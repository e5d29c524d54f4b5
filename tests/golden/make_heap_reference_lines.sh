#!/bin/sh
# Regenerates expected/heap_reference_lines.json, the recorded reference output of the command lines the heap-ordered seeding tests
# run (tests/test_oracle_heap_seed.py: --print-seeds dumps; tests/test_gpu_heap_seed.py: CLI output), as digests in the form
# tests/oracle_lib.py:reference_lines stores them. The tests are run once with MM2_RECORD_REFERENCE set, which makes them run the
# reference build (oracle/_ref, from `make -C oracle ref`) on the same inputs and record its output; the GPU file's comparisons with
# this library then fail without a CUDA device, after recording.
set -e
cd "$(dirname "$0")/../.."
out=${TMPDIR:-/tmp}/heap_reference_lines.$$.json
rm -f "$out"
MM2_RECORD_REFERENCE=$out python -m pytest -q tests/test_oracle_heap_seed.py
MM2_RECORD_REFERENCE=$out python -m pytest -q -m gpu -k cli tests/test_gpu_heap_seed.py || true
mv "$out" tests/golden/expected/heap_reference_lines.json
