#!/bin/sh
# Regenerates expected/long_reference_lines.json, the recorded reference output of the command lines the long-read tests run
# (tests/test_gpu_long_reads.py and tests/test_emu_long_reads.py, inputs from tests/long_reads.py), as digests in the form
# tests/oracle_lib.py:reference_lines stores them. The tests are run once with MM2_RECORD_REFERENCE set, which makes them run the
# reference build (oracle/_ref, from `make -C oracle ref`) on the same inputs and record its output; the comparisons with this
# library then fail without a CUDA device (GPU file) or are skipped, after recording.
set -e
cd "$(dirname "$0")/../.."
out=${TMPDIR:-/tmp}/long_reference_lines.$$.json
rm -f "$out"
MM2_RECORD_REFERENCE=$out python -m pytest -q -m gpu -k cli tests/test_gpu_long_reads.py || true
MM2_RECORD_REFERENCE=$out python -m pytest -q -k cli tests/test_emu_long_reads.py || true
mv "$out" tests/golden/expected/long_reference_lines.json
