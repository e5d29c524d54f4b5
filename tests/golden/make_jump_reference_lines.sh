#!/bin/sh
# Regenerates expected/jump_reference_lines.json, the recorded reference output of the command lines tests/test_gpu_jump.py runs
# (digests as tests/oracle_lib.py:reference_lines stores them). The test file is run once with MM2_RECORD_REFERENCE set, which makes
# it run the reference build (oracle/_ref, from `make -C oracle ref`) on the same inputs and record its output. The --pass1 input is
# this library's own --write-junc output, so the run needs a CUDA device.
set -e
cd "$(dirname "$0")/../.."
out=${TMPDIR:-/tmp}/jump_reference_lines.$$.json
rm -f "$out"
MM2_RECORD_REFERENCE=$out python -m pytest -q tests/test_gpu_jump.py
mv "$out" tests/golden/expected/jump_reference_lines.json
