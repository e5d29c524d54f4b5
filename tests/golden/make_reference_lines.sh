#!/bin/sh
# Regenerates the recorded reference outputs that the parity tests compare against:
#  * expected/reference_lines.json -- digests of what the reference binary prints for every command line those tests run
#    (tests/oracle_lib.py:reference_lines);
#  * expected/reference_values.json -- results of reference library calls (tests/oracle_lib.py:reference_values);
#  * data/MT-human.mmi.gz -- the reference's index file of data/MT-human.fa.
# The tests are run once with MM2_RECORD_REFERENCE set, which makes them call the reference build (oracle/_ref, from
# `make -C oracle ref`) on the same inputs and record its results. Needs that build and a CUDA device.
set -e
cd "$(dirname "$0")/../.."
out=${TMPDIR:-/tmp}/reference_lines.$$.json
rm -f "$out" "$out.values.json"
MM2_RECORD_REFERENCE=$out python -m pytest -q tests/test_emu_e2e.py tests/test_emu_api.py tests/test_oracle_seed.py \
    tests/test_gpu_e2e.py tests/test_gpu_zz_splice.py tests/test_gpuext_options.py tests/test_gpu_chain_cli.py tests/test_index_cases_vs_ref.py tests/test_gpu_index_cli.py
mv "$out" tests/golden/expected/reference_lines.json
mv "$out.values.json" tests/golden/expected/reference_values.json
oracle/_ref/minimap2 -t 2 -d tests/golden/data/MT-human.mmi tests/golden/data/MT-human.fa
gzip -9 -n -f tests/golden/data/MT-human.mmi
# an HPC index and an even-k index with b = 2k < 14 (tests/index_cases.py: REF_MMI)
oracle/_ref/minimap2 -t 2 -H -w 10 -k 19 -d tests/golden/data/MT-human.H.w10k19.mmi tests/golden/data/MT-human.fa
oracle/_ref/minimap2 -t 2 -w 4 -k 6 -d tests/golden/data/MT-human.w4k6.mmi tests/golden/data/MT-human.fa
gzip -9 -n -f tests/golden/data/MT-human.H.w10k19.mmi tests/golden/data/MT-human.w4k6.mmi
