"""CPU: a reduced set of tests/test_gpu_index.py -- the index build (sketch kernels on the packed S, CUB sort and run-length
encoding, the open-addressing table, the sorted counts behind mm_idx_cal_max_occ), mm_idx_dump / mm_idx_load and the device probe,
unmodified CUDA sources under the SIMT emulator of tests/cuda_emu, against the oracle on every build path of tests/index_cases.py."""
import ctypes as C
import os
import sys
import numpy as np
import pytest
import oracle_lib as O
import index_cases as IC
import seed_check as SC

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))
sys.path.insert(0, O.ROOT)


@pytest.fixture(scope="module")
def emu():
    import build_emu
    L = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    L.mmb_ctx_create.restype = C.c_void_p
    IC.setup(L)
    SC.setup(L)
    return L, C.c_void_p(L.mmb_ctx_create(0))


@pytest.mark.parametrize("p", IC.PARAMS, ids=IC.PARAM_IDS)
def test_emulated_index_build_matches_oracle(emu, p, tmp_path):
    w, k, is_hpc = p
    L, _ = emu
    exp, wrapped = IC.check_device_index(L, IC.contigs(w, k, is_hpc, 5, scale=0.1), w, k, is_hpc, tmp_path)
    assert int(exp.cnt.max()) >= 300
    assert wrapped == IC.wraps(exp.keys, k)


def test_some_cases_probe_across_the_table_end():
    """in several cases (reduced and full size) the table's last slot is filled and absent keys homed there probe on from slot 0"""
    for seed, scale in ((5, 0.1), (11, 1.0)):
        n = sum(IC.wraps(IC.oracle_canon(IC.contigs(w, k, h, seed, scale), w, k, h).keys, k) for w, k, h in IC.PARAMS)
        assert n >= 3, (seed, scale, n)


@pytest.mark.parametrize("fx", IC.REF_MMI, ids=[f[0] for f in IC.REF_MMI])
def test_emulated_load_of_reference_mmi(emu, fx, tmp_path):
    """a .mmi the reference wrote (HPC; even k with b = 2k < 14) loads and probes as the oracle's index of the same sequence"""
    IC.check_reference_mmi(emu[0], *fx, tmp_path)


@pytest.mark.parametrize("p", IC.PARTS_PARAMS)
def test_emulated_index_parts_match_reference(emu, p, tmp_path):
    """-I: mm_idx_reader_read's parts (idx_gen's mini-batch rule) against the reference's recorded parts"""
    IC.check_parts(emu[0], *p, tmp_path)


def test_emulated_hpc_seed_stage_matches_oracle(emu):
    """the seeding stage with an HPC index: seed spans differ from k in the query sketch, the lookups and the anchors"""
    L, ctx = emu
    contigs, reads = SC.repeat_rich_case(6, 40_000, 4, 1500, rep=0.5)
    rng = np.random.default_rng(6)
    reads.append(IC._hpc_runs(rng, 600, 40))
    contigs.append(np.frombuffer(IC._hpc_runs(rng, 4000, 40) + reads[-1], dtype=np.uint8))
    st = SC.check_case(L, ctx, contigs, reads, w=10, k=19, is_hpc=1)
    assert st["anchors"] > 300
