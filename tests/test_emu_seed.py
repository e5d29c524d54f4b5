"""CPU: the seeding-stage kernels (mzflt / lookup / select / expand / sort_radix / sort_exact_*), unmodified CUDA sources under the SIMT
emulator, against the oracle (see tests/seed_check.py)."""
import ctypes as C
import os
import sys
import pytest
import oracle_lib as O
import seed_check as SC

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))


@pytest.fixture(scope="module")
def emu():
    import build_emu
    L = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    L.mmb_ctx_create.restype = C.c_void_p
    SC.setup(L)
    return L, C.c_void_p(L.mmb_ctx_create(0))


@pytest.mark.parametrize("cfg", [dict(), dict(mid_occ=4, occ_dist=100), dict(mid_occ=6, occ_dist=0), dict(flag=0x100000), dict(w=5, mid_occ=8, q_occ_frac=0.0)])
def test_emulated_seed_stage_matches_oracle(emu, cfg):
    L, ctx = emu
    contigs, reads = SC.repeat_rich_case(3, 60_000, 5, 1500, rep=0.5)
    st = SC.check_case(L, ctx, contigs, reads, **cfg)
    assert st["anchors"] > 500 and st["big"] >= 3


def test_emulated_seed_stage_sort_ties(emu):
    """many equal sort keys in reads with more than 64 anchors: the stable radix order is detected as tied and redone by the exact
    emulation of the reference's unstable sort"""
    L, ctx = emu
    contigs, reads = SC.repeat_rich_case(8, 30_000, 3, 2500, rep=0.8, n_contigs=1)
    st = SC.check_case(L, ctx, contigs, reads, mid_occ=50, max_max_occ=400, occ_dist=50)
    assert st["ties"] >= 1


def test_emulated_seed_stage_long_reads(emu):
    """reads with more than SEL_CAP (2048) minimizers after the query-side filter: select_kernel keeps their seeds in global memory"""
    L, ctx = emu
    contigs, reads = SC.repeat_rich_case(4, 60_000, 4, 8000, rep=0.5)
    cfg = dict(w=5, mid_occ=8, q_occ_frac=0.01)
    assert max(SC.n_minimizers(r, cfg["w"], 15, cfg["mid_occ"], cfg["q_occ_frac"]) for r in reads) > 2048
    st = SC.check_case(L, ctx, contigs, reads, **cfg)
    assert st["anchors"] > 500 and st["big"] >= 3


def test_emulated_seed_stage_capacity_edges(emu):
    """2048 / 2049 minimizers in both query-side filter kernels and in select_kernel, q_occ_max / q_occ_max + 1 minimizers, and streaks
    at the 128-entry heap's cap (see seed_check.check_edges)"""
    L, ctx = emu
    SC.check_edges(L, ctx)
