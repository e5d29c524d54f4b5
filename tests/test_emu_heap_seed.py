"""CPU: heap-ordered seeding (MM_F_HEAP_SORT) through the kernel-level entry mmb_seed_batch_host, the unmodified CUDA sources under the
SIMT emulator, against the restatement of the heap merge (tests/heap_cases.py:HeapOracle, pinned to the reference by
tests/test_oracle_heap_seed.py). The
reads with equal keys are replayed by heap_merge_kernel: with its heap in shared memory, in the global-memory fallback, and for an
oversize read."""
import ctypes as C
import os
import sys
import pytest
import oracle_lib as O
import seed_check as SC
import heap_cases as H

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))


@pytest.fixture(scope="module")
def emu():
    import build_emu
    L = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    L.mmb_ctx_create.restype = C.c_void_p
    SC.setup(L)
    return L, C.c_void_p(L.mmb_ctx_create(0))


def _case():
    contigs, reads = H.mixed_case(21, 60_000, 6, 2500, 40, rep=0.6, n_contigs=2)
    big_ctg, big_read = H.oversize_case()
    return contigs + [big_ctg], reads + [big_read]


@pytest.mark.parametrize("cfg", [dict(mid_occ=30), dict(mid_occ=30, occ_dist=100), dict(mid_occ=30, flag=0x100000), dict(mid_occ=30, flag=0x200000)])
def test_emulated_heap_seed_matches_oracle(emu, cfg):
    L, ctx = emu
    contigs, reads = _case()
    kw = dict(cfg, flag=cfg.get("flag", 0) | H.HEAP)
    H.check_device(L, ctx, contigs, reads, **cfg)
    idx = H.HeapOracle([bytes(c) for c in contigs], ["chr%d" % i for i in range(len(contigs))], 10, 15)
    oracle_kw = dict(kw, flag=kw["flag"] & ~H.HEAP)
    pc = H.path_counts(idx, reads, oracle_kw)
    st = H.tie_stats(idx, [bytes(r) for r in reads], [None] * len(reads), 10, 15, oracle_kw)
    idx.close()
    assert pc["smem"] >= 1 and pc["global_"] >= 1 and pc["oversize"] == 1, pc
    strands = "+" if kw["flag"] & 0x100000 else "-" if kw["flag"] & 0x200000 else "+-"
    H.assert_covered(st, strands=strands, skip=bool(kw["flag"] & H.SKIP))


def test_emulated_heap_flag_off_is_default(emu):
    """without the flag the same batch gives the sorted order (the default path is unchanged)"""
    L, ctx = emu
    contigs, reads = _case()
    SC.check_case(L, ctx, contigs, reads, mid_occ=30)
