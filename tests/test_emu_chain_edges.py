"""CPU: a reduced set of tests/test_gpu_chain_edges.py -- the chaining kernels (unmodified CUDA sources under the SIMT emulator of
tests/cuda_emu) against the reference chainers at their parameter edges, on one mixed batch of every read shape of
tests/chain_cases.py except the reads of more than 10^5 anchors."""
import ctypes as C
import os
import sys
import numpy as np
import pytest
import oracle_lib as O
import chain_cases as CC

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))
sys.path.insert(0, O.ROOT)


@pytest.fixture(scope="module")
def emu():
    import build_emu
    L = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    L.mmb_ctx_create.restype = C.c_void_p
    return L, C.c_void_p(L.mmb_ctx_create(0))


@pytest.fixture(scope="module")
def reads():
    return CC.read_mix(np.random.default_rng(7), n_noisy=4, scale=0.4)


def call(emu, fn, reads, par, *extra):
    """fn over the batch through the host-buffer entry; extra: arguments between par and n_reads (the rescue's), then qlen after a_off"""
    L, ctx = emu
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    for i, a in enumerate(reads):
        off[i + 1] = off[i] + len(a)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in reads]))
    n = len(reads)
    n_u, n_v = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    u, ao = np.zeros(int(off[-1]) + 1, dtype=np.uint64), np.zeros((int(off[-1]) + 1, 2), dtype=np.uint64)
    ptr = lambda x: C.c_void_p(x.ctypes.data)
    if extra:
        r, ql = extra
        getattr(L, fn)(ctx, C.byref(par), C.byref(r), n, ptr(cat), ptr(off), ptr(np.ascontiguousarray(ql, dtype=np.int32)),
                       ptr(n_u), ptr(n_v), ptr(u), ptr(ao))
    else:
        getattr(L, fn)(ctx, C.byref(par), n, ptr(cat), ptr(off), ptr(n_u), ptr(n_v), ptr(u), ptr(ao))
    return [(u[int(off[i]):int(off[i]) + n_u[i]].copy(), ao[int(off[i]):int(off[i]) + n_v[i]].copy()) for i in range(n)]


DP = [CC.dp_par(max_iter=m) for m in (-1, 0, 33)] + \
    [CC.dp_par(max_skip=0, max_iter=1), CC.dp_par(max_skip=32, bw=20, pen_skip=CC.pen(3)),
     CC.dp_par(max_dist_x=300, max_dist_y=300, bw=300, max_iter=2, min_cnt=2, min_sc=20),
     CC.dp_par(max_dist_x=30, max_dist_y=30, bw=50), CC.dp_par(max_dist_x=200000, max_dist_y=100, bw=500, is_cdna=1, min_sc=20)]


@pytest.mark.parametrize("i", range(len(DP)))
def test_emulated_chain_dp_edges(emu, reads, i):
    p = DP[i]
    got = call(emu, "mmb_chain_batch_host", reads, CC.chain_par(p))
    assert CC.check_all(got, reads, lambda a: CC.expect_dp(a, p), str(p)) > 0


RMQ = [CC.rmq_par(cap=12, max_dist_inner=-5), CC.rmq_par(max_dist_inner=20000, max_skip=0, pen_skip=CC.pen(1))]


@pytest.mark.parametrize("i", range(len(RMQ)))
def test_emulated_chain_rmq_edges(emu, reads, i):
    p = RMQ[i]
    rs = [CC.y_zero(a) for a in reads]
    got = call(emu, "mmb_chain_rmq_batch_host", rs, CC.chain_par(p))
    assert CC.check_all(got, rs, lambda a: CC.expect_rmq(a, p), str(p)) > 0


RESCUES = [(CC.dp_par(max_iter=0), dict(bw_long=20000, rescue_size=1000, rescue_ratio=2.0, max_dist=5000, max_dist_inner=1000, cap=100000)),
           (CC.rmq_par(), dict(bw_long=20000, rescue_size=1000, rescue_ratio=0.3, max_dist=5000, max_dist_inner=0, cap=64))]


@pytest.mark.parametrize("i", range(len(RESCUES)))
def test_emulated_chain_rescue(emu, reads, i):
    p, r = RESCUES[i]
    rng = np.random.default_rng(31 + i)
    rs = reads + [CC.tandem(rng, copies=3, n=120) for _ in range(4)]
    ql = CC.rescue_qlens(rng, rs, p, r)
    got = call(emu, "mmb_chain_rescue_batch_host", rs, CC.chain_par(p), CC.rescue_par(r), ql)
    n_rescued = 0
    for k, a in enumerate(rs):
        u, b, rescued = CC.expect_rescue(a, ql[k], p, r)
        CC.assert_same(got[k], (u, b), "rescue %d read %d (qlen %d, rescued %d)" % (i, k, ql[k], rescued))
        n_rescued += rescued
    assert 0 < n_rescued < len(rs)
