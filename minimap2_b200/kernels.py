"""Kernel-level host-buffer entry points (the C-ABI calls in include/mm_b200.h), used by the parity tests."""
import ctypes as C
import numpy as np
from ._lib import lib, KswJob, KswRes, KswScore, ChainPar, RescuePar


def make_score(mat, q, e, q2, e2, noncan=0, junc_bonus=0, junc_pen=0, zd_skip=0):
    sc = KswScore()
    for i in range(25):
        sc.mat[i] = int(mat[i])
    sc.q, sc.e, sc.q2, sc.e2 = q, e, q2, e2
    sc.noncan, sc.junc_bonus, sc.junc_pen = noncan, junc_bonus, junc_pen
    sc.zd_skip = zd_skip
    return sc


def ksw_batch(ctx, score, pairs, params):
    """pairs: list of (q, t) uint8 nt4 arrays; params: list of dict(w, zdrop, end_bonus, flag).
    Returns a list of dicts shaped like the oracle's (tests/oracle_lib.ez_dict)."""
    n = len(pairs)
    if n == 0:
        return []
    qcat = np.concatenate([np.asarray(p[0], dtype=np.uint8) for p in pairs])
    tcat = np.concatenate([np.asarray(p[1], dtype=np.uint8) for p in pairs])
    jobs = (KswJob * n)()
    qo = to = 0
    tot = 0
    for i, ((q, t), pr) in enumerate(zip(pairs, params)):
        j = jobs[i]
        j.q_start, j.t_start, j.q_step, j.t_step = qo, to, 1, 1
        j.qlen, j.tlen = len(q), len(t)
        j.w, j.zdrop, j.end_bonus, j.flag = pr["w"], pr["zdrop"], pr["end_bonus"], pr["flag"]
        qo += len(q); to += len(t); tot += len(q) + len(t) + 2
    res = (KswRes * n)()
    cig = np.zeros(tot, dtype=np.uint32)
    used = lib().mmb_ksw_batch_host(ctx.h, C.byref(score), n, jobs, qcat.ctypes.data, len(qcat), tcat.ctypes.data, len(tcat),
                                    res, cig.ctypes.data, len(cig))
    assert used >= 0, used
    out = []
    for i in range(n):
        r = res[i]
        out.append(dict(max=r.max, zdropped=r.zdropped, max_q=r.max_q, max_t=r.max_t, mqe=r.mqe, mqe_t=r.mqe_t, mte=r.mte,
                        mte_q=r.mte_q, score=r.score, n_cigar=r.n_cigar, reach_end=r.reach_end,
                        cigar=[int(x) for x in cig[r.cigar_off:r.cigar_off + r.n_cigar]]))
    return out


def sketch_batch(ctx, seqs, w, k, is_hpc=0, rid0=0):
    """seqs: list of bytes. Returns a list of (n_i, 2) uint64 arrays (x, y) like mm_sketch's mm128_t output."""
    n = len(seqs)
    off = np.zeros(n + 1, dtype=np.int64)
    for i, s in enumerate(seqs):
        off[i + 1] = off[i] + len(s)
    cat = b"".join(seqs)
    buf = np.frombuffer(cat, dtype=np.uint8)
    n_out = np.zeros(n, dtype=np.int64)
    cap = max(int(off[-1]), 1)
    out = np.zeros((cap, 2), dtype=np.uint64)
    tot = lib().mmb_sketch_batch_host(ctx.h, n, buf.ctypes.data, off.ctypes.data, w, k, is_hpc, rid0, out.ctypes.data, cap, n_out.ctypes.data)
    assert tot <= cap
    res, o = [], 0
    for i in range(n):
        res.append(out[o:o + n_out[i]].copy()); o += int(n_out[i])
    assert o == tot
    return res


def _chain_io(anchor_arrays):
    """concatenated anchors, offsets and output buffers of the chaining entries"""
    n = len(anchor_arrays)
    off = np.zeros(n + 1, dtype=np.int64)
    for i, a in enumerate(anchor_arrays):
        off[i + 1] = off[i] + len(a)
    tot = int(off[-1])
    cat = np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in anchor_arrays]) if tot else np.zeros((0, 2), dtype=np.uint64)
    cat = np.ascontiguousarray(cat)
    n_u = np.zeros(n, dtype=np.int32); n_v = np.zeros(n, dtype=np.int32)
    u = np.zeros(tot + 1, dtype=np.uint64); ao = np.zeros((tot + 1, 2), dtype=np.uint64)
    return off, cat, n_u, n_v, u, ao


def _chain_out(off, n_u, n_v, u, ao):
    return [(u[int(off[i]):int(off[i]) + n_u[i]].copy(), ao[int(off[i]):int(off[i]) + n_v[i]].copy()) for i in range(len(n_u))]


def chain_batch(ctx, anchor_arrays, max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc, pen_gap, pen_skip=0.0, is_cdna=0, n_seg=1):
    """anchor_arrays: list of (n_i,2) uint64 arrays sorted by x. Returns list of (u, a) like mg_lchain_dp."""
    off, cat, n_u, n_v, u, ao = _chain_io(anchor_arrays)
    par = ChainPar(max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc, pen_gap, pen_skip, is_cdna, n_seg, 0, 0, 0)
    lib().mmb_chain_batch_host(ctx.h, C.byref(par), len(n_u), cat.ctypes.data, off.ctypes.data, n_u.ctypes.data, n_v.ctypes.data, u.ctypes.data, ao.ctypes.data)
    return _chain_out(off, n_u, n_v, u, ao)


def chain_rmq_batch(ctx, anchor_arrays, max_dist, max_dist_inner, bw, max_skip, cap, min_cnt, min_sc, pen_gap, pen_skip=0.0):
    """mg_lchain_rmq on every read (anchors sorted by x). Returns list of (u, a)."""
    off, cat, n_u, n_v, u, ao = _chain_io(anchor_arrays)
    par = ChainPar(max_dist, max_dist, bw, max_skip, 5000, min_cnt, min_sc, pen_gap, pen_skip, 0, 1, 1, max_dist_inner, cap)
    lib().mmb_chain_rmq_batch_host(ctx.h, C.byref(par), len(n_u), cat.ctypes.data, off.ctypes.data, n_u.ctypes.data, n_v.ctypes.data, u.ctypes.data, ao.ctypes.data)
    return _chain_out(off, n_u, n_v, u, ao)


def chain_rescue_batch(ctx, anchor_arrays, qlens, par, rescue):
    """The mapper's chaining stage (map.c:262-292) on every read: the first chainer that par (a ChainPar; use_rmq selects
    mg_lchain_rmq) describes, then the long-join rescue (a RescuePar) of the reads it selects by their query length qlens[i].
    Returns list of (u, a)."""
    off, cat, n_u, n_v, u, ao = _chain_io(anchor_arrays)
    ql = np.ascontiguousarray(qlens, dtype=np.int32)
    assert len(ql) == len(n_u)
    lib().mmb_chain_rescue_batch_host(ctx.h, C.byref(par), C.byref(rescue), len(n_u), cat.ctypes.data, off.ctypes.data, ql.ctypes.data,
                                      n_u.ctypes.data, n_v.ctypes.data, u.ctypes.data, ao.ctypes.data)
    return _chain_out(off, n_u, n_v, u, ao)


def idx_lookup(idx, keys, L=None):
    """The device hash table of idx (an mm_idx_t pointer) probed for every key, as the seeding kernels probe it. Returns (cnt, occ_off,
    occ): occurrences of keys[i] (0: absent) and their words occ[occ_off[i]:occ_off[i + 1]], in stored order. L: the library to call
    (default: this package's)."""
    L = L or lib()
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    n = len(keys)
    cnt, occ_off = np.zeros(max(n, 1), dtype=np.uint32), np.zeros(n + 1, dtype=np.int64)
    occ = np.zeros(1, dtype=np.uint64)
    for _ in range(2):  # the second call when the first capacity was too small
        tot = L.mmb_idx_lookup_host(C.c_void_p(idx), C.c_int64(n), C.c_void_p(keys.ctypes.data), C.c_void_p(cnt.ctypes.data),
                                    C.c_void_p(occ.ctypes.data), C.c_int64(len(occ)), C.c_void_p(occ_off.ctypes.data))
        if tot <= len(occ):
            break
        occ = np.zeros(tot, dtype=np.uint64)
    return cnt[:n], occ_off, occ[:tot]


SORT_ROUTE_NONE, SORT_ROUTE_OVERSIZE, SORT_ROUTE_NETWORK, SORT_ROUTE_EXACT, SORT_ROUTE_GLOBAL = -1, 5, 8, 16, 32  # MMB_SORT_ROUTE_*


def anchor_sort_batch(ctx, arrays, L=None):
    """The seeding stage's anchor sort (radix_sort_128x) on every read. arrays: list of (n_i, 2) uint64 anchor arrays. Returns (sorted
    arrays, routes): routes[i] is read i's path through the sort kernels (MMB_SORT_ROUTE_* in include/mm_b200.h). ctx: a Context or a
    context handle; L: the library to call (default: this package's; declare_anchor_sort() gives another one the argtypes)."""
    n = len(arrays)
    off = np.zeros(n + 1, dtype=np.int64)
    for i, a in enumerate(arrays):
        off[i + 1] = off[i] + len(a)
    tot = int(off[-1])
    cat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in arrays]) if tot else np.zeros((1, 2), dtype=np.uint64))
    out = np.zeros((max(tot, 1), 2), dtype=np.uint64)
    route = np.zeros(max(n, 1), dtype=np.int32)
    got = (L or lib()).mmb_anchor_sort_host(getattr(ctx, "h", ctx), n, cat.ctypes.data, off.ctypes.data, out.ctypes.data, route.ctypes.data)
    assert got == tot, (got, tot)
    return [out[int(off[i]):int(off[i + 1])].copy() for i in range(n)], route[:n]


class JumpHit(C.Structure):  # mmb_jump_hit_t (include/mm_b200.h)
    _fields_ = [("rid", C.c_int32), ("rs", C.c_int32), ("re", C.c_int32), ("qs", C.c_int32), ("qe", C.c_int32), ("rev", C.c_int32),
                ("qlen", C.c_int32), ("n_cigar", C.c_int32), ("q_off", C.c_int64), ("cig_first", C.c_uint32), ("cig_last", C.c_uint32)]


class JumpSide(C.Structure):  # mmb_jump_side_t
    _fields_ = [("act", C.c_int32), ("l", C.c_int32), ("off", C.c_int32), ("off2", C.c_int32), ("mm0", C.c_int32)]


class JumpDec(C.Structure):  # mmb_jump_dec_t
    _fields_ = [("side", JumpSide * 2)]


def jump_batch(ctx, idx, map_opt, reads, hits, L=None):
    """K5 (junction jumps) on the device. idx: mm_idx_t pointer with a jump table (mm_idx_jjump_read); map_opt: MapOpt (a, b,
    jump_min_match); reads: list of bytes (ASCII); hits: list of dicts with read (index into reads), rid, rs, re, qs, qe, rev and cigar
    (list of uint32 words). Returns one ((act, l, off, off2, mm0) left, (...) right) pair per hit. L: the library to call (default:
    this package's)."""
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    for i, s in enumerate(reads):
        off[i + 1] = off[i] + len(s)
    buf = np.frombuffer(b"".join(reads) + b"\0", dtype=np.uint8)
    n = len(hits)
    h = (JumpHit * max(n, 1))()
    for i, x in enumerate(hits):
        e = h[i]
        e.rid, e.rs, e.re, e.qs, e.qe, e.rev = x["rid"], x["rs"], x["re"], x["qs"], x["qe"], x["rev"]
        e.qlen, e.n_cigar, e.q_off = len(reads[x["read"]]), len(x["cigar"]), int(off[x["read"]])
        e.cig_first, e.cig_last = x["cigar"][0], x["cigar"][-1]
    out = (JumpDec * max(n, 1))()
    ret = (L or lib()).mmb_jump_batch_host(C.c_void_p(ctx.h), idx, C.byref(map_opt), len(reads), C.c_void_p(buf.ctypes.data),
                                    C.c_void_p(off.ctypes.data), n, h, out)
    assert ret == 0, "mmb_jump_batch_host: the index has no jump table"
    return [tuple((s.act, s.l, s.off, s.off2, s.mm0) for s in out[i].side) for i in range(n)]
