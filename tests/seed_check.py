"""Shared checker of the seeding stage (K1 sketch -> query-side filter -> index lookup -> streak selection -> anchor expansion -> anchor
sort) through the kernel-level C entry mmb_seed_batch_host, against the oracle restatement (oracle/mm2o_seed.c, itself pinned to the
reference's --print-seeds dump in tests/test_oracle_seed.py): sorted anchors incl. the tie order of the unstable radix sort, rep_len
and the kept seeds' mini_pos words. Used by tests/test_emu_seed.py (CPU, SIMT emulator) and tests/test_gpu_seed.py (GPU)."""
import ctypes as C
import numpy as np
import oracle_lib as O
import synth


def setup(L):
    L.mm_idx_str.restype = C.c_void_p
    L.mm_idx_str.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
    L.mm_idx_destroy.argtypes = [C.c_void_p]
    L.mmb_seed_batch_host.restype = C.c_int64
    L.mmb_seed_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]


def device_seeds(L, ctx, mi, reads, flag, mid_occ, q_occ_frac, max_max_occ, occ_dist):
    n = len(reads)
    off = np.zeros(n + 1, dtype=np.int64)
    for i, s in enumerate(reads):
        off[i + 1] = off[i] + len(s)
    buf = np.frombuffer(b"".join(reads) + b"\0", dtype=np.uint8)
    a_off = np.zeros(n + 1, dtype=np.int64); rep = np.zeros(n, dtype=np.int32); nmini = np.zeros(n, dtype=np.int32)
    a_cap = 4_000_000
    a = np.zeros((a_cap, 2), dtype=np.uint64); mp = np.zeros(int(off[-1]) + 16, dtype=np.uint64)
    tot = L.mmb_seed_batch_host(ctx, mi, n, buf.ctypes.data, off.ctypes.data, flag, mid_occ, q_occ_frac, max_max_occ, occ_dist,
                                a_off.ctypes.data, rep.ctypes.data, nmini.ctypes.data, a.ctypes.data, a_cap, mp.ctypes.data, len(mp))
    assert tot >= 0 and tot == a_off[-1]
    out, o = [], 0
    for i in range(n):
        out.append((a[int(a_off[i]):int(a_off[i + 1])].copy(), int(rep[i]), mp[o:o + int(nmini[i])].copy()))
        o += int(nmini[i])
    return out


def check_case(L, ctx, contigs, reads, w=10, k=15, flag=0, mid_occ=10, q_occ_frac=0.01, max_max_occ=4095, occ_dist=500, is_hpc=0):
    names = ["chr%d" % i for i in range(len(contigs))]
    seqs = [bytes(c) for c in contigs]
    arr = (C.c_char_p * len(seqs))(*seqs); nm = (C.c_char_p * len(seqs))(*[x.encode() for x in names])
    mi = L.mm_idx_str(w, k, is_hpc, 14, len(seqs), arr, nm)
    reads = [bytes(r) for r in reads]
    got = device_seeds(L, ctx, mi, reads, flag, mid_occ, q_occ_frac, max_max_occ, occ_dist)
    idx = O.OracleIndex(seqs, names, w, k, is_hpc)
    stats = dict(anchors=0, ties=0, big=0, wide=0)
    for i, s in enumerate(reads):
        ea, erep, emp = idx.anchors(s, flag=flag, mid_occ=mid_occ, q_occ_frac=q_occ_frac, max_max_occ=max_max_occ, occ_dist=occ_dist) if len(s) else (np.zeros((0, 2), dtype=np.uint64), 0, np.zeros(0, dtype=np.uint64))
        ga, grep_, gmp = got[i]
        assert grep_ == erep, (i, grep_, erep)
        assert len(gmp) == len(emp) and (gmp == emp).all(), (i, len(gmp), len(emp))
        assert ga.shape == ea.shape, (i, ga.shape, ea.shape)
        assert (ga == ea).all(), (i, int(np.argmax((ga != ea).any(axis=1))))
        stats["anchors"] += len(ea)
        if len(ga):  # sort keys that differ in more than 33 bit positions: the radix kernels leave such reads to sort_block_kernel
            stats["wide"] += int(bin(int(np.bitwise_or.reduce(ga[:, 0] ^ ga[0, 0]))).count("1") > 33)
        if len(ea) > 64:
            stats["big"] += 1
            stats["ties"] += int((ea[1:, 0] == ea[:-1, 0]).any())
    idx.close()
    L.mm_idx_destroy(mi)
    return stats


def n_minimizers(seq, w, k, q_occ_max, q_occ_frac):
    """minimizers of a read after the query-side filter (mm_seed_mz_flt, seed.c:5-28), from the oracle's sketch"""
    x = O.oracle_sketch(bytes(seq), w, k)[:, 0]
    n = len(x)
    if n <= q_occ_max or q_occ_frac <= 0 or q_occ_max <= 0:
        return n
    _, inv, cnt = np.unique(x, return_inverse=True, return_counts=True)
    c = cnt[inv]
    return int((~(((c > q_occ_max) & (c > np.float32(n) * np.float32(q_occ_frac))) | (x == 0))).sum())


def repeat_rich_case(seed, glen, n_reads, rlen, rep=0.4, n_contigs=2):
    """genome with copied segments (several query minimizers hit the same reference position => equal sort keys, long occurrence lists,
    high-occurrence streaks) and reads with errors, some chimeric, one made of tandem copies"""
    contigs = synth.random_genome(glen, seed, n_contigs=n_contigs, repeat_frac=rep)
    reads = synth.make_reads(contigs, n_reads, rlen, 0.08, seed + 50, chimeric_frac=0.1)
    reads.append(bytes(contigs[0][500:900]) * 5)
    reads.append(b"ACGT")
    return contigs, reads


def n_sketch(seq, w, k):
    """minimizers of a read before the query-side filter"""
    return len(O.oracle_sketch(bytes(seq), w, k))


def trim_to_count(seq, target, count):
    """the shortest prefix of seq with count(prefix) == target minimizers (count: n_sketch or n_minimizers with their parameters bound)"""
    lo, hi = 0, len(seq)
    assert count(seq) >= target, (count(seq), target)
    while lo < hi:  # the shortest prefix with at least target
        mid = (lo + hi) // 2
        if count(seq[:mid]) >= target:
            hi = mid
        else:
            lo = mid + 1
    for ln in range(lo, min(len(seq), lo + 64) + 1):
        if count(seq[:ln]) == target:
            return bytes(seq[:ln])
    raise ValueError("no prefix with %d minimizers" % target)


def read_counts(seq, w, k):
    """how often each minimizer of the read occurs in it (what mm_seed_mz_flt compares with q_occ_max and n * q_occ_frac)"""
    _, cnt = np.unique(O.oracle_sketch(bytes(seq), w, k)[:, 0], return_counts=True)
    return cnt


def streaks(seq, contigs, w, k, max_occ, occ_dist):
    """mm_seed_select's stretches of seeds with more than max_occ occurrences (seed.c:56-96), from the oracle's sketches: per stretch,
    (its number of seeds, max_high_occ = (pe - ps) / occ_dist + .499) before the 128-entry cap"""
    occ = {}
    for c in contigs:
        for x in O.oracle_sketch(bytes(c), w, k)[:, 0] >> np.uint64(8):
            occ[int(x)] = occ.get(int(x), 0) + 1
    mz = O.oracle_sketch(bytes(seq), w, k)
    seeds = [(int(y & np.uint64(0xffffffff)) >> 1, occ[int(x >> np.uint64(8))]) for x, y in mz if int(x >> np.uint64(8)) in occ]
    out, last0 = [], -1
    for i in range(len(seeds) + 1):
        if i == len(seeds) or seeds[i][1] <= max_occ:
            if i - last0 > 1:
                ps = 0 if last0 < 0 else seeds[last0][0]
                pe = len(seq) if i == len(seeds) else seeds[i][0]
                out.append((i - last0 - 1, int((pe - ps) / occ_dist + .499)))
            last0 = i
    return out


def edge_genome(seed):
    """a random genome with a 2 kb segment copied 20 times (seeds with 20 occurrences: high-occurrence stretches) and tandem arrays of a
    40-bp, a 37-bp and a 7-bp unit (minimizers that occur many times in one read)"""
    rng = np.random.default_rng(seed)
    rnd = lambda n: bytes(synth.ALPHA[rng.integers(0, 4, n)])
    rep, u40, u37, u7 = rnd(2000), rnd(40), rnd(37), b"ACGGTCA"
    ctg0 = b"".join(rnd(3000) + rep for _ in range(20)) + rnd(3000)
    ctg1 = rnd(20_000) + u40 * 40 + rnd(500) + u37 * 11 + rnd(500) + u7 * 12 + rnd(20_000)
    return [ctg0, ctg1], dict(rep=rep, u40=u40, u37=u37, u7=u7, flank=ctg1[:20_000], rnd=rnd)


def mzflt_edge_reads(parts, w=10, k=15, q_occ_max=10):
    """reads of exactly 2048 and 2049 minimizers before the query-side filter (mzflt_smem_kernel / mzflt_kernel), each opening with
    tandem arrays whose minimizers occur q_occ_max times and more in the read; reads of q_occ_max and q_occ_max + 1 minimizers of one
    7-bp unit (the filter's n <= q_occ_max exit)"""
    body = parts["u37"] * 11 + parts["u40"] * 40 + parts["flank"] + parts["rnd"](20_000)
    out = [trim_to_count(body, n, lambda s: n_sketch(s, w, k)) for n in (2048, 2049)]
    out += [trim_to_count(parts["u7"] * 40, n, lambda s: n_sketch(s, w, k)) for n in (q_occ_max, q_occ_max + 1)]
    return out


def select_edge_reads(parts, w=10, k=15):
    """reads of exactly 2048 and 2049 minimizers (SEL_CAP: select_kernel's shared or global seed tables) that open with copies of the
    repeated segment, so streak selection has stretches of high-occurrence seeds to thin"""
    body = parts["rep"] + parts["flank"] + parts["rep"][:900] + parts["rnd"](20_000)
    return [trim_to_count(body, n, lambda s: n_sketch(s, w, k)) for n in (2048, 2049)]


def streak_edge_reads(contigs, parts, w=10, k=15, max_occ=10, occ_dist=10, want=(128, 129)):
    """one stretch of high-occurrence seeds (a prefix of the repeated segment between unique flanks) per wanted max_high_occ; the stretch
    length is searched with streaks()"""
    fl0, fl1 = parts["flank"][:300], parts["flank"][5000:5300]
    found = {}
    for ln in range(1100, 1500):
        s = fl0 + parts["rep"][:ln] + fl1
        st = streaks(s, contigs, w, k, max_occ, occ_dist)
        for n_seed, mho in st:
            if mho in want and mho not in found and n_seed > mho:
                found[mho] = s
        if len(found) == len(want):
            break
    assert len(found) == len(want), sorted(found)
    return [found[m] for m in want] + [fl0 + parts["rep"] + fl1]


def check_edges(L, ctx, seed=3, w=10, k=15, q_occ_max=10):
    """the seeding stage at its capacity edges against the oracle, each case first asserting from the oracle side that both sides of its
    boundary occur: 2048 / 2049 minimizers before the query-side filter with entries both filter kernels drop (one occurring exactly
    q_occ_max times); q_occ_max / q_occ_max + 1 minimizers; 2048 / 2049 minimizers in select_kernel with streak selection on; stretches
    whose max_high_occ is 128, 129 and far above the streak heap's 128 entries"""
    contigs, parts = edge_genome(seed)
    mz = mzflt_edge_reads(parts, w, k, q_occ_max)
    frac = 0.001  # n * q_occ_frac < q_occ_max: q_occ_max decides
    assert [n_sketch(s, w, k) for s in mz] == [2048, 2049, q_occ_max, q_occ_max + 1]
    for s in mz[:2]:
        cnt = read_counts(s, w, k)
        assert (cnt == q_occ_max).any() and (cnt > q_occ_max).any() and q_occ_max > n_sketch(s, w, k) * frac
        assert n_minimizers(s, w, k, q_occ_max, frac) < n_sketch(s, w, k)
    assert n_minimizers(mz[2], w, k, q_occ_max, frac) == q_occ_max and n_minimizers(mz[3], w, k, q_occ_max, frac) == 0
    check_case(L, ctx, contigs, mz, w=w, k=k, mid_occ=q_occ_max, q_occ_frac=frac)
    sel = select_edge_reads(parts, w, k)
    assert [n_sketch(s, w, k) for s in sel] == [2048, 2049]
    for s in sel:
        assert any(n_seed > mho > 0 for n_seed, mho in streaks(s, contigs, w, k, q_occ_max, 200))
    check_case(L, ctx, contigs, sel, w=w, k=k, mid_occ=q_occ_max, q_occ_frac=0.0, occ_dist=200)
    stk = streak_edge_reads(contigs, parts, w, k, q_occ_max, 10)
    mho = [max(m for _, m in streaks(s, contigs, w, k, q_occ_max, 10)) for s in stk]
    assert mho[:2] == [128, 129] and mho[2] > 150, mho
    check_case(L, ctx, contigs, stk, w=w, k=k, mid_occ=q_occ_max, q_occ_frac=0.0, occ_dist=10)
