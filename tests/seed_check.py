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


def check_case(L, ctx, contigs, reads, w=10, k=15, flag=0, mid_occ=10, q_occ_frac=0.01, max_max_occ=4095, occ_dist=500):
    names = ["chr%d" % i for i in range(len(contigs))]
    seqs = [bytes(c) for c in contigs]
    arr = (C.c_char_p * len(seqs))(*seqs); nm = (C.c_char_p * len(seqs))(*[x.encode() for x in names])
    mi = L.mm_idx_str(w, k, 0, 14, len(seqs), arr, nm)
    reads = [bytes(r) for r in reads]
    got = device_seeds(L, ctx, mi, reads, flag, mid_occ, q_occ_frac, max_max_occ, occ_dist)
    idx = O.OracleIndex(seqs, names, w, k)
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
