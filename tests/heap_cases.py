"""Heap-ordered seeding (MM_F_HEAP_SORT, `--heap-sort=yes`: collect_seed_hits_heap, map.c:102-166): the restatement the tests compare
against, the reference's recorded output, inputs and counters. Used by tests/test_oracle_heap_seed.py, tests/test_emu_heap_seed.py and
tests/test_gpu_heap_seed.py.

HeapOracle restates the heap merge on top of the oracle's seeding stage (oracle/mm2o_seed.c): that stage gives the kept seeds (their
mini_pos words, in seed order), rep_len and the tandem flags, the oracle index gives every seed's occurrence list, and the merge itself,
skip_seed and the anchor formulas are written out here. The heap merge differs from the sorted order only where anchors have equal x,
so every case is built from repeat-rich genomes and tandem reads, at long and at short read lengths, and tie_stats() counts the
situations the order depends on: ties in small reads, on both strands, between occurrences that differ only in the strand bit (see
assert_covered), and groups of equal occurrences that skip_seed thins."""
import ctypes as C
import json
import os
import numpy as np
import oracle_lib as O
import seed_check as SC
import synth

HEAP = 0x400000                       # MM_F_HEAP_SORT
F_NO_DIAG, F_NO_DUAL, F_FOR_ONLY, F_REV_ONLY, F_QSTRAND = 0x001, 0x002, 0x100000, 0x200000, 0x100000000
SKIP = F_NO_DIAG | F_NO_DUAL | F_FOR_ONLY | F_REV_ONLY  # the flags under which skip_seed drops occurrences
SEED_TANDEM, SEED_SELF, SEED_SEG_SHIFT = 1 << 42, 1 << 43, 48
M32, HI32 = 0xffffffff, 0xffffffff00000000
REF_LINES = os.path.join(O.ROOT, "tests", "golden", "expected", "heap_reference_lines.json")


def reference_lines(args, records=None):
    """the reference binary's recorded output of `minimap2 <args>` (oracle_lib's digest form), from expected/heap_reference_lines.json.
    With MM2_RECORD_REFERENCE set, oracle_lib runs the reference binary and records into that file instead
    (tests/golden/make_heap_reference_lines.sh)."""
    if os.environ.get("MM2_RECORD_REFERENCE"):
        return O.reference_lines(args, records=records)
    key = O.input_key(args)
    tab = json.load(open(REF_LINES))
    assert key in tab, "no recorded reference output for these inputs: minimap2 " + key
    return O.RecordedLines(tab[key])


def _sift(hx, hy, i, n):
    """ksort.h's heap sift-down (ksort.h:44-56) with heap_lt(a, b) = a.x > b.x (map.c:74): a min-heap on x alone. The smaller child
    is followed, and the entry stops only above a child whose x is strictly larger, so it sinks below children with an equal x."""
    tx, ty = hx[i], hy[i]
    while True:
        k = 2 * i + 1
        if k >= n:
            break
        if k != n - 1 and hx[k] > hx[k + 1]:
            k += 1
        if hx[k] > tx:
            break
        hx[i], hy[i] = hx[k], hy[k]
        i = k
    hx[i], hy[i] = tx, ty


class HeapOracle:
    """OracleIndex with the anchor order of collect_seed_hits_heap: anchors(..., heap=True)"""

    def __init__(self, seqs, names, w, k, is_hpc=0):
        self.idx = O.OracleIndex(seqs, names, w, k, is_hpc)
        self.w, self.k, self.is_hpc = w, k, is_hpc
        self.names = [n.encode() for n in names]
        self.lens = [len(x) for x in seqs]
        self._get = O.oracle().mm2o_idx_get
        self._get.restype = C.POINTER(C.c_uint64)
        self._get.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_int)]

    def close(self):
        self.idx.close()

    def _occ(self, key):
        n = C.c_int(0)
        p = self._get(self.idx.h, key, C.byref(n))
        return p[:n.value] if n.value else []

    def _skip(self, flag, r, q_pos, qname, qlen):
        """skip_seed (map.c:78-100): (dropped, is_self)"""
        is_self = False
        if qname is not None and flag & (F_NO_DIAG | F_NO_DUAL):
            rid = r >> 32
            nm = self.names[rid]
            cmp = (qname > nm) - (qname < nm)
            if flag & F_NO_DIAG and cmp == 0 and self.lens[rid] == qlen:
                if (r & M32) >> 1 == q_pos >> 1:
                    return True, False
                if r & 1 == q_pos & 1:
                    is_self = True
            if flag & F_NO_DUAL and cmp > 0:
                return True, is_self
        if flag & (F_FOR_ONLY | F_REV_ONLY):
            if r & 1 == q_pos & 1:
                if flag & F_REV_ONLY:
                    return True, is_self
            elif flag & F_FOR_ONLY:
                return True, is_self
        return False, is_self

    def anchors(self, seq, qname=None, flag=0, mid_occ=10, q_occ_frac=0.01, max_max_occ=4095, occ_dist=500, heap=True):
        """(anchors, rep_len, mini_pos) of one read; heap=False gives the oracle's sorted order (collect_seed_hits)"""
        s = seq if isinstance(seq, bytes) else bytes(seq)
        kw = dict(mid_occ=mid_occ, q_occ_frac=q_occ_frac, max_max_occ=max_max_occ, occ_dist=occ_dist)
        if not heap:
            return self.idx.anchors(s, qname=qname, flag=flag & ~HEAP, **kw)
        # the kept seeds, rep_len and tandem flags do not depend on skip_seed or the anchor formulas: take them from the sorted path
        # with neither, where every kept seed has at least one anchor
        plain, rep, mp = self.idx.anchors(s, flag=0, **kw)
        qlen = len(s)
        tandem = {}
        for x, y in plain:
            x, y = int(x), int(y)
            span, yq = y >> 32 & 0xff, y & M32
            pos = qlen - yq - 2 + span if x >> 63 else yq
            tandem[pos] = bool(y & SEED_TANDEM)
        mz = O.oracle_sketch(s, self.w, self.k, is_hpc=self.is_hpc)
        by_pos = {int(y) >> 1 & 0x7fffffff: (int(x), int(y)) for x, y in mz}
        seeds = []  # (q_pos, span, seg_id, tandem, occurrences) in the order of m[] (map.c:114)
        for w in mp:
            x, y = by_pos[int(w) & M32]
            seeds.append((y & M32, x & 0xff, y >> 32, tandem[int(w) & M32], self._occ(x >> 8)))
        qn = None if qname is None else (qname.encode() if isinstance(qname, str) else qname)
        hx = [q[4][0] for q in seeds]
        hy = [i << 32 for i in range(len(seeds))]
        size = len(seeds)
        for i in range(size // 2 - 1, -1, -1):  # ks_heapmake
            _sift(hx, hy, i, size)
        fwd, rev = [], []
        while size > 0:
            r, i, j = hx[0], hy[0] >> 32, hy[0] & M32
            q_pos, span, seg, tnd, occ = seeds[i]
            drop, is_self = self._skip(flag, r, q_pos, qn, qlen)
            if not drop:  # map.c:128-143: the reverse formula without query strand, in every mode
                rpos = (r & M32) >> 1
                if r & 1 == q_pos & 1:
                    x, y, out = (r & HI32) | rpos, span << 32 | q_pos >> 1, fwd
                else:
                    x, y, out = 1 << 63 | (r & HI32) | rpos, span << 32 | ((qlen - ((q_pos >> 1) + 1 - span) - 1) & M32), rev
                y |= seg << SEED_SEG_SHIFT
                if tnd:
                    y |= SEED_TANDEM
                if is_self:
                    y |= SEED_SELF
                out.append((x, y))
            if j + 1 < len(occ):  # the seed's next occurrence replaces the top, or the heap shrinks
                hx[0], hy[0] = occ[j + 1], hy[0] + 1
            else:
                size -= 1
                hx[0], hy[0] = hx[size], hy[size]
            _sift(hx, hy, 0, size)
        a = np.array(fwd + rev, dtype=np.uint64).reshape(-1, 2)
        return a, rep, mp


def check_device(L, ctx, contigs, reads, w=10, k=15, flag=0, mid_occ=10, q_occ_frac=0.01, max_max_occ=4095, occ_dist=500):
    """the seeding stage through mmb_seed_batch_host with MM_F_HEAP_SORT against HeapOracle: anchors in order, rep_len, mini_pos"""
    names = ["chr%d" % i for i in range(len(contigs))]
    seqs = [bytes(c) for c in contigs]
    arr = (C.c_char_p * len(seqs))(*seqs); nm = (C.c_char_p * len(seqs))(*[x.encode() for x in names])
    mi = L.mm_idx_str(w, k, 0, 14, len(seqs), arr, nm)
    reads = [bytes(r) for r in reads]
    got = SC.device_seeds(L, ctx, mi, reads, flag | HEAP, mid_occ, q_occ_frac, max_max_occ, occ_dist)
    ho = HeapOracle(seqs, names, w, k)
    n_a = 0
    for i, s in enumerate(reads):
        ea, erep, emp = ho.anchors(s, flag=flag, mid_occ=mid_occ, q_occ_frac=q_occ_frac, max_max_occ=max_max_occ, occ_dist=occ_dist) \
            if len(s) else (np.zeros((0, 2), dtype=np.uint64), 0, np.zeros(0, dtype=np.uint64))
        ga, grep_, gmp = got[i]
        assert grep_ == erep, (i, grep_, erep)
        assert len(gmp) == len(emp) and (gmp == emp).all(), (i, len(gmp), len(emp))
        assert ga.shape == ea.shape, (i, ga.shape, ea.shape)
        assert (ga == ea).all(), (i, int(np.argmax((ga != ea).any(axis=1))))
        n_a += len(ea)
    ho.close()
    L.mm_idx_destroy(mi)
    return n_a


def mixed_case(seed, glen, n_long, long_len, n_short, rep=0.6, n_contigs=2):
    """seed_check.repeat_rich_case's genome and long reads (with its tandem read), plus short reads of 150-300 bp from the same genome,
    some of them tandem copies of a short unit"""
    contigs, reads = SC.repeat_rich_case(seed, glen, n_long, long_len, rep=rep, n_contigs=n_contigs)
    for j, ln in enumerate((150, 200, 250, 300)):
        reads += synth.make_reads(contigs, n_short // 4, ln, 0.03, seed + 70 + j, chimeric_frac=0.0)
    c0 = bytes(contigs[0])
    rc = lambda s: bytes(synth.revcomp(np.frombuffer(s, dtype=np.uint8)))
    for j in range(8):
        # a 30-58 bp unit repeated to 240 or 80 bp, and its reverse complement: one occurrence hit by several query positions (forward, then
        # reverse ties in reads of <= 64 anchors)
        u = c0[1000 + 997 * j:1000 + 997 * j + 30 + 4 * j]
        t = (u * 8)[:240 if j % 2 == 0 else 80]
        reads += [t, rc(t)]
        # a segment followed by its reverse complement: the same occurrence is hit from both query strands, once as a forward and once
        # as a reverse anchor, so a strand restriction keeps one of them
        s = c0[20_000 + 1500 * j:20_000 + 1500 * j + (100 if j < 4 else 1200)]
        reads.append(s + rc(s))
    reads.append(rc(reads[len(reads) - 1 - 8 * 3 - 4 * (n_short // 4)]))  # repeat_rich_case's long tandem read, reverse complemented
    return contigs, reads


def _qstrand(seq, w, k, is_hpc=0):
    """query position -> strand bit of the minimizer ending there"""
    mz = O.oracle_sketch(bytes(seq), w, k, is_hpc=is_hpc)
    return {int(y) >> 1 & 0x7fffffff: int(y) & 1 for y in mz[:, 1]}


def _occurrences(a, qlen, strand_at):
    """the occurrence word r = rid<<32 | pos<<1 | strand behind every anchor of the plain (not query-strand) formulas"""
    out = []
    for x, y in a:
        x, y = int(x), int(y)
        rev, span, yq = x >> 63, y >> 32 & 0xff, y & 0xffffffff
        qpos = qlen - yq - 2 + span if rev else yq
        s = strand_at[qpos] ^ rev
        out.append((x >> 32 & 0x7fffffff) << 32 | (x & 0xffffffff) << 1 | s)
    return out


def tie_stats(idx, reads, qnames, w, k, kw):
    """counters over HeapOracle's anchors of every read (kw: HeapOracle.anchors arguments incl. flag)"""
    st = dict(reads=0, anchors=0, tie_reads=0, small_tie_reads=0, fwd_ties=0, rev_ties=0, strand_r_ties=0, thinned=0, differs=0)
    flag = kw.get("flag", 0)
    for s, qn in zip(reads, qnames):
        if not len(s):
            continue
        a, _, _ = idx.anchors(s, qname=qn, heap=True, **kw)
        st["reads"] += 1
        st["anchors"] += len(a)
        strand_at = _qstrand(s, w, k)
        if flag & SKIP:  # equal occurrences of which skip_seed drops some and keeps some
            kw0 = dict(kw, flag=flag & ~SKIP)
            a0, _, _ = idx.anchors(s, qname=qn, heap=True, **kw0)
            c0, c1 = {}, {}
            for v in _occurrences(a0, len(s), strand_at):
                c0[v] = c0.get(v, 0) + 1
            for v in _occurrences(a, len(s), strand_at):
                c1[v] = c1.get(v, 0) + 1
            st["thinned"] += sum(1 for v, c in c1.items() if c < c0.get(v, 0) and c0[v] >= 2)
        if len(a) < 2:
            continue
        eq = a[1:, 0] == a[:-1, 0]
        if not eq.any():
            continue
        st["tie_reads"] += 1
        st["small_tie_reads"] += int(len(a) <= 64)
        rev = (a[:-1, 0] >> np.uint64(63)).astype(bool)
        st["fwd_ties"] += int((eq & ~rev).sum())
        st["rev_ties"] += int((eq & rev).sum())
        r = _occurrences(a, len(s), strand_at)
        st["strand_r_ties"] += sum(1 for i in np.nonzero(eq)[0] if r[i] != r[i + 1])
        srt, _, _ = idx.anchors(s, qname=qn, heap=False, **kw)
        st["differs"] += int(not (srt == a).all())
    return st


def assert_covered(st, strands="+-", skip=False):
    """the situations the heap order depends on occur in the case: ties in reads of <= 64 anchors, ties on each strand the mode keeps,
    a heap order that differs from the sorted one, and (skip) equal occurrences thinned by skip_seed. strand_r_ties is counted but not
    required: the sketch gives every (contig, position) one minimizer, so an index never holds two occurrences that differ only in the
    strand bit, and equal x always comes from equal occurrences."""
    assert st["small_tie_reads"] >= 1, st
    assert ("+" not in strands or st["fwd_ties"] >= 1) and ("-" not in strands or st["rev_ties"] >= 1), st
    assert st["differs"] >= 1, st
    if skip:
        assert st["thinned"] >= 1, st


def oversize_case(unit_len=500, copies=24, seed=31):
    """a contig holding a tandem array of one unit and a read made of copies of the unit on both strands: every seed hits every copy,
    so the read has more than 16384 anchors (the sort kernels' oversize class) and more kept seeds than a shared-memory heap holds"""
    rng = np.random.default_rng(seed)
    u = bytes(synth.ALPHA[rng.integers(0, 4, unit_len)])
    flank = bytes(synth.ALPHA[rng.integers(0, 4, 5000)])
    half = u * (copies // 2)  # both strands, so that a strand restriction still leaves an oversize read
    return flank + u * copies + flank, half + bytes(synth.revcomp(np.frombuffer(half, dtype=np.uint8)))


def path_counts(idx, reads, kw, smem_cap=128, oversize=16384):
    """reads with equal keys whose heap fits in shared memory / needs the global fallback, and oversize reads (idx: HeapOracle)"""
    c = dict(smem=0, global_=0, oversize=0)
    for s in reads:
        if not len(s):
            continue
        a, _, mp = idx.anchors(bytes(s), heap=True, **kw)
        if len(a) > oversize:
            c["oversize"] += 1
        elif len(a) > 1 and (a[1:, 0] == a[:-1, 0]).any():
            c["smem" if len(mp) <= smem_cap else "global_"] += 1
    return c
