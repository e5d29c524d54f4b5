"""Index build cases and checkers shared by tests/test_index_cases_vs_ref.py (the oracle against the reference library),
tests/test_emu_index.py (the build kernels under the SIMT emulator) and tests/test_gpu_index.py (on the device).

A case is a set of contigs and sketch parameters (w, k, is_hpc). Every build path of mmb_sketch_device is covered:
sketch_tile_kernel<true> (odd k <= 15), sketch_tile_kernel<false> (odd k 17-27) and the chunk-replay sketch_kernel (even k, w + k > 64,
HPC), which reads the packed S. An index is compared in its canonical form: header, names, lengths, the S words, and the keys in
ascending order, each with its occurrence list in stored order (index.c:264-266 sorts it by position)."""
import ctypes as C
import hashlib
import os
import numpy as np
import oracle_lib as O
import synth

MM_I_HPC, MM_I_NO_SEQ = 0x1, 0x2
BUCKET_BITS = 14
INT32_MAX = (1 << 31) - 1

# (w, k, is_hpc) of every build path; the comment names the sketch kernel the build takes
PARAMS = [
    (10, 15, 0), (1, 5, 0), (3, 7, 0),      # sketch_tile_kernel<true>
    (19, 19, 0), (37, 27, 0),               # sketch_tile_kernel<false>
    (10, 14, 0), (5, 28, 0),                # even k: sketch_kernel
    (50, 21, 0), (200, 15, 0),              # w + k > 64: sketch_kernel
    (10, 19, 1), (5, 19, 1), (10, 15, 1),   # HPC (map-pb, ava-pb, -H): sketch_kernel, one chunk per contig
]
PARAM_IDS = ["w%dk%d%s" % (w, k, "H" if h else "") for w, k, h in PARAMS]

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def _rand(rng, n, alphabet=b"ACGT"):
    return bytes(np.frombuffer(alphabet, dtype=np.uint8)[rng.integers(0, len(alphabet), n)])


def _hpc_runs(rng, n_runs, max_run):
    """homopolymer runs of 1..max_run bases, neighbouring runs of different bases"""
    out, last = [], -1
    for _ in range(n_runs):
        b = int(rng.integers(0, 3))
        b = b if b < last else b + 1 if last >= 0 else int(rng.integers(0, 4))
        last = b
        out.append(bytes([ACGT[b]]) * int(min(max_run, 1 + rng.geometric(0.3) if rng.random() < 0.9 else rng.integers(1, max_run + 1))))
    return b"".join(out)


def _span_edges(k):
    """k-mers whose HPC span is exactly 254..257: one long run among runs of one base (span = run + k - 1), for the
    `kmer_span < 256` test of sketch.c:111"""
    out = []
    for span in (254, 255, 256, 257):
        out.append(b"ACGTCAGT" * 3 + b"ACTGACGTAC"[:k - 1] + b"G" * (span - (k - 1)) + b"TCATGCATCA"[:k - 1] + b"CAGTGCA" * 3)
    return b"".join(out)


def contigs(w, k, is_hpc, seed, scale=1.0):
    """the contigs of one case (ASCII bytes): lengths at the sketch's edges, contigs that start anywhere inside a 32-bit word of S, all-N
    contigs, IUPAC codes and lowercase, many tiny contigs, tandem repeats with thousands of copies and, for HPC, homopolymer runs of 1-400
    and spans of exactly 255 and 256. scale shrinks the bulky parts (the emulator runs a reduced set)."""
    rng = np.random.default_rng(seed)
    out = []
    for n in (0, 1, k - 1, k, w + k - 1, w + k, 31, 32, 33, 63, 2047, 2048, 2049, 4097):
        out.append(_rand(rng, n))
    out.append(b"N" * 300)
    out.append(_rand(rng, 700, b"ACGTRYKMSWBDHVN"))
    out.append(_rand(rng, 900, b"ACGTacgtNn"))
    out.append(_rand(rng, 200) + b"N" * 40 + _rand(rng, 5) + b"N" + _rand(rng, 300))
    out += [_rand(rng, int(rng.integers(1, w + k + 3))) for _ in range(int(3000 * scale))]
    out.append(b"AT" * 200 + b"ACGT" * 150 + b"A" * 300 + _rand(rng, 400))  # symmetric k-mers (even k), ties inside windows
    unit = _rand(rng, 37)
    out.append(_rand(rng, 500) + unit * int(3000 * scale) + _rand(rng, 500))
    out.append(bytes(synth.random_genome(int(60_000 * scale) + 5000, seed + 1, repeat_frac=0.3)[0]))
    out.append(_hpc_runs(rng, int(4000 * scale), 400))
    if is_hpc:
        out.append(_span_edges(k) + _hpc_runs(rng, 300, 30) + _span_edges(k))
    return out


def names_of(ctgs):
    return ["ctg%d" % i for i in range(len(ctgs))]


# ---------------- canonical form ----------------
class Canon:
    """header (w, k, b, n_seq, flag), names, lengths, the S words (None with MM_I_NO_SEQ), and keys in ascending order with counts and
    their occurrence words, each key's list in stored order"""

    def __init__(self, hdr, names, lens, S, keys, cnt, pos):
        self.hdr, self.names, self.lens, self.S = tuple(int(x) for x in hdr), list(names), np.asarray(lens, dtype=np.uint32), S
        self.keys, self.cnt, self.pos = keys, cnt, pos

    def off(self):
        o = np.zeros(len(self.cnt) + 1, dtype=np.int64)
        np.cumsum(self.cnt, out=o[1:])
        return o

    def digest(self):
        h = hashlib.sha1(repr((self.hdr, self.names)).encode())
        for a in (self.lens, self.S if self.S is not None else np.zeros(0, dtype=np.uint32), self.keys, self.cnt, self.pos):
            h.update(np.ascontiguousarray(a).tobytes())
        return h.hexdigest()

    def assert_equal(self, o, what=""):
        assert self.hdr == o.hdr, (what, self.hdr, o.hdr)
        assert self.names == o.names and (self.lens == o.lens).all(), what
        assert (self.S is None) == (o.S is None) and (self.S is None or (len(self.S) == len(o.S) and (self.S == o.S).all())), (what, "S")
        assert len(self.keys) == len(o.keys), (what, len(self.keys), len(o.keys))
        bad = np.flatnonzero((self.keys != o.keys) | (self.cnt != o.cnt))
        assert len(bad) == 0, (what, "key/count differ at rank %d" % bad[0], int(self.keys[bad[0]]), int(o.keys[bad[0]]))
        bad = np.flatnonzero(self.pos != o.pos)
        assert len(bad) == 0, (what, "occurrence differs at %d" % bad[0])


def _gather(starts, cnt):
    """indices start[i] .. start[i] + cnt[i] - 1, i ascending"""
    tot = int(cnt.sum())
    first = np.zeros(len(cnt), dtype=np.int64)
    np.cumsum(cnt[:-1], out=first[1:])
    return np.repeat(starts.astype(np.int64) - first, cnt.astype(np.int64)) + np.arange(tot, dtype=np.int64)


def parse_mmi(buf):
    """every index in a .mmi byte string (several back to back with -I), each as a Canon (index.c:475-569)"""
    parts, o = [], 0
    while o < len(buf):
        assert buf[o:o + 4] == b"MMI\x02", "bad magic at %d" % o
        hdr = np.frombuffer(buf, dtype=np.uint32, count=5, offset=o + 4)
        w, k, b, n_seq, flag = (int(x) for x in hdr)
        o += 24
        names, lens = [], np.zeros(n_seq, dtype=np.uint32)
        for i in range(n_seq):
            ln = buf[o]
            names.append(buf[o + 1:o + 1 + ln].decode())
            o += 1 + ln
            lens[i] = np.frombuffer(buf, dtype=np.uint32, count=1, offset=o)[0]
            o += 4
        ks, cs, ps = [], [], []
        for bi in range(1 << b):
            np_ = int(np.frombuffer(buf, dtype=np.int32, count=1, offset=o)[0])
            p = np.frombuffer(buf, dtype=np.uint64, count=np_, offset=o + 4)
            o += 4 + 8 * np_
            size = int(np.frombuffer(buf, dtype=np.uint32, count=1, offset=o)[0])
            o += 4
            if size == 0:
                continue
            kv = np.frombuffer(buf, dtype=np.uint64, count=2 * size, offset=o).reshape(-1, 2)
            o += 16 * size
            single = (kv[:, 0] & 1).astype(bool)
            cnt = np.where(single, 1, kv[:, 1] & 0xffffffff).astype(np.uint32)
            comb = np.concatenate([p, kv[single, 1]])
            start = np.where(single, len(p) + np.cumsum(single) - 1, (kv[:, 1] >> np.uint64(32)).astype(np.int64))
            ks.append((kv[:, 0] >> np.uint64(1) << np.uint64(b)) | np.uint64(bi))
            cs.append(cnt)
            ps.append(comb[_gather(start, cnt)])
        keys = np.concatenate(ks) if ks else np.zeros(0, dtype=np.uint64)
        cnt = np.concatenate(cs) if cs else np.zeros(0, dtype=np.uint32)
        pos = np.concatenate(ps) if ps else np.zeros(0, dtype=np.uint64)
        order = np.argsort(keys, kind="stable")
        first = np.zeros(len(cnt), dtype=np.int64)
        np.cumsum(cnt[:-1], out=first[1:])
        pos = pos[_gather(first[order], cnt[order])]
        S = None
        if not flag & MM_I_NO_SEQ:
            nw = (int(lens.astype(np.int64).sum()) + 7) // 8
            S = np.frombuffer(buf, dtype=np.uint32, count=nw, offset=o).copy()
            o += 4 * nw
        parts.append(Canon((w, k, b, n_seq, flag), names, lens, S, keys[order], cnt[order], pos))
    return parts


NT4 = np.full(256, 4, dtype=np.uint32)
for _c, _v in zip(b"ACGTUacgtu", (0, 1, 2, 3, 3, 0, 1, 2, 3, 3)):
    NT4[_c] = _v


def pack_S(ctgs):
    """the 4-bit packed S of index.c:351-357"""
    cat = np.frombuffer(b"".join(ctgs) + b"\0" * 8, dtype=np.uint8)[:sum(len(c) for c in ctgs)]
    n = len(cat)
    v = np.zeros((n + 7) // 8 * 8, dtype=np.uint32)
    v[:n] = NT4[cat]
    v = v.reshape(-1, 8) << (np.arange(8, dtype=np.uint32) * 4)
    return np.bitwise_or.reduce(v, axis=1).astype(np.uint32) if n else np.zeros(0, dtype=np.uint32)


def oracle_canon(ctgs, w, k, is_hpc, names=None):
    """the oracle's index (oracle/mm2o_seed.c restates worker_post) in canonical form, with the header mm_idx_str writes"""
    names = names_of(ctgs) if names is None else names
    idx = O.OracleIndex(ctgs, names, w, k, is_hpc)
    L = O.oracle()
    L.mm2o_idx_keys.restype = C.c_int64
    kp, sp, pp = C.POINTER(C.c_uint64)(), C.POINTER(C.c_int64)(), C.POINTER(C.c_uint64)()
    n = L.mm2o_idx_keys(idx.h, C.byref(kp), C.byref(sp), C.byref(pp))
    keys = np.ctypeslib.as_array(kp, (n,)).copy() if n else np.zeros(0, dtype=np.uint64)
    start = np.ctypeslib.as_array(sp, (n + 1,)).copy()
    pos = np.ctypeslib.as_array(pp, (int(start[-1]),)).copy() if start[-1] else np.zeros(0, dtype=np.uint64)
    idx.close()
    flag = MM_I_HPC if is_hpc else 0
    hdr = (max(w, 1), k, min(BUCKET_BITS, 2 * k), len(ctgs), flag)  # mm_idx_init, index.c:52-61
    return Canon(hdr, names, [len(c) for c in ctgs], pack_S(ctgs), keys, np.diff(start).astype(np.uint32), pos)


# ---------------- mid_occ (mm_idx_cal_max_occ, index.c:198-220) ----------------
F_FIXED = (1.0, 0.5, 0.01, 2e-4, 1e-6)


def f_values(n):
    """the fixed fractions, and for a few ranks m the float32 values of f at and around the one where (1. - f) * n crosses m"""
    fs = list(F_FIXED)
    for m in sorted({n - 1, (n * 999) // 1000, n // 2, n // 3, 1}):
        if 0 < m < n:
            f = np.float32(1.0 - m / n)
            for g in (np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))):
                if 0 < g <= 1:
                    fs.append(float(g))
    return fs


def max_occ(cnt, f):
    """mm_idx_cal_max_occ from the occurrence counts: the (uint32)((1. - f) * n)-th smallest count, plus one; f is a C float"""
    f = float(np.float32(f))
    if f <= 0 or len(cnt) == 0:
        return INT32_MAX
    return int(np.sort(cnt)[int((1.0 - f) * len(cnt))]) + 1


# ---------------- a library's index (this one's, the emulator's or the reference's) ----------------
_libc = C.CDLL("libc.so.6")
_libc.fopen.restype = C.c_void_p
_libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
_libc.fclose.argtypes = [C.c_void_p]


def setup(L):
    L.mm_idx_str.restype = C.c_void_p
    L.mm_idx_str.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
    L.mm_idx_destroy.argtypes = [C.c_void_p]
    L.mm_idx_dump.argtypes = [C.c_void_p, C.c_void_p]
    L.mm_idx_load.restype = C.c_void_p
    L.mm_idx_load.argtypes = [C.c_void_p]
    L.mm_idx_cal_max_occ.restype = C.c_int32
    L.mm_idx_cal_max_occ.argtypes = [C.c_void_p, C.c_float]
    if hasattr(L, "mmb_idx_lookup_host"):
        L.mmb_idx_lookup_host.restype = C.c_int64


def build(L, ctgs, w, k, is_hpc, names=None):
    """mm_idx_str of L on the contigs"""
    names = names_of(ctgs) if names is None else names
    arr = (C.c_char_p * len(ctgs))(*[bytes(c) for c in ctgs])
    nm = (C.c_char_p * len(ctgs))(*[x.encode() for x in names])
    return L.mm_idx_str(w, k, is_hpc, BUCKET_BITS, len(ctgs), arr, nm)


def dump(L, mi, path):
    """mm_idx_dump of L into path; returns the bytes"""
    fp = _libc.fopen(str(path).encode(), b"wb")
    L.mm_idx_dump(fp, mi)
    _libc.fclose(fp)
    return open(path, "rb").read()


def load(L, path):
    fp = _libc.fopen(str(path).encode(), b"rb")
    mi = L.mm_idx_load(fp)
    _libc.fclose(fp)
    return mi


def recorded(name, ref_canon_fn):
    """the reference index's digest and mid_occ values, recorded with O.reference_values; ref_canon_fn() -> (Canon, {f: value})"""
    def compute():
        c, mo = ref_canon_fn()
        return dict(digest=c.digest(), n_keys=len(c.keys), max_occ=[[repr(f), v] for f, v in mo.items()])
    return O.reference_values("index:" + name, compute)


def case_name(w, k, is_hpc, seed, scale):
    return "w%d.k%d.hpc%d.seed%d.scale%g" % (w, k, is_hpc, seed, scale)


# ---------------- absent keys ----------------
GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def tab_bits(n_keys):
    """the table size finish_table() picks (index.cu): load factor <= 0.5, at least 2^10 slots"""
    bits = 10
    while (1 << bits) < n_keys * 2:
        bits += 1
    return bits


def slot_of(keys, bits):
    """idx_slot_of (index.h)"""
    with np.errstate(over="ignore"):
        return (np.asarray(keys, dtype=np.uint64) * GOLDEN) >> np.uint64(64 - bits)


def absent_keys(keys, k, rng):
    """keys that are not in the index: every present key with one bit flipped (within the 2k hash bits) when that gives an absent key,
    and keys whose home slot is the last slot of the table"""
    mask = np.uint64((1 << 2 * k) - 1)
    present = np.asarray(keys, dtype=np.uint64)
    flip = (present ^ (np.uint64(1) << rng.integers(0, 2 * k, len(present)).astype(np.uint64))) & mask
    last = np.uint64((1 << tab_bits(len(present))) - 1)
    tail = []
    for _ in range(64):
        cand = rng.integers(0, 1 << min(2 * k, 63), 1 << 20, dtype=np.uint64) & mask
        tail.append(cand[slot_of(cand, tab_bits(len(present))) == last])
        if sum(len(t) for t in tail) >= 16:
            break
    out = np.unique(np.concatenate([flip] + tail))
    return out[~np.isin(out, present)]


def last_slot_occupied(keys):
    """whether linear probing fills the table's last slot (the set of filled slots does not depend on the insertion order). Then a
    probe for an absent key whose home is the last slot crosses the end of the table to slot 0."""
    bits = tab_bits(len(keys))
    h = np.sort(slot_of(keys, bits).astype(np.int64))
    i = np.arange(len(h))
    return len(h) > 0 and int((i + np.maximum.accumulate(h - i)).max()) >= (1 << bits) - 1  # slot of the i-th home, before wrapping


def wraps(keys, k):
    """whether check_lookup's absent keys include a probe that crosses the end of the table: the last slot is filled and some absent
    key has its home there (with k = 5 every 10-bit key homed there may be present)"""
    bits = tab_bits(len(keys))
    return bool(last_slot_occupied(keys) and (slot_of(absent_keys(keys, k, np.random.default_rng(0)), bits) == np.uint64((1 << bits) - 1)).any())


# ---------------- the device index against the oracle ----------------
def check_lookup(L, mi, exp, k, rng):
    """the device table probed for every key (idx_lookup) equals the oracle's lists; absent keys find nothing. Returns whether some of
    those probes crossed the end of the table."""
    from minimap2_b200 import kernels as K
    cnt, off, occ = K.idx_lookup(mi, exp.keys, L)
    assert (cnt == exp.cnt).all(), ("count", int(np.flatnonzero(cnt != exp.cnt)[0]))
    assert (off == exp.off()).all() and len(occ) == len(exp.pos)
    bad = np.flatnonzero(occ != exp.pos)
    assert len(bad) == 0, ("occurrence", int(bad[0]))
    absent = absent_keys(exp.keys, k, rng)
    cnt, off, occ = K.idx_lookup(mi, absent, L)
    assert not cnt.any() and len(occ) == 0
    bits = tab_bits(len(exp.keys))
    return last_slot_occupied(exp.keys) and bool((slot_of(absent, bits) == np.uint64((1 << bits) - 1)).any())


def check_device_index(L, ctgs, w, k, is_hpc, tmp_path, max_occ_values=None, rng=None):
    """mm_idx_str of L (the build kernels) against the oracle: the dump in canonical form, every lookup, mm_idx_cal_max_occ at every
    fraction of f_values (max_occ_values: {f: value} recorded from the reference; default: computed from the oracle's counts), and the
    same after mm_idx_dump -> mm_idx_load -> mm_idx_dump. Returns the oracle's canonical index, and whether some probe for an absent
    key crossed the end of the table."""
    rng = rng or np.random.default_rng(3)
    exp = oracle_canon(ctgs, w, k, is_hpc)
    mo = max_occ_values or {f: max_occ(exp.cnt, f) for f in f_values(len(exp.keys))}
    mi = build(L, ctgs, w, k, is_hpc)
    got, = parse_mmi(dump(L, mi, tmp_path / "a.mmi"))
    exp.assert_equal(got, "mm_idx_str")
    wrapped = check_lookup(L, mi, exp, k, rng)
    for f, v in mo.items():
        assert L.mm_idx_cal_max_occ(mi, f) == v, (f, v)
    mi2 = load(L, tmp_path / "a.mmi")
    L.mm_idx_destroy(mi)
    assert mi2
    again, = parse_mmi(dump(L, mi2, tmp_path / "b.mmi"))
    exp.assert_equal(again, "dump -> load -> dump")
    assert check_lookup(L, mi2, exp, k, rng) == wrapped
    for f, v in mo.items():
        assert L.mm_idx_cal_max_occ(mi2, f) == v, ("loaded", f, v)
    L.mm_idx_destroy(mi2)
    return exp, wrapped


# ---------------- -I: an index in parts (idx_gen's mini-batch rule, index.c:389-408 and bseq.c:80-119) ----------------
def parts_fasta(path, seed):
    """contigs whose lengths sum exactly to the mini-batch size of PARTS_OPT at some record ends, and others that do not"""
    rng = np.random.default_rng(seed)
    lens = [1000] * 10 + [int(x) for x in rng.integers(1, 3000, 20)] + [2500, 2500] + [int(x) for x in rng.integers(1, 400, 30)]
    names = ["p%d" % i for i in range(len(lens))]
    seqs = [np.frombuffer(_rand(rng, n), dtype=np.uint8) for n in lens]
    synth.write_fasta(str(path), names, seqs)
    return dict(zip(names, (bytes(x) for x in seqs)))


PARTS_OPT = [(5000, 12000), (5000, 5000), (1000, 30000), (64, 1)]  # (mini_batch_size, batch_size)


def read_parts(L, fn, w, k, is_hpc, mini_batch_size, batch_size, tmp_path):
    """every part mm_idx_reader_read of L makes of fn, in canonical form; the multi-part file the reader writes as it goes (-d) must
    hold the same parts"""
    from minimap2_b200.api import IdxOpt
    # private function objects (L[name] makes a new one): the attributes of L keep the types minimap2_b200.api gives them
    reader_open, reader_read, reader_close = L["mm_idx_reader_open"], L["mm_idx_reader_read"], L["mm_idx_reader_close"]
    reader_open.restype = C.c_void_p
    reader_open.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.c_char_p]
    reader_read.restype = C.c_void_p
    reader_read.argtypes = [C.c_void_p, C.c_int]
    reader_close.argtypes = [C.c_void_p]
    io = IdxOpt(k=k, w=w, flag=MM_I_HPC if is_hpc else 0, bucket_bits=BUCKET_BITS, mini_batch_size=mini_batch_size, batch_size=batch_size)
    rd = reader_open(str(fn).encode(), C.byref(io), str(tmp_path / "all.mmi").encode())
    assert rd
    out = []
    while True:
        mi = reader_read(rd, 1)
        if not mi:
            break
        out += parse_mmi(dump(L, mi, tmp_path / "part.mmi"))
        L.mm_idx_destroy(mi)
    reader_close(rd)
    d = [c.digest() for c in parse_mmi(open(tmp_path / "all.mmi", "rb").read())]  # what `-d` writes: the parts back to back
    assert d == [c.digest() for c in out]
    return out


PARTS_PARAMS = [(10, 15, 0), (10, 19, 1)]


def parts_name(w, k, is_hpc, mbs, bs):
    return "index-parts:w%d.k%d.hpc%d.mb%d.b%d" % (w, k, is_hpc, mbs, bs)


def check_parts(L, w, k, is_hpc, tmp_path):
    """the parts of L's reader equal the reference's, recorded by tests/test_index_cases_vs_ref.py"""
    parts_fasta(tmp_path / "parts.fa", 9)
    for mbs, bs in PARTS_OPT:
        got = read_parts(L, tmp_path / "parts.fa", w, k, is_hpc, mbs, bs, tmp_path)
        rec = O.reference_values(parts_name(w, k, is_hpc, mbs, bs), None)
        assert [c.names for c in got] == rec["names"], (mbs, bs)
        assert [c.digest() for c in got] == rec["digests"], (mbs, bs)


# ---------------- .mmi files the reference wrote (tests/golden/make_reference_lines.sh) ----------------
GOLD_DATA = os.path.join(O.ROOT, "tests", "golden", "data")
# (fixture, w, k, is_hpc): the reference's `-d` of data/MT-human.fa with these parameters
REF_MMI = [("MT-human.H.w10k19.mmi.gz", 10, 19, 1), ("MT-human.w4k6.mmi.gz", 4, 6, 0)]


def read_fasta(fn):
    names, seqs = [], []
    for blk in open(fn, "rb").read().split(b">")[1:]:
        head, _, body = blk.partition(b"\n")
        names.append(head.split()[0].decode())
        seqs.append(body.replace(b"\n", b""))
    return names, seqs


def check_reference_mmi(L, fn, w, k, is_hpc, tmp_path):
    """the reference's .mmi equals the oracle's index of MT-human.fa; L loads it, and its dump and every probe agree"""
    import gzip
    names, seqs = read_fasta(os.path.join(GOLD_DATA, "MT-human.fa"))
    exp = oracle_canon(seqs, w, k, is_hpc, names=names)
    raw = gzip.open(os.path.join(GOLD_DATA, fn)).read()
    ref, = parse_mmi(raw)
    exp.assert_equal(ref, fn)
    open(tmp_path / "ref.mmi", "wb").write(raw)
    mi = load(L, tmp_path / "ref.mmi")
    assert mi
    got, = parse_mmi(dump(L, mi, tmp_path / "again.mmi"))
    exp.assert_equal(got, fn + " loaded")
    check_lookup(L, mi, exp, k, np.random.default_rng(2))
    for f in f_values(len(exp.keys)):
        assert L.mm_idx_cal_max_occ(mi, f) == max_occ(exp.cnt, f), f
    L.mm_idx_destroy(mi)


# ---------------- mapping with HPC, even-k and wide-window indexes through the CLI ----------------
def cli_inputs(d, tag, glen, n_reads, seed):
    """a homopolymer-rich reference of three contigs (random stretches between homopolymer runs of 1-12 bases) and reads sampled from
    it with 8% errors, half of them reverse-complemented. Returns the two file names, relative to d."""
    rng = np.random.default_rng(seed)
    ctgs = []
    for n in (glen // 2, glen // 3, glen - glen // 2 - glen // 3):
        parts, tot = [], 0
        while tot < n:
            parts.append(_rand(rng, int(rng.integers(50, 400))) if rng.random() < 0.5 else _hpc_runs(rng, int(rng.integers(30, 200)), 12))
            tot += len(parts[-1])
        ctgs.append(np.frombuffer(b"".join(parts)[:n], dtype=np.uint8))
    reads = []
    for i in range(n_reads):
        c = ctgs[i % 3]
        ln = int(rng.integers(800, min(6000, len(c) // 2)))
        s = int(rng.integers(0, len(c) - ln))
        r = synth.mutate_ascii(c[s:s + ln], rng, 0.08)
        reads.append(synth.revcomp(r) if i % 2 else r)
    rf, qf = tag + "_ref.fa", tag + "_reads.fa"
    synth.write_fasta(os.path.join(d, rf), ["hp%d" % i for i in range(3)], [bytes(c) for c in ctgs])
    synth.write_fasta(os.path.join(d, qf), ["r%d" % i for i in range(n_reads)], [bytes(r) for r in reads])
    return rf, qf


def cli_lines(rf, qf, I="60k"):
    """the option lines of the CLI tests: map-pb and ava-pb (HPC), -H, even k, w + k > 64, and an HPC index in -I parts"""
    return [["-x", "map-pb", "-c", "--cs", rf, qf], ["-x", "map-pb", "-a", rf, qf], ["-x", "ava-pb", qf, qf],
            ["-H", "-k", "15", "-w", "10", "-c", rf, qf], ["-k", "14", "-w", "10", "-c", rf, qf], ["-k", "21", "-w", "50", "-c", rf, qf],
            ["-x", "map-pb", "-I", I, "-c", rf, qf]]
