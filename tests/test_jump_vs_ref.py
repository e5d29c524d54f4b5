"""CPU: junction jumps against the unmodified reference library.
- The jump table (mm_idx_jjump_read from an annotation BED, then merged with a pass-1 BED): every entry, strand and flag included,
  through mm_idx_jump_get on random windows.
- Thousands of synthetic spliced hits: the reference's mm_jump_split against this library's host apply step (mmb_jump_apply) fed
  with the decisions of the restatement in jump_cases.py; every field of mm_reg1_t and mm_extra_t, CIGAR included.
The product library is used without a device: the index object is built on the host only (no device table)."""
import ctypes as C
import os
import numpy as np
import pytest
import oracle_lib as O
import jump_cases as J
from minimap2_b200._lib import lib
from minimap2_b200.api import IdxOpt, MapOpt, Idx, IdxSeq, Reg1, Extra

pytestmark = pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
libc = C.CDLL(None)
libc.malloc.restype = C.c_void_p
libc.malloc.argtypes = [C.c_size_t]


class Jj1(C.Structure):  # mm_idx_jjump1_t (mmpriv.h:59-63)
    _fields_ = [("off", C.c_int32), ("off2", C.c_int32), ("cnt", C.c_int32), ("strand", C.c_int16), ("flag", C.c_uint16)]


def _setup(L):
    L.mm_idx_jjump_read.restype = C.c_int
    L.mm_idx_jjump_read.argtypes = [C.POINTER(Idx), C.c_char_p, C.c_int, C.c_int]
    L.mm_idx_jump_get.restype = C.POINTER(Jj1)
    L.mm_idx_jump_get.argtypes = [C.POINTER(Idx), C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    return L


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = J.make_data(seed=11)
    dirname = J.write_data(d, str(tmp_path_factory.mktemp("jump")))
    rng = np.random.default_rng(5)
    lines = []  # a pass-1 BED: annotated introns and new ones, scores around the threshold of 5
    for b in d["bed"]:
        f = b.split("\t")
        if f[3] in ("dup", "decoy"):
            lines.append("%s\t%s\t%s\tp1\t%d\t%s" % (f[0], f[1], f[2], int(rng.integers(2, 9)), "+-"[int(rng.integers(0, 2))]))
    for i in range(40):
        c = int(rng.integers(0, len(d["names"])))
        st = int(rng.integers(100, len(d["contigs"][c]) - 1000))
        lines.append("%s\t%d\t%d\tp1n\t%d\t%s" % (d["names"][c], st, st + int(rng.integers(50, 800)), int(rng.integers(3, 8)), "+-"[i % 2]))
    with open(os.path.join(dirname, "pass1.bed"), "w") as f:
        f.write("\n".join(lines) + "\n")
    d["dir"] = dirname
    return d


def ref_index(R, d):
    """the reference's index of ref.fa, read as its command line reads it (-x splice: k=15, w=5)"""
    R.mm_idx_reader_open.restype = C.c_void_p
    R.mm_idx_reader_open.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.c_char_p]
    R.mm_idx_reader_read.restype = C.POINTER(Idx)
    R.mm_idx_reader_read.argtypes = [C.c_void_p, C.c_int]
    R.mm_idx_reader_close.argtypes = [C.c_void_p]
    io, mo = IdxOpt(), MapOpt()
    R.mm_set_opt(None, C.byref(io), C.byref(mo))
    R.mm_set_opt(b"splice", C.byref(io), C.byref(mo))
    rd = R.mm_idx_reader_open(os.path.join(d["dir"], "ref.fa").encode(), C.byref(io), None)
    mi = R.mm_idx_reader_read(rd, 1)
    R.mm_idx_reader_close(rd)
    return mi


def host_index(d):
    """an mm_idx_t of this library with the contig names and lengths only (no sequence, no device side)"""
    mi = Idx()
    n = len(d["contigs"])
    seq = (IdxSeq * (n + 1))()
    keep = [nm.encode() for nm in d["names"]]
    off = 0
    for i in range(n):
        seq[i].name, seq[i].offset, seq[i].len = keep[i], off, len(d["contigs"][i])
        off += len(d["contigs"][i])
    mi.n_seq, mi.seq = n, seq
    mi._keep = (seq, keep)
    return mi


def entries(L, mi, cid, st, en):
    n = C.c_int32(0)
    p = L.mm_idx_jump_get(mi, cid, st, en, C.byref(n))
    return [(p[i].off, p[i].off2, p[i].cnt, p[i].strand, p[i].flag) for i in range(n.value)]


def test_table_matches_reference(data):
    R, L = _setup(O.ref()), _setup(lib())
    rmi, omi = ref_index(R, data), host_index(data)
    anno, p1 = os.path.join(data["dir"], "anno.bed").encode(), os.path.join(data["dir"], "pass1.bed").encode()
    rng = np.random.default_rng(3)
    for step, (fn, flag, min_sc) in enumerate([(anno, J.MM_JUNC_ANNO, -1), (p1, 2, 5)]):
        assert R.mm_idx_jjump_read(rmi, fn, flag, min_sc) == 0
        assert L.mm_idx_jjump_read(C.byref(omi), fn, flag, min_sc) == 0
        n_total = 0
        for cid, s in enumerate(data["contigs"]):
            full = entries(R, rmi, cid, -1, len(s))
            assert entries(L, C.byref(omi), cid, -1, len(s)) == full
            n_total += len(full)
            assert len(set((e[0], e[1]) for e in full)) == len(full)
            for _ in range(300):
                st = int(rng.integers(-50, len(s) + 50))
                en = st + int(rng.integers(0, 2000)) if rng.random() < 0.9 else -1
                assert entries(L, C.byref(omi), cid, st, en) == entries(R, rmi, cid, st, en), (step, cid, st, en)
        assert n_total > 50
        if step == 0:  # the opposite-strand copies of an intron merge into one entry per end, whose strand is the replayed sort's
            assert any(e[2] > 1 for cid in range(len(data["contigs"])) for e in entries(R, rmi, cid, -1, 1 << 30))
    assert entries(L, C.byref(omi), len(data["contigs"]), 0, 100) == []  # contig id out of range


def test_missing_file_leaves_table(data):
    L = _setup(lib())
    omi = host_index(data)
    assert L.mm_idx_jjump_read(C.byref(omi), b"/nonexistent/anno.bed", 1, -1) == -1
    assert not omi.J


def _make_reg(h, qlen, rng):
    cig = h["cigar"]
    cap = len(cig) + 7
    cap = 1 << (cap - 1).bit_length()
    p = libc.malloc(cap * 4)
    ex = Extra.from_address(p)
    ex.capacity, ex.dp_score, ex.dp_max, ex.dp_max2, ex.dp_max0 = cap, int(rng.integers(50, 500)), int(rng.integers(50, 500)), 0, int(rng.integers(50, 500))
    ex.n_ambi_ts, ex.n_cigar = int(rng.integers(0, 3)) << 30, len(cig)
    (C.c_uint32 * len(cig)).from_address(p + C.sizeof(Extra))[:] = cig
    r = Reg1()
    r.id = r.parent = 0
    r.rid, r.rs, r.re, r.qs, r.qe = h["rid"], h["rs"], h["re"], h["qs"], h["qe"]
    r.blen = h["re"] - h["rs"]
    r.mlen = r.blen - int(rng.integers(0, 5))
    r.bits = 60 | h["rev"] << 10 | (int(len(cig) > 1) << 27)
    r.p = C.cast(p, C.POINTER(Extra))
    return r


def _reg_state(r):
    head = bytes(C.string_at(C.addressof(r), 72))
    ex = r.p.contents
    cig = list((C.c_uint32 * ex.n_cigar).from_address(C.addressof(ex) + C.sizeof(Extra)))
    return head, (ex.capacity, ex.dp_score, ex.dp_max, ex.dp_max2, ex.dp_max0, ex.n_ambi_ts, ex.n_cigar), cig


@pytest.mark.parametrize("jmm", [3, 5])
def test_split_matches_reference(data, jmm):
    R, L = _setup(O.ref()), _setup(lib())
    rmi, omi = ref_index(R, data), host_index(data)
    anno = os.path.join(data["dir"], "anno.bed").encode()
    assert R.mm_idx_jjump_read(rmi, anno, J.MM_JUNC_ANNO, -1) == 0
    assert L.mm_idx_jjump_read(C.byref(omi), anno, J.MM_JUNC_ANNO, -1) == 0
    io, mo = IdxOpt(), MapOpt()
    R.mm_set_opt(None, C.byref(io), C.byref(mo))
    assert R.mm_set_opt(b"splice", C.byref(io), C.byref(mo)) == 0
    mo.jump_min_match = jmm
    L.mmb_jump_apply.argtypes = [C.POINTER(MapOpt), C.c_int, C.POINTER(Reg1), C.c_void_p]
    from minimap2_b200.kernels import JumpDec
    tables = [[(e[0], e[1], e[4]) for e in entries(L, C.byref(omi), c, -1, len(s))] for c, s in enumerate(data["contigs"])]
    t4 = [J.NT4[np.frombuffer(s, dtype=np.uint8)] for s in data["contigs"]]
    rng = np.random.default_rng(17 + jmm)
    hits = J.hit_variants(data, rng)
    assert len(hits) > 1000
    n_changed, acts = 0, set()
    for h in hits:
        q = data["reads"][h["read"]][1]
        seed = int(rng.integers(0, 1 << 30))
        rr, orr = _make_reg(h, len(q), np.random.default_rng(seed)), _make_reg(h, len(q), np.random.default_rng(seed))
        before = _reg_state(rr)
        R.mm_jump_split(None, rmi, C.byref(mo), len(q), q, C.byref(rr), 0)
        left, right = J.decide(h, q, t4[h["rid"]], tables[h["rid"]], mo.a, mo.b, jmm)
        dec = JumpDec()
        for k, s in enumerate((left, right)):
            dec.side[k].act, dec.side[k].l, dec.side[k].off, dec.side[k].off2, dec.side[k].mm0 = s
        L.mmb_jump_apply(C.byref(mo), len(q), C.byref(orr), C.byref(dec))
        exp = _reg_state(rr)
        assert _reg_state(orr) == exp, (h, left, right)
        n_changed += exp != before
        acts.update((left[0], right[0]))
        libc.free(C.cast(rr.p, C.c_void_p)), libc.free(C.cast(orr.p, C.c_void_p))
    assert n_changed > 100 and {1, 2} <= acts, (n_changed, acts)
