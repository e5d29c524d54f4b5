"""GPU parity of the index build (DESIGN rows f1 and f3) on every build path of tests/index_cases.py: mm_idx_str on the device against
the oracle and the reference's recorded digest, key by key (dump, device-table probe, absent keys, wrap-around), mm_idx_cal_max_occ
against the reference's recorded values, dump -> load -> dump, and the seeding stage on an HPC index."""
import ctypes as C
import numpy as np
import pytest
import index_cases as IC
import oracle_lib as O
import seed_check as SC
import synth

pytestmark = pytest.mark.gpu

SEED = 11  # the cases of tests/test_index_cases_vs_ref.py, whose reference values are recorded


@pytest.fixture(scope="module")
def dev():
    import minimap2_b200 as mb
    from minimap2_b200._lib import lib
    L = lib()
    IC.setup(L)
    SC.setup(L)
    c = mb.Context(0)
    yield L, C.c_void_p(c.h)
    c.close()


def _ref_canon(ctgs, w, k, is_hpc, tmp_path):
    R = O.ref()
    IC.setup(R)
    mi = IC.build(R, ctgs, w, k, is_hpc)
    c, = IC.parse_mmi(IC.dump(R, mi, tmp_path / "ref.mmi"))
    mo = {f: R.mm_idx_cal_max_occ(mi, f) for f in IC.f_values(len(c.keys))}
    R.mm_idx_destroy(mi)
    return c, mo


@pytest.mark.parametrize("p", IC.PARAMS, ids=IC.PARAM_IDS)
def test_index_build_matches_reference(dev, p, tmp_path):
    w, k, is_hpc = p
    L, _ = dev
    ctgs = IC.contigs(w, k, is_hpc, SEED)
    rec = IC.recorded(IC.case_name(w, k, is_hpc, SEED, 1.0), lambda: _ref_canon(ctgs, w, k, is_hpc, tmp_path))
    mo = {float(f): v for f, v in rec["max_occ"]}
    exp, wrapped = IC.check_device_index(L, ctgs, w, k, is_hpc, tmp_path, max_occ_values=mo)
    assert exp.digest() == rec["digest"] and len(exp.keys) == rec["n_keys"]
    assert wrapped == IC.wraps(exp.keys, k)


@pytest.mark.parametrize("fx", IC.REF_MMI, ids=[f[0] for f in IC.REF_MMI])
def test_load_of_reference_mmi(dev, fx, tmp_path):
    """a .mmi the reference wrote (HPC; even k with b = 2k < 14) loads and probes as the oracle's index of the same sequence"""
    IC.check_reference_mmi(dev[0], *fx, tmp_path)


@pytest.mark.parametrize("p", IC.PARTS_PARAMS)
def test_index_parts_match_reference(dev, p, tmp_path):
    """-I: mm_idx_reader_read's parts (idx_gen's mini-batch rule) against the reference's recorded parts"""
    IC.check_parts(dev[0], *p, tmp_path)


def test_index_of_many_contigs_and_a_long_repeat(dev, tmp_path):
    """10^4 tiny contigs next to 2 Mbp with repeats, under the default and the HPC sketch"""
    L, _ = dev
    rng = np.random.default_rng(4)
    ctgs = [bytes(synth.ALPHA[rng.integers(0, 4, int(n))]) for n in rng.integers(0, 60, 10_000)]
    ctgs += [bytes(c) for c in synth.random_genome(2_000_000, 4, n_contigs=3, repeat_frac=0.5)]
    for w, k, is_hpc in ((10, 15, 0), (10, 19, 1), (10, 14, 0)):
        IC.check_device_index(L, ctgs, w, k, is_hpc, tmp_path)


@pytest.mark.parametrize("cfg", [dict(w=10, k=19), dict(w=5, k=19, mid_occ=30), dict(w=10, k=15)])
def test_hpc_seed_stage_matches_oracle(dev, cfg):
    """the seeding stage with an HPC index: seed spans differ from k in the query sketch, the lookups and the anchors"""
    L, ctx = dev
    contigs, reads = SC.repeat_rich_case(7, 300_000, 60, 4000, rep=0.35, n_contigs=3)
    rng = np.random.default_rng(7)
    hp = [IC._hpc_runs(rng, 1500, 60) for _ in range(6)]
    contigs.append(np.frombuffer(b"".join(hp), dtype=np.uint8))
    reads += [h[100:2500] for h in hp]
    st = SC.check_case(L, ctx, contigs, reads, is_hpc=1, **cfg)
    assert st["anchors"] > 10_000


def test_index_of_a_200_mbp_genome(dev, tmp_path):
    """the 200 Mbp synthetic genome of mmb_synth_index, written out with mmb_idx_write_fasta: its index against the oracle's"""
    L, _ = dev
    L.mmb_synth_index.restype = C.c_void_p
    L.mmb_synth_index.argtypes = [C.c_uint64, C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int]
    L.mmb_idx_write_fasta.argtypes = [C.c_void_p, C.c_char_p]
    mi = L.mmb_synth_index(200_000_000, 24, 5, 10, 15, IC.BUCKET_BITS)
    assert L.mmb_idx_write_fasta(mi, str(tmp_path / "g.fa").encode()) == 0
    names, seqs = IC.read_fasta(tmp_path / "g.fa")
    exp = IC.oracle_canon(seqs, 10, 15, 0, names=names)
    got, = IC.parse_mmi(IC.dump(L, mi, tmp_path / "g.mmi"))
    exp.assert_equal(got, "200 Mbp")
    IC.check_lookup(L, mi, exp, 15, np.random.default_rng(8))
    L.mm_idx_destroy(mi)


@pytest.mark.parametrize("p", [(10, 15, 0)], ids=["w10k15"])
def test_contigs_past_2g_in_S(dev, p, tmp_path):
    """(odd k: the chunk-replay sketch kernel is quadratic inside long N stretches, DESIGN section 7) two leading all-N contigs of 2^30 + 2 and 2^30 + 3 bases, so that every later contig starts past 2^31 in S (the reference sketches
    a contig's length as an int, so one contig of more than 2^31 - 1 bases is not an input it can index)"""
    w, k, is_hpc = p
    L, _ = dev
    head = [b"N" * ((1 << 30) + 2), b"N" * ((1 << 30) + 3)]
    tail = IC.contigs(w, k, is_hpc, 3, scale=0.2)
    names = IC.names_of(head + tail)
    exp = IC.oracle_canon([b"", b""] + tail, w, k, is_hpc, names=names)  # rids as in the full index; the N contigs have no minimizers
    mi = IC.build(L, head + tail, w, k, is_hpc, names=names)
    got, = IC.parse_mmi(IC.dump(L, mi, tmp_path / "big.mmi"))
    assert got.names == names and list(got.lens) == [len(c) for c in head + tail]
    assert (got.keys == exp.keys).all() and (got.cnt == exp.cnt).all() and (got.pos == exp.pos).all()
    S_tail = IC.pack_S([b"N" * 5] + tail)  # 2^31 is a multiple of 8 bases: S words from 2^28 on hold five N codes, then the tail
    assert (got.S[1 << 28:] == S_tail).all()
    IC.check_lookup(L, mi, exp, k, np.random.default_rng(9))
    L.mm_idx_destroy(mi)
