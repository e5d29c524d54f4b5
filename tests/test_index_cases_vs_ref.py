"""CPU: the oracle's index (oracle/mm2o_seed.c, the restatement of worker_post the index tests compare against) equals the reference's,
key by key, on every case of tests/index_cases.py: the reference's mm_idx_str read back through its mm_idx_dump and through mm_idx_get
for every key, and mm_idx_cal_max_occ at fractions on both sides of its truncation edges. The reference index's digest and mid_occ
values are recorded here (tests/golden/expected/reference_values.json) for the device tests."""
import ctypes as C
import numpy as np
import pytest
import oracle_lib as O
import index_cases as IC

pytestmark = pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")

SEED = 11


def ref_index(ctgs, w, k, is_hpc, tmp_path):
    R = O.ref()
    IC.setup(R)
    R.refshim_idx_get.restype = C.c_int
    R.refshim_idx_get.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int]
    mi = IC.build(R, ctgs, w, k, is_hpc)
    canon, = IC.parse_mmi(IC.dump(R, mi, tmp_path / "ref.mmi"))
    return R, mi, canon


@pytest.mark.parametrize("p", IC.PARAMS, ids=IC.PARAM_IDS)
def test_oracle_index_equals_reference(p, tmp_path):
    w, k, is_hpc = p
    ctgs = IC.contigs(w, k, is_hpc, SEED)
    R, mi, ref = ref_index(ctgs, w, k, is_hpc, tmp_path)
    exp = IC.oracle_canon(ctgs, w, k, is_hpc)
    exp.assert_equal(ref, "oracle vs the reference's dump")
    # mm_idx_get of every key, and of absent keys
    off, buf = exp.off(), np.zeros(int(exp.cnt.max()) if len(exp.cnt) else 1, dtype=np.uint64)
    for i, key in enumerate(exp.keys):
        n = R.refshim_idx_get(mi, int(key), buf.ctypes.data, len(buf))
        assert n == exp.cnt[i] and (buf[:n] == exp.pos[off[i]:off[i + 1]]).all(), (i, int(key))
    for key in IC.absent_keys(exp.keys, k, np.random.default_rng(1))[:2000]:
        assert R.refshim_idx_get(mi, int(key), buf.ctypes.data, len(buf)) == 0
    mo = {f: R.mm_idx_cal_max_occ(mi, f) for f in IC.f_values(len(exp.keys))}
    for f, v in mo.items():
        assert v == IC.max_occ(exp.cnt, f), (f, v)
    rec = IC.recorded(IC.case_name(w, k, is_hpc, SEED, 1.0), lambda: (ref, mo))
    assert rec["digest"] == ref.digest() and rec["n_keys"] == len(ref.keys)
    assert [[repr(f), v] for f, v in mo.items()] == rec["max_occ"]
    R.mm_idx_destroy(mi)
    # sanity of the case itself: the edges it is meant to reach
    assert int(exp.cnt.max()) >= 1000


@pytest.mark.parametrize("p", IC.PARTS_PARAMS)
def test_oracle_index_parts_equal_reference(p, tmp_path):
    """-I: the parts the reference's reader cuts (mini-batches of whole records, a part ends at the first mini-batch boundary past the
    batch size), each equal to the oracle's index of its contigs"""
    w, k, is_hpc = p
    seqs = IC.parts_fasta(tmp_path / "parts.fa", 9)
    R = O.ref()
    IC.setup(R)
    for mbs, bs in IC.PARTS_OPT:
        parts = IC.read_parts(R, tmp_path / "parts.fa", w, k, is_hpc, mbs, bs, tmp_path)
        assert len(parts) > 1 and sum(c.hdr[3] for c in parts) == len(seqs)
        for c in parts:
            IC.oracle_canon([seqs[n] for n in c.names], w, k, is_hpc, names=c.names).assert_equal(c, (mbs, bs))
        rec = O.reference_values(IC.parts_name(w, k, is_hpc, mbs, bs),
                                 lambda: dict(names=[c.names for c in parts], digests=[c.digest() for c in parts]))
        assert rec == dict(names=[c.names for c in parts], digests=[c.digest() for c in parts])
