"""GPU parity for K4 (finalize.cu): the per-hit tail of the alignment driver -- CIGAR stitching (mm_append_cigar), mm_fix_cigar and
mm_update_extra (align.c:105-334) -- through the C-ABI entry mmb_tail_batch_host against the oracle (oracle/mm2o_extra.c) and against
the committed outputs of the reference's own functions (tests/golden/vectors_tail.npz). Bit-exact: CIGAR words, blen, mlen, n_ambi,
dp_max, the coordinate shifts of a dropped leading gap."""
import os
import numpy as np
import pytest
import tail_cases as T

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vectors_tail.npz")


@pytest.fixture(scope="module")
def ctx():
    import minimap2_b200 as mb
    c = mb.Context(0)
    yield c
    c.close()


def test_tail_matches_oracle(ctx):
    import minimap2_b200 as mb
    rng = np.random.default_rng(77)
    cases = [T.make_case(rng) for _ in range(3000)]
    got = T.run_device(ctx, mb.lib(), cases)
    bad = [i for i, c in enumerate(cases) if not T.same(got[i], T.run_oracle(c))]
    assert not bad, bad[:10]


def test_tail_other_gap_costs(ctx):  # the logarithmic gap term with other q / e
    import minimap2_b200 as mb
    rng = np.random.default_rng(78)
    cases = [T.make_case(rng) for _ in range(500)]
    for q, e in ((6, 2), (5, 4), (16, 1)):
        got = T.run_device(ctx, mb.lib(), cases, q, e)
        bad = [i for i, c in enumerate(cases) if not T.same(got[i], T.run_oracle(c, q, e))]
        assert not bad, (q, e, bad[:10])


def test_tail_matches_reference_vectors(ctx):
    import minimap2_b200 as mb
    z = np.load(GOLD)
    rng = np.random.default_rng(int(z["seed"]))
    cases = [T.make_case(rng) for _ in range(int(z["n"]))]
    exp = T.unpack_results(z["stats"], z["cigars"])
    got = T.run_device(ctx, mb.lib(), cases)
    bad = [i for i in range(len(cases)) if not T.same(got[i], exp[i])]
    assert not bad, bad[:10]


def test_tail_long_hit(ctx):
    """hits of read scale: ~40 pieces and thousands of operations; and hits of a megabase read, with thousands of pieces and more than
    65,535 operations (stage 1's 32-piece groups and stage 2's 32-operation chunks carry state thousands of times), one of them
    without empty operations, all in one launch with short hits"""
    import minimap2_b200 as mb
    rng = np.random.default_rng(79)

    def stitched(n_parts, low_complexity, no_empty=False):
        parts = []
        while len(parts) < n_parts:
            p = T.make_case(rng, low_complexity=low_complexity)
            if not (no_empty and any((int(w) >> 4) == 0 for pc in p["pieces"] for w in pc)):
                parts.append(p)
        q = np.concatenate([p["qseq"] for p in parts]); t = np.concatenate([p["tseq"] for p in parts])
        pieces = [np.concatenate(p["pieces"]) if p["pieces"] else np.zeros(0, np.uint32) for p in parts]
        return dict(read=q, rev=0, qs=0, qseq=q, tseq=t, target=np.concatenate([t, np.zeros(16, np.uint8)]), t0=0, pieces=pieces, qspan=len(q), tspan=len(t))
    big = [stitched(40, False) for _ in range(8)]
    huge = [stitched(7000, True), stitched(7600, False, no_empty=True)]
    short = [T.make_case(rng) for _ in range(64)]
    cases = short[:32] + huge[:1] + short[32:] + huge[1:] + big
    got = T.run_device(ctx, mb.lib(), cases)
    for i, (g, c) in enumerate(zip(got, cases)):
        e = T.run_oracle(c)
        assert T.same(g, e), (i, len(c["pieces"]), e["n_cigar"])
    assert all(len(c["pieces"]) >= 2000 and T.run_oracle(c)["n_cigar"] > 65535 for c in huge)
