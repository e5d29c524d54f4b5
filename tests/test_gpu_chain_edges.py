"""GPU: the chaining kernels at their parameter edges against the reference chainers (tests/chain_cases.py). Every configuration
runs as one batch that mixes all the read shapes, reads of more than 10^5 anchors included, so the reads also share scratch and
sort stacks as they do in the mapper.
  DP (chain_fill_kernel + backtrack + compaction) vs mg_lchain_dp: max_skip and max_iter across the warp width (max_iter 0 and -1
  included), small bw, max_dist_x < bw, cDNA, skip penalties, min_sc / min_cnt on the keep/drop edge.
  RMQ (chain_rescue_kernel as the first chainer) vs mg_lchain_rmq: evicting tree caps, the max_dist_inner clamps, y = 0.
  Long-join rescue (mmb_chain_rescue_batch_host: the mapper's chaining stage) vs mg_lchain_dp / mg_lchain_rmq, radix_sort_128x and
  mg_lchain_rmq at bw_long composed as map.c:275-291 does, with query lengths on both sides of the selection rule."""
import numpy as np
import pytest
import chain_cases as CC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import minimap2_b200 as mb
    c = mb.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def reads():
    return CC.read_mix(np.random.default_rng(2024), n_noisy=40, n_huge=2)


def run_dp(ctx, reads, p):
    from minimap2_b200 import kernels as K
    return K.chain_batch(ctx, reads, p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"], p["min_sc"],
                         p["pen_gap"], p["pen_skip"], p["is_cdna"])


def run_rmq(ctx, reads, p):
    from minimap2_b200 import kernels as K
    return K.chain_rmq_batch(ctx, reads, p["max_dist"], p["max_dist_inner"], p["bw"], p["max_skip"], p["cap"], p["min_cnt"], p["min_sc"],
                             p["pen_gap"], p["pen_skip"])


@pytest.mark.parametrize("i", range(len(CC.DP_EDGES)))
def test_chain_dp_edges(ctx, reads, i):
    p = CC.DP_EDGES[i]
    assert CC.check_all(run_dp(ctx, reads, p), reads, lambda a: CC.expect_dp(a, p), str(p)) > 0


def test_chain_dp_score_edges(ctx, reads):
    for p in CC.score_edges(reads[:30], CC.dp_par(max_iter=64)):
        assert CC.check_all(run_dp(ctx, reads, p), reads, lambda a: CC.expect_dp(a, p), str(p)) > 0


@pytest.mark.parametrize("i", range(len(CC.RMQ_EDGES)))
def test_chain_rmq_edges(ctx, reads, i):
    p = CC.RMQ_EDGES[i]
    rs = [CC.y_zero(a) for a in reads]
    assert CC.check_all(run_rmq(ctx, rs, p), rs, lambda a: CC.expect_rmq(a, p), str(p)) > 0


RESCUES = [  # (first chainer, rescue): selection by size only, by ratio only, map-ont's rule, and an RMQ first chainer (asm)
    (CC.dp_par(), dict(bw_long=20000, rescue_size=1000, rescue_ratio=2.0, max_dist=5000, max_dist_inner=1000, cap=100000)),
    (CC.dp_par(max_iter=0), dict(bw_long=20000, rescue_size=10 ** 8, rescue_ratio=0.8, max_dist=5000, max_dist_inner=1000, cap=100000)),
    (CC.dp_par(bw=100, pen_skip=CC.pen(1)), dict(bw_long=5000, rescue_size=1000, rescue_ratio=0.1, max_dist=3000, max_dist_inner=0, cap=64)),
    (CC.rmq_par(), dict(bw_long=20000, rescue_size=1000, rescue_ratio=0.3, max_dist=5000, max_dist_inner=1000, cap=100000)),
]


@pytest.mark.parametrize("i", range(len(RESCUES)))
def test_chain_rescue(ctx, reads, i):
    from minimap2_b200 import kernels as K
    p, r = RESCUES[i]
    rng = np.random.default_rng(77 + i)
    rs = reads + [CC.tandem(rng, copies=3, n=200) for _ in range(6)]  # two or three chains with equal x among the compacted anchors
    ql = CC.rescue_qlens(rng, rs, p, r)
    got = K.chain_rescue_batch(ctx, rs, ql, CC.chain_par(p), CC.rescue_par(r))
    n_rescued = n_kept = 0
    for k, a in enumerate(rs):
        u, b, rescued = CC.expect_rescue(a, ql[k], p, r)
        CC.assert_same(got[k], (u, b), "rescue %d read %d (%d anchors, qlen %d, rescued %d)" % (i, k, len(a), ql[k], rescued))
        n_rescued += rescued
        n_kept += not rescued
    assert n_rescued > 0 and n_kept > 0, (n_rescued, n_kept)
