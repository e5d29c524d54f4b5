"""CPU: the C restatement of the chainers in oracle/ against the reference's own functions on the generators and parameter edges of
tests/chain_cases.py, so that the chaining tests stay exact on a machine where only the restatement is built."""
import numpy as np
import pytest
import oracle_lib as O
import chain_cases as CC

pytestmark = pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")


@pytest.fixture(scope="module")
def reads():
    return CC.read_mix(np.random.default_rng(2024), n_noisy=40, n_huge=1)


def same(x, y):
    return len(x[0]) == len(y[0]) and (x[0] == y[0]).all() and x[1].shape == y[1].shape and (x[1] == y[1]).all()


def test_oracle_lchain_dp_edges(reads):
    for p in CC.DP_EDGES:
        for i, a in enumerate(reads):
            x = O.oracle_lchain_dp(a, p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"], p["min_sc"],
                                   p["pen_gap"], p["pen_skip"], p["is_cdna"])
            assert same(x, O.ref_lchain_dp(a, p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"],
                                           p["min_sc"], p["pen_gap"], p["pen_skip"], p["is_cdna"])), (p, i)


def test_oracle_lchain_rmq_edges(reads):
    for p in CC.RMQ_EDGES:
        for i, a in enumerate(reads):
            a = CC.y_zero(a)
            args = (p["max_dist"], p["max_dist_inner"], p["bw"], p["max_skip"], p["cap"], p["min_cnt"], p["min_sc"], p["pen_gap"], p["pen_skip"])
            assert same(O.oracle_lchain_rmq(a, *args), O.ref_lchain_rmq(a, *args)), (p, i)


def test_oracle_sort128_on_compacted_chains(reads):
    """the rescue's re-sort of compacted anchors, ties in x included"""
    for a in reads:
        _, b = O.ref_lchain_dp(a, 5000, 5000, 500, 25, 5000, 3, 40, CC.pen(0.8), 0.0)
        assert (O.oracle_sort128(b) == O.ref_sort128(b)).all()
