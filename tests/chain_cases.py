"""Anchor sets and checkers for the chaining kernels (chain.cu), shared by the device tests and their emulated copies.

Anchors are the reference's: x = rev<<63 | rid<<32 | rpos, y = flags<<40 | span<<32 | qpos, sorted by x in radix_sort_128x's
order. The generators aim at the places where the warp-level DP, the backtrack and the rescue can part from the sequential
reference: per-anchor spans (1..255, often larger than the gap), the seed flag bits 40-43, dense collinear chains (windows of
hundreds of candidates, predecessor marks inside and beyond the current 32-wide chunk), tandem copies (ties in f, in x and in both
backtrack sorts), contigs whose x values lie closer than max_dist_x across the boundary, query positions at 0, anchor counts on the
warp and sort edges, and reads of more than 10^5 anchors.

Expected results come from the reference's own functions (mg_lchain_dp, mg_lchain_rmq, radix_sort_128x through oracle/_ref) when
that build is present; otherwise from the C restatement in oracle/, which tests/test_chain_cases_vs_ref.py holds equal to the
reference on these same generators."""
import numpy as np
import oracle_lib as O

FLAGS = [1 << 40, 1 << 41, 1 << 42, 1 << 43]  # MM_SEED_LONG_JOIN, _IGNORE, _TANDEM, _SELF
EDGE_COUNTS = [0, 1, 2, 31, 32, 33, 64, 65, 66]


def pen(scale, k=15):
    """a chaining penalty as map.c computes it: float scale * 0.01 * k in double, stored as float"""
    return float(np.float32(float(np.float32(scale)) * 0.01 * k))


def _rows(rng, rid, rev, r0, q0, n, step=(1, 3), jitter=0.0, spans=(1, 255), flags=True):
    rows = []
    q, r = q0, r0
    for _ in range(n):
        sp = int(rng.integers(spans[0], spans[1] + 1))
        fl = sum(f for f in FLAGS if rng.random() < 0.15) if flags else 0
        rows.append(((rev << 63) | (rid << 32) | (r & 0xffffffff), fl | (sp << 32) | (q & 0xffffffff)))
        st = int(rng.integers(step[0], step[1] + 1))
        q += st
        r += st + (int(rng.integers(-4, 5)) if rng.random() < jitter else 0)
    return rows


def _sorted(rows):
    a = np.array(rows, dtype=np.uint64).reshape(-1, 2)
    return O.oracle_sort128(a)


def dense_chain(rng, n=600, q0=None):
    """one collinear chain with steps of 1..3 bases, plus a second copy shifted on the reference (predecessors both near and far)"""
    q0 = int(rng.integers(0, 3)) if q0 is None else q0
    r0 = int(rng.integers(1000, 50000))
    rows = _rows(rng, 0, 0, r0, q0, n, jitter=0.05)
    rows += _rows(rng, 0, 0, r0 + int(rng.integers(200, 400)), q0 + 5, n // 3, step=(1, 3), jitter=0.2)
    return _sorted(rows)


def tandem(rng, copies=12, n=80):
    """one query stretch hit at many reference positions (equal f, equal y), and one reference stretch hit by several query
    positions (runs of equal x)"""
    rows = []
    r0, q0, period = int(rng.integers(1000, 9000)), int(rng.integers(0, 50)), int(rng.integers(30, 120))
    base = _rows(rng, 1, 0, r0, q0, n, step=(2, 6), spans=(15, 15), flags=False)
    for c in range(copies):  # same query positions, reference shifted by one period per copy
        rows += [(x + c * period, y) for x, y in base]
    for c in range(1, 4):  # same reference positions, query shifted
        rows += [(x, y + c * period) for x, y in base[: n // 2]]
    return _sorted(rows)


def multi_contig(rng, n=300):
    """chains on several contigs and both strands; contigs 2 and 3 meet where rid 2 ends near 2^32, so x across the boundary
    differs by less than max_dist_x"""
    rows = []
    for rid, rev in [(0, 0), (0, 1), (1, 0), (1, 1)]:
        rows += _rows(rng, rid, rev, int(rng.integers(100, 20000)), int(rng.integers(0, 100)), n // 4, step=(5, 60), jitter=0.3)
    top = (1 << 32) - int(rng.integers(200, 1500))
    rows += _rows(rng, 2, 0, top, 10, 40, step=(5, 30))
    rows = [(x, y) for x, y in rows if (x >> 32) != 2 or (x & 0xffffffff) >= top]  # no wrap inside rid 2
    rows += _rows(rng, 3, 0, int(rng.integers(0, 50)), 400, 40, step=(5, 30))
    return _sorted(rows)


def equal_f_scatter(rng, n=300):
    """anchors 1..30 bases apart on one contig with random query positions and one span: few of them chain, so most share
    f = span. When max_ii falls out of max_dist_x, its recomputation meets many equal f and must keep the largest j; under a
    small max_iter the anchors that follow reach it only through the max_ii shortcut"""
    rows, x = [], int(rng.integers(1000, 5000))
    for _ in range(n):
        x += int(rng.integers(1, 31))
        rows.append((x, (15 << 32) | int(rng.integers(0, 2000))))
    return _sorted(rows)


def noisy_chains(rng, n_chain=3, n_noise=200, qlen=6000):
    """sparse chains with gaps of 1..150 and random spans, plus noise anywhere (the shape of real seed hits)"""
    rows = []
    for _ in range(n_chain):
        rid, rev = int(rng.integers(0, 3)), int(rng.integers(0, 2))
        q, r = int(rng.integers(0, 200)), int(rng.integers(1000, 100000))
        while q < qlen:
            sp = int(rng.integers(1, 256))
            rows.append(((rev << 63) | (rid << 32) | r, sum(f for f in FLAGS if rng.random() < 0.1) | (sp << 32) | q))
            st = int(rng.integers(1, 150))
            q += st
            r += st + (int(rng.integers(-8, 9)) if rng.random() < 0.3 else 0)
    for _ in range(n_noise):
        rows.append(((int(rng.integers(0, 2)) << 63) | (int(rng.integers(0, 3)) << 32) | int(rng.integers(0, 200000)),
                     (int(rng.integers(1, 256)) << 32) | int(rng.integers(0, qlen))))
    return _sorted(rows) if rows else np.zeros((0, 2), dtype=np.uint64)


def with_count(rng, n):
    """exactly n anchors from a dense chain with some noise (warp-chunk edges at 32/64, insertion/radix sort edge at 64/65)"""
    if n == 0:
        return np.zeros((0, 2), dtype=np.uint64)
    a = np.concatenate([dense_chain(rng, n=max(n, 8)), noisy_chains(rng, 1, n)])
    keep = np.sort(rng.choice(len(a), n, replace=False))
    return _sorted([tuple(int(v) for v in r) for r in a[keep]])


def huge(rng, n=110_000):
    """more than 10^5 anchors: many dense chains over several contigs (deep radix levels, a large per-read sort stack)"""
    rows = []
    while len(rows) < n:
        rows += _rows(rng, int(rng.integers(0, 8)), int(rng.integers(0, 2)), int(rng.integers(0, 1 << 30)), int(rng.integers(0, 100)),
                      int(rng.integers(500, 4000)), step=(1, 12), jitter=0.1)
    return _sorted(rows[:n])


def y_zero(a):
    """a copy with the first anchors' y set to 0 (query position 0, span 0, no flags)"""
    a = a.copy()
    a[: min(3, len(a)), 1] = 0
    return _sorted([tuple(int(v) for v in r) for r in a])


def read_mix(rng, n_noisy=24, n_huge=0, scale=1.0):
    """one batch with every read shape above; scale shrinks the dense and tandem reads (the emulated tests)"""
    reads = [with_count(rng, n) for n in EDGE_COUNTS]
    reads += [dense_chain(rng, n=int(600 * scale)), dense_chain(rng, n=int(1500 * scale), q0=0), tandem(rng, n=int(80 * scale)),
              tandem(rng, copies=int(40 * scale), n=40), multi_contig(rng), equal_f_scatter(rng), equal_f_scatter(rng, n=int(1000 * scale))]
    reads += [noisy_chains(rng, int(rng.integers(0, 5)), int(rng.integers(0, 400))) for _ in range(n_noisy)]
    reads += [huge(rng) for _ in range(n_huge)]
    order = rng.permutation(len(reads))
    return [reads[i] for i in order]


# ---- expected results --------------------------------------------------------------------------------------------------------

def _fn(name):
    return getattr(O, ("ref_" if O.have_ref() else "oracle_") + name)


def expect_dp(a, p):
    """p: dict of mg_lchain_dp's arguments (max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc, pen_gap, pen_skip, is_cdna)"""
    return _fn("lchain_dp")(a, p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"], p["min_sc"],
                            p["pen_gap"], p["pen_skip"], p["is_cdna"])


def expect_rmq(a, p):
    """p: dict of mg_lchain_rmq's arguments (max_dist, max_dist_inner, bw, max_skip, cap, min_cnt, min_sc, pen_gap, pen_skip)"""
    return _fn("lchain_rmq")(a, p["max_dist"], p["max_dist_inner"], p["bw"], p["max_skip"], p["cap"], p["min_cnt"], p["min_sc"],
                             p["pen_gap"], p["pen_skip"])


def rescue_selected(u, b, qlen, rescue_size, rescue_ratio):
    """map.c:283-285 on a first-round result: more than one chain, and the best chain leaves more than rescue_size query bases
    unchained or spans more than qlen * rescue_ratio (a float product)"""
    if len(u) <= 1:
        return False
    st, en = int(np.int32(np.uint32(b[0, 1] & 0xffffffff))), int(np.int32(np.uint32(b[int(u[0] & 0xffffffff) - 1, 1] & 0xffffffff)))
    return qlen - (en - st) > rescue_size or np.float32(en - st) > np.float32(qlen) * np.float32(rescue_ratio)


def best_span(u, b):
    """en - st of the first chain, as map.c:284 computes it"""
    return int(np.int32(np.uint32(b[int(u[0] & 0xffffffff) - 1, 1] & 0xffffffff))) - int(np.int32(np.uint32(b[0, 1] & 0xffffffff)))


def first_round(a, p):
    """p: the first chainer's parameters, as a dict for expect_rmq (when p['use_rmq']) or expect_dp"""
    return expect_rmq(a, p) if p.get("use_rmq") else expect_dp(a, p)


def expect_rescue(a, qlen, p, r):
    """map.c:275-291 composed from the reference's functions: the first chainer, then, for a selected read, radix_sort_128x over
    the compacted anchors and mg_lchain_rmq at bw_long. r: bw_long, rescue_size, rescue_ratio, max_dist, max_dist_inner, cap.
    Returns (u, b, rescued)."""
    u, b = first_round(a, p)
    if not rescue_selected(u, b, qlen, r["rescue_size"], r["rescue_ratio"]):
        return u, b, False
    s = _fn("sort128")(b)
    u, b = _fn("lchain_rmq")(s, r["max_dist"], r["max_dist_inner"], r["bw_long"], p["max_skip"], r["cap"], p["min_cnt"], p["min_sc"],
                             p["pen_gap"], p["pen_skip"])
    return u, b, True


def assert_same(got, exp, what):
    """got, exp: (u, anchors) of one read; any difference fails, with the first differing chain or anchor named"""
    gu, ga = got
    eu, ea = exp
    assert len(gu) == len(eu), "%s: %d chains, expected %d" % (what, len(gu), len(eu))
    d = np.nonzero(gu != eu)[0]
    assert len(d) == 0, "%s: chain %d u=%#x, expected %#x" % (what, d[0], int(gu[d[0]]), int(eu[d[0]]))
    assert ga.shape == ea.shape, "%s: %d anchors, expected %d" % (what, len(ga), len(ea))
    d = np.nonzero((ga != ea).any(axis=1))[0]
    assert len(d) == 0, "%s: anchor %d (%#x, %#x), expected (%#x, %#x)" % (what, d[0], *map(int, ga[d[0]]), *map(int, ea[d[0]]))


def check_all(got, reads, expect, what):
    """compare every read of a batch; returns the number of chains seen, so callers can check a case was not vacuous"""
    n_chains = 0
    for i, a in enumerate(reads):
        e = expect(a)
        assert_same(got[i], e[:2], "%s read %d (%d anchors)" % (what, i, len(a)))
        n_chains += len(e[0])
    return n_chains


# ---- parameter sets ----------------------------------------------------------------------------------------------------------

def dp_par(**kw):
    """map-ont's chaining parameters (k = 15), with overrides"""
    p = dict(max_dist_x=5000, max_dist_y=5000, bw=500, max_skip=25, max_iter=5000, min_cnt=3, min_sc=40, pen_gap=pen(0.8), pen_skip=0.0, is_cdna=0)
    p.update(kw)
    return p


def rmq_par(**kw):
    """asm5's first chainer (mg_lchain_rmq), with overrides"""
    p = dict(use_rmq=1, max_dist=5000, max_dist_inner=1000, bw=500, max_skip=25, cap=100000, min_cnt=3, min_sc=40, pen_gap=pen(0.8), pen_skip=0.0)
    p.update(kw)
    return p


def chain_par(p):
    """the ChainPar of a dp_par()/rmq_par() dict, as map.cu fills it"""
    from minimap2_b200._lib import ChainPar
    if p.get("use_rmq"):
        return ChainPar(p["max_dist"], p["max_dist"], p["bw"], p["max_skip"], 5000, p["min_cnt"], p["min_sc"], p["pen_gap"], p["pen_skip"],
                        0, 1, 1, p["max_dist_inner"], p["cap"])
    return ChainPar(p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"], p["min_sc"], p["pen_gap"],
                    p["pen_skip"], p["is_cdna"], 1, 0, 0, 0)


def rescue_par(r):
    from minimap2_b200._lib import RescuePar
    return RescuePar(r["bw_long"], r["rescue_size"], r["rescue_ratio"], r["max_dist"], r["max_dist_inner"], r["cap"])


# DP edges: max_skip and max_iter across the warp width and the early exits, small bw (candidates rejected by dd > bw, chains cut
# by bk_end's max_drop = bw), max_dist_x below bw (raised to bw), cDNA with max_dist_y on both sides of bw, skip penalties
DP_EDGES = [dp_par(max_skip=s) for s in (0, 1, 2, 31, 32, 33)] + \
    [dp_par(max_iter=m) for m in (-1, 0, 1, 2, 31, 32, 33, 64)] + \
    [dp_par(max_dist_x=300, max_dist_y=300, bw=300, max_iter=2, min_cnt=2, min_sc=20),
     dp_par(max_dist_x=300, max_dist_y=300, bw=300, max_iter=3, max_skip=0, min_cnt=2, min_sc=20),
     dp_par(max_skip=0, max_iter=1), dp_par(max_skip=1, max_iter=33, pen_skip=pen(1)), dp_par(max_skip=32, max_iter=0, pen_skip=pen(0.5)),
     dp_par(max_iter=-1, pen_skip=pen(3)),
     dp_par(bw=20), dp_par(bw=8, max_skip=2), dp_par(max_dist_x=30, max_dist_y=30, bw=50), dp_par(max_dist_x=10, max_dist_y=4000, bw=200),
     dp_par(max_dist_x=200000, max_dist_y=100, bw=500, is_cdna=1, min_sc=20), dp_par(max_dist_x=200000, max_dist_y=2000, bw=500, is_cdna=1),
     dp_par(pen_skip=pen(0.5)), dp_par(pen_skip=pen(1)), dp_par(pen_skip=pen(3), max_skip=2)]

# RMQ edges: a tree cap small enough to evict, max_dist_inner 0 / negative / above max_dist (the clamps), skip penalties
RMQ_EDGES = [rmq_par(cap=12), rmq_par(cap=64, max_skip=2), rmq_par(max_dist_inner=0), rmq_par(max_dist_inner=-5),
             rmq_par(max_dist_inner=20000), rmq_par(pen_skip=pen(1)), rmq_par(max_dist=300, max_dist_inner=300, bw=100, max_skip=0),
             rmq_par(bw=20, pen_skip=pen(3), min_cnt=2, min_sc=20)]


def score_edges(reads, p):
    """min_sc / min_cnt values that put chains exactly on the keep/drop edge: the median chain's score and anchor count under p,
    as (kept, dropped) parameter sets"""
    sc, cnt = [], []
    for a in reads:
        u, _ = expect_dp(a, p)
        sc += [int(x >> 32) for x in u]
        cnt += [int(x & 0xffffffff) for x in u]
    s, c = int(np.median(sc)), int(np.median(cnt))
    return dict(p, min_sc=s, min_cnt=c), dict(p, min_sc=s + 1, min_cnt=c + 1)


def rescue_qlens(rng, reads, p, r):
    """per-read query lengths on the rescue's edges: qlen - (en - st) equal to rescue_size and one more, and (en - st) just under
    and just over qlen * rescue_ratio in float; reads with fewer than two chains get random lengths"""
    ql = []
    for i, a in enumerate(reads):
        u, b = first_round(a, p)
        if len(u) < 2:
            ql.append(int(rng.integers(100, 20000)))
            continue
        L = best_span(u, b)
        kind = i % 5
        if kind == 0:
            ql.append(r["rescue_size"] + L)          # not selected by size
        elif kind == 1:
            ql.append(r["rescue_size"] + L + 1)      # selected by size
        elif kind in (2, 3):                          # the smallest qlen with L <= qlen * ratio, and the one below it
            q = max(int(L / r["rescue_ratio"]) - 3, 1)
            while np.float32(L) > np.float32(q) * np.float32(r["rescue_ratio"]):
                q += 1
            ql.append(q if kind == 2 else q - 1)
        else:
            ql.append(int(rng.integers(max(L, 1), 4 * max(L, 1) + 2)))
    return ql
