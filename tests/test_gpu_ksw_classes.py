"""GPU: every K3 launch class (tests/ksw_classes.py: 18 fast-path widths, 5 universal tiers for each of the dual-affine and spliced
passes, the ll kernel) against the oracle, bit-exact, one launch per batch, at the edges of each class, under every scoring regime
with its own code path, with batches larger than the resident workers (every worker takes a second, shorter job), and with a
workspace large enough that the 2 GiB bound shrinks the grid."""
import collections
import os
import numpy as np
import pytest
import ksw_classes as KC

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(KC.SMEM_MAXLEN_ENV in os.environ, reason="the tier bounds are lowered by " + KC.SMEM_MAXLEN_ENV)]

RUN = collections.Counter()  # jobs checked per class


@pytest.fixture(scope="module")
def ctx():
    import minimap2_b200 as mb
    c = mb.Context(0)
    yield c
    c.close()


def check(ctx, score, jobs, cls):
    import minimap2_b200 as mb
    RUN[cls] += KC.check_batch(mb.lib(), ctx.h, score, jobs, cls)


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("score", KC.REGIMES, ids=str)
def test_every_class_under_scoring(ctx, score):
    """each fast width and dual-affine tier the scoring can reach, and the ll kernel: edge shapes, one batch per class"""
    rng = np.random.default_rng(sum(map(ord, score.name)))
    for cls in KC.FAST_CLASSES + [c for c in KC.UNIV_CLASSES if c.startswith("extd2")] + ["ll"]:
        if KC.reachable(cls, score):
            check(ctx, score, KC.class_jobs(rng, cls, score), cls)


def test_packed_limit_routing():
    """2*max(q+e,q2+e2) + max|s| + 8 == 127 is the last scoring the packed kernel takes; 128 goes to the scalar kernel. (The device half:
    the JOB_ZDROP scan is only done by the packed kernel, and the batches above check it is there, or absent, per class.)"""
    assert KC.PK_LIMIT.pk_limit_sum()[0] == 127 and KC.PK_LIMIT.pk_ok()
    assert KC.PK_LIMIT_1.pk_limit_sum()[0] == 128 and not KC.PK_LIMIT_1.pk_ok()
    job = KC.make_job(np.zeros(100, np.uint8), np.zeros(100, np.uint8), flag=KC.APPROX)
    assert KC.is_packed(KC.route(job, KC.PK_LIMIT)) and not KC.is_packed(KC.route(job, KC.PK_LIMIT_1))


@pytest.mark.parametrize("score", [KC.MAP_ONT, KC.PK_LIMIT_1], ids=str)
def test_fast_one_and_two_jobs(ctx, score):
    """batches of one job and of two (which share a warp in the 16-lane packed classes)"""
    rng = np.random.default_rng(4)
    for cls in KC.FAST_CLASSES:
        if KC.reachable(cls, score):
            jobs = KC.fast_jobs(rng, int(cls[4:]), score, n_odd=False)
            check(ctx, score, jobs[-1:], cls)
            check(ctx, score, [jobs[0], jobs[-1]], cls)


def test_band_edge_of_fast_path(ctx):
    """w == max(qlen,tlen) is the narrowest band the fast path takes; w == max-1 goes to the universal kernel"""
    rng = np.random.default_rng(5)
    for tlen in (64, 200, 512):
        for qlen in (tlen - 3, tlen, tlen + 9):
            q, t = KC.related(rng, qlen, tlen, err=0.1)
            m = max(qlen, tlen)
            for w in (m, m - 1):
                job = KC.make_job(q, t, w=w, zdrop=400, flag=KC.APPROX | KC.JOB_ZDROP)
                cls = KC.route(job, KC.MAP_ONT)
                assert cls.startswith("fast") == (w == m), (qlen, tlen, w, cls)
                check(ctx, KC.MAP_ONT, [job], cls)


@pytest.mark.parametrize("score", KC.SPLICE_SCORINGS, ids=str)
def test_spliced_tiers(ctx, score):
    """ksw_exts2 in all five tiers, forward and reversed targets, both splice models"""
    rng = np.random.default_rng(sum(map(ord, score.name)))
    for k in range(KC.N_TIERS):
        for model in (KC.FLANK | KC.CMPLX, KC.FLANK):
            check(ctx, score, KC.exts2_jobs(rng, k, score, model), "exts2_t%d" % k)


@pytest.mark.parametrize("k", [3, 4])
def test_spliced_with_junctions(ctx, k):
    """annotated junctions (mmb_ctx_set_junctions) in the CTA tier and in the HBM-state tier, where their flags are OR-ed into the score
    row kept in HBM"""
    rng = np.random.default_rng(80 + k)
    score = KC.SPLICE_SCORINGS[0]
    jobs = KC.exts2_jobs(rng, k, score, KC.FLANK, with_junc=True)
    assert sum(len(j["introns"]) for j in jobs) >= 4
    changed = sum(KC.expected(j, score) != KC.expected(dict(j, introns=[]), score) for j in jobs)
    assert changed >= 1  # the annotation changes some of the expected results
    check(ctx, score, jobs, "exts2_t%d" % k)


def test_ll_more_jobs_than_groups(ctx):
    """ksw_ll_kernel with more jobs than its persistent groups (n_sm * 64): groups take several jobs"""
    rng = np.random.default_rng(6)
    jobs = KC.ll_jobs(rng, n_sm() * KC.LL_GROUPS_PER_SM + 37)
    check(ctx, KC.MAP_ONT, jobs, "ll")


def reuse_jobs(rng, cls, n_long, n_short):
    """n_long long jobs of one class, then n_short short ones. The queue runs longest first and n_long is at least the class's resident
    workers, so the first job of every worker is a long one, and each short job goes to a worker that has run a long job before it.
    The long jobs are long in the dimension that picks the class and modest in the other, which keeps the oracle cheap."""
    jobs = []
    if cls == "ll":
        for v in range(n_long + n_short):
            ql, tl = (int(rng.integers(48, 65)), int(rng.integers(100, 129))) if v < n_long else (int(rng.integers(1, 9)), int(rng.integers(1, 25)))
            q, t = KC.related(rng, ql, tl, err=0.15, n_frac=0.02 if v % 7 == 0 else 0.0)
            jobs.append(KC.make_job(q, t, w=4, zdrop=2, end_bonus=0, flag=KC.JOB_LL | (KC.T_COMP if v % 3 == 1 else 0), q_rev=v % 2 == 1))
        return jobs
    if cls.startswith("fast"):
        k = int(cls[4:]); lo, hi = KC.fast_lo(k), KC.fast_bound(k)
        for v in range(n_long + n_short):
            ql, tl = (int(rng.integers(48, 97)), hi) if v < n_long else (int(rng.integers(1, 7)), int(rng.integers(lo, (lo + hi) // 2 + 1)))
            q, t = KC.related(rng, ql, tl, err=0.1, n_frac=0.02 if v % 7 == 0 else 0.0)
            jobs.append(KC.make_job(q, t, w=-1, zdrop=400, flag=KC.APPROX | (KC.JOB_ZDROP if v % 2 else 0), q_rev=v % 3 == 1))
        return jobs
    k = KC.tier_of(cls); lo, hi = KC.tier_lo(k), min(KC.TIERS[k][0], 20000)
    for v in range(n_long + n_short):
        if v < n_long:
            m, ql = hi, min(hi, 32 if k < KC.N_TIERS - 1 else 16)
        else:
            m, ql = int(rng.integers(lo, lo + (hi - lo) // 4 + 1)), int(rng.integers(1, 9))
        q, t = KC.related(rng, ql, m, err=0.1)
        if v % 32:
            q, t = t, q  # the long side mostly on the query: the oracle's time grows with the target length times the rows
        jobs.append(KC.make_job(q, t, w=-1, zdrop=[400, -1][v % 2], end_bonus=-1, flag=[0, KC.EXT, KC.EXT | KC.RIGHT | KC.REVC][v % 3],
                                t_rev=v % 4 == 3, q_rev=v % 5 == 1))
    return jobs


def _reuse_cases():
    """one class of each family: the last 16-lane and the last 32-lane packed width, the last scalar width, the first and the last warp
    tier, the CTA tier, the HBM-state tier, and the ll kernel"""
    packed = range(KC.NS, KC.NC)
    warp = [k for k in range(KC.N_TIERS) if KC.TIERS[k][1] == 32]
    cta = [k for k in range(KC.N_TIERS - 1) if KC.TIERS[k][1] > 32]
    fast = [max(k for k in packed if KC.LNW[k] == 16), max(k for k in packed if KC.LNW[k] == 32), KC.NS - 1]
    return ([("fast%d" % k, KC.MAP_ONT if k >= KC.NS else KC.PK_LIMIT_1) for k in fast]
            + [("extd2_t%d" % k, KC.MAP_ONT) for k in sorted({warp[0], warp[-1], cta[0], KC.N_TIERS - 1})] + [("ll", KC.MAP_ONT)])


@pytest.mark.parametrize("cls,score", _reuse_cases(), ids=lambda x: str(x))
def test_worker_reuse(ctx, cls, score):
    """a batch larger than the resident-worker bound of its class, long jobs first: every worker goes on from a long job to short ones
    and must not see the shared memory or workspace state of the job before"""
    rng = np.random.default_rng(sum(map(ord, cls)))
    n = KC.resident_bound(cls, n_sm())
    check(ctx, score, reuse_jobs(rng, cls, n, n + 53), cls)


def test_workspace_bound_halves_grid(ctx):
    """the HBM-state tier with 20000 x 20000 jobs at w = 751: each worker's traceback rows alone take ~31 MB, so the grid is halved until
    the launch's workspace is within 2 GiB (ksw_extd2.cu:849) and the workers take the remaining jobs in turn"""
    rng = np.random.default_rng(7)
    jobs = []
    for v in range(3):
        t = KC.rand_seq(rng, 20000); q = KC.O.mutate(t, rng, err=0.05)[:20000]
        q = np.concatenate([q, KC.rand_seq(rng, 20000 - len(q))])
        jobs.append(KC.make_job(q, t, w=751, zdrop=-1, flag=[KC.EXT, 0, KC.EXT | KC.RIGHT | KC.REVC][v]))
    for v in range(70):
        q, t = KC.related(rng, int(rng.integers(1, 5)), 13001 + v, err=0.1)
        jobs.append(KC.make_job(q, t, w=-1, zdrop=400, flag=[0, KC.EXT][v % 2], t_rev=v % 3 == 0))
    # the host's bound on the traceback rows of one worker, and the HBM state of one worker (mmb_ksw_launch)
    maxp = max((len(j["q"]) + len(j["t"]) - 1) * (((min(len(j["q"]), len(j["t"]), (j["w"] if j["w"] >= 0 else 1 << 30) + 1) + 15) // 16 + 1) * 16) + 16
               for j in jobs)
    L = (max(len(j["t"]) for j in jobs) + 15) // 16 * 16; LQ = (max(len(j["q"]) for j in jobs) + 15) // 16 * 16
    gws = (16 * L + LQ + 64 + 1024 + 255) // 256 * 256
    assert min(len(jobs), n_sm()) * (maxp + gws) > 2 << 30
    check(ctx, KC.MAP_ONT, jobs, "extd2_t4")


def test_zz_every_class_exercised(request):
    """every class the routing mirror enumerates was run by the tests above (fails when a class is added without cases)"""
    names = {it.originalname for it in request.session.items if it.module is request.module}
    wanted = {n for n in dir(request.module) if n.startswith("test_") and n != "test_zz_every_class_exercised"}
    if not wanted <= names:
        pytest.skip("only part of this module was selected")
    missing = [c for c in KC.ALL_CLASSES if RUN[c] == 0]
    print("jobs per class:", dict(sorted(RUN.items())))
    assert not missing, missing
