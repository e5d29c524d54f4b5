"""CPU: one or two edge jobs of every K3 launch class (tests/ksw_classes.py) through the SIMT emulator, with the same one-launch and
oracle checks as tests/test_gpu_ksw_classes.py, so that a routing or width regression fails without a GPU."""
import os
import numpy as np
import pytest
import ksw_classes as KC

pytestmark = pytest.mark.skipif(KC.SMEM_MAXLEN_ENV in os.environ, reason="the tier bounds are lowered by " + KC.SMEM_MAXLEN_ENV)


@pytest.fixture(scope="module")
def emu():
    import test_emu_ksw as E
    return E.load_emu()


def small_edge_jobs(rng, cls, score):
    """the class's lower and upper edge, the long side only: the emulator runs one OS thread per CUDA thread"""
    if cls == "ll":
        return KC.ll_jobs(rng, 3)
    if cls.startswith("fast"):
        k = int(cls[4:])
        lo, hi = KC.fast_lo(k), KC.fast_bound(k)
        out = []
        for v, (ql, tl) in enumerate(((1 if k % 2 else 9, lo), (int(rng.integers(4, 40)), hi))):
            q, t = KC.related(rng, ql, tl, err=0.1, n_frac=0.05)
            out.append(KC.make_job(q, t, w=[-1, max(ql, tl)][v], zdrop=400, flag=KC.APPROX | KC.JOB_ZDROP | (KC.GENERIC if score.generic else 0),
                                   q_rev=v == 1, t_rev=k % 3 == 0))
        return out
    k = KC.tier_of(cls)
    lo, hi = KC.tier_lo(k), KC.TIERS[k][0]
    out = []
    for v, m in enumerate((lo, hi)):
        q, t = KC.related(rng, int(rng.integers(1, 6)), m, err=0.1, n_frac=0.02)
        if v:
            q, t = t, q  # the long side on the query
        flag = [0, KC.EXT | KC.RIGHT | KC.REVC][v]
        if cls.startswith("exts2"):
            out.append(KC.make_job(q, t, zdrop=200, flag=flag | KC.SPF | KC.FLANK | KC.JOB_SPLICE, t_rev=v == 1))
        else:
            out.append(KC.make_job(q, t, w=[-1, 17][v], zdrop=200, flag=flag | KC.T_COMP * v, q_rev=v == 0))
    return out


# the warp tiers only: the CTA tier and the HBM-state tier take minutes here (the latter runs in test_emu_ksw.test_emulated_hbm_state_tier)
EMU_CLASSES = [c for c in KC.ALL_CLASSES if c.startswith("fast") or c == "ll" or KC.TIERS[KC.tier_of(c)][1] == 32]


@pytest.mark.parametrize("score", [KC.MAP_ONT, KC.PK_LIMIT, KC.PK_LIMIT_1], ids=str)
def test_emulated_class_edges(emu, score):
    L, ctx = emu[0], emu[1]
    rng = np.random.default_rng(sum(map(ord, score.name)))
    n_cls = 0
    for cls in EMU_CLASSES:
        if not KC.reachable(cls, score) or (score is not KC.MAP_ONT and not cls.startswith("fast")):
            continue  # the universal and ll kernels do not depend on the packed kernel's limit
        sc = KC.SPLICE_SCORINGS[0] if cls.startswith("exts2") else score
        KC.check_batch(L, ctx, sc, small_edge_jobs(rng, cls, sc), cls)
        n_cls += 1
    assert n_cls == (KC.NC - KC.NS if score.pk_ok() else KC.NS) + (len(EMU_CLASSES) - KC.NC if score is KC.MAP_ONT else 0)


def test_emulated_scan_of_ambiguous_bases(emu):
    """ambiguous bases under --score-N 0 and 2. With a 0 matrix entry the DP scores them -e2 (ksw2_extd2_sse.c:87), in the packed and the
    universal kernel, while the packed kernel's z-drop scan keeps the matrix entry, as mm_test_zdrop does (align.c:61-89)"""
    L, ctx = emu[0], emu[1]
    rng = np.random.default_rng(11)
    for name in ("sc_ambi0", "sc_ambi2"):
        score = [s for s in KC.REGIMES if s.name == name][0]
        for cls, flag in (("fast%d" % KC.NS, KC.APPROX | KC.JOB_ZDROP), ("extd2_t0", 0), ("extd2_t0", KC.EXT)):
            jobs = []
            for v in range(5):
                q, t = KC.related(rng, int(rng.integers(30, 120)), 64, err=0.1, n_frac=0.15)
                jobs.append(KC.make_job(q, t, w=-1 if cls != "extd2_t0" else 40, zdrop=400, flag=flag))
            KC.check_batch(L, ctx, score, jobs, cls)


@pytest.mark.parametrize("name", ["swapped-gaps", "asm5-swapped"])
def test_emulated_swapped_gap_costs(emu, name):
    """gap costs with q2+e2 < q+e: the kernels reorder the two pairs like ksw_extd2_sse (:78) but start the score from the caller's q+e
    (:68, :358), in the packed or the scalar kernel and in the universal kernel"""
    L, ctx = emu[0], emu[1]
    score = [s for s in KC.REGIMES if s.name == name][0]
    rng = np.random.default_rng(sum(map(ord, name)))
    n_cls = 0
    for cls in EMU_CLASSES:
        if KC.reachable(cls, score) and not cls.startswith("exts2"):
            KC.check_batch(L, ctx, score, small_edge_jobs(rng, cls, score), cls)
            n_cls += 1
    assert n_cls == (KC.NC - KC.NS if score.pk_ok() else KC.NS) + len([c for c in EMU_CLASSES if c.startswith("extd2") or c == "ll"])
