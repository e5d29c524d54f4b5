"""CPU: the product's K3 CUDA kernels (ksw_pk_kernel, ksw_fast_kernel, ksw_extd2_kernel, ksw_ll_kernel -- the unmodified sources of
minimap2_b200/csrc/ksw_fast.cu and ksw_extd2.cu) executed by the SIMT emulator of tests/cuda_emu (one OS thread per CUDA thread)
and compared with the oracle, job for job. This checks kernel LOGIC in the CPU suite; the -m gpu tests remain the parity proof on
the real device."""
import ctypes as C
import os
import sys
import numpy as np
import pytest
import oracle_lib as O

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))
sys.path.insert(0, O.ROOT)
EXT, RIGHT, REVC, APPROX, SCORE_ONLY = 0x40, 0x02, 0x80, 0x08, 0x01
JOB_LL, JOB_ZDROP = 0x20000, 0x40000


def load_emu():
    import build_emu
    from minimap2_b200._lib import KswJob, KswRes, KswScore
    L = C.CDLL(build_emu.build("mmb_emu_k3", ["mmb_ctx.cu", "ksw_fast.cu", "ksw_extd2.cu"]))
    L.mmb_ctx_create.restype = C.c_void_p
    L.mmb_ksw_batch_host.restype = C.c_int64
    L.mmb_ksw_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64]
    ctx = C.c_void_p(L.mmb_ctx_create(0))
    assert ctx.value
    return L, ctx, KswJob, KswRes, KswScore


@pytest.fixture(scope="module")
def emu():
    return load_emu()


def run_jobs(emu, mat, q, e, q2, e2, pairs, params, zd_skip=0):
    L, ctx, KswJob, KswRes, KswScore = emu
    n = len(pairs)
    qcat = np.concatenate([np.asarray(p[0], dtype=np.uint8) for p in pairs]); tcat = np.concatenate([np.asarray(p[1], dtype=np.uint8) for p in pairs])
    jobs = (KswJob * n)(); qo = to = tot = 0
    for i, ((qq, tt), pr) in enumerate(zip(pairs, params)):
        j = jobs[i]
        j.q_start, j.t_start, j.q_step, j.t_step, j.qlen, j.tlen = qo, to, 1, 1, len(qq), len(tt)
        j.w, j.zdrop, j.end_bonus, j.flag = pr["w"], pr["zdrop"], pr["end_bonus"], pr["flag"]
        qo += len(qq); to += len(tt); tot += len(qq) + len(tt) + 2
    sc = KswScore()
    for i in range(25):
        sc.mat[i] = int(mat[i])
    sc.q, sc.e, sc.q2, sc.e2 = q, e, q2, e2
    sc.zd_skip = zd_skip
    res = (KswRes * n)(); cig = np.zeros(tot, dtype=np.uint32)
    used = L.mmb_ksw_batch_host(ctx, C.byref(sc), n, jobs, qcat.ctypes.data, len(qcat), tcat.ctypes.data, len(tcat), res, cig.ctypes.data, len(cig))
    assert used >= 0
    out = []
    for i in range(n):
        r = res[i]
        out.append((dict(max=r.max, zdropped=r.zdropped, max_q=r.max_q, max_t=r.max_t, mqe=r.mqe, mqe_t=r.mqe_t, mte=r.mte, mte_q=r.mte_q, score=r.score,
                         n_cigar=r.n_cigar, reach_end=r.reach_end, cigar=[int(x) for x in cig[r.cigar_off:r.cigar_off + r.n_cigar]]),
                    (r.zd_max, r.zd_t0, r.zd_t1, r.zd_q0, r.zd_q1)))
    return out


def zdrop_scan(q, t, mat, cigar, gq, ge):
    """mm_test_zdrop's scan (align.c:61-89) in plain Python: max_zdrop and pos"""
    score, mx, mi, mj, i, j, zd, pos = 0, -(1 << 31), -1, -1, 0, 0, 0, [-1, -1, -1, -1]

    def upd(sc, ii, jj):
        nonlocal mx, mi, mj, zd, pos
        if sc < mx:
            li, lj = ii - mi, jj - mj
            z = mx - sc - abs(li - lj) * ge
            if z > zd:
                zd, pos = z, [mi, ii, mj, jj]
        else:
            mx, mi, mj = sc, ii, jj
    for c in cigar:
        op, ln = c & 0xf, c >> 4
        if op == 0:
            for l in range(ln):
                score += int(mat[int(t[i + l]) * 5 + int(q[j + l])]); upd(score, i + l, j + l)
            i += ln; j += ln
        else:
            score -= gq + ge * ln
            if op == 1: j += ln
            else: i += ln
            upd(score, i, j)
    return (zd, *pos)


def test_emulated_kernels_match_oracle(emu):
    rng = np.random.default_rng(2024)
    mat = O.simple_mat(2, 4, 1)
    pairs, params = [], []
    for it in range(90):
        tl = int(rng.integers(1, 330)) if it % 5 else int(rng.integers(260, 520))
        t = rng.integers(0, 4, tl).astype(np.uint8)
        q = O.mutate(t, rng, err=float(rng.choice([0.0, 0.05, 0.15, 0.35])))
        if len(q) == 0:
            q = np.array([0], dtype=np.uint8)
        if rng.random() < 0.2:
            q[rng.integers(0, len(q))] = 4; t[rng.integers(0, len(t))] = 4
        kind = it % 6
        if kind in (0, 1, 2):   # gap fills: packed kernel (+ the in-kernel z-drop scan)
            pr = dict(w=30001, zdrop=400, end_bonus=-1, flag=APPROX | JOB_ZDROP)
        elif kind == 3:         # extensions through the universal kernel
            pr = dict(w=int(rng.choice([751, 40, 17])), zdrop=int(rng.choice([400, 100, -1])), end_bonus=int(rng.choice([-1, 10])), flag=int(rng.choice([EXT, EXT | RIGHT | REVC])))
        elif kind == 4:         # exact global alignment, band-limited or not
            pr = dict(w=int(rng.choice([-1, 30, 5])), zdrop=int(rng.choice([-1, 200])), end_bonus=-1, flag=int(rng.choice([0, RIGHT, SCORE_ONLY])))
        else:                   # local score probe (ksw_ll_i16): w = gap open, zdrop = gap extension
            pr = dict(w=4, zdrop=2, end_bonus=0, flag=JOB_LL)
        pairs.append((q, t)); params.append(pr)
    got = run_jobs(emu, mat, 4, 2, 24, 1, pairs, params)
    n_zd = 0
    for i, ((qq, tt), pr) in enumerate(zip(pairs, params)):
        g, zd = got[i]
        if pr["flag"] & JOB_LL:
            sc, qe, te = O.oracle_ll_i16(qq, tt, mat, 4, 2)
            assert (g["score"], g["max_q"], g["max_t"]) == (sc, qe, te), (i, g)
            continue
        exp = O.oracle_extd2(qq, tt, mat, 4, 2, 24, 1, pr["w"], pr["zdrop"], pr["end_bonus"], pr["flag"] & 0xff)
        assert g == exp, (i, len(qq), len(tt), pr, {k: (g[k], exp[k]) for k in exp if g[k] != exp[k]})
        if (pr["flag"] & JOB_ZDROP) and zd[0] >= 0:
            assert zd == zdrop_scan(qq, tt, mat, exp["cigar"], 4, 2), (i, zd)
            n_zd += 1
    assert n_zd >= 20


def small_spliced_pair(rng, n_exon, err, introns_out=None, intron_len=(30, 200)):
    ex = [rng.integers(0, 4, int(rng.integers(20, 90))).astype(np.uint8) for _ in range(n_exon)]
    parts = [ex[0]]; pos = len(ex[0])
    for k in range(1, n_exon):
        intron = rng.integers(0, 4, int(rng.integers(*intron_len))).astype(np.uint8)
        sig = int(rng.integers(0, 5))
        if sig < 3: intron[:2] = [2, 3]; intron[-2:] = [0, 2]
        elif sig == 3: intron[:2] = [2, 1]; intron[-2:] = [0, 2]
        if introns_out is not None:
            introns_out.append((pos, pos + len(intron)))
        pos += len(intron) + len(ex[k])
        parts += [intron, ex[k]]
    q = O.mutate(np.concatenate(ex), rng, err=err)
    return (q if len(q) else np.array([0], dtype=np.uint8)), np.concatenate(parts)


def check_splice_jobs(emu, rng, models, n_jobs, max_exons, with_junc=False, with_score=False):
    L, ctx, KswJob, KswRes, KswScore = emu
    SPF, SPR, JOB_SPLICE = 0x100, 0x200, 0x80000
    mat = O.simple_mat(1, 2, 1)
    for model in models:  # the model bits are per batch (mm_mapopt_t), the strand bits per job
        pairs, params, true_introns = [], [], []
        for it in range(n_jobs):
            true_introns.append([])
            q, t = small_spliced_pair(rng, int(rng.integers(1, max_exons + 1)), float(rng.choice([0.0, 0.03, 0.1])), true_introns[-1])
            if rng.random() < 0.1:
                q[rng.integers(0, len(q))] = 4
            base = int(rng.choice([0, APPROX, EXT, EXT | RIGHT | REVC, RIGHT]))
            pairs.append((q, t)); params.append(dict(w=[-1, 17, 300][it % 3], zdrop=int(rng.choice([-1, 200])), end_bonus=int(rng.choice([-1, 10])), flag=base | int(rng.choice([SPF, SPR])) | model | JOB_SPLICE))  # w: ksw_exts2 has no band, whatever bandwidth the driver passes along
        n = len(pairs)
        qcat = np.concatenate([p[0] for p in pairs]); tcat = np.concatenate([p[1] for p in pairs])
        jobs = (KswJob * n)(); qo = to = tot = 0
        introns, juncs = [], [None] * n
        score_tabs = [{}, {}]
        for i, ((qq, tt), pr) in enumerate(zip(pairs, params)):
            j = jobs[i]
            j.q_start, j.t_start, j.q_step, j.t_step, j.qlen, j.tlen = qo, to, 1, 1, len(qq), len(tt)
            j.w, j.zdrop, j.end_bonus, j.flag = pr["w"], pr["zdrop"], pr["end_bonus"], pr["flag"]
            if with_score:
                # splice-score tables per strand in the coordinates of the concatenated target (mmb_ctx_set_splice_scores): scores at the
                # true intron ends, at shifted decoys and at random places; a job sees the entries strictly inside its window
                lt = len(tt); sd = 1 if pr["flag"] & SPR else 0
                j.flag = pr["flag"] = pr["flag"] | 0x1000
                for tab in (0, 1):
                    cand = {}
                    for st, en in true_introns[i]:
                        for pos_, typ in ((st, 0), (en - 1, 1)) if rng.random() < 0.5 else ((en - 1, 0), (st, 1)):
                            cand[to + pos_ + int(rng.choice([0, 0, 0, 1, -2]))] = (int(rng.integers(60, 80)) << 1) | typ
                    for _ in range(max(1, lt // 25)):
                        cand[to + int(rng.integers(0, lt))] = (int(rng.integers(50, 78)) << 1) | int(rng.integers(0, 2))
                    cand[to] = (70 << 1) | 1  # on the window edge: not strictly inside, must be ignored
                    for pos_, v in cand.items():
                        if to <= pos_ < to + lt:
                            score_tabs[tab][pos_] = v
                flags = np.full(lt, 0xff, dtype=np.uint8)
                for pos_, v in score_tabs[sd].items():
                    if to < pos_ < to + lt:
                        flags[pos_ - to] = v
                if i % 2:
                    j.t_start, j.t_step = to + lt - 1, -1
                    pairs[i] = (qq, tt[::-1].copy()); flags = flags[::-1].copy()
                juncs[i] = flags
            if with_junc:
                # annotated introns in the coordinates of the concatenated target: inside this job's window, or sticking out of it
                # (those must be ignored, index.c:816); every other job reads its target backwards (t_step = -1, reversed junc[])
                lt = len(tt); flags = np.zeros(lt, dtype=np.uint8)
                cand = [(to + int(rng.integers(-5, lt)), int(rng.integers(1, 60))) for _ in range(max(1, lt // 30))]
                cand = [(st, st + ln) for st, ln in cand]
                for st, en in true_introns[i]:  # the real introns, some of them shifted by a few bases
                    d = int(rng.choice([0, 0, 0, -2, 3]))
                    cand.append((to + st + d, to + en + d))
                for st, en in cand:
                    sd = int(rng.choice([1, -1, -1, 1, 0]))
                    introns.append((st, en, sd))
                    if st >= to and en <= to + lt and sd != 0:
                        flags[st - to] |= 1 if sd > 0 else 8; flags[en - 1 - to] |= 2 if sd > 0 else 4
                if i % 2:
                    j.t_start, j.t_step = to + lt - 1, -1
                    pairs[i] = (qq, tt[::-1].copy()); flags = flags[::-1].copy()
                juncs[i] = flags
            qo += len(qq); to += len(tt); tot += len(qq) + len(tt) + 2
        if with_junc:
            # the device reads a reversed job backwards from the forward array, so tcat stays as built; pairs[i] now holds what the oracle sees
            introns.sort(key=lambda x: x[0])
            st = np.array([x[0] for x in introns], dtype=np.int64); en = np.array([x[1] for x in introns], dtype=np.int64); sd = np.array([x[2] for x in introns], dtype=np.int8)
            assert L.mmb_ctx_set_junctions(ctx, C.c_int64(len(introns)), st.ctypes.data_as(C.c_void_p), en.ctypes.data_as(C.c_void_p), sd.ctypes.data_as(C.c_void_p)) == 0
        if with_score:
            for tab in (0, 1):
                ps = np.array(sorted(score_tabs[tab]), dtype=np.int64); vs = np.array([score_tabs[tab][x] for x in ps], dtype=np.uint8)
                assert L.mmb_ctx_set_splice_scores(ctx, tab, C.c_int64(len(ps)), ps.ctypes.data_as(C.c_void_p), vs.ctypes.data_as(C.c_void_p)) == 0
        sc = KswScore()
        for i in range(25):
            sc.mat[i] = int(mat[i])
        sc.q, sc.e, sc.q2, sc.e2, sc.noncan, sc.junc_bonus, sc.junc_pen = 2, 1, 32, 0, 9, 9, 5
        res = (KswRes * n)(); cig = np.zeros(tot, dtype=np.uint32)
        used = L.mmb_ksw_batch_host(ctx, C.byref(sc), n, jobs, qcat.ctypes.data, len(qcat), tcat.ctypes.data, len(tcat), res, cig.ctypes.data, len(cig))
        assert used >= 0
        if with_junc:
            L.mmb_ctx_set_junctions(ctx, C.c_int64(0), None, None, None)
        if with_score:
            for tab in (0, 1):
                L.mmb_ctx_set_splice_scores(ctx, tab, C.c_int64(0), None, None)
        n_changed = 0
        for i, ((qq, tt), pr) in enumerate(zip(pairs, params)):
            r = res[i]
            g = dict(max=r.max, zdropped=r.zdropped, max_q=r.max_q, max_t=r.max_t, mqe=r.mqe, mqe_t=r.mqe_t, mte=r.mte, mte_q=r.mte_q, score=r.score,
                     n_cigar=r.n_cigar, reach_end=r.reach_end, cigar=[int(x) for x in cig[r.cigar_off:r.cigar_off + r.n_cigar]])
            exp = O.oracle_exts2(qq, tt, mat, 2, 1, 32, 9, pr["zdrop"], pr["end_bonus"], 9, 5, pr["flag"] & 0x1fff, juncs[i])
            if with_junc or with_score:
                n_changed += exp != O.oracle_exts2(qq, tt, mat, 2, 1, 32, 9, pr["zdrop"], pr["end_bonus"], 9, 5, pr["flag"] & 0x1fff)
            assert g == exp, (hex(model), i, len(qq), len(tt), hex(pr["flag"]), {k: (g[k], exp[k]) for k in exp if g[k] != exp[k] and k != "cigar"}, g["cigar"][:8], exp["cigar"][:8])
        assert not (with_junc or with_score) or n_changed >= 3, n_changed  # the annotation really changed some of the expected results


def test_emulated_splice_kernel_with_junction_annotation(emu):
    """the annotated-junction branch of ksw_exts2_sse (:220-241) in the spliced kernel: the flags are derived on the device from a
    sorted intron table (mmb_ctx_set_junctions) with mm_idx_bed_junc's window rule, for forward and reversed targets"""
    FLANK, CMPLX = 0x400, 0x800
    check_splice_jobs(emu, np.random.default_rng(78), (FLANK | CMPLX, 0), 24, 3, with_junc=True)


def test_emulated_splice_kernel_with_splice_scores(emu):
    """the splice-score branch of ksw_exts2_sse (:213-219): junc[] bytes assembled on the device from per-strand position tables
    (mmb_ctx_set_splice_scores) with mm_idx_spsc_get's window rule, forward and reversed targets"""
    FLANK, CMPLX = 0x400, 0x800
    check_splice_jobs(emu, np.random.default_rng(79), (FLANK | CMPLX, 0), 24, 3, with_score=True)


def test_emulated_splice_kernel_matches_oracle(emu):
    """ksw_extd2_kernel<G, SP=true> (ksw_exts2_sse: intron state, donor/acceptor signals) under the emulator vs the oracle's restatement"""
    FLANK, CMPLX = 0x400, 0x800
    check_splice_jobs(emu, np.random.default_rng(77), (FLANK | CMPLX, FLANK), 24, 4)


def test_emulated_hbm_state_tier():
    """the tier that keeps the DP state in HBM (targets > 13000 on the device): MM_B200_KSW_SMEM_MAXLEN moves tiny jobs there. The
    library reads the variable once, hence the separate process."""
    import subprocess
    env = dict(os.environ, MM_B200_KSW_SMEM_MAXLEN="48")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "hbm-tier"], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=1800)
    assert p.returncode == 0 and b"HBM_TIER_OK" in p.stdout, p.stdout.decode()[-2000:]


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "hbm-tier":
    e = load_emu()
    rng = np.random.default_rng(5)
    mat = O.simple_mat(2, 4, 1)
    pairs, params = [], []
    for it in range(3):
        t = rng.integers(0, 4, int(rng.integers(60, 110))).astype(np.uint8)
        q = O.mutate(t, rng, err=0.1)
        pairs.append((q, t)); params.append(dict(w=int(rng.choice([-1, 20])), zdrop=200, end_bonus=-1, flag=[0, EXT, EXT | RIGHT | REVC][it % 3]))
    for (g, _), (qq, tt), pr in zip(run_jobs(e, mat, 4, 2, 24, 1, pairs, params), pairs, params):
        assert g == O.oracle_extd2(qq, tt, mat, 4, 2, 24, 1, pr["w"], pr["zdrop"], pr["end_bonus"], pr["flag"])
    check_splice_jobs(e, rng, (0x400 | 0x800,), 3, 2)
    try:
        check_splice_jobs(e, rng, (0x400,), 2, 2, with_junc=True)  # junction flags OR-ed into the score row that lives in HBM here
    except AssertionError as ex:
        if not (ex.args and isinstance(ex.args[0], int)):  # too few jobs for the "annotation changed something" count: not a failure
            raise
    print("HBM_TIER_OK")


def check_zdrop_scan_skip(run, mat):
    """mmb_ksw_score_t::zd_skip: the kernel may answer "no drop" (0) without scanning, but only when the true largest drop is within the
    threshold; every other job still carries the exact scan. Shared by the emulated and the device test."""
    rng = np.random.default_rng(99)
    pairs, params = [], []
    for it in range(120):
        t = rng.integers(0, 4, int(rng.integers(40, 380))).astype(np.uint8)
        q = O.mutate(t, rng, err=float(rng.choice([0.02, 0.08, 0.15, 0.3])))
        if it % 7 == 0 and len(q) > 30:  # a junk stretch: a large drop
            a = int(rng.integers(5, len(q) - 20)); q[a:a + 15] = rng.integers(0, 4, 15)
        if len(q) == 0:
            q = np.array([0], dtype=np.uint8)
        pairs.append((q, t)); params.append(dict(w=30001, zdrop=400, end_bonus=-1, flag=APPROX | JOB_ZDROP))
    n_skip = n_scan = 0
    for thr in (60, 200):
        got = run(mat, 4, 2, 24, 1, pairs, params, thr)
        for (qq, tt), (g, zd) in zip(pairs, got):
            exp = O.oracle_extd2(qq, tt, mat, 4, 2, 24, 1, 30001, 400, -1, APPROX)
            assert g == exp
            true = zdrop_scan(qq, tt, mat, exp["cigar"], 4, 2)
            if zd == true:
                n_scan += 1
            else:  # skipped: reported as "no drop", and the true drop really is within the threshold
                assert zd[0] == 0 and true[0] <= thr, (zd, true, thr)
                n_skip += 1
    assert n_skip >= 40 and n_scan >= 40, (n_skip, n_scan)


def test_emulated_zdrop_scan_skip(emu):
    check_zdrop_scan_skip(lambda *a: run_jobs(emu, *a), O.simple_mat(2, 4, 1))
