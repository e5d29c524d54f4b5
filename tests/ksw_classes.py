"""Mirror of the K3 (ksw2) launch routing: which kernel and which width or tier every job of a batch lands in.

mmb_ksw_launch (minimap2_b200/csrc/ksw_extd2.cu) sends each job to exactly one launch class:
  * "fast<k>"  : the fast path of mmb_ksw_fast_plan (ksw_fast.cu), width k of the CW/CPW/LNW tables. k < NS is the scalar
                 ksw_fast_kernel, k >= NS the packed ksw_pk_kernel.
  * "extd2_t<k>" / "exts2_t<k>": tier k of the universal ksw_extd2_kernel, dual-affine or spliced pass; the last tier keeps
                 the DP state in HBM.
  * "ll"       : ksw_ll_kernel (MMB_JOB_LL).
The width and tier tables are parsed from the .cu sources, so a class that is added or moved shows up here (and in the coverage
test of tests/test_gpu_ksw_classes.py) without editing this file.

Also here: edge shapes per class, and a batch runner over mmb_ksw_batch_host for the device library and the SIMT emulator alike.
"""
import ctypes as C
import os
import re
import numpy as np
import oracle_lib as O

CSRC = os.path.join(O.ROOT, "minimap2_b200", "csrc")

SCORE_ONLY, RIGHT, GENERIC, APPROX, APPROX_DROP, EXT, REVC = 0x01, 0x02, 0x04, 0x08, 0x10, 0x40, 0x80
SPF, SPR, FLANK, CMPLX, SPSC = 0x100, 0x200, 0x400, 0x800, 0x1000
Q_COMP, JOB_LL, JOB_ZDROP, JOB_SPLICE, T_COMP = 0x10000, 0x20000, 0x40000, 0x80000, 0x100000
NEG_INF = -0x40000000


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _int_expr(s):
    """an integer constant of the C sources: a literal, a << b or a * b"""
    for op, f in (("<<", lambda a, b: a << b), ("*", lambda a, b: a * b)):
        if op in s:
            a, b = s.split(op, 1)
            return f(_int_expr(a), _int_expr(b))
    return int(s)


def _int_table(src, name):
    m = re.search(r"static const int %s\[\] = \{([^}]*)\};" % name, src)
    assert m, name
    return [int(x) for x in m.group(1).replace(" ", "").split(",") if x]


_FAST = _src("ksw_fast.cu")
_UNIV = _src("ksw_extd2.cu")
CW, CPW, LNW = (_int_table(_FAST, n) for n in ("CW", "CPW", "LNW"))
_m = re.search(r"const int NS = (\d+), NC = (\d+);", _FAST)
NS, NC = int(_m.group(1)), int(_m.group(2))
assert len(CW) == len(CPW) == len(LNW) == NC and 0 < NS < NC
FAST_THREADS = int(re.search(r"const int threads = (\d+), nwk = threads / 32;", _FAST).group(1))
# fast-path eligibility limits (mmb_ksw_fast_eligible, ksw_fast.cu:665-673)
_m = re.search(r"j\.tlen > (\d+) \|\| j\.qlen > (\d+)\) return false;", _FAST)
FAST_MAX_TLEN, FAST_MAX_QLEN = int(_m.group(1)), int(_m.group(2))
# universal tiers {max(qlen,tlen) bound, group size, workers per CTA} (mmb_ksw_launch, ksw_extd2.cu:738-743)
_m = re.search(r"Tier tiers\[\] = \{(.*?)\};", _UNIV)
TIERS = [tuple(_int_expr(v) for v in t.split(",")) for t in re.findall(r"\{([^{}]*)\}", _m.group(1))]
N_TIERS = int(re.search(r"const int n_tiers = (\d+);", _UNIV).group(1))
assert len(TIERS) == N_TIERS
# ksw_ll_kernel: 128 threads per CTA, 8 threads per job; persistent groups = n_sm * 16 * 4 (ksw_extd2.cu:783-785)
LL_THREADS, LL_JOBS_PER_CTA = 128, 16
LL_GROUPS_PER_SM = _int_expr(re.search(r"ctx->n_sm \* (\d+ \* \d+)\);", _UNIV).group(1))
# MM_B200_KSW_SMEM_MAXLEN (a test hook of mmb_ksw_launch) lowers the tier bounds; the class edges here assume it is not set
SMEM_MAXLEN_ENV = "MM_B200_KSW_SMEM_MAXLEN"
assert SMEM_MAXLEN_ENV in _UNIV

FAST_CLASSES = ["fast%d" % k for k in range(NC)]
UNIV_CLASSES = ["%s_t%d" % (p, k) for p in ("extd2", "exts2") for k in range(N_TIERS)]
ALL_CLASSES = FAST_CLASSES + UNIV_CLASSES + ["ll"]


def fast_bound(k):
    return LNW[k] * CW[k]


def fast_lo(k):
    """smallest tlen of width k: one past the previous width of the same kernel"""
    return 1 if k in (0, NS) else fast_bound(k - 1) + 1


def is_packed(cls):
    return cls.startswith("fast") and int(cls[4:]) >= NS


def tier_of(cls):
    return int(cls.split("_t")[1])


def tier_lo(k):
    return 1 if k == 0 else TIERS[k - 1][0] + 1


class Scoring:
    """a mmb_ksw_score_t: match/mismatch/sc_ambi (+ transition) matrix and gap costs as the mapper's options give them"""

    def __init__(self, name, a, b, q, e, q2, e2, sc_ambi=1, transition=0, noncan=0, junc_bonus=0, junc_pen=0):
        self.name, self.a, self.b, self.q, self.e, self.q2, self.e2 = name, a, b, q, e, q2, e2
        self.mat = O.simple_mat(a, b, sc_ambi, transition)
        self.generic = transition != 0
        self.noncan, self.junc_bonus, self.junc_pen = noncan, junc_bonus, junc_pen

    def pk_limit_sum(self):
        """2*max(q+e,q2+e2) + max|s| + 8 (ksw_fast.cu:697-698): the packed kernel takes the scoring when this is <= 127"""
        q, e, q2, e2 = self.q, self.e, self.q2, self.e2
        if q2 + e2 < q + e:
            q, e, q2, e2 = q2, e2, q, e
        mch, mis = int(self.mat[0]), int(self.mat[1])
        scn = -e2 if self.mat[24] == 0 else int(self.mat[24])
        return 2 * max(q + e, q2 + e2) + max(abs(mch), abs(mis), abs(scn)) + 8, mch, mis, scn

    def pk_ok(self):
        s, mch, mis, scn = self.pk_limit_sum()
        return s <= 127 and mch > 0 and mis <= 0 and scn <= 0

    def __repr__(self):
        return self.name


def fast_eligible(job):
    """mmb_ksw_fast_eligible (ksw_fast.cu:665-673)"""
    f, qlen, tlen = job["flag"], len(job["qbuf"]), len(job["tbuf"])
    if f & (JOB_LL | JOB_SPLICE | T_COMP | SCORE_ONLY | RIGHT | APPROX_DROP | EXT):
        return False
    if not f & APPROX:
        return False
    if qlen <= 0 or tlen <= 0 or tlen > FAST_MAX_TLEN or qlen > FAST_MAX_QLEN:
        return False
    w = max(qlen, tlen) if job["w"] < 0 else job["w"]
    return w >= max(qlen, tlen)


def route(job, score):
    """the launch class mmb_ksw_launch gives this job (ksw_extd2.cu:747-760, ksw_fast.cu:705-711)"""
    f, qlen, tlen = job["flag"], len(job["qbuf"]), len(job["tbuf"])
    if f & JOB_LL:
        return "ll"
    spl = (f & JOB_SPLICE) != 0
    if not spl and fast_eligible(job):
        pk = score.pk_ok() and not f & GENERIC
        k, last = (NS, NC - 1) if pk else (0, NS - 1)
        while k < last and fast_bound(k) < tlen:
            k += 1
        return "fast%d" % k
    m, k = max(qlen, tlen), 0
    while k < N_TIERS and m > TIERS[k][0]:
        k += 1
    assert k < N_TIERS, "longer than the last tier: aborts by design"
    return "%s_t%d" % ("exts2" if spl else "extd2", k)


def workers_per_cta(cls):
    """jobs a CTA of this class works on at once"""
    if cls == "ll":
        return LL_JOBS_PER_CTA
    if cls.startswith("fast"):
        k = int(cls[4:])
        return FAST_THREADS // 32 * (32 // LNW[k])
    return TIERS[tier_of(cls)][2]


def threads_per_cta(cls):
    if cls == "ll":
        return LL_THREADS
    if cls.startswith("fast"):
        return FAST_THREADS
    _, G, nw = TIERS[tier_of(cls)]
    return G * nw


def resident_bound(cls, n_sm, max_threads_per_sm=2048):
    """an upper bound on the workers of a persistent launch of this class: every SM full of CTAs, limited by threads only"""
    return n_sm * (max_threads_per_sm // threads_per_cta(cls)) * workers_per_cta(cls)


# ---------------- sequences ----------------
def comp(a):
    a = np.asarray(a, dtype=np.uint8)
    return np.where(a < 4, 3 - a, a).astype(np.uint8)


def rand_seq(rng, n):
    return rng.integers(0, 4, n).astype(np.uint8)


def related(rng, qlen, tlen, err=0.1, n_frac=0.0):
    """a target of tlen bases and a query of exactly qlen bases derived from it (mutated, then cut or padded)"""
    t = rand_seq(rng, tlen)
    q = O.mutate(t[:qlen + qlen // 4 + 8], rng, err=err)[:qlen]
    if len(q) < qlen:
        q = np.concatenate([q, rand_seq(rng, qlen - len(q))])
    if n_frac > 0:
        for s in (q, t):
            s[rng.random(len(s)) < n_frac] = 4
            s[rng.integers(0, len(s))] = 4
    return q, t


def make_job(q, t, w=-1, zdrop=-1, end_bonus=-1, flag=0, q_rev=False, t_rev=False, introns=None):
    """a job whose kernel view is (q, t): the buffers hold what the kernel must read backwards and/or complement to see them.
    introns: annotated introns (st, en, strand) in the coordinates of the kernel view of the target."""
    qb = comp(q) if flag & Q_COMP else np.asarray(q, dtype=np.uint8)
    tb = comp(t) if flag & T_COMP else np.asarray(t, dtype=np.uint8)
    if q_rev:
        qb = qb[::-1]
    if t_rev:
        tb = tb[::-1]
    return dict(qbuf=np.ascontiguousarray(qb), tbuf=np.ascontiguousarray(tb), q_rev=q_rev, t_rev=t_rev, q=np.asarray(q, dtype=np.uint8),
                t=np.asarray(t, dtype=np.uint8), w=w, zdrop=zdrop, end_bonus=end_bonus, flag=flag, introns=introns or [])


def junc_flags(job):
    """junc[] of the reference's ksw_exts2_sse call for this job (mm_idx_bed_junc over the window, index.c:802-826)"""
    if not job["introns"]:
        return None
    tl = len(job["t"])
    fl = np.zeros(tl, dtype=np.uint8)
    for st, en, sd in job["introns"]:  # flags in forward target coordinates, reversed with the target for a reversed job (align.c:787-790)
        if job["t_rev"]:
            st, en = tl - en, tl - st
        if sd != 0:
            fl[st] |= 1 if sd > 0 else 8
            fl[en - 1] |= 2 if sd > 0 else 4
    return fl[::-1].copy() if job["t_rev"] else fl


# ---------------- running a batch ----------------
def run_batch(lib, ctx_h, score, jobs):
    """all jobs through mmb_ksw_batch_host in one call. Returns (results, zdrop scans, kernel launches the call made)."""
    from minimap2_b200._lib import KswJob, KswRes
    from minimap2_b200 import kernels as K
    lib.mmb_launch_count.restype = C.c_uint64
    lib.mmb_launch_count.argtypes = [C.c_void_p, C.c_int]
    n = len(jobs)
    qcat = np.ascontiguousarray(np.concatenate([j["qbuf"] for j in jobs]))
    tcat = np.ascontiguousarray(np.concatenate([j["tbuf"] for j in jobs]))
    cj = (KswJob * n)()
    qo = to = tot = 0
    introns = []
    for i, jb in enumerate(jobs):
        c, ql, tl = cj[i], len(jb["qbuf"]), len(jb["tbuf"])
        c.q_start, c.q_step = (qo + ql - 1, -1) if jb["q_rev"] else (qo, 1)
        c.t_start, c.t_step = (to + tl - 1, -1) if jb["t_rev"] else (to, 1)
        c.qlen, c.tlen, c.w, c.zdrop, c.end_bonus, c.flag = ql, tl, jb["w"], jb["zdrop"], jb["end_bonus"], jb["flag"]
        for st, en, sd in jb["introns"]:  # view coordinates -> concatenated-buffer coordinates
            introns.append((to + tl - en, to + tl - st, sd) if jb["t_rev"] else (to + st, to + en, sd))
        qo += ql; to += tl; tot += ql + tl + 2
    if introns:
        introns.sort(key=lambda x: x[0])
        st = np.array([x[0] for x in introns], dtype=np.int64); en = np.array([x[1] for x in introns], dtype=np.int64)
        sd = np.array([x[2] for x in introns], dtype=np.int8)
        assert lib.mmb_ctx_set_junctions(ctx_h, C.c_int64(len(introns)), st.ctypes.data_as(C.c_void_p), en.ctypes.data_as(C.c_void_p),
                                         sd.ctypes.data_as(C.c_void_p)) == 0
    sc = K.make_score(score.mat, score.q, score.e, score.q2, score.e2, score.noncan, score.junc_bonus, score.junc_pen)
    res = (KswRes * n)()
    cig = np.zeros(tot, dtype=np.uint32)
    lib.mmb_launch_count(ctx_h, 1)
    try:
        used = lib.mmb_ksw_batch_host(ctx_h, C.byref(sc), n, cj, qcat.ctypes.data, len(qcat), tcat.ctypes.data, len(tcat), res,
                                      cig.ctypes.data, len(cig))
    finally:
        if introns:
            lib.mmb_ctx_set_junctions(ctx_h, C.c_int64(0), None, None, None)
    launches = lib.mmb_launch_count(ctx_h, 1)
    assert used >= 0, used
    out, zds = [], []
    for i in range(n):
        r = res[i]
        out.append(dict(max=r.max, zdropped=r.zdropped, max_q=r.max_q, max_t=r.max_t, mqe=r.mqe, mqe_t=r.mqe_t, mte=r.mte, mte_q=r.mte_q,
                        score=r.score, n_cigar=r.n_cigar, reach_end=r.reach_end, cigar=[int(x) for x in cig[r.cigar_off:r.cigar_off + r.n_cigar]]))
        zds.append((r.zd_max, r.zd_t0, r.zd_t1, r.zd_q0, r.zd_q1))
    return out, zds, launches


def expected(job, score):
    """the oracle's answer for the job's kernel view"""
    q, t, f = job["q"], job["t"], job["flag"]
    if f & JOB_LL:
        return O.oracle_ll_i16(q, t, score.mat, job["w"], job["zdrop"])
    if f & JOB_SPLICE:
        return O.oracle_exts2(q, t, score.mat, score.q, score.e, score.q2, score.noncan, job["zdrop"], job["end_bonus"], score.junc_bonus,
                              score.junc_pen, f & 0x1fff, junc_flags(job))
    return O.oracle_extd2(q, t, score.mat, score.q, score.e, score.q2, score.e2, job["w"], job["zdrop"], job["end_bonus"], f & 0xff)


def check_batch(lib, ctx_h, score, jobs, cls):
    """one class, one launch, every job bit-exact against the oracle; z-drop scans exact in the packed classes, absent elsewhere.
    Returns the number of jobs checked."""
    import test_emu_ksw as E
    for i, jb in enumerate(jobs):
        assert route(jb, score) == cls, (i, route(jb, score), cls)
    got, zds, launches = run_batch(lib, ctx_h, score, jobs)
    assert launches == 1, (cls, score, launches)
    for i, (jb, g, zd) in enumerate(zip(jobs, got, zds)):
        exp = expected(jb, score)
        what = (cls, score, i, len(jb["q"]), len(jb["t"]), jb["w"], hex(jb["flag"]), jb["q_rev"], jb["t_rev"])
        if jb["flag"] & JOB_LL:
            assert (g["score"], g["max_q"], g["max_t"]) == exp, (what, g, exp)
            continue
        assert g == exp, (what, {k: (g[k], exp[k]) for k in exp if g[k] != exp[k] and k != "cigar"}, g["cigar"][:6], exp["cigar"][:6])
        if (jb["flag"] & JOB_ZDROP) and is_packed(cls):
            assert zd == E.zdrop_scan(jb["q"], jb["t"], score.mat, exp["cigar"], score.q, score.e), (what, zd)
        else:
            assert zd[0] == -1, (what, zd)
    return len(jobs)


# ---------------- edge shapes per class ----------------
def edge_tlens(lo, hi):
    return sorted({lo, (lo + hi) // 2, hi})


def fast_jobs(rng, k, score, n_odd=True):
    """jobs of width k at both edges of its tlen range and inside it, qlen from 1 to the fast path's limit, every band form that
    keeps the job on the fast path, N bases, reversed and complemented reads"""
    jobs = []
    lo, hi = fast_lo(k), fast_bound(k)
    gen = GENERIC if score.generic else 0
    for ti, tlen in enumerate(edge_tlens(lo, hi)):
        qlens = [1, max(1, tlen + int(rng.integers(-8, 9))), FAST_MAX_QLEN if ti != 1 else int(rng.integers(2, 700))]
        for qi, qlen in enumerate(qlens):
            v = len(jobs)
            q, t = related(rng, qlen, tlen, err=float(rng.choice([0.02, 0.1, 0.25])), n_frac=0.02 if v % 3 == 0 else 0.0)
            w = [-1, max(qlen, tlen), 30001][v % 3]
            flag = APPROX | gen | (JOB_ZDROP if v % 2 == 0 else 0) | (Q_COMP if v % 4 == 1 else 0)
            jobs.append(make_job(q, t, w=w, zdrop=400, flag=flag, q_rev=v % 3 == 1, t_rev=v % 4 == 2))
    if n_odd and len(jobs) % 2 == 0:
        jobs.pop()
    return jobs


def univ_shapes(rng, k):
    """(qlen, tlen, w) at both edges of tier k's max(qlen,tlen) range and inside it. Long shapes are asymmetric or narrow-banded so the
    oracle stays cheap. The last tier is only reached up to 20000: on its own bound of 1 << 20 the oracle alone takes minutes."""
    lo, hi = tier_lo(k), TIERS[k][0]
    out = []
    for m in edge_tlens(lo, hi) if hi <= 20000 else [lo, 20000]:
        if m <= 1100:
            out += [(m, max(1, m - int(rng.integers(0, 20))), -1), (max(1, m // 3), m, 17), (m, m, 100), (1, m, 751)]
        else:
            out += [(int(rng.integers(20, 200)), m, -1), (m, int(rng.integers(1, 120)), 751), (m, m, 17), (m, m, 100)]
    return out


UNIV_FLAGS = [0, EXT, EXT | RIGHT | REVC, RIGHT, SCORE_ONLY, APPROX]


def extd2_jobs(rng, k, score):
    jobs = []
    gen = GENERIC if score.generic else 0
    for qlen, tlen, w in univ_shapes(rng, k):
        v = len(jobs)
        if qlen == tlen and w > 0:  # a square shape on a narrow band: an end extension
            t = rand_seq(rng, tlen); q = O.mutate(t, rng, err=0.08)[:qlen]
            q = np.concatenate([q, rand_seq(rng, qlen - len(q))])
            if v % 3 == 0:
                q[rng.integers(0, qlen, 3)] = 4; t[rng.integers(0, tlen, 3)] = 4
        else:
            q, t = related(rng, qlen, tlen, err=0.1, n_frac=0.01 if v % 3 == 0 else 0.0)
        flag = UNIV_FLAGS[v % len(UNIV_FLAGS)]
        if flag == APPROX and (w < 0 or w >= max(qlen, tlen)):
            w = max(1, max(qlen, tlen) - 1)  # too narrow for the fast path by one
        flag |= gen | (T_COMP if v % 3 == 1 else 0) | (Q_COMP if v % 5 == 2 else 0)
        jobs.append(make_job(q, t, w=w, zdrop=[400, -1, 200][v % 3], end_bonus=[-1, 10][v % 2], flag=flag, q_rev=v % 2 == 1, t_rev=v % 4 == 3))
    return jobs


def spliced_pair(rng, tlen, n_exon, err=0.03):
    """tests/test_emu_ksw.small_spliced_pair with introns long enough for a target of tlen bases, the target padded to exactly tlen"""
    import test_emu_ksw as E
    introns = []
    span = max(30, (tlen - 90 * n_exon) // max(1, n_exon - 1))
    q, t = E.small_spliced_pair(rng, n_exon, err, introns, intron_len=(max(30, span // 2), max(31, span)))
    while len(t) > tlen:
        n_exon = max(1, n_exon - 1); introns = []
        q, t = E.small_spliced_pair(rng, n_exon, err, introns, intron_len=(30, max(31, (tlen - 90 * n_exon) // max(1, n_exon - 1))))
    t = np.concatenate([t, rand_seq(rng, tlen - len(t))])
    return q, t, introns


def exts2_jobs(rng, k, score, model, with_junc=False):
    jobs = []
    lo, hi = tier_lo(k), TIERS[k][0]
    tls = edge_tlens(max(lo, 40), hi) if hi <= 20000 else [lo, 20000]
    base = [0, APPROX, EXT, EXT | RIGHT | REVC, RIGHT]
    for tlen in tls:
        for r in range(2):
            v = len(jobs)
            q, t, ints = spliced_pair(rng, tlen, int(rng.integers(2, 5)) if tlen > 100 else 1)
            if v % 3 == 0:
                q[rng.integers(0, len(q))] = 4
            flag = base[v % len(base)] | (SPF if v % 2 == 0 else SPR) | model | JOB_SPLICE
            introns = []
            if with_junc:
                introns = [(st, en, [1, -1][i % 2]) for i, (st, en) in enumerate(ints)]
                introns += [(st + 2, en + 2, 1) for st, en in ints[:1] if en + 2 <= tlen]  # a shifted decoy
            jobs.append(make_job(q, t, w=[-1, 17, 300][v % 3], zdrop=[200, -1][v % 2], end_bonus=[-1, 10][v % 2], flag=flag,
                                 t_rev=v % 2 == 1, introns=introns))
    return jobs


def ll_jobs(rng, n, qmax=60, tmax=80):
    jobs = []
    for v in range(n):
        qlen = 1 if v % 17 == 0 else int(rng.integers(1, qmax + 1))
        q, t = related(rng, qlen, int(rng.integers(max(1, qlen // 2), tmax + 1)), err=0.15, n_frac=0.02 if v % 5 == 0 else 0.0)
        if v % 4 == 0:  # a local hit inside a longer target
            t = np.concatenate([rand_seq(rng, int(rng.integers(0, 30))), t])
        flag = JOB_LL | (T_COMP if v % 3 == 1 else 0) | (Q_COMP if v % 3 == 2 else 0)
        jobs.append(make_job(q, t, w=4, zdrop=2, end_bonus=0, flag=flag, q_rev=v % 2 == 1, t_rev=v % 5 == 3))  # w = gap open, zdrop = gap extension
    return jobs


def class_jobs(rng, cls, score, model=FLANK | CMPLX):
    if cls.startswith("fast"):
        return fast_jobs(rng, int(cls[4:]), score)
    if cls.startswith("extd2"):
        return extd2_jobs(rng, tier_of(cls), score)
    if cls.startswith("exts2"):
        return exts2_jobs(rng, tier_of(cls), score, model)
    return ll_jobs(rng, 41)


def reachable(cls, score):
    """whether a scoring can put any job into this class"""
    if cls.startswith("fast"):
        return is_packed(cls) == (score.pk_ok() and not score.generic)
    return True


# ---------------- scorings ----------------
MAP_ONT = Scoring("map-ont", 2, 4, 4, 2, 24, 1)
PK_LIMIT = Scoring("pk-limit", 2, 5, 4, 2, 56, 1)       # 2*max(q+e,q2+e2) + max|s| + 8 == 127: the packed kernel's last scoring
PK_LIMIT_1 = Scoring("pk-limit+1", 2, 6, 4, 2, 56, 1)   # == 128 (mismatch one larger): the scalar kernel
REGIMES = [
    MAP_ONT,
    Scoring("asm5", 1, 19, 39, 3, 81, 1),
    Scoring("generic-ts", 2, 4, 4, 2, 24, 1, transition=2),
    Scoring("sc_ambi0", 2, 4, 4, 2, 24, 1, sc_ambi=0),
    Scoring("sc_ambi2", 2, 4, 4, 2, 24, 1, sc_ambi=2),
    Scoring("swapped-gaps", 2, 4, 24, 1, 4, 2),           # q2+e2 < q+e: the kernels reorder the pairs (ksw2_extd2_sse.c:78)
    Scoring("asm5-swapped", 1, 19, 81, 1, 39, 3),         # the same on the scalar kernel
    Scoring("single-affine", 2, 4, 4, 2, 4, 2),
    PK_LIMIT,
    PK_LIMIT_1,
]
SPLICE_SCORINGS = [Scoring("splice", 1, 2, 2, 1, 32, 0, noncan=9, junc_bonus=9, junc_pen=5),
                   Scoring("splice-sc_ambi0", 1, 2, 2, 1, 32, 0, sc_ambi=0, noncan=9, junc_bonus=9, junc_pen=5),
                   Scoring("splice-sc_ambi2", 2, 4, 4, 2, 24, 0, sc_ambi=2, noncan=5, junc_bonus=9, junc_pen=5)]
