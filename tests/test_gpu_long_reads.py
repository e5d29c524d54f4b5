"""GPU: the mapper at the read lengths long-read users have (20 kb to 1.1 Mb; tests/long_reads.py), stage by stage against the oracle and
the reference, and end to end against the reference binary's recorded output (tests/golden/expected/long_reference_lines.json).
  * seeding (mmb_seed_batch_host) against the oracle with map-ont's, lr:hq's and lr:hqae's seeding parameters, on reads whose
    minimizers overflow the query filter's and the seed selection's shared-memory tables (mzflt_kernel, select_kernel through
    SelGlobal), where the query-occurrence filter drops repeats, and with more than 16,384 and 10^5 anchors;
  * the anchor sort (mmb_anchor_sort_host) on those anchors against the reference's radix_sort_128x, order and route;
  * the chainers on the same anchors against the reference's: the DP at map-ont's parameters, the RMQ chainer at lr:hqae's and the
    long-join rescue at the default bw_long;
  * CLI output byte for byte: map-ont with --cs, -a with and without -L (CIGARs of more than 65,535 operations), -K below one read,
    --max-qlen, --no-long-join, FASTQ.gz input; lr:hq, map-hifi, lr:hqae, map-iclr and map-iclr-prerender on HiFi reads; and a batch
    that the mapper splits into 12 concurrent groups."""
import ctypes as C
import gzip
import os
import subprocess
import numpy as np
import pytest
import oracle_lib as O
import seed_check as SC
import sort_cases as S
import chain_cases as CC
import long_reads as LR

pytestmark = pytest.mark.gpu
MINE = os.path.join(O.ROOT, "minimap2_b200", "minimap2-b200")


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return LR.write_all(str(tmp_path_factory.mktemp("long")))


@pytest.fixture(scope="module")
def dev():
    import minimap2_b200 as mb
    from minimap2_b200._lib import lib
    L = lib()
    SC.setup(L)
    c = mb.Context(0)
    yield L, C.c_void_p(c.h), c
    c.close()


# seeding cases: (read set, preset whose seeding parameters apply); lr:hqae on the ONT reads gives the reads of more than 10^5 anchors
CASES = [("ont_set", "map-ont"), ("hifi_set", "lr:hq"), ("hifi_set", "lr:hqae"), ("ont_set", "lr:hqae")]
_seeds = {}


def seeds(dev, data, i):
    """the seeding stage of case i checked against the oracle (once per module); returns (parameters, reads, the oracle's anchors)"""
    if i not in _seeds:
        L, ctx, _ = dev
        which, preset = CASES[i]
        par = LR.seed_params(data["ctgs"], preset)
        reads = [bytes(r) for r in data[which][1]]
        keep = []
        SC.check_case(L, ctx, data["ctgs"], reads, keep=keep, **par)
        _seeds[i] = par, reads, keep
    return _seeds[i]


@pytest.mark.parametrize("i", range(len(CASES)))
def test_long_seed_stage(dev, data, i):
    par, reads, anchors = seeds(dev, data, i)
    w, k, m = par["w"], par["k"], par["mid_occ"]
    n_sk = [SC.n_sketch(r, w, k) for r in reads]
    n_mz = [SC.n_minimizers(r, w, k, m, par["q_occ_frac"]) for r in reads]
    n_a = [len(a) for a in anchors]
    assert sum(n > 2048 for n in n_sk) >= 10 and sum(n > 2048 for n in n_mz) >= 10, (n_sk, n_mz)  # mzflt_kernel; select_kernel, SelGlobal
    assert sum(a < b for a, b in zip(n_mz, n_sk)) >= 1  # the query-occurrence filter drops minimizers
    if CASES[i] != ("hifi_set", "lr:hq"):
        assert max(n_a) > 16384, max(n_a)  # oversize reads: the global exact walker
    if CASES[i] == ("ont_set", "lr:hqae"):
        assert max(n_a) > 100_000, max(n_a)


@pytest.mark.parametrize("i", [0, 3])
def test_long_anchor_sort(dev, data, i):
    """the oracle's anchor keys of every read in a fixed shuffled order, sorted by the sort kernels"""
    _, _, anchors = seeds(dev, data, i)
    rng = np.random.default_rng(40 + i)
    cases = [("read%d" % j, rng.permutation(a[:, 0])) for j, a in enumerate(anchors)]
    seen = S.check_batch(dev[2], cases)
    assert seen[S.OVERSIZE] >= 1 and sum(v for r, v in seen.items() if r >= 0 and r & S.EXACT) >= 1, seen


def test_long_chain_dp(dev, data):
    """mg_lchain_dp at map-ont's parameters, on the map-ont anchors and on the lr:hqae ones (reads of more than 10^5 anchors)"""
    from minimap2_b200 import kernels as K
    p = CC.dp_par()
    for i in (0, 3):
        _, _, anchors = seeds(dev, data, i)
        got = K.chain_batch(dev[2], anchors, p["max_dist_x"], p["max_dist_y"], p["bw"], p["max_skip"], p["max_iter"], p["min_cnt"],
                            p["min_sc"], p["pen_gap"], p["pen_skip"], p["is_cdna"])
        assert CC.check_all(got, anchors, lambda a: CC.expect_dp(a, p), "dp case %d" % i) > 0
    assert max(len(a) for a in anchors) > 100_000


def test_long_chain_rmq(dev, data):
    """mg_lchain_rmq at lr:hqae's parameters (max_gap 5000, rmq_inner_dist 5000, chain_gap_scale 5 at k = 25)"""
    from minimap2_b200 import kernels as K
    p = CC.rmq_par(max_dist=5000, max_dist_inner=5000, pen_gap=CC.pen(5.0, 25))
    for i in (2, 3):
        _, _, anchors = seeds(dev, data, i)
        got = K.chain_rmq_batch(dev[2], anchors, p["max_dist"], p["max_dist_inner"], p["bw"], p["max_skip"], p["cap"], p["min_cnt"],
                                p["min_sc"], p["pen_gap"], p["pen_skip"])
        assert CC.check_all(got, anchors, lambda a: CC.expect_rmq(a, p), "rmq case %d" % i) > 0


def test_long_chain_rescue(dev, data):
    """the long-join rescue as map-ont runs it (bw_long 20000, rmq_rescue_size 1000, rmq_rescue_ratio 0.1) on the map-ont anchors with
    the reads' own lengths; the chimeric, inverted and structurally varied reads are rescued"""
    from minimap2_b200 import kernels as K
    p, r = CC.dp_par(), dict(bw_long=20000, rescue_size=1000, rescue_ratio=0.1, max_dist=5000, max_dist_inner=1000, cap=100000)
    _, reads, anchors = seeds(dev, data, 0)
    ql = [len(s) for s in reads]
    got = K.chain_rescue_batch(dev[2], anchors, ql, CC.chain_par(p), CC.rescue_par(r))
    n_rescued = 0
    for j, a in enumerate(anchors):
        u, b, rescued = CC.expect_rescue(a, ql[j], p, r)
        CC.assert_same(got[j], (u, b), "rescue read %d (%d anchors, qlen %d, rescued %d)" % (j, len(a), ql[j], rescued))
        n_rescued += rescued
    assert 0 < n_rescued < len(anchors), n_rescued


# ---------------- CLI parity ----------------
def _mine(args):
    p = subprocess.run([MINE] + (["-t", "8"] if "-t" not in args else []) + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1800)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    return p.stdout.decode().splitlines()


def _max_qlen(data):
    """a read length N with reads both longer and shorter than N"""
    return sorted(len(r) for r in data["ont_set"][1])[len(data["ont_set"][1]) // 2]


ONT_LINES = {"cs": ["-x", "map-ont", "-c", "--cs"], "sam_long_cigar": ["-x", "map-ont", "-a", "-L"], "sam": ["-x", "map-ont", "-a"],
             "minibatch": ["-x", "map-ont", "-c", "-K", "400k"], "max_qlen": ["-x", "map-ont", "-c", "--max-qlen", None],
             "cigar": ["-x", "map-ont", "-c"], "no_long_join": ["-x", "map-ont", "-c", "--no-long-join"]}


@pytest.mark.parametrize("name", list(ONT_LINES))
def test_long_cli_ont(data, name):
    opts = [str(_max_qlen(data)) if o is None else o for o in ONT_LINES[name]]
    args = opts + [data["ref"], data["ont"]]
    ref = LR.reference_lines(args)
    got = _mine(args)
    O.assert_matches_reference(got, ref)
    assert len(ref) > 0
    if name == "sam_long_cigar":  # some CIGAR has more than 65,535 operations: the CIGAR field holds a placeholder, the CIGAR goes to CG:B:I
        assert any("\tCG:B:I," in l for l in got)
    if name == "max_qlen":
        n = _max_qlen(data)
        lens = dict(zip(data["ont_set"][0], map(len, data["ont_set"][1])))
        mapped = {l.split("\t")[0] for l in got}
        assert any(lens[q] == n for q in mapped) and all(lens[q] <= n for q in mapped)
    if name == "no_long_join":  # the rescue changes the reference's output on these reads
        assert LR.reference_lines(ONT_LINES["cigar"] + [data["ref"], data["ont"]]).all != ref.all


def test_long_cli_fastq_gz(data):
    """FASTQ.gz input of the ONT set and an unmappable read of 4.3 Mbases, SAM: SEQ and QUAL of records of up to 1.1 Mb, and of one
    whose sequence and quality lines are each longer than the reader's 4 MB buffer"""
    args = ["-x", "map-ont", "-a", data["ref"], data["ont_fq"]]
    ref = LR.reference_lines(args)
    got = _mine(args)
    O.assert_matches_reference(got, ref)
    with gzip.open(data["ont_fq"], "rt") as f:
        recs = f.read().split("\n")
    qual = {recs[i][1:].split()[0]: recs[i + 3] for i in range(0, len(recs) - 3, 4)}
    prim = [l.split("\t") for l in got if not l.startswith("@") and not int(l.split("\t")[1]) & 0x900]
    assert any(len(f[10]) > 700_000 for f in prim) and any(len(f[10]) > 4 << 20 for f in prim)
    for f in prim:
        q = qual[f[0]]
        assert f[10] in ("*", q, q[::-1]), f[0]


HIFI_LINES = [["-x", "lr:hq", "-c", "--cs"], ["-x", "map-hifi", "-a", "--MD"], ["-x", "lr:hqae", "-c", "--cs"], ["-x", "map-iclr", "-c"],
              ["-x", "map-iclr-prerender", "-c"]]


@pytest.mark.parametrize("i", range(len(HIFI_LINES)))
def test_long_cli_hifi(data, i):
    args = HIFI_LINES[i] + [data["ref"], data["hifi"]]
    ref = LR.reference_lines(args)
    O.assert_matches_reference(_mine(args), ref)
    assert len(ref) > 0


def test_long_cli_scheduler_groups(data):
    """one mini-batch of at least 768 reads and 4 Mbases: the mapper runs it as 12 concurrent groups (map_batch_pass), with the
    ultra-long reads in the first, a middle and the last group"""
    reads = data["sched_set"][1]
    assert len(reads) >= 64 * 12 and sum(map(len, reads)) >= 4_000_000
    args = ["-x", "map-ont", "-c", "-t", "16", data["ref"], data["sched"]]
    ref = LR.reference_lines(args)
    O.assert_matches_reference(_mine(args), ref)
    assert len(ref) > 0
