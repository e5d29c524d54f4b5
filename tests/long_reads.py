"""Long-read inputs for tests/test_gpu_long_reads.py and, reduced, tests/test_emu_long_reads.py: a repeat-rich genome and read sets at
the lengths long-read users map (20 kb to 1.1 Mb), built deterministically from numpy seeds. The recorded reference outputs
(tests/golden/expected/long_reference_lines.json) are keyed by the SHA-1 of the files written here, so any change to these generators
needs the records made again (tests/golden/make_long_reference_lines.sh).

Genome (genome()): contigs of random sequence with
  * segmental duplications of 20-80 kb at 0.5-3% divergence, some inverted (seeds with a few occurrences, chains on two copies);
  * a tandem array of a 171-bp monomer at 0.5-2% per-copy divergence (minimizers with about as many occurrences as copies: the
    query-side occurrence filter, high-occurrence streaks, reads of more than 10^5 anchors);
  * microsatellites of 1-6 bp units, 0.5-5 kb long;
  * a 10 kb run of N inside one contig.
Read sets: ont_set() (ONT-like errors, 20-300 kb, three reads of 0.7-1.1 Mb that align end to end, reads inside the tandem array,
chimeras, inversions, large insertions and deletions, an N run), hifi_set() (15-60 kb at 0.1-1% error) and sched_set() (at least
768 reads and 4 Mbases: enough for the mapper to split one mini-batch into 12 groups)."""
import gzip
import io
import json
import os
import numpy as np
import oracle_lib as O
import synth

A = synth.ALPHA


def _rnd(rng, n):
    return A[rng.integers(0, 4, n)]


def _copy_diverged(rng, src, div):
    """src with substitutions and small indels at rate div, cut or padded to len(src)"""
    out = synth.mutate_ascii(src, rng, div)
    return out[:len(src)] if len(out) >= len(src) else np.concatenate([out, src[len(out):]])


def genome(seed=1, lens=(3_200_000, 2_600_000, 2_200_000, 2_000_000), n_segdup=12, segdup=(20_000, 80_000), n_mono=1500,
           n_sat=40, n_run=10_000):
    """contigs (ASCII uint8 arrays) and a dict of where the features lie: 'array' = (contig, start, end) of the tandem array,
    'nrun' = (contig, start, end) of the N run, 'avoid' = per contig the (start, end) intervals reads that must align end to
    end stay out of"""
    rng = np.random.default_rng(seed)
    ctgs = [_rnd(rng, n) for n in lens]
    avoid = [[] for _ in lens]
    for _ in range(n_segdup):
        ln = int(rng.integers(segdup[0], segdup[1] + 1))
        cs, cd = int(rng.integers(0, len(ctgs))), int(rng.integers(0, len(ctgs)))
        s, d = int(rng.integers(0, len(ctgs[cs]) - ln)), int(rng.integers(0, len(ctgs[cd]) - ln))
        src = ctgs[cs][s:s + ln].copy()
        if rng.random() < 0.4:
            src = synth.revcomp(src)
        ctgs[cd][d:d + ln] = _copy_diverged(rng, src, float(rng.uniform(0.005, 0.03)))
    mono = _rnd(rng, 171)
    arr = np.concatenate([_copy_diverged(rng, mono, float(rng.uniform(0.005, 0.02))) for _ in range(n_mono)])
    a0 = len(ctgs[1]) // 2
    ctgs[1][a0:a0 + len(arr)] = arr
    avoid[1].append((a0 - 50_000, a0 + len(arr) + 50_000))
    for _ in range(n_sat):
        unit = _rnd(rng, int(rng.integers(1, 7)))
        ln = int(rng.integers(500, 5001))
        c = int(rng.integers(0, len(ctgs)))
        p = int(rng.integers(0, len(ctgs[c]) - ln))
        ctgs[c][p:p + ln] = _copy_diverged(rng, np.resize(unit, ln), 0.01)
    cn = min(2, len(ctgs) - 1)
    r0 = len(ctgs[cn]) // 3
    ctgs[cn][r0:r0 + n_run] = ord("N")
    avoid[cn].append((r0 - 10_000, r0 + n_run + 10_000))
    return ctgs, dict(array=(1, a0, a0 + len(arr)), nrun=(cn, r0, r0 + n_run), avoid=avoid)


def _place(rng, ctgs, ln, avoid=None):
    """(contig, start) of a read of length ln, outside the avoid intervals when given"""
    while True:
        c = int(rng.integers(0, len(ctgs)))
        if len(ctgs[c]) <= ln:
            continue
        s = int(rng.integers(0, len(ctgs[c]) - ln))
        if avoid is None or all(s + ln <= a or s >= b for a, b in avoid[c]):
            return c, s


def _ont(rng, seg, err=None):
    rd = synth.mutate_ascii(seg, rng, float(rng.uniform(0.08, 0.12)) if err is None else err)
    return synth.revcomp(rd) if rng.random() < 0.5 else rd


def _loguniform(rng, lo, hi):
    return int(np.exp(rng.uniform(np.log(lo), np.log(hi))))


def ont_set(ctgs, info, seed=2, n=60, rlen=(20_000, 300_000), n_ultra=3, ultra=(700_000, 1_100_000), special=True):
    """(names, reads): n reads of log-uniform length with 8-12% ONT-like errors, then the ultra-long reads and, with special, the
    reads of particular shapes (their names say which)"""
    rng = np.random.default_rng(seed)
    names, reads = [], []
    for i in range(n):
        ln = _loguniform(rng, *rlen)
        c, s = _place(rng, ctgs, ln)
        names.append("ont%03d" % i); reads.append(_ont(rng, ctgs[c][s:s + ln]))
    for i in range(n_ultra):
        ln = int(rng.integers(ultra[0], ultra[1] + 1))
        c, s = _place(rng, ctgs, ln, info["avoid"])
        names.append("ultra%d" % i); reads.append(_ont(rng, ctgs[c][s:s + ln]))
    if not special:
        return names, reads
    ac, a0, a1 = info["array"]
    for i in range(2):  # mostly inside the tandem array, with a unique flank on one side
        ln = int(rng.integers(120_000, 180_000))
        s = a0 - 15_000 if i == 0 else a1 + 15_000 - ln
        names.append("tandem%d" % i); reads.append(_ont(rng, ctgs[ac][s:s + ln]))
    for i in range(2):  # two pieces from different contigs
        l0, l1 = int(rng.integers(30_000, 80_000)), int(rng.integers(30_000, 80_000))
        c0, s0 = _place(rng, ctgs, l0, info["avoid"])
        c1, s1 = _place(rng, ctgs, l1, info["avoid"])
        while c1 == c0:
            c1, s1 = _place(rng, ctgs, l1, info["avoid"])
        names.append("chimera%d" % i); reads.append(_ont(rng, np.concatenate([ctgs[c0][s0:s0 + l0], synth.revcomp(ctgs[c1][s1:s1 + l1])])))
    for i in range(2):  # a 5-30 kb inversion in the middle
        inv = int(rng.integers(5_000, 30_001)); ln = inv + int(rng.integers(40_000, 80_000))
        c, s = _place(rng, ctgs, ln, info["avoid"])
        seg = ctgs[c][s:s + ln].copy(); m = (ln - inv) // 2
        seg[m:m + inv] = synth.revcomp(seg[m:m + inv])
        names.append("inversion%d" % i); reads.append(_ont(rng, seg))
    for i in range(2):  # a 10-20 kb insertion (i = 0) or deletion (i = 1), larger than max_gap
        sv = int(rng.integers(10_000, 20_001)); ln = int(rng.integers(60_000, 100_000))
        c, s = _place(rng, ctgs, ln + sv, info["avoid"])
        seg = ctgs[c][s:s + ln + sv]; m = ln // 2
        seg = np.concatenate([seg[:m], _rnd(rng, sv), seg[m:ln]]) if i == 0 else np.concatenate([seg[:m], seg[m + sv:]])
        names.append(("insertion%d" if i == 0 else "deletion%d") % i); reads.append(_ont(rng, seg))
    ln = int(rng.integers(40_000, 80_000))  # a 5 kb N run inside the read
    c, s = _place(rng, ctgs, ln, info["avoid"])
    rd = synth.mutate_ascii(ctgs[c][s:s + ln], rng, 0.1)
    m = len(rd) // 2
    names.append("nrun0"); reads.append(np.concatenate([rd[:m], np.full(5000, ord("N"), dtype=np.uint8), rd[m:]]))
    return names, reads


def hifi_set(ctgs, seed=3, n=200, rlen=(15_000, 60_000)):
    rng = np.random.default_rng(seed)
    names, reads = [], []
    for i in range(n):
        ln = int(rng.integers(rlen[0], rlen[1] + 1))
        c, s = _place(rng, ctgs, ln)
        names.append("hifi%03d" % i); reads.append(_ont(rng, ctgs[c][s:s + ln], float(rng.uniform(0.001, 0.01))))
    return names, reads


def sched_set(ctgs, info, seed=4, n=800, rlen=(5_000, 40_000)):
    """n ONT reads of 5-40 kb with three ultra-long reads first, in the middle and last"""
    rng = np.random.default_rng(seed)
    names, reads = [], []
    for i in range(n):
        ln = _loguniform(rng, *rlen)
        c, s = _place(rng, ctgs, ln)
        names.append("s%04d" % i); reads.append(_ont(rng, ctgs[c][s:s + ln]))
    un, ur = ont_set(ctgs, info, seed=seed + 100, n=0, n_ultra=3, special=False)
    for p, nm, rd in zip((0, len(reads) // 2, len(reads) + 2), un, ur):
        names.insert(p, nm); reads.insert(p, rd)
    return names, reads


def qualities(seed, reads):
    rng = np.random.default_rng(seed)
    return [bytes((rng.integers(2, 42, len(r)) + 33).astype(np.uint8)) for r in reads]


def write_fastq_gz(path, names, reads, quals):
    with gzip.GzipFile(path, "wb", mtime=0) as g, io.BufferedWriter(g) as f:  # mtime 0: the same bytes on every run
        for n, s, q in zip(names, reads, quals):
            f.write(b"@" + n.encode() + b" len=%d\n" % len(s) + bytes(s) + b"\n+\n" + q + b"\n")


def write_all(d, small=False):
    """writes the genome and the read sets under directory d; returns a dict of the paths and the sets. small: the reduced case of the
    emulated tests (a 2 Mbp genome with a 60 kb tandem array, seven reads of 30-100 kb)"""
    if small:
        ctgs, info = genome(seed=21, lens=(1_100_000, 900_000), n_segdup=3, n_mono=350, n_sat=10)
        info["avoid"] = [[] for _ in ctgs]
        names, reads = ont_set(ctgs, info, seed=22, n=5, rlen=(30_000, 60_000), n_ultra=1, ultra=(100_000, 100_000), special=False)
        ac, a0, a1 = info["array"]
        names.append("tandem0"); reads.append(_ont(np.random.default_rng(23), ctgs[ac][a0 - 10_000:a1]))
        out = dict(ref=os.path.join(d, "small_ref.fa"), ont=os.path.join(d, "small_ont.fa"), ctgs=ctgs, info=info, ont_set=(names, reads))
        synth.write_fasta(out["ref"], ["chr%d" % i for i in range(len(ctgs))], ctgs)
        synth.write_fasta(out["ont"], names, reads)
        return out
    ctgs, info = genome()
    out = dict(ref=os.path.join(d, "long_ref.fa"), ont=os.path.join(d, "long_ont.fa"), ont_fq=os.path.join(d, "long_ont.fq.gz"),
               hifi=os.path.join(d, "long_hifi.fa"), sched=os.path.join(d, "long_sched.fa"), ctgs=ctgs, info=info)
    synth.write_fasta(out["ref"], ["chr%d" % i for i in range(len(ctgs))], ctgs)
    out["ont_set"] = ont_set(ctgs, info)
    synth.write_fasta(out["ont"], *out["ont_set"])
    fq_names, fq_reads = out["ont_set"][0] + ["allN"], out["ont_set"][1] + [np.full(4_300_000, ord("N"), dtype=np.uint8)]
    write_fastq_gz(out["ont_fq"], fq_names, fq_reads, qualities(5, fq_reads))  # the last record is longer than the reader's buffer
    out["hifi_set"] = hifi_set(ctgs)
    synth.write_fasta(out["hifi"], *out["hifi_set"])
    out["sched_set"] = sched_set(ctgs, info)
    synth.write_fasta(out["sched"], *out["sched_set"])
    return out


# ---------------- seeding parameters of the presets, and the reference's recorded output ----------------
# (w, k, min_mid_occ, max_mid_occ, occ_dist) of map-ont, lr:hq / map-hifi and lr:hqae (options.c); q_occ_frac 0.01, max_max_occ 4095
PRESETS = {"map-ont": (10, 15, 10, 1000, 500), "lr:hq": (19, 19, 50, 500, 500), "lr:hqae": (51, 25, 50, 500, 200)}


def mid_occ(ctgs, w, k, lo, hi, f=2e-4):
    """mid_occ as mm_mapopt_update sets it: mm_idx_cal_max_occ(f) over the index's minimizers, clamped to [lo, hi]"""
    import index_cases as IC
    x = np.concatenate([O.oracle_sketch(bytes(c), w, k)[:, 0] >> np.uint64(8) for c in ctgs])
    _, cnt = np.unique(x, return_counts=True)
    return min(max(IC.max_occ(cnt, f), lo), hi)


def seed_params(ctgs, preset):
    w, k, lo, hi, od = PRESETS[preset]
    return dict(w=w, k=k, mid_occ=mid_occ(ctgs, w, k, lo, hi), q_occ_frac=0.01, max_max_occ=4095, occ_dist=od)


REF_LINES = os.path.join(O.ROOT, "tests", "golden", "expected", "long_reference_lines.json")


def reference_lines(args):
    """the reference binary's recorded output of `minimap2 <args>` (oracle_lib's digest form), from expected/long_reference_lines.json.
    With MM2_RECORD_REFERENCE set, oracle_lib runs the reference binary and records into that file instead
    (tests/golden/make_long_reference_lines.sh)."""
    if os.environ.get("MM2_RECORD_REFERENCE"):
        return O.reference_lines(args)
    key = O.input_key(args)
    tab = json.load(open(REF_LINES))
    assert key in tab, "no recorded reference output for these inputs: minimap2 " + key
    return O.RecordedLines(tab[key])
