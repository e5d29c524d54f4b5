"""GPU: junction jumps (-j, --pass1, --jump-min-match) and --write-junc.
- K5 (jump.cuh) through mmb_jump_batch_host against the restatement in jump_cases.py, hit for hit.
- The command line, byte for byte against the reference's recorded output, on the jump_cases data set; each run with jumps also
  differs from the same run without them in a stated number of lines. The recorded output of these command lines is kept in
  tests/golden/expected/jump_reference_lines.json (tests/golden/make_jump_reference_lines.sh regenerates it).
Marker gpu_ext, like the other optional splice inputs (--junc-bed, --spsc)."""
import ctypes as C
import json
import os
import numpy as np
import pytest
import oracle_lib as O
import jump_cases as J
from test_gpu_e2e import run, MINE

pytestmark = pytest.mark.gpu_ext
REF_LINES = os.path.join(O.ROOT, "tests", "golden", "expected", "jump_reference_lines.json")


def compare(args):
    """this library's CLI output for args against the reference's recorded output of the same command (oracle_lib's digest form).
    With MM2_RECORD_REFERENCE set, oracle_lib runs the reference binary and records into that file instead."""
    if os.environ.get("MM2_RECORD_REFERENCE"):
        ref = O.reference_lines(args)
    else:
        key = O.input_key(args)
        tab = json.load(open(REF_LINES))
        assert key in tab, "no recorded reference output for these inputs: minimap2 " + key
        ref = O.RecordedLines(tab[key])
    O.assert_matches_reference(run(MINE, ["-t", "8"] + args), ref)
    return len(ref)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = J.make_data(seed=11)
    d["dir"] = J.write_data(d, str(tmp_path_factory.mktemp("jump")))
    return d


def _paths(d, *names):
    return [os.path.join(d["dir"], n) for n in names]


def _n_differ(a, b):
    assert len(a) == len(b)
    return sum(x != y for x, y in zip(a, b))


def test_k5_matches_restatement(data):
    import minimap2_b200 as mb
    from minimap2_b200 import kernels as K
    from minimap2_b200.api import Aligner
    al = Aligner(_paths(data, "ref.fa")[0], preset="splice")
    L = mb.lib()
    L.mm_idx_jjump_read.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int]
    assert L.mm_idx_jjump_read(C.cast(al._idx, C.c_void_p), _paths(data, "anno.bed")[0].encode(), J.MM_JUNC_ANNO, -1) == 0
    hits = J.hit_variants(data, np.random.default_rng(23))
    reads = [s for _, s in data["reads"]]
    t4 = [J.NT4[np.frombuffer(s, dtype=np.uint8)] for s in data["contigs"]]
    from test_jump_vs_ref import entries, _setup
    _setup(L)
    tables = [[(e[0], e[1], e[4]) for e in entries(L, al._idx, c, -1, len(s))] for c, s in enumerate(data["contigs"])]
    ctx = mb.Context(0)
    acts = set()
    for jmm in (3, 5, 30):
        al.map_opt.jump_min_match = jmm
        got = K.jump_batch(ctx, al._idx, al.map_opt, reads, hits)
        for h, g in zip(hits, got):
            exp = J.decide(h, reads[h["read"]], t4[h["rid"]], tables[h["rid"]], al.map_opt.a, al.map_opt.b, jmm)
            assert g == exp, (h, g, exp)
            acts.update((g[0][0], g[1][0]))
    assert {0, 1, 2} <= acts
    ctx.close()


def test_jumps_vs_reference(data):
    ref, qry, anno = _paths(data, "ref.fa", "reads.fa", "anno.bed")
    for args, min_diff in ((["-x", "splice", "-c", "--cs", "-j", anno], 150), (["-x", "splice", "-a", "-j", anno, "--jump-min-match", "5"], 100)):
        compare(args + [ref, qry])
        with_j = run(MINE, ["-t", "8"] + args + [ref, qry])
        k = args.index("-j")
        without = run(MINE, ["-t", "8"] + args[:k] + args[k + 2:] + [ref, qry])
        assert _n_differ([l for l in with_j if not l.startswith("@PG")], [l for l in without if not l.startswith("@PG")]) >= min_diff


def test_two_pass_vs_reference(data):
    """--write-junc, then its output as --pass1 next to the annotation"""
    ref, qry, anno = _paths(data, "ref.fa", "reads.fa", "anno.bed")
    compare(["-x", "splice", "--write-junc", ref, qry])
    junc = os.path.join(data["dir"], "junc.bed")
    with open(junc, "w") as f:
        f.write("".join(l + "\n" for l in run(MINE, ["-x", "splice", "--write-junc", ref, qry])))
    compare(["-x", "splice", "-c", "--pass1", junc, "-j", anno, ref, qry])
    compare(["-x", "splice", "-c", "--pass1", junc, ref, qry])
    assert _n_differ(run(MINE, ["-x", "splice", "-c", "--pass1", junc, ref, qry]), run(MINE, ["-x", "splice", "-c", ref, qry])) >= 150


def test_jumps_with_junction_bed_vs_reference(data):
    ref, qry, anno = _paths(data, "ref.fa", "reads.fa", "anno.bed")
    compare(["-x", "splice", "-c", "--junc-bed", anno, "-j", anno, ref, qry])


def test_refusals(data):
    import subprocess
    ref, qry, anno = _paths(data, "ref.fa", "reads.fa", "anno.bed")
    p = subprocess.run([MINE, "-x", "splice", "-c", "--eqx", "-j", anno, ref, qry], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600)
    assert p.returncode == 1 and b"--eqx" in p.stderr and p.stdout == b""
    p = subprocess.run([MINE, "-x", "splice", "-c", "-j", anno + ".missing", ref, qry], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600)
    assert p.returncode == 0 and b"failed to load the jump BED file" in p.stderr
    assert p.stdout.decode().splitlines() == run(MINE, ["-x", "splice", "-c", ref, qry])
