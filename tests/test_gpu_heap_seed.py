"""GPU: heap-ordered seeding (`--heap-sort=yes`, MM_F_HEAP_SORT; collect_seed_hits_heap, map.c:102-166).
  * kernel level: mmb_seed_batch_host with the flag against the restatement of the heap merge (tests/heap_cases.py:HeapOracle) on
    thousands of reads, long and short, with the situations the order depends on counted;
  * CLI: byte-identical to the reference binary's recorded output (tests/golden/expected/heap_reference_lines.json) with every long-read
    preset and chainer, the re-chaining pass and query-strand mode; `--heap-sort=no` gives the default output;
  * API: mm_map with the flag (api.Aligner(extra_flags=MM_F_HEAP_SORT)) returns the CLI's hits."""
import ctypes as C
import os
import subprocess
import pytest
import oracle_lib as O
import seed_check as SC
import synth
import heap_cases as H

pytestmark = pytest.mark.gpu
MINE = os.path.join(O.ROOT, "minimap2_b200", "minimap2-b200")
DATA = os.path.join(O.ROOT, "tests", "golden", "data")
D = lambda f: os.path.join(DATA, f)
ONT = [D("synth-ref.fa"), D("synth-ont.fa")]


@pytest.fixture(scope="module")
def dev():
    import minimap2_b200 as mb
    from minimap2_b200._lib import lib
    L = lib()
    SC.setup(L)
    c = mb.Context(0)
    yield L, C.c_void_p(c.h)
    c.close()


@pytest.mark.parametrize("cfg", [dict(mid_occ=10), dict(mid_occ=6, occ_dist=100), dict(mid_occ=10, flag=0x100000), dict(mid_occ=10, flag=0x200000),
                                 dict(w=19, k=19, mid_occ=20)])
def test_heap_seed_stage_matches_oracle(dev, cfg):
    L, ctx = dev
    contigs, reads = H.mixed_case(41, 1_000_000, 400, 4000, 4000, rep=0.6, n_contigs=3)
    big_ctg, big_read = H.oversize_case(unit_len=6000, copies=6)  # occurrences and query multiplicity within mid_occ = 6
    contigs, reads = contigs + [big_ctg], reads + [big_read]
    H.check_device(L, ctx, contigs, reads, **cfg)
    w, k = cfg.get("w", 10), cfg.get("k", 15)
    idx = H.HeapOracle([bytes(c) for c in contigs], ["chr%d" % i for i in range(len(contigs))], w, k)
    okw = {a: b for a, b in cfg.items() if a not in ("w", "k")}
    okw.setdefault("flag", 0)
    pc = H.path_counts(idx, reads, okw)
    st = H.tie_stats(idx, [bytes(r) for r in reads], [None] * len(reads), w, k, okw)
    idx.close()
    assert st["reads"] > 4000 and pc["smem"] >= 5 and pc["global_"] >= 1 and pc["oversize"] >= 1, (pc, st)
    strands = "+" if okw["flag"] & 0x100000 else "-" if okw["flag"] & 0x200000 else "+-"
    H.assert_covered(st, strands=strands, skip=bool(okw["flag"] & H.SKIP))


def _repeat_rich_files(tmp_path):
    contigs, reads = H.mixed_case(51, 300_000, 60, 3000, 400, rep=0.6, n_contigs=3)
    rf, qf = str(tmp_path / "ref.fa"), str(tmp_path / "reads.fa")
    synth.write_fasta(rf, ["chr%d" % i for i in range(len(contigs))], contigs)
    synth.write_fasta(qf, ["rd%04d" % i for i in range(len(reads))], reads)
    return [rf, qf]


LINES = [(["-x", "map-ont", "-c", "--heap-sort=yes"], ONT),
         (["-x", "map-hifi", "-a", "--heap-sort=yes"], [D("synth-ref.fa"), D("synth-hifi.fa")]),
         (["-x", "ava-ont", "--heap-sort=yes"], [D("synth-ont.fa"), D("synth-ont.fa")]),
         (["-x", "splice", "--heap-sort=yes"], [D("synth-gene.fa"), D("synth-cdna.fa")]),
         (["-x", "asm5", "--heap-sort=yes"], [D("MT-human.fa"), D("MT-orang.fa")]),
         (["-x", "map-ont", "--qstrand", "--heap-sort=yes"], ONT),
         (["-x", "map-ont", "-c", "--heap-sort=yes"], None),
         (["-x", "map-ont", "-f", "10,1000", "--heap-sort=yes"], None),
         (["-x", "ava-ont", "--heap-sort=yes"], None),
         (["-x", "map-ont", "--qstrand", "--heap-sort=yes"], None)]
# on the repeat-rich inputs in query-strand mode the heap path is visible: the reference prints something else without --heap-sort=yes
DIFFERS = {9}


def _mine(args):
    p = subprocess.run([MINE, "-t", "8"] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1200)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    return p.stdout.decode().splitlines()


@pytest.mark.parametrize("i", range(len(LINES)))
def test_heap_sort_cli_matches_reference(tmp_path, i):
    opts, files = LINES[i]
    if files is None:
        files = _repeat_rich_files(tmp_path)
        if "ava-ont" in opts:
            files = [files[1], files[1]]
    ref = H.reference_lines(opts + files)
    if i in DIFFERS:
        assert H.reference_lines([o for o in opts if o != "--heap-sort=yes"] + files).all != ref.all
    O.assert_matches_reference(_mine(opts + files), ref)
    assert len(ref) > 0


def test_heap_sort_no_is_default():
    assert _mine(["-x", "map-ont", "-c", "--heap-sort=yes", "--heap-sort=no"] + ONT) == _mine(["-x", "map-ont", "-c"] + ONT)


def test_api_heap_sort_maps_as_cli():
    from minimap2_b200.api import Aligner
    al = Aligner(ONT[0], preset="map-ont", extra_flags=H.HEAP)
    assert al
    got = []
    names, seqs = [], []
    for l in open(ONT[1]):
        if l.startswith(">"):
            names.append(l[1:].split()[0]); seqs.append("")
        else:
            seqs[-1] += l.strip()
    for name, s in zip(names, seqs):
        for h in al.map(s):
            got.append((name, h.q_st, h.q_en, "+" if h.strand > 0 else "-", h.ctg, h.r_st, h.r_en, h.mlen, h.blen, h.mapq))
    al.close()
    cli = [tuple(f[:1] + [int(f[2]), int(f[3]), f[4], f[5], int(f[7]), int(f[8]), int(f[9]), int(f[10]), int(f[11])])
           for f in (l.split("\t") for l in _mine(["-x", "map-ont", "-c", "--heap-sort=yes"] + ONT))]
    assert len(got) > 0 and sorted(got) == sorted(cli)
