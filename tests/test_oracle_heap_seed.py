"""CPU: the restatement of the heap-ordered anchor collection (tests/heap_cases.py:HeapOracle, the k-way heap merge of
collect_seed_hits_heap, map.c:102-166) against the unmodified reference's own stage dump (`minimap2 --print-seeds --heap-sort=yes`,
recorded in tests/golden/expected/heap_reference_lines.json): every anchor in order, and rep_len, for every read. The inputs are built
so that the order depends on the heap's history, and each test asserts that it does."""
import json
import pytest
import synth
import heap_cases as H
from test_oracle_seed import oracle_seed_dump, check


def ref_seed_dump(args):
    """the reference's --print-seeds dump (stderr), one JSON record per read, in the form tests/test_oracle_seed.py records"""
    def records(out, err):
        reads, cur = [], None
        for l in err.splitlines():
            f = l.split("\t")
            if f[0] == "QR":
                cur = dict(name=f[1], rep=None, sd=[]); reads.append(cur)
            elif f[0] == "RS":
                cur["rep"] = int(f[1])
            elif f[0] == "SD":
                cur["sd"].append((f[1], int(f[2]), f[3], int(f[4]), int(f[5])))
        return [json.dumps(r) for r in reads]
    return H.reference_lines(["--print-seeds"] + args, records=records)


def _run(tmp_path, extra, kw, w, k, strands="+-", ava=False):
    contigs, reads = H.mixed_case(11, 200_000, 40, 3000, 200, rep=0.6, n_contigs=3) if not ava else \
        H.mixed_case(12, 60_000, 30, 3000, 100, rep=0.5, n_contigs=1)
    qnames = ["rd%03d" % i for i in range(len(reads))]
    qf = str(tmp_path / "reads.fa")
    synth.write_fasta(qf, qnames, reads)
    if ava:
        names, seqs, args = qnames, reads, [qf, qf]
    else:
        names, seqs = ["chr%d" % i for i in range(len(contigs))], contigs
        rf = str(tmp_path / "ref.fa")
        synth.write_fasta(rf, names, contigs)
        args = [rf, qf]
    ref = ref_seed_dump(["--heap-sort=yes"] + extra + args)
    idx = H.HeapOracle([bytes(c) for c in seqs], names, w, k)
    reads = [bytes(r) for r in reads]
    check(ref, oracle_seed_dump(idx, names, reads, qnames, **kw))
    st = H.tie_stats(idx, reads, qnames, w, k, kw)
    idx.close()
    H.assert_covered(st, strands=strands, skip=bool(kw.get("flag", 0) & H.SKIP))


@pytest.mark.parametrize("cfg", [dict(extra=["-f", "10"], kw=dict(mid_occ=10)),
                                 dict(extra=["-f", "6", "-e", "100"], kw=dict(mid_occ=6, occ_dist=100)),
                                 dict(extra=["-f", "10", "--for-only"], kw=dict(mid_occ=10, flag=0x100000), strands="+"),
                                 dict(extra=["-f", "10", "--rev-only"], kw=dict(mid_occ=10, flag=0x200000), strands="-")])
def test_heap_seed_order_map_ont(tmp_path, cfg):
    _run(tmp_path, ["-x", "map-ont"] + cfg["extra"], cfg["kw"], 10, 15, strands=cfg.get("strands", "+-"))


def test_heap_seed_order_map_hifi(tmp_path):
    _run(tmp_path, ["-x", "map-hifi", "-f", "20"], dict(mid_occ=20), 19, 19)


def test_heap_seed_order_all_vs_all(tmp_path):
    """ava-ont with the reads as their own reference: skip_seed's diagonal and dual tests thin groups of equal occurrences"""
    _run(tmp_path, ["-x", "ava-ont", "-f", "20"], dict(mid_occ=20, occ_dist=0, flag=0x001 | 0x002), 5, 15, ava=True)
