"""Cost of junction jumps on the GPU: maps a spliced read set (jump_cases generator, about 10^5 reads from genes of 14 to 21 exons;
the read lengths run from tens of bases to about 3 kb and the median is printed) with -x splice, without and then
with an annotation jump table, and prints one JSON line: the device name and power limit, the mapping time of both runs (host clock
around mm_map_batch, which returns after the device work; profiling off), the time of the jump stage's kernel (K5: CUDA events of the
profiling family it is counted in, with and without the table, in a separate run whose read groups run one after another so that
the events time one group's kernels only), and how many hits the jumps changed. Usage: python tests/jump_probe.py [--genes N] [--reads-per-gene M]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import jump_cases as J
import minimap2_b200 as mb
from minimap2_b200.api import Aligner, Reg1, Extra

PROF_OTHER = 5


def hit_sig(n_regs, regs):
    out = []
    for i in range(len(n_regs)):
        arr = C.cast(C.c_void_p(int(regs[i])), C.POINTER(Reg1)) if regs[i] else None
        for j in range(n_regs[i]):
            r = arr[j]
            ex = r.p.contents if r.p else None
            cig = tuple((C.c_uint32 * ex.n_cigar).from_address(C.addressof(ex) + C.sizeof(Extra))) if ex else ()
            out.append((i, r.rs, r.re, r.qs, r.qe, cig))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--reads-per-gene", type=int, default=50)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    d = J.make_data(seed=7, n_contigs=10, genes_per_contig=a.genes // 10, reads_per_gene=a.reads_per_gene, n_exons=(14, 22))
    tmp = tempfile.mkdtemp(prefix="jump_probe.")
    J.write_data(d, tmp)
    reads = [s for _, s in d["reads"]]
    buf = np.frombuffer(b"".join(reads), dtype=np.uint8)
    qlens = np.array([len(s) for s in reads], dtype=np.int32)
    names = [n for n, _ in d["reads"]]
    al = Aligner(os.path.join(tmp, "ref.fa"), preset="splice", n_threads=16)
    L = mb.lib()
    L.mm_idx_jjump_read.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int]
    prep = al.prepare_batch(buf, qlens, names)
    res = {}
    for tag in ("no_jump", "jump"):
        if tag == "jump":
            assert L.mm_idx_jjump_read(C.cast(al._idx, C.c_void_p), os.path.join(tmp, "anno.bed").encode(), J.MM_JUNC_ANNO, -1) == 0
        nr, rg, _ = al.map_prepared(prep)  # warm-up
        sig = hit_sig(nr, rg)
        Aligner.free_batch(nr, rg)
        ts = []
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            nr, rg, _ = al.map_prepared(prep)
            ts.append(time.perf_counter() - t0)
            Aligner.free_batch(nr, rg)
        L.mmb_set_groups(-12)
        L.mmb_profile_enable_all(1)
        L.mmb_profile_ms_all(PROF_OTHER, 1)
        nr, rg, _ = al.map_prepared(prep)
        Aligner.free_batch(nr, rg)
        other_ms = L.mmb_profile_ms_all(PROF_OTHER, 1)
        L.mmb_profile_enable_all(0)
        L.mmb_set_groups(0)
        res[tag] = dict(map_s=min(ts), other_family_ms=other_ms, sig=sig)
    changed = sum(x != y for x, y in zip(res["jump"]["sig"], res["no_jump"]["sig"]))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE).stdout.decode().strip()
    k5_ms = res["jump"]["other_family_ms"] - res["no_jump"]["other_family_ms"]
    print(json.dumps(dict(gpu=gpu, n_reads=len(reads), bases=int(qlens.sum()), median_read_len=int(np.median(qlens)), n_hits=len(res["jump"]["sig"]), hits_changed=changed,
                          map_s_without=round(res["no_jump"]["map_s"], 4), map_s_with=round(res["jump"]["map_s"], 4),
                          k5_ms=round(k5_ms, 3), k5_share_of_step=round(k5_ms / 1e3 / res["jump"]["map_s"], 5))))


if __name__ == "__main__":
    main()
