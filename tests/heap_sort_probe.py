"""Cost of heap-ordered seeding (`--heap-sort=yes`, MM_F_HEAP_SORT) on the GPU. Two workloads on bench.py's synthetic map-ont genome:
the bench's map-ont read set (reads of 10 kb), and about 10^6 reads of 150 bp mapped with the same long-read preset. Each is mapped
with the flag off and on, alternately, and the probe prints one JSON line: the device name and power limit, and per workload and
mode the mapping time (host clock around mm_map_batch, which returns after the device work; profiling off; best of the rounds), the
device time of the seed and sort profiling families (CUDA events, in a separate run whose read groups run one after another), the
kernel launches of one mapping, and the number of reads whose anchors have equal keys (the reads heap mode replays; counted by a
child process with the sort stage's statistics switched on). Usage: python tests/heap_sort_probe.py [--long-reads N] [--short-reads N]"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from minimap2_b200 import api
from minimap2_b200.api import Aligner

HEAP = 0x400000
PROF_SEED, PROF_SORT = 1, 2


def workloads(L, idx, a):
    out = []
    for tag, n, ln in (("map-ont_10kb", a.long_reads, 10000), ("map-ont_150bp", a.short_reads, 150)):
        buf = np.zeros(n * ln, dtype=np.uint8)
        L.mmb_synth_reads(idx, n, ln, 12, 0.10, 0.40, 0.25, buf.ctypes.data)
        out.append((tag, buf, np.full(n, ln, dtype=np.int32)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-mbp", type=float, default=3000.0)
    ap.add_argument("--long-reads", type=int, default=30000)
    ap.add_argument("--short-reads", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--count-ties", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    ties = {}
    if not a.count_ties:  # first, while this process holds no device memory: the child maps once in heap mode with the sort statistics on
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--count-ties", "--genome-mbp", str(a.genome_mbp), "--long-reads", str(a.long_reads),
                            "--short-reads", str(a.short_reads)], env=dict(os.environ, MM_B200_SORT_STATS="1"), stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert p.returncode == 0, p.stderr.decode()[-2000:]
        cur = None
        for l in p.stderr.decode().splitlines():
            if l.startswith("[workload] "):
                cur = l.split()[1]
                ties[cur] = 0
            m = re.search(r" ties=(\d+)", l)
            if m and cur:
                ties[cur] += int(m.group(1))
    L = api._setup()
    L.mmb_profile_ms_all.restype = C.c_double
    L.mmb_launch_count_all.restype = C.c_uint64
    idx = L.mmb_synth_index(int(a.genome_mbp * 1e6), 24, 11, 10, 15, 14)
    al = Aligner(preset="map-ont", _idx=idx, n_threads=16)
    base_flag = al.map_opt.flag
    wls = workloads(L, idx, a)
    if a.count_ties:  # child: one heap-mode mapping per workload, the sort statistics go to stderr
        al.map_opt.flag = base_flag | HEAP
        for tag, buf, qlens in wls:
            print("[workload] " + tag, file=sys.stderr, flush=True)
            nr, rg, _ = al.map_prepared(al.prepare_batch(buf, qlens))
            Aligner.free_batch(nr, rg)
        return
    res = {}
    for tag, buf, qlens in wls:
        prep = al.prepare_batch(buf, qlens)
        r = {m: dict(map_s=[]) for m in ("off", "on")}
        for m in ("off", "on"):  # warm-up
            al.map_opt.flag = base_flag | (HEAP if m == "on" else 0)
            nr, rg, _ = al.map_prepared(prep)
            Aligner.free_batch(nr, rg)
        for _ in range(a.rounds):
            for m in ("off", "on"):
                al.map_opt.flag = base_flag | (HEAP if m == "on" else 0)
                L.mmb_launch_count_all(1)
                t0 = time.perf_counter()
                nr, rg, _ = al.map_prepared(prep)
                r[m]["map_s"].append(time.perf_counter() - t0)
                r[m]["launches"] = int(L.mmb_launch_count_all(1))
                r[m]["n_hits"] = int(nr.sum())
                Aligner.free_batch(nr, rg)
        for m in ("off", "on"):
            al.map_opt.flag = base_flag | (HEAP if m == "on" else 0)
            L.mmb_set_groups(-12)
            L.mmb_profile_enable_all(1)
            L.mmb_profile_ms_all(PROF_SEED, 1), L.mmb_profile_ms_all(PROF_SORT, 1)
            nr, rg, _ = al.map_prepared(prep)
            Aligner.free_batch(nr, rg)
            r[m]["seed_ms"] = round(L.mmb_profile_ms_all(PROF_SEED, 1), 2)
            r[m]["sort_ms"] = round(L.mmb_profile_ms_all(PROF_SORT, 1), 2)
            L.mmb_profile_enable_all(0)
            L.mmb_set_groups(0)
            r[m]["map_s"] = round(min(r[m]["map_s"]), 4)
        res[tag] = dict(n_reads=len(qlens), read_len=int(qlens[0]), reads_with_ties=ties[tag], **{"heap_" + m: v for m, v in r.items()})
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE).stdout.decode().strip()
    print(json.dumps(dict(gpu=gpu, genome_mbp=a.genome_mbp, workloads=res)))


if __name__ == "__main__":
    main()
