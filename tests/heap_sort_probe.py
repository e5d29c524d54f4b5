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


def reads_with_ties(L, idx, opt, flag, buf, qlens, chunk=2000):
    """reads whose sorted anchors (first seeding pass, at mid_occ) have equal neighbouring keys and at most 16384 anchors: the reads the
    sort kernels list for the heap merge in heap mode"""
    L.mmb_seed_batch_host.restype = C.c_int64
    L.mmb_seed_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
    ctx = L.mmb_ctx_create(0)
    off_all = np.concatenate([[0], np.cumsum(qlens, dtype=np.int64)])
    n_tie = 0
    for r0 in range(0, len(qlens), chunk):
        r1 = min(r0 + chunk, len(qlens))
        off = off_all[r0:r1 + 1] - off_all[r0]
        seq = np.concatenate([buf[off_all[r0]:off_all[r1]], np.zeros(1, dtype=np.uint8)])
        a_off = np.zeros(r1 - r0 + 1, dtype=np.int64); rep = np.zeros(r1 - r0, dtype=np.int32); nmini = np.zeros(r1 - r0, dtype=np.int32)
        a = np.zeros((1, 2), dtype=np.uint64)
        for _ in range(2):  # the second call with room for every anchor
            tot = L.mmb_seed_batch_host(ctx, idx, r1 - r0, seq.ctypes.data, off.ctypes.data, flag, opt.mid_occ, opt.q_occ_frac, opt.max_max_occ,
                                        opt.occ_dist, a_off.ctypes.data, rep.ctypes.data, nmini.ctypes.data, a.ctypes.data, len(a), None, 0)
            if tot >= 0:
                break
            a = np.zeros((int(a_off[-1]) + 1, 2), dtype=np.uint64)
        eq = np.zeros(len(a), dtype=bool)
        eq[1:] = a[1:, 0] == a[:-1, 0]
        for i in range(r1 - r0):
            s, e = int(a_off[i]), int(a_off[i + 1])
            n_tie += int(e - s <= 16384 and eq[s + 1:e].any())
    L.mmb_ctx_destroy(ctx)
    return n_tie


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-mbp", type=float, default=3000.0)
    ap.add_argument("--long-reads", type=int, default=30000)
    ap.add_argument("--short-reads", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    L = api._setup()
    L.mmb_profile_ms_all.restype = C.c_double
    L.mmb_launch_count_all.restype = C.c_uint64
    idx = L.mmb_synth_index(int(a.genome_mbp * 1e6), 24, 11, 10, 15, 14)
    al = Aligner(preset="map-ont", _idx=idx, n_threads=16)
    base_flag = al.map_opt.flag
    wls = workloads(L, idx, a)
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
        res[tag] = dict(n_reads=len(qlens), read_len=int(qlens[0]), reads_with_ties=reads_with_ties(L, idx, al.map_opt, base_flag, buf, qlens), **{"heap_" + m: v for m, v in r.items()})
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE).stdout.decode().strip()
    print(json.dumps(dict(gpu=gpu, genome_mbp=a.genome_mbp, workloads=res)))


if __name__ == "__main__":
    main()
