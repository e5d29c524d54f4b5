"""Scheduler timeline of the bench workload (not a pytest; needs a GPU):

  python tests/sched_timeline.py [--workload map-ont] [--pairs 4] [--slots 4,8] [--trace-steps 2] [--out DIR]

Builds bench.py's input for the workload (same synthetic index and reads), warms up, then runs steps with the reads resident in
HBM (A, what bench.py's `value` times) and with host buffers (B, `e2e`) alternately, ABAB..., so that an order effect between
the two cannot pass for a difference between them. For every step it prints the wall time and, from the scheduler timeline
(mmb_timeline_get: host timestamps the scheduler records at each phase boundary without synchronising anything):
  gate      time the groups spent waiting for a device slot (sum over groups; stage 1 / waves)
  dev       time the groups held a slot (sum over groups)
  host      time the groups spent in host phases (sum over groups), and the host time spent while holding a slot
  noslot    wall time during which no group held a device slot
  end1      when the last group finished stage 1
and the host phases summed over groups. Then, in a separate run under torch.profiler (CUDA activity), it reports per step the
union of kernel execution intervals over all streams and the GPU-idle time (wall minus that union).
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GATE_REQ, GATE_GRANT, GATE_REL, ENQUEUED, SYNC, HOST_BEGIN, HOST_END = range(7)
PHASES = ["concat", "hits", "replay", "tail_prep", "tail_apply", "jobs", "ksw_plan", "scatter", "finalize"]
MAX_GROUPS = 16


def union_len(iv):
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        tot += cur_e - cur_s
    return tot


def overlap(iv, jv):
    """total length of the intersection of two interval lists (each without self-overlap)"""
    tot = 0.0
    for s, e in iv:
        for s2, e2 in jv:
            tot += max(0.0, min(e, e2) - max(s, s2))
    return tot


def read_timeline(L):
    out = {}
    for g in range(MAX_GROUPS):
        n = L.mmb_timeline_get(g, None, 0)
        if n <= 0:
            continue
        arr = (C.c_double * (3 * n))()
        L.mmb_timeline_get(g, arr, n)
        out[g] = [(arr[3 * i], int(arr[3 * i + 1]), int(arr[3 * i + 2])) for i in range(n)]
    return out


def analyse(tl, t0, t1):
    """per-step summary of the timeline of every group (times in ms)"""
    slots_all, gate = [], [0.0, 0.0]
    dev = host = host_in_slot = 0.0
    phase = [0.0] * len(PHASES)
    n_sync = 0
    end1 = 0.0
    groups = {}
    for g, recs in tl.items():
        req, grant, hb = {}, {}, {}
        held, hostiv = [], []
        first_grant1 = rel1 = None
        for t, ev, arg in recs:
            if ev == GATE_REQ:
                req[arg] = t
            elif ev == GATE_GRANT:
                grant[arg] = t
                gate[arg] += t - req.pop(arg, t)
                if arg == 0 and first_grant1 is None:
                    first_grant1 = t
            elif ev == GATE_REL:
                s = grant.pop(arg, t)
                held.append((s, t))
                if arg == 0:
                    rel1 = t
                    end1 = max(end1, t - t0)
            elif ev == HOST_BEGIN:
                hb[arg] = t
            elif ev == HOST_END:
                s = hb.pop(arg, t)
                phase[arg] += t - s
                hostiv.append((s, t))
            elif ev == SYNC:
                n_sync += 1
        slots_all += held
        dev += sum(e - s for s, e in held)
        host += sum(e - s for s, e in hostiv)
        host_in_slot += overlap(hostiv, held)
        groups[g] = {"grant1": None if first_grant1 is None else 1e3 * (first_grant1 - t0), "rel1": None if rel1 is None else 1e3 * (rel1 - t0),
                     "end": 1e3 * (recs[-1][0] - t0)}
    noslot = (t1 - t0) - union_len([(max(s, t0), min(e, t1)) for s, e in slots_all if e > s])
    return {"wall": 1e3 * (t1 - t0), "gate1": 1e3 * gate[0], "gatew": 1e3 * gate[1], "dev": 1e3 * dev, "host": 1e3 * host,
            "host_in_slot": 1e3 * host_in_slot, "noslot": 1e3 * noslot, "end1": 1e3 * end1, "syncs": n_sync,
            "phases": {PHASES[k]: 1e3 * v for k, v in enumerate(phase)}, "groups": groups}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="map-ont")
    ap.add_argument("--reads", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=4, help="A/B step pairs per slot count")
    ap.add_argument("--slots", default="0", help="comma-separated device slot counts to run (0: the scheduler's default)")
    ap.add_argument("--trace-steps", type=int, default=2, help="A and B steps each in the profiler run (0: no trace)")
    ap.add_argument("--out", default=None, help="directory for timeline.json and the profiler trace")
    a = ap.parse_args()

    from bench import WORKLOADS, gen_reads, apply_output_flags
    wl = dict(WORKLOADS[a.workload])
    if a.reads:
        wl["reads"] = a.reads
    n_reads, read_len = int(wl["reads"]), int(wl["read_len"])
    ncpu = os.cpu_count() or 1
    os.environ.setdefault("MM_B200_HOST_THREADS", str(ncpu // 2))  # as bench.py sets it for one rank
    import numpy as np
    import torch
    torch.cuda.set_device(0)
    from minimap2_b200 import api
    L = api._setup()
    L.mmb_timeline_enable.argtypes = [C.c_int]
    L.mmb_timeline_now.restype = C.c_double
    L.mmb_timeline_get.restype = C.c_int64
    L.mmb_timeline_get.argtypes = [C.c_int, C.c_void_p, C.c_int64]
    L.mmb_set_gpu_slots.argtypes = [C.c_int]
    if wl["kind"] != "genomic":
        sys.exit("sched_timeline: genomic workloads only (map-ont, map-hifi)")
    gidx = L.mmb_synth_index(int(wl["genome_mbp"] * 1e6), int(wl["contigs"]), 11, wl["w"], wl["k"], 14)
    buf = np.zeros(n_reads * read_len, dtype=np.uint8)
    gen_reads(L, gidx, wl, n_reads, read_len, 12, buf)
    al = api.Aligner(preset=wl["preset"], _idx=gidx, n_threads=ncpu)
    al.map_opt.flag &= ~0x004
    apply_output_flags(al.map_opt, wl)
    prepared = al.prepare_batch(buf, np.full(n_reads, read_len, dtype=np.int32), ["r%d" % i for i in range(n_reads)])
    name = torch.cuda.get_device_name(0)
    print("device: %s; %s; %d reads x %d bp; %d logical CPUs, host pool %s" % (name, a.workload, n_reads, read_len, ncpu, os.environ["MM_B200_HOST_THREADS"]), flush=True)

    def step(resident, timeline=True):
        L.mmb_set_resident_reads(1 if resident else 0)
        L.mmb_timeline_enable(1 if timeline else 0)
        t0 = L.mmb_timeline_now()
        n_regs, regs, _ = al.map_prepared(prepared)
        torch.cuda.synchronize()
        t1 = L.mmb_timeline_now()
        L.mmb_timeline_enable(0)
        res = analyse(read_timeline(L), t0, t1) if timeline else {"wall": 1e3 * (t1 - t0)}
        al.free_batch(n_regs, regs)
        return res

    for _ in range(a.warmup):
        step(True, False)
    results = []
    for slots in [int(x) for x in a.slots.split(",")]:
        L.mmb_set_gpu_slots(slots)
        print("\nslots %s  (ms; gate/dev/host summed over groups)" % (slots or "default"))
        print("%-4s %7s %7s %7s %7s %7s %7s %7s %7s  %s" % ("mode", "wall", "noslot", "end1", "gate1", "gatew", "dev", "host", "h@slot",
                                                       " ".join("%9s" % p for p in PHASES)))
        rows = {"A": [], "B": []}
        for i in range(a.pairs):
            for mode in "AB":
                r = step(mode == "A")
                r["mode"], r["slots"] = mode, slots
                rows[mode].append(r)
                results.append(r)
                print("%-4s %7.1f %7.1f %7.1f %7.1f %7.1f %7.1f %7.1f %7.1f  %s" % (
                    mode, r["wall"], r["noslot"], r["end1"], r["gate1"], r["gatew"], r["dev"], r["host"], r["host_in_slot"],
                    " ".join("%9.1f" % r["phases"][p] for p in PHASES)), flush=True)
        for mode in "AB":
            w = sorted(r["wall"] for r in rows[mode])
            print("  %s: median wall %.1f ms (min %.1f, max %.1f), median no-slot %.1f ms" % (
                mode, w[len(w) // 2], w[0], w[-1], sorted(r["noslot"] for r in rows[mode])[len(w) // 2]))
        last = rows["A"][-1]
        print("  last A step, per group (ms from step start): stage-1 grant / release / end")
        print("  " + "  ".join("g%d %.0f/%.0f/%.0f" % (g, v["grant1"] or -1, v["rel1"] or -1, v["end"]) for g, v in sorted(last["groups"].items())))
    L.mmb_set_gpu_slots(0)

    trace = None
    if a.trace_steps > 0:
        from torch.profiler import profile, ProfilerActivity, record_function
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for i in range(a.trace_steps):
                for mode in "AB":
                    with record_function("step_%s_%d" % (mode, i)):
                        step(mode == "A", False)
        path = os.path.join(a.out or "/tmp", "sched_%d.pt.trace.json" % os.getpid())
        prof.export_chrome_trace(path)
        ev = json.load(open(path)).get("traceEvents", [])
        kern = [(e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("ph") == "X" and e.get("cat") == "kernel"]
        copies = [(e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("ph") == "X" and e.get("cat") in ("gpu_memcpy", "gpu_memset")]
        wins = sorted((e["name"], e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("ph") == "X" and str(e.get("name", "")).startswith("step_")
                      and e.get("cat") == "user_annotation")
        print("\nprofiler run (CUDA activity; slower than the timed runs): %d kernels, %d copies" % (len(kern), len(copies)))
        trace = []
        for nm, s, e in wins:
            kin = [(max(s, x), min(e, y)) for x, y in kern if y > s and x < e]
            cin = [(max(s, x), min(e, y)) for x, y in copies if y > s and x < e]
            busy, busy_c = union_len(kin) / 1e3, union_len(kin + cin) / 1e3
            wall = (e - s) / 1e3
            trace.append({"step": nm, "wall": wall, "kernel_busy": busy, "gpu_idle": wall - busy, "idle_no_copy": wall - busy_c,
                          "kernel_sum": sum(y - x for x, y in kin) / 1e3})
            print("  %-9s wall %7.1f ms  kernel-busy union %7.1f  GPU idle %6.1f  (idle incl. copies as busy %6.1f; kernel time summed %7.1f)" % (
                nm, wall, busy, wall - busy, wall - busy_c, trace[-1]["kernel_sum"]))
        if not a.out:
            os.unlink(path)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "timeline.json"), "w") as f:
            json.dump({"device": name, "workload": a.workload, "steps": results, "trace": trace}, f)
    al.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
