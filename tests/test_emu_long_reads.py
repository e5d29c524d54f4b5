"""CPU: a reduced case of tests/test_gpu_long_reads.py under the SIMT emulator of tests/cuda_emu (every CUDA kernel source unchanged): a
2 Mbp genome with a 60 kb tandem array and seven ONT-like reads of 30-100 kb (tests/long_reads.py, write_all(small=True)). The seeding
stage against the oracle at map-ont's and lr:hqae's seeding parameters (reads of more than 2048 minimizers, minimizers the query filter
drops, a read of more than 8,192 anchors), the chaining stage (DP chainer and long-join rescue) against the reference's, and two command lines
against the reference binary's recorded output (tests/golden/expected/long_reference_lines.json)."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np
import pytest
import oracle_lib as O
import seed_check as SC
import chain_cases as CC
import long_reads as LR

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))
sys.path.insert(0, O.ROOT)


@pytest.fixture(scope="module")
def emu():
    import build_emu
    L = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    L.mmb_ctx_create.restype = C.c_void_p
    SC.setup(L)
    return L, C.c_void_p(L.mmb_ctx_create(0))


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return LR.write_all(str(tmp_path_factory.mktemp("long_small")), small=True)


_seeds = {}


def seeds(emu, data, preset):
    if preset not in _seeds:
        L, ctx = emu
        par = LR.seed_params(data["ctgs"], preset)
        reads = [bytes(r) for r in data["ont_set"][1]]
        keep = []
        SC.check_case(L, ctx, data["ctgs"], reads, keep=keep, **par)
        _seeds[preset] = par, reads, keep
    return _seeds[preset]


@pytest.mark.parametrize("preset", ["map-ont", "lr:hqae"])
def test_emulated_long_seed_stage(emu, data, preset):
    par, reads, anchors = seeds(emu, data, preset)
    w, k = par["w"], par["k"]
    n_sk = [SC.n_sketch(r, w, k) for r in reads]
    n_mz = [SC.n_minimizers(r, w, k, par["mid_occ"], par["q_occ_frac"]) for r in reads]
    assert sum(n > 2048 for n in n_mz) >= (3 if preset == "map-ont" else 1), n_mz  # select_kernel's global seed table
    if preset == "map-ont":  # mid_occ 10: the query-occurrence filter drops the tandem read's repeats
        assert any(a < b for a, b in zip(n_mz, n_sk)), (n_sk, n_mz)
    if preset == "lr:hqae":  # the tandem-array read: the largest shared-memory sort class
        assert max(len(a) for a in anchors) > 8192


def _call(L, ctx, fn, reads, par, *extra):
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    for i, a in enumerate(reads):
        off[i + 1] = off[i] + len(a)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in reads]))
    n = len(reads)
    n_u, n_v = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    u, ao = np.zeros(int(off[-1]) + 1, dtype=np.uint64), np.zeros((int(off[-1]) + 1, 2), dtype=np.uint64)
    ptr = lambda x: C.c_void_p(x.ctypes.data)
    if extra:
        r, ql = extra
        getattr(L, fn)(ctx, C.byref(par), C.byref(r), n, ptr(cat), ptr(off), ptr(np.ascontiguousarray(ql, dtype=np.int32)), ptr(n_u), ptr(n_v),
                       ptr(u), ptr(ao))
    else:
        getattr(L, fn)(ctx, C.byref(par), n, ptr(cat), ptr(off), ptr(n_u), ptr(n_v), ptr(u), ptr(ao))
    return [(u[int(off[i]):int(off[i]) + n_u[i]].copy(), ao[int(off[i]):int(off[i]) + n_v[i]].copy()) for i in range(n)]


def test_emulated_long_chain(emu, data):
    """the chaining stage as map-ont runs it: the DP chainer, then the long-join rescue at the default bw_long, with the reads' own
    lengths"""
    L, ctx = emu
    _, reads, anchors = seeds(emu, data, "map-ont")
    p, r = CC.dp_par(), dict(bw_long=20000, rescue_size=1000, rescue_ratio=0.1, max_dist=5000, max_dist_inner=1000, cap=100000)
    ql = [len(s) for s in reads]
    got = _call(L, ctx, "mmb_chain_rescue_batch_host", anchors, CC.chain_par(p), CC.rescue_par(r), ql)
    for j, a in enumerate(anchors):
        u, b, rescued = CC.expect_rescue(a, ql[j], p, r)
        CC.assert_same(got[j], (u, b), "rescue read %d (%d anchors, rescued %d)" % (j, len(a), rescued))


@pytest.fixture(scope="module")
def emu_cli():
    import build_emu
    lib = build_emu.build("mmb_emu_all", build_emu.ALL, extra=())
    exe = os.path.join(os.path.dirname(lib), "minimap2-emu")
    main = os.path.join(O.ROOT, "minimap2_b200", "cli", "main.cc")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(lib), os.path.getmtime(main)):
        subprocess.check_call(["g++", "-O1", "-I" + os.path.join(O.ROOT, "include"), "-o", exe, main, "-L" + os.path.dirname(lib), "-lmmb_emu_all",
                               "-Wl,-rpath,$ORIGIN", "-lpthread"])
    return exe


def _max_qlen(data):
    return sorted(len(r) for r in data["ont_set"][1])[2]


# no base-level alignment under the emulator (seconds per kilobase): mapping positions and chains only, of the three shortest reads
CLI = {"map_ont": ["-x", "map-ont", "--max-qlen", None], "lr_hqae": ["-x", "lr:hqae", "--max-qlen", None]}


@pytest.mark.parametrize("name", list(CLI))
def test_emulated_long_cli(emu_cli, data, name):
    n = _max_qlen(data)
    args = [str(n) if o is None else o for o in CLI[name]] + [data["ref"], data["ont"]]
    ref = LR.reference_lines(args)
    p = subprocess.run([emu_cli, "-t", "8"] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    got = p.stdout.decode().splitlines()
    O.assert_matches_reference(got, ref)
    lens = dict(zip(data["ont_set"][0], map(len, data["ont_set"][1])))
    mapped = {l.split("\t")[0] for l in got}
    assert any(lens[q] == n for q in mapped) and all(lens[q] <= n for q in mapped)  # the read of exactly N bases kept, longer ones dropped
