"""CPU: K5 (junction jumps, jump.cuh) under the SIMT emulator, through mmb_jump_batch_host on the emulated product library, against
the restatement in jump_cases.py, over the hit sets of test_jump_vs_ref.py."""
import ctypes as C
import os
import sys
import types
import numpy as np
import jump_cases as J
import oracle_lib as O
from minimap2_b200 import kernels as K
from minimap2_b200.api import IdxOpt, MapOpt, Idx

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))


def test_emulated_k5_matches_restatement(tmp_path):
    import build_emu
    E = C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=()))
    d = J.make_data(seed=11)
    J.write_data(d, str(tmp_path))
    E.mm_set_opt.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.POINTER(MapOpt)]
    E.mm_idx_str.restype = C.POINTER(Idx)
    E.mm_idx_jjump_read.argtypes = [C.POINTER(Idx), C.c_char_p, C.c_int, C.c_int]
    E.mmb_ctx_create.restype = C.c_void_p
    io, mo = IdxOpt(), MapOpt()
    E.mm_set_opt(None, C.byref(io), C.byref(mo))
    E.mm_set_opt(b"splice", C.byref(io), C.byref(mo))
    seqs = (C.c_char_p * len(d["contigs"]))(*d["contigs"])
    names = (C.c_char_p * len(d["names"]))(*[n.encode() for n in d["names"]])
    mi = E.mm_idx_str(io.w, io.k, 0, io.bucket_bits, len(d["contigs"]), seqs, names)
    assert E.mm_idx_jjump_read(mi, str(tmp_path / "anno.bed").encode(), J.MM_JUNC_ANNO, -1) == 0
    from test_jump_vs_ref import entries, _setup
    _setup(E)
    tables = [[(e[0], e[1], e[4]) for e in entries(E, mi, c, -1, len(s))] for c, s in enumerate(d["contigs"])]
    t4 = [J.NT4[np.frombuffer(s, dtype=np.uint8)] for s in d["contigs"]]
    hits = J.hit_variants(d, np.random.default_rng(23))
    reads = [s for _, s in d["reads"]]
    ctx = types.SimpleNamespace(h=E.mmb_ctx_create(0))
    acts = set()
    for jmm in (3, 30):
        mo.jump_min_match = jmm
        got = K.jump_batch(ctx, mi, mo, reads, hits, L=E)
        for h, g in zip(hits, got):
            assert g == J.decide(h, reads[h["read"]], t4[h["rid"]], tables[h["rid"]], mo.a, mo.b, jmm), h
            acts.update((g[0][0], g[1][0]))
    assert {0, 1, 2} <= acts
