"""Loader for the product library libminimap2_b200.so (hand-written sm_90a CUDA + host C++ behind a C ABI).

There is no CPU fallback: if the library is missing this raises, and every GPU entry point aborts/raises when no
CUDA device is present. Nothing under oracle/ is ever imported from here."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libminimap2_b200.so")
_lib = None


class KswJob(C.Structure):  # mmb_ksw_job_t (include/mm_b200.h)
    _fields_ = [("q_start", C.c_int64), ("t_start", C.c_int64), ("q_step", C.c_int32), ("t_step", C.c_int32),
                ("qlen", C.c_int32), ("tlen", C.c_int32), ("w", C.c_int32), ("zdrop", C.c_int32),
                ("end_bonus", C.c_int32), ("flag", C.c_int32)]


class KswRes(C.Structure):  # mmb_ksw_res_t
    _fields_ = [("max", C.c_int32), ("zdropped", C.c_int32), ("max_q", C.c_int32), ("max_t", C.c_int32),
                ("mqe", C.c_int32), ("mqe_t", C.c_int32), ("mte", C.c_int32), ("mte_q", C.c_int32),
                ("score", C.c_int32), ("n_cigar", C.c_int32), ("reach_end", C.c_int32), ("cigar_off", C.c_uint32),
                ("zd_max", C.c_int32), ("zd_t0", C.c_int32), ("zd_t1", C.c_int32), ("zd_q0", C.c_int32), ("zd_q1", C.c_int32)]


class KswScore(C.Structure):  # mmb_ksw_score_t
    _fields_ = [("mat", C.c_int8 * 25), ("q", C.c_int8), ("e", C.c_int8), ("q2", C.c_int8), ("e2", C.c_int8),
                ("noncan", C.c_int8), ("junc_bonus", C.c_int8), ("junc_pen", C.c_int8), ("zd_skip", C.c_int16)]


class ChainPar(C.Structure):  # mmb_chain_par_t
    _fields_ = [("max_dist_x", C.c_int32), ("max_dist_y", C.c_int32), ("bw", C.c_int32), ("max_skip", C.c_int32),
                ("max_iter", C.c_int32), ("min_cnt", C.c_int32), ("min_sc", C.c_int32),
                ("chn_pen_gap", C.c_float), ("chn_pen_skip", C.c_float), ("is_cdna", C.c_int32), ("n_seg", C.c_int32),
                ("use_rmq", C.c_int32), ("max_dist_inner", C.c_int32), ("rmq_size_cap", C.c_int32)]


class RescuePar(C.Structure):  # mmb_rescue_par_t
    _fields_ = [("bw_long", C.c_int32), ("rescue_size", C.c_int32), ("rescue_ratio", C.c_float),
                ("max_dist", C.c_int32), ("max_dist_inner", C.c_int32), ("rmq_size_cap", C.c_int32)]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("minimap2_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(no CPU fallback exists)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.mmb_device_count.restype = C.c_int
        L.mmb_ctx_create.restype = C.c_void_p
        L.mmb_ctx_create.argtypes = [C.c_int]
        L.mmb_ctx_destroy.argtypes = [C.c_void_p]
        L.mmb_ctx_stream.restype = C.c_void_p
        L.mmb_ctx_stream.argtypes = [C.c_void_p]
        L.mmb_launch_count.restype = C.c_uint64
        L.mmb_launch_count.argtypes = [C.c_void_p, C.c_int]
        L.mmb_profile_enable.argtypes = [C.c_void_p, C.c_int]
        L.mmb_profile_ms.restype = C.c_double
        L.mmb_profile_ms.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.mmb_profile_units.restype = C.c_uint64
        L.mmb_profile_units.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.mmb_ksw_batch_host.restype = C.c_int64
        L.mmb_ksw_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                         C.c_int64, C.c_void_p, C.c_void_p, C.c_int64]
        L.mmb_sketch_batch_host.restype = C.c_int64
        L.mmb_sketch_batch_host.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint32,
                                            C.c_void_p, C.c_int64, C.c_void_p]
        L.mmb_chain_batch_host.restype = C.c_int
        L.mmb_chain_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.mmb_chain_rmq_batch_host.restype = C.c_int
        L.mmb_chain_rmq_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.mmb_chain_rescue_batch_host.restype = C.c_int
        L.mmb_chain_rescue_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.mmb_idx_lookup_host.restype = C.c_int64
        L.mmb_idx_lookup_host.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        _lib = L
    return _lib


class Context:
    """One per GPU (mmb_ctx_t)."""

    def __init__(self, device=0):
        L = lib()
        if L.mmb_device_count() <= 0:
            raise RuntimeError("minimap2_b200: no CUDA device visible; this library has no CPU path")
        self.h = L.mmb_ctx_create(device)
        if not self.h:
            raise RuntimeError("minimap2_b200: mmb_ctx_create(%d) failed" % device)
        self.device = device

    def close(self):
        if self.h:
            lib().mmb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
