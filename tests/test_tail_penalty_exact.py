"""CPU: the gap penalty of mm_update_extra (align.c:283,292), q + e * mg_log2(1 + len), is exact in 2^-32 fixed point.

The reference keeps that function's running score in double. The host driver (Driver::update_extra, csrc/align.cc) and the device
tail (finalize_kernel, csrc/finalize.cu) keep it as an int64 in units of 2^-32, with q and e taken as int8_t. That is the same
arithmetic only if every penalty times 2^32 is an integer the double holds exactly. This file checks that for every int8_t pair
(q, e), with mmx_log2 (csrc/mm_algo.cuh) restated bit for bit in float32."""
import ctypes as C

import numpy as np

import oracle_lib as O


def mmx_log2(x):
    """mmx_log2 on a float32 array: the same bit operations and the same float32 evaluation order"""
    i = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = (((i >> np.uint32(23)) & np.uint32(255)).astype(np.int32) - 128).astype(np.float32)
    z = ((i & np.uint32(~(255 << 23) & 0xFFFFFFFF)) + np.uint32(127 << 23)).view(np.float32)
    return r + ((np.float32(-0.34484843) * z + np.float32(2.02466578)) * z - np.float32(0.67487759))


def gap_log2(lens):
    """mmx_log2(1.0 + len) as the callers evaluate it: 1.0 + len in double, rounded to float"""
    return mmx_log2((1.0 + np.asarray(lens, dtype=np.float64)).astype(np.float32))


def spread_of_lengths():
    p2 = [1 << k for k in range(32)]
    lens = set(range(1, 4097)) | set(p2) | {v + d for v in p2 for d in (-1, 1)}
    lens |= set(np.random.default_rng(7).integers(1, 1 << 28, 2000).tolist())
    return np.array(sorted(v for v in lens if 1 <= v <= 1 << 31), dtype=np.int64)


def test_restatement_matches_oracle():
    L = O.oracle()
    L.mm2o_log2.restype, L.mm2o_log2.argtypes = C.c_float, [C.c_float]
    lens = spread_of_lengths()
    got = gap_log2(lens)
    exp = np.array([L.mm2o_log2(float(np.float32(1.0 + v))) for v in lens], dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


def test_log2_in_range():
    """mmx_log2(1 + len) lies in [1, 33): a float that is a multiple of 2^-23"""
    for lens in (np.arange(1, (1 << 24) + 1, dtype=np.int64), np.array([1 << k for k in range(32)], dtype=np.int64)):
        r = gap_log2(lens)
        assert r.min() >= 1.0 and r.max() < 33.0, (r.min(), r.max())


def test_penalty_exact_in_fixed_point():
    """for every int8_t (q, e): (q + e * r) * 2^32 is computed exactly in double, is an integer and is below 2^45 in magnitude"""
    r = gap_log2(spread_of_lengths()).astype(np.float64)
    r_fx = r * 2.0 ** 32
    assert np.all(r_fx == np.floor(r_fx))
    r_fx = r_fx.astype(np.int64)                   # exact: r < 33, so r * 2^32 < 2^38
    q = np.arange(-128, 128, dtype=np.int64)[:, None]
    for e in range(-128, 128):
        pen = (q.astype(np.float64) + float(e) * r[None, :]) * 2.0 ** 32   # the callers' double arithmetic
        exact = (q << 32) + e * r_fx[None, :]      # the same value in integers
        assert np.all(np.abs(exact) < 1 << 45)
        assert np.array_equal(pen, exact.astype(np.float64)), e   # exact < 2^45 converts to double without rounding
    qq, ee = np.meshgrid(np.arange(-128, 128, dtype=np.int64), np.arange(-128, 128, dtype=np.int64))
    pen = (qq + ee).astype(np.float64) * 2.0 ** 32  # the penalty without the log term
    assert np.array_equal(pen, ((qq + ee) << 32).astype(np.float64)) and np.all(np.abs(pen) < 2.0 ** 45)
