"""Cases and checkers of the anchor sort alone (the sort block of the seeding stage, radix_sort_128x of map.c:202) through
kernels.anchor_sort_batch (mmb_anchor_sort_host). Used by tests/test_gpu_anchor_sort.py and, on a reduced set, tests/test_emu_anchor_sort.py.

Expected order: the reference's own radix_sort_128x (oracle_lib.ref_sort128). Every anchor's y is read << 32 | index, so the order of
equal keys is seen. Expected route: route() below, from the anchor count n, the number of key bits that vary, nb = popcount(OR(x ^ x0)),
and whether the reference's output has equal neighbours -- what the kernels' routing must decide:
  * n = 0: no route; n <= 1024 << c: shared-memory radix class c (0-4); n > 16384: oversize (sort_exact_kernel, global memory);
  * nb > 33 (32 position bits plus the strand bit): the radix kernels hand the read on to the network sort (sort_block_kernel);
  * equal keys and n > 64: listed for the exact emulation of the unstable sort (sort_exact_smem_kernel), which passes reads of more than
    15360 anchors on to sort_exact_kernel.
Each generator returns a list of (name, x) with x the uint64 keys of one read in input order."""
import collections
import numpy as np
import oracle_lib as O

NONE, OVERSIZE, NETWORK, EXACT, GLOBAL = -1, 5, 8, 16, 32  # MMB_SORT_ROUTE_* (include/mm_b200.h)
CAP0, N_CLS, TIE_MIN_N, EXACT_SMEM_CAP = 1024, 5, 64, 15360
# every route a read can take: no anchors; a class, with or without the network sort and the exact listing; the two ways on to the
# global-memory walker (only class 4 holds reads of more than 15360 anchors); oversize
ALL_ROUTES = sorted({NONE, OVERSIZE} | {c | f for c in range(N_CLS) for f in (0, NETWORK, EXACT, NETWORK | EXACT)}
                    | {4 | EXACT | GLOBAL, 4 | NETWORK | EXACT | GLOBAL})
U64 = np.uint64


def n_vary(x):
    x = np.asarray(x, dtype=U64)
    return 0 if len(x) == 0 else bin(int(np.bitwise_or.reduce(x ^ x[0]))).count("1")


def has_ties(sorted_x):
    return len(sorted_x) > 1 and bool((sorted_x[1:] == sorted_x[:-1]).any())


def route(x, ref_sorted_x):
    n = len(x)
    if n == 0:
        return NONE
    c, cap = 0, CAP0
    while c < N_CLS - 1 and n > cap:
        c, cap = c + 1, cap << 1
    if n > cap:
        return OVERSIZE
    r = c | (NETWORK if n_vary(x) > 33 else 0)
    if n > TIE_MIN_N and has_ties(ref_sorted_x):
        r |= EXACT | (GLOBAL if n > EXACT_SMEM_CAP else 0)
    return r


def anchors(rd, x):
    a = np.zeros((len(x), 2), dtype=U64)
    a[:, 0] = x
    a[:, 1] = (U64(rd) << U64(32)) | np.arange(len(x), dtype=U64)
    return a


def check_batch(ctx, cases, L=None):
    """sorts every case in one batch and compares order and route with the reference; returns a Counter of the routes seen"""
    from minimap2_b200 import kernels as K
    arrs = [anchors(i, x) for i, (_, x) in enumerate(cases)]
    got, routes = K.anchor_sort_batch(ctx, arrs, L=L)
    seen = collections.Counter()
    for i, ((name, x), a, g) in enumerate(zip(cases, arrs, got)):
        ref = O.ref_sort128(a)
        assert g.shape == ref.shape, (name, g.shape, ref.shape)
        if not (g == ref).all():
            j = int(np.argmax((g != ref).any(axis=1)))
            raise AssertionError("%s (n=%d, nb=%d): first difference at %d: got %s, reference %s" % (name, len(x), n_vary(x), j, g[j], ref[j]))
        want = route(x, ref[:, 0])
        assert routes[i] == want, (name, len(x), n_vary(x), int(routes[i]), want)
        seen[want] += 1
    return seen


# ---------------- key construction ----------------
def scatter(v, mask):
    """places the low bits of v on the set bits of mask, in order"""
    v = np.asarray(v, dtype=U64)
    out = np.zeros(len(v), dtype=U64)
    k = 0
    for b in range(64):
        if mask >> b & 1:
            out |= ((v >> U64(k)) & U64(1)) << U64(b)
            k += 1
    return out


def keys(rng, n, mask, ties, base=None):
    """n keys that vary exactly in the bits of mask (when n allows), with (ties=True) or without equal keys; base: the other bits"""
    nb = bin(mask).count("1")
    base = int(rng.integers(0, 1 << 63, dtype=np.uint64)) * 2 + int(rng.integers(0, 2)) if base is None else base
    base &= ~mask & ((1 << 64) - 1)
    space = 1 << nb
    if n == 0:
        return np.zeros(0, dtype=U64)
    if not ties and n > space:
        raise ValueError("no %d distinct keys in %d bits" % (n, nb))
    n_dist = n if not ties else max(1, min(space, n - max(1, n // 4)))
    if space <= 1 << 22:
        vals = rng.choice(space, size=min(space, n_dist + 2), replace=False).astype(U64)
    else:
        vals = rng.integers(0, space if nb < 64 else 1 << 64, size=n_dist + 32, dtype=np.uint64)
        vals = rng.permutation(np.unique(vals))
    top = U64(space - 1)
    if nb > 0:  # every bit of the mask varies: one key all zeros, one all ones there
        vals = np.concatenate([np.array([0, top][:min(2, n_dist)], dtype=U64), vals[(vals != U64(0)) & (vals != top)]])
    vals = vals[:n_dist]
    assert len(vals) == n_dist
    v = vals if not ties else np.concatenate([vals, rng.choice(vals, size=n - n_dist)])
    return scatter(rng.permutation(v), mask) | U64(base)


def bits(*ranges):
    m = 0
    for lo, hi in ranges:  # bits lo..hi inclusive
        m |= ((1 << (hi - lo + 1)) - 1) << lo
    return m


POS = bits((0, 27))  # typical mapper keys: strand << 63 | contig << 32 | position


def real_mask(n_ctg_bits=3):
    return POS | bits((32, 32 + n_ctg_bits - 1)) | 1 << 63


# ---------------- generator families ----------------
SIZES = [1, 2, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 2049, 4096, 4097, 8192, 8193, 15359, 15360, 15361, 16383, 16384, 16385]


def sizes(rng, ns=SIZES, oversize=(40_000, 120_000, 200_000)):
    """every class boundary, with and without equal keys; reads without anchors; oversize reads"""
    out = [("n0", np.zeros(0, dtype=U64))]
    for n in list(ns) + list(oversize):
        out.append(("n%d_distinct" % n, keys(rng, n, real_mask(), False)))
        if n >= 2:
            out.append(("n%d_ties" % n, keys(rng, n, real_mask(), True)))
    return out


WIDTHS = [0, 1, 7, 8, 9, 16, 24, 31, 32, 33, 34, 64]


def width_mask(rng, nb, scattered):
    if nb == 64:
        return (1 << 64) - 1
    if not scattered:
        return bits((0, nb - 1)) if nb <= 32 else bits((0, 31)) | bits((64 - (nb - 32), 63))  # position bits, then strand / contig from the top
    return sum(1 << int(b) for b in rng.choice(64, size=nb, replace=False))


def widths(rng, ns=(300, 3000)):
    """key widths around the byte digits of the radix passes and the 32/33-bit limit of the squeezed key, contiguous and scattered"""
    out = []
    for nb in WIDTHS:
        for n in ns:
            for scattered in (False, True) if 0 < nb < 64 else (False,):
                m = width_mask(rng, nb, scattered)
                tag = "nb%d_%s_n%d" % (nb, "scat" if scattered else "low", n)
                if n <= 1 << nb:
                    out.append((tag + "_distinct", keys(rng, n, m, False)))
                out.append((tag + "_ties", keys(rng, n, m, True)))
    return out


def placement(rng, n=2000):
    """where the varying bits sit: a single bit at 0 and at 63; runs split over position, contig and strand bits; runs across byte
    boundaries; a byte without varying bits between bytes that vary (the exact walker's vary mask skips it)"""
    masks = dict(bit0=1, bit63=1 << 63, pos_ctg_strand=bits((0, 27), (32, 35), (63, 63)), pos_strand=bits((0, 31), (63, 63)),
                 straddle_4_11=bits((4, 11)), straddle_4_19=bits((4, 19)), straddle_28_36=bits((28, 36)), straddle_60_63_0_3=bits((0, 3), (60, 63)),
                 gap_byte1=bits((0, 7), (16, 23)), gap_byte6=bits((40, 47), (56, 63)), gap_bytes_1_to_6=bits((0, 7), (56, 63)),
                 sparse_one_per_byte=sum(1 << (8 * i + 3) for i in range(8)))
    out = []
    for name, m in masks.items():
        nb = bin(m).count("1")
        if n <= 1 << nb:
            out.append((name + "_distinct", keys(rng, n, m, False)))
        out.append((name + "_ties", keys(rng, n, m, True)))
        out.append((name + "_n2", keys(rng, 2, m, False)))
    return out


def _distinct(rng, n, mask=POS):
    return keys(rng, n, mask, False)


def tie_shapes(rng):
    """equal keys where the unstable order depends on them: one pair at either end; groups of 2 to 300; all keys equal; a bucket of
    exactly 64 (insertion sort) and one of 65 (next level) below the top level; buckets whose elements all share the level's digit;
    ranges of 1024 or more that reach a second level (the warp-wide walk); ranges of more than 64 that reach byte 0"""
    out = []
    for n in (65, 100, 3000):
        x = _distinct(rng, n)
        s = np.sort(x)
        a, b = x.copy(), x.copy()
        a[a == s[1]] = s[0]  # the smallest key twice
        b[b == s[-2]] = s[-1]  # the largest key twice
        out += [("pair_first_n%d" % n, a), ("pair_last_n%d" % n, b)]
    for g in (2, 3, 17, 64, 65, 150, 300):
        n_grp = max(2, 3000 // g)
        vals = _distinct(rng, n_grp)
        out.append(("groups_of_%d" % g, rng.permutation(np.repeat(vals, g))))
    sz = rng.integers(2, 301, size=40)
    out.append(("groups_2_to_300", rng.permutation(np.repeat(_distinct(rng, len(sz)), sz))))
    for n in (65, 1000, 5000):
        out.append(("all_equal_n%d" % n, np.full(n, U64(0x8000000300001234), dtype=U64)))
    # top varying byte (bits 8-15): digit 1 holds exactly 64 keys, digit 2 exactly 65, digit 3 exactly 63, the others 10; the low byte
    # is drawn from a few values, so every bucket has equal keys
    for lo_vals in (4, 40):
        cnt = {1: 64, 2: 65, 3: 63}
        hi = np.concatenate([np.full(cnt.get(d, 10), d, dtype=U64) for d in range(0, 12)])
        lo = rng.integers(0, lo_vals, size=len(hi)).astype(U64)
        out.append(("bucket_64_65_lo%d" % lo_vals, rng.permutation(hi << U64(8) | lo) | U64(7 << 32)))
    # the same one level lower: the top byte (bits 16-23) splits the read in three ranges; below it (bits 8-15) buckets of exactly 64 and
    # 65 keys, and a range whose keys all share that digit
    grp = {(0, 0): 64, (0, 1): 65, (0, 2): 30, (1, 0): 100, (1, 1): 64, (2, 3): 65}
    x = np.concatenate([np.full(c, m << 16 | h << 8, dtype=U64) for (m, h), c in grp.items()])
    out.append(("bucket_64_65_level3", rng.permutation(x | rng.integers(0, 6, size=len(x)).astype(U64))))
    # buckets whose keys share the digit of their level: digit 0 of the top byte varies below in the middle byte, digit 1 holds keys
    # that all share their middle byte and vary in the low byte only (the reference's pass counts them and moves nothing)
    a = (U64(0) << U64(16)) | (rng.integers(0, 200, size=900).astype(U64) << U64(8)) | rng.integers(0, 256, size=900).astype(U64)
    b = (U64(1) << U64(16)) | (U64(0x5a) << U64(8)) | rng.integers(0, 50, size=700).astype(U64)
    c = (U64(2) << U64(16)) | (U64(0x11) << U64(8)) | rng.integers(0, 20, size=1500).astype(U64)  # >= 1024: the warp-wide walk skips it too
    out.append(("shared_digit_buckets", rng.permutation(np.concatenate([a, b, c]))))
    # ranges of >= 1024 keys at a second and a third level
    hi = rng.integers(0, 3, size=4500).astype(U64)
    out.append(("wide_ranges_level2", (hi << U64(8)) | rng.integers(0, 256, size=4500).astype(U64)))
    x = (rng.integers(0, 2, size=9000).astype(U64) << U64(40)) | (rng.integers(0, 2, size=9000).astype(U64) << U64(24)) | rng.integers(0, 256, size=9000).astype(U64)
    out.append(("wide_ranges_level3", x | U64(1 << 63)))
    # ranges of more than 64 keys that reach byte 0 (no level below it)
    x = (rng.integers(0, 4, size=2000).astype(U64) << U64(8)) | rng.integers(0, 8, size=2000).astype(U64)
    out.append(("ranges_reach_byte0", x))
    x = (rng.integers(0, 2, size=14000).astype(U64) << U64(32)) | rng.integers(0, 5, size=14000).astype(U64)
    out.append(("ranges_reach_byte0_large", x))
    return out


def combined(rng):
    """keys wider than 33 bits with equal keys: from the network sort on to the exact emulation, in every class and over 15360"""
    out = []
    for n in (65, 500, 1500, 3000, 6000, 12000, 15360, 15361, 16384):
        out.append(("wide_ties_n%d" % n, keys(rng, n, real_mask(6) | bits((48, 55)), True)))
        out.append(("wide_distinct_n%d" % n, keys(rng, n, real_mask(6) | bits((48, 55)), False)))
    # nb = 33 where the two strand blocks meet on equal position bits: neighbours differ only in the squeezed key's 33rd bit
    for n in (100, 3000):
        lo = keys(rng, n // 2, bits((0, 30)), False, base=0)
        hi = np.concatenate([lo.max(keepdims=True), keys(rng, n - n // 2 - 1, bits((0, 30)), False, base=0) | U64(1 << 31)])
        out.append(("strand_flag_boundary_n%d" % n, rng.permutation(np.concatenate([lo, hi | U64(1 << 63)]))))
    return out


def grid_batch(rng, n_cls0=3000, n_cls4=300, n_net=300, n_exact=400):
    """more reads per class than the class's grid (n_sm x occupancy), so the grid-stride loops take several turns; in one batch"""
    out = []
    for i in range(n_cls0):
        n = int(rng.integers(2, 1025))
        out.append(("cls0_%d" % i, keys(rng, n, real_mask(), i % 2 == 1)))
    for i in range(n_cls4):
        n = int(rng.integers(8193, 16385))
        out.append(("cls4_%d" % i, keys(rng, n, real_mask(), i % 4 == 1)))
    for i in range(n_net):
        n = int(rng.integers(2, 4097))
        out.append(("net_%d" % i, keys(rng, n, real_mask(6) | bits((48, 50)), i % 2 == 1)))
    for i in range(n_exact):
        n = int(rng.integers(65, 3000))
        out.append(("exact_%d" % i, keys(rng, n, bits((0, 11)), True)))
    return out


FAMILIES = dict(sizes=sizes, widths=widths, placement=placement, tie_shapes=tie_shapes, combined=combined)


def everything(seed=7):
    out = []
    for name, f in FAMILIES.items():
        out += [(name + "/" + t, x) for t, x in f(np.random.default_rng(seed + len(name)))]
    return out
