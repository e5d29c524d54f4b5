"""GPU parity, kernel level: the seeding stage K2a/K2b (query-side filter, index lookup on the device hash table, streak selection,
skip_seed's strand rule, anchor expansion, anchor sort incl. the reference's unstable tie order) through mmb_seed_batch_host against the
oracle restatement (oracle/mm2o_seed.c). See tests/seed_check.py."""
import ctypes as C
import numpy as np
import pytest
import seed_check as SC
import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import minimap2_b200 as mb
    from minimap2_b200._lib import lib
    L = lib()
    SC.setup(L)
    c = mb.Context(0)
    yield L, C.c_void_p(c.h)
    c.close()


@pytest.mark.parametrize("cfg", [dict(), dict(mid_occ=6, occ_dist=100), dict(mid_occ=8, occ_dist=0), dict(q_occ_frac=0.0), dict(flag=0x100000), dict(flag=0x200000),
                                 dict(w=5, mid_occ=20), dict(w=19, k=19, mid_occ=50)])
def test_seed_stage_matches_oracle(dev, cfg):
    L, ctx = dev
    contigs, reads = SC.repeat_rich_case(5, 400_000, 120, 4000, rep=0.35, n_contigs=3)
    st = SC.check_case(L, ctx, contigs, reads, **cfg)
    assert st["anchors"] > 10_000 and st["big"] > 50


def test_seed_stage_sort_ties_and_size_classes(dev):
    """repeat-rich genome and long reads: anchor counts from a handful to > 16384 per read (every shared-memory class of the radix sort and
    the global-memory fallback), many reads with equal sort keys (exact emulation of the unstable radix sort)"""
    L, ctx = dev
    contigs, reads = SC.repeat_rich_case(9, 200_000, 40, 12000, rep=0.8, n_contigs=1)
    reads += [r[:n] for r, n in zip(reads[:12], (200, 500, 900, 1500, 2500, 3500, 5000, 7000, 9000, 10000, 11000, 11500))]
    st = SC.check_case(L, ctx, contigs, reads, mid_occ=60, max_max_occ=600, occ_dist=100)
    assert st["ties"] >= 5


def test_seed_stage_wide_keys(dev):
    """sort keys that differ in more than 33 bit positions, as on a human reference: the radix kernels hand these reads to
    sort_block_kernel, and the ones with equal keys on to the exact emulation. 64 contigs give 6 contig bits; the last one holds a
    reverse-complemented copy of chr0 at 2^27 - 2^14 after N padding, so positions differ in bits 0-26, plus the strand bit."""
    L, ctx = dev
    contigs = synth.random_genome(640_000, 13, n_contigs=63, repeat_frac=0.3)
    seg = contigs[0]
    contigs.append(np.concatenate([np.full((1 << 27) - (1 << 14), ord("N"), dtype=np.uint8), synth.revcomp(seg)]))
    reads = synth.make_reads([seg], 40, 4000, 0.08, 63) + [bytes(seg[1000:9000]) * 2]  # the tandem read has equal keys
    st = SC.check_case(L, ctx, contigs, reads, mid_occ=20)
    assert st["wide"] >= 40 and st["ties"] >= 1


@pytest.mark.parametrize("seed", [3, 4])
def test_seed_stage_capacity_edges(dev, seed):
    """2048 / 2049 minimizers in both query-side filter kernels and in select_kernel, q_occ_max / q_occ_max + 1 minimizers, and streaks
    at the 128-entry heap's cap (see seed_check.check_edges)"""
    L, ctx = dev
    SC.check_edges(L, ctx, seed=seed)
