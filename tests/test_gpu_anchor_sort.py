"""GPU: the anchor sort alone (mmb_anchor_sort_host: the seeding stage's sort kernels with the same launches) against the reference's
radix_sort_128x, anchor for anchor including the order of equal keys, and the path every read takes through the kernels, at every
class boundary, key width, bit placement and tie shape of tests/sort_cases.py, and with more reads per class than the class's grid."""
import collections
import numpy as np
import pytest
import sort_cases as S

pytestmark = pytest.mark.gpu

SEEN = collections.Counter()  # reads checked per route


@pytest.fixture(scope="module")
def ctx():
    import minimap2_b200 as mb
    c = mb.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("family", list(S.FAMILIES))
def test_anchor_sort_family(ctx, family):
    SEEN.update(S.check_batch(ctx, S.FAMILIES[family](np.random.default_rng(11 + len(family)))))


def test_anchor_sort_every_shape_in_one_batch(ctx):
    SEEN.update(S.check_batch(ctx, S.everything(seed=23)))


def test_anchor_sort_more_reads_than_grid(ctx):
    """class 0 (128-thread CTAs: at most 16 per SM), class 4 (1024 threads: at most 2 per SM), the network sort and the exact walker
    (at most 2 and 1 CTAs per SM) each get more reads than their grid holds, so every grid-stride loop turns more than once"""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    seen = S.check_batch(ctx, S.grid_batch(np.random.default_rng(5)))
    SEEN.update(seen)
    by = lambda f: sum(v for r, v in seen.items() if f(r))
    assert by(lambda r: r >= 0 and r & 7 == 0 and not r & S.NETWORK) > 16 * n_sm, seen
    assert by(lambda r: r >= 0 and r & 7 == 4 and not r & S.NETWORK) > 2 * n_sm, seen
    assert by(lambda r: r >= 0 and r & S.NETWORK) > 2 * n_sm, seen
    assert by(lambda r: r >= 0 and r & S.EXACT) > n_sm, seen


def test_zz_every_route_exercised(request):
    """every route the kernels can give a read was checked by the tests above"""
    names = {it.originalname for it in request.session.items if it.module is request.module}
    wanted = {n for n in dir(request.module) if n.startswith("test_") and n != "test_zz_every_route_exercised"}
    if not wanted <= names:
        pytest.skip("only part of this module was selected")
    print("reads per route:", dict(sorted(SEEN.items())))
    missing = [r for r in S.ALL_ROUTES if SEEN[r] == 0]
    assert not missing, missing
