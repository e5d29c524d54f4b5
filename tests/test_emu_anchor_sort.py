"""CPU: the anchor sort alone (mmb_anchor_sort_host), the unmodified CUDA sources under the SIMT emulator, against the reference's
radix_sort_128x and the expected route of every read (tests/sort_cases.py), on a reduced set: every class boundary with one oversize
read, key widths at 300 anchors, and the placement, tie and combined shapes. The whole module takes about a minute."""
import collections
import ctypes as C
import os
import sys
import numpy as np
import pytest
import oracle_lib as O
import sort_cases as S

sys.path.insert(0, os.path.join(O.ROOT, "tests", "cuda_emu"))

SEEN = collections.Counter()
REDUCED = dict(sizes=lambda rng: S.sizes(rng, oversize=(40_000,)), widths=lambda rng: S.widths(rng, ns=(300,)),
               placement=S.placement, tie_shapes=S.tie_shapes, combined=S.combined)


@pytest.fixture(scope="module")
def emu():
    import build_emu
    from minimap2_b200._lib import declare_anchor_sort
    L = declare_anchor_sort(C.CDLL(build_emu.build("mmb_emu_all", build_emu.ALL, extra=())))
    L.mmb_ctx_create.restype = C.c_void_p
    return L, C.c_void_p(L.mmb_ctx_create(0))


@pytest.mark.parametrize("family", list(REDUCED))
def test_emulated_anchor_sort(emu, family):
    L, ctx = emu
    SEEN.update(S.check_batch(ctx, REDUCED[family](np.random.default_rng(3 + len(family))), L=L))


def test_zz_every_route_exercised(request):
    names = {it.originalname for it in request.session.items if it.module is request.module}
    if "test_emulated_anchor_sort" not in names:
        pytest.skip("only part of this module was selected")
    missing = [r for r in S.ALL_ROUTES if SEEN[r] == 0]
    assert not missing, (missing, dict(SEEN))
