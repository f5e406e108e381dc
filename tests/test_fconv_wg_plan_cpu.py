"""Plans of the two-warpgroup forward and weight gradient of the fp32 first-layer convolution (mnb_fconv2d_fwd_wg /
mnb_fconv2d_wgrad_wg), checked on the host through mnb_fconv2d_wg_plan and mnb_fconv2d_wgrad_wg_scratch_bytes (no
launch, no GPU): the edges of both covers in both directions, that neither covers a shape the old kernels refuse, the
shared memory of every forward plan, and the forward plans of the bench stems."""
import ctypes as C

import pytest

from tests import fconv_plan_util as FU

SMEM_BUDGET = 227 * 1024 - 2560


def wg_plan(sh):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(FU.FIELDS))()
    if L.load().mnb_fconv2d_wg_plan(C.byref(sh), out, len(FU.FIELDS)) != 0:
        return None
    return dict(zip(FU.FIELDS, list(out)))


# (B, C, H, W, K, R), accepted
EDGES = [
    ((8, 3, 32, 32, 256, 5), True),     # the NIN-GC stem
    ((8, 3, 32, 32, 192, 5), True),     # the NIN stem
    ((8, 3, 32, 32, 129, 5), True),     # Cout = 129: N = 192
    ((8, 3, 32, 32, 128, 5), False),    # Cout = 128
    ((8, 3, 32, 32, 64, 3), False),     # the ResNet stem
    ((8, 3, 32, 32, 193, 5), True),     # N = 256
    ((8, 1, 32, 32, 257, 3), False),    # Cout = 257
    ((8, 3, 32, 64, 256, 5), True),     # W = 64: one row per tile
    ((8, 3, 64, 128, 256, 5), False),   # W = 128: fwd_tc only
    ((8, 3, 32, 8, 256, 3), True),      # W = 8
    ((8, 3, 64, 4, 256, 3), False),     # W = 4: refused by fwd_tc
    ((8, 3, 4, 16, 256, 3), False),     # H * W = 64: refused by fwd_tc
    ((8, 2, 32, 32, 176, 7), False),    # C*R*S = 98: 3 im2col buffers do not fit
    ((8, 5, 32, 32, 256, 3), True),     # C*R*S = 45, KP = 48
    ((8, 3, 32, 32, 256, 4), False),    # even filter
    ((8191, 3, 32, 32, 256, 5), True),  # B * K * H * W = 2^31 - 2^18
    ((8192, 3, 32, 32, 256, 5), False),
]


@pytest.mark.parametrize("shape,ok", EDGES, ids=[str(e[0]) for e in EDGES])
def test_cover_edges(shape, ok):
    p = wg_plan(FU.shape(*shape))
    assert (p is not None) == ok, (shape, p)
    if p is not None:
        assert FU.plan(FU.shape(*shape), False) is not None   # never more than fwd_tc's cover
        assert p["smem_bytes"] <= SMEM_BUDGET and 3 <= p["nbuf_a"] <= 4, p
        assert p["NP"] in (192, 256) and p["NP"] >= shape[4] and p["TH"] * shape[3] == 64, p


@pytest.mark.parametrize("cid", list(FU.CASES))
def test_cases_within_fwd_tc_cover(cid):
    sh = FU.shape(*FU.CASES[cid].shape)
    p = wg_plan(sh)
    if p is not None:
        assert FU.plan(sh, False) is not None and p["smem_bytes"] <= SMEM_BUDGET, (cid, p)


@pytest.mark.parametrize("shape,want", [
    ((256, 3, 32, 32, 256, 5), dict(NP=256, KP=80, TH=2, n_tiles=4096, grid=132, nbuf_a=3, patch_floats=648)),
    ((256, 3, 32, 32, 192, 5), dict(NP=192, KP=80, TH=2, n_tiles=4096, grid=132, nbuf_a=4, patch_floats=648)),
], ids=["ningc_stem", "nin_stem"])
def test_bench_stem_plans(shape, want):
    p = wg_plan(FU.shape(*shape))
    assert p is not None and {k: p[k] for k in want} == want, p
    # the converter warpgroup prefetches FWG_PF = 6 patch elements per thread: the whole patch
    assert p["patch_floats"] <= 6 * 128


# weight gradient: (B, C, H, W, K, R), accepted by mnb_fconv2d_wgrad_wg
WGRAD_EDGES = [
    ((8, 3, 32, 32, 256, 5), True),     # the NIN-GC stem
    ((8, 3, 32, 32, 192, 5), True),     # the NIN stem
    ((8, 3, 32, 32, 129, 5), True),     # four 64-channel blocks
    ((8, 3, 32, 32, 128, 5), False),    # two blocks: wgrad_tc
    ((8, 3, 32, 32, 256, 3), False),    # C*R*S = 27, KP = 32
    ((8, 2, 32, 32, 256, 6), False),    # even filter
    ((8, 4, 32, 32, 256, 4), False),
    ((8, 3, 32, 128, 256, 5), True),    # W = 128: 128-position tiles as in wgrad_tc
    ((8, 3, 4, 16, 256, 5), False),     # H * W = 64: refused by wgrad_tc
]


@pytest.mark.parametrize("shape,ok", WGRAD_EDGES, ids=[str(e[0]) for e in WGRAD_EDGES])
def test_wgrad_cover_edges(shape, ok):
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = FU.shape(*shape)
    n = int(lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(sh)))
    assert (n >= 0) == ok, (shape, n)
    if ok:   # the same plan as wgrad_tc: one partial per CTA of the same grid
        assert n == int(lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh)))
        assert FU.plan(sh, True) is not None
