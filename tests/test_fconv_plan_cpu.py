"""Plans of the fp32 first-layer convolution (mnb_conv_fp32_tc.cu), checked on the host through mnb_fconv2d_plan (no
launch, no GPU): the edges of its cover in both directions, the weight-gradient scratch size, the plans each case of
test_gpu_fconv_fp64.py was written for, and that those cases together reach every plan path of the two kernels."""
import ctypes as C

import pytest

from tests import fconv_plan_util as FU


def _plan(B, Cc, H, W, K, R, wgrad):
    return FU.plan(FU.shape(B, Cc, H, W, K, R), wgrad)


# (B, C, H, W, K, R), forward accepted, weight gradient accepted
EDGES = [
    ((8, 5, 32, 32, 128, 5), True, True),        # C*R*S = 125
    ((8, 129, 32, 32, 16, 1), False, False),     # C*R*S = 129
    ((8, 1, 32, 32, 256, 3), True, True),        # K = 256
    ((8, 1, 32, 32, 257, 3), False, False),
    ((8, 3, 32, 8, 16, 3), True, True),          # W = 8
    ((8, 3, 32, 128, 16, 3), True, True),        # W = 128
    ((8, 3, 64, 4, 16, 3), False, False),        # W = 4
    ((8, 3, 16, 256, 16, 3), False, False),      # W = 256
    ((8, 3, 48, 48, 16, 3), False, False),       # 48 does not divide 128
    ((8, 3, 8, 16, 16, 3), True, True),          # H * W = 128
    ((8, 3, 4, 16, 16, 3), False, False),        # H * W = 64: not a whole tile
    ((8, 2, 32, 32, 176, 7), True, False),       # C*R*S = 98: shared memory
    ((8, 2, 32, 32, 177, 7), False, False),
    ((8, 2, 32, 32, 128, 7), True, True),
    ((8, 2, 32, 32, 129, 7), True, False),
    ((8, 5, 32, 32, 129, 5), False, False),      # C*R*S = 125: shared memory
    ((8191, 3, 32, 32, 256, 5), True, True),     # B * K * H * W = 2^31 - 2^18
    ((8192, 3, 32, 32, 256, 5), False, False),   # = 2^31
]


@pytest.mark.parametrize("shape,fwd,wgrad", EDGES, ids=[str(e[0]) for e in EDGES])
def test_cover_edges(shape, fwd, wgrad):
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = FU.shape(*shape)
    for kind, want in (("fwd", fwd), ("wgrad", wgrad)):
        out = (C.c_int32 * len(FU.FIELDS))()
        rc = lib.mnb_fconv2d_plan(C.byref(sh), int(kind == "wgrad"), out, len(FU.FIELDS))
        if want:
            assert rc == 0, (kind, lib.mnb_last_error())
            p = dict(zip(FU.FIELDS, out))
            assert p["smem_bytes"] <= 227 * 1024 - 2560, (kind, p)
        else:
            assert rc == L.E_UNSUPPORTED, kind
            assert b"fp32 tc conv" in lib.mnb_last_error(), kind
    assert (lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh)) >= 0) == wgrad


def test_plan_fields_follow_the_shape():
    """fields against the formulas of tcfp32::plan: paddings, tile rows, patch size, grid"""
    for B, Cc, H, W, K, R in [(256, 3, 32, 32, 256, 5), (1, 3, 32, 32, 192, 5), (7, 2, 16, 64, 40, 3), (3, 1, 128, 128, 8, 1)]:
        for wgrad in (False, True):
            p = _plan(B, Cc, H, W, K, R, wgrad)
            TH = 128 // W
            assert p["KP"] == -(-Cc * R * R // 16) * 16
            assert p["NP"] == -(-K // (128 if wgrad else 16)) * (128 if wgrad else 16)
            assert p["TH"] == TH and p["n_tiles"] == B * H // TH
            assert p["grid"] == min(p["n_tiles"], FU.NUM_SMS)
            assert p["patch_floats"] == Cc * (TH + R - 1) * (W + R - 1)
            assert p["nbuf_a"] in (1, 2) and (not wgrad or p["nbuf_a"] == 2)
    # a short output buffer takes only the leading fields
    from micronet_b200 import _lib as L
    out = (C.c_int32 * 3)(-7, -7, -7)
    assert L.load().mnb_fconv2d_plan(C.byref(FU.shape(2, 3, 32, 32, 40, 5)), 0, out, 2) == 0
    assert list(out) == [48, 80, -7]
    assert L.load().mnb_fconv2d_plan(C.byref(FU.shape(2, 3, 32, 32, 40, 5)), 0, None, 0) == 0


def test_wgrad_scratch_is_one_partial_per_cta():
    """one fp32 partial dw per CTA, also when there are more tiles than SMs (grid = min(n_tiles, 132))"""
    from micronet_b200 import _lib as L
    lib = L.load()
    for shape in [(256, 3, 32, 32, 256, 5), (256, 3, 32, 32, 192, 5), (1, 3, 32, 32, 256, 5), (40, 8, 32, 32, 64, 3)]:
        B, Cc, H, W, K, R = shape
        p = _plan(*shape, True)
        need = lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(FU.shape(*shape)))
        assert need == p["grid"] * K * Cc * R * R * 4
    assert _plan(256, 3, 32, 32, 256, 5, True)["grid"] == 132 < 2048


def test_gpu_cases_run_the_plans_they_were_written_for():
    for c in FU.CASES.values():
        sh = FU.shape(*c.shape)
        for kind, want in (("fwd", c.fwd), ("wgrad", c.wgrad)):
            got = FU.plan(sh, kind == "wgrad")
            if want is None:
                assert got is None, (c.id, kind, got)
            else:
                assert got is not None, (c.id, kind)
                assert {k: got[k] for k in want} == want, (c.id, kind, got)


def test_gpu_cases_cover_every_plan_path():
    fwd = {i: FU.plan(FU.shape(*FU.CASES[i].shape), False) for i in FU.CASES}
    wg = {i: FU.plan(FU.shape(*FU.CASES[i].shape), True) for i in FU.CASES}
    onehot = {i: fwd[i] for i in FU.ONEHOT_FWD}
    sparse = {i: wg[i] for i in FU.SPARSE_WGRAD}
    rand_f = {i: fwd[i] for i in FU.RANDOM if fwd[i]}
    rand_w = {i: wg[i] for i in FU.RANDOM if wg[i]}
    bench = {(256, 3, 32, 32, 256, 5), (256, 3, 32, 32, 192, 5)}
    for group in (onehot, rand_f):
        assert bench <= {FU.CASES[i].shape for i in group}
        for nbuf in (1, 2):
            assert any(p["nbuf_a"] == nbuf and p["n_tiles"] > p["grid"] for p in group.values()), nbuf
        assert any(p["NP"] % 32 == 16 and p["n_tiles"] > p["grid"] for p in group.values())
        assert any(p["patch_floats"] > FU.PATCH_PREFETCH for p in group.values())
        assert {1, 16} <= {p["TH"] for p in group.values()}
    for group in (sparse, rand_w):
        assert bench <= {FU.CASES[i].shape for i in group}
        assert {128, 256} <= {p["NP"] for p in group.values()}
        assert any(p["patch_floats"] > FU.PATCH_PREFETCH for p in group.values())
        assert any(p["n_tiles"] > p["grid"] and p["n_tiles"] % p["grid"] for p in group.values())
    assert {1, 16} <= {p["TH"] for p in rand_w.values()}
    assert any(p["grid"] < FU.NUM_SMS for p in rand_f.values())
    # forward on the engine, weight gradient refused (the module falls back to ATen for it)
    assert any(fwd[i] and not wg[i] for i in FU.RANDOM)
