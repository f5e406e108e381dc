"""The two-warpgroup forward and weight gradient of the fp32 first-layer convolution (mnb_fconv2d_fwd_wg /
mnb_fconv2d_wgrad_wg, DESIGN 4.8) byte for byte against mnb_fconv2d_fwd_tc / mnb_fconv2d_wgrad_tc.  The forward: at every case of tests/fconv_plan_util.py it covers, at the bench stems' batch and at the edges of
its cover, on random operands, operands spanning a wide dynamic range (the lo pieces matter), one-hot filters and signed
zeros.  Each launch writes a NaN-prefilled output, twice: equal results, error flag clear.  Also the module route
(EngineFloatConv2d forward and backward) against the old entry points, and refusals outside the cover with nothing
launched.  Byte equality at N = 192 / 256 is also the check that an MMA's result for one element does not depend on the
N width it is issued with.  The weight gradient: every covered case, random, wide-range, sparse and signed-zero
operands, NaN-prefilled dw and scratch, two launches, refusals."""
import ctypes as C
import zlib

import pytest
import torch

from tests import fconv_plan_util as FU

pytestmark = pytest.mark.gpu
DEV = "cuda"

EXTRA = {
    "ningc_stem_b256": (256, 3, 32, 32, 256, 5),
    "nin_stem_b256": (256, 3, 32, 32, 192, 5),
    "k129": (4, 3, 32, 32, 129, 5),         # N = 192, 63 padded columns
    "k193_kp48": (4, 5, 32, 32, 193, 3),    # N = 256, KP = 48
    "w64": (4, 3, 32, 64, 256, 5),          # one image row per tile
    "w8": (4, 3, 32, 8, 200, 3),            # eight rows per tile
}
# the cases of fconv_plan_util the two-warpgroup plan covers (test_every_case_is_listed keeps the list whole)
FU_COVERED = ["ningc_stem", "nin_stem", "b1"]


def _lib():
    from micronet_b200 import _lib as L
    return L, L.load()


def _wg_covers(shape):
    L, lib = _lib()
    return lib.mnb_fconv2d_wg_plan(C.byref(FU.shape(*shape)), None, 0) == 0


def _cases():
    out = {cid: c.shape for cid, c in FU.CASES.items()}
    out.update(EXTRA)
    return out


def _operands(shape, kind, seed):
    B, Cc, H, W, K, R = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cc, H, W, generator=g)
    w = torch.randn(K, Cc, R, R, generator=g) * 0.1
    bias = torch.randn(K, generator=g)
    if kind == "wide":
        x = x * torch.exp2(torch.randint(-40, 40, x.shape, generator=g).float())
        w = w * torch.exp2(torch.randint(-30, 30, w.shape, generator=g).float())
    elif kind == "onehot":
        w = torch.zeros_like(w)
        idx = torch.randint(0, Cc * R * R, (K,), generator=g)
        w.view(K, -1)[torch.arange(K), idx] = torch.randn(K, generator=g)
    elif kind == "zeros":
        x = torch.where(torch.rand(x.shape, generator=g) < 0.5, x, torch.zeros_like(x))
        x = torch.where(torch.rand(x.shape, generator=g) < 0.5, x, -torch.zeros_like(x))
        w = torch.where(torch.rand(w.shape, generator=g) < 0.5, w, -torch.zeros_like(w))
        bias = None
    return x.to(DEV), w.to(DEV), None if bias is None else bias.to(DEV)


def _run(entry, shape, x, w, bias):
    """two launches onto NaN-prefilled outputs: bitwise equal, flag clear"""
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    sh = FU.shape(*shape)
    err = L.tc_err_flag(torch.device(DEV))
    outs = []
    for _ in range(2):
        y = torch.full((B, K, H, W), float("nan"), device=DEV)
        L.check(getattr(lib, entry)(C.byref(sh), x.data_ptr(), w.data_ptr(), L.ptr(bias), y.data_ptr(), err.data_ptr(),
                                    L.stream()), entry)
        outs.append(y)
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), entry
    return outs[0]


def test_every_case_is_listed():
    assert [cid for cid, c in FU.CASES.items() if _wg_covers(c.shape)] == FU_COVERED
    for cid in EXTRA:
        assert _wg_covers(EXTRA[cid]), cid


@pytest.mark.parametrize("kind", ["random", "wide", "onehot", "zeros"])
@pytest.mark.parametrize("cid", FU_COVERED + list(EXTRA))
def test_forward_bytes_equal_fwd_tc(cid, kind):
    shape = _cases()[cid]
    x, w, bias = _operands(shape, kind, zlib.crc32(repr((cid, kind)).encode()))
    y_old = _run("mnb_fconv2d_fwd_tc", shape, x, w, bias)
    y_new = _run("mnb_fconv2d_fwd_wg", shape, x, w, bias)
    assert torch.equal(y_old.view(torch.int32), y_new.view(torch.int32)), (cid, kind)


@pytest.mark.parametrize("shape", [(8, 3, 32, 32, 64, 3), (8, 3, 32, 32, 128, 5), (8, 3, 64, 128, 256, 5),
                                   (8, 2, 32, 32, 176, 7), (8, 3, 4, 16, 256, 3)])
def test_refused_outside_cover(shape):
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    x = torch.zeros(B, Cc, H, W, device=DEV)
    w = torch.zeros(K, Cc, R, R, device=DEV)
    y = torch.zeros(B, K, H, W, device=DEV)
    n0 = L.launch_count()
    rc = lib.mnb_fconv2d_fwd_wg(C.byref(FU.shape(*shape)), x.data_ptr(), w.data_ptr(), None, y.data_ptr(),
                                L.tc_err_flag(x.device).data_ptr(), L.stream())
    assert rc == L.E_UNSUPPORTED and L.launch_count() == n0


@pytest.mark.parametrize("cid", ["ningc_stem_b256", "nin_stem_b256"])
def test_module_route_bytes_equal_old_entry_points(cid):
    from micronet_b200.fused import EngineFloatConv2d
    L, lib = _lib()
    B, Cc, H, W, K, R = EXTRA[cid]
    torch.manual_seed(zlib.crc32(cid.encode()))
    m = EngineFloatConv2d(Cc, K, R, padding=R // 2).to(DEV)
    x = torch.randn(B, Cc, H, W, device=DEV)
    dy = torch.randn(B, K, H, W, device=DEV)
    n0 = L.launch_count()
    y = m(x)
    y.backward(dy)
    torch.cuda.synchronize()
    assert L.launch_count() > n0
    sh = FU.shape(B, Cc, H, W, K, R)
    y_old = _run("mnb_fconv2d_fwd_tc", (B, Cc, H, W, K, R), x, m.weight.detach(), m.bias.detach())
    assert torch.equal(y.detach().view(torch.int32), y_old.view(torch.int32))
    dw = torch.full_like(m.weight, float("nan"))
    scratch = torch.empty(int(lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh))), dtype=torch.uint8, device=DEV)
    L.check(lib.mnb_fconv2d_wgrad_tc(C.byref(sh), dy.data_ptr(), x.data_ptr(), dw.data_ptr(), scratch.data_ptr(),
                                     L.tc_err_flag(x.device).data_ptr(), L.stream()), "wgrad")
    torch.cuda.synchronize()
    assert torch.equal(m.weight.grad.view(torch.int32), dw.view(torch.int32))


# the weight gradient: mnb_fconv2d_wgrad_wg against mnb_fconv2d_wgrad_tc
WGRAD_COVERED = ["ningc_stem", "nin_stem", "b1", "ningc_stem_b256", "nin_stem_b256", "k129", "w64"]


def _wgrad(entry, shape, dy, x):
    """two launches onto NaN-prefilled dw and scratch: bitwise equal, flag clear"""
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    sh = FU.shape(*shape)
    err = L.tc_err_flag(torch.device(DEV))
    nbytes = int(getattr(lib, entry + "_scratch_bytes")(C.byref(sh)))
    assert nbytes > 0
    outs = []
    for _ in range(2):
        dw = torch.full((K, Cc, R, R), float("nan"), device=DEV)
        scratch = torch.full((nbytes // 4,), float("nan"), device=DEV)
        L.check(getattr(lib, entry)(C.byref(sh), dy.data_ptr(), x.data_ptr(), dw.data_ptr(), scratch.data_ptr(),
                                    err.data_ptr(), L.stream()), entry)
        outs.append(dw)
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), entry
    return outs[0]


def test_wgrad_cover_is_listed():
    L, lib = _lib()
    covered = [cid for cid, s in _cases().items() if lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(FU.shape(*s))) >= 0]
    assert sorted(covered) == sorted(WGRAD_COVERED)
    for cid in covered:   # never more than wgrad_tc's cover, the same scratch (one partial per CTA)
        sh = FU.shape(*_cases()[cid])
        assert lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(sh)) == lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh))


@pytest.mark.parametrize("kind", ["random", "wide", "sparse", "zeros"])
@pytest.mark.parametrize("cid", WGRAD_COVERED)
def test_wgrad_bytes_equal_wgrad_tc(cid, kind):
    B, Cc, H, W, K, R = shape = _cases()[cid]
    g = torch.Generator().manual_seed(zlib.crc32(repr((cid, kind, "wgrad")).encode()))
    x = torch.randn(B, Cc, H, W, generator=g)
    dy = torch.randn(B, K, H, W, generator=g)
    if kind == "wide":
        x = x * torch.exp2(torch.randint(-30, 30, x.shape, generator=g).float())
        dy = dy * torch.exp2(torch.randint(-30, 30, dy.shape, generator=g).float())
    elif kind == "sparse":
        dy = dy * (torch.rand(dy.shape, generator=g) < 1e-3)
    elif kind == "zeros":
        x = torch.where(torch.rand(x.shape, generator=g) < 0.5, x, -torch.zeros_like(x))
        dy = torch.where(torch.rand(dy.shape, generator=g) < 0.5, dy, -torch.zeros_like(dy))
    x, dy = x.to(DEV), dy.to(DEV)
    dw_old = _wgrad("mnb_fconv2d_wgrad_tc", shape, dy, x)
    dw_new = _wgrad("mnb_fconv2d_wgrad_wg", shape, dy, x)
    assert torch.equal(dw_old.view(torch.int32), dw_new.view(torch.int32)), (cid, kind)


@pytest.mark.parametrize("shape", [(8, 3, 32, 32, 128, 5), (8, 3, 32, 32, 256, 3), (8, 2, 32, 32, 176, 7)])
def test_wgrad_refused_outside_cover(shape):
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    x = torch.zeros(B, Cc, H, W, device=DEV)
    dy = torch.zeros(B, K, H, W, device=DEV)
    dw = torch.zeros(K, Cc, R, R, device=DEV)
    scratch = torch.zeros(1 << 20, device=DEV)
    n0 = L.launch_count()
    rc = lib.mnb_fconv2d_wgrad_wg(C.byref(FU.shape(*shape)), dy.data_ptr(), x.data_ptr(), dw.data_ptr(),
                                  scratch.data_ptr(), L.tc_err_flag(x.device).data_ptr(), L.stream())
    assert rc == L.E_UNSUPPORTED and L.launch_count() == n0
    assert lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(FU.shape(*shape))) == -1
