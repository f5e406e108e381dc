"""The fp32 first-layer convolution (mnb_fconv2d_fwd_tc / mnb_fconv2d_wgrad_tc, DESIGN 4.8) element by element, at the
bench stems' batch and at every plan path (tests/fconv_plan_util.py pins the plan of each case).

Every launch goes to the C entry points, onto NaN-prefilled outputs and scratch, twice: the two results must be bitwise
equal, the error flag 0.

* one-hot filters: y[b, n, p] = fp32(x[b, c_n, p + tap_n] * w_n + bias_n) bit for bit.  Three operand variants, each
  needing a different set of the six kept piece products (hi/mid/lo = the exact bf16 split of an fp32 value):
  A full-significand x, w_n = +-2^e (lo.hi, mid.hi, hi.hi); B x = +-2^k, full-significand w (hi.lo, hi.mid, hi.hi);
  C x = +-(1 + 2^-a) 2^k, w = +-(1 + 2^-b) 2^e, a, b in {9, 10, 11} (mid.mid).
* sparse dy (one or two +-2^e-style entries per output channel): dw[n, c, r, s] is one exact product, or fp32(a + b) of
  two, bit for bit, with the entries at image corners, in the first and last image and in the last tile of a CTA that runs
  the most tiles; the second entry in a tile of another CTA, or in another 32-position step of the same CTA.
* random operands against fp64, element-wise, with R = the same operation on |operands| (+ |bias|) in fp64:
  forward |y - y64| <= (KR + 3) u R, weight gradient |dw - dw64| <= c u R, u = 2^-24 (see _wgrad_c).
* the module routes: EngineFloatConv2d, QuantConv2dFn without an activation quantizer, ATen where the kernels refuse."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as TF

from tests import fconv_plan_util as FU

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _lib():
    from micronet_b200 import _lib as L
    return L, L.load()


def _expect_plan(case, wgrad):
    p = FU.plan(FU.shape(*case.shape), wgrad)
    want = case.wgrad if wgrad else case.fwd
    assert p is not None and {k: p[k] for k in want} == want, (case.id, wgrad, p)
    return p


def _nan(shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _fwd(shape, x, w, bias):
    """two launches on NaN-prefilled outputs: bitwise equal, flag clear"""
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    sh = FU.shape(*shape)
    outs = []
    for _ in range(2):
        y = _nan((B, K, H, W))
        L.check(lib.mnb_fconv2d_fwd_tc(C.byref(sh), x.data_ptr(), w.data_ptr(), L.ptr(bias), y.data_ptr(),
                                       L.tc_err_flag(x.device).data_ptr(), L.stream()), "fconv2d_fwd_tc")
        outs.append(y)
    L.tc_check()
    assert int(L.tc_err_flag(x.device).item()) == 0
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "forward not deterministic"
    return outs[0]


def _wgrad(shape, dy, x):
    L, lib = _lib()
    B, Cc, H, W, K, R = shape
    sh = FU.shape(*shape)
    need = int(lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh)))
    assert need > 0
    outs = []
    for _ in range(2):
        dw = _nan((K, Cc, R, R))
        scratch = _nan((need // 4,))
        L.check(lib.mnb_fconv2d_wgrad_tc(C.byref(sh), dy.data_ptr(), x.data_ptr(), dw.data_ptr(), scratch.data_ptr(),
                                         L.tc_err_flag(x.device).data_ptr(), L.stream()), "fconv2d_wgrad_tc")
        outs.append(dw)
    L.tc_check()
    assert int(L.tc_err_flag(x.device).item()) == 0
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "weight gradient not deterministic"
    return outs[0]


# ------------------------------------------------------------------------------------------------ operand variants
def _full(n, g, lo, hi):
    """+-(24-bit significand in [1, 2)) * 2^U(lo, hi)"""
    m = torch.randint(2 ** 23, 2 ** 24, (n,), generator=g).double() * 2.0 ** -23
    e = torch.randint(lo, hi + 1, (n,), generator=g)
    s = torch.randint(0, 2, (n,), generator=g) * 2 - 1
    return (s * torch.ldexp(m, e)).float()


def _pow2(n, g, lo, hi):
    e = torch.randint(lo, hi + 1, (n,), generator=g)
    s = torch.randint(0, 2, (n,), generator=g) * 2 - 1
    return (s * torch.ldexp(torch.ones(n, dtype=torch.float64), e)).float()


def _near1(n, g, lo, hi):
    """+-(1 + 2^-a) 2^k, a in {9, 10, 11}: hi piece 1, mid piece 2^-a"""
    a = torch.randint(9, 12, (n,), generator=g)
    return (_pow2(n, g, lo, hi).double() * (1 + torch.ldexp(torch.ones(n, dtype=torch.float64), -a))).float()


VARIANTS = {"A": (_full, _pow2), "B": (_pow2, _full), "C": (_near1, _near1)}   # (activation, weight / dy) generators


# ------------------------------------------------------------------------------------------------ a. one-hot forward
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("cid", FU.ONEHOT_FWD)
def test_forward_one_hot_is_exact(cid, variant, bias):
    case = FU.CASES[cid]
    _expect_plan(case, False)
    B, Cc, H, W, K, R = case.shape
    KR = Cc * R * R
    g = torch.Generator().manual_seed(_seed(cid, variant, bias))
    gx, gw = VARIANTS[variant]
    x = gx(B * Cc * H * W, g, -20, 20).view(B, Cc, H, W).to(DEV)
    cols = TF.unfold(x, R, padding=R // 2)                  # [B, KR, H*W], exact copies, 0 outside the image
    launches = -(-KR // K)
    for launch in range(launches):                            # every im2col column is some channel's tap
        kk = (torch.arange(K) + launch * K) % KR
        wn = gw(K, g, -10, 10)
        w = torch.zeros(K, KR)
        w[torch.arange(K), kk] = wn
        b = _full(K, g, -20, 20).to(DEV) if bias else None
        y = _fwd(case.shape, x, w.view(K, Cc, R, R).to(DEV), b)
        ref = cols[:, kk.to(DEV), :] * wn.to(DEV)[None, :, None]
        ref = ref + (b if bias else torch.zeros(K, device=DEV))[None, :, None]
        y = y.view(B, K, H * W)
        bad = y != ref
        assert not bad.any(), (f"{cid} {variant} launch {launch}: {int(bad.sum())} of {y.numel()} differ, first at "
                               f"{bad.nonzero()[0].tolist()}: {y[bad][0].item()!r} vs {ref[bad][0].item()!r}")


# ------------------------------------------------------------------------------------------------ b. sparse-dy weight gradient
def _positions(case, p, g):
    """one (b, h, w) per output channel: the four corners of the first and the last image, the first, a middle and the
    last position of the last tile of CTA 0 (one of the CTAs that run the most tiles), then random positions"""
    B, Cc, H, W, K, R = case.shape
    TH, grid, n_tiles = p["TH"], p["grid"], p["n_tiles"]
    tpi = H // TH
    last = (n_tiles - 1) // grid * grid
    fixed = [(b, h, w) for b in (0, B - 1) for h in (0, H - 1) for w in (0, W - 1)]
    fixed += [(last // tpi, (last % tpi) * TH + m // W, m % W) for m in (0, 69, 127)]
    rnd = [(int(torch.randint(0, B, (1,), generator=g)), int(torch.randint(0, H, (1,), generator=g)),
            int(torch.randint(0, W, (1,), generator=g))) for _ in range(max(0, K - len(fixed)))]
    return (fixed + rnd)[:K]


def _second(case, p, pos, mode):
    """the position of a second entry: same offset in the next tile (owned by the next CTA), or 32 positions further
    inside the same tile (another weight-gradient step of the same CTA)"""
    B, Cc, H, W, K, R = case.shape
    TH, n_tiles = p["TH"], p["n_tiles"]
    tpi = H // TH
    b, h, w = pos
    t, m = b * tpi + h // TH, (h % TH) * W + w
    if mode == "other_cta":
        t = (t + 1) % n_tiles
    else:
        m = (m + 32) % 128
    return t // tpi, (t % tpi) * TH + m // W, m % W


@pytest.mark.parametrize("mode", ["one", "other_cta", "other_step"])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("cid", FU.SPARSE_WGRAD)
def test_wgrad_sparse_dy_is_exact(cid, variant, mode):
    case = FU.CASES[cid]
    p = _expect_plan(case, True)
    B, Cc, H, W, K, R = case.shape
    g = torch.Generator().manual_seed(_seed(cid, variant, mode))
    gx, gd = VARIANTS[variant]
    x = gx(B * Cc * H * W, g, -20, 20).view(B, Cc, H, W).to(DEV)
    cols = TF.unfold(x, R, padding=R // 2)
    dy = torch.zeros(B, K, H, W, device=DEV)
    chan = torch.arange(K)
    entries = [_positions(case, p, g)]
    if mode != "one":
        entries.append([_second(case, p, q, mode) for q in entries[0]])
    ref = None
    for pos in entries:
        bs, hs, ws = (torch.tensor(v) for v in zip(*pos))
        d = gd(K, g, -10, 10).to(DEV)
        dy[bs, chan, hs, ws] = d
        term = cols[bs.to(DEV), :, (hs * W + ws).to(DEV)] * d[:, None]     # [K, KR], exact products
        ref = term if ref is None else ref + term                          # one round-to-nearest add
    dw = _wgrad(case.shape, dy, x).view(K, -1)
    bad = dw != ref
    assert not bad.any(), (f"{cid} {variant} {mode}: {int(bad.sum())} of {dw.numel()} differ, first at "
                           f"{bad.nonzero()[0].tolist()}: {dw[bad][0].item()!r} vs {ref[bad][0].item()!r}")


# ------------------------------------------------------------------------------------------------ c. random vs fp64
def _wgrad_c(p):
    """error constant of the weight gradient, from its summation structure (first order, in units of u = 2^-24 of R):
    2            the dropped piece products (<= 2 u |x||dy| per term, as in the forward);
    24           one 32-position step = 12 MMAs into a register accumulator, each rounding (or truncating) <= 2 u;
    S            S = 4 ceil(n_tiles / grid) steps added into the CTA's running sum with round-to-nearest adds;
    grid         the CTAs' partial sums added one after another in reduce_partials_kernel.
    NIN-GC stem at batch 256: 2 + 24 + 64 + 132 = 222."""
    return 2 + 24 + 4 * -(-p["n_tiles"] // p["grid"]) + p["grid"]


def _operands(shape, kind, g):
    B, Cc, H, W, K, R = shape

    def spread(*s):
        n = math.prod(s)
        v = torch.randn(n, generator=g) * torch.ldexp(torch.ones(n), torch.randint(-8, 9, (n,), generator=g))
        return (v.abs() if kind == "positive" else v).view(*s).to(DEV)

    x, w, b, dy = spread(B, Cc, H, W), spread(K, Cc, R, R), spread(K), spread(B, K, H, W)
    dy[torch.rand(dy.shape, generator=g).to(DEV) < 0.25] = 0.0     # exact zeros
    return x, w, b, dy


def _fwd64(x, w, b, R):
    y64 = TF.conv2d(x.double(), w.double(), b.double(), padding=R // 2)
    r64 = TF.conv2d(x.double().abs(), w.double().abs(), b.double().abs(), padding=R // 2)
    return y64, r64


def _wgrad64(x, dy, wshape, R):
    d64 = torch.nn.grad.conv2d_weight(x.double(), wshape, dy.double(), padding=R // 2)
    r64 = torch.nn.grad.conv2d_weight(x.double().abs(), wshape, dy.double().abs(), padding=R // 2)
    return d64, r64


def _worst(got, ref, r64, c, what):
    ratio = ((got.double() - ref).abs() / r64.clamp_min(1e-300)).max().item() / U
    print(f"{what}: worst err/R = {ratio:.2f} u (bound {c} u)")
    assert torch.isfinite(got).all(), what
    assert ((got.double() - ref).abs() <= c * U * r64).all(), f"{what}: worst err/R = {ratio:.2f} u > {c} u"


@pytest.mark.parametrize("kind", ["spread", "positive"])
@pytest.mark.parametrize("cid", FU.RANDOM)
def test_random_against_fp64(cid, kind):
    case = FU.CASES[cid]
    B, Cc, H, W, K, R = case.shape
    KR = Cc * R * R
    g = torch.Generator().manual_seed(_seed(cid, kind))
    x, w, b, dy = _operands(case.shape, kind, g)
    _expect_plan(case, False)
    y = _fwd(case.shape, x, w, b)
    y64, r64 = _fwd64(x, w, b, R)
    _worst(y, y64, r64, KR + 3, f"{cid} {kind} forward")
    del y, y64, r64
    if case.wgrad is not None:
        p = _expect_plan(case, True)
        dw = _wgrad(case.shape, dy, x)
        d64, r64 = _wgrad64(x, dy, w.shape, R)
        _worst(dw, d64, r64, _wgrad_c(p), f"{cid} {kind} weight gradient")
    else:
        assert FU.plan(FU.shape(*case.shape), True) is None


# ------------------------------------------------------------------------------------------------ d. module routes
class _PresumDy(torch.autograd.Function):
    """identity whose backward tags the gradient with a channel sum, as a fused BatchNorm consumer does"""

    @staticmethod
    def forward(ctx, y, presum):
        ctx.presum = presum
        return y.view_as(y)

    @staticmethod
    def backward(ctx, g):
        g = g.clone()
        g._mnb_channel_sum = ctx.presum
        return g, None


def _module_case(shape, presummed, seed):
    from micronet_b200.fused import EngineFloatConv2d
    B, Cc, H, W, K, R = shape
    g = torch.Generator().manual_seed(seed)
    x, w, b, dy = _operands(shape, "spread", g)
    conv = EngineFloatConv2d(Cc, K, R, 1, R // 2).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(w)
        conv.bias.copy_(b)
    y = conv(x)
    presum = torch.randn(K, generator=g).to(DEV) if presummed else None
    (_PresumDy.apply(y, presum) if presummed else y).backward(dy)
    return x, w, b, dy, y.detach(), conv.weight.grad, conv.bias.grad, presum


@pytest.mark.parametrize("presummed", [False, True], ids=["channel_sums", "presummed"])
@pytest.mark.parametrize("cid", ["ningc_stem", "nin_stem"])
def test_engine_float_conv_module_at_bench_stems(cid, presummed):
    case = FU.CASES[cid]
    B, Cc, H, W, K, R = case.shape
    p = _expect_plan(case, True)
    x, w, b, dy, y, dw, db, presum = _module_case(case.shape, presummed, 11)
    # the module runs the same kernels: bitwise the C entry points' results
    assert torch.equal(y, _fwd(case.shape, x, w, b))
    assert torch.equal(dw, _wgrad(case.shape, dy, x))
    y64, r64 = _fwd64(x, w, b, R)
    _worst(y, y64, r64, Cc * R * R + 3, f"{cid} module forward")
    d64, r64 = _wgrad64(x, dy, w.shape, R)
    _worst(dw, d64, r64, _wgrad_c(p), f"{cid} module weight gradient")
    if presummed:
        assert torch.equal(db, presum)
    else:
        # channel_sums: any summation order of B*H*W terms is within (B*H*W) u of the sum of |dy|
        n = B * H * W
        _worst(db, dy.double().sum((0, 2, 3)), dy.double().abs().sum((0, 2, 3)), n, f"{cid} module bias gradient")


def test_quant_conv_fn_first_layer_route_runs_the_fp32_kernels():
    """QuantConv2dFn without an activation quantizer on an fp32 input (the DoReFa / IAO first layer) runs
    mnb_fconv2d_fwd_tc and mnb_fconv2d_wgrad_tc: same results as the C entry points, both recorded by KernelTimer"""
    from micronet_b200 import functional as F_
    case = FU.CASES["nin_stem"]
    B, Cc, H, W, K, R = shape = (16,) + case.shape[1:]
    g = torch.Generator().manual_seed(3)
    x, w, b, dy = _operands(shape, "spread", g)
    wq = w.clone().requires_grad_(True)
    old, F_.TIMER = F_.TIMER, F_.KernelTimer()
    try:
        y = F_.quant_conv2d(x, wq, b, None, None, None, (1, 1), (R // 2, R // 2), (1, 1), 1)
        y.backward(dy)
        kinds = [r[0] for r in F_.TIMER.records]
    finally:
        F_.TIMER = old
    assert "fconv_fwd_tc" in kinds and "fconv_wgrad_tc" in kinds, kinds
    assert torch.equal(y.detach(), _fwd(shape, x, w, b))
    assert torch.equal(wq.grad, _wgrad(shape, dy, x))


# (B, C, H, W, K, R): forward on the engine with the weight gradient on ATen, and a shape both kernels refuse
@pytest.mark.parametrize("shape", [(8, 2, 32, 32, 144, 7), (2, 3, 48, 48, 16, 3)], ids=["mixed_kr98_k144", "refused_48x48"])
def test_module_fallbacks_against_fp64(shape):
    B, Cc, H, W, K, R = shape
    fwd_plan, wg_plan = FU.plan(FU.shape(*shape), False), FU.plan(FU.shape(*shape), True)
    assert wg_plan is None and (fwd_plan is not None) == (H == 32)
    x, w, b, dy, y, dw, db, _ = _module_case(shape, False, 5)
    if fwd_plan is not None:
        assert torch.equal(y, _fwd(shape, x, w, b))
    y64, r64 = _fwd64(x, w, b, R)
    _worst(y, y64, r64, Cc * R * R + 3, f"{shape} module forward")
    # ATen's weight gradient: its summation order is its own; any order of B*H*W terms is within (B*H*W + 1) u R
    d64, r64 = _wgrad64(x, dy, w.shape, R)
    _worst(dw, d64, r64, B * H * W + 1, f"{shape} module weight gradient (ATen)")


def test_refused_launch_leaves_outputs_untouched():
    L, lib = _lib()
    shape = (2, 3, 48, 48, 16, 3)
    sh = FU.shape(*shape)
    x = torch.randn(2, 3, 48, 48, device=DEV)
    w = torch.randn(16, 3, 3, 3, device=DEV)
    dy = torch.randn(2, 16, 48, 48, device=DEV)
    y, dw, scratch = _nan((2, 16, 48, 48)), _nan((16, 3, 3, 3)), _nan((1024,))
    torch.cuda.synchronize()
    before = L.launch_count()
    err = L.tc_err_flag(x.device).data_ptr()
    assert lib.mnb_fconv2d_fwd_tc(C.byref(sh), x.data_ptr(), w.data_ptr(), None, y.data_ptr(), err, L.stream()) \
        == L.E_UNSUPPORTED
    assert lib.mnb_fconv2d_wgrad_tc(C.byref(sh), dy.data_ptr(), x.data_ptr(), dw.data_ptr(), scratch.data_ptr(), err,
                                    L.stream()) == L.E_UNSUPPORTED
    assert L.launch_count() == before
    torch.cuda.synchronize()
    assert torch.isnan(y).all() and torch.isnan(dw).all() and torch.isnan(scratch).all()
