"""Fused wgmma forward conv (mnb_fq_conv2d_fwd_tc) against the generic kernels, the standalone
quantizer kernel (codes / STE bits must be identical) and ATen-CPU conv2d.

The "tc" leg turns the packed-operand family off (L.PK_MODE = "off"): with a quantizer spec QuantConv2dFn would otherwise
take that family first, whatever USE_TC says.  Inside the documented cover (DESIGN.md §4.1/§4.2) the leg must have run
fwd_tc / dgrad_tc / wgrad_tc; the shapes instantiate every group width 16..160 of conv_tc_kernel, forward (K/g) and data
gradient (C/g).

The second half of the file runs every case of tests/tc_conv_cases.py through the C ABI against fp64, element by element:
integer operands bitwise against the exact epilogue, raw fp32 operands within the fp32 accumulation bound, operand buffers
that switch between exact and inexact entries (stale mid / lo pieces), the STE mask of the data gradient and the inexact
flag of the weight gradient."""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests.oracle_util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# B, C, H, W, K, R, groups           (stride 1, 'same' padding)
SHAPES = [
    (4, 256, 32, 32, 256, 1, 2),     # NIN-GC conv 2/3
    (4, 256, 16, 16, 512, 3, 16),    # NIN-GC conv 4
    (4, 512, 16, 16, 512, 1, 4),     # NIN-GC conv 5/6
    (4, 512, 8, 8, 1024, 3, 32),     # NIN-GC conv 7
    (5, 1024, 8, 8, 1024, 1, 8),     # NIN-GC conv 8 (odd batch: partial 2-image tile)
    (3, 192, 32, 32, 160, 1, 1),     # NIN conv 2
    (2, 64, 32, 32, 64, 3, 1),       # ResNet conv2_x
    (2, 32, 16, 16, 32, 5, 1),       # 5x5
    (3, 48, 4, 4, 64, 1, 1),         # 4x4 images, 8 per tile
    (2, 16, 12, 12, 16, 3, 1),       # W not a power of two
    (2, 48, 16, 16, 80, 3, 1),       # group widths: forward 80, data gradient 48
    (2, 96, 16, 16, 112, 3, 1),      # weights of the group (189 KB) do not fit in shared memory: generic kernels
    (2, 96, 16, 16, 112, 1, 1),      # 112 / 96
    (2, 144, 8, 8, 48, 3, 1),        # 48 / 144
    (2, 112, 8, 8, 144, 1, 1),       # 144 / 112
    (2, 80, 8, 8, 96, 1, 1),         # 96 / 80
]


def _tc_cover(shape, which):
    """inside the cover of the fused tensor-core kernels (DESIGN.md §4.1 / §4.2) for these stride-1 'same' shapes?"""
    B, C, H, W, K, R, G = shape
    if (C // G) % 16 or (K // G) % 16 or W > 64 or (W * 4) % 16:
        return False
    n = {"fwd": K // G, "dgrad": C // G, "wgrad": 0}[which]       # accumulator columns of the kernel instance
    # forward and dgrad keep the bf16 weights of a group resident next to at least two staging slots: 128 KB is inside
    # what the plan leaves at these tile sizes
    fits = which == "wgrad" or R * R * (C // G) * (K // G) * 2 <= 128 * 1024
    return n <= 160 and fits and (which != "wgrad" or C // G <= 256)


def _legs(use_tc):
    """switch the engine to the fused tensor-core kernels (packed-operand family off) or to the generic fallback;
    returns a restore function"""
    from micronet_b200 import _lib as L, functional as F_
    old = (L.USE_TC, L.PK_MODE, F_.TIMER)
    L.USE_TC = use_tc
    if use_tc:
        L.PK_MODE = "off"
    F_.TIMER = F_.KernelTimer()

    def restore():
        kinds = {k for k, _, _, _ in F_.TIMER.records}
        L.USE_TC, L.PK_MODE, F_.TIMER = old
        return kinds
    return restore


def _run(x, wq, bias, w_int, w_scale, spec, R, G, use_tc):
    from micronet_b200 import functional as F_
    restore = _legs(use_tc)
    try:
        xg = x.clone().requires_grad_(True)
        y = F_.quant_conv2d(xg, wq, bias, w_int, w_scale, spec, (1, 1), (R // 2, R // 2), (1, 1), G)
        torch.cuda.synchronize()
    finally:
        kinds = restore()
    return y, kinds


@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
@pytest.mark.parametrize("mode", ["raw_pm1", "raw_fp32", "dorefa8", "dorefa4", "iao_sym", "iao_asym"])
def test_tc_forward_matches_generic_and_cpu(shape, mode):
    from micronet_b200 import _lib as L, functional as F_
    B, C, H, W, K, R, G = shape
    g = torch.Generator().manual_seed(hash((shape, mode)) % (1 << 31))
    if mode == "raw_pm1":
        x = torch.randint(0, 2, (B, C, H, W), generator=g).float() * 2 - 1
    else:
        x = torch.randn(B, C, H, W, generator=g) * 3
    lim = 1 if mode.startswith("raw") else (255 if mode == "dorefa8" else (15 if mode == "dorefa4" else 127))
    w_int = torch.randint(-lim, lim + 1, (K, C // G, R, R), generator=g, dtype=torch.int16)
    w_scale = torch.rand(K, generator=g) * 0.02 + 0.001
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    bias = torch.randn(K, generator=g)
    spec = None
    bufs = {}
    if mode.startswith("dorefa"):
        spec = F_.ActSpec(L.ACT_DOREFA, bits=int(mode[6:]))
    elif mode.startswith("iao"):
        sym = mode == "iao_sym"
        qmin, qmax = (-128, 127) if sym else (0, 255)
        mn, mx = torch.tensor([-7.5]), torch.tensor([8.25])
        if sym:
            s = torch.max(mn.abs(), mx.abs()) / 127.5
            zp = torch.zeros(1)
        else:
            s = (mx - mn) / 255.0
            zp = torch.sign(mn) * torch.floor((mn / s).abs() + 0.5)
        bufs = {k: v.to(DEV) for k, v in dict(scale=s, zero_point=zp, obs_min=mn, obs_max=mx).items()}
        spec = F_.ActSpec(L.ACT_IAO, qmin=qmin, qmax=qmax, q_type=0 if sym else 1, **bufs)
    xd, wqd, bd, wid, wsd = (t.to(DEV) for t in (x, wq, bias, w_int, w_scale))
    err = L.tc_err_flag(torch.device(DEV))
    err.zero_()
    n0 = L.launch_count()
    y_tc, kinds = _run(xd, wqd, bd, wid, wsd, spec, R, G, True)
    assert err.item() == 0, f"tensor-core pipeline timed out, code {err.item()}"
    if _tc_cover(shape, "fwd"):
        # fwd_tc is recorded whether or not the kernel ran; the generic kind only when the generic kernel did
        assert "fwd_tc" in kinds and "fwd" not in kinds, kinds
    assert not any(k.endswith("_pk") for k in kinds), kinds
    y_gen, _ = _run(xd, wqd, bd, wid, wsd, spec, R, G, False)
    assert torch.isfinite(y_tc).all()
    # both paths are exact on integer levels; on raw fp32 they differ only by fp32 summation order
    assert rel_err(y_tc, y_gen) <= (5e-6 if mode == "raw_fp32" else 1e-6), f"tc vs generic {rel_err(y_tc, y_gen)}"
    # CPU reference: conv2d of the dequantized operands
    if spec is None:
        xq = x
    else:
        _, _, xqd = F_.act_quant_raw(xd, spec, False, False, True)
        xq = xqd.cpu()
    want = TF.conv2d(xq.double(), wq.double(), bias.double(), 1, R // 2, 1, G).float()
    assert rel_err(y_tc, want) <= 1e-5, f"tc vs cpu {rel_err(y_tc, want)}"


@pytest.mark.parametrize("shape", SHAPES[:5] + SHAPES[6:8], ids=str)
@pytest.mark.parametrize("mode", ["dorefa8", "iao_sym"])
def test_tc_forward_emits_identical_codes_and_bits(shape, mode):
    import ctypes as C
    from micronet_b200 import _lib as L, functional as F_
    lib = L.load()
    B, Cc, H, W, K, R, G = shape
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(B, Cc, H, W, generator=g) * 4).to(DEV)
    w_int = torch.randint(-127, 128, (K, Cc // G, R, R), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) * 0.02 + 0.001).to(DEV)
    if mode == "dorefa8":
        spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
    else:
        bufs = dict(scale=torch.tensor([9.0 / 127.5]), zero_point=torch.zeros(1), obs_min=torch.tensor([-9.0]),
                    obs_max=torch.tensor([7.0]))
        spec = F_.ActSpec(L.ACT_IAO, qmin=-128, qmax=127, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})
    codes_ref, bits_ref, _ = F_.act_quant_raw(x, spec, True, True, False)
    sh = L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, R // 2, R // 2, 1, 1, G)
    y = torch.empty(B, K, H, W, device=DEV)
    codes = torch.full(x.shape, 77, dtype=torch.uint8, device=DEV)
    bits = torch.zeros_like(bits_ref)
    err = L.tc_err_flag(torch.device(DEV)); err.zero_()
    qp = spec.struct()
    wpack = torch.empty(w_int.numel(), dtype=torch.int16, device=DEV)
    rc = lib.mnb_fq_conv2d_fwd_tc(C.byref(sh), x.data_ptr(), C.byref(qp), w_int.data_ptr(), w_scale.data_ptr(), None,
                                  y.data_ptr(), codes.data_ptr(), bits.data_ptr(), wpack.data_ptr(), err.data_ptr(),
                                  L.stream())
    if rc == L.E_UNSUPPORTED:
        pytest.skip("geometry not covered by the tensor-core kernel")
    L.check(rc, "fq_conv2d_fwd_tc")
    torch.cuda.synchronize()
    assert err.item() == 0
    assert torch.equal(codes, codes_ref)
    assert torch.equal(bits, bits_ref)


@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
@pytest.mark.parametrize("mode", ["raw", "dorefa8", "iao_sym"])
def test_tc_dgrad_matches_generic_and_cpu(shape, mode):
    """dx through the tensor-core dgrad (weight scale folded into dy, exact 3-term split, fused STE)."""
    from micronet_b200 import _lib as L, functional as F_
    B, C, H, W, K, R, G = shape
    g = torch.Generator().manual_seed(hash((shape, mode, "dgrad")) % (1 << 31))
    x = torch.randn(B, C, H, W, generator=g) * 4
    lim = 1 if mode == "raw" else 127
    w_int = torch.randint(-lim, lim + 1, (K, C // G, R, R), generator=g, dtype=torch.int16)
    w_scale = torch.rand(K, generator=g) * 0.02 + 0.001
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    spec = None
    if mode == "dorefa8":
        spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
    elif mode == "iao_sym":
        bufs = dict(scale=torch.tensor([9.0 / 127.5]), zero_point=torch.zeros(1), obs_min=torch.tensor([-9.0]),
                    obs_max=torch.tensor([7.0]))
        spec = F_.ActSpec(L.ACT_IAO, qmin=-128, qmax=127, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})
    go = torch.randn(B, K, H, W, generator=g)
    err = L.tc_err_flag(torch.device(DEV)); err.zero_()
    grads, kinds = {}, {}
    for use_tc in (True, False):
        restore = _legs(use_tc)
        try:
            xg = x.to(DEV).requires_grad_(True)
            y = F_.quant_conv2d(xg, wq.to(DEV), None, w_int.to(DEV), w_scale.to(DEV), spec, (1, 1), (R // 2, R // 2), (1, 1), G)
            y.backward(go.to(DEV))
            torch.cuda.synchronize()
            grads[use_tc] = xg.grad.clone()
        finally:
            kinds[use_tc] = restore()
    assert err.item() == 0, f"tensor-core pipeline timed out, code {err.item()}"
    if _tc_cover(shape, "dgrad"):
        assert "dgrad_tc" in kinds[True] and "dgrad" not in kinds[True], kinds[True]
    assert not any(k.endswith("_pk") for k in kinds[True]), kinds[True]
    assert rel_err(grads[True], grads[False]) <= 5e-6, rel_err(grads[True], grads[False])  # fp32 summation order
    # CPU: autograd of conv2d on the dequantized input
    from oracle import reference_port as O
    xr = x.clone().requires_grad_(True)
    if mode == "raw":
        xq = xr
    elif mode == "dorefa8":
        xq = O.dorefa_quantize_activation(xr, 8)
    else:
        s = torch.tensor([9.0 / 127.5])
        v = xr / s
        r = O._RoundRangeSTE.apply(v, torch.tensor([-9.0]) / s, torch.tensor([7.0]) / s, 0)
        xq = torch.clamp(r, -128, 127) * s
    TF.conv2d(xq, wq, None, 1, R // 2, 1, G).backward(go)
    assert rel_err(grads[True], xr.grad) <= 1e-5, rel_err(grads[True], xr.grad)


@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
@pytest.mark.parametrize("mode", ["raw_pm1", "raw_fp32", "dorefa8", "iao_sym"])
def test_tc_wgrad_matches_generic_and_cpu(shape, mode):
    """dWq through the tensor-core wgrad (MN-major operands, register accumulators, deterministic
    two-stage reduction); raw fp32 inputs that are not bf16-exact take the device-side fallback."""
    from micronet_b200 import _lib as L, functional as F_
    from oracle import reference_port as O
    B, C, H, W, K, R, G = shape
    g = torch.Generator().manual_seed(hash((shape, mode, "wgrad")) % (1 << 31))
    if mode == "raw_pm1":
        x = torch.randint(0, 2, (B, C, H, W), generator=g).float() * 2 - 1
    else:
        x = torch.randn(B, C, H, W, generator=g) * 4
    lim = 1 if mode.startswith("raw") else 127
    w_int = torch.randint(-lim, lim + 1, (K, C // G, R, R), generator=g, dtype=torch.int16)
    w_scale = torch.rand(K, generator=g) * 0.02 + 0.001
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    spec = None
    if mode == "dorefa8":
        spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
    elif mode == "iao_sym":
        bufs = dict(scale=torch.tensor([9.0 / 127.5]), zero_point=torch.zeros(1), obs_min=torch.tensor([-9.0]),
                    obs_max=torch.tensor([7.0]))
        spec = F_.ActSpec(L.ACT_IAO, qmin=-128, qmax=127, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})
    go = torch.randn(B, K, H, W, generator=g)
    err = L.tc_err_flag(torch.device(DEV)); err.zero_()
    grads, kinds = {}, {}
    for use_tc in (True, False):
        restore = _legs(use_tc)
        try:
            wg = wq.to(DEV).requires_grad_(True)
            y = F_.quant_conv2d(x.to(DEV), wg, None, w_int.to(DEV), w_scale.to(DEV), spec, (1, 1), (R // 2, R // 2), (1, 1), G)
            y.backward(go.to(DEV))
            torch.cuda.synchronize()
            grads[use_tc] = wg.grad.clone()
        finally:
            kinds[use_tc] = restore()
    assert err.item() == 0, f"tensor-core pipeline timed out, code {err.item()}"
    if _tc_cover(shape, "wgrad") and mode != "raw_fp32":
        assert "wgrad_tc" in kinds[True] and "wgrad" not in kinds[True], kinds[True]
    assert not any(k.endswith("_pk") for k in kinds[True]), kinds[True]
    assert torch.isfinite(grads[True]).all()
    assert rel_err(grads[True], grads[False]) <= 1e-5, rel_err(grads[True], grads[False])
    if mode.startswith("raw"):
        xq = x
    elif mode == "dorefa8":
        xq = O.dorefa_quantize_activation(x, 8)
    else:
        s = torch.tensor([9.0 / 127.5])
        xq = torch.clamp(O.round_half_away(x / s), -128, 127) * s
    wr = wq.clone().double().requires_grad_(True)
    TF.conv2d(xq.double(), wr, None, 1, R // 2, 1, G).backward(go.double())
    assert rel_err(grads[True], wr.grad) <= 1e-5, rel_err(grads[True], wr.grad)


def test_backward_stays_on_the_family_of_the_forward():
    """the backward of a layer whose forward ran on the fused tensor-core kernels runs dgrad_tc / wgrad_tc even when
    L.USE_TC changes between forward and backward, with the gradients of a run that never changes it"""
    from micronet_b200 import _lib as L, functional as F_
    B, C, H, W, K, R, G = SHAPES[0]
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(B, C, H, W, generator=g) * 4).to(DEV)
    w_int = torch.randint(-127, 128, (K, C // G, R, R), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) * 0.02 + 0.001).to(DEV)
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    go = torch.randn(B, K, H, W, generator=g).to(DEV)
    spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
    grads, kinds = {}, {}
    for flip in (False, True):
        restore = _legs(True)
        try:
            xg, wg = x.clone().requires_grad_(True), wq.clone().requires_grad_(True)
            y = F_.quant_conv2d(xg, wg, None, w_int, w_scale, spec, (1, 1), (R // 2, R // 2), (1, 1), G)
            if flip:
                L.USE_TC = False
            y.backward(go)
            torch.cuda.synchronize()
            grads[flip] = (xg.grad, wg.grad)
        finally:
            kinds[flip] = restore()
        assert {"fwd_tc", "dgrad_tc", "wgrad_tc"} <= kinds[flip], (flip, kinds[flip])
        assert not {"fwd", "dgrad", "wgrad"} & kinds[flip], (flip, kinds[flip])
    L.tc_check()
    assert torch.equal(grads[True][0], grads[False][0]) and torch.equal(grads[True][1], grads[False][1])


# =====================================================================================================================
# Every case of tests/tc_conv_cases.py, through the C ABI, element by element against fp64.  Outputs are NaN-filled before
# each launch, every launch runs twice with bitwise-identical results and a clean error flag, and every case's plan is the
# pinned one (the launchers plan with the function the query reports).
from tests import tc_conv_cases as T  # noqa: E402

FWD_CASES = [c for c in T.CASES if c.fwd is not None]
DGRAD_CASES = [c for c in T.CASES if c.dgrad is not None]
WGRAD_CASES = [c for c in T.CASES if c.wgrad is not None]
SMALL = lambda cases: [c for c in cases if c.id not in T.MODEL_CASES]   # noqa: E731
EPS = 2.0 ** -24


def _pinned(case):
    assert T.plans(case.shape) == (case.fwd, case.dgrad, case.wgrad), case.id


def _twice(fn):
    """run ``fn`` (returns a tuple of output tensors) twice: identical bits, no NaN left, error flag clean"""
    from micronet_b200 import _lib as L
    err = L.tc_err_flag(torch.device(DEV))
    err.zero_()
    a = fn()
    b = fn()
    torch.cuda.synchronize()
    assert err.item() == 0, f"tensor-core pipeline timed out, code {err.item()}"
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8) if u.dtype == torch.float32 else u,
                           v.view(torch.uint8) if v.dtype == torch.float32 else v), "two launches differ"
        if u.dtype == torch.float32:
            assert not torch.isnan(u).any(), "outputs left unwritten"
    return a


def _ulp(v):
    v = v.float().abs()
    return (torch.nextafter(v, torch.full_like(v, float("inf"))) - v).double()


def _fmaf_exact(sum64, scale, bias):
    """float32(fmaf(float32(sum), scale, bias)) per element from the exact fp64 sum, correctly rounded"""
    from tests.pk_plan_util import fmaf32
    return fmaf32(sum64.float(), scale.view(1, -1, 1, 1), bias.view(1, -1, 1, 1))


def _check_bound(got, ref, absref, n, scale=1.0, what=""):
    """|got - ref| <= n 2^-24 |scale| absref + one ulp of the result, per element; returns the worst ratio"""
    bound = n * EPS * abs(scale) * absref + _ulp(ref)
    d = (got.double() - ref).abs()
    ratio = (d / bound).max().item()
    assert ratio <= 1.0, f"{what}: error {ratio:.3f} x the element-wise bound"
    return ratio


def _specs(mode):
    """(ActSpec or None, a_scale as fp32 tensor, level offset added to the codes)"""
    from micronet_b200 import _lib as L, functional as F_
    one = torch.ones(1, device=DEV)
    if mode in ("pm1", "raw"):
        return None, one, 0.0
    if mode.startswith("dorefa"):
        bits = int(mode[6:])
        return F_.ActSpec(L.ACT_DOREFA, bits=bits), F_._dorefa_scale_tensor(bits, torch.device(DEV)), 0.0
    sym = mode == "iao_sym"
    qmin, qmax = (-128, 127) if sym else (0, 255)
    mn, mx = torch.tensor([-7.5]), torch.tensor([8.25])
    s = torch.max(mn.abs(), mx.abs()) / 127.5 if sym else (mx - mn) / 255.0
    zp = torch.zeros(1) if sym else torch.sign(mn) * torch.floor((mn / s).abs() + 0.5)
    bufs = {k: v.to(DEV) for k, v in dict(scale=s, zero_point=zp, obs_min=mn, obs_max=mx).items()}
    spec = F_.ActSpec(L.ACT_IAO, qmin=qmin, qmax=qmax, q_type=0 if sym else 1, **bufs)
    return spec, bufs["scale"], float(qmin + zp.item())


def _input(shape, mode, g):
    B, Cc, H, W = shape
    if mode == "pm1":
        return (torch.randint(0, 2, shape, generator=g, device=DEV).float() * 2 - 1)
    if mode.startswith("dorefa"):   # clip edges 0 and 10 (0.1 x in [0, 1]) among the values
        x = torch.rand(shape, generator=g, device=DEV) * 14 - 2
    else:
        x = torch.randn(shape, generator=g, device=DEV) * 4
    edges = torch.tensor([0.0, 10.0] if mode.startswith("dorefa") else [-7.5, 8.25, 0.0], device=DEV)
    pick = torch.randint(0, 8, shape, generator=g, device=DEV)
    return torch.where(pick < len(edges), edges[pick.clamp(max=len(edges) - 1)], x)


def _weights(K, cg, R, lim, g, pow2_scale=False):
    w_int = torch.randint(-lim, lim + 1, (K, cg, R, R), generator=g, device=DEV, dtype=torch.int16)
    if pow2_scale:
        w_scale = 2.0 ** torch.randint(-3, 3, (K,), generator=g, device=DEV).float()
    else:
        w_scale = torch.rand(K, generator=g, device=DEV) * 0.02 + 0.001
    return w_int, w_scale


def _fwd(case, x, spec, w_int, w_scale, bias, want_codes=False):
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    B, Cc, H, W, K, R, G = case.shape
    sh = T.conv_shape(case.shape)

    def run():
        y = torch.full((B, K, H, W), float("nan"), device=DEV)
        codes = torch.full(x.shape, 77, dtype=torch.uint8, device=DEV) if spec is not None else None
        bits = torch.zeros((x.numel() + 31) // 32, dtype=torch.int32, device=DEV) if spec is not None else None
        wpack = torch.empty(w_int.numel(), dtype=torch.int16, device=DEV)
        qp = spec.struct() if spec is not None else None
        L.check(lib.mnb_fq_conv2d_fwd_tc(C.byref(sh), x.data_ptr(), None if qp is None else C.byref(qp), w_int.data_ptr(),
                                         w_scale.data_ptr(), L.ptr(bias), y.data_ptr(), L.ptr(codes), L.ptr(bits),
                                         wpack.data_ptr(), L.tc_err_flag(x.device).data_ptr(), L.stream()), "fwd_tc")
        return (y,) if spec is None else (y, codes, bits)
    return _twice(run)


def _levels(x, spec, codes, offset):
    """the integer level the kernel multiplies: the fused quantizer's code plus its offset (codes equal the standalone
    quantizer's), or x itself"""
    from micronet_b200 import functional as F_
    if spec is None:
        return x.double()
    ref_codes, _, _ = F_.act_quant_raw(x, spec, True, False, False)
    assert torch.equal(codes, ref_codes), "fused quantizer codes differ from the standalone quantizer's"
    return codes.double() + offset


@pytest.mark.parametrize("mode", ["pm1", "dorefa4", "dorefa8", "iao_sym", "iao_asym"])
@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: c.id)
def test_forward_integer_operands_equal_the_exact_epilogue(case, mode):
    """integer operands with every partial sum below 2^24: y is bitwise fmaf(sum, a_scale * w_scale, bias) of the exact
    sum (the fp32 accumulation is exact), at every element"""
    if case.id in T.MODEL_CASES and mode not in ("pm1", "dorefa4"):
        pytest.skip("model shapes: the wbwtab operands and one quantizer")
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(hash((case.id, mode)) % (1 << 31))
    spec, a_scale, off = _specs(mode)
    emax = 1 if spec is None else 255
    lim = 1 if mode == "pm1" else max(1, min(127, (2 ** 24 - 1) // ((Cc // G) * R * R * emax)))
    x = _input((B, Cc, H, W), mode, g)
    w_int, w_scale = _weights(K, Cc // G, R, lim, g)
    bias = torch.randn(K, generator=g, device=DEV)
    out = _fwd(case, x, spec, w_int, w_scale, bias)
    e = _levels(x, spec, out[1] if spec is not None else None, off)
    s64 = TF.conv2d(e, w_int.double(), None, 1, R // 2, 1, G)
    assert s64.abs().max().item() < 2 ** 24
    sc = (a_scale * w_scale).float()                     # __fmul_rn(a_scale, w_scale[n]) of the kernel's constants
    bad = out[0] != _fmaf_exact(s64, sc, bias)
    assert not bad.any(), f"{int(bad.sum())} elements differ from the exact epilogue, first at {bad.nonzero()[0].tolist()}"


def test_forward_sums_past_2_24_keep_the_fp32_bound():
    """8-bit levels, 1568 terms per output: sums reach ~2^25.  The round-1 forward accumulates in fp32 and does not
    segment, so it is held to the fp32 accumulation bound, not to the exact sum"""
    case = T.BY_ID["cc16_mma_off_7x7"]
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(5)
    spec, a_scale, off = _specs("dorefa8")
    x = torch.full((B, Cc, H, W), 10.0, device=DEV) - torch.rand((B, Cc, H, W), generator=g, device=DEV) * 0.2
    w_int = (127 - torch.randint(0, 3, (K, Cc // G, R, R), generator=g, device=DEV)).to(torch.int16)
    w_scale, bias = torch.full((K,), 2.0 ** -20, device=DEV), torch.zeros(K, device=DEV)
    y, codes, _ = _fwd(case, x, spec, w_int, w_scale, bias)
    e = _levels(x, spec, codes, off)
    s64 = TF.conv2d(e, w_int.double(), None, 1, R // 2, 1, G)
    assert s64.abs().max().item() > 2 ** 25
    sc = (a_scale * w_scale).float().double().view(1, -1, 1, 1)
    a64 = TF.conv2d(e.abs(), w_int.double().abs(), None, 1, R // 2, 1, G)
    ratio = _check_bound(y, s64 * sc, a64 * sc, (Cc // G) * R * R, what="sums past 2^24")
    print(f"sums past 2^24: worst error {ratio:.3f} x bound, exact elements {(y.double() == s64 * sc).float().mean():.3f}")


@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: c.id)
def test_forward_raw_fp32_within_the_fp32_bound(case):
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(hash(case.id) % (1 << 31))
    x = torch.randn((B, Cc, H, W), generator=g, device=DEV) * 3
    w_int, w_scale = _weights(K, Cc // G, R, 1, g)
    bias = torch.randn(K, generator=g, device=DEV)
    (y,) = _fwd(case, x, None, w_int, w_scale, bias)
    s64 = TF.conv2d(x.double(), w_int.double(), None, 1, R // 2, 1, G)
    a64 = TF.conv2d(x.double().abs(), w_int.double().abs(), None, 1, R // 2, 1, G)
    sc = w_scale.double().view(1, -1, 1, 1)
    ratio = _check_bound(y, s64 * sc + bias.double().view(1, -1, 1, 1), a64 * sc, 3 * R * R * (Cc // G), what=case.id)
    print(f"raw fp32 forward {case.id}: worst error {ratio:.3f} x bound")


# ---- mixed exactness: operand buffers that go exact -> inexact -> exact, entry by entry and chunk by chunk
EXACT, SPARSE_A, SPARSE_B, DENSE = range(4)
INEXACT = 1.0 + 2.0 ** -9


def _mixed(shape, seed):
    """values in {-1, 0, 1} with a few 1 + 2^-9 (not bf16-exact); each (image, 32-channel chunk) has one state:
    EXACT (and whole 8-channel entries zero), SPARSE_A / SPARSE_B (disjoint sets of inexact entries), DENSE (every entry
    inexact).  Returns (tensor, states [B, C/32])"""
    B, Cc, H, W = shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randint(0, 2, shape, generator=g, device=DEV).float() * 2 - 1
    c = torch.arange(Cc, device=DEV).view(1, -1, 1, 1)
    pos = torch.arange(H * W, device=DEV).view(1, 1, H, W)
    states = torch.randint(0, 4, (B, (Cc + 31) // 32), generator=g, device=DEV)
    st = states.repeat_interleave(32, dim=1)[:, :Cc].view(B, Cc, 1, 1)
    key = (pos + c // 8) % 5
    zero = (st == EXACT) & ((pos + c // 8) % 3 == 0)
    inexact = ((st == SPARSE_A) & (key == 0) & (c % 8 == 3)) | ((st == SPARSE_B) & (key == 2) & (c % 8 == 3)) | \
              ((st == DENSE) & (c % 8 == 5))
    x = torch.where(zero, torch.zeros_like(x), x)
    return torch.where(inexact, x * INEXACT, x), states.cpu()


def _buffer_transitions(plan, chunk_states):
    """simulate the CTA schedule of a forward / dgrad plan: for every operand buffer, the set of (previous state, state)
    of the chunks converted into it; chunk_states(tile, group, chunk) -> state"""
    grid, n_slabs, slab, nchunk, nop = plan["grid"], plan["n_slabs"], plan["slab_groups"], plan["nchunk"], plan["nop"]
    seen = {ob: set() for ob in range(nop)}
    for blk in range(grid):
        s, rank = blk % n_slabs, blk // n_slabs
        ctas = (grid - s + n_slabs - 1) // n_slabs
        ob, last = -1, {}
        for tile in range(rank, plan["n_tiles"], ctas):
            for gi in range(slab):
                for ch in range(nchunk):
                    ob = (ob + 1) % nop
                    now = chunk_states(tile, s * slab + gi, ch)
                    if ob in last:
                        seen[ob].add((last[ob], now))
                    last[ob] = now
    return seen


def _assert_all_transitions(seen):
    for ob, tr in seen.items():
        kinds = {
            "inexact entry -> exact entry": any(a != EXACT and b in (SPARSE_A, SPARSE_B) and a != b for a, b in tr),
            "exact entry -> inexact entry": any(a in (EXACT, SPARSE_A, SPARSE_B) and b != EXACT and a != b for a, b in tr),
            "inexact chunk -> fully exact chunk": any(a != EXACT and b == EXACT for a, b in tr),
            "fully exact chunk -> inexact chunk": any(a == EXACT and b != EXACT for a, b in tr),
        }
        assert all(kinds.values()), (ob, kinds)


def test_forward_mixed_exactness_is_exact():
    """stale mid / lo pieces of an entry that was inexact the last time its operand buffer was used must not reach the
    MMAs: every sum is exact in fp32, so any stale piece is an element-wise error"""
    case = T.BY_ID["mixed_3x3"]
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    x, states = _mixed((B, Cc, H, W), 17)
    p = T.fd(case.fwd[0])
    assert p["CC"] == 32 and p["TB"] == 1 and p["row_tiles"] == 1
    _assert_all_transitions(_buffer_transitions(p, lambda tile, gi, ch: int(states[tile, ch])))
    g = torch.Generator(device=DEV).manual_seed(3)
    w_int, w_scale = _weights(K, Cc // G, R, 1, g)
    bias = torch.randn(K, generator=g, device=DEV)
    (y,) = _fwd(case, x, None, w_int, w_scale, bias)
    s64 = TF.conv2d(x.double(), w_int.double(), None, 1, R // 2, 1, G)
    assert torch.equal(s64.float().double(), s64)
    bad = y != _fmaf_exact(s64, w_scale, bias)
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


def _dgrad(case, dy, w_int, w_scale, bits=None, spec=None):
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    B, Cc, H, W, K, R, G = case.shape
    sh = T.conv_shape(case.shape)

    def run():
        dx = torch.full((B, Cc, H, W), float("nan"), device=DEV)
        wpack = torch.empty(w_int.numel(), dtype=torch.int16, device=DEV)
        qp = spec.struct() if spec is not None else None
        L.check(lib.mnb_conv2d_dgrad_tc(C.byref(sh), dy.data_ptr(), w_int.data_ptr(), w_scale.data_ptr(), L.ptr(bits),
                                        None if qp is None else C.byref(qp), dx.data_ptr(), wpack.data_ptr(),
                                        L.tc_err_flag(dy.device).data_ptr(), L.stream()), "dgrad_tc")
        return (dx,)
    return _twice(run)[0]


def test_dgrad_mixed_exactness_is_exact():
    case = T.BY_ID["mixed_3x3"]
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    dy, states = _mixed((B, K, H, W), 23)
    p = T.fd(case.dgrad)
    assert p["CC"] == 32 and p["nchunk"] == 1
    _assert_all_transitions(_buffer_transitions(p, lambda tile, gi, ch: int(states[tile, ch])))
    g = torch.Generator(device=DEV).manual_seed(4)
    w_int, w_scale = _weights(K, Cc // G, R, 1, g, pow2_scale=True)    # dy * w_scale keeps its exactness
    dx = _dgrad(case, dy, w_int, w_scale)
    d = dy.double() * w_scale.double().view(1, -1, 1, 1)
    want = TF.conv_transpose2d(d, w_int.double(), None, 1, R // 2, 0, G)
    assert torch.equal(want.float().double(), want)
    bad = dx.double() != want
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


def _ste_mask(x, mode):
    """the reference quantizer's STE pass mask (its autograd on the CPU)"""
    from oracle import reference_port as O
    xr = x.cpu().clone().requires_grad_(True)
    if mode.startswith("dorefa"):
        xq = O.dorefa_quantize_activation(xr, int(mode[6:]))
    else:
        s = torch.tensor([9.0 / 127.5])
        xq = torch.clamp(O._RoundRangeSTE.apply(xr / s, torch.tensor([-9.0]) / s, torch.tensor([7.0]) / s, 0), -128, 127) * s
    xq.sum().backward()
    return (xr.grad != 0).to(DEV)


@pytest.mark.parametrize("mode", ["plain", "dorefa4", "iao_sym"])
@pytest.mark.parametrize("case", DGRAD_CASES, ids=lambda c: c.id)
def test_dgrad_within_the_fp32_bound_and_masked_exactly(case, mode):
    """dx against the fp64 transposed conv of fp32(dy * w_scale[k]) (the kernel's __fmul_rn) and the integer weights;
    with a quantizer, the STE bits of the standalone quantizer (inputs on the clip edges): masked positions exactly 0"""
    from micronet_b200 import _lib as L, functional as F_
    if case.id in T.MODEL_CASES and mode != "plain":
        pytest.skip("model shapes: plain data gradient (wbwtab)")
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(hash((case.id, mode, "dgrad")) % (1 << 31))
    spec = bits = None
    gain = 1.0
    if mode != "plain":
        if mode == "dorefa4":
            spec = F_.ActSpec(L.ACT_DOREFA, bits=4)
            gain = 0.1
            x = _input((B, Cc, H, W), mode, g)
        else:
            bufs = dict(scale=torch.tensor([9.0 / 127.5]), zero_point=torch.zeros(1), obs_min=torch.tensor([-9.0]),
                        obs_max=torch.tensor([7.0]))
            spec = F_.ActSpec(L.ACT_IAO, qmin=-128, qmax=127, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})
            x = torch.randn((B, Cc, H, W), generator=g, device=DEV) * 5
            x.view(-1)[::7] = -9.0
            x.view(-1)[3::7] = 7.0
            x.view(-1)[5::7] = 9.0
        _, bits, _ = F_.act_quant_raw(x, spec, False, True, False)
    dy = torch.randn((B, K, H, W), generator=g, device=DEV)
    w_int, w_scale = _weights(K, Cc // G, R, 127, g)
    dx = _dgrad(case, dy, w_int, w_scale, bits, spec)
    d = (dy * w_scale.view(1, -1, 1, 1)).double()                  # fp32 product, as __fmul_rn
    want = TF.conv_transpose2d(d, w_int.double(), None, 1, R // 2, 0, G)
    absw = TF.conv_transpose2d(d.abs(), w_int.double().abs(), None, 1, R // 2, 0, G)
    n = 3 * R * R * (K // G)
    if spec is None:
        ratio = _check_bound(dx, want, absw, n, what=case.id)
    else:
        mask = _ste_mask(x, mode)
        idx = torch.arange(x.numel(), device=DEV)
        kbits = ((bits.view(-1)[idx >> 5] >> (idx & 31)) & 1).view(x.shape).bool()
        assert torch.equal(kbits, mask), "quantizer STE bits differ from the reference's pass mask"
        assert 0 < mask.float().mean().item() < 1
        assert (dx[~mask] == 0).all(), "masked positions not exactly 0"
        # pass positions: the fp32 sum times the fp32 gain, one more rounding
        ratio = _check_bound(dx[mask], (want * gain)[mask], (absw * gain)[mask] + _ulp(want * gain)[mask] / EPS / n, n,
                             what=case.id)
    print(f"dgrad {case.id} {mode}: worst error {ratio:.3f} x bound")


def _wgrad(case, dy, x, spec):
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    B, Cc, H, W, K, R, G = case.shape
    sh = T.conv_shape(case.shape)
    nbytes = int(lib.mnb_wgrad_tc_scratch_bytes(C.byref(sh)))
    assert nbytes > 0

    def run():
        dw = torch.full((K, Cc // G, R, R), float("nan"), device=DEV)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        qp = spec.struct() if spec is not None else None
        L.check(lib.mnb_conv2d_wgrad_tc(C.byref(sh), dy.data_ptr(), x.data_ptr(), None if qp is None else C.byref(qp),
                                        dw.data_ptr(), ws.data_ptr(), flag.data_ptr(),
                                        L.tc_err_flag(dy.device).data_ptr(), L.stream()), "wgrad_tc")
        return dw, flag
    return _twice(run)


@pytest.mark.parametrize("mode", ["pm1", "dorefa8", "iao_asym"])
@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: c.id)
def test_wgrad_within_the_fp32_bound(case, mode):
    """dWq = a_scale * sum dy * e_a against fp64, element by element, including the reduce kernel's a_scale; the inexact
    flag stays 0 (every operand is an exact level or +-1)"""
    if case.id in T.MODEL_CASES and mode != "pm1":
        pytest.skip("model shapes: the wbwtab operands")
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(hash((case.id, mode, "wgrad")) % (1 << 31))
    spec, a_scale, off = _specs(mode)
    x = _input((B, Cc, H, W), mode, g)
    dy = torch.randn((B, K, H, W), generator=g, device=DEV)
    dw, flag = _wgrad(case, dy, x, spec)
    assert flag.item() == 0
    if spec is None:
        e = x.double()
    else:
        from micronet_b200 import functional as F_
        codes, _, _ = F_.act_quant_raw(x, spec, True, False, False)
        e = codes.double() + off
    s64 = torch.nn.grad.conv2d_weight(e, dw.shape, dy.double(), 1, R // 2, 1, G)
    a64 = torch.nn.grad.conv2d_weight(e.abs(), dw.shape, dy.double().abs(), 1, R // 2, 1, G)
    sc = float(a_scale.item())
    ratio = _check_bound(dw, s64 * sc, a64 * sc, 3 * B * H * W, what=case.id)
    print(f"wgrad {case.id} {mode}: worst error {ratio:.3f} x bound")


@pytest.mark.parametrize("case", [T.BY_ID[i] for i in ("ng16_tb_ragged", "ng32_h_ragged", "ng112_slab2", "gc_3x3g16")],
                         ids=lambda c: c.id)
def test_wgrad_inexact_flag_and_the_conditional_overwrite(case):
    """one inexact raw activation (the tensor's last element) sets the flag; functional._wgrad then returns bitwise what
    mnb_conv2d_wgrad computes"""
    import ctypes as C
    import types
    from micronet_b200 import _lib as L, functional as F_
    lib = L.load()
    _pinned(case)
    B, Cc, H, W, K, R, G = case.shape
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randint(0, 2, (B, Cc, H, W), generator=g, device=DEV).float() * 2 - 1
    dy = torch.randn((B, K, H, W), generator=g, device=DEV)
    assert _wgrad(case, dy, x, None)[1].item() == 0
    x.view(-1)[-1] = INEXACT
    assert _wgrad(case, dy, x, None)[1].item() == 1
    sh = T.conv_shape(case.shape)
    wq = torch.randn((K, Cc // G, R, R), generator=g, device=DEV)
    ctx = types.SimpleNamespace(sh=sh, spec=None, codes=None, x=x, wq=wq)
    got = F_._wgrad(ctx, dy, tc=True)
    ops = L.ConvOperands()
    ops.a_f32 = x.data_ptr()
    ws = torch.empty(max(int(lib.mnb_wgrad_scratch_bytes(C.byref(sh))), 4), dtype=torch.uint8, device=DEV)
    want = torch.full_like(wq, float("nan"))
    L.check(lib.mnb_conv2d_wgrad(C.byref(sh), dy.data_ptr(), C.byref(ops), want.data_ptr(), ws.data_ptr(), L.stream()),
            "conv2d_wgrad")
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
