"""Fused wgmma forward conv (mnb_fq_conv2d_fwd_tc) against the generic kernels, the standalone
quantizer kernel (codes / STE bits must be identical) and ATen-CPU conv2d.

The "tc" leg turns the packed-operand family off (L.PK_MODE = "off"): with a quantizer spec QuantConv2dFn would otherwise
take that family first, whatever USE_TC says.  Inside the documented cover (DESIGN.md §4.1/§4.2) the leg must have run
fwd_tc / dgrad_tc / wgrad_tc; the shapes instantiate every group width 16..160 of conv_tc_kernel, forward (K/g) and data
gradient (C/g)."""
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
