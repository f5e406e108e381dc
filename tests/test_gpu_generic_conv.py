"""The generic implicit-GEMM convolution kernels (mnb_conv_generic.cu) against fp64, through the C ABI, at the geometries
only they serve (tests/generic_conv_cases.py); then the same kernels reached through QuantConv2dFn and ConvTranspose2dFn.

- forward, integer path (u8 codes x int16 levels): bit for bit the exact integer sum, scaled with the kernel's epilogue
  fl(fl(S) * fl(a_scale * w_scale)) + bias; also past 2^31 (DoReFa 8-bit codes 255 against levels 255);
- forward, fp32 path; dgrad; wgrad: element-wise |got - ref64| <= (n + 2) * 2^-24 * (|a| * |w|)64 (+ 2^-24 |bias|), n the
  length of the dot product: a single dropped or misplaced tap breaks it, where a per-tensor relative error would not;
- dgrad with the STE: bit for bit the STE op sequence of mnb_act_ste_one applied to the kernel's own plain result;
- wgrad: the split-K reduction is deterministic, and the flag-predicated variant runs or leaves dwq untouched.

Every output is NaN-filled before a call: an element the kernel leaves unwritten fails the comparison."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as TF
from torch.nn.grad import conv2d_input, conv2d_weight

from tests.generic_conv_cases import CASES, conv_shape, out_hw

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
NAN = float("nan")
F32_01 = float(np.float32(0.1))     # the DoReFa STE multiplies by 0.1 in fp32


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _geom(case):
    B, Cin, H, W, K, (R, S), st, pad, dil, G = case
    P, Q = out_hw(case)
    return dict(B=B, C=Cin, H=H, W=W, K=K, R=R, S=S, P=P, Q=Q, G=G, conv=dict(stride=st, padding=pad, dilation=dil, groups=G))


def assert_within(got, ref, absref, n, what, extra=0, bias=None):
    """|got - ref| <= (n + 2 + extra) * 2^-24 * absref (+ 2^-24 |bias|), element-wise, nothing left NaN"""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan = torch.isnan(got)
    assert not nan.any(), f"{what}: {int(nan.sum())} of {got.numel()} elements left unwritten"
    lim = (n + 2 + extra) * U * absref
    if bias is not None:
        lim = lim + U * bias.double().abs().view(1, -1, 1, 1)
    err = (got - ref).abs()
    bad = err > lim
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {got.numel()} elements outside the bound, first at "
                           f"{bad.nonzero()[0].tolist()}: err {err[bad][0].item():.3e} > {lim[bad][0].item():.3e}")


def _assert_bitwise(got, want, what):
    got = got.detach().cpu()
    nan = torch.isnan(got)
    assert not nan.any(), f"{what}: {int(nan.sum())} of {got.numel()} elements left unwritten"
    diff = got.view(torch.int32) != want.view(torch.int32)
    assert not diff.any(), (f"{what}: {int(diff.sum())} of {got.numel()} elements differ, first at {diff.nonzero()[0].tolist()}:"
                            f" {got[diff][0].item()!r} != {want[diff][0].item()!r}")


# ---------------------------------------------------------------- integer operands of the forward
# name -> (code range, a_offset, zero_point or None, a_scale, weight levels)
VARIANTS = {
    "dorefa4": (16, 0, None, 1.0 / 15, "dorefa4"),
    "dorefa8": (256, 0, None, 1.0 / 255, "dorefa8"),
    "iao_sym": (256, -128, 0.0, 0.0371, "sym127"),
    "iao_asym": (256, 0, -37.0, 0.0213, "sym127"),
}


def _levels(kind, shape, g):
    if kind == "dorefa4":
        return torch.randint(0, 16, shape, generator=g, dtype=torch.int16) * 2 - 15
    if kind == "dorefa8":
        return torch.randint(0, 256, shape, generator=g, dtype=torch.int16) * 2 - 255
    return torch.randint(-127, 128, shape, generator=g, dtype=torch.int16)


class _Act:
    """u8 codes of one variant, on the device, with their ConvOperands fields and their effective integers e on the CPU"""

    def __init__(self, variant, shape, g):
        ncode, self.offset, zp, sc, self.wkind = VARIANTS[variant]
        self.codes = torch.randint(0, ncode, shape, generator=g, dtype=torch.uint8)
        self.zp = None if zp is None else torch.tensor([zp], dtype=torch.float32)
        self.scale = torch.tensor([sc], dtype=torch.float32)
        self.e = self.codes.long() + self.offset + (0 if zp is None else int(zp))
        self.dev = [t.to(DEV) if t is not None else None for t in (self.codes, self.zp, self.scale)]

    def ops(self):
        from micronet_b200 import _lib as L
        codes, zp, sc = self.dev
        return L.ConvOperands(a_codes=codes.data_ptr(), a_offset=self.offset, a_offset_zp=L.ptr(zp), a_scale=sc.data_ptr())

    def dequantized(self):
        """fl(e * a_scale): the kernel's fp32 activation operand"""
        return self.e.float() * self.scale


def _launch_fwd(case, ops):
    from micronet_b200 import _lib as L
    g = _geom(case)
    y = torch.full((g["B"], g["K"], g["P"], g["Q"]), NAN, device=DEV)
    L.check(L.load().mnb_conv2d_fwd(C.byref(conv_shape(case)), C.byref(ops), y.data_ptr(), L.stream()), "conv2d_fwd")
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", CASES)
def test_forward_integer_path_is_exact(name, variant):
    case = CASES[name]
    g, gen = _geom(case), _gen("fwd_int", name, variant)
    act = _Act(variant, (g["B"], g["C"], g["H"], g["W"]), gen)
    w_int = _levels(act.wkind, (g["K"], g["C"] // g["G"], g["R"], g["S"]), gen)
    w_scale = torch.rand(g["K"], generator=gen) * 0.02 + 0.001
    bias = torch.randn(g["K"], generator=gen)
    dev = [t.to(DEV) for t in (w_int, w_scale, bias)]
    ops = act.ops()
    ops.w_int, ops.w_scale, ops.bias = dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr()
    y = _launch_fwd(case, ops)
    # every partial sum is an integer below 2^53: the fp64 convolution of the integers is the exact sum
    s = TF.conv2d(act.e.double(), w_int.double(), None, **g["conv"])
    assert s.abs().max() < 2 ** 31
    want = s.float() * (act.scale * w_scale).view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)
    _assert_bitwise(y, want, f"{name} {variant}")


@pytest.mark.parametrize("act_kind", ["f32", "codes"])
@pytest.mark.parametrize("name", CASES)
def test_forward_fp32_path_within_the_elementwise_bound(name, act_kind):
    """fp32 x fp32, and u8 codes (asymmetric IAO: offset and zero-point) dequantized by the kernel x fp32 weights"""
    from micronet_b200 import _lib as L
    case = CASES[name]
    g, gen = _geom(case), _gen("fwd_f32", name, act_kind)
    shape = (g["B"], g["C"], g["H"], g["W"])
    if act_kind == "f32":
        a = torch.randn(shape, generator=gen)
        a_dev = a.to(DEV)
        ops = L.ConvOperands(a_f32=a_dev.data_ptr())
    else:
        act = _Act("iao_asym", shape, gen)
        a = act.dequantized()
        ops = act.ops()
    w = torch.randn(g["K"], g["C"] // g["G"], g["R"], g["S"], generator=gen) * 0.1
    bias = torch.randn(g["K"], generator=gen)
    w_dev, b_dev = w.to(DEV), bias.to(DEV)
    ops.w_f32, ops.bias = w_dev.data_ptr(), b_dev.data_ptr()
    y = _launch_fwd(case, ops)
    ref = TF.conv2d(a.double(), w.double(), bias.double(), **g["conv"])
    absref = TF.conv2d(a.double().abs(), w.double().abs(), None, **g["conv"])
    assert_within(y, ref, absref, (g["C"] // g["G"]) * g["R"] * g["S"], f"{name} fwd {act_kind}", bias=bias)


# ---------------------------------------------------------------- dgrad
def _ste_spec(kind):
    from micronet_b200 import _lib as L, functional as F_
    if kind == "dorefa8":
        return F_.ActSpec(L.ACT_DOREFA, bits=8)
    mn, mx = torch.tensor([-7.5]), torch.tensor([8.25])
    s = (mx - mn) / 255.0
    zp = torch.sign(mn) * torch.floor((mn / s).abs() + 0.5)
    bufs = {k: v.to(DEV) for k, v in dict(scale=s, zero_point=zp, obs_min=mn, obs_max=mx).items()}
    return F_.ActSpec(L.ACT_IAO, qmin=0, qmax=255, q_type=1, **bufs)


def _mask(bits, shape):
    """the STE pass flags of a u32 bit mask, element i at bit i % 32 of word i / 32"""
    n = math.prod(shape)
    words = bits.cpu().numpy().view(np.uint32)
    idx = np.arange(n)
    return torch.from_numpy(((words[idx >> 5] >> (idx & 31).astype(np.uint32)) & 1).astype(bool)).view(shape)


def _ste(spec, g, mask):
    """mnb_act_ste_one's op sequence in fp32 ATen-CPU ops (which divide, where ATen-CUDA multiplies by a reciprocal)"""
    from micronet_b200 import _lib as L
    if spec.mode == L.ACT_DOREFA:
        s = torch.tensor(1.0 / 255, dtype=torch.float32)
        v = ((g * s) / s) * torch.tensor(0.1, dtype=torch.float32)
    else:
        s = spec.scale.cpu().view(())
        v = (g * s) / s
    return torch.where(mask, v, torch.zeros((), dtype=torch.float32))


def _launch_dgrad(case, dy, wq, bits=None, spec=None):
    from micronet_b200 import _lib as L
    g = _geom(case)
    dx = torch.full((g["B"], g["C"], g["H"], g["W"]), NAN, device=DEV)
    qp = spec.struct() if spec is not None else None
    L.check(L.load().mnb_conv2d_dgrad(C.byref(conv_shape(case)), dy.data_ptr(), wq.data_ptr(), L.ptr(bits),
                                      None if qp is None else C.byref(qp), dx.data_ptr(), L.stream()), "conv2d_dgrad")
    torch.cuda.synchronize()
    return dx


@pytest.mark.parametrize("ste", [None, "dorefa8", "iao_asym"])
@pytest.mark.parametrize("name", CASES)
def test_dgrad_against_fp64_and_the_ste(name, ste):
    from micronet_b200 import functional as F_
    case = CASES[name]
    g, gen = _geom(case), _gen("dgrad", name, ste)
    xshape = (g["B"], g["C"], g["H"], g["W"])
    dy = torch.randn(g["B"], g["K"], g["P"], g["Q"], generator=gen)
    wq = torch.randn(g["K"], g["C"] // g["G"], g["R"], g["S"], generator=gen) * 0.1
    dy_dev, wq_dev = dy.to(DEV), wq.to(DEV)
    dx = _launch_dgrad(case, dy_dev, wq_dev)
    ref = conv2d_input(xshape, wq.double(), dy.double(), **g["conv"])
    absref = conv2d_input(xshape, wq.double().abs(), dy.double().abs(), **g["conv"])
    # (stride 3: input positions no output reads have absref == 0, so the bound holds them to exactly 0)
    assert_within(dx, ref, absref, (g["K"] // g["G"]) * g["R"] * g["S"], f"{name} dgrad")
    if ste is None:
        return
    spec = _ste_spec(ste)
    x = torch.randn(xshape, generator=gen) * 6
    _, bits, _ = F_.act_quant_raw(x.to(DEV), spec, False, True, False)
    mask = _mask(bits, xshape)
    assert 0.05 < mask.float().mean() < 0.95, "the STE mask must have both values"
    dx_ste = _launch_dgrad(case, dy_dev, wq_dev, bits, spec)
    _assert_bitwise(dx_ste, _ste(spec, dx.cpu(), mask), f"{name} dgrad + {ste} STE")


# ---------------------------------------------------------------- wgrad
@pytest.mark.parametrize("act_kind", ["f32", "codes"])
@pytest.mark.parametrize("name", CASES)
def test_wgrad_against_fp64_deterministic_and_conditional(name, act_kind):
    """split-K wgrad on fp32 activations, and on u8 codes (asymmetric IAO), whose reduction multiplies by a_scale"""
    from micronet_b200 import _lib as L
    lib = L.load()
    case = CASES[name]
    g, gen = _geom(case), _gen("wgrad", name, act_kind)
    shape = (g["B"], g["C"], g["H"], g["W"])
    if act_kind == "f32":
        a = torch.randn(shape, generator=gen)
        a_dev = a.to(DEV)
        ops = L.ConvOperands(a_f32=a_dev.data_ptr())
        a64 = a.double()
    else:
        act = _Act("iao_asym", shape, gen)
        ops = act.ops()
        a64 = act.e.double() * act.scale.double()     # exact: the kernel scales the reduced sum of dy * e
    dy = torch.randn(g["B"], g["K"], g["P"], g["Q"], generator=gen)
    dy_dev = dy.to(DEV)
    wshape = (g["K"], g["C"] // g["G"], g["R"], g["S"])
    sh = conv_shape(case)
    ws = torch.empty(max(int(lib.mnb_wgrad_scratch_bytes(C.byref(sh))), 4), dtype=torch.uint8, device=DEV)

    def run(flag=None):
        dw = torch.full(wshape, NAN, device=DEV)
        if flag is None:
            rc = lib.mnb_conv2d_wgrad(C.byref(sh), dy_dev.data_ptr(), C.byref(ops), dw.data_ptr(), ws.data_ptr(), L.stream())
        else:
            f = torch.tensor([flag], dtype=torch.int32, device=DEV)
            rc = lib.mnb_conv2d_wgrad_cond(C.byref(sh), dy_dev.data_ptr(), C.byref(ops), dw.data_ptr(), ws.data_ptr(),
                                           f.data_ptr(), L.stream())
        L.check(rc, "conv2d_wgrad")
        torch.cuda.synchronize()
        return dw.cpu()

    dw = run()
    ref = conv2d_weight(a64, wshape, dy.double(), **g["conv"])
    absref = conv2d_weight(a64.abs(), wshape, dy.double().abs(), **g["conv"])
    assert_within(dw, ref, absref, g["B"] * g["P"] * g["Q"], f"{name} wgrad {act_kind}")
    _assert_bitwise(run(), dw, f"{name} wgrad {act_kind}, second call")          # rank-order reduction
    assert torch.isnan(run(flag=0)).all(), "wgrad_cond with the flag at 0 wrote dwq"
    _assert_bitwise(run(flag=1), dw, f"{name} wgrad_cond {act_kind}")


# ---------------------------------------------------------------- integer sums past 2^31
S32 = {
    "1x1_C33025": (2, 33025, 2, 2, 3, (1, 1), (1, 1), (0, 0), (1, 1), 1),     # 65025 * 33025 < 2^31 - 1
    "1x1_C33026": (2, 33026, 2, 2, 3, (1, 1), (1, 1), (0, 0), (1, 1), 1),     # 65025 * 33026 > 2^31 - 1
    "3x3_C3670": (1, 3670, 3, 3, 3, (3, 3), (1, 1), (1, 1), (1, 1), 1),       # centre: 65025 * 9 * 3670 > 2^31 - 1
}


@pytest.mark.parametrize("name", S32)
def test_integer_sums_past_int32_stay_exact(name):
    """DoReFa 8-bit codes 255 against weight levels +255: the forward's integer sum must not wrap"""
    from micronet_b200 import _lib as L
    case = S32[name]
    g = _geom(case)
    codes = torch.full((g["B"], g["C"], g["H"], g["W"]), 255, dtype=torch.uint8, device=DEV)
    w_int = torch.full((g["K"], g["C"], g["R"], g["S"]), 255, dtype=torch.int16, device=DEV)
    one = torch.ones(g["K"], dtype=torch.float32, device=DEV)
    ops = L.ConvOperands(a_codes=codes.data_ptr(), a_scale=one.data_ptr(), w_int=w_int.data_ptr(), w_scale=one.data_ptr())
    y = _launch_fwd(case, ops)

    def taps(n, p):   # filter rows (columns) of output row (column) p inside the image: 'same' 3x3 or 1x1
        return sum(0 <= p - 1 + r < n for r in range(3)) if g["R"] == 3 else 1

    # exact sums in Python integers, 65025 per in-image tap and channel, rounded once to fp32 (scales 1, no bias)
    want = torch.tensor([[float(np.float32(65025 * g["C"] * taps(g["H"], p) * taps(g["W"], q))) for q in range(g["Q"])]
                         for p in range(g["P"])], dtype=torch.float32).expand(g["B"], g["K"], g["P"], g["Q"])
    if name != "1x1_C33025":
        assert want.max() > 2 ** 31
    _assert_bitwise(y, want.contiguous(), name)


# ---------------------------------------------------------------- through the autograd Functions
# (B, C, H, W, K, R, stride, padding, dilation): shapes the packed-operand family and the round-1 tensor-core kernels refuse
DISPATCH = {
    "dilation2": (2, 32, 12, 12, 48, 3, 1, 2, 2),
    "stride3": (2, 32, 14, 14, 32, 3, 3, 1, 1),
    "s2_odd": (2, 32, 13, 13, 64, 3, 2, 1, 1),
    "pad_wide": (2, 16, 10, 10, 32, 3, 1, 3, 1),
}
SCHEMES = ["dorefa_w8a8", "dorefa_w4a4", "iao_sym", "iao_asym", "wbwtab_ternary", "float"]


def _scheme(scheme, x_shape, K, Cg, R, gen):
    """-> (x, wq, w_int, w_scale, spec, STE factor)"""
    from micronet_b200 import _lib as L, functional as F_
    wshape = (K, Cg, R, R)
    w_scale = torch.rand(K, generator=gen) * 0.02 + 0.001
    x = torch.randn(x_shape, generator=gen) * 4
    spec, factor = None, 1.0
    if scheme.startswith("dorefa"):
        bits = 8 if scheme.endswith("8") else 4
        w_int = torch.randint(0, 2 ** bits, wshape, generator=gen, dtype=torch.int16) * 2 - (2 ** bits - 1)
        spec, factor = F_.ActSpec(L.ACT_DOREFA, bits=bits), F32_01
        x = x * 2.5
    elif scheme == "iao_sym":
        w_int = torch.randint(-127, 128, wshape, generator=gen, dtype=torch.int16)
        bufs = dict(scale=torch.tensor([9.0 / 127.5]), zero_point=torch.zeros(1), obs_min=torch.tensor([-9.0]),
                    obs_max=torch.tensor([7.0]))
        spec = F_.ActSpec(L.ACT_IAO, qmin=-128, qmax=127, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})
    elif scheme == "iao_asym":
        w_int = torch.randint(-127, 128, wshape, generator=gen, dtype=torch.int16)
        spec = _ste_spec("iao_asym")
    elif scheme == "wbwtab_ternary":
        w_int = torch.randint(-1, 2, wshape, generator=gen, dtype=torch.int16)
        x = torch.randint(0, 2, x_shape, generator=gen).float() * 2 - 1
    else:
        wq = torch.randn(wshape, generator=gen) * 0.1
        return x, wq, None, None, None, factor
    return x, w_int.float() * w_scale.view(-1, 1, 1, 1), w_int, w_scale, spec, factor


@pytest.mark.parametrize("scheme", SCHEMES)
@pytest.mark.parametrize("name", DISPATCH)
def test_quant_conv_on_the_generic_kernels(name, scheme):
    """QuantConv2dFn where only the generic kernels have cover: y, dx and dwq against fp64, teacher-forced on the
    engine's activation operand and STE mask (both tested bit for bit elsewhere)"""
    from micronet_b200 import _lib as L, functional as F_
    B, Cin, H, W, K, R, st, pad, dil = DISPATCH[name]
    gen = _gen("dispatch", name, scheme)
    x, wq, w_int, w_scale, spec, factor = _scheme(scheme, (B, Cin, H, W), K, Cin, R, gen)
    bias = torch.randn(K, generator=gen)
    conv = dict(stride=(st, st), padding=(pad, pad), dilation=(dil, dil), groups=1)
    xe, we = x.to(DEV).requires_grad_(True), wq.to(DEV).requires_grad_(True)
    dev = [None if t is None else t.to(DEV) for t in (w_int, w_scale, bias)]
    old = F_.TIMER
    F_.TIMER = F_.KernelTimer()
    try:
        y = F_.quant_conv2d(xe, we, dev[2], dev[0], dev[1], spec, (st, st), (pad, pad), (dil, dil), 1)
        family = y.grad_fn.family
        go = torch.randn(y.shape, generator=gen)
        y.backward(go.to(DEV))
        torch.cuda.synchronize()
        kinds = {k for k, _, _, _ in F_.TIMER.records}
    finally:
        F_.TIMER = old
    L.tc_check()
    assert family in ("generic", "tc"), family
    assert {"fwd", "dgrad", "wgrad"} <= kinds, kinds
    assert not any(k.endswith("_pk") for k in kinds), kinds
    if spec is None:
        xq, mask = x, torch.ones(x.shape, dtype=torch.bool)
    else:
        _, bits, xq = F_.act_quant_raw(x.to(DEV), spec, False, True, True)
        xq, mask = xq.cpu(), _mask(bits, x.shape)
    n_fwd, n_dx, n_dw = Cin * R * R, K * R * R, B * y.shape[2] * y.shape[3]
    x64, w64, go64 = xq.double().requires_grad_(True), wq.double().requires_grad_(True), go.double()
    y64 = TF.conv2d(x64, w64, bias.double(), **conv)
    y64.backward(go64)
    xa, wa = xq.double().abs().requires_grad_(True), wq.double().abs().requires_grad_(True)
    ya = TF.conv2d(xa, wa, None, **conv)
    ya.backward(go64.abs())
    # integer path: the operands' own roundings (xq, wq) and the epilogue's three add up to less than n + 2 of the bound
    assert_within(y, y64.detach(), ya.detach(), n_fwd, f"{name} {scheme} y", bias=bias)
    # the STE: ((g * s) / s) (* 0.1) adds up to three roundings of the masked gradient
    m = mask.double()
    assert_within(xe.grad, x64.grad * factor * m, xa.grad * factor * m, n_dx, f"{name} {scheme} dx", extra=3)
    # codes: the kernel scales the fp32 sum of dy * e once; xq = fl(e * s) is one more rounding
    assert_within(we.grad, w64.grad, wa.grad, n_dw, f"{name} {scheme} dwq", extra=1)


# B, Cin, H, W, Cout, (R, S), stride, padding, output_padding, groups, dilation
TRANSPOSED = {
    "unequal_stride_pad": (2, 12, 7, 9, 20, (3, 4), (2, 3), (1, 2), (1, 2), 1, (1, 1)),
    "dilation_2_1": (2, 16, 6, 5, 12, (3, 3), (1, 1), (2, 1), (0, 0), 1, (2, 1)),
    "groups_cg10": (2, 36, 8, 8, 30, (3, 3), (2, 2), (1, 1), (1, 1), 3, (1, 1)),
}


@pytest.mark.parametrize("name", TRANSPOSED)
def test_conv_transpose_on_the_generic_kernels(name):
    from micronet_b200 import _lib as L, functional as F_
    B, Ci, H, W, Co, (R, S), st, pad, op, G, dil = TRANSPOSED[name]
    gen = _gen("transposed", name)
    x = torch.randn(B, Ci, H, W, generator=gen)
    w = torch.randn(Ci, Co // G, R, S, generator=gen) * 0.2
    bias = torch.randn(Co, generator=gen)
    xe, we, be = (t.to(DEV).requires_grad_(True) for t in (x, w, bias))
    old = F_.TIMER
    F_.TIMER = F_.KernelTimer()
    try:
        y = F_.conv_transpose2d(xe, we, be, st, pad, op, G, dil)
        go = torch.randn(y.shape, generator=gen)
        y.backward(go.to(DEV))
        torch.cuda.synchronize()
        kinds = {k for k, _, _, _ in F_.TIMER.records}
    finally:
        F_.TIMER = old
    L.tc_check()
    assert {"dgrad", "fwd", "wgrad"} <= kinds and not any(k.endswith("_pk") for k in kinds), kinds
    x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, bias))
    y64 = TF.conv_transpose2d(x64, w64, b64, st, pad, op, G, dil)
    y64.backward(go.double())
    xa, wa, ba = (t.double().abs().requires_grad_(True) for t in (x, w, bias))
    ya = TF.conv_transpose2d(xa, wa, None, st, pad, op, G, dil)
    ya.backward(go.double().abs())
    # y = the generic dgrad (Ci / G * R * S products), then + bias in its own pass
    assert_within(y, y64.detach(), ya.detach(), Ci // G * R * S, f"{name} y", bias=bias)
    assert_within(xe.grad, x64.grad, xa.grad, Co // G * R * S, f"{name} dx")
    assert_within(we.grad, w64.grad, wa.grad, B * H * W, f"{name} dw")
    nb = B * y.shape[2] * y.shape[3]
    gabs = go.double().abs().sum(dim=(0, 2, 3))
    assert_within(be.grad.view(1, -1, 1, 1), b64.grad.view(1, -1, 1, 1), gabs.view(1, -1, 1, 1), nb, f"{name} db")
