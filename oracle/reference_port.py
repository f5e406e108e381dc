"""CPU oracle for the micronet fake-quant conv/linear hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in ``micronet_b200/`` may import this file;
only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` execute it, and there only as the
checker (or as the timed CPU baseline), never as the product.

What it is: a from-scratch restatement, in plain fp32 PyTorch-CPU ops, of the
arithmetic the reference performs in

* ``micronet/compression/quantization/wqaq/dorefa/quantize.py``  (alias DF)
* ``micronet/compression/quantization/wbwtab/quantize.py``        (alias WB)
* ``micronet/compression/quantization/wqaq/iao/quantize.py``      (alias IAO)

All arithmetic of the reference lives in a third-party dependency that is not
in the reference tree: PyTorch/ATen (``requirements.txt:1`` ``torch>=1.1.0``,
unpinned).  The oracle therefore uses the very same ATen CPU ops in the same
order (true fp32 division, ``sign*floor(abs+0.5)`` rounding, Sleef ``tanh``,
oneDNN ``conv2d``), so that on this container it is bit-identical to the
reference on every quantity we compare.

Pinning: the reference ships no golden vectors / known-answer tests
(SURVEY.md §4, §8c).  The oracle is pinned against the reference ITSELF,
imported unmodified (a checkout named by ``MICRONET_REFERENCE``) by
``tests/golden/make_golden.py``; the resulting fixtures are committed under
``tests/golden/`` and checked by ``tests/test_oracle_golden.py`` (CPU suite).

Layout of this file (each block cites the reference lines it follows):
  1. rounding primitives                      DF:11-21, IAO:144-168
  2. DoReFa quantizers                        DF:25-73
  3. wbwtab quantizers                        WB:11-149
  4. IAO observers / quantizers               IAO:15-321
  5. module surface (conv / linear / bnfuse)  DF:76-199, WB:152-195,
                                              IAO:325-507, 652-994, 997-1157
  6. IAO activation-only wrappers             IAO:1160-1498
  7. prepare() tree rewriters                 DF:202-323, WB:247-347, IAO:1501-1824
"""
from __future__ import annotations

import copy

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

# --------------------------------------------------------------------------
# 1. rounding primitives
# --------------------------------------------------------------------------


def round_half_away(v: torch.Tensor) -> torch.Tensor:
    """``sign(v) * floor(|v| + 0.5)`` evaluated in fp32 (DF:13-16, IAO:158-159).

    Note the fp32 quirk: ``0.49999997 + 0.5`` rounds to ``1.0`` so the level is
    1, not 0; ``torch.round`` (half-to-even) is NOT equivalent."""
    return torch.sign(v) * torch.floor(torch.abs(v) + 0.5)


class _RoundIdentitySTE(Function):
    """DF:11-21 — forward half-away rounding, backward identity."""

    @staticmethod
    def forward(ctx, v):
        return round_half_away(v)

    @staticmethod
    def backward(ctx, g):
        return g.clone()


class _RoundRangeSTE(Function):
    """IAO:144-168 — same forward; backward zeroes the gradient outside the
    observed range expressed in level units."""

    @staticmethod
    def forward(ctx, v, lo_obs, hi_obs, q_type):
        if q_type == 0:
            hi = torch.max(torch.abs(lo_obs), torch.abs(hi_obs))
            lo = -hi
        else:
            hi, lo = hi_obs, lo_obs
        ctx.save_for_backward(v, lo, hi)
        return round_half_away(v)

    @staticmethod
    def backward(ctx, g):
        v, lo, hi = ctx.saved_tensors
        gi = g.clone()
        gi[v.gt(hi)] = 0
        gi[v.lt(lo)] = 0
        return gi, None, None, None


# --------------------------------------------------------------------------
# 2. DoReFa (DF:25-73)
# --------------------------------------------------------------------------


def dorefa_quantize_activation(x: torch.Tensor, a_bits: int) -> torch.Tensor:
    """DF:36-46.  levels = round(clamp(0.1 x, 0, 1) / s), s = 1/(2^a - 1)."""
    if a_bits == 32:
        return x
    assert a_bits != 1, "binary quantization is not supported by DoReFa"
    s = 1 / float(2**a_bits - 1)
    c = torch.clamp(x * 0.1, 0, 1)
    return _RoundIdentitySTE.apply(c / s) * s


def dorefa_activation_levels(x: torch.Tensor, a_bits: int) -> torch.Tensor:
    """Integer levels (as fp32) of DF:43-45, for bit-exact parity checks."""
    s = 1 / float(2**a_bits - 1)
    return round_half_away(torch.clamp(x * 0.1, 0, 1) / s)


def dorefa_quantize_weight(w: torch.Tensor, w_bits: int) -> torch.Tensor:
    """DF:61-73.  tanh -> /2/max|.| + 0.5 -> round to 2^w-1 levels -> 2q-1."""
    if w_bits == 32:
        return w
    assert w_bits != 1, "binary quantization is not supported by DoReFa"
    s = 1 / float(2**w_bits - 1)
    t = torch.tanh(w)
    o = t / 2 / torch.max(torch.abs(t)) + 0.5
    q = _RoundIdentitySTE.apply(o / s) * s
    return 2 * q - 1


def dorefa_weight_levels(w: torch.Tensor, w_bits: int):
    """(levels k in [0, 2^w-1] as fp32, pre-round value) of DF:68-71."""
    s = 1 / float(2**w_bits - 1)
    t = torch.tanh(w)
    pre = (t / 2 / torch.max(torch.abs(t)) + 0.5) / s
    return round_half_away(pre), pre


# --------------------------------------------------------------------------
# 3. wbwtab (WB:11-149)
# --------------------------------------------------------------------------


class _BinaryActivationFn(Function):
    """WB:11-36 — sign with 0 -> +1; saturate-STE backward."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        y = torch.sign(x)
        y[y == 0] = 1
        return y

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        gi = g.clone()
        gi[x.ge(1.0)] = 0
        gi[x.le(-1.0)] = 0
        return gi


class _SignSTE(Function):
    """WB:40-51 — sign with 0 -> +1, identity backward."""

    @staticmethod
    def forward(ctx, w):
        y = torch.sign(w)
        y[y == 0] = 1
        return y

    @staticmethod
    def backward(ctx, g):
        return g.clone()


class _TernarySTE(Function):
    """WB:55-75 — per-output-channel threshold 0.7*E|w|, levels {-1,0,1}."""

    @staticmethod
    def forward(ctx, w):
        e = torch.mean(torch.abs(w), (3, 2, 1), keepdim=True)
        thr = e * 0.7
        t = torch.sign(torch.sign(w + thr) + torch.sign(w + (-thr)))
        return t, thr

    @staticmethod
    def backward(ctx, g, g_thr):
        return g.clone()


def wb_binarize_activation(x):
    return _BinaryActivationFn.apply(x)


def wb_quantize_weight(w: torch.Tensor, W: int) -> torch.Tensor:
    """WB:118-149.  W==2 mutates ``w.data`` in place (mean-centre over dim 1,
    clamp to [-1,1]; WB:98-102) — that side effect is part of the contract."""
    if W == 2:
        m = w.data.mean(1, keepdim=True)
        w.data.sub_(m)
        w.data.clamp_(-1.0, 1.0)
        alpha = torch.mean(torch.abs(w), (3, 2, 1), keepdim=True)
        return _SignSTE.apply(w) * alpha
    if W == 3:
        keep = w.clone()
        t, thr = _TernarySTE.apply(w)
        mag = torch.abs(keep)
        small = mag.le(thr)
        big = mag.gt(thr)
        mag[small] = 0
        num = torch.sum(mag.clone(), (3, 2, 1), keepdim=True)
        cnt = torch.sum(big, (3, 2, 1), keepdim=True).float()
        return t * (num / cnt)
    return w


class WbActivationQuantizer(nn.Module):
    """WB:79-94 (replaces nn.ReLU in prepared models)."""

    def __init__(self, A=2):
        super().__init__()
        self.A = A
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        return wb_binarize_activation(x) if self.A == 2 else self.relu(x)


# --------------------------------------------------------------------------
# 4. IAO observers and quantizers (IAO:15-321)
# --------------------------------------------------------------------------


def _obs_shape(level, channels):
    return {"L": (1,), "C": (channels, 1, 1, 1), "FC": (channels, 1)}[level]


class RangeObserver(nn.Module):
    """IAO:15-113.  ``ema=False`` -> MinMaxObserver (running extremum),
    ``ema=True`` -> MovingAverageMinMaxObserver."""

    def __init__(self, q_level, out_channels, ema, momentum=0.1):
        super().__init__()
        self.q_level, self.out_channels = q_level, out_channels
        self.ema, self.momentum = ema, momentum
        self.num_flag = 0
        shape = _obs_shape(q_level, out_channels)
        self.register_buffer("min_val", torch.zeros(shape, dtype=torch.float32))
        self.register_buffer("max_val", torch.zeros(shape, dtype=torch.float32))

    @torch.no_grad()
    def forward(self, x):
        if self.q_level == "L":
            lo, hi = torch.min(x), torch.max(x)
        elif self.q_level == "C":
            flat = torch.flatten(x, start_dim=1)
            lo = torch.min(flat, 1)[0].reshape(self.min_val.shape)
            hi = torch.max(flat, 1)[0].reshape(self.max_val.shape)
        else:
            lo = torch.min(x, 1, keepdim=True)[0]
            hi = torch.max(x, 1, keepdim=True)[0]
        if self.num_flag == 0:
            self.num_flag += 1
        elif self.ema:
            lo = (1 - self.momentum) * self.min_val + self.momentum * lo
            hi = (1 - self.momentum) * self.max_val + self.momentum * hi
        else:
            lo = torch.min(lo, self.min_val)
            hi = torch.max(hi, self.max_val)
        self.min_val.copy_(lo)
        self.max_val.copy_(hi)


class PercentileObserver(nn.Module):
    """IAO:116-139 ("HistogramObserver"): EMA of the k-th smallest |x|,
    k = int(percentile * numel).  ``min_val`` is never written."""

    def __init__(self, q_level="L", momentum=0.1, percentile=0.9999):
        super().__init__()
        self.q_level, self.momentum, self.percentile = q_level, momentum, percentile
        self.num_flag = 0
        self.out_channels = None
        self.register_buffer("min_val", torch.zeros((1), dtype=torch.float32))
        self.register_buffer("max_val", torch.zeros((1), dtype=torch.float32))

    @torch.no_grad()
    def forward(self, x):
        flat = x.abs().view(-1)
        cur = torch.kthvalue(flat, int(self.percentile * flat.size(0)), dim=0)[0]
        if self.num_flag == 0:
            self.num_flag += 1
            new = cur
        else:
            new = (1 - self.momentum) * self.max_val + self.momentum * cur
        self.max_val.copy_(new)


class FakeQuantizer(nn.Module):
    """IAO:171-321.  ``symmetric`` picks Signed+Symmetric vs Unsigned+Asymmetric;
    ``is_activation`` picks the level range (IAO:243-288)."""

    def __init__(self, bits, observer, is_activation, symmetric, qaft=False, union=False):
        super().__init__()
        self.bits, self.observer = bits, observer
        self.activation_weight_flag = 1 if is_activation else 0
        self.symmetric, self.qaft, self.union = symmetric, qaft, union
        self.q_type = 0
        shape = _obs_shape(observer.q_level, observer.out_channels)
        self.register_buffer("scale", torch.ones(shape, dtype=torch.float32))
        self.register_buffer("zero_point", torch.zeros(shape, dtype=torch.float32))
        self.register_buffer(
            "eps", torch.tensor(torch.finfo(torch.float32).eps, dtype=torch.float32)
        )
        if symmetric:
            half = 1 << (bits - 1)
            lo, hi = (-half, half - 1) if is_activation else (-(half - 1), half - 1)
        else:
            lo, hi = (0, (1 << bits) - 1) if is_activation else (0, (1 << bits) - 2)
        self.register_buffer("quant_min_val", torch.tensor(lo, dtype=torch.float32))
        self.register_buffer("quant_max_val", torch.tensor(hi, dtype=torch.float32))

    def update_qparams(self):
        span = float(self.quant_max_val - self.quant_min_val)
        if self.symmetric:  # IAO:292-305
            self.q_type = 0
            fr = torch.max(torch.abs(self.observer.min_val), torch.abs(self.observer.max_val))
            s = torch.max(fr / (span / 2), self.eps)
            zp = torch.zeros_like(s)
        else:  # IAO:309-321
            self.q_type = 1
            fr = self.observer.max_val - self.observer.min_val
            s = torch.max(fr / span, self.eps)
            zp = torch.sign(self.observer.min_val) * torch.floor(
                torch.abs(self.observer.min_val / s) + 0.5
            )
        self.scale.copy_(s)
        self.zero_point.copy_(zp)

    def levels(self, x):
        """clamped integer levels (fp32) for parity checks; no state change."""
        v = x / self.scale - self.zero_point
        return torch.clamp(round_half_away(v), self.quant_min_val, self.quant_max_val)

    def forward(self, x):  # IAO:214-240
        if self.bits == 32:
            return x
        assert self.bits != 1, "binary quantization is not supported by IAO"
        if not self.qaft and self.training:
            if not self.union:
                self.observer(x)
            self.update_qparams()
        r = _RoundRangeSTE.apply(
            x / self.scale.clone() - self.zero_point,
            self.observer.min_val / self.scale - self.zero_point,
            self.observer.max_val / self.scale - self.zero_point,
            self.q_type,
        )
        return (torch.clamp(r, self.quant_min_val, self.quant_max_val) + self.zero_point) * self.scale.clone()


def _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile, union=False):
    if ptq:  # IAO:450-456
        return FakeQuantizer(a_bits, PercentileObserver("L", percentile=percentile), True, True, qaft, union)
    return FakeQuantizer(a_bits, RangeObserver("L", None, ema=True), True, q_type == 0, qaft, union)


def _iao_weight_quantizer(w_bits, q_type, q_level, weight_observer, out_channels, qaft, ptq, fc=False):
    level = ("FC" if fc else "C") if q_level == 0 else "L"
    obs = RangeObserver(level, out_channels if q_level == 0 else None, ema=(weight_observer != 0))
    return FakeQuantizer(w_bits, obs, False, True if ptq else (q_type == 0), qaft)


# --------------------------------------------------------------------------
# 5. module surface
# --------------------------------------------------------------------------


class DorefaQuantConv2d(nn.Conv2d):
    """DF:76-122."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, padding_mode="zeros", a_bits=8, w_bits=8, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, padding_mode)
        self.a_bits, self.w_bits, self.quant_inference = a_bits, w_bits, quant_inference

    def forward(self, x):
        qx = dorefa_quantize_activation(x, self.a_bits)
        qw = self.weight if self.quant_inference else dorefa_quantize_weight(self.weight, self.w_bits)
        return F.conv2d(qx, qw, self.bias, self.stride, self.padding, self.dilation, self.groups)


class DorefaQuantLinear(nn.Linear):
    """DF:177-199."""

    def __init__(self, in_features, out_features, bias=True, a_bits=8, w_bits=8, quant_inference=False):
        super().__init__(in_features, out_features, bias)
        self.a_bits, self.w_bits, self.quant_inference = a_bits, w_bits, quant_inference

    def forward(self, x):
        qx = dorefa_quantize_activation(x, self.a_bits)
        qw = self.weight if self.quant_inference else dorefa_quantize_weight(self.weight, self.w_bits)
        return F.linear(qx, qw, self.bias)


class WbQuantConv2d(nn.Conv2d):
    """WB:152-195 — only the weight is quantized here."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, padding_mode="zeros", W=2, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, padding_mode)
        self.W, self.quant_inference = W, quant_inference

    def forward(self, x):
        qw = self.weight if self.quant_inference else wb_quantize_weight(self.weight, self.W)
        return F.conv2d(x, qw, self.bias, self.stride, self.padding, self.dilation, self.groups)


class IaoQuantConv2d(nn.Conv2d):
    """IAO:325-507."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=True, padding_mode="zeros", a_bits=8, w_bits=8, q_type=0, q_level=0,
                 weight_observer=0, quant_inference=False, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _iao_weight_quantizer(w_bits, q_type, q_level, weight_observer, out_channels, qaft, ptq)

    def forward(self, x):
        qx = self.activation_quantizer(x)
        qw = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F.conv2d(qx, qw, self.bias, self.stride, self.padding, self.dilation, self.groups)


class IaoQuantConvTranspose2d(nn.ConvTranspose2d):
    """IAO:510-636: per-layer ("L") observers for both operands whatever q_level says (the reference hard-codes them)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, groups=1,
                 bias=True, dilation=1, padding_mode="zeros", a_bits=8, w_bits=8, q_type=0, weight_observer=0,
                 quant_inference=False, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, output_padding, groups, bias, dilation,
                         padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _iao_weight_quantizer(w_bits, q_type, 1, weight_observer, None, qaft, ptq)

    def forward(self, x):
        qx = self.activation_quantizer(x)
        qw = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F.conv_transpose2d(qx, qw, self.bias, self.stride, self.padding, self.output_padding, self.groups,
                                  self.dilation)


class IaoQuantBNFuseConv2d(IaoQuantConv2d):
    """IAO:652-994."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                 groups=1, bias=False, padding_mode="zeros", eps=1e-5, momentum=0.1, a_bits=8, w_bits=8,
                 q_type=0, q_level=0, weight_observer=0, pretrained_model=False, qaft=False, ptq=False,
                 percentile=0.9999, bn_fuse_calib=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode, a_bits=a_bits, w_bits=w_bits, q_type=q_type, q_level=q_level,
                         weight_observer=weight_observer, qaft=qaft, ptq=ptq, percentile=percentile)
        self.num_flag = 0
        self.pretrained_model, self.qaft, self.bn_fuse_calib = pretrained_model, qaft, bn_fuse_calib
        self.eps, self.momentum = eps, momentum
        self.gamma = nn.Parameter(torch.empty(out_channels).uniform_())
        self.beta = nn.Parameter(torch.zeros(out_channels))
        self.register_buffer("running_mean", torch.zeros(out_channels, dtype=torch.float32))
        self.register_buffer("running_var", torch.ones(out_channels, dtype=torch.float32))

    def _conv(self, x, w, b):
        return F.conv2d(x, w, b, self.stride, self.padding, self.dilation, self.groups)

    def forward(self, x):
        use_batch = (not self.qaft) and self.training
        if use_batch:  # IAO:843-901
            pre = self._conv(x, self.weight, self.bias)
            b_mean = torch.mean(pre, dim=[0, 2, 3])
            b_var = torch.var(pre, dim=[0, 2, 3])  # unbiased
            with torch.no_grad():
                if (not self.pretrained_model) and self.num_flag == 0:
                    self.num_flag += 1
                    r_mean, r_var = b_mean, b_var
                else:
                    r_mean = (1 - self.momentum) * self.running_mean + self.momentum * b_mean
                    r_var = (1 - self.momentum) * self.running_var + self.momentum * b_var
                self.running_mean.copy_(r_mean)
                self.running_var.copy_(r_var)
            mean, var = b_mean, b_var
        else:  # IAO:903-935
            mean, var = self.running_mean, self.running_var
        g = self.gamma / torch.sqrt(var + self.eps)
        if self.bias is not None:
            b_fused = (self.beta + (self.bias - mean) * g).reshape(-1)
        else:
            b_fused = (self.beta - mean * g).reshape(-1)
        if use_batch and self.bn_fuse_calib:
            w_fused = self.weight * (self.gamma / torch.sqrt(self.running_var + self.eps)).reshape(-1, 1, 1, 1)
        else:
            w_fused = self.weight * g.reshape(-1, 1, 1, 1)
        qx = self.activation_quantizer(x)
        qw = self.weight_quantizer(w_fused)
        if use_batch and self.bn_fuse_calib:  # IAO:957-972
            y = self._conv(qx, qw, None)
            y *= (torch.sqrt(self.running_var + self.eps) / torch.sqrt(b_var + self.eps)).reshape(1, -1, 1, 1)
            y += b_fused.reshape(1, -1, 1, 1)
            return y
        return self._conv(qx, qw, b_fused)


class IaoQuantLinear(nn.Linear):
    """IAO:997-1157."""

    def __init__(self, in_features, out_features, bias=True, a_bits=8, w_bits=8, q_type=0, q_level=0,
                 weight_observer=0, quant_inference=False, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_features, out_features, bias)
        self.quant_inference = quant_inference
        self.activation_quantizer = _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _iao_weight_quantizer(
            w_bits, q_type, q_level, weight_observer, out_features, qaft, ptq, fc=True)

    def forward(self, x):
        qx = self.activation_quantizer(x)
        qw = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F.linear(qx, qw, self.bias)


# --------------------------------------------------------------------------
# 6. IAO activation-only wrappers (IAO:1160-1498) — §8(f1) "next" row
# --------------------------------------------------------------------------


class IaoQuantThenOp(nn.Module):
    """quantize the input, then apply ``op`` (ReLU / LeakyReLU / Sigmoid / pools)."""

    def __init__(self, op, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__()
        self.op = op
        self.activation_quantizer = _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, x):
        return self.op(self.activation_quantizer(x))


class IaoQuantAdd(nn.Module):
    """IAO:1441-1498 — shared (union) range for the two addends."""

    def __init__(self, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__()
        if ptq:
            self.observer_res = PercentileObserver("L", percentile=percentile)
            self.observer_shortcut = PercentileObserver("L", percentile=percentile)
        else:
            self.observer_res = RangeObserver("L", None, ema=True)
            self.observer_shortcut = RangeObserver("L", None, ema=True)
        self.activation_quantizer = _iao_act_quantizer(a_bits, q_type, qaft, ptq, percentile, union=True)

    def forward(self, res, shortcut):
        self.observer_res(res)
        self.observer_shortcut(shortcut)
        q = self.activation_quantizer
        q.observer.min_val = torch.min(self.observer_res.min_val, self.observer_shortcut.min_val)
        q.observer.max_val = torch.max(self.observer_res.max_val, self.observer_shortcut.max_val)
        return q(res) + q(shortcut)


# --------------------------------------------------------------------------
# 7. prepare() (DF:202-323, WB:247-347, IAO:1501-1824)
# --------------------------------------------------------------------------


def _conv_kwargs(c):
    return dict(stride=c.stride, padding=c.padding, dilation=c.dilation, groups=c.groups,
                bias=c.bias is not None, padding_mode=c.padding_mode)


def _adopt(dst, src):
    dst.weight.data = src.weight
    if src.bias is not None:
        dst.bias.data = src.bias
    return dst


def prepare_dorefa(model, inplace=False, a_bits=8, w_bits=8, quant_inference=False):
    model = model if inplace else copy.deepcopy(model)
    seen = [0]

    def walk(mod):
        for name, ch in mod.named_children():
            if isinstance(ch, nn.Conv2d):
                seen[0] += 1
                if seen[0] > 1:
                    mod._modules[name] = _adopt(DorefaQuantConv2d(
                        ch.in_channels, ch.out_channels, ch.kernel_size, a_bits=a_bits, w_bits=w_bits,
                        quant_inference=quant_inference, **_conv_kwargs(ch)), ch)
            elif isinstance(ch, nn.Linear):
                seen[0] += 1
                if seen[0] > 1:
                    mod._modules[name] = _adopt(DorefaQuantLinear(
                        ch.in_features, ch.out_features, bias=ch.bias is not None, a_bits=a_bits,
                        w_bits=w_bits, quant_inference=quant_inference), ch)
            else:
                walk(ch)

    walk(model)
    return model


def prepare_wbwtab(model, inplace=False, A=2, W=2, quant_inference=False):
    model = model if inplace else copy.deepcopy(model)
    total = sum(isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)) for m in model.modules())
    seen = [0]

    def walk(mod):
        for name, ch in mod.named_children():
            if isinstance(ch, nn.Conv2d):
                seen[0] += 1
                if 1 < seen[0] < total:
                    mod._modules[name] = _adopt(WbQuantConv2d(
                        ch.in_channels, ch.out_channels, ch.kernel_size, W=W,
                        quant_inference=quant_inference, **_conv_kwargs(ch)), ch)
            elif isinstance(ch, nn.ReLU):
                if 0 < seen[0] < total:
                    mod._modules[name] = WbActivationQuantizer(A=A)
            else:
                walk(ch)

    walk(model)
    return model


def prepare_iao(model, inplace=False, a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0,
                bn_fuse=False, bn_fuse_calib=False, quant_inference=False, pretrained_model=False,
                qaft=False, ptq=False, percentile=0.9999, add_type=None):
    """``add_type``: the residual-add module class of the model zoo in use
    (the reference hard-codes ``micronet.base_module.op.Add``, IAO:1760)."""
    model = model if inplace else copy.deepcopy(model)
    qa = dict(a_bits=a_bits, q_type=q_type, qaft=qaft, ptq=ptq, percentile=percentile)
    qw = dict(w_bits=w_bits, q_level=q_level, weight_observer=weight_observer)

    def walk(mod):
        pending = None
        for name, ch in mod.named_children():
            if isinstance(ch, nn.Conv2d):
                if bn_fuse:
                    pending = (name, ch)
                else:
                    mod._modules[name] = _adopt(IaoQuantConv2d(
                        ch.in_channels, ch.out_channels, ch.kernel_size, quant_inference=quant_inference,
                        **_conv_kwargs(ch), **qa, **qw), ch)
            elif isinstance(ch, nn.BatchNorm2d):
                if bn_fuse:
                    cname, conv = pending
                    fused = _adopt(IaoQuantBNFuseConv2d(
                        conv.in_channels, conv.out_channels, conv.kernel_size, eps=ch.eps,
                        momentum=ch.momentum, pretrained_model=pretrained_model,
                        bn_fuse_calib=bn_fuse_calib, **_conv_kwargs(conv), **qa, **qw), conv)
                    fused.gamma.data = ch.weight
                    fused.beta.data = ch.bias
                    fused.running_mean.copy_(ch.running_mean)
                    fused.running_var.copy_(ch.running_var)
                    mod._modules[cname] = fused
                    mod._modules[name] = nn.Identity()
            elif isinstance(ch, nn.Linear):
                mod._modules[name] = _adopt(IaoQuantLinear(
                    ch.in_features, ch.out_features, bias=ch.bias is not None,
                    quant_inference=quant_inference, **qa, **qw), ch)
            elif isinstance(ch, (nn.LeakyReLU, nn.Sigmoid, nn.MaxPool2d, nn.AvgPool2d, nn.AdaptiveAvgPool2d)):
                mod._modules[name] = IaoQuantThenOp(copy.deepcopy(ch), **qa)
            elif add_type is not None and isinstance(ch, add_type):
                mod._modules[name] = IaoQuantAdd(**qa)
            else:
                walk(ch)

    walk(model)
    return model
