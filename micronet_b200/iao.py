"""Integer-arithmetic-only (IAO) QAT / PTQ / QAFT modules on the H100 engine.

Drop-in for the reference's ``micronet/compression/quantization/wqaq/iao/quantize.py``:
same class names, constructor signatures (IAO:326-346, 653-676, 998-1012), attribute names,
registered buffers (so reference checkpoints load: IAO:45-60, 182-204, 247-286) and
``prepare`` rules (IAO:1501-1824).  Observers, scale / zero-point updates, fake-quant, the
convolutions and their backward all run as sm_90a kernels with no host synchronisation."""
from __future__ import annotations

import copy

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import frozen_graph as FG
from . import functional as F_


# ********************* observers (IAO:15-139) *********************
def _range_shape(q_level, out_channels):
    if q_level == "L":
        return (1,)
    if q_level == "C":
        return (out_channels, 1, 1, 1)
    if q_level == "FC":
        return (out_channels, 1)
    raise ValueError(f"unknown q_level {q_level!r}")


class ObserverBase(nn.Module):
    kind = 0  # 0 running min/max, 1 EMA min/max, 2 EMA percentile of |x|
    momentum = 0.1
    percentile = 0.0

    def __init__(self, q_level):
        super().__init__()
        self.q_level = q_level

    def _register_range(self, out_channels):
        shape = _range_shape(self.q_level, out_channels)
        self.register_buffer("min_val", torch.zeros(shape, dtype=torch.float32))
        self.register_buffer("max_val", torch.zeros(shape, dtype=torch.float32))

    def observe(self, input, quantizer=None):
        """one kernel: range reduction, running/EMA update of min_val/max_val and, when a
        quantizer is given, its update_qparams (IAO:292-321) in the same launch."""
        L.require_cuda(input, self.min_val)
        lib = L.load()
        x = input.detach().contiguous()
        rows = 1 if self.q_level == "L" else self.min_val.numel()
        first = 1 if self.num_flag == 0 else 0
        if first:
            self.num_flag += 1
        if quantizer is not None:
            quantizer.q_type = 0 if quantizer.symmetric else 1
            args = (1, 1 if quantizer.symmetric else 0, quantizer.qmin, quantizer.qmax,
                    quantizer.scale.data_ptr(), quantizer.zero_point.data_ptr())
        else:
            args = (0, 1, 0, 1, None, None)
        L.check(lib.mnb_iao_observe(x.data_ptr(), x.numel(), rows, self.kind, first, float(self.momentum),
                                    float(self.percentile), self.min_val.data_ptr(), self.max_val.data_ptr(),
                                    *args, L.scratch(x.device).data_ptr(), L.stream()), "iao_observe")

    @torch.no_grad()
    def forward(self, input):
        self.observe(input)


class MinMaxObserver(ObserverBase):
    kind = 0

    def __init__(self, q_level, out_channels):
        super().__init__(q_level)
        self.num_flag = 0
        self.out_channels = out_channels
        self._register_range(out_channels)


class MovingAverageMinMaxObserver(ObserverBase):
    kind = 1

    def __init__(self, q_level, out_channels, momentum=0.1):
        super().__init__(q_level)
        self.momentum = momentum
        self.num_flag = 0
        self.out_channels = out_channels
        self._register_range(out_channels)


class HistogramObserver(ObserverBase):
    """IAO:116-139: EMA of kthvalue(|x|, int(percentile * numel)); min_val is never written."""
    kind = 2

    def __init__(self, q_level, momentum=0.1, percentile=0.9999):
        super().__init__(q_level)
        self.momentum = momentum
        self.percentile = percentile
        self.num_flag = 0
        self.out_channels = None
        self.register_buffer("min_val", torch.zeros((1), dtype=torch.float32))
        self.register_buffer("max_val", torch.zeros((1), dtype=torch.float32))


# ********************* quantizers (IAO:171-321) *********************
class Quantizer(nn.Module):
    symmetric = True

    def __init__(self, bits, observer, activation_weight_flag, qaft=False, union=False):
        super().__init__()
        self.bits = bits
        self.observer = observer
        self.activation_weight_flag = activation_weight_flag
        self.qaft = qaft
        self.union = union
        self.q_type = 0
        shape = _range_shape(observer.q_level, observer.out_channels)
        self.register_buffer("scale", torch.ones(shape, dtype=torch.float32))
        self.register_buffer("zero_point", torch.zeros(shape, dtype=torch.float32))
        self.register_buffer("eps", torch.tensor((torch.finfo(torch.float32).eps), dtype=torch.float32))
        self.qmin, self.qmax = self._level_range()
        self.register_buffer("quant_min_val", torch.tensor((self.qmin), dtype=torch.float32))
        self.register_buffer("quant_max_val", torch.tensor((self.qmax), dtype=torch.float32))

    def _level_range(self):
        raise NotImplementedError

    def _check_bits(self):
        if self.bits == 1:
            print("！Binary quantization is not supported ！")
            assert self.bits != 1
        if self.bits != 32 and not (2 <= self.bits <= 8):
            raise NotImplementedError(f"micronet_b200: IAO bits must be 2..8 or 32 on the CUDA path, got {self.bits}")

    def update_qparams(self):
        """refresh scale / zero_point from the observer's current range (device kernel)."""
        lib = L.load()
        self.q_type = 0 if self.symmetric else 1
        obs = self.observer
        L.check(lib.mnb_iao_update_qparams(obs.min_val.data_ptr(), obs.max_val.data_ptr(), self.scale.numel(),
                                           1 if self.symmetric else 0, self.qmin, self.qmax,
                                           self.scale.data_ptr(), self.zero_point.data_ptr(), L.stream()),
                "iao_update_qparams")

    def refresh(self, input):
        """the training-time side effects of IAO:221-226 (observer + qparams)."""
        if not self.qaft and self.training:
            if not self.union:
                with torch.no_grad():
                    self.observer.observe(input, self)
            else:
                self.update_qparams()

    def act_spec(self):
        obs = self.observer
        return F_.ActSpec(L.ACT_IAO, bits=self.bits, qmin=self.qmin, qmax=self.qmax, q_type=self.q_type,
                          scale=self.scale, zero_point=self.zero_point, obs_min=obs.min_val,
                          obs_max=obs.max_val)

    def prepare_activation(self, input):
        """-> ActSpec for the fused conv (None when bits == 32)."""
        if self.bits == 32:
            return None
        self._check_bits()
        self.refresh(input)
        return self.act_spec()

    def quantize_weight(self, weight):
        """-> (wq, w_int, w_scale); integer operands only for symmetric quantizers."""
        if self.bits == 32:
            return weight, None, None
        self._check_bits()
        self.refresh(weight)
        obs = self.observer
        wq, w_int, w_scale = F_.IaoWeightFn.apply(weight, self.scale, self.zero_point, obs.min_val,
                                                   obs.max_val, self.q_type, self.qmin, self.qmax)
        if not self.symmetric:
            w_int = w_scale = None
        return wq, w_int, w_scale

    def forward(self, input):
        if self.bits == 32:
            return input
        if self.activation_weight_flag == 0 and input.dim() in (2, 4) and self.scale.numel() > 1:
            return self.quantize_weight(input)[0]
        spec = self.prepare_activation(input)
        return F_.ActQuantFn.apply(input, spec)


class SignedQuantizer(Quantizer):
    def _level_range(self):
        if self.bits == 32:
            return 0, 1
        half = 1 << (self.bits - 1)
        if self.activation_weight_flag == 0:
            return -(half - 1), half - 1
        if self.activation_weight_flag == 1:
            return -half, half - 1
        print("activation_weight_flag error")
        return -half, half - 1


class UnsignedQuantizer(Quantizer):
    def _level_range(self):
        if self.bits == 32:
            return 0, 1
        if self.activation_weight_flag == 0:
            return 0, (1 << self.bits) - 2
        if self.activation_weight_flag == 1:
            return 0, (1 << self.bits) - 1
        print("activation_weight_flag error")
        return 0, (1 << self.bits) - 1


class SymmetricQuantizer(SignedQuantizer):
    symmetric = True


class AsymmetricQuantizer(UnsignedQuantizer):
    symmetric = False


def _activation_quantizer(a_bits, q_type, qaft, ptq, percentile, union=False):
    if ptq:  # IAO:450-456 — PTQ always calibrates a symmetric percentile range
        return SymmetricQuantizer(bits=a_bits, observer=HistogramObserver(q_level="L", percentile=percentile),
                                  activation_weight_flag=1, qaft=qaft, union=union)
    cls = SymmetricQuantizer if q_type == 0 else AsymmetricQuantizer
    return cls(bits=a_bits, observer=MovingAverageMinMaxObserver(q_level="L", out_channels=None),
               activation_weight_flag=1, qaft=qaft, union=union)


def _weight_quantizer(w_bits, q_type, q_level, weight_observer, out_channels, qaft, ptq, channel_level="C"):
    obs_cls = MinMaxObserver if weight_observer == 0 else MovingAverageMinMaxObserver
    if q_level == 0:
        observer = obs_cls(q_level=channel_level, out_channels=out_channels)
    else:
        observer = obs_cls(q_level="L", out_channels=None)
    cls = SymmetricQuantizer if (ptq or q_type == 0) else AsymmetricQuantizer
    return cls(bits=w_bits, observer=observer, activation_weight_flag=0, qaft=qaft)


def stored_fake_quant(quantizer, w):
    """the weight fake-quant of the reference's eval forward (IAO:214-240: no observer or qparam update) with the stored
    scale / zero point, in torch ops so that it runs wherever the converter does: (clamp(r, qmin, qmax) + zp) * s with
    r = sign(v) * floor(|v| + 0.5), v = w / s - zp - the op sequence of iao_weight_fwd_kernel and act_quant_fwd_kernel
    (per-channel and per-layer weights).  -> (fake-quantized ``w``, un-clamped levels r)"""
    v = w / quantizer.scale - quantizer.zero_point
    r = torch.sign(v) * torch.floor(v.abs() + 0.5)
    return (r.clamp(quantizer.qmin, quantizer.qmax) + quantizer.zero_point) * quantizer.scale, r


def _holds_levels(conv):
    """does the weight of a ``quant_inference`` conv with a symmetric 2..8-bit weight quantizer hold that quantizer's output
    (bn_fuse.iao_quantize_inference_weights)?  Finite, every level in range, and quantizing it again reproduces it bit for
    bit; raw folded fp32 weights fail the last test."""
    q = conv.weight_quantizer
    if not (conv.quant_inference and _sym_quantizer(q)):
        return False
    w = conv.weight.detach()
    wq, r = stored_fake_quant(q, w)
    return bool(torch.isfinite(w).all()) and bool(((r >= q.qmin) & (r <= q.qmax)).all()) and torch.equal(wq, w)


def _int_weights(conv):
    """does ``conv`` run on integer weights when frozen?  A QAT conv quantizes its own; a ``quant_inference`` conv only when
    freeze_inference found its stored weight to be its quantizer's levels (``_int_levels``, DESIGN.md 4.18)"""
    return not conv.quant_inference or conv.__dict__.get("_int_levels") is not None


_OPEN_RANGE = {}    # device -> (-inf, +inf) observer range of _frozen_spec


def _frozen_spec(conv, spec):
    """the activation spec of a frozen conv's forward and of the epilogue that writes its plane.  A deployment conv with
    levels gets an unbounded observer range in place of its own: the converter does not copy the observer (neither does
    the reference's), so its range is [0, 0], and the range only feeds the STE mask, which no frozen forward reads - but
    the epilogues' level certification (mnb_act_levels) re-derives every level within rounding distance of the range's
    ends exactly, i.e. every zero that a ReLU left, which made the linked convs 2.8x slower (DESIGN.md 4.18).  Levels are
    unchanged: that path only decides how they are computed."""
    if spec is None or conv.__dict__.get("_int_levels") is None:
        return spec
    dev = spec.scale.device
    if dev not in _OPEN_RANGE:
        _OPEN_RANGE[dev] = (torch.full((1,), -float("inf"), device=dev), torch.full((1,), float("inf"), device=dev))
    return F_.ActSpec(spec.mode, spec.bits, spec.qmin, spec.qmax, spec.q_type, spec.scale, spec.zero_point,
                      *_OPEN_RANGE[dev])


def _int8_ok(conv):
    """was ``conv`` frozen with int8=True, with integer weights that fit s8 (symmetric, 2..8 bits)?  Its activation
    quantizer and shape are checked per call (functional._i8_route)."""
    wq = conv.weight_quantizer
    return bool(conv.__dict__.get("_int8", False)) and _int_weights(conv) and wq.symmetric and 2 <= wq.bits <= 8


def _consumer_of(producer):
    """F_.Consumer for the conv that freeze_inference linked behind ``producer`` (None without a link)"""
    link = producer.__dict__.get("_post_consumer")
    if link is None:
        return None
    nxt, only = (link.cconv, True) if isinstance(link, _BlockLink) else link
    if not nxt._use_frozen() or not _int_weights(nxt):
        return None
    aq, wq = nxt.activation_quantizer, nxt.weight_quantizer
    if aq.bits == 32 or wq.bits == 32 or not wq.symmetric:
        return None
    spec = _frozen_spec(nxt, aq.act_spec())
    if isinstance(link, _BlockLink):
        return link.consumer(spec, _int8_ok(nxt))
    return F_.Consumer(nxt, spec, nxt.__dict__.get("_pre_relu", False), only, tuple(nxt.weight.shape), tuple(nxt.stride),
                       tuple(nxt.padding), tuple(nxt.dilation), nxt.groups, True, int8=_int8_ok(nxt))


# ********************* quantized conv / linear *********************
class QuantConv2d(nn.Conv2d):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", a_bits=8, w_bits=8, q_type=0, q_level=0,
                 weight_observer=0, quant_inference=False, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = _activation_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _weight_quantizer(w_bits, q_type, q_level, weight_observer, out_channels,
                                                  qaft, ptq)

    def _quant_conv(self, input, weight, bias):
        spec = self.activation_quantizer.prepare_activation(input)
        if not self.quant_inference:
            wq, w_int, w_scale = self.weight_quantizer.quantize_weight(weight)
        else:
            wq, w_int, w_scale = weight, None, None
        if L.KEEP_DEBUG:   # tests: the fake-quantized weight of this call (tie-excuse rule for BN-fused weights)
            self.__dict__["_dbg_wq"] = wq.detach()
        return F_.quant_conv2d(input, wq, bias, w_int, w_scale, spec, self.stride, self.padding,
                               self.dilation, self.groups)

    def _frozen_operands(self, make):
        """inference fast path (freeze_inference): the quantized weights of an eval-mode module are computed once;
        ``make`` returns (weight to quantize, bias).  Invalidated when any parameter / buffer is written in place."""
        def ops():
            weight, bias = make()
            if not self.quant_inference:
                wq, w_int, w_scale = self.weight_quantizer.quantize_weight(weight)
            elif _int_weights(self):
                wq, w_int, w_scale = self._stored_levels(weight)
            else:
                wq, w_int, w_scale = weight, None, None
            wq = wq.detach()
            (w_int if w_int is not None else wq)._mnb_pk_cache = {}
            return wq, w_int, w_scale, None if bias is None else bias.detach()
        return FG.cached_operands(self, "_frozen", ops)

    def _stored_levels(self, weight):
        """(wq, w_int, w_scale) of a ``quant_inference`` conv whose stored weight freeze_inference accepted as levels: the
        weight quantizer run on it (levels clamped to range), which must give the stored weight back bit for bit.  A weight
        written since with other values is refused: the planes this conv reads and writes assume those levels."""
        wq, w_int, w_scale = self.weight_quantizer.quantize_weight(weight)
        if not (bool(torch.isfinite(weight).all()) and torch.equal(wq, weight)):
            raise RuntimeError(f"micronet_b200: the weight of {self.__dict__['_int_levels']!r} no longer holds its weight "
                               "quantizer's levels; call iao.freeze_inference(model) again")
        return wq, w_int, w_scale

    def _use_frozen(self):
        return self.__dict__.get("_frozen_inference", False) and not self.training and not torch.is_grad_enabled()

    def _in_shuffle(self, x):
        """the channel shuffle of this conv's block that freeze_inference moved into the producer's epilogue, applied here
        when the producer wrote fp32 instead (no plane came, or the module runs un-frozen)"""
        sg = self.__dict__.get("_mnb_in_shuffle", 1)
        return x if sg == 1 else FG.shuffle(F_.materialized(x), sg)

    def _frozen_forward(self, input, make):
        """eval forward of a frozen module: cached quantized weights, the operand plane its producer may have written
        (F_.handed_plane) and the plane it writes for its own consumer (freeze_inference's ``_post_consumer``)"""
        wq, w_int, w_scale, bias = self._frozen_operands(make)
        plane = F_.handed_plane(self, input)
        if plane is None:
            input = self._in_shuffle(input)
        aq = self.activation_quantizer
        spec = _frozen_spec(self, aq.act_spec() if plane is not None else aq.prepare_activation(input))
        return F_.frozen_conv(input, plane, wq, bias, w_int, w_scale, spec, self.stride, self.padding, self.dilation,
                              self.groups, pre_relu=self.__dict__.get("_pre_relu", False),
                              consumer=_consumer_of(self), int8=_int8_ok(self))

    def forward(self, input):
        if self._use_frozen():
            return self._frozen_forward(input, lambda: (self.weight, self.bias))
        return self._quant_conv(self._in_shuffle(input), self.weight, self.bias)


class QuantConvTranspose2d(nn.ConvTranspose2d):
    """IAO:510-636.  Both quantizers observe per layer ("L"), whatever the model-level q_level is (the reference hard-codes
    them); the transposed convolution runs on the engine's convolution kernels with the roles swapped
    (functional.ConvTranspose2dFn)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, groups=1, bias=True,
                 dilation=1, padding_mode="zeros", a_bits=8, w_bits=8, q_type=0, weight_observer=0, quant_inference=False,
                 qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, output_padding, groups, bias, dilation,
                         padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = _activation_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _weight_quantizer(w_bits, q_type, 1, weight_observer, None, qaft, ptq)

    def forward(self, input):
        L.require_cuda(input, self.weight)
        quant_input = self.activation_quantizer(input)
        quant_weight = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F_.conv_transpose2d(quant_input, quant_weight, self.bias, self.stride, self.padding, self.output_padding,
                                   self.groups, self.dilation)


def reshape_to_activation(input):
    return input.reshape(1, -1, 1, 1)


def reshape_to_weight(input):
    return input.reshape(-1, 1, 1, 1)


def reshape_to_bias(input):
    return input.reshape(-1)


class QuantBNFuseConv2d(QuantConv2d):
    """IAO:652-994: BN folded into (w, b) BEFORE quantisation.  Training uses the batch
    statistics of an un-quantised conv of the same input (two convs forward, gradients
    through both); eval / QAFT fold the running statistics."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=False, padding_mode="zeros", eps=1e-5, momentum=0.1, a_bits=8, w_bits=8, q_type=0,
                 q_level=0, weight_observer=0, pretrained_model=False, qaft=False, ptq=False,
                 percentile=0.9999, bn_fuse_calib=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode, a_bits=a_bits, w_bits=w_bits, q_type=q_type, q_level=q_level,
                         weight_observer=weight_observer, quant_inference=False, qaft=qaft, ptq=ptq,
                         percentile=percentile)
        self.num_flag = 0
        self.pretrained_model = pretrained_model
        self.qaft = qaft
        self.bn_fuse_calib = bn_fuse_calib
        self.eps = eps
        self.momentum = momentum
        self.gamma = nn.Parameter(torch.empty(out_channels))
        self.beta = nn.Parameter(torch.empty(out_channels))
        self.register_buffer("running_mean", torch.zeros((out_channels), dtype=torch.float32))
        self.register_buffer("running_var", torch.ones((out_channels), dtype=torch.float32))
        nn.init.uniform_(self.gamma)
        nn.init.zeros_(self.beta)

    def _fold_running(self):
        ratio = self.gamma / torch.sqrt(self.running_var + self.eps)
        if self.bias is not None:
            bias_fused = reshape_to_bias(self.beta + (self.bias - self.running_mean) * ratio)
        else:
            bias_fused = reshape_to_bias(self.beta - self.running_mean * ratio)
        return self.weight * reshape_to_weight(ratio), bias_fused

    def forward(self, input):
        if self._use_frozen():   # eval / running statistics (IAO:903-935), folded and quantized once
            return self._frozen_forward(input, self._fold_running)
        input = self._in_shuffle(input)
        use_batch = (not self.qaft) and self.training
        if use_batch:
            # un-quantised conv only to obtain the BN batch statistics (IAO:843-855)
            pre = F_.quant_conv2d(input, self.weight, self.bias, None, None, None, self.stride, self.padding,
                                  self.dilation, self.groups)
            batch_mean, batch_var = F_.channel_mean_var(pre)
            first = (not self.pretrained_model) and self.num_flag == 0
            if first:
                self.num_flag += 1
            L.check(L.load().mnb_bn_fold_running(self.running_mean.data_ptr(), self.running_var.data_ptr(),
                                                 batch_mean.detach().contiguous().data_ptr(),
                                                 batch_var.detach().contiguous().data_ptr(), self.running_mean.numel(),
                                                 float(self.momentum), 1 if first else 0, L.stream()), "bn_fold_running")
            mean, var = batch_mean, batch_var
        else:
            mean, var = self.running_mean, self.running_var
        if use_batch and self.bn_fuse_calib:
            # calibration variant (IAO:936-945): the weight is folded with the RUNNING variance, the bias with the batch one
            ratio = self.gamma / torch.sqrt(var + self.eps)
            if self.bias is not None:
                bias_fused = reshape_to_bias(self.beta + (self.bias - mean) * ratio)
            else:
                bias_fused = reshape_to_bias(self.beta - mean * ratio)
            weight_fused = self.weight * reshape_to_weight(self.gamma / torch.sqrt(self.running_var + self.eps))
        else:
            weight_fused, bias_fused = F_.BNFoldFn.apply(self.weight, self.bias, self.gamma, self.beta, mean, var, self.eps)
        if use_batch and self.bn_fuse_calib:  # IAO:957-972
            output = self._quant_conv(input, weight_fused, None)
            output = output * reshape_to_activation(
                torch.sqrt(self.running_var + self.eps) / torch.sqrt(batch_var + self.eps))
            return output + reshape_to_activation(bias_fused)
        return self._quant_conv(input, weight_fused, bias_fused)


class QuantLinear(nn.Linear):
    def __init__(self, in_features, out_features, bias=True, a_bits=8, w_bits=8, q_type=0, q_level=0,
                 weight_observer=0, quant_inference=False, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(in_features, out_features, bias)
        self.quant_inference = quant_inference
        self.activation_quantizer = _activation_quantizer(a_bits, q_type, qaft, ptq, percentile)
        self.weight_quantizer = _weight_quantizer(w_bits, q_type, q_level, weight_observer, out_features,
                                                  qaft, ptq, channel_level="FC")

    def forward(self, input):
        spec = self.activation_quantizer.prepare_activation(input)
        if not self.quant_inference:
            wq, w_int, w_scale = self.weight_quantizer.quantize_weight(self.weight)
        else:
            wq, w_int, w_scale = self.weight, None, None
        return F_.quant_linear(input, wq, self.bias, w_int, w_scale, spec)


# ********************* activation-only wrappers (IAO:1160-1498, SURVEY §8 f1) *********************
class _QuantInput:
    def _make_aq(self, a_bits, q_type, qaft, ptq, percentile):
        self.activation_quantizer = _activation_quantizer(a_bits, q_type, qaft, ptq, percentile)


class QuantReLU(nn.ReLU, _QuantInput):
    def __init__(self, inplace=False, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(inplace)
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return F.relu(self.activation_quantizer(input), self.inplace)


class QuantLeakyReLU(nn.LeakyReLU, _QuantInput):
    def __init__(self, negative_slope=0.01, inplace=False, a_bits=8, q_type=0, qaft=False, ptq=False,
                 percentile=0.9999):
        super().__init__(negative_slope, inplace)
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return F.leaky_relu(self.activation_quantizer(input), self.negative_slope, self.inplace)


class QuantSigmoid(nn.Sigmoid, _QuantInput):
    def __init__(self, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__()
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return torch.sigmoid(self.activation_quantizer(input))


class QuantMaxPool2d(nn.MaxPool2d, _QuantInput):
    def __init__(self, kernel_size, stride=None, padding=0, dilation=1, return_indices=False,
                 ceil_mode=False, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(kernel_size, stride, padding, dilation, return_indices, ceil_mode)
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return F.max_pool2d(self.activation_quantizer(input), self.kernel_size, self.stride, self.padding,
                            self.dilation, ceil_mode=self.ceil_mode, return_indices=self.return_indices)


class QuantAvgPool2d(nn.AvgPool2d, _QuantInput):
    def __init__(self, kernel_size, stride=None, padding=0, ceil_mode=False, count_include_pad=True,
                 divisor_override=None, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(kernel_size, stride, padding, ceil_mode, count_include_pad, divisor_override)
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return F.avg_pool2d(self.activation_quantizer(input), self.kernel_size, self.stride, self.padding,
                            self.ceil_mode, self.count_include_pad, self.divisor_override)


class QuantAdaptiveAvgPool2d(nn.AdaptiveAvgPool2d, _QuantInput):
    def __init__(self, output_size, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__(output_size)
        self._make_aq(a_bits, q_type, qaft, ptq, percentile)

    def forward(self, input):
        return F.adaptive_avg_pool2d(self.activation_quantizer(input), self.output_size)


class QuantAdd(nn.Module):
    """IAO:1441-1498: both addends share one (union) range."""

    def __init__(self, a_bits=8, q_type=0, qaft=False, ptq=False, percentile=0.9999):
        super().__init__()
        if not ptq:
            self.observer_res = MovingAverageMinMaxObserver(q_level="L", out_channels=None)
            self.observer_shortcut = MovingAverageMinMaxObserver(q_level="L", out_channels=None)
        else:
            self.observer_res = HistogramObserver(q_level="L", percentile=percentile)
            self.observer_shortcut = HistogramObserver(q_level="L", percentile=percentile)
        self.activation_quantizer = _activation_quantizer(a_bits, q_type, qaft, ptq, percentile, union=True)

    def forward(self, res, shortcut):
        q = self.activation_quantizer
        frozen = self.__dict__.get("_frozen_inference", False) and not self.training
        if not frozen:
            # the reference refreshes the two observers on every call, eval included (IAO:1483-1494); in eval they only
            # feed the STE range of a backward pass, so a frozen inference model (freeze_inference) skips them
            self.observer_res(res)
            self.observer_shortcut(shortcut)
            # in place (the reference rebinds the attributes): a CUDA graph captured here keeps writing the buffers it
            # captured, so a rebinding eager step between replays would leave the module holding a stale range
            obs = q.observer
            with torch.no_grad():
                torch.minimum(self.observer_res.min_val, self.observer_shortcut.min_val, out=obs.min_val)
                torch.maximum(self.observer_res.max_val, self.observer_shortcut.max_val, out=obs.max_val)
        if q.bits == 32:
            return res + shortcut
        q._check_bits()
        q.refresh(res)          # union quantizer: update_qparams only (training, not QAFT)
        relu = bool(frozen and self.__dict__.get("_fuse_relu", False))
        if frozen and not torch.is_grad_enabled():
            return F_.frozen_quant_add(res, shortcut, q.act_spec(), relu, consumer=_consumer_of(self))
        return F_.QuantAddFn.apply(res, shortcut, q.act_spec(), relu)


# ********************* prepare (IAO:1501-1824) *********************
def _is_add(module):
    return type(module).__name__ == "Add"


def _adopt(dst, src):
    dst.weight.data = src.weight
    if src.bias is not None:
        dst.bias.data = src.bias
    return dst


def add_quant_op(module, a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0, bn_fuse=False,
                 bn_fuse_calib=False, quant_inference=False, pretrained_model=False, qaft=False, ptq=False,
                 percentile=0.9999):
    kw = dict(a_bits=a_bits, w_bits=w_bits, q_type=q_type, q_level=q_level, weight_observer=weight_observer,
              bn_fuse=bn_fuse, bn_fuse_calib=bn_fuse_calib, quant_inference=quant_inference,
              pretrained_model=pretrained_model, qaft=qaft, ptq=ptq, percentile=percentile)
    aq = dict(a_bits=a_bits, q_type=q_type, qaft=qaft, ptq=ptq, percentile=percentile)
    wq = dict(w_bits=w_bits, q_level=q_level, weight_observer=weight_observer)
    conv_name_temp = conv_child_temp = None
    for name, child in module.named_children():
        if isinstance(child, nn.Conv2d):
            if bn_fuse:
                conv_name_temp, conv_child_temp = name, child
            else:
                module._modules[name] = _adopt(QuantConv2d(
                    child.in_channels, child.out_channels, child.kernel_size, stride=child.stride,
                    padding=child.padding, dilation=child.dilation, groups=child.groups,
                    bias=child.bias is not None, padding_mode=child.padding_mode,
                    quant_inference=quant_inference, **aq, **wq), child)
        elif isinstance(child, nn.BatchNorm2d):
            if bn_fuse:
                conv = conv_child_temp
                fused = _adopt(QuantBNFuseConv2d(
                    conv.in_channels, conv.out_channels, conv.kernel_size, stride=conv.stride,
                    padding=conv.padding, dilation=conv.dilation, groups=conv.groups,
                    bias=conv.bias is not None, padding_mode=conv.padding_mode, eps=child.eps,
                    momentum=child.momentum, pretrained_model=pretrained_model, bn_fuse_calib=bn_fuse_calib,
                    **aq, **wq), conv)
                fused.gamma.data = child.weight
                fused.beta.data = child.bias
                fused.running_mean.copy_(child.running_mean)
                fused.running_var.copy_(child.running_var)
                module._modules[conv_name_temp] = fused
                module._modules[name] = nn.Identity()
        elif isinstance(child, nn.ConvTranspose2d):   # IAO:1606-1640 (never BN-fused in the reference either)
            module._modules[name] = _adopt(QuantConvTranspose2d(
                child.in_channels, child.out_channels, child.kernel_size, stride=child.stride, padding=child.padding,
                output_padding=child.output_padding, groups=child.groups, bias=child.bias is not None,
                dilation=child.dilation, padding_mode=child.padding_mode, a_bits=a_bits, w_bits=w_bits, q_type=q_type,
                weight_observer=weight_observer, quant_inference=quant_inference, qaft=qaft, ptq=ptq,
                percentile=percentile), child)
        elif isinstance(child, nn.Linear):
            module._modules[name] = _adopt(QuantLinear(
                child.in_features, child.out_features, bias=child.bias is not None,
                quant_inference=quant_inference, **aq, **wq), child)
        # nn.ReLU is deliberately left alone (IAO:1705-1709)
        elif isinstance(child, nn.LeakyReLU):
            module._modules[name] = QuantLeakyReLU(negative_slope=child.negative_slope, inplace=child.inplace, **aq)
        elif isinstance(child, nn.Sigmoid):
            module._modules[name] = QuantSigmoid(**aq)
        elif isinstance(child, nn.MaxPool2d):
            module._modules[name] = QuantMaxPool2d(kernel_size=child.kernel_size, stride=child.stride,
                                                   padding=child.padding, **aq)
        elif isinstance(child, nn.AvgPool2d):
            module._modules[name] = QuantAvgPool2d(kernel_size=child.kernel_size, stride=child.stride,
                                                   padding=child.padding, **aq)
        elif isinstance(child, nn.AdaptiveAvgPool2d):
            module._modules[name] = QuantAdaptiveAvgPool2d(output_size=child.output_size, **aq)
        elif _is_add(child):
            module._modules[name] = QuantAdd(**aq)
        else:
            add_quant_op(child, **kw)


def freeze_inference(model, enable=True, handoff=True, int8=False):
    """Opt-in inference fast path for an IAO-prepared model in eval mode (BASELINE.json configs[4], iao/main.py:511-519):
    * every quant conv folds + quantizes its weights and packs their tensor-core image ONCE (re-done when a parameter or
      buffer is written in place);
    * QuantAdd stops refreshing its observers, which cannot influence an eval forward;
    * an nn.ReLU whose only consumer is the next quant conv of an nn.Sequential is folded into that conv's operand packer,
      and the nn.ReLU behind a residual QuantAdd (``self.act(self.add(res, shortcut))`` blocks) into the add kernel.
    * ``handoff``: producers write the bf16 operand plane of the conv that consumes them (conv epilogue -> next conv of an
      nn.Sequential, QuantAdd -> first conv of the next residual block; mnb_pk_conv_post / mnb_quant_add_pack_fwd), so those
      convs need no separate quantize + pack pass and the Sequential intermediates are never written as fp32.
    * ``int8``: every quant conv with a symmetric activation quantizer (q_type 0) and symmetric weights of 2..8 bits runs
      its forward on int8 operands (s8 x s8 -> s32 wgmma, mnb_pk_i8_conv) where the int8 plan covers its shape; the others
      keep the bf16 path.  Hand-offs then carry the plane format the consumer reads.
    * ``handoff``, NIN / NIN-GC-style graphs (``nn.Sequential`` of conv-bn-relu blocks, nin.py / nin_gc.py, prepared with
      ``bn_fuse=True``): a block (conv, nn.Identity or nothing, nn.ReLU) is linked to the first conv of the next block when
      both convs and any QuantMaxPool2d in between have symmetric (q_type 0) IAO quantizers and the pool is square with
      2 * p <= k in front of a stride-1 conv.  The producer's epilogue applies the ReLU, the next block's channel shuffle and
      the pool's quantizer (the consumer's without a pool) and writes a level plane; the pool max-pools that plane and
      requantizes it to the consumer's levels (mnb_pk_plane_maxpool_requant).  No fp32 activation is written in between.
      A link whose consumer block shuffles its input is taken only where it pays (DESIGN.md 4.16): the shuffled epilogue
      stores one element at a time, so such a link is made only across a pool (whose fake-quant and max-pool passes it
      saves) and only for an int8 plane (1-byte stores); the others write fp32 as before.
      Blocks with a live nn.BatchNorm2d (``bn_fuse=False``) and asymmetric quantizers keep the fp32 path.
    * deployment graphs (``bn_fuse.iao_model_bn_fuse`` -> ``bn_fuse.iao_quantize_inference_weights``): an eval-mode
      ``quant_inference`` conv with a symmetric 2..8-bit weight quantizer whose stored weight is that quantizer's output
      (finite, levels in range, re-quantized bit for bit) runs on those integer levels and links like the QAT conv it came
      from; its logits are bitwise those of the frozen QAT graph (DESIGN.md 4.18).  Any other ``quant_inference`` conv (raw
      folded weights, asymmetric weights) keeps its fp32 weight and is not linked; a later in-place write of a weight that
      no longer verifies raises at the next forward.
    Outputs are bit-identical to the un-frozen eval forward (a deployment graph's: to the frozen QAT graph's);
    ``enable=False`` restores the modules."""
    FG.undo(model, _UNDO)
    if not enable:
        return model
    rw = FG.Rewrite(model, _UNDO)
    for name, m in model.named_modules():
        if isinstance(m, (QuantConv2d, QuantLinear, QuantAdd)):
            rw.set_dict(m, "_frozen_inference", True)
            rw.set_dict(m, "_int8", bool(int8))
            rw.forget(m, "_frozen")
            if isinstance(m, QuantConv2d) and not m.training and _holds_levels(m):
                rw.set_dict(m, "_int_levels", name or type(m).__name__)    # named in the error of a later mismatch
    for m in model.modules():
        if isinstance(m, nn.Sequential):
            kids = [(n, k) for n, k in m.named_children() if not isinstance(k, nn.Identity)]
            for (n0, k0), (n1, k1) in zip(kids, kids[1:]):
                if type(k0) is nn.ReLU and isinstance(k1, QuantConv2d) and _int_weights(k1):
                    rw.set_dict(k1, "_pre_relu", True)
                    rw.set_child(m, n0, nn.Identity())
        add, act = m._modules.get("add"), m._modules.get("act")
        if isinstance(add, QuantAdd) and type(act) is nn.ReLU:
            rw.set_dict(add, "_fuse_relu", True)
            rw.set_child(m, "act", nn.Identity())
    if handoff:
        _link_consumers(model, rw)
        _link_blocks(model, rw)
    return model


_UNDO = "_mnb_iao_undo"


class _BlockLink(FG.Link):
    """frozen_graph.Link of two conv-bn-relu blocks of an IAO graph: the producer applies the ReLU, the consumer block's
    shuffle and the IAO quantizer of the QuantMaxPool2d in between (the consumer's without one).  A shuffled link hands
    over int8 planes only (_shuffled_link_pays)."""

    def consumer(self, spec, int8):
        c = self.cconv
        pool_spec = None if self.pool is None else self.pool[0].activation_quantizer.act_spec()
        return F_.Consumer(c, spec, True, True, tuple(c.weight.shape), tuple(c.stride), tuple(c.padding), tuple(c.dilation),
                           c.groups, True, int8=int8, shuffle_groups=self.sg, pool=self.pool, post_spec=pool_spec,
                           formats=None if self.sg == 1 else ("i8",))


def _shuffled_link_pays(pool, cconv):
    """link a producer to a consumer block that shuffles its input?  The shuffled epilogue stores one level at a time
    (2 bytes scattered per element for a bf16 plane, 1 for int8), where the fp32 path runs the conv with its plain epilogue
    (or pk_gc3_kernel for the narrow grouped 3x3 layers), ATen ReLU, the shuffle copy and the consumer's pack.  Measured on
    an H100 (DESIGN.md 4.16) this pays only when the link also replaces a pool's fake-quant and max-pool passes and the
    plane is int8: so a pool in between and a consumer frozen with int8 operands (the link then hands over int8 planes
    only; in any other format the producer writes fp32)."""
    return pool is not None and _int8_ok(cconv)


def _sym_quantizer(q):
    return isinstance(q, Quantizer) and q.symmetric and 2 <= q.bits <= 8


def _block_conv(conv):
    """can ``conv`` produce or consume a level plane of a block link?  A frozen eval-mode conv with symmetric 2..8-bit IAO
    quantizers and integer weights (_int_weights)"""
    return (isinstance(conv, QuantConv2d) and conv.__dict__.get("_frozen_inference", False) and not conv.training
            and _int_weights(conv) and _sym_quantizer(conv.activation_quantizer)
            and _sym_quantizer(conv.weight_quantizer))


def _conv_relu(blk):
    """(conv, nn.ReLU) of a conv-bn-relu block whose BatchNorm prepare(bn_fuse=True) folded into the conv, else None"""
    bp = FG.block_parts(blk) if hasattr(blk, "channel_shuffle_flag") else None
    if bp is None or len(bp[1]) != 1 or type(bp[1][0]) is not nn.ReLU:
        return None
    return bp[0], bp[1][0]


def _pool_cover(m):
    """(k, s, p) of a QuantMaxPool2d that mnb_pk_plane_maxpool_requant runs, else None"""
    from .fused import _pool_cfg
    if type(m) is not QuantMaxPool2d or m.training or not _sym_quantizer(m.activation_quantizer):
        return None
    return _pool_cfg(m)


def _requant_pool(link, plane, x, k, s, p):
    from . import pk as PK
    q_in = link.pool[0].activation_quantizer.act_spec().struct()
    q_out = link.cconv.activation_quantizer.act_spec().struct()
    return PK.plane_maxpool_requant(plane, *x.shape, k, s, p, q_in, q_out, int8=x._mnb_pk_pre[3] == "i8")


def _no_check(m):
    """absorbed IAO modules run un-frozen in training mode: a producer tags its output only on the frozen eval path"""


def _link_blocks(model, rw):
    """block -> block links of NIN / NIN-GC-style graphs (see freeze_inference)"""
    import functools
    for (conv, relu), pool, cfg, nxt, cconv, _ in FG.block_pairs(model, _conv_relu, _pool_cover):
        if (not (_block_conv(conv) and _block_conv(cconv)) or not hasattr(nxt, "channel_shuffle_flag")
                or (pool is not None and tuple(cconv.stride) != (1, 1))):
            continue
        sg = FG.block_shuffle(nxt)
        if sg > 1 and not _shuffled_link_pays(pool, cconv):
            continue
        link = _BlockLink(cconv, None, relu, sg, None if pool is None else (pool,) + cfg)
        rw.set_dict(conv, "_post_consumer", link)
        rw.override(relu, FG.absorbed_forward, _no_check, relu, link.target)
        if pool is not None:
            rw.override(pool, FG.pool_forward, _no_check, functools.partial(_requant_pool, link), FG.pool_as_usual, pool, link)
        if sg > 1:
            rw.move_shuffle(nxt, cconv, sg)


def _first_quant_conv(seq):
    kids = [k for k in seq.children() if not isinstance(k, nn.Identity)] if isinstance(seq, nn.Sequential) else []
    return kids[0] if kids and isinstance(kids[0], QuantConv2d) else None


def _link_consumers(model, rw):
    """producer -> consumer links of the frozen graph (the consumer's operand plane is then written by the producer):
    * two quant convs that are adjacent in an nn.Sequential (the nn.ReLU between them already folded away): the first
      one's epilogue writes the second one's plane and no fp32 tensor at all - nobody else can read a Sequential's
      intermediate;
    * a residual block's QuantAdd (with its trailing ReLU folded in) -> the first conv of the NEXT block's
      ``residual_function``: the add kernel writes fp32 (next shortcut) and that conv's plane.
    A link is only a hint: the consumer takes the plane only if the tensor it receives is the tagged, unmodified producer
    output (F_.handed_plane), so a wrong guess about the data flow costs a wasted write, never a wrong result."""
    for m in model.modules():
        if isinstance(m, nn.Sequential):
            kids = [k for k in m.children() if not isinstance(k, nn.Identity)]
            for k0, k1 in zip(kids, kids[1:]):
                if isinstance(k0, QuantConv2d) and isinstance(k1, QuantConv2d):
                    rw.set_dict(k0, "_post_consumer", (k1, True))
    blocks = [m for m in model.modules() if isinstance(m._modules.get("add"), QuantAdd)
              and _first_quant_conv(m._modules.get("residual_function")) is not None]
    for b0, b1 in zip(blocks, blocks[1:]):
        if b0._modules["add"].__dict__.get("_fuse_relu", False):
            rw.set_dict(b0._modules["add"], "_post_consumer", (_first_quant_conv(b1._modules["residual_function"]), False))


def prepare(model, inplace=False, a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0, bn_fuse=False,
            bn_fuse_calib=False, quant_inference=False, pretrained_model=False, qaft=False, ptq=False,
            percentile=0.9999, fuse=False):
    """``fuse`` (extension, off by default): engine max-pool kernels and channel-shuffle folding
    (micronet_b200.fused); parameters, state_dict keys and results are unchanged."""
    if not inplace:
        model = copy.deepcopy(model)
    add_quant_op(model, a_bits=a_bits, w_bits=w_bits, q_type=q_type, q_level=q_level,
                 weight_observer=weight_observer, bn_fuse=bn_fuse, bn_fuse_calib=bn_fuse_calib,
                 quant_inference=quant_inference, pretrained_model=pretrained_model, qaft=qaft, ptq=ptq,
                 percentile=percentile)
    if fuse:
        from .fused import fuse_blocks
        fuse_blocks(model)
    return model
