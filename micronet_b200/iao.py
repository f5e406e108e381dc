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


def _consumer_of(producer):
    """F_.Consumer for the conv that freeze_inference linked behind ``producer`` (None without a link)"""
    link = producer.__dict__.get("_post_consumer")
    if link is None:
        return None
    nxt, only = link
    if not nxt._use_frozen() or nxt.quant_inference:
        return None
    aq, wq = nxt.activation_quantizer, nxt.weight_quantizer
    if aq.bits == 32 or wq.bits == 32 or not wq.symmetric:
        return None
    return F_.Consumer(nxt, aq.act_spec(), nxt.__dict__.get("_pre_relu", False), only, tuple(nxt.weight.shape), tuple(nxt.stride),
                       tuple(nxt.padding), tuple(nxt.dilation), nxt.groups, True)


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
        key = tuple(t._version for t in list(self.parameters()) + list(self.buffers()))
        fr = self.__dict__.get("_frozen")
        if fr is None or fr[0] != key:
            weight, bias = make()
            if not self.quant_inference:
                wq, w_int, w_scale = self.weight_quantizer.quantize_weight(weight)
            else:
                wq, w_int, w_scale = weight, None, None
            wq = wq.detach()
            (w_int if w_int is not None else wq)._mnb_pk_cache = {}
            fr = (key, wq, w_int, w_scale, None if bias is None else bias.detach())
            self.__dict__["_frozen"] = fr
        return fr[1:]

    def _use_frozen(self):
        return self.__dict__.get("_frozen_inference", False) and not self.training and not torch.is_grad_enabled()

    def _frozen_forward(self, input, make):
        """eval forward of a frozen module: cached quantized weights, the operand plane its producer may have written
        (F_.handed_plane) and the plane it writes for its own consumer (freeze_inference's ``_post_consumer``)"""
        wq, w_int, w_scale, bias = self._frozen_operands(make)
        plane = F_.handed_plane(self, input)
        aq = self.activation_quantizer
        spec = aq.act_spec() if plane is not None else aq.prepare_activation(input)
        return F_.frozen_conv(input, plane, wq, bias, w_int, w_scale, spec, self.stride, self.padding, self.dilation,
                              self.groups, pre_relu=self.__dict__.get("_pre_relu", False),
                              consumer=_consumer_of(self))

    def forward(self, input):
        if self._use_frozen():
            return self._frozen_forward(input, lambda: (self.weight, self.bias))
        return self._quant_conv(input, self.weight, self.bias)


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
            obs = q.observer
            obs.min_val = torch.min(self.observer_res.min_val, self.observer_shortcut.min_val)
            obs.max_val = torch.max(self.observer_res.max_val, self.observer_shortcut.max_val)
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


def freeze_inference(model, enable=True, handoff=True):
    """Opt-in inference fast path for an IAO-prepared model in eval mode (BASELINE.json configs[4], iao/main.py:511-519):
    * every quant conv folds + quantizes its weights and packs their tensor-core image ONCE (re-done when a parameter or
      buffer is written in place);
    * QuantAdd stops refreshing its observers, which cannot influence an eval forward;
    * an nn.ReLU whose only consumer is the next quant conv of an nn.Sequential is folded into that conv's operand packer,
      and the nn.ReLU behind a residual QuantAdd (``self.act(self.add(res, shortcut))`` blocks) into the add kernel.
    * ``handoff``: producers write the bf16 operand plane of the conv that consumes them (conv epilogue -> next conv of an
      nn.Sequential, QuantAdd -> first conv of the next residual block; mnb_pk_conv_post / mnb_quant_add_pack_fwd), so those
      convs need no separate quantize + pack pass and the Sequential intermediates are never written as fp32.
    Outputs are bit-identical to the un-frozen eval forward; ``enable=False`` restores the modules."""
    for m in model.modules():
        if isinstance(m, (QuantConv2d, QuantLinear, QuantAdd)):
            m.__dict__["_frozen_inference"] = bool(enable)
            m.__dict__.pop("_frozen", None)
            m.__dict__.pop("_pre_relu", None)
            m.__dict__.pop("_fuse_relu", None)
            m.__dict__.pop("_post_consumer", None)
    for m in model.modules():
        saved = m.__dict__.setdefault("_mnb_saved_relus", {})
        for name, relu in list(saved.items()):       # undo an earlier rewrite first
            m._modules[name] = relu
        saved.clear()
        if not enable:
            continue
        if isinstance(m, nn.Sequential):
            kids = [(n, k) for n, k in m.named_children() if not isinstance(k, nn.Identity)]
            for (n0, k0), (n1, k1) in zip(kids, kids[1:]):
                if type(k0) is nn.ReLU and isinstance(k1, QuantConv2d) and not k1.quant_inference:
                    k1.__dict__["_pre_relu"] = True
                    saved[n0] = k0
                    m._modules[n0] = nn.Identity()
        add, act = m._modules.get("add"), m._modules.get("act")
        if isinstance(add, QuantAdd) and type(act) is nn.ReLU:
            add.__dict__["_fuse_relu"] = True
            saved["act"] = act
            m._modules["act"] = nn.Identity()
    if enable and handoff:
        _link_consumers(model)
    return model


def _first_quant_conv(seq):
    kids = [k for k in seq.children() if not isinstance(k, nn.Identity)] if isinstance(seq, nn.Sequential) else []
    return kids[0] if kids and isinstance(kids[0], QuantConv2d) else None


def _link_consumers(model):
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
                    k0.__dict__["_post_consumer"] = (k1, True)
    blocks = [m for m in model.modules() if isinstance(m._modules.get("add"), QuantAdd)
              and _first_quant_conv(m._modules.get("residual_function")) is not None]
    for b0, b1 in zip(blocks, blocks[1:]):
        if b0._modules["add"].__dict__.get("_fuse_relu", False):
            b0._modules["add"].__dict__["_post_consumer"] = (_first_quant_conv(b1._modules["residual_function"]), False)


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
