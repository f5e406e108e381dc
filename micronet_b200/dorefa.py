"""DoReFa k-bit QAT modules on the H100 engine.

Drop-in for the reference's ``micronet/compression/quantization/wqaq/dorefa/quantize.py``:
same class names, constructor signatures (DF:77-91, DF:178-186), attribute names and
``prepare`` rules (DF:202-323).  The quantizers are stateless, so ``state_dict`` holds only
``weight`` / ``bias`` exactly like the reference."""
from __future__ import annotations

import copy

import torch.nn as nn

from . import _lib as L
from . import functional as F_


class ActivationQuantizer(nn.Module):
    """DF:25-46: clamp(0.1 x, 0, 1) quantized to 2^a - 1 levels."""

    def __init__(self, a_bits):
        super().__init__()
        self.a_bits = a_bits

    def spec(self):
        if self.a_bits == 32:
            return None
        if self.a_bits == 1:
            print("！Binary quantization is not supported ！")
            assert self.a_bits != 1
        return F_.ActSpec(L.ACT_DOREFA, bits=self.a_bits)

    def forward(self, input):
        spec = self.spec()
        return input if spec is None else F_.ActQuantFn.apply(input, spec)


class WeightQuantizer(nn.Module):
    """DF:50-73: tanh -> normalise by the global max -> 2^w - 1 levels -> [-1, 1]."""

    def __init__(self, w_bits):
        super().__init__()
        self.w_bits = w_bits

    def quantize(self, weight):
        """(wq, w_int, w_scale); w_int/w_scale are None when the weight is passed through."""
        if self.w_bits == 32:
            return weight, None, None
        if self.w_bits == 1:
            print("！Binary quantization is not supported ！")
            assert self.w_bits != 1
        return F_.DorefaWeightFn.apply(weight, self.w_bits)

    def forward(self, input):
        return self.quantize(input)[0]


class QuantConv2d(nn.Conv2d):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", a_bits=8, w_bits=8, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = ActivationQuantizer(a_bits=a_bits)
        self.weight_quantizer = WeightQuantizer(w_bits=w_bits)

    def forward(self, input):
        spec = self.activation_quantizer.spec()
        if not self.quant_inference:
            wq, w_int, w_scale = self.weight_quantizer.quantize(self.weight)
        else:
            wq, w_int, w_scale = self.weight, None, None
        # padding_mode is accepted but, as in the reference (DF:113-121), padding is always zeros
        return F_.quant_conv2d(input, wq, self.bias, w_int, w_scale, spec, self.stride, self.padding,
                               self.dilation, self.groups)


class QuantConvTranspose2d(nn.ConvTranspose2d):
    """DF:125-174.  The reference hands (dilation, groups, bias) POSITIONALLY to ``nn.ConvTranspose2d.__init__``, whose order is
    (groups, bias, dilation): with current PyTorch its forward raises ``TypeError`` (dilation = (True, True)), so there is no
    reference behaviour to reproduce beyond the intent - activation quantizer, weight quantizer, ``F.conv_transpose2d`` - which
    is what this module does, with the constructor arguments taken by name.  The transposed convolution runs on the engine's
    convolution kernels with the roles swapped (functional.ConvTranspose2dFn)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", a_bits=8, w_bits=8, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                         output_padding=output_padding, groups=groups, bias=bias, dilation=dilation,
                         padding_mode=padding_mode)
        self.quant_inference = quant_inference
        self.activation_quantizer = ActivationQuantizer(a_bits=a_bits)
        self.weight_quantizer = WeightQuantizer(w_bits=w_bits)

    def forward(self, input):
        L.require_cuda(input, self.weight)
        quant_input = self.activation_quantizer(input)
        quant_weight = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F_.conv_transpose2d(quant_input, quant_weight, self.bias, self.stride, self.padding, self.output_padding,
                                   self.groups, self.dilation)


class QuantLinear(nn.Linear):
    def __init__(self, in_features, out_features, bias=True, a_bits=8, w_bits=8, quant_inference=False):
        super().__init__(in_features, out_features, bias)
        self.quant_inference = quant_inference
        self.activation_quantizer = ActivationQuantizer(a_bits=a_bits)
        self.weight_quantizer = WeightQuantizer(w_bits=w_bits)

    def forward(self, input):
        spec = self.activation_quantizer.spec()
        if not self.quant_inference:
            wq, w_int, w_scale = self.weight_quantizer.quantize(self.weight)
        else:
            wq, w_int, w_scale = self.weight, None, None
        return F_.quant_linear(input, wq, self.bias, w_int, w_scale, spec)


def _adopt(dst, src):
    dst.weight.data = src.weight
    if src.bias is not None:
        dst.bias.data = src.bias
    return dst


def add_quant_op(module, layer_counter, a_bits=8, w_bits=8, quant_inference=False):
    """DF:202-309: every conv / linear except the first one becomes a quant module."""
    for name, child in module.named_children():
        if isinstance(child, nn.Conv2d):
            layer_counter[0] += 1
            if layer_counter[0] > 1:
                module._modules[name] = _adopt(QuantConv2d(
                    child.in_channels, child.out_channels, child.kernel_size, stride=child.stride,
                    padding=child.padding, dilation=child.dilation, groups=child.groups,
                    bias=child.bias is not None, padding_mode=child.padding_mode, a_bits=a_bits,
                    w_bits=w_bits, quant_inference=quant_inference), child)
        elif isinstance(child, nn.ConvTranspose2d):
            layer_counter[0] += 1
            if layer_counter[0] > 1:     # DF:236-277
                module._modules[name] = _adopt(QuantConvTranspose2d(
                    child.in_channels, child.out_channels, child.kernel_size, stride=child.stride,
                    padding=child.padding, output_padding=child.output_padding, dilation=child.dilation,
                    groups=child.groups, bias=child.bias is not None, padding_mode=child.padding_mode, a_bits=a_bits,
                    w_bits=w_bits, quant_inference=quant_inference), child)
        elif isinstance(child, nn.Linear):
            layer_counter[0] += 1
            if layer_counter[0] > 1:
                module._modules[name] = _adopt(QuantLinear(
                    child.in_features, child.out_features, bias=child.bias is not None, a_bits=a_bits,
                    w_bits=w_bits, quant_inference=quant_inference), child)
        else:
            add_quant_op(child, layer_counter, a_bits=a_bits, w_bits=w_bits, quant_inference=quant_inference)


def prepare(model, inplace=False, a_bits=8, w_bits=8, quant_inference=False, fuse=False):
    """``fuse`` (extension, off by default): engine max-pool kernels and channel-shuffle folding around the
    quantized convolutions (micronet_b200.fused); parameters, state_dict keys and results are unchanged."""
    if not inplace:
        model = copy.deepcopy(model)
    add_quant_op(model, [0], a_bits=a_bits, w_bits=w_bits, quant_inference=quant_inference)
    if fuse:
        from .fused import fuse_blocks
        fuse_blocks(model)
    return model
