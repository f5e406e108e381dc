"""Binary / ternary weight, binary activation QAT modules on the H100 engine.

Drop-in for the reference's ``micronet/compression/quantization/wbwtab/quantize.py``
(constructor signatures WB:80, WB:106, WB:153-166; ``prepare`` rules WB:247-347)."""
from __future__ import annotations

import copy

import torch.nn as nn

from . import _lib as L
from . import functional as F_


class ActivationQuantizer(nn.Module):
    """WB:79-94: A == 2 -> sign(x) (0 -> +1) with the saturate-STE; otherwise ReLU."""

    def __init__(self, A=2):
        super().__init__()
        self.A = A
        self.relu = nn.ReLU(inplace=True)

    def binary(self, input):
        y = F_.ActQuantFn.apply(input, F_.ActSpec(L.ACT_SIGN))
        y._mnb_pm1 = True     # exactly +-1: a consuming conv may read it as one bf16 piece / one bit per value
        return y

    def forward(self, input):
        return self.binary(input) if self.A == 2 else self.relu(input)


class WeightQuantizer(nn.Module):
    """WB:105-149: W == 2 binary (in-place mean-centre + clamp of the parameter, then
    sign * E|w|), W == 3 ternary (threshold 0.7 E|w|, scaled by the mean surviving |w|)."""

    def __init__(self, W=2):
        super().__init__()
        self.W = W

    def quantize(self, weight):
        if self.W == 2 or self.W == 3:
            return F_.WbWeightFn.apply(weight, self.W)
        return weight, None, None

    def forward(self, input):
        return self.quantize(input)[0]


class QuantConv2d(nn.Conv2d):
    codes_out = False   # set by fused.fuse_wbwtab_blocks: the only reader is this block's BatchNormBinarize2d (int16 hand-off)

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", W=2, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode)
        self.quant_inference = quant_inference
        self.weight_quantizer = WeightQuantizer(W=W)

    def forward(self, input):
        if not self.quant_inference:
            wq, w_int, w_scale = self.weight_quantizer.quantize(self.weight)
        else:
            wq, w_int, w_scale = self.weight, None, None
        # the input is NOT quantized here (WB:181-195): it is whatever the previous block produced
        # (+-1 after an ActivationQuantizer(A=2), plain fp32 when A == 32)
        return F_.quant_conv2d(input, wq, self.bias, w_int, w_scale, None, self.stride, self.padding,
                               self.dilation, self.groups, codes_out=bool(self.codes_out) and w_int is not None)


class QuantConvTranspose2d(nn.ConvTranspose2d):
    """WB:198-244 (only the weight is quantized; the input is whatever the previous block produced).  Like DF:125-174 the
    reference passes (dilation, groups, bias) positionally in the wrong order and its forward raises ``TypeError`` under
    current PyTorch: this module implements the intent - ``F.conv_transpose2d(x, Wq(w), bias, ...)`` - with the constructor
    arguments taken by name, on the engine's convolution kernels with the roles swapped (functional.ConvTranspose2dFn).
    The per-channel statistics of the weight quantizer run over dim 0 of the [C_in, C_out / g, R, S] weight, exactly as
    WB:105-149 would compute them."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", W=2, quant_inference=False):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                         output_padding=output_padding, groups=groups, bias=bias, dilation=dilation,
                         padding_mode=padding_mode)
        self.quant_inference = quant_inference
        self.weight_quantizer = WeightQuantizer(W=W)

    def forward(self, input):
        L.require_cuda(input, self.weight)
        tnn_bin_weight = self.weight if self.quant_inference else self.weight_quantizer(self.weight)
        return F_.conv_transpose2d(input, tnn_bin_weight, self.bias, self.stride, self.padding, self.output_padding,
                                   self.groups, self.dilation)


def _adopt(dst, src):
    dst.weight.data = src.weight
    if src.bias is not None:
        dst.bias.data = src.bias
    return dst


def add_quant_op(module, layer_counter, layer_num, A=2, W=2, quant_inference=False):
    """WB:247-331: all convs but the first and the last are quantized; every ReLU that
    follows conv 1 .. L-1 becomes an ActivationQuantizer."""
    for name, child in module.named_children():
        if isinstance(child, nn.Conv2d):
            layer_counter[0] += 1
            if 1 < layer_counter[0] < layer_num:
                module._modules[name] = _adopt(QuantConv2d(
                    child.in_channels, child.out_channels, child.kernel_size, stride=child.stride,
                    padding=child.padding, dilation=child.dilation, groups=child.groups,
                    bias=child.bias is not None, padding_mode=child.padding_mode, W=W,
                    quant_inference=quant_inference), child)
        elif isinstance(child, nn.ConvTranspose2d):
            layer_counter[0] += 1
            if 1 < layer_counter[0] < layer_num:     # WB:280-318
                module._modules[name] = _adopt(QuantConvTranspose2d(
                    child.in_channels, child.out_channels, child.kernel_size, stride=child.stride,
                    padding=child.padding, output_padding=child.output_padding, dilation=child.dilation,
                    groups=child.groups, bias=child.bias is not None, padding_mode=child.padding_mode, W=W,
                    quant_inference=quant_inference), child)
        elif isinstance(child, nn.ReLU):
            if 0 < layer_counter[0] < layer_num:
                module._modules[name] = ActivationQuantizer(A=A)
        else:
            add_quant_op(child, layer_counter, layer_num, A=A, W=W, quant_inference=quant_inference)


def prepare(model, inplace=False, A=2, W=2, quant_inference=False, fuse_bn=False):
    """``fuse_bn`` (extension, off by default): additionally fuse BatchNorm2d + binarizer pairs, max-pools and
    channel shuffles around the quantized convolutions (micronet_b200.fused); parameters, buffers, state_dict
    keys and results are unchanged."""
    if not inplace:
        model = copy.deepcopy(model)
    layer_num = sum(isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)) for m in model.modules())
    add_quant_op(model, [0], layer_num, A=A, W=W, quant_inference=quant_inference)
    if fuse_bn and A == 2:
        from .fused import fuse_wbwtab_blocks
        fuse_wbwtab_blocks(model)
    return model
