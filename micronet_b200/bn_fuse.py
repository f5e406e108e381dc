"""Inference-graph converters (SURVEY 8 f3): the reference's two ``bn_fuse`` scripts as library functions.

* ``wbwtab_model_bn_fuse`` - ``wbwtab/bn_fuse/bn_fuse.py:20-105``.  Walks the children in registration order; every
  ``nn.Conv2d`` (quantized or not) that is followed by a sibling ``nn.BatchNorm2d`` absorbs it.  The first
  ``bin_bn_fuse_num`` BatchNorms (= the number of ``ActivationQuantizer`` modules in the model: each of them feeds a
  binarizer) are folded the sign-preserving way - ``sign(bn(z)) = sign(gamma) * sign(z - mean + beta * std / gamma)`` - so
  the weights stay +-1 / ternary and only the bias changes (channels with gamma < 0 flip the sign of weight and bias);
  the rest is the ordinary fold.  Fused convs 2 .. bin_bn_fuse_num become ``wbwtab.QuantConv2d(quant_inference=True)``,
  the others plain ``nn.Conv2d``; the BatchNorm is replaced by ``nn.Identity``.
* ``wbwtab_quantize_inference_weights`` - the weight step that follows in the reference (
  ``bn_fused_model_test.py:191-194``): every wbwtab ``QuantConv2d`` stores its quantized weight alpha_k * {-1, 0, +1}.
* ``iao_model_bn_fuse`` - ``wqaq/iao/bn_fuse/bn_fuse.py:20-73``.  Every ``iao.QuantBNFuseConv2d`` becomes an
  ``iao.QuantConv2d(quant_inference=True, bias=True)`` holding the folded weight / bias (running statistics) and the
  calibrated scale / zero-point buffers of both quantizers.
* ``iao_quantize_inference_weights`` - its weight step (``bn_fused_model_test.py:199-201``): every such conv stores its
  fake-quantized weight, which ``iao.freeze_inference`` runs on the integer levels.

The reference scripts read ``W`` / bit widths / ``q_type`` / ``q_level`` from their command line; here they are arguments
(wbwtab) or read off the module being replaced (iao)."""
from __future__ import annotations

import copy

import torch
import torch.nn as nn

from . import iao as _iao
from . import wbwtab as _wb


def _bn_terms(bn_like, gamma, beta):
    mean = bn_like.running_mean
    std = torch.sqrt(bn_like.running_var + bn_like.eps)
    return mean, std, gamma, beta


def _wbwtab_fuse_pair(conv, bn, counter, n_bin, W):
    mean, std, gamma, beta = _bn_terms(bn, bn.weight, bn.bias)
    w = conv.weight
    b = conv.bias if conv.bias is not None else mean.new_zeros(mean.shape)
    if 1 <= counter <= n_bin:
        # this BatchNorm feeds a binarizer: keep the integer weights, move everything into the bias
        w_f, b_f = w.clone(), b.clone()
        pos, neg = gamma.data.gt(0), gamma.data.lt(0)
        w_f[pos] = w[pos]
        b_f[pos] = b[pos] - mean[pos] + beta[pos] * (std[pos] / gamma[pos])
        w_f[neg] = w[neg] * -1
        b_f[neg] = mean[neg] - b[neg] - beta[neg] * (std[neg] / gamma[neg])
    else:
        w_f = w * (gamma / std).reshape([conv.out_channels, 1, 1, 1])
        b_f = beta + (b - mean) * (gamma / std)
    geometry = dict(stride=conv.stride, padding=conv.padding, dilation=conv.dilation, groups=conv.groups, bias=True,
                    padding_mode=conv.padding_mode)
    if 2 <= counter <= n_bin:
        fused = _wb.QuantConv2d(conv.in_channels, conv.out_channels, conv.kernel_size, W=W, quant_inference=True, **geometry)
    else:
        fused = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, **geometry)
    fused.weight.data = w_f
    fused.bias.data = b_f
    return fused


def _wbwtab_walk(module, state, W):
    last = None
    for name, child in module.named_children():
        if isinstance(child, nn.Conv2d):
            last = (name, child)
        elif isinstance(child, nn.BatchNorm2d):
            if last is None:
                raise ValueError("bn_fuse: BatchNorm2d without a preceding Conv2d sibling")
            state["counter"] += 1
            module._modules[last[0]] = _wbwtab_fuse_pair(last[1], child, state["counter"], state["n_bin"], W)
            module._modules[name] = nn.Identity()
        else:
            _wbwtab_walk(child, state, W)


def wbwtab_model_bn_fuse(model, W=2, inplace=False):
    """``model``: a wbwtab-prepared model (``wbwtab.prepare(..., quant_inference=True)``) with trained statistics"""
    if not inplace:
        model = copy.deepcopy(model)
    n_bin = sum(isinstance(m, _wb.ActivationQuantizer) for m in model.modules())
    _wbwtab_walk(model, {"counter": 0, "n_bin": n_bin}, W)
    return model


def _iao_fuse_one(m):
    mean, std, gamma, beta = _bn_terms(m, m.gamma, m.beta)
    w = m.weight
    b = m.bias if m.bias is not None else mean.new_zeros(mean.shape)
    w_f = w * (gamma / std).reshape([m.out_channels, 1, 1, 1])
    b_f = beta + (b - mean) * (gamma / std)
    aq, wq = m.activation_quantizer, m.weight_quantizer
    fused = _iao.QuantConv2d(m.in_channels, m.out_channels, m.kernel_size, stride=m.stride, padding=m.padding,
                             dilation=m.dilation, groups=m.groups, bias=True, padding_mode=m.padding_mode,
                             a_bits=aq.bits, w_bits=wq.bits, q_type=0 if wq.symmetric else 1,
                             q_level=0 if wq.observer.q_level == "C" else 1, quant_inference=True).to(w.device)
    fused.weight.data = w_f
    fused.bias.data = b_f
    for src, dst in ((aq, fused.activation_quantizer), (wq, fused.weight_quantizer)):
        dst.scale.copy_(src.scale)
        dst.zero_point.copy_(src.zero_point)
        dst.eps.copy_(src.eps)
    return fused


def _iao_walk(module):
    for name, child in module.named_children():
        if isinstance(child, _iao.QuantBNFuseConv2d):
            module._modules[name] = _iao_fuse_one(child)
        else:
            _iao_walk(child)


@torch.no_grad()
def iao_model_bn_fuse(model, inplace=False):
    if not inplace:
        model = copy.deepcopy(model)
    _iao_walk(model)
    return model


@torch.no_grad()
def wbwtab_quantize_inference_weights(model):
    """the second step of the reference's deployment flow (``wbwtab/bn_fuse/bn_fused_model_test.py:191-194``): every wbwtab
    ``QuantConv2d`` of a BN-fused model stores its quantized weight, ``m.weight.data = m.weight_quantizer(m.weight)``, so a
    ``quant_inference`` layer holds alpha_k * {-1, 0, +1} (what ``wbwtab.freeze_inference`` runs on the XNOR kernels)"""
    for m in model.modules():
        if isinstance(m, _wb.QuantConv2d):
            m.weight.data = m.weight_quantizer(m.weight)
    return model


@torch.no_grad()
def dorefa_quantize_inference_weights(model):
    """the weight step of the reference's DoReFa deployment flow (``wqaq/dorefa/quant_model_test/quant_model_test.py:
    191-194``): every DoReFa ``QuantConv2d`` stores its quantized weight, ``m.weight.data = m.weight_quantizer(m.weight)``, so
    a ``quant_inference`` layer holds the levels (2 k - n) / n, n = 2^w - 1, that ``dorefa.freeze_inference`` recovers"""
    from . import dorefa as _df
    for m in model.modules():
        if isinstance(m, _df.QuantConv2d):
            m.weight.data = m.weight_quantizer(m.weight)
    return model


@torch.no_grad()
def iao_quantize_inference_weights(model):
    """the weight step of the reference's IAO deployment flow (``wqaq/iao/bn_fuse/bn_fused_model_test.py:199-201``, on the
    model in eval mode): every IAO ``QuantConv2d`` with ``quant_inference=True`` (``iao_model_bn_fuse``'s output) stores
    ``m.weight_quantizer(m.weight)`` with the stored scale / zero point and no observer or qparam update, per-channel and
    per-layer alike, so it holds the levels ``fl(L * s)`` that ``iao.freeze_inference`` recovers.  Evaluated with
    ``iao.stored_fake_quant`` (torch ops, the kernels' op sequence), so a model converted on the CPU takes the step there."""
    for m in model.modules():
        if isinstance(m, _iao.QuantConv2d) and m.quant_inference and m.weight_quantizer.bits != 32:
            m.weight.data = _iao.stored_fake_quant(m.weight_quantizer, m.weight)[0]
    return model
