"""DoReFa k-bit QAT modules on the H100 engine.

Drop-in for the reference's ``micronet/compression/quantization/wqaq/dorefa/quantize.py``:
same class names, constructor signatures (DF:77-91, DF:178-186), attribute names and
``prepare`` rules (DF:202-323).  The quantizers are stateless, so ``state_dict`` holds only
``weight`` / ``bias`` exactly like the reference."""
from __future__ import annotations

import copy
import functools

import torch.nn as nn

from . import _lib as L
from . import frozen_graph as FG
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
        if "_mnb_frozen" in self.__dict__:      # set by freeze_inference
            return _frozen_conv_forward(self, input)
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


# --------------------------------------------------------------------------
# frozen inference graphs on level planes
# --------------------------------------------------------------------------
def frozen_levels(conv):
    """(wq, w_int i16 [K, C/g, R, S], w_scale f32 [K]) of a DoReFa conv with 2..8-bit weights, or None when its weights cannot be
    frozen.  A QAT layer takes them from its weight quantizer (DF:50-73).  A ``quant_inference`` layer holds that quantizer's
    output (bn_fuse.dorefa_quantize_inference_weights, quant_model_test.py:191-194): v = 2 k / n - 1 with n = 2^w - 1, so the
    level is the odd integer round(v * n); anything else (raw fp32 weights, NaN) is refused."""
    import torch
    bits = conv.weight_quantizer.w_bits
    if not 2 <= bits <= 8:
        return None
    if not conv.quant_inference:
        wq, w_int, w_scale = conv.weight_quantizer.quantize(conv.weight)
        return wq.detach(), w_int.detach(), w_scale.detach()
    n = float(2 ** bits - 1)
    v = conv.weight.detach()
    lv = torch.round(v * n)
    tol = 4 * torch.finfo(torch.float32).eps       # the reconstruction must match v to fp32 rounding
    ok = (bool(torch.isfinite(v).all()) and bool((lv.abs() <= n).all()) and bool((lv.remainder(2) == 1).all())
          and bool(((lv / n - v).abs() <= tol).all()))
    if not ok:
        return None
    return v, lv.to(torch.int16), torch.full((v.shape[0],), 1.0 / n, dtype=torch.float32, device=v.device)


def _freezable(conv):
    if not isinstance(conv, QuantConv2d) or conv.padding_mode != "zeros" or isinstance(conv.padding, str):
        return False
    if not (2 <= conv.activation_quantizer.a_bits <= 8 and 2 <= conv.weight_quantizer.w_bits <= 8):
        return False
    return not conv.quant_inference or frozen_levels(conv) is not None


_check_eval = functools.partial(FG.check_eval, "dorefa")


def _frozen_operands(conv):
    """(wq, w_int, w_scale, bias) computed once; re-done when a parameter or buffer is written in place"""
    def make():
        lv = frozen_levels(conv)
        if lv is None:
            raise RuntimeError("micronet_b200: the weights of a frozen DoReFa layer changed to values that are not weight "
                               "quantizer levels; call dorefa.freeze_inference(model) again")
        lv[1]._mnb_pk_cache = {}          # the packed weight images are built once per shape (functional.frozen_conv)
        return tuple(lv) + (None if conv.bias is None else conv.bias.detach(),)
    return FG.cached_operands(conv, "_mnb_ops", make)


class _Link(FG.Link):
    """frozen_graph.Link whose producer applies the eval BatchNorm (running statistics) before the ReLU and the consumer's
    DoReFa quantizer; a max-pool in between runs as mnb_pk_plane_maxpool"""

    def consumer(self):
        c = self.cconv
        return F_.Consumer(c, c.activation_quantizer.spec(), self.relu, True, tuple(c.weight.shape), tuple(c.stride),
                           tuple(c.padding), tuple(c.dilation), c.groups, True, int8=c.__dict__["_mnb_frozen"]["int8"],
                           bn=self.bn_tensors(), shuffle_groups=self.sg, pool=self.pool)


def _frozen_conv_forward(conv, x):
    """eval forward of a frozen DoReFa conv: cached weight levels, the plane its producer wrote (if it got one) and, with a
    link, its consumer's plane written by the epilogue (BatchNorm, ReLU and shuffle folded in)"""
    _check_eval(conv)
    wq, w_int, w_scale, bias = _frozen_operands(conv)
    spec = conv.activation_quantizer.spec()
    plane = F_.handed_plane(conv, x)
    if plane is None:
        if getattr(x, "_mnb_pk_q", None) is not None:     # a BatchNormReluQuant2d that ran un-linked wrote this conv's plane
            return F_.quant_conv2d(x, wq, bias, w_int, w_scale, spec, conv.stride, conv.padding, conv.dilation, conv.groups)
        x = F_.materialized(x)
        sg = conv.__dict__.get("_mnb_in_shuffle", 1)
        if sg > 1:
            x = FG.shuffle(x, sg)     # the block's channel shuffle that freeze_inference moved into the producer
    info = conv.__dict__["_mnb_frozen"]
    link = info.get("link")
    return F_.frozen_conv(x, plane, wq, bias, w_int, w_scale, spec, conv.stride, conv.padding, conv.dilation, conv.groups,
                          consumer=link.consumer() if link is not None else None, int8=info["int8"])


def _plane_pool(plane, x, k, s, p):
    from . import pk as PK
    return PK.plane_maxpool(plane, *x.shape, k, s, p, int8=x._mnb_pk_pre[3] == "i8")


def _stem_forward(bn, link, x):
    """eval BatchNorm + ReLU behind the un-quantized stem conv, written straight as the first quantized conv's level plane
    (mnb_bn_relu_quant_pack_fwd / _i8_fwd) with the consumer block's shuffle"""
    import ctypes as C
    import torch
    from . import pk as PK
    _check_eval(bn)
    x = F_.materialized(x)
    if x.dim() == 4 and x.is_cuda and x.dtype == torch.float32:
        consumer = link.consumer()
        fmt = consumer.format(tuple(x.shape))
        if fmt is not None:
            b, c, h, w = x.shape
            x = x.contiguous()
            mean, invstd, gamma, beta = (t.data_ptr() for t in consumer.bn)
            qp = consumer.spec.struct()
            lib = L.load()
            if fmt == "i8":
                plane = PK.consumer_plane_i8(b, c, h, w, x.device)
                rc = lib.mnb_bn_relu_quant_pack_i8_fwd(x.data_ptr(), b, c, h * w, mean, invstd, gamma, beta, C.byref(qp),
                                                       consumer.sg, plane.data_ptr(), L.stream())
            else:
                plane = PK.consumer_plane(b, c, h, w, x.device)
                bits = torch.empty((x.numel() + 31) // 32, dtype=torch.int32, device=x.device)   # STE mask (unused)
                rc = lib.mnb_bn_relu_quant_pack_fwd(x.data_ptr(), b, c, h * w, mean, invstd, gamma, beta, C.byref(qp),
                                                    consumer.sg, plane.data_ptr(), bits.data_ptr(), L.stream())
            if rc == 0:
                return F_.tag(torch.empty(x.shape, dtype=torch.float32, device="meta"), consumer.target, plane, fmt)
            if rc != L.E_UNSUPPORTED:
                L.check(rc, "bn_relu_quant_pack (stem)")
    return type(bn).forward(bn, x)


def _conv_bn_act(blk):
    """(conv, BatchNorm, nn.ReLU or None, relu applied?) of one of the reference's conv-bn-relu blocks, else None"""
    from .fused import BatchNormReluQuant2d
    bp = FG.block_parts(blk) if hasattr(blk, "channel_shuffle_flag") else None
    if bp is None or len(bp[1]) not in (1, 2):
        return None
    bn, act = bp[1][0], (bp[1][1] if len(bp[1]) == 2 else None)
    if type(bn) not in (nn.BatchNorm2d, BatchNormReluQuant2d) or not (bn.affine and bn.track_running_stats):
        return None
    if act is not None and (type(act) is not nn.ReLU or isinstance(bn, BatchNormReluQuant2d)):
        return None
    return bp[0], bn, act, act is not None or isinstance(bn, BatchNormReluQuant2d)


_UNDO = "_mnb_dorefa_undo"


def freeze_inference(model, enable=True, int8=False):
    """Inference on level planes for a DoReFa model in eval mode (NIN / NIN-GC-style ``nn.Sequential`` of conv-bn-relu
    blocks; the reference times this graph in wqaq/dorefa/quant_model_test/quant_model_test.py:185-194):
    * every eval-mode QuantConv2d with 2..8-bit quantizers quantizes and packs its weights ONCE (re-done when a parameter or
      buffer is written in place);
    * linking, from the conv-bn-relu block (QuantConv2d, nn.BatchNorm2d or fused.BatchNormReluQuant2d, nn.ReLU or nothing) to
      the first conv of the next block, when that conv is frozen and any max-pool in between is square with 2 * p <= k and
      feeds a stride-1 conv: the producer conv's epilogue applies the eval BatchNorm (running statistics), the ReLU, the
      consumer's quantizer and the next block's channel shuffle and writes the consumer's level plane (mnb_pk_conv_post /
      mnb_pk_i8_conv); the pool runs on that plane (mnb_pk_plane_maxpool); no fp32 activation is written in between;
    * the un-quantized stem conv's BatchNorm + ReLU write the first quantized conv's plane (mnb_bn_relu_quant_pack_fwd or
      its int8 form); the last conv of the model writes fp32 as before;
    * ``int8``: convs with activation and weight quantizers of at most 7 bits run on int8 operands where the int8 plan
      covers them (NIN-GC W4A4); 8-bit layers keep the bf16 planes.
    Covered graphs: ``prepare(...)`` and ``prepare(..., fuse=True)`` in eval mode, and the deployment graph
    ``prepare(quant_inference=True)`` -> ``bn_fuse.dorefa_quantize_inference_weights``; a layer whose weights are not
    quantizer levels (raw fp32 weights) stays un-frozen, and so does the producer in front of it.
    A consumer takes a plane only from the unmodified tagged producer output; when the kernels refuse a shape at run time the
    absorbed modules run as usual.  Numerics (DESIGN.md 4.15): the levels equal the fused BatchNormReluQuant2d's bit for bit;
    where the un-frozen graph ran ATen's BatchNorm a level on a rounding boundary may differ by one.  Parameters, buffers
    and state_dict keys are unchanged; ``enable=False`` restores the modules (needed before training)."""
    from .fused import EngineFloatConv2d
    FG.undo(model, _UNDO)
    if not enable:
        return model
    rw = FG.Rewrite(model, _UNDO)
    frozen = set()
    for m in model.modules():
        if isinstance(m, QuantConv2d) and not m.training and _freezable(m):
            small = m.activation_quantizer.a_bits <= 7 and m.weight_quantizer.w_bits <= 7
            m.__dict__["_mnb_frozen"] = {"int8": bool(int8) and small, "link": None}
            rw.forget(m, "_mnb_frozen", "_mnb_ops")
            frozen.add(m)
    for (conv, bn, act, relu), pool, cfg, nxt, cconv, _ in FG.block_pairs(model, _conv_bn_act, FG.max_pool_cfg):
        if cconv not in frozen or not hasattr(nxt, "channel_shuffle_flag") or (pool is not None and tuple(cconv.stride) != (1, 1)):
            continue
        flag_sg = FG.block_shuffle(nxt)
        fold_sg = int(getattr(pool if pool is not None else bn, "out_shuffle_groups", 1))   # folded by fuse=True
        stem = type(conv) in (nn.Conv2d, EngineFloatConv2d)
        if not (conv in frozen or (stem and relu and (pool is not None or tuple(cconv.stride) == (1, 1)))):
            continue
        link = _Link(cconv, bn, relu, max(flag_sg, fold_sg), None if pool is None else (pool,) + cfg)
        target = link.target
        if stem:
            rw.override(bn, _stem_forward, bn, link)
        else:
            conv.__dict__["_mnb_frozen"]["link"] = link
            rw.override(bn, FG.absorbed_forward, _check_eval, bn, target)
        if act is not None:
            rw.override(act, FG.absorbed_forward, _check_eval, act, target)
        if pool is not None:
            rw.override(pool, FG.pool_forward, _check_eval, _plane_pool, FG.pool_as_usual, pool, link)
        if flag_sg > 1:
            rw.move_shuffle(nxt, cconv, flag_sg)
    return model
