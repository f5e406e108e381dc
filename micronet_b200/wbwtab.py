"""Binary / ternary weight, binary activation QAT modules on the H100 engine.

Drop-in for the reference's ``micronet/compression/quantization/wbwtab/quantize.py``
(constructor signatures WB:80, WB:106, WB:153-166; ``prepare`` rules WB:247-347)."""
from __future__ import annotations

import copy
import functools

import torch.nn as nn

from . import _lib as L
from . import frozen_graph as FG
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


# --------------------------------------------------------------------------
# frozen inference graphs on bit planes
# --------------------------------------------------------------------------
_UNDO = "_mnb_xnor_undo"
_check_eval = functools.partial(FG.check_eval, "wbwtab")


def frozen_levels(conv):
    """(w_int i16 [K, C/g, R, S], alpha f32 [K]) of a wbwtab conv for the XNOR kernels, or None when its weights cannot be
    frozen.  A ``quant_inference`` layer holds alpha_k * {-1, 0, +1} (bn_fuse.wbwtab_quantize_inference_weights): the levels
    are recovered exactly, anything else (raw fp32 weights, NaN) is refused.  A QAT layer takes them from its weight
    quantizer (W = 2 centres the parameter in place, as every forward of the un-frozen layer does); a NaN alpha (an all-zero
    ternary channel, 0 / 0) is refused: a sign bit cannot carry NaN."""
    import torch
    if conv.quant_inference:
        w = conv.weight.detach()
        alpha = w.abs().amax(dim=(1, 2, 3))
        a4 = alpha.view(-1, 1, 1, 1)
        lv = torch.where(a4 > 0, w / torch.where(a4 > 0, a4, torch.ones_like(a4)), torch.zeros_like(w)).round()
        if not torch.equal(lv * a4, w):
            return None
        w_int = lv.to(torch.int16)
    else:
        if conv.weight_quantizer.W not in (2, 3):
            return None
        _, w_int, alpha = conv.weight_quantizer.quantize(conv.weight)
        w_int, alpha = w_int.detach(), alpha.detach()
    if not bool(torch.isfinite(alpha).all()):
        return None
    return w_int, alpha


def _frozen_kernel(conv):
    """the kernel a frozen layer runs, from its geometry: "xnor" inside the XNOR kernel's cover, else "b1" inside the binary
    tensor-core convolution's (DESIGN.md 4.19), else None; None also when frozen_levels would refuse the weights (for a QAT
    ternary layer: an all-zero channel, alpha 0 / 0)"""
    from . import b1 as B1, xnor as XN
    if not isinstance(conv, QuantConv2d) or conv.padding_mode != "zeros" or isinstance(conv.padding, str):
        return None
    k = conv.kernel_size[0]
    sh = L.ConvShape(1, conv.in_channels, max(8, k), max(8, k), conv.out_channels, k, conv.kernel_size[1], conv.stride[0],
                     conv.stride[1], conv.padding[0], conv.padding[1], conv.dilation[0], conv.dilation[1], conv.groups)
    kind = "xnor" if XN.supported(sh) else ("b1" if B1.supported(sh) else None)
    if kind is None:
        return None
    if conv.quant_inference:
        ok = frozen_levels(conv) is not None
    elif conv.weight_quantizer.W == 3:
        ok = bool((conv.weight.detach().abs().amax(dim=(1, 2, 3)) > 0).all())
    else:
        ok = conv.weight_quantizer.W == 2
    return kind if ok else None


class _Link:
    """what a frozen producer writes for its consumer: format (bit plane for a frozen XNOR conv, bf16 +-1 plane for the
    un-quantized head), the consumer's groups, and the modules the epilogue stands for (the eval BatchNorm of a
    BatchNormBinarize2d or an ActivationQuantizer, a 2x2 max-pool, the consumer block's channel shuffle)"""

    def __init__(self, consumer, fmt, out_groups, act, pool, shuffle_groups):
        self.consumer, self.fmt, self.out_groups = consumer, fmt, out_groups
        self.act, self.pool, self.sg = act, pool, shuffle_groups

    @property
    def pool2(self):
        from .fused import BatchNormBinarize2d
        return bool(self.act.pool2) if isinstance(self.act, BatchNormBinarize2d) else self.pool is not None

    def post(self):
        """(mnb_xnor_post, the tensors it points to)"""
        import torch
        from . import xnor as XN
        from .fused import BatchNormBinarize2d
        bn = None
        if isinstance(self.act, BatchNormBinarize2d):
            a = self.act      # eval BatchNorm: running statistics, invstd exactly as BatchNormBinarize2d computes it
            bn = (a.running_mean, torch.rsqrt(a.running_var + a.eps), a.weight.detach(), a.bias.detach())
        return XN.post_struct(self.fmt, self.out_groups, self.sg, self.pool2, bn), bn

    def out_shape(self, b, c, h, w):
        return (b, c, h // 2, w // 2) if self.pool2 else (b, c, h, w)

    def tail(self, y):
        """the absorbed modules, run as they would run un-frozen (planes the kernels refuse at run time)"""
        from .fused import BatchNormBinarize2d
        if isinstance(self.act, BatchNormBinarize2d):
            y = type(self.act).forward(self.act, y)     # BatchNorm + sign [+ pool] [+ shuffle]
        else:
            y = self.act.binary(y)
            if self.pool is not None:
                y = self.pool(y)
            if self.sg > 1:
                y = FG.shuffle(y, self.sg)
                y._mnb_pm1 = True
        return y

    def tag(self, plane, shape, device):
        import torch
        if self.fmt == L.XNOR_PM1_BF16:
            y = torch.empty(shape, dtype=torch.float32, device=device)      # the placeholder of a plane-only producer
            y._mnb_pk_pm1, y._mnb_plane_only, y._mnb_pm1 = plane, True, True
            return y
        y = torch.empty(shape, dtype=torch.float32, device="meta")         # shape only: the data lives in the plane
        return F_.tag(y, self.consumer, plane, "b1" if self.fmt == L.XNOR_B1_PLANE else "bits", groups=self.out_groups)


def _out_buffer(nbytes, fmt, device):
    import torch
    if fmt in (L.XNOR_BITS, L.XNOR_B1_PLANE):
        return torch.empty(nbytes // 4, dtype=torch.int32, device=device)
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


class _PlanePool(nn.Module):
    """a MaxPool2d(k, s, p) between a frozen producer and a frozen b1 consumer: the pool of the +-1 tensor taken on its b1
    plane (mnb_b1_plane_maxpool); any other input runs the original pool"""

    def __init__(self, pool, cfg, consumer):
        super().__init__()
        self.__dict__["pool"] = pool        # not a sub-module: state_dict unchanged
        self.k, self.s, self.p = cfg
        self.link = FG.Link(consumer, None, None, 1, (self,) + tuple(cfg))
        self.train(pool.training)

    def forward(self, x):
        return FG.pool_forward(_check_eval, _b1_pool, _b1_pool_fallback, self, self.link, x, timed=False)


def _b1_pool(plane, x, k, s, p):
    from . import b1 as B1
    rc, out, _ = B1.plane_maxpool(plane, x.shape, x._mnb_pk_pre[4]["groups"], k, s, p)
    if rc == 0:
        return out
    if rc != L.E_UNSUPPORTED:
        L.check(rc, "b1_plane_maxpool")
    return None


def _b1_pool_fallback(pp, link, x, plane):
    return pp.pool(F_.materialized(x))


def _frozen_conv_operands(conv):
    """(w_int, alpha, bias, XNOR weight image) computed once; re-done when a parameter or buffer is written in place"""
    def make():
        lv = frozen_levels(conv)
        if lv is None:
            raise RuntimeError("micronet_b200: the weights of a frozen wbwtab layer changed to values the XNOR kernel cannot "
                               "hold (NaN alpha or not alpha * {-1, 0, 1}); call wbwtab.freeze_inference(model) again")
        return lv[0], lv[1], None if conv.bias is None else conv.bias.detach(), {}
    return FG.cached_operands(conv, "_mnb_ops", make)


def _record(rw, conv, kernel, fmt, link):
    """the record of a frozen conv (or stem binarizer), read by its forward: the kernel it runs, the format it hands over,
    its link"""
    rw.set_dict(conv, "_mnb_frozen", {"kernel": kernel, "fmt": fmt, "link": link})
    rw.set_dict(conv, "_mnb_frozen_plan", (kernel, fmt))


def _frozen_conv_forward(conv, x):
    """XNOR (or, outside its cover, binary tensor-core) conv whose epilogue applies the absorbed BatchNorm / binarizer /
    pool / shuffle and writes the consumer's operand"""
    from . import b1 as B1, xnor as XN
    rec = conv.__dict__["_mnb_frozen"]
    kind, link = rec["kernel"], rec["link"]
    K = B1 if kind == "b1" else XN
    _check_eval(conv)
    w_int, alpha, bias, images = _frozen_conv_operands(conv)
    sh = F_._shape_struct(x.shape, conv.weight.shape, conv.stride, conv.padding, conv.dilation, conv.groups)
    post, keep = link.post()
    nbytes = K.post_bytes(sh, post)
    if nbytes >= 0:
        plane = F_.handed_plane(conv, x)
        if plane is None:
            plane = K.pack_act(F_.materialized(x).contiguous(), conv.groups)
        if "w_img" not in images:
            images["w_img"] = K.pack_weight(sh, w_int)
        out = _out_buffer(nbytes, link.fmt, alpha.device)
        rc = F_._timed(f"fwd_{kind}_post", sh, lambda: K.conv_post(sh, plane, images["w_img"], post, out, alpha=alpha, bias=bias))
        del keep
        if rc == 0:
            p, q = F_._out_hw(sh)
            return link.tag(out, link.out_shape(x.shape[0], conv.out_channels, p, q), alpha.device)
        if rc != L.E_UNSUPPORTED:
            L.check(rc, f"{kind}_conv_post")
    # outside the kernel's cover: the un-frozen layer, then the modules its epilogue stands for
    wq = w_int.float() * alpha.view(-1, 1, 1, 1)
    y = F_.quant_conv2d(F_.materialized(x), wq, bias, w_int, alpha, None, conv.stride, conv.padding, conv.dilation, conv.groups)
    return link.tail(y)


def _frozen_stem_forward(act, x):
    """the binarizer behind the un-quantized stem conv: [eval BatchNorm] + sign [+ pool] [+ shuffle] straight into the
    first XNOR layer's bit plane"""
    import torch
    from . import b1 as B1, xnor as XN
    link = act.__dict__["_mnb_frozen"]["link"]
    K = B1 if link.fmt == L.XNOR_B1_PLANE else XN
    _check_eval(act)
    x = F_.materialized(x)
    if x.dim() == 4 and x.is_cuda and x.dtype == torch.float32:
        b, c, h, w = x.shape
        post, keep = link.post()
        oh, ow = (h // 2, w // 2) if link.pool2 else (h, w)
        nbytes = int((L.load().mnb_b1_act_bytes if K is B1 else L.load().mnb_xnor_act_bytes)(b, c, oh, ow, link.out_groups))
        if nbytes >= 0 and not (link.pool2 and (h | w) & 1):
            out = _out_buffer(nbytes, link.fmt, x.device)
            x = x.contiguous()
            rc = K.pack_act_post(x, post, out)
            del keep
            if rc == 0:
                return link.tag(out, (b, c, oh, ow), x.device)
            if rc != L.E_UNSUPPORTED:
                L.check(rc, "pack_act_post")
    return link.tail(x)


def _bit_block(blk):
    """(conv, binarizer) of a conv-bn-act block that ends in a binarizer (BatchNormBinarize2d, or a BatchNorm-fused conv
    followed by ActivationQuantizer(A=2)), else None"""
    from .fused import BatchNormBinarize2d
    bp = FG.block_parts(blk)
    if bp is None or len(bp[1]) != 1:
        return None
    act = bp[1][0]
    if isinstance(act, BatchNormBinarize2d) or (type(act) is ActivationQuantizer and act.A == 2):
        return bp[0], act
    return None


def _head_conv(conv):
    from .fused import EnginePmConv2d
    return (type(conv) in (nn.Conv2d, EnginePmConv2d) and conv.in_channels % 8 == 0 and conv.padding_mode == "zeros"
            and not isinstance(conv.padding, str))


def _freeze_bits(model, rw):
    """link the conv-bn-act blocks that end in a binarizer (see freeze_inference)"""
    from .fused import BatchNormBinarize2d, EnginePmConv2d
    frozen = {}             # conv -> the kernel it runs frozen ("xnor" / "b1")
    links = []
    # from the last block back: a producer is frozen only when its consumer reads what it writes
    for (conv, act), pool, cfg, nxt, cconv, slot in reversed(list(FG.block_pairs(model, _bit_block, FG.max_pool_cfg))):
        bnb = isinstance(act, BatchNormBinarize2d)
        fold = ppool = None
        if pool is not None:
            if cfg == (2, 2, 0) and not bnb:
                fold = pool         # the 2x2 pool moves into the epilogue
            elif cfg != (2, 2, 0) and int(getattr(pool, "out_shuffle_groups", 1)) == 1:
                ppool = pool        # taken on the consumer's b1 plane (mnb_b1_plane_maxpool), if it has one
            else:
                continue
        shuffled = FG.block_shuffle(nxt) > 1
        if bnb and shuffled:
            continue        # a shuffle the fused producer did not take (not a graph prepare(fuse_bn=True) builds)
        sg = FG.block_shuffle(nxt) if shuffled else (int(act.out_shuffle_groups) if bnb else 1)
        ckind = frozen.get(cconv)
        if ppool is not None and ckind != "b1":
            continue        # a pool the epilogue cannot take and no b1 plane to take it on
        if ckind is not None:
            link = _Link(cconv, L.XNOR_B1_PLANE if ckind == "b1" else L.XNOR_BITS, cconv.groups, act, fold, sg)
        elif (_head_conv(cconv) and not isinstance(cconv, QuantConv2d) and sg == 1 and pool is None
              and not (bnb and act.pool2)):
            link = _Link(cconv, L.XNOR_PM1_BF16, 1, act, None, 1)
        else:
            continue
        kind = None
        if isinstance(conv, QuantConv2d):
            kind = _frozen_kernel(conv)
            # an XNOR producer has no b1-plane epilogue: in front of a b1 consumer it runs un-frozen
            if kind is None or (kind == "xnor" and link.fmt == L.XNOR_B1_PLANE):
                continue
            frozen[conv] = kind
        elif link.fmt == L.XNOR_PM1_BF16:
            continue
        links.append((conv, kind, link, cfg, slot, ppool, nxt, shuffled))
    for conv, kind, link, cfg, slot, ppool, nxt, shuffled in links:
        if ppool is not None:
            # the pool reads what the producer writes and hands its pooled plane to the consumer
            link.consumer = _PlanePool(ppool, cfg, link.consumer)
            rw.set_child(*slot, link.consumer)
        if kind is not None:
            _record(rw, conv, kind, link.fmt, link)
            rw.forget(conv, "_mnb_ops")
            rw.override(conv, _frozen_conv_forward, conv)
            rw.override(link.act, FG.absorbed_forward, _check_eval, link.act, None)    # done in the conv's epilogue
        else:
            _record(rw, link.act, "b1" if link.fmt == L.XNOR_B1_PLANE else "xnor", link.fmt, link)
            rw.override(link.act, _frozen_stem_forward, link.act)
        if link.pool is not None:
            rw.set_child(*slot, nn.Identity())
        if shuffled:
            rw.set_attr(nxt, "channel_shuffle_flag", 0)
        if link.fmt == L.XNOR_PM1_BF16 and type(link.consumer) is nn.Conv2d:
            # the BatchNorm-fused head reads the +-1 plane on the packed-operand family (same parameters)
            h = link.consumer
            pm = EnginePmConv2d(h.in_channels, h.out_channels, h.kernel_size, h.stride, h.padding, h.dilation, h.groups,
                                h.bias is not None, h.padding_mode)
            pm.weight, pm.bias = h.weight, h.bias
            pm.train(h.training)
            for n, k in list(nxt.named_children()):
                if k is h:
                    rw.set_child(nxt, n, pm)


# --------------------------------------------------------------------------
# frozen inference graphs with fp32 activations (A = 32): term-plane hand-offs (DESIGN.md 4.20)
# --------------------------------------------------------------------------
A32_TERMS = 3       # exact bf16 pieces of an fp32 activation (the packed-operand family's split, pk.pack_act with qp None)
A32_PLANE = "terms3"


def _a32_block(blk):
    """(conv, BatchNorm, ReLU) of a conv-bn-act block of an A=32 model (the act: ActivationQuantizer(A=32), WB:79-94, or the
    nn.ReLU behind the head), else None"""
    parts = [k for k in blk.children() if not isinstance(k, nn.Identity)]
    if len(parts) != 3 or not isinstance(parts[0], nn.Conv2d):
        return None
    conv, bn, act = parts
    if type(bn) is not nn.BatchNorm2d or not (bn.affine and bn.track_running_stats):
        return None
    if not ((type(act) is ActivationQuantizer and act.A == 32) or type(act) is nn.ReLU):
        return None
    return conv, bn, act


def _a32_freezable(conv):
    """does this QuantConv2d run frozen on term planes: binary / ternary weights whose levels freeze (frozen_levels: a finite
    alpha), zero padding, and a packed-operand forward at terms (3, 1) on a nominal shape (batch 1, 32 x 32)"""
    from . import pk as PK
    if (type(conv) is not QuantConv2d or conv.training or conv.padding_mode != "zeros" or isinstance(conv.padding, str)
            or conv.weight_quantizer.W not in (2, 3)):
        return False
    # (as _frozen_kernel: the QAT weight quantizer is not run here, W = 2 would centre the parameter in place)
    if conv.quant_inference:
        if frozen_levels(conv) is None:
            return False
    elif conv.weight_quantizer.W == 3 and not bool((conv.weight.detach().abs().amax(dim=(1, 2, 3)) > 0).all()):
        return False
    sh = L.ConvShape(1, conv.in_channels, 32, 32, conv.out_channels, conv.kernel_size[0], conv.kernel_size[1], conv.stride[0],
                     conv.stride[1], conv.padding[0], conv.padding[1], conv.dilation[0], conv.dilation[1], conv.groups)
    return L.PK_MODE != "off" and PK.supported(sh, 0, A32_TERMS, 1)


class _TermLink(FG.Link):
    """frozen_graph.Link of an A=32 graph: the producer applies the eval BatchNorm before the ReLU and the consumer block's
    channel shuffle and writes the consumer's term planes; the max-pool in between runs on them"""

    def __init__(self, cconv, bn, sg, pool):
        super().__init__(cconv, bn, None, sg, pool)

    @property
    def split(self):
        return self.cconv.stride[0] == 2 and self.pool is None

    def read_shape(self, out_shape):
        if self.pool is None:
            return tuple(out_shape)
        _, k, s, p = self.pool
        b, c, h, w = out_shape
        return (b, c, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)

    def accepts(self, out_shape):
        """will the consumer read the term plane of a producer output of this shape (the pk forward at terms (3, 1) on its
        plain, unsplit or phase-split plane)?"""
        from . import pk as PK
        c = self.cconv
        b, ch, h, w = self.read_shape(out_shape)
        if ch != c.in_channels or PK.padded(ch, c.groups) or ch % 8:
            return False
        if self.sg > 1 and (ch % self.sg or self.split):
            return False
        if self.split and (h | w) & 1:
            return False
        sh = F_._shape_struct((b, ch, h, w), c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
        return L.PK_MODE != "off" and PK.supported(sh, 0, A32_TERMS, 1)

    def tag(self, plane, shape):
        import torch
        y = torch.empty(shape, dtype=torch.float32, device="meta")   # shape only: the data lives in the term plane
        return F_.tag(y, self.target, plane, "terms", split=self.split, terms=A32_TERMS)


def _terms_pool(plane, x, k, s, p):
    from . import pk as PK
    rc, out = PK.plane_maxpool_terms(plane, *x.shape, k, s, p, A32_TERMS)
    if rc == 0:
        return out
    if rc != L.E_UNSUPPORTED:
        L.check(rc, "pk_plane_maxpool_terms")
    return None


def _terms_pool_fallback(pool, link, x, plane):
    """the pool as usual on the decoded tensor, in the producer's channel order: a refused plane holds the consumer's
    (shuffled) order, and the consumer applies its block's shuffle itself when no plane arrives (shuffle with C / sg groups
    is the inverse of the shuffle with sg)"""
    y = F_.materialized(x)
    if plane is not None and link.sg > 1:
        y = FG.shuffle(y, y.shape[1] // link.sg)
    return type(pool).forward(pool, y)


# the max-pool between a frozen producer and its consumer, on the producer's term plane (mnb_pk_plane_maxpool_terms)
_a32_pool_forward = functools.partial(FG.pool_forward, _check_eval, _terms_pool, _terms_pool_fallback)


def _a32_produce(link, y):
    """eval BatchNorm + ReLU of the fp32 tensor y written as its consumer's term planes with the consumer block's shuffle
    (mnb_bn_relu_pack_terms_fwd): the tagged placeholder, or None when the producer does not take y (y is left as it is)"""
    import torch
    from . import pk as PK
    if not (y.dim() == 4 and y.is_cuda and y.dtype == torch.float32 and not link.split and link.accepts(y.shape)):
        return None
    b, c, h, w = y.shape
    y = y.contiguous()
    plane = PK.terms_plane(b, c, h, w, A32_TERMS, y.device)
    rc = PK.bn_relu_pack_terms(y, link.bn_tensors(), True, link.sg, A32_TERMS, plane)
    if rc == 0:
        return link.tag(plane, y.shape)
    if rc != L.E_UNSUPPORTED:
        L.check(rc, "bn_relu_pack_terms")
    return None


def _a32_stem_forward(bn, link, x):
    """the BatchNorm behind the fp32 stem conv: with the ReLU and the consumer block's shuffle, written straight as the first
    quantized conv's term plane (_a32_produce); the BatchNorm as usual where the producer does not take the tensor"""
    _check_eval(bn)
    x = F_.materialized(x)
    out = _a32_produce(link, x)
    return out if out is not None else type(bn).forward(bn, x)


def _epilogue_hand_off(link, sh):
    """does the conv's epilogue write its consumer's term planes?  Else it writes fp32 and the stem producer writes the planes
    from it.  Not for a segmented plan (mnb_pk_conv_post refuses it), nor for a shuffled link: its epilogue stores each
    element as three scattered 2-byte pieces, several times slower than the fp32 output plus the producer's whole-unit stores
    (harness/wbwtab_a32_infer_probe.py compares both per layer, DESIGN.md 4.20)"""
    from . import pk as PK
    return link.sg == 1 and not PK.segmented(sh, 0, A32_TERMS, 1)


def _a32_conv_forward(conv, x):
    """eval forward of a frozen A=32 conv: its cached weight levels and (3, 1) weight image, the term plane its producer wrote
    (else its own pack of x) and, with a link, its consumer's term plane written by the epilogue (BatchNorm, ReLU, shuffle)"""
    import torch
    from . import pk as PK
    _check_eval(conv)
    link = conv.__dict__["_mnb_frozen"]["link"]
    w_int, alpha, bias, images = _frozen_conv_operands(conv)
    plane = F_.handed_plane(conv, x)
    if plane is None:
        x = F_.materialized(x)
        sg = conv.__dict__.get("_mnb_in_shuffle", 1)
        if sg > 1:
            x = FG.shuffle(x, sg)      # the block's channel shuffle that freeze_inference moved into the producer
    sh = F_._shape_struct(x.shape, conv.weight.shape, conv.stride, conv.padding, conv.dilation, conv.groups)
    p, q = F_._out_hw(sh)
    out_shape = (x.shape[0], conv.out_channels, p, q)
    if L.PK_MODE == "off" or not PK.supported(sh, 0, A32_TERMS, 1) or (plane is None and x.dtype != torch.float32):
        # outside the cover: the un-frozen layer on the decoded input
        wq = w_int.float() * alpha.view(-1, 1, 1, 1)
        return F_.quant_conv2d(F_.materialized(x), wq, bias, w_int, alpha, None, conv.stride, conv.padding, conv.dilation,
                               conv.groups)
    dev = alpha.device
    if plane is None:
        L.require_cuda(x, conv.weight)
        plane, _ = PK.pack_act(x.contiguous(), None, A32_TERMS, phase_split=sh.stride_h == 2, groups=conv.groups)
    key = ("terms", PK._key(sh))
    if key not in images:
        images[key] = PK.pack_weight(sh, 0, A32_TERMS, 1, w_int=w_int)
    w_img = images[key]
    hand = link is not None and link.accepts(out_shape) and not PK.padded(conv.out_channels, conv.groups)
    if hand and _epilogue_hand_off(link, sh):
        cplane = PK.terms_plane(*out_shape, A32_TERMS, dev)
        rc = F_._timed("fwd_pk_terms", sh, lambda: PK.conv_post_terms(sh, plane, w_img, None, cplane, A32_TERMS, True,
                                                                       link.split, n_scale=alpha, bias=bias,
                                                                       bn=link.bn_tensors(), shuffle_groups=link.sg))
        if rc == 0:
            return link.tag(cplane, out_shape)
        if rc != L.E_UNSUPPORTED:
            L.check(rc, "pk_conv_post (term planes)")
    y = torch.empty(out_shape, dtype=torch.float32, device=dev)
    L.check(F_._timed("fwd_pk", sh, lambda: PK.conv(sh, 0, plane, A32_TERMS, w_img, 1, y, n_scale=alpha, bias=bias)),
            "pk_conv fwd")
    if hand:
        # no consumer epilogue: the stem producer writes the plane from the fp32 output, the same op sequence
        out = _a32_produce(link, y)
        if out is not None:
            return out
    # no consumer plane: fp32 output; the absorbed modules (BatchNorm, ReLU, pool) run as usual on it
    return y


def _freeze_a32(model, rw):
    """link the A=32 conv-bn-act blocks (DESIGN.md 4.20)"""
    from .fused import EngineFloatConv2d
    frozen = {p[0] for p in FG.blocks(model, _a32_block) if _a32_freezable(p[0])}
    for conv in frozen:
        _record(rw, conv, "pk", "fp32", None)
        rw.forget(conv, "_mnb_ops")
        rw.override(conv, _a32_conv_forward, conv)
    for (conv, bn, act), pool, cfg, nxt, cconv, _ in FG.block_pairs(model, _a32_block, FG.max_pool_cfg):
        if cconv not in frozen or bn.training or (pool is not None and tuple(cconv.stride) != (1, 1)):
            continue
        if pool is not None and int(getattr(pool, "out_shuffle_groups", 1)) != 1:
            continue
        stem = type(conv) in (nn.Conv2d, EngineFloatConv2d)
        if not (conv in frozen or stem):
            continue
        sg = FG.block_shuffle(nxt)
        link = _TermLink(cconv, bn, sg, None if pool is None else (pool,) + cfg)
        if stem:
            rw.override(bn, _a32_stem_forward, bn, link)
        else:
            _record(rw, conv, "pk", A32_PLANE, link)
            rw.override(bn, FG.absorbed_forward, _check_eval, bn, link.target)
        rw.override(act, FG.absorbed_forward, _check_eval, act, link.target)
        if pool is not None:
            rw.override(pool, _a32_pool_forward, pool, link)
        if sg > 1:
            rw.move_shuffle(nxt, cconv, sg)


def freeze_inference(model, enable=True):
    """Inference on bit planes for a wbwtab model in eval mode (NIN-GC-style ``nn.Sequential`` of conv-bn-act blocks):
    every binary / ternary conv whose output is binarized for a consumer runs the XNOR-popcount kernel (outside its cover,
    e.g. NIN's 160 / 192-channel layers: the binary tensor-core convolution, DESIGN.md 4.19) with its weights
    quantized and packed ONCE (re-done when a parameter is written in place), and its epilogue writes the consumer's operand
    directly - the sign bits of the next XNOR layer (mnb_xnor_conv_post), or the +-1 bf16 plane of the un-quantized head -
    so no fp32 activation crosses between two binarized layers.  The binarizer behind the stem conv writes the first
    layer's bit plane (mnb_xnor_pack_act_post).  Covered graphs:
    * the QAT graph with fused producers (``prepare(..., fuse_bn=True)``, then ``.eval()``): each layer's
      BatchNormBinarize2d (running statistics, folded pool, channel shuffle) moves into the conv's epilogue;
    * the reference's deployment graph (``prepare(quant_inference=True)`` -> ``bn_fuse.wbwtab_model_bn_fuse`` ->
      ``bn_fuse.wbwtab_quantize_inference_weights``): the ActivationQuantizer, the following MaxPool2d(2, 2) and the next
      block's channel shuffle move into the epilogue, and the BatchNorm-fused head conv reads the +-1 plane on the
      packed-operand tensor cores (fused.EnginePmConv2d).
    A layer whose weights are not of the form alpha_k * {-1, 0, +1} with a finite alpha (raw fp32 weights, an all-zero
    ternary channel) stays un-frozen, and so does every producer without a frozen consumer.  A consumer takes a plane only
    from the unmodified tagged producer output; anything else reads ``functional.materialized`` of what it receives.  The
    logits equal the un-frozen eval forward's bit for bit (same integer sums, same fmaf, same BatchNorm op sequence).
    Models with fp32 activations (``prepare(A=32, W=2|3)``: conv -> nn.BatchNorm2d -> ActivationQuantizer(A=32), a ReLU) hand
    their activations over as term planes instead (DESIGN.md 4.20): every eval-mode binary / ternary QuantConv2d whose levels
    freeze and whose shape the packed-operand forward covers at terms (3, 1) runs on its weight levels, quantized and packed
    once; a block linked to the next block's frozen conv (across a max-pool with 2 p <= k in front of a stride-1 conv) writes
    that conv's three exact bf16 pieces of ReLU(BatchNorm(y)) in the next block's channel order from its epilogue
    (mnb_pk_conv_post with terms_out), the pool runs on the plane (mnb_pk_plane_maxpool_terms), and the fp32 stem conv's
    BatchNorm + ReLU write the first plane (mnb_bn_relu_pack_terms_fwd).  The last quantized conv writes fp32 for the head.
    Each frozen conv holds its record ``_mnb_frozen``: the kernel it runs, the format it hands over and its link;
    ``_mnb_frozen_plan`` is (kernel, format): ("xnor" or "b1", the XNOR post format) on bit planes, ("pk", "terms3") for an
    A=32 conv writing term planes and ("pk", "fp32") for one writing fp32.  The logits
    equal a block-by-block composition of those kernels bit for bit; against the un-frozen forward (another conv kernel,
    ATen's BatchNorm) they agree to the fp32 contract.
    Parameters, buffers and state_dict keys are unchanged; ``enable=False`` restores the modules (needed before training)."""
    FG.undo(model, _UNDO)
    if not enable:
        return model
    rw = FG.Rewrite(model, _UNDO)
    _freeze_bits(model, rw)
    _freeze_a32(model, rw)
    return model
