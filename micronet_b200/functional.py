"""autograd.Function wrappers around the C-ABI kernels.

Each Function mirrors one autograd node (or a fused chain of nodes) of the
reference's forward path; the math each kernel implements is documented in
``include/micronet_b200.h`` with the reference file:line it replaces."""
from __future__ import annotations

import ctypes as C

import torch
from torch.autograd import Function

from . import _lib as L


# --------------------------------------------------------------------------
# optional per-launch device timing of the conv kernels (bench.py's roofline leg)
# --------------------------------------------------------------------------
class KernelTimer:
    """records a CUDA-event pair on the launching (current) stream around each conv kernel call"""

    def __init__(self):
        self.records = []  # (kind, shape tuple, start event, end event)

    def run(self, kind, sh, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = fn()
        b.record()
        self.records.append((kind, tuple(getattr(sh, f) for f, _ in sh._fields_), a, b))
        return rc

    def summary(self):
        """{(kind, shape): [ms, ...]} — call after torch.cuda.synchronize()"""
        out = {}
        for kind, shape, a, b in self.records:
            out.setdefault((kind, shape), []).append(a.elapsed_time(b))
        return out


TIMER = None  # set to a KernelTimer to enable


def _timed(kind, sh, fn):
    return fn() if TIMER is None else TIMER.run(kind, sh, fn)


# --------------------------------------------------------------------------
# activation quantizer description
# --------------------------------------------------------------------------
class ActSpec:
    """Which activation fake-quantizer to run and where its device-resident
    parameters live (tensors are the module's registered buffers)."""

    __slots__ = ("mode", "bits", "qmin", "qmax", "q_type", "scale", "zero_point", "obs_min", "obs_max")

    def __init__(self, mode, bits=8, qmin=0, qmax=255, q_type=0, scale=None, zero_point=None,
                 obs_min=None, obs_max=None):
        self.mode, self.bits, self.qmin, self.qmax, self.q_type = mode, bits, qmin, qmax, q_type
        self.scale, self.zero_point, self.obs_min, self.obs_max = scale, zero_point, obs_min, obs_max

    def struct(self):
        return L.ActQParams(self.mode, self.bits, self.qmin, self.qmax, self.q_type, L.ptr(self.scale),
                            L.ptr(self.zero_point), L.ptr(self.obs_min), L.ptr(self.obs_max))

    def frozen(self):
        """copy with private clones of the device scalars: what backward must see is the forward-time scale / range
        (the reference uses self.scale.clone(), IAO:228-239), not whatever a later forward of the module wrote"""
        if self.mode != L.ACT_IAO:
            return self
        snap = torch.cat([self.scale.reshape(1), self.zero_point.reshape(1), self.obs_min.reshape(1), self.obs_max.reshape(1)])
        return ActSpec(self.mode, self.bits, self.qmin, self.qmax, self.q_type, snap[0:1], snap[1:2], snap[2:3], snap[3:4])

    # decoding of the u8 codes: effective integer e = code + offset (+ zero_point), value = e * scale
    @property
    def code_offset(self):
        if self.mode == L.ACT_IAO:
            return self.qmin
        if self.mode == L.ACT_SIGN:
            return -1
        return 0


def _dorefa_scale_tensor(bits, device, _cache={}):
    key = (bits, device.type, device.index)
    if key not in _cache:
        # Python double 1/(2^a-1), cast to fp32 exactly as ATen does for `tensor / python_float`
        _cache[key] = torch.tensor([1.0 / float(2 ** bits - 1)], dtype=torch.float32, device=device)
    return _cache[key]


def act_quant_raw(x, spec: ActSpec, want_codes, want_bits, want_xq):
    """run the activation quantizer kernel; returns (codes, pass_bits, xq)"""
    L.require_cuda(x)
    lib = L.load()
    x = x.contiguous()
    n = x.numel()
    codes = torch.empty(x.shape, dtype=torch.uint8, device=x.device) if want_codes else None
    bits = torch.empty((n + 31) // 32, dtype=torch.int32, device=x.device) if want_bits else None
    xq = torch.empty_like(x) if want_xq else None
    qp = spec.struct()
    L.check(lib.mnb_act_quant_fwd(x.data_ptr(), n, C.byref(qp), L.ptr(codes), L.ptr(bits), L.ptr(xq),
                                  L.stream()), "act_quant_fwd")
    return codes, bits, xq


class ActQuantFn(Function):
    """standalone fake-quant of an activation tensor (reference: ActivationQuantizer /
    Quantizer.forward returning the dequantized tensor)."""

    @staticmethod
    def forward(ctx, x, spec: ActSpec):
        _, bits, xq = act_quant_raw(x, spec, False, ctx.needs_input_grad[0], True)
        ctx.spec, ctx.bits = (spec.frozen() if ctx.needs_input_grad[0] else spec), bits
        return xq

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        g = g.contiguous()
        dx = torch.empty_like(g)
        qp = ctx.spec.struct()
        L.check(lib.mnb_act_quant_bwd(g.data_ptr(), ctx.bits.data_ptr(), g.numel(), C.byref(qp),
                                      dx.data_ptr(), L.stream()), "act_quant_bwd")
        return dx, None


class QuantAddFn(Function):
    """IAO QuantAdd (IAO:1441-1498): Q(res) + Q(shortcut) with the shared quantizer, one kernel each way"""

    @staticmethod
    def forward(ctx, a, b, spec: ActSpec, relu=False):
        L.require_cuda(a, b)
        lib = L.load()
        a, b = a.contiguous(), b.contiguous()
        assert a.shape == b.shape, "QuantAdd: operand shapes differ"
        n = a.numel()
        out = torch.empty_like(a)
        words = (n + 31) // 32
        ba = torch.empty(words, dtype=torch.int32, device=a.device) if ctx.needs_input_grad[0] else None
        bb = torch.empty(words, dtype=torch.int32, device=a.device) if ctx.needs_input_grad[1] else None
        qp = spec.struct()
        assert not (relu and (ba is not None or bb is not None)), "the folded ReLU is an inference-only fusion"
        L.check(lib.mnb_quant_add_fwd(a.data_ptr(), b.data_ptr(), n, C.byref(qp), out.data_ptr(), L.ptr(ba), L.ptr(bb),
                                      1 if relu else 0, L.stream()), "quant_add_fwd")
        ctx.spec, ctx.ba, ctx.bb = spec.frozen() if (ba is not None or bb is not None) else spec, ba, bb
        return out

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        g = g.contiguous()
        da = torch.empty_like(g) if ctx.ba is not None else None
        db = torch.empty_like(g) if ctx.bb is not None else None
        qp = ctx.spec.struct()
        L.check(lib.mnb_quant_add_bwd(g.data_ptr(), L.ptr(ctx.ba), L.ptr(ctx.bb), g.numel(), C.byref(qp), L.ptr(da),
                                      L.ptr(db), L.stream()), "quant_add_bwd")
        return da, db, None, None


# --------------------------------------------------------------------------
# weight quantizers: return (wq fp32, w_int i16, w_scale f32[K])
# --------------------------------------------------------------------------
class DorefaWeightFn(Function):
    @staticmethod
    def forward(ctx, w, w_bits):
        L.require_cuda(w)
        lib = L.load()
        w = w.contiguous()
        n, k = w.numel(), w.shape[0]
        wq = torch.empty_like(w)
        w_int = torch.empty(w.shape, dtype=torch.int16, device=w.device)
        w_scale = torch.empty(k, dtype=torch.float32, device=w.device)
        aux = torch.empty(n + 4, dtype=torch.float32, device=w.device)
        L.check(lib.mnb_dorefa_weight_fwd(w.data_ptr(), n, k, w_bits, w_int.data_ptr(), w_scale.data_ptr(),
                                          wq.data_ptr(), aux.data_ptr(), L.scratch(w.device).data_ptr(),
                                          L.stream()), "dorefa_weight_fwd")
        ctx.aux, ctx.w_bits = aux, w_bits
        ctx.mark_non_differentiable(w_int, w_scale)
        return wq, w_int, w_scale

    @staticmethod
    def backward(ctx, g, _gi, _gs):
        lib = L.load()
        g = g.contiguous()
        dw = torch.empty_like(g)
        L.check(lib.mnb_dorefa_weight_bwd(g.data_ptr(), ctx.aux.data_ptr(), g.numel(), ctx.w_bits,
                                          dw.data_ptr(), L.scratch(g.device).data_ptr(), L.stream()),
                "dorefa_weight_bwd")
        return dw, None


class WbWeightFn(Function):
    """wbwtab binary / ternary weights.  W == 2 mutates ``w`` in place (WB:98-102)."""

    @staticmethod
    def forward(ctx, w, W):
        L.require_cuda(w)
        lib = L.load()
        assert w.is_contiguous() and w.dim() == 4
        k, cpg, khw = w.shape[0], w.shape[1], w.shape[2] * w.shape[3]
        wq = torch.empty_like(w)
        w_int = torch.empty(w.shape, dtype=torch.int16, device=w.device)
        w_scale = torch.empty(k, dtype=torch.float32, device=w.device)
        aux = torch.empty(3 * k, dtype=torch.float32, device=w.device)
        L.check(lib.mnb_wb_weight_fwd(w.data_ptr(), k, cpg, khw, W, w_int.data_ptr(), w_scale.data_ptr(),
                                      wq.data_ptr(), aux.data_ptr(), L.stream()), "wb_weight_fwd")
        ctx.w, ctx.aux, ctx.W = w.detach(), aux, W  # gradient is taken at the (mutated) parameter values
        ctx.mark_non_differentiable(w_int, w_scale)
        return wq, w_int, w_scale

    @staticmethod
    def backward(ctx, g, _gi, _gs):
        lib = L.load()
        g = g.contiguous()
        w = ctx.w
        dw = torch.empty_like(g)
        L.check(lib.mnb_wb_weight_bwd(g.data_ptr(), w.data_ptr(), ctx.aux.data_ptr(), w.shape[0], w.shape[1],
                                      w.shape[2] * w.shape[3], ctx.W, dw.data_ptr(), L.stream()),
                "wb_weight_bwd")
        return dw, None


class IaoWeightFn(Function):
    """IAO fake-quant of a weight tensor with (already refreshed) per-row or per-layer qparams."""

    @staticmethod
    def forward(ctx, w, scale, zero_point, obs_min, obs_max, q_type, qmin, qmax):
        L.require_cuda(w)
        lib = L.load()
        w = w.contiguous()
        n, k, rows = w.numel(), w.shape[0], scale.numel()
        wq = torch.empty_like(w)
        w_int = torch.empty(w.shape, dtype=torch.int16, device=w.device)
        w_scale = torch.empty(k, dtype=torch.float32, device=w.device)
        keep = torch.empty(w.shape, dtype=torch.uint8, device=w.device)
        L.check(lib.mnb_iao_weight_fwd(w.data_ptr(), n, k, rows, scale.data_ptr(), zero_point.data_ptr(),
                                       obs_min.data_ptr(), obs_max.data_ptr(), q_type, qmin, qmax,
                                       w_int.data_ptr(), w_scale.data_ptr(), wq.data_ptr(), keep.data_ptr(),
                                       L.stream()), "iao_weight_fwd")
        ctx.keep, ctx.scale, ctx.k, ctx.rows = keep, scale, k, rows
        ctx.mark_non_differentiable(w_int, w_scale)
        return wq, w_int, w_scale

    @staticmethod
    def backward(ctx, g, _gi, _gs):
        lib = L.load()
        g = g.contiguous()
        dw = torch.empty_like(g)
        L.check(lib.mnb_iao_weight_bwd(g.data_ptr(), ctx.keep.data_ptr(), ctx.scale.data_ptr(), g.numel(),
                                       ctx.k, ctx.rows, dw.data_ptr(), L.stream()), "iao_weight_bwd")
        return (dw,) + (None,) * 7


# --------------------------------------------------------------------------
# the fake-quantized convolution
# --------------------------------------------------------------------------
def _shape_struct(x_shape, w_shape, stride, padding, dilation, groups):
    b, c, h, w = x_shape
    k, _, r, s = w_shape
    return L.ConvShape(b, c, h, w, k, r, s, stride[0], stride[1], padding[0], padding[1],
                       dilation[0], dilation[1], groups)


def _out_hw(sh: L.ConvShape):
    p = (sh.in_h + 2 * sh.pad_h - sh.dil_h * (sh.ker_h - 1) - 1) // sh.stride_h + 1
    q = (sh.in_w + 2 * sh.pad_w - sh.dil_w * (sh.ker_w - 1) - 1) // sh.stride_w + 1
    return p, q


def channel_sums(x4):
    """sum over (B, H, W) of a [B, C, H, W] tensor -> [C] (bias gradient)."""
    lib = L.load()
    b, c = x4.shape[0], x4.shape[1]
    hw = x4.numel() // (b * c)
    out = torch.empty(2 * c, dtype=torch.float32, device=x4.device)
    L.check(lib.mnb_channel_stats(x4.data_ptr(), b, c, hw, 0, out.data_ptr(),
                                  L.scratch(x4.device, c).data_ptr(), L.stream()), "channel_stats")
    return out[:c]



def materialized(t):
    """the values of a producer output: ``t`` itself, or - for a plane-only output of a fused BatchNorm + binarizer (its fp32
    storage was never written) - the +-1 tensor rebuilt from the bf16 operand plane [b][c/8][h][w][8], or - for a wbwtab conv
    that handed its output to its BatchNorm as int16 codes (``codes_out``) - that output decoded with the conv epilogue's own
    fmaf, or - for the output of a frozen wbwtab layer (wbwtab.freeze_inference) - the +-1 tensor its consumer's bit plane or
    b1 plane encodes, or the fp32 tensor whose exact pieces a frozen A=32 producer wrote (term planes).  A meta-shaped
    output with a level plane (bf16 / i8) cannot be decoded and raises.
    Plumbing for tests, hooks and readers outside the fused producers; the training step never calls it."""
    pre = getattr(t, "_mnb_pk_pre", None)
    if pre is not None:
        _, plane, _, fmt, info = pre
        if fmt == "bits":
            from . import xnor as XN
            return XN.unpack(plane, t.shape, info["groups"])
        if fmt == "b1":
            from . import b1 as B1
            return B1.unpack(plane, t.shape, info["groups"])
        if fmt == "terms":
            from . import pk as PK
            return PK.unpack_terms(plane, t.shape, info["terms"], split=info["split"])
        if t.device.type == "meta":
            raise RuntimeError(f"micronet_b200: a {fmt} operand plane cannot be decoded")
    codes = getattr(t, "_mnb_codes", None)
    if codes is not None:
        b, c = t.shape[0], t.shape[1]
        out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
        L.check(L.load().mnb_codes_decode(codes[0].data_ptr(), codes[1].data_ptr(), b, c, t.numel() // (b * c), out.data_ptr(),
                                          L.stream()), "codes_decode")
        return out
    if not getattr(t, "_mnb_plane_only", False):
        return t
    b, c, h, w = t.shape
    plane = t._mnb_pk_pm1.view(torch.bfloat16).view(b, c // 8, h, w, 8)
    return plane.permute(0, 1, 4, 2, 3).reshape(b, c, h, w).float()


def _pk_terms(spec, w_int, pm1=False):
    """(terms of the activation operand, terms of the weight operand) on the packed-operand path; ``pm1``: the raw input is
    known to hold only +-1 (output of a binarizer): one bf16 piece is exact"""
    T = L.PK_TERMS
    if spec is None:
        ta = 1 if pm1 else T
    else:
        ta = 2 if (spec.mode == L.ACT_IAO and spec.q_type == 1) else 1   # asymmetric: |level + zero_point| may exceed 256
    return ta, (1 if w_int is not None else T)


def _pk_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, prepacked=None, pre_relu=False, pm1=False, codes_out=False,
                prepacked_bits=None, train_post=None):
    """forward on the packed-operand tensor-core family; returns False when the shape is outside its cover.
    ``prepacked``: the operand plane a fused producer (fused.BNReluQuantFn) already wrote - x itself holds no data then;
    ``prepacked_bits``: the STE mask that producer wrote with it for this layer's data gradient (QAFT hand-offs; without it
    the producer applies the mask in its own backward).
    ``train_post``: the Consumer of a QAFT hand-off (iao.prepare(fuse=True)): the epilogue writes its plane and STE mask
    (mnb_pk_conv_post_train) and y is left unwritten, tagged with both; where that epilogue refuses, y as usual.
    ``codes_out`` (wbwtab layer on a +-1 input whose only reader is its fused BatchNorm + binarizer): the exact integer sums
    go out as int16 codes with their decode pair, tagged on y as ``_mnb_codes``; y itself is then not written.  Shapes the
    int16 hand-off does not cover write y as usual."""
    from . import pk as PK
    need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    ta, tw = _pk_terms(spec, w_int, pm1)
    if not PK.supported(sh, 0, ta, tw):
        return False
    # the backward of a layer stays in the family its forward ran in (saved operands are packed): check its cover now
    Tb = L.PK_TERMS_BWD
    if need_dx and not PK.supported(sh, 1, Tb, 1 if w_int is not None else Tb):
        return False
    if need_dw and not PK.wgrad_supported(sh, Tb, min(ta, Tb)):
        return False
    qp = spec.struct() if spec is not None else None
    if prepacked is not None:
        x_pk, bits8 = prepacked, prepacked_bits
    else:
        x_pk, bits8 = PK.pack_act(x, qp, ta, phase_split=sh.stride_h == 2, want_bits=need_dx, relu=pre_relu,
                                  groups=sh.groups)
    w_img = PK.weight_image(sh, ta, tw, w_int=w_int, w_f32=None if w_int is not None else wq)
    # backward must see the forward-time scale (the reference clones it too); no clone needed without autograd
    a_scale, a_const = PK.act_scale(spec, clone=need_dx or need_dw)
    rc = L.E_UNSUPPORTED
    if codes_out and w_int is not None and ta == 1 and tw == 1:
        codes = torch.empty(y.shape, dtype=torch.int16, device=y.device)
        dec = torch.empty(2 * y.shape[1], dtype=torch.float32, device=y.device)
        rc = _timed("fwd_pk", sh, lambda: PK.run_conv_codes(sh, x_pk, w_img, codes, dec, n_scale=w_scale, a_scale=a_scale,
                                                            a_scale_const=a_const, bias=bias))
        if rc == 0:
            y._mnb_codes = (codes, dec)
    if train_post is not None and w_int is not None:
        cplane, cbits = PK.consumer_plane(*y.shape, y.device), PK.consumer_bits(*y.shape, y.device)
        cqp = train_post.post_spec.struct()
        rc = _timed("fwd_pk", sh, lambda: PK.conv_post(sh, x_pk, ta, w_img, tw, None, cqp, cplane, True, train_post.split,
                                                       n_scale=w_scale, a_scale=a_scale, a_scale_const=a_const, bias=bias,
                                                       post_bits=cbits))
        if rc == 0:
            tag(y, train_post.target, cplane, "bf16", bits=cbits)
    if rc == L.E_UNSUPPORTED:
        rc = _timed("fwd_pk", sh, lambda: PK.run_conv(sh, 0, x_pk, ta, w_img, tw, y,
                                                      n_scale=w_scale if w_int is not None else None, a_scale=a_scale,
                                                      a_scale_const=a_const, bias=bias))
    if rc == L.E_UNSUPPORTED:
        return False
    L.check(rc, "pk_conv fwd")
    ctx.pk_x, ctx.pk_ta, ctx.pk_bits8, ctx.pk_prepacked = x_pk, ta, bits8, prepacked is not None and bits8 is None
    # the quantizer's STE gain on the data gradient, and the scale of the saved activation levels in the weight gradient
    ctx.pk_gain = 0.1 if (spec is not None and spec.mode == L.ACT_DOREFA) else 1.0
    ctx.pk_wg_scale = None
    if spec is not None:
        ctx.pk_wg_scale = a_scale if spec.mode == L.ACT_IAO else _dorefa_scale_tensor(spec.bits, x.device)
    if spec is None and w_int is not None and need_dw and not PK.padded(sh.out_c, sh.groups):
        # a fused BatchNorm + binarizer consuming y may write this layer's gradient operand itself (fused.BNSignFn; plain
        # planes only: a group-padded dy plane is packed here)
        y._mnb_pk_conv = (w_scale if need_dx else None, Tb)
    return True


def _pk_backward(ctx, dy):
    """data and weight gradients of a layer whose forward ran on the packed-operand path"""
    from . import pk as PK
    sh = ctx.sh
    T = L.PK_TERMS_BWD     # pieces of dy and of an fp32 second operand (see _lib.PK_TERMS_BWD)
    int_w = ctx.w_int is not None
    need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    # dy is packed once for both gradients; the data gradient wants the per-channel weight scale folded in (it sits on
    # the reduction dimension there), the weight gradient divides it out again (mnb_pk_wgrad's kdiv)
    fold = int_w and need_dx
    pre = getattr(dy, "_mnb_pk_dy", None)     # written by the consumer's fused BatchNorm backward (fused.BNSignFn): dy holds no data
    if pre is not None:
        if pre[1] != T or (pre[2] is not None) != fold or PK.padded(sh.out_c, sh.groups):
            raise RuntimeError("micronet_b200: packed gradient operand does not match this layer's backward configuration")
        dy_pk = pre[0]
    else:
        dy_pk, _ = PK.pack_act(dy, None, T, ch_scale=ctx.w_scale if fold else None, groups=sh.groups)
    dx = dwq = None
    tw = 1 if int_w else T
    tx = min(ctx.pk_ta, T)     # a 3-piece saved input contributes its two leading pieces
    kdiv = ctx.w_scale if fold else None
    # a fused producer applies the STE mask itself (it owns the mask bits): plain data gradient times the quantizer's gain
    plain_gain = ctx.pk_gain if ctx.pk_prepacked else 1.0
    if need_dx:
        w_img = PK.pack_weight(sh, 1, T, tw, w_int=ctx.w_int, w_f32=None if int_w else ctx.wq,
                               kzero=ctx.w_scale if int_w else None)
        dx = torch.empty((sh.batch, sh.in_c, sh.in_h, sh.in_w), dtype=torch.float32, device=dy.device)
    if need_dx and need_dw and pre is not None and PK.bwd1x1_taken(sh, T, tx, tw):
        # 1x1 layers whose dy a fused BatchNorm + binarizer backward packed (the wbwtab graphs): both gradients in one pass
        # over dy (mnb_pk_bwd1x1).  The DoReFa graphs keep the two launches, which their span tests time kernel by kernel.
        dwq = torch.empty_like(ctx.wq)
        L.check(_timed("bwd1x1_pk", sh, lambda: PK.run_bwd(sh, dy_pk, T, ctx.pk_x, tx, w_img, tw, dx, dwq, bits8=ctx.pk_bits8,
                                                           gain=ctx.pk_gain, a_scale_const=plain_gain,
                                                           a_scale=ctx.pk_wg_scale, kdiv=kdiv)), "pk_bwd1x1")
        return dx, dwq
    if need_dx:
        L.check(_timed("dgrad_pk", sh, lambda: PK.run_conv(sh, 1, dy_pk, T, w_img, tw, dx, bits8=ctx.pk_bits8, gain=ctx.pk_gain,
                                                           a_scale_const=plain_gain)), "pk_conv dgrad")
    if need_dw:
        dwq = torch.empty_like(ctx.wq)
        L.check(_timed("wgrad_pk", sh, lambda: PK.run_wgrad(sh, dy_pk, T, ctx.pk_x, tx, dwq, a_scale=ctx.pk_wg_scale,
                                                            kdiv=kdiv)), "pk_wgrad")
    return dx, dwq


def _xnor_forward(x, w_int, w_scale, bias, sh, y, groups):
    """wbwtab inference forward on +-1 activations: bit-packed XNOR-popcount kernel where it is expected to beat the
    tensor-core forward.  Same integer sums, same fmaf epilogue: bit-identical to the packed-operand path.  Only taken
    where no backward follows (training steps multiply real-valued gradients and want the bf16 operand plane the forward
    already read), so it saves nothing."""
    from . import xnor as XN
    # Both convolution kernels are dominated by the fp32 output they write, and the popc pipe gives the bit kernel no
    # arithmetic edge over the tensor cores on +-1 operands.  The operand it reads is 16 x smaller (1 bit vs one bf16 per
    # activation), so a layer that has to pack its own input saves most of its pack pass (harness/xnor_probe.py times both
    # forms layer by layer; not yet measured on the H100).  Hence XNOR only when no producer-written plane came with x;
    # where a fused BatchNorm + binarizer already wrote the bf16 plane, the pack pass is free and the tensor-core forward
    # runs.
    if not XN.supported(sh) or getattr(x, "_mnb_pk_pm1", None) is not None:
        return False
    a_bits = XN.pack_act(materialized(x), groups)
    rc = _timed("fwd_xnor", sh, lambda: XN.conv(sh, a_bits, XN.pack_weight(sh, w_int), y, alpha=w_scale, bias=bias))
    if rc == L.E_UNSUPPORTED:
        return False
    L.check(rc, "xnor_conv_fwd")
    return True


def _save_unpacked(ctx, x, spec, codes, bits, keep_x):
    """what the backward of the round-1, fconv and generic families reads: the quantizer with its forward-time parameters
    (the forward kernel may have refreshed them), its u8 codes and STE mask bits, and the fp32 input where a kernel reads it"""
    if spec is not None and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]):
        spec = spec.frozen()
    ctx.spec, ctx.codes, ctx.bits = spec, codes, bits
    ctx.x = x if keep_x else None


def _act_operands(spec, codes, x):
    """ConvOperands with the activation side filled in: the u8 codes of the quantizer ``spec`` or the fp32 tensor x"""
    ops = L.ConvOperands()
    if codes is None:
        ops.a_f32 = x.data_ptr()
        return ops
    ops.a_codes, ops.a_offset = codes.data_ptr(), spec.code_offset
    if spec.mode == L.ACT_IAO:
        ops.a_offset_zp, ops.a_scale = L.ptr(spec.zero_point), L.ptr(spec.scale)
    elif spec.mode == L.ACT_DOREFA:
        ops.a_scale = _dorefa_scale_tensor(spec.bits, codes.device).data_ptr()
    return ops


def _tc_forward(ctx, x, w_int, w_scale, bias, spec, sh, y):
    """round-1 fused wgmma forward (mnb_fq_conv2d_fwd_tc): the activation quantizer runs inside the operand staging of the
    tensor-core conv and also writes the u8 codes and STE mask bits the backward reads.  False outside its cover."""
    lib = L.load()
    qp = codes = bits = None
    if spec is not None:
        qp = spec.struct()
        codes = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
        if ctx.needs_input_grad[0]:
            bits = torch.zeros((x.numel() + 31) // 32, dtype=torch.int32, device=x.device)
    wpack = torch.empty(w_int.numel(), dtype=torch.int16, device=x.device)
    rc = _timed("fwd_tc", sh, lambda: lib.mnb_fq_conv2d_fwd_tc(
        C.byref(sh), x.data_ptr(), None if qp is None else C.byref(qp), w_int.data_ptr(),
        w_scale.data_ptr(), L.ptr(bias), y.data_ptr(), L.ptr(codes), L.ptr(bits), wpack.data_ptr(),
        L.tc_err_flag(x.device).data_ptr(), L.stream()))
    if rc == L.E_UNSUPPORTED:
        return False
    L.check(rc, "fq_conv2d_fwd_tc")
    _save_unpacked(ctx, x, spec, codes, bits, keep_x=True)
    return True


def fconv_fwd(sh, x, w, bias, y, kind=None):
    """fp32-accurate im2col conv of an un-quantized input with few channels (first layer) on the tensor cores:
    mnb_fconv2d_fwd_wg where its plan covers the shape, mnb_fconv2d_fwd_tc otherwise (the same bits).  Returns the entry
    point's code: MNB_E_UNSUPPORTED outside both covers.  ``kind``: record the launch under it in TIMER."""
    lib = L.load()
    args = (C.byref(sh), x.data_ptr(), w.data_ptr(), L.ptr(bias), y.data_ptr(), L.tc_err_flag(x.device).data_ptr(),
            L.stream())

    def run():
        rc = lib.mnb_fconv2d_fwd_wg(*args)
        return lib.mnb_fconv2d_fwd_tc(*args) if rc == L.E_UNSUPPORTED else rc
    return run() if kind is None else _timed(kind, sh, run)


def fconv_wgrad(sh, dy, x, dw, kind=None):
    """weight gradient of the fconv_fwd layer: mnb_fconv2d_wgrad_wg where its plan covers the shape,
    mnb_fconv2d_wgrad_tc otherwise (the same bits); False where neither has a plan.  ``kind`` as for fconv_fwd."""
    lib = L.load()
    entry = lib.mnb_fconv2d_wgrad_wg
    fbytes = int(lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(sh)))
    if fbytes < 0:
        entry = lib.mnb_fconv2d_wgrad_tc
        fbytes = int(lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh)))
    if fbytes < 0:
        return False
    ws = torch.empty(max(fbytes, 4), dtype=torch.uint8, device=dy.device)

    def run():
        return entry(C.byref(sh), dy.data_ptr(), x.data_ptr(), dw.data_ptr(), ws.data_ptr(),
                     L.tc_err_flag(dy.device).data_ptr(), L.stream())
    L.check(run() if kind is None else _timed(kind, sh, run), "fconv2d_wgrad")
    return True


def _fconv_forward(ctx, x, wq, bias, sh, y):
    """un-quantized input with few channels (first layer): fconv_fwd.  False outside its cover."""
    rc = fconv_fwd(sh, x, wq, bias, y, "fconv_fwd_tc")
    if rc == L.E_UNSUPPORTED:
        return False
    L.check(rc, "fconv2d_fwd_tc")
    _save_unpacked(ctx, x, None, None, None, keep_x=True)
    return True


def _generic_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, keep_x):
    """implicit-GEMM forward of any shape (mnb_conv2d_fwd) on the codes of the standalone quantizer kernel"""
    lib = L.load()
    codes = bits = None
    if spec is not None:
        codes, bits, _ = act_quant_raw(x, spec, True, ctx.needs_input_grad[0], False)
    ops = _act_operands(spec, codes, x)
    if codes is not None and w_int is not None:
        ops.w_int, ops.w_scale = w_int.data_ptr(), w_scale.data_ptr()
    else:
        ops.w_f32 = wq.data_ptr()
    ops.bias = L.ptr(bias)
    L.check(_timed("fwd", sh, lambda: lib.mnb_conv2d_fwd(C.byref(sh), C.byref(ops), y.data_ptr(), L.stream())), "conv2d_fwd")
    _save_unpacked(ctx, x, spec, codes, bits, keep_x=keep_x or codes is None)


def _dgrad(ctx, dy, tc):
    """data gradient of an unpacked layer: mnb_conv2d_dgrad_tc first when ``tc`` (integer weights), mnb_conv2d_dgrad for
    whatever it refuses"""
    lib = L.load()
    sh, spec = ctx.sh, ctx.spec
    dx = torch.empty((sh.batch, sh.in_c, sh.in_h, sh.in_w), dtype=torch.float32, device=dy.device)
    qp = spec.struct() if spec is not None else None
    bits_ptr = ctx.bits.data_ptr() if spec is not None else None
    rc = L.E_UNSUPPORTED
    if tc:
        wpack = torch.empty(ctx.w_int.numel(), dtype=torch.int16, device=dy.device)
        rc = _timed("dgrad_tc", sh, lambda: lib.mnb_conv2d_dgrad_tc(
            C.byref(sh), dy.data_ptr(), ctx.w_int.data_ptr(), ctx.w_scale.data_ptr(), bits_ptr,
            None if qp is None else C.byref(qp), dx.data_ptr(), wpack.data_ptr(),
            L.tc_err_flag(dy.device).data_ptr(), L.stream()))
    if rc == L.E_UNSUPPORTED:
        rc = _timed("dgrad", sh, lambda: lib.mnb_conv2d_dgrad(
            C.byref(sh), dy.data_ptr(), ctx.wq.data_ptr(), bits_ptr, None if qp is None else C.byref(qp),
            dx.data_ptr(), L.stream()))
    L.check(rc, "conv2d_dgrad")
    return dx


def _wgrad(ctx, dy, tc):
    """weight gradient of an unpacked layer: mnb_conv2d_wgrad_tc first when ``tc`` (integer weights; raw fp32 activations
    that are not bf16-exact then take mnb_conv2d_wgrad_cond, on the device), mnb_conv2d_wgrad for whatever it refuses"""
    lib = L.load()
    sh, spec = ctx.sh, ctx.spec
    dwq = torch.empty_like(ctx.wq)
    ops = _act_operands(spec, ctx.codes, ctx.x)
    nbytes = int(lib.mnb_wgrad_scratch_bytes(C.byref(sh)))
    tbytes = int(lib.mnb_wgrad_tc_scratch_bytes(C.byref(sh))) if tc else 0
    if tbytes > 0:
        qp = spec.struct() if spec is not None else None
        ws = torch.empty(max(tbytes, nbytes, 4), dtype=torch.uint8, device=dy.device)
        inexact = torch.zeros(1, dtype=torch.int32, device=dy.device)
        rc = _timed("wgrad_tc", sh, lambda: lib.mnb_conv2d_wgrad_tc(
            C.byref(sh), dy.data_ptr(), ctx.x.data_ptr(), None if qp is None else C.byref(qp),
            dwq.data_ptr(), ws.data_ptr(), inexact.data_ptr(), L.tc_err_flag(dy.device).data_ptr(), L.stream()))
        if rc == 0:
            if spec is None:
                L.check(lib.mnb_conv2d_wgrad_cond(C.byref(sh), dy.data_ptr(), C.byref(ops), dwq.data_ptr(),
                                                  ws.data_ptr(), inexact.data_ptr(), L.stream()), "conv2d_wgrad_cond")
            return dwq
        if rc != L.E_UNSUPPORTED:
            L.check(rc, "conv2d_wgrad_tc")
    ws = torch.empty(max(nbytes, 4), dtype=torch.uint8, device=dy.device)
    L.check(_timed("wgrad", sh, lambda: lib.mnb_conv2d_wgrad(
        C.byref(sh), dy.data_ptr(), C.byref(ops), dwq.data_ptr(), ws.data_ptr(), L.stream())), "conv2d_wgrad")
    return dwq


def _fconv_wgrad(ctx, dy):
    """weight gradient on fconv_wgrad; None where it has no plan"""
    dwq = torch.empty_like(ctx.wq)
    return dwq if fconv_wgrad(ctx.sh, dy, ctx.x, dwq, "fconv_wgrad_tc") else None


class QuantConv2dFn(Function):
    """y = conv2d(Q_a(x), wq, bias) with the activation quantizer fused on the input side
    and the clip-STE fused into dgrad.  ``spec`` None => x is used as fp32 (wbwtab, a_bits=32).

    The forward picks one kernel family and records it as ``ctx.family``; the backward runs that family's gradients
    (DESIGN.md 4.9, "Dispatch")."""

    @staticmethod
    def forward(ctx, x, wq, bias, w_int, w_scale, spec, stride, padding, dilation, groups, pre_relu=False, no_grad=False,
                codes_out=False, handed=None, train_post=None):
        from . import pk as PK
        L.require_cuda(x, wq)
        assert not (pre_relu and any(ctx.needs_input_grad)), "the folded ReLU is an inference-only fusion"
        x = x.contiguous()
        wq = wq.contiguous()
        sh = _shape_struct(x.shape, wq.shape, stride, padding, dilation, groups)
        p, q = _out_hw(sh)
        y = torch.empty((x.shape[0], wq.shape[0], p, q), dtype=torch.float32, device=x.device)
        ctx.sh, ctx.wq, ctx.has_bias = sh, wq, bias is not None
        ctx.w_int, ctx.w_scale = (w_int, w_scale) if w_int is not None else (None, None)
        pk_on = L.PK_MODE != "off"
        pm1 = x.dtype == torch.float32 and getattr(x, "_mnb_pm1", False)   # exactly +-1 (a binarizer's output)
        pm1_plane = getattr(x, "_mnb_pk_pm1", None)   # that +-1 tensor as the bf16 plane a fused BatchNorm + binarizer wrote
        # producers write plain planes: a conv that reads a group-padded plane (pk.padded) packs its own
        padded_in = PK.padded(sh.in_c, sh.groups)
        plane = pm1_plane if (pm1_plane is not None and not padded_in and pm1_plane.numel() == x.numel() * 2) else None
        pkq = getattr(x, "_mnb_pk_q", None)   # operand plane written by a fused BN + ReLU + quantizer producer
        if pkq is not None and padded_in:
            raise RuntimeError("micronet_b200: a fused producer's packed output reached a conv that reads group-padded planes")
        plane_only = getattr(x, "_mnb_plane_only", False)
        if plane_only and padded_in:
            x, plane_only = materialized(x), False
        if (spec is None and w_int is not None and pm1 and not pre_relu
                and (no_grad or not any(ctx.needs_input_grad[:3])) and _xnor_forward(x, w_int, w_scale, bias, sh, y, groups)):
            family = "xnor"
        elif handed is not None:
            # a QAFT producer's epilogue (or the plane pool behind it) wrote this layer's plane and STE mask; the layer may
            # in turn write its own consumer's (train_post)
            if not _pk_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, prepacked=handed[0], prepacked_bits=handed[1],
                               train_post=train_post):
                raise RuntimeError("micronet_b200: handed-over plane in front of a conv outside the packed-operand cover")
            family = "pk"
        elif pkq is not None:
            if spec is None or spec.mode != L.ACT_DOREFA or spec.bits != pkq[1] or w_int is None:
                raise RuntimeError("micronet_b200: a fused producer's packed output reached a conv with another quantizer")
            if not _pk_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, prepacked=pkq[0]):
                raise RuntimeError("micronet_b200: fused producer output in front of a conv outside the packed-operand cover")
            family = "pk"
        elif ((pk_on and x.dtype == torch.float32 and (L.PK_MODE == "all" or spec is not None) and not plane_only
               and _pk_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, pre_relu=pre_relu, train_post=train_post))
              # wbwtab layer behind a fused BatchNorm + binarizer: +-1 input (one exact bf16 piece).  With the producer's
              # plane the layer is pure TMA -> MMA; 3x3 layers win on the packed-operand family even when they pack
              # themselves (measured per layer, DESIGN.md 6).  Outside the cover: the round-1 fused kernels below.
              # Group-padded layers (no producer plane, no round-1 cover) take it too
              or (L.PK_WBWTAB and pk_on and spec is None and w_int is not None and pm1
                  and (pm1_plane is not None or sh.ker_h * sh.ker_w > 1 or padded_in)
                  and _pk_forward(ctx, x, wq, bias, w_int, w_scale, None, sh, y, prepacked=plane, pm1=True,
                                  codes_out=codes_out))
              # un-quantized conv behind a binarizer (the 10-way head of a wbwtab model, fused.EnginePmConv2d): the +-1
              # input is ONE exact bf16 piece - the producer's plane when it wrote one - against exact pieces of the fp32
              # weights
              or (pk_on and spec is None and w_int is None and pm1 and not pre_relu
                  and _pk_forward(ctx, x, wq, bias, None, None, None, sh, y, prepacked=plane, pm1=True))):
            family = "pk"
        else:
            # outside the packed-operand cover: the kernels below read the fp32 values, with the folded ReLU as its own pass
            if plane_only:
                x = materialized(x)
            if pre_relu:
                x = torch.relu(x)
            f32 = x.dtype == torch.float32
            if L.USE_TC and w_int is not None and f32 and _tc_forward(ctx, x, w_int, w_scale, bias, spec, sh, y):
                family = "tc"
            elif L.USE_TC and spec is None and f32 and _fconv_forward(ctx, x, wq, bias, sh, y):
                family = "fconv"
            elif pk_on and f32 and _pk_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y):
                family = "pk"
            else:
                # the round-1 backward kernels also cover shapes whose forward they refuse (the data gradient reads K
                # channels and writes C): with integer weights the layer takes the round-1 backward
                tc = L.USE_TC and w_int is not None
                _generic_forward(ctx, x, wq, bias, w_int, w_scale, spec, sh, y, keep_x=tc)
                family = "tc" if tc else "generic"
        ctx.family = family
        return y

    @staticmethod
    def backward(ctx, dy):
        # a fused BatchNorm+binarize consumer already reduced its dx (= this dy) over (B, H, W): fused.BNSignFn
        presummed = getattr(dy, "_mnb_channel_sum", None)
        dy = dy.contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        db = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = presummed if presummed is not None and presummed.numel() == dy.shape[1] else channel_sums(dy)
        dx = dwq = None
        if ctx.family == "pk":
            dx, dwq = _pk_backward(ctx, dy)
        elif ctx.family == "tc":
            dx = _dgrad(ctx, dy, tc=True) if need_dx else None
            dwq = _wgrad(ctx, dy, tc=True) if need_dw else None
        elif ctx.family == "fconv":
            # integer weights (a wbwtab layer the round-1 forward refused): the round-1 kernels may still take the gradients
            tc = ctx.w_int is not None
            dx = _dgrad(ctx, dy, tc) if need_dx else None
            if need_dw:
                dwq = _fconv_wgrad(ctx, dy)
                if dwq is None:
                    dwq = _wgrad(ctx, dy, tc)
        else:
            dx = _dgrad(ctx, dy, tc=False) if need_dx else None
            dwq = _wgrad(ctx, dy, tc=False) if need_dw else None
        return dx, dwq, db, None, None, None, None, None, None, None, None, None, None, None, None


def quant_conv2d(x, wq, bias, w_int, w_scale, spec, stride, padding, dilation, groups, pre_relu=False, codes_out=False,
                 handed=None, train_post=None):
    """``handed`` / ``train_post``: the two ends of a QAFT hand-off (QuantConv2dFn, _pk_forward)"""
    # (autograd runs a Function's forward with grad mode off and needs_input_grad ignores torch.no_grad(): whether this call
    # will ever be differentiated is only known out here)
    return QuantConv2dFn.apply(x, wq, bias, w_int, w_scale, spec, tuple(stride), tuple(padding),
                               tuple(dilation), groups, pre_relu, not torch.is_grad_enabled(), codes_out, handed, train_post)


# --------------------------------------------------------------------------
# transposed convolution (IAO.QuantConvTranspose2d, IAO:510-636)
# --------------------------------------------------------------------------
def _pk_plain(sh, mode, a, w, out, T):
    """fp32 x fp32 convolution (mode 0) / data gradient (mode 1) of shape ``sh`` on the packed-operand tensor-core family:
    both operands as T exact bf16 pieces.  False when the shape is outside its cover."""
    from . import pk as PK
    # (group-padded shapes keep the generic kernels here: the transposed conv's planes are not packed group-padded)
    if L.PK_MODE == "off" or PK.padded_conv(sh) or not PK.supported(sh, mode, T, T):
        return False
    a_pk, _ = PK.pack_act(a, None, T, phase_split=(mode == 0 and sh.stride_h == 2))
    w_img = PK.pack_weight(sh, mode, T, T, w_f32=w)
    rc = _timed("fwd_pk" if mode == 0 else "dgrad_pk", sh, lambda: PK.conv(sh, mode, a_pk, T, w_img, T, out))
    if rc == L.E_UNSUPPORTED:
        return False
    L.check(rc, "pk_conv (plain)")
    return True


class ConvTranspose2dFn(Function):
    """y = F.conv_transpose2d(x, w, bias, stride, padding, output_padding, groups, dilation) on the engine's convolution
    kernels.  A transposed convolution IS the data gradient of the convolution S that maps y-space to x-space (w is
    already stored as S's weight [K = C_in][C_out / g][R][S]):

        forward   y  = dgrad_S(dy := x, w)            backward  dx = fwd_S(gy, w),  dw = wgrad_S(x := gy, dy := x)

    so the three kernels of QuantConv2dFn serve it with the roles swapped: the packed-operand tensor-core family where it
    has cover (exact bf16 pieces of the fp32 operands), the generic implicit-GEMM kernels elsewhere."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, padding, output_padding, groups, dilation):
        L.require_cuda(x, w)
        L.require_f32(x, w)
        lib = L.load()
        x, w = x.contiguous(), w.contiguous()
        b, cin, h, wd = x.shape
        if w.shape[0] != cin or cin % groups:
            raise ValueError("conv_transpose2d: weight must be [C_in, C_out / groups, R, S]")
        cout = w.shape[1] * groups
        oh = (h - 1) * stride[0] - 2 * padding[0] + dilation[0] * (w.shape[2] - 1) + output_padding[0] + 1
        ow = (wd - 1) * stride[1] - 2 * padding[1] + dilation[1] * (w.shape[3] - 1) + output_padding[1] + 1
        sh = _shape_struct((b, cout, oh, ow), w.shape, stride, padding, dilation, groups)
        if _out_hw(sh) != (h, wd):
            raise ValueError("conv_transpose2d: output_padding must be smaller than the stride")
        y = torch.empty((b, cout, oh, ow), dtype=torch.float32, device=x.device)
        if not _pk_plain(sh, 1, x, w, y, L.PK_TERMS):
            L.check(_timed("dgrad", sh, lambda: lib.mnb_conv2d_dgrad(C.byref(sh), x.data_ptr(), w.data_ptr(), None, None,
                                                                      y.data_ptr(), L.stream())), "conv2d_dgrad")
        if bias is not None:
            y += bias.view(1, -1, 1, 1)
        ctx.save_for_backward(x, w)
        ctx.sh, ctx.has_bias = sh, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        from . import pk as PK
        lib = L.load()
        x, w = ctx.saved_tensors
        sh = ctx.sh
        gy = gy.contiguous()
        gx = gw = gb = None
        T = L.PK_TERMS_BWD
        if ctx.needs_input_grad[0]:
            gx = torch.empty_like(x)
            if not _pk_plain(sh, 0, gy, w, gx, T):
                ops = L.ConvOperands()
                ops.a_f32, ops.w_f32 = gy.data_ptr(), w.data_ptr()
                L.check(_timed("fwd", sh, lambda: lib.mnb_conv2d_fwd(C.byref(sh), C.byref(ops), gx.data_ptr(), L.stream())),
                        "conv2d_fwd")
        if ctx.needs_input_grad[1]:
            gw = torch.empty_like(w)
            done = False
            if L.PK_MODE != "off" and not PK.padded_conv(sh) and PK.wgrad_supported(sh, T, T):
                x_pk, _ = PK.pack_act(x, None, T)                                   # S's output-gradient operand
                g_pk, _ = PK.pack_act(gy, None, T, phase_split=sh.stride_h == 2)    # S's input operand
                rc = _timed("wgrad_pk", sh, lambda: PK.wgrad(sh, x_pk, T, g_pk, T, gw))
                if rc != L.E_UNSUPPORTED:
                    L.check(rc, "pk_wgrad (transposed conv)")
                    done = True
            if not done:
                ops = L.ConvOperands()
                ops.a_f32 = gy.data_ptr()
                ws = torch.empty(max(int(lib.mnb_wgrad_scratch_bytes(C.byref(sh))), 4), dtype=torch.uint8, device=gy.device)
                L.check(_timed("wgrad", sh, lambda: lib.mnb_conv2d_wgrad(C.byref(sh), x.data_ptr(), C.byref(ops), gw.data_ptr(),
                                                                         ws.data_ptr(), L.stream())), "conv2d_wgrad")
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = channel_sums(gy)
        return gx, gw, gb, None, None, None, None, None


def conv_transpose2d(x, w, bias, stride, padding, output_padding, groups, dilation):
    return ConvTranspose2dFn.apply(x, w, bias, tuple(stride), tuple(padding), tuple(output_padding), groups, tuple(dilation))


# --------------------------------------------------------------------------
# frozen inference graphs (iao.freeze_inference): producer -> consumer hand-off of packed operand planes
# --------------------------------------------------------------------------
class Consumer:
    """the quantized conv that reads a producer's output next (set up by iao.freeze_inference): its frozen activation
    quantizer, the nn.ReLU in between (folded away), its geometry, whether anybody else needs the fp32 tensor, and
    whether it was frozen with int8 operands (``int8``: then ``format`` tells which plane it reads)"""

    def __init__(self, module, spec, relu, only, w_shape, stride, padding, dilation, groups, int_weights, int8=False, bn=None,
                 shuffle_groups=1, pool=None, post_spec=None, formats=None):
        self.module, self.spec, self.relu, self.only = module, spec, bool(relu), bool(only)
        self.w_shape, self.stride, self.padding, self.dilation, self.groups = w_shape, stride, padding, dilation, groups
        self.int_weights, self.int8 = int_weights, bool(int8)
        # DoReFa graphs (dorefa.freeze_inference): the eval BatchNorm (mean, invstd, gamma, beta) the producer's epilogue applies
        # before the ReLU, the consumer block's channel shuffle, and a max-pool in between: pool = (module, k, s, p), run as
        # mnb_pk_plane_maxpool on the producer's full-resolution plane, so the producer tags its output for that module
        self.bn, self.sg, self.pool = bn, int(shuffle_groups), pool
        self.target = module if pool is None else pool[0]
        # the quantizer whose levels the producer writes: the consumer's own, or - IAO graphs (iao.freeze_inference) - that of
        # the QuantMaxPool2d in between, whose pool kernel requantizes them to the consumer's (mnb_pk_plane_maxpool_requant)
        self.post_spec = spec if post_spec is None else post_spec
        # the plane formats this link hands over (None: any); for any other format the producer writes fp32
        self.formats = formats

    def read_shape(self, out_shape):
        """the activation the consumer reads when the producer writes ``out_shape``"""
        if self.pool is None:
            return tuple(out_shape)
        _, k, s, p = self.pool
        b, c, h, w = out_shape
        return (b, c, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)

    def format(self, out_shape):
        """operand plane the consumer's forward reads for this producer output: "i8" (int8 conv), "bf16" (packed-operand conv
        with a one-piece plane) or None (a producer cannot write its operand).  frozen_conv takes the same decision."""
        act_shape = self.read_shape(out_shape)
        if self.sg > 1 and (out_shape[1] % 16 or out_shape[1] % self.sg or self.split):
            return None       # the epilogue stores a shuffled plane of whole units only, never phase-split
        fmt = None
        if self.int8 and act_shape[1] == self.w_shape[1] * self.groups:
            sh = _shape_struct(act_shape, self.w_shape, self.stride, self.padding, self.dilation, self.groups)
            if _i8_route(self.spec, self.int_weights, sh):
                fmt = "i8"
        if fmt is None and self.accepts(act_shape):
            fmt = "bf16"
        return fmt if self.formats is None or fmt in self.formats else None

    def accepts(self, act_shape):
        """will the consumer's forward run on the packed-operand family with a one-piece plane of this activation?"""
        from . import pk as PK
        sp = self.spec
        if sp is None or not self.int_weights or not (2 <= sp.bits <= 8) or _pk_terms(sp, True)[0] != 1:
            return False
        if act_shape[1] != self.w_shape[1] * self.groups:
            return False
        if PK.padded(act_shape[1], self.groups):     # producers write plain planes; this conv reads a group-padded one
            return False
        sh = _shape_struct(act_shape, self.w_shape, self.stride, self.padding, self.dilation, self.groups)
        if sh.stride_h == 2 and ((act_shape[2] | act_shape[3]) & 1):
            return False
        return L.PK_MODE != "off" and PK.supported(sh, 0, 1, 1)

    @property
    def split(self):
        return self.stride[0] == 2 and self.pool is None


def train_consumer_ok(consumer, out_shape):
    """can a QAFT producer writing ``out_shape`` hand ``consumer`` its plane?  The consumer's forward takes a one-piece plane
    of the activation it reads (Consumer.accepts) and its data and weight gradients stay on the packed-operand family."""
    from . import pk as PK
    act = consumer.read_shape(out_shape)
    if not consumer.accepts(act):
        return False
    sh = _shape_struct(act, consumer.w_shape, consumer.stride, consumer.padding, consumer.dilation, consumer.groups)
    Tb = L.PK_TERMS_BWD
    return PK.supported(sh, 1, Tb, 1) and PK.wgrad_supported(sh, Tb, 1)


def handed_train(module, x):
    """(plane, STE mask) a QAFT producer wrote for ``module`` when ``x`` is its tagged output, else None"""
    plane = handed_plane(module, x)
    return None if plane is None or "bits" not in x._mnb_pk_pre[4] else (plane, x._mnb_pk_pre[4]["bits"])


class PlanePoolFn(Function):
    """the QuantMaxPool2d between two linked blocks of a QAFT step (iao.prepare(fuse=True)) on the producer's plane of the
    pool quantizer's levels: max-pool, window indices, requantization to the consumer's levels and their STE mask in one
    kernel (mnb_pk_plane_maxpool_requant_train); the returned tensor is a shape-carrying placeholder tagged with that plane
    for ``target``.  Backward: max_pool2d, ActQuantFn and nn.ReLU backward in one kernel (mnb_pk_plane_maxpool_requant_bwd)."""

    @staticmethod
    def forward(ctx, x, plane, bits, k, s, p, spec_p, spec_c, target):
        from . import pk as PK
        b, c, h, w = x.shape
        q_in = spec_p.frozen()     # the pool's backward sees the forward-time scale, as ActQuantFn's does
        out, arg, cbits = _timed("plane_pool", L.ConvShape(b, c, h, w, c, k, k, s, s, p, p, 1, 1, 1),
                                 lambda: PK.plane_maxpool_requant_train(plane, b, c, h, w, k, s, p, q_in.struct(),
                                                                        spec_c.struct()))
        y = torch.empty((b, c, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1), dtype=torch.float32, device=x.device)
        ctx.arg, ctx.bits, ctx.spec, ctx.cfg = arg, bits, q_in, (b, c, h, w, k, s, p)
        return tag(y, target, out, "bf16", bits=cbits)

    @staticmethod
    def backward(ctx, g):
        from . import pk as PK
        b, c, h, w, k, s, p = ctx.cfg
        qp = ctx.spec.struct()
        dx = _timed("plane_pool_bwd", L.ConvShape(b, c, h, w, c, k, k, s, s, p, p, 1, 1, 1),
                    lambda: PK.plane_maxpool_requant_bwd(g.contiguous(), ctx.arg, ctx.bits, b, c, h, w, k, s, p, qp))
        return dx, None, None, None, None, None, None, None, None


DECODABLE = ("bits", "b1", "terms")     # plane formats materialized decodes; level planes ("bf16", "i8") it cannot


def tag(y, target, plane, fmt, **meta):
    """tag producer output ``y`` with the plane it wrote for module ``target``, in format ``fmt`` ("bf16" / "i8" level
    planes, "bits" / "b1" planes with their ``groups``, "terms" planes with ``split`` and ``terms``)"""
    y._mnb_pk_pre = (target, plane, y._version, fmt, meta)
    return y


def handed_plane(module, x):
    """the plane a frozen producer wrote for ``module`` when ``x`` is that producer's output, else None.  The plane goes
    to its target only, at the groups it was packed for (bit / b1 planes), and, for an output that also holds values (a
    tagged fp32 tensor), only while ``x._version`` is the one it was tagged at.  A meta-shaped output holds nothing but its
    plane, so no in-place write can make the two disagree: its version is not checked.  A meta-shaped output that
    reaches another module raises unless its plane decodes (functional.materialized: bit, b1 and term planes)."""
    pre = getattr(x, "_mnb_pk_pre", None)
    meta = x.device.type == "meta"
    if pre is not None:
        target, plane, version, fmt, info = pre
        g = info.get("groups")
        if target is module and (meta or x._version == version) and (g is None or getattr(module, "groups", g) == g):
            return plane
    if meta and (pre is None or pre[3] not in DECODABLE):
        raise RuntimeError("micronet_b200: a plane-only producer output reached a module it was not produced for")
    return None


def _i8_route(spec, w_int, sh):
    """does a conv frozen with int8=True run this forward on the int8 kernels?  Symmetric IAO activations with 2..8 bits
    and levels in [-128, 127] (the quantizer test of the C side: an asymmetric quantizer reports q_type 0 until its first
    update_qparams, its level range tells) or DoReFa activations with 2..7 bits (levels 0 .. 2^a - 1), integer weights (the
    module checks they fit s8) and a shape the int8 plan takes; everything else keeps the bf16 path."""
    from . import pk as PK
    if spec is None or w_int is None or L.PK_MODE == "off":
        return False
    if spec.mode == L.ACT_DOREFA:
        ok = 2 <= spec.bits <= 7
    else:
        ok = spec.mode == L.ACT_IAO and spec.q_type == 0 and 2 <= spec.bits <= 8 and -128 <= spec.qmin and spec.qmax <= 127
    return ok and PK.i8_supported(sh)


def _i8_producer_writes_plane(out_channels, groups):
    """can an int8 conv's epilogue write its consumer's int8 plane?  It stores whole 16-channel units, so every N tile
    must start on one: a grouped producer needs output channels per group % 16 == 0 (mnb_pk_i8_conv refuses others)"""
    return groups == 1 or (out_channels // groups) % 16 == 0


@torch.no_grad()
def frozen_conv(x, plane, wq, bias, w_int, w_scale, spec, stride, padding, dilation, groups, pre_relu=False, consumer=None,
                int8=False):
    """eval forward of a frozen quantized conv.  ``plane``: operand plane its producer already wrote (x holds no data
    then); ``consumer``: write the next conv's plane from the epilogue (mnb_pk_conv_post); ``int8``: the module was frozen
    with int8 operands (the int8 kernels run where _i8_route allows)."""
    from . import pk as PK
    stride, padding, dilation = tuple(stride), tuple(padding), tuple(dilation)
    sh = _shape_struct(x.shape, wq.shape, stride, padding, dilation, groups)
    p, q = _out_hw(sh)
    out_shape = (x.shape[0], wq.shape[0], p, q)
    fmt = "i8" if int8 and _i8_route(spec, w_int, sh) else "bf16"
    if plane is not None and x._mnb_pk_pre[3] != fmt:
        raise RuntimeError(f"micronet_b200: a {x._mnb_pk_pre[3]} operand plane reached a conv that reads {fmt}")
    # a producer hands its consumer a plane only when both run the same format; otherwise the consumer packs its own
    cfmt = consumer.format(out_shape) if consumer is not None else None
    if fmt == "i8":
        hand = cfmt == "i8" and _i8_producer_writes_plane(wq.shape[0], groups)
        return _frozen_conv_i8(x, plane, bias, w_int, w_scale, spec, sh, out_shape, pre_relu, consumer if hand else None)
    ta, tw = _pk_terms(spec, w_int)
    # a segmented producer plan (two level pieces of an asymmetric quantizer) takes no fused consumer: the consumer packs
    # its own operand from y.  Nor does a grouped producer with output channels per group % 8 != 0 (mnb_pk_conv_post stores
    # whole octets of a group)
    fused = cfmt == "bf16" and not PK.segmented(sh, 0, ta, tw) and not PK.padded(sh.out_c, groups)
    if (plane is None and not fused) or spec is None or w_int is None or L.PK_MODE == "off" or not PK.supported(sh, 0, ta, tw):
        if plane is not None:
            raise RuntimeError("micronet_b200: handed-over plane in front of a conv outside the packed-operand cover")
        return quant_conv2d(x, wq, bias, w_int, w_scale, spec, stride, padding, dilation, groups, pre_relu=pre_relu)
    dev = wq.device
    if plane is None:
        L.require_cuda(x, wq)
        plane, _ = PK.pack_act(x.contiguous(), spec.struct(), ta, phase_split=sh.stride_h == 2, relu=pre_relu, groups=groups)
    w_img = PK.weight_image(sh, ta, tw, w_int=w_int)
    a_scale, a_const = PK.act_scale(spec)
    if not fused:
        y = torch.empty(out_shape, dtype=torch.float32, device=dev)
        L.check(_timed("fwd_pk", sh, lambda: PK.conv(sh, 0, plane, ta, w_img, tw, y, n_scale=w_scale, a_scale=a_scale,
                                                     a_scale_const=a_const, bias=bias)), "pk_conv fwd")
        return y
    y = None if consumer.only else torch.empty(out_shape, dtype=torch.float32, device=dev)
    cplane = PK.consumer_plane(*out_shape, dev)
    cqp = consumer.post_spec.struct()
    L.check(_timed("fwd_pk", sh, lambda: PK.conv_post(sh, plane, ta, w_img, tw, y, cqp, cplane, consumer.relu, consumer.split,
                                                      n_scale=w_scale, a_scale=a_scale, a_scale_const=a_const, bias=bias,
                                                      bn=consumer.bn, shuffle_groups=consumer.sg)),
            "pk_conv_post")
    if y is None:
        y = torch.empty(out_shape, dtype=torch.float32, device="meta")   # shape only: the data lives in the consumer's plane
    return tag(y, consumer.target, cplane, "bf16")


def _frozen_conv_i8(x, plane, bias, w_int, w_scale, spec, sh, out_shape, pre_relu, consumer):
    """frozen_conv on the int8 kernels (mnb_pk_i8_*); ``consumer``: an int8 consumer whose plane the epilogue writes"""
    from . import pk as PK
    dev = w_int.device
    if plane is None:
        L.require_cuda(x, w_int)
        plane = PK.pack_act_i8(x.contiguous(), spec.struct(), phase_split=sh.stride_h == 2, relu=pre_relu)
    w_img = PK.weight_image(sh, w_int=w_int, i8=True)
    a_scale, a_const = PK.act_scale(spec)
    if consumer is None:
        y = torch.empty(out_shape, dtype=torch.float32, device=dev)
        L.check(_timed("fwd_pk_i8", sh, lambda: PK.conv_i8(sh, plane, w_img, y, n_scale=w_scale, a_scale=a_scale,
                                                           a_scale_const=a_const, bias=bias)), "pk_i8_conv")
        return y
    y = None if consumer.only else torch.empty(out_shape, dtype=torch.float32, device=dev)
    cplane = PK.consumer_plane_i8(*out_shape, dev)
    post = (consumer.post_spec.struct(), cplane, consumer.relu, consumer.split, consumer.bn, consumer.sg)
    L.check(_timed("fwd_pk_i8", sh, lambda: PK.conv_i8(sh, plane, w_img, y, n_scale=w_scale, a_scale=a_scale,
                                                       a_scale_const=a_const, bias=bias, post=post)), "pk_i8_conv")
    if y is None:
        y = torch.empty(out_shape, dtype=torch.float32, device="meta")
    return tag(y, consumer.target, cplane, "i8")


@torch.no_grad()
def frozen_quant_add(a, b, spec, relu, consumer=None):
    """eval forward of a frozen QuantAdd; with a ``consumer`` the kernel also writes the next conv's operand plane, in the
    format that conv reads (bf16 or int8)"""
    cfmt = consumer.format(tuple(a.shape)) if consumer is not None and a.dim() == 4 else None
    if cfmt is None:
        return QuantAddFn.apply(a, b, spec, relu)
    from . import pk as PK
    L.require_cuda(a, b)
    lib = L.load()
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape, "QuantAdd: operand shapes differ"
    out = torch.empty_like(a)
    i8 = cfmt == "i8"
    cplane = (PK.consumer_plane_i8 if i8 else PK.consumer_plane)(*a.shape, a.device)
    qp, cqp = spec.struct(), consumer.spec.struct()
    post = L.PkPost(C.pointer(cqp), 1 if (consumer.relu and not relu) else 0, 1 if consumer.split else 0, cplane.data_ptr())
    fn = lib.mnb_quant_add_pack_i8_fwd if i8 else lib.mnb_quant_add_pack_fwd
    L.check(fn(a.data_ptr(), b.data_ptr(), a.shape[0], a.shape[1], a.shape[2], a.shape[3], C.byref(qp), 1 if relu else 0,
               out.data_ptr(), C.byref(post), L.stream()), "quant_add_pack_i8_fwd" if i8 else "quant_add_pack_fwd")
    return tag(out, consumer.target, cplane, cfmt)


def quant_linear(x, wq, bias, w_int, w_scale, spec):
    """F.linear on the same kernels: [*, C] -> 1x1 conv on a [N, C, 1, 1] view."""
    lead = x.shape[:-1]
    x4 = x.reshape(-1, x.shape[-1], 1, 1)
    w4 = wq.reshape(wq.shape[0], wq.shape[1], 1, 1)
    wi4 = None if w_int is None else w_int.reshape(w4.shape)
    y = QuantConv2dFn.apply(x4, w4, bias, wi4, w_scale, spec, (1, 1), (0, 0), (1, 1), 1)
    return y.reshape(*lead, wq.shape[0])


class BNFoldFn(Function):
    """IAO:903-945: (weight, bias) with the BatchNorm statistics folded in, one kernel each way"""

    @staticmethod
    def forward(ctx, weight, bias, gamma, beta, mean, var, eps):
        L.require_cuda(weight, gamma)
        lib = L.load()
        weight = weight.contiguous()
        k, n = weight.shape[0], weight.numel() // weight.shape[0]
        mean, var = mean.contiguous(), var.contiguous()
        w_f = torch.empty_like(weight)
        b_f = torch.empty(k, dtype=torch.float32, device=weight.device)
        L.check(lib.mnb_bn_fold_fwd(weight.data_ptr(), k, n, gamma.data_ptr(), beta.data_ptr(), L.ptr(bias), mean.data_ptr(),
                                    var.data_ptr(), float(eps), w_f.data_ptr(), b_f.data_ptr(), L.stream()), "bn_fold_fwd")
        ctx.save_for_backward(weight, bias, gamma, mean, var)
        ctx.eps = eps
        return w_f, b_f

    @staticmethod
    def backward(ctx, dw_f, db_f):
        lib = L.load()
        weight, bias, gamma, mean, var = ctx.saved_tensors
        k, n = weight.shape[0], weight.numel() // weight.shape[0]
        if dw_f is None:
            dw_f = torch.zeros_like(weight)
        dw_f = dw_f.contiguous()
        db_f = None if db_f is None else db_f.contiguous()
        dw = torch.empty_like(weight) if ctx.needs_input_grad[0] else None
        out6 = torch.empty((k, 6), dtype=torch.float32, device=weight.device)
        L.check(lib.mnb_bn_fold_bwd(dw_f.data_ptr(), L.ptr(db_f), weight.data_ptr(), k, n, gamma.data_ptr(), L.ptr(bias),
                                    mean.data_ptr(), var.data_ptr(), float(ctx.eps), L.ptr(dw), out6.data_ptr(), L.stream()),
                "bn_fold_bwd")
        g = ctx.needs_input_grad
        return (dw, out6[:, 2] if (bias is not None and g[1]) else None, out6[:, 0] if g[2] else None,
                out6[:, 1] if g[3] else None, out6[:, 3] if g[4] else None, out6[:, 4] if g[5] else None, None)


# --------------------------------------------------------------------------
# per-channel batch statistics (BN-fuse training path, IAO:853-855)
# --------------------------------------------------------------------------
class ChannelMeanVarFn(Function):
    @staticmethod
    def forward(ctx, x):
        L.require_cuda(x)
        lib = L.load()
        x = x.contiguous()
        b, c = x.shape[0], x.shape[1]
        hw = x.numel() // (b * c)
        out = torch.empty(2 * c, dtype=torch.float32, device=x.device)
        L.check(lib.mnb_channel_stats(x.data_ptr(), b, c, hw, 1, out.data_ptr(),
                                      L.scratch(x.device, c).data_ptr(), L.stream()), "channel_stats")
        mean, var = out[:c], out[c:]
        ctx.save_for_backward(x, mean)
        return mean, var

    @staticmethod
    def backward(ctx, dmean, dvar):
        lib = L.load()
        x, mean = ctx.saved_tensors
        b, c = x.shape[0], x.shape[1]
        hw = x.numel() // (b * c)
        dmean = torch.zeros_like(mean) if dmean is None else dmean.contiguous()
        dvar = torch.zeros_like(mean) if dvar is None else dvar.contiguous()
        dx = torch.empty_like(x)
        L.check(lib.mnb_channel_stats_bwd(x.data_ptr(), mean.contiguous().data_ptr(), dmean.data_ptr(),
                                          dvar.data_ptr(), b, c, hw, dx.data_ptr(), L.stream()),
                "channel_stats_bwd")
        return dx


def channel_mean_var(x):
    return ChannelMeanVarFn.apply(x)
