"""Python side of the packed-operand tensor-core family (``csrc/mnb_pk.cu``).

Every conv of the QAT models that the fused kernels of ``mnb_conv_tc_*.cu`` cannot take (weights that do not fit in
shared memory, stride 2, 5x5 filters, 4x4 or 224x224 images ...) and every fused-quantizer layer runs here:

    pack_act    fp32 NCHW -> bf16 term planes [t][b][c/8][h][w][8] (fake-quantize, or exact split of an fp32 tensor)
    pack_weight integer levels / fp32 weights -> the bf16 operand image of one (shape, mode)
    conv        TMA -> wgmma (register accumulators) -> epilogue (forward: scale + bias; data gradient: STE mask)
    wgrad       the same boxes read as MN-major operands, split over the batch, deterministic reduction
    wgrad_taps  wgrad of narrow grouped 3x3 layers with all nine taps of a CTA in registers
    gc3_conv    forward / data gradient of the same layers with whole images as M tiles (same result as conv)
    bwd1x1      data gradient and weight gradient of a 1x1 layer in one pass over dy (same results as conv + wgrad)

The layers of the engine go through run_conv / run_conv_codes / run_wgrad / run_bwd, which pick among those kernels
(``PK_GC3``, ``PK_WG_TAPS``, ``PK_BWD1X1``); the single-kernel calls stay for tests and probes that compare the kernels directly.

Reference math: F.conv2d of the fake-quantized tensors (WB:186, DF:113, IAO:498/843/947) and ATen's
convolution_backward."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L

_plan_cache = {}


def _key(sh):
    return tuple(getattr(sh, f) for f, _ in sh._fields_)


def supported(sh, mode, terms_a, terms_w):
    """does mnb_pk_conv cover this (shape, mode)?  (host-only plan query, cached)"""
    k = ("c", _key(sh), mode, terms_a, terms_w)
    if k not in _plan_cache:
        _plan_cache[k] = L.load().mnb_pk_conv_plan(C.byref(sh), mode, terms_a, terms_w, None) == 0
    return _plan_cache[k]


def segmented(sh, mode, terms_a, terms_w):
    """does the plan run segmented accumulation (several piece products per K-step, long K loop)?  Such plans take no
    fused consumer (mnb_pk_conv_post refuses them).  Host-only plan query, cached."""
    k = ("s", _key(sh), mode, terms_a, terms_w)
    if k not in _plan_cache:
        out = (C.c_int32 * 17)()
        _plan_cache[k] = L.load().mnb_pk_conv_plan_ex(C.byref(sh), mode, terms_a, terms_w, out, 17) == 0 and out[16] != 0
    return _plan_cache[k]


def wgrad_supported(sh, terms_dy, terms_x):
    k = ("w", _key(sh), terms_dy, terms_x)
    if k not in _plan_cache:
        _plan_cache[k] = int(L.load().mnb_pk_wgrad_scratch_bytes(C.byref(sh), terms_dy, terms_x))
    return _plan_cache[k] >= 0


def padded(channels, groups):
    """is the operand plane of a grouped conv reading ``channels`` channels group-padded (DESIGN.md 4.17)?  Then its
    layout differs from a plain plane of the same tensor, and no plane in the plain layout may be handed to that conv."""
    return groups > 1 and (channels // groups) % 8 != 0


def padded_conv(sh):
    """does any operand plane of conv ``sh`` (x: input channels per group, dy: output channels per group) use the padded layout?"""
    return padded(sh.in_c, sh.groups) or padded(sh.out_c, sh.groups)


def pack_act(x, qp, terms, ch_scale=None, phase_split=False, want_bits=False, relu=False, groups=1):
    """-> (planes u8[terms * B * ceil(C/8) * H * W * 16], bits8 u8[B, ceil(C/8), H, W] or None).  ``groups``: the plane is the
    operand of a grouped conv; group-padded (mnb_pk_pack_act_grouped) where C / groups % 8 != 0, the plain plane otherwise."""
    lib = L.load()
    b, c, h, w = x.shape
    pad = padded(c, groups)
    c8 = groups * ((c // groups + 7) // 8) if pad else (c + 7) // 8
    nbytes = int(lib.mnb_pk_grouped_act_bytes(b, c, h, w, terms, groups) if pad else lib.mnb_pk_act_bytes(b, c, h, w, terms))
    out = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    bits = None
    if qp is not None and want_bits:
        bits = torch.empty((b, c8, h, w), dtype=torch.uint8, device=x.device)
    args = (x.data_ptr(), b, c, h, w, None if qp is None else C.byref(qp), terms, L.ptr(ch_scale), 1 if phase_split else 0,
            1 if relu else 0, out.data_ptr(), L.ptr(bits))
    if pad:
        L.check(lib.mnb_pk_pack_act_grouped(*args, groups, L.stream()), "pk_pack_act_grouped")
    else:
        L.check(lib.mnb_pk_pack_act_relu(*args, L.stream()), "pk_pack_act")
    return out, bits


def pack_weight(sh, mode, terms_a, terms_w, w_int=None, w_f32=None, kzero=None):
    lib = L.load()
    nbytes = int(lib.mnb_pk_wimage_bytes(C.byref(sh), mode, terms_a, terms_w))
    if nbytes < 0:
        raise ValueError("micronet_b200.pk: shape outside the cover of the packed-operand convolution")
    dev = (w_int if w_int is not None else w_f32).device
    img = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    L.check(lib.mnb_pk_pack_weight(C.byref(sh), mode, terms_a, terms_w, L.ptr(w_int), L.ptr(w_f32), L.ptr(kzero),
                                   img.data_ptr(), L.stream()), "pk_pack_weight")
    return img


def weight_image(sh, terms_a=1, terms_w=1, w_int=None, w_f32=None, i8=False):
    """forward weight image of pack_weight (or of pack_weight_i8 with ``i8``).  Frozen (inference) modules hang a dict
    ``_mnb_pk_cache`` on their cached weight tensor: the image is then built once per shape."""
    src = w_int if w_int is not None else w_f32
    cache = getattr(src, "_mnb_pk_cache", None)
    key = (_key(sh), "i8") if i8 else (_key(sh), terms_a, terms_w)
    img = cache.get(key) if cache is not None else None
    if img is None:
        img = pack_weight_i8(sh, w_int) if i8 else pack_weight(sh, 0, terms_a, terms_w, w_int=w_int, w_f32=w_f32)
        if cache is not None:
            cache[key] = img
    return img


def act_scale(spec, clone=False):
    """(a_scale, a_scale_const) of the forward epilogues for the activation quantizer ``spec`` (functional.ActSpec or None):
    IAO's device scalar - a private copy with ``clone``, for a backward that must see the forward-time scale - or DoReFa's
    1 / (2^a - 1)"""
    if spec is not None and spec.mode == L.ACT_IAO:
        return (spec.scale.clone() if clone else spec.scale), 1.0
    if spec is not None and spec.mode == L.ACT_DOREFA:
        return None, 1.0 / float(2 ** spec.bits - 1)
    return None, 1.0


def conv(sh, mode, a_pk, terms_a, w_img, terms_w, out, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None,
         bits8=None, gain=1.0):
    lib = L.load()
    return lib.mnb_pk_conv(C.byref(sh), mode, a_pk.data_ptr(), terms_a, w_img.data_ptr(), terms_w, L.ptr(n_scale),
                           L.ptr(a_scale), float(a_scale_const), L.ptr(bias), L.ptr(bits8), float(gain), out.data_ptr(),
                           L.tc_err_flag(out.device).data_ptr(), L.stream())


def conv_codes(sh, a_pk, w_img, codes, dec, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None, level_bound=1):
    """forward conv of one +-1 piece against one piece of integer weight levels (|level| <= level_bound) whose exact sums go
    out as int16 ``codes`` plus the epilogue's decode pair ``dec`` [2, K] (mnb_pk_conv_codes); returns the C status"""
    return L.load().mnb_pk_conv_codes(C.byref(sh), a_pk.data_ptr(), 1, w_img.data_ptr(), 1, L.ptr(n_scale), L.ptr(a_scale),
                                      float(a_scale_const), L.ptr(bias), int(level_bound), codes.data_ptr(), dec.data_ptr(),
                                      L.tc_err_flag(codes.device).data_ptr(), L.stream())


def codes_fit(in_channels, groups, kernel_size, level_bound=1):
    """the int16 bound of mnb_pk_conv_codes: every sum of (C/g) * R * S terms +-1 x level fits in an int16"""
    r, s = (kernel_size, kernel_size) if isinstance(kernel_size, int) else kernel_size
    return (in_channels // groups) * r * s * level_bound <= 32767


def consumer_plane(b, c, h, w, device):
    """empty operand plane (one bf16 piece) of a conv that reads a [b, c, h, w] activation"""
    return torch.empty(int(L.load().mnb_pk_act_bytes(b, c, h, w, 1)), dtype=torch.uint8, device=device)


def post_struct(qp, plane, relu, split, bn=None, shuffle_groups=1):
    """mnb_pk_post of a consumer; ``bn`` = (mean, invstd, gamma, beta) of an eval BatchNorm in front of its [ReLU +] quantizer"""
    post = L.PkPost(C.pointer(qp), 1 if relu else 0, 1 if split else 0, plane.data_ptr())
    if bn is not None:
        post.bn_mean, post.bn_invstd, post.bn_gamma, post.bn_beta = (t.data_ptr() for t in bn)
    post.shuffle_groups = int(shuffle_groups)
    return post


def conv_post(sh, a_pk, terms_a, w_img, terms_w, out, post_qp, post_plane, post_relu, post_split, n_scale=None, a_scale=None,
              a_scale_const=1.0, bias=None, bn=None, shuffle_groups=1):
    """forward conv whose epilogue also writes the consumer's operand plane (frozen inference graphs); out may be None"""
    lib = L.load()
    post = post_struct(post_qp, post_plane, post_relu, post_split, bn, shuffle_groups)
    return lib.mnb_pk_conv_post(C.byref(sh), a_pk.data_ptr(), terms_a, w_img.data_ptr(), terms_w, L.ptr(n_scale), L.ptr(a_scale),
                                float(a_scale_const), L.ptr(bias), L.ptr(out), C.byref(post),
                                L.tc_err_flag(a_pk.device).data_ptr(), L.stream())


# ---- term planes as a hand-off (frozen wbwtab graphs with fp32 activations): the consumer reads an fp32 value as T exact pieces
def terms_plane(b, c, h, w, terms, device):
    """empty term planes (``terms`` bf16 pieces) of a conv that reads a [b, c, h, w] fp32 activation"""
    return torch.empty(terms * int(L.load().mnb_pk_act_bytes(b, c, h, w, 1)), dtype=torch.uint8, device=device)


def unpack_terms(plane, shape, terms, split=False):
    """the fp32 [b, c, h, w] tensor a term plane holds (p0 + p1 + p2, exact); ``split``: phase-split layout"""
    b, c, h, w = shape
    c8 = (c + 7) // 8
    pl = plane.view(torch.bfloat16).float()
    if split:
        pl = pl.view(terms, b, 2, 2, c8, h // 2, w // 2, 8).permute(0, 1, 4, 7, 5, 2, 6, 3).reshape(terms, b, c8 * 8, h, w)
    else:
        pl = pl.view(terms, b, c8, h, w, 8).permute(0, 1, 2, 5, 3, 4).reshape(terms, b, c8 * 8, h, w)
    out = pl[0].clone()
    for t in range(1, terms):
        out += pl[t]
    return out[:, :c].contiguous()


def conv_post_terms(sh, a_pk, w_img, out, plane, terms, relu=True, split=False, n_scale=None, bias=None, bn=None,
                    shuffle_groups=1):
    """forward conv (activation ``terms``-piece plane, one piece of integer weight levels) whose epilogue writes the
    consumer's ``terms`` term planes of [BatchNorm] [ReLU] [shuffle] of its output; out may be None.  Returns the C status."""
    post = L.PkPost(None, 1 if relu else 0, 1 if split else 0, plane.data_ptr())
    if bn is not None:
        post.bn_mean, post.bn_invstd, post.bn_gamma, post.bn_beta = (t.data_ptr() for t in bn)
    post.shuffle_groups, post.terms_out = int(shuffle_groups), int(terms)
    return L.load().mnb_pk_conv_post(C.byref(sh), a_pk.data_ptr(), terms, w_img.data_ptr(), 1, L.ptr(n_scale), None, 1.0,
                                     L.ptr(bias), L.ptr(out), C.byref(post), L.tc_err_flag(a_pk.device).data_ptr(), L.stream())


def bn_relu_pack_terms(x, bn, relu, shuffle_groups, terms, plane):
    """mnb_bn_relu_pack_terms_fwd of a contiguous fp32 [b, c, h, w] x into ``plane``; bn = (mean, invstd, gamma, beta) or None.
    Returns the C status."""
    b, c, h, w = x.shape
    mean, invstd, gamma, beta = (None,) * 4 if bn is None else (t.data_ptr() for t in bn)
    return L.load().mnb_bn_relu_pack_terms_fwd(x.data_ptr(), b, c, h * w, mean, invstd, gamma, beta, 1 if relu else 0,
                                               int(shuffle_groups), terms, plane.data_ptr(), L.stream())


def plane_maxpool_terms(plane, b, c, h, w, k, s, p, terms):
    """(C status, pooled term planes) of max_pool2d(k, s, p) of the fp32 tensor a term plane holds (mnb_pk_plane_maxpool_terms)"""
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    out = terms_plane(b, c, oh, ow, terms, plane.device)
    return L.load().mnb_pk_plane_maxpool_terms(plane.data_ptr(), b, c, h, w, k, s, p, terms, out.data_ptr(), L.stream()), out


# ---- int8 operands (frozen inference graphs, symmetric IAO): planes [b][c/16][h][w][16] s8, s8 x s8 -> s32 wgmma
def i8_plan(sh):
    """plan of mnb_pk_i8_conv as a list of the 21 mnb_pk_conv_plan_ex fields, None outside the int8 cover (host only)"""
    out = (C.c_int32 * 21)()
    return list(out) if L.load().mnb_pk_i8_conv_plan(C.byref(sh), out, 21) == 0 else None


def i8_supported(sh):
    """does mnb_pk_i8_conv cover this forward shape?  (host-only plan query, cached)"""
    k = ("i8", _key(sh))
    if k not in _plan_cache:
        _plan_cache[k] = L.load().mnb_pk_i8_conv_plan(C.byref(sh), None, 0) == 0
    return _plan_cache[k]


def consumer_plane_i8(b, c, h, w, device):
    """empty int8 operand plane of a conv that reads a [b, c, h, w] activation"""
    return torch.empty(int(L.load().mnb_pk_i8_act_bytes(b, c, h, w)), dtype=torch.uint8, device=device)


def pack_act_i8(x, qp, phase_split=False, relu=False):
    """fp32 NCHW -> int8 level plane of a symmetric IAO quantizer"""
    b, c, h, w = x.shape
    out = consumer_plane_i8(b, c, h, w, x.device)
    L.check(L.load().mnb_pk_i8_pack_act(x.data_ptr(), b, c, h, w, C.byref(qp), 1 if phase_split else 0, 1 if relu else 0,
                                        out.data_ptr(), L.stream()), "pk_i8_pack_act")
    return out


def plane_maxpool(plane, b, c, h, w, k, s, p, int8=False):
    """max_pool2d(k, s, p) of a level plane of a [b, c, h, w] activation (mnb_pk_plane_maxpool) -> the pooled plane"""
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    out = (consumer_plane_i8 if int8 else consumer_plane)(b, c, oh, ow, plane.device)
    L.check(L.load().mnb_pk_plane_maxpool(plane.data_ptr(), b, c, h, w, k, s, p, 1 if int8 else 0, out.data_ptr(), L.stream()),
            "pk_plane_maxpool")
    return out


def plane_maxpool_requant(plane, b, c, h, w, k, s, p, q_in, q_out, int8=False):
    """the IAO QuantMaxPool2d between two frozen convs on a plane of its own quantizer's levels (q_in, an ActQParams):
    max_pool2d(k, s, p), requantized to the consumer's quantizer q_out (mnb_pk_plane_maxpool_requant) -> the consumer's plane"""
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    out = (consumer_plane_i8 if int8 else consumer_plane)(b, c, oh, ow, plane.device)
    L.check(L.load().mnb_pk_plane_maxpool_requant(plane.data_ptr(), b, c, h, w, k, s, p, 1 if int8 else 0, C.byref(q_in),
                                                  C.byref(q_out), out.data_ptr(), L.stream()), "pk_plane_maxpool_requant")
    return out


def pack_weight_i8(sh, w_int):
    nbytes = int(L.load().mnb_pk_i8_wimage_bytes(C.byref(sh)))
    if nbytes < 0:
        raise ValueError("micronet_b200.pk: shape outside the cover of the int8 convolution")
    img = torch.empty(nbytes, dtype=torch.uint8, device=w_int.device)
    L.check(L.load().mnb_pk_i8_pack_weight(C.byref(sh), w_int.data_ptr(), img.data_ptr(), L.stream()), "pk_i8_pack_weight")
    return img


def conv_i8(sh, a_pk, w_img, out, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None, post=None):
    """forward conv of an int8 plane; ``post`` = (quantizer struct, int8 plane, relu, phase split[, BatchNorm tensors,
    shuffle groups]) of the consumer whose plane the epilogue writes as well (out may then be None).  Returns the C status."""
    pp = None
    if post is not None:
        pp = C.byref(post_struct(*post))
    return L.load().mnb_pk_i8_conv(C.byref(sh), a_pk.data_ptr(), w_img.data_ptr(), L.ptr(n_scale), L.ptr(a_scale),
                                   float(a_scale_const), L.ptr(bias), L.ptr(out), pp, L.tc_err_flag(a_pk.device).data_ptr(),
                                   L.stream())


def wgrad(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=None, kdiv=None):
    lib = L.load()
    nbytes = int(lib.mnb_pk_wgrad_scratch_bytes(C.byref(sh), terms_dy, terms_x))
    if nbytes < 0:
        return L.E_UNSUPPORTED
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dw.device)
    return lib.mnb_pk_wgrad(C.byref(sh), dy_pk.data_ptr(), terms_dy, x_pk.data_ptr(), terms_x, L.ptr(a_scale),
                            L.ptr(kdiv), dw.data_ptr(), ws.data_ptr(), L.tc_err_flag(dw.device).data_ptr(), L.stream())


def wgrad_taps_plan(sh, terms_dy, terms_x):
    """plan of mnb_pk_wgrad_taps as a dict, None outside its cover (host-only plan query, cached)"""
    k = ("wt", _key(sh), terms_dy, terms_x)
    if k not in _plan_cache:
        out = (C.c_int32 * 12)()
        ok = L.load().mnb_pk_wgrad_taps_plan(C.byref(sh), terms_dy, terms_x, out, 12) == 0
        names = ("blocks", "splits", "NI", "nstage", "BW", "TH", "stg_per_split", "smem_bytes", "acc_regs")
        plan = None
        if ok:
            plan = dict(zip(names, out[:9]))
            plan["scratch_bytes"] = out[9] | (out[10] << 31)
            plan["npairs"] = out[11]
        _plan_cache[k] = plan
    return _plan_cache[k]


def wgrad_taps(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=None, kdiv=None):
    """mnb_pk_wgrad_taps: same operands as wgrad and the same result bit for bit; returns the C status"""
    plan = wgrad_taps_plan(sh, terms_dy, terms_x)
    if plan is None:
        return L.E_UNSUPPORTED
    ws = torch.empty(plan["scratch_bytes"], dtype=torch.uint8, device=dw.device)
    return L.load().mnb_pk_wgrad_taps(C.byref(sh), dy_pk.data_ptr(), terms_dy, x_pk.data_ptr(), terms_x, L.ptr(a_scale),
                                      L.ptr(kdiv), dw.data_ptr(), ws.data_ptr(), L.tc_err_flag(dw.device).data_ptr(), L.stream())


def bwd1x1_plan(sh, terms_dy, terms_x, terms_w):
    """plan of mnb_pk_bwd1x1 as a dict, None outside its cover (host-only plan query, cached)"""
    k = ("b1", _key(sh), terms_dy, terms_x, terms_w)
    if k not in _plan_cache:
        out = (C.c_int32 * 15)()
        ok = L.load().mnb_pk_bwd1x1_plan(C.byref(sh), terms_dy, terms_x, terms_w, out, 15) == 0
        plan = None
        if ok:
            names = ("groups", "splits", "NI", "nstage", "BW", "TH", "stg_per_split", "smem_bytes", "nsub", "nstg_total",
                     "dgrad_chain")
            plan = dict(zip(names, out[:11]))
            plan["scratch_bytes"] = out[11] | (out[12] << 31)
            plan["npairs"], plan["Nc"] = out[13], out[14]
        _plan_cache[k] = plan
    return _plan_cache[k]


def bwd1x1(sh, dy_pk, terms_dy, x_pk, terms_x, w_img, terms_w, dx, dw, bits8=None, gain=1.0, a_scale_const=1.0, a_scale=None,
           kdiv=None):
    """mnb_pk_bwd1x1: conv(sh, 1, dy_pk, terms_dy, w_img, terms_w, dx, bits8=, gain=, a_scale_const=) followed by
    wgrad(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=, kdiv=), the same results bit for bit; returns the C status"""
    plan = bwd1x1_plan(sh, terms_dy, terms_x, terms_w)
    if plan is None:
        return L.E_UNSUPPORTED
    ws = torch.empty(plan["scratch_bytes"], dtype=torch.uint8, device=dw.device)
    return L.load().mnb_pk_bwd1x1(C.byref(sh), dy_pk.data_ptr(), terms_dy, x_pk.data_ptr(), terms_x, w_img.data_ptr(), terms_w,
                                  float(a_scale_const), L.ptr(bits8), float(gain), dx.data_ptr(), L.ptr(a_scale), L.ptr(kdiv),
                                  dw.data_ptr(), ws.data_ptr(), L.tc_err_flag(dw.device).data_ptr(), L.stream())


def gc3_plan(sh, mode, terms_a, terms_w):
    """plan of mnb_pk_gc3_conv as a dict, None outside its cover (host-only plan query, cached).  ``chain``: the MMAs of
    one accumulator in issue order as (filter tap r * 3 + s, streamed-operand piece, weight piece, 16-channel K-step)"""
    k = ("g3", _key(sh), mode, terms_a, terms_w)
    if k not in _plan_cache:
        out = (C.c_int32 * (10 + 4 * 128))()
        ok = L.load().mnb_pk_gc3_plan(C.byref(sh), mode, terms_a, terms_w, out, len(out)) == 0
        plan = None
        if ok:
            names = ("groups_per_block", "images_per_tile", "m_blocks", "nstage", "smem_bytes", "ctas", "tiles", "chain_len",
                     "Nt", "mma_warpgroups")
            plan = dict(zip(names, out[:10]))
            plan["chain"] = [tuple(out[10 + 4 * i:14 + 4 * i]) for i in range(plan["chain_len"])]
        _plan_cache[k] = plan
    return _plan_cache[k]


def gc3_conv(sh, mode, a_pk, terms_a, w_img, terms_w, out, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None,
             bits8=None, gain=1.0):
    """mnb_pk_gc3_conv: same arguments as conv and the same result bit for bit; returns the C status"""
    return L.load().mnb_pk_gc3_conv(C.byref(sh), mode, a_pk.data_ptr(), terms_a, w_img.data_ptr(), terms_w, L.ptr(n_scale),
                                    L.ptr(a_scale), float(a_scale_const), L.ptr(bias), L.ptr(bits8), float(gain),
                                    out.data_ptr(), L.tc_err_flag(out.device).data_ptr(), L.stream())


def gc3_conv_codes(sh, a_pk, w_img, codes, dec, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None, level_bound=1):
    """mnb_pk_gc3_conv_codes: same arguments as conv_codes and the same codes and decode pair; returns the C status"""
    return L.load().mnb_pk_gc3_conv_codes(C.byref(sh), a_pk.data_ptr(), 1, w_img.data_ptr(), 1, L.ptr(n_scale), L.ptr(a_scale),
                                          float(a_scale_const), L.ptr(bias), int(level_bound), codes.data_ptr(), dec.data_ptr(),
                                          L.tc_err_flag(codes.device).data_ptr(), L.stream())


# ---- kernel choice of the engine's layers
def run_conv(sh, mode, a_pk, terms_a, w_img, terms_w, out, **epilogue):
    """forward (mode 0) or data gradient (mode 1) with conv's arguments: on gc3_conv where its plan covers the shape and
    PK_GC3 allows, on conv otherwise and for whatever gc3_conv refuses.  Returns the C status."""
    if L.PK_GC3 and gc3_plan(sh, mode, terms_a, terms_w) is not None:
        rc = gc3_conv(sh, mode, a_pk, terms_a, w_img, terms_w, out, **epilogue)
        if rc != L.E_UNSUPPORTED:
            return rc
    return conv(sh, mode, a_pk, terms_a, w_img, terms_w, out, **epilogue)


def run_conv_codes(sh, a_pk, w_img, codes, dec, **epilogue):
    """conv_codes with the same choice as run_conv: gc3_conv_codes first where it applies.  Returns the C status."""
    if L.PK_GC3 and gc3_plan(sh, 0, 1, 1) is not None:
        rc = gc3_conv_codes(sh, a_pk, w_img, codes, dec, **epilogue)
        if rc != L.E_UNSUPPORTED:
            return rc
    return conv_codes(sh, a_pk, w_img, codes, dec, **epilogue)


def run_wgrad(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=None, kdiv=None):
    """weight gradient with wgrad's arguments: on wgrad_taps where its plan covers the shape and PK_WG_TAPS allows, on
    wgrad otherwise.  Returns the C status."""
    fn = wgrad_taps if L.PK_WG_TAPS and wgrad_taps_plan(sh, terms_dy, terms_x) is not None else wgrad
    return fn(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=a_scale, kdiv=kdiv)


def bwd1x1_taken(sh, terms_dy, terms_x, terms_w):
    """does run_bwd take mnb_pk_bwd1x1 for this layer?"""
    return L.PK_BWD1X1 and bwd1x1_plan(sh, terms_dy, terms_x, terms_w) is not None


def run_bwd(sh, dy_pk, terms_dy, x_pk, terms_x, w_img, terms_w, dx, dw, bits8=None, gain=1.0, a_scale_const=1.0, a_scale=None,
            kdiv=None):
    """data and weight gradient: on bwd1x1 where its plan covers the shape and PK_BWD1X1 allows, otherwise run_conv
    (mode 1) followed by run_wgrad.  Returns the C status of the first call that fails, or 0."""
    if bwd1x1_taken(sh, terms_dy, terms_x, terms_w):
        return bwd1x1(sh, dy_pk, terms_dy, x_pk, terms_x, w_img, terms_w, dx, dw, bits8=bits8, gain=gain,
                      a_scale_const=a_scale_const, a_scale=a_scale, kdiv=kdiv)
    rc = run_conv(sh, 1, dy_pk, terms_dy, w_img, terms_w, dx, bits8=bits8, gain=gain, a_scale_const=a_scale_const)
    if rc != 0:
        return rc
    return run_wgrad(sh, dy_pk, terms_dy, x_pk, terms_x, dw, a_scale=a_scale, kdiv=kdiv)
