"""Python side of the packed-operand tensor-core family (``csrc/mnb_pk.cu``).

Every conv of the QAT models that the fused kernels of ``mnb_conv_tc_*.cu`` cannot take (weights that do not fit in
shared memory, stride 2, 5x5 filters, 4x4 or 224x224 images ...) and every fused-quantizer layer runs here:

    pack_act    fp32 NCHW -> bf16 term planes [t][b][c/8][h][w][8] (fake-quantize, or exact split of an fp32 tensor)
    pack_weight integer levels / fp32 weights -> the bf16 operand image of one (shape, mode)
    conv        TMA -> wgmma (register accumulators) -> epilogue (forward: scale + bias; data gradient: STE mask)
    wgrad       the same boxes read as MN-major operands, split over the batch, deterministic reduction
    wgrad_taps  wgrad of narrow grouped 3x3 layers with all nine taps of a CTA in registers

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


def pack_act(x, qp, terms, ch_scale=None, phase_split=False, want_bits=False, relu=False):
    """-> (planes u8[terms * B * ceil(C/8) * H * W * 16], bits8 u8[B, ceil(C/8), H, W] or None)"""
    lib = L.load()
    b, c, h, w = x.shape
    nbytes = int(lib.mnb_pk_act_bytes(b, c, h, w, terms))
    out = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    bits = None
    if qp is not None and want_bits:
        bits = torch.empty((b, (c + 7) // 8, h, w), dtype=torch.uint8, device=x.device)
    L.check(lib.mnb_pk_pack_act_relu(x.data_ptr(), b, c, h, w, None if qp is None else C.byref(qp), terms, L.ptr(ch_scale),
                                     1 if phase_split else 0, 1 if relu else 0, out.data_ptr(), L.ptr(bits), L.stream()),
            "pk_pack_act")
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


def conv_post(sh, a_pk, terms_a, w_img, terms_w, out, post_qp, post_plane, post_relu, post_split, n_scale=None, a_scale=None,
              a_scale_const=1.0, bias=None):
    """forward conv whose epilogue also writes the consumer's operand plane (frozen inference graphs); out may be None"""
    lib = L.load()
    post = L.PkPost(C.pointer(post_qp), 1 if post_relu else 0, 1 if post_split else 0, post_plane.data_ptr())
    return lib.mnb_pk_conv_post(C.byref(sh), a_pk.data_ptr(), terms_a, w_img.data_ptr(), terms_w, L.ptr(n_scale), L.ptr(a_scale),
                                float(a_scale_const), L.ptr(bias), L.ptr(out), C.byref(post),
                                L.tc_err_flag(a_pk.device).data_ptr(), L.stream())


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


def pack_weight_i8(sh, w_int):
    nbytes = int(L.load().mnb_pk_i8_wimage_bytes(C.byref(sh)))
    if nbytes < 0:
        raise ValueError("micronet_b200.pk: shape outside the cover of the int8 convolution")
    img = torch.empty(nbytes, dtype=torch.uint8, device=w_int.device)
    L.check(L.load().mnb_pk_i8_pack_weight(C.byref(sh), w_int.data_ptr(), img.data_ptr(), L.stream()), "pk_i8_pack_weight")
    return img


def conv_i8(sh, a_pk, w_img, out, n_scale=None, a_scale=None, a_scale_const=1.0, bias=None, post=None):
    """forward conv of an int8 plane; ``post`` = (quantizer struct, int8 plane, relu, phase split) of the consumer whose
    plane the epilogue writes as well (out may then be None).  Returns the C status."""
    pp = None
    if post is not None:
        qp, plane, relu, split = post
        pp = C.byref(L.PkPost(C.pointer(qp), 1 if relu else 0, 1 if split else 0, plane.data_ptr()))
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
