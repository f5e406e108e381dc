"""Python side of the bit-packed XNOR-popcount forward (``csrc/mnb_xnor.cu``) for wbwtab layers.

    pack_act     fp32 NCHW -> sign bit planes u32 [B][G][ceil(C/g / 32)][H][W]      (WB:11-36: sign(x), 0 -> +1)
    pack_weight  i16 levels {-1, 0, +1} -> sign / non-zero words + popcount / border tables   (WB:40-75, 98-146)
    conv         y = fmaf(popc(N) - 2 popc(N & (A ^ S)), alpha[k], bias[k])       (WB:181-195, forward only)

The integer sum is exact, so the result equals the packed-operand tensor-core forward bit for bit; which of the two runs a
given layer is decided from measurements (``harness/xnor_probe.py`` -> ``profiles/r2_xnor_vs_tc.md``, DESIGN.md 4.11)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L

_sup_cache = {}


def supported(sh):
    k = tuple(getattr(sh, f) for f, _ in sh._fields_)
    if k not in _sup_cache:
        _sup_cache[k] = L.load().mnb_xnor_supported(C.byref(sh)) == 1
    return _sup_cache[k]


PLAN_FIELDS = ("R", "NW", "border", "px", "post", "ksplit", "kb", "pblocks", "smem", "refused")


def plan(sh, post=None):
    """the launch plan of ``conv`` (post None) / ``conv_post`` for shape ``sh`` (mnb_xnor_plan, host only): a dict of
    PLAN_FIELDS, or None outside the cover.  ``refused`` 1: the launch returns MNB_E_UNSUPPORTED."""
    out = (C.c_int32 * len(PLAN_FIELDS))()
    rc = L.load().mnb_xnor_plan(C.byref(sh), None if post is None else C.byref(post), out)
    if rc == L.E_UNSUPPORTED:
        return None
    L.check(rc, "xnor_plan")
    return dict(zip(PLAN_FIELDS, out))


def pack_act(x, groups):
    lib = L.load()
    b, c, h, w = x.shape
    nbytes = int(lib.mnb_xnor_act_bytes(b, c, h, w, groups))
    if nbytes < 0:
        raise ValueError("micronet_b200.xnor: channels not divisible by groups")
    out = torch.empty(nbytes // 4, dtype=torch.int32, device=x.device)
    L.check(lib.mnb_xnor_pack_act(x.data_ptr(), b, c, h, w, groups, out.data_ptr(), L.stream()), "xnor_pack_act")
    return out


def pack_weight(sh, w_int):
    lib = L.load()
    nbytes = int(lib.mnb_xnor_wimage_bytes(C.byref(sh)))
    if nbytes < 0:
        raise ValueError("micronet_b200.xnor: shape outside the cover of the XNOR-popcount convolution")
    img = torch.empty(nbytes // 4, dtype=torch.int32, device=w_int.device)
    L.check(lib.mnb_xnor_pack_weight(C.byref(sh), w_int.data_ptr(), img.data_ptr(), L.stream()), "xnor_pack_weight")
    return img


def conv(sh, a_bits, w_img, out, alpha=None, bias=None):
    return L.load().mnb_xnor_conv_fwd(C.byref(sh), a_bits.data_ptr(), w_img.data_ptr(), L.ptr(alpha), L.ptr(bias),
                                      out.data_ptr(), L.stream())


def post_struct(fmt, out_groups=1, shuffle_groups=1, pool2=False, bn=None):
    """mnb_xnor_post: ``bn`` = (mean, invstd, gamma, beta) fp32 [C] device tensors of an eval BatchNorm, or None"""
    ptrs = [None] * 4 if bn is None else [t.data_ptr() for t in bn]
    return L.XnorPost(fmt, int(out_groups), int(shuffle_groups), 1 if pool2 else 0, *ptrs)


def post_bytes(sh, post):
    return int(L.load().mnb_xnor_post_bytes(C.byref(sh), C.byref(post)))


def conv_post(sh, a_bits, w_img, post, out, alpha=None, bias=None):
    """the convolution with the sign-bit epilogue: ``out`` (post_bytes(sh, post) bytes) receives the consumer's operand"""
    return L.load().mnb_xnor_conv_post(C.byref(sh), a_bits.data_ptr(), w_img.data_ptr(), L.ptr(alpha), L.ptr(bias),
                                       C.byref(post), out.data_ptr(), L.stream())


def pack_act_post(x, post, out):
    b, c, h, w = x.shape
    return L.load().mnb_xnor_pack_act_post(x.data_ptr(), b, c, h, w, C.byref(post), out.data_ptr(), L.stream())


def unpack(bits, shape, groups):
    """bit plane u32 [B][G][ceil(C/g / 32)][H][W] -> the +-1 fp32 tensor [B, C, H, W] it encodes (for readers outside the
    frozen graph: tests, hooks, a module the plane was not written for)"""
    b, c, h, w = shape
    cg = c // groups
    nw = (cg + 31) // 32
    words = bits.view(b, groups, nw, h, w)
    ch = torch.arange(c, device=bits.device)
    sel = words[:, ch // cg, (ch % cg) // 32]                                  # [B, C, H, W] word of each channel
    bit = (sel >> ((ch % cg) % 32).view(1, c, 1, 1).to(torch.int32)) & 1           # bit of the channel within its group
    return (bit * 2 - 1).float()
