"""Python side of the binary tensor-core forward (``csrc/mnb_b1.cu``) for wbwtab layers outside the XNOR kernel's cover.

    pack_act       fp32 NCHW -> b1 plane [B][G * u][H][W][16 B], u = ceil(C/g / 64)   (WB:11-36: sign(x), 0 -> +1)
    pack_weight    i16 levels {-1, 0, +1} -> B image: plus = [P | M], minus = [M | P] per output channel   (WB:55-75)
    conv           y = fmaf(D_plus - D_minus, alpha[k], bias[k])                      (WB:181-195, forward only)
    conv_post      the same sum through mnb_xnor_post's epilogue into a bit, bf16 or b1 plane
    plane_maxpool  MaxPool2d(k, s, p) on a b1 plane (NIN's 3 / 2 / 1 pools, models/nin.py)

The integer sum is exact, so the result equals the XNOR and packed-operand forwards bit for bit (DESIGN.md 4.19)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L

_sup_cache = {}


def supported(sh):
    k = tuple(getattr(sh, f) for f, _ in sh._fields_)
    if k not in _sup_cache:
        _sup_cache[k] = L.load().mnb_b1_supported(C.byref(sh)) == 1
    return _sup_cache[k]


PLAN_FIELDS = ("Nt", "n_ntiles", "u", "ksteps", "G", "col_tiles", "Wt", "BW", "TH", "TB", "row_tiles", "n_mtiles", "TG",
               "ntg", "nstage", "post", "smem")


def plan(sh, post=None):
    """the launch plan of ``conv`` (post None) / ``conv_post`` for shape ``sh`` (mnb_b1_plan, host only): a dict of
    PLAN_FIELDS, or None outside the cover"""
    out = (C.c_int32 * len(PLAN_FIELDS))()
    rc = L.load().mnb_b1_plan(C.byref(sh), None if post is None else C.byref(post), out)
    if rc == L.E_UNSUPPORTED:
        return None
    L.check(rc, "b1_plan")
    return dict(zip(PLAN_FIELDS, out))


def act_bytes(b, c, h, w, groups):
    return int(L.load().mnb_b1_act_bytes(b, c, h, w, groups))


def empty_plane(nbytes, device):
    return torch.empty(nbytes // 4, dtype=torch.int32, device=device)


def pack_act(x, groups):
    lib = L.load()
    b, c, h, w = x.shape
    nbytes = act_bytes(b, c, h, w, groups)
    if nbytes < 0:
        raise ValueError("micronet_b200.b1: channels not divisible by groups")
    out = empty_plane(nbytes, x.device)
    L.check(lib.mnb_b1_pack_act(x.data_ptr(), b, c, h, w, groups, out.data_ptr(), L.stream()), "b1_pack_act")
    return out


def pack_act_post(x, post, out):
    b, c, h, w = x.shape
    return L.load().mnb_b1_pack_act_post(x.data_ptr(), b, c, h, w, C.byref(post), out.data_ptr(), L.stream())


def pack_weight(sh, w_int):
    lib = L.load()
    nbytes = int(lib.mnb_b1_wimage_bytes(C.byref(sh)))
    if nbytes < 0:
        raise ValueError("micronet_b200.b1: shape outside the cover of the binary tensor-core convolution")
    img = torch.empty(nbytes // 4, dtype=torch.int32, device=w_int.device)
    L.check(lib.mnb_b1_pack_weight(C.byref(sh), w_int.data_ptr(), img.data_ptr(), L.stream()), "b1_pack_weight")
    return img


def conv(sh, a_plane, w_img, out, alpha=None, bias=None):
    return L.load().mnb_b1_conv_fwd(C.byref(sh), a_plane.data_ptr(), w_img.data_ptr(), L.ptr(alpha), L.ptr(bias),
                                    out.data_ptr(), L.tc_err_flag(out.device).data_ptr(), L.stream())


def post_bytes(sh, post):
    return int(L.load().mnb_b1_post_bytes(C.byref(sh), C.byref(post)))


def conv_post(sh, a_plane, w_img, post, out, alpha=None, bias=None):
    """the convolution with the sign epilogue: ``out`` (post_bytes(sh, post) bytes) receives the consumer's operand"""
    return L.load().mnb_b1_conv_post(C.byref(sh), a_plane.data_ptr(), w_img.data_ptr(), L.ptr(alpha), L.ptr(bias),
                                     C.byref(post), out.data_ptr(), L.tc_err_flag(out.device).data_ptr(), L.stream())


def plane_maxpool(plane, shape, groups, k, s, p):
    """MaxPool2d(k, s, p) of the +-1 tensor ``shape`` = (B, C, H, W) encoded by ``plane``: (pooled plane, pooled shape)"""
    b, c, h, w = shape
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    out = empty_plane(act_bytes(b, c, oh, ow, groups), plane.device)
    rc = L.load().mnb_b1_plane_maxpool(plane.data_ptr(), b, c, groups, h, w, k, s, p, out.data_ptr(), L.stream())
    return rc, out, (b, c, oh, ow)


def unpack(plane, shape, groups):
    """b1 plane -> the fp32 tensor [B, C, H, W] it encodes (+1, -1, or 0 where neither bit is set) - for readers outside
    the frozen graph: tests, hooks, a module the plane was not written for"""
    b, c, h, w = shape
    cg = c // groups
    u = (cg + 63) // 64
    words = plane.view(torch.int32).view(b, groups, u, h, w, 4)
    ch = torch.arange(c, device=plane.device)
    sel = words[:, ch // cg, (ch % cg) // 64]                                 # [B, C, H, W, 4] unit of each channel
    j = ((ch % cg) % 64).view(1, c, 1, 1)
    word = (j // 32).unsqueeze(-1)
    shift = (j % 32).to(torch.int32)
    pos = (torch.gather(sel, 4, word.expand(b, c, h, w, 1)).squeeze(-1) >> shift) & 1
    neg = (torch.gather(sel, 4, (word + 2).expand(b, c, h, w, 1)).squeeze(-1) >> shift) & 1
    return (pos - neg).float()
