"""Host-side checks of the int8 operands of the packed-operand family (mnb_pk_i8_*), no GPU needed:

* the int8 plan (mnb_pk_i8_conv_plan) covers every conv of the ResNet-18 bench models (32 x 32 and 224 x 224) inside shared
  memory and the register budget of the accumulators, and the int8 plane holds 16 channels per 16 bytes;
* the int8 entry points refuse requests outside their cover on the host, before launching (the pointers are fakes that
  are never dereferenced)."""
import ctypes as C

import pytest

from tests import pk_plan_util as PU


def _resnet_convs():
    return [c for c in PU.model_convs() if c[0].startswith(("res32_", "res224_"))]


@pytest.mark.parametrize("conv", _resnet_convs(), ids=lambda c: c[0])
def test_int8_plan_covers_the_resnet_convs(conv):
    from micronet_b200 import _lib as L
    lib = L.load()
    name, B, Cc, H, W, K, R, st, pad, G = conv
    sh = PU.shape(B, Cc, H, W, K, R, st, pad, G)
    p = PU.i8_plan(sh)
    assert p is not None, (name, lib.mnb_last_error())
    assert 0 < p["smem"] <= PU.budget("mnb_pk.cu", "kSmemBudget"), (name, p)
    assert p["acc"] == p["MT"] * p["Nt"] and p["acc"] <= 128 and p["Nt"] in PU.CONV_NT, (name, p)
    assert p["segmented"] == 0 and p["npairs"] == 1 and p["ny"] == 1 and p["CC"] % 32 == 0, (name, p)
    assert 1 <= p["n_items"] < (1 << 22) and p["n_mtiles"] < (1 << 22), (name, p)
    wimg = int(lib.mnb_pk_i8_wimage_bytes(C.byref(sh)))
    assert wimg == p["wimg_lo"] + (p["wimg_hi"] << 31) and wimg >= 16
    # one 16-byte vector per pixel and 16 channels: half the bytes of the bf16 plane of the same activation
    assert int(lib.mnb_pk_i8_act_bytes(B, Cc, H, W)) == B * ((Cc + 15) // 16) * H * W * 16
    if Cc % 16 == 0:
        assert 2 * int(lib.mnb_pk_i8_act_bytes(B, Cc, H, W)) == int(lib.mnb_pk_act_bytes(B, Cc, H, W, 1))


def test_int8_entry_points_refuse_before_launching():
    from micronet_b200 import _lib as L
    lib = L.load()
    fake = 4096
    sym = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, fake, fake, fake, fake)
    asym = L.ActQParams(L.ACT_IAO, 8, 0, 255, 1, fake, fake, fake, fake)
    nine = L.ActQParams(L.ACT_IAO, 9, -256, 255, 0, fake, fake, fake, fake)
    dorefa = L.ActQParams(L.ACT_DOREFA, 8, 0, 255, 0, fake, fake, fake, fake)
    for bad in (asym, nine, dorefa):
        assert lib.mnb_pk_i8_pack_act(fake, 2, 16, 8, 8, C.byref(bad), 0, 0, fake, None) == L.E_UNSUPPORTED
        post = L.PkPost(C.pointer(bad), 0, 0, fake)
        assert lib.mnb_quant_add_pack_i8_fwd(fake, fake, 2, 16, 8, 8, C.byref(sym), 0, fake, C.byref(post), None) == L.E_UNSUPPORTED
        sh = PU.shape(2, 16, 8, 8, 32, 3, 1, 1, 1)
        rc = lib.mnb_pk_i8_conv(C.byref(sh), fake, fake, None, None, 1.0, None, None, C.byref(post), fake, None)
        assert rc == L.E_UNSUPPORTED and b"symmetric" in lib.mnb_last_error(), rc
    # grouped convs: GEMM-K channels per group must be a multiple of 16 (one 16-byte unit)
    g8 = PU.shape(2, 32, 8, 8, 32, 3, 1, 1, 4)
    assert PU.conv_plan(g8, 0, 1, 1) is not None and PU.i8_plan(g8) is None
    assert lib.mnb_pk_i8_wimage_bytes(C.byref(g8)) == -1
    rc = lib.mnb_pk_i8_conv(C.byref(g8), fake, fake, None, None, 1.0, None, fake, None, fake, None)
    assert rc == L.E_UNSUPPORTED and b"% 16" in lib.mnb_last_error()
    assert lib.mnb_pk_i8_pack_weight(C.byref(g8), fake, fake, None) == L.E_UNSUPPORTED
    # a grouped producer whose channels per group are not a multiple of 16 writes no int8 consumer plane
    g16 = PU.shape(2, 64, 8, 8, 32, 3, 1, 1, 4)                   # 16 in, 8 out per group
    post = L.PkPost(C.pointer(sym), 0, 0, fake)
    assert lib.mnb_pk_i8_conv(C.byref(g16), fake, fake, None, None, 1.0, None, None, C.byref(post), fake, None) == L.E_UNSUPPORTED
    # no output at all
    sh = PU.shape(2, 16, 8, 8, 32, 3, 1, 1, 1)
    assert lib.mnb_pk_i8_conv(C.byref(sh), fake, fake, None, None, 1.0, None, None, None, fake, None) == -1
    assert b"post" in lib.mnb_last_error()


def test_python_route_takes_the_c_side_rules():
    """functional decides on the host what the C entry points would refuse: a quantizer whose levels leave s8 (an
    asymmetric one reports q_type 0 until its first update_qparams; its level range tells) keeps the bf16 path, and a
    grouped int8 producer hands off a plane only when its output channels per group fill whole 16-channel units"""
    from micronet_b200 import _lib as L, functional as F_
    sh = PU.shape(2, 64, 8, 8, 32, 3, 1, 1, 4)
    w = object()                                       # stands for the integer weights (only their presence is read)
    sym = F_.ActSpec(L.ACT_IAO, bits=8, qmin=-128, qmax=127, q_type=0)
    fresh_asym = F_.ActSpec(L.ACT_IAO, bits=8, qmin=0, qmax=255, q_type=0)
    assert F_._i8_route(sym, w, sh) and not F_._i8_route(fresh_asym, w, sh)
    assert not F_._i8_route(F_.ActSpec(L.ACT_IAO, bits=8, qmin=-128, qmax=127, q_type=1), w, sh)
    assert not F_._i8_route(sym, None, sh)
    assert F_._i8_producer_writes_plane(32, 1) and F_._i8_producer_writes_plane(64, 4)
    assert not F_._i8_producer_writes_plane(32, 4)     # 8 output channels per group: mnb_pk_i8_conv refuses the post
    lib = L.load()
    fake = 4096
    qp = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, fake, fake, fake, fake)
    post = L.PkPost(C.pointer(qp), 0, 0, fake)
    assert lib.mnb_pk_i8_conv(C.byref(sh), fake, fake, None, None, 1.0, None, None, C.byref(post), fake, None) == L.E_UNSUPPORTED
