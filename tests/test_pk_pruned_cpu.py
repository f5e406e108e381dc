"""Host-side checks of the group-padded operand planes (DESIGN.md 4.17), no GPU needed:

* the plans of the packed-operand family cover every conv of a channel-pruned NIN-GC (the reference README's
  group + prune cfg 154 162 144 304 320 320 608 584): forward at the piece counts the three schemes use, data gradient and
  weight gradient;
* the plans of every conv of the bench models at every terms configuration are those recorded in
  tests/pk_plan_bench_table.py (BENCH_PLANS): a change to any of them must be deliberate and recorded there;
* the specialised kernels (pk_gc3, pk_wgrad_taps, int8) refuse padded shapes, so the engine runs them on mnb_pk_conv /
  mnb_pk_wgrad;
* the Python hand-off decisions never hand a plain plane to a conv that reads a group-padded one."""
import ctypes as C

import pytest

from tests import pk_plan_util as PU
from tests.pk_plan_bench_table import BENCH_PLANS, CONFIGS

README_CFG = [154, 162, 144, 304, 320, 320, 608, 584]


def pruned_convs(cfg=README_CFG, batch=256):
    """(name, B, C, H, W, K, R, stride, pad, groups) of the grouped convs of harness.models.NINGC(cfg) at 32 x 32"""
    c = cfg
    return [("L1", batch, c[0], 32, 32, c[1], 1, 1, 0, 2), ("L2", batch, c[1], 32, 32, c[2], 1, 1, 0, 2),
            ("L3", batch, c[2], 16, 16, c[3], 3, 1, 1, 16), ("L4", batch, c[3], 16, 16, c[4], 1, 1, 0, 4),
            ("L5", batch, c[4], 16, 16, c[5], 1, 1, 0, 4), ("L6", batch, c[5], 8, 8, c[6], 3, 1, 1, 32),
            ("L7", batch, c[6], 8, 8, c[7], 1, 1, 0, 8)]


def _sh(conv):
    _, B, Cc, H, W, K, R, st, pad, G = conv
    return PU.shape(B, Cc, H, W, K, R, st, pad, G)


@pytest.mark.parametrize("conv", pruned_convs(), ids=lambda c: c[0])
def test_plans_cover_the_pruned_nin_gc(conv):
    from micronet_b200 import _lib as L, pk as PK
    lib = L.load()
    sh = _sh(conv)
    name, B, Cc, H, W, K, R, st, pad, G = conv
    assert PK.padded_conv(sh) == (name != "L5"), name
    Tb = L.PK_TERMS_BWD
    # forward: levels x integer weights (DoReFa, symmetric IAO, wbwtab), two level pieces x integer weights (asymmetric
    # IAO), +-1 x fp32 pieces, fp32 x fp32; data gradient against integer / fp32 weights
    for mode, ta, tw in ((0, 1, 1), (0, 2, 1), (0, 1, 3), (0, 3, 3), (1, Tb, 1), (1, Tb, Tb)):
        p = PU.conv_plan(sh, mode, ta, tw)
        assert p is not None, (name, mode, ta, tw, lib.mnb_last_error())
        assert p["Nt"] in PU.CONV_NT and p["acc"] <= 128 and p["ny"] == 1, (name, p)
    for t_dy, t_x in ((Tb, 1), (Tb, Tb)):
        p = PU.wgrad_plan(sh, t_dy, t_x)
        assert p is not None, (name, t_dy, t_x, lib.mnb_last_error())
        assert p["Nc"] in PU.WGRAD_NC, (name, p)
    # plane bytes: G groups of ceil(C/G / 8) octets per position
    for ch in (Cc, K):
        want = B * G * ((ch // G + 7) // 8) * H * W * 16
        assert int(lib.mnb_pk_grouped_act_bytes(B, ch, H, W, 1, G)) == want
        if not PK.padded(ch, G):
            assert want == int(lib.mnb_pk_act_bytes(B, ch, H, W, 1))


@pytest.mark.parametrize("cg,kg", [(1, 8), (7, 5), (9, 16), (17, 3), (77, 81), (10, 19)])
def test_plans_cover_edge_channel_counts(cg, kg):
    for R, st, pad in ((1, 1, 0), (3, 1, 1), (3, 2, 1), (1, 2, 0)):
        sh = PU.shape(4, 4 * cg, 16, 16, 4 * kg, R, st, pad, 4)
        for mode, ta, tw in ((0, 1, 1), (0, 3, 3), (1, 2, 1), (1, 2, 2)):
            assert PU.conv_plan(sh, mode, ta, tw) is not None, (cg, kg, R, st, mode, ta, tw)
        for t_dy, t_x in ((2, 1), (2, 2)):
            assert PU.wgrad_plan(sh, t_dy, t_x) is not None, (cg, kg, R, st)


def _bench_rows():
    """(conv, kind, name, mode / terms..., recorded plan) of every bench-model conv at every configuration of the table"""
    table = {r[:5]: r[5] for r in BENCH_PLANS}
    rows = [(conv, kind, conv[0], a, b, c, table.pop((kind, conv[0], a, b, c), "not recorded"))
            for conv in PU.model_convs() for kind, a, b, c in CONFIGS]
    assert not table, f"recorded plans of convs or configurations the bench models do not have: {sorted(table)}"
    return rows


@pytest.mark.parametrize("row", _bench_rows(), ids=lambda r: f"{r[1]}-{r[2]}-{r[3]}-{r[4]}-{r[5]}")
def test_bench_plans_are_unchanged(row):
    import ctypes
    from micronet_b200 import _lib as L
    conv, kind, _, a, b, c, want = row
    lib = L.load()
    sh = _sh(conv)
    if kind == "c":
        out = (ctypes.c_int32 * 21)()
        rc = lib.mnb_pk_conv_plan_ex(C.byref(sh), a, b, c, out, 21)
    else:
        out = (ctypes.c_int32 * 10)()
        rc = lib.mnb_pk_wgrad_plan(C.byref(sh), a, b, out, 10)
    assert (tuple(out) if rc == 0 else None) == want


@pytest.mark.parametrize("conv", pruned_convs(), ids=lambda c: c[0])
def test_specialised_kernels_refuse_padded_shapes(conv):
    from micronet_b200 import _lib as L, pk as PK
    sh = _sh(conv)
    if not PK.padded_conv(sh):
        pytest.skip("not a group-padded shape")
    lib = L.load()
    for mode, ta, tw in ((0, 1, 1), (1, 2, 1)):
        assert PK.gc3_plan(sh, mode, ta, tw) is None
        assert lib.mnb_pk_gc3_plan(C.byref(sh), mode, ta, tw, None, 0) == L.E_UNSUPPORTED
    assert PK.wgrad_taps_plan(sh, 2, 1) is None
    assert lib.mnb_pk_wgrad_taps_plan(C.byref(sh), 2, 1, None, 0) == L.E_UNSUPPORTED
    assert not PK.i8_supported(sh)
    # and their entry points refuse before launching (fake pointers, never dereferenced)
    fake = C.c_void_p(16)
    assert lib.mnb_pk_gc3_conv(C.byref(sh), 0, fake, 1, fake, 1, None, None, 1.0, None, None, 1.0, fake, fake,
                               None) == L.E_UNSUPPORTED
    assert lib.mnb_pk_wgrad_taps(C.byref(sh), fake, 2, fake, 1, None, None, fake, fake, fake, None) == L.E_UNSUPPORTED


def test_consumer_plane_epilogue_keeps_its_cover():
    """mnb_pk_conv_post writes whole octets of a group: a producer with output channels per group % 8 != 0 is refused"""
    from micronet_b200 import _lib as L, functional as F_
    lib = L.load()
    sh = PU.shape(2, 160, 8, 8, 162, 1, 1, 0, 2)          # 80 -> 81 channels per group
    qp = F_.ActSpec(L.ACT_DOREFA, bits=4).struct()
    fake = C.c_void_p(16)
    post = L.PkPost(C.pointer(qp), 0, 0, fake)
    assert lib.mnb_pk_conv_post(C.byref(sh), fake, 1, fake, 1, None, None, 1.0, None, fake, C.byref(post), fake,
                                None) == L.E_UNSUPPORTED


def test_padded_predicate():
    from micronet_b200 import pk as PK
    assert not PK.padded(154, 1) and not PK.padded(160, 2) and not PK.padded(320, 4)
    assert PK.padded(154, 2) and PK.padded(144, 16) and PK.padded(608, 32)


@pytest.mark.parametrize("groups,cin", [(2, 154), (16, 144), (4, 320)])
def test_frozen_consumer_refuses_padded_planes(groups, cin):
    """functional.Consumer decides every frozen hand-off (IAO block links, DoReFa links and stem): a consumer that reads a
    group-padded plane gets no producer-written plane in any format"""
    from micronet_b200 import _lib as L, functional as F_, pk as PK
    spec = F_.ActSpec(L.ACT_DOREFA, bits=4)
    cons = F_.Consumer(None, spec, True, True, (64, cin // groups, 1, 1), (1, 1), (0, 0), (1, 1), groups, True)
    act = (8, cin, 16, 16)
    assert cons.accepts(act) == (not PK.padded(cin, groups))
    assert (cons.format(act) is None) == PK.padded(cin, groups)
    cons8 = F_.Consumer(None, spec, True, True, (64, cin // groups, 1, 1), (1, 1), (0, 0), (1, 1), groups, True, int8=True)
    if PK.padded(cin, groups):
        assert cons8.format(act) is None


def _block(cin, cout, k, groups, shuffle):
    from harness.models import ConvBNReLU
    return ConvBNReLU(cin, cout, k, 1, k // 2, groups=groups, channel_shuffle=shuffle, shuffle_groups=2)


@pytest.mark.parametrize("cfg", [[152, 168, 144], [160, 160, 144]], ids=["pruned", "aligned"])
def test_fused_producers_skip_padded_consumers(cfg):
    """fuse_blocks: no plane-only BatchNorm + binarizer (wbwtab) and no BatchNorm + ReLU + quantizer producer (DoReFa) in
    front of a conv that reads a group-padded plane (152 = 2 x 76 and 168 = 2 x 84 channels: whole octets overall, not per
    group)"""
    import copy
    import torch.nn as nn
    import micronet_b200 as E
    from micronet_b200 import fused as FU, pk as PK
    base = nn.Sequential(_block(3, cfg[0], 3, 1, 0), _block(cfg[0], cfg[1], 1, 2, 0), _block(cfg[1], cfg[2], 1, 2, 0))
    padded = PK.padded(cfg[0], 2)
    wb = E.wbwtab.prepare(copy.deepcopy(base), W=3, A=2, fuse_bn=True)
    prods = [m for m in wb.modules() if isinstance(m, FU.BatchNormBinarize2d)]
    assert len(prods) >= 2
    assert prods[0].plane_only == (not padded)
    df = E.dorefa.prepare(copy.deepcopy(base), a_bits=4, w_bits=4, fuse=True)
    n_fused = sum(isinstance(m, FU.BatchNormReluQuant2d) for m in df.modules())
    assert n_fused == (0 if padded else 2)
