"""Packed-operand convolutions (csrc/mnb_pk.cu) at the plans the bench models run, and at plans forced through the MNB_PK_*
knobs, against fp64 ATen convolutions of the same operands.

The small shapes of test_gpu_pk.py all run one M tile per work item.  Each case here first asks the host-side plan query
for the plan it was written for (N tile, M tiles per item, segmented accumulation, output phases, ...) and fails if the
heuristics now choose another one, instead of quietly testing something else.  Then:

* outputs start as NaN, consumer planes as 0xFF bytes, so a position or channel the epilogue never writes is caught;
* integer operands must be bit-exact (|sum| < 2^24), the 3-piece forward within 3e-6 of the largest element, and 2-piece
  backward results element-wise within c * R, R = the same convolution of |operands| in fp64 (c = 2^-15 for the data
  gradient, 2^-14 for the weight gradient, whose accumulation chains reach 256 MMAs; a dropped or doubled piece product
  is ~2^-8 R);
* a second launch must give bitwise-identical results (the reductions are deterministic)."""
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as TF

from tests import pk_plan_util as PU

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

C_DGRAD, C_WGRAD = 2.0 ** -15, 2.0 ** -14

# kind: "fwd" (mode 0), "dgrad" (mode 1), "wgrad"; shape: (B, C, H, W, K, R, stride, pad, groups); terms: (streamed operand,
# weight / x operand); expect: plan fields the case is pinned to; env: MNB_PK_* knobs; mask: STE mask on the data gradient
Case = namedtuple("Case", "id kind shape terms expect env mask", defaults=({}, False))

CASES = [
    # ---- natural multi-tile plans of the bench models, at reduced batch
    Case("gc3x3g16_fwd", "fwd", (32, 256, 16, 16, 512, 3, 1, 1, 16), (1, 1), dict(Nt=32, MT=4, segmented=0, ny=1)),
    Case("gc3x3g16_dgrad21_ste", "dgrad", (32, 256, 16, 16, 512, 3, 1, 1, 16), (2, 1), dict(Nt=16, MT=4, segmented=0, ny=1),
         mask=True),
    Case("gc3x3g32_fwd", "fwd", (8, 512, 8, 8, 1024, 3, 1, 1, 32), (1, 1), dict(Nt=32, MT=2, segmented=0, ny=1)),
    Case("gc3x3g32_dgrad21_ste", "dgrad", (8, 512, 8, 8, 1024, 3, 1, 1, 32), (2, 1), dict(Nt=16, MT=2, segmented=0, ny=1),
         mask=True),
    Case("res64_fwd33", "fwd", (64, 64, 32, 32, 64, 3, 1, 1, 1), (3, 3), dict(Nt=64, MT=2, segmented=1, ny=1)),
    Case("res64_fwd11", "fwd", (64, 64, 32, 32, 64, 3, 1, 1, 1), (1, 1), dict(Nt=64, MT=1, segmented=0, ny=1, col_tiles=2)),
    Case("res64_dgrad21", "dgrad", (64, 64, 32, 32, 64, 3, 1, 1, 1), (2, 1), dict(Nt=64, MT=2, segmented=1, ny=1)),
    Case("res64_dgrad22", "dgrad", (64, 64, 32, 32, 64, 3, 1, 1, 1), (2, 2), dict(Nt=64, MT=2, segmented=1, ny=1)),
    Case("stem_dgrad21", "dgrad", (64, 3, 32, 32, 64, 3, 1, 1, 1), (2, 1), dict(Nt=16, MT=2, segmented=1, ny=1)),
    Case("res128s2_dgrad21_ste", "dgrad", (64, 64, 32, 32, 128, 3, 2, 1, 1), (2, 1), dict(Nt=64, MT=2, segmented=0, ny=4),
         mask=True),
    Case("res128s2_dgrad22", "dgrad", (64, 64, 32, 32, 128, 3, 2, 1, 1), (2, 2), dict(Nt=64, MT=2, segmented=1, ny=4)),
    Case("res128sc_dgrad21", "dgrad", (32, 64, 32, 32, 128, 1, 2, 0, 1), (2, 1), dict(Nt=64, MT=2, segmented=0, ny=4)),
    Case("res256s2_dgrad21", "dgrad", (16, 128, 16, 16, 256, 3, 2, 1, 1), (2, 1), dict(Nt=128, MT=1, segmented=1, ny=4)),
    Case("res256sc_dgrad21_ste", "dgrad", (16, 128, 16, 16, 256, 1, 2, 0, 1), (2, 1), dict(Nt=128, MT=1, segmented=0, ny=4),
         mask=True),
    # ---- plans forced through the knobs: partial last M group, pipeline depth, column tiles, short segments
    Case("mt2_partial", "fwd", (3, 64, 28, 28, 64, 3, 1, 1, 1), (1, 1), dict(Nt=64, MT=2, n_mtiles=21, n_mgroups=11),
         {"MNB_PK_MT": "2"}),
    Case("mt4_partial", "fwd", (3, 64, 32, 32, 32, 3, 1, 1, 1), (1, 1), dict(Nt=32, MT=4, n_mtiles=30, n_mgroups=8),
         {"MNB_PK_MT": "4"}),
    Case("mt4_partial_seg", "fwd", (3, 64, 32, 32, 32, 3, 1, 1, 1), (3, 3),
         dict(Nt=32, MT=4, segmented=1, n_mtiles=33, n_mgroups=9), {"MNB_PK_MT": "4"}),
    Case("mt2_partial_seg48", "fwd", (3, 64, 32, 32, 48, 3, 1, 1, 1), (3, 3),
         dict(Nt=48, MT=2, segmented=1, n_mtiles=33, n_mgroups=17), {"MNB_PK_MT": "2"}),
    Case("mt2_dgrad21_ste", "dgrad", (3, 64, 28, 28, 48, 3, 1, 1, 1), (2, 1), dict(Nt=64, MT=2, n_mtiles=21, n_mgroups=11),
         {"MNB_PK_MT": "2"}, True),
    Case("stages2", "fwd", (4, 16, 8, 8, 32, 3, 1, 1, 1), (1, 1), dict(nstage=2), {"MNB_PK_STAGES": "2"}),
    Case("stages4", "fwd", (4, 16, 8, 8, 32, 3, 1, 1, 1), (1, 1), dict(nstage=4), {"MNB_PK_STAGES": "4"}),
    Case("stages8", "fwd", (4, 16, 8, 8, 32, 3, 1, 1, 1), (1, 1), dict(nstage=8), {"MNB_PK_STAGES": "8"}),
    Case("stages2_seg", "fwd", (3, 64, 16, 16, 64, 3, 1, 1, 1), (3, 3), dict(nstage=2, segmented=1), {"MNB_PK_STAGES": "2"}),
    Case("coltiles3", "fwd", (2, 32, 8, 24, 32, 3, 1, 1, 1), (1, 1), dict(col_tiles=3), {"MNB_PK_COLTILES": "3"}),
    Case("coltiles2_dgrad21", "dgrad", (2, 32, 16, 16, 48, 3, 1, 1, 1), (2, 1), dict(col_tiles=2), {"MNB_PK_COLTILES": "2"}),
    Case("seg_mmas8", "fwd", (3, 64, 16, 16, 64, 3, 1, 1, 1), (3, 3), dict(segmented=1, seg_len=1), {"MNB_PK_SEG_MMAS": "8"}),
    Case("seg_mmas8_dgrad22", "dgrad", (3, 64, 16, 16, 64, 3, 1, 1, 1), (2, 2), dict(segmented=1, seg_len=1),
         {"MNB_PK_SEG_MMAS": "8"}),
    Case("seg32_fwd", "fwd", (2, 64, 16, 16, 32, 3, 1, 1, 1), (3, 3), dict(Nt=32, MT=1, segmented=1)),
    Case("seg48_fwd", "fwd", (2, 64, 16, 16, 48, 3, 1, 1, 1), (3, 3), dict(Nt=48, MT=1, segmented=1)),
    # ---- weight gradient
    Case("wg_nc48", "wgrad", (2, 48, 16, 16, 64, 3, 1, 1, 1), (2, 1), dict(Nc=48, gm=1)),
    Case("wg_nc112", "wgrad", (2, 112, 16, 16, 64, 3, 1, 1, 1), (2, 1), dict(Nc=112, tpg=1, gm=1)),
    Case("wg_gc3x3g16_22", "wgrad", (16, 256, 16, 16, 512, 3, 1, 1, 16), (2, 2), dict(Nc=64, gm=4)),
    Case("wg_res64_21", "wgrad", (16, 64, 32, 32, 64, 3, 1, 1, 1), (2, 1), dict(Nc=64, tpg=2, gm=1)),
    Case("wg_stem_22", "wgrad", (16, 3, 32, 32, 64, 3, 1, 1, 1), (2, 2), dict(Nc=16, gm=1)),
    Case("wg_chain16", "wgrad", (8, 64, 16, 16, 64, 3, 1, 1, 1), (2, 1), dict(Nc=64, splits=32), {"MNB_PK_WG_CHAIN": "16"}),
    Case("wg_merge0", "wgrad", (4, 256, 8, 8, 512, 3, 1, 1, 16), (2, 1), dict(Nc=16, gm=1), {"MNB_PK_WG_MERGE": "0"}),
    Case("wg_nc48_forced", "wgrad", (2, 96, 16, 16, 64, 3, 1, 1, 1), (2, 1), dict(Nc=48, n_ctiles=2), {"MNB_PK_WG_NC": "48"}),
]


def plan_of(case):
    """the plan of a case (call with the case's environment set)"""
    sh = PU.shape(*case.shape)
    if case.kind == "wgrad":
        return PU.wgrad_plan(sh, *case.terms)
    return PU.conv_plan(sh, 0 if case.kind == "fwd" else 1, *case.terms)


def _ints(shape, gen, lim):
    return torch.randint(-lim, lim + 1, shape, generator=gen).double()


def _pieces(t, gen):
    """fp32 test data with full 24-bit significands"""
    return torch.randn(t, generator=gen, dtype=torch.float64).float().double()


def _run_twice(launch, out):
    from micronet_b200 import _lib as L
    res = []
    for _ in range(2):
        if out.dtype == torch.uint8:
            out.fill_(0xFF)
        else:
            out.fill_(float("nan"))
        L.check(launch(), "pk launch")
        torch.cuda.synchronize()
        res.append(out.clone())
    L.tc_check()
    if out.dtype != torch.uint8:
        assert not torch.isnan(res[0]).any(), "outputs the kernel never wrote"
    assert torch.equal(res[0], res[1]), "second launch differs: the result is not deterministic"
    return res[0]


def _elementwise(got, ref, R, c):
    assert not torch.isnan(got).any(), "outputs the kernel never wrote"
    err = (got.double() - ref).abs()
    ratio = (err / R.clamp_min(1e-300)).max().item()
    assert (err <= c * R).all(), f"worst err / R = {ratio:.3e} > c = {c:.3e}"
    return ratio


def _fwd(case):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = case.shape
    ta, tw = case.terms
    sh = PU.shape(*case.shape)
    g = torch.Generator().manual_seed(sum(map(ord, case.id)))
    if tw == 1:
        lim_x = 127 if ta == 1 else 500               # 2 pieces: levels of an asymmetric quantizer (code + zero point)
        lim_w = 127 if (Cc // G) * R * R * lim_x <= (1 << 24) // 127 else 15
        x, w = _ints((B, Cc, H, W), g, lim_x), _ints((K, Cc // G, R, R), g, lim_w)
        assert (Cc // G) * R * R * lim_x * lim_w < (1 << 24)
        img = PK.pack_weight(sh, 0, ta, tw, w_int=w.to(DEV, torch.int16))
    else:
        x, w = _pieces((B, Cc, H, W), g) * 2, (_pieces((K, Cc // G, R, R), g) * 0.1).float().double()
        img = PK.pack_weight(sh, 0, ta, tw, w_f32=w.float().to(DEV))
    x, w = x.to(DEV), w.to(DEV)
    x_pk, _ = PK.pack_act(x.float(), None, ta, phase_split=st == 2)
    ref = TF.conv2d(x, w, None, st, pad, 1, G)
    y = torch.empty(ref.shape, dtype=torch.float32, device=DEV)
    y = _run_twice(lambda: PK.conv(sh, 0, x_pk, ta, img, tw, y), y)
    if tw == 1:
        assert torch.equal(y.double(), ref), (y.double() - ref).abs().max().item()
    else:
        assert not torch.isnan(y).any()
        err = (y.double() - ref).abs().max().item() / ref.abs().max().item()
        assert err <= 3e-6, err


def _dgrad(case):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = case.shape
    ta, tw = case.terms
    sh = PU.shape(*case.shape)
    g = torch.Generator().manual_seed(sum(map(ord, case.id)))
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    dy = _pieces((B, K, P, Q), g).to(DEV)
    if tw == 1:                                      # integer weight levels, the scale folded into dy
        w_int = torch.randint(-127, 128, (K, Cc // G, R, R), generator=g, dtype=torch.int16).to(DEV)
        w_scale = (torch.rand(K, generator=g, dtype=torch.float64) * 0.02 + 0.001).float().to(DEV)
        w_scale[0] = 0.0                             # a dead channel contributes nothing
        wq = w_int.double() * w_scale.double().view(-1, 1, 1, 1)
        dy_pk, _ = PK.pack_act(dy.float(), None, ta, ch_scale=w_scale)
        img = PK.pack_weight(sh, 1, ta, tw, w_int=w_int, kzero=w_scale)
        # the packed dy is dy * w_scale rounded to fp32: that product is the operand the kernel is measured against
        dys = (dy.float() * w_scale.view(1, -1, 1, 1)).double()
        wo = w_int.double()
    else:                                            # fp32 weights in pieces (the statistics conv of QuantBNFuseConv2d)
        wq = _pieces((K, Cc // G, R, R), g).to(DEV) * 0.05
        dy_pk, _ = PK.pack_act(dy.float(), None, ta)
        img = PK.pack_weight(sh, 1, ta, tw, w_f32=wq.float())
        dys, wo = dy, wq.float().double()
    ref = torch.nn.grad.conv2d_input((B, Cc, H, W), wo, dys, st, pad, 1, G)
    Rb = torch.nn.grad.conv2d_input((B, Cc, H, W), wo.abs(), dys.abs(), st, pad, 1, G)
    bits8, gain = None, 1.0
    if case.mask:
        bits8 = torch.randint(0, 256, (B, (Cc + 7) // 8, H, W), generator=g, dtype=torch.uint8).to(DEV)
        keep = torch.stack([(bits8 >> j) & 1 for j in range(8)], dim=2).reshape(B, -1, H, W)[:, :Cc].double()
        gain = 0.1
        ref, Rb = ref * keep * gain, Rb * keep * gain
    dx = torch.empty((B, Cc, H, W), dtype=torch.float32, device=DEV)
    dx = _run_twice(lambda: PK.conv(sh, 1, dy_pk, ta, img, tw, dx, bits8=bits8, gain=gain), dx)
    ratio = _elementwise(dx, ref, Rb, C_DGRAD)
    print(f"{case.id}: worst err / R = {ratio:.3e}")


def _wgrad(case):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = case.shape
    td, tx = case.terms
    sh = PU.shape(*case.shape)
    g = torch.Generator().manual_seed(sum(map(ord, case.id)))
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    dy = _pieces((B, K, P, Q), g).to(DEV)
    if tx == 1:
        x = _ints((B, Cc, H, W), g, 127).to(DEV)
        kdiv = (torch.rand(K, generator=g, dtype=torch.float64) + 0.5).float().to(DEV)
        a_scale = torch.tensor([0.03125], device=DEV)          # a power of two: the reference scales exactly
        dy_pk, _ = PK.pack_act(dy.float(), None, td, ch_scale=kdiv)
        mul = 0.03125
        dys = (dy.float() * kdiv.view(1, -1, 1, 1)).double() / kdiv.double().view(1, -1, 1, 1)
    else:
        x = _pieces((B, Cc, H, W), g).to(DEV) * 2
        kdiv = a_scale = None
        dy_pk, _ = PK.pack_act(dy.float(), None, td)
        mul, dys = 1.0, dy
    x_pk, _ = PK.pack_act(x.float(), None, tx, phase_split=st == 2)
    ref = torch.nn.grad.conv2d_weight(x, (K, Cc // G, R, R), dys, st, pad, 1, G) * mul
    Rb = torch.nn.grad.conv2d_weight(x.abs(), (K, Cc // G, R, R), dys.abs(), st, pad, 1, G) * mul
    dw = torch.empty((K, Cc // G, R, R), dtype=torch.float32, device=DEV)
    dw = _run_twice(lambda: PK.wgrad(sh, dy_pk, td, x_pk, tx, dw, a_scale=a_scale, kdiv=kdiv), dw)
    ratio = _elementwise(dw, ref, Rb, C_WGRAD)
    print(f"{case.id}: worst err / R = {ratio:.3e}")


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_pinned_plan_matches_fp64(case, monkeypatch):
    for k, v in case.env.items():      # before the weight packer too: the image layout depends on the plan
        monkeypatch.setenv(k, v)
    plan = plan_of(case)
    assert plan is not None, f"{case.id}: shape outside the cover"
    got = {k: plan[k] for k in case.expect}
    assert got == case.expect, f"{case.id}: the plan changed: {got} != {case.expect} (full plan {plan})"
    {"fwd": _fwd, "dgrad": _dgrad, "wgrad": _wgrad}[case.kind](case)


# ---- fused consumer behind a segmented producer plan (frozen inference graphs)
# asymmetric IAO producer: its levels (code + zero point) take two bf16 pieces, so with 3x3 x 64 channels the K loop is
# segmented; the consumer is a symmetric IAO conv (one-piece plane)
POST_SHAPE = (4, 64, 16, 16, 128, 3, 1, 1, 1)
POST_PLAN = dict(segmented=1, npairs=2, Nt=128)


def _iao(scale, sym, dev=DEV):
    from micronet_b200 import _lib as L, functional as F_
    zp = 0.0 if sym else -101.0
    lo, hi = (-127.5 * scale, 127.5 * scale) if sym else ((0 + zp) * scale, (255 + zp) * scale)
    bufs = dict(scale=torch.tensor([scale]), zero_point=torch.tensor([zp]), obs_min=torch.tensor([lo]), obs_max=torch.tensor([hi]))
    return F_.ActSpec(L.ACT_IAO, qmin=-128 if sym else 0, qmax=127 if sym else 255, q_type=0 if sym else 1,
                      **{k: v.to(dev) for k, v in bufs.items()})


def _post_operands():
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = POST_SHAPE
    g = torch.Generator().manual_seed(21)
    x = (torch.randn(B, Cc, H, W, generator=g) * 3).to(DEV)
    w_int = torch.randint(-127, 128, (K, Cc, R, R), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) * 0.01 + 0.001).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    spec, nxt = _iao(0.05, False), _iao(0.11, True)
    sh = PU.shape(*POST_SHAPE)
    x_pk, _ = PK.pack_act(x, spec.struct(), 2)
    w_img = PK.pack_weight(sh, 0, 2, 1, w_int=w_int)
    y_ref = torch.empty(B, K, H, W, device=DEV)
    from micronet_b200 import _lib as L
    L.check(PK.conv(sh, 0, x_pk, 2, w_img, 1, y_ref, n_scale=w_scale, a_scale=spec.scale, bias=bias), "conv")
    return sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref


def _check_post(with_out):
    """mnb_pk_conv_post on the segmented plan either refuses it before launching or writes exactly what the unfused pair
    writes; it must never return success with the consumer plane (or y) left unwritten"""
    from micronet_b200 import _lib as L, pk as PK
    plan = PU.conv_plan(PU.shape(*POST_SHAPE), 0, 2, 1)
    assert {k: plan[k] for k in POST_PLAN} == POST_PLAN, plan
    sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref = _post_operands()
    B, Cc, H, W, K = POST_SHAPE[:5]
    for relu in (False, True):
        for split in (False, True):
            want, _ = PK.pack_act(y_ref, nxt.struct(), 1, phase_split=split, relu=relu)
            plane = PK.consumer_plane(B, K, H, W, DEV).fill_(0xFF)
            y = torch.full_like(y_ref, float("nan")) if with_out else None
            rc = PK.conv_post(sh, x_pk, 2, w_img, 1, y, nxt.struct(), plane, relu, split, n_scale=w_scale,
                              a_scale=spec.scale, bias=bias)
            torch.cuda.synchronize()
            if rc == L.E_UNSUPPORTED:
                assert (plane == 0xFF).all() and (y is None or torch.isnan(y).all()), "refused, yet something was written"
                continue
            L.check(rc, "conv_post")
            assert torch.equal(plane, want), ("consumer plane", relu, split)
            if with_out:
                assert torch.equal(y, y_ref), ("y", relu, split)
    L.tc_check()


def test_conv_post_on_a_segmented_producer_plan_with_out():
    _check_post(True)


def test_conv_post_on_a_segmented_producer_plan_plane_only():
    _check_post(False)


@pytest.mark.parametrize("only", [False, True], ids=["y_kept", "plane_only"])
def test_frozen_conv_behind_an_asymmetric_producer_hands_the_right_plane(only):
    """functional.frozen_conv with a consumer: whatever path it takes, y equals the plain conv and the plane the consumer
    reads equals the consumer's own quantizer applied to y"""
    from micronet_b200 import functional as F_, pk as PK
    sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref = _post_operands()
    B, Cc, H, W, K, R, st, pad, G = POST_SHAPE
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    consumer_mod = torch.nn.Identity()
    for relu in (False, True):
        cons = F_.Consumer(consumer_mod, nxt, relu, only, (K, K, 3, 3), (1, 1), (1, 1), (1, 1), 1, True)
        assert cons.accepts((B, K, H, W))
        y = F_.frozen_conv(x, None, wq, bias, w_int, w_scale, spec, (1, 1), (1, 1), (1, 1), 1, consumer=cons)
        torch.cuda.synchronize()
        plane = F_.handed_plane(consumer_mod, y)
        want, _ = PK.pack_act(y_ref, nxt.struct(), 1, relu=relu)
        if plane is None:            # not fused: y holds the data, the consumer packs it itself
            assert torch.equal(y, y_ref)
            got, _ = PK.pack_act(y, nxt.struct(), 1, relu=relu)
            assert torch.equal(got, want)
        else:
            assert torch.equal(plane, want), relu
            if y.device.type != "meta":
                assert torch.equal(y, y_ref)
