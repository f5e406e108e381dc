"""Grouped convolutions with any number of channels per group on the packed-operand family: group-padded operand planes
(DESIGN.md 4.17), from the packer up to the QAT step of a channel-pruned NIN-GC.

Kernel level: the six padded layers of the reference README's pruned NIN-GC (cfg 154 162 144 304 320 320 608 584) at a
small batch and edge shapes against fp64, with the packed-operand family's bounds: integer operands exact, three fp32 pieces to fp32
rounding, two dy pieces within 2^-15 (data gradient) / 2^-14 (weight gradient) of the same convolution of the absolute
values.  Module and model level: the layers take ``family == "pk"`` and no generic kernel, with results against the oracle;
CUDA-graph replay against eager steps; frozen inference against the un-frozen eval forward."""
import copy

import pytest
import torch
import torch.nn.functional as TF

from tests.pk_plan_util import within
from tests.test_pk_pruned_cpu import README_CFG, pruned_convs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_DGRAD, C_WGRAD = 2.0 ** -15, 2.0 ** -14

# B, C, H, W, K, R, stride, pad, groups
README_SHAPES = [(2,) + c[2:] for c in pruned_convs() if c[0] != "L5"]
EDGE_SHAPES = [
    (2, 4, 12, 12, 16, 3, 1, 1, 4),       # 1 input channel per group
    (2, 28, 10, 10, 20, 3, 1, 1, 4),      # 7 / 5
    (2, 36, 8, 8, 64, 1, 1, 0, 4),        # 9 / 16
    (2, 34, 16, 16, 6, 3, 2, 1, 2),       # 17 / 3, stride 2
    (2, 32, 16, 16, 44, 1, 2, 0, 4),      # 8 / 11: only the output side padded, stride-2 1x1
    (3, 154, 9, 9, 162, 1, 1, 0, 2),      # odd image: several images per M tile
]
SHAPES = README_SHAPES + EDGE_SHAPES
IDS = ["x".join(map(str, s)) for s in SHAPES]


def _sh(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, st, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def _unpack(planes, terms, B, Cc, G, H, W):
    """-> (values [B, C, H, W], padding channels [B, G, pad, H, W]) of a group-padded plane"""
    cg = Cc // G
    k8 = (cg + 7) // 8
    t = planes.view(torch.bfloat16).view(terms, B, G, k8, H, W, 8).float().sum(0)
    t = t.permute(0, 1, 2, 5, 3, 4).reshape(B, G, k8 * 8, H, W)
    return t[:, :, :cg].reshape(B, Cc, H, W), t[:, :, cg:]


def _unbits(bits8, B, Cc, G, H, W):
    cg = Cc // G
    k8 = (cg + 7) // 8
    t = torch.stack([(bits8.view(B, G, k8, H, W) >> j) & 1 for j in range(8)], dim=3).reshape(B, G, k8 * 8, H, W)
    return t[:, :, :cg].reshape(B, Cc, H, W), t[:, :, cg:]


def _seed(shape, k):
    return torch.Generator().manual_seed(abs(hash(shape)) % (1 << 31) + k)


@pytest.mark.parametrize("cg,G", [(1, 4), (7, 3), (9, 2), (17, 2), (77, 2), (19, 16)])
def test_grouped_planes_hold_exact_pieces_levels_and_masks(cg, G):
    from micronet_b200 import _lib as L, functional as F_, pk as PK
    g = torch.Generator().manual_seed(cg * 31 + G)
    B, H, W, Cc = 2, 6, 10, cg * G
    x = (torch.randn(B, Cc, H, W, generator=g) * 3).to(DEV)
    sc = (torch.rand(Cc, generator=g) + 0.5).to(DEV)
    for terms in (1, 2, 3):
        planes, _ = PK.pack_act(x, None, terms, ch_scale=sc, groups=G)
        assert planes.numel() == int(L.load().mnb_pk_grouped_act_bytes(B, Cc, H, W, terms, G))
        back, pad = _unpack(planes, terms, B, Cc, G, H, W)
        want = x * sc.view(1, -1, 1, 1)
        err = (back - want).abs().max().item() / want.abs().max().item()
        assert err <= (2.0 ** -8, 2.0 ** -16, 0.0)[terms - 1] * 1.01, (terms, err)
        assert not pad.any()
    # DoReFa levels round(clamp(0.1 x, 0, 1) * 15) and the STE mask: 0.1 x = (k + 0.25) / 15 lies inside [0, 1], and some
    # inputs outside it (clamped, no pass)
    from oracle import reference_port as O
    lv = torch.randint(0, 15, (B, Cc, H, W), generator=g).float()
    xq = (lv + 0.25) / 1.5
    out = torch.rand(B, Cc, H, W, generator=g) < 0.2
    xq = torch.where(out, torch.where(lv > 7, 15.0, -5.0), xq)
    want = O.dorefa_activation_levels(xq, 4).to(DEV)
    xq = xq.to(DEV)
    qp = F_.ActSpec(L.ACT_DOREFA, bits=4).struct()
    for split in (False, True):
        planes, bits8 = PK.pack_act(xq, qp, 1, want_bits=True, groups=G, phase_split=split)
        if split:      # octet (h%2*2 + w%2) * C8 + c/8 of an [H/2, W/2] plane
            k8 = (cg + 7) // 8
            ph = planes.view(torch.bfloat16).view(B, 4, G, k8, H // 2, W // 2, 8).float()
            for a in range(2):
                for b in range(2):
                    got = ph[:, a * 2 + b].permute(0, 1, 2, 5, 3, 4).reshape(B, G, k8 * 8, H // 2, W // 2)
                    assert torch.equal(got[:, :, :cg].reshape(B, Cc, H // 2, W // 2), want[:, :, a::2, b::2])
                    assert not got[:, :, cg:].any()
            continue
        levels, pad = _unpack(planes, 1, B, Cc, G, H, W)
        assert torch.equal(levels, want) and not pad.any()
        passed, bpad = _unbits(bits8, B, Cc, G, H, W)
        assert torch.equal(passed.bool(), ~out.to(DEV)) and not bpad.any()


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_forward_integer_operands_are_exact(shape):
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    g = _seed(shape, 0)
    x = torch.randint(-127, 128, (B, Cc, H, W), generator=g).float().to(DEV)
    w = torch.randint(-127, 128, (K, Cc // G, R, R), generator=g).float().to(DEV)
    sh = _sh(shape)
    x_pk, _ = PK.pack_act(x, None, 1, phase_split=st == 2, groups=G)
    img = PK.pack_weight(sh, 0, 1, 1, w_int=w.to(torch.int16))
    ref = TF.conv2d(x.double(), w.double(), None, st, pad, 1, G)
    y = torch.full(ref.shape, float("nan"), dtype=torch.float32, device=DEV)
    L.check(PK.run_conv(sh, 0, x_pk, 1, img, 1, y), "pk_conv")
    torch.cuda.synchronize()
    L.tc_check()
    assert torch.equal(y.double(), ref), (y.double() - ref).abs().max().item()


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_forward_fp32_operands_scale_and_bias(shape):
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    g = _seed(shape, 1)
    x = (torch.randn(B, Cc, H, W, generator=g) * 2).to(DEV)
    w = (torch.randn(K, Cc // G, R, R, generator=g) * 0.1).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    nsc = (torch.rand(K, generator=g) + 0.5).to(DEV)
    sh = _sh(shape)
    x_pk, _ = PK.pack_act(x, None, 3, phase_split=st == 2, groups=G)
    img = PK.pack_weight(sh, 0, 3, 3, w_f32=w)
    ref = TF.conv2d(x.double(), w.double(), None, st, pad, 1, G) * (0.25 * nsc.double()).view(1, -1, 1, 1) \
        + bias.double().view(1, -1, 1, 1)
    y = torch.full(ref.shape, float("nan"), dtype=torch.float32, device=DEV)
    L.check(PK.conv(sh, 0, x_pk, 3, img, 3, y, n_scale=nsc, a_scale_const=0.25, bias=bias), "pk_conv")
    torch.cuda.synchronize()
    L.tc_check()
    err = (y.double() - ref).abs().max().item() / ref.abs().max().item()
    assert err <= 3e-6, err


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_data_gradient_with_ste_mask(shape):
    """two dy pieces (the models' PK_TERMS_BWD) with the per-channel weight scale folded in, STE mask in the padded layout"""
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    g = _seed(shape, 2)
    terms = 2
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    dy = torch.randn(B, K, P, Q, generator=g).to(DEV)
    w_int = torch.randint(-127, 128, (K, Cc // G, R, R), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) * 0.02 + 0.001).to(DEV)
    w_scale[0] = 0.0                       # a dead channel contributes nothing
    wq = w_int.double() * w_scale.double().view(-1, 1, 1, 1)
    ref = torch.nn.grad.conv2d_input((B, Cc, H, W), wq, dy.double(), st, pad, 1, G)
    sh = _sh(shape)
    dy_pk, _ = PK.pack_act(dy, None, terms, ch_scale=w_scale, groups=G)
    _, dpad = _unpack(dy_pk, terms, B, K, G, P, Q)
    assert not dpad.any()
    img = PK.pack_weight(sh, 1, terms, 1, w_int=w_int, kzero=w_scale)
    dys = (dy * w_scale.view(1, -1, 1, 1)).double()
    Rb = torch.nn.grad.conv2d_input((B, Cc, H, W), w_int.double().abs(), dys.abs(), st, pad, 1, G)
    k8 = (Cc // G + 7) // 8
    bits8 = torch.randint(0, 256, (B, G * k8, H, W), generator=g, dtype=torch.uint8).to(DEV)   # padding bits set too
    keep = _unbits(bits8, B, Cc, G, H, W)[0].double()
    ref, Rb = ref * keep * 0.1, Rb * keep * 0.1
    dx = torch.full((B, Cc, H, W), float("nan"), dtype=torch.float32, device=DEV)
    L.check(PK.run_conv(sh, 1, dy_pk, terms, img, 1, dx, bits8=bits8, gain=0.1), "pk_conv dgrad")
    torch.cuda.synchronize()
    L.tc_check()
    print(f"worst err / R = {within(dx, ref, Rb, C_DGRAD):.3e}")


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
@pytest.mark.parametrize("kind", ["levels", "fp32"])
def test_weight_gradient(shape, kind):
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    g = _seed(shape, 3)
    terms = 2
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    dy = torch.randn(B, K, P, Q, generator=g).to(DEV)
    sh = _sh(shape)
    tx = 1 if kind == "levels" else terms
    assert PK.wgrad_supported(sh, terms, tx)
    if kind == "levels":
        x = torch.randint(-128, 128, (B, Cc, H, W), generator=g).float().to(DEV)
        a_scale = torch.tensor([0.031], device=DEV)
        kdiv = (torch.rand(K, generator=g) + 0.5).to(DEV)
        dy_pk, _ = PK.pack_act(dy, None, terms, ch_scale=kdiv, groups=G)
        mul = 0.031
        dys = (dy * kdiv.view(1, -1, 1, 1)).double() / kdiv.double().view(1, -1, 1, 1)
    else:
        x = (torch.randn(B, Cc, H, W, generator=g) * 2).to(DEV)
        a_scale, kdiv, mul = None, None, 1.0
        dy_pk, _ = PK.pack_act(dy, None, terms, groups=G)
        dys = dy.double()
    x_pk, _ = PK.pack_act(x, None, tx, phase_split=st == 2, groups=G)
    ref = torch.nn.grad.conv2d_weight(x.double(), (K, Cc // G, R, R), dys, st, pad, 1, G) * mul
    dw = torch.full((K, Cc // G, R, R), float("nan"), dtype=torch.float32, device=DEV)
    L.check(PK.run_wgrad(sh, dy_pk, terms, x_pk, tx, dw, a_scale=a_scale, kdiv=kdiv), "pk_wgrad")
    torch.cuda.synchronize()
    L.tc_check()
    Rb = torch.nn.grad.conv2d_weight(x.double().abs(), (K, Cc // G, R, R), dys.abs(), st, pad, 1, G) * mul
    print(f"worst err / R = {within(dw, ref, Rb, C_WGRAD):.3e}")


# ---- module level: one padded layer per scheme against the oracle port
def _layer_pair(scheme, cin, cout, k, groups):
    import micronet_b200 as E
    from oracle import reference_port as O
    torch.manual_seed(7)
    pad = k // 2
    if scheme == "dorefa":
        e = E.dorefa.QuantConv2d(cin, cout, k, padding=pad, groups=groups, a_bits=4, w_bits=4)
        o = O.DorefaQuantConv2d(cin, cout, k, padding=pad, groups=groups, a_bits=4, w_bits=4)
    elif scheme == "iao":
        e = E.iao.QuantConv2d(cin, cout, k, padding=pad, groups=groups, bias=False)
        o = O.IaoQuantConv2d(cin, cout, k, padding=pad, groups=groups, bias=False)
    else:
        e = E.wbwtab.QuantConv2d(cin, cout, k, padding=pad, groups=groups, W=3)
        o = O.WbQuantConv2d(cin, cout, k, padding=pad, groups=groups, W=3)
    o.load_state_dict(e.state_dict())
    return e.to(DEV), o


@pytest.mark.parametrize("scheme", ["dorefa", "iao", "wbwtab"])
@pytest.mark.parametrize("layer", ["L1", "L3", "L6"])
def test_module_runs_padded_layers_on_the_packed_family(scheme, layer):
    from micronet_b200 import _lib as L, functional as F_
    _, _, cin, hw, _, cout, k, _, _, groups = next(c for c in pruned_convs() if c[0] == layer)
    e, o = _layer_pair(scheme, cin, cout, k, groups)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(4, cin, hw, hw, generator=g) * 2
    if scheme == "wbwtab":
        x = torch.where(x >= 0, 1.0, -1.0)              # a binarizer's output
    xe = x.to(DEV).requires_grad_(True)
    if scheme == "wbwtab":
        xe_in = xe * 1.0
        xe_in._mnb_pm1 = True
    else:
        xe_in = xe
    xo = x.clone().requires_grad_(True)
    e.train(); o.train()
    F_.TIMER = F_.KernelTimer()
    try:
        ye = e(xe_in)
        yo = o(xo)
        gy = torch.randn(yo.shape, generator=g)
        ye.backward(gy.to(DEV))
        yo.backward(gy)
        torch.cuda.synchronize()
        kinds = {kd for kd, _, _, _ in F_.TIMER.records}
    finally:
        F_.TIMER = None
    L.tc_check()
    assert {"fwd_pk", "dgrad_pk", "wgrad_pk"} <= kinds, kinds
    assert not kinds & {"fwd", "dgrad", "wgrad", "fwd_tc", "dgrad_tc", "wgrad_tc"}, kinds
    # output and data gradient within 1e-5 of the largest element, the weight gradient (two dy pieces, long reductions)
    # within 2e-5 as smoke() holds the packed-operand family's
    for what, a, b, tol in (("y", ye, yo, 1e-5), ("dx", xe.grad, xo.grad, 1e-5), ("dw", e.weight.grad, o.weight.grad, 2e-5)):
        rel = (a.detach().cpu() - b.detach()).abs().max().item() / b.detach().abs().max().item()
        assert rel <= tol, (scheme, layer, what, rel)


# ---- model level: QAT steps of the README-cfg NIN-GC
def _pruned(scheme):
    from harness import models as zoo, train as H
    torch.manual_seed(1)
    base = zoo.init_like_reference(zoo.NINGC(README_CFG))
    if scheme == "wbwtab":
        kw, extra = dict(W=3, A=2), dict(fuse_bn=True)
    else:
        kw, extra = dict(a_bits=4, w_bits=4), dict(fuse=True)
    eng = H.prepare_engine(copy.deepcopy(base), scheme, **kw, **extra).to(DEV)
    ora = H.prepare_oracle(copy.deepcopy(base), scheme, **kw)
    return eng, ora


def _grouped_shapes():
    """ConvShape tuples of the quantized grouped convs of the README-cfg NIN-GC at batch 32"""
    from micronet_b200 import _lib as L
    out = set()
    for _, _, Cc, H, W, K, R, st, pad, G in pruned_convs(batch=32):
        out.add(tuple(getattr(L.ConvShape(32, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G), f)
                      for f, _ in L.ConvShape._fields_))
    return out


@pytest.mark.parametrize("scheme", ["wbwtab", "dorefa"])
def test_pruned_qat_step_on_the_packed_family(scheme):
    from harness import train as H
    from micronet_b200 import _lib as L, functional as F_
    eng, ora = _pruned(scheme)
    x, t = H.synthetic_batch(32, 32, seed=3)
    eng.train(); ora.train()
    # teacher forcing: every padded conv's input as the engine saw it, fed to the oracle's conv of the same name (a
    # binarized graph amplifies a sign flip of a BatchNorm output at zero into different logits, so the logits of the two
    # graphs are not compared; L5 reads a fused producer's plane, its fp32 input is never written)
    from micronet_b200 import pk as PK
    seen_io, hooks = {}, []
    for name, m in eng.named_modules():
        if isinstance(m, torch.nn.Conv2d) and (PK.padded(m.in_channels, m.groups) or PK.padded(m.out_channels, m.groups)):
            hooks.append(m.register_forward_hook(
                lambda mod, inp, out, name=name: seen_io.__setitem__(
                    name, (F_.materialized(inp[0]).detach().cpu(), F_.materialized(out).detach().cpu()))))
    F_.TIMER = F_.KernelTimer()
    try:
        ye = eng(x.to(DEV))
        TF.cross_entropy(ye, t.to(DEV)).backward()
        torch.cuda.synchronize()
        recs = [(kd, shp) for kd, shp, _, _ in F_.TIMER.records]
    finally:
        F_.TIMER = None
        for hk in hooks:
            hk.remove()
    L.tc_check()
    ora_mods = dict(ora.named_modules())
    assert len(seen_io) == 6, sorted(seen_io)
    with torch.no_grad():
        for name, (inp, got) in seen_io.items():
            want = ora_mods[name](inp)
            rel = (got - want).abs().max().item() / want.abs().max().item()
            assert rel <= 1e-5, (scheme, name, rel)
    grouped = _grouped_shapes()
    seen = {shp for _, shp in recs if shp in grouped}
    assert seen == grouped, grouped - seen
    kinds = {kd for kd, shp in recs if shp in grouped}
    assert kinds <= {"fwd_pk", "dgrad_pk", "wgrad_pk"}, kinds     # no generic or round-1 kernel
    assert {"fwd_pk", "dgrad_pk", "wgrad_pk"} <= kinds


@pytest.mark.parametrize("scheme", ["wbwtab", "dorefa"])
def test_pruned_graph_replay_equals_eager_steps(scheme):
    from harness import train as H
    from micronet_b200 import _lib as L

    def run(graph):
        eng, _ = _pruned(scheme)
        st = H.QatStepper(eng, lr=0.01, wd=1e-5, flat=True, graph=graph, graph_warmup=2)
        losses = []
        for i in range(5):
            x, t = H.synthetic_batch(32, 32, seed=40 + i % 2, device=DEV)
            losses.append(st.step(x, t).detach().clone())
        torch.cuda.synchronize()
        if graph:
            assert st.graph is not None, st.graph_error
        return torch.stack(losses).cpu(), [p.detach().cpu().clone() for p in eng.parameters()]

    le, pe = run(False)
    lg, pg = run(True)
    L.tc_check()
    assert torch.equal(le, lg), (le, lg)
    assert all(torch.equal(a, b) for a, b in zip(pe, pg))


# ---- frozen inference of the pruned model
def _calibrated_iao():
    import micronet_b200 as E
    from harness import models as zoo, train as H
    torch.manual_seed(1)
    base = zoo.init_like_reference(zoo.NINGC(README_CFG))
    m = E.iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True).to(DEV)
    m.train()
    with torch.no_grad():
        for i in range(2):
            m(H.synthetic_batch(32, 32, seed=20 + i, device=DEV)[0])
    return m.eval()


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_frozen_iao_pruned_logits(i8):
    from harness import train as H
    from micronet_b200 import _lib as L, functional as F_, iao
    m = _calibrated_iao()
    x = H.synthetic_batch(16, 32, seed=5, device=DEV)[0]
    with torch.no_grad():
        plain = m(x)
    off = copy.deepcopy(m)
    iao.freeze_inference(off, handoff=False, int8=i8)
    iao.freeze_inference(m, int8=i8)
    F_.TIMER = F_.KernelTimer()
    try:
        with torch.no_grad():
            want, got = off(x), m(x)
        torch.cuda.synchronize()
        recs = [(kd, shp) for kd, shp, _, _ in F_.TIMER.records]
    finally:
        F_.TIMER = None
    L.tc_check()
    assert torch.equal(got, want)
    if not i8:
        assert torch.equal(got, plain)        # the un-frozen eval forward, bit for bit
    else:                                     # int8 where the int8 plan covers a layer (L5 only): levels equal, fp32 sums
        rel = (got - plain).abs().max().item() / plain.abs().max().item()
        assert rel <= 1e-5, rel
    grouped = {s[1:] for s in _grouped_shapes()}
    kinds = {kd for kd, shp in recs if shp[1:] in grouped}
    assert "fwd" not in kinds and "fwd_tc" not in kinds, kinds
    iao.freeze_inference(m, enable=False)


def test_frozen_dorefa_pruned_logits():
    from harness import models as zoo, train as H
    import micronet_b200 as E
    from micronet_b200 import _lib as L
    torch.manual_seed(1)
    base = zoo.init_like_reference(zoo.NINGC(README_CFG))
    m = E.dorefa.prepare(base, a_bits=4, w_bits=4, fuse=True).to(DEV)
    m.train()
    with torch.no_grad():
        m(H.synthetic_batch(16, 32, seed=21, device=DEV)[0])
    m.eval()
    x = H.synthetic_batch(8, 32, seed=4, device=DEV)[0]
    with torch.no_grad():
        plain = m(x)
    E.dorefa.freeze_inference(m)
    with torch.no_grad():
        got = m(x)
    torch.cuda.synchronize()
    L.tc_check()
    # the padded consumers take no link (their producers write fp32 and ATen's BatchNorm runs as un-frozen); the one link
    # left (L4 -> L5: 76 -> 80 channels per group, consumer not padded) applies BatchNorm in the epilogue, where a level on a
    # rounding boundary may differ by one from ATen's (DESIGN.md 4.15): logits close, not bitwise
    rel = (got - plain).abs().max().item() / plain.abs().max().item()
    assert rel <= 2e-2, rel
    E.dorefa.freeze_inference(m, enable=False)
    with torch.no_grad():
        assert torch.equal(m(x), plain)
