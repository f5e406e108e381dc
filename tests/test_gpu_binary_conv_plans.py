"""The two binary forward convolutions (csrc/mnb_xnor.cu, csrc/mnb_b1.cu) at every case of tests/binary_conv_cases.py: each
kernel instance, plan feature and frozen-model layer the list pins.

Forward: the plan is the pinned one; with alpha = 1 and no bias the fp32 output (started as NaN) equals the fp64
convolution of the +-1 / {-1, 0, +1} tensors exactly (binary and ternary weights, an all-zero output channel, +0 and -0
inputs); with alpha and bias it is byte-equal to the packed-operand tensor-core forward and to the other binary kernel where
both cover the shape, and within one ulp of fp64 S * alpha + bias (mnb_pk_conv has no plan for 1x1 convolutions with
padding: those small cases are compared whole in fp64).  Batch-256 cases compare a few images in fp64 (at M-tile and
image-block boundaries and the last image) and the whole tensor against mnb_pk_conv.
Epilogue: the output buffer starts as 0xFF bytes; every format decodes to the un-fused BatchNorm -> sign -> pool -> shuffle
sequence and is byte-equal to its packer's plane of those signs (padding bits zero).
Every case runs twice with bitwise-identical results and leaves the tensor-core error flag clean.

Also: the b1 plane max-pool against ATen at every pool freeze_inference hands it, and the frozen README-cfg pruned NIN-GC
(wbwtab W3/A2 and W2/A2) against its un-frozen eval forward and, teacher-forced, against the oracle."""
import copy
import zlib

import pytest
import torch
import torch.nn.functional as TF

from harness import models as zoo
from tests import binary_conv_cases as BC, pk_plan_util as PU
from tests.test_gpu_wbwtab_frozen import _bn, _bn_sign

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _kmod(kernel):
    from micronet_b200 import b1 as B1, xnor as X
    return X if kernel == "xnor" else B1


def _operands(shape, seed, ternary):
    B, Cc, H, W, K, R, st, pad, G = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cc, H, W, generator=g)
    x[0, 0, 0, 0] = 0.0                 # sign(0) -> +1 (WB:15-16)
    x[-1, -1, -1, -1] = -0.0
    x[0, :, H // 2, W // 2] = -0.0      # a pixel of -0.0 in every channel
    if ternary:
        w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g)
    else:
        w = torch.randint(0, 2, (K, Cc // G, R, R), generator=g) * 2 - 1
    w[min(1, K - 1)] = 0                 # an all-zero output channel
    alpha = torch.rand(K, generator=g) * 0.05 + 0.01
    bias = torch.randn(K, generator=g)
    return x.to(DEV), w.to(torch.int16).to(DEV), alpha.to(DEV), bias.to(DEV), g


def _fwd(kernel, shape, x, w, alpha, bias, ops=None):
    """fp32 forward of ``kernel`` (output started as NaN); ops: cached (activation plane, weight image)"""
    from micronet_b200 import _lib as L
    K_ = _kmod(kernel)
    sh = BC.conv_shape(shape)
    G = shape[8]
    if ops is None:
        ops = (K_.pack_act(x, G), K_.pack_weight(sh, w))
    P_, Q_ = BC.out_hw(shape)
    y = torch.full((shape[0], shape[4], P_, Q_), float("nan"), device=DEV)
    L.check(K_.conv(sh, ops[0], ops[1], y, alpha=alpha, bias=bias), f"{kernel} conv")
    return y, ops


def _pk_fwd(shape, x, w, alpha, bias):
    from micronet_b200 import _lib as L, pk as PK
    sh = BC.conv_shape(shape)
    planes = PK.pack_act(torch.where(x < 0, -1.0, 1.0), None, 1, groups=shape[8])[0]
    P_, Q_ = BC.out_hw(shape)
    y = torch.full((shape[0], shape[4], P_, Q_), float("nan"), device=DEV)
    L.check(PK.conv(sh, 0, planes, 1, PK.pack_weight(sh, 0, 1, 1, w_int=w), 1, y, n_scale=alpha, bias=bias), "pk conv")
    return y


def _images(case):
    """the images compared in fp64: all of a small batch; at batch 256 the first two, the last two, both sides of the
    middle and of the first M-tile boundary (b1: TB images per M tile)"""
    B = case.shape[0]
    if B <= 8:
        return list(range(B))
    tb = BC.plan_of(case.kernel, case.shape)["TB"] if case.kernel == "b1" else 1
    return sorted({0, 1, tb - 1, tb, B // 2 - 1, B // 2, B - 2, B - 1})


def _ulp(y):
    a = y.abs()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


def _seed(case):
    return zlib.crc32(case.id.encode())


def _check_forward(case, ternary):
    """the forward checks of one case; returns (x, w, alpha, bias, y, ops) of the alpha / bias run"""
    from micronet_b200 import b1 as B1, xnor as X
    B, Cc, H, W, K, R, st, pad, G = case.shape
    x, w, alpha, bias, g = _operands(case.shape, _seed(case) + int(ternary), ternary)
    idx = _images(case)
    ref = TF.conv2d(torch.where(x[idx] < 0, -1.0, 1.0).double().cpu(), w.double().cpu(), None, st, pad, 1, G)
    # exact integer sums
    y1, ops = _fwd(case.kernel, case.shape, x, w, torch.ones_like(alpha), None)
    assert torch.equal(y1[idx].cpu().double(), ref), case.id
    # alpha and bias: the fmaf epilogue, one rounding of S * alpha + bias
    y, _ = _fwd(case.kernel, case.shape, x, w, alpha, bias, ops)
    want = ref * alpha.double().cpu().view(1, -1, 1, 1) + bias.double().cpu().view(1, -1, 1, 1)
    yi = y[idx].cpu()
    assert bool(((yi.double() - want).abs() <= _ulp(yi).double()).all()), case.id
    # the packed-operand forward, where it covers the shape (not 1x1 with padding, not the grouped stride-2 case); every
    # case it leaves out has a batch small enough for the whole tensor to be compared in fp64 above
    if PU.conv_plan(BC.conv_shape(case.shape), 0, 1, 1) is not None:
        assert torch.equal(y, _pk_fwd(case.shape, x, w, alpha, bias)), case.id
    else:
        assert B <= 8, case.id
    other = "b1" if case.kernel == "xnor" else "xnor"
    if (B1 if other == "b1" else X).supported(BC.conv_shape(case.shape)):
        assert torch.equal(y, _fwd(other, case.shape, x, w, alpha, bias)[0]), case.id
    again, _ = _fwd(case.kernel, case.shape, x, w, alpha, bias, ops)
    assert torch.equal(again, y), case.id
    return x, w, alpha, bias, y, ops, g


def _signs(y, bn, pool, sg):
    s = _bn_sign(y, bn)
    if pool:
        s = TF.max_pool2d(s, 2, 2)
    if sg > 1:
        s = zoo.shuffle_channels(s, sg)
    return s.contiguous()


def _run_post(kernel, case, ops, alpha, bias, bn):
    from micronet_b200 import _lib as L
    K_ = _kmod(kernel)
    sh = BC.conv_shape(case.shape)
    ps = BC.post_struct(case.post, bn)
    n = K_.post_bytes(sh, ps)
    assert n > 0, case.id
    out = torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV)        # unwritten or un-cleared bits show
    L.check(K_.conv_post(sh, ops[0], ops[1], ps, out, alpha=alpha, bias=bias), f"{kernel} conv_post")
    return out


def _check_post(case, x, w, alpha, bias, y, ops, g):
    from micronet_b200 import b1 as B1, xnor as X
    post = case.post
    K = case.shape[4]
    bn = _bn(K, g) if post.bn else None
    out = _run_post(case.kernel, case, ops, alpha, bias, bn)
    want = _signs(y, bn, post.pool, post.sg)
    b, c, h, ww = want.shape
    if post.fmt == "bits":
        assert torch.equal(X.unpack(out.view(torch.int32), want.shape, post.og), want), case.id
        assert torch.equal(out.view(torch.int32), X.pack_act(want, post.og)), case.id
    elif post.fmt == "b1":
        assert torch.equal(B1.unpack(out.view(torch.int32), want.shape, post.og), want), case.id
        assert torch.equal(out.view(torch.int32), B1.pack_act(want, post.og)), case.id
    else:
        plane = want.view(b, c // 8, 8, h, ww).permute(0, 1, 3, 4, 2).contiguous().to(torch.bfloat16)
        assert torch.equal(out.view(torch.bfloat16).view(b, c // 8, h, ww, 8).float(), plane.float()), case.id
        assert torch.equal(out, plane.view(torch.uint8).view(-1)), case.id
    assert torch.equal(_run_post(case.kernel, case, ops, alpha, bias, bn), out), case.id     # deterministic
    # the other kernel's epilogue, where it covers the shape and writes the format
    other = "b1" if case.kernel == "xnor" else "xnor"
    if post.fmt != "b1" and BC.plan_of(other, case.shape, post) is not None:
        O = _kmod(other)
        oops = (O.pack_act(x, case.shape[8]), O.pack_weight(BC.conv_shape(case.shape), w))
        assert torch.equal(_run_post(other, case, oops, alpha, bias, bn), out), case.id


@pytest.mark.parametrize("case", BC.CASES, ids=[c.id for c in BC.CASES])
def test_case(case):
    assert BC.plan_tuple(case.kernel, BC.plan_of(case.kernel, case.shape, case.post)) == tuple(case.plan), case.id
    _check_forward(case, ternary=False)
    x, w, alpha, bias, y, ops, g = _check_forward(case, ternary=True)
    if case.post is not None:
        _check_post(case, x, w, alpha, bias, y, ops, g)


def _freeze_pools():
    """every (k, s, p) wbwtab.freeze_inference hands to the b1 plane pool: MaxPool2d of the engine's cover (square,
    k <= 15, 2p <= k, floor mode) other than the folded 2x2 / 2; strides 1, 2, 3 and k"""
    out = []
    for k in range(1, 16):
        for p in range(0, k // 2 + 1):
            for s in sorted({1, 2, 3, k}):
                if (k, s, p) != (2, 2, 0):
                    out.append((k, s, p))
    return out


@pytest.mark.parametrize("cg", [(96, 1), (140, 2), (150, 3)], ids=["c96g1", "c140g2", "c150g3"])
def test_plane_pool_is_atens_max_pool_at_every_frozen_pool(cg):
    from micronet_b200 import _lib as L, b1 as B1
    from micronet_b200.fused import _pool_cfg
    C, G = cg
    g = torch.Generator().manual_seed(C)
    x = torch.randn(2, C, 15, 17, generator=g)
    x[0, :, 3, 4] = 0.0
    x[1, :, 7, 7] = -0.0
    x = x.to(DEV)
    pm1 = torch.where(x < 0, -1.0, 1.0)
    plane = B1.pack_act(x, G)
    pools = _freeze_pools()
    assert len(pools) > 200
    for k, s, p in pools:
        assert _pool_cfg(torch.nn.MaxPool2d(k, s, p)) == (k, s, p)
        rc, out, oshape = B1.plane_maxpool(plane, x.shape, G, k, s, p)
        L.check(rc, "b1 plane_maxpool")
        want = TF.max_pool2d(pm1, k, s, p)
        assert oshape == tuple(want.shape), (k, s, p)
        assert torch.equal(B1.unpack(out, oshape, G), want), (k, s, p)
        assert torch.equal(out, B1.pack_act(want.contiguous(), G)), (k, s, p)


# ---- model level: the README-cfg pruned NIN-GC
def _pruned_base():
    from tests.test_pk_pruned_cpu import README_CFG
    torch.manual_seed(1)
    base = zoo.init_like_reference(zoo.NINGC(README_CFG))
    g = torch.Generator().manual_seed(11)
    for mod in base.modules():          # trained-looking BatchNorm statistics (fresh ones are 0 / 1)
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
            mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
            mod.weight.data.copy_(torch.randn(mod.num_features, generator=g))
            mod.bias.data.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
    return base


def _pruned_engine(W):
    from harness import train as H
    return H.prepare_engine(_pruned_base(), "wbwtab", W=W, A=2, fuse_bn=True).to(DEV).eval()


@pytest.mark.parametrize("W", [3, 2])
def test_pruned_frozen_logits_are_bit_identical(W):
    from harness import train as H
    from micronet_b200 import _lib as L, functional as F_, wbwtab
    ref_m, fz = _pruned_engine(W), _pruned_engine(W)
    x, _ = H.synthetic_batch(256, 32, seed=5, device=DEV)
    with torch.no_grad():
        ref = ref_m(x)
        wbwtab.freeze_inference(fz)
        plan = [c.__dict__.get("_mnb_frozen_plan") for c in fz.modules() if isinstance(c, wbwtab.QuantConv2d)]
        assert plan == [("xnor", L.XNOR_BITS)] * 6 + [("xnor", L.XNOR_PM1_BF16)]
        F_.TIMER = F_.KernelTimer()
        try:
            got = fz(x)
            torch.cuda.synchronize()
            kinds = [r[0] for r in F_.TIMER.records]
        finally:
            F_.TIMER = None
        assert torch.equal(got, ref)
        # the CPU link plan: one epilogue launch per frozen conv, of the conv kinds only the head's forward besides
        assert kinds == [f"fwd_{k}_post" for k, _ in plan] + ["fwd_pk"], kinds
        # each hand-off, read back through functional.materialized (the bit plane at the consumer's groups of 76 - 81
        # channels), is the +-1 input the un-frozen consumer conv sees after BatchNorm, sign, pool and shuffle
        qr = [c for c in ref_m.modules() if isinstance(c, wbwtab.QuantConv2d)]
        qf = [c for c in fz.modules() if isinstance(c, wbwtab.QuantConv2d)]
        seen_in, seen_out = {}, {}
        hooks = [c.register_forward_pre_hook(lambda m, a, i=i: seen_in.__setitem__(i, F_.materialized(a[0]).clone()))
                 for i, c in enumerate(qr)]
        hooks += [c.register_forward_hook(lambda m, a, o, i=i: seen_out.__setitem__(i, F_.materialized(o).clone()))
                  for i, c in enumerate(qf)]
        try:
            ref_m(x)
            fz(x)
        finally:
            for hk in hooks:
                hk.remove()
        for i in range(len(qf) - 1):
            assert torch.equal(seen_out[i], seen_in[i + 1]), f"L{i + 1} -> L{i + 2}"
        st = H.InferStepper(fz, graph=True)
        for _ in range(4):
            out = st.step(x)
        assert st.graph is not None, st.graph_error
        assert torch.equal(out, ref)
        wbwtab.freeze_inference(fz, enable=False)
        assert torch.equal(fz(x), ref_m(x))      # W = 2: both centre their weights a second time


@pytest.mark.parametrize("W", [3, 2])
def test_pruned_eval_convs_against_the_oracle_teacher_forced(W):
    """each binarized conv of the un-frozen eval forward against the oracle port's conv of the same name, fed the +-1 input
    the engine's conv saw: within 1e-5 of the largest element, and a sign may differ only where the oracle's value is
    within fp32 rounding of 0"""
    from harness import train as H
    from micronet_b200 import functional as F_, wbwtab
    eng = _pruned_engine(W)
    ora = H.prepare_oracle(copy.deepcopy(_pruned_base()), "wbwtab", W=W, A=2).eval()
    seen, hooks = {}, []
    for name, m in eng.named_modules():
        if isinstance(m, wbwtab.QuantConv2d):
            hooks.append(m.register_forward_hook(lambda mod, inp, out, name=name: seen.__setitem__(
                name, (F_.materialized(inp[0]).detach().cpu(), F_.materialized(out).detach().cpu()))))
    x, _ = H.synthetic_batch(32, 32, seed=2, device=DEV)
    try:
        with torch.no_grad():
            eng(x)
            torch.cuda.synchronize()
    finally:
        for hk in hooks:
            hk.remove()
    assert len(seen) == 7, sorted(seen)
    ora_mods = dict(ora.named_modules())
    with torch.no_grad():
        for name, (inp, got) in seen.items():
            assert bool(((inp == 1) | (inp == -1)).all()), name
            c = ora_mods[name]
            want = c(inp)
            err = (got - want).abs().max() / want.abs().max()
            assert err < 1e-5, (name, err)
            flip = (got < 0) != (want < 0)
            taps = c.in_channels // c.groups * c.kernel_size[0] * c.kernel_size[1]
            tol = 2.0 ** -23 * (c.weight.abs().amax() * taps + c.bias.abs().amax())
            assert bool((want[flip].abs() <= tol).all()), name
