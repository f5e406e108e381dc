"""Frozen wbwtab inference graphs on bit planes (wbwtab.freeze_inference): the sign-bit epilogue of the XNOR convolution
(mnb_xnor_conv_post) and the stem producer (mnb_xnor_pack_act_post) word for word against the un-fused sequence, the
frozen headline QAT graph bit-identical to its un-frozen eval forward (eagerly and under CUDA-graph replay), and the
reference's deployment graph against a per-layer composition of existing kernels and against the oracle."""
import pytest
import torch

from harness import models as zoo
from tests.test_gpu_xnor import IDS, SHAPES, _sh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _bn(K, g):
    mean = torch.randn(K, generator=g) * 3
    var = torch.rand(K, generator=g) * 4 + 0.1
    gamma = torch.randn(K, generator=g)
    gamma[0] = -gamma[0].abs()
    beta = torch.randn(K, generator=g)
    return [t.to(DEV) for t in (mean, torch.rsqrt(var.to(DEV) + 1e-5).cpu(), gamma, beta)]


def _bn_sign(y, bn):
    """+-1 of the eval BatchNorm + binarizer producer (mnb_bn_sign_fwd), or the plain sign without a BatchNorm"""
    from micronet_b200 import _lib as L
    if bn is None:
        return torch.where(y < 0, -1.0, 1.0)
    mean, invstd, gamma, beta = bn
    b, c = y.shape[0], y.shape[1]
    out = torch.empty_like(y)
    pass_bits = torch.empty((y.numel() + 31) // 32, dtype=torch.int32, device=DEV)
    L.check(L.load().mnb_bn_sign_fwd(y.data_ptr(), b, c, y.numel() // (b * c), mean.data_ptr(), invstd.data_ptr(),
                                     gamma.data_ptr(), beta.data_ptr(), 1, out.data_ptr(), pass_bits.data_ptr(), L.stream()),
            "bn_sign_fwd")
    return out


def _reference_bits(y, bn, pool, sg, G):
    """the un-fused sequence: eval BatchNorm in the producers' op order -> sign -> max-pool -> shuffle -> mnb_xnor_pack_act"""
    from micronet_b200 import xnor as X
    s = _bn_sign(y, bn)
    if pool:
        s = torch.nn.functional.max_pool2d(s, 2, 2)
    if sg > 1:
        s = zoo.shuffle_channels(s, sg)
    return X.pack_act(s.contiguous(), G)


@pytest.mark.parametrize("combo", ["plain", "bn", "bn_pool", "bn_shuffle", "bn_pool_shuffle", "pool_shuffle"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_bit_epilogue_matches_the_unfused_sequence(shape, combo):
    from micronet_b200 import _lib as L, xnor as X
    B, Cc, H, W, K, R, st, pad, G = shape
    g = torch.Generator().manual_seed(sum(shape) + len(combo))
    x = torch.randn(B, Cc, H, W, generator=g).to(DEV)
    w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g).to(torch.int16).to(DEV)
    alpha = (torch.rand(K, generator=g) * 0.05 + 0.01).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    sh = _sh(shape)
    bits, img = X.pack_act(x, G), X.pack_weight(sh, w)
    y = torch.empty((B, K, (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1), device=DEV)
    L.check(X.conv(sh, bits, img, y, alpha=alpha, bias=bias), "xnor conv")
    bn = _bn(K, g) if "bn" in combo else None
    pool = "pool" in combo
    sg = next(s for s in (4, 2, 1) if K % s == 0) if "shuffle" in combo else 1
    og = next(q for q in (8, 2, 1) if K % q == 0)           # consumer groups
    post = X.post_struct(L.XNOR_BITS, og, sg, pool, bn)
    n = X.post_bytes(sh, post)
    if pool and (y.shape[2] % 2 or y.shape[3] % 2):
        assert n == -1
        return
    out = torch.full((n // 4,), -1, dtype=torch.int32, device=DEV)     # garbage: the kernel zeroes it first
    L.check(X.conv_post(sh, bits, img, post, out, alpha=alpha, bias=bias), "xnor conv_post")
    assert torch.equal(out, _reference_bits(y, bn, pool, sg, og))
    # the stem producer on the fp32 output: same bits
    out2 = torch.full_like(out, -1)
    L.check(X.pack_act_post(y, post, out2), "xnor pack_act_post")
    assert torch.equal(out2, out)


@pytest.mark.parametrize("shape", [s for s in SHAPES if s[4] % 8 == 0], ids=[i for s, i in zip(SHAPES, IDS) if s[4] % 8 == 0])
def test_bf16_epilogue_matches_the_packed_producer(shape):
    from micronet_b200 import _lib as L, xnor as X
    B, Cc, H, W, K, R, st, pad, G = shape
    g = torch.Generator().manual_seed(sum(shape) + 7)
    x = torch.randn(B, Cc, H, W, generator=g).to(DEV)
    w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g).to(torch.int16).to(DEV)
    alpha = (torch.rand(K, generator=g) * 0.05 + 0.01).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    sh = _sh(shape)
    bits, img = X.pack_act(x, G), X.pack_weight(sh, w)
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    y = torch.empty((B, K, P, Q), device=DEV)
    L.check(X.conv(sh, bits, img, y, alpha=alpha, bias=bias), "xnor conv")
    bn = _bn(K, g)
    post = X.post_struct(L.XNOR_PM1_BF16, 1, 1, False, bn)
    out = torch.zeros(X.post_bytes(sh, post), dtype=torch.uint8, device=DEV)
    L.check(X.conv_post(sh, bits, img, post, out, alpha=alpha, bias=bias), "xnor conv_post bf16")
    if (P * Q) % 32 == 0:
        ref = torch.zeros_like(out)
        pass_bits = torch.empty((y.numel() + 31) // 32, dtype=torch.int32, device=DEV)
        mean, invstd, gamma, beta = bn
        L.check(L.load().mnb_bn_sign_fwd_packed(y.data_ptr(), B, K, P * Q, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                                beta.data_ptr(), 1, None, pass_bits.data_ptr(), ref.data_ptr(), L.stream()),
                "bn_sign_fwd_packed")
        assert torch.equal(out, ref)
    s = _bn_sign(y, bn)
    got = out.view(torch.bfloat16).view(B, K // 8, P, Q, 8).permute(0, 1, 4, 2, 3).reshape(B, K, P, Q).float()
    assert torch.equal(got, s)


def _g2(W, seed=0):
    from harness import train as H
    base = H.build_float_model("nin_gc", seed=seed)
    m = H.prepare_engine(base, "wbwtab", W=W, A=2, fuse_bn=True).to(DEV)
    g = torch.Generator().manual_seed(seed + 11)
    for mod in m.modules():          # trained-looking BatchNorm statistics (fresh ones are 0 / 1)
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
            mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
            mod.weight.data.copy_(torch.randn(mod.num_features, generator=g))
            mod.bias.data.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
    return m.eval()


@pytest.mark.parametrize("W", [3, 2])
def test_g2_frozen_logits_are_bit_identical(W):
    from harness import train as H
    from micronet_b200 import functional as F_, wbwtab
    ref_m, fz = _g2(W), _g2(W)
    x, _ = H.synthetic_batch(256, 32, seed=5, device=DEV)
    with torch.no_grad():
        ref = ref_m(x)
        wbwtab.freeze_inference(fz)
        F_.TIMER = F_.KernelTimer()
        try:
            got = fz(x)
            torch.cuda.synchronize()
            kinds = [r[0] for r in F_.TIMER.records]
        finally:
            F_.TIMER = None
        assert torch.equal(got, ref)
        # L1 - L7 each one XNOR launch with the epilogue, nothing else of the conv kinds but the head's forward
        assert kinds.count("fwd_xnor_post") == 7 and kinds.count("fwd_pk") == 1 and len(kinds) == 8, kinds
        again = fz(x)
        assert torch.equal(again, ref)
        st = H.InferStepper(fz, graph=True)
        for _ in range(4):
            out = st.step(x)
        assert st.graph is not None, st.graph_error
        assert torch.equal(out, ref)
        wbwtab.freeze_inference(fz, enable=False)
        assert torch.equal(fz(x), ref_m(x))      # W = 2: both centre their weights a second time


def test_g2_frozen_forward_writes_no_fp32_between_stem_and_head():
    """allocator bytes of one frozen forward at batch 256: the stem's fp32 output, the bit planes, the head's bf16 plane and
    logits - an fp32 layer output of L1 - L7 (>= 8 MB) would exceed the bound"""
    from harness import train as H
    from micronet_b200 import wbwtab
    m = wbwtab.freeze_inference(_g2(3))
    x, _ = H.synthetic_batch(256, 32, seed=5, device=DEV)
    with torch.no_grad():
        m(x)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m(x)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    B = 256
    stem = B * 256 * 32 * 32 * 4                          # EngineFloatConv2d output, fp32
    bits = B * 256 * 32 * 32 // 8 * 2                     # the largest bit planes (two alive at a time), generously
    head_in = 2 * B * 1024 * 8 * 8 * 2                    # bf16 plane + its placeholder's fp32 storage
    assert peak <= stem + bits + head_in + (4 << 20), (peak, stem)


def _g1(W, seed=0):
    """prepare(quant_inference=True) -> wbwtab_model_bn_fuse -> wbwtab_quantize_inference_weights, with randomised BN"""
    import micronet_b200 as E
    from harness import train as H
    base = H.build_float_model("nin_gc", seed=seed)
    g = torch.Generator().manual_seed(seed + 3)
    for mod in base.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
            mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
            mod.weight.data.copy_(torch.randn(mod.num_features, generator=g))
            mod.bias.data.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
    m = E.wbwtab.prepare(base, W=W, A=2, quant_inference=True)
    m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=W).to(DEV)
    return E.bn_fuse.wbwtab_quantize_inference_weights(m).eval()


def _g1_composed(m, x):
    """per-layer composition of existing kernels with the frozen layers' (w_int, alpha, bias): XNOR conv (fp32) -> sign ->
    max-pool -> shuffle, stem and head as the un-frozen model runs them"""
    from micronet_b200 import _lib as L, wbwtab, xnor as X
    from micronet_b200 import functional as F_
    seq = m.model
    h = x
    for blk in seq.children():
        if isinstance(blk, torch.nn.MaxPool2d):
            h = torch.nn.functional.max_pool2d(h, 2, 2)
            continue
        if isinstance(blk, torch.nn.AvgPool2d):
            h = blk(h)
            continue
        if blk.channel_shuffle_flag:
            h = zoo.shuffle_channels(h, blk.shuffle_groups)
        if isinstance(blk.conv, wbwtab.QuantConv2d):
            c = blk.conv
            w_int, alpha = wbwtab.frozen_levels(c)
            sh = F_._shape_struct(h.shape, c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
            y = torch.empty((h.shape[0], c.out_channels, h.shape[2], h.shape[3]), device=DEV)
            L.check(X.conv(sh, X.pack_act(h.contiguous(), c.groups), X.pack_weight(sh, w_int), y, alpha=alpha, bias=c.bias), "")
            h = torch.where(y < 0, -1.0, 1.0)
        elif blk.conv.in_channels >= 64:
            # the head on the packed-operand family, +-1 input as one bf16 piece (fused.EnginePmConv2d's route)
            c = blk.conv
            h._mnb_pm1 = True
            h = torch.relu(F_.quant_conv2d(h, c.weight, c.bias, None, None, None, c.stride, c.padding, c.dilation, c.groups))
        else:
            h = blk(h)
    return h.view(h.shape[0], -1)


@pytest.mark.parametrize("W", [3, 2])
def test_g1_frozen_matches_the_composed_kernels(W):
    from harness import train as H
    from micronet_b200 import wbwtab
    m = _g1(W)
    x, _ = H.synthetic_batch(256, 32, seed=9, device=DEV)
    with torch.no_grad():
        ref = _g1_composed(m, x)
        wbwtab.freeze_inference(m)
        got = m(x)
        assert torch.equal(got, ref)
        wbwtab.freeze_inference(m, enable=False)


def test_g1_frozen_against_the_oracle_teacher_forced():
    """each frozen layer's pre-sign value against the oracle port's fp32 convolution of the same +-1 input with the
    pre-quantized weights (bn_fused_model_test.py:191-194): within 1e-5 relative, and a sign may differ only where the oracle
    value is within fp32 rounding of 0 (SURVEY 7.2.1)"""
    from harness import train as H
    from micronet_b200 import _lib as L, wbwtab, xnor as X
    from micronet_b200 import functional as F_
    m = _g1(3)
    x, _ = H.synthetic_batch(32, 32, seed=2, device=DEV)
    h = x
    with torch.no_grad():
        for blk in m.model.children():
            if isinstance(blk, (torch.nn.MaxPool2d, torch.nn.AvgPool2d)):
                h = blk(h)
                continue
            if blk.channel_shuffle_flag:
                h = zoo.shuffle_channels(h, blk.shuffle_groups)
            if not isinstance(blk.conv, wbwtab.QuantConv2d):
                h = blk(h)
                continue
            c = blk.conv
            w_int, alpha = wbwtab.frozen_levels(c)
            sh = F_._shape_struct(h.shape, c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
            y = torch.empty((h.shape[0], c.out_channels, h.shape[2], h.shape[3]), device=DEV)
            L.check(X.conv(sh, X.pack_act(h.contiguous(), c.groups), X.pack_weight(sh, w_int), y, alpha=alpha, bias=c.bias), "")
            ora = torch.nn.functional.conv2d(h.cpu(), c.weight.cpu(), c.bias.cpu(), c.stride, c.padding, c.dilation, c.groups)
            err = (y.cpu() - ora).abs().max() / ora.abs().max()
            assert err < 1e-5, err
            flip = (y.cpu() < 0) != (ora < 0)
            tol = 2.0 ** -23 * (c.weight.abs().amax().cpu() * c.in_channels // c.groups * 9 + c.bias.abs().amax().cpu())
            assert bool((ora[flip].abs() <= tol).all())
            h = torch.where(ora.to(DEV) < 0, -1.0, 1.0)                 # teacher-forced: the oracle's signs go on
