"""Frozen wbwtab inference with fp32 activations (prepare(A=32, W=2|3)) on term planes: the conv epilogue that writes its
consumer's three exact bf16 pieces (mnb_pk_conv_post with terms_out), the stem producer (mnb_bn_relu_pack_terms_fwd) and the
term-plane max-pool (mnb_pk_plane_maxpool_terms) bitwise against their decoded compositions, and the frozen NIN / NIN-GC
logits bitwise against a block-by-block composition of those kernels and within the fp32 contract of an fp64 evaluation."""
import pytest
import torch
import torch.nn.functional as F

from harness import train as H
from harness.wbwtab_a32_compose import blocks as _blocks, composed as _composed, parts as _parts
from tests.test_wbwtab_frozen_nin_cpu import RefNIN

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 3


@pytest.fixture(autouse=True)
def _tc_clean():
    cudnn = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False   # the stem / head convs run on ATen
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = cudnn
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _shuffle(x, g):
    b, c = x.shape[0], x.shape[1]
    return x.view(b, g, c // g, *x.shape[2:]).transpose(1, 2).contiguous().view(x.shape) if g > 1 else x


def _bn_stats(c, seed):
    g = torch.Generator().manual_seed(seed)
    mean, var = torch.randn(c, generator=g) * 0.3, torch.rand(c, generator=g) + 0.5
    gamma, beta = torch.randn(c, generator=g), torch.randn(c, generator=g) * 0.3
    return tuple(t.to(DEV) for t in (mean, torch.rsqrt(var + 1e-5), gamma, beta))


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
EPI_CASES = [
    # (B, C, H, K, R, pad, groups, shuffle groups, stride-2 consumer); plans at terms (3, 1) that are not segmented
    (4, 64, 16, 64, 1, 0, 1, 1, False),
    (4, 64, 16, 64, 1, 0, 1, 4, False),
    (4, 32, 16, 64, 3, 1, 1, 1, False),
    (2, 256, 8, 256, 1, 0, 2, 2, False),
    (2, 128, 8, 512, 1, 0, 4, 16, False),
    (2, 256, 16, 512, 3, 1, 16, 2, False),
    (4, 96, 16, 192, 1, 0, 1, 1, True),
    (3, 48, 10, 80, 1, 0, 1, 1, True),
]


@pytest.mark.parametrize("bn_on", [True, False])
@pytest.mark.parametrize("case", EPI_CASES)
def test_epilogue_term_planes_match_the_composition(case, bn_on):
    """fwd conv with the term-plane epilogue == fp32 conv -> stem producer (BatchNorm + ReLU + shuffle -> term planes), and
    for a stride-2 consumer == the phase-split pack of that producer's decoded tensor; the fp32 output written alongside is
    the plain conv's"""
    from micronet_b200 import _lib as L, pk as PK
    from micronet_b200 import functional as F_
    B, C, Hh, K, R, pad, G, sg, split = case
    torch.manual_seed(sum(case[:6]))
    x = torch.randn(B, C, Hh, Hh, device=DEV) * 2
    w_int = torch.randint(-1, 2, (K, C // G, R, R), device=DEV, dtype=torch.int16)
    alpha = torch.rand(K, device=DEV) + 0.1
    bias = torch.randn(K, device=DEV) * 0.5
    bn = _bn_stats(K, K + R) if bn_on else None
    sh = F_._shape_struct(x.shape, w_int.shape, (1, 1), (pad, pad), (1, 1), G)
    a_pk, _ = PK.pack_act(x, None, T, groups=G)
    w_img = PK.pack_weight(sh, 0, T, 1, w_int=w_int)
    y = torch.empty(B, K, Hh, Hh, device=DEV)
    L.check(PK.conv(sh, 0, a_pk, T, w_img, 1, y, n_scale=alpha, bias=bias), "pk_conv")
    ref = PK.terms_plane(B, K, Hh, Hh, T, DEV)
    L.check(PK.bn_relu_pack_terms(y, bn, True, sg, T, ref), "bn_relu_pack_terms")
    if split:
        ref, _ = PK.pack_act(PK.unpack_terms(ref, y.shape, T), None, T, phase_split=True)
    got = PK.terms_plane(B, K, Hh, Hh, T, DEV)
    y2 = torch.full_like(y, float("nan"))
    L.check(PK.conv_post_terms(sh, a_pk, w_img, y2, got, T, True, split, n_scale=alpha, bias=bias, bn=bn, shuffle_groups=sg),
            "pk_conv_post terms")
    torch.cuda.synchronize()
    assert torch.equal(got, ref)
    assert torch.equal(y2, y)
    # without BatchNorm the stem producer is exact: the plane decodes to shuffle(relu(y))
    if bn is None and not split:
        assert torch.equal(PK.unpack_terms(got, y.shape, T), _shuffle(torch.relu(y), sg))


def test_stem_producer_against_fp64():
    from micronet_b200 import _lib as L, pk as PK
    torch.manual_seed(3)
    x = torch.randn(8, 64, 32, 32, device=DEV) * 3
    mean, invstd, gamma, beta = _bn_stats(64, 9)
    plane = PK.terms_plane(*x.shape, T, DEV)
    L.check(PK.bn_relu_pack_terms(x, (mean, invstd, gamma, beta), True, 4, T, plane), "bn_relu_pack_terms")
    got = PK.unpack_terms(plane, x.shape, T).double()
    v = lambda t: t.double().view(1, -1, 1, 1)     # noqa: E731
    d, gs = x.double() - v(mean), v(gamma) * v(invstd)
    ref = _shuffle(torch.relu(d * gs + v(beta)), 4)
    # three fp32 roundings (x - mean, gamma * invstd, the fma), each within 2^-24 of the magnitude it rounds
    bound = _shuffle(2.0 ** -22 * ((d * gs).abs() + v(beta).abs()), 4)
    assert ((got - ref).abs() <= bound).all()


@pytest.mark.parametrize("kps", [(3, 2, 1), (2, 2, 0), (3, 1, 1)])
def test_term_pool_matches_aten_max_pool(kps):
    from micronet_b200 import _lib as L, pk as PK
    k, s, p = kps
    torch.manual_seed(k * 10 + s)
    x = torch.relu(torch.randn(4, 40, 17, 16, device=DEV))
    x[:, :, ::3, ::2] = 0.0                      # ties between zeros
    plane, _ = PK.pack_act(x, None, T)
    rc, got = PK.plane_maxpool_terms(plane, *x.shape, k, s, p, T)
    L.check(rc, "plane_maxpool_terms")
    ref, _ = PK.pack_act(F.max_pool2d(PK.unpack_terms(plane, x.shape, T), k, s, p), None, T)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


def test_kernel_refusals_launch_nothing():
    """MNB_E_ARG for a partial BatchNorm set, MNB_E_UNSUPPORTED for a segmented plan, a shuffle that does not divide C_out
    and a shuffle with phase_split: all before anything is launched"""
    from micronet_b200 import _lib as L, pk as PK
    from micronet_b200 import functional as F_
    x = torch.randn(2, 64, 8, 8, device=DEV)
    w_int = torch.randint(-1, 2, (48, 64, 3, 3), device=DEV, dtype=torch.int16)
    alpha = torch.ones(48, device=DEV)
    sh = F_._shape_struct(x.shape, w_int.shape, (1, 1), (1, 1), (1, 1), 1)
    a_pk, _ = PK.pack_act(x, None, T)
    w_img = PK.pack_weight(sh, 0, T, 1, w_int=w_int)
    plane = PK.terms_plane(2, 48, 8, 8, T, DEV)
    mean = torch.zeros(48, device=DEV)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    post = L.PkPost(None, 1, 0, plane.data_ptr())
    post.terms_out, post.bn_mean = T, mean.data_ptr()
    import ctypes as C
    lib = L.load()
    args = lambda: (C.byref(sh), a_pk.data_ptr(), T, w_img.data_ptr(), 1, alpha.data_ptr(), None, 1.0, None, None,  # noqa
                    C.byref(post), L.tc_err_flag(x.device).data_ptr(), L.stream())
    assert lib.mnb_pk_conv_post(*args()) == -1                                           # partial BatchNorm
    post.bn_mean = None
    post.shuffle_groups = 5
    assert lib.mnb_pk_conv_post(*args()) == L.E_UNSUPPORTED                              # 5 does not divide 48
    post.shuffle_groups, post.phase_split = 2, 1
    assert lib.mnb_pk_conv_post(*args()) == L.E_UNSUPPORTED                              # shuffle + phase split
    post.shuffle_groups, post.phase_split = 1, 0
    post.terms_out = 4
    assert lib.mnb_pk_conv_post(*args()) == -1                                           # terms_out 1..3
    post.terms_out = T
    seg = L.ConvShape(2, 64, 8, 8, 48, 3, 3, 1, 1, 1, 1, 1, 1, 1)   # this very conv: its plan at (3, 1) is segmented
    assert PK.segmented(seg, 0, T, 1)
    assert PK.conv_post_terms(sh, a_pk, w_img, None, plane, T, True) == L.E_UNSUPPORTED          # segmented plan
    # C_out = 12, ungrouped: the epilogue stores whole 8-channel units, so a partial last unit is refused
    w12 = torch.randint(-1, 2, (12, 64, 1, 1), device=DEV, dtype=torch.int16)
    sh12 = F_._shape_struct(x.shape, w12.shape, (1, 1), (0, 0), (1, 1), 1)
    assert PK.supported(sh12, 0, T, 1) and not PK.segmented(sh12, 0, T, 1)
    img12 = PK.pack_weight(sh12, 0, T, 1, w_int=w12)
    plane12 = PK.terms_plane(2, 12, 8, 8, T, DEV)
    y12 = torch.empty(2, 12, 8, 8, device=DEV)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    assert PK.conv_post_terms(sh12, a_pk, img12, y12, plane12, T, True, n_scale=alpha[:12]) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def test_pool_fallback_keeps_the_channel_order():
    """a term-plane pool the kernel refuses runs the module on the decoded tensor in the producer's channel order (the plane
    holds the consumer's shuffled order; the consumer applies its block's shuffle itself when no plane arrives)"""
    from micronet_b200 import _lib as L, pk as PK, wbwtab
    torch.manual_seed(4)
    y = torch.randn(2, 32, 8, 8, device=DEV)
    plane = PK.terms_plane(*y.shape, T, DEV)
    L.check(PK.bn_relu_pack_terms(y, None, True, 4, T, plane), "bn_relu_pack_terms")
    pool = torch.nn.MaxPool2d(2, 2).eval()
    # (k, s, p) = (3, 2, 2) as the plane pool's geometry: 2 p > k, which mnb_pk_plane_maxpool_terms refuses
    link = wbwtab._TermLink(torch.nn.Conv2d(32, 32, 1), None, 4, (pool, 3, 2, 2))
    out = wbwtab._a32_pool_forward(pool, link, link.tag(plane, y.shape))
    assert getattr(out, "_mnb_terms", None) is None
    assert torch.equal(out, F.max_pool2d(torch.relu(y), 2, 2))


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _randomise_bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
            mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
            mod.weight.data.copy_(torch.randn(mod.num_features, generator=g))
            mod.bias.data.copy_(torch.randn(mod.num_features, generator=g) * 0.3)


def _model(name, W, seed=0):
    import micronet_b200 as E
    if name == "ref_nin":
        torch.manual_seed(seed)
        base = RefNIN()
    else:
        base = H.build_float_model(name, seed=seed)
    _randomise_bn(base, seed + 11)
    return E.wbwtab.prepare(base, W=W, A=32).to(DEV).eval()


def _fp64(m, x):
    """the graph in fp64 on the CPU: weight levels x alpha, running-statistics BatchNorm"""
    from micronet_b200 import wbwtab
    h = x.double().cpu()
    for blk in _blocks(m):
        if not hasattr(blk, "conv"):
            h = blk(h)           # the pools
            continue
        if getattr(blk, "channel_shuffle_flag", 0):
            h = _shuffle(h, int(blk.shuffle_groups))
        c, bn = _parts(blk)[0], _parts(blk)[1]
        if type(c) is wbwtab.QuantConv2d:
            w_int, alpha = wbwtab.frozen_levels(c)
            w = w_int.double().cpu() * alpha.double().cpu().view(-1, 1, 1, 1)
        else:
            w = c.weight.detach().double().cpu()
        b = None if c.bias is None else c.bias.detach().double().cpu()
        h = F.conv2d(h, w, b, c.stride, c.padding, c.dilation, c.groups)
        h = F.batch_norm(h, bn.running_mean.double().cpu(), bn.running_var.double().cpu(), bn.weight.detach().double().cpu(),
                         bn.bias.detach().double().cpu(), False, 0.0, bn.eps)
        h = torch.relu(h)
    return h.view(h.shape[0], -1)


WORST = {}


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("name", ["nin", "nin_gc", "ref_nin", "nin_b256", "nin_gc_b256"])
def test_frozen_logits_equal_the_composition(name, W):
    from micronet_b200 import functional as F_, wbwtab
    name, _, batch = name.partition("_b")     # "_b256": the batch the benchmark runs the NIN models at
    batch = int(batch) if batch else 32
    ref_m, fz = _model(name, W), _model(name, W)
    x, _ = H.synthetic_batch(batch, 32, seed=5, device=DEV)
    with torch.no_grad():
        ref, reads = _composed(ref_m, x)
        unfrozen = ref_m(x)
        wbwtab.freeze_inference(fz)
        seen = []
        qconvs = [k for k in fz.modules() if type(k) is wbwtab.QuantConv2d]
        hooks = [c.register_forward_pre_hook(lambda mod, inp: seen.append(F_.materialized(inp[0]))) for c in qconvs]
        got = fz(x)
        for hk in hooks:
            hk.remove()
        torch.cuda.synchronize()
        assert torch.equal(got, ref)
        # every plane a quantized layer reads decodes to the composition's tensor (L1 .. L7; shuffles applied by producers)
        assert len(seen) == len(reads) == 7
        for i, (a, b) in enumerate(zip(seen, reads)):
            assert torch.equal(a, b), f"L{i + 1}"
        ref64 = _fp64(ref_m, x)
        scale = ref64.abs().max().item()
        err_f = (got.double().cpu() - ref64).abs().max().item() / scale
        err_u = (unfrozen.double().cpu() - ref64).abs().max().item() / scale
        WORST[(name, W, batch)] = (err_f, err_u)
        print(f"\n{name} W{W}: max |logit - fp64| / max |fp64|: frozen {err_f:.3e}, un-frozen {err_u:.3e}")
        assert err_f <= 1e-5 and err_u <= 1e-5


@pytest.mark.parametrize("name", ["nin", "nin_gc"])
def test_launch_kinds(name, monkeypatch):
    """between the stem and the head: no ATen BatchNorm, ReLU or pool and no pack_act - one conv launch per quantized layer,
    the plane pools and the stem producer"""
    from micronet_b200 import functional as F_, pk as PK, wbwtab
    fz = _model(name, 3)
    wbwtab.freeze_inference(fz)
    x, _ = H.synthetic_batch(16, 32, seed=7, device=DEV)
    calls = {"bn": 0, "relu": 0, "pool": 0, "pack_act": 0, "stem": 0}

    def spy(key, fn):
        def run(*a, **k):
            calls[key] += 1
            return fn(*a, **k)
        return run
    monkeypatch.setattr(F, "batch_norm", spy("bn", F.batch_norm))
    monkeypatch.setattr(F, "relu", spy("relu", F.relu))
    monkeypatch.setattr(F, "max_pool2d", spy("pool", F.max_pool2d))
    monkeypatch.setattr(PK, "pack_act", spy("pack_act", PK.pack_act))
    monkeypatch.setattr(PK, "bn_relu_pack_terms", spy("stem", PK.bn_relu_pack_terms))
    with torch.no_grad():
        fz(x)
        F_.TIMER = F_.KernelTimer()
        for k in calls:
            calls[k] = 0
        try:
            fz(x)
            torch.cuda.synchronize()
            kinds = [r[0] for r in F_.TIMER.records]
        finally:
            F_.TIMER = None
    # producers without a consumer epilogue - NIN's L3 and L6 (segmented plans) and every NIN-GC link (shuffled) - write fp32,
    # then the stem producer writes the plane
    sep = 2 if name == "nin" else 6
    # ATen: L7's BatchNorm + ReLU (its consumer is the un-quantized head) and the head block's own
    assert calls == {"bn": 2, "relu": 2, "pool": 0, "pack_act": 0, "stem": 1 + sep}, calls
    assert kinds.count("fwd_pk_terms") == 6 - sep and kinds.count("fwd_pk") == 1 + sep, kinds
    assert kinds.count("plane_pool") == 2 and len(kinds) == 9, kinds


@pytest.mark.parametrize("name", ["nin", "nin_gc"])
def test_cuda_graph_replay_equals_eager(name):
    from micronet_b200 import wbwtab
    fz = _model(name, 2)
    wbwtab.freeze_inference(fz)
    x, _ = H.synthetic_batch(64, 32, seed=8, device=DEV)
    with torch.no_grad():
        eager = fz(x)
        st = H.InferStepper(fz, graph=True)
        for _ in range(4):
            out = st.step(x)
        assert st.graph is not None, st.graph_error
        assert torch.equal(out, eager)


def test_weight_write_repacks_and_restore():
    import micronet_b200 as E
    ref_m, fz = _model("nin_gc", 3), _model("nin_gc", 3)
    tree = [type(k) for k in fz.modules()]
    x, _ = H.synthetic_batch(32, 32, seed=6, device=DEV)
    with torch.no_grad():
        unfrozen = fz(x)
        E.wbwtab.freeze_inference(fz)
        fz(x)
        qa = [c for c in ref_m.modules() if type(c) is E.wbwtab.QuantConv2d]
        qb = [c for c in fz.modules() if type(c) is E.wbwtab.QuantConv2d]
        for c in (qa[2], qb[2]):
            c.weight.mul_(-1.0)
        assert torch.equal(fz(x), _composed(ref_m, x)[0])
        for c in (qa[2], qb[2]):
            c.weight.mul_(-1.0)
        E.wbwtab.freeze_inference(fz, enable=False)
        assert [type(k) for k in fz.modules()] == tree
        assert torch.equal(fz(x), unfrozen)
