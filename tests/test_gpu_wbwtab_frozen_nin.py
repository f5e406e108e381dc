"""Frozen wbwtab inference on NIN (models/nin.py, for the harness NIN and a reference-structured NIN without
channel_shuffle_flag): every binarized layer runs the binary tensor-core convolution with its epilogue writing the next
layer's b1 plane (mnb_b1_conv_post), the 3 / 2 / 1 pools run on the planes, and the head reads a bf16 +-1 plane.  The frozen
logits equal the un-frozen eval forward's bit for bit (QAT graph and deployment graph), eagerly and under CUDA-graph replay."""
import pytest
import torch

from harness import train as H
from tests.test_wbwtab_frozen_nin_cpu import RefNIN

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _randomise_bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():          # trained-looking BatchNorm statistics (fresh ones are 0 / 1)
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.3)
            mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
            mod.weight.data.copy_(torch.randn(mod.num_features, generator=g))
            mod.bias.data.copy_(torch.randn(mod.num_features, generator=g) * 0.3)


def _model(name, graph, W, seed=0):
    import micronet_b200 as E
    if name == "ref_nin":
        torch.manual_seed(seed)
        base = RefNIN()
    else:
        base = H.build_float_model("nin", seed=seed)
    _randomise_bn(base, seed + 11)
    if graph == "G2":
        m = E.wbwtab.prepare(base, W=W, A=2, fuse_bn=True).to(DEV)
    else:
        m = E.wbwtab.prepare(base, W=W, A=2, quant_inference=True)
        m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=W).to(DEV)
        m = E.bn_fuse.wbwtab_quantize_inference_weights(m)
    return m.eval()


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _g1_composed(m, x):
    """per-layer composition of existing kernels with the frozen layers' (w_int, alpha, bias): packed-operand conv (fp32) ->
    sign -> ATen max-pool, stem and head as the un-frozen model runs them"""
    from micronet_b200 import _lib as L, pk as PK, wbwtab
    from micronet_b200 import functional as F_
    h = x
    for blk in m.model.children():
        if isinstance(blk, (torch.nn.MaxPool2d, torch.nn.AvgPool2d)):
            h = blk(h)
            continue
        c = blk.conv
        if isinstance(c, wbwtab.QuantConv2d):
            w_int, alpha = wbwtab.frozen_levels(c)
            sh = F_._shape_struct(h.shape, c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
            y = torch.empty((h.shape[0], c.out_channels, h.shape[2], h.shape[3]), device=DEV)
            planes = PK.pack_act(h.contiguous(), None, 1, groups=c.groups)[0]
            L.check(PK.conv(sh, 0, planes, 1, PK.pack_weight(sh, 0, 1, 1, w_int=w_int), 1, y, n_scale=alpha, bias=c.bias), "")
            h = torch.where(y < 0, -1.0, 1.0)
        elif c.in_channels >= 64:
            # the head on the packed-operand family, +-1 input as one bf16 piece (fused.EnginePmConv2d's route)
            h._mnb_pm1 = True
            h = torch.relu(F_.quant_conv2d(h, c.weight, c.bias, None, None, None, c.stride, c.padding, c.dilation, c.groups))
        else:
            h = blk(h)
    return h.view(h.shape[0], -1)


@pytest.mark.parametrize("graph", ["G2", "G1"])
@pytest.mark.parametrize("W", [3, 2])
@pytest.mark.parametrize("name", ["nin", "ref_nin"])
def test_frozen_nin_logits_are_bit_identical(name, W, graph):
    from micronet_b200 import functional as F_, wbwtab
    ref_m, fz = _model(name, graph, W), _model(name, graph, W)
    tree = [type(k) for k in fz.modules()]
    sd = {k: v.clone() for k, v in fz.state_dict().items()}
    x, _ = H.synthetic_batch(256, 32, seed=5, device=DEV)
    with torch.no_grad():
        # G2: the un-frozen eval forward; G1: the per-layer composition with the frozen layers' (w_int, alpha, bias)
        ref = ref_m(x) if graph == "G2" else _g1_composed(ref_m, x)
        wbwtab.freeze_inference(fz)
        F_.TIMER = F_.KernelTimer()
        try:
            got = fz(x)
            torch.cuda.synchronize()
            kinds = [r[0] for r in F_.TIMER.records]
        finally:
            F_.TIMER = None
        assert torch.equal(got, ref)
        # L1 - L7 each one binary tensor-core launch with the epilogue; of the conv kinds only the head's forward besides
        assert kinds.count("fwd_b1_post") == 7 and kinds.count("fwd_pk") == 1 and len(kinds) == 8, kinds
        st = H.InferStepper(fz, graph=True)
        for _ in range(4):
            out = st.step(x)
        assert st.graph is not None, st.graph_error
        assert torch.equal(out, ref)
        wbwtab.freeze_inference(fz, enable=False)
        assert [type(k) for k in fz.modules()] == tree and fz.state_dict().keys() == sd.keys()
        if W == 3:   # (W = 2 centres its weights in place on every forward, frozen or not)
            assert all(torch.equal(v, sd[k]) for k, v in fz.state_dict().items())
        assert torch.equal(fz(x), ref_m(x))


def test_weight_written_in_place_is_repacked():
    import micronet_b200 as E
    ref_m, fz = _model("nin", "G2", 3), _model("nin", "G2", 3)
    E.wbwtab.freeze_inference(fz)
    x, _ = H.synthetic_batch(64, 32, seed=6, device=DEV)
    qa = [c for c in ref_m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    qb = [c for c in fz.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    with torch.no_grad():
        fz(x)
        for c in (qa[2], qb[2]):
            c.weight.mul_(-1.0)
        assert torch.equal(fz(x), ref_m(x))


def test_nan_alpha_layer_stays_unfrozen():
    import micronet_b200 as E
    ref_m, fz = _model("nin", "G2", 3), _model("nin", "G2", 3)
    for m in (ref_m, fz):
        q = [c for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
        with torch.no_grad():
            q[3].weight[5].zero_()            # an all-zero ternary channel: alpha = 0 / 0
    E.wbwtab.freeze_inference(fz)
    plan = [c.__dict__.get("_mnb_frozen_plan") for c in fz.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    assert plan[3] is None and plan[2] is None and plan[4] is not None
    x, _ = H.synthetic_batch(64, 32, seed=7, device=DEV)
    with torch.no_grad():
        torch.testing.assert_close(fz(x), ref_m(x), rtol=0, atol=0, equal_nan=True)
