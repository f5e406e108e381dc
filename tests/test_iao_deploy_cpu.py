"""CPU side of frozen IAO deployment graphs (bn_fuse.iao_model_bn_fuse -> bn_fuse.iao_quantize_inference_weights ->
iao.freeze_inference): the weight step against the reference's own flow (tests/golden/make_golden_iao_deploy.py), which
stored weights freeze_inference accepts as integer levels and which it refuses, that the link plan of the deployment
graphs of NIN, NIN-GC (default and pruned cfg) and ResNet-18 is the plan of the QAT graphs they came from, and that
``enable=False`` restores the module tree and the state_dict.  Host logic only - runs without a GPU."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from harness import models as zoo
from tests.oracle_util import load_golden
from tests.test_bn_fuse_cpu import converted_iao

NIN_CFG = [64, 32, 32, 64, 64, 64, 64, 64]
GC_CFG = [32, 32, 32, 64, 64, 64, 128, 128]
PRUNED_CFG = [154, 162, 144, 304, 320, 320, 608, 584]      # DESIGN.md 4.17


def _deploy(qat):
    from micronet_b200 import bn_fuse
    return bn_fuse.iao_quantize_inference_weights(bn_fuse.iao_model_bn_fuse(qat)).eval()


@pytest.mark.parametrize("q_level", [0, 1], ids=["per_channel", "per_layer"])
def test_weight_step_matches_the_reference_flow(q_level):
    gold = load_golden("iao_deploy", f"t0_l{q_level}")
    from micronet_b200 import bn_fuse
    inf = bn_fuse.iao_quantize_inference_weights(converted_iao(gold, 0, q_level).eval())
    want = {k[7:]: v for k, v in gold.items() if k.startswith("deploy.")}
    got = inf.state_dict()
    assert set(got) == set(want)
    for k, v in want.items():
        assert np.array_equal(got[k].numpy(), v), k
    # the step changed the weights, and every quant_inference conv is then accepted as levels
    raw = converted_iao(gold, 0, q_level).state_dict()
    assert any(not torch.equal(raw[k], got[k]) for k in got if k.endswith(".weight"))
    _freeze(inf)
    convs = _inference_convs(inf)
    assert len(convs) == 9 and all("_int_levels" in c.__dict__ for c in convs.values())


def _inference_convs(m):
    from micronet_b200 import iao
    return {n: c for n, c in m.named_modules() if isinstance(c, iao.QuantConv2d) and c.quant_inference}


def _freeze(m, **kw):
    from micronet_b200 import iao
    return iao.freeze_inference(m, **kw)


def _stepped(q_level=0):
    from micronet_b200 import bn_fuse
    gold = load_golden("iao_deploy", f"t0_l{q_level}")
    return bn_fuse.iao_quantize_inference_weights(converted_iao(gold, 0, q_level).eval())


def _accepted(m):
    return {n for n, c in _inference_convs(m).items() if "_int_levels" in c.__dict__}


def test_raw_folded_weights_are_refused():
    gold = load_golden("iao_deploy", "t0_l0")
    m = converted_iao(gold, 0, 0).eval()
    _freeze(m, int8=True)
    assert _accepted(m) == set()
    assert not any(k in c.__dict__ for c in m.modules() for k in ("_pre_relu", "forward", "_mnb_in_shuffle", "_post_consumer"))


# one element of a stepped layer replaced: (stored value, that element's scale, weight quantizer) -> new value
EDITS = {
    "one_ulp": lambda v, s, q: torch.nextafter(v, torch.tensor(float("inf"))),
    "out_of_range": lambda v, s, q: (q.qmax + 1) * s,      # fl(L * s) with L = qmax + 1: the clamp changes it
    "nan": lambda v, s, q: torch.tensor(float("nan")),
    "inf": lambda v, s, q: torch.tensor(float("inf")),
}


@pytest.mark.parametrize("q_level", [0, 1], ids=["per_channel", "per_layer"])
@pytest.mark.parametrize("edit", list(EDITS))
def test_edited_weights_are_refused(edit, q_level):
    """one element of one stepped layer changed: that layer keeps its fp32 weight, the producer in front of it gets no
    consumer for it, and every other layer is still accepted"""
    from micronet_b200 import iao
    m = _stepped(q_level)
    mods = dict(m.named_modules())
    victim = mods["model.4.conv"]
    q = victim.weight_quantizer
    with torch.no_grad():
        w = victim.weight.view(-1)
        i = int(w.abs().argmax())
        s = q.scale.view(-1)[i // victim.weight[0].numel() if q.scale.numel() > 1 else 0]
        w[i] = EDITS[edit](w[i], s, q)
    _freeze(m, int8=True)
    assert _accepted(m) == set(_inference_convs(m)) - {"model.4.conv"}
    assert not iao._int_weights(victim) and not iao._int8_ok(victim)
    with torch.no_grad():
        assert iao._consumer_of(mods["model.2.conv"]) is None
    # the same layer with its stepped weight back is accepted again
    victim.weight.data = _stepped(q_level).model[4].conv.weight.data
    _freeze(m, int8=True)
    assert _accepted(m) == set(_inference_convs(m))
    with torch.no_grad():
        assert iao._consumer_of(mods["model.2.conv"]) is not None


def test_asymmetric_and_training_mode_are_refused():
    from micronet_b200 import bn_fuse
    gold = load_golden("bnfuse", "iao_t1_l1")
    m = bn_fuse.iao_quantize_inference_weights(converted_iao(gold, 1, 1).eval())
    _freeze(m, int8=True)
    assert _accepted(m) == set()
    m = _stepped(0).train()
    _freeze(m)
    assert _accepted(m) == set()


def _qat(kind, ptq=False, q_level=0):
    """an eval-mode ``prepare(bn_fuse=True)`` model with randomised BatchNorm statistics and weight scales taken from the
    folded weights (no calibration pass: the engine's observers run on the GPU only)"""
    from micronet_b200 import iao
    torch.manual_seed(0)
    if kind == "resnet":
        base = zoo.resnet18()
    else:
        cfg = {"nin": NIN_CFG, "gc": GC_CFG, "pruned": PRUNED_CFG}[kind]
        base = zoo.init_like_reference(zoo.NIN(cfg) if kind == "nin" else zoo.NINGC(cfg))
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for bn in base.modules():
            if isinstance(bn, nn.BatchNorm2d):
                bn.running_mean.copy_(torch.randn(bn.num_features, generator=g) * 0.3)
                bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
                bn.weight.copy_(torch.rand(bn.num_features, generator=g) + 0.3)
    m = iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=q_level, bn_fuse=True, ptq=ptq).eval()
    with torch.no_grad():
        for c in m.modules():
            if isinstance(c, iao.QuantBNFuseConv2d):
                w = c._fold_running()[0]
                s = (w.abs().amax(dim=(1, 2, 3), keepdim=True) if q_level == 0 else w.abs().max().reshape(1)) / 127
                c.weight_quantizer.scale.copy_(s.clamp_min(1e-8))
    return m


def _plan(m):
    """everything freeze_inference decided, by module name"""
    from micronet_b200 import iao
    names = {id(mod): n for n, mod in m.named_modules()}
    out = {}
    with torch.no_grad():
        for n, mod in m.named_modules():
            d = mod.__dict__
            link = d.get("_post_consumer")
            if isinstance(link, iao._BlockLink):
                link = ("block", names[id(link.cconv)], None if link.pool is None else (names[id(link.pool[0])],) + link.pool[1:],
                        link.sg)
            elif link is not None:
                link = (names[id(link[0])], link[1])
            consumer = iao._consumer_of(mod) if isinstance(mod, (iao.QuantConv2d, iao.QuantAdd)) else None
            out[n] = (link, d.get("_pre_relu", False), d.get("_fuse_relu", False), d.get("_mnb_in_shuffle", 1),
                      "forward" in d, getattr(mod, "channel_shuffle_flag", None),
                      iao._int8_ok(mod) if isinstance(mod, iao.QuantConv2d) else None,
                      None if consumer is None else (consumer.relu, consumer.only, consumer.int8, consumer.sg,
                                                     consumer.formats))
    return out


@pytest.mark.parametrize("kind", ["nin", "gc", "pruned", "resnet"])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
@pytest.mark.parametrize("q_level,ptq", [(0, False), (1, False), (0, True)], ids=["per_channel", "per_layer", "ptq"])
def test_deployment_plan_is_the_qat_plan(kind, i8, q_level, ptq):
    qat = _qat(kind, ptq, q_level)
    dep = _deploy(qat)
    _freeze(qat, int8=i8)
    _freeze(dep, int8=i8)
    want = _plan(qat)
    assert any(row[0] is not None for row in want.values())      # the QAT graph links something
    assert _plan(dep) == want
    assert _accepted(dep) == set(_inference_convs(dep))


def test_enable_false_restores_the_deployment_graph():
    m = _deploy(_qat("gc"))
    before = repr(m), {k: v.clone() for k, v in m.state_dict().items()}, [getattr(k, "channel_shuffle_flag", None)
                                                                          for k in m.modules()]
    _freeze(m, int8=True)
    assert _accepted(m) and any("forward" in c.__dict__ for c in m.modules())
    _freeze(m, enable=False)
    assert repr(m) == before[0]
    assert [getattr(k, "channel_shuffle_flag", None) for k in m.modules()] == before[2]
    sd = m.state_dict()
    assert sd.keys() == before[1].keys() and all(torch.equal(v, before[1][k]) for k, v in sd.items())
    assert not any(k in c.__dict__ for c in m.modules()
                   for k in ("forward", "_post_consumer", "_mnb_in_shuffle", "_int_levels", "_pre_relu"))
