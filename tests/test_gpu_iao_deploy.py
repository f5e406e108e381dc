"""Frozen IAO deployment graphs on the GPU (bn_fuse.iao_model_bn_fuse -> bn_fuse.iao_quantize_inference_weights ->
iao.freeze_inference): the weight step against the engine's weight quantizer, the logits bitwise against the frozen QAT graph
the deployment graph came from (NIN, NIN-GC, pruned NIN-GC, ResNet-18; per-channel and per-layer weights; QAT and PTQ
calibration; bf16 and int8 planes; eager and CUDA-graph replay) with the same conv launches, the reference's own deployment
output, raw converter output unchanged, and the refusal of a weight rewritten after freezing."""
import collections
import copy

import pytest
import torch

from harness import train as H
from harness.wbwtab_infer_probe import _randomise_bn
from tests.oracle_util import load_golden, rel_err
from tests.test_bn_fuse_cpu import converted_iao

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRUNED_CFG = [154, 162, 144, 304, 320, 320, 608, 584]      # DESIGN.md 4.17


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _calibrated(arch, q_level, ptq, hw=32, batch=32):
    import micronet_b200 as E
    from harness import models as zoo
    if arch == "nin_gc_pruned":
        torch.manual_seed(1)
        base = zoo.init_like_reference(zoo.NINGC(PRUNED_CFG))
    else:
        base = H.build_float_model(arch, seed=1)
    with torch.no_grad():
        _randomise_bn(base, 7)
    m = E.iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=q_level, bn_fuse=True, ptq=ptq).to(DEV)
    m.train()
    with torch.no_grad():
        for i in range(2):
            m(H.synthetic_batch(batch, hw, seed=20 + i, device=DEV)[0])
    return m.eval()


def _pair(arch, q_level, ptq, hw=32, batch=32):
    """(frozen QAT graph, frozen deployment graph converted from the same calibrated state)"""
    from micronet_b200 import bn_fuse
    qat = _calibrated(arch, q_level, ptq, hw, batch)
    dep = bn_fuse.iao_quantize_inference_weights(bn_fuse.iao_model_bn_fuse(qat)).eval()
    return qat, dep


def _launches(m, x):
    from micronet_b200 import functional as F_
    F_.TIMER = F_.KernelTimer()
    try:
        with torch.no_grad():
            y = m(x)
        torch.cuda.synchronize()
        return y, collections.Counter(kind for kind, *_ in F_.TIMER.records)
    finally:
        F_.TIMER = None


def _graph_logits(m, x):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            m(x)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr), torch.no_grad():
        out = m(x)
    gr.replay()
    torch.cuda.synchronize()
    return out.clone()


def _check_bitwise(qat, dep, x, i8):
    from micronet_b200 import iao
    iao.freeze_inference(qat, int8=i8)
    iao.freeze_inference(dep, int8=i8)
    convs = [c for c in dep.modules() if isinstance(c, iao.QuantConv2d) and c.quant_inference]
    assert convs and all("_int_levels" in c.__dict__ for c in convs)
    want, kinds_qat = _launches(qat, x)
    got, kinds_dep = _launches(dep, x)
    assert torch.equal(got, want), float((got - want).abs().max())
    assert kinds_dep == kinds_qat and kinds_dep
    assert torch.equal(_graph_logits(dep, x), want)
    # the operands the two graphs run on: the same levels, scales and bias bit for bit
    q_convs = [c for c in qat.modules() if isinstance(c, iao.QuantConv2d)]
    for a, b in zip(q_convs, convs):
        fa, fb = a.__dict__["_frozen"], b.__dict__["_frozen"]
        for ta, tb in zip(fa[1:], fb[1:]):
            assert torch.equal(ta, tb)


@pytest.mark.parametrize("arch", ["nin", "nin_gc", "nin_gc_pruned", "resnet18"])
@pytest.mark.parametrize("q_level,ptq", [(0, False), (1, False), (0, True)], ids=["per_channel", "per_layer", "ptq"])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_deployment_logits_are_the_qat_logits(arch, q_level, ptq, i8):
    qat, dep = _pair(arch, q_level, ptq)
    _check_bitwise(qat, dep, H.synthetic_batch(32, 32, seed=5, device=DEV)[0], i8)


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_resnet18_deployment_at_224(i8):
    qat, dep = _pair("resnet18", 0, True, hw=224, batch=8)
    _check_bitwise(qat, dep, H.synthetic_batch(8, 224, seed=5, device=DEV)[0], i8)


@pytest.mark.parametrize("arch", ["nin_gc", "resnet18"])
@pytest.mark.parametrize("q_level", [0, 1], ids=["per_channel", "per_layer"])
def test_weight_step_is_the_engine_weight_quantizer(arch, q_level):
    """the step's torch-op fake-quant is bitwise the engine's weight quantizer in eval mode: IaoWeightFn per channel,
    Quantizer.forward's activation branch (act_quant_fwd_kernel) per layer"""
    from micronet_b200 import bn_fuse, iao
    qat = _calibrated(arch, q_level, False)
    raw = bn_fuse.iao_model_bn_fuse(qat).eval()
    n = 0
    with torch.no_grad():
        for c in raw.modules():
            if isinstance(c, iao.QuantConv2d) and c.quant_inference:
                q = c.weight_quantizer
                assert torch.equal(iao.stored_fake_quant(q, c.weight)[0], q(c.weight))
                n += 1
    assert n > 0


@pytest.mark.parametrize("q_level", [0, 1], ids=["per_channel", "per_layer"])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_against_the_reference_deployment_flow(q_level, i8):
    from micronet_b200 import bn_fuse, iao
    gold = load_golden("iao_deploy", f"t0_l{q_level}")
    m = bn_fuse.iao_quantize_inference_weights(converted_iao(gold, 0, q_level)).to(DEV).eval()
    iao.freeze_inference(m, int8=i8)
    assert all("_int_levels" in c.__dict__ for c in m.modules() if isinstance(c, iao.QuantConv2d))
    with torch.no_grad():
        y = m(torch.from_numpy(gold["x"]).to(DEV))
    # 8-bit activation levels of 9 layers: one level on the other side of a rounding tie moves a logit by ~1e-4 relative
    assert rel_err(y, gold["y"]) <= 2e-4, rel_err(y, gold["y"])


@pytest.mark.parametrize("q", [(0, 0), (1, 1)], ids=["sym_per_channel", "asym_per_layer"])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_raw_converter_output_is_unchanged(q, i8):
    """no weight step: freeze_inference keeps every conv on its fp32 weight, and the logits are those of the un-frozen
    converted model"""
    from micronet_b200 import iao
    gold = load_golden("bnfuse", f"iao_t{q[0]}_l{q[1]}")
    m = converted_iao(gold, *q).to(DEV).eval()
    x = torch.from_numpy(gold["x"]).to(DEV)
    with torch.no_grad():
        plain = m(x)
    iao.freeze_inference(m, int8=i8)
    assert not any("_int_levels" in c.__dict__ or "_post_consumer" in c.__dict__ for c in m.modules())
    with torch.no_grad():
        assert torch.equal(m(x), plain)
    assert torch.equal(_graph_logits(m, x), plain)


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_weight_rewritten_after_freezing_raises(i8):
    from micronet_b200 import iao
    _, dep = _pair("nin", 0, False, batch=8)
    iao.freeze_inference(dep, int8=i8)
    x = H.synthetic_batch(8, 32, seed=5, device=DEV)[0]
    with torch.no_grad():
        want = dep(x)
        conv = dep.model[4].conv
        conv.weight.copy_(conv.weight.clone())             # the same levels written in place: verified again, accepted
        assert torch.equal(dep(x), want)
        conv.weight.mul_(1.001)
        with pytest.raises(RuntimeError, match=r"model\.4\.conv.*freeze_inference"):
            dep(x)
        with pytest.raises(RuntimeError, match=r"model\.4\.conv"):
            dep(x)                                         # still refused: nothing was cached
    iao.freeze_inference(dep, int8=i8)                     # re-frozen: that layer now runs on its fp32 weight
    assert "_int_levels" not in conv.__dict__
    with torch.no_grad():
        assert dep(x).shape == want.shape
