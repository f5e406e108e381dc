"""The wbwtab training graphs that run on the round-1 fused tensor-core convolutions: full-precision-activation models
(A = 32, every covered conv: exact 3-piece split forward and data gradient, weight gradient through the inexact flag and
mnb_conv2d_wgrad_cond) and the un-fused A = 2 graph, teacher-forced layer by layer against the oracle; and an A = 32 QAT
step replayed from a CUDA graph, where the wgrad_cond overwrite is predicated on a device flag, against eager steps."""
import copy

import pytest
import torch

from tests import tc_conv_cases as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _expected(shape, kinds):
    """what the conv of ``shape`` must have run, given the kernel kinds recorded for it"""
    B, Cc, H, W, K, R, G = shape
    bad = []
    fwd_ok = T.refusal("fwd", shape) is None
    if fwd_ok and ("fwd_tc" not in kinds or "fwd" in kinds):
        bad.append("fwd_tc did not run")
    if not fwd_ok and "fwd" not in kinds:
        # a refused forward goes to the packed-operand family, whose backward is its own
        return bad if any(k.endswith("_pk") for k in kinds) else bad + [f"no forward recorded: {kinds}"]
    dgrad_ok = T.refusal("dgrad", shape) is None
    if "dgrad_tc" not in kinds or (dgrad_ok == ("dgrad" in kinds)):
        bad.append(f"dgrad: plan {'accepts' if dgrad_ok else 'refuses'}, ran {kinds}")
    wgrad_ok = T.refusal("wgrad", shape) is None
    if wgrad_ok != ("wgrad_tc" in kinds) or wgrad_ok == ("wgrad" in kinds):
        bad.append(f"wgrad: plan {'accepts' if wgrad_ok else 'refuses'}, ran {kinds}")
    return bad


@pytest.mark.parametrize("model,W,A", [("nin_gc", 3, 32), ("nin", 2, 32), ("nin_gc", 3, 2)],
                         ids=["nin_gc_w3a32", "nin_w2a32", "nin_gc_w3a2_unfused"])
def test_wbwtab_graph_layers_teacher_forced(model, W, A):
    from harness import train as H
    from micronet_b200 import _lib as L, functional as F_, wbwtab
    from tests.test_gpu_parity import _teacher_forced
    base = H.build_float_model(model, seed=1)
    om = H.prepare_oracle(copy.deepcopy(base), "wbwtab", W=W, A=A)
    om.train()
    em = H.prepare_engine(copy.deepcopy(base), "wbwtab", W=W, A=A).to(DEV)
    em.train()
    for m in list(om.modules()) + list(em.modules()):
        if isinstance(m, torch.nn.ReLU):     # an A = 32 ActivationQuantizer is its block's ReLU: replayed on a leaf tensor
            m.inplace = False
    x, t = H.synthetic_batch(8, 32, seed=21)
    old = F_.TIMER
    F_.TIMER = F_.KernelTimer()
    try:
        _teacher_forced(om, em, x, t)
        records = F_.TIMER.records
    finally:
        F_.TIMER = old
    L.tc_check()
    by_shape = {}
    for kind, sh, _, _ in records:
        by_shape.setdefault(sh, set()).add(kind)
    convs = [m for m in em.modules() if isinstance(m, wbwtab.QuantConv2d)]
    assert len(convs) == 7
    bad, ran = [], set()
    for sh, kinds in by_shape.items():
        B, Cc, H_, W_, K, R, _, st, _, pad, _, _, _, G = sh
        if not any(c.in_channels == Cc and c.out_channels == K and c.kernel_size[0] == R and c.groups == G for c in convs):
            continue
        shape = (B, Cc, H_, W_, K, R, G)
        bad += [(shape, b) for b in _expected(shape, kinds)]
        ran |= kinds
    assert not bad, bad
    assert {"fwd_tc", "dgrad_tc", "wgrad_tc"} <= ran, ran


def test_a32_qat_graph_replay_equals_eager_steps():
    """NIN-GC W3 A = 32 (every conv forward on fwd_tc, weight gradients through the flag-predicated wgrad_cond): a step
    replayed from a CUDA graph computes what the eager step computes, bit for bit"""
    from harness import train as H
    from micronet_b200 import _lib as L
    base = H.build_float_model("nin_gc", seed=1)
    batches = [tuple(v.to(DEV) for v in H.synthetic_batch(8, 32, seed=40 + i)) for i in range(2)]
    runs = {}
    for graph in (False, True):
        m = H.prepare_engine(copy.deepcopy(base), "wbwtab", W=3, A=32).to(DEV)
        st = H.QatStepper(m, flat=True, graph=graph, graph_warmup=2)
        losses = [st.step(*batches[i % 2]).detach().clone() for i in range(5)]
        torch.cuda.synchronize()
        if graph:
            assert st.graph is not None, st.graph_error
        runs[graph] = (losses, [p.detach().clone() for p in m.parameters()])
    L.tc_check()
    for a, b in zip(runs[False][0], runs[True][0]):
        assert torch.equal(a.reshape(1).view(torch.uint8), b.reshape(1).view(torch.uint8))
    for a, b in zip(runs[False][1], runs[True][1]):
        assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
