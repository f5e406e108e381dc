#!/usr/bin/env python
"""Golden fixtures for the IAO deployment flow (bn_fuse.iao_model_bn_fuse -> bn_fuse.iao_quantize_inference_weights ->
iao.freeze_inference), generated FROM THE REFERENCE'S OWN SCRIPTS: its IAO ``bn_fuse.py`` converter, run as
make_golden_bnfuse.py runs it (the stale ``device=`` keyword dropped), then the weight step of
``bn_fused_model_test.py:199-201`` on the model in eval mode,

    for m in model.modules():
        if isinstance(m, quantize.QuantConv2d):
            m.weight.data = m.weight_quantizer(m.weight)

for NIN-GC W8A8 with symmetric per-channel and symmetric per-layer weight quantizers.

Needs a checkout of the reference (MICRONET_REFERENCE=<path>, 666DZY666/micronet @ c31cdd28); the tests only read the
committed fixtures:

    python tests/golden/make_golden_iao_deploy.py

Recorded: the float model's initial state, the calibrated ``prepare(bn_fuse=True)`` state, the state_dict of the
weight-stepped deployment model, and its eval output on a seeded input."""
import argparse
import copy
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_bnfuse as B  # noqa: E402  (exits without MICRONET_REFERENCE)

CFG = [16, 16, 16, 32, 32, 32, 64, 64]


def deploy_case(q_level):
    from models import nin_gc as ref_nin_gc
    q, b = B.load_scheme(os.path.join("wqaq", "iao"))
    torch.manual_seed(41 + q_level)
    base = ref_nin_gc.Net(cfg=CFG)
    B.randomize_bn(base, 13)
    out = {f"init.{k}": v.numpy().copy() for k, v in base.state_dict().items()}
    model = copy.deepcopy(base)
    q.prepare(model, inplace=True, a_bits=8, w_bits=8, q_type=0, q_level=q_level, weight_observer=0, bn_fuse=True,
              pretrained_model=True)
    model.train()
    g = torch.Generator().manual_seed(8)
    with torch.no_grad():
        for _ in range(2):
            model(torch.randn(4, 3, 32, 32, generator=g))
    for k, v in model.state_dict().items():
        out[f"calibrated.{k}"] = v.numpy().copy()
    b.args = argparse.Namespace(a_bits=8, w_bits=8, q_type=0, q_level=q_level)
    b.device = "cpu"
    b.quantize = types.SimpleNamespace(QuantBNFuseConv2d=q.QuantBNFuseConv2d,
                                       QuantConv2d=lambda *a, device=None, **k: q.QuantConv2d(*a, **k))
    with torch.no_grad():
        inf = b.model_bn_fuse(model)
    inf.eval()
    for m in inf.modules():                                 # bn_fused_model_test.py:199-201
        if isinstance(m, q.QuantConv2d):
            m.weight.data = m.weight_quantizer(m.weight)
    x = torch.randn(4, 3, 32, 32, generator=g)
    with torch.no_grad():
        y = inf(x)
    out["x"], out["y"] = x.numpy(), y.numpy()
    for k, v in inf.state_dict().items():
        out[f"deploy.{k}"] = v.numpy().copy()
    name = f"iao_deploy_t0_l{q_level}"
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
    print("wrote", name, len(out), "arrays")


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(B.REF, "micronet"))
    deploy_case(0)
    deploy_case(1)
