#!/usr/bin/env python
"""Golden fixtures for the inference-graph converters (SURVEY 8 f3), generated FROM THE REFERENCE'S OWN bn_fuse SCRIPTS.

Needs a checkout of the reference (MICRONET_REFERENCE=<path>, 666DZY666/micronet @ c31cdd28); the tests only read the
committed fixtures:

    python tests/golden/make_golden_bnfuse.py

The reference converters are scripts that read ``args`` / ``bn_counter`` / ``bin_bn_fuse_num`` / ``device`` as module
globals; this file loads each script as a module (its ``__main__`` block does not run), sets those globals the way the
script's main block does, and calls its ``model_bn_fuse``.  Recorded: the float model's initial state, the state_dict and
module types of the converted model, and its eval output on a seeded input."""
import argparse
import copy
import importlib.util
import os
import sys

import numpy as np
import torch

REF = os.environ.get("MICRONET_REFERENCE")
if not REF:
    sys.exit("make_golden_bnfuse.py: set MICRONET_REFERENCE to a checkout of 666DZY666/micronet @ c31cdd28")
HERE = os.path.dirname(os.path.abspath(__file__))
QDIR = os.path.join(REF, "micronet", "compression", "quantization")


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_scheme(sub):
    """-> (quantize module, bn_fuse module) of one scheme, wired the way the script expects (``import quantize``)"""
    sys.path.insert(0, REF)                                 # `from micronet.base_module.op import *` (iao)
    sys.path.insert(0, os.path.join(REF, "micronet"))       # `from models import nin_gc, nin`
    q = _load(os.path.join(QDIR, sub, "quantize.py"), "quantize")
    b = _load(os.path.join(QDIR, sub, "bn_fuse", "bn_fuse.py"), "ref_bn_fuse_" + sub.replace("/", "_"))
    del sys.modules["quantize"]
    sys.path.pop(0)
    sys.path.pop(0)
    return q, b


def randomize_bn(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.3)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_((torch.rand(m.num_features, generator=g) + 0.3) * torch.where(
                    torch.rand(m.num_features, generator=g) < 0.3, -1.0, 1.0))      # some negative gammas
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.3)


def save(name, out):
    np.savez_compressed(os.path.join(HERE, f"bnfuse_{name}.npz"), **out)
    print("wrote", name, len(out), "arrays")


CFG = [16, 16, 16, 32, 32, 32, 64, 64]


def wbwtab_case(W):
    from models import nin_gc as ref_nin_gc
    q, b = load_scheme("wbwtab")
    torch.manual_seed(11 + W)
    base = ref_nin_gc.Net(cfg=CFG)
    randomize_bn(base, 5)
    out = {f"init.{k}": v.numpy().copy() for k, v in base.state_dict().items()}
    train = copy.deepcopy(base)
    q.prepare(train, inplace=True, A=2, W=W)
    inf = copy.deepcopy(base)
    q.prepare(inf, inplace=True, A=2, W=W, quant_inference=True)
    inf.load_state_dict(train.state_dict())
    b.args = argparse.Namespace(W=W, A=2)
    b.bn_counter = 0
    b.bin_bn_fuse_num = sum(isinstance(m, q.ActivationQuantizer) for m in inf.modules())
    b.model_bn_fuse(inf, inplace=True)
    inf.eval()
    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        y = inf(x)
    out["x"], out["y"] = x.numpy(), y.numpy()
    for k, v in inf.state_dict().items():
        out[f"fused.{k}"] = v.numpy().copy()
    out["types"] = np.array([f"{n}:{type(m).__name__}" for n, m in inf.named_modules()])
    save(f"wbwtab_W{W}", out)


def iao_case(q_type, q_level):
    from models import nin_gc as ref_nin_gc
    q, b = load_scheme(os.path.join("wqaq", "iao"))
    torch.manual_seed(23 + q_type * 2 + q_level)
    base = ref_nin_gc.Net(cfg=CFG)
    randomize_bn(base, 9)
    out = {f"init.{k}": v.numpy().copy() for k, v in base.state_dict().items()}
    model = copy.deepcopy(base)
    q.prepare(model, inplace=True, a_bits=8, w_bits=8, q_type=q_type, q_level=q_level, weight_observer=0, bn_fuse=True,
              pretrained_model=True)
    model.train()
    g = torch.Generator().manual_seed(4)
    calib = [torch.randn(4, 3, 32, 32, generator=g) for _ in range(2)]
    with torch.no_grad():
        for c in calib:
            model(c)
    for i, c in enumerate(calib):
        out[f"calib{i}"] = c.numpy()
    for k, v in model.state_dict().items():
        out[f"calibrated.{k}"] = v.numpy().copy()
    b.args = argparse.Namespace(a_bits=8, w_bits=8, q_type=q_type, q_level=q_level)
    b.device = "cpu"
    # the script passes a stale ``device=`` keyword that the reference's own QuantConv2d (IAO:326-346) no longer accepts
    # (TypeError as shipped); the keyword is dropped here, nothing else of the script is touched
    import types
    b.quantize = types.SimpleNamespace(QuantBNFuseConv2d=q.QuantBNFuseConv2d,
                                       QuantConv2d=lambda *a, device=None, **k: q.QuantConv2d(*a, **k))
    with torch.no_grad():
        inf = b.model_bn_fuse(model)
    inf.eval()
    x = torch.randn(4, 3, 32, 32, generator=g)
    with torch.no_grad():
        y = inf(x)
    out["x"], out["y"] = x.numpy(), y.numpy()
    for k, v in inf.state_dict().items():
        out[f"fused.{k}"] = v.numpy().copy()
    out["types"] = np.array([f"{n}:{type(m).__name__}" for n, m in inf.named_modules()])
    save(f"iao_t{q_type}_l{q_level}", out)


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(REF, "micronet"))
    wbwtab_case(2)
    wbwtab_case(3)
    iao_case(0, 0)
    iao_case(1, 1)
