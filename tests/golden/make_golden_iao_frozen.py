#!/usr/bin/env python
"""Golden fixture for frozen IAO NIN-GC inference graphs (iao.freeze_inference block links), generated FROM THE REFERENCE'S
OWN IAO modules: the reference's nin_gc.Net at a small cfg, its ``prepare(..., bn_fuse=True)`` (W8A8, symmetric,
per-channel weights - the IAO configuration of the reference README), calibration batches in train mode under no_grad,
then the eval forward of that prepared model (QuantMaxPool2d pools included) on a seeded input.

Needs a checkout of the reference (MICRONET_REFERENCE=<path>, 666DZY666/micronet @ c31cdd28); the tests only read the
committed fixture:

    python tests/golden/make_golden_iao_frozen.py

Recorded: the calibrated state_dict (float weights, folded BatchNorm statistics, observer ranges and scales), the eval
input and the eval output."""
import copy
import importlib.util
import os
import sys

import numpy as np
import torch

REF = os.environ.get("MICRONET_REFERENCE")
if not REF:
    sys.exit("make_golden_iao_frozen.py: set MICRONET_REFERENCE to a checkout of 666DZY666/micronet @ c31cdd28")
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = [32, 32, 32, 64, 64, 64, 128, 128]


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def main():
    sys.path.insert(0, REF)                                 # `from micronet.base_module.op import *` (iao)
    sys.path.insert(0, os.path.join(REF, "micronet"))       # `from models import nin_gc`
    from models import nin_gc as ref_nin_gc
    q = _load(os.path.join(REF, "micronet", "compression", "quantization", "wqaq", "iao", "quantize.py"), "ref_iao_quantize")
    torch.manual_seed(31)
    base = ref_nin_gc.Net(cfg=CFG)
    g = torch.Generator().manual_seed(6)
    with torch.no_grad():
        for m in base.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.3)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.3)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.3)
    out = {}
    model = copy.deepcopy(base)
    q.prepare(model, inplace=True, a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0, bn_fuse=True,
              pretrained_model=True)
    model.train()
    calib = [torch.randn(8, 3, 32, 32, generator=g) for _ in range(3)]
    with torch.no_grad():
        for c in calib:
            model(c)
    for k, v in model.state_dict().items():
        out[f"calibrated.{k}"] = v.numpy().copy()
    model.eval()
    x = torch.randn(8, 3, 32, 32, generator=g)
    with torch.no_grad():
        y = model(x)
    out["x"], out["y"] = x.numpy(), y.numpy()
    np.savez_compressed(os.path.join(HERE, "iao_frozen_nin_gc_w8a8.npz"), **out)
    print("wrote iao_frozen_nin_gc_w8a8", len(out), "arrays, y", tuple(y.shape))


if __name__ == "__main__":
    main()
