#!/usr/bin/env python
"""Generate the golden fixtures in this directory FROM THE REFERENCE ITSELF.

Needs a checkout of the reference (666DZY666/micronet @ c31cdd28); the tests only read the committed fixtures:

    MICRONET_REFERENCE=<path to the checkout> python tests/golden/make_golden.py

For every case below it instantiates the reference's own module
(``micronet.compression.quantization.{wbwtab,wqaq.dorefa,wqaq.iao}.quantize``),
drives it with seeded synthetic inputs for a few training steps plus one eval
step, and records inputs, outputs, gradients and the post-step state_dict.
The committed ``*.npz`` files are what pins ``oracle/reference_port.py``
(tests/test_oracle_golden.py) and, through it, the CUDA path.
"""
import json
import os
import sys

import numpy as np
import torch

REF = os.environ.get("MICRONET_REFERENCE")
if not REF:
    sys.exit("make_golden.py: set MICRONET_REFERENCE to a checkout of 666DZY666/micronet @ c31cdd28")
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import micronet.compression.quantization.wbwtab.quantize as ref_wb  # noqa: E402
import micronet.compression.quantization.wqaq.dorefa.quantize as ref_df  # noqa: E402
import micronet.compression.quantization.wqaq.iao.quantize as ref_iao  # noqa: E402
from micronet.models import nin as ref_nin, nin_gc as ref_nin_gc, resnet as ref_resnet  # noqa: E402

from tests.golden.cases import LAYER_CASES, MODEL_CASES, make_input  # noqa: E402

REF_CLASSES = {
    ("dorefa", "conv"): ref_df.QuantConv2d,
    ("dorefa", "linear"): ref_df.QuantLinear,
    ("wbwtab", "conv"): ref_wb.QuantConv2d,
    ("iao", "conv"): ref_iao.QuantConv2d,
    ("iao", "bnfuse"): ref_iao.QuantBNFuseConv2d,
    ("iao", "linear"): ref_iao.QuantLinear,
    ("iao", "convT"): ref_iao.QuantConvTranspose2d,
}


def run_layer_case(case):
    torch.manual_seed(case["seed"])
    mod = REF_CLASSES[(case["scheme"], case["kind"])](*case["args"], **case["kwargs"])
    out = {}
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if n == "weight":
                p.mul_(case.get("weight_gain", 1.0))
            if n == "bias":
                p.uniform_(-0.5, 0.5)
            if n == "beta":
                p.uniform_(-0.3, 0.3)
    for n, t in mod.state_dict().items():
        out[f"init.{n}"] = t.detach().clone().numpy()
    steps = case["train_steps"] + case["eval_steps"]
    for i in range(steps):
        training = i < case["train_steps"]
        mod.train(training)
        x = make_input(case, i).requires_grad_(True)
        y = mod(x)
        go = torch.randn(y.shape, generator=torch.Generator().manual_seed(1000 + case["seed"] * 17 + i))
        out[f"s{i}.x"] = x.detach().numpy().copy()
        out[f"s{i}.y"] = y.detach().numpy().copy()
        out[f"s{i}.go"] = go.numpy().copy()
        if training or case.get("eval_backward", False):
            mod.zero_grad()
            y.backward(go)
            out[f"s{i}.dx"] = x.grad.numpy().copy()
            for n, p in mod.named_parameters():
                out[f"s{i}.d.{n}"] = p.grad.detach().numpy().copy()
        for n, t in mod.state_dict().items():
            out[f"s{i}.state.{n}"] = t.detach().clone().numpy()
        # integer levels actually used by this forward (fp32-valued)
        if case["scheme"] == "dorefa":
            ab, wb = case["kwargs"].get("a_bits", 8), case["kwargs"].get("w_bits", 8)
            out[f"s{i}.lvl_a"] = (mod.activation_quantizer(x.detach()) * float(2**ab - 1)).round().numpy()
            out[f"s{i}.lvl_w"] = ((mod.weight_quantizer(mod.weight.detach()) + 1) / 2 * float(2**wb - 1)).round().numpy()
        elif case["scheme"] == "iao":
            mod.eval()
            aq, wq = mod.activation_quantizer, mod.weight_quantizer
            with torch.no_grad():
                out[f"s{i}.lvl_a"] = (aq(x.detach()) / aq.scale - aq.zero_point).round().numpy()
    return out


def run_model_case(case):
    from harness import models as zoo

    torch.manual_seed(case["seed"])
    if case["model"] == "nin_gc":
        mine, ref = zoo.NINGC(case["cfg"]), ref_nin_gc.Net(case["cfg"])
    elif case["model"] == "nin":
        mine, ref = zoo.NIN(case["cfg"]), ref_nin.Net(case["cfg"])
    else:
        mine = zoo.ResNet(widths=tuple(case["cfg"]))
        ref = ref_resnet.resnet18()
        # shrink the reference resnet to the same widths
        ref = _narrow_resnet(case["cfg"])
    zoo.init_like_reference(mine)
    ref.load_state_dict(mine.state_dict())
    out = {f"init.{k}": v.numpy().copy() for k, v in mine.state_dict().items()}
    if case["scheme"] == "wbwtab":
        ref = ref_wb.prepare(ref, inplace=True, **case["prepare"])
    elif case["scheme"] == "dorefa":
        ref = ref_df.prepare(ref, inplace=True, **case["prepare"])
    else:
        ref = ref_iao.prepare(ref, inplace=True, **case["prepare"])
    params = [{"params": [p], "lr": case["lr"], "weight_decay": case["wd"]} for p in ref.parameters()]
    opt = torch.optim.Adam(params, lr=case["lr"], weight_decay=case["wd"])
    crit = torch.nn.CrossEntropyLoss()
    ref.train()
    for i in range(case["steps"]):
        g = torch.Generator().manual_seed(case["seed"] * 31 + i)
        x = torch.randn(case["batch"], 3, case["hw"], case["hw"], generator=g)
        t = torch.randint(0, 10, (case["batch"],), generator=g)
        y = ref(x)
        loss = crit(y, t)
        opt.zero_grad()
        loss.backward()
        out[f"s{i}.x"], out[f"s{i}.t"] = x.numpy().copy(), t.numpy().copy()
        out[f"s{i}.logits"], out[f"s{i}.loss"] = y.detach().numpy().copy(), np.float32(loss.item())
        for n, p in ref.named_parameters():
            if p.grad is not None and (n.endswith("weight") or n.endswith("gamma")):
                out[f"s{i}.gradnorm.{n}"] = np.float32(p.grad.norm().item())
        opt.step()
    for n, t in ref.state_dict().items():
        out[f"final.{n}"] = t.detach().numpy().copy()
    return out


def _narrow_resnet(widths):
    r = ref_resnet.ResNet.__new__(ref_resnet.ResNet)
    torch.nn.Module.__init__(r)
    nn = torch.nn
    r.in_channels = widths[0]
    r.conv1 = nn.Sequential(nn.Conv2d(3, widths[0], kernel_size=3, padding=1, bias=False),
                            nn.BatchNorm2d(widths[0]), nn.ReLU(inplace=True))
    r.conv2_x = r._make_layer(ref_resnet.BasicBlock, widths[0], 2, 1)
    r.conv3_x = r._make_layer(ref_resnet.BasicBlock, widths[1], 2, 2)
    r.conv4_x = r._make_layer(ref_resnet.BasicBlock, widths[2], 2, 2)
    r.conv5_x = r._make_layer(ref_resnet.BasicBlock, widths[3], 2, 2)
    r.avg_pool = nn.AdaptiveAvgPool2d((1, 1))
    r.fc = nn.Linear(widths[3], 10)
    return r


def main():
    torch.set_num_threads(1)  # fixed summation order for the fixtures
    only_new = "--only-new" in sys.argv     # keep the committed fixtures, generate the cases that have none yet
    for case in LAYER_CASES:
        if only_new and os.path.exists(os.path.join(HERE, f"layer_{case['name']}.npz")):
            continue
        arrays = run_layer_case(case)
        np.savez_compressed(os.path.join(HERE, f"layer_{case['name']}.npz"), **arrays)
        print("layer", case["name"], sum(a.nbytes for a in arrays.values()) // 1024, "KiB raw")
    for case in MODEL_CASES:
        if only_new and os.path.exists(os.path.join(HERE, f"model_{case['name']}.npz")):
            continue
        arrays = run_model_case(case)
        np.savez_compressed(os.path.join(HERE, f"model_{case['name']}.npz"), **arrays)
        print("model", case["name"], sum(a.nbytes for a in arrays.values()) // 1024, "KiB raw")
    with open(os.path.join(HERE, "MANIFEST.json"), "w") as f:
        json.dump({"torch": torch.__version__, "reference": "666DZY666/micronet@c31cdd28",
                   "layer_cases": [c["name"] for c in LAYER_CASES],
                   "model_cases": [c["name"] for c in MODEL_CASES]}, f, indent=1)


if __name__ == "__main__":
    main()
