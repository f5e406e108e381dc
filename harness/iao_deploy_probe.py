"""Frozen IAO deployment graphs (bn_fuse.iao_model_bn_fuse -> bn_fuse.iao_quantize_inference_weights ->
iao.freeze_inference) against the un-frozen deployment graph and the frozen QAT graph they came from.

    python -m harness.iao_deploy_probe [--rounds 5] [--reps 20] [--out FILE]

Workloads: NIN and NIN-GC at their default cfg at batch 256 on synthetic 3x32x32 inputs, ResNet-18 (BASELINE.json
configs[4]) at batch 64 on synthetic 3x224x224 inputs; IAO W8A8 symmetric with per-channel weights and ``bn_fuse=True``
(the README's IAO row), randomised BatchNorm statistics, calibrated in train mode under no_grad on two synthetic batches
(NIN / NIN-GC QAT observers, ResNet-18 PTQ), then converted with the weight step.  Five models per workload - the
un-frozen deployment graph, and the frozen deployment and frozen QAT graphs with bf16 planes and with ``int8=True`` - are
each captured into a CUDA graph (harness.train.InferStepper) and replayed alternately over several rounds; a round times
``reps`` replays with CUDA events, the median round is reported.  The logits of each frozen deployment graph are compared
bitwise with those of the frozen QAT graph of the same plane format.  The card, its power limit and SM clock come from a
read-only nvidia-smi query."""
from __future__ import annotations

import argparse
import copy
import os
import statistics

import torch

from harness import train as H
from harness.wbwtab_infer_probe import _card, _randomise_bn, _time

WORKLOADS = (("nin", 256, 32, False), ("nin_gc", 256, 32, False), ("resnet18", 64, 224, True))


def build(arch, dev, batch, hw, ptq):
    import micronet_b200 as E
    base = H.build_float_model(arch, seed=1)
    with torch.no_grad():
        _randomise_bn(base, 7)
    m = E.iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True, ptq=ptq).to(dev)
    m.train()
    with torch.no_grad():
        for i in range(2):
            m(H.synthetic_batch(batch, hw, seed=20 + i, device=dev)[0])
    return m.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    from micronet_b200 import bn_fuse, iao
    dev = torch.device("cuda:0")
    lines = [f"card: {_card()}"]
    print(lines[-1], flush=True)
    for arch, B, hw, ptq in WORKLOADS:
        qat = build(arch, dev, B, hw, ptq)
        dep = bn_fuse.iao_quantize_inference_weights(bn_fuse.iao_model_bn_fuse(qat)).eval()
        models = {"deploy un-frozen": dep}
        for i8 in (False, True):
            tag = "int8" if i8 else "bf16"
            models[f"deploy frozen {tag}"] = iao.freeze_inference(copy.deepcopy(dep), int8=i8)
            models[f"QAT frozen {tag}"] = iao.freeze_inference(copy.deepcopy(qat), int8=i8)
        x, _ = H.synthetic_batch(B, hw, seed=3, device=dev)
        sts = {k: H.InferStepper(m, graph=True) for k, m in models.items()}
        for st in sts.values():
            for _ in range(4):
                st.step(x)
            assert st.graph is not None, st.graph_error
        times = {k: [] for k in sts}
        for _ in range(args.rounds):
            for k, st in sts.items():
                times[k].append(_time(st, x, args.reps))
        med = {k: statistics.median(v) for k, v in times.items()}
        base = med["deploy un-frozen"]
        name = f"{arch} W8A8 {'PTQ' if ptq else 'QAT'} batch {B} {hw}x{hw}"
        for k in sts:
            same = ""
            if k.startswith("deploy frozen"):
                tag = k.split()[-1]
                eq = torch.equal(sts[k].step(x).clone(), sts[f"QAT frozen {tag}"].step(x).clone())
                same = f"; logits bitwise equal to QAT frozen {tag}: {eq}"
            lines.append(f"{name}: {k} {med[k]:.3f} ms ({B / med[k]:.1f} k img/s), x{base / med[k]:.2f} over deploy "
                         f"un-frozen; rounds {[round(t, 3) for t in times[k]]}{same}")
            print(lines[-1], flush=True)
        del sts, models, qat, dep
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
