"""bf16 vs int8 operands on the frozen ResNet-18 PTQ inference graph (workload resnet18_iao_ptq_224: batch 64 at 224 x 224,
2 calibration batches): whole-model CUDA-graph replays of iao.freeze_inference() and freeze_inference(int8=True) in one
process, alternating A/B over three rounds, an eager per-layer table of fwd_pk vs fwd_pk_i8 CUDA-event times per conv shape,
the launch count of one forward of each, and a bitwise comparison of the two logits tensors.  Prints one JSON object (GPU
name and power limit included; the power limit is read with a read-only nvidia-smi query).

    python -m harness.int8_probe [--batch 64] [--iters 20] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def _graph(model, x):
    with torch.no_grad():
        for _ in range(2):
            model(x)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = model(x)
    return g, out


def _replay_ms(g, iters):
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _layer_table(model, x, reps=5):
    """{conv shape: median CUDA-event ms per forward} of the fwd_pk / fwd_pk_i8 records of eager forwards"""
    from micronet_b200 import functional as F_
    with torch.no_grad():
        model(x)
        F_.TIMER = F_.KernelTimer()
        try:
            for _ in range(reps):
                model(x)
            torch.cuda.synchronize()
            summ = F_.TIMER.summary()
        finally:
            F_.TIMER = None
    out = {}
    for (kind, shape), ms in summ.items():
        if kind in ("fwd_pk", "fwd_pk_i8"):
            per = sorted(ms)
            out.setdefault(shape, {})[kind] = per[len(per) // 2]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on cuda:0"
    from harness import train as H
    from micronet_b200 import _lib as L, iao
    dev = torch.device("cuda:0")
    w = H.WORKLOADS["resnet18_iao_ptq_224"]
    B = args.batch
    model = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"]).to(dev)
    x = H.synthetic_batch(B, w["hw"], seed=100)[0].to(dev)
    st = H.InferStepper(model)
    st.calibrate([H.synthetic_batch(max(2, B // 8), w["hw"], seed=50 + i)[0].to(dev) for i in range(w["calib_batches"])])

    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "workload": "resnet18_iao_ptq_224",
           "batch": B, "iters": args.iters}
    modes = {"bf16": False, "int8": True}
    graphs, outs, launches, tables, keep = {}, {}, {}, {}, []
    for name, i8 in modes.items():
        # the captured graph reads the frozen weights / packed images made before the capture: re-freezing drops the
        # modules' references to them, so they are kept alive here
        keep.append([m.__dict__.get("_frozen") for m in model.modules()])
        iao.freeze_inference(model, int8=i8)
        with torch.no_grad():
            model(x)
            n0 = L.launch_count()
            outs[name] = model(x).clone()
            torch.cuda.synchronize()
            launches[name] = L.launch_count() - n0
        tables[name] = _layer_table(model, x)
        graphs[name] = _graph(model, x)
    res["logits_bitwise_equal"] = bool(torch.equal(outs["bf16"], outs["int8"]))
    res["graph_logits_bitwise_equal"] = bool(torch.equal(graphs["bf16"][1], graphs["int8"][1]))
    res["launches_per_forward"] = launches
    rounds = []
    for _ in range(args.rounds):
        r = {}
        for name in modes:                       # A/B alternating inside every round
            r[name] = _replay_ms(graphs[name][0], args.iters)
        rounds.append(r)
    res["rounds_ms"] = rounds
    for name in modes:
        ms = sorted(r[name] for r in rounds)[len(rounds) // 2]
        res[f"{name}_ms_median"] = ms
        res[f"{name}_img_s"] = B / (ms / 1e3)
    rows = []
    fields = [f for f, _ in L.ConvShape._fields_]
    for shape in sorted(set(tables["bf16"]) | set(tables["int8"])):
        s = dict(zip(fields, shape))
        b16, i8 = tables["bf16"].get(shape, {}).get("fwd_pk"), tables["int8"].get(shape, {}).get("fwd_pk_i8")
        rows.append({"shape": f"{s['in_c']}->{s['out_c']} {s['ker_h']}x{s['ker_w']} s{s['stride_h']} @{s['in_h']}",
                     "fwd_pk_ms": b16, "fwd_pk_i8_ms": i8, "speedup": (b16 / i8) if (b16 and i8) else None})
    res["layers"] = rows
    txt = json.dumps(res)
    print(txt)
    if args.json:
        with open(args.json, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
