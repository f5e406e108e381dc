"""Frozen wbwtab inference on bit planes (wbwtab.freeze_inference) against the un-frozen eval forward.

    python -m harness.wbwtab_infer_probe [--batches 256,1024] [--rounds 5] [--reps 20]

Workload: NIN-GC W3/A2 eval forward on synthetic 3x32x32 inputs, in the two graphs a user deploys:
* G2, the headline QAT graph (``wbwtab.prepare(W=3, A=2, fuse_bn=True)``, ``.eval()``);
* G1, the reference's deployment graph (``prepare(quant_inference=True)`` -> ``bn_fuse.wbwtab_model_bn_fuse`` ->
  ``bn_fuse.wbwtab_quantize_inference_weights``).
Un-frozen and frozen models are each captured into a CUDA graph (harness.train.InferStepper) and replayed alternately over
several rounds; a round times ``reps`` replays with CUDA events, the median round is reported.  A per-kernel table (device
time per forward, torch.profiler) of one eager forward of each at batch 256 follows.  The card, its power limit and SM clock
come from a read-only nvidia-smi query.  ``--out FILE`` also writes the report to FILE."""
from __future__ import annotations

import argparse
import copy
import os
import statistics
import subprocess

import torch

from harness import train as H


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers still stand; say that the card could not be read
        return f"nvidia-smi unavailable ({type(e).__name__})"


def _randomise_bn(model, seed):
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.3)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
            m.weight.data.copy_(torch.randn(m.num_features, generator=g))
            m.bias.data.copy_(torch.randn(m.num_features, generator=g) * 0.3)


def build(graph, dev):
    import micronet_b200 as E
    base = H.build_float_model("nin_gc", seed=1)
    _randomise_bn(base, 7)
    if graph == "G2":
        m = E.wbwtab.prepare(base, W=3, A=2, fuse_bn=True).to(dev)
    else:
        m = E.wbwtab.prepare(base, W=3, A=2, quant_inference=True)
        m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=3).to(dev)
        m = E.bn_fuse.wbwtab_quantize_inference_weights(m)
    return m.eval()


def _time(st, x, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        st.step(x)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _kernel_table(model, x):
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model(x)
            torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        if t > 0:
            rows[ev.key] = (t, ev.count)
    return sorted(rows.items(), key=lambda kv: -kv[1][0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1024")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    from micronet_b200 import wbwtab
    dev = torch.device("cuda:0")
    lines = [f"card: {_card()}"]
    for graph in ("G2", "G1"):
        for B in [int(v) for v in args.batches.split(",")]:
            x, _ = H.synthetic_batch(B, 32, seed=3, device=dev)
            un = build(graph, dev)
            fz = wbwtab.freeze_inference(copy.deepcopy(un))
            sts = {"un-frozen": H.InferStepper(un, graph=True), "frozen": H.InferStepper(fz, graph=True)}
            note = ""
            try:
                with torch.no_grad():
                    same = torch.equal(un(x), fz(x))
            except ValueError as e:      # a kernel of the un-frozen path refuses this batch: time the frozen graph alone
                note, same = f"un-frozen path refused: {e}", None
                del sts["un-frozen"]
            for st in sts.values():
                for _ in range(4):
                    st.step(x)
                assert st.graph is not None, st.graph_error
            times = {k: [] for k in sts}
            for _ in range(args.rounds):
                for k, st in sts.items():
                    times[k].append(_time(st, x, args.reps))
            f = statistics.median(times["frozen"])
            if note:
                lines.append(f"{graph} batch {B}: frozen {f:.3f} ms ({B / f:.1f} k img/s); {note}")
            else:
                u = statistics.median(times["un-frozen"])
                lines.append(f"{graph} batch {B}: un-frozen {u:.3f} ms ({B / u:.1f} k img/s), frozen {f:.3f} ms "
                             f"({B / f:.1f} k img/s), x{u / f:.2f}; logits bitwise equal: {same}; rounds un-frozen "
                             f"{[round(t, 3) for t in times['un-frozen']]} frozen {[round(t, 3) for t in times['frozen']]}")
            print(lines[-1], flush=True)
            if B == 256:
                start = len(lines)
                for k, m in (("un-frozen", un), ("frozen", fz)):
                    lines.append(f"  {graph} {k}, batch 256, device us per forward (torch.profiler, eager):")
                    for name, (t, n) in _kernel_table(m, x)[:16]:
                        lines.append(f"    {t:9.1f} us  x{n:<3d} {name[:110]}")
                print("\n".join(lines[-(len(lines) - start):]), flush=True)
            del sts, un, fz
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
