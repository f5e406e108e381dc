"""Frozen DoReFa inference on level planes (dorefa.freeze_inference) against the un-frozen eval forward.

    python -m harness.dorefa_infer_probe [--batch 256] [--rounds 5] [--reps 20] [--out FILE]

Workloads: the two DoReFa configs of BASELINE.json in eval mode on synthetic 3x32x32 inputs, as ``dorefa.prepare(...)``
graphs with non-trivial BatchNorm statistics: NIN W8A8 (bf16 planes) and NIN-GC W4A4 (bf16 planes, and int8 operands with
``int8=True``).  Un-frozen and frozen models are each captured into a CUDA graph (harness.train.InferStepper) and replayed
alternately over several rounds; a round times ``reps`` replays with CUDA events, the median round is reported.  The frozen
logits of the timed model are compared bitwise with the block-by-block composition of existing kernels that
tests/test_gpu_dorefa_frozen.py checks.  A per-kernel table (device time per forward, torch.profiler) of one eager forward
of each follows.  The card, its power limit and SM clock come from a read-only nvidia-smi query."""
from __future__ import annotations

import argparse
import copy
import os
import statistics

import torch

from harness import train as H
from harness.wbwtab_infer_probe import _card, _kernel_table, _randomise_bn, _time

CONFIGS = [("NIN W8A8", "nin", 8, False), ("NIN-GC W4A4", "nin_gc", 4, False), ("NIN-GC W4A4 int8", "nin_gc", 4, True)]


def build(arch, bits, dev):
    import micronet_b200 as E
    base = H.build_float_model(arch, seed=1)
    _randomise_bn(base, 7)
    return E.dorefa.prepare(base, a_bits=bits, w_bits=bits).to(dev).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    from micronet_b200 import dorefa
    from tests.test_gpu_dorefa_frozen import _reference_logits
    dev = torch.device("cuda:0")
    B = args.batch
    lines = [f"card: {_card()}"]
    x, _ = H.synthetic_batch(B, 32, seed=3, device=dev)
    for name, arch, bits, i8 in CONFIGS:
        un = build(arch, bits, dev)
        fz = copy.deepcopy(un)
        ref = _reference_logits(fz, x, bits, i8)
        dorefa.freeze_inference(fz, int8=i8)
        sts = {"un-frozen": H.InferStepper(un, graph=True), "frozen": H.InferStepper(fz, graph=True)}
        for st in sts.values():
            for _ in range(4):
                st.step(x)
            assert st.graph is not None, st.graph_error
        times = {k: [] for k in sts}
        for _ in range(args.rounds):
            for k, st in sts.items():
                times[k].append(_time(st, x, args.reps))
        with torch.no_grad():
            got, base = fz(x), un(x)
        same = torch.equal(got, ref)
        diff = (got - base).abs().max().item()
        u, f = statistics.median(times["un-frozen"]), statistics.median(times["frozen"])
        lines.append(f"{name} batch {B}: un-frozen {u:.3f} ms ({B / u:.1f} k img/s), frozen {f:.3f} ms ({B / f:.1f} k img/s), "
                     f"x{u / f:.2f}; frozen logits bitwise equal to the block composition: {same}; max |frozen - un-frozen| "
                     f"{diff:.3g}; rounds un-frozen {[round(t, 3) for t in times['un-frozen']]} frozen "
                     f"{[round(t, 3) for t in times['frozen']]}")
        print(lines[-1], flush=True)
        start = len(lines)
        for k, m in (("un-frozen", un), ("frozen", fz)):
            lines.append(f"  {name} {k}, batch {B}, device us per forward (torch.profiler, eager):")
            for kname, (t, n) in _kernel_table(m, x)[:16]:
                lines.append(f"    {t:9.1f} us  x{n:<3d} {kname[:110]}")
        print("\n".join(lines[start:]), flush=True)
        del sts, un, fz
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
