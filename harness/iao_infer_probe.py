"""Frozen IAO inference of NIN / NIN-GC with block hand-offs (iao.freeze_inference, handoff=True) against the same frozen
graph without them (handoff=False).

    python -m harness.iao_infer_probe [--batch 256] [--rounds 5] [--reps 20] [--out FILE]

Workloads: NIN and NIN-GC at their default cfg, IAO W8A8 symmetric with per-channel weights and ``bn_fuse=True`` (the IAO
configuration of the reference README), non-trivial BatchNorm statistics, calibrated in train mode under no_grad on two
synthetic batches, then eval on synthetic 3x32x32 inputs.  For bf16 planes and for ``int8=True`` the two frozen models are
each captured into a CUDA graph (harness.train.InferStepper) and replayed alternately over several rounds; a round times
``reps`` replays with CUDA events, the median round is reported.  The logits of the two timed variants are compared
bitwise.  A per-kernel table (device time per forward, torch.profiler) of one eager forward of each follows.  The card,
its power limit and SM clock come from a read-only nvidia-smi query."""
from __future__ import annotations

import argparse
import copy
import os
import statistics

import torch

from harness import train as H
from harness.wbwtab_infer_probe import _card, _kernel_table, _randomise_bn, _time


def build(arch, dev, batch):
    import micronet_b200 as E
    base = H.build_float_model(arch, seed=1)
    with torch.no_grad():
        _randomise_bn(base, 7)
    m = E.iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True).to(dev)
    m.train()
    with torch.no_grad():
        for i in range(2):
            m(H.synthetic_batch(batch, 32, seed=20 + i, device=dev)[0])
    return m.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    from micronet_b200 import iao
    dev = torch.device("cuda:0")
    B = args.batch
    lines = [f"card: {_card()}"]
    x, _ = H.synthetic_batch(B, 32, seed=3, device=dev)
    for arch in ("nin", "nin_gc"):
        calibrated = build(arch, dev, B)
        for i8 in (False, True):
            name = f"{'NIN' if arch == 'nin' else 'NIN-GC'} W8A8 {'int8' if i8 else 'bf16'}"
            off, on = copy.deepcopy(calibrated), copy.deepcopy(calibrated)
            iao.freeze_inference(off, handoff=False, int8=i8)
            iao.freeze_inference(on, handoff=True, int8=i8)
            sts = {"handoff=False": H.InferStepper(off, graph=True), "handoff=True": H.InferStepper(on, graph=True)}
            for st in sts.values():
                for _ in range(4):
                    st.step(x)
                assert st.graph is not None, st.graph_error
            times = {k: [] for k in sts}
            for _ in range(args.rounds):
                for k, st in sts.items():
                    times[k].append(_time(st, x, args.reps))
            same = torch.equal(sts["handoff=True"].step(x).clone(), sts["handoff=False"].step(x).clone())
            u, f = statistics.median(times["handoff=False"]), statistics.median(times["handoff=True"])
            lines.append(f"{name} batch {B}: handoff=False {u:.3f} ms ({B / u:.1f} k img/s), handoff=True {f:.3f} ms "
                         f"({B / f:.1f} k img/s), x{u / f:.2f}; logits bitwise equal: {same}; rounds handoff=False "
                         f"{[round(t, 3) for t in times['handoff=False']]} handoff=True "
                         f"{[round(t, 3) for t in times['handoff=True']]}")
            print(lines[-1], flush=True)
            start = len(lines)
            for k, m in (("handoff=False", off), ("handoff=True", on)):
                lines.append(f"  {name} {k}, batch {B}, device us per forward (torch.profiler, eager):")
                for kname, (t, n) in _kernel_table(m, x)[:16]:
                    lines.append(f"    {t:9.1f} us  x{n:<3d} {kname[:110]}")
            print("\n".join(lines[start:]), flush=True)
            del sts, off, on
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
