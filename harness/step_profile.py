"""Per-kernel split of the headline QAT step (NIN-GC wbwtab W3/A2, batch 256) under torch.profiler.

    python -m harness.step_profile --out DIR [--steps 5] [--warmup 5] [--batch 256]

Runs the bench model's step eagerly (no CUDA graph, so that the profiler sees every launch) in a process of its own and
writes DIR/step_profile.json and DIR/step_profile.txt: per kernel name the launches and device microseconds per step and,
for the fused BatchNorm producers and the batch-statistics kernel, the bytes each launch has to move (computed from the
shapes of the BatchNormBinarize2d inputs seen in the profiled steps) and the achieved GB/s.  Prints the card's name and
power limit with the table.  The profiler slows the host, not the kernels: end-to-end step times come from bench.py."""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from harness import train as H  # noqa: E402

HEADLINE = "nin_gc_wbwtab_w3a2"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError) as e:
        return f"unknown ({type(e).__name__})"


def producer_bytes(rec, terms_dy):
    """{kernel base name: bytes one launch moves} for one BatchNormBinarize2d call.  x is read at 4 bytes per element, or
    2 when it arrives as the producing conv's int16 codes; pass bits are 1/8 byte per element; the bf16 operand planes 2
    bytes per element and piece.  The pooled reduce pass reads x at the window winners only, but those are spread over
    every 32-byte sector of x: it is counted as a full read."""
    n, xb, pooled, plane_only, pk_conv = rec["n"], rec["xb"], rec["pool2"], rec["plane_only"], rec["pk_conv"]
    bits = n / 8
    out = {"channel_stats_kernel": n * xb}
    if pooled:
        out["bn_sign_pool_fwd_kernel"] = n * xb + n + n / 4 + bits                 # x, pooled +-1 fp32, arg-max bytes, bits
        out["bn_sign_pool_bwd_reduce_kernel"] = n * xb + n + n / 4 + bits          # x, pooled gradient, arg-max, bits
        if pk_conv:
            out["bn_sign_pool_bwd_pack_kernel"] = n * xb + n + n / 4 + bits + 2 * n * terms_dy
        else:
            out["bn_sign_pool_bwd_apply_kernel"] = n * xb + n + n / 4 + bits + 4 * n
    else:
        out["bn_sign_packed_fwd_kernel"] = n * xb + 2 * n + bits + (0 if plane_only else 4 * n)
        out["bn_sign_bwd_reduce_kernel"] = n * xb + 4 * n + bits                   # x, g, bits
        if pk_conv:
            out["bn_sign_bwd_pack_kernel"] = n * xb + 4 * n + bits + 2 * n * terms_dy
        else:
            out["bn_sign_bwd_apply_kernel"] = n * xb + 4 * n + bits + 4 * n
    return out


def base_name(kernel):
    """'void pk::bn_sign_bwd_pack_kernel<4, short>(...)' -> 'bn_sign_bwd_pack_kernel'"""
    head = kernel.split("(")[0]
    head = re.sub(r"<.*$", "", head)
    return head.split("::")[-1].split(" ")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_profile: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    from micronet_b200 import _lib as L
    from micronet_b200.fused import BatchNormBinarize2d
    w = H.WORKLOADS[HEADLINE]
    dev = torch.device("cuda:0")
    model = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w.get("engine_extra", {})).to(dev)
    stepper = H.QatStepper(model, lr=0.01, wd=w["wd"], flat=True, graph=False)
    batches = [H.synthetic_batch(args.batch, w["hw"], seed=100 + i, device=dev) for i in range(2)]
    for i in range(args.warmup):
        stepper.step(*batches[i % 2])
    torch.cuda.synchronize()

    calls = []

    def hook(mod, inp):
        x = inp[0]
        calls.append({"n": x.numel(), "xb": 2 if getattr(x, "_mnb_codes", None) is not None else 4,
                      "pool2": bool(mod.pool2), "plane_only": bool(mod.plane_only) and not mod.pool2,
                      "pk_conv": getattr(x, "_mnb_pk_conv", None) is not None})

    handles = [m.register_forward_pre_hook(hook) for m in model.modules() if isinstance(m, BatchNormBinarize2d)]
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(args.steps):
            stepper.step(*batches[i % 2])
        torch.cuda.synchronize()
    for h in handles:
        h.remove()

    terms_dy = L.PK_TERMS_BWD
    want = {}
    for rec in calls:
        for k, b in producer_bytes(rec, terms_dy).items():
            want[k] = want.get(k, 0.0) + b
    kern = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = kern.setdefault(e.name, {"launches": 0, "us": 0.0})
        d["launches"] += 1
        d["us"] += e.device_time
    rows, total_us = [], sum(d["us"] for d in kern.values()) / args.steps
    for name, d in kern.items():
        row = {"kernel": name, "base": base_name(name), "launches_per_step": d["launches"] / args.steps,
               "us_per_step": d["us"] / args.steps}
        rows.append(row)
    # bytes of a producer kernel: shared out over the template instances of one base name in proportion to their launches
    by_base = {}
    for r in rows:
        by_base.setdefault(r["base"], []).append(r)
    for base, rs in by_base.items():
        if base not in want:
            continue
        launches = sum(r["launches_per_step"] for r in rs)
        bytes_step = want[base] / args.steps
        us = sum(r["us_per_step"] for r in rs)
        for r in rs:
            r["bytes_per_launch"] = bytes_step / launches
        rs[0]["group_bytes_per_step"] = bytes_step
        rs[0]["group_GBps"] = bytes_step / (us * 1e-6) / 1e9
    rows.sort(key=lambda r: -r["us_per_step"])
    res = {"card": card(), "workload": HEADLINE, "batch": args.batch, "steps": args.steps,
           "device_us_per_step": total_us, "kernels": rows}
    with open(os.path.join(args.out, "step_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    lines = [f"card: {res['card']}", f"{HEADLINE}, batch {args.batch}, eager step, {args.steps} profiled steps; "
             f"device time per step {total_us / 1e3:.3f} ms (sum of kernel times)", "",
             f"{'us/step':>9} {'share':>6} {'launch':>6} {'MB/launch':>9} {'GB/s':>7}  kernel"]
    for r in rows:
        mb = f"{r['bytes_per_launch'] / 1e6:9.1f}" if "bytes_per_launch" in r else " " * 9
        gbs = f"{r['group_GBps']:7.0f}" if "group_GBps" in r else " " * 7
        lines.append(f"{r['us_per_step']:9.1f} {r['us_per_step'] / total_us:6.1%} {r['launches_per_step']:6.1f} {mb} {gbs}  "
                     f"{r['kernel'][:110]}")
    txt = "\n".join(lines)
    with open(os.path.join(args.out, "step_profile.txt"), "w") as f:
        f.write(txt + "\n")
    print(txt)


if __name__ == "__main__":
    main()
