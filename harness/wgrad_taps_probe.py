"""Time mnb_pk_wgrad (all pk layers) against mnb_pk_wgrad_taps (narrow grouped 3x3 layers) at the two grouped 3x3 layers
of the NIN-GC bench model, batch 256, the operands the QAT step gives them: dy in two bf16 pieces, x as one +-1 plane.

    python -m harness.wgrad_taps_probe [--iters 50] [--rounds 5]

The two kernels run alternately, `iters` launches per timed window with CUDA events, over 4 rotating operand sets; the
median window per kernel is reported with the card name and power limit, and the largest difference of the two results
relative to max |dw|."""
import argparse
import json
import subprocess

import torch

from micronet_b200 import _lib as L, pk as PK

SHAPES = {"g16 256->512 @16": (256, 256, 16, 16, 512, 16), "g32 512->1024 @8": (256, 512, 8, 8, 1024, 32)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # the timing does not depend on it
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {type(e).__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "layers": {}}
    for name, (B, Cc, H, W, K, G) in SHAPES.items():
        sh = L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, 1, 1, 1, 1, G)
        g = torch.Generator().manual_seed(7)
        ops = []
        for _ in range(4):
            dy = torch.randn(B, K, H, W, generator=g).to(dev)
            x = torch.randint(0, 2, (B, Cc, H, W), generator=g).float().mul_(2).sub_(1).to(dev)
            ops.append((PK.pack_act(dy, None, 2)[0], PK.pack_act(x, None, 1)[0]))
        dws = {k: torch.empty(K, Cc // G, 3, 3, device=dev) for k in ("old", "new")}
        fns = {"old": PK.wgrad, "new": PK.wgrad_taps}

        def window(k):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.iters):
                dy_pk, x_pk = ops[i % 4]
                L.check(fns[k](sh, dy_pk, 2, x_pk, 1, dws[k]), k)
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) * 1e3 / args.iters

        for k in fns:   # warm-up
            window(k)
        t = {"old": [], "new": []}
        for _ in range(args.rounds):
            for k in fns:
                t[k].append(window(k))
        L.tc_check()
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        diff = ((dws["new"] - dws["old"]).abs().max() / dws["old"].abs().max()).item()
        out["layers"][name] = {"old_us": med["old"], "new_us": med["new"], "speedup": med["old"] / med["new"],
                               "old_windows_us": t["old"], "new_windows_us": t["new"], "plan": PK.wgrad_taps_plan(sh, 2, 1),
                               "max_rel_diff": diff}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
