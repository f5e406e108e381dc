"""Time mnb_pk_conv_codes / mnb_pk_conv (all pk layers) against mnb_pk_gc3_conv_codes / mnb_pk_gc3_conv (narrow grouped 3x3
layers): the forward (int16 codes, as the QAT step writes them) and the data gradient of the two grouped 3x3 layers of the
NIN-GC bench model, batch 256, with the operands the step gives them: x as one +-1 plane, integer weight levels, dy in two
bf16 pieces.

    python -m harness.gc3_probe [--iters 50] [--rounds 5]

Old and new run alternately, `iters` launches per timed window with CUDA events, over 4 rotating operand sets; the median
window per launch is reported with the card name and power limit, and whether the two results are bit-identical."""
import argparse
import json

import torch

from harness.wgrad_taps_probe import card
from micronet_b200 import _lib as L, pk as PK

SHAPES = {"g16 256->512 @16": (256, 256, 16, 16, 512, 16), "g32 512->1024 @8": (256, 512, 8, 8, 1024, 32)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "layers": {}}
    total = {"old": 0.0, "new": 0.0}
    for name, (B, Cc, H, W, K, G) in SHAPES.items():
        sh = L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, 1, 1, 1, 1, G)
        g = torch.Generator().manual_seed(7)
        ops = []
        for _ in range(4):
            x = torch.randint(0, 2, (B, Cc, H, W), generator=g).float().mul_(2).sub_(1).to(dev)
            dy = torch.randn(B, K, H, W, generator=g).to(dev)
            ops.append((PK.pack_act(x, None, 1)[0], PK.pack_act(dy, None, 2)[0]))
        w = torch.randint(-1, 2, (K, Cc // G, 3, 3), generator=g).to(torch.int16).to(dev)
        w_scale = (torch.rand(K, generator=g) + 0.5).to(dev)
        wf = PK.pack_weight(sh, 0, 1, 1, w_int=w)
        wd = PK.pack_weight(sh, 1, 2, 1, w_int=w, kzero=w_scale)
        res = {k: (torch.empty(B, K, H, W, dtype=torch.int16, device=dev), torch.empty(2 * K, device=dev),
                   torch.empty(B, Cc, H, W, device=dev)) for k in ("old", "new")}
        launches = {
            "fwd": {"old": lambda i, r: PK.conv_codes(sh, ops[i][0], wf, r[0], r[1], n_scale=w_scale),
                    "new": lambda i, r: PK.gc3_conv_codes(sh, ops[i][0], wf, r[0], r[1], n_scale=w_scale)},
            "dgrad": {"old": lambda i, r: PK.conv(sh, 1, ops[i][1], 2, wd, 1, r[2]),
                      "new": lambda i, r: PK.gc3_conv(sh, 1, ops[i][1], 2, wd, 1, r[2])},
        }
        layer = {"plans": {kind: {k: v for k, v in PK.gc3_plan(sh, *m).items() if k != "chain"}
                           for kind, m in (("fwd", (0, 1, 1)), ("dgrad", (1, 2, 1)))}}
        for kind, fns in launches.items():
            def window(k):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(args.iters):
                    L.check(fns[k](i % 4, res[k]), f"{kind} {k}")
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
            idx = (0, 1) if kind == "fwd" else (2,)
            same = all(torch.equal(res["old"][j].view(torch.int16) if j == 0 else res["old"][j].view(torch.int32),
                                   res["new"][j].view(torch.int16) if j == 0 else res["new"][j].view(torch.int32)) for j in idx)
            for k in med:
                total[k] += med[k]
            layer[kind] = {"old_us": med["old"], "new_us": med["new"], "speedup": med["old"] / med["new"],
                           "old_windows_us": t["old"], "new_windows_us": t["new"], "bit_identical": same}
        out["layers"][name] = layer
    out["four_launches_us"] = {"old": total["old"], "new": total["new"]}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
