"""Time mnb_pk_bwd1x1 (data and weight gradient in one pass over dy) against mnb_pk_conv (data gradient) followed by
mnb_pk_wgrad at the 1x1 grouped layers of the NIN-GC bench model, batch 256, with the operands the wbwtab QAT step gives
them: dy in two bf16 pieces, x as one +-1 plane, ternary weights as one piece, the STE mask applied by the producer.

    python -m harness.pk_bwd1x1_probe [--iters 50] [--rounds 5]

The two paths run alternately, `iters` launches per timed window with CUDA events, over 4 rotating operand sets; the
median window per path is reported in microseconds and as bytes-based GB/s (each path's compulsory HBM traffic: dy, x
and the weight image read, dx written, dW partials written and read back), with the card name and power limit, and
whether the two results are byte-equal."""
import argparse
import json

import torch

from harness.wgrad_taps_probe import card
from micronet_b200 import _lib as L, pk as PK

# B, C, H, W, K, groups: L1 / L2, L4 / L5, L7
SHAPES = {"L1/L2 256->256 g2 @32": (256, 256, 32, 32, 256, 2), "L4/L5 512->512 g4 @16": (256, 512, 16, 16, 512, 4),
          "L7 1024->1024 g8 @8": (256, 1024, 8, 8, 1024, 8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "layers": {}}
    for name, (B, Cc, H, W, K, G) in SHAPES.items():
        sh = L.ConvShape(B, Cc, H, W, K, 1, 1, 1, 1, 0, 0, 1, 1, G)
        plan = PK.bwd1x1_plan(sh, 2, 1, 1)
        g = torch.Generator().manual_seed(7)
        ops = []
        for _ in range(4):
            dy = torch.randn(B, K, H, W, generator=g).to(dev)
            x = torch.randint(0, 2, (B, Cc, H, W), generator=g).float().mul_(2).sub_(1).to(dev)
            w_int = torch.randint(-1, 2, (K, Cc // G, 1, 1), generator=g).to(torch.int16).to(dev)
            ops.append((PK.pack_act(dy, None, 2, groups=G)[0], PK.pack_act(x, None, 1, groups=G)[0],
                        PK.pack_weight(sh, 1, 2, 1, w_int=w_int)))
        res = {k: (torch.empty(B, Cc, H, W, device=dev), torch.empty(K, Cc // G, 1, 1, device=dev)) for k in ("sep", "fused")}

        def sep(dy_pk, x_pk, w_img, dx, dw):
            L.check(PK.conv(sh, 1, dy_pk, 2, w_img, 1, dx, a_scale_const=0.25), "pk_conv dgrad")
            L.check(PK.wgrad(sh, dy_pk, 2, x_pk, 1, dw), "pk_wgrad")

        def fused(dy_pk, x_pk, w_img, dx, dw):
            L.check(PK.bwd1x1(sh, dy_pk, 2, x_pk, 1, w_img, 1, dx, dw, a_scale_const=0.25), "pk_bwd1x1")

        fns = {"sep": sep, "fused": fused}

        def window(k):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.iters):
                fns[k](*ops[i % 4], *res[k])
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) * 1e3 / args.iters

        for k in fns:   # warm-up
            window(k)
        t = {k: [] for k in fns}
        for _ in range(args.rounds):
            for k in fns:
                t[k].append(window(k))
        L.tc_check()
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        n_out = B * K * H * W
        dy_b, x_b, dx_b = n_out * 4, B * Cc * H * W * 2, B * Cc * H * W * 4
        w_b = ops[0][2].numel()
        part_b = plan["scratch_bytes"] * 2
        bytes_ = {"sep": 2 * dy_b + x_b + w_b + dx_b + part_b, "fused": dy_b + x_b + w_b + dx_b + part_b}
        same = all(torch.equal(res["sep"][i].view(torch.int32), res["fused"][i].view(torch.int32)) for i in range(2))
        out["layers"][name] = {
            "sep_us": med["sep"], "fused_us": med["fused"], "speedup": med["sep"] / med["fused"],
            "sep_GBps": bytes_["sep"] / med["sep"] * 1e-3, "fused_GBps": bytes_["fused"] / med["fused"] * 1e-3,
            "sep_bytes": bytes_["sep"], "fused_bytes": bytes_["fused"],
            "sep_windows_us": t["sep"], "fused_windows_us": t["fused"], "byte_equal": same, "plan": plan}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
