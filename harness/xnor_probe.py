"""XNOR-popcount forward (csrc/mnb_xnor.cu) against the packed-operand tensor-core forward (csrc/mnb_pk.cu) on the wbwtab
layers of NIN-GC at the bench batch: CUDA events around each kernel, inputs rotated over 4 buffers.  The table this prints
is the evidence for the choice in functional._xnor_forward (north_star: the XNOR kernel is "picked when ncu shows it beating the
tensor-core path").

    python -m harness.xnor_probe [--batch 256] [--json out.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name, C, H, W, K, R, pad, groups   (harness/models.py NINGC, reference models/nin_gc.py:62-147)
LAYERS = [
    ("1x1 g2 256->256 @32", 256, 32, 32, 256, 1, 0, 2),
    ("3x3 g16 256->512 @16", 256, 16, 16, 512, 3, 1, 16),
    ("1x1 g4 512->512 @16", 512, 16, 16, 512, 1, 0, 4),
    ("3x3 g32 512->1024 @8", 512, 8, 8, 1024, 3, 1, 32),
    ("1x1 g8 1024->1024 @8", 1024, 8, 8, 1024, 1, 0, 8),
]


ITERS = 20


def timeit(fn, iters=None):
    iters = iters or ITERS
    fn(0)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--only", default=None, help="substring of the layer name (ncu target: one layer)")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from micronet_b200 import _lib as L, pk as PK, xnor as X
    dev = torch.device("cuda:0")
    pk_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    hbm = json.load(open(pk_path))["hbm_gbs"] if os.path.exists(pk_path) else 6650.0
    B, nb, rows = args.batch, 4, []
    global ITERS
    ITERS = args.iters
    for name, Cc, H, W, K, R, pad, G in LAYERS:
        if args.only and args.only not in name:
            continue
        sh = L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, pad, pad, 1, 1, G)
        xs = [torch.where(torch.randn(B, Cc, H, W, device=dev) < 0, -1.0, 1.0) for _ in range(nb)]
        ys = [torch.empty(B, K, H, W, device=dev) for _ in range(nb)]
        w_int = torch.randint(-1, 2, (K, Cc // G, R, R), dtype=torch.int16, device=dev)
        alpha = torch.rand(K, device=dev) * 0.05 + 0.01
        bias = torch.randn(K, device=dev)
        rec = {"layer": name, "out_MB": B * K * H * W * 4 / 1e6,
               "roof_us_fp32_surface": (4.0 * (B * Cc * H * W + B * K * H * W)) / (hbm * 1e9) * 1e6,
               "roof_us_out_only": (4.0 * B * K * H * W) / (hbm * 1e9) * 1e6}
        bits = [X.pack_act(x, G) for x in xs]
        ximg = X.pack_weight(sh, w_int)
        rec["xnor_conv"] = timeit(lambda i: L.check(X.conv(sh, bits[i % nb], ximg, ys[i % nb], alpha=alpha, bias=bias), "x"))
        rec["xnor_pack_act"] = timeit(lambda i: X.pack_act(xs[i % nb], G))
        rec["xnor_pack_w"] = timeit(lambda i: X.pack_weight(sh, w_int))
        planes = [PK.pack_act(x, None, 1)[0] for x in xs]
        pimg = PK.pack_weight(sh, 0, 1, 1, w_int=w_int)
        rec["tc_conv"] = timeit(lambda i: L.check(PK.conv(sh, 0, planes[i % nb], 1, pimg, 1, ys[i % nb], n_scale=alpha, bias=bias), "p"))
        rec["tc_pack_act"] = timeit(lambda i: PK.pack_act(xs[i % nb], None, 1))
        rec["tc_pack_w"] = timeit(lambda i: PK.pack_weight(sh, 0, 1, 1, w_int=w_int))
        L.tc_check()
        ya, yb = torch.empty_like(ys[0]), torch.empty_like(ys[0])
        L.check(X.conv(sh, bits[0], ximg, ya, alpha=alpha, bias=bias), "x")
        L.check(PK.conv(sh, 0, planes[0], 1, pimg, 1, yb, n_scale=alpha, bias=bias), "p")
        rec["bit_identical"] = bool(torch.equal(ya, yb))
        rec["winner_conv_only"] = "xnor" if rec["xnor_conv"] < rec["tc_conv"] else "tensor-core"
        rec["winner_with_pack"] = "xnor" if rec["xnor_conv"] + rec["xnor_pack_act"] < rec["tc_conv"] + rec["tc_pack_act"] else "tensor-core"
        rows.append(rec)
        print(json.dumps(rec))
        del xs, ys, bits, planes
        torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
