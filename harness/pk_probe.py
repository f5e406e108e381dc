"""Timing probe of the packed-operand kernels (csrc/mnb_pk.cu) on isolated layers: CUDA events around each kernel,
inputs rotated over 4 buffers (> L2 for the big layers), per-kernel roofline from SURVEY.md 8(d).

    python -m harness.pk_probe [--json out.json] [--batch 256]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name, C, H, W, K, R, stride, pad, groups
LAYERS = [
    ("resnet conv2_x 64->64 3x3 @32", 64, 32, 32, 64, 3, 1, 1, 1),
    ("resnet conv3_1 64->128 3x3 s2", 64, 32, 32, 128, 3, 2, 1, 1),
    ("resnet conv3_x 128->128 3x3 @16", 128, 16, 16, 128, 3, 1, 1, 1),
    ("resnet conv4_x 256->256 3x3 @8", 256, 8, 8, 256, 3, 1, 1, 1),
    ("resnet conv5_x 512->512 3x3 @4", 512, 4, 4, 512, 3, 1, 1, 1),
    ("nin 5x5 96->192 @16", 96, 16, 16, 192, 5, 1, 2, 1),
    ("ptq224 conv2_x 64->64 3x3 @224 (use --batch 64)", 64, 224, 224, 64, 3, 1, 1, 1),
    ("ptq224 conv3_x 128->128 3x3 @112 (use --batch 64)", 128, 112, 112, 128, 3, 1, 1, 1),
    ("nin-gc 1x1 g2 256->256 @32", 256, 32, 32, 256, 1, 1, 0, 2),
    ("nin-gc 3x3 g16 256->512 @16", 256, 16, 16, 512, 3, 1, 1, 16),
    ("nin-gc 1x1 g4 512->512 @16", 512, 16, 16, 512, 1, 1, 0, 4),
    ("nin-gc 3x3 g32 512->1024 @8", 512, 8, 8, 1024, 3, 1, 1, 32),
    ("nin-gc 1x1 g8 1024->1024 @8", 1024, 8, 8, 1024, 1, 1, 0, 8),
]


def timeit(fn, iters=10):
    fn()
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
    ap.add_argument("--only", default=None)
    ap.add_argument("--compact", action="store_true", help="also print one short line per layer on stderr")
    args = ap.parse_args()
    from micronet_b200 import _lib as L, pk as PK
    dev = torch.device("cuda:0")
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}
    hbm, tfl = peaks["hbm_gbs"], peaks["bf16_tflops"]
    rows = []
    B = args.batch
    for name, Cc, H, W, K, R, st, pad, G in LAYERS:
        if args.only and args.only not in name:
            continue
        sh = L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)
        P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
        flops = 2.0 * B * K * P * Q * (Cc // G) * R * R
        nbytes = 4.0 * (B * Cc * H * W + B * K * P * Q) + 4.0 * K * (Cc // G) * R * R
        roof = max(flops / (tfl * 1e12), nbytes / (hbm * 1e9)) * 1e6
        nb = 4
        xs = [torch.randn(B, Cc, H, W, device=dev) for _ in range(nb)]
        dys = [torch.randn(B, K, P, Q, device=dev) for _ in range(nb)]
        w_int = torch.randint(-127, 128, (K, Cc // G, R, R), dtype=torch.int16, device=dev)
        w_f = torch.randn(K, Cc // G, R, R, device=dev) * 0.05
        w_scale = torch.rand(K, device=dev) * 0.01 + 0.001
        y = torch.empty(B, K, P, Q, device=dev)
        dx = torch.empty(B, Cc, H, W, device=dev)
        dw = torch.empty(K, Cc // G, R, R, device=dev)
        from micronet_b200 import functional as F_
        spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
        qp = spec.struct()
        split = st == 2
        rec = {"layer": name, "roof_us": roof, "GFLOP": flops / 1e9, "MB": nbytes / 1e6}
        rec["pack_x_quant"] = timeit(lambda i=0: PK.pack_act(xs[i % nb], qp, 1, phase_split=split, want_bits=True))
        rec["pack_x_raw3"] = timeit(lambda i=0: PK.pack_act(xs[i % nb], None, 3, phase_split=split))
        rec["pack_dy3"] = timeit(lambda i=0: PK.pack_act(dys[i % nb], None, 3, ch_scale=w_scale))
        xq = [PK.pack_act(x, qp, 1, phase_split=split)[0] for x in xs]
        xr = [PK.pack_act(x, None, 3, phase_split=split)[0] for x in xs]
        dyp = [PK.pack_act(d, None, 3)[0] for d in dys]
        rec["pack_w"] = timeit(lambda i=0: PK.pack_weight(sh, 0, 1, 1, w_int=w_int))
        img11 = PK.pack_weight(sh, 0, 1, 1, w_int=w_int)
        img33 = PK.pack_weight(sh, 0, 3, 3, w_f32=w_f)
        imgd = PK.pack_weight(sh, 1, 3, 1, w_int=w_int)
        imgd3 = PK.pack_weight(sh, 1, 3, 3, w_f32=w_f)
        rec["fwd_1x1"] = timeit(lambda i=0: L.check(PK.conv(sh, 0, xq[i % nb], 1, img11, 1, y, n_scale=w_scale), "c"))
        rec["fwd_3x3"] = timeit(lambda i=0: L.check(PK.conv(sh, 0, xr[i % nb], 3, img33, 3, y), "c"))
        rec["dgrad_3x1"] = timeit(lambda i=0: L.check(PK.conv(sh, 1, dyp[i % nb], 3, imgd, 1, dx), "c"))
        rec["dgrad_3x3"] = timeit(lambda i=0: L.check(PK.conv(sh, 1, dyp[i % nb], 3, imgd3, 3, dx), "c"))
        # what the QAT backward actually runs since round 2 (L.PK_TERMS_BWD = 2 pieces)
        xr2 = [PK.pack_act(x, None, 2, phase_split=split)[0] for x in xs]
        dyp2 = [PK.pack_act(d, None, 2)[0] for d in dys]
        imgd2 = PK.pack_weight(sh, 1, 2, 2, w_f32=w_f)
        imgd21 = PK.pack_weight(sh, 1, 2, 1, w_int=w_int)
        rec["dgrad_2x1"] = timeit(lambda i=0: L.check(PK.conv(sh, 1, dyp2[i % nb], 2, imgd21, 1, dx), "c"))
        rec["dgrad_2x2"] = timeit(lambda i=0: L.check(PK.conv(sh, 1, dyp2[i % nb], 2, imgd2, 2, dx), "c"))
        if PK.wgrad_supported(sh, 2, 1):
            rec["wgrad_2x1"] = timeit(lambda i=0: L.check(PK.wgrad(sh, dyp2[i % nb], 2, xq[i % nb], 1, dw), "w"))
            rec["wgrad_2x2"] = timeit(lambda i=0: L.check(PK.wgrad(sh, dyp2[i % nb], 2, xr2[i % nb], 2, dw), "w"))
        del xr2, dyp2
        if PK.wgrad_supported(sh, 3, 1):
            rec["wgrad_3x1"] = timeit(lambda i=0: L.check(PK.wgrad(sh, dyp[i % nb], 3, xq[i % nb], 1, dw), "w"))
            rec["wgrad_3x3"] = timeit(lambda i=0: L.check(PK.wgrad(sh, dyp[i % nb], 3, xr[i % nb], 3, dw), "w"))
        plan = (C.c_int32 * 16)()
        L.load().mnb_pk_conv_plan(C.byref(sh), 0, 1, 1, plan)
        rec["plan_fwd"] = dict(zip("Nt ntiles MT CC chunks nstage smem acc TH TB BW n_mtiles n_items ny".split(), list(plan)[2:]))
        L.tc_check()
        rows.append(rec)
        print(json.dumps(rec))
        if args.compact:
            print("  " + name + ": " + " ".join(f"{k}={v:.0f}" for k, v in rec.items() if isinstance(v, float) and k not in ("GFLOP", "MB")),
                  file=sys.stderr)
        del xs, dys, xq, xr, dyp
        torch.cuda.empty_cache()
    if args.json:
        json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
