"""Binary tensor-core convolution (csrc/mnb_b1.cu) per launch against the kernels a layer runs without it.

    python -m harness.b1_probe [--batch 256] [--reps 50] [--out FILE]

At batch 256 on synthetic +-1 activations and ternary weights, CUDA events around ``reps`` back-to-back launches (after a
warm-up), median of 5 rounds, microseconds per launch:
* NIN's seven binarized layers (models/nin.py): b1 forward (fp32 out), b1 post (BatchNorm + sign into the next layer's b1
  plane), and the packed-operand tensor-core forward (bf16 +-1 plane, fp32 out) that the layer runs un-frozen;
* the whole NIN W3/A2 eval forward (G2 and G1) un-frozen against frozen at batch 256 and 1024, CUDA-graph replays
  alternated, with logits equality (G2) or the largest logit difference (G1);
* NIN-GC's five 1x1 layers: b1 post, XNOR post (bit plane out) and the packed-operand forward - evidence for a later choice,
  these layers stay on the XNOR kernel.
The card, its power limit and SM clock come from a read-only nvidia-smi query.  Every timed output is checked once against
the packed-operand forward (fp32) or the XNOR epilogue (bit plane) before timing."""
from __future__ import annotations

import argparse
import statistics

import torch

from harness.wbwtab_infer_probe import _card

# C, H, K, R, pad, groups
NIN = [("L1", 192, 32, 160, 1, 0, 1), ("L2", 160, 32, 96, 1, 0, 1), ("L3", 96, 16, 192, 5, 2, 1),
       ("L4", 192, 16, 192, 1, 0, 1), ("L5", 192, 16, 192, 1, 0, 1), ("L6", 192, 8, 192, 3, 1, 1), ("L7", 192, 8, 192, 1, 0, 1)]
NINGC = [("L1", 256, 32, 256, 1, 0, 2), ("L2", 256, 32, 256, 1, 0, 2), ("L4", 512, 16, 512, 1, 0, 4),
         ("L5", 512, 16, 512, 1, 0, 4), ("L7", 1024, 8, 1024, 1, 0, 8)]


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        rounds.append(a.elapsed_time(b) * 1000.0 / reps)
    return statistics.median(rounds)


def layer(batch, C, H, K, R, pad, G, reps, with_xnor):
    from micronet_b200 import _lib as L, b1 as B1, pk as PK, xnor as X
    dev = "cuda:0"
    g = torch.Generator().manual_seed(C + K + R)
    x = torch.where(torch.randn(batch, C, H, H, generator=g) < 0, -1.0, 1.0).to(dev)
    w = torch.randint(-1, 2, (K, C // G, R, R), generator=g).to(torch.int16).to(dev)
    alpha = (torch.rand(K, generator=g) * 0.05 + 0.01).to(dev)
    bias = torch.randn(K, generator=g).to(dev)
    bn = [torch.randn(K, generator=g).to(dev), (torch.rand(K, generator=g) + 0.5).to(dev), torch.randn(K, generator=g).to(dev),
          torch.randn(K, generator=g).to(dev)]
    sh = L.ConvShape(batch, C, H, H, K, R, R, 1, 1, pad, pad, 1, 1, G)
    P = H + 2 * pad - R + 1
    plane, img = B1.pack_act(x, G), B1.pack_weight(sh, w)
    y = torch.empty(batch, K, P, P, device=dev)
    post = X.post_struct(L.XNOR_B1_PLANE, G, 1, False, bn)
    out = B1.empty_plane(B1.post_bytes(sh, post), dev)
    pk_plane = PK.pack_act(x, None, 1, groups=G)[0]
    pk_img = PK.pack_weight(sh, 0, 1, 1, w_int=w)
    y_pk = torch.empty_like(y)
    L.check(B1.conv(sh, plane, img, y, alpha=alpha, bias=bias), "b1 conv")
    L.check(PK.conv(sh, 0, pk_plane, 1, pk_img, 1, y_pk, n_scale=alpha, bias=bias), "pk conv")
    assert torch.equal(y, y_pk)
    row = {
        "b1_fwd": _time(lambda: B1.conv(sh, plane, img, y, alpha=alpha, bias=bias), reps),
        "b1_post": _time(lambda: B1.conv_post(sh, plane, img, post, out, alpha=alpha, bias=bias), reps),
        "pk_fwd": _time(lambda: PK.conv(sh, 0, pk_plane, 1, pk_img, 1, y_pk, n_scale=alpha, bias=bias), reps),
    }
    if with_xnor:
        xpost = X.post_struct(L.XNOR_BITS, G, 1, False, bn)
        bits, ximg = X.pack_act(x, G), X.pack_weight(sh, w)
        xo = torch.empty(X.post_bytes(sh, xpost) // 4, dtype=torch.int32, device=dev)
        bo = torch.empty_like(xo)
        L.check(X.conv_post(sh, bits, ximg, xpost, xo, alpha=alpha, bias=bias), "xnor conv_post")
        L.check(B1.conv_post(sh, plane, img, xpost, bo, alpha=alpha, bias=bias), "b1 conv_post")
        assert torch.equal(xo, bo)
        row["xnor_post"] = _time(lambda: X.conv_post(sh, bits, ximg, xpost, xo, alpha=alpha, bias=bias), reps)
    L.tc_check()
    return row


def whole_nin(batches, rounds=5, reps=20):
    """NIN W3/A2 eval forward, G2 and G1, un-frozen against frozen: CUDA-graph replays alternated, median round"""
    import micronet_b200 as E
    from harness import train as H
    from tests.test_gpu_wbwtab_frozen_nin import _model
    lines = []
    for graph in ("G2", "G1"):
        ref_m, fz = _model("nin", graph, 3), _model("nin", graph, 3)
        E.wbwtab.freeze_inference(fz)
        for b in batches:
            x, _ = H.synthetic_batch(b, 32, seed=5, device="cuda:0")
            sa, sb = H.InferStepper(ref_m, graph=True), H.InferStepper(fz, graph=True)
            with torch.no_grad():
                ya, yb = sa.step(x), sb.step(x)
                # G2 is bit-identical to its un-frozen forward; G1's un-frozen convs multiply the fp32 weights alpha * level
                # on another kernel, so the frozen logits equal the per-layer composition instead (the GPU tests pin both)
                equal = torch.equal(ya, yb) if graph == "G2" else f"max |d| {float((ya - yb).abs().max()):.2e}"
                ta, tb = [], []
                for _ in range(rounds):
                    for st, t in ((sa, ta), (sb, tb)):
                        t.append(_time(lambda: st.step(x), reps))
            lines.append(f"NIN {graph} batch {b}: un-frozen {statistics.median(ta):8.1f} us  frozen {statistics.median(tb):8.1f} us"
                         f"  logits equal {equal}  (graphs {sa.graph is not None}/{sb.graph is not None})")
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = [f"card: {_card()}", f"batch {a.batch}, us per launch (median of 5 rounds x {a.reps})"]
    for model, layers, with_xnor in (("NIN", NIN, False), ("NIN-GC", NINGC, True)):
        for name, C, H, K, R, pad, G in layers:
            row = layer(a.batch, C, H, K, R, pad, G, a.reps, with_xnor)
            cells = "  ".join(f"{k} {v:8.1f}" for k, v in row.items())
            lines.append(f"{model:6s} {name} {C}->{K} {R}x{R} g{G} {H}x{H}:  {cells}")
    lines += whole_nin((256, 1024))
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
