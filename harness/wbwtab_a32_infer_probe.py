"""Frozen wbwtab inference with fp32 activations on term planes (wbwtab.freeze_inference on ``prepare(A=32, W=2|3)``) against
the un-frozen eval forward.

    python -m harness.wbwtab_a32_infer_probe [--batch 256] [--rounds 5] [--reps 20] [--out FILE]

Workloads: NIN and NIN-GC at W=2 (binary) and W=3 (ternary) weights with A=32 (fp32 activations, the ReLU of WB:79-94) in
eval mode on synthetic 3x32x32 inputs, with non-trivial BatchNorm statistics.  Un-frozen and frozen models are each captured
into a CUDA graph (harness.train.InferStepper) and replayed alternately over several rounds; a round times ``reps`` replays
with CUDA events, the median round is reported.  The frozen logits of the timed model are compared bitwise with the
block-by-block composition of harness/wbwtab_a32_compose.py (cuDNN in deterministic mode for the stem and head convs, in
both graphs).  A per-kernel table (device time per forward, torch.profiler) of one eager forward of each
follows, then each linked layer's two hand-off routes timed on its own shape: the conv epilogue writing the consumer's
term planes against the fp32 conv plus the stand-alone producer.  The card, its power limit and SM clock come from a
read-only nvidia-smi query."""
from __future__ import annotations

import argparse
import copy
import os
import statistics

import torch

from harness import train as H
from harness.wbwtab_infer_probe import _card, _kernel_table, _randomise_bn, _time

CONFIGS = [("NIN W2/A32", "nin", 2), ("NIN W3/A32", "nin", 3), ("NIN-GC W2/A32", "nin_gc", 2), ("NIN-GC W3/A32", "nin_gc", 3)]


def build(arch, W, dev):
    import micronet_b200 as E
    base = H.build_float_model(arch, seed=1)
    _randomise_bn(base, 7)
    return E.wbwtab.prepare(base, W=W, A=32).to(dev).eval()


def _event_us(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return 1000.0 * start.elapsed_time(end) / reps


def layer_routes(fz, x, rounds, reps):
    """per linked layer of a frozen model whose plan takes a consumer epilogue: us per launch of (a) the conv whose epilogue
    writes the consumer's term planes and (b) the fp32 conv followed by the stem producer (the route wbwtab takes for shuffled
    links), on the layer's own shape; median of ``rounds`` alternating rounds of ``reps`` launches"""
    from micronet_b200 import _lib as L, pk as PK, wbwtab
    from micronet_b200 import functional as F_
    convs = [c for c in fz.modules() if type(c) is wbwtab.QuantConv2d]
    shapes = {}
    def record(m, args):
        shapes.setdefault(m, tuple(args[0].shape))
    hooks = [c.register_forward_pre_hook(record) for c in convs]
    with torch.no_grad():
        fz(x)
    for h in hooks:
        h.remove()
    rows = []
    for i, c in enumerate(convs):
        rec = c.__dict__.get("_mnb_frozen")
        link = None if rec is None or rec["fmt"] != wbwtab.A32_PLANE else rec["link"]
        sh = F_._shape_struct(shapes[c], c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
        if link is None or link.split or PK.segmented(sh, 0, wbwtab.A32_TERMS, 1):
            continue
        w_int, alpha, bias, _ = wbwtab._frozen_conv_operands(c)
        plane, _ = PK.pack_act(torch.relu(torch.randn(shapes[c], device=x.device)), None, wbwtab.A32_TERMS, groups=c.groups)
        w_img = PK.pack_weight(sh, 0, wbwtab.A32_TERMS, 1, w_int=w_int)
        out_shape = (sh.batch, c.out_channels) + F_._out_hw(sh)
        y = torch.empty(out_shape, device=x.device)
        cplane = PK.terms_plane(*out_shape, wbwtab.A32_TERMS, x.device)
        bn = link.bn_tensors()

        def epi():
            L.check(PK.conv_post_terms(sh, plane, w_img, None, cplane, wbwtab.A32_TERMS, True, False, n_scale=alpha, bias=bias,
                                       bn=bn, shuffle_groups=link.sg), "conv_post_terms")

        def conv():
            L.check(PK.conv(sh, 0, plane, wbwtab.A32_TERMS, w_img, 1, y, n_scale=alpha, bias=bias), "pk_conv")

        def prod():
            L.check(PK.bn_relu_pack_terms(y, bn, True, link.sg, wbwtab.A32_TERMS, cplane), "bn_relu_pack_terms")
        t = {"epi": [], "conv": [], "prod": []}
        for fn in (epi, conv, prod):
            _event_us(fn, 3)
        for _ in range(rounds):
            for k, fn in (("epi", epi), ("conv", conv), ("prod", prod)):
                t[k].append(_event_us(fn, reps))
        e, cv, pr = (statistics.median(t[k]) for k in ("epi", "conv", "prod"))
        rows.append(f"    L{i + 1} {sh.in_c}->{sh.out_c} g{sh.groups} {sh.ker_h}x{sh.ker_w} {sh.in_h}x{sh.in_w} shuffle {link.sg}: "
                    f"epilogue {e:.1f} us, fp32 conv {cv:.1f} + producer {pr:.1f} = {cv + pr:.1f} us")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    from micronet_b200 import wbwtab
    from harness.wbwtab_a32_compose import composed
    dev = torch.device("cuda:0")
    B = args.batch
    lines = [f"card: {_card()}"]
    x, _ = H.synthetic_batch(B, 32, seed=3, device=dev)
    for name, arch, W in CONFIGS:
        un = build(arch, W, dev)
        fz, comp = copy.deepcopy(un), copy.deepcopy(un)
        with torch.no_grad():
            ref = composed(comp, x)[0]
        del comp
        wbwtab.freeze_inference(fz)
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
        rel = ((got - base).abs().max() / base.abs().max()).item()
        u, f = statistics.median(times["un-frozen"]), statistics.median(times["frozen"])
        lines.append(f"{name} batch {B}: un-frozen {u:.3f} ms ({B / u:.1f} k img/s), frozen {f:.3f} ms ({B / f:.1f} k img/s), "
                     f"x{u / f:.2f}; frozen logits bitwise equal to the block composition: {same}; max |frozen - un-frozen| / "
                     f"max |un-frozen| {rel:.3g}; rounds un-frozen {[round(t, 3) for t in times['un-frozen']]} frozen "
                     f"{[round(t, 3) for t in times['frozen']]}")
        print(lines[-1], flush=True)
        start = len(lines)
        for k, m in (("un-frozen", un), ("frozen", fz)):
            lines.append(f"  {name} {k}, batch {B}, device us per forward (torch.profiler, eager):")
            for kname, (t, n) in _kernel_table(m, x)[:16]:
                lines.append(f"    {t:9.1f} us  x{n:<3d} {kname[:110]}")
        lines.append(f"  {name}, batch {B}: term-plane hand-off per linked layer, epilogue against fp32 conv + stem producer:")
        lines += layer_routes(fz, x, args.rounds, args.reps)
        print("\n".join(lines[start:]), flush=True)
        del sts, un, fz
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
