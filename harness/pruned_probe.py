"""Speed of the channel-pruned NIN-GC (reference README cfg 154 162 144 304 320 320 608 584) on group-padded planes.

    python -m harness.pruned_probe --layers                      # per padded layer, batch 256: pk path vs generic kernels
    python -m harness.pruned_probe --step [--parent DIR]         # pruned QAT step (CUDA-graph replay), this tree vs DIR

--layers: forward, data gradient and weight gradient of every padded grouped layer with DoReFa 4-bit levels and 4-bit
weights, each as the engine runs it on the packed-operand family (operand packing included) against the generic CUDA-core
entry points called directly (with their activation quantizer pass); CUDA events, the two paths in alternating windows,
median of 5.  --step: wbwtab W3A2 (fuse_bn) and DoReFa W4A4 (fuse, and un-fused) QAT steps of the pruned model at batch 256
through
QatStepper(flat=True, graph=True), run in child processes alternating between this tree and the tree at --parent (a
checkout of another commit with its library built); the losses of the timed steps are compared, and a tree that cannot run
a graph is reported with its error.  Prints JSON lines; with
--out the same lines go to that file."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = [154, 162, 144, 304, 320, 320, 608, 584]


def _emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def _timeit(fns, iters, windows=5):
    """median ms per call of each fn over ``windows`` windows of ``iters`` calls, the fns alternating window by window"""
    import torch
    for fn in fns:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = [[] for _ in fns]
    for _ in range(windows):
        for i, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            res[i].append(a.elapsed_time(b) / iters)
    return [statistics.median(r) for r in res]


def layers(out, batch=256, iters=20):
    import torch
    from micronet_b200 import _lib as L, functional as F_, pk as PK
    lib = L.load()
    dev = torch.device("cuda:0")
    c = CFG
    convs = [("L1", c[0], 32, c[1], 1, 2), ("L2", c[1], 32, c[2], 1, 2), ("L3", c[2], 16, c[3], 3, 16),
             ("L4", c[3], 16, c[4], 1, 4), ("L6", c[5], 8, c[6], 3, 32), ("L7", c[6], 8, c[7], 1, 8)]
    g = torch.Generator().manual_seed(0)
    for name, cin, hw, cout, k, G in convs:
        pad = k // 2
        sh = L.ConvShape(batch, cin, hw, hw, cout, k, k, 1, 1, pad, pad, 1, 1, G)
        x = torch.rand(batch, cin, hw, hw, generator=g).to(dev)
        dy = torch.randn(batch, cout, hw, hw, generator=g).to(dev)
        w_int = torch.randint(-7, 8, (cout, cin // G, k, k), generator=g, dtype=torch.int16).to(dev)
        w_scale = (torch.rand(cout, generator=g) * 0.02 + 0.001).to(dev)
        wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
        spec = F_.ActSpec(L.ACT_DOREFA, bits=4)
        qp = spec.struct()
        y = torch.empty(batch, cout, hw, hw, device=dev)
        dx = torch.empty_like(x)
        dw = torch.empty_like(wq)
        a_scale, a_const = PK.act_scale(spec)
        x_pk, bits8 = PK.pack_act(x, qp, 1, want_bits=True, groups=G)
        img = PK.weight_image(sh, 1, 1, w_int=w_int)
        dy_pk, _ = PK.pack_act(dy, None, 2, ch_scale=w_scale, groups=G)
        codes, bits, _ = F_.act_quant_raw(x, spec, True, True, False)
        ops = F_._act_operands(spec, codes, x)
        ops.w_int, ops.w_scale = w_int.data_ptr(), w_scale.data_ptr()
        ws = torch.empty(max(int(lib.mnb_wgrad_scratch_bytes(C.byref(sh))), 4), dtype=torch.uint8, device=dev)
        wg_scale = F_._dorefa_scale_tensor(4, dev)

        def pk_fwd():
            xp, _ = PK.pack_act(x, qp, 1, want_bits=True, groups=G)
            L.check(PK.run_conv(sh, 0, xp, 1, img, 1, y, n_scale=w_scale, a_scale=a_scale, a_scale_const=a_const), "fwd")

        def gen_fwd():
            cd, _, _ = F_.act_quant_raw(x, spec, True, True, False)
            o = F_._act_operands(spec, cd, x)
            o.w_int, o.w_scale = w_int.data_ptr(), w_scale.data_ptr()
            L.check(lib.mnb_conv2d_fwd(C.byref(sh), C.byref(o), y.data_ptr(), L.stream()), "conv2d_fwd")

        def pk_dgrad():
            dp, _ = PK.pack_act(dy, None, 2, ch_scale=w_scale, groups=G)
            wi = PK.pack_weight(sh, 1, 2, 1, w_int=w_int, kzero=w_scale)
            L.check(PK.run_conv(sh, 1, dp, 2, wi, 1, dx, bits8=bits8, gain=0.1), "dgrad")

        def gen_dgrad():
            L.check(lib.mnb_conv2d_dgrad(C.byref(sh), dy.data_ptr(), wq.data_ptr(), bits.data_ptr(), C.byref(qp),
                                         dx.data_ptr(), L.stream()), "conv2d_dgrad")

        def pk_wgrad():
            L.check(PK.run_wgrad(sh, dy_pk, 2, x_pk, 1, dw, a_scale=wg_scale, kdiv=w_scale), "wgrad")

        def gen_wgrad():
            L.check(lib.mnb_conv2d_wgrad(C.byref(sh), dy.data_ptr(), C.byref(ops), dw.data_ptr(), ws.data_ptr(), L.stream()),
                    "conv2d_wgrad")

        rec = dict(kind="layer", layer=name, shape=[batch, cin, hw, hw, cout, k, G])
        for what, a, b in (("fwd", pk_fwd, gen_fwd), ("dgrad", pk_dgrad, gen_dgrad), ("wgrad", pk_wgrad, gen_wgrad)):
            tp, tg = _timeit([a, b], iters)
            rec[what] = dict(pk_ms=round(tp, 4), generic_ms=round(tg, 4), speedup=round(tg / tp, 2))
        L.tc_check()
        _emit(rec, out)


def step_child(scheme, batch, windows, iters, fuse=True):
    """one tree's pruned QAT step: JSON with the window medians and the losses of the timed steps"""
    import torch
    from harness import models as zoo, train as H
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    base = zoo.init_like_reference(zoo.NINGC(CFG))
    kw = dict(W=3, A=2, fuse_bn=fuse) if scheme == "wbwtab" else dict(a_bits=4, w_bits=4, fuse=fuse)
    eng = H.prepare_engine(base, scheme, **kw).to(dev)
    st = H.QatStepper(eng, lr=0.01, wd=1e-5, flat=True, graph=True)
    data = [H.synthetic_batch(batch, 32, seed=100 + i, device=dev) for i in range(4)]
    for i in range(6):
        st.step(*data[i % 4])
    torch.cuda.synchronize()
    times, losses = [], []
    for w in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(iters):
            losses.append(st.step(*data[i % 4]).detach().clone())
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / iters)
    from micronet_b200 import _lib as L
    L.tc_check()
    return dict(ms=times, graph=st.graph is not None, losses=[float(v) for v in torch.stack(losses).cpu()])


def step(out, parent, batch=256, rounds=3, iters=10):
    trees = [("this", ROOT)] + ([("parent", os.path.abspath(parent))] if parent else [])
    for scheme, fuse in (("wbwtab", True), ("dorefa", True), ("dorefa", False)):
        res, errors = {name: [] for name, _ in trees}, {}
        for _ in range(rounds):
            for name, tree in trees:        # alternating child processes
                # this file's step_child on the other tree's package and harness
                cmd = [sys.executable, "-c", f"import sys, json, importlib.util as U; sys.path.insert(0, {tree!r}); "
                       f"s = U.spec_from_file_location('pruned_probe', {os.path.abspath(__file__)!r}); "
                       f"m = U.module_from_spec(s); s.loader.exec_module(m); "
                       f"print('RESULT', json.dumps(m.step_child({scheme!r}, {batch}, 1, {iters}, {fuse})))"]
                env = dict(os.environ, PYTHONPATH=tree)
                p = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True)
                line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
                if p.returncode or not line:     # e.g. a tree that cannot run this graph at all: reported, not timed
                    errors[name] = (p.stderr.strip().splitlines() or ["no output"])[-1][:300]
                    continue
                res[name].append(json.loads(line[0][7:]))
        rec = dict(kind="step", scheme=scheme, fuse=fuse, batch=batch)
        for name, err in errors.items():
            rec[name + "_error"] = err
        for name, rs in res.items():
            if not rs:
                continue
            rec[name + "_ms"] = round(statistics.median(r["ms"][0] for r in rs), 3)
            rec[name + "_graph"] = all(r["graph"] for r in rs)
        if parent and res["this"] and res["parent"]:
            a, b = res["this"][0]["losses"], res["parent"][0]["losses"]
            rec["first_loss_diff"] = abs(a[0] - b[0])
            rec["max_loss_diff"] = max(abs(x - y) for x, y in zip(a, b))
            rec["losses_equal"] = a == b
            rec["speedup"] = round(rec["parent_ms"] / rec["this_ms"], 2)
        _emit(rec, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", action="store_true")
    ap.add_argument("--step", action="store_true")
    ap.add_argument("--parent", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pruned_probe measures on the GPU: no CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    _emit(dict(kind="device", gpu=smi), a.out)
    if a.layers:
        layers(a.out)
    if a.step:
        step(a.out, a.parent)


if __name__ == "__main__":
    main()
