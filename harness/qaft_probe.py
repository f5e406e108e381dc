"""Step time of the IAO W8A8 BN-fused QAFT step of NIN and NIN-GC with and without the hand-offs of
iao.prepare(fuse=True), batch 256, FlatAdam, CUDA-graph replay.

    python -m harness.qaft_probe --out DIR [--runs 3] [--steps 50] [--warmup 5] [--batch 256]

Every measurement runs in a fresh process, linked and un-linked alternating, ``--runs`` times each; the card's name and power
limit are read in the same call.  Each process first calibrates the quantizers with two QAT forwards (the QAT -> QAFT flow
of the README recipes) from the same seed.  The first run of each variant dumps its loss and parameters after its steps
(DIR/<model>_<variant>.pt); the two dumps must be equal byte for byte.  A last pair of processes profiles a few eager steps
with torch.profiler and lists the device time per kernel (harness.step_profile's naming).  Writes DIR/qaft_probe.json."""
import argparse
import copy
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from harness import train as H  # noqa: E402
from harness.step_profile import base_name, card  # noqa: E402

MODELS = ("nin", "nin_gc")


def build(model, fuse, batch, dev):
    from micronet_b200 import iao
    base = H.build_float_model(model)
    qat = iao.prepare(copy.deepcopy(base), a_bits=8, w_bits=8, bn_fuse=True).to(dev).train()
    with torch.no_grad():
        for s in (11, 12):
            qat(H.synthetic_batch(batch, 32, seed=s, device=dev)[0])
    m = iao.prepare(base, a_bits=8, w_bits=8, bn_fuse=True, qaft=True, fuse=fuse).to(dev)
    m.load_state_dict(qat.state_dict())
    return m.train()


def child(args):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = build(args.model, bool(args.fuse), args.batch, dev)
    batches = [H.synthetic_batch(args.batch, 32, seed=100 + i, device=dev) for i in range(2)]
    if args.profile:
        st = H.QatStepper(m, lr=1e-3, wd=1e-5, flat=True, graph=False)
        for i in range(args.warmup):
            st.step(*batches[i % 2])
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for i in range(5):
                st.step(*batches[i % 2])
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                kern[base_name(e.name)] = kern.get(base_name(e.name), 0.0) + e.device_time / 5
        print(json.dumps({"kernels_us_per_step": dict(sorted(kern.items(), key=lambda kv: -kv[1]))}))
        return
    st = H.QatStepper(m, lr=1e-3, wd=1e-5, flat=True, graph=True)
    for i in range(args.warmup):
        st.step(*batches[i % 2])     # no reference kept: a live loss keeps AccumulateGrad nodes that break the capture
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(args.steps):
        loss = st.step(*batches[i % 2])
    b.record()
    torch.cuda.synchronize()
    from micronet_b200 import _lib as L
    L.tc_check()
    if args.dump:
        torch.save({"loss": loss.detach().cpu(), **{n: p.detach().cpu() for n, p in m.named_parameters()}}, args.dump)
    print(json.dumps({"ms_per_step": a.elapsed_time(b) / args.steps, "graph": st.graph is not None,
                      "graph_error": st.graph_error}))


def run_child(args, model, fuse, extra):
    cmd = [sys.executable, "-m", "harness.qaft_probe", "--child", "--model", model, "--fuse", str(fuse), "--steps",
           str(args.steps), "--warmup", str(args.warmup), "--batch", str(args.batch)] + extra
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    if out.returncode != 0:
        raise SystemExit(f"qaft_probe child {model} fuse={fuse} failed:\n{out.stderr[-3000:]}")
    return json.loads(out.stdout.strip().splitlines()[-1])


def same_bytes(pa, pb):
    a, b = torch.load(pa), torch.load(pb)
    return a.keys() == b.keys() and all(a[k].numpy().tobytes() == b[k].numpy().tobytes() for k in a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--model", default="nin")
    ap.add_argument("--fuse", type=int, default=0)
    ap.add_argument("--dump")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qaft_probe: no CUDA device")
    if args.child:
        return child(args)
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card(), "batch": args.batch, "steps": args.steps, "models": {}}
    print("card:", res["card"])
    for model in MODELS:
        r = {"unlinked_ms": [], "linked_ms": []}
        for i in range(args.runs):
            for fuse in (0, 1):
                extra = ["--dump", os.path.join(args.out, f"{model}_{fuse}.pt")] if i == 0 else []
                out = run_child(args, model, fuse, extra)
                r["linked_ms" if fuse else "unlinked_ms"].append(out["ms_per_step"])
                if not out["graph"]:
                    r["graph_error"] = out["graph_error"]
        r["bytes_equal"] = same_bytes(os.path.join(args.out, f"{model}_0.pt"), os.path.join(args.out, f"{model}_1.pt"))
        for fuse in (0, 1):
            r["linked_kernels_us" if fuse else "unlinked_kernels_us"] = run_child(args, model, fuse, ["--profile"])[
                "kernels_us_per_step"]
        res["models"][model] = r
        print(f"{model}: un-linked {['%.3f' % v for v in r['unlinked_ms']]} ms, linked {['%.3f' % v for v in r['linked_ms']]}"
              f" ms per step, outputs byte-equal: {r['bytes_equal']}")
        for fuse in (0, 1):
            key = "linked_kernels_us" if fuse else "unlinked_kernels_us"
            top = list(r[key].items())[:12]
            print(f"  {'linked' if fuse else 'un-linked'}: device us per step {sum(r[key].values()):.0f}; top kernels: "
                  + ", ".join(f"{k} {v:.0f}" for k, v in top))
    with open(os.path.join(args.out, "qaft_probe.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
