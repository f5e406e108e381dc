"""A/B of two builds of libmicronet_b200.so on the bench workloads, alternating in one session.

    python -m harness.wgmma_ab --old-lib OLD.so --out DIR [--rounds 3] [--steps 20] [--extra-rounds 2]

OLD.so is a library built from another commit (e.g. `git archive <commit>` extracted into a git-ignored directory and
built there with `python -m micronet_b200.build`); the other build is the one in the tree.  Every run is a fresh
`bench.py` process; between runs the in-tree library file is replaced by the build under test, and the tree's own build
is put back at the end.  Per round and build:
* the headline workload with `--kernels-json` (per-kernel CUDA-event times), `--dump-outputs` in the first round;
* then, `--extra-rounds` times each, short runs of the other workloads (the PTQ inference one with `--dump-outputs`).
Writes every bench line and kernel table under DIR and prints one JSON summary (also DIR/summary.json): the card's name
and power limit, img/s per run, the per-kernel medians of both builds, and whether the dumps of the two builds are
bit-identical.  The dumps themselves (up to ~100 MB per build) go to a temporary directory that is removed at the end."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "micronet_b200", "lib", "libmicronet_b200.so")
HEADLINE = "nin_gc_wbwtab_w3a2"
OTHERS = ["nin_dorefa_w8a8", "nin_gc_dorefa_w4a4", "resnet18_iao_w8a8_bnfuse", "resnet18_iao_ptq_224"]
INFERENCE = "resnet18_iao_ptq_224"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError) as e:
        return f"unknown ({type(e).__name__})"


def install(src):
    tmp = LIB_PATH + ".ab_tmp"
    shutil.copyfile(src, tmp)
    os.replace(tmp, LIB_PATH)


def bench(out_dir, tag, argv):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--no-extra",
                        *argv], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    with open(os.path.join(out_dir, tag + ".log"), "w") as f:
        f.write(p.stdout + "\n--- stderr ---\n" + p.stderr)
    if p.returncode != 0:
        raise SystemExit(f"bench.py {' '.join(argv)} failed ({p.returncode}), see {tag}.log:\n{p.stderr[-2000:]}")
    return json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])


def same_files(a, b):
    import numpy as np
    names = sorted(os.listdir(a))
    if names != sorted(os.listdir(b)):
        return False
    for n in names:
        x, y = np.load(os.path.join(a, n)), np.load(os.path.join(b, n))
        if x.shape != y.shape or x.tobytes() != y.tobytes():
            return False
    return True


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old-lib", required=True, help="the other build of libmicronet_b200.so")
    ap.add_argument("--out", required=True, help="directory for bench lines, kernel tables and dumps")
    ap.add_argument("--rounds", type=int, default=3, help="headline runs per build")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--extra-rounds", type=int, default=2, help="runs per build of each other workload")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    keep = tempfile.mkdtemp(prefix="mnb_ab_")
    libs = {"old": os.path.join(keep, "old.so"), "new": os.path.join(keep, "new.so")}
    shutil.copyfile(os.path.abspath(args.old_lib), libs["old"])
    shutil.copyfile(LIB_PATH, libs["new"])
    res = {"card": card(), "headline": {"old": [], "new": []}, "others": {}}
    tables = {"old": [], "new": []}
    try:
        for r in range(args.rounds):
            for tag in ("old", "new"):
                install(libs[tag])
                kj = os.path.join(args.out, f"kernels_{tag}_{r}.json")
                argv = ["--steps", str(args.steps), "--warmup", str(args.warmup), "--kernels-json", kj]
                if r == 0:
                    argv += ["--dump-outputs", os.path.join(keep, f"dump_{HEADLINE}_{tag}")]
                line = bench(args.out, f"{HEADLINE}_{tag}_{r}", argv)
                res["headline"][tag].append({"value": line["value"], "e2e": line["e2e"]["value"],
                                             "ms_per_step": line["ms_per_step"], "clocks": line.get("clocks")})
                tables[tag].append(json.load(open(kj))["kernels"])
        for wl in OTHERS:
            runs = {"old": [], "new": []}
            for r in range(args.extra_rounds):
                for tag in ("old", "new"):
                    install(libs[tag])
                    argv = ["--workload", wl, "--steps", "10", "--warmup", "3"]
                    if r == 0 and wl == INFERENCE:
                        argv += ["--dump-outputs", os.path.join(keep, f"dump_{wl}_{tag}")]
                    runs[tag].append(bench(args.out, f"{wl}_{tag}_{r}", argv)["value"])
            res["others"][wl] = runs
        res["dumps_bit_identical"] = {wl: same_files(os.path.join(keep, f"dump_{wl}_old"), os.path.join(keep, f"dump_{wl}_new"))
                                      for wl in (HEADLINE, INFERENCE)}
    finally:
        install(libs["new"])
        shutil.rmtree(keep, ignore_errors=True)
    h = {tag: [x["value"] for x in v] for tag, v in res["headline"].items()}
    res["headline_gain"] = {"min_new_over_max_old": min(h["new"]) / max(h["old"]) - 1,
                            "median_new_over_median_old": median(h["new"]) / median(h["old"]) - 1}
    # per-kernel medians (µs per launch) over the headline rounds
    rows = {}
    for tag in ("old", "new"):
        for t in tables[tag]:
            for k in t:
                rows.setdefault((k["kind"], tuple(k["shape"])), {"old": [], "new": []})[tag].append(k["avg_us"])
    res["kernels_us"] = sorted(({"kind": k, "shape": list(s), "old": median(v["old"]) if v["old"] else None,
                                 "new": median(v["new"]) if v["new"] else None} for (k, s), v in rows.items()),
                               key=lambda d: -(d["old"] or 0))
    txt = json.dumps(res, indent=1)
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        f.write(txt + "\n")
    print(txt)


if __name__ == "__main__":
    main()
