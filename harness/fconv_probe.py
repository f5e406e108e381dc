"""A/B timing of the fp32 first-layer convolution's entry points at the bench stems (batch 256):
mnb_fconv2d_fwd_tc against mnb_fconv2d_fwd_wg, mnb_fconv2d_wgrad_tc against mnb_fconv2d_wgrad_wg (each new entry point
where its plan covers the stem).

    python harness/fconv_probe.py [--batch 256] [--windows 5] [--launches 50]

The versions alternate window by window; each window runs `launches` launches over 4 rotating operand sets, and the
median window is reported in us per launch next to the HBM floor (the fp32 y written / dy read at 3.35 TB/s) and the
tensor floor (the six bf16 piece products at 989 TFLOP/s, H100 SXM data sheet).  The outputs of the two forward entry
points, and those of the two weight-gradient entry points, are compared byte for byte."""
import argparse
import ctypes as C
import statistics
import subprocess

import torch

STEMS = {"ningc_stem": (3, 32, 32, 256, 5), "nin_stem": (3, 32, 32, 192, 5), "res_stem": (3, 32, 32, 64, 3)}
HBM_BPS, BF16_FLOPS = 3.35e12, 989e12
NSETS = 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def window_us(fn, launches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(launches):
        fn(i % NSETS)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def ab(fns, windows, launches):
    """median us per launch of each named fn, windows alternating between them"""
    for fn in fns.values():
        for i in range(2 * NSETS):
            fn(i % NSETS)
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            times[k].append(window_us(fn, launches))
    return {k: statistics.median(v) for k, v in times.items()}


def run_stem(lib, L, name, B, windows, launches):
    Cc, H, W, K, R = STEMS[name]
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    xs = [torch.randn(B, Cc, H, W, device=dev, generator=g) for _ in range(NSETS)]
    ws = [torch.randn(K, Cc, R, R, device=dev, generator=g) * 0.1 for _ in range(NSETS)]
    bs = [torch.randn(K, device=dev, generator=g) for _ in range(NSETS)]
    dys = [torch.randn(B, K, H, W, device=dev, generator=g) for _ in range(NSETS)]
    y_old = torch.empty(B, K, H, W, device=dev)
    y_new = torch.empty_like(y_old)
    dw_old = torch.empty_like(ws[0])
    dw_new = torch.empty_like(ws[0])
    sh = L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, R // 2, R // 2, 1, 1, 1)
    scratch = torch.empty(int(lib.mnb_fconv2d_wgrad_tc_scratch_bytes(C.byref(sh))), dtype=torch.uint8, device=dev)
    has_fwd = lib.mnb_fconv2d_wg_plan(C.byref(sh), None, 0) == 0
    has_wg = int(lib.mnb_fconv2d_wgrad_wg_scratch_bytes(C.byref(sh))) >= 0
    err = L.tc_err_flag(dev)

    def fwd(entry, y):
        return lambda i: L.check(entry(C.byref(sh), xs[i].data_ptr(), ws[i].data_ptr(), bs[i].data_ptr(), y.data_ptr(),
                                       err.data_ptr(), L.stream()), name)

    def wgrad(entry, dw):
        return lambda i: L.check(entry(C.byref(sh), dys[i].data_ptr(), xs[i].data_ptr(), dw.data_ptr(),
                                       scratch.data_ptr(), err.data_ptr(), L.stream()), name)

    fns = {"fwd_tc": fwd(lib.mnb_fconv2d_fwd_tc, y_old), "wgrad_tc": wgrad(lib.mnb_fconv2d_wgrad_tc, dw_old)}
    if has_fwd:
        fns["fwd_wg"] = fwd(lib.mnb_fconv2d_fwd_wg, y_new)
    if has_wg:
        fns["wgrad_wg"] = wgrad(lib.mnb_fconv2d_wgrad_wg, dw_new)
    t = ab(fns, windows, launches)
    same = True
    for i in range(NSETS):
        for old, new, out_old, out_new in (("fwd_tc", "fwd_wg", y_old, y_new), ("wgrad_tc", "wgrad_wg", dw_old, dw_new)):
            if new in fns:
                out_new.fill_(float("nan"))
                fns[old](i)
                fns[new](i)
                torch.cuda.synchronize()
                same &= torch.equal(out_old.view(torch.int32), out_new.view(torch.int32))
    assert int(err.item()) == 0, f"error flag {int(err.item())}"
    big = B * K * H * W * 4
    flops = 2 * B * H * W * K * ((Cc * R * R + 15) // 16 * 16) * 6
    hbm, tens = big / HBM_BPS * 1e6, flops / BF16_FLOPS * 1e6
    cols = []
    for old, new in (("fwd_tc", "fwd_wg"), ("wgrad_tc", "wgrad_wg")):
        cols.append(f"{old} {t[old]:.1f} us" + (f" {new} {t[new]:.1f} us ({t[old] / t[new]:.2f}x)" if new in t else ""))
    print(f"{name} B={B}: floors hbm {hbm:.0f} us, tensor {tens:.0f} us | {'  '.join(cols)} | outputs byte-equal: {same}",
          flush=True)
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--stems", default=",".join(STEMS))
    a = ap.parse_args()
    from micronet_b200 import _lib as L
    lib = L.load()
    print("card:", card(), flush=True)
    ok = all([run_stem(lib, L, s, a.batch, a.windows, a.launches) for s in a.stems.split(",")])
    print("card:", card(), flush=True)
    raise SystemExit(0 if ok else 1)


if __name__ == "__main__":
    main()
