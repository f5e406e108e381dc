"""Micro-benchmark (GPU): cycles per wgmma M64 x N x K16 (bf16, smem operands) from one warpgroup."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micronet_b200 import _lib as L
lib = L.load()
dev = torch.device("cuda:0")
out = torch.zeros(2, dtype=torch.int64, device=dev)
err = torch.zeros(1, dtype=torch.int32, device=dev)
iters = 2000
for mn in (0, 1):
    for N in (16, 32, 64, 128, 256):
        for n_acc in (1, 4):
            if n_acc * N > 512:
                continue
            for shift in (0, 19, 100):  # 100+: per-thread (lane 0) issue loop instead of the warp-converged one
                L.check(lib.mnb_selftest_mma_rate(N, n_acc, shift, iters, mn, out.data_ptr(), err.data_ptr(), L.stream()), "rate")
                torch.cuda.synchronize()
                o = out.cpu()
                print(f"{'MN' if mn else 'K '}-major N={N:3d} acc={n_acc} shift={shift:2d}: {o[0].item() / iters:7.1f} cyc/MMA total, {o[1].item() / iters:6.1f} issue")
