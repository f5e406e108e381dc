"""Debug: where do the roles of the tensor-core conv kernel wait?  (needs a GPU)

    python harness/tc_role_profile.py

Prints, per layer shape of NIN-GC at batch 256 and per kernel (fwd / dgrad), the fraction of the
kernel's cycles each warp role (TMA producer, the two MMA warpgroups, converters) spent inside
pipeline waits.  The role that barely waits is the bottleneck."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micronet_b200 import _lib as L, functional as F_  # noqa: E402

SHAPES = [(256, 256, 32, 32, 256, 1, 2), (256, 256, 16, 16, 512, 3, 16), (256, 512, 16, 16, 512, 1, 4),
          (256, 512, 8, 8, 1024, 3, 32), (256, 1024, 8, 8, 1024, 1, 8)]
NAMES = ("tma", "mma0", "mma1", "conv")


def main():
    dev = torch.device("cuda:0")
    lib = L.load()
    prof = torch.zeros(16, dtype=torch.int64, device=dev)
    for (B, C, H, W, K, R, G) in SHAPES:
        g = torch.Generator().manual_seed(1)
        x = (torch.randint(0, 2, (B, C, H, W), generator=g).float() * 2 - 1).to(dev).requires_grad_(True)
        w_int = torch.randint(-1, 2, (K, C // G, R, R), generator=g, dtype=torch.int16).to(dev)
        w_scale = (torch.rand(K, generator=g) * 0.02 + 0.001).to(dev)
        wq = (w_int.float() * w_scale.view(-1, 1, 1, 1)).requires_grad_(True)
        go = torch.randn(B, K, H, W, generator=g).to(dev)
        for phase in ("fwd", "dgrad"):
            for rep in range(3):
                xg = x.detach().requires_grad_(True)
                if phase == "fwd":
                    prof.zero_(); torch.cuda.synchronize()
                    lib.mnb_set_tc_profile_buffer(prof.data_ptr())
                y = F_.quant_conv2d(xg, wq, None, w_int, w_scale, None, (1, 1), (R // 2, R // 2), (1, 1), G)
                torch.cuda.synchronize()
                if phase == "fwd":
                    lib.mnb_set_tc_profile_buffer(None)
                    continue
                prof.zero_(); torch.cuda.synchronize()
                lib.mnb_set_tc_profile_buffer(prof.data_ptr())
                gx, = torch.autograd.grad(y, xg, go)
                torch.cuda.synchronize()
                lib.mnb_set_tc_profile_buffer(None)
            p = prof.cpu().view(4, 4).double()
            line = f"{phase:5s} {str((B, C, H, W, K, R, G)):38s}"
            for i, n in enumerate(NAMES):
                tot = max(p[i, 3].item(), 1.0)
                line += f" | {n}: wait {100 * p[i, 0] / tot:4.0f}% +{100 * p[i, 1] / tot:4.0f}% +{100 * p[i, 2] / tot:3.0f}%"
            print(line + f" | cycles/CTA {p[1, 3].item() / 132:.0f}")


if __name__ == "__main__":
    main()
