"""Host-only plan query of the fp32 first-layer convolution (mnb_fconv2d_plan) decoded to dicts, and the cases of
test_gpu_fconv_fp64.py with the plans each was written for, so that test_fconv_plan_cpu.py can check on the host that
they still reach those plans and, together, every plan path of mnb_conv_fp32_tc.cu."""
import ctypes as C
from collections import namedtuple

FIELDS = "NP KP TH n_tiles grid nbuf_a smem_bytes patch_floats".split()
NUM_SMS = 132
# patch_commit moves the first PF * nconv floats of a patch through registers, the rest in its remainder loop
PATCH_PREFETCH = 4 * (512 - 32 - 128)


def shape(B, Cc, H, W, K, R):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, R // 2, R // 2, 1, 1, 1)


def plan(sh, wgrad):
    """plan of mnb_fconv2d_fwd_tc (wgrad False) or mnb_fconv2d_wgrad_tc (wgrad True); None if the shape is refused"""
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(FIELDS))()
    if L.load().mnb_fconv2d_plan(C.byref(sh), int(bool(wgrad)), out, len(FIELDS)) != 0:
        return None
    return dict(zip(FIELDS, list(out)))


# shape: (B, C, H, W, K, R); fwd / wgrad: the plan fields the case was written for, None = refused by that kernel
Case = namedtuple("Case", "id shape fwd wgrad")

CASES = {c.id: c for c in [
    # the bench stems at the bench batch: single operand buffer, 2048 tiles over 132 CTAs (68 of them run 16 tiles)
    Case("ningc_stem", (256, 3, 32, 32, 256, 5), dict(NP=256, TH=4, n_tiles=2048, grid=132, nbuf_a=1),
         dict(NP=256, n_tiles=2048, grid=132)),
    Case("nin_stem", (256, 3, 32, 32, 192, 5), dict(NP=192, TH=4, n_tiles=2048, grid=132, nbuf_a=1),
         dict(NP=256, n_tiles=2048, grid=132)),
    # double-buffered operand, 512 tiles; one 128-channel half in the weight gradient
    Case("res_stem", (64, 3, 32, 32, 64, 3), dict(NP=64, KP=32, n_tiles=512, grid=132, nbuf_a=2),
         dict(NP=128, n_tiles=512, grid=132)),
    # 8 x 6 x 34 = 1632-float patch: the remainder loop of patch_commit
    Case("patch_tail", (40, 8, 32, 32, 64, 3), dict(NP=64, KP=80, n_tiles=320, grid=132, patch_floats=1632),
         dict(NP=128, n_tiles=320, grid=132, patch_floats=1632)),
    # NP % 32 == 16: the last 32-channel slab reads B rows past NP, four tiles per CTA
    Case("np48", (66, 5, 32, 32, 40, 5), dict(NP=48, KP=128, n_tiles=528, grid=132),
         dict(NP=128, KP=128, n_tiles=528, grid=132)),
    # C*R*S = 125 at the largest K both kernels accept
    Case("kr125_k128", (8, 5, 32, 32, 128, 5), dict(NP=128, KP=128, n_tiles=64, grid=64),
         dict(NP=128, KP=128, n_tiles=64, grid=64)),
    # C*R*S = 98: the forward goes up to K = 176, the weight gradient only to 128
    Case("kr98_k176", (8, 2, 32, 32, 176, 7), dict(NP=176, KP=112, nbuf_a=1), None),
    Case("kr98_k144", (8, 2, 32, 32, 144, 7), dict(NP=144, KP=112), None),
    Case("kr98_k128", (8, 2, 32, 32, 128, 7), dict(NP=128, KP=112), dict(NP=128, KP=112)),
    # 16 rows of 8 per tile / one row of 128 per tile, both with more tiles than CTAs
    Case("w8", (96, 3, 32, 8, 32, 3), dict(TH=16, n_tiles=192, grid=132), dict(TH=16, n_tiles=192, grid=132)),
    Case("w128", (4, 3, 64, 128, 32, 5), dict(TH=1, n_tiles=256, grid=132), dict(TH=1, n_tiles=256, grid=132)),
    # batch 1: fewer tiles than SMs
    Case("b1", (1, 3, 32, 32, 256, 5), dict(NP=256, n_tiles=8, grid=8), dict(NP=256, n_tiles=8, grid=8)),
]}

# which cases each part of the GPU test runs
ONEHOT_FWD = ["ningc_stem", "nin_stem", "res_stem", "patch_tail", "np48", "w8", "w128", "kr98_k176"]
SPARSE_WGRAD = ["ningc_stem", "nin_stem", "patch_tail", "np48", "w128"]
RANDOM = list(CASES)
