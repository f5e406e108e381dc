"""One case list for the round-1 fused tensor-core convolutions: the forward and data-gradient kernel conv_tc_kernel<NG>
(csrc/mnb_conv_tc_fwd.cu, mnb_fq_conv2d_fwd_tc / mnb_conv2d_dgrad_tc) and the weight-gradient kernel
(csrc/mnb_conv_tc_wgrad.cu, mnb_conv2d_wgrad_tc).

Each case is a stride-1 'same' conv shape (B, C, H, W, K, R, groups) with the plans it was written for, as the launchers'
own plan functions report them (mnb_tc_conv_plan / mnb_wgrad_tc_plan): the forward plan for a raw fp32 input and for a
fused quantizer (they differ in the operand buffers: three bf16 pieces against one level), the data-gradient plan and the
weight-gradient plan; None where that launcher refuses the shape.  tests/test_tc_conv_plan_cpu.py checks on the host that
the list launches every kernel instance, reaches every plan feature below and every refusal reason, covers the
quantized convs of the wbwtab NIN / NIN-GC training graphs, and that each plan is still the pinned one;
tests/test_gpu_tc_conv.py runs every case against fp64."""
import ctypes as C
from collections import namedtuple

Case = namedtuple("Case", "id shape fwd dgrad wgrad")       # fwd: (raw fp32 plan, quantizer plan) or None

FWD_FIELDS = ("NG TB TH row_tiles n_tiles CC nchunk nst nop slab_groups n_slabs collapsed smem BW npos_in grid "
              "n_mma_off").split()
WGRAD_FIELDS = "Gb nsplit tap_groups tpc n_block CC TH TB nbuf nst ranks n_slabs smem npos_d npos_x n_tiles".split()
INSTANCES = list(range(16, 161, 16))       # conv_tc_kernel<NG>: output channels per group (dgrad: input channels per group)


def conv_shape(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, R // 2, R // 2, 1, 1, G)


def _last_error():
    from micronet_b200 import _lib as L
    return L.load().mnb_last_error().decode()


def fwd_plan(shape, quant_mode=0, dgrad=False):
    """plan tuple of mnb_fq_conv2d_fwd_tc (quant_mode 0: raw fp32 input) or mnb_conv2d_dgrad_tc; None where refused"""
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(FWD_FIELDS))()
    rc = L.load().mnb_tc_conv_plan(C.byref(conv_shape(shape)), int(dgrad), quant_mode, out, len(out))
    if rc == L.E_UNSUPPORTED:
        return None
    L.check(rc, "tc_conv_plan")
    return tuple(out)


def wgrad_plan(shape, quant_mode=0):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(WGRAD_FIELDS))()
    rc = L.load().mnb_wgrad_tc_plan(C.byref(conv_shape(shape)), quant_mode, out, len(out))
    if rc == L.E_UNSUPPORTED:
        return None
    L.check(rc, "wgrad_tc_plan")
    return tuple(out)


def refusal(kind, shape):
    """the reason (mnb_last_error) the launcher of ``kind`` ("fwd" / "dgrad" / "wgrad") refuses ``shape``, None if it
    accepts it"""
    p = wgrad_plan(shape) if kind == "wgrad" else fwd_plan(shape, 0, kind == "dgrad")
    return None if p is not None else _last_error().split(": ", 1)[1]


def plans(shape):
    """(fwd, dgrad, wgrad) in the format of Case"""
    f0, f1 = fwd_plan(shape, 0), fwd_plan(shape, 1)
    return (None if f0 is None else (f0, f1)), fwd_plan(shape, dgrad=True), wgrad_plan(shape)


def fd(plan):
    return dict(zip(FWD_FIELDS, plan))


def wd(plan):
    return dict(zip(WGRAD_FIELDS, plan))


# (B, C, H, W, K, R, groups); the pinned plans follow each shape
CASES = []


def _c(id, shape, fwd, dgrad, wgrad):
    CASES.append(Case(id, shape, fwd, dgrad, wgrad))


# NG 16: several images per tile, B % TB != 0 (11 images, 8 per tile); 1x1 on the collapsed tensor map
_c("ng16_tb_ragged", (11, 16, 4, 4, 16, 1, 1),
    ((16, 8, 4, 1, 2, 16, 1, 8, 4, 1, 1, 1, 132608, 4, 128, 2, 1), (16, 8, 4, 1, 2, 16, 1, 8, 4, 1, 1, 1, 99840, 4, 128, 2, 1)),
    (16, 8, 4, 1, 2, 16, 1, 8, 4, 1, 1, 1, 132608, 4, 128, 2, 1),
    (1, 1, 1, 1, 16, 16, 4, 8, 1, 8, 2, 1, 167936, 128, 128, 2))
# NG 32: 3x3, H % TH != 0 (7 rows per tile of a 16-row plane), CC 32
_c("ng32_h_ragged", (2, 32, 16, 16, 32, 3, 1),
    ((32, 1, 7, 3, 6, 32, 1, 4, 3, 1, 1, 0, 225280, 18, 200, 6, 18), (32, 1, 7, 3, 6, 32, 1, 7, 4, 1, 1, 0, 216064, 18, 200, 6, 18)),
    (32, 1, 7, 3, 6, 32, 1, 4, 3, 1, 1, 0, 225280, 18, 200, 6, 18),
    (1, 1, 1, 9, 32, 32, 4, 1, 2, 7, 8, 1, 225280, 80, 120, 8))
# NG 16 / 32 at TH = 1: a padded row of 66 positions
_c("ng32_th1_w64", (2, 16, 5, 64, 32, 3, 1),
    ((32, 1, 1, 5, 10, 16, 1, 5, 4, 1, 1, 0, 217088, 66, 336, 10, 9), (32, 1, 1, 5, 10, 16, 1, 8, 4, 1, 1, 0, 167936, 66, 336, 10, 9)),
    (16, 1, 1, 5, 10, 32, 1, 2, 2, 1, 1, 0, 204800, 66, 336, 10, 18),
    (1, 1, 1, 9, 16, 16, 1, 1, 2, 7, 10, 1, 223232, 80, 216, 10))
# CC 16 through converter capacity (32 channels per group, 376 operand positions), forward and dgrad
_c("cc16_converter", (2, 32, 6, 60, 32, 3, 1),
    ((32, 1, 2, 3, 6, 16, 2, 5, 3, 1, 1, 0, 221184, 62, 376, 6, 9), (32, 1, 2, 3, 6, 16, 2, 8, 4, 1, 1, 0, 206848, 62, 376, 6, 9)),
    (32, 1, 2, 3, 6, 16, 2, 5, 3, 1, 1, 0, 221184, 62, 376, 6, 9),
    (1, 1, 1, 9, 32, 32, 1, 1, 2, 4, 12, 1, 215040, 64, 192, 12))
# CC 16 through the 64-entry mma_off table: 7x7
_c("cc16_mma_off_7x7", (2, 32, 9, 8, 32, 7, 1),
    ((32, 1, 9, 1, 2, 16, 2, 6, 2, 1, 1, 0, 222208, 14, 304, 2, 49), (32, 1, 9, 1, 2, 16, 2, 8, 4, 1, 1, 0, 218112, 14, 304, 2, 49)),
    (32, 1, 9, 1, 2, 16, 2, 6, 2, 1, 1, 0, 222208, 14, 304, 2, 49),
    (1, 1, 4, 13, 32, 32, 5, 1, 2, 7, 4, 4, 224256, 80, 176, 4))
# NG 48: W = 44 (not a power of two), H*W % 32 != 0, CC 16 through cin_g % 32
_c("ng48_w44", (2, 48, 12, 44, 48, 3, 1),
    ((48, 1, 2, 6, 12, 16, 3, 5, 4, 1, 1, 0, 222720, 46, 280, 12, 9), (48, 1, 2, 6, 12, 16, 3, 8, 4, 1, 1, 0, 184832, 46, 280, 12, 9)),
    (48, 1, 2, 6, 12, 16, 3, 5, 4, 1, 1, 0, 222720, 46, 280, 12, 9),
    (1, 1, 1, 9, 48, 16, 2, 1, 2, 4, 12, 1, 229376, 96, 192, 12))
# NG 80 / 32: H*W % 32 != 0
_c("ng80_12x12", (3, 32, 12, 12, 80, 3, 1),
    ((80, 1, 9, 2, 6, 32, 1, 5, 2, 1, 1, 0, 219136, 14, 184, 6, 18), (80, 1, 9, 2, 6, 32, 1, 6, 4, 1, 1, 0, 211968, 14, 184, 6, 18)),
    (32, 1, 9, 2, 6, 16, 5, 8, 4, 1, 1, 0, 201728, 14, 184, 6, 9),
    (1, 1, 1, 9, 32, 16, 6, 1, 2, 8, 6, 1, 212992, 96, 128, 6))
# NG 64 / 80
_c("ng64_3x3", (2, 80, 8, 8, 64, 3, 1),
    ((64, 1, 8, 1, 2, 16, 5, 8, 4, 1, 1, 0, 208896, 10, 152, 2, 9), (64, 1, 8, 1, 2, 16, 5, 8, 4, 1, 1, 0, 169984, 10, 152, 2, 9)),
    (80, 1, 8, 1, 2, 32, 2, 5, 2, 1, 1, 0, 219136, 10, 152, 2, 18),
    (1, 1, 2, 5, 80, 16, 8, 1, 2, 8, 2, 2, 198656, 80, 104, 2))
# NG 48 / 96: dgrad over 96 channels per group
_c("ng48_1x1", (3, 96, 8, 8, 48, 1, 1),
    ((48, 2, 8, 1, 2, 32, 3, 6, 4, 1, 1, 1, 223232, 8, 128, 2, 2), (48, 2, 8, 1, 2, 32, 3, 8, 4, 1, 1, 1, 190464, 8, 128, 2, 2)),
    (96, 2, 8, 1, 2, 16, 3, 8, 4, 1, 1, 1, 141312, 8, 128, 2, 1),
    (1, 1, 1, 1, 96, 16, 8, 2, 1, 8, 2, 1, 188416, 128, 128, 2))
# NG 96 / 64: two chunks per group
_c("ng96_3x3", (3, 64, 8, 8, 96, 3, 1),
    ((96, 1, 8, 1, 3, 32, 2, 3, 2, 1, 1, 0, 217088, 10, 152, 3, 18), (96, 1, 8, 1, 3, 32, 2, 5, 4, 1, 1, 0, 218112, 10, 152, 3, 18)),
    (64, 1, 8, 1, 3, 32, 3, 3, 2, 1, 1, 0, 217088, 10, 152, 3, 18),
    (1, 1, 2, 5, 64, 32, 8, 1, 2, 7, 3, 2, 221184, 80, 104, 3))
# NG 112: two groups in one slab
_c("ng112_slab2", (2, 224, 8, 8, 224, 1, 2),
    ((112, 2, 8, 1, 1, 16, 7, 8, 4, 2, 1, 1, 182272, 8, 128, 1, 1), (112, 2, 8, 1, 1, 16, 7, 8, 4, 2, 1, 1, 149504, 8, 128, 1, 1)),
    (112, 2, 8, 1, 1, 16, 7, 8, 4, 2, 1, 1, 182272, 8, 128, 1, 1),
    (1, 1, 1, 1, 112, 16, 8, 2, 1, 8, 1, 2, 192512, 128, 128, 1))
# NG 144: nine CC-16 chunks; wgrad: ragged channel split (144 = 128 + 16)
_c("ng144", (2, 144, 8, 8, 144, 1, 1),
    ((144, 2, 8, 1, 1, 16, 9, 8, 4, 1, 1, 1, 173568, 8, 128, 1, 1), (144, 2, 8, 1, 1, 16, 9, 8, 4, 1, 1, 1, 140800, 8, 128, 1, 1)),
    (144, 2, 8, 1, 1, 16, 9, 8, 4, 1, 1, 1, 173568, 8, 128, 1, 1),
    (1, 2, 1, 1, 144, 16, 8, 2, 1, 8, 1, 2, 200704, 128, 128, 1))
# NG 160; wgrad: ragged channel split at CC 32 (160 = 128 + 32)
_c("ng160", (2, 160, 8, 8, 160, 1, 1),
    ((160, 2, 8, 1, 1, 32, 5, 5, 3, 1, 1, 1, 224256, 8, 128, 1, 2), (160, 2, 8, 1, 1, 32, 5, 7, 4, 1, 1, 1, 216064, 8, 128, 1, 2)),
    (160, 2, 8, 1, 1, 32, 5, 5, 3, 1, 1, 1, 224256, 8, 128, 1, 2),
    (1, 2, 1, 1, 160, 32, 8, 2, 1, 5, 1, 2, 221184, 128, 128, 1))
# the largest accepted H (255): 32-row tiles, the last one ragged
_c("h255", (2, 32, 255, 4, 16, 1, 1),
    ((16, 1, 32, 8, 16, 32, 1, 6, 4, 1, 1, 1, 215040, 4, 128, 16, 2), (16, 1, 32, 8, 16, 32, 1, 8, 4, 1, 1, 1, 182272, 4, 128, 16, 2)),
    (32, 1, 32, 8, 16, 16, 1, 8, 4, 1, 1, 1, 133120, 4, 128, 16, 1),
    (1, 1, 1, 1, 32, 16, 32, 1, 1, 8, 16, 1, 172032, 128, 128, 16))
# dgrad: three 96-channel groups per slab, clamped by the 288-float scale array
_c("dgrad_slab288", (2, 96, 8, 8, 576, 1, 6),
    ((96, 2, 8, 1, 1, 16, 1, 8, 4, 2, 3, 1, 138240, 8, 128, 3, 1), (96, 2, 8, 1, 1, 16, 1, 8, 4, 2, 3, 1, 105472, 8, 128, 3, 1)),
    (16, 2, 8, 1, 1, 32, 3, 6, 4, 3, 2, 1, 223232, 8, 128, 2, 2),
    (1, 1, 1, 1, 16, 16, 8, 2, 1, 8, 1, 6, 167936, 128, 128, 1))
# fwd refused (256 output channels); dgrad NG 32 over 8 chunks; wgrad: an even channel split
_c("k256", (2, 32, 8, 8, 256, 1, 1),
    None,
    (32, 2, 8, 1, 1, 32, 8, 5, 4, 1, 1, 1, 214016, 8, 128, 1, 2),
    (1, 2, 1, 1, 32, 32, 8, 2, 1, 7, 1, 2, 221184, 128, 128, 1))
# many chunks per CTA: 1024 tiles over 132 CTAs, every operand buffer reused (mixed-exactness tests)
_c("mixed_3x3", (1024, 64, 8, 8, 32, 3, 1),
    ((32, 1, 8, 1, 1024, 32, 2, 5, 4, 1, 1, 0, 222208, 10, 152, 132, 18), (32, 1, 8, 1, 1024, 32, 2, 8, 4, 1, 1, 0, 175104, 10, 152, 132, 18)),
    (64, 1, 8, 1, 1024, 32, 1, 5, 4, 1, 1, 0, 222208, 10, 152, 132, 18),
    (1, 1, 2, 5, 64, 32, 8, 1, 2, 7, 66, 2, 221184, 80, 104, 1024))
# 1x1, 8 x 8, one tile: wgrad with ranks = 1
_c("one_tile", (1, 32, 8, 8, 32, 1, 1),
    ((32, 1, 8, 1, 1, 32, 1, 8, 4, 1, 1, 1, 183296, 8, 128, 1, 2), (32, 1, 8, 1, 1, 32, 1, 8, 4, 1, 1, 1, 117760, 8, 128, 1, 2)),
    (32, 1, 8, 1, 1, 32, 1, 8, 4, 1, 1, 1, 183296, 8, 128, 1, 2),
    (1, 1, 1, 1, 32, 32, 8, 1, 1, 8, 1, 1, 118784, 64, 64, 1))

# ---- the quantized convs of the wbwtab NIN / NIN-GC training graphs at the bench batch (256): the unfused A = 2 graph runs
# the 1x1 layers on this family, the A = 32 graphs every quantized conv the launchers accept
_c("nin_1x1a", (256, 192, 32, 32, 160, 1, 1),
    ((160, 1, 4, 8, 2048, 32, 6, 4, 3, 1, 1, 1, 218112, 32, 128, 132, 2), (160, 1, 4, 8, 2048, 32, 6, 7, 4, 1, 1, 1, 226304, 32, 128, 132, 2)),
    None,
    (1, 2, 1, 1, 192, 32, 4, 1, 1, 5, 66, 2, 229376, 128, 128, 2048))
_c("nin_1x1b", (256, 160, 32, 32, 96, 1, 1),
    ((96, 1, 4, 8, 2048, 32, 5, 4, 4, 1, 1, 1, 211968, 32, 128, 132, 2), (96, 1, 4, 8, 2048, 32, 5, 8, 4, 1, 1, 1, 211968, 32, 128, 132, 2)),
    (160, 1, 4, 8, 2048, 32, 3, 4, 4, 1, 1, 1, 211968, 32, 128, 132, 2),
    (1, 1, 1, 1, 160, 32, 4, 1, 1, 5, 132, 1, 221184, 128, 128, 2048))
_c("nin_5x5", (256, 96, 16, 16, 192, 5, 1),
    None,
    None,
    (1, 2, 5, 5, 96, 32, 3, 1, 2, 5, 13, 10, 229376, 64, 152, 1536))
_c("nin_1x1c", (256, 192, 16, 16, 192, 1, 1),
    None,
    None,
    (1, 2, 1, 1, 192, 32, 8, 1, 1, 5, 66, 2, 229376, 128, 128, 512))
_c("nin_3x3", (256, 192, 8, 8, 192, 3, 1),
    None,
    None,
    (1, 2, 5, 2, 192, 32, 4, 1, 2, 8, 13, 10, 178176, 48, 72, 512))
_c("nin_1x1d", (256, 192, 8, 8, 192, 1, 1),
    None,
    None,
    (1, 2, 1, 1, 192, 32, 8, 2, 1, 5, 66, 2, 229376, 128, 128, 128))
_c("gc_1x1g2", (256, 256, 32, 32, 256, 1, 2),
    ((128, 1, 4, 8, 2048, 32, 4, 4, 3, 2, 1, 1, 222208, 32, 128, 132, 2), (128, 1, 4, 8, 2048, 32, 4, 6, 4, 2, 1, 1, 214016, 32, 128, 132, 2)),
    (128, 1, 4, 8, 2048, 32, 4, 4, 3, 2, 1, 1, 222208, 32, 128, 132, 2),
    (1, 1, 1, 1, 128, 32, 4, 1, 1, 6, 66, 2, 229376, 128, 128, 2048))
_c("gc_3x3g16", (256, 256, 16, 16, 512, 3, 16),
    ((32, 1, 7, 3, 768, 16, 1, 8, 4, 4, 4, 0, 204800, 18, 200, 132, 9), (32, 1, 7, 3, 768, 16, 1, 8, 4, 4, 4, 0, 153600, 18, 200, 132, 9)),
    (16, 1, 7, 3, 768, 32, 1, 5, 2, 4, 4, 0, 223232, 18, 200, 132, 18),
    (4, 1, 2, 5, 64, 32, 4, 1, 2, 6, 16, 8, 227328, 80, 120, 1024))
_c("gc_1x1g4", (256, 512, 16, 16, 512, 1, 4),
    ((128, 1, 8, 2, 512, 32, 4, 4, 3, 2, 2, 1, 222208, 16, 128, 132, 2), (128, 1, 8, 2, 512, 32, 4, 6, 4, 2, 2, 1, 214016, 16, 128, 132, 2)),
    (128, 1, 8, 2, 512, 32, 4, 4, 3, 2, 2, 1, 222208, 16, 128, 132, 2),
    (1, 1, 1, 1, 128, 32, 8, 1, 1, 6, 33, 4, 229376, 128, 128, 512))
_c("gc_3x3g32", (256, 512, 8, 8, 1024, 3, 32),
    ((32, 1, 8, 1, 256, 16, 1, 8, 4, 4, 8, 0, 153600, 10, 152, 132, 9), (32, 1, 8, 1, 256, 16, 1, 8, 4, 4, 8, 0, 114688, 10, 152, 132, 9)),
    (16, 1, 8, 1, 256, 32, 1, 5, 4, 4, 8, 0, 222208, 10, 152, 132, 18),
    (4, 1, 2, 5, 64, 32, 8, 1, 2, 7, 8, 16, 221184, 80, 104, 256))
_c("gc_1x1g8", (256, 1024, 8, 8, 1024, 1, 8),
    ((128, 2, 8, 1, 128, 32, 4, 4, 3, 2, 4, 1, 222208, 8, 128, 132, 2), (128, 2, 8, 1, 128, 32, 4, 6, 4, 2, 4, 1, 214016, 8, 128, 132, 2)),
    (128, 2, 8, 1, 128, 32, 4, 4, 3, 2, 4, 1, 222208, 8, 128, 132, 2),
    (1, 1, 1, 1, 128, 32, 8, 2, 1, 6, 16, 8, 229376, 128, 128, 128))

MODEL_CASES = {"nin_1x1a", "nin_1x1b", "nin_5x5", "nin_1x1c", "nin_3x3", "nin_1x1d",
               "gc_1x1g2", "gc_3x3g16", "gc_1x1g4", "gc_3x3g32", "gc_1x1g8"}
BY_ID = {c.id: c for c in CASES}

# ---- shapes each launcher refuses, one per refusal reason of its plan(): (id, kind, (B, C, H, W, K, R, stride, pad, G),
# reason)
REFUSALS = [
    ("fwd_stride2", "fwd", (2, 16, 8, 8, 16, 3, 2, 1, 1), "stride/dilation != 1"),
    ("fwd_valid_3x3", "fwd", (2, 16, 8, 8, 16, 3, 1, 0, 1), "not a 'same' odd square filter"),
    ("fwd_cin24", "fwd", (2, 24, 8, 8, 16, 1, 1, 0, 1), "channels per group"),
    ("fwd_cout176", "fwd", (2, 16, 8, 8, 176, 1, 1, 0, 1), "channels per group"),
    ("fwd_w72", "fwd", (2, 16, 8, 72, 16, 1, 1, 0, 1), "image size"),
    ("fwd_h256", "fwd", (2, 16, 256, 4, 16, 1, 1, 0, 1), "image size"),
    ("fwd_row130", "fwd", (1, 16, 4, 64, 16, 67, 1, 33, 1), "padded row wider than 128 positions"),
    ("fwd_converter_7x7_w64", "fwd", (1, 16, 8, 64, 16, 7, 1, 3, 1), "tile too large for the converter"),
    ("fwd_9x9", "fwd", (1, 16, 8, 8, 16, 9, 1, 4, 1), "more than 64 filter taps"),
    ("fwd_weights_3x3_160", "fwd", (2, 160, 8, 8, 160, 3, 1, 1, 1), "weights of one group do not fit in shared memory"),
    ("dgrad_k304", "dgrad", (2, 16, 8, 8, 304, 1, 1, 0, 1), "more than 288 gradient channels per group"),
    ("dgrad_nin_5x5", "dgrad", (256, 96, 16, 16, 192, 5, 1, 2, 1), "weights of one group do not fit in shared memory"),
    ("wgrad_stride2", "wgrad", (2, 16, 8, 8, 16, 3, 2, 1, 1), "stride/dilation != 1"),
    ("wgrad_valid_3x3", "wgrad", (2, 16, 8, 8, 16, 3, 1, 0, 1), "not a 'same' odd square filter"),
    ("wgrad_cin24", "wgrad", (2, 24, 8, 8, 16, 1, 1, 0, 1), "channels per group"),
    ("wgrad_w72", "wgrad", (2, 16, 8, 72, 16, 1, 1, 0, 1), "image size"),
    ("wgrad_cg272_ng128", "wgrad", (2, 272, 8, 8, 128, 1, 1, 0, 1), "more than 256 activation channels per group"),
    ("wgrad_cg272_ng16", "wgrad", (2, 272, 8, 8, 16, 1, 1, 0, 1), "too many accumulator columns per CTA"),
    ("wgrad_row130", "wgrad", (1, 16, 4, 64, 16, 67, 1, 33, 1), "padded row wider than 128 positions"),
    ("wgrad_7x7_w60", "wgrad", (1, 16, 1, 60, 16, 7, 1, 3, 1), "shared memory budget"),
]
# refusals no shape can reach, and why (a sweep over 400k shapes in the coverage test finds none of them)
UNREACHABLE = {
    ("fwd", "shared memory budget"):
        "the slab is sized from the budget left after staging and operand buffers, and the rings only grow while they fit",
    ("wgrad", "ragged channel split"):
        "CC is 16 whenever a split group has Ng % 32 != 0, and Ng is a multiple of 16",
}


def conv_shape9(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, st, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def refusal9(kind, shape):
    """refusal reason of a general (B, C, H, W, K, R, stride, pad, G) shape, None if accepted"""
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = conv_shape9(shape)
    if kind == "wgrad":
        rc = lib.mnb_wgrad_tc_plan(C.byref(sh), 0, None, 0)
    else:
        rc = lib.mnb_tc_conv_plan(C.byref(sh), int(kind == "dgrad"), 0, None, 0)
    if rc == 0:
        return None
    assert rc == L.E_UNSUPPORTED, (kind, shape, rc)
    return _last_error().split(": ", 1)[1]


def launches(case):
    """[(kind, plan dict)] of every launch a case makes: the forward raw and quantized, the data and weight gradients"""
    out = []
    if case.fwd is not None:
        out += [("fwd", fd(case.fwd[0])), ("fwdq", fd(case.fwd[1]))]
    if case.dgrad is not None:
        out.append(("dgrad", fd(case.dgrad)))
    if case.wgrad is not None:
        out.append(("wgrad", wd(case.wgrad)))
    return out


def features(case, kind, p):
    """the plan features (names) one launch of a case reaches"""
    B, Cc, H, W, K, R, G = case.shape
    f = set()
    if kind == "wgrad":
        Ng = K // G
        if p["nsplit"] > 1:
            f.add("wgrad channel split, ragged" if Ng % 128 else "wgrad channel split, even")
            if Ng % 128:
                f.add(f"wgrad ragged channel split at CC {p['CC']}")
        for name, on in (("tap groups", p["tap_groups"] > 1), ("Gb > 1", p["Gb"] > 1), ("TB > 1", p["TB"] > 1),
                         ("ranks = 1", p["ranks"] == 1), ("ranks > 1", p["ranks"] > 1)):
            if on:
                f.add(f"wgrad {name}")
        f.add(f"wgrad CC {p['CC']}")
        f.add(f"wgrad nbuf {p['nbuf']}")
        return f
    d = "dgrad" if kind == "dgrad" else "fwd"
    cin_g, cout_g = (K // G, Cc // G) if d == "dgrad" else (Cc // G, K // G)
    if p["TB"] > 1 and B % p["TB"]:
        f.add(f"{d} TB > 1, B % TB != 0")
    if H % p["TH"]:
        f.add(f"{d} H % TH != 0")
    if p["TH"] == 1:
        f.add(f"{d} TH = 1")
    if H == 255:
        f.add(f"{d} H = 255")
    if W & (W - 1):
        f.add(f"{d} W not a power of two")
    if p["CC"] == 32:
        f.add(f"{d} CC 32")
    elif cin_g % 32:
        f.add(f"{d} CC 16: channels per group")
    elif p["npos_in"] * 4 > 6 * 224:
        f.add(f"{d} CC 16: converter capacity")
    elif R * R * 2 > 64:
        f.add(f"{d} CC 16: mma_off table")
    if p["slab_groups"] > 1:
        f.add(f"{d} slab_groups > 1")
    if p["n_slabs"] > 1:
        f.add(f"{d} n_slabs > 1")
    f.add(f"{d} {'collapsed' if p['collapsed'] else '4-d'} tensor map")
    if kind == "dgrad":
        # the 288-float scale array, not the 256 columns of the forward constants, bounds the slab
        if p["slab_groups"] * cin_g <= 288 < (p["slab_groups"] + 1) * cin_g and 256 // cout_g > p["slab_groups"]:
            f.add("dgrad slab clamped at 288 channels")
        if (H * W) % 32:
            f.add("dgrad STE bits, H*W % 32 != 0")
    if kind == "fwdq":
        if (H * W) % 32:
            f.add("fwd pass bits, H*W % 32 != 0")
        elif R == 1 and (p["TH"] * W) % 32 == 0:
            f.add("fwd pass bits, whole words")
        else:
            f.add("fwd pass bits, shared word per entry")
    return f


WANTED_FEATURES = {
    f"{d} {name}" for d in ("fwd", "dgrad") for name in (
        "TB > 1, B % TB != 0", "H % TH != 0", "TH = 1", "H = 255", "W not a power of two", "CC 32",
        "CC 16: channels per group", "CC 16: converter capacity", "CC 16: mma_off table", "slab_groups > 1",
        "n_slabs > 1", "collapsed tensor map", "4-d tensor map")
} | {
    "dgrad slab clamped at 288 channels", "dgrad STE bits, H*W % 32 != 0",
    "fwd pass bits, H*W % 32 != 0", "fwd pass bits, whole words", "fwd pass bits, shared word per entry",
    "wgrad channel split, ragged", "wgrad channel split, even", "wgrad ragged channel split at CC 16",
    "wgrad ragged channel split at CC 32", "wgrad tap groups", "wgrad Gb > 1", "wgrad TB > 1", "wgrad ranks = 1",
    "wgrad ranks > 1", "wgrad CC 16", "wgrad CC 32", "wgrad nbuf 1", "wgrad nbuf 2",
}
