"""One case list for the two binary forward convolutions of frozen wbwtab inference: the XNOR-popcount kernel
(csrc/mnb_xnor.cu) and the binary tensor-core kernel (csrc/mnb_b1.cu).

Each case names the kernel, the conv shape (B, C, H, W, K, R, stride, pad, groups), an optional sign epilogue (the
consumer's format, groups, channel shuffle, 2x2 pool, BatchNorm) and the launch plan it was written for, as returned by
``xnor.plan`` / ``b1.plan`` (the launchers' own plan functions).  tests/test_binary_conv_coverage_cpu.py checks on the host
that the list launches every kernel instance, reaches every plan feature below and every conv of the frozen NIN, NIN-GC and
pruned NIN-GC graphs, and that each plan is still the pinned one; tests/test_gpu_binary_conv_plans.py runs every case
against fp64 and the other forward kernels.

Every case also runs the forward without an epilogue at its shape (the fp32 output the epilogue is checked against), so
a post case launches two instances: (.., POST = False) and (.., POST = True)."""
from collections import namedtuple

from micronet_b200 import _lib as L

Post = namedtuple("Post", "fmt og sg pool bn")        # fmt: "bits" | "bf16" | "b1"; og: the consumer's groups
Case = namedtuple("Case", "id kernel shape post plan")

FMT = {"bits": L.XNOR_BITS, "bf16": L.XNOR_PM1_BF16, "b1": L.XNOR_B1_PLANE}

# the instances each kernel can launch (mnb_xnor.cu pick(), mnb_b1.cu kNt)
XNOR_RNW = [(1, 1), (1, 2), (1, 3), (1, 4), (1, 8), (3, 1), (3, 2), (3, 4), (5, 1), (5, 2)]
XNOR_INSTANCES = [(r, nw, border, post) for r, nw in XNOR_RNW for border in (0, 1) for post in (0, 1)]
B1_NT = [32, 64, 128, 192]
B1_INSTANCES = [(nt, post) for nt in B1_NT for post in (0, 1)]


def _x(id, shape, post, plan):
    return Case(id, "xnor", shape, post, plan)


def _b(id, shape, post, plan):
    return Case(id, "b1", shape, post, plan)


P = Post
# XNOR plan fields: R, NW, border, px, post, ksplit, kb, pblocks, smem, refused
# b1 plan fields:   Nt, n_ntiles, u, ksteps, G, col_tiles, Wt, BW, TH, TB, row_tiles, n_mtiles, TG, ntg, nstage, post, smem
CASES = [
    # ---- XNOR: every (R, NW) without / with border, without / with the sign epilogue ----------------------------------------
    # 1x1, NW 1: full words; odd pixel count at two pixels per thread; 1x1 with padding 1 is the border variant
    _x("x1w1", (2, 32, 9, 9, 45, 1, 1, 0, 1), None, (1, 1, 0, 2, 0, 6, 8, 1, 512, 0)),
    _x("x1w1_pad1_oddpix", (1, 32, 9, 9, 45, 1, 1, 1, 1), None, (1, 1, 1, 2, 0, 6, 8, 1, 512, 0)),
    _x("x1w1_bits_og3", (2, 32, 8, 8, 48, 1, 1, 0, 1), P("bits", 3, 1, False, False), (1, 1, 0, 2, 1, 6, 8, 1, 640, 0)),
    _x("x1w1_pad1_bf16_bn", (2, 32, 6, 6, 40, 1, 1, 1, 1), P("bf16", 1, 1, False, True), (1, 1, 1, 2, 1, 5, 8, 1, 640, 0)),
    # 1x1, NW 2 (48 channels per group: ragged second word); stride 2
    _x("x1w2_s2", (2, 96, 9, 9, 36, 1, 2, 0, 2), None, (1, 2, 0, 2, 0, 3, 6, 1, 384, 0)),
    _x("x1w2_pad1", (3, 96, 7, 7, 36, 1, 1, 1, 2), None, (1, 2, 1, 2, 0, 3, 6, 1, 384, 0)),
    _x("x1w2_bits_pool_bn", (2, 96, 8, 8, 60, 1, 1, 0, 2), P("bits", 2, 1, True, True), (1, 2, 0, 2, 1, 4, 8, 1, 640, 0)),
    _x("x1w2_pad1_bits_shuffle", (2, 96, 6, 6, 72, 1, 1, 1, 2), P("bits", 4, 3, False, True),
        (1, 2, 1, 2, 1, 5, 8, 1, 640, 0)),
    # 1x1, NW 3: the pruned NIN-GC's 77 / 81 / 76 / 80 channels per group
    _x("x1w3", (2, 154, 9, 9, 162, 1, 1, 0, 2), None, (1, 3, 0, 2, 0, 9, 9, 1, 576, 0)),
    _x("x1w3_pad1", (2, 154, 5, 7, 46, 1, 1, 1, 2), None, (1, 3, 1, 2, 0, 3, 8, 1, 512, 0)),
    _x("x1w3_bits_og16_pool_shuffle", (2, 162, 8, 8, 144, 1, 1, 0, 2), P("bits", 16, 2, True, True),
        (1, 3, 0, 2, 1, 9, 8, 1, 640, 0)),
    _x("x1w3_pad1_bf16_shuffle", (2, 160, 6, 6, 88, 1, 1, 1, 2), P("bf16", 1, 4, False, False),
        (1, 3, 1, 2, 1, 5, 9, 1, 720, 0)),
    # 1x1, NW 4
    _x("x1w4", (2, 128, 9, 9, 100, 1, 1, 0, 1), None, (1, 4, 0, 2, 0, 12, 9, 1, 576, 0)),
    _x("x1w4_pad1", (1, 128, 8, 9, 20, 1, 1, 1, 1), None, (1, 4, 1, 2, 0, 3, 7, 1, 448, 0)),
    _x("x1w4_bits_og5", (3, 256, 8, 8, 120, 1, 1, 0, 2), P("bits", 5, 1, False, True), (1, 4, 0, 2, 1, 7, 9, 1, 720, 0)),
    _x("x1w4_pad1_bits_pool", (2, 128, 6, 6, 64, 1, 1, 1, 1), P("bits", 2, 2, True, False),
        (1, 4, 1, 2, 1, 8, 8, 1, 640, 0)),
    # 1x1, NW 8 (250 channels: ragged eighth word)
    _x("x1w8", (2, 250, 9, 9, 30, 1, 1, 0, 1), None, (1, 8, 0, 2, 0, 4, 8, 1, 768, 0)),
    _x("x1w8_pad1", (1, 250, 7, 7, 27, 1, 1, 1, 1), None, (1, 8, 1, 2, 0, 4, 7, 1, 672, 0)),
    _x("x1w8_bits", (2, 250, 8, 8, 66, 1, 1, 0, 1), P("bits", 3, 1, False, True), (1, 8, 0, 2, 1, 8, 9, 1, 1008, 0)),
    _x("x1w8_pad1_bf16", (2, 256, 6, 6, 24, 1, 1, 1, 1), P("bf16", 1, 1, False, True), (1, 8, 1, 2, 1, 3, 8, 1, 896, 0)),
    # 3x3, NW 1 (9 channels per group, 16 groups); 'valid' 3x3 is the border-free variant
    _x("x3w1", (2, 144, 9, 9, 80, 3, 1, 0, 16), None, (3, 1, 0, 1, 0, 1, 5, 1, 880, 0)),
    _x("x3w1_pad1", (2, 144, 8, 8, 304, 3, 1, 1, 16), None, (3, 1, 1, 1, 0, 3, 7, 1, 1232, 0)),
    _x("x3w1_bits_pool", (2, 144, 10, 10, 304, 3, 1, 0, 16), P("bits", 4, 16, True, True),
        (3, 1, 0, 1, 1, 3, 7, 1, 1344, 0)),
    _x("x3w1_pad1_bits_og8", (2, 320, 8, 8, 608, 3, 1, 1, 32), P("bits", 8, 32, False, True),
        (3, 1, 1, 1, 1, 3, 7, 1, 1344, 0)),
    # 3x3, NW 2; stride 2 on an odd plane
    _x("x3w2", (2, 80, 9, 9, 36, 3, 1, 0, 2), None, (3, 2, 0, 1, 0, 3, 6, 1, 1440, 0)),
    _x("x3w2_s2_pad1", (2, 80, 15, 13, 40, 3, 2, 1, 2), None, (3, 2, 1, 1, 0, 3, 7, 1, 1680, 0)),
    _x("x3w2_bits_og6", (2, 80, 10, 10, 36, 3, 1, 0, 2), P("bits", 6, 1, False, False), (3, 2, 0, 1, 1, 3, 6, 1, 1536, 0)),
    _x("x3w2_pad1_bf16_shuffle_bn", (2, 80, 8, 8, 48, 3, 1, 1, 2), P("bf16", 1, 2, False, True),
        (3, 2, 1, 1, 1, 3, 8, 1, 2048, 0)),
    # 3x3, NW 4; padding wider than R / 2
    _x("x3w4", (2, 100, 9, 9, 21, 3, 1, 0, 1), None, (3, 4, 0, 1, 0, 3, 7, 1, 2576, 0)),
    _x("x3w4_pad2", (2, 128, 7, 7, 64, 3, 1, 2, 1), None, (3, 4, 1, 1, 0, 8, 8, 1, 2944, 0)),
    _x("x3w4_bits", (2, 100, 10, 10, 50, 3, 1, 0, 1), P("bits", 2, 5, True, True), (3, 4, 0, 1, 1, 6, 9, 1, 3456, 0)),
    _x("x3w4_pad1_bits_og3", (1, 100, 8, 8, 51, 3, 1, 1, 1), P("bits", 3, 1, False, True),
        (3, 4, 1, 1, 1, 6, 9, 1, 3456, 0)),
    # 5x5, NW 1 and 2
    _x("x5w1", (2, 24, 9, 9, 20, 5, 1, 0, 1), None, (5, 1, 0, 1, 0, 3, 7, 1, 2688, 0)),
    _x("x5w1_pad2", (2, 24, 9, 9, 20, 5, 1, 2, 1), None, (5, 1, 1, 1, 0, 3, 7, 1, 2688, 0)),
    _x("x5w1_bits_pool", (2, 24, 12, 12, 40, 5, 1, 0, 1), P("bits", 1, 1, True, True), (5, 1, 0, 1, 1, 5, 8, 1, 3200, 0)),
    _x("x5w1_pad3_bits", (2, 24, 6, 6, 40, 5, 1, 3, 1), P("bits", 2, 2, False, False), (5, 1, 1, 1, 1, 5, 8, 1, 3200, 0)),
    _x("x5w2", (2, 96, 9, 9, 30, 5, 1, 0, 2), None, (5, 2, 0, 1, 0, 2, 8, 1, 4608, 0)),
    _x("x5w2_pad2", (2, 96, 8, 8, 192, 5, 1, 2, 2), None, (5, 2, 1, 1, 0, 11, 9, 1, 5184, 0)),
    _x("x5w2_bf16", (2, 96, 12, 12, 40, 5, 1, 0, 2), P("bf16", 1, 1, False, True), (5, 2, 0, 1, 1, 3, 7, 1, 4144, 0)),
    _x("x5w2_pad2_bits_og3", (2, 96, 8, 8, 42, 5, 1, 2, 2), P("bits", 3, 2, False, True), (5, 2, 1, 1, 1, 3, 7, 1, 4144, 0)),

    # ---- b1: every N tile without / with the epilogue, the epilogue's three formats at every N tile -------------------------
    # Nt 32 (up to 16 output channels per group)
    _b("b32_partial_unit", (2, 70, 9, 13, 12, 3, 1, 1, 1), None, (32, 1, 2, 1, 1, 1, 13, 15, 8, 1, 2, 4, 9, 1, 4, 0, 59008)),
    _b("b32_b1_oddu_g2_tb", (2, 40, 8, 8, 16, 1, 1, 0, 2), P("b1", 2, 1, False, True),
        (32, 1, 1, 1, 2, 1, 8, 8, 8, 2, 1, 1, 1, 1, 4, 1, 49152)),
    _b("b32_bits_pool", (3, 64, 10, 10, 16, 3, 1, 1, 1), P("bits", 1, 1, True, True),
        (32, 1, 1, 1, 1, 1, 10, 12, 10, 1, 1, 3, 9, 1, 4, 1, 57984)),
    _b("b32_bf16_shuffle", (2, 96, 9, 9, 16, 3, 1, 1, 1), P("bf16", 1, 2, False, True),
        (32, 1, 2, 1, 1, 1, 9, 11, 9, 1, 1, 2, 9, 1, 4, 1, 55296)),
    # Nt 64 (17 - 32 channels); 150 channels per group: three units, the third k-step's second unit the next group's
    _b("b64_oddu_g2_cols_1x1", (2, 300, 3, 130, 48, 1, 1, 0, 2), None,
        (64, 1, 3, 2, 2, 4, 33, 33, 3, 1, 1, 8, 1, 1, 4, 0, 49152)),
    _b("b64_b1_5x5_ragged_taps", (2, 64, 12, 12, 32, 5, 1, 2, 1), P("b1", 2, 2, True, True),
        (64, 1, 1, 1, 1, 1, 12, 16, 8, 1, 2, 4, 13, 2, 4, 1, 134400)),
    _b("b64_bits_cols_3x3", (1, 130, 4, 140, 30, 3, 1, 1, 1), P("bits", 3, 1, False, True),
        (64, 1, 3, 2, 1, 5, 28, 30, 4, 1, 1, 5, 9, 1, 4, 1, 99968)),
    _b("b64_bf16", (2, 192, 8, 8, 32, 1, 1, 0, 1), P("bf16", 1, 1, False, False),
        (64, 1, 3, 2, 1, 1, 8, 8, 8, 2, 1, 1, 1, 1, 4, 1, 49152)),
    # Nt 128 (33 - 64 channels); 7x7 in five tap groups, the last ragged
    _b("b128_7x7", (1, 192, 7, 7, 64, 7, 1, 3, 1), None, (128, 1, 3, 2, 1, 1, 7, 13, 7, 1, 1, 1, 10, 5, 4, 0, 189440)),
    _b("b128_b1_g2", (2, 130, 9, 13, 66, 3, 1, 1, 2), P("b1", 3, 1, False, True),
        (128, 1, 2, 1, 2, 1, 13, 15, 8, 1, 2, 4, 9, 1, 4, 1, 169600)),
    _b("b128_bits_og3", (2, 192, 8, 8, 120, 1, 1, 0, 2), P("bits", 3, 4, True, True),
        (128, 1, 2, 1, 2, 1, 8, 8, 8, 2, 1, 1, 1, 1, 4, 1, 49152)),
    _b("b128_bf16_shuffle", (2, 160, 8, 8, 64, 3, 1, 1, 1), P("bf16", 1, 4, False, True),
        (128, 1, 3, 2, 1, 1, 8, 10, 8, 1, 1, 2, 9, 1, 4, 1, 162816)),
    # Nt 192 (65 - 96 channels, and several N tiles beyond)
    _b("b192_ntiles3", (2, 64, 8, 8, 200, 1, 1, 0, 1), None, (192, 3, 1, 1, 1, 1, 8, 8, 8, 2, 1, 1, 1, 1, 4, 0, 49152)),
    _b("b192_b1_og3_pool", (2, 192, 8, 8, 180, 3, 1, 1, 1), P("b1", 3, 3, True, True),
        (192, 2, 3, 2, 1, 1, 8, 10, 8, 1, 1, 2, 5, 2, 4, 1, 138240)),
    _b("b192_bits_ntiles2", (2, 96, 8, 8, 192, 1, 1, 0, 1), P("bits", 4, 1, False, True),
        (192, 2, 2, 1, 1, 1, 8, 8, 8, 2, 1, 1, 1, 1, 4, 1, 49152)),
    _b("b192_bf16_5x5", (2, 96, 8, 8, 160, 5, 1, 2, 1), P("bf16", 1, 1, False, True),
        (192, 2, 2, 1, 1, 1, 8, 12, 8, 1, 1, 2, 7, 4, 4, 1, 193536)),
    # pipeline depth: two and three stages (the wide 7x7 boxes), four everywhere else
    _b("b192_7x7_two_stages", (1, 64, 1, 122, 96, 7, 1, 3, 1), None,
        (192, 1, 1, 1, 1, 1, 122, 128, 1, 1, 1, 1, 7, 7, 2, 0, 157952)),
    _b("b128_7x7_three_stages", (1, 64, 4, 60, 64, 7, 1, 3, 1), None,
        (128, 1, 1, 1, 1, 1, 60, 66, 2, 1, 2, 2, 10, 5, 3, 0, 182272)),
]

# ---- every binarized conv of the frozen NIN, NIN-GC and README-cfg pruned NIN-GC graphs (wbwtab.freeze_inference of the
# fuse_bn QAT graph), at batch 256 and 4: (model, layer, (C, H, W, K, R, pad, G), post)
MODEL_LAYERS = [
    ("nin", "L1", (192, 32, 32, 160, 1, 0, 1), P("b1", 1, 1, False, True)),
    ("nin", "L2", (160, 32, 32, 96, 1, 0, 1), P("b1", 1, 1, False, True)),
    ("nin", "L3", (96, 16, 16, 192, 5, 2, 1), P("b1", 1, 1, False, True)),
    ("nin", "L4", (192, 16, 16, 192, 1, 0, 1), P("b1", 1, 1, False, True)),
    ("nin", "L5", (192, 16, 16, 192, 1, 0, 1), P("b1", 1, 1, False, True)),
    ("nin", "L6", (192, 8, 8, 192, 3, 1, 1), P("b1", 1, 1, False, True)),
    ("nin", "L7", (192, 8, 8, 192, 1, 0, 1), P("bf16", 1, 1, False, True)),
    ("nin_gc", "L1", (256, 32, 32, 256, 1, 0, 2), P("bits", 2, 2, False, True)),
    ("nin_gc", "L2", (256, 32, 32, 256, 1, 0, 2), P("bits", 16, 2, True, True)),
    ("nin_gc", "L3", (256, 16, 16, 512, 3, 1, 16), P("bits", 4, 16, False, True)),
    ("nin_gc", "L4", (512, 16, 16, 512, 1, 0, 4), P("bits", 4, 4, False, True)),
    ("nin_gc", "L5", (512, 16, 16, 512, 1, 0, 4), P("bits", 32, 4, True, True)),
    ("nin_gc", "L6", (512, 8, 8, 1024, 3, 1, 32), P("bits", 8, 32, False, True)),
    ("nin_gc", "L7", (1024, 8, 8, 1024, 1, 0, 8), P("bf16", 1, 1, False, True)),
    ("pruned", "L1", (154, 32, 32, 162, 1, 0, 2), P("bits", 2, 2, False, True)),
    ("pruned", "L2", (162, 32, 32, 144, 1, 0, 2), P("bits", 16, 2, True, True)),
    ("pruned", "L3", (144, 16, 16, 304, 3, 1, 16), P("bits", 4, 16, False, True)),
    ("pruned", "L4", (304, 16, 16, 320, 1, 0, 4), P("bits", 4, 4, False, True)),
    ("pruned", "L5", (320, 16, 16, 320, 1, 0, 4), P("bits", 32, 4, True, True)),
    ("pruned", "L6", (320, 8, 8, 608, 3, 1, 32), P("bits", 8, 32, False, True)),
    ("pruned", "L7", (608, 8, 8, 584, 1, 0, 8), P("bf16", 1, 1, False, True)),
]
MODEL_KERNEL = {"nin": "b1", "nin_gc": "xnor", "pruned": "xnor"}
MODEL_BATCHES = (256, 4)
MODEL_PLANS = {
    ('nin', 'L1', 256): (192, 2, 3, 2, 1, 1, 32, 32, 4, 1, 8, 2048, 1, 1, 4, 1, 49152),
    ('nin', 'L2', 256): (192, 1, 3, 2, 1, 1, 32, 32, 4, 1, 8, 2048, 1, 1, 4, 1, 49152),
    ('nin', 'L3', 256): (192, 2, 2, 1, 1, 1, 16, 20, 6, 1, 3, 768, 7, 4, 4, 1, 201216),
    ('nin', 'L4', 256): (192, 2, 3, 2, 1, 1, 16, 16, 8, 1, 2, 512, 1, 1, 4, 1, 49152),
    ('nin', 'L5', 256): (192, 2, 3, 2, 1, 1, 16, 16, 8, 1, 2, 512, 1, 1, 4, 1, 49152),
    ('nin', 'L6', 256): (192, 2, 3, 2, 1, 1, 8, 10, 8, 1, 1, 256, 5, 2, 4, 1, 138240),
    ('nin', 'L7', 256): (192, 2, 3, 2, 1, 1, 8, 8, 8, 2, 1, 128, 1, 1, 4, 1, 49152),
    ('nin_gc', 'L1', 256): (1, 4, 0, 2, 1, 1, 128, 512, 10240, 0),
    ('nin_gc', 'L2', 256): (1, 4, 0, 2, 1, 1, 128, 512, 10240, 0),
    ('nin_gc', 'L3', 256): (3, 1, 1, 1, 1, 1, 32, 256, 6144, 0),
    ('nin_gc', 'L4', 256): (1, 4, 0, 2, 1, 2, 64, 128, 5120, 0),
    ('nin_gc', 'L5', 256): (1, 4, 0, 2, 1, 2, 64, 128, 5120, 0),
    ('nin_gc', 'L6', 256): (3, 1, 1, 1, 1, 1, 32, 64, 6144, 0),
    ('nin_gc', 'L7', 256): (1, 4, 0, 2, 1, 3, 43, 32, 3440, 0),
    ('pruned', 'L1', 256): (1, 3, 0, 2, 1, 1, 81, 512, 6480, 0),
    ('pruned', 'L2', 256): (1, 3, 0, 2, 1, 1, 72, 512, 5760, 0),
    ('pruned', 'L3', 256): (3, 1, 1, 1, 1, 1, 19, 256, 3648, 0),
    ('pruned', 'L4', 256): (1, 3, 0, 2, 1, 2, 40, 128, 3200, 0),
    ('pruned', 'L5', 256): (1, 3, 0, 2, 1, 2, 40, 128, 3200, 0),
    ('pruned', 'L6', 256): (3, 1, 1, 1, 1, 1, 19, 64, 3648, 0),
    ('pruned', 'L7', 256): (1, 3, 0, 2, 1, 3, 25, 32, 2000, 0),
    ('nin', 'L1', 4): (192, 2, 3, 2, 1, 1, 32, 32, 4, 1, 8, 32, 1, 1, 4, 1, 49152),
    ('nin', 'L2', 4): (192, 1, 3, 2, 1, 1, 32, 32, 4, 1, 8, 32, 1, 1, 4, 1, 49152),
    ('nin', 'L3', 4): (192, 2, 2, 1, 1, 1, 16, 20, 6, 1, 3, 12, 7, 4, 4, 1, 201216),
    ('nin', 'L4', 4): (192, 2, 3, 2, 1, 1, 16, 16, 8, 1, 2, 8, 1, 1, 4, 1, 49152),
    ('nin', 'L5', 4): (192, 2, 3, 2, 1, 1, 16, 16, 8, 1, 2, 8, 1, 1, 4, 1, 49152),
    ('nin', 'L6', 4): (192, 2, 3, 2, 1, 1, 8, 10, 8, 1, 1, 4, 5, 2, 4, 1, 138240),
    ('nin', 'L7', 4): (192, 2, 3, 2, 1, 1, 8, 8, 8, 2, 1, 2, 1, 1, 4, 1, 49152),
    ('nin_gc', 'L1', 4): (1, 4, 0, 2, 1, 15, 9, 8, 720, 0),
    ('nin_gc', 'L2', 4): (1, 4, 0, 2, 1, 15, 9, 8, 720, 0),
    ('nin_gc', 'L3', 4): (3, 1, 1, 1, 1, 4, 8, 4, 1536, 0),
    ('nin_gc', 'L4', 4): (1, 4, 0, 2, 1, 15, 9, 2, 720, 0),
    ('nin_gc', 'L5', 4): (1, 4, 0, 2, 1, 15, 9, 2, 720, 0),
    ('nin_gc', 'L6', 4): (3, 1, 1, 1, 1, 4, 8, 1, 1536, 0),
    ('nin_gc', 'L7', 4): (1, 4, 0, 2, 1, 15, 9, 1, 720, 0),
    ('pruned', 'L1', 4): (1, 3, 0, 2, 1, 9, 9, 8, 720, 0),
    ('pruned', 'L2', 4): (1, 3, 0, 2, 1, 9, 8, 8, 640, 0),
    ('pruned', 'L3', 4): (3, 1, 1, 1, 1, 3, 7, 4, 1344, 0),
    ('pruned', 'L4', 4): (1, 3, 0, 2, 1, 9, 9, 2, 720, 0),
    ('pruned', 'L5', 4): (1, 3, 0, 2, 1, 9, 9, 2, 720, 0),
    ('pruned', 'L6', 4): (3, 1, 1, 1, 1, 3, 7, 1, 1344, 0),
    ('pruned', 'L7', 4): (1, 3, 0, 2, 1, 9, 9, 1, 720, 0),
}

CASES += [Case(f"{m}_{layer}_b{B}", MODEL_KERNEL[m], (B, c, h, w, k, r, 1, pad, g), post, MODEL_PLANS[(m, layer, B)])
          for B in MODEL_BATCHES for m, layer, (c, h, w, k, r, pad, g), post in MODEL_LAYERS]


# ---- host-side helpers shared by the coverage and GPU tests
def conv_shape(shape):
    B, Cc, H, W, K, R, st, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def out_hw(shape):
    B, Cc, H, W, K, R, st, pad, G = shape
    return (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1


def post_struct(post, bn=None):
    """mnb_xnor_post of a case's epilogue; ``bn``: the four [K] device tensors when post.bn"""
    from micronet_b200 import xnor as X
    return X.post_struct(FMT[post.fmt], post.og, post.sg, post.pool, bn if post.bn else None)


def plan_of(kernel, shape, post=None):
    """the plan dict the kernel's launcher uses for this shape (None outside the cover)"""
    from micronet_b200 import b1 as B1, xnor as X
    K = X if kernel == "xnor" else B1
    return K.plan(conv_shape(shape), None if post is None else post_struct(post))


def plan_tuple(kernel, plan):
    from micronet_b200 import b1 as B1, xnor as X
    return tuple(plan[f] for f in (X if kernel == "xnor" else B1).PLAN_FIELDS)


def launches(case):
    """[(kernel, plan)] of every launch a case makes: the plain forward, and the epilogue's if it has one"""
    out = [(case.kernel, plan_of(case.kernel, case.shape))]
    if case.post is not None:
        out.append((case.kernel, plan_of(case.kernel, case.shape, case.post)))
    return out


def instance(kernel, plan):
    if kernel == "xnor":
        return (plan["R"], plan["NW"], plan["border"], plan["post"])
    return (plan["Nt"], plan["post"])


def _xnor_dest_units(K, post):
    """destination unit (bit-plane word of the consumer's group, or bf16 octet) of every producer channel"""
    cpg = K // post.sg
    out = []
    for c in range(K):
        cd = (c % cpg) * post.sg + c // cpg if post.sg > 1 else c
        if post.fmt == "bf16":
            out.append(cd >> 3)
        else:
            ocg = K // post.og
            out.append((cd // ocg) * ((ocg + 31) // 32) + (cd % ocg) // 32)
    return out


def features(case, plan):
    """the plan features (names) this launch of a case reaches"""
    B, Cc, H, W, K, R, st, pad, G = case.shape
    P_, Q_ = out_hw(case.shape)
    cin_g, cout_g = Cc // G, K // G
    post = case.post if plan["post"] else None
    f = set()
    if case.kernel == "xnor":
        if st == 2:
            f.add("xnor stride 2")
        if R > 1 and pad > R // 2:
            f.add("xnor padding wider than R/2")
        if plan["px"] == 2 and (B * P_ * Q_) % 2:
            f.add("xnor px 2, odd pixel count")
        if plan["ksplit"] > 1 and cout_g % plan["kb"]:
            f.add("xnor ragged last k-slice")
        if post is not None:
            if post.fmt == "bits" and (K // post.og) % 32:
                f.add("xnor bits, consumer group not a multiple of 32")
            if post.fmt == "bf16":
                f.add("xnor bf16 with shuffle" if post.sg > 1 else "xnor bf16 without shuffle")
            if post.pool:
                f.add("xnor 2x2 pool")
            if post.bn:
                f.add("xnor BatchNorm")
            if plan["ksplit"] > 1:
                units = _xnor_dest_units(K, post)
                writers = {}
                for c in range(K):
                    writers.setdefault((c // cout_g, units[c]), set()).add((c % cout_g) // plan["kb"])
                if any(len(s) > 1 for s in writers.values()):
                    f.add(f"xnor {post.fmt}: one destination unit written by several k-slices")
    else:
        if plan["n_ntiles"] > 1:
            f.add("b1 several N tiles")
        if plan["col_tiles"] > 1:
            f.add(f"b1 several column tiles, {R}x{R}")
        if plan["TB"] > 1:
            f.add("b1 several images per M tile")
        if plan["ntg"] > 1 and (R * R) % plan["TG"]:
            f.add("b1 ragged last tap group")
        if plan["u"] % 2 and G > 1:
            f.add("b1 odd units per group, G > 1")
        if cin_g % 64:
            f.add("b1 partial last unit")
        f.add(f"b1 {plan['nstage']} pipeline stages")
        if post is not None:
            f.add(f"b1 {post.fmt} at Nt {plan['Nt']}")
            if post.pool:
                f.add("b1 2x2 pool")
            if post.sg > 1:
                f.add("b1 shuffle")
            if post.bn:
                f.add("b1 BatchNorm")
    return f


WANTED_FEATURES = {
    "xnor stride 2", "xnor padding wider than R/2", "xnor px 2, odd pixel count", "xnor ragged last k-slice",
    "xnor bits, consumer group not a multiple of 32", "xnor bf16 with shuffle", "xnor bf16 without shuffle",
    "xnor 2x2 pool", "xnor BatchNorm", "xnor bits: one destination unit written by several k-slices",
    "xnor bf16: one destination unit written by several k-slices",
    "b1 several N tiles", "b1 several column tiles, 1x1", "b1 several column tiles, 3x3", "b1 several images per M tile",
    "b1 ragged last tap group", "b1 odd units per group, G > 1", "b1 partial last unit",
    "b1 2 pipeline stages", "b1 3 pipeline stages", "b1 4 pipeline stages",
    "b1 2x2 pool", "b1 shuffle", "b1 BatchNorm",
} | {f"b1 {fmt} at Nt {nt}" for fmt in ("bits", "bf16", "b1") for nt in B1_NT}
