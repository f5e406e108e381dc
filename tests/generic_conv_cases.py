"""Geometries of the generic implicit-GEMM convolution kernels (mnb_conv_generic.cu), shared by the host-side plan test
(test_generic_conv_plan_cpu.py) and the fp64 comparison on the GPU (test_gpu_generic_conv.py).

Each case: (B, C, H, W, K, (R, S), (sh, sw), (ph, pw), (dh, dw), G).  Together they reach every template instance of the
three kernels, every cap of the split-K weight-gradient plan and both tile edges; test_generic_conv_plan_cpu.py checks
that they still do."""

CASES = {
    # packed-operand family refuses stride 2 on odd images; Ng = 96 needs two BN-64 column tiles
    "s2_odd": (2, 64, 15, 15, 96, (3, 3), (2, 2), (1, 1), (1, 1), 1),
    "dilation2": (3, 48, 16, 12, 40, (3, 3), (1, 1), (2, 2), (2, 2), 1),
    # dx has positions no output reads: they must be exactly 0
    "stride3": (2, 32, 20, 20, 32, (3, 3), (3, 3), (0, 0), (1, 1), 1),
    # unequal strides, padding wider than the filter, dilation in one direction
    "mixed": (2, 24, 9, 13, 20, (3, 5), (2, 1), (3, 0), (1, 2), 1),
    # Cg = 10, Ng = 15
    "grouped_1x7": (2, 30, 17, 11, 45, (1, 7), (1, 1), (0, 3), (1, 1), 3),
    # grid.z = 64
    "depthwise": (2, 64, 14, 14, 64, (3, 3), (1, 1), (1, 1), (1, 1), 64),
    # 10-way head on a [B, C, 1, 1] view (F.linear): M = 33 < BM
    "head": (33, 512, 1, 1, 10, (1, 1), (1, 1), (0, 0), (1, 1), 1),
    # ImageNet stem: outside the fp32 tensor-core cover
    "stem7x7": (1, 3, 224, 224, 64, (7, 7), (2, 2), (3, 3), (1, 1), 1),
    # weight gradient: Cg*R*S = 27 takes the BN-32 instance; stride 2 and dilation 2 on an odd RGB image
    "rgb_s2_d2": (2, 3, 17, 17, 16, (3, 3), (2, 2), (2, 2), (2, 2), 1),
    # weight gradient runs 256 splits
    "split_cap256": (64, 1, 32, 32, 10, (3, 3), (1, 1), (1, 1), (1, 1), 1),
    # Kd = 507 in 3 splits of 176, 176 and 155 (the Kd / 128 cap)
    "split_ragged": (3, 16, 13, 13, 16, (3, 3), (1, 1), (1, 1), (1, 1), 1),
    # Kd = 16: one split
    "split_single": (1, 64, 8, 8, 256, (3, 3), (2, 2), (1, 1), (1, 1), 1),
}


def out_hw(case):
    B, C, H, W, K, (R, S), (sh, sw), (ph, pw), (dh, dw), G = case
    return (H + 2 * ph - dh * (R - 1) - 1) // sh + 1, (W + 2 * pw - dw * (S - 1) - 1) // sw + 1


def conv_shape(case):
    """the mnb_conv_shape of a case"""
    from micronet_b200 import _lib as L
    B, C, H, W, K, (R, S), (sh, sw), (ph, pw), (dh, dw), G = case
    return L.ConvShape(B, C, H, W, K, R, S, sh, sw, ph, pw, dh, dw, G)
