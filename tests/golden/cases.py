"""Case tables shared by ``make_golden.py`` (reference side) and
the parity tests (oracle / CUDA side).  Pure data + a seeded input generator."""
import torch


def make_input(case, step):
    g = torch.Generator().manual_seed(case["seed"] * 101 + step)
    shape = case["x_shape"]
    kind = case.get("x_kind", "randn")
    if kind == "pm1":  # binarised activations, as produced by wbwtab's ActivationQuantizer
        return (torch.randint(0, 2, shape, generator=g).float() * 2 - 1)
    x = torch.randn(shape, generator=g) * case.get("x_gain", 1.0)
    if kind == "relu":  # post-BN-ReLU statistics
        x = torch.relu(x)
    # later steps drift in range so EMA / running-min-max observers are exercised
    return x * (1.0 + 0.25 * step)


def _c(name, scheme, kind, args, kwargs, x_shape, seed, train_steps=2, eval_steps=1, **extra):
    d = dict(name=name, scheme=scheme, kind=kind, args=list(args), kwargs=dict(kwargs),
             x_shape=list(x_shape), seed=seed, train_steps=train_steps, eval_steps=eval_steps)
    d.update(extra)
    return d


LAYER_CASES = [
    # ---- DoReFa (DF:76-199) -------------------------------------------------
    _c("dorefa_w8a8_3x3", "dorefa", "conv", (8, 12, 3), dict(padding=1, a_bits=8, w_bits=8),
       (2, 8, 9, 9), 1, x_gain=4.0, weight_gain=3.0),
    _c("dorefa_w4a4_1x1_g2", "dorefa", "conv", (8, 16, 1), dict(groups=2, a_bits=4, w_bits=4),
       (3, 8, 8, 8), 2, x_gain=4.0, x_kind="relu", weight_gain=3.0),
    _c("dorefa_w2a2_5x5_s2", "dorefa", "conv", (4, 6, 5), dict(stride=2, padding=2, a_bits=2, w_bits=2, bias=False),
       (2, 4, 11, 11), 3, x_gain=5.0, weight_gain=4.0),
    _c("dorefa_w8a32", "dorefa", "conv", (4, 6, 3), dict(padding=1, a_bits=32, w_bits=8),
       (2, 4, 6, 6), 4, weight_gain=2.0),
    _c("dorefa_linear_w8a8", "dorefa", "linear", (20, 7), dict(a_bits=8, w_bits=8),
       (5, 20), 5, x_gain=4.0, weight_gain=3.0),
    # ---- wbwtab (WB:152-195) --------------------------------------------------
    _c("wb_ternary_pm1_3x3_g4", "wbwtab", "conv", (16, 8, 3), dict(padding=1, groups=4, W=3),
       (2, 16, 8, 8), 6, x_kind="pm1"),
    _c("wb_binary_pm1_1x1_g2", "wbwtab", "conv", (8, 8, 1), dict(groups=2, W=2),
       (2, 8, 8, 8), 7, x_kind="pm1", weight_gain=6.0),
    _c("wb_ternary_fp32_3x3", "wbwtab", "conv", (6, 8, 3), dict(padding=1, W=3, bias=False),
       (2, 6, 7, 7), 8),
    _c("wb_binary_fp32_5x5", "wbwtab", "conv", (3, 4, 5), dict(padding=2, W=2),
       (2, 3, 8, 8), 9, weight_gain=8.0),
    _c("wb_w32", "wbwtab", "conv", (4, 4, 3), dict(padding=1, W=32),
       (2, 4, 6, 6), 10),
    # ---- IAO (IAO:325-507, 997-1157) -----------------------------------------------
    _c("iao_sym_pc_minmax", "iao", "conv", (8, 12, 3), dict(padding=1, q_type=0, q_level=0, weight_observer=0),
       (2, 8, 9, 9), 11, train_steps=3),
    _c("iao_sym_pl_ema", "iao", "conv", (8, 8, 1), dict(groups=2, q_type=0, q_level=1, weight_observer=1),
       (2, 8, 8, 8), 12, train_steps=3, x_kind="relu"),
    _c("iao_asym_pc_minmax", "iao", "conv", (6, 8, 3), dict(padding=1, stride=2, q_type=1, q_level=0, weight_observer=0),
       (2, 6, 9, 9), 13, train_steps=3),
    _c("iao_asym_pl_ema_relu", "iao", "conv", (6, 8, 3), dict(padding=1, q_type=1, q_level=1, weight_observer=1, bias=False),
       (2, 6, 8, 8), 14, train_steps=3, x_kind="relu"),
    _c("iao_w4a4_sym", "iao", "conv", (8, 8, 3), dict(padding=1, a_bits=4, w_bits=4),
       (2, 8, 8, 8), 15, train_steps=2),
    _c("iao_ptq", "iao", "conv", (8, 8, 3), dict(padding=1, ptq=True, percentile=0.99),
       (2, 8, 8, 8), 16, train_steps=2),
    _c("iao_linear_sym_pc", "iao", "linear", (24, 10), dict(q_type=0, q_level=0),
       (6, 24), 17, train_steps=2),
    _c("iao_linear_asym_pl", "iao", "linear", (24, 10), dict(q_type=1, q_level=1),
       (6, 24), 18, train_steps=2),
    # ---- IAO transposed conv (IAO:510-636) ---------------------------------------------
    _c("iao_convT_sym_s2", "iao", "convT", (8, 6, 3), dict(stride=2, padding=1, output_padding=1, q_type=0),
       (2, 8, 7, 7), 24, train_steps=3),
    _c("iao_convT_asym_g2_ema", "iao", "convT", (8, 12, 4), dict(stride=2, padding=1, groups=2, q_type=1, weight_observer=1),
       (2, 8, 6, 6), 25, train_steps=3, x_kind="relu"),
    _c("iao_convT_s1_nobias", "iao", "convT", (6, 8, 3), dict(padding=1, bias=False, a_bits=4, w_bits=4),
       (3, 6, 8, 8), 26, train_steps=2),
    # ---- IAO BN-fuse (IAO:652-994) ---------------------------------------------------
    _c("iao_bnfuse_sym_pc", "iao", "bnfuse", (8, 12, 3), dict(padding=1),
       (4, 8, 8, 8), 19, train_steps=3),
    _c("iao_bnfuse_bias_s2", "iao", "bnfuse", (8, 8, 3), dict(padding=1, stride=2, bias=True),
       (4, 8, 9, 9), 20, train_steps=2),
    _c("iao_bnfuse_calib", "iao", "bnfuse", (6, 8, 1), dict(bn_fuse_calib=True, pretrained_model=True),
       (4, 6, 8, 8), 21, train_steps=2),
    _c("iao_bnfuse_asym_pl", "iao", "bnfuse", (6, 8, 3), dict(padding=1, q_type=1, q_level=1),
       (4, 6, 8, 8), 22, train_steps=2),
    _c("iao_bnfuse_qaft", "iao", "bnfuse", (6, 8, 3), dict(padding=1, qaft=True),
       (4, 6, 8, 8), 23, train_steps=1, eval_steps=1),
]


MODEL_CASES = [
    dict(name="nin_gc_wb_ternary", model="nin_gc", cfg=[32, 32, 32, 64, 64, 64, 128, 128], scheme="wbwtab",
         prepare=dict(A=2, W=3), batch=4, hw=32, steps=2, seed=41, lr=0.01, wd=0.0),
    dict(name="nin_gc_wb_binary", model="nin_gc", cfg=[32, 32, 32, 64, 64, 64, 128, 128], scheme="wbwtab",
         prepare=dict(A=2, W=2), batch=4, hw=32, steps=2, seed=42, lr=0.01, wd=0.0),
    dict(name="nin_dorefa_w8a8", model="nin", cfg=[24, 20, 12, 24, 24, 24, 24, 24], scheme="dorefa",
         prepare=dict(a_bits=8, w_bits=8), batch=4, hw=32, steps=2, seed=43, lr=0.01, wd=1e-5),
    dict(name="nin_gc_dorefa_w4a4", model="nin_gc", cfg=[32, 32, 32, 64, 64, 64, 128, 128], scheme="dorefa",
         prepare=dict(a_bits=4, w_bits=4), batch=4, hw=32, steps=2, seed=44, lr=0.01, wd=1e-5),
    dict(name="resnet_iao_bnfuse", model="resnet", cfg=[4, 8, 16, 32], scheme="iao",
         prepare=dict(a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0, bn_fuse=True),
         batch=4, hw=16, steps=2, seed=45, lr=0.01, wd=1e-5),
]
