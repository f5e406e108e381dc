"""One case list for the packed-operand family's general kernels: pk_conv_kernel rows 0 (bf16), 1 (segmented) and 2 (int8)
behind mnb_pk_conv / mnb_pk_i8_conv, and pk_wgrad_kernel<Nc> + wg_reduce_kernel behind mnb_pk_wgrad.

test_pk_conv_coverage_cpu.py checks on the host that every pinned plan still holds and that the list reaches every kernel
instance, plan feature, epilogue form and refusal reason; test_gpu_pk_conv_fp64.py runs every case against fp64.

Case fields:
  mode    "fwd" (mnb_pk_conv mode 0), "dgrad" (mode 1), "i8" (mnb_pk_i8_conv), "wgrad" (mnb_pk_wgrad)
  shape   (B, C, H, W, K, R, S, stride, pad_h, pad_w, groups[, dilation])
  terms   (streamed operand, weight / x operand) pieces
  ops     "int": integer levels, one piece per operand (dgrad / wgrad: dy packed with the case's pieces, the later ones zero);
          "asym": streamed operand holds two-piece integer levels (|level| up to 383, as asymmetric IAO levels);
          "f32": split fp32 streamed operand (and fp32 weights / x where that side has more than one piece, integer levels
                 where it has one);
          "pm1": +-1 streamed operand (one exact piece) against split fp32 weights
  epi     forward: n_scale (bool), a_scale ("dev" device scalar / "const"), bias (bool);
          dgrad: gain (STE mask with this gain) or None (no mask, a_scale_const = const);
          wgrad: a_scale (bool), kdiv (bool)
  pin     plan fields (tests.pk_plan_util names) the case was written for
  env     MNB_PK_* knobs set around the plan query and the launch
  bench   the bench launch the case stands for ("" for none)
  refuse  substring of the refusal text, for a case whose launch must be refused
  maxnorm split fp32 cases: also |err| <= maxnorm * max |ref| (0: the element-wise bound alone)
"""
from collections import namedtuple

Case = namedtuple("Case", "id mode shape terms ops epi pin env bench refuse maxnorm", defaults=({}, {}, {}, "", "", 0.0))

E_FULL = dict(n_scale=True, a_scale="dev", bias=True)
E_NONE = dict(n_scale=False, a_scale="const", bias=False)
E_SCALE = dict(n_scale=True, a_scale="const", bias=False)
E_BIAS = dict(n_scale=False, a_scale="dev", bias=True)
D_STE = dict(gain=0.1)
D_CONST = dict(gain=None, const=1.0)
W_ALL = dict(a_scale=True, kdiv=True)
W_NONE = dict(a_scale=False, kdiv=False)

CASES = [
    # ---- plain bf16 forward (row 0): every N tile; R != S, pad_h != pad_w, kg % 16 != 0, ng % 16 != 0
    Case("fwd_nt16_3x1", "fwd", (2, 24, 9, 7, 16, 3, 1, 1, 1, 0, 1), (1, 1), "int", E_FULL, dict(Nt=16, segmented=0)),
    Case("fwd_nt32_1x3", "fwd", (3, 32, 12, 10, 32, 1, 3, 1, 0, 1, 1), (1, 1), "int", E_NONE, dict(Nt=32, segmented=0)),
    Case("fwd_nt48_s2", "fwd", (2, 40, 8, 8, 40, 3, 3, 2, 1, 1, 1), (1, 1), "int", E_SCALE, dict(Nt=48, segmented=0)),
    Case("fwd_nt64_mt2", "fwd", (3, 64, 28, 28, 64, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_BIAS, dict(Nt=64, MT=2, n_mtiles=21),
         {"MNB_PK_MT": "2"}),
    Case("fwd_nt96_5x3", "fwd", (2, 48, 8, 8, 80, 5, 3, 1, 2, 1, 1), (1, 1), "int", E_FULL, dict(Nt=96, segmented=0)),
    Case("fwd_nt128_ntiles", "fwd", (2, 16, 6, 6, 200, 1, 1, 1, 0, 0, 1), (1, 1), "int", E_FULL, dict(Nt=128, n_ntiles=2)),
    Case("fwd_grouped_padded", "fwd", (2, 36, 8, 8, 24, 3, 3, 1, 1, 1, 3), (1, 1), "int", E_FULL, dict(Nt=16, segmented=0)),
    Case("fwd_tb", "fwd", (8, 16, 4, 4, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(TB=3)),
    Case("fwd_items", "fwd", (32, 64, 16, 16, 1024, 1, 1, 1, 0, 0, 4), (1, 1), "int", E_FULL, dict(Nt=128, n_ntiles=2, n_items=512)),
    Case("fwd_chunks", "fwd", (1, 600, 10, 10, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=32)),
    Case("fwd_taps_per_kph", "fwd", (2, 64, 12, 12, 128, 5, 5, 1, 2, 2, 1), (1, 1), "int", E_FULL, dict(Nt=128, ntmpl0=3)),
    Case("fwd_mt4_partial", "fwd", (3, 64, 32, 32, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=32, MT=4),
         {"MNB_PK_MT": "4"}),
    Case("fwd_coltiles3", "fwd", (2, 32, 9, 10, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(col_tiles=3),
         {"MNB_PK_COLTILES": "3"}),
    Case("fwd_stages2", "fwd", (4, 16, 8, 8, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(nstage=2), {"MNB_PK_STAGES": "2"}),
    Case("fwd_stages4", "fwd", (4, 16, 8, 8, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(nstage=4), {"MNB_PK_STAGES": "4"}),
    Case("fwd_stages8", "fwd", (4, 16, 8, 8, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(nstage=8), {"MNB_PK_STAGES": "8"}),
    # ---- segmented forward (row 1): asymmetric two-piece levels (2, 1) at every N tile, fp32 x levels (3, 1), fp32 (3, 3)
    Case("seg_nt16_asym", "fwd", (2, 64, 8, 8, 16, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_FULL, dict(Nt=16, segmented=1, npairs=2)),
    Case("seg_nt32_asym", "fwd", (2, 64, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_NONE, dict(Nt=32, segmented=1)),
    Case("seg_nt48_asym", "fwd", (2, 64, 8, 8, 48, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_SCALE, dict(Nt=48, segmented=1)),
    Case("seg_nt64_asym", "fwd", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_BIAS, dict(Nt=64, segmented=1)),
    Case("seg_nt96_asym", "fwd", (2, 64, 8, 8, 96, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_FULL, dict(Nt=96, segmented=1)),
    Case("seg_nt128_asym", "fwd", (2, 64, 8, 8, 128, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_FULL, dict(Nt=128, segmented=1)),
    Case("seg_31_f32", "fwd", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", E_FULL, dict(segmented=1, npairs=3)),
    Case("seg_33_f32", "fwd", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (3, 3), "f32", E_BIAS, dict(segmented=1, npairs=6)),
    Case("seg_len1_asym", "fwd", (3, 64, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 1), "asym", E_FULL, dict(segmented=1, seg_len=1),
         {"MNB_PK_SEG_MMAS": "8"}),
    Case("seg_s2_grouped_asym", "fwd", (2, 144, 8, 8, 48, 3, 3, 2, 1, 1, 2), (2, 1), "asym", E_FULL, dict(segmented=1)),
    # ---- data gradient, rows 0 and 1, integer dy (two pieces, the second zero): bit-exact STE / gain epilogues
    Case("dg_nt16_rows", "dgrad", (2, 16, 40, 40, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=16, TH=3)),
    Case("dg_nt32", "dgrad", (2, 32, 8, 8, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=1.0), dict(Nt=32, segmented=0)),
    Case("dg_nt48", "dgrad", (2, 40, 8, 8, 16, 3, 2, 1, 1, 0, 1), (2, 1), "int", dict(gain=None, const=0.1), dict(Nt=48, segmented=0)),
    Case("dg_nt64", "dgrad", (2, 64, 8, 8, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=64, segmented=0)),
    Case("dg_nt96", "dgrad", (2, 96, 8, 8, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=1.0), dict(Nt=96, segmented=0)),
    Case("dg_nt128", "dgrad", (2, 200, 8, 8, 16, 1, 1, 1, 0, 0, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=128, n_ntiles=2)),
    Case("dg_seg_nt16", "dgrad", (2, 16, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=16, segmented=1)),
    Case("dg_seg_nt32", "dgrad", (2, 32, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=None, const=1.0), dict(Nt=32, segmented=1)),
    Case("dg_seg_nt48", "dgrad", (2, 48, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=1.0), dict(Nt=48, segmented=1)),
    Case("dg_seg_nt64", "dgrad", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=64, segmented=1)),
    Case("dg_seg_nt96", "dgrad", (2, 80, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=96, segmented=1)),
    Case("dg_seg_nt128", "dgrad", (2, 128, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(Nt=128, segmented=1)),
    Case("dg_s2", "dgrad", (2, 32, 8, 8, 48, 3, 3, 2, 1, 1, 1), (2, 1), "int", dict(gain=0.1), dict(ny=4)),
    Case("dg_s2_1x1", "dgrad", (2, 32, 8, 8, 64, 1, 1, 2, 0, 0, 1), (2, 1), "int", dict(gain=1.0), dict(ny=4)),
    Case("dg_grouped_padded", "dgrad", (2, 36, 8, 8, 24, 3, 3, 1, 1, 1, 3), (2, 1), "int", dict(gain=0.1), dict(Nt=16)),
    Case("dg_grouped_padded_seg", "dgrad", (2, 60, 8, 8, 240, 3, 3, 1, 1, 1, 3), (2, 1), "int", dict(gain=1.0), dict(segmented=1)),
    Case("dg_22_f32", "dgrad", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 2), "f32", dict(gain=None, const=1.0), dict(npairs=3)),
    # ---- int8 forward (row 2): every N tile
    Case("i8_nt16", "i8", (2, 32, 8, 8, 16, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=16)),
    Case("i8_nt32", "i8", (2, 24, 8, 8, 32, 3, 1, 1, 1, 0, 1), (1, 1), "int", E_NONE, dict(Nt=32)),
    Case("i8_nt48", "i8", (2, 32, 8, 8, 40, 3, 3, 2, 1, 1, 1), (1, 1), "int", E_SCALE, dict(Nt=48)),
    Case("i8_nt64", "i8", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 2), (1, 1), "int", E_BIAS, dict(Nt=32)),
    Case("i8_nt64b", "i8", (2, 48, 8, 8, 64, 1, 1, 1, 0, 0, 1), (1, 1), "int", E_FULL, dict(Nt=64)),
    Case("i8_nt96", "i8", (2, 32, 8, 8, 96, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=96)),
    Case("i8_nt128", "i8", (2, 32, 6, 6, 200, 1, 1, 1, 0, 0, 1), (1, 1), "int", E_FULL, dict(Nt=128, n_ntiles=2)),
    # ---- weight gradient: every N tile, integer dy and x (bit-exact), a_scale / kdiv each given or not
    Case("wg_nc16", "wgrad", (2, 16, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(Nc=16)),
    Case("wg_nc32", "wgrad", (2, 32, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=False, kdiv=True), dict(Nc=32)),
    Case("wg_nc48", "wgrad", (2, 48, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=False), dict(Nc=48)),
    Case("wg_nc64", "wgrad", (2, 64, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=False, kdiv=False), dict(Nc=64)),
    Case("wg_nc80", "wgrad", (2, 80, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(Nc=80)),
    Case("wg_nc96", "wgrad", (2, 96, 8, 8, 32, 1, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(Nc=96)),
    Case("wg_nc112", "wgrad", (2, 112, 8, 8, 32, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(Nc=112)),
    Case("wg_nc128_ktiles", "wgrad", (2, 128, 6, 6, 200, 3, 1, 1, 1, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         dict(Nc=128, n_ktiles=2)),
    Case("wg_ctiles", "wgrad", (2, 200, 6, 6, 32, 1, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         dict(n_ctiles=2)),
    Case("wg_gm2", "wgrad", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 2), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(gm=2)),
    Case("wg_gm4_padded", "wgrad", (2, 48, 8, 8, 48, 3, 3, 1, 1, 1, 4), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(gm=4)),
    Case("wg_gm8", "wgrad", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 8), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(gm=8)),
    Case("wg_gm16", "wgrad", (2, 128, 8, 8, 128, 3, 3, 1, 1, 1, 16), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(gm=16)),
    Case("wg_s2_kph4", "wgrad", (2, 32, 8, 8, 32, 3, 3, 2, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         dict(nkph_used=4)),
    Case("wg_s2_kph2", "wgrad", (2, 32, 8, 8, 32, 1, 2, 2, 0, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         dict(nkph_used=2)),
    Case("wg_ni_short", "wgrad", (9, 16, 4, 4, 16, 1, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict(NI=5, nsub=9)),
    Case("wg_splits_short", "wgrad", (1005, 16, 4, 4, 16, 1, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         dict(splits=101, stg_per_split=2)),
    Case("wg_raster_pass2", "wgrad", (1, 32, 2, 126, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True), dict()),
    Case("wg_7x7_33_f32", "wgrad", (1, 96, 6, 2, 32, 7, 7, 1, 5, 5, 1), (3, 3), "f32", dict(a_scale=False, kdiv=False), dict(Nc=48)),
    Case("wg_22_f32", "wgrad", (2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1), (2, 2), "f32", dict(a_scale=False, kdiv=False), dict()),
    # ---- plans the older packed-operand tests reached and the cases above do not: three-piece dy (the exact split), the
    # bench models' multi-tile and phase-split plans, fp32 dy against integer weights with the STE mask; the fp32 backward
    # with three dy pieces also keeps its max-norm bound
    Case("pk_fwd11_3x64x32x32_64_3x3s1g1", "fwd", (3, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL,
         dict(segmented=0, Nt=64, MT=1, ny=1)),
    Case("pk_fwd33_2x3x32x32_64_3x3s1g1", "fwd", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 3), "f32", E_FULL,
         dict(segmented=0, Nt=64, MT=1, ny=1)),
    Case("pk_fwd33_2x96x16x16_192_5x5s1g1", "fwd", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=96, MT=1, ny=1)),
    Case("pk_fwd33_2x160x32x32_96_1x1s1g1", "fwd", (2, 160, 32, 32, 96, 1, 1, 1, 0, 0, 1), (3, 3), "f32", E_FULL,
         dict(segmented=0, Nt=96, MT=1, ny=1)),
    Case("pk_fwd33_2x192x8x8_10_1x1s1g1", "fwd", (2, 192, 8, 8, 10, 1, 1, 1, 0, 0, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=16, MT=1, ny=1)),
    Case("pk_fwd33_2x256x16x16_512_3x3s1g16", "fwd", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (3, 3), "f32", E_FULL,
         dict(segmented=0, Nt=32, MT=1, ny=1)),
    Case("pk_fwd33_2x32x9x9_48_3x3s1g1", "fwd", (2, 32, 9, 9, 48, 3, 3, 1, 0, 0, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=48, MT=1, ny=1)),
    Case("gc3x3g32_fwd", "fwd", (8, 512, 8, 8, 1024, 3, 3, 1, 1, 1, 32), (1, 1), "int", E_FULL,
         dict(segmented=0, Nt=32, MT=2, ny=1)),
    Case("mt4_partial_seg", "fwd", (3, 64, 32, 32, 32, 3, 3, 1, 1, 1, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=32, MT=4, ny=1, n_mtiles=33, n_mgroups=9), {"MNB_PK_MT": "4"}),
    Case("mt2_partial_seg48", "fwd", (3, 64, 32, 32, 48, 3, 3, 1, 1, 1, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=48, MT=2, ny=1, n_mtiles=33, n_mgroups=17), {"MNB_PK_MT": "2"}),
    Case("seg32_fwd", "fwd", (2, 64, 16, 16, 32, 3, 3, 1, 1, 1, 1), (3, 3), "f32", E_FULL,
         dict(segmented=1, Nt=32, MT=1, ny=1)),
    Case("pk_dgrad31_3x64x32x32_64_3x3s1g1", "dgrad", (3, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=64, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad21_3x64x32x32_128_3x3s2g1", "dgrad", (3, 64, 32, 32, 128, 3, 3, 2, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=64, MT=1, ny=4)),
    Case("pk_dgrad31_3x64x32x32_128_3x3s2g1", "dgrad", (3, 64, 32, 32, 128, 3, 3, 2, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=64, MT=1, ny=4), maxnorm=3e-06),
    Case("pk_dgrad31_3x64x32x32_128_1x1s2g1", "dgrad", (3, 64, 32, 32, 128, 1, 1, 2, 0, 0, 1), (3, 1), "f32", D_STE,
         dict(segmented=0, Nt=64, MT=1, ny=4), maxnorm=3e-06),
    Case("pk_dgrad31_5x128x16x16_128_3x3s1g1", "dgrad", (5, 128, 16, 16, 128, 3, 3, 1, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=128, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_4x256x8x8_512_3x3s2g1", "dgrad", (4, 256, 8, 8, 512, 3, 3, 2, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=128, MT=1, ny=4), maxnorm=3e-06),
    Case("pk_dgrad31_2x3x32x32_64_3x3s1g1", "dgrad", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=16, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_2x96x16x16_192_5x5s1g1", "dgrad", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=96, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_2x192x32x32_160_1x1s1g1", "dgrad", (2, 192, 32, 32, 160, 1, 1, 1, 0, 0, 1), (3, 1), "f32", D_STE,
         dict(segmented=0, Nt=96, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_2x256x16x16_512_3x3s1g16", "dgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (3, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_2x256x32x32_256_1x1s1g2", "dgrad", (2, 256, 32, 32, 256, 1, 1, 1, 0, 0, 2), (3, 1), "f32", D_STE,
         dict(segmented=0, Nt=128, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad21_1x3x64x64_16_7x7s2g1", "dgrad", (1, 3, 64, 64, 16, 7, 7, 2, 3, 3, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=1, ny=4)),
    Case("pk_dgrad31_1x3x64x64_16_7x7s2g1", "dgrad", (1, 3, 64, 64, 16, 7, 7, 2, 3, 3, 1), (3, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=1, ny=4), maxnorm=3e-06),
    Case("pk_dgrad31_2x32x9x9_48_3x3s1g1", "dgrad", (2, 32, 9, 9, 48, 3, 3, 1, 0, 0, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=32, MT=1, ny=1), maxnorm=3e-06),
    Case("pk_dgrad31_2x48x16x16_64_3x3s1g1", "dgrad", (2, 48, 16, 16, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", D_STE,
         dict(segmented=1, Nt=48, MT=1, ny=1), maxnorm=3e-06),
    Case("gc3x3g16_dgrad21_ste", "dgrad", (32, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=4, ny=1)),
    Case("gc3x3g32_dgrad21_ste", "dgrad", (8, 512, 8, 8, 1024, 3, 3, 1, 1, 1, 32), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=2, ny=1)),
    Case("stem_dgrad21", "dgrad", (64, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_CONST,
         dict(segmented=1, Nt=16, MT=2, ny=1)),
    Case("mt2_dgrad21_ste", "dgrad", (3, 64, 28, 28, 48, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=64, MT=2, ny=1, n_mtiles=21, n_mgroups=11), {"MNB_PK_MT": "2"}),
    Case("i8_stem_224", "i8", (1, 3, 224, 224, 64, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=64, MT=2)),
    Case("i8_sc_1x1_s2", "i8", (4, 64, 16, 16, 128, 1, 1, 2, 0, 0, 1), (1, 1), "int", E_FULL, dict(Nt=128, MT=1)),
    Case("i8_nt48_s1", "i8", (4, 48, 16, 16, 48, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL, dict(Nt=48, MT=1)),
    Case("i8_mt4_nt32", "i8", (8, 64, 16, 16, 32, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL,
         dict(Nt=32, MT=4), {"MNB_PK_MT": "4"}),
    Case("pk_wgrad31_3x64x32x32_64_3x3s1g1", "wgrad", (3, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", W_ALL,
         dict(Nc=64, tpg=2, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_3x64x32x32_64_3x3s1g1", "wgrad", (3, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=64, tpg=2, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_3x64x32x32_128_3x3s2g1", "wgrad", (3, 64, 32, 32, 128, 3, 3, 2, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=32, tpg=3, gm=1), maxnorm=3e-06),
    Case("pk_wgrad31_3x64x32x32_128_1x1s2g1", "wgrad", (3, 64, 32, 32, 128, 1, 1, 2, 0, 0, 1), (3, 1), "f32", W_ALL,
         dict(Nc=64, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_3x64x32x32_128_1x1s2g1", "wgrad", (3, 64, 32, 32, 128, 1, 1, 2, 0, 0, 1), (3, 3), "f32", W_NONE,
         dict(Nc=64, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad31_5x128x16x16_128_3x3s1g1", "wgrad", (5, 128, 16, 16, 128, 3, 3, 1, 1, 1, 1), (3, 1), "f32", W_ALL,
         dict(Nc=128, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_5x128x16x16_128_3x3s1g1", "wgrad", (5, 128, 16, 16, 128, 3, 3, 1, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=128, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x3x32x32_64_3x3s1g1", "wgrad", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (2, 2), "f32", W_NONE,
         dict(Nc=16, tpg=5, gm=1)),
    Case("pk_wgrad31_2x3x32x32_64_3x3s1g1", "wgrad", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", W_ALL,
         dict(Nc=16, tpg=5, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_2x3x32x32_64_3x3s1g1", "wgrad", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=16, tpg=5, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x96x16x16_192_5x5s1g1", "wgrad", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (2, 2), "f32", W_NONE,
         dict(Nc=96, tpg=1, gm=1)),
    Case("pk_wgrad31_2x96x16x16_192_5x5s1g1", "wgrad", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (3, 1), "f32", W_ALL,
         dict(Nc=96, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_2x192x8x8_192_3x3s1g1", "wgrad", (2, 192, 8, 8, 192, 3, 3, 1, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=96, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x160x32x32_96_1x1s1g1", "wgrad", (2, 160, 32, 32, 96, 1, 1, 1, 0, 0, 1), (2, 2), "f32", W_NONE,
         dict(Nc=80, tpg=1, gm=1)),
    Case("pk_wgrad31_2x160x32x32_96_1x1s1g1", "wgrad", (2, 160, 32, 32, 96, 1, 1, 1, 0, 0, 1), (3, 1), "f32", W_ALL,
         dict(Nc=80, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_2x160x32x32_96_1x1s1g1", "wgrad", (2, 160, 32, 32, 96, 1, 1, 1, 0, 0, 1), (3, 3), "f32", W_NONE,
         dict(Nc=80, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x256x16x16_512_3x3s1g16", "wgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (2, 2), "f32", W_NONE,
         dict(Nc=64, tpg=2, gm=4)),
    Case("pk_wgrad31_2x256x16x16_512_3x3s1g16", "wgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (3, 1), "f32", W_ALL,
         dict(Nc=64, tpg=2, gm=4), maxnorm=3e-06),
    Case("pk_wgrad33_2x256x16x16_512_3x3s1g16", "wgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (3, 3), "f32", W_NONE,
         dict(Nc=64, tpg=2, gm=4), maxnorm=3e-06),
    Case("pk_wgrad22_2x32x9x9_48_3x3s1g1", "wgrad", (2, 32, 9, 9, 48, 3, 3, 1, 0, 0, 1), (2, 2), "f32", W_NONE,
         dict(Nc=32, tpg=3, gm=1)),
    Case("pk_wgrad31_2x32x9x9_48_3x3s1g1", "wgrad", (2, 32, 9, 9, 48, 3, 3, 1, 0, 0, 1), (3, 1), "f32", W_ALL,
         dict(Nc=32, tpg=3, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x48x16x16_64_3x3s1g1", "wgrad", (2, 48, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 2), "f32", W_NONE,
         dict(Nc=48, tpg=2, gm=1)),
    Case("pk_wgrad31_2x48x16x16_64_3x3s1g1", "wgrad", (2, 48, 16, 16, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", W_ALL,
         dict(Nc=48, tpg=2, gm=1), maxnorm=3e-06),
    Case("pk_wgrad22_2x112x16x16_64_3x3s1g1", "wgrad", (2, 112, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 2), "f32", W_NONE,
         dict(Nc=112, tpg=1, gm=1)),
    Case("pk_wgrad31_2x112x16x16_64_3x3s1g1", "wgrad", (2, 112, 16, 16, 64, 3, 3, 1, 1, 1, 1), (3, 1), "f32", W_ALL,
         dict(Nc=112, tpg=1, gm=1), maxnorm=3e-06),
    Case("pk_wgrad33_2x112x16x16_64_3x3s1g1", "wgrad", (2, 112, 16, 16, 64, 3, 3, 1, 1, 1, 1), (3, 3), "f32", W_NONE,
         dict(Nc=112, tpg=1, gm=1), maxnorm=3e-06),
    Case("wg_chain16", "wgrad", (8, 64, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", W_ALL,
         dict(Nc=64, splits=32), {"MNB_PK_WG_CHAIN": "16"}),
    Case("wg_merge0", "wgrad", (4, 256, 8, 8, 512, 3, 3, 1, 1, 1, 16), (2, 1), "f32", W_ALL,
         dict(Nc=16, gm=1), {"MNB_PK_WG_MERGE": "0"}),
    Case("wg_nc48_forced", "wgrad", (2, 96, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", W_ALL,
         dict(Nc=48, n_ctiles=2), {"MNB_PK_WG_NC": "48"}),
    # ---- fp32 dy (two nonzero pieces) at the (2, 1) plans the older tests ran so and the integer cases above reach with
    # the second dy piece zero
    Case("res64_dgrad21", "dgrad", (64, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_CONST,
         dict(segmented=1, Nt=64, MT=2, ny=1)),
    Case("res128s2_dgrad21_ste", "dgrad", (64, 64, 32, 32, 128, 3, 3, 2, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=64, MT=2, ny=4)),
    Case("res256s2_dgrad21", "dgrad", (16, 128, 16, 16, 256, 3, 3, 2, 1, 1, 1), (2, 1), "f32", D_CONST,
         dict(segmented=1, Nt=128, MT=1, ny=4)),
    Case("res256sc_dgrad21_ste", "dgrad", (16, 128, 16, 16, 256, 1, 1, 2, 0, 0, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=128, MT=1, ny=4)),
    Case("coltiles2_dgrad21", "dgrad", (2, 32, 16, 16, 48, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_CONST,
         dict(segmented=0, Nt=32, MT=1, ny=1, col_tiles=2), {"MNB_PK_COLTILES": "2"}),
    Case("pk_dgrad21_f32_3x64x32x32_64_3x3s1g1", "dgrad", (3, 64, 32, 32, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=1, Nt=64, MT=1, ny=1)),
    Case("pk_dgrad21_f32_5x128x16x16_128_3x3s1g1", "dgrad", (5, 128, 16, 16, 128, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=1, Nt=128, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x3x32x32_64_3x3s1g1", "dgrad", (2, 3, 32, 32, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=1, Nt=16, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x96x16x16_192_5x5s1g1", "dgrad", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (2, 1), "f32", D_STE,
         dict(segmented=1, Nt=96, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x192x32x32_160_1x1s1g1", "dgrad", (2, 192, 32, 32, 160, 1, 1, 1, 0, 0, 1), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=96, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x256x16x16_512_3x3s1g16", "dgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=16, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x256x32x32_256_1x1s1g2", "dgrad", (2, 256, 32, 32, 256, 1, 1, 1, 0, 0, 2), (2, 1), "f32", D_STE,
         dict(segmented=0, Nt=128, MT=1, ny=1)),
    Case("pk_dgrad21_f32_2x48x16x16_64_3x3s1g1", "dgrad", (2, 48, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", D_STE,
         dict(segmented=1, Nt=48, MT=1, ny=1)),
    Case("wg_nc112_f32", "wgrad", (2, 112, 16, 16, 64, 3, 3, 1, 1, 1, 1), (2, 1), "f32", W_ALL,
         dict(Nc=112, tpg=1, gm=1)),
    Case("pk_wgrad21_f32_3x64x32x32_128_1x1s2g1", "wgrad", (3, 64, 32, 32, 128, 1, 1, 2, 0, 0, 1), (2, 1), "f32", W_ALL,
         dict(Nc=64, tpg=1, gm=1)),
    Case("pk_wgrad21_f32_5x128x16x16_128_3x3s1g1", "wgrad", (5, 128, 16, 16, 128, 3, 3, 1, 1, 1, 1), (2, 1), "f32", W_ALL,
         dict(Nc=128, tpg=1, gm=1)),
    Case("pk_wgrad21_f32_2x96x16x16_192_5x5s1g1", "wgrad", (2, 96, 16, 16, 192, 5, 5, 1, 2, 2, 1), (2, 1), "f32", W_ALL,
         dict(Nc=96, tpg=1, gm=1)),
    Case("pk_wgrad21_f32_2x160x32x32_96_1x1s1g1", "wgrad", (2, 160, 32, 32, 96, 1, 1, 1, 0, 0, 1), (2, 1), "f32", W_ALL,
         dict(Nc=80, tpg=1, gm=1)),
    Case("pk_wgrad21_f32_2x256x16x16_512_3x3s1g16", "wgrad", (2, 256, 16, 16, 512, 3, 3, 1, 1, 1, 16), (2, 1), "f32", W_ALL,
         dict(Nc=64, tpg=2, gm=4)),
    Case("pk_wgrad21_f32_2x32x9x9_48_3x3s1g1", "wgrad", (2, 32, 9, 9, 48, 3, 3, 1, 0, 0, 1), (2, 1), "f32", W_ALL,
         dict(Nc=32, tpg=3, gm=1)),
    # ---- refusals (launch refuses with the query's code and text, writes nothing)
    Case("no_fwd_dilation", "fwd", (1, 16, 8, 8, 16, 3, 3, 1, 1, 1, 1, 2), (1, 1), "int", E_FULL, refuse="dilation != 1"),
    Case("no_fwd_stride3", "fwd", (1, 16, 9, 9, 16, 3, 3, 3, 1, 1, 1), (1, 1), "int", E_FULL, refuse="stride must be 1 or 2"),
    Case("no_fwd_pad", "fwd", (1, 16, 8, 8, 16, 3, 1, 1, 1, 1, 1), (1, 1), "int", E_FULL, refuse="padding larger than the filter"),
    Case("no_fwd_odd_s2", "fwd", (1, 16, 9, 8, 16, 3, 3, 2, 1, 1, 1), (1, 1), "int", E_FULL, refuse="stride 2 needs even H and W"),
    Case("no_fwd_empty", "fwd", (1, 16, 2, 8, 16, 5, 1, 1, 0, 0, 1), (1, 1), "int", E_FULL, refuse="empty output"),
    Case("no_fwd_taps", "fwd", (1, 16, 12, 12, 16, 9, 9, 1, 4, 4, 1), (1, 1), "int", E_FULL, refuse="more than 64 filter taps"),
    Case("no_dg_taps", "dgrad", (1, 16, 12, 12, 16, 9, 9, 1, 4, 4, 1), (2, 1), "int", dict(gain=1.0),
         refuse="more than 64 filter taps"),
    Case("no_i8_grouped", "i8", (1, 48, 8, 8, 48, 3, 3, 1, 1, 1, 2), (1, 1), "int", E_FULL,
         refuse="grouped int8 conv needs GEMM-K channels per group % 16 == 0"),
    Case("no_fwd_prog", "fwd", (1, 1536, 2, 4, 256, 7, 7, 2, 2, 2, 16), (2, 1), "asym", E_FULL,
         refuse="MMA program longer than 512 entries"),
    Case("no_dg_prog", "dgrad", (1, 16, 2, 2, 96, 7, 7, 2, 3, 3, 1), (2, 1), "int", dict(gain=1.0),
         refuse="MMA program longer than 512 entries"),
    Case("no_wg_row", "wgrad", (1, 16, 4, 130, 16, 3, 3, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="row wider than 128 positions"),
    Case("no_wg_taps", "wgrad", (1, 16, 12, 12, 16, 9, 9, 1, 4, 4, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="more than 64 taps"),
    Case("no_wg_pad", "wgrad", (1, 16, 8, 8, 16, 3, 1, 1, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="pk wgrad: padding larger than the filter"),
    Case("no_wg_raster", "wgrad", (1, 16, 70, 100, 16, 63, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="no raster fits shared memory"),
    Case("no_wg_empty", "wgrad", (1, 16, 2, 8, 16, 5, 1, 1, 0, 0, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="pk wgrad: empty output"),
    Case("no_wg_dilation", "wgrad", (1, 16, 8, 8, 16, 3, 3, 1, 1, 1, 1, 2), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="pk wgrad: dilation != 1"),
    Case("no_wg_odd_s2", "wgrad", (1, 16, 9, 8, 16, 3, 3, 2, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="pk wgrad: stride 2 needs even H and W"),
    Case("no_i8_overflow", "i8", (1, 16400, 4, 4, 16, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL,
         refuse="int8 sums could overflow s32"),
    Case("no_fwd_wimage", "fwd", (1, 8192, 4, 4, 8192, 3, 3, 1, 1, 1, 1), (1, 1), "int", E_FULL,
         refuse="weight image larger than 1 GiB"),
    Case("no_wg_stride", "wgrad", (1, 16, 9, 9, 16, 3, 3, 3, 1, 1, 1), (2, 1), "int", dict(a_scale=True, kdiv=True),
         refuse="pk wgrad: stride"),
]

# refusal reasons of make_plan / conv_route / conv_mma / make_wg_plan_nc that no shape can reach, and why
UNREACHABLE = {
    "filter too wide": "a halo of 96 columns needs 97 taps in one output phase, refused first as more than 64 filter taps",
    "box dimension": "Wt <= 128 - halo by the column tiling, TH <= 128 and the halo rows <= 63 keep BW <= 128, THH < 256, TB <= 128",
    "accumulators exceed the register budget": "MT is only raised (heuristic or MNB_PK_MT) while MT * Nt <= 128; wgrad tpg <= 128 / Nc",
    "plan with Nt": "make_plan picks Nt from kNtSizes and MT with MT * Nt <= 128",
    "MMA program offset overflow": "every program offset lies inside one pipeline stage, < 227 KB = 14.5K 16-byte units",
    "issue program too long": "make_wg_plan falls back to a narrower N tile; at Nc = 16 every filter fits (8 taps per CTA)",
}


def _bench_case(workload, fn, sh, mode, ta, tw):
    """the case of one recorded bench launch: integer levels where the operands are integer, split fp32 otherwise"""
    B, Cc, H, W, K, R, S, st, _, ph, pw, dil, _, G = sh
    shape = (B, Cc, H, W, K, R, S, st, ph, pw, G)
    name = f"bench_{workload}_{B}x{Cc}x{H}x{W}_{K}_{R}x{S}s{st}g{G}"
    gain = 0.1 if "dorefa" in workload else 1.0
    if mode == 2:
        return Case(f"{name}_wgrad{ta}{tw}", "wgrad", shape, (ta, tw), "int" if tw == 1 else "f32",
                    dict(a_scale=tw == 1, kdiv=tw == 1), bench=workload)
    if mode == 1:
        return Case(f"{name}_dgrad{ta}{tw}", "dgrad", shape, (ta, tw), "int" if tw == 1 else "f32",
                    dict(gain=gain) if tw == 1 else dict(gain=None, const=1.0), bench=workload)
    ops = "int" if (ta, tw) == (1, 1) else ("pm1" if ta == 1 else "f32")
    return Case(f"{name}_fwd{ta}{tw}", "fwd", shape, (ta, tw), ops, E_FULL if ops == "int" else E_BIAS, bench=workload)


def _bench_cases():
    from tests.pk_conv_bench_launches import BENCH_LAUNCHES
    return [_bench_case(*launch) for launch in BENCH_LAUNCHES]


CASES += _bench_cases()

# reachable refusal reasons that no case holds yet (shapes far outside the models: huge shared-memory stages or tap counts);
# the host sweep still checks that query and launch agree on them wherever it meets them
UNCASED = {
    "fewer than two pipeline stages fit": "forward / data-gradient stage of more than half the shared-memory budget",
    "one 16-channel stage does not fit in shared memory": "tall filters (R near 64) on rows of 128 positions",
    "too many tap groups": "more than 16 tap groups of one output phase: many taps with a stage too large for several",
    "fewer than two stages fit": "wgrad sub-block of just over half the shared-memory budget",
}

