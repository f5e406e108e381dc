"""Pinned cases of the narrow grouped 3x3 convolutions (csrc/mnb_pk.cu, pk_gc3_kernel behind mnb_pk_gc3_conv and
mnb_pk_gc3_conv_codes), shared by tests/test_gc3_coverage_cpu.py (host: plans, features, refusals, the bench launches) and
tests/test_gpu_gc3_fp64.py (device: every case against an fp64 reference).

A case: shape (B, C, H, W, K, pad_h, pad_w, G) of a 3x3 stride-1 conv with 16 input and 32 output channels per group;
mode - "fwd" (mnb_pk_gc3_conv mode 0, fp32 out), "codes" (mnb_pk_gc3_conv_codes: int16 sums and the decode pair) or
"dgrad" (mnb_pk_gc3_conv mode 1); operands -

    pm1      activations +-1, weights in {-1, 0, 1}
    dorefa4  DoReFa 4-bit levels: activations 0 .. 15, weights odd in -15 .. 15
    int8     symmetric int8-range levels: fp32 forward |x|, |w| <= 127; codes |x| <= 113, |w| <= 2 (within the int16 bound)
    int      data gradient on integer dy, |dy| <= 255 (bf16-exact: the second piece is 0), weights in -3 .. 3
    real     data gradient on random dy, two pieces, w_scale folded into dy, some kzero channels

epi - the epilogue arguments: forward n_scale (per-channel tensor or none), a_scale ("tensor": a device scalar, or the
constant), bias (tensor or none); data gradient gain (the STE mask bits8 with that gain) or a_scale (a_scale_const alone);
expect - the plan fields of mnb_pk_gc3_plan the case is pinned to; model - (workload, layer) of the bench launch the case
stands for, at the bench batch."""
from collections import namedtuple

Case = namedtuple("Case", "id shape mode operands epi expect model", defaults=(None,))

# fields of mnb_pk_gc3_plan (out[0..9])
PLAN_FIELDS = "GB TB nmb nstage smem ctas tiles chain Nt ncons".split()
MODES = ("fwd", "codes", "dgrad")
TERMS = {"fwd": (1, 1), "codes": (1, 1), "dgrad": (2, 1)}      # (pieces of the streamed operand, pieces of the weights)


def _c(id, shape, mode, operands, epi, expect, model=None):
    return Case(id, shape, mode, operands, epi, expect, model)


CASES = [
    # ---- the bench launches at batch 256: the forward (codes for wbwtab, fp32 on 4-bit levels for DoReFa) and the data
    # gradient.  wbwtab: behind the fused BatchNorm + binarizer + max-pool producer, which owns the STE mask (a_scale_const
    # 1, no mask).  DoReFa: a max-pool sits between the producer and the layer, so the layer packs its own input and keeps
    # the STE mask bits8 with the gain 0.1
    _c("f_g16_b256_dorefa4", (256, 256, 16, 16, 512, 1, 1, 16), "fwd", "dorefa4", dict(n_scale=1, a_scale=1 / 15, bias=1),
       dict(GB=1, TB=1, nmb=5, nstage=6, ctas=128, tiles=256, Nt=32), model=('nin_gc_dorefa_w4a4', 'gc3x3g16')),
    _c("f_g32_b256_dorefa4", (256, 512, 8, 8, 1024, 1, 1, 32), "fwd", "dorefa4", dict(n_scale=1, a_scale=1 / 15, bias=1),
       dict(GB=1, TB=4, nmb=6, nstage=6, ctas=128, tiles=64, Nt=32), model=('nin_gc_dorefa_w4a4', 'gc3x3g32')),
    _c("c_g16_b256_pm1", (256, 256, 16, 16, 512, 1, 1, 16), "codes", "pm1", dict(n_scale=1, a_scale=1.0, bias=1),
       dict(GB=1, TB=1, nmb=5, nstage=6, ctas=128, tiles=256, Nt=32), model=('nin_gc_wbwtab_w3a2', 'gc3x3g16')),
    _c("c_g32_b256_pm1", (256, 512, 8, 8, 1024, 1, 1, 32), "codes", "pm1", dict(n_scale=1, a_scale=1.0, bias=1),
       dict(GB=1, TB=4, nmb=6, nstage=6, ctas=128, tiles=64, Nt=32), model=('nin_gc_wbwtab_w3a2', 'gc3x3g32')),
    _c("d_g16_b256_wbwtab", (256, 256, 16, 16, 512, 1, 1, 16), "dgrad", "real", dict(a_scale=1.0),
       dict(GB=1, TB=1, nmb=5, nstage=3, ctas=128, tiles=256, Nt=16), model=('nin_gc_wbwtab_w3a2', 'gc3x3g16')),
    _c("d_g32_b256_wbwtab", (256, 512, 8, 8, 1024, 1, 1, 32), "dgrad", "real", dict(a_scale=1.0),
       dict(GB=1, TB=2, nmb=3, nstage=6, ctas=128, tiles=128, Nt=16), model=('nin_gc_wbwtab_w3a2', 'gc3x3g32')),
    _c("d_g16_b256_dorefa", (256, 256, 16, 16, 512, 1, 1, 16), "dgrad", "real", dict(gain=0.1),
       dict(GB=1, TB=1, nmb=5, nstage=3, ctas=128, tiles=256, Nt=16), model=('nin_gc_dorefa_w4a4', 'gc3x3g16')),
    _c("d_g32_b256_dorefa", (256, 512, 8, 8, 1024, 1, 1, 32), "dgrad", "real", dict(gain=0.1),
       dict(GB=1, TB=2, nmb=3, nstage=6, ctas=128, tiles=128, Nt=16), model=('nin_gc_dorefa_w4a4', 'gc3x3g32')),
    # ---- forward and codes: every plan feature, on each operand kind
    _c("f_1x1_gb4", (1, 64, 1, 1, 128, 1, 1, 4), "fwd", "pm1", dict(n_scale=1, a_scale="tensor", bias=1),
       dict(GB=4, TB=1, nmb=1, nstage=6, ctas=1, tiles=1, Nt=32)),
    _c("c_1x1_gb4", (1, 64, 1, 1, 128, 1, 1, 4), "codes", "dorefa4", dict(n_scale=1, a_scale=0.37, bias=0),
       dict(GB=4, TB=1, nmb=1, nstage=6, ctas=1, tiles=1, Nt=32)),
    _c("f_row40_nmb3", (1, 64, 1, 40, 128, 2, 2, 4), "fwd", "int8", dict(n_scale=1, a_scale=0.37, bias=0),
       dict(GB=2, TB=1, nmb=3, nstage=6, ctas=2, tiles=1, Nt=32)),
    _c("c_row40_nmb3", (1, 64, 1, 40, 128, 2, 2, 4), "codes", "pm1", dict(n_scale=1, a_scale="tensor", bias=1),
       dict(GB=2, TB=1, nmb=3, nstage=6, ctas=2, tiles=1, Nt=32)),
    _c("f_row126_widest", (1, 64, 1, 126, 128, 1, 1, 4), "fwd", "int8", dict(n_scale=0, a_scale=0.25, bias=0),
       dict(GB=2, TB=1, nmb=2, nstage=6, ctas=2, tiles=1, Nt=32)),
    _c("c_row126_widest", (1, 64, 1, 126, 128, 1, 1, 4), "codes", "pm1", dict(n_scale=0, a_scale="tensor", bias=1),
       dict(GB=2, TB=1, nmb=2, nstage=6, ctas=2, tiles=1, Nt=32)),
    _c("f_g64_3tiles", (5, 1024, 1, 64, 2048, 2, 2, 64), "fwd", "dorefa4", dict(n_scale=0, a_scale="tensor", bias=1),
       dict(GB=1, TB=1, nmb=4, nstage=6, ctas=128, tiles=5, Nt=32)),
    _c("c_g64_3tiles", (5, 1024, 1, 64, 2048, 2, 2, 64), "codes", "int8", dict(n_scale=0, a_scale=0.25, bias=0),
       dict(GB=1, TB=1, nmb=4, nstage=6, ctas=128, tiles=5, Nt=32)),
    _c("f_g64_4tiles_st3_asym", (7, 1024, 1, 100, 2048, 2, 0, 64), "fwd", "int8", dict(n_scale=1, a_scale="tensor", bias=1),
       dict(GB=1, TB=1, nmb=5, nstage=3, ctas=128, tiles=7, Nt=32)),
    _c("c_g64_4tiles_st3_asym", (7, 1024, 1, 100, 2048, 2, 0, 64), "codes", "pm1", dict(n_scale=1, a_scale=0.37, bias=0),
       dict(GB=1, TB=1, nmb=5, nstage=3, ctas=128, tiles=7, Nt=32)),
    _c("f_g64_short_2tiles", (5, 1024, 1, 40, 2048, 2, 2, 64), "fwd", "pm1", dict(n_scale=0, a_scale=0.25, bias=0),
       dict(GB=1, TB=2, nmb=6, nstage=6, ctas=128, tiles=3, Nt=32)),
    _c("c_g64_short_2tiles", (5, 1024, 1, 40, 2048, 2, 2, 64), "codes", "dorefa4", dict(n_scale=0, a_scale="tensor", bias=1),
       dict(GB=1, TB=2, nmb=6, nstage=6, ctas=128, tiles=3, Nt=32)),
    _c("f_asym_5x3_short", (37, 64, 5, 3, 128, 0, 2, 4), "fwd", "pm1", dict(n_scale=1, a_scale="tensor", bias=1),
       dict(GB=4, TB=4, nmb=2, nstage=6, ctas=10, tiles=10, Nt=32)),
    _c("c_asym_5x3_short", (37, 64, 5, 3, 128, 0, 2, 4), "codes", "dorefa4", dict(n_scale=1, a_scale=0.37, bias=0),
       dict(GB=4, TB=4, nmb=2, nstage=6, ctas=10, tiles=10, Nt=32)),
    # ---- data gradient: every plan feature, on integer and real dy, STE mask and constant
    _c("d_1x1_gb4", (1, 64, 1, 1, 128, 1, 1, 4), "dgrad", "int", dict(gain=0.1),
       dict(GB=4, TB=1, nmb=1, nstage=6, ctas=1, tiles=1, Nt=16)),
    _c("d_1x1_b9_gb2", (9, 64, 1, 1, 128, 1, 1, 4), "dgrad", "real", dict(a_scale=0.1),
       dict(GB=2, TB=8, nmb=1, nstage=6, ctas=4, tiles=2, Nt=16)),
    _c("d_2x96_nmb4", (1, 64, 2, 96, 128, 1, 0, 4), "dgrad", "int", dict(a_scale=0.5),
       dict(GB=1, TB=1, nmb=4, nstage=3, ctas=4, tiles=1, Nt=16)),
    _c("d_9x34_nmb6", (1, 64, 9, 34, 128, 0, 0, 4), "dgrad", "int", dict(gain=0.1),
       dict(GB=1, TB=1, nmb=6, nstage=3, ctas=4, tiles=1, Nt=16)),
    _c("d_row126_widest", (1, 64, 1, 126, 128, 1, 1, 4), "dgrad", "real", dict(gain=0.1),
       dict(GB=1, TB=1, nmb=2, nstage=3, ctas=4, tiles=1, Nt=16)),
    _c("d_g64_3tiles", (5, 1024, 1, 40, 2048, 1, 0, 64), "dgrad", "real", dict(gain=0.1),
       dict(GB=1, TB=1, nmb=1, nstage=6, ctas=128, tiles=5, Nt=16)),
    _c("d_g64_short_2tiles", (5, 1024, 1, 30, 2048, 1, 0, 64), "dgrad", "real", dict(a_scale=0.1),
       dict(GB=1, TB=2, nmb=2, nstage=6, ctas=128, tiles=3, Nt=16)),
    _c("d_pad2_7x9", (4, 128, 7, 9, 256, 2, 2, 8), "dgrad", "int", dict(a_scale=0.5),
       dict(GB=1, TB=2, nmb=3, nstage=6, ctas=16, tiles=2, Nt=16)),
]

# ---- refusals: (id, mode, conv shape (B, C, H, W, K, R, S, stride, stride, pad_h, pad_w, dil, dil, G), pieces, env, launch,
# code, text).  launch: "" (the plan query refuses; the launch must return the same code and text), "unaligned_out",
# "unaligned_a" (the launcher refuses an operand or output off a 16-byte boundary) or "codes_bound" (the int16 bound of
# mnb_pk_gc3_conv_codes)
Refusal = namedtuple("Refusal", "id mode shape terms env launch code text")
_SH = (4, 64, 8, 8, 128, 3, 3, 1, 1, 1, 1, 1, 1, 4)


def _sh(**kw):
    names = "B C H W K R S sh sw ph pw dh dw G".split()
    v = dict(zip(names, _SH))
    v.update(kw)
    return tuple(v[n] for n in names)


REFUSALS = [
    Refusal("not_3x3", "fwd", _sh(R=5, S=5, ph=2, pw=2), (1, 1), {}, "", "E_UNSUPPORTED", "pk gc3: filter is not 3x3"),
    Refusal("not_3x3_1x3", "dgrad", _sh(R=1, ph=0), (2, 1), {}, "", "E_UNSUPPORTED", "pk gc3: filter is not 3x3"),
    Refusal("stride2", "fwd", _sh(sh=2, sw=2), (1, 1), {}, "", "E_UNSUPPORTED", "pk gc3: stride or dilation != 1"),
    Refusal("dilation2", "dgrad", _sh(dh=2, dw=2), (2, 1), {}, "", "E_UNSUPPORTED", "pk gc3: stride or dilation != 1"),
    Refusal("pad3", "fwd", _sh(ph=3), (1, 1), {}, "", "E_UNSUPPORTED", "pk gc3: padding outside 0..2"),
    Refusal("pad_w3_dgrad", "dgrad", _sh(pw=3), (2, 1), {}, "", "E_UNSUPPORTED", "pk gc3: padding outside 0..2"),
    Refusal("cin32", "fwd", _sh(C=128), (1, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: needs 16 / 32 channels per group and groups % 4 == 0"),
    Refusal("groups6", "dgrad", _sh(C=96, K=192, G=6), (2, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: needs 16 / 32 channels per group and groups % 4 == 0"),
    Refusal("fwd_two_pieces", "fwd", _sh(), (2, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: the forward takes one activation piece and one weight piece"),
    Refusal("dgrad_three_pieces", "dgrad", _sh(), (3, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: the data gradient takes two dy pieces and one weight piece"),
    Refusal("dgrad_segmented", "dgrad", _sh(), (2, 1), {"MNB_PK_SEG_MMAS": "16"}, "", "E_UNSUPPORTED",
            "pk gc3: plan is segmented or tiled along N"),
    Refusal("empty_output", "fwd", _sh(H=1, W=5, ph=0, pw=0), (1, 1), {}, "", "E_UNSUPPORTED", "pk conv: empty output"),
    Refusal("empty_output_dgrad", "dgrad", _sh(H=2, W=5, ph=0, pw=1), (2, 1), {}, "", "E_UNSUPPORTED",
            "pk conv: empty output"),
    Refusal("row127", "fwd", _sh(B=1, H=1, W=127), (1, 1), {}, "", "E_UNSUPPORTED", "pk gc3: image larger than one box"),
    Refusal("row129_pad0", "codes", _sh(B=1, H=3, W=129, ph=0, pw=0), (1, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: image larger than one box"),
    Refusal("row127_dgrad", "dgrad", _sh(B=1, H=1, W=127), (2, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: image larger than one box"),
    Refusal("image32", "fwd", _sh(B=1, H=32, W=32), (1, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: no image tile fits the accumulators and shared memory"),
    Refusal("image32_dgrad", "dgrad", _sh(B=1, H=32, W=32), (2, 1), {}, "", "E_UNSUPPORTED",
            "pk gc3: no image tile fits the accumulators and shared memory"),
    Refusal("unaligned_out", "fwd", _sh(), (1, 1), {}, "unaligned_out", "E_UNSUPPORTED",
            "pk gc3: operands and output must be 16-byte aligned"),
    Refusal("unaligned_codes", "codes", _sh(), (1, 1), {}, "unaligned_out", "E_UNSUPPORTED",
            "pk gc3: operands and output must be 16-byte aligned"),
    Refusal("unaligned_dy", "dgrad", _sh(), (2, 1), {}, "unaligned_a", "E_UNSUPPORTED",
            "pk gc3: operands and output must be 16-byte aligned"),
    Refusal("codes_bound", "codes", _sh(), (1, 1), {}, "codes_bound", "E_UNSUPPORTED",
            "pk_gc3_conv_codes: sums of 16 x 3 x 3 terms of level 228 may exceed int16"),
]
# level bound of the codes_bound refusal: 16 x 9 x 228 > 32767 >= 16 x 9 x 227
CODES_BOUND_REFUSED = 228

# refusal reasons of make_gc3_plan that no shape reaches, and why: a host sweep (test_gc3_coverage_cpu.py) confirms that
# none of its shapes returns them
UNREACHABLE = {
    "descriptor range": "a stage ring and the weights fit the 223 KiB shared-memory budget, below the 2^18-byte range of "
                        "a descriptor, and npos <= 8 m64 blocks plus two halo rows of at most 128 positions",
    "MMA chain longer than 128": "a chain is 9 taps x piece pairs (1 or 2) x K-steps (1 or 2): at most 36 MMAs",
    "MMA offset overflow": "A offsets stay within two stages of the ring and B offsets within one group's weight image, "
                           "both below 2^16 16-byte units",
}


def conv_shape(shape):
    """ConvShape of a case's (B, C, H, W, K, pad_h, pad_w, G)"""
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, ph, pw, G = shape
    return L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, ph, pw, 1, 1, G)


def refusal_shape(r):
    from micronet_b200 import _lib as L
    return L.ConvShape(*r.shape)


def query(sh, mode, terms, chain=False):
    """mnb_pk_gc3_plan of a ConvShape as a dict (with the chain as (tap, A piece, B piece, K-step) tuples if ``chain``); on
    a refusal (code, error text)"""
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    out = (C.c_int32 * (10 + 4 * 128))()
    rc = lib.mnb_pk_gc3_plan(C.byref(sh), 1 if mode == "dgrad" else 0, terms[0], terms[1], out, len(out))
    if rc != 0:
        return rc, lib.mnb_last_error().decode(errors="replace")
    p = dict(zip(PLAN_FIELDS, list(out[:10])))
    if chain:
        p["chain_mmas"] = [tuple(out[10 + 4 * i:14 + 4 * i]) for i in range(p["chain"])]
    return p


def plan_of(case):
    return query(conv_shape(case.shape), case.mode, TERMS[case.mode])


def out_hw(shape, mode):
    """(rows, columns) of the output raster: the forward output, or the data gradient's dx"""
    B, Cc, H, W, K, ph, pw, G = shape
    return (H, W) if mode == "dgrad" else (H + 2 * ph - 2, W + 2 * pw - 2)


def tiles_per_cta(plan, G):
    """image tiles the busiest CTA of a group block walks: ceil(tiles / CTAs per block)"""
    cpb = plan["ctas"] // (G // plan["GB"])
    return -(-plan["tiles"] // cpb)


def features(case, plan):
    """the plan and shape features a case reaches"""
    B, Cc, H, W, K, ph, pw, G = case.shape
    oh, ow = out_hw(case.shape, case.mode)
    tpc = tiles_per_cta(plan, G)
    f = {f"GB{plan['GB']}", f"nmb{plan['nmb']}", f"nstage{plan['nstage']}", f"pad_h{ph}", f"pad_w{pw}",
         "TB1" if plan["TB"] == 1 else "TB>1", f"G{G}"}
    if tpc == 1:
        f.add("tiles_per_cta1")
    elif tpc == 2:
        f.add("tiles_per_cta2")
    elif tpc <= plan["nstage"]:
        f.add("tiles_per_cta3..nstage")
    else:
        f.add("tiles_per_cta>nstage")
    if B % plan["TB"] and tpc > 1:
        f.add("short_last_tile_of_several")
    if ph != pw:
        f.add("pad_h!=pad_w")
    if oh != ow:
        f.add("non_square")
    if oh == 1:
        f.add("one_row")
    if ow == 1:
        f.add("one_column")
    if ow + 2 == 128:         # the raster's row pitch is ow + 2 (3x3 halo): 128 = the widest a box takes
        f.add("widest_row")
    return f
