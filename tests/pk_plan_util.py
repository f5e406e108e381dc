"""Host-only plan queries of the packed-operand family (mnb_pk_conv_plan_ex / mnb_pk_wgrad_plan) decoded to dicts, and the
plan signatures the coverage test compares.  No GPU needed: the plans are computed on the host, with the same MNB_PK_*
environment knobs the launches read."""
import ctypes as C

CONV_FIELDS = ("wimg_lo wimg_hi Nt n_ntiles MT CC chunks nstage smem acc TH TB BW n_mtiles n_items ny "
               "segmented seg_len npairs col_tiles n_mgroups").split()
WGRAD_FIELDS = "Nc n_ctiles tpg n_tg gm splits NI nstage BW TH".split()

# the kernel instances the library is built with (mnb_pk.cu: kNtSizes, wfns)
CONV_NT = (16, 32, 48, 64, 96, 128)
WGRAD_NC = (16, 32, 48, 64, 80, 96, 112, 128)


def shape(B, Cc, H, W, K, R, st, pad, G):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def conv_plan(sh, mode, ta, tw):
    """plan of mnb_pk_conv for (shape, mode, terms); None if the shape is outside the cover"""
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(CONV_FIELDS))()
    if L.load().mnb_pk_conv_plan_ex(C.byref(sh), mode, ta, tw, out, len(CONV_FIELDS)) != 0:
        return None
    return dict(zip(CONV_FIELDS, list(out)))


def wgrad_plan(sh, t_dy, t_x):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * len(WGRAD_FIELDS))()
    if L.load().mnb_pk_wgrad_plan(C.byref(sh), t_dy, t_x, out, len(WGRAD_FIELDS)) != 0:
        return None
    return dict(zip(WGRAD_FIELDS, list(out)))


def conv_signature(p):
    """what selects the code path of pk_conv_kernel: instance (SEG, Nt), M tiles per item, output phases"""
    return (bool(p["segmented"]), p["Nt"], p["MT"], p["ny"])


def wgrad_signature(p):
    """instance Nc, several tap groups, merged groups"""
    return (p["Nc"], p["tpg"] > 1, p["gm"] > 1)
