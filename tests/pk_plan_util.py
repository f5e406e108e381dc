"""Shared helpers of the packed-operand family's tests.

* Host-only plan queries (mnb_pk_conv_plan_ex / mnb_pk_i8_conv_plan / mnb_pk_wgrad_plan) decoded to dicts, the plan
  signatures the coverage tests compare, and ``env``, which sets the MNB_PK_* knobs the plan query and the launch read.
* The convolutions of the bench models and the shared-memory limits their plans must respect.
* The fp64 references of the GPU tests: the element-wise bound check ``within`` and the correctly rounded fp32 fmaf."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMIT = 227 * 1024          # opt-in shared memory per block on sm_90 (H100)
RESERVED = 1024             # per-block reservation that cuobjdump's SHARED figure includes

# every field the plan queries write, in order (mnb_pk_conv_plan: the first 16 conv fields)
CONV_FIELDS = ("wimg_lo wimg_hi Nt n_ntiles MT CC chunks nstage smem acc TH TB BW n_mtiles n_items ny "
               "segmented seg_len npairs col_tiles n_mgroups "
               "ntmpl0 ntmpl1 ntmpl2 ntmpl3 ntap0 ntap1 ntap2 ntap3 words last_seg").split()
WGRAD_FIELDS = "Nc n_ctiles tpg n_tg gm splits NI nstage BW TH n_ktiles nkph_used stg_per_split nsub prog nstg_total".split()

# the kernel instances the library is built with (mnb_pk.cu: kNtSizes, wfns)
CONV_NT = (16, 32, 48, 64, 96, 128)
WGRAD_NC = (16, 32, 48, 64, 80, 96, 112, 128)


class env:
    """sets the given environment variables (MNB_PK_* knobs) inside the block and restores the old values after it; the
    plan cache of micronet_b200.pk, keyed by shape only, is cleared on both sides of a block that sets any"""

    def __init__(self, env):
        self.env, self.old = env, {}

    def _clear(self):
        if self.env:
            from micronet_b200 import pk as PK
            PK._plan_cache.clear()

    def __enter__(self):
        for k, v in self.env.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = v
        self._clear()

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        self._clear()


def budget(src, name):
    """the value of `constexpr int <name> = ...;` in micronet_b200/csrc/<src>"""
    text = open(os.path.join(ROOT, "micronet_b200", "csrc", src)).read()
    m = re.search(r"constexpr int %s = ([0-9*+\- ]+);" % name, text)
    assert m, (src, name)
    return int(eval(m.group(1)))      # e.g. "227 * 1024 - 3072"


def model_convs():
    """(name, B, C, H, W, K, R, stride, pad, groups) of every conv of the bench models (harness/models.py)"""
    out = []
    B = 256
    gc = [("gc1x1g2", 256, 32, 256, 1, 1, 0, 2), ("gc3x3g16", 256, 16, 512, 3, 1, 1, 16), ("gc1x1g4", 512, 16, 512, 1, 1, 0, 4),
          ("gc3x3g32", 512, 8, 1024, 3, 1, 1, 32), ("gc1x1g8", 1024, 8, 1024, 1, 1, 0, 8), ("gc_head", 1024, 8, 10, 1, 1, 0, 1)]
    nin = [("nin1x1a", 192, 32, 160, 1, 1, 0, 1), ("nin1x1b", 160, 32, 96, 1, 1, 0, 1), ("nin5x5", 96, 16, 192, 5, 1, 2, 1),
           ("nin1x1c", 192, 16, 192, 1, 1, 0, 1), ("nin3x3", 192, 8, 192, 3, 1, 1, 1), ("nin1x1d", 192, 8, 192, 1, 1, 0, 1),
           ("nin_head", 192, 8, 10, 1, 1, 0, 1)]
    for n, c, h, k, r, st, p, g in gc + nin:
        out.append((n, B, c, h, h, k, r, st, p, g))
    for hw, b, tag in ((32, 256, "res32"), (224, 64, "res224")):
        c, h = 64, hw
        out.append((f"{tag}_stem", b, 3, h, h, 64, 3, 1, 1, 1))
        for width in (64, 128, 256, 512):
            if width != 64:
                out.append((f"{tag}_{width}_s2", b, c, h, h, width, 3, 2, 1, 1))
                out.append((f"{tag}_{width}_sc", b, c, h, h, width, 1, 2, 0, 1))
                h //= 2
            out.append((f"{tag}_{width}", b, width, h, h, width, 3, 1, 1, 1))
            c = width
    return out


# ---- plans
def shape(B, Cc, H, W, K, R, st, pad, G):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def case_shape(s):
    """ConvShape of a case shape (B, C, H, W, K, R, S, stride, pad_h, pad_w, groups[, dilation])"""
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, S, st, ph, pw, G = s[:11]
    dil = s[11] if len(s) > 11 else 1
    return L.ConvShape(B, Cc, H, W, K, R, S, st, st, ph, pw, dil, dil, G)


def query(mode, sh, terms):
    """(code, error text, plan dict) of the host-only query of a launch mode: "fwd", "dgrad", "i8" or "wgrad" """
    from micronet_b200 import _lib as L
    lib = L.load()
    if mode == "wgrad":
        out = (C.c_int32 * len(WGRAD_FIELDS))()
        rc = lib.mnb_pk_wgrad_plan(C.byref(sh), terms[0], terms[1], out, len(out))
        names = WGRAD_FIELDS
    else:
        out = (C.c_int32 * len(CONV_FIELDS))()
        if mode == "i8":
            rc = lib.mnb_pk_i8_conv_plan(C.byref(sh), out, len(out))
        else:
            rc = lib.mnb_pk_conv_plan_ex(C.byref(sh), 0 if mode == "fwd" else 1, terms[0], terms[1], out, len(out))
        names = CONV_FIELDS
    text = lib.mnb_last_error() if rc else b""
    return rc, text, (dict(zip(names, list(out))) if rc == 0 else None)


def conv_plan(sh, mode, ta, tw):
    """plan of mnb_pk_conv for (shape, mode, terms); None if the shape is outside the cover"""
    return query("dgrad" if mode else "fwd", sh, (ta, tw))[2]


def wgrad_plan(sh, t_dy, t_x):
    return query("wgrad", sh, (t_dy, t_x))[2]


def i8_plan(sh):
    return query("i8", sh, (1, 1))[2]


def conv_signature(p):
    """what selects the code path of pk_conv_kernel: instance (SEG, Nt), M tiles per item, output phases"""
    return (bool(p["segmented"]), p["Nt"], p["MT"], p["ny"])


def wgrad_signature(p):
    """instance Nc, several tap groups, merged groups"""
    return (p["Nc"], p["tpg"] > 1, p["gm"] > 1)


def i8_signature(p, stride):
    """instance Nt of the int8 kernel, M tiles per item, phase-split operand"""
    return (p["Nt"], p["MT"], stride == 2)


# ---- fp64 references
def within(got, ref, R, c):
    """element-wise |got - ref| <= c * R; returns the worst err / R, which the message carries"""
    import torch
    assert not torch.isnan(got).any(), "outputs the kernel never wrote"
    err = (got.double() - ref).abs()
    ratio = (err / R.clamp_min(1e-300)).max().item()
    assert (err <= c * R).all(), f"worst err / R = {ratio:.3e} > c = {c:.3e}"
    return ratio


def fmaf32(a, b, c, stats=None):
    """fp32 fmaf(a, b, c) of float32 tensors (broadcasting), correctly rounded: t = a * b is exact in fp64, s = fl64(t + c)
    with its exact error e (TwoSum), and s rounded to fp32 - wrong only where s lies on an fp32 midpoint and e != 0, where
    the neighbour on e's side is the answer.  ``stats["midpoints"]`` counts the elements whose s is an fp32 midpoint."""
    import torch
    t = a.double() * b.double()                # exact: 24 x 24 significant bits
    c = c.double()
    s = t + c
    bb = s - t
    e = (t - (s - bb)) + (c - bb)
    r = s.float()
    r64 = r.double()
    toward = torch.where(s > r64, torch.full_like(r, float("inf")), torch.full_like(r, float("-inf")))
    nb = torch.nextafter(r, toward)
    mid = (s != r64) & ((s - r64).abs() * 2 == (nb.double() - r64).abs())
    # at a midpoint RN picked r (ties to even) from s alone; the exact value s + e lies on nb's side iff e points away from r
    up = mid & (e != 0) & ((e > 0) == (nb.double() > r64))
    if stats is not None:
        stats["midpoints"] = stats.get("midpoints", 0) + int(mid.sum())
    return torch.where(up, nb, r)
