"""Host side of mnb_pk_wgrad_taps (csrc/mnb_pk.cu): its cover among the bench models' convolutions, the plan's register,
shared-memory and accumulation-chain limits, refusals before any launch, and the compiled kernel (no spills, every
launched instance exercised by tests/test_gpu_pk_wgrad_taps.py)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from tests.pk_plan_util import LIMIT, RESERVED, budget, model_convs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAPS_LAYERS = {"gc3x3g16", "gc3x3g32"}
E_ARG = -1   # MNB_E_ARG


def _sh(B, Cc, H, W, K, R, st, pad, G):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def _plan(sh, t_dy, t_x):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * 12)()
    rc = L.load().mnb_pk_wgrad_taps_plan(C.byref(sh), t_dy, t_x, out, 12)
    return rc, list(out)


@pytest.mark.parametrize("conv", model_convs(), ids=lambda c: c[0])
def test_cover_is_exactly_the_grouped_3x3_layers(conv):
    from micronet_b200 import _lib as L
    name, B, Cc, H, W, K, R, st, pad, G = conv
    rc, _ = _plan(_sh(B, Cc, H, W, K, R, st, pad, G), 2, 1)
    assert (rc == 0) == (name in TAPS_LAYERS), (name, rc)
    if rc:
        assert rc == L.E_UNSUPPORTED


@pytest.mark.parametrize("terms", [(1, 1), (2, 1), (2, 2), (3, 1), (3, 3)])
@pytest.mark.parametrize("B", [1, 3, 37, 256])
@pytest.mark.parametrize("layer", [(256, 16, 512, 16), (512, 8, 1024, 32)], ids=["g16", "g32"])
def test_plan_limits(layer, B, terms):
    from micronet_b200 import _lib as L
    Cc, H, K, G = layer
    sh = _sh(B, Cc, H, H, K, 3, 1, 1, G)
    rc, v = _plan(sh, *terms)
    assert rc == 0
    blocks, splits, NI, nstage, BW, TH, spp, smem, acc, s_lo, s_hi, npairs = v
    assert blocks == G // 4 and acc == 9 * 16
    # registers: 144 accumulators within the 232 the MMA warpgroups raise to (128 * 40 + 256 * 232 = 384 * 168)
    assert 128 * 40 + 256 * 232 <= 384 * 168
    assert 2 <= nstage <= 8 and 0 < smem <= budget("mnb_pk.cu", "kSmemBudget") and smem + RESERVED <= LIMIT
    assert BW >= H + 2 and (BW * TH) % 16 == 0
    nstg = -(-B * -(-H // TH) // NI)
    assert splits == -(-nstg // spp) and (splits - 1) * spp < nstg
    assert spp * NI * (BW * TH // 16) * npairs <= 256, "accumulation chain longer than 256 MMAs"
    assert (s_lo | (s_hi << 31)) == splits * blocks * 9 * 64 * 128 * 4
    # the accumulation chains and the reduction of mnb_pk_wgrad: its merged block, raster, stages and batch splits
    old = (C.c_int32 * 10)()
    assert L.load().mnb_pk_wgrad_plan(C.byref(sh), *terms, old, 10) == 0
    Nc, n_ctiles, _, _, gm, o_splits, o_NI, o_nstage, o_BW, o_TH = list(old)
    assert (Nc, n_ctiles, gm, o_splits, o_NI, o_BW, o_TH) == (64, 1, 4, splits, NI, BW, TH)
    assert nstage >= o_nstage


@pytest.mark.parametrize("bad", [
    dict(R=5, pad=2), dict(R=1, pad=0), dict(st=2), dict(G=8, Cc=256), dict(G=16, K=256), dict(G=6, Cc=96, K=192),
    dict(pad=3), dict(H=1, pad=0), dict(W=127),
], ids=["5x5", "1x1", "stride2", "cin32", "cout16", "groups6", "pad3", "empty", "row129"])
def test_refuses_outside_the_cover_before_any_launch(bad):
    from micronet_b200 import _lib as L
    a = dict(B=4, Cc=256, H=16, W=16, K=512, R=3, st=1, pad=1, G=16)
    a.update(bad)
    sh = _sh(a["B"], a["Cc"], a["H"], a["W"], a["K"], a["R"], a["st"], a["pad"], a["G"])
    lib = L.load()
    n0 = L.launch_count()
    assert _plan(sh, 2, 1)[0] == L.E_UNSUPPORTED
    dummy = C.c_void_p(16)
    assert lib.mnb_pk_wgrad_taps(C.byref(sh), dummy, 2, dummy, 1, None, None, dummy, dummy, dummy, None) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def test_refuses_null_operands_and_bad_terms():
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = _sh(4, 256, 16, 16, 512, 3, 1, 1, 16)
    n0 = L.launch_count()
    dummy = C.c_void_p(16)
    assert lib.mnb_pk_wgrad_taps(C.byref(sh), None, 2, dummy, 1, None, None, dummy, dummy, dummy, None) == E_ARG
    assert lib.mnb_pk_wgrad_taps(C.byref(sh), dummy, 4, dummy, 1, None, None, dummy, dummy, dummy, None) == E_ARG
    assert _plan(sh, 0, 1)[0] == E_ARG
    assert L.launch_count() == n0


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_kernel_has_no_spills():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = [(n, u) for n, u in re.findall(r"Function (\S+?):\s*\n\s*(.*)", out) if "pk_wgrad_taps_kernel" in n]
    assert len(funcs) == 1, "exactly one instance of pk_wgrad_taps_kernel, launched by every GPU case"
    usage = funcs[0][1]
    assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), usage
    static = int(re.search(r"SHARED:(\d+)", usage).group(1)) - RESERVED
    assert static + budget("mnb_pk.cu", "kSmemBudget") <= LIMIT


def test_gpu_cases_cover_the_bench_layers_and_the_edges():
    """the GPU file launches the kernel at both bench layers (batch 256 and small), a short last split, a short last stage
    (several sub-blocks per stage), padding 0 and 2, one to three pieces per operand, and a two-stage raster"""
    import importlib
    gpu = importlib.import_module("tests.test_gpu_pk_wgrad_taps")
    seen = set()
    for case, terms in gpu.CASES:
        B, Cc, H, W, K, pad, G = case
        rc, v = _plan(_sh(B, Cc, H, W, K, 3, 1, pad, G), *terms)
        assert rc == 0, case
        blocks, splits, NI, nstage, BW, TH, spp = v[:7]
        nsub = B * -(-(H + 2 * pad - 2) // TH)
        nstg = -(-nsub // NI)
        seen.add("g16" if (Cc, H, K) == (256, 16, 512) else "g32" if (Cc, H, K) == (512, 8, 1024) else "other")
        if B == 256:
            seen.add("b256")
        if nstg % spp:
            seen.add("short split")
        if nsub % NI:
            seen.add("short stage")
        seen |= {f"pad{pad}", f"ta{terms[0]}", f"tx{terms[1]}", f"nstage{min(nstage, 3)}"}
    want = {"g16", "g32", "other", "b256", "short split", "short stage", "pad0", "pad1", "pad2", "ta1", "ta2", "ta3",
            "tx1", "tx2", "tx3", "nstage2", "nstage3"}
    assert want <= seen, want - seen
