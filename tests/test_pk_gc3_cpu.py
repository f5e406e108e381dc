"""Host side of mnb_pk_gc3_conv / mnb_pk_gc3_conv_codes (csrc/mnb_pk.cu): the cover among the bench models' convolutions,
refusals before any launch, the data-gradient MMA chain against mnb_pk_conv's plan, and the compiled kernels (no spills,
at most the wgmma waits tests/test_wgmma_issue_cpu.py allows)."""
import ctypes as C
import re
import shutil
import subprocess

import pytest

from tests.pk_plan_util import LIMIT, RESERVED, budget, model_convs

GC3_LAYERS = {"gc3x3g16", "gc3x3g32"}
E_ARG = -1   # MNB_E_ARG


def _sh(B, Cc, H, W, K, R, st, pad, G):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def _plan(sh, mode, ta, tw):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * (10 + 4 * 128))()
    rc = L.load().mnb_pk_gc3_plan(C.byref(sh), mode, ta, tw, out, len(out))
    return rc, list(out)


@pytest.mark.parametrize("conv", model_convs(), ids=lambda c: c[0])
def test_cover_is_exactly_the_grouped_3x3_layers(conv):
    from micronet_b200 import _lib as L
    name, B, Cc, H, W, K, R, st, pad, G = conv
    for mode, ta, tw in ((0, 1, 1), (1, 2, 1)):
        rc, _ = _plan(_sh(B, Cc, H, W, K, R, st, pad, G), mode, ta, tw)
        assert (rc == 0) == (name in GC3_LAYERS), (name, mode, rc)
        if rc:
            assert rc == L.E_UNSUPPORTED


def _pairs(ta, tw):
    """piece products of make_pairs: i + j <= max(ta, tw) - 1, smallest first"""
    lim = max(ta, tw) - 1
    return [(a, s - a) for s in range(lim, -1, -1) for a in range(ta) if 0 <= s - a < tw]


@pytest.mark.parametrize("B", [1, 3, 37, 256])
@pytest.mark.parametrize("pad", [0, 1, 2])
@pytest.mark.parametrize("layer", [(256, 16, 512, 16), (512, 8, 1024, 32)], ids=["g16", "g32"])
def test_data_gradient_chain_is_the_plan_of_mnb_pk_conv(layer, pad, B):
    """every dx element sees the chain of make_plan(mode 1): K chunks -> piece pairs -> taps -> K-steps"""
    from micronet_b200 import _lib as L
    Cc, H, K, G = layer
    sh = _sh(B, Cc, H, H, K, 3, 1, pad, G)
    rc, v = _plan(sh, 1, 2, 1)
    assert rc == 0
    old = (C.c_int32 * 21)()
    assert L.load().mnb_pk_conv_plan_ex(C.byref(sh), 1, 2, 1, old, 21) == 0
    CC, chunks, segmented, npairs = old[5], old[6], old[16], old[18]
    assert not segmented and v[8] == old[2] == 16
    taps = [r * 3 + s for r in range(3) for s in range(3)]
    want = [(t, a, b, cc * (CC // 16) + j) for cc in range(chunks) for a, b in _pairs(2, 1) for t in taps
            for j in range(CC // 16)]
    assert len(_pairs(2, 1)) == npairs
    n = v[7]
    assert n == len(want) == 36
    assert [tuple(v[10 + 4 * i:14 + 4 * i]) for i in range(n)] == want


@pytest.mark.parametrize("B", [1, 5, 256])
@pytest.mark.parametrize("layer", [(256, 16, 512, 16), (512, 8, 1024, 32)], ids=["g16", "g32"])
def test_plan_limits(layer, B):
    Cc, H, K, G = layer
    for mode, ta, nt in ((0, 1, 32), (1, 2, 16)):
        rc, v = _plan(_sh(B, Cc, H, H, K, 3, 1, 1, G), mode, ta, 1)
        assert rc == 0
        gb, tb, nmb, nstage, smem, ctas, tiles, nchain, Nt, ncons = v[:10]
        assert Nt == nt and G % gb == 0 and 1 <= tb <= B and tiles == -(-B // tb)
        assert nmb * 64 >= (tb - 1) * (H + 2) ** 2 + (H - 1) * (H + 2) + H, "M tile shorter than the image raster"
        assert nmb * nt // 2 <= 96, "accumulators over the register budget"
        # every ring slot belongs to one MMA warpgroup (stage k: slot k % nstage, warpgroup k % ncons)
        assert ncons == 3 and nstage % ncons == 0 and ncons <= nstage <= 8 and 0 < smem <= budget("mnb_pk.cu", "kGc3SmemBudget")
        assert ctas <= 132 and ctas % (G // gb) == 0


@pytest.mark.parametrize("bad", [
    dict(R=5, pad=2), dict(R=1, pad=0), dict(st=2), dict(G=8, Cc=256), dict(G=16, K=256), dict(G=6, Cc=96, K=192),
    dict(pad=3), dict(H=1, pad=0),
], ids=["5x5", "1x1", "stride2", "cin32", "cout16", "groups6", "pad3", "empty"])
def test_refuses_outside_the_cover_before_any_launch(bad):
    from micronet_b200 import _lib as L
    a = dict(B=4, Cc=256, H=16, W=16, K=512, R=3, st=1, pad=1, G=16)
    a.update(bad)
    sh = _sh(a["B"], a["Cc"], a["H"], a["W"], a["K"], a["R"], a["st"], a["pad"], a["G"])
    lib = L.load()
    n0 = L.launch_count()
    d = C.c_void_p(16)
    for mode, ta in ((0, 1), (1, 2)):
        assert _plan(sh, mode, ta, 1)[0] == L.E_UNSUPPORTED
        assert lib.mnb_pk_gc3_conv(C.byref(sh), mode, d, ta, d, 1, None, None, 1.0, None, None, 1.0, d, d, None) == L.E_UNSUPPORTED
    assert lib.mnb_pk_gc3_conv_codes(C.byref(sh), d, 1, d, 1, None, None, 1.0, None, 1, d, d, d, None) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def test_refuses_other_piece_counts_and_null_operands():
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = _sh(4, 256, 16, 16, 512, 3, 1, 1, 16)
    n0 = L.launch_count()
    d = C.c_void_p(16)
    # forward: one piece each; data gradient: two dy pieces, one weight piece
    for mode, ta, tw in ((0, 2, 1), (0, 1, 2), (1, 1, 1), (1, 3, 1), (1, 2, 2)):
        assert _plan(sh, mode, ta, tw)[0] == L.E_UNSUPPORTED, (mode, ta, tw)
    assert _plan(sh, 2, 1, 1)[0] == E_ARG
    assert _plan(sh, 0, 0, 1)[0] == E_ARG
    assert lib.mnb_pk_gc3_conv(C.byref(sh), 0, None, 1, d, 1, None, None, 1.0, None, None, 1.0, d, d, None) == E_ARG
    assert lib.mnb_pk_gc3_conv(C.byref(sh), 0, d, 1, d, 1, None, None, 1.0, None, None, 1.0, None, d, None) == E_ARG
    assert lib.mnb_pk_gc3_conv_codes(C.byref(sh), d, 1, d, 1, None, None, 1.0, None, 1, None, d, d, None) == E_ARG
    # a level bound whose sums may leave int16
    assert lib.mnb_pk_gc3_conv_codes(C.byref(sh), d, 1, d, 1, None, None, 1.0, None, 300, d, d, d, None) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def _gc3_functions(flag):
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", flag, L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return out


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_kernels_have_no_spills_and_fit_shared_memory():
    out = _gc3_functions("-res-usage")
    funcs = [(n, u) for n, u in re.findall(r"Function (\S+?):\s*\n\s*(.*)", out) if "pk_gc3_kernel" in n]
    assert len(funcs) == 2, "one instance per N tile (32: forward, 16: data gradient)"
    for n, usage in funcs:
        assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), (n, usage)
        static = int(re.search(r"SHARED:(\d+)", usage).group(1)) - RESERVED
        assert static + budget("mnb_pk.cu", "kGc3SmemBudget") + RESERVED <= LIMIT, (n, usage)


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_kernels_do_not_wait_after_every_wgmma():
    from tests.test_wgmma_issue_cpu import MAX_WAITS
    out = _gc3_functions("-sass")
    seen = 0
    for name, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        if "pk_gc3_kernel" not in name:
            continue
        seen += 1
        assert re.search(r"\bHGMMA\.", body), name
        assert len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body)) <= MAX_WAITS, name
    assert seen == 2


def test_refuses_unaligned_tensors_before_any_launch():
    """an operand or output off a 16-byte boundary is refused (the caller then takes mnb_pk_conv / mnb_pk_conv_codes)"""
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = _sh(4, 256, 16, 16, 512, 3, 1, 1, 16)
    n0 = L.launch_count()
    d, odd = C.c_void_p(16), C.c_void_p(20)
    assert lib.mnb_pk_gc3_conv(C.byref(sh), 0, d, 1, d, 1, None, None, 1.0, None, None, 1.0, odd, d, None) == L.E_UNSUPPORTED
    assert lib.mnb_pk_gc3_conv(C.byref(sh), 1, odd, 2, d, 1, None, None, 1.0, None, None, 1.0, d, d, None) == L.E_UNSUPPORTED
    assert lib.mnb_pk_gc3_conv_codes(C.byref(sh), d, 1, odd, 1, None, None, 1.0, None, 1, d, d, d, None) == L.E_UNSUPPORTED
    assert L.launch_count() == n0
