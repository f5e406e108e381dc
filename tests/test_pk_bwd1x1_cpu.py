"""Host side of mnb_pk_bwd1x1 (csrc/mnb_pk.cu): its cover among the bench models' convolutions, the plan against
mnb_pk_wgrad_plan's (raster, batch splits, stage order), the shared-memory budget, every refusal before any launch, and
the compiled kernel (no spills)."""
import ctypes as C
import re
import shutil
import subprocess

import pytest

from tests.pk_conv_bench_launches import BENCH_LAUNCHES
from tests.pk_plan_util import LIMIT, RESERVED, budget

E_ARG = -1   # MNB_E_ARG


def _sh(B, Cc, H, W, K, R=1, st=1, pad=0, G=1):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def _plan(sh, t_dy=2, t_x=1, t_w=1):
    from micronet_b200 import _lib as L
    out = (C.c_int32 * 15)()
    rc = L.load().mnb_pk_bwd1x1_plan(C.byref(sh), t_dy, t_x, t_w, out, 15)
    return rc, list(out)


def _wgrad_launches():
    return sorted({(f, (t_dy, t_x)) for _, kind, f, _, t_dy, t_x in BENCH_LAUNCHES if kind == "wgrad"})


@pytest.mark.parametrize("launch", _wgrad_launches(), ids=lambda l: "x".join(map(str, l[0])))
def test_cover_is_exactly_the_grouped_1x1_layers(launch):
    """among the bench weight-gradient launches: the 1x1 grouped layers of NIN-GC (128 channels per group)"""
    from micronet_b200 import _lib as L
    f, (t_dy, t_x) = launch
    sh = L.ConvShape(*f)
    rc, _ = _plan(sh, t_dy, t_x, 1)
    B, Cc, H, W, K, R = f[:6]
    G = f[-1]
    want = R == 1 and G > 1 and B == 256 and Cc // G == 128 and K // G == 128
    assert (rc == 0) == want, (f, rc)
    if rc:
        assert rc == L.E_UNSUPPORTED


def test_cover_has_the_five_wbwtab_layers():
    layers = [f for w, kind, f, *_ in BENCH_LAUNCHES if w == "nin_gc_wbwtab_w3a2" and kind == "wgrad"]
    covered = {f for f in layers if _plan(_sh(*f[:5], R=f[5], st=f[7], pad=f[9], G=f[-1]))[0] == 0}
    # L1 / L2 share 256 -> 256 g2 @ 32, L4 / L5 512 -> 512 g4 @ 16, L7 is 1024 -> 1024 g8 @ 8
    assert {(f[1], f[2], f[-1]) for f in covered} == {(256, 32, 2), (512, 16, 4), (1024, 8, 8)}


@pytest.mark.parametrize("terms", [(1, 1, 1), (2, 1, 1), (1, 2, 2), (2, 1, 3)])
@pytest.mark.parametrize("shape", [(256, 256, 32, 32, 256, 2), (256, 512, 16, 16, 512, 4), (256, 1024, 8, 8, 1024, 8),
                                   (5, 128, 32, 32, 64, 1), (7, 64, 16, 16, 128, 1), (3, 192, 8, 8, 96, 2),
                                   (9, 256, 11, 16, 256, 2)],
                         ids=["L1", "L4", "L7", "cin128-cout64", "cin64-cout128", "g2-96-48", "partial"])
def test_plan_matches_the_wgrad_plan(shape, terms):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, G = shape
    sh = _sh(B, Cc, H, W, K, G=G)
    rc, v = _plan(sh, *terms)
    assert rc == 0, rc
    groups, splits, NI, nstage, BW, TH, spp, smem, nsub, nstg, chain, s_lo, s_hi, npairs, Nc = v
    old = (C.c_int32 * 16)()
    assert L.load().mnb_pk_wgrad_plan(C.byref(sh), terms[0], terms[1], old, 16) == 0
    o = list(old)
    o_Nc, o_nct, o_tpg, o_ntg, o_gm, o_splits, o_NI, _, o_BW, o_TH, o_nkt, o_nkph, o_spp, o_nsub, _, o_nstg = o
    assert (o_nct, o_tpg, o_ntg, o_gm, o_nkt, o_nkph) == (1, 1, 1, 1, 1, 1)
    assert (groups, Nc, splits, NI, BW, TH, spp, nsub, nstg) == (G, o_Nc, o_splits, o_NI, o_BW, o_TH, o_spp, o_nsub, o_nstg)
    assert BW * TH == 64
    assert 2 <= nstage <= 8 and 0 < smem <= budget("mnb_pk.cu", "kSmemBudget") and smem + RESERVED <= LIMIT
    assert (s_lo | (s_hi << 31)) == splits * G * Nc * 128 * 4
    # the data-gradient chain of mnb_pk_conv's plan: piece pairs x 16-channel K-steps over the output channels of a group
    pairs_dg = sum(1 for a in range(terms[0]) for b in range(terms[2]) if a + b <= max(terms[0], terms[2]) - 1)
    assert chain == pairs_dg * -(-(K // G) // 16)


# (shape overrides, piece counts (dy, x, w), environment, the refusal text of make_bwd_plan)
REFUSALS = [
    (dict(R=3, pad=1), (2, 1, 1), {}, "filter is not 1x1"),
    (dict(st=2), (2, 1, 1), {}, "stride or dilation != 1"),
    (dict(pad=1), (2, 1, 1), {}, "padding != 0"),
    (dict(Cc=512, K=512), (2, 1, 1), {}, "more than 128 channels per group"),
    (dict(Cc=256, K=512), (2, 1, 1), {}, "more than 128 channels per group"),
    (dict(Cc=200, K=200), (2, 1, 1), {}, "group-padded operand planes"),
    (dict(Cc=128, K=128), (2, 1, 1), {}, "weight-gradient block is not one whole group"),
    (dict(H=2, W=2), (2, 1, 1), {}, "sub-block raster is not 64 positions"),
    (dict(H=32, W=48), (2, 1, 1), {}, "sub-block raster is not 64 positions"),
    (dict(Cc=80, K=80, G=1), (2, 1, 1), {}, "data-gradient N tile differs from the weight-gradient tile"),
    (dict(), (2, 1, 1), {"MNB_PK_SEG_MMAS": "4"}, "segmented data-gradient plan"),
    (dict(), (2, 1, 2), {}, "data-gradient K-steps beyond the dy box"),
]


@pytest.mark.parametrize("bad,terms,env,why", REFUSALS, ids=[f"{r[3][:24]}-{i}" for i, r in enumerate(REFUSALS)])
def test_refuses_outside_the_cover_before_any_launch(bad, terms, env, why, monkeypatch):
    from micronet_b200 import _lib as L
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    a = dict(B=4, Cc=256, H=16, W=16, K=256, R=1, st=1, pad=0, G=2)
    a.update(bad)
    sh = _sh(a["B"], a["Cc"], a["H"], a["W"], a["K"], a["R"], a["st"], a["pad"], a["G"])
    lib = L.load()
    n0 = L.launch_count()
    assert _plan(sh, *terms)[0] == L.E_UNSUPPORTED
    assert why in lib.mnb_last_error().decode()
    d = C.c_void_p(16)
    assert lib.mnb_pk_bwd1x1(C.byref(sh), d, terms[0], d, terms[1], d, terms[2], 1.0, None, 1.0, d, None, None, d, d, d,
                             None) == L.E_UNSUPPORTED
    assert why in lib.mnb_last_error().decode()
    assert L.launch_count() == n0


def test_every_refusal_in_the_source_has_a_case():
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "micronet_b200", "csrc",
                            "mnb_pk.cu")).read()
    body = src[src.index("static int make_bwd_plan"):src.index("struct BwdParams")]
    reasons = set(re.findall(r'return no\("([^"]+)"\)', body))
    missing = reasons - {r[3] for r in REFUSALS}
    # (a 64-position sub-block is at most (227 KB - 2 KB) / 4 - the wgrad raster's first pass - so two stages of it always
    # fit next to a weight image of three 32 KB pieces)
    assert missing <= {"fewer than two stages fit next to the weight image"}, missing


def test_refuses_null_operands_and_bad_terms():
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = _sh(4, 256, 16, 16, 256, G=2)
    n0 = L.launch_count()
    d = C.c_void_p(16)
    assert lib.mnb_pk_bwd1x1(C.byref(sh), None, 2, d, 1, d, 1, 1.0, None, 1.0, d, None, None, d, d, d, None) == E_ARG
    assert lib.mnb_pk_bwd1x1(C.byref(sh), d, 2, d, 1, None, 1, 1.0, None, 1.0, d, None, None, d, d, d, None) == E_ARG
    assert lib.mnb_pk_bwd1x1(C.byref(sh), d, 4, d, 1, d, 1, 1.0, None, 1.0, d, None, None, d, d, d, None) == E_ARG
    assert _plan(sh, 2, 1, 0)[0] == E_ARG
    assert L.launch_count() == n0


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_kernel_has_no_spills():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = [(n, u) for n, u in re.findall(r"Function (\S+?):\s*\n\s*(.*)", out) if "pk_bwd1x1_kernel" in n]
    assert len(funcs) == 4, "pk_bwd1x1_kernel<32, 64, 96, 128>"
    for name, usage in funcs:
        assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), (name, usage)
        static = int(re.search(r"SHARED:(\d+)", usage).group(1)) - RESERVED
        assert static + budget("mnb_pk.cu", "kSmemBudget") <= LIMIT
