"""Host side of the generic convolution kernels (mnb_conv_generic.cu), no GPU needed: a mirror of the geometry check, the
column-tile choice and the split-K weight-gradient plan, held against mnb_wgrad_scratch_bytes (= splits * K * Cg * R * S * 4
bytes) for the shared case list and a seeded sweep; the case list reaches every template instance, every cap of the
plan and both tile edges; bad shapes are refused before any launch."""
import ctypes as C

import numpy as np
import pytest

from tests.generic_conv_cases import CASES, conv_shape

BM, BK, NUM_SMS = 64, 16, 132   # mnb_conv_generic.cu tiles, MNB_NUM_SMS


def _lib():
    from micronet_b200 import _lib as L, build
    build.build()
    return L, L.load()


def geom(case):
    """make_geom: None where the shape is refused"""
    B, Cin, H, W, K, (R, S), (sh, sw), (ph, pw), (dh, dw), G = case
    if min(B, Cin, H, W, K, R, S, sh, sw, dh, dw, G) <= 0 or min(ph, pw) < 0 or Cin % G or K % G:
        return None
    P = (H + 2 * ph - dh * (R - 1) - 1) // sh + 1
    Q = (W + 2 * pw - dw * (S - 1) - 1) // sw + 1
    if P <= 0 or Q <= 0:
        return None
    return dict(B=B, C=Cin, H=H, W=W, K=K, RS=R * S, G=G, P=P, Q=Q, Cg=Cin // G, Ng=K // G)


def pick_bn(n):
    return 16 if n <= 16 else (32 if n <= 32 else 64)


def cdiv(a, b):
    return -(-a // b)


def wgrad_plan(g):
    """(bn, splits, k_per_split, binding cap) of wgrad_plan"""
    Nd, Kd = g["Cg"] * g["RS"], g["B"] * g["P"] * g["Q"]
    bn = pick_bn(Nd)
    tiles = cdiv(g["Ng"], BM) * cdiv(Nd, bn) * g["G"]
    want = max(1, NUM_SMS * 4 // tiles)
    maxs = max(1, Kd // (BK * 8))
    splits = min(want, maxs, 256)
    cap = "256" if splits == 256 else ("kd" if splits == maxs else "want")
    kps = cdiv(cdiv(Kd, splits), BK) * BK
    return bn, cdiv(Kd, kps), kps, cap


def launches(g):
    """per kernel: (template BN, GEMM M, GEMM N) as the entry points launch them"""
    Nd = g["Cg"] * g["RS"]
    return {"fwd": (pick_bn(g["Ng"]), g["B"] * g["P"] * g["Q"], g["Ng"]),
            "dgrad": (pick_bn(g["Cg"]), g["B"] * g["H"] * g["W"], g["Cg"]),
            "wgrad": (pick_bn(Nd), g["Ng"], Nd)}


def _scratch_bytes(lib, case):
    return int(lib.mnb_wgrad_scratch_bytes(C.byref(conv_shape(case))))


def test_plan_mirror_matches_the_library_on_the_cases():
    L, lib = _lib()
    for name, case in CASES.items():
        g = geom(case)
        assert g is not None, name
        _, splits, kps, _ = wgrad_plan(g)
        assert _scratch_bytes(lib, case) == splits * g["K"] * g["Cg"] * g["RS"] * 4, name
        Kd = g["B"] * g["P"] * g["Q"]
        assert kps % BK == 0 and (splits - 1) * kps < Kd <= splits * kps, name   # no empty split


def test_plan_mirror_matches_the_library_on_a_sweep():
    L, lib = _lib()
    rng = np.random.default_rng(20261017)
    caps, refused = set(), 0
    for _ in range(4000):
        G = int(rng.choice([1, 1, 1, 2, 3, 4, 8]))
        R, S = (int(v) for v in rng.integers(1, 8, 2))
        case = (int(rng.integers(1, 70)), G * int(rng.integers(1, 40)), int(rng.integers(1, 40)), int(rng.integers(1, 40)),
                G * int(rng.integers(1, 80)), (R, S), tuple(int(v) for v in rng.integers(1, 5, 2)),
                tuple(int(v) for v in rng.integers(0, 5, 2)), tuple(int(v) for v in rng.integers(1, 4, 2)), G)
        if rng.random() < 0.05:   # channels that groups do not divide
            case = case[:1] + (case[1] + 1,) + case[2:]
        g = geom(case)
        got = _scratch_bytes(lib, case)
        if g is None:
            refused += 1
            assert got == -1, case
            continue
        _, splits, _, cap = wgrad_plan(g)
        caps.add(cap)
        assert got == splits * g["K"] * g["Cg"] * g["RS"] * 4, case
    assert refused > 100 and caps == {"256", "kd", "want"}, (refused, caps)


def test_cases_reach_every_instance_cap_and_edge():
    """every case runs every path of test_gpu_generic_conv.py: forward on the integer and the fp32 path, dgrad with and
    without the STE, wgrad on codes and on fp32 activations"""
    bns = {"fwd": set(), "dgrad": set(), "wgrad": set()}
    ragged_m = {"fwd": False, "dgrad": False, "wgrad": False}
    two_cols = dict(ragged_m)
    caps, split_counts, ragged_split = set(), set(), False
    for case in CASES.values():
        g = geom(case)
        for kern, (bn, M, N) in launches(g).items():
            bns[kern].add(bn)
            ragged_m[kern] |= M % BM != 0
            two_cols[kern] |= N > bn
        _, splits, kps, cap = wgrad_plan(g)
        caps.add(cap)
        split_counts.add(splits)
        ragged_split |= g["B"] * g["P"] * g["Q"] % kps != 0 and splits > 1
    assert all(b == {16, 32, 64} for b in bns.values()), bns
    assert all(ragged_m.values()), ragged_m            # M % 64 != 0
    assert all(two_cols.values()), two_cols            # more than one grid.y tile
    assert 1 in split_counts and 256 in split_counts and "kd" in caps, (split_counts, caps)
    assert ragged_split
    g = geom(CASES["split_ragged"])
    assert wgrad_plan(g)[1:3] == (3, 176) and g["B"] * g["P"] * g["Q"] == 507
    assert wgrad_plan(geom(CASES["split_cap256"]))[1] == 256
    assert wgrad_plan(geom(CASES["split_single"]))[1] == 1


@pytest.mark.parametrize("bad, what", [
    ((2, 8, 4, 4, 8, (5, 5), (1, 1), (0, 0), (1, 1), 1), b"empty"),        # filter larger than the image
    ((2, 8, 4, 4, 8, (5, 5), (2, 2), (0, 0), (1, 1), 1), b"empty"),        # ... by one row, at stride 2
    ((2, 8, 3, 9, 8, (3, 3), (3, 1), (0, 0), (2, 1), 1), b"empty"),        # dilated filter, stride 3
    ((2, 6, 8, 8, 4, (3, 3), (1, 1), (1, 1), (1, 1), 4), b"groups"),       # 6 input channels, 4 groups
    ((2, 8, 8, 8, 6, (3, 3), (1, 1), (1, 1), (1, 1), 4), b"groups"),       # 6 output channels, 4 groups
    ((2, 8, 8, 8, 8, (3, 3), (0, 1), (1, 1), (1, 1), 1), b"stride"),       # zero stride
    ((2, 8, 8, 8, 8, (3, 3), (1, 1), (1, 1), (1, 0), 1), b"dilation"),     # zero dilation
    ((2, 8, 8, 8, 8, (3, 3), (1, 1), (-1, 1), (1, 1), 1), b"padding"),     # negative padding
])
def test_bad_shapes_are_refused_before_launch(bad, what):
    L, lib = _lib()
    assert geom(bad) is None
    fake = 4096   # never dereferenced: every call must be refused on the host
    sh = conv_shape(bad)
    ops = L.ConvOperands(a_f32=fake, w_f32=fake)
    assert lib.mnb_conv2d_fwd(C.byref(sh), C.byref(ops), fake, None) == -1
    assert what in lib.mnb_last_error()
    assert lib.mnb_conv2d_dgrad(C.byref(sh), fake, fake, None, None, fake, None) == -1
    assert what in lib.mnb_last_error()
    assert lib.mnb_conv2d_wgrad(C.byref(sh), fake, C.byref(ops), fake, fake, None) == -1
    assert what in lib.mnb_last_error()
    assert lib.mnb_conv2d_wgrad_cond(C.byref(sh), fake, C.byref(ops), fake, fake, fake, None) == -1
    assert lib.mnb_wgrad_scratch_bytes(C.byref(sh)) == -1
