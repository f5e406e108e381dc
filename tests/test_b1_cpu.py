"""CPU side of the binary tensor-core forward (csrc/mnb_b1.cu): the host-only cover and byte-count queries, a numpy replay of
the operand encoding (p / n activation halves, plus = [P | M] and minus = [M | P] weight columns, AND + popc) against a plain
convolution of the +-1 / ternary tensors (WB:11-36, 55-75, 181-195), and the compiled kernel's SASS: binary tensor-core
MMAs (BGMMA) with at most four warpgroup waits per function.  The GPU results are pinned by tests/test_gpu_b1_conv.py."""
import ctypes as C
import re
import shutil
import subprocess

import numpy as np
import pytest

# B, C, H, W, K, R, pad, groups
NIN = [(256, 192, 32, 32, 160, 1, 0, 1), (256, 160, 32, 32, 96, 1, 0, 1), (256, 96, 16, 16, 192, 5, 2, 1),
       (256, 192, 16, 16, 192, 1, 0, 1), (256, 192, 16, 16, 192, 1, 0, 1), (256, 192, 8, 8, 192, 3, 1, 1),
       (256, 192, 8, 8, 192, 1, 0, 1)]
NINGC_1X1 = [(256, 256, 32, 32, 256, 1, 0, 2), (256, 256, 32, 32, 256, 1, 0, 2), (256, 512, 16, 16, 512, 1, 0, 4),
             (256, 512, 16, 16, 512, 1, 0, 4), (256, 1024, 8, 8, 1024, 1, 0, 8)]
EDGE = [(1, 1, 9, 13, 3, 3, 1, 1), (1, 63, 9, 13, 5, 3, 1, 1), (1, 65, 1, 1, 1, 1, 0, 1), (2, 70, 9, 13, 33, 7, 3, 1),
        (2, 64, 7, 7, 24, 7, 0, 1), (3, 96, 7, 7, 40, 5, 2, 1), (2, 130, 9, 13, 66, 3, 1, 2), (1, 4096, 2, 2, 999, 1, 0, 1)]


def _sh(B, Cc, H, W, K, R, pad, G, stride=1, dil=1, S=None):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, Cc, H, W, K, R, R if S is None else S, stride, stride, pad, pad, dil, dil, G)


@pytest.mark.parametrize("shape", NIN + NINGC_1X1 + EDGE)
def test_cover_accepts(shape):
    from micronet_b200 import _lib as L
    assert L.load().mnb_b1_supported(C.byref(_sh(*shape))) == 1


@pytest.mark.parametrize("kw", [dict(stride=2), dict(dil=2), dict(S=1), dict(R=9, pad=4), dict(R=3, pad=2)],
                         ids=["stride2", "dilation2", "3x1", "9x9", "pad_beyond_half"])
def test_cover_refuses(kw):
    from micronet_b200 import _lib as L
    args = dict(B=2, Cc=64, H=16, W=16, K=32, R=3, pad=1, G=1)
    args.update(kw)
    sh = _sh(args.pop("B"), args.pop("Cc"), args.pop("H"), args.pop("W"), args.pop("K"), args.pop("R"), args.pop("pad"),
             args.pop("G"), **args)
    lib = L.load()
    assert lib.mnb_b1_supported(C.byref(sh)) == 0
    assert lib.mnb_b1_wimage_bytes(C.byref(sh)) == -1
    # refused before any launch: null device pointers are never touched
    assert lib.mnb_b1_conv_fwd(C.byref(sh), 16, 16, None, None, 16, 16, None) == L.E_UNSUPPORTED
    assert lib.mnb_b1_pack_weight(C.byref(sh), 16, 16, None) == L.E_UNSUPPORTED


def test_byte_counts_follow_the_layout():
    from micronet_b200 import _lib as L, xnor as X
    lib = L.load()
    # [B][G * ceil(C/g / 64)][H][W][16 B]
    assert lib.mnb_b1_act_bytes(2, 192, 8, 8, 1) == 2 * 3 * 64 * 16
    assert lib.mnb_b1_act_bytes(2, 130, 9, 13, 2) == 2 * 2 * 2 * 117 * 16
    assert lib.mnb_b1_act_bytes(1, 1, 1, 1, 1) == 16
    assert lib.mnb_b1_act_bytes(1, 10, 1, 1, 3) == -1
    # weights: [G][n-tiles][k-steps][taps][2][Nt][16 B], two columns per output channel, at most 192 per tile
    assert lib.mnb_b1_wimage_bytes(C.byref(_sh(*NIN[0]))) == 1 * 2 * 2 * 1 * 2 * 192 * 16   # 320 columns: 2 x 192
    assert lib.mnb_b1_wimage_bytes(C.byref(_sh(*NIN[2]))) == 1 * 2 * 1 * 25 * 2 * 192 * 16   # 384 columns: 2 x 192
    assert lib.mnb_b1_wimage_bytes(C.byref(_sh(*EDGE[0]))) == 1 * 1 * 1 * 9 * 2 * 32 * 16
    # post outputs: bit plane, bf16 plane, b1 plane of the consumer's groups (pooled)
    sh = _sh(*NIN[5])
    for fmt, og, pool, want in ((L.XNOR_BITS, 1, False, 256 * 6 * 64 * 4), (L.XNOR_PM1_BF16, 1, False, 256 * 192 * 64 * 2),
                                (L.XNOR_B1_PLANE, 1, False, 256 * 3 * 64 * 16), (L.XNOR_B1_PLANE, 2, True, 256 * 2 * 2 * 16 * 16),
                                (L.XNOR_PM1_BF16, 1, True, -1)):
        assert lib.mnb_b1_post_bytes(C.byref(sh), C.byref(X.post_struct(fmt, og, 1, pool))) == want
    # the XNOR entry points keep refusing the new format
    xs = _sh(4, 256, 8, 8, 256, 1, 0, 2)
    assert lib.mnb_xnor_post_bytes(C.byref(xs), C.byref(X.post_struct(L.XNOR_B1_PLANE, 1))) == -1


def _bits64(flags):
    """flags [..., n <= 64] of bool -> uint64 words (bit j = flags[..., j])"""
    w = np.zeros(flags.shape[:-1], dtype=np.uint64)
    for j in range(flags.shape[-1]):
        w |= flags[..., j].astype(np.uint64) << np.uint64(j)
    return w


def _popc(a):
    return np.vectorize(lambda v: bin(int(v)).count("1"), otypes=[np.int64])(a)


@pytest.mark.parametrize("cg", [1, 63, 64, 65, 130])
def test_encoding_gives_the_exact_sum(cg):
    """numpy replay of one output pixel's K steps: activation units [p | n] against weight columns plus / minus"""
    rng = np.random.default_rng(cg)
    a = rng.choice([-1, 1], size=cg)
    w = rng.integers(-1, 2, size=(5, cg))
    u = (cg + 63) // 64
    units = 2 * ((u + 1) // 2)                               # whole K steps: the last may carry a padding unit
    p = np.zeros((units, 64), bool); n = np.zeros((units, 64), bool)
    P = np.zeros((5, units, 64), bool); M = np.zeros((5, units, 64), bool)
    for c in range(cg):
        p[c // 64, c % 64] = a[c] == 1; n[c // 64, c % 64] = a[c] == -1
        P[:, c // 64, c % 64] = w[:, c] == 1; M[:, c // 64, c % 64] = w[:, c] == -1
    if units > u:   # a padding unit of the box holds arbitrary bits (the next group's channels): its weights are zero
        p[u:] = rng.random((units - u, 64)) < 0.5; n[u:] = ~p[u:]
    act = np.stack([_bits64(p), _bits64(n)], -1)                      # [units, 2]: the 128 bits of each unit
    plus = np.stack([_bits64(P), _bits64(M)], -1)                     # [5, units, 2]
    minus = np.stack([_bits64(M), _bits64(P)], -1)
    d_plus = _popc(act[None] & plus).sum(axis=(1, 2))
    d_minus = _popc(act[None] & minus).sum(axis=(1, 2))
    assert np.array_equal(d_plus - d_minus, w @ a)


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_has_binary_mmas_and_few_waits():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for name, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        if "b111conv_kernel" in name:
            funcs[name] = (len(re.findall(r"\bBGMMA\.64x\d+x256\.AND\.POPC\b", body)),
                           len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body)))
    nts = {int(m.group(1)) for n in funcs if (m := re.search(r"conv_kernelILi(\d+)ELb", n))}
    assert nts == {32, 64, 128, 192} and len(funcs) == 8, funcs
    assert all(c[0] >= 1 and c[1] <= 4 for c in funcs.values()), funcs
