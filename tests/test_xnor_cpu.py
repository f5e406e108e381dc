"""CPU side of the bit-packed XNOR-popcount forward (csrc/mnb_xnor.cu): the host-only C-ABI queries, and a numpy replay of the
kernel's arithmetic - bit planes, sign / non-zero weight words, `popc(N) - 2 popc(N & (A ^ S))`, out-of-image taps read as
A = 0 and corrected through the 2-D prefix table of per-tap weight sums - against a plain convolution of the +-1 / ternary
tensors (WB:11-36, 55-75, 181-195).  The GPU kernel itself is pinned by tests/test_gpu_xnor.py; this test keeps the algorithm
and the layouts checkable without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as TF


def _popc(a):
    a = a.astype(np.uint64)
    return np.array([bin(int(v)).count("1") for v in a.ravel()], dtype=np.int64).reshape(a.shape)


def _pack_bits(flags):
    """flags [..., n <= 32] of bool -> uint32 words (bit j = flags[..., j])"""
    w = np.zeros(flags.shape[:-1], dtype=np.uint64)
    for j in range(flags.shape[-1]):
        w |= flags[..., j].astype(np.uint64) << np.uint64(j)
    return w


def xnor_conv_model(x, w, stride, pad, groups):
    """numpy replay of mnb_xnor_pack_act + mnb_xnor_pack_weight + xnor::conv_kernel (integer sums)"""
    B, Cc, H, W = x.shape
    K, cg, R, S = w.shape
    kg = K // groups
    nw = (cg + 31) // 32
    P, Q = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
    # activation bits [B][G][nw][H][W]: bit = not (x < 0)
    abits = np.zeros((B, groups, nw, H, W), dtype=np.uint64)
    for g in range(groups):
        for n in range(nw):
            ch = x[:, g * cg + 32 * n: g * cg + min(32 * n + 32, cg)]          # [B, <=32, H, W]
            abits[:, g, n] = _pack_bits(np.moveaxis(~(ch < 0), 1, -1))
    # weight words [K][tap][nw] (sign, non-zero), per-tap sums, prefix table
    ws = np.zeros((K, R * S, nw), dtype=np.uint64)
    wn = np.zeros_like(ws)
    wsum = np.zeros((K, R, S), dtype=np.int64)
    for n in range(nw):
        blk = w[:, 32 * n: min(32 * n + 32, cg)]                                  # [K, <=32, R, S]
        ws[:, :, n] = _pack_bits(np.moveaxis(blk > 0, 1, -1)).reshape(K, R * S)
        wn[:, :, n] = _pack_bits(np.moveaxis(blk != 0, 1, -1)).reshape(K, R * S)
    wsum[:] = w.sum(axis=1)
    nz_total = _popc(wn).sum(axis=(1, 2))
    prefix = np.zeros((K, R + 1, S + 1), dtype=np.int64)
    prefix[:, 1:, 1:] = wsum.cumsum(axis=1).cumsum(axis=2)
    out = np.zeros((B, K, P, Q), dtype=np.int64)
    for b in range(B):
        for p in range(P):
            for q in range(Q):
                ih0, iw0 = p * stride - pad, q * stride - pad
                r0, r1 = max(0, -ih0), max(max(0, -ih0), min(R, H - ih0))
                s0, s1 = max(0, -iw0), max(max(0, -iw0), min(S, W - iw0))
                for g in range(groups):
                    a = np.zeros((R * S, nw), dtype=np.uint64)                    # out-of-image taps read 0
                    for r in range(r0, r1):
                        for s_ in range(s0, s1):
                            a[r * S + s_] = abits[b, g, :, ih0 + r, iw0 + s_]
                    ks = slice(g * kg, (g + 1) * kg)
                    cnt = _popc(wn[ks] & (a[None] ^ ws[ks])).sum(axis=(1, 2))
                    acc = nz_total[ks] - 2 * cnt
                    pk = prefix[ks]
                    rect = pk[:, r1, s1] - pk[:, r0, s1] - pk[:, r1, s0] + pk[:, r0, s0]
                    out[b, ks, p, q] = acc + pk[:, R, S] - rect
    return out


CASES = [  # B, C, H, W, K, R, stride, pad, groups, ternary
    (2, 32, 5, 6, 8, 1, 1, 0, 2, True),
    (2, 16, 6, 5, 8, 3, 1, 1, 1, True),      # 16 channels: half-used words
    (1, 48, 7, 7, 6, 3, 2, 1, 2, False),     # stride 2, ragged 24-channel groups
    (1, 40, 6, 6, 4, 5, 1, 2, 1, True),      # 5x5, two words with a ragged tail
    (1, 8, 4, 4, 4, 3, 1, 2, 1, True),       # padding wider than 'same': pixels whose taps are all outside
]


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_xnor_arithmetic_model_matches_a_convolution(case):
    B, Cc, H, W, K, R, st, pad, G, tern = case
    g = torch.Generator().manual_seed(sum(int(v) for v in case))
    x = torch.randn(B, Cc, H, W, generator=g)
    x[0, 0, 0, 0] = 0.0                                           # sign(0) -> +1
    w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g) if tern else torch.randint(0, 2, (K, Cc // G, R, R), generator=g) * 2 - 1
    ref = TF.conv2d(torch.where(x < 0, -1.0, 1.0).double(), w.double(), None, st, pad, 1, G).numpy()
    got = xnor_conv_model(x.numpy(), w.numpy().astype(np.int64), st, pad, G)
    assert np.array_equal(got, ref.astype(np.int64))


@pytest.mark.parametrize("cg,groups", [(24, 3), (77, 2), (81, 2), (16, 16), (64, 2)])
def test_unpack_reads_each_channel_at_its_bit_within_the_group(cg, groups):
    """xnor.unpack (functional.materialized of a frozen layer's bit plane) against the layout of the numpy packer above:
    channel j of a group sits at bit j % 32 of word j // 32, also when C/g is not a multiple of 32 (the pruned NIN-GC)"""
    from micronet_b200 import xnor as X
    g = torch.Generator().manual_seed(cg * groups)
    x = torch.randn(2, cg * groups, 3, 5, generator=g)
    nw = (cg + 31) // 32
    words = np.zeros((2, groups, nw, 3, 5), dtype=np.uint64)
    for gi in range(groups):
        for n in range(nw):
            ch = x[:, gi * cg + 32 * n: gi * cg + min(32 * n + 32, cg)].numpy()
            words[:, gi, n] = _pack_bits(np.moveaxis(~(ch < 0), 1, -1))
    bits = torch.from_numpy(words.astype(np.uint32).view(np.int32).reshape(-1))
    assert torch.equal(X.unpack(bits, x.shape, groups), torch.where(x < 0, -1.0, 1.0))


def test_xnor_host_queries():
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = L.ConvShape(4, 256, 16, 16, 512, 3, 3, 1, 1, 1, 1, 1, 1, 16)
    assert lib.mnb_xnor_supported(C.byref(sh)) == 1
    assert lib.mnb_xnor_act_bytes(4, 256, 16, 16, 16) == 4 * 16 * 1 * 256 * 4          # one (half-used) word per group
    nw, TW = 1, 9
    assert lib.mnb_xnor_wimage_bytes(C.byref(sh)) == 512 * (2 * TW + 1 + 16) * 4
    assert lib.mnb_xnor_act_bytes(4, 250, 16, 16, 16) == -1                                # channels not divisible by groups
    for bad in (L.ConvShape(4, 256, 16, 16, 512, 3, 3, 1, 1, 1, 1, 2, 2, 16),              # dilation
                L.ConvShape(4, 256, 16, 16, 512, 7, 7, 1, 1, 3, 3, 1, 1, 16),              # 7x7: no kernel variant
                L.ConvShape(4, 2048, 16, 16, 64, 3, 3, 1, 1, 1, 1, 1, 1, 1)):              # 64 words per tap
        assert lib.mnb_xnor_supported(C.byref(bad)) == 0
        assert lib.mnb_xnor_wimage_bytes(C.byref(bad)) == -1


def test_reciprocal_divmod_is_exact_on_its_range():
    """pk::FastDiv (mnb_pk.cu): q = trunc(float(n) * (1 / float(d))) corrected by one step; exact for n < 2^22 (the launcher
    rejects larger index spaces).  Same arithmetic in numpy float32."""
    rng = np.random.default_rng(0)
    for d in list(range(1, 260)) + [511, 768, 1024, 2047, 3072, 4096, 65535, (1 << 22) - 1]:
        inv = np.float32(1.0) / np.float32(d)
        n = np.concatenate([rng.integers(0, 1 << 22, 3000), np.arange(0, 3000), np.arange((1 << 22) - 3000, 1 << 22)]).astype(np.uint32)
        q = np.trunc(n.astype(np.float32) * inv).astype(np.int64)
        r = n.astype(np.int64) - q * d
        lo = r < 0
        q[lo] -= 1; r[lo] += d
        hi = r >= d
        q[hi] += 1; r[hi] -= d
        assert np.array_equal(q, n // d) and np.array_equal(r, n % d), d
