"""The fused BatchNorm producers, kernel by kernel, at the bench models' planes and at their decision edges:

* mnb_bn_sign_fwd (v4 / scalar), mnb_bn_sign_fwd_packed (VEC 4 / 2 / 1, with and without y), mnb_bn_sign_pool_fwd and
  mnb_bn_relu_quant_pack_fwd against an fp32 emulation of the documented formula bn = fma(fl(x - mu), fl(gamma invstd),
  beta): every decision (sign with 0 -> +1, saturate-STE pass bit |bn| < 1, DoReFa level, relu-and-clamp mask, pooled
  arg-max) bit for bit, every output word written, nothing past the end touched;
* the same decisions against plain fp64 BatchNorm semantics (nn.functional.batch_norm, then the oracle's binarizer /
  DoReFa quantizer): they may differ only within the fp32 rounding of a decision boundary;
* mnb_bn_sign_bwd / mnb_bn_sign_pool_bwd (training 1, 0 and 2 = reduce only) and the two _pack apply passes against fp64,
  with bounds derived from the number of fp32 roundings each kernel puts between the exact value and its result
  (u = 2^-24), and the packed gradient pieces decoded and checked exactly.

Each kernel is handed mean / invstd / gamma / beta directly (not statistics it computes itself), so these tests do not
depend on mnb_bn_batch_stats (tests/test_gpu_quant_kernels.py pins that one).  Every case asserts the launch path it
expects through a Python restatement of the host-side choice (fwd_path, bwd_path, pack_vec, plane_splits below)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as TF

from tests.test_gpu_quant_kernels import NUM_SMS, U, _eq, _first_diff, _gen

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U64 = 2.0 ** -53
E_UNSUPPORTED = -2
SPLIT_SLOTS = 32          # FUSED_SPLITS in mnb_fused.cu


# ============================================================================ launch-path restatements (mnb_fused.cu,
# mnb_conv_packed.cu, mnb_pk.cu).  Pointers are integer addresses; None stands for NULL (always "aligned").
def _aligned(a, *ptrs):
    return all(p is None or p % a == 0 for p in ptrs)


def fwd_path(n, hw, x, y):
    """mnb_bn_sign_fwd: planes_vectorizable(n, hw, x, y) -> bn_sign_fwd_v4_kernel, else the scalar bn_sign_fwd_kernel"""
    return "v4" if hw % 4 == 0 and n < 2 ** 31 and _aligned(16, x, y) else "scalar"


def bwd_path(n, hw, x, g, dx):
    """mnb_bn_sign_bwd: planes_vectorizable(n, hw, x, g, dx) -> the VEC reduce / apply kernels, else the scalar ones"""
    return "vec" if hw % 4 == 0 and n < 2 ** 31 and _aligned(16, x, g, dx) else "scalar"


def pack_vec(hw, *ptrs):
    """VEC of bn_sign_bwd_pack_kernel (ptrs = g, x, dx) and of bn_sign_packed_fwd_kernel (ptrs = x, y): 4 for hw % 128 == 0
    and 16-byte aligned pointers, 2 for hw % 64 == 0 and 8-byte aligned ones, else 1"""
    if hw % 128 == 0 and _aligned(16, *ptrs):
        return 4
    if hw % 64 == 0 and _aligned(8, *ptrs):
        return 2
    return 1


def plane_splits(batch, per, channels):
    """batch splits of the reduce / apply grids: min(32, batch, per / 2048), capped at ceil(2 * 8 * 132 / channels)"""
    want = -(-(2 * 8 * NUM_SMS) // channels)
    return max(1, min(SPLIT_SLOTS, batch, per // 2048, want))


def split_images(batch, splits):
    """images of the largest split: split s covers [batch * s / splits, batch * (s + 1) / splits)"""
    return max((batch * (s + 1)) // splits - (batch * s) // splits for s in range(splits))


def reduce_chain(path, batch, hw, splits):
    """longest fp32 accumulation a term passes through in the reduce pass before the fp64 hand-over.
    vec:    two accumulators per thread, each adds (t0 + t1) + (t2 + t3) once per 2 * 256 float4 of the split: 2 + steps.
    scalar: one accumulator per image and thread, ceil(hw / 256) steps.
    pool:   two accumulators per thread, each adds the two window winners of one lane item per 2 * 256 items: 2 * steps."""
    imgs = split_images(batch, splits)
    if path == "vec":
        return 2 + -(-imgs * hw // 4 // 512)
    if path == "scalar":
        return -(-hw // 256)
    return 2 * -(-imgs * (hw // 8) // 512)


def apply_chain(path, batch, hw, splits):
    """the same for the dx channel sum of the apply pass: vec adds a pair-summed float4 (2 + steps over 512 float4),
    scalar one dx per step (ceil(hw / 256)), pool one accumulator adding a pair-summed group of 8 per 256 items"""
    imgs = split_images(batch, splits)
    if path == "vec":
        return 2 + -(-imgs * hw // 4 // 512)
    if path == "scalar":
        return -(-hw // 256)
    return 3 + -(-imgs * (hw // 8) // 256)


# ============================================================================ buffers, layouts, decoders
def _lib():
    from micronet_b200 import _lib as L
    return L, L.load()


class Guarded:
    """``n`` elements of ``dtype`` at byte offset ``off`` of a sentinel-filled buffer with 256 guard bytes behind them:
    ``intact()`` says whether every byte outside the view still holds the sentinel"""

    def __init__(self, n, dtype, off=0, fill=0xFF):
        self.nbytes = n * torch.empty((), dtype=dtype).element_size()
        self.off, self.fill = off, fill
        self.buf = torch.full((off + self.nbytes + 256,), fill, dtype=torch.uint8, device=DEV)
        self.t = self.buf[off:off + self.nbytes].view(dtype)

    @property
    def ptr(self):
        return self.t.data_ptr()

    def intact(self):
        return bool((self.buf[:self.off] == self.fill).all()) and bool((self.buf[self.off + self.nbytes:] == self.fill).all())

    def untouched(self):
        return bool((self.buf == self.fill).all())


def _shuffle(x, sg):
    """channel order of a folded shuffle: out[:, a * sg + b] = in[:, b * (C / sg) + a] (harness.models.shuffle_channels)"""
    if sg == 1:
        return x
    b, c = x.shape[:2]
    return x.reshape(b, sg, c // sg, *x.shape[2:]).transpose(1, 2).reshape(x.shape)


def _unshuffle(x, sg):
    if sg == 1:
        return x
    b, c = x.shape[:2]
    return x.reshape(b, c // sg, sg, *x.shape[2:]).transpose(1, 2).reshape(x.shape)


def decode_bits(words, n):
    """flat NCHW pass words -> bool[n] (bit i of word w = element 32 w + i) and whether every bit past n is 0.
    The pooled kernels write the same layout byte-wise: the nibble of float4 i of x (its four elements) goes to byte i / 2,
    bits 4 (i % 2) .. 4 (i % 2) + 3, i.e. bit 4 i + e of the little-endian word stream for element 4 i + e."""
    w = words.reshape(-1).view(torch.int32)
    sh = torch.arange(32, dtype=torch.int32, device=w.device)
    bits = ((w.view(-1, 1) >> sh) & 1).to(torch.bool).reshape(-1)
    return bits[:n], not bool(bits[n:].any())


def decode_plane(plane, T, B, Cc, hw):
    """bf16 term planes [t][B][C/8][H][W][8] -> fp32 [t][B][C][H*W] (channel c8 * 8 + j)"""
    t = plane.reshape(-1).view(torch.bfloat16).view(T, B, Cc // 8, hw, 8)
    return t.permute(0, 1, 2, 4, 3).reshape(T, B, Cc, hw).float()


def first_max_of_signs(bn):
    """window index (r * 2 + s) ATen's max_pool2d picks among the +-1 signs of each 2x2 window: scan r0c0, r0c1, r1c0,
    r1c1 and replace on strictly greater, i.e. the first +1, else element 0; and the pooled value"""
    B, Cc, H, W = bn.shape
    pos = ~(bn < 0)
    w = pos.view(B, Cc, H // 2, 2, W // 2, 2)
    p = torch.stack([w[:, :, :, 0, :, 0], w[:, :, :, 0, :, 1], w[:, :, :, 1, :, 0], w[:, :, :, 1, :, 1]], -1)
    arg = p.to(torch.uint8).argmax(-1).to(torch.uint8)          # first maximum; 0 when no +1
    return arg, torch.where(p.any(-1), 1.0, -1.0)


def windows_of(mask):
    B, Cc, H, W = mask.shape
    return mask.view(B, Cc, H // 2, 2, W // 2, 2).any(5).any(3)


# ============================================================================ references
def emulate_bn(x, mean, invstd, gamma, beta):
    """fp32 emulation of the producers' bn = fmaf(fl(x - mu), fl(gamma * invstd), beta), exact for every element.
    The subtraction and the product are fp32 operations; the product p of two fp32 values is exact in fp64, and TwoSum
    gives the fp64 sum s = fl64(p + beta) together with its exact error e (s + e == p + beta).  Converting s to fp32 is the
    fma's single rounding except where s lies exactly on an fp32 rounding midpoint while e != 0: the fp64 rounding moved the
    exact value onto the tie, and the sign of e says which neighbour the fma rounds to.  Those double-rounding elements are
    resolved that way; their count is returned (a handful at most: the fp64 sum has 29 bits to spare)."""
    B, Cc = x.shape[:2]
    v = (1, Cc, 1, 1)
    k = (gamma * invstd).double().view(v)
    b = beta.double().view(v)
    bn = torch.empty_like(x)
    n_mid = 0
    for lo_i, hi_i in _chunks(B):
        p = (x[lo_i:hi_i] - mean.view(v)).double() * k
        s = p + b
        bb = s - p
        e = (p - (s - bb)) + (b - bb)
        del p, bb
        f = s.float()
        lo = f.double()
        other = torch.nextafter(f, torch.where(s > lo, math.inf, -math.inf).float())
        mid = (s != lo) & ((lo + other.double()) * 0.5 == s) & (e != 0)
        fix = torch.where(e > 0, torch.maximum(f, other), torch.minimum(f, other))
        bn[lo_i:hi_i] = torch.where(mid, fix, f)
        n_mid += int(mid.sum())
    return bn, n_mid


def dorefa_levels(y, a_bits):
    """the engine's standalone DoReFa quantizer (functional.act_quant_raw, bit-exact to the oracle) on y"""
    from micronet_b200 import _lib as L, functional as F_
    codes, _, _ = F_.act_quant_raw(y, F_.ActSpec(L.ACT_DOREFA, bits=a_bits), True, False, False)
    return codes.float()


def dorefa_mask(bn):
    """relu'(bn) * [0 <= fl(0.1f * relu(bn)) <= 1]  (relu'(0) = 0)"""
    return (bn > 0) & (bn * torch.tensor(0.1, dtype=torch.float32, device=bn.device) <= 1)


def semantic_check(x, mean, invstd, gamma, beta, kind, a_bits, got):
    """plain fp64 semantics: nn.functional.batch_norm with the given statistics (running_var = invstd^-2 - eps), then the
    oracle's binarizer / DoReFa quantizer.  The fp32 formula carries |bn32 - bn64| <= 4 u (|x - mu| |gamma invstd| + |beta|)
    (three roundings, the first two relative to terms of that size); a decision may differ only where bn64 lies within that
    distance of its boundary (0, +-1; DoReFa: 0, 10 and the level ties, the latter through the x 0.1 / s scaling plus 4 u
    of the quantizer's own arithmetic), and such elements may be at most 1e-4 of the total."""
    from oracle import reference_port as O
    Cc, v, eps = x.shape[1], (1, x.shape[1], 1, 1), 1e-5
    x64, m64, i64 = x.double(), mean.double(), invstd.double()
    bn64 = TF.batch_norm(x64, m64, i64 ** -2 - eps, gamma.double(), beta.double(), False, 0.0, eps)
    e = 4 * U * ((x64 - m64.view(v)).abs() * (gamma.double() * i64).abs().view(v) + beta.double().abs().view(v))
    del x64
    n = bn64.numel()
    checks = []
    if kind == "dorefa":
        s = 1.0 / (2 ** a_bits - 1)
        lev = O.dorefa_activation_levels(torch.relu(bn64), a_bits)
        pre = torch.clamp(0.1 * bn64, 0, 1) / s
        frac = (pre - torch.floor(pre) - 0.5).abs()
        near_lev = frac <= 0.1 * e / s + 4 * U * (pre + 1)
        checks.append(("level", got["level"] != lev, near_lev | (bn64.abs() <= e) | ((bn64 - 10).abs() <= e + 10 * U)))
        mask = (bn64 > 0) & (0.1 * bn64 <= 1)
        checks.append(("mask", got["mask"] != mask, (bn64.abs() <= e) | ((bn64 - 10).abs() <= e + 40 * U)))
    else:
        b = bn64.clone().requires_grad_(True)
        ysem = O.wb_binarize_activation(b)
        ysem.backward(torch.ones_like(ysem))
        passm = b.grad != 0
        near0 = bn64.abs() <= e
        if "pooled" in got:      # the oracle's binarizer, then max_pool2d
            checks.append(("pooled y", got["pooled"] != TF.max_pool2d(ysem.detach(), 2, 2), windows_of(near0)))
        else:
            checks.append(("sign", got["sign"] != ysem.detach(), near0))
        checks.append(("pass", got["pass_"] != passm, (bn64.abs() - 1).abs() <= e))
        del b, ysem
    for name, differ, near in checks:
        far = differ & ~near
        assert not far.any(), f"{name}: {int(far.sum())} decisions differ from fp64 away from a boundary"
        assert int(differ.sum()) <= max(1, int(1e-4 * n)), f"{name}: {int(differ.sum())} of {n} differ from fp64"


def _chunks(B):
    step = max(1, -(-B // 8))
    return [(lo, min(B, lo + step)) for lo in range(0, B, step)]


def _xhat64(x, mean, invstd):
    v = (1, x.shape[1], 1, 1)
    return (x.double() - mean.double().view(v)) * invstd.double().view(v)


def bwd_reference(gm, x, mean, invstd, gamma):
    """fp64 sums of nn.BatchNorm2d's backward of the masked gradient gm (fp32, exact g * mask, own channel order) with the
    given fp32 statistics, xhat = (x - mean) invstd: per image and channel sum gm and sum gm xhat (DB, DG are their sums over
    the batch), and the magnitudes the kernel's roundings are relative to, A1 = sum |gm|, A2 = sum |gm xhat|.  Computed
    eight images at a time to keep the fp64 temporaries small."""
    B, Cc = x.shape[:2]
    db_img, dg_img = torch.zeros(B, Cc, dtype=torch.float64, device=DEV), torch.zeros(B, Cc, dtype=torch.float64, device=DEV)
    A1, A2 = torch.zeros(Cc, dtype=torch.float64, device=DEV), torch.zeros(Cc, dtype=torch.float64, device=DEV)
    for lo, hi in _chunks(B):
        g = gm[lo:hi].double()
        gx = g * _xhat64(x[lo:hi], mean, invstd)
        db_img[lo:hi], dg_img[lo:hi] = g.sum((2, 3)), gx.sum((2, 3))
        A1 += g.abs().sum((0, 2, 3))
        A2 += gx.abs().sum((0, 2, 3))
    return dict(db_img=db_img, dg_img=dg_img, DB=db_img.sum(0), DG=dg_img.sum(0), A1=A1, A2=A2,
                k=gamma.double() * invstd.double())


def check_reductions(ref, dgamma, dbeta, chain, N, batch, splits):
    """dbeta = sum gm: each term passes <= chain fp32 additions before the fp64 hand-over, the fp64 partials add N
    roundings of 2^-53 at most and the result is rounded to fp32 once:  |dbeta - DB| <= (chain + 1) u A1 + N 2^-53 A1 + u |DB|.
    dgamma = sum gm fl(fl(x - mu) invstd): three more roundings per term (the subtraction, the product with invstd, the
    product with gm):  |dgamma - DG| <= (chain + 4) u A2 + N 2^-53 A2 + u |DG|.
    With several splits, the bound must be sharp enough to see the last split dropped (or counted twice: the same change)
    in every channel: that split's fp64 share of DB or of DG must exceed its bound."""
    b_db = (chain + 1) * U * ref["A1"] + N * U64 * ref["A1"] + U * ref["DB"].abs()
    b_dg = (chain + 4) * U * ref["A2"] + N * U64 * ref["A2"] + U * ref["DG"].abs()
    e_db = (dbeta.double() - ref["DB"]).abs()
    e_dg = (dgamma.double() - ref["DG"]).abs()
    assert (e_db <= b_db).all(), f"dbeta: worst {(e_db / b_db).max().item():.3f} x the bound"
    assert (e_dg <= b_dg).all(), f"dgamma: worst {(e_dg / b_dg).max().item():.3f} x the bound"
    if splits > 1:
        lo = (batch * (splits - 1)) // splits
        db_last, dg_last = ref["db_img"][lo:].sum(0).abs(), ref["dg_img"][lo:].sum(0).abs()
        assert ((db_last > b_db) | (dg_last > b_dg)).all(), "bound too loose to see a dropped split"
    return b_db, b_dg


def check_dx(dx, gm, x, mean, invstd, ref, b_db, b_dg, N, what):
    """dx = fl(k fl(fl(gm - db) - fl(xhat dg))), k = fl(gamma invstd), db = fl(dbeta fl(1 / N)), dg likewise,
    xhat = fl(fl(x - mu) invstd), against dx64 = k (gm - DB / N - xhat DG / N) in fp64.  The longest path (xhat dg) passes
    8 roundings (xhat 2, 1 / N, dg, the product, the subtraction, k, the final product), each relative to a term no larger
    than the three terms' absolute sum (a contracted fma only removes roundings), so
        |dx - dx64| <= 10 u |k| (|gm| + |DB| / N + |xhat DG| / N) + |k| (bound(dbeta) + |xhat| bound(dgamma)) / N,
    where the second part carries the errors of the kernel's own dbeta / dgamma (check_reductions)."""
    v = (1, dx.shape[1], 1, 1)
    k, DBn, DGn = ref["k"].view(v), (ref["DB"] / N).view(v), (ref["DG"] / N).view(v)
    b1, b2 = (b_db / N).view(v), (b_dg / N).view(v)
    worst = 0.0
    for lo, hi in _chunks(dx.shape[0]):
        xh, g = _xhat64(x[lo:hi], mean, invstd), gm[lo:hi].double()
        err = (dx[lo:hi].double() - k * (g - DBn - xh * DGn)).abs()
        bound = 10 * U * k.abs() * (g.abs() + DBn.abs() + (xh * DGn).abs()) + k.abs() * (b1 + xh.abs() * b2) + 1e-300
        worst = max(worst, (err / bound).max().item())
    assert worst <= 1.0, f"{what}: worst {worst:.3f} x the bound"


def check_dx_sum(dx_sum, dx, chain, what):
    """channel sums of the dx the kernel wrote: each dx passes <= chain fp32 additions, then fp64 and one final rounding:
    |s - S| <= chain u sum |dx| + N 2^-53 sum |dx| + u |S|"""
    d = dx.double()
    S, A = d.sum((0, 2, 3)), d.abs().sum((0, 2, 3))
    N = dx.numel() // dx.shape[1]
    bound = chain * U * A + N * U64 * A + U * S.abs() + 1e-300
    err = (dx_sum.double() - S).abs()
    assert (err <= bound).all(), f"{what}: worst {(err / bound).max().item():.3f} x the bound"


def check_pieces(plane, T, B, Cc, hw, v, what):
    """decoded pieces of one call against the fp32 value v = fl(dx * ch_scale) (v = dx without ch_scale):
    T = 3: p0 + p1 + p2 == v exactly (the 3-piece split of an fp32 value is exact; the sum is taken in fp64, where it is
    exact too); T = 1, 2: piece t == the round-to-nearest bf16 of the fp32 residual v - p0 - ... - p(t-1)."""
    p = decode_plane(plane, T, B, Cc, hw)
    v = v.reshape(B, Cc, hw)
    if T == 3:
        s = p[0].double() + p[1].double() + p[2].double()
        assert torch.equal(s, v.double()), f"{what}: {_first_diff(s, v.double())}"
        return
    r = v
    for t in range(T):
        want = r.to(torch.bfloat16).float()
        assert _eq(p[t], want), f"{what}: piece {t}: {_first_diff(p[t], want)}"
        r = r - want


# ============================================================================ cases
# The producer planes of the three bench workloads that use them, derived from the models (test_bn_producers_cpu.py
# checks this list against harness.models + the prepare passes): (C, H, W, out_shuffle_groups, pool2, a_bits)
BENCH_PLANES = {
    "nin_gc_wbwtab_w3a2": [(256, 32, 32, 1, False, None), (256, 32, 32, 2, False, None), (256, 32, 32, 2, True, None),
                           (512, 16, 16, 16, False, None), (512, 16, 16, 4, False, None), (512, 16, 16, 4, True, None),
                           (1024, 8, 8, 32, False, None), (1024, 8, 8, 1, False, None)],
    "nin_dorefa_w8a8": [(192, 32, 32, 1, False, 8), (160, 32, 32, 1, False, 8), (192, 16, 16, 1, False, 8),
                        (192, 16, 16, 1, False, 8), (192, 8, 8, 1, False, 8), (192, 8, 8, 1, False, 8)],
    "nin_gc_dorefa_w4a4": [(256, 32, 32, 1, False, 4), (256, 32, 32, 2, False, 4), (512, 16, 16, 16, False, 4),
                           (512, 16, 16, 4, False, 4), (1024, 8, 8, 32, False, 4), (1024, 8, 8, 1, False, 4)],
}


def bench_planes(workload):
    """(C, H, W, out_shuffle_groups, pool2, a_bits) of every fused producer the workload's prepare pass creates, in module
    order, with H, W taken from a CPU forward of the un-prepared model"""
    import copy
    import micronet_b200 as E
    from harness import models as zoo
    from micronet_b200.fused import BatchNormBinarize2d, BatchNormReluQuant2d
    base = zoo.NIN() if workload == "nin_dorefa_w8a8" else zoo.NINGC()
    shapes = {}
    hooks = [m.register_forward_hook(lambda m, i, o, n=n: shapes.__setitem__(n, tuple(i[0].shape[2:])))
             for n, m in base.named_modules() if isinstance(m, nn.BatchNorm2d)]
    with torch.no_grad():
        base(torch.zeros(1, 3, 32, 32))
    for h in hooks:
        h.remove()
    m = copy.deepcopy(base)
    if workload == "nin_gc_wbwtab_w3a2":
        E.wbwtab.prepare(m, inplace=True, A=2, W=3, fuse_bn=True)
    else:
        bits = 8 if workload == "nin_dorefa_w8a8" else 4
        E.dorefa.prepare(m, inplace=True, a_bits=bits, w_bits=bits, fuse=True)
    out = []
    for n, mod in m.named_modules():
        if isinstance(mod, BatchNormBinarize2d):
            out.append((mod.num_features, *shapes[n], int(mod.out_shuffle_groups), bool(mod.pool2), None))
        elif isinstance(mod, BatchNormReluQuant2d):
            out.append((mod.num_features, *shapes[n], int(mod.out_shuffle_groups), False, int(mod.a_bits)))
    return out


def _plane(workload, C_, H, sg, pool=False):
    p = [q for q in BENCH_PLANES[workload] if q[0] == C_ and q[1] == H and q[3] == sg and q[4] == pool]
    assert p, (workload, C_, H, sg, pool)
    return p[0]


# (B, C, H, W, sg, kind, a_bits, byte offset of x / g / dx, expected (forward path, backward path, pack VEC, splits))
# kind "sign": mnb_bn_sign_fwd (+ _fwd_packed where C % 8 == 0 and hw % 32 == 0), mnb_bn_sign_bwd (+ mnb_bn_sign_bwd_pack);
# "pool": the pooled pair; "dorefa": mnb_bn_relu_quant_pack_fwd + mnb_bn_sign_bwd.  Splits per plane_splits.
def _case(B, plane, off, expect, id):
    Cc, H, W, sg, pool, a_bits = plane
    kind = "dorefa" if a_bits else ("pool" if pool else "sign")
    return pytest.param(B, Cc, H, W, sg, kind, a_bits, off, expect, id=id)


HL, NIN, GC = "nin_gc_wbwtab_w3a2", "nin_dorefa_w8a8", "nin_gc_dorefa_w4a4"
CASES = [
    # headline, batch 256
    _case(256, _plane(HL, 256, 32, 2), 0, ("v4", "vec", 4, 9), "hl-256x256@32-sg2-v4-vec-pack4-9splits"),
    _case(256, _plane(HL, 256, 32, 2, True), 0, ("pool", "pool", None, 9), "hl-256x256@32-pool-sg2-9splits"),
    _case(256, _plane(HL, 512, 16, 16), 0, ("v4", "vec", 4, 5), "hl-256x512@16-sg16-v4-vec-pack4-5splits"),
    _case(256, _plane(HL, 512, 16, 4, True), 0, ("pool", "pool", None, 5), "hl-256x512@16-pool-sg4-5splits"),
    _case(256, _plane(HL, 1024, 8, 32), 0, ("v4", "vec", 2, 3), "hl-256x1024@8-sg32-hw64-pack2-3splits"),
    _case(32, _plane(HL, 1024, 8, 1), 0, ("v4", "vec", 2, 1), "hl-32x1024@8-sg1-pack2-1split"),
    # DoReFa: NIN at a_bits 8, NIN-GC at a_bits 4; one plane of each at batch 256
    _case(256, _plane(NIN, 192, 32, 1), 0, ("dorefa", "vec", None, 11), "nin-256x192@32-a8-11splits"),
    _case(32, _plane(NIN, 160, 32, 1), 0, ("dorefa", "vec", None, 14), "nin-32x160@32-a8-14splits"),
    _case(32, _plane(NIN, 192, 16, 1), 0, ("dorefa", "vec", None, 4), "nin-32x192@16-a8-4splits"),
    _case(64, _plane(NIN, 192, 8, 1), 0, ("dorefa", "vec", None, 2), "nin-64x192@8-a8-2splits"),
    _case(32, _plane(GC, 256, 32, 2), 0, ("dorefa", "vec", None, 9), "gc-32x256@32-sg2-a4-9splits"),
    _case(32, _plane(GC, 512, 16, 16), 0, ("dorefa", "vec", None, 4), "gc-32x512@16-sg16-a4-4splits"),
    _case(256, _plane(GC, 1024, 8, 32), 0, ("dorefa", "vec", None, 3), "gc-256x1024@8-sg32-a4-3splits"),
    # path edges at small batch
    _case(8, (64, 4, 8, 4, False, None), 0, ("v4", "vec", 1, 1), "hw32-v4-vec-pack1-1split"),
    _case(37, (8, 4, 8, 1, False, 2), 0, ("dorefa", "vec", None, 1), "c8-hw32-a2-batch37-1split"),
    _case(5, (24, 7, 6, 3, False, None), 0, ("scalar", "scalar", None, 1), "hw42-scalar-1split"),
    _case(37, (8, 45, 43, 2, False, None), 0, ("scalar", "scalar", None, 32), "c8-hw1935-scalar-batch37-32splits"),
    _case(16, (64, 16, 16, 4, False, None), 4, ("scalar", "scalar", 1, 2), "offset4-scalar-pack1-2splits"),
    _case(16, (64, 16, 16, 4, False, None), 8, ("scalar", "scalar", 2, 2), "offset8-scalar-pack2-2splits"),
    _case(37, (8, 32, 32, 1, False, None), 0, ("v4", "vec", 4, 18), "c8-batch37-vec-pack4-18splits"),
    _case(37, (8, 8, 16, 1, True, None), 0, ("pool", "pool", None, 2), "c8-batch37-pool-2splits"),
    _case(2, (8184, 4, 8, 4, False, None), 0, ("v4", "vec", 1, 1), "c8184-hw32-pack1-1split"),
    _case(2, (8184, 4, 8, 1, True, None), 0, ("pool", "pool", None, 1), "c8184-pool-1split"),
]


def _make_inputs(B, Cc, H, W, kind, off, seed):
    """x ~ N(mu_c, sd_c) in a guarded (possibly offset) buffer; mean / invstd the fp32 batch statistics of x; gamma, beta
    spread so that bn crosses every decision boundary often: binarizer |gamma| in [0.5, 1.5] (every 8th negative),
    beta ~ 0.3 N(0, 1); DoReFa gamma in [1, 5], beta ~ 2 + 2 N(0, 1), so 0.1 bn spans the quantizer's [0, 1] and beyond"""
    g = _gen(seed)
    n = B * Cc * H * W
    xb = Guarded(n, torch.float32, off)
    sd = torch.rand(Cc, generator=g, device=DEV) + 0.5
    mu = (torch.rand(Cc, generator=g, device=DEV) - 0.5) * 4
    x = xb.t.view(B, Cc, H, W)
    x.copy_(torch.randn(B, Cc, H, W, generator=g, device=DEV) * sd.view(1, -1, 1, 1) + mu.view(1, -1, 1, 1))
    mean = x.mean((0, 2, 3))
    invstd = torch.rsqrt(x.var((0, 2, 3), unbiased=False) + 1e-5)
    if kind == "dorefa":
        gamma = torch.rand(Cc, generator=g, device=DEV) * 4 + 1
        beta = torch.randn(Cc, generator=g, device=DEV) * 2 + 2
    else:
        gamma = (torch.rand(Cc, generator=g, device=DEV) + 0.5) * torch.where(torch.arange(Cc, device=DEV) % 8 == 5, -1.0, 1.0)
        beta = torch.randn(Cc, generator=g, device=DEV) * 0.3
    return xb, x, mean, invstd, gamma, beta


def run_forward(kind, x, mean, invstd, gamma, beta, sg, a_bits, off):
    """one call of the case's forward kernel into sentinel-filled guarded outputs; returns the decoded outputs"""
    L, lib = _lib()
    B, Cc, H, W = x.shape
    hw, n = H * W, x.numel()
    words = Guarded(-(-n // 32), torch.int32, 0, fill=0xA5)
    args = (mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), beta.data_ptr())
    out = {"words": words}
    if kind == "pool":
        y = Guarded(n // 4, torch.float32)
        arg = Guarded(n // 4, torch.uint8)
        L.check(lib.mnb_bn_sign_pool_fwd(x.data_ptr(), B, Cc, H, W, *args, sg, y.ptr, words.ptr, arg.ptr, L.stream()),
                "bn_sign_pool_fwd")
        out.update(y=y, arg=arg)
    elif kind == "dorefa":
        from micronet_b200 import functional as F_
        qp = F_.ActSpec(L.ACT_DOREFA, bits=a_bits).struct()
        plane = Guarded(n, torch.bfloat16)
        L.check(lib.mnb_bn_relu_quant_pack_fwd(x.data_ptr(), B, Cc, hw, *args, C.byref(qp), sg, plane.ptr, words.ptr,
                                               L.stream()), "bn_relu_quant_pack_fwd")
        out.update(plane=plane)
    else:
        y = Guarded(n, torch.float32, off)
        L.check(lib.mnb_bn_sign_fwd(x.data_ptr(), B, Cc, hw, *args, sg, y.ptr, words.ptr, L.stream()), "bn_sign_fwd")
        out.update(y=y, path=fwd_path(n, hw, x.data_ptr(), y.ptr))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,Cc,H,W,sg,kind,a_bits,off,expect", CASES)
def test_forward_exact_against_fp32_emulation(B, Cc, H, W, sg, kind, a_bits, off, expect):
    """every decision of the forward kernels bit for bit against emulate_bn; every output word written (sentinel-filled
    outputs), nothing outside them touched; the packed forward's bf16 plane equals its own y in the shuffled order and y /
    pass words equal mnb_bn_sign_fwd's, with y and with y = NULL.  Then the semantic check against fp64 BatchNorm."""
    L, lib = _lib()
    hw, n = H * W, B * Cc * H * W
    xb, x, mean, invstd, gamma, beta = _make_inputs(B, Cc, H, W, kind, off, seed=B + Cc + H + sg)
    out = run_forward(kind, x, mean, invstd, gamma, beta, sg, a_bits, off)
    bn, n_mid = emulate_bn(x, mean, invstd, gamma, beta)
    assert n_mid <= 4, f"{n_mid} double-rounding midpoints: the emulation's premise does not hold"
    words, ok = decode_bits(out["words"].t, n)
    assert ok and out["words"].intact(), "pass words: bits past the end set or guard overwritten"
    words = words.view(B, Cc, H, W)
    got = {}
    if kind == "pool":
        assert expect[0] == "pool"
        arg_w, y_w = first_max_of_signs(bn)
        arg = out["arg"].t.view(B, Cc, H // 2, W // 2)
        y = _unshuffle(out["y"].t.view(B, Cc, H // 2, W // 2), sg)
        assert out["arg"].intact() and out["y"].intact()
        assert torch.equal(arg, arg_w), f"arg-max: {_first_diff(arg, arg_w)}"
        assert torch.equal(y, y_w), f"pooled y: {_first_diff(y, y_w)}"
        assert torch.equal(words, bn.abs() < 1), f"pass: {_first_diff(words, bn.abs() < 1)}"
        got.update(pooled=y, pass_=words)
    elif kind == "dorefa":
        lev = _unshuffle(decode_plane(out["plane"].t, 1, B, Cc, hw)[0].view(B, Cc, H, W), sg)
        assert out["plane"].intact()
        want_lev = dorefa_levels(torch.relu(bn), a_bits)
        want_mask = dorefa_mask(bn)
        assert torch.equal(lev, want_lev), f"levels: {_first_diff(lev, want_lev)}"
        assert torch.equal(words, want_mask), f"mask: {_first_diff(words, want_mask)}"
        got.update(level=lev, mask=words)
    else:
        assert out["path"] == expect[0], out["path"]
        y = out["y"].t.view(B, Cc, H, W)
        assert out["y"].intact()
        want_y = _shuffle(torch.where(bn < 0, -1.0, 1.0), sg)
        assert torch.equal(y, want_y), f"y: {_first_diff(y, want_y)}"
        assert torch.equal(words, bn.abs() < 1), f"pass: {_first_diff(words, bn.abs() < 1)}"
        got.update(sign=_unshuffle(y, sg), pass_=words)
        # the packed forward: plane == y (shuffled order), its y and pass words == these, also with y = NULL
        for with_y in (True, False):
            y2 = Guarded(n, torch.float32, off) if with_y else None
            w2 = Guarded(-(-n // 32), torch.int32, 0, fill=0xA5)
            plane = Guarded(n, torch.bfloat16)
            rc = lib.mnb_bn_sign_fwd_packed(x.data_ptr(), B, Cc, hw, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                            beta.data_ptr(), sg, y2.ptr if with_y else None, w2.ptr, plane.ptr, L.stream())
            if Cc % 8 or hw % 32:
                assert expect[2] is None and rc == E_UNSUPPORTED, rc
                assert plane.untouched() and w2.untouched(), "a refused call wrote something"
                continue
            L.check(rc, "bn_sign_fwd_packed")
            torch.cuda.synchronize()
            assert pack_vec(hw, x.data_ptr(), y2.ptr if with_y else None) == expect[2]
            pl = decode_plane(plane.t, 1, B, Cc, hw)[0].view(B, Cc, H, W)
            assert plane.intact() and torch.equal(pl, y), f"plane != y: {_first_diff(pl, y)}"
            assert w2.intact() and torch.equal(w2.t, out["words"].t), "pass words of the packed forward"
            if with_y:
                assert y2.intact() and torch.equal(y2.t, out["y"].t), "y of the packed forward"
    del out
    semantic_check(x, mean, invstd, gamma, beta, kind, a_bits, got)
    del bn, got, xb
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B,Cc,H,W,sg,kind,a_bits,off,expect", CASES)
def test_backward_against_fp64(B, Cc, H, W, sg, kind, a_bits, off, expect):
    """mnb_bn_sign_bwd / mnb_bn_sign_pool_bwd behind the case's forward (its pass bits and arg-max, checked exactly by
    test_forward_exact_against_fp32_emulation, give the mask):
    * training = 1: dbeta / dgamma (check_reductions, including the dropped-split test), dx (check_dx), dx_channel_sum
      (check_dx_sum);
    * training = 2 (reduce only): the same dbeta / dgamma bit for bit, dx untouched;
    * training = 0: dx = fl(fl(gamma invstd) g m) exactly (one product, no statistics terms);
    * the _pack apply passes from training 1's dgamma / dbeta: their fp32 dx (check_dx) and the decoded pieces exactly
      (check_pieces), T = 3 with ch_scale, T = 2 with ch_scale = NULL and dx = NULL, T = 1 with ch_scale; the pooled
      pieces against the non-pack pooled dx of the same reduce pass times ch_scale.
    g has a non-zero mean (the conv's gradient is not centred) so every split carries a large share of dbeta."""
    L, lib = _lib()
    hw, n, N = H * W, B * Cc * H * W, B * H * W
    seed = B + Cc + H + sg
    xb, x, mean, invstd, gamma, beta = _make_inputs(B, Cc, H, W, kind, off, seed=seed)
    fwd = run_forward(kind, x, mean, invstd, gamma, beta, sg, a_bits, off)
    m = decode_bits(fwd["words"].t, n)[0].view(B, Cc, H, W)
    words = fwd["words"].ptr
    gen = _gen(seed + 1)
    pool = kind == "pool"
    if pool:
        OH, OW = H // 2, W // 2
        g_own = 1 + 0.25 * torch.randn(B, Cc, OH, OW, generator=gen, device=DEV)
        gb = Guarded(n // 4, torch.float32)
        arg = fwd["arg"].t.view(B, Cc, OH, OW)
        win = torch.zeros(B, Cc, OH, OW, 4, device=DEV)
        win.scatter_(-1, arg.long().unsqueeze(-1), g_own.unsqueeze(-1))      # the pooled gradient goes to the winner
        gfull = win.view(B, Cc, OH, OW, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, Cc, H, W)
        del win
    else:
        xh = ((x - mean.view(1, -1, 1, 1)) * invstd.view(1, -1, 1, 1))
        g_own = 1 + 4 * xh + 0.25 * torch.randn(B, Cc, H, W, generator=gen, device=DEV)
        del xh
        gb = Guarded(n, torch.float32, off)
        gfull = g_own
    gb.t.copy_(_shuffle(g_own, sg).reshape(-1))
    gm = torch.where(m, gfull, torch.zeros((), device=DEV))
    del gfull, m
    splits = plane_splits(B, N, Cc)
    assert splits == expect[3], splits
    stats = (mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr())
    scratch = L.scratch(x.device, Cc).data_ptr()
    sums = {}

    def call(training, dx):
        out = torch.full((3 * Cc,), float("nan"), device=DEV)
        if pool:
            rc = lib.mnb_bn_sign_pool_bwd(gb.ptr, words, fwd["arg"].ptr, x.data_ptr(), B, Cc, H, W, *stats, training, sg,
                                          dx.ptr, out[:Cc].data_ptr(), out[Cc:2 * Cc].data_ptr(), out[2 * Cc:].data_ptr(),
                                          scratch, L.stream())
        else:
            rc = lib.mnb_bn_sign_bwd(gb.ptr, words, x.data_ptr(), B, Cc, hw, *stats, training, sg, dx.ptr,
                                     out[:Cc].data_ptr(), out[Cc:2 * Cc].data_ptr(), out[2 * Cc:].data_ptr(), scratch,
                                     L.stream())
        L.check(rc, f"bwd training={training}")
        torch.cuda.synchronize()
        return out[:Cc], out[Cc:2 * Cc], out[2 * Cc:]

    # training = 1
    dx1 = Guarded(n, torch.float32, off)
    path = "pool" if pool else bwd_path(n, hw, x.data_ptr(), gb.ptr, dx1.ptr)
    assert path == expect[1], path
    dg, db, ds = call(1, dx1)
    assert dx1.intact()
    dx = dx1.t.view(B, Cc, H, W)
    ref = bwd_reference(gm, x, mean, invstd, gamma)
    b_db, b_dg = check_reductions(ref, dg, db, reduce_chain(path, B, hw, splits), N, B, splits)
    check_dx(dx, gm, x, mean, invstd, ref, b_db, b_dg, N, "dx (training)")
    check_dx_sum(ds, dx, apply_chain(path, B, hw, splits), "dx_channel_sum (training)")
    # training = 2: the reduce pass alone
    dx2 = Guarded(n, torch.float32, off)
    dg2, db2, ds2 = call(2, dx2)
    assert dx2.untouched(), "training = 2 wrote dx"
    assert _eq(dg2, dg) and _eq(db2, db), "the reduce-only pass differs from the reduce pass of training = 1"
    assert torch.isnan(ds2).all(), "training = 2 wrote dx_channel_sum"
    del dx2
    # training = 0: fixed statistics, dx = k * g * m
    dx0 = Guarded(n, torch.float32, off)
    dg0, db0, ds0 = call(0, dx0)
    assert dx0.intact()
    k32 = (gamma * invstd).view(1, -1, 1, 1)
    want0 = k32 * gm
    assert _eq(dx0.t, want0), f"dx (eval): {_first_diff(dx0.t, want0)}"
    assert _eq(dg0, dg) and _eq(db0, db)
    check_dx_sum(ds0, dx0.t.view(B, Cc, H, W), apply_chain(path, B, hw, splits), "dx_channel_sum (eval)")
    del dx0, want0
    # the packed apply passes
    sc = torch.rand(Cc, generator=gen, device=DEV) * 0.02 + 0.001       # a conv's per-channel weight scale
    if kind == "dorefa":
        return
    for T, scale, with_dx in ((3, sc, True), (2, None, False), (1, sc, False)):
        plane = Guarded(T * n, torch.bfloat16)
        if pool:
            rc = lib.mnb_bn_sign_pool_bwd_pack(gb.ptr, words, fwd["arg"].ptr, x.data_ptr(), B, Cc, H, W, *stats,
                                               dg.data_ptr(), db.data_ptr(), sg, L.ptr(scale), T, plane.ptr, L.stream())
            L.check(rc, "bn_sign_pool_bwd_pack")
            dref = dx                       # the non-pack pooled dx of the same reduce pass
        else:
            dxp = Guarded(n, torch.float32, off) if with_dx else None
            rc = lib.mnb_bn_sign_bwd_pack(gb.ptr, words, x.data_ptr(), B, Cc, hw, *stats, dg.data_ptr(), db.data_ptr(), sg,
                                          L.ptr(scale), T, dxp.ptr if with_dx else None, plane.ptr, L.stream())
            if expect[2] is None:
                assert rc == E_UNSUPPORTED and plane.untouched(), rc
                break
            L.check(rc, "bn_sign_bwd_pack")
            assert pack_vec(hw, gb.ptr, x.data_ptr(), dxp.ptr if with_dx else None) == expect[2]
            if with_dx:
                torch.cuda.synchronize()
                assert dxp.intact()
                dpk = dxp.t.view(B, Cc, H, W)
                check_dx(dpk, gm, x, mean, invstd, ref, b_db, b_dg, N, "dx (pack)")
                # both apply passes round dx the same way (bn_bwd_centre): the pieces are those of the non-pack dx
                assert _eq(dpk, dx), f"dx of the pack pass vs mnb_bn_sign_bwd: {_first_diff(dpk, dx)}"
            dref = dpk                      # the T = 3 call's dx: the same fp32 values every call computes
        torch.cuda.synchronize()
        assert plane.intact()
        v = dref * scale.view(1, -1, 1, 1) if scale is not None else dref
        check_pieces(plane.t, T, B, Cc, hw, v, f"T={T} ch_scale={'yes' if scale is not None else 'NULL'}")
        del plane, v
    del xb, gb, gm, dx1, ref
    torch.cuda.empty_cache()


# ============================================================================ pinned decision edges
def _steps(v, k):
    """v and its k fp32 neighbours on each side"""
    out, lo, hi = [np.float32(v)], np.float32(v), np.float32(v)
    for _ in range(k):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return out


def dorefa_edge_values(a_bits):
    """(b10, its successor, [(bn, level)] at rounding ties): b10 = the largest fp32 bn with fl(0.1f bn) <= 1 (mask 1, the
    successor's is 0); a tie bn has fl(fl(0.1f bn) / s) == level - 1/2 exactly, s = fl(1 / (2^a - 1)), so the quantizer's
    floor(. + 0.5) must give ``level``"""
    tenth, one = np.float32(0.1), np.float32(1)
    b = np.float32(10)
    while np.float32(b * tenth) > one:
        b = np.nextafter(b, np.float32(0))
    while np.float32(np.nextafter(b, np.float32(np.inf)) * tenth) <= one:
        b = np.nextafter(b, np.float32(np.inf))
    s = np.float32(1.0 / (2 ** a_bits - 1))
    ties = []
    for lev in range(min(2 ** a_bits - 1, 48)):
        for c in _steps((lev + 0.5) * float(s), 8):
            if np.float32(c / s) != np.float32(lev + 0.5):
                continue
            hit = [x for x in _steps(float(c) / 0.1, 16) if np.float32(x * tenth) == c]
            if hit:
                ties.append((hit[0], lev + 1))
                break
    return b, np.nextafter(b, np.float32(np.inf)), ties


def _edge_plane(kind, a_bits, B=2, Cc=16, H=8, W=16):
    """bn values placed by construction: gamma = 2^(c % 5 - 2), invstd = 1, mean = 0, beta = +0 (even c) / -0 (odd c), so
    fma(x - 0, gamma, beta) = x gamma exactly and x = bn / gamma reproduces any chosen bn (bn = -0 needs x = -0 in an odd
    channel).  Every 2x2 window takes one of the 16 sign patterns, its magnitudes cycle through the edge values."""
    if kind == "dorefa":
        b10, above, ties = dorefa_edge_values(a_bits)
        mags = [0.0, b10, above, 20.0, 5.0] + [t for t, _ in ties]
    else:
        n1 = float(np.nextafter(np.float32(1), np.float32(0)))
        mags = [0.0, 1.0, n1, float(np.nextafter(np.float32(1), np.float32(2))), 0.5, 2.0 ** -30, 1.5]
    mags = torch.tensor(np.array(mags, dtype=np.float32), device=DEV)
    nw = B * Cc * (H // 2) * (W // 2)
    pat = torch.arange(nw, device=DEV) % 16
    e = torch.arange(4, device=DEV)
    neg = ((pat.view(-1, 1) >> e) & 1).bool()
    if kind == "dorefa":
        neg = neg & (torch.arange(nw, device=DEV).view(-1, 1) % 3 == 0)     # keep most of them positive
    mag = mags[torch.arange(nw * 4, device=DEV) % len(mags)].view(nw, 4)
    val = torch.where(neg, -mag, mag)                                     # -0.0 where a zero magnitude meets a minus
    bn = val.view(B, Cc, H // 2, W // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, Cc, H, W)
    c = torch.arange(Cc, device=DEV)
    gamma = torch.pow(2.0, (c % 5 - 2).float())
    beta = torch.where(c % 2 == 1, -0.0, 0.0)
    x = bn / gamma.view(1, -1, 1, 1)
    # a -0 bn needs an odd channel (beta = -0): in even channels it comes out +0, which the checks below see as such
    mean, invstd = torch.zeros(Cc, device=DEV), torch.ones(Cc, device=DEV)
    return x, mean, invstd, gamma, beta


@pytest.mark.parametrize("variant,a_bits", [("sign-v4", None), ("sign-scalar", None), ("packed", None), ("pool", None),
                                            ("dorefa", 2), ("dorefa", 4), ("dorefa", 8)])
def test_forward_decisions_at_pinned_edges(variant, a_bits):
    """bn = +0 and -0 give +1; |bn| = 1 gives pass 0 and nextafter(1, 0) pass 1; DoReFa: bn = +-0 gives level 0 and mask
    0, the largest bn with fl(0.1f bn) == 1 mask 1 and level 2^a - 1, the next float above it mask 0, rounding ties round
    up; pooled windows all -1 (arg 0, -1), all +1 (arg 0, +1) and mixed (the first +1).  Each asserted directly, and every
    element against the emulation (exact here: no rounding anywhere)."""
    L, lib = _lib()
    kind = "dorefa" if variant == "dorefa" else ("pool" if variant == "pool" else "sign")
    off = 4 if variant == "sign-scalar" else 0
    x0, mean, invstd, gamma, beta = _edge_plane(kind, a_bits)
    B, Cc, H, W = x0.shape
    n, hw = x0.numel(), H * W
    xb = Guarded(n, torch.float32, off)
    x = xb.t.view(B, Cc, H, W)
    x.copy_(x0)
    bn, n_mid = emulate_bn(x, mean, invstd, gamma, beta)
    assert n_mid == 0
    zero = bn == 0
    assert (zero & torch.signbit(bn)).any() and (zero & ~torch.signbit(bn)).any(), "construction: both signed zeros"
    if variant == "packed":
        y, words, plane = Guarded(n, torch.float32), Guarded(n // 32, torch.int32, fill=0xA5), Guarded(n, torch.bfloat16)
        L.check(lib.mnb_bn_sign_fwd_packed(x.data_ptr(), B, Cc, hw, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                           beta.data_ptr(), 1, y.ptr, words.ptr, plane.ptr, L.stream()), "fwd_packed")
        torch.cuda.synchronize()
        assert pack_vec(hw, x.data_ptr(), y.ptr) == 4
        assert torch.equal(decode_plane(plane.t, 1, B, Cc, hw)[0].view(B, Cc, H, W), y.t.view(B, Cc, H, W))
        out = dict(y=y, words=words)
    else:
        out = run_forward(kind, x, mean, invstd, gamma, beta, 1, a_bits, off)
        if kind == "sign":
            assert out["path"] == ("scalar" if off else "v4")
    p, ok = decode_bits(out["words"].t, n)
    p = p.view(B, Cc, H, W)
    assert ok and out["words"].intact()
    if kind == "dorefa":
        b10, above, ties = dorefa_edge_values(a_bits)
        lev = decode_plane(out["plane"].t, 1, B, Cc, hw)[0].view(B, Cc, H, W)
        top = 2 ** a_bits - 1
        assert (lev[zero] == 0).all() and not p[zero].any(), "bn = 0: level 0, mask 0"
        at10, past = bn == float(b10), bn == float(above)
        assert at10.any() and past.any()
        assert p[at10].all() and (lev[at10] == top).all(), "fl(0.1 bn) == 1: mask 1, top level"
        assert not p[past].any() and (lev[past] == top).all(), "next float above: mask 0"
        assert len(ties) >= min(top, 48) // 2, f"construction: only {len(ties)} ties"
        for t, want in ties:
            at = bn == float(t)
            assert at.any() and (lev[at] == want).all(), (float(t), want, lev[at].unique())
        assert torch.equal(lev, dorefa_levels(torch.relu(bn), a_bits))
        assert torch.equal(p, dorefa_mask(bn))
        return
    one = bn.abs() == 1
    below = bn.abs() == float(np.nextafter(np.float32(1), np.float32(0)))
    assert one.any() and below.any()
    assert not p[one].any() and p[below].all(), "|bn| = 1 must not pass, nextafter(1, 0) must"
    assert torch.equal(p, bn.abs() < 1)
    if kind == "pool":
        arg = out["arg"].t.view(B, Cc, H // 2, W // 2)
        y = out["y"].t.view(B, Cc, H // 2, W // 2)
        pos = ~(bn < 0)
        w = pos.view(B, Cc, H // 2, 2, W // 2, 2)
        cnt = w.sum((3, 5))
        assert (cnt == 0).any() and (cnt == 4).any() and ((cnt > 0) & (cnt < 4)).any()
        assert (arg[cnt == 0] == 0).all() and (y[cnt == 0] == -1).all(), "all -1: element 0, -1"
        assert (arg[cnt == 4] == 0).all() and (y[cnt == 4] == 1).all(), "all +1: element 0, +1"
        want_arg, want_y = first_max_of_signs(bn)
        assert torch.equal(arg, want_arg) and torch.equal(y, want_y)
        # ATen itself on the oracle's +-1 tensor: the same winners
        ys = torch.where(bn < 0, -1.0, 1.0)
        _, idx = TF.max_pool2d(ys, 2, 2, return_indices=True)
        r, s = idx // W % 2, idx % W % 2
        assert torch.equal(arg.long(), r * 2 + s), "first-maximum rule differs from ATen's max_pool2d"
        return
    y = out["y"].t.view(B, Cc, H, W)
    assert (y[zero] == 1).all(), "bn = +-0 must give +1"
    assert torch.equal(y, torch.where(bn < 0, -1.0, 1.0))


# ============================================================================ module level: fused.BatchNormReluQuant2d
@pytest.mark.parametrize("B,plane", [
    pytest.param(16, _plane(NIN, 192, 16, 1), id="nin-16x192@16-a8"),
    pytest.param(8, _plane(NIN, 160, 32, 1), id="nin-8x160@32-a8"),
    pytest.param(8, _plane(GC, 512, 16, 16), id="gc-8x512@16-sg16-a4"),
])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_bn_relu_quant_module_against_fp64(B, plane, training):
    """the whole module (statistics, producer, backward through mnb_bn_sign_bwd with its relu-and-clamp mask).  The
    statistics it used are recomputed with mnb_bn_batch_stats on copies of the running buffers (deterministic: the same
    bits), or read from the running buffers in eval mode, so the kernel checks above apply unchanged: levels and mask
    exact against the emulation (the reference restated for these statistics), dgamma / dbeta / dx within the bounds of
    check_reductions / check_dx (eval: dx = fl(k g m) exactly), running statistics and num_batches_tracked bit for bit.
    The statistics themselves against fp64 are test_gpu_quant_kernels.test_bn_batch_stats_vs_fp64_and_running_updates."""
    from micronet_b200.fused import BatchNormReluQuant2d
    L, lib = _lib()
    Cc, H, W, sg, _, a_bits = plane
    hw, N = H * W, B * H * W
    g0 = _gen(Cc + H + B)
    mod = BatchNormReluQuant2d(Cc).to(DEV)
    mod.a_bits, mod.out_shuffle_groups = a_bits, sg
    with torch.no_grad():
        mod.weight.copy_(torch.rand(Cc, generator=g0, device=DEV) * 4 + 1)
        mod.bias.copy_(torch.randn(Cc, generator=g0, device=DEV) * 2 + 2)
        mod.running_mean.copy_(torch.randn(Cc, generator=g0, device=DEV))
        mod.running_var.copy_(torch.rand(Cc, generator=g0, device=DEV) + 0.5)
    mod.train(training)
    x = torch.randn(B, Cc, H, W, generator=g0, device=DEV) * 1.5 + 0.5
    rm, rv, nbt = mod.running_mean.clone(), mod.running_var.clone(), mod.num_batches_tracked.clone()
    xg = x.clone().requires_grad_(True)
    y = mod(xg)
    packed, bits = y._mnb_pk_q
    assert bits == a_bits
    if training:
        stats = torch.empty(2 * Cc, device=DEV)
        L.check(lib.mnb_bn_batch_stats(x.data_ptr(), B, Cc, hw, float(mod.eps), float(mod.momentum), rm.data_ptr(),
                                       rv.data_ptr(), nbt.data_ptr(), stats.data_ptr(), L.scratch(x.device, Cc).data_ptr(),
                                       L.stream()), "bn_batch_stats")
        mean, invstd = stats[:Cc], stats[Cc:]
        assert _eq(mod.running_mean, rm) and _eq(mod.running_var, rv) and int(mod.num_batches_tracked) == int(nbt) == 1
    else:
        mean, invstd = rm, torch.rsqrt(rv + mod.eps)
        assert _eq(mod.running_mean, rm) and _eq(mod.running_var, rv) and int(mod.num_batches_tracked) == 0
    gamma = mod.weight.detach()
    bn, _ = emulate_bn(x, mean, invstd, gamma, mod.bias.detach())
    lev = _unshuffle(decode_plane(packed, 1, B, Cc, hw)[0].view(B, Cc, H, W), sg)
    want = dorefa_levels(torch.relu(bn), a_bits)
    assert torch.equal(lev, want), f"levels: {_first_diff(lev, want)}"
    semantic_check(x, mean, invstd, gamma, mod.bias.detach(), "dorefa", a_bits, dict(level=lev, mask=dorefa_mask(bn)))
    g = torch.randn(B, Cc, H, W, generator=g0, device=DEV)          # in the module's output (shuffled) channel order
    y.backward(g)
    gm = torch.where(dorefa_mask(bn), _unshuffle(g, sg), torch.zeros((), device=DEV))
    splits = plane_splits(B, N, Cc)
    ref = bwd_reference(gm, x, mean, invstd, gamma)
    b_db, b_dg = check_reductions(ref, mod.weight.grad, mod.bias.grad, reduce_chain("vec", B, hw, splits), N, B, 1)
    if training:
        check_dx(xg.grad, gm, x, mean, invstd, ref, b_db, b_dg, N, "dx (module, training)")
    else:
        want_dx = (gamma * invstd).view(1, -1, 1, 1) * gm
        assert _eq(xg.grad, want_dx), f"dx (module, eval): {_first_diff(xg.grad, want_dx)}"


@pytest.mark.parametrize("shape,sg", [pytest.param((4, 20, 8, 8), 4, id="C20-C%8"), pytest.param((4, 16, 6, 6), 2, id="hw36-hw%32")])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_bn_relu_quant_module_falls_back_outside_the_fused_cover(shape, sg, training):
    """C % 8 != 0 or hw % 32 != 0: the module is nn.BatchNorm2d -> ReLU [-> the folded shuffle], the same ATen ops as the
    un-fused block, so output, gradients and running statistics equal them bit for bit, and no producer kernel runs"""
    from micronet_b200.fused import BatchNormReluQuant2d
    L, _ = _lib()
    B, Cc, H, W = shape
    g0 = _gen(Cc + H)
    ref = nn.BatchNorm2d(Cc).to(DEV)
    with torch.no_grad():
        ref.weight.copy_(torch.rand(Cc, generator=g0, device=DEV) + 0.5)
        ref.bias.copy_(torch.randn(Cc, generator=g0, device=DEV))
    mod = BatchNormReluQuant2d(Cc).to(DEV)
    mod.load_state_dict(ref.state_dict())
    mod.a_bits, mod.out_shuffle_groups = 4, sg
    ref.train(training); mod.train(training)
    x = torch.randn(shape, generator=g0, device=DEV) * 2
    g = torch.randn(shape, generator=g0, device=DEV)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    n0 = L.launch_count()
    ya = mod(xa)
    assert L.launch_count() == n0, "a producer kernel ran outside its cover"
    assert not hasattr(ya, "_mnb_pk_q")
    yb = _shuffle(torch.relu(ref(xb)), sg)
    assert torch.equal(ya, yb)
    ya.backward(g); yb.backward(g)
    assert torch.equal(xa.grad, xb.grad)
    assert torch.equal(mod.weight.grad, ref.weight.grad) and torch.equal(mod.bias.grad, ref.bias.grad)
    assert torch.equal(mod.running_mean, ref.running_mean) and torch.equal(mod.running_var, ref.running_var)
