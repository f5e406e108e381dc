"""Consumer-plane epilogues of the packed-operand convolutions (mnb_pk_conv_post, mnb_pk_i8_conv with a consumer) against a
host reference, at every case of tests/pk_post_cases.py: every (epilogue path, N tile) instance, the plan features, several
work items per CTA, and every linked conv of the frozen graphs at the batch the benchmark runs them.  Behind a segmented
producer plan (asymmetric levels), mnb_pk_conv_post refuses before launching or writes what the unfused pair writes, and
functional.frozen_conv hands the consumer the plane its own quantizer makes of y.

Operands are integer levels, so the conv sum S is exact (|S| < 2^24, asserted; S is computed on the device in fp64 and
must be integral).  Each launch writes into an fp32 ``out`` filled with NaN and a plane filled with 0x5A followed by guard
bytes; it runs twice and both runs must give the same bits, and the tensor-core error flag must stay clean.

Bit-exact check: the epilogue's documented fp32 op sequence, evaluated from S:
    scv = fl(a_scale * n_scale);  y = fmaf(S, scv, bias);  [BatchNorm: fmaf(fl(y - mean), fl(gamma * invstd), beta)];
    [ReLU];  the oracle's quantizer (levels + zero point), or the sequential round-to-nearest bf16 split into pieces.
fmaf is emulated as an fp64 sum rounded to fp32; the only elements that double rounding can flip are those whose fp64 sum
is exactly halfway between two fp32 values, and those are settled by the sign of the sum's exact TwoSum error.  Every plane byte
(levels, zeroed channel padding, every phase, the shuffled destination) and the guard bytes must match; ``out`` too.

fp64 check (against a reference that copies a wrong op order): the chain in fp64 without intermediate rounding, quantized
in fp64.  Levels may differ by exactly one, and only where the fp64 value lies within the fp32 chain's error bound of a
rounding boundary; term planes must stay within that bound of the fp64 value.

Boundary channels place values on the quantizer's rounding boundaries and clamp edges: some channels have n_scale = 0 (y is
the bias, set to a boundary or one ulp beside it), others a power-of-two scale of one ulp of a boundary bias and a single
+-1 weight tap, so y steps through the consecutive fp32 values around that boundary."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests import pk_plan_util as PU
from tests import pk_post_cases as P

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 256
EPS = 2.0 ** -24


# ---- fp32 arithmetic of the reference
def round_half_away(v):
    return torch.sign(v) * torch.floor(torch.abs(v) + 0.5)


def quant_levels(x, qd):
    """the oracle's quantizer on fp32 x: the stored level (IAO: clamped level + zero point) as fp32"""
    if qd["kind"] == "dorefa":
        s = torch.tensor(1.0 / float((1 << qd["bits"]) - 1), dtype=torch.float32, device=x.device)
        c = torch.clamp(x * torch.tensor(0.1, dtype=torch.float32, device=x.device), 0, 1)
        return round_half_away(c / s)
    sc = torch.tensor(qd["scale"], dtype=torch.float32, device=x.device)
    zp = torch.tensor(qd["zp"], dtype=torch.float32, device=x.device)
    return torch.clamp(round_half_away(x / sc - zp), qd["qmin"], qd["qmax"]) + zp


def quant_levels_fp64(x, qd):
    """(level, distance of the quantizer's pre-rounding value to the nearest rounding boundary, in its own units, value)"""
    if qd["kind"] == "dorefa":
        s = float(np.float32(1.0 / float((1 << qd["bits"]) - 1)))
        u = torch.clamp(x * 0.1, 0, 1) / s + 0.5
        return torch.floor(u), (u - torch.round(u)).abs(), u
    v = x / qd["scale"] - qd["zp"]
    lev = torch.clamp(torch.sign(v) * torch.floor(v.abs() + 0.5), qd["qmin"], qd["qmax"]) + qd["zp"]
    frac = v.abs() - torch.floor(v.abs())
    return lev, (frac - 0.5).abs(), v


def edges(qd):
    """fp32 values at every rounding boundary and clamp edge of a quantizer"""
    if qd["kind"] == "dorefa":
        n = (1 << qd["bits"]) - 1
        s = float(np.float32(1.0 / n))
        e = [(k + 0.5) * s * 10.0 for k in range(n)] + [0.0, 10.0]
    else:
        e = [(k + 0.5 + qd["zp"]) * qd["scale"] for k in range(qd["qmin"] - 2, qd["qmax"] + 2)]
    return [float(np.float32(v)) for v in e]


def qrange(qd):
    if qd is None:
        return 0.0, 4.0
    if qd["kind"] == "dorefa":
        return 5.0, 6.0
    lo, hi = (qd["qmin"] + qd["zp"]) * qd["scale"], (qd["qmax"] + qd["zp"]) * qd["scale"]
    return (lo + hi) / 2, (hi - lo) / 2 * 1.15


# ---- operands of a case
def operands(case, gen):
    B, Cc, H, W, K, R, st, pad, G = case.shape
    kg = Cc // G
    lim_a = 127
    lim_w = 127
    while kg * R * R * lim_a * lim_w >= (1 << 24):
        lim_w //= 2
    x = torch.randint(-lim_a, lim_a + 1, (B, Cc, H, W), generator=gen).float()
    # the first image holds small levels only: the single-tap boundary channels below then step through every fp32 value
    # within a few ulps of their boundary, where the quantizer's fast path hands over to the IEEE division
    x[0] = torch.randint(-4, 5, (Cc, H, W), generator=gen).float()
    w = torch.randint(-lim_w, lim_w + 1, (K, kg, R, R), generator=gen).float()
    qd = P.qparams(case.q)[1] if case.q else None
    centre, half = qrange(qd)
    # per-channel roles: 0 normal, 1 one-ulp steps around a boundary bias (a single +-1 weight tap), 2 n_scale = 0
    role = torch.zeros(K, dtype=torch.int64)
    if qd is not None:
        role[1::4] = 1
        role[3::8] = 2
    e = edges(qd) if qd is not None else [1.0]
    n_scale = torch.zeros(K)
    bias = torch.zeros(K)
    std = math.sqrt(kg * R * R) * lim_a * lim_w / 3.0
    bnd = 0
    for k in range(K):
        if role[k] == 1:
            w[k].zero_()
            w[k].view(-1)[int(torch.randint(0, kg * R * R, (1,), generator=gen))] = 1.0 if k % 3 else -1.0
            b = e[bnd % len(e)]
            bnd += 1
            n_scale[k] = 2.0 ** (math.frexp(b)[1] - 24) if b != 0 else 2.0 ** -30
            bias[k] = b
        elif role[k] == 2:
            b = np.float32(e[bnd % len(e)])
            bnd += 1
            step = (k // 8) % 3 - 1
            if step:
                b = np.nextafter(b, np.float32(step * np.inf))
            n_scale[k], bias[k] = 0.0, float(b)
        else:
            n_scale[k] = float(np.float32(half / std * (0.5 + float(torch.rand(1, generator=gen)))))
            bias[k] = centre + half * 0.3 * float(torch.randn(1, generator=gen))
    bn = None
    if case.bn:
        mean = torch.randn(K, generator=gen) * half * 0.2
        invstd = torch.rand(K, generator=gen) + 0.5
        gamma = (torch.rand(K, generator=gen) + 0.5) * torch.where(torch.rand(K, generator=gen) < 0.2, -1.0, 1.0)
        beta = torch.randn(K, generator=gen) * half * 0.2
        fixed = role > 0       # boundary channels pass y through the BatchNorm unchanged
        mean[fixed], invstd[fixed], gamma[fixed], beta[fixed] = 0.0, 1.0, 1.0, 0.0
        bn = [t.float().contiguous() for t in (mean, invstd, gamma, beta)]
    return x, w, n_scale.float(), bias.float(), bn, qd, role


def encode(vals, K, cpu, split, sg):
    """stored values [B, K, OH, OW] (fp32) -> the bytes of the consumer plane (bf16 for cpu 8, int8 for cpu 16)"""
    B, _, OH, OW = vals.shape
    if sg > 1:
        cpg = K // sg
        c = torch.arange(K, device=vals.device)
        dst = (c % cpg) * sg + c // cpg
        sh = torch.empty_like(vals)
        sh[:, dst] = vals
        vals = sh
    units = (K + cpu - 1) // cpu
    if units * cpu != K:
        vals = torch.cat([vals, torch.zeros(B, units * cpu - K, OH, OW, device=vals.device)], 1)
    v = vals.view(B, units, cpu, OH, OW)
    if split:
        v = v.view(B, units, cpu, OH // 2, 2, OW // 2, 2).permute(0, 4, 6, 1, 3, 5, 2)
    else:
        v = v.permute(0, 1, 3, 4, 2)
    v = v.contiguous()
    if cpu == 16:
        return v.to(torch.int8).view(torch.uint8).flatten()
    return v.to(torch.bfloat16).view(torch.uint8).flatten()


def decode_terms(plane_bytes, K, shape4, split, terms):
    """sum of the term pieces per (b, consumer channel, h, w), in fp64 (unshuffled positions: consumer channel order)"""
    B, _, OH, OW = shape4
    units = (K + 7) // 8
    pl = plane_bytes.view(torch.bfloat16).double().view(terms, -1)
    if split:
        v = pl.view(terms, B, 2, 2, units, OH // 2, OW // 2, 8).permute(0, 1, 4, 7, 5, 2, 6, 3)
    else:
        v = pl.view(terms, B, units, OH, OW, 8).permute(0, 1, 2, 5, 3, 4)
    return v.reshape(terms, B, units * 8, OH, OW)[:, :, :K].sum(0)


def unshuffle(vals, K, sg):
    if sg <= 1:
        return vals
    cpg = K // sg
    c = torch.arange(K, device=vals.device)
    return vals[:, (c % cpg) * sg + c // cpg]


def _launch(case, sh, a_pk, w_img, n_scale, bias, out, post):
    from micronet_b200 import _lib as L
    lib = L.load()
    err = L.tc_err_flag(torch.device(DEV)).data_ptr()
    if case.path in P.I8_PATHS:
        return lib.mnb_pk_i8_conv(C.byref(sh), a_pk.data_ptr(), w_img.data_ptr(), n_scale.data_ptr(), None, 1.0,
                                  bias.data_ptr(), L.ptr(out), C.byref(post), err, L.stream())
    return lib.mnb_pk_conv_post(C.byref(sh), a_pk.data_ptr(), case.ta, w_img.data_ptr(), 1, n_scale.data_ptr(), None, 1.0,
                                bias.data_ptr(), L.ptr(out), C.byref(post), err, L.stream())


def run_case(case, monkeypatch):
    from micronet_b200 import _lib as L, pk as PK
    for k, v in case.env.items():      # before the weight packer too: the image layout depends on the plan
        monkeypatch.setenv(k, v)
    plan = P.plan_of(case)
    assert isinstance(plan, dict), f"{case.id}: refused {plan}"
    got = {k: plan[k] for k in case.expect}
    assert got == case.expect and plan["path"] == P.PATHS[case.path], \
        f"{case.id}: the plan changed: {got} != {case.expect} (full plan {plan})"
    B, Cc, H, W, K, R, st, pad, G = case.shape
    OH, OW = P.out_hw(case.shape)
    gen = torch.Generator().manual_seed(sum(map(ord, case.id)))
    x, w, n_scale, bias, bn, qd, role = operands(case, gen)
    x, w, n_scale, bias = x.to(DEV), w.to(DEV), n_scale.to(DEV), bias.to(DEV)
    bn = [t.to(DEV) for t in bn] if bn is not None else None
    sh = P.conv_shape(case.shape)
    i8 = case.path in P.I8_PATHS
    cpu = 16 if i8 else 8
    if i8:
        # a symmetric 8-bit quantizer of scale 1: the int8 levels are x itself
        unit = [torch.tensor([v], device=DEV) for v in (1.0, 0.0, -127.5, 127.5)]
        unit_q = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, *(t.data_ptr() for t in unit))
        a_pk = PK.pack_act_i8(x, unit_q, phase_split=st == 2)
        w_img = PK.pack_weight_i8(sh, w.to(torch.int16))
    else:
        a_pk, _ = PK.pack_act(x, None, case.ta, phase_split=st == 2)
        w_img = PK.pack_weight(sh, 0, case.ta, 1, w_int=w.to(torch.int16))
    # the exact sums, on the device in fp64
    S = TF.conv2d(x.double(), w.double(), None, st, pad, 1, G)
    assert torch.equal(S, S.round()) and S.abs().max().item() < 2 ** 24
    # consumer quantizer and buffers
    terms = case.terms
    unit_bytes = int(L.load().mnb_pk_i8_act_bytes(B, K, OH, OW)) if i8 else int(L.load().mnb_pk_act_bytes(B, K, OH, OW, 1))
    nbytes = unit_bytes * max(terms, 1)
    buf = torch.empty(nbytes + GUARD, dtype=torch.uint8, device=DEV)
    out = torch.empty((B, K, OH, OW), dtype=torch.float32, device=DEV) if case.out else None
    qs, keep_q = None, []
    if case.q:
        qs, _, keep_q = P.qparams(case.q, DEV)
    bn_ptrs = tuple(t.data_ptr() for t in bn) if bn is not None else (None,) * 4
    post = P.post_struct(qs, buf.data_ptr(), case.relu, case.split, bn_ptrs, case.sg, terms)
    results = []
    for _ in range(2):
        buf.fill_(0x5A)
        if out is not None:
            out.fill_(float("nan"))
        L.check(_launch(case, sh, a_pk, w_img, n_scale, bias, out, post), case.id)
        torch.cuda.synchronize()
        results.append((buf.clone(), None if out is None else out.clone()))
    L.tc_check()
    assert torch.equal(results[0][0], results[1][0]), "second launch differs (plane)"
    if out is not None:
        assert torch.equal(results[0][1].view(torch.int32), results[1][1].view(torch.int32)), "second launch differs (out)"
    plane, yout = results[0]
    assert (plane[nbytes:] == 0x5A).all(), "guard bytes behind the plane were written"
    # ---- bit-exact reference of the fp32 op sequence
    stats = {}
    scv = n_scale.view(1, -1, 1, 1)                  # a_scale = 1: scv = fl(1 * n_scale) = n_scale
    y = PU.fmaf32(S.float(), scv, bias.view(1, -1, 1, 1), stats)
    if out is not None:
        assert not torch.isnan(yout).any(), "out positions the epilogue never wrote"
        assert torch.equal(yout.view(torch.int32), y.view(torch.int32)), \
            f"out: {(yout != y).sum().item()} elements differ"
    v = y
    if bn is not None:
        mean, invstd, gamma, beta = (t.view(1, -1, 1, 1) for t in bn)
        v = PU.fmaf32(v - mean, gamma * invstd, beta.expand_as(v), stats)
    if case.relu:
        v = torch.clamp_min(v, 0.0)
    # fp64 chain, no intermediate rounding
    S64 = S
    y64 = S64 * n_scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    Mx = S64.abs() * n_scale.double().view(1, -1, 1, 1) + bias.double().abs().view(1, -1, 1, 1)
    v64 = y64
    if bn is not None:
        mean, invstd, gamma, beta = (t.double().view(1, -1, 1, 1) for t in bn)
        gs = gamma * invstd
        v64 = (y64 - mean) * gs + beta
        Mx = (Mx + mean.abs()) * gs.abs() + beta.abs()
    if case.relu:
        v64 = torch.clamp_min(v64, 0.0)
    ex = 4 * EPS * Mx                                   # error bound of the fp32 chain on the quantizer input
    if terms:
        pieces, r = [], v
        for _ in range(3):
            p = r.to(torch.bfloat16)
            pieces.append(p.float())
            r = r - p.float()
        assert torch.equal(pieces[0].double() + pieces[1].double() + pieces[2].double(), v.double()), \
            "three bf16 pieces do not hold the fp32 value"
        want = torch.cat([encode(pieces[t], K, 8, case.split, case.sg) for t in range(terms)])
        got = plane[:nbytes]
        bad = (got != want).sum().item()
        assert bad == 0, f"{case.id}: {bad} of {nbytes} term-plane bytes differ"
        dec = unshuffle(decode_terms(got, K, (B, K, OH, OW), case.split, terms), K, case.sg)
        ratio = None
        if terms == 3:      # (fewer pieces hold the value truncated: their bits are checked against the split above)
            assert torch.equal(dec, v.double())
            err = (dec - v64).abs()
            assert (err <= ex).all(), f"{case.id}: term planes off the fp64 chain by more than 4 * 2^-24 * M"
            ratio = (err / ex.clamp_min(1e-300)).max().item()
        print(f"{case.id}: terms {terms}, worst |pieces - fp64 chain| / bound = {ratio}, "
              f"fma midpoints settled: {stats.get('midpoints', 0)}")
        return ratio
    lev = quant_levels(v, qd)
    want = encode(lev, K, cpu, case.split, case.sg)
    got = plane[:nbytes]
    bad = (got != want).sum().item()
    assert bad == 0, f"{case.id}: {bad} of {nbytes} plane bytes differ"
    if qd["kind"] == "dorefa":
        _assert_boundaries_straddled(v, lev, role, bias, qd)
    # fp64 check
    lev64, dist, u = quant_levels_fp64(v64, qd)
    if qd["kind"] == "dorefa":
        s = float(np.float32(1.0 / float((1 << qd["bits"]) - 1)))
        du = 0.1 * ex / s + 8 * EPS * (u.abs() + 1)
    else:
        du = ex / qd["scale"] + 8 * EPS * (u.abs() + abs(qd["zp"]) + 1)
    diff = (lev.double() - lev64).abs()
    near = diff != 0
    assert ((diff <= 1) & (~near | (dist <= du))).all(), \
        f"{case.id}: levels differ from the fp64 chain away from a rounding boundary"
    placed = (role > 0).to(DEV).view(1, -1, 1, 1).expand_as(near)
    print(f"{case.id}: one level off the fp64 chain near a boundary: {int((near & ~placed).sum())} elements of the random "
          f"channels, {int((near & placed).sum())} of the boundary channels ({int((dist <= du).sum())} within the bound of a "
          f"boundary); fma midpoints settled: {stats.get('midpoints', 0)}")
    return None


def _assert_boundaries_straddled(v, lev, role, bias, qd):
    """every one-ulp-step channel of a DoReFa consumer (boundaries fall after the x 0.1, as in the adversarial inputs of
    test_gpu_parity) holds levels on both sides of its boundary, and some of its values fall into the window in which
    mnb_act_levels redoes the fast reciprocal product with the IEEE division"""
    n = (1 << qd["bits"]) - 1
    s = np.float32(1.0 / n)
    rinv = np.float32(np.float32(1.0) / s)
    c = torch.clamp(v * torch.tensor(0.1, dtype=torch.float32, device=v.device), 0, 1)
    pa = c * float(rinv)
    f = pa + 0.5
    d = f - torch.floor(f)
    delta = 4e-7 * (pa + 1.0)
    redo = (d < delta) | (d > 1.0 - delta)
    bad = []
    for k in (role == 1).nonzero().flatten().tolist():
        b = float(bias[k])
        if b <= 0.0 or b >= 10.0:             # the clamp edges: no rounding boundary there
            continue
        if lev[:, k].unique().numel() < 2 or not bool(redo[:, k].any()):
            bad.append((k, b))
    assert not bad, f"boundary channels that do not straddle their boundary or miss the redo window: {bad[:8]}"


@pytest.mark.parametrize("case", P.ALL_CASES, ids=[c.id for c in P.ALL_CASES])
def test_epilogue_matches_the_reference(case, monkeypatch):
    run_case(case, monkeypatch)


@pytest.mark.parametrize("ref", P.REFUSALS, ids=[r.id for r in P.REFUSALS])
def test_refused_launch_writes_nothing(ref):
    """a refused consumer returns its code before launching: sentinels and guard bytes stay, the code is the query's"""
    from micronet_b200 import _lib as L
    lib = L.load()
    q_post, _ = P.host_post(ref.opts)
    want = P.query(ref.shape, ref.cpu, ref.ta, q_post)
    assert isinstance(want, tuple) and want[0] == {"E_ARG": -1, "E_UNSUPPORTED": L.E_UNSUPPORTED}[ref.code], want
    assert ref.text in want[1], want
    big = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    buf = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device=DEV)
    B, Cc, H, W, K = ref.shape[:5]
    OH, OW = P.out_hw(ref.shape)
    out = torch.full((B, K, OH, OW), float("nan"), device=DEV)
    vec = torch.ones(4096, device=DEV)
    qs, keep = None, []
    if ref.opts.get("q"):
        qs, _, keep = P.qparams(ref.opts["q"], DEV)
    bn = ref.opts.get("bn")
    ptrs = (vec.data_ptr(), vec.data_ptr() + 1024, vec.data_ptr() + 2048, vec.data_ptr() + 4096)
    bn_ptrs = ptrs if bn == "all" else (ptrs[0], None, ptrs[2], ptrs[3]) if bn == "partial" else (None,) * 4
    post = P.post_struct(qs, buf.data_ptr(), 1, ref.opts.get("split", 0), bn_ptrs, ref.opts.get("sg", 1),
                         ref.opts.get("terms", 0))
    sh = P.conv_shape(ref.shape)
    n0 = L.launch_count()
    err = L.tc_err_flag(torch.device(DEV)).data_ptr()
    if ref.cpu == 16:
        rc = lib.mnb_pk_i8_conv(C.byref(sh), big.data_ptr(), big.data_ptr(), vec.data_ptr(), None, 1.0, vec.data_ptr(),
                                out.data_ptr(), C.byref(post), err, L.stream())
    else:
        rc = lib.mnb_pk_conv_post(C.byref(sh), big.data_ptr(), ref.ta, big.data_ptr(), 1, vec.data_ptr(), None, 1.0,
                                  vec.data_ptr(), out.data_ptr(), C.byref(post), err, L.stream())
    torch.cuda.synchronize()
    assert rc == want[0] and L.launch_count() == n0, (rc, want)
    assert lib.mnb_last_error().decode(errors="replace") == want[1]
    assert (buf == 0x5A).all() and torch.isnan(out).all(), "refused, yet something was written"


# ---- the other plane producers of the frozen ResNet-18 graph, at its 224 x 64 planes
def _guarded_plane(nbytes):
    return torch.full((nbytes + GUARD,), 0x5A, dtype=torch.uint8, device=DEV)


def _edge_values(qd, n, gen):
    """n fp32 values on and one ulp beside the rounding boundaries and clamp edges of a quantizer"""
    e = torch.tensor(edges(qd), dtype=torch.float32)
    pick = e[torch.randint(0, e.numel(), (n,), generator=gen)]
    step = torch.randint(-1, 2, (n,), generator=gen).float()
    return torch.nextafter(pick, pick + step * math.inf).where(step != 0, pick)


# (B, C, H, W, phase split): the QuantAdd of each residual stage writes the plane of the next block's first conv (stride 2
# behind the first three stages)
ADD_PLANES = [(64, 64, 224, 224, True), (64, 128, 112, 112, True), (64, 256, 56, 56, True), (64, 512, 28, 28, False)]


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
@pytest.mark.parametrize("plane", ADD_PLANES, ids=lambda p: f"{p[1]}x{p[2]}" + ("_split" if p[4] else ""))
def test_quant_add_pack_matches_the_reference(plane, i8):
    """mnb_quant_add_pack_fwd / _i8: out = ReLU(Q(a) + Q(b)) bit for bit, and the consumer plane = the consumer's quantizer
    of it, every byte, guard bytes untouched"""
    from micronet_b200 import _lib as L
    B, Cc, H, W, split = plane
    gen = torch.Generator().manual_seed(Cc + 7 * int(i8))
    qa, da, keep_a = P.qparams("iao8", DEV)
    qn, dn, keep_n = P.qparams("iao8", DEV, rng=(-2.9, 4.1))
    a = torch.randn(B, Cc, H, W, generator=gen) * 2.5
    b = torch.randn(B, Cc, H, W, generator=gen) * 2.5
    m = a.numel() // 16                      # a sixteenth of each input on the boundaries of the add's quantizer
    a.view(-1)[:m] = _edge_values(da, m, gen)
    b.view(-1)[-m:] = _edge_values(da, m, gen)
    a, b = a.to(DEV), b.to(DEV)
    cpu = 16 if i8 else 8
    lib = L.load()
    nbytes = int(lib.mnb_pk_i8_act_bytes(B, Cc, H, W)) if i8 else int(lib.mnb_pk_act_bytes(B, Cc, H, W, 1))
    buf = _guarded_plane(nbytes)
    out = torch.full((B, Cc, H, W), float("nan"), device=DEV)
    post = P.post_struct(qn, buf.data_ptr(), 0, split, (None,) * 4, 1, 0)
    fn = lib.mnb_quant_add_pack_i8_fwd if i8 else lib.mnb_quant_add_pack_fwd
    res = []
    for _ in range(2):
        buf.fill_(0x5A)
        out.fill_(float("nan"))
        L.check(fn(a.data_ptr(), b.data_ptr(), B, Cc, H, W, C.byref(qa), 1, out.data_ptr(), C.byref(post), L.stream()),
                "quant_add_pack")
        torch.cuda.synchronize()
        res.append((buf.clone(), out.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1].view(torch.int32), res[1][1].view(torch.int32))
    sc = torch.tensor(da["scale"], dtype=torch.float32, device=DEV)
    t = torch.clamp_min(quant_levels(a, da) * sc + quant_levels(b, da) * sc, 0.0)
    assert torch.equal(res[0][1].view(torch.int32), t.view(torch.int32)), "QuantAdd output differs"
    want = encode(quant_levels(t, dn), Cc, cpu, split, 1)
    got = res[0][0]
    assert (got[nbytes:] == 0x5A).all(), "guard bytes behind the plane were written"
    bad = (got[:nbytes] != want).sum().item()
    assert bad == 0, f"{bad} of {nbytes} plane bytes differ"


# (B, C, H, W, k, s, p): the IAO QuantMaxPool2d of the frozen NIN / NIN-GC graphs on planes of the ResNet-18 224 x 64 sizes
POOL_PLANES = [(64, 64, 224, 224, 3, 2, 1), (64, 128, 112, 112, 2, 2, 0), (64, 256, 56, 56, 3, 2, 1)]


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
@pytest.mark.parametrize("plane", POOL_PLANES, ids=lambda p: f"{p[1]}x{p[2]}_k{p[4]}s{p[5]}p{p[6]}")
def test_plane_maxpool_requant_matches_the_reference(plane, i8):
    """mnb_pk_plane_maxpool_requant: the consumer's quantizer of max_pool2d of the pool quantizer's dequantized levels"""
    from micronet_b200 import _lib as L
    B, Cc, H, W, k, s, p = plane
    gen = torch.Generator().manual_seed(Cc + k + 3 * int(i8))
    qi, di, keep_i = P.qparams("iao8", DEV)
    qo, do, keep_o = P.qparams("iao8", DEV, rng=(-2.3, 3.1))
    cpu = 16 if i8 else 8
    lev_in = torch.randint(-128, 128, (B, Cc, H, W), generator=gen).float().to(DEV)
    src = encode(lev_in, Cc, cpu, False, 1)
    OH, OW = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    lib = L.load()
    nbytes = int(lib.mnb_pk_i8_act_bytes(B, Cc, OH, OW)) if i8 else int(lib.mnb_pk_act_bytes(B, Cc, OH, OW, 1))
    buf = _guarded_plane(nbytes)
    res = []
    for _ in range(2):
        buf.fill_(0x5A)
        L.check(lib.mnb_pk_plane_maxpool_requant(src.data_ptr(), B, Cc, H, W, k, s, p, int(i8), C.byref(qi), C.byref(qo),
                                                 buf.data_ptr(), L.stream()), "plane_maxpool_requant")
        torch.cuda.synchronize()
        res.append(buf.clone())
    assert torch.equal(res[0], res[1])
    sc = torch.tensor(di["scale"], dtype=torch.float32, device=DEV)
    vals = torch.clamp(lev_in, di["qmin"], di["qmax"]) * sc
    pooled = TF.max_pool2d(vals, k, s, p)
    want = encode(quant_levels(pooled, do), Cc, cpu, False, 1)
    got = res[0]
    assert (got[nbytes:] == 0x5A).all(), "guard bytes behind the plane were written"
    bad = (got[:nbytes] != want).sum().item()
    assert bad == 0, f"{bad} of {nbytes} plane bytes differ"


# ---- fused consumer behind a segmented producer plan (frozen inference graphs)
# asymmetric IAO producer: its levels (code + zero point) take two bf16 pieces, so with 3x3 x 64 channels the K loop is
# segmented; the consumer is a symmetric IAO conv (one-piece plane)
POST_SHAPE = (4, 64, 16, 16, 128, 3, 1, 1, 1)
POST_PLAN = dict(segmented=1, npairs=2, Nt=128)


def _iao(scale, sym, dev=DEV):
    from micronet_b200 import _lib as L, functional as F_
    zp = 0.0 if sym else -101.0
    lo, hi = (-127.5 * scale, 127.5 * scale) if sym else ((0 + zp) * scale, (255 + zp) * scale)
    bufs = dict(scale=torch.tensor([scale]), zero_point=torch.tensor([zp]), obs_min=torch.tensor([lo]), obs_max=torch.tensor([hi]))
    return F_.ActSpec(L.ACT_IAO, qmin=-128 if sym else 0, qmax=127 if sym else 255, q_type=0 if sym else 1,
                      **{k: v.to(dev) for k, v in bufs.items()})


def _post_operands():
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = POST_SHAPE
    g = torch.Generator().manual_seed(21)
    x = (torch.randn(B, Cc, H, W, generator=g) * 3).to(DEV)
    w_int = torch.randint(-127, 128, (K, Cc, R, R), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) * 0.01 + 0.001).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    spec, nxt = _iao(0.05, False), _iao(0.11, True)
    sh = PU.shape(*POST_SHAPE)
    x_pk, _ = PK.pack_act(x, spec.struct(), 2)
    w_img = PK.pack_weight(sh, 0, 2, 1, w_int=w_int)
    y_ref = torch.empty(B, K, H, W, device=DEV)
    from micronet_b200 import _lib as L
    L.check(PK.conv(sh, 0, x_pk, 2, w_img, 1, y_ref, n_scale=w_scale, a_scale=spec.scale, bias=bias), "conv")
    return sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref


def _check_post(with_out):
    """mnb_pk_conv_post on the segmented plan either refuses it before launching or writes exactly what the unfused pair
    writes; it must never return success with the consumer plane (or y) left unwritten"""
    from micronet_b200 import _lib as L, pk as PK
    plan = PU.conv_plan(PU.shape(*POST_SHAPE), 0, 2, 1)
    assert {k: plan[k] for k in POST_PLAN} == POST_PLAN, plan
    sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref = _post_operands()
    B, Cc, H, W, K = POST_SHAPE[:5]
    for relu in (False, True):
        for split in (False, True):
            want, _ = PK.pack_act(y_ref, nxt.struct(), 1, phase_split=split, relu=relu)
            plane = PK.consumer_plane(B, K, H, W, DEV).fill_(0xFF)
            y = torch.full_like(y_ref, float("nan")) if with_out else None
            rc = PK.conv_post(sh, x_pk, 2, w_img, 1, y, nxt.struct(), plane, relu, split, n_scale=w_scale,
                              a_scale=spec.scale, bias=bias)
            torch.cuda.synchronize()
            if rc == L.E_UNSUPPORTED:
                assert (plane == 0xFF).all() and (y is None or torch.isnan(y).all()), "refused, yet something was written"
                continue
            L.check(rc, "conv_post")
            assert torch.equal(plane, want), ("consumer plane", relu, split)
            if with_out:
                assert torch.equal(y, y_ref), ("y", relu, split)
    L.tc_check()


def test_conv_post_on_a_segmented_producer_plan_with_out():
    _check_post(True)


def test_conv_post_on_a_segmented_producer_plan_plane_only():
    _check_post(False)


@pytest.mark.parametrize("only", [False, True], ids=["y_kept", "plane_only"])
def test_frozen_conv_behind_an_asymmetric_producer_hands_the_right_plane(only):
    """functional.frozen_conv with a consumer: whatever path it takes, y equals the plain conv and the plane the consumer
    reads equals the consumer's own quantizer applied to y"""
    from micronet_b200 import functional as F_, pk as PK
    sh, x, x_pk, w_int, w_img, w_scale, bias, spec, nxt, y_ref = _post_operands()
    B, Cc, H, W, K, R, st, pad, G = POST_SHAPE
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    consumer_mod = torch.nn.Identity()
    for relu in (False, True):
        cons = F_.Consumer(consumer_mod, nxt, relu, only, (K, K, 3, 3), (1, 1), (1, 1), (1, 1), 1, True)
        assert cons.accepts((B, K, H, W))
        y = F_.frozen_conv(x, None, wq, bias, w_int, w_scale, spec, (1, 1), (1, 1), (1, 1), 1, consumer=cons)
        torch.cuda.synchronize()
        plane = F_.handed_plane(consumer_mod, y)
        want, _ = PK.pack_act(y_ref, nxt.struct(), 1, relu=relu)
        if plane is None:            # not fused: y holds the data, the consumer packs it itself
            assert torch.equal(y, y_ref)
            got, _ = PK.pack_act(y, nxt.struct(), 1, relu=relu)
            assert torch.equal(got, want)
        else:
            assert torch.equal(plane, want), relu
            if y.device.type != "meta":
                assert torch.equal(y, y_ref)
