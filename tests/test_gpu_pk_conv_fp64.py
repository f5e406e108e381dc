"""The packed-operand family's general kernels (mnb_pk_conv, mnb_pk_i8_conv, mnb_pk_wgrad) at every case of
tests/pk_conv_cases.py - the synthetic plan cases and every launch of the bench workloads at the bench batch - against fp64
convolutions of the same operands (computed on the GPU in float64).

* Outputs start as NaN with a NaN guard tail past their end, the weight gradient's scratch as 0x5A bytes; each launch runs
  twice and must give the same bits, leave the guard and the tensor-core error flag untouched.
* Integer operands are bit-exact: every partial sum is an exact integer below 2^24 (level bounds are chosen per shape so
  that kg x taps x |a| x |w| < 2^24; two-piece asymmetric levels up to 383 on the segmented plans), so the conv sum S is
  the fp64 one and the epilogue is checked bit for bit:
    forward / int8      y  = fmaf(S, sc, bias),   sc = fl(a_scale * n_scale[k]) (or a_scale alone), bias 0 when absent;
                        the int8 result also equals mnb_pk_conv's on the same levels bit for bit;
    data gradient       dx = fl(S * gain) where the STE mask passes, +0.0 where it does not; without a mask
                        fmaf(S, a_scale_const, 0);
    weight gradient     dw = fl(S * fl(a_scale / kdiv[k])), fl(S * a_scale), fl(S * fl(1 / kdiv[k])) or S.
  fmaf is evaluated in fp64 (the product is exact) with the one double-rounding case, a sum on an fp32 midpoint, settled
  by the sign of the sum's exact TwoSum error.
* Split fp32 operands are held element-wise: |got - ref| <= c * R, R = the same convolution of |operands| in fp64 (times
  |scale|, plus |bias|).  c per configuration:
    forward (3, 1), (3, 3), (1, 3): the pieces of each operand are exact; the dropped piece products of (3, 3) sum below
      2^-22 R; a segment's chain of <= 64 MMAs (truncating adds) and the RN adds of the segments stay below ~2^-21 R.
      c = 2^-20.  A dropped kept product or a lost segment is caught when its magnitude exceeds 2^-20 R: every product of
      the leading pieces, the second-piece products of (3, 1) / (3, 3) on these operands, and any lost segment of the
      plans here; the smallest kept products (2^-16 of the operand magnitudes, times a sum of mixed signs) can be smaller.
      Each is also held to max |err| <= 3e-6 max |ref|, which R does not imply under cancellation.
    data gradient: dy keeps two pieces (2^-16 relative truncation of dy) over chains of <= 64 MMAs: c = 2^-15.
    weight gradient: dy keeps two pieces, and the chains reach 256 MMAs before their RN split adds: c = 2^-14.
  A case with ``maxnorm`` is held to max |err| <= maxnorm * max |ref| as well.  With an fp32 dy against integer weights
  the weights' per-channel scale is folded into dy (one channel's scale 0), as the models' data gradient does.  The worst
  err / R of every configuration is printed.
* Refusal cases return the query's code and text, launch nothing, and leave outputs and guards untouched."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as TF

from tests import pk_conv_cases as PC
from tests.pk_plan_util import case_shape as shape, env, fmaf32, query

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 64
C_FWD, C_DGRAD, C_WGRAD = 2.0 ** -20, 2.0 ** -15, 2.0 ** -14
MAX_FWD = 3e-6
WORST = {}


def _nan(n):
    return torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=DEV)


def _rand_int(shape, bound, g):
    return torch.randint(-bound, bound + 1, shape, generator=g, device=DEV).float()


def _bounds(kg, taps, a_max, w_max):
    """(|a|, |w|) level bounds at most (a_max, w_max) with kg * taps * |a| * |w| < 2^24 (every partial sum exact)"""
    a, w = a_max, w_max
    while kg * taps * a * w >= 2 ** 24:
        if a >= w:
            a = max(1, a // 2)
        else:
            w = max(1, w // 2)
    return a, w


def _ref_conv(x, w, case):
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    return TF.conv2d(x.double(), w.double(), stride=st, padding=(ph, pw), groups=G)


def _ref_dgrad(dy, w, case):
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    P, Q = dy.shape[2:]
    op = (H - ((P - 1) * st - 2 * ph + R), W - ((Q - 1) * st - 2 * pw + S))
    return TF.conv_transpose2d(dy.double(), w.double(), stride=st, padding=(ph, pw), output_padding=op, groups=G)


def _ref_wgrad(x, dy, case):
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    return torch.nn.grad.conv2d_weight(x.double(), (K, Cc // G, R, S), dy.double(), stride=st, padding=(ph, pw), groups=G)


def _launch_twice(fn, out, n, scratch=None):
    from micronet_b200 import _lib as L
    flag = L.tc_err_flag(torch.device(DEV))
    flag.zero_()
    assert fn() == 0, L.load().mnb_last_error()
    torch.cuda.synchronize()
    first = out.clone()
    if scratch is not None:
        scratch.fill_(0x5A)                    # a partial tile the second launch skips would keep the poison
    assert fn() == 0, L.load().mnb_last_error()
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int32), out.view(torch.int32)), "second launch differs"
    assert torch.isnan(out[n:]).all(), "guard tail written"
    assert int(flag.item()) == 0, "tensor-core error flag set"
    return out[:n]


def _bits_equal(got, want, what):
    bad = (got.contiguous().view(torch.int32) != want.float().contiguous().view(torch.int32)).reshape(-1)
    nbad = int(bad.sum())
    if nbad:
        i = bad.nonzero()[:5, 0]
        raise AssertionError(f"{what}: {nbad} elements differ, first at {i.tolist()}: got {got.reshape(-1)[i].tolist()}, "
                             f"want {want.reshape(-1)[i].tolist()}")


def _bound(got, ref, R, c, key, maxnorm=0.0):
    """|got - ref| <= c * R element-wise and, where maxnorm is given, max |got - ref| <= maxnorm * max |ref|"""
    err = (got.double() - ref).abs()
    ratio = float((err / R.clamp_min(1e-30)).max())
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    print(f"worst err/R {key}: {WORST[key]:.3e}")
    assert torch.isfinite(got).all()
    assert bool((err <= c * R).all()), f"{key}: err/R {ratio:.3e} > {c:.3e}"
    if maxnorm:
        rel = float(err.max()) / float(ref.abs().max())
        WORST[key + " max-norm"] = max(WORST.get(key + " max-norm", 0.0), rel)
        print(f"worst max|err|/max|ref| {key}: {WORST[key + ' max-norm']:.3e}")
        assert rel <= maxnorm, f"{key}: max|err| / max|ref| {rel:.3e} > {maxnorm:.1e}"


def _iao_spec(scale=1.0, bits=8):
    from micronet_b200 import _lib as L, functional as F_
    half = 1 << (bits - 1)
    bufs = dict(scale=torch.tensor([scale]), zero_point=torch.zeros(1), obs_min=torch.tensor([-(half - 0.5) * scale]),
                obs_max=torch.tensor([(half - 0.5) * scale]))
    return F_.ActSpec(L.ACT_IAO, bits=bits, qmin=-half, qmax=half - 1, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})


def _fwd(case, g):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    ta, tw = case.terms
    sh = shape(case.shape)
    amax = 383 if case.ops == "asym" else (127 if case.mode == "i8" else 8)
    ab, wb = _bounds(Cc // G, R * S, amax, 127 if case.mode == "i8" else 7)
    if case.ops == "f32":
        x = torch.randn(B, Cc, H, W, generator=g, device=DEV)
    elif case.ops == "pm1":
        x = (torch.rand(B, Cc, H, W, generator=g, device=DEV) < 0.5).float() * 2 - 1
    else:
        x = _rand_int((B, Cc, H, W), ab, g)
    w_int = _rand_int((K, Cc // G, R, S), wb, g)
    w_f32 = torch.randn(K, Cc // G, R, S, generator=g, device=DEV) if tw > 1 else None
    n_scale = (torch.rand(K, generator=g, device=DEV) + 0.5) if case.epi["n_scale"] else None
    a_dev = torch.tensor([0.37], device=DEV) if case.epi["a_scale"] == "dev" else None
    a_const = 0.043
    bias = torch.randn(K, generator=g, device=DEV) if case.epi["bias"] else None
    P, Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1
    n = B * K * P * Q
    out = _nan(n)
    if case.mode == "i8":
        a_pk = PK.pack_act_i8(x, _iao_spec().struct(), phase_split=st == 2)
        w_img = PK.pack_weight_i8(sh, w_int.to(torch.int16))
        fn = lambda: PK.conv_i8(sh, a_pk, w_img, out, n_scale=n_scale, a_scale=a_dev, a_scale_const=a_const, bias=bias)
        # the bf16 kernel on the same levels, which the int8 result must equal bit for bit
        b_pk, _ = PK.pack_act(x, None, 1, phase_split=st == 2)
        b_img = PK.pack_weight(sh, 0, 1, 1, w_int=w_int.to(torch.int16))
        b_out = _nan(n)
        fn_bf16 = lambda: PK.conv(sh, 0, b_pk, 1, b_img, 1, b_out, n_scale=n_scale, a_scale=a_dev, a_scale_const=a_const,
                                  bias=bias)
    else:
        a_pk, _ = PK.pack_act(x, None, ta, phase_split=st == 2, groups=G)
        w_img = PK.pack_weight(sh, 0, ta, tw, w_f32=w_f32) if w_f32 is not None else \
            PK.pack_weight(sh, 0, ta, tw, w_int=w_int.to(torch.int16))
        fn = lambda: PK.conv(sh, 0, a_pk, ta, w_img, tw, out, n_scale=n_scale, a_scale=a_dev, a_scale_const=a_const, bias=bias)
    got = _launch_twice(fn, out, n).view(B, K, P, Q)
    if case.mode == "i8":
        _bits_equal(got, _launch_twice(fn_bf16, b_out, n).view(B, K, P, Q), f"{case.id}: int8 against bf16")
    w = w_f32 if w_f32 is not None else w_int
    Ssum = _ref_conv(x, w, case)
    a = torch.tensor(0.37 if a_dev is not None else a_const, dtype=torch.float32, device=DEV)
    sc = (a * n_scale) if n_scale is not None else a.expand(K)
    bs = bias if bias is not None else torch.zeros(K, device=DEV)
    sc4, bs4 = sc.view(1, K, 1, 1), bs.view(1, K, 1, 1)
    if case.ops in ("f32", "pm1"):
        ref = Ssum * sc4.double() + bs4.double()
        Rm = _ref_conv(x.abs(), w.abs(), case) * sc4.double().abs() + bs4.double().abs()
        _bound(got, ref, Rm, C_FWD, f"fwd {case.terms}", MAX_FWD)
    else:
        assert float(Ssum.abs().max()) < 2 ** 24
        S32 = Ssum.float()
        _bits_equal(got, fmaf32(S32, sc4.expand_as(S32), bs4.expand_as(S32)), case.id)


def _dgrad(case, g):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    ta, tw = case.terms
    sh = shape(case.shape)
    P, Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1
    f32 = case.ops == "f32"
    db, wb = _bounds(K // G, R * S, 8, 7)
    dy = torch.randn(B, K, P, Q, generator=g, device=DEV) if f32 else _rand_int((B, K, P, Q), db, g)
    w_scale = None
    if f32 and tw > 1:
        w = torch.randn(K, Cc // G, R, S, generator=g, device=DEV)
        w_img = PK.pack_weight(sh, 1, ta, tw, w_f32=w)
    else:
        w = _rand_int((K, Cc // G, R, S), 127 if f32 else wb, g)
        if f32:     # integer weight levels with their per-channel scale folded into dy, one channel's scale 0 (kzero)
            w_scale = torch.rand(K, generator=g, device=DEV) * 0.02 + 0.001
            w_scale[0] = 0.0
        w_img = PK.pack_weight(sh, 1, ta, tw, w_int=w.to(torch.int16), kzero=w_scale)
    dy_pk, _ = PK.pack_act(dy, None, ta, ch_scale=w_scale, groups=G)
    if w_scale is not None:
        dy = dy * w_scale.view(1, -1, 1, 1)      # the fp32 product is the operand the kernel splits
    gain, const = case.epi["gain"], case.epi.get("const", 1.0)
    c8o = G * (-(-(Cc // G) // 8))
    bits = torch.randint(0, 256, (B, c8o, H, W), generator=g, device=DEV, dtype=torch.uint8) if gain is not None else None
    n = B * Cc * H * W
    out = _nan(n)
    fn = lambda: PK.conv(sh, 1, dy_pk, ta, w_img, tw, out, bits8=bits, gain=gain if gain is not None else 1.0,
                         a_scale_const=const)
    got = _launch_twice(fn, out, n).view(B, Cc, H, W)
    Ssum = _ref_dgrad(dy, w, case)
    mask = None
    if bits is not None:
        cg = Cc // G
        ch = torch.arange(Cc, device=DEV)
        octet = (ch // cg) * (-(-cg // 8)) + (ch % cg) // 8
        bitno = ((ch % cg) % 8).view(1, Cc, 1, 1)
        mask = ((bits.index_select(1, octet).int() >> bitno) & 1).bool()
    if f32:
        mul = gain if mask is not None else const
        ref, Rm = Ssum * mul, _ref_dgrad(dy.abs(), w.abs(), case) * abs(mul)
        if mask is not None:
            ref, Rm = torch.where(mask, ref, torch.zeros_like(ref)), torch.where(mask, Rm, torch.zeros_like(Rm))
        _bound(got, ref, Rm, C_DGRAD, f"dgrad {case.terms}", case.maxnorm)
        return
    assert float(Ssum.abs().max()) < 2 ** 24
    S32 = Ssum.float()
    if mask is None:
        want = fmaf32(S32, torch.full_like(S32, const), torch.zeros_like(S32))
    else:
        want = torch.where(mask, S32 * torch.tensor(gain, dtype=torch.float32, device=DEV), torch.zeros_like(S32))
    _bits_equal(got, want, case.id)


def _wgrad(case, g):
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    ta, tx = case.terms
    sh = shape(case.shape)
    P, Q = (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1
    f32 = case.ops == "f32"
    db, xb = _bounds(B * P * Q, 1, 8, 8)
    dy = torch.randn(B, K, P, Q, generator=g, device=DEV) if f32 else _rand_int((B, K, P, Q), db, g)
    x = torch.randn(B, Cc, H, W, generator=g, device=DEV) if f32 and tx > 1 else _rand_int((B, Cc, H, W), 127 if f32 else xb, g)
    a = torch.tensor([0.37], device=DEV) if case.epi["a_scale"] else None
    kdiv = (torch.rand(K, generator=g, device=DEV) + 0.5) if case.epi["kdiv"] else None
    n = K * (Cc // G) * R * S
    out = _nan(n)
    dy_pk, _ = PK.pack_act(dy, None, ta, groups=G)
    x_pk, _ = PK.pack_act(x, None, tx, phase_split=st == 2, groups=G)
    lib = L.load()
    nbytes = int(lib.mnb_pk_wgrad_scratch_bytes(C.byref(sh), ta, tx))
    assert nbytes >= 0, lib.mnb_last_error()
    scratch = torch.full((nbytes + 16,), 0x5A, dtype=torch.uint8, device=DEV)
    flag = L.tc_err_flag(torch.device(DEV))
    fn = lambda: lib.mnb_pk_wgrad(C.byref(sh), dy_pk.data_ptr(), ta, x_pk.data_ptr(), tx, L.ptr(a), L.ptr(kdiv), out.data_ptr(),
                                  scratch.data_ptr(), flag.data_ptr(), L.stream())
    got = _launch_twice(fn, out, n, scratch).view(K, Cc // G, R, S)
    Ssum = _ref_wgrad(x, dy, case)
    mul = torch.ones(K, device=DEV)
    if a is not None or kdiv is not None:
        av = a if a is not None else torch.ones(1, device=DEV)
        mul = (av / kdiv) if kdiv is not None else av.expand(K)      # fp32 division: RN, as __fdiv_rn
    mul = mul.view(K, 1, 1, 1)
    if f32:
        Rm = _ref_wgrad(x.abs(), dy.abs(), case) * mul.double().abs()
        _bound(got, Ssum * mul.double(), Rm, C_WGRAD, f"wgrad {case.terms}", case.maxnorm)
        return
    assert float(Ssum.abs().max()) < 2 ** 24
    S32 = Ssum.float()
    _bits_equal(got, S32 if a is None and kdiv is None else S32 * mul, case.id)


def _refusal(case):
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = shape(case.shape)
    q_rc, q_text, _ = query(case.mode, sh, case.terms)
    assert q_rc != 0
    buf = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    out = _nan(4096)
    flag = L.tc_err_flag(torch.device(DEV))
    n0 = L.launch_count()
    p, o, e = buf.data_ptr(), out.data_ptr(), flag.data_ptr()
    if case.mode == "wgrad":
        rc = lib.mnb_pk_wgrad(C.byref(sh), p, case.terms[0], p, case.terms[1], None, None, o, p, e, L.stream())
    elif case.mode == "i8":
        rc = lib.mnb_pk_i8_conv(C.byref(sh), p, p, None, None, 1.0, None, o, None, e, L.stream())
    else:
        rc = lib.mnb_pk_conv(C.byref(sh), 0 if case.mode == "fwd" else 1, p, case.terms[0], p, case.terms[1], None, None, 1.0,
                             None, None, 1.0, o, e, L.stream())
    text = lib.mnb_last_error()
    torch.cuda.synchronize()
    assert (rc, text) == (q_rc, q_text), (case.id, rc, text, q_rc, q_text)
    assert L.launch_count() == n0, "a refused launch launched a kernel"
    assert torch.isnan(out).all(), "a refused launch wrote its output"


@pytest.mark.parametrize("case", PC.CASES, ids=lambda c: c.id)
def test_case_against_fp64(case):
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case.id)))
    with env(case.env):            # the knobs change the plan, hence the weight image as well as the launch
        if case.refuse:
            _refusal(case)
        elif case.mode in ("fwd", "i8"):
            _fwd(case, g)
        elif case.mode == "dgrad":
            _dgrad(case, g)
        else:
            _wgrad(case, g)
    torch.cuda.empty_cache()
