"""Narrow grouped 3x3 convolutions (mnb_pk_gc3_conv / mnb_pk_gc3_conv_codes, pk_gc3_kernel) against fp64 at every case of
tests/gc3_cases.py: every plan feature the query can take, the four bench launches of both NIN-GC workloads at batch 256,
and every refusal.

Every launch goes through the C entry points.  Outputs start as NaN (fp32) or -32768 (codes), the decode pair as NaN; each
output is a view at the front of a larger buffer whose tail holds a sentinel that must survive.  Every launch runs twice
with bitwise-identical results, and the tensor-core error flag must stay clean.

* Forward on integer levels (+-1 x ternary, DoReFa 4-bit, int8 range): the exact sum S (fp64, exact below 2^24).  codes
  = S; the decode pair = (fl(a_scale * n_scale[k]), bias[k]) bit for bit; the fp32 output = fmaf(S, fl(a_scale * n_scale[k]),
  bias[k]) bit for bit (fmaf emulated in fp64, double-rounding midpoints settled by the TwoSum error).
* Data gradient on integer dy (|dy| <= 255 is bf16-exact, so the second piece is 0): exact, so dx = fl(S * a_scale_const)
  or, under the STE mask, fl(S * gain), masked-out positions +0.0, bit for bit.
* Data gradient on real dy (two pieces, w_scale folded into dy, kzero channels): element-wise within 2^-15 R, R the same
  convolution of |dy| and |w| in fp64, and byte-equal to mnb_pk_conv, which pins the order of the MMA chain."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests import gc3_cases as P
from tests.pk_plan_util import fmaf32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TAIL = 64                       # sentinel elements behind every output
F_SENT, I_SENT = -7.25, 0x1234
C_DGRAD = 2.0 ** -15
CODES = {"E_ARG": -1, "E_UNSUPPORTED": -2}


def _guarded(n, dtype, fill, sentinel):
    """(view of n elements filled with ``fill``, whole buffer) - the n + TAIL tail elements hold ``sentinel``"""
    buf = torch.empty(n + TAIL, dtype=dtype, device=DEV)
    buf[:n] = fill
    buf[n:] = sentinel
    return buf[:n], buf


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _tail_ok(buf, n, sentinel):
    t = buf[n:]
    return bool((_bits(t) == _bits(torch.full_like(t, sentinel))).all())


# ---- operands
def _levels(kind, shape_x, shape_w, gen, mode):
    if kind == "pm1":
        x = torch.randint(0, 2, shape_x, generator=gen).float() * 2 - 1
        w = torch.randint(-1, 2, shape_w, generator=gen)
        return x, w, 1
    if kind == "dorefa4":
        x = torch.randint(0, 16, shape_x, generator=gen).float()
        w = torch.randint(0, 16, shape_w, generator=gen) * 2 - 15
        return x, w, 15 * 15
    # int8 range: the fp32 forward takes the full range; codes stay within the int16 bound (113 x 2 <= 227)
    la, lw = (127, 127) if mode == "fwd" else (113, 2)
    x = torch.randint(-la, la + 1, shape_x, generator=gen).float()
    w = torch.randint(-lw, lw + 1, shape_w, generator=gen)
    return x, w, la * lw


def _forward_epilogue(case, K, gen):
    e = case.epi
    n_scale = (torch.rand(K, generator=gen) + 0.5).to(DEV) if e["n_scale"] else None
    bias = torch.randn(K, generator=gen).to(DEV) if e["bias"] else None
    if e["a_scale"] == "tensor":
        a_t = torch.tensor([0.4375 + float(torch.rand(1, generator=gen)) * 0.1], device=DEV)
        a_const, a_f32 = 1.0, a_t
    else:
        a_t, a_const = None, float(e["a_scale"])
        a_f32 = torch.tensor([np.float32(a_const)], device=DEV)
    scv = a_f32.expand(K) * n_scale if n_scale is not None else a_f32.expand(K).clone()     # fp32 product: fl(a * n)
    bsv = bias if bias is not None else torch.zeros(K, device=DEV)
    return n_scale, a_t, a_const, bias, scv.contiguous(), bsv


def _run_twice(launch, outs, what):
    """launch twice into freshly filled outputs; returns the clones of the first run's buffers"""
    from micronet_b200 import _lib as L
    runs = []
    for _ in range(2):
        for view, buf, fill, sent, n in outs:
            view.fill_(fill)
            buf[n:] = sent
        L.check(launch(), what)
        torch.cuda.synchronize()
        runs.append([buf.clone() for _, buf, *_ in outs])
    L.tc_check()
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b)), f"{what}: the second launch differs"
    for (view, buf, fill, sent, n), got in zip(outs, runs[0]):
        assert _tail_ok(got, n, sent), f"{what}: written past the end of the output"
    return [r[:o[4]] for r, o in zip(runs[0], outs)]


def _check_plan(case):
    plan = P.plan_of(case)
    assert isinstance(plan, dict), f"{case.id}: refused {plan}"
    got = {k: plan[k] for k in case.expect}
    assert got == case.expect, f"{case.id}: the plan changed: {got} != {case.expect}"
    return plan


FWD_CASES = [c for c in P.CASES if c.mode in ("fwd", "codes")]
DGRAD_CASES = [c for c in P.CASES if c.mode == "dgrad"]


@pytest.mark.parametrize("case", FWD_CASES, ids=[c.id for c in FWD_CASES])
def test_forward_matches_the_exact_sum(case):
    from micronet_b200 import _lib as L, pk as PK
    _check_plan(case)
    B, Cc, H, W, K, ph, pw, G = case.shape
    OH, OW = P.out_hw(case.shape, case.mode)
    sh = P.conv_shape(case.shape)
    gen = torch.Generator().manual_seed(sum(map(ord, case.id)))
    x, w, bound = _levels(case.operands, (B, Cc, H, W), (K, Cc // G, 3, 3), gen, case.mode)
    x, w = x.to(DEV), w.to(torch.int16).to(DEV)
    n_scale, a_t, a_const, bias, scv, bsv = _forward_epilogue(case, K, gen)
    x_pk, _ = PK.pack_act(x, None, 1)
    w_img = PK.pack_weight(sh, 0, 1, 1, w_int=w)
    S = TF.conv2d(x.double(), w.double(), None, 1, (ph, pw), 1, G)
    assert torch.equal(S, S.round()) and S.abs().max().item() < 2 ** 24
    lib = L.load()
    err = L.tc_err_flag(torch.device(DEV)).data_ptr()
    n = B * K * OH * OW
    if case.mode == "codes":
        dec, dec_buf = _guarded(2 * K, torch.float32, float("nan"), F_SENT)
        assert S.abs().max().item() <= 16 * 9 * bound <= 32767
        codes, codes_buf = _guarded(n, torch.int16, -32768, I_SENT)
        got_codes, got_dec = _run_twice(
            lambda: lib.mnb_pk_gc3_conv_codes(C.byref(sh), x_pk.data_ptr(), 1, w_img.data_ptr(), 1, L.ptr(n_scale),
                                              L.ptr(a_t), a_const, L.ptr(bias), bound, codes.data_ptr(), dec.data_ptr(),
                                              err, L.stream()),
            [(codes, codes_buf, -32768, I_SENT, n), (dec, dec_buf, float("nan"), F_SENT, 2 * K)], case.id)
        bad = (got_codes.view(B, K, OH, OW).long() != S.long()).sum().item()
        assert bad == 0, f"{case.id}: {bad} of {n} codes differ from the exact sum"
    else:
        out, out_buf = _guarded(n, torch.float32, float("nan"), F_SENT)
        (got,) = _run_twice(
            lambda: lib.mnb_pk_gc3_conv(C.byref(sh), 0, x_pk.data_ptr(), 1, w_img.data_ptr(), 1, L.ptr(n_scale), L.ptr(a_t),
                                        a_const, L.ptr(bias), None, 1.0, out.data_ptr(), err, L.stream()),
            [(out, out_buf, float("nan"), F_SENT, n)], case.id)
        stats = {}
        want = fmaf32(S.float(), scv.view(1, -1, 1, 1), bsv.view(1, -1, 1, 1), stats)
        got = got.view(B, K, OH, OW)
        assert not torch.isnan(got).any(), f"{case.id}: output elements never written"
        bad = (_bits(got) != _bits(want)).sum().item()
        assert bad == 0, f"{case.id}: {bad} of {n} outputs differ from fmaf(S, fl(a_scale * n_scale), bias)"
        got_dec = None          # (the decode pair belongs to the codes entry point)
        print(f"{case.id}: fma midpoints settled: {stats.get('midpoints', 0)}")
    if got_dec is not None:
        want_dec = torch.cat([scv, bsv])
        assert torch.equal(_bits(got_dec), _bits(want_dec)), \
            f"{case.id}: decode pair differs in {(_bits(got_dec) != _bits(want_dec)).sum().item()} of {2 * K} elements"


def _dgrad_operands(case, gen):
    B, Cc, H, W, K, ph, pw, G = case.shape
    OH, OW = H + 2 * ph - 2, W + 2 * pw - 2
    w = torch.randint(-3, 4, (K, Cc // G, 3, 3), generator=gen)
    if case.operands == "int":
        dy = torch.randint(-255, 256, (B, K, OH, OW), generator=gen).float()
        w_scale = torch.ones(K)
    else:
        dy = torch.randn(B, K, OH, OW, generator=gen)
        w_scale = torch.rand(K, generator=gen) + 0.5
    w_scale[::7] = 0.0                     # channels whose weights read as zero (kzero)
    return dy.to(DEV), w.to(torch.int16).to(DEV), w_scale.to(DEV)


@pytest.mark.parametrize("case", DGRAD_CASES, ids=[c.id for c in DGRAD_CASES])
def test_data_gradient_matches_fp64(case):
    from micronet_b200 import _lib as L, pk as PK
    _check_plan(case)
    B, Cc, H, W, K, ph, pw, G = case.shape
    sh = P.conv_shape(case.shape)
    gen = torch.Generator().manual_seed(sum(map(ord, case.id)))
    dy, w, w_scale = _dgrad_operands(case, gen)
    dy_pk, _ = PK.pack_act(dy, None, 2, ch_scale=w_scale, groups=G)
    w_img = PK.pack_weight(sh, 1, 2, 1, w_int=w, kzero=w_scale)
    mask = "gain" in case.epi
    gain = float(case.epi.get("gain", 1.0))
    a_const = float(case.epi.get("a_scale", 1.0))
    bits8 = torch.randint(0, 256, (B, (Cc + 7) // 8, H, W), generator=gen).to(torch.uint8).to(DEV) if mask else None
    lib = L.load()
    err = L.tc_err_flag(torch.device(DEV)).data_ptr()
    n = B * Cc * H * W
    out, out_buf = _guarded(n, torch.float32, float("nan"), F_SENT)
    (got,) = _run_twice(
        lambda: lib.mnb_pk_gc3_conv(C.byref(sh), 1, dy_pk.data_ptr(), 2, w_img.data_ptr(), 1, None, None, a_const, None,
                                    L.ptr(bits8), gain, out.data_ptr(), err, L.stream()),
        [(out, out_buf, float("nan"), F_SENT, n)], case.id)
    got = got.view(B, Cc, H, W)
    assert not torch.isnan(got).any(), f"{case.id}: dx elements never written"
    dyf = dy.double() * w_scale.double().view(1, -1, 1, 1)
    D = TF.conv_transpose2d(dyf, w.double(), None, 1, (ph, pw), 0, G)
    keep = None
    if mask:
        c = torch.arange(Cc, device=DEV)
        keep = ((bits8.long()[:, c // 8] >> (c % 8).view(1, -1, 1, 1)) & 1).bool()
    if case.operands == "int":
        assert torch.equal(D, D.round()) and D.abs().max().item() < 2 ** 24
        fac = torch.tensor(np.float32(gain if mask else a_const), device=DEV)
        want = D.float() * fac + 0.0                       # fl(S * factor); + 0.0: the kernel's zero sums are +0
        if mask:
            want = torch.where(keep, want, torch.zeros_like(want))
        bad = (_bits(got) != _bits(want)).sum().item()
        assert bad == 0, f"{case.id}: {bad} of {n} dx elements differ from the exact result"
        if mask:
            assert (_bits(got[~keep]) == 0).all(), "masked-out positions are not +0.0"
        return
    fac = gain if mask else a_const
    R = TF.conv_transpose2d(dyf.abs(), w.double().abs(), None, 1, (ph, pw), 0, G) * fac
    ref = D * fac
    if mask:
        ref = torch.where(keep, ref, torch.zeros_like(ref))
        R = torch.where(keep, R, torch.zeros_like(R))
        assert (_bits(got[~keep]) == 0).all(), "masked-out positions are not +0.0"
    e = (got.double() - ref).abs()
    assert (e <= C_DGRAD * R).all(), f"{case.id}: dx off the fp64 result by more than 2^-15 R"
    ratio = (e / R.clamp_min(1e-300)).max().item() / C_DGRAD
    # the same bits as mnb_pk_conv: the same chain of MMAs in the same order
    old = torch.full((B, Cc, H, W), float("nan"), device=DEV)
    L.check(PK.conv(sh, 1, dy_pk, 2, w_img, 1, old, None, None, a_const, None, bits8, gain), "pk_conv")
    torch.cuda.synchronize()
    L.tc_check()
    diff = (_bits(got) != _bits(old)).sum().item()
    assert diff == 0, f"{case.id}: differs from mnb_pk_conv in {diff} of {n} elements"
    print(f"{case.id}: worst |dx - fp64| / (2^-15 R) = {ratio:.3g}")


@pytest.mark.parametrize("ref", P.REFUSALS, ids=[r.id for r in P.REFUSALS])
def test_refused_launch_writes_nothing(ref, monkeypatch):
    """a refused launch returns the query's code and text (or, past the plan, the launcher's), launches nothing and
    writes nothing"""
    from micronet_b200 import _lib as L, pk as PK
    for k, v in ref.env.items():
        monkeypatch.setenv(k, v)
    PK._plan_cache.clear()
    lib = L.load()
    sh = P.refusal_shape(ref)
    B, Cc, H, W, K, R, S, st, _, ph, pw, dil, _, G = ref.shape
    want = P.query(sh, ref.mode, ref.terms)
    if ref.launch:
        assert isinstance(want, dict), want
        want = (CODES[ref.code], ref.text)
    else:
        assert want == (CODES[ref.code], ref.text), want
    OH, OW = (H + 2 * ph - dil * (R - 1) - 1) // st + 1, (W + 2 * pw - dil * (S - 1) - 1) // st + 1
    if ref.mode == "dgrad":
        a_bytes = lib.mnb_pk_act_bytes(B, K, max(OH, 1), max(OW, 1), 3)
        n_out = B * Cc * H * W
    else:
        a_bytes = lib.mnb_pk_act_bytes(B, Cc, H, W, 3)
        n_out = B * K * max(OH, 1) * max(OW, 1)
    a = torch.zeros(int(a_bytes) + 4096, dtype=torch.uint8, device=DEV)
    wimg = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    vec = torch.ones(max(K, Cc) + 64, device=DEV)
    err = L.tc_err_flag(torch.device(DEV)).data_ptr()
    a_ptr = a.data_ptr() + (4 if ref.launch == "unaligned_a" else 0)
    off = 1 if ref.launch == "unaligned_out" else 0        # one element: 4 (fp32) or 2 (int16) bytes off
    n0 = L.launch_count()
    if ref.mode == "codes":
        out, buf = _guarded(n_out + 1, torch.int16, -32768, I_SENT)
        bound = P.CODES_BOUND_REFUSED if ref.launch == "codes_bound" else 1
        dec, dec_buf = _guarded(2 * K, torch.float32, float("nan"), F_SENT)
        rc = lib.mnb_pk_gc3_conv_codes(C.byref(sh), a_ptr, ref.terms[0], wimg.data_ptr(), ref.terms[1], vec.data_ptr(), None,
                                       1.0, vec.data_ptr(), bound, out[off:].data_ptr(), dec.data_ptr(), err, L.stream())
    else:
        out, buf = _guarded(n_out + 1, torch.float32, float("nan"), F_SENT)
        dec = dec_buf = None
        mode = 1 if ref.mode == "dgrad" else 0
        rc = lib.mnb_pk_gc3_conv(C.byref(sh), mode, a_ptr, ref.terms[0], wimg.data_ptr(), ref.terms[1],
                                 vec.data_ptr() if mode == 0 else None, None, 1.0, vec.data_ptr() if mode == 0 else None,
                                 None, 1.0, out[off:].data_ptr(), err, L.stream())
    text = lib.mnb_last_error().decode(errors="replace")
    torch.cuda.synchronize()
    assert (rc, text) == want and L.launch_count() == n0, (rc, text, want)
    if out.dtype == torch.int16:
        assert (out == -32768).all() and _tail_ok(buf, n_out + 1, I_SENT), "refused, yet codes were written"
        assert torch.isnan(dec).all() and _tail_ok(dec_buf, 2 * K, F_SENT), "refused, yet the decode pair was written"
    else:
        assert torch.isnan(out).all() and _tail_ok(buf, n_out + 1, F_SENT), "refused, yet the output was written"
    L.tc_check()


@pytest.mark.parametrize("fuse", [True, False], ids=["fused", "unfused"])
def test_dorefa_w4a4_step_runs_gc3_and_matches_the_other_kernels(fuse):
    """one QAT step of the bench DoReFa W4A4 NIN-GC model (fused producers, and un-fused): both grouped 3x3 layers run the
    gc3 forward (a_scale_const 1/15), the gc3 data gradient (the STE mask with the gain 0.1) and the taps weight gradient,
    and the loss and every gradient are bit-identical to the step with MNB_PK_GC3 / MNB_PK_WG_TAPS off"""
    from harness import train as H
    from micronet_b200 import _lib as L, pk as PK
    w = H.WORKLOADS["nin_gc_dorefa_w4a4"]
    extra = dict(w["engine_extra"], fuse=fuse)
    base = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **extra)
    x, t = H.synthetic_batch(8, w["hw"], seed=11, device=DEV)
    calls = []
    real = (PK.gc3_conv, PK.gc3_conv_codes, PK.wgrad_taps)

    def spy_conv(sh, mode, *args, **kw):
        calls.append((sh.in_c, sh.groups, "fwd" if mode == 0 else "dgrad", kw.get("bits8") is not None,
                      float(kw.get("a_scale_const", 1.0)), float(kw.get("gain", 1.0))))
        return real[0](sh, mode, *args, **kw)

    def spy_codes(sh, *args, **kw):
        calls.append((sh.in_c, sh.groups, "codes", False, 0.0, 0.0))
        return real[1](sh, *args, **kw)

    def spy_taps(sh, *args, **kw):
        calls.append((sh.in_c, sh.groups, "wgrad_taps", False, 0.0, 0.0))
        return real[2](sh, *args, **kw)

    res = {}
    saved = (L.PK_GC3, L.PK_WG_TAPS)
    try:
        PK.gc3_conv, PK.gc3_conv_codes, PK.wgrad_taps = spy_conv, spy_codes, spy_taps
        for on in (False, True):
            L.PK_GC3 = L.PK_WG_TAPS = on
            n_calls = len(calls)
            m = copy.deepcopy(base).to(DEV).train()
            loss = torch.nn.functional.cross_entropy(m(x), t)
            loss.backward()
            torch.cuda.synchronize()
            if not on:
                assert len(calls) == n_calls, calls[n_calls:]
            res[on] = (loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    finally:
        L.PK_GC3, L.PK_WG_TAPS = saved
        PK.gc3_conv, PK.gc3_conv_codes, PK.wgrad_taps = real
    L.tc_check()
    # (mask, a_scale_const, gain) of a data gradient: a max-pool sits between each grouped layer and the BatchNorm + ReLU +
    # quantizer in front of it, so even the fused model packs the layer's input in the conv and keeps the STE mask bits8 with
    # the gain 0.1 (a fused producer owning the mask would hand over a_scale_const = 0.1 and no mask)
    forms = {(True, 1.0, 0.1)}
    got = sorted((c, g, k, m, round(a, 7), round(gn, 7)) for c, g, k, m, a, gn in calls)
    layers = ((256, 16), (512, 32))
    assert sorted(x[:3] for x in got) == sorted((c, g, k) for c, g in layers for k in ("fwd", "dgrad", "wgrad_taps")), got
    for c, g, k, m, a, gn in got:
        if k == "fwd":
            assert (m, a, gn) == (False, round(1.0 / 15, 7), 1.0), (c, g, k, m, a, gn)
        elif k == "dgrad":
            assert (m, a, gn) in {(x, round(y, 7), round(z, 7)) for x, y, z in forms}, (c, g, k, m, a, gn)
    print(f"{'fused' if fuse else 'unfused'}: gc3 launches {got}")
    assert torch.equal(res[False][0], res[True][0])
    assert res[False][1].keys() == res[True][1].keys()
    for n in res[True][1]:
        assert torch.equal(res[False][1][n], res[True][1][n]), n
