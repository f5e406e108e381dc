"""mnb_pk_gc3_conv / mnb_pk_gc3_conv_codes (csrc/mnb_pk.cu): forward and data gradient of the narrow grouped 3x3 layers with
whole images as M tiles, against mnb_pk_conv / mnb_pk_conv_codes, whose results they must reproduce byte for byte: the
forward sums are exact integers, and every data-gradient element sees the same chain of MMAs as in mnb_pk_conv's plan.
Outputs start as NaN (codes as -32768, which no sum of 144 terms +-1 x level 1 reaches), so an element the kernels never
write fails."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# B, C, H, W, K, pad, groups (3x3, stride 1; 16 input / 32 output channels per group)
CASES = [
    (256, 256, 16, 16, 512, 1, 16), (256, 512, 8, 8, 1024, 1, 32),   # the bench layers at batch 256
    (3, 256, 16, 16, 512, 1, 16), (2, 512, 8, 8, 1024, 1, 32),       # small batches
    (5, 512, 8, 8, 1024, 1, 32),                                      # short last image tile
    (3, 256, 16, 16, 512, 0, 16),                                     # 'valid' padding, short last tile
    (4, 128, 7, 9, 256, 2, 8),                                        # padding 2, odd non-square image, 8 groups
]
IDS = ["g16-b256", "g32-b256", "g16-b3", "g32-b2", "g32-b5-short", "g16-pad0", "pad2-odd"]


def _sh(case):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, pad, G = case
    return L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, pad, pad, 1, 1, G)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f"{what}: differs from mnb_pk_conv in {(_bits(a) != _bits(b)).sum().item()} elements"


def _check(fn, *args):
    from micronet_b200 import _lib as L
    L.check(fn(*args), fn.__name__)
    torch.cuda.synchronize()
    L.tc_check()


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_forward_codes_and_fp32(case):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, pad, G = case
    sh = _sh(case)
    assert PK.gc3_plan(sh, 0, 1, 1) is not None, "shape outside the cover"
    P, Q = H + 2 * pad - 2, W + 2 * pad - 2
    g = torch.Generator().manual_seed(3 + CASES.index(case))
    x = torch.randint(0, 2, (B, Cc, H, W), generator=g).float().mul_(2).sub_(1).to(DEV)
    w = torch.randint(-1, 2, (K, Cc // G, 3, 3), generator=g).to(torch.int16).to(DEV)
    n_scale = (torch.rand(K, generator=g) + 0.5).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    a_scale = torch.tensor([0.37], device=DEV)
    x_pk, _ = PK.pack_act(x, None, 1)
    w_img = PK.pack_weight(sh, 0, 1, 1, w_int=w)
    res = {}
    for name, fn in (("old", PK.conv_codes), ("new", PK.gc3_conv_codes), ("again", PK.gc3_conv_codes)):
        codes = torch.full((B, K, P, Q), -32768, dtype=torch.int16, device=DEV)
        dec = torch.full((2 * K,), float("nan"), device=DEV)
        _check(fn, sh, x_pk, w_img, codes, dec, n_scale, a_scale, 1.0, bias)
        res[name] = (codes, dec)
    assert (res["old"][0] != -32768).all()
    for name in ("new", "again"):
        _same(res[name][0], res["old"][0], f"codes ({name})")
        _same(res[name][1], res["old"][1], f"decode pair ({name})")
    # the fp32 form: with and without the per-channel scale / bias, the activation scale as a constant
    for kw in (dict(n_scale=n_scale, a_scale=a_scale, bias=bias), dict(a_scale_const=0.25)):
        outs = {}
        for name, fn in (("old", PK.conv), ("new", PK.gc3_conv), ("again", PK.gc3_conv)):
            y = torch.full((B, K, P, Q), float("nan"), device=DEV)
            _check(fn, sh, 0, x_pk, 1, w_img, 1, y, *[kw.get(k) for k in ("n_scale", "a_scale")], kw.get("a_scale_const", 1.0),
                   kw.get("bias"))
            outs[name] = y
        assert not torch.isnan(outs["old"]).any()
        _same(outs["new"], outs["old"], "fp32 forward")
        _same(outs["again"], outs["old"], "fp32 forward (second run)")


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("mask", [False, True], ids=["plain", "ste-mask"])
def test_data_gradient(case, mask):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, pad, G = case
    sh = _sh(case)
    assert PK.gc3_plan(sh, 1, 2, 1) is not None, "shape outside the cover"
    P, Q = H + 2 * pad - 2, W + 2 * pad - 2
    g = torch.Generator().manual_seed(41 + CASES.index(case))
    dy = torch.randn(B, K, P, Q, generator=g).to(DEV)
    w = torch.randint(-3, 4, (K, Cc // G, 3, 3), generator=g).to(torch.int16).to(DEV)
    w_scale = (torch.rand(K, generator=g) + 0.5).to(DEV)
    w_scale[::7] = 0.0                        # channels whose weights read as zero (kzero)
    dy_pk, _ = PK.pack_act(dy, None, 2, ch_scale=w_scale)
    w_img = PK.pack_weight(sh, 1, 2, 1, w_int=w, kzero=w_scale)
    bits8 = torch.randint(0, 256, (B, (Cc + 7) // 8, H, W), generator=g).to(torch.uint8).to(DEV) if mask else None
    outs = {}
    for name, fn in (("old", PK.conv), ("new", PK.gc3_conv), ("again", PK.gc3_conv)):
        dx = torch.full((B, Cc, H, W), float("nan"), device=DEV)
        _check(fn, sh, 1, dy_pk, 2, w_img, 1, dx, None, None, 0.1 if not mask else 1.0, None, bits8, 0.1)
        outs[name] = dx
    assert not torch.isnan(outs["old"]).any()
    _same(outs["new"], outs["old"], "data gradient")
    _same(outs["again"], outs["old"], "data gradient (second run)")


def test_headline_model_step_with_and_without_the_gc3_plan():
    """one QAT step of the fused NIN-GC wbwtab W3/A2 model with gc3_plan forced to refuse every shape and as it is: the new
    kernels run for exactly the forward and the data gradient of the two grouped 3x3 layers, and the loss and every gradient
    are bit-identical"""
    from harness import train as H
    from micronet_b200 import _lib as L, pk as PK
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    base = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w["engine_extra"])
    x, t = H.synthetic_batch(16, w["hw"], seed=5, device=DEV)
    calls = []
    real = (PK.gc3_conv, PK.gc3_conv_codes, PK.gc3_plan)

    def spy_conv(sh, mode, *args, **kw):
        calls.append((sh.in_c, sh.out_c, sh.groups, "fwd" if mode == 0 else "dgrad"))
        return real[0](sh, mode, *args, **kw)

    def spy_codes(sh, *args, **kw):
        calls.append((sh.in_c, sh.out_c, sh.groups, "fwd"))
        return real[1](sh, *args, **kw)

    res = {}
    try:
        PK.gc3_conv, PK.gc3_conv_codes = spy_conv, spy_codes
        for on in (False, True):
            PK.gc3_plan = real[2] if on else (lambda *a: None)
            n_calls = len(calls)
            m = copy.deepcopy(base).to(DEV).train()
            loss = torch.nn.functional.cross_entropy(m(x), t)
            loss.backward()
            torch.cuda.synchronize()
            assert len(calls) - n_calls == (4 if on else 0)
            res[on] = (loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    finally:
        PK.gc3_conv, PK.gc3_conv_codes, PK.gc3_plan = real
    L.tc_check()
    assert sorted(calls) == [(256, 512, 16, "dgrad"), (256, 512, 16, "fwd"), (512, 1024, 32, "dgrad"),
                             (512, 1024, 32, "fwd")], calls
    assert torch.equal(res[False][0], res[True][0])
    assert res[False][1].keys() == res[True][1].keys()
    for n in res[True][1]:
        assert torch.equal(res[False][1][n], res[True][1][n]), n


def test_refused_gc3_launches_fall_back_to_mnb_pk_conv():
    """a shape the plan covers but whose launch mnb_pk_gc3_conv* refuses (MNB_E_UNSUPPORTED, e.g. an unaligned tensor) runs on
    mnb_pk_conv / mnb_pk_conv_codes instead: the step still takes the packed-operand path and gives the same loss and
    gradients as with gc3_plan forced to refuse every shape"""
    from harness import train as H
    from micronet_b200 import _lib as L, pk as PK
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    base = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w["engine_extra"])
    x, t = H.synthetic_batch(8, w["hw"], seed=9, device=DEV)
    real = (PK.gc3_conv, PK.gc3_conv_codes, PK.conv, PK.conv_codes, PK.gc3_plan)
    refused, old_calls = [], []

    def refuse(sh, *args, **kw):
        refused.append((sh.in_c, sh.groups))
        return L.E_UNSUPPORTED

    def count_conv(sh, *args, **kw):
        old_calls.append((sh.in_c, sh.groups))
        return real[2](sh, *args, **kw)

    def count_codes(sh, *args, **kw):
        old_calls.append((sh.in_c, sh.groups))
        return real[3](sh, *args, **kw)

    res = {}
    try:
        PK.conv, PK.conv_codes = count_conv, count_codes
        for on in (False, True):
            PK.gc3_plan = real[4] if on else (lambda *a: None)
            PK.gc3_conv, PK.gc3_conv_codes = (refuse, refuse) if on else real[:2]
            n_old = len(old_calls)
            m = copy.deepcopy(base).to(DEV).train()
            loss = torch.nn.functional.cross_entropy(m(x), t)
            loss.backward()
            torch.cuda.synchronize()
            res[on] = (loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None},
                       sorted(old_calls[n_old:]))
    finally:
        PK.gc3_conv, PK.gc3_conv_codes, PK.conv, PK.conv_codes, PK.gc3_plan = real
    L.tc_check()
    assert sorted(set(refused)) == [(256, 16), (512, 32)] and len(refused) == 4, refused
    assert res[True][2] == res[False][2], "the refused launches did not all run on mnb_pk_conv"
    assert torch.equal(res[False][0], res[True][0])
    for n in res[True][1]:
        assert torch.equal(res[False][1][n], res[True][1][n]), n
