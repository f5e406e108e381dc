"""mnb_pk_bwd1x1 (csrc/mnb_pk.cu): data and weight gradient of a 1x1 grouped convolution in one pass over dy, against
mnb_pk_conv (data gradient) followed by mnb_pk_wgrad on the same operands, whose results it must reproduce byte for byte
(every accumulator sees the same chain of MMAs, the batch splits are reduced in the same order).

Every case runs twice, once into outputs filled with NaN and once into outputs filled with 0x5A bytes, so an element the
kernel never writes fails either way."""
import copy

import pytest
import torch

from tests.pk_conv_bench_launches import BENCH_LAUNCHES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bench_cases():
    """the 1x1 layers of the bench launches the fused kernel covers, with their piece counts (dy, x); weights: one piece"""
    from micronet_b200 import _lib as L, pk as PK
    out = []
    for _, kind, f, _, t_dy, t_x in BENCH_LAUNCHES:
        if kind != "wgrad" or f[5] != 1:
            continue
        case = (f[0], f[1], f[2], f[3], f[4], f[-1])
        if PK.bwd1x1_plan(L.ConvShape(*f), t_dy, t_x, 1) is not None and (case, (t_dy, t_x, 1)) not in out:
            out.append((case, (t_dy, t_x, 1)))
    return out


# B, C, H, W, K, groups (1x1, stride 1, no padding)
SYNTH = [
    ((4, 128, 32, 32, 128, 1), (2, 1, 1)),        # G = 1
    ((6, 256, 16, 16, 256, 2), (2, 1, 1)),        # G = 2
    ((5, 512, 8, 8, 512, 4), (1, 2, 2)),          # G = 4, two x and two weight pieces
    ((3, 1024, 8, 8, 1024, 8), (2, 1, 3)),        # G = 8, three weight pieces
    ((3, 64, 16, 16, 64, 1), (2, 2, 3)),          # cin_g 64, two x pieces
    ((37, 256, 32, 32, 256, 2), (2, 1, 1)),       # short last split
    ((9, 32, 8, 8, 128, 1), (1, 1, 1)),           # cin_g 32: two sub-blocks per stage, short last stage
    ((7, 256, 11, 16, 256, 2), (2, 1, 1)),        # 11 rows: partial last sub-block
    ((5, 256, 32, 32, 128, 2), (2, 1, 1)),        # cin_g 128, cout_g 64
    ((4, 128, 16, 16, 256, 2), (2, 1, 1)),        # cin_g 64, cout_g 128
    ((4, 32, 16, 16, 128, 1), (3, 1, 2)),         # cin_g 32, cout_g 128, three dy pieces
    ((3, 192, 8, 8, 96, 2), (1, 1, 1)),           # cin_g 96, cout_g 48, one piece each
]
SYNTH_IDS = ["g1", "g2", "g4-t122", "g8-t213", "cin64-t223", "short-split", "short-stage", "partial-sub", "cin128-cout64",
             "cin64-cout128", "cin32-cout128-t312", "cin96-cout48-t1"]


def _sh(case):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, G = case
    return L.ConvShape(B, Cc, H, W, K, 1, 1, 1, 1, 0, 0, 1, 1, G)


def _operands(case, terms, seed, mask, levels):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, G = case
    t, tx, tw = terms
    g = torch.Generator().manual_seed(seed)
    dy = torch.randn(B, K, H, W, generator=g).to(DEV)
    if levels:   # the wbwtab layers: ternary levels with per-channel scale folded into dy, divided out of dW
        w_int = torch.randint(-1, 2, (K, Cc // G, 1, 1), generator=g).to(torch.int16).to(DEV)
        w_scale = (torch.rand(K, generator=g) + 0.5).to(DEV)
        dy_pk, _ = PK.pack_act(dy, None, t, ch_scale=w_scale, groups=G)
        w_img = PK.pack_weight(_sh(case), 1, t, tw, w_int=w_int, kzero=w_scale)
        x = torch.randint(-1, 2, (B, Cc, H, W), generator=g).float().to(DEV)
        a_scale, kdiv = torch.tensor([0.031], device=DEV), w_scale
    else:
        wq = torch.randn(K, Cc // G, 1, 1, generator=g).to(DEV)
        dy_pk, _ = PK.pack_act(dy, None, t, groups=G)
        w_img = PK.pack_weight(_sh(case), 1, t, tw, w_f32=wq)
        x = torch.randn(B, Cc, H, W, generator=g).to(DEV)
        a_scale, kdiv = None, None
    x_pk, _ = PK.pack_act(x, None, tx, groups=G)
    bits8 = torch.randint(0, 256, (B, (Cc + 7) // 8, H, W), generator=g).to(torch.uint8).to(DEV) if mask else None
    return dy_pk, x_pk, w_img, bits8, a_scale, kdiv


def _outputs(case, fill):
    B, Cc, H, W, K, G = case
    dx = torch.empty((B, Cc, H, W), device=DEV)
    dw = torch.empty((K, Cc // G, 1, 1), device=DEV)
    for o in (dx, dw):
        if fill == "nan":
            o.fill_(float("nan"))
        else:
            o.view(torch.uint8).fill_(0x5A)
    return dx, dw


def _check(case, terms, seed, mask, levels):
    from micronet_b200 import _lib as L, pk as PK
    sh = _sh(case)
    t, tx, tw = terms
    assert PK.bwd1x1_plan(sh, t, tx, tw) is not None, "shape outside the cover"
    dy_pk, x_pk, w_img, bits8, a_scale, kdiv = _operands(case, terms, seed, mask, levels)
    epi = dict(bits8=bits8, gain=0.1 if mask else 1.0, a_scale_const=1.0 if mask else 0.25)
    ref_dx, ref_dw = _outputs(case, "nan")
    L.check(PK.conv(sh, 1, dy_pk, t, w_img, tw, ref_dx, **epi), "pk_conv dgrad")
    L.check(PK.wgrad(sh, dy_pk, t, x_pk, tx, ref_dw, a_scale=a_scale, kdiv=kdiv), "pk_wgrad")
    torch.cuda.synchronize()
    L.tc_check()
    assert not torch.isnan(ref_dx).any() and not torch.isnan(ref_dw).any()
    for fill in ("nan", "5a"):
        dx, dw = _outputs(case, fill)
        L.check(PK.bwd1x1(sh, dy_pk, t, x_pk, tx, w_img, tw, dx, dw, a_scale=a_scale, kdiv=kdiv, **epi), "pk_bwd1x1")
        torch.cuda.synchronize()
        L.tc_check()
        assert torch.equal(dx.view(torch.int32), ref_dx.view(torch.int32)), f"dx differs ({fill})"
        assert torch.equal(dw.view(torch.int32), ref_dw.view(torch.int32)), f"dW differs ({fill})"


@pytest.mark.parametrize("mask", [False, True], ids=["plain", "ste"])
def test_bench_layers(mask):
    cases = _bench_cases()
    assert {(c[1], c[2], c[-1]) for c, _ in cases} == {(256, 32, 2), (512, 16, 4), (1024, 8, 8)}
    for i, (case, terms) in enumerate(cases):
        _check(case, terms, 100 + i, mask, levels=True)


@pytest.mark.parametrize("case,terms", SYNTH, ids=SYNTH_IDS)
@pytest.mark.parametrize("mask", [False, True], ids=["plain", "ste"])
def test_synthetic(case, terms, mask):
    from micronet_b200 import pk as PK
    plan = PK.bwd1x1_plan(_sh(case), *terms)
    B, Cc, H, W, K, G = case
    if B == 37:
        assert plan["nstg_total"] % plan["stg_per_split"] != 0, "the case wants a short last split"
    if B == 9:
        assert plan["NI"] > 1 and plan["nsub"] % plan["NI"] != 0, "the case wants a short last stage"
    if B == 7:
        assert H % plan["TH"] != 0, "the case wants a partial last sub-block"
    _check(case, terms, 7 + SYNTH.index((case, terms)), mask, levels=terms[2] == 1)


def test_headline_model_step_fused_and_separate():
    """one QAT step of the fused NIN-GC wbwtab W3/A2 model with MNB_PK_BWD1X1=0 and =1: the fused kernel runs for exactly
    the five 1x1 grouped layers, and the loss and every gradient are bit-identical"""
    from harness import train as H
    from micronet_b200 import _lib as L, pk as PK
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    base = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w["engine_extra"])
    x, t = H.synthetic_batch(16, w["hw"], seed=5, device=DEV)
    calls = []
    real = PK.bwd1x1

    def spy(sh, *args, **kw):
        calls.append((sh.in_c, sh.out_c, sh.groups))
        return real(sh, *args, **kw)

    res = {}
    saved = L.PK_BWD1X1
    try:
        PK.bwd1x1 = spy
        for on in (False, True):
            L.PK_BWD1X1 = on
            n_calls = len(calls)
            m = copy.deepcopy(base).to(DEV).train()
            loss = torch.nn.functional.cross_entropy(m(x), t)
            loss.backward()
            torch.cuda.synchronize()
            assert len(calls) - n_calls == (5 if on else 0)
            res[on] = (loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    finally:
        L.PK_BWD1X1, PK.bwd1x1 = saved, real
    L.tc_check()
    assert sorted(calls) == sorted([(256, 256, 2)] * 2 + [(512, 512, 4)] * 2 + [(1024, 1024, 8)]), calls
    assert torch.equal(res[False][0], res[True][0])
    assert res[False][1].keys() == res[True][1].keys()
    for n in res[True][1]:
        assert torch.equal(res[False][1][n], res[True][1][n]), n
