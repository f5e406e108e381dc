"""mnb_pk_wgrad_taps (csrc/mnb_pk.cu): weight gradient of the narrow grouped 3x3 layers with all nine taps of a CTA in
registers, against an fp64 convolution of the same operands and against mnb_pk_wgrad, whose result it must reproduce bit
for bit (same accumulation chains, batch splits and reduction order).

Bound: element-wise |dw - ref| <= 2^-14 * R, R = the same weight gradient of |dy| and |x| in fp64 (chains of <= 256 MMAs
between round-to-nearest adds, two bf16 pieces of dy), the bound test_gpu_pk_conv_fp64.py holds mnb_pk_wgrad to.
Results start as NaN, so an element the kernels never write fails."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_WGRAD = 2.0 ** -14

# B, C, H, W, K, pad, groups (3x3, stride 1; 16 input / 32 output channels per group)
G16, G32 = (256, 256, 16, 16, 512, 1, 16), (256, 512, 8, 8, 1024, 1, 32)
CASES = [
    (G16, (2, 1)), (G16, (2, 2)), (G32, (2, 1)), (G32, (2, 2)),                      # the bench layers at batch 256
    ((3, 256, 16, 16, 512, 1, 16), (2, 1)), ((2, 512, 8, 8, 1024, 1, 32), (2, 2)),   # small batches
    ((37, 256, 16, 16, 512, 1, 16), (2, 1)),       # partial last split
    ((5, 64, 4, 4, 128, 1, 4), (2, 1)),            # 4x4 images: several sub-blocks per stage, short last stage; 4 groups
    ((3, 64, 9, 7, 128, 0, 4), (1, 1)),            # 'valid' padding, odd non-square image, one piece each
    ((2, 128, 6, 5, 256, 2, 8), (3, 3)),           # padding 2, three pieces (six piece products)
    ((1, 64, 3, 94, 128, 1, 4), (2, 1)),           # one 96-position raster row per sub-block, two stages
]
IDS = ["g16-b256-t21", "g16-b256-t22", "g32-b256-t21", "g32-b256-t22", "g16-b3", "g32-b2-t22", "g16-b37-partial-split",
       "4x4-g4", "valid-odd", "pad2-t33", "row96"]


def _sh(case):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, pad, G = case
    return L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, pad, pad, 1, 1, G)


def _operands(case, terms, seed, levels):
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, pad, G = case
    g = torch.Generator().manual_seed(seed)
    P, Q = H + 2 * pad - 2, W + 2 * pad - 2
    dy = torch.randn(B, K, P, Q, generator=g).to(DEV)
    t, tx = terms
    if levels:   # integer levels, activation scale and the per-channel factor dy was packed with (the models' layout)
        x = torch.randint(-1, 2, (B, Cc, H, W), generator=g).float().to(DEV)
        a_scale = torch.tensor([0.031], device=DEV)
        kdiv = (torch.rand(K, generator=g) + 0.5).to(DEV)
        dy_pk, _ = PK.pack_act(dy, None, t, ch_scale=kdiv)
        mul = 0.031 / kdiv.double().view(-1, 1, 1, 1)
    else:
        x = torch.randn(B, Cc, H, W, generator=g).to(DEV)
        a_scale, kdiv, mul = None, None, 1.0
        dy_pk, _ = PK.pack_act(dy, None, t)
    x_pk, _ = PK.pack_act(x, None, tx)
    # the operands the kernels multiply: the sums of the pieces in the planes
    xs, dys = _unpack(x_pk, tx, B, Cc, H, W).double(), _unpack(dy_pk, t, B, K, P, Q).double()
    shp = (K, Cc // G, 3, 3)
    ref = torch.nn.grad.conv2d_weight(xs, shp, dys, 1, pad, 1, G) * mul
    Rb = torch.nn.grad.conv2d_weight(xs.abs(), shp, dys.abs(), 1, pad, 1, G) * (mul.abs() if levels else 1.0)
    return dy_pk, x_pk, a_scale, kdiv, ref, Rb


def _run(fn, case, *args, **kw):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, pad, G = case
    dw = torch.full((K, Cc // G, 3, 3), float("nan"), dtype=torch.float32, device=DEV)
    L.check(fn(_sh(case), *args[:2], args[2], *args[3:4], dw, **kw), fn.__name__)
    torch.cuda.synchronize()
    L.tc_check()
    return dw


def _within(got, ref, R, c):
    assert not torch.isnan(got).any(), "outputs the kernel never wrote"
    err = (got.double() - ref).abs()
    ratio = (err / R.clamp_min(1e-300)).max().item()
    assert (err <= c * R).all(), f"worst err / R = {ratio:.3e} > c = {c:.3e}"


@pytest.mark.parametrize("case,terms", CASES, ids=IDS)
@pytest.mark.parametrize("levels", [False, True], ids=["fp32", "levels"])
def test_taps_weight_gradient(case, terms, levels):
    from micronet_b200 import pk as PK
    t, tx = terms
    sh = _sh(case)
    plan = PK.wgrad_taps_plan(sh, t, tx)
    assert plan is not None, "shape outside the cover"
    B, Cc, H, W, K, pad, G = case
    nstg = -(-B * -(-(H + 2 * pad - 2) // plan["TH"]) // plan["NI"])
    if B == 37:
        assert nstg % plan["stg_per_split"] != 0, "the case wants a short last split"
    dy_pk, x_pk, a_scale, kdiv, ref, Rb = _operands(case, terms, 11 + CASES.index((case, terms)), levels)
    kw = dict(a_scale=a_scale, kdiv=kdiv)
    new = _run(PK.wgrad_taps, case, dy_pk, t, x_pk, tx, **kw)
    _within(new, ref, Rb, C_WGRAD)
    again = _run(PK.wgrad_taps, case, dy_pk, t, x_pk, tx, **kw)
    assert torch.equal(new, again), "two runs differ"
    old = _run(PK.wgrad, case, dy_pk, t, x_pk, tx, **kw)
    assert torch.equal(new, old), f"differs from mnb_pk_wgrad by up to {(new - old).abs().max().item():.3e}"


def test_headline_model_step_with_and_without_the_taps_plan():
    """one QAT step of the fused NIN-GC wbwtab W3/A2 model with wgrad_taps_plan forced to refuse every shape and as it is: the
    new kernel runs for exactly the two grouped 3x3 layers, and the loss and every gradient are bit-identical"""
    from harness import train as H
    from micronet_b200 import _lib as L, pk as PK
    from micronet_b200 import functional as F_
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    base = H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w["engine_extra"])
    x, t = H.synthetic_batch(16, w["hw"], seed=5, device=DEV)
    calls = []
    real_taps, real_plan = PK.wgrad_taps, PK.wgrad_taps_plan

    def spy_taps(sh, *args, **kw):
        calls.append((sh.in_c, sh.out_c, sh.groups))
        return real_taps(sh, *args, **kw)

    res = {}
    try:
        PK.wgrad_taps = spy_taps
        for on in (False, True):
            PK.wgrad_taps_plan = real_plan if on else (lambda *a: None)   # wgrad_taps reads it too: only on the old leg
            n_calls = len(calls)
            m = copy.deepcopy(base).to(DEV).train()
            loss = torch.nn.functional.cross_entropy(m(x), t)
            loss.backward()
            torch.cuda.synchronize()
            assert len(calls) - n_calls == (2 if on else 0)
            res[on] = (loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None})
    finally:
        PK.wgrad_taps, PK.wgrad_taps_plan = real_taps, real_plan
    L.tc_check()
    assert sorted(calls) == [(256, 512, 16), (512, 1024, 32)], calls
    assert torch.equal(res[False][0], res[True][0])
    assert res[False][1].keys() == res[True][1].keys()
    for n in res[True][1]:
        assert torch.equal(res[False][1][n], res[True][1][n]), n


def _unpack(planes, terms, B, Cc, H, W):
    c8 = (Cc + 7) // 8
    t = planes.view(torch.bfloat16).view(terms, B, c8, H, W, 8).float().sum(0)
    return t.permute(0, 1, 4, 2, 3).reshape(B, c8 * 8, H, W)[:, :Cc]
