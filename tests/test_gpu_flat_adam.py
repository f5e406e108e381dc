"""mnb_adam_step (micronet_b200.FlatAdam) element by element against an fp64 evaluation of torch.optim.Adam's formulas,
started from the same fp32 state, at bucket sizes around the launcher's grid cap (132 * 8 blocks of 256 threads = 270,336
threads: larger buckets run the grid-stride loop more than once) and at the bench models' bucket sizes.

Error bound (first order, u = 2^-24), from the kernel's operations; the hyper-parameters reach it as fp32, so their
rounding counts too (e1 / e2 = relative error of 1 - fp32(beta1) / 1 - fp32(beta2) against the exact 1 - beta, eb = that of
fp32(beta2), ebc1 / ebc2 = that of the bias corrections bc = 1 - fp32(beta)^step, which mnb_adam_step computes from the
fp32 betas it is given while torch uses the Python floats: at step 2 with beta2 = 0.999, ebc2 = 1.3e-5, about 216 u).
nvcc may contract a multiply and an add into one FMA: that drops a rounding, the bound holds either way.
  g' = fma(wd, p, g)                        Eg = u (|g'| + 2 wd |p|)
  m' = m + (g' - m)(1 - b1)                 Em = u |m'| + (1 - b1)((|g'| + |m|)(2u + e1) + Eg)
  v' = fma(1 - b2, g' g', v b2)             Ev = u v' + (1 - b2)(g'^2 (2u + e2) + 2 |g'| Eg) + b2 v (2u + eb)
  d  = sqrt(v') / fp32(sqrt(bc2)) + eps     Ed = dsqrt + sqrt(v') / sqrt(bc2) (3u + ebc2 / 2) + eps u + u d,
                                            dsqrt = min(Ev / sqrt(v'), sqrt(Ev)) / sqrt(bc2)
  r  = m' / d                               Er = u |r| + Em / d + |r| Ed / d
  p' = p - (lr / bc1) r                     Ep = u |p'| + (lr / bc1)((4u + ebc1) |r| + Er)   (lr, bc1 rounded, a division, a product)
with every quantity on the right taken from the fp64 evaluation."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
GRID_THREADS = 132 * 8 * 256


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _adam64(p, g, m, v, lr, b1, b2, eps, wd, step):
    """torch.optim.Adam (foreach=False, no amsgrad) in fp64 from the fp32 state; returns (p, m, v) and their bounds"""
    p, g, m, v = (t.double() for t in (p, g, m, v))
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    gg = g + wd * p if wd else g
    m1 = m + (gg - m) * (1 - b1)
    v1 = v * b2 + (1 - b2) * gg * gg
    sbc2 = bc2 ** 0.5
    d = v1.sqrt() / sbc2 + eps
    r = m1 / d
    p1 = p - (lr / bc1) * r
    e1 = abs((1 - _f32(b1)) - (1 - b1)) / (1 - b1)
    e2 = abs((1 - _f32(b2)) - (1 - b2)) / (1 - b2)
    eb = abs(_f32(b2) - b2) / b2
    ebc1 = abs((1 - _f32(b1) ** step) - bc1) / bc1     # the launcher's bias corrections start from fp32(beta)
    ebc2 = abs((1 - _f32(b2) ** step) - bc2) / bc2
    Eg = U * (gg.abs() + 2 * wd * p.abs())
    Em = U * m1.abs() + (1 - b1) * ((gg.abs() + m.abs()) * (2 * U + e1) + Eg)
    Ev = U * v1 + (1 - b2) * (gg * gg * (2 * U + e2) + 2 * gg.abs() * Eg) + b2 * v * (2 * U + eb)
    dsqrt = torch.minimum(Ev / v1.sqrt().clamp_min(1e-300), Ev.sqrt()) / sbc2
    Ed = dsqrt + v1.sqrt() / sbc2 * (3 * U + ebc2 / 2) + eps * U + U * d
    Er = U * r.abs() + Em / d + r.abs() * Ed / d
    Ep = U * p1.abs() + (lr / bc1) * ((4 * U + ebc1) * r.abs() + Er)
    return (p1, m1, v1), (Ep, Em, Ev)


def _launch(p, g, m, v, lr, b1, b2, eps, wd, step):
    from micronet_b200 import _lib as L
    L.check(L.load().mnb_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr, b1, b2, eps, wd,
                                   step, L.stream()), "adam_step")


def _state(n, gen, grad_scale=1.0, step=1):
    p = torch.randn(n, generator=gen) * 0.1
    g = torch.randn(n, generator=gen) * grad_scale
    g[torch.rand(n, generator=gen) < 0.1] = 0.0
    if step == 1:
        m, v = torch.zeros(n), torch.zeros(n)
    else:
        m = torch.randn(n, generator=gen) * grad_scale * 0.3
        v = torch.rand(n, generator=gen) * grad_scale ** 2
    return [t.to(DEV) for t in (p, g, m, v)]


def _check(got, ref, bound, what):
    worst = ((got.double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
    print(f"{what}: worst err / bound = {worst:.3f}")
    assert torch.isfinite(got).all(), what
    assert ((got.double() - ref).abs() <= bound).all(), f"{what}: worst err / bound = {worst:.3f}"


SIZES = [1, 255, 257, GRID_THREADS - 1, GRID_THREADS, GRID_THREADS + 1, 591_390, 969_822]


@pytest.mark.parametrize("wd", [0.0, 1e-5])
@pytest.mark.parametrize("step", [1, 2, 10_000])
@pytest.mark.parametrize("n", SIZES)
def test_adam_step_against_fp64(n, step, wd):
    gen = torch.Generator().manual_seed(n * 7 + step)
    lr, b1, b2, eps = 0.01, 0.9, 0.999, 1e-8
    p, g, m, v = _state(n, gen, step=step)
    (p64, m64, v64), (Ep, Em, Ev) = _adam64(p, g, m, v, lr, b1, b2, eps, wd, step)
    p0 = p.clone()
    _launch(p, g, m, v, lr, b1, b2, eps, wd, step)
    torch.cuda.synchronize()
    _check(m, m64, Em, f"n={n} step={step} wd={wd} exp_avg")
    _check(v, v64, Ev, f"n={n} step={step} wd={wd} exp_avg_sq")
    _check(p, p64, Ep, f"n={n} step={step} wd={wd} param")
    # every element the fp64 step moves by more than two units in the last place moved, the tail of the bucket (second
    # pass of the grid-stride loop) included
    must = (p64 - p0.double()).abs() > p0.double().abs() * 4 * U
    assert must[GRID_THREADS - 1:].any() or n <= GRID_THREADS
    assert (p != p0)[must].all()


@pytest.mark.parametrize("step", [1, 2, 10_000])
def test_tiny_gradients_against_fp64(step):
    """|g| ~ 1e-12: sqrt(v) is far below eps"""
    n = GRID_THREADS + 4097
    gen = torch.Generator().manual_seed(step)
    p, g, m, v = _state(n, gen, grad_scale=1e-12, step=step)
    (p64, m64, v64), (Ep, Em, Ev) = _adam64(p, g, m, v, 0.01, 0.9, 0.999, 1e-8, 0.0, step)
    _launch(p, g, m, v, 0.01, 0.9, 0.999, 1e-8, 0.0, step)
    torch.cuda.synchronize()
    assert (v64.sqrt() < 1e-3 * 1e-8).all()
    _check(m, m64, Em, f"tiny step={step} exp_avg")
    _check(v, v64, Ev, f"tiny step={step} exp_avg_sq")
    _check(p, p64, Ep, f"tiny step={step} param")


def test_zero_state_keeps_parameters_bitwise():
    n = GRID_THREADS + 1000
    p = torch.randn(n, device=DEV)
    p0 = p.clone()
    g, m, v = (torch.zeros(n, device=DEV) for _ in range(3))
    for step in (1, 2, 10_000):
        _launch(p, g, m, v, 0.01, 0.9, 0.999, 1e-8, 0.0, step)
    torch.cuda.synchronize()
    assert torch.equal(p.view(torch.int32), p0.view(torch.int32))
    assert not m.any() and not v.any()


def test_empty_bucket_launches_nothing():
    from micronet_b200 import _lib as L
    t = torch.zeros(1, device=DEV)
    before = L.launch_count()
    assert L.load().mnb_adam_step(t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), 0, 0.01, 0.9, 0.999, 1e-8, 0.0, 1,
                                  L.stream()) == 0
    assert L.launch_count() == before


@pytest.mark.parametrize("step", [1, 3])
def test_non_finite_gradients_like_torch(step):
    """NaN / +-Inf gradients: exactly the elements torch.optim.Adam(foreach=False) makes non-finite become non-finite"""
    n = GRID_THREADS + 777
    gen = torch.Generator().manual_seed(17 + step)
    p, g, m, v = _state(n, gen, step=step)
    idx = torch.randperm(n, generator=gen)[:300].to(DEV)
    g[idx[:100]] = float("nan")
    g[idx[100:200]] = float("inf")
    g[idx[200:]] = float("-inf")
    tp = p.clone().requires_grad_(True)
    tp.grad = g.clone()
    opt = torch.optim.Adam([tp], lr=0.01, weight_decay=1e-5, foreach=False)
    opt.state[tp] = {"step": torch.tensor(float(step - 1)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    opt.step()
    _launch(p, g, m, v, 0.01, 0.9, 0.999, 1e-8, 1e-5, step)
    torch.cuda.synchronize()
    st = opt.state[tp]
    for name, a, b in (("param", p, tp.detach()), ("exp_avg", m, st["exp_avg"]), ("exp_avg_sq", v, st["exp_avg_sq"])):
        assert torch.equal(torch.isfinite(a), torch.isfinite(b)), name
    assert not torch.isfinite(p[idx]).any()


def test_flat_adam_on_the_headline_model_matches_torch_adam():
    """FlatAdam on the prepared NIN-GC wbwtab W3A2 model (591,390 parameters) with the gradients of one QAT forward and
    backward, against torch.optim.Adam set up as the reference does (one group per tensor) from the same parameters,
    moments and step count: p, m, v within the sum of both implementations' bounds (torch evaluates the same formulas with
    its own roundings: Adam's bound with e2 = max of both scalar roundings, twice)."""
    import torch.nn as nn
    from micronet_b200 import FlatAdam
    from harness import train as T
    w = T.WORKLOADS["nin_gc_wbwtab_w3a2"]
    model = T.prepare_engine(T.build_float_model("nin_gc"), "wbwtab", **w["prepare"], **w["engine_extra"]).to(DEV)
    opt = FlatAdam(model.parameters(), lr=0.01, weight_decay=w["wd"])
    assert opt.flat_p.numel() == 591_390
    x, t = T.synthetic_batch(64, 32, 0, DEV)
    model.train()
    opt.zero_grad()
    nn.CrossEntropyLoss()(model(x), t).backward()
    gen = torch.Generator().manual_seed(9)
    step = 5
    opt.step_count = step - 1
    opt.exp_avg.copy_((torch.randn(opt.flat_p.numel(), generator=gen) * 1e-3).to(DEV))
    opt.exp_avg_sq.copy_((torch.rand(opt.flat_p.numel(), generator=gen) * 1e-6).to(DEV))
    flat_g = opt.bucket.flat.clone()
    assert flat_g[GRID_THREADS:].count_nonzero() > 0
    p0, m0, v0 = opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
    # torch.optim.Adam on copies of the same tensors, one group per tensor (harness.train.make_optimizer)
    tparams = [nn.Parameter(p.detach().clone()) for p in opt.params]
    topt = torch.optim.Adam([{"params": [q], "lr": 0.01, "weight_decay": w["wd"]} for q in tparams], lr=0.01,
                            weight_decay=w["wd"], foreach=False)
    off = 0
    for q, p in zip(tparams, opt.params):
        n = q.numel()
        q.grad = p.grad.detach().clone()
        topt.state[q] = {"step": torch.tensor(float(step - 1)), "exp_avg": m0[off:off + n].view_as(q).clone(),
                         "exp_avg_sq": v0[off:off + n].view_as(q).clone()}
        off += n
    opt.step()
    topt.step()
    torch.cuda.synchronize()
    tp = torch.cat([q.detach().reshape(-1) for q in tparams])
    tm = torch.cat([topt.state[q]["exp_avg"].reshape(-1) for q in tparams])
    tv = torch.cat([topt.state[q]["exp_avg_sq"].reshape(-1) for q in tparams])
    (p64, m64, v64), (Ep, Em, Ev) = _adam64(p0, flat_g, m0, v0, 0.01, 0.9, 0.999, 1e-8, w["wd"], step)
    _check(opt.flat_p, tp.double(), 2 * Ep, "FlatAdam vs torch.optim.Adam param")
    _check(opt.exp_avg, tm.double(), 2 * Em, "FlatAdam vs torch.optim.Adam exp_avg")
    _check(opt.exp_avg_sq, tv.double(), 2 * Ev, "FlatAdam vs torch.optim.Adam exp_avg_sq")
    # the second pass of the grid-stride loop: every element with a gradient moved
    tail = slice(GRID_THREADS - 1, None)
    nz = flat_g[tail] != 0
    assert (opt.exp_avg[tail] != m0[tail])[nz].all()
    assert (opt.flat_p[tail] != p0[tail])[nz & ((p64 - p0.double())[tail].abs() > p0[tail].abs().double() * 4 * U)].all()
