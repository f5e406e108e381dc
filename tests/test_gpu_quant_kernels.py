"""The quantizer, observer and statistics kernels of mnb_quant.cu at the bench models' tensor sizes and at their numeric
edges, each against a plain reference of the same operation:

* the CPU oracle (oracle/reference_port.py, fp32 ATen) where DESIGN.md §3 promises bit-exact results: observer state,
  scales, zero-points, integer levels, fake-quantized tensors and STE masks;
* fp64 torch where the kernel's result depends on a summation order: every bound below is derived from the number of
  fp32 roundings the kernel's arithmetic puts between the exact value and its result (u = 2^-24).

Every case id names the kernel path it reaches; the comment next to it gives the launch arithmetic (from the launchers in
mnb_quant.cu) that puts it there.  132 is the SM count the launchers size their grids by (MNB_NUM_SMS)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24           # unit roundoff of fp32 (round to nearest)
NUM_SMS = 132
N_ACT = 256 * 64 * 32 * 32   # first IAO activation of ResNet-18 at batch 256: 16.8 M


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _eq(a, b):
    """bit-exact (NaN == NaN, +0 == -0 as torch.equal has it)"""
    a, b = a.detach().cpu().reshape(-1), b.detach().cpu().reshape(-1)
    na, nb = torch.isnan(a), torch.isnan(b)
    return a.shape == b.shape and torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _first_diff(a, b):
    a, b = a.detach().cpu().reshape(-1), b.detach().cpu().reshape(-1)
    i = int((a != b).nonzero()[0]) if (a != b).any() else -1
    return f"{int((a != b).sum())} of {a.numel()} differ, first at {i}: {a[i].item() if i >= 0 else ''} vs {b[i].item() if i >= 0 else ''}"


# ============================================================================ 1. observers + update_qparams
# observe_global_kernel (rows = 1): min(ceil(n / 2048), 1024) blocks x 256 threads, grid-stride by blocks * 256; the last
# block to finish reduces the per-block partials and re-arms the counter in the shared scratch buffer.
# observe_rows_kernel (rows = out_c): one 128-thread block per row, block-stride over the row.
def _quantizers(kind, rows, bits, symmetric, is_act):
    import micronet_b200 as E
    from oracle import reference_port as O
    level, oc = ("L", None) if rows == 1 else ("C", rows)
    eobs = E.iao.MinMaxObserver(level, oc) if kind == "minmax" else E.iao.MovingAverageMinMaxObserver(level, oc)
    ecls = E.iao.SymmetricQuantizer if symmetric else E.iao.AsymmetricQuantizer
    eq = ecls(bits=bits, observer=eobs, activation_weight_flag=1 if is_act else 0).to(DEV)
    oq = O.FakeQuantizer(bits, O.RangeObserver(level, oc, ema=(kind == "ema")), is_act, symmetric)
    return eq, oq


def _observe(eq, oq, x):
    """one observer step with update_qparams: one kernel on the engine side"""
    eq.observer.observe(x, eq)
    oq.observer(x.cpu())
    oq.update_qparams()


def _check_qstate(eq, oq, what):
    for name, e, o in (("min_val", eq.observer.min_val, oq.observer.min_val),
                       ("max_val", eq.observer.max_val, oq.observer.max_val),
                       ("scale", eq.scale, oq.scale), ("zero_point", eq.zero_point, oq.zero_point)):
        assert _eq(e, o), f"{what}: {name}: {_first_diff(e, o)}"


def _steps(n, rows, seed, count):
    """count inputs whose range grows, shrinks and moves (MinMax keeps the running extremum, EMA follows)"""
    g = _gen(seed)
    shape = (n,) if rows == 1 else (rows, n // rows)
    out = []
    for i, (sc, off) in enumerate(((1.0, 0.0), (2.5, 0.3), (0.5, -0.2), (1.5, 1.0))[:count]):
        out.append(torch.randn(shape, generator=g, device=DEV) * sc + off)
    return out


OBS_CASES = [
    # id, n, rows, observer, bits, symmetric, activation (True: levels [-2^(b-1), 2^(b-1)-1] / [0, 2^b-1])
    pytest.param(1, 1, "ema", 8, False, True, id="global-1block-n1"),                          # 1 block, 1 live thread
    pytest.param(255, 1, "minmax", 4, True, False, id="global-1block-n255"),                   # 1 block, last warp partial
    pytest.param(2049, 1, "ema", 2, True, True, id="global-2blocks-n2049"),                    # 2 blocks, 1 element in the 2nd sweep
    pytest.param((1 << 21) + 3, 1, "minmax", 8, False, False, id="global-1024blocks-9sweeps-n2M+3"),   # ceil(n/2048) = 1025 -> 1024 blocks; 262,144 per sweep
    pytest.param((1 << 21) + 3, 1, "ema", 4, False, True, id="global-1024blocks-9sweeps-n2M+3-ema"),
    pytest.param(N_ACT, 1, "ema", 8, True, True, id="global-1024blocks-64sweeps-n16.8M"),    # 16,777,216 / 262,144 = 64 sweeps
    pytest.param(N_ACT, 1, "ema", 8, False, True, id="global-1024blocks-64sweeps-n16.8M-asym"),
    pytest.param(512 * 4608, 512, "minmax", 8, True, False, id="rows512x4608-36passes"),       # ResNet-18 512x512x3x3: 4608 / 128 = 36 per thread
    pytest.param(512 * 4608, 512, "ema", 4, False, False, id="rows512x4608-36passes-ema-asym"),
    pytest.param(10 * 512, 10, "ema", 2, False, False, id="rows10x512-4passes"),
    pytest.param(10 * 512, 10, "minmax", 8, True, False, id="rows10x512-4passes-sym"),
    pytest.param(1000, 1000, "minmax", 4, False, False, id="rows1000x1-1thread"),              # one live thread per block
    pytest.param(1000, 1000, "ema", 8, True, False, id="rows1000x1-1thread-ema"),
]


@pytest.mark.parametrize("n,rows,kind,bits,symmetric,is_act", OBS_CASES)
def test_observer_and_qparams_match_oracle(n, rows, kind, bits, symmetric, is_act):
    """4 steps from first = 1: min_val, max_val, scale and zero_point bit-exact after every step (IAO:15-113, 292-321)"""
    eq, oq = _quantizers(kind, rows, bits, symmetric, is_act)
    for i, x in enumerate(_steps(n, rows, 7 + n % 1000 + rows, 4 if n < N_ACT else 3)):
        _observe(eq, oq, x)
        _check_qstate(eq, oq, f"step {i}")
    # update_qparams on its own (the union quantizer of QuantAdd): the same scale / zero_point from the stored range
    eq.scale.fill_(-1.0); eq.zero_point.fill_(-1.0)
    eq.update_qparams()
    _check_qstate(eq, oq, "update_qparams")


def _edge_inputs(n, rows, seed):
    """(name, tensor) pairs: constant, all-negative, all-positive, signed zeros, and one extreme element placed at the
    first element, the last element, and the last element the last block reads (rows: first / last element of a row,
    and the last row)"""
    g = _gen(seed)
    shape = (n,) if rows == 1 else (rows, n // rows)
    r = torch.randn(shape, generator=g, device=DEV)
    out = [("constant", torch.full(shape, 3.25, device=DEV)), ("zeros", torch.zeros(shape, device=DEV)),
           ("all-negative", -(r.abs() + 0.125)), ("all-positive", r.abs() + 0.125)]
    z = torch.zeros(shape, device=DEV)
    z.view(-1)[::3] = -0.0
    out.append(("signed-zeros", z))
    flat_pos = [0, n - 1]
    if rows == 1:
        blocks = min(-(-n // 2048), 1024)
        stride = blocks * 256
        first_of_last = (blocks - 1) * 256 + 255                  # thread 255 of the last block
        if first_of_last < n:
            flat_pos.append(first_of_last + ((n - 1 - first_of_last) // stride) * stride)   # its final sweep
    else:
        inner = n // rows
        flat_pos += [inner - 1, (rows - 1) * inner, (rows - 1) * inner + inner // 2]
    for p in sorted(set(flat_pos)):
        for sgn in (1.0, -1.0):
            t = r.clone()
            t.view(-1)[p] = sgn * 1e3
            out.append((f"extreme{'+' if sgn > 0 else '-'}@{p}", t))
    return out


@pytest.mark.parametrize("n,rows", [
    pytest.param(2049, 1, id="global-2blocks"),
    pytest.param((1 << 21) + 3, 1, id="global-1024blocks-9sweeps"),
    pytest.param(64 * 4608, 64, id="rows64x4608-36passes"),
    pytest.param(7 * 130, 7, id="rows7x130-2passes"),
])
@pytest.mark.parametrize("symmetric", [True, False], ids=["sym", "asym"])
def test_observer_edges_match_oracle(n, rows, symmetric):
    """constant tensors (max = min: the scale clamps to FLT_EPSILON), single-signed tensors, +-0.0, and the extreme value
    in the first element, the last element and the last block's final sweep; first step and one EMA step each"""
    for name, x in _edge_inputs(n, rows, 11 + rows):
        eq, oq = _quantizers("ema", rows, 8, symmetric, True)
        _observe(eq, oq, x)
        _check_qstate(eq, oq, f"{name} first")
        _observe(eq, oq, x * 0.5 - 0.25)
        _check_qstate(eq, oq, f"{name} ema")
    # the clamp: a constant tensor gives the FLT_EPSILON scale on both sides
    eq, oq = _quantizers("minmax", rows, 8, False, True)
    _observe(eq, oq, torch.full((n,) if rows == 1 else (rows, n // rows), 3.25, device=DEV))
    assert (eq.scale.cpu() == torch.finfo(torch.float32).eps).all()


def test_counter_rearm_across_back_to_back_reductions():
    """last-block-done kernels share the block counter at the head of L.scratch: observers of different n (1024, 2 and 1
    blocks) and the DoReFa weight quantizer (1024-block forward and backward reductions) are queued back to back with no
    synchronisation; every result must still be exact, so each kernel re-armed the counter for the next one"""
    from micronet_b200 import functional as F_
    qs = [_quantizers("ema", 1, 8, False, True), _quantizers("minmax", 1, 4, True, True), _quantizers("ema", 1, 8, True, True)]
    sizes = [(1 << 21) + 3, 2049, 1]
    xs = [[torch.randn(n, generator=_gen(100 + 10 * j + k), device=DEV) * (k + 1) for k in range(2)]
          for j, n in enumerate(sizes)]
    w = torch.randn(192, 96, 5, 5, generator=_gen(5), device=DEV) * 0.3       # NIN 96->192 5x5: 460,800
    w_small = torch.randn(3, 4, 5, 5, generator=_gen(6), device=DEV)
    g = torch.randn(w.shape, generator=_gen(7), device=DEV)
    out = []
    for k in range(2):
        for (eq, _), x in zip(qs, xs):
            eq.observer.observe(x[k], eq)
        wg = w.clone().requires_grad_(True)
        wq, _, _ = F_.DorefaWeightFn.apply(wg, 4)
        wq.backward(g)
        wq_small, _, _ = F_.DorefaWeightFn.apply(w_small, 8)
        out.append((wq.detach(), wg.grad, wq_small))
    torch.cuda.synchronize()
    for (_, oq), x in zip(qs, xs):
        for k in range(2):
            oq.observer(x[k].cpu()); oq.update_qparams()
    for (eq, oq) in qs:
        _check_qstate(eq, oq, "queued back to back")
    # the DoReFa results of one call on its own, the scratch counter at 0 before and after (these kernels are
    # deterministic: max, integer tie count, fixed-order fp64 partial sums); test_dorefa_weight_matches_oracle pins them
    # to the oracle
    wg = w.clone().requires_grad_(True)
    wq_alone, _, _ = F_.DorefaWeightFn.apply(wg, 4)
    wq_alone.backward(g)
    wq_small_alone, _, _ = F_.DorefaWeightFn.apply(w_small, 8)
    torch.cuda.synchronize()
    for k in range(2):
        wq, dw, wq_small = out[k]
        assert _eq(wq, wq_alone) and _eq(wq_small, wq_small_alone), f"call {k}: DoReFa forward"
        assert _eq(dw, wg.grad), f"call {k}: DoReFa backward {_first_diff(dw, wg.grad)}"


def test_observer_ema_step_replayed_from_a_cuda_graph():
    """an EMA observer step (with update_qparams) captured once and replayed k times equals k eager oracle steps"""
    eq, oq = _quantizers("ema", 1, 8, False, True)
    x0 = torch.randn((1 << 21) + 3, generator=_gen(21), device=DEV)
    _observe(eq, oq, x0)                      # the first call (first = 1 is decided on the host) runs eagerly
    torch.cuda.synchronize()
    static = torch.randn_like(x0) * 3 + 0.5
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eq.observer.observe(static, eq)
    torch.cuda.synchronize()
    _check_qstate(eq, oq, "capture must not run the step")
    xs = static.cpu()
    for k in range(6):
        graph.replay()
        oq.observer(xs); oq.update_qparams()
        torch.cuda.synchronize()
        _check_qstate(eq, oq, f"replay {k + 1}")


# ============================================================================ 2. weight quantizers
def _rel(a, b, skip=None):
    """max |a - b| / max |b| over the elements not in ``skip`` (flat indices)"""
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    d = (a - b).abs()
    if skip is not None and len(skip):
        d[skip] = 0
    den = b.abs().max().item()
    return d.max().item() / den if den else d.max().item()


def _argmax_set(w):
    t = torch.tanh(w.detach().cpu()).abs().reshape(-1)
    return (t == t.max()).nonzero().reshape(-1)


def _tie_excused(pre, got, want):
    """(mismatches, mismatches not within 2 ulp of a k + 0.5 rounding tie) of DoReFa weight levels (DESIGN §3)"""
    bad = got != want
    if not bad.any():
        return 0, 0
    frac = np.abs(np.abs(pre[bad]) % 1.0 - 0.5)
    ulp = np.spacing(np.abs(pre[bad]).astype(np.float32))
    return int(bad.sum()), int((frac > 2 * ulp).sum())


def _dorefa_check(w, bits, g, what):
    """DoReFa weight quantizer (DF:61-73) forward and backward against the oracle.  Levels and w_scale bit-exact (the tie
    excuse of DESIGN §3 for the tanh); wq bit-exact wherever the level agrees; the gradient within 1e-5 of max|dw| except at
    the arg-max of |tanh w|, whose gradient collects the cancelling sum -sum(G t / 2) / m^2 over the whole tensor: 1e-3 of
    the larger of max|dw| and that sum's absolute value (the tolerances of test_gpu_parity._teacher_forced)."""
    from micronet_b200 import functional as F_
    from oracle import reference_port as O
    L = 2 ** bits - 1
    wg = w.clone().requires_grad_(True)
    wq, w_int, w_scale = F_.DorefaWeightFn.apply(wg, bits)
    wq.backward(g)
    wo = w.cpu().requires_grad_(True)
    yo = O.dorefa_quantize_weight(wo, bits)
    yo.backward(g.cpu())
    k_ref, pre = O.dorefa_weight_levels(w.cpu(), bits)
    k = (w_int.cpu().int() + L) // 2
    nbad, unexcused = _tie_excused(pre.numpy(), k.float().numpy(), k_ref.numpy())
    assert unexcused == 0, f"{what}: {nbad} level mismatches, {unexcused} not at a tie"
    assert (w_scale.cpu() == np.float32(1.0 / L)).all(), what
    same = (k.float() == k_ref).reshape(-1)
    assert _eq(wq.reshape(-1)[same.to(DEV)], yo.detach().reshape(-1)[same]), f"{what}: wq"
    am = _argmax_set(w)
    assert _rel(wg.grad, wo.grad, skip=am) <= 1e-5, f"{what}: dw {_rel(wg.grad, wo.grad, skip=am):.2e}"
    # the arg-max elements: the absolute value of the sum they collect
    t = torch.tanh(w.cpu().double()).reshape(-1)
    m = t.abs().max().item()
    G = 2.0 * g.cpu().double().reshape(-1)
    s_abs = ((G * t / 2).abs().sum().item() / (m * m) / len(am) + G[am].abs().max().item() / (2 * m)) * (1 - m * m)
    den = max(wo.grad.abs().max().item(), s_abs)
    d = (wg.grad.cpu().reshape(-1)[am].double() - wo.grad.reshape(-1)[am].double()).abs().max().item()
    assert d <= 1e-3 * den, f"{what}: arg-max gradient {d / den:.2e}"
    return wg.grad, wo.grad


@pytest.mark.parametrize("shape,bits", [
    pytest.param((1, 1, 1, 1), 4, id="n1-1block"),                     # 1 block; the single element is the arg-max
    pytest.param((3, 4, 5, 5), 2, id="n300-2blocks"),                  # ceil(300 / 256) = 2 blocks
    pytest.param((5, 52429, 1, 1), 8, id="n262145-1024blocks-2sweeps"),    # 1025 -> 1024 blocks, 1 element in the 2nd sweep
    pytest.param((192, 96, 5, 5), 4, id="n460800-1024blocks-2sweeps"),     # NIN 96->192 5x5, 1.76 sweeps of 262,144
])
def test_dorefa_weight_matches_oracle(shape, bits):
    w = torch.randn(shape, generator=_gen(sum(shape)), device=DEV) * 0.4
    g = torch.randn(shape, generator=_gen(sum(shape) + 1), device=DEV)
    _dorefa_check(w, bits, g, str(shape))


@pytest.mark.parametrize("n,bits", [pytest.param(300, 4, id="n300-2blocks"),
                                    pytest.param(460800, 8, id="n460800-1024blocks")])
def test_dorefa_weight_gradient_splits_evenly_among_ties(n, bits):
    """torch.max's backward spreads the gradient of m = max|tanh w| evenly over every element attaining it
    (dorefa_w_bwd_kernel: share = dm / count, with the sign of t).  Ties at m < 1: several +0.75 and -0.75 weights, all
    with the same upstream gradient, so every +m tie must get the same dw, every -m tie the same, and (dw+ - dw-) / 2 /
    (1 - m^2) is the share, checked against dm / count in fp64.  Saturated ties: |w| > 9.1 gives tanh = 1.0f exactly;
    those elements have dw = 0 (1 - t^2 = 0), the others still match."""
    g0 = torch.Generator().manual_seed(n)
    w = (torch.rand(n, generator=g0) * 1.4 - 0.7)                       # |w| < 0.7 < 0.75
    idx = torch.randperm(n, generator=g0)
    pos, neg = idx[:5], idx[5:9]
    w[pos], w[neg] = 0.75, -0.75
    g = torch.randn(n, generator=g0)
    g[pos], g[neg] = 0.375, 0.375
    wd, gd = w.reshape(n, 1, 1, 1).to(DEV), g.reshape(n, 1, 1, 1).to(DEV)
    dw, dwo = _dorefa_check(wd, bits, gd, "ties at 0.75")
    dw = dw.cpu().reshape(-1).double()
    assert (dw[pos] == dw[pos[0]]).all() and (dw[neg] == dw[neg[0]]).all(), (dw[pos], dw[neg])
    t = torch.tanh(w.double())
    m = t.abs().max().item()
    s = np.float32(1.0 / (2 ** bits - 1))
    G = ((g.float() * 2) * torch.tensor(s)) / torch.tensor(s)            # the upstream gradient of o, as both compute it
    dm = (-(G.double() * t / 2) / (m * m)).sum().item()
    share = (dw[pos[0]] - dw[neg[0]]).item() / 2 / (1 - m * m)
    dm_abs = ((G.double() * t / 2).abs() / (m * m)).sum().item()
    # the kernel's dm is an fp64 sum of fp32 terms of <= 5 roundings each: |error| <= 5 u dm_abs (+ the tanh's ulp)
    assert abs(share - dm / 9) <= 1e-5 * dm_abs / 9, (share, dm / 9)
    # saturated ties of both signs among the same weights
    w2 = w.clone()
    w2[pos], w2[neg] = 9.5, -12.0
    w2[idx[9:40]] = 20.0
    dw2, _ = _dorefa_check(w2.reshape(n, 1, 1, 1).to(DEV), bits, gd, "saturated ties")
    sat = (w2.abs() > 9.1)
    assert (dw2.cpu().reshape(-1)[sat] == 0).all()


# ---------------------------------------------------------------- wbwtab (WB:98-149): one 128-thread block per output channel
@pytest.mark.parametrize("shape", [
    pytest.param((8, 1, 3, 3), id="cpg1-9taps"),                      # mean over a single channel: the centred weight is 0
    pytest.param((16, 200, 1, 1), id="cpg200-1tap"),                  # one thread walks 200 channels
    pytest.param((32, 64, 3, 3), id="cpg64-inner576-5passes"),        # 576 / 128 -> 5 block-stride passes
    pytest.param((256, 256, 3, 3), id="cpg256-inner2304-18passes"),   # NIN-GC-sized layer
])
def test_wbwtab_binary_weight_matches_oracle(shape):
    """W = 2: the in-place mean-centring over the input channels (per tap) and clamp to [-1, 1] (WB:98-102), then
    sign * E|w| per output channel.  The mutated parameter: the kernel sums the cpg values in fp64 and rounds the mean
    once; the oracle's fp32 ATen sum rounds up to cpg - 1 times, so the two centred weights differ by at most
    (cpg + 1) u mean|w| + 2 u |w - mean| (both subtractions rounded).  Levels bit-exact; wq and dw within 1e-5."""
    from micronet_b200 import functional as F_
    from oracle import reference_port as O
    w0 = torch.randn(shape, generator=_gen(shape[1]), device=DEV) * 0.6 + 0.1
    g = torch.randn(shape, generator=_gen(shape[1] + 1), device=DEV)
    we = w0.clone().requires_grad_(True)
    wq, w_int, w_scale = F_.WbWeightFn.apply(we, 2)
    wq.backward(g)
    wo = torch.nn.Parameter(w0.cpu())
    yo = O.wb_quantize_weight(wo, 2)
    yo.backward(g.cpu())
    cpg = shape[1]
    w64 = w0.cpu().double()
    mabs = w64.abs().mean(1, keepdim=True)
    bound = (cpg + 1) * U * mabs + 2 * U * (w64 - w64.mean(1, keepdim=True)).abs() + 1e-30
    d = (we.detach().cpu().double() - wo.detach().double()).abs()
    assert (d <= bound).all(), f"mutated weight: worst {(d / bound).max().item():.2f} x the bound"
    lv = torch.sign(wo.detach()); lv[lv == 0] = 1
    assert torch.equal(w_int.cpu().float(), lv)
    alpha_o = wo.detach().abs().mean((1, 2, 3))
    assert _rel(w_scale, alpha_o) <= 1e-5 and _rel(wq, yo) <= 1e-5 and _rel(we.grad, wo.grad) <= 1e-5


def _ternary_rows(out_c, inner, rng, ties=2, zero_rows=()):
    """out_c rows of ``inner`` weights with ``ties`` elements exactly at +-thr, thr = fl(0.7f * fl(sum|w| / inner))
    (WB:55-75), computed identically by any summation order: every |w| < 1 is a multiple of 2^-G with inner < 2^(24 - G),
    so every partial sum of |w| is exact in fp32, and thr itself is picked on that grid"""
    G = 24 - math.ceil(math.log2(inner + 1))
    grid = 2.0 ** -G
    seven = np.float32(0.7)
    rows = []
    for r in range(out_c):
        if r in zero_rows:
            rows.append(np.zeros(inner, np.float32))
            continue
        units = np.arange(int(0.40 * inner / grid), int(0.50 * inner / grid), dtype=np.int64)
        S = units * grid                                     # sum |w|, exact in fp64 and fp32
        E = (S / inner).astype(np.float32)                   # fp64 quotient rounded once = fp32 quotient of the exact sum
        thr = (seven * E).astype(np.float32)
        on_grid = (thr.astype(np.float64) / grid) == np.round(thr.astype(np.float64) / grid)
        cand = np.nonzero(on_grid & (thr > 0))[0]
        assert len(cand), (inner, G)
        j = cand[rng.integers(len(cand))]
        t_units = int(round(float(thr[j]) / grid))
        rest = int(units[j]) - ties * t_units                # grid units left for the other inner - ties weights
        n_rest = inner - ties
        p = 0.5 + 0.5 * rng.random(n_rest)                  # shares within 4/3 of the mean: every |w| stays < 1
        mag = np.floor(p / p.sum() * rest).astype(np.int64)
        mag[rng.permutation(n_rest)[:rest - int(mag.sum())]] += 1     # settle the total exactly on the grid
        assert mag.sum() == rest and mag.max() < 2 ** G
        vals = np.concatenate([mag, np.full(ties, t_units)]).astype(np.float64) * grid
        sign = np.where(rng.random(inner) < 0.5, -1.0, 1.0)
        sign[n_rest:] = [1.0 if i % 2 == 0 else -1.0 for i in range(ties)]
        row = (vals * sign).astype(np.float32)
        rows.append(row[rng.permutation(inner)])
    return np.stack(rows)


@pytest.mark.parametrize("cpg,khw,zero_row", [
    pytest.param(1, 9, None, id="cpg1-inner9-shorter-than-block"),           # 9 of the 128 threads hold a weight
    pytest.param(128, 1, 2, id="inner128-one-pass-zero-channel"),            # exactly one block-stride pass
    pytest.param(256, 9, 0, id="inner2304-18passes-zero-channel"),           # 2304 / 128 = 18 passes
])
def test_wbwtab_ternary_weight_matches_oracle(cpg, khw, zero_row):
    """W = 3 (WB:55-75, 132-146).  Weights exactly at +-thr: the reference gives them level sign(sign(2 thr) + 0) = +-1 but
    leaves them out of alpha = mean(|w| > thr) (its count uses gt): the kernel must do the same.  An all-zero channel has
    thr = 0, no element above it and alpha = 0 / 0: the reference produces NaN for that channel's alpha, every wq of the
    channel (0 * NaN) and its whole weight gradient; the kernel must produce exactly that, and leave the other channels
    finite.  Levels, alpha and wq bit-exact (every sum here is exact, see _ternary_rows); dw within 1e-5."""
    from micronet_b200 import functional as F_
    from oracle import reference_port as O
    out_c = 6
    rows = _ternary_rows(out_c, cpg * khw, np.random.default_rng(cpg * 7 + khw), zero_rows=() if zero_row is None else (zero_row,))
    w0 = torch.from_numpy(rows).reshape(out_c, cpg, int(math.isqrt(khw)), -1)
    g = torch.randn(w0.shape, generator=torch.Generator().manual_seed(3))
    t_o, thr_o = O._TernarySTE.apply(w0.clone())
    E = torch.from_numpy(np.abs(rows).sum(1).astype(np.float32) / np.float32(cpg * khw))
    assert torch.equal(thr_o.reshape(-1), E * np.float32(0.7)), "test construction: thr is not the expected exact value"
    at_thr = (w0.abs() == thr_o) & (thr_o > 0)
    assert int(at_thr.sum()) >= 2 * (out_c - (zero_row is not None))
    we = w0.to(DEV).requires_grad_(True)
    wq, w_int, w_scale = F_.WbWeightFn.apply(we, 3)
    wq.backward(g.to(DEV))
    wo = w0.clone().requires_grad_(True)
    yo = O.wb_quantize_weight(wo, 3)
    yo.backward(g)
    assert torch.equal(w_int.cpu().float(), t_o), _first_diff(w_int.float(), t_o)
    assert (t_o[at_thr].abs() == 1).all()                     # what the reference gives a weight exactly at +-thr
    alpha_o = (yo.detach() / torch.where(t_o == 0, torch.ones_like(t_o), t_o)).abs().amax((1, 2, 3))
    keep = torch.ones(out_c, dtype=torch.bool)
    if zero_row is not None:
        keep[zero_row] = False
        assert torch.isnan(yo.detach()[zero_row]).all() and torch.isnan(wo.grad[zero_row]).all()   # the reference's NaNs
        assert torch.isnan(w_scale[zero_row]).item()
    assert _eq(w_scale.cpu()[keep], alpha_o[keep]), _first_diff(w_scale.cpu()[keep], alpha_o[keep])
    assert _eq(wq, yo), _first_diff(wq, yo)
    assert torch.equal(torch.isnan(we.grad.cpu()), torch.isnan(wo.grad))
    assert _rel(we.grad[keep.to(DEV)], wo.grad[keep]) <= 1e-5


# ---------------------------------------------------------------- IAO weights (IAO:214-240)
# iao_weight_fwd/bwd_kernel: min(ceil(n / 256), 132 * 8 = 1056) blocks x 256 threads, grid-stride by 270,336.
def _iao_crafted(shape, per_channel, symmetric, bits, rng):
    """weights whose first-step scale is a power of two, so that w / s lands exactly on k + 1/2 (rounding ties) and the
    row's extremes land exactly on lo / hi.  Symmetric: |w| <= Q s with +-Q s present (Q = 2^(b-1) - 1, s = Q s / Q
    exactly).  Asymmetric: w in [-z s, (Q - z) s] with both ends present (Q = 2^b - 2), so zero_point = -z."""
    out_c, inner = shape[0], int(np.prod(shape[1:]))
    rows = out_c if per_channel else 1
    Q = (1 << (bits - 1)) - 1 if symmetric else (1 << bits) - 2
    w = np.empty((rows, out_c * inner // rows), np.float64)
    for r in range(rows):
        s = 2.0 ** -(5 + r % 4)
        lo_k, hi_k = (-Q, Q) if symmetric else (-(int(rng.integers(1, Q)) if Q > 1 else 1), None)
        if not symmetric:
            hi_k = Q + lo_k
        k = rng.integers(lo_k, hi_k, w.shape[1]).astype(np.float64) + 0.5     # exact ties k + 1/2 inside [lo, hi]
        k[rng.random(w.shape[1]) < 0.3] -= 0.5                                  # and exact levels
        k[0], k[-1] = lo_k, hi_k                                                # the range ends exactly
        w[r] = k * s
    return torch.from_numpy(w.astype(np.float32).reshape(shape))


@pytest.mark.parametrize("shape,q_level,q_type,bits,observer", [
    pytest.param((512, 512, 3, 3), 0, 0, 8, 1, id="perchannel-sym8-2.36M-1056blocks-9sweeps"),    # 2,359,296 / 270,336
    pytest.param((512, 512, 3, 3), 1, 1, 8, 1, id="perlayer-asym8-2.36M-1056blocks-9sweeps"),
    pytest.param((64, 64, 3, 3), 1, 0, 4, 0, id="perlayer-sym4-144blocks-1sweep"),
    pytest.param((64, 64, 3, 3), 0, 1, 4, 1, id="perchannel-asym4-144blocks-1sweep"),
    pytest.param((16, 3, 3, 3), 0, 1, 2, 0, id="perchannel-asym2-2blocks"),
    pytest.param((10, 512), 0, 0, 2, 1, id="fc-perchannel-sym2-20blocks"),
])
def test_iao_weight_matches_oracle(shape, q_level, q_type, bits, observer):
    """observer + update_qparams + fake-quant of a weight, three training steps.  Step 0: crafted weights (exact ties at
    w/s = k + 1/2, the row extremes exactly at lo / hi).  Steps 1, 2: the weight grows by 1.7 then shrinks; under the EMA
    observer the range lags, so elements lie past hi and past qmax: clamped, and their gradient is cut.  Observer state,
    scale, zero_point, integer levels, w_scale and wq bit-exact; the gradient (g * s / s where the STE passes, else 0) too,
    which pins the pass mask; the elements at lo / hi must pass."""
    import micronet_b200 as E
    from micronet_b200 import functional as F_
    from oracle import reference_port as O
    per_channel = q_level == 0
    out_c = shape[0]
    fc = len(shape) == 2
    eq = E.iao._weight_quantizer(bits, q_type, q_level, observer, out_c, False, False, channel_level="FC" if fc else "C").to(DEV)
    oq = O._iao_weight_quantizer(bits, q_type, q_level, observer, out_c, False, False, fc=fc)
    eq.train(); oq.train()
    w0 = _iao_crafted(shape, per_channel, q_type == 0, bits, np.random.default_rng(out_c + bits))
    noise = torch.randn(shape, generator=torch.Generator().manual_seed(1)) * w0.abs().max() * 0.05
    cut_seen = False
    for step, w in enumerate((w0, w0 * 1.7 + noise, w0 * 0.6)):
        g = torch.randn(shape, generator=torch.Generator().manual_seed(10 + step))
        we = w.to(DEV).requires_grad_(True)
        eq.refresh(we)
        obs = eq.observer
        wq, w_int, w_scale = F_.IaoWeightFn.apply(we, eq.scale, eq.zero_point, obs.min_val, obs.max_val, eq.q_type,
                                                 eq.qmin, eq.qmax)
        wq.backward(g.to(DEV))
        wo = w.clone().requires_grad_(True)
        yo = oq(wo)
        yo.backward(g)
        _check_qstate(eq, oq, f"step {step}")
        lv = oq.levels(w) + oq.zero_point
        assert torch.equal(w_int.cpu().float(), lv), f"step {step}: levels {_first_diff(w_int.float(), lv)}"
        assert _eq(w_scale, oq.scale.reshape(-1).expand(out_c)), f"step {step}: w_scale"
        assert _eq(wq, yo), f"step {step}: wq {_first_diff(wq, yo)}"
        assert _eq(we.grad, wo.grad), f"step {step}: dw {_first_diff(we.grad, wo.grad)}"
        passed = we.grad.cpu() != 0
        if step == 0:
            w2 = w.reshape(out_c if per_channel else 1, -1)
            ends = torch.zeros_like(w2, dtype=torch.bool)
            ends[:, 0] = ends[:, -1] = True
            assert passed.reshape(w2.shape)[ends].all(), "elements exactly at lo / hi must pass the STE"
            v = (w / oq.scale - oq.zero_point).reshape(-1)
            assert ((v.abs() % 1) == 0.5).sum() > w.numel() // 4, "test construction: too few exact rounding ties"
        cut_seen |= bool((~passed).any())
    if observer == 1:
        assert cut_seen, "the EMA steps should have put elements past hi"


# ============================================================================ 3. activation quantizer and QuantAdd
# act_quant_fwd_kernel / quant_add_fwd_kernel: min(ceil(n / 1024), 1056) blocks x 256 threads; each warp owns 128
# consecutive elements and writes 4 pass-bit words; grid-stride by 1056 * 1024 = 1,081,344 elements.
def _pack_bits(mask):
    m = np.asarray(mask, dtype=bool).reshape(-1)
    m = np.concatenate([m, np.zeros((-len(m)) % 32, bool)])
    return np.packbits(m, bitorder="little").view("<u4")


ACT_SHAPES = [
    pytest.param((1, 1, 1, 1), id="n1-1warp-tailword1bit"),
    pytest.param((1, 13, 17, 19), id="n4199-5blocks-tailword7bits"),      # 4199 % 32 = 7, % 128 = 103
    pytest.param((3, 5, 31, 29), id="n13485-14blocks-tailword13bits"),    # 13485 % 32 = 13
    pytest.param((256, 64, 32, 32), id="n16.8M-1056blocks-16sweeps"),    # 16,777,216 / 1,081,344 = 15.5
]


@pytest.mark.parametrize("shape", ACT_SHAPES)
@pytest.mark.parametrize("bits,q_type", [(8, 0), (4, 1)], ids=["sym8", "asym4"])
def test_iao_activation_quantizer_matches_oracle(shape, bits, q_type):
    """the IAO activation quantizer (EMA observer + qparams + fake-quant, IAO:214-240): outputs, input gradients and
    state bit-exact over three steps; the pass-bit words (including the tail word of n % 32 != 0, whose bits past n
    must be 0) equal the oracle's STE mask"""
    import micronet_b200 as E
    from micronet_b200 import functional as F_
    from oracle import reference_port as O
    eq = E.iao._activation_quantizer(bits, q_type, False, False, 0.9999).to(DEV)
    oq = O._iao_act_quantizer(bits, q_type, False, False, 0.9999)
    eq.train(); oq.train()
    big = shape[0] == 256
    for step in range(2 if big else 3):
        x = torch.randn(shape, generator=_gen(step), device=DEV) * (1 + step) + 0.3 * step
        g = torch.randn(shape, generator=_gen(50 + step), device=DEV)
        xe = x.clone().requires_grad_(True)
        ye = eq(xe)
        ye.backward(g)
        xo = x.cpu().requires_grad_(True)
        yo = oq(xo)
        yo.backward(g.cpu())
        _check_qstate(eq, oq, f"step {step}")
        assert _eq(ye, yo), f"step {step}: {_first_diff(ye, yo)}"
        assert _eq(xe.grad, xo.grad), f"step {step}: dx {_first_diff(xe.grad, xo.grad)}"
        _, bits_e, _ = F_.act_quant_raw(x, eq.act_spec(), False, True, False)
        ones = torch.ones_like(xo)
        xo2 = x.cpu().requires_grad_(True)
        oq.eval(); oq(xo2).backward(ones); oq.train()
        assert np.array_equal(bits_e.cpu().numpy().view("<u4"), _pack_bits(xo2.grad.numpy() != 0)), f"step {step}: pass bits"


@pytest.mark.parametrize("shape", ACT_SHAPES)
def test_dorefa_activation_quantizer_matches_oracle(shape):
    """DoReFa activation (DF:36-46) at the same sizes: outputs, gradients and pass bits bit-exact"""
    from micronet_b200 import _lib as L, functional as F_
    from oracle import reference_port as O
    x = torch.randn(shape, generator=_gen(3), device=DEV) * 6 + 2
    g = torch.randn(shape, generator=_gen(4), device=DEV)
    spec = F_.ActSpec(L.ACT_DOREFA, bits=4)
    xe = x.clone().requires_grad_(True)
    ye = F_.ActQuantFn.apply(xe, spec)
    ye.backward(g)
    xo = x.cpu().requires_grad_(True)
    yo = O.dorefa_quantize_activation(xo, 4)
    yo.backward(g.cpu())
    assert _eq(ye, yo) and _eq(xe.grad, xo.grad)
    _, bits_e, _ = F_.act_quant_raw(x, spec, False, True, False)
    t = x.cpu() * np.float32(0.1)
    assert np.array_equal(bits_e.cpu().numpy().view("<u4"), _pack_bits(((t >= 0) & (t <= 1)).numpy()))


@pytest.mark.parametrize("shape", ACT_SHAPES)
@pytest.mark.parametrize("bits,q_type", [(8, 0), (8, 1)], ids=["sym8", "asym8"])
def test_quant_add_matches_oracle(shape, bits, q_type):
    """QuantAdd (IAO:1441-1498): two EMA observers, the union range, Q(a) + Q(b) in one kernel, and both STE masks in the
    backward: sum, both input gradients and all observer state bit-exact"""
    import micronet_b200 as E
    from oracle import reference_port as O
    e = E.iao.QuantAdd(a_bits=bits, q_type=q_type).to(DEV)
    o = O.IaoQuantAdd(a_bits=bits, q_type=q_type)
    e.train(); o.train()
    for step in range(2 if shape[0] == 256 else 3):
        a = torch.randn(shape, generator=_gen(60 + step), device=DEV) * (1.5 + step)
        b = torch.relu(torch.randn(shape, generator=_gen(70 + step), device=DEV)) * 1.7
        g = torch.randn(shape, generator=_gen(80 + step), device=DEV)
        ae, be = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        ao, bo = a.cpu().requires_grad_(True), b.cpu().requires_grad_(True)
        ye, yo = e(ae, be), o(ao, bo)
        ye.backward(g); yo.backward(g.cpu())
        assert _eq(ye, yo), f"step {step}: sum {_first_diff(ye, yo)}"
        assert _eq(ae.grad, ao.grad) and _eq(be.grad, bo.grad), f"step {step}: gradients"
        _check_qstate(e.activation_quantizer, o.activation_quantizer, f"step {step}")
        for name in ("observer_res", "observer_shortcut"):
            assert _eq(getattr(e, name).min_val, getattr(o, name).min_val), name
            assert _eq(getattr(e, name).max_val, getattr(o, name).max_val), name


# ============================================================================ 4. statistics
def _stats_launch(batch, channels, hw, aligned):
    """(splits, vector path?, fp32 chain length per thread) of channel_stats_kernel, as mnb_channel_stats /
    mnb_bn_batch_stats launch it: grid (channels, splits) of 256 threads, splits = min(32, batch, batch*hw / 2048) capped
    at ceil(2112 / channels) (~2 waves of 8 blocks per SM).  Vector path (hw % 4 == 0, 16-byte aligned x): each thread
    keeps 4 fp32 accumulators and adds one float4 per step to each, over the split's (image, offset) pairs, so a chain has
    ceil(images * hw / 4 / 1024) steps.  Scalar path: one fp32 accumulator per image, ceil(hw / 256) steps, then fp64."""
    per = batch * hw
    splits = max(1, min(32, batch, per // 2048))
    splits = max(1, min(splits, -(-(2 * 8 * NUM_SMS) // channels)))
    vec = hw % 4 == 0 and aligned
    imgs = -(-batch // splits)
    chain = -(-imgs * hw // 4096) if vec else -(-hw // 256)
    return splits, vec, chain


STATS_SHAPES = [
    # (batch, channels, h, w), |mean| / std, misaligned view, expected (splits, vector path, chain) of _stats_launch
    pytest.param((256, 256, 32, 32), 1.0, False, (9, True, 8), id="ningc-256x256x32x32-9splits-vec-chain8"),
    pytest.param((256, 512, 16, 16), 1.0, False, (5, True, 4), id="ningc-256x512x16x16-5splits-vec-chain4"),
    pytest.param((256, 1024, 8, 8), 1.0, False, (3, True, 2), id="ningc-256x1024x8x8-3splits-vec-chain2"),
    pytest.param((256, 512, 4, 4), 1.0, False, (2, True, 1), id="resnet-256x512x4x4-2splits-vec-chain1"),
    pytest.param((2, 8, 1, 1), 1.0, False, (1, False, 1), id="batchxhw2-1split-scalar"),
    pytest.param((1, 6, 1, 2), 1.0, False, (1, False, 1), id="batch1xhw2-1split-scalar"),
    pytest.param((256, 64, 7, 7), 1.0, False, (6, False, 1), id="256x64x7x7-6splits-scalar-hw49"),
    pytest.param((9, 20, 13, 7), 1.0, False, (1, False, 1), id="9x20x13x7-1split-scalar-hw91"),
    pytest.param((64, 96, 16, 16), 1.0, True, (8, False, 1), id="64x96x16x16-8splits-misaligned-scalar"),
    pytest.param((64, 32, 8, 8), 1e5, False, (2, True, 1), id="64x32x8x8-2splits-vec-mean1e5"),
    pytest.param((64, 32, 9, 9), 1e5, False, (2, False, 1), id="64x32x9x9-2splits-scalar-mean1e5"),
    pytest.param((4, 8192, 2, 2), 1.0, False, (1, True, 1), id="4x8192x2x2-1split-vec-8192channels"),
]
BN_SHAPES = [p for p in STATS_SHAPES if p.id.split("-")[0] in ("ningc", "resnet", "batchxhw2", "256x64x7x7", "64x96x16x16",
                                                                "64x32x8x8", "4x8192x2x2")]


def _stats_input(shape, mean_over_std, misaligned, seed):
    b, c, h, w = shape
    n = b * c * h * w
    g = _gen(seed)
    base = torch.empty(n + (1 if misaligned else 0), device=DEV)
    x = base[1:] if misaligned else base
    x = x.view(shape)
    sd = torch.rand(c, generator=g, device=DEV) + 0.5
    if mean_over_std > 1:    # |mean| / std between mean_over_std and 4 mean_over_std, both signs
        mu = (torch.rand(c, generator=g, device=DEV) + 1) * mean_over_std * sd * torch.where(torch.arange(c, device=DEV) % 2 == 0, 1.5, -2.0)
    else:
        mu = (torch.rand(c, generator=g, device=DEV) - 0.5) * 4
    x.copy_(torch.randn(shape, generator=g, device=DEV) * sd.view(1, c, 1, 1) + mu.view(1, c, 1, 1))
    x[0, :, 0, 0] += 4 * sd      # the pivot (each channel's first value) sits 4 std off the mean: see _stats_reference
    if misaligned:
        assert x.data_ptr() % 16 == 4 and x.is_contiguous()
    return x


def _stats_reference(x, launch):
    """fp64 statistics of x and the error bounds of the kernel's results.

    The kernel sums d = x - p (p = the channel's first value, x[0, c, 0, 0]) in fp32 chains of `chain` steps per thread,
    then in fp64.  Each d and d^2 passes through at most chain + 4 (vector: subtraction, two pair adds, the chain, the fp64
    hand-over) resp. chain + 6 roundings of relative size u, so
        |s1 - S1| <= (chain + 4) u A1,   |s2 - S2| <= (chain + 6) u A2,   A1 = sum |d|, A2 = sum d^2,
    and mean = p + s1 / N, var = (s2 - N dmean^2) / (N - 1) carry
        mean: (chain + 4) u A1 / N + u |mean|                         (the last term: the fp32 result)
        var:  ((chain + 6) u A2 + 2 |dmean| (chain + 4) u A1) / (N - 1) + u var.
    (chain + 6) u is below 1e-6 for every case here, while one dropped or double-counted split changes s2 by a 1 / splits
    share of A2 (>= 1/32 = 3e-2): the variance bound fails by four orders of magnitude.  The mean fails too, because the
    pivot sits 4 std off the mean, so every split's s1 is ~ -4 std per element.  The test asserts, for the last split, that
    dropping it (or counting it twice: the same change) would break both bounds in every channel.  With one split the
    same holds for one thread's chain (a 1/256 share)."""
    b, c = x.shape[0], x.shape[1]
    hw = x.numel() // (b * c)
    xd = x.double().reshape(b, c, hw)
    p = xd[0, :, 0]
    d = xd - p.view(1, c, 1)
    s1_img, s2_img, a1_img = d.sum(2), (d * d).sum(2), d.abs().sum(2)
    N = b * hw
    S1, S2, A1 = s1_img.sum(0), s2_img.sum(0), a1_img.sum(0)
    dm = S1 / N
    mean = p + dm
    ss = S2 - N * dm * dm
    var = ss / max(N - 1, 1)
    splits, _, chain = launch
    k1, k2 = (chain + 4) * U, (chain + 6) * U
    b_mean = k1 * A1 / N + U * mean.abs()
    b_ss = k2 * S2 + 2 * dm.abs() * k1 * A1
    b_var = b_ss / max(N - 1, 1) + U * var
    if splits > 1:   # the bounds are sharp enough to see one split dropped or counted twice
        lo, hi = (b * (splits - 1)) // splits, b
        sp1, sp2 = s1_img[lo:hi].sum(0), s2_img[lo:hi].sum(0)
        ss_drop = (S2 - sp2) - N * ((S1 - sp1) / N) ** 2
        dmean_drop, dvar_drop = (sp1 / N).abs(), (ss_drop - ss).abs() / max(N - 1, 1)
        assert ((dmean_drop > b_mean) & (dvar_drop > b_var)).all(), "bound too loose to see a dropped split"
    return dict(N=N, mean=mean, var=var, ss=ss, b_mean=b_mean, b_ss=b_ss, b_var=b_var, p=p)


@pytest.mark.parametrize("shape,mean_over_std,misaligned,path", STATS_SHAPES)
def test_channel_mean_var_and_backward_vs_fp64(shape, mean_over_std, misaligned, path):
    """channel_mean_var (IAO:853-855: mean, unbiased var) and channel_stats_bwd against fp64, bounds of _stats_reference.
    Backward: dx = dmean / N + dvar * 2 / (N - 1) * (x - mean), elementwise in fp32 with the forward's fp32 mean, so
        |dx - dx64| <= 6 u (|a| + |b| |x - mean|) + |b| * bound(mean),   a = dmean / N, b = 2 dvar / (N - 1)."""
    from micronet_b200 import functional as F_
    b, c, h, w = shape
    launch = _stats_launch(b, c, h * w, not misaligned)
    assert launch == path, launch
    x = _stats_input(shape, mean_over_std, misaligned, seed=c + h)
    ref = _stats_reference(x, launch)
    xe = x.detach().requires_grad_(True)
    m, v = F_.channel_mean_var(xe)
    em = (m.double() - ref["mean"]).abs()
    ev = (v.double() - ref["var"]).abs()
    assert (em <= ref["b_mean"]).all(), f"mean: worst {(em / ref['b_mean']).max().item():.3f} x the bound"
    assert (ev <= ref["b_var"]).all(), f"var: worst {(ev / ref['b_var']).max().item():.3f} x the bound"
    gm = torch.randn(c, generator=_gen(1), device=DEV)
    gv = torch.randn(c, generator=_gen(2), device=DEV)
    (m * gm + v * gv).sum().backward()
    N = ref["N"]
    a = gm.double() / N
    bb = gv.double() * 2 / max(N - 1, 1)
    dev = x.double() - ref["mean"].view(1, c, 1, 1)
    want = a.view(1, c, 1, 1) + bb.view(1, c, 1, 1) * dev
    bound = 6 * U * (a.abs().view(1, c, 1, 1) + (bb.abs().view(1, c, 1, 1) * dev.abs())) \
        + (bb.abs() * ref["b_mean"]).view(1, c, 1, 1)
    err = (xe.grad.double() - want).abs()
    assert (err <= bound).all(), f"dx: worst {(err / bound).max().item():.3f} x the bound"
    # channel sums (as_mean_var = 0, the bias gradient): no pivot, |sum - S| <= (chain + 4) u sum|x| + u |sum|
    s = F_.channel_sums(x)
    xs = x.double()
    S = xs.sum((0, 2, 3))
    es = (s.double() - S).abs()
    bs = (launch[2] + 4) * U * xs.abs().sum((0, 2, 3)) + U * S.abs()
    assert (es <= bs).all(), f"channel sums: worst {(es / bs).max().item():.3f} x the bound"


@pytest.mark.parametrize("shape,mean_over_std,misaligned,path", BN_SHAPES)
def test_bn_batch_stats_vs_fp64_and_running_updates(shape, mean_over_std, misaligned, path):
    """mnb_bn_batch_stats (the fused BatchNorm producers' training statistics): mean and invstd = (ss / N + eps)^-1/2
    against fp64, with |invstd - ref| <= invstd (bound(ss) / N / 2 / (var_b + eps) + 2 u); then three calls' running_mean,
    running_var and num_batches_tracked bit-exact against the fp32 update r = fl(fl((1 - m) r) + fl(m batch)) applied to
    the kernel's own batch statistics, read back (the unbiased variance through channel_mean_var, which runs the same
    partial sums and finaliser arithmetic)."""
    from micronet_b200 import _lib as L, functional as F_
    b, c, h, w = shape
    hw = h * w
    launch = _stats_launch(b, c, hw, not misaligned)
    assert launch == path, launch
    eps, mom = 1e-5, 0.1
    rm = torch.randn(c, generator=_gen(9), device=DEV)
    rv = torch.rand(c, generator=_gen(10), device=DEV) + 0.5
    nbt = torch.tensor(5, dtype=torch.int64, device=DEV)
    keep, m32 = torch.tensor(1.0) - torch.tensor(mom, dtype=torch.float32), torch.tensor(mom, dtype=torch.float32)
    want_m, want_v = rm.cpu(), rv.cpu()
    lib = L.load()
    for step in range(3):
        x = _stats_input(shape, mean_over_std, misaligned, seed=100 * step + c)
        stats = torch.empty(2 * c, device=DEV)
        L.check(lib.mnb_bn_batch_stats(x.data_ptr(), b, c, hw, eps, mom, rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(),
                                       stats.data_ptr(), L.scratch(x.device, c).data_ptr(), L.stream()), "bn_batch_stats")
        mean_k, var_k = F_.channel_mean_var(x)
        assert _eq(mean_k, stats[:c]), "channel_mean_var and bn_batch_stats disagree on the batch mean"
        if step == 0:
            ref = _stats_reference(x, launch)
            N = ref["N"]
            vb = ref["ss"] / N
            inv = 1.0 / torch.sqrt(vb + eps)
            assert ((stats[:c].double() - ref["mean"]).abs() <= ref["b_mean"]).all(), "mean"
            b_inv = inv * (ref["b_ss"] / N / 2 / (vb + eps) + 2 * U)
            e_inv = (stats[c:].double() - inv).abs()
            assert (e_inv <= b_inv).all(), f"invstd: worst {(e_inv / b_inv).max().item():.3f} x the bound"
        want_m = keep * want_m + m32 * mean_k.cpu()
        want_v = keep * want_v + m32 * var_k.cpu()
        assert _eq(rm, want_m), f"step {step}: running_mean {_first_diff(rm, want_m)}"
        assert _eq(rv, want_v), f"step {step}: running_var {_first_diff(rv, want_v)}"
        assert int(nbt.item()) == 6 + step


# ---------------------------------------------------------------- BatchNorm fold of QuantBNFuseConv2d (IAO:903-945)
# bn_fold_fwd/bwd_kernel: one 256-thread block per output channel, block-stride over the C/g * R * S weights of the row.
@pytest.mark.parametrize("wshape", [
    pytest.param((64, 3, 3, 3), id="stem-64x27-1pass"),
    pytest.param((64, 64, 3, 3), id="64x576-3passes"),
    pytest.param((128, 64, 1, 1), id="shortcut-128x64-1pass"),
    pytest.param((256, 128, 3, 3), id="256x1152-5passes"),
    pytest.param((512, 512, 3, 3), id="512x4608-18passes"),
])
@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
def test_bn_fold_vs_fp64_autograd(wshape, with_bias):
    """BNFoldFn (mnb_bn_fold_fwd / _bwd) against fp64 autograd of ratio = gamma / sqrt(var + eps), w_f = w * ratio,
    b_f = beta + (bias - mean) * ratio (beta - mean * ratio without bias).  Counting the fp32 roundings of each output
    (ratio = g / sqrt(var + eps): 2.5 u; the dot product dratio is an fp64 sum rounded once, plus the rounded
    bias - mean: 2 u) gives at most 7.5 u for dvar, the longest chain; every output is held to 12 u times the same
    expression evaluated on absolute values.  mnb_bn_fold_running: three calls (copy, then EMA) bit-exact against
    the fp32 formula r = fl(fl((1 - m) r) + fl(m batch))."""
    from micronet_b200 import _lib as L, functional as F_
    k = wshape[0]
    g = torch.Generator().manual_seed(k + (1 if with_bias else 0))
    w = torch.randn(wshape, generator=g) * 0.2
    bias = torch.randn(k, generator=g) if with_bias else None
    gamma, beta = torch.rand(k, generator=g) + 0.5, torch.randn(k, generator=g)
    mean, var = torch.randn(k, generator=g) * 3, torch.rand(k, generator=g) * 2 + 1e-3
    dwf, dbf = torch.randn(wshape, generator=g), torch.randn(k, generator=g)
    eps = 1e-5
    dev = [t.to(DEV).requires_grad_(True) if t is not None else None for t in (w, bias, gamma, beta, mean, var)]
    wf, bf = F_.BNFoldFn.apply(*dev, eps)
    torch.autograd.backward([wf, bf], [dwf.to(DEV), dbf.to(DEV)])
    r = [t.double().requires_grad_(True) if t is not None else None for t in (w, bias, gamma, beta, mean, var)]
    w6, b6, g6, be6, m6, v6 = r
    ratio = g6 / torch.sqrt(v6 + eps)
    wf6 = w6 * ratio.view(-1, 1, 1, 1)
    bf6 = be6 + (b6 - m6) * ratio if b6 is not None else be6 - m6 * ratio
    torch.autograd.backward([wf6, bf6], [dwf.double(), dbf.double()])
    # absolute-value evaluations (magnitudes the roundings are relative to)
    ra = ratio.detach().abs()
    diff_abs = (b6.detach().abs() if b6 is not None else 0) + m6.detach().abs()
    sq = torch.sqrt(v6.detach() + eps)
    Mr = (dwf.double() * w6.detach()).abs().sum((1, 2, 3)) + dbf.double().abs() * diff_abs
    checks = [
        ("w_f", wf, wf6, (w6.detach() * ra.view(-1, 1, 1, 1)).abs()),
        ("b_f", bf, bf6, be6.detach().abs() + diff_abs * ra),
        ("dw", dev[0].grad, w6.grad, (dwf.double() * ra.view(-1, 1, 1, 1)).abs()),
        ("dgamma", dev[2].grad, g6.grad, Mr / sq),
        ("dbeta", dev[3].grad, be6.grad, dbf.double().abs()),
        ("dmean", dev[4].grad, m6.grad, dbf.double().abs() * ra),
        ("dvar", dev[5].grad, v6.grad, 0.5 * Mr * g6.detach().abs() / (sq ** 3)),
    ]
    if with_bias:
        checks.append(("dbias", dev[1].grad, b6.grad, dbf.double().abs() * ra))
    for name, got, want, mag in checks:
        err = (got.detach().cpu().double() - want.detach()).abs()
        bound = 12 * U * mag + 1e-300
        assert (err <= bound).all(), f"{name}: worst {(err / bound).max().item():.3f} x the bound"
    # running statistics (IAO:858-876): first call copies, later calls r = (1 - m) r + m batch in fp32
    rm, rv = torch.zeros(k, device=DEV), torch.ones(k, device=DEV)
    mom = 0.1
    keep, m32 = torch.tensor(np.float32(1.0 - mom)), torch.tensor(np.float32(mom))
    want_m, want_v = None, None
    for step in range(3):
        bm, bv = torch.randn(k, generator=g) * 2, torch.rand(k, generator=g) + 0.1
        bm_d, bv_d = bm.to(DEV), bv.to(DEV)
        L.check(L.load().mnb_bn_fold_running(rm.data_ptr(), rv.data_ptr(), bm_d.data_ptr(), bv_d.data_ptr(),
                                             k, mom, 1 if step == 0 else 0, L.stream()), "bn_fold_running")
        torch.cuda.synchronize()
        want_m, want_v = (bm, bv) if step == 0 else (keep * want_m + m32 * bm, keep * want_v + m32 * bv)
        assert _eq(rm, want_m) and _eq(rv, want_v), f"running step {step}"
