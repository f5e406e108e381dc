"""The int16 hand-off between a wbwtab conv and its fused BatchNorm + binarizer (mnb_pk_conv_codes and the _codes producers).

* every _codes producer, on random int16 codes and a random decode pair, writes byte for byte what its fp32 namesake writes
  when fed the decoded tensor (mnb_codes_decode): statistics and running statistics, pass bits, +-1 output and operand
  plane, arg-max bytes, dgamma / dbeta / dx / channel sums, packed gradient pieces - at the planes of the bench model's
  seven wbwtab convs (batch 256, with their folded shuffles and pools) and at edge planes that take the VEC 2 / VEC 1 /
  scalar paths;
* mnb_pk_conv_codes decoded equals mnb_pk_conv's fp32 output bit for bit at the plans of L1..L7, and its decode pair is the
  epilogue's (weight scale, bias);
* shapes outside the int16 cover are refused with MNB_E_UNSUPPORTED and the layer falls back to the fp32 output;
* fused NIN-GC QAT steps with codes_out set and cleared give bit-identical losses, gradients, parameters and statistics."""
import copy

import pytest
import torch

from micronet_b200 import _lib as L, functional as F_, pk as PK

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (batch, channels, H, W, out_shuffle_groups, pooled) of the BatchNorm producers behind L1..L7 of the bench model, then edges
BENCH = [(256, 256, 32, 32, 2, False), (256, 256, 32, 32, 2, True), (256, 512, 16, 16, 16, False),
         (256, 512, 16, 16, 4, False), (256, 512, 16, 16, 4, True), (256, 1024, 8, 8, 32, False),
         (256, 1024, 8, 8, 1, False)]
EDGES = [(6, 16, 4, 8, 2, False),      # H*W = 32: VEC 1 of the packed kernels
         (5, 24, 8, 8, 1, False),      # H*W = 64: VEC 2
         (3, 16, 5, 5, 1, False),      # H*W = 25: scalar reduce / apply, no packed form
         (3, 16, 6, 8, 2, True)]       # pooled, odd number of window pairs per row


def _t(n, dtype=torch.float32):
    return torch.empty(n, dtype=dtype, device=DEV)


def _random_codes(shape, seed, bound=144):
    g = torch.Generator(device=DEV).manual_seed(seed)
    codes = torch.randint(-bound, bound + 1, shape, generator=g, device=DEV, dtype=torch.int32).to(torch.int16)
    c = shape[1]
    dec = torch.cat([torch.rand(c, generator=g, device=DEV) * 0.02 + 1e-3, torch.randn(c, generator=g, device=DEV) * 0.3])
    return codes, dec


def _decode(codes, dec):
    b, c = codes.shape[0], codes.shape[1]
    x = torch.empty(codes.shape, dtype=torch.float32, device=DEV)
    L.check(L.load().mnb_codes_decode(codes.data_ptr(), dec.data_ptr(), b, c, codes.numel() // (b * c), x.data_ptr(),
                                      L.stream()), "codes_decode")
    return x


def _same(a, b, what):
    a, b = a.reshape(-1).contiguous().view(torch.uint8), b.reshape(-1).contiguous().view(torch.uint8)
    bad = (a != b).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.numel()} bytes differ, first at {bad[0].item()}"


def _both(fn32, fncodes, x, codes, dec, outs_factory, call):
    """call(fn, xargs, outs) for the fp32 form on x and the _codes form on (codes, dec), each with fresh outputs"""
    o32, oc = outs_factory(), outs_factory()
    call(fn32, (x.data_ptr(),), o32)
    call(fncodes, (codes.data_ptr(), dec.data_ptr()), oc)
    torch.cuda.synchronize()
    return o32, oc


def _bn_params(c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    mean = torch.randn(c, generator=g, device=DEV) * 0.5
    invstd = torch.rand(c, generator=g, device=DEV) * 2 + 0.5
    gamma = torch.randn(c, generator=g, device=DEV)
    beta = torch.randn(c, generator=g, device=DEV) * 0.3
    return mean, invstd, gamma, beta


@pytest.mark.parametrize("shape", BENCH + EDGES, ids=lambda s: "x".join(map(str, s[:4])) + f"_sg{s[4]}" + ("_pool" if s[5] else ""))
def test_codes_producers_match_fp32_forms(shape):
    B, Cc, H, W, sg, pooled = shape
    hw, n = H * W, B * Cc * H * W
    lib = L.load()
    codes, dec = _random_codes((B, Cc, H, W), seed=B * 7 + Cc + hw)
    x = _decode(codes, dec)
    mean, invstd, gamma, beta = _bn_params(Cc, seed=Cc + hw)
    st = L.stream()
    scratch = L.scratch(torch.device(DEV), Cc)

    # batch statistics (+ running statistics and step counter)
    def stats_outs():
        return [_t(2 * Cc), torch.full((Cc,), 0.25, device=DEV), torch.full((Cc,), 2.0, device=DEV),
                torch.zeros(1, dtype=torch.int64, device=DEV)]
    o32, oc = _both(lib.mnb_bn_batch_stats, lib.mnb_bn_batch_stats_codes, x, codes, dec, stats_outs,
                    lambda fn, xa, o: L.check(fn(*xa, B, Cc, hw, 1e-5, 0.1, o[1].data_ptr(), o[2].data_ptr(), o[3].data_ptr(),
                                                 o[0].data_ptr(), scratch.data_ptr(), st), "stats"))
    for a, b, w in zip(o32, oc, ("mean_invstd", "running_mean", "running_var", "num_batches_tracked")):
        _same(a, b, w)

    bits_words = (n + 31) // 32
    if pooled:
        def fwd_outs():
            return [_t(n // 4), _t(bits_words, torch.int32), _t(n // 4, torch.uint8)]
        o32, oc = _both(lib.mnb_bn_sign_pool_fwd, lib.mnb_bn_sign_pool_fwd_codes, x, codes, dec, fwd_outs,
                        lambda fn, xa, o: L.check(fn(*xa, B, Cc, H, W, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                                     beta.data_ptr(), sg, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(),
                                                     st), "pool fwd"))
        for a, b, w in zip(o32, oc, ("y", "bits", "argmax")):
            _same(a, b, w)
        bits, arg = o32[1], o32[2]
        g = torch.randn(n // 4, device=DEV)
        for training in (1, 0, 2):
            def bwd_outs():
                return [_t(n), _t(3 * Cc)]
            o32, oc = _both(lib.mnb_bn_sign_pool_bwd, lib.mnb_bn_sign_pool_bwd_codes, x, codes, dec, bwd_outs,
                            lambda fn, xa, o: L.check(fn(g.data_ptr(), bits.data_ptr(), arg.data_ptr(), *xa, B, Cc, H, W,
                                                         mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), training, sg,
                                                         o[0].data_ptr(), o[1].data_ptr(), o[1][Cc:].data_ptr(),
                                                         None if training == 2 else o[1][2 * Cc:].data_ptr(),
                                                         scratch.data_ptr(), st), "pool bwd"))
            _same(o32[1][:2 * Cc], oc[1][:2 * Cc], f"dgamma / dbeta, training {training}")
            if training != 2:
                _same(o32[0], oc[0], f"dx, training {training}")
                _same(o32[1][2 * Cc:], oc[1][2 * Cc:], f"dx channel sums, training {training}")
        dgb = o32[1]
        for T in (1, 2):
            o32, oc = _both(lib.mnb_bn_sign_pool_bwd_pack, lib.mnb_bn_sign_pool_bwd_pack_codes, x, codes, dec,
                            lambda: [_t(T * n * 2, torch.uint8)],
                            lambda fn, xa, o: L.check(fn(g.data_ptr(), bits.data_ptr(), arg.data_ptr(), *xa, B, Cc, H, W,
                                                         mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), dgb.data_ptr(),
                                                         dgb[Cc:].data_ptr(), sg, invstd.data_ptr(), T, o[0].data_ptr(), st),
                                                      "pool bwd pack"))
            _same(o32[0], oc[0], f"packed gradient, {T} pieces")
        return

    packed = Cc % 8 == 0 and hw % 32 == 0
    if packed:
        for with_y in (True, False):
            def fwd_outs():
                return [_t(n), _t(bits_words, torch.int32), _t(n * 2, torch.uint8)]
            o32, oc = _both(lib.mnb_bn_sign_fwd_packed, lib.mnb_bn_sign_fwd_packed_codes, x, codes, dec, fwd_outs,
                            lambda fn, xa, o: L.check(fn(*xa, B, Cc, hw, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                                         beta.data_ptr(), sg, o[0].data_ptr() if with_y else None,
                                                         o[1].data_ptr(), o[2].data_ptr(), st), "packed fwd"))
            for a, b, w in zip(o32 if with_y else o32[1:], oc if with_y else oc[1:], ("y", "bits", "plane")[0 if with_y else 1:]):
                _same(a, b, w)
        bits = o32[1]
    else:
        bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (bits_words,), dtype=torch.int32, device=DEV)
    g = torch.randn(n, device=DEV)
    for training in (1, 0, 2):
        o32, oc = _both(lib.mnb_bn_sign_bwd, lib.mnb_bn_sign_bwd_codes, x, codes, dec, lambda: [_t(n), _t(3 * Cc)],
                        lambda fn, xa, o: L.check(fn(g.data_ptr(), bits.data_ptr(), *xa, B, Cc, hw, mean.data_ptr(),
                                                     invstd.data_ptr(), gamma.data_ptr(), training, sg, o[0].data_ptr(),
                                                     o[1].data_ptr(), o[1][Cc:].data_ptr(),
                                                     None if training == 2 else o[1][2 * Cc:].data_ptr(), scratch.data_ptr(),
                                                     st), "bwd"))
        _same(o32[1][:2 * Cc], oc[1][:2 * Cc], f"dgamma / dbeta, training {training}")
        if training != 2:
            _same(o32[0], oc[0], f"dx, training {training}")
            _same(o32[1][2 * Cc:], oc[1][2 * Cc:], f"dx channel sums, training {training}")
    dgb = o32[1]
    if packed:
        for T in (1, 2):
            for with_dx in (True, False):
                o32, oc = _both(lib.mnb_bn_sign_bwd_pack, lib.mnb_bn_sign_bwd_pack_codes, x, codes, dec,
                                lambda: [_t(T * n * 2, torch.uint8), _t(n)],
                                lambda fn, xa, o: L.check(fn(g.data_ptr(), bits.data_ptr(), *xa, B, Cc, hw, mean.data_ptr(),
                                                             invstd.data_ptr(), gamma.data_ptr(), dgb.data_ptr(),
                                                             dgb[Cc:].data_ptr(), sg, invstd.data_ptr(), T,
                                                             o[1].data_ptr() if with_dx else None, o[0].data_ptr(), st),
                                                          "bwd pack"))
                _same(o32[0], oc[0], f"packed gradient, {T} pieces")
                if with_dx:
                    _same(o32[1], oc[1], "dx of the pack pass")


# (C_in, H, K, R, groups) of L1..L7 at batch 256
CONVS = [(256, 32, 256, 1, 2), (256, 32, 256, 1, 2), (256, 16, 512, 3, 16), (512, 16, 512, 1, 4), (512, 16, 512, 1, 4),
         (512, 8, 1024, 3, 32), (1024, 8, 1024, 1, 8)]


def _conv_operands(cin, h, k, r, groups, batch=256, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sh = L.ConvShape(batch, cin, h, h, k, r, r, 1, 1, r // 2, r // 2, 1, 1, groups)
    x = torch.where(torch.rand(batch, cin, h, h, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    w_int = torch.randint(-1, 2, (k, cin // groups, r, r), generator=g, device=DEV, dtype=torch.int32).to(torch.int16)
    w_scale = torch.rand(k, generator=g, device=DEV) * 0.05 + 1e-3
    bias = torch.randn(k, generator=g, device=DEV) * 0.1
    return sh, x, w_int, w_scale, bias


@pytest.mark.parametrize("layer", range(1, 8), ids=lambda i: f"L{i}")
def test_conv_codes_decode_to_the_fp32_output(layer):
    cin, h, k, r, groups = CONVS[layer - 1]
    sh, x, w_int, w_scale, bias = _conv_operands(cin, h, k, r, groups, seed=layer)
    assert PK.supported(sh, 0, 1, 1) and not PK.segmented(sh, 0, 1, 1) and PK.codes_fit(cin, groups, r)
    x_pk, _ = PK.pack_act(x, None, 1)
    w_img = PK.pack_weight(sh, 0, 1, 1, w_int=w_int)
    y = torch.empty(256, k, h, h, device=DEV)
    L.check(PK.conv(sh, 0, x_pk, 1, w_img, 1, y, n_scale=w_scale, bias=bias), "pk_conv")
    codes = torch.full((256, k, h, h), 12345, dtype=torch.int16, device=DEV)
    dec = torch.full((2 * k,), float("nan"), device=DEV)
    L.check(PK.conv_codes(sh, x_pk, w_img, codes, dec, n_scale=w_scale, bias=bias), "pk_conv_codes")
    torch.cuda.synchronize()
    L.tc_check()
    _same(dec[:k], w_scale, "decode scale")
    _same(dec[k:], bias, "decode bias")
    assert codes.abs().max().item() <= (cin // groups) * r * r
    _same(_decode(codes, dec), y, f"L{layer} decoded codes vs fp32 output")


def test_conv_codes_refusals_fall_back_to_fp32():
    lib = L.load()
    # over the int16 bound: 4096 x 3 x 3 terms of level 1 (host check, before any plan or launch)
    sh = L.ConvShape(2, 4096, 4, 4, 16, 3, 3, 1, 1, 1, 1, 1, 1, 1)
    codes, dec = _t(2 * 16 * 16, torch.int16), _t(32)
    dummy = _t(64)
    rc = lib.mnb_pk_conv_codes(sh, dummy.data_ptr(), 1, dummy.data_ptr(), 1, None, None, 1.0, None, 1, codes.data_ptr(),
                               dec.data_ptr(), L.tc_err_flag(torch.device(DEV)).data_ptr(), L.stream())
    assert rc == L.E_UNSUPPORTED
    # two-piece operands (the plan itself is supported) and a segmented plan
    sh, x, w_int, w_scale, bias = _conv_operands(64, 8, 64, 3, 1, batch=4, seed=9)
    x_pk, _ = PK.pack_act(x, None, 2)
    w_img = PK.pack_weight(sh, 0, 2, 1, w_int=w_int)
    rc = lib.mnb_pk_conv_codes(sh, x_pk.data_ptr(), 2, w_img.data_ptr(), 1, w_scale.data_ptr(), None, 1.0, bias.data_ptr(), 1,
                               codes.data_ptr(), dec.data_ptr(), L.tc_err_flag(torch.device(DEV)).data_ptr(), L.stream())
    assert rc == L.E_UNSUPPORTED
    seg = next(((tA, tW) for tA, tW in ((3, 3), (2, 3), (3, 2)) if PK.segmented(sh, 0, tA, tW)), None)
    if seg is not None:
        rc = lib.mnb_pk_conv_codes(sh, x_pk.data_ptr(), seg[0], w_img.data_ptr(), seg[1], None, None, 1.0, None, 1,
                                   codes.data_ptr(), dec.data_ptr(), L.tc_err_flag(torch.device(DEV)).data_ptr(), L.stream())
        assert rc == L.E_UNSUPPORTED
    # the layer: a marked conv over the bound writes its fp32 output, identical to the unmarked one
    from micronet_b200 import wbwtab
    torch.manual_seed(3)
    conv = wbwtab.QuantConv2d(4096, 16, 3, padding=1, W=3).to(DEV)
    xin = torch.where(torch.rand(2, 4096, 8, 8, device=DEV) < 0.5, -1.0, 1.0)
    outs = []
    for flag in (True, False):
        conv.codes_out = flag
        xi = xin.clone()
        xi._mnb_pm1 = True
        y = conv(xi)
        assert getattr(y, "_mnb_codes", None) is None
        outs.append(y.detach().clone())
    _same(outs[0], outs[1], "fallback output")


def _step_model(codes_out, base):
    from harness import train as H
    m = copy.deepcopy(base)
    from micronet_b200 import wbwtab
    n = 0
    for mod in m.modules():
        if isinstance(mod, wbwtab.QuantConv2d) and mod.codes_out:
            n += 1
            mod.codes_out = codes_out
    assert n == 7, n
    return m.to(DEV), H.QatStepper(m, lr=0.01, wd=0.0, flat=True, graph=False)


def test_qat_steps_identical_with_and_without_codes():
    from harness import train as H
    from micronet_b200.fused import BatchNormBinarize2d
    base = H.prepare_engine(H.build_float_model("nin_gc"), "wbwtab", W=3, A=2, fuse_bn=True)
    batches = [H.synthetic_batch(64, 32, seed=40 + i, device=DEV) for i in range(3)]
    runs = {}
    for flag in (True, False):
        model, stepper = _step_model(flag, base)
        seen = []
        hooks = [m.register_forward_pre_hook(lambda mod, inp: seen.append(getattr(inp[0], "_mnb_codes", None) is not None))
                 for m in model.modules() if isinstance(m, BatchNormBinarize2d)]
        losses = [stepper.step(x, t).detach().clone() for x, t in batches]
        torch.cuda.synchronize()
        for h in hooks:
            h.remove()
        assert sum(seen) == (7 * len(batches) if flag else 0), seen
        runs[flag] = (losses, {k: v.detach().clone() for k, v in model.state_dict().items()},
                      {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None})
    (l1, s1, g1), (l0, s0, g0) = runs[True], runs[False]
    for a, b in zip(l1, l0):
        _same(a, b, "loss")
    assert s1.keys() == s0.keys() and g1.keys() == g0.keys() and len(g1) > 0
    for k in s1:
        _same(s1[k], s0[k], k)
    for k in g1:
        _same(g1[k], g0[k], "grad " + k)
    # the decode rebuilds a marked conv's output as its fp32 epilogue would have written it
    model, _ = _step_model(True, base)
    model.train()
    block = model.model[1]
    captured = {}
    block.bn.register_forward_pre_hook(lambda mod, inp: captured.setdefault("x", inp[0]))
    x0 = batches[0][0]
    model(x0)
    y_codes = F_.materialized(captured["x"])
    block.conv.codes_out = False
    captured.clear()
    model(x0)
    _same(y_codes, captured["x"], "materialized codes")
