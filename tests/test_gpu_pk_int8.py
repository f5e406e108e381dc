"""int8 operands of the packed-operand family (mnb_pk_i8_*, iao.freeze_inference(int8=True)) on the H100.

* the kernel at every plan it can take: the "i8" cases of tests/pk_conv_cases.py in test_gpu_pk_conv_fp64.py (bit for bit
  the fp64 sum's fmaf(S, scale, bias) and mnb_pk_conv's result on the same levels);
* above 2^24: the s32 sum is exact and rounded once;
* packers and hand-offs: pack_act_i8 holds the levels of the bf16 plane, the consumer-plane epilogue and
  mnb_quant_add_pack_i8_fwd write exactly pack_act_i8 of their fp32 result;
* models: freeze_inference(int8=True) logits are bitwise equal to freeze_inference() and to the plain eval forward."""
import collections
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

def _iao_spec(scale, bits=8):
    from micronet_b200 import _lib as L, functional as F_
    half = 1 << (bits - 1)
    bufs = dict(scale=torch.tensor([scale]), zero_point=torch.zeros(1), obs_min=torch.tensor([-(half - 0.5) * scale]),
                obs_max=torch.tensor([(half - 0.5) * scale]))
    return F_.ActSpec(L.ACT_IAO, bits=bits, qmin=-half, qmax=half - 1, q_type=0, **{k: v.to(DEV) for k, v in bufs.items()})


def _levels_i8(plane, B, Cc, H, W, split=False):
    """int8 plane -> levels [B, C, H, W] (split: [B, 4, C, H/2, W/2])"""
    u = -(-Cc // 16)
    v = plane.view(torch.int8).float()
    if split:
        return v.view(B, 4, u, H // 2, W // 2, 16).permute(0, 1, 2, 5, 3, 4).reshape(B, 4, u * 16, H // 2, W // 2)[:, :, :Cc]
    return v.view(B, u, H, W, 16).permute(0, 1, 4, 2, 3).reshape(B, u * 16, H, W)[:, :Cc]


def _levels_bf16(plane, B, Cc, H, W, split=False):
    o = -(-Cc // 8)
    v = plane.view(torch.bfloat16).float()
    if split:
        return v.view(B, 4, o, H // 2, W // 2, 8).permute(0, 1, 2, 5, 3, 4).reshape(B, 4, o * 8, H // 2, W // 2)[:, :, :Cc]
    return v.view(B, o, H, W, 8).permute(0, 1, 4, 2, 3).reshape(B, o * 8, H, W)[:, :Cc]


def _case_operands(B, Cc, H, W, K, R, st, pad, G, seed, extreme=False):
    from micronet_b200 import _lib as L
    g = torch.Generator(device=DEV).manual_seed(seed)
    if extreme:   # levels at and next to the extremes: every product in [126^2, 128 x 127], sums of arbitrary parity
        xl = -128.0 + torch.randint(0, 2, (B, Cc, H, W), generator=g, device=DEV).float()
        w_int = (-127 + torch.randint(0, 2, (K, Cc // G, R, R), generator=g, device=DEV)).to(torch.int16)
        w_scale, bias = torch.ones(K, device=DEV), torch.zeros(K, device=DEV)
    else:
        xl = torch.randint(-128, 128, (B, Cc, H, W), generator=g, device=DEV).float()
        w_int = torch.randint(-127, 128, (K, Cc // G, R, R), generator=g, device=DEV, dtype=torch.int16)
        w_scale = torch.rand(K, generator=g, device=DEV) * 0.01 + 0.001
        bias = torch.randn(K, generator=g, device=DEV)
    sh = L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)
    return sh, xl, w_int, w_scale, bias


def _run_case(shape, seed=11, extreme=False):
    """(int8 result, bf16 result, exact fp64 sum) of one shape (B, C, H, W, K, R, stride, pad, groups); asserts the repeat
    is bitwise identical"""
    from micronet_b200 import _lib as L, pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    sh, xl, w_int, w_scale, bias = _case_operands(B, Cc, H, W, K, R, st, pad, G, seed, extreme)
    spec = _iao_spec(1.0)                    # scale 1: the levels are the input values themselves
    a_scale = torch.ones(1, device=DEV)
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    x8 = PK.pack_act_i8(xl, spec.struct(), phase_split=st == 2)
    w8 = PK.pack_weight_i8(sh, w_int)
    outs = []
    for _ in range(2):
        y = torch.full((B, K, P, Q), float("nan"), device=DEV)
        L.check(PK.conv_i8(sh, x8, w8, y, n_scale=w_scale, a_scale=a_scale, bias=bias), "pk_i8_conv")
        outs.append(y)
    xb, _ = PK.pack_act(xl, spec.struct(), 1, phase_split=st == 2)
    wb = PK.pack_weight(sh, 0, 1, 1, w_int=w_int)
    yb = torch.full((B, K, P, Q), float("nan"), device=DEV)
    L.check(PK.conv(sh, 0, xb, 1, wb, 1, yb, n_scale=w_scale, a_scale=a_scale, bias=bias), "pk_conv")
    torch.cuda.synchronize()
    L.tc_check()
    assert torch.equal(outs[0], outs[1]), "the repeat differs"
    s64 = torch.nn.functional.conv2d(xl.double(), w_int.double(), stride=st, padding=pad, groups=G)
    return outs[0], yb, s64, w_scale, bias


def test_sums_above_2_24_are_exact_and_rounded_once():
    """sums of ~7.4e7 that fp32 cannot hold: the s32 accumulators keep them exact, so the result is the exact sum rounded
    once (scale 1, bias 0), where an fp32 accumulation (the bf16 kernel's) rounds its partial sums on the way"""
    y8, yb, s64, _, _ = _run_case((1, 512, 8, 8, 64, 3, 1, 1, 1), extreme=True)
    assert s64.abs().min().item() > 2 ** 24                         # >= 512 x 4 x 126^2 even in the corners
    want = s64.float()                                              # the exact integer sum rounded once to fp32
    assert (want.double() != s64).float().mean().item() > 0.5       # most exact sums are not fp32 numbers
    assert torch.equal(y8, want), (y8 != want).sum().item()         # __int2float_rn is that single rounding
    assert not torch.equal(yb, want), "the fp32-accumulating bf16 kernel was expected to round some partial sums"


def test_pack_act_i8_holds_the_bf16_planes_levels():
    from micronet_b200 import pk as PK
    torch.manual_seed(3)
    B, Cc, H, W = 3, 40, 10, 12
    x = torch.randn(B, Cc, H, W, device=DEV) * 4
    spec = _iao_spec(0.05)
    for relu in (False, True):
        for split in (False, True):
            p8 = PK.pack_act_i8(x, spec.struct(), phase_split=split, relu=relu)
            pb, _ = PK.pack_act(x, spec.struct(), 1, phase_split=split, relu=relu)
            assert torch.equal(_levels_i8(p8, B, Cc, H, W, split), _levels_bf16(pb, B, Cc, H, W, split)), (relu, split)
            u = -(-Cc // 16)
            last = p8.view(torch.int8).view(B, 4 if split else 1, u, -1, 16)[:, :, -1, :, Cc % 16:]
            assert not last.any(), "channels beyond C must be zero"


def test_consumer_plane_epilogue_and_quant_add_write_pack_act_i8():
    from micronet_b200 import _lib as L, functional as F_, pk as PK
    torch.manual_seed(5)
    B, Cc, H, W, K = 4, 64, 16, 16, 96
    x = torch.randn(B, Cc, H, W, device=DEV) * 3
    w_int = torch.randint(-127, 128, (K, Cc, 3, 3), dtype=torch.int16, device=DEV)
    w_scale = torch.rand(K, device=DEV) * 0.01 + 0.001
    bias = torch.randn(K, device=DEV)
    spec, nxt = _iao_spec(0.05), _iao_spec(0.11)
    sh = L.ConvShape(B, Cc, H, W, K, 3, 3, 1, 1, 1, 1, 1, 1, 1)
    x8 = PK.pack_act_i8(x, spec.struct())
    w8 = PK.pack_weight_i8(sh, w_int)
    y_ref = torch.empty(B, K, H, W, device=DEV)
    L.check(PK.conv_i8(sh, x8, w8, y_ref, n_scale=w_scale, a_scale=spec.scale, bias=bias), "conv_i8")
    for relu in (False, True):
        for split in (False, True):
            want = PK.pack_act_i8(y_ref, nxt.struct(), phase_split=split, relu=relu)
            for with_out in (True, False):
                y = torch.full_like(y_ref, float("nan")) if with_out else None
                plane = PK.consumer_plane_i8(B, K, H, W, DEV)
                L.check(PK.conv_i8(sh, x8, w8, y, n_scale=w_scale, a_scale=spec.scale, bias=bias,
                                   post=(nxt.struct(), plane, relu, split)), "conv_i8 post")
                assert torch.equal(plane, want), (relu, split, with_out)
                if with_out:
                    assert torch.equal(y, y_ref)
    a, b = torch.randn(B, K, H, W, device=DEV) * 4, torch.randn(B, K, H, W, device=DEV) * 4
    add = _iao_spec(0.07)
    lib = L.load()
    for relu in (False, True):
        ref = F_.QuantAddFn.apply(a, b, add, relu)
        for split in (False, True):
            for next_relu in (False, True):
                want = PK.pack_act_i8(ref, nxt.struct(), phase_split=split, relu=next_relu)
                out = torch.full_like(a, float("nan"))
                plane = PK.consumer_plane_i8(B, K, H, W, DEV)
                qp, cqp = add.struct(), nxt.struct()
                post = L.PkPost(C.pointer(cqp), 1 if next_relu else 0, 1 if split else 0, plane.data_ptr())
                L.check(lib.mnb_quant_add_pack_i8_fwd(a.data_ptr(), b.data_ptr(), B, K, H, W, C.byref(qp), 1 if relu else 0,
                                                      out.data_ptr(), C.byref(post), L.stream()), "quant_add_pack_i8")
                assert torch.equal(out, ref) and torch.equal(plane, want), (relu, split, next_relu)
    L.tc_check()


# ---------------------------------------------------------------------------------------------------------------- models
PTQ = dict(a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0, bn_fuse=True, pretrained_model=True, ptq=True,
           percentile=0.999999)


def _resnet(widths, hw, seed=4, **over):
    from harness import models as zoo, train as H
    torch.manual_seed(seed)
    base = zoo.init_like_reference(zoo.ResNet(widths=widths))
    with torch.no_grad():
        for m in base.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.2); m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5); m.bias.normal_(0, 0.2)
    eng = H.prepare_engine(base, "iao", **dict(PTQ, **over)).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    return eng, torch.randn(2, 3, hw, hw, generator=g), torch.randn(2, 3, hw, hw, generator=g)


def _ningc(seed=6):
    from harness import models as zoo, train as H
    torch.manual_seed(seed)
    base = zoo.init_like_reference(zoo.NINGC())
    eng = H.prepare_engine(base, "iao", a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    return eng, torch.randn(4, 3, 32, 32, generator=g), torch.randn(4, 3, 32, 32, generator=g)


def _quant_convs(model):
    from micronet_b200 import iao
    return [m for m in model.modules() if isinstance(m, iao.QuantConv2d)]


def _compare(eng, calib, x, expect_i8=True, extra_launches=0):
    """plain eval vs freeze_inference() vs freeze_inference(int8=True): bitwise equal logits, equal launch counts, and
    (expect_i8) an fwd_pk_i8 timer record for every quantized conv inside the int8 cover"""
    from micronet_b200 import iao, _lib as L, functional as F_, pk as PK
    xd = x.to(DEV)
    with torch.no_grad():
        eng.train(); eng(calib.to(DEV)); eng.eval()
        plain = eng(xd).clone()
        iao.freeze_inference(eng)
        bf = eng(xd).clone()
        n0 = L.launch_count(); eng(xd); n_bf = L.launch_count() - n0
        iao.freeze_inference(eng, int8=True)
        i8a = eng(xd).clone()
        n0 = L.launch_count(); i8b = eng(xd).clone(); n_i8 = L.launch_count() - n0
        shapes = []
        hooks = [m.register_forward_pre_hook(lambda mod, inp, m=m: shapes.append((m, tuple(inp[0].shape))))
                 for m in _quant_convs(eng)]
        F_.TIMER = F_.KernelTimer()
        try:
            eng(xd)
            torch.cuda.synchronize()
            kinds = collections.Counter(k for k, *_ in F_.TIMER.records)
        finally:
            F_.TIMER = None
            for h in hooks:
                h.remove()
        cover = sum(iao._int8_ok(m) and m.activation_quantizer.q_type == 0 and
                    PK.i8_supported(F_._shape_struct(s, tuple(m.weight.shape), tuple(m.stride), tuple(m.padding),
                                                     tuple(m.dilation), m.groups)) for m, s in shapes)
        iao.freeze_inference(eng, enable=False)
    L.tc_check()
    assert torch.equal(plain, bf), "bf16 frozen path differs from the eval forward"
    assert torch.equal(i8a, plain) and torch.equal(i8b, plain), (i8a - plain).abs().max().item()
    assert n_i8 == n_bf + extra_launches, (n_i8, n_bf)
    # every quantized conv in the cover (symmetric IAO activations, s8 weights, a shape the int8 plan takes) ran int8
    assert kinds["fwd_pk_i8"] == cover, (kinds, cover, len(shapes))
    if expect_i8:
        assert cover == len(shapes), (cover, len(shapes))
    else:
        assert cover == 0 and kinds["fwd_pk_i8"] == 0, kinds
    return plain


@pytest.mark.parametrize("name,over", [("per_channel", {}), ("per_layer", dict(q_level=1)),
                                       ("w4a4", dict(a_bits=4, w_bits=4))])
def test_frozen_int8_resnet_is_bit_identical(name, over):
    eng, calib, x = _resnet((16, 32, 64, 128), 64, **over)
    _compare(eng, calib, x)


def test_frozen_int8_resnet18_at_224_is_bit_identical():
    eng, calib, x = _resnet((64, 128, 256, 512), 224)
    _compare(eng, calib, x)


def test_frozen_int8_resnet18_at_224_bench_batch_is_bit_identical():
    """the ResNet-18 PTQ graph at 224 x 64, the batch of the benchmark's inference metric: bf16 and int8 frozen logits equal
    the un-frozen eval forward bit for bit"""
    eng, calib, _ = _resnet((64, 128, 256, 512), 224)
    x = torch.randn(64, 3, 224, 224, generator=torch.Generator().manual_seed(64))
    _compare(eng, calib, x)


def test_frozen_int8_ningc_is_bit_identical():
    eng, calib, x = _ningc()
    _compare(eng, calib, x)


def test_grouped_producer_with_8_outputs_per_group_hands_off_no_int8_plane():
    """16 in / 8 out channels per group: the int8 conv takes it, but its epilogue cannot write whole 16-channel units of the
    consumer's int8 plane (the bf16 epilogue writes 8-channel octets and hands off): the producer writes fp32 and the
    consumer packs its own plane - one launch more than the bf16 frozen graph, same logits"""
    from harness import train as H
    torch.manual_seed(8)
    nn = torch.nn
    base = nn.Sequential(nn.Conv2d(16, 64, 3, padding=1), nn.ReLU(), nn.Conv2d(64, 32, 3, padding=1, groups=4), nn.ReLU(),
                         nn.Conv2d(32, 64, 3, padding=1))
    eng = H.prepare_engine(base, "iao", a_bits=8, w_bits=8, q_type=0, q_level=0, weight_observer=0).to(DEV)
    g = torch.Generator().manual_seed(9)
    _compare(eng, torch.randn(4, 16, 16, 16, generator=g), torch.randn(4, 16, 16, 16, generator=g), extra_launches=1)


def test_asymmetric_model_runs_no_int8_kernel():
    eng, calib, x = _resnet((16, 32, 64, 128), 64, q_type=1, ptq=False, percentile=0.9999)
    _compare(eng, calib, x, expect_i8=False)


def test_cuda_graph_replay_gives_the_eager_result():
    from harness import train as H
    from micronet_b200 import iao
    eng, calib, x = _resnet((16, 32, 64, 128), 64)
    st = H.InferStepper(eng, graph=True)
    st.calibrate([calib.to(DEV)])
    iao.freeze_inference(eng, int8=True)
    xd = x.to(DEV)
    with torch.no_grad():
        eager = eng(xd).clone()
    outs = [st.step(xd).clone() for _ in range(4)]
    assert st.graph is not None, st.graph_error
    for o in outs:
        assert torch.equal(o, eager)
