"""Packers and module path of the packed-operand tensor-core family (csrc/mnb_pk.cu): the activation packer's bf16
pieces, its fused quantizer and STE flags against the standalone kernels, and QuantConv2dFn end to end on the packed
family.  The convolutions themselves are held against fp64 at every case of tests/pk_conv_cases.py by
test_gpu_pk_conv_fp64.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _unpack(planes, terms, B, Cc, H, W):
    c8 = (Cc + 7) // 8
    t = planes.view(torch.bfloat16).view(terms, B, c8, H, W, 8).float().sum(0)
    return t.permute(0, 1, 4, 2, 3).reshape(B, c8 * 8, H, W)[:, :Cc]


def test_pack_act_planes_hold_exact_pieces():
    from micronet_b200 import pk as PK
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(3, 19, 6, 10, generator=g) * 3).to(DEV)
    for terms in (1, 2, 3):
        planes, _ = PK.pack_act(x, None, terms)
        back = _unpack(planes, terms, 3, 19, 6, 10)
        err = (back - x).abs().max().item() / x.abs().max().item()
        assert err <= (2.0 ** -8, 2.0 ** -16, 0.0)[terms - 1] * 1.01, (terms, err)
    sc = (torch.rand(19, generator=g) + 0.5).to(DEV)
    planes, _ = PK.pack_act(x, None, 3, ch_scale=sc)
    assert torch.equal(_unpack(planes, 3, 3, 19, 6, 10), x * sc.view(1, -1, 1, 1))
    # phase split: octet (h%2*2 + w%2)*C8 + c/8 of an [H/2, W/2] plane
    planes, _ = PK.pack_act(x, None, 3, phase_split=True)
    ph = planes.view(torch.bfloat16).view(3, 3, 4, 3, 3, 5, 8).float().sum(0)      # [b][phase][c8][h/2][w/2][8]
    for a in range(2):
        for b in range(2):
            got = ph[:, a * 2 + b].permute(0, 1, 4, 2, 3).reshape(3, 24, 3, 5)[:, :19]
            assert torch.equal(got, x[:, :, a::2, b::2])


@pytest.mark.parametrize("mode", ["dorefa4", "dorefa8", "iao_sym", "iao_asym"])
def test_pack_act_quantizer_matches_the_standalone_kernel(mode):
    from micronet_b200 import _lib as L, functional as F_, pk as PK
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(2, 24, 8, 8, generator=g) * 4).to(DEV)
    if mode.startswith("dorefa"):
        spec = F_.ActSpec(L.ACT_DOREFA, bits=int(mode[6:]))
        terms, scale, zp = 1, 1.0 / (2 ** int(mode[6:]) - 1), 0.0
    else:
        sym = mode == "iao_sym"
        s = torch.tensor([0.037], device=DEV)
        z = torch.tensor([0.0 if sym else -101.0], device=DEV)
        lo, hi = torch.tensor([-4.5], device=DEV), torch.tensor([4.9], device=DEV)
        spec = F_.ActSpec(L.ACT_IAO, bits=8, qmin=-128 if sym else 0, qmax=127 if sym else 255, q_type=0 if sym else 1,
                          scale=s, zero_point=z, obs_min=lo, obs_max=hi)
        terms, scale, zp = (1 if sym else 2), 0.037, z.item()
    codes, bits, xq = F_.act_quant_raw(x, spec, True, True, True)
    qp = spec.struct()
    planes, bits8 = PK.pack_act(x, qp, terms, want_bits=True)
    lev = _unpack(planes, terms, 2, 24, 8, 8)
    want = codes.float() + spec.code_offset + zp
    assert torch.equal(lev, want)
    # STE flags: bit j of bits8[b, c/8, h, w] = flat NCHW bit of channel 8*(c/8) + j
    flat = bits.view(torch.int32)
    idx = torch.arange(x.numel(), device=DEV)
    passed = ((flat[idx // 32] >> (idx % 32)) & 1).view(x.shape).bool()
    got = torch.stack([(bits8 >> j) & 1 for j in range(8)], dim=2).reshape(2, 24, 8, 8).bool()
    assert torch.equal(got, passed)


def test_module_path_uses_the_packed_family_for_resnet_shapes():
    """QuantConv2dFn end to end (IAO symmetric quantizer, stride 2) against the generic CUDA-core kernels"""
    from micronet_b200 import _lib as L, functional as F_
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(4, 64, 16, 16, generator=g) * 2).to(DEV)
    w_int = torch.randint(-127, 128, (128, 64, 3, 3), generator=g, dtype=torch.int16).to(DEV)
    w_scale = (torch.rand(128, generator=g) * 0.02 + 0.001).to(DEV)
    wq = w_int.float() * w_scale.view(-1, 1, 1, 1)
    bias = torch.randn(128, generator=g).to(DEV)
    s, z = torch.tensor([0.04], device=DEV), torch.tensor([0.0], device=DEV)
    lo, hi = torch.tensor([-5.0], device=DEV), torch.tensor([5.1], device=DEV)
    spec = F_.ActSpec(L.ACT_IAO, bits=8, qmin=-128, qmax=127, q_type=0, scale=s, zero_point=z, obs_min=lo, obs_max=hi)
    gy = torch.randn(4, 128, 8, 8, generator=g).to(DEV)
    res = {}
    for mode in ("auto", "off"):
        L.PK_MODE = mode
        try:
            F_.TIMER = F_.KernelTimer()
            xg, wg = x.clone().requires_grad_(True), wq.clone().requires_grad_(True)
            y = F_.quant_conv2d(xg, wg, bias, w_int, w_scale, spec, (2, 2), (1, 1), (1, 1), 1)
            y.backward(gy)
            torch.cuda.synchronize()
            kinds = {k for k, _, _, _ in F_.TIMER.records}
            res[mode] = (y.detach(), xg.grad, wg.grad, kinds)
        finally:
            L.PK_MODE = "auto"
            F_.TIMER = None
    assert {"fwd_pk", "dgrad_pk", "wgrad_pk"} <= res["auto"][3], res["auto"][3]
    assert not any(k.endswith("_pk") for k in res["off"][3])
    for a, b, tol in zip(res["auto"][:3], res["off"][:3], (1e-6, 1e-5, 1e-5)):
        assert (a - b).abs().max().item() <= tol * b.abs().max().item()
    L.tc_check()
