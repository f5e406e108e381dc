"""IAO.QuantConvTranspose2d (IAO:510-636, SURVEY 8 row f4) on the engine: functional.ConvTranspose2dFn runs the transposed
convolution as the data gradient of the mirrored convolution (tensor-core packed-operand family where it has cover, generic
kernels elsewhere).  The three golden cases generated from the reference run in test_gpu_parity.py::test_layer_case_matches_golden;
here: larger shapes against the CPU oracle / fp64 ATen, the kernel families actually taken, and prepare()."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as TF

from tests.oracle_util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# B, Cin, H, W, Cout, R, stride, pad, output_padding, groups, dilation
SHAPES = [
    (4, 64, 16, 16, 32, 4, 2, 1, 0, 1, 1),     # the usual 2x up-sampling decoder layer
    (3, 32, 8, 8, 64, 3, 2, 1, 1, 1, 1),       # output_padding
    (2, 64, 12, 12, 64, 3, 1, 1, 0, 2, 1),     # stride 1, groups
    (2, 16, 7, 9, 24, 3, 1, 0, 0, 1, 2),       # dilation 2: outside the tensor-core cover -> generic kernels
    (2, 6, 5, 5, 4, 5, 3, 2, 2, 1, 1),         # few channels, stride 3
]
IDS = ["x".join(map(str, s)) for s in SHAPES]


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_conv_transpose_fn_matches_fp64(shape):
    from micronet_b200 import _lib as L, functional as F_
    B, Ci, H, W, Co, R, st, pad, op, G, dil = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Ci, Co // G, R, R, generator=g) * 0.2
    bias = torch.randn(Co, generator=g)
    xe, we, be = (t.to(DEV).requires_grad_(True) for t in (x, w, bias))
    F_.TIMER = F_.KernelTimer()
    try:
        y = F_.conv_transpose2d(xe, we, be, (st, st), (pad, pad), (op, op), G, (dil, dil))
        go = torch.randn(y.shape, generator=g)
        y.backward(go.to(DEV))
        torch.cuda.synchronize()
        kinds = {k for k, _, _, _ in F_.TIMER.records}
    finally:
        F_.TIMER = None
    L.tc_check()
    xd, wd, bd = (t.double().requires_grad_(True) for t in (x, w, bias))
    yd = TF.conv_transpose2d(xd, wd, bd, st, pad, op, G, dil)
    yd.backward(go.double())
    assert y.shape == yd.shape
    assert rel_err(y.detach(), yd.detach()) <= 3e-6
    assert rel_err(xe.grad, xd.grad) <= 1e-5
    assert rel_err(we.grad, wd.grad) <= 1e-5
    assert rel_err(be.grad, bd.grad) <= 1e-5
    if dil == 1 and Ci >= 16:
        assert {"dgrad_pk", "fwd_pk", "wgrad_pk"} <= kinds, kinds       # the tensor-core family, roles swapped
        assert not {"dgrad", "fwd", "wgrad"} & kinds, kinds             # (a _pk kind is recorded even when it refused)
    if dil == 2:
        assert {"dgrad", "fwd", "wgrad"} <= kinds, kinds


@pytest.mark.parametrize("q_type", [0, 1], ids=["sym", "asym"])
def test_quant_conv_transpose_module_matches_the_oracle(q_type):
    from micronet_b200 import iao
    from oracle import reference_port as O
    torch.manual_seed(10 + q_type)
    kw = dict(stride=2, padding=1, output_padding=1, q_type=q_type)
    me = iao.QuantConvTranspose2d(32, 48, 3, **kw)
    mo = O.IaoQuantConvTranspose2d(32, 48, 3, **kw)
    mo.load_state_dict(me.state_dict())
    me.to(DEV).train(); mo.train()
    for step in range(3):
        x = torch.randn(4, 32, 10, 10) * (1.0 + 0.3 * step)
        xe, xo = x.to(DEV).requires_grad_(True), x.clone().requires_grad_(True)
        ye, yo = me(xe), mo(xo)
        go = torch.randn(yo.shape)
        me.zero_grad(); mo.zero_grad()
        ye.backward(go.to(DEV)); yo.backward(go)
        assert rel_err(ye.detach(), yo.detach()) <= 1e-5, step
        assert rel_err(xe.grad, xo.grad) <= 1e-5, step
        assert rel_err(me.weight.grad, mo.weight.grad) <= 1e-5, step
        assert rel_err(me.bias.grad, mo.bias.grad) <= 1e-5, step
        so = mo.state_dict()
        for k, v in me.state_dict().items():     # observer ranges, scales, zero-points: bit-exact
            if "quantizer" in k:
                assert torch.equal(v.cpu(), so[k]), (step, k)
    me.eval(); mo.eval()
    x = torch.randn(2, 32, 10, 10)
    with torch.no_grad():
        assert rel_err(me(x.to(DEV)), mo(x)) <= 1e-5


def test_prepare_replaces_conv_transpose():
    from micronet_b200 import iao
    from oracle import reference_port as O
    torch.manual_seed(3)
    net = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.ConvTranspose2d(16, 8, 4, stride=2, padding=1))
    eng = iao.prepare(copy.deepcopy(net), inplace=True).to(DEV)
    assert isinstance(eng[2], iao.QuantConvTranspose2d)
    assert set(eng.state_dict().keys()) >= {"2.weight", "2.bias", "2.activation_quantizer.scale", "2.weight_quantizer.scale"}
    ora = nn.Sequential(O.IaoQuantConv2d(3, 16, 3, padding=1), nn.ReLU(), O.IaoQuantConvTranspose2d(16, 8, 4, stride=2, padding=1))
    ora.load_state_dict(eng.state_dict())
    eng.train(); ora.train()
    x = torch.randn(2, 3, 12, 12)
    ye, yo = eng(x.to(DEV)), ora(x)
    assert ye.shape == (2, 8, 24, 24) and rel_err(ye.detach(), yo.detach()) <= 1e-5
