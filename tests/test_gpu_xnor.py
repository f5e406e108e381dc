"""Bit-packed XNOR-popcount forward (csrc/mnb_xnor.cu) for wbwtab layers: exact integer sums against an fp64 convolution
of the +-1 / ternary operands, bit-identical outputs against the packed-operand tensor-core forward, and the module-level
result against the CPU oracle of WB.QuantConv2d (WB:181-195) within the 1e-5 contract."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as TF

from tests.oracle_util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# B, C, H, W, K, R, stride, pad, groups
SHAPES = [
    (3, 256, 32, 32, 256, 1, 1, 0, 2),     # NIN-GC 1x1 g2
    (3, 256, 16, 16, 512, 3, 1, 1, 16),    # NIN-GC 3x3 g16 (16 channels per group: half-used words)
    (3, 512, 16, 16, 512, 1, 1, 0, 4),
    (5, 512, 8, 8, 1024, 3, 1, 1, 32),
    (5, 1024, 8, 8, 1024, 1, 1, 0, 8),
    (2, 96, 16, 16, 192, 5, 1, 2, 2),      # 5x5, 48 channels per group (two words, ragged tail)
    (2, 64, 15, 13, 40, 3, 2, 1, 1),       # stride 2, odd image, K not a multiple of anything
    (2, 24, 9, 9, 12, 3, 1, 0, 1),         # 'valid' padding, 24 channels (ragged word)
    (2, 128, 7, 7, 64, 3, 1, 2, 1),        # padding wider than the usual 'same'
    (33, 32, 1, 1, 10, 1, 1, 0, 1),        # linear-layer view
]
IDS = ["x".join(map(str, s)) for s in SHAPES]


def _sh(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, st, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


@pytest.mark.parametrize("ternary", [False, True], ids=["binary", "ternary"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_xnor_sums_are_exact(shape, ternary):
    from micronet_b200 import _lib as L, xnor as X
    B, Cc, H, W, K, R, st, pad, G = shape
    g = torch.Generator().manual_seed(sum(shape) + int(ternary))
    x = torch.randn(B, Cc, H, W, generator=g)
    x[0, 0, 0, 0] = 0.0          # sign(0) -> +1 (WB:15-16)
    x[0, -1, -1, -1] = -0.0
    if ternary:
        w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g)
    else:
        w = torch.randint(0, 2, (K, Cc // G, R, R), generator=g) * 2 - 1
    a = torch.where(x < 0, -1.0, 1.0).double()
    ref = TF.conv2d(a, w.double(), None, st, pad, 1, G)
    sh = _sh(shape)
    assert X.supported(sh)
    bits = X.pack_act(x.to(DEV), G)
    img = X.pack_weight(sh, w.to(torch.int16).to(DEV))
    y = torch.full(ref.shape, float("nan"), device=DEV)
    L.check(X.conv(sh, bits, img, y), "xnor conv")
    assert torch.equal(y.cpu().double(), ref)
    alpha = (torch.rand(K, generator=g) * 0.05 + 0.01).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    L.check(X.conv(sh, bits, img, y, alpha=alpha, bias=bias), "xnor conv")
    want = torch.addcmul(bias.view(1, -1, 1, 1).cpu(), ref.float(), alpha.view(1, -1, 1, 1).cpu())   # one rounding, like fmaf
    assert rel_err(y, want) <= 2e-7


@pytest.mark.parametrize("shape", SHAPES[:5], ids=IDS[:5])
def test_xnor_equals_the_tensor_core_forward_bit_for_bit(shape):
    from micronet_b200 import _lib as L, pk as PK, xnor as X
    B, Cc, H, W, K, R, st, pad, G = shape
    g = torch.Generator().manual_seed(7 + sum(shape))
    x = torch.randn(B, Cc, H, W, generator=g).to(DEV)
    w_int = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g).to(torch.int16).to(DEV)
    alpha = (torch.rand(K, generator=g) * 0.05 + 0.01).to(DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    sh = _sh(shape)
    y_x = torch.empty(B, K, H, W, device=DEV)
    L.check(X.conv(sh, X.pack_act(x, G), X.pack_weight(sh, w_int), y_x, alpha=alpha, bias=bias), "xnor conv")
    pm1 = torch.where(x < 0, -1.0, 1.0)
    planes, _ = PK.pack_act(pm1, None, 1)
    y_t = torch.empty_like(y_x)
    L.check(PK.conv(sh, 0, planes, 1, PK.pack_weight(sh, 0, 1, 1, w_int=w_int), 1, y_t, n_scale=alpha, bias=bias), "pk conv")
    L.tc_check()
    assert torch.equal(y_x, y_t)


@pytest.mark.parametrize("W", [2, 3], ids=["binary", "ternary"])
def test_eval_module_takes_the_xnor_path_and_matches_the_oracle(W):
    """WB.QuantConv2d in eval mode (no autograd) on a +-1 input without a producer-written plane: the engine takes the XNOR
    forward; result vs the CPU oracle"""
    from micronet_b200 import functional as F_, wbwtab
    from oracle import reference_port as O
    torch.manual_seed(3 + W)
    conv_e = wbwtab.QuantConv2d(64, 96, 3, padding=1, groups=2, W=W)
    conv_o = O.WbQuantConv2d(64, 96, 3, padding=1, groups=2, W=W)
    conv_o.load_state_dict(conv_e.state_dict())
    x = torch.where(torch.randn(4, 64, 12, 12) < 0, -1.0, 1.0)
    conv_e.to(DEV).eval(); conv_o.eval()
    try:
        F_.TIMER = F_.KernelTimer()
        with torch.no_grad():
            xe = x.to(DEV)
            xe._mnb_pm1 = True
            ye = conv_e(xe)
        kinds = {k for k, _, _, _ in F_.TIMER.records}
    finally:
        F_.TIMER = None
    with torch.no_grad():
        yo = conv_o(x)
    assert "fwd_xnor" in kinds, kinds
    assert rel_err(ye, yo) <= 1e-5
