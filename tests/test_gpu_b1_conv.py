"""Binary tensor-core forward (csrc/mnb_b1.cu): fp32 outputs byte-equal to the packed-operand tensor-core forward and to the
XNOR kernel where it covers the shape, exact integer sums against fp64, the post epilogue's three output formats against
the un-fused sequence (BatchNorm -> sign -> pool -> shuffle -> packer), the plane max-pool against ATen, and the packers."""
import pytest
import torch
import torch.nn.functional as TF

from harness import models as zoo
from tests.test_gpu_wbwtab_frozen import _bn, _bn_sign

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# B, C, H, W, K, R, pad, groups
NIN = [
    (256, 192, 32, 32, 160, 1, 0, 1),
    (256, 160, 32, 32, 96, 1, 0, 1),
    (256, 96, 16, 16, 192, 5, 2, 1),
    (256, 192, 16, 16, 192, 1, 0, 1),
    (256, 192, 8, 8, 192, 3, 1, 1),
    (256, 192, 8, 8, 192, 1, 0, 1),
]
NINGC_1X1 = [
    (256, 256, 32, 32, 256, 1, 0, 2),
    (256, 512, 16, 16, 512, 1, 0, 4),
    (256, 1024, 8, 8, 1024, 1, 0, 8),
]
EDGE = [(1, c, 9, 13, k, 3, 1, 1) for c, k in ((1, 3), (63, 5), (64, 7), (65, 9), (127, 11), (160, 13), (192, 15))] + [
    (2, 70, 9, 13, 33, 7, 3, 1),      # 7x7 on a 9 x 13 plane
    (2, 64, 7, 7, 24, 7, 3, 1),       # 7x7 on 7 x 7
    (3, 96, 7, 7, 40, 5, 2, 1),       # 5x5 pad 2
    (3, 96, 7, 7, 40, 5, 0, 1),       # 5x5 pad 0
    (2, 130, 9, 13, 66, 3, 1, 2),     # two groups of 65 channels: the second group starts on a unit boundary
]
SHAPES = NIN + NINGC_1X1 + EDGE
IDS = ["x".join(map(str, s)) for s in SHAPES]


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _sh(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, pad, pad, 1, 1, G)


def _operands(shape, seed, ternary=True):
    B, Cc, H, W, K, R, pad, G = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cc, H, W, generator=g)
    x[0, 0, 0, 0] = 0.0          # sign(0) -> +1 (WB:15-16)
    x[0, -1, -1, -1] = -0.0
    if ternary:
        w = torch.randint(-1, 2, (K, Cc // G, R, R), generator=g)
        w[0] = 0                 # an all-zero output channel
    else:
        w = torch.randint(0, 2, (K, Cc // G, R, R), generator=g) * 2 - 1
    alpha = torch.rand(K, generator=g) * 0.05 + 0.01
    bias = torch.randn(K, generator=g)
    return x.to(DEV), w.to(torch.int16).to(DEV), alpha.to(DEV), bias.to(DEV), g


def _b1_fwd(shape, x, w, alpha, bias):
    from micronet_b200 import _lib as L, b1 as B1
    B, Cc, H, W, K, R, pad, G = shape
    sh = _sh(shape)
    assert B1.supported(sh)
    y = torch.full((B, K, H + 2 * pad - R + 1, W + 2 * pad - R + 1), float("nan"), device=DEV)
    L.check(B1.conv(sh, B1.pack_act(x, G), B1.pack_weight(sh, w), y, alpha=alpha, bias=bias), "b1 conv")
    return y


def _pk_fwd(shape, x, w, alpha, bias, out_shape):
    from micronet_b200 import _lib as L, pk as PK
    sh = _sh(shape)
    G = shape[7]
    pm1 = torch.where(x < 0, -1.0, 1.0)
    planes = PK.pack_act(pm1, None, 1, groups=G)[0]
    y = torch.empty(out_shape, device=DEV)
    L.check(PK.conv(sh, 0, planes, 1, PK.pack_weight(sh, 0, 1, 1, w_int=w), 1, y, n_scale=alpha, bias=bias), "pk conv")
    return y


@pytest.mark.parametrize("ternary", [False, True], ids=["binary", "ternary"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_b1_equals_the_tensor_core_forward_and_fp64(shape, ternary):
    from micronet_b200 import _lib as L, xnor as X
    B, Cc, H, W, K, R, pad, G = shape
    x, w, alpha, bias, _ = _operands(shape, sum(shape) + int(ternary), ternary)
    y = _b1_fwd(shape, x, w, alpha, bias)
    if B <= 4:   # exact integer sums (alpha = 1, no bias) against fp64
        a = torch.where(x < 0, -1.0, 1.0).double()
        ref = TF.conv2d(a, w.double(), None, 1, pad, 1, G)
        ones = torch.ones_like(alpha)
        assert torch.equal(_b1_fwd(shape, x, w, ones, None).double(), ref)
    assert torch.equal(y, _pk_fwd(shape, x, w, alpha, bias, y.shape))
    sh = _sh(shape)
    if X.supported(sh):
        y_x = torch.empty_like(y)
        L.check(X.conv(sh, X.pack_act(x, G), X.pack_weight(sh, w), y_x, alpha=alpha, bias=bias), "xnor conv")
        assert torch.equal(y, y_x)


def _post_case(shape, combo, seed):
    B, Cc, H, W, K, R, pad, G = shape
    x, w, alpha, bias, g = _operands(shape, seed)
    y = _b1_fwd(shape, x, w, alpha, bias)
    bn = _bn(K, g) if "bn" in combo else None
    pool = "pool" in combo
    sg = next(s for s in (4, 2, 1) if K % s == 0) if "shuffle" in combo else 1
    return x, w, alpha, bias, y, bn, pool, sg


def _signs(y, bn, pool, sg):
    s = _bn_sign(y, bn)
    if pool:
        s = TF.max_pool2d(s, 2, 2)
    if sg > 1:
        s = zoo.shuffle_channels(s, sg)
    return s.contiguous()


COMBOS = ["plain", "bn", "bn_pool", "bn_shuffle", "bn_pool_shuffle", "pool_shuffle"]
POST_SHAPES = [(4,) + s[1:] for s in NIN + NINGC_1X1] + EDGE[-3:]
POST_IDS = ["x".join(map(str, s)) for s in POST_SHAPES]


@pytest.mark.parametrize("combo", COMBOS)
@pytest.mark.parametrize("shape", POST_SHAPES, ids=POST_IDS)
def test_post_planes_decode_to_the_unfused_sequence(shape, combo):
    from micronet_b200 import _lib as L, b1 as B1, xnor as X
    B, Cc, H, W, K, R, pad, G = shape
    x, w, alpha, bias, y, bn, pool, sg = _post_case(shape, combo, sum(shape) + len(combo))
    sh = _sh(shape)
    plane_in, img = B1.pack_act(x, G), B1.pack_weight(sh, w)
    if pool and (y.shape[2] % 2 or y.shape[3] % 2):
        assert B1.post_bytes(sh, X.post_struct(L.XNOR_B1_PLANE, 1, sg, pool, bn)) == -1
        return
    want = _signs(y, bn, pool, sg)
    og = next(q for q in (3, 2, 1) if K % q == 0)        # the consumer's groups
    # b1 plane: decodes to the signs, and is byte-equal to the packer's plane of them (padding bits zero)
    post = X.post_struct(L.XNOR_B1_PLANE, og, sg, pool, bn)
    out = B1.empty_plane(B1.post_bytes(sh, post), DEV)
    out.fill_(-1)
    L.check(B1.conv_post(sh, plane_in, img, post, out, alpha=alpha, bias=bias), "b1 conv_post")
    assert torch.equal(B1.unpack(out, want.shape, og), want)
    assert torch.equal(out, B1.pack_act(want, og))
    # bit plane: byte-equal to the XNOR packer's bits of the signs (and to the XNOR kernel's own epilogue where it covers)
    post = X.post_struct(L.XNOR_BITS, og, sg, pool, bn)
    bits = torch.full((B1.post_bytes(sh, post) // 4,), -1, dtype=torch.int32, device=DEV)
    L.check(B1.conv_post(sh, plane_in, img, post, bits, alpha=alpha, bias=bias), "b1 conv_post bits")
    assert torch.equal(bits, X.pack_act(want, og))
    xsh = L.ConvShape(B, Cc, H, W, K, R, R, 1, 1, pad, pad, 1, 1, G)
    if X.supported(xsh):
        xb = torch.empty_like(bits)
        L.check(X.conv_post(xsh, X.pack_act(x, G), X.pack_weight(xsh, w), post, xb, alpha=alpha, bias=bias), "xnor conv_post")
        assert torch.equal(bits, xb)
    # bf16 +-1 plane [b][c/8][h][w][8] (no pool)
    if not pool and K % 8 == 0:
        post = X.post_struct(L.XNOR_PM1_BF16, 1, sg, False, bn)
        pm = torch.empty(B1.post_bytes(sh, post), dtype=torch.uint8, device=DEV)
        L.check(B1.conv_post(sh, plane_in, img, post, pm, alpha=alpha, bias=bias), "b1 conv_post bf16")
        b, c, h, ww = want.shape
        dec = pm.view(torch.bfloat16).view(b, c // 8, h, ww, 8).permute(0, 1, 4, 2, 3).reshape(b, c, h, ww).float()
        assert torch.equal(dec, want)


@pytest.mark.parametrize("hw", [32, 15])
@pytest.mark.parametrize("cg", [(96, 1), (192, 2), (160, 1)])
def test_plane_pool_is_atens_max_pool(hw, cg):
    from micronet_b200 import _lib as L, b1 as B1
    C, G = cg
    g = torch.Generator().manual_seed(hw + C)
    x = torch.randn(3, C, hw, hw, generator=g).to(DEV)
    plane = B1.pack_act(x, G)
    rc, out, oshape = B1.plane_maxpool(plane, x.shape, G, 3, 2, 1)
    L.check(rc, "b1 plane_maxpool")
    want = TF.max_pool2d(torch.where(x < 0, -1.0, 1.0), 3, 2, 1)
    assert oshape == tuple(want.shape) and oshape[2] == (hw + 1) // 2
    assert torch.equal(B1.unpack(out, oshape, G), want)
    assert torch.equal(out, B1.pack_act(want.contiguous(), G))


@pytest.mark.parametrize("combo", ["plain", "bn", "bn_pool", "bn_pool_shuffle"])
def test_packers_decode_to_the_signs(combo):
    from micronet_b200 import _lib as L, b1 as B1, xnor as X
    g = torch.Generator().manual_seed(len(combo))
    x = torch.randn(3, 192, 16, 16, generator=g)
    x[0, :8, 0, 0] = 0.0
    x[0, 8:16, 0, 0] = -0.0
    x[1, :4, 1, 1] = float("nan")
    x = x.to(DEV)
    want = torch.where(x < 0, -1.0, 1.0)
    for G in (1, 2, 3):
        assert torch.equal(B1.unpack(B1.pack_act(x, G), x.shape, G), want)
    bn = _bn(192, g) if "bn" in combo else None
    pool, sg = "pool" in combo, 4 if "shuffle" in combo else 1
    post = X.post_struct(L.XNOR_B1_PLANE, 2, sg, pool, bn)
    oshape = (3, 192, 8, 8) if pool else tuple(x.shape)
    out = B1.empty_plane(B1.act_bytes(*oshape, 2), DEV)
    L.check(B1.pack_act_post(x, post, out), "b1 pack_act_post")
    assert torch.equal(out, B1.pack_act(_signs(x, bn, pool, sg), 2))
