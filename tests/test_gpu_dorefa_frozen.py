"""Frozen DoReFa inference graphs on level planes (dorefa.freeze_inference): the consumer epilogue of the packed-operand
convolution with BatchNorm, ReLU and channel shuffle (mnb_pk_conv_post / mnb_pk_i8_conv) byte for byte against the fp32
output -> mnb_bn_relu_quant_pack_fwd composition, the plane max-pool against torch.max_pool2d of the decoded levels, whole
NIN / NIN-GC models bitwise against a block-by-block composition of existing kernels, the fused graph bitwise against its
un-frozen eval forward, the ATen-BatchNorm graph teacher-forced, and the deployment graph against the oracle."""
import copy
import zlib

import pytest
import torch

from harness import models as zoo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _stats(K, g):
    mean = (torch.randn(K, generator=g) * 0.5).to(DEV)
    var = (torch.rand(K, generator=g) * 2 + 0.05).to(DEV)
    gamma = torch.randn(K, generator=g).to(DEV)
    beta = (torch.randn(K, generator=g) * 2).to(DEV)
    return mean, torch.rsqrt(var + 1e-5), gamma, beta


def _spec(bits):
    from micronet_b200 import _lib as L, functional as F_
    return F_.ActSpec(L.ACT_DOREFA, bits=bits)


def _bn_relu_plane(y, bn, bits, sg, i8):
    """the un-fused producer: eval BatchNorm + ReLU + DoReFa quantizer (+ shuffle) from the fp32 conv output"""
    import ctypes as C
    from micronet_b200 import _lib as L, pk as PK
    b, c, h, w = y.shape
    qp = _spec(bits).struct()
    args = [t.data_ptr() for t in bn]
    lib = L.load()
    if i8:
        out = PK.consumer_plane_i8(b, c, h, w, y.device)
        L.check(lib.mnb_bn_relu_quant_pack_i8_fwd(y.data_ptr(), b, c, h * w, *args, C.byref(qp), sg, out.data_ptr(), L.stream()),
                "bn_relu_quant_pack_i8_fwd")
    else:
        out = PK.consumer_plane(b, c, h, w, y.device)
        bits_ = torch.empty((y.numel() + 31) // 32, dtype=torch.int32, device=y.device)
        L.check(lib.mnb_bn_relu_quant_pack_fwd(y.data_ptr(), b, c, h * w, *args, C.byref(qp), sg, out.data_ptr(),
                                               bits_.data_ptr(), L.stream()), "bn_relu_quant_pack_fwd")
    return out


def _pack(x, bits, i8):
    from micronet_b200 import pk as PK
    if i8:
        return PK.pack_act_i8(x.contiguous(), _spec(bits).struct())
    return PK.pack_act(x.contiguous(), _spec(bits).struct(), 1)[0]


def _conv(sh, plane, w_int, w_scale, a_bits, bias, i8, y=None, post=None):
    from micronet_b200 import _lib as L, pk as PK
    a_const = 1.0 / float(2 ** a_bits - 1)
    if i8:
        img = PK.pack_weight_i8(sh, w_int)
        rc = PK.conv_i8(sh, plane, img, y, n_scale=w_scale, a_scale_const=a_const, bias=bias, post=post)
    else:
        img = PK.pack_weight(sh, 0, 1, 1, w_int=w_int)
        if post is None:
            rc = PK.conv(sh, 0, plane, 1, img, 1, y, n_scale=w_scale, a_scale_const=a_const, bias=bias)
        else:
            qp, cplane, relu, split, bn, sg = post
            rc = PK.conv_post(sh, plane, 1, img, 1, y, qp, cplane, relu, split, n_scale=w_scale, a_scale_const=a_const, bias=bias,
                              bn=bn, shuffle_groups=sg)
    L.check(rc, "pk conv")


# (name, C, H, K, R, pad, groups, shuffle groups of the consumer): NIN and NIN-GC layers
SHAPES = [("nin_l1", 192, 32, 160, 1, 0, 1, 2), ("nin_l3", 96, 16, 192, 5, 2, 1, 2), ("nin_l6", 192, 8, 192, 3, 1, 1, 2),
          ("gc_l1", 256, 32, 256, 1, 0, 2, 2), ("gc_l3", 256, 16, 512, 3, 1, 16, 16), ("gc_l4", 512, 16, 512, 1, 0, 4, 4),
          ("gc_l6", 512, 8, 1024, 3, 1, 32, 32), ("gc_l7", 1024, 8, 1024, 1, 0, 8, 8)]


@pytest.mark.parametrize("combo", ["plain", "bn", "bn_relu", "bn_relu_shuffle"])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_epilogue_plane_matches_the_composition(shape, i8, combo):
    from micronet_b200 import _lib as L, pk as PK
    name, Cc, H, K, R, pad, G, sg = shape
    bits = 4 if i8 or name.startswith("gc") else 8
    g = torch.Generator().manual_seed(zlib.crc32((name + combo).encode()))
    n = 2 ** bits - 1
    B = 2
    x = (torch.rand(B, Cc, H, H, generator=g) * 12 - 1).to(DEV)
    w_int = (torch.randint(0, n + 1, (K, Cc // G, R, R), generator=g) * 2 - n).to(torch.int16).to(DEV)
    w_scale = torch.full((K,), 1.0 / n, device=DEV)
    bias = torch.randn(K, generator=g).to(DEV)
    bn = _stats(K, g)
    sh = L.ConvShape(B, Cc, H, H, K, R, R, 1, 1, pad, pad, 1, 1, G)
    plane = _pack(x, bits, i8)
    y = torch.empty(B, K, H, H, device=DEV)
    _conv(sh, plane, w_int, w_scale, bits, bias, i8, y=y)
    use_bn, relu, s = combo != "plain", "relu" in combo, sg if "shuffle" in combo else 1
    # reference: mnb_bn_relu_quant_pack_fwd from the fp32 output (DoReFa's clamp at 0 makes the ReLU a no-op on the levels,
    # so "bn" compares against it too); without a BatchNorm the consumer's own packer
    ref = _bn_relu_plane(y, bn, bits, s, i8) if use_bn else _pack(y, bits, i8)
    out = (PK.consumer_plane_i8 if i8 else PK.consumer_plane)(B, K, H, H, DEV)
    out.fill_(0x5a)
    y2 = torch.empty_like(y)
    post = (_spec(bits).struct(), out, relu, False, bn if use_bn else None, s)
    _conv(sh, plane, w_int, w_scale, bits, bias, i8, y=y2, post=post)
    torch.cuda.synchronize()
    assert torch.equal(y2, y)
    assert torch.equal(out, ref), (out != ref).sum().item()


def _decode(plane, b, c, h, w, i8):
    u = 16 if i8 else 8
    v = plane.view(torch.int8 if i8 else torch.bfloat16).view(b, c // u, h, w, u)
    return v.permute(0, 1, 4, 2, 3).reshape(b, c, h, w).float()


def _encode(lev, i8):
    b, c, h, w = lev.shape
    u = 16 if i8 else 8
    t = lev.view(b, c // u, u, h, w).permute(0, 1, 3, 4, 2).contiguous()
    return (t.to(torch.int8) if i8 else t.to(torch.bfloat16)).view(torch.uint8).reshape(-1)


@pytest.mark.parametrize("kps", [(3, 2, 1), (2, 2, 0)])
@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_plane_pool_matches_max_pool_of_the_levels(kps, i8):
    from micronet_b200 import pk as PK
    k, s, p = kps
    b, c, h, w = 3, 96 if not i8 else 112, 32, 32
    g = torch.Generator().manual_seed(7)
    x = (torch.rand(b, c, h, w, generator=g) * 11).to(DEV)
    plane = _pack(x, 4 if i8 else 8, i8)
    out = PK.plane_maxpool(plane, b, c, h, w, k, s, p, int8=i8)
    ref = _encode(torch.nn.functional.max_pool2d(_decode(plane, b, c, h, w, i8), k, s, p), i8)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def _model(kind, a_bits, w_bits, fuse=False, pools=True, deploy=False):
    from micronet_b200 import dorefa as DF
    torch.manual_seed(3)
    base = zoo.init_like_reference(zoo.NIN() if kind == "nin" else zoo.NINGC())
    g = torch.Generator().manual_seed(11)
    for m in base.modules():
        if isinstance(m, torch.nn.BatchNorm2d):     # non-trivial running statistics and affine parameters
            k = m.num_features
            m.running_mean.copy_(torch.randn(k, generator=g) * 0.3)
            m.running_var.copy_(torch.rand(k, generator=g) * 2 + 0.2)
            m.weight.data.copy_(torch.randn(k, generator=g) * 0.5 + 1.5)
            m.bias.data.copy_(torch.randn(k, generator=g) * 2 + 3)
    if not pools:
        for name, m in list(base.model.named_children()):
            if isinstance(m, torch.nn.MaxPool2d):
                base.model._modules[name] = torch.nn.Identity()
    m = DF.prepare(base, a_bits=a_bits, w_bits=w_bits, fuse=fuse, quant_inference=deploy).to(DEV).eval()
    return m


def _reference_logits(m, x, a_bits, i8):
    """the frozen graph evaluated block by block through existing kernels: packed conv fp32 -> mnb_bn_relu_quant_pack_fwd
    (running statistics, next block's shuffle) -> max-pool of the decoded levels -> the next conv on that plane"""
    from micronet_b200 import dorefa as DF, functional as F_
    kids = list(m.model.children())
    with torch.no_grad():
        y = kids[0].conv(x)
        plane, shape, i = None, None, 0
        while True:
            blk = kids[i]
            j = i + 1
            pool = kids[j] if isinstance(kids[j], torch.nn.MaxPool2d) else None
            j += pool is not None
            nxt = kids[j]
            if not hasattr(nxt, "channel_shuffle_flag"):
                out = blk.relu(blk.bn(y))
                return kids[j](out).view(x.shape[0], -1)
            sg = nxt.shuffle_groups if nxt.channel_shuffle_flag else 1
            mean, invstd = blk.bn.running_mean, torch.rsqrt(blk.bn.running_var + blk.bn.eps)
            plane = _bn_relu_plane(y, (mean, invstd, blk.bn.weight, blk.bn.bias), a_bits, sg, i8)
            b, c, h, w = y.shape
            if pool is not None:
                k, s, p = pool.kernel_size, pool.stride, pool.padding
                lev = torch.nn.functional.max_pool2d(_decode(plane, b, c, h, w, i8), k, s, p)
                plane, (h, w) = _encode(lev, i8), lev.shape[2:]
            conv = nxt.conv
            _, w_int, w_scale = DF.frozen_levels(conv)
            sh = F_._shape_struct((b, c, h, w), conv.weight.shape, conv.stride, conv.padding, conv.dilation, conv.groups)
            y = torch.empty((b, conv.out_channels, h, w), device=DEV)
            _conv(sh, plane, w_int, w_scale, a_bits, conv.bias, i8, y=y)
            i = j


def _graph_logits(m, x):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            m(x)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr), torch.no_grad():
        out = m(x)
    gr.replay()
    torch.cuda.synchronize()
    return out.clone()


# batch 256: the batch the benchmark runs the NIN models at
@pytest.mark.parametrize("kind,a,w,i8,batch", [("nin", 8, 8, False, 8), ("gc", 4, 4, False, 8), ("gc", 4, 4, True, 8),
                                               ("nin", 8, 8, False, 256), ("gc", 4, 4, False, 256), ("gc", 4, 4, True, 256)],
                         ids=["nin_w8a8", "gc_w4a4", "gc_w4a4_int8", "nin_w8a8_b256", "gc_w4a4_b256", "gc_w4a4_int8_b256"])
def test_frozen_logits_equal_the_block_composition(kind, a, w, i8, batch):
    from harness import train as H
    from micronet_b200 import dorefa as DF
    m = _model(kind, a, w)
    x, _ = H.synthetic_batch(batch, 32, seed=4, device=DEV)
    ref = _reference_logits(m, x, a, i8)
    DF.freeze_inference(m, int8=i8)
    with torch.no_grad():
        got = m(x)
    torch.cuda.synchronize()
    assert torch.equal(got, ref), (got - ref).abs().max().item()
    assert torch.equal(_graph_logits(m, x), ref)
    DF.freeze_inference(m, enable=False)


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_fused_graph_bitwise_against_unfrozen(i8):
    """prepare(fuse=True) without pools: every absorbed block ran BatchNormReluQuant2d un-frozen, the same op sequence"""
    from harness import train as H
    from micronet_b200 import dorefa as DF
    m = _model("gc", 4, 4, fuse=True, pools=False)
    x, _ = H.synthetic_batch(4, 32, seed=5, device=DEV)
    with torch.no_grad():
        ref = m(x)
    DF.freeze_inference(m, int8=i8)
    with torch.no_grad():
        got = m(x)
    torch.cuda.synchronize()
    assert torch.equal(got, ref), (got - ref).abs().max().item()
    assert torch.equal(_graph_logits(m, x), ref)
    DF.freeze_inference(m, enable=False)


def test_aten_batchnorm_levels_teacher_forced():
    """where the un-frozen graph ran ATen's eval BatchNorm, each block's levels equal the frozen producer's except where the
    fp32 BatchNorm output lies within 2 ulp of a level boundary (DESIGN.md 4.15)"""
    from harness import train as H
    m = _model("nin", 8, 8)
    x, _ = H.synthetic_batch(8, 32, seed=6, device=DEV)
    outs = []
    hooks = [blk.conv.register_forward_hook(lambda mod, i, o: outs.append(o.detach().clone()))
             for blk in m.model.children() if hasattr(blk, "channel_shuffle_flag")]
    with torch.no_grad():
        m(x)
    for hk in hooks:
        hk.remove()
    blocks = [b for b in m.model.children() if hasattr(b, "channel_shuffle_flag")]
    n = 255.0
    excused = total = 0
    for blk, y in zip(blocks[:-1], outs[:-1]):
        bn = blk.bn
        with torch.no_grad():
            a = torch.relu(bn(y))
        b, c, h, w = y.shape
        mine = _decode(_bn_relu_plane(y, (bn.running_mean, torch.rsqrt(bn.running_var + bn.eps), bn.weight, bn.bias), 8, 1,
                                      False), b, c, h, w, False)
        theirs = _decode(_pack(a, 8, False), b, c, h, w, False)
        diff = mine != theirs
        total += a.numel()
        if diff.any():
            ad = a[diff].double()
            k = torch.floor(ad * 0.1 * n)                        # the boundary between level k and k + 1
            bound = (k + 0.5) / n * 10
            ulp = (torch.nextafter(ad.float(), torch.full_like(ad.float(), float("inf"))) - ad.float()).double()
            assert bool(((ad - bound).abs() <= 2 * ulp).all())
            assert bool(((mine[diff] - theirs[diff]).abs() == 1).all())
            excused += int(diff.sum())
    print(f"excused levels: {excused} of {total}")


def test_deployment_graph_against_the_oracle():
    """prepare(quant_inference=True) + bn_fuse.dorefa_quantize_inference_weights: each frozen conv, fed the oracle's input of
    that layer, within 1e-5 relative of the oracle port's output (teacher-forced, layer by layer)"""
    from harness import train as H
    from micronet_b200 import bn_fuse, dorefa as DF, functional as F_
    from oracle import reference_port as RP
    m = _model("gc", 4, 4, deploy=True)
    bn_fuse.dorefa_quantize_inference_weights(m)
    base = copy.deepcopy(m).cpu()
    ora = RP.prepare_dorefa(zoo.NINGC(), a_bits=4, w_bits=4, quant_inference=True)
    ora.load_state_dict(base.state_dict())
    ora.eval()
    seen = []
    convs = [c for c in ora.modules() if isinstance(c, torch.nn.Conv2d)][1:]
    hooks = [c.register_forward_hook(lambda mod, i, o: seen.append((i[0].detach(), o.detach()))) for c in convs]
    x, _ = H.synthetic_batch(4, 32, seed=8, device="cpu")
    with torch.no_grad():
        ora(x)
    for hk in hooks:
        hk.remove()
    DF.freeze_inference(m)
    mine = [c for c in m.modules() if isinstance(c, DF.QuantConv2d)]
    assert len(mine) == len(seen) and all("_mnb_frozen" in c.__dict__ for c in mine)
    for c, (inp, out) in zip(mine, seen):
        wq, w_int, w_scale, bias = DF._frozen_operands(c)
        y = F_.frozen_conv(inp.to(DEV), None, wq, bias, w_int, w_scale, c.activation_quantizer.spec(), c.stride, c.padding,
                           c.dilation, c.groups)
        err = (y.cpu() - out).abs().max() / out.abs().max()
        assert err < 1e-5, err
    DF.freeze_inference(m, enable=False)


def test_no_fp32_intermediates():
    """a frozen NIN-GC forward launches packed-conv posts, plane pools, the stem producer, the stem and head convs and the
    avg-pool, and allocates no fp32 activation between the stem producer and the head"""
    from harness import train as H
    from micronet_b200 import dorefa as DF, functional as F_
    m = _model("gc", 4, 4, fuse=True)
    x, _ = H.synthetic_batch(8, 32, seed=9, device=DEV)
    DF.freeze_inference(m, int8=True)
    with torch.no_grad():
        m(x)
    F_.TIMER = F_.KernelTimer()
    try:
        with torch.no_grad():
            m(x)
        torch.cuda.synchronize()
        kinds = [k for k, *_ in F_.TIMER.records]
    finally:
        F_.TIMER = None
    assert kinds.count("plane_pool") == 2
    assert set(kinds) <= {"fwd_pk", "fwd_pk_i8", "plane_pool"}, kinds
    # fp32 activations allocated on the device: only the stem conv's output and the head conv's
    sizes = []
    orig = torch.empty

    def spy(*a, **k):
        t = orig(*a, **k)
        if t.dtype == torch.float32 and t.device.type == "cuda" and t.dim() == 4:
            sizes.append(tuple(t.shape))
        return t
    torch.empty = spy
    try:
        with torch.no_grad():
            m(x)
    finally:
        torch.empty = orig
    assert sorted(sizes) == [(8, 10, 8, 8), (8, 256, 32, 32)], sizes
