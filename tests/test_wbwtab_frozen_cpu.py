"""CPU side of frozen wbwtab inference graphs (wbwtab.freeze_inference, mnb_xnor_conv_post / mnb_xnor_pack_act_post):
host refusals of the new entry points (fake device pointers: nothing may be launched), a numpy model of where the epilogue
puts each sign bit (consumer group / word / bit under a channel shuffle and a folded 2x2 pool), and the graph rewrite on
CPU-built models - which layers freeze, which modules are switched off, and that ``enable=False`` restores everything."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from harness import models as zoo

CFG = [32, 32, 32, 64, 64, 64, 256, 256]     # head 256 -> 10: EnginePmConv2d, as at full width
FAKE = 1 << 20          # never dereferenced: every call below is refused on the host


def _post(fmt=0, groups=1, sg=1, pool=0, bn=False):
    from micronet_b200 import _lib as L
    p = [FAKE] * 4 if bn else [None] * 4
    return L.XnorPost(fmt, groups, sg, pool, *p)


def _sh(B=2, C_=64, H=8, W=8, K=64, R=1, pad=0, groups=2):
    from micronet_b200 import _lib as L
    return L.ConvShape(B, C_, H, W, K, R, R, 1, 1, pad, pad, 1, 1, groups)


def test_conv_post_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()

    def call(sh, post):
        return lib.mnb_xnor_conv_post(C.byref(sh), FAKE, FAKE, None, None, None if post is None else C.byref(post), FAKE, None)

    n0 = L.launch_count()
    assert call(_sh(), None) == -1                                     # no consumer description
    assert call(_sh(), _post(fmt=7)) == -1                             # unknown format
    assert call(_sh(), _post(groups=3)) == -1                          # consumer groups do not divide 64
    assert call(_sh(), _post(sg=5)) == -1                              # shuffle groups do not divide 64
    bad_bn = _post()
    bad_bn.bn_mean = FAKE                                              # one of four BatchNorm pointers
    assert call(_sh(), bad_bn) == -1
    assert call(_sh(H=7, W=8), _post(pool=1)) == -2                    # pool over an odd plane
    assert call(_sh(), _post(fmt=1, pool=1)) == -2                     # bf16 plane with a pool
    assert call(_sh(K=60, groups=2), _post(fmt=1)) == -2               # bf16 plane needs C % 8 == 0
    assert call(_sh(R=7, pad=3), _post()) == -2                        # conv shape outside the XNOR cover
    assert lib.mnb_xnor_post_bytes(C.byref(_sh(H=7)), C.byref(_post(pool=1))) == -1
    assert L.launch_count() == n0


def test_pack_act_post_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    n0 = L.launch_count()
    assert lib.mnb_xnor_pack_act_post(FAKE, 2, 64, 8, 8, None, FAKE, None) == -1
    assert lib.mnb_xnor_pack_act_post(FAKE, 2, 64, 7, 8, C.byref(_post(pool=1)), FAKE, None) == -2
    assert lib.mnb_xnor_pack_act_post(FAKE, 2, 64, 8, 8, C.byref(_post(fmt=1)), FAKE, None) == -2   # bit planes only
    assert lib.mnb_xnor_pack_act_post(FAKE, 2, 64, 8, 8, C.byref(_post(groups=3)), FAKE, None) == -1
    assert L.launch_count() == n0


def test_post_bytes():
    from micronet_b200 import _lib as L
    lib = L.load()
    # 64 channels for a consumer with 16 groups: 4 channels per group, one (partly used) word per group
    assert lib.mnb_xnor_post_bytes(C.byref(_sh()), C.byref(_post(groups=16))) == 2 * 16 * 1 * 64 * 4
    assert lib.mnb_xnor_post_bytes(C.byref(_sh()), C.byref(_post(groups=16, pool=1))) == 2 * 16 * 1 * 16 * 4
    assert lib.mnb_xnor_post_bytes(C.byref(_sh()), C.byref(_post(fmt=1))) == 2 * 64 * 64 * 2


def _dest(c, K, sg, cin_o):
    """xnor::post_dest for the bit plane: (consumer group, word, bit) of producer channel c"""
    cpg = K // sg
    cd = (c % cpg) * sg + c // cpg if sg > 1 else c
    g, r = cd // cin_o, cd % cin_o
    return g, r // 32, r % 32


@pytest.mark.parametrize("K,sg,G,pool", [(64, 1, 2, False), (64, 2, 16, True), (256, 16, 4, False), (128, 32, 8, True),
                                        (96, 4, 3, True)])
def test_bit_destinations_model_pool_shuffle_pack(K, sg, G, pool):
    """scatter the sign bits the way the epilogue does (per producer channel, OR into the destination word, pooled pixels
    OR-ed together) and compare with the un-fused sequence: sign -> max-pool -> shuffle_channels -> mnb_xnor_pack_act"""
    rng = np.random.default_rng(K + sg + G)
    B, P, Q = 2, 4, 6
    v = rng.standard_normal((B, K, P, Q)).astype(np.float32)
    v[0, 0, 0, 0] = -0.0                                            # -0.0 -> +1
    cin_o = K // G
    nw = (cin_o + 31) // 32
    OP, OQ = (P // 2, Q // 2) if pool else (P, Q)
    got = np.zeros((B, G, nw, OP, OQ), dtype=np.uint64)
    for c in range(K):
        g, n, j = _dest(c, K, sg, cin_o)
        bit = (~(v[:, c] < 0)).astype(np.uint64)
        if pool:
            bit = bit[:, 0::2, 0::2] | bit[:, 1::2, 0::2] | bit[:, 0::2, 1::2] | bit[:, 1::2, 1::2]
        got[:, g, n] |= bit << np.uint64(j)
    t = torch.where(torch.from_numpy(v) < 0, -1.0, 1.0)
    if pool:
        t = torch.nn.functional.max_pool2d(t, 2, 2)
    if sg > 1:
        t = zoo.shuffle_channels(t, sg)
    want = np.zeros_like(got)
    for g in range(G):
        for n in range(nw):
            ch = t[:, g * cin_o + 32 * n: g * cin_o + min(32 * n + 32, cin_o)].numpy()
            for j in range(ch.shape[1]):
                want[:, g, n] |= (ch[:, j] > 0).astype(np.uint64) << np.uint64(j)
    assert np.array_equal(got, want)
    # the stem producer gathers instead: consumer channel cd reads producer channel (cd mod sg) * K/sg + cd div sg
    for cd in range(K):
        c = (cd % sg) * (K // sg) + cd // sg if sg > 1 else cd
        g, n, j = _dest(c, K, sg, cin_o)
        assert (g * cin_o + 32 * n + j) == cd


def _g2():
    import micronet_b200 as E
    torch.manual_seed(0)
    return E.wbwtab.prepare(zoo.init_like_reference(zoo.NINGC(CFG)), W=3, A=2, fuse_bn=True).eval()


def _g1(raw=None, nan=None):
    """the reference's deployment graph built on the CPU: BN-fused, weights alpha_k * {-1, 0, +1} written directly (the
    weight step itself runs the engine's quantizer kernel)"""
    import micronet_b200 as E
    torch.manual_seed(0)
    m = E.wbwtab.prepare(zoo.init_like_reference(zoo.NINGC(CFG)), W=3, A=2, quant_inference=True)
    m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=3)
    convs = [c for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    for c in convs:
        k = c.weight.shape[0]
        lv = torch.randint(-1, 2, c.weight.shape).float()
        c.weight.data = lv * (torch.rand(k) + 0.1).view(-1, 1, 1, 1)
    if raw is not None:
        convs[raw].weight.data = torch.randn(convs[raw].weight.shape)
    if nan is not None:
        convs[nan].weight.data[0] = float("nan")
    return m.eval()


def _frozen_convs(m):
    import micronet_b200 as E
    return [i for i, c in enumerate(c for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)) if "_mnb_frozen" in c.__dict__]


def _snapshot(m):
    return ([(n, type(k).__name__, getattr(k, "channel_shuffle_flag", None)) for n, k in m.named_modules()],
            {k: v.clone() for k, v in m.state_dict().items()})


def _same(a, b):
    assert a[0] == b[0]
    assert a[1].keys() == b[1].keys() and all(torch.equal(a[1][k], b[1][k]) for k in a[1])


def test_g2_records_and_restore():
    import micronet_b200 as E
    from micronet_b200.fused import BatchNormBinarize2d
    m = _g2()
    before = _snapshot(m)
    E.wbwtab.freeze_inference(m)
    assert _frozen_convs(m) == list(range(7))                          # L1 .. L7
    bnb = [k for k in m.modules() if isinstance(k, BatchNormBinarize2d)]
    assert len(bnb) == 8 and all("forward" in k.__dict__ for k in bnb)     # stem producer + seven absorbed
    # nothing structural moved: the fused graph already folded pools and shuffles
    _same(before, _snapshot(m))
    E.wbwtab.freeze_inference(m, enable=False)
    assert _frozen_convs(m) == [] and not any("forward" in k.__dict__ for k in m.modules())
    _same(before, _snapshot(m))


def test_g2_all_zero_ternary_channel_has_no_record():
    import micronet_b200 as E
    m = _g2()
    convs = [c for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    convs[3].weight.data[5].zero_()                                    # alpha = 0 / 0 = NaN
    E.wbwtab.freeze_inference(m)
    # L4 stays un-frozen; a producer is frozen only when its consumer reads what it writes, so L1 - L3 and the stem keep
    # their un-frozen path and L5 - L7 run on bit planes
    assert _frozen_convs(m) == [4, 5, 6]


def test_g1_records_and_restore():
    import micronet_b200 as E
    from micronet_b200.fused import EnginePmConv2d
    m = _g1()
    before = _snapshot(m)
    E.wbwtab.freeze_inference(m)
    assert _frozen_convs(m) == list(range(7))
    seq = m.model
    assert all(isinstance(seq._modules[n], nn.Identity) for n in ("3", "7"))           # both 2x2 pools folded
    assert all(getattr(b, "channel_shuffle_flag", 0) == 0 for b in seq.children())     # every shuffle folded
    assert isinstance(seq._modules["10"].conv, EnginePmConv2d)                        # the head reads the bf16 plane
    aqs = [k for k in m.modules() if isinstance(k, E.wbwtab.ActivationQuantizer)]
    assert len(aqs) == 8 and all("forward" in k.__dict__ for k in aqs)
    assert m.state_dict().keys() == before[1].keys()
    E.wbwtab.freeze_inference(m, enable=False)
    _same(before, _snapshot(m))
    assert type(seq._modules["10"].conv) is nn.Conv2d


@pytest.mark.parametrize("what", ["raw", "nan"])
def test_g1_records_no_weights_that_are_not_ternary_levels(what):
    import micronet_b200 as E
    from micronet_b200.fused import EnginePmConv2d
    m = _g1(**{what: 3})                                               # L4: raw fp32 weights, or a NaN channel
    E.wbwtab.freeze_inference(m)
    assert _frozen_convs(m) == [4, 5, 6]                              # L5 - L7; L1 - L3 have no frozen consumer
    assert isinstance(m.model._modules["3"], nn.MaxPool2d)             # the pool behind L2 stays
    assert isinstance(m.model._modules["7"], nn.Identity)              # the pool behind L5 moved into its epilogue
    assert isinstance(m.model._modules["10"].conv, EnginePmConv2d)
