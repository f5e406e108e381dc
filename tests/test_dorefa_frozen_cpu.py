"""CPU side of frozen DoReFa inference graphs (dorefa.freeze_inference): host refusals of the extended consumer epilogue
(BatchNorm, channel shuffle), the plane max-pool and the int8 stem producer (fake device pointers: nothing may be launched),
the shuffle destination map, and the graph rewrite on CPU-built NIN / NIN-GC models - which convs freeze and link, which
pools and shuffles are absorbed, and that ``enable=False`` restores the module tree and the state_dict."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn as nn

from harness import models as zoo

FAKE = 1 << 20          # never dereferenced: every call below is refused on the host
NIN_CFG = [64, 32, 32, 64, 64, 64, 64, 64]
GC_CFG = [32, 32, 32, 64, 64, 64, 128, 128]


def _q(bits=4):
    from micronet_b200 import _lib as L
    return L.ActQParams(L.ACT_DOREFA, bits, 0, 2 ** bits - 1, 0, None, None, None, None)


def _post(q, bn=(None,) * 4, sg=0, split=0):
    from micronet_b200 import _lib as L
    return L.PkPost(C.pointer(q), 1, split, FAKE, *bn, sg)


def test_consumer_epilogue_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = L.ConvShape(2, 64, 8, 8, 64, 1, 1, 1, 1, 0, 0, 1, 1, 2)
    q4 = _q(4)
    n0 = L.launch_count()

    def bf16(post):
        return lib.mnb_pk_conv_post(C.byref(sh), FAKE, 1, FAKE, 1, None, None, 1.0, None, None, C.byref(post), FAKE, None)

    def i8(post):
        return lib.mnb_pk_i8_conv(C.byref(sh), FAKE, FAKE, None, None, 1.0, None, None, C.byref(post), FAKE, None)

    for call in (bf16, i8):
        assert call(_post(q4, bn=(FAKE, FAKE, None, FAKE))) == -1            # a partial set of BatchNorm pointers
        assert call(_post(q4, bn=(FAKE, None, None, None))) == -1
        assert call(_post(q4, sg=3)) == L.E_UNSUPPORTED                        # 3 does not divide 64 channels
        assert call(_post(q4, sg=2, split=1)) == L.E_UNSUPPORTED               # shuffle + stride-2 consumer
        assert call(_post(q4, sg=-1)) == -1
    # 8-bit DoReFa levels reach 255: no int8 plane (the message names the symmetric IAO rule as before)
    assert i8(_post(_q(8))) == L.E_UNSUPPORTED and b"symmetric" in lib.mnb_last_error()
    assert lib.mnb_pk_i8_pack_act(FAKE, 2, 16, 8, 8, C.byref(_q(8)), 0, 0, FAKE, None) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def test_plane_pool_and_stem_producer_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    n0 = L.launch_count()
    pool = lib.mnb_pk_plane_maxpool
    assert pool(None, 2, 64, 8, 8, 2, 2, 0, 0, FAKE, None) == -1
    assert pool(FAKE, 2, 64, 8, 8, 2, 2, 0, 0, FAKE, None) == -1                # in place
    assert pool(FAKE, 2, 64, 8, 8, 3, 2, 2, 0, FAKE + 4096, None) == L.E_UNSUPPORTED   # 2 * p > k
    assert pool(FAKE, 2, 64, 8, 8, 0, 2, 0, 1, FAKE + 4096, None) == L.E_UNSUPPORTED
    assert pool(FAKE, 2, 64, 8, 8, 2, 2, 0, 0, FAKE + 8, None) == -1             # misaligned output
    stem = lib.mnb_bn_relu_quant_pack_i8_fwd
    args = (FAKE,) * 4
    assert stem(FAKE, 2, 64, 64, *args, C.byref(_q(8)), 1, FAKE, None) == L.E_UNSUPPORTED       # 8-bit: no s8 levels
    iao = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, FAKE, FAKE, FAKE, FAKE)
    assert stem(FAKE, 2, 64, 64, *args, C.byref(iao), 1, FAKE, None) == L.E_UNSUPPORTED         # DoReFa producer only
    assert stem(FAKE, 2, 40, 64, *args, C.byref(_q(4)), 1, FAKE, None) == L.E_UNSUPPORTED       # C % 16
    assert stem(FAKE, 2, 64, 48, *args, C.byref(_q(4)), 1, FAKE, None) == L.E_UNSUPPORTED       # H*W % 32
    assert stem(FAKE, 2, 64, 64, *args, C.byref(_q(4)), 3, FAKE, None) == -1                    # shuffle groups
    assert stem(FAKE, 2, 64, 64, None, FAKE, FAKE, FAKE, C.byref(_q(4)), 1, FAKE, None) == -1
    assert L.launch_count() == n0


@pytest.mark.parametrize("C_,sg", [(32, 2), (64, 16), (128, 4), (256, 32)])
def test_shuffle_destination_matches_shuffle_channels(C_, sg):
    """the epilogue stores producer channel c as consumer channel (c % cpg) * sg + c / cpg"""
    x = torch.arange(C_, dtype=torch.float32).view(1, C_, 1, 1)
    y = zoo.shuffle_channels(x, sg).view(-1)
    cpg = C_ // sg
    for c in range(C_):
        assert int(y[(c % cpg) * sg + c // cpg]) == c


def _model(kind, mode, a_bits=4, w_bits=4):
    from micronet_b200 import dorefa as DF, bn_fuse
    torch.manual_seed(0)
    base = zoo.init_like_reference(zoo.NIN(NIN_CFG) if kind == "nin" else zoo.NINGC(GC_CFG))
    if mode == "deploy":
        m = DF.prepare(base, a_bits=a_bits, w_bits=w_bits, quant_inference=True)
        with torch.no_grad():       # what bn_fuse.dorefa_quantize_inference_weights stores (DF:50-73, reference arithmetic)
            for c in m.modules():
                if isinstance(c, DF.QuantConv2d):
                    t = torch.tanh(c.weight)
                    t = t / 2 / t.abs().max() + 0.5
                    s = 1 / float(2 ** w_bits - 1)
                    c.weight.data = 2 * (torch.round(t / s) * s) - 1
        assert callable(bn_fuse.dorefa_quantize_inference_weights)
    else:
        m = DF.prepare(base, a_bits=a_bits, w_bits=w_bits, fuse=(mode == "fuse"))
    return m.eval()


def _snapshot(m):
    return repr(m), {k: v.clone() for k, v in m.state_dict().items()}, \
        [getattr(k, "channel_shuffle_flag", None) for k in m.modules()]


def _links(m):
    from micronet_b200 import dorefa as DF
    kids = [k for k in m.model.children()]
    frozen = [isinstance(k, nn.Module) and any("_mnb_frozen" in c.__dict__ for c in k.modules()) for k in kids]
    linked = []
    for k in kids:
        conv = next(iter(k.children()), None)
        if isinstance(conv, DF.QuantConv2d) and "_mnb_frozen" in conv.__dict__:
            linked.append(conv.__dict__["_mnb_frozen"]["link"] is not None)
        elif hasattr(k, "channel_shuffle_flag"):
            linked.append("forward" in list(k.children())[1].__dict__)      # the stem's BatchNorm
        else:
            linked.append("forward" in k.__dict__)                          # a pool on the level plane
    return frozen, linked


@pytest.mark.parametrize("kind", ["nin", "gc"])
@pytest.mark.parametrize("mode", ["plain", "fuse", "deploy"])
def test_recognition_and_restore(kind, mode):
    from micronet_b200 import dorefa as DF
    m = _model(kind, mode)
    before = _snapshot(m)
    DF.freeze_inference(m)
    frozen, linked = _links(m)
    # stem, two blocks, pool, three blocks, pool, two blocks, head, avg-pool
    assert frozen == [False] + [True] * 2 + [False] + [True] * 3 + [False] + [True] * 3 + [False]
    assert linked == [True] * 10 + [False, False], linked
    if kind == "gc":
        # every shuffle moved into its producer: no block shuffles its input any more
        assert all(not getattr(k, "channel_shuffle_flag", 0) for k in m.modules())
    assert m.state_dict().keys() == before[1].keys()
    assert all(torch.equal(v, before[1][k]) for k, v in m.state_dict().items())
    DF.freeze_inference(m, enable=False)
    after = _snapshot(m)
    assert after[0] == before[0] and after[2] == before[2]
    assert all(torch.equal(v, before[1][k]) for k, v in after[1].items())
    assert not any(k in c.__dict__ for c in m.modules() for k in ("forward", "_mnb_frozen", "_mnb_in_shuffle"))


def test_raw_deployment_weights_stay_unfrozen():
    from micronet_b200 import dorefa as DF
    m = _model("gc", "deploy")
    kids = list(m.model.children())
    raw = next(iter(kids[5].children()))
    with torch.no_grad():
        raw.weight.add_(1e-3)                     # no longer odd levels over 2^w - 1
    DF.freeze_inference(m)
    assert "_mnb_frozen" not in raw.__dict__
    prod = next(iter(kids[4].children()))        # the producer in front of it writes fp32 as before
    assert prod.__dict__["_mnb_frozen"]["link"] is None
    assert "forward" not in list(kids[4].children())[1].__dict__
    assert kids[5].channel_shuffle_flag == 1
    DF.freeze_inference(m, enable=False)


def test_int8_flag_and_training_mode():
    from micronet_b200 import dorefa as DF
    m = _model("gc", "plain")
    DF.freeze_inference(m, int8=True)
    assert all(c.__dict__["_mnb_frozen"]["int8"] for c in m.modules() if "_mnb_frozen" in c.__dict__)
    conv = next(iter(list(m.model.children())[1].children()))
    conv.train()
    with pytest.raises(RuntimeError, match="frozen"):
        conv(torch.zeros(1, GC_CFG[0], 8, 8))
    m8 = _model("nin", "plain", a_bits=8, w_bits=8)
    DF.freeze_inference(m8, int8=True)
    assert not any(c.__dict__["_mnb_frozen"]["int8"] for c in m8.modules() if "_mnb_frozen" in c.__dict__)
    # a model frozen in training mode freezes nothing
    t = copy.deepcopy(_model("nin", "plain")).train()
    DF.freeze_inference(t)
    assert not any("_mnb_frozen" in c.__dict__ for c in t.modules())
