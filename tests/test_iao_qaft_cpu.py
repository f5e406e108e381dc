"""CPU side of the QAFT hand-offs of BN-fused IAO NIN / NIN-GC models (iao.prepare(bn_fuse=True, qaft=True, fuse=True)):
host refusals of the training consumer epilogue (mnb_pk_conv_post_train, its plan query) and of the training plane
pool and its backward (fake device pointers: nothing may be launched), which blocks link, which pools run on the plane and
that no shuffle moves, that every other configuration links nothing, and that module types, repr, state_dict, shuffle flags
and iao.freeze_inference (records, links, enable=False) are those of the same model prepared without ``fuse``."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from harness import models as zoo

FAKE = 1 << 20          # never dereferenced: every call below is refused on the host
NIN_CFG = [64, 32, 32, 64, 64, 64, 64, 64]
GC_CFG = [32, 32, 32, 64, 64, 64, 128, 128]
PRUNED_CFG = [154, 162, 144, 304, 320, 320, 608, 584]


def _iao_q(bits=8, q_type=0, qmin=None, qmax=None):
    from micronet_b200 import _lib as L
    half = 1 << (bits - 1)
    qmin = -half if qmin is None else qmin
    qmax = half - 1 if qmax is None else qmax
    return L.ActQParams(L.ACT_IAO, bits, qmin, qmax, q_type, FAKE, FAKE, FAKE, FAKE)


def _shape(b=4, c=64, h=16, w=16, k=64, r=1, groups=1):
    from micronet_b200 import _lib as L
    return L.ConvShape(b, c, h, w, k, r, r, 1, 1, r // 2, r // 2, 1, 1, groups)


def test_train_epilogue_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    q8, n0 = _iao_q(8), L.launch_count()

    def post(q=q8, **kw):
        p = L.PkPost(None if q is None else C.pointer(q), 1, 0, FAKE)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    def plan(p, sh=None):
        return lib.mnb_pk_conv_post_train_plan(C.byref(sh or _shape()), 1, 1, C.byref(p), None, 0)

    def launch(p, sh=None, bits=FAKE):
        return lib.mnb_pk_conv_post_train(C.byref(sh or _shape()), FAKE, 1, FAKE, 1, None, None, 1.0, None, None, C.byref(p),
                                          bits, FAKE, None)

    assert plan(post()) == 0                                          # the cover: a plain bf16 plane of a symmetric IAO quantizer
    out = (C.c_int32 * 10)()
    assert lib.mnb_pk_conv_post_train_plan(C.byref(_shape()), 1, 1, C.byref(post()), out, 10) == 0 and out[0] == 3
    assert lib.mnb_pk_conv_post_plan(C.byref(_shape()), 1, 1, 8, C.byref(post()), out, 10) == 0 and out[0] == 0
    assert launch(post(), bits=None) == -1
    assert lib.mnb_pk_conv_post_train_plan(C.byref(_shape()), 1, 1, None, None, 0) == -1
    for p in (post(q=_iao_q(8, q_type=1, qmin=0, qmax=255)),         # asymmetric consumer
              post(q=L.ActQParams(L.ACT_DOREFA, 4, 0, 15, 0, None, None, None, None)),
              post(shuffle_groups=2),                                 # shuffled consumer plane
              post(bn_mean=FAKE, bn_invstd=FAKE, bn_gamma=FAKE, bn_beta=FAKE)):
        assert plan(p) == L.E_UNSUPPORTED and launch(p) == L.E_UNSUPPORTED
        assert b"STE mask" in lib.mnb_last_error()
    term = post(q=None, terms_out=2)                                  # term planes carry no STE mask
    assert plan(term) == L.E_UNSUPPORTED and launch(term) == L.E_UNSUPPORTED
    # a producer storing partial 8-channel units, grouped or not
    assert plan(post(), sh=_shape(c=12, k=12, groups=2)) == L.E_UNSUPPORTED
    assert plan(post(), sh=_shape(k=12)) == L.E_UNSUPPORTED and launch(post(), sh=_shape(k=12)) == L.E_UNSUPPORTED
    assert lib.mnb_pk_conv_post_plan(C.byref(_shape(k=12)), 1, 1, 8, C.byref(post()), None, 0) == 0   # no mask: accepted
    assert L.launch_count() == n0


def test_train_pool_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    q8, n0 = _iao_q(8), L.launch_count()

    def fwd(k=2, s=2, p=0, c=64, q_in=q8, q_out=q8, out=FAKE + 4096, arg=FAKE + 8192):
        return lib.mnb_pk_plane_maxpool_requant_train(FAKE, 2, c, 8, 8, k, s, p, None if q_in is None else C.byref(q_in),
                                                      None if q_out is None else C.byref(q_out), out, arg, FAKE, None)

    def bwd(k=2, s=2, p=0, c=64, q_in=q8, arg=FAKE + 8192):
        return lib.mnb_pk_plane_maxpool_requant_bwd(FAKE, arg, FAKE, 2, c, 8, 8, k, s, p, None if q_in is None else C.byref(q_in),
                                                    FAKE + 4096, None)

    for call in (fwd, bwd):
        assert call(q_in=None) == -1
        assert call(arg=FAKE + 4) == -1                               # window indices: 8-byte units
        assert call(3, 2, 2) == L.E_UNSUPPORTED                       # 2 * p > k
        assert call(16, 16, 0) == L.E_UNSUPPORTED                     # k > 15: the index byte
        assert call(c=60) == L.E_UNSUPPORTED                          # whole 8-channel units only
        assert call(q_in=_iao_q(8, q_type=1, qmin=0, qmax=255)) == L.E_UNSUPPORTED
        assert b"symmetric IAO" in lib.mnb_last_error()
        nulls = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, None, None, None, None)
        assert call(q_in=nulls) == -1
    assert fwd(out=FAKE) == -1                                        # in place
    assert fwd(out=FAKE + 8) == -1                                    # misaligned plane
    assert fwd(q_out=None) == -1
    assert fwd(q_out=_iao_q(4, q_type=1, qmin=0, qmax=15)) == L.E_UNSUPPORTED
    assert L.launch_count() == n0


def _model(kind, fuse=True, q_type=0, bn_fuse=True, qaft=True, ptq=False, a_bits=8, w_bits=8):
    from micronet_b200 import iao
    torch.manual_seed(0)
    if kind == "resnet":
        base = zoo.resnet18()
    else:
        cfg = {"nin": NIN_CFG, "gc": GC_CFG, "pruned": PRUNED_CFG}[kind]
        base = zoo.init_like_reference(zoo.NIN(cfg) if kind == "nin" else zoo.NINGC(cfg))
    return iao.prepare(base, a_bits=a_bits, w_bits=w_bits, q_type=q_type, bn_fuse=bn_fuse, qaft=qaft, ptq=ptq, fuse=fuse)


def _plan(m):
    """per child of model.model: does its conv hand its consumer a plane / does the pool run on the plane?"""
    out = []
    for k in m.model.children():
        conv = next(iter(k.children()), None)
        if isinstance(conv, nn.Conv2d):
            out.append("_mnb_train_link" in conv.__dict__)
        else:
            out.append("forward" in k.__dict__)
    return out


# per child of model.model (stem, two blocks, pool, three blocks, pool, two blocks, head, avg-pool): only links across a pool
# are made (a pool-less link costs more than it saves), so NIN links blocks 2 and 5 across its two pools and runs both pools
# on the plane.  NIN-GC's pools sit in front of blocks that shuffle their input (a shuffled bf16 epilogue does not pay,
# iao._shuffled_link_pays): it links nothing, nor does the README-pruned NIN-GC.
WANT = {"nin": [False, False, True, True, False, False, True, True, False, False, False, False], "gc": [False] * 12,
        "pruned": [False] * 12}


@pytest.mark.parametrize("kind", ["nin", "gc", "pruned"])
@pytest.mark.parametrize("ptq", [False, True])
def test_link_plan(kind, ptq):
    m = _model(kind, ptq=ptq)
    want = WANT[kind]
    assert _plan(m) == want
    kids = list(m.model.children())
    for i in (3, 7):
        if want[i]:
            link = next(iter(kids[i - 1].children())).__dict__["_mnb_train_link"]
            assert link.pool[0] is kids[i] and link.pool[1:] == (3, 2, 1)
            assert link.cconv is next(iter(kids[i + 1].children())) and link.target is kids[i]
    # the ReLU of every linked block passes the plane through, the others run as usual
    assert [("forward" in k.relu.__dict__) for k in kids if hasattr(k, "relu")] == [w for k, w in zip(kids, want)
                                                                                    if hasattr(k, "relu")]
    # no shuffle moves
    assert not any("_mnb_in_shuffle" in c.__dict__ for c in m.modules())
    ref = _model(kind, fuse=False, ptq=ptq)
    assert [getattr(k, "channel_shuffle_flag", None) for k in m.modules()] == \
        [getattr(k, "channel_shuffle_flag", None) for k in ref.modules()]


@pytest.mark.parametrize("why", ["q_type1", "bn_live", "qat", "a32", "w32", "no_fuse"])
def test_excluded_graphs_link_nothing(why):
    kw = {"q_type1": dict(q_type=1), "bn_live": dict(bn_fuse=False), "qat": dict(qaft=False), "a32": dict(a_bits=32),
          "w32": dict(w_bits=32), "no_fuse": dict(fuse=False)}[why]
    m = _model("nin", **kw)
    assert _plan(m) == [False] * 12
    assert not any(k in c.__dict__ for c in m.modules() for k in ("forward", "_mnb_train_link"))


def test_resnet_links_nothing():
    m = _model("resnet")
    assert not any(k in c.__dict__ for c in m.modules() for k in ("forward", "_mnb_train_link"))


def test_pool_outside_cover_is_not_crossed():
    from micronet_b200 import iao
    base = zoo.init_like_reference(zoo.NIN(NIN_CFG))
    base.model[3] = nn.MaxPool2d(kernel_size=(3, 2), stride=2, padding=1)     # a non-square window: not covered
    m = iao.prepare(base, bn_fuse=True, qaft=True, fuse=True)
    assert _plan(m) == [False] * 6 + [True, True] + [False] * 4


@pytest.mark.parametrize("kind", ["nin", "gc"])
def test_modules_state_dict_and_freeze_unchanged(kind):
    from micronet_b200 import iao
    m, ref = _model(kind), _model(kind, fuse=False)
    assert repr(m) == repr(ref)
    assert [type(k) for k in m.modules()] == [type(k) for k in ref.modules()]
    assert m.state_dict().keys() == ref.state_dict().keys()
    assert all(torch.equal(v, ref.state_dict()[k]) for k, v in m.state_dict().items())
    before = {id(c): dict(c.__dict__) for c in m.modules()}
    m.eval()
    ref.eval()

    def records(model):
        names = {id(mod): n for n, mod in model.named_modules()}
        return [(r[0], names.get(id(r[1])), r[2]) for r in model.__dict__["_mnb_iao_undo"]]

    def links(model):
        out = []
        for n, mod in model.named_modules():
            link = mod.__dict__.get("_post_consumer")
            if link is not None:
                out.append((n, type(link).__name__, id(link.cconv) in {id(x) for x in model.modules()}))
        return out

    for i8 in (False, True):
        iao.freeze_inference(m, int8=i8)
        iao.freeze_inference(ref, int8=i8)
        assert records(m) == records(ref)
        assert links(m) == links(ref)
        assert repr(m) == repr(ref)
        iao.freeze_inference(m, enable=False)
        iao.freeze_inference(ref, enable=False)
        # the training links and overrides are back, nothing of the freeze is left
        after = {id(c): dict(c.__dict__) for c in m.modules()}
        assert after.keys() == before.keys()
        for k, d in after.items():
            assert d.keys() == before[k].keys()
        assert _plan(m) == WANT[kind]


def test_cleared_qaft_flag_stops_the_hand_off():
    """a link is made from the qaft flags at prepare time; a quantizer whose flag is cleared later (to resume QAT on the same
    modules) would refresh its observer from the producer's unwritten output, so the producer re-checks them per call"""
    m = _model("nin").train()
    conv = m.model[2].conv
    link = conv.__dict__["_mnb_train_link"]
    assert link.frozen_quantizers(conv)
    for q in (link.cconv.activation_quantizer, link.pool[0].activation_quantizer, conv.weight_quantizer):
        q.qaft = False
        assert not link.frozen_quantizers(conv)
        q.qaft = True
    assert link.frozen_quantizers(conv)
