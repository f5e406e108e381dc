"""frozen_graph, the host-side rewriting the three schemes' freeze_inference share: ``enable=False`` restores every module as
it was before the first freeze, freezing twice gives the plan of freezing once, and the one tag reader hands a plane only to
its target (unchanged version, matching groups), raises for a level plane anywhere else and lets decodable planes fall
through.  CPU only: freezing needs the library's plan queries, no GPU."""
import pytest
import torch
import torch.nn as nn

from harness import models as zoo
from harness import train as H

GC_CFG = [32, 32, 32, 64, 64, 64, 128, 128]
NIN_CFG = [64, 32, 32, 64, 64, 64, 64, 64]


def _wbwtab(name, **kw):
    import micronet_b200 as E
    m = E.wbwtab.prepare(H.build_float_model(name, seed=1), W=3, **kw)
    if kw.get("quant_inference"):
        # the reference's deployment graph: BN-fused, weights alpha_k * {-1, 0, +1} written directly (the weight step
        # itself runs the engine's quantizer kernel)
        m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=3)
        for c in m.modules():
            if isinstance(c, E.wbwtab.QuantConv2d):
                lv = torch.randint(-1, 2, c.weight.shape).float()
                c.weight.data = lv * (torch.rand(c.weight.shape[0]) + 0.1).view(-1, 1, 1, 1)
    return m.eval()


def _dorefa(kind, **kw):
    from micronet_b200 import dorefa
    torch.manual_seed(0)
    base = zoo.init_like_reference(zoo.NIN(NIN_CFG) if kind == "nin" else zoo.NINGC(GC_CFG))
    return dorefa.prepare(base, a_bits=4, w_bits=4, **kw).eval()


def _iao(kind, deploy=False):
    from micronet_b200 import bn_fuse, iao
    torch.manual_seed(0)
    base = zoo.resnet18() if kind == "resnet" else zoo.init_like_reference(zoo.NINGC(GC_CFG))
    m = iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True).eval()
    return bn_fuse.iao_quantize_inference_weights(bn_fuse.iao_model_bn_fuse(m)).eval() if deploy else m


GRAPHS = {
    "wbwtab_nin_gc_fused": (lambda: _wbwtab("nin_gc", A=2, fuse_bn=True), "wbwtab", {}),
    "wbwtab_nin_gc_deploy": (lambda: _wbwtab("nin_gc", A=2, quant_inference=True), "wbwtab", {}),
    "wbwtab_nin_b1": (lambda: _wbwtab("nin", A=2, fuse_bn=True), "wbwtab", {}),
    "wbwtab_nin_b1_deploy": (lambda: _wbwtab("nin", A=2, quant_inference=True), "wbwtab", {}),
    "wbwtab_nin_gc_a32": (lambda: _wbwtab("nin_gc", A=32), "wbwtab", {}),
    "wbwtab_nin_a32": (lambda: _wbwtab("nin", A=32), "wbwtab", {}),
    "dorefa_nin": (lambda: _dorefa("nin"), "dorefa", {}),
    "dorefa_nin_gc_fused_int8": (lambda: _dorefa("gc", fuse=True), "dorefa", {"int8": True}),
    "iao_nin_gc_int8": (lambda: _iao("gc"), "iao", {"int8": True}),
    "iao_nin_gc_deploy": (lambda: _iao("gc", deploy=True), "iao", {}),
    "iao_resnet18": (lambda: _iao("resnet"), "iao", {}),
}


def _freeze(m, scheme, **kw):
    import micronet_b200 as E
    return getattr(E, scheme).freeze_inference(m, **kw)


def _state(m):
    """every module: its __dict__ (keys and the identity of each value), children and state_dict"""
    mods = [(n, k, dict((a, id(v)) for a, v in k.__dict__.items()), dict(k._modules)) for n, k in m.named_modules()]
    return mods, {k: v.clone() for k, v in m.state_dict().items()}


def _describe(v, names, depth=0):
    """a freeze's plan without object identities: modules by name, links by their public attributes"""
    if isinstance(v, nn.Module):
        return names.get(id(v), type(v).__name__)
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape))
    if isinstance(v, (tuple, list)):
        return tuple(_describe(x, names, depth) for x in v)
    if isinstance(v, dict):
        return tuple(sorted((k, _describe(x, names, depth)) for k, x in v.items()))
    if hasattr(v, "__dict__") and not callable(v) and depth < 2:
        return (type(v).__name__,) + tuple(sorted((k, _describe(x, names, depth + 1)) for k, x in vars(v).items()
                                                  if not k.startswith("_")))
    if callable(v):
        return ("callable",)
    return v


def _plan(m):
    names = {id(k): n for n, k in m.named_modules()}
    return [(n, type(k).__name__, _describe({a: v for a, v in k.__dict__.items() if a.startswith("_mnb") or a in (
        "forward", "channel_shuffle_flag", "_frozen_inference", "_int8", "_int_levels", "_pre_relu", "_fuse_relu",
        "_post_consumer")}, names)) for n, k in m.named_modules()]


@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_undo_restores_every_module(graph):
    build, scheme, kw = GRAPHS[graph]
    m = build()
    mods, sd = _state(m)
    _freeze(m, scheme, **kw)
    assert _plan(m) != _plan(build()), "nothing was frozen"
    _freeze(m, scheme, enable=False)
    mods2, sd2 = _state(m)
    assert len(mods2) == len(mods)
    for (n, k, d, kids), (n2, k2, d2, kids2) in zip(mods, mods2):
        assert n == n2 and k is k2, (n, n2)
        assert d == d2, (n, sorted(set(d) ^ set(d2)), [a for a in d if a in d2 and d[a] != d2[a]])
        assert kids.keys() == kids2.keys() and all(kids[a] is kids2[a] for a in kids), n
    assert sd.keys() == sd2.keys() and all(torch.equal(sd[k], sd2[k]) for k in sd)


@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_freezing_twice_gives_the_plan_of_freezing_once(graph):
    build, scheme, kw = GRAPHS[graph]
    m = build()
    _freeze(m, scheme, **kw)
    once = _plan(m)
    _freeze(m, scheme, **kw)
    assert _plan(m) == once


def test_tag_reader_rules():
    from micronet_b200 import functional as F_
    conv, other, g4 = nn.Conv2d(8, 8, 1, groups=2), nn.Conv2d(8, 8, 1, groups=2), nn.Conv2d(8, 8, 1, groups=4)
    plane = torch.zeros(4, dtype=torch.int32)

    def meta():
        return torch.empty(1, 8, 2, 2, device="meta")

    # a bit plane: its target at its groups only; anywhere else it falls through to functional.materialized
    bits = F_.tag(meta(), conv, plane, "bits", groups=2)
    assert F_.handed_plane(conv, bits) is plane
    assert F_.handed_plane(other, bits) is None and F_.handed_plane(g4, bits) is None
    b1 = F_.tag(meta(), conv, plane, "b1", groups=2)
    assert F_.handed_plane(conv, b1) is plane and F_.handed_plane(g4, b1) is None
    terms = F_.tag(meta(), conv, plane, "terms", split=False, terms=3)
    assert F_.handed_plane(conv, terms) is plane and F_.handed_plane(other, terms) is None
    # a meta-shaped output holds nothing but its plane: an in-place write changes no value, the version is not checked
    terms.add_(1)
    assert F_.handed_plane(conv, terms) is plane
    # a level plane cannot be decoded: at any module but its target a meta-shaped one raises, and so does an untagged one
    for fmt in ("bf16", "i8"):
        lv = F_.tag(meta(), conv, plane, fmt)
        assert F_.handed_plane(conv, lv) is plane
        with pytest.raises(RuntimeError, match="not produced for"):
            F_.handed_plane(other, lv)
        with pytest.raises(RuntimeError, match="cannot be decoded"):
            F_.materialized(lv)
    with pytest.raises(RuntimeError, match="not produced for"):
        F_.handed_plane(conv, meta())
    # an output that also holds values (a QuantAdd's fp32 sum): its plane only while the tensor is unmodified
    y = F_.tag(torch.zeros(1, 8, 2, 2), conv, plane, "bf16")
    assert F_.handed_plane(conv, y) is plane and F_.handed_plane(other, y) is None and F_.materialized(y) is y
    y.add_(1)
    assert F_.handed_plane(conv, y) is None
