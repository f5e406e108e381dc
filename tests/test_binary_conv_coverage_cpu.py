"""Coverage of the two binary forward convolutions (csrc/mnb_xnor.cu, csrc/mnb_b1.cu) by tests/binary_conv_cases.py, checked
on the host with the launchers' own plan functions (xnor.plan / b1.plan; no GPU needed):

* every conv_kernel instance of both kernels is launched by some case,
* every plan feature the case list is written for is reached,
* every case's plan is still the one pinned beside it,
* every binarized conv of the frozen NIN, NIN-GC and README-cfg pruned NIN-GC graphs (wbwtab.freeze_inference on the CPU)
  runs a plan some case runs,

so a change of the plan heuristics or of the case list that leaves an instance, a feature or a model layer untested fails
here, naming it.  Also pins the link plan of the pruned NIN-GC (which layer freezes on which kernel, what each hand-off
writes)."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from tests import binary_conv_cases as BC


def _launches():
    """[(case id, kernel, plan)] of every launch of the case list"""
    out = []
    for case in BC.CASES:
        for kernel, plan in BC.launches(case):
            assert plan is not None, f"{case.id}: outside the {kernel} kernel's cover"
            out.append((case, kernel, plan))
    return out


def test_every_kernel_instance_is_launched():
    got = {(k, BC.instance(k, p)) for _, k, p in _launches()}
    missing = [("xnor", i) for i in BC.XNOR_INSTANCES if ("xnor", i) not in got]
    missing += [("b1", i) for i in BC.B1_INSTANCES if ("b1", i) not in got]
    assert not missing, ("instances no case launches (xnor: R, NW, BORDER, POST; b1: Nt, POST): "
                         f"{missing}")


def test_every_plan_feature_is_reached():
    got = set()
    for case, _, plan in _launches():
        got |= BC.features(case, plan)
    assert not BC.WANTED_FEATURES - got, f"plan features no case reaches: {sorted(BC.WANTED_FEATURES - got)}"
    assert len(BC.WANTED_FEATURES) >= 35


def test_no_launch_is_refused():
    refused = [case.id for case, k, p in _launches() if k == "xnor" and p["refused"]]
    assert not refused, refused


def test_every_case_runs_its_pinned_plan():
    ids = [c.id for c in BC.CASES]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    changed = {}
    for case in BC.CASES:
        got = BC.plan_tuple(case.kernel, BC.plan_of(case.kernel, case.shape, case.post))
        if got != tuple(case.plan):
            changed[case.id] = {"pinned": case.plan, "now": got}
    assert not changed, f"plans that changed under the cases written for them: {changed}"


# ---- frozen graphs, frozen on the CPU (only host-side cover queries run)
def _model(name):
    import micronet_b200 as E
    from harness import models as zoo, train as H
    from tests.test_pk_pruned_cpu import README_CFG
    if name == "pruned":
        torch.manual_seed(1)
        base = zoo.init_like_reference(zoo.NINGC(README_CFG))
    else:
        base = H.build_float_model(name, seed=1)
    return E.wbwtab.prepare(base, W=3, A=2, fuse_bn=True).eval()


def _conv_inputs(m, hw=32):
    """{conv: (C, H, W) of its input} for a 32 x 32 image through the model's nn.Sequential"""
    out, c, h, w = {}, 3, hw, hw
    for blk in m.model.children():
        if isinstance(blk, nn.MaxPool2d):
            k, s, p = blk.kernel_size, blk.stride, blk.padding
            h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
            continue
        if isinstance(blk, (nn.AvgPool2d, nn.Identity)):
            continue
        cv = blk.conv
        out[cv] = (c, h, w)
        k, s, p = cv.kernel_size[0], cv.stride[0], cv.padding[0]
        c, h, w = cv.out_channels, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        if any(getattr(k_, "pool2", False) for k_ in blk.children()):      # a pool folded into the fused producer
            h, w = h // 2, w // 2
    return out


def _link(conv):
    """the (_Link, kernel) of a frozen conv's record, or None when the conv stayed un-frozen"""
    rec = conv.__dict__.get("_mnb_frozen")
    return None if rec is None else (rec["link"], rec["kernel"])


def _post_of(link):
    from micronet_b200 import fused
    fmt = {v: k for k, v in BC.FMT.items()}[link.fmt]
    return BC.Post(fmt, link.out_groups, link.sg, link.pool2, isinstance(link.act, fused.BatchNormBinarize2d))


def _frozen_layers(name):
    """[(layer, kernel or None, shape at batch 1, post)] of the binarized convs of a frozen model"""
    import micronet_b200 as E
    m = _model(name)
    ins = _conv_inputs(m)
    E.wbwtab.freeze_inference(m)
    out = []
    convs = [c for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]
    for i, conv in enumerate(convs):
        c, h, w = ins[conv]
        shape = (1, c, h, w, conv.out_channels, conv.kernel_size[0], conv.stride[0], conv.padding[0], conv.groups)
        lk = _link(conv)
        out.append((f"L{i + 1}", None if lk is None else lk[1], shape, None if lk is None else _post_of(lk[0])))
    return m, out


@pytest.fixture(scope="module")
def frozen():
    return {name: _frozen_layers(name) for name in ("nin", "nin_gc", "pruned")}


def test_frozen_records_are_covered_by_cases(frozen):
    tested = {(k, BC.plan_tuple(k, p)) for _, k, p in _launches()}
    missing, n = [], 0
    for name, (_, layers) in frozen.items():
        for layer, kernel, shape, post in layers:
            assert kernel is not None, f"{name} {layer} stays un-frozen"
            for B in BC.MODEL_BATCHES:
                sh = (B,) + shape[1:]
                for p in (None, post):
                    sig = (kernel, BC.plan_tuple(kernel, BC.plan_of(kernel, sh, p)))
                    n += 1
                    if sig not in tested:
                        missing.append((name, layer, B, "post" if p else "fwd", sig))
    assert n == 2 * 2 * 21
    assert not missing, f"plans of frozen-graph convs no case runs: {missing}"


def test_model_cases_are_the_frozen_records(frozen):
    """MODEL_LAYERS is what freeze_inference links today: same kernel, geometry and hand-off for every layer"""
    want = [(m, layer, BC.MODEL_KERNEL[m], geo, post) for m, layer, geo, post in BC.MODEL_LAYERS]
    got = []
    for name, (_, layers) in frozen.items():
        for layer, kernel, (_, c, h, w, k, r, st, pad, g), post in layers:
            assert st == 1
            got.append((name, layer, kernel, (c, h, w, k, r, pad, g), post))
    assert got == want


def test_pruned_nin_gc_frozen_records(frozen):
    """README-cfg pruned NIN-GC (154 162 144 304 320 320 608 584): all seven binarized convs freeze on the XNOR kernel
    (76 - 81 channels per group on the 1x1 layers: three words, the third partial), each epilogue writes its consumer's bit
    plane at the consumer's groups with the consumer block's shuffle and the folded 2x2 pools, the last one the head's bf16
    plane; the stem's binarizer writes L1's bit plane"""
    from micronet_b200 import _lib as L, fused
    m, layers = frozen["pruned"]
    plan = [(layer, kernel, shape[8], post) for layer, kernel, shape, post in layers]
    P = BC.Post
    assert plan == [
        ("L1", "xnor", 2, P("bits", 2, 2, False, True)),
        ("L2", "xnor", 2, P("bits", 16, 2, True, True)),
        ("L3", "xnor", 16, P("bits", 4, 16, False, True)),
        ("L4", "xnor", 4, P("bits", 4, 4, False, True)),
        ("L5", "xnor", 4, P("bits", 32, 4, True, True)),
        ("L6", "xnor", 32, P("bits", 8, 32, False, True)),
        ("L7", "xnor", 8, P("bf16", 1, 1, False, True)),
    ]
    nws = [BC.plan_of(k, s)["NW"] for _, k, s, _ in layers]
    assert nws == [3, 3, 1, 3, 3, 1, 3]
    # the stem's binarizer: a producer of L1's bit plane (2 groups of 77 channels)
    acts = [k for k in m.modules() if isinstance(k, fused.BatchNormBinarize2d)]
    stem = acts[0].__dict__.get("_mnb_frozen")
    assert stem is not None and stem["link"].fmt == L.XNOR_BITS and stem["link"].out_groups == 2
    assert all("forward" in k.__dict__ for k in acts[1:])     # absorbed into the conv epilogues
    assert not any(type(k).__name__ == "_PlanePool" for k in m.modules())


def test_plan_query_and_launcher_agree_on_refusal():
    """a plan the query marks refused is refused by the launcher before anything is launched (the pointers below are never
    dereferenced); the query returns None outside the cover and refuses a malformed epilogue"""
    from micronet_b200 import _lib as L, b1 as B1, xnor as X
    lib = L.load()
    sh = BC.conv_shape((1, 65536, 2, 2, 65536, 1, 1, 0, 65536))      # one channel per group: 65536 (group, k-slice) blocks
    p = X.plan(sh)
    assert p is not None and p["refused"] == 1 and X.supported(sh)
    fake = 4096
    assert lib.mnb_xnor_conv_fwd(C.byref(sh), fake, fake, None, None, fake, None) == L.E_UNSUPPORTED
    assert X.plan(BC.conv_shape((1, 64, 9, 9, 8, 7, 1, 3, 1))) is None            # 7x7: b1 only
    assert B1.plan(BC.conv_shape((1, 64, 9, 9, 8, 3, 2, 1, 1))) is None           # stride 2: XNOR only
    odd = BC.conv_shape((1, 64, 9, 9, 8, 3, 1, 1, 1))
    assert X.plan(odd, X.post_struct(L.XNOR_BITS, 1, 1, True)) is None           # a 2x2 pool over a 9 x 9 plane
    assert B1.plan(odd, X.post_struct(L.XNOR_B1_PLANE, 1, 1, True)) is None
    with pytest.raises(ValueError):
        X.plan(odd, X.post_struct(L.XNOR_BITS, 3, 1, False))                    # 3 consumer groups of 8 channels
    assert X.plan(odd, X.post_struct(L.XNOR_BITS, 2, 1, False))["post"] == 1
    assert B1.plan(odd)["post"] == 0 and B1.plan(odd, X.post_struct(L.XNOR_PM1_BF16, 1, 1, False))["post"] == 1
