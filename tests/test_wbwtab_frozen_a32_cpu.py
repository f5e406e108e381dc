"""Host-side link plan of wbwtab.freeze_inference on fp32-activation models (prepare(A=32, W=2|3)): which convs run frozen
on term planes, which pools run on the plane, the shuffle each link carries, the packed-operand plan of every quantized layer
at terms (3, 1), the graphs that must stay as they are, the new C-ABI symbols and the SASS of the new kernel instances.
Builds and freezes on the CPU: only host-side cover queries run."""
import ctypes
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn as nn

from harness import train as H
from tests.test_wbwtab_frozen_nin_cpu import RefNIN


def _model(name, W, A=32):
    import micronet_b200 as E
    if name == "ref_nin":
        torch.manual_seed(1)
        base = RefNIN()
    else:
        base = H.build_float_model(name, seed=1)
    return E.wbwtab.prepare(base, W=W, A=A).eval()


def _quant_convs(m):
    import micronet_b200 as E
    return [c for c in m.modules() if type(c) is E.wbwtab.QuantConv2d]


def _plan(m):
    return [c.__dict__.get("_mnb_frozen_plan") for c in _quant_convs(m)]


def _links(m):
    """the link of each quantized conv that writes term planes (None for the others)"""
    recs = [c.__dict__.get("_mnb_frozen") for c in _quant_convs(m)]
    return [r["link"] if r is not None and r["fmt"] == "terms3" else None for r in recs]


def _overridden(m, cls):
    return [k for k in m.modules() if type(k) is cls and "forward" in k.__dict__]


TERMS, FP32 = ("pk", "terms3"), ("pk", "fp32")


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("name", ["nin", "ref_nin"])
def test_nin_frozen_records(name, W):
    import micronet_b200 as E
    m = _model(name, W)
    tree = [type(k) for k in m.modules()]
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    E.wbwtab.freeze_inference(m)
    # L1 - L6 write their consumer's term planes, L7 writes fp32 for the un-quantized head
    assert _plan(m) == [TERMS] * 6 + [FP32]
    links = _links(m)
    assert all(lk.sg == 1 for lk in links[:6]) and links[6] is None
    pools = [lk.pool for lk in links[:6] if lk.pool is not None]
    assert [p[1:] for p in pools] == [(3, 2, 1)] * 2
    assert len(_overridden(m, nn.MaxPool2d)) == 2
    # every BatchNorm but the head's passes the plane through (the stem's is the stem producer); every ReLU but the
    # head's and L7's too
    assert len(_overridden(m, nn.BatchNorm2d)) == 7
    assert [type(k) for k in m.modules()] == tree
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    E.wbwtab.freeze_inference(m, enable=False)
    assert [type(k) for k in m.modules()] == tree and _plan(m) == [None] * 7 and _links(m) == [None] * 7
    assert not _overridden(m, nn.BatchNorm2d) and not _overridden(m, nn.MaxPool2d)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())


@pytest.mark.parametrize("W", [2, 3])
def test_nin_gc_frozen_records(W):
    import micronet_b200 as E
    m = _model("nin_gc", W)
    flags = [getattr(b, "channel_shuffle_flag", None) for b in m.model.children()]
    assert sum(bool(f) for f in flags) == 6
    E.wbwtab.freeze_inference(m)
    assert _plan(m) == [TERMS] * 6 + [FP32]
    links = _links(m)
    # the shuffle each link writes: that of the consumer block (nin_gc.py: L2 <- 2, L3 <- 2, L4 <- 2, L5 <- 16, L6 <- 4,
    # L7 <- 32 groups; harness cfg), and the 2x2 pools in front of L3 and L6
    assert [lk.sg for lk in links[:6]] == [2, 2, 16, 4, 4, 32]
    assert [None if lk.pool is None else lk.pool[1:] for lk in links[:6]] == [None, (2, 2, 0), None, None, (2, 2, 0), None]
    # every shuffled consumer block had its flag cleared: its producer writes the shuffled plane
    assert not any(getattr(b, "channel_shuffle_flag", 0) for b in m.model.children())
    assert [c.__dict__.get("_mnb_in_shuffle", 1) for c in _quant_convs(m)] == [1, 2, 2, 16, 4, 4, 32]
    E.wbwtab.freeze_inference(m, enable=False)
    assert [getattr(b, "channel_shuffle_flag", None) for b in m.model.children()] == flags
    assert all("_mnb_in_shuffle" not in c.__dict__ for c in _quant_convs(m))


def _layer_shapes(name, batch=256):
    """ConvShape of the forward of every quantized layer (convs 2 .. L-1) at batch 256 on 32 x 32 images"""
    from micronet_b200 import functional as F_
    base = H.build_float_model(name, seed=1)
    shapes = []
    for c in [k for k in base.modules() if isinstance(k, nn.Conv2d)][1:-1]:
        c.register_forward_pre_hook(lambda mod, inp: shapes.append(
            F_._shape_struct(inp[0].shape, mod.weight.shape, mod.stride, mod.padding, mod.dilation, mod.groups)))
    base.to("meta").eval()(torch.empty(batch, 3, 32, 32, device="meta"))
    return shapes


# the quantized layers whose plan at terms (3, 1) is segmented (long K loop): mnb_pk_conv_post refuses them, so they write
# fp32 and the stem producer (mnb_bn_relu_pack_terms_fwd) writes their consumer's term planes from it, as it does behind
# every shuffled link (wbwtab._epilogue_hand_off)
SEGMENTED = {"nin": {3, 6}, "nin_gc": set()}


@pytest.mark.parametrize("name", ["nin", "nin_gc"])
def test_record_table_at_terms_3_1(name):
    """mnb_pk_conv_plan_ex of every quantized layer at batch 256 and how its output reaches its consumer"""
    from micronet_b200 import _lib as L
    shapes = _layer_shapes(name)
    assert len(shapes) == 7
    m = _model(name, 3)
    import micronet_b200 as E
    E.wbwtab.freeze_inference(m)
    links = _links(m)
    print(f"\n{name}: layer  C->K  g  RxS  HxW | Nt MT nstage smem_bytes segmented npairs | hand-off")
    seg = set()
    for i, sh in enumerate(shapes):
        out = (ctypes.c_int32 * 21)()
        rc = L.load().mnb_pk_conv_plan_ex(ctypes.byref(sh), 0, 3, 1, out, 21)
        assert rc == 0, f"L{i + 1} outside the packed-operand cover at terms (3, 1)"
        assert out[18] == 3, "one piece product per activation piece"
        if out[16]:
            seg.add(i + 1)
        how = ("fp32 to the un-quantized head" if links[i] is None else
               "fp32, then the stem producer writes the term planes" if out[16] or links[i].sg > 1 else
               "epilogue writes the term planes")
        print(f"  L{i + 1} {sh.in_c}->{sh.out_c} g{sh.groups} {sh.ker_h}x{sh.ker_w} {sh.in_h}x{sh.in_w} | "
              f"{out[2]} {out[4]} {out[7]} {out[8]} {out[16]} {out[18]} | {how}")
    assert seg == SEGMENTED[name]
    assert [lk is not None for lk in links] == [True] * 6 + [False]


def test_a2_plan_unchanged():
    import micronet_b200 as E
    from micronet_b200 import _lib as L
    m = E.wbwtab.prepare(H.build_float_model("nin_gc", seed=1), W=3, A=2, fuse_bn=True).eval()
    E.wbwtab.freeze_inference(m)
    xnor, bf16 = ("xnor", L.XNOR_BITS), ("xnor", L.XNOR_PM1_BF16)
    assert _plan(m) == [xnor] * 6 + [bf16] and _links(m) == [None] * 7
    assert not _overridden(m, nn.BatchNorm2d) and not _overridden(m, nn.MaxPool2d)


def test_all_zero_ternary_channel_and_w32_stay_unfrozen():
    import micronet_b200 as E
    m = _model("nin", 3)
    convs = _quant_convs(m)
    with torch.no_grad():
        convs[3].weight[5].zero_()           # alpha 0 / 0 on one channel of L4
    E.wbwtab.freeze_inference(m)
    # L4 stays un-frozen, and so does L3's link into it (L3 then writes fp32)
    assert _plan(m) == [TERMS, TERMS, FP32, None, TERMS, TERMS, FP32]
    assert _links(m)[2] is None
    E.wbwtab.freeze_inference(m, enable=False)
    m32 = _model("nin", 32)
    E.wbwtab.freeze_inference(m32)
    assert _plan(m32) == [None] * 7
    assert not _overridden(m32, nn.BatchNorm2d) and not _overridden(m32, nn.MaxPool2d)


def test_training_mode_stays_unfrozen():
    import micronet_b200 as E
    m = _model("nin", 2).train()
    E.wbwtab.freeze_inference(m)
    assert _plan(m) == [None] * 7


def test_symbols_exported():
    from micronet_b200 import _lib as L
    lib = L.load()
    for name in ("mnb_pk_plane_maxpool_terms", "mnb_bn_relu_pack_terms_fwd"):
        assert hasattr(lib, name) and name in L.PROTOTYPES
    assert [f for f, _ in L.PkPost._fields_][-1] == "terms_out"


def test_host_refusals_launch_nothing():
    """host-side refusals of the new entry points (no device pointer is touched before them)"""
    from micronet_b200 import _lib as L
    E_ARG = -1
    lib = L.load()
    n0 = L.launch_count()
    fake = 1 << 20      # 16-byte aligned, never dereferenced: every call below returns before a launch
    assert lib.mnb_pk_plane_maxpool_terms(fake, 2, 16, 8, 8, 3, 2, 2, 3, fake + 4096, None) == L.E_UNSUPPORTED   # 2p > k
    assert lib.mnb_pk_plane_maxpool_terms(fake, 2, 16, 8, 8, 2, 2, 0, 4, fake + 4096, None) == E_ARG          # terms
    assert lib.mnb_bn_relu_pack_terms_fwd(fake, 2, 12, 64, None, None, None, None, 1, 1, 3, fake + 4096, None) == L.E_UNSUPPORTED
    assert lib.mnb_bn_relu_pack_terms_fwd(fake, 2, 16, 64, fake, None, None, None, 1, 1, 3, fake + 4096, None) == E_ARG
    assert lib.mnb_bn_relu_pack_terms_fwd(fake, 2, 16, 64, None, None, None, None, 1, 3, 3, fake + 4096, None) == L.E_UNSUPPORTED
    # the term-plane epilogue stores whole 8-channel units: C_out per group % 8 != 0 is refused, ungrouped (12) or grouped
    for k, g in ((12, 1), (20, 1), (24, 2)):
        sh = L.ConvShape(2, 16, 8, 8, k, 1, 1, 1, 1, 0, 0, 1, 1, g)
        post = L.PkPost(None, 1, 0, fake + 8192)
        post.terms_out = 3
        assert lib.mnb_pk_conv_post(ctypes.byref(sh), fake, 3, fake + 4096, 1, None, None, 1.0, None, None, ctypes.byref(post),
                                    fake + 12288, None) == L.E_UNSUPPORTED, (k, g)
    assert L.launch_count() == n0


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_term_plane_instances_do_not_spill():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for name, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        if re.search(r"pk_conv_kernelILb0ELi\d+ELb0ELb0ELb1EE", name) or "plane_maxpool_terms_kernel" in name or \
                "bn_relu_pack_terms_kernel" in name:
            funcs[name] = len(re.findall(r"\b(?:STL|LDL)(?:\.\w+)*\b", body))
    nts = {int(m.group(1)) for n in funcs if (m := re.search(r"pk_conv_kernelILb0ELi(\d+)E", n))}
    assert nts == {16, 32, 48, 64, 96, 128} and len(funcs) == 8, sorted(funcs)
    assert all(v == 0 for v in funcs.values()), funcs
