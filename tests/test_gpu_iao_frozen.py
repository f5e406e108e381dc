"""Frozen IAO inference graphs of NIN / NIN-GC on level planes (iao.freeze_inference block links): the requantizing plane
max-pool (mnb_pk_plane_maxpool_requant) byte for byte against the composition of existing kernels it replaces, whole
W8A8 bn_fuse models with ``handoff=True`` bitwise against ``handoff=False`` (bf16 and int8, per-channel and per-layer
weights, PTQ, eager and under CUDA-graph replay), and a small NIN-GC against the eval output of the reference's own
``prepare(bn_fuse=True)`` model."""
import copy

import pytest
import torch
import torch.nn.functional as F

from harness import train as H
from harness.wbwtab_infer_probe import _randomise_bn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _tc_clean():
    yield
    from micronet_b200 import _lib as L
    torch.cuda.synchronize()
    L.tc_check()


def _quantizer(scale, bits=8):
    from micronet_b200 import iao
    q = iao.SymmetricQuantizer(bits=bits, observer=iao.MovingAverageMinMaxObserver(q_level="L", out_channels=None),
                               activation_weight_flag=1).to(DEV).eval()
    q.scale.fill_(scale)
    q.observer.max_val.fill_(scale * (q.qmax + 0.5))
    q.observer.min_val.fill_(-scale * (q.qmax + 0.5))
    return q


def _decode_bf16(plane, b, c, h, w):
    return plane.view(torch.bfloat16).view(b, c // 8, h, w, 8).permute(0, 1, 4, 2, 3).reshape(b, c, h, w).float()


def _decode_i8(plane, b, c, h, w):
    return plane.view(torch.int8).view(b, c // 16, h, w, 16).permute(0, 1, 4, 2, 3).reshape(b, c, h, w).float()


# NIN: 3x3 / 2 / 1 pools on 96- and 192-channel 32x32 / 16x16 planes; NIN-GC: 2x2 / 2 / 0 on 256 / 512 channels; batch 256.
# Two pool scales: one from the data (general fp32 rounding) and 2^-4, a power of two, so that the consumer ratio 2.0 makes
# every odd level an exact half-way quotient (t = L / 2: the round-half-away path at ties).  The activations are signed
# (the kernel does not assume a ReLU in front), so the consumer ratio 0.1 reaches both of its clamps.
PLANES = [(256, 96, 32, 32, 3, 2, 1), (256, 192, 16, 16, 3, 2, 1), (256, 256, 32, 32, 2, 2, 0), (256, 512, 16, 16, 2, 2, 0)]
SCALES = [(1.0, 8), (1.37, 8), (0.5, 8), (0.213, 8), (2.0, 8), (0.1, 8), (3.0, 4)]


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
@pytest.mark.parametrize("shape", PLANES, ids=lambda s: "x".join(map(str, s)))
def test_requant_pool_matches_the_kernel_composition(shape, i8):
    from micronet_b200 import functional as F_
    from micronet_b200 import pk as PK
    b, c, h, w, k, s, p = shape
    decode = _decode_i8 if i8 else _decode_bf16
    g = torch.Generator(device=DEV).manual_seed(b + c + h + k)
    y = torch.randn(b, c, h, w, device=DEV, generator=g) * 4.0
    y[:, :, ::5, ::3] = 0.0
    for s_p in (float(y.abs().max()) / 127.0, 2.0 ** -4):
        qp = _quantizer(s_p)
        sp = qp.act_spec()
        plane = PK.pack_act_i8(y, sp.struct()) if i8 else PK.pack_act(y, sp.struct(), 1)[0]
        xq = F_.ActQuantFn.apply(y, sp)
        levels = decode(plane, b, c, h, w)
        assert torch.equal(levels * qp.scale, xq)            # v = fl(L * s_p): what the pool quantizer writes
        pooled = F.max_pool2d(xq, k, s, p)
        pooled_lv = F.max_pool2d(levels, k, s, p)
        oh, ow = pooled.shape[2:]
        for ratio, bits in SCALES:
            qc = _quantizer(s_p * ratio, bits)
            sc = qc.act_spec()
            got = PK.plane_maxpool_requant(plane, b, c, h, w, k, s, p, sp.struct(), sc.struct(), int8=i8)
            want = PK.pack_act_i8(pooled, sc.struct()) if i8 else PK.pack_act(pooled, sc.struct(), 1)[0]
            assert got.shape == want.shape
            assert torch.equal(got, want), (s_p, ratio, bits, int((got != want).sum()))
            lv = decode(got, b, c, oh, ow)
            if ratio < 1:                                    # the upper clamp of the consumer
                assert float(lv.max()) == qc.qmax
            if ratio == 0.1:                                 # and the lower one
                assert float(lv.min()) == qc.qmin
            if ratio == 2.0 and s_p == 2.0 ** -4:            # exact ties went through the device table
                odd = pooled_lv.remainder(2) == 1
                assert bool(odd.any()) and torch.equal(lv[odd].abs(), (pooled_lv[odd].abs() + 1) / 2)


def _calibrated(arch, q_level=0, ptq=False, batch=32):
    import micronet_b200 as E
    base = H.build_float_model(arch, seed=1)
    with torch.no_grad():
        _randomise_bn(base, 7)
    m = E.iao.prepare(base, a_bits=8, w_bits=8, q_type=0, q_level=q_level, bn_fuse=True, ptq=ptq).to(DEV)
    m.train()
    with torch.no_grad():
        for i in range(2):
            m(H.synthetic_batch(batch, 32, seed=20 + i, device=DEV)[0])
    return m.eval()


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


def _pool_outputs(m):
    """forward hooks on the pools between blocks: the device of what each one returned ("meta": it ran on the plane)"""
    from micronet_b200 import iao
    seen, hooks = [], []
    for mod in m.model.children():
        if isinstance(mod, iao.QuantMaxPool2d):
            hooks.append(mod.register_forward_hook(lambda _m, _i, out: seen.append(out.device.type)))
    return seen, hooks


@pytest.mark.parametrize("arch", ["nin", "nin_gc"])
@pytest.mark.parametrize("q_level,ptq", [(0, False), (1, False), (0, True)], ids=["per_channel", "per_layer", "ptq"])
# batch 256: the batch the benchmark runs the NIN models at
@pytest.mark.parametrize("i8,batch", [(False, 32), (True, 32), (False, 256), (True, 256)],
                         ids=["bf16", "int8", "bf16_b256", "int8_b256"])
def test_handoff_logits_bitwise(arch, q_level, ptq, i8, batch):
    from micronet_b200 import iao
    m = _calibrated(arch, q_level, ptq)
    x = H.synthetic_batch(batch, 32, seed=5, device=DEV)[0]
    with torch.no_grad():
        plain = m(x)
    off = copy.deepcopy(m)
    iao.freeze_inference(off, handoff=False, int8=i8)
    iao.freeze_inference(m, int8=i8)
    seen, hooks = _pool_outputs(m)
    with torch.no_grad():
        want, got = off(x), m(x)
    for hk in hooks:
        hk.remove()
    # NIN: both pools run on the producer's level plane.  NIN-GC: its pools sit in front of shuffling blocks, linked only
    # with int8 planes (iao._shuffled_link_pays); with bf16 planes they run as usual
    assert seen == (["meta", "meta"] if arch == "nin" or i8 else ["cuda", "cuda"]), seen
    assert torch.equal(got, want)
    if not i8:
        assert torch.equal(got, plain)                       # the un-frozen eval forward, bit for bit
    assert torch.equal(_graph_logits(m, x), want)
    assert torch.equal(_graph_logits(off, x), want)
    # restore: the un-frozen forward again, shuffles back in their blocks
    iao.freeze_inference(m, enable=False)
    with torch.no_grad():
        assert torch.equal(m(x), plain)


def test_training_mode_after_freeze_runs_unfrozen():
    """a frozen NIN-GC put back into training mode runs its usual forward: the moved shuffles are applied by the convs"""
    from micronet_b200 import iao
    m = _calibrated("nin_gc", batch=8)
    ref = copy.deepcopy(m)
    iao.freeze_inference(m)
    x = H.synthetic_batch(8, 32, seed=9, device=DEV)[0]
    with torch.no_grad():
        m.train(), ref.train()
        a, b = m(x), ref(x)
    assert torch.equal(a, b)


@pytest.mark.parametrize("i8", [False, True], ids=["bf16", "int8"])
def test_small_nin_gc_against_the_reference(i8):
    from micronet_b200 import iao
    from harness import models as zoo
    from tests.oracle_util import load_golden, rel_err
    gold = load_golden("iao", "frozen_nin_gc_w8a8")
    m = iao.prepare(zoo.NINGC([32, 32, 32, 64, 64, 64, 128, 128]), a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True,
                    pretrained_model=True)
    m.load_state_dict({k[11:]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("calibrated.")})
    m = m.to(DEV).eval()
    x = torch.from_numpy(gold["x"]).to(DEV)
    off = copy.deepcopy(m)
    iao.freeze_inference(off, handoff=False, int8=i8)
    iao.freeze_inference(m, int8=i8)
    with torch.no_grad():
        y, y_off = m(x), off(x)
    assert torch.equal(y, y_off)
    # 8-bit activation levels of 9 layers: one level on the other side of a rounding tie moves a logit by ~1e-4 relative
    assert rel_err(y, gold["y"]) <= 2e-4, rel_err(y, gold["y"])
