"""CPU side of frozen IAO inference graphs of NIN / NIN-GC (iao.freeze_inference, block links): host refusals of the
requantizing plane max-pool (fake device pointers: nothing may be launched), its 256-entry table against the oracle's IAO
quantizer, and the graph rewrite on CPU-built models - which convs link, which pools run on the plane, which shuffles move,
that ResNet-18 keeps exactly its conv -> conv and QuantAdd -> conv links, and that ``enable=False`` restores the module
tree, the state_dict and every ``channel_shuffle_flag``."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from harness import models as zoo

FAKE = 1 << 20          # never dereferenced: every call below is refused on the host
NIN_CFG = [64, 32, 32, 64, 64, 64, 64, 64]
GC_CFG = [32, 32, 32, 64, 64, 64, 128, 128]


def _iao_q(bits=8, q_type=0, qmin=None, qmax=None):
    from micronet_b200 import _lib as L
    half = 1 << (bits - 1)
    qmin = -half if qmin is None else qmin
    qmax = half - 1 if qmax is None else qmax
    return L.ActQParams(L.ACT_IAO, bits, qmin, qmax, q_type, FAKE, FAKE, FAKE, FAKE)


def test_requant_pool_refusals():
    from micronet_b200 import _lib as L
    lib = L.load()
    pool = lib.mnb_pk_plane_maxpool_requant
    q8, n0 = _iao_q(8), L.launch_count()

    def call(*a, q_in=q8, q_out=q8, out=FAKE + 4096):
        return pool(FAKE, 2, 64, 8, 8, *a, None if q_in is None else C.byref(q_in), None if q_out is None else C.byref(q_out),
                    out, None)

    assert call(2, 2, 0, 0, q_in=None) == -1
    assert call(2, 2, 0, 1, q_out=None) == -1
    assert call(2, 2, 0, 0, out=FAKE) == -1                                     # in place
    assert call(2, 2, 0, 0, out=FAKE + 8) == -1                                 # misaligned output
    assert call(3, 2, 2, 0) == L.E_UNSUPPORTED                                  # 2 * p > k
    assert call(0, 2, 0, 1) == L.E_UNSUPPORTED
    assert call(2, 2, 0, 0, q_in=_iao_q(8, q_type=1, qmin=0, qmax=255)) == L.E_UNSUPPORTED     # asymmetric pool
    assert call(2, 2, 0, 1, q_out=_iao_q(8, q_type=1, qmin=0, qmax=255)) == L.E_UNSUPPORTED    # asymmetric consumer
    assert b"symmetric IAO" in lib.mnb_last_error()
    dorefa = L.ActQParams(L.ACT_DOREFA, 4, 0, 15, 0, None, None, None, None)
    assert call(2, 2, 0, 0, q_in=dorefa) == L.E_UNSUPPORTED
    assert call(2, 2, 0, 0, q_out=dorefa) == L.E_UNSUPPORTED
    assert call(2, 2, 0, 0, q_in=_iao_q(1, qmin=-1, qmax=0)) == L.E_UNSUPPORTED               # 1 bit
    nulls = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, None, None, None, None)
    assert call(2, 2, 0, 0, q_in=nulls) == -1
    assert L.launch_count() == n0


def _host_table(s_in, s_out, qmin_in, qmax_in, qmin_out, qmax_out):
    """the table mnb_pk_plane_maxpool_requant builds, one entry per stored level -128..127, in numpy fp32: the pool's
    fake-quantized value fl(L * s_in), then the consumer's clamp(sign(t) * floor(|t| + 0.5)) with t = fl(v / s_out)"""
    f = np.float32
    lev = np.clip(np.arange(-128, 128), qmin_in, qmax_in).astype(f)
    v = (lev + f(0)) * f(s_in)
    t = v / f(s_out)
    r = np.sign(t) * np.floor(np.abs(t) + f(0.5))
    return np.clip(r, f(qmin_out), f(qmax_out)).astype(f), v


# (s_pool, s_consumer, pool bits, consumer bits): exact half-way ties (0.5 / 1.0, 0.75 / 0.5), fp32-rounded quotients next to
# ties (0.1 / 0.2, 0.3 / 0.6), both clamps of the consumer (s_consumer << s_pool), 4-bit consumers, a scale of FLT_EPSILON
CASES = [(0.5, 1.0, 8, 8), (0.75, 0.5, 8, 8), (0.1, 0.2, 8, 8), (0.3, 0.6, 8, 8), (0.02, 0.003, 8, 8), (1.0, 0.01, 8, 8),
         (0.05, 0.35, 8, 4), (0.0123, 0.0456, 8, 8), (2.0 ** -23, 2.0 ** -20, 8, 8), (0.07, 0.07, 4, 8), (0.1, 0.1, 8, 8)]


@pytest.mark.parametrize("s_in,s_out,b_in,b_out", CASES)
def test_requant_table_matches_oracle_quantizers(s_in, s_out, b_in, b_out):
    from oracle import reference_port as O
    qp = O._iao_act_quantizer(b_in, 0, False, False, 0.9999).eval()
    qc = O._iao_act_quantizer(b_out, 0, False, False, 0.9999).eval()
    qp.scale.fill_(s_in)
    qc.scale.fill_(s_out)
    lo_in, hi_in = int(qp.quant_min_val), int(qp.quant_max_val)
    lo_out, hi_out = int(qc.quant_min_val), int(qc.quant_max_val)
    tab, v = _host_table(s_in, s_out, lo_in, hi_in, lo_out, hi_out)
    # the oracle pool quantizer's output for inputs that land on each of its levels, requantized by the oracle consumer
    lev = torch.arange(lo_in, hi_in + 1, dtype=torch.float32)
    xp = qp(lev * qp.scale)
    assert torch.equal(qp.levels(xp), lev)
    assert np.array_equal(xp.numpy(), v[lo_in + 128:hi_in + 129])
    want = qc.levels(xp).numpy()
    assert np.array_equal(tab[lo_in + 128:hi_in + 129], want)
    # monotone, so the table commutes with the window max
    assert (np.diff(tab) >= 0).all()


def test_requant_cases_hit_ties_and_clamps():
    ties = clamp_lo = clamp_hi = 0
    for s_in, s_out, b_in, b_out in CASES:
        half_in, half_out = 1 << (b_in - 1), 1 << (b_out - 1)
        tab, v = _host_table(s_in, s_out, -half_in, half_in - 1, -half_out, half_out - 1)
        t = v / np.float32(s_out)
        ties += int((np.abs(t) % 1 == 0.5).sum())
        clamp_lo += int((t < -half_out).sum())
        clamp_hi += int((t > half_out - 1).sum())
    assert ties > 0 and clamp_lo > 0 and clamp_hi > 0, (ties, clamp_lo, clamp_hi)


def _model(kind, q_type=0, bn_fuse=True, ptq=False, q_level=0):
    from micronet_b200 import iao
    torch.manual_seed(0)
    if kind == "resnet":
        base = zoo.resnet18()
    else:
        base = zoo.init_like_reference(zoo.NIN(NIN_CFG) if kind == "nin" else zoo.NINGC(GC_CFG))
    return iao.prepare(base, a_bits=8, w_bits=8, q_type=q_type, q_level=q_level, bn_fuse=bn_fuse, ptq=ptq).eval()


def _snapshot(m):
    return repr(m), {k: v.clone() for k, v in m.state_dict().items()}, \
        [getattr(k, "channel_shuffle_flag", None) for k in m.modules()]


def _block_links(m):
    """per child of model.model: does its conv link to the next block / does the pool run on the plane?"""
    from micronet_b200 import iao
    out = []
    for k in m.model.children():
        conv = next(iter(k.children()), None)
        if isinstance(conv, iao.QuantConv2d):
            out.append(isinstance(conv.__dict__.get("_post_consumer"), iao._BlockLink))
        else:
            out.append("forward" in k.__dict__)
    return out


# per child of model.model (stem, two blocks, pool, three blocks, pool, two blocks, head, avg-pool): NIN links every block
# to the next and runs both pools on the plane.  NIN-GC links its two unshuffled pairs (stem -> block 1, block 7 -> head);
# its shuffled links are taken only across a pool with int8 planes (blocks 2 and 5 and both pools); the grouped 3x3 layers
# (blocks 3 and 6) and the other 1x1 blocks keep writing fp32.  The head writes fp32, the avg-pool is untouched.
WANT = {("nin", False): [True] * 10 + [False, False], ("nin", True): [True] * 10 + [False, False],
        ("gc", False): [True] + [False] * 8 + [True, False, False],
        ("gc", True): [True, False, True, True, False, False, True, True, False, True, False, False]}


@pytest.mark.parametrize("kind", ["nin", "gc"])
@pytest.mark.parametrize("ptq", [False, True])
def test_block_links_and_restore(kind, ptq):
    _check_links_and_restore(kind, ptq, False)


@pytest.mark.parametrize("kind", ["nin", "gc"])
@pytest.mark.parametrize("ptq", [False, True])
def test_block_links_and_restore_int8(kind, ptq):
    _check_links_and_restore(kind, ptq, True)


def _check_links_and_restore(kind, ptq, i8):
    from micronet_b200 import iao
    m = _model(kind, ptq=ptq)
    before = _snapshot(m)
    iao.freeze_inference(m, int8=i8)
    want = WANT[(kind, i8)]
    assert _block_links(m) == want
    kids = list(m.model.children())
    for i in (3, 7):
        if not want[i]:
            continue
        link = next(iter(kids[i - 1].children())).__dict__["_post_consumer"]
        assert link.pool[0] is kids[i] and link.pool[1:] == ((3, 2, 1) if kind == "nin" else (2, 2, 0))
        assert link.cconv is next(iter(kids[i + 1].children()))
    # the ReLU of every linked block passes the plane through, the others run as usual
    assert [("forward" in k.relu.__dict__) for k in kids if hasattr(k, "relu")] == [w for k, w in zip(kids, want)
                                                                                    if hasattr(k, "relu")]
    if kind == "gc":
        # a shuffle moves into the producer only with its link: blocks 3 and 6 behind the int8 pool links
        sg = [next(iter(k.children())).__dict__.get("_mnb_in_shuffle", 1) for k in kids if hasattr(k, "channel_shuffle_flag")]
        flags = [k.channel_shuffle_flag for k in kids if hasattr(k, "channel_shuffle_flag")]
        if i8:
            assert sg == [1, 1, 1, 2, 1, 1, 4, 1, 1] and flags == [0, 0, 1, 0, 1, 1, 0, 1, 0]
        else:
            assert sg == [1] * 9 and _snapshot(m)[2] == before[2]
    assert m.state_dict().keys() == before[1].keys()
    assert all(torch.equal(v, before[1][k]) for k, v in m.state_dict().items())
    iao.freeze_inference(m, int8=i8)                             # freezing twice rewrites from the restored graph
    assert _block_links(m) == want
    iao.freeze_inference(m, enable=False)
    after = _snapshot(m)
    assert after[0] == before[0] and after[2] == before[2]
    assert all(torch.equal(v, before[1][k]) for k, v in after[1].items())
    assert not any(k in c.__dict__ for c in m.modules() for k in ("forward", "_post_consumer", "_mnb_in_shuffle"))


def test_shuffled_links_hand_over_int8_planes_only():
    """a shuffled link of an int8 graph restricts its consumer to int8 planes: where the consumer would read bf16 the
    producer writes fp32 instead of a shuffled bf16 plane"""
    from micronet_b200 import iao
    m = _model("gc")
    iao.freeze_inference(m, int8=True)
    kids = list(m.model.children())
    shuffled = next(iter(kids[2].children())).__dict__["_post_consumer"]
    plain = next(iter(kids[0].children())).__dict__["_post_consumer"]
    assert shuffled.sg == 2 and plain.sg == 1
    spec = shuffled.cconv.activation_quantizer.act_spec()
    assert shuffled.consumer(spec, True).formats == ("i8",)
    assert shuffled.consumer(spec, False).format((2, GC_CFG[2], 16, 16)) is None      # a bf16 consumer: no hand-off
    assert plain.consumer(plain.cconv.activation_quantizer.act_spec(), False).formats is None
    iao.freeze_inference(m, enable=False)


def test_handoff_false_links_no_blocks():
    from micronet_b200 import iao
    m = _model("gc")
    before = _snapshot(m)
    iao.freeze_inference(m, handoff=False)
    assert _block_links(m) == [False] * 12
    assert _snapshot(m)[2] == before[2]


@pytest.mark.parametrize("why", ["q_type1", "bn_live"])
def test_refused_graphs_link_nothing(why):
    from micronet_b200 import iao
    m = _model("gc", q_type=1) if why == "q_type1" else _model("gc", bn_fuse=False)
    before = _snapshot(m)
    iao.freeze_inference(m, int8=True)
    assert _block_links(m) == [False] * 12
    assert _snapshot(m)[2] == before[2]
    assert not any("forward" in c.__dict__ for c in m.modules())
    iao.freeze_inference(m, enable=False)


def test_pool_outside_cover_is_not_crossed():
    from micronet_b200 import iao
    m = _model("gc")
    old = m.model[3]
    m.model[3] = iao.QuantMaxPool2d(kernel_size=2, stride=2, padding=0, ceil_mode=True)   # ceil mode: not covered
    m.model[3].activation_quantizer.load_state_dict(old.activation_quantizer.state_dict())
    m.eval()
    iao.freeze_inference(m, int8=True)
    assert _block_links(m) == [True, False, False, False, False, False, True, True, False, True, False, False]
    assert m.model[4].channel_shuffle_flag == 1 and "_mnb_in_shuffle" not in m.model[4].conv.__dict__
    iao.freeze_inference(m, enable=False)


def _all_links(m):
    names = {id(mod): n for n, mod in m.named_modules()}
    out = set()
    for n, mod in m.named_modules():
        link = mod.__dict__.get("_post_consumer")
        if link is not None:
            out.add((n, names[id(link[0])], link[1]))
    return out


def test_resnet18_links_and_undo_record():
    """ResNet-18 keeps exactly the links of its two rules: adjacent convs of a residual_function, QuantAdd -> first conv of
    the next block; no block link, no override"""
    from micronet_b200 import iao
    m = _model("resnet")
    iao.freeze_inference(m, int8=True)
    blocks = [f"conv{s}_x.{i}" for s in range(2, 6) for i in range(2)]
    want = {(f"{b}.residual_function.0", f"{b}.residual_function.3", True) for b in blocks}
    want |= {(f"{b0}.add", f"{b1}.residual_function.0", False) for b0, b1 in zip(blocks, blocks[1:])}
    assert _all_links(m) == want
    assert not any("forward" in c.__dict__ or "_mnb_in_shuffle" in c.__dict__ for c in m.modules())
    # the undo record holds the flags, the folded ReLUs and the links above: no block link moved a shuffle or a pool
    flags = {"_frozen_inference", "_int8", "_frozen", "_int_levels", "_pre_relu", "_fuse_relu", "_post_consumer"}
    for rec in m.__dict__["_mnb_iao_undo"]:
        assert (rec[0] == "dict" and rec[2] in flags) or (rec[0] == "child" and type(rec[3]) is nn.ReLU), rec
    iao.freeze_inference(m, enable=False)
    assert _all_links(m) == set()
