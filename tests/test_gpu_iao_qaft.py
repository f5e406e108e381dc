"""QAFT hand-offs of BN-fused IAO NIN / NIN-GC models on the GPU (iao.prepare(bn_fuse=True, qaft=True, fuse=True)):

* every linked producer's epilogue writes the plane and STE mask that the consumer's pack_act of ReLU(y) writes, bit for bit
  (with a pool in between: the pool quantizer's levels, and relu'(y) & its pass flags);
* the training plane pool, forward and backward, equals ActQuantFn + ATen max_pool2d (+ their backward and ReLU's), bit for
  bit, on inputs full of ties;
* in a full training forward every link fires: each linked conv and pool hands its consumer a tagged plane, also where a
  conv both reads a handed plane and writes one (a chain of pooled blocks);
* one QAFT step (W8A8 and W4A4, NIN, NIN-GC and that chain), linked against un-linked from identical state: loss, every
  gradient and every parameter after FlatAdam are bitwise equal; three CUDA-graph replays equal eager steps;
* an un-linked QAFT step of NIN matches the oracle port layer by layer (tests.test_gpu_parity's teacher-forced contract).

The quantizers are calibrated by two QAT forwards first (the README's QAT -> QAFT flow): fresh QAFT quantizers have the
unit scale and an empty observer range, whose STE passes nothing."""
import copy

import pytest
import torch
import torch.nn.functional as TF

from harness import models as zoo
from harness import train as H

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NIN_CFG = [192, 160, 96, 192, 192, 192, 192, 192]
GC_CFG = [256, 256, 256, 512, 512, 512, 1024, 1024]


class Chain(zoo._SeqNet):
    """conv-bn-relu blocks with a 3 / 2 / 1 pool behind each: the middle block reads a handed plane and writes one"""

    def __init__(self):
        super().__init__()
        self.model = torch.nn.Sequential(zoo.ConvBNReLU(3, 64, 3, 1, 1), torch.nn.MaxPool2d(3, 2, 1),
                                         zoo.ConvBNReLU(64, 96, 3, 1, 1), torch.nn.MaxPool2d(3, 2, 1),
                                         zoo.ConvBNReLU(96, 10, 1), torch.nn.AvgPool2d(8))


def _float_model(kind):
    return zoo.init_like_reference({"nin": lambda: zoo.NIN(NIN_CFG), "gc": lambda: zoo.NINGC(GC_CFG), "chain": Chain}[kind]())


def _calibrated(kind, bits=8, ptq=False, batch=16, seed=1):
    """(float model, state_dict of a QAT model after two training-mode forwards): scales, ranges and running statistics"""
    from micronet_b200 import iao
    torch.manual_seed(seed)
    base = _float_model(kind)
    qat = iao.prepare(copy.deepcopy(base), a_bits=bits, w_bits=bits, bn_fuse=True, ptq=ptq).to(DEV).train()
    with torch.no_grad():
        for s in (11, 12):
            qat(H.synthetic_batch(batch, 32, seed=s, device=DEV)[0])
    return base, qat.state_dict()


def _qaft(base, state, fuse, bits=8, ptq=False):
    from micronet_b200 import iao
    m = iao.prepare(copy.deepcopy(base), a_bits=bits, w_bits=bits, bn_fuse=True, qaft=True, ptq=ptq, fuse=fuse).to(DEV)
    m.load_state_dict(state)
    return m.train()


def _octet_bits(mask):
    """bool [b, c, h, w] -> bits8 [b, c/8, h, w] (bit j = channel 8 * (c/8) + j)"""
    b, c, h, w = mask.shape
    m = mask.view(b, c // 8, 8, h, w).to(torch.int32)
    return (m << torch.arange(8, device=mask.device, dtype=torch.int32).view(1, 1, 8, 1, 1)).sum(2).to(torch.uint8)


def _links(m):
    return [(conv, conv.__dict__["_mnb_train_link"]) for conv in m.modules() if "_mnb_train_link" in conv.__dict__]


# linked producers per model: NIN's two pooled pairs; NIN-GC's pools sit in front of shuffled blocks, so it links nothing
N_LINKS = {"nin": 2, "gc": 0, "chain": 2}


@pytest.mark.parametrize("kind", ["nin", "chain"])
def test_epilogue_plane_and_bits_equal_pack_act(kind):
    from micronet_b200 import pk as PK
    base, state = _calibrated(kind)
    ref, fused = _qaft(base, state, False), _qaft(base, state, True)
    seen = {}
    names = {id(mod): n for n, mod in ref.named_modules()}
    hooks = [mod.register_forward_hook(lambda mod, i, o: seen.__setitem__(names[id(mod)], (i[0].detach().clone(),
                                                                                           o.detach().clone())))
             for mod in ref.modules() if isinstance(mod, torch.nn.Conv2d)]
    x, _ = H.synthetic_batch(8, 32, seed=5, device=DEV)
    with torch.no_grad():
        ref(x)
    for h in hooks:
        h.remove()
    fnames = {id(mod): n for n, mod in fused.named_modules()}
    links = _links(fused)
    assert len(links) == N_LINKS[kind]
    for conv, link in links:
        inp, y = seen[fnames[id(conv)]]
        with torch.no_grad():
            out = conv(inp)
        pre = out._mnb_pk_pre
        assert pre[0] is link.target, fnames[id(conv)]
        q = (link.pool[0] if link.pool is not None else link.cconv).activation_quantizer.act_spec()
        plane, bits = PK.pack_act(torch.relu(y).contiguous(), q.struct(), 1, want_bits=True)
        assert torch.equal(pre[1], plane), fnames[id(conv)]
        assert torch.equal(pre[4]["bits"], bits & _octet_bits(y > 0)), fnames[id(conv)]


@pytest.mark.parametrize("shape,k,s,p", [((4, 96, 32, 32), 3, 2, 1), ((4, 192, 16, 16), 3, 2, 1), ((4, 256, 32, 32), 2, 2, 0),
                                         ((2, 64, 9, 7), 3, 2, 1)])
@pytest.mark.parametrize("bits", [8, 4])
def test_plane_pool_equals_actquant_maxpool(shape, k, s, p, bits):
    from micronet_b200 import iao, functional as F_, pk as PK
    torch.manual_seed(3)
    qp = iao.QuantMaxPool2d(k, s, p, a_bits=bits, qaft=True).to(DEV).activation_quantizer
    qc = iao.QuantMaxPool2d(k, s, p, a_bits=bits, qaft=True).to(DEV).activation_quantizer
    half = 1 << (bits - 1)
    qp.scale.fill_(0.05)
    qp.observer.min_val.fill_(-0.05 * (half - 3))
    qp.observer.max_val.fill_(0.05 * (half - 3))          # some levels past the range: STE zeros
    qc.scale.fill_(0.07)
    qc.observer.min_val.fill_(-0.07 * (half - 2))
    qc.observer.max_val.fill_(0.07 * (half - 2))
    sp, sc = qp.act_spec(), qc.act_spec()
    # levels of a few values only: every window is full of ties, and exact zeros for ReLU
    y = (torch.randint(-3, half + 2, shape, device=DEV).float() * 0.05).contiguous()
    b, c, h, w = shape
    plane, pbits = PK.pack_act(torch.relu(y), sp.struct(), 1, want_bits=True)
    pbits = pbits & _octet_bits(y > 0)
    out, arg, cbits = PK.plane_maxpool_requant_train(plane, b, c, h, w, k, s, p, sp.struct(), sc.struct())
    yr = y.clone().requires_grad_(True)
    xq = F_.ActQuantFn.apply(torch.relu(yr), sp)
    m, idx = TF.max_pool2d(xq, k, s, p, return_indices=True)
    want_plane, want_bits = PK.pack_act(m.detach().contiguous(), sc.struct(), 1, want_bits=True)
    assert torch.equal(out, want_plane) and torch.equal(cbits, want_bits)
    oh, ow = m.shape[2], m.shape[3]
    ih, iw = idx // w, idx % w
    r = ih - (torch.arange(oh, device=DEV).view(1, 1, oh, 1) * s - p)
    q = iw - (torch.arange(ow, device=DEV).view(1, 1, 1, ow) * s - p)
    got = arg.permute(0, 1, 4, 2, 3).reshape(b, c, oh, ow).long()
    assert torch.equal(got, r * k + q)
    g = torch.randn(m.shape, device=DEV)
    m.backward(g)
    dx = PK.plane_maxpool_requant_bwd(g, arg, pbits, b, c, h, w, k, s, p, sp.frozen().struct())
    assert torch.equal(dx, yr.grad)
    assert (dx != 0).any() and (dx == 0).any()


@pytest.mark.parametrize("kind", ["nin", "gc", "chain"])
def test_every_link_fires_in_a_training_forward(kind, monkeypatch):
    """a link that silently falls back (the producer writes fp32, the pool fake-quantizes it) computes the same numbers, so
    the step tests cannot see it: here every linked conv's and pool's output must carry the plane and mask it hands over"""
    from micronet_b200 import iao
    base, state = _calibrated(kind)
    m = _qaft(base, state, True)
    links = _links(m)
    assert len(links) == N_LINKS[kind]
    tagged = {}

    def hook(key, target):
        def h(mod, inp, out):
            pre = getattr(out, "_mnb_pk_pre", None)
            tagged[key] = pre is not None and pre[0] is target and "bits" in pre[4]
        return h

    hooks = []
    for conv, link in links:
        hooks.append(conv.register_forward_hook(hook(("conv", id(conv)), link.target)))
        if link.pool is not None:
            hooks.append(link.pool[0].register_forward_hook(hook(("pool", id(conv)), link.cconv)))
    # the class forward of QuantMaxPool2d (fake-quant + ATen max-pool) may run only for the pools no link crosses
    fell_back = []
    plain = iao.QuantMaxPool2d.forward
    monkeypatch.setattr(iao.QuantMaxPool2d, "forward", lambda self, x: fell_back.append(self) or plain(self, x))
    x, t = H.synthetic_batch(8, 32, seed=7, device=DEV)
    TF.cross_entropy(m(x), t).backward()
    for h in hooks:
        h.remove()
    assert len(tagged) == 2 * N_LINKS[kind] and all(tagged.values()), tagged
    linked_pools = {id(link.pool[0]) for _, link in links if link.pool is not None}
    assert not any(id(p) in linked_pools for p in fell_back)
    assert len(fell_back) == sum(1 for k in m.modules() if isinstance(k, iao.QuantMaxPool2d)) - len(linked_pools)


def _step(m, x, t, opt):
    loss = TF.cross_entropy(m(x), t)
    opt.zero_grad()
    loss.backward()
    grads = [p.grad.clone() for p in m.parameters()]
    opt.step()
    return loss.detach(), grads


@pytest.mark.parametrize("kind", ["nin", "gc", "chain"])
@pytest.mark.parametrize("bits", [8, 4])
def test_qaft_step_linked_equals_unlinked(kind, bits):
    from micronet_b200 import FlatAdam, _lib as L
    base, state = _calibrated(kind, bits=bits, batch=32)
    ref, fused = _qaft(base, state, False, bits), _qaft(base, state, True, bits)
    o_ref = FlatAdam(ref.parameters(), lr=1e-3, weight_decay=1e-5)
    o_fused = FlatAdam(fused.parameters(), lr=1e-3, weight_decay=1e-5)
    for s in (21, 22):
        x, t = H.synthetic_batch(32, 32, seed=s, device=DEV)
        la, ga = _step(ref, x, t, o_ref)
        n0 = L.launch_count()
        lb, gb = _step(fused, x, t, o_fused)
        torch.cuda.synchronize()
        assert L.launch_count() > n0
        assert torch.equal(la, lb)
        for (n, _), a, b_ in zip(ref.named_parameters(), ga, gb):
            assert torch.equal(a, b_), n
        assert any(g.abs().sum() > 0 for g in gb[:4])
        for (n, a), b_ in zip(ref.named_parameters(), fused.parameters()):
            assert torch.equal(a, b_), n
    L.tc_check()


def test_qaft_graph_replay_equals_eager():
    base, state = _calibrated("nin", batch=32)
    eager, graphed = _qaft(base, state, True), _qaft(base, state, True)
    se = H.QatStepper(eager, lr=1e-3, wd=1e-5, flat=True, graph=False)
    sg = H.QatStepper(graphed, lr=1e-3, wd=1e-5, flat=True, graph=True, graph_warmup=1)
    for s in range(4):                     # one eager warm-up step, then the capture and three replays
        x, t = H.synthetic_batch(32, 32, seed=30 + s, device=DEV)
        # (detached at once: a loss kept alive keeps its autograd graph, whose AccumulateGrad nodes would break the capture)
        la, lb = se.step(x, t).detach(), sg.step(x, t).detach()
        torch.cuda.synchronize()
        assert torch.equal(la, lb), s
    assert sg.graph is not None, sg.graph_error
    for (n, a), b_ in zip(eager.named_parameters(), graphed.parameters()):
        assert torch.equal(a, b_), n


def test_unlinked_qaft_step_matches_oracle():
    """the QAFT step of NIN against the independent oracle port: every quantized layer, fed the oracle's own inputs and
    output gradient, reproduces the oracle's output and gradients (tests.test_gpu_parity._teacher_forced: 1e-5 with the
    tie-excuse rules for BN-fused weight levels).  Whole-model logits are not a contract here: one activation level on the
    other side of a rounding tie moves them by far more than the fp32 error of any layer."""
    from oracle import reference_port as O
    from tests.test_gpu_parity import _teacher_forced
    base, state = _calibrated("nin", batch=8)
    em = _qaft(base, state, False)
    om = O.prepare_iao(copy.deepcopy(base), bn_fuse=True, qaft=True, add_type=zoo.Add)
    om.load_state_dict({k: v.cpu() for k, v in state.items()})
    om.train()
    x, t = H.synthetic_batch(4, 32, seed=41)
    _teacher_forced(om, em, x, t)
