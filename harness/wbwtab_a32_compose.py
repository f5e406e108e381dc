"""The reference chain of a frozen wbwtab A=32 graph (wbwtab.freeze_inference on ``prepare(A=32, W=2|3)``, DESIGN.md 4.20),
composed block by block from the engine's kernels: the frozen logits must equal it bit for bit.  Used by
tests/test_gpu_wbwtab_frozen_a32.py and harness/wbwtab_a32_infer_probe.py."""
import torch


def blocks(m):
    return list(m.model.children())


def parts(blk):
    return [k for k in blk.children() if not isinstance(k, torch.nn.Identity)]


def composed(m, x):
    """the block-by-block composition of the kernels on an un-frozen model: stem conv (as the model runs it) -> stem producer
    -> for every quantized layer pk conv (fp32, terms (3, 1), the frozen (w_int, alpha, bias)) -> stem producer (BatchNorm +
    ReLU + next block's shuffle -> term planes) [-> term-plane pool]; the last quantized layer's output and the head run as
    the un-frozen model runs them.  Returns (logits, the decoded plane each quantized layer reads)."""
    from micronet_b200 import _lib as L, pk as PK, wbwtab
    from micronet_b200 import functional as F_
    T = wbwtab.A32_TERMS
    kids = blocks(m)
    qidx = [i for i, b in enumerate(kids) if hasattr(b, "conv") and type(b.conv) is wbwtab.QuantConv2d]
    first, last = qidx[0], qidx[-1]
    stem = kids[0]
    h = stem.conv(x)
    reads = []

    def producer(y, bn, nxt):
        sg = int(nxt.shuffle_groups) if getattr(nxt, "channel_shuffle_flag", 0) else 1
        stats = (bn.running_mean, torch.rsqrt(bn.running_var + bn.eps), bn.weight.detach(), bn.bias.detach())
        plane = PK.terms_plane(*y.shape, T, y.device)
        L.check(PK.bn_relu_pack_terms(y.contiguous(), stats, True, sg, T, plane), "bn_relu_pack_terms")
        return plane

    plane, shape = producer(h, parts(stem)[1], kids[first]), h.shape
    i = first
    while i <= last:
        blk = kids[i]
        if isinstance(blk, torch.nn.MaxPool2d):
            k, s, p = blk.kernel_size, blk.stride, blk.padding
            rc, plane = PK.plane_maxpool_terms(plane, *shape, k, s, p, T)
            L.check(rc, "pool")
            shape = (shape[0], shape[1], (shape[2] + 2 * p - k) // s + 1, (shape[3] + 2 * p - k) // s + 1)
            i += 1
            continue
        c, bn = parts(blk)[0], parts(blk)[1]
        reads.append(PK.unpack_terms(plane, shape, T))
        w_int, alpha = wbwtab.frozen_levels(c)
        sh = F_._shape_struct(shape, c.weight.shape, c.stride, c.padding, c.dilation, c.groups)
        y = torch.empty((shape[0], c.out_channels) + F_._out_hw(sh), device=x.device)
        L.check(PK.conv(sh, 0, plane, T, PK.pack_weight(sh, 0, T, 1, w_int=w_int), 1, y, n_scale=alpha, bias=c.bias), "pk")
        if i == last:
            h = parts(blk)[2](bn(y))
            break
        j = i + 1 + isinstance(kids[i + 1], torch.nn.MaxPool2d)
        plane, shape = producer(y, bn, kids[j]), y.shape
        i += 1
    for blk in kids[last + 1:]:
        h = blk(h)
    return h.view(h.shape[0], -1), reads
