"""Scheme-independent parts of the frozen inference graphs of all three schemes (dorefa.freeze_inference,
iao.freeze_inference, wbwtab.freeze_inference): finding the reference's conv-bn-act blocks (nin.py / nin_gc.py
``ConvBNReLU``) and the max-pool between two of them in an ``nn.Sequential``, the producer -> consumer link, the
instance-level ``forward`` overrides that pass a producer's plane (tagged by functional.tag, read by
functional.handed_plane, decoded by functional.materialized) through the absorbed modules and run a max-pool on it, moving
a block's channel shuffle into its producer, the versioned operand cache, the eval check, and the undo record that
``enable=False`` replays.  Each scheme decides which blocks it links, what its kernels are and what it does where they
refuse a shape."""
from __future__ import annotations

import functools

import torch
import torch.nn as nn

from . import _lib as L
from . import functional as F_

def shuffle(x, groups):
    b, c = x.shape[0], x.shape[1]
    return x.view(b, groups, c // groups, *x.shape[2:]).transpose(1, 2).contiguous().view(x.shape)


def block_parts(blk):
    """(conv, the modules behind it with nn.Identity left out) of one of the reference's conv-bn-act blocks - nin_gc.py's
    (with ``channel_shuffle_flag``) or nin.py's (without) - else None"""
    parts = [k for k in blk.children() if not isinstance(k, nn.Identity)]
    if not parts or not isinstance(parts[0], nn.Conv2d):
        return None
    return parts[0], parts[1:]


def blocks(model, parse):
    """parse(block) of every child of an nn.Sequential that ``parse`` accepts"""
    for seq in [m for m in model.modules() if isinstance(m, nn.Sequential)]:
        for k in seq.children():
            parsed = None if isinstance(k, nn.Identity) else parse(k)
            if parsed is not None:
                yield parsed


def block_pairs(model, parse, pool_cfg):
    """(parse(block), pool, (k, s, p) or None, next block, its first conv, (the nn.Sequential, the pool's name) or None) for
    every block of an nn.Sequential that ``parse`` accepts and that is followed - directly or across one max-pool that
    ``pool_cfg`` covers - by another conv-bn-act block.  A pool that ``pool_cfg`` refuses ends the pair."""
    for seq in [m for m in model.modules() if isinstance(m, nn.Sequential)]:
        kids = [(n, k) for n, k in seq.named_children() if not isinstance(k, nn.Identity)]
        for i, (_, blk) in enumerate(kids):
            parsed = parse(blk)
            if parsed is None:
                continue
            j, pool, cfg, slot = i + 1, None, None, None
            if j < len(kids):
                cfg = pool_cfg(kids[j][1])
                if cfg is not None:
                    pool, slot, j = kids[j][1], (seq, kids[j][0]), j + 1
            nparts = block_parts(kids[j][1]) if j < len(kids) else None
            if nparts is not None:
                yield parsed, pool, cfg, kids[j][1], nparts[0], slot


def max_pool_cfg(m):
    """(k, s, p) of an nn.MaxPool2d / fused.EngineMaxPool2d the engine's pool kernels cover, else None"""
    from .fused import EngineMaxPool2d, _pool_cfg
    return _pool_cfg(m) if type(m) in (nn.MaxPool2d, EngineMaxPool2d) else None


def block_shuffle(nxt):
    """shuffle groups of the channel shuffle a block applies to its input (1: none)"""
    sg = int(getattr(nxt, "shuffle_groups", 1))
    return sg if getattr(nxt, "channel_shuffle_flag", 0) and sg > 1 else 1


def check_eval(scheme, m):
    if m.training:
        raise RuntimeError(f"micronet_b200: this module is frozen for inference ({scheme}.freeze_inference); call "
                           "freeze_inference(model, enable=False) before training it")


def cached_operands(m, name, make):
    """make() of a frozen module, kept in ``m.__dict__[name]`` as (key, *operands) and re-done when a parameter or buffer
    of ``m`` is written in place.  The key is taken after make: wbwtab's W = 2 quantizer centres its parameter in place."""
    def key():
        return tuple(t._version for t in list(m.parameters()) + list(m.buffers()))
    fr = m.__dict__.get(name)
    if fr is None or fr[0] != key():
        ops = tuple(make())
        fr = m.__dict__[name] = (key(),) + ops
    return fr[1:]


class Link:
    """a producer -> consumer hand-off of a frozen graph: the consumer conv, the eval BatchNorm and ReLU the producer applies,
    the consumer block's channel shuffle and the max-pool (module, k, s, p) in between, which runs on the plane"""

    def __init__(self, cconv, bn, relu, sg, pool):
        self.cconv, self.bn, self.relu, self.sg, self.pool = cconv, bn, relu, int(sg), pool
        self.target = pool[0] if pool is not None else cconv
        self._invstd = None

    def bn_tensors(self):
        """(mean, invstd, gamma, beta) of the eval BatchNorm (running statistics); invstd as the un-frozen eval BatchNorm
        computes it, re-computed when running_var changes"""
        bn = self.bn
        rv = bn.running_var
        key = (rv.data_ptr(), rv._version, float(bn.eps))
        if self._invstd is None or self._invstd[0] != key:
            self._invstd = (key, torch.rsqrt(rv + bn.eps))
        return bn.running_mean, self._invstd[1], bn.weight.detach(), bn.bias.detach()


class Rewrite:
    """the instance-level changes of one freeze, recorded on the model under ``key`` so that ``undo`` restores them"""

    def __init__(self, model, key):
        self.log = model.__dict__.setdefault(key, [])

    def set_dict(self, m, name, value):
        m.__dict__[name] = value
        self.log.append(("dict", m, name))

    def forget(self, m, *names):
        """entries a frozen module adds to its own ``__dict__`` later (operand caches)"""
        self.log += [("dict", m, n) for n in names]

    def set_attr(self, m, name, value):
        self.log.append(("attr", m, name, getattr(m, name)))
        setattr(m, name, value)

    def set_child(self, parent, name, new):
        self.log.append(("child", parent, name, parent._modules[name]))
        parent._modules[name] = new

    def override(self, m, fn, *args, **kw):
        self.set_dict(m, "forward", functools.partial(fn, *args, **kw))

    def move_shuffle(self, nxt, cconv, sg):
        """the producer applies block ``nxt``'s input shuffle; ``cconv`` applies it itself when no plane comes"""
        self.set_attr(nxt, "channel_shuffle_flag", 0)
        self.set_dict(cconv, "_mnb_in_shuffle", sg)


def undo(model, key):
    for rec in reversed(model.__dict__.pop(key, [])):
        if rec[0] == "attr":
            setattr(rec[1], rec[2], rec[3])
        elif rec[0] == "child":
            rec[1]._modules[rec[2]] = rec[3]
        else:
            rec[1].__dict__.pop(rec[2], None)


def absorbed_forward(check, m, target, x):
    """BatchNorm / ReLU / binarizer whose work a producer did for ``target``: pass its tagged output through, run as usual
    otherwise.  ``target`` None: the producer runs the module itself on every path, so everything passes through."""
    pre = getattr(x, "_mnb_pk_pre", None)
    if target is None or (pre is not None and pre[0] is target):
        check(m)
        return x
    return type(m).forward(m, x)


def pool_forward(check, run, fallback, pool, link, x, timed=True):
    """the max-pool between a producer and its consumer, on the producer's plane: ``run(plane, x, k, s, p)`` returns the
    consumer's plane at the pooled size, or None where its kernel refuses the shape; ``fallback(pool, link, x, plane)``
    runs the pool on anything else (``plane``: the refused plane, or None)"""
    plane = F_.handed_plane(pool, x)
    if plane is not None:
        check(pool)
        _, k, s, p = link.pool
        b, c, h, w = x.shape
        if timed:
            out = F_._timed("plane_pool", L.ConvShape(b, c, h, w, c, k, k, s, s, p, p, 1, 1, 1),
                            lambda: run(plane, x, k, s, p))
        else:
            out = run(plane, x, k, s, p)
        if out is not None:
            y = torch.empty((b, c, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1), dtype=torch.float32, device="meta")
            _, _, _, fmt, info = x._mnb_pk_pre
            return F_.tag(y, link.cconv, out, fmt, **info)
    return fallback(pool, link, x, plane)


def pool_as_usual(pool, link, x, plane):
    return type(pool).forward(pool, F_.materialized(x))
