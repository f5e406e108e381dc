"""Scheme-independent parts of the frozen inference graphs on level planes (dorefa.freeze_inference, iao.freeze_inference):
finding the reference's conv-bn-relu blocks (nin.py / nin_gc.py ``ConvBNReLU``) and the max-pool between two of them in an
``nn.Sequential``, the producer -> consumer link, the instance-level ``forward`` overrides that pass a producer's tagged
plane through the absorbed modules, moving a block's channel shuffle into its producer, and the undo record that
``enable=False`` replays.  Each scheme decides which blocks it links and what its pool kernel is."""
from __future__ import annotations

import functools

import torch.nn as nn

from . import _lib as L
from . import functional as F_


def shuffle(x, groups):
    b, c = x.shape[0], x.shape[1]
    return x.view(b, groups, c // groups, *x.shape[2:]).transpose(1, 2).contiguous().view(x.shape)


def block_parts(blk):
    """(conv, the modules behind it with nn.Identity left out) of one of the reference's conv-bn-relu blocks, else None"""
    if not hasattr(blk, "channel_shuffle_flag"):
        return None
    parts = [k for k in blk.children() if not isinstance(k, nn.Identity)]
    if not parts or not isinstance(parts[0], nn.Conv2d):
        return None
    return parts[0], parts[1:]


def block_pairs(model, parse, pool_cfg):
    """(parse(block), pool, (k, s, p) or None, next block, its first conv) for every block of an nn.Sequential that
    ``parse`` accepts and that is followed - directly or across one max-pool that ``pool_cfg`` covers - by another
    conv-bn-relu block.  A pool that ``pool_cfg`` refuses ends the pair."""
    for seq in [m for m in model.modules() if isinstance(m, nn.Sequential)]:
        kids = [k for k in seq.children() if not isinstance(k, nn.Identity)]
        for i, blk in enumerate(kids):
            parsed = parse(blk)
            if parsed is None:
                continue
            j, pool, cfg = i + 1, None, None
            if j < len(kids):
                cfg = pool_cfg(kids[j])
                if cfg is not None:
                    pool, j = kids[j], j + 1
            if j >= len(kids) or not hasattr(kids[j], "channel_shuffle_flag"):
                continue
            nxt = kids[j]
            nparts = [k for k in nxt.children() if not isinstance(k, nn.Identity)]
            yield parsed, pool, cfg, nxt, (nparts[0] if nparts else None)


def block_shuffle(nxt):
    """shuffle groups of the channel shuffle a block applies to its input (1: none)"""
    return int(nxt.shuffle_groups) if nxt.channel_shuffle_flag and int(getattr(nxt, "shuffle_groups", 1)) > 1 else 1


class Link:
    """a producer -> consumer hand-off of a frozen graph: the consumer conv, the eval BatchNorm and ReLU the producer applies,
    the consumer block's channel shuffle and the max-pool (module, k, s, p) in between, which runs on the level plane"""

    def __init__(self, cconv, bn, relu, sg, pool):
        self.cconv, self.bn, self.relu, self.sg, self.pool = cconv, bn, relu, sg, pool
        self.target = pool[0] if pool is not None else cconv


class Rewrite:
    """the instance-level changes of one freeze, recorded on the model under ``key`` so that ``undo`` restores them"""

    def __init__(self, model, key):
        self.key = key
        self.log = model.__dict__.setdefault(key, [])

    def set_dict(self, m, name, value):
        m.__dict__[name] = value
        self.log.append(("dict", m, name))

    def forget(self, m, *names):
        self.log += [("dict", m, n) for n in names]

    def override(self, m, fn, *args):
        self.set_dict(m, "forward", functools.partial(fn, *args))

    def move_shuffle(self, nxt, cconv, sg):
        """the producer applies block ``nxt``'s input shuffle; ``cconv`` applies it itself when no plane comes"""
        self.log.append(("attr", nxt, "channel_shuffle_flag", nxt.channel_shuffle_flag))
        nxt.channel_shuffle_flag = 0
        self.set_dict(cconv, "_mnb_in_shuffle", sg)


def undo(model, key):
    for rec in reversed(model.__dict__.pop(key, [])):
        if rec[0] == "attr":
            setattr(rec[1], rec[2], rec[3])
        else:
            rec[1].__dict__.pop(rec[2], None)


def absorbed_forward(check, m, target, x):
    """BatchNorm / ReLU whose work a producer did for ``target``: pass its tagged output through, run as usual otherwise"""
    pre = getattr(x, "_mnb_pk_pre", None)
    if pre is not None and pre[0] is target:
        check(m)
        return x
    return type(m).forward(m, x)


def pool_forward(check, run, pool, link, x):
    """the max-pool between a producer and its consumer, on the producer's level plane: ``run(plane, b, c, h, w, k, s, p,
    int8)`` returns the consumer's plane at the pooled size; the module runs as usual on anything but that plane"""
    import torch
    plane = F_.handed_plane(pool, x)
    if plane is None:
        return type(pool).forward(pool, x)
    check(pool)
    _, k, s, p = link.pool
    b, c, h, w = x.shape
    fmt = x._mnb_pk_pre[3]
    out = F_._timed("plane_pool", L.ConvShape(b, c, h, w, c, k, k, s, s, p, p, 1, 1, 1),
                    lambda: run(plane, b, c, h, w, k, s, p, fmt == "i8"))
    y = torch.empty((b, c, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1), dtype=torch.float32, device="meta")
    y._mnb_pk_pre = (link.cconv, out, y._version, fmt)
    return y
