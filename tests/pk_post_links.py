"""The producer -> consumer links of the frozen inference graphs, taken from freeze_inference's host-side link planning on CPU
models: for every linked conv, its forward shape at the batch the benchmark runs the graph, the consumer-plane epilogue it
launches (tests/pk_post_cases.py paths) and the consumer options (shuffle groups, eval BatchNorm, phase split, ReLU).

frozen_conv (functional.py) and wbwtab._a32_conv_forward decide per call whether a link hands over a plane and in which
format; the rules below are those decisions, evaluated with the host-only plan queries.  Links that hand over nothing run
the plain conv and do not appear."""
import torch
import torch.nn as nn

from tests import pk_post_cases as P


def _conv_inputs(base, batch, hw):
    """{module name: input shape} of every nn.Conv2d of a float model (a meta-device forward: no data)"""
    out = {}
    hooks = [m.register_forward_pre_hook(lambda mod, inp, n=n: out.__setitem__(n, tuple(inp[0].shape)))
             for n, m in base.named_modules() if isinstance(m, nn.Conv2d)]
    base.to("meta").eval()(torch.empty(batch, 3, hw, hw, device="meta"))
    for h in hooks:
        h.remove()
    return out


def _shape(inp, conv):
    B, Cc, H, W = inp
    assert conv.kernel_size[0] == conv.kernel_size[1] and conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1]
    return (B, Cc, H, W, conv.out_channels, conv.kernel_size[0], conv.stride[0], conv.padding[0], conv.groups)


def _read_shape(shape, cconv, pool):
    B, Cc, H, W, K, R, st, pad, G = shape
    oh, ow = P.out_hw(shape)
    if pool is not None:
        _, k, s, p = pool
        oh, ow = (oh + 2 * p - k) // s + 1, (ow + 2 * p - k) // s + 1
    return (B, K, oh, ow, cconv.out_channels, cconv.kernel_size[0], cconv.stride[0], cconv.padding[0], cconv.groups)


def _route(shape, cconv, pool, sg, bn, relu, q, int8, formats=None):
    """(path, options) of the epilogue a producer of ``shape`` launches for this consumer, or None (no hand-off).  int8: the
    graph was frozen with int8=True and the consumer's quantizer fits s8 (functional._i8_route, Consumer.format)."""
    from micronet_b200 import pk as PK
    B, Cc, H, W, K, R, st, pad, G = shape
    split = cconv.stride[0] == 2 and pool is None
    read = _read_shape(shape, cconv, pool)
    if sg > 1 and (K % 16 or K % sg or split):
        return None
    out_shape_ok = read[1] == cconv.in_channels
    csh = P.conv_shape(read)
    fmt = None
    if int8 and out_shape_ok and PK.i8_supported(csh):
        fmt = "i8"
    elif out_shape_ok and not PK.padded(read[1], cconv.groups) and not (cconv.stride[0] == 2 and (read[2] | read[3]) & 1) \
            and PK.supported(csh, 0, 1, 1):
        fmt = "bf16"
    if formats is not None and fmt not in formats:
        return None
    psh = P.conv_shape(shape)
    if fmt == "i8":
        if not PK.i8_supported(psh) or not (G == 1 or (K // G) % 16 == 0):
            return None
        path = "xpost_i8" if bn or sg > 1 else "levels_i8"
    elif fmt == "bf16":
        if PK.segmented(psh, 0, 1, 1) or PK.padded(K, G) or not PK.supported(psh, 0, 1, 1):
            return None
        path = "xpost" if bn or sg > 1 else "levels"
    else:
        return None
    return path, dict(q=q, sg=sg, bn=bool(bn), split=split, relu=bool(relu), terms=0, ta=1)


def _iao(base_fn, name, batch, hw, int8):
    from micronet_b200 import iao
    shapes = _conv_inputs(base_fn(), batch, hw)
    torch.manual_seed(0)
    m = iao.prepare(base_fn(), a_bits=8, w_bits=8, q_type=0, q_level=0, bn_fuse=True, ptq=True).eval()
    iao.freeze_inference(m, int8=int8)
    out = {}
    for n, c in m.named_modules():
        link = c.__dict__.get("_post_consumer")
        if link is None or not isinstance(c, nn.Conv2d):
            continue                     # (QuantAdd producers: tests/test_gpu_pk_post.py checks them separately)
        if isinstance(link, iao._BlockLink):
            cconv, sg, pool, relu, formats = link.cconv, link.sg, link.pool, True, (None if link.sg == 1 else ("i8",))
        else:
            cconv, sg, pool, relu, formats = link[0], 1, None, link[0].__dict__.get("_pre_relu", False), None
        shape = _shape(shapes[n], c)
        r = _route(shape, cconv, pool, sg, False, relu, "iao8", int8, formats)
        if r is not None:
            out[(name, n)] = (shape,) + r
    return out


def _dorefa(base_fn, name, batch, a, w):
    from micronet_b200 import dorefa as DF
    shapes = _conv_inputs(base_fn(), batch, 32)
    torch.manual_seed(0)
    m = DF.prepare(base_fn(), a_bits=a, w_bits=w).eval()
    DF.freeze_inference(m)
    out = {}
    for n, c in m.named_modules():
        info = c.__dict__.get("_mnb_frozen")
        link = None if info is None else info.get("link")
        if link is None or not isinstance(c, nn.Conv2d):
            continue
        shape = _shape(shapes[n], c)
        r = _route(shape, link.cconv, link.pool, link.sg, link.bn is not None, link.relu, f"dorefa{a}", False)
        if r is not None:
            out[(name, n)] = (shape,) + r
    return out


def _a32(base_fn, name, batch):
    from micronet_b200 import pk as PK, wbwtab
    shapes = _conv_inputs(base_fn(), batch, 32)
    m = wbwtab.prepare(base_fn(), W=3, A=32).eval()
    wbwtab.freeze_inference(m)
    out = {}
    for n, c in m.named_modules():
        rec = c.__dict__.get("_mnb_frozen")
        link = None if rec is None or rec["fmt"] != wbwtab.A32_PLANE else rec["link"]
        if link is None:
            continue
        shape = _shape(shapes[n], c)
        psh = P.conv_shape(shape)
        # wbwtab._a32_conv_forward: the epilogue writes the term planes of an unshuffled link on a non-segmented plan
        if not link.accepts((shape[0], shape[4]) + P.out_hw(shape)) or PK.padded(shape[4], shape[8]) or \
                not wbwtab._epilogue_hand_off(link, psh):
            continue
        out[(name, n)] = (shape, "terms", dict(q=None, sg=link.sg, bn=True, split=link.split, relu=True, terms=3,
                                                ta=wbwtab.A32_TERMS))
    return out


def linked_convs():
    """{(graph, conv name): (shape, path, options)} of every conv whose epilogue writes its consumer's plane"""
    from harness import models as zoo, train as H
    nin = lambda: H.build_float_model("nin", seed=1)
    gc = lambda: H.build_float_model("nin_gc", seed=1)
    out = {}
    out.update(_iao(zoo.resnet18, "resnet18_iao_ptq_224", 64, 224, False))
    out.update(_iao(zoo.resnet18, "resnet18_iao_ptq_224_int8", 64, 224, True))
    out.update(_iao(nin, "nin_iao", 256, 32, False))
    out.update(_iao(nin, "nin_iao_int8", 256, 32, True))
    out.update(_iao(gc, "nin_gc_iao", 256, 32, False))
    out.update(_iao(gc, "nin_gc_iao_int8", 256, 32, True))
    out.update(_dorefa(nin, "nin_dorefa_w8a8", 256, 8, 8))
    out.update(_dorefa(gc, "nin_gc_dorefa_w4a4", 256, 4, 4))
    out.update(_a32(nin, "nin_wbwtab_a32", 256))
    out.update(_a32(gc, "nin_gc_wbwtab_a32", 256))
    return out


def case_options(c):
    return dict(q=c.q, sg=c.sg, bn=bool(c.bn), split=bool(c.split), relu=bool(c.relu), terms=c.terms, ta=c.ta)
