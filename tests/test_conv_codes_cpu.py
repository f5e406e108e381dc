"""Where the int16 hand-off of a wbwtab conv to its BatchNorm applies (fused._mark_codes_out), and the host-side bound of
mnb_pk_conv_codes; no GPU needed (the refused calls return before any plan or launch, their pointers are never read)."""
import ctypes as C

import pytest

FAKE = 4096


def _bench_model():
    from harness import train as H
    w = H.WORKLOADS["nin_gc_wbwtab_w3a2"]
    return H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"], **w.get("engine_extra", {}))


def test_rewrite_marks_exactly_the_seven_wbwtab_convs():
    from micronet_b200 import wbwtab
    from micronet_b200.fused import BatchNormBinarize2d
    model = _bench_model()
    blocks = list(model.model.children())
    marked = [i for i, blk in enumerate(blocks) if getattr(getattr(blk, "conv", None), "codes_out", False)]
    assert marked == [1, 2, 4, 5, 6, 8, 9], marked          # L1, L2, (pool), L3, L4, L5, (pool), L6, L7
    for i in marked:
        assert isinstance(blocks[i].conv, wbwtab.QuantConv2d) and isinstance(blocks[i].bn, BatchNormBinarize2d)
    assert sum(isinstance(m, wbwtab.QuantConv2d) and m.codes_out for m in model.modules()) == 7


def test_inference_and_unfused_convs_are_not_marked():
    from harness import train as H
    from micronet_b200 import wbwtab
    inf = H.prepare_engine(H.build_float_model("nin_gc"), "wbwtab", W=3, A=2, fuse_bn=True, quant_inference=True)
    assert not any(getattr(m, "codes_out", False) for m in inf.modules())
    plain = H.prepare_engine(H.build_float_model("nin_gc"), "wbwtab", W=3, A=2)
    assert not any(isinstance(m, wbwtab.QuantConv2d) and m.codes_out for m in plain.modules())


def test_int16_bound_matches_the_shapes():
    from micronet_b200 import pk as PK, wbwtab
    terms = sorted({(m.in_channels // m.groups) * m.kernel_size[0] * m.kernel_size[1]
                    for m in _bench_model().modules() if isinstance(m, wbwtab.QuantConv2d)})
    assert terms == [128, 144]                               # 1x1 layers and the two grouped 3x3 layers
    assert PK.codes_fit(32767, 1, 1) and not PK.codes_fit(32768, 1, 1)
    assert PK.codes_fit(3640, 1, 3) and not PK.codes_fit(3641, 1, 3)
    assert PK.codes_fit(16383, 1, 1, level_bound=2) and not PK.codes_fit(16384, 1, 1, level_bound=2)


@pytest.mark.parametrize("cin,groups,r,level", [(32768, 1, 1, 1), (3641, 1, 3, 1), (16384, 1, 1, 2), (65536, 2, 1, 1)])
def test_host_refuses_sums_over_int16(cin, groups, r, level):
    from micronet_b200 import _lib as L
    lib = L.load()
    sh = L.ConvShape(1, cin, 4, 4, 8 * groups, r, r, 1, 1, r // 2, r // 2, 1, 1, groups)
    rc = lib.mnb_pk_conv_codes(C.byref(sh), FAKE, 1, FAKE, 1, None, None, 1.0, None, level, FAKE, FAKE, FAKE, None)
    assert rc == L.E_UNSUPPORTED, rc
    assert "int16" in lib.mnb_last_error().decode()
