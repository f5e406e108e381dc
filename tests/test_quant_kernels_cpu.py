"""Host-side refusals of the quantizer, observer and statistics entry points (mnb_quant.cu), no GPU needed.

Every call below passes argument checks up to the one under test and fails exactly there: the entry point must return
MNB_E_ARG with a message naming the problem, before launching anything.  The pointers are fakes that are never
dereferenced (a launch would fault on them), and no CUDA call is made, so the test runs without a device."""
import ctypes as C

import pytest

FAKE = 4096
E_ARG = -1


def _lib():
    from micronet_b200 import _lib as L
    return L.load()


def _refused(rc, lib, *words):
    assert rc == E_ARG, rc
    msg = lib.mnb_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("entry", ["channel_stats", "bn_batch_stats"])
def test_statistics_refuse_more_than_8192_channels(entry):
    """the completion counters of the split finaliser are a fixed 8192-entry array in the scratch buffer"""
    lib = _lib()
    for c in (8193, 16384):     # (8192 itself launches; test_gpu_quant_kernels.py runs it)
        if entry == "channel_stats":
            rc = lib.mnb_channel_stats(FAKE, 2, c, 4, 1, FAKE, FAKE, None)
        else:
            rc = lib.mnb_bn_batch_stats(FAKE, 2, c, 4, 1e-5, 0.1, FAKE, FAKE, FAKE, FAKE, FAKE, None)
        _refused(rc, lib, "8192", str(c))


def test_channel_stats_refuses_an_unknown_output_kind():
    lib = _lib()
    _refused(lib.mnb_channel_stats(FAKE, 2, 8, 4, 3, FAKE, FAKE, None), lib, "as_mean_var")


def test_bn_batch_stats_refuses_a_single_value_per_channel():
    """the unbiased variance of the running estimate divides by N - 1"""
    lib = _lib()
    _refused(lib.mnb_bn_batch_stats(FAKE, 1, 8, 1, 1e-5, 0.1, FAKE, FAKE, FAKE, FAKE, FAKE, None), lib, "more than one")


@pytest.mark.parametrize("n,rows", [(10, 3), (4608 * 512 + 1, 512), (7, 2)])
def test_observer_refuses_n_not_a_multiple_of_rows(n, rows):
    lib = _lib()
    for kind in (0, 1):
        rc = lib.mnb_iao_observe(FAKE, n, rows, kind, 1, 0.1, 0.0, FAKE, FAKE, 1, 1, -127, 127, FAKE, FAKE, FAKE, None)
        _refused(rc, lib, "observer")


@pytest.mark.parametrize("n,percentile", [(1000, 0.0009), (1000, 0.0), (1000, 1.5), (1, 0.5)])
def test_percentile_observer_refuses_k_outside_1_to_n(n, percentile):
    """k = int(percentile * n), as the reference's kthvalue call computes it; k = 0 or k > n has no k-th value"""
    lib = _lib()
    rc = lib.mnb_iao_observe(FAKE, n, 1, 2, 1, 0.1, percentile, FAKE, FAKE, 1, 1, -128, 127, FAKE, FAKE, FAKE, None)
    _refused(rc, lib, "kthvalue", f"n={n}")


def test_percentile_observer_refuses_per_channel_rows():
    lib = _lib()
    rc = lib.mnb_iao_observe(FAKE, 64, 4, 2, 1, 0.1, 0.5, FAKE, FAKE, 1, 1, -128, 127, FAKE, FAKE, FAKE, None)
    _refused(rc, lib, "per-layer")


def test_observer_refuses_an_unknown_kind_and_missing_qparams():
    lib = _lib()
    _refused(lib.mnb_iao_observe(FAKE, 64, 1, 3, 1, 0.1, 0.0, FAKE, FAKE, 0, 1, 0, 1, None, None, FAKE, None), lib, "kind 3")
    _refused(lib.mnb_iao_observe(FAKE, 64, 1, 0, 1, 0.1, 0.0, FAKE, FAKE, 1, 1, 0, 255, None, None, FAKE, None), lib, "qparams")
    _refused(lib.mnb_iao_update_qparams(FAKE, FAKE, 4, 1, 5, 5, FAKE, FAKE, None), lib, "qparams")


@pytest.mark.parametrize("w_bits", [1, 9, 0, 16, 32])
def test_dorefa_weight_refuses_bits_outside_2_to_8(w_bits):
    lib = _lib()
    _refused(lib.mnb_dorefa_weight_fwd(FAKE, 300, 3, w_bits, FAKE, FAKE, FAKE, FAKE, FAKE, None), lib, "w_bits", str(w_bits))
    _refused(lib.mnb_dorefa_weight_bwd(FAKE, FAKE, 300, w_bits, FAKE, FAKE, None), lib, "w_bits", str(w_bits))


@pytest.mark.parametrize("W", [0, 1, 4, 32])
def test_wbwtab_weight_refuses_W_other_than_2_or_3(W):
    lib = _lib()
    _refused(lib.mnb_wb_weight_fwd(FAKE, 4, 3, 9, W, FAKE, FAKE, FAKE, FAKE, None), lib, f"got {W}")
    _refused(lib.mnb_wb_weight_bwd(FAKE, FAKE, FAKE, 4, 3, 9, W, FAKE, None), lib, f"got {W}")


@pytest.mark.parametrize("rows", [0, 2, 7, 9])
def test_iao_weight_refuses_rows_other_than_1_or_out_c(rows):
    """rows picks the scale of element i: scale[0] (per layer) or scale[i / inner] (per output channel); any other count
    would read scales that do not exist, in the forward and in the backward"""
    lib = _lib()
    out_c, numel = 8, 8 * 27
    rc = lib.mnb_iao_weight_fwd(FAKE, numel, out_c, rows, FAKE, FAKE, FAKE, FAKE, 0, -127, 127, FAKE, FAKE, FAKE, FAKE, None)
    _refused(rc, lib, "rows")
    _refused(lib.mnb_iao_weight_bwd(FAKE, FAKE, FAKE, numel, out_c, rows, FAKE, None), lib, "rows")


def test_activation_quantizer_refuses_bad_qparams():
    from micronet_b200 import _lib as L
    lib = _lib()
    for qp, word in ((L.ActQParams(L.ACT_DOREFA, 9, 0, 0, 0, None, None, None, None), "a_bits"),
                     (L.ActQParams(L.ACT_IAO, 8, 0, 256, 0, FAKE, FAKE, FAKE, FAKE), "u8"),
                     (L.ActQParams(L.ACT_IAO, 8, 0, 255, 0, None, FAKE, FAKE, FAKE), "NULL"),
                     (L.ActQParams(7, 8, 0, 255, 0, None, None, None, None), "mode 7")):
        _refused(lib.mnb_act_quant_fwd(FAKE, 100, C.byref(qp), None, FAKE, FAKE, None), lib, word)
        _refused(lib.mnb_act_quant_bwd(FAKE, FAKE, 100, C.byref(qp), FAKE, None), lib, word)
    sign = L.ActQParams(L.ACT_SIGN, 1, 0, 0, 0, None, None, None, None)
    _refused(lib.mnb_quant_add_fwd(FAKE, FAKE, 100, C.byref(sign), FAKE, FAKE, FAKE, 0, None), lib, "QuantAdd")
