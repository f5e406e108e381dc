"""Host-side refusals of the fused BatchNorm producers (mnb_fused.cu, mnb_conv_packed.cu, mnb_pk.cu) and the launch-path
restatements tests/test_gpu_bn_producers.py asserts its cases with, no GPU needed.

Every refused call fails before anything is launched: MNB_E_UNSUPPORTED (-2) for a plane outside a kernel's cover (the
caller then takes another path), MNB_E_ARG (-1) for arguments no path accepts.  The pointers are fakes that are never
dereferenced (a launch would fault on them), and no CUDA call is made."""
import ctypes as C

import pytest

from tests.test_gpu_bn_producers import (BENCH_PLANES, apply_chain, bench_planes, bwd_path, fwd_path, pack_vec,
                                         plane_splits, reduce_chain)

FAKE = 4096          # 16-byte aligned
E_ARG, E_UNSUPPORTED = -1, -2


def _lib():
    from micronet_b200 import _lib as L
    return L, L.load()


def _rc(rc, want, lib, *words):
    assert rc == want, (rc, lib.mnb_last_error().decode())
    msg = lib.mnb_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def _fwd_packed(lib, B=2, Cc=16, hw=64, sg=1, x=FAKE, y=FAKE, plane=FAKE):
    return lib.mnb_bn_sign_fwd_packed(x, B, Cc, hw, FAKE, FAKE, FAKE, FAKE, sg, y, FAKE, plane, None)


def _relu_quant(lib, qp, B=2, Cc=16, hw=64, sg=1, plane=FAKE):
    return lib.mnb_bn_relu_quant_pack_fwd(FAKE, B, Cc, hw, FAKE, FAKE, FAKE, FAKE, C.byref(qp), sg, plane, FAKE, None)


def _bwd_pack(lib, B=2, Cc=16, hw=64, sg=1, terms=3, plane=FAKE):
    return lib.mnb_bn_sign_bwd_pack(FAKE, FAKE, FAKE, B, Cc, hw, FAKE, FAKE, FAKE, FAKE, FAKE, sg, FAKE, terms, FAKE, plane,
                                    None)


def _pool_fwd(lib, B=2, Cc=16, H=8, W=16, sg=1, x=FAKE, y=FAKE):
    return lib.mnb_bn_sign_pool_fwd(x, B, Cc, H, W, FAKE, FAKE, FAKE, FAKE, sg, y, FAKE, FAKE, None)


def _pool_bwd(lib, B=2, Cc=16, H=8, W=16, sg=1, g=FAKE, x=FAKE, dx=FAKE):
    return lib.mnb_bn_sign_pool_bwd(g, FAKE, FAKE, x, B, Cc, H, W, FAKE, FAKE, FAKE, 1, sg, dx, FAKE, FAKE, None, FAKE, None)


def _pool_bwd_pack(lib, B=2, Cc=16, H=8, W=16, sg=1, terms=3, g=FAKE, x=FAKE, plane=FAKE):
    return lib.mnb_bn_sign_pool_bwd_pack(g, FAKE, FAKE, x, B, Cc, H, W, FAKE, FAKE, FAKE, FAKE, FAKE, sg, FAKE, terms, plane,
                                         None)


@pytest.mark.parametrize("what", ["C%8", "hw%32", "plane+8"])
def test_packed_producers_refuse_planes_outside_their_cover(what):
    """the plane layout [B][C/8][H][W][8] needs C % 8 == 0; a warp owns 32 consecutive positions (hw % 32 == 0); the plane
    is written with 16-byte stores"""
    from micronet_b200 import functional as F_
    L, lib = _lib()
    kw = {"C%8": dict(Cc=20), "hw%32": dict(hw=48), "plane+8": dict(plane=FAKE + 8)}[what]
    qp = F_.ActSpec(L.ACT_DOREFA, bits=4).struct()
    _rc(_fwd_packed(lib, **kw), E_UNSUPPORTED, lib)
    _rc(_relu_quant(lib, qp, **kw), E_UNSUPPORTED, lib)
    _rc(_bwd_pack(lib, **kw), E_UNSUPPORTED, lib)


@pytest.mark.parametrize("what", ["odd H", "W%8", "x+4", "y+8", "2^31 elements"])
def test_pooled_producers_refuse_planes_outside_their_cover(what):
    """one lane owns two float4 of x in rows 2 oh and 2 oh + 1: even H, W % 8 == 0, 16-byte aligned x / y / dx / plane,
    and 32-bit element indices (< 2^31 elements)"""
    L, lib = _lib()
    big = dict(B=4096, Cc=64, H=128, W=128)                              # 2^32 elements
    shape = {"odd H": dict(H=7), "W%8": dict(W=12), "2^31 elements": big}.get(what, {})
    fwd_ptr = {"x+4": dict(x=FAKE + 4), "y+8": dict(y=FAKE + 8)}.get(what, {})
    bwd_ptr = {"x+4": dict(x=FAKE + 4), "y+8": dict(dx=FAKE + 8)}.get(what, {})
    pack_ptr = {"x+4": dict(x=FAKE + 4), "y+8": dict(plane=FAKE + 8)}.get(what, {})
    _rc(_pool_fwd(lib, **shape, **fwd_ptr), E_UNSUPPORTED, lib, "bn_sign_pool")
    _rc(_pool_bwd(lib, **shape, **bwd_ptr), E_UNSUPPORTED, lib, "bn_sign_pool")
    _rc(_pool_bwd_pack(lib, **shape, **pack_ptr), E_UNSUPPORTED, lib)


def test_pooled_backward_refuses_a_misaligned_pooled_gradient():
    """g is read as float2: the non-pack pass refuses it as an argument error, the pack pass as outside its cover"""
    L, lib = _lib()
    _rc(_pool_bwd(lib, g=FAKE + 4), E_ARG, lib, "8-byte")
    _rc(_pool_bwd_pack(lib, g=FAKE + 4), E_UNSUPPORTED, lib)
    _rc(_pool_bwd_pack(lib, Cc=12, H=8, W=16), E_UNSUPPORTED, lib)     # C % 8 for the plane


@pytest.mark.parametrize("sg", [3, 7, 0])
def test_every_producer_refuses_a_shuffle_group_that_does_not_divide_C(sg):
    from micronet_b200 import functional as F_
    L, lib = _lib()
    qp = F_.ActSpec(L.ACT_DOREFA, bits=4).struct()
    word = "shuffle groups"
    _rc(lib.mnb_bn_sign_fwd(FAKE, 2, 16, 64, FAKE, FAKE, FAKE, FAKE, sg, FAKE, FAKE, None), E_ARG, lib, word)
    _rc(lib.mnb_bn_sign_bwd(FAKE, FAKE, FAKE, 2, 16, 64, FAKE, FAKE, FAKE, 1, sg, FAKE, FAKE, FAKE, None, FAKE, None),
        E_ARG, lib, word)
    _rc(_fwd_packed(lib, sg=sg), E_ARG, lib, word)
    _rc(_relu_quant(lib, qp, sg=sg), E_ARG, lib, word)
    _rc(_bwd_pack(lib, sg=sg), E_ARG, lib, word)
    _rc(_pool_fwd(lib, sg=sg), E_ARG, lib, word)
    _rc(_pool_bwd(lib, sg=sg), E_ARG, lib, word)
    _rc(_pool_bwd_pack(lib, sg=sg), E_ARG, lib, word)


@pytest.mark.parametrize("terms", [0, 4, -1])
def test_packed_backward_refuses_terms_outside_1_to_3(terms):
    L, lib = _lib()
    _rc(_bwd_pack(lib, terms=terms), E_ARG, lib, "bn_sign_bwd_pack")
    _rc(_pool_bwd_pack(lib, terms=terms), E_ARG, lib, "bn_sign_pool_bwd_pack")


def test_relu_quant_producer_refuses_a_quantizer_other_than_dorefa_2_to_8_bits():
    L, lib = _lib()
    for mode, bits in ((L.ACT_IAO, 8), (L.ACT_SIGN, 1), (L.ACT_DOREFA, 1), (L.ACT_DOREFA, 9), (7, 4)):
        qp = L.ActQParams(mode, bits, 0, 255, 0, None, None, None, None)
        _rc(_relu_quant(lib, qp), E_ARG, lib, "DoReFa")


def test_reduction_producers_refuse_more_than_8192_channels():
    """the split finalisers' completion counters are a fixed 8192-entry array of the scratch buffer"""
    L, lib = _lib()
    _rc(lib.mnb_bn_sign_bwd(FAKE, FAKE, FAKE, 2, 8200, 32, FAKE, FAKE, FAKE, 1, 1, FAKE, FAKE, FAKE, None, FAKE, None),
        E_ARG, lib, "bn_sign_bwd shape")
    _rc(_pool_bwd(lib, Cc=8200), E_ARG, lib, "bn_sign_pool shape")


# ---------------------------------------------------------------- the launch-path restatements, worked by hand
def test_plane_splits_hand_worked():
    # min(32, batch, batch * hw / 2048, ceil(2112 / C))
    assert plane_splits(256, 256 * 1024, 256) == 9        # 2112 / 256 = 8.25 -> 9
    assert plane_splits(256, 256 * 256, 512) == 5         # 4.125 -> 5
    assert plane_splits(256, 256 * 64, 1024) == 3         # 2.06 -> 3; 16384 / 2048 = 8
    assert plane_splits(37, 37 * 1935, 8) == 32           # 71595 / 2048 = 34, 2112 / 8 = 264, batch 37: the 32 slots
    assert plane_splits(8, 8 * 32, 64) == 1               # 256 / 2048 = 0 -> at least one
    assert plane_splits(2, 2 * 32, 8184) == 1             # ceil(2112 / 8184) = 1


def test_launch_paths_hand_worked():
    a = 1 << 20
    assert fwd_path(256 * 256 * 1024, 1024, a, a) == "v4"
    assert fwd_path(5 * 24 * 42, 42, a, a) == "scalar"               # hw % 4
    assert fwd_path(16 * 64 * 256, 256, a + 4, a + 4) == "scalar"    # 4-byte offset
    assert fwd_path(16 * 64 * 256, 256, a + 8, a + 8) == "scalar"    # 8-byte offset: still not 16
    assert bwd_path(8, 4, a, a, a + 16) == "vec" and bwd_path(8, 4, a, a + 4, a) == "scalar"
    assert fwd_path(2 ** 31, 1024, a, a) == "scalar"                 # 32-bit float4 indices
    assert pack_vec(1024, a, a, a) == 4 and pack_vec(1024, a, a, None) == 4
    assert pack_vec(64, a, a, a) == 2                                # the headline's 1024-channel 8x8 layers
    assert pack_vec(32, a, a, a) == 1
    assert pack_vec(256, a + 8, a + 8, a + 8) == 2 and pack_vec(256, a + 4, a + 4, None) == 1
    assert pack_vec(1024, a, a + 8, None) == 2
    # accumulation chains: vec = 2 pair adds + ceil(images * hw / 4 / 512); scalar ceil(hw / 256); pooled reduce
    # 2 * ceil(images * hw / 8 / 512), pooled apply 3 + ceil(images * hw / 8 / 256)
    assert reduce_chain("vec", 256, 1024, 9) == 2 + 15                # 29 images * 256 float4 / 512 = 14.5
    assert reduce_chain("scalar", 37, 1935, 32) == 8
    assert reduce_chain("pool", 256, 1024, 9) == 2 * 8                # 29 * 128 / 512 = 7.25
    assert apply_chain("pool", 256, 1024, 9) == 3 + 15


@pytest.mark.parametrize("workload", sorted(BENCH_PLANES))
def test_bench_producer_planes_are_the_ones_the_gpu_tests_run(workload):
    """the producer planes the prepare passes create in the bench models, derived from harness.models: a model change
    that moves a producer to a new plane must show up here (and in the cases of test_gpu_bn_producers.py)"""
    assert bench_planes(workload) == BENCH_PLANES[workload]
