"""Coverage of the packed-operand family by the GPU suite, checked on the host (no GPU needed).

The plan of a convolution (mnb_pk_conv_plan_ex / mnb_pk_wgrad_plan) selects the kernel instance and the code paths
inside it: segmented accumulation, the N tile, the number of M tiles per work item, the output phases of a stride-2 data
gradient; for the weight gradient the N tile, several taps per CTA and merged groups.  This test enumerates those
signatures for every conv of the bench models at every terms configuration the models use, and for every case of the
GPU tests (test_gpu_pk.py, test_gpu_pk_plans.py) with their environment overrides, and requires

* every model signature to be reached by some GPU case, and
* every pk_conv_kernel<SEG, Nt> and pk_wgrad_kernel<Nc> instance to be launched by some GPU case,

so a change of the plan heuristics or of a test list that leaves a production plan or an instance untested fails here,
naming what is now uncovered."""
import os

import pytest

from tests import pk_plan_util as PU
from tests.test_pk_plan_cpu import _model_convs

FWD_TERMS = [(1, 1), (2, 1), (3, 3), (1, 3)]     # integer levels, asymmetric levels, fp32 x fp32, fp32 x levels
BWD_TERMS = [(2, 1), (2, 2)]                     # two dy pieces (PK_TERMS_BWD) x integer / fp32 second operand


class _env:
    def __init__(self, env):
        self.env, self.old = env, {}

    def __enter__(self):
        for k, v in self.env.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _model_signatures():
    """{conv signature: [where]}, {wgrad signature: [where]} of the bench models"""
    conv, wgrad = {}, {}
    for name, B, Cc, H, W, K, R, st, pad, G in _model_convs():
        sh = PU.shape(B, Cc, H, W, K, R, st, pad, G)
        train = not name.startswith("res224")      # the 224 x 224 workload is inference only
        cfgs = [(0, t) for t in FWD_TERMS] + ([(1, t) for t in BWD_TERMS] if train else [])
        for mode, terms in cfgs:
            p = PU.conv_plan(sh, mode, *terms)
            if p is not None:
                conv.setdefault(PU.conv_signature(p), []).append(f"{name} mode {mode} terms {terms}")
        if train:
            for terms in BWD_TERMS:
                p = PU.wgrad_plan(sh, *terms)
                if p is not None:
                    wgrad.setdefault(PU.wgrad_signature(p), []).append(f"{name} wgrad terms {terms}")
    return conv, wgrad


def _gpu_cases():
    """(test id, kind, plan) of every launch of the GPU tests"""
    from tests import test_gpu_pk as T1, test_gpu_pk_plans as T2
    out = []
    for kind, s, terms in T1.plan_configs():
        sh = PU.shape(*s)
        p = PU.wgrad_plan(sh, *terms) if kind == "wgrad" else PU.conv_plan(sh, 0 if kind == "fwd" else 1, *terms)
        if p is not None:                      # (test_gpu_pk.py skips shapes outside the weight-gradient cover)
            out.append((f"test_gpu_pk {kind} {s} {terms}", kind, p))
    for case in T2.CASES:
        with _env(case.env):
            p = T2.plan_of(case)
        assert p is not None, case.id
        out.append((f"test_gpu_pk_plans {case.id}", case.kind, p))
    return out


@pytest.fixture(scope="module")
def cases():
    return _gpu_cases()


def test_model_conv_signatures_are_covered_by_gpu_cases(cases):
    model, _ = _model_signatures()
    assert len(model) >= 10, sorted(model)
    tested = {PU.conv_signature(p) for _, kind, p in cases if kind != "wgrad"}
    missing = {sig: model[sig][:3] for sig in model if sig not in tested}
    assert not missing, f"plans (segmented, Nt, MT, ny) of the bench models no GPU case runs: {missing}"


def test_model_wgrad_signatures_are_covered_by_gpu_cases(cases):
    _, model = _model_signatures()
    assert len(model) >= 5, sorted(model)
    tested = {PU.wgrad_signature(p) for _, kind, p in cases if kind == "wgrad"}
    missing = {sig: model[sig][:3] for sig in model if sig not in tested}
    assert not missing, f"weight-gradient plans (Nc, tpg > 1, gm > 1) of the bench models no GPU case runs: {missing}"


def test_every_kernel_instance_is_launched(cases):
    conv = {(bool(p["segmented"]), p["Nt"]) for _, kind, p in cases if kind != "wgrad"}
    want = {(seg, nt) for seg in (False, True) for nt in PU.CONV_NT}
    assert not want - conv, f"pk_conv_kernel<SEG, Nt> instances no GPU case launches: {sorted(want - conv)}"
    wg = {p["Nc"] for _, kind, p in cases if kind == "wgrad"}
    assert not set(PU.WGRAD_NC) - wg, f"pk_wgrad_kernel<Nc> instances no GPU case launches: {sorted(set(PU.WGRAD_NC) - wg)}"


def test_plan_query_agrees_with_the_16_field_query():
    """mnb_pk_conv_plan is mnb_pk_conv_plan_ex's first 16 fields; the wgrad query agrees with the scratch size"""
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    for name, B, Cc, H, W, K, R, st, pad, G in _model_convs()[::3]:
        sh = PU.shape(B, Cc, H, W, K, R, st, pad, G)
        old = (C.c_int32 * 16)()
        assert lib.mnb_pk_conv_plan(C.byref(sh), 0, 1, 1, old) == 0
        p = PU.conv_plan(sh, 0, 1, 1)
        assert list(old) == [p[f] for f in PU.CONV_FIELDS[:16]], name
        assert p["acc"] == p["MT"] * p["Nt"] and p["n_mgroups"] == -(-p["n_mtiles"] // p["MT"]), name
        assert p["n_items"] % p["n_mgroups"] == 0 and p["npairs"] == 1 and p["segmented"] == 0, name
        short = (C.c_int32 * 3)(-7, -7, -7)
        assert lib.mnb_pk_conv_plan_ex(C.byref(sh), 0, 1, 1, short, 2) == 0 and list(short)[2] == -7   # writes n fields only
        w = PU.wgrad_plan(sh, 2, 1)
        assert (w is None) == (lib.mnb_pk_wgrad_scratch_bytes(C.byref(sh), 2, 1) < 0), name
        if w is not None:
            assert w["tpg"] * w["Nc"] <= 128 and w["Nc"] in PU.WGRAD_NC, (name, w)


def test_conv_post_refuses_a_segmented_plan_before_launching():
    """a fused consumer epilogue exists only in the single-product kernels: mnb_pk_conv_post must refuse a segmented
    producer plan on the host (the pointers below are never dereferenced), not launch and leave the plane unwritten"""
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    fake = 4096
    qp = L.ActQParams(L.ACT_IAO, 8, -128, 127, 0, fake, fake, fake, fake)
    post = L.PkPost(C.pointer(qp), 0, 0, fake)
    sh = PU.shape(4, 64, 16, 16, 128, 3, 1, 1, 1)
    assert PU.conv_plan(sh, 0, 2, 1)["segmented"] == 1
    rc = lib.mnb_pk_conv_post(C.byref(sh), fake, 2, fake, 1, None, None, 1.0, None, None, C.byref(post), fake, None)
    assert rc == L.E_UNSUPPORTED and b"segmented" in lib.mnb_last_error()
    from micronet_b200 import pk as PK
    assert PK.segmented(sh, 0, 2, 1) and not PK.segmented(sh, 0, 1, 1)
