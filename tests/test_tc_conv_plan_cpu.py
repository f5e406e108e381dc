"""Coverage of the round-1 fused tensor-core convolutions (csrc/mnb_conv_tc_fwd.cu, csrc/mnb_conv_tc_wgrad.cu) by
tests/tc_conv_cases.py, checked on the host with the launchers' own plan functions (mnb_tc_conv_plan / mnb_wgrad_tc_plan; no
GPU needed):

* every conv_tc_kernel<NG> instance is launched by some case, in forward and in data-gradient mode,
* every plan feature the case list is written for is reached,
* every case's plan is still the one pinned beside it,
* every refusal reason of both plan() functions is reached by a refusal case, or is listed as unreachable,
* every quantized conv of the wbwtab NIN / NIN-GC training graphs (A = 2 unfused: the 1x1 layers; A = 32: all of them)
  runs a plan some case runs, or is refused with a listed reason,

so a change of the plan heuristics or of the case list that leaves an instance, a feature or a model layer untested fails
here, naming it."""
import itertools
import os
import re

import pytest

from tests import tc_conv_cases as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _launches():
    return [(case, kind, p) for case in T.CASES for kind, p in T.launches(case)]


def test_every_kernel_instance_is_launched():
    got = {("dgrad" if k == "dgrad" else "fwd", p["NG"]) for _, k, p in _launches() if k != "wgrad"}
    missing = [(d, ng) for d in ("fwd", "dgrad") for ng in T.INSTANCES if (d, ng) not in got]
    assert not missing, f"conv_tc_kernel<NG> instances no case launches (mode, NG): {missing}"


def test_every_plan_feature_is_reached():
    got = set()
    for case, kind, p in _launches():
        got |= T.features(case, kind, p)
    assert not T.WANTED_FEATURES - got, f"plan features no case reaches: {sorted(T.WANTED_FEATURES - got)}"
    assert len(T.WANTED_FEATURES) >= 40


def test_every_case_runs_its_pinned_plan():
    ids = [c.id for c in T.CASES]
    assert len(ids) == len(set(ids)), "duplicate case ids"
    changed = {}
    for case in T.CASES:
        now = T.plans(case.shape)
        if now != (case.fwd, case.dgrad, case.wgrad):
            changed[case.id] = {"pinned": (case.fwd, case.dgrad, case.wgrad), "now": now}
    assert not changed, f"plans that changed under the cases written for them: {changed}"


def _reasons(src):
    text = open(os.path.join(ROOT, "micronet_b200", "csrc", src)).read()
    return set(re.findall(r'unsupported\("([^"]+)"\)', text))


def test_every_refusal_reason_is_reached():
    want = {("fwd", r) for r in _reasons("mnb_conv_tc_fwd.cu")} | {("wgrad", r) for r in _reasons("mnb_conv_tc_wgrad.cu")}
    assert len(want) >= 18
    wrong = []
    for id, kind, shape, reason in T.REFUSALS:
        got = T.refusal9(kind, shape)
        if got != reason:
            wrong.append((id, reason, got))
    assert not wrong, f"refusal cases refused for another reason (id, pinned, now): {wrong}"
    reached = {("fwd" if k == "dgrad" else k, r) for _, k, _, r in T.REFUSALS}
    missing = want - reached - set(T.UNREACHABLE)
    assert not missing, f"refusal reasons no case reaches: {sorted(missing)}"
    assert not set(T.UNREACHABLE) - want, "UNREACHABLE names a reason the sources no longer have"
    assert not set(T.UNREACHABLE) & reached


def test_unreachable_refusals_stay_unreachable():
    """the reasons listed as unreachable are not met over a sweep of group widths, filters and planes"""
    seen = set()
    for cg, ng, G, R, W, H in itertools.product(range(16, 337, 16), range(16, 337, 16), (1, 3), (1, 3, 5, 7),
                                               (4, 44, 60, 64), (7, 255)):
        shape = (2, cg * G, H, W, ng * G, R, 1, R // 2, G)
        for kind in ("fwd", "dgrad", "wgrad"):
            r = T.refusal9(kind, shape)
            if r is not None:
                seen.add(("fwd" if kind == "dgrad" else kind, r))
    assert not seen & set(T.UNREACHABLE), seen & set(T.UNREACHABLE)
    assert len(seen) >= 7


def _model_convs():
    from tests.pk_plan_util import model_convs as convs
    out = []
    for name, B, Cc, H, W, K, R, st, pad, G in convs():
        if name.startswith(("gc", "nin")) and not name.endswith("head"):
            assert st == 1 and pad == R // 2
            out.append((name, (B, Cc, H, W, K, R, G)))
    return out


def test_model_convs_are_covered_by_cases():
    """A = 32: every quantized conv of NIN and NIN-GC; A = 2 unfused: their 1x1 convs (the 3x3 / 5x5 ones take the
    packed-operand family).  Both graphs' convs run (fwd, dgrad, wgrad) plans some case runs, or are refused with a reason
    a refusal case pins."""
    tested = {(k, tuple(p.values())) for _, k, p in _launches()}
    reasons = {("fwd" if k == "dgrad" else k, r) for _, k, _, r in T.REFUSALS}     # forward and dgrad share plan()
    convs = _model_convs()
    assert len(convs) == 11
    missing = []
    for name, shape in convs:
        f, d, w = T.plans(shape)
        for kind, p in (("fwd", f and f[0]), ("dgrad", d), ("wgrad", w)):
            if p is None:
                r = T.refusal(kind, shape)
                if ("fwd" if kind == "dgrad" else kind, r) not in reasons:
                    missing.append((name, kind, "refused: " + r))
            elif (kind, p) not in tested:
                missing.append((name, kind, p))
    assert not missing, f"model convs whose plan no case runs: {missing}"
    for name, shape in convs:
        assert any(c.shape == shape for c in T.CASES if c.id in T.MODEL_CASES), name


def test_model_conv_plans():
    """which launcher takes which model conv (the training tests assert that these launches happen)"""
    acc = {name: tuple(T.refusal(k, s) is None for k in ("fwd", "dgrad", "wgrad")) for name, s in _model_convs()}
    assert acc == {
        "gc1x1g2": (True, True, True), "gc3x3g16": (True, True, True), "gc1x1g4": (True, True, True),
        "gc3x3g32": (True, True, True), "gc1x1g8": (True, True, True),
        "nin1x1a": (True, False, True), "nin1x1b": (True, True, True), "nin5x5": (False, False, True),
        "nin1x1c": (False, False, True), "nin3x3": (False, False, True), "nin1x1d": (False, False, True),
    }
    nin5 = dict(_model_convs())["nin5x5"]
    assert T.refusal("fwd", nin5) == "channels per group"                     # 192 output channels
    assert T.refusal("dgrad", nin5) == "weights of one group do not fit in shared memory"
    w = T.wd(T.wgrad_plan(nin5))
    assert (w["nsplit"], w["tap_groups"]) == (2, 5)
    assert T.refusal("dgrad", dict(_model_convs())["nin1x1a"]) == "channels per group"   # NG = 192


@pytest.mark.parametrize("kind", ["fwd", "dgrad", "wgrad"])
def test_plan_query_refuses_bad_arguments(kind):
    from micronet_b200 import _lib as L
    lib = L.load()
    if kind == "wgrad":
        assert lib.mnb_wgrad_tc_plan(None, 0, None, 0) < 0
    else:
        assert lib.mnb_tc_conv_plan(None, int(kind == "dgrad"), 0, None, 0) < 0
