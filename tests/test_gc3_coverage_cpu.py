"""Coverage of the narrow grouped 3x3 convolutions (pk_gc3_kernel) by tests/test_gpu_gc3_fp64.py, checked on the host (no
GPU needed).

mnb_pk_gc3_plan runs the launcher's own make_gc3_plan.  This test requires

* every pinned plan of tests/gc3_cases.py to hold;
* every plan feature (groups per CTA block, m64 blocks, ring stages, image tiles per CTA, images per tile, short last
  tiles), padding and image edge to be reached by some case in each mode (forward fp32, codes, data gradient), on every
  operand kind and epilogue form;
* every refusal reason the host can reach to be listed, with the code and text of the query, and the others to be
  unreachable over a host sweep;
* the four bench launches of both NIN-GC workloads at batch 256 to be cases;
* the MNB_PK_* knobs that make_plan reads to keep the gc3 chain that of mnb_pk_conv's plan (the weight packer and the
  kernel read the same environment) or to refuse,

so deleting a case or a refusal, or a change of the plan heuristics that moves a case elsewhere, fails here naming what
lost its cover."""
import os
import re
import types

import pytest

from tests import gc3_cases as P
from tests import pk_plan_util as PU

CODES = {"E_ARG": -1, "E_UNSUPPORTED": -2}
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "micronet_b200", "csrc", "mnb_pk.cu")


@pytest.fixture(scope="module")
def plans():
    return {c.id: P.plan_of(c) for c in P.CASES}


def test_case_ids_are_unique():
    ids = [c.id for c in P.CASES] + [r.id for r in P.REFUSALS]
    assert len(ids) == len(set(ids))


def test_pinned_plans_hold(plans):
    bad = {}
    for c in P.CASES:
        p = plans[c.id]
        if not isinstance(p, dict):
            bad[c.id] = p
            continue
        got = {k: p[k] for k in c.expect}
        nt = 16 if c.mode == "dgrad" else 32
        if got != c.expect or p["Nt"] != nt or p["ncons"] != 3:
            bad[c.id] = (got, c.expect)
    assert not bad, f"plans changed or refused: {bad}"


# what each mode must reach (the host sweep below shows every one of them reachable in both plan modes)
WANT = ({"GB1", "GB2", "GB4", "nstage3", "nstage6", "TB1", "TB>1", "short_last_tile_of_several", "pad_h!=pad_w",
         "non_square", "one_row", "one_column", "widest_row", "G4", "G64"}
        | {f"nmb{i}" for i in range(1, 7)} | {f"pad_h{i}" for i in range(3)} | {f"pad_w{i}" for i in range(3)}
        | {f"tiles_per_cta{t}" for t in ("1", "2", "3..nstage", ">nstage")})
OPERANDS = {"fwd": {"pm1", "dorefa4", "int8"}, "codes": {"pm1", "dorefa4", "int8"}, "dgrad": {"int", "real"}}


def _epi_forms(c):
    e = c.epi
    if c.mode == "dgrad":
        return {"mask" if "gain" in e else "a_scale_const"}
    return {"n_scale" if e["n_scale"] else "no_n_scale", "a_scale_tensor" if e["a_scale"] == "tensor" else "a_scale_const",
            "bias" if e["bias"] else "no_bias"}


EPI_WANT = {"fwd": {"n_scale", "no_n_scale", "a_scale_tensor", "a_scale_const", "bias", "no_bias"},
            "codes": {"n_scale", "no_n_scale", "a_scale_tensor", "a_scale_const", "bias", "no_bias"},
            "dgrad": {"mask", "a_scale_const"}}


def test_every_feature_is_covered(plans):
    missing = {}
    for mode in P.MODES:
        got = set()
        for c in P.CASES:
            if c.mode == mode:
                got |= P.features(c, plans[c.id])
        if WANT - got:
            missing[mode] = sorted(WANT - got)
    assert not missing, f"plan features no case of the mode reaches: {missing}"


def test_every_operand_kind_and_epilogue_is_covered(plans):
    missing = {}
    for mode in P.MODES:
        cs = [c for c in P.CASES if c.mode == mode]
        ops = {c.operands for c in cs}
        epis = set().union(*(_epi_forms(c) for c in cs))
        if ops != OPERANDS[mode] or EPI_WANT[mode] - epis:
            missing[mode] = (sorted(OPERANDS[mode] ^ ops), sorted(EPI_WANT[mode] - epis))
        # both data-gradient operand kinds take both epilogue forms, and several groups per CTA block
        if mode == "dgrad":
            for kind in ("int", "real"):
                k = [c for c in cs if c.operands == kind]
                if set().union(*(_epi_forms(c) for c in k)) != EPI_WANT["dgrad"] or all(plans[c.id]["GB"] == 1 for c in k):
                    missing[f"dgrad_{kind}"] = "needs the mask, the constant and a case with GB > 1"
    # several groups per CTA block on every forward operand kind too
    for mode in ("fwd", "codes"):
        if not any(plans[c.id]["GB"] > 1 and c.mode == mode and c.epi["bias"] for c in P.CASES):
            missing[f"{mode}_gb_bias"] = "a case with GB > 1 and a bias"
    assert not missing, f"(operand kinds, epilogue forms) no case of the mode reaches: {missing}"


def _required_items(c, p):
    """what a case contributes to the coverage the tests above require: (mode, feature), (mode, operand kind), (mode,
    epilogue form), and the per-kind and GB > 1 combinations"""
    s = {(c.mode, f) for f in P.features(c, p) & WANT}
    s |= {(c.mode, "operands " + c.operands)} | {(c.mode, e) for e in _epi_forms(c)}
    if c.mode == "dgrad":
        s |= {(c.mode, c.operands, e) for e in _epi_forms(c)}
        if p["GB"] > 1:
            s.add((c.mode, c.operands, "GB>1"))
    elif p["GB"] > 1 and c.epi["bias"]:
        s.add((c.mode, "GB>1 with a bias"))
    return s


def test_every_case_is_needed(plans):
    """every case other than the bench launches is the only one to reach something the coverage requires, so that deleting
    any single case fails one of the coverage tests, naming what lost its cover"""
    items = {c.id: _required_items(c, plans[c.id]) for c in P.CASES}
    spare = []
    for c in P.CASES:
        if c.model:
            continue
        others = set().union(*(v for k, v in items.items() if k != c.id))
        if not items[c.id] - others:
            spare.append(c.id)
    assert not spare, f"cases whose coverage other cases already give (drop them or give them a feature of their own): {spare}"


def test_widest_row_is_the_last_before_the_box_refusal(plans):
    """the widest-row cases are the widest the query accepts: one column more is the 'image larger than one box' refusal"""
    for c in P.CASES:
        if "widest_row" not in P.features(c, plans[c.id]):
            continue
        B, Cc, H, W, K, ph, pw, G = c.shape
        got = P.query(P.conv_shape((B, Cc, H, W + 1, K, ph, pw, G)), c.mode, P.TERMS[c.mode])
        assert isinstance(got, tuple) and "image larger than one box" in got[1], (c.id, got)


# the modes each refusal reason is listed for
REFUSAL_MODES = {
    "pk gc3: filter is not 3x3": ("fwd", "dgrad"),
    "pk gc3: stride or dilation != 1": ("fwd", "dgrad"),
    "pk gc3: padding outside 0..2": ("fwd", "dgrad"),
    "pk gc3: needs 16 / 32 channels per group and groups % 4 == 0": ("fwd", "dgrad"),
    "pk gc3: the forward takes one activation piece and one weight piece": ("fwd",),
    "pk gc3: the data gradient takes two dy pieces and one weight piece": ("dgrad",),
    "pk gc3: plan is segmented or tiled along N": ("dgrad",),     # a forward plan has one piece pair: never segmented
    "pk conv: empty output": ("fwd", "dgrad"),
    "pk gc3: image larger than one box": ("fwd", "codes", "dgrad"),
    "pk gc3: no image tile fits the accumulators and shared memory": ("fwd", "dgrad"),
    "pk gc3: operands and output must be 16-byte aligned": ("fwd", "codes", "dgrad"),
    "pk_gc3_conv_codes: sums of 16 x 3 x 3 terms": ("codes",),
}


def _make_gc3_plan_reasons():
    src = open(SRC).read()
    body = src[src.index("static int make_gc3_plan("):]
    body = body[:body.index("\n}\n")]
    return set(re.findall(r'\bno\("([^"]+)"\)', body))


def test_every_refusal_reason_is_listed_and_agrees_with_the_query():
    from micronet_b200 import _lib as L
    bad = {}
    for r in P.REFUSALS:
        with PU.env(r.env):
            got = P.query(P.refusal_shape(r), r.mode, r.terms)
        if r.launch:
            # the plan accepts; the launcher refuses (alignment, the codes bound)
            if not isinstance(got, dict):
                bad[r.id] = got
        elif not isinstance(got, tuple) or got[0] != CODES[r.code] or got[1] != r.text:
            bad[r.id] = got
    assert not bad, bad
    listed = {r.text for r in P.REFUSALS}
    # one refusal per (reason, mode) in every mode where the reason can be met: the forward plan query serves the fp32 and
    # the codes entry points alike, so the codes mode only lists what its own entry point adds
    keys = [(r.text.split(" of level")[0], r.mode) for r in P.REFUSALS]
    assert len(keys) == len(set(keys)), "two refusals stand for the same (reason, mode)"
    want = {(t, m) for t, ms in REFUSAL_MODES.items() for m in ms}
    missing = sorted(want - set(keys))
    assert not missing, f"(reason, mode) no listed refusal reaches: {missing}"
    assert set(keys) <= want, sorted(set(keys) - want)
    reasons = {f"pk gc3: {t}" for t in _make_gc3_plan_reasons()}
    unreachable = {f"pk gc3: {t}" for t in P.UNREACHABLE}
    missing = sorted(reasons - listed - unreachable)
    assert not missing, f"refusal reasons of make_gc3_plan no listed shape reaches: {missing}"
    assert not (listed & unreachable), "a reason listed as unreachable has a refusal shape"
    assert unreachable <= reasons, f"unreachable reasons make_gc3_plan no longer has: {sorted(unreachable - reasons)}"
    # the refusals of the launchers and of make_plan
    for want in ("pk conv: empty output", "pk gc3: operands and output must be 16-byte aligned",
                 f"pk_gc3_conv_codes: sums of 16 x 3 x 3 terms of level {P.CODES_BOUND_REFUSED} may exceed int16"):
        assert want in listed, want
    assert L.E_UNSUPPORTED == CODES["E_UNSUPPORTED"]


def test_sweep_reaches_the_listed_reasons_only():
    """a host sweep over shapes, paddings and batches: every refusal is a listed reason, the unreachable ones never occur,
    and every wanted plan feature occurs in both plan modes"""
    reached = {"fwd": set(), "dgrad": set()}
    texts = set()
    n = 0
    for mode in ("fwd", "dgrad"):
        for B in (1, 2, 3, 5, 7, 37):
            for G in (4, 64):
                for H in (1, 2, 3, 4, 6, 9, 16, 33):
                    for W in (1, 3, 18, 30, 33, 34, 40, 61, 63, 64, 83, 96, 100, 104, 126, 127, 130):
                        for ph in range(3):
                            for pw in range(3):
                                shape = (B, 16 * G, H, W, 32 * G, ph, pw, G)
                                p = P.query(P.conv_shape(shape), mode, P.TERMS[mode])
                                n += 1
                                if isinstance(p, tuple):
                                    texts.add(p[1])
                                    continue
                                reached[mode] |= P.features(P.Case("s", shape, mode, "", {}, {}), p)
    assert n > 20000
    listed = {r.text for r in P.REFUSALS if not r.launch}
    assert texts <= listed, f"refusals the sweep meets that no listed shape reaches: {sorted(texts - listed)}"
    assert not any(u in t for t in texts for u in P.UNREACHABLE)
    for mode in reached:
        assert WANT <= reached[mode], (mode, sorted(WANT - reached[mode]))


# ---- the bench launches of the two NIN-GC workloads
def _bench_launches():
    """(workload, layer, mode, shape, pieces) of every gc3 launch of a bench step at batch 256: the forward and the data
    gradient of the grouped 3x3 layers, at the piece counts the engine gives them"""
    from micronet_b200 import _lib as L, functional as F_
    Tb = min(L.PK_TERMS, L.PK_TERMS_BWD)
    out = []
    for name, B, Cc, H, W, K, R, st, pad, G in PU.model_convs():
        if not name.startswith("gc") or R != 3:
            continue
        shape = (B, Cc, H, W, K, pad, pad, G)
        for wl, spec, pm1 in (("nin_gc_wbwtab_w3a2", None, True),
                              ("nin_gc_dorefa_w4a4", types.SimpleNamespace(mode=L.ACT_DOREFA, q_type=0, bits=4), False)):
            ta, tw = F_._pk_terms(spec, True, pm1)
            fwd = "codes" if wl.startswith("nin_gc_wbwtab") else "fwd"
            out.append((wl, name, fwd, shape, (ta, tw)))
            out.append((wl, name, "dgrad", shape, (Tb, 1)))
    return out


def test_every_bench_launch_is_a_case(plans):
    launches = _bench_launches()
    assert {(wl, n) for wl, n, *_ in launches} == {(w, n) for w in ("nin_gc_wbwtab_w3a2", "nin_gc_dorefa_w4a4")
                                                   for n in ("gc3x3g16", "gc3x3g32")}
    missing = []
    for wl, name, mode, shape, terms in launches:
        hits = [c for c in P.CASES if c.model == (wl, name) and c.mode == mode and tuple(c.shape) == shape]
        if not hits or P.TERMS[mode] != terms or not isinstance(plans[hits[0].id], dict):
            missing.append((wl, name, mode, shape, terms))
    assert not missing, f"bench launches no case runs: {missing}"
    assert len([c for c in P.CASES if c.model]) == len(launches)
    # the epilogues of the bench launches: DoReFa forward at a_scale_const 1/15 with n_scale and bias, data gradient under
    # the STE mask with the gain 0.1 (tests/test_gpu_gc3_fp64.py checks that route in the model step); wbwtab forward as
    # codes, data gradient behind the fused producer at a_scale_const 1
    for c in P.CASES:
        if c.model and c.mode == "dgrad":
            assert c.epi == ({"gain": 0.1} if "dorefa" in c.model[0] else {"a_scale": 1.0}) and c.operands == "real", c.id
        elif c.model and c.mode == "fwd":
            assert c.operands == "dorefa4" and c.epi == {"n_scale": 1, "a_scale": 1 / 15, "bias": 1}, c.id
        elif c.model:
            assert c.operands == "pm1", c.id


def _expected_chain(conv_plan, mode):
    """the chain of make_plan's program for one accumulator: K chunks -> piece pairs (small products first) -> the nine
    taps -> K-steps, when the nine taps form one stage template (TG = 9)"""
    ta, tw = P.TERMS[mode]
    lim = max(ta, tw) - 1
    pairs = [(a, s - a) for s in range(lim, -1, -1) for a in range(ta) if 0 <= s - a < tw]
    ks = conv_plan["CC"] // 16
    return [(t, a, b, cc * ks + j) for cc in range(conv_plan["chunks"]) for a, b in pairs for t in range(9)
            for j in range(ks)]


@pytest.mark.parametrize("env", [{}, {"MNB_PK_COLTILES": "2"}, {"MNB_PK_COLTILES": "3"}, {"MNB_PK_MT": "2"},
                                 {"MNB_PK_MT": "4"}, {"MNB_PK_STAGES": "2"}, {"MNB_PK_STAGES": "4"},
                                 {"MNB_PK_SEG_MMAS": "16"}, {"MNB_PK_SEG_MMAS": "36"}],
                         ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()) or "default")
def test_make_plan_knobs_keep_the_chain_of_mnb_pk_conv(env):
    """under every MNB_PK_* knob make_plan reads, the gc3 plan of each bench layer either refuses or runs the chain of
    mnb_pk_conv_plan_ex's plan (chunks, K-steps, piece pairs); the weight image is packed by that plan, so this is the one
    way the image could disagree with the kernel's program"""
    from micronet_b200 import pk as PK
    seen = 0
    with PU.env(env):
        for c in P.CASES:
            if not c.model:
                continue
            sh = P.conv_shape(c.shape)
            mode = 1 if c.mode == "dgrad" else 0
            g = P.query(sh, c.mode, P.TERMS[c.mode], chain=True)
            cp = PU.conv_plan(sh, mode, *P.TERMS[c.mode])
            # the cached Python query agrees with the C query under the same environment
            pg = PK.gc3_plan(sh, mode, *P.TERMS[c.mode])
            if isinstance(g, tuple):
                assert pg is None and cp is not None and (cp["segmented"] or cp["n_ntiles"] > 1), (c.id, g, cp)
                assert "segmented" in g[1]
                continue
            seen += 1
            assert pg is not None and pg["chain"] == g["chain_mmas"]
            assert not cp["segmented"] and cp["n_ntiles"] == 1 and cp["Nt"] == g["Nt"]
            assert g["chain_mmas"] == _expected_chain(cp, c.mode), (c.id, env)
    segmenting = "MNB_PK_SEG_MMAS" in env and int(env["MNB_PK_SEG_MMAS"]) < 36
    assert seen == (4 if segmenting else 8), seen     # a segmented plan refuses the data gradient only
