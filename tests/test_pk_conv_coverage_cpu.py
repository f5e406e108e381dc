"""Coverage of the packed-operand family's general kernels by tests/pk_conv_cases.py, checked on the host (no GPU needed).

* every case's plan still has the fields it was pinned to, and refusal cases are still refused for their reason;
* the cases reach every pk_conv_kernel instance of rows 0 / 1 (forward and data gradient) and row 2 (int8), every
  pk_wgrad_kernel<Nc>, every plan feature and epilogue form listed below, and every refusal reason of the source that a
  shape can reach (the others are listed in pk_conv_cases.UNREACHABLE with the reason);
* the cases reach every plan signature of the bench models' convs at every terms configuration the models use (forward,
  data gradient, weight gradient, and int8 for the ResNet convs), and every (mode, terms, signature) the older
  packed-operand tests launched (RETIRED_LAUNCHES), and set every MNB_PK_* knob those launches set;
* a seeded sweep of random shapes at the term counts the models use meets no refusal reason outside that list, and for
  every shape the plan query and the launch agree: the launch, given a misaligned operand pointer, returns the query's code
  and text where the query refuses, and fails at the operand's tensor map (before any kernel launch) where it accepts;
* the 7x7 stride-2 data gradient whose MMA program does not fit is refused by the query, so the layer runs on the
  generic kernels instead of failing in its backward."""
import ctypes as C
import os
import random
import re

import pytest

from tests import pk_conv_cases as PC
from tests import pk_plan_util as PU
from tests.pk_plan_util import case_shape as shape, query

ROOT = PU.ROOT
FWD_TERMS = [(1, 1), (2, 1), (3, 3), (1, 3)]     # integer levels, asymmetric levels, fp32 x fp32, fp32 x levels
BWD_TERMS = [(2, 1), (2, 2)]                     # two dy pieces (PK_TERMS_BWD) x integer / fp32 second operand
MISALIGNED = 4096 + 8        # never dereferenced: the first tensor map refuses a base that is not 16-byte aligned
SMEM_BUDGET = 227 * 1024 - 3072


def fake_launch(mode, sh, terms):
    """(code, text) of the launch with a misaligned streamed operand: refusals come first, else the tensor map fails"""
    from micronet_b200 import _lib as L
    lib = L.load()
    f = MISALIGNED
    if mode == "wgrad":
        rc = lib.mnb_pk_wgrad(C.byref(sh), f, terms[0], f, terms[1], None, None, f, f, f, None)
    elif mode == "i8":
        rc = lib.mnb_pk_i8_conv(C.byref(sh), f, f, None, None, 1.0, None, f, None, f, None)
    else:
        rc = lib.mnb_pk_conv(C.byref(sh), 0 if mode == "fwd" else 1, f, terms[0], f, terms[1], None, None, 1.0, None, None, 1.0,
                             f, f, None)
    return rc, (lib.mnb_last_error() if rc else b"")


def case_plan(case):
    with PU.env(case.env):
        return query(case.mode, shape(case.shape), case.terms)


@pytest.fixture(scope="module")
def plans():
    return {c.id: case_plan(c) for c in PC.CASES}


# ---- what the cases must reach
def conv_features(case, p):
    """plan features of a forward / data-gradient / int8 case"""
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    fwd = case.mode != "dgrad"
    kg, ng = (Cc // G, K // G) if fwd else (K // G, Cc // G)
    OHr, OWr = ((H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1) if fwd else (H // st, W // st)
    cpu = 16 if case.mode == "i8" else 8
    nk16 = -(-kg // (2 * cpu))
    ksteps = p["CC"] // (2 * cpu)
    wt = -(-OWr // p["col_tiles"])
    kph = {((r - ph) & 1) * 2 + ((q - pw) & 1) for r in range(R) for q in range(S)} if (fwd and st == 2) else {0}
    m = case.mode
    f = {f"{m} MT{p['MT']}" + (" partial last M group" if p["n_mtiles"] % p["MT"] else "")}
    f |= {f"{m} nstage {p['nstage']}", f"{m} npairs {p['npairs']}"}
    if p["TB"] > 1: f.add(f"{m} TB > 1")
    if p["col_tiles"] > 1 and OWr % wt: f.add(f"{m} partial last column tile")
    if OHr % p["TH"]: f.add(f"{m} partial last row tile")
    if p["chunks"] > 1 and nk16 % ksteps: f.add(f"{m} ragged last K chunk")
    if kg % 16: f.add(f"{m} kg % 16 != 0")
    if any(p[f"ntmpl{y}"] > (len(kph) if y == 0 else 1) for y in range(p["ny"])): f.add(f"{m} several tap groups in a k-phase")
    if fwd and st == 2: f.add(f"{m} stride 2 (4 k-phases)")
    if p["ny"] == 4: f.add(f"{m} 4 output phases")
    if p["ny"] == 4 and min(p[f"ntap{y}"] for y in range(4)) == 0: f.add(f"{m} output phase without a tap")
    if p["n_ntiles"] > 1 and ng % p["Nt"]: f.add(f"{m} partial last N tile")
    if ng % 16: f.add(f"{m} ng % 16 != 0")
    if G > 1 and (kg % 8 or ng % 8) and cpu == 8: f.add(f"{m} group-padded planes")
    if p["segmented"]:
        f.add(f"{m} seg_len {'1' if p['seg_len'] == 1 else '> 1'}")
        if p["last_seg"] < p["seg_len"]: f.add(f"{m} partial last segment")
    if p["n_items"] > 132 // p["ny"] and (p["n_ntiles"] > 1 or G > 1): f.add(f"{m} more items than CTAs, N tile / group change")
    return f


def wgrad_features(case, p):
    B, Cc, H, W, K, R, S, st, ph, pw, G = case.shape[:11]
    cin = (-(-(Cc // G) // 8) * 8 if G > 1 else Cc // G) * p["gm"]
    f = {f"wgrad gm {p['gm']}", f"wgrad nkph_used {p['nkph_used']}", f"wgrad nstage {p['nstage']}"}
    if p["n_ctiles"] > 1 and cin % p["Nc"]: f.add("wgrad partial last c tile")
    if p["n_ktiles"] > 1: f.add("wgrad n_ktiles > 1")
    if p["tpg"] > 1 and (R * S) % p["tpg"]: f.add("wgrad short last tap group")
    if G > 1 and ((Cc // G) % 8 or (K // G) % 8): f.add("wgrad group-padded channels")
    if p["NI"] > 1 and p["nsub"] % p["NI"]: f.add("wgrad NI > 1, short last stage")
    if p["splits"] > 1 and p["nstg_total"] % p["stg_per_split"]: f.add("wgrad splits > 1, short last split")
    # raster from the second shared-memory pass: its sub-block is over the first pass's limit
    hlo = max(0, max(-((r - ph) >> (st - 1)) for r in range(R)))
    hhi = max(0, max((r - ph) >> (st - 1) for r in range(R)))
    dyb = -(-(16 * p["TH"] * p["BW"] * 16) // 128) * 128
    xb = -(-((p["Nc"] // 8) * (p["TH"] + hlo + hhi) * p["BW"] * 16 + 256) // 128) * 128
    if case.terms[0] * dyb + case.terms[1] * p["nkph_used"] * xb > (SMEM_BUDGET - 2048) // 4:
        f.add("wgrad raster from the second shared-memory pass")
    return f


def epilogue_forms(case):
    e = case.epi
    if case.mode in ("fwd", "i8"):
        return {f"{case.mode} n_scale {e['n_scale']}", f"{case.mode} a_scale {e['a_scale']}", f"{case.mode} bias {e['bias']}"}
    if case.mode == "dgrad":
        return {f"dgrad STE mask gain {e['gain']}" if e["gain"] is not None else "dgrad a_scale_const alone"}
    return {f"wgrad a_scale {e['a_scale']}", f"wgrad kdiv {e['kdiv']}"}


WANT_FEATURES = (
    {f"{m} MT{t} partial last M group" for m in ("fwd",) for t in (2, 4)} | {"dgrad MT2 partial last M group"} |
    {"fwd MT1", "dgrad MT1"} |
    {f"{m} {f}" for m in ("fwd", "dgrad") for f in ("TB > 1", "partial last row tile", "kg % 16 != 0", "partial last N tile",
                                                   "ng % 16 != 0", "group-padded planes")} |
    {"fwd partial last column tile", "fwd ragged last K chunk", "fwd several tap groups in a k-phase", "fwd stride 2 (4 k-phases)",
     "dgrad 4 output phases", "dgrad output phase without a tap", "fwd more items than CTAs, N tile / group change"} |
    {f"fwd nstage {n}" for n in (2, 4, 8)} | {"fwd seg_len 1", "fwd seg_len > 1", "fwd partial last segment", "dgrad seg_len > 1"} |
    {"fwd npairs 1", "fwd npairs 2", "fwd npairs 3", "fwd npairs 6", "dgrad npairs 2", "dgrad npairs 3"} |
    {"i8 partial last N tile", "i8 kg % 16 != 0"} |
    {"wgrad partial last c tile", "wgrad n_ktiles > 1", "wgrad short last tap group", "wgrad group-padded channels",
     "wgrad NI > 1, short last stage", "wgrad splits > 1, short last split", "wgrad raster from the second shared-memory pass"} |
    {f"wgrad gm {g}" for g in (1, 2, 4, 8, 16)} | {f"wgrad nkph_used {k}" for k in (1, 2, 4)} | {"wgrad nstage 2", "wgrad nstage 4"})

WANT_EPILOGUES = (
    {f"{m} n_scale {v}" for m in ("fwd", "i8") for v in (True, False)} | {f"{m} a_scale {v}" for m in ("fwd", "i8") for v in ("dev", "const")} |
    {f"{m} bias {v}" for m in ("fwd", "i8") for v in (True, False)} |
    {"dgrad STE mask gain 0.1", "dgrad STE mask gain 1.0", "dgrad a_scale_const alone"} |
    {f"wgrad {k} {v}" for k in ("a_scale", "kdiv") for v in (True, False)})


def covered(plans):
    """{item: [case ids]} of instances, features, epilogue forms and (reason, mode)"""
    cov = {}
    for case in PC.CASES:
        rc, text, p = plans[case.id]
        items = set()
        if case.refuse:
            items.add(("refusal", case.refuse, case.mode))
        elif case.mode == "wgrad":
            items |= {("instance", "wgrad", p["Nc"])} | wgrad_features(case, p) | epilogue_forms(case)
        else:
            row = 2 if case.mode == "i8" else p["segmented"]
            items |= {("instance", case.mode, row, p["Nt"])} | conv_features(case, p) | epilogue_forms(case)
        for it in items:
            cov.setdefault(it, []).append(case.id)
    return cov


def test_case_ids_are_unique():
    ids = [c.id for c in PC.CASES]
    assert len(ids) == len(set(ids)), [i for i in ids if ids.count(i) > 1]


@pytest.mark.parametrize("case", PC.CASES, ids=lambda c: c.id)
def test_pinned_plan_holds(case, plans):
    rc, text, p = plans[case.id]
    if case.refuse:
        assert rc != 0 and case.refuse.encode() in text, (case.id, rc, text)
        return
    assert rc == 0, (case.id, text)
    got = {k: p[k] for k in case.pin}
    assert got == case.pin, f"{case.id}: the plan heuristics changed, the case no longer runs the plan it was written for"


def test_every_kernel_instance_is_reached(plans):
    cov = covered(plans)
    want = {("instance", m, row, nt) for m in ("fwd", "dgrad") for row in (0, 1) for nt in PU.CONV_NT}
    want |= {("instance", "i8", 2, nt) for nt in PU.CONV_NT} | {("instance", "wgrad", nc) for nc in PU.WGRAD_NC}
    missing = sorted(want - set(cov))
    assert not missing, f"kernel instances no case launches: {missing}"


def test_every_plan_feature_and_epilogue_is_reached(plans):
    cov = covered(plans)
    missing = sorted((WANT_FEATURES | WANT_EPILOGUES) - set(cov))
    assert not missing, f"plan features / epilogue forms no case reaches: {missing}"


def _source_reasons():
    """refusal texts of make_plan, conv_route (without a consumer), conv_mma and make_wg_plan_nc"""
    src = open(os.path.join(ROOT, "micronet_b200", "csrc", "mnb_pk.cu")).read()
    def body(name):
        i = src.index(f"static int {name}(")
        return src[i:src.index("\n}\n", i)]
    reasons = set()
    for name in ("make_plan", "conv_mma"):
        reasons |= set(re.findall(r'unsupported\("([^"%]+)', body(name)))
        reasons |= set(re.findall(r'mnb_fail\(MNB_E_\w+, "pk conv: ([^"%]+)', body(name)))
    route = body("conv_route")
    route = route[route.index("int ki = -1"):]          # the checks that apply without a consumer
    reasons |= {m.strip() for m in re.findall(r'"pk conv: ([^"%]+)', route)}
    reasons |= {("wgrad", m.strip()) for m in re.findall(r'"pk wgrad: ([^"%(]+)', body("make_wg_plan_nc"))}
    return reasons


def test_every_refusal_reason_is_cased_or_listed(plans):
    cov = covered(plans)
    cased = {(it[2] == "wgrad", it[1]) for it in cov if it[0] == "refusal"}
    for r in _source_reasons():
        wg = isinstance(r, tuple)
        text = r[1] if wg else r
        hit = any(w == wg and (text in c or c in text) for w, c in cased) or any(u in text for u in PC.UNREACHABLE)
        hit = hit or any(u in text for u in PC.UNCASED)
        assert hit, f"refusal reason {'pk wgrad' if wg else 'pk conv'}: {text!r} has no case and is not listed as unreachable"


@pytest.mark.parametrize("case", [c for c in PC.CASES if c.refuse], ids=lambda c: c.id)
def test_refusal_launch_returns_the_query_code_and_text(case):
    with PU.env(case.env):
        sh = shape(case.shape)
        q = query(case.mode, sh, case.terms)
        f = fake_launch(case.mode, sh, case.terms)
    assert q[0] != 0 and (q[0], q[1]) == f, (case.id, q[:2], f)


# ---- the sweep
_MODES = [("fwd", (1, 1)), ("fwd", (2, 1)), ("fwd", (3, 1)), ("fwd", (3, 3)), ("dgrad", (2, 1)), ("dgrad", (2, 2)),
          ("i8", (1, 1)), ("wgrad", (2, 1)), ("wgrad", (2, 2)), ("wgrad", (3, 3))]


def _random_shape(rng):
    G = rng.choice([1, 1, 1, 2, 3, 4, 8, 16])
    cg, kg = rng.choice([1, 3, 8, 12, 16, 24, 32, 48, 64, 96, 128, 192]), rng.choice([1, 3, 8, 12, 16, 24, 32, 48, 64, 96, 128, 256])
    R, S = rng.randint(1, 9), rng.randint(1, 9)
    st = rng.choice([1, 1, 2, 2, 3])
    ph, pw = rng.randint(0, R), rng.randint(0, S)
    H, W = rng.randint(1, 40), rng.randint(1, 140)
    if st == 2 and rng.random() < 0.8:
        H, W = H + (H & 1), W + (W & 1)
    dil = 2 if rng.random() < 0.01 else 1
    return (rng.randint(1, 8), cg * G, H, W, kg * G, R, S, st, ph, pw, G, dil)


def test_sweep_query_and_launch_agree():
    from micronet_b200 import _lib as L
    rng = random.Random(20251018)
    # reasons listed as unreachable are not known: the sweep meeting one fails and names it
    known = {r if isinstance(r, str) else r[1] for r in _source_reasons()}
    known = {k for k in known if not any(u in k for u in PC.UNREACHABLE)}
    known |= {"bad conv shape", "conv shape"}
    n, refused, reasons = 0, 0, set()
    while n < 20000:
        s = _random_shape(rng)
        sh = shape(s)
        for mode, terms in _MODES:
            if mode == "wgrad" and s[11] == 1 and rng.random() < 0.5:
                continue
            q_rc, q_text, _ = query(mode, sh, terms)
            f_rc, f_text = fake_launch(mode, sh, terms)
            if q_rc:
                refused += 1
                assert (f_rc, f_text) == (q_rc, q_text), (mode, terms, s, q_text, f_text)
                t = q_text.decode()
                assert any(k in t for k in known), f"refusal outside the known reasons (or listed unreachable): {mode} {terms} {s}: {t}"
                reasons.add(t.split(":")[1].split("(")[0].strip() if ":" in t else t)
            else:
                assert f_rc != 0 and b"cuTensorMapEncodeTiled" in f_text, (mode, terms, s, f_rc, f_text)
        n += 1
    assert refused > 1000, refused
    assert any("MMA program longer" in r for r in reasons), sorted(reasons)


# ---- plan signatures: the bench models' and the retired tests'
# (mode, terms, plan signature, operand kind, MNB_PK_* knobs) of every launch of the packed-operand tests the case list
# replaced: 20 ResNet / NIN / NIN-GC shapes at forward (1, 1) / (3, 3), data gradient (2, 1) / (3, 1) and weight gradient
# (2, 1) / (2, 2) / (3, 1) / (3, 3), the bench models' multi-tile plans at reduced batch, the plans forced through the
# knobs, and the int8 cases (signature (Nt, MT, phase split)).  Their backward ran on fp32 dy (every dy piece nonzero), so a
# case of the same kind must reach each one.
RETIRED_LAUNCHES = [
    ("dgrad", (2, 1), (False, 128, 1, 1), "f32", ()), ("dgrad", (2, 1), (False, 128, 1, 4), "f32", ()),
    ("dgrad", (2, 1), (False, 16, 1, 1), "f32", ()), ("dgrad", (2, 1), (False, 16, 1, 4), "f32", ()),
    ("dgrad", (2, 1), (False, 16, 2, 1), "f32", ()), ("dgrad", (2, 1), (False, 16, 4, 1), "f32", ()),
    ("dgrad", (2, 1), (False, 32, 1, 1), "f32", (("MNB_PK_COLTILES", "2"),)), ("dgrad", (2, 1), (False, 32, 1, 1), "f32", ()),
    ("dgrad", (2, 1), (False, 64, 1, 4), "f32", ()), ("dgrad", (2, 1), (False, 64, 2, 1), "f32", (("MNB_PK_MT", "2"),)),
    ("dgrad", (2, 1), (False, 64, 2, 4), "f32", ()), ("dgrad", (2, 1), (False, 96, 1, 1), "f32", ()),
    ("dgrad", (2, 1), (True, 128, 1, 1), "f32", ()), ("dgrad", (2, 1), (True, 128, 1, 4), "f32", ()),
    ("dgrad", (2, 1), (True, 16, 1, 1), "f32", ()), ("dgrad", (2, 1), (True, 16, 2, 1), "f32", ()),
    ("dgrad", (2, 1), (True, 48, 1, 1), "f32", ()), ("dgrad", (2, 1), (True, 64, 1, 1), "f32", ()),
    ("dgrad", (2, 1), (True, 64, 2, 1), "f32", ()), ("dgrad", (2, 1), (True, 96, 1, 1), "f32", ()),
    ("dgrad", (2, 2), (True, 64, 1, 1), "f32", (("MNB_PK_SEG_MMAS", "8"),)), ("dgrad", (2, 2), (True, 64, 2, 1), "f32", ()),
    ("dgrad", (2, 2), (True, 64, 2, 4), "f32", ()), ("dgrad", (3, 1), (False, 128, 1, 1), "f32", ()),
    ("dgrad", (3, 1), (False, 16, 1, 1), "f32", ()), ("dgrad", (3, 1), (False, 16, 1, 4), "f32", ()),
    ("dgrad", (3, 1), (False, 64, 1, 4), "f32", ()), ("dgrad", (3, 1), (False, 96, 1, 1), "f32", ()),
    ("dgrad", (3, 1), (True, 128, 1, 1), "f32", ()), ("dgrad", (3, 1), (True, 128, 1, 4), "f32", ()),
    ("dgrad", (3, 1), (True, 16, 1, 1), "f32", ()), ("dgrad", (3, 1), (True, 32, 1, 1), "f32", ()),
    ("dgrad", (3, 1), (True, 48, 1, 1), "f32", ()), ("dgrad", (3, 1), (True, 64, 1, 1), "f32", ()),
    ("dgrad", (3, 1), (True, 64, 1, 4), "f32", ()), ("dgrad", (3, 1), (True, 96, 1, 1), "f32", ()),
    ("fwd", (1, 1), (False, 128, 1, 1), "int", ()), ("fwd", (1, 1), (False, 16, 1, 1), "int", ()),
    ("fwd", (1, 1), (False, 32, 1, 1), "int", (("MNB_PK_COLTILES", "3"),)),
    ("fwd", (1, 1), (False, 32, 1, 1), "int", (("MNB_PK_STAGES", "2"),)),
    ("fwd", (1, 1), (False, 32, 1, 1), "int", (("MNB_PK_STAGES", "4"),)),
    ("fwd", (1, 1), (False, 32, 1, 1), "int", (("MNB_PK_STAGES", "8"),)), ("fwd", (1, 1), (False, 32, 1, 1), "int", ()),
    ("fwd", (1, 1), (False, 32, 2, 1), "int", ()), ("fwd", (1, 1), (False, 32, 4, 1), "int", (("MNB_PK_MT", "4"),)),
    ("fwd", (1, 1), (False, 32, 4, 1), "int", ()), ("fwd", (1, 1), (False, 48, 1, 1), "int", ()),
    ("fwd", (1, 1), (False, 64, 1, 1), "int", ()), ("fwd", (1, 1), (False, 64, 2, 1), "int", (("MNB_PK_MT", "2"),)),
    ("fwd", (1, 1), (False, 96, 1, 1), "int", ()), ("fwd", (3, 3), (False, 128, 1, 1), "f32", ()),
    ("fwd", (3, 3), (False, 32, 1, 1), "f32", ()), ("fwd", (3, 3), (False, 64, 1, 1), "f32", ()),
    ("fwd", (3, 3), (False, 96, 1, 1), "f32", ()), ("fwd", (3, 3), (True, 128, 1, 1), "f32", ()),
    ("fwd", (3, 3), (True, 16, 1, 1), "f32", ()), ("fwd", (3, 3), (True, 32, 1, 1), "f32", ()),
    ("fwd", (3, 3), (True, 32, 4, 1), "f32", (("MNB_PK_MT", "4"),)), ("fwd", (3, 3), (True, 48, 1, 1), "f32", ()),
    ("fwd", (3, 3), (True, 48, 2, 1), "f32", (("MNB_PK_MT", "2"),)),
    ("fwd", (3, 3), (True, 64, 1, 1), "f32", (("MNB_PK_SEG_MMAS", "8"),)),
    ("fwd", (3, 3), (True, 64, 1, 1), "f32", (("MNB_PK_STAGES", "2"),)), ("fwd", (3, 3), (True, 64, 1, 1), "f32", ()),
    ("fwd", (3, 3), (True, 64, 2, 1), "f32", ()), ("fwd", (3, 3), (True, 96, 1, 1), "f32", ()),
    ("i8", (1, 1), (128, 1, False), "int", (("MNB_PK_MT", "1"),)),
    ("i8", (1, 1), (128, 1, False), "int", (("MNB_PK_STAGES", "2"),)),
    ("i8", (1, 1), (128, 1, False), "int", (("MNB_PK_STAGES", "4"),)), ("i8", (1, 1), (128, 1, False), "int", ()),
    ("i8", (1, 1), (128, 1, True), "int", ()), ("i8", (1, 1), (16, 1, False), "int", ()),
    ("i8", (1, 1), (32, 1, False), "int", ()), ("i8", (1, 1), (32, 4, False), "int", (("MNB_PK_MT", "4"),)),
    ("i8", (1, 1), (48, 1, False), "int", ()), ("i8", (1, 1), (64, 1, False), "int", (("MNB_PK_COLTILES", "3"),)),
    ("i8", (1, 1), (64, 1, False), "int", ()), ("i8", (1, 1), (64, 2, False), "int", (("MNB_PK_MT", "2"),)),
    ("i8", (1, 1), (64, 2, False), "int", ()), ("i8", (1, 1), (96, 1, False), "int", ()),
    ("wgrad", (2, 1), (112, False, False), "f32", ()), ("wgrad", (2, 1), (128, False, False), "f32", ()),
    ("wgrad", (2, 1), (16, True, False), "f32", (("MNB_PK_WG_MERGE", "0"),)), ("wgrad", (2, 1), (16, True, False), "f32", ()),
    ("wgrad", (2, 1), (32, True, False), "f32", ()), ("wgrad", (2, 1), (48, True, False), "f32", (("MNB_PK_WG_NC", "48"),)),
    ("wgrad", (2, 1), (48, True, False), "f32", ()), ("wgrad", (2, 1), (64, False, False), "f32", ()),
    ("wgrad", (2, 1), (64, True, False), "f32", (("MNB_PK_WG_CHAIN", "16"),)), ("wgrad", (2, 1), (64, True, False), "f32", ()),
    ("wgrad", (2, 1), (64, True, True), "f32", ()), ("wgrad", (2, 1), (80, False, False), "f32", ()),
    ("wgrad", (2, 1), (96, False, False), "f32", ()), ("wgrad", (2, 2), (112, False, False), "f32", ()),
    ("wgrad", (2, 2), (128, False, False), "f32", ()), ("wgrad", (2, 2), (16, True, False), "f32", ()),
    ("wgrad", (2, 2), (32, True, False), "f32", ()), ("wgrad", (2, 2), (48, True, False), "f32", ()),
    ("wgrad", (2, 2), (64, False, False), "f32", ()), ("wgrad", (2, 2), (64, True, False), "f32", ()),
    ("wgrad", (2, 2), (64, True, True), "f32", ()), ("wgrad", (2, 2), (80, False, False), "f32", ()),
    ("wgrad", (2, 2), (96, False, False), "f32", ()), ("wgrad", (3, 1), (112, False, False), "f32", ()),
    ("wgrad", (3, 1), (128, False, False), "f32", ()), ("wgrad", (3, 1), (16, True, False), "f32", ()),
    ("wgrad", (3, 1), (32, True, False), "f32", ()), ("wgrad", (3, 1), (48, True, False), "f32", ()),
    ("wgrad", (3, 1), (64, False, False), "f32", ()), ("wgrad", (3, 1), (64, True, False), "f32", ()),
    ("wgrad", (3, 1), (64, True, True), "f32", ()), ("wgrad", (3, 1), (80, False, False), "f32", ()),
    ("wgrad", (3, 1), (96, False, False), "f32", ()), ("wgrad", (3, 3), (112, False, False), "f32", ()),
    ("wgrad", (3, 3), (128, False, False), "f32", ()), ("wgrad", (3, 3), (16, True, False), "f32", ()),
    ("wgrad", (3, 3), (32, True, False), "f32", ()), ("wgrad", (3, 3), (48, True, False), "f32", ()),
    ("wgrad", (3, 3), (64, False, False), "f32", ()), ("wgrad", (3, 3), (64, True, False), "f32", ()),
    ("wgrad", (3, 3), (64, True, True), "f32", ()), ("wgrad", (3, 3), (80, False, False), "f32", ()),
    ("wgrad", (3, 3), (96, False, False), "f32", ()),
]


def signature(case, p):
    if case.mode == "wgrad":
        return PU.wgrad_signature(p)
    if case.mode == "i8":
        return PU.i8_signature(p, case.shape[7])
    return PU.conv_signature(p)


def case_signatures(plans):
    """{(mode, terms, plan signature, operand kind)} of the cases"""
    return {(c.mode, c.terms, signature(c, plans[c.id][2]), c.ops) for c in PC.CASES if not c.refuse}


def test_every_retired_launch_is_reached(plans):
    held = case_signatures(plans)
    missing = [r for r in RETIRED_LAUNCHES if r[:4] not in held]
    assert not missing, f"(mode, terms, plan signature, operand kind, knobs) of retired launches no case reaches: {missing}"


def test_every_knob_of_the_retired_launches_is_set_by_a_case():
    want = {k for r in RETIRED_LAUNCHES for k, _ in r[4]}
    missing = sorted(want - {k for c in PC.CASES for k in c.env})
    assert not missing, f"MNB_PK_* knobs no case sets: {missing}"


def _model_signatures():
    """{conv signature: [where]}, {wgrad signature: [where]}, {int8 signature: [where]} of the bench models"""
    conv, wgrad, i8 = {}, {}, {}
    for name, B, Cc, H, W, K, R, st, pad, G in PU.model_convs():
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
        if name.startswith(("res32_", "res224_")):
            p = PU.i8_plan(sh)
            assert p is not None, name
            i8.setdefault(PU.i8_signature(p, st), []).append(name)
    return conv, wgrad, i8


def test_model_signatures_are_reached(plans):
    model = dict(zip(("conv", "wgrad", "i8"), _model_signatures()))
    assert len(model["conv"]) >= 10 and len(model["wgrad"]) >= 5 and len(model["i8"]) >= 3, model
    held = {}
    for mode, terms, sig, _ in case_signatures(plans):
        held.setdefault({"fwd": "conv", "dgrad": "conv"}.get(mode, mode), set()).add(sig)
    missing = {(kind, sig): where[:3] for kind, sigs in model.items()
               for sig, where in sigs.items() if sig not in held[kind]}
    assert not missing, f"plan signatures of the bench models no case reaches (conv: segmented, Nt, MT, ny; wgrad: Nc, " \
                        f"tpg > 1, gm > 1; i8: Nt, MT, phase split): {missing}"


def test_plan_query_agrees_with_the_16_field_query():
    """mnb_pk_conv_plan is mnb_pk_conv_plan_ex's first 16 fields; the wgrad query agrees with the scratch size"""
    from micronet_b200 import _lib as L
    lib = L.load()
    for name, B, Cc, H, W, K, R, st, pad, G in PU.model_convs()[::3]:
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


def test_7x7_stride2_dgrad_is_refused_and_routed_to_the_generic_kernels():
    """the data gradient at (2, 1) of this shape needs an MMA program over 512 words: the query refuses it, so the layer's
    forward never commits it to the packed family (the launch in its backward would refuse)"""
    from types import SimpleNamespace
    from micronet_b200 import _lib as L, functional as F, pk as PK
    sh = shape((1, 16, 2, 2, 96, 7, 7, 2, 3, 3, 1))
    assert PK.supported(sh, 0, 1, 1)
    assert not PK.supported(sh, 1, 2, 1)
    rc, text, _ = query("dgrad", sh, (2, 1))
    assert rc == L.E_UNSUPPORTED and b"MMA program longer than 512 entries" in text
    assert fake_launch("dgrad", sh, (2, 1)) == (rc, text)
    # QuantConv2dFn's forward asks _pk_forward first; it declines the layer before touching any tensor (the backward's data
    # gradient is outside the cover), and the forward takes the next family.  Integer weights, a DoReFa activation.
    assert L.PK_TERMS_BWD == 2
    ctx = SimpleNamespace(needs_input_grad=(True, True, False))
    spec = SimpleNamespace(mode=L.ACT_DOREFA, q_type=0, bits=4)
    assert F._pk_forward(ctx, None, None, None, object(), None, spec, sh, None) is False
    assert not hasattr(ctx, "pk_x")


def test_every_bench_launch_is_a_case():
    """every launch the bench workloads send to mnb_pk_conv / mnb_pk_wgrad (tests/pk_conv_bench_launches.py, at the bench
    batch) is a case, and the table accounts for every conv of the bench models: each one's forward is a recorded launch,
    or a recorded consumer-plane launch, or is taken by gc3 (pk.gc3_plan), or runs on another family (the fp32 stems)"""
    from micronet_b200 import pk as PK
    from tests.pk_conv_bench_launches import BENCH_LAUNCHES, POST_LAUNCHES
    held = {(c.shape, {"fwd": 0, "dgrad": 1, "wgrad": 2}[c.mode], c.terms) for c in PC.CASES if c.bench}
    missing = []
    for wl, fn, sh, mode, ta, tw in BENCH_LAUNCHES:
        B, Cc, H, W, K, R, S, st, _, ph, pw, dil, _, G = sh
        if ((B, Cc, H, W, K, R, S, st, ph, pw, G), mode, (ta, tw)) not in held:
            missing.append((wl, sh, mode, ta, tw))
    assert not missing, f"bench launches no case holds: {missing}"
    fwd_shapes = {tuple(sh) for wl, fn, sh, mode, ta, tw in BENCH_LAUNCHES + POST_LAUNCHES if mode == 0}
    unaccounted = []
    for name, B, Cc, H, W, K, R, st, pad, G in PU.model_convs():
        sh = PU.shape(B, Cc, H, W, K, R, st, pad, G)
        if PK._key(sh) in fwd_shapes or PK.gc3_plan(sh, 0, 1, 1) is not None or Cc == 3:
            continue
        unaccounted.append(name)
    assert not unaccounted, f"bench-model convs with no recorded packed-operand forward: {unaccounted}"
