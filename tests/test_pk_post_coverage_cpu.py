"""Coverage of the consumer-plane epilogues by tests/test_gpu_pk_post.py, checked on the host (no GPU needed).

mnb_pk_conv_post_plan runs the launcher's own route (conv_route in csrc/mnb_pk.cu): the epilogue path - the instance row
of pk_conv_kernel - and the plan.  This test requires

* every pinned plan of tests/pk_post_cases.py to hold, and every case to take the path it names;
* every (epilogue path, N tile) instance, every option and plan feature to be reached by some case, with several work
  items per CTA on every path and consecutive items of a CTA on different N tiles and groups;
* every refusal reason the host can reach to be listed, with the code and text of the query;
* every linked conv of the frozen graphs at the batch the benchmark runs them to be a case,

so deleting a case, or a change of the plan heuristics that moves a case elsewhere, fails here naming what lost its cover.
mnb_pk_conv_post also refuses a segmented producer plan on the host, before launching."""
import pytest

from tests import pk_post_cases as P
from tests import pk_plan_util as PU

E_ARG = -1


@pytest.fixture(scope="module")
def plans():
    out = {}
    for c in P.ALL_CASES:
        with PU.env(c.env):
            out[c.id] = P.plan_of(c)
    return out


def test_case_ids_are_unique():
    ids = [c.id for c in P.ALL_CASES] + [r.id for r in P.REFUSALS]
    assert len(ids) == len(set(ids))


def test_pinned_plans_hold(plans):
    bad = {}
    for c in P.ALL_CASES:
        p = plans[c.id]
        if not isinstance(p, dict):
            bad[c.id] = p
            continue
        got = {k: p[k] for k in c.expect}
        if got != c.expect or p["path"] != P.PATHS[c.path] or p["ny"] != 1 or p["segmented"]:
            bad[c.id] = (got, c.expect, p)
    assert not bad, f"plans changed or refused: {bad}"


def test_every_instance_is_launched(plans):
    got = {(p["path"], p["Nt"]) for p in plans.values() if isinstance(p, dict)}
    want = {(P.PATHS[path], nt) for path in P.PATHS for nt in P.NT}
    names = {v: k for k, v in P.PATHS.items()}
    missing = sorted((names[a], nt) for a, nt in want - got)
    assert not missing, f"(epilogue path, Nt) instances no case launches: {missing}"


def _features(c, p):
    B, Cc, H, W, K, R, st, pad, G = c.shape
    f = {"relu" if c.relu else "no_relu", "out" if c.out else "plane_only"}
    if p["n_ntiles"] * p["Nt"] > K // G:
        f.add("partial_n_tile")
    if K % 8:
        f.add("k_mod8")
    if p["n_mtiles"] % p["MT"]:
        f.add("partial_m_group")
    if p["MT"] > 1:
        f.add("mt>1")
    if p["col_tiles"] > 1:
        f.add("col_tiles>1")
    if st == 2:
        f.add("stride2_producer")
    if c.split:
        f.add("phase_split")
    if G > 1:
        f.add("grouped")
    if c.bn:
        f.add("bn")
        if not c.relu:
            f.add("bn_no_relu")
    if c.sg > 1:
        f.add("shuffle")
        if G > 1:
            f.add("grouped_shuffle")
    if c.q:
        f.add(f"q_{c.q}")
    if c.terms:
        f.add(f"terms{c.terms}")
    if c.ta > 1:
        f.add(f"ta{c.ta}")
    seq = P.items_of_cta(p, G)
    if p["n_items"] > p["gx"]:
        f.add("multi_item")
        if len({nt for nt, _ in seq}) > 1 and len({g for _, g in seq}) > 1 and \
                all(a[0] != b[0] and a[1] != b[1] for a, b in zip(seq, seq[1:])):
            f.add("multi_item_new_tile_and_group")
    return f


# what every path must reach; the quantizers of the level paths between them
WANT = {
    "levels": {"partial_n_tile", "k_mod8", "partial_m_group", "col_tiles>1", "stride2_producer", "phase_split", "grouped",
               "multi_item_new_tile_and_group", "relu", "no_relu", "out", "plane_only"},
    "levels_i8": {"partial_n_tile", "k_mod8", "partial_m_group", "col_tiles>1", "stride2_producer", "phase_split", "grouped",
                  "multi_item_new_tile_and_group", "relu", "no_relu", "out", "plane_only"},
    "xpost": {"partial_n_tile", "k_mod8", "partial_m_group", "col_tiles>1", "stride2_producer", "phase_split", "grouped", "bn",
              "bn_no_relu", "shuffle", "grouped_shuffle", "multi_item_new_tile_and_group", "relu", "no_relu", "out", "plane_only"},
    "xpost_i8": {"partial_n_tile", "k_mod8", "partial_m_group", "col_tiles>1", "stride2_producer", "phase_split", "grouped",
                 "bn", "bn_no_relu", "shuffle", "grouped_shuffle", "multi_item_new_tile_and_group", "relu", "no_relu", "out", "plane_only"},
    "terms": {"partial_n_tile", "partial_m_group", "col_tiles>1", "stride2_producer", "phase_split", "grouped", "bn", "bn_no_relu",
              "shuffle", "grouped_shuffle", "multi_item_new_tile_and_group", "relu", "no_relu", "out", "plane_only", "terms1", "terms2",
              "terms3", "ta3"},
}
QUANTIZERS = {"levels": {"dorefa2", "dorefa4", "dorefa8", "iao8", "iao4", "iao8a"},
              "xpost": {"dorefa2", "dorefa4", "dorefa8", "iao8", "iao4", "iao8a"},
              "levels_i8": {"dorefa2", "dorefa4", "dorefa7", "iao8", "iao4"},
              "xpost_i8": {"dorefa2", "dorefa4", "dorefa7", "iao8", "iao4"}}


def test_every_option_is_covered(plans):
    missing = {}
    for path, want in WANT.items():
        got = set()
        for c in P.CASES:
            if c.path == path:
                got |= _features(c, plans[c.id])
        want = want | {f"q_{q}" for q in QUANTIZERS.get(path, ())}
        if want - got:
            missing[path] = sorted(want - got)
    assert not missing, f"options no case of the path reaches: {missing}"


def test_forward_plans_run_one_output_phase():
    """the unreachable instance feature: a consumer is forward-only, and no forward plan runs several output phases (ny = 4
    is the data gradient of a stride-2 conv), so the epilogue never stores at phase y > 0"""
    n = 0
    for B in (1, 3, 64):
        for Cc, K in ((16, 16), (64, 128), (96, 40), (256, 512)):
            for H in (6, 8, 14, 32, 56):
                for R, st, pad in ((1, 1, 0), (3, 1, 1), (3, 2, 1), (1, 2, 0), (5, 1, 2)):
                    for G in (1, 2, 8):
                        if Cc % G or K % G:
                            continue
                        for cpu in (8, 16):
                            p = P.query((B, Cc, H, H, K, R, st, pad, G), cpu, 1, None)
                            if isinstance(p, dict):
                                assert p["ny"] == 1, (B, Cc, H, K, R, st, G, cpu, p)
                                n += 1
    assert n > 500, n


def test_every_refusal_reason_is_listed_and_agrees_with_the_launcher_text():
    codes = {"E_ARG": E_ARG, "E_UNSUPPORTED": -2}
    bad = {}
    for r in P.REFUSALS:
        post, _ = P.host_post(r.opts)
        got = P.query(r.shape, r.cpu, r.ta, post)
        if not isinstance(got, tuple) or got[0] != codes[r.code] or r.text not in got[1]:
            bad[r.id] = got
    assert not bad, bad
    # the refusal reasons of conv_route a consumer can reach, one listed shape each; a reason with two variants (bf16 and int8
    # plane, quantizer, grouped or not) needs both
    def key(r, text):
        return (text, r.cpu, r.shape[8] > 1, r.opts.get("q"))
    reasons = {("all four", 8, False, "iao8"), ("% 4 == 0", 8, False, "iao8"), ("do not divide", 8, False, "iao8"),
               ("channel shuffle in front of a stride-2 consumer", 8, False, "iao8"), ("channels per unit", 8, False, "iao8"),
               ("channels per unit", 16, False, "iao8"), ("int8 plane needs", 16, False, "dorefa8"),
               ("int8 plane needs", 16, False, "iao8a"), ("int8 consumer plane of a grouped conv", 16, True, "iao8"),
               ("fused consumer of a grouped conv", 8, True, "iao8"), ("term planes need", 8, False, None),
               ("term planes need", 8, True, None), ("term planes (1..3)", 8, False, None), ("odd-sized", 8, False, "iao8"),
               ("segmented", 8, False, "iao8"), ("DoReFa or IAO", 8, False, "sign"), ("2..8 bits", 8, False, "dorefa9"),
               ("terms_out without one", 8, False, "iao8")}
    got = set()
    for r in P.REFUSALS:
        text = P.query(r.shape, r.cpu, r.ta, P.host_post(r.opts)[0])[1]
        got |= {k for k in reasons if k[0] in text and k == key(r, k[0])}
    missing = sorted(reasons - got, key=str)
    assert not missing, f"refusal reasons no listed shape reaches: {missing}"


def test_query_without_consumer_is_the_plain_plan():
    """post NULL: the plain / int8 instance row and the plan of mnb_pk_conv_plan_ex / mnb_pk_i8_conv_plan"""
    from tests import pk_plan_util as PU
    for shape in ((2, 16, 8, 8, 16, 3, 1, 1, 1), (4, 64, 16, 16, 128, 3, 1, 1, 1), (8, 64, 32, 32, 128, 3, 2, 1, 1)):
        sh = PU.shape(*shape)
        for ta in (1, 2):
            p, q = P.query(shape, 8, ta, None), PU.conv_plan(sh, 0, ta, 1)
            assert p["path"] == (1 if q["segmented"] else 0)
            assert all(p[k] == q[k] for k in ("Nt", "MT", "n_mtiles", "n_items", "ny", "col_tiles", "n_ntiles", "segmented"))
        p = P.query(shape, 16, 1, None)
        assert p["path"] == 2
    assert P.query((2, 16, 8, 8, 16, 1, 1, 0, 1), 12, 1, None)[0] == E_ARG


@pytest.fixture(scope="module")
def links():
    from tests import pk_post_links as K
    return K.linked_convs()


def test_every_recorded_link_is_a_case(links, plans):
    """every conv that freeze_inference links to its consumer, at the graph's bench batch, is a case with the same shape,
    epilogue path and consumer options (shuffle, BatchNorm, phase split, ReLU, quantizer, term planes), and the case lists it"""
    from tests import pk_post_links as K
    graphs = {g for g, _ in links}
    assert graphs >= {"resnet18_iao_ptq_224", "resnet18_iao_ptq_224_int8", "nin_iao", "nin_gc_iao", "nin_gc_iao_int8",
                      "nin_dorefa_w8a8", "nin_gc_dorefa_w4a4", "nin_wbwtab_a32"}, sorted(graphs)
    by_link = {}
    for c in P.MODEL_CASES:
        for who in c.model:
            by_link[who] = c
    missing, wrong = [], {}
    for key, (shape, path, opts) in links.items():
        c = by_link.get(key)
        if c is None:
            missing.append((key, shape, path, opts))
        elif (tuple(c.shape), c.path, K.case_options(c)) != (tuple(shape), path, opts) or plans[c.id]["path"] != P.PATHS[path]:
            wrong[key] = ((c.id, c.shape, c.path, K.case_options(c)), (shape, path, opts))
    stale = sorted(set(by_link) - set(links))
    assert not missing and not wrong and not stale, \
        f"links no case runs: {missing}; cases that differ from their link: {wrong}; cases of links that no longer exist: {stale}"


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
