"""Pinned cases of the packed-operand convolutions' consumer-plane epilogues (csrc/mnb_pk.cu, mnb_pk_conv_post and
mnb_pk_i8_conv with a consumer), shared by tests/test_pk_post_coverage_cpu.py (host: plans, instances, options, refusals)
and tests/test_gpu_pk_post.py (device: every case against a host reference of the epilogue's fp32 op sequence).

The epilogue path of a launch is the instance row conv_route picks (mnb_pk_conv_post_plan, out[0]):

    levels    0  bf16 level plane: scale + bias [-> ReLU] -> consumer quantizer
    levels_i8 2  the same into an int8 plane (s8 operands, s32 sums)
    xpost     3  bf16 level plane behind an eval BatchNorm and / or a channel shuffle
    xpost_i8  4  the same into an int8 plane
    terms     5  bf16 term planes: [BatchNorm] [ReLU] [shuffle] and the value's exact split into 1..3 bf16 pieces

Each path is compiled for the six N tiles (Nt 16 .. 128): 30 instances, every one of them reachable.  Not reachable: a
producer with several output phases (ny = 4).  Only the data gradient of a stride-2 conv runs four phases, and a consumer
is a forward-only option (mnb_pk_conv_post is mode 0); a stride-2 producer runs ny = 1 with four k-phases of its input.
test_pk_post_coverage_cpu.py sweeps forward shapes to show that.

A case: shape (B, C, H, W, K, R, stride, pad, groups); path; q the consumer quantizer (dorefa<bits>, iao<bits> symmetric,
iao8a asymmetric with a zero point; None for term planes); relu; split (the consumer is a stride-2 conv: phase-split
plane); bn (eval BatchNorm in front); sg (shuffle groups); terms (term planes written); ta (activation pieces of the
producer: the frozen wbwtab graphs read 3); out (fp32 y kept, or NULL); env (MNB_PK_* knobs); expect (the plan fields
the case is pinned to); model (the frozen graph conv it stands for, at that graph's batch)."""
from collections import namedtuple

Case = namedtuple("Case", "id shape path q relu split bn sg terms ta out env expect model",
                  defaults=(True, False, False, 1, 0, 1, True, {}, {}, None))

PATHS = {"levels": 0, "levels_i8": 2, "xpost": 3, "xpost_i8": 4, "terms": 5}
I8_PATHS = ("levels_i8", "xpost_i8")
NT = (16, 32, 48, 64, 96, 128)
# fields of mnb_pk_conv_post_plan
PLAN_FIELDS = "path Nt MT n_mtiles n_items ny col_tiles n_ntiles gx segmented".split()


def _c(id, shape, path, q, expect, **kw):
    return Case(id, shape, path, q, expect=expect, **kw)


CASES = [
    # ---- bf16 level plane (path 0), one case per N tile
    _c("lv16_dorefa4", (2, 16, 8, 8, 16, 3, 1, 1, 1), "levels", "dorefa4",
       dict(Nt=16, MT=1, n_mtiles=2, n_items=2, col_tiles=1, n_ntiles=1)),
    _c("lv32_s2_split_iao8", (2, 16, 16, 16, 32, 3, 2, 1, 1), "levels", "iao8",
       dict(Nt=32, MT=1, n_mtiles=2, n_items=2, col_tiles=1, n_ntiles=1), relu=False, split=True, out=False),
    _c("lv48_partial_iao8a", (2, 24, 8, 8, 40, 1, 1, 0, 1), "levels", "iao8a",
       dict(Nt=48, MT=1, n_mtiles=1, n_items=1, col_tiles=1, n_ntiles=1)),
    _c("lv64_g2_dorefa8", (2, 32, 8, 8, 128, 3, 1, 1, 2), "levels", "dorefa8",
       dict(Nt=64, MT=1, n_mtiles=2, n_items=4, col_tiles=1, n_ntiles=1)),
    _c("lv96_k90_iao4", (2, 16, 8, 8, 90, 3, 1, 1, 1), "levels", "iao4",
       dict(Nt=96, MT=1, n_mtiles=2, n_items=2, col_tiles=1, n_ntiles=1), out=False),
    _c("lv128_cols2_dorefa2", (2, 16, 8, 40, 128, 3, 1, 1, 1), "levels", "dorefa2",
       dict(Nt=128, MT=1, col_tiles=2, n_ntiles=1), env={"MNB_PK_COLTILES": "2"}),
    _c("lv64_mt2_partial_iao8", (3, 16, 28, 28, 64, 3, 1, 1, 1), "levels", "iao8",
       dict(Nt=64, MT=2, n_mtiles=21, n_items=11), env={"MNB_PK_MT": "2"}),
    _c("lv_multi_g3_dorefa4", (6, 48, 16, 16, 1560, 1, 1, 0, 3), "levels", "dorefa4",
       dict(Nt=128, MT=1, n_ntiles=5, n_items=180, gx=132)),
    # ---- int8 level plane (path 2)
    _c("i8_16_iao8", (2, 32, 8, 8, 16, 3, 1, 1, 1), "levels_i8", "iao8",
       dict(Nt=16, MT=1, n_mtiles=2, n_items=2, n_ntiles=1)),
    _c("i8_32_s2_split_dorefa4", (2, 32, 16, 16, 32, 3, 2, 1, 1), "levels_i8", "dorefa4",
       dict(Nt=32, MT=1, n_mtiles=2, n_items=2), split=True),
    _c("i8_48_partial_iao4", (2, 32, 8, 8, 40, 1, 1, 0, 1), "levels_i8", "iao4",
       dict(Nt=48, MT=1, n_items=1), out=False),
    _c("i8_64_g2_dorefa7", (2, 64, 8, 8, 128, 3, 1, 1, 2), "levels_i8", "dorefa7",
       dict(Nt=64, MT=1, n_mtiles=2, n_items=4)),
    _c("i8_96_k90_iao8", (2, 32, 8, 8, 90, 3, 1, 1, 1), "levels_i8", "iao8",
       dict(Nt=96, MT=1, n_items=2), relu=False),
    _c("i8_128_cols2_dorefa2", (2, 32, 8, 40, 128, 3, 1, 1, 1), "levels_i8", "dorefa2",
       dict(Nt=128, col_tiles=2), env={"MNB_PK_COLTILES": "2"}),
    _c("i8_64_mt2_partial_iao8", (3, 32, 28, 28, 64, 3, 1, 1, 1), "levels_i8", "iao8",
       dict(Nt=64, MT=2, n_mtiles=21, n_items=11), env={"MNB_PK_MT": "2"}),
    _c("i8_multi_g3_iao8", (6, 48, 16, 16, 1584, 1, 1, 0, 3), "levels_i8", "iao8",
       dict(Nt=128, MT=1, n_ntiles=5, n_items=180, gx=132)),
    # ---- bf16 level plane behind BatchNorm / shuffle (path 3)
    _c("xp16_bn_dorefa4", (2, 16, 8, 8, 16, 3, 1, 1, 1), "xpost", "dorefa4", dict(Nt=16, n_items=2), bn=True),
    _c("xp32_sg2_iao8", (2, 16, 8, 8, 32, 1, 1, 0, 1), "xpost", "iao8", dict(Nt=32, n_items=1), sg=2, out=False),
    _c("xp48_bn_partial_iao8a", (2, 16, 8, 8, 44, 3, 1, 1, 1), "xpost", "iao8a", dict(Nt=48, n_items=2), bn=True),
    _c("xp64_g2_bn_sg4_dorefa8", (2, 32, 8, 8, 128, 1, 1, 0, 2), "xpost", "dorefa8", dict(Nt=64, n_items=2), bn=True, sg=4),
    _c("xp96_bn_split_iao4", (2, 16, 16, 16, 92, 3, 2, 1, 1), "xpost", "iao4", dict(Nt=96, n_items=2), bn=True, split=True,
       relu=False),
    _c("xp128_bn_sg16_dorefa2", (2, 16, 8, 40, 128, 1, 1, 0, 1), "xpost", "dorefa2", dict(Nt=128, col_tiles=2), bn=True, sg=16,
       env={"MNB_PK_COLTILES": "2"}),
    _c("xp64_mt2_partial_bn_iao8", (3, 16, 28, 28, 64, 3, 1, 1, 1), "xpost", "iao8",
       dict(Nt=64, MT=2, n_mtiles=21, n_items=11), bn=True, env={"MNB_PK_MT": "2"}),
    _c("xp_multi_g3_bn_sg4_dorefa4", (6, 48, 16, 16, 1560, 1, 1, 0, 3), "xpost", "dorefa4",
       dict(Nt=128, n_ntiles=5, n_items=180, gx=132), bn=True, sg=4),
    # ---- int8 level plane behind BatchNorm / shuffle (path 4)
    _c("xi16_bn_iao8", (2, 32, 8, 8, 16, 3, 1, 1, 1), "xpost_i8", "iao8", dict(Nt=16, n_items=2), bn=True),
    _c("xi32_sg2_dorefa4", (2, 32, 8, 8, 32, 1, 1, 0, 1), "xpost_i8", "dorefa4", dict(Nt=32, n_items=1), sg=2),
    _c("xi48_bn_partial_iao4", (2, 32, 8, 8, 44, 1, 1, 0, 1), "xpost_i8", "iao4", dict(Nt=48, n_items=1), bn=True, out=False),
    _c("xi64_g2_bn_sg4_dorefa7", (2, 64, 8, 8, 128, 1, 1, 0, 2), "xpost_i8", "dorefa7", dict(Nt=64, n_items=2), bn=True, sg=4),
    _c("xi96_bn_split_iao8", (2, 32, 16, 16, 92, 3, 2, 1, 1), "xpost_i8", "iao8", dict(Nt=96, n_items=2), bn=True, split=True),
    _c("xi128_bn_sg8_dorefa2", (2, 32, 8, 40, 128, 1, 1, 0, 1), "xpost_i8", "dorefa2", dict(Nt=128, col_tiles=2), bn=True,
       sg=8, relu=False, env={"MNB_PK_COLTILES": "2"}),
    _c("xi64_mt2_partial_sg4_iao8", (3, 32, 28, 28, 64, 3, 1, 1, 1), "xpost_i8", "iao8",
       dict(Nt=64, MT=2, n_mtiles=21, n_items=11), sg=4, env={"MNB_PK_MT": "2"}),
    _c("xi_multi_g3_bn_sg4_iao8", (6, 48, 16, 16, 1584, 1, 1, 0, 3), "xpost_i8", "iao8",
       dict(Nt=128, n_ntiles=5, n_items=180, gx=132), bn=True, sg=4),
    # ---- term planes (path 5)
    _c("tm16_t3_bn", (2, 16, 8, 8, 16, 3, 1, 1, 1), "terms", None, dict(Nt=16, n_items=2), bn=True, terms=3),
    _c("tm32_t1_bn_sg2", (2, 16, 8, 8, 32, 1, 1, 0, 1), "terms", None, dict(Nt=32, n_items=1), bn=True, sg=2, terms=1,
       out=False),
    _c("tm48_t2_partial", (2, 16, 8, 8, 40, 1, 1, 0, 1), "terms", None, dict(Nt=48, n_items=1), terms=2, relu=False),
    _c("tm64_g2_bn_sg4_t3", (2, 32, 8, 8, 128, 1, 1, 0, 2), "terms", None, dict(Nt=64, n_items=2), bn=True, sg=4, terms=3,
       relu=False),
    _c("tm96_bn_split_t3", (2, 16, 16, 16, 88, 3, 2, 1, 1), "terms", None, dict(Nt=96, n_items=2), bn=True, split=True, terms=3),
    _c("tm128_cols2_t3_ta3", (2, 16, 8, 40, 128, 3, 1, 1, 1), "terms", None, dict(Nt=128, col_tiles=2), terms=3, ta=3,
       env={"MNB_PK_COLTILES": "2"}),
    _c("tm64_mt2_partial_t2", (3, 16, 28, 28, 64, 3, 1, 1, 1), "terms", None, dict(Nt=64, MT=2, n_mtiles=21, n_items=11),
       bn=True, terms=2, env={"MNB_PK_MT": "2"}),
    _c("tm_multi_g3_bn_sg4_t3", (6, 48, 16, 16, 1560, 1, 1, 0, 3), "terms", None,
       dict(Nt=128, n_ntiles=5, n_items=180, gx=132), bn=True, sg=4, terms=3),
]

# ---- every linked conv of the frozen graphs at the batch the benchmark runs them, one case per distinct (shape, path,
# consumer options); ``model`` lists the (graph, conv) links it stands for.  tests/pk_post_links.py derives the links from
# freeze_inference's link planning on CPU models, and test_pk_post_coverage_cpu.py requires each of them to be a case here.
def _m(id, shape, path, q, expect, model, **kw):
    return Case(id, shape, path, q, out=False, expect=expect, model=tuple(model), **kw)


MODEL_CASES = [
    _m("m_nin_df_192x32_160_1x1", (256, 192, 32, 32, 160, 1, 1, 0, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=2),
       [('nin_dorefa_w8a8', 'model.1.conv')], bn=True),
    _m("m_nin_df_160x32_96_1x1", (256, 160, 32, 32, 96, 1, 1, 0, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_dorefa_w8a8', 'model.2.conv')], bn=True),
    _m("m_nin_df_96x16_192_5x5", (256, 96, 16, 16, 192, 5, 1, 2, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=768, n_items=1536, col_tiles=1, n_ntiles=2),
       [('nin_dorefa_w8a8', 'model.4.conv')], bn=True),
    _m("m_nin_df_192x16_192_1x1", (256, 192, 16, 16, 192, 1, 1, 0, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=512, n_items=1024, col_tiles=1, n_ntiles=2),
       [('nin_dorefa_w8a8', 'model.5.conv'), ('nin_dorefa_w8a8', 'model.6.conv')], bn=True),
    _m("m_nin_df_192x8_192_3x3", (256, 192, 8, 8, 192, 3, 1, 1, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=256, n_items=512, col_tiles=1, n_ntiles=2),
       [('nin_dorefa_w8a8', 'model.8.conv')], bn=True),
    _m("m_nin_df_192x8_192_1x1", (256, 192, 8, 8, 192, 1, 1, 0, 1), "xpost", 'dorefa8', dict(Nt=96, MT=1, n_mtiles=128, n_items=256, col_tiles=1, n_ntiles=2),
       [('nin_dorefa_w8a8', 'model.9.conv')], bn=True),
    _m("m_gc_df_256x32_256_1x1g2_sg2", (256, 256, 32, 32, 256, 1, 1, 0, 2), "xpost", 'dorefa4', dict(Nt=128, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=1),
       [('nin_gc_dorefa_w4a4', 'model.1.conv'), ('nin_gc_dorefa_w4a4', 'model.2.conv')], bn=True, sg=2),
    _m("m_gc_df_256x16_512_3x3g16_sg16", (256, 256, 16, 16, 512, 3, 1, 1, 16), "xpost", 'dorefa4', dict(Nt=32, MT=4, n_mtiles=768, n_items=3072, col_tiles=1, n_ntiles=1),
       [('nin_gc_dorefa_w4a4', 'model.4.conv')], bn=True, sg=16),
    _m("m_gc_df_512x16_512_1x1g4_sg4", (256, 512, 16, 16, 512, 1, 1, 0, 4), "xpost", 'dorefa4', dict(Nt=128, MT=1, n_mtiles=512, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_gc_dorefa_w4a4', 'model.5.conv'), ('nin_gc_dorefa_w4a4', 'model.6.conv')], bn=True, sg=4),
    _m("m_gc_df_512x8_1024_3x3g32_sg32", (256, 512, 8, 8, 1024, 3, 1, 1, 32), "xpost", 'dorefa4', dict(Nt=32, MT=4, n_mtiles=256, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_gc_dorefa_w4a4', 'model.8.conv')], bn=True, sg=32),
    _m("m_gc_df_1024x8_1024_1x1g8", (256, 1024, 8, 8, 1024, 1, 1, 0, 8), "xpost", 'dorefa4', dict(Nt=128, MT=1, n_mtiles=128, n_items=1024, col_tiles=1, n_ntiles=1),
       [('nin_gc_dorefa_w4a4', 'model.9.conv')], bn=True),
    _m("m_gc_iao_3x32_256_5x5", (256, 3, 32, 32, 256, 5, 1, 2, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=2816, n_items=5632, col_tiles=1, n_ntiles=2),
       [('nin_gc_iao', 'model.0.conv')]),
    _m("m_gc_iao_1024x8_1024_1x1g8", (256, 1024, 8, 8, 1024, 1, 1, 0, 8), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=128, n_items=1024, col_tiles=1, n_ntiles=1),
       [('nin_gc_iao', 'model.9.conv')]),
    _m("m_gc_iao_i8_3x32_256_5x5", (256, 3, 32, 32, 256, 5, 1, 2, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=2816, n_items=5632, col_tiles=1, n_ntiles=2),
       [('nin_gc_iao_int8', 'model.0.conv')]),
    _m("m_gc_iao_i8_256x32_256_1x1g2_sg2", (256, 256, 32, 32, 256, 1, 1, 0, 2), "xpost_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=1),
       [('nin_gc_iao_int8', 'model.2.conv')], sg=2),
    _m("m_gc_iao_i8_512x16_512_1x1g4_sg4", (256, 512, 16, 16, 512, 1, 1, 0, 4), "xpost_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=512, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_gc_iao_int8', 'model.6.conv')], sg=4),
    _m("m_gc_iao_i8_1024x8_1024_1x1g8", (256, 1024, 8, 8, 1024, 1, 1, 0, 8), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=128, n_items=1024, col_tiles=1, n_ntiles=1),
       [('nin_gc_iao_int8', 'model.9.conv')]),
    _m("m_nin_iao_3x32_192_5x5", (256, 3, 32, 32, 192, 5, 1, 2, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=2816, n_items=5632, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.0.conv')]),
    _m("m_nin_iao_192x32_160_1x1", (256, 192, 32, 32, 160, 1, 1, 0, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.1.conv')]),
    _m("m_nin_iao_160x32_96_1x1", (256, 160, 32, 32, 96, 1, 1, 0, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_iao', 'model.2.conv')]),
    _m("m_nin_iao_96x16_192_5x5", (256, 96, 16, 16, 192, 5, 1, 2, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=768, n_items=1536, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.4.conv')]),
    _m("m_nin_iao_192x16_192_1x1", (256, 192, 16, 16, 192, 1, 1, 0, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=512, n_items=1024, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.5.conv'), ('nin_iao', 'model.6.conv')]),
    _m("m_nin_iao_192x8_192_3x3", (256, 192, 8, 8, 192, 3, 1, 1, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=256, n_items=512, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.8.conv')]),
    _m("m_nin_iao_192x8_192_1x1", (256, 192, 8, 8, 192, 1, 1, 0, 1), "levels", 'iao8', dict(Nt=96, MT=1, n_mtiles=128, n_items=256, col_tiles=1, n_ntiles=2),
       [('nin_iao', 'model.9.conv')]),
    _m("m_nin_iao_i8_3x32_192_5x5", (256, 3, 32, 32, 192, 5, 1, 2, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=2816, n_items=5632, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.0.conv')]),
    _m("m_nin_iao_i8_192x32_160_1x1", (256, 192, 32, 32, 160, 1, 1, 0, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.1.conv')]),
    _m("m_nin_iao_i8_160x32_96_1x1", (256, 160, 32, 32, 96, 1, 1, 0, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=2048, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_iao_int8', 'model.2.conv')]),
    _m("m_nin_iao_i8_96x16_192_5x5", (256, 96, 16, 16, 192, 5, 1, 2, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=768, n_items=1536, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.4.conv')]),
    _m("m_nin_iao_i8_192x16_192_1x1", (256, 192, 16, 16, 192, 1, 1, 0, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=512, n_items=1024, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.5.conv'), ('nin_iao_int8', 'model.6.conv')]),
    _m("m_nin_iao_i8_192x8_192_3x3", (256, 192, 8, 8, 192, 3, 1, 1, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=256, n_items=512, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.8.conv')]),
    _m("m_nin_iao_i8_192x8_192_1x1", (256, 192, 8, 8, 192, 1, 1, 0, 1), "levels_i8", 'iao8', dict(Nt=96, MT=1, n_mtiles=128, n_items=256, col_tiles=1, n_ntiles=2),
       [('nin_iao_int8', 'model.9.conv')]),
    _m("m_nin_a32_192x32_160_1x1", (256, 192, 32, 32, 160, 1, 1, 0, 1), "terms", None, dict(Nt=96, MT=1, n_mtiles=2048, n_items=4096, col_tiles=1, n_ntiles=2),
       [('nin_wbwtab_a32', 'model.1.conv')], bn=True, terms=3, ta=3),
    _m("m_nin_a32_160x32_96_1x1", (256, 160, 32, 32, 96, 1, 1, 0, 1), "terms", None, dict(Nt=96, MT=1, n_mtiles=2048, n_items=2048, col_tiles=1, n_ntiles=1),
       [('nin_wbwtab_a32', 'model.2.conv')], bn=True, terms=3, ta=3),
    _m("m_nin_a32_192x16_192_1x1", (256, 192, 16, 16, 192, 1, 1, 0, 1), "terms", None, dict(Nt=96, MT=1, n_mtiles=512, n_items=1024, col_tiles=1, n_ntiles=2),
       [('nin_wbwtab_a32', 'model.5.conv'), ('nin_wbwtab_a32', 'model.6.conv')], bn=True, terms=3, ta=3),
    _m("m_r18_64x224_64_3x3", (64, 64, 224, 224, 64, 3, 1, 1, 1), "levels", 'iao8', dict(Nt=64, MT=2, n_mtiles=28672, n_items=14336, col_tiles=8, n_ntiles=1),
       [('resnet18_iao_ptq_224', 'conv2_x.0.residual_function.0'), ('resnet18_iao_ptq_224', 'conv2_x.1.residual_function.0')]),
    _m("m_r18_64x224_128_3x3s2", (64, 64, 224, 224, 128, 3, 2, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=7168, n_items=7168, col_tiles=2, n_ntiles=1),
       [('resnet18_iao_ptq_224', 'conv3_x.0.residual_function.0')]),
    _m("m_r18_128x112_128_3x3", (64, 128, 112, 112, 128, 3, 1, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=7168, n_items=7168, col_tiles=4, n_ntiles=1),
       [('resnet18_iao_ptq_224', 'conv3_x.1.residual_function.0')]),
    _m("m_r18_128x112_256_3x3s2", (64, 128, 112, 112, 256, 3, 2, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=1792, n_items=3584, col_tiles=1, n_ntiles=2),
       [('resnet18_iao_ptq_224', 'conv4_x.0.residual_function.0')]),
    _m("m_r18_256x56_256_3x3", (64, 256, 56, 56, 256, 3, 1, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=1792, n_items=3584, col_tiles=2, n_ntiles=2),
       [('resnet18_iao_ptq_224', 'conv4_x.1.residual_function.0')]),
    _m("m_r18_256x56_512_3x3s2", (64, 256, 56, 56, 512, 3, 2, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=448, n_items=1792, col_tiles=1, n_ntiles=4),
       [('resnet18_iao_ptq_224', 'conv5_x.0.residual_function.0')]),
    _m("m_r18_512x28_512_3x3", (64, 512, 28, 28, 512, 3, 1, 1, 1), "levels", 'iao8', dict(Nt=128, MT=1, n_mtiles=448, n_items=1792, col_tiles=1, n_ntiles=4),
       [('resnet18_iao_ptq_224', 'conv5_x.1.residual_function.0')]),
    _m("m_r18i8_64x224_64_3x3", (64, 64, 224, 224, 64, 3, 1, 1, 1), "levels_i8", 'iao8', dict(Nt=64, MT=2, n_mtiles=28672, n_items=14336, col_tiles=8, n_ntiles=1),
       [('resnet18_iao_ptq_224_int8', 'conv2_x.0.residual_function.0'), ('resnet18_iao_ptq_224_int8', 'conv2_x.1.residual_function.0')]),
    _m("m_r18i8_64x224_128_3x3s2", (64, 64, 224, 224, 128, 3, 2, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=7168, n_items=7168, col_tiles=2, n_ntiles=1),
       [('resnet18_iao_ptq_224_int8', 'conv3_x.0.residual_function.0')]),
    _m("m_r18i8_128x112_128_3x3", (64, 128, 112, 112, 128, 3, 1, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=7168, n_items=7168, col_tiles=4, n_ntiles=1),
       [('resnet18_iao_ptq_224_int8', 'conv3_x.1.residual_function.0')]),
    _m("m_r18i8_128x112_256_3x3s2", (64, 128, 112, 112, 256, 3, 2, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=1792, n_items=3584, col_tiles=1, n_ntiles=2),
       [('resnet18_iao_ptq_224_int8', 'conv4_x.0.residual_function.0')]),
    _m("m_r18i8_256x56_256_3x3", (64, 256, 56, 56, 256, 3, 1, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=1792, n_items=3584, col_tiles=2, n_ntiles=2),
       [('resnet18_iao_ptq_224_int8', 'conv4_x.1.residual_function.0')]),
    _m("m_r18i8_256x56_512_3x3s2", (64, 256, 56, 56, 512, 3, 2, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=448, n_items=1792, col_tiles=1, n_ntiles=4),
       [('resnet18_iao_ptq_224_int8', 'conv5_x.0.residual_function.0')]),
    _m("m_r18i8_512x28_512_3x3", (64, 512, 28, 28, 512, 3, 1, 1, 1), "levels_i8", 'iao8', dict(Nt=128, MT=1, n_mtiles=448, n_items=1792, col_tiles=1, n_ntiles=4),
       [('resnet18_iao_ptq_224_int8', 'conv5_x.1.residual_function.0')]),
]
ALL_CASES = CASES + MODEL_CASES

# ---- refusals: one shape per reason the host can reach; (id, shape, cpu, ta, post options, return code name, error text)
# post options: q, bn ("all" / "partial"), sg, split, terms
Refusal = namedtuple("Refusal", "id shape cpu ta opts code text")
REFUSALS = [
    Refusal("bn_partial", (2, 16, 8, 8, 16, 1, 1, 0, 1), 8, 1, dict(q="iao8", bn="partial"), "E_ARG", "all four"),
    Refusal("bn_nout_mod4", (2, 16, 8, 8, 18, 1, 1, 0, 1), 8, 1, dict(q="iao8", bn="all"), "E_UNSUPPORTED", "% 4 == 0"),
    Refusal("sg_not_dividing", (2, 16, 8, 8, 32, 1, 1, 0, 1), 8, 1, dict(q="iao8", sg=3), "E_UNSUPPORTED", "do not divide"),
    Refusal("sg_with_split", (2, 16, 8, 8, 32, 1, 1, 0, 1), 8, 1, dict(q="iao8", sg=2, split=1), "E_UNSUPPORTED",
            "shuffle in front of a stride-2 consumer"),
    Refusal("sg_nout_mod_unit", (2, 16, 8, 8, 12, 1, 1, 0, 1), 8, 1, dict(q="iao8", sg=2), "E_UNSUPPORTED",
            "channels per unit"),
    Refusal("sg_nout_mod_unit_i8", (2, 32, 8, 8, 24, 1, 1, 0, 1), 16, 1, dict(q="iao8", sg=2), "E_UNSUPPORTED",
            "channels per unit"),
    Refusal("i8_quantizer_rule", (2, 32, 8, 8, 32, 1, 1, 0, 1), 16, 1, dict(q="dorefa8"), "E_UNSUPPORTED", "int8 plane needs"),
    Refusal("i8_quantizer_asym", (2, 32, 8, 8, 32, 1, 1, 0, 1), 16, 1, dict(q="iao8a"), "E_UNSUPPORTED", "int8 plane needs"),
    Refusal("i8_grouped_ng16", (2, 64, 8, 8, 48, 1, 1, 0, 2), 16, 1, dict(q="iao8"), "E_UNSUPPORTED", "% 16 == 0"),
    Refusal("grouped_ng8", (2, 32, 8, 8, 24, 1, 1, 0, 2), 8, 1, dict(q="iao8"), "E_UNSUPPORTED", "per group % 8 == 0"),
    Refusal("terms_ng8", (2, 16, 8, 8, 12, 1, 1, 0, 1), 8, 1, dict(terms=3), "E_UNSUPPORTED", "term planes need"),
    Refusal("terms_grouped_ng8", (2, 32, 8, 8, 24, 1, 1, 0, 2), 8, 1, dict(terms=3), "E_UNSUPPORTED", "term planes need"),
    Refusal("terms_gt3", (2, 16, 8, 8, 16, 1, 1, 0, 1), 8, 1, dict(terms=4), "E_ARG", "term planes (1..3)"),
    Refusal("split_odd_plane", (2, 16, 7, 7, 16, 1, 1, 0, 1), 8, 1, dict(q="iao8", split=1), "E_UNSUPPORTED", "odd-sized"),
    Refusal("segmented_plan", (4, 64, 16, 16, 128, 3, 1, 1, 1), 8, 2, dict(q="iao8"), "E_UNSUPPORTED", "segmented"),
    Refusal("q_mode_sign", (2, 16, 8, 8, 16, 1, 1, 0, 1), 8, 1, dict(q="sign"), "E_ARG", "DoReFa or IAO"),
    Refusal("q_bits9", (2, 16, 8, 8, 16, 1, 1, 0, 1), 8, 1, dict(q="dorefa9"), "E_ARG", "2..8 bits"),
    Refusal("q_with_terms", (2, 16, 8, 8, 16, 1, 1, 0, 1), 8, 1, dict(q="iao8", terms=2), "E_ARG", "terms_out without one"),
]


def conv_shape(shape):
    from micronet_b200 import _lib as L
    B, Cc, H, W, K, R, st, pad, G = shape
    return L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)


def out_hw(shape):
    B, Cc, H, W, K, R, st, pad, G = shape
    return (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1


def qparams(q, device=None, rng=(-3.7, 5.3)):
    """(ActQParams struct, quantizer description dict, tensors kept alive) of a consumer quantizer name; the IAO scalars
    live on ``device`` (None: fake aligned host addresses, for host-only queries that never read them); ``rng``: the IAO
    observer range"""
    from micronet_b200 import _lib as L
    if q.startswith("dorefa"):
        bits = int(q[6:])
        return L.ActQParams(L.ACT_DOREFA, bits, 0, (1 << bits) - 1, 0, None, None, None, None), dict(kind="dorefa", bits=bits), []
    if q == "sign":
        return L.ActQParams(L.ACT_SIGN, 1, -1, 1, 0, None, None, None, None), dict(kind="sign"), []
    sym = not q.endswith("a")
    bits = int(q[3:].rstrip("a"))
    qmin, qmax = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if sym else (0, (1 << bits) - 1)
    import torch
    mn, mx = torch.tensor([rng[0]]), torch.tensor([rng[1]])
    if sym:
        sc = (torch.max(mn.abs(), mx.abs()) / ((qmax - qmin) / 2)).float()
        zp = torch.zeros(1)
    else:
        sc = ((mx - mn) / float(qmax - qmin)).float()
        zp = torch.sign(mn) * torch.floor((mn / sc).abs() + 0.5)
    desc = dict(kind="iao", bits=bits, qmin=qmin, qmax=qmax, scale=float(sc), zp=float(zp), sym=sym)
    if device is None:
        fake = [1 << 20, (1 << 20) + 16, (1 << 20) + 32, (1 << 20) + 48]
        return L.ActQParams(L.ACT_IAO, bits, qmin, qmax, 0 if sym else 1, *fake), desc, []
    bufs = [t.to(device) for t in (sc, zp, mn, mx)]
    return L.ActQParams(L.ACT_IAO, bits, qmin, qmax, 0 if sym else 1, *(t.data_ptr() for t in bufs)), desc, bufs


def post_struct(q_struct, plane_ptr, relu, split, bn_ptrs, sg, terms):
    """mnb_pk_post from plain values; bn_ptrs = four addresses (or None entries)"""
    import ctypes as C
    from micronet_b200 import _lib as L
    post = L.PkPost(C.pointer(q_struct) if q_struct is not None else None, int(relu), int(split), plane_ptr)
    post.bn_mean, post.bn_invstd, post.bn_gamma, post.bn_beta = bn_ptrs
    post.shuffle_groups, post.terms_out = int(sg), int(terms)
    return post


FAKE = 1 << 22     # 16-byte aligned host address; the plan query compares and checks pointers, never dereferences them


def host_post(case_or_opts):
    """(mnb_pk_post, kept objects) with fake addresses for the host query of a case or of a refusal's options"""
    if isinstance(case_or_opts, Case):
        c = case_or_opts
        opts = dict(q=c.q, bn="all" if c.bn else None, sg=c.sg, split=int(c.split), terms=c.terms, relu=c.relu)
    else:
        opts = case_or_opts
    qs = None
    if opts.get("q"):
        qs, _, _ = qparams(opts["q"])
    bn = opts.get("bn")
    bn_ptrs = (FAKE + 64, FAKE + 128, FAKE + 192, FAKE + 256) if bn == "all" else \
        (FAKE + 64, None, FAKE + 192, FAKE + 256) if bn == "partial" else (None,) * 4
    post = post_struct(qs, FAKE + 4096, opts.get("relu", True), opts.get("split", 0), bn_ptrs, opts.get("sg", 1),
                       opts.get("terms", 0))
    return post, qs


def cpu_of(path):
    return 16 if path in I8_PATHS else 8


def plan_of(case):
    """mnb_pk_conv_post_plan of a case as a dict (call with the case's environment set); (rc, error text) on a refusal"""
    return query(case.shape, cpu_of(case.path), case.ta, host_post(case)[0])


def query(shape, cpu, ta, post):
    import ctypes as C
    from micronet_b200 import _lib as L
    lib = L.load()
    out = (C.c_int32 * len(PLAN_FIELDS))()
    rc = lib.mnb_pk_conv_post_plan(C.byref(conv_shape(shape)), ta, 1, cpu, C.byref(post) if post is not None else None, out,
                                   len(PLAN_FIELDS))
    if rc != 0:
        return rc, lib.mnb_last_error().decode(errors="replace")
    return dict(zip(PLAN_FIELDS, list(out)))


def items_of_cta(plan, G, cta=0):
    """(N tile, group) of the work items CTA ``cta`` runs one after the other (the kernel's item decode)"""
    out = []
    for it in range(cta, plan["n_items"], plan["gx"]):
        out.append((it % plan["n_ntiles"], (it // plan["n_ntiles"]) % G))
    return out
