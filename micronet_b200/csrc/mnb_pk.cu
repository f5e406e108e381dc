// Packed-operand ("pk") tensor-core convolution family: any conv geometry of the QAT models on Hopper wgmma.
//
// Why a second family next to mnb_conv_tc_fwd.cu / mnb_conv_tc_wgrad.cu: those kernels keep the whole weight
// slab of a group resident in shared memory and convert fp32 activations inside the kernel, which limits them
// to small grouped layers (NIN-GC).  ResNet-18 (up to 512 -> 512 3x3 = 9.4 MB of weights, stride 2, 4x4 images),
// NIN's 5x5 96 -> 192 and 224x224 inputs need the B operand STREAMED and N / W tiling.  Here every operand
// reaches the kernel already in the layout the tensor core reads:
//
//   activations / gradients : bf16 "term planes"  pk[t][b][c/8][h][w][8]   (16 bytes = 8 channels of one pixel)
//                             t = 0 .. T-1 exact pieces of an fp32 value (x = p0 + p1 + p2, 8 significand bits each)
//                             or ONE plane of exact integer levels (fake-quantized activations);
//   weights                 : bf16 image [n-tile][group][stage][term][tap][c/8][n][8] (K-major, rows = n), written
//                             once per optimizer step by pk_pack_weight_kernel;
//
// so the convolution itself is the canonical Hopper pipeline TMA -> wgmma (register accumulators) -> epilogue with no
// converter warps.  A 5-D tensor map (8, W, H, B, C/8) with the channel-octet dimension declared LAST makes one
// box land in shared memory as op[c/8][position][8]: the wgmma K-major no-swizzle canonical layout with the
// positions of the zero-padded tile as GEMM rows (halo rows AND columns zero-filled by the TMA unit), so filter tap
// (r, s) is the same buffer with the descriptor start address moved by (r*BW + s)*16 bytes: implicit GEMM without
// im2col.  The same buffers read as MN-major operands give the weight gradient (positions = reduction dimension).
//
// Stride-2 convolutions use the space-to-depth form: the pack kernel writes the four (h%2, w%2) phase planes as extra
// channel octets, every filter tap then is a stride-1 tap of ONE phase plane with a shift in {-1, 0} (data gradient:
// four output phases, each a stride-1 conv of dy with a subset of the taps).
//
// Exactness: integer levels (|e| <= 256) are exact in bf16, products exact, fp32 accumulation in registers.  fp32 operands
// are split into T exact bf16 pieces; the products p_i * q_j with i + j < max(Ta, Tb) are accumulated, smallest first.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

namespace pk {

constexpr int MAXST = 8;           // operand ring (power of two: ring index = counter & mask)
constexpr int MAXTAP = 64, MAXTMPL = 16, MAXY = 4, MAXPAIR = 6, MAXPROG = 512;
constexpr int kSmemBudget = 227 * 1024 - 3072;   // dynamic shared memory the kernels may ask for
constexpr int kNtSizes[] = {16, 32, 48, 64, 96, 128};   // N tiles the convolution kernel is instantiated for

// ---------------------------------------------------------------------------------------------------------
// plan: everything about a (shape, mode) pair that the weight packer and the convolution must agree on
// ---------------------------------------------------------------------------------------------------------
struct Tmpl { int kph, tap0, ntap, blk_off, blk_bytes; };   // one (k-phase, tap group): a pipeline stage template

struct Plan {
  int mode;                 // 0 forward, 1 data gradient
  int B, G, R, S, stride;
  int HA, WA, C8A, nkph;    // A planes as stored: spatial dims, octets per k-phase (all groups), k-phases
  int kg, ng, NOUT;         // GEMM-K / GEMM-N channels per group, total output channels
  int OHr, OWr, OH, OW, omul, ny;   // raster (per output phase) and real output dims
  int hlo, hhi, wlo, whi;
  int Wt, BW, TH, THH, TB, npos, col_tiles, row_tiles, img_tiles, n_mtiles;
  int Nt, n_ntiles, MT, n_mgroups, n_items;
  int CC, ksteps, chunks;   // K-chunk channels (multiple of 16), MMAs along K per chunk, chunks per k-phase
  int TA, TBk, npairs, pair_a[MAXPAIR], pair_b[MAXPAIR];
  int ntmpl[MAXY], ntap[MAXY];
  Tmpl tmpl[MAXY][MAXTMPL];
  int tap_aoff[MAXY][MAXTAP];            // A start-row offset of a tap inside the box (16-byte units)
  short tap_r[MAXY][MAXTAP], tap_s[MAXY][MAXTAP];
  int img_bytes[MAXY], y_off[MAXY];      // bytes of one (n-tile, group) weight image of output phase y; prefix offsets
  int64_t wimg_bytes;
  int a_box_bytes, a_bytes, b_off, stage_bytes, nstage, st_log2, smem_bytes, off_stg;
  int segmented, seg_len;   // stages per accumulation segment (segmented mode)
  int cpu;                  // channels per 16-byte unit of the operands: 8 (bf16), 16 (int8)
};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

static void make_pairs(int TA, int TBk, Plan& p) {
  // pieces have magnitudes 2^-8i: accumulate the products p_i q_j with i + j <= max(TA, TBk) - 1, smallest first
  const int lim = std::max(TA, TBk) - 1;
  p.npairs = 0;
  for (int sum = lim; sum >= 0; --sum)
    for (int a = 0; a < TA; ++a) {
      const int b = sum - a;
      if (b < 0 || b >= TBk) continue;
      if (p.npairs < MAXPAIR) { p.pair_a[p.npairs] = a; p.pair_b[p.npairs] = b; ++p.npairs; }
    }
}

static int unsupported(const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "pk conv: %s", why); }

// mode 0: y = conv2d(x, w); mode 1: dx = conv_transpose(dy, w).  TA / TBk: term planes of the streamed / weight operand.
// cpu: channels per 16-byte operand unit - 8 for bf16 planes (K-step of 16 channels), 16 for int8 planes (K-step of 32
// channels: one s8 K32 MMA reads the same 32 bytes per row as one bf16 K16 MMA, so every byte-level quantity below is
// shared).  int8 plans are forward, single-product (TA = TBk = 1) and never segmented.
static int make_plan(const mnb_conv_shape* s, int mode, int TA, int TBk, Plan& p, int cpu = 8) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  memset(&p, 0, sizeof(p));
  const int C = s->in_c, K = s->out_c, G = s->groups, H = s->in_h, W = s->in_w, R = s->ker_h, S = s->ker_w;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && H > 0 && W > 0 && G > 0 && C % G == 0 && K % G == 0 && R > 0 && S > 0,
              "bad conv shape");
  MNB_REQUIRE(TA >= 1 && TA <= 3 && TBk >= 1 && TBk <= 3, "term counts must be 1..3");
  MNB_REQUIRE(cpu == 8 || (cpu == 16 && mode == 0 && TA == 1 && TBk == 1), "int8 plans are single-product forward plans");
  if (s->dil_h != 1 || s->dil_w != 1) return unsupported("dilation != 1");
  if (s->stride_h != s->stride_w || (s->stride_h != 1 && s->stride_h != 2)) return unsupported("stride must be 1 or 2");
  const int st = s->stride_h, ph_ = s->pad_h, pw_ = s->pad_w;
  if (ph_ > R - 1 || pw_ > S - 1) return unsupported("padding larger than the filter");
  const int P = (H + 2 * ph_ - R) / st + 1, Q = (W + 2 * pw_ - S) / st + 1;
  if (P < 1 || Q < 1) return unsupported("empty output");
  if (st == 2 && ((H | W) & 1)) return unsupported("stride 2 needs even H and W");
  const int cin_g = C / G, cout_g = K / G;
  p.mode = mode; p.B = s->batch; p.G = G; p.R = R; p.S = S; p.stride = st;
  p.TA = TA; p.TBk = TBk; p.cpu = cpu;
  make_pairs(TA, TBk, p);
  if (mode == 0) {
    p.kg = cin_g; p.ng = cout_g; p.NOUT = K;
    p.nkph = st == 2 ? 4 : 1;
    p.HA = H / st; p.WA = W / st; p.C8A = ceil_div(C, cpu);
    p.OHr = P; p.OWr = Q; p.OH = P; p.OW = Q; p.omul = 1; p.ny = 1;
  } else {
    p.kg = cout_g; p.ng = cin_g; p.NOUT = C;
    p.nkph = 1; p.HA = P; p.WA = Q; p.C8A = ceil_div(K, 8);
    p.OHr = H / st; p.OWr = W / st; p.OH = H; p.OW = W; p.omul = st; p.ny = st == 2 ? 4 : 1;
  }
  if (cpu == 16 && G > 1 && (p.kg % cpu)) return unsupported("grouped int8 conv needs GEMM-K channels per group % 16 == 0");
  // bf16 planes of a grouped conv are group-padded: group g's K-octets start at octet g * ceil(kg / 8) (DESIGN.md 4.17;
  // the same octets as ceil(C / 8) whenever kg % 8 == 0 or G == 1)
  if (cpu == 8) p.C8A = G * ceil_div(p.kg, 8);
  // s32 accumulators: |level| <= 128 (activations) times |level| <= 127 (symmetric weights) over kg x taps products
  if (cpu == 16 && (int64_t)p.kg * R * S * 128 * 127 > (int64_t)INT32_MAX) return unsupported("int8 sums could overflow s32");
  // ---- taps: (k-phase, shift) of every filter tap, per output phase
  struct Tap { int kph, sh, sw, r, s; };
  Tap taps[MAXY][MAXTAP];
  int hlo = 0, hhi = 0, wlo = 0, whi = 0;
  for (int y = 0; y < p.ny; ++y) {
    int n = 0;
    const int ya = y >> 1, yb = y & 1;
    for (int kph = 0; kph < p.nkph; ++kph)       // taps sorted by k-phase
      for (int r = 0; r < R; ++r)
        for (int q = 0; q < S; ++q) {
          int kp = 0, sh, sw;
          if (mode == 0) {
            const int dr = r - ph_, ds = q - pw_;
            if (st == 1) { sh = dr; sw = ds; }
            else {
              const int fh = dr & 1, fw = ds & 1;
              kp = fh * 2 + fw; sh = (dr - fh) / 2; sw = (ds - fw) / 2;
            }
          } else {
            if (st == 1) { sh = ph_ - r; sw = pw_ - q; }
            else {
              const int th = ya + ph_ - r, tw = yb + pw_ - q;
              if ((th & 1) || (tw & 1)) continue;
              sh = th / 2; sw = tw / 2;   // exact (even), also for negatives
            }
          }
          if (kp != kph) continue;
          if (n >= MAXTAP) return unsupported("more than 64 filter taps");
          taps[y][n++] = Tap{kph, sh, sw, r, q};
          hlo = std::max(hlo, -sh); hhi = std::max(hhi, sh); wlo = std::max(wlo, -sw); whi = std::max(whi, sw);
        }
    p.ntap[y] = n;
  }
  p.hlo = hlo; p.hhi = hhi; p.wlo = wlo; p.whi = whi;
  // ---- M tile: 128 consecutive positions of the zero-padded tile raster (tb, row, col)
  const int halo_w = wlo + whi;
  if (halo_w >= 96) return unsupported("filter too wide");
  // Column tiling: a tile is TH rows of Wt columns, rastered with the row pitch BW = Wt + halo, and its last valid position
  // must be < 128.  Narrower tiles often hold MORE valid positions (224 wide: 1 x 112 = 112 vs 4 x 28 = 112 with a third
  // of the halo rows; 32 wide: 3 x 32 = 96 vs 7 x 16 = 112) - every tile costs the same MMAs, and the halo rows are re-read
  // (THH * BW) / (TH * Wt) times.  cost = tiles per image * (1 + 0.25 * read amplification) * (1 + 3.2 / Wt)
  {
    const int ct_min = ceil_div(p.OWr, 128 - halo_w);
    double best = 1e30;
    // (the single-product kernels gain from narrower tiles, while the segmented split-fp32 kernels keep the widest tiling
    // unless it re-reads its halo rows more than ~2.2 x, as on 112- and 224-wide planes)
    int ct_max = std::min(p.OWr, ct_min + 14);
    if (p.npairs > 1) {
      const int wt0 = ceil_div(p.OWr, ct_min), bw0 = wt0 + halo_w;
      const int th0 = std::max(1, std::min(p.OHr, (128 - wt0) / bw0 + 1));
      if ((double)((th0 + hlo + hhi) * bw0) / (double)(th0 * wt0) <= 2.2) ct_max = ct_min;
    }
    for (int ct = ct_min; ct <= ct_max; ++ct) {
      const int wt = ceil_div(p.OWr, ct), bw = wt + halo_w;
      if (ceil_div(p.OWr, wt) != ct) continue;                       // same tiling as a smaller ct
      const int th = std::max(1, std::min(p.OHr, (128 - wt) / bw + 1));
      const double amp = (double)((th + hlo + hhi) * bw) / (double)(th * wt);
      // (+ a mild preference for long rows: the epilogue's fp32 stores cover Wt * 4 contiguous bytes per channel and row)
      const double cost = (double)ct * ceil_div(p.OHr, th) * (1.0 + 0.25 * amp) * (1.0 + 3.2 / wt);
      if (cost < best - 1e-9) { best = cost; p.col_tiles = ct; p.Wt = wt; p.BW = bw; p.TH = th; }
    }
    if (const char* e = getenv("MNB_PK_COLTILES")) {                 // experiments: force the number of column tiles
      const int ct = atoi(e);
      if (ct >= ct_min && ct <= p.OWr) {
        p.col_tiles = ct; p.Wt = ceil_div(p.OWr, ct); p.col_tiles = ceil_div(p.OWr, p.Wt); p.BW = p.Wt + halo_w;
        p.TH = std::max(1, std::min(p.OHr, (128 - p.Wt) / p.BW + 1));
      }
    }
  }
  p.THH = p.TH + hlo + hhi;
  p.TB = 1;
  if (p.TH == p.OHr && p.col_tiles == 1) {
    const int last = (p.TH - 1) * p.BW + p.Wt;             // rows used by the last image of a tile
    p.TB = std::max(1, std::min(p.B, (128 - last) / (p.THH * p.BW) + 1));
  }
  if (p.BW > 128 || p.THH > 256 || p.TB > 256) return unsupported("box dimension");
  p.npos = p.TB * p.THH * p.BW;
  p.row_tiles = ceil_div(p.OHr, p.TH);
  p.img_tiles = ceil_div(p.B, p.TB);
  p.n_mtiles = p.img_tiles * p.row_tiles * p.col_tiles;
  // ---- N tile
  const int ng16 = round_up(p.ng, 16);
  // Split fp32 operands (more than one piece product per K-step) run in SEGMENTED mode: the tensor core does not round the
  // running fp32 accumulator to nearest after every instruction, so the K loop is cut into segments of <= ~64 MMAs, each
  // into zeroed accumulators, and the segments are added into running sums with round-to-nearest fp32 adds.  A K loop that
  // is short anyway needs no segments: the whole chain of one accumulator (taps x piece pairs x K-steps) is then no longer
  // than a segment would be.
  {
    int seg_target = 64;
    if (const char* e = getenv("MNB_PK_SEG_MMAS")) seg_target = std::max(1, atoi(e));
    int chain = 0;
    for (int y = 0; y < p.ny; ++y) chain = std::max(chain, p.ntap[y] * p.npairs * ceil_div(p.kg, 16));
    p.segmented = p.npairs > 1 && chain > seg_target;
  }
  // N tile: the accumulators of a thread are MT x Nt / 2 registers (two warpgroups, 64 rows each), so Nt <= 128, and Nt is
  // one of the widths the kernel is instantiated for (kNtSizes); the weight image zero-pads the columns beyond ng
  {
    const int ntiles = ceil_div(ng16, 128);
    const int want = round_up(ceil_div(ng16, ntiles), 16);
    p.Nt = 128;
    for (int v : kNtSizes) if (v >= want) { p.Nt = v; break; }
  }
  p.n_ntiles = ceil_div(p.ng, p.Nt);
  // M tiles per work item: every item streams the WHOLE weight block of its (N tile, group) from L2, so at MT = 1 the
  // L2 -> shared-memory bandwidth on the re-fetched weights bounds the kernel.  MT M tiles share one weight fetch (registers: MT x Nt <= 128).
  // The items are dealt to MNB_NUM_SMS persistent CTAs, so a larger MT is taken only while it costs no wave efficiency.
  p.MT = 1;
  {
    auto wave_eff = [&](int mt) {
      const int64_t items = (int64_t)ceil_div(p.n_mtiles, mt) * p.n_ntiles * G;
      const int64_t ctas = std::max<int64_t>(1, MNB_NUM_SMS / p.ny);
      return (double)items / (double)(ceil_div((int)std::min<int64_t>(items, 1 << 30), (int)ctas) * ctas);
    };
    const int cap = std::max(1, 128 / p.Nt);
    for (int mt = 2; mt <= std::min(4, cap); mt *= 2) {
      if (p.n_mtiles < mt) break;
      if ((int64_t)ceil_div(p.n_mtiles, mt) * p.n_ntiles * G * p.ny < 120) break;
      if (wave_eff(mt) >= wave_eff(1) - 0.04) p.MT = mt;
    }
  }
  if (const char* e = getenv("MNB_PK_MT")) {
    const int v = atoi(e);
    if ((v == 1 || v == 2 || v == 4) && v * p.Nt <= 128) p.MT = v;
  }
  p.n_mgroups = ceil_div(p.n_mtiles, p.MT);
  p.n_items = p.n_mgroups * p.n_ntiles * G;
  // ---- K chunking and tap groups: one stage = MT * TA boxes of CC channels + the weights of (chunk, tap group)
  const int nk16 = ceil_div(p.kg, 2 * cpu);      // K-steps (16 bf16 / 32 int8 channels = 32 bytes per row)
  int maxtap_kph = 1;
  for (int y = 0; y < p.ny; ++y)
    for (int i = 0, run = 0; i < p.ntap[y]; ++i) {
      run = (i > 0 && taps[y][i].kph == taps[y][i - 1].kph) ? run + 1 : 1;
      maxtap_kph = std::max(maxtap_kph, run);
    }
  const int a16 = p.MT * TA * round_up(2 * p.npos * 16, 128);     // A bytes per K-step (2 units)
  auto b16 = [&](int tg) { return TBk * tg * 2 * p.Nt * 16; };   // B bytes per K-step
  const int stage_target = 56 * 1024;
  int TG = std::min(maxtap_kph, 25);
  while (TG > 1 && a16 + b16(TG) > stage_target) --TG;
  if (a16 + b16(TG) > (kSmemBudget - 8192) / 2) return unsupported("one 16-channel stage does not fit in shared memory");
  int cc16 = std::max(1, std::min(nk16, stage_target / (a16 + b16(TG))));
  cc16 = std::min(cc16, 16);
  p.chunks = ceil_div(nk16, cc16);
  cc16 = ceil_div(nk16, p.chunks);            // balance the chunks
  p.CC = cc16 * 2 * cpu; p.ksteps = cc16;
  p.a_box_bytes = (p.CC / cpu) * p.npos * 16;
  p.a_bytes = round_up(p.a_box_bytes, 128);
  p.b_off = p.MT * TA * p.a_bytes;
  // ---- stage templates and the weight-image layout
  int64_t total = 0;
  int max_blk = 0;
  for (int y = 0; y < p.ny; ++y) {
    int nt = 0, off = 0;
    for (int i = 0; i < p.ntap[y];) {
      int j = i;
      while (j < p.ntap[y] && taps[y][j].kph == taps[y][i].kph && j - i < TG) ++j;
      if (nt >= MAXTMPL) return unsupported("too many tap groups");
      Tmpl& t = p.tmpl[y][nt++];
      t.kph = taps[y][i].kph; t.tap0 = i; t.ntap = j - i;
      t.blk_bytes = TBk * t.ntap * (p.CC / cpu) * p.Nt * 16;
      t.blk_off = off;
      off += p.chunks * t.blk_bytes;
      max_blk = std::max(max_blk, t.blk_bytes);
      i = j;
    }
    p.ntmpl[y] = nt;
    p.img_bytes[y] = off;
    p.y_off[y] = (int)total;
    total += (int64_t)off * p.n_ntiles * G;
    if (total > (int64_t)1 << 30) return unsupported("weight image larger than 1 GiB");
    for (int i = 0; i < p.ntap[y]; ++i) {
      p.tap_aoff[y][i] = (taps[y][i].sh + hlo) * p.BW + (taps[y][i].sw + wlo);
      p.tap_r[y][i] = (short)taps[y][i].r; p.tap_s[y][i] = (short)taps[y][i].s;
    }
  }
  p.wimg_bytes = std::max<int64_t>(total, 16);
  p.seg_len = 1 << 30;
  if (p.segmented) {
    const int per_stage = TG * p.npairs * p.ksteps;     // MMAs per accumulator and stage (upper bound)
    int target = 64;
    if (const char* e = getenv("MNB_PK_SEG_MMAS")) target = std::max(1, atoi(e));
    p.seg_len = std::max(1, target / per_stage);
  }
  p.stage_bytes = round_up(p.b_off + max_blk, 1024);
  // slack behind the last stage: MMAs of invalid halo rows read up to 128 + max tap offset rows past a plane start
  const int slack = round_up((128 + (hlo + hhi) * p.BW + halo_w + 8) * 16, 1024);
  const int stg = 32 * tc::kStageLd * 4;   // 128 x 32 epilogue staging tile behind the slack
  int nst = (kSmemBudget - slack - stg) / p.stage_bytes;
  if (nst < 2) return unsupported("fewer than two pipeline stages fit");
  p.nstage = nst >= 8 ? 8 : (nst >= 4 ? 4 : 2);
  if (const char* e = getenv("MNB_PK_STAGES")) { const int v = atoi(e); if ((v == 2 || v == 4 || v == 8) && v <= nst) p.nstage = v; }
  p.st_log2 = p.nstage == 8 ? 3 : (p.nstage == 4 ? 2 : 1);
  p.off_stg = p.nstage * p.stage_bytes + slack;
  p.smem_bytes = p.off_stg + stg;
  if (p.MT * p.Nt > 128) return unsupported("accumulators exceed the register budget");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// operand packers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// four integer levels (exact floats in [-128, 127]) -> four s8 bytes, first in the lowest byte
__device__ __forceinline__ uint32_t pack4_s8(float a, float b, float c, float d) {
  return ((uint32_t)__float2int_rn(a) & 0xffu) | (((uint32_t)__float2int_rn(b) & 0xffu) << 8) |
         (((uint32_t)__float2int_rn(c) & 0xffu) << 16) | ((uint32_t)__float2int_rn(d) << 24);
}
__device__ __forceinline__ uint4 pack16_s8(const float (&l)[16]) {
  return make_uint4(pack4_s8(l[0], l[1], l[2], l[3]), pack4_s8(l[4], l[5], l[6], l[7]), pack4_s8(l[8], l[9], l[10], l[11]),
                    pack4_s8(l[12], l[13], l[14], l[15]));
}

// fp32 NCHW -> bf16 term planes [t][b][octet][h][w][8]; one thread = one pixel of one channel octet.
//   QUANT = 0: planes are the exact pieces of x (* ch_scale[c] when given)
//   QUANT = 1: plane 0.. hold the fake-quantized integer level e = code + a_off (+ zero point) (exact; two pieces when
//              |e| can exceed 256), bits8[b][c/8][h][w] bit j = STE pass flag of channel 8*(c/8) + j
// phase_split: octet index (h%2 * 2 + w%2) * C8 + c/8 of a [.., H/2, W/2] plane (stride-2 consumers)
// GROUPED: the group-padded plane of a grouped conv with cg channels per group, cg % 8 != 0: group g's channel j sits at
// plane channel g * kg8 * 8 + j (kg8 = ceil(cg / 8) octets per group), the padding channels are zero in every plane and mask.
template <int QUANT, bool GROUPED>
__device__ __forceinline__ void pack_act_body(const float* __restrict__ x, int B, int C, int H, int W, int C8, int terms,
                                              const float* __restrict__ ch_scale, mnb_act_qparams qp, int phase_split,
                                              uint4* __restrict__ out, int64_t plane_vecs, uint8_t* __restrict__ bits8, int relu,
                                              int cg, int kg8) {
  MnbActQ q;
  float zp = 0.f;
  if (QUANT) {
    q = mnb_load_actq(qp);
    if (qp.mode == MNB_ACT_IAO && qp.zero_point) zp = __ldg(qp.zero_point);
  }
  // grid = (chunks of the H*W plane, B * C8 planes): 32-bit index arithmetic only (no per-pixel divisions)
  const uint32_t HW = (uint32_t)H * (uint32_t)W;
  // block = (positions, planes): small images put several planes into one 256-thread block
  const uint32_t plane = blockIdx.y * blockDim.y + threadIdx.y;                 // b * C8 + c8
  if (plane >= (uint32_t)B * (uint32_t)C8) return;
  const uint32_t b = plane / (uint32_t)C8, c8 = plane - b * (uint32_t)C8;
  // first channel of the octet, and (GROUPED) its index inside its group: channels jb + j >= cg are padding
  uint32_t cb = c8 * 8, jb = 0;
  if (GROUPED) {
    const uint32_t g = c8 / (uint32_t)kg8;
    jb = (c8 - g * (uint32_t)kg8) * 8;
    cb = g * (uint32_t)cg + jb;
  }
  for (uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x; pos < HW; pos += gridDim.x * blockDim.x) {
    const int64_t idx = (int64_t)plane * HW + pos;
    float v[8];
    uint32_t passbits = 0;
    const float* src = x + ((int64_t)b * C + (GROUPED ? cb : c8 * 8)) * HW + pos;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = GROUPED ? (int)cb + j : (int)c8 * 8 + j;
      const bool in = GROUPED ? (int)jb + j < cg : c < C;
      float val = in ? __ldg(src + (int64_t)j * HW) : 0.f;
      if (relu) val = fmaxf(val, 0.f);          // a preceding nn.ReLU folded into the packer (inference graphs)
      if (!QUANT && ch_scale) val = in ? __fmul_rn(val, __ldg(ch_scale + c)) : 0.f;
      v[j] = val;
    }
    if (QUANT) {   // level itself (code + a_off) as a float, eight channels in straight-line code
      float lev[8];
      mnb_act_levels<8>(q, v, lev, passbits);
      uint32_t live = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool in = GROUPED ? (int)jb + j < cg : (int)c8 * 8 + j < C;
        v[j] = in ? lev[j] + zp : 0.f;
        live |= in ? (1u << j) : 0u;
      }
      passbits &= live;
    }
    int64_t dst;
    if (phase_split) {
      const uint32_t h = pos / (uint32_t)W, w = pos - h * (uint32_t)W;
      const uint32_t oct = ((h & 1u) * 2u + (w & 1u)) * (uint32_t)C8 + c8;
      dst = (((int64_t)b * 4 * C8 + oct) * (H >> 1) + (h >> 1)) * (W >> 1) + (w >> 1);
    } else {
      dst = idx;
    }
    for (int tm = 0; tm < terms; ++tm) {
      uint32_t pk4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        pk4[j] = pack2(v[2 * j], v[2 * j + 1]);
        v[2 * j] -= __uint_as_float(pk4[j] << 16);
        v[2 * j + 1] -= __uint_as_float(pk4[j] & 0xffff0000u);
      }
      out[(int64_t)tm * plane_vecs + dst] = make_uint4(pk4[0], pk4[1], pk4[2], pk4[3]);
    }
    if (QUANT && bits8) bits8[idx] = (uint8_t)passbits;
  }
}

template <int QUANT>
__global__ void __launch_bounds__(256) pack_act_kernel(const float* __restrict__ x, int B, int C, int H, int W, int C8,
                                                       int terms, const float* __restrict__ ch_scale, mnb_act_qparams qp,
                                                       int a_off, int phase_split, uint4* __restrict__ out,
                                                       int64_t plane_vecs, uint8_t* __restrict__ bits8, int relu) {
  pack_act_body<QUANT, false>(x, B, C, H, W, C8, terms, ch_scale, qp, phase_split, out, plane_vecs, bits8, relu, 0, 1);
}

// C8 = groups * kg8 octets per position
template <int QUANT>
__global__ void __launch_bounds__(256) pack_act_grouped_kernel(const float* __restrict__ x, int B, int C, int H, int W, int C8,
                                                               int terms, const float* __restrict__ ch_scale, mnb_act_qparams qp,
                                                               int phase_split, uint4* __restrict__ out, int64_t plane_vecs,
                                                               uint8_t* __restrict__ bits8, int relu, int cg, int kg8) {
  pack_act_body<QUANT, true>(x, B, C, H, W, C8, terms, ch_scale, qp, phase_split, out, plane_vecs, bits8, relu, cg, kg8);
}

// fp32 NCHW -> int8 level plane [b][c/16][h][w][16] of a symmetric IAO quantizer (levels in [-128, 127]): the levels of
// pack_act_kernel<1> with one piece, stored as s8; one thread = one pixel of one 16-channel unit.  phase_split: unit index
// (h%2 * 2 + w%2) * C16 + c/16 of a [.., H/2, W/2] plane (stride-2 consumers).  No STE bits (inference only).
__global__ void __launch_bounds__(256) pack_act_i8_kernel(const float* __restrict__ x, int B, int C, int H, int W, int C16,
                                                          mnb_act_qparams qp, int phase_split, int relu, uint4* __restrict__ out) {
  const MnbActQ q = mnb_load_actq(qp);
  const float zp = (qp.mode == MNB_ACT_IAO && qp.zero_point) ? __ldg(qp.zero_point) : 0.f;
  const uint32_t HW = (uint32_t)H * (uint32_t)W;
  const uint32_t plane = blockIdx.y * blockDim.y + threadIdx.y;                 // b * C16 + c16
  if (plane >= (uint32_t)B * (uint32_t)C16) return;
  const uint32_t b = plane / (uint32_t)C16, c16 = plane - b * (uint32_t)C16;
  for (uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x; pos < HW; pos += gridDim.x * blockDim.x) {
    const float* src = x + ((int64_t)b * C + c16 * 16) * HW + pos;
    float v[16], lev[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float val = (int)c16 * 16 + j < C ? __ldg(src + (int64_t)j * HW) : 0.f;
      if (relu) val = fmaxf(val, 0.f);
      v[j] = val;
    }
    uint32_t passbits;
    mnb_act_levels<16>(q, v, lev, passbits);
#pragma unroll
    for (int j = 0; j < 16; ++j) lev[j] = (int)c16 * 16 + j < C ? lev[j] + zp : 0.f;
    int64_t dst;
    if (phase_split) {
      const uint32_t h = pos / (uint32_t)W, w = pos - h * (uint32_t)W;
      const uint32_t u = ((h & 1u) * 2u + (w & 1u)) * (uint32_t)C16 + c16;
      dst = (((int64_t)b * 4 * C16 + u) * (H >> 1) + (h >> 1)) * (W >> 1) + (w >> 1);
    } else {
      dst = (int64_t)plane * HW + pos;
    }
    out[dst] = pack16_s8(lev);
  }
}

// BatchNorm2d + ReLU + DoReFa activation quantizer + operand packing in ONE pass (SURVEY.md 8 f2 for the DoReFa blocks
// conv -> nn.BatchNorm2d -> nn.ReLU -> [channel_shuffle] -> QuantConv2d, nin_gc.py:53-59 + DF:36-46): reads the conv output
// once, writes the integer levels of the NEXT conv's activation quantizer as its packed bf16 plane (2 B / element, in the
// output channel order of the folded shuffle) and the combined STE mask  relu'(bn) * [0.1 bn <= 1]  as flat NCHW bits in the
// producer's own channel order - exactly what mnb_bn_sign_bwd consumes, so the backward needs no new kernel.  The fp32
// BatchNorm / ReLU outputs and the separate quantize + pack pass never touch HBM.
// one warp = 32 consecutive positions of one OUTPUT channel octet of one image
__global__ void __launch_bounds__(256) bn_relu_quant_pack_kernel(const float* __restrict__ x, int batch, int channels, int hw,
                                                                 int sg, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, mnb_act_qparams qp,
                                                                 uint32_t* __restrict__ bits, uint4* __restrict__ xp) {
  const int lane = threadIdx.x & 31;
  const int c8n = channels / 8, p32n = hw / 32, cpg = channels / sg;
  const int64_t items = (int64_t)batch * c8n * p32n;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const MnbActQ q = mnb_load_actq(qp);
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
    const int p32 = (int)(w % p32n);
    const int64_t t = w / p32n;
    const int oc8 = (int)(t % c8n), b = (int)(t / c8n);
    const int pos = p32 * 32 + lane;
    float lev[8], yv[8], bnv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int oc = oc8 * 8 + j;
      const int c = sg > 1 ? (oc % sg) * cpg + oc / sg : oc;   // inverse of out[:, a*sg + b] = in[:, b*cpg + a]
      const int64_t fi = ((int64_t)b * channels + c) * hw + pos;
      bnv[j] = fmaf(__ldg(x + fi) - __ldg(mean + c), __ldg(gamma + c) * __ldg(invstd + c), __ldg(beta + c));
      yv[j] = fmaxf(bnv[j], 0.f);                              // nn.ReLU
    }
    uint32_t passbits;
    mnb_act_levels<8>(q, yv, lev, passbits);                   // DoReFa: pass = 0 <= 0.1 y <= 1
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int oc = oc8 * 8 + j;
      const int c = sg > 1 ? (oc % sg) * cpg + oc / sg : oc;
      const int64_t fi = ((int64_t)b * channels + c) * hw + pos;
      const uint32_t word = __ballot_sync(0xffffffffu, ((passbits >> j) & 1u) && bnv[j] > 0.f);   // relu'(0) = 0
      if (lane == 0) bits[fi >> 5] = word;
    }
    xp[((int64_t)b * c8n + oc8) * hw + pos] = make_uint4(pack2(lev[0], lev[1]), pack2(lev[2], lev[3]), pack2(lev[4], lev[5]),
                                                          pack2(lev[6], lev[7]));
  }
}

// bn_relu_quant_pack_kernel writing the int8 plane [b][c/16][hw][16] of a DoReFa quantizer with 2..7 bits (inference only:
// no STE bits); same BatchNorm, ReLU and shuffle sequence.  One warp = 32 consecutive positions of one output unit.
__global__ void __launch_bounds__(256) bn_relu_quant_pack_i8_kernel(const float* __restrict__ x, int batch, int channels, int hw,
                                                                    int sg, const float* __restrict__ mean,
                                                                    const float* __restrict__ invstd,
                                                                    const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, mnb_act_qparams qp,
                                                                    uint4* __restrict__ xp) {
  const int lane = threadIdx.x & 31;
  const int c16n = channels / 16, p32n = hw / 32, cpg = channels / sg;
  const int64_t items = (int64_t)batch * c16n * p32n;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const MnbActQ q = mnb_load_actq(qp);
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
    const int p32 = (int)(w % p32n);
    const int64_t t = w / p32n;
    const int oc16 = (int)(t % c16n), b = (int)(t / c16n);
    const int pos = p32 * 32 + lane;
    float lev[16], yv[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int oc = oc16 * 16 + j;
      const int c = sg > 1 ? (oc % sg) * cpg + oc / sg : oc;
      const int64_t fi = ((int64_t)b * channels + c) * hw + pos;
      yv[j] = fmaxf(fmaf(__ldg(x + fi) - __ldg(mean + c), __ldg(gamma + c) * __ldg(invstd + c), __ldg(beta + c)), 0.f);
    }
    uint32_t passbits;
    mnb_act_levels<16>(q, yv, lev, passbits);
    xp[((int64_t)b * c16n + oc16) * hw + pos] = pack16_s8(lev);
  }
}

// The requantizing table of an IAO max-pool (mnb_pk_plane_maxpool_requant), one entry per stored level P in [-128, 127]
// (entry P + 128): the pool quantizer's dequantized value v = fl((P + zp_in) * s_in), exactly what ActQuantFn writes
// (act_quant_fwd_kernel), requantized by the consumer's quantizer with the exact op sequence of mnb_act_quantize_one
// (__fdiv_rn, mnb_round_half_away, clamp) and stored as the consumer's plane value fl(level + zp_out): bf16 bits, or the
// s8 byte in the low 8 bits.  Symmetric quantizers have zero_point 0, so P is the pool quantizer's level itself.
template <bool I8>
__device__ __forceinline__ void build_requant_table(const mnb_act_qparams& qin, const mnb_act_qparams& qout, uint16_t* tab) {
  const MnbActQ a = mnb_load_actq(qin), b = mnb_load_actq(qout);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    const float lev = (float)min(max(i - 128, a.qmin), a.qmax);
    const float v = __fmul_rn(__fadd_rn(lev, a.zp), a.s);
    bool pass;
    float xq;
    const float o = __fadd_rn((float)(mnb_act_quantize_one(b, v, pass, xq) + b.qmin), b.zp);
    if constexpr (I8) tab[i] = (uint16_t)((uint32_t)__float2int_rn(o) & 0xffu);
    else tab[i] = __bfloat16_as_ushort(__float2bfloat16_rn(o));
  }
}

// window max of a level plane [b][unit][H][W][16 B] (bf16 or s8 levels), unit by unit, padding skipped: the plane of
// max_pool2d(k, s, p) of the decoded activations, because every quantizer whose levels a plane holds is monotone
// non-decreasing.  One thread = one output position of one unit.  REQ: the window max goes out through the requantizing
// table ``tab`` of an IAO pool quantizer -> consumer quantizer pair (build_requant_table; monotone as well, so it commutes
// with the max).
template <bool I8, bool REQ>
__device__ __forceinline__ void plane_maxpool_body(const uint4* __restrict__ in, int64_t planes, int H, int W, int k, int s,
                                                   int pad, int OH, int OW, uint4* __restrict__ out, const uint16_t* tab) {
  const int64_t total = planes * OH * OW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int ow = (int)(idx % OW);
    const int64_t t = idx / OW;
    const int oh = (int)(t % OH);
    const uint4* src = in + (t / OH) * H * W;
    const int h0 = oh * s - pad, w0 = ow * s - pad;
    uint4 m = make_uint4(0, 0, 0, 0);
    bool first = true;
    for (int i = max(h0, 0); i < min(h0 + k, H); ++i)
      for (int j = max(w0, 0); j < min(w0 + k, W); ++j) {
        const uint4 v = __ldg(src + (int64_t)i * W + j);
        if (first) { m = v; first = false; continue; }
        uint32_t* mm = reinterpret_cast<uint32_t*>(&m);
        const uint32_t* vv = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if constexpr (I8) {
            mm[e] = __vmaxs4(mm[e], vv[e]);
          } else {
            __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&mm[e]);
            const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&vv[e]);
            a = __hmax2(a, b);
            mm[e] = *reinterpret_cast<uint32_t*>(&a);
          }
        }
      }
    if constexpr (REQ) {
      uint32_t* mm = reinterpret_cast<uint32_t*>(&m);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const uint32_t v = mm[e];
        if constexpr (I8) {      // s8 level + 128 == its byte with the sign bit flipped
          const uint32_t x = v ^ 0x80808080u;
          mm[e] = (uint32_t)tab[x & 0xffu] | ((uint32_t)tab[(x >> 8) & 0xffu] << 8) |
                  ((uint32_t)tab[(x >> 16) & 0xffu] << 16) | ((uint32_t)tab[x >> 24] << 24);
        } else {                 // bf16 holding an integer level in [-128, 127]
          const int lo = min(max(__float2int_rz(__uint_as_float(v << 16)) + 128, 0), 255);
          const int hi = min(max(__float2int_rz(__uint_as_float(v & 0xffff0000u)) + 128, 0), 255);
          mm[e] = (uint32_t)tab[lo] | ((uint32_t)tab[hi] << 16);
        }
      }
    }
    out[idx] = m;
  }
}

template <bool I8>
__global__ void __launch_bounds__(256) plane_maxpool_kernel(const uint4* __restrict__ in, int64_t planes, int H, int W, int k,
                                                            int s, int pad, int OH, int OW, uint4* __restrict__ out) {
  plane_maxpool_body<I8, false>(in, planes, H, W, k, s, pad, OH, OW, out, nullptr);
}

// the IAO pool (IAO:1285-1343) between two frozen convs: table built once per CTA, then the window max through it
template <bool I8>
__global__ void __launch_bounds__(256) plane_maxpool_requant_kernel(const uint4* __restrict__ in, int64_t planes, int H, int W,
                                                                    int k, int s, int pad, int OH, int OW,
                                                                    uint4* __restrict__ out, mnb_act_qparams qin,
                                                                    mnb_act_qparams qout) {
  // 512 bytes, the kernel's only shared memory.  ptxas reports 1024: this file's dynamic shared array (pk::smem) is aligned
  // to 1024 bytes, so every kernel's static shared memory is rounded up to that alignment.
  __shared__ uint16_t tab[256];
  build_requant_table<I8>(qin, qout, tab);
  __syncthreads();
  plane_maxpool_body<I8, true>(in, planes, H, W, k, s, pad, OH, OW, out, tab);
}

// the exact split of pack_act_body: piece t of each of 8 values into unit dst[t * term_vecs], residues carried over
__device__ __forceinline__ void store_terms8(float (&v)[8], int terms, uint4* __restrict__ dst, int64_t term_vecs) {
  for (int tm = 0; tm < terms; ++tm) {
    uint32_t pk4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      pk4[j] = pack2(v[2 * j], v[2 * j + 1]);
      v[2 * j] -= __uint_as_float(pk4[j] << 16);
      v[2 * j + 1] -= __uint_as_float(pk4[j] & 0xffff0000u);
    }
    dst[(int64_t)tm * term_vecs] = make_uint4(pk4[0], pk4[1], pk4[2], pk4[3]);
  }
}

// max_pool2d(k, s, p) of an fp32 tensor held as `terms` exact bf16 pieces [t][b][c/8][H][W][8] (mnb_pk_plane_maxpool_terms):
// each value is rebuilt as p0 + p1 + p2 (exact: the pieces are the successive rounding residues of pack_act_body), the window
// max is taken with ATen's rule (row-major window order, the first of equal values stays, NaN wins) and split again.  One
// thread = one output position of one 8-channel unit.
__global__ void __launch_bounds__(256) plane_maxpool_terms_kernel(const uint4* __restrict__ in, int64_t planes, int H, int W,
                                                                  int k, int s, int pad, int OH, int OW, int terms,
                                                                  uint4* __restrict__ out) {
  const int64_t total = planes * OH * OW, in_vecs = planes * H * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int ow = (int)(idx % OW);
    const int64_t t = idx / OW;
    const int oh = (int)(t % OH);
    const uint4* src = in + (t / OH) * H * W;
    const int h0 = oh * s - pad, w0 = ow * s - pad;
    float m[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = -INFINITY;     // ATen's start value: the first window value always replaces it
    for (int i = max(h0, 0); i < min(h0 + k, H); ++i)
      for (int j = max(w0, 0); j < min(w0 + k, W); ++j) {
        const uint4* px = src + (int64_t)i * W + j;
        float v[8];
#pragma unroll
        for (int tm = 0; tm < 3; ++tm) {
          if (tm >= terms) break;
          const uint4 u = __ldg(px + (int64_t)tm * in_vecs);
          const float f[8] = {__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                              __uint_as_float(u.y & 0xffff0000u), __uint_as_float(u.z << 16), __uint_as_float(u.z & 0xffff0000u),
                              __uint_as_float(u.w << 16), __uint_as_float(u.w & 0xffff0000u)};
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = tm ? v[e] + f[e] : f[e];
        }
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (v[e] > m[e] || v[e] != v[e]) m[e] = v[e];
      }
    store_terms8(m, terms, out + idx, total);
  }
}

// eval BatchNorm [-> ReLU] [-> channel shuffle] of an fp32 NCHW tensor into the consumer's term planes (mnb_bn_relu_pack_terms_fwd):
// the op sequence of the XTERMS conv epilogue.  One thread = one position of one consumer 8-channel unit; a block's threads
// take consecutive positions, so each channel's loads coalesce.
__global__ void __launch_bounds__(256) bn_relu_pack_terms_kernel(const float* __restrict__ x, int batch, int channels, int hw,
                                                                 int sg, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, int relu, int terms,
                                                                 uint4* __restrict__ xp) {
  const int c8n = channels / 8, cpg = channels / sg;
  const int64_t total = (int64_t)batch * c8n * hw;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int pos = (int)(idx % hw);
    const int64_t t = idx / hw;
    const int oc8 = (int)(t % c8n), b = (int)(t / c8n);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int oc = oc8 * 8 + j;
      const int c = sg > 1 ? (oc % sg) * cpg + oc / sg : oc;   // inverse of out[:, a*sg + b] = in[:, b*cpg + a]
      float y = __ldg(x + ((int64_t)b * channels + c) * hw + pos);
      if (mean) y = fmaf(__fsub_rn(y, __ldg(mean + c)), __fmul_rn(__ldg(gamma + c), __ldg(invstd + c)), __ldg(beta + c));
      v[j] = relu ? fmaxf(y, 0.f) : y;
    }
    store_terms8(v, terms, xp + idx, total);
  }
}

// IAO QuantAdd of a frozen inference graph + the consuming conv's quantizer and operand packing in one pass (see
// mnb_quant_add_pack_fwd): one thread = one pixel of one 16-byte unit of the consumer's plane (CPU = 8 channels as bf16,
// or 16 channels as int8 for an int8 consumer), same arithmetic as quant_add_fwd_kernel (mnb_quant.cu) followed by
// pack_act_kernel<1> / pack_act_i8_kernel.
template <int CPU>
__global__ void __launch_bounds__(256) quant_add_pack_kernel(const float* __restrict__ a, const float* __restrict__ b, int B, int C,
                                                             int H, int W, int C8, mnb_act_qparams qadd, int relu,
                                                             float* __restrict__ out, mnb_act_qparams qnext, int next_relu,
                                                             int phase_split, uint4* __restrict__ out_pk) {
  const MnbActQ q = mnb_load_actq(qadd), qn = mnb_load_actq(qnext);
  const float zpn = (qnext.mode == MNB_ACT_IAO && qnext.zero_point) ? __ldg(qnext.zero_point) : 0.f;
  const uint32_t HW = (uint32_t)H * (uint32_t)W;
  const uint32_t plane = blockIdx.y * blockDim.y + threadIdx.y;                 // b * C8 + c8
  if (plane >= (uint32_t)B * (uint32_t)C8) return;
  const uint32_t bi = plane / (uint32_t)C8, c8 = plane - bi * (uint32_t)C8;
  for (uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x; pos < HW; pos += gridDim.x * blockDim.x) {
    const int64_t base = ((int64_t)bi * C + c8 * CPU) * HW + pos;
    float va[CPU], vb[CPU], lev[CPU];
#pragma unroll
    for (int j = 0; j < CPU; ++j) {
      const bool live = (int)c8 * CPU + j < C;
      va[j] = live ? __ldg(a + base + (int64_t)j * HW) : 0.f;
      vb[j] = live ? __ldg(b + base + (int64_t)j * HW) : 0.f;
    }
    // Q(a), Q(b): the level as a float (IAO: clamp(round(x/s - zp)), value = (level + zp) * s; DoReFa: value = level * s)
    float la[CPU], lb[CPU], sum[CPU];
    uint32_t pbits;
    mnb_act_levels<CPU>(q, va, la, pbits);
    mnb_act_levels<CPU>(q, vb, lb, pbits);
#pragma unroll
    for (int j = 0; j < CPU; ++j) {
      const bool live = (int)c8 * CPU + j < C;
      float oa, ob;
      if (q.mode == MNB_ACT_DOREFA) { oa = __fmul_rn(la[j], q.s); ob = __fmul_rn(lb[j], q.s); }
      else { oa = __fmul_rn(__fadd_rn(la[j], q.zp), q.s); ob = __fmul_rn(__fadd_rn(lb[j], q.zp), q.s); }
      float t = __fadd_rn(oa, ob);
      if (relu) t = fmaxf(t, 0.f);
      if (live) out[base + (int64_t)j * HW] = t;
      sum[j] = next_relu ? fmaxf(t, 0.f) : t;
    }
    mnb_act_levels<CPU>(qn, sum, lev, pbits);
#pragma unroll
    for (int j = 0; j < CPU; ++j) lev[j] = ((int)c8 * CPU + j < C) ? lev[j] + zpn : 0.f;
    int64_t dst;
    if (phase_split) {
      const uint32_t h = pos / (uint32_t)W, w = pos - h * (uint32_t)W;
      const uint32_t oct = ((h & 1u) * 2u + (w & 1u)) * (uint32_t)C8 + c8;
      dst = (((int64_t)bi * 4 * C8 + oct) * (H >> 1) + (h >> 1)) * (W >> 1) + (w >> 1);
    } else {
      dst = (int64_t)plane * HW + pos;
    }
    if constexpr (CPU == 16) out_pk[dst] = pack16_s8(lev);
    else out_pk[dst] = make_uint4(pack2(lev[0], lev[1]), pack2(lev[2], lev[3]), pack2(lev[4], lev[5]), pack2(lev[6], lev[7]));
  }
}

template <int VEC> struct PkVec;
template <> struct PkVec<1> { typedef float type; };
template <> struct PkVec<2> { typedef float2 type; };
template <> struct PkVec<4> { typedef float4 type; };

// Second pass of the fused BatchNorm + binarizer backward (mnb_bn_sign_bwd: dgamma / dbeta already reduced) that writes the
// gradient of the PRODUCING convolution's output directly as that convolution's packed operand: `terms` exact bf16 pieces
// of  dx * ch_scale[c]  in the plane layout [t][b][c/8][h][w][8] (and, optionally, plain fp32 dx).  The conv's data- and
// weight-gradient kernels then start from TMA loads; the separate pack pass (read 4 B, write 4 B per element) is gone.
//   dx = gamma * invstd * (g * pass - dbeta / N - xhat * dgamma / N)            (training-mode BatchNorm, saturate STE)
// One warp = 32 * VEC consecutive pixels of one channel octet (the conv's own channel order; g is read in the shuffled
// order); a lane owns VEC consecutive pixels: 16-byte loads of g and x (VEC = 4), one word of pass bits per channel, VEC
// consecutive 16-byte pixels per piece plane (one pixel per thread with 4-byte loads is far below HBM bandwidth).
// XT = int16_t (also in the pooled form below): x as a wbwtab conv's codes + decode pair `dec` (mnb_common.cuh x_load).
template <int VEC, typename XT>
__global__ void __launch_bounds__(256) bn_sign_bwd_pack_kernel(const float* __restrict__ g, const uint32_t* __restrict__ bits,
                                                               const XT* __restrict__ x, const float* __restrict__ dec,
                                                               int batch, int channels, int hw,
                                                               int sg, float inv_count, const float* __restrict__ mean,
                                                               const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                               const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                                                               const float* __restrict__ ch_scale, int terms,
                                                               float* __restrict__ dx, uint4* __restrict__ out, int64_t plane_vecs) {
  typedef typename PkVec<VEC>::type T;
  const int lane = threadIdx.x & 31;
  const int c8n = channels / 8, cpg = channels / sg, chunks = hw / (32 * VEC);
  const int64_t items = (int64_t)batch * c8n * chunks;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
    const int ch = (int)(w % chunks);
    const int64_t pl = w / chunks;                                // b * c8n + c8
    const int c8 = (int)(pl % c8n), b = (int)(pl / c8n);
    const int pos = (ch * 32 + lane) * VEC;
    T gv[8];
    float xf[8][VEC];
    uint32_t bw[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c8 * 8 + j;
      const int oc = sg > 1 ? (c % cpg) * sg + c / cpg : c;      // out[:, a*sg + b] = in[:, b*cpg + a]
      const int64_t fi = ((int64_t)b * channels + c) * hw + pos;
      gv[j] = __ldg(reinterpret_cast<const T*>(g + ((int64_t)b * channels + oc) * hw + pos));
      x_load<VEC>(x + fi, x_dec<XT>(dec, channels, c), xf[j]);
      bw[j] = __ldg(bits + (fi >> 5)) >> (fi & 31);              // bit i = pass flag of pixel pos + i
    }
    float v[VEC][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c8 * 8 + j;
      const float mu = __ldg(mean + c), is = __ldg(invstd + c), k = __ldg(gamma + c) * is;
      const float db = __ldg(dbeta + c) * inv_count, dg = __ldg(dgamma + c) * inv_count;
      const float sc = ch_scale ? __ldg(ch_scale + c) : 1.f;
      const float* gf = reinterpret_cast<const float*>(&gv[j]);
      T dv;
      float* df = reinterpret_cast<float*>(&dv);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float t = ((bw[j] >> i) & 1u) ? gf[i] : 0.f;
        t = bn_bwd_centre(t, db, (xf[j][i] - mu) * is, dg);
        t = k * t;
        df[i] = t;
        v[i][j] = ch_scale ? __fmul_rn(t, sc) : t;
      }
      if (dx) *reinterpret_cast<T*>(dx + ((int64_t)b * channels + c) * hw + pos) = dv;
    }
    const int64_t dst = pl * hw + pos;
    for (int tm = 0; tm < terms; ++tm) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        uint32_t pk4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          pk4[j] = pack2(v[i][2 * j], v[i][2 * j + 1]);
          v[i][2 * j] -= __uint_as_float(pk4[j] << 16);
          v[i][2 * j + 1] -= __uint_as_float(pk4[j] & 0xffff0000u);
        }
        out[(int64_t)tm * plane_vecs + dst + i] = make_uint4(pk4[0], pk4[1], pk4[2], pk4[3]);
      }
    }
  }
}

// The same for a producer with the 2x2 max-pool folded in (mnb_bn_sign_pool_*): second pass of its backward writing the
// full-resolution gradient of the producing conv's output as that conv's packed operand.  One lane = two horizontally
// adjacent pooling windows (4 x 2 pixels) of the 8 channels of one octet: per channel one float2 of the pooled gradient
// (read in the shuffled order), the two window arg-max bytes, the pass nibbles and two float4 of x; per piece plane two
// runs of 4 consecutive 16-byte pixels.  Layouts of arg / bits8 as written by bn_sign_pool_fwd_kernel (mnb_fused.cu).
template <typename XT>
__global__ void __launch_bounds__(256) bn_sign_pool_bwd_pack_kernel(const float2* __restrict__ g, const uchar2* __restrict__ arg,
                                                                    const uint8_t* __restrict__ bits8, const XT* __restrict__ x,
                                                                    const float* __restrict__ dec, int batch, int channels, int H, int W4, int sg, float inv_count,
                                                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                    const float* __restrict__ gamma, const float* __restrict__ dgamma,
                                                                    const float* __restrict__ dbeta, const float* __restrict__ ch_scale,
                                                                    int terms, uint4* __restrict__ out, int64_t plane_vecs) {
  const uint32_t OH = (uint32_t)H / 2u, OW2 = (uint32_t)W4, c8n = (uint32_t)channels / 8u, cpg = (uint32_t)channels / (uint32_t)sg;
  const uint32_t per_plane = OH * OW2;                                       // lane items per (image, channel) plane
  const int64_t total = (int64_t)batch * c8n * per_plane;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t rem = (uint32_t)(it % per_plane);
    const int64_t pl = it / per_plane;                                      // b * c8n + c8
    const uint32_t c8 = (uint32_t)(pl % c8n), b = (uint32_t)(pl / c8n);
    const uint32_t oh = rem / OW2, j = rem - oh * OW2;
    float v[8][8];                                                            // [pixel e: row (e >> 2), column (e & 3)][channel]
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint32_t c = c8 * 8u + q;
      const uint32_t oc = sg > 1 ? (c % cpg) * (uint32_t)sg + c / cpg : c;
      const uint32_t plane = b * (uint32_t)channels + c;
      const float2 gv = __ldg(g + ((size_t)(b * (uint32_t)channels + oc) * OH + oh) * OW2 + j);
      const uchar2 a = arg[((size_t)plane * OH + oh) * OW2 + j];
      const uint32_t i0 = (plane * (uint32_t)H + 2u * oh) * (uint32_t)W4 + j, i1 = i0 + (uint32_t)W4;
      const uint32_t n0 = (bits8[i0 >> 1] >> (4u * (i0 & 1u))) & 15u, n1 = (bits8[i1 >> 1] >> (4u * (i1 & 1u))) & 15u;
      const XDec d = x_dec<XT>(dec, channels, (int)c);
      const float4 r0 = x_load4(x + 4 * i0, d), r1 = x_load4(x + 4 * i1, d);
      const float mu = __ldg(mean + c), is = __ldg(invstd + c), k = __ldg(gamma + c) * is;
      const float db = __ldg(dbeta + c) * inv_count, dg = __ldg(dgamma + c) * inv_count;
      const float sc = ch_scale ? __ldg(ch_scale + c) : 1.f;
      const uint32_t e0 = (a.x >> 1) * 4u + (a.x & 1u), e1 = (a.y >> 1) * 4u + 2u + (a.y & 1u);
      const uint32_t nib = n0 | (n1 << 4);
      const float xs[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = 0.f;
        if ((uint32_t)e == e0 && ((nib >> e) & 1u)) t = gv.x;
        if ((uint32_t)e == e1 && ((nib >> e) & 1u)) t = gv.y;
        t = bn_bwd_centre(t, db, (xs[e] - mu) * is, dg);
        t = k * t;
        v[e][q] = ch_scale ? __fmul_rn(t, sc) : t;
      }
    }
    const int64_t dst0 = (pl * H + 2 * oh) * (int64_t)(4 * W4) + 4 * j;     // pixel (2 oh, 4 j) of this octet plane
    for (int tm = 0; tm < terms; ++tm) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        uint32_t pk4[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          pk4[q] = pack2(v[e][2 * q], v[e][2 * q + 1]);
          v[e][2 * q] -= __uint_as_float(pk4[q] << 16);
          v[e][2 * q + 1] -= __uint_as_float(pk4[q] & 0xffff0000u);
        }
        out[(int64_t)tm * plane_vecs + dst0 + (e >> 2) * (int64_t)(4 * W4) + (e & 3)] = make_uint4(pk4[0], pk4[1], pk4[2], pk4[3]);
      }
    }
  }
}

struct PackWParams {
  Plan pl;
  const int16_t* w_int; const float* w_f32; const float* kzero;   // kzero[k] == 0 -> the weights of channel k read as 0 (dgrad)
  int cin_g, cout_g;
};

// weights (int16 levels or fp32) -> bf16 image of the plan; one thread = one 16-byte vector (8 GEMM-K channels).
// CPU = 16: int16 levels in [-127, 127] -> int8 image [n-tile][group][stage][tap][c/16][n][16] (16 GEMM-K channels per vector).
template <int CPU>
__global__ void __launch_bounds__(256) pack_weight_kernel(const __grid_constant__ PackWParams pp, uint4* __restrict__ out) {
  const Plan& p = pp.pl;
  const int64_t total = p.wimg_bytes / 16;
  const int RS = p.R * p.S;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (int64_t)gridDim.x * blockDim.x) {
    int64_t byte = v * 16;
    int y = 0;
    for (int yy = 1; yy < p.ny; ++yy) if (byte >= p.y_off[yy]) y = yy;
    byte -= p.y_off[y];
    if (p.img_bytes[y] == 0) continue;
    const int ntg = (int)(byte / p.img_bytes[y]);
    int rem = (int)(byte - (int64_t)ntg * p.img_bytes[y]);
    if (ntg >= p.n_ntiles * p.G) continue;
    const int nt = ntg / p.G, g = ntg - nt * p.G;
    int t = 0;
    for (int tt = 1; tt < p.ntmpl[y]; ++tt) if (rem >= p.tmpl[y][tt].blk_off) t = tt;
    const Tmpl tp = p.tmpl[y][t];
    rem -= tp.blk_off;
    const int cc = rem / tp.blk_bytes;
    rem -= cc * tp.blk_bytes;
    const int per_tap = (p.CC / CPU) * p.Nt * 16, per_term = tp.ntap * per_tap;
    const int term = rem / per_term;
    rem -= term * per_term;
    const int tapi = rem / per_tap;
    rem -= tapi * per_tap;
    const int c8l = rem / (p.Nt * 16), n = (rem - c8l * (p.Nt * 16)) / 16;
    const int r = p.tap_r[y][tp.tap0 + tapi], s = p.tap_s[y][tp.tap0 + tapi];
    const int nn = nt * p.Nt + n;                 // GEMM-N channel within the group
    float val[CPU];
#pragma unroll
    for (int e = 0; e < CPU; ++e) {
      const int kk = cc * p.CC + c8l * CPU + e;   // GEMM-K channel within the group
      float x = 0.f;
      if (kk < p.kg && nn < p.ng) {
        int64_t src;
        int kout;
        if (p.mode == 0) { kout = g * pp.cout_g + nn; src = ((int64_t)kout * pp.cin_g + kk) * RS + r * p.S + s; }
        else { kout = g * pp.cout_g + kk; src = ((int64_t)kout * pp.cin_g + nn) * RS + r * p.S + s; }
        x = pp.w_int ? (float)__ldg(pp.w_int + src) : __ldg(pp.w_f32 + src);
        if (pp.kzero && __ldg(pp.kzero + kout) == 0.f) x = 0.f;
      }
      val[e] = x;
    }
    if constexpr (CPU == 16) {
      out[v] = pack16_s8(val);
    } else {
      uint32_t pk4[4];
      for (int tm = 0; tm <= term; ++tm) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          pk4[j] = pack2(val[2 * j], val[2 * j + 1]);
          val[2 * j] -= __uint_as_float(pk4[j] << 16);
          val[2 * j + 1] -= __uint_as_float(pk4[j] & 0xffff0000u);
        }
      }
      out[v] = make_uint4(pk4[0], pk4[1], pk4[2], pk4[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// the convolution kernel (forward and data gradient)
// ---------------------------------------------------------------------------------------------------------
struct ConvParams {
  // parameter block of the MMA warpgroups
  struct Mma {
    uint32_t n_items, chunks, ksteps, MT, Nt, npairs, st_mask, st_log2, stage16, a_mt16, a_term16, a_k16, b_off16,
        b_tap16, b_k16, a_lbo, b_lbo, seg_len;
    uint32_t ntmpl[MAXY];
    // The MMA "program": one 32-bit word per (filter tap, piece pair, K-step) of a stage template = A offset | B offset << 16
    // (16-byte units inside the stage); the issue loop is then  load word, two adds, MMA.
    uint16_t tmpl_begin[MAXY][MAXTMPL], tmpl_cnt[MAXY][MAXTMPL];   // in groups of four words
    alignas(16) uint4 prog4[MAXPROG / 4];                          // padded with 0xffffffff to whole groups
  } m;
  // TMA role
  int n_items, n_ntiles, G, MT, TA, chunks, CC8, C8A, kg8, stage_bytes, a_bytes, a_box_bytes, b_off, st_mask, st_log2;
  int Wt, TH, TB, wlo, hlo, col_tiles, row_tiles, n_mtiles;
  int ntmpl[MAXY], tmpl_kph[MAXY][MAXTMPL], tmpl_blk_off[MAXY][MAXTMPL], tmpl_blk_bytes[MAXY][MAXTMPL];
  int img_bytes[MAXY], y_off[MAXY];
  const uint8_t* w_img;
  // epilogue
  int B, THH, BW, OHr, OWr, OH, OW, omul, ny, ng, Nt, NOUT, C8O, smem_bytes, off_stg, mode;
  int dbg;                  // MNB_PK_DEBUG (timing experiments only): 1 no epilogue stores, 2 no MMAs
  const float* n_scale;     // [NOUT] per-output-channel scale or NULL
  const float* a_scale;     // device scalar multiplied into n_scale, or NULL
  float a_scale_const;
  const float* bias;        // [NOUT] or NULL
  const uint8_t* bits8;     // dgrad STE mask [B][C8O][OH][OW] or NULL
  float gain;               // dgrad: factor on passed gradients (DoReFa 0.1)
  float* out;               // fp32 NCHW result, or NULL when only the packed output below is wanted
  // int16 codes (mnb_pk_conv_codes, single-product forward plans only): the exact integer sums as NCHW int16 instead of out,
  // and dec[2][NOUT] = the (scale, bias) pair of the epilogue, so that a reader rebuilds out as fmaf(code, scale, bias)
  int16_t* codes;
  float* dec;
  // fused consumer (inference graphs): the epilogue also applies [ReLU +] the NEXT conv's activation quantizer and writes
  // that conv's operand plane [b][c/8][h][w][8] bf16, or [b][c/16][h][w][16] int8 in the int8 kernels (space-to-depth
  // phase planes for a stride-2 consumer; C8O = 16-byte units per position)
  uint4* post_out;
  mnb_act_qparams post_q;
  int post_relu, post_split;
  // eval BatchNorm between the conv and the consumer's [ReLU +] quantizer (all four or none) and the consumer block's
  // channel shuffle (post_sg > 1: producer channel c lands at consumer channel (c % cpg) * sg + c / cpg, cpg = NOUT / sg)
  const float *post_mean, *post_invstd, *post_gamma, *post_beta;
  int post_sg;
  int* err;
  // XTERMS instances (no consumer quantizer): the consumer's fp32 operand as post_terms exact bf16 pieces (after err, so
  // the parameter offsets of every other instance stay as they were)
  int post_terms;
};

struct alignas(16) ConvShared {
  uint64_t full[MAXST], empty[MAXST];
  uint32_t abort;
  alignas(16) float epi_scale[256];
  alignas(16) float epi_bias[256];
  uint16_t epi_dst[256];     // consumer channel of each channel of the N tile (shuffled consumer plane only)
};

template <int NEPI>
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NEPI) : "memory"); }

// n = q * d + r for n < 2^22 through one float multiply (the compiler's 32-bit integer division is a ~25-instruction dependent
// chain, and the TMA-issuing lane decodes every work item with it).  q from the reciprocal is within +-1: corrected exactly.
struct FastDiv {
  uint32_t d; float inv;
  __device__ __forceinline__ explicit FastDiv(int dd) : d((uint32_t)dd), inv(1.0f / (float)dd) {}
  __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const {
    q = __float2uint_rz(__uint2float_rz(n) * inv);
    r = n - q * d;
    if ((int32_t)r < 0) { --q; r += d; } else if (r >= d) { ++q; r -= d; }
  }
};

constexpr int kConvThreads = 384;   // warp 0 TMA, warps 4..11 two MMA + epilogue warpgroups (warps 1..3 idle)

// Warpgroup wg issues the wgmma of GEMM rows 64*wg .. 64*wg+63 of every M tile of the item (accumulators in registers:
// MT x NT / 2 per thread, plan: MT * Nt <= 128).  SEG: segmented accumulation (split fp32 operands): every segment of
// at most seg_len stages starts from zero and is added into running sums with round-to-nearest fp32 adds.
// Epilogue: 32 accumulator columns at a time through a 128 x 32 staging tile; thread et of the 256 then owns position
// (et % 128) of the tile raster and one 16-column slot (et / 128) of the two.
// I8: int8 operands (16 channels per 16-byte unit, s8 K32 MMAs into s32 accumulators, exact); the sums are converted to
// fp32 once (__int2float_rn) ahead of the same epilogue, and a consumer plane is written as int8.
// XPOST (forward with a consumer plane only): the consumer plane with an eval BatchNorm and / or a channel shuffle in front of
// the quantizer.  Instances of their own: with both epilogues in one instance the plain consumer plane's code (the IAO frozen
// graphs) loses registers to the other and ran 22-25% slower on frozen ResNet-18 (DESIGN.md 4.15).
// XTERMS (bf16 forward with a consumer plane only, no consumer quantizer): [eval BatchNorm] [-> ReLU] [-> shuffle] and the
// value's exact split into post_terms bf16 pieces, the term planes mnb_pk_pack_act writes from the same fp32 tensor (frozen
// wbwtab graphs with fp32 activations, DESIGN.md 4.20).  Instances of their own for the same reason.
template <bool SEG, int NT, bool I8 = false, bool XPOST = false, bool XTERMS = false>
__global__ void __launch_bounds__(kConvThreads, 1)
pk_conv_kernel(const __grid_constant__ CUtensorMap tmap0, const __grid_constant__ CUtensorMap tmap1,
               const __grid_constant__ CUtensorMap tmap2, const __grid_constant__ ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ ConvShared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < MAXST; ++i) { tc::mbar_init(&sh.full[i], 1); tc::mbar_init(&sh.empty[i], 8); }
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmap0);
    if (p.TA > 1) tc::prefetch_tmap(&tmap1);
    if (p.TA > 2) tc::prefetch_tmap(&tmap2);
  }
  // rows behind a box that only invalid accumulator rows read must at least be finite
  for (int i = tid; i < p.smem_bytes / 16; i += kConvThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp == 0) {
    // ================================================================= TMA producer
    if (lane == 0) {
      const int y = blockIdx.y;
      uint32_t sc = 0;
      const FastDiv d_nt(p.n_ntiles), d_g(p.G), d_ct(p.col_tiles), d_rt(p.row_tiles);
      for (int it = blockIdx.x; it < p.n_items; it += gridDim.x) {
        uint32_t nt, r1, g, mg;
        d_nt.divmod((uint32_t)it, r1, nt);
        d_g.divmod(r1, mg, g);
        const uint8_t* wsrc = p.w_img + (size_t)p.y_off[y] + (size_t)(nt * p.G + g) * (size_t)p.img_bytes[y];
        for (int t = 0; t < p.ntmpl[y]; ++t) {
          const int kph = p.tmpl_kph[y][t];
          const uint32_t blk = (uint32_t)p.tmpl_blk_bytes[y][t];
          const uint8_t* bsrc = wsrc + p.tmpl_blk_off[y][t];
          for (int cc = 0; cc < p.chunks; ++cc, ++sc) {
            const uint32_t slot = sc & (uint32_t)p.st_mask, ph = (sc >> p.st_log2) & 1u;
            if (!tc::mbar_wait(&sh.empty[slot], ph ^ 1u, p.err, 701)) goto done;
            // MNB_PK_DEBUG bits 8 / 16 (timing experiments only): leave out the activation boxes / the weight block
            const bool ld_a = !(p.dbg & 8), ld_b = !(p.dbg & 16);
            tc::mbar_arrive_expect_tx(&sh.full[slot], (ld_a ? (uint32_t)(p.MT * p.TA * p.a_box_bytes) : 0u) + (ld_b ? blk : 0u));
            uint8_t* sbase = smem + (size_t)slot * p.stage_bytes;
            const int c8 = kph * p.C8A + g * p.kg8 + cc * p.CC8;
            for (int mt = 0; mt < (ld_a ? p.MT : 0); ++mt) {
              const uint32_t tile = mg * (uint32_t)p.MT + (uint32_t)mt;
              uint32_t ct, r2, rt, bt;
              d_ct.divmod(tile, r2, ct);
              d_rt.divmod(r2, bt, rt);
              const int cw = (int)ct * p.Wt - p.wlo, chh = (int)rt * p.TH - p.hlo, cb = (int)bt * p.TB;
              tc::tma_load_4d(sbase + (size_t)(mt * p.TA) * p.a_bytes, &tmap0, &sh.full[slot], 2 * cw, chh, cb, c8);
              if (p.TA > 1) tc::tma_load_4d(sbase + (size_t)(mt * p.TA + 1) * p.a_bytes, &tmap1, &sh.full[slot], 2 * cw, chh, cb, c8);
              if (p.TA > 2) tc::tma_load_4d(sbase + (size_t)(mt * p.TA + 2) * p.a_bytes, &tmap2, &sh.full[slot], 2 * cw, chh, cb, c8);
            }
            if (ld_b) tc::bulk_load_1d(sbase + p.b_off, bsrc + (size_t)cc * blk, blk, &sh.full[slot]);
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ================================================================= MMA warpgroups + epilogue
    constexpr int NEPI = 256, NR = NT / 2, MAXMT = 128 / NT;
    const int wg = (warp - 4) >> 2, et = tid - 128;
    const int m = et & 127, half = et >> 7;          // epilogue: accumulator row (= tile raster position), slot parity
    float* stage = reinterpret_cast<float*>(smem + p.off_stg);
    const int tb = m / (p.THH * p.BW);
    const int rem = m - tb * (p.THH * p.BW);
    const int th = rem / p.BW, wc = rem - th * p.BW;
    const bool row_ok = tb < p.TB && th < p.TH && wc < p.Wt;
    const int y = blockIdx.y, ya = p.ny == 4 ? (y >> 1) : 0, yb = p.ny == 4 ? (y & 1) : 0;
    const int64_t plane = (int64_t)p.OH * p.OW;
    const float a_sc = p.a_scale ? __ldg(p.a_scale) : p.a_scale_const;
    MnbActQ pq;
    float pzp = 0.f;
    if (!XTERMS && p.post_out) {
      pq = mnb_load_actq(p.post_q);
      if (p.post_q.mode == MNB_ACT_IAO && p.post_q.zero_point) pzp = __ldg(p.post_q.zero_point);
    }
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), p.m.a_lbo, 128) + (uint64_t)(64 * wg);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), p.m.b_lbo, 128) + (uint64_t)p.m.b_off16;
    const uint32_t a_lo0 = (uint32_t)a_desc0, b_lo0 = (uint32_t)b_desc0;
    const uint64_t a_hi = a_desc0 & 0xffffffff00000000ull, b_hi = b_desc0 & 0xffffffff00000000ull;
    uint32_t sc = 0;
    const FastDiv e_nt(p.n_ntiles), e_g(p.G), e_ct(p.col_tiles), e_rt(p.row_tiles);
    for (int it = blockIdx.x; it < p.n_items; it += gridDim.x) {
      uint32_t nt_u, r1_u, g_u, mg_u;
      e_nt.divmod((uint32_t)it, r1_u, nt_u);
      e_g.divmod(r1_u, mg_u, g_u);
      const int nt = (int)nt_u, g = (int)g_u, mg = (int)mg_u;
      const int n_base = g * p.ng + nt * p.Nt;                // first output channel of this N tile
      const int n_cnt = min(p.Nt, p.ng - nt * p.Nt);
      // per-channel constants of this N tile (the previous item's readers are done: barrier at the end of the loop body)
      for (int n = et; n < p.Nt; n += NEPI) {
        float scv = 1.f, bs = 0.f;
        if (n < n_cnt) {
          scv = p.n_scale ? __fmul_rn(a_sc, __ldg(p.n_scale + n_base + n)) : a_sc;
          if (p.bias) bs = __ldg(p.bias + n_base + n);
        }
        sh.epi_scale[n] = scv; sh.epi_bias[n] = bs;
        if constexpr (XPOST || XTERMS) {
          if (p.post_sg > 1 && n < n_cnt) {
            const int c = n_base + n, cpg = p.NOUT / p.post_sg;
            sh.epi_dst[n] = (uint16_t)((c % cpg) * p.post_sg + c / cpg);
          }
        }
        if constexpr (!SEG && !I8) {   // one snapshot of the decode pair: from the items of M group 0
          if (p.dec && mg == 0 && y == 0 && n < n_cnt) { p.dec[n_base + n] = scv; p.dec[p.NOUT + n_base + n] = bs; }
        }
      }
      // ---- MMAs of the item: every stage of every template, all M tiles
      float acc[MAXMT][NR];
      float rs[SEG ? MAXMT : 1][SEG ? NR : 1];
#pragma unroll
      for (int mt = 0; mt < MAXMT; ++mt) tc::zero_acc(acc[mt]);
      if (SEG) {
#pragma unroll
        for (int mt = 0; mt < MAXMT; ++mt) tc::zero_acc(rs[mt]);
      }
      uint32_t seg_pos = 0;
      for (uint32_t t = 0; t < p.m.ntmpl[y]; ++t) {
        const uint32_t pb = p.m.tmpl_begin[y][t], pc = p.m.tmpl_cnt[y][t];
        for (uint32_t cc = 0; cc < p.m.chunks; ++cc, ++sc) {
          const uint32_t slot = sc & p.m.st_mask, ph = (sc >> p.m.st_log2) & 1u;
          tc::mbar_wait_soft(&sh.full[slot], ph, p.err, 703, &sh.abort);
          const uint32_t s16 = slot * p.m.stage16;
          tc::wg_fence();
#pragma unroll
          for (int mt = 0; mt < MAXMT; ++mt) tc::fence_acc(acc[mt]);
          if (!(p.dbg & 2)) {
#pragma unroll
            for (int mt = 0; mt < MAXMT; ++mt) {
              if (mt >= (int)p.m.MT) break;
              const uint32_t a_base = a_lo0 + s16 + (uint32_t)mt * p.m.a_mt16, b_base = b_lo0 + s16;
              // flat program: one word per MMA of this stage template (tap x piece pair x K-step) = A offset | B offset << 16,
              // padded with 0xffffffff to groups of four
              for (uint32_t e = 0; e < pc; ++e) {
                const uint4 w4 = p.m.prog4[pb + e];
                const uint32_t w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  if (w[k] == 0xffffffffu) continue;
                  if constexpr (I8)   // s32 accumulators in the registers of acc (zero bits = 0 either way)
                    tc::Mma<NT>::s8(reinterpret_cast<int32_t(&)[NR]>(acc[mt]), a_hi | (uint64_t)(a_base + (w[k] & 0xffffu)),
                                    b_hi | (uint64_t)(b_base + (w[k] >> 16)), 1);
                  else
                    tc::Mma<NT>::template bf16<0, 0>(acc[mt], a_hi | (uint64_t)(a_base + (w[k] & 0xffffu)),
                                                      b_hi | (uint64_t)(b_base + (w[k] >> 16)), 1);
                }
              }
            }
          }
          tc::wg_commit();
          tc::wg_wait<0>();
#pragma unroll
          for (int mt = 0; mt < MAXMT; ++mt) tc::fence_acc(acc[mt]);
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(&sh.empty[slot]);   // this warp's reads of the stage are done
          if (SEG && ++seg_pos == p.m.seg_len) {            // segment complete: into the running sums
            seg_pos = 0;
#pragma unroll
            for (int mt = 0; mt < MAXMT; ++mt) {
#pragma unroll
              for (int i = 0; i < NR; ++i) { rs[SEG ? mt : 0][SEG ? i : 0] = __fadd_rn(rs[SEG ? mt : 0][SEG ? i : 0], acc[mt][i]); acc[mt][i] = 0.f; }
            }
          }
        }
      }
      if (SEG) {   // the last (partial) segment
#pragma unroll
        for (int mt = 0; mt < MAXMT; ++mt) {
#pragma unroll
          for (int i = 0; i < NR; ++i) rs[SEG ? mt : 0][SEG ? i : 0] = __fadd_rn(rs[SEG ? mt : 0][SEG ? i : 0], acc[mt][i]);
        }
      }
      if constexpr (I8) {   // exact s32 sums -> fp32, rounded once (exact below 2^24, where the bf16 kernels agree)
#pragma unroll
        for (int mt = 0; mt < MAXMT; ++mt) {
#pragma unroll
          for (int i = 0; i < NR; ++i) acc[mt][i] = __int2float_rn(__float_as_int(acc[mt][i]));
        }
      }
      // ---- epilogue
      int mt_cur = -1;
      bool valid = false;
      int64_t orow = 0;      // element offset of this thread's output position in channel n_base of out / codes
      const uint8_t* brow = nullptr;
      int64_t prow = 0;      // vector index of this thread's position in octet 0 of the consumer's operand plane
      // one slot = 16 accumulator columns of one M tile
      auto do_slot = [&](const int mt, const int c16, const float (&r)[16]) {
        const int n0 = c16 * 16;
        if (mt != mt_cur) {   // output row of this thread in M tile mt
          mt_cur = mt;
          const int tile = mg * p.MT + mt;
          uint32_t ct_u, r2_u, rt_u, bt_u;
          e_ct.divmod((uint32_t)tile, r2_u, ct_u);
          e_rt.divmod(r2_u, bt_u, rt_u);
          const int ct = (int)ct_u, rt = (int)rt_u, bt = (int)bt_u;
          const int b = bt * p.TB + tb, i = rt * p.TH + th, j = ct * p.Wt + wc;
          valid = row_ok && tile < p.n_mtiles && b < p.B && i < p.OHr && j < p.OWr;
          const int oh = i * p.omul + ya, ow = j * p.omul + yb;
          orow = ((int64_t)b * p.NOUT + n_base) * plane + (int64_t)oh * p.OW + ow;
          brow = p.bits8 ? p.bits8 + (int64_t)b * p.C8O * plane + (int64_t)oh * p.OW + ow : nullptr;
          if (p.post_out) {
            if (p.post_split)   // octet index (h%2 * 2 + w%2) * C8 + c/8 of a [.., OH/2, OW/2] plane
              prow = (((int64_t)b * 4 * p.C8O + ((oh & 1) * 2 + (ow & 1)) * p.C8O) * (p.OH >> 1) + (oh >> 1)) * (p.OW >> 1) + (ow >> 1);
            else
              prow = ((int64_t)b * p.C8O * p.OH + oh) * p.OW + ow;
          }
        }
        if (!valid || n0 >= n_cnt || (p.dbg & 1)) return;
        if (!SEG && !I8 && p.codes) {   // exact integer sums (|r| <= 32767: checked on the host) as int16
          int16_t* cp = p.codes + orow + (int64_t)n0 * plane;
#pragma unroll
          for (int k = 0; k < 16; ++k, cp += plane)
            if (n0 + k < n_cnt) *cp = (int16_t)__float2int_rn(r[k]);
          return;
        }
        if constexpr (XTERMS) {
          // one 8-channel unit at a time (C_out per group % 8 == 0, refused otherwise on the host: an octet is all valid or
          // all past the tile): the value after [BatchNorm] [ReLU], split into pieces exactly as pack_act_body splits an
          // fp32 tensor
          float* op0 = p.out + orow + (int64_t)n0 * plane;
          const int64_t oct_stride = p.post_split ? (int64_t)(p.OH >> 1) * (p.OW >> 1) : plane;
          const int64_t term_vecs = (int64_t)p.B * p.C8O * plane;     // 16-byte units per term plane
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            if (n0 + 8 * o >= n_cnt) break;
            float v[8];
#pragma unroll
            for (int h4 = 0; h4 < 2; ++h4) {
              const int k0 = 8 * o + 4 * h4;
              const float4 sc4 = *reinterpret_cast<const float4*>(&sh.epi_scale[n0 + k0]);
              const float4 bs4 = *reinterpret_cast<const float4*>(&sh.epi_bias[n0 + k0]);
              const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, bsv[4] = {bs4.x, bs4.y, bs4.z, bs4.w};
              float mu[4] = {0.f, 0.f, 0.f, 0.f}, gs[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
              if (p.post_mean) {   // 16-byte aligned arrays, C_out % 4 == 0 (checked on the host)
                const int c0 = n_base + n0 + k0;
                const float4 m4 = __ldg(reinterpret_cast<const float4*>(p.post_mean + c0));
                const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.post_gamma + c0));
                const float4 i4 = __ldg(reinterpret_cast<const float4*>(p.post_invstd + c0));
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.post_beta + c0));
                mu[0] = m4.x; mu[1] = m4.y; mu[2] = m4.z; mu[3] = m4.w;
                gs[0] = __fmul_rn(g4.x, i4.x); gs[1] = __fmul_rn(g4.y, i4.y); gs[2] = __fmul_rn(g4.z, i4.z); gs[3] = __fmul_rn(g4.w, i4.w);
                be[0] = b4.x; be[1] = b4.y; be[2] = b4.z; be[3] = b4.w;
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float t = fmaf(r[k0 + j], scv[j], bsv[j]);
                if (p.out) op0[(int64_t)(k0 + j) * plane] = t;
                if (p.post_mean) t = fmaf(__fsub_rn(t, mu[j]), gs[j], be[j]);
                v[4 * h4 + j] = p.post_relu ? fmaxf(t, 0.f) : t;
              }
            }
            if (p.post_sg > 1) {   // consecutive channels land in different consumer units: one element at a time
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int oc = sh.epi_dst[n0 + 8 * o + j];
                __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.post_out) + (prow + (int64_t)(oc >> 3) * oct_stride) * 8 + (oc & 7);
                float t = v[j];
                for (int tm = 0; tm < p.post_terms; ++tm) {
                  const uint32_t w = pack2(t, 0.f);
                  dst[(int64_t)tm * term_vecs * 8] = __ushort_as_bfloat16((unsigned short)(w & 0xffffu));
                  t -= __uint_as_float(w << 16);
                }
              }
            } else {
              store_terms8(v, p.post_terms, p.post_out + prow + (int64_t)(((n_base + n0) >> 3) + o) * oct_stride, term_vecs);
            }
          }
          return;
        }
        if constexpr (XPOST) {
          float* op0 = p.out + orow + (int64_t)n0 * plane;
          // consumer plane with an eval BatchNorm in front of the [ReLU +] quantizer (the op sequence of
          // bn_relu_quant_pack_kernel) and / or the consumer block's channel shuffle.  Four chunks of four channels (the
          // quantizer is elementwise) with the packed words carried over: few values are live at a time, which keeps these
          // instances free of spills.
          const int64_t oct_stride = p.post_split ? (int64_t)(p.OH >> 1) * (p.OW >> 1) : plane;
          uint32_t pw[4];     // packed words of the current 16-byte unit (bf16: 8 channels, int8: 16 channels)
#pragma unroll
          for (int qc = 0; qc < 4; ++qc) {
            if (!I8 && qc >= 2 && n0 + 8 >= n_cnt) break;
            float lev[4], yv[4];
            // 16-byte loads of the chunk's per-channel constants (BatchNorm arrays: 16-byte aligned, C_out % 4 == 0, checked
            // on the host; a chunk past the tile's last channel re-reads the first one)
            const float4 sc4 = *reinterpret_cast<const float4*>(&sh.epi_scale[n0 + 4 * qc]);
            const float4 bs4 = *reinterpret_cast<const float4*>(&sh.epi_bias[n0 + 4 * qc]);
            const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, bsv[4] = {bs4.x, bs4.y, bs4.z, bs4.w};
            float mu[4] = {0.f, 0.f, 0.f, 0.f}, gs[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
            if (p.post_mean) {
              const int c0 = n_base + n0 + (n0 + 4 * qc < n_cnt ? 4 * qc : 0);
              const float4 m4 = __ldg(reinterpret_cast<const float4*>(p.post_mean + c0));
              const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.post_gamma + c0));
              const float4 i4 = __ldg(reinterpret_cast<const float4*>(p.post_invstd + c0));
              const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.post_beta + c0));
              mu[0] = m4.x; mu[1] = m4.y; mu[2] = m4.z; mu[3] = m4.w;
              gs[0] = __fmul_rn(g4.x, i4.x); gs[1] = __fmul_rn(g4.y, i4.y); gs[2] = __fmul_rn(g4.z, i4.z); gs[3] = __fmul_rn(g4.w, i4.w);
              be[0] = b4.x; be[1] = b4.y; be[2] = b4.z; be[3] = b4.w;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int k = 4 * qc + j;
              float v = fmaf(r[k], scv[j], bsv[j]);
              if (p.out && n0 + k < n_cnt) op0[(int64_t)k * plane] = v;
              if (p.post_mean) v = fmaf(__fsub_rn(v, mu[j]), gs[j], be[j]);
              yv[j] = p.post_relu ? fmaxf(v, 0.f) : v;
            }
            uint32_t passbits;
            mnb_act_levels<4>(pq, yv, lev, passbits);
#pragma unroll
            for (int j = 0; j < 4; ++j) lev[j] = n0 + 4 * qc + j < n_cnt ? lev[j] + pzp : 0.f;
            if (p.post_sg > 1) {   // consecutive channels land in different consumer units: one element at a time
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (n0 + 4 * qc + j >= n_cnt) continue;
                const int oc = sh.epi_dst[n0 + 4 * qc + j];
                if constexpr (I8)
                  reinterpret_cast<int8_t*>(p.post_out)[(prow + (int64_t)(oc >> 4) * oct_stride) * 16 + (oc & 15)] =
                      (int8_t)__float2int_rn(lev[j]);
                else
                  reinterpret_cast<__nv_bfloat16*>(p.post_out)[(prow + (int64_t)(oc >> 3) * oct_stride) * 8 + (oc & 7)] =
                      __float2bfloat16_rn(lev[j]);
              }
            } else if constexpr (I8) {   // one 16-channel unit (n_base + n0 is a multiple of 16: checked on the host)
              pw[qc] = pack4_s8(lev[0], lev[1], lev[2], lev[3]);
              if (qc == 3) p.post_out[prow + (int64_t)((n_base + n0) >> 4) * oct_stride] = make_uint4(pw[0], pw[1], pw[2], pw[3]);
            } else {
              pw[2 * (qc & 1)] = pack2(lev[0], lev[1]);
              pw[2 * (qc & 1) + 1] = pack2(lev[2], lev[3]);
              if (qc & 1)
                p.post_out[prow + (int64_t)(((n_base + n0) >> 3) + (qc >> 1)) * oct_stride] = make_uint4(pw[0], pw[1], pw[2], pw[3]);
            }
          }
          return;
        }
        float sc[16], bs[16];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const float4 a = *reinterpret_cast<const float4*>(&sh.epi_scale[n0 + 4 * v]);
          const float4 c = *reinterpret_cast<const float4*>(&sh.epi_bias[n0 + 4 * v]);
          sc[4 * v] = a.x; sc[4 * v + 1] = a.y; sc[4 * v + 2] = a.z; sc[4 * v + 3] = a.w;
          bs[4 * v] = c.x; bs[4 * v + 1] = c.y; bs[4 * v + 2] = c.z; bs[4 * v + 3] = c.w;
        }
        float* op = p.out + orow + (int64_t)n0 * plane;
        if (!SEG && p.post_out) {   // (the host refuses a consumer plane on segmented plans)
          // forward conv of a frozen inference graph: y = acc * scale + bias [-> ReLU] -> consumer's quantizer -> bf16 levels
          float lev[16], yv[16];
#pragma unroll
          for (int k = 0; k < 16; ++k) {
            const float v = fmaf(r[k], sc[k], bs[k]);
            if (p.out && n0 + k < n_cnt) op[(int64_t)k * plane] = v;
            yv[k] = p.post_relu ? fmaxf(v, 0.f) : v;
          }
          uint32_t passbits;
          mnb_act_levels<16>(pq, yv, lev, passbits);
#pragma unroll
          for (int k = 0; k < 16; ++k) lev[k] = n0 + k < n_cnt ? lev[k] + pzp : 0.f;
          const int64_t oct_stride = p.post_split ? (int64_t)(p.OH >> 1) * (p.OW >> 1) : plane;
          if constexpr (I8) {   // one 16-channel unit (n_base + n0 is a multiple of 16: checked on the host)
            p.post_out[prow + (int64_t)((n_base + n0) >> 4) * oct_stride] = pack16_s8(lev);
          } else {
            const int oc8 = (n_base + n0) >> 3;
            uint4* dst = p.post_out + prow + (int64_t)oc8 * oct_stride;
            dst[0] = make_uint4(pack2(lev[0], lev[1]), pack2(lev[2], lev[3]), pack2(lev[4], lev[5]), pack2(lev[6], lev[7]));
            if (n0 + 8 < n_cnt)
              dst[oct_stride] = make_uint4(pack2(lev[8], lev[9]), pack2(lev[10], lev[11]), pack2(lev[12], lev[13]), pack2(lev[14], lev[15]));
          }
        } else if (p.mode == 0 || !brow) {
#pragma unroll
          for (int k = 0; k < 16; ++k, op += plane)
            if (n0 + k < n_cnt) *op = fmaf(r[k], sc[k], bs[k]);
        } else {
          // STE of the activation quantizer that fed the forward conv: the reference computes ((g*s)*pass)/s (IAO) or
          // (((g*s)/s)*pass)*0.1 (DoReFa); (g*s)/s is g to within one ulp, so g itself is passed
          // mask octet of channel nt * Nt + n0 of group g (a multiple of 8) in the group-padded mask: C8O / G octets per group
          // (the int8 instances run forward plans only)
          const int oc0 = I8 ? (n_base + n0) >> 3 : g * (p.C8O / p.G) + ((nt * p.Nt + n0) >> 3);
          const uint32_t m0 = __ldg(brow + (int64_t)oc0 * plane);
          const uint32_t m1 = (n0 + 8 < n_cnt) ? __ldg(brow + (int64_t)(oc0 + 1) * plane) : 0u;
          const uint32_t mask = m0 | (m1 << 8);
#pragma unroll
          for (int k = 0; k < 16; ++k, op += plane)
            if (n0 + k < n_cnt) *op = ((mask >> k) & 1u) ? r[k] * p.gain : 0.f;
        }
      };
      // columns of the item in M-tile-major order: L = mt * NT + n; round rnd stages L in [32 rnd, 32 rnd + 32)
      const int ncols = (int)p.m.MT * NT;
#pragma unroll
      for (int rnd = 0; rnd < (MAXMT * NT + 31) / 32; ++rnd) {
        if (32 * rnd >= ncols) break;
        epi_bar_sync<NEPI>();   // every thread is done with the previous staging tile (and, first round, epi_scale is written)
#pragma unroll
        for (int mt = 0; mt < MAXMT; ++mt) {
          const int lo = mt * NT > 32 * rnd ? mt * NT : 32 * rnd;
          const int hi = (mt + 1) * NT < 32 * rnd + 32 ? (mt + 1) * NT : 32 * rnd + 32;
          if (lo >= hi) continue;
          float* dst = stage + (lo - 32 * rnd) * tc::kStageLd;
          if constexpr (SEG) tc::frag_cols_to_smem(rs[mt], dst, tc::kStageLd, 64 * wg, lo - mt * NT, hi - lo);
          else tc::frag_cols_to_smem(acc[mt], dst, tc::kStageLd, 64 * wg, lo - mt * NT, hi - lo);
        }
        epi_bar_sync<NEPI>();
        const int L0 = 32 * rnd + 16 * half;
        if (L0 < ncols) {
          float r[16];
#pragma unroll
          for (int k = 0; k < 16; ++k) r[k] = stage[(16 * half + k) * tc::kStageLd + m];
          do_slot(L0 / NT, (L0 % NT) >> 4, r);
        }
      }
      epi_bar_sync<NEPI>();   // everyone is done with epi_scale / epi_bias and the staging tile of this item
    }
  }
done:
  __syncthreads();
}

// Map over term plane `t` of a packed tensor [b][octet][h][w][8 x bf16].  The TMA unit's cost is per box ROW whatever
// its length (with the 16-byte channel octet as innermost dimension every position would be a row), so the 16-byte pixels
// of one image row are declared as ONE dimension of 8-byte elements:
// dims (2*W, H, B, octets), box (2*BW, rows, images, octets) - same shared-memory image [octet][image][row][col][16 B],
// halo columns still zero-filled (start coordinate -2*wlo: a multiple of 16 bytes).
static int make_pk_tmap(CUtensorMap* m, const void* base, int64_t plane_bytes, int t, int B, int C8tot, int H, int W,
                        int bw, int bh, int bb, int bc8) {
  const uint64_t HW = (uint64_t)H * W;
  uint64_t dims[4] = {(uint64_t)W * 2, (uint64_t)H, (uint64_t)B, (uint64_t)C8tot};
  uint64_t strides[3] = {(uint64_t)W * 16, (uint64_t)C8tot * HW * 16, HW * 16};
  uint32_t box[4] = {(uint32_t)bw * 2, (uint32_t)bh, (uint32_t)bb, (uint32_t)bc8};
  return mnb_make_tmap_strided(m, reinterpret_cast<const uint8_t*>(base) + (int64_t)t * plane_bytes, 8, 4, dims, strides, box);
}

template <typename K>
static int set_max_smem(K kernel, int bytes) {
  // the attribute is a property of the function on a device: set it once per (function, device).  Keyed by the function
  // ADDRESS (instantiations of one template share their pointer TYPE, so a per-type static would cover only the first)
  static const void* seen_fn[32];
  static int seen_dev[32], nseen = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const void* fn = reinterpret_cast<const void*>(kernel);
  for (int i = 0; i < nseen; ++i)
    if (seen_fn[i] == fn && seen_dev[i] == dev) return 0;
  cudaError_t ce = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
  if (nseen < 32) { seen_fn[nseen] = fn; seen_dev[nseen] = dev; ++nseen; }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// weight gradient: dW[k][c][tap] = sum over positions of dy[pos][k] * x[pos + tap][c]   (MN-major operands)
// ---------------------------------------------------------------------------------------------------------
struct WgPlan {
  int B, G, R, S, stride, ntap;
  int P, Q, K8, HX, WX, C8X, nkph;      // dy dims / octets; x planes as stored
  int cin_g, cout_g, gm;       // plane channels per (merged) group; gm = original groups per merged group
  int cin_o, cout_o;           // channels per original group
  int hlo, hhi, wlo, whi, BW, TH, THH, rows_dy, rows_x, row_tiles;
  int Nc, n_ctiles, n_ktiles, tpg, n_tg, NI, nsub, nstg_total, splits, stg_per_split;
  int TA, TX, npairs, pair_a[MAXPAIR], pair_b[MAXPAIR];
  int tap_kph[MAXTAP], tap_off[MAXTAP];   // per tap: k-phase plane and start-row offset in the x block
  int kph_used[4], nkph_used, kph_slot[4];
  int dy_box_bytes, x_box_bytes, dy_bytes, x_bytes, sub_bytes, stage_bytes, nstage, st_log2, smem_bytes;
  int64_t partial_floats;
};

constexpr int kWgProg4 = MAXPAIR * MAXTAP / 4 + MAXPAIR * 16;   // uint4 entries of the wgrad issue program (WgParams)

static int make_wg_plan_nc(const mnb_conv_shape* s, int TA, int TX, WgPlan& p, int nc_cap) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  memset(&p, 0, sizeof(p));
  const int C = s->in_c, K = s->out_c, G = s->groups, H = s->in_h, W = s->in_w, R = s->ker_h, S = s->ker_w;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && H > 0 && W > 0 && G > 0 && C % G == 0 && K % G == 0, "bad conv shape");
  if (s->dil_h != 1 || s->dil_w != 1) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: dilation != 1");
  if (s->stride_h != s->stride_w || (s->stride_h != 1 && s->stride_h != 2)) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: stride");
  const int st = s->stride_h, ph_ = s->pad_h, pw_ = s->pad_w;
  if (ph_ > R - 1 || pw_ > S - 1) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: padding larger than the filter");
  if (st == 2 && ((H | W) & 1)) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: stride 2 needs even H and W");
  if (R * S > MAXTAP) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: more than 64 taps");
  p.B = s->batch; p.G = G; p.R = R; p.S = S; p.stride = st; p.ntap = R * S;
  p.P = (H + 2 * ph_ - R) / st + 1; p.Q = (W + 2 * pw_ - S) / st + 1;
  if (p.P < 1 || p.Q < 1) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: empty output");
  p.cin_o = C / G; p.cout_o = K / G;
  // group-padded planes (DESIGN.md 4.17): a group spans round_up(channels per group, 8) plane channels on either side
  p.cin_g = G > 1 ? round_up(p.cin_o, 8) : p.cin_o; p.cout_g = G > 1 ? round_up(p.cout_o, 8) : p.cout_o;
  // Small groups are MERGED: gm neighbouring groups form one 128-row accumulator block (rows = their output channels,
  // columns = their input channels); a narrow MMA uses the tensor core poorly, so computing the discarded off-diagonal
  // blocks costs little and the MMA count drops by gm.  The reduction kernel keeps the diagonal blocks only.
  p.gm = 1;
  while (G % (p.gm * 2) == 0 && p.gm * 2 * p.cout_g <= 128 && p.gm * 2 * p.cin_g <= 128) p.gm *= 2;
  if (const char* e = getenv("MNB_PK_WG_MERGE")) { if (atoi(e) == 0) p.gm = 1; }
  p.G = G / p.gm; p.cin_g *= p.gm; p.cout_g *= p.gm;
  p.K8 = ceil_div(p.G * p.cout_g, 8); p.C8X = ceil_div(p.G * p.cin_g, 8);
  p.nkph = st == 2 ? 4 : 1; p.HX = H / st; p.WX = W / st;
  p.TA = TA; p.TX = TX;
  { Plan tmp; memset(&tmp, 0, sizeof(tmp)); make_pairs(TA, TX, tmp); p.npairs = tmp.npairs;
    for (int i = 0; i < tmp.npairs; ++i) { p.pair_a[i] = tmp.pair_a[i]; p.pair_b[i] = tmp.pair_b[i]; } }
  int sh_[MAXTAP], sw_[MAXTAP];
  int hlo = 0, hhi = 0, wlo = 0, whi = 0;
  for (int i = 0; i < 4; ++i) p.kph_slot[i] = -1;
  for (int r = 0; r < R; ++r)
    for (int q = 0; q < S; ++q) {
      const int t = r * S + q, dr = r - ph_, ds = q - pw_;
      int kp = 0, sh = dr, sw = ds;
      if (st == 2) { const int fh = dr & 1, fw = ds & 1; kp = fh * 2 + fw; sh = (dr - fh) / 2; sw = (ds - fw) / 2; }
      p.tap_kph[t] = kp; sh_[t] = sh; sw_[t] = sw;
      if (p.kph_slot[kp] < 0) { p.kph_slot[kp] = p.nkph_used; p.kph_used[p.nkph_used++] = kp; }
      hlo = std::max(hlo, -sh); hhi = std::max(hhi, sh); wlo = std::max(wlo, -sw); whi = std::max(whi, sw);
    }
  p.hlo = hlo; p.hhi = hhi; p.wlo = wlo; p.whi = whi;
  // raster: rows of BW >= Q + halo columns; TH * BW must be a multiple of 16 (MMA K-steps of 16 positions)
  const int need = p.Q + wlo + whi;
  if (need > 128) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: row wider than 128 positions");
  // N tile over input channels and TAP GROUPS: one CTA accumulates tpg taps x Nc columns (tpg x Nc <= 128: registers).
  // Wide MMAs use the tensor core best, so the N tile is made as wide as the layer allows (up to 128) and the taps are split
  // over CTAs instead (each tap group re-reads the operands, mostly from L2).
  int nc = std::min(nc_cap, round_up(p.cin_g, 16));
  if (const char* e = getenv("MNB_PK_WG_NC")) nc = std::max(16, std::min(nc, atoi(e) / 16 * 16));
  p.n_ctiles = ceil_div(p.cin_g, nc);
  p.Nc = round_up(ceil_div(p.cin_g, p.n_ctiles), 16);      // balance the tiles
  p.n_ctiles = ceil_div(p.cin_g, p.Nc);
  p.n_ktiles = ceil_div(p.cout_g, 128);
  p.tpg = std::max(1, std::min(p.ntap, 128 / p.Nc));       // accumulators: tpg x Nc / 2 registers per thread
  p.n_tg = ceil_div(p.ntap, p.tpg);
  p.tpg = ceil_div(p.ntap, p.n_tg);                        // balance the groups
  if (p.tpg * p.Nc > 128) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: accumulators exceed the register budget");
  // the issue program holds ceil(tpg / 4) groups of four x-offsets per (piece pair, tap group): many tap groups of a wide N
  // tile (7x7 filters at Nc > 64: one tap per CTA) with several piece pairs overflow it; make_wg_plan then tries a narrower tile
  if ((int64_t)p.npairs * p.n_tg * ceil_div(p.tpg, 4) > kWgProg4)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: issue program too long (%d piece pairs x %d tap groups)", p.npairs, p.n_tg);
  // stage = NI sub-blocks (one image row-tile each): dy [TA][16 octets][rows_dy], x [TX][k-phase][Nc/8][rows_x].
  // Pick the raster (BW, TH) with the best useful fraction whose sub-block fits four times (else twice).
  auto sub_bytes_of = [&](int bw, int th) {
    const int dyb = round_up(16 * th * bw * 16, 128);
    const int xb = round_up((p.Nc / 8) * (th + hlo + hhi) * bw * 16 + 16 * 16, 128);
    return TA * dyb + TX * p.nkph_used * xb;
  };
  int best_bw = 0, best_th = 0;
  double best_score = -1;
  for (int pass = 0; pass < 2 && !best_bw; ++pass) {
    const int limit = (kSmemBudget - 2048) / (pass == 0 ? 4 : 2);
    for (int bw = need; bw <= std::min(128, need + 15); ++bw)
      for (int th = 1; th <= p.P; ++th) {
        if ((th * bw) % 16) continue;
        if (th + hlo + hhi > 256 || sub_bytes_of(bw, th) > limit) continue;
        const double eff = (double)p.Q / bw, fill = std::min(1.0, (double)th * bw / 64.0);
        const double score = eff * (0.5 + 0.5 * fill);
        if (score > best_score) { best_score = score; best_bw = bw; best_th = th; }
      }
  }
  if (!best_bw) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: no raster fits shared memory (N tile %d)", p.Nc);
  p.BW = best_bw; p.TH = best_th; p.THH = p.TH + hlo + hhi;
  p.rows_dy = p.TH * p.BW; p.rows_x = p.THH * p.BW;
  p.row_tiles = ceil_div(p.P, p.TH);
  for (int t = 0; t < p.ntap; ++t) p.tap_off[t] = (sh_[t] + hlo) * p.BW + (sw_[t] + wlo);
  p.dy_box_bytes = 16 * p.rows_dy * 16;
  p.x_box_bytes = (p.Nc / 8) * p.rows_x * 16;
  p.dy_bytes = round_up(p.dy_box_bytes, 128);
  p.x_bytes = round_up(p.x_box_bytes + 16 * 16, 128);       // + slack rows read past the last plane (must stay finite: zeroed)
  p.sub_bytes = TA * p.dy_bytes + TX * p.nkph_used * p.x_bytes;
  p.nsub = p.B * p.row_tiles;
  const int stage_target = 52 * 1024;
  p.NI = std::max(1, std::min(std::min(p.nsub, 8), stage_target / p.sub_bytes));
  p.stage_bytes = round_up(p.NI * p.sub_bytes, 1024);
  const int nst = (kSmemBudget - 1024) / p.stage_bytes;
  if (nst < 2) return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad: fewer than two stages fit");
  p.nstage = nst >= 4 ? 4 : 2;
  p.st_log2 = p.nstage == 4 ? 2 : 1;
  p.smem_bytes = p.nstage * p.stage_bytes + 1024;
  p.nstg_total = ceil_div(p.nsub, p.NI);
  const int n_kc = p.n_ktiles * p.n_ctiles * p.G * p.n_tg;
  p.splits = std::max(1, std::min(p.nstg_total, std::max(1, MNB_NUM_SMS / n_kc)));
  // keep accumulation chains short (the tensor core does not round the running fp32 sum to nearest after every
  // instruction): one accumulator takes <= ~256 MMAs; the partial sums are added with RN adds
  const int chain_per_stage = p.NI * (p.rows_dy / 16) * p.npairs;
  int chain_max = 256;
  if (const char* e = getenv("MNB_PK_WG_CHAIN")) chain_max = std::max(1, atoi(e));
  while (p.splits < p.nstg_total && (int64_t)ceil_div(p.nstg_total, p.splits) * chain_per_stage > chain_max) ++p.splits;
  p.stg_per_split = ceil_div(p.nstg_total, p.splits);
  p.splits = ceil_div(p.nstg_total, p.stg_per_split);
  p.partial_floats = (int64_t)p.splits * p.G * p.n_ktiles * p.n_ctiles * p.ntap * p.Nc * 128;
  return 0;
}

// the widest N tile whose operand blocks fit shared memory next to the dy planes (split fp32 x and stride-2 phase planes are
// several times larger than one plane of integer levels)
static int make_wg_plan(const mnb_conv_shape* s, int TA, int TX, WgPlan& p) {
  int rc = MNB_E_UNSUPPORTED;
  for (int cap = 128; cap >= 16; cap /= 2) {
    rc = make_wg_plan_nc(s, TA, TX, p, cap);
    if (rc != MNB_E_UNSUPPORTED) return rc;
  }
  return rc;
}

struct WgParams {
  struct Mma {
    uint32_t stg_per_split, nstg_total, NI, ksteps, ntap, tpg, n_tg, Nc, npairs, st_mask, st_log2, stage16, sub16, dy_term16, x_off16,
        x_term16, x_kph16, dy_sbo, x_sbo, nsub;
    uint32_t pair_a16[MAXPAIR], pair_b16[MAXPAIR];   // piece-plane offsets of the pairs (16-byte units)
    // per (piece pair, tap group, tap): x-operand offsets = pair plane + k-phase slot + tap row offset, in groups of four
    // (0xffffffff behind the last tap of a group)
    alignas(16) uint4 progb4[kWgProg4];
    uint32_t g4;                        // uint4 entries per (pair, tap group) = ceil(tpg / 4)
  } m;
  int G, n_ktiles, n_ctiles, n_tg, tpg, splits, stg_per_split, nstg_total, NI, nsub, row_tiles, TA, TX, nkph_used, kph_used[4];
  int K8, C8X, cout_g8, cin_g8, Nc8, TH, hlo, wlo, stage_bytes, sub_bytes, dy_bytes, x_bytes, dy_box_bytes, x_box_bytes,
      st_mask, st_log2, smem_bytes, ntap, Nc, cout_g, cin_g;
  float* partial;
  int* err;
};

struct alignas(16) WgShared {
  uint64_t full[MAXST], empty[MAXST];
  uint32_t abort;
};

constexpr int kWgThreads = 384;   // warp 0 TMA, warps 4..11 two MMA warpgroups (warps 1..3 idle)

// Warpgroup wg accumulates gradient channels (GEMM rows) 64*wg .. 64*wg+63 of the k tile for every tap of the CTA's tap
// group: tpg x NC / 2 registers per thread (plan: tpg * Nc <= 128).
template <int NC>
__global__ void __launch_bounds__(kWgThreads, 1)
pk_wgrad_kernel(const __grid_constant__ CUtensorMap dy0, const __grid_constant__ CUtensorMap dy1,
                const __grid_constant__ CUtensorMap dy2, const __grid_constant__ CUtensorMap x0,
                const __grid_constant__ CUtensorMap x1, const __grid_constant__ CUtensorMap x2,
                const __grid_constant__ WgParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ WgShared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < MAXST; ++i) { tc::mbar_init(&sh.full[i], 1); tc::mbar_init(&sh.empty[i], 8); }
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&dy0); tc::prefetch_tmap(&x0);
  }
  // every row an MMA can read must be finite (positions are the reduction dimension here): zero everything once,
  // the TMA boxes never touch the slack rows
  for (int i = tid; i < p.smem_bytes / 16; i += kWgThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();
  // work item of this CTA: blockIdx.x = (((g * n_ktiles + kt) * n_ctiles + ct) * n_tg + tap group), blockIdx.y = split
  const int split = blockIdx.y;
  const int tg = blockIdx.x % p.n_tg;
  const int r0 = blockIdx.x / p.n_tg;
  const int t0 = tg * p.tpg, tn = min(p.tpg, p.ntap - t0);    // this CTA's filter taps
  const int ct = r0 % p.n_ctiles;
  const int r1 = r0 / p.n_ctiles;
  const int kt = r1 % p.n_ktiles, g = r1 / p.n_ktiles;
  const int stg0 = split * p.stg_per_split, stg1 = min(p.nstg_total, stg0 + p.stg_per_split);

  if (warp == 0) {
    if (lane == 0) {
      uint32_t sc = 0;
      const int k8 = g * p.cout_g8 + kt * 16, c8 = g * p.cin_g8 + ct * p.Nc8;
      for (int stg = stg0; stg < stg1; ++stg, ++sc) {
        const uint32_t slot = sc & (uint32_t)p.st_mask, ph = (sc >> p.st_log2) & 1u;
        if (!tc::mbar_wait(&sh.empty[slot], ph ^ 1u, p.err, 711)) goto done;
        const int sub0 = stg * p.NI, nsubs = min(p.NI, p.nsub - sub0);
        tc::mbar_arrive_expect_tx(&sh.full[slot], (uint32_t)(nsubs * (p.TA * p.dy_box_bytes + p.TX * p.nkph_used * p.x_box_bytes)));
        for (int si = 0; si < nsubs; ++si) {
          const int sub = sub0 + si;
          const int b = sub / p.row_tiles, rt = sub - b * p.row_tiles;
          uint8_t* sb = smem + (size_t)slot * p.stage_bytes + (size_t)si * p.sub_bytes;
          const int h0 = rt * p.TH;
          tc::tma_load_4d(sb, &dy0, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 1) tc::tma_load_4d(sb + p.dy_bytes, &dy1, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 2) tc::tma_load_4d(sb + 2 * p.dy_bytes, &dy2, &sh.full[slot], 0, h0, b, k8);
          uint8_t* xb = sb + (size_t)p.TA * p.dy_bytes;
          for (int tx = 0; tx < p.TX; ++tx)
            for (int ks = 0; ks < p.nkph_used; ++ks) {
              const CUtensorMap* tm = tx == 0 ? &x0 : (tx == 1 ? &x1 : &x2);
              tc::tma_load_4d(xb + (size_t)(tx * p.nkph_used + ks) * p.x_bytes, tm, &sh.full[slot], -2 * p.wlo, h0 - p.hlo, b,
                              p.kph_used[ks] * p.C8X + c8);
            }
        }
        // sub-blocks of a short last stage keep their previous (finite) contents; the MMA loop skips them
      }
    }
  } else if (warp >= 4) {
    constexpr int NR = NC / 2, MAXTPG = 128 / NC;
    const int wg = (warp - 4) >> 2;
    const uint64_t a_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.m.dy_sbo) + (uint64_t)((8u * wg * p.m.dy_sbo) >> 4);
    const uint64_t b_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.m.x_sbo) + (uint64_t)p.m.x_off16;
    const uint32_t a_lo0 = (uint32_t)a_desc0, b_lo0 = (uint32_t)b_desc0;
    const uint64_t a_hi = a_desc0 & 0xffffffff00000000ull, b_hi = b_desc0 & 0xffffffff00000000ull;
    const uint32_t* prog = reinterpret_cast<const uint32_t*>(p.m.progb4);
    const uint32_t tgm = blockIdx.x % p.m.n_tg;
    const uint32_t tnm = min(p.m.tpg, p.m.ntap - tgm * p.m.tpg);
    float acc[MAXTPG][NR];
#pragma unroll
    for (int t = 0; t < MAXTPG; ++t) tc::zero_acc(acc[t]);
    uint32_t sc = 0;
    for (int stg = stg0; stg < stg1; ++stg, ++sc) {
      const uint32_t slot = sc & p.m.st_mask, ph = (sc >> p.m.st_log2) & 1u;
      tc::mbar_wait_soft(&sh.full[slot], ph, p.err, 712, &sh.abort);
      const uint32_t nsubs = min(p.m.NI, p.m.nsub - (uint32_t)stg * p.m.NI);
      tc::wg_fence();
#pragma unroll
      for (int t = 0; t < MAXTPG; ++t) tc::fence_acc(acc[t]);
      for (uint32_t si = 0; si < nsubs; ++si) {
        const uint32_t s16 = slot * p.m.stage16 + si * p.m.sub16;
        uint32_t arow = a_lo0 + s16, brow = b_lo0 + s16;
        for (uint32_t j = 0; j < p.m.ksteps; ++j, arow += 16u, brow += 16u) {
          for (uint32_t pr = 0; pr < p.m.npairs; ++pr) {
            const uint64_t ad = a_hi | (uint64_t)(arow + p.m.pair_a16[pr]);
            const uint32_t* pw = prog + (size_t)(pr * p.m.n_tg + tgm) * p.m.g4 * 4;
#pragma unroll
            for (int t = 0; t < MAXTPG; ++t) {
              if (t >= (int)tnm) break;
              tc::Mma<NC>::template bf16<1, 1>(acc[t], ad, b_hi | (uint64_t)(brow + pw[t]), 1);
            }
          }
        }
      }
      tc::wg_commit();
      tc::wg_wait<0>();
#pragma unroll
      for (int t = 0; t < MAXTPG; ++t) tc::fence_acc(acc[t]);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.empty[slot]);
    }
    // partial[split][g][kt][ct][tap][c][k]: straight from the fragment (row = k, column = c)
    float* dst = p.partial + ((((int64_t)split * p.G + g) * p.n_ktiles + kt) * p.n_ctiles + ct) * (int64_t)(p.ntap * p.Nc * 128) +
                 (int64_t)t0 * p.Nc * 128;
    const int fr = 64 * wg + 16 * ((warp - 4) & 3) + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
    for (int t = 0; t < MAXTPG; ++t) {
      if (t >= tn) break;
#pragma unroll
      for (int j = 0; j < NR / 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          dst[(int64_t)(t * p.Nc + 8 * j + fc + (e & 1)) * 128 + fr + 8 * (e >> 1)] = acc[t][4 * j + e];
    }
  }
done:
  __syncthreads();
}

// dw[k][c][tap] = mul(k) * sum over splits (fixed order: deterministic); mul = a_scale / kdiv[k] (either may be NULL).
// G merged groups of gm original groups each: only the diagonal (same original group) blocks are read.
// One block = the 128 output channels of a k tile for ONE (input channel, tap): the partials are read along k, their
// contiguous dimension (512-byte runs per warp), four splits in flight per thread; |W| threads in total.
__global__ void __launch_bounds__(128) wg_reduce_kernel(const float* __restrict__ partial, int splits, int G, int gm, int n_ktiles,
                                                        int n_ctiles, int ntap, int Nc, int cout_g, int cin_g, int cout_p,
                                                        int cin_p, const float* __restrict__ a_scale,
                                                        const float* __restrict__ kdiv, float* __restrict__ dw) {
  // cout_g / cin_g: channels per ORIGINAL group; cout_p / cin_p: the plane channels it spans (group-padded planes: rounded
  // up to 8, only the real (k, c) entries are read).  grid = (cin_g * ntap, k tiles of the original group, original groups)
  const int go = blockIdx.z, ktile = blockIdx.y;
  const int c = blockIdx.x / ntap, tap = blockIdx.x - c * ntap;
  const int g = go / gm, gi = go - g * gm;
  const int kk = ktile * 128 + threadIdx.x;         // output channel inside the original group
  if (kk >= cout_g) return;
  const int64_t tile = (int64_t)ntap * Nc * 128;
  const int64_t split_stride = (int64_t)G * n_ktiles * n_ctiles * tile;
  const int km = gi * cout_p + kk, cm = gi * cin_p + c;     // row / column inside the merged group
  const int kt = km >> 7, kl = km & 127, ct = cm / Nc, cl = cm - ct * Nc;
  const float* src = partial + (((int64_t)g * n_ktiles + kt) * n_ctiles + ct) * tile + ((int64_t)tap * Nc + cl) * 128 + kl;
  float acc = 0.f;
  int s = 0;
  for (; s + 4 <= splits; s += 4) {
    const float v0 = __ldg(src + (int64_t)s * split_stride), v1 = __ldg(src + (int64_t)(s + 1) * split_stride),
                v2 = __ldg(src + (int64_t)(s + 2) * split_stride), v3 = __ldg(src + (int64_t)(s + 3) * split_stride);
    acc = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(acc, v0), v1), v2), v3);
  }
  for (; s < splits; ++s) acc = __fadd_rn(acc, __ldg(src + (int64_t)s * split_stride));
  const int kout = go * cout_g + kk;
  if (a_scale || kdiv) {
    const float as = a_scale ? __ldg(a_scale) : 1.f;
    acc = __fmul_rn(acc, kdiv ? __fdiv_rn(as, __ldg(kdiv + kout)) : as);
  }
  dw[((int64_t)kout * cin_g + c) * ntap + tap] = acc;
}

// ---------------------------------------------------------------------------------------------------------
// weight gradient of narrow grouped 3x3 convolutions with every filter tap in registers
// ---------------------------------------------------------------------------------------------------------
// pk_wgrad_kernel merges four groups of 16 input / 32 output channels into one 128 x 64 accumulator block per tap and keeps
// tpg x Nc <= 128 accumulator columns, so such a layer runs as 5 tap groups, each re-reading every operand byte, with 3/4
// of its MMAs landing in discarded off-diagonal blocks.  Here one CTA owns the same 4-group block for ALL nine taps: MMA
// warpgroup wg multiplies its 64 dy rows (groups 2wg, 2wg + 1) by those two groups' 32 x columns only (m64n32k16, half of
// the products discarded instead of 3/4), 9 x 16 = 144 fp32 accumulators per thread, so each stage is loaded once.
// The register file is split with setmaxnreg: TMA warpgroup 40, MMA warpgroups 232 (128 * 40 + 256 * 232 = 384 * 168).
constexpr int kTapsN = 9;                                     // taps held in registers: 3 x 3 filters
constexpr int kTapsCin = 16, kTapsCout = 32, kTapsGm = 4;     // channels per group; groups per CTA block
constexpr int kTapsTmaRegs = 40, kTapsMmaRegs = 232;

// The cover: stride 1, 3 x 3, 16 / 32 channels per group, groups % 4 == 0.  The raster, the stages and the batch splits
// are those of make_wg_plan for the same shape, so every accumulator runs the same chain of MMAs in the same order and
// the splits are reduced in the same order: the result is bit for bit that of pk_wgrad_kernel.  Only the ring depth
// differs (any count up to MAXST instead of 2, 4 or 8: it does not change the arithmetic).
static int make_wgt_plan(const mnb_conv_shape* s, int TA, int TX, WgPlan& p) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  MNB_REQUIRE(TA >= 1 && TA <= 3 && TX >= 1 && TX <= 3, "term counts must be 1..3");
  const int C = s->in_c, K = s->out_c, G = s->groups;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && s->in_h > 0 && s->in_w > 0 && G > 0 && C % G == 0 && K % G == 0,
              "bad conv shape");
  auto no = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "pk wgrad taps: %s", why); };
  if (s->ker_h != 3 || s->ker_w != 3) return no("filter is not 3x3");
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return no("stride or dilation != 1");
  if (s->pad_h < 0 || s->pad_w < 0 || s->pad_h > 2 || s->pad_w > 2) return no("padding outside 0..2");
  if (C / G != kTapsCin || K / G != kTapsCout || G % kTapsGm) return no("needs 16 / 32 channels per group and groups % 4 == 0");
  if (int e = make_wg_plan(s, TA, TX, p)) return e;
  // the same block as pk_wgrad_kernel's: 4 merged groups, one 128-channel k tile, one 64-channel c tile (MNB_PK_WG_* knobs
  // that change it leave the shape to pk_wgrad_kernel)
  if (p.gm != kTapsGm || p.Nc != 64 || p.n_ctiles != 1 || p.n_ktiles != 1 || p.nkph_used != 1) return no("merged block");
  p.tpg = kTapsN; p.n_tg = 1;
  p.nstage = std::min(MAXST, (kSmemBudget - 1024) / p.stage_bytes);
  p.smem_bytes = p.nstage * p.stage_bytes + 1024;
  p.partial_floats = (int64_t)p.splits * p.G * kTapsN * p.Nc * 128;
  return 0;
}

struct WgtParams {
  uint32_t stg_per_split, nstg_total, NI, nsub, ksteps, npairs, nstage, stage16, sub16, dy_sbo, x_sbo, x_off16;
  uint32_t pair_a16[MAXPAIR], pair_b16[MAXPAIR];   // dy / x piece-plane offsets of each piece pair (16-byte units)
  uint32_t tap16[kTapsN];                          // x start-row offset of each tap (16-byte units)
  int row_tiles, TA, TX, TH, hlo, wlo, stage_bytes, sub_bytes, dy_bytes, x_bytes, dy_box_bytes, x_box_bytes, smem_bytes;
  float* partial;
  int* err;
};

constexpr int kWgtThreads = 384;   // warpgroup 0: TMA (warp 0, lane 0), warpgroups 1, 2: MMA

// CTA (blockIdx.x = 4-group block, blockIdx.y = batch split).  partial[split][block][tap][c 0..63][k 0..127] as
// wg_reduce_kernel reads it (G = blocks, one k tile, one c tile, Nc = 64); only the diagonal (same group) 32 x 16 blocks are
// written, the reduction reads nothing else.
__global__ void __launch_bounds__(kWgtThreads, 1)
pk_wgrad_taps_kernel(const __grid_constant__ CUtensorMap dy0, const __grid_constant__ CUtensorMap dy1,
                     const __grid_constant__ CUtensorMap dy2, const __grid_constant__ CUtensorMap x0,
                     const __grid_constant__ CUtensorMap x1, const __grid_constant__ CUtensorMap x2,
                     const __grid_constant__ WgtParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ WgShared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < MAXST; ++i) { tc::mbar_init(&sh.full[i], 1); tc::mbar_init(&sh.empty[i], 8); }
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&dy0); tc::prefetch_tmap(&x0);
  }
  // every row an MMA can read must be finite (positions are the reduction dimension): zero everything once
  for (int i = tid; i < p.smem_bytes / 16; i += kWgtThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();
  const int blk = blockIdx.x, split = blockIdx.y;
  const uint32_t stg0 = (uint32_t)split * p.stg_per_split, stg1 = min(p.nstg_total, stg0 + p.stg_per_split);

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kTapsTmaRegs));
    if (warp == 0 && lane == 0) {
      uint32_t slot = 0, ph = 0;
      const int k8 = blk * (kTapsGm * kTapsCout / 8), c8 = blk * (kTapsGm * kTapsCin / 8);
      for (uint32_t stg = stg0; stg < stg1; ++stg) {
        if (!tc::mbar_wait(&sh.empty[slot], ph ^ 1u, p.err, 721)) break;
        const int sub0 = (int)(stg * p.NI), nsubs = min((int)p.NI, (int)p.nsub - sub0);
        tc::mbar_arrive_expect_tx(&sh.full[slot], (uint32_t)(nsubs * (p.TA * p.dy_box_bytes + p.TX * p.x_box_bytes)));
        for (int si = 0; si < nsubs; ++si) {
          const int sub = sub0 + si;
          const int b = sub / p.row_tiles, h0 = (sub - b * p.row_tiles) * p.TH;
          uint8_t* sb = smem + (size_t)slot * p.stage_bytes + (size_t)si * p.sub_bytes;
          tc::tma_load_4d(sb, &dy0, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 1) tc::tma_load_4d(sb + p.dy_bytes, &dy1, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 2) tc::tma_load_4d(sb + 2 * p.dy_bytes, &dy2, &sh.full[slot], 0, h0, b, k8);
          uint8_t* xb = sb + (size_t)p.TA * p.dy_bytes;
          tc::tma_load_4d(xb, &x0, &sh.full[slot], -2 * p.wlo, h0 - p.hlo, b, c8);
          if (p.TX > 1) tc::tma_load_4d(xb + p.x_bytes, &x1, &sh.full[slot], -2 * p.wlo, h0 - p.hlo, b, c8);
          if (p.TX > 2) tc::tma_load_4d(xb + 2 * p.x_bytes, &x2, &sh.full[slot], -2 * p.wlo, h0 - p.hlo, b, c8);
        }
        // sub-blocks of a short last stage keep their previous (finite) contents; the MMA loop skips them
        if (++slot == p.nstage) { slot = 0; ph ^= 1u; }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kTapsMmaRegs));
    const int wg = (warp - 4) >> 2, w4 = (warp - 4) & 3;
    // A: the warpgroup's 64 dy channels (octets 8wg ..), B: its two groups' 32 x channels (octets 4wg ..)
    const uint64_t a_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.dy_sbo) + (uint64_t)((8u * wg * p.dy_sbo) >> 4);
    const uint64_t b_desc0 =
        tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.x_sbo) + (uint64_t)(p.x_off16 + ((4u * wg * p.x_sbo) >> 4));
    const uint32_t a_lo0 = (uint32_t)a_desc0, b_lo0 = (uint32_t)b_desc0;
    const uint64_t a_hi = a_desc0 & 0xffffffff00000000ull, b_hi = b_desc0 & 0xffffffff00000000ull;
    float acc[kTapsN][16];
#pragma unroll
    for (int t = 0; t < kTapsN; ++t) tc::zero_acc(acc[t]);
    uint32_t slot = 0, ph = 0;
    for (uint32_t stg = stg0; stg < stg1; ++stg) {
      tc::mbar_wait_soft(&sh.full[slot], ph, p.err, 722, &sh.abort);
      const uint32_t nsubs = min(p.NI, p.nsub - stg * p.NI);
      tc::wg_fence();
#pragma unroll
      for (int t = 0; t < kTapsN; ++t) tc::fence_acc(acc[t]);
      for (uint32_t si = 0; si < nsubs; ++si) {
        const uint32_t s16 = slot * p.stage16 + si * p.sub16;
        for (uint32_t j = 0; j < p.ksteps; ++j) {
          for (uint32_t pr = 0; pr < p.npairs; ++pr) {
            const uint64_t ad = a_hi | (uint64_t)(a_lo0 + s16 + 16u * j + p.pair_a16[pr]);
            const uint32_t bb = b_lo0 + s16 + 16u * j + p.pair_b16[pr];
#pragma unroll
            for (int t = 0; t < kTapsN; ++t) tc::Mma<32>::bf16<1, 1>(acc[t], ad, b_hi | (uint64_t)(bb + p.tap16[t]), 1);
          }
        }
      }
      tc::wg_commit();
      tc::wg_wait<0>();
#pragma unroll
      for (int t = 0; t < kTapsN; ++t) tc::fence_acc(acc[t]);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.empty[slot]);
      if (++slot == p.nstage) { slot = 0; ph ^= 1u; }
    }
    // fragment d[4j + 2i + c] = D[16 w4 + lane/4 + 8i][8j + 2(lane%4) + c]: rows of group (w4 >> 1), columns of group (j >> 1)
    float* dst = p.partial + ((int64_t)split * gridDim.x + blk) * (int64_t)(kTapsN * 64 * 128);
    const int kr = 64 * wg + 16 * w4 + (lane >> 2), cb = 32 * wg + 2 * (lane & 3);
#pragma unroll
    for (int t = 0; t < kTapsN; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if ((j >> 1) != (w4 >> 1)) continue;
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[(int64_t)(t * 64 + cb + 8 * j + (e & 1)) * 128 + kr + 8 * (e >> 1)] = acc[t][4 * j + e];
      }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// data and weight gradient of a 1x1 grouped convolution in one pass over dy
// ---------------------------------------------------------------------------------------------------------
// pk_conv_kernel (data gradient) and pk_wgrad_kernel read the same dy boxes op[c/8][position][8] from HBM, one K-major and
// one MN-major.  Here one CTA per (group, batch split) of the weight gradient's own plan streams each box once and feeds
// both MMAs from it: the wgrad MMAs exactly as pk_wgrad_kernel issues them (same split partials, reduced by
// wg_reduce_kernel), and per sub-block of 64 positions the data-gradient MMAs against the group's weight image, resident
// in shared memory, in the piece-pair / K-step order of make_plan's data-gradient program for the same shape.  Every
// accumulator sees the chain of MMAs it sees in the two separate kernels, so dx and dW are theirs bit for bit.
// The register file is split with setmaxnreg as in pk_wgrad_taps_kernel: wgrad Nc / 2 + dgrad Nc / 4 accumulators per thread.
constexpr int kBwdThreads = 384;   // warpgroup 0: TMA (warp 0, lane 0), warpgroups 1, 2: MMA + data-gradient epilogue
constexpr int kBwdRows = 64;       // positions per sub-block: one m64 block of data-gradient rows
constexpr int kBwdProg = 64;       // data-gradient MMAs per accumulator chain
constexpr int kBwdTmaRegs = 40, kBwdMmaRegs = 232;

struct BwdPlan {
  WgPlan wg;          // raster, sub-blocks, stages and splits (make_wg_plan; only the ring depth differs)
  Plan dg;            // data-gradient plan of the same shape (make_plan mode 1): N tile, K chunks, piece pairs
  int nprog, off_w, w_bytes, nstage, smem_bytes;
};

// The cover: stride 1, 1x1, no padding, channels per group <= 128 on either side and not group-padded, one 64-position
// sub-block raster, and data-gradient / weight-gradient plans that tile a group the same way (one N tile as wide as the
// wgrad's input-channel tile, one K box).
static int make_bwd_plan(const mnb_conv_shape* s, int TA, int TX, int TW, BwdPlan& b) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  MNB_REQUIRE(TA >= 1 && TA <= 3 && TX >= 1 && TX <= 3 && TW >= 1 && TW <= 3, "term counts must be 1..3");
  memset(&b, 0, sizeof(b));
  const int C = s->in_c, K = s->out_c, G = s->groups;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && s->in_h > 0 && s->in_w > 0 && G > 0 && C % G == 0 && K % G == 0,
              "bad conv shape");
  auto no = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "pk bwd1x1: %s", why); };
  if (s->ker_h != 1 || s->ker_w != 1) return no("filter is not 1x1");
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return no("stride or dilation != 1");
  if (s->pad_h != 0 || s->pad_w != 0) return no("padding != 0");
  if (C / G > 128 || K / G > 128) return no("more than 128 channels per group");
  if (G > 1 && ((C / G) % 8 || (K / G) % 8)) return no("group-padded operand planes");
  if (int e = make_wg_plan(s, TA, TX, b.wg)) return e;
  if (int e = make_plan(s, 1, TA, TW, b.dg)) return e;
  const WgPlan& w = b.wg;
  const Plan& d = b.dg;
  if (w.gm != 1 || w.n_ktiles != 1 || w.n_ctiles != 1 || w.n_tg != 1) return no("weight-gradient block is not one whole group");
  if (w.rows_dy != kBwdRows) return no("sub-block raster is not 64 positions");
  if (d.n_ntiles != 1 || d.Nt != w.Nc || d.Nt % 32) return no("data-gradient N tile differs from the weight-gradient tile");
  if (d.segmented) return no("segmented data-gradient plan");
  if (d.chunks * d.ksteps * 16 > 128) return no("data-gradient K-steps beyond the dy box");
  b.nprog = d.chunks * d.npairs * d.ksteps;
  // (one filter tap, <= 8 K-steps of at most 6 piece pairs: one stage template and at most 48 MMAs)
  if (d.ny != 1 || d.ntmpl[0] != 1 || b.nprog > kBwdProg)
    return mnb_fail(MNB_E_ARG, "pk bwd1x1: data-gradient plan with %d templates, %d MMAs", d.ntmpl[0], b.nprog);
  b.w_bytes = round_up(d.img_bytes[0], 1024);
  b.nstage = std::min(MAXST, (kSmemBudget - 1024 - b.w_bytes) / w.stage_bytes);
  if (b.nstage < 2) return no("fewer than two stages fit next to the weight image");
  b.off_w = b.nstage * w.stage_bytes + 1024;
  b.smem_bytes = b.off_w + b.w_bytes;
  return 0;
}

struct BwdParams {
  // weight gradient (pk_wgrad_kernel's quantities for tpg = 1, one tap)
  uint32_t stg_per_split, nstg_total, NI, nsub, ksteps, npairs, nstage, stage16, sub16, dy_sbo, x_sbo, x_off16;
  uint32_t pair_a16[MAXPAIR], pair_b16[MAXPAIR];
  int row_tiles, TA, TX, TH, stage_bytes, sub_bytes, dy_bytes, x_bytes, dy_box_bytes, x_box_bytes, smem_bytes, cout_g8, cin_g8;
  float* partial;
  // data gradient: chain of (A offset in the sub-block | B offset in the weight image << 16), 16-byte units
  uint32_t nprog, dg_lbo, w_lbo, off_w, w_bytes, img_bytes;
  uint32_t prog[kBwdProg];
  const uint8_t* w_img;
  int B, P, Q, BW, C, cin_g, C8O;
  float a_scale_const, gain;
  float bias0;              // 0: pk_conv_kernel's epilogue adds its (zero) bias with the same fmaf
  const uint8_t* bits8;     // STE mask [B][C8O][P][Q] or NULL
  float* dx;
  int* err;
};

// CTA (blockIdx.x = group, blockIdx.y = batch split).  NC: input channels per group rounded up to 16 (wgrad N, dgrad N tile)
template <int NC>
__global__ void __launch_bounds__(kBwdThreads, 1)
pk_bwd1x1_kernel(const __grid_constant__ CUtensorMap dy0, const __grid_constant__ CUtensorMap dy1,
                 const __grid_constant__ CUtensorMap dy2, const __grid_constant__ CUtensorMap x0,
                 const __grid_constant__ CUtensorMap x1, const __grid_constant__ CUtensorMap x2,
                 const __grid_constant__ BwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ WgShared sh;
  __shared__ uint64_t wbar;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < MAXST; ++i) { tc::mbar_init(&sh.full[i], 1); tc::mbar_init(&sh.empty[i], 8); }
    tc::mbar_init(&wbar, 1);
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&dy0); tc::prefetch_tmap(&x0);
  }
  // every row an MMA can read must be finite (positions are the wgrad's reduction dimension): zero the ring once
  for (int i = tid; i < (int)p.off_w / 16; i += kBwdThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();
  const int g = blockIdx.x, split = blockIdx.y;
  const uint32_t stg0 = (uint32_t)split * p.stg_per_split, stg1 = min(p.nstg_total, stg0 + p.stg_per_split);

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kBwdTmaRegs));
    if (warp == 0 && lane == 0) {
      // the group's data-gradient weight image (n tile 0, group g), once
      tc::mbar_arrive_expect_tx(&wbar, p.img_bytes);
      tc::bulk_load_1d(smem + p.off_w, p.w_img + (size_t)g * p.img_bytes, p.img_bytes, &wbar);
      uint32_t slot = 0, ph = 0;
      const int k8 = g * p.cout_g8, c8 = g * p.cin_g8;
      for (uint32_t stg = stg0; stg < stg1; ++stg) {
        if (!tc::mbar_wait(&sh.empty[slot], ph ^ 1u, p.err, 731)) break;
        const int sub0 = (int)(stg * p.NI), nsubs = min((int)p.NI, (int)p.nsub - sub0);
        tc::mbar_arrive_expect_tx(&sh.full[slot], (uint32_t)(nsubs * (p.TA * p.dy_box_bytes + p.TX * p.x_box_bytes)));
        for (int si = 0; si < nsubs; ++si) {
          const int sub = sub0 + si;
          const int b = sub / p.row_tiles, h0 = (sub - b * p.row_tiles) * p.TH;
          uint8_t* sb = smem + (size_t)slot * p.stage_bytes + (size_t)si * p.sub_bytes;
          tc::tma_load_4d(sb, &dy0, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 1) tc::tma_load_4d(sb + p.dy_bytes, &dy1, &sh.full[slot], 0, h0, b, k8);
          if (p.TA > 2) tc::tma_load_4d(sb + 2 * p.dy_bytes, &dy2, &sh.full[slot], 0, h0, b, k8);
          uint8_t* xb = sb + (size_t)p.TA * p.dy_bytes;
          tc::tma_load_4d(xb, &x0, &sh.full[slot], 0, h0, b, c8);
          if (p.TX > 1) tc::tma_load_4d(xb + p.x_bytes, &x1, &sh.full[slot], 0, h0, b, c8);
          if (p.TX > 2) tc::tma_load_4d(xb + 2 * p.x_bytes, &x2, &sh.full[slot], 0, h0, b, c8);
        }
        // sub-blocks of a short last stage keep their previous (finite) contents; the MMA loop skips them
        if (++slot == p.nstage) { slot = 0; ph ^= 1u; }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kBwdMmaRegs));
    constexpr int NR = NC / 2, ND = NC / 2, NRD = ND / 2;
    const int wg = (warp - 4) >> 2, w4 = (warp - 4) & 3;
    // wgrad: A = the warpgroup's 64 dy channels (MN-major), B = the x channels (MN-major)
    const uint64_t a_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.dy_sbo) + (uint64_t)((8u * wg * p.dy_sbo) >> 4);
    const uint64_t b_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(smem), 128, p.x_sbo) + (uint64_t)p.x_off16;
    // dgrad: A = the 64 positions of the sub-block (K-major: dy channels along K), B = the warpgroup's half of the N tile
    const uint64_t da_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), p.dg_lbo, 128);
    const uint64_t db_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem + p.off_w), p.w_lbo, 128) + (uint64_t)(ND * wg);
    const uint32_t a_lo0 = (uint32_t)a_desc0, b_lo0 = (uint32_t)b_desc0, da_lo0 = (uint32_t)da_desc0, db_lo0 = (uint32_t)db_desc0;
    const uint64_t a_hi = a_desc0 & 0xffffffff00000000ull, b_hi = b_desc0 & 0xffffffff00000000ull;
    const uint64_t da_hi = da_desc0 & 0xffffffff00000000ull, db_hi = db_desc0 & 0xffffffff00000000ull;
    // data-gradient epilogue: fragment d[4j + 2i + c] = D[position 16 w4 + lane/4 + 8i][channel ND wg + 8j + 2(lane%4) + c]
    const int64_t plane = (int64_t)p.P * p.Q;
    const int n_lo = ND * wg + 2 * (lane & 3);
    float acc[NR], dacc[NRD];
    tc::zero_acc(acc);
    tc::mbar_wait_soft(&wbar, 0, p.err, 733, &sh.abort);
    uint32_t slot = 0, ph = 0;
    for (uint32_t stg = stg0; stg < stg1; ++stg) {
      tc::mbar_wait_soft(&sh.full[slot], ph, p.err, 732, &sh.abort);
      const uint32_t nsubs = min(p.NI, p.nsub - stg * p.NI);
      for (uint32_t si = 0; si < nsubs; ++si) {
        const uint32_t s16 = slot * p.stage16 + si * p.sub16;
        tc::zero_acc(dacc);
        tc::wg_fence();
        tc::fence_acc(acc);
        tc::fence_acc(dacc);
        for (uint32_t j = 0; j < p.ksteps; ++j)
          for (uint32_t pr = 0; pr < p.npairs; ++pr)
            tc::Mma<NC>::template bf16<1, 1>(acc, a_hi | (uint64_t)(a_lo0 + s16 + 16u * j + p.pair_a16[pr]),
                                             b_hi | (uint64_t)(b_lo0 + s16 + 16u * j + p.pair_b16[pr]), 1);
        for (uint32_t e = 0; e < p.nprog; ++e) {
          const uint32_t w = p.prog[e];
          tc::Mma<ND>::template bf16<0, 0>(dacc, da_hi | (uint64_t)(da_lo0 + s16 + (w & 0xffffu)),
                                           db_hi | (uint64_t)(db_lo0 + (w >> 16)), 1);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::fence_acc(acc);
        tc::fence_acc(dacc);
        // dx of the sub-block: pk_conv_kernel's data-gradient epilogue (a_scale_const, or the STE mask times gain)
        const int sub = (int)((stg * p.NI) + si);
        const int b = sub / p.row_tiles, h0 = (sub - b * p.row_tiles) * p.TH;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int m = 16 * w4 + (lane >> 2) + 8 * i;
          const int oh = h0 + m / p.BW, ow = m - (m / p.BW) * p.BW;
          if (oh >= p.P || ow >= p.Q) continue;
          float* orow = p.dx + ((int64_t)b * p.C + g * p.cin_g) * plane + (int64_t)oh * p.Q + ow;
          const uint8_t* brow = p.bits8 ? p.bits8 + ((int64_t)b * p.C8O + g * (p.cin_g >> 3)) * plane + (int64_t)oh * p.Q + ow : nullptr;
#pragma unroll
          for (int j = 0; j < ND / 8; ++j) {
            const int n = n_lo + 8 * j;     // channels n, n + 1 (same octet)
            if (n >= p.cin_g) continue;
            if (brow) {
              const uint32_t mk = __ldg(brow + (int64_t)(n >> 3) * plane) >> (n & 7);
              orow[(int64_t)n * plane] = (mk & 1u) ? dacc[4 * j + 2 * i] * p.gain : 0.f;
              if (n + 1 < p.cin_g) orow[(int64_t)(n + 1) * plane] = (mk & 2u) ? dacc[4 * j + 2 * i + 1] * p.gain : 0.f;
            } else {
              orow[(int64_t)n * plane] = fmaf(dacc[4 * j + 2 * i], p.a_scale_const, p.bias0);
              if (n + 1 < p.cin_g) orow[(int64_t)(n + 1) * plane] = fmaf(dacc[4 * j + 2 * i + 1], p.a_scale_const, p.bias0);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.empty[slot]);
      if (++slot == p.nstage) { slot = 0; ph ^= 1u; }
    }
    // partial[split][g][c][k]: pk_wgrad_kernel's layout for one k tile, one c tile, one tap
    float* dst = p.partial + ((int64_t)split * gridDim.x + g) * (int64_t)(NC * 128);
    const int fr = 64 * wg + 16 * w4 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < NR / 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) dst[(int64_t)(8 * j + fc + (e & 1)) * 128 + fr + 8 * (e >> 1)] = acc[4 * j + e];
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// forward and data gradient of narrow grouped 3x3 convolutions with whole images as M tiles
// ---------------------------------------------------------------------------------------------------------
// pk_conv_kernel tiles these layers (16 / 32 channels per group) into 128-row M tiles of a few image rows: a 16 x 16 image
// takes three row tiles (7 + 7 + 2 rows), an 8 x 8 image fills half of one, and every work item is 9..36 short MMAs followed
// by an epilogue that both MMA warpgroups wait for.  Here a CTA owns GB consecutive groups for the whole launch (their
// weight images stay in shared memory) and walks over image tiles: one stage = the zero-padded boxes of TB whole images
// with the channels of all GB groups, the M tile = the image raster itself (ceil(rows / 64) m64 blocks, no row tiles).
// The three MMA warpgroups take turns on the stages: while one runs its epilogue the others issue MMAs.  The
// epilogue goes through a per-warpgroup staging tile [image][channel][position], so that the output of one (image, group)
// - a contiguous NCHW run of ng * H * W elements - leaves in 16-byte stores.
// Every output element sees the MMA chain of make_plan's plan for the same shape (taps, piece pairs, K-steps and their
// order; one N tile of exactly the group's channels), so the result is bit for bit that of pk_conv_kernel (DESIGN.md 4.9).
constexpr int kGc3MaxMb = 8;                       // m64 blocks per M tile
constexpr int kGc3MaxProg = 128;                   // MMAs per accumulator chain
constexpr int kGc3Cons = 3;                        // MMA + epilogue warpgroups
constexpr int kGc3Threads = 128 * (1 + kGc3Cons);  // warpgroup 0: TMA (warp 0, lane 0), warpgroups 1 .. 3: MMA + epilogue
constexpr int kGc3SmemBudget = 227 * 1024 - 4096;  // dynamic shared memory (the static part holds barriers and constants)
// registers: 128 * 40 + 384 * 152 <= 65536; the accumulators of an M tile are (m64 blocks) x NT / 2 per thread
constexpr int kGc3TmaRegs = 40, kGc3MmaRegs = 152;
__host__ __device__ constexpr int gc3_max_mb(int nt) { return nt == 32 ? 6 : kGc3MaxMb; }

struct Gc3Plan {
  Plan pl;                  // make_plan's plan of the same (shape, mode, pieces): the chain and the weight image
  int GB, nblk, TB, n_tiles, cpb, BW, THH, npos, nmb, plane, SP;
  int a_box_bytes, a_piece_bytes, stage_bytes, nstage, w_bytes, stg_bytes, off_stage, off_stg, off_rowmap, smem_bytes;
  int nprog;
  uint32_t prog[kGc3MaxProg];               // A offset | B offset << 16 (16-byte units) of each MMA of the chain, in order
  int16_t chain[kGc3MaxProg][4];            // (tap r * S + s, piece of A, piece of B, K-step) of each MMA (plan queries)
};

struct Gc3Params {
  uint32_t prog[kGc3MaxProg];
  int nprog, mode, TA, GB, ng, kg8, NOUT, B, TB, n_tiles, cpb, nmb, npos, BW, THH, OH, OW, plane, SP, C8O, wlo, hlo;
  int a_box_bytes, a_piece_bytes, stage_bytes, nstage, w_bytes, img_bytes, stg_bytes, off_stage, off_stg, off_rowmap, smem_bytes;
  const uint8_t* w_img;
  const float* n_scale;
  const float* a_scale;
  float a_scale_const;
  const float* bias;
  const uint8_t* bits8;
  float gain;
  float* out;
  int16_t* codes;
  float* dec;
  int* err;
};

static int make_gc3_plan(const mnb_conv_shape* s, int mode, int TA, int TBk, Gc3Plan& g) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  MNB_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (forward) or 1 (data gradient)");
  MNB_REQUIRE(TA >= 1 && TA <= 3 && TBk >= 1 && TBk <= 3, "term counts must be 1..3");
  memset(&g, 0, sizeof(g));
  auto no = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "pk gc3: %s", why); };
  const int C = s->in_c, K = s->out_c, G = s->groups;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && s->in_h > 0 && s->in_w > 0 && G > 0 && C % G == 0 && K % G == 0,
              "bad conv shape");
  if (s->ker_h != 3 || s->ker_w != 3) return no("filter is not 3x3");
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return no("stride or dilation != 1");
  if (s->pad_h < 0 || s->pad_w < 0 || s->pad_h > 2 || s->pad_w > 2) return no("padding outside 0..2");
  if (C / G != 16 || K / G != 32 || G % 4) return no("needs 16 / 32 channels per group and groups % 4 == 0");
  if (mode == 0 && (TA != 1 || TBk != 1)) return no("the forward takes one activation piece and one weight piece");
  if (mode == 1 && (TA != 2 || TBk != 1)) return no("the data gradient takes two dy pieces and one weight piece");
  Plan& p = g.pl;
  if (int e = make_plan(s, mode, TA, TBk, p)) return e;
  if (p.segmented || p.ny != 1 || p.nkph != 1 || p.n_ntiles != 1 || p.Nt != p.ng) return no("plan is segmented or tiled along N");
  // raster: whole images, row pitch BW, TB images per M tile
  g.BW = p.OWr + p.wlo + p.whi; g.THH = p.OHr + p.hlo + p.hhi; g.plane = p.OHr * p.OWr;
  if (2 * g.BW > 256 || g.THH > 256) return no("image larger than one box");
  g.SP = g.plane + ((4 - g.plane % 16) + 16) % 16;     // channel pitch of the staging tile: = 4 (mod 16), conflict-free writes
  const int kg8 = p.kg / 8, img_bytes = p.img_bytes[0];
  const int static_slack = 1024;
  double best = -1;
  for (int pass = 0; pass < 2 && best < 0; ++pass) {
    // stages: a multiple of kGc3Cons, so that every ring slot belongs to ONE warpgroup (stage k -> slot k % nstage, warpgroup
    // k % kGc3Cons).  A slot shared by two warpgroups would let the consumer of stage k + nstage wait on full[slot] while
    // stage k's load is still in flight: the phase it waits for has the parity of the phase before stage k, the wait would
    // pass at once, and its arrivals on empty[slot] would release stage k's slot early.  Within one warpgroup the waits on
    // a slot are ordered, so a waiter is never more than one phase ahead.
    const int min_st = pass == 0 ? 2 * kGc3Cons : kGc3Cons;
    for (int tb = std::min(p.B, 16); tb >= 1; --tb) {
      const int rows = (tb - 1) * g.THH * g.BW + (p.OHr - 1) * g.BW + p.OWr;
      const int nmb = ceil_div(rows, 64);
      if (nmb > gc3_max_mb(p.Nt)) continue;
      const double eff = (double)tb * g.plane / (64.0 * nmb);
      if (eff <= best + 1e-9) continue;
      for (int gb = 4; gb >= 1; gb /= 2) {
        if (G % gb) continue;
        const int npos = tb * g.THH * g.BW;
        const int box = gb * kg8 * npos * 16, piece = round_up(box, 128);
        const int stage = round_up(TA * piece, 1024);
        const int wb = round_up(gb * img_bytes, 1024);
        const int stg = round_up(tb * p.ng * g.SP * 4, 128);
        // MMAs of invalid rows read up to nmb * 64 + the largest tap offset rows past the start of the last octet
        const int over = std::max(0, nmb * 64 + (p.hlo + p.hhi) * g.BW + p.wlo + p.whi - npos);
        const int slack = round_up(over * 16 + 16, 1024);
        const int rowmap = kGc3MaxMb * 64 * 4;
        const int fixed = wb + slack + kGc3Cons * stg + rowmap + static_slack;
        const int nst = std::min(MAXST, (kGc3SmemBudget - fixed) / stage) / kGc3Cons * kGc3Cons;
        if (nst < min_st) continue;
        best = eff;
        g.TB = tb; g.nmb = nmb; g.npos = npos; g.GB = gb; g.a_box_bytes = box; g.a_piece_bytes = piece; g.stage_bytes = stage;
        g.nstage = nst; g.w_bytes = gb * img_bytes; g.stg_bytes = stg;
        g.off_stage = wb; g.off_stg = wb + nst * stage + slack; g.off_rowmap = g.off_stg + kGc3Cons * stg;
        g.smem_bytes = g.off_rowmap + rowmap;
        break;
      }
    }
  }
  if (best < 0) return no("no image tile fits the accumulators and shared memory");
  if (g.npos * 16 >= (1 << 18) || g.stage_bytes * g.nstage + g.w_bytes > (1 << 18)) return no("descriptor range");
  g.nblk = G / g.GB;
  g.n_tiles = ceil_div(p.B, g.TB);
  g.cpb = std::max(1, std::min(g.n_tiles, MNB_NUM_SMS / g.nblk));
  // the chain of make_plan: stage templates -> K chunks -> piece pairs (small products first) -> taps -> K-steps, the issue
  // order of pk_conv_kernel's program; A offsets for this raster, B offsets into the plan's weight image of one group
  const int ph = s->pad_h, pw = s->pad_w;
  const int b_tap16 = (p.CC / 8) * p.Nt, a_piece16 = g.a_piece_bytes >> 4;
  g.nprog = 0;
  for (int t = 0; t < p.ntmpl[0]; ++t) {
    const Tmpl& tp = p.tmpl[0][t];
    for (int cc = 0; cc < p.chunks; ++cc)
      for (int pr = 0; pr < p.npairs; ++pr)
        for (int i = 0; i < tp.ntap; ++i)
          for (int j = 0; j < p.ksteps; ++j) {
            if (g.nprog >= kGc3MaxProg) return no("MMA chain longer than 128");
            const int r = p.tap_r[0][tp.tap0 + i], q = p.tap_s[0][tp.tap0 + i];
            const int sh = mode == 0 ? r - ph : ph - r, sw = mode == 0 ? q - pw : pw - q;
            const int ks = cc * p.ksteps + j;
            const int a16 = (sh + p.hlo) * g.BW + (sw + p.wlo) + p.pair_a[pr] * a_piece16 + ks * 2 * g.npos;
            const int b16 = (tp.blk_off + cc * tp.blk_bytes) / 16 + i * b_tap16 + p.pair_b[pr] * tp.ntap * b_tap16 + j * 2 * p.Nt;
            if (a16 > 0xffff || b16 > 0xffff) return no("MMA offset overflow");
            g.chain[g.nprog][0] = (int16_t)(r * 3 + q); g.chain[g.nprog][1] = (int16_t)p.pair_a[pr];
            g.chain[g.nprog][2] = (int16_t)p.pair_b[pr]; g.chain[g.nprog][3] = (int16_t)ks;
            g.prog[g.nprog++] = (uint32_t)a16 | ((uint32_t)b16 << 16);
          }
  }
  return 0;
}

__device__ __forceinline__ void gc3_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// One output element of the epilogue, exactly as pk_conv_kernel's do_slot computes it (r: the accumulator).
struct Gc3Out {
  const Gc3Params& p;
  const float* sc;
  const float* bs;
  __device__ __forceinline__ float f32(float r, int n, int b, int ch, int pos) const {
    if (p.mode == 1 && p.bits8) {
      const uint32_t m = __ldg(p.bits8 + ((int64_t)b * p.C8O + (ch >> 3)) * p.plane + pos);
      return ((m >> (ch & 7)) & 1u) ? r * p.gain : 0.f;
    }
    return fmaf(r, sc[n], bs[n]);
  }
};

template <int NT>
__global__ void __launch_bounds__(kGc3Threads, 1)
pk_gc3_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1, const __grid_constant__ Gc3Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t full[MAXST], empty[MAXST], wfull;
  __shared__ uint32_t abort_flag;
  __shared__ alignas(16) float s_scale[128], s_bias[128];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int blk = blockIdx.x / p.cpb, cta = blockIdx.x - blk * p.cpb;   // group block; CTA within the block
  const int n_base = blk * p.GB * p.ng;                                 // first output channel of the block
  int* rowmap = reinterpret_cast<int*>(smem + p.off_rowmap);
  if (tid == 0) {
    for (int i = 0; i < MAXST; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 4); }
    tc::mbar_init(&wfull, 1);
    abort_flag = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tm0);
    if (p.TA > 1) tc::prefetch_tmap(&tm1);
  }
  // rows behind the boxes that only invalid accumulator rows read must be finite
  for (int i = tid; i < p.off_rowmap / 16; i += kGc3Threads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  // M row -> staging index image * ng * SP + position, or -1 for a halo / padding row
  for (int m = tid; m < kGc3MaxMb * 64; m += kGc3Threads) {
    const int img = p.THH * p.BW, tb = m / img, rem = m - tb * img, th = rem / p.BW, wc = rem - th * p.BW;
    rowmap[m] = (tb < p.TB && th < p.OH && wc < p.OW) ? tb * p.ng * p.SP + th * p.OW + wc : -1;
  }
  {
    const float a_sc = p.a_scale ? __ldg(p.a_scale) : p.a_scale_const;
    for (int n = tid; n < p.GB * p.ng; n += kGc3Threads) {
      const float scv = p.n_scale ? __fmul_rn(a_sc, __ldg(p.n_scale + n_base + n)) : a_sc;
      const float bsv = p.bias ? __ldg(p.bias + n_base + n) : 0.f;
      s_scale[n] = scv; s_bias[n] = bsv;
      if (p.dec && cta == 0) { p.dec[n_base + n] = scv; p.dec[p.NOUT + n_base + n] = bsv; }
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kGc3TmaRegs));
    if (warp == 0 && lane == 0) {
      tc::mbar_arrive_expect_tx(&wfull, (uint32_t)p.w_bytes);
      tc::bulk_load_1d(smem, p.w_img + (size_t)blk * p.w_bytes, (uint32_t)p.w_bytes, &wfull);
      const int c8 = blk * p.GB * p.kg8;
      uint32_t slot = 0, ph = 0;
      for (int t = cta; t < p.n_tiles; t += p.cpb) {
        if (!tc::mbar_wait(&empty[slot], ph ^ 1u, p.err, 731)) break;
        tc::mbar_arrive_expect_tx(&full[slot], (uint32_t)(p.TA * p.a_box_bytes));
        uint8_t* sb = smem + p.off_stage + (size_t)slot * p.stage_bytes;
        tc::tma_load_4d(sb, &tm0, &full[slot], -2 * p.wlo, -p.hlo, t * p.TB, c8);
        if (p.TA > 1) tc::tma_load_4d(sb + p.a_piece_bytes, &tm1, &full[slot], -2 * p.wlo, -p.hlo, t * p.TB, c8);
        if (++slot == (uint32_t)p.nstage) { slot = 0; ph ^= 1u; }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kGc3MmaRegs));
    constexpr int NR = NT / 2, MAXMB = gc3_max_mb(NT);
    const int wg = (warp - 4) >> 2, w4 = (warp - 4) & 3, et = tid - 128 * (wg + 1);
    float* stg = reinterpret_cast<float*>(smem + p.off_stg + (size_t)wg * p.stg_bytes);
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), (uint32_t)p.npos * 16u, 128);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), (uint32_t)NT * 16u, 128);
    const uint32_t a_lo0 = (uint32_t)a_desc0, b_lo0 = (uint32_t)b_desc0;
    const uint64_t a_hi = a_desc0 & 0xffffffff00000000ull, b_hi = b_desc0 & 0xffffffff00000000ull;
    const int fr = 16 * w4 + (lane >> 2), fc = 2 * (lane & 3);      // fragment row / column of d[0]
    const FastDiv d_plane(p.plane);
    tc::mbar_wait_soft(&wfull, 0, p.err, 733, &abort_flag);
    // this warpgroup's stages: every kGc3Cons-th one of the CTA's sequence (k = wg, wg + kGc3Cons, ...)
    for (int k = wg, t = cta + wg * p.cpb; t < p.n_tiles; k += kGc3Cons, t += kGc3Cons * p.cpb) {
      const uint32_t slot = (uint32_t)k % (uint32_t)p.nstage, ph = ((uint32_t)k / (uint32_t)p.nstage) & 1u;
      tc::mbar_wait_soft(&full[slot], ph, p.err, 732, &abort_flag);
      const uint32_t s16 = (uint32_t)(p.off_stage + (int)slot * p.stage_bytes) >> 4;
      for (int gl = 0; gl < p.GB; ++gl) {
        float acc[MAXMB][NR];
#pragma unroll
        for (int mb = 0; mb < MAXMB; ++mb) tc::zero_acc(acc[mb]);
        tc::wg_fence();
#pragma unroll
        for (int mb = 0; mb < MAXMB; ++mb) tc::fence_acc(acc[mb]);
        const uint32_t a_base = a_lo0 + s16 + (uint32_t)(gl * p.kg8 * p.npos), b_base = b_lo0 + (uint32_t)((gl * p.img_bytes) >> 4);
#pragma unroll
        for (int mb = 0; mb < MAXMB; ++mb) {
          if (mb >= p.nmb) break;
          for (int e = 0; e < p.nprog; ++e) {
            const uint32_t w = p.prog[e];
            tc::Mma<NT>::template bf16<0, 0>(acc[mb], a_hi | (uint64_t)(a_base + 64u * mb + (w & 0xffffu)),
                                              b_hi | (uint64_t)(b_base + (w >> 16)), 1);
          }
        }
        tc::wg_commit();
        tc::wg_wait<0>();
#pragma unroll
        for (int mb = 0; mb < MAXMB; ++mb) tc::fence_acc(acc[mb]);
        if (gl == p.GB - 1) {   // this warp's reads of the stage are done
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(&empty[slot]);
        }
        gc3_bar(1 + wg);        // the previous copy-out is done with the staging tile
#pragma unroll
        for (int mb = 0; mb < MAXMB; ++mb) {
          if (mb >= p.nmb) break;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int dst = rowmap[64 * mb + fr + 8 * i];
            if (dst < 0) continue;
#pragma unroll
            for (int j = 0; j < NR / 4; ++j) {
              stg[dst + (8 * j + fc) * p.SP] = acc[mb][4 * j + 2 * i];
              stg[dst + (8 * j + fc + 1) * p.SP] = acc[mb][4 * j + 2 * i + 1];
            }
          }
        }
        gc3_bar(1 + wg);
        // copy-out: image b of the tile, channels ch0 .. ch0 + ng: one contiguous NCHW run of ng * plane elements
        const int ch0 = n_base + gl * p.ng, E = p.ng * p.plane;
        const float* sc = s_scale + gl * p.ng;
        const float* bs = s_bias + gl * p.ng;
        const Gc3Out og{p, sc, bs};
        for (int tb = 0; tb < p.TB; ++tb) {
          const int b = t * p.TB + tb;
          if (b >= p.B) break;
          const float* src = stg + tb * p.ng * p.SP;
          if (p.codes) {
            uint4* dst = reinterpret_cast<uint4*>(p.codes + ((int64_t)b * p.NOUT + ch0) * p.plane);
            for (int v = et; v < E / 8; v += 128) {
              uint32_t n, pos;
              d_plane.divmod((uint32_t)(8 * v), n, pos);
              uint32_t wv[4];
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const uint32_t c = (uint32_t)(int16_t)__float2int_rn(src[n * p.SP + pos]) & 0xffffu;
                wv[i >> 1] = (i & 1) ? (wv[i >> 1] | (c << 16)) : c;
                if (++pos == (uint32_t)p.plane) { pos = 0; ++n; }
              }
              dst[v] = make_uint4(wv[0], wv[1], wv[2], wv[3]);
            }
          } else {
            float4* dst = reinterpret_cast<float4*>(p.out + ((int64_t)b * p.NOUT + ch0) * p.plane);
            for (int v = et; v < E / 4; v += 128) {
              uint32_t n, pos;
              d_plane.divmod((uint32_t)(4 * v), n, pos);
              float r[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                r[i] = og.f32(src[n * p.SP + pos], (int)n, b, ch0 + (int)n, (int)pos);
                if (++pos == (uint32_t)p.plane) { pos = 0; ++n; }
              }
              dst[v] = make_float4(r[0], r[1], r[2], r[3]);
            }
          }
        }
      }
    }
  }
  __syncthreads();
}

}  // namespace pk

// =========================================================================================================
// C-ABI
// =========================================================================================================
// launch geometry of the packers that give one thread one position of one (image, 16-byte unit) plane: block =
// (positions, planes), small images put several planes into one 256-thread block.  false: the planes exceed the grid.
static bool unit_grid(int batch, int units, int hw, dim3& blocks, dim3& threads) {
  const int tx = std::min(256, (hw + 31) / 32 * 32), ty = 256 / tx;     // threads along positions / planes per block
  const int planes = batch * units, gy = (planes + ty - 1) / ty;
  const int bx = std::max(1, std::min((hw + tx - 1) / tx, std::max(1, (MNB_NUM_SMS * 16) / std::max(1, gy))));
  blocks = dim3(bx, gy); threads = dim3(tx, ty);
  return gy <= 65535;
}

// the quantizers whose levels fit s8: symmetric IAO with 2..8 bits, DoReFa with 2..7 bits (levels 0 .. 2^a - 1); the only
// ones an int8 plane holds
static bool i8_quantizer(const mnb_act_qparams* q) {
  if (q->mode == MNB_ACT_DOREFA) return q->bits >= 2 && q->bits <= 7;
  return q->mode == MNB_ACT_IAO && q->q_type == 0 && q->bits >= 2 && q->bits <= 8 && q->qmin >= -128 && q->qmax <= 127;
}
static const char* const kI8QuantizerRule =
    "int8 plane needs a symmetric IAO quantizer with 2..8 bits or a DoReFa quantizer with 2..7 bits (8-bit DoReFa levels "
    "reach 255)";

// mnb_quant_add_pack_fwd (CPU = 8: bf16 consumer plane) and mnb_quant_add_pack_i8_fwd (CPU = 16: int8 consumer plane)
template <int CPU>
static int quant_add_pack(const float* a, const float* b, int32_t batch, int32_t channels, int32_t h, int32_t w,
                          const mnb_act_qparams* qp, int32_t relu, float* out, const mnb_pk_post* post, mnb_stream_t stream) {
  MNB_REQUIRE(a && b && qp && out && post && post->q && post->out_pk, "NULL quant_add_pack pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0, "bad quant_add_pack shape");
  MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA || qp->mode == MNB_ACT_IAO, "QuantAdd takes a DoReFa or IAO quantizer");
  if (CPU == 16) {
    if (!i8_quantizer(post->q)) return mnb_fail(MNB_E_UNSUPPORTED, "quant_add_pack: %s", kI8QuantizerRule);
  } else {
    MNB_REQUIRE(post->q->mode == MNB_ACT_DOREFA || post->q->mode == MNB_ACT_IAO, "consumer quantizer must be DoReFa or IAO");
  }
  MNB_REQUIRE(post->q->bits >= 2 && post->q->bits <= 8 && qp->bits >= 2 && qp->bits <= 8, "quantizers must have 2..8 bits");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(post->out_pk) & 15) == 0, "packed tensor must be 16-byte aligned");
  if (post->phase_split) MNB_REQUIRE(((h | w) & 1) == 0, "phase split needs even H and W");
  const int units = (channels + CPU - 1) / CPU;
  dim3 blocks, threads;
  if (!unit_grid(batch, units, h * w, blocks, threads))
    return mnb_fail(MNB_E_UNSUPPORTED, "quant_add_pack: %d (image, unit) planes exceed the grid", batch * units);
  pk::quant_add_pack_kernel<CPU><<<blocks, threads, 0, (cudaStream_t)stream>>>(
      a, b, batch, channels, h, w, units, *qp, relu, out, *post->q, post->relu, post->phase_split,
      reinterpret_cast<uint4*>(post->out_pk));
  MNB_LAUNCHED(1);
  return 0;
}

// the first min(n, 31) fields of mnb_pk_conv_plan_ex / mnb_pk_i8_conv_plan (words: MMA program words of the plan)
static void plan_fields(const pk::Plan& p, int words, int32_t* out, int32_t n) {
  // stages of the last accumulation segment of an output-phase-0 item (segmented plans; 0 otherwise)
  const int last_seg = p.segmented ? (p.ntmpl[0] * p.chunks - 1) % p.seg_len + 1 : 0;
  const int v[31] = {(int)(p.wimg_bytes & 0x7fffffff), (int)(p.wimg_bytes >> 31), p.Nt, p.n_ntiles, p.MT, p.CC, p.chunks, p.nstage,
                     p.smem_bytes, p.MT * p.Nt, p.TH, p.TB, p.BW, p.n_mtiles, p.n_items, p.ny,
                     p.segmented, p.segmented ? p.seg_len : 0, p.npairs, p.col_tiles, p.n_mgroups,
                     p.ntmpl[0], p.ntmpl[1], p.ntmpl[2], p.ntmpl[3], p.ntap[0], p.ntap[1], p.ntap[2], p.ntap[3], words, last_seg};
  for (int i = 0; i < std::min(n, 31); ++i) out[i] = v[i];
}

extern "C" int64_t mnb_pk_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t terms) {
  return (int64_t)terms * batch * ((channels + 7) / 8) * h * w * 16;
}

extern "C" int mnb_pk_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w,
                               const mnb_act_qparams* qp, int32_t terms, const float* ch_scale, int32_t phase_split,
                               void* out_pk, uint8_t* bits8, mnb_stream_t stream) {
  return mnb_pk_pack_act_relu(x, batch, channels, h, w, qp, terms, ch_scale, phase_split, 0, out_pk, bits8, stream);
}

extern "C" int mnb_pk_pack_act_relu(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w,
                                    const mnb_act_qparams* qp, int32_t terms, const float* ch_scale, int32_t phase_split,
                                    int32_t relu, void* out_pk, uint8_t* bits8, mnb_stream_t stream) {
  MNB_REQUIRE(x && out_pk, "NULL pk_pack_act pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && terms >= 1 && terms <= 3, "bad pk_pack_act arguments");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(out_pk) & 15) == 0, "packed tensor must be 16-byte aligned");
  if (phase_split) MNB_REQUIRE(((h | w) & 1) == 0, "phase split needs even H and W");
  const int C8 = (channels + 7) / 8;
  const int64_t plane_vecs = (int64_t)batch * C8 * h * w;
  MNB_REQUIRE((int64_t)batch * C8 <= 65535 * 8 && (int64_t)h * w < (1ll << 31), "pk_pack_act: too many (image, octet) planes");
  dim3 blocks, threads;
  if (!unit_grid(batch, C8, h * w, blocks, threads))
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_pack_act: %d (image, octet) planes exceed the grid", batch * C8);
  cudaStream_t st = (cudaStream_t)stream;
  if (qp) {
    MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA || qp->mode == MNB_ACT_IAO || qp->mode == MNB_ACT_SIGN, "unknown activation quantizer");
    if (qp->mode == MNB_ACT_DOREFA) MNB_REQUIRE(qp->bits >= 2 && qp->bits <= 8, "DoReFa a_bits must be in [2,8]");
    const int a_off = qp->mode == MNB_ACT_IAO ? qp->qmin : (qp->mode == MNB_ACT_SIGN ? -1 : 0);
    pk::pack_act_kernel<1><<<blocks, threads, 0, st>>>(x, batch, channels, h, w, C8, terms, nullptr, *qp, a_off, phase_split,
                                                   reinterpret_cast<uint4*>(out_pk), plane_vecs, bits8, relu);
  } else {
    mnb_act_qparams none{};
    pk::pack_act_kernel<0><<<blocks, threads, 0, st>>>(x, batch, channels, h, w, C8, terms, ch_scale, none, 0, phase_split,
                                                   reinterpret_cast<uint4*>(out_pk), plane_vecs, nullptr, relu);
  }
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int64_t mnb_pk_grouped_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t terms, int32_t groups) {
  if (groups < 1 || channels % groups) return -1;
  return (int64_t)terms * batch * groups * ((channels / groups + 7) / 8) * h * w * 16;
}

extern "C" int mnb_pk_pack_act_grouped(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w,
                                       const mnb_act_qparams* qp, int32_t terms, const float* ch_scale, int32_t phase_split,
                                       int32_t relu, void* out_pk, uint8_t* bits8, int32_t groups, mnb_stream_t stream) {
  MNB_REQUIRE(x && out_pk, "NULL pk_pack_act_grouped pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && terms >= 1 && terms <= 3 && groups >= 1 && channels % groups == 0,
              "bad pk_pack_act_grouped arguments");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(out_pk) & 15) == 0, "packed tensor must be 16-byte aligned");
  if (phase_split) MNB_REQUIRE(((h | w) & 1) == 0, "phase split needs even H and W");
  const int cg = channels / groups;
  if (groups == 1 || cg % 8 == 0)   // the padded layout is the plain one: one kernel for it
    return mnb_pk_pack_act_relu(x, batch, channels, h, w, qp, terms, ch_scale, phase_split, relu, out_pk, bits8, stream);
  const int kg8 = (cg + 7) / 8, C8 = groups * kg8;
  const int64_t plane_vecs = (int64_t)batch * C8 * h * w;
  MNB_REQUIRE((int64_t)batch * C8 <= 65535 * 8 && (int64_t)h * w < (1ll << 31), "pk_pack_act_grouped: too many (image, octet) planes");
  dim3 blocks, threads;
  if (!unit_grid(batch, C8, h * w, blocks, threads))
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_pack_act_grouped: %d (image, octet) planes exceed the grid", batch * C8);
  cudaStream_t st = (cudaStream_t)stream;
  if (qp) {
    MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA || qp->mode == MNB_ACT_IAO || qp->mode == MNB_ACT_SIGN, "unknown activation quantizer");
    if (qp->mode == MNB_ACT_DOREFA) MNB_REQUIRE(qp->bits >= 2 && qp->bits <= 8, "DoReFa a_bits must be in [2,8]");
    pk::pack_act_grouped_kernel<1><<<blocks, threads, 0, st>>>(x, batch, channels, h, w, C8, terms, nullptr, *qp, phase_split,
                                                               reinterpret_cast<uint4*>(out_pk), plane_vecs, bits8, relu, cg, kg8);
  } else {
    mnb_act_qparams none{};
    pk::pack_act_grouped_kernel<0><<<blocks, threads, 0, st>>>(x, batch, channels, h, w, C8, terms, ch_scale, none, phase_split,
                                                               reinterpret_cast<uint4*>(out_pk), plane_vecs, nullptr, relu, cg,
                                                               kg8);
  }
  MNB_LAUNCHED(1);
  return 0;
}

template <typename XT>
static int bn_sign_bwd_pack(const float* g, const uint32_t* pass_bits, const XT* x, const float* dec, int32_t batch,
                            int32_t channels, int32_t hw, const float* mean, const float* invstd, const float* gamma,
                            const float* dgamma, const float* dbeta, int32_t out_shuffle_groups, const float* ch_scale,
                            int32_t terms, float* dx, void* dy_packed, mnb_stream_t stream) {
  MNB_REQUIRE(g && pass_bits && x && mean && invstd && gamma && dgamma && dbeta && dy_packed, "NULL bn_sign_bwd_pack pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0 && terms >= 1 && terms <= 3, "bad bn_sign_bwd_pack arguments");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  if (channels % 8 || (reinterpret_cast<uintptr_t>(dy_packed) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "packed BatchNorm backward needs channels %% 8 == 0 and a 16-byte aligned output");
  if (hw % 32) return mnb_fail(MNB_E_UNSUPPORTED, "packed BatchNorm backward needs H*W %% 32 == 0");
  const int c8n = channels / 8;
  auto al = [](const void* p, int a) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(a - 1)) == 0; };
  constexpr int xs = (int)sizeof(XT);   // x is loaded VEC elements at a time
  const int vec = (hw % 128 == 0 && al(g, 16) && al(x, 4 * xs) && al(dx, 16)) ? 4
                  : ((hw % 64 == 0 && al(g, 8) && al(x, 2 * xs) && al(dx, 8)) ? 2 : 1);
  const int64_t warps = (int64_t)batch * c8n * (hw / (32 * vec));
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(warps, 8), (int64_t)MNB_NUM_SMS * 8);
  const float inv_count = 1.f / (float)((int64_t)batch * hw);
  uint4* outp = reinterpret_cast<uint4*>(dy_packed);
  const int64_t plane_vecs = (int64_t)batch * c8n * hw;
  cudaStream_t st = (cudaStream_t)stream;
#define MNB_BWD_PACK(V)                                                                                                          \
  pk::bn_sign_bwd_pack_kernel<V, XT><<<blocks, 256, 0, st>>>(g, pass_bits, x, dec, batch, channels, hw, out_shuffle_groups,     \
                                                             inv_count, mean, invstd, gamma, dgamma, dbeta, ch_scale, terms, dx, \
                                                             outp, plane_vecs)
  if (vec == 4) MNB_BWD_PACK(4); else if (vec == 2) MNB_BWD_PACK(2); else MNB_BWD_PACK(1);
#undef MNB_BWD_PACK
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_sign_bwd_pack(const float* g, const uint32_t* pass_bits, const float* x, int32_t batch, int32_t channels,
                                    int32_t hw, const float* mean, const float* invstd, const float* gamma, const float* dgamma,
                                    const float* dbeta, int32_t out_shuffle_groups, const float* ch_scale, int32_t terms,
                                    float* dx, void* dy_packed, mnb_stream_t stream) {
  return bn_sign_bwd_pack<float>(g, pass_bits, x, nullptr, batch, channels, hw, mean, invstd, gamma, dgamma, dbeta,
                                 out_shuffle_groups, ch_scale, terms, dx, dy_packed, stream);
}

extern "C" int mnb_bn_sign_bwd_pack_codes(const float* g, const uint32_t* pass_bits, const int16_t* codes, const float* dec,
                                          int32_t batch, int32_t channels, int32_t hw, const float* mean, const float* invstd,
                                          const float* gamma, const float* dgamma, const float* dbeta, int32_t out_shuffle_groups,
                                          const float* ch_scale, int32_t terms, float* dx, void* dy_packed, mnb_stream_t stream) {
  MNB_REQUIRE(dec, "NULL decode pair");
  return bn_sign_bwd_pack<int16_t>(g, pass_bits, codes, dec, batch, channels, hw, mean, invstd, gamma, dgamma, dbeta,
                                   out_shuffle_groups, ch_scale, terms, dx, dy_packed, stream);
}

template <typename XT>
static int bn_sign_pool_bwd_pack(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const XT* x, const float* dec,
                                 int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean, const float* invstd,
                                 const float* gamma, const float* dgamma, const float* dbeta, int32_t out_shuffle_groups,
                                 const float* ch_scale, int32_t terms, void* dy_packed, mnb_stream_t stream) {
  MNB_REQUIRE(g && pass_bits && argmax && x && mean && invstd && gamma && dgamma && dbeta && dy_packed, "NULL bn_sign_pool_bwd_pack pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && H > 0 && W > 0 && terms >= 1 && terms <= 3, "bad bn_sign_pool_bwd_pack arguments");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  if ((H & 1) || (W & 7) || channels % 8 || (int64_t)batch * channels * H * W >= (1ll << 31) ||
      (reinterpret_cast<uintptr_t>(x) & (4 * sizeof(XT) - 1)) || (reinterpret_cast<uintptr_t>(dy_packed) & 15) ||
      (reinterpret_cast<uintptr_t>(g) & 7))
    return mnb_fail(MNB_E_UNSUPPORTED, "packed pooled BatchNorm backward needs even H, W %% 8 == 0, channels %% 8 == 0, aligned tensors");
  const int c8n = channels / 8;
  const int64_t total = (int64_t)batch * c8n * (H / 2) * (W / 4);
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(total, 256), (int64_t)MNB_NUM_SMS * 8);
  pk::bn_sign_pool_bwd_pack_kernel<XT><<<blocks, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(g), reinterpret_cast<const uchar2*>(argmax), reinterpret_cast<const uint8_t*>(pass_bits),
      x, dec, batch, channels, H, W / 4, out_shuffle_groups, 1.f / (float)((int64_t)batch * H * W), mean,
      invstd, gamma, dgamma, dbeta, ch_scale, terms, reinterpret_cast<uint4*>(dy_packed), (int64_t)batch * c8n * H * W);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_sign_pool_bwd_pack(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const float* x,
                                         int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean,
                                         const float* invstd, const float* gamma, const float* dgamma, const float* dbeta,
                                         int32_t out_shuffle_groups, const float* ch_scale, int32_t terms, void* dy_packed,
                                         mnb_stream_t stream) {
  return bn_sign_pool_bwd_pack<float>(g, pass_bits, argmax, x, nullptr, batch, channels, H, W, mean, invstd, gamma, dgamma, dbeta,
                                      out_shuffle_groups, ch_scale, terms, dy_packed, stream);
}

extern "C" int mnb_bn_sign_pool_bwd_pack_codes(const float* g, const uint32_t* pass_bits, const uint8_t* argmax,
                                               const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t H,
                                               int32_t W, const float* mean, const float* invstd, const float* gamma,
                                               const float* dgamma, const float* dbeta, int32_t out_shuffle_groups,
                                               const float* ch_scale, int32_t terms, void* dy_packed, mnb_stream_t stream) {
  MNB_REQUIRE(dec, "NULL decode pair");
  return bn_sign_pool_bwd_pack<int16_t>(g, pass_bits, argmax, codes, dec, batch, channels, H, W, mean, invstd, gamma, dgamma,
                                        dbeta, out_shuffle_groups, ch_scale, terms, dy_packed, stream);
}

extern "C" int mnb_quant_add_pack_fwd(const float* a, const float* b, int32_t batch, int32_t channels, int32_t h, int32_t w,
                                      const mnb_act_qparams* qp, int32_t relu, float* out, const mnb_pk_post* post,
                                      mnb_stream_t stream) {
  return quant_add_pack<8>(a, b, batch, channels, h, w, qp, relu, out, post, stream);
}

extern "C" int mnb_bn_relu_quant_pack_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                                          const float* invstd, const float* gamma, const float* beta,
                                          const mnb_act_qparams* qp, int32_t out_shuffle_groups, void* x_packed,
                                          uint32_t* pass_bits, mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && invstd && gamma && beta && qp && x_packed && pass_bits, "NULL bn_relu_quant_pack pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0, "bad bn_relu_quant_pack shape");
  MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA && qp->bits >= 2 && qp->bits <= 8, "the fused producer takes a DoReFa quantizer with 2..8 bits");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  if (channels % 8 || hw % 32 || (reinterpret_cast<uintptr_t>(x_packed) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "fused producer needs channels %% 8 == 0, H*W %% 32 == 0, 16-byte aligned output");
  const int64_t warps = (int64_t)batch * (channels / 8) * (hw / 32);
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(warps, 8), (int64_t)MNB_NUM_SMS * 16);
  pk::bn_relu_quant_pack_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, batch, channels, hw, out_shuffle_groups, mean, invstd,
                                                                       gamma, beta, *qp, pass_bits,
                                                                       reinterpret_cast<uint4*>(x_packed));
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_relu_quant_pack_i8_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                                             const float* invstd, const float* gamma, const float* beta,
                                             const mnb_act_qparams* qp, int32_t out_shuffle_groups, void* x_packed,
                                             mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && invstd && gamma && beta && qp && x_packed, "NULL bn_relu_quant_pack_i8 pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0, "bad bn_relu_quant_pack_i8 shape");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  if (qp->mode != MNB_ACT_DOREFA || !i8_quantizer(qp))
    return mnb_fail(MNB_E_UNSUPPORTED, "bn_relu_quant_pack_i8: the int8 producer takes a DoReFa quantizer with 2..7 bits");
  if (channels % 16 || hw % 32 || (reinterpret_cast<uintptr_t>(x_packed) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "int8 producer needs channels %% 16 == 0, H*W %% 32 == 0, 16-byte aligned output");
  const int64_t warps = (int64_t)batch * (channels / 16) * (hw / 32);
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(warps, 8), (int64_t)MNB_NUM_SMS * 16);
  pk::bn_relu_quant_pack_i8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, batch, channels, hw, out_shuffle_groups, mean,
                                                                          invstd, gamma, beta, *qp,
                                                                          reinterpret_cast<uint4*>(x_packed));
  MNB_LAUNCHED(1);
  return 0;
}

// mnb_pk_plane_maxpool (q_in == NULL) and mnb_pk_plane_maxpool_requant: same cover, same grid
static int plane_maxpool(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k, int32_t s,
                         int32_t p, int32_t int8, const mnb_act_qparams* q_in, const mnb_act_qparams* q_out, void* out_pk,
                         mnb_stream_t stream) {
  MNB_REQUIRE(in_pk && out_pk && in_pk != out_pk, "NULL or aliased pk_plane_maxpool pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0, "bad pk_plane_maxpool shape");
  MNB_REQUIRE(((reinterpret_cast<uintptr_t>(in_pk) | reinterpret_cast<uintptr_t>(out_pk)) & 15) == 0,
              "packed tensors must be 16-byte aligned");
  if (k < 1 || s < 1 || p < 0 || 2 * p > k || h + 2 * p < k || w + 2 * p < k)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_plane_maxpool: kernel %d, stride %d, padding %d on %d x %d (needs 2 * p <= k)", k, s,
                    p, h, w);
  if (q_in) {
    for (const mnb_act_qparams* q : {q_in, q_out})
      if (q->mode != MNB_ACT_IAO || q->q_type != 0 || q->bits < 2 || q->bits > 8 || q->qmin < -128 || q->qmax > 127)
        return mnb_fail(MNB_E_UNSUPPORTED, "pk_plane_maxpool_requant: both quantizers must be symmetric IAO (q_type 0) with "
                                           "2..8 bits and levels in [-128, 127]");
    MNB_REQUIRE(q_in->scale && q_in->zero_point && q_in->obs_min && q_in->obs_max && q_out->scale && q_out->zero_point &&
                    q_out->obs_min && q_out->obs_max,
                "NULL IAO quantizer scalar");
  }
  const int oh = (h + 2 * p - k) / s + 1, ow = (w + 2 * p - k) / s + 1;
  const int64_t planes = (int64_t)batch * ((channels + (int8 ? 15 : 7)) / (int8 ? 16 : 8));
  const int64_t total = planes * oh * ow;
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(total, 256), (int64_t)MNB_NUM_SMS * 16);
  const uint4* src = reinterpret_cast<const uint4*>(in_pk);
  uint4* dst = reinterpret_cast<uint4*>(out_pk);
  if (q_in) {
    auto kern = int8 ? pk::plane_maxpool_requant_kernel<true> : pk::plane_maxpool_requant_kernel<false>;
    kern<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, planes, h, w, k, s, p, oh, ow, dst, *q_in, *q_out);
  } else {
    auto kern = int8 ? pk::plane_maxpool_kernel<true> : pk::plane_maxpool_kernel<false>;
    kern<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, planes, h, w, k, s, p, oh, ow, dst);
  }
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_pk_plane_maxpool(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k,
                                    int32_t s, int32_t p, int32_t int8, void* out_pk, mnb_stream_t stream) {
  return plane_maxpool(in_pk, batch, channels, h, w, k, s, p, int8, nullptr, nullptr, out_pk, stream);
}

extern "C" int mnb_pk_plane_maxpool_requant(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k,
                                            int32_t s, int32_t p, int32_t int8, const mnb_act_qparams* q_in,
                                            const mnb_act_qparams* q_out, void* out_pk, mnb_stream_t stream) {
  MNB_REQUIRE(q_in && q_out, "NULL pk_plane_maxpool_requant quantizer");
  return plane_maxpool(in_pk, batch, channels, h, w, k, s, p, int8, q_in, q_out, out_pk, stream);
}

extern "C" int mnb_pk_plane_maxpool_terms(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k,
                                          int32_t s, int32_t p, int32_t terms, void* out_pk, mnb_stream_t stream) {
  MNB_REQUIRE(in_pk && out_pk && in_pk != out_pk, "NULL or aliased pk_plane_maxpool_terms pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && terms >= 1 && terms <= 3, "bad pk_plane_maxpool_terms arguments");
  MNB_REQUIRE(((reinterpret_cast<uintptr_t>(in_pk) | reinterpret_cast<uintptr_t>(out_pk)) & 15) == 0,
              "packed tensors must be 16-byte aligned");
  if (k < 1 || s < 1 || p < 0 || 2 * p > k || h + 2 * p < k || w + 2 * p < k)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_plane_maxpool_terms: kernel %d, stride %d, padding %d on %d x %d (needs 2 * p <= k)",
                    k, s, p, h, w);
  const int oh = (h + 2 * p - k) / s + 1, ow = (w + 2 * p - k) / s + 1;
  const int64_t planes = (int64_t)batch * ((channels + 7) / 8);
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(planes * oh * ow, 256), (int64_t)MNB_NUM_SMS * 16);
  pk::plane_maxpool_terms_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(in_pk), planes, h, w, k,
                                                                            s, p, oh, ow, terms, reinterpret_cast<uint4*>(out_pk));
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_relu_pack_terms_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                                          const float* invstd, const float* gamma, const float* beta, int32_t relu,
                                          int32_t out_shuffle_groups, int32_t terms, void* x_packed, mnb_stream_t stream) {
  MNB_REQUIRE(x && x_packed, "NULL bn_relu_pack_terms pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0 && terms >= 1 && terms <= 3, "bad bn_relu_pack_terms arguments");
  const int nbn = (mean != nullptr) + (invstd != nullptr) + (gamma != nullptr) + (beta != nullptr);
  MNB_REQUIRE(nbn == 0 || nbn == 4, "bn_relu_pack_terms: the BatchNorm needs all four of mean, invstd, gamma, beta");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(x_packed) & 15) == 0, "packed tensor must be 16-byte aligned");
  MNB_REQUIRE(out_shuffle_groups >= 1, "bn_relu_pack_terms: shuffle groups %d", out_shuffle_groups);
  if (channels % 8 || channels % out_shuffle_groups)
    return mnb_fail(MNB_E_UNSUPPORTED, "bn_relu_pack_terms: needs channels %% 8 == 0 and shuffle groups %d dividing %d channels",
                    out_shuffle_groups, channels);
  const int64_t total = (int64_t)batch * (channels / 8) * hw;
  const int blocks = (int)std::min<int64_t>(mnb_ceil_div(total, 256), (int64_t)MNB_NUM_SMS * 16);
  pk::bn_relu_pack_terms_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, batch, channels, hw, out_shuffle_groups, mean, invstd,
                                                                           gamma, beta, relu, terms,
                                                                           reinterpret_cast<uint4*>(x_packed));
  MNB_LAUNCHED(1);
  return 0;
}

// host only: out[0..15] = {wimg_bytes(lo), wimg_bytes(hi), Nt, n_ntiles, MT, CC, chunks, nstage, smem_bytes, accumulator
//                          columns MT * Nt, TH, TB, BW, n_mtiles, n_items, ny},
//            out[16..20] = {segmented, seg_len, npairs, col_tiles, n_mgroups},
//            out[21..30] = {stage templates (tap groups) of output phases 0..3, filter taps of output phases 0..3, MMA program
//                           words, stages of the last accumulation segment of a phase-0 item (0: not segmented)};
//            the first min(n, 31) are written.  Refuses what mnb_pk_conv refuses on the host, with its code and error text.
static int conv_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int cpu, pk::Plan& pl, int& words);

extern "C" int mnb_pk_conv_plan_ex(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out,
                                   int32_t n) {
  pk::Plan p;
  int words = 0;
  if (int e = conv_plan(s, mode, terms_a, terms_w, 8, p, words)) return e;
  if (out) plan_fields(p, words, out, n);
  return 0;
}

extern "C" int mnb_pk_conv_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out16) {
  return mnb_pk_conv_plan_ex(s, mode, terms_a, terms_w, out16, 16);
}

// -1 where mnb_pk_conv_plan_ex refuses
extern "C" int64_t mnb_pk_wimage_bytes(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w) {
  pk::Plan p;
  int words = 0;
  if (conv_plan(s, mode, terms_a, terms_w, 8, p, words)) return -1;
  return p.wimg_bytes;
}

extern "C" int mnb_pk_pack_weight(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w,
                                  const int16_t* w_int, const float* w_f32, const float* kzero, void* w_img,
                                  mnb_stream_t stream) {
  MNB_REQUIRE((w_int != nullptr) != (w_f32 != nullptr), "exactly one of w_int / w_f32");
  MNB_REQUIRE(w_img && (reinterpret_cast<uintptr_t>(w_img) & 15) == 0, "weight image must be 16-byte aligned");
  pk::PackWParams pp;
  if (int e = pk::make_plan(s, mode, terms_a, terms_w, pp.pl)) return e;
  pp.w_int = w_int; pp.w_f32 = w_f32; pp.kzero = kzero;
  pp.cin_g = s->in_c / s->groups; pp.cout_g = s->out_c / s->groups;
  const int64_t vecs = pp.pl.wimg_bytes / 16;
  const int blocks = (int)std::min<int64_t>((vecs + 255) / 256, (int64_t)MNB_NUM_SMS * 8);
  pk::pack_weight_kernel<8><<<blocks, 256, 0, (cudaStream_t)stream>>>(pp, reinterpret_cast<uint4*>(w_img));
  MNB_LAUNCHED(1);
  return 0;
}

// The epilogue route of a conv launch: the consumer checks of mnb_pk_conv_post / mnb_pk_i8_conv (before anything is
// launched) and the pk_conv_kernel instance row that runs it - 0 plain, 1 segmented (no consumer), 2 int8, 3 XPOST,
// 4 XPOST int8, 5 XTERMS - together with the index range of the kernel's work-item arithmetic.  Host only: the launcher and
// mnb_pk_conv_post_plan share it, so the query refuses what a launch refuses, with the same code and error text.
static int conv_route(const pk::Plan& pl, int32_t mode, const uint8_t* bits8, const mnb_pk_post* post, int cpu, int& row) {
  using namespace pk;
  if (post) {   // BatchNorm and channel shuffle in front of the consumer's quantizer
    const int nbn = (post->bn_mean != nullptr) + (post->bn_invstd != nullptr) + (post->bn_gamma != nullptr) + (post->bn_beta != nullptr);
    MNB_REQUIRE(nbn == 0 || nbn == 4, "pk conv: the consumer's BatchNorm needs all four of mean, invstd, gamma, beta");
    if (nbn) {
      MNB_REQUIRE(((reinterpret_cast<uintptr_t>(post->bn_mean) | reinterpret_cast<uintptr_t>(post->bn_invstd) |
                    reinterpret_cast<uintptr_t>(post->bn_gamma) | reinterpret_cast<uintptr_t>(post->bn_beta)) & 15) == 0,
                  "pk conv: the consumer's BatchNorm arrays must be 16-byte aligned");
      if (pl.NOUT % 4) return unsupported("the consumer's BatchNorm needs output channels % 4 == 0");
    }
    MNB_REQUIRE(post->shuffle_groups >= 0, "pk conv: shuffle groups %d", post->shuffle_groups);
    if (post->shuffle_groups > 1) {
      if (pl.NOUT % post->shuffle_groups) return unsupported("shuffle groups do not divide the output channels");
      if (post->phase_split) return unsupported("channel shuffle in front of a stride-2 consumer");
      if (pl.NOUT % cpu) return unsupported("shuffled consumer plane needs output channels % channels per unit == 0");
    }
  }
  if (post && cpu == 16) {   // int8 consumer plane: s8 levels, 16-channel units
    MNB_REQUIRE(post->q && post->out_pk && (reinterpret_cast<uintptr_t>(post->out_pk) & 15) == 0, "pk conv: consumer plane / quantizer");
    if (!i8_quantizer(post->q)) return unsupported(kI8QuantizerRule);
    if (pl.G > 1 && (pl.ng % 16)) return unsupported("int8 consumer plane of a grouped conv needs channels per group % 16 == 0");
  }
  const bool terms_out = post && !post->q && post->terms_out > 0;    // consumer term planes (no quantizer)
  if (post) {
    MNB_REQUIRE(mode == 0 && !bits8, "pk conv: a fused consumer is a forward-only (inference) option");
    MNB_REQUIRE(post->out_pk && (reinterpret_cast<uintptr_t>(post->out_pk) & 15) == 0, "pk conv: consumer plane");
    if (terms_out) {
      MNB_REQUIRE(post->terms_out <= 3, "pk conv: %d consumer term planes (1..3)", post->terms_out);
      // the XTERMS epilogue stores whole 8-channel units without a per-channel tail (grouped or not)
      if (pl.ng % 8) return unsupported("consumer term planes need output channels per group % 8 == 0");
    } else {
      MNB_REQUIRE(post->q && post->terms_out == 0, "pk conv: a consumer quantizer, or terms_out without one");
      MNB_REQUIRE(post->q->mode == MNB_ACT_DOREFA || post->q->mode == MNB_ACT_IAO, "pk conv: consumer quantizer must be DoReFa or IAO");
      MNB_REQUIRE(post->q->bits >= 2 && post->q->bits <= 8, "pk conv: consumer levels must fit one bf16 piece (2..8 bits)");
    }
    if (pl.G > 1 && (pl.ng % 8)) return unsupported("fused consumer of a grouped conv needs channels per group % 8 == 0");
    if (post->phase_split && ((pl.OH | pl.OW) & 1)) return unsupported("stride-2 consumer of an odd-sized plane");
    // the consumer epilogue is compiled into the single-product kernels only: in the segmented ones (several piece
    // products, e.g. an asymmetric-IAO producer whose levels take two pieces) it costs register spills on every launch
    if (pl.segmented) return unsupported("fused consumer of a segmented (multi-piece) plan");
  }
  int ki = -1;
  for (int i = 0; i < 6; ++i) if (kNtSizes[i] == pl.Nt) ki = i;
  if (ki < 0 || pl.MT * pl.Nt > 128) return mnb_fail(MNB_E_ARG, "pk conv: plan with Nt %d, MT %d", pl.Nt, pl.MT);
  if (pl.n_items >= (1 << 22) || pl.n_mtiles >= (1 << 22))     // FastDiv's exact range (fp32 reciprocal + one correction step)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk conv: %d work items / %d M tiles exceed the index arithmetic of the kernel", pl.n_items, pl.n_mtiles);
  const bool xpost = post && (post->bn_mean || post->shuffle_groups > 1);   // (segmented plans refuse a post above)
  row = terms_out ? 5 : cpu == 16 ? (xpost ? 4 : 2) : (pl.segmented ? 1 : (xpost ? 3 : 0));
  return 0;
}

// The MMA warpgroups' parameter block of a plan, with its program: one word per (piece pair, tap, K-step) of every stage
// template.  Host only: the launcher writes it into the kernel's parameters and the plan queries build it too, so that a
// program that does not fit (length or 16-bit offsets) is refused by the query with the launch's code and error text.
// words: program words used (each template padded to a group of four).
static int conv_mma(const pk::Plan& pl, int cpu, pk::ConvParams::Mma& m, int& words) {
  using namespace pk;
  memset(&m, 0, sizeof(m));
  m.n_items = pl.n_items; m.chunks = pl.chunks; m.ksteps = pl.ksteps; m.MT = pl.MT; m.Nt = pl.Nt; m.npairs = pl.npairs;
  m.st_mask = pl.nstage - 1; m.st_log2 = pl.st_log2; m.stage16 = pl.stage_bytes >> 4;
  m.a_term16 = pl.a_bytes >> 4; m.a_mt16 = (pl.TA * pl.a_bytes) >> 4; m.a_k16 = 2 * pl.npos;
  m.b_off16 = pl.b_off >> 4; m.b_tap16 = (pl.CC / cpu) * pl.Nt; m.b_k16 = 2 * pl.Nt;
  m.a_lbo = (uint32_t)pl.npos * 16u; m.b_lbo = (uint32_t)pl.Nt * 16u;
  m.seg_len = (uint32_t)pl.seg_len;
  int nprog = 0;
  uint32_t* prog = reinterpret_cast<uint32_t*>(m.prog4);
  for (int i = 0; i < MAXPROG; ++i) prog[i] = 0xffffffffu;    // padding words: no MMA
  for (int y = 0; y < pl.ny; ++y) {
    m.ntmpl[y] = pl.ntmpl[y];
    for (int t = 0; t < pl.ntmpl[y]; ++t) {
      const Tmpl& tp = pl.tmpl[y][t];
      const int cnt = tp.ntap * pl.npairs * pl.ksteps;
      nprog = (nprog + 3) & ~3;                       // every template starts on a group of four words
      m.tmpl_begin[y][t] = (uint16_t)(nprog / 4); m.tmpl_cnt[y][t] = (uint16_t)((cnt + 3) / 4);
      if (nprog + ((cnt + 3) & ~3) > MAXPROG) return unsupported("MMA program longer than 512 entries");
      for (int pr = 0; pr < pl.npairs; ++pr)          // piece pairs outermost: small products first
        for (int i = 0; i < tp.ntap; ++i)
          for (int j = 0; j < pl.ksteps; ++j) {
            const uint32_t a16 = (uint32_t)pl.tap_aoff[y][tp.tap0 + i] + (uint32_t)pl.pair_a[pr] * m.a_term16 + (uint32_t)j * m.a_k16;
            const uint32_t b16 = (uint32_t)i * m.b_tap16 + (uint32_t)pl.pair_b[pr] * (uint32_t)tp.ntap * m.b_tap16 + (uint32_t)j * m.b_k16;
            if (a16 > 0xffffu || b16 > 0xffffu) return mnb_fail(MNB_E_ARG, "pk conv: MMA program offset overflow");
            prog[nprog++] = a16 | (b16 << 16);
          }
    }
  }
  words = (nprog + 3) & ~3;
  return 0;
}

// The plan of a plain (no consumer) pk_conv_kernel launch and everything that launch refuses on the host: make_plan,
// conv_route and the MMA program.  The plan queries and the weight-image size use it.  words: as conv_mma.
static int conv_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int cpu, pk::Plan& pl, int& words) {
  if (int e = pk::make_plan(s, mode, terms_a, terms_w, pl, cpu)) return e;
  int row = 0;
  if (int e = conv_route(pl, mode, nullptr, nullptr, cpu, row)) return e;
  pk::ConvParams::Mma m;   // the program itself is not kept (2.4 KB on the stack: queries may run on any host thread)
  return conv_mma(pl, cpu, m, words);
}

static int pk_conv_impl(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img,
                        int32_t terms_w, const float* n_scale, const float* a_scale, float a_scale_const,
                        const float* bias, const uint8_t* bits8, float gain, float* out, const mnb_pk_post* post,
                        int32_t* err_flag, mnb_stream_t stream, int cpu = 8, int16_t* codes = nullptr, float* dec = nullptr) {
  using namespace pk;
  MNB_REQUIRE(s && a_pk && w_img && (out || post || codes) && err_flag, "NULL pk_conv pointer");
  Plan pl;
  if (int e = make_plan(s, mode, terms_a, terms_w, pl, cpu)) return e;
  if (codes) {
    MNB_REQUIRE(mode == 0 && cpu == 8 && !out && !post && !bits8 && dec, "pk conv: int16 codes are a plain forward output");
    // the int16 store is compiled into the single-product kernels only; one piece per operand keeps the sums exact integers
    if (pl.segmented || terms_a != 1 || terms_w != 1)
      return unsupported("int16 codes need one activation piece, one weight piece and a non-segmented plan");
  }
  int row = 0;
  if (int e = conv_route(pl, mode, bits8, post, cpu, row)) return e;
  const bool terms_out = row == 5;
  static ConvParams p;   // large POD: filled per call (single host thread per process)
  memset(&p, 0, sizeof(p));
  int nprog = 0;
  if (int e = conv_mma(pl, cpu, p.m, nprog)) return e;
  for (int y = 0; y < pl.ny; ++y) {
    p.ntmpl[y] = pl.ntmpl[y];
    for (int t = 0; t < pl.ntmpl[y]; ++t) {
      const Tmpl& tp = pl.tmpl[y][t];
      p.tmpl_kph[y][t] = tp.kph; p.tmpl_blk_off[y][t] = tp.blk_off; p.tmpl_blk_bytes[y][t] = tp.blk_bytes;
    }
    p.img_bytes[y] = pl.img_bytes[y]; p.y_off[y] = pl.y_off[y];
  }
  p.n_items = pl.n_items; p.n_ntiles = pl.n_ntiles; p.G = pl.G; p.MT = pl.MT; p.TA = pl.TA; p.chunks = pl.chunks;
  p.CC8 = pl.CC / cpu; p.C8A = pl.C8A; p.kg8 = ceil_div(pl.kg, cpu); p.stage_bytes = pl.stage_bytes; p.a_bytes = pl.a_bytes;
  p.a_box_bytes = pl.a_box_bytes; p.b_off = pl.b_off; p.st_mask = pl.nstage - 1; p.st_log2 = pl.st_log2;
  p.Wt = pl.Wt; p.TH = pl.TH; p.TB = pl.TB; p.wlo = pl.wlo; p.hlo = pl.hlo; p.col_tiles = pl.col_tiles; p.row_tiles = pl.row_tiles;
  p.n_mtiles = pl.n_mtiles;
  p.w_img = reinterpret_cast<const uint8_t*>(w_img);
  p.B = pl.B; p.THH = pl.THH; p.BW = pl.BW; p.OHr = pl.OHr; p.OWr = pl.OWr; p.OH = pl.OH; p.OW = pl.OW; p.omul = pl.omul; p.ny = pl.ny;
  // units per position of the output-side planes: the STE mask of a data gradient is group-padded like its operand plane
  p.ng = pl.ng; p.Nt = pl.Nt; p.NOUT = pl.NOUT; p.C8O = cpu == 8 ? pl.G * ceil_div(pl.ng, 8) : ceil_div(pl.NOUT, cpu); p.smem_bytes = pl.smem_bytes; p.off_stg = pl.off_stg;
  p.mode = mode;
  p.n_scale = n_scale; p.a_scale = a_scale; p.a_scale_const = a_scale_const; p.bias = bias; p.bits8 = bits8; p.gain = gain;
  p.out = out; p.err = err_flag; p.codes = codes; p.dec = dec;
  if (post) {
    p.post_out = reinterpret_cast<uint4*>(post->out_pk); p.post_relu = post->relu; p.post_split = post->phase_split;
    if (!terms_out) p.post_q = *post->q;
    p.post_mean = post->bn_mean; p.post_invstd = post->bn_invstd; p.post_gamma = post->bn_gamma; p.post_beta = post->bn_beta;
    p.post_sg = post->shuffle_groups;
    p.post_terms = terms_out ? post->terms_out : 0;
  }
  { static const int dbg = [] { const char* e = getenv("MNB_PK_DEBUG"); return e ? atoi(e) : 0; }(); p.dbg = dbg; }
  CUtensorMap tm[3];
  const int C8tot = pl.nkph * pl.C8A;
  const int64_t plane_bytes = (int64_t)pl.B * C8tot * pl.HA * pl.WA * 16;
  for (int t = 0; t < 3; ++t) {
    const int tt = t < pl.TA ? t : 0;
    if (int e = make_pk_tmap(&tm[t], a_pk, plane_bytes, tt, pl.B, C8tot, pl.HA, pl.WA, pl.BW, pl.THH, pl.TB, pl.CC / cpu)) return e;
  }
  const int gx = std::max(1, std::min(pl.n_items, MNB_NUM_SMS / pl.ny));
  using ConvFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const ConvParams);
#define MNB_PK_CONV_FNS(SEG, I8, X, T) {pk_conv_kernel<SEG, 16, I8, X, T>, pk_conv_kernel<SEG, 32, I8, X, T>,                       \
                                        pk_conv_kernel<SEG, 48, I8, X, T>, pk_conv_kernel<SEG, 64, I8, X, T>,                       \
                                        pk_conv_kernel<SEG, 96, I8, X, T>, pk_conv_kernel<SEG, 128, I8, X, T>}
  static const ConvFn fns[6][6] = {MNB_PK_CONV_FNS(false, false, false, false), MNB_PK_CONV_FNS(true, false, false, false),
                                   MNB_PK_CONV_FNS(false, true, false, false), MNB_PK_CONV_FNS(false, false, true, false),
                                   MNB_PK_CONV_FNS(false, true, true, false), MNB_PK_CONV_FNS(false, false, false, true)};
#undef MNB_PK_CONV_FNS
  int ki = 0;
  while (kNtSizes[ki] != pl.Nt) ++ki;     // (conv_route refuses any other N tile)
  const ConvFn fn = fns[row][ki];
  if (int e = set_max_smem(fn, kSmemBudget)) return e;
  fn<<<dim3(gx, pl.ny), kConvThreads, pl.smem_bytes, (cudaStream_t)stream>>>(tm[0], tm[1], tm[2], p);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_pk_conv(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img,
                           int32_t terms_w, const float* n_scale, const float* a_scale, float a_scale_const,
                           const float* bias, const uint8_t* bits8, float gain, float* out, int32_t* err_flag,
                           mnb_stream_t stream) {
  MNB_REQUIRE(out, "NULL pk_conv output");
  return pk_conv_impl(s, mode, a_pk, terms_a, w_img, terms_w, n_scale, a_scale, a_scale_const, bias, bits8, gain, out, nullptr,
                      err_flag, stream);
}

extern "C" int mnb_pk_conv_post(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                                const float* n_scale, const float* a_scale, float a_scale_const, const float* bias,
                                float* out, const mnb_pk_post* post, int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(post, "NULL consumer description");
  return pk_conv_impl(s, 0, a_pk, terms_a, w_img, terms_w, n_scale, a_scale, a_scale_const, bias, nullptr, 1.f, out, post,
                      err_flag, stream);
}

// host only: out = {epilogue path (conv_route's instance row), Nt, MT, n_mtiles, n_items, ny, col_tiles, n_ntiles, CTAs per
//            output phase, segmented}; the first min(n, 10) are written
extern "C" int mnb_pk_conv_post_plan(const mnb_conv_shape* s, int32_t terms_a, int32_t terms_w, int32_t cpu,
                                     const mnb_pk_post* post, int32_t* out, int32_t n) {
  MNB_REQUIRE(s && (cpu == 8 || cpu == 16), "pk conv post plan: shape, 8 or 16 channels per unit");
  pk::Plan pl;
  if (int e = pk::make_plan(s, 0, terms_a, terms_w, pl, cpu)) return e;
  int row = 0;
  if (int e = conv_route(pl, 0, nullptr, post, cpu, row)) return e;
  pk::ConvParams::Mma m;   // (not kept: see conv_plan)
  int words = 0;
  if (int e = conv_mma(pl, cpu, m, words)) return e;
  if (out) {
    const int gx = std::max(1, std::min(pl.n_items, MNB_NUM_SMS / pl.ny));
    const int v[10] = {row, pl.Nt, pl.MT, pl.n_mtiles, pl.n_items, pl.ny, pl.col_tiles, pl.n_ntiles, gx, pl.segmented};
    for (int i = 0; i < std::min(n, 10); ++i) out[i] = v[i];
  }
  return 0;
}

extern "C" int mnb_pk_conv_codes(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                                 const float* n_scale, const float* a_scale, float a_scale_const, const float* bias,
                                 int32_t level_bound, int16_t* codes, float* dec, int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(s && codes && dec, "NULL pk_conv_codes pointer");
  MNB_REQUIRE(level_bound >= 1 && s->groups >= 1, "pk_conv_codes: level bound %d", level_bound);
  // |sum| <= (C/g) * R * S * max|level| for a +-1 activation plane: the bound under which every sum is an exact int16
  if ((int64_t)(s->in_c / s->groups) * s->ker_h * s->ker_w * level_bound > 32767)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_conv_codes: sums of %d x %d x %d terms of level %d may exceed int16", s->in_c / s->groups,
                    s->ker_h, s->ker_w, level_bound);
  return pk_conv_impl(s, 0, a_pk, terms_a, w_img, terms_w, n_scale, a_scale, a_scale_const, bias, nullptr, 1.f, nullptr, nullptr,
                      err_flag, stream, 8, codes, dec);
}

// ---- int8 operands (inference): symmetric IAO levels as s8, s8 x s8 -> s32 wgmma

extern "C" int64_t mnb_pk_i8_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w) {
  return (int64_t)batch * ((channels + 15) / 16) * h * w * 16;
}

extern "C" int mnb_pk_i8_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_act_qparams* qp,
                                  int32_t phase_split, int32_t relu, void* out_pk, mnb_stream_t stream) {
  MNB_REQUIRE(x && qp && out_pk, "NULL pk_i8_pack_act pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0, "bad pk_i8_pack_act arguments");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(out_pk) & 15) == 0, "packed tensor must be 16-byte aligned");
  if (!i8_quantizer(qp)) return mnb_fail(MNB_E_UNSUPPORTED, "pk_i8_pack_act: %s", kI8QuantizerRule);
  if (phase_split) MNB_REQUIRE(((h | w) & 1) == 0, "phase split needs even H and W");
  MNB_REQUIRE((int64_t)h * w < (1ll << 31), "pk_i8_pack_act: plane too large");
  const int C16 = (channels + 15) / 16;
  dim3 blocks, threads;
  if (!unit_grid(batch, C16, h * w, blocks, threads))
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_i8_pack_act: %d (image, unit) planes exceed the grid", batch * C16);
  pk::pack_act_i8_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(x, batch, channels, h, w, C16, *qp, phase_split,
                                                                               relu, reinterpret_cast<uint4*>(out_pk));
  MNB_LAUNCHED(1);
  return 0;
}

// host only: the fields of mnb_pk_conv_plan_ex for the int8 forward; refuses what mnb_pk_i8_conv refuses without a consumer
extern "C" int mnb_pk_i8_conv_plan(const mnb_conv_shape* s, int32_t* out, int32_t n) {
  pk::Plan p;
  int words = 0;
  if (int e = conv_plan(s, 0, 1, 1, 16, p, words)) return e;
  if (out) plan_fields(p, words, out, n);
  return 0;
}

extern "C" int64_t mnb_pk_i8_wimage_bytes(const mnb_conv_shape* s) {
  pk::Plan p;
  int words = 0;
  if (conv_plan(s, 0, 1, 1, 16, p, words)) return -1;
  return p.wimg_bytes;
}

extern "C" int mnb_pk_i8_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream) {
  MNB_REQUIRE(w_int, "NULL pk_i8_pack_weight levels");
  MNB_REQUIRE(w_img && (reinterpret_cast<uintptr_t>(w_img) & 15) == 0, "weight image must be 16-byte aligned");
  pk::PackWParams pp;
  if (int e = pk::make_plan(s, 0, 1, 1, pp.pl, 16)) return e;
  pp.w_int = w_int; pp.w_f32 = nullptr; pp.kzero = nullptr;
  pp.cin_g = s->in_c / s->groups; pp.cout_g = s->out_c / s->groups;
  const int64_t vecs = pp.pl.wimg_bytes / 16;
  const int blocks = (int)std::min<int64_t>((vecs + 255) / 256, (int64_t)MNB_NUM_SMS * 8);
  pk::pack_weight_kernel<16><<<blocks, 256, 0, (cudaStream_t)stream>>>(pp, reinterpret_cast<uint4*>(w_img));
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_pk_i8_conv(const mnb_conv_shape* s, const void* a_pk, const void* w_img, const float* n_scale,
                              const float* a_scale, float a_scale_const, const float* bias, float* out, const mnb_pk_post* post,
                              int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(out || post, "pk_i8_conv: NULL out needs a consumer plane (post)");
  return pk_conv_impl(s, 0, a_pk, 1, w_img, 1, n_scale, a_scale, a_scale_const, bias, nullptr, 1.f, out, post, err_flag, stream, 16);
}

extern "C" int mnb_quant_add_pack_i8_fwd(const float* a, const float* b, int32_t batch, int32_t channels, int32_t h, int32_t w,
                                         const mnb_act_qparams* qp, int32_t relu, float* out, const mnb_pk_post* post,
                                         mnb_stream_t stream) {
  return quant_add_pack<16>(a, b, batch, channels, h, w, qp, relu, out, post, stream);
}

extern "C" int64_t mnb_pk_wgrad_scratch_bytes(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x) {
  pk::WgPlan p;
  if (pk::make_wg_plan(s, terms_dy, terms_x, p)) return -1;
  return p.partial_floats * 4;
}

// host only: out = {Nc, n_ctiles, tpg, n_tg, gm, splits, NI, nstage, BW, TH, n_ktiles, nkph_used, stg_per_split, nsub,
//                   issue-program entries (uint4: piece pairs x tap groups x ceil(tpg / 4)), nstg_total};
//            the first min(n, 16) are written.  Refuses what mnb_pk_wgrad refuses on the host, with its code and error text.
extern "C" int mnb_pk_wgrad_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t* out, int32_t n) {
  pk::WgPlan p;
  if (int e = pk::make_wg_plan(s, terms_dy, terms_x, p)) return e;
  if (out) {
    const int v[16] = {p.Nc, p.n_ctiles, p.tpg, p.n_tg, p.gm, p.splits, p.NI, p.nstage, p.BW, p.TH, p.n_ktiles, p.nkph_used,
                       p.stg_per_split, p.nsub, p.npairs * p.n_tg * ((p.tpg + 3) / 4), p.nstg_total};
    for (int i = 0; i < std::min(n, 16); ++i) out[i] = v[i];
  }
  return 0;
}

// dw[k][c][r][s] = mul(k) * sum_{b,p,q} dy[b,k,p,q] * x[b,c,p*st+r-pad, q*st+s-pad];  mul(k) = a_scale[0] / kdiv[k]
// (a_scale: activation scale when x_pk holds integer levels; kdiv: the per-channel factor dy_pk was pre-multiplied with)
extern "C" int mnb_pk_wgrad(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                            const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag,
                            mnb_stream_t stream) {
  using namespace pk;
  MNB_REQUIRE(s && dy_pk && x_pk && dw && scratch && err_flag, "NULL pk_wgrad pointer");
  WgPlan pl;
  if (int e = make_wg_plan(s, terms_dy, terms_x, pl)) return e;
  static WgParams p;
  memset(&p, 0, sizeof(p));
  WgParams::Mma& m = p.m;
  m.stg_per_split = pl.stg_per_split; m.nstg_total = pl.nstg_total; m.NI = pl.NI; m.ksteps = pl.rows_dy / 16; m.ntap = pl.ntap;
  m.Nc = pl.Nc; m.tpg = pl.tpg; m.n_tg = pl.n_tg; m.npairs = pl.npairs; m.st_mask = pl.nstage - 1; m.st_log2 = pl.st_log2; m.stage16 = pl.stage_bytes >> 4;
  m.sub16 = pl.sub_bytes >> 4; m.dy_term16 = pl.dy_bytes >> 4; m.x_off16 = (pl.TA * pl.dy_bytes) >> 4;
  m.x_term16 = (pl.nkph_used * pl.x_bytes) >> 4; m.x_kph16 = pl.x_bytes >> 4;
  m.dy_sbo = (uint32_t)pl.rows_dy * 16u; m.x_sbo = (uint32_t)pl.rows_x * 16u; m.nsub = pl.nsub;
  for (int i = 0; i < pl.npairs; ++i) { m.pair_a16[i] = pl.pair_a[i] * m.dy_term16; m.pair_b16[i] = pl.pair_b[i] * m.x_term16; }
  {
    m.g4 = (uint32_t)ceil_div(pl.tpg, 4);      // (make_wg_plan_nc refuses programs longer than progb4)
    uint32_t* prog = reinterpret_cast<uint32_t*>(m.progb4);
    for (size_t i = 0; i < sizeof(m.progb4) / 4; ++i) prog[i] = 0xffffffffu;
    for (int i = 0; i < pl.npairs; ++i)
      for (int tg = 0; tg < pl.n_tg; ++tg)
        for (int tt = 0; tt < pl.tpg && tg * pl.tpg + tt < pl.ntap; ++tt) {
          const int t = tg * pl.tpg + tt;
          prog[((size_t)(i * pl.n_tg + tg) * m.g4) * 4 + tt] = m.pair_b16[i] + pl.kph_slot[pl.tap_kph[t]] * m.x_kph16 + pl.tap_off[t];
        }
  }
  p.G = pl.G; p.n_ktiles = pl.n_ktiles; p.n_ctiles = pl.n_ctiles; p.n_tg = pl.n_tg; p.tpg = pl.tpg; p.splits = pl.splits; p.stg_per_split = pl.stg_per_split;
  p.nstg_total = pl.nstg_total; p.NI = pl.NI; p.nsub = pl.nsub; p.row_tiles = pl.row_tiles; p.TA = pl.TA; p.TX = pl.TX;
  p.nkph_used = pl.nkph_used;
  for (int i = 0; i < 4; ++i) p.kph_used[i] = pl.kph_used[i];
  p.K8 = pl.K8; p.C8X = pl.C8X; p.cout_g8 = pl.cout_g / 8; p.cin_g8 = pl.cin_g / 8; p.Nc8 = pl.Nc / 8; p.TH = pl.TH; p.hlo = pl.hlo;
  p.wlo = pl.wlo; p.stage_bytes = pl.stage_bytes; p.sub_bytes = pl.sub_bytes; p.dy_bytes = pl.dy_bytes; p.x_bytes = pl.x_bytes;
  p.dy_box_bytes = pl.dy_box_bytes; p.x_box_bytes = pl.x_box_bytes; p.st_mask = pl.nstage - 1; p.st_log2 = pl.st_log2;
  p.smem_bytes = pl.smem_bytes; p.ntap = pl.ntap; p.Nc = pl.Nc; p.cout_g = pl.cout_g; p.cin_g = pl.cin_g;
  p.partial = reinterpret_cast<float*>(scratch); p.err = err_flag;
  CUtensorMap tdy[3], tx[3];
  const int64_t dy_plane = (int64_t)pl.B * pl.K8 * pl.P * pl.Q * 16;
  const int C8tot = pl.nkph * pl.C8X;
  const int64_t x_plane = (int64_t)pl.B * C8tot * pl.HX * pl.WX * 16;
  for (int t = 0; t < 3; ++t) {
    if (int e = make_pk_tmap(&tdy[t], dy_pk, dy_plane, t < pl.TA ? t : 0, pl.B, pl.K8, pl.P, pl.Q, pl.BW, pl.TH, 1, 16)) return e;
    if (int e = make_pk_tmap(&tx[t], x_pk, x_plane, t < pl.TX ? t : 0, pl.B, C8tot, pl.HX, pl.WX, pl.BW, pl.THH, 1, pl.Nc / 8)) return e;
  }
  using WgFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                        const CUtensorMap, const WgParams);
  static const WgFn wfns[8] = {pk_wgrad_kernel<16>, pk_wgrad_kernel<32>, pk_wgrad_kernel<48>, pk_wgrad_kernel<64>,
                               pk_wgrad_kernel<80>, pk_wgrad_kernel<96>, pk_wgrad_kernel<112>, pk_wgrad_kernel<128>};
  if (pl.Nc % 16 || pl.Nc < 16 || pl.Nc > 128) return mnb_fail(MNB_E_ARG, "pk wgrad: plan with Nc %d", pl.Nc);
  const WgFn wfn = wfns[pl.Nc / 16 - 1];
  if (int e = set_max_smem(wfn, kSmemBudget)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  wfn<<<dim3(pl.G * pl.n_ktiles * pl.n_ctiles * pl.n_tg, pl.splits), kWgThreads, pl.smem_bytes, st>>>(tdy[0], tdy[1], tdy[2], tx[0],
                                                                                                     tx[1], tx[2], p);
  {
    const dim3 rgrid(pl.cin_o * pl.ntap, (pl.cout_o + 127) / 128, pl.G * pl.gm);
    wg_reduce_kernel<<<rgrid, 128, 0, st>>>(p.partial, pl.splits, pl.G, pl.gm, pl.n_ktiles, pl.n_ctiles, pl.ntap, pl.Nc, pl.cout_o,
                                            pl.cin_o, pl.cout_g / pl.gm, pl.cin_g / pl.gm, a_scale, kdiv, dw);
  }
  MNB_LAUNCHED(2);
  return 0;
}

// host only: out = {blocks, splits, NI, nstage, BW, TH, stg_per_split, smem_bytes, accumulators per MMA thread,
//                   scratch bytes (lo), scratch bytes (hi), npairs}; the first min(n, 12) are written
extern "C" int mnb_pk_wgrad_taps_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t* out, int32_t n) {
  pk::WgPlan p;
  if (int e = pk::make_wgt_plan(s, terms_dy, terms_x, p)) return e;
  if (out) {
    const int64_t sb = p.partial_floats * 4;
    const int v[12] = {p.G, p.splits, p.NI, p.nstage, p.BW, p.TH, p.stg_per_split, p.smem_bytes, pk::kTapsN * 16,
                       (int)(sb & 0x7fffffff), (int)(sb >> 31), p.npairs};
    for (int i = 0; i < std::min(n, 12); ++i) out[i] = v[i];
  }
  return 0;
}

// mnb_pk_wgrad for the shapes of mnb_pk_wgrad_taps_plan's cover (same operands, the same result bit for bit: same chains,
// same batch splits, same reduction); scratch: the plan's scratch bytes
extern "C" int mnb_pk_wgrad_taps(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                                 const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag,
                                 mnb_stream_t stream) {
  using namespace pk;
  MNB_REQUIRE(s && dy_pk && x_pk && dw && scratch && err_flag, "NULL pk_wgrad_taps pointer");
  WgPlan pl;
  if (int e = make_wgt_plan(s, terms_dy, terms_x, pl)) return e;
  WgtParams p;
  memset(&p, 0, sizeof(p));
  p.stg_per_split = pl.stg_per_split; p.nstg_total = pl.nstg_total; p.NI = pl.NI; p.nsub = pl.nsub; p.ksteps = pl.rows_dy / 16;
  p.npairs = pl.npairs; p.nstage = pl.nstage; p.stage16 = pl.stage_bytes >> 4; p.sub16 = pl.sub_bytes >> 4;
  p.dy_sbo = (uint32_t)pl.rows_dy * 16u; p.x_sbo = (uint32_t)pl.rows_x * 16u; p.x_off16 = (pl.TA * pl.dy_bytes) >> 4;
  for (int i = 0; i < pl.npairs; ++i) {
    p.pair_a16[i] = (uint32_t)(pl.pair_a[i] * pl.dy_bytes) >> 4;
    p.pair_b16[i] = (uint32_t)(pl.pair_b[i] * pl.x_bytes) >> 4;
  }
  for (int t = 0; t < kTapsN; ++t) p.tap16[t] = (uint32_t)pl.tap_off[t];
  p.row_tiles = pl.row_tiles; p.TA = pl.TA; p.TX = pl.TX; p.TH = pl.TH; p.hlo = pl.hlo; p.wlo = pl.wlo;
  p.stage_bytes = pl.stage_bytes; p.sub_bytes = pl.sub_bytes; p.dy_bytes = pl.dy_bytes; p.x_bytes = pl.x_bytes;
  p.dy_box_bytes = pl.dy_box_bytes; p.x_box_bytes = pl.x_box_bytes; p.smem_bytes = pl.smem_bytes;
  p.partial = reinterpret_cast<float*>(scratch); p.err = err_flag;
  CUtensorMap tdy[3], tx[3];
  const int64_t dy_plane = (int64_t)pl.B * pl.K8 * pl.P * pl.Q * 16;
  const int64_t x_plane = (int64_t)pl.B * pl.C8X * pl.HX * pl.WX * 16;
  for (int t = 0; t < 3; ++t) {
    if (int e = make_pk_tmap(&tdy[t], dy_pk, dy_plane, t < pl.TA ? t : 0, pl.B, pl.K8, pl.P, pl.Q, pl.BW, pl.TH, 1, 16)) return e;
    if (int e = make_pk_tmap(&tx[t], x_pk, x_plane, t < pl.TX ? t : 0, pl.B, pl.C8X, pl.HX, pl.WX, pl.BW, pl.THH, 1, 8)) return e;
  }
  if (int e = set_max_smem(pk_wgrad_taps_kernel, kSmemBudget)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  pk_wgrad_taps_kernel<<<dim3(pl.G, pl.splits), kWgtThreads, pl.smem_bytes, st>>>(tdy[0], tdy[1], tdy[2], tx[0], tx[1], tx[2], p);
  const dim3 rgrid(kTapsCin * kTapsN, 1, pl.G * kTapsGm);
  wg_reduce_kernel<<<rgrid, 128, 0, st>>>(p.partial, pl.splits, pl.G, kTapsGm, 1, 1, kTapsN, pl.Nc, kTapsCout, kTapsCin, kTapsCout,
                                          kTapsCin, a_scale, kdiv, dw);
  MNB_LAUNCHED(2);
  return 0;
}

// ---- data and weight gradient of 1x1 grouped convolutions in one pass over dy (pk_bwd1x1_kernel)

// host only: out = {groups, splits, NI, nstage, BW, TH, stg_per_split, smem_bytes, nsub, nstg_total, data-gradient MMAs per
// chain, scratch bytes (lo), scratch bytes (hi), npairs (wgrad), N tile}; the first min(n, 15) are written.  Refuses what
// mnb_pk_bwd1x1 refuses on the host, with its code and error text.
extern "C" int mnb_pk_bwd1x1_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t terms_w, int32_t* out,
                                  int32_t n) {
  pk::BwdPlan b;
  if (int e = pk::make_bwd_plan(s, terms_dy, terms_x, terms_w, b)) return e;
  if (out) {
    const pk::WgPlan& w = b.wg;
    const int64_t sb = w.partial_floats * 4;
    const int v[15] = {w.G, w.splits, w.NI, b.nstage, w.BW, w.TH, w.stg_per_split, b.smem_bytes, w.nsub, w.nstg_total, b.nprog,
                       (int)(sb & 0x7fffffff), (int)(sb >> 31), w.npairs, w.Nc};
    for (int i = 0; i < std::min(n, 15); ++i) out[i] = v[i];
  }
  return 0;
}

// mnb_pk_conv (mode 1, data gradient into dx) followed by mnb_pk_wgrad (into dw) for the shapes of mnb_pk_bwd1x1_plan's cover,
// with the same operands - w_img: the data-gradient weight image of mnb_pk_pack_weight (mode 1, terms_dy, terms_w) - and the
// same results bit for bit.  The data-gradient epilogue is the one mnb_pk_conv runs without n_scale, a_scale or bias:
// dx = acc * a_scale_const, or with bits8 (STE mask) dx = pass ? acc * gain : 0.  scratch: the plan's scratch bytes.
extern "C" int mnb_pk_bwd1x1(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                             const void* w_img, int32_t terms_w, float a_scale_const, const uint8_t* bits8, float gain, float* dx,
                             const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag,
                             mnb_stream_t stream) {
  using namespace pk;
  MNB_REQUIRE(s && dy_pk && x_pk && w_img && dx && dw && scratch && err_flag, "NULL pk_bwd1x1 pointer");
  BwdPlan b;
  if (int e = make_bwd_plan(s, terms_dy, terms_x, terms_w, b)) return e;
  const WgPlan& pl = b.wg;
  const Plan& d = b.dg;
  static BwdParams p;   // filled per call (single host thread per process)
  memset(&p, 0, sizeof(p));
  p.stg_per_split = pl.stg_per_split; p.nstg_total = pl.nstg_total; p.NI = pl.NI; p.nsub = pl.nsub; p.ksteps = pl.rows_dy / 16;
  p.npairs = pl.npairs; p.nstage = b.nstage; p.stage16 = pl.stage_bytes >> 4; p.sub16 = pl.sub_bytes >> 4;
  p.dy_sbo = (uint32_t)pl.rows_dy * 16u; p.x_sbo = (uint32_t)pl.rows_x * 16u; p.x_off16 = (pl.TA * pl.dy_bytes) >> 4;
  for (int i = 0; i < pl.npairs; ++i) {
    p.pair_a16[i] = (uint32_t)(pl.pair_a[i] * pl.dy_bytes) >> 4;
    p.pair_b16[i] = (uint32_t)(pl.pair_b[i] * pl.x_bytes) >> 4;
  }
  p.row_tiles = pl.row_tiles; p.TA = pl.TA; p.TX = pl.TX; p.TH = pl.TH;
  p.stage_bytes = pl.stage_bytes; p.sub_bytes = pl.sub_bytes; p.dy_bytes = pl.dy_bytes; p.x_bytes = pl.x_bytes;
  p.dy_box_bytes = pl.dy_box_bytes; p.x_box_bytes = pl.x_box_bytes; p.smem_bytes = b.smem_bytes;
  p.cout_g8 = pl.cout_g / 8; p.cin_g8 = pl.cin_g / 8;
  p.partial = reinterpret_cast<float*>(scratch);
  // the data-gradient chain of make_plan's program (conv_mma: chunk, piece pair, K-step), re-addressed: A in the sub-block's
  // dy box (octet stride = rows_dy * 16 bytes), B in the resident weight image (chunk blocks of blk_bytes)
  p.nprog = (uint32_t)b.nprog;
  {
    const int b_tap16 = (d.CC / 8) * d.Nt, blk16 = d.tmpl[0][0].blk_bytes >> 4;
    int e = 0;
    for (int cc = 0; cc < d.chunks; ++cc)
      for (int pr = 0; pr < d.npairs; ++pr)
        for (int j = 0; j < d.ksteps; ++j) {
          const uint32_t a16 = (uint32_t)(d.pair_a[pr] * pl.dy_bytes / 16 + (cc * d.ksteps + j) * 2 * pl.rows_dy);
          const uint32_t b16 = (uint32_t)(cc * blk16 + d.pair_b[pr] * b_tap16 + j * 2 * d.Nt);
          if (a16 > 0xffffu || b16 > 0xffffu) return mnb_fail(MNB_E_ARG, "pk bwd1x1: MMA program offset overflow");
          p.prog[e++] = a16 | (b16 << 16);
        }
  }
  p.dg_lbo = (uint32_t)pl.rows_dy * 16u; p.w_lbo = (uint32_t)d.Nt * 16u; p.off_w = (uint32_t)b.off_w;
  p.w_bytes = (uint32_t)b.w_bytes; p.img_bytes = (uint32_t)d.img_bytes[0];
  p.w_img = reinterpret_cast<const uint8_t*>(w_img);
  p.B = pl.B; p.P = pl.P; p.Q = pl.Q; p.BW = pl.BW; p.C = s->in_c; p.cin_g = s->in_c / s->groups;
  p.C8O = s->groups * ceil_div(p.cin_g, 8);
  p.a_scale_const = a_scale_const; p.gain = gain; p.bias0 = 0.f; p.bits8 = bits8; p.dx = dx; p.err = err_flag;
  CUtensorMap tdy[3], tx[3];
  const int64_t dy_plane = (int64_t)pl.B * pl.K8 * pl.P * pl.Q * 16;
  const int64_t x_plane = (int64_t)pl.B * pl.C8X * pl.HX * pl.WX * 16;
  for (int t = 0; t < 3; ++t) {
    if (int e = make_pk_tmap(&tdy[t], dy_pk, dy_plane, t < pl.TA ? t : 0, pl.B, pl.K8, pl.P, pl.Q, pl.BW, pl.TH, 1, 16)) return e;
    if (int e = make_pk_tmap(&tx[t], x_pk, x_plane, t < pl.TX ? t : 0, pl.B, pl.C8X, pl.HX, pl.WX, pl.BW, pl.THH, 1, pl.Nc / 8)) return e;
  }
  using BwdFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                         const CUtensorMap, const BwdParams);
  static const BwdFn fns[4] = {pk_bwd1x1_kernel<32>, pk_bwd1x1_kernel<64>, pk_bwd1x1_kernel<96>, pk_bwd1x1_kernel<128>};
  const BwdFn fn = fns[pl.Nc / 32 - 1];     // (make_bwd_plan: Nc % 32 == 0, Nc <= 128)
  if (int e = set_max_smem(fn, kSmemBudget)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  fn<<<dim3(pl.G, pl.splits), kBwdThreads, b.smem_bytes, st>>>(tdy[0], tdy[1], tdy[2], tx[0], tx[1], tx[2], p);
  const dim3 rgrid(pl.cin_o, 1, pl.G);
  wg_reduce_kernel<<<rgrid, 128, 0, st>>>(p.partial, pl.splits, pl.G, 1, 1, 1, 1, pl.Nc, pl.cout_o, pl.cin_o, pl.cout_g, pl.cin_g,
                                          a_scale, kdiv, dw);
  MNB_LAUNCHED(2);
  return 0;
}

// ---- forward and data gradient of narrow grouped 3x3 convolutions (pk_gc3_kernel)

// host only: out[0..9] = {groups per CTA block, images per M tile, m64 blocks per M tile, stages, shared-memory bytes, CTAs,
// image tiles, MMAs per accumulator chain, N tile, MMA warpgroups}, then 4 values per MMA of the chain in issue order:
// (filter tap r * 3 + s, piece of the streamed operand, piece of the weights, 16-channel K-step); the first n are written
extern "C" int mnb_pk_gc3_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out, int32_t n) {
  static pk::Gc3Plan g;   // large POD (single host thread per process)
  if (int e = pk::make_gc3_plan(s, mode, terms_a, terms_w, g)) return e;
  if (out) {
    const int v[10] = {g.GB, g.TB, g.nmb, g.nstage, g.smem_bytes, g.nblk * g.cpb, g.n_tiles, g.nprog, g.pl.Nt, pk::kGc3Cons};
    for (int i = 0; i < std::min(n, 10); ++i) out[i] = v[i];
    for (int i = 10; i < n && (i - 10) / 4 < g.nprog; ++i) out[i] = g.chain[(i - 10) / 4][(i - 10) % 4];
  }
  return 0;
}

static int pk_gc3_impl(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                       const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, const uint8_t* bits8,
                       float gain, float* out, int16_t* codes, float* dec, int32_t* err_flag, mnb_stream_t stream) {
  using namespace pk;
  MNB_REQUIRE(s && a_pk && w_img && (out != nullptr) != (codes != nullptr) && err_flag, "NULL pk_gc3 pointer");
  static Gc3Plan g;
  if (int e = make_gc3_plan(s, mode, terms_a, terms_w, g)) return e;
  MNB_REQUIRE(g.nstage % kGc3Cons == 0, "pk gc3: %d stages are not a whole number per MMA warpgroup", g.nstage);
  const Plan& pl = g.pl;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(a_pk) || !al16(w_img) || !al16(out ? (const void*)out : (const void*)codes))
    return mnb_fail(MNB_E_UNSUPPORTED, "pk gc3: operands and output must be 16-byte aligned");
  static Gc3Params p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < g.nprog; ++i) p.prog[i] = g.prog[i];
  p.nprog = g.nprog; p.mode = mode; p.TA = terms_a; p.GB = g.GB; p.ng = pl.ng; p.kg8 = pl.kg / 8; p.NOUT = pl.NOUT; p.B = pl.B;
  p.TB = g.TB; p.n_tiles = g.n_tiles; p.cpb = g.cpb; p.nmb = g.nmb; p.npos = g.npos; p.BW = g.BW; p.THH = g.THH; p.OH = pl.OHr;
  p.OW = pl.OWr; p.plane = g.plane; p.SP = g.SP; p.C8O = ceil_div(pl.NOUT, 8); p.wlo = pl.wlo; p.hlo = pl.hlo;
  p.a_box_bytes = g.a_box_bytes; p.a_piece_bytes = g.a_piece_bytes; p.stage_bytes = g.stage_bytes; p.nstage = g.nstage;
  p.w_bytes = g.w_bytes; p.img_bytes = pl.img_bytes[0]; p.stg_bytes = g.stg_bytes; p.off_stage = g.off_stage; p.off_stg = g.off_stg;
  p.off_rowmap = g.off_rowmap; p.smem_bytes = g.smem_bytes;
  p.w_img = reinterpret_cast<const uint8_t*>(w_img);
  p.n_scale = n_scale; p.a_scale = a_scale; p.a_scale_const = a_scale_const; p.bias = bias; p.bits8 = mode == 1 ? bits8 : nullptr;
  p.gain = gain; p.out = out; p.codes = codes; p.dec = dec; p.err = err_flag;
  CUtensorMap tm[2];
  const int64_t plane_bytes = (int64_t)pl.B * pl.C8A * pl.HA * pl.WA * 16;
  for (int t = 0; t < 2; ++t)
    if (int e = make_pk_tmap(&tm[t], a_pk, plane_bytes, t < terms_a ? t : 0, pl.B, pl.C8A, pl.HA, pl.WA, g.BW, g.THH, g.TB,
                             g.GB * p.kg8))
      return e;
  auto fn = pl.Nt == 32 ? pk_gc3_kernel<32> : pk_gc3_kernel<16>;
  if (pl.Nt != 16 && pl.Nt != 32) return mnb_fail(MNB_E_ARG, "pk gc3: plan with Nt %d", pl.Nt);
  if (int e = set_max_smem(fn, kGc3SmemBudget)) return e;
  fn<<<g.nblk * g.cpb, kGc3Threads, g.smem_bytes, (cudaStream_t)stream>>>(tm[0], tm[1], p);
  MNB_LAUNCHED(1);
  return 0;
}

// mnb_pk_conv (mode 0: fp32 forward, mode 1: data gradient) for the shapes of mnb_pk_gc3_plan's cover: the same operands, weight
// image and epilogue arguments, the same result bit for bit
extern "C" int mnb_pk_gc3_conv(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img,
                               int32_t terms_w, const float* n_scale, const float* a_scale, float a_scale_const,
                               const float* bias, const uint8_t* bits8, float gain, float* out, int32_t* err_flag,
                               mnb_stream_t stream) {
  MNB_REQUIRE(out, "NULL pk_gc3_conv output");
  return pk_gc3_impl(s, mode, a_pk, terms_a, w_img, terms_w, n_scale, a_scale, a_scale_const, bias, bits8, gain, out, nullptr,
                     nullptr, err_flag, stream);
}

// mnb_pk_conv_codes for the forward shapes of mnb_pk_gc3_plan's cover: the same codes and decode pair
extern "C" int mnb_pk_gc3_conv_codes(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img,
                                     int32_t terms_w, const float* n_scale, const float* a_scale, float a_scale_const,
                                     const float* bias, int32_t level_bound, int16_t* codes, float* dec, int32_t* err_flag,
                                     mnb_stream_t stream) {
  MNB_REQUIRE(s && codes && dec, "NULL pk_gc3_conv_codes pointer");
  MNB_REQUIRE(level_bound >= 1 && s->groups >= 1, "pk_gc3_conv_codes: level bound %d", level_bound);
  if ((int64_t)(s->in_c / s->groups) * s->ker_h * s->ker_w * level_bound > 32767)
    return mnb_fail(MNB_E_UNSUPPORTED, "pk_gc3_conv_codes: sums of %d x %d x %d terms of level %d may exceed int16",
                    s->in_c / s->groups, s->ker_h, s->ker_w, level_bound);
  return pk_gc3_impl(s, 0, a_pk, terms_a, w_img, terms_w, n_scale, a_scale, a_scale_const, bias, nullptr, 1.f, nullptr, codes, dec,
                     err_flag, stream);
}
