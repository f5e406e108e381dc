// Binary tensor-core forward convolution for wbwtab inference layers: wgmma m64nNk256.s32.b1.b1.and.popc on Hopper.
//
// Reference math (WB:11-36, 55-75, 181-195): y = bias + alpha[k] * sum_{c,r,s} a[c] * w[k][c][r][s] with a = sign(x) in
// {-1, +1} (0 -> +1), w in {-1, +1} or {-1, 0, +1}, out-of-image taps 0.  The XNOR kernel (mnb_xnor.cu) computes it on the
// popc pipe for the layers its templates cover (at most 8 words of 32 channels per group on 1x1, 4 on 3x3, 2 on 5x5); NIN's
// 160- and 192-channel layers (models/nin.py) are outside that cover.  This kernel takes them to the binary tensor cores.
//
// Operands ("b1 plane", the byte geometry of the bf16 / int8 planes of mnb_pk.cu):
//   activations [B][G * u][H][W][16 B], u = ceil(C/g / 64): one 16-byte unit = 64 channels of one pixel,
//               bits 0-63 p = [a == +1], bits 64-127 n = [a == -1]; p = n = 0 is a 0 (halo, channel and group padding)
//   weights     [G][n-tile][k-step][tap][2 units][Nt columns][16 B]: output channel k owns columns 2k (plus = [P | M]) and
//               2k + 1 (minus = [M | P]), P = [w == +1], M = [w == -1]; columns and units past the layer are zero.
// With AND + popc over the 256 bits of a K step (two units):
//   D_plus - D_minus = sum p P + n M - p M - n P = sum (P - M)(p - n) = sum w * a,
// the exact integer of mnb_xnor_conv_fwd and mnb_pk_conv; a zero weight or a zero activation contributes nothing, so the
// halo zero-filled by the TMA unit and whatever a padding unit of the box holds (the next group's first unit) need no
// border tables.  Adjacent columns put D_plus and D_minus in one thread's fragment registers (d[4j + 2i] and d[4j + 2i + 1]).
//
// Pipeline (the pk forward's, DESIGN.md 4.9): a 4-D tensor map (16-byte pixels as pairs of 8-byte elements, H, B, units)
// lands a box of the zero-padded tile as [unit][image][row][col][16 B] - the K-major no-swizzle canonical layout with the
// tile raster as GEMM rows - so filter tap (r, s) is the same buffer with the descriptor start moved by (r * BW + s) rows.
// One TMA thread feeds a ring of (k-step, tap group) stages; two MMA warpgroups (rows 0-63 / 64-127 of the M tile) issue one
// wgmma per tap into s32 register accumulators and run the epilogue themselves.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

namespace b1 {

constexpr int kThreads = 384;                 // warp 0: TMA, warps 4-11: two MMA + epilogue warpgroups (1-3 idle)
constexpr int kMaxStages = 4;
constexpr int kSmemBudget = 227 * 1024 - 3072;   // dynamic shared memory: the 227 KB block limit less the static Shared
constexpr int kNt[] = {32, 64, 128, 192};     // B columns (two per output channel) the kernel is instantiated for
constexpr int kMaxCh = 96;                    // output channels of the widest N tile
constexpr int kMaxR = 7;

__host__ __device__ inline int units_per_group(int cin_g) { return (cin_g + 63) / 64; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// everything about a conv shape that the weight packer, the host launcher and the kernel agree on
struct Plan {
  int B, G, H, W, P, Q, R, pad, cin_g, cout_g, u, GU, ksteps, taps;
  int Nt, n_ntiles;
  int Wt, BW, TH, THH, TB, col_tiles, row_tiles, n_mtiles, npos;
  int TG, ntg;                       // taps per stage, tap groups
  int a_bytes, b_bytes, stage_bytes, nstage, smem_bytes;
  int64_t wimg_bytes;
};

static int check_shape(const mnb_conv_shape* s) {
  MNB_REQUIRE(s != nullptr, "b1: null shape");
  MNB_REQUIRE(s->batch > 0 && s->in_c > 0 && s->out_c > 0 && s->groups > 0 && s->in_c % s->groups == 0 &&
                  s->out_c % s->groups == 0 && s->in_h > 0 && s->in_w > 0, "b1: bad conv shape");
  if (s->ker_h != s->ker_w || s->ker_h < 1 || s->ker_h > kMaxR) return MNB_E_UNSUPPORTED;
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return MNB_E_UNSUPPORTED;
  if (s->pad_h != s->pad_w || s->pad_h < 0 || s->pad_h > s->ker_h / 2) return MNB_E_UNSUPPORTED;
  const int P = s->in_h + 2 * s->pad_h - s->ker_h + 1, Q = s->in_w + 2 * s->pad_w - s->ker_w + 1;
  if (P < 1 || Q < 1) return MNB_E_UNSUPPORTED;
  return 0;
}

static int make_plan(const mnb_conv_shape* s, Plan& p) {
  const int rc = check_shape(s);
  if (rc != 0) return rc;
  memset(&p, 0, sizeof(p));
  p.B = s->batch; p.G = s->groups; p.H = s->in_h; p.W = s->in_w; p.R = s->ker_h; p.pad = s->pad_h;
  p.P = p.H + 2 * p.pad - p.R + 1; p.Q = p.W + 2 * p.pad - p.R + 1;
  p.cin_g = s->in_c / p.G; p.cout_g = s->out_c / p.G;
  p.u = units_per_group(p.cin_g); p.GU = p.G * p.u; p.ksteps = ceil_div(p.u, 2); p.taps = p.R * p.R;
  // N tile: the accumulators of a thread are Nt / 2 s32 registers; at most 192 columns (96 output channels) keeps the
  // epilogue free of spills at 288 threads
  {
    const int cols = 2 * p.cout_g;
    p.n_ntiles = ceil_div(cols, 192);
    const int want = ceil_div(cols, p.n_ntiles);
    p.Nt = 192;
    for (int v : kNt) if (v >= want) { p.Nt = v; break; }
    p.n_ntiles = ceil_div(cols, p.Nt);
  }
  // M tile: 128 consecutive positions of the zero-padded tile raster (image, row, col), rows of Wt outputs at pitch BW
  const int halo = p.R - 1;
  {
    const int ct_min = ceil_div(p.Q, 128 - halo);
    double best = 1e30;
    for (int ct = ct_min; ct <= std::min(p.Q, ct_min + 14); ++ct) {
      const int wt = ceil_div(p.Q, ct), bw = wt + halo;
      if (ceil_div(p.Q, wt) != ct) continue;
      const int th = std::max(1, std::min(p.P, (128 - wt) / bw + 1));
      const double amp = (double)((th + halo) * bw) / (double)(th * wt);
      const double cost = (double)ct * ceil_div(p.P, th) * (1.0 + 0.25 * amp);
      if (cost < best - 1e-9) { best = cost; p.col_tiles = ct; p.Wt = wt; p.BW = bw; p.TH = th; }
    }
  }
  if (p.col_tiles == 0) return mnb_fail(MNB_E_UNSUPPORTED, "b1 conv: no column tiling of a %d-wide plane", p.Q);
  p.THH = p.TH + halo;
  p.TB = 1;
  if (p.TH == p.P && p.col_tiles == 1) {
    const int last = (p.TH - 1) * p.BW + p.Wt;
    p.TB = std::max(1, std::min(p.B, (128 - last) / (p.THH * p.BW) + 1));
  }
  if (p.BW > 128 || p.THH > 256) return mnb_fail(MNB_E_UNSUPPORTED, "b1 conv: box dimension");
  p.npos = p.TB * p.THH * p.BW;
  p.row_tiles = ceil_div(p.P, p.TH);
  p.n_mtiles = ceil_div(p.B, p.TB) * p.row_tiles * p.col_tiles;
  // stages: one k-step (two units of the box) and a group of taps; at most 48 KB of weights per stage
  const int per_tap = 2 * p.Nt * 16;
  const int tg_max = std::max(1, std::min(p.taps, 48 * 1024 / per_tap));
  p.ntg = ceil_div(p.taps, tg_max);
  p.TG = ceil_div(p.taps, p.ntg);
  p.a_bytes = round_up(2 * p.npos * 16, 128);
  p.b_bytes = p.TG * per_tap;
  p.stage_bytes = round_up(p.a_bytes + p.b_bytes, 128);
  // rows past a box that only invalid accumulator rows read: up to 128 + the largest tap offset behind the last stage
  const int slack = round_up((128 + halo * p.BW + halo + 8) * 16, 128);
  p.nstage = std::min(kMaxStages, (kSmemBudget - slack) / p.stage_bytes);
  if (p.nstage < 2) return mnb_fail(MNB_E_UNSUPPORTED, "b1 conv: fewer than two pipeline stages fit");
  // (at least the post epilogue's staging rows: 128 x one word per output channel of the widest tile)
  p.smem_bytes = std::max(p.nstage * p.stage_bytes + slack, 128 * kMaxCh * 4);
  p.wimg_bytes = (int64_t)p.G * p.n_ntiles * p.ksteps * p.taps * per_tap;
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// packers
// ------------------------------------------------------------------------------------------------------------------
// fp32 NCHW [-> eval BatchNorm] -> sign [-> 2x2 max-pool: OR of the window] [-> channel shuffle] -> b1 plane of a consumer
// with G groups.  One thread per 16-byte unit, gathering its (up to) 64 channels through the inverse shuffle; the plain
// packer is the case without BatchNorm, pool and shuffle.
__global__ void __launch_bounds__(256) pack_act_kernel(const float* __restrict__ x, int B, int Cc, int H, int W, int G, int sg,
                                                       int pool, const float* __restrict__ mean, const float* __restrict__ invstd,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       uint4* __restrict__ out) {
  const int cin_g = Cc / G, u = units_per_group(cin_g), cpg = Cc / sg;
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W, OHW = OH * OW, HW = H * W;
  const int64_t total = (int64_t)B * G * u * OHW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int opix = (int)(i % OHW);
    int64_t t = i / OHW;
    const int gu = (int)(t % (G * u));
    const int b = (int)(t / (G * u));
    const int g = gu / u, c0 = (gu - g * u) * 64, cnt = min(64, cin_g - c0);
    const int oh = opix / OW, ow = opix - oh * OW;
    const int pix = pool ? (2 * oh) * W + 2 * ow : opix;
    uint64_t pos = 0, neg = 0;
    for (int j = 0; j < cnt; ++j) {
      const int cd = g * cin_g + c0 + j;
      const int c = sg > 1 ? (cd % sg) * cpg + cd / sg : cd;   // inverse of the producer's shuffle
      const float* src = x + ((int64_t)b * Cc + c) * HW + pix;
      float mu = 0.f, k = 1.f, be = 0.f;
      if (mean) { mu = __ldg(mean + c); k = __ldg(gamma + c) * __ldg(invstd + c); be = __ldg(beta + c); }
      bool plus = false;
      for (int q = 0; q < (pool ? 4 : 1); ++q) {
        float v = __ldg(src + (q >> 1) * W + (q & 1));
        if (mean) v = fmaf(v - mu, k, be);
        plus |= !(v < 0.f);
      }
      if (plus) pos |= 1ull << j; else neg |= 1ull << j;
    }
    out[i] = make_uint4((uint32_t)pos, (uint32_t)(pos >> 32), (uint32_t)neg, (uint32_t)(neg >> 32));
  }
}

// i16 levels [K][C/g][R][S] -> weight image; one thread per 16-byte record (column of one unit of one tap)
__global__ void __launch_bounds__(256) pack_weight_kernel(const int16_t* __restrict__ w, int G, int cin_g, int cout_g, int taps,
                                                          int ksteps, int n_ntiles, int Nt, uint4* __restrict__ out) {
  const int64_t total = (int64_t)G * n_ntiles * ksteps * taps * 2 * Nt;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    const int col = (int)(t % Nt); t /= Nt;
    const int half = (int)(t % 2); t /= 2;
    const int tap = (int)(t % taps); t /= taps;
    const int ks = (int)(t % ksteps); t /= ksteps;
    const int nt = (int)(t % n_ntiles);
    const int g = (int)(t / n_ntiles);
    const int k = (nt * Nt + col) >> 1;
    uint64_t P = 0, M = 0;
    if (k < cout_g) {
      const int c0 = (2 * ks + half) * 64;
      const int16_t* wk = w + ((int64_t)(g * cout_g + k) * cin_g) * taps + tap;
      for (int j = 0; j < 64 && c0 + j < cin_g; ++j) {
        const int v = wk[(int64_t)(c0 + j) * taps];
        if (v > 0) P |= 1ull << j;
        if (v < 0) M |= 1ull << j;
      }
    }
    const uint64_t lo = (col & 1) ? M : P, hi = (col & 1) ? P : M;
    out[i] = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
  }
}

// the b1 plane of a post-conv consumer before the epilogue ANDs / ORs into it: every valid channel -1 (n set, p clear),
// padding channels 0
__global__ void __launch_bounds__(256) fill_neg_kernel(uint4* __restrict__ out, int64_t total, int u, int cin_g, int hw) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int unit = (int)((i / hw) % u);
    const int cnt = min(64, cin_g - unit * 64);
    const uint64_t m = cnt >= 64 ? ~0ull : ((1ull << cnt) - 1ull);
    out[i] = make_uint4(0u, 0u, (uint32_t)m, (uint32_t)(m >> 32));
  }
}

// MaxPool2d(k, s, p) on a b1 plane (floor mode, 2p <= k: every window holds an in-image pixel): p = OR of the window's p,
// n = (OR n) & !p.  One thread per output unit.
__global__ void __launch_bounds__(256) plane_maxpool_kernel(const uint4* __restrict__ in, int64_t planes, int H, int W, int k,
                                                            int s, int pad, int OH, int OW, uint4* __restrict__ out) {
  const int64_t total = planes * OH * OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ow = (int)(i % OW);
    const int oh = (int)((i / OW) % OH);
    const int64_t pl = i / ((int64_t)OH * OW);
    const uint4* src = in + pl * H * W;
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
    for (int r = 0; r < k; ++r) {
      const int ih = oh * s - pad + r;
      if (ih < 0 || ih >= H) continue;
      for (int q = 0; q < k; ++q) {
        const int iw = ow * s - pad + q;
        if (iw < 0 || iw >= W) continue;
        const uint4 v = __ldg(src + ih * W + iw);
        acc.x |= v.x; acc.y |= v.y; acc.z |= v.z; acc.w |= v.w;
      }
    }
    acc.z &= ~acc.x; acc.w &= ~acc.y;
    out[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// the convolution
// ------------------------------------------------------------------------------------------------------------------
struct Params {
  int B, G, P, Q, R, pad, BW, Wt, TH, THH, TB, col_tiles, row_tiles, npos;
  int u, ksteps, taps, TG, ntg, cout_g, Nt, a_bytes, stage_bytes, nstage;
  const uint8_t* w_img;
  int64_t wtile_bytes;                        // weight bytes of one (group, n-tile)
  const float* alpha;                         // [K] or NULL (= 1)
  const float* bias;                          // [K] or NULL
  float* y;                                   // fp32 NCHW (conv_fwd)
  // post epilogue (conv_post): BatchNorm constants (mean NULL = none), output format, the consumer's geometry, 2x2 pool
  const float *bn_mean, *bn_invstd, *bn_gamma, *bn_beta;
  void* out;
  int fmt, sg, out_cin_g, out_units, pool;    // out_units: words (bits) / units (b1) / octets (bf16) per image and pixel
  int* err;                                   // pipeline-timeout flag (L.tc_check): 711 TMA side, 713 MMA side
};

struct alignas(16) Shared {
  uint64_t full[kMaxStages], empty[kMaxStages];
  uint32_t abort;
  float alpha[kMaxCh], bias[kMaxCh];
  float4 bn[kMaxCh];                           // POST: {mean, gamma * invstd, beta, destination}
  // POST into bit / b1 planes: the tile's channels in runs that share one 32-bit destination word (key = dest >> 5);
  // channel e sets bit (dest & 31) of staging row word[slot[e]]
  int key[kMaxCh];
  uint8_t slot[kMaxCh];
  int nslots;
};

// destination of output channel c in the consumer's operand (after the producer's shuffle: channel c lands at
// (c mod C/sg) * sg + c div C/sg):  bits: (word << 5) | bit;  b1 plane: (unit << 6) | bit;  bf16 plane: the channel
__device__ __forceinline__ int post_dest(int c, int K, const Params& p) {
  const int cpg = K / p.sg;
  const int cd = p.sg > 1 ? (c % cpg) * p.sg + c / cpg : c;
  if (p.fmt == MNB_XNOR_PM1_BF16) return cd;
  const int g = cd / p.out_cin_g, r = cd - g * p.out_cin_g;
  if (p.fmt == MNB_XNOR_BITS) return ((g * ((p.out_cin_g + 31) >> 5) + (r >> 5)) << 5) | (r & 31);
  return ((g * units_per_group(p.out_cin_g) + (r >> 6)) << 6) | (r & 63);
}

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int NT, bool POST>
__global__ void __launch_bounds__(kThreads, 1) conv_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ Params p) {
  constexpr int NR = NT / 2;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mt = blockIdx.x, nt = blockIdx.y, g = blockIdx.z;
  const int K = p.G * p.cout_g;
  const int k0 = nt * (NT / 2);                                  // first output channel of the tile within the group
  const int kcnt = min(NT / 2, p.cout_g - k0);

  if (tid == 0) {
    for (int i = 0; i < kMaxStages; ++i) { tc::mbar_init(&sh.full[i], 1); tc::mbar_init(&sh.empty[i], 8); }
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmap);
  }
  for (int e = tid; e < kcnt; e += kThreads) {
    const int c = g * p.cout_g + k0 + e;
    sh.alpha[e] = p.alpha ? __ldg(p.alpha + c) : 1.f;
    sh.bias[e] = p.bias ? __ldg(p.bias + c) : 0.f;
    if (POST) {
      float4 v = make_float4(0.f, 1.f, 0.f, 0.f);
      if (p.bn_mean) v = make_float4(__ldg(p.bn_mean + c), __ldg(p.bn_gamma + c) * __ldg(p.bn_invstd + c), __ldg(p.bn_beta + c), 0.f);
      v.w = __int_as_float(post_dest(c, K, p));
      sh.bn[e] = v;
    }
  }
  __syncthreads();
  if (POST && p.fmt != MNB_XNOR_PM1_BF16 && warp == 4) {
    // runs of equal destination words: a slot per run (a word reached again after another run gets a second slot - two
    // ORs into one word, still exact)
    int base = 0;
    for (int e0 = 0; e0 < kcnt; e0 += 32) {
      const int e = e0 + lane;
      const int k = e < kcnt ? (__float_as_int(sh.bn[e].w) >> 5) : -1;
      const int prev = e == 0 ? -2 : (e < kcnt ? (__float_as_int(sh.bn[e - 1].w) >> 5) : -1);
      const uint32_t starts = __ballot_sync(0xffffffffu, e < kcnt && k != prev);
      const int sl = base + __popc(starts & ((2u << lane) - 1u)) - 1;
      if (e < kcnt) { sh.slot[e] = (uint8_t)sl; if (k != prev) sh.key[sl] = k; }
      base += __popc(starts);
    }
    if (lane == 0) sh.nslots = base;
  }
  __syncthreads();

  const int ct = mt % p.col_tiles, rt = (mt / p.col_tiles) % p.row_tiles, bt = mt / (p.col_tiles * p.row_tiles);
  const int nstages = p.ksteps * p.ntg;
  if (warp >= 4) {
    // ================================================================= MMA warpgroups + epilogue
    const int wg = (warp >> 2) - 1;
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), (uint32_t)(p.npos * 16), 128) + (uint64_t)(64 * wg);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(smem), (uint32_t)(NT * 16), 128) + (uint64_t)(p.a_bytes >> 4);
    int32_t acc[NR];
    tc::zero_acc(acc);
    for (int st = 0; st < nstages; ++st) {
      const int slot = st % p.nstage, ph = (st / p.nstage) & 1;
      tc::mbar_wait_soft(&sh.full[slot], ph, p.err, 713, &sh.abort);
      const int ks = st / p.ntg, t0 = (st - ks * p.ntg) * p.TG, nta = min(p.TG, p.taps - t0);
      const uint64_t s16 = (uint64_t)((slot * p.stage_bytes) >> 4);
      tc::wg_fence();
      tc::fence_acc(acc);
      int r = t0 / p.R, q = t0 - r * p.R;
      // (one MMA per iteration: ptxas serializes the taps of a stage here either way - C7520, DESIGN.md 4.19 - and the
      // unrolled form carries a wait per copy)
#pragma unroll 1
      for (int ti = 0; ti < nta; ++ti) {
        tc::Mma<NT>::b1(acc, a_desc0 + s16 + (uint64_t)(r * p.BW + q), b_desc0 + s16 + (uint64_t)(ti * 2 * NT), 1);
        if (++q == p.R) { q = 0; ++r; }
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::fence_acc(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.empty[slot]);
    }

    // ---- epilogue: thread (warp w, lane l) holds rows 64 wg + 16 (w % 4) + l / 4 + 8 i and, per j, the plus / minus columns
    // of output channel 4 j + l % 4 of the tile
    const int PQ = p.P * p.Q;
    const int OQ = POST && p.pool ? p.Q >> 1 : p.Q;
    const int64_t out_hw = POST && p.pool ? (int64_t)(p.P >> 1) * (p.Q >> 1) : (int64_t)PQ;
    bool valid[2];
    int64_t obase[2];       // fwd: offset of (b, channel 0, oh, ow) in y; post: image b's unit-0 offset + output pixel
    // bit / b1 planes: the sign bits are first collected per (slot, row) in the drained pipeline buffers, then written with
    // one global OR (b1: OR of p, AND of n) per destination word and row
    const bool staged = POST && p.fmt != MNB_XNOR_PM1_BF16;
    uint32_t* stg = reinterpret_cast<uint32_t*>(smem);
    if (staged) {
      epi_bar_sync();                                     // both warpgroups are done reading the stages
      for (int i = tid - 128; i < sh.nslots * 128; i += 256) stg[i] = 0u;
      epi_bar_sync();
    }
  #pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * i;
      const int tb = m / (p.THH * p.BW), rem = m - tb * (p.THH * p.BW), th = rem / p.BW, wc = rem - th * p.BW;
      const int b = bt * p.TB + tb, oh = rt * p.TH + th, ow = ct * p.Wt + wc;
      valid[i] = tb < p.TB && th < p.TH && wc < p.Wt && b < p.B && oh < p.P && ow < p.Q;
      if (!POST) {
        obase[i] = ((int64_t)b * K + g * p.cout_g + k0) * PQ + (int64_t)oh * p.Q + ow;
      } else {
        const int opix = p.pool ? (oh >> 1) * OQ + (ow >> 1) : oh * p.Q + ow;
        obase[i] = (int64_t)b * p.out_units * out_hw + opix;
      }
    }
  #pragma unroll
    for (int j = 0; j < NR / 4; ++j) {
      const int e = 4 * j + (lane & 3);
      if (e >= kcnt) continue;
      const float al = sh.alpha[e], bs = sh.bias[e];
  #pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        const float v0 = fmaf((float)(acc[4 * j + 2 * i] - acc[4 * j + 2 * i + 1]), al, bs);
        if (!POST) {
          p.y[obase[i] + (int64_t)e * PQ] = v0;
          continue;
        }
        // the BN + sign producers' op sequence (mnb_conv_packed.cu): bn = fmaf(v - mean, gamma * invstd, beta), bit = !(bn < 0)
        const float4 c = sh.bn[e];
        const float v = p.bn_mean ? fmaf(v0 - c.x, c.y, c.z) : v0;
        const bool plus = !(v < 0.f);
        const int dest = __float_as_int(c.w);
        if (!staged) {
          reinterpret_cast<uint16_t*>(p.out)[(obase[i] + (int64_t)(dest >> 3) * out_hw) * 8 + (dest & 7)] = plus ? 0x3F80u : 0xBF80u;
        } else if (plus) {
          const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * i;
          atomicOr(stg + sh.slot[e] * 128 + m, 1u << (dest & 31));
        }
      }
    }
    if (staged) {
      epi_bar_sync();
      // thread -> (row m, slots m / 128 + 2 k): consecutive threads write consecutive output pixels of one word plane
      const int m = (tid - 128) & 127;
      const int tb = m / (p.THH * p.BW), rem = m - tb * (p.THH * p.BW), th = rem / p.BW, wc = rem - th * p.BW;
      const int b = bt * p.TB + tb, oh = rt * p.TH + th, ow = ct * p.Wt + wc;
      if (tb < p.TB && th < p.TH && wc < p.Wt && b < p.B && oh < p.P && ow < p.Q) {
        const int64_t ob = (int64_t)b * p.out_units * out_hw + (p.pool ? (oh >> 1) * OQ + (ow >> 1) : oh * p.Q + ow);
        uint32_t* out = reinterpret_cast<uint32_t*>(p.out);
        for (int sl = (tid - 128) >> 7; sl < sh.nslots; sl += 2) {
          const uint32_t bits = stg[sl * 128 + m];
          const int key = sh.key[sl];
          if (p.fmt == MNB_XNOR_BITS) {
            if (bits) atomicOr(out + ob + (int64_t)key * out_hw, bits);
          } else if (bits) {   // b1 plane, pre-filled with n set: +1 sets p and clears n (any +1 of a pooled window wins)
            uint32_t* w = out + (ob + (int64_t)(key >> 1) * out_hw) * 4 + (key & 1);
            atomicOr(w, bits);
            atomicAnd(w + 2, ~bits);
          }
        }
      }
    }
  } else if (warp == 0) {
    // ================================================================= TMA producer
    if (lane == 0) {
      const uint8_t* wsrc = p.w_img + (int64_t)(g * (int)gridDim.y + nt) * p.wtile_bytes;
      const int per_tap = 2 * NT * 16;
      const int cw = ct * p.Wt - p.pad, chh = rt * p.TH - p.pad, cb = bt * p.TB;
      for (int st = 0; st < nstages; ++st) {
        const int slot = st % p.nstage, ph = (st / p.nstage) & 1;
        if (!tc::mbar_wait(&sh.empty[slot], ph ^ 1, p.err, 711)) break;
        const int ks = st / p.ntg, t0 = (st - ks * p.ntg) * p.TG, nta = min(p.TG, p.taps - t0);
        tc::mbar_arrive_expect_tx(&sh.full[slot], (uint32_t)(2 * p.npos * 16 + nta * per_tap));
        uint8_t* sbase = smem + (size_t)slot * p.stage_bytes;
        // units g*u + 2ks and + 1 (a unit past the group holds the next group's channels or is zero-filled: its weights are 0)
        tc::tma_load_4d(sbase, &tmap, &sh.full[slot], 2 * cw, chh, cb, g * p.u + 2 * ks);
        tc::bulk_load_1d(sbase + p.a_bytes, wsrc + ((int64_t)ks * p.taps + t0) * per_tap, (uint32_t)(nta * per_tap), &sh.full[slot]);
      }
    }
  }
}

template <int NT, bool POST>
static int set_smem(int bytes) {
  static int done_dev = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (done_dev == dev) return 0;
  cudaError_t e = cudaFuncSetAttribute(conv_kernel<NT, POST>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return mnb_fail((int)e, "b1 conv: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  done_dev = dev;
  return 0;
}

template <int NT, bool POST>
static int launch_nt(const Plan& pl, const CUtensorMap& tmap, const Params& p, cudaStream_t stream) {
  const int rc = set_smem<NT, POST>(kSmemBudget);
  if (rc != 0) return rc;
  dim3 grid((unsigned)pl.n_mtiles, (unsigned)pl.n_ntiles, (unsigned)pl.G);
  conv_kernel<NT, POST><<<grid, kThreads, pl.smem_bytes, stream>>>(tmap, p);
  MNB_LAUNCHED(1);
  return 0;
}

// the consumer description of mnb_b1_conv_post / mnb_b1_pack_act_post for C producer channels on a P x Q plane
static int check_post(const mnb_xnor_post* post, int C, int P, int Q) {
  MNB_REQUIRE(post != nullptr, "b1 post: null consumer description");
  MNB_REQUIRE(post->format == MNB_XNOR_BITS || post->format == MNB_XNOR_PM1_BF16 || post->format == MNB_XNOR_B1_PLANE,
              "b1 post: unknown format %d", post->format);
  MNB_REQUIRE(post->shuffle_groups >= 1 && C % post->shuffle_groups == 0, "b1 post: shuffle groups %d do not divide %d channels",
              post->shuffle_groups, C);
  MNB_REQUIRE(post->pool2 == 0 || post->pool2 == 1, "b1 post: pool2 must be 0 or 1");
  const bool any_bn = post->bn_mean || post->bn_invstd || post->bn_gamma || post->bn_beta;
  MNB_REQUIRE(!any_bn || (post->bn_mean && post->bn_invstd && post->bn_gamma && post->bn_beta),
              "b1 post: BatchNorm needs all four of mean, invstd, gamma, beta");
  if (post->format == MNB_XNOR_PM1_BF16) {
    if (post->pool2) return mnb_fail(MNB_E_UNSUPPORTED, "b1 post: the bf16 plane takes no folded pool");
    if (C % 8) return mnb_fail(MNB_E_UNSUPPORTED, "b1 post: the bf16 plane needs C %% 8 == 0");
  } else {
    MNB_REQUIRE(post->out_groups >= 1 && C % post->out_groups == 0, "b1 post: consumer groups %d do not divide %d channels",
                post->out_groups, C);
  }
  if (post->pool2 && ((P | Q) & 1)) return mnb_fail(MNB_E_UNSUPPORTED, "b1 post: a 2x2 pool over an odd plane (%d x %d)", P, Q);
  return 0;
}

static int64_t post_bytes(int B, int C, int OH, int OW, const mnb_xnor_post* post) {
  if (post->format == MNB_XNOR_PM1_BF16) return (int64_t)B * C * OH * OW * 2;
  const int cg = C / post->out_groups;
  if (post->format == MNB_XNOR_BITS) return (int64_t)B * post->out_groups * ((cg + 31) / 32) * OH * OW * 4;
  return (int64_t)B * post->out_groups * units_per_group(cg) * OH * OW * 16;
}

static int run_conv(const mnb_conv_shape* s, const void* a_plane, const void* w_img, const float* alpha, const float* bias,
                    const mnb_xnor_post* post, void* out, int32_t* err_flag, mnb_stream_t stream) {
  Plan pl;
  int rc = make_plan(s, pl);
  if (rc != 0) return rc;
  MNB_REQUIRE(a_plane && w_img && out && err_flag, "b1 conv: null pointer");
  CUtensorMap tmap;
  {
    const uint64_t HW = (uint64_t)pl.H * pl.W;
    uint64_t dims[4] = {(uint64_t)pl.W * 2, (uint64_t)pl.H, (uint64_t)pl.B, (uint64_t)pl.GU};
    uint64_t strides[3] = {(uint64_t)pl.W * 16, (uint64_t)pl.GU * HW * 16, HW * 16};
    uint32_t box[4] = {(uint32_t)pl.BW * 2, (uint32_t)pl.THH, (uint32_t)pl.TB, 2u};
    rc = mnb_make_tmap_strided(&tmap, a_plane, 8, 4, dims, strides, box);
    if (rc != 0) return rc;
  }
  Params p;
  memset(&p, 0, sizeof(p));
  p.B = pl.B; p.G = pl.G; p.P = pl.P; p.Q = pl.Q; p.R = pl.R; p.pad = pl.pad; p.BW = pl.BW; p.Wt = pl.Wt; p.TH = pl.TH;
  p.THH = pl.THH; p.TB = pl.TB; p.col_tiles = pl.col_tiles; p.row_tiles = pl.row_tiles; p.npos = pl.npos;
  p.u = pl.u; p.ksteps = pl.ksteps; p.taps = pl.taps; p.TG = pl.TG; p.ntg = pl.ntg; p.cout_g = pl.cout_g; p.Nt = pl.Nt;
  p.a_bytes = pl.a_bytes; p.stage_bytes = pl.stage_bytes; p.nstage = pl.nstage;
  p.w_img = (const uint8_t*)w_img;
  p.wtile_bytes = (int64_t)pl.ksteps * pl.taps * 2 * pl.Nt * 16;
  p.alpha = alpha; p.bias = bias; p.err = err_flag;
  cudaStream_t st = (cudaStream_t)stream;
  if (post) {
    rc = check_post(post, s->out_c, pl.P, pl.Q);
    if (rc != 0) return rc;
    if (post->format == MNB_XNOR_PM1_BF16 && (reinterpret_cast<uintptr_t>(out) & 15))
      return mnb_fail(MNB_E_UNSUPPORTED, "b1 conv_post: the bf16 plane must be 16-byte aligned");
    p.bn_mean = post->bn_mean; p.bn_invstd = post->bn_invstd; p.bn_gamma = post->bn_gamma; p.bn_beta = post->bn_beta;
    p.out = out; p.fmt = post->format; p.sg = post->shuffle_groups; p.pool = post->pool2;
    const int C = s->out_c;
    const int OH = post->pool2 ? pl.P / 2 : pl.P, OW = post->pool2 ? pl.Q / 2 : pl.Q;
    if (post->format == MNB_XNOR_PM1_BF16) {
      p.out_cin_g = C; p.out_units = C / 8;
    } else {
      p.out_cin_g = C / post->out_groups;
      p.out_units = post->out_groups * (post->format == MNB_XNOR_BITS ? (p.out_cin_g + 31) / 32 : units_per_group(p.out_cin_g));
    }
    // bits and b1 planes are OR-ed (and AND-ed) into: several blocks and the four pixels of a pooled window write one word
    const int64_t nbytes = post_bytes(pl.B, C, OH, OW, post);
    if (post->format == MNB_XNOR_BITS) {
      cudaError_t e = cudaMemsetAsync(out, 0, (size_t)nbytes, st);
      if (e != cudaSuccess) return mnb_fail((int)e, "b1 conv_post: memset failed: %s", cudaGetErrorString(e));
    } else if (post->format == MNB_XNOR_B1_PLANE) {
      const int64_t total = nbytes / 16;
      const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)MNB_NUM_SMS * 16);
      fill_neg_kernel<<<blocks, 256, 0, st>>>((uint4*)out, total, units_per_group(p.out_cin_g), p.out_cin_g, OH * OW);
      MNB_LAUNCHED(1);
    }
  } else {
    p.y = (float*)out;
  }
#define B1_CASE(n)                                                                                      \
  if (pl.Nt == n) return post ? launch_nt<n, true>(pl, tmap, p, st) : launch_nt<n, false>(pl, tmap, p, st);
  B1_CASE(32) B1_CASE(64) B1_CASE(128) B1_CASE(192)
#undef B1_CASE
  return mnb_fail(MNB_E_UNSUPPORTED, "b1 conv: no kernel for N tile %d", pl.Nt);
}

static int launch_pack_act(const float* x, int B, int C, int H, int W, int G, int sg, int pool, const mnb_xnor_post* bn, void* out,
                           mnb_stream_t stream) {
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W;
  const int64_t total = (int64_t)B * G * units_per_group(C / G) * OH * OW;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)MNB_NUM_SMS * 16);
  pack_act_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, B, C, H, W, G, sg, pool, bn ? bn->bn_mean : nullptr,
                                                            bn ? bn->bn_invstd : nullptr, bn ? bn->bn_gamma : nullptr,
                                                            bn ? bn->bn_beta : nullptr, (uint4*)out);
  MNB_LAUNCHED(1);
  return 0;
}

}  // namespace b1

extern "C" {

int mnb_b1_supported(const mnb_conv_shape* s) {
  b1::Plan pl;
  const int rc = b1::make_plan(s, pl);
  return rc == 0 ? 1 : (rc == MNB_E_UNSUPPORTED ? 0 : rc);
}

int64_t mnb_b1_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups) {
  if (batch <= 0 || channels <= 0 || h <= 0 || w <= 0 || groups <= 0 || channels % groups) return -1;
  return (int64_t)batch * groups * b1::units_per_group(channels / groups) * h * w * 16;
}

int mnb_b1_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups, void* out_plane,
                    mnb_stream_t stream) {
  MNB_REQUIRE(x && out_plane, "b1_pack_act: null pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && groups > 0 && channels % groups == 0, "b1_pack_act: bad shape");
  return b1::launch_pack_act(x, batch, channels, h, w, groups, 1, 0, nullptr, out_plane, stream);
}

int mnb_b1_pack_act_post(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_xnor_post* post,
                         void* out_plane, mnb_stream_t stream) {
  MNB_REQUIRE(x && out_plane, "b1_pack_act_post: null pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0, "b1_pack_act_post: bad shape");
  const int rc = b1::check_post(post, channels, h, w);
  if (rc != 0) return rc;
  if (post->format != MNB_XNOR_B1_PLANE) return mnb_fail(MNB_E_UNSUPPORTED, "b1_pack_act_post: writes b1 planes only");
  return b1::launch_pack_act(x, batch, channels, h, w, post->out_groups, post->shuffle_groups, post->pool2,
                             post->bn_mean ? post : nullptr, out_plane, stream);
}

int64_t mnb_b1_wimage_bytes(const mnb_conv_shape* s) {
  b1::Plan pl;
  if (b1::make_plan(s, pl) != 0) return -1;
  return pl.wimg_bytes;
}

int mnb_b1_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream) {
  b1::Plan pl;
  const int rc = b1::make_plan(s, pl);
  if (rc != 0) return rc;
  MNB_REQUIRE(w_int && w_img, "b1_pack_weight: null pointer");
  const int64_t total = pl.wimg_bytes / 16;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)MNB_NUM_SMS * 16);
  b1::pack_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w_int, pl.G, pl.cin_g, pl.cout_g, pl.taps, pl.ksteps,
                                                                   pl.n_ntiles, pl.Nt, (uint4*)w_img);
  MNB_LAUNCHED(1);
  return 0;
}

int mnb_b1_plan(const mnb_conv_shape* s, const mnb_xnor_post* post, int32_t* out) {
  b1::Plan pl;
  int rc = b1::make_plan(s, pl);
  if (rc != 0) return rc;
  MNB_REQUIRE(out != nullptr, "b1_plan: null output");
  if (post) {
    rc = b1::check_post(post, s->out_c, pl.P, pl.Q);
    if (rc != 0) return rc;
  }
  const int32_t v[] = {pl.Nt, pl.n_ntiles, pl.u, pl.ksteps, pl.G, pl.col_tiles, pl.Wt, pl.BW, pl.TH, pl.TB, pl.row_tiles,
                       pl.n_mtiles, pl.TG, pl.ntg, pl.nstage, post != nullptr, pl.smem_bytes};
  for (int i = 0; i < 17; ++i) out[i] = v[i];
  return 0;
}

int mnb_b1_conv_fwd(const mnb_conv_shape* s, const void* a_plane, const void* w_img, const float* alpha, const float* bias,
                    float* y, int32_t* err_flag, mnb_stream_t stream) {
  return b1::run_conv(s, a_plane, w_img, alpha, bias, nullptr, y, err_flag, stream);
}

int64_t mnb_b1_post_bytes(const mnb_conv_shape* s, const mnb_xnor_post* post) {
  b1::Plan pl;
  if (b1::make_plan(s, pl) != 0 || b1::check_post(post, s->out_c, pl.P, pl.Q) != 0) return -1;
  const int OH = post->pool2 ? pl.P / 2 : pl.P, OW = post->pool2 ? pl.Q / 2 : pl.Q;
  return b1::post_bytes(pl.B, s->out_c, OH, OW, post);
}

int mnb_b1_conv_post(const mnb_conv_shape* s, const void* a_plane, const void* w_img, const float* alpha, const float* bias,
                     const mnb_xnor_post* post, void* out, int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(post != nullptr, "b1_conv_post: null consumer description");
  return b1::run_conv(s, a_plane, w_img, alpha, bias, post, out, err_flag, stream);
}

int mnb_b1_plane_maxpool(const void* in_plane, int32_t batch, int32_t channels, int32_t groups, int32_t h, int32_t w, int32_t k,
                         int32_t s, int32_t p, void* out_plane, mnb_stream_t stream) {
  MNB_REQUIRE(in_plane && out_plane, "b1_plane_maxpool: null pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && groups > 0 && channels % groups == 0 && h > 0 && w > 0 && k > 0 && s > 0 && p >= 0,
              "b1_plane_maxpool: bad shape");
  if (2 * p > k) return mnb_fail(MNB_E_UNSUPPORTED, "b1_plane_maxpool: padding %d beyond half the window %d", p, k);
  const int OH = (h + 2 * p - k) / s + 1, OW = (w + 2 * p - k) / s + 1;
  if (h + 2 * p < k || w + 2 * p < k) return mnb_fail(MNB_E_UNSUPPORTED, "b1_plane_maxpool: window larger than the plane");
  const int64_t planes = (int64_t)batch * groups * b1::units_per_group(channels / groups);
  const int64_t total = planes * OH * OW;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)MNB_NUM_SMS * 16);
  b1::plane_maxpool_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint4*)in_plane, planes, h, w, k, s, p, OH, OW,
                                                                     (uint4*)out_plane);
  MNB_LAUNCHED(1);
  return 0;
}

}  // extern "C"
