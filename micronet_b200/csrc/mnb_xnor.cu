// Bit-packed XNOR-popcount forward convolution for the wbwtab scheme (binary activations, binary or ternary weights).
//
// BASELINE.json north_star: "the wbwtab binary/ternary case additionally gets a bit-packed XNOR-popcount kernel picked
// when ncu shows it beating the tensor-core path".  This file is that kernel; harness/xnor_probe.py times it against the
// packed-operand tensor-core forward (mnb_pk.cu) layer by layer and functional._xnor_forward picks per layer (DESIGN.md 4.12).
//
// Reference math (WB:11-36, 55-75, 98-146, 181-195): y = bias + alpha[k] * sum_{c,r,s} a[c] * w[k][c][r][s] with
// a = sign(x) in {-1, +1} (0 -> +1) and w in {-1, +1} (binary) or {-1, 0, +1} (ternary); out-of-image taps contribute 0.
// With one bit per value (A = [a == +1], S = [w == +1], N = [w != 0]):
//     sum_c a*w = popc(N) - 2 * popc(N & (A ^ S))
// The sum is an exact integer, so the result is bit-identical to the tensor-core path (same fmaf epilogue).
//
// Out-of-image taps read A = 0 (all "-1"), which adds -sum_c w[k][c][tap] to the full-filter sum; border pixels add the
// weight sums of their missing taps back from a 2-D prefix table (valid taps always form a rectangle of the filter).
//
// Layouts
//   activation bits  u32 [B][G][NW][H][W]      NW = ceil(C/g / 32); bit j of word n = channel g*C/g + 32 n + j
//   weight image     u32 [K][2][TW] (S words then N words, TW = R*S*NW, tap-major) followed by
//                    i32 [K][1 + (R+1)*(S+1)]  (popc total of N, then the prefix table of per-tap weight sums)
#include "mnb_common.cuh"

namespace xnor {

constexpr int NTHREADS = 256;

__host__ __device__ inline int words_per_group(int cin_g) { return (cin_g + 31) / 32; }

// ------------------------------------------------------------------------------------------------------------------
// activation packer: fp32 NCHW -> sign bit planes (x >= 0 or x == -0 -> 1: torch.sign(x) with 0 -> +1; NaN -> 1 like
// the engine's other binarizers, which test !(x < 0))
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS) pack_act_kernel(const float* __restrict__ x, int B, int Cc, int HW, int G,
                                                            uint32_t* __restrict__ out) {
  const int cin_g = Cc / G, nw = words_per_group(cin_g);
  const int64_t total = (int64_t)B * G * nw * HW;
  for (int64_t i = (int64_t)blockIdx.x * NTHREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * NTHREADS) {
    const int pix = (int)(i % HW);
    int64_t t = i / HW;
    const int n = (int)(t % nw); t /= nw;
    const int g = (int)(t % G);
    const int b = (int)(t / G);
    const int c0 = n * 32, cnt = min(32, cin_g - c0);
    const float* src = x + ((int64_t)b * Cc + (int64_t)g * cin_g + c0) * HW + pix;
    uint32_t word = 0;
#pragma unroll 8
    for (int j = 0; j < cnt; ++j) word |= (!(__ldg(src + (int64_t)j * HW) < 0.f) ? 1u : 0u) << j;
    out[i] = word;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// weight packer: integer levels [K][C/g][R][S] -> sign / non-zero words + popcount and prefix tables, one block per k
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) pack_weight_kernel(const int16_t* __restrict__ w, int K, int cin_g, int R, int S,
                                                          uint32_t* __restrict__ words, int32_t* __restrict__ tabs) {
  const int k = blockIdx.x, nw = words_per_group(cin_g), taps = R * S, TW = taps * nw;
  const int tabn = 1 + (R + 1) * (S + 1);
  __shared__ int32_t wsum[64];   // per-tap weight sums (taps <= 64)
  __shared__ int32_t nzc[64];
  const int16_t* wk = w + (int64_t)k * cin_g * taps;
  for (int t = threadIdx.x; t < taps; t += blockDim.x) { wsum[t] = 0; nzc[t] = 0; }
  __syncthreads();
  for (int e = threadIdx.x; e < TW; e += blockDim.x) {
    const int tap = e / nw, n = e % nw;
    uint32_t sw = 0, nz = 0;
    int sum = 0;
    for (int j = 0; j < 32 && n * 32 + j < cin_g; ++j) {
      const int v = wk[(int64_t)(n * 32 + j) * taps + tap];
      sw |= (v > 0 ? 1u : 0u) << j;
      nz |= (v != 0 ? 1u : 0u) << j;
      sum += (v > 0) - (v < 0);
    }
    words[((int64_t)k * 2 + 0) * TW + e] = sw;
    words[((int64_t)k * 2 + 1) * TW + e] = nz;
    atomicAdd(&wsum[tap], sum);
    atomicAdd(&nzc[tap], __popc(nz));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot = 0;
    for (int t = 0; t < taps; ++t) tot += nzc[t];
    tabs[(int64_t)k * tabn] = tot;
  }
  // prefix table P[i][j] = sum_{r < i, s < j} wsum[r][s]
  for (int e = threadIdx.x; e < (R + 1) * (S + 1); e += blockDim.x) {
    const int i = e / (S + 1), j = e % (S + 1);
    int acc = 0;
    for (int r = 0; r < i; ++r)
      for (int s = 0; s < j; ++s) acc += wsum[r * S + s];
    tabs[(int64_t)k * tabn + 1 + e] = acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// forward: one thread = PX output pixels (256 apart: coalesced), looping over the output channels of its block's
// (group, k-slice); the slice's weight words and per-channel constants sit in shared memory and are read as warp-wide
// broadcasts (three 16-byte loads per channel for the 128-channel 1x1 layers, shared by the PX pixels), activation words stay
// in registers: the kernel is instruction-issue bound, so per-output instructions are what this layout saves.
// ------------------------------------------------------------------------------------------------------------------
struct Params {
  const uint32_t* abits;
  const uint32_t* wwords;
  const int32_t* wtabs;
  const float* alpha;   // [K] or NULL (= 1)
  const float* bias;    // [K] or NULL
  float* y;
  int B, G, cin_g, cout_g, H, W, P, Q, R, S, stride, pad, kb, ksplit;
  // sign-bit epilogue (conv_kernel<..., true>, mnb_xnor_conv_post): BatchNorm constants (mean NULL = none), the consumer's
  // output format, unit geometry and the 2x2 pool
  const float *bn_mean, *bn_invstd, *bn_gamma, *bn_beta;
  void* out;
  int fmt, sg, out_cin_g, out_nw, pool;
};

// destination of output channel c in the consumer's plane, packed as (unit << 5) | bit: unit = (group, word) of the bit plane
// or the channel octet of the bf16 plane.  The producer's channel shuffle moves channel c to (c mod C/sg) * sg + c div (C/sg).
__host__ __device__ inline int post_dest(int c, int K, int fmt, int sg, int out_cin_g, int out_nw) {
  const int cpg = K / sg;
  const int cd = sg > 1 ? (c % cpg) * sg + c / cpg : c;
  if (fmt == MNB_XNOR_PM1_BF16) return ((cd >> 3) << 5) | (cd & 7);
  const int g = cd / out_cin_g, r = cd - g * out_cin_g;
  return ((g * out_nw + (r >> 5)) << 5) | (r & 31);
}

// flush one destination unit of one output pixel: OR the collected sign bits into the (zeroed) bit plane, or store the
// +-1 channels of the octet as bf16 (one 16-byte store when this thread holds all eight)
__device__ __forceinline__ void post_flush(const Params& p, int64_t base, int64_t unit_stride, int unit, uint32_t bits,
                                           uint32_t have) {
  if (unit < 0) return;
  if (p.fmt == MNB_XNOR_BITS) {
    if (bits) atomicOr(reinterpret_cast<uint32_t*>(p.out) + base + (int64_t)unit * unit_stride, bits);
    return;
  }
  uint16_t* o = reinterpret_cast<uint16_t*>(p.out) + (base + (int64_t)unit * unit_stride) * 8;
  if (have == 0xFFu) {
    uint32_t h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = (bits >> j) & 1u ? 0x3F80u : 0xBF80u;
    *reinterpret_cast<uint4*>(o) = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
  } else {
    for (int j = 0; j < 8; ++j)
      if ((have >> j) & 1u) o[j] = (bits >> j) & 1u ? 0x3F80u : 0xBF80u;
  }
}

// pixels per thread: two where the receptive field is a few words (1x1 layers: the per-channel shared-memory loads and loop
// overhead are shared), one where it is nine or more (3x3 / 5x5: 2 x 9 activation words + border state cost occupancy)
template <int R_, int NW_> struct PxOf { static constexpr int value = (R_ * R_ * NW_ <= 8) ? 2 : 1; };

// shared-memory record of one output channel: [S words TW][N words TW][popc(N) total, alpha, bias, 0][prefix table (R+1)^2]
template <int R_, int NW_>
struct Rec {
  static constexpr int TW = R_ * R_ * NW_;
  static constexpr int TWP = (TW + 3) & ~3;                       // 16-byte aligned sections
  static constexpr int TAB = (R_ + 1) * (R_ + 1);
  static constexpr int WORDS = 2 * TWP + 4 + ((TAB + 3) & ~3);
};

template <int R_, int NW_, bool BORDER, bool POST>
__global__ void __launch_bounds__(NTHREADS) conv_kernel(const Params p) {
  constexpr int PX = PxOf<R_, NW_>::value;
  typedef Rec<R_, NW_> RC;
  constexpr int TW = RC::TW;
  extern __shared__ __align__(16) uint32_t smem[];
  const int tabn = 1 + RC::TAB;
  const int g = blockIdx.y / p.ksplit, ks = blockIdx.y % p.ksplit;
  const int k0 = g * p.cout_g + ks * p.kb;                // first output channel of this block
  const int kcnt = min(p.kb, p.cout_g - ks * p.kb);
  // POST: per channel {mean, gamma * invstd, beta, destination} after the records (the BN+sign producers' constants)
  float4* pcst = reinterpret_cast<float4*>(smem + p.kb * RC::WORDS);
  if (POST) {
    const int K = p.G * p.cout_g;
    for (int e = threadIdx.x; e < kcnt; e += NTHREADS) {
      const int c = k0 + e;
      float4 v = make_float4(0.f, 1.f, 0.f, 0.f);
      if (p.bn_mean) v = make_float4(__ldg(p.bn_mean + c), __ldg(p.bn_gamma + c) * __ldg(p.bn_invstd + c), __ldg(p.bn_beta + c), 0.f);
      v.w = __int_as_float(post_dest(c, K, p.fmt, p.sg, p.out_cin_g, p.out_nw));
      pcst[e] = v;
    }
  }
  for (int e = threadIdx.x; e < kcnt * RC::WORDS; e += NTHREADS) {
    const int k = e / RC::WORDS, o = e - k * RC::WORDS;
    uint32_t v = 0;
    if (o < RC::TWP) { if (o < TW) v = __ldg(p.wwords + ((int64_t)(k0 + k) * 2 + 0) * TW + o); }
    else if (o < 2 * RC::TWP) { if (o - RC::TWP < TW) v = __ldg(p.wwords + ((int64_t)(k0 + k) * 2 + 1) * TW + (o - RC::TWP)); }
    else if (o == 2 * RC::TWP) v = (uint32_t)__ldg(p.wtabs + (int64_t)(k0 + k) * tabn);
    else if (o == 2 * RC::TWP + 1) v = __float_as_uint(p.alpha ? __ldg(p.alpha + k0 + k) : 1.f);
    else if (o == 2 * RC::TWP + 2) v = __float_as_uint(p.bias ? __ldg(p.bias + k0 + k) : 0.f);
    else if (o >= 2 * RC::TWP + 4 && o - (2 * RC::TWP + 4) < RC::TAB)
      v = (uint32_t)__ldg(p.wtabs + (int64_t)(k0 + k) * tabn + 1 + (o - (2 * RC::TWP + 4)));
    smem[e] = v;
  }
  __syncthreads();

  const int PQ = p.P * p.Q, HW = p.H * p.W;
  const int64_t npix = (int64_t)p.B * PQ;
  uint32_t a[PX][TW];
  bool live[PX];
  float* yp[PX];
  int r0[PX], r1[PX], s0[PX], s1[PX];
  bool border[PX];
  int64_t obase[PX];
  int cu[PX];                 // POST: destination unit being collected (-1: none), its bits and the channels seen
  uint32_t cb[PX], chv[PX];
  const int64_t out_hw = POST && p.pool ? (int64_t)(p.P >> 1) * (p.Q >> 1) : (int64_t)PQ;
  const int units = !POST ? 0 : p.fmt == MNB_XNOR_BITS ? p.out_nw * ((p.G * p.cout_g) / p.out_cin_g) : (p.G * p.cout_g) >> 3;
#pragma unroll
  for (int x = 0; x < PX; ++x) {
    const int64_t pix = ((int64_t)blockIdx.x * PX + x) * NTHREADS + threadIdx.x;
    live[x] = pix < npix;
    const int64_t pc = live[x] ? pix : 0;
    const int b = (int)(pc / PQ), pq = (int)(pc % PQ);
    const int op = pq / p.Q, oq = pq % p.Q;
    const int ih0 = op * p.stride - p.pad, iw0 = oq * p.stride - p.pad;
    // activation words of this pixel's receptive field (0 where the tap is outside the image)
    const uint32_t* ab = p.abits + ((int64_t)b * p.G + g) * NW_ * HW;
#pragma unroll
    for (int r = 0; r < R_; ++r)
#pragma unroll
      for (int s = 0; s < R_; ++s) {
        const int ih = ih0 + r, iw = iw0 + s;
        const bool ok = !BORDER || (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W);
#pragma unroll
        for (int n = 0; n < NW_; ++n) a[x][(r * R_ + s) * NW_ + n] = ok ? __ldg(ab + (int64_t)n * HW + ih * p.W + iw) : 0u;
      }
    // valid taps: rows [r0, r1) x columns [s0, s1)
    r0[x] = max(0, -ih0); r1[x] = max(r0[x], min(R_, p.H - ih0));
    s0[x] = max(0, -iw0); s1[x] = max(s0[x], min(R_, p.W - iw0));
    border[x] = BORDER && ((r0[x] != 0) || (r1[x] != R_) || (s0[x] != 0) || (s1[x] != R_));
    if (POST) {
      // destination pixel (pooled: the 2x2 window's output) and the offset of unit 0 of this image
      const int opq = p.pool ? (op >> 1) * (p.Q >> 1) + (oq >> 1) : pq;
      obase[x] = (int64_t)b * units * out_hw + opq;
      cu[x] = -1; cb[x] = 0u; chv[x] = 0u;
    } else {
      yp[x] = p.y + ((int64_t)b * p.G * p.cout_g + k0) * PQ + pq;
    }
  }

#pragma unroll 2
  for (int k = 0; k < kcnt; ++k) {
    const uint32_t* rec = smem + k * RC::WORDS;
    uint32_t ws[TW], wn[TW];
#pragma unroll
    for (int t = 0; t < TW; ++t) { ws[t] = rec[t]; wn[t] = rec[RC::TWP + t]; }
    const uint4 cst = *reinterpret_cast<const uint4*>(rec + 2 * RC::TWP);     // popc(N) total, alpha, bias
    const float al = __uint_as_float(cst.y), bs = __uint_as_float(cst.z);
#pragma unroll
    for (int x = 0; x < PX; ++x) {
      int cnt = 0;
#pragma unroll
      for (int t = 0; t < TW; ++t) cnt += __popc(wn[t] & (a[x][t] ^ ws[t]));
      int acc = (int)cst.x - 2 * cnt;
      if (BORDER && border[x]) {
        const int32_t* P = reinterpret_cast<const int32_t*>(rec + 2 * RC::TWP + 4);
        const int rect = P[r1[x] * (R_ + 1) + s1[x]] - P[r0[x] * (R_ + 1) + s1[x]] - P[r1[x] * (R_ + 1) + s0[x]] +
                         P[r0[x] * (R_ + 1) + s0[x]];
        acc += P[R_ * (R_ + 1) + R_] - rect;
      }
      if (!POST) {
        if (live[x]) yp[x][(int64_t)k * PQ] = fmaf((float)acc, al, bs);
      } else {
        // the BN+sign producers' op sequence (mnb_conv_packed.cu): bn = fmaf(v - mean, gamma * invstd, beta), bit = !(bn < 0)
        const float4 pc = pcst[k];
        float v = fmaf((float)acc, al, bs);
        if (p.bn_mean) v = fmaf(v - pc.x, pc.y, pc.z);
        const int dest = __float_as_int(pc.w), unit = dest >> 5, j = dest & 31;
        if (unit != cu[x]) {
          if (live[x]) post_flush(p, obase[x], out_hw, cu[x], cb[x], chv[x]);
          cu[x] = unit; cb[x] = 0u; chv[x] = 0u;
        }
        cb[x] |= (v < 0.f ? 0u : 1u) << j;
        chv[x] |= 1u << j;
      }
    }
  }
  if (POST) {
#pragma unroll
    for (int x = 0; x < PX; ++x)
      if (live[x]) post_flush(p, obase[x], out_hw, cu[x], cb[x], chv[x]);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// stem producer: fp32 NCHW [-> eval BatchNorm] -> sign [-> 2x2 max-pool] [-> channel shuffle] -> the consumer's bit plane.
// One thread per output word, gathering its (up to) 32 channels through the inverse shuffle; the pooled bit is the OR of the
// window's four sign bits (the max of +-1 values).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS) pack_act_post_kernel(const float* __restrict__ x, int B, int Cc, int H, int W,
                                                                 int G, int sg, int pool, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, uint32_t* __restrict__ out) {
  const int cin_g = Cc / G, nw = words_per_group(cin_g), cpg = Cc / sg;
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W, OHW = OH * OW, HW = H * W;
  const int64_t total = (int64_t)B * G * nw * OHW;
  for (int64_t i = (int64_t)blockIdx.x * NTHREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * NTHREADS) {
    const int opix = (int)(i % OHW);
    int64_t t = i / OHW;
    const int n = (int)(t % nw); t /= nw;
    const int g = (int)(t % G);
    const int b = (int)(t / G);
    const int oh = opix / OW, ow = opix % OW;
    const int pix = pool ? (2 * oh) * W + 2 * ow : opix;
    const int c0 = n * 32, cnt = min(32, cin_g - c0);
    uint32_t word = 0;
    for (int j = 0; j < cnt; ++j) {
      const int cd = g * cin_g + c0 + j;
      const int c = sg > 1 ? (cd % sg) * cpg + cd / sg : cd;   // inverse of the producer's shuffle
      const float* src = x + ((int64_t)b * Cc + c) * HW + pix;
      float mu = 0.f, k = 1.f, be = 0.f;
      if (mean) { mu = __ldg(mean + c); k = __ldg(gamma + c) * __ldg(invstd + c); be = __ldg(beta + c); }
      uint32_t bit = 0;
      for (int q = 0; q < (pool ? 4 : 1); ++q) {
        float v = __ldg(src + (q >> 1) * W + (q & 1));
        if (mean) v = fmaf(v - mu, k, be);
        bit |= v < 0.f ? 0u : 1u;
      }
      word |= bit << j;
    }
    out[i] = word;
  }
}

typedef void (*KernelFn)(const Params);
static KernelFn pick(int R, int nw, bool border, int* rec_words, int* px = nullptr, bool post = false) {
#define XN_CASE(r, n)                                                                                 \
  if (R == r && nw == n) {                                                                            \
    if (rec_words) *rec_words = Rec<r, n>::WORDS;                                                     \
    if (px) *px = PxOf<r, n>::value;                                                                  \
    if (post) return border ? conv_kernel<r, n, true, true> : conv_kernel<r, n, false, true>;         \
    return border ? conv_kernel<r, n, true, false> : conv_kernel<r, n, false, false>;                 \
  }
  XN_CASE(1, 1) XN_CASE(1, 2) XN_CASE(1, 3) XN_CASE(1, 4) XN_CASE(1, 8)
  XN_CASE(3, 1) XN_CASE(3, 2) XN_CASE(3, 4)
  XN_CASE(5, 1) XN_CASE(5, 2)
#undef XN_CASE
  return nullptr;
}

static int check_shape(const mnb_conv_shape* s) {
  MNB_REQUIRE(s != nullptr, "xnor: null shape");
  MNB_REQUIRE(s->batch > 0 && s->in_c > 0 && s->out_c > 0 && s->groups > 0 && s->in_c % s->groups == 0 &&
                  s->out_c % s->groups == 0, "xnor: bad channel counts");
  if (s->ker_h != s->ker_w || s->stride_h != s->stride_w || s->pad_h != s->pad_w || s->dil_h != 1 || s->dil_w != 1)
    return MNB_E_UNSUPPORTED;
  if (s->ker_h * s->ker_w > 64) return MNB_E_UNSUPPORTED;
  if (pick(s->ker_h, words_per_group(s->in_c / s->groups), true, nullptr) == nullptr) return MNB_E_UNSUPPORTED;
  const int P = (s->in_h + 2 * s->pad_h - s->ker_h) / s->stride_h + 1, Q = (s->in_w + 2 * s->pad_w - s->ker_w) / s->stride_w + 1;
  if (P <= 0 || Q <= 0) return MNB_E_UNSUPPORTED;
  return 0;
}

// the launch configuration of a shape that has passed check_shape: kernel instance, k-slices, grid and shared memory
struct Plan {
  int P, Q, nw, border, px, post, ksplit, kb, pblocks, smem, grid_y;
  bool refused;              // shared memory or grid beyond what the launch allows: MNB_E_UNSUPPORTED, nothing launched
  KernelFn fn;
};

static void make_plan(const mnb_conv_shape* s, bool post, Plan& pl) {
  const int cout_g = s->out_c / s->groups, R = s->ker_h;
  pl.P = (s->in_h + 2 * s->pad_h - R) / s->stride_h + 1;
  pl.Q = (s->in_w + 2 * s->pad_w - s->ker_w) / s->stride_w + 1;
  pl.nw = words_per_group(s->in_c / s->groups);
  // border handling only where a tap can leave the image (never for an un-padded filter that fits)
  pl.border = s->pad_h > 0 || (pl.P - 1) * s->stride_h + R > s->in_h || (pl.Q - 1) * s->stride_w + s->ker_w > s->in_w;
  pl.post = post;
  int rec_words = 0;
  pl.px = 1;
  pl.fn = pick(R, pl.nw, pl.border, &rec_words, &pl.px, post);
  const int per_k = rec_words * 4 + (post ? 16 : 0);     // shared-memory bytes per output channel
  const int64_t npix = (int64_t)s->batch * pl.P * pl.Q;
  pl.pblocks = (int)((npix + NTHREADS * pl.px - 1) / (NTHREADS * pl.px));
  // k-slices: enough blocks for ~4 per SM, at most 40 KB of channel records per block
  int ksplit = 1;
  while (cout_g / ksplit > 8 && ((int64_t)pl.pblocks * s->groups * ksplit < 4 * MNB_NUM_SMS ||
                                 (int64_t)((cout_g + ksplit - 1) / ksplit) * per_k > 40 * 1024))
    ++ksplit;
  pl.kb = (cout_g + ksplit - 1) / ksplit;
  pl.ksplit = (cout_g + pl.kb - 1) / pl.kb;
  pl.smem = pl.kb * per_k;
  pl.grid_y = s->groups * pl.ksplit;
  pl.refused = pl.smem > 48 * 1024 || pl.grid_y > 65535;
}

// post: NULL for the fp32 output of mnb_xnor_conv_fwd.  The shape has passed check_shape (and check_post when post is set).
static int launch(const mnb_conv_shape* s, const void* a_bits, const void* w_img, const float* alpha, const float* bias,
                  const mnb_xnor_post* post, void* out, mnb_stream_t stream) {
  Plan pl;
  make_plan(s, post != nullptr, pl);
  if (pl.refused) return MNB_E_UNSUPPORTED;
  Params p;
  p.B = s->batch; p.G = s->groups; p.cin_g = s->in_c / s->groups; p.cout_g = s->out_c / s->groups;
  p.H = s->in_h; p.W = s->in_w; p.R = s->ker_h; p.S = s->ker_w; p.stride = s->stride_h; p.pad = s->pad_h;
  p.P = pl.P; p.Q = pl.Q;
  p.kb = pl.kb; p.ksplit = pl.ksplit;
  const int TW = p.R * p.S * pl.nw;
  const uint32_t* words = (const uint32_t*)w_img;
  p.abits = (const uint32_t*)a_bits;
  p.wwords = words;
  p.wtabs = (const int32_t*)(words + (int64_t)s->out_c * 2 * TW);
  p.alpha = alpha; p.bias = bias;
  p.y = post ? nullptr : (float*)out;
  p.bn_mean = p.bn_invstd = p.bn_gamma = p.bn_beta = nullptr;
  p.out = nullptr;
  p.fmt = p.sg = p.out_cin_g = p.out_nw = p.pool = 0;
  if (post) {
    p.bn_mean = post->bn_mean; p.bn_invstd = post->bn_invstd; p.bn_gamma = post->bn_gamma; p.bn_beta = post->bn_beta;
    p.out = out;
    p.fmt = post->format; p.sg = post->shuffle_groups; p.pool = post->pool2;
    p.out_cin_g = s->out_c / post->out_groups; p.out_nw = words_per_group(p.out_cin_g);
  }
  dim3 grid((unsigned)pl.pblocks, (unsigned)pl.grid_y);
  pl.fn<<<grid, NTHREADS, (size_t)pl.smem, (cudaStream_t)stream>>>(p);
  MNB_LAUNCHED(1);
  return 0;
}

// the consumer description of mnb_xnor_conv_post / mnb_xnor_pack_act_post for C producer channels on a P x Q plane
// (P = Q = 0: plane size not known yet, only the channel rules are checked)
static int check_post(const mnb_xnor_post* post, int C, int P, int Q) {
  MNB_REQUIRE(post != nullptr, "xnor post: null consumer description");
  MNB_REQUIRE(post->format == MNB_XNOR_BITS || post->format == MNB_XNOR_PM1_BF16, "xnor post: unknown format %d", post->format);
  MNB_REQUIRE(post->shuffle_groups >= 1 && C % post->shuffle_groups == 0, "xnor post: shuffle groups %d do not divide %d channels",
              post->shuffle_groups, C);
  MNB_REQUIRE(post->pool2 == 0 || post->pool2 == 1, "xnor post: pool2 must be 0 or 1");
  const bool any_bn = post->bn_mean || post->bn_invstd || post->bn_gamma || post->bn_beta;
  MNB_REQUIRE(!any_bn || (post->bn_mean && post->bn_invstd && post->bn_gamma && post->bn_beta),
              "xnor post: BatchNorm needs all four of mean, invstd, gamma, beta");
  if (post->format == MNB_XNOR_BITS) {
    MNB_REQUIRE(post->out_groups >= 1 && C % post->out_groups == 0, "xnor post: consumer groups %d do not divide %d channels",
                post->out_groups, C);
  } else {
    if (post->pool2) return mnb_fail(MNB_E_UNSUPPORTED, "xnor post: the bf16 plane takes no folded pool");
    if (C % 8) return mnb_fail(MNB_E_UNSUPPORTED, "xnor post: the bf16 plane needs C %% 8 == 0");
  }
  if (post->pool2 && ((P | Q) & 1)) return mnb_fail(MNB_E_UNSUPPORTED, "xnor post: a 2x2 pool over an odd plane (%d x %d)", P, Q);
  return 0;
}

}  // namespace xnor

extern "C" {

int mnb_xnor_supported(const mnb_conv_shape* s) {
  const int rc = xnor::check_shape(s);
  return rc == 0 ? 1 : (rc == MNB_E_UNSUPPORTED ? 0 : rc);
}

int64_t mnb_xnor_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups) {
  if (batch <= 0 || channels <= 0 || groups <= 0 || channels % groups) return -1;
  return (int64_t)batch * groups * xnor::words_per_group(channels / groups) * h * w * 4;
}

int mnb_xnor_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups, void* out_bits,
                      mnb_stream_t stream) {
  MNB_REQUIRE(x && out_bits, "xnor_pack_act: null pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && groups > 0 && channels % groups == 0, "xnor_pack_act: bad shape");
  const int64_t total = mnb_xnor_act_bytes(batch, channels, h, w, groups) / 4;
  const int blocks = (int)std::min<int64_t>((total + xnor::NTHREADS - 1) / xnor::NTHREADS, (int64_t)MNB_NUM_SMS * 16);
  xnor::pack_act_kernel<<<blocks, xnor::NTHREADS, 0, (cudaStream_t)stream>>>(x, batch, channels, h * w, groups,
                                                                             (uint32_t*)out_bits);
  MNB_LAUNCHED(1);
  return 0;
}

int64_t mnb_xnor_wimage_bytes(const mnb_conv_shape* s) {
  if (xnor::check_shape(s) != 0) return -1;
  const int nw = xnor::words_per_group(s->in_c / s->groups), TW = s->ker_h * s->ker_w * nw;
  return (int64_t)s->out_c * (2 * TW + 1 + (s->ker_h + 1) * (s->ker_w + 1)) * 4;
}

int mnb_xnor_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream) {
  const int rc = xnor::check_shape(s);
  if (rc != 0) return rc;
  MNB_REQUIRE(w_int && w_img, "xnor_pack_weight: null pointer");
  const int nw = xnor::words_per_group(s->in_c / s->groups), TW = s->ker_h * s->ker_w * nw;
  uint32_t* words = (uint32_t*)w_img;
  int32_t* tabs = (int32_t*)(words + (int64_t)s->out_c * 2 * TW);
  xnor::pack_weight_kernel<<<s->out_c, 128, 0, (cudaStream_t)stream>>>(w_int, s->out_c, s->in_c / s->groups, s->ker_h, s->ker_w,
                                                                       words, tabs);
  MNB_LAUNCHED(1);
  return 0;
}

int mnb_xnor_conv_fwd(const mnb_conv_shape* s, const void* a_bits, const void* w_img, const float* alpha, const float* bias,
                      float* y, mnb_stream_t stream) {
  const int rc = xnor::check_shape(s);
  if (rc != 0) return rc;
  MNB_REQUIRE(a_bits && w_img && y, "xnor_conv_fwd: null pointer");
  return xnor::launch(s, a_bits, w_img, alpha, bias, nullptr, y, stream);
}

int64_t mnb_xnor_post_bytes(const mnb_conv_shape* s, const mnb_xnor_post* post) {
  if (xnor::check_shape(s) != 0 || xnor::check_post(post, s->out_c, 0, 0) != 0) return -1;
  const int P = (s->in_h + 2 * s->pad_h - s->ker_h) / s->stride_h + 1, Q = (s->in_w + 2 * s->pad_w - s->ker_w) / s->stride_w + 1;
  if (post->pool2 && ((P | Q) & 1)) return -1;
  const int OH = post->pool2 ? P / 2 : P, OW = post->pool2 ? Q / 2 : Q;
  if (post->format == MNB_XNOR_PM1_BF16) return (int64_t)s->batch * s->out_c * OH * OW * 2;
  return mnb_xnor_act_bytes(s->batch, s->out_c, OH, OW, post->out_groups);
}

int mnb_xnor_conv_post(const mnb_conv_shape* s, const void* a_bits, const void* w_img, const float* alpha, const float* bias,
                       const mnb_xnor_post* post, void* out, mnb_stream_t stream) {
  int rc = xnor::check_shape(s);
  if (rc != 0) return rc;
  MNB_REQUIRE(a_bits && w_img && out, "xnor_conv_post: null pointer");
  const int P = (s->in_h + 2 * s->pad_h - s->ker_h) / s->stride_h + 1, Q = (s->in_w + 2 * s->pad_w - s->ker_w) / s->stride_w + 1;
  rc = xnor::check_post(post, s->out_c, P, Q);
  if (rc != 0) return rc;
  if (post->format == MNB_XNOR_PM1_BF16 && (reinterpret_cast<uintptr_t>(out) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "xnor_conv_post: the bf16 plane must be 16-byte aligned");
  if (post->format == MNB_XNOR_BITS) {
    // bits are OR-ed in (several blocks, and the four pixels of a pooled window, write one word): zero the plane first
    const int64_t nbytes = mnb_xnor_post_bytes(s, post);
    cudaError_t e = cudaMemsetAsync(out, 0, (size_t)nbytes, (cudaStream_t)stream);
    if (e != cudaSuccess) return mnb_fail((int)e, "xnor_conv_post: memset failed: %s", cudaGetErrorString(e));
  }
  return xnor::launch(s, a_bits, w_img, alpha, bias, post, out, stream);
}

int mnb_xnor_plan(const mnb_conv_shape* s, const mnb_xnor_post* post, int32_t* out) {
  int rc = xnor::check_shape(s);
  if (rc != 0) return rc;
  MNB_REQUIRE(out != nullptr, "xnor_plan: null output");
  xnor::Plan pl;
  xnor::make_plan(s, post != nullptr, pl);
  if (post) {
    rc = xnor::check_post(post, s->out_c, pl.P, pl.Q);
    if (rc != 0) return rc;
  }
  const int32_t v[] = {s->ker_h, pl.nw, pl.border, pl.px, pl.post, pl.ksplit, pl.kb, pl.pblocks, pl.smem, pl.refused};
  for (int i = 0; i < 10; ++i) out[i] = v[i];
  return 0;
}

int mnb_xnor_pack_act_post(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_xnor_post* post,
                           void* out_bits, mnb_stream_t stream) {
  MNB_REQUIRE(x && out_bits, "xnor_pack_act_post: null pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0, "xnor_pack_act_post: bad shape");
  const int rc = xnor::check_post(post, channels, h, w);
  if (rc != 0) return rc;
  if (post->format != MNB_XNOR_BITS) return mnb_fail(MNB_E_UNSUPPORTED, "xnor_pack_act_post: writes bit planes only");
  const int OH = post->pool2 ? h / 2 : h, OW = post->pool2 ? w / 2 : w;
  const int64_t total = mnb_xnor_act_bytes(batch, channels, OH, OW, post->out_groups) / 4;
  const int blocks = (int)std::min<int64_t>((total + xnor::NTHREADS - 1) / xnor::NTHREADS, (int64_t)MNB_NUM_SMS * 16);
  xnor::pack_act_post_kernel<<<blocks, xnor::NTHREADS, 0, (cudaStream_t)stream>>>(
      x, batch, channels, h, w, post->out_groups, post->shuffle_groups, post->pool2, post->bn_mean, post->bn_invstd,
      post->bn_gamma, post->bn_beta, (uint32_t*)out_bits);
  MNB_LAUNCHED(1);
  return 0;
}

}  // extern "C"
