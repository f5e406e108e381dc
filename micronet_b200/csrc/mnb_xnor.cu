// Bit-packed XNOR-popcount forward convolution for the wbwtab scheme (binary activations, binary or ternary weights).
//
// BASELINE.json north_star: "the wbwtab binary/ternary case additionally gets a bit-packed XNOR-popcount kernel picked
// when ncu shows it beating the tensor-core path".  This file is that kernel; harness/xnor_probe.py times it against the
// packed-operand tensor-core forward (mnb_pk.cu) layer by layer and functional.xnor_preferred picks per layer (DESIGN.md 4.12).
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
};

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

template <int R_, int NW_, bool BORDER>
__global__ void __launch_bounds__(NTHREADS) conv_kernel(const Params p) {
  constexpr int PX = PxOf<R_, NW_>::value;
  typedef Rec<R_, NW_> RC;
  constexpr int TW = RC::TW;
  extern __shared__ __align__(16) uint32_t smem[];
  const int tabn = 1 + RC::TAB;
  const int g = blockIdx.y / p.ksplit, ks = blockIdx.y % p.ksplit;
  const int k0 = g * p.cout_g + ks * p.kb;                // first output channel of this block
  const int kcnt = min(p.kb, p.cout_g - ks * p.kb);
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
    yp[x] = p.y + ((int64_t)b * p.G * p.cout_g + k0) * PQ + pq;
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
      if (live[x]) yp[x][(int64_t)k * PQ] = fmaf((float)acc, al, bs);
    }
  }
}

typedef void (*KernelFn)(const Params);
static KernelFn pick(int R, int nw, bool border, int* rec_words, int* px = nullptr) {
#define XN_CASE(r, n)                                                                     \
  if (R == r && nw == n) {                                                                \
    if (rec_words) *rec_words = Rec<r, n>::WORDS;                                         \
    if (px) *px = PxOf<r, n>::value;                                                      \
    return border ? conv_kernel<r, n, true> : conv_kernel<r, n, false>;                   \
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
  xnor::Params p;
  p.B = s->batch; p.G = s->groups; p.cin_g = s->in_c / s->groups; p.cout_g = s->out_c / s->groups;
  p.H = s->in_h; p.W = s->in_w; p.R = s->ker_h; p.S = s->ker_w; p.stride = s->stride_h; p.pad = s->pad_h;
  p.P = (p.H + 2 * p.pad - p.R) / p.stride + 1;
  p.Q = (p.W + 2 * p.pad - p.S) / p.stride + 1;
  const int nw = xnor::words_per_group(p.cin_g), TW = p.R * p.S * nw;
  // border handling only where a tap can leave the image (never for an un-padded filter that fits)
  const bool border = p.pad > 0 || (p.P - 1) * p.stride + p.R > p.H || (p.Q - 1) * p.stride + p.S > p.W;
  int rec_words = 0, px = 1;
  xnor::KernelFn fn = xnor::pick(p.R, nw, border, &rec_words, &px);
  const int64_t npix = (int64_t)p.B * p.P * p.Q;
  const int pblocks = (int)((npix + xnor::NTHREADS * px - 1) / (xnor::NTHREADS * px));
  // k-slices: enough blocks for ~4 per SM, at most 40 KB of channel records per block
  int ksplit = 1;
  while (p.cout_g / ksplit > 8 && ((int64_t)pblocks * p.G * ksplit < 4 * MNB_NUM_SMS ||
                                   (int64_t)((p.cout_g + ksplit - 1) / ksplit) * rec_words * 4 > 40 * 1024))
    ++ksplit;
  p.kb = (p.cout_g + ksplit - 1) / ksplit;
  p.ksplit = (p.cout_g + p.kb - 1) / p.kb;
  const size_t smem = (size_t)p.kb * rec_words * 4;
  if (smem > 48 * 1024) return MNB_E_UNSUPPORTED;
  const uint32_t* words = (const uint32_t*)w_img;
  p.abits = (const uint32_t*)a_bits;
  p.wwords = words;
  p.wtabs = (const int32_t*)(words + (int64_t)s->out_c * 2 * TW);
  p.alpha = alpha; p.bias = bias; p.y = y;
  dim3 grid((unsigned)pblocks, (unsigned)(p.G * p.ksplit));
  if (grid.y > 65535) return MNB_E_UNSUPPORTED;
  fn<<<grid, xnor::NTHREADS, smem, (cudaStream_t)stream>>>(p);
  MNB_LAUNCHED(1);
  return 0;
}

}  // extern "C"
