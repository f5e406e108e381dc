// Producer-side fusions around the quantized convolutions of a wbwtab-prepared block (SURVEY.md 8 f2):
//
//   conv -> BatchNorm2d(train) -> ActivationQuantizer(A=2) [-> MaxPool2d] -> channel_shuffle -> next conv
//
//  * bn_sign:  y = sign(gamma * (x - mean) * invstd + beta), 0 -> +1, saturate STE |bn| < 1  (WB:11-36 on top of
//              nn.BatchNorm2d), one read of x and one write of y forward; two passes backward (channel reductions, apply)
//              that also produce the channel sums of dx (the preceding convolution's bias gradient).
//  * maxpool:  nn.MaxPool2d forward / backward with a one-byte window index instead of int64 indices; same
//              first-maximum tie rule and the same accumulation order as ATen's kernels.
//  * every producer can write its output with the channel permutation of the next block's channel_shuffle
//    (nin_gc.py:9-21) folded in, and read the incoming gradient through the same permutation, so the shuffle copies
//    disappear:  out[:, a * sg + b] = in[:, b * (C / sg) + a].
//
// All of it is HBM-bound plane streaming: float4 accesses, 32-bit index arithmetic, grid sized from the channel
// count x batch splits; reductions are deterministic (fixed split order, last-block-done finalisation).
#include <algorithm>

#include "mnb_common.cuh"

static inline cudaStream_t S(mnb_stream_t s) { return (cudaStream_t)s; }
constexpr int FUSED_SPLITS = 32;  // must not exceed the 32 split slots of the scratch layout (mnb_observe_scratch_bytes)

__device__ __forceinline__ uint32_t shuffled_channel(uint32_t c, uint32_t sg, uint32_t cpg) {
  return sg > 1 ? (c % cpg) * sg + c / cpg : c;
}

// ------------------------------------------------------------------ BatchNorm + sign, forward
__global__ void __launch_bounds__(256) bn_sign_fwd_v4_kernel(const float4* __restrict__ x, uint32_t n4, uint32_t channels,
                                                             uint32_t hw4, uint32_t sg, const float* __restrict__ mean,
                                                             const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float4* __restrict__ y,
                                                             uint32_t* __restrict__ bits) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t n4_up = (n4 + 31u) & ~31u;  // warp-uniform trip count (shuffles below)
  const uint32_t cpg = channels / sg;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n4_up; i += stride) {
    uint32_t nib = 0;
    if (i < n4) {
      const uint32_t plane = i / hw4, off = i - plane * hw4;
      const uint32_t b = plane / channels, c = plane - b * channels;
      const float mu = __ldg(mean + c), sc = __ldg(gamma + c) * __ldg(invstd + c), be = __ldg(beta + c);
      const float4 v = __ldg(x + i);
      const float b0 = fmaf(v.x - mu, sc, be), b1 = fmaf(v.y - mu, sc, be), b2 = fmaf(v.z - mu, sc, be),
                  b3 = fmaf(v.w - mu, sc, be);
      const uint32_t o = (b * channels + shuffled_channel(c, sg, cpg)) * hw4 + off;
      y[o] = make_float4(b0 < 0.f ? -1.f : 1.f, b1 < 0.f ? -1.f : 1.f, b2 < 0.f ? -1.f : 1.f, b3 < 0.f ? -1.f : 1.f);
      nib = (uint32_t)(fabsf(b0) < 1.f) | ((uint32_t)(fabsf(b1) < 1.f) << 1) | ((uint32_t)(fabsf(b2) < 1.f) << 2) |
            ((uint32_t)(fabsf(b3) < 1.f) << 3);
    }
    uint32_t w = nib << (4 * (lane & 7));
    w |= __shfl_xor_sync(0xffffffffu, w, 1);
    w |= __shfl_xor_sync(0xffffffffu, w, 2);
    w |= __shfl_xor_sync(0xffffffffu, w, 4);
    if ((lane & 7) == 0 && i < n4) bits[i >> 3] = w;
  }
}

// any plane size (scalar accesses, 64-bit indices)
__global__ void __launch_bounds__(256) bn_sign_fwd_kernel(const float* __restrict__ x, int64_t n, int channels, int hw,
                                                          int sg, const float* __restrict__ mean,
                                                          const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float* __restrict__ y,
                                                          uint32_t* __restrict__ bits) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t cpg = (uint32_t)(channels / sg);
  for (int64_t base = warp * 32; base < n; base += nwarps * 32) {
    const int64_t i = base + lane;
    bool pass = false;
    if (i < n) {
      const int64_t plane = i / hw;
      const int c = (int)(plane % channels);
      const float sc = __ldg(gamma + c) * __ldg(invstd + c);
      const float bn = fmaf(__ldg(x + i) - __ldg(mean + c), sc, __ldg(beta + c));
      pass = fabsf(bn) < 1.f;
      const int64_t o = (plane - c + shuffled_channel((uint32_t)c, (uint32_t)sg, cpg)) * hw + (i - plane * hw);
      y[o] = bn < 0.f ? -1.f : 1.f;
    }
    const uint32_t word = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) bits[base >> 5] = word;
  }
}

// ------------------------------------------------------------------ BatchNorm + sign, backward
// pass 1: dbeta = sum g*pass, dgamma = sum g*pass*xhat per channel.  `g` is indexed through the output permutation.
template <bool VEC>
__global__ void __launch_bounds__(256) bn_sign_bwd_reduce_kernel(const float* __restrict__ g, const uint32_t* __restrict__ bits,
                                                                 const float* __restrict__ x, int batch, int channels, int hw,
                                                                 int sg, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd, float* __restrict__ dgamma,
                                                                 float* __restrict__ dbeta, uint32_t* counters,
                                                                 double* partial) {
  __shared__ double red[32];
  __shared__ bool last;
  const int c = blockIdx.x, sp = blockIdx.y, nsp = gridDim.y;
  const int oc = (int)shuffled_channel((uint32_t)c, (uint32_t)sg, (uint32_t)(channels / sg));
  const float mu = __ldg(mean + c), is = __ldg(invstd + c);
  const int b_lo = (int)((int64_t)batch * sp / nsp), b_hi = (int)((int64_t)batch * (sp + 1) / nsp);
  double s1, s2;
  if (VEC) {
    const uint32_t hw4 = (uint32_t)hw >> 2, total = (uint32_t)(b_hi - b_lo) * hw4;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float f1[2] = {0.f, 0.f}, f2[2] = {0.f, 0.f};
    for (uint32_t t0 = threadIdx.x; t0 < total; t0 += 2 * blockDim.x) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t t = t0 + u * blockDim.x;
        if (t < total) {
          const uint32_t b = t / hw4, i = t - b * hw4;
          const uint32_t fi4 = ((uint32_t)(b_lo + b) * channels + c) * hw4 + i;
          const uint32_t go4 = ((uint32_t)(b_lo + b) * channels + oc) * hw4 + i;
          const uint32_t nib = (__ldg(bits + (fi4 >> 3)) >> (4 * (fi4 & 7))) & 15u;
          const float4 gv = __ldg(g4 + go4), xv = __ldg(x4 + fi4);
          const float g0 = (nib & 1u) ? gv.x : 0.f, g1 = (nib & 2u) ? gv.y : 0.f, g2 = (nib & 4u) ? gv.z : 0.f,
                      g3 = (nib & 8u) ? gv.w : 0.f;
          f1[u] += (g0 + g1) + (g2 + g3);
          f2[u] += (g0 * ((xv.x - mu) * is) + g1 * ((xv.y - mu) * is)) + (g2 * ((xv.z - mu) * is) + g3 * ((xv.w - mu) * is));
        }
      }
    }
    s1 = (double)f1[0] + (double)f1[1];
    s2 = (double)f2[0] + (double)f2[1];
  } else {
    s1 = 0.0; s2 = 0.0;
    for (int b = b_lo; b < b_hi; ++b) {
      const int64_t off = ((int64_t)b * channels + c) * hw, goff = ((int64_t)b * channels + oc) * hw;
      float f1 = 0.f, f2 = 0.f;
      for (int i = threadIdx.x; i < hw; i += blockDim.x) {
        const int64_t fi = off + i;
        const bool pass = (__ldg(bits + (fi >> 5)) >> (fi & 31)) & 1u;
        const float gv = pass ? __ldg(g + goff + i) : 0.f;
        f1 += gv;
        f2 += gv * ((__ldg(x + fi) - mu) * is);
      }
      s1 += (double)f1; s2 += (double)f2;
    }
  }
  s1 = mnb_block_reduce(s1, MnbSum(), 0.0, red);
  s2 = mnb_block_reduce(s2, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    partial[((int64_t)c * nsp + sp) * 2 + 0] = s1;
    partial[((int64_t)c * nsp + sp) * 2 + 1] = s2;
    __threadfence();
    last = (atomicAdd(counters + c, 1u) == (uint32_t)nsp - 1);
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  s1 = 0.0; s2 = 0.0;
  for (int j = 0; j < nsp; ++j) { s1 += partial[((int64_t)c * nsp + j) * 2]; s2 += partial[((int64_t)c * nsp + j) * 2 + 1]; }
  dbeta[c] = (float)s1;
  dgamma[c] = (float)s2;
  counters[c] = 0;
}

// pass 2: dx = gamma * invstd * (g*pass - dbeta/N - xhat * dgamma/N)  (training) or gamma * invstd * g*pass (eval),
// plus the per-channel sum of the dx values just written (what the producing convolution needs as its bias gradient).
template <bool VEC>
__global__ void __launch_bounds__(256) bn_sign_bwd_apply_kernel(const float* __restrict__ g, const uint32_t* __restrict__ bits,
                                                                const float* __restrict__ x, int batch, int channels, int hw,
                                                                int sg, float inv_count, const float* __restrict__ mean,
                                                                const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                                                                int training, float* __restrict__ dx, float* __restrict__ dx_sum,
                                                                uint32_t* counters, double* partial) {
  __shared__ double red[32];
  __shared__ bool last;
  const int c = blockIdx.x, sp = blockIdx.y, nsp = gridDim.y;
  const int oc = (int)shuffled_channel((uint32_t)c, (uint32_t)sg, (uint32_t)(channels / sg));
  const float mu = __ldg(mean + c), is = __ldg(invstd + c), k = __ldg(gamma + c) * is;
  const float db = training ? __ldg(dbeta + c) * inv_count : 0.f, dg = training ? __ldg(dgamma + c) * inv_count : 0.f;
  const int b_lo = (int)((int64_t)batch * sp / nsp), b_hi = (int)((int64_t)batch * (sp + 1) / nsp);
  double s;
  if (VEC) {
    const uint32_t hw4 = (uint32_t)hw >> 2, total = (uint32_t)(b_hi - b_lo) * hw4;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* dx4 = reinterpret_cast<float4*>(dx);
    float f[2] = {0.f, 0.f};
    for (uint32_t t0 = threadIdx.x; t0 < total; t0 += 2 * blockDim.x) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t t = t0 + u * blockDim.x;
        if (t < total) {
          const uint32_t b = t / hw4, i = t - b * hw4;
          const uint32_t fi4 = ((uint32_t)(b_lo + b) * channels + c) * hw4 + i;
          const uint32_t go4 = ((uint32_t)(b_lo + b) * channels + oc) * hw4 + i;
          const uint32_t nib = (__ldg(bits + (fi4 >> 3)) >> (4 * (fi4 & 7))) & 15u;
          const float4 gv = __ldg(g4 + go4);
          float v0 = (nib & 1u) ? gv.x : 0.f, v1 = (nib & 2u) ? gv.y : 0.f, v2 = (nib & 4u) ? gv.z : 0.f,
                v3 = (nib & 8u) ? gv.w : 0.f;
          if (training) {
            const float4 xv = __ldg(x4 + fi4);
            v0 = bn_bwd_centre(v0, db, (xv.x - mu) * is, dg);
            v1 = bn_bwd_centre(v1, db, (xv.y - mu) * is, dg);
            v2 = bn_bwd_centre(v2, db, (xv.z - mu) * is, dg);
            v3 = bn_bwd_centre(v3, db, (xv.w - mu) * is, dg);
          }
          const float4 o = make_float4(k * v0, k * v1, k * v2, k * v3);
          dx4[fi4] = o;
          f[u] += (o.x + o.y) + (o.z + o.w);
        }
      }
    }
    s = (double)f[0] + (double)f[1];
  } else {
    s = 0.0;
    for (int b = b_lo; b < b_hi; ++b) {
      const int64_t off = ((int64_t)b * channels + c) * hw, goff = ((int64_t)b * channels + oc) * hw;
      float f = 0.f;
      for (int i = threadIdx.x; i < hw; i += blockDim.x) {
        const int64_t fi = off + i;
        const bool pass = (__ldg(bits + (fi >> 5)) >> (fi & 31)) & 1u;
        float v = pass ? __ldg(g + goff + i) : 0.f;
        if (training) v = bn_bwd_centre(v, db, (__ldg(x + fi) - mu) * is, dg);
        v = k * v;
        dx[fi] = v;
        f += v;
      }
      s += (double)f;
    }
  }
  if (!dx_sum) return;
  s = mnb_block_reduce(s, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    partial[((int64_t)c * nsp + sp) * 2] = s;
    __threadfence();
    last = (atomicAdd(counters + c, 1u) == (uint32_t)nsp - 1);
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  s = 0.0;
  for (int j = 0; j < nsp; ++j) s += partial[((int64_t)c * nsp + j) * 2];
  dx_sum[c] = (float)s;
  counters[c] = 0;
}

static bool planes_vectorizable(int64_t n, int hw, const void* a, const void* b, const void* c) {
  return (hw & 3) == 0 && n < (1ll << 31) &&
         (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15) == 0;
}
// (channels x splits) blocks: about two waves of 8 resident 256-thread blocks per SM, so that every block streams
// >= ~100 KB (small blocks spend as long being scheduled as loading)
static int plane_splits(int batch, int64_t per, int channels) {
  const int64_t want = (2 * 8 * MNB_NUM_SMS + channels - 1) / channels;
  return (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(std::min<int64_t>(FUSED_SPLITS, batch), per / 2048), want));
}

extern "C" int mnb_bn_sign_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                               const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups,
                               float* y, uint32_t* pass_bits, mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && invstd && gamma && beta && y && pass_bits, "NULL bn_sign_fwd pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0, "bad bn_sign_fwd shape");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  const int64_t n = (int64_t)batch * channels * hw;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  if (planes_vectorizable(n, hw, x, y, nullptr))
    bn_sign_fwd_v4_kernel<<<blocks, 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), (uint32_t)(n / 4),
                                                         (uint32_t)channels, (uint32_t)(hw / 4), (uint32_t)out_shuffle_groups,
                                                         mean, invstd, gamma, beta, reinterpret_cast<float4*>(y), pass_bits);
  else
    bn_sign_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(x, n, channels, hw, out_shuffle_groups, mean, invstd, gamma, beta, y,
                                                      pass_bits);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_sign_bwd(const float* g, const uint32_t* pass_bits, const float* x, int32_t batch, int32_t channels,
                               int32_t hw, const float* mean, const float* invstd, const float* gamma, int32_t training,
                               int32_t out_shuffle_groups, float* dx, float* dgamma, float* dbeta, float* dx_channel_sum,
                               void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(g && pass_bits && x && mean && invstd && gamma && dx && dgamma && dbeta && scratch, "NULL bn_sign_bwd pointer");
  MNB_REQUIRE(batch > 0 && channels > 0 && channels <= 8192 && hw > 0, "bad bn_sign_bwd shape");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  const int64_t n = (int64_t)batch * channels * hw;
  const int64_t per = (int64_t)batch * hw;
  const int splits = plane_splits(batch, per, channels);
  uint32_t* counters = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(scratch) + 16384);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 49152);
  const dim3 grid(channels, splits);
  const float inv_count = 1.f / (float)per;
  if (planes_vectorizable(n, hw, x, g, dx)) {
    bn_sign_bwd_reduce_kernel<true><<<grid, 256, 0, S(stream)>>>(g, pass_bits, x, batch, channels, hw, out_shuffle_groups, mean,
                                                                 invstd, dgamma, dbeta, counters, partial);
    if (training == 2) { MNB_LAUNCHED(1); return 0; }   // reduce pass only: the caller applies (mnb_bn_sign_bwd_pack)
    bn_sign_bwd_apply_kernel<true><<<grid, 256, 0, S(stream)>>>(g, pass_bits, x, batch, channels, hw, out_shuffle_groups,
                                                                inv_count, mean, invstd, gamma, dgamma, dbeta, training, dx,
                                                                dx_channel_sum, counters, partial);
  } else {
    bn_sign_bwd_reduce_kernel<false><<<grid, 256, 0, S(stream)>>>(g, pass_bits, x, batch, channels, hw, out_shuffle_groups, mean,
                                                                  invstd, dgamma, dbeta, counters, partial);
    if (training == 2) { MNB_LAUNCHED(1); return 0; }
    bn_sign_bwd_apply_kernel<false><<<grid, 256, 0, S(stream)>>>(g, pass_bits, x, batch, channels, hw, out_shuffle_groups,
                                                                 inv_count, mean, invstd, gamma, dgamma, dbeta, training, dx,
                                                                 dx_channel_sum, counters, partial);
  }
  MNB_LAUNCHED(2);
  return 0;
}

// ------------------------------------------------------------------ BatchNorm + sign + MaxPool2d(2, 2) in one pass
// The full-resolution +-1 tensor is never written: forward reads x once and writes the pooled signs (plus the STE
// pass bits of all inputs and the window argmax); backward routes the pooled gradient to the window winner, applies
// the STE mask and the batch-norm backward without materialising the un-pooled gradient.
// One thread owns two horizontally adjacent windows = two float4 of x (rows 2oh and 2oh + 1).  W % 8 == 0, H even.
struct PoolGeom { uint32_t channels, H, W4, OH, OW2, sg; };

__device__ __forceinline__ uint32_t first_max_of_signs(bool p0, bool p1, bool p2, bool p3) {
  // ATen's max_pool scan order (r0c0, r0c1, r1c0, r1c1), replace on strictly greater: the first +1, else element 0
  return p0 ? 0u : (p1 ? 1u : (p2 ? 2u : (p3 ? 3u : 0u)));
}

__global__ void __launch_bounds__(256) bn_sign_pool_fwd_kernel(const float4* __restrict__ x, uint32_t n_pairs, PoolGeom gm,
                                                               const float* __restrict__ mean, const float* __restrict__ invstd,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               float2* __restrict__ y, uchar2* __restrict__ arg,
                                                               uint8_t* __restrict__ bits8) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t n_up = (n_pairs + 31u) & ~31u;
  const uint32_t cpg = gm.channels / gm.sg;
  for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < n_up; o += stride) {
    uint32_t nib = 0, i0 = 0;
    const bool live = o < n_pairs;
    if (live) {
      const uint32_t j = o % gm.OW2, t = o / gm.OW2;
      const uint32_t oh = t % gm.OH, plane = t / gm.OH;
      const uint32_t b = plane / gm.channels, c = plane - b * gm.channels;
      i0 = (plane * gm.H + 2 * oh) * gm.W4 + j;
      const float mu = __ldg(mean + c), sc = __ldg(gamma + c) * __ldg(invstd + c), be = __ldg(beta + c);
      const float4 r0 = __ldg(x + i0), r1 = __ldg(x + i0 + gm.W4);
      const float v[8] = {fmaf(r0.x - mu, sc, be), fmaf(r0.y - mu, sc, be), fmaf(r0.z - mu, sc, be), fmaf(r0.w - mu, sc, be),
                          fmaf(r1.x - mu, sc, be), fmaf(r1.y - mu, sc, be), fmaf(r1.z - mu, sc, be), fmaf(r1.w - mu, sc, be)};
      bool pos[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) { pos[e] = !(v[e] < 0.f); nib |= (uint32_t)(fabsf(v[e]) < 1.f) << e; }
      const uint32_t a0 = first_max_of_signs(pos[0], pos[1], pos[4], pos[5]);
      const uint32_t a1 = first_max_of_signs(pos[2], pos[3], pos[6], pos[7]);
      const float m0 = (pos[0] | pos[1] | pos[4] | pos[5]) ? 1.f : -1.f, m1 = (pos[2] | pos[3] | pos[6] | pos[7]) ? 1.f : -1.f;
      const uint32_t oplane = b * gm.channels + shuffled_channel(c, gm.sg, cpg);
      y[(oplane * gm.OH + oh) * gm.OW2 + j] = make_float2(m0, m1);
      arg[o] = make_uchar2((unsigned char)a0, (unsigned char)a1);
    }
    // pass nibbles: bits 0-3 = row 2oh (float4 index i0), bits 4-7 = row 2oh+1 (i0 + W4); two lanes share a byte
    const uint32_t other = __shfl_xor_sync(0xffffffffu, nib, 1);
    if (live && (threadIdx.x & 1) == 0) {
      bits8[i0 >> 1] = (uint8_t)((nib & 15u) | ((other & 15u) << 4));
      bits8[(i0 + gm.W4) >> 1] = (uint8_t)((nib >> 4) | (other & 0xf0u));
    }
  }
}

// pass 1 of the backward: dbeta = sum gm, dgamma = sum gm * xhat with gm = pooled gradient at the window winner x pass bit
__global__ void __launch_bounds__(256) bn_sign_pool_bwd_reduce_kernel(const float2* __restrict__ g, const uchar2* __restrict__ arg,
                                                                      const uint8_t* __restrict__ bits8, const float* __restrict__ x,
                                                                      int batch, PoolGeom gm, const float* __restrict__ mean,
                                                                      const float* __restrict__ invstd, float* __restrict__ dgamma,
                                                                      float* __restrict__ dbeta, uint32_t* counters, double* partial) {
  __shared__ double red[32];
  __shared__ bool last;
  const uint32_t c = blockIdx.x, sp = blockIdx.y, nsp = gridDim.y;
  const uint32_t oc = shuffled_channel(c, gm.sg, gm.channels / gm.sg);
  const float mu = __ldg(mean + c), is = __ldg(invstd + c);
  const uint32_t b_lo = (uint32_t)((int64_t)batch * sp / nsp), b_hi = (uint32_t)((int64_t)batch * (sp + 1) / nsp);
  const uint32_t per_img = gm.OH * gm.OW2, total = (b_hi - b_lo) * per_img;
  float f1[2] = {0.f, 0.f}, f2[2] = {0.f, 0.f};
  for (uint32_t t0 = threadIdx.x; t0 < total; t0 += 2 * blockDim.x) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint32_t t = t0 + u * blockDim.x;
      if (t < total) {
        const uint32_t b = b_lo + t / per_img, rem = t % per_img;
        const uint32_t oh = rem / gm.OW2, j = rem - oh * gm.OW2;
        const uint32_t plane = b * gm.channels + c;
        const float2 gv = __ldg(g + ((b * gm.channels + oc) * gm.OH + oh) * gm.OW2 + j);
        const uchar2 a = arg[(plane * gm.OH + oh) * gm.OW2 + j];
        const uint32_t i0 = (plane * gm.H + 2 * oh) * gm.W4 + j;
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const uint32_t aw = w ? a.y : a.x;
          const uint32_t i4 = i0 + (aw >> 1) * gm.W4, col = 2u * w + (aw & 1u);
          const bool pass = (bits8[i4 >> 1] >> (4u * (i4 & 1u) + col)) & 1u;
          const float gmv = pass ? (w ? gv.y : gv.x) : 0.f;
          f1[u] += gmv;
          f2[u] += gmv * ((__ldg(x + 4u * i4 + col) - mu) * is);
        }
      }
    }
  }
  double s1 = mnb_block_reduce((double)f1[0] + (double)f1[1], MnbSum(), 0.0, red);
  double s2 = mnb_block_reduce((double)f2[0] + (double)f2[1], MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    partial[((int64_t)c * nsp + sp) * 2 + 0] = s1;
    partial[((int64_t)c * nsp + sp) * 2 + 1] = s2;
    __threadfence();
    last = (atomicAdd(counters + c, 1u) == nsp - 1);
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  s1 = 0.0; s2 = 0.0;
  for (uint32_t j = 0; j < nsp; ++j) { s1 += partial[((int64_t)c * nsp + j) * 2]; s2 += partial[((int64_t)c * nsp + j) * 2 + 1]; }
  dbeta[c] = (float)s1;
  dgamma[c] = (float)s2;
  counters[c] = 0;
}

// pass 2: dx over the full-resolution plane (+ its channel sums)
__global__ void __launch_bounds__(256) bn_sign_pool_bwd_apply_kernel(const float2* __restrict__ g, const uchar2* __restrict__ arg,
                                                                     const uint8_t* __restrict__ bits8, const float4* __restrict__ x,
                                                                     int batch, PoolGeom gm, float inv_count,
                                                                     const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                     const float* __restrict__ gamma, const float* __restrict__ dgamma,
                                                                     const float* __restrict__ dbeta, int training,
                                                                     float4* __restrict__ dx, float* __restrict__ dx_sum,
                                                                     uint32_t* counters, double* partial) {
  __shared__ double red[32];
  __shared__ bool last;
  const uint32_t c = blockIdx.x, sp = blockIdx.y, nsp = gridDim.y;
  const uint32_t oc = shuffled_channel(c, gm.sg, gm.channels / gm.sg);
  const float mu = __ldg(mean + c), is = __ldg(invstd + c), k = __ldg(gamma + c) * is;
  const float db = training ? __ldg(dbeta + c) * inv_count : 0.f, dg = training ? __ldg(dgamma + c) * inv_count : 0.f;
  const uint32_t b_lo = (uint32_t)((int64_t)batch * sp / nsp), b_hi = (uint32_t)((int64_t)batch * (sp + 1) / nsp);
  const uint32_t per_img = gm.OH * gm.OW2, total = (b_hi - b_lo) * per_img;
  float f = 0.f;
  for (uint32_t t = threadIdx.x; t < total; t += blockDim.x) {
    const uint32_t b = b_lo + t / per_img, rem = t % per_img;
    const uint32_t oh = rem / gm.OW2, j = rem - oh * gm.OW2;
    const uint32_t plane = b * gm.channels + c;
    const float2 gv = __ldg(g + ((b * gm.channels + oc) * gm.OH + oh) * gm.OW2 + j);
    const uchar2 a = arg[(plane * gm.OH + oh) * gm.OW2 + j];
    const uint32_t i0 = (plane * gm.H + 2 * oh) * gm.W4 + j, i1 = i0 + gm.W4;
    const uint32_t n0 = (bits8[i0 >> 1] >> (4u * (i0 & 1u))) & 15u, n1 = (bits8[i1 >> 1] >> (4u * (i1 & 1u))) & 15u;
    // masked gradient of the eight inputs: the pooled gradient at each window's winner, if its pass bit is set
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    {
      const uint32_t e0 = (a.x >> 1) * 4u + (a.x & 1u), e1 = (a.y >> 1) * 4u + 2u + (a.y & 1u);
      const uint32_t nib = n0 | (n1 << 4);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if ((uint32_t)e == e0 && ((nib >> e) & 1u)) v[e] = gv.x;
        if ((uint32_t)e == e1 && ((nib >> e) & 1u)) v[e] = gv.y;
      }
    }
    if (training) {
      const float4 r0 = __ldg(x + i0), r1 = __ldg(x + i1);
      const float xs[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = bn_bwd_centre(v[e], db, (xs[e] - mu) * is, dg);
    }
    const float4 o0 = make_float4(k * v[0], k * v[1], k * v[2], k * v[3]), o1 = make_float4(k * v[4], k * v[5], k * v[6], k * v[7]);
    dx[i0] = o0;
    dx[i1] = o1;
    f += ((o0.x + o0.y) + (o0.z + o0.w)) + ((o1.x + o1.y) + (o1.z + o1.w));
  }
  if (!dx_sum) return;
  double s = mnb_block_reduce((double)f, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    partial[((int64_t)c * nsp + sp) * 2] = s;
    __threadfence();
    last = (atomicAdd(counters + c, 1u) == nsp - 1);
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  s = 0.0;
  for (uint32_t j = 0; j < nsp; ++j) s += partial[((int64_t)c * nsp + j) * 2];
  dx_sum[c] = (float)s;
  counters[c] = 0;
}

static int pool_geom(int batch, int channels, int H, int W, int sg, const void* a, const void* b, const void* c, PoolGeom& gm) {
  MNB_REQUIRE(batch > 0 && channels > 0 && channels <= 8192 && H > 0 && W > 0, "bad bn_sign_pool shape");
  MNB_REQUIRE(sg >= 1 && channels % sg == 0, "shuffle groups %d do not divide %d channels", sg, channels);
  if ((H & 1) || (W & 7) || (int64_t)batch * channels * H * W >= (1ll << 31) ||
      (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "bn_sign_pool needs even H, W %% 8 == 0, < 2^31 elements, 16-byte aligned tensors");
  gm = PoolGeom{(uint32_t)channels, (uint32_t)H, (uint32_t)(W / 4), (uint32_t)(H / 2), (uint32_t)(W / 4), (uint32_t)sg};
  return 0;
}

extern "C" int mnb_bn_sign_pool_fwd(const float* x, int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean,
                                    const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups,
                                    float* y, uint32_t* pass_bits, uint8_t* argmax, mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && invstd && gamma && beta && y && pass_bits && argmax, "NULL bn_sign_pool_fwd pointer");
  PoolGeom gm;
  if (int e = pool_geom(batch, channels, H, W, out_shuffle_groups, x, y, nullptr, gm)) return e;
  const uint32_t n_pairs = (uint32_t)((int64_t)batch * channels * gm.OH * gm.OW2);
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n_pairs, 256), MNB_NUM_SMS * 16);
  bn_sign_pool_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), n_pairs, gm, mean, invstd, gamma, beta,
                                                         reinterpret_cast<float2*>(y), reinterpret_cast<uchar2*>(argmax),
                                                         reinterpret_cast<uint8_t*>(pass_bits));
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_sign_pool_bwd(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const float* x, int32_t batch,
                                    int32_t channels, int32_t H, int32_t W, const float* mean, const float* invstd,
                                    const float* gamma, int32_t training, int32_t out_shuffle_groups, float* dx, float* dgamma,
                                    float* dbeta, float* dx_channel_sum, void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(g && pass_bits && argmax && x && mean && invstd && gamma && dx && dgamma && dbeta && scratch,
              "NULL bn_sign_pool_bwd pointer");
  PoolGeom gm;
  if (int e = pool_geom(batch, channels, H, W, out_shuffle_groups, x, dx, nullptr, gm)) return e;
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(g) & 7) == 0, "pooled gradient must be 8-byte aligned");
  const int64_t per = (int64_t)batch * H * W;
  const int splits = plane_splits(batch, per, channels);
  uint32_t* counters = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(scratch) + 16384);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 49152);
  const dim3 grid(channels, splits);
  const uint8_t* bits8 = reinterpret_cast<const uint8_t*>(pass_bits);
  bn_sign_pool_bwd_reduce_kernel<<<grid, 256, 0, S(stream)>>>(reinterpret_cast<const float2*>(g),
                                                              reinterpret_cast<const uchar2*>(argmax), bits8, x, batch, gm, mean,
                                                              invstd, dgamma, dbeta, counters, partial);
  if (training == 2) { MNB_LAUNCHED(1); return 0; }   // reduce pass only: the caller applies (mnb_bn_sign_pool_bwd_pack)
  bn_sign_pool_bwd_apply_kernel<<<grid, 256, 0, S(stream)>>>(reinterpret_cast<const float2*>(g),
                                                             reinterpret_cast<const uchar2*>(argmax), bits8,
                                                             reinterpret_cast<const float4*>(x), batch, gm, 1.f / (float)per, mean,
                                                             invstd, gamma, dgamma, dbeta, training,
                                                             reinterpret_cast<float4*>(dx), dx_channel_sum, counters, partial);
  MNB_LAUNCHED(2);
  return 0;
}

// ------------------------------------------------------------------ MaxPool2d with a one-byte window index
// Tie rule of ATen's max_pool_forward_nchw: scan the window row-major, replace on (v > best) || isnan(v): the first
// maximum wins.  The stored byte is r * k + s of the winner (window coordinates, counted from the unclipped corner).
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const float* __restrict__ x, int64_t n_out, int channels, int H, int W,
                                                          int OH, int OW, int k, int st, int pad, int sg,
                                                          float* __restrict__ y, uint8_t* __restrict__ arg) {
  const uint32_t cpg = (uint32_t)(channels / sg);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += stride) {
    const int ow = (int)(o % OW);
    const int64_t t = o / OW;
    const int oh = (int)(t % OH);
    const int64_t plane = t / OH;
    const int c = (int)(plane % channels);
    const float* src = x + plane * H * W;
    const int h0 = oh * st - pad, w0 = ow * st - pad;
    float best = -INFINITY;
    int bi = -1;
    for (int r = 0; r < k; ++r) {
      const int h = h0 + r;
      if (h < 0 || h >= H) continue;
      for (int s = 0; s < k; ++s) {
        const int w = w0 + s;
        if (w < 0 || w >= W) continue;
        const float v = __ldg(src + h * W + w);
        if (bi < 0 || v > best || isnan(v)) { best = v; bi = r * k + s; }
      }
    }
    const int64_t oplane = plane - c + shuffled_channel((uint32_t)c, (uint32_t)sg, cpg);
    y[(oplane * OH + oh) * OW + ow] = best;
    arg[o] = (uint8_t)bi;
  }
}

// k = stride = 2, pad 0, even W: one thread makes two adjacent outputs from two float4 rows
__global__ void __launch_bounds__(256) maxpool2x2_fwd_kernel(const float4* __restrict__ x, uint32_t n_pairs, uint32_t channels,
                                                             uint32_t OH, uint32_t OW2, uint32_t W4, uint32_t H, uint32_t sg,
                                                             float2* __restrict__ y, uchar2* __restrict__ arg) {
  const uint32_t cpg = channels / sg;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < n_pairs; o += stride) {
    const uint32_t j = o % OW2, t = o / OW2;
    const uint32_t oh = t % OH, plane = t / OH;
    const uint32_t b = plane / channels, c = plane - b * channels;
    const float4 r0 = __ldg(x + (plane * H + 2 * oh) * W4 + j), r1 = __ldg(x + (plane * H + 2 * oh + 1) * W4 + j);
    float m0 = r0.x; uint32_t a0 = 0;
    if (r0.y > m0 || isnan(r0.y)) { m0 = r0.y; a0 = 1; }
    if (r1.x > m0 || isnan(r1.x)) { m0 = r1.x; a0 = 2; }
    if (r1.y > m0 || isnan(r1.y)) { m0 = r1.y; a0 = 3; }
    float m1 = r0.z; uint32_t a1 = 0;
    if (r0.w > m1 || isnan(r0.w)) { m1 = r0.w; a1 = 1; }
    if (r1.z > m1 || isnan(r1.z)) { m1 = r1.z; a1 = 2; }
    if (r1.w > m1 || isnan(r1.w)) { m1 = r1.w; a1 = 3; }
    const uint32_t oplane = b * channels + shuffled_channel(c, sg, cpg);
    y[(oplane * OH + oh) * OW2 + j] = make_float2(m0, m1);
    arg[o] = make_uchar2((unsigned char)a0, (unsigned char)a1);
  }
}

// gather form (one thread per input element), windows visited in (oh, ow) order like ATen's max_pool_backward_nchw
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const float* __restrict__ g, const uint8_t* __restrict__ arg,
                                                          int64_t n_in, int channels, int H, int W, int OH, int OW, int k, int st,
                                                          int pad, int sg, float* __restrict__ dx) {
  const uint32_t cpg = (uint32_t)(channels / sg);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += stride) {
    const int w = (int)(i % W);
    const int64_t t = i / W;
    const int h = (int)(t % H);
    const int64_t plane = t / H;
    const int c = (int)(plane % channels);
    const int64_t oplane = plane - c + shuffled_channel((uint32_t)c, (uint32_t)sg, cpg);
    const int oh_lo = (h + pad < k) ? 0 : (h + pad - k) / st + 1, oh_hi = min((h + pad) / st + 1, OH);
    const int ow_lo = (w + pad < k) ? 0 : (w + pad - k) / st + 1, ow_hi = min((w + pad) / st + 1, OW);
    float acc = 0.f;
    for (int oh = oh_lo; oh < oh_hi; ++oh)
      for (int ow = ow_lo; ow < ow_hi; ++ow) {
        const int r = h - (oh * st - pad), s = w - (ow * st - pad);
        if ((int)arg[(plane * OH + oh) * OW + ow] == r * k + s) acc += __ldg(g + (oplane * OH + oh) * OW + ow);
      }
    dx[i] = acc;
  }
}

__global__ void __launch_bounds__(256) maxpool2x2_bwd_kernel(const float2* __restrict__ g, const uchar2* __restrict__ arg,
                                                             uint32_t n_pairs, uint32_t channels, uint32_t OH, uint32_t OW2,
                                                             uint32_t W4, uint32_t H, uint32_t sg, float4* __restrict__ dx) {
  const uint32_t cpg = channels / sg;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < n_pairs; o += stride) {
    const uint32_t j = o % OW2, t = o / OW2;
    const uint32_t oh = t % OH, plane = t / OH;
    const uint32_t b = plane / channels, c = plane - b * channels;
    const uint32_t oplane = b * channels + shuffled_channel(c, sg, cpg);
    const float2 gv = __ldg(g + (oplane * OH + oh) * OW2 + j);
    const uchar2 a = arg[o];
    dx[(plane * H + 2 * oh) * W4 + j] = make_float4(a.x == 0 ? gv.x : 0.f, a.x == 1 ? gv.x : 0.f, a.y == 0 ? gv.y : 0.f,
                                                    a.y == 1 ? gv.y : 0.f);
    dx[(plane * H + 2 * oh + 1) * W4 + j] = make_float4(a.x == 2 ? gv.x : 0.f, a.x == 3 ? gv.x : 0.f, a.y == 2 ? gv.y : 0.f,
                                                        a.y == 3 ? gv.y : 0.f);
  }
}

static int pool_out(int in, int k, int st, int pad) { return (in + 2 * pad - k) / st + 1; }
static bool pool_is_2x2(int H, int W, int k, int st, int pad, int64_t n_in, const void* a, const void* b) {
  return k == 2 && st == 2 && pad == 0 && (W & 3) == 0 && (H & 1) == 0 && n_in < (1ll << 31) &&
         (((uintptr_t)a | (uintptr_t)b) & 15) == 0;
}

extern "C" int mnb_maxpool2d_fwd(const float* x, int32_t batch, int32_t channels, int32_t H, int32_t W, int32_t kernel,
                                 int32_t stride, int32_t pad, int32_t out_shuffle_groups, float* y, uint8_t* argmax,
                                 mnb_stream_t stream) {
  MNB_REQUIRE(x && y && argmax && batch > 0 && channels > 0 && H > 0 && W > 0, "bad maxpool2d_fwd arguments");
  MNB_REQUIRE(kernel >= 1 && kernel <= 15 && stride >= 1 && pad >= 0 && 2 * pad <= kernel, "maxpool kernel %d stride %d pad %d",
              kernel, stride, pad);
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  const int OH = pool_out(H, kernel, stride, pad), OW = pool_out(W, kernel, stride, pad);
  MNB_REQUIRE(OH > 0 && OW > 0, "maxpool output is empty");
  const int64_t planes = (int64_t)batch * channels, n_out = planes * OH * OW;
  if (pool_is_2x2(H, W, kernel, stride, pad, planes * H * W, x, y)) {
    const uint32_t n_pairs = (uint32_t)(n_out / 2);
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n_pairs, 256), MNB_NUM_SMS * 16);
    maxpool2x2_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), n_pairs, (uint32_t)channels,
                                                         (uint32_t)OH, (uint32_t)(OW / 2), (uint32_t)(W / 4), (uint32_t)H,
                                                         (uint32_t)out_shuffle_groups, reinterpret_cast<float2*>(y),
                                                         reinterpret_cast<uchar2*>(argmax));
  } else {
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n_out, 256), MNB_NUM_SMS * 16);
    maxpool_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(x, n_out, channels, H, W, OH, OW, kernel, stride, pad, out_shuffle_groups,
                                                      y, argmax);
  }
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_maxpool2d_bwd(const float* g, const uint8_t* argmax, int32_t batch, int32_t channels, int32_t H, int32_t W,
                                 int32_t kernel, int32_t stride, int32_t pad, int32_t out_shuffle_groups, float* dx,
                                 mnb_stream_t stream) {
  MNB_REQUIRE(g && dx && argmax && batch > 0 && channels > 0 && H > 0 && W > 0, "bad maxpool2d_bwd arguments");
  MNB_REQUIRE(kernel >= 1 && kernel <= 15 && stride >= 1 && pad >= 0 && 2 * pad <= kernel, "maxpool kernel %d stride %d pad %d",
              kernel, stride, pad);
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  const int OH = pool_out(H, kernel, stride, pad), OW = pool_out(W, kernel, stride, pad);
  MNB_REQUIRE(OH > 0 && OW > 0, "maxpool output is empty");
  const int64_t planes = (int64_t)batch * channels, n_in = planes * H * W;
  if (pool_is_2x2(H, W, kernel, stride, pad, n_in, g, dx) && (((uintptr_t)g) & 7) == 0) {
    const uint32_t n_pairs = (uint32_t)(planes * OH * OW / 2);
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n_pairs, 256), MNB_NUM_SMS * 16);
    maxpool2x2_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(reinterpret_cast<const float2*>(g), reinterpret_cast<const uchar2*>(argmax),
                                                         n_pairs, (uint32_t)channels, (uint32_t)OH, (uint32_t)(OW / 2),
                                                         (uint32_t)(W / 4), (uint32_t)H, (uint32_t)out_shuffle_groups,
                                                         reinterpret_cast<float4*>(dx));
  } else {
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n_in, 256), MNB_NUM_SMS * 16);
    maxpool_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(g, argmax, n_in, channels, H, W, OH, OW, kernel, stride, pad,
                                                      out_shuffle_groups, dx);
  }
  MNB_LAUNCHED(1);
  return 0;
}
