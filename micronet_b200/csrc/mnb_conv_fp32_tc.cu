// fp32 convolution with few input channels (the un-quantized FIRST layer of every QAT model: 3 -> 192/256,
// 5x5 or 3x3; nin_gc.py:82, nin.py, resnet.py) on Hopper tensor cores (wgmma): forward and weight gradient.
//
// C*R*S (75 for 3x5x5) is far too small a reduction for the per-tap implicit GEMM of mnb_conv_tc_fwd.cu
// (one MMA K-step would carry 3 real channels out of 16), so this layer uses a real im2col operand, built in
// shared memory from a zero-padded input patch:
//
//   forward : y[b, n, pos]  = bias[n] + sum_kk  Xcol[pos, kk] * w[n, kk]      M = 128 positions, N = Cout, K = kk
//   wgrad   : dw[n, kk]     = sum_{b, pos}      dy[b, n, pos] * Xcol[pos, kk] M = 128 channels,  N = kk,   K = positions
//
// fp32 accuracy on bf16 tensor cores: every fp32 value is split exactly into three bf16 pieces (hi + mid + lo) and
// the six products down to 2^-16 relative weight (hh, hm, mh, hl, lh, mm) are accumulated in fp32; the dropped
// pieces are <= 2^-24 relative: the error is that of an fp32 convolution with a different summation order.
//
// Both kernels are persistent (one CTA per SM), HBM-bound by the one large tensor they stream (y written once,
// dy read once): forward 128 positions x Cout x 4 B per tile, weight gradient 32 positions x Cout x 4 B per step.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

namespace tcfp32 {

constexpr int NTHREADS = 512;
constexpr int kMaxDynSmem = 227 * 1024 - 2560;
constexpr int SUB = 32;  // positions per weight-gradient step

struct Params {
  int B, C, K, H, W, R, pad;
  int KR, KP;         // C*R*R and its multiple-of-16 padding
  int NP;             // forward: Cout padded to 16 (MMA N); wgrad: Cout padded to 128 (MMA M halves)
  int TH, PH, PW;     // tile = TH full rows (TH * W = 128); patch = C x PH x PW floats (zero padded)
  int tiles_per_img, n_tiles;
  int nbuf_a;
  int off_b, off_a, off_patch, off_tab, off_sum, off_stg, sum_bytes, a_term_bytes, a_buf_bytes, b_term_bytes, patch_bytes;
  const float* x; const float* w; const float* bias; float* y;
  const float* dy; float* partial;
  int* err;
};

struct alignas(16) Shared {
  uint64_t a_full[2], a_empty[2];
  uint32_t abort;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void split3_pair(float a, float b, uint32_t& hp, uint32_t& mp, uint32_t& lp) {
  hp = pack_bf16x2(a, b);
  const float ra = a - __uint_as_float(hp << 16), rb = b - __uint_as_float(hp & 0xffff0000u);
  mp = pack_bf16x2(ra, rb);
  const float la = ra - __uint_as_float(mp << 16), lb = rb - __uint_as_float(mp & 0xffff0000u);
  lp = pack_bf16x2(la, lb);
}
// eight fp32 values -> one 16-byte row of each of the three operand planes
__device__ __forceinline__ void store_split8(const float (&v)[8], uint8_t* dst, int term_bytes) {
  uint32_t hp[4], mp[4], lp[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split3_pair(v[2 * j], v[2 * j + 1], hp[j], mp[j], lp[j]);
  *reinterpret_cast<uint4*>(dst) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
  *reinterpret_cast<uint4*>(dst + term_bytes) = make_uint4(mp[0], mp[1], mp[2], mp[3]);
  *reinterpret_cast<uint4*>(dst + 2 * term_bytes) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
}
__device__ __forceinline__ void conv_bar_sync(int nthreads) {  // named barrier 1: converter warps only
  asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
}
__device__ __forceinline__ void mma_bar_sync() {  // named barrier 2: the MMA warpgroup (warps 4..7)
  asm volatile("bar.sync 2, 128;" ::: "memory");
}

// The six (A piece, B piece) products kept, SMALLEST FIRST: the 2^-16 and 2^-8 products are added while the running
// fp32 accumulator is still tiny, so whatever rounding the tensor core applies to it acts on the small terms at their
// own magnitude and only the hi x hi MMAs run at full magnitude.
__device__ __constant__ int kProdA[6] = {1, 2, 0, 1, 0, 0};
__device__ __constant__ int kProdB[6] = {1, 0, 2, 0, 1, 0};

// zero-padded input patch of one tile: patch[c][pr][pc] = x[b, c, h0 - pad + pr, pc - pad].  It is fetched one tile
// ahead: the first PF elements of every converter thread wait in registers while the current tile is converted
// (patch_fetch), and are written to the other patch buffer afterwards (patch_commit, which also moves the rare
// remainder of a patch larger than PF * nconv directly).
constexpr int PF = 4;
__device__ __forceinline__ float patch_element(const Params& p, int i, int b, int h0) {
  const int pc = i % p.PW, t = i / p.PW;
  const int pr = t % p.PH, c = t / p.PH;
  const int h = h0 - p.pad + pr, w = pc - p.pad;
  return (h >= 0 && h < p.H && w >= 0 && w < p.W) ? __ldg(p.x + (((int64_t)b * p.C + c) * p.H + h) * p.W + w) : 0.f;
}
template <int NPF = PF>
__device__ __forceinline__ void patch_fetch(const Params& p, int tile, int ct, int nconv, float (&v)[NPF]) {
  const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
  const int n = p.C * p.PH * p.PW;
#pragma unroll
  for (int k = 0; k < NPF; ++k) {
    const int i = ct + k * nconv;
    v[k] = i < n ? patch_element(p, i, b, h0) : 0.f;
  }
}
template <int NPF = PF>
__device__ __forceinline__ void patch_commit(const Params& p, float* patch, int tile, int ct, int nconv, const float (&v)[NPF]) {
  const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
  const int n = p.C * p.PH * p.PW;
#pragma unroll
  for (int k = 0; k < NPF; ++k) {
    const int i = ct + k * nconv;
    if (i < n) patch[i] = v[k];
  }
  for (int i = ct + NPF * nconv; i < n; i += nconv) patch[i] = patch_element(p, i, b, h0);
}

// ------------------------------------------------------------------------------------------------ forward
// warps: 4..7 = MMA warpgroup (wgmma + epilogue), the other 11 except warp 0 = im2col converters
constexpr int FWD_NCONV = NTHREADS - 32 - 128;

__global__ void __launch_bounds__(NTHREADS, 1) fwd_kernel(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Shared sh;
  __shared__ __align__(16) float epi_bias[256];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* bop = smem + p.off_b;
  uint8_t* aop = smem + p.off_a;
  int* tab = reinterpret_cast<int*>(smem + p.off_tab);
  const int kchunks = p.KP / 8;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&sh.a_full[i], FWD_NCONV / 32); tc::mbar_init(&sh.a_empty[i], 4);
    }
    sh.abort = 0;
    tc::fence_barrier_init();
  }
  for (int n = tid; n < 256; n += NTHREADS) epi_bias[n] = (p.bias && n < p.K) ? __ldg(p.bias + n) : 0.f;
  // resident B operand: w[n][kk] as K-major core matrices [piece][kk / 8][n][8], zero beyond Cout / KR
  for (int i = tid; i < kchunks * p.NP; i += NTHREADS) {
    const int j = i / p.NP, n = i - j * p.NP;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int kk = j * 8 + e;
      v[e] = (n < p.K && kk < p.KR) ? __ldg(p.w + (int64_t)n * p.KR + kk) : 0.f;
    }
    store_split8(v, bop + (size_t)i * 16, p.b_term_bytes);
  }
  for (int kk = tid; kk < p.KP; kk += NTHREADS) {
    int off = -1;
    if (kk < p.KR) {
      const int s = kk % p.R, t = kk / p.R;
      const int r = t % p.R, c = t / p.R;
      off = (c * p.PH + r) * p.PW + s;
    }
    tab[kk] = off;
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp >= 4 && warp < 8) {
    // ================================================================= MMA warpgroup: wgmma -> + bias -> y (NCHW)
    // 32 output channels at a time: both 64-row halves of the tile in registers (m64n32), through a 128 x 32 staging tile
    // so that thread m stores position m of every channel (coalesced NCHW rows)
    const int m = (warp - 4) * 32 + lane;
    float* stage = reinterpret_cast<float*>(smem + p.off_stg);
    const int64_t plane = (int64_t)p.H * p.W;
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(aop), 128u * 16u, 128u);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(bop), (uint32_t)p.NP * 16u, 128u);
    const uint32_t a_term16 = (uint32_t)p.a_term_bytes >> 4, b_term16 = (uint32_t)p.b_term_bytes >> 4;
    const uint32_t a_buf16 = (uint32_t)p.a_buf_bytes >> 4;
    const uint32_t a_step16 = 2u * 128u, b_step16 = 2u * (uint32_t)p.NP;   // one K16 step = two 8-wide chunks
    uint32_t t = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++t) {
      const uint32_t ab = p.nbuf_a == 2 ? (t & 1u) : 0u, aph = p.nbuf_a == 2 ? ((t >> 1) & 1u) : (t & 1u);
      tc::mbar_wait_soft(&sh.a_full[ab], aph, p.err, 502, &sh.abort);
      const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
      float* dst = p.y + (int64_t)b * p.K * plane + (int64_t)h0 * p.W + m;
      for (int n0 = 0; n0 < p.NP; n0 += 32) {
        float acc0[16], acc1[16];
        tc::zero_acc(acc0); tc::zero_acc(acc1);
        tc::wg_fence();
        tc::fence_acc(acc0); tc::fence_acc(acc1);
        for (int q = 0; q < 6; ++q) {
          const uint64_t aq = a_desc0 + (uint64_t)(ab * a_buf16 + (uint32_t)kProdA[q] * a_term16);
          const uint64_t bq = b_desc0 + (uint64_t)((uint32_t)kProdB[q] * b_term16 + (uint32_t)n0);
          // kept rolled: unrolled, ptxas puts a warpgroup.arrive in a divergent path and waits after every wgmma (C7520)
#pragma unroll 1
          for (int ks = 0; ks < p.KP / 16; ++ks) {
            const uint64_t ad = aq + (uint64_t)((uint32_t)ks * a_step16), bd = bq + (uint64_t)((uint32_t)ks * b_step16);
            tc::Mma<32>::bf16<0, 0>(acc0, ad, bd, 1);
            tc::Mma<32>::bf16<0, 0>(acc1, ad + 64u, bd, 1);   // rows 64..127: 64 core-matrix rows further
          }
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::fence_acc(acc0); tc::fence_acc(acc1);
        if (n0 + 32 >= p.NP) {   // the tile's last MMAs retired: its operand buffer is free
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(&sh.a_empty[ab]);
        }
        mma_bar_sync();          // every thread is done reading the previous staging tile
        tc::frag_to_smem(acc0, stage, tc::kStageLd, 0);
        tc::frag_to_smem(acc1, stage, tc::kStageLd, 64);
        mma_bar_sync();
        // bias as vector loads from shared memory up front so that the store loop is a pure FADD + STG stream (a
        // per-element bias load serialises against the stores)
        float bs[32];
#pragma unroll
        for (int v = 0; v < 8; ++v) {
          const float4 c4 = *reinterpret_cast<const float4*>(&epi_bias[n0 + 4 * v]);
          bs[4 * v] = c4.x; bs[4 * v + 1] = c4.y; bs[4 * v + 2] = c4.z; bs[4 * v + 3] = c4.w;
        }
        float* op = dst + (int64_t)n0 * plane;
#pragma unroll
        for (int j = 0; j < 32; ++j, op += plane)
          if (n0 + j < p.K) *op = stage[j * tc::kStageLd + m] + bs[j];
      }
    }
  } else {
    // ================================================================= converters: patch -> im2col A operand
    if (warp == 0) goto done;
    const int ct = warp < 4 ? tid - 32 : tid - 32 - 128;   // 0 .. FWD_NCONV-1
    float* patch0 = reinterpret_cast<float*>(smem + p.off_patch);
    const int items = 128 * kchunks;
    const int patch_floats = p.patch_bytes / 4;
    float pre[PF];
    if ((int)blockIdx.x < p.n_tiles) {
      patch_fetch(p, blockIdx.x, ct, FWD_NCONV, pre);
      patch_commit(p, patch0, blockIdx.x, ct, FWD_NCONV, pre);
    }
    uint32_t t = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++t) {
      const float* patch = patch0 + (size_t)(t & 1u) * patch_floats;
      conv_bar_sync(FWD_NCONV);   // every converter committed its part of this tile's patch
      const int next = tile + (int)gridDim.x;
      if (next < p.n_tiles) patch_fetch(p, next, ct, FWD_NCONV, pre);
      const uint32_t ab = p.nbuf_a == 2 ? (t & 1u) : 0u, aph = p.nbuf_a == 2 ? ((t >> 1) & 1u) : (t & 1u);
      if (!tc::mbar_wait(&sh.a_empty[ab], aph ^ 1u, p.err, 504)) break;
      uint8_t* abuf = aop + (size_t)ab * p.a_buf_bytes;
      for (int i = ct; i < items; i += FWD_NCONV) {
        const int j = i >> 7, m = i & 127;
        const int base = (m / p.W) * p.PW + (m % p.W);
        int off[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) off[e] = tab[j * 8 + e];
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = off[e] >= 0 ? patch[off[e] + base] : 0.f;
        store_split8(v, abuf + (size_t)i * 16, p.a_term_bytes);
      }
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.a_full[ab]);
      if (next < p.n_tiles) patch_commit(p, patch0 + (size_t)((t + 1) & 1u) * patch_floats, next, ct, FWD_NCONV, pre);
    }
  }
done:
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ weight gradient
// warps: 4..7 = MMA warpgroup, the other 11 except warp 0 = converters (dy split + im2col of x).
// A register accumulator only ever holds ONE step (12 MMAs per column set): the MMA warpgroup adds it into an fp32
// running sum in shared memory with round-to-nearest adds.  Short accumulation chains keep the tensor core's
// accumulator rounding (see kProdA) at the size of one step's terms.
constexpr int WG_NCONV = NTHREADS - 32 - 128;

__global__ void __launch_bounds__(NTHREADS, 1) wgrad_kernel(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* bop = smem + p.off_b;   // Xcol^T : [buf][piece][pos / 8][kk][8 pos]
  uint8_t* aop = smem + p.off_a;   // dy     : [buf][piece][pos / 8][channel][8 pos]
  int* tab = reinterpret_cast<int*>(smem + p.off_tab);
  const int halves = p.NP / 128;
  const int nsub = 128 / SUB;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&sh.a_full[i], WG_NCONV / 32); tc::mbar_init(&sh.a_empty[i], 4);
    }
    sh.abort = 0;
    tc::fence_barrier_init();
  }
  // operand buffers start as zeros (channel rows >= Cout and im2col rows >= KR are never written), and so does the
  // running sum that follows them
  for (int i = tid; i < (2 * (p.a_buf_bytes + 3 * p.b_term_bytes) + p.sum_bytes) / 16; i += NTHREADS)
    reinterpret_cast<uint4*>(smem + p.off_b)[i] = make_uint4(0, 0, 0, 0);
  for (int kk = tid; kk < p.KP; kk += NTHREADS) {
    int off = -1;
    if (kk < p.KR) {
      const int s = kk % p.R, t = kk / p.R;
      const int r = t % p.R, c = t / p.R;
      off = (c * p.PH + r) * p.PW + s;
    }
    tab[kk] = off;
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const int b_buf_bytes = 3 * p.b_term_bytes;

  if (warp >= 4 && warp < 8) {
    // ================================================================= MMA warpgroup: wgmma -> fp32 running sum -> partial dw
    // per step and 128-channel half: 32 im2col columns at a time, both 64-row halves in registers (m64n32), added into
    // the running sum straight from the fragment (every (channel, column) element belongs to exactly one thread)
    const int m = (warp - 4) * 32 + lane, wq = warp - 4;
    float* sum = reinterpret_cast<float*>(smem + p.off_sum);   // [half][kk][128 channels]
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(aop), (uint32_t)p.NP * 16u, 128u);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(bop), (uint32_t)p.KP * 16u, 128u);
    const uint32_t a_term16 = (uint32_t)p.a_term_bytes >> 4, b_term16 = (uint32_t)p.b_term_bytes >> 4;
    const uint32_t a_buf16 = (uint32_t)p.a_buf_bytes >> 4, b_buf16 = (uint32_t)b_buf_bytes >> 4;
    const uint32_t a_step16 = 2u * (uint32_t)p.NP, b_step16 = 2u * (uint32_t)p.KP;
    const int fr = 16 * wq + (lane >> 2), fc = 2 * (lane & 3);   // fragment row / column of this thread
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
      for (int sub = 0; sub < nsub; ++sub, ++it) {
        const uint32_t ob = it & 1u, oph = (it >> 1) & 1u;
        tc::mbar_wait_soft(&sh.a_full[ob], oph, p.err, 511, &sh.abort);
        for (int hf = 0; hf < halves; ++hf) {
          for (int k0 = 0; k0 < p.KP; k0 += 32) {
            float acc0[16], acc1[16];
            tc::zero_acc(acc0); tc::zero_acc(acc1);
            tc::wg_fence();
            tc::fence_acc(acc0); tc::fence_acc(acc1);
            for (int q = 0; q < 6; ++q) {
              const uint64_t aq = a_desc0 + (uint64_t)(ob * a_buf16 + (uint32_t)kProdA[q] * a_term16 + (uint32_t)hf * 128u);
              const uint64_t bq = b_desc0 + (uint64_t)(ob * b_buf16 + (uint32_t)kProdB[q] * b_term16 + (uint32_t)k0);
#pragma unroll
              for (int ks = 0; ks < SUB / 16; ++ks) {
                const uint64_t ad = aq + (uint64_t)((uint32_t)ks * a_step16), bd = bq + (uint64_t)((uint32_t)ks * b_step16);
                tc::Mma<32>::bf16<0, 0>(acc0, ad, bd, 1);
                tc::Mma<32>::bf16<0, 0>(acc1, ad + 64u, bd, 1);
              }
            }
            tc::wg_commit();
            tc::wg_wait<0>();
            tc::fence_acc(acc0); tc::fence_acc(acc1);
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int col = k0 + 8 * j + fc + (e & 1), row = fr + 8 * (e >> 1);
                if (col < p.KP) {
                  float* s0 = sum + ((hf * p.KP) + col) * 128 + row;
                  s0[0] = __fadd_rn(s0[0], acc0[4 * j + e]);
                  s0[64] = __fadd_rn(s0[64], acc1[4 * j + e]);
                }
              }
          }
        }
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&sh.a_empty[ob]);
      }
    }
    mma_bar_sync();   // running sums complete (written by other threads of the warpgroup)
    float* mine = p.partial + (int64_t)blockIdx.x * p.K * p.KR;
    for (int hf = 0; hf < halves; ++hf) {
      const int n = hf * 128 + m;
      if (n < p.K)
        for (int kk = 0; kk < p.KR; ++kk) mine[(int64_t)n * p.KR + kk] = sum[((hf * p.KP) + kk) * 128 + m];
    }
  } else if (warp != 0) {
    // ================================================================= converters
    const int ct = warp < 4 ? tid - 32 : tid - 32 - 128;
    float* patch0 = reinterpret_cast<float*>(smem + p.off_patch);
    const int64_t plane = (int64_t)p.H * p.W;
    const int d_items = p.K * (SUB / 8), x_items = p.KR * (SUB / 8);
    const int patch_floats = p.patch_bytes / 4;
    // dy is fetched one step (32 positions) ahead into registers: up to DMAX x 32 bytes per thread in flight while the
    // previous step is split and stored
    constexpr int DMAX = 3;
    float4 dpre[DMAX][2];
    auto fetch_dy = [&](int tile, int sub) {
      const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
      const float* dy_tile = p.dy + (int64_t)b * p.K * plane + (int64_t)h0 * p.W + sub * SUB;
#pragma unroll
      for (int k = 0; k < DMAX; ++k) {
        const int i = ct + k * WG_NCONV;
        if (i < d_items) {
          const int n = i / (SUB / 8), j = i - n * (SUB / 8);
          const float4* src = reinterpret_cast<const float4*>(dy_tile + (int64_t)n * plane + j * 8);
          dpre[k][0] = __ldg(src); dpre[k][1] = __ldg(src + 1);
        }
      }
    };
    float pre[PF];
    if ((int)blockIdx.x < p.n_tiles) {
      patch_fetch(p, blockIdx.x, ct, WG_NCONV, pre);
      patch_commit(p, patch0, blockIdx.x, ct, WG_NCONV, pre);
      fetch_dy(blockIdx.x, 0);
    }
    uint32_t it = 0, t = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++t) {
      const float* patch = patch0 + (size_t)(t & 1u) * patch_floats;
      conv_bar_sync(WG_NCONV);
      const int next = tile + (int)gridDim.x;
      if (next < p.n_tiles) patch_fetch(p, next, ct, WG_NCONV, pre);
      for (int sub = 0; sub < nsub; ++sub, ++it) {
        const uint32_t ob = it & 1u, oph = (it >> 1) & 1u;
        float4 dcur[DMAX][2];
#pragma unroll
        for (int k = 0; k < DMAX; ++k) { dcur[k][0] = dpre[k][0]; dcur[k][1] = dpre[k][1]; }
        if (sub + 1 < nsub) fetch_dy(tile, sub + 1);
        else if (next < p.n_tiles) fetch_dy(next, 0);
        if (!tc::mbar_wait(&sh.a_empty[ob], oph ^ 1u, p.err, 512)) goto done;
        uint8_t* abuf = aop + (size_t)ob * p.a_buf_bytes;
        uint8_t* bbuf = bop + (size_t)ob * b_buf_bytes;
        // dy: item = (channel n, 8-position chunk j): 32 contiguous bytes of global memory
#pragma unroll
        for (int k = 0; k < DMAX; ++k) {
          const int i = ct + k * WG_NCONV;
          if (i < d_items) {
            const int n = i / (SUB / 8), j = i - n * (SUB / 8);
            const float v[8] = {dcur[k][0].x, dcur[k][0].y, dcur[k][0].z, dcur[k][0].w,
                                dcur[k][1].x, dcur[k][1].y, dcur[k][1].z, dcur[k][1].w};
            store_split8(v, abuf + ((size_t)j * p.NP + n) * 16, p.a_term_bytes);
          }
        }
        // Xcol^T: item = (kk, 8-position chunk j): 8 consecutive patch columns
        for (int i = ct; i < x_items; i += WG_NCONV) {
          const int kk = i / (SUB / 8), j = i - kk * (SUB / 8);
          const int m = sub * SUB + j * 8;
          const float* src = patch + tab[kk] + (m / p.W) * p.PW + (m % p.W);
          float v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = src[e];
          store_split8(v, bbuf + ((size_t)j * p.KP + kk) * 16, p.b_term_bytes);
        }
        tc::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&sh.a_full[ob]);
      }
      if (next < p.n_tiles) patch_commit(p, patch0 + (size_t)((t + 1) & 1u) * patch_floats, next, ct, WG_NCONV, pre);
    }
  }
done:
  __syncthreads();
}

__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ partial, int n, int ranks,
                                                              float* __restrict__ dw) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < ranks; ++j) s += partial[(int64_t)j * n + i];
    dw[i] = s;
  }
}

static int plan(const mnb_conv_shape* s, bool wgrad, Params& p, int& smem_bytes) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  auto unsupported = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "fp32 tc conv: %s", why); };
  p.B = s->batch; p.C = s->in_c; p.K = s->out_c; p.H = s->in_h; p.W = s->in_w; p.R = s->ker_h;
  MNB_REQUIRE(p.B > 0 && p.C > 0 && p.K > 0 && p.H > 0 && p.W > 0 && s->groups > 0, "bad conv shape");
  if (s->groups != 1 || s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1)
    return unsupported("groups / stride / dilation != 1");
  if (s->ker_h != s->ker_w || (p.R & 1) == 0 || s->pad_h != p.R / 2 || s->pad_w != p.R / 2)
    return unsupported("not a 'same' odd square filter");
  p.pad = p.R / 2;
  p.KR = p.C * p.R * p.R;
  p.KP = (p.KR + 15) / 16 * 16;
  if (p.KP > 128) return unsupported("C*R*S > 128 (use the per-tap implicit GEMM)");
  if (p.K > 256) return unsupported("more than 256 output channels");   // also: K * 4 dy items <= DMAX * WG_NCONV
  if (p.W < 8 || p.W > 128 || 128 % p.W || (p.H * p.W) % 128) return unsupported("image rows do not tile into 128 positions");
  if ((int64_t)p.B * p.K * p.H * p.W >= (1ll << 31)) return unsupported("tensor too large");
  p.TH = 128 / p.W;
  p.PH = p.TH + 2 * p.pad; p.PW = p.W + 2 * p.pad;
  p.tiles_per_img = p.H / p.TH;
  p.n_tiles = p.B * p.tiles_per_img;
  p.patch_bytes = (p.C * p.PH * p.PW * 4 + 8 * 4 + 15) / 16 * 16;   // + slack: the wgrad gather of a padded kk row may overrun
  const int kchunks = p.KP / 8;
  if (!wgrad) {
    p.NP = (p.K + 15) / 16 * 16;
    p.b_term_bytes = kchunks * p.NP * 16;
    p.a_term_bytes = kchunks * 128 * 16;
    p.a_buf_bytes = 3 * p.a_term_bytes;
    p.off_b = 0;
    p.off_a = 3 * p.b_term_bytes;
    for (p.nbuf_a = 2; p.nbuf_a >= 1; --p.nbuf_a) {
      p.off_patch = p.off_a + p.nbuf_a * p.a_buf_bytes;
      p.off_tab = p.off_patch + 2 * p.patch_bytes;
      p.off_stg = (p.off_tab + p.KP * 4 + 15) / 16 * 16;
      smem_bytes = p.off_stg + 32 * tc::kStageLd * 4;   // 128 x 32 staging tile of the epilogue
      if (smem_bytes <= kMaxDynSmem) break;
    }
    if (p.nbuf_a < 1) return unsupported("shared memory budget");
  } else {
    p.NP = (p.K + 127) / 128 * 128;
    p.a_term_bytes = (SUB / 8) * p.NP * 16;
    p.a_buf_bytes = 3 * p.a_term_bytes;
    p.b_term_bytes = (SUB / 8) * p.KP * 16;
    // [B buf0][B buf1][A buf0][A buf1][running sum] contiguous (zeroed in one sweep by the kernel)
    p.off_b = 0;
    p.off_a = 2 * 3 * p.b_term_bytes;
    p.off_sum = p.off_a + 2 * p.a_buf_bytes;
    p.sum_bytes = (p.NP / 128) * p.KP * 128 * 4;
    p.off_patch = p.off_sum + p.sum_bytes;
    p.off_tab = p.off_patch + 2 * p.patch_bytes;
    smem_bytes = p.off_tab + p.KP * 4;
    p.nbuf_a = 2;
    if (smem_bytes > kMaxDynSmem) return unsupported("shared memory budget");
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ forward, two MMA warpgroups
// fwd_kernel runs a 128-position tile as 8 slabs of 32 channels on one warpgroup (MMA, wait, staging epilogue, one after
// another), and at the bench stems only one im2col buffer fits next to its weight image.  Here a tile is 64 positions and
// one m64nN MMA spans every output channel (N = Cout rounded up to 192 or 256), so A is read once per K-step
// instead of once per slab; two MMA warpgroups take alternate tiles, so one runs its epilogue while the other issues MMAs,
// and 3..4 im2col buffers let the converters build tile t + 2 meanwhile.  The epilogue stores straight from the fragment:
// the 8 row-lanes of a column are 8 consecutive positions of one channel, whole 32-byte sectors of y.
// Every output element sees fwd_kernel's chain: a zeroed accumulator, the kProdA / kProdB products in order with the
// same K-steps over the same split3_pair pieces (zero beyond KR and Cout), then + bias in fp32.  An MMA's result for one
// element does not depend on the N width or the 64-row block it is issued with (DESIGN.md 4.9), so y is bit for bit
// fwd_kernel's.  The plan never covers a shape fwd_kernel refuses.
// Measured on an H100 SXM (700 W), batch 256, 32 x 32: 3 -> 256 5x5 252 -> 164 us, 3 -> 192 5x5 194 -> 135 us per launch.
constexpr int FWG_THREADS = 384;   // warpgroup 0: im2col converters; warpgroups 1, 2: MMA + epilogue on alternate tiles
constexpr int FWG_NCONV = 128;
constexpr int FWG_PF = 6;          // FWG_PF * FWG_NCONV >= the bench stems' 648-float patch: no element waits on its load
constexpr int FWG_MAXBUF = 4;
constexpr int FWG_CONV_REGS = 56, FWG_MMA_REGS = 224;   // 128 * 56 + 256 * 224 <= 65536 (m64n256: 128 accumulators)

struct alignas(16) FwgShared {
  uint64_t full[FWG_MAXBUF], empty[FWG_MAXBUF];
  uint32_t abort;
};

template <int N>
__global__ void __launch_bounds__(FWG_THREADS, 1) fwd_wg_kernel(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ FwgShared sh;
  __shared__ __align__(16) float epi_bias[N];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* bop = smem + p.off_b;
  uint8_t* aop = smem + p.off_a;
  int* tab = reinterpret_cast<int*>(smem + p.off_tab);
  const int kchunks = p.KP / 8;

  if (tid == 0) {
    for (int i = 0; i < FWG_MAXBUF; ++i) {
      tc::mbar_init(&sh.full[i], FWG_NCONV / 32); tc::mbar_init(&sh.empty[i], 4);
    }
    sh.abort = 0;
    tc::fence_barrier_init();
  }
  for (int n = tid; n < N; n += FWG_THREADS) epi_bias[n] = (p.bias && n < p.K) ? __ldg(p.bias + n) : 0.f;
  // resident B operand, as in fwd_kernel with NP = N
  for (int i = tid; i < kchunks * N; i += FWG_THREADS) {
    const int j = i / N, n = i - j * N;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int kk = j * 8 + e;
      v[e] = (n < p.K && kk < p.KR) ? __ldg(p.w + (int64_t)n * p.KR + kk) : 0.f;
    }
    store_split8(v, bop + (size_t)i * 16, p.b_term_bytes);
  }
  for (int kk = tid; kk < p.KP; kk += FWG_THREADS) {
    int off = -1;
    if (kk < p.KR) {
      const int s = kk % p.R, t = kk / p.R;
      const int r = t % p.R, c = t / p.R;
      off = (c * p.PH + r) * p.PW + s;
    }
    tab[kk] = off;
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  // local tile t of this CTA = tile blockIdx.x + t * gridDim.x, im2col buffer t % nbuf_a, MMA warpgroup t % 2
  const int n_local = (int)blockIdx.x < p.n_tiles ? (p.n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (warp < FWG_NCONV / 32) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FWG_CONV_REGS));
    // ================================================================= converters: patch -> im2col A operand
    const int ct = tid;
    float* patch0 = reinterpret_cast<float*>(smem + p.off_patch);
    const int items = 64 * kchunks;
    const int patch_floats = p.patch_bytes / 4;
    float pre[FWG_PF];
    if (n_local > 0) {
      patch_fetch(p, blockIdx.x, ct, FWG_NCONV, pre);
      patch_commit(p, patch0, blockIdx.x, ct, FWG_NCONV, pre);
    }
    for (int t = 0; t < n_local; ++t) {
      const int tile = (int)blockIdx.x + t * (int)gridDim.x;
      const float* patch = patch0 + (size_t)(t & 1) * patch_floats;
      conv_bar_sync(FWG_NCONV);   // every converter committed its part of this tile's patch
      const int next = tile + (int)gridDim.x;
      if (next < p.n_tiles) patch_fetch(p, next, ct, FWG_NCONV, pre);
      const int ab = t % p.nbuf_a;
      const uint32_t aph = (uint32_t)(t / p.nbuf_a) & 1u;
      if (!tc::mbar_wait(&sh.empty[ab], aph ^ 1u, p.err, 506)) break;
      uint8_t* abuf = aop + (size_t)ab * p.a_buf_bytes;
      for (int i = ct; i < items; i += FWG_NCONV) {
        const int j = i >> 6, m = i & 63;
        const int base = (m / p.W) * p.PW + (m % p.W);
        int off[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) off[e] = tab[j * 8 + e];
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = off[e] >= 0 ? patch[off[e] + base] : 0.f;
        store_split8(v, abuf + (size_t)i * 16, p.a_term_bytes);
      }
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.full[ab]);
      if (next < p.n_tiles) patch_commit(p, patch0 + (size_t)((t + 1) & 1) * patch_floats, next, ct, FWG_NCONV, pre);
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FWG_MMA_REGS));
    // ================================================================= MMA warpgroups: wgmma -> + bias -> y (NCHW)
    const int wg = (warp - FWG_NCONV / 32) >> 2, w4 = warp & 3;
    const int64_t plane = (int64_t)p.H * p.W;
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(aop), 64u * 16u, 128u);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(bop), (uint32_t)N * 16u, 128u);
    const uint32_t a_term16 = (uint32_t)p.a_term_bytes >> 4, b_term16 = (uint32_t)p.b_term_bytes >> 4;
    const uint32_t a_buf16 = (uint32_t)p.a_buf_bytes >> 4;
    const uint32_t a_step16 = 2u * 64u, b_step16 = 2u * (uint32_t)N;   // one K16 step = two 8-wide chunks
    const int ksteps = p.KP / 16;
    // fragment: acc[4j + 2i + c] = D[row 16 w4 + lane / 4 + 8i][column 8j + 2 (lane % 4) + c]
    const int fr = 16 * w4 + (lane >> 2), fc = 2 * (lane & 3);
    for (int t = wg; t < n_local; t += 2) {
      const int tile = (int)blockIdx.x + t * (int)gridDim.x;
      const int ab = t % p.nbuf_a;
      tc::mbar_wait_soft(&sh.full[ab], (uint32_t)(t / p.nbuf_a) & 1u, p.err, 505, &sh.abort);
      float acc[N / 2];
      tc::zero_acc(acc);
      tc::wg_fence();
      tc::fence_acc(acc);
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const uint64_t aq = a_desc0 + (uint64_t)((uint32_t)ab * a_buf16 + (uint32_t)kProdA[q] * a_term16);
        const uint64_t bq = b_desc0 + (uint64_t)((uint32_t)kProdB[q] * b_term16);
        for (int ks = 0; ks < ksteps; ++ks)
          tc::Mma<N>::template bf16<0, 0>(acc, aq + (uint64_t)((uint32_t)ks * a_step16), bq + (uint64_t)((uint32_t)ks * b_step16), 1);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::fence_acc(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.empty[ab]);   // the tile's MMAs retired: its operand buffer is free
      const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
      float* dst = p.y + (int64_t)b * p.K * plane + (int64_t)h0 * p.W + fr;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int n = 8 * j + fc;
        const float2 bs = *reinterpret_cast<const float2*>(&epi_bias[n]);
        float* o = dst + (int64_t)n * plane;
        if (n < p.K) { o[0] = __fadd_rn(acc[4 * j], bs.x); o[8] = __fadd_rn(acc[4 * j + 2], bs.x); }
        if (n + 1 < p.K) { o[plane] = __fadd_rn(acc[4 * j + 1], bs.y); o[plane + 8] = __fadd_rn(acc[4 * j + 3], bs.y); }
      }
    }
  }
  __syncthreads();
}

static int grid_size(const Params& p) { return std::max(1, std::min(p.n_tiles, MNB_NUM_SMS)); }

// plan of fwd_wg_kernel: fwd_kernel's cover (whose checks it runs first) where a 64-position tile holds whole rows
// (W <= 64) and at least 3 im2col buffers fit next to the weight image
static int plan_wg(const mnb_conv_shape* s, Params& p, int& smem_bytes) {
  if (int e = plan(s, false, p, smem_bytes)) return e;
  auto unsupported = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "fp32 tc conv (two warpgroups): %s", why); };
  if (64 % p.W) return unsupported("image rows do not tile into 64 positions");
  // at narrow N a tile's MMAs are too short to hide the converters and the epilogue: the 3 -> 64 stem measured slower
  if (p.K <= 128) return unsupported("128 output channels or fewer");
  p.TH = 64 / p.W;
  p.PH = p.TH + 2 * p.pad;
  p.tiles_per_img = p.H / p.TH;
  p.n_tiles = p.B * p.tiles_per_img;
  p.patch_bytes = (p.C * p.PH * p.PW * 4 + 8 * 4 + 15) / 16 * 16;
  p.NP = p.K <= 192 ? 192 : 256;
  const int kchunks = p.KP / 8;
  p.b_term_bytes = kchunks * p.NP * 16;
  p.a_term_bytes = kchunks * 64 * 16;
  p.a_buf_bytes = 3 * p.a_term_bytes;
  p.off_b = 0;
  p.off_a = 3 * p.b_term_bytes;
  for (p.nbuf_a = FWG_MAXBUF; p.nbuf_a >= 3; --p.nbuf_a) {
    p.off_patch = p.off_a + p.nbuf_a * p.a_buf_bytes;
    p.off_tab = p.off_patch + 2 * p.patch_bytes;
    smem_bytes = p.off_tab + p.KP * 4;
    if (smem_bytes <= kMaxDynSmem) break;
  }
  if (p.nbuf_a < 3) return unsupported("shared memory budget (3 im2col buffers)");
  return 0;
}

template <int N>
static int launch_fwd_wg(const Params& p, int smem_bytes, mnb_stream_t stream) {
  static bool attr_set = false;   // one per instantiation
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(fwd_wg_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set = true;
  }
  fwd_wg_kernel<N><<<grid_size(p), FWG_THREADS, smem_bytes, (cudaStream_t)stream>>>(p);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------------------------------------ weight gradient, two MMA warpgroups
// wgrad_kernel issues m64n32 over KP = 80 in three slabs (96 columns for 80), waits after every 24 MMAs and then adds each
// fragment into a running sum in shared memory (4-way bank conflicts on every read and write).  Here two MMA warpgroups
// each own every other 64-channel block (blocks wg, wg + 2) and one m64nKP MMA spans all im2col columns; the running sums
// stay in registers (a (channel, kk) element lives in the same thread of the same fragment for the whole launch), and a
// ring of 3 dy / Xcol stages lets warpgroup 0 convert two steps ahead.
// Bit identity with wgrad_kernel: the same plan (tiles, grid, CTA i takes tiles i, i + grid, ...), the same 32-position
// steps in order, per step and element one 12-MMA chain (kProdA / kProdB order, 2 K-steps each) from a zeroed
// accumulator added with __fadd_rn into a running sum that starts at 0, one partial per CTA, reduce_partials_kernel.
constexpr int WWG_THREADS = 384;   // warpgroup 0: converters (dy split + im2col of x); warpgroups 1, 2: MMA
constexpr int WWG_NCONV = 128;
constexpr int WWG_DMAX = 8;        // dy items (channel, 8 positions) per converter and step: 4 * Cout <= 8 * 128
constexpr int WWG_NBUF = 3;
constexpr int WWG_KP = 80;         // the 3 x 5 x 5 stems

template <int KP>
__global__ void __launch_bounds__(WWG_THREADS, 1) wgrad_wg_kernel(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ FwgShared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* bop = smem + p.off_b;   // Xcol^T : [buf][piece][pos / 8][kk][8 pos]
  uint8_t* aop = smem + p.off_a;   // dy     : [buf][piece][pos / 8][channel][8 pos]
  int* tab = reinterpret_cast<int*>(smem + p.off_tab);
  const int nsub = 128 / SUB;
  const int b_buf_bytes = 3 * p.b_term_bytes;

  if (tid == 0) {
    for (int i = 0; i < WWG_NBUF; ++i) {
      tc::mbar_init(&sh.full[i], WWG_NCONV / 32); tc::mbar_init(&sh.empty[i], 8);
    }
    sh.abort = 0;
    tc::fence_barrier_init();
  }
  // operand buffers start as zeros: channel rows >= Cout and im2col rows >= KR are never written
  for (int i = tid; i < WWG_NBUF * (p.a_buf_bytes + b_buf_bytes) / 16; i += WWG_THREADS)
    reinterpret_cast<uint4*>(smem + p.off_b)[i] = make_uint4(0, 0, 0, 0);
  for (int kk = tid; kk < p.KP; kk += WWG_THREADS) {
    int off = -1;
    if (kk < p.KR) {
      const int s = kk % p.R, t = kk / p.R;
      const int r = t % p.R, c = t / p.R;
      off = (c * p.PH + r) * p.PW + s;
    }
    tab[kk] = off;
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp >= 4) {
    // ================================================================= MMA warpgroups: wgmma -> register running sums -> partial dw
    const int wg = (warp - 4) >> 2, w4 = warp & 3;
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(aop), (uint32_t)p.NP * 16u, 128u);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(bop), (uint32_t)KP * 16u, 128u);
    const uint32_t a_term16 = (uint32_t)p.a_term_bytes >> 4, b_term16 = (uint32_t)p.b_term_bytes >> 4;
    const uint32_t a_buf16 = (uint32_t)p.a_buf_bytes >> 4, b_buf16 = (uint32_t)b_buf_bytes >> 4;
    const uint32_t a_step16 = 2u * (uint32_t)p.NP, b_step16 = 2u * (uint32_t)KP;
    float sum0[KP / 2], sum1[KP / 2];   // blocks wg, wg + 2
    tc::zero_acc(sum0); tc::zero_acc(sum1);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
      for (int sub = 0; sub < nsub; ++sub, ++it) {
        const uint32_t ob = it % WWG_NBUF, oph = (it / WWG_NBUF) & 1u;
        tc::mbar_wait_soft(&sh.full[ob], oph, p.err, 515, &sh.abort);
#pragma unroll 1
        for (int mb = 0; mb < 2; ++mb) {   // 64-channel blocks wg, wg + 2; rolled: two chains in one block serialise the wgmma
          float acc[KP / 2];
          tc::zero_acc(acc);
          tc::wg_fence();
          tc::fence_acc(acc);
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const uint64_t aq = a_desc0 + (uint64_t)(ob * a_buf16 + (uint32_t)kProdA[q] * a_term16 + (uint32_t)(wg + 2 * mb) * 64u);
            const uint64_t bq = b_desc0 + (uint64_t)(ob * b_buf16 + (uint32_t)kProdB[q] * b_term16);
#pragma unroll
            for (int ks = 0; ks < SUB / 16; ++ks)
              tc::Mma<KP>::template bf16<0, 0>(acc, aq + (uint64_t)((uint32_t)ks * a_step16), bq + (uint64_t)((uint32_t)ks * b_step16), 1);
          }
          tc::wg_commit();
          tc::wg_wait<0>();
          tc::fence_acc(acc);
#pragma unroll
          for (int i = 0; i < KP / 2; ++i) {
            if (mb == 0) sum0[i] = __fadd_rn(sum0[i], acc[i]);
            else sum1[i] = __fadd_rn(sum1[i], acc[i]);
          }
        }
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&sh.empty[ob]);
      }
    }
    // fragment: sum[mb][4j + 2i + c] = dw[channel 64 (wg + 2 mb) + 16 w4 + lane / 4 + 8i][kk 8j + 2 (lane % 4) + c]
    float* mine = p.partial + (int64_t)blockIdx.x * p.K * p.KR;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
      for (int e = 0; e < KP / 2; ++e) {
        const int n = 64 * (wg + 2 * mb) + 16 * w4 + (lane >> 2) + 8 * ((e >> 1) & 1);
        const int kk = 8 * (e >> 2) + 2 * (lane & 3) + (e & 1);
        if (n < p.K && kk < p.KR) mine[(int64_t)n * p.KR + kk] = mb == 0 ? sum0[e] : sum1[e];
      }
    }
  } else {
    // ================================================================= converters: wgrad_kernel's, with each step's dy loaded
    // when the step starts (a register copy of the next step's dy does not fit next to it): the ring runs them ahead
    const int ct = tid;
    float* patch0 = reinterpret_cast<float*>(smem + p.off_patch);
    const int64_t plane = (int64_t)p.H * p.W;
    const int d_items = p.K * (SUB / 8), x_items = p.KR * (SUB / 8);
    const int patch_floats = p.patch_bytes / 4;
    float4 dpre[WWG_DMAX][2];
    auto fetch_dy = [&](int tile, int sub) {
      const int b = tile / p.tiles_per_img, h0 = (tile - b * p.tiles_per_img) * p.TH;
      const float* dy_tile = p.dy + (int64_t)b * p.K * plane + (int64_t)h0 * p.W + sub * SUB;
#pragma unroll
      for (int k = 0; k < WWG_DMAX; ++k) {
        const int i = ct + k * WWG_NCONV;
        if (i < d_items) {
          const int n = i / (SUB / 8), j = i - n * (SUB / 8);
          const float4* src = reinterpret_cast<const float4*>(dy_tile + (int64_t)n * plane + j * 8);
          dpre[k][0] = __ldg(src); dpre[k][1] = __ldg(src + 1);
        }
      }
    };
    float pre[PF];
    if ((int)blockIdx.x < p.n_tiles) {
      patch_fetch(p, blockIdx.x, ct, WWG_NCONV, pre);
      patch_commit(p, patch0, blockIdx.x, ct, WWG_NCONV, pre);
    }
    uint32_t it = 0, t = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++t) {
      const float* patch = patch0 + (size_t)(t & 1u) * patch_floats;
      conv_bar_sync(WWG_NCONV);
      const int next = tile + (int)gridDim.x;
      if (next < p.n_tiles) patch_fetch(p, next, ct, WWG_NCONV, pre);
      for (int sub = 0; sub < nsub; ++sub, ++it) {
        const uint32_t ob = it % WWG_NBUF, oph = (it / WWG_NBUF) & 1u;
        fetch_dy(tile, sub);
        const auto& dcur = dpre;
        if (!tc::mbar_wait(&sh.empty[ob], oph ^ 1u, p.err, 516)) goto done;
        uint8_t* abuf = aop + (size_t)ob * p.a_buf_bytes;
        uint8_t* bbuf = bop + (size_t)ob * b_buf_bytes;
#pragma unroll
        for (int k = 0; k < WWG_DMAX; ++k) {
          const int i = ct + k * WWG_NCONV;
          if (i < d_items) {
            const int n = i / (SUB / 8), j = i - n * (SUB / 8);
            const float v[8] = {dcur[k][0].x, dcur[k][0].y, dcur[k][0].z, dcur[k][0].w,
                                dcur[k][1].x, dcur[k][1].y, dcur[k][1].z, dcur[k][1].w};
            store_split8(v, abuf + ((size_t)j * p.NP + n) * 16, p.a_term_bytes);
          }
        }
        for (int i = ct; i < x_items; i += WWG_NCONV) {
          const int kk = i / (SUB / 8), j = i - kk * (SUB / 8);
          const int m = sub * SUB + j * 8;
          const float* src = patch + tab[kk] + (m / p.W) * p.PW + (m % p.W);
          float v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = src[e];
          store_split8(v, bbuf + ((size_t)j * KP + kk) * 16, p.b_term_bytes);
        }
        tc::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&sh.full[ob]);
      }
      if (next < p.n_tiles) patch_commit(p, patch0 + (size_t)((t + 1) & 1u) * patch_floats, next, ct, WWG_NCONV, pre);
    }
  }
done:
  __syncthreads();
}

// plan of wgrad_wg_kernel: wgrad_kernel's plan (whose tiles, grid and partials it keeps) at KP = 80 and 129..256 output
// channels (four 64-channel blocks, two per MMA warpgroup: a branch around a block would serialise the wgmma), with a ring of 3
// stages in place of 2 stages and the shared-memory running sum
static int plan_wgrad_wg(const mnb_conv_shape* s, Params& p, int& smem_bytes) {
  if (int e = plan(s, true, p, smem_bytes)) return e;
  if (p.KP != WWG_KP) return mnb_fail(MNB_E_UNSUPPORTED, "fp32 tc wgrad (two warpgroups): C*R*S not in 65..80");
  if (p.NP != 256) return mnb_fail(MNB_E_UNSUPPORTED, "fp32 tc wgrad (two warpgroups): 128 output channels or fewer");
  p.off_b = 0;
  p.off_a = WWG_NBUF * 3 * p.b_term_bytes;
  p.off_patch = p.off_a + WWG_NBUF * p.a_buf_bytes;
  p.off_tab = p.off_patch + 2 * p.patch_bytes;
  p.sum_bytes = 0;
  p.nbuf_a = WWG_NBUF;
  smem_bytes = p.off_tab + p.KP * 4;
  if (smem_bytes > kMaxDynSmem) return mnb_fail(MNB_E_UNSUPPORTED, "fp32 tc wgrad (two warpgroups): shared memory budget");
  return 0;
}

}  // namespace tcfp32

extern "C" int mnb_fconv2d_plan(const mnb_conv_shape* s, int32_t wgrad, int32_t* out, int32_t n) {
  tcfp32::Params p{};
  int smem_bytes = 0;
  if (int e = tcfp32::plan(s, wgrad != 0, p, smem_bytes)) return e;
  const int v[8] = {p.NP, p.KP, p.TH, p.n_tiles, tcfp32::grid_size(p), p.nbuf_a, smem_bytes, p.C * p.PH * p.PW};
  if (out)
    for (int i = 0; i < std::min(n, 8); ++i) out[i] = v[i];
  return 0;
}

extern "C" int mnb_fconv2d_fwd_tc(const mnb_conv_shape* s, const float* x, const float* w, const float* bias, float* y,
                                  int32_t* err_flag, mnb_stream_t stream) {
  using namespace tcfp32;
  MNB_REQUIRE(s && x && w && y && err_flag, "NULL pointer");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan(s, false, p, smem_bytes)) return e;
  p.x = x; p.w = w; p.bias = bias; p.y = y; p.err = err_flag;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set = true;
  }
  fwd_kernel<<<grid_size(p), NTHREADS, smem_bytes, (cudaStream_t)stream>>>(p);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_fconv2d_wg_plan(const mnb_conv_shape* s, int32_t* out, int32_t n) {
  tcfp32::Params p{};
  int smem_bytes = 0;
  if (int e = tcfp32::plan_wg(s, p, smem_bytes)) return e;
  const int v[8] = {p.NP, p.KP, p.TH, p.n_tiles, tcfp32::grid_size(p), p.nbuf_a, smem_bytes, p.C * p.PH * p.PW};
  if (out)
    for (int i = 0; i < std::min(n, 8); ++i) out[i] = v[i];
  return 0;
}

extern "C" int mnb_fconv2d_fwd_wg(const mnb_conv_shape* s, const float* x, const float* w, const float* bias, float* y,
                                  int32_t* err_flag, mnb_stream_t stream) {
  using namespace tcfp32;
  MNB_REQUIRE(s && x && w && y && err_flag, "NULL pointer");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan_wg(s, p, smem_bytes)) return e;
  p.x = x; p.w = w; p.bias = bias; p.y = y; p.err = err_flag;
  return p.NP == 192 ? launch_fwd_wg<192>(p, smem_bytes, stream) : launch_fwd_wg<256>(p, smem_bytes, stream);
}

extern "C" int64_t mnb_fconv2d_wgrad_tc_scratch_bytes(const mnb_conv_shape* s) {
  tcfp32::Params p{};
  int smem = 0;
  if (tcfp32::plan(s, true, p, smem)) return -1;
  return (int64_t)tcfp32::grid_size(p) * p.K * p.KR * 4;
}

extern "C" int mnb_fconv2d_wgrad_tc(const mnb_conv_shape* s, const float* dy, const float* x, float* dw, void* scratch,
                                    int32_t* err_flag, mnb_stream_t stream) {
  using namespace tcfp32;
  MNB_REQUIRE(s && dy && x && dw && scratch && err_flag, "NULL pointer");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(dy) & 15) == 0, "dy must be 16-byte aligned");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan(s, true, p, smem_bytes)) return e;
  p.x = x; p.dy = dy; p.partial = reinterpret_cast<float*>(scratch); p.err = err_flag;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set = true;
  }
  const int grid = grid_size(p);
  cudaStream_t st = (cudaStream_t)stream;
  wgrad_kernel<<<grid, NTHREADS, smem_bytes, st>>>(p);
  const int n = p.K * p.KR;
  reduce_partials_kernel<<<std::min(mnb_ceil_div(n, 256), MNB_NUM_SMS * 4), 256, 0, st>>>(p.partial, n, grid, dw);
  MNB_LAUNCHED(2);
  return 0;
}

extern "C" int64_t mnb_fconv2d_wgrad_wg_scratch_bytes(const mnb_conv_shape* s) {
  tcfp32::Params p{};
  int smem = 0;
  if (tcfp32::plan_wgrad_wg(s, p, smem)) return -1;
  return (int64_t)tcfp32::grid_size(p) * p.K * p.KR * 4;
}

extern "C" int mnb_fconv2d_wgrad_wg(const mnb_conv_shape* s, const float* dy, const float* x, float* dw, void* scratch,
                                    int32_t* err_flag, mnb_stream_t stream) {
  using namespace tcfp32;
  MNB_REQUIRE(s && dy && x && dw && scratch && err_flag, "NULL pointer");
  MNB_REQUIRE((reinterpret_cast<uintptr_t>(dy) & 15) == 0, "dy must be 16-byte aligned");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan_wgrad_wg(s, p, smem_bytes)) return e;
  p.x = x; p.dy = dy; p.partial = reinterpret_cast<float*>(scratch); p.err = err_flag;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(wgrad_wg_kernel<WWG_KP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set = true;
  }
  const int grid = grid_size(p);
  cudaStream_t st = (cudaStream_t)stream;
  wgrad_wg_kernel<WWG_KP><<<grid, WWG_THREADS, smem_bytes, st>>>(p);
  const int n = p.K * p.KR;
  reduce_partials_kernel<<<std::min(mnb_ceil_div(n, 256), MNB_NUM_SMS * 4), 256, 0, st>>>(p.partial, n, grid, dw);
  MNB_LAUNCHED(2);
  return 0;
}
