// Packed bf16 output of the BatchNorm + binarizer producer: mnb_bn_sign_fwd_packed = mnb_bn_sign_fwd plus
// xp[b][c/8][h][w][8] (bf16 +-1, OUTPUT channel order) - the operand plane the packed-operand tensor-core family
// (mnb_pk.cu) reads with TMA, so that a wbwtab layer behind a fused BatchNorm + binarizer needs no pack pass and no
// converter warps (fused.BNSignFn -> functional._pk_forward(prepacked=...)).
// (The round-1 consumer kernel that lived in this file was superseded by mnb_pk.cu before it ever ran and is gone.)
#include <cuda_bf16.h>

#include <algorithm>

#include "mnb_common.cuh"

namespace tcpacked {

template <int VEC> struct VecT;
template <> struct VecT<1> { typedef float type; };
template <> struct VecT<2> { typedef float2 type; };
template <> struct VecT<4> { typedef float4 type; };

template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
  typedef typename VecT<VEC>::type T;
  T t;
  float* f = reinterpret_cast<float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) f[i] = v[i];
  *reinterpret_cast<T*>(p) = t;
}

// ---------------------------------------------------------------------------------------------- producer
// One warp = 32 * VEC consecutive positions of one OUTPUT channel octet of one image; a lane owns VEC consecutive positions
// (16-byte loads of x for VEC = 4, VEC consecutive 16-byte pixels of the plane = 64 contiguous bytes per lane: one position
// per lane with 4-byte accesses leaves this stream far below HBM bandwidth).  y is optional - a consuming conv of the
// packed-operand family reads only the plane.  XT = int16_t: x as a wbwtab conv's codes + decode pair (mnb_common.cuh).
template <int VEC, typename XT>
__global__ void __launch_bounds__(256) bn_sign_packed_fwd_kernel(const XT* __restrict__ x, const float* __restrict__ dec,
                                                                 int batch, int channels, int hw, int sg, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, float* __restrict__ y,
                                                                 uint32_t* __restrict__ bits, uint4* __restrict__ xp) {
  constexpr int LPW = 32 / VEC;                 // lanes that share one 32-position word of pass bits
  const int lane = threadIdx.x & 31;
  const int c8n = channels / 8, chunks = hw / (32 * VEC), cpg = channels / sg;
  const int64_t items = (int64_t)batch * c8n * chunks;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items; w += nwarps) {
    const int ch = (int)(w % chunks);
    const int64_t t = w / chunks;
    const int oc8 = (int)(t % c8n), b = (int)(t / c8n);
    const int pos = (ch * 32 + lane) * VEC;
    float v[8][VEC];
    int cc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int oc = oc8 * 8 + j;
      cc[j] = sg > 1 ? (oc % sg) * cpg + oc / sg : oc;   // inverse of out[:, a*sg + b] = in[:, b*cpg + a]
      x_load<VEC>(x + ((int64_t)b * channels + cc[j]) * hw + pos, x_dec<XT>(dec, channels, cc[j]), v[j]);
    }
    uint32_t h[VEC][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = cc[j];
      const float mu = __ldg(mean + c), k = __ldg(gamma + c) * __ldg(invstd + c), be = __ldg(beta + c);
      uint32_t pass = 0;
      float yv[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float bn = fmaf(v[j][i] - mu, k, be);
        const bool neg = bn < 0.f;
        yv[i] = neg ? -1.f : 1.f;
        h[i][j] = neg ? 0xBF80u : 0x3F80u;   // bf16 -1 / +1
        pass |= (fabsf(bn) < 1.f ? 1u : 0u) << i;
      }
      if (y) store_vec<VEC>(y + ((int64_t)b * channels + oc8 * 8 + j) * hw + pos, yv);
      // pass bits: flat NCHW bit index of the producer's own channel order, 32 positions per word
      uint32_t word = pass << (VEC * (lane % LPW));
#pragma unroll
      for (int o = 1; o < LPW; o <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, o);
      if (lane % LPW == 0) bits[(((int64_t)b * channels + c) * hw + pos) >> 5] = word;
    }
    uint4* dst = xp + ((int64_t)b * c8n + oc8) * hw + pos;
#pragma unroll
    for (int i = 0; i < VEC; ++i)
      dst[i] = make_uint4(h[i][0] | (h[i][1] << 16), h[i][2] | (h[i][3] << 16), h[i][4] | (h[i][5] << 16), h[i][6] | (h[i][7] << 16));
  }
}

}  // namespace tcpacked

template <typename XT>
static int bn_sign_fwd_packed(const XT* x, const float* dec, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                              const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups, float* y,
                              uint32_t* pass_bits, void* x_packed, mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && invstd && gamma && beta && pass_bits && x_packed, "NULL bn_sign_fwd_packed pointer");   // y may be NULL
  MNB_REQUIRE(batch > 0 && channels > 0 && hw > 0, "bad bn_sign_fwd_packed shape");
  MNB_REQUIRE(out_shuffle_groups >= 1 && channels % out_shuffle_groups == 0, "shuffle groups %d do not divide %d channels",
              out_shuffle_groups, channels);
  if (channels % 8 || hw % 32 || (reinterpret_cast<uintptr_t>(x_packed) & 15))
    return mnb_fail(MNB_E_UNSUPPORTED, "packed producer needs channels %% 8 == 0, H*W %% 32 == 0, 16-byte aligned output");
  constexpr uintptr_t xa4 = 4 * sizeof(XT) - 1, xa2 = 2 * sizeof(XT) - 1;   // alignment of a 4- / 2-element load of x
  const int vec = (hw % 128 == 0 && (reinterpret_cast<uintptr_t>(x) & xa4) == 0 && (!y || (reinterpret_cast<uintptr_t>(y) & 15) == 0)) ? 4
                  : ((hw % 64 == 0 && (reinterpret_cast<uintptr_t>(x) & xa2) == 0 && (!y || (reinterpret_cast<uintptr_t>(y) & 7) == 0)) ? 2 : 1);
  const int64_t warps = (int64_t)batch * (channels / 8) * (hw / (32 * vec));
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(warps, 8), MNB_NUM_SMS * 8);
  uint4* xp = reinterpret_cast<uint4*>(x_packed);
  cudaStream_t st = (cudaStream_t)stream;
  if (vec == 4)
    tcpacked::bn_sign_packed_fwd_kernel<4, XT><<<blocks, 256, 0, st>>>(x, dec, batch, channels, hw, out_shuffle_groups, mean, invstd, gamma, beta, y, pass_bits, xp);
  else if (vec == 2)
    tcpacked::bn_sign_packed_fwd_kernel<2, XT><<<blocks, 256, 0, st>>>(x, dec, batch, channels, hw, out_shuffle_groups, mean, invstd, gamma, beta, y, pass_bits, xp);
  else
    tcpacked::bn_sign_packed_fwd_kernel<1, XT><<<blocks, 256, 0, st>>>(x, dec, batch, channels, hw, out_shuffle_groups, mean, invstd, gamma, beta, y, pass_bits, xp);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_sign_fwd_packed(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                                      const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups,
                                      float* y, uint32_t* pass_bits, void* x_packed, mnb_stream_t stream) {
  return bn_sign_fwd_packed<float>(x, nullptr, batch, channels, hw, mean, invstd, gamma, beta, out_shuffle_groups, y, pass_bits,
                                   x_packed, stream);
}

extern "C" int mnb_bn_sign_fwd_packed_codes(const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t hw,
                                            const float* mean, const float* invstd, const float* gamma, const float* beta,
                                            int32_t out_shuffle_groups, float* y, uint32_t* pass_bits, void* x_packed,
                                            mnb_stream_t stream) {
  MNB_REQUIRE(dec, "NULL decode pair");
  return bn_sign_fwd_packed<int16_t>(codes, dec, batch, channels, hw, mean, invstd, gamma, beta, out_shuffle_groups, y, pass_bits,
                                     x_packed, stream);
}
