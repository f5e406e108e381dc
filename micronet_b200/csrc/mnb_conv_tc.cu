// wgmma / TMA tensor-core plumbing of the fake-quant convolution (sm_90a only).
//
// Host-side tensor-map encoding, and two hardware self-tests exported through the C-ABI.  They pin the two
// things that cannot be checked on a CPU-only build box - the wgmma shared-memory descriptor encodings (K-major
// and MN-major operands) and the TMA box geometry with out-of-bounds zero fill - on tiny problems with known
// answers, under bounded waits (a wrong descriptor must fail a test, not hang a GPU).
#include <cuda.h>
#include <cuda_bf16.h>

#include <mutex>
#include <type_traits>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

// ------------------------------------------------------------------ host: tensor-map encoding
namespace {

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

}  // namespace

// rank-`rank` tiled map over a dense tensor; dims/box innermost-first; elem_bytes 4 (f32) / 2 / 1
int mnb_make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                  const uint32_t* box) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return mnb_fail(MNB_E_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  // driver-API call: make sure this host thread (e.g. an autograd worker) has the primary context bound - once per
  // thread (a cudaFree inside a stream capture would invalidate the capture)
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bdim[5], estr[5];
  uint64_t stride = (uint64_t)elem_bytes;
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    stride *= dims[i];
    if (i < rank - 1) gstr[i] = stride;  // byte stride of dimension i+1
  }
  CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                           : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return mnb_fail(MNB_E_ARG, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int mnb_make_tmap_strided(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return mnb_fail(MNB_E_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  { static thread_local bool ctx_bound = false; if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; } }
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i < rank - 1) gstr[i] = strides_bytes[i];
  }
  CUtensorMapDataType dt = elem_bytes == 8 ? CU_TENSOR_MAP_DATA_TYPE_UINT64
                           : elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                           : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return mnb_fail(MNB_E_ARG, "cuTensorMapEncodeTiled (strided) failed with CUresult %d", (int)r);
  return 0;
}

// ------------------------------------------------------------------ self-test 1: wgmma descriptors
// D[128 x N] = A[128 x K] * B[N x K]^T, operands converted by threads into the K-major no-swizzle
// canonical layout  buf[k_chunk][row][16 bytes]  (SBO = 128 B, LBO = rows * 16 B).  One warpgroup computes the two
// 64-row halves with N = 128 instructions (columns >= N are discarded).
template <bool INT8>
__global__ void __launch_bounds__(128) selftest_umma_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                            float* __restrict__ D, int N, int K, int* err) {
  constexpr int EPC = INT8 ? 16 : 8;  // elements per 16-byte chunk
  __shared__ __align__(128) uint8_t a_s[128 * 64 * 2];
  __shared__ __align__(128) uint8_t b_s[128 * 64 * 2];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int nchunk = K / EPC;
  for (int i = tid; i < (int)sizeof(b_s) / 16; i += 128) reinterpret_cast<uint4*>(b_s)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (int kc = 0; kc < nchunk; ++kc) {
    uint8_t* dst = a_s + ((size_t)kc * 128 + tid) * 16;
    for (int e = 0; e < EPC; ++e) {
      float v = A[(size_t)tid * K + kc * EPC + e];
      if (INT8) reinterpret_cast<int8_t*>(dst)[e] = (int8_t)v;
      else reinterpret_cast<__nv_bfloat16*>(dst)[e] = __float2bfloat16_rn(v);
    }
    if (tid < N) {
      uint8_t* db = b_s + ((size_t)kc * N + tid) * 16;
      for (int e = 0; e < EPC; ++e) {
        float v = B[(size_t)tid * K + kc * EPC + e];
        if (INT8) reinterpret_cast<int8_t*>(db)[e] = (int8_t)v;
        else reinterpret_cast<__nv_bfloat16*>(db)[e] = __float2bfloat16_rn(v);
      }
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const int ksteps = nchunk / 2;   // one MMA K-step = two 16-byte chunks (16 bf16 / 32 int8)
  for (int h = 0; h < 2; ++h) {
    typename std::conditional<INT8, int32_t, float>::type acc[64];
    tc::zero_acc(acc);
    tc::wg_fence();
    tc::fence_acc(acc);
    for (int ks = 0; ks < ksteps; ++ks) {
      const uint64_t ad = tc::smem_desc_kmajor_noswz(tc::smem_u32(a_s) + ks * 2 * 128 * 16 + h * 64 * 16, 128 * 16, 128);
      const uint64_t bd = tc::smem_desc_kmajor_noswz(tc::smem_u32(b_s) + ks * 2 * N * 16, N * 16, 128);
      if constexpr (INT8) tc::mma_s8_n128(acc, ad, bd, 1);
      else tc::Mma<128>::bf16<0, 0>(acc, ad, bd, 1);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::fence_acc(acc);
    const int r = h * 64 + 16 * w + (lane >> 2), c = 2 * (lane & 3);
    for (int j = 0; j < 16; ++j)
      for (int e = 0; e < 4; ++e) {
        const int row = r + 8 * (e >> 1), col = 8 * j + c + (e & 1);
        if (col < N) D[(size_t)row * N + col] = (float)acc[4 * j + e];
      }
  }
}

// MN-major variant (the weight-gradient kernels' operand form): operands stored as buf[m/8][k][8 elements],
// i.e. D[128 x N] = sum_k At[k][m] * Bt[k][n] with both operands "transposed" in shared memory.
__global__ void __launch_bounds__(128) selftest_umma_mn_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                               float* __restrict__ D, int N, int K, int* err) {
  __shared__ __align__(128) uint8_t a_s[128 * 64 * 2];
  __shared__ __align__(128) uint8_t b_s[128 * 64 * 2];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < (int)sizeof(b_s) / 16; i += 128) reinterpret_cast<uint4*>(b_s)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    reinterpret_cast<__nv_bfloat16*>(a_s)[((size_t)(tid >> 3) * K + k) * 8 + (tid & 7)] = __float2bfloat16_rn(A[(size_t)tid * K + k]);
    if (tid < N)
      reinterpret_cast<__nv_bfloat16*>(b_s)[((size_t)(tid >> 3) * K + k) * 8 + (tid & 7)] = __float2bfloat16_rn(B[(size_t)tid * K + k]);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  for (int h = 0; h < 2; ++h) {
    float acc[64];
    tc::zero_acc(acc);
    tc::wg_fence();
    tc::fence_acc(acc);
    for (int ks = 0; ks < K / 16; ++ks) {
      const uint64_t ad = tc::smem_desc_mnmajor_noswz(tc::smem_u32(a_s) + ks * 256 + h * 8 * K * 16, 128, K * 16);
      const uint64_t bd = tc::smem_desc_mnmajor_noswz(tc::smem_u32(b_s) + ks * 256, 128, K * 16);
      tc::Mma<128>::bf16<1, 1>(acc, ad, bd, 1);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::fence_acc(acc);
    const int r = h * 64 + 16 * w + (lane >> 2), c = 2 * (lane & 3);
    for (int j = 0; j < 16; ++j)
      for (int e = 0; e < 4; ++e) {
        const int row = r + 8 * (e >> 1), col = 8 * j + c + (e & 1);
        if (col < N) D[(size_t)row * N + col] = acc[4 * j + e];
      }
  }
}

extern "C" int mnb_selftest_umma(const float* A, const float* B, float* D, int32_t N, int32_t K, int32_t int8,
                                 int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(A && B && D && err_flag, "NULL self-test pointers");
  MNB_REQUIRE(N >= 16 && N <= 128 && N % 16 == 0, "self-test N must be a multiple of 16 in [16,128]");
  MNB_REQUIRE(K >= 32 && K <= (int8 == 1 ? 128 : 64) && K % 32 == 0, "self-test K out of range");
  if (int8 == 2) {
    MNB_REQUIRE(K <= 64, "MN-major self-test K <= 64");
    selftest_umma_mn_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(A, B, D, N, K, err_flag);
  } else if (int8) selftest_umma_kernel<true><<<1, 128, 0, (cudaStream_t)stream>>>(A, B, D, N, K, err_flag);
  else selftest_umma_kernel<false><<<1, 128, 0, (cudaStream_t)stream>>>(A, B, D, N, K, err_flag);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ self-test 2: TMA box + OOB fill
__global__ void __launch_bounds__(128) selftest_tma_kernel(const __grid_constant__ CUtensorMap tmap, int c0, int c1,
                                                           int c2, int box_elems, float* __restrict__ out, int* err) {
  extern __shared__ __align__(128) uint8_t dyn[];
  __shared__ __align__(8) uint64_t bar;
  float* buf = reinterpret_cast<float*>(dyn);
  if (threadIdx.x == 0) {
    tc::mbar_init(&bar, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    tc::mbar_arrive_expect_tx(&bar, (uint32_t)box_elems * 4u);
    tc::tma_load_3d(buf, &tmap, &bar, c0, c1, c2);
  }
  bool ok = tc::mbar_wait(&bar, 0, err, 201);
  if (ok)
    for (int i = threadIdx.x; i < box_elems; i += blockDim.x) out[i] = buf[i];
}

extern "C" int mnb_selftest_tma3d(const float* src, const int64_t* dims3, const int32_t* box3, const int32_t* coord3,
                                  float* out, int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(src && dims3 && box3 && coord3 && out && err_flag, "NULL self-test pointers");
  CUtensorMap tmap;
  uint64_t dims[3] = {(uint64_t)dims3[0], (uint64_t)dims3[1], (uint64_t)dims3[2]};
  uint32_t box[3] = {(uint32_t)box3[0], (uint32_t)box3[1], (uint32_t)box3[2]};
  if (int e = mnb_make_tmap(&tmap, src, 4, 3, dims, box)) return e;
  int elems = box3[0] * box3[1] * box3[2];
  MNB_REQUIRE(elems * 4 <= 48 * 1024, "self-test box too large");
  selftest_tma_kernel<<<1, 128, elems * 4, (cudaStream_t)stream>>>(tmap, coord3[0], coord3[1], coord3[2], elems, out,
                                                                    err_flag);
  MNB_LAUNCHED(1);
  return 0;
}


// ------------------------------------------------------------------ micro-benchmark: MMA issue / execution rate
// `iters` back-to-back wgmma (M=64, N, K=16, bf16, no-swizzle operands of zeros) from one warpgroup into one register
// accumulator; A start address shifted by `a_shift16` 16-byte units.
// out[0] = SM cycles from first issue until the last MMA retired, out[1] = cycles spent issuing.
template <int N>
__global__ void __launch_bounds__(128) mma_rate_kernel(int a_shift16, int iters, int mn_major, long long* out) {
  __shared__ __align__(1024) uint8_t ab[48 * 1024 - 1024];
  const int tid = threadIdx.x;
  for (int i = tid; i < (int)sizeof(ab) / 16; i += 128) reinterpret_cast<uint4*>(ab)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();
  const uint32_t a_addr = tc::smem_u32(ab) + (uint32_t)(a_shift16 % 100) * 16u, b_addr = tc::smem_u32(ab) + 24 * 1024;
  const uint64_t ad = mn_major ? tc::smem_desc_mnmajor_noswz(a_addr, 128, 136 * 16) : tc::smem_desc_kmajor_noswz(a_addr, 136 * 16, 128);
  const uint64_t bd = mn_major ? tc::smem_desc_mnmajor_noswz(b_addr, 128, 136 * 16) : tc::smem_desc_kmajor_noswz(b_addr, (uint32_t)N * 16, 128);
  float acc[N / 2];
  tc::zero_acc(acc);
  tc::wg_fence();
  tc::fence_acc(acc);
  const long long t0 = clock64();
  if (mn_major) for (int i = 0; i < iters; ++i) tc::Mma<N>::template bf16<1, 1>(acc, ad + (i & 3), bd, 1);
  else for (int i = 0; i < iters; ++i) tc::Mma<N>::template bf16<0, 0>(acc, ad + (i & 3), bd, 1);
  const long long t1 = clock64();
  tc::wg_commit();
  tc::wg_wait<0>();
  tc::fence_acc(acc);
  const long long t2 = clock64();
  if (tid == 0) { out[0] = acc[0] == 0.f ? (t2 - t0) : -1; out[1] = t1 - t0; }
}

extern "C" int mnb_selftest_mma_rate(int32_t N, int32_t n_acc, int32_t a_shift16, int32_t iters, int32_t mn_major,
                                     int64_t* out2, int32_t* err_flag, mnb_stream_t stream) {
  MNB_REQUIRE(out2 && err_flag && n_acc >= 1 && iters >= 0, "bad mma_rate arguments");
  long long* o = reinterpret_cast<long long*>(out2);
  cudaStream_t st = (cudaStream_t)stream;
  switch (N) {
    case 32: mma_rate_kernel<32><<<1, 128, 0, st>>>(a_shift16, iters, mn_major, o); break;
    case 64: mma_rate_kernel<64><<<1, 128, 0, st>>>(a_shift16, iters, mn_major, o); break;
    case 128: mma_rate_kernel<128><<<1, 128, 0, st>>>(a_shift16, iters, mn_major, o); break;
    default: return mnb_fail(MNB_E_UNSUPPORTED, "mma_rate: N must be 32, 64 or 128");
  }
  MNB_LAUNCHED(1);
  return 0;
}
