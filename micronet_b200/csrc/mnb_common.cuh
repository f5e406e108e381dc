// Shared helpers for the micronet_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "../../include/micronet_b200.h"

int mnb_fail(int code, const char* fmt, ...);
void mnb_count_launches(int n);

#define MNB_REQUIRE(cond, ...)                            \
  do {                                                    \
    if (!(cond)) return mnb_fail(MNB_E_ARG, __VA_ARGS__); \
  } while (0)

// call after every launch: surfaces launch-configuration errors as return codes
#define MNB_LAUNCHED(nlaunch)                                                        \
  do {                                                                               \
    mnb_count_launches(nlaunch);                                                     \
    cudaError_t e__ = cudaGetLastError();                                            \
    if (e__ != cudaSuccess) return mnb_fail((int)e__, "%s:%d launch failed: %s", __FILE__, __LINE__, \
                                            cudaGetErrorString(e__));                \
  } while (0)

static inline int mnb_ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
constexpr int MNB_NUM_SMS = 132;  // H100 SXM

// ---- exact-rounding primitives (never contracted into FMA, never fast-math) ----

// sign(v) * floor(|v| + 0.5) in fp32 — DF:13-16 / IAO:158-159, including the
// fp32 double-rounding quirk (0.49999997 -> 1).  rintf/roundf are both wrong here.
__device__ __forceinline__ float mnb_round_half_away(float v) {
  float r = floorf(__fadd_rn(fabsf(v), 0.5f));
  return v > 0.f ? r : (v < 0.f ? -r : 0.f);
}
// torch.sign: -1 / 0 / +1
__device__ __forceinline__ float mnb_sign0(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// order-preserving float <-> uint32 (for atomic / integer min-max)
__device__ __forceinline__ uint32_t mnb_f2ord(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float mnb_ord2f(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

template <typename T, typename Op>
__device__ __forceinline__ T mnb_warp_reduce(T v, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide reduction; result valid in every thread.  `smem` holds >= 32 T.
template <typename T, typename Op>
__device__ __forceinline__ T mnb_block_reduce(T v, Op op, T identity, T* smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = mnb_warp_reduce(v, op);
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (lane < nw) ? smem[lane] : identity;
  r = mnb_warp_reduce(r, op);
  return r;
}
struct MnbMin { template <typename T> __device__ T operator()(T a, T b) const { return a < b ? a : b; } };
struct MnbMax { template <typename T> __device__ T operator()(T a, T b) const { return a > b ? a : b; } };
struct MnbSum { template <typename T> __device__ T operator()(T a, T b) const { return a + b; } };

// The centred gradient of the BatchNorm backward, g_masked - dbeta / N - xhat * dgamma / N, with its rounding pinned: one
// subtraction, then one fma.  Every apply pass of the fused producers (mnb_fused.cu, and the _pack passes of mnb_pk.cu that
// write the same dx as packed pieces) calls this, so they all produce the same fp32 dx bit for bit; written as a plain
// expression, nvcc's fma contraction was free to round it differently in each kernel.
__device__ __forceinline__ float bn_bwd_centre(float g, float db, float xhat, float dg) {
  return fmaf(-xhat, dg, __fsub_rn(g, db));
}

// ---- the x operand of the fused BatchNorm producers: fp32 values (XT = float), or the exact int16 accumulator codes of a
// wbwtab convolution (XT = int16_t, written by mnb_pk_conv_codes) with the per-channel decode pair dec[c] / dec[C + c] that
// conv's epilogue used: x = fmaf(code, dec[c], dec[C + c]) is the value its fp32 epilogue stores, bit for bit.  Loads are
// VEC elements wide (16 bytes of fp32 = 8 bytes of codes); nothing else of a producer depends on XT.
struct XDec { float s, b; };
template <typename XT> struct XVec;
template <> struct XVec<float> { typedef float t1; typedef float2 t2; typedef float4 t4; };
template <> struct XVec<int16_t> { typedef short t1; typedef short2 t2; typedef short4 t4; };

template <typename XT>
__device__ __forceinline__ XDec x_dec(const float* dec, int channels, int c) {
  if constexpr (sizeof(XT) == 4) return XDec{1.f, 0.f};
  else return XDec{__ldg(dec + c), __ldg(dec + channels + c)};
}
template <typename XT>
__device__ __forceinline__ float x_val(XT q, XDec d) {
  if constexpr (sizeof(XT) == 4) return q;
  else return fmaf((float)q, d.s, d.b);
}
template <int VEC, typename XT>
__device__ __forceinline__ void x_load(const XT* p, XDec d, float (&v)[VEC]) {
  if constexpr (VEC == 1) {
    v[0] = x_val<XT>(__ldg(reinterpret_cast<const typename XVec<XT>::t1*>(p)), d);
  } else if constexpr (VEC == 2) {
    const typename XVec<XT>::t2 t = __ldg(reinterpret_cast<const typename XVec<XT>::t2*>(p));
    v[0] = x_val<XT>(t.x, d); v[1] = x_val<XT>(t.y, d);
  } else {
    static_assert(VEC == 4, "x_load: 1, 2 or 4 elements");
    const typename XVec<XT>::t4 t = __ldg(reinterpret_cast<const typename XVec<XT>::t4*>(p));
    v[0] = x_val<XT>(t.x, d); v[1] = x_val<XT>(t.y, d); v[2] = x_val<XT>(t.z, d); v[3] = x_val<XT>(t.w, d);
  }
}
template <typename XT>
__device__ __forceinline__ float4 x_load4(const XT* p, XDec d) {
  float v[4];
  x_load<4>(p, d, v);
  return make_float4(v[0], v[1], v[2], v[3]);
}

// ---- the activation quantizer, shared by the standalone kernel and the fused conv loaders ----
struct MnbActQ {
  int mode, qmin, qmax;
  float s, zp, lo, hi;
  float rinv;  // fl(1 / s): reciprocal used by the certified fast path below
};

__device__ __forceinline__ MnbActQ mnb_load_actq(const mnb_act_qparams& p) {
  MnbActQ q;
  q.mode = p.mode; q.qmin = p.qmin; q.qmax = p.qmax;
  q.s = 1.f; q.zp = 0.f; q.lo = 0.f; q.hi = 0.f; q.rinv = 1.f;
  if (p.mode == MNB_ACT_DOREFA) {
    q.s = (float)(1.0 / (double)((1 << p.bits) - 1));  // Python: 1 / float(2**a - 1), cast to fp32 by ATen
  } else if (p.mode == MNB_ACT_IAO) {
    q.s = __ldg(p.scale);
    q.zp = __ldg(p.zero_point);
    float a = __fsub_rn(__fdiv_rn(__ldg(p.obs_min), q.s), q.zp);
    float b = __fsub_rn(__fdiv_rn(__ldg(p.obs_max), q.s), q.zp);
    if (p.q_type == 0) { q.hi = fmaxf(fabsf(a), fabsf(b)); q.lo = -q.hi; }
    else { q.lo = a; q.hi = b; }
  }
  q.rinv = __fdiv_rn(1.f, q.s);
  return q;
}

// returns the clamped level; sets pass (STE gradient mask) and xq (dequantized value)
__device__ __forceinline__ int mnb_act_quantize_one(const MnbActQ& q, float x, bool& pass, float& xq) {
  if (q.mode == MNB_ACT_DOREFA) {
    float t = __fmul_rn(x, 0.1f);
    pass = (t >= 0.f) && (t <= 1.f);
    float c = fminf(fmaxf(t, 0.f), 1.f);
    float r = floorf(__fadd_rn(__fdiv_rn(c, q.s), 0.5f));  // c >= 0: sign*floor(|.|+0.5)
    xq = __fmul_rn(r, q.s);
    return (int)r;
  } else if (q.mode == MNB_ACT_IAO) {
    float v = __fsub_rn(__fdiv_rn(x, q.s), q.zp);
    float r = mnb_round_half_away(v);
    float c = fminf(fmaxf(r, (float)q.qmin), (float)q.qmax);
    pass = !(v > q.hi) && !(v < q.lo) && (r >= (float)q.qmin) && (r <= (float)q.qmax);
    xq = __fmul_rn(__fadd_rn(c, q.zp), q.s);
    return (int)c - q.qmin;
  } else {  // SIGN
    bool pos = !(x < 0.f);
    pass = !(x >= 1.0f) && !(x <= -1.0f);
    xq = pos ? 1.f : -1.f;
    return pos ? 2 : 0;
  }
}

// Same level code and STE mask as mnb_act_quantize_one, without the IEEE division in the common case.
// v' = x * fl(1/s) differs from the reference's fl(x / s) by at most ~3 ulp; the rounded level (and the
// range comparisons) can only differ when v' lies within `delta` of a decision boundary, and exactly those
// elements (about 1e-4 of them) take the exact path.  The result is therefore bit-identical.
__device__ __forceinline__ int mnb_act_code_certified(const MnbActQ& q, float x, bool& pass) {
  if (q.mode == MNB_ACT_DOREFA) {
    const float t = __fmul_rn(x, 0.1f);
    pass = (t >= 0.f) && (t <= 1.f);
    const float c = fminf(fmaxf(t, 0.f), 1.f);
    const float pa = c * q.rinv;
    const float f = pa + 0.5f;
    float r = floorf(f);
    const float d = f - r, delta = 4e-7f * (pa + 1.f);
    if (d < delta || d > 1.f - delta) r = floorf(__fadd_rn(__fdiv_rn(c, q.s), 0.5f));
    return (int)r;
  } else if (q.mode == MNB_ACT_IAO) {
    const float xa = x * q.rinv;
    float v = xa - q.zp;
    const float av = fabsf(v);
    const float f = av + 0.5f;
    float ra = floorf(f);
    const float d = f - ra, delta = 4e-7f * (fabsf(xa) + fabsf(q.zp) + 1.f);
    const bool near_edge = fabsf(v - q.hi) < delta || fabsf(v - q.lo) < delta;
    if (d < delta || d > 1.f - delta || near_edge || av < delta) {
      v = __fsub_rn(__fdiv_rn(x, q.s), q.zp);
      ra = floorf(__fadd_rn(fabsf(v), 0.5f));
    }
    const float r = v > 0.f ? ra : (v < 0.f ? -ra : 0.f);
    const float cl = fminf(fmaxf(r, (float)q.qmin), (float)q.qmax);
    pass = !(v > q.hi) && !(v < q.lo) && (r >= (float)q.qmin) && (r <= (float)q.qmax);
    return (int)cl - q.qmin;
  } else {
    const bool pos = !(x < 0.f);
    pass = !(x >= 1.0f) && !(x <= -1.0f);
    return pos ? 2 : 0;
  }
}

// Same decisions as mnb_act_code_certified, returning the effective integer level AS A FLOAT (level - qmin + a_off
// arithmetic folded away: DoReFa -> k, IAO -> clamp(round(x/s - zp)), SIGN -> +-1) with no float <-> int conversions:
// the operand packers of the tensor-core path are instruction-bound, not bandwidth-bound, on the quantizer.
__device__ __forceinline__ float mnb_act_level_certified(const MnbActQ& q, float x, bool& pass) {
  if (q.mode == MNB_ACT_DOREFA) {
    const float t = __fmul_rn(x, 0.1f);
    pass = (t >= 0.f) && (t <= 1.f);
    const float c = fminf(fmaxf(t, 0.f), 1.f);
    const float pa = c * q.rinv;
    const float f = pa + 0.5f;
    float r = floorf(f);
    const float d = f - r, delta = 4e-7f * (pa + 1.f);
    if (d < delta || d > 1.f - delta) r = floorf(__fadd_rn(__fdiv_rn(c, q.s), 0.5f));
    return r;
  } else if (q.mode == MNB_ACT_IAO) {
    const float xa = x * q.rinv;
    float v = xa - q.zp;
    const float av = fabsf(v);
    const float f = av + 0.5f;
    float ra = floorf(f);
    const float d = f - ra, delta = 4e-7f * (fabsf(xa) + fabsf(q.zp) + 1.f);
    const bool near_edge = fabsf(v - q.hi) < delta || fabsf(v - q.lo) < delta;
    if (d < delta || d > 1.f - delta || near_edge || av < delta) {
      v = __fsub_rn(__fdiv_rn(x, q.s), q.zp);
      ra = floorf(__fadd_rn(fabsf(v), 0.5f));
    }
    const float r = v > 0.f ? ra : (v < 0.f ? -ra : 0.f);
    pass = !(v > q.hi) && !(v < q.lo) && (r >= (float)q.qmin) && (r <= (float)q.qmax);
    return fminf(fmaxf(r, (float)q.qmin), (float)q.qmax);
  } else {
    pass = !(x >= 1.0f) && !(x <= -1.0f);
    return !(x < 0.f) ? 1.f : -1.f;
  }
}

// Branch-free first half of mnb_act_level_certified: the provisional level / pass flag from the reciprocal product, and
// `exact` = this element sits within `delta` of a decision boundary and must be redone with the IEEE division
// (mnb_act_level_certified does that).  Callers evaluate a whole vector of elements with this straight-line code and
// take ONE rarely-taken branch for the flagged ones: with the fallback branch inside every element the epilogue cannot
// overlap the elements' dependent chains.
__device__ __forceinline__ float mnb_act_level_fast(const MnbActQ& q, float x, bool& pass, bool& exact) {
  if (q.mode == MNB_ACT_DOREFA) {
    const float t = __fmul_rn(x, 0.1f);
    pass = (t >= 0.f) && (t <= 1.f);
    const float c = fminf(fmaxf(t, 0.f), 1.f);
    const float pa = c * q.rinv;
    const float f = pa + 0.5f;
    const float r = floorf(f);
    const float d = f - r, delta = 4e-7f * (pa + 1.f);
    exact = d < delta || d > 1.f - delta;
    return r;
  } else if (q.mode == MNB_ACT_IAO) {
    const float xa = x * q.rinv;
    const float v = xa - q.zp;
    const float av = fabsf(v);
    const float f = av + 0.5f;
    const float ra = floorf(f);
    const float d = f - ra, delta = 4e-7f * (fabsf(xa) + fabsf(q.zp) + 1.f);
    // (no `av < delta` test here: it guards the SIGN of v, which only matters when ra >= 1, i.e. av >= 0.5 - and a
    // ReLU output is exactly 0 for half of its elements, every one of which would take the slow path)
    exact = d < delta || d > 1.f - delta || fabsf(v - q.hi) < delta || fabsf(v - q.lo) < delta;
    const float r = v > 0.f ? ra : (v < 0.f ? -ra : 0.f);
    pass = !(v > q.hi) && !(v < q.lo) && (r >= (float)q.qmin) && (r <= (float)q.qmax);
    return fminf(fmaxf(r, (float)q.qmin), (float)q.qmax);
  } else {
    exact = false;
    pass = !(x >= 1.0f) && !(x <= -1.0f);
    return !(x < 0.f) ? 1.f : -1.f;
  }
}

// N levels at once: straight-line fast path for all, one branch for the (about 1e-4 of the) elements that need the exact
// division.  lev[k] = effective level as a float (see mnb_act_level_certified), passbits bit k = STE pass flag.
template <int N>
__device__ __forceinline__ void mnb_act_levels(const MnbActQ& q, const float (&x)[N], float (&lev)[N], uint32_t& passbits) {
  uint32_t redo = 0;
  passbits = 0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    bool pass, exact;
    lev[k] = mnb_act_level_fast(q, x[k], pass, exact);
    passbits |= pass ? (1u << k) : 0u;
    redo |= exact ? (1u << k) : 0u;
  }
  if (redo) {
#pragma unroll 1
    for (int k = 0; k < N; ++k) {
      if (!((redo >> k) & 1u)) continue;
      bool pass;
      float xv = 0.f;            // register arrays: dynamic element k through select chains, no local memory
#pragma unroll
      for (int j = 0; j < N; ++j)
        if (j == k) xv = x[j];
      const float l = mnb_act_level_certified(q, xv, pass);
#pragma unroll
      for (int j = 0; j < N; ++j)
        if (j == k) lev[j] = l;
      passbits = (passbits & ~(1u << k)) | (pass ? (1u << k) : 0u);
    }
  }
}

__device__ __forceinline__ float mnb_act_ste_one(const MnbActQ& q, float g, bool pass) {
  if (q.mode == MNB_ACT_DOREFA) return __fmul_rn(pass ? __fdiv_rn(__fmul_rn(g, q.s), q.s) : 0.f, 0.1f);
  if (q.mode == MNB_ACT_IAO) return pass ? __fdiv_rn(__fmul_rn(g, q.s), q.s) : 0.f;
  return pass ? g : 0.f;
}
