// Quantizer / observer kernels of the fake-quant hot path (HBM-bound elementwise + reductions).
// Reference semantics: DF:11-73, WB:11-149, IAO:15-321 (see include/micronet_b200.h).
#include <math.h>
#include <stdarg.h>
#include <stdio.h>

#include <atomic>

#include "mnb_common.cuh"

// ------------------------------------------------------------------ error plumbing
static thread_local char g_mnb_err[512] = "";
static std::atomic<int64_t> g_mnb_launches{0};

int mnb_fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_mnb_err, sizeof(g_mnb_err), fmt, ap);
  va_end(ap);
  return code;
}
void mnb_count_launches(int n) { g_mnb_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" int mnb_version(void) { return 100; }
extern "C" const char* mnb_last_error(void) { return g_mnb_err; }
extern "C" int64_t mnb_launch_count(void) { return g_mnb_launches.load(); }

static inline cudaStream_t S(mnb_stream_t s) { return (cudaStream_t)s; }

// ------------------------------------------------------------------ activation fake-quant
// Each warp owns 128 consecutive elements: lane l touches l, l+32, l+64, l+96 (coalesced 128 B
// loads, 32 B code stores, one ballot word per 32 elements).  5.125 B/element of HBM traffic.
__global__ void __launch_bounds__(256) act_quant_fwd_kernel(const float* __restrict__ x, int64_t n,
                                                            mnb_act_qparams p, uint8_t* __restrict__ codes,
                                                            uint32_t* __restrict__ bits,
                                                            float* __restrict__ xq) {
  const MnbActQ q = mnb_load_actq(p);
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * 128; base < n; base += nwarps * 128) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t i = base + lane + 32 * j;
      v[j] = (i < n) ? __ldg(x + i) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t i = base + lane + 32 * j;
      bool pass;
      const int c = mnb_act_code_certified(q, v[j], pass);  // bit-identical to mnb_act_quantize_one
      float o;
      if (q.mode == MNB_ACT_DOREFA) o = __fmul_rn((float)c, q.s);
      else if (q.mode == MNB_ACT_IAO) o = __fmul_rn(__fadd_rn((float)(c + q.qmin), q.zp), q.s);
      else o = c ? 1.f : -1.f;
      bool live = i < n;
      uint32_t word = __ballot_sync(0xffffffffu, live && pass);
      if (live) {
        if (codes) codes[i] = (uint8_t)c;
        if (xq) xq[i] = o;
      }
      if (bits && lane == 0 && (base + 32 * j) < n) bits[(base >> 5) + j] = word;
    }
  }
}

__global__ void __launch_bounds__(256) act_quant_bwd_kernel(const float* __restrict__ g,
                                                            const uint32_t* __restrict__ bits, int64_t n,
                                                            mnb_act_qparams p, float* __restrict__ dx) {
  const MnbActQ q = mnb_load_actq(p);
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    bool pass = (__ldg(bits + (i >> 5)) >> (i & 31)) & 1u;
    dx[i] = mnb_act_ste_one(q, __ldg(g + i), pass);
  }
}

static int check_actq(const mnb_act_qparams* qp) {
  MNB_REQUIRE(qp != nullptr, "act qparams is NULL");
  if (qp->mode == MNB_ACT_DOREFA) {
    MNB_REQUIRE(qp->bits >= 2 && qp->bits <= 8, "DoReFa a_bits must be in [2,8] for the CUDA path, got %d", qp->bits);
  } else if (qp->mode == MNB_ACT_IAO) {
    MNB_REQUIRE(qp->scale && qp->zero_point && qp->obs_min && qp->obs_max, "IAO qparams pointers are NULL");
    MNB_REQUIRE(qp->qmax > qp->qmin && qp->qmax - qp->qmin <= 255, "IAO level range [%d,%d] does not fit u8 codes", qp->qmin, qp->qmax);
  } else {
    MNB_REQUIRE(qp->mode == MNB_ACT_SIGN, "unknown activation quantizer mode %d", qp->mode);
  }
  return 0;
}

extern "C" int mnb_act_quant_fwd(const float* x, int64_t n, const mnb_act_qparams* qp, uint8_t* codes,
                                 uint32_t* pass_bits, float* xq, mnb_stream_t stream) {
  if (int e = check_actq(qp)) return e;
  MNB_REQUIRE(x != nullptr && n >= 0, "x is NULL or n < 0");
  if (n == 0) return 0;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  act_quant_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(x, n, *qp, codes, pass_bits, xq);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_act_quant_bwd(const float* g, const uint32_t* pass_bits, int64_t n,
                                 const mnb_act_qparams* qp, float* dx, mnb_stream_t stream) {
  if (int e = check_actq(qp)) return e;
  MNB_REQUIRE(g && pass_bits && dx && n >= 0, "NULL pointer");
  if (n == 0) return 0;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  act_quant_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(g, pass_bits, n, *qp, dx);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ observers + qparams
struct ObsCfg {
  int kind, first, update_q, symmetric, qmin, qmax;
  float c_prev, c_cur;  // (float)(1 - momentum), (float)momentum
};

__device__ __forceinline__ void observer_update_row(const ObsCfg& c, float cur_min, float cur_max,
                                                    float* min_val, float* max_val, float* scale,
                                                    float* zero_point, bool touch_min) {
  float mn = cur_min, mx = cur_max;
  if (!c.first) {
    if (c.kind == 0) {  // MinMaxObserver IAO:70-72
      mn = fminf(cur_min, *min_val);
      mx = fmaxf(cur_max, *max_val);
    } else {  // EMA IAO:110-111 / 138
      mn = __fadd_rn(__fmul_rn(c.c_prev, *min_val), __fmul_rn(c.c_cur, cur_min));
      mx = __fadd_rn(__fmul_rn(c.c_prev, *max_val), __fmul_rn(c.c_cur, cur_max));
    }
  }
  if (touch_min) *min_val = mn; else mn = *min_val;  // HistogramObserver never writes min_val
  *max_val = mx;
  if (!c.update_q) return;
  const float span = (float)(c.qmax - c.qmin);
  float s, zp;
  if (c.symmetric) {  // IAO:292-305
    float fr = fmaxf(fabsf(mn), fabsf(mx));
    s = fmaxf(__fdiv_rn(fr, (float)((double)span / 2.0)), FLT_EPSILON);
    zp = 0.f;
  } else {  // IAO:309-321
    s = fmaxf(__fdiv_rn(__fsub_rn(mx, mn), span), FLT_EPSILON);
    zp = mnb_sign0(mn) * floorf(__fadd_rn(fabsf(__fdiv_rn(mn, s)), 0.5f));
  }
  *scale = s;
  *zero_point = zp;
}

// scratch layout (bytes): [0,4) block counter | [64, 64+4*MAXB) partial min | then partial max
constexpr int OBS_MAXB = 1024;

__global__ void __launch_bounds__(256) observe_global_kernel(const float* __restrict__ x, int64_t n, ObsCfg c,
                                                             float* min_val, float* max_val, float* scale,
                                                             float* zero_point, uint32_t* scratch) {
  __shared__ float red[32];
  __shared__ bool last;
  float mn = FLT_MAX, mx = -FLT_MAX;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float v = __ldg(x + i);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  mn = mnb_block_reduce(mn, MnbMin(), FLT_MAX, red);
  mx = mnb_block_reduce(mx, MnbMax(), -FLT_MAX, red);
  float* pmin = reinterpret_cast<float*>(scratch + 16);
  float* pmax = pmin + OBS_MAXB;
  if (threadIdx.x == 0) {
    pmin[blockIdx.x] = mn;
    pmax[blockIdx.x] = mx;
    __threadfence();
    last = (atomicAdd(scratch, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  mn = FLT_MAX; mx = -FLT_MAX;
  for (int b = threadIdx.x; b < gridDim.x; b += blockDim.x) {
    mn = fminf(mn, pmin[b]);
    mx = fmaxf(mx, pmax[b]);
  }
  mn = mnb_block_reduce(mn, MnbMin(), FLT_MAX, red);
  mx = mnb_block_reduce(mx, MnbMax(), -FLT_MAX, red);
  if (threadIdx.x == 0) {
    observer_update_row(c, mn, mx, min_val, max_val, scale, zero_point, true);
    scratch[0] = 0;  // re-arm
  }
}

// per-row (out-channel) ranges of a weight tensor: one block per row.
__global__ void __launch_bounds__(128) observe_rows_kernel(const float* __restrict__ x, int64_t inner, ObsCfg c,
                                                           float* min_val, float* max_val, float* scale,
                                                           float* zero_point) {
  __shared__ float red[32];
  const int r = blockIdx.x;
  const float* row = x + (int64_t)r * inner;
  float mn = FLT_MAX, mx = -FLT_MAX;
  for (int64_t i = threadIdx.x; i < inner; i += blockDim.x) {
    float v = __ldg(row + i);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  mn = mnb_block_reduce(mn, MnbMin(), FLT_MAX, red);
  mx = mnb_block_reduce(mx, MnbMax(), -FLT_MAX, red);
  if (threadIdx.x == 0)
    observer_update_row(c, mn, mx, min_val + r, max_val + r, scale ? scale + r : nullptr,
                        zero_point ? zero_point + r : nullptr, true);
}

// ---- percentile (k-th smallest |x|) by 4-pass MSB-first radix select on the fp32 bit pattern ----
// scratch: [256, 256+4*256) u32 histograms (zero on entry; re-zeroed by the finalize kernel)
__device__ __forceinline__ void radix_prefix(const uint32_t* hist, int pass, uint64_t k, uint32_t& prefix,
                                             uint64_t& krem) {
  prefix = 0; krem = k;  // k is 1-indexed
  for (int p = 0; p < pass; ++p) {
    const uint32_t* h = hist + p * 256;
    uint64_t acc = 0; int d = 0;
    for (; d < 256; ++d) {
      uint64_t cnt = h[d];
      if (acc + cnt >= krem) break;
      acc += cnt;
    }
    krem -= acc;
    prefix = (prefix << 8) | (uint32_t)d;
  }
}

__global__ void __launch_bounds__(256) radix_hist_kernel(const float* __restrict__ x, int64_t n, int pass,
                                                         uint64_t k, uint32_t* hist) {
  __shared__ uint32_t sh[256];
  __shared__ uint32_t s_prefix;
  sh[threadIdx.x] = 0;
  if (threadIdx.x == 0) { uint32_t pf; uint64_t kr; radix_prefix(hist, pass, k, pf, kr); s_prefix = pf; }
  __syncthreads();
  const uint32_t prefix = s_prefix;
  const int shift = 24 - 8 * pass;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint32_t u = __float_as_uint(fabsf(__ldg(x + i)));
    bool match = (pass == 0) || ((u >> (shift + 8)) == prefix);
    if (match) atomicAdd(&sh[(u >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&hist[pass * 256 + threadIdx.x], sh[threadIdx.x]);
}

__global__ void radix_finalize_kernel(uint64_t k, ObsCfg c, float* min_val, float* max_val, float* scale,
                                      float* zero_point, uint32_t* hist) {
  if (threadIdx.x == 0) {
    uint32_t pf; uint64_t kr;
    radix_prefix(hist, 4, k, pf, kr);
    float kth = __uint_as_float(pf);
    observer_update_row(c, 0.f, kth, min_val, max_val, scale, zero_point, false);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) hist[i] = 0;
}

extern "C" int64_t mnb_observe_scratch_bytes(int64_t n, int32_t rows) {
  (void)n;
  // [0,16K): block counter, min/max partials, 4x256 radix histograms
  // [16K,48K): per-channel completion counters of channel_stats (fixed size: the layout must not
  //            depend on the channel count, or one call's partial sums alias another call's counters)
  // [48K,...): channel_stats partial sums, rows * 32 splits * 2 doubles
  return 49152 + (int64_t)rows * (32 * 16);
}

extern "C" int mnb_iao_observe(const float* x, int64_t n, int32_t rows, int32_t observer_kind, int32_t first,
                               double momentum, double percentile, float* min_val, float* max_val,
                               int32_t update_qparams, int32_t symmetric, int32_t qmin, int32_t qmax,
                               float* scale, float* zero_point, void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(x && min_val && max_val && n > 0 && rows >= 1 && n % rows == 0, "bad observer arguments");
  MNB_REQUIRE(observer_kind >= 0 && observer_kind <= 2, "observer kind %d", observer_kind);
  MNB_REQUIRE(!update_qparams || (scale && zero_point && qmax > qmin), "qparams buffers missing");
  ObsCfg c{observer_kind, first, update_qparams, symmetric, qmin, qmax, (float)(1.0 - momentum), (float)momentum};
  if (observer_kind == 2) {
    MNB_REQUIRE(rows == 1 && scratch, "percentile observer is per-layer and needs scratch");
    int64_t k = (int64_t)(percentile * (double)n);  // Python: int(percentile * numel)
    MNB_REQUIRE(k >= 1 && k <= n, "kthvalue: k=%lld out of range for n=%lld", (long long)k, (long long)n);
    uint32_t* hist = reinterpret_cast<uint32_t*>(scratch) + 2560;  // past the min/max partials
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 8), MNB_NUM_SMS * 4);
    for (int pass = 0; pass < 4; ++pass)
      radix_hist_kernel<<<blocks, 256, 0, S(stream)>>>(x, n, pass, (uint64_t)k, hist);
    radix_finalize_kernel<<<1, 256, 0, S(stream)>>>((uint64_t)k, c, min_val, max_val, scale, zero_point, hist);
    MNB_LAUNCHED(5);
    return 0;
  }
  if (rows == 1) {
    MNB_REQUIRE(scratch != nullptr, "global observer needs scratch");
    int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 8), OBS_MAXB);
    observe_global_kernel<<<blocks, 256, 0, S(stream)>>>(x, n, c, min_val, max_val, scale, zero_point,
                                                          reinterpret_cast<uint32_t*>(scratch));
  } else {
    observe_rows_kernel<<<rows, 128, 0, S(stream)>>>(x, n / rows, c, min_val, max_val, scale, zero_point);
  }
  MNB_LAUNCHED(1);
  return 0;
}

__global__ void update_qparams_kernel(float* min_val, float* max_val, int rows, ObsCfg c, float* scale,
                                      float* zero_point) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  c.first = 1;  // keep the observed range untouched: "first" branch copies cur -> stored
  observer_update_row(c, min_val[r], max_val[r], min_val + r, max_val + r, scale + r, zero_point + r, true);
}

extern "C" int mnb_iao_update_qparams(const float* min_val, const float* max_val, int32_t rows,
                                      int32_t symmetric, int32_t qmin, int32_t qmax, float* scale,
                                      float* zero_point, mnb_stream_t stream) {
  MNB_REQUIRE(min_val && max_val && scale && zero_point && rows >= 1 && qmax > qmin, "bad qparams arguments");
  ObsCfg c{0, 1, 1, symmetric, qmin, qmax, 0.f, 0.f};
  update_qparams_kernel<<<mnb_ceil_div(rows, 128), 128, 0, S(stream)>>>(
      const_cast<float*>(min_val), const_cast<float*>(max_val), rows, c, scale, zero_point);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ DoReFa weight quantizer (DF:61-73)
// aux layout: [0,numel) tanh(w) | numel+0: m = max|t| | numel+1: number of elements attaining it
__global__ void __launch_bounds__(256) dorefa_w_tanh_max_kernel(const float* __restrict__ w, int64_t n,
                                                                float* __restrict__ aux, uint32_t* scratch) {
  __shared__ float red[32];
  __shared__ bool last;
  float m = 0.f;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    // correctly-rounded fp32 tanh via fp64 (ATen-CPU uses Sleef, <= 1 ulp from this; SURVEY §7.2.1d)
    float t = (float)tanh((double)__ldg(w + i));
    aux[i] = t;
    m = fmaxf(m, fabsf(t));
  }
  m = mnb_block_reduce(m, MnbMax(), 0.f, red);
  float* pmax = reinterpret_cast<float*>(scratch + 16);
  if (threadIdx.x == 0) {
    pmax[blockIdx.x] = m;
    __threadfence();
    last = (atomicAdd(scratch, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  m = 0.f;
  for (int b = threadIdx.x; b < gridDim.x; b += blockDim.x) m = fmaxf(m, pmax[b]);
  m = mnb_block_reduce(m, MnbMax(), 0.f, red);
  if (threadIdx.x == 0) { aux[n] = m; aux[n + 1] = 0.f; scratch[0] = 0; }
}

__global__ void __launch_bounds__(256) dorefa_w_quant_kernel(int64_t n, int out_c, int w_bits,
                                                             float* __restrict__ aux, int16_t* __restrict__ w_int,
                                                             float* __restrict__ w_scale, float* __restrict__ wq) {
  const int L = (1 << w_bits) - 1;
  const float s = (float)(1.0 / (double)L);
  const float m = aux[n];
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int ties = 0;
  for (; i < n; i += stride) {
    float t = aux[i];
    if (fabsf(t) == m) ++ties;
    float o = __fadd_rn(__fdiv_rn(__fmul_rn(t, 0.5f), m), 0.5f);  // t / 2 / max|t| + 0.5
    float kf = mnb_round_half_away(__fdiv_rn(o, s));
    float q = __fmul_rn(kf, s);
    if (wq) wq[i] = __fsub_rn(__fmul_rn(2.f, q), 1.f);
    if (w_int) w_int[i] = (int16_t)(2 * (int)kf - L);
    if (w_scale && i < out_c) w_scale[i] = s;
  }
  ties = mnb_warp_reduce(ties, MnbSum());
  if ((threadIdx.x & 31) == 0 && ties) atomicAdd(aux + n + 1, (float)ties);
}

extern "C" int mnb_dorefa_weight_fwd(const float* w, int64_t numel, int32_t out_c, int32_t w_bits,
                                     int16_t* w_int, float* w_scale, float* wq, float* aux, void* scratch,
                                     mnb_stream_t stream) {
  MNB_REQUIRE(w && aux && scratch && numel > 0 && out_c > 0 && out_c <= numel, "bad DoReFa weight arguments");
  MNB_REQUIRE(w_bits >= 2 && w_bits <= 8, "DoReFa w_bits must be in [2,8] for the CUDA path, got %d", w_bits);
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(numel, 256), OBS_MAXB);
  dorefa_w_tanh_max_kernel<<<blocks, 256, 0, S(stream)>>>(w, numel, aux, reinterpret_cast<uint32_t*>(scratch));
  dorefa_w_quant_kernel<<<blocks, 256, 0, S(stream)>>>(numel, out_c, w_bits, aux, w_int, w_scale, wq);
  MNB_LAUNCHED(2);
  return 0;
}

// backward: wq = 2*R(o/s)*s - 1, o = (t/2)/m + 0.5, m = max|t|, t = tanh(w)
__global__ void __launch_bounds__(256) dorefa_w_bwd_reduce_kernel(const float* __restrict__ g,
                                                                  const float* __restrict__ aux, int64_t n,
                                                                  float s, double* partial, uint32_t* counter,
                                                                  double* result) {
  __shared__ double red[32];
  __shared__ bool last;
  const float m = aux[n];
  double acc = 0.0;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float G = __fdiv_rn(__fmul_rn(__fmul_rn(__ldg(g + i), 2.f), s), s);
    float a = __fmul_rn(aux[i], 0.5f);
    acc += (double)(-__fdiv_rn(__fmul_rn(G, a), __fmul_rn(m, m)));  // div backward: -grad*a/(b*b)
  }
  acc = mnb_block_reduce(acc, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = acc;
    __threadfence();
    last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  acc = 0.0;
  for (int b = threadIdx.x; b < gridDim.x; b += blockDim.x) acc += partial[b];
  acc = mnb_block_reduce(acc, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) { *result = acc; *counter = 0; }
}

__global__ void __launch_bounds__(256) dorefa_w_bwd_kernel(const float* __restrict__ g,
                                                           const float* __restrict__ aux, int64_t n, float s,
                                                           const double* dm_sum, float* __restrict__ dw) {
  const float m = aux[n];
  const float share = (float)(*dm_sum) / aux[n + 1];  // evenly split among arg-max ties (torch.max backward)
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float t = aux[i];
    float G = __fdiv_rn(__fmul_rn(__fmul_rn(__ldg(g + i), 2.f), s), s);
    float dt = __fmul_rn(__fdiv_rn(G, m), 0.5f);
    if (fabsf(t) == m) dt = __fadd_rn(dt, __fmul_rn(share, mnb_sign0(t)));
    dw[i] = __fmul_rn(dt, __fsub_rn(1.f, __fmul_rn(t, t)));
  }
}

extern "C" int mnb_dorefa_weight_bwd(const float* g_wq, const float* aux, int64_t numel, int32_t w_bits,
                                     float* dw, void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(g_wq && aux && dw && scratch && numel > 0, "bad DoReFa weight-bwd arguments");
  MNB_REQUIRE(w_bits >= 2 && w_bits <= 8, "DoReFa w_bits must be in [2,8], got %d", w_bits);
  const float s = (float)(1.0 / (double)((1 << w_bits) - 1));
  uint32_t* counter = reinterpret_cast<uint32_t*>(scratch);
  double* result = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 32);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 64);
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(numel, 256), OBS_MAXB);
  dorefa_w_bwd_reduce_kernel<<<blocks, 256, 0, S(stream)>>>(g_wq, aux, numel, s, partial, counter, result);
  dorefa_w_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(g_wq, aux, numel, s, result, dw);
  MNB_LAUNCHED(2);
  return 0;
}

// ------------------------------------------------------------------ wbwtab weight quantizer (WB:98-149)
// one block per output channel; the row (in_c_per_group * ker_hw floats) is small (<= a few K)
__global__ void __launch_bounds__(128) wb_weight_fwd_kernel(float* __restrict__ w, int cpg, int khw, int W,
                                                            int16_t* __restrict__ w_int,
                                                            float* __restrict__ w_scale, float* __restrict__ wq,
                                                            float* __restrict__ aux, int out_c) {
  __shared__ double redd[32];
  const int k = blockIdx.x;
  const int inner = cpg * khw;
  float* row = w + (int64_t)k * inner;
  if (W == 2) {
    // WB:98-102 — in place: subtract the mean over the input-channel dim (per tap), clamp to [-1,1]
    for (int rs = threadIdx.x; rs < khw; rs += blockDim.x) {
      double sum = 0.0;
      for (int c = 0; c < cpg; ++c) sum += (double)row[c * khw + rs];
      float mean = (float)(sum / (double)cpg);
      for (int c = 0; c < cpg; ++c) {
        float v = __fsub_rn(row[c * khw + rs], mean);
        row[c * khw + rs] = fminf(fmaxf(v, -1.f), 1.f);
      }
    }
    __syncthreads();
  }
  double asum = 0.0;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) asum += (double)fabsf(row[i]);
  asum = mnb_block_reduce(asum, MnbSum(), 0.0, redd);
  const float E = (float)(asum / (double)inner);  // channel-level E|w|  (WB:59 / WB:124)
  if (W == 2) {
    for (int i = threadIdx.x; i < inner; i += blockDim.x) {
      float sg = row[i] < 0.f ? -1.f : 1.f;  // sign with 0 -> +1
      int64_t o = (int64_t)k * inner + i;
      if (w_int) w_int[o] = (int16_t)sg;
      if (wq) wq[o] = __fmul_rn(sg, E);
    }
    if (threadIdx.x == 0) { if (w_scale) w_scale[k] = E; aux[k] = E; aux[out_c + k] = 0.f; aux[2 * out_c + k] = (float)inner; }
    return;
  }
  // ternary, WB:55-75 + WB:132-146
  const float thr = __fmul_rn(E, 0.7f);
  double num = 0.0; int cnt = 0;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    float a = fabsf(row[i]);
    if (a > thr) { num += (double)a; ++cnt; }
  }
  num = mnb_block_reduce(num, MnbSum(), 0.0, redd);
  double cntd = mnb_block_reduce((double)cnt, MnbSum(), 0.0, redd);
  const float alpha = __fdiv_rn((float)num, (float)cntd);
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    float v = row[i];
    float t = mnb_sign0(mnb_sign0(__fadd_rn(v, thr)) + mnb_sign0(__fadd_rn(v, -thr)));
    int64_t o = (int64_t)k * inner + i;
    if (w_int) w_int[o] = (int16_t)t;
    if (wq) wq[o] = __fmul_rn(t, alpha);
  }
  if (threadIdx.x == 0) { if (w_scale) w_scale[k] = alpha; aux[k] = alpha; aux[out_c + k] = thr; aux[2 * out_c + k] = (float)cntd; }
}

__global__ void __launch_bounds__(128) wb_weight_bwd_kernel(const float* __restrict__ g,
                                                            const float* __restrict__ w,
                                                            const float* __restrict__ aux, int inner, int W,
                                                            int out_c, float* __restrict__ dw) {
  __shared__ double redd[32];
  const int k = blockIdx.x;
  const float alpha = aux[k], thr = aux[out_c + k], cnt = aux[2 * out_c + k];
  const float* grow = g + (int64_t)k * inner;
  const float* wrow = w + (int64_t)k * inner;
  double da = 0.0;  // d alpha = sum g * level
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    float v = wrow[i];
    float lv = (W == 2) ? (v < 0.f ? -1.f : 1.f)
                        : mnb_sign0(mnb_sign0(__fadd_rn(v, thr)) + mnb_sign0(__fadd_rn(v, -thr)));
    da += (double)__fmul_rn(grow[i], lv);
  }
  da = mnb_block_reduce(da, MnbSum(), 0.0, redd);
  const float share = __fdiv_rn((float)da, cnt);  // mean / (num/cnt) backward
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    float v = wrow[i];
    bool big = (W == 2) ? true : (fabsf(v) > thr);
    float extra = big ? __fmul_rn(share, mnb_sign0(v)) : 0.f;
    dw[(int64_t)k * inner + i] = __fadd_rn(__fmul_rn(grow[i], alpha), extra);
  }
}

extern "C" int mnb_wb_weight_fwd(float* w, int32_t out_c, int32_t in_c_per_group, int32_t ker_hw, int32_t W,
                                 int16_t* w_int, float* w_scale, float* wq, float* aux, mnb_stream_t stream) {
  MNB_REQUIRE(w && aux && out_c > 0 && in_c_per_group > 0 && ker_hw > 0, "bad wbwtab weight arguments");
  MNB_REQUIRE(W == 2 || W == 3, "wbwtab W must be 2 (binary) or 3 (ternary), got %d", W);
  wb_weight_fwd_kernel<<<out_c, 128, 0, S(stream)>>>(w, in_c_per_group, ker_hw, W, w_int, w_scale, wq, aux, out_c);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_wb_weight_bwd(const float* g_wq, const float* w, const float* aux, int32_t out_c,
                                 int32_t in_c_per_group, int32_t ker_hw, int32_t W, float* dw,
                                 mnb_stream_t stream) {
  MNB_REQUIRE(g_wq && w && aux && dw && out_c > 0, "bad wbwtab weight-bwd arguments");
  MNB_REQUIRE(W == 2 || W == 3, "wbwtab W must be 2 or 3, got %d", W);
  wb_weight_bwd_kernel<<<out_c, 128, 0, S(stream)>>>(g_wq, w, aux, in_c_per_group * ker_hw, W, out_c, dw);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ IAO weight quantizer (IAO:214-240)
__global__ void __launch_bounds__(256) iao_weight_fwd_kernel(const float* __restrict__ w, int64_t n, int64_t inner,
                                                             int out_c, int rows, const float* __restrict__ scale,
                                                             const float* __restrict__ zero_point,
                                                             const float* __restrict__ obs_min,
                                                             const float* __restrict__ obs_max, int q_type,
                                                             int qmin, int qmax, int16_t* __restrict__ w_int,
                                                             float* __restrict__ w_scale, float* __restrict__ wq,
                                                             uint8_t* __restrict__ pass) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const int r = rows == 1 ? 0 : (int)(i / inner);
    const float s = __ldg(scale + r), zp = __ldg(zero_point + r);
    float a = __fsub_rn(__fdiv_rn(__ldg(obs_min + r), s), zp);
    float b = __fsub_rn(__fdiv_rn(__ldg(obs_max + r), s), zp);
    float lo, hi;
    if (q_type == 0) { hi = fmaxf(fabsf(a), fabsf(b)); lo = -hi; } else { lo = a; hi = b; }
    float v = __fsub_rn(__fdiv_rn(__ldg(w + i), s), zp);
    float rr = mnb_round_half_away(v);
    float c = fminf(fmaxf(rr, (float)qmin), (float)qmax);
    bool ok = !(v > hi) && !(v < lo) && (rr >= (float)qmin) && (rr <= (float)qmax);
    float e = __fadd_rn(c, zp);
    if (wq) wq[i] = __fmul_rn(e, s);
    if (w_int) w_int[i] = (int16_t)fminf(fmaxf(e, -32768.f), 32767.f);
    if (pass) pass[i] = ok ? 1 : 0;
    if (w_scale && i < out_c) w_scale[i] = __ldg(scale + (rows == 1 ? 0 : i));
  }
}

__global__ void __launch_bounds__(256) iao_weight_bwd_kernel(const float* __restrict__ g,
                                                             const uint8_t* __restrict__ pass,
                                                             const float* __restrict__ scale, int64_t n,
                                                             int64_t inner, int rows, float* __restrict__ dw) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const float s = __ldg(scale + (rows == 1 ? 0 : (int)(i / inner)));
    dw[i] = pass[i] ? __fdiv_rn(__fmul_rn(__ldg(g + i), s), s) : 0.f;
  }
}

extern "C" int mnb_iao_weight_fwd(const float* w, int64_t numel, int32_t out_c, int32_t rows, const float* scale,
                                  const float* zero_point, const float* obs_min, const float* obs_max,
                                  int32_t q_type, int32_t qmin, int32_t qmax, int16_t* w_int, float* w_scale,
                                  float* wq, uint8_t* pass, mnb_stream_t stream) {
  MNB_REQUIRE(w && scale && zero_point && obs_min && obs_max && numel > 0, "bad IAO weight arguments");
  MNB_REQUIRE(out_c > 0 && numel % out_c == 0 && (rows == 1 || rows == out_c), "rows must be 1 or out_c");
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(numel, 256), MNB_NUM_SMS * 8);
  iao_weight_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(w, numel, numel / out_c, out_c, rows, scale, zero_point,
                                                        obs_min, obs_max, q_type, qmin, qmax, w_int, w_scale, wq, pass);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_iao_weight_bwd(const float* g_wq, const uint8_t* pass, const float* scale, int64_t numel,
                                  int32_t out_c, int32_t rows, float* dw, mnb_stream_t stream) {
  MNB_REQUIRE(g_wq && pass && scale && dw && numel > 0 && out_c > 0 && numel % out_c == 0, "bad IAO weight-bwd arguments");
  MNB_REQUIRE(rows == 1 || rows == out_c, "rows must be 1 or out_c, got %d for out_c = %d", rows, out_c);
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(numel, 256), MNB_NUM_SMS * 8);
  iao_weight_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(g_wq, pass, scale, numel, numel / out_c, rows, dw);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ per-channel statistics (IAO:853-855)
// grid (channels, splits): fp64 partial sums, last split-block of a channel finalises.
constexpr int STATS_SPLITS = 32;

struct MnbBnUpdate {
  double eps; float momentum;
  float* running_mean; float* running_var; long long* num_batches_tracked;
};

__global__ void __launch_bounds__(256) channel_stats_kernel(const float* __restrict__ x, int batch, int channels,
                                                            int hw, int as_mean_var, float* __restrict__ stats,
                                                            uint32_t* counters, double* partial, MnbBnUpdate bn) {
  __shared__ double red[32];
  __shared__ bool last;
  const int c = blockIdx.x, sp = blockIdx.y, nsp = gridDim.y;
  const int64_t per = (int64_t)batch * hw;
  double s1 = 0.0, s2 = 0.0;
  // Sums are taken of (x - pivot), pivot = the channel's first value: sum(x^2) - N mean^2 in fp32 partials cancels
  // catastrophically when |mean| >> std (a conv with a large bias); the shifted form is exact to fp32 rounding of the
  // deviations (as_mean_var == 0, plain sums for bias gradients, keeps pivot 0).
  const float pivot = as_mean_var ? __ldg(x + (int64_t)c * hw) : 0.f;
  // images [b_lo, b_hi) of this split.  The (image, offset) pairs of the split are walked as one flat index
  // space so that small planes (8x8) still keep every thread loading; fp32 partials per thread, fp64 across.
  const int b_lo = (int)((int64_t)batch * sp / nsp), b_hi = (int)((int64_t)batch * (sp + 1) / nsp);
  const bool vec = (hw & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  if (vec) {
    const uint32_t hw4 = (uint32_t)hw >> 2, total = (uint32_t)(b_hi - b_lo) * hw4;
    const float4* base = reinterpret_cast<const float4*>(x);
    float f1[4] = {0.f, 0.f, 0.f, 0.f}, f2[4] = {0.f, 0.f, 0.f, 0.f};
    for (uint32_t t0 = threadIdx.x; t0 < total; t0 += 4 * blockDim.x) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t t = t0 + u * blockDim.x;
        if (t < total) {
          const uint32_t b = t / hw4, i = t - b * hw4;
          float4 v = __ldg(base + ((int64_t)(b_lo + b) * channels + c) * hw4 + i);
          v.x -= pivot; v.y -= pivot; v.z -= pivot; v.w -= pivot;
          f1[u] += (v.x + v.y) + (v.z + v.w);
          f2[u] += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
        }
      }
    }
    s1 = ((double)f1[0] + (double)f1[1]) + ((double)f1[2] + (double)f1[3]);
    s2 = ((double)f2[0] + (double)f2[1]) + ((double)f2[2] + (double)f2[3]);
  } else {
    for (int b = b_lo; b < b_hi; ++b) {
      const float* plane = x + ((int64_t)b * channels + c) * hw;
      float f1 = 0.f, f2 = 0.f;
      for (int i = threadIdx.x; i < hw; i += blockDim.x) {
        const float v = __ldg(plane + i) - pivot;
        f1 += v; f2 += v * v;
      }
      s1 += (double)f1;
      s2 += (double)f2;
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
  if (as_mean_var) {
    const double dmean = s1 / (double)per;          // mean of the deviations from the pivot
    double mean = (double)pivot + dmean;
    double ss = s2 - (double)per * dmean * dmean;
    if (ss < 0.0) ss = 0.0;
    double var = ss / (double)(per - 1);  // unbiased (torch.var default)
    stats[c] = (float)mean;
    if (as_mean_var == 2) {  // batch-norm flavour: biased variance for normalisation, unbiased for the running estimate
      stats[channels + c] = (float)(ss / (double)per);
      stats[2 * channels + c] = (float)var;
    } else if (as_mean_var == 3) {
      // nn.BatchNorm2d training step in the finaliser: invstd for the normalisation, running statistics updated
      // with the module's momentum (running = (1 - m) * running + m * batch; unbiased variance), step counter
      stats[channels + c] = (float)(1.0 / sqrt(ss / (double)per + bn.eps));
      const float m = bn.momentum;
      bn.running_mean[c] = __fadd_rn(__fmul_rn(1.f - m, bn.running_mean[c]), __fmul_rn(m, (float)mean));
      bn.running_var[c] = __fadd_rn(__fmul_rn(1.f - m, bn.running_var[c]), __fmul_rn(m, (float)var));
      if (c == 0 && bn.num_batches_tracked) *bn.num_batches_tracked += 1;
    } else {
      stats[channels + c] = (float)var;
    }
  } else {
    stats[c] = (float)s1;
    stats[channels + c] = (float)s2;
  }
  counters[c] = 0;
}

__global__ void __launch_bounds__(256) channel_stats_bwd_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ mean,
                                                                const float* __restrict__ dmean,
                                                                const float* __restrict__ dvar, int batch,
                                                                int channels, int hw, float* __restrict__ dx) {
  const int64_t n = (int64_t)batch * channels * hw;
  const float N = (float)((int64_t)batch * hw);
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    int c = (int)((i / hw) % channels);
    float a = __fdiv_rn(__ldg(dmean + c), N);
    float b = __fmul_rn(__ldg(dvar + c), __fdiv_rn(2.f, N - 1.f));
    dx[i] = __fadd_rn(a, __fmul_rn(b, __fsub_rn(__ldg(x + i), __ldg(mean + c))));
  }
}

extern "C" int mnb_channel_stats(const float* x, int32_t batch, int32_t channels, int32_t hw,
                                 int32_t as_mean_var, float* stats, void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(x && stats && scratch && batch > 0 && channels > 0 && hw > 0, "bad channel_stats arguments");
  MNB_REQUIRE(channels <= 8192, "channel_stats supports at most 8192 channels, got %d", channels);
  int64_t per = (int64_t)batch * hw;
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(STATS_SPLITS, batch), per / 2048));
  splits = std::max(1, std::min(splits, (2 * 8 * MNB_NUM_SMS + channels - 1) / channels));  // ~2 waves of fat blocks
  uint32_t* counters = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(scratch) + 16384);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 49152);
  MNB_REQUIRE(as_mean_var >= 0 && as_mean_var <= 2, "as_mean_var must be 0, 1 or 2");
  channel_stats_kernel<<<dim3(channels, splits), 256, 0, S(stream)>>>(x, batch, channels, hw, as_mean_var, stats,
                                                                       counters, partial, MnbBnUpdate{});
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_batch_stats(const float* x, int32_t batch, int32_t channels, int32_t hw, double eps, double momentum,
                                  float* running_mean, float* running_var, int64_t* num_batches_tracked,
                                  float* mean_invstd, void* scratch, mnb_stream_t stream) {
  MNB_REQUIRE(x && running_mean && running_var && mean_invstd && scratch && batch > 0 && channels > 0 && hw > 0,
              "bad bn_batch_stats arguments");
  MNB_REQUIRE(channels <= 8192, "bn_batch_stats supports at most 8192 channels, got %d", channels);
  MNB_REQUIRE((int64_t)batch * hw > 1, "batch statistics need more than one value per channel");
  int64_t per = (int64_t)batch * hw;
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(STATS_SPLITS, batch), per / 2048));
  splits = std::max(1, std::min(splits, (2 * 8 * MNB_NUM_SMS + channels - 1) / channels));  // ~2 waves of fat blocks
  uint32_t* counters = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(scratch) + 16384);
  double* partial = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 49152);
  MnbBnUpdate bn{eps, (float)momentum, running_mean, running_var, reinterpret_cast<long long*>(num_batches_tracked)};
  channel_stats_kernel<<<dim3(channels, splits), 256, 0, S(stream)>>>(x, batch, channels, hw, 3, mean_invstd, counters,
                                                                       partial, bn);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_channel_stats_bwd(const float* x, const float* mean, const float* dmean, const float* dvar,
                                     int32_t batch, int32_t channels, int32_t hw, float* dx,
                                     mnb_stream_t stream) {
  MNB_REQUIRE(x && mean && dmean && dvar && dx && batch > 0 && channels > 0 && hw > 0, "bad channel_stats_bwd arguments");
  int64_t n = (int64_t)batch * channels * hw;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  channel_stats_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(x, mean, dmean, dvar, batch, channels, hw, dx);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ fused Adam over a flat parameter bucket
// torch.optim.Adam (no amsgrad, L2 weight decay folded into the gradient) on one contiguous fp32 buffer:
// the optimizer step of the QAT loop (wbwtab/main.py:84, one param group per tensor with identical
// hyper-parameters) as a single HBM-bound launch instead of ~5 launches per parameter tensor.
__global__ void __launch_bounds__(256) adam_step_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                        float lr, float b1, float b2, float eps, float wd,
                                                        float bc1, float sqrt_bc2) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float step_size = lr / bc1;
  for (; i < n; i += stride) {
    float gi = g[i];
    const float pi = p[i];
    if (wd != 0.f) gi = fmaf(wd, pi, gi);
    const float mi = m[i] + (gi - m[i]) * (1.f - b1);          // exp_avg.lerp_(grad, 1 - beta1)
    const float vi = fmaf(1.f - b2, gi * gi, v[i] * b2);       // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(vi) / sqrt_bc2 + eps;
    m[i] = mi; v[i] = vi;
    p[i] = pi - step_size * (mi / denom);
  }
}

extern "C" int mnb_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int32_t step, mnb_stream_t stream) {
  MNB_REQUIRE(p && g && m && v && n >= 0 && step >= 1, "bad Adam arguments");
  if (n == 0) return 0;
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float sqrt_bc2 = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256), MNB_NUM_SMS * 8);
  adam_step_kernel<<<blocks, 256, 0, S(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, sqrt_bc2);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ IAO QuantAdd (IAO:1441-1498), one pass
// out = Q(a) + Q(b) with the shared (union-range) quantizer: one read of each addend, one write of the sum, the two
// STE pass masks for the backward pass.  Replaces two fake-quant launches and the ATen add (5 launches with their
// intermediate tensors); the arithmetic per element is that of act_quant_fwd_kernel followed by __fadd_rn.
__global__ void __launch_bounds__(256) quant_add_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                            int64_t n, mnb_act_qparams p, float* __restrict__ out,
                                                            uint32_t* __restrict__ bits_a, uint32_t* __restrict__ bits_b,
                                                            int relu) {
  const MnbActQ q = mnb_load_actq(p);
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * 128; base < n; base += nwarps * 128) {
    float va[4], vb[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t i = base + lane + 32 * j;
      va[j] = (i < n) ? __ldg(a + i) : 0.f;
      vb[j] = (i < n) ? __ldg(b + i) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t i = base + lane + 32 * j;
      bool pa, pb;
      const int ca = mnb_act_code_certified(q, va[j], pa), cb = mnb_act_code_certified(q, vb[j], pb);
      float oa, ob;
      if (q.mode == MNB_ACT_DOREFA) { oa = __fmul_rn((float)ca, q.s); ob = __fmul_rn((float)cb, q.s); }
      else {
        oa = __fmul_rn(__fadd_rn((float)(ca + q.qmin), q.zp), q.s);
        ob = __fmul_rn(__fadd_rn((float)(cb + q.qmin), q.zp), q.s);
      }
      const bool live = i < n;
      const uint32_t wa = __ballot_sync(0xffffffffu, live && pa), wb = __ballot_sync(0xffffffffu, live && pb);
      if (live) { const float sum = __fadd_rn(oa, ob); out[i] = relu ? fmaxf(sum, 0.f) : sum; }
      if (lane == 0 && (base + 32 * j) < n) {
        if (bits_a) bits_a[(base >> 5) + j] = wa;
        if (bits_b) bits_b[(base >> 5) + j] = wb;
      }
    }
  }
}

__global__ void __launch_bounds__(256) quant_add_bwd_kernel(const float* __restrict__ g, const uint32_t* __restrict__ bits_a,
                                                            const uint32_t* __restrict__ bits_b, int64_t n,
                                                            mnb_act_qparams p, float* __restrict__ da, float* __restrict__ db) {
  const MnbActQ q = mnb_load_actq(p);
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const float gv = __ldg(g + i);
    if (da) da[i] = mnb_act_ste_one(q, gv, (__ldg(bits_a + (i >> 5)) >> (i & 31)) & 1u);
    if (db) db[i] = mnb_act_ste_one(q, gv, (__ldg(bits_b + (i >> 5)) >> (i & 31)) & 1u);
  }
}

extern "C" int mnb_quant_add_fwd(const float* a, const float* b, int64_t n, const mnb_act_qparams* qp, float* out,
                                 uint32_t* pass_bits_a, uint32_t* pass_bits_b, int32_t relu, mnb_stream_t stream) {
  if (int e = check_actq(qp)) return e;
  MNB_REQUIRE(qp->mode != MNB_ACT_SIGN, "QuantAdd takes a DoReFa or IAO quantizer");
  MNB_REQUIRE(a && b && out && n >= 0, "NULL pointer");
  if (n == 0) return 0;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  quant_add_fwd_kernel<<<blocks, 256, 0, S(stream)>>>(a, b, n, *qp, out, pass_bits_a, pass_bits_b, relu);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_quant_add_bwd(const float* g, const uint32_t* pass_bits_a, const uint32_t* pass_bits_b, int64_t n,
                                 const mnb_act_qparams* qp, float* da, float* db, mnb_stream_t stream) {
  if (int e = check_actq(qp)) return e;
  MNB_REQUIRE(g && n >= 0 && (da == nullptr || pass_bits_a) && (db == nullptr || pass_bits_b), "NULL pointer");
  if (n == 0) return 0;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256 * 4), MNB_NUM_SMS * 8);
  quant_add_bwd_kernel<<<blocks, 256, 0, S(stream)>>>(g, pass_bits_a, pass_bits_b, n, *qp, da, db);
  MNB_LAUNCHED(1);
  return 0;
}

// ------------------------------------------------------------------ IAO BN-fuse: fold BatchNorm into (weight, bias)
// IAO:903-945 (QuantBNFuseConv2d.forward):  ratio = gamma / sqrt(var + eps);  w_f = w * ratio[k];
// b_f = beta + (bias - mean) * ratio   (bias may be absent: beta - mean * ratio).  The reference composes this from ~10
// ATen launches per layer forward and ~25 backward (broadcast multiplies, reshapes, reductions); here it is one launch each
// way, one block per output channel.  Same operation order and roundings as the ATen composition.
__global__ void __launch_bounds__(256) bn_fold_fwd_kernel(const float* __restrict__ w, int n, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, const float* __restrict__ bias,
                                                          const float* __restrict__ mean, const float* __restrict__ var,
                                                          float eps, float* __restrict__ w_f, float* __restrict__ b_f) {
  const int k = blockIdx.x;
  const float ratio = __fdiv_rn(__ldg(gamma + k), __fsqrt_rn(__fadd_rn(__ldg(var + k), eps)));
  if (threadIdx.x == 0) {
    const float m = __ldg(mean + k);
    b_f[k] = bias ? __fadd_rn(__ldg(beta + k), __fmul_rn(__fsub_rn(__ldg(bias + k), m), ratio))
                  : __fsub_rn(__ldg(beta + k), __fmul_rn(m, ratio));
  }
  const float* wk = w + (int64_t)k * n;
  float* ok = w_f + (int64_t)k * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) ok[i] = __fmul_rn(__ldg(wk + i), ratio);
}

// backward of the fold: dw = dw_f * ratio;  dratio = sum_i dw_f * w + db_f * (bias - mean);  dgamma = dratio / sqrt(var + eps);
// dvar = -0.5 * dratio * gamma * (var + eps)^-1.5;  dmean = -db_f * ratio;  dbeta = db_f;  dbias = db_f * ratio.
// out6[k*6 ..] = {dgamma, dbeta, dbias, dmean, dvar, -}
__global__ void __launch_bounds__(256) bn_fold_bwd_kernel(const float* __restrict__ dw_f, const float* __restrict__ db_f,
                                                          const float* __restrict__ w, int n, const float* __restrict__ gamma,
                                                          const float* __restrict__ bias, const float* __restrict__ mean,
                                                          const float* __restrict__ var, float eps, float* __restrict__ dw,
                                                          float* __restrict__ out6) {
  __shared__ double red[32];
  const int k = blockIdx.x;
  const float ve = __fadd_rn(__ldg(var + k), eps);
  const float sq = __fsqrt_rn(ve);
  const float g = __ldg(gamma + k);
  const float ratio = __fdiv_rn(g, sq);
  const float* dk = dw_f + (int64_t)k * n;
  const float* wk = w + (int64_t)k * n;
  float* ok = dw ? dw + (int64_t)k * n : nullptr;
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float d = __ldg(dk + i);
    s += (double)d * (double)__ldg(wk + i);
    if (ok) ok[i] = __fmul_rn(d, ratio);
  }
  s = mnb_block_reduce(s, MnbSum(), 0.0, red);
  if (threadIdx.x == 0) {
    const float db = db_f ? __ldg(db_f + k) : 0.f;
    const float m = __ldg(mean + k);
    const float diff = bias ? __fsub_rn(__ldg(bias + k), m) : -m;
    const float dratio = (float)(s + (double)db * (double)diff);
    float* o = out6 + (int64_t)k * 6;
    o[0] = __fdiv_rn(dratio, sq);                               // dgamma
    o[1] = db;                                                  // dbeta
    o[2] = db * ratio;                                          // dbias
    o[3] = -db * ratio;                                         // dmean
    o[4] = -0.5f * dratio * g / (ve * sq);                      // dvar
    o[5] = 0.f;
  }
}

// running_mean / running_var update of QuantBNFuseConv2d (IAO:858-876): first call copies the batch statistics, later calls
// r = (1 - momentum) * r + momentum * batch   (Python doubles cast to fp32 by ATen, then mul, mul, add)
__global__ void __launch_bounds__(256) bn_fold_running_kernel(float* __restrict__ rm, float* __restrict__ rv,
                                                              const float* __restrict__ bm, const float* __restrict__ bv, int n,
                                                              float keep, float mom, int first) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (first) { rm[i] = __ldg(bm + i); rv[i] = __ldg(bv + i); }
  else {
    rm[i] = __fadd_rn(__fmul_rn(keep, rm[i]), __fmul_rn(mom, __ldg(bm + i)));
    rv[i] = __fadd_rn(__fmul_rn(keep, rv[i]), __fmul_rn(mom, __ldg(bv + i)));
  }
}

extern "C" int mnb_bn_fold_fwd(const float* w, int32_t out_c, int32_t per_channel, const float* gamma, const float* beta,
                               const float* bias, const float* mean, const float* var, double eps, float* w_fused,
                               float* b_fused, mnb_stream_t stream) {
  MNB_REQUIRE(w && gamma && beta && mean && var && w_fused && b_fused && out_c > 0 && per_channel > 0, "bad bn_fold_fwd arguments");
  bn_fold_fwd_kernel<<<out_c, 256, 0, S(stream)>>>(w, per_channel, gamma, beta, bias, mean, var, (float)eps, w_fused, b_fused);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_fold_bwd(const float* dw_fused, const float* db_fused, const float* w, int32_t out_c, int32_t per_channel,
                               const float* gamma, const float* bias, const float* mean, const float* var, double eps, float* dw,
                               float* out6, mnb_stream_t stream) {
  MNB_REQUIRE(dw_fused && w && gamma && mean && var && out6 && out_c > 0 && per_channel > 0, "bad bn_fold_bwd arguments");
  bn_fold_bwd_kernel<<<out_c, 256, 0, S(stream)>>>(dw_fused, db_fused, w, per_channel, gamma, bias, mean, var, (float)eps, dw, out6);
  MNB_LAUNCHED(1);
  return 0;
}

extern "C" int mnb_bn_fold_running(float* running_mean, float* running_var, const float* batch_mean, const float* batch_var,
                                   int32_t n, double momentum, int32_t first, mnb_stream_t stream) {
  MNB_REQUIRE(running_mean && running_var && batch_mean && batch_var && n > 0, "bad bn_fold_running arguments");
  bn_fold_running_kernel<<<mnb_ceil_div(n, 256), 256, 0, S(stream)>>>(running_mean, running_var, batch_mean, batch_var, n,
                                                                      (float)(1.0 - momentum), (float)momentum, first);
  MNB_LAUNCHED(1);
  return 0;
}
