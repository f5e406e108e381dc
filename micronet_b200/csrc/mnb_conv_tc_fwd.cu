// Fused fake-quant convolution on Hopper tensor cores (wgmma): forward and data-gradient.
//
// Both are "same"-padded stride-1 correlations of an fp32 NCHW tensor with small-integer weights:
//
//   forward : y[b, gNg+n, h, w] = bias[n] + (s_a * s_w[n]) * sum_{c,r,s} e_a[b, gCg+c, h+r-p, w+s-p] * e_w[gNg+n, c, r, s]
//   dgrad   : dx[b, gCg+c, h, w] = STE( sum_{k,r,s} (dy * s_w[k])[b, gNg+k, h+r-p, w+s-p] * e_w[gNg+k, c, R-1-r, S-1-s] )
//
// Data flow per CTA (persistent, one CTA per SM, bound to a slab of groups whose integer weights
// stay resident in shared memory as bf16):
//
//   TMA warp    : cp.async.bulk.tensor.4d box (W, TH+2p, CC, TB) of the fp32 input -> staging ring;
//                 rows above / below the image are zero-filled by the TMA unit
//   7 converter : staging fp32 -> integer level (DoReFa / IAO fake-quant) or exact 3-way bf16 split
//     warps       of a raw / pre-scaled fp32 value -> "position-major" bf16 operand
//                 op[c/8][position][8 ch], position = row*(W+2p) + col of the zero-padded tile.
//                 This IS the wgmma K-major no-swizzle canonical layout with positions as GEMM rows,
//                 so filter tap (r, s) is the same buffer with the descriptor start address moved by
//                 (r*BW + s)*16 bytes: implicit GEMM without any im2col copy.  Side outputs of the
//                 fused quantizer: u8 level codes + STE pass bits for the backward pass.
//   2 MMA       : wgmma bf16 x bf16 -> fp32 accumulators in registers, one warpgroup per 64 positions;
//     warpgroups  every operand is an exact small integer or an exact bf16 piece of an fp32 value,
//                 M = 128 positions, N = output channels of the group, K = 16 channels per MMA; then the
//                 epilogue: scale + bias (fwd) or STE mask (dgrad) -> coalesced fp32 NCHW stores
#include <cuda.h>
#include <cstdlib>
#include <cuda_bf16.h>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

namespace tcconv {

constexpr int NTHREADS = 512;
constexpr int NCONV = 224;  // converter threads (warps 1..3 and 12..15); warps 4..11 are the two MMA warpgroups
constexpr int NCW = NCONV / 32;
constexpr int MAXST = 8, BASEST = 4, MAXOP = 4;  // staging ring / operand ring: as deep as shared memory allows (plan())
constexpr int kMaxNG = 160;  // output channels per group: the accumulator row of one thread is NG / 2 registers
constexpr int KMAX = 6;     // operand entries per converter thread and chunk
constexpr int kMaxDynSmem = 227 * 1024 - 6144;  // 227 KB per CTA minus the static block below (5 KB)
constexpr int kStgBytes = 2 * 32 * 68 * 4;        // two 64 x 32 epilogue staging tiles (tc::kStageLd64)
constexpr int kPlanSmem = kMaxDynSmem - kStgBytes;

struct Params {
  // tensors: input [B, Cin, H, W], output [B, Cout, H, W]
  int B, Cin, Cout, H, W, R, S, pad, G, cin_g, cout_g;
  int BW, TH, THH, TB, CC, nchunk, nst, nop;
  int npos_in, row_tiles, n_tiles, slab_groups, n_slabs;
  int quant_mode;   // 0: raw fp32 input (exact 3-term split); else MNB_ACT_DOREFA / MNB_ACT_IAO
  int dgrad;        // 1: weights transposed + flipped, per-input-channel pre-scale, STE epilogue
  int dbg;          // MNB_TC_DEBUG (timing experiments only): 1 no converter fence, 2 no converter work, 4 no epilogue stores, 8 no MMAs
  int a_offset;
  int stage_bytes, op_term_bytes, op_buf_bytes, b_group_bytes, off_stage, off_op, off_b, off_stg;
  float a_scale_const;
  mnb_act_qparams qp;
  const int16_t* w_int;     // [K, Cg, R, S] integer weights (K = fwd output channels)
  const uint8_t* w_pack;    // bf16 B-operand image [g][tap][k/8][n][8], written by pack_b_kernel
  const float* w_scale;     // [K]
  const float* a_scale;     // device scalar (IAO) or NULL
  const float* bias;        // fwd only
  const uint32_t* ste_bits; // dgrad only (may be NULL: plain dgrad)
  float* out;
  uint8_t* codes; uint32_t* pass_bits;  // fwd side outputs of the fused quantizer
  int* err;
  long long* prof;  // optional debug counters (cycles): see mnb_set_tc_profile_buffer
  // per (tap, k-step): start-address offsets (16-byte units) of the A and B operands.  Kept in the kernel parameters
  // (constant bank), NOT in shared memory: the MMA warps' descriptor arithmetic then stays in uniform registers.
  uint2 mma_off[64];
};

struct alignas(16) Shared {
  uint64_t stage_full[MAXST], stage_empty[MAXST], op_full[MAXOP], op_empty[MAXOP], b_full;
  uint32_t abort;
  uint32_t op_flags[MAXOP][NCW];
  alignas(16) float epi_scale[288];   // per output channel of the slab (fixed for the whole kernel)
  alignas(16) float epi_bias[288];
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
// (a, b) -> packed bf16 pairs of the exact pieces hi, mid, lo with a = hi_a + mid_a + lo_a (same for b)
__device__ __forceinline__ void split3_pair(float a, float b, uint32_t& hp, uint32_t& mp, uint32_t& lp) {
  hp = pack_bf16x2(a, b);
  const float ra = a - __uint_as_float(hp << 16), rb = b - __uint_as_float(hp & 0xffff0000u);
  mp = pack_bf16x2(ra, rb);
  const float la = ra - __uint_as_float(mp << 16), lb = rb - __uint_as_float(mp & 0xffff0000u);
  lp = pack_bf16x2(la, lb);
}

// debug instrumentation: time spent inside a bounded wait, accumulated per role
#define PROF_WAIT(slot, call)                                   \
  do {                                                          \
    long long t0__ = p.prof ? clock64() : 0;                    \
    const bool ok__ = (call);                                   \
    if (p.prof) prof_acc[slot] += clock64() - t0__;             \
    if (!ok__) goto done;                                       \
  } while (0)

#define PROF_SOFT(slot, call)                                   \
  do {                                                          \
    long long t0__ = p.prof ? clock64() : 0;                    \
    call;                                                       \
    if (p.prof) prof_acc[slot] += clock64() - t0__;             \
  } while (0)

__device__ __forceinline__ void wg_bar_sync(int wg) {  // named barriers 2, 3: one MMA warpgroup
  asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
}

template <int NG>   // output channels per group (GEMM N)
__global__ void __launch_bounds__(NTHREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_in, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* stage_base = smem + p.off_stage;
  uint8_t* op_base = smem + p.off_op;
  uint8_t* b_base = smem + p.off_b;
  long long prof_acc[3] = {0, 0, 0};
  const long long prof_t0 = p.prof ? clock64() : 0;

  // ---- work assignment: CTA -> slab of groups; the slab's tiles are dealt round-robin
  const int slab = blockIdx.x % p.n_slabs;
  const int rank_in_slab = blockIdx.x / p.n_slabs;
  const int ctas_in_slab = (gridDim.x - slab + p.n_slabs - 1) / p.n_slabs;
  const int g_first = slab * p.slab_groups;
  const int g_count = min(p.slab_groups, p.G - g_first);

  // ---- one-time setup
  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) { tc::mbar_init(&sh.stage_full[i], 1); tc::mbar_init(&sh.stage_empty[i], NCONV / 32); }
    for (int i = 0; i < MAXOP; ++i) { tc::mbar_init(&sh.op_full[i], NCONV / 32); tc::mbar_init(&sh.op_empty[i], 8); }
    tc::mbar_init(&sh.b_full, 1);
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmap_in);
  }
  if (tid < MAXOP * NCW) sh.op_flags[tid / NCW][tid % NCW] = 0;
  if (tid == 0) sh.abort = 0;
  // zero the operand buffers once: the mid / lo planes are only rewritten when a chunk needs them
  for (int i = tid; i < p.nop * p.op_buf_bytes / 16; i += NTHREADS)
    reinterpret_cast<uint4*>(op_base)[i] = make_uint4(0, 0, 0, 0);
  // per-channel constants of this slab, loaded once: forward = epilogue scale / bias per output channel,
  // dgrad = weight scale per INPUT channel (folded into dy while it is converted)
  if (p.dgrad) {
    const int ch_first = g_first * p.cin_g;
    for (int n = tid; n < g_count * p.cin_g && n < 288; n += NTHREADS) sh.epi_scale[n] = __ldg(p.w_scale + ch_first + n);
  } else {
    const float a_sc0 = p.a_scale ? __ldg(p.a_scale) : p.a_scale_const;
    const int ch_first = g_first * p.cout_g;
    for (int n = tid; n < g_count * p.cout_g; n += NTHREADS) {
      sh.epi_scale[n] = __fmul_rn(a_sc0, __ldg(p.w_scale + ch_first + n));
      sh.epi_bias[n] = p.bias ? __ldg(p.bias + ch_first + n) : 0.f;
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp == 0) {
    // ================================================================= TMA producer
    if (lane == 0) {
      // resident B operand of this slab: one bulk copy of the pre-packed bf16 image (L2 -> smem)
      {
        const uint32_t bytes = (uint32_t)(g_count * p.b_group_bytes);
        tc::mbar_arrive_expect_tx(&sh.b_full, bytes);
        tc::bulk_load_1d(b_base, p.w_pack + (size_t)g_first * p.b_group_bytes, bytes, &sh.b_full);
      }
      // ring positions are advanced incrementally: a runtime `it % nst` costs a ~100-cycle integer division, and these
      // per-chunk loops are pure latency chains (nothing else to issue while the quotient is computed)
      int st = -1;
      uint32_t ph = 1;
      for (int tile = rank_in_slab; tile < p.n_tiles; tile += ctas_in_slab) {
        const int bt = tile / p.row_tiles, rt = tile - bt * p.row_tiles;
        const int b0 = bt * p.TB, h0 = rt * p.TH;
        for (int gi = 0; gi < g_count; ++gi) {
          for (int ch = 0; ch < p.nchunk; ++ch) {
            if (++st == p.nst) st = 0;
            ph ^= (st == 0);
            PROF_WAIT(0, tc::mbar_wait(&sh.stage_empty[st], ph ^ 1, p.err, 301));
            tc::mbar_arrive_expect_tx(&sh.stage_full[st], (uint32_t)p.stage_bytes);
            if (p.pad == 0)   // un-padded tile rows are contiguous: one long row per channel (see launch())
              tc::tma_load_3d(stage_base + (size_t)st * p.stage_bytes, &tmap_in, &sh.stage_full[st], h0 * p.W,
                              (g_first + gi) * p.cin_g + ch * p.CC, b0);
            else
              tc::tma_load_4d(stage_base + (size_t)st * p.stage_bytes, &tmap_in, &sh.stage_full[st], 0, h0 - p.pad,
                              (g_first + gi) * p.cin_g + ch * p.CC, b0);
          }
        }
      }
    }
  } else if (warp >= 4 && warp < 12) {
    // ================================================================= MMA warpgroups + epilogue
    // Warpgroup wg (warps 4..7 / 8..11) owns GEMM rows (= padded-tile positions) 64*wg .. 64*wg+63 of every group's
    // accumulator (m64 x NG in registers).  Epilogue: 32 columns at a time through a 64 x 32 staging tile; thread lt of
    // the warpgroup then owns position 64*wg + lt%64 and 16 of the 32 columns (lt / 64), stored as coalesced NCHW rows.
    const int wg = (warp - 4) >> 2, lt = tid - 128 * (wg + 1);
    float* stage = reinterpret_cast<float*>(smem + p.off_stg) + wg * 32 * tc::kStageLd64;
    const int pos = 64 * wg + (lt & 63), ehalf = lt >> 6;
    const int tb = pos / (p.THH * p.BW);
    const int rem = pos - tb * (p.THH * p.BW);
    const int th = rem / p.BW, wc = rem - th * p.BW;
    MnbActQ ste;
    if (p.dgrad && p.ste_bits) ste = mnb_load_actq(p.qp);
    const int64_t plane = (int64_t)p.H * p.W;
    const int ch_first = g_first * p.cout_g;
    const uint32_t a_lbo = (uint32_t)p.npos_in * 16u, b_lbo = (uint32_t)p.cout_g * 16u;
    // descriptors differ only in the 14-bit start-address field: build once, then add (bytes >> 4)
    const uint64_t a_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(op_base), a_lbo, 128) + (uint64_t)(64 * wg);
    const uint64_t b_desc0 = tc::smem_desc_kmajor_noswz(tc::smem_u32(b_base), b_lbo, 128);
    const uint32_t a_term = (uint32_t)p.op_term_bytes >> 4, a_buf = (uint32_t)p.op_buf_bytes >> 4;
    const uint32_t b_chunk = (uint32_t)((p.CC / 8) * p.cout_g * 16) >> 4, b_group = (uint32_t)p.b_group_bytes >> 4;
    const int ksteps = p.CC / 16;
    const int max_terms = p.quant_mode == 0 ? 3 : 1;
    PROF_SOFT(0, tc::mbar_wait_soft(&sh.b_full, 0, p.err, 307, &sh.abort));
    int ob = -1;
    uint32_t oph = 1;
    for (int tile = rank_in_slab; tile < p.n_tiles; tile += ctas_in_slab) {
      const int bt = tile / p.row_tiles, rt = tile - bt * p.row_tiles;
      const int b = bt * p.TB + tb, h = rt * p.TH + th;
      const bool valid = tb < p.TB && th < p.TH && wc < p.W && b < p.B && h < p.H;
      float* orow = p.out + (((int64_t)b * p.Cout + ch_first) * p.H + h) * p.W + wc;
      const int64_t obase = (((int64_t)b * p.Cout + ch_first) * p.H + h) * p.W + wc;
      for (int gi = 0; gi < g_count; ++gi) {
        float acc[NG / 2];
        tc::zero_acc(acc);
        for (int ch = 0; ch < p.nchunk; ++ch) {
          if (++ob == p.nop) ob = 0;
          oph ^= (ob == 0);
          PROF_SOFT(1, tc::mbar_wait_soft(&sh.op_full[ob], oph, p.err, 303, &sh.abort));
          bool need_low = false;  // mid / lo planes needed for this chunk?
          if (p.quant_mode == 0) {
            uint32_t any = 0;
#pragma unroll
            for (int w8 = 0; w8 < NCW; ++w8) any |= sh.op_flags[ob][w8];
            need_low = __any_sync(0xffffffffu, any != 0);
          }
          const uint64_t a_chunk = a_desc0 + (uint64_t)((uint32_t)ob * a_buf);
          const uint64_t b_chunk_d = b_desc0 + (uint64_t)((uint32_t)gi * b_group + (uint32_t)ch * b_chunk);
          const long long tmma0 = p.prof ? clock64() : 0;
          const int n_off = (p.dbg & 8) ? 0 : p.R * p.S * ksteps;
          tc::wg_fence();
          tc::fence_acc(acc);
          if (max_terms == 3 && need_low) {
            for (int e = 0; e < n_off; ++e) {
              const uint2 off = p.mma_off[e];
              const uint64_t ad = a_chunk + (uint64_t)off.x, bd = b_chunk_d + (uint64_t)off.y;
              tc::Mma<NG>::template bf16<0, 0>(acc, ad, bd, 1);
              tc::Mma<NG>::template bf16<0, 0>(acc, ad + a_term, bd, 1);
              tc::Mma<NG>::template bf16<0, 0>(acc, ad + 2 * a_term, bd, 1);
            }
          } else {
            for (int e = 0; e < n_off; ++e) {
              const uint2 off = p.mma_off[e];
              tc::Mma<NG>::template bf16<0, 0>(acc, a_chunk + (uint64_t)off.x, b_chunk_d + (uint64_t)off.y, 1);
            }
          }
          tc::wg_commit();
          tc::wg_wait<0>();
          tc::fence_acc(acc);
          if (p.prof) prof_acc[2] += clock64() - tmma0;
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(&sh.op_empty[ob]);  // this warp's share of the operand buffer is read
        }
        const int gcol = gi * p.cout_g;
#pragma unroll
        for (int c0 = 0; c0 < NG; c0 += 32) {
          wg_bar_sync(wg);   // the previous staging tile has been read
          tc::frag_cols_to_smem(acc, stage, tc::kStageLd64, 0, c0, 32);
          wg_bar_sync(wg);
          const int nb = gcol + c0 + 16 * ehalf;   // first slab column of this thread
          if (c0 + 16 * ehalf >= NG || !valid || (p.dbg & 4)) continue;
          float r[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) r[j] = stage[(16 * ehalf + j) * tc::kStageLd64 + (lt & 63)];
          if (!p.dgrad) {
            // scale / bias of the 16 columns as vector loads up front, then a pure FFMA + STG stream
            float sc[16], bs[16];
#pragma unroll
            for (int v = 0; v < 4; ++v) {
              const float4 a = *reinterpret_cast<const float4*>(&sh.epi_scale[nb + 4 * v]);
              const float4 c = *reinterpret_cast<const float4*>(&sh.epi_bias[nb + 4 * v]);
              sc[4 * v] = a.x; sc[4 * v + 1] = a.y; sc[4 * v + 2] = a.z; sc[4 * v + 3] = a.w;
              bs[4 * v] = c.x; bs[4 * v + 1] = c.y; bs[4 * v + 2] = c.z; bs[4 * v + 3] = c.w;
            }
            float* op = orow + (int64_t)nb * plane;
#pragma unroll
            for (int j = 0; j < 16; ++j, op += plane) *op = fmaf(r[j], sc[j], bs[j]);
          } else if (p.ste_bits) {
            // the 16 channel planes' mask words first (independent loads), then select + store.  The reference's STE
            // computes ((g*s)*pass)/s (IAO) or (((g*s)/s)*pass)*0.1 (DoReFa); (g*s)/s is g to within one ulp, so the
            // epilogue passes g itself (well inside the 1e-5 contract).
            const int64_t fi0 = obase + (int64_t)nb * plane;
            const uint32_t shift = (uint32_t)(fi0 & 31);
            const bool same_bit = (plane & 31) == 0;
            uint32_t wbits[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) wbits[j] = __ldg(p.ste_bits + ((fi0 + (int64_t)j * plane) >> 5));
            const float gain = ste.mode == MNB_ACT_DOREFA ? 0.1f : 1.f;
            float* op = orow + (int64_t)nb * plane;
#pragma unroll
            for (int j = 0; j < 16; ++j, op += plane) {
              const uint32_t sh_j = same_bit ? shift : (uint32_t)((fi0 + (int64_t)j * plane) & 31);
              const bool pass = (wbits[j] >> sh_j) & 1u;
              *op = pass ? r[j] * gain : 0.f;
            }
          } else {
            float* op = orow + (int64_t)nb * plane;
#pragma unroll
            for (int j = 0; j < 16; ++j, op += plane) *op = r[j];
          }
        }
      }
    }
  } else {
    // ================================================================= converters (warps 1..3, 12..15)
    const int ct = warp >= 12 ? tid - 384 + 96 : tid - 32;
    const int cw = ct >> 5;
    MnbActQ q;
    if (p.quant_mode != 0) q = mnb_load_actq(p.qp);
    const int a_off = p.a_offset + ((p.quant_mode == MNB_ACT_IAO && p.qp.zero_point) ? (int)__ldg(p.qp.zero_point) : 0);
    const int per_img = p.THH * p.BW;
    const int total = p.npos_in * (p.CC / 8);
    const int chstride = p.THH * p.W;  // floats between consecutive channels in the staging box
    // per-thread operand entries: fixed for the whole kernel (depend on the tile geometry only)
    int soff[KMAX];   // staging float offset of channel 0 of the entry's 8-channel group, -1: halo / dead
    int meta[KMAX];   // hr | tb << 8 | c8 << 16 | w << 20
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      const int idx = ct + k * NCONV;
      soff[k] = -1; meta[k] = 0;
      if (idx < total) {
        const int c8 = idx / p.npos_in, ip = idx - c8 * p.npos_in;
        const int tb = ip / per_img;
        const int rem = ip - tb * per_img;
        const int hr = rem / p.BW, wc = rem - hr * p.BW;
        const int w = wc - p.pad;
        if (tb < p.TB && w >= 0 && w < p.W) {
          soff[k] = ((tb * p.CC + c8 * 8) * p.THH + hr) * p.W + w;
          meta[k] = hr | (tb << 8) | (c8 << 16) | (w << 20);
        }
      }
    }
    uint32_t dirty_all = 0;   // 8 bits per operand buffer (KMAX <= 8 entries per thread), kept in one register
    int st = -1, ob = -1;
    uint32_t ph = 1, oph = 1;
    for (int tile = rank_in_slab; tile < p.n_tiles; tile += ctas_in_slab) {
      const int bt = tile / p.row_tiles, rt = tile - bt * p.row_tiles;
      const int b0 = bt * p.TB, h0 = rt * p.TH;
      for (int gi = 0; gi < g_count; ++gi) {
        for (int ch = 0; ch < p.nchunk; ++ch) {
          if (++st == p.nst) st = 0;
          ph ^= (st == 0);
          if (++ob == p.nop) ob = 0;
          oph ^= (ob == 0);
          PROF_WAIT(0, tc::mbar_wait(&sh.op_empty[ob], oph ^ 1, p.err, 306));
          PROF_WAIT(1, tc::mbar_wait(&sh.stage_full[st], ph, p.err, 305));
          // did THIS thread leave non-zero mid / lo pieces in its entries of this buffer last time?
          // (entries are owned by fixed threads, so dirtiness is thread-private state)
          const uint32_t dirty = (dirty_all >> (8 * ob)) & 0xffu;
          uint32_t now_dirty = 0;
          const float* stg = reinterpret_cast<const float*>(stage_base + (size_t)st * p.stage_bytes);
          uint8_t* opb = op_base + (size_t)ob * p.op_buf_bytes;
          const int cbase = (g_first + gi) * p.cin_g + ch * p.CC;
          uint32_t any_low = 0;
#pragma unroll
          for (int k = 0; k < KMAX; ++k) {
            if ((ct & ~31) + k * NCONV >= total || (p.dbg & 2)) break;  // warp-uniform
            const int idx = ct + k * NCONV;
            const bool live = idx < total;
            const int so = soff[k];
            uint32_t u[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) u[j] = so >= 0 ? __float_as_uint(stg[so + j * chstride]) : 0u;
            uint4 hi;
            if (p.quant_mode == 0) {
              if (p.dgrad) {  // fold the per-input-channel weight scale into the gradient operand
                const float* sc = &sh.epi_scale[gi * p.cin_g + ch * p.CC + ((meta[k] >> 16) & 15) * 8];
                const float4 s0 = *reinterpret_cast<const float4*>(sc), s1 = *reinterpret_cast<const float4*>(sc + 4);
                u[0] = __float_as_uint(__fmul_rn(__uint_as_float(u[0]), s0.x)); u[1] = __float_as_uint(__fmul_rn(__uint_as_float(u[1]), s0.y));
                u[2] = __float_as_uint(__fmul_rn(__uint_as_float(u[2]), s0.z)); u[3] = __float_as_uint(__fmul_rn(__uint_as_float(u[3]), s0.w));
                u[4] = __float_as_uint(__fmul_rn(__uint_as_float(u[4]), s1.x)); u[5] = __float_as_uint(__fmul_rn(__uint_as_float(u[5]), s1.y));
                u[6] = __float_as_uint(__fmul_rn(__uint_as_float(u[6]), s1.z)); u[7] = __float_as_uint(__fmul_rn(__uint_as_float(u[7]), s1.w));
              }
              uint32_t low = 0;
#pragma unroll
              for (int j = 0; j < 8; ++j) low |= u[j] & 0xffffu;
              if (low == 0) {
                // already bf16-exact (e.g. +-1 activations): the high halves ARE the operand
                hi = make_uint4(__byte_perm(u[0], u[1], 0x7632), __byte_perm(u[2], u[3], 0x7632),
                                __byte_perm(u[4], u[5], 0x7632), __byte_perm(u[6], u[7], 0x7632));
                if (((dirty >> k) & 1u) && live) {
                  *reinterpret_cast<uint4*>(opb + (size_t)p.op_term_bytes + (size_t)idx * 16) = make_uint4(0, 0, 0, 0);
                  *reinterpret_cast<uint4*>(opb + (size_t)2 * p.op_term_bytes + (size_t)idx * 16) = make_uint4(0, 0, 0, 0);
                }
              } else {
                // exact 3-way split x = hi + mid + lo (8 + 8 + 8 significand bits), two values per
                // cvt.rn.bf16x2 so that the three planes cost ~13 instructions per pair
                uint32_t hp[4], mp[4], lp[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) split3_pair(__uint_as_float(u[2 * j]), __uint_as_float(u[2 * j + 1]), hp[j], mp[j], lp[j]);
                any_low = 1;
                now_dirty |= 1u << k;
                hi = make_uint4(hp[0], hp[1], hp[2], hp[3]);
                if (live) {
                  *reinterpret_cast<uint4*>(opb + (size_t)p.op_term_bytes + (size_t)idx * 16) = make_uint4(mp[0], mp[1], mp[2], mp[3]);
                  *reinterpret_cast<uint4*>(opb + (size_t)2 * p.op_term_bytes + (size_t)idx * 16) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
                }
              }
            } else {
              // fused fake-quant: integer level (exact in bf16), plus the saved codes / STE bits
              const int hr = meta[k] & 255, tb = (meta[k] >> 8) & 255, c8 = (meta[k] >> 16) & 15, w = meta[k] >> 20;
              const int h = h0 - p.pad + hr, b = b0 + tb;
              const bool inside = so >= 0 && h >= 0 && h < p.H && b < p.B;
              const bool owned = inside && hr >= p.pad && hr < p.pad + p.TH;
              float e[8];
              const int64_t plane = (int64_t)p.H * p.W;
              const int64_t fi0 = (((int64_t)b * p.Cin + cbase + c8 * 8) * p.H + h) * p.W + w;
              // the 8 channels of an entry sit at the same pixel: when H*W is a multiple of 32 they share
              // the bit position and the lane grouping, so one match_any serves all eight
              const bool shared_group = (plane & 31) == 0;
              // un-padded tiles whose per-image part is a multiple of 32 pixels: the warp's 32 positions are
              // exactly one aligned mask word -> plain ballot + store, no atomics
              const bool whole_word = shared_group && p.pad == 0 && ((p.TH * p.W) & 31) == 0 &&
                                      __all_sync(0xffffffffu, owned);  // (warp-uniform)
              uint32_t peers0 = 0;
              if (p.pass_bits && shared_group && !whole_word)
                peers0 = __match_any_sync(0xffffffffu, owned ? (uint32_t)(fi0 >> 5) : 0xffffffffu);
              const bool leader0 = owned && (__ffs(peers0) - 1) == lane;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                bool pass;
                const int code = mnb_act_code_certified(q, __uint_as_float(u[j]), pass);
                e[j] = inside ? (float)(code + a_off) : 0.f;
                const int64_t fi = fi0 + (int64_t)j * plane;
                if (p.codes && owned) p.codes[fi] = (uint8_t)code;
                if (p.pass_bits) {
                  const uint32_t mine = (owned && pass) ? (1u << (fi & 31)) : 0u;
                  if (whole_word) {
                    const uint32_t wordv = __ballot_sync(0xffffffffu, mine != 0u);
                    if (lane == 0) p.pass_bits[fi >> 5] = wordv;
                  } else if (shared_group) {
                    const uint32_t val = __reduce_or_sync(peers0, mine);
                    if (leader0 && val) atomicOr(p.pass_bits + (fi >> 5), val);
                  } else {
                    // lanes that fall into the same 32-bit word combine their bits: one atomic per word
                    const uint32_t word = owned ? (uint32_t)(fi >> 5) : 0xffffffffu;
                    const uint32_t peers = __match_any_sync(0xffffffffu, word);
                    const uint32_t val = __reduce_or_sync(peers, mine);
                    if (owned && val && (__ffs(peers) - 1) == lane) atomicOr(p.pass_bits + word, val);
                  }
                }
              }
              hi = make_uint4(pack_bf16x2(e[0], e[1]), pack_bf16x2(e[2], e[3]), pack_bf16x2(e[4], e[5]), pack_bf16x2(e[6], e[7]));
            }
            if (live) *reinterpret_cast<uint4*>(opb + (size_t)idx * 16) = hi;
          }
          dirty_all = (dirty_all & ~(0xffu << (8 * ob))) | (now_dirty << (8 * ob));
          if (p.quant_mode == 0) {
            any_low = __reduce_or_sync(0xffffffffu, any_low);
            if (lane == 0) sh.op_flags[ob][cw] = any_low;
          }
          if (!(p.dbg & 1)) tc::fence_proxy_async_smem();   // every writer publishes its smem stores to the async proxy
          __syncwarp();
          if (lane == 0) {                // one arrival per warp: 16 instead of 512 smem atomics per chunk
            tc::mbar_arrive(&sh.op_full[ob]);
            tc::mbar_arrive(&sh.stage_empty[st]);
          }
        }
      }
    }
  }
done:
  if (p.prof && lane == 0 && (warp == 0 || warp == 4 || warp == 8 || warp == 12)) {
    // slots: [role 0..3 = tma, mma warpgroup 0, mma warpgroup 1, converter][wait a, wait b, wait c, total]
    const int role = warp == 0 ? 0 : (warp == 4 ? 1 : (warp == 8 ? 2 : 3));
    atomicAdd(reinterpret_cast<unsigned long long*>(p.prof + role * 4 + 0), (unsigned long long)prof_acc[0]);
    atomicAdd(reinterpret_cast<unsigned long long*>(p.prof + role * 4 + 1), (unsigned long long)prof_acc[1]);
    atomicAdd(reinterpret_cast<unsigned long long*>(p.prof + role * 4 + 2), (unsigned long long)prof_acc[2]);
    atomicAdd(reinterpret_cast<unsigned long long*>(p.prof + role * 4 + 3), (unsigned long long)(clock64() - prof_t0));
  }
  __syncthreads();
}

static long long* g_prof_buffer = nullptr;

// bf16 B-operand image of the integer weights: out[g][tap][k/8][n][8] (K-major no-swizzle, rows = n);
// forward: n = output channel, k = input channel; dgrad: n = input channel, k = output channel, taps flipped
__global__ void __launch_bounds__(256) pack_b_kernel(const int16_t* __restrict__ w_int, __nv_bfloat16* __restrict__ out,
                                                     int G, int cin_g, int cout_g, int RS, int dgrad) {
  const int per_group = RS * cin_g * cout_g;
  const int total = G * per_group;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    // idx enumerates the destination: [g][tap][c8][n][e]
    const int g = idx / per_group;
    int r = idx - g * per_group;
    const int tap = r / (cin_g * cout_g);
    r -= tap * (cin_g * cout_g);
    const int c8 = r / (cout_g * 8);
    r -= c8 * (cout_g * 8);
    const int n = r >> 3, c = c8 * 8 + (r & 7);
    int64_t src;
    if (!dgrad) src = ((int64_t)(g * cout_g + n) * cin_g + c) * RS + tap;
    else src = ((int64_t)(g * cin_g + c) * cout_g + n) * RS + (RS - 1 - tap);
    out[idx] = __float2bfloat16_rn((float)__ldg(w_int + src));
  }
}

// geometry + shared-memory plan shared by forward and dgrad; returns 0 / MNB_E_UNSUPPORTED / error
static int plan(const mnb_conv_shape* s, bool dgrad, int quant_mode, Params& p, int& smem_bytes) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  const int C = s->in_c, K = s->out_c, G = s->groups;
  MNB_REQUIRE(s->batch > 0 && C > 0 && K > 0 && s->in_h > 0 && s->in_w > 0 && G > 0 && C % G == 0 && K % G == 0,
              "bad conv shape");
  auto unsupported = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "tc conv: %s", why); };
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return unsupported("stride/dilation != 1");
  p.R = s->ker_h; p.S = s->ker_w;
  if (p.R != p.S || (p.R & 1) == 0 || s->pad_h != p.R / 2 || s->pad_w != p.R / 2) return unsupported("not a 'same' odd square filter");
  p.B = s->batch; p.H = s->in_h; p.W = s->in_w; p.G = G; p.pad = p.R / 2;
  p.dgrad = dgrad ? 1 : 0;
  p.Cin = dgrad ? K : C; p.Cout = dgrad ? C : K;
  p.cin_g = p.Cin / G; p.cout_g = p.Cout / G;
  if (p.cin_g % 16 || p.cout_g % 16 || p.cout_g > kMaxNG) return unsupported("channels per group");
  if ((p.W * 4) % 16 || p.W > 64 || p.H > 255) return unsupported("image size");
  p.BW = p.W + 2 * p.pad;
  p.TH = std::min(p.H, 128 / p.BW);
  if (p.TH < 1) return unsupported("padded row wider than 128 positions");
  p.THH = p.TH + 2 * p.pad;
  p.TB = 1;
  if (p.pad == 0 && p.TH == p.H) p.TB = std::max(1, std::min(p.B, 128 / (p.H * p.W)));  // small images: several per tile
  p.CC = (p.cin_g % 32 == 0) ? 32 : 16;
  p.nchunk = p.cin_g / p.CC;
  const int halo = (p.R - 1) * p.BW + (p.S - 1);
  const int npos = std::max(p.TB * p.THH * p.BW, 128) + halo;  // MMA rows read [tap_off, tap_off + 128)
  p.npos_in = (npos + 7) / 8 * 8;
  if (p.npos_in * (p.CC / 8) > KMAX * NCONV) {
    p.CC = 16; p.nchunk = p.cin_g / 16;
    if (p.npos_in * 2 > KMAX * NCONV) return unsupported("tile too large for the converter");
  }
  // the per-(tap, k-step) descriptor offsets live in a 64-entry kernel-parameter table (Params::mma_off)
  if (p.R * p.S * (p.CC / 16) > 64) {
    p.CC = 16; p.nchunk = p.cin_g / 16;
    if (p.R * p.S > 64) return unsupported("more than 64 filter taps");
  }
  p.row_tiles = (p.H + p.TH - 1) / p.TH;
  p.n_tiles = ((p.B + p.TB - 1) / p.TB) * p.row_tiles;
  p.quant_mode = quant_mode;
  p.stage_bytes = p.W * p.THH * p.CC * p.TB * 4;
  p.op_term_bytes = p.npos_in * (p.CC / 8) * 16;
  p.op_buf_bytes = p.op_term_bytes * (quant_mode == 0 ? 3 : 1);
  p.b_group_bytes = p.R * p.S * p.cin_g * p.cout_g * 2;
  p.nst = BASEST;
  p.nop = 2;
  int fixed = 0, budget = 0;
  for (;; --p.nst) {
    fixed = (p.nst * p.stage_bytes + 1023) / 1024 * 1024 + (p.nop * p.op_buf_bytes + 1023) / 1024 * 1024;
    budget = kPlanSmem - fixed;
    if (budget >= p.b_group_bytes || p.nst == 2) break;
  }
  if (budget < p.b_group_bytes) return unsupported("weights of one group do not fit in shared memory");
  int max_groups = std::max(1, std::min(p.G, std::min(budget / p.b_group_bytes, std::max(1, 64 * 1024 / p.b_group_bytes))));
  max_groups = std::max(1, std::min(max_groups, 256 / p.cout_g));  // per-channel constants of a slab: <= 256 columns
  if (dgrad) {  // per-input-channel scales of the slab are staged in a 288-float shared array
    if (p.cin_g > 288) return unsupported("more than 288 gradient channels per group");
    max_groups = std::max(1, std::min(max_groups, 288 / p.cin_g));
  }
  while (p.G % max_groups) --max_groups;  // equal slabs: every CTA does the same work per tile
  p.slab_groups = max_groups;
  p.n_slabs = p.G / p.slab_groups;
  // The pipeline floor is TMA latency x bytes in flight, so every kilobyte the weights and operands leave free becomes
  // staging slots.
  auto fits = [&](int nst, int nop) {
    return (nst * p.stage_bytes + 1023) / 1024 * 1024 + (nop * p.op_buf_bytes + 1023) / 1024 * 1024 +
               p.slab_groups * p.b_group_bytes <= kPlanSmem;
  };
  // Spare shared memory goes to the OPERAND ring first: the converter -> MMA -> release -> converter round trip has a
  // fixed latency even with no work in it, and more operand buffers hide it.
  while (p.nop < MAXOP && fits(p.nst, p.nop + 1)) ++p.nop;
  while (p.nst < MAXST && fits(p.nst + 1, p.nop)) ++p.nst;
  p.off_stage = 0;
  p.off_op = (p.nst * p.stage_bytes + 1023) / 1024 * 1024;
  p.off_b = p.off_op + (p.nop * p.op_buf_bytes + 1023) / 1024 * 1024;
  p.off_stg = (p.off_b + p.slab_groups * p.b_group_bytes + 15) / 16 * 16;
  smem_bytes = p.off_stg + kStgBytes;
  if (smem_bytes > kMaxDynSmem) return unsupported("shared memory budget");
  return 0;
}

// persistent CTAs: one per SM, at least one per slab
static int grid_size(const Params& p) {
  const int64_t items = (int64_t)p.n_tiles * p.n_slabs;
  return std::max((int)std::min<int64_t>(items, MNB_NUM_SMS), p.n_slabs);
}

static int launch(const Params& p, const void* in, int smem_bytes, cudaStream_t st) {
  {
    const int total = p.G * p.b_group_bytes / 2;
    pack_b_kernel<<<std::min(mnb_ceil_div(total, 256), MNB_NUM_SMS * 4), 256, 0, st>>>(
        p.w_int, reinterpret_cast<__nv_bfloat16*>(const_cast<uint8_t*>(p.w_pack)), p.G, p.cin_g, p.cout_g, p.R * p.S, p.dgrad);
  }
  CUtensorMap tmap;
  if (p.pad == 0) {
    // The TMA unit's cost is per box row, whatever its length: a 1x1 filter
    // needs no halo, so H and W collapse into one dimension and a tile is TH*W contiguous floats per channel
    // (4 x fewer rows than W-wide ones at 32x32).  Same shared-memory image as the 4-D box.
    uint64_t dims[3] = {(uint64_t)p.H * p.W, (uint64_t)p.Cin, (uint64_t)p.B};
    uint32_t box[3] = {(uint32_t)(p.TH * p.W), (uint32_t)p.CC, (uint32_t)p.TB};
    if (int e = mnb_make_tmap(&tmap, in, 4, 3, dims, box)) return e;
  } else {
    uint64_t dims[4] = {(uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Cin, (uint64_t)p.B};
    uint32_t box[4] = {(uint32_t)p.W, (uint32_t)p.THH, (uint32_t)p.CC, (uint32_t)p.TB};
    if (int e = mnb_make_tmap(&tmap, in, 4, 4, dims, box)) return e;
  }
  using KernelFn = void (*)(const CUtensorMap, const Params);
  static const KernelFn kernels[kMaxNG / 16] = {conv_tc_kernel<16>,  conv_tc_kernel<32>,  conv_tc_kernel<48>,  conv_tc_kernel<64>,
                                                conv_tc_kernel<80>,  conv_tc_kernel<96>,  conv_tc_kernel<112>, conv_tc_kernel<128>,
                                                conv_tc_kernel<144>, conv_tc_kernel<160>};
  static bool attr_set[kMaxNG / 16] = {};
  const int ki = p.cout_g / 16 - 1;
  if (!attr_set[ki]) {
    cudaError_t ce = cudaFuncSetAttribute(kernels[ki], cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set[ki] = true;
  }
  const int grid = grid_size(p);
  Params pp = p;
  pp.prof = g_prof_buffer;
  {
    static const int dbg = [] { const char* e = getenv("MNB_TC_DEBUG"); return e ? atoi(e) : 0; }();
    pp.dbg = dbg;
  }
  {
    const int ks = p.CC / 16, c8_per_group = p.cin_g / 8;
    for (int e = 0; e < p.R * p.S * ks && e < 64; ++e) {
      const int tap = e / ks, j = e - tap * ks;
      const int r = tap / p.S, s2 = tap - r * p.S;
      pp.mma_off[e] = make_uint2((uint32_t)(r * p.BW + s2) + (uint32_t)j * (uint32_t)(2 * p.npos_in),
                                 (uint32_t)tap * (uint32_t)(c8_per_group * p.cout_g) + (uint32_t)j * (uint32_t)(2 * p.cout_g));
    }
  }
  kernels[ki]<<<grid, NTHREADS, smem_bytes, st>>>(tmap, pp);
  MNB_LAUNCHED(2);
  return 0;
}

}  // namespace tcconv

// debug hook: device buffer of 16 int64 cycle counters (NULL disables); see PROF_WAIT above
extern "C" void mnb_set_tc_profile_buffer(void* dev_ptr) { tcconv::g_prof_buffer = reinterpret_cast<long long*>(dev_ptr); }

extern "C" int mnb_tc_conv_plan(const mnb_conv_shape* s, int32_t dgrad, int32_t quant_mode, int32_t* out, int32_t n) {
  tcconv::Params p{};
  int smem_bytes = 0;
  // the data gradient always splits fp32 dy: its launcher plans with quant_mode 0
  if (int e = tcconv::plan(s, dgrad != 0, dgrad ? 0 : quant_mode, p, smem_bytes)) return e;
  const int v[17] = {p.cout_g, p.TB, p.TH, p.row_tiles, p.n_tiles, p.CC, p.nchunk, p.nst, p.nop, p.slab_groups,
                     p.n_slabs, p.pad == 0, smem_bytes, p.BW, p.npos_in, tcconv::grid_size(p), p.R * p.S * (p.CC / 16)};
  if (out)
    for (int i = 0; i < std::min(n, 17); ++i) out[i] = v[i];
  return 0;
}

extern "C" int mnb_fq_conv2d_fwd_tc(const mnb_conv_shape* s, const float* x, const mnb_act_qparams* qp,
                                    const int16_t* w_int, const float* w_scale, const float* bias, float* y,
                                    uint8_t* codes, uint32_t* pass_bits, void* wpack_scratch, int32_t* err_flag,
                                    mnb_stream_t stream) {
  using namespace tcconv;
  MNB_REQUIRE(s && x && w_int && w_scale && y && err_flag && wpack_scratch, "NULL pointer");
  if (qp) MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA || qp->mode == MNB_ACT_IAO, "fused quantizer must be DoReFa or IAO");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan(s, false, qp ? qp->mode : 0, p, smem_bytes)) return e;
  if (qp) {
    if (qp->mode == MNB_ACT_DOREFA) MNB_REQUIRE(qp->bits >= 2 && qp->bits <= 8, "DoReFa a_bits must be in [2,8]");
    p.qp = *qp;
    p.a_offset = qp->mode == MNB_ACT_IAO ? qp->qmin : 0;
  }
  p.a_scale = (qp && qp->mode == MNB_ACT_IAO) ? qp->scale : nullptr;
  p.a_scale_const = (qp && qp->mode == MNB_ACT_DOREFA) ? (float)(1.0 / (double)((1 << qp->bits) - 1)) : 1.f;
  p.w_int = w_int; p.w_scale = w_scale; p.bias = bias; p.out = y; p.codes = codes; p.pass_bits = pass_bits;
  p.err = err_flag; p.w_pack = reinterpret_cast<const uint8_t*>(wpack_scratch);
  return launch(p, x, smem_bytes, (cudaStream_t)stream);
}

extern "C" int mnb_conv2d_dgrad_tc(const mnb_conv_shape* s, const float* dy, const int16_t* w_int,
                                   const float* w_scale, const uint32_t* pass_bits, const mnb_act_qparams* qp,
                                   float* dx, void* wpack_scratch, int32_t* err_flag, mnb_stream_t stream) {
  using namespace tcconv;
  MNB_REQUIRE(s && dy && w_int && w_scale && dx && err_flag && wpack_scratch, "NULL pointer");
  MNB_REQUIRE((pass_bits == nullptr) == (qp == nullptr), "pass_bits and qp go together");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan(s, true, 0, p, smem_bytes)) return e;
  if (qp) p.qp = *qp;
  p.a_scale_const = 1.f;
  p.w_int = w_int; p.w_scale = w_scale; p.ste_bits = pass_bits; p.out = dx; p.err = err_flag;
  p.w_pack = reinterpret_cast<const uint8_t*>(wpack_scratch);
  return launch(p, dy, smem_bytes, (cudaStream_t)stream);
}
