// Weight gradient of the fake-quant convolution on Hopper tensor cores (wgmma).
//
//   dWq[gNg+k, c, r, s] = s_a * sum_{b,h,w} dy[b, gNg+k, h, w] * e_a[b, gCg+c, h+r-p, w+s-p]
//
// The reduction runs over pixels, so both MMA operands are the position-major bf16 buffers the
// forward kernel builds (op[ch/8][position][8 ch]) - read here as MN-major wgmma operands:
//   A = dy^T  (128 gradient channels  x 16 positions per MMA), exact 3-term bf16 split of fp32 dy
//   B = e_a^T (N activation channels  x 16 positions per MMA), exact integer levels re-quantized
//                                                              from the fp32 input (or +-1 / bf16-exact raw x)
// and a filter tap (r, s) is again just a shifted start address of B.  Every CTA owns a block of gradient
// channels and streams its share of the pixel tiles through TMA -> converter warps -> MMA warpgroup; the warpgroup
// accumulates one tile's D[tap][128 x 32 columns] in registers at a time and adds it (fp32, round to nearest) into
// the CTA's partial dW in global memory (L2-resident); a second kernel reduces the partials in a fixed order
// (deterministic).
#include <cuda.h>
#include <cuda_bf16.h>

#include "mnb_common.cuh"
#include "mnb_tc.cuh"

namespace tcwgrad {

constexpr int NTHREADS = 512, NCONV = 320, MAXST = 8, BASEST = 4;  // warp 0 TMA, warps 4..7 MMA, converters: warps 2, 3, 8..15
constexpr int KX = 4, KD = 3;  // operand entries per converter thread: activation / gradient chunks
constexpr int kMaxDynSmem = 227 * 1024 - 2048;

struct Params {
  int B, C, K, H, W, R, S, pad, G, Cg, Ng;
  int BW, TH, THH, TB, CC, nst;
  int npos_x, npos_d, ksteps, row_tiles, n_tiles;   // npos_d: gradient positions per tile (multiple of 16)
  int op_buf_bytes, nbuf;                            // one {activation, 3 x gradient} operand buffer; nbuf (1|2) are cycled
  int Gb, nsplit, n_block, n_slabs, ranks;
  int tap_groups, tpc;   // filter taps are split over `tap_groups` CTA sets of `tpc` taps
  int quant_mode, a_offset;
  int slot_bytes, stage_x_bytes, stage_d_bytes, xop_bytes, dop_term_bytes, off_stage, off_xop, off_dop;
  mnb_act_qparams qp;
  float* partial;     // [ranks][K * Cg * RS]
  int* err;
  int* inexact;       // set when a raw fp32 activation is not bf16-exact (result then invalid)
};

struct alignas(16) Shared {
  uint64_t stage_full[MAXST], stage_empty[MAXST], op_full[2], op_empty[2];
  uint32_t abort;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// (a, b) -> packed bf16 pairs of the exact pieces hi, mid, lo with a = hi_a + mid_a + lo_a (same for b)
__device__ __forceinline__ void split3_pair(float a, float b, uint32_t& hp, uint32_t& mp, uint32_t& lp) {
  hp = pack_bf16x2(a, b);
  const float ra = a - __uint_as_float(hp << 16), rb = b - __uint_as_float(hp & 0xffff0000u);
  mp = pack_bf16x2(ra, rb);
  const float la = ra - __uint_as_float(mp << 16), lb = rb - __uint_as_float(mp & 0xffff0000u);
  lp = pack_bf16x2(la, lb);
}

__global__ void __launch_bounds__(NTHREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy,
                const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* stage_base = smem + p.off_stage;
  uint8_t* xop = smem + p.off_xop;
  uint8_t* dop = smem + p.off_dop;
  const int RS = p.R * p.S;

  // ---- block of gradient channels owned by this CTA
  const int slab = blockIdx.x % p.n_slabs, rank = blockIdx.x / p.n_slabs;
  const int tg = slab % p.tap_groups, cb = slab / p.tap_groups;   // tap group, channel block
  const int gbi = cb / p.nsplit, ms = cb - gbi * p.nsplit;
  const int tap0 = tg * p.tpc, tap1 = min(RS, tap0 + p.tpc);
  const int dy_ch0 = gbi * p.Gb * p.Ng + ms * 128;
  const int m_real = min(128, p.Gb * p.Ng - ms * 128);
  const int x_ch0 = gbi * p.Gb * p.Cg;
  const int x_chunks = p.n_block / p.CC, d_chunks = m_real / p.CC;
  const int my_tiles = (p.n_tiles > rank) ? (p.n_tiles - rank + p.ranks - 1) / p.ranks : 0;

  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) { tc::mbar_init(&sh.stage_full[i], 1); tc::mbar_init(&sh.stage_empty[i], NCONV / 32); }
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&sh.op_full[i], NCONV / 32); tc::mbar_init(&sh.op_empty[i], 4); }
    sh.abort = 0;
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmap_x);
    tc::prefetch_tmap(&tmap_dy);
  }
  // operand buffers start as zeros: padded columns / rows and unused channel rows are never written
  for (int i = tid; i < p.nbuf * p.op_buf_bytes / 16; i += NTHREADS)
    reinterpret_cast<uint4*>(xop)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async_smem();
  __syncthreads();
  const int64_t wsize = (int64_t)p.K * p.Cg * RS;
  float* mine = p.partial + (int64_t)rank * wsize;   // this CTA's partial dW

  if (warp == 0) {
    // ================================================================= TMA producer
    if (lane == 0) {
      int st = -1;          // ring position advanced incrementally (no per-chunk integer division)
      uint32_t ph = 1;
      for (int tile = rank; tile < p.n_tiles; tile += p.ranks) {
        const int bt = tile / p.row_tiles, rt = tile - bt * p.row_tiles;
        const int b0 = bt * p.TB, h0 = rt * p.TH;
        for (int ch = 0; ch < x_chunks + d_chunks; ++ch) {
          if (++st == p.nst) st = 0;
          ph ^= (st == 0);
          if (!tc::mbar_wait(&sh.stage_empty[st], ph ^ 1, p.err, 401)) goto done;
          uint8_t* dst = stage_base + (size_t)st * p.slot_bytes;
          if (ch < x_chunks) {
            tc::mbar_arrive_expect_tx(&sh.stage_full[st], (uint32_t)p.stage_x_bytes);
            if (p.pad == 0) tc::tma_load_3d(dst, &tmap_x, &sh.stage_full[st], h0 * p.W, x_ch0 + ch * p.CC, b0);
            else tc::tma_load_4d(dst, &tmap_x, &sh.stage_full[st], 0, h0 - p.pad, x_ch0 + ch * p.CC, b0);
          } else {
            tc::mbar_arrive_expect_tx(&sh.stage_full[st], (uint32_t)p.stage_d_bytes);
            tc::tma_load_3d(dst, &tmap_dy, &sh.stage_full[st], h0 * p.W, dy_ch0 + (ch - x_chunks) * p.CC, b0);
          }
        }
      }
    }
  } else if (warp >= 4 && warp < 8) {
    // ================================================================= MMA warpgroup -> partial dW
    // per tile, tap and 32 activation channels: both 64-row halves of the 128 gradient channels in registers (m64n32),
    // then added into the partial straight from the fragment (every element belongs to exactly one thread)
    const int wq = warp - 4, fr = 16 * wq + (lane >> 2), fc = 2 * (lane & 3);
    const uint64_t b_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(xop), 128, (uint32_t)p.npos_x * 16u);
    const uint64_t a_desc0 = tc::smem_desc_mnmajor_noswz(tc::smem_u32(dop), 128, (uint32_t)p.npos_d * 16u);
    const uint32_t buf16 = (uint32_t)p.op_buf_bytes >> 4;
    const uint32_t a_term = (uint32_t)p.dop_term_bytes >> 4, a_half = 8u * (uint32_t)p.npos_d;
    uint32_t t = 0;
    for (int tile = rank; tile < p.n_tiles; tile += p.ranks, ++t) {
      const uint32_t ob = p.nbuf == 2 ? (t & 1u) : 0u, oph = p.nbuf == 2 ? ((t >> 1) & 1u) : (t & 1u);
      tc::mbar_wait_soft(&sh.op_full[ob], oph, p.err, 402, &sh.abort);
      for (int tap = tap0; tap < tap1; ++tap) {
        const int r = tap / p.S, s2 = tap - r * p.S;
        const uint64_t b_tap = b_desc0 + (uint64_t)(ob * buf16 + (uint32_t)(r * p.BW + s2));
        for (int n0 = 0; n0 < p.n_block; n0 += 32) {
          float acc0[16], acc1[16];
          tc::zero_acc(acc0); tc::zero_acc(acc1);
          tc::wg_fence();
          tc::fence_acc(acc0); tc::fence_acc(acc1);
          const uint64_t b_n = b_tap + (uint64_t)((uint32_t)(n0 / 8) * (uint32_t)p.npos_x);
          for (int ps = 0; ps < p.ksteps; ++ps) {
            const uint64_t bd = b_n + (uint64_t)(ps * 16);   // 16 positions x 16 bytes = 256 B
            const uint64_t ad = a_desc0 + (uint64_t)(ob * buf16 + (uint32_t)(ps * 16));
#pragma unroll
            for (int term = 0; term < 3; ++term) {
              tc::Mma<32>::bf16<1, 1>(acc0, ad + term * a_term, bd, 1);
              tc::Mma<32>::bf16<1, 1>(acc1, ad + term * a_term + a_half, bd, 1);
            }
          }
          tc::wg_commit();
          tc::wg_wait<0>();
          tc::fence_acc(acc0); tc::fence_acc(acc1);
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int row = fr + 8 * ((e >> 1) & 1) + 64 * (e >> 2), n = n0 + 8 * j + fc + (e & 1);
              const float v = (e >> 2) ? acc1[4 * j + (e & 3)] : acc0[4 * j + (e & 3)];
              if (row < m_real && n < p.n_block) {
                const int k_abs = dy_ch0 + row, xg = (x_ch0 + n) / p.Cg;
                if (xg == k_abs / p.Ng) {
                  float* dst = mine + ((int64_t)k_abs * p.Cg + (x_ch0 + n - xg * p.Cg)) * RS + tap;
                  *dst = t == 0 ? v : __fadd_rn(*dst, v);
                }
              }
            }
        }
      }
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.op_empty[ob]);
    }
    if (my_tiles == 0) {   // a rank without tiles contributes zeros
      const int m = wq * 32 + lane, k_abs = dy_ch0 + m, k_group = k_abs / p.Ng;
      if (m < m_real)
        for (int tap = tap0; tap < tap1; ++tap)
          for (int n = 0; n < p.n_block; ++n) {
            const int xg = (x_ch0 + n) / p.Cg;
            if (xg == k_group) mine[((int64_t)k_abs * p.Cg + (x_ch0 + n - xg * p.Cg)) * RS + tap] = 0.f;
          }
    }
  } else if (warp >= 2) {
    // ================================================================= converters (warps 2, 3, 8..15)
    const int ct = warp < 4 ? tid - 64 : tid - 64 - 128;
    MnbActQ q;
    if (p.quant_mode != 0) q = mnb_load_actq(p.qp);
    const int a_off = p.a_offset + ((p.quant_mode == MNB_ACT_IAO && p.qp.zero_point) ? (int)__ldg(p.qp.zero_point) : 0);
    const int per_img = p.THH * p.BW, c8s = p.CC / 8;
    const int total_x = p.npos_x * c8s;
    const int nvalid = p.TB * p.TH * p.W;
    const int total_d = nvalid * c8s;
    int xso[KX], xmeta[KX];
#pragma unroll
    for (int k = 0; k < KX; ++k) {
      const int idx = ct + k * NCONV;
      xso[k] = -1; xmeta[k] = 0;
      if (idx < total_x) {
        const int c8 = idx / p.npos_x, ip = idx - c8 * p.npos_x;
        const int tb = ip / per_img;
        const int rem = ip - tb * per_img;
        const int hr = rem / p.BW, wc = rem - hr * p.BW;
        const int w = wc - p.pad;
        if (tb < p.TB && w >= 0 && w < p.W) {
          xso[k] = ((tb * p.CC + c8 * 8) * p.THH + hr) * p.W + w;
          xmeta[k] = hr | (tb << 8);
        }
      }
    }
    int dso[KD], ddst[KD];
#pragma unroll
    for (int k = 0; k < KD; ++k) {
      const int idx = ct + k * NCONV;
      dso[k] = -1; ddst[k] = 0;
      if (idx < total_d) {
        const int c8 = idx / nvalid, vp = idx - c8 * nvalid;
        const int tb = vp / (p.TH * p.W);
        const int rem = vp - tb * (p.TH * p.W);
        const int th = rem / p.W, w = rem - th * p.W;
        dso[k] = ((tb * p.CC + c8 * 8) * p.TH + th) * p.W + w;
        ddst[k] = (c8 * p.npos_d + (tb * p.THH + th) * p.BW + w) * 16;  // byte offset inside a chunk's 8-ch groups
      }
    }
    const int x_chstride = p.THH * p.W, d_chstride = p.TH * p.W;
    uint32_t t = 0;
    int st = -1;
    uint32_t ph = 1;
    for (int tile = rank; tile < p.n_tiles; tile += p.ranks, ++t) {
      const int bt = tile / p.row_tiles, rt = tile - bt * p.row_tiles;
      const int b0 = bt * p.TB, h0 = rt * p.TH;
      const uint32_t ob = p.nbuf == 2 ? (t & 1u) : 0u, oph = p.nbuf == 2 ? ((t >> 1) & 1u) : (t & 1u);
      if (!tc::mbar_wait(&sh.op_empty[ob], oph ^ 1, p.err, 404)) goto done;  // MMAs of the tile two back retired
      uint8_t* xop_b = xop + (size_t)ob * p.op_buf_bytes;
      uint8_t* dop_b = dop + (size_t)ob * p.op_buf_bytes;
      for (int ch = 0; ch < x_chunks + d_chunks; ++ch) {
        if (++st == p.nst) st = 0;
        ph ^= (st == 0);
        if (!tc::mbar_wait(&sh.stage_full[st], ph, p.err, 405)) goto done;
        const float* stg = reinterpret_cast<const float*>(stage_base + (size_t)st * p.slot_bytes);
        if (ch < x_chunks) {
          uint8_t* dstb = xop_b + (size_t)ch * c8s * p.npos_x * 16;
#pragma unroll
          for (int k = 0; k < KX; ++k) {
            const int idx = ct + k * NCONV;
            if (idx >= total_x) break;
            const int so = xso[k];
            if (so < 0) continue;  // halo column / dead position: stays zero
            uint32_t u[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) u[j] = __float_as_uint(stg[so + j * x_chstride]);
            uint4 v;
            if (p.quant_mode == 0) {
              uint32_t low = 0;
#pragma unroll
              for (int j = 0; j < 8; ++j) low |= u[j] & 0xffffu;
              if (low) atomicOr(p.inexact, 1);
              v = make_uint4(__byte_perm(u[0], u[1], 0x7632), __byte_perm(u[2], u[3], 0x7632),
                             __byte_perm(u[4], u[5], 0x7632), __byte_perm(u[6], u[7], 0x7632));
            } else {
              const int hr = xmeta[k] & 255, tb = xmeta[k] >> 8;
              const int h = h0 - p.pad + hr;
              const bool inside = h >= 0 && h < p.H && (b0 + tb) < p.B;
              float e[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                bool pass;
                const int code = mnb_act_code_certified(q, __uint_as_float(u[j]), pass);
                e[j] = inside ? (float)(code + a_off) : 0.f;
              }
              v = make_uint4(pack_bf16x2(e[0], e[1]), pack_bf16x2(e[2], e[3]), pack_bf16x2(e[4], e[5]), pack_bf16x2(e[6], e[7]));
            }
            *reinterpret_cast<uint4*>(dstb + (size_t)idx * 16) = v;
          }
        } else {
          const int dch = ch - x_chunks;
          uint8_t* dstb = dop_b + (size_t)dch * c8s * p.npos_d * 16;
#pragma unroll
          for (int k = 0; k < KD; ++k) {
            if (ct + k * NCONV >= total_d) break;
            const int so = dso[k];
            uint32_t hp[4], mp[4], lp[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
              split3_pair(stg[so + (2 * j) * d_chstride], stg[so + (2 * j + 1) * d_chstride], hp[j], mp[j], lp[j]);
            uint8_t* d0 = dstb + ddst[k];
            *reinterpret_cast<uint4*>(d0) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
            *reinterpret_cast<uint4*>(d0 + p.dop_term_bytes) = make_uint4(mp[0], mp[1], mp[2], mp[3]);
            *reinterpret_cast<uint4*>(d0 + 2 * p.dop_term_bytes) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
          }
        }
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&sh.stage_empty[st]);
      }
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&sh.op_full[ob]);
    }
  }
done:
  __syncthreads();
}

__global__ void __launch_bounds__(256) wgrad_tc_reduce_kernel(const float* __restrict__ partial, int64_t n, int ranks,
                                                              const float* a_scale, float a_scale_const,
                                                              float* __restrict__ dwq) {
  const float sc = a_scale ? __ldg(a_scale) : a_scale_const;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // four chains in flight, fixed order: deterministic
    int j = 0;
    for (; j + 4 <= ranks; j += 4) {
      s0 += partial[(int64_t)j * n + i];
      s1 += partial[(int64_t)(j + 1) * n + i];
      s2 += partial[(int64_t)(j + 2) * n + i];
      s3 += partial[(int64_t)(j + 3) * n + i];
    }
    for (; j < ranks; ++j) s0 += partial[(int64_t)j * n + i];
    dwq[i] = __fmul_rn((s0 + s1) + (s2 + s3), sc);
  }
}

static int plan(const mnb_conv_shape* s, int quant_mode, Params& p, int& smem_bytes) {
  MNB_REQUIRE(s != nullptr, "conv shape is NULL");
  auto unsupported = [](const char* why) { return mnb_fail(MNB_E_UNSUPPORTED, "tc wgrad: %s", why); };
  p.B = s->batch; p.C = s->in_c; p.K = s->out_c; p.H = s->in_h; p.W = s->in_w; p.R = s->ker_h; p.S = s->ker_w; p.G = s->groups;
  MNB_REQUIRE(p.B > 0 && p.C > 0 && p.K > 0 && p.H > 0 && p.W > 0 && p.G > 0 && p.C % p.G == 0 && p.K % p.G == 0, "bad conv shape");
  if (s->stride_h != 1 || s->stride_w != 1 || s->dil_h != 1 || s->dil_w != 1) return unsupported("stride/dilation != 1");
  if (p.R != p.S || (p.R & 1) == 0 || s->pad_h != p.R / 2 || s->pad_w != p.R / 2) return unsupported("not a 'same' odd square filter");
  p.pad = p.R / 2; p.Cg = p.C / p.G; p.Ng = p.K / p.G;
  const int RS = p.R * p.S;
  if (p.Cg % 16 || p.Ng % 16) return unsupported("channels per group");
  if ((p.W * 4) % 16 || p.W > 64 || p.H > 255) return unsupported("image size");
  // block of gradient channels: Gb whole groups (Gb*Ng <= 128) or a 128-slice of one big group; taps may be split over
  // `tap_groups` CTA sets (each re-reading the inputs) to bound the MMA work of one CTA per tile.
  p.Gb = 1; p.nsplit = 1; p.tap_groups = 1; p.tpc = RS;
  if (p.Ng >= 128) {
    p.nsplit = (p.Ng + 127) / 128;
    if (p.Cg > 256) return unsupported("more than 256 activation channels per group");
    p.tpc = std::min(RS, 512 / p.Cg);
    if (p.tpc < 1) return unsupported("too many accumulator columns per CTA");
    p.tap_groups = (RS + p.tpc - 1) / p.tpc;
    p.tpc = (RS + p.tap_groups - 1) / p.tap_groups;
  } else {
    double best = 1e30;
    for (int gb = 1; gb <= p.G; ++gb) {
      if (p.G % gb || gb * p.Ng > 128 || gb * p.Cg > 256) continue;
      int tpc = std::min(RS, 512 / (gb * p.Cg));
      if (tpc < 1) continue;
      const int tgs = (RS + tpc - 1) / tpc;
      tpc = (RS + tgs - 1) / tgs;
      const double mma = tpc * 24.0 * 61.0;
      const double bytes = 4.0 * 128.0 * gb * (p.Cg * 1.3 + p.Ng);   // rough bytes per tile (activation halo ~1.3x)
      const double cost = tgs * std::max(mma, bytes / 23.0) / gb;
      if (cost < best) { best = cost; p.Gb = gb; p.tpc = tpc; p.tap_groups = tgs; }
    }
  }
  p.n_block = p.Gb * p.Cg;
  if (p.n_block > 256 || p.tpc * p.n_block > 512) return unsupported("too many accumulator columns per CTA");
  int cc0 = 32;
  if (p.n_block % 32 || (p.Gb * p.Ng) % 32 || (p.nsplit > 1 && p.Ng % 32)) cc0 = 16;
  if (p.nsplit > 1 && (p.Ng % 128) % cc0) return unsupported("ragged channel split");
  p.n_slabs = (p.G / p.Gb) * p.nsplit * p.tap_groups;
  p.BW = p.W + 2 * p.pad;
  const int th_max = std::min(p.H, 128 / p.BW);
  if (th_max < 1) return unsupported("padded row wider than 128 positions");
  const int halo = (p.R - 1) * p.BW + (p.S - 1);
  // rows per tile: the largest that lets TWO operand buffers (converter and MMA overlap) plus a staging
  // ring of >= 3 slots fit in shared memory
  bool ok = false;
  auto try_tile = [&](int TH, int TB, int nbuf) -> bool {
    p.TH = TH; p.TB = TB; p.nbuf = nbuf;
    p.THH = p.TH + 2 * p.pad;
    p.npos_d = ((p.pad > 0 ? p.TH * p.BW : p.TB * p.TH * p.W) + 15) / 16 * 16;
    if (p.npos_d > 128) return false;
    p.ksteps = p.npos_d / 16;
    p.npos_x = (p.npos_d + halo + 7) / 8 * 8;
    p.CC = cc0;
    if (p.npos_x * (p.CC / 8) > KX * NCONV || p.TB * p.TH * p.W * (p.CC / 8) > KD * NCONV) {
      if (p.CC == 32 && p.npos_x * 2 <= KX * NCONV) p.CC = 16; else return false;
    }
    p.stage_x_bytes = p.W * p.THH * p.CC * p.TB * 4;
    p.stage_d_bytes = p.W * p.TH * p.CC * p.TB * 4;
    p.slot_bytes = (std::max(p.stage_x_bytes, p.stage_d_bytes) + 127) / 128 * 128;
    p.xop_bytes = (p.n_block / 8) * p.npos_x * 16;
    p.dop_term_bytes = 16 * p.npos_d * 16;  // 128 channel rows (16 groups of 8) x npos_d positions
    p.op_buf_bytes = (p.xop_bytes + 3 * p.dop_term_bytes + 1023) / 1024 * 1024;
    p.off_xop = 0;
    p.off_dop = p.xop_bytes;
    p.off_stage = p.nbuf * p.op_buf_bytes;
    p.nst = BASEST;
    while (p.nst > 3 && p.off_stage + p.nst * p.slot_bytes > kMaxDynSmem) --p.nst;
    if (p.off_stage + p.nst * p.slot_bytes > kMaxDynSmem) return false;
    while (p.nst < MAXST && p.off_stage + (p.nst + 1) * p.slot_bytes <= kMaxDynSmem) ++p.nst;  // more bytes in flight
    smem_bytes = p.off_stage + p.nst * p.slot_bytes;
    return true;
  };
  // 1x1 filters (no halo re-reads, few MMAs per tile): one 128-position operand set, converter and MMA
  // alternate.  Filters with taps: two smaller operand sets so that the (tap-heavy) MMAs overlap the converter.
  if (p.pad == 0) {
    const int TH = th_max;
    const int tb = (TH == p.H) ? std::max(1, std::min(p.B, 128 / (p.H * p.W))) : 1;
    ok = try_tile(TH, tb, 1);
  }
  if (!ok) {
    int best_th = 0, best_tb = 0, best_tiles = 1 << 30;
    for (int TH = th_max; TH >= 1; --TH) {
      const int tb_max = (p.pad == 0 && TH == p.H) ? std::max(1, std::min(p.B, 128 / (p.H * p.W))) : 1;
      for (int TB = tb_max; TB >= 1; TB >>= 1) {
        if (!try_tile(TH, TB, 2)) continue;
        const int tiles = ((p.B + TB - 1) / TB) * ((p.H + TH - 1) / TH);
        if (tiles <= best_tiles) { best_tiles = tiles; best_th = TH; best_tb = TB; }  // ties: smaller tile
        break;
      }
    }
    ok = best_th > 0 && try_tile(best_th, best_tb, 2);
  }
  if (!ok) return unsupported("shared memory budget");
  p.row_tiles = (p.H + p.TH - 1) / p.TH;
  p.n_tiles = ((p.B + p.TB - 1) / p.TB) * p.row_tiles;
  p.ranks = std::max(1, std::min(p.n_tiles, MNB_NUM_SMS / p.n_slabs));  // one wave of CTAs
  p.quant_mode = quant_mode;
  return 0;
}

}  // namespace tcwgrad

extern "C" int mnb_wgrad_tc_plan(const mnb_conv_shape* s, int32_t quant_mode, int32_t* out, int32_t n) {
  tcwgrad::Params p{};
  int smem_bytes = 0;
  if (int e = tcwgrad::plan(s, quant_mode, p, smem_bytes)) return e;
  const int v[16] = {p.Gb, p.nsplit, p.tap_groups, p.tpc, p.n_block, p.CC, p.TH, p.TB, p.nbuf, p.nst, p.ranks,
                     p.n_slabs, smem_bytes, p.npos_d, p.npos_x, p.n_tiles};
  if (out)
    for (int i = 0; i < std::min(n, 16); ++i) out[i] = v[i];
  return 0;
}

extern "C" int64_t mnb_wgrad_tc_scratch_bytes(const mnb_conv_shape* s) {
  tcwgrad::Params p{};
  int smem = 0;
  if (tcwgrad::plan(s, 0, p, smem)) return -1;
  return (int64_t)p.ranks * p.K * p.Cg * p.R * p.S * 4;
}

extern "C" int mnb_conv2d_wgrad_tc(const mnb_conv_shape* s, const float* dy, const float* x, const mnb_act_qparams* qp,
                                   float* dwq, void* scratch, int32_t* inexact_flag, int32_t* err_flag,
                                   mnb_stream_t stream) {
  using namespace tcwgrad;
  MNB_REQUIRE(s && dy && x && dwq && scratch && inexact_flag && err_flag, "NULL pointer");
  if (qp) MNB_REQUIRE(qp->mode == MNB_ACT_DOREFA || qp->mode == MNB_ACT_IAO, "fused quantizer must be DoReFa or IAO");
  Params p{};
  int smem_bytes = 0;
  if (int e = plan(s, qp ? qp->mode : 0, p, smem_bytes)) return e;
  if (qp) {
    if (qp->mode == MNB_ACT_DOREFA) MNB_REQUIRE(qp->bits >= 2 && qp->bits <= 8, "DoReFa a_bits must be in [2,8]");
    p.qp = *qp;
    p.a_offset = qp->mode == MNB_ACT_IAO ? qp->qmin : 0;
  }
  p.partial = reinterpret_cast<float*>(scratch); p.err = err_flag; p.inexact = inexact_flag;
  CUtensorMap tx, td;
  // TMA cost is per box row: tiles without a halo (dy always, x of a 1x1 filter) are read as ONE contiguous row of
  // TH*W floats per channel over a collapsed (H*W, C, B) view; rows past the image end are zero-filled as before.
  uint64_t dd[3] = {(uint64_t)p.H * p.W, (uint64_t)p.K, (uint64_t)p.B};
  uint32_t bd[3] = {(uint32_t)(p.TH * p.W), (uint32_t)p.CC, (uint32_t)p.TB};
  if (int e = mnb_make_tmap(&td, dy, 4, 3, dd, bd)) return e;
  if (p.pad == 0) {
    uint64_t dx[3] = {(uint64_t)p.H * p.W, (uint64_t)p.C, (uint64_t)p.B};
    uint32_t bx[3] = {(uint32_t)(p.TH * p.W), (uint32_t)p.CC, (uint32_t)p.TB};
    if (int e = mnb_make_tmap(&tx, x, 4, 3, dx, bx)) return e;
  } else {
    uint64_t dx[4] = {(uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.C, (uint64_t)p.B};
    uint32_t bx[4] = {(uint32_t)p.W, (uint32_t)p.THH, (uint32_t)p.CC, (uint32_t)p.TB};
    if (int e = mnb_make_tmap(&tx, x, 4, 4, dx, bx)) return e;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
    if (ce != cudaSuccess) return mnb_fail((int)ce, "cudaFuncSetAttribute: %s", cudaGetErrorString(ce));
    attr_set = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  wgrad_tc_kernel<<<p.n_slabs * p.ranks, NTHREADS, smem_bytes, st>>>(tx, td, p);
  const int64_t n = (int64_t)p.K * p.Cg * p.R * p.S;
  const float a_const = (qp && qp->mode == MNB_ACT_DOREFA) ? (float)(1.0 / (double)((1 << qp->bits) - 1)) : 1.f;
  const float* a_ptr = (qp && qp->mode == MNB_ACT_IAO) ? qp->scale : nullptr;
  int blocks = (int)std::min<int64_t>(mnb_ceil_div(n, 256), MNB_NUM_SMS * 8);
  wgrad_tc_reduce_kernel<<<blocks, 256, 0, st>>>(p.partial, n, p.ranks, a_ptr, a_const, dwq);
  MNB_LAUNCHED(2);
  return 0;
}
