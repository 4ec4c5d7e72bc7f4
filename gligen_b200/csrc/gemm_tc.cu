// wgmma / TMA GEMM and implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[M,N] = epilogue( A[M,K] . W[N,K]^T )           bf16 operands, fp32 accumulation in registers
//
// Persistent, warp-specialised, three warpgroups per CTA (384 threads):
//   warpgroup 0   : TMA producer (one elected lane of warp 0: cp.async.bulk.tensor -> 128B-swizzled smem ring,
//                   mbarrier complete_tx); gives most of its registers to the consumers (setmaxnreg)
//   warpgroups 1-2: consumers, each owning 64 rows of the 128 x BN tile: wgmma.mma_async m64nBNk16 on the smem
//                   descriptors, fp32 accumulators in registers, then the epilogue straight from registers
//                   (LayerNorm fold / bias / time-embedding row bias / SiLU / GELU / tanh-gate / residual / GEGLU ->
//                   bf16 or fp32 global stores, per-row LayerNorm partial sums of what is stored)
//
// Two consumer schedules:
//   PP = false (cooperative): both consumer warpgroups share one 128 x BN work item, 64 rows each, and run its epilogue
//                  together while the tensor pipe idles.
//   PP = true  (ping-pong): each consumer warpgroup owns whole 128 x BN work items (two m64 x BN accumulators, rows 0-63 and
//                  64-127 of the same A stage): warpgroup 0 takes the CTA's even items, warpgroup 1 the odd ones.  An MMA
//                  token passed through two named barriers lets only one of them issue wgmmas at a time, so one warpgroup's
//                  epilogue runs under the other's mainloop.  The producer feeds both through the same in-order ring; each
//                  warpgroup steps its ring position over the stages of the other's items.  GEGLU items are 128 packed weight
//                  rows [64 x | 64 gate] cut from the 256-row [128 x | 128 gate] layout: B is staged as two 64-row boxes.
//
// Two cluster shapes of the same code:
//   CTA2 = false : one CTA per 128 x BN tile.
//   CTA2 = true  : a cluster of two CTAs per 256 x BN tile: each CTA stages its own 128 rows of A and loads HALF of the
//                  B tile with a TMA multicast into both CTAs, so every weight byte fetched from L2 feeds two CTAs.
//                  A stage is refilled only when the consumers of BOTH CTAs have released it (remote mbarrier arrives).
//
// B-resident mode (b_res): when a CTA's whole weight tile W[n_blk*BN .. +BN, 0..K) fits in shared memory next to a few
// A stages (the K = 320 / 640 projections), every CTA keeps ONE n-tile for its lifetime, loads that weight tile once and
// streams only A tiles.
//
// conv_mode: the A operand is gathered by an im2col-mode TMA map over the NHWC activation (C, W, H, B): a load of tap
// (dy, dx) fills the 128 rows of an A stage with that tap's input pixel for 128 consecutive output pixels in (b, y, x)
// order, across row and image boundaries, and TMA's out-of-bounds zero fill implements the padding.  A 3x3 convolution is
// 9*Cin/64 K-steps of the same pipeline with no im2col buffer, and its 128-row blocks are those of a plain GEMM over the
// B*H*W output pixels, at any H and W.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"
#include "../../include/gligen_b200.h"

namespace glg {

struct GemmKParams {
  int M, N, num_kb, kb_per_tap;
  int tiles_m, tiles_n;          // tiles_m counts 128-row (CTA2: 256-row) blocks
  int conv, HW, Wd;
  void* out; long long ldc; int out_fp32;
  const float* bias; const float* rowbias; long long ld_rowbias; int rows_per_batch;
  int act; const float* gate; const bf16* residual; long long ldr;
  // LayerNorm fold (consumer side): per-row partial (sum, sumsq) of A over K, column sums of the weights
  const float* ln_stats; int ln_slots; const float* ln_colsum; float ln_eps; float inv_k;
  // producer side: per-row partial (sum, sumsq) of the values this GEMM stores
  float* stats_out; int stats_slots;
  // batch-strided output rows: address = (row / orpb) * obs + (row % orpb) * ldc   (orpb == 0: uniform rows)
  int orpb; long long obs;
  // split-K: `splits` CTAs share one output tile, each reducing a contiguous range of K steps into its own fp32
  // slab ws[split][M][N]; splitk_reduce_kernel sums the slabs in a fixed order and applies the epilogue.
  int splits; float* ws;
  int stages;                     // depth of the smem ring (runtime: B-resident mode trades stages for the weight tile)
  int b_res;                      // 1: weights resident in smem, one n-tile per CTA for its lifetime
  long long stats_stride;         // stats_out / ln_stats are SLOT-major: element (slot, row) at [slot * stride + row]
  long long ln_stride;
};

template <int BN, bool CTA2> struct GemmCfg {
  static constexpr int BM = 128, BK = 64;
  static constexpr int THREADS = 384;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int B_HALF = B_BYTES / 2;                         // CTA2: the share of B one CTA loads
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int MAX_STAGES = 12;
  static constexpr int BAR_BYTES = 1024;                             // barriers live in FRONT of the tiles (runtime stage count)
  static constexpr int SMEM_MAX = 227 * 1024;
  static_assert(8 * (2 * MAX_STAGES + 1) <= BAR_BYTES, "barrier area");
  static_assert(B_HALF % 1024 == 0, "each half of the B stage must keep the 1024-byte swizzle alignment");
};

__device__ __forceinline__ void setmaxnreg_dec40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void setmaxnreg_inc232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }
// named barriers 1 / 2 (0 is __syncthreads): the ping-pong MMA token of consumer warpgroup 0 / 1, 256 threads each
__device__ __forceinline__ void named_bar_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

// GEGLU: first packed weight row of the x half of n-tile n_blk of width BN (the gate rows follow 128 rows later).
// BN = 256 is one whole [128 x | 128 gate] block; BN = 128 is the upper or lower 64 x rows of one.
template <int BN> __device__ __forceinline__ int geglu_xrow(int n_blk) { return (n_blk * BN / 256) * 256 + (n_blk * (BN / 2)) % 128; }

__device__ __forceinline__ float act_f(int act, float v) {
  if (act == GLG_ACT_SILU) return silu_f(v);
  if (act == GLG_ACT_GELU) return gelu_erf_f(v);
  if (act == GLG_ACT_QUICK_GELU) return quick_gelu_f(v);
  return v;
}

// ---- epilogue of one 64-row x BN accumulator held by a consumer warpgroup ---------------------------------------
// wgmma m64nN D fragment: warp w of the warpgroup holds rows 16 w + lane / 4 (regs 4 j + 0, 1) and + 8 (regs 4 j + 2, 3),
// columns 8 j + 2 (lane % 4) + {0, 1}, for j = 0 .. N / 8 - 1.
// The epilogue walks 32-column chunks and issues every global load of a chunk (bias, LayerNorm column sums, row bias,
// residual; both rows of the thread) before the chunk's first store: the compiler cannot move a load across a store that
// may alias it, so loads interleaved with stores would cost one L2 round trip per 8 columns.
// ACT = false compiles the activation out: the fully unrolled epilogue is instruction-fetch bound, and the inlined
// SiLU / GELU / quick-GELU branches of every element (which no UNet projection takes) cost the GEMMs 14 % of their time.
template <int BN, bool GEGLU, bool ACT>
__device__ __forceinline__ void epilogue_tile(const GemmKParams& p, float (&d)[BN / 2], int row_base, int n_blk, float gate, int lane) {
  const int cq = 2 * (lane & 3);
  int row[2]; bool row_ok[2]; size_t out_off[2];
  float ln_rstd[2] = {1.f, 1.f}, c1[2] = {0.f, 0.f};     // LayerNorm fold: rstd * acc + (bias - rstd * mu * colsum)
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    row[hr] = row_base + hr * 8;
    row_ok[hr] = row[hr] < p.M;
    out_off[hr] = p.orpb ? (size_t)(row[hr] / p.orpb) * p.obs + (size_t)(row[hr] % p.orpb) * p.ldc : (size_t)row[hr] * p.ldc;
  }
  if (p.ln_stats) {
    const float2* sp = reinterpret_cast<const float2*>(p.ln_stats);
    const int r0 = row_ok[0] ? row[0] : 0, r1 = row_ok[1] ? row[1] : 0;
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
    for (int i = 0; i < p.ln_slots; ++i) {                 // fixed order
      const float2 t0 = __ldg(sp + (size_t)i * p.ln_stride + r0), t1 = __ldg(sp + (size_t)i * p.ln_stride + r1);
      s1[0] += t0.x; s2[0] += t0.y; s1[1] += t1.x; s2[1] += t1.y;
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const float mu = s1[hr] * p.inv_k;
      ln_rstd[hr] = rsqrtf(fmaxf(s2[hr] * p.inv_k - mu * mu, 0.f) + p.ln_eps);
      c1[hr] = -ln_rstd[hr] * mu;
    }
  }
  if constexpr (GEGLU) {
    constexpr int HALF = BN / 2;                    // tile columns [HALF x | HALF gate], packed weight rows x and x + 128
    const int xrow = geglu_xrow<BN>(n_blk);
#pragma unroll
    for (int ch = 0; ch < HALF / 32; ++ch) {
      float2 bx[4], bg[4], cx[4], cg[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int wcol = xrow + 32 * ch + 8 * jj + cq;
        bx[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + wcol));
        bg[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + wcol + 128));
        if (p.ln_stats) {
          cx[jj] = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + wcol));
          cg[jj] = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + wcol + 128));
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * ch + jj;
          float bx0 = bx[jj].x, bx1 = bx[jj].y, bg0 = bg[jj].x, bg1 = bg[jj].y;
          if (p.ln_stats) {
            bx0 = fmaf(cx[jj].x, c1[hr], bx0); bx1 = fmaf(cx[jj].y, c1[hr], bx1);
            bg0 = fmaf(cg[jj].x, c1[hr], bg0); bg1 = fmaf(cg[jj].y, c1[hr], bg1);
          }
          const float x0 = fmaf(d[4 * j + 2 * hr], ln_rstd[hr], bx0), x1 = fmaf(d[4 * j + 2 * hr + 1], ln_rstd[hr], bx1);
          const float g0 = fmaf(d[HALF / 2 + 4 * j + 2 * hr], ln_rstd[hr], bg0), g1 = fmaf(d[HALF / 2 + 4 * j + 2 * hr + 1], ln_rstd[hr], bg1);
          if (row_ok[hr])
            *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.out) + out_off[hr] + n_blk * HALF + 8 * j + cq) = pack_bf16x2(geglu_f(x0, g0), geglu_f(x1, g1));
        }
      }
    }
  } else {
    const float* rb[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) rb[hr] = (p.rowbias && row_ok[hr]) ? p.rowbias + (size_t)(row[hr] / p.rows_per_batch) * p.ld_rowbias : nullptr;
#pragma unroll
    for (int ch = 0; ch < BN / 32; ++ch) {          // 32-column chunks: one LayerNorm-statistics slot each
      float2 bias[4], cs[4], rbv[2][4];
      uint32_t res[2][4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int n0 = n_blk * BN + 32 * ch + 8 * jj + cq;
        bias[jj] = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n0)) : make_float2(0.f, 0.f);
        if (p.ln_stats) cs[jj] = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + n0));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          if (rb[hr]) rbv[hr][jj] = __ldg(reinterpret_cast<const float2*>(rb[hr] + n0));
          if (p.residual && row_ok[hr]) res[hr][jj] = __ldg(reinterpret_cast<const unsigned int*>(p.residual + (size_t)row[hr] * p.ldr + n0));
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float st_sum = 0.f, st_sq = 0.f;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * ch + jj;
          const int n0 = n_blk * BN + 8 * j + cq;
          float v0 = d[4 * j + 2 * hr], v1 = d[4 * j + 2 * hr + 1];
          if (p.ln_stats) {
            v0 = fmaf(v0, ln_rstd[hr], fmaf(cs[jj].x, c1[hr], bias[jj].x));
            v1 = fmaf(v1, ln_rstd[hr], fmaf(cs[jj].y, c1[hr], bias[jj].y));
          } else if (p.bias) { v0 += bias[jj].x; v1 += bias[jj].y; }
          if (rb[hr]) { v0 += rbv[hr][jj].x; v1 += rbv[hr][jj].y; }
          if constexpr (ACT) { v0 = act_f(p.act, v0); v1 = act_f(p.act, v1); }
          if (p.gate) { v0 *= gate; v1 *= gate; }
          if (p.residual && row_ok[hr]) {
            const float2 r = unpack_bf16x2(res[hr][jj]);
            v0 += r.x; v1 += r.y;
          }
          if (p.out_fp32) {
            if (row_ok[hr]) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + out_off[hr] + n0) = make_float2(v0, v1);
          } else {
            const uint32_t pk = pack_bf16x2(v0, v1);
            if (row_ok[hr]) *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.out) + out_off[hr] + n0) = pk;
            // statistics of the values AS STORED (bf16-rounded): exactly what the consumer GEMM reads
            const float2 f = unpack_bf16x2(pk);
            st_sum += f.x + f.y;
            st_sq = fmaf(f.x, f.x, fmaf(f.y, f.y, st_sq));
          }
        }
        if (p.stats_out && !p.out_fp32) {
          // one partial per 32-column chunk, slot = global chunk index: independent of the tile shape, so the consumer's
          // fixed-order sum is bit-identical whatever tile width produced the rows.  The four lanes of a row reduce in
          // a fixed butterfly order.
          st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 1); st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 1);
          st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 2); st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 2);
          if ((lane & 3) == 0 && row_ok[hr])
            reinterpret_cast<float2*>(p.stats_out)[(size_t)((n_blk * BN >> 5) + ch) * p.stats_stride + row[hr]] = make_float2(st_sum, st_sq);
        }
      }
    }
  }
}

// split-K: raw fp32 accumulators -> ws[split][row][n]
template <int BN>
__device__ __forceinline__ void epilogue_partial(const GemmKParams& p, const float (&d)[BN / 2], int row_base, int n_blk, int split, int lane) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = row_base + hr * 8;
    if (row >= p.M) continue;
    float* dst = p.ws + ((size_t)split * p.M + row) * p.N + (size_t)n_blk * BN + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(d[4 * j + 2 * hr], d[4 * j + 2 * hr + 1]);
  }
}

// out[row][n..n+7] = sum_s ws[s][row][n..] (fixed order) + bias + rowbias, SiLU, gate, + residual  -> bf16
__global__ void splitk_reduce_kernel(const GemmKParams p) {
  pdl_trigger();
  pdl_wait();
  const int nv = p.N >> 3;
  const long long total = (long long)p.M * nv;
  const float gate = p.gate ? __ldg(p.gate) : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / nv), n0 = (int)(i % nv) * 8;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < p.splits; ++s) {
      const float4* w4 = reinterpret_cast<const float4*>(p.ws + ((size_t)s * p.M + row) * p.N + n0);
      const float4 a = w4[0], b = w4[1];
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __ldg(p.bias + n0 + j);
    }
    if (p.rowbias) {
      const float* rb = p.rowbias + (size_t)(row / p.rows_per_batch) * p.ld_rowbias + n0;
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __ldg(rb + j);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = act_f(p.act, v[j]);
    if (p.gate) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= gate;
    }
    if (p.residual) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(p.residual + (size_t)row * p.ldr + n0));
      float2 f;
      f = unpack_bf16x2(u.x); v[0] += f.x; v[1] += f.y;
      f = unpack_bf16x2(u.y); v[2] += f.x; v[3] += f.y;
      f = unpack_bf16x2(u.z); v[4] += f.x; v[5] += f.y;
      f = unpack_bf16x2(u.w); v[6] += f.x; v[7] += f.y;
    }
    const size_t out_off = p.orpb ? (size_t)(row / p.orpb) * p.obs + (size_t)(row % p.orpb) * p.ldc : (size_t)row * p.ldc;
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]); o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(p.out) + out_off + n0) = o;
  }
}

template <int BN, bool GEGLU, bool CTA2, bool PP>
__global__ void __launch_bounds__(384, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) {
  using Cfg = GemmCfg<BN, CTA2>;
  constexpr int MAXST = Cfg::MAX_STAGES;
  constexpr int ROWS_PER_TILE = CTA2 ? 256 : 128;
  constexpr bool B_SPLIT = GEGLU && PP;                               // B staged as two BN/2-row boxes (x rows, gate rows)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t bar_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t base = bar_base + Cfg::BAR_BYTES;                   // tiles (1024-byte aligned)
  const int STAGES = p.stages;
  const bool bres = !CTA2 && p.b_res != 0;
  const uint32_t stage_bytes = bres ? (uint32_t)Cfg::A_BYTES : (uint32_t)Cfg::STAGE_BYTES;
  const uint32_t bres_base = base + (uint32_t)STAGES * Cfg::A_BYTES;  // resident weight tile: num_kb x [BN rows x 128 B]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (MAXST + s); };
  const uint32_t bfull_bar = bar_base + 8u * (2 * MAXST);
  // first weight row of half q (BN/2 rows) of the B tile of n-tile n_blk
  auto b_row = [&](int n_blk, int q) { return B_SPLIT ? geglu_xrow<BN>(n_blk) + q * 128 : n_blk * BN + q * (BN / 2); };

  pdl_trigger();          // the next kernel may start its prologue while this one runs (it waits before touching memory)
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t rank = CTA2 ? cluster_ctarank() : 0u;
  const int unit = CTA2 ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;          // CTA or CTA-pair index
  const int num_units = CTA2 ? (int)(gridDim.x >> 1) : (int)gridDim.x;

  if (threadIdx.x == 0) {
    // a stage is free again when every consumer warp that reads it (8 per CTA; ping-pong: the 4 of the owning warpgroup)
    // of every CTA that receives it has released it
    constexpr uint32_t releasers = (PP ? 4 : 8) * (CTA2 ? 2 : 1);
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), releasers); }
    mbar_init(bfull_bar, 1);
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) { tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB); }
  if constexpr (CTA2) cluster_sync_all(); else __syncthreads();
  pdl_wait();             // everything above overlapped the previous kernel's tail; global data is touched only below

  const int total_work = p.tiles_m * p.tiles_n * p.splits;
  // work item `it` of this CTA (pair) -> (m_blk, n_blk, split).  Streaming: round robin over all (tile, split) items.
  // B-resident: the CTA keeps n-tile unit % tiles_n and walks m-blocks (the grid is a whole multiple of tiles_n).
  const int per_n = bres ? num_units / p.tiles_n : 1;
  auto get_work = [&](int it, int& tile, int& split, int& m_blk, int& n_blk) -> bool {
    if (bres) {
      n_blk = unit % p.tiles_n;
      m_blk = unit / p.tiles_n + it * per_n;
      split = 0;
      tile = m_blk * p.tiles_n + n_blk;
      return m_blk < p.tiles_m;
    }
    const int work = unit + it * num_units;
    if (work >= total_work) return false;
    tile = work / p.splits; split = work - tile * p.splits;
    m_blk = tile / p.tiles_n; n_blk = tile - m_blk * p.tiles_n;
    return true;
  };

  if (wg == 0) {
    setmaxnreg_dec40();
    if (warp == 0) {
      // ===================== TMA producer: whole warp walks the loop, one elected lane issues =====================
      const bool leader = elect_one();
      int stage = 0; uint32_t phase = 0;
      if (bres && leader) {
        // the CTA's weight tile, once: num_kb boxes of [BN rows x 64 columns] on one barrier
        const int nblk = unit % p.tiles_n;
        mbar_arrive_expect_tx(bfull_bar, (uint32_t)p.num_kb * Cfg::B_BYTES);
        for (int kb = 0; kb < p.num_kb; ++kb) {
          const uint32_t dst = bres_base + (uint32_t)kb * Cfg::B_BYTES;
          tma_load_2d(dst, &tmB, bfull_bar, kb * 64, b_row(nblk, 0));
          if constexpr (B_SPLIT) tma_load_2d(dst + Cfg::B_HALF, &tmB, bfull_bar, kb * 64, b_row(nblk, 1));
        }
      }
      int tile, split, m_blk, n_blk;
      for (int it = 0; get_work(it, tile, split, m_blk, n_blk); ++it) {
        const int kb_lo = (split * p.num_kb) / p.splits, kb_n = ((split + 1) * p.num_kb) / p.splits - kb_lo;
        const int row0 = m_blk * ROWS_PER_TILE + (int)rank * 128;
        int b0 = 0, y0 = 0, x0 = 0;                    // conv: the tile's first output pixel
        if (p.conv) {
          b0 = row0 / p.HW;
          y0 = (row0 - b0 * p.HW) / p.Wd;
          x0 = row0 - b0 * p.HW - y0 * p.Wd;
        }
        // K steps are visited in a per-tile rotated order: tiles running at the same time would otherwise request
        // the very same weight (and activation) lines from L2 in lockstep; the rotation spreads them over slices.
        // (fp32 accumulation order depends only on the tile index -> results stay reproducible.)  B-resident tiles
        // fetch no weights per tile and walk K in order (the consumers index the resident tile by K step).
        int kb = bres ? kb_lo : kb_lo + (int)(((unsigned)tile * 3u) % (unsigned)kb_n);
        for (int it2 = 0; it2 < kb_n; ++it2, kb = (kb + 1 == kb_lo + kb_n) ? kb_lo : kb + 1) {
          mbar_wait<false>(empty_bar(stage), phase ^ 1u);
          const uint32_t a_dst = base + stage * stage_bytes;
          const uint32_t b_dst = a_dst + Cfg::A_BYTES;
          if (leader) {
            mbar_arrive_expect_tx(full_bar(stage), bres ? Cfg::A_BYTES : Cfg::STAGE_BYTES);
            int ca = kb * 64, cb_off = 0;
            if (p.conv) {
              const int tap = kb / p.kb_per_tap;
              const int cb = kb - tap * p.kb_per_tap;
              const int dy = tap / 3, dx = tap - (tap / 3) * 3;
              // bounding-box start (x0 - 1, y0 - 1): tap (0, 0) of the first output pixel
              tma_load_im2col_4d(a_dst, &tmA, full_bar(stage), cb * 64, x0 - 1, y0 - 1, b0, (uint16_t)dx, (uint16_t)dy);
              ca = cb * 64; cb_off = tap * p.N;
            } else {
              tma_load_2d(a_dst, &tmA, full_bar(stage), kb * 64, row0);
            }
            if constexpr (CTA2) {
              tma_load_2d_mc(b_dst + rank * Cfg::B_HALF, &tmB, full_bar(stage), ca, cb_off + b_row(n_blk, (int)rank), (uint16_t)3);
            } else if (!bres) {
              if constexpr (B_SPLIT) {
                tma_load_2d(b_dst, &tmB, full_bar(stage), ca, cb_off + b_row(n_blk, 0));
                tma_load_2d(b_dst + Cfg::B_HALF, &tmB, full_bar(stage), ca, cb_off + b_row(n_blk, 1));
              } else {
                tma_load_2d(b_dst, &tmB, full_bar(stage), ca, cb_off + n_blk * BN);
              }
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== consumers =====================
    // cooperative: warpgroup 1 / 2 own accumulator rows [0, 64) / [64, 128) of every item;
    // ping-pong: warpgroup 1 / 2 own the even / odd items of this CTA, all 128 rows (accumulator halves d[0], d[1])
    setmaxnreg_inc232();
    const int cw = wg - 1;
    constexpr int MH = PP ? 2 : 1;
    const float gate = p.gate ? __ldg(p.gate) : 1.0f;
    uint32_t empty0 = empty_bar(0), empty0_peer = 0;
    if constexpr (CTA2) empty0_peer = mapa_cluster(empty_bar(0), rank ^ 1u);
    if (bres) mbar_wait<false>(bfull_bar, 0);
    int stage = 0; uint32_t phase = 0;
    auto release = [&](int s) {
      if (lane == 0) {
        mbar_arrive(empty0 + 8u * s);
        if constexpr (CTA2) mbar_arrive_cluster(empty0_peer + 8u * s);
      }
    };
    float d[MH][BN / 2];
    int tile, split, m_blk, n_blk;
    for (int it = 0; get_work(it, tile, split, m_blk, n_blk); ++it) {
      const int kb_n = ((split + 1) * p.num_kb) / p.splits - (split * p.num_kb) / p.splits;
      if (PP && (it & 1) != cw) {                // the other warpgroup's item: step over its stages
        stage += kb_n;
        while (stage >= STAGES) { stage -= STAGES; phase ^= 1u; }
        continue;
      }
      if (PP && it > 0) named_bar_sync(1 + cw);  // the MMA token, passed on by the owner of item it - 1
      int prev = -1;
      for (int kb = 0; kb < kb_n; ++kb) {
        mbar_wait<false>(full_bar(stage), phase);
        const uint32_t a_addr = base + stage * stage_bytes + (uint32_t)(PP ? 0 : cw) * (64 * 128);
        const uint64_t bdesc = gmma_desc_kmajor_sw128(bres ? bres_base + (uint32_t)kb * Cfg::B_BYTES : base + stage * stage_bytes + Cfg::A_BYTES);
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) wgmma_fence_regs(d[mh]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {    // 4 x K=16 inside one 64-wide (128 B) swizzle atom: +32 B per step
#pragma unroll
          for (int mh = 0; mh < MH; ++mh)
            Wgmma<BN>::mma(d[mh], gmma_desc_kmajor_sw128(a_addr + (uint32_t)mh * (64 * 128)) + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                 // the previous stage's MMAs are done: hand its buffers back to the producer
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) wgmma_fence_regs(d[mh]);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      if constexpr (PP) {                        // all MMAs of this item are issued: pass the token to the next item's owner
        int t2, s2, m2, n2;
        if (get_work(it + 1, t2, s2, m2, n2)) named_bar_arrive(2 - cw);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) wgmma_fence_regs(d[mh]);
      if (prev >= 0) release(prev);
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) {
        const int row_base = m_blk * ROWS_PER_TILE + (int)rank * 128 + (PP ? mh : cw) * 64 + (warp & 3) * 16 + (lane >> 2);
        if (p.splits > 1) epilogue_partial<BN>(p, d[mh], row_base, n_blk, split, lane);
        else if (!GEGLU && p.act) epilogue_tile<BN, GEGLU, true>(p, d[mh], row_base, n_blk, gate, lane);
        else epilogue_tile<BN, GEGLU, false>(p, d[mh], row_base, n_blk, gate, lane);
      }
    }
  }
  // no CTA of a pair may exit while its peer can still multicast into its smem or arrive on its barriers
  if constexpr (CTA2) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// launch
// ------------------------------------------------------------------------------------------------
template <int BN, bool GEGLU, bool CTA2, bool PP>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, size_t smem, cudaStream_t st) {
  using Cfg = GemmCfg<BN, CTA2>;
  static bool attr_set = false;
  auto kern = gemm_tc_kernel<BN, GEGLU, CTA2, PP>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_MAX);
    if (e != cudaSuccess) return set_error(std::string("cudaFuncSetAttribute(gemm): ") + cudaGetErrorString(e));
    attr_set = true;
  }
  const int tiles = p.tiles_m * p.tiles_n * p.splits;
  int grid;
  if (p.b_res) {
    grid = (num_sms() / p.tiles_n) * p.tiles_n;          // one n-tile per CTA for its lifetime
  } else if (CTA2) {
    const int pairs = num_sms() / 2;
    grid = 2 * (tiles < pairs ? tiles : pairs);
  } else {
    grid = tiles < num_sms() ? tiles : num_sms();
  }
  cudaError_t e = launch_k(kern, dim3(grid), dim3(Cfg::THREADS), smem, st, CTA2 ? 2 : 1, ta, tb, p);
  count_launch();
  if (e != cudaSuccess) return set_error(std::string("gemm launch: ") + cudaGetErrorString(e));
  if (check_launch("gemm launch")) return -1;
  if (p.splits > 1) {
    const long long total = (long long)p.M * (p.N / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    e = launch_k(splitk_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, st, 1, p);
    count_launch();
    if (e != cudaSuccess) return set_error(std::string("splitk reduce launch: ") + cudaGetErrorString(e));
    return check_launch("splitk reduce launch");
  }
  return 0;
}

int g_force_bn = 0;     // test hooks (glg_debug_force_bn / glg_debug_gemm_cta2 / glg_debug_splitk)
int g_splitk_mode = 0;  // 0 = heuristic, 1 = never, 2 = split whenever legal
int g_cta2_mode = -1;   // 0 = heuristic, 1 = never pair, 2 = pair whenever legal; -1 = read GLG_GEMM_CTA2 (default 0)
int g_bres_mode = -1;   // B-resident tiles: 0 = heuristic, 1 = never, 2 = whenever legal; -1 = read GLG_GEMM_BRES (default 1)
int g_pp_mode = 0;      // ping-pong consumers (glg_debug_gemm_pp): 0 = heuristic, 1 = never, 2 = whenever legal

static constexpr long long kTileMax = 227 * 1024 - 1024 - 1024;     // dynamic smem minus alignment slack and barriers

// A stages left beside a resident [BN x K] weight tile (0: does not fit)
static int bres_stages(int bn, int num_kb) {
  const long long left = kTileMax - (long long)num_kb * bn * 128;
  if (left < 3 * 16384) return 0;
  const int st = (int)(left / 16384);
  return st > 12 ? 12 : st;
}

// Tile / split choice by a small time model (cycles, H100 data-sheet rates, not tuned by measurement):
//   per 64-wide K step an SM needs max(MMA = 4*BN: 128 x BN x 64 MACs at 2048 bf16 MAC/clk, operand bytes / ~32 B/clk of
//   L2->SM bandwidth) cycles (a pair stages 128 + BN/2 operand rows per SM instead of 128 + BN); a CTA pays ~3000 cycles
//   of fixed cost per work item; split-K adds a reduce pass over splits * M * N fp32.  The least estimated time wins.
// Schedule: ping-pong only where a forced-tile sweep (scripts/sweep_bn.py, H100 80GB HBM3 at 400 W) measured it ahead of
// every cooperative tile: 3x3 convolutions with M >= 8192 on 64-wide tiles (SD levels 0-1 at 8 rows: 0.72-0.87x the
// time of the cooperative tile the model picks) and GEGLU with M <= 512 (0.87x).  Elsewhere it measured level or slower.
static bool pingpong_pays(int M, int bn, bool geglu, bool conv) {
  return (conv && M >= 8192 && bn == 64) || (geglu && M <= 512);
}

static void pick_tile(int M, int N, int num_kb, bool geglu, bool conv, int max_splits, long long ws_bytes,
                      int* bn_out, int* cta2_out, int* splits_out, int* bres_out, int* pp_out) {
  if (g_cta2_mode < 0) {
    const char* e = getenv("GLG_GEMM_CTA2");
    g_cta2_mode = e ? atoi(e) : 0;
  }
  if (g_bres_mode < 0) {
    const char* e = getenv("GLG_GEMM_BRES");
    g_bres_mode = e ? atoi(e) : 1;      // opt-in
  }
  const int sms = num_sms();
  const int cands[4] = {256, 160, 128, 64};
  float best = 1e30f; int best_bn = 0, best_pair = 0, best_s = 1, best_res = 0, best_pp = 0;
  for (int pair = 0; pair < 2; ++pair) {
    if (pair && (g_cta2_mode == 1 || M <= 128)) continue;
    // the heuristic pairs only large, long-K plain GEMMs with N % 256 == 0 and the larger 3x3 convolutions
    if (pair && g_cta2_mode == 0 && !conv && (N % 256 || num_kb < 16 || M < 4096)) continue;
    if (pair && g_cta2_mode == 0 && conv && M < 2048) continue;
    if (!pair && g_cta2_mode == 2 && M > 128) {
      bool any = false;
      for (int i = 0; i < 3; ++i) any |= (N % cands[i] == 0) && (!geglu || cands[i] == 256);
      if (any) continue;
    }
    for (int i = 0; i < 4; ++i) {
      const int bn = cands[i];
      if (N % bn) continue;
      if (geglu && bn != 256) continue;
      if (g_force_bn && bn != g_force_bn && (N % g_force_bn == 0) && !geglu) continue;
      if (pair && bn < 128) continue;                    // per-CTA half of B must stay a whole number of KiB
      if (pair && g_cta2_mode == 0 && !conv && bn != 256) continue;
      for (int pp = 0; pp < 2; ++pp) {
        // ping-pong holds 128 x BN fp32 accumulators per warpgroup in 168 registers: BN <= 128 (GEGLU: 128-row halves of
        // the 256 tile); 128 x 160 spills
        if (pp && (g_pp_mode == 1 || (!geglu && bn > 128))) continue;
        if (pp && g_pp_mode == 0 && !pingpong_pays(M, bn, geglu, conv)) continue;
        const int kbn = (pp && geglu) ? 128 : bn;        // width of one work item
        // ping-pong where it measured ahead (heuristic) or wherever legal (test hook): preferred over every cooperative tile
        const float force = pp ? 1e-3f : 1.0f;
        const int rows = pair ? 256 : 128;
        const int tiles = ((M + rows - 1) / rows) * (N / kbn);
        const int units = pair ? sms / 2 : sms;
        const float mma = 4.0f * kbn;
        const float l2 = 4.0f * (pair ? 128.0f + 0.5f * kbn : 128.0f + kbn);
        const float per_kb = mma > l2 ? mma : l2;
        for (int sp = 1; sp <= (pair ? 1 : max_splits); ++sp) {
          if (sp > 1 && (num_kb / sp < (g_splitk_mode == 2 ? 4 : 16) || (long long)sp * M * N * 4 > ws_bytes)) break;
          if (sp > 1 && tiles * 2 > units && g_splitk_mode != 2) break;        // only when the tile grid leaves >= half the SMs idle
          if (g_splitk_mode == 2 && max_splits > 1 && sp == 1 && num_kb >= 8) continue;      // test hook: force a split
          const int waves = (tiles * sp + units - 1) / units;
          const int kb_cta = (num_kb + sp - 1) / sp;
          float t = (float)waves * (per_kb * kb_cta + 3000.0f);
          if (sp > 1) t += 12000.0f + (float)sp * M * N * 4.0f / (sms * 40.0f);     // slab round trip + reduce launch
          const int ctas = (pair ? 2 : 1) * (tiles * sp < units ? tiles * sp : units);
          t *= 1.0f + 0.10f * (1.0f - (float)ctas / (float)sms);     // idle SMs: prefer the finer decomposition
          t *= force;
          if (t < best) { best = t; best_bn = bn; best_pair = pair; best_s = sp; best_res = 0; best_pp = pp; }
        }
        // B-resident: one n-tile per CTA, weights loaded once per CTA, only A streams (plain GEMMs, single CTAs)
        const int tiles_n = N / kbn, tiles_m = (M + 127) / 128;
        if (!pair && !conv && g_bres_mode != 1 && tiles_n <= sms && bres_stages(kbn, num_kb) > 0) {
          const int per_n = sms / tiles_n;
          if (tiles_m >= 2 * per_n || g_bres_mode == 2) {
            const int waves = (tiles_m + per_n - 1) / per_n;
            const float l2a = 4.0f * 128.0f;
            float t = (float)waves * ((mma > l2a ? mma : l2a) * num_kb + 3000.0f) + 4.0f * kbn * num_kb;
            const int ctas = per_n * tiles_n;
            t *= 1.0f + 0.10f * (1.0f - (float)ctas / (float)sms);
            if (g_bres_mode == 2) t = -1.0f / (float)bn / force;   // test hook: force (widest legal tile)
            else t *= force;
            if (t < best) { best = t; best_bn = bn; best_pair = 0; best_s = 1; best_res = 1; best_pp = pp; }
          }
        }
      }
    }
  }
  *bn_out = best_bn; *cta2_out = best_pair; *splits_out = best_s; *bres_out = best_res; *pp_out = best_pp;
}

}  // namespace glg

using namespace glg;

extern "C" void glg_debug_force_bn(int bn) { glg::g_force_bn = bn; }
// test hook (host only, no CUDA work): what the tile picker chooses for a problem; out[3] = {BN, paired CTAs, K splits}
extern "C" void glg_debug_pick_tile(int M, int N, int K, int geglu, int conv, int can_split, long long ws_bytes, int* out) {
  int bres = 0, pp = 0;
  glg::pick_tile(M, N, (conv ? 9 : 1) * (K / 64), geglu != 0, conv != 0, can_split ? 8 : 1, ws_bytes, &out[0], &out[1], &out[2], &bres, &pp);
  out[1] |= bres << 8;           // bit 8 of the "paired" word: B-resident
}
// test hook (host only): 1 when the tile picker runs the problem on the ping-pong schedule
extern "C" int glg_debug_pick_pingpong(int M, int N, int K, int geglu, int conv, int can_split, long long ws_bytes) {
  int bn, pair, sp, bres, pp = 0;
  glg::pick_tile(M, N, (conv ? 9 : 1) * (K / 64), geglu != 0, conv != 0, can_split ? 8 : 1, ws_bytes, &bn, &pair, &sp, &bres, &pp);
  return pp;
}
extern "C" void glg_debug_gemm_pp(int mode) { glg::g_pp_mode = mode; }
extern "C" void glg_debug_gemm_bres(int mode) { glg::g_bres_mode = mode; }
extern "C" void glg_debug_gemm_cta2(int mode) { glg::g_cta2_mode = mode; }
extern "C" void glg_debug_splitk(int mode) { glg::g_splitk_mode = mode; }

extern "C" int glg_gemm(const GlgGemmArgs* a, void* stream) {
  if (!a) return set_error("glg_gemm: null args");
  if (a->K <= 0 || a->K % 64) return set_error("glg_gemm: K must be a positive multiple of 64");
  if (a->M <= 0 || a->N <= 0) return set_error("glg_gemm: M, N must be positive");
  if ((a->lda % 8) || (a->ldc % 8) || (a->residual && (a->ldr % 8))) return set_error("glg_gemm: leading dims must be multiples of 8");
  if (((uintptr_t)a->A | (uintptr_t)a->W | (uintptr_t)a->out | (uintptr_t)a->residual) & 15) return set_error("glg_gemm: pointers must be 16-byte aligned");
  if (a->rowbias && ((a->ld_rowbias % 4) || a->rows_per_batch <= 0)) return set_error("glg_gemm: bad rowbias args");
  if (a->geglu && (a->N % 256 || !a->bias || a->out_fp32)) return set_error("glg_gemm: geglu needs N % 256 == 0, a bias and bf16 output");
  int bn = 0, cta2 = 0, splits = 1, bres = 0, pp = 0;
  const bool can_split = a->splitk_ws && g_splitk_mode != 1 && !a->geglu && !a->ln_stats && !a->stats_out && !a->out_fp32 &&
                         !((uintptr_t)a->splitk_ws & 15);
  pick_tile(a->M, a->N, (a->conv_mode ? 9 : 1) * (a->K / 64), a->geglu != 0, a->conv_mode != 0, can_split ? 8 : 1,
            a->splitk_ws_bytes, &bn, &cta2, &splits, &bres, &pp);
  if (!bn) return set_error("glg_gemm: N must be a multiple of 64");
  const int kbn = (pp && a->geglu) ? 128 : bn;                     // width of one work item (ping-pong GEGLU: half a packed tile)
  GemmKParams p;
  memset(&p, 0, sizeof(p));
  const int rows_per_tile = cta2 ? 256 : 128;
  p.M = a->M; p.N = a->N;
  p.kb_per_tap = a->K / 64;
  p.num_kb = a->conv_mode ? 9 * p.kb_per_tap : p.kb_per_tap;
  p.tiles_m = (a->M + rows_per_tile - 1) / rows_per_tile;
  p.tiles_n = a->N / kbn;
  p.conv = a->conv_mode;
  p.out = a->out; p.ldc = a->ldc; p.out_fp32 = a->out_fp32;
  p.bias = a->bias; p.rowbias = a->rowbias; p.ld_rowbias = a->ld_rowbias; p.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : 1;
  p.act = a->act; p.gate = a->gate; p.residual = reinterpret_cast<const bf16*>(a->residual); p.ldr = a->ldr;
  if (a->ln_stats) {
    if (!a->ln_colsum || a->ln_slots <= 0 || a->conv_mode) return set_error("glg_gemm: LayerNorm fold needs ln_colsum, ln_slots > 0 and a plain GEMM");
    if (((uintptr_t)a->ln_stats & 7) || ((uintptr_t)a->ln_colsum & 15)) return set_error("glg_gemm: ln_stats / ln_colsum alignment");
    if (a->ln_slot_stride > 0 && a->ln_slot_stride < a->M) return set_error("glg_gemm: ln_slot_stride < M");
    p.ln_stats = a->ln_stats; p.ln_slots = a->ln_slots; p.ln_colsum = a->ln_colsum; p.ln_eps = a->ln_eps; p.inv_k = 1.0f / (float)a->K;
  }
  if (a->stats_out) {
    if (a->geglu || a->out_fp32 || a->stats_slots * 32 != a->N || ((uintptr_t)a->stats_out & 7))
      return set_error("glg_gemm: stats_out needs a bf16 non-GEGLU output and stats_slots == N / 32");
    p.stats_out = a->stats_out; p.stats_slots = a->stats_slots;
  }
  if (a->out_rows_per_batch > 0) {
    if (a->out_batch_stride % 8) return set_error("glg_gemm: out_batch_stride must be a multiple of 8");
    p.orpb = a->out_rows_per_batch; p.obs = a->out_batch_stride;
  }
  if (a->bias && ((uintptr_t)a->bias & 15)) return set_error("glg_gemm: bias must be 16-byte aligned");

  p.splits = splits;
  p.ws = splits > 1 ? reinterpret_cast<float*>(a->splitk_ws) : nullptr;
  p.b_res = bres;
  const long long stage_bytes = bres ? 16384 : 128 * 128 + kbn * 128;
  const long long fixed = bres ? (long long)p.num_kb * kbn * 128 : 0;
  long long stages = (kTileMax - fixed) / stage_bytes;
  const int cap = bres ? 12 : 8;
  p.stages = (int)(stages > cap ? cap : stages);
  if (p.stages < 2) return set_error("glg_gemm: internal: shared memory budget");
  const size_t smem = (size_t)(p.stages * stage_bytes + fixed) + 1024 + 1024;
  if (a->stats_out) p.stats_stride = a->stats_slot_stride > 0 ? a->stats_slot_stride : a->M;
  if (a->ln_stats) p.ln_stride = a->ln_slot_stride > 0 ? a->ln_slot_stride : a->M;

  // a pair: each CTA multicasts half of the B tile; ping-pong GEGLU: x and gate rows are two boxes
  const uint32_t brows = (uint32_t)(cta2 || (pp && a->geglu) ? kbn / 2 : kbn);
  CUtensorMap ta, tb;
  if (a->conv_mode) {
    const int H = a->H, W = a->Wd, B = a->Bn;
    if (H <= 0 || W <= 0 || B <= 0 || (long long)B * H * W != a->M) return set_error("glg_gemm: conv dims do not match M");
    const int HW = H * W;
    p.HW = HW; p.Wd = W;
    const uint64_t dims[4] = {(uint64_t)a->K, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[3] = {(uint64_t)a->lda * 2, (uint64_t)a->lda * 2 * W, (uint64_t)a->lda * 2 * HW};
    if (get_tmap_bf16_im2col3x3(&ta, a->A, dims, str, 64, 128)) return -1;
    const uint64_t wd[2] = {(uint64_t)a->K, (uint64_t)a->N * 9};
    const uint64_t ws[1] = {(uint64_t)a->K * 2};
    const uint32_t wb[2] = {64, brows};
    if (get_tmap_bf16(&tb, a->W, 2, wd, ws, wb)) return -1;
  } else {
    const uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
    const uint64_t str[1] = {(uint64_t)a->lda * 2};
    const uint32_t box[2] = {64, 128};
    if (get_tmap_bf16(&ta, a->A, 2, dims, str, box)) return -1;
    const uint64_t wd[2] = {(uint64_t)a->K, (uint64_t)a->N};
    const uint64_t ws[1] = {(uint64_t)a->K * 2};
    const uint32_t wb[2] = {64, brows};
    if (get_tmap_bf16(&tb, a->W, 2, wd, ws, wb)) return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (pp) {
    if (cta2) {
      if (a->geglu) return launch_gemm<128, true, true, true>(ta, tb, p, smem, st);
      switch (bn) {
        case 128: return launch_gemm<128, false, true, true>(ta, tb, p, smem, st);
      }
    } else {
      if (a->geglu) return launch_gemm<128, true, false, true>(ta, tb, p, smem, st);
      switch (bn) {
        case 128: return launch_gemm<128, false, false, true>(ta, tb, p, smem, st);
        case 64:  return launch_gemm<64, false, false, true>(ta, tb, p, smem, st);
      }
    }
  } else if (cta2) {
    if (a->geglu) return launch_gemm<256, true, true, false>(ta, tb, p, smem, st);
    switch (bn) {
      case 256: return launch_gemm<256, false, true, false>(ta, tb, p, smem, st);
      case 160: return launch_gemm<160, false, true, false>(ta, tb, p, smem, st);
      case 128: return launch_gemm<128, false, true, false>(ta, tb, p, smem, st);
    }
  } else {
    if (a->geglu) return launch_gemm<256, true, false, false>(ta, tb, p, smem, st);
    switch (bn) {
      case 256: return launch_gemm<256, false, false, false>(ta, tb, p, smem, st);
      case 160: return launch_gemm<160, false, false, false>(ta, tb, p, smem, st);
      case 128: return launch_gemm<128, false, false, false>(ta, tb, p, smem, st);
      case 64:  return launch_gemm<64, false, false, false>(ta, tb, p, smem, st);
    }
  }
  return set_error("glg_gemm: internal: bad tile");
}
