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
//
// Epilogue kinds (EPI): the epilogue is unrolled over every element of the tile, and its time follows the length of that
// code rather than its memory traffic (DESIGN §5).  So each epilogue flag the production plans combine is a compile-time
// bit: a false bit removes that flag's loads, arithmetic and branches.  Each kind's kernels live in a namespace of their
// own, `glg::<kind>::gemm_tc_kernel<BN, GEGLU, CTA2, PP>`, instantiated only for the tiles the plans pick with that kind
// (GLG_GEMM_INSTANCES_*, spread over the gemm_tc_bn*.cu units); every other combination runs `epi_generic`, which reads
// every flag at run time.  The header is shared by gemm_tc.cu (tile picker, dispatch) and those units.
#pragma once
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

// epilogue kind bits.  EPI_GENERIC reads every flag from GemmKParams at run time; its kernel holds two epilogue copies,
// with and without the activation, and picks one per launch from p.act.
enum : int {
  EPI_LN = 1, EPI_BIAS = 2, EPI_ROWBIAS = 4, EPI_GATE = 8, EPI_RES = 16, EPI_STATS = 32, EPI_F32 = 64, EPI_ORPB = 128,
  EPI_ACT = 256, EPI_GENERIC = 512,
};

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
// EPI (the epilogue kind) fixes which flags exist at compile time; EPI_GENERIC tests each at run time.  Every element
// that remains goes through the same operations in the same order whichever kind runs it.  Without EPI_ACT the
// activation is compiled out: the inlined SiLU / GELU / quick-GELU branches of every element cost the GEMMs 14 % of
// their time when they were present but not taken.
template <int BN, bool GEGLU, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmKParams& p, float (&d)[BN / 2], int row_base, int n_blk, float gate, int lane) {
  constexpr bool GEN = (EPI & EPI_GENERIC) != 0, ACT = (EPI & EPI_ACT) != 0;
  const bool has_ln = GEN ? p.ln_stats != nullptr : (EPI & EPI_LN) != 0;
  const bool has_bias = GEN ? p.bias != nullptr : (EPI & EPI_BIAS) != 0;
  const bool has_rowbias = GEN ? p.rowbias != nullptr : (EPI & EPI_ROWBIAS) != 0;
  const bool has_gate = GEN ? p.gate != nullptr : (EPI & EPI_GATE) != 0;
  const bool has_res = GEN ? p.residual != nullptr : (EPI & EPI_RES) != 0;
  const bool has_stats = GEN ? p.stats_out != nullptr : (EPI & EPI_STATS) != 0;
  const bool out_f32 = GEN ? p.out_fp32 != 0 : (EPI & EPI_F32) != 0;
  const bool has_orpb = GEN ? p.orpb != 0 : (EPI & EPI_ORPB) != 0;
  const int cq = 2 * (lane & 3);
  int row[2]; bool row_ok[2]; size_t out_off[2];
  float ln_rstd[2] = {1.f, 1.f}, c1[2] = {0.f, 0.f};     // LayerNorm fold: rstd * acc + (bias - rstd * mu * colsum)
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    row[hr] = row_base + hr * 8;
    row_ok[hr] = row[hr] < p.M;
    out_off[hr] = has_orpb ? (size_t)(row[hr] / p.orpb) * p.obs + (size_t)(row[hr] % p.orpb) * p.ldc : (size_t)row[hr] * p.ldc;
  }
  if (has_ln) {
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
        if (has_ln) {
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
          if (has_ln) {
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
    for (int hr = 0; hr < 2; ++hr) rb[hr] = (has_rowbias && row_ok[hr]) ? p.rowbias + (size_t)(row[hr] / p.rows_per_batch) * p.ld_rowbias : nullptr;
#pragma unroll
    for (int ch = 0; ch < BN / 32; ++ch) {          // 32-column chunks: one LayerNorm-statistics slot each
      float2 bias[4], cs[4], rbv[2][4];
      uint32_t res[2][4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int n0 = n_blk * BN + 32 * ch + 8 * jj + cq;
        bias[jj] = has_bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n0)) : make_float2(0.f, 0.f);
        if (has_ln) cs[jj] = __ldg(reinterpret_cast<const float2*>(p.ln_colsum + n0));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          if (rb[hr]) rbv[hr][jj] = __ldg(reinterpret_cast<const float2*>(rb[hr] + n0));
          if (has_res && row_ok[hr]) res[hr][jj] = __ldg(reinterpret_cast<const unsigned int*>(p.residual + (size_t)row[hr] * p.ldr + n0));
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
          if (has_ln) {
            v0 = fmaf(v0, ln_rstd[hr], fmaf(cs[jj].x, c1[hr], bias[jj].x));
            v1 = fmaf(v1, ln_rstd[hr], fmaf(cs[jj].y, c1[hr], bias[jj].y));
          } else if (has_bias) { v0 += bias[jj].x; v1 += bias[jj].y; }
          if (rb[hr]) { v0 += rbv[hr][jj].x; v1 += rbv[hr][jj].y; }
          if constexpr (ACT) { v0 = act_f(p.act, v0); v1 = act_f(p.act, v1); }
          if (has_gate) { v0 *= gate; v1 *= gate; }
          if (has_res && row_ok[hr]) {
            const float2 r = unpack_bf16x2(res[hr][jj]);
            v0 += r.x; v1 += r.y;
          }
          if (out_f32) {
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
        if (has_stats && !out_f32) {
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

// The whole kernel; each epilogue kind's __global__ wrapper below inlines it.
template <int BN, bool GEGLU, bool CTA2, bool PP, int EPI>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmKParams& p) {
  using Cfg = GemmCfg<BN, CTA2>;
  constexpr int MAXST = Cfg::MAX_STAGES;
  constexpr int ROWS_PER_TILE = CTA2 ? 256 : 128;
  constexpr bool B_SPLIT = GEGLU && PP;                               // B staged as two BN/2-row boxes (x rows, gate rows)
  constexpr bool MAY_SPLIT = EPI == 0 || (EPI & EPI_GENERIC) != 0;
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
        // split-K items store raw partials: the dispatch gives them kind 0 (or the generic kernel)
        if (MAY_SPLIT && p.splits > 1) epilogue_partial<BN>(p, d[mh], row_base, n_blk, split, lane);
        else if constexpr ((EPI & EPI_GENERIC) != 0) {
          if (!GEGLU && p.act) epilogue_tile<BN, GEGLU, EPI | EPI_ACT>(p, d[mh], row_base, n_blk, gate, lane);
          else epilogue_tile<BN, GEGLU, EPI>(p, d[mh], row_base, n_blk, gate, lane);
        } else {
          epilogue_tile<BN, GEGLU, EPI>(p, d[mh], row_base, n_blk, gate, lane);
        }
      }
    }
  }
  // no CTA of a pair may exit while its peer can still multicast into its smem or arrive on its barriers
  if constexpr (CTA2) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// epilogue kinds and their kernels
// ------------------------------------------------------------------------------------------------
// (namespace, EPI) of every kind.  Kinds other than epi_generic are exact: a launch gets one only when its runtime flags
// are those bits (gemm_tc.cu epilogue_kind).
#define GLG_GEMM_EPI_KINDS(X)                                                  \
  X(epi_generic, EPI_GENERIC)                                                  \
  X(epi_none, 0)                                                               \
  X(epi_bias, EPI_BIAS)                                                        \
  X(epi_bias_act, EPI_BIAS | EPI_ACT)                                          \
  X(epi_bias_f32, EPI_BIAS | EPI_F32)                                          \
  X(epi_bias_rowbias, EPI_BIAS | EPI_ROWBIAS)                                  \
  X(epi_bias_res, EPI_BIAS | EPI_RES)                                          \
  X(epi_bias_stats, EPI_BIAS | EPI_STATS)                                      \
  X(epi_bias_res_stats, EPI_BIAS | EPI_RES | EPI_STATS)                        \
  X(epi_bias_gate_res_stats, EPI_BIAS | EPI_GATE | EPI_RES | EPI_STATS)        \
  X(epi_ln_bias, EPI_LN | EPI_BIAS)                                            \
  X(epi_ln_bias_orpb, EPI_LN | EPI_BIAS | EPI_ORPB)

// one launch of a tile kernel over its persistent grid
template <int BN, bool CTA2, typename Kern>
int launch_gemm_grid(Kern kern, const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, size_t smem, cudaStream_t st) {
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
  cudaError_t e = launch_k(kern, dim3(grid), dim3(GemmCfg<BN, CTA2>::THREADS), smem, st, CTA2 ? 2 : 1, ta, tb, p);
  count_launch();
  if (e != cudaSuccess) return set_error(std::string("gemm launch: ") + cudaGetErrorString(e));
  return check_launch("gemm launch");
}

using GemmLaunchFn = int (*)(const CUtensorMap&, const CUtensorMap&, const GemmKParams&, size_t, cudaStream_t);

#define GLG_GEMM_DECLARE_KIND(NS, EPI_BITS)                                                                              \
  namespace NS {                                                                                                         \
  constexpr int kEpi = EPI_BITS;                                                                                         \
  template <int BN, bool GEGLU, bool CTA2, bool PP>                                                                      \
  int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, size_t smem, cudaStream_t st);          \
  }
GLG_GEMM_EPI_KINDS(GLG_GEMM_DECLARE_KIND)

// The tile kernel of one kind, launched once (no split-K reduce: glg_gemm launches that).  Defined only in the units that
// instantiate kernels (GLG_GEMM_KERNEL_UNIT), so gemm_tc.cu compiles none.
#ifdef GLG_GEMM_KERNEL_UNIT
#define GLG_GEMM_DEFINE_KIND(NS, EPI_BITS)                                                                               \
  namespace NS {                                                                                                         \
  template <int BN, bool GEGLU, bool CTA2, bool PP>                                                                      \
  __global__ void __launch_bounds__(384, 1)                                                                              \
  gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) { \
    gemm_tc_body<BN, GEGLU, CTA2, PP, kEpi>(tmA, tmB, p);                                                                \
  }                                                                                                                      \
  template <int BN, bool GEGLU, bool CTA2, bool PP>                                                                      \
  int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& p, size_t smem, cudaStream_t st) {         \
    static bool attr_set = false;                                                                                        \
    auto kern = gemm_tc_kernel<BN, GEGLU, CTA2, PP>;                                                                     \
    if (!attr_set) {                                                                                                     \
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN, CTA2>::SMEM_MAX); \
      if (e != cudaSuccess) return set_error(std::string("cudaFuncSetAttribute(gemm): ") + cudaGetErrorString(e));       \
      attr_set = true;                                                                                                   \
    }                                                                                                                    \
    return launch_gemm_grid<BN, CTA2>(kern, ta, tb, p, smem, st);                                                        \
  }                                                                                                                      \
  }
GLG_GEMM_EPI_KINDS(GLG_GEMM_DEFINE_KIND)
#endif

// Every instantiation: X(BN, GEGLU, CTA2, PP, kind).  A kind is instantiated for the tiles the tile picker gives its calls
// in the production plans (tests/schedule_census.py enumerates them); epi_generic for every tile glg_gemm can launch.
// Ping-pong GEGLU runs 128-wide items of the packed 256-row tile.  At BN = 256 the residual kinds and the paired row-bias
// kind are left out: with their flags fixed, ptxas spills 8-56 bytes in them (the generic kernels do not spill).
#define GLG_GEMM_GENERIC(X, BN, GEGLU, CTA2, PP) X(BN, GEGLU, CTA2, PP, epi_generic)
#define GLG_GEMM_UNET_COOP(X, BN)                                                                                          \
  X(BN, false, false, false, epi_none) X(BN, false, false, false, epi_bias) X(BN, false, false, false, epi_bias_f32)      \
  X(BN, false, false, false, epi_bias_res) X(BN, false, false, false, epi_bias_stats)                                     \
  X(BN, false, false, false, epi_bias_res_stats) X(BN, false, false, false, epi_bias_gate_res_stats)                      \
  X(BN, false, false, false, epi_ln_bias) X(BN, false, false, false, epi_ln_bias_orpb)
#define GLG_GEMM_CONV(X, BN, CTA2, PP)                                                                                     \
  X(BN, false, CTA2, PP, epi_bias) X(BN, false, CTA2, PP, epi_bias_rowbias) X(BN, false, CTA2, PP, epi_bias_res)

#define GLG_GEMM_INSTANCES_BN64(X)                                                                                         \
  GLG_GEMM_GENERIC(X, 64, false, false, false) GLG_GEMM_GENERIC(X, 64, false, false, true)                                \
  GLG_GEMM_UNET_COOP(X, 64) X(64, false, false, false, epi_bias_act) X(64, false, false, false, epi_bias_rowbias)         \
  GLG_GEMM_CONV(X, 64, false, true)
#define GLG_GEMM_INSTANCES_BN128(X)                                                                                        \
  GLG_GEMM_GENERIC(X, 128, false, false, false) GLG_GEMM_GENERIC(X, 128, false, true, false)                              \
  GLG_GEMM_GENERIC(X, 128, false, false, true) GLG_GEMM_GENERIC(X, 128, false, true, true)                                \
  GLG_GEMM_GENERIC(X, 128, true, false, true) GLG_GEMM_GENERIC(X, 128, true, true, true)                                  \
  GLG_GEMM_UNET_COOP(X, 128) GLG_GEMM_CONV(X, 128, true, false) X(128, true, false, true, epi_ln_bias)
#define GLG_GEMM_INSTANCES_BN160(X)                                                                                        \
  GLG_GEMM_GENERIC(X, 160, false, false, false) GLG_GEMM_GENERIC(X, 160, false, true, false)                              \
  GLG_GEMM_UNET_COOP(X, 160) GLG_GEMM_CONV(X, 160, true, false)
#define GLG_GEMM_INSTANCES_BN256(X)                                                                                        \
  GLG_GEMM_GENERIC(X, 256, false, false, false) GLG_GEMM_GENERIC(X, 256, false, true, false)                              \
  GLG_GEMM_GENERIC(X, 256, true, false, false) GLG_GEMM_GENERIC(X, 256, true, true, false)                                \
  X(256, false, false, false, epi_none) X(256, false, false, false, epi_bias) X(256, false, false, false, epi_bias_act)    \
  X(256, false, false, false, epi_bias_stats) X(256, false, false, false, epi_ln_bias)                                    \
  X(256, false, false, false, epi_ln_bias_orpb)                                                                           \
  X(256, false, true, false, epi_bias) X(256, false, true, false, epi_bias_f32) X(256, false, true, false, epi_bias_stats) \
  X(256, false, true, false, epi_ln_bias) X(256, false, true, false, epi_ln_bias_orpb)                                    \
  X(256, true, false, false, epi_ln_bias) X(256, true, true, false, epi_ln_bias)
#define GLG_GEMM_INSTANCES(X)                                                                                              \
  GLG_GEMM_INSTANCES_BN64(X) GLG_GEMM_INSTANCES_BN128(X) GLG_GEMM_INSTANCES_BN160(X) GLG_GEMM_INSTANCES_BN256(X)

#define GLG_GEMM_INSTANTIATE(BN, GEGLU, CTA2, PP, NS)                                                                    \
  template int NS::launch<BN, GEGLU, CTA2, PP>(const CUtensorMap&, const CUtensorMap&, const GemmKParams&, size_t, cudaStream_t);

}  // namespace glg
