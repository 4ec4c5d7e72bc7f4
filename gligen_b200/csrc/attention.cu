// Fused (flash-style) multi-head attention for the GLIGEN transformer blocks.
//
//   O = softmax(Q K^T * scale) V      per (batch, head); online softmax in fp32; scores stay on chip.
//
// Data path: 64-query x 64-key tiles, 4 warps (16 query rows each), bf16 mma.sync m16n8k16 with
// ldmatrix-fed operands, K/V tiles double-buffered with cp.async.  Head dims 8..160 (multiple of 8)
// are zero-padded to a multiple of 16 in shared memory only.  Ragged key lengths (T+G grounding
// tokens, 77 text tokens) are masked to -inf in the last tile.
//
// Two instantiations: the short-key kernel (Lk <= 128: K and V loaded once, four query tiles per CTA), which also
// implements the causal mask of the 77-token CLIP text encoder, and the streamed kernel (one CTA per 64 query rows, key
// tiles double-buffered), kept as a test reference.  Long key sets run on attn_wgmma_kernel below.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <string>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"
#include "../../include/gligen_b200.h"

namespace glg {

struct AttnKParams {
  const bf16* q; const bf16* k; const bf16* v; bf16* o;
  long long q_row, k_row, v_row, o_row, q_batch, k_batch, v_batch, o_batch;
  int heads, d, Lq, Lk;
  float scale_log2;
  int causal;                     // key j is masked for query i when j > i (short-key kernel only)
  int poly;                       // of every 8 score pairs of a row, the last `poly` take exp2 from ex2_poly3 (FMA pipe)
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exp2 of score pair j (0..7) of a 64-key tile: the last `poly` pairs of every 8 on the FMA pipe, the rest on the MUFU
__device__ __forceinline__ float exp2_share(float x, int j, int poly) { return j >= 8 - poly ? ex2_poly3(x) : fast_exp2(x); }

template <int DPAD>
struct AttnCfg {
  static constexpr int BM = 64, BN = 64;
  static constexpr int LDS = DPAD + 8;                 // padded row (elements): (DPAD+8)*2 B == 16*odd (mod 128) -> conflict-free ldmatrix
  static constexpr int TILE_ELEMS = 64 * LDS;
  static constexpr int SMEM_BYTES = 5 * TILE_ELEMS * 2;  // Q + 2xK + 2xV
};

// Copy a 64-row tile of one head into shared memory: rows [row0, row0+64) of a [L, *] matrix with row
// stride `ld`, first d columns (d/8 16-byte chunks per row).  Rows >= L are zero-filled.
template <int DPAD>
__device__ __forceinline__ void load_tile(uint32_t smem_tile, const bf16* g, long long ld, int row0, int L, int d) {
  constexpr int LDS = AttnCfg<DPAD>::LDS;
  const int chunks = d >> 3;
  const int total = 64 * chunks;
  for (int i = threadIdx.x; i < total; i += 128) {
    const int r = i / chunks, c = i - r * chunks;
    const int gr = row0 + r;
    const bool ok = gr < L;
    const bf16* src = g + (ok ? (long long)gr * ld + c * 8 : 0);
    cp_async16(smem_tile + (uint32_t)(r * LDS + c * 8) * 2u, src, ok ? 16 : 0);
  }
}

template <int DPAD, bool SHORT>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnKParams p) {
  // SHORT (Lk <= 128, the 77-token text context of cross attention): K and V (<= 2 tiles) are loaded ONCE and the
  // CTA walks QT = 4 consecutive 64-row query tiles with a double-buffered Q, instead of one CTA (and one K/V
  // fetch, one launch-latency chain) per 64 query rows.
  pdl_trigger();
  pdl_wait();
  using Cfg = AttnCfg<DPAD>;
  constexpr int LDS = Cfg::LDS;
  constexpr int KSTEPS = DPAD / 16;       // k-steps of QK^T
  constexpr int DT = DPAD / 8;            // n-tiles of the output
  constexpr int NQ = SHORT ? 2 : 1;       // Q buffers
  constexpr int QT = SHORT ? 4 : 1;       // query tiles per CTA
  extern __shared__ __align__(16) uint8_t attn_smem[];
  const uint32_t sQ0 = smem_u32(attn_smem);
  const uint32_t sK = sQ0 + NQ * Cfg::TILE_ELEMS * 2;
  const uint32_t sV = sK + 2 * Cfg::TILE_ELEMS * 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int d = p.d;
  const bf16* gq = p.q + (long long)b * p.q_batch + (long long)h * d;
  const bf16* gk = p.k + (long long)b * p.k_batch + (long long)h * d;
  const bf16* gv = p.v + (long long)b * p.v_batch + (long long)h * d;

  // zero the padded columns [d, DPAD) of every tile once (cp.async never writes them)
  if (d < DPAD) {
    const int padc = DPAD - d;                   // multiple of 8
    for (int i = threadIdx.x; i < (4 + NQ) * 64 * (padc / 8); i += 128) {
      const int row = i / (padc / 8), c = i - row * (padc / 8);
      *reinterpret_cast<uint4*>(attn_smem + ((size_t)row * LDS + d + c * 8) * 2) = make_uint4(0, 0, 0, 0);
    }
  }
  const int nkt = (p.Lk + 63) / 64;
  const int qbase = blockIdx.x * 64 * QT;
  load_tile<DPAD>(sQ0, gq, p.q_row, qbase, p.Lq, d);
  load_tile<DPAD>(sK, gk, p.k_row, 0, p.Lk, d);
  load_tile<DPAD>(sV, gv, p.v_row, 0, p.Lk, d);
  if (SHORT && nkt > 1) {
    load_tile<DPAD>(sK + Cfg::TILE_ELEMS * 2, gk, p.k_row, 64, p.Lk, d);
    load_tile<DPAD>(sV + Cfg::TILE_ELEMS * 2, gv, p.v_row, 64, p.Lk, d);
  }
  cp_async_commit();

  float o_acc[DT][4];
  float m_run[2], l_run[2];
  auto reset_state = [&]() {
#pragma unroll
    for (int j = 0; j < DT; ++j) { o_acc[j][0] = o_acc[j][1] = o_acc[j][2] = o_acc[j][3] = 0.f; }
    m_run[0] = m_run[1] = -INFINITY;
    l_run[0] = l_run[1] = 0.f;
  };
  reset_state();

  const uint32_t q_lane_off = (uint32_t)((warp * 16 + (lane & 15)) * LDS + (lane >> 4) * 8) * 2u;
  // K (non-transposed) ldmatrix lane offsets: matrix m = lane/8 -> key += (m/2)*8, col += (m%2)*8
  const uint32_t k_lane_off = (uint32_t)((((lane >> 4) * 8) + (lane & 7)) * LDS + ((lane >> 3) & 1) * 8) * 2u;
  // V (transposed) ldmatrix lane offsets: matrix m = lane/8 -> key += (m%2)*8, dcol += (m/2)*8
  const uint32_t v_lane_off = (uint32_t)(((((lane >> 3) & 1) * 8) + (lane & 7)) * LDS + (lane >> 4) * 8) * 2u;

  // one 64-key tile: S = Q K^T, mask, online softmax, O += P V
  auto compute_tile = [&](uint32_t sQ, uint32_t sKb, uint32_t sVb, int kt, int q0) {
    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {
      uint32_t a0, a1, a2, a3;
      ldsm_x4(sQ + q_lane_off + kk * 32, a0, a1, a2, a3);
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(sKb + k_lane_off + (uint32_t)(jp * 16 * LDS) * 2u + kk * 32, b0, b1, b2, b3);
        mma_bf16_16816(s[2 * jp], a0, a1, a2, a3, b0, b1);
        mma_bf16_16816(s[2 * jp + 1], a0, a1, a2, a3, b2, b3);
      }
    }
    // ---- mask ragged tail
    if (kt == nkt - 1 && (p.Lk & 63)) {
      const int kbase = kt * 64 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kbase + j * 8;
        if (key >= p.Lk) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
        if (key + 1 >= p.Lk) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
      }
    }
    if (SHORT && p.causal) {
      const int r0 = q0 + warp * 16 + (lane >> 2);
      const int kbase = kt * 64 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kbase + j * 8;
        if (key > r0) s[j][0] = -INFINITY;
        if (key + 1 > r0) s[j][1] = -INFINITY;
        if (key > r0 + 8) s[j][2] = -INFINITY;
        if (key + 1 > r0 + 8) s[j][3] = -INFINITY;
      }
    }
    // ---- online softmax (rows g = lane/4 and g+8)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m_run[0], mx0), mn1 = fmaxf(m_run[1], mx1);
    const float corr0 = fast_exp2((m_run[0] - mn0) * p.scale_log2);
    const float corr1 = fast_exp2((m_run[1] - mn1) * p.scale_log2);
    m_run[0] = mn0; m_run[1] = mn1;
    const float ms0 = mn0 * p.scale_log2, ms1 = mn1 * p.scale_log2;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t pa[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2_share(fmaf(s[j][0], p.scale_log2, -ms0), j, p.poly);
      const float p1 = exp2_share(fmaf(s[j][1], p.scale_log2, -ms0), j, p.poly);
      const float p2 = exp2_share(fmaf(s[j][2], p.scale_log2, -ms1), j, p.poly);
      const float p3 = exp2_share(fmaf(s[j][3], p.scale_log2, -ms1), j, p.poly);
      // the row sum uses the bf16-rounded probabilities that actually enter the PV product
      const uint32_t u01 = pack_bf16x2(p0, p1), u23 = pack_bf16x2(p2, p3);
      const float2 f01 = unpack_bf16x2(u01), f23 = unpack_bf16x2(u23);
      rs0 += f01.x + f01.y;
      rs1 += f23.x + f23.y;
      pa[j][0] = u01; pa[j][1] = u23;
    }
    l_run[0] = l_run[0] * corr0 + rs0;
    l_run[1] = l_run[1] * corr1 + rs1;
#pragma unroll
    for (int j = 0; j < DT; ++j) {
      o_acc[j][0] *= corr0; o_acc[j][1] *= corr0;
      o_acc[j][2] *= corr1; o_acc[j][3] *= corr1;
    }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t a0 = pa[2 * kk][0], a1 = pa[2 * kk][1], a2 = pa[2 * kk + 1][0], a3 = pa[2 * kk + 1][1];
#pragma unroll
      for (int jp = 0; jp < DT / 2; ++jp) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(sVb + v_lane_off + (uint32_t)(kk * 16 * LDS + jp * 16) * 2u, b0, b1, b2, b3);
        mma_bf16_16816(o_acc[2 * jp], a0, a1, a2, a3, b0, b1);
        mma_bf16_16816(o_acc[2 * jp + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  };
  // O /= l, write bf16 rows [q0, q0 + 64)
  auto finalize = [&](int q0) {
  float l0 = l_run[0], l1 = l_run[1];
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
  bf16* go = p.o + (long long)b * p.o_batch + (long long)h * d;
#pragma unroll
  for (int j = 0; j < DT; ++j) {
    const int col = j * 8 + 2 * (lane & 3);
    if (col < d) {
      if (r0 < p.Lq) *reinterpret_cast<uint32_t*>(go + (long long)r0 * p.o_row + col) = pack_bf16x2(o_acc[j][0] * inv0, o_acc[j][1] * inv0);
      if (r1 < p.Lq) *reinterpret_cast<uint32_t*>(go + (long long)r1 * p.o_row + col) = pack_bf16x2(o_acc[j][2] * inv1, o_acc[j][3] * inv1);
    }
  }
  };

  if constexpr (!SHORT) {
    for (int kt = 0; kt < nkt; ++kt) {
      const int buf = kt & 1;
      if (kt + 1 < nkt) {
        load_tile<DPAD>(sK + (buf ^ 1) * Cfg::TILE_ELEMS * 2, gk, p.k_row, (kt + 1) * 64, p.Lk, d);
        load_tile<DPAD>(sV + (buf ^ 1) * Cfg::TILE_ELEMS * 2, gv, p.v_row, (kt + 1) * 64, p.Lk, d);
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      compute_tile(sQ0, sK + buf * Cfg::TILE_ELEMS * 2, sV + buf * Cfg::TILE_ELEMS * 2, kt, qbase);
      __syncthreads();
    }
    finalize(qbase);
  } else {
    for (int s = 0; s < QT; ++s) {
      const int q0 = qbase + s * 64;
      if (q0 >= p.Lq) break;
      const bool more = (s + 1 < QT) && (q0 + 64 < p.Lq);
      if (more) {
        load_tile<DPAD>(sQ0 + ((s + 1) & 1) * Cfg::TILE_ELEMS * 2, gq, p.q_row, q0 + 64, p.Lq, d);
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      reset_state();
      for (int kt = 0; kt < nkt; ++kt)
        compute_tile(sQ0 + (s & 1) * Cfg::TILE_ELEMS * 2, sK + kt * Cfg::TILE_ELEMS * 2, sV + kt * Cfg::TILE_ELEMS * 2, kt, q0);
      finalize(q0);
      __syncthreads();            // this Q buffer is refilled two iterations later
    }
  }
}

template <int DPAD, bool SHORT>
static int launch_attn2(const AttnKParams& p, int B, cudaStream_t st) {
  using Cfg = AttnCfg<DPAD>;
  static bool attr_set = false;
  auto kern = attn_fwd_kernel<DPAD, SHORT>;
  constexpr int smem = (SHORT ? 6 : 5) * Cfg::TILE_ELEMS * 2;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return set_error(std::string("cudaFuncSetAttribute(attn): ") + cudaGetErrorString(e));
    attr_set = true;
  }
  const int rows_per_cta = SHORT ? 256 : 64;
  dim3 grid((p.Lq + rows_per_cta - 1) / rows_per_cta, p.heads, B);
  launch_k(kern, dim3(grid), dim3(128), smem, st, 1, p);
  count_launch();
  return check_launch("attention launch");
}
// ------------------------------------------------------------------------------------------------------------------
// Hopper flash attention for long key sets (Lk > 128: self attention and the fuser's attention over [visual ; grounding]).
// 288 threads: warp 8 loads Q once and streams K/V tiles of 64 keys through a TMA + mbarrier ring; warpgroups 0 / 1 each
// own 64 of the CTA's 128 query rows.  Per key tile: S = Q K^T with wgmma (both operands in shared memory), online softmax
// in registers, O += P V with wgmma taking P straight from registers and V as a transposed (MN-major) operand.
// Every tile is one 5-D TMA box {8 elements, rows, d/8 chunks, head, batch} that lands as [chunk][row][8 elements]: the
// non-swizzled core-matrix layout wgmma reads, with the zero padding of d up to DPAD and of ragged rows done by the TMA.
int g_attn_poly = 0;          // test hook (glg_debug_attn_poly_share): FMA-pipe share of the long-key kernels' exponentials

template <int DPAD>
struct HAttnCfg {
  static constexpr int BM = 128, BN = 64;
  static constexpr int Q_BYTES = BM * DPAD * 2;
  static constexpr int KV_BYTES = BN * DPAD * 2;
  static constexpr int STAGES = (Q_BYTES + 6 * KV_BYTES <= 200 * 1024) ? 3 : 2;
  static constexpr int SMEM = 1024 /*barriers*/ + 1024 /*align*/ + Q_BYTES + STAGES * 2 * KV_BYTES;
};

struct HAttnParams {
  bf16* o; long long o_row, o_batch;
  int d, Lq, Lk;
  float scale_log2;
  int poly;                       // FMA-pipe share of the exponentials, as AttnKParams::poly
};

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// non-swizzled wgmma descriptor: lbo / sbo = byte strides between core matrices (8 rows x 16 B) along the leading
// (K for K-major, K too for MN-major in the "interleave" layout) and the strided dimension
__device__ __forceinline__ uint64_t gmma_desc_interleave(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

template <int DPAD>
__global__ void __launch_bounds__(288, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, const HAttnParams p) {
  using Cfg = HAttnCfg<DPAD>;
  constexpr int ST = Cfg::STAGES;
  extern __shared__ uint8_t hattn_smem[];
  const uint32_t bar = (smem_u32(hattn_smem) + 1023u) & ~1023u;
  const uint32_t qbar = bar;
  auto full_bar = [&](int s) { return bar + 8u + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 8u + 8u * (ST + s); };
  const uint32_t sQ = bar + 1024u;
  auto sK = [&](int s) { return sQ + Cfg::Q_BYTES + (uint32_t)s * 2u * Cfg::KV_BYTES; };
  auto sV = [&](int s) { return sK(s) + Cfg::KV_BYTES; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * Cfg::BM;
  const int nkt = (p.Lk + 63) / 64;
  pdl_trigger();
  if (threadIdx.x == 0) {
    mbar_init(qbar, 1);
    for (int s = 0; s < ST; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }   // 8 consumer warps
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    // ===================== producer: Q once, then K/V tiles through the ring =====================
    if (lane == 0) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
      mbar_arrive_expect_tx(qbar, Cfg::Q_BYTES);
      tma_load_5d(sQ, &tmQ, qbar, 0, q0, 0, h, b);
      for (int kt = 0; kt < nkt; ++kt) {
        const int s = kt % ST;
        mbar_wait<false>(empty_bar(s), ((kt / ST) & 1) ^ 1u);
        mbar_arrive_expect_tx(full_bar(s), 2 * Cfg::KV_BYTES);
        tma_load_5d(sK(s), &tmK, full_bar(s), 0, kt * 64, 0, h, b);
        tma_load_5d(sV(s), &tmV, full_bar(s), 0, kt * 64, 0, h, b);
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile =====================
  const int wg = warp >> 2, wq = warp & 3;
  constexpr int DT = DPAD / 8;
  float o_acc[DPAD / 2];
#pragma unroll
  for (int i = 0; i < DPAD / 2; ++i) o_acc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  // Q: [chunk][128 rows][8]; this warpgroup's 64 rows start 64 * 16 B into every chunk
  const uint64_t dq = gmma_desc_interleave(sQ + (uint32_t)wg * 64u * 16u, 128u * 16u, 128u);
  mbar_wait<false>(qbar, 0);
  for (int kt = 0; kt < nkt; ++kt) {
    const int s = kt % ST;
    mbar_wait<false>(full_bar(s), (kt / ST) & 1);
    // ---- S = Q K^T: K [chunk][64 keys][8] is K-major (contraction over d)
    float sc[32];
    const uint64_t dk = gmma_desc_interleave(sK(s), 64u * 16u, 128u);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DPAD / 16; ++kk)            // 16 d-columns = two chunks per step
      Wgmma<64>::mma(sc, dq + (uint64_t)((kk * 2 * 128 * 16) >> 4), dk + (uint64_t)((kk * 2 * 64 * 16) >> 4), kk > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    // ---- mask the ragged last key tile (fragment: regs 4 j + {0,1} row r, 4 j + {2,3} row r + 8, cols 8 j + 2 (lane % 4))
    if (kt == nkt - 1 && (p.Lk & 63)) {
      const int kbase = kt * 64 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kbase + j * 8;
        if (key >= p.Lk) { sc[4 * j] = -INFINITY; sc[4 * j + 2] = -INFINITY; }
        if (key + 1 >= p.Lk) { sc[4 * j + 1] = -INFINITY; sc[4 * j + 3] = -INFINITY; }
      }
    }
    // ---- online softmax over the four lanes of a row
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx0 = fmaxf(mx0, fmaxf(sc[4 * j], sc[4 * j + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m_run[0], mx0), mn1 = fmaxf(m_run[1], mx1);
    const float corr0 = fast_exp2((m_run[0] - mn0) * p.scale_log2), corr1 = fast_exp2((m_run[1] - mn1) * p.scale_log2);
    m_run[0] = mn0; m_run[1] = mn1;
    const float ms0 = mn0 * p.scale_log2, ms1 = mn1 * p.scale_log2;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t pa[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t u01 = pack_bf16x2(exp2_share(fmaf(sc[4 * j], p.scale_log2, -ms0), j, p.poly),
                                       exp2_share(fmaf(sc[4 * j + 1], p.scale_log2, -ms0), j, p.poly));
      const uint32_t u23 = pack_bf16x2(exp2_share(fmaf(sc[4 * j + 2], p.scale_log2, -ms1), j, p.poly),
                                       exp2_share(fmaf(sc[4 * j + 3], p.scale_log2, -ms1), j, p.poly));
      const float2 f01 = unpack_bf16x2(u01), f23 = unpack_bf16x2(u23);     // row sums of what enters P.V
      rs0 += f01.x + f01.y; rs1 += f23.x + f23.y;
      pa[j][0] = u01; pa[j][1] = u23;
    }
    l_run[0] = l_run[0] * corr0 + rs0;
    l_run[1] = l_run[1] * corr1 + rs1;
#pragma unroll
    for (int j = 0; j < DT; ++j) {
      o_acc[4 * j] *= corr0; o_acc[4 * j + 1] *= corr0;
      o_acc[4 * j + 2] *= corr1; o_acc[4 * j + 3] *= corr1;
    }
    // ---- O += P V: V [chunk][64 keys][8] is the MN-major B operand (8-key groups 128 B apart, d chunks 1024 B apart)
    const uint64_t dv = gmma_desc_interleave(sV(s), 128u, 64u * 16u);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t a[4] = {pa[2 * kk][0], pa[2 * kk][1], pa[2 * kk + 1][0], pa[2 * kk + 1][1]};
      WgmmaRS<DPAD>::mma(o_acc, a, dv + (uint64_t)((kk * 2 * 128) >> 4));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o_acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(s));         // K and V of this stage are consumed
  }
  // ---- O /= l, bf16 rows
  float l0 = l_run[0], l1 = l_run[1];
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = q0 + wg * 64 + wq * 16 + (lane >> 2), r1 = r0 + 8;
  bf16* go = p.o + (long long)b * p.o_batch + (long long)h * p.d;
#pragma unroll
  for (int j = 0; j < DT; ++j) {
    const int col = j * 8 + 2 * (lane & 3);
    if (col < p.d) {
      if (r0 < p.Lq) *reinterpret_cast<uint32_t*>(go + (long long)r0 * p.o_row + col) = pack_bf16x2(o_acc[4 * j] * inv0, o_acc[4 * j + 1] * inv0);
      if (r1 < p.Lq) *reinterpret_cast<uint32_t*>(go + (long long)r1 * p.o_row + col) = pack_bf16x2(o_acc[4 * j + 2] * inv1, o_acc[4 * j + 3] * inv1);
    }
  }
}

// tensor map of one operand: {8 elements, rows, d/8 chunks, head, batch} -> smem [chunk][rows][8]
static int attn_tmap(CUtensorMap* m, const void* ptr, long long row, long long batch, int L, int d, int heads, int B, int box_rows, int dpad) {
  const uint64_t dims[5] = {8, (uint64_t)L, (uint64_t)(d / 8), (uint64_t)heads, (uint64_t)B};
  const uint64_t str[4] = {(uint64_t)row * 2, 16, (uint64_t)d * 2, (uint64_t)(B > 1 ? batch : row) * 2};
  const uint32_t box[5] = {8, (uint32_t)box_rows, (uint32_t)(dpad / 8), 1, 1};
  return get_tmap_bf16_sw(m, ptr, 5, dims, str, box, 0);
}

template <int DPAD>
static int launch_attn_wgmma(const GlgAttnArgs* a, cudaStream_t st) {
  using Cfg = HAttnCfg<DPAD>;
  static bool attr_set = false;
  auto kern = attn_wgmma_kernel<DPAD>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(std::string("cudaFuncSetAttribute(attn wgmma): ") + cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tq, tk, tv;
  if (attn_tmap(&tq, a->q, a->q_row, a->q_batch, a->Lq, a->d_head, a->heads, a->B, Cfg::BM, DPAD) ||
      attn_tmap(&tk, a->k, a->k_row, a->k_batch, a->Lk, a->d_head, a->heads, a->B, Cfg::BN, DPAD) ||
      attn_tmap(&tv, a->v, a->v_row, a->v_batch, a->Lk, a->d_head, a->heads, a->B, Cfg::BN, DPAD)) return -1;
  HAttnParams p;
  p.o = (bf16*)a->out; p.o_row = a->o_row; p.o_batch = a->o_batch;
  p.d = a->d_head; p.Lq = a->Lq; p.Lk = a->Lk;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.poly = g_attn_poly;
  dim3 grid((a->Lq + Cfg::BM - 1) / Cfg::BM, a->heads, a->B);
  cudaError_t e = launch_k(kern, grid, dim3(288), Cfg::SMEM, st, 1, tq, tk, tv, p);
  count_launch();
  if (e != cudaSuccess) return set_error(std::string("attention (wgmma) launch: ") + cudaGetErrorString(e));
  return check_launch("attention (wgmma) launch");
}

static int attention_wgmma(const GlgAttnArgs* a, cudaStream_t st) {
  switch ((a->d_head + 15) / 16 * 16) {
    case 16: return launch_attn_wgmma<16>(a, st);
    case 32: return launch_attn_wgmma<32>(a, st);
    case 48: return launch_attn_wgmma<48>(a, st);
    case 64: return launch_attn_wgmma<64>(a, st);
    case 80: return launch_attn_wgmma<80>(a, st);
    case 96: return launch_attn_wgmma<96>(a, st);
    case 112: return launch_attn_wgmma<112>(a, st);
    case 128: return launch_attn_wgmma<128>(a, st);
    case 144: return launch_attn_wgmma<144>(a, st);
    case 160: return launch_attn_wgmma<160>(a, st);
  }
  return set_error("glg_attention: unsupported head dim");
}

template <int DPAD>
static int launch_attn(const AttnKParams& p, int B, bool short_keys, cudaStream_t st) {
  return short_keys ? launch_attn2<DPAD, true>(p, B, st) : launch_attn2<DPAD, false>(p, B, st);
}

int g_attn_mode = 0;          // test hook (glg_debug_attn_mode): 0 = auto (short-key mma.sync kernel for Lk <= 128, wgmma kernel above), 1 = the
                              // streamed mma.sync kernel for every key length, 2 = the wgmma kernel for every key length,
                              // 3 = the short-key kernel wherever Lk <= 128 (causal attention always takes the short-key kernel)

}  // namespace glg

using namespace glg;

extern "C" void glg_debug_attn_mode(int mode) { glg::g_attn_mode = mode; }
extern "C" void glg_debug_attn_poly_share(int poly) { glg::g_attn_poly = poly < 0 ? 0 : poly > 8 ? 8 : poly; }

extern "C" int glg_attention(const GlgAttnArgs* a, void* stream) {
  if (!a) return set_error("glg_attention: null args");
  if (a->d_head <= 0 || a->d_head % 8 || a->d_head > 160) return set_error("glg_attention: d_head must be a multiple of 8 in [8,160]");
  if (a->Lq <= 0 || a->Lk <= 0 || a->B <= 0 || a->heads <= 0) return set_error("glg_attention: bad sizes");
  if ((a->q_row | a->k_row | a->v_row | a->q_batch | a->k_batch | a->v_batch) % 8) return set_error("glg_attention: q/k/v strides must be multiples of 8 elements");
  if ((a->o_row | a->o_batch) % 2) return set_error("glg_attention: output strides must be even");
  if (((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) & 15) return set_error("glg_attention: q/k/v must be 16-byte aligned");
  if (a->causal && a->Lk > 128) return set_error("glg_attention: causal attention needs Lk <= 128");
  AttnKParams p;
  p.q = (const bf16*)a->q; p.k = (const bf16*)a->k; p.v = (const bf16*)a->v; p.o = (bf16*)a->out;
  p.q_row = a->q_row; p.k_row = a->k_row; p.v_row = a->v_row; p.o_row = a->o_row;
  p.q_batch = a->q_batch; p.k_batch = a->k_batch; p.v_batch = a->v_batch; p.o_batch = a->o_batch;
  p.heads = a->heads; p.d = a->d_head; p.Lq = a->Lq; p.Lk = a->Lk;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.causal = a->causal;
  const bool short_keys = a->Lk <= 128 && (a->causal || g_attn_mode == 0 || g_attn_mode == 3);
  p.poly = short_keys ? 0 : g_attn_poly;           // the short-key kernel keeps every exponential on the MUFU
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!a->causal && ((g_attn_mode == 0 && !short_keys) || g_attn_mode == 2)) return attention_wgmma(a, st);
  const int dpad = (a->d_head + 15) / 16 * 16;
  switch (dpad) {
    case 16: return launch_attn<16>(p, a->B, short_keys, st);
    case 32: return launch_attn<32>(p, a->B, short_keys, st);
    case 48: return launch_attn<48>(p, a->B, short_keys, st);
    case 64: return launch_attn<64>(p, a->B, short_keys, st);
    case 80: return launch_attn<80>(p, a->B, short_keys, st);
    case 96: return launch_attn<96>(p, a->B, short_keys, st);
    case 112: return launch_attn<112>(p, a->B, short_keys, st);
    case 128: return launch_attn<128>(p, a->B, short_keys, st);
    case 144: return launch_attn<144>(p, a->B, short_keys, st);
    case 160: return launch_attn<160>(p, a->B, short_keys, st);
  }
  return set_error("glg_attention: unsupported head dim");
}
