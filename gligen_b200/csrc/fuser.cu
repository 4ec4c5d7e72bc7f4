// The gatedSA2 fuser's residual (reference ldm/modules/attention.py:251-297, GatedSelfAttentionDense2.forward):
//
//     x[b, y*n + x', c] = bf16( x[b, y*n + x', c] + gate * bicubic_{g->n}(grid[b])[y, x', c] )
//
// grid holds the to_out projections of the G = g*g grounding rows (fp32, row-major tokens), which the reference reshapes to a
// g x g image and resamples with F.interpolate(mode='bicubic') onto the n x n visual grid before the gated add.  One pass over x:
// the grid of one image and one 32-channel slot sits in shared memory, every thread owns 8 channels of one pixel (16-byte loads
// and stores of x), and the four threads of a pixel's slot reduce the LayerNorm partials (sum, sum of squares) of the values
// they stored - the stats_out contract of glg_gemm, so fuser.ff.1 folds norm2 on them unchanged.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include "common.cuh"
#include "internal.h"
#include "../../include/gligen_b200.h"

namespace glg {

constexpr int GR_THREADS = 256;                 // 64 pixels x 4 threads (8 channels each = one 32-channel slot)
constexpr int GR_PIX = GR_THREADS / 4;
constexpr int GR_BAND = 512;                    // output pixels per CTA: the grid tile is loaded once per 512 pixels
constexpr int GR_MAX_G = 19;                    // g * g * 32 fp32 of shared memory <= 48 KiB

__global__ void __launch_bounds__(GR_THREADS) grid_resample_gate_kernel(const float* __restrict__ grid, long long grid_batch, bf16* x,
                                                                        long long ldx, const float* __restrict__ gate, float* __restrict__ stats,
                                                                        long long slot_stride, int g, int n, int C) {
  extern __shared__ float4 sgrid4[];           // [g * g tokens][32 channels of this slot]
  const int slots = C >> 5;
  const int b = blockIdx.y / slots, slot = blockIdx.y % slots;
  pdl_trigger();
  pdl_wait();
  const float* src = grid + (long long)b * grid_batch + slot * 32;
  const int gg = g * g;
  for (int i = threadIdx.x; i < gg * 8; i += GR_THREADS)
    sgrid4[i] = __ldg(reinterpret_cast<const float4*>(src + (long long)(i >> 3) * C) + (i & 7));
  __syncthreads();

  const float gv = __ldg(gate);
  const float sc = (float)g / (float)n;         // area_pixel_compute_scale (align_corners = False), as resize_plane
  const int q = threadIdx.x & 3;                // channels slot*32 + 8q .. +7
  const long long T = (long long)n * n;
  const int p_lo = blockIdx.x * GR_BAND;
  const int p_hi = (int)min((long long)p_lo + GR_BAND, T);
  const float* sg = reinterpret_cast<const float*>(sgrid4) + q * 8;
#pragma unroll 2
  for (int it = 0; it < GR_BAND / GR_PIX; ++it) {
    const int p = p_lo + it * GR_PIX + (threadIdx.x >> 2);
    const bool active = p < p_hi;               // the warp stays converged for the shuffles below
    float s = 0.f, sq = 0.f;
    const long long row = (long long)b * T + p;
    if (active) {
      const int oy = p / n, ox = p - oy * n;
      const float ry = sc * ((float)oy + 0.5f) - 0.5f, rx = sc * ((float)ox + 0.5f) - 0.5f;
      const float fy = floorf(ry), fx = floorf(rx);
      const int iy = (int)fy, ix = (int)fx;
      float cy[4], cx[4];
      cubic_coeffs(ry - fy, cy);
      cubic_coeffs(rx - fx, cx);
      float acc[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[c] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int yy = min(max(iy - 1 + j, 0), g - 1);
        float r[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) r[c] = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int xx = min(max(ix - 1 + k, 0), g - 1);
          const float4* t = reinterpret_cast<const float4*>(sg + (yy * g + xx) * 32);
          const float4 a = t[0], bb = t[1];
          r[0] = fmaf(cx[k], a.x, r[0]); r[1] = fmaf(cx[k], a.y, r[1]); r[2] = fmaf(cx[k], a.z, r[2]); r[3] = fmaf(cx[k], a.w, r[3]);
          r[4] = fmaf(cx[k], bb.x, r[4]); r[5] = fmaf(cx[k], bb.y, r[5]); r[6] = fmaf(cx[k], bb.z, r[6]); r[7] = fmaf(cx[k], bb.w, r[7]);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = fmaf(cy[j], r[c], acc[c]);
      }
      bf16* xp = x + row * ldx + slot * 32 + q * 8;
      const uint4 u = *reinterpret_cast<const uint4*>(xp);
      const uint32_t in[4] = {u.x, u.y, u.z, u.w};
      uint32_t out[4];
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const float2 xv = unpack_bf16x2(in[h]);
        out[h] = pack_bf16x2(fmaf(gv, acc[2 * h], xv.x), fmaf(gv, acc[2 * h + 1], xv.y));
        const float2 st = unpack_bf16x2(out[h]);           // statistics of the stored (rounded) values
        s += st.x + st.y;
        sq = fmaf(st.x, st.x, fmaf(st.y, st.y, sq));
      }
      *reinterpret_cast<uint4*>(xp) = make_uint4(out[0], out[1], out[2], out[3]);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    sq += __shfl_xor_sync(0xffffffffu, sq, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    sq += __shfl_xor_sync(0xffffffffu, sq, 2);
    if (active && q == 0) *reinterpret_cast<float2*>(stats + ((long long)slot * slot_stride + row) * 2) = make_float2(s, sq);
  }
}

}  // namespace glg

using namespace glg;

extern "C" int glg_grid_resample_gate(const float* grid, int64_t grid_batch_stride, void* x, int64_t ldx, const float* gate, float* stats_out,
                                      int64_t stats_slot_stride, int32_t B, int32_t g, int32_t n, int32_t C, void* stream) {
  if (!grid || !x || !gate || !stats_out) return set_error("glg_grid_resample_gate: null pointer");
  if (B < 1 || g < 1 || n < 1) return set_error("glg_grid_resample_gate: B, g and n must be >= 1");
  if (g > GR_MAX_G) return set_error("glg_grid_resample_gate: g must be <= 19 (the grid tile of one 32-channel slot lives in 48 KiB of shared memory)");
  if (C < 32 || C % 32) return set_error("glg_grid_resample_gate: C must be a positive multiple of 32");
  if (B > 1 && grid_batch_stride < (int64_t)g * g * C) return set_error("glg_grid_resample_gate: grid_batch_stride < g*g*C");
  if (grid_batch_stride % 4 || ((uintptr_t)grid & 15)) return set_error("glg_grid_resample_gate: grid must be 16-byte aligned, its batch stride a multiple of 4");
  if (ldx < C || ldx % 8 || ((uintptr_t)x & 15)) return set_error("glg_grid_resample_gate: x must be 16-byte aligned with ldx >= C, a multiple of 8");
  const long long T = (long long)n * n;
  if ((long long)B * T > 0x7fffffffLL) return set_error("glg_grid_resample_gate: B*n*n exceeds 2^31 rows");
  if (stats_slot_stride < (int64_t)B * T || ((uintptr_t)stats_out & 7)) return set_error("glg_grid_resample_gate: stats_slot_stride < B*n*n or stats_out not 8-byte aligned");
  const dim3 blocks((unsigned)((T + GR_BAND - 1) / GR_BAND), (unsigned)(B * (C / 32)));
  if (blocks.y > 65535u) return set_error("glg_grid_resample_gate: B*C/32 exceeds 65535");
  launch_k(grid_resample_gate_kernel, blocks, dim3(GR_THREADS), (size_t)g * g * 32 * sizeof(float), reinterpret_cast<cudaStream_t>(stream), 1,
           grid, (long long)grid_batch_stride, (bf16*)x, (long long)ldx, gate, stats_out, (long long)stats_slot_stride, g, n, C);
  count_launch();
  return check_launch("grid_resample_gate launch");
}
