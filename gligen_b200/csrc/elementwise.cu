// Small CUDA-core kernels around the tensor-core path: edge convolutions (Cin=4/9 and Cout=4),
// nearest-2x upsample, stride-2 im2col, embeddings, PositionNet feature rows, sampler update.
// All are HBM- or latency-bound; the rule here is coalesced 16-byte accesses and one launch per op.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <string>

#include "common.cuh"
#include "internal.h"
#include "../../include/gligen_b200.h"

namespace glg {

static inline unsigned blocks_for(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  if (b > 2147483647LL) b = 2147483647LL;
  return (unsigned)(b < 1 ? 1 : b);
}

// ---- first conv: NCHW fp32 (x | extra) -> NHWC bf16.  w packed [9][Cin][Cout] fp32. -----------------
// Wide-latent variant (W % 4 == 0, weights fit shared memory): persistent blocks stage the whole [9][Cin][Cout] fp32
// weight once; a thread owns 4 consecutive pixels x 8 output channels, so every weight vector read from smem feeds 32
// FMAs and every input row segment (6 values) feeds three taps.
__global__ void __launch_bounds__(256) conv_in_px4_kernel(const float* __restrict__ x, int C0, const float* __restrict__ extra, int C1,
                                   const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out,
                                   long long ldo, int B, int H, int W, int Cout) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float cin_sw[];      // [9 * Cin][Cout]
  const int Cin = C0 + C1;
  const int nw4 = 9 * Cin * Cout / 4;
  for (int i = threadIdx.x; i < nw4; i += blockDim.x)
    reinterpret_cast<float4*>(cin_sw)[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
  __syncthreads();
  const int cov = Cout >> 3, Wq = W >> 2;
  const long long total = (long long)B * H * Wq * cov;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cov);
    const long long g = i / cov;
    const int x0 = (int)(g % Wq) * 4;
    const int yh = (int)((g / Wq) % H);
    const int b = (int)(g / ((long long)Wq * H));
    float acc[4][8];
    {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c8 * 8)), b1 = __ldg(reinterpret_cast<const float4*>(bias + c8 * 8 + 4));
#pragma unroll
      for (int px = 0; px < 4; ++px) {
        acc[px][0] = b0.x; acc[px][1] = b0.y; acc[px][2] = b0.z; acc[px][3] = b0.w;
        acc[px][4] = b1.x; acc[px][5] = b1.y; acc[px][6] = b1.z; acc[px][7] = b1.w;
      }
    }
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int yy = yh + dy - 1;
      if (yy < 0 || yy >= H) continue;
      for (int ci = 0; ci < Cin; ++ci) {
        const float* row = ci < C0 ? x + (((long long)b * C0 + ci) * H + yy) * W : extra + (((long long)b * C1 + (ci - C0)) * H + yy) * W;
        float r[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          const int xx = x0 + k - 1;
          r[k] = (xx >= 0 && xx < W) ? __ldg(row + xx) : 0.f;
        }
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const float* wp = cin_sw + ((dy * 3 + dx) * Cin + ci) * Cout + c8 * 8;
          const float4 w0 = *reinterpret_cast<const float4*>(wp), w1 = *reinterpret_cast<const float4*>(wp + 4);
#pragma unroll
          for (int px = 0; px < 4; ++px) {
            const float v = r[px + dx];
            acc[px][0] = fmaf(v, w0.x, acc[px][0]); acc[px][1] = fmaf(v, w0.y, acc[px][1]);
            acc[px][2] = fmaf(v, w0.z, acc[px][2]); acc[px][3] = fmaf(v, w0.w, acc[px][3]);
            acc[px][4] = fmaf(v, w1.x, acc[px][4]); acc[px][5] = fmaf(v, w1.y, acc[px][5]);
            acc[px][6] = fmaf(v, w1.z, acc[px][6]); acc[px][7] = fmaf(v, w1.w, acc[px][7]);
          }
        }
      }
    }
    const long long pix0 = ((long long)b * H + yh) * W + x0;
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      uint4 u;
      u.x = pack_bf16x2(acc[px][0], acc[px][1]); u.y = pack_bf16x2(acc[px][2], acc[px][3]);
      u.z = pack_bf16x2(acc[px][4], acc[px][5]); u.w = pack_bf16x2(acc[px][6], acc[px][7]);
      *reinterpret_cast<uint4*>(out + (pix0 + px) * ldo + c8 * 8) = u;
    }
  }
}

__global__ void conv_in_kernel(const float* __restrict__ x, int C0, const float* __restrict__ extra, int C1,
                               const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out,
                               long long ldo, int B, int H, int W, int Cout) {
  pdl_trigger();
  pdl_wait();
  const int cov = Cout >> 3;
  const long long total = (long long)B * H * W * cov;
  const int Cin = C0 + C1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cov);
    const long long pix = i / cov;
    const int xw = (int)(pix % W);
    const int yh = (int)((pix / W) % H);
    const int b = (int)(pix / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bias[c8 * 8 + j];
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = yh + tap / 3 - 1, xx = xw + tap % 3 - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      for (int ci = 0; ci < Cin; ++ci) {
        const float v = ci < C0 ? __ldg(x + (((long long)b * C0 + ci) * H + yy) * W + xx)
                                : __ldg(extra + (((long long)b * C1 + (ci - C0)) * H + yy) * W + xx);
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + ((long long)tap * Cin + ci) * Cout + c8 * 8));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + ((long long)tap * Cin + ci) * Cout + c8 * 8 + 4));
        acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]); acc[2] = fmaf(v, w0.z, acc[2]); acc[3] = fmaf(v, w0.w, acc[3]);
        acc[4] = fmaf(v, w1.x, acc[4]); acc[5] = fmaf(v, w1.y, acc[5]); acc[6] = fmaf(v, w1.z, acc[6]); acc[7] = fmaf(v, w1.w, acc[7]);
      }
    }
    uint4 u;
    u.x = pack_bf16x2(acc[0], acc[1]); u.y = pack_bf16x2(acc[2], acc[3]);
    u.z = pack_bf16x2(acc[4], acc[5]); u.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + pix * ldo + c8 * 8) = u;
  }
}

// ---- last conv: NHWC bf16 -> NCHW fp32, Cout <= 8.  w packed [9][Cout][Cin] fp32.  One warp per pixel.
// Wide-latent variant (W % 8 == 0): one warp owns 8 consecutive pixels, so each weight vector it loads is used for
// 8 pixels (the per-pixel kernel below re-reads all 9 x COUT x Cin weights for every pixel).
template <int COUT>
__global__ void __launch_bounds__(256) conv_out_px8_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ w,
                                    const float* __restrict__ bias, float* __restrict__ out, int B, int H, int W, int Cin) {
  pdl_trigger();
  pdl_wait();
  const int Wo = W >> 3;
  const long long grp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (grp >= (long long)B * H * Wo) return;
  const int lane = threadIdx.x & 31;
  const int x0 = (int)(grp % Wo) * 8;
  const int yh = (int)((grp / Wo) % H);
  const int b = (int)(grp / ((long long)Wo * H));
  float acc[8][COUT];
#pragma unroll
  for (int px = 0; px < 8; ++px)
#pragma unroll
    for (int j = 0; j < COUT; ++j) acc[px][j] = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = yh + tap / 3 - 1, dx = tap % 3 - 1;
    if (yy < 0 || yy >= H) continue;
    const bf16* xrow = x + (((long long)b * H + yy) * W) * ldx;
    for (int c = lane * 8; c < Cin; c += 256) {
      float wv[COUT][8];
#pragma unroll
      for (int co = 0; co < COUT; ++co) {
        const float* wp = w + ((long long)tap * COUT + co) * Cin + c;
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp)), w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
        wv[co][0] = w0.x; wv[co][1] = w0.y; wv[co][2] = w0.z; wv[co][3] = w0.w;
        wv[co][4] = w1.x; wv[co][5] = w1.y; wv[co][6] = w1.z; wv[co][7] = w1.w;
      }
#pragma unroll
      for (int px = 0; px < 8; ++px) {
        const int xx = x0 + px + dx;
        if (xx < 0 || xx >= W) continue;
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xrow + (long long)xx * ldx + c));
        float v[8];
        float2 f;
        f = unpack_bf16x2(u.x); v[0] = f.x; v[1] = f.y;
        f = unpack_bf16x2(u.y); v[2] = f.x; v[3] = f.y;
        f = unpack_bf16x2(u.z); v[4] = f.x; v[5] = f.y;
        f = unpack_bf16x2(u.w); v[6] = f.x; v[7] = f.y;
#pragma unroll
        for (int co = 0; co < COUT; ++co)
          acc[px][co] += v[0] * wv[co][0] + v[1] * wv[co][1] + v[2] * wv[co][2] + v[3] * wv[co][3] + v[4] * wv[co][4] +
                         v[5] * wv[co][5] + v[6] * wv[co][6] + v[7] * wv[co][7];
      }
    }
  }
#pragma unroll
  for (int px = 0; px < 8; ++px)
#pragma unroll
    for (int co = 0; co < COUT; ++co) {
      const float sum = warp_sum(acc[px][co]);
      if (lane == ((px * COUT + co) & 31)) out[(((long long)b * COUT + co) * H + yh) * W + x0 + px] = sum + bias[co];
    }
}

template <int COUT>
__global__ void conv_out_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ w,
                                const float* __restrict__ bias, float* __restrict__ out, int B, int H, int W, int Cin) {
  pdl_trigger();
  pdl_wait();
  const long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= (long long)B * H * W) return;
  const int lane = threadIdx.x & 31;
  const int xw = (int)(pix % W);
  const int yh = (int)((pix / W) % H);
  const int b = (int)(pix / ((long long)W * H));
  float acc[COUT];
#pragma unroll
  for (int j = 0; j < COUT; ++j) acc[j] = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = yh + tap / 3 - 1, xx = xw + tap % 3 - 1;
    if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
    const bf16* xp = x + (((long long)b * H + yy) * W + xx) * ldx;
    for (int c = lane * 8; c < Cin; c += 256) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(xp + c));
      float v[8];
      float2 f;
      f = unpack_bf16x2(u.x); v[0] = f.x; v[1] = f.y;
      f = unpack_bf16x2(u.y); v[2] = f.x; v[3] = f.y;
      f = unpack_bf16x2(u.z); v[4] = f.x; v[5] = f.y;
      f = unpack_bf16x2(u.w); v[6] = f.x; v[7] = f.y;
#pragma unroll
      for (int co = 0; co < COUT; ++co) {
        const float* wp = w + ((long long)tap * COUT + co) * Cin + c;
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
        acc[co] += v[0] * w0.x + v[1] * w0.y + v[2] * w0.z + v[3] * w0.w + v[4] * w1.x + v[5] * w1.y + v[6] * w1.z + v[7] * w1.w;
      }
    }
  }
#pragma unroll
  for (int co = 0; co < COUT; ++co) {
    const float s = warp_sum(acc[co]);
    if (lane == 0) out[(((long long)b * COUT + co) * H + yh) * W + xw] = s + bias[co];
  }
}

__global__ void upsample2x_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy,
                                  int B, int H, int W, int C) {
  pdl_trigger();
  pdl_wait();
  const int vec = C >> 3;
  const int Ho = 2 * H, Wo = 2 * W;
  const long long total = (long long)B * Ho * Wo * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vec);
    const long long pix = i / vec;
    const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((long long)Wo * Ho));
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + (yo >> 1)) * W + (xo >> 1)) * ldx + cv * 8));
    *reinterpret_cast<uint4*>(y + pix * ldy + cv * 8) = u;
  }
}

__global__ void im2col_s2_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, int B, int H, int W, int C, int pad_lo) {
  pdl_trigger();
  pdl_wait();
  const int vec = C >> 3;
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)B * Ho * Wo * 9 * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vec);
    long long t = i / vec;
    const int tap = (int)(t % 9);
    const long long pix = t / 9;
    const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((long long)Wo * Ho));
    const int yy = 2 * yo + tap / 3 - pad_lo, xx = 2 * xo + tap % 3 - pad_lo;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < H && xx >= 0 && xx < W)
      u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * ldx + cv * 8));
    *reinterpret_cast<uint4*>(y + (pix * 9 + tap) * C + cv * 8) = u;
  }
}

__global__ void copy_rows_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy, long long rows, int C) {
  pdl_trigger();
  pdl_wait();
  const int vec = C >> 3;
  const long long total = rows * vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vec; const int cv = (int)(i % vec);
    *reinterpret_cast<uint4*>(y + r * ldy + cv * 8) = __ldg(reinterpret_cast<const uint4*>(x + r * ldx + cv * 8));
  }
}

// T = long long (integer grid timesteps) or float (fractional model time); util.py:170 evaluates timesteps.float() * freqs, so both
// round t to fp32 first and share every instruction after that: integer-valued t gives the same bits through either entry point
template <typename T>
__global__ void timestep_embedding_kernel(const T* __restrict__ t, bf16* __restrict__ out, int B, int dim) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * dim) return;
  const int b = i / dim, j = i % dim;
  const int half = dim / 2;
  const int k = j < half ? j : j - half;
  const float freq = expf(-9.210340371976184f * (float)k / (float)half);   // ln(10000)
  const float arg = (float)t[b] * freq;
  out[i] = __float2bfloat16(j < half ? cosf(arg) : sinf(arg));
}

__global__ void position_features_kernel(const float* __restrict__ feat, long long feat_bs, const float* __restrict__ feat_mask,
                                         const float* __restrict__ null_feat, const float* __restrict__ coords,
                                         const float* __restrict__ pos_mask, const float* __restrict__ null_pos,
                                         bf16* __restrict__ out, long long ldo, int B, int N, int F, int ncoord, int freqs) {
  pdl_trigger();
  pdl_wait();
  const int P = freqs * 2 * ncoord;
  const long long total = (long long)B * N * ldo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % ldo);
    const long long row = i / ldo;
    const int n = (int)(row % N), b = (int)(row / N);
    float v = 0.f;
    if (j < F) {
      const float m = feat_mask[row];
      v = feat[(long long)b * feat_bs + (long long)n * F + j] * m + (1.f - m) * null_feat[j];
    } else if (j < F + P) {
      const int pj = j - F;
      const int k = pj / (2 * ncoord);
      const int rem = pj - k * 2 * ncoord;
      const int is_cos = rem / ncoord, c = rem - is_cos * ncoord;
      const float f = powf(100.f, (float)k / (float)freqs);
      const float a = f * coords[row * ncoord + c];
      const float e = is_cos ? cosf(a) : sinf(a);
      const float m = pos_mask[row];
      v = e * m + (1.f - m) * null_pos[pj];
    }
    out[i] = __float2bfloat16(v);
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long n) {
  pdl_trigger();
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(x[i]);
}

__global__ void sampler_update_kernel(const float* __restrict__ x, const float* __restrict__ ec, const float* __restrict__ eu, float g,
                                      const float* __restrict__ o1, const float* __restrict__ o2, const float* __restrict__ o3,
                                      float c0, float c1, float c2, float c3, float sqrt_at, float sqrt_1m_at,
                                      float sqrt_aprev, float sqrt_1m_aprev,
                                      float* __restrict__ e_out, float* __restrict__ x_prev, long long n) {
  pdl_trigger();
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float e = ec[i];
    if (eu) { const float u = eu[i]; e = u + g * (e - u); }
    if (e_out) e_out[i] = e;
    float ep = c0 * e;
    if (o1) ep += c1 * o1[i];
    if (o2) ep += c2 * o2[i];
    if (o3) ep += c3 * o3[i];
    const float pred_x0 = (x[i] - sqrt_1m_at * ep) / sqrt_at;
    x_prev[i] = sqrt_aprev * pred_x0 + sqrt_1m_aprev * ep;
  }
}

// One DPM-Solver++ multistep update (include/gligen_b200.h, glg_dpm_update).  Elements [0, 4 n4) move as float4 (every
// pointer 16-byte aligned, checked on the host), the tail [4 n4, n) one float at a time.
struct DpmScalars {
  float g, alpha, sigma, cx, k0, k1, k2;
};

__device__ __forceinline__ void dpm_element(float x, float ec, float eu, float m1, float m2, bool cfg, const DpmScalars& s,
                                            float& m0, float& xp) {
  float e = ec;
  if (cfg) e = eu + s.g * (ec - eu);
  m0 = (x - s.sigma * e) / s.alpha;
  xp = s.cx * x + s.k0 * m0 + s.k1 * m1 + s.k2 * m2;
}

__global__ void __launch_bounds__(256) dpm_update_kernel(const float* __restrict__ x, const float* __restrict__ ec, const float* __restrict__ eu,
                                                         const float* __restrict__ m1, const float* __restrict__ m2, DpmScalars s,
                                                         float* __restrict__ x0_out, float* __restrict__ x_prev, long long n4, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool cfg = eu != nullptr;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = tid; i < n4; i += stride) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
    const float4 cv = __ldg(reinterpret_cast<const float4*>(ec) + i);
    const float4 uv = cfg ? __ldg(reinterpret_cast<const float4*>(eu) + i) : zero;
    const float4 p1 = m1 ? __ldg(reinterpret_cast<const float4*>(m1) + i) : zero;
    const float4 p2 = m2 ? __ldg(reinterpret_cast<const float4*>(m2) + i) : zero;
    float4 m0, xp;
    dpm_element(xv.x, cv.x, uv.x, p1.x, p2.x, cfg, s, m0.x, xp.x);
    dpm_element(xv.y, cv.y, uv.y, p1.y, p2.y, cfg, s, m0.y, xp.y);
    dpm_element(xv.z, cv.z, uv.z, p1.z, p2.z, cfg, s, m0.z, xp.z);
    dpm_element(xv.w, cv.w, uv.w, p1.w, p2.w, cfg, s, m0.w, xp.w);
    reinterpret_cast<float4*>(x0_out)[i] = m0;
    reinterpret_cast<float4*>(x_prev)[i] = xp;
  }
  for (long long i = 4 * n4 + tid; i < n; i += stride) {
    float m0, xp;
    dpm_element(x[i], ec[i], cfg ? eu[i] : 0.f, m1 ? m1[i] : 0.f, m2 ? m2[i] : 0.f, cfg, s, m0, xp);
    x0_out[i] = m0;
    x_prev[i] = xp;
  }
}

// One UniPC step (include/gligen_b200.h, glg_unipc_update): the corrector for the point just evaluated, then the predictor
// from the corrected state.  Elements [0, 4 n4) move as float4 (every pointer 16-byte aligned, checked on the host), the tail
// [4 n4, n) one float at a time.
struct UniPCScalars {
  float g, alpha, sigma, cc, c0, c1, c2, c3, pc, p0, p1, p2;
};

__device__ __forceinline__ void unipc_element(float x, float xcp, float ec, float eu, float m1, float m2, float m3, bool cfg, bool corr,
                                              const UniPCScalars& s, float& m0, float& xc, float& xn) {
  float e = ec;
  if (cfg) e = eu + s.g * (ec - eu);
  m0 = (x - s.sigma * e) / s.alpha;
  xc = corr ? s.cc * xcp + s.c0 * m0 + s.c1 * m1 + s.c2 * m2 + s.c3 * m3 : x;
  xn = s.pc * xc + s.p0 * m0 + s.p1 * m1 + s.p2 * m2;
}

__global__ void __launch_bounds__(256) unipc_update_kernel(const float* __restrict__ x, const float* __restrict__ xcp,
                                                           const float* __restrict__ ec, const float* __restrict__ eu,
                                                           const float* __restrict__ m1, const float* __restrict__ m2,
                                                           const float* __restrict__ m3, UniPCScalars s, float* __restrict__ m_out,
                                                           float* __restrict__ xc_out, float* __restrict__ x_next, long long n4, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool cfg = eu != nullptr, corr = xcp != nullptr;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = tid; i < n4; i += stride) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
    const float4 cp = corr ? __ldg(reinterpret_cast<const float4*>(xcp) + i) : zero;
    const float4 cv = __ldg(reinterpret_cast<const float4*>(ec) + i);
    const float4 uv = cfg ? __ldg(reinterpret_cast<const float4*>(eu) + i) : zero;
    const float4 h1 = m1 ? __ldg(reinterpret_cast<const float4*>(m1) + i) : zero;
    const float4 h2 = m2 ? __ldg(reinterpret_cast<const float4*>(m2) + i) : zero;
    const float4 h3 = m3 ? __ldg(reinterpret_cast<const float4*>(m3) + i) : zero;
    float4 m0, xc, xn;
    unipc_element(xv.x, cp.x, cv.x, uv.x, h1.x, h2.x, h3.x, cfg, corr, s, m0.x, xc.x, xn.x);
    unipc_element(xv.y, cp.y, cv.y, uv.y, h1.y, h2.y, h3.y, cfg, corr, s, m0.y, xc.y, xn.y);
    unipc_element(xv.z, cp.z, cv.z, uv.z, h1.z, h2.z, h3.z, cfg, corr, s, m0.z, xc.z, xn.z);
    unipc_element(xv.w, cp.w, cv.w, uv.w, h1.w, h2.w, h3.w, cfg, corr, s, m0.w, xc.w, xn.w);
    reinterpret_cast<float4*>(m_out)[i] = m0;
    reinterpret_cast<float4*>(xc_out)[i] = xc;
    reinterpret_cast<float4*>(x_next)[i] = xn;
  }
  for (long long i = 4 * n4 + tid; i < n; i += stride) {
    float m0, xc, xn;
    unipc_element(x[i], corr ? xcp[i] : 0.f, ec[i], cfg ? eu[i] : 0.f, m1 ? m1[i] : 0.f, m2 ? m2[i] : 0.f, m3 ? m3[i] : 0.f, cfg, corr, s,
                  m0, xc, xn);
    m_out[i] = m0;
    xc_out[i] = xc;
    x_next[i] = xn;
  }
}

// One stochastic sampler step (include/gligen_b200.h, glg_sde_update): DDIM with eta > 0 or DPM-Solver++ 2M SDE.  Elements
// [0, 4 n4) move as float4 (every pointer 16-byte aligned, checked on the host), the tail [4 n4, n) one float at a time.
struct SdeScalars {
  float g, alpha, sigma, cx, k0, k1, ce, cz;
};

__device__ __forceinline__ void sde_element(float x, float ec, float eu, float m1, float z, bool cfg, const SdeScalars& s, float& m0,
                                            float& xn) {
  float e = ec;
  if (cfg) e = eu + s.g * (ec - eu);
  m0 = (x - s.sigma * e) / s.alpha;
  xn = s.cx * x + s.k0 * m0 + s.k1 * m1 + s.ce * e + s.cz * z;
}

__global__ void __launch_bounds__(256) sde_update_kernel(const float* __restrict__ x, const float* __restrict__ ec, const float* __restrict__ eu,
                                                         const float* __restrict__ m1, const float* __restrict__ z, SdeScalars s,
                                                         float* __restrict__ x0_out, float* __restrict__ x_next, long long n4, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool cfg = eu != nullptr;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = tid; i < n4; i += stride) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
    const float4 cv = __ldg(reinterpret_cast<const float4*>(ec) + i);
    const float4 uv = cfg ? __ldg(reinterpret_cast<const float4*>(eu) + i) : zero;
    const float4 p1 = m1 ? __ldg(reinterpret_cast<const float4*>(m1) + i) : zero;
    const float4 zv = __ldg(reinterpret_cast<const float4*>(z) + i);
    float4 m0, xn;
    sde_element(xv.x, cv.x, uv.x, p1.x, zv.x, cfg, s, m0.x, xn.x);
    sde_element(xv.y, cv.y, uv.y, p1.y, zv.y, cfg, s, m0.y, xn.y);
    sde_element(xv.z, cv.z, uv.z, p1.z, zv.z, cfg, s, m0.z, xn.z);
    sde_element(xv.w, cv.w, uv.w, p1.w, zv.w, cfg, s, m0.w, xn.w);
    if (x0_out) reinterpret_cast<float4*>(x0_out)[i] = m0;
    reinterpret_cast<float4*>(x_next)[i] = xn;
  }
  for (long long i = 4 * n4 + tid; i < n; i += stride) {
    float m0, xn;
    sde_element(x[i], ec[i], cfg ? eu[i] : 0.f, m1 ? m1[i] : 0.f, z[i], cfg, s, m0, xn);
    if (x0_out) x0_out[i] = m0;
    x_next[i] = xn;
  }
}

}  // namespace glg

namespace glg {
// Row softmax of an fp32 score matrix -> bf16 probabilities (sum of a row = 1 before rounding): one CTA per row.
// Used by the VAE decoder's single-head attention over H*W tokens (model.py:178-202), whose head dim (512) is too wide
// for the flash kernels' register-resident output tile: QK^T and P.V run as glg_gemm, the scores make one round trip through L2.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, long long lds, bf16* __restrict__ p, long long ldp,
                                                          int cols, float scale_log2) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[8];
  const float* row = s + (long long)blockIdx.x * lds;
  bf16* out = p + (long long)blockIdx.x * ldp;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int c = threadIdx.x * 4; c < cols; c += 1024) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  const float ms = mx * scale_log2;
  float sum = 0.f;
  for (int c = threadIdx.x * 4; c < cols; c += 1024) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    sum += exp2f(fmaf(v.x, scale_log2, -ms)) + exp2f(fmaf(v.y, scale_log2, -ms)) + exp2f(fmaf(v.z, scale_log2, -ms)) + exp2f(fmaf(v.w, scale_log2, -ms));
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];           // fixed order
  const float inv = 1.0f / tot;
  for (int c = threadIdx.x * 4; c < cols; c += 1024) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
    uint2 u;
    u.x = pack_bf16x2(exp2f(fmaf(v.x, scale_log2, -ms)) * inv, exp2f(fmaf(v.y, scale_log2, -ms)) * inv);
    u.y = pack_bf16x2(exp2f(fmaf(v.z, scale_log2, -ms)) * inv, exp2f(fmaf(v.w, scale_log2, -ms)) * inv);
    *reinterpret_cast<uint2*>(out + c) = u;
  }
}
}  // namespace glg

using namespace glg;
#define ST reinterpret_cast<cudaStream_t>(stream)

extern "C" int glg_conv_in(const float* x, int32_t C0, const float* extra, int32_t C1, const float* w, const float* bias,
                           void* out, int64_t ldo, int32_t B, int32_t H, int32_t Wd, int32_t Cout, void* stream) {
  if (Cout % 8 || ldo % 8) return set_error("glg_conv_in: Cout and ldo must be multiples of 8");
  if (C1 > 0 && !extra) return set_error("glg_conv_in: extra channels requested but pointer is null");
  const long long total = (long long)B * H * Wd * (Cout / 8);
  const size_t wbytes = (size_t)9 * (C0 + C1) * Cout * sizeof(float);
  if (Wd % 4 == 0 && wbytes <= 110 * 1024 && total >= 4 * 256 * 64) {
    static size_t attr_bytes = 0;
    if (wbytes > attr_bytes) {
      cudaError_t e = cudaFuncSetAttribute(conv_in_px4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wbytes);
      if (e != cudaSuccess) return set_error(std::string("cudaFuncSetAttribute(conv_in): ") + cudaGetErrorString(e));
      attr_bytes = wbytes;
    }
    unsigned grid = blocks_for(total / 4, 256);
    const unsigned cap = 2u * (unsigned)num_sms();
    if (grid > cap) grid = cap;
    launch_k(conv_in_px4_kernel, dim3(grid), dim3(256), wbytes, ST, 1, x, C0, extra, C1, w, bias, (bf16*)out, ldo, B, H, Wd, Cout);
  } else {
    launch_k(conv_in_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, ST, 1, x, C0, extra, C1, w, bias, (bf16*)out, ldo, B, H, Wd, Cout);
  }
  count_launch();
  return check_launch("conv_in launch");
}

extern "C" int glg_conv_out(const void* x, int64_t ldx, const float* w, const float* bias, float* out,
                            int32_t B, int32_t H, int32_t Wd, int32_t Cin, int32_t Cout, void* stream) {
  if (Cin % 8 || ldx % 8) return set_error("glg_conv_out: Cin and ldx must be multiples of 8");
  const long long pix = (long long)B * H * Wd;
  if (Wd % 8 == 0 && (Cout == 4 || Cout == 3)) {
    if (Cout == 4) launch_k(conv_out_px8_kernel<4>, dim3(blocks_for(pix / 8, 8)), dim3(256), 0, ST, 1, (const bf16*)x, ldx, w, bias, out, B, H, Wd, Cin);
    else launch_k(conv_out_px8_kernel<3>, dim3(blocks_for(pix / 8, 8)), dim3(256), 0, ST, 1, (const bf16*)x, ldx, w, bias, out, B, H, Wd, Cin);
    count_launch();
    return check_launch("conv_out launch");
  }
  const unsigned grid = blocks_for(pix, 8);
  if (Cout == 4) launch_k(conv_out_kernel<4>, dim3(grid), dim3(256), 0, ST, 1, (const bf16*)x, ldx, w, bias, out, B, H, Wd, Cin);
  else if (Cout == 8) launch_k(conv_out_kernel<8>, dim3(grid), dim3(256), 0, ST, 1, (const bf16*)x, ldx, w, bias, out, B, H, Wd, Cin);
  else if (Cout == 3) launch_k(conv_out_kernel<3>, dim3(grid), dim3(256), 0, ST, 1, (const bf16*)x, ldx, w, bias, out, B, H, Wd, Cin);
  else return set_error("glg_conv_out: Cout must be 3, 4 or 8");
  count_launch();
  return check_launch("conv_out launch");
}

extern "C" int glg_softmax_rows(const float* s, int64_t lds, void* p, int64_t ldp, int64_t rows, int32_t cols, float scale, void* stream) {
  // the kernel reads 4 scores as one float4 and writes 4 probabilities as one 8-byte store per thread and step
  if (cols <= 0 || cols % 4 || ldp % 4 || lds % 4 || ((uintptr_t)s & 15) || ((uintptr_t)p & 7))
    return set_error("glg_softmax_rows: cols % 4, lds % 4, ldp % 4, s 16-byte and p 8-byte aligned required");
  if (rows <= 0) return 0;
  launch_k(softmax_rows_kernel, dim3((unsigned)rows), dim3(256), 0, ST, 1, s, (long long)lds, (bf16*)p, (long long)ldp, cols, scale * 1.4426950408889634f);
  count_launch();
  return check_launch("softmax_rows launch");
}

extern "C" int glg_upsample2x(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t B, int32_t H, int32_t Wd, int32_t C, void* stream) {
  if (C % 8 || ldx % 8 || ldy % 8) return set_error("glg_upsample2x: C and leading dims must be multiples of 8");
  const long long total = (long long)B * 4 * H * Wd * (C / 8);
  launch_k(upsample2x_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, ST, 1, (const bf16*)x, ldx, (bf16*)y, ldy, B, H, Wd, C);
  count_launch();
  return check_launch("upsample2x launch");
}

extern "C" int glg_im2col_s2_pad(const void* x, int64_t ldx, void* y, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t pad_lo, void* stream) {
  if (C % 8 || ldx % 8 || (H & 1) || (Wd & 1)) return set_error("glg_im2col_s2: C % 8, even H/W required");
  if (pad_lo != 0 && pad_lo != 1) return set_error("glg_im2col_s2_pad: pad_lo must be 0 (pad right/bottom only) or 1 (symmetric)");
  const long long total = (long long)B * (H / 2) * (Wd / 2) * 9 * (C / 8);
  launch_k(im2col_s2_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, ST, 1, (const bf16*)x, ldx, (bf16*)y, B, H, Wd, C, pad_lo);
  count_launch();
  return check_launch("im2col_s2 launch");
}

extern "C" int glg_im2col_s2(const void* x, int64_t ldx, void* y, int32_t B, int32_t H, int32_t Wd, int32_t C, void* stream) {
  return glg_im2col_s2_pad(x, ldx, y, B, H, Wd, C, 1, stream);
}

extern "C" int glg_copy_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int32_t C, void* stream) {
  if (C % 8 || ldx % 8 || ldy % 8) return set_error("glg_copy_rows: C and leading dims must be multiples of 8");
  launch_k(copy_rows_kernel, dim3(blocks_for(rows * (C / 8), 256)), dim3(256), 0, ST, 1, (const bf16*)x, ldx, (bf16*)y, ldy, rows, C);
  count_launch();
  return check_launch("copy_rows launch");
}

extern "C" int glg_timestep_embedding(const int64_t* t, void* out, int32_t B, int32_t dim, void* stream) {
  if (dim % 2) return set_error("glg_timestep_embedding: dim must be even");
  launch_k(timestep_embedding_kernel<long long>, dim3(blocks_for((long long)B * dim, 256)), dim3(256), 0, ST, 1, (const long long*)t, (bf16*)out, B, dim);
  count_launch();
  return check_launch("timestep_embedding launch");
}

extern "C" int glg_timestep_embedding_f32(const float* t, void* out, int32_t B, int32_t dim, void* stream) {
  if (dim % 2) return set_error("glg_timestep_embedding_f32: dim must be even");
  launch_k(timestep_embedding_kernel<float>, dim3(blocks_for((long long)B * dim, 256)), dim3(256), 0, ST, 1, t, (bf16*)out, B, dim);
  count_launch();
  return check_launch("timestep_embedding_f32 launch");
}

extern "C" int glg_position_features(const float* feat, int64_t feat_batch_stride, const float* feat_mask, const float* null_feat,
                                     const float* coords, const float* pos_mask, const float* null_pos, void* out, int64_t ldo,
                                     int32_t B, int32_t N, int32_t F, int32_t ncoord, int32_t freqs, void* stream) {
  if (ldo < F + freqs * 2 * ncoord) return set_error("glg_position_features: ldo too small");
  launch_k(position_features_kernel, dim3(blocks_for((long long)B * N * ldo, 256)), dim3(256), 0, ST, 1, feat, feat_batch_stride, feat_mask, null_feat, coords,
                                                                                    pos_mask, null_pos, (bf16*)out, ldo, B, N, F, ncoord, freqs);
  count_launch();
  return check_launch("position_features launch");
}

extern "C" int glg_cast_f32_bf16(const float* x, void* y, int64_t n, void* stream) {
  launch_k(cast_f32_bf16_kernel, dim3(blocks_for(n, 256) > 4096 ? 4096 : blocks_for(n, 256)), dim3(256), 0, ST, 1, x, (bf16*)y, n);
  count_launch();
  return check_launch("cast launch");
}

extern "C" int glg_sampler_update(const float* x, const float* e_cond, const float* e_uncond, float guidance,
                                  const float* old1, const float* old2, const float* old3,
                                  float c0, float c1, float c2, float c3, float a_t, float a_prev,
                                  float* e_out, float* x_prev, int64_t n, void* stream) {
  launch_k(sampler_update_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ST, 1, x, e_cond, e_uncond, guidance, old1, old2, old3, c0, c1, c2, c3,
                                                            sqrtf(a_t), sqrtf(1.f - a_t), sqrtf(a_prev), sqrtf(1.f - a_prev), e_out, x_prev, n);
  count_launch();
  return check_launch("sampler_update launch");
}

extern "C" int glg_dpm_update(const float* x, const float* e_cond, const float* e_uncond, float guidance, const float* m1, const float* m2,
                              float alpha, float sigma, float cx, float k0, float k1, float k2, float* x0_out, float* x_prev, int64_t n,
                              void* stream) {
  if (!x || !e_cond || !x0_out || !x_prev) return set_error("glg_dpm_update: x, e_cond, x0_out and x_prev are required");
  if (n < 0) return set_error("glg_dpm_update: n must be >= 0");
  if (n == 0) return 0;
  const uintptr_t bits = (uintptr_t)x | (uintptr_t)e_cond | (uintptr_t)e_uncond | (uintptr_t)m1 | (uintptr_t)m2 | (uintptr_t)x0_out |
                         (uintptr_t)x_prev;
  const long long n4 = (bits & 15) ? 0 : n / 4;          // a misaligned view takes the scalar path for all of n
  const DpmScalars s{guidance, alpha, sigma, cx, k0, k1, k2};
  const unsigned grid = blocks_for(n4 > 0 ? n4 : n, 256);
  launch_k(dpm_update_kernel, dim3(grid > 4096 ? 4096 : grid), dim3(256), 0, ST, 1, x, e_cond, e_uncond, m1, m2, s, x0_out, x_prev, n4, (long long)n);
  count_launch();
  return check_launch("dpm_update launch");
}

extern "C" int glg_unipc_update(const float* x, const float* xc_prev, const float* e_cond, const float* e_uncond, float guidance,
                                const float* m1, const float* m2, const float* m3, float alpha, float sigma, float cc, float c0, float c1,
                                float c2, float c3, float pc, float p0, float p1, float p2, float* m_out, float* xc_out, float* x_next,
                                int64_t n, void* stream) {
  if (!x || !e_cond || !m_out || !xc_out || !x_next) return set_error("glg_unipc_update: x, e_cond, m_out, xc_out and x_next are required");
  if (n < 0) return set_error("glg_unipc_update: n must be >= 0");
  if (n == 0) return 0;
  const uintptr_t bits = (uintptr_t)x | (uintptr_t)xc_prev | (uintptr_t)e_cond | (uintptr_t)e_uncond | (uintptr_t)m1 | (uintptr_t)m2 |
                         (uintptr_t)m3 | (uintptr_t)m_out | (uintptr_t)xc_out | (uintptr_t)x_next;
  const long long n4 = (bits & 15) ? 0 : n / 4;          // a misaligned view takes the scalar path for all of n
  const UniPCScalars s{guidance, alpha, sigma, cc, c0, c1, c2, c3, pc, p0, p1, p2};
  const unsigned grid = blocks_for(n4 > 0 ? n4 : n, 256);
  launch_k(unipc_update_kernel, dim3(grid > 4096 ? 4096 : grid), dim3(256), 0, ST, 1, x, xc_prev, e_cond, e_uncond, m1, m2, m3, s, m_out,
           xc_out, x_next, n4, (long long)n);
  count_launch();
  return check_launch("unipc_update launch");
}

extern "C" int glg_sde_update(const float* x, const float* e_cond, const float* e_uncond, float guidance, const float* m1, const float* z,
                              float alpha, float sigma, float cx, float k0, float k1, float ce, float cz, float* x0_out, float* x_next,
                              int64_t n, void* stream) {
  if (n < 0) return set_error("glg_sde_update: n must be >= 0");
  if (n == 0) return 0;                                  // empty tensors may carry null pointers
  if (!x || !e_cond || !z || !x_next) return set_error("glg_sde_update: x, e_cond, z and x_next are required");
  const uintptr_t bits = (uintptr_t)x | (uintptr_t)e_cond | (uintptr_t)e_uncond | (uintptr_t)m1 | (uintptr_t)z | (uintptr_t)x0_out |
                         (uintptr_t)x_next;
  const long long n4 = (bits & 15) ? 0 : n / 4;          // a misaligned view takes the scalar path for all of n
  const SdeScalars s{guidance, alpha, sigma, cx, k0, k1, ce, cz};
  const unsigned grid = blocks_for(n4 > 0 ? n4 : n, 256);
  launch_k(sde_update_kernel, dim3(grid > 4096 ? 4096 : grid), dim3(256), 0, ST, 1, x, e_cond, e_uncond, m1, z, s, x0_out, x_next, n4, (long long)n);
  count_launch();
  return check_launch("sde_update launch");
}
