// Front-end kernels of the spatial grounding modalities (hed / canny / depth / normal / semantic maps; SURVEY 8f-4):
// the ConvNeXt-tiny grounding tokenizer (reference ldm/modules/diffusionmodules/convnext.py, *_grounding_net.py) and the
// grounding downsamplers (*_grounding_downsampler.py).  They run ONCE per sample (timestep-invariant), are CUDA-core,
// HBM / latency bound, and exist so that the whole conditioning path stays on this library: the dense layers between them
// (stem / downsample patch convolutions, pointwise MLPs of the ConvNeXt blocks, PositionNet MLP) are glg_gemm calls.
//   patchify      k x k stride-k patches -> GEMM rows  (Conv2d(k, stride k) == GEMM over patches; nearest resize fused in)
//   layernorm_rows per-row LayerNorm over the first C columns of strided rows (channels_first LayerNorm of an NHWC tensor)
//   dwconv7_ln    depthwise 7x7 + bias + LayerNorm(eps 1e-6) in one pass (convnext.py:40-44)
//   resize_plane  bicubic (A = -0.75, align_corners = False) / nearest resampling of NCHW fp32 planes (F.interpolate)
//   conv2d_small  direct k x k convolution with <= 16 output channels on NCHW fp32 (+ SiLU), nearest resize fused in
// and the CLIP towers' front / back ends: embed_tokens (text), clip_vision_embed (CLS + patches + positions + pre-LayerNorm) and
// clip_image_head (post-LayerNorm of the CLS row, visual projection, GLIGEN's reprojection) for the image tower.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <string>

#include "common.cuh"
#include "internal.h"
#include "../../include/gligen_b200.h"

namespace glg {

static inline unsigned fe_blocks(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  if (b > 1048576LL) b = 1048576LL;
  return (unsigned)(b < 1 ? 1 : b);
}

// F.interpolate(mode="nearest"): src = min(floor(dst * (in / out)), in - 1), the scale computed in fp32 as ATen does
__device__ __forceinline__ int nearest_src(int dst, float scale, int in_size) {
  const int s = (int)floorf((float)dst * scale);
  return s < in_size - 1 ? s : in_size - 1;
}

// ---- patchify, NCHW fp32 source sampled on a virtual Hv x Wv grid (nearest) ------------------------------------------
// out[(b, oy, ox)][(ky * k + kx) * C + c] = x[b, c, src(oy * k + ky), src(ox * k + kx)];  columns [k*k*C, ldo) = 0
__global__ void patchify_nchw_kernel(const float* __restrict__ x, bf16* __restrict__ out, long long ldo, int B, int C, int Hs, int Ws,
                                     int Hv, int Wv, int k) {
  pdl_trigger();
  pdl_wait();
  const int Ho = Hv / k, Wo = Wv / k, kkc = k * k * C;
  const float sh = (float)Hs / (float)Hv, sw = (float)Ws / (float)Wv;
  const long long total = (long long)B * Ho * Wo * ldo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % ldo);
    const long long row = i / ldo;
    float v = 0.f;
    if (col < kkc) {
      const int c = col % C, tap = col / C, ky = tap / k, kx = tap % k;
      const int ox = (int)(row % Wo), oy = (int)((row / Wo) % Ho), b = (int)(row / ((long long)Wo * Ho));
      const int sy = nearest_src(oy * k + ky, sh, Hs), sx = nearest_src(ox * k + kx, sw, Ws);
      v = __ldg(x + (((long long)b * C + c) * Hs + sy) * Ws + sx);
    }
    out[i] = __float2bfloat16(v);
  }
}

// ---- patchify, NHWC bf16 source (C % 8 == 0): out[(b, oy, ox)][(ky * k + kx) * C + c] = x[b, oy*k+ky, ox*k+kx, c] ----------
__global__ void patchify_nhwc_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ out, long long ldo, int B, int H, int W,
                                     int C, int k) {
  pdl_trigger();
  pdl_wait();
  const int Ho = H / k, Wo = W / k, c8n = C >> 3, chunks = k * k * c8n;
  const long long total = (long long)B * Ho * Wo * chunks;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % chunks);
    const long long row = i / chunks;
    const int c8 = ch % c8n, tap = ch / c8n, ky = tap / k, kx = tap % k;
    const int ox = (int)(row % Wo), oy = (int)((row / Wo) % Ho), b = (int)(row / ((long long)Wo * Ho));
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + oy * k + ky) * W + ox * k + kx) * ldx + c8 * 8));
    *reinterpret_cast<uint4*>(out + row * ldo + (long long)tap * C + c8 * 8) = u;
  }
}

// ---- LayerNorm over the first C columns of strided bf16 rows; one warp per row; columns [C, Cpad) of y are zeroed -----------
// (two-pass in registers: mean, then mean of squared deviations - the reference's channels_first form, convnext.py:135-139)
constexpr int LNR_MAX_CHUNKS = 4;          // C <= 32 * 8 * 4 = 1024
template <bool F32OUT>                     // F32OUT: y is fp32 (the text encoder's last_hidden_state), no padding columns
__global__ void __launch_bounds__(256) layernorm_rows_kernel(const bf16* __restrict__ x, long long ldx, void* __restrict__ yv, long long ldy,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             long long rows, int C, int Cpad, float eps) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int c8n = C >> 3;
  float v[LNR_MAX_CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < c8n) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + row * ldx + c8 * 8);
      float2 f;
      f = unpack_bf16x2(u.x); v[i][0] = f.x; v[i][1] = f.y;
      f = unpack_bf16x2(u.y); v[i][2] = f.x; v[i][3] = f.y;
      f = unpack_bf16x2(u.z); v[i][4] = f.x; v[i][5] = f.y;
      f = unpack_bf16x2(u.w); v[i][6] = f.x; v[i][7] = f.y;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    if (lane + 32 * i < c8n) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q = fmaf(d, d, q); }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < c8n) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf((v[i][j] - mean) * rstd, __ldg(gamma + c8 * 8 + j), __ldg(beta + c8 * 8 + j));
      if (F32OUT) {
        float* y = reinterpret_cast<float*>(yv) + row * ldy + c8 * 8;
        *reinterpret_cast<float4*>(y) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(y + 4) = make_float4(o[4], o[5], o[6], o[7]);
      } else {
        uint4 u;
        u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]); u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
        *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(yv) + row * ldy + c8 * 8) = u;
      }
    } else if (!F32OUT && c8 * 8 < Cpad) {
      *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(yv) + row * ldy + c8 * 8) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

// ---- depthwise 7x7 (pad 3) + bias + LayerNorm over channels, NHWC bf16; one warp per output pixel --------------------------
// w packed [49][C] fp32 (tap-major); lanes own channel pairs p = lane + 32 i; columns [C, Cpad) of y are zeroed.
constexpr int DW_MAX_PAIRS = 12;           // C <= 768
__global__ void __launch_bounds__(256) dwconv7_ln_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy,
                                                         const float* __restrict__ w, const float* __restrict__ bias,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                                         int B, int H, int W, int C, int Cpad, float eps) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= (long long)B * H * W) return;
  const int xw = (int)(pix % W), yh = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  const int np = C >> 1;
  float2 acc[DW_MAX_PAIRS];
#pragma unroll
  for (int i = 0; i < DW_MAX_PAIRS; ++i) {
    const int p = lane + 32 * i;
    acc[i] = p < np ? __ldg(reinterpret_cast<const float2*>(bias) + p) : make_float2(0.f, 0.f);
  }
  for (int ky = 0; ky < 7; ++ky) {
    const int yy = yh + ky - 3;
    if (yy < 0 || yy >= H) continue;
    for (int kx = 0; kx < 7; ++kx) {
      const int xx = xw + kx - 3;
      if (xx < 0 || xx >= W) continue;
      const bf16* xr = x + (((long long)b * H + yy) * W + xx) * ldx;
      const float2* wr = reinterpret_cast<const float2*>(w + (long long)(ky * 7 + kx) * C);
#pragma unroll
      for (int i = 0; i < DW_MAX_PAIRS; ++i) {
        const int p = lane + 32 * i;
        if (p < np) {
          const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xr + 2 * p));
          const float2 ww = __ldg(wr + p);
          acc[i].x = fmaf(f.x, ww.x, acc[i].x);
          acc[i].y = fmaf(f.y, ww.y, acc[i].y);
        }
      }
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < DW_MAX_PAIRS; ++i)
    if (lane + 32 * i < np) s += acc[i].x + acc[i].y;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < DW_MAX_PAIRS; ++i)
    if (lane + 32 * i < np) { const float d0 = acc[i].x - mean, d1 = acc[i].y - mean; q = fmaf(d0, d0, fmaf(d1, d1, q)); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  bf16* yr = y + pix * ldy;
#pragma unroll
  for (int i = 0; i < DW_MAX_PAIRS; ++i) {
    const int p = lane + 32 * i;
    if (p < np) {
      const float2 g = __ldg(reinterpret_cast<const float2*>(gamma) + p), bt = __ldg(reinterpret_cast<const float2*>(beta) + p);
      *reinterpret_cast<uint32_t*>(yr + 2 * p) = pack_bf16x2(fmaf((acc[i].x - mean) * rstd, g.x, bt.x), fmaf((acc[i].y - mean) * rstd, g.y, bt.y));
    } else if (2 * p < Cpad) {
      *reinterpret_cast<uint32_t*>(yr + 2 * p) = 0u;
    }
  }
}

// ---- F.interpolate on NCHW fp32 planes: mode 0 nearest, 1 bicubic (align_corners=False, A = -0.75, border-clamped taps) ----
__device__ __forceinline__ float cubic1(float t, float A) { return ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f; }
__device__ __forceinline__ float cubic2(float t, float A) { return ((A * t - 5.f * A) * t + 8.f * A) * t - 4.f * A; }
__device__ __forceinline__ void cubic_coeffs(float t, float* c) {
  const float A = -0.75f;
  c[0] = cubic2(t + 1.f, A); c[1] = cubic1(t, A); c[2] = cubic1(1.f - t, A); c[3] = cubic2(2.f - t, A);
}
__global__ void resize_plane_kernel(const float* __restrict__ x, long long x_batch, float* __restrict__ y, int B, int C, int Hs, int Ws,
                                    int Ho, int Wo, int mode) {
  pdl_trigger();
  pdl_wait();
  const float sh = (float)Hs / (float)Ho, sw = (float)Ws / (float)Wo;
  const long long total = (long long)B * C * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), c = (int)((i / ((long long)Wo * Ho)) % C), b = (int)(i / ((long long)Wo * Ho * C));
    const float* src = x + (long long)b * x_batch + (long long)c * Hs * Ws;
    if (mode == 0) {
      y[i] = __ldg(src + (long long)nearest_src(oy, sh, Hs) * Ws + nearest_src(ox, sw, Ws));
      continue;
    }
    const float ry = sh * ((float)oy + 0.5f) - 0.5f, rx = sw * ((float)ox + 0.5f) - 0.5f;
    const float fy = floorf(ry), fx = floorf(rx);
    const int iy = (int)fy, ix = (int)fx;
    float cy[4], cx[4];
    cubic_coeffs(ry - fy, cy);
    cubic_coeffs(rx - fx, cx);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int yy = min(max(iy - 1 + j, 0), Hs - 1);
      float r = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int xx = min(max(ix - 1 + k, 0), Ws - 1);
        r = fmaf(cx[k], __ldg(src + (long long)yy * Ws + xx), r);
      }
      acc = fmaf(cy[j], r, acc);
    }
    y[i] = acc;
  }
}

// ---- direct convolution, <= 16 output channels, NCHW fp32 in / out; the input is the source resampled (nearest) onto a
// virtual Hv x Wv grid (Hv == Hs, Wv == Ws: no resampling).  w packed [Cin * k * k][CO] fp32.  One thread per output pixel.
template <int CO>
__global__ void __launch_bounds__(128) conv2d_small_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                           float* __restrict__ y, int B, int Cin, int Hs, int Ws, int Hv, int Wv, int k, int stride,
                                                           int pad, int Ho, int Wo, int silu) {
  pdl_trigger();
  pdl_wait();
  const float sh = (float)Hs / (float)Hv, sw = (float)Ws / (float)Wv;
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), b = (int)(i / ((long long)Wo * Ho));
    float acc[CO];
#pragma unroll
    for (int j = 0; j < CO; ++j) acc[j] = __ldg(bias + j);
    for (int ky = 0; ky < k; ++ky) {
      const int vy = oy * stride - pad + ky;
      if (vy < 0 || vy >= Hv) continue;
      const int sy = nearest_src(vy, sh, Hs);
      for (int kx = 0; kx < k; ++kx) {
        const int vx = ox * stride - pad + kx;
        if (vx < 0 || vx >= Wv) continue;
        const int sx = nearest_src(vx, sw, Ws);
        const float* xp = x + ((long long)b * Cin * Hs + sy) * Ws + sx;
        const float* wp = w + (long long)(ky * k + kx) * CO;
        for (int ci = 0; ci < Cin; ++ci) {
          const float v = __ldg(xp + (long long)ci * Hs * Ws);
          const float* wr = wp + (long long)ci * k * k * CO;
#pragma unroll
          for (int j = 0; j < CO; ++j) acc[j] = fmaf(v, __ldg(wr + j), acc[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < CO; ++j) {
      const float v = silu ? silu_f(acc[j]) : acc[j];
      y[(((long long)b * CO + j) * Ho + oy) * Wo + ox] = v;
    }
  }
}

// ---- grounding tokens of a spatial map (hed_grounding_net.py:47-56): y[b, t, :] = x[b, t, :] * m[b] + null * (1 - m[b]) + pos[t, :] -------
__global__ void spatial_tokens_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ mask, const float* __restrict__ null_feat,
                                      const float* __restrict__ pos, bf16* __restrict__ y, long long ldy, int B, int n, int C) {
  pdl_trigger();
  pdl_wait();
  const int c8n = C >> 3;
  const long long total = (long long)B * n * c8n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % c8n);
    const long long row = i / c8n;
    const int t = (int)(row % n), b = (int)(row / n);
    const float m = __ldg(mask + b);
    const uint4 u = *reinterpret_cast<const uint4*>(x + row * ldx + c8 * 8);
    float v[8];
    float2 f;
    f = unpack_bf16x2(u.x); v[0] = f.x; v[1] = f.y;
    f = unpack_bf16x2(u.y); v[2] = f.x; v[3] = f.y;
    f = unpack_bf16x2(u.z); v[4] = f.x; v[5] = f.y;
    f = unpack_bf16x2(u.w); v[6] = f.x; v[7] = f.y;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = v[j] * m + __ldg(null_feat + c8 * 8 + j) * (1.f - m) + __ldg(pos + (long long)t * C + c8 * 8 + j);
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]); o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(y + row * ldy + c8 * 8) = o;
  }
}

// ---- text-encoder input rows (transformers CLIPTextEmbeddings): out[b, l, :] = bf16(table[ids[b, l], :] + pos[l, :]) ---------------
// ids outside [0, vocab) are clamped (a corrupt id must not read out of bounds).
__global__ void embed_tokens_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table, long long vocab, const float* __restrict__ pos,
                                    bf16* __restrict__ out, long long ldo, int B, int L, int C) {
  pdl_trigger();
  pdl_wait();
  const int c8n = C >> 3;
  const long long total = (long long)B * L * c8n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % c8n);
    const long long row = i / c8n;
    const int l = (int)(row % L);
    long long id = ids[row];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const float4* t = reinterpret_cast<const float4*>(table + id * C + c8 * 8);
    const float4* p = reinterpret_cast<const float4*>(pos + (long long)l * C + c8 * 8);
    const float4 t0 = __ldg(t), t1 = __ldg(t + 1), p0 = __ldg(p), p1 = __ldg(p + 1);
    uint4 o;
    o.x = pack_bf16x2(t0.x + p0.x, t0.y + p0.y); o.y = pack_bf16x2(t0.z + p0.z, t0.w + p0.w);
    o.z = pack_bf16x2(t1.x + p1.x, t1.y + p1.y); o.w = pack_bf16x2(t1.z + p1.z, t1.w + p1.w);
    *reinterpret_cast<uint4*>(out + row * ldo + c8 * 8) = o;
  }
}

// ---- image-tower input rows (transformers CLIPVisionEmbeddings + pre_layrnorm); one warp per output row -------------------
// row n*(P+1) + 0 is LN(cls + pos[0]), row n*(P+1) + 1 + p is LN(patch[n*P + p] + pos[1 + p]); the add is fp32 and the statistics
// are two-pass fp32 in registers (as layernorm_rows_kernel), bf16 out.
__global__ void __launch_bounds__(256) clip_vision_embed_kernel(const float* __restrict__ patch, long long ldp, const float* __restrict__ cls,
                                                                const float* __restrict__ pos, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, bf16* __restrict__ x, long long ldx,
                                                                int N, int P, int C, float eps) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= (long long)N * (P + 1)) return;
  const int t = (int)(row % (P + 1));
  const long long n = row / (P + 1);
  const float* src = t == 0 ? cls : patch + (n * P + t - 1) * ldp;
  const float* pr = pos + (long long)t * C;
  const int c8n = C >> 3;
  float v[LNR_MAX_CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < c8n) {
      const float4 a0 = *reinterpret_cast<const float4*>(src + c8 * 8), a1 = *reinterpret_cast<const float4*>(src + c8 * 8 + 4);
      const float4 p0 = __ldg(reinterpret_cast<const float4*>(pr + c8 * 8)), p1 = __ldg(reinterpret_cast<const float4*>(pr + c8 * 8 + 4));
      v[i][0] = a0.x + p0.x; v[i][1] = a0.y + p0.y; v[i][2] = a0.z + p0.z; v[i][3] = a0.w + p0.w;
      v[i][4] = a1.x + p1.x; v[i][5] = a1.y + p1.y; v[i][6] = a1.z + p1.z; v[i][7] = a1.w + p1.w;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    if (lane + 32 * i < c8n) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q = fmaf(d, d, q); }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < LNR_MAX_CHUNKS; ++i) {
    const int c8 = lane + 32 * i;
    if (c8 < c8n) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf((v[i][j] - mean) * rstd, __ldg(gamma + c8 * 8 + j), __ldg(beta + c8 * 8 + j));
      uint4 u;
      u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]); u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(x + row * ldx + c8 * 8) = u;
    }
  }
}

// ---- image-tower head, one CTA per image, fp32 on CUDA cores (transformers CLIPVisionTransformer pooling + visual_projection,
// then GLIGEN's reprojection).  Every reduction has a fixed order for a fixed blockDim, so results are bit-reproducible.
constexpr int HEAD_THREADS = 256;
__device__ __forceinline__ float head_block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                  // red[] may still be read by the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < HEAD_THREADS / 32; ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(HEAD_THREADS) clip_image_head_kernel(const bf16* __restrict__ x, long long x_batch,
                                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                       const float* __restrict__ wproj, const float* __restrict__ proj,
                                                                       float target_norm, float* __restrict__ pooled, float* __restrict__ embeds,
                                                                       float* __restrict__ feature, int C, int D, float eps) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float head_smem[];
  float* y = head_smem;                             // [C]  post_layernorm(CLS row)
  float* e = head_smem + C;                         // [D]  image_embeds
  __shared__ float red[HEAD_THREADS / 32];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bf16* xr = x + (long long)n * x_batch;      // the CLS token is row 0 of image n
  float s = 0.f;
  for (int c = tid; c < C; c += HEAD_THREADS) { const float v = __bfloat162float(xr[c]); y[c] = v; s += v; }
  const float mean = head_block_sum(s, red) / (float)C;
  float q = 0.f;
  for (int c = tid; c < C; c += HEAD_THREADS) { const float d = y[c] - mean; q = fmaf(d, d, q); }
  const float rstd = rsqrtf(head_block_sum(q, red) / (float)C + eps);
  for (int c = tid; c < C; c += HEAD_THREADS) {
    const float v = fmaf((y[c] - mean) * rstd, gamma[c], beta[c]);
    y[c] = v;
    pooled[(long long)n * C + c] = v;
  }
  __syncthreads();
  // image_embeds[d] = y . wproj[d, :]: one warp per output, lanes stride the row (coalesced), butterfly sum
  for (int d = warp; d < D; d += HEAD_THREADS / 32) {
    const float* wr = wproj + (long long)d * C;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(y[c], __ldg(wr + c), a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) { e[d] = a; embeds[(long long)n * D + d] = a; }
  }
  if (proj == nullptr) return;
  __syncthreads();
  // f[j] = sum_d e[d] proj[d, j]: one thread per output column (coalesced rows of proj), sequential over d
  float* f = feature + (long long)n * D;
  float sq = 0.f;
  for (int j = tid; j < D; j += HEAD_THREADS) {
    float a = 0.f;
    for (int d = 0; d < D; ++d) a = fmaf(e[d], __ldg(proj + (long long)d * D + j), a);
    f[j] = a;
    sq = fmaf(a, a, sq);
  }
  const float scale = target_norm / sqrtf(head_block_sum(sq, red));
  for (int j = tid; j < D; j += HEAD_THREADS) f[j] *= scale;   // each thread rescales the columns it wrote
}

}  // namespace glg

using namespace glg;
#define ST reinterpret_cast<cudaStream_t>(stream)

extern "C" int glg_spatial_tokens(const void* x, int64_t ldx, const float* mask, const float* null_feat, const float* pos, void* y, int64_t ldy,
                                  int32_t B, int32_t n, int32_t C, void* stream) {
  if (C % 8 || ldx % 8 || ldy % 8 || (((uintptr_t)x | (uintptr_t)y) & 15)) return set_error("glg_spatial_tokens: C, ldx, ldy must be multiples of 8, pointers 16-byte aligned");
  const long long total = (long long)B * n * (C / 8);
  if (total <= 0) return 0;
  launch_k(spatial_tokens_kernel, dim3(fe_blocks(total, 256)), dim3(256), 0, ST, 1, (const bf16*)x, (long long)ldx, mask, null_feat, pos, (bf16*)y, (long long)ldy, B, n, C);
  count_launch();
  return check_launch("spatial_tokens launch");
}

extern "C" int glg_patchify_nchw(const float* x, void* out, int64_t ldo, int32_t B, int32_t C, int32_t Hs, int32_t Ws, int32_t Hv, int32_t Wv,
                                 int32_t k, void* stream) {
  if (k <= 0 || Hv % k || Wv % k) return set_error("glg_patchify_nchw: the (virtual) grid must be a multiple of the patch size");
  if (ldo < (int64_t)k * k * C) return set_error("glg_patchify_nchw: ldo < k*k*C");
  const long long total = (long long)B * (Hv / k) * (Wv / k) * ldo;
  launch_k(patchify_nchw_kernel, dim3(fe_blocks(total, 256)), dim3(256), 0, ST, 1, x, (bf16*)out, (long long)ldo, B, C, Hs, Ws, Hv, Wv, k);
  count_launch();
  return check_launch("patchify_nchw launch");
}

extern "C" int glg_patchify_nhwc(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t k,
                                 void* stream) {
  if (k <= 0 || H % k || Wd % k) return set_error("glg_patchify_nhwc: H, W must be multiples of the patch size");
  if (C % 8 || ldx % 8 || ldo % 8 || (((uintptr_t)x | (uintptr_t)out) & 15)) return set_error("glg_patchify_nhwc: C, ldx, ldo must be multiples of 8 and the pointers 16-byte aligned");
  if (ldo < (int64_t)k * k * C) return set_error("glg_patchify_nhwc: ldo < k*k*C");
  const long long total = (long long)B * (H / k) * (Wd / k) * k * k * (C / 8);
  launch_k(patchify_nhwc_kernel, dim3(fe_blocks(total, 256)), dim3(256), 0, ST, 1, (const bf16*)x, (long long)ldx, (bf16*)out, (long long)ldo, B, H, Wd, C, k);
  count_launch();
  return check_launch("patchify_nhwc launch");
}

extern "C" int glg_layernorm_rows(const void* x, int64_t ldx, void* y, int64_t ldy, const float* gamma, const float* beta, int64_t rows,
                                  int32_t C, int32_t Cpad, float eps, void* stream) {
  if (C <= 0 || C % 8 || C > 256 * LNR_MAX_CHUNKS || Cpad % 8 || Cpad < C || Cpad > 256 * LNR_MAX_CHUNKS)
    return set_error("glg_layernorm_rows: C, Cpad must be multiples of 8 with C <= Cpad <= 1024");
  if (ldx % 8 || ldy % 8 || (((uintptr_t)x | (uintptr_t)y) & 15)) return set_error("glg_layernorm_rows: leading dims must be multiples of 8, pointers 16-byte aligned");
  if (rows <= 0) return 0;
  launch_k(layernorm_rows_kernel<false>, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, ST, 1, (const bf16*)x, (long long)ldx, y, (long long)ldy, gamma, beta,
           (long long)rows, C, Cpad, eps);
  count_launch();
  return check_launch("layernorm_rows launch");
}

extern "C" int glg_layernorm_rows_f32(const void* x, int64_t ldx, float* y, int64_t ldy, const float* gamma, const float* beta, int64_t rows,
                                      int32_t C, float eps, void* stream) {
  if (C <= 0 || C % 8 || C > 256 * LNR_MAX_CHUNKS) return set_error("glg_layernorm_rows_f32: C must be a multiple of 8, <= 1024");
  if (ldx % 8 || ldy % 4 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15)) return set_error("glg_layernorm_rows_f32: ldx % 8, ldy % 4, 16-byte aligned pointers");
  if (rows <= 0) return 0;
  launch_k(layernorm_rows_kernel<true>, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, ST, 1, (const bf16*)x, (long long)ldx, (void*)y, (long long)ldy, gamma, beta,
           (long long)rows, C, C, eps);
  count_launch();
  return check_launch("layernorm_rows_f32 launch");
}

extern "C" int glg_embed_tokens(const int64_t* ids, const float* table, int64_t vocab, const float* pos, void* out, int64_t ldo, int32_t B, int32_t L,
                                int32_t C, void* stream) {
  if (C % 8 || ldo % 8 || ((uintptr_t)out & 15) || (((uintptr_t)table | (uintptr_t)pos) & 15)) return set_error("glg_embed_tokens: C, ldo must be multiples of 8, pointers 16-byte aligned");
  const long long total = (long long)B * L * (C / 8);
  if (total <= 0) return 0;
  launch_k(embed_tokens_kernel, dim3(fe_blocks(total, 256)), dim3(256), 0, ST, 1, ids, table, (long long)vocab, pos, (bf16*)out, (long long)ldo, B, L, C);
  count_launch();
  return check_launch("embed_tokens launch");
}

extern "C" int glg_clip_vision_embed(const float* patch, int64_t ldp, const float* cls, const float* pos, const float* gamma, const float* beta,
                                     void* x, int64_t ldx, int32_t N, int32_t P, int32_t C, float eps, void* stream) {
  if (C <= 0 || C % 8 || C > 256 * LNR_MAX_CHUNKS) return set_error("glg_clip_vision_embed: C must be a multiple of 8, <= 1024");
  if (N < 0 || P < 0) return set_error("glg_clip_vision_embed: negative N or P");
  if (ldp % 4 || ldx % 8 || (((uintptr_t)patch | (uintptr_t)cls | (uintptr_t)pos | (uintptr_t)x) & 15))
    return set_error("glg_clip_vision_embed: ldp % 4, ldx % 8, 16-byte aligned pointers");
  const long long rows = (long long)N * (P + 1);
  if (rows == 0) return 0;
  launch_k(clip_vision_embed_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, ST, 1, patch, (long long)ldp, cls, pos, gamma, beta,
           (bf16*)x, (long long)ldx, N, P, C, eps);
  count_launch();
  return check_launch("clip_vision_embed launch");
}

extern "C" int glg_clip_image_head(const void* x, int64_t x_batch, const float* gamma, const float* beta, const float* w_proj, const float* proj,
                                   float target_norm, float* pooled, float* embeds, float* feature, int32_t N, int32_t C, int32_t D, float eps,
                                   void* stream) {
  if (C <= 0 || D <= 0 || C + D > 12288) return set_error("glg_clip_image_head: need C, D > 0 and C + D <= 12288 (48 KiB of shared memory)");
  if ((proj == nullptr) != (feature == nullptr)) return set_error("glg_clip_image_head: proj and feature go together");
  if (N <= 0) return 0;
  launch_k(clip_image_head_kernel, dim3((unsigned)N), dim3(HEAD_THREADS), (size_t)(C + D) * sizeof(float), ST, 1, (const bf16*)x, (long long)x_batch,
           gamma, beta, w_proj, proj, target_norm, pooled, embeds, feature, C, D, eps);
  count_launch();
  return check_launch("clip_image_head launch");
}

extern "C" int glg_dwconv7_ln(const void* x, int64_t ldx, void* y, int64_t ldy, const float* w, const float* bias, const float* gamma,
                              const float* beta, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t Cpad, float eps, void* stream) {
  if (C <= 0 || C % 2 || C > 64 * DW_MAX_PAIRS || Cpad % 2 || Cpad < C || Cpad > 64 * DW_MAX_PAIRS)
    return set_error("glg_dwconv7_ln: C, Cpad must be even with C <= Cpad <= 768");
  if (ldx % 2 || ldy % 2 || (((uintptr_t)x | (uintptr_t)y) & 3) || (((uintptr_t)w | (uintptr_t)bias | (uintptr_t)gamma | (uintptr_t)beta) & 7))
    return set_error("glg_dwconv7_ln: alignment");
  const long long pix = (long long)B * H * Wd;
  launch_k(dwconv7_ln_kernel, dim3((unsigned)((pix + 7) / 8)), dim3(256), 0, ST, 1, (const bf16*)x, (long long)ldx, (bf16*)y, (long long)ldy, w, bias, gamma, beta,
           B, H, Wd, C, Cpad, eps);
  count_launch();
  return check_launch("dwconv7_ln launch");
}

extern "C" int glg_resize_plane(const float* x, int64_t x_batch_stride, float* y, int32_t B, int32_t C, int32_t Hs, int32_t Ws, int32_t Ho, int32_t Wo,
                                int32_t mode, void* stream) {
  if (mode != 0 && mode != 1) return set_error("glg_resize_plane: mode must be 0 (nearest) or 1 (bicubic)");
  const long long total = (long long)B * C * Ho * Wo;
  if (total <= 0) return 0;
  launch_k(resize_plane_kernel, dim3(fe_blocks(total, 256)), dim3(256), 0, ST, 1, x, (long long)x_batch_stride, y, B, C, Hs, Ws, Ho, Wo, mode);
  count_launch();
  return check_launch("resize_plane launch");
}

extern "C" int glg_conv2d_small(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t Cin, int32_t Hs, int32_t Ws, int32_t Hv,
                                int32_t Wv, int32_t Cout, int32_t k, int32_t stride, int32_t pad, int32_t silu, void* stream) {
  if (k <= 0 || stride <= 0 || pad < 0) return set_error("glg_conv2d_small: bad geometry");
  const int Ho = (Hv + 2 * pad - k) / stride + 1, Wo = (Wv + 2 * pad - k) / stride + 1;
  const long long total = (long long)B * Ho * Wo;
  if (total <= 0) return set_error("glg_conv2d_small: empty output");
  const dim3 grid(fe_blocks(total, 128)), block(128);
  switch (Cout) {
    case 3: launch_k(conv2d_small_kernel<3>, grid, block, 0, ST, 1, x, w, bias, y, B, Cin, Hs, Ws, Hv, Wv, k, stride, pad, Ho, Wo, silu); break;
    case 4: launch_k(conv2d_small_kernel<4>, grid, block, 0, ST, 1, x, w, bias, y, B, Cin, Hs, Ws, Hv, Wv, k, stride, pad, Ho, Wo, silu); break;
    case 8: launch_k(conv2d_small_kernel<8>, grid, block, 0, ST, 1, x, w, bias, y, B, Cin, Hs, Ws, Hv, Wv, k, stride, pad, Ho, Wo, silu); break;
    case 16: launch_k(conv2d_small_kernel<16>, grid, block, 0, ST, 1, x, w, bias, y, B, Cin, Hs, Ws, Hv, Wv, k, stride, pad, Ho, Wo, silu); break;
    default: return set_error("glg_conv2d_small: Cout must be 3, 4, 8 or 16");
  }
  count_launch();
  return check_launch("conv2d_small launch");
}
