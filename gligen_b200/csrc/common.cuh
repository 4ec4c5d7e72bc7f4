// Shared device-side helpers for the sm_90a kernels: mbarrier, TMA, wgmma, clusters, small math.
// Everything here is inline PTX written for sm_90a (no CUTLASS dependency).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace glg {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// With GLG_PDL=1 every kernel is launched with cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel
// in the stream may be scheduled (and run its prologue: barrier init, descriptor prefetch) while this
// one drains; pdl_wait() blocks until the previous grid has completed and its memory is visible, so it must precede
// the first access to global data.  Without the launch attribute both are no-ops.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}
// non-suspending poll (mbarrier.test_wait): the thread keeps its issue slot instead of being parked by the hardware
__device__ __forceinline__ uint32_t mbar_test_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Wait with a watchdog: a protocol bug traps (-> cudaErrorLaunchFailure at the next sync) instead of
// hanging the GPU.  The watchdog only runs on the slow path.  VERBOSE = false leaves out the printf: a function call
// between wgmma.mma_async and its wait makes ptxas serialise the warpgroup MMAs.
template <bool VERBOSE = true>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
#pragma unroll 1
  for (int i = 0; i < 256; ++i)           // common case: the phase completes within a few (HW-suspended) polls - no timer read on this path
    if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (true) {
#pragma unroll 1
    for (int i = 0; i < 64; ++i)          // the timer read is slow: keep it off the wake-up path
      if (mbar_try_wait(bar, parity)) return;
    if (globaltimer_ns() - t0 > 4000000000ull) {  // 4 s
      if (VERBOSE) printf("glg: mbarrier timeout block %d thread %d bar %u parity %u\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// Busy-polling wait (no hardware suspend between polls): lowest wake-up latency, at the price of issue slots.  Falls back to the
// suspending wait (with its watchdog) after 4096 polls.
__device__ __forceinline__ void mbar_wait_spin(uint32_t bar, uint32_t parity) {
#pragma unroll 1
  for (int i = 0; i < 4096; ++i)
    if (mbar_test_wait(bar, parity)) return;
  mbar_wait(bar, parity);
}

// One leader lane of a fully converged warp.  The single-thread TMA producer runs the whole warp through its loop and
// predicates the issue on this flag, so the compiler does not wrap every UTMALDG in a loop over "the active lanes".
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ TMA (tiled and im2col tensor maps)
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// im2col mode over (C, W, H, B): the map's pixels-per-column pixels, walked through its bounding box from position (w, h, n) in
// (n, h, w) order, each read at (w + dw, h + dh)
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const void* tmap, uint32_t bar, int c, int w, int h, int n,
                                                   uint16_t dw, uint16_t dh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(dw), "h"(dh)
      : "memory");
}

// ------------------------------------------------------------------ wgmma (sm_90a warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Shared-memory matrix descriptor, K-major operand, 128B swizzle, rows of 64 bf16 (=128 B), 8-row core-matrix groups
// 1024 B apart (SBO); the tile base must be 1024-byte aligned.  Advancing K by 16 elements adds 32 B (= 2 in the
// start-address field) inside the swizzle atom.
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // start address  [0,14)
  d |= (uint64_t)1 << 16;                              // LBO (unused for swizzled K-major) [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;                    // SBO = 1024 B  [32,46)
  d |= (uint64_t)1 << 62;                              // layout type = SWIZZLE_128B [62,64)
  return d;
}

// ------------------------------------------------------------------ clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa_cluster(uint32_t local_addr, uint32_t cta) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(cta));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// TMA load delivered to the same smem offset of every CTA in `mask`; each destination CTA's mbarrier at `bar`'s
// offset receives the bytes it got
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// ------------------------------------------------------------------ math
// exp2 on the FMA / ALU pipes (Cody-Waite split + Taylor cubic on [-0.5, 0.5]: relative error 1.2e-4 mean, 7.9e-4 max at
// |f| = 0.5, against 2e-3 for the bf16 rounding of P; tests/test_exp2_poly_cpu.py): the attention softmax can move a share
// of its exponentials off the MUFU pipe (16 exp2 / clk / SM), which bounds it at small head dims.
__device__ __forceinline__ float ex2_poly3(float x) {
  x = fmaxf(x, -125.0f);
  const float t = x + 12582912.0f;                 // 1.5 * 2^23: round(x) lands in the low mantissa bits
  const float f = x - (t - 12582912.0f);
  float p = fmaf(0.05550411f, f, 0.24022651f);
  p = fmaf(p, f, 0.69314718f);
  p = fmaf(p, f, 1.0f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// x * sigmoid(x); __fdividef: 2 ulp, no IEEE-division slow path (a CALL per element in the epilogues)
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// CLIP's activation (transformers "quick_gelu": x * sigmoid(1.702 x))
__device__ __forceinline__ float quick_gelu_f(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }
// erf(z) ~= z P(z^2) / Q(z^2) on |z| <= 4 (clamped; |erf(4)-1| < 2e-8): own least-squares rational fit,
// max abs error 3.3e-7 in fp32 (checked against scipy.special.erf), branch-free: 11 FMA + 1 rcp.
__device__ __forceinline__ float erf_rational(float z) {
  z = fminf(fmaxf(z, -4.0f), 4.0f);
  const float z2 = z * z;
  float pn = 2.0269792457838776e-06f;
  pn = fmaf(pn, z2, 0.0002861879765987396f);
  pn = fmaf(pn, z2, 0.003845315193757415f);
  pn = fmaf(pn, z2, 0.05298357829451561f);
  pn = fmaf(pn, z2, 0.1923242062330246f);
  pn = fmaf(pn, z2, 1.128378987312317f);
  float qn = 3.7925383367110044e-05f;
  qn = fmaf(qn, z2, 0.0011811800068244338f);
  qn = fmaf(qn, z2, 0.015125652775168419f);
  qn = fmaf(qn, z2, 0.11488588154315948f);
  qn = fmaf(qn, z2, 0.5037747621536255f);
  qn = fmaf(qn, z2, 1.0f);
  return __fdividef(z * pn, qn);
}
// exact (erf) GELU of attention.py:44 (F.gelu default); abs error < 1e-6, far below bf16 resolution
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erf_rational(x * 0.70710678118654752f)); }
// Cheaper erf for the GEGLU epilogue (the FF1 GEMMs are bound by the epilogue's instruction issue, not by the tensor
// pipe: 128 x 128 GELUs per 2560 MMA cycles): z P3(z^2) / Q3(z^2) on |z| <= 3.2 (clamped; 1 - erf(3.2) = 6e-6), own
// least-squares fit: max abs error 3.4e-6 on erf, 1.5e-5 on gelu(x) over all x - three decimal orders below the bf16
// resolution of the stored product.  7 FMA + 1 rcp instead of 11 FMA + 1 rcp.
__device__ __forceinline__ float erf_rational3(float z) {
  z = fminf(fmaxf(z, -3.2f), 3.2f);
  const float z2 = z * z;
  float pn = 0.0007654472137801349f;
  pn = fmaf(pn, z2, 0.04346451908349991f);
  pn = fmaf(pn, z2, 0.15304264426231384f);
  pn = fmaf(pn, z2, 1.1283873319625854f);
  float qn = 0.009417801164090633f;
  qn = fmaf(qn, z2, 0.09465143829584122f);
  qn = fmaf(qn, z2, 0.4690375328063965f);
  qn = fmaf(qn, z2, 1.0f);
  return __fdividef(z * pn, qn);
}
// x * gelu_erf(g) for the GEGLU epilogue: 0.5 g (1 + erf(g / sqrt 2)) as one FMA on h = 0.5 g
__device__ __forceinline__ float geglu_f(float x, float g) {
  const float h = 0.5f * g;
  return x * fmaf(h, erf_rational3(g * 0.70710678118654752f), h);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace glg
