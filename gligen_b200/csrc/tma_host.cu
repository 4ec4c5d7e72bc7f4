// Host-side CUtensorMap cache (bf16, zero OOB fill; tiled and im2col maps) shared by the GEMM/conv and attention launchers.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <mutex>
#include <unordered_map>
#include <string>

#include "internal.h"

namespace glg {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                     CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void* driver_entry(const char* name) {
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess) return ptr;
  return nullptr;
}
static PFN_encodeTiled get_encode_fn() {
  static const PFN_encodeTiled fn = reinterpret_cast<PFN_encodeTiled>(driver_entry("cuTensorMapEncodeTiled"));
  return fn;
}
static PFN_encodeIm2col get_encode_im2col_fn() {
  static const PFN_encodeIm2col fn = reinterpret_cast<PFN_encodeIm2col>(driver_entry("cuTensorMapEncodeIm2col"));
  return fn;
}

enum TmapKind { kTiled = 0, kIm2col3x3 = 1 };
struct TmapKey {
  const void* ptr; uint64_t d[5]; uint64_t s[4]; uint32_t box[5]; int rank; int swizzle; int kind;
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) { h ^= w[i]; h *= 1099511628211ull; }
    return h;
  }
};
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmaps;
static std::mutex g_tmap_mu;

// bf16 tensor map, 128B swizzle, zero OOB fill.  dims/strides innermost first; strides in bytes (rank-1 of them).
int get_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides,
                  const uint32_t* box) {
  return get_tmap_bf16_sw(out, ptr, rank, dims, strides, box, 128);
}

// same with the swizzle width chosen by the caller (0: none, 64 or 128 bytes); rank up to 5
int get_tmap_bf16_sw(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box, int swizzle_bytes) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = ptr; key.rank = rank; key.swizzle = swizzle_bytes;
  for (int i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.box[i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) key.s[i] = strides[i];
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  auto it = g_tmaps.find(key);
  if (it != g_tmaps.end()) { *out = it->second; return 0; }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if (rank < 1 || rank > 5) return set_error("tensor map rank must be 1..5");
  cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides[i];
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 0 ? CU_TENSOR_MAP_SWIZZLE_NONE : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu stride0 %llu box %u %u %u %u ptr %p",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
             (unsigned long long)(rank > 1 ? strides[0] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
             rank > 3 ? box[3] : 0, ptr);
    return set_error(buf);
  }
  if (g_tmaps.size() >= 8192) g_tmaps.clear();     // callers that pass ever-new buffers must not grow the cache without bound
  g_tmaps.emplace(key, m);
  *out = m;
  return 0;
}

// im2col tensor map of a 3x3 / pad 1 / stride 1 convolution over an NHWC activation, dims (C, W, H, B).  The bounding box
// runs from -1 to W-2 (H-2) in each spatial dim: one position per output pixel, at the input pixel of its tap (0, 0).  A load
// at start (c, x-1, y-1, b) with im2col offsets (dx, dy) fills `pixels` smem rows of `channels` (128-byte, swizzled) with
// the input of tap (dy, dx) for `pixels` consecutive output pixels in (b, y, x) order, crossing row and image boundaries;
// padding and pixels past the last image read as zeros.
int get_tmap_bf16_im2col3x3(CUtensorMap* out, const void* ptr, const uint64_t* dims, const uint64_t* strides, uint32_t channels,
                            uint32_t pixels) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = ptr; key.rank = 4; key.swizzle = 128; key.kind = kIm2col3x3;
  for (int i = 0; i < 4; ++i) key.d[i] = dims[i];
  for (int i = 0; i < 3; ++i) key.s[i] = strides[i];
  key.box[0] = channels; key.box[1] = pixels;
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  auto it = g_tmaps.find(key);
  if (it != g_tmaps.end()) { *out = it->second; return 0; }
  PFN_encodeIm2col enc = get_encode_im2col_fn();
  if (!enc) return set_error("cuTensorMapEncodeIm2col entry point unavailable (no CUDA driver?)");
  cuuint64_t gd[4]; cuuint64_t gs[3];
  for (int i = 0; i < 4; ++i) gd[i] = dims[i];
  for (int i = 0; i < 3; ++i) gs[i] = strides[i];
  const int lower[2] = {-1, -1}, upper[2] = {-1, -1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), gd, gs, lower, upper, channels, pixels, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeIm2col failed (%d): dims %llu %llu %llu %llu stride0 %llu channels %u pixels %u ptr %p",
             (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
             (unsigned long long)strides[0], channels, pixels, ptr);
    return set_error(buf);
  }
  if (g_tmaps.size() >= 8192) g_tmaps.clear();
  g_tmaps.emplace(key, m);
  *out = m;
  return 0;
}

static int g_num_sms = 0;
int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}


}  // namespace glg
