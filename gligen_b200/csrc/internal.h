// Library-internal helpers shared by the translation units of libgligen_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>

namespace glg {
// records a thread-local error message and returns -1
int set_error(const std::string& msg);
void count_launch();
// returns 0 or records the error
int check_launch(const char* what);
// bf16 tiled tensor map with 128B swizzle and zero out-of-bounds fill (host-side cache keyed by all
// arguments).  dims/box innermost first; strides in BYTES for dims 1..rank-1.  Returns 0 or records the error.
int get_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides, const uint32_t* box);
// swizzle_bytes: 0 (none), 64 or 128; rank 1..5
int get_tmap_bf16_sw(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides, const uint32_t* box, int swizzle_bytes);
int num_sms();
bool pdl_enabled();     // GLG_PDL env (default off)
int pdl_mode();         // 0 off, 1 every launch, 2 only launches whose grid leaves SMs idle (fewer CTAs than SMs): their prologue
                        // (launch latency, barrier init) overlaps the tail of the kernel before them

// Launch with programmatic dependent launch (and optionally a thread-block cluster along x).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  const int pm = pdl_mode();
  if (pm == 1 || (pm == 2 && (long long)grid.x * grid.y * grid.z < (long long)num_sms())) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
}  // namespace glg
