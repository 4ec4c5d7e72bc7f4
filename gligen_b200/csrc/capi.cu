// C-ABI plumbing: error strings, launch counter.
#include <cuda_runtime.h>
#include <stdlib.h>
#include <atomic>
#include <string>

#include "internal.h"
#include "../../include/gligen_b200.h"

namespace glg {
static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

int set_error(const std::string& msg) {
  g_err = msg;
  return -1;
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(std::string(what) + ": " + cudaGetErrorString(e));
  return 0;
}
int pdl_mode() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("GLG_PDL");
    v = e ? atoi(e) : 0;            // opt-in
  }
  return v;
}
bool pdl_enabled() { return pdl_mode() != 0; }
}  // namespace glg

extern "C" int glg_abi_version(void) { return GLG_ABI_VERSION; }
extern "C" const char* glg_last_error(void) { return glg::g_err.c_str(); }
extern "C" int64_t glg_launch_count(void) { return glg::g_launches.load(); }
extern "C" void glg_reset_launch_count(void) { glg::g_launches.store(0); }
