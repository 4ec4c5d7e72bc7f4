// Engine-level C ABI: run a whole UNet forward from an exported plan file, without any Python at run time.
//
// `gligen_b200/export.py` serialises one (batch rows, grounding slots, context length) plan of gligen_b200.engine.Engine:
// the packed weights, the sizes of every workspace buffer, and the ordered list of op-level C-ABI calls with every
// pointer argument expressed as (buffer, byte offset).  This file loads such a plan (allocates the buffers, uploads the
// weights, patches the pointers) and replays it on a stream:
//
//     glg_engine_load(path, &e);
//     glg_engine_buffer(e, "in:x", &p, &n);  cudaMemcpyAsync(p, x, n, ...);      // likewise in:t, in:context, in:coords, ...
//     glg_engine_run(e, /*static part*/ 1, fuser_on, stream);                    // once per prompt / grounding input
//     glg_engine_run(e, /*per-step part*/ 0, fuser_on, stream);                  // every sampler step (CUDA-graph capturable)
//     glg_engine_buffer(e, "out", &p, &n);                                       // eps [rows, 4, H, W] fp32
//
// This is the `gligen_create / gligen_load_tensor / gligen_unet_forward` contract of SURVEY 8(b) in exported-plan form:
// weight packing and plan construction stay in gligen_b200/engine.py (run once, at export); the per-step path is native.
// Replaces UNetModel.forward (openaimodel.py:420-464) for a host that cannot embed Python.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

#include "internal.h"
#include "../../include/gligen_b200.h"

namespace glg {

struct EArg {
  char tag;                       // 'P' pointer, 'I' int64, 'F' float, 'S' struct bytes, 'T' stream
  void* p = nullptr;
  long long i = 0;
  float f = 0.f;
  std::vector<uint8_t> s;
};
struct EOp {
  std::string name;
  uint32_t flags;                 // bit 0: fuser-only, bit 1: static (timestep-invariant)
  std::vector<EArg> args;
};
struct EBuf {
  std::string name;
  void* ptr = nullptr;
  uint64_t bytes = 0;
};

}  // namespace glg

struct GlgEngine {
  std::vector<glg::EBuf> bufs;
  std::vector<glg::EOp> ops;
  std::map<std::string, int> by_name;
};

using namespace glg;

namespace {
struct Reader {
  FILE* f;
  bool ok = true;
  void raw(void* dst, size_t n) { if (ok && fread(dst, 1, n, f) != n) ok = false; }
  uint32_t u32() { uint32_t v = 0; raw(&v, 4); return v; }
  uint64_t u64() { uint64_t v = 0; raw(&v, 8); return v; }
  std::string str(size_t n) { std::vector<char> b(n + 1, 0); raw(b.data(), n); return std::string(b.data()); }
};

void* resolve(const GlgEngine* e, uint32_t buf, uint64_t off) {
  if (buf == 0xFFFFFFFFu) return nullptr;
  return static_cast<uint8_t*>(e->bufs[buf].ptr) + off;
}

#define A_P(k) (a[k].p)
#define A_I(k) (a[k].i)
#define A_I32(k) ((int32_t)a[k].i)
#define A_F(k) (a[k].f)

int dispatch(const EOp& op, void* st) {
  const std::vector<EArg>& a = op.args;
  const std::string& n = op.name;
  if (n == "glg_gemm") return glg_gemm(reinterpret_cast<const GlgGemmArgs*>(a[0].s.data()), st);
  if (n == "glg_attention") return glg_attention(reinterpret_cast<const GlgAttnArgs*>(a[0].s.data()), st);
  if (n == "glg_groupnorm")
    return glg_groupnorm(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), (float*)A_P(6), A_I32(7), A_I32(8), A_I32(9),
                         A_I32(10), A_F(11), A_I32(12), st);
  if (n == "glg_layernorm")
    return glg_layernorm(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), A_I32(6), A_I32(7), A_I32(8), A_F(9), st);
  if (n == "glg_conv_in")
    return glg_conv_in((const float*)A_P(0), A_I32(1), (const float*)A_P(2), A_I32(3), (const float*)A_P(4), (const float*)A_P(5), A_P(6), A_I(7),
                       A_I32(8), A_I32(9), A_I32(10), A_I32(11), st);
  if (n == "glg_conv_out")
    return glg_conv_out(A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (float*)A_P(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), A_I32(9), st);
  if (n == "glg_upsample2x") return glg_upsample2x(A_P(0), A_I(1), A_P(2), A_I(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), st);
  if (n == "glg_im2col_s2") return glg_im2col_s2(A_P(0), A_I(1), A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), st);
  if (n == "glg_im2col_s2_pad") return glg_im2col_s2_pad(A_P(0), A_I(1), A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), st);
  if (n == "glg_timestep_embedding") return glg_timestep_embedding((const int64_t*)A_P(0), A_P(1), A_I32(2), A_I32(3), st);
  if (n == "glg_position_features")
    return glg_position_features((const float*)A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (const float*)A_P(4), (const float*)A_P(5),
                                 (const float*)A_P(6), A_P(7), A_I(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12), A_I32(13), st);
  if (n == "glg_cast_f32_bf16") return glg_cast_f32_bf16((const float*)A_P(0), A_P(1), A_I(2), st);
  if (n == "glg_softmax_rows") return glg_softmax_rows((const float*)A_P(0), A_I(1), A_P(2), A_I(3), A_I(4), A_I32(5), A_F(6), st);
  if (n == "glg_copy_rows") return glg_copy_rows(A_P(0), A_I(1), A_P(2), A_I(3), A_I(4), A_I32(5), st);
  // spatial grounding modalities: ConvNeXt tokenizer + grounding downsampler steps (static part of the plan)
  if (n == "glg_patchify_nchw")
    return glg_patchify_nchw((const float*)A_P(0), A_P(1), A_I(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), A_I32(9), st);
  if (n == "glg_patchify_nhwc") return glg_patchify_nhwc(A_P(0), A_I(1), A_P(2), A_I(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), st);
  if (n == "glg_layernorm_rows")
    return glg_layernorm_rows(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), A_I(6), A_I32(7), A_I32(8), A_F(9), st);
  if (n == "glg_dwconv7_ln")
    return glg_dwconv7_ln(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), (const float*)A_P(6), (const float*)A_P(7),
                          A_I32(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12), A_F(13), st);
  if (n == "glg_spatial_tokens")
    return glg_spatial_tokens(A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (const float*)A_P(4), A_P(5), A_I(6), A_I32(7), A_I32(8),
                              A_I32(9), st);
  if (n == "glg_resize_plane")
    return glg_resize_plane((const float*)A_P(0), A_I(1), (float*)A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), A_I32(9), st);
  if (n == "glg_conv2d_small")
    return glg_conv2d_small((const float*)A_P(0), (const float*)A_P(1), (const float*)A_P(2), (float*)A_P(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7),
                            A_I32(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12), A_I32(13), A_I32(14), st);
  // gatedSA2 fuser: the resampled, gated residual of the grounding rows (per step)
  if (n == "glg_grid_resample_gate")
    return glg_grid_resample_gate((const float*)A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (float*)A_P(5), A_I(6), A_I32(7), A_I32(8),
                                  A_I32(9), A_I32(10), st);
  return set_error("glg_engine_run: unknown op '" + n + "' in the plan");
}
}  // namespace

extern "C" int glg_engine_destroy(GlgEngine* e) {
  if (!e) return 0;
  for (auto& b : e->bufs)
    if (b.ptr) cudaFree(b.ptr);
  delete e;
  return 0;
}

extern "C" int glg_engine_load(const char* path, GlgEngine** out) {
  if (!path || !out) return set_error("glg_engine_load: null argument");
  FILE* f = fopen(path, "rb");
  if (!f) return set_error(std::string("glg_engine_load: cannot open ") + path);
  Reader r{f};
  char magic[8];
  r.raw(magic, 8);
  if (!r.ok || memcmp(magic, "GLGPLAN1", 8)) { fclose(f); return set_error("glg_engine_load: not a GLGPLAN1 file"); }
  if (r.u32() != (uint32_t)GLG_ABI_VERSION) { fclose(f); return set_error("glg_engine_load: plan was exported for another ABI version"); }
  GlgEngine* e = new GlgEngine();
  const uint32_t nb = r.u32();
  std::vector<uint8_t> stage;
  for (uint32_t i = 0; i < nb && r.ok; ++i) {
    EBuf b;
    b.bytes = r.u64();
    const uint32_t has_data = r.u32();
    b.name = r.str(48);
    const size_t alloc = b.bytes < 256 ? 256 : (size_t)b.bytes;
    if (cudaMalloc(&b.ptr, alloc) != cudaSuccess) { fclose(f); glg_engine_destroy(e); return set_error("glg_engine_load: cudaMalloc failed for buffer " + b.name); }
    cudaMemset(b.ptr, 0, alloc);                      // workspace starts zeroed (GroupNorm barrier counters rely on it)
    if (has_data) {
      stage.resize((size_t)b.bytes);
      r.raw(stage.data(), (size_t)b.bytes);
      if (r.ok) cudaMemcpy(b.ptr, stage.data(), (size_t)b.bytes, cudaMemcpyHostToDevice);
    }
    e->by_name[b.name] = (int)e->bufs.size();
    e->bufs.push_back(b);
  }
  const uint32_t no = r.u32();
  for (uint32_t i = 0; i < no && r.ok; ++i) {
    EOp op;
    op.name = r.str(32);
    op.flags = r.u32();
    const uint32_t na = r.u32();
    for (uint32_t k = 0; k < na && r.ok; ++k) {
      EArg a;
      r.raw(&a.tag, 1);
      if (a.tag == 'P') { const uint32_t b = r.u32(); const uint64_t off = r.u64(); if (b != 0xFFFFFFFFu && b >= e->bufs.size()) r.ok = false; else a.p = resolve(e, b, off); }
      else if (a.tag == 'I') { uint64_t v = r.u64(); memcpy(&a.i, &v, 8); }
      else if (a.tag == 'F') { uint32_t v = r.u32(); memcpy(&a.f, &v, 4); }
      else if (a.tag == 'T') { }
      else if (a.tag == 'S') {
        const uint32_t nbytes = r.u32();
        a.s.resize(nbytes);
        r.raw(a.s.data(), nbytes);
        const uint32_t nfix = r.u32();
        for (uint32_t x = 0; x < nfix && r.ok; ++x) {
          const uint32_t field = r.u32(), b = r.u32();
          const uint64_t off = r.u64();
          if (field + 8 > nbytes || (b != 0xFFFFFFFFu && b >= e->bufs.size())) { r.ok = false; break; }
          void* p = resolve(e, b, off);
          memcpy(a.s.data() + field, &p, 8);
        }
      } else r.ok = false;
      op.args.push_back(std::move(a));
    }
    e->ops.push_back(std::move(op));
  }
  fclose(f);
  if (!r.ok) { glg_engine_destroy(e); return set_error("glg_engine_load: truncated or corrupt plan file"); }
  cudaDeviceSynchronize();
  *out = e;
  return 0;
}

extern "C" int glg_engine_buffer(GlgEngine* e, const char* name, void** ptr, int64_t* bytes) {
  if (!e || !name) return set_error("glg_engine_buffer: null argument");
  auto it = e->by_name.find(name);
  if (it == e->by_name.end()) return set_error(std::string("glg_engine_buffer: no buffer named ") + name);
  if (ptr) *ptr = e->bufs[it->second].ptr;
  if (bytes) *bytes = (int64_t)e->bufs[it->second].bytes;
  return 0;
}

// copies between caller memory (host or device: cudaMemcpyDefault) and a named buffer, ordered on `stream`
extern "C" int glg_engine_write(GlgEngine* e, const char* name, const void* src, int64_t bytes, void* stream) {
  void* dst = nullptr; int64_t n = 0;
  if (glg_engine_buffer(e, name, &dst, &n)) return -1;
  if (bytes > n) return set_error(std::string("glg_engine_write: ") + name + " is smaller than the source");
  cudaError_t err = cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, reinterpret_cast<cudaStream_t>(stream));
  return err == cudaSuccess ? 0 : set_error(std::string("glg_engine_write: ") + cudaGetErrorString(err));
}
extern "C" int glg_engine_read(GlgEngine* e, const char* name, void* dst, int64_t bytes, void* stream) {
  void* src = nullptr; int64_t n = 0;
  if (glg_engine_buffer(e, name, &src, &n)) return -1;
  if (bytes > n) return set_error(std::string("glg_engine_read: ") + name + " is smaller than the destination");
  cudaError_t err = cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, reinterpret_cast<cudaStream_t>(stream));
  return err == cudaSuccess ? 0 : set_error(std::string("glg_engine_read: ") + cudaGetErrorString(err));
}

// static_part = 1: the timestep-invariant ops (PositionNet, text K/V, grounding K/V) - run when the prompt / grounding input
// changes; 0: everything else - run every step.  fuser_on = 0 skips the gated self-attention ops (scale == 0).
extern "C" int glg_engine_run(GlgEngine* e, int32_t static_part, int32_t fuser_on, void* stream) {
  if (!e) return set_error("glg_engine_run: null engine");
  for (const EOp& op : e->ops) {
    const bool fuser = op.flags & 1u, stat = (op.flags & 2u) != 0;
    if (stat != (static_part != 0)) continue;
    if (fuser && !fuser_on && !stat) continue;
    const int rc = dispatch(op, stream);
    if (rc) return rc;
  }
  return 0;
}

extern "C" int64_t glg_engine_num_ops(GlgEngine* e) { return e ? (int64_t)e->ops.size() : -1; }
