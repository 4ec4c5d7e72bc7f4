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
//
// A plan file comes from outside the library (it may be truncated, stale or edited), so glg_engine_load checks every op
// against the table of calls below - name, argument count, argument tags, struct sizes, pointer (buffer, offset) ranges -
// before it allocates anything, and refuses the whole plan on the first mismatch.  glg_engine_run only replays checked ops.
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

constexpr uint32_t kNullBuf = 0xFFFFFFFFu;   // pointer argument that is NULL

struct Fixup {
  uint32_t at;                    // 'S': byte offset of the pointer field in the struct ('P': unused)
  uint32_t buf;                   // buffer index or kNullBuf
  uint64_t off;                   // byte offset into that buffer
};
struct EArg {
  char tag;                       // 'P' pointer, 'I' int64, 'F' float, 'S' struct bytes, 'T' stream
  void* p = nullptr;
  long long i = 0;
  float f = 0.f;
  std::vector<uint8_t> s;
  std::vector<Fixup> fix;         // 'P': the one pointer, 'S': its pointer fields; patched once the buffers are allocated
};
// One op-level call a plan may contain.  `tags` has one letter per parameter of its declaration in include/gligen_b200.h, as
// gligen_b200/export.py writes it: 'P' pointer, 'I' integer (any width), 'F' float, 'S' struct passed by pointer (of `sbytes`
// bytes), 'T' the trailing stream.
struct OpDef {
  const char* name;
  const char* tags;
  size_t sbytes;
  int (*run)(const EArg* a, void* st);
};
struct EOp {
  const OpDef* def;
  uint32_t flags;                 // bit 0: fuser-only, bit 1: static (timestep-invariant)
  std::vector<EArg> args;
};
struct EBuf {
  std::string name;
  void* ptr = nullptr;
  uint64_t bytes = 0;
  int64_t file_at = -1;           // where the contents start in the plan file; -1: workspace (zero-filled)
};

}  // namespace glg

struct GlgEngine {
  std::vector<glg::EBuf> bufs;
  std::vector<glg::EOp> ops;
  std::map<std::string, int> by_name;
};

using namespace glg;

namespace {

#define A_P(k) (a[k].p)
#define A_I(k) (a[k].i)
#define A_I32(k) ((int32_t)a[k].i)
#define A_F(k) (a[k].f)
#define CALL(...) [](const EArg* a, void* st) -> int { return __VA_ARGS__; }

// every call glg_engine_load accepts in a plan (tests/test_abi_cpu.py checks the tags against the header's declarations)
const OpDef kOps[] = {
    {"glg_gemm", "ST", sizeof(GlgGemmArgs), CALL(glg_gemm(reinterpret_cast<const GlgGemmArgs*>(a[0].s.data()), st))},
    {"glg_attention", "ST", sizeof(GlgAttnArgs), CALL(glg_attention(reinterpret_cast<const GlgAttnArgs*>(a[0].s.data()), st))},
    {"glg_groupnorm", "PIPIPPPIIIIFIT", 0,
     CALL(glg_groupnorm(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), (float*)A_P(6), A_I32(7), A_I32(8),
                        A_I32(9), A_I32(10), A_F(11), A_I32(12), st))},
    {"glg_layernorm", "PIPIPPIIIFT", 0,
     CALL(glg_layernorm(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), A_I32(6), A_I32(7), A_I32(8), A_F(9), st))},
    {"glg_conv_in", "PIPIPPPIIIIIT", 0,
     CALL(glg_conv_in((const float*)A_P(0), A_I32(1), (const float*)A_P(2), A_I32(3), (const float*)A_P(4), (const float*)A_P(5), A_P(6), A_I(7),
                      A_I32(8), A_I32(9), A_I32(10), A_I32(11), st))},
    {"glg_conv_out", "PIPPPIIIIIT", 0,
     CALL(glg_conv_out(A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (float*)A_P(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8),
                       A_I32(9), st))},
    {"glg_upsample2x", "PIPIIIIIT", 0, CALL(glg_upsample2x(A_P(0), A_I(1), A_P(2), A_I(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), st))},
    {"glg_im2col_s2", "PIPIIIIT", 0, CALL(glg_im2col_s2(A_P(0), A_I(1), A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), st))},
    {"glg_im2col_s2_pad", "PIPIIIIIT", 0, CALL(glg_im2col_s2_pad(A_P(0), A_I(1), A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), st))},
    {"glg_timestep_embedding", "PPIIT", 0, CALL(glg_timestep_embedding((const int64_t*)A_P(0), A_P(1), A_I32(2), A_I32(3), st))},
    {"glg_timestep_embedding_f32", "PPIIT", 0, CALL(glg_timestep_embedding_f32((const float*)A_P(0), A_P(1), A_I32(2), A_I32(3), st))},
    {"glg_position_features", "PIPPPPPPIIIIIIT", 0,
     CALL(glg_position_features((const float*)A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (const float*)A_P(4),
                                (const float*)A_P(5), (const float*)A_P(6), A_P(7), A_I(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12),
                                A_I32(13), st))},
    {"glg_cast_f32_bf16", "PPIT", 0, CALL(glg_cast_f32_bf16((const float*)A_P(0), A_P(1), A_I(2), st))},
    {"glg_softmax_rows", "PIPIIIFT", 0, CALL(glg_softmax_rows((const float*)A_P(0), A_I(1), A_P(2), A_I(3), A_I(4), A_I32(5), A_F(6), st))},
    {"glg_copy_rows", "PIPIIIT", 0, CALL(glg_copy_rows(A_P(0), A_I(1), A_P(2), A_I(3), A_I(4), A_I32(5), st))},
    // spatial grounding modalities: ConvNeXt tokenizer + grounding downsampler steps (static part of the plan)
    {"glg_patchify_nchw", "PPIIIIIIIIT", 0,
     CALL(glg_patchify_nchw((const float*)A_P(0), A_P(1), A_I(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), A_I32(9), st))},
    {"glg_patchify_nhwc", "PIPIIIIIIT", 0,
     CALL(glg_patchify_nhwc(A_P(0), A_I(1), A_P(2), A_I(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), st))},
    {"glg_layernorm_rows", "PIPIPPIIIFT", 0,
     CALL(glg_layernorm_rows(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), A_I(6), A_I32(7), A_I32(8), A_F(9),
                             st))},
    {"glg_dwconv7_ln", "PIPIPPPPIIIIIFT", 0,
     CALL(glg_dwconv7_ln(A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (const float*)A_P(5), (const float*)A_P(6),
                         (const float*)A_P(7), A_I32(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12), A_F(13), st))},
    {"glg_spatial_tokens", "PIPPPPIIIIT", 0,
     CALL(glg_spatial_tokens(A_P(0), A_I(1), (const float*)A_P(2), (const float*)A_P(3), (const float*)A_P(4), A_P(5), A_I(6), A_I32(7),
                             A_I32(8), A_I32(9), st))},
    {"glg_resize_plane", "PIPIIIIIIIT", 0,
     CALL(glg_resize_plane((const float*)A_P(0), A_I(1), (float*)A_P(2), A_I32(3), A_I32(4), A_I32(5), A_I32(6), A_I32(7), A_I32(8), A_I32(9),
                           st))},
    {"glg_conv2d_small", "PPPPIIIIIIIIIIIT", 0,
     CALL(glg_conv2d_small((const float*)A_P(0), (const float*)A_P(1), (const float*)A_P(2), (float*)A_P(3), A_I32(4), A_I32(5), A_I32(6),
                           A_I32(7), A_I32(8), A_I32(9), A_I32(10), A_I32(11), A_I32(12), A_I32(13), A_I32(14), st))},
    // gatedSA2 fuser: the resampled, gated residual of the grounding rows (per step)
    {"glg_grid_resample_gate", "PIPIPPIIIIIT", 0,
     CALL(glg_grid_resample_gate((const float*)A_P(0), A_I(1), A_P(2), A_I(3), (const float*)A_P(4), (float*)A_P(5), A_I(6), A_I32(7),
                                 A_I32(8), A_I32(9), A_I32(10), st))},
};

const OpDef* find_op(const std::string& name) {
  for (const OpDef& d : kOps)
    if (name == d.name) return &d;
  return nullptr;
}

struct Reader {
  FILE* f;
  bool ok = true;
  void raw(void* dst, size_t n) { if (ok && fread(dst, 1, n, f) != n) ok = false; }
  uint32_t u32() { uint32_t v = 0; raw(&v, 4); return v; }
  uint64_t u64() { uint64_t v = 0; raw(&v, 8); return v; }
  std::string str(size_t n) { std::vector<char> b(n + 1, 0); raw(b.data(), n); return std::string(b.data()); }
  void skip(uint64_t n) { if (ok && fseeko(f, (off_t)n, SEEK_CUR) != 0) ok = false; }
};

// "" when (buf, off) names a byte inside a buffer of the plan (or buf is kNullBuf), else what is wrong
std::string check_ptr(const std::vector<EBuf>& bufs, uint32_t buf, uint64_t off) {
  if (buf == kNullBuf) return "";
  if (buf >= bufs.size()) return "names buffer " + std::to_string(buf) + ", but the plan has " + std::to_string(bufs.size());
  if (off >= bufs[buf].bytes)
    return "points at byte " + std::to_string(off) + " of buffer '" + bufs[buf].name + "', which holds " + std::to_string(bufs[buf].bytes);
  return "";
}

// Reads one op and checks it against its table entry: "" or what is wrong (r.ok = false: the file ended first).
std::string read_op(Reader& r, const std::vector<EBuf>& bufs, EOp& op) {
  const std::string name = r.str(32);
  op.flags = r.u32();
  const uint32_t na = r.u32();
  if (!r.ok) return "";
  op.def = find_op(name);
  if (!op.def) return "unknown op '" + name + "'";
  const std::string where = name + " ";
  if (na != strlen(op.def->tags))
    return where + "has " + std::to_string(na) + " arguments, expected " + std::to_string(strlen(op.def->tags));
  for (uint32_t k = 0; k < na && r.ok; ++k) {
    EArg a;
    r.raw(&a.tag, 1);
    if (!r.ok) return "";
    const std::string arg = where + "argument " + std::to_string(k) + " ";
    if (a.tag != op.def->tags[k])
      return arg + "is tagged '" + std::string(1, a.tag) + "', expected '" + std::string(1, op.def->tags[k]) + "'";
    if (a.tag == 'P') {
      const uint32_t b = r.u32();
      const uint64_t off = r.u64();
      const std::string bad = r.ok ? check_ptr(bufs, b, off) : "";
      if (!bad.empty()) return arg + bad;
      a.fix.push_back({0, b, off});
    } else if (a.tag == 'I') {
      const uint64_t v = r.u64();
      memcpy(&a.i, &v, 8);
    } else if (a.tag == 'F') {
      const uint32_t v = r.u32();
      memcpy(&a.f, &v, 4);
    } else if (a.tag == 'S') {
      const uint32_t nbytes = r.u32();
      if (!r.ok) return "";
      if (nbytes != op.def->sbytes)
        return arg + "holds " + std::to_string(nbytes) + " bytes, expected " + std::to_string(op.def->sbytes);
      a.s.resize(nbytes);
      r.raw(a.s.data(), nbytes);
      const uint32_t nfix = r.u32();
      for (uint32_t x = 0; x < nfix && r.ok; ++x) {
        const uint32_t field = r.u32(), b = r.u32();
        const uint64_t off = r.u64();
        if (!r.ok) return "";
        if ((uint64_t)field + 8 > nbytes) return arg + "has a pointer at byte " + std::to_string(field) + ", past its end";
        const std::string bad = check_ptr(bufs, b, off);
        if (!bad.empty()) return arg + "field at byte " + std::to_string(field) + " " + bad;
        a.fix.push_back({field, b, off});
      }
    }
    op.args.push_back(std::move(a));
  }
  return "";
}

void* resolve(const GlgEngine* e, const Fixup& x) {
  return x.buf == kNullBuf ? nullptr : static_cast<uint8_t*>(e->bufs[x.buf].ptr) + x.off;
}

// First pass: the buffer table (contents skipped) and every op, checked.  "" or the reason to refuse the plan.
std::string read_plan(Reader& r, GlgEngine* e) {
  char magic[8];
  r.raw(magic, 8);
  if (!r.ok || memcmp(magic, "GLGPLAN1", 8)) return "not a GLGPLAN1 file";
  if (r.u32() != (uint32_t)GLG_ABI_VERSION) return r.ok ? "plan was exported for another ABI version" : "truncated or corrupt plan file";
  const uint32_t nb = r.u32();
  for (uint32_t i = 0; i < nb && r.ok; ++i) {
    EBuf b;
    b.bytes = r.u64();
    const uint32_t has_data = r.u32();
    b.name = r.str(48);
    if (has_data) {
      b.file_at = (int64_t)ftello(r.f);
      r.skip(b.bytes);
    }
    e->by_name[b.name] = (int)e->bufs.size();
    e->bufs.push_back(b);
  }
  const uint32_t no = r.u32();
  for (uint32_t i = 0; i < no && r.ok; ++i) {
    EOp op;
    const std::string bad = read_op(r, e->bufs, op);
    if (!bad.empty()) return "op " + std::to_string(i) + ": " + bad;
    e->ops.push_back(std::move(op));
  }
  return r.ok ? "" : "truncated or corrupt plan file";
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
  GlgEngine* e = new GlgEngine();
  const std::string bad = read_plan(r, e);
  if (!bad.empty()) { fclose(f); glg_engine_destroy(e); return set_error("glg_engine_load: " + bad); }
  // second pass: allocate every buffer, upload the contents of the weight buffers, patch the pointers
  std::vector<uint8_t> stage;
  for (EBuf& b : e->bufs) {
    const size_t alloc = b.bytes < 256 ? 256 : (size_t)b.bytes;
    if (cudaMalloc(&b.ptr, alloc) != cudaSuccess) {
      const std::string msg = "glg_engine_load: cudaMalloc failed for buffer " + b.name;
      fclose(f);
      glg_engine_destroy(e);
      return set_error(msg);
    }
    cudaMemset(b.ptr, 0, alloc);                      // workspace starts zeroed (GroupNorm barrier counters rely on it)
    if (b.file_at >= 0) {
      stage.resize((size_t)b.bytes);
      if (fseeko(f, (off_t)b.file_at, SEEK_SET) != 0) r.ok = false;
      r.raw(stage.data(), (size_t)b.bytes);
      if (!r.ok) { fclose(f); glg_engine_destroy(e); return set_error("glg_engine_load: truncated or corrupt plan file"); }
      cudaMemcpy(b.ptr, stage.data(), (size_t)b.bytes, cudaMemcpyHostToDevice);
    }
  }
  fclose(f);
  for (EOp& op : e->ops)
    for (EArg& a : op.args) {
      if (a.tag == 'P') {
        a.p = resolve(e, a.fix[0]);
        continue;
      }
      for (const Fixup& x : a.fix) {                 // 'S'
        void* p = resolve(e, x);
        memcpy(a.s.data() + x.at, &p, 8);
      }
    }
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
    const int rc = op.def->run(op.args.data(), stream);
    if (rc) return rc;
  }
  return 0;
}

extern "C" int64_t glg_engine_num_ops(GlgEngine* e) { return e ? (int64_t)e->ops.size() : -1; }
