// wgmma / TMA GEMM and implicit-GEMM 3x3 convolution for sm_90a: host side (tile picker, epilogue-kind dispatch,
// launches) and the split-K reduce kernel.  The tile kernels are in gemm_tc.cuh, instantiated by gemm_tc_bn*.cu.
#include "gemm_tc.cuh"

namespace glg {

// out[row][n..n+7] = sum_s ws[s][row][n..] (fixed order) + bias + rowbias, SiLU, gate, + residual  -> bf16
__global__ void splitk_reduce_kernel(const GemmKParams p) {
  pdl_trigger();
  pdl_wait();
  const int nv = p.N >> 3;
  const long long total = (long long)p.M * nv;
  const float gate = p.gate ? __ldg(p.gate) : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / nv), n0 = (int)(i % nv) * 8;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < p.splits; ++s) {
      const float4* w4 = reinterpret_cast<const float4*>(p.ws + ((size_t)s * p.M + row) * p.N + n0);
      const float4 a = w4[0], b = w4[1];
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __ldg(p.bias + n0 + j);
    }
    if (p.rowbias) {
      const float* rb = p.rowbias + (size_t)(row / p.rows_per_batch) * p.ld_rowbias + n0;
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __ldg(rb + j);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = act_f(p.act, v[j]);
    if (p.gate) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= gate;
    }
    if (p.residual) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(p.residual + (size_t)row * p.ldr + n0));
      float2 f;
      f = unpack_bf16x2(u.x); v[0] += f.x; v[1] += f.y;
      f = unpack_bf16x2(u.y); v[2] += f.x; v[3] += f.y;
      f = unpack_bf16x2(u.z); v[4] += f.x; v[5] += f.y;
      f = unpack_bf16x2(u.w); v[6] += f.x; v[7] += f.y;
    }
    const size_t out_off = p.orpb ? (size_t)(row / p.orpb) * p.obs + (size_t)(row % p.orpb) * p.ldc : (size_t)row * p.ldc;
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]); o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(p.out) + out_off + n0) = o;
  }
}

// ------------------------------------------------------------------------------------------------
// launch
// ------------------------------------------------------------------------------------------------
int g_force_bn = 0;     // test hooks (glg_debug_force_bn / glg_debug_gemm_cta2 / glg_debug_splitk)
int g_splitk_mode = 0;  // 0 = heuristic, 1 = never, 2 = split whenever legal
int g_cta2_mode = -1;   // 0 = heuristic, 1 = never pair, 2 = pair whenever legal; -1 = read GLG_GEMM_CTA2 (default 0)
int g_bres_mode = -1;   // B-resident tiles: 0 = heuristic, 1 = never, 2 = whenever legal; -1 = read GLG_GEMM_BRES (default 1)
int g_pp_mode = 0;      // ping-pong consumers (glg_debug_gemm_pp): 0 = heuristic, 1 = never, 2 = whenever legal

static constexpr long long kTileMax = 227 * 1024 - 1024 - 1024;     // dynamic smem minus alignment slack and barriers

// A stages left beside a resident [BN x K] weight tile (0: does not fit)
static int bres_stages(int bn, int num_kb) {
  const long long left = kTileMax - (long long)num_kb * bn * 128;
  if (left < 3 * 16384) return 0;
  const int st = (int)(left / 16384);
  return st > 12 ? 12 : st;
}

// Tile / split choice by a small time model (cycles, H100 data-sheet rates, not tuned by measurement):
//   per 64-wide K step an SM needs max(MMA = 4*BN: 128 x BN x 64 MACs at 2048 bf16 MAC/clk, operand bytes / ~32 B/clk of
//   L2->SM bandwidth) cycles (a pair stages 128 + BN/2 operand rows per SM instead of 128 + BN); a CTA pays ~3000 cycles
//   of fixed cost per work item; split-K adds a reduce pass over splits * M * N fp32.  The least estimated time wins.
// Schedule: ping-pong only where a forced-tile sweep (scripts/sweep_bn.py, H100 80GB HBM3 at 400 W) measured it ahead of
// every cooperative tile: 3x3 convolutions with M >= 8192 on 64-wide tiles (SD levels 0-1 at 8 rows: 0.72-0.87x the
// time of the cooperative tile the model picks) and GEGLU with M <= 512 (0.87x).  Elsewhere it measured level or slower.
static bool pingpong_pays(int M, int bn, bool geglu, bool conv) {
  return (conv && M >= 8192 && bn == 64) || (geglu && M <= 512);
}

static void pick_tile(int M, int N, int num_kb, bool geglu, bool conv, int max_splits, long long ws_bytes,
                      int* bn_out, int* cta2_out, int* splits_out, int* bres_out, int* pp_out) {
  if (g_cta2_mode < 0) {
    const char* e = getenv("GLG_GEMM_CTA2");
    g_cta2_mode = e ? atoi(e) : 0;
  }
  if (g_bres_mode < 0) {
    const char* e = getenv("GLG_GEMM_BRES");
    g_bres_mode = e ? atoi(e) : 1;      // opt-in
  }
  const int sms = num_sms();
  const int cands[4] = {256, 160, 128, 64};
  float best = 1e30f; int best_bn = 0, best_pair = 0, best_s = 1, best_res = 0, best_pp = 0;
  for (int pair = 0; pair < 2; ++pair) {
    if (pair && (g_cta2_mode == 1 || M <= 128)) continue;
    // the heuristic pairs only large, long-K plain GEMMs with N % 256 == 0 and the larger 3x3 convolutions
    if (pair && g_cta2_mode == 0 && !conv && (N % 256 || num_kb < 16 || M < 4096)) continue;
    if (pair && g_cta2_mode == 0 && conv && M < 2048) continue;
    if (!pair && g_cta2_mode == 2 && M > 128) {
      bool any = false;
      for (int i = 0; i < 3; ++i) any |= (N % cands[i] == 0) && (!geglu || cands[i] == 256);
      if (any) continue;
    }
    for (int i = 0; i < 4; ++i) {
      const int bn = cands[i];
      if (N % bn) continue;
      if (geglu && bn != 256) continue;
      if (g_force_bn && bn != g_force_bn && (N % g_force_bn == 0) && !geglu) continue;
      if (pair && bn < 128) continue;                    // per-CTA half of B must stay a whole number of KiB
      if (pair && g_cta2_mode == 0 && !conv && bn != 256) continue;
      for (int pp = 0; pp < 2; ++pp) {
        // ping-pong holds 128 x BN fp32 accumulators per warpgroup in 168 registers: BN <= 128 (GEGLU: 128-row halves of
        // the 256 tile); 128 x 160 spills
        if (pp && (g_pp_mode == 1 || (!geglu && bn > 128))) continue;
        if (pp && g_pp_mode == 0 && !pingpong_pays(M, bn, geglu, conv)) continue;
        const int kbn = (pp && geglu) ? 128 : bn;        // width of one work item
        // ping-pong where it measured ahead (heuristic) or wherever legal (test hook): preferred over every cooperative tile
        const float force = pp ? 1e-3f : 1.0f;
        const int rows = pair ? 256 : 128;
        const int tiles = ((M + rows - 1) / rows) * (N / kbn);
        const int units = pair ? sms / 2 : sms;
        const float mma = 4.0f * kbn;
        const float l2 = 4.0f * (pair ? 128.0f + 0.5f * kbn : 128.0f + kbn);
        const float per_kb = mma > l2 ? mma : l2;
        for (int sp = 1; sp <= (pair ? 1 : max_splits); ++sp) {
          if (sp > 1 && (num_kb / sp < (g_splitk_mode == 2 ? 4 : 16) || (long long)sp * M * N * 4 > ws_bytes)) break;
          if (sp > 1 && tiles * 2 > units && g_splitk_mode != 2) break;        // only when the tile grid leaves >= half the SMs idle
          if (g_splitk_mode == 2 && max_splits > 1 && sp == 1 && num_kb >= 8) continue;      // test hook: force a split
          const int waves = (tiles * sp + units - 1) / units;
          const int kb_cta = (num_kb + sp - 1) / sp;
          float t = (float)waves * (per_kb * kb_cta + 3000.0f);
          if (sp > 1) t += 12000.0f + (float)sp * M * N * 4.0f / (sms * 40.0f);     // slab round trip + reduce launch
          const int ctas = (pair ? 2 : 1) * (tiles * sp < units ? tiles * sp : units);
          t *= 1.0f + 0.10f * (1.0f - (float)ctas / (float)sms);     // idle SMs: prefer the finer decomposition
          t *= force;
          if (t < best) { best = t; best_bn = bn; best_pair = pair; best_s = sp; best_res = 0; best_pp = pp; }
        }
        // B-resident: one n-tile per CTA, weights loaded once per CTA, only A streams (plain GEMMs, single CTAs)
        const int tiles_n = N / kbn, tiles_m = (M + 127) / 128;
        if (!pair && !conv && g_bres_mode != 1 && tiles_n <= sms && bres_stages(kbn, num_kb) > 0) {
          const int per_n = sms / tiles_n;
          if (tiles_m >= 2 * per_n || g_bres_mode == 2) {
            const int waves = (tiles_m + per_n - 1) / per_n;
            const float l2a = 4.0f * 128.0f;
            float t = (float)waves * ((mma > l2a ? mma : l2a) * num_kb + 3000.0f) + 4.0f * kbn * num_kb;
            const int ctas = per_n * tiles_n;
            t *= 1.0f + 0.10f * (1.0f - (float)ctas / (float)sms);
            if (g_bres_mode == 2) t = -1.0f / (float)bn / force;   // test hook: force (widest legal tile)
            else t *= force;
            if (t < best) { best = t; best_bn = bn; best_pair = 0; best_s = 1; best_res = 1; best_pp = pp; }
          }
        }
      }
    }
  }
  *bn_out = best_bn; *cta2_out = best_pair; *splits_out = best_s; *bres_out = best_res; *pp_out = best_pp;
}


// ---- epilogue kinds -----------------------------------------------------------------------------------------------------
struct GemmInstance { int bn; bool geglu, cta2, pp; int epi; GemmLaunchFn fn; };
#define GLG_GEMM_TABLE_ROW(BN, GEGLU, CTA2, PP, NS) {BN, GEGLU, CTA2, PP, NS::kEpi, &NS::launch<BN, GEGLU, CTA2, PP>},
static const GemmInstance kGemmInstances[] = {GLG_GEMM_INSTANCES(GLG_GEMM_TABLE_ROW)};

// template BN of a launch: ping-pong GEGLU runs 128-wide items of the packed 256-row tile
static int bn_launch(int bn, bool geglu, bool pp) { return pp && geglu ? 128 : bn; }

// the epilogue's runtime flags as EPI bits; a split-K launch's tile kernel stores raw partials (the reduce kernel
// applies the flags), so it needs none
static int epilogue_flags(const GemmKParams& p) {
  if (p.splits > 1) return 0;
  return (p.ln_stats ? EPI_LN : 0) | (p.bias ? EPI_BIAS : 0) | (p.rowbias ? EPI_ROWBIAS : 0) | (p.gate ? EPI_GATE : 0) |
         (p.residual ? EPI_RES : 0) | (p.stats_out ? EPI_STATS : 0) | (p.out_fp32 ? EPI_F32 : 0) | (p.orpb ? EPI_ORPB : 0) |
         (p.act ? EPI_ACT : 0);
}

// the kernel of a tile with these flags: the kind equal to the flags where it is instantiated for the tile, else the
// generic kernel (nullptr: no such tile)
static const GemmInstance* find_instance(int bn, bool geglu, bool cta2, bool pp, int flags) {
  const GemmInstance* generic = nullptr;
  for (const GemmInstance& g : kGemmInstances) {
    if (g.bn != bn || g.geglu != geglu || g.cta2 != cta2 || g.pp != pp) continue;
    if (g.epi == flags) return &g;
    if (g.epi == EPI_GENERIC) generic = &g;
  }
  return generic;
}
}  // namespace glg

using namespace glg;

extern "C" void glg_debug_force_bn(int bn) { glg::g_force_bn = bn; }
// test hook (host only, no CUDA work): what the tile picker chooses for a problem; out[3] = {BN, paired CTAs, K splits}
extern "C" void glg_debug_pick_tile(int M, int N, int K, int geglu, int conv, int can_split, long long ws_bytes, int* out) {
  int bres = 0, pp = 0;
  glg::pick_tile(M, N, (conv ? 9 : 1) * (K / 64), geglu != 0, conv != 0, can_split ? 8 : 1, ws_bytes, &out[0], &out[1], &out[2], &bres, &pp);
  out[1] |= bres << 8;           // bit 8 of the "paired" word: B-resident
}
// test hook (host only): 1 when the tile picker runs the problem on the ping-pong schedule
extern "C" int glg_debug_pick_pingpong(int M, int N, int K, int geglu, int conv, int can_split, long long ws_bytes) {
  int bn, pair, sp, bres, pp = 0;
  glg::pick_tile(M, N, (conv ? 9 : 1) * (K / 64), geglu != 0, conv != 0, can_split ? 8 : 1, ws_bytes, &bn, &pair, &sp, &bres, &pp);
  return pp;
}
// test hook (host only): the epilogue kind (EPI bits; 512 = the generic kernel) glg_gemm runs for a problem whose
// epilogue flags are `flags` (EPI bits of GemmKParams: see gemm_tc.cuh)
extern "C" int glg_debug_epilogue_kind(int M, int N, int K, int geglu, int conv, int can_split, long long ws_bytes, int flags) {
  int bn, pair, sp, bres, pp = 0;
  glg::pick_tile(M, N, (conv ? 9 : 1) * (K / 64), geglu != 0, conv != 0, can_split ? 8 : 1, ws_bytes, &bn, &pair, &sp, &bres, &pp);
  const glg::GemmInstance* g = glg::find_instance(glg::bn_launch(bn, geglu != 0, pp != 0), geglu != 0, pair != 0, pp != 0, sp > 1 ? 0 : flags);
  return g ? g->epi : -1;
}
extern "C" void glg_debug_gemm_pp(int mode) { glg::g_pp_mode = mode; }
extern "C" void glg_debug_gemm_bres(int mode) { glg::g_bres_mode = mode; }
extern "C" void glg_debug_gemm_cta2(int mode) { glg::g_cta2_mode = mode; }
extern "C" void glg_debug_splitk(int mode) { glg::g_splitk_mode = mode; }

extern "C" int glg_gemm(const GlgGemmArgs* a, void* stream) {
  if (!a) return set_error("glg_gemm: null args");
  if (a->K <= 0 || a->K % 64) return set_error("glg_gemm: K must be a positive multiple of 64");
  if (a->M <= 0 || a->N <= 0) return set_error("glg_gemm: M, N must be positive");
  if ((a->lda % 8) || (a->ldc % 8) || (a->residual && (a->ldr % 8))) return set_error("glg_gemm: leading dims must be multiples of 8");
  if (((uintptr_t)a->A | (uintptr_t)a->W | (uintptr_t)a->out | (uintptr_t)a->residual) & 15) return set_error("glg_gemm: pointers must be 16-byte aligned");
  if (a->rowbias && ((a->ld_rowbias % 4) || a->rows_per_batch <= 0)) return set_error("glg_gemm: bad rowbias args");
  if (a->geglu && (a->N % 256 || !a->bias || a->out_fp32)) return set_error("glg_gemm: geglu needs N % 256 == 0, a bias and bf16 output");
  int bn = 0, cta2 = 0, splits = 1, bres = 0, pp = 0;
  const bool can_split = a->splitk_ws && g_splitk_mode != 1 && !a->geglu && !a->ln_stats && !a->stats_out && !a->out_fp32 &&
                         !((uintptr_t)a->splitk_ws & 15);
  pick_tile(a->M, a->N, (a->conv_mode ? 9 : 1) * (a->K / 64), a->geglu != 0, a->conv_mode != 0, can_split ? 8 : 1,
            a->splitk_ws_bytes, &bn, &cta2, &splits, &bres, &pp);
  if (!bn) return set_error("glg_gemm: N must be a multiple of 64");
  const int kbn = bn_launch(bn, a->geglu != 0, pp != 0);          // width of one work item (ping-pong GEGLU: half a packed tile)
  GemmKParams p;
  memset(&p, 0, sizeof(p));
  const int rows_per_tile = cta2 ? 256 : 128;
  p.M = a->M; p.N = a->N;
  p.kb_per_tap = a->K / 64;
  p.num_kb = a->conv_mode ? 9 * p.kb_per_tap : p.kb_per_tap;
  p.tiles_m = (a->M + rows_per_tile - 1) / rows_per_tile;
  p.tiles_n = a->N / kbn;
  p.conv = a->conv_mode;
  p.out = a->out; p.ldc = a->ldc; p.out_fp32 = a->out_fp32;
  p.bias = a->bias; p.rowbias = a->rowbias; p.ld_rowbias = a->ld_rowbias; p.rows_per_batch = a->rows_per_batch > 0 ? a->rows_per_batch : 1;
  p.act = a->act; p.gate = a->gate; p.residual = reinterpret_cast<const bf16*>(a->residual); p.ldr = a->ldr;
  if (a->ln_stats) {
    if (!a->ln_colsum || a->ln_slots <= 0 || a->conv_mode) return set_error("glg_gemm: LayerNorm fold needs ln_colsum, ln_slots > 0 and a plain GEMM");
    if (((uintptr_t)a->ln_stats & 7) || ((uintptr_t)a->ln_colsum & 15)) return set_error("glg_gemm: ln_stats / ln_colsum alignment");
    if (a->ln_slot_stride > 0 && a->ln_slot_stride < a->M) return set_error("glg_gemm: ln_slot_stride < M");
    p.ln_stats = a->ln_stats; p.ln_slots = a->ln_slots; p.ln_colsum = a->ln_colsum; p.ln_eps = a->ln_eps; p.inv_k = 1.0f / (float)a->K;
  }
  if (a->stats_out) {
    if (a->geglu || a->out_fp32 || a->stats_slots * 32 != a->N || ((uintptr_t)a->stats_out & 7))
      return set_error("glg_gemm: stats_out needs a bf16 non-GEGLU output and stats_slots == N / 32");
    p.stats_out = a->stats_out; p.stats_slots = a->stats_slots;
  }
  if (a->out_rows_per_batch > 0) {
    if (a->out_batch_stride % 8) return set_error("glg_gemm: out_batch_stride must be a multiple of 8");
    p.orpb = a->out_rows_per_batch; p.obs = a->out_batch_stride;
  }
  if (a->bias && ((uintptr_t)a->bias & 15)) return set_error("glg_gemm: bias must be 16-byte aligned");

  p.splits = splits;
  p.ws = splits > 1 ? reinterpret_cast<float*>(a->splitk_ws) : nullptr;
  p.b_res = bres;
  const long long stage_bytes = bres ? 16384 : 128 * 128 + kbn * 128;
  const long long fixed = bres ? (long long)p.num_kb * kbn * 128 : 0;
  long long stages = (kTileMax - fixed) / stage_bytes;
  const int cap = bres ? 12 : 8;
  p.stages = (int)(stages > cap ? cap : stages);
  if (p.stages < 2) return set_error("glg_gemm: internal: shared memory budget");
  const size_t smem = (size_t)(p.stages * stage_bytes + fixed) + 1024 + 1024;
  if (a->stats_out) p.stats_stride = a->stats_slot_stride > 0 ? a->stats_slot_stride : a->M;
  if (a->ln_stats) p.ln_stride = a->ln_slot_stride > 0 ? a->ln_slot_stride : a->M;

  // a pair: each CTA multicasts half of the B tile; ping-pong GEGLU: x and gate rows are two boxes
  const uint32_t brows = (uint32_t)(cta2 || (pp && a->geglu) ? kbn / 2 : kbn);
  CUtensorMap ta, tb;
  if (a->conv_mode) {
    const int H = a->H, W = a->Wd, B = a->Bn;
    if (H <= 0 || W <= 0 || B <= 0 || (long long)B * H * W != a->M) return set_error("glg_gemm: conv dims do not match M");
    const int HW = H * W;
    p.HW = HW; p.Wd = W;
    const uint64_t dims[4] = {(uint64_t)a->K, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[3] = {(uint64_t)a->lda * 2, (uint64_t)a->lda * 2 * W, (uint64_t)a->lda * 2 * HW};
    if (get_tmap_bf16_im2col3x3(&ta, a->A, dims, str, 64, 128)) return -1;
    const uint64_t wd[2] = {(uint64_t)a->K, (uint64_t)a->N * 9};
    const uint64_t ws[1] = {(uint64_t)a->K * 2};
    const uint32_t wb[2] = {64, brows};
    if (get_tmap_bf16(&tb, a->W, 2, wd, ws, wb)) return -1;
  } else {
    const uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
    const uint64_t str[1] = {(uint64_t)a->lda * 2};
    const uint32_t box[2] = {64, 128};
    if (get_tmap_bf16(&ta, a->A, 2, dims, str, box)) return -1;
    const uint64_t wd[2] = {(uint64_t)a->K, (uint64_t)a->N};
    const uint64_t ws[1] = {(uint64_t)a->K * 2};
    const uint32_t wb[2] = {64, brows};
    if (get_tmap_bf16(&tb, a->W, 2, wd, ws, wb)) return -1;
  }
  const GemmInstance* inst = find_instance(kbn, a->geglu != 0, cta2 != 0, pp != 0, epilogue_flags(p));
  if (!inst) return set_error("glg_gemm: internal: bad tile");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (inst->fn(ta, tb, p, smem, st)) return -1;
  if (p.splits > 1) {
    const long long total = (long long)p.M * (p.N / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    cudaError_t e = launch_k(splitk_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, st, 1, p);
    count_launch();
    if (e != cudaSuccess) return set_error(std::string("splitk reduce launch: ") + cudaGetErrorString(e));
    return check_launch("splitk reduce launch");
  }
  return 0;
}
