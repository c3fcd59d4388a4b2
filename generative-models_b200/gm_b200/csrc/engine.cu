// libgm_b200.so — host side of the C ABI (include/gm_b200.h): context, GEMM plans
// (TMA tensor maps + launch config), the GAN train-step engine.  No torch types.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "gm_b200.h"
#include "gemm_wgmma.cuh"
#include "kernels.cuh"
#include "conv_ops.cuh"

using namespace gm;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct gm_ctx {
  int device = 0;
  int num_sms = 0;
  PFN_encodeTiled encode = nullptr;
  std::string err;
  long long launches = 0;     // kernels launched by this context (counted by launch() only; gm_launch_count)
  // Run-time switches, read from the environment by gm_ctx_create:
  bool pdl = true;            // programmatic stream serialisation on every launch (GM_NO_PDL=1 off; gm_ctx_set_pdl)
  bool tma_store = true;      // GM_NO_TMA_STORE=1: epilogue stores through LDS + STG only
  bool tn208 = true;          // GM_TN208=0: every wide TN plan takes the 256-wide tile (the previous route)
  float* scratch = nullptr;   // split-K partials for the generic gm_gemm_bf16
  size_t scratch_bytes = 0;
  void* red = nullptr;        // scratch of the conv building blocks' two-stage reductions (engine_conv.inl)
  size_t red_bytes = 0;
  void* loss_zero = nullptr;  // 64 zero bytes: bias / Fisher state / completion counter for gm_loss_rows
  long long plan_lo = 0;      // > 0 while an engine in split-operand mode builds its plans: element offset of the lo planes
  // gm_prof_enable: 0 off, 1 CUDA events around every GEMM launch (gm_prof_collect sums them by plan kind), 2 around every
  // launch (gm_prof_report sums them by kernel name: in-stream durations including the launch gaps)
  int prof = 0;
  // name: level 2 only; kind -1: not a GEMM.  launches: 2 for a GEMM run as a main and a companion grid (launch_pp208),
  // timed as one span: an event between the two grids would hold the companion back until the main grid completes
  struct ProfRec { const char* name; int kind; double flops; cudaEvent_t e0, e1; int launches; };
  std::vector<ProfRec> prof_recs;
};

static int fail(gm_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}
#define CU_OK(ctx, expr)                                                                          \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return fail(ctx, GM_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int rup(int a, int b) { return cdiv(a, b) * b; }

// on-device batch sampler (kernels.cuh: Sampler): permutation of [0, n) keyed by (seed, epoch-or-step)
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
static Sampler make_sampler(long long n, uint64_t seed, uint64_t round, uint64_t offset, const unsigned long long* step_ptr = nullptr) {
  Sampler sp;
  sp.n = n > 0 ? unsigned(n) : 0u;
  int bits = 2;
  while (bits < 32 && (1ull << bits) < (unsigned long long)(n > 0 ? n : 1)) ++bits;
  if (bits & 1) ++bits;
  sp.half_bits = unsigned(bits / 2);
  sp.seed_mix = splitmix64(seed);
  sp.key = sampler_key(sp.seed_mix, round);
  sp.offset = offset;
  sp.step_ptr = step_ptr;      // device-step mode: the kernel derives the key from *step_ptr instead of `round`
  return sp;
}
static const Sampler kNoSampler = {0u, 1u, 0ull, 0ull, nullptr, 0ull};

// ------------------------------------------------------------------ tensor maps
// 2-D bf16 row-major matrix: `inner` contiguous elements per row (logical extent, may
// be smaller than ld), `outer` rows, 128-byte swizzle, OOB elements read as zero.
static int make_tmap(gm_ctx* c, CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld,
                     uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld * 2) % 16 != 0)
    return fail(c, GM_ERR_ARG, "tensor map: pointer/ld must be 16-byte aligned (ptr=%p ld=%llu)", ptr, (unsigned long long)ld);
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = c->encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(c, GM_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d", int(r));
  return GM_OK;
}

// ------------------------------------------------------------------ GEMM plans
enum PlanKind { PK_NT_208 = 0, PK_NT_64, PK_TN_256, PK_TN_64 };

struct GemmPlan {
  CUtensorMap tmA, tmB;
  CUtensorMap tmA2, tmB2;   // residual (lo) planes of the operands in split mode, else copies of tmA / tmB
  // MN-major 208-wide plans: 16-column tail boxes of tmB / tmB2 (32-byte swizzle).  K-major 208-wide plans: the boxes of
  // the cluster ranks' shorter B shares (b_share_rows)
  CUtensorMap tmBt, tmB2t;
  CUtensorMap tmBc;         // K-major 208-wide plans: B in the 104-row shares of a 2-CTA companion grid (launch_pp208)
  // output map of the K-major bf16 kernels (16-row x 32-column box, 64-byte swizzle), encoded at the first
  // launch because the epilogue (output pointer / leading dimension) is set after plan_gemm
  mutable CUtensorMap tmC;
  mutable int tmc_state;   // 0: not encoded yet, 1: in use, 2: output not eligible (STG path)
  GemmParams p;
  int kind;
  int bn;         // tile width: the TN kind (PK_TN_256) runs 208- or 256-wide tiles
  int grid;
  double flops;   // algorithmic 2*M*N*K of the logical problem (no padding)
  bool one_grid;  // gm_gemm_bf16: one GEMM kernel per call, never a main + companion pair (launch_pp208)
};

// Profile name of a GEMM launch: plan kind and epilogue signature, output type, K class, split (interned)
static const char* gemm_name(const GemmPlan& pl) {
  static const char* kKind[4] = {"gemm_nt208", "gemm_nt64", "gemm_tn", "gemm_tn64"};
  static std::map<int, std::string> names;
  const GemmParams& q = pl.p;
  const bool f32 = q.epi == EPI_F32, klong = q.K >= 512, split = q.nparts == 3;
  const int key = epi_sig(q) | (pl.kind | f32 << 2 | klong << 3 | split << 4 | (pl.bn == 208) << 5) << kEpiSigBits;
  auto it = names.find(key);
  if (it == names.end()) {
    char buf[128];
    char kind[32];
    snprintf(kind, sizeof kind, pl.kind == PK_TN_256 ? "%s%d" : "%s", kKind[pl.kind], pl.bn);
    snprintf(buf, sizeof buf, "%s[act%d aux%d%s%s%s%s%s K%s%s]", kind, q.act, q.aux_mode, q.bias ? " bias" : "",
             dot_has_w(q.dot) ? " dot" : "", q.dot == DOT_W_PRE ? " pre" : (q.dot == DOT_W_MASK ? " mask" : ""),
             q.dot == DOT_SQ ? " sq" : "", f32 ? " f32" : "", klong ? "long" : "short", split ? " split" : "");
    it = names.emplace(key, buf).first;
  }
  return it->second.c_str();
}

// What launch() accounts a kernel as: its name (a GEMM is named by its plan), whether it takes programmatic stream
// serialisation, and for a GEMM its plan (kind for gm_prof_collect), the FLOPs of this launch's share of the plan and
// its cluster size.  span: SPAN_OWN times the launch on its own; a main grid (SPAN_OPEN) and the companion grid right
// behind it (SPAN_CLOSE) share one profile record, which counts both launches.
enum : int { SPAN_OWN = 0, SPAN_OPEN = 1, SPAN_CLOSE = 2 };
struct KernelTag {
  const char* name;
  bool pdl = true;
  const GemmPlan* plan = nullptr;
  int cluster = 1;
  double flops = 0.0;
  int span = SPAN_OWN;
  KernelTag(const char* n, bool pdl_ = true) : name(n), pdl(pdl_) {}
  KernelTag(const GemmPlan& pl, int cl, double fl, int sp) : name(nullptr), plan(&pl), cluster(cl), flops(fl), span(sp) {}
};

// Launch configuration; `at` receives its attributes.  With `pdl` the grid may become resident while its predecessor
// drains, and blocks in griddepcontrol.wait (first statement of every kernel, after the prologue in the GEMM) until the
// predecessor completed.
static cudaLaunchConfig_t launch_cfg(dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster, bool pdl,
                                     cudaLaunchAttribute (&at)[2]) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = at;
  if (cluster > 1) {
    at[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    at[cfg.numAttrs].val.clusterDim.x = cluster;
    at[cfg.numAttrs].val.clusterDim.y = 1;
    at[cfg.numAttrs].val.clusterDim.z = 1;
    ++cfg.numAttrs;
  }
  if (pdl) {
    at[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg.numAttrs;
  }
  return cfg;
}

// Every kernel of the library is launched here: a failed launch ends the entry point with GM_ERR_CUDA (nothing after it
// is enqueued), a successful one is counted (gm_launch_count) and, when the context's profiling level asks for it, timed.
template <typename... KArgs, typename... Args>
[[nodiscard]] static int launch(gm_ctx* c, const KernelTag& k, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                cudaStream_t s, Args&&... args) {
  cudaLaunchAttribute at[2];
  const cudaLaunchConfig_t cfg = launch_cfg(grid, block, smem, s, k.cluster, k.pdl && c->pdl, at);
  const bool timed = c->prof == 2 || (c->prof == 1 && k.plan);
  // SPAN_CLOSE continues the record its main grid opened (launch_pp208 launches the two back to back)
  const bool opens = timed && k.span != SPAN_CLOSE;
  gm_ctx::ProfRec r;
  if (opens) {
    r.name = c->prof == 2 ? (k.plan ? gemm_name(*k.plan) : k.name) : nullptr;
    r.kind = k.plan ? k.plan->kind : -1;
    r.flops = k.flops;
    r.launches = 1;
    CU_OK(c, cudaEventCreate(&r.e0));
    CU_OK(c, cudaEventCreate(&r.e1));
    CU_OK(c, cudaEventRecord(r.e0, s));
  }
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();   // a launch error is not sticky: leave no trace of it for the caller's next runtime call
    if (opens) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    else if (timed) cudaEventRecord(c->prof_recs.back().e1, s);   // close the main grid's record on its own
    return fail(c, GM_ERR_CUDA, "%s launch failed: %s", k.plan ? gemm_name(*k.plan) : k.name, cudaGetErrorString(e));
  }
  c->launches++;
  if (timed) {
    if (opens) c->prof_recs.push_back(r);
    gm_ctx::ProfRec& rec = c->prof_recs.back();
    if (!opens) { rec.launches++; rec.flops += k.flops; }
    if (k.span != SPAN_OPEN) CU_OK(c, cudaEventRecord(rec.e1, s));
  }
  return GM_OK;
}

// One grid of a plan's product: all of it (the default), or the main or companion share of a two-grid plan (launch_pp208):
// m-tiles [m_tile0, m_tile0 + m_tiles), at most `clusters` clusters, B through tmB (the companion's 2-CTA B shares).
struct GridPart {
  int m_tile0 = 0, m_tiles = 0;   // m_tiles 0: all of the plan's
  int clusters = 0;               // 0: as many as the device holds at once
  int span = SPAN_OWN;
  const CUtensorMap* tmB = nullptr;
};

// The instance's function, configured on the current device at its first use: the opt-in to > 48 KB dynamic shared
// memory is per (function, device); so is the number of clusters that fit at once (*mc; 0 unclustered)
template <int BN, bool AMN, bool BMN, int EPI = kEpiUniversal, bool SPLIT = false, bool PP = false,
          int CL = kGemmCluster<BN, AMN, BMN>, int ROLE = PDL_SINGLE>
static int inst_clusters(gm_ctx* c, const GemmPlan& pl, cudaStream_t s, int* mc) {
  using Cfg = GemmCfg<BN, !AMN, PP>;
  auto kern = gemm_wgmma_kernel<BN, AMN, BMN, EPI, SPLIT, PP, CL, ROLE>;
  static bool configured[64] = {};
  static int max_clusters[64] = {};
  int dev = 0;
  CU_OK(c, cudaGetDevice(&dev));
  const bool cached = dev >= 0 && dev < 64;
  *mc = cached ? max_clusters[dev] : 0;
  if (!cached || !configured[dev]) {
    CU_OK(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (CL > 1) {
      cudaLaunchAttribute at[2];
      const cudaLaunchConfig_t cfg = launch_cfg(dim3(CL), dim3(kGemmThreads), Cfg::SMEM_BYTES, s, CL, false, at);
      CU_OK(c, cudaOccupancyMaxActiveClusters(mc, kern, &cfg));
      if (*mc < 1) return fail(c, GM_ERR_CUDA, "%s: no %d-CTA cluster fits on device %d", gemm_name(pl), CL, dev);
    }
    if (cached) { max_clusters[dev] = *mc; configured[dev] = true; }
  }
  return GM_OK;
}

template <int BN, bool AMN, bool BMN, int EPI = kEpiUniversal, bool SPLIT = false, bool PP = false,
          int CL = kGemmCluster<BN, AMN, BMN>, int ROLE = PDL_SINGLE>
static int launch_inst(gm_ctx* c, const GemmPlan& pl, cudaStream_t s, const GridPart& part = GridPart()) {
  using Cfg = GemmCfg<BN, !AMN, PP>;
  auto kern = gemm_wgmma_kernel<BN, AMN, BMN, EPI, SPLIT, PP, CL, ROLE>;
  int mc = 0;
  if (int rc = inst_clusters<BN, AMN, BMN, EPI, SPLIT, PP, CL, ROLE>(c, pl, s, &mc)) return rc;
  GemmParams prm = pl.p;
  double flops = pl.flops;
  if (part.m_tiles > 0) {
    prm.m_tile0 = part.m_tile0;
    prm.m_tiles = part.m_tiles;
    const int end = (part.m_tile0 + part.m_tiles) * BM, rows = (end < prm.M ? end : prm.M) - part.m_tile0 * BM;
    flops = pl.flops * double(rows) / double(prm.M);
  }
  if (part.clusters > 0 && part.clusters < mc) mc = part.clusters;
  dim3 grid(pl.grid);
  if (CL > 1) {
    // persistent: one cluster per item, up to the clusters the device holds at once (a GPC need not hold a multiple of CL
    // SMs).  K-major clusters group CL m-tiles, MN-major ones pair n-tiles (of an even count)
    const int items = (BMN ? prm.m_tiles * (prm.n_tiles / CL) : cdiv(prm.m_tiles, CL) * prm.n_tiles) * prm.splits;
    grid = dim3(CL * (items < mc ? items : mc));
  }
  prm.tma_store = pl.tmc_state == 1 ? 1 : 0;
  // fp32 rows take float4 stores only where every row of every split starts on 16 bytes (ldc = 30: row 1 is at byte 120)
  prm.f32_vec = prm.epi == EPI_F32 && !(reinterpret_cast<uintptr_t>(prm.part) & 15) && prm.ldp % 4 == 0 && prm.part_stride % 4 == 0;
  return launch(c, KernelTag(pl, CL, flops, part.span), kern, grid, kGemmThreads, Cfg::SMEM_BYTES, s, pl.tmA,
                part.tmB ? *part.tmB : pl.tmB, pl.tmC, pl.tmA2, pl.tmB2, pl.tmBt, pl.tmB2t, prm);
}

// TN kind: the 256-wide tile, or the 208-wide one as 2-CTA clusters over n-tile pairs (an even n-tile count, plan_gemm)
template <bool SPLIT>
static int launch_tn(gm_ctx* c, const GemmPlan& pl, cudaStream_t s) {
  if (pl.bn == 256) return launch_inst<256, true, true, kEpiUniversal, SPLIT>(c, pl, s);
  return launch_inst<208, true, true, kEpiUniversal, SPLIT, false, 2>(c, pl, s);
}

// split-operand plans (gm_prec GM_PREC_SPLIT): the universal epilogue with the residual-plane paths compiled in.  Their
// K-major 208-wide kernel keeps 2-CTA clusters: it runs cooperatively, and as 4-CTA clusters (30 fit on an H100, 120 SMs)
// it slowed the split-precision step by 5% (DESIGN §5)
constexpr int kNtSplitCl = 2;
template <int BN, bool AMN, bool BMN>
static int launch_split(gm_ctx* c, const GemmPlan& pl, cudaStream_t s) {
  if constexpr (BN == 208 && !AMN) return launch_inst<BN, AMN, BMN, kEpiUniversal, true, false, kNtSplitCl>(c, pl, s);
  else return launch_inst<BN, AMN, BMN, kEpiUniversal, true>(c, pl, s);
}

// Per-SM rate of the 2-CTA ping-pong instance (a companion grid) over that of the 4-CTA one: 2-CTA clusters load B once
// per 64-row half for two m-tiles, 43 008 instead of 29 696 B per 128 rows and k-block.  Measured on an H100 SXM at 700 W
// (DESIGN §5) with the whole GEMM as 66 2-CTA clusters against 30 4-CTA clusters at B = 65536: 0.72 for d1 on 2B rows,
// 0.79 for g2 and dx.  The lower one, rounded down; every train-step split is the same for rates from 0.7 to 1.
constexpr double kCompanionRate = 0.7;

// Two-grid split of a K-major 208-wide ping-pong plan.  30 4-CTA clusters fit on an H100 SXM: 120 SMs, since some GPCs
// hold 4k + 2 SMs, and the last of a plan's rounds of 30 items is mostly empty (512 items: 17.07 rounds run as 18).  So a
// plan of two or more rounds runs m-tiles [0, 4 g) as the main grid of 4-CTA clusters and m-tiles [4 g, m_tiles) in
// pairs as a companion grid of 2-CTA clusters on the SMs left over, (num_sms - 4 main_clusters) / 2 clusters.  g makes
// the two grids finish together, at the companion's rate kCompanionRate; among equal finishes the largest g.  Returns 0
// (one grid) where that finishes no sooner.  Every (m-tile, n-tile) keeps its k order, warp, lane and epilogue code, so
// outputs are bit-identical to the single grid's.
static int companion_groups(const GemmParams& p, int main_clusters, int comp_clusters) {
  if (comp_clusters < 1 || main_clusters < 1 || p.splits != 1) return 0;
  const int single = cdiv(cdiv(p.m_tiles, 4) * p.n_tiles, main_clusters);
  if (single < 2) return 0;
  int best = 0;
  double best_t = single;
  for (int g = 1; 4 * g < p.m_tiles; ++g) {
    const double t_main = cdiv(g * p.n_tiles, main_clusters);
    const double t_comp = cdiv(cdiv(p.m_tiles - 4 * g, 2) * p.n_tiles, comp_clusters) / kCompanionRate;
    const double t = t_main > t_comp ? t_main : t_comp;
    if (t < best_t || (best && t == best_t)) { best = g; best_t = t; }
  }
  return best;
}

// A ping-pong plan: one grid of 4-CTA clusters, or a main and a companion grid (companion_groups; PDL_* for their order)
template <int EPI>
static int launch_pp208(gm_ctx* c, const GemmPlan& pl, cudaStream_t s) {
  int mc4 = 0;
  if (int rc = inst_clusters<208, false, false, EPI, false, true, 4>(c, pl, s, &mc4)) return rc;
  // the companion overlaps the main grid only through programmatic dependent launch
  const int g = c->pdl && !pl.one_grid ? companion_groups(pl.p, mc4, (c->num_sms - 4 * mc4) / 2) : 0;
  if (g == 0) return launch_inst<208, false, false, EPI, false, true, 4>(c, pl, s);
  const bool timed = c->prof != 0;
  GridPart main;
  main.m_tiles = 4 * g;
  main.span = timed ? SPAN_OPEN : SPAN_OWN;
  if (int rc = launch_inst<208, false, false, EPI, false, true, 4, PDL_MAIN>(c, pl, s, main)) return rc;
  GridPart comp;
  comp.m_tile0 = 4 * g;
  comp.m_tiles = pl.p.m_tiles - 4 * g;
  comp.clusters = (c->num_sms - 4 * mc4) / 2;
  comp.span = timed ? SPAN_CLOSE : SPAN_OWN;
  comp.tmB = &pl.tmBc;
  return launch_inst<208, false, false, EPI, false, true, 2, PDL_COMPANION>(c, pl, s, comp);
}

// K-major 128x208 kernel: the compile-time-specialised instance of the plan's epilogue signature when the train steps use
// that signature, else the universal instance.  The specialised instances run their consumer warpgroups in ping-pong, so
// each half-tile's epilogue hides under the other warpgroup's wgmma; the 4-CTA cluster's multicast keeps the B feed of
// the half-tiles at that of the cooperative loop (DESIGN §3).
static int launch_nt208(gm_ctx* c, const GemmPlan& pl, cudaStream_t s) {
  const GemmParams& p = pl.p;
  if (p.epi != EPI_BF16) return launch_inst<208, false, false>(c, pl, s);
#define NT208(S) case S: return launch_pp208<S>(c, pl, s)
  switch (epi_sig(p)) {
    NT208(epi_sig(ACT_RELU, AUX_NONE, true, DOT_NONE));
    NT208(epi_sig(ACT_SIGMOID, AUX_NONE, true, DOT_NONE));
    NT208(epi_sig(ACT_RELU, AUX_NONE, true, DOT_W));
    NT208(epi_sig(ACT_RELU, AUX_NONE, true, DOT_W_MASK));
    NT208(epi_sig(ACT_RELU, AUX_NONE, true, DOT_W_PRE));
    NT208(epi_sig(ACT_NONE, AUX_NONE, false, DOT_NONE));
    NT208(epi_sig(ACT_NONE, AUX_NONE, false, DOT_SQ));
    NT208(epi_sig(ACT_NONE, AUX_SIGMOID_GRAD, false, DOT_NONE));
    NT208(epi_sig(ACT_NONE, AUX_RELU_MASK, false, DOT_NONE));
    NT208(epi_sig(ACT_NONE, AUX_NONZERO_MASK, false, DOT_NONE));
    NT208(epi_sig(ACT_NONE, AUX_L1, true, DOT_NONE));
    NT208(epi_sig(ACT_SIGMOID, AUX_VAE_OUT, true, DOT_NONE));
    default: return launch_inst<208, false, false>(c, pl, s);
  }
#undef NT208
}

[[nodiscard]] static int launch_plan(gm_ctx* c, const GemmPlan& pl, cudaStream_t s) {
  if (pl.tmc_state == 0) {
    const GemmParams& p = pl.p;
    const bool nt = pl.kind == PK_NT_208 || pl.kind == PK_NT_64;
    pl.tmc_state = 2;
    // the bulk store serves the pure activation epilogues only; the aux / row-dot epilogues keep LDS + STG
    // (a fence + wait for the bulk store would sit in their longer per-block dependency chain)
    if (c->tma_store && nt && epi_plain(p.aux_mode, p.dot) && p.nparts == 1 && p.epi == EPI_BF16 && p.out != nullptr && !(reinterpret_cast<uintptr_t>(p.out) & 15) &&
        (p.ldo * 2) % 16 == 0 && p.out_cols > 0) {
      int rc = make_tmap(c, &pl.tmC, p.out, uint64_t(p.out_cols), uint64_t(p.M), uint64_t(p.ldo), kEpiCols, kEpiRows, CU_TENSOR_MAP_SWIZZLE_64B);
      if (rc) return rc;
      pl.tmc_state = 1;
    }
  }
  if (pl.p.nparts == 3) {
    switch (pl.kind) {
      case PK_NT_208: return launch_split<208, false, false>(c, pl, s);
      case PK_NT_64: return launch_split<64, false, false>(c, pl, s);
      case PK_TN_256: return launch_tn<true>(c, pl, s);
      default: return launch_split<64, true, true>(c, pl, s);
    }
  }
  switch (pl.kind) {
    case PK_NT_208: return launch_nt208(c, pl, s);
    case PK_NT_64: return launch_inst<64, false, false>(c, pl, s);
    case PK_TN_256: return launch_tn<false>(c, pl, s);
    default: return launch_inst<64, true, true>(c, pl, s);
  }
}

// mode 0 (NT): A [M, lda] K-contiguous, B [N, ldb] K-contiguous.
// mode 1 (TN): A [K, lda] M-contiguous, B [K, ldb] N-contiguous.
// `ncover` = number of output columns the tiling must cover (>= N; out_cols for bf16).
static int plan_gemm(gm_ctx* c, GemmPlan* pl, int mode, int M, int N, int K, const void* A, int lda, const void* B,
                     int ldb, int ncover, int max_splits) {
  memset(pl, 0, sizeof *pl);
  if (M <= 0 || N <= 0 || K <= 0) return fail(c, GM_ERR_ARG, "gemm: bad extents %d %d %d", M, N, K);
  const int ntcl = c->plan_lo > 0 ? kNtSplitCl : kGemmCluster<208, false, false>;   // the launch_split / launch_nt208 instance
  int bn, boxn = 0, boxm = BM, boxn_t = 0;
  if (mode == 0) {
    if (ncover <= 64) { pl->kind = PK_NT_64; bn = 64; boxn = 64; }
    else {   // the cluster ranks' taller and shorter B shares (tmB, tmBt); 64-row A boxes
      pl->kind = PK_NT_208; bn = 208; boxm = kGemmABoxRows<208, false>;
      boxn = b_share_rows(208, ntcl, 0); boxn_t = b_share_rows(208, ntcl, ntcl - 1);
    }
    int rc = make_tmap(c, &pl->tmA, A, K, M, lda, BK, boxm);
    if (rc) return rc;
    rc = make_tmap(c, &pl->tmB, B, K, N, ldb, BK, boxn);
    if (rc) return rc;
    if (boxn_t && (rc = make_tmap(c, &pl->tmBt, B, K, N, ldb, BK, boxn_t))) return rc;
    if (boxn_t && c->plan_lo == 0 && (rc = make_tmap(c, &pl->tmBc, B, K, N, ldb, BK, b_share_rows(208, 2, 0)))) return rc;
  } else {
    // K (batch rows) need not be a multiple of 64: rows past the extent are TMA zero-fill.  Wide outputs take the 208-wide
    // tile, run as 2-CTA clusters over n-tile pairs, wherever it needs an even number of n-tiles and no more than the
    // 256-wide one (400 and 401 columns: 416 instead of 512 computed), so tile count, split count and each output's
    // k-block order stay those of the 256-wide tile.  An odd count keeps the 256-wide tile: unclustered, the 208-wide
    // one slowed the DCGAN step (DESIGN §5)
    const int n208 = cdiv(ncover, 208);
    if (ncover <= 64) { pl->kind = PK_TN_64; bn = 64; }
    else { pl->kind = PK_TN_256; bn = c->tn208 && n208 % 2 == 0 && n208 <= cdiv(ncover, 256) ? 208 : 256; }
    int rc = make_tmap(c, &pl->tmA, A, M, K, lda, 64, BK);
    if (rc) return rc;
    rc = make_tmap(c, &pl->tmB, B, N, K, ldb, 64, BK);
    if (rc) return rc;
    if (bn == 208 && (rc = make_tmap(c, &pl->tmBt, B, N, K, ldb, kTnTail, BK, CU_TENSOR_MAP_SWIZZLE_32B))) return rc;
  }
  pl->bn = bn;
  GemmParams& p = pl->p;
  pl->flops = 2.0 * M * N * K;
  p.M = M; p.N = N; p.K = K;
  p.m_tiles = cdiv(M, BM);
  p.n_tiles = cdiv(ncover, bn);
  p.kblocks = cdiv(K, BK);
  p.nparts = 1; p.kb_part = p.kblocks; p.lo_off = 0;
  pl->tmA2 = pl->tmA; pl->tmB2 = pl->tmB; pl->tmB2t = pl->tmBt;
  if (c->plan_lo > 0) {
    // split operands: second tensor maps on the residual planes, contraction over (hi,hi), (hi,lo), (lo,hi)
    const __nv_bfloat16* A2 = static_cast<const __nv_bfloat16*>(A) + c->plan_lo;
    const __nv_bfloat16* B2 = static_cast<const __nv_bfloat16*>(B) + c->plan_lo;
    int rc;
    if (mode == 0) {
      if ((rc = make_tmap(c, &pl->tmA2, A2, K, M, lda, BK, boxm))) return rc;
      if ((rc = make_tmap(c, &pl->tmB2, B2, K, N, ldb, BK, boxn))) return rc;
      if (boxn_t && (rc = make_tmap(c, &pl->tmB2t, B2, K, N, ldb, BK, boxn_t))) return rc;
    } else {
      if ((rc = make_tmap(c, &pl->tmA2, A2, M, K, lda, 64, BK))) return rc;
      if ((rc = make_tmap(c, &pl->tmB2, B2, N, K, ldb, 64, BK))) return rc;
      if (bn == 208 && (rc = make_tmap(c, &pl->tmB2t, B2, N, K, ldb, kTnTail, BK, CU_TENSOR_MAP_SWIZZLE_32B))) return rc;
    }
    p.nparts = 3; p.kblocks = 3 * p.kb_part; p.lo_off = c->plan_lo;
  }
  const int tiles = p.m_tiles * p.n_tiles;   // work items per split
  const int slots = c->num_sms;               // CTAs resident at once (one per SM)
  int splits = 1;
  if (max_splits > 1) {
    splits = slots / tiles;
    if (splits > max_splits) splits = max_splits;
    if (splits > p.kblocks) splits = p.kblocks;
    if (splits < 1) splits = 1;
  }
  p.kb_per_split = cdiv(p.kblocks, splits);
  p.splits = cdiv(p.kblocks, p.kb_per_split);
  const int total = tiles * p.splits;
  pl->grid = total < slots ? total : slots;
  return GM_OK;
}

// out[r * ld + c] = sum over splits of part[split * stride + r * ld + c] for the logical [rows, cols] block only: columns
// [cols, ld) belong to the caller and are left as they are (no split writes them, so their partials are stale scratch)
__global__ void reduce_partials_kernel(const float* __restrict__ part, int nsplit, long long stride, long long rows, int cols,
                                       int ld, float* __restrict__ out) {
  griddep_sync();
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= rows * cols) return;
  const long long i = cols == ld ? k : (k / cols) * ld + k % cols;
  float t = 0.f;
  for (int s0 = 0; s0 < nsplit; s0 += 8) {     // eight partials in flight, summed in split order
    float a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] = (s0 + u < nsplit) ? part[i + (long long)(s0 + u) * stride] : 0.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) t += a[u];
  }
  out[i] = t;
}

// ------------------------------------------------------------------ ctx
extern "C" int gm_version(void) { return 100; }

extern "C" int gm_ctx_create(int device, gm_ctx** out) {
  if (!out) return GM_ERR_ARG;
  *out = nullptr;
  gm_ctx* c = new gm_ctx();
  c->device = device;
  *out = c;  // returned even on failure so the caller can read gm_last_error
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0)
    return fail(c, GM_ERR_CUDA, "no CUDA device visible: this library has no CPU fallback");
  CU_OK(c, cudaSetDevice(device));
  cudaDeviceProp prop;
  CU_OK(c, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(c, GM_ERR_UNSUPPORTED, "device is sm_%d%d; this library is built for sm_90a (H100) only", prop.major, prop.minor);
  c->num_sms = prop.multiProcessorCount;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  CU_OK(c, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) return fail(c, GM_ERR_CUDA, "cuTensorMapEncodeTiled not available");
  c->encode = reinterpret_cast<PFN_encodeTiled>(fn);
  const char* np = getenv("GM_NO_PDL");
  c->pdl = !(np && np[0] == '1');
  const char* nts = getenv("GM_NO_TMA_STORE");
  c->tma_store = !(nts && nts[0] == '1');
  const char* tn = getenv("GM_TN208");
  c->tn208 = !(tn && tn[0] == '0');
  return GM_OK;
}
extern "C" int gm_ctx_destroy(gm_ctx* c) {
  if (!c) return GM_OK;
  if (c->scratch) cudaFree(c->scratch);
  if (c->red) cudaFree(c->red);
  if (c->loss_zero) cudaFree(c->loss_zero);
  delete c;
  return GM_OK;
}
extern "C" const char* gm_last_error(const gm_ctx* c) { return c ? c->err.c_str() : "null ctx"; }
extern "C" int gm_ctx_num_sms(const gm_ctx* c) { return c ? c->num_sms : 0; }
extern "C" long long gm_launch_count(gm_ctx* c, int reset) {
  if (!c) return 0;
  const long long n = c->launches;
  if (reset) c->launches = 0;
  return n;
}

extern "C" int gm_prof_enable(gm_ctx* c, int on) {
  if (!c) return GM_ERR_ARG;
  c->prof = on == 1 || on == 2 ? on : 0;
  return GM_OK;
}
// level-2 profile (gm_prof_enable(ctx, 2)): synchronises, then writes "name,launches,total_ms\n" lines (one per kernel
// name, GEMMs named by plan kind + epilogue) into buf; returns the number of bytes needed (0 if nothing was recorded)
extern "C" int gm_prof_report(gm_ctx* c, char* buf, int buflen) {
  if (!c) return GM_ERR_ARG;
  CU_OK(c, cudaDeviceSynchronize());
  std::map<std::string, std::pair<long long, double>> agg;
  std::vector<std::string> order;
  for (auto& r : c->prof_recs) {
    if (r.name) {   // recorded at level 2
      float t = 0.f;
      cudaEventElapsedTime(&t, r.e0, r.e1);
      auto it = agg.find(r.name);
      if (it == agg.end()) { order.push_back(r.name); it = agg.emplace(r.name, std::make_pair(0ll, 0.0)).first; }
      it->second.first += r.launches; it->second.second += t;
    }
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  c->prof_recs.clear();
  std::string out;
  for (auto& n : order) {
    char line[256];
    snprintf(line, sizeof line, "%s,%lld,%.6f\n", n.c_str(), agg[n].first, agg[n].second);
    out += line;
  }
  if (buf && buflen > 0) { strncpy(buf, out.c_str(), size_t(buflen) - 1); buf[buflen - 1] = 0; }
  return int(out.size()) + 1;
}
// Synchronises the device, then sums per plan kind (0: NT 128x208, 1: NT 128x64,
// 2: TN 128x256 split-K, 3: TN 128x64 split-K) the launch durations (ms), algorithmic
// FLOPs and launch counts recorded since the last collect.
extern "C" int gm_prof_collect(gm_ctx* c, double* ms, double* flops, long long* count) {
  if (!c || !ms || !flops || !count) return GM_ERR_ARG;
  for (int i = 0; i < 4; ++i) { ms[i] = 0; flops[i] = 0; count[i] = 0; }
  CU_OK(c, cudaDeviceSynchronize());
  for (auto& r : c->prof_recs) {
    if (r.kind >= 0) {
      float t = 0.f;
      cudaEventElapsedTime(&t, r.e0, r.e1);
      ms[r.kind] += t; flops[r.kind] += r.flops; count[r.kind] += r.launches;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  c->prof_recs.clear();
  return GM_OK;
}

// ------------------------------------------------------------------ generic GEMM / Adam
extern "C" int gm_gemm_bf16(gm_ctx* c, const gm_gemm_desc* d, gm_stream stream) {
  if (!c || !d) return GM_ERR_ARG;
  if (!c->encode) return fail(c, GM_ERR_STATE, "context has no device");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  GemmPlan pl;
  const bool f32 = d->out_kind == 1;
  const int ncover = f32 ? d->N : (d->out_cols > d->N ? d->out_cols : d->N);
  // every descriptor the kernels cannot run as written is refused here, before anything is launched
  auto misaligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) != 0; };
  if (d->out_kind != 0 && d->out_kind != 1) return fail(c, GM_ERR_ARG, "gemm: out_kind %d is not 0 (bf16) or 1 (fp32)", d->out_kind);
  if (d->mode != 0 && d->mode != 1) return fail(c, GM_ERR_ARG, "gemm: mode %d is not 0 (NT) or 1 (TN)", d->mode);
  if (d->mode == 1 && !f32) return fail(c, GM_ERR_ARG, "gemm: a TN (mode 1) product has an fp32 output only");
  if (d->act < ACT_NONE || d->act > ACT_LRELU) return fail(c, GM_ERR_ARG, "gemm: act %d is outside 0..3", d->act);
  if (d->aux_mode < AUX_NONE || d->aux_mode > AUX_VAE_OUT) return fail(c, GM_ERR_ARG, "gemm: aux_mode %d is outside 0..3", d->aux_mode);
  if ((d->aux_mode != AUX_NONE) != (d->aux_dev != nullptr)) return fail(c, GM_ERR_ARG, "gemm: aux_dev needs a nonzero aux_mode and the reverse");
  if (!d->C_dev || misaligned(d->C_dev)) return fail(c, GM_ERR_ARG, "gemm: C_dev must be a 16-byte aligned pointer");
  if (misaligned(d->aux_dev) || misaligned(d->bias_dev) || misaligned(d->dot_w_dev))
    return fail(c, GM_ERR_ARG, "gemm: aux_dev, bias_dev and dot_w_dev must be 16-byte aligned");
  if (f32) {
    if (d->pad_one || d->bias_dev || d->act != ACT_NONE || d->aux_dev || d->dot_w_dev || d->dot_out_dev || (d->out_cols != 0 && d->out_cols != d->N))
      return fail(c, GM_ERR_ARG, "gemm: an fp32 output takes no epilogue (out_cols, pad_one, bias, act, aux, dot)");
    const int row_len = d->transpose ? d->M : d->N;
    if (d->ldc < row_len) return fail(c, GM_ERR_ARG, "gemm: fp32 ldc %d is below the stored row length %d", d->ldc, row_len);
  } else {
    if (d->N % 16) return fail(c, GM_ERR_ARG, "bf16 output needs N %% 16 == 0 (N=%d)", d->N);
    if (d->transpose) return fail(c, GM_ERR_ARG, "gemm: transpose applies to an fp32 output only");
    if (ncover % 8 || d->ldc % 8 || d->ldc < ncover)
      return fail(c, GM_ERR_ARG, "gemm: bf16 output needs out_cols %% 8 == 0, ldc %% 8 == 0 and ldc >= out_cols (out_cols=%d ldc=%d)", ncover, d->ldc);
    if (d->aux_dev && (d->ld_aux % 8 || d->ld_aux < ncover))
      return fail(c, GM_ERR_ARG, "gemm: aux needs ld_aux %% 8 == 0 and ld_aux >= out_cols (ld_aux=%d out_cols=%d)", d->ld_aux, ncover);
    if (d->dot_w_dev && !d->dot_out_dev) return fail(c, GM_ERR_ARG, "gemm: dot_w_dev needs dot_out_dev");
    if (d->dot_out_dev && d->dot_ld < d->M) return fail(c, GM_ERR_ARG, "gemm: dot_ld %d is below M %d", d->dot_ld, d->M);
  }
  int rc = plan_gemm(c, &pl, d->mode, d->M, d->N, d->K, d->A_dev, d->lda, d->B_dev, d->ldb, ncover, f32 ? 64 : 1);
  if (rc) return rc;
  pl.one_grid = true;
  GemmParams& p = pl.p;
  if (!f32) {
    p.epi = EPI_BF16;
    p.out = static_cast<__nv_bfloat16*>(d->C_dev);
    p.ldo = d->ldc;
    p.out_cols = ncover;
    p.pad_one = d->pad_one;
    p.bias = d->bias_dev;
    p.act = d->act;
    p.act_slope = d->act_slope;
    p.aux = static_cast<const __nv_bfloat16*>(d->aux_dev);
    p.ld_aux = d->ld_aux;
    p.aux_mode = d->aux_mode;
    p.dot = d->dot_w_dev ? DOT_W : DOT_NONE;
    p.dot_w = d->dot_w_dev;
    p.dot_out = d->dot_out_dev;
    p.dot_ld = d->dot_ld;
    return launch_plan(c, pl, s);
  }
  p.epi = EPI_F32;
  p.transpose = d->transpose;
  p.ldp = d->ldc;
  const long long per = (long long)(d->transpose ? d->N : d->M) * d->ldc;
  if (p.splits == 1) {
    p.part = static_cast<float*>(d->C_dev);
    p.part_stride = 0;
    return launch_plan(c, pl, s);
  }
  const size_t need = size_t(per) * p.splits * sizeof(float);
  if (need > c->scratch_bytes) {
    if (c->scratch) cudaFree(c->scratch);
    c->scratch = nullptr;
    c->scratch_bytes = 0;
    CU_OK(c, cudaMalloc(&c->scratch, need));
    c->scratch_bytes = need;
  }
  p.part = c->scratch;
  p.part_stride = per;
  rc = launch_plan(c, pl, s);
  if (rc) return rc;
  const long long rows = d->transpose ? d->N : d->M;
  const int cols = d->transpose ? d->M : d->N;
  return launch(c, "reduce_partials_kernel", reduce_partials_kernel, unsigned((rows * cols + 255) / 256), 256, 0, s, c->scratch, p.splits, per,
             rows, cols, d->ldc, static_cast<float*>(d->C_dev));
}

static void fill_adam(AdamParams& a, const gm_adam_hp* hp, int step) {
  a.lr = hp->lr; a.b1 = hp->beta1; a.b2 = hp->beta2; a.eps = hp->eps; a.wd = hp->weight_decay; a.clamp = hp->clamp;
  a.bc1 = float(1.0 - pow(double(hp->beta1), double(step)));
  a.bc2_sqrt = float(sqrt(1.0 - pow(double(hp->beta2), double(step))));
  a.update = 1;
}

extern "C" int gm_adam_step_lr(gm_ctx* c, float* p, const float* g, float* m, float* v, int n, const gm_adam_hp* hp,
                               const float* lr_scale_dev, int step, gm_stream stream) {
  if (!c || !p || !g || !m || !v || !hp || n <= 0 || step <= 0) return fail(c, GM_ERR_ARG, "gm_adam_step: bad argument");
  AdamParams a;
  memset(&a, 0, sizeof a);
  a.p = p; a.g = g; a.m = m; a.v = v; a.total = n; a.nseg = 0;
  fill_adam(a, hp, step);
  a.lr_scale = lr_scale_dev;
  return launch(c, "adam_kernel", adam_kernel, cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream), a);
}

extern "C" int gm_adam_step(gm_ctx* c, float* p, const float* g, float* m, float* v, int n, const gm_adam_hp* hp,
                            int step, gm_stream stream) {
  return gm_adam_step_lr(c, p, g, m, v, n, hp, nullptr, step, stream);
}

// ------------------------------------------------------------------ bf16 arena
// Every bf16 buffer of an engine (activations, hidden gradients, operand copies of the weights) is carved from ONE
// allocation; in split-operand mode (gm_prec GM_PREC_SPLIT) the allocation is twice as large and the second half
// holds the residual (lo) planes, so the lo twin of ANY bf16 pointer p of the engine is p + lo_off.
struct BfArena {
  std::vector<std::pair<__nv_bfloat16**, size_t>> reqs;
  __nv_bfloat16* base = nullptr;
  size_t total = 0;        // elements of one plane
  long long lo_off = 0;    // 0 in bf16 mode
  void request(__nv_bfloat16** p, size_t n) { reqs.push_back({p, (n + 511) / 512 * 512}); }   // 1 KB granules (TMA alignment)
  cudaError_t finalize(bool split) {
    total = 0;
    for (auto& r : reqs) total += r.second;
    total += 512;
    const size_t bytes = total * sizeof(__nv_bfloat16) * (split ? 2 : 1);
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) return e;
    e = cudaMemset(q, 0, bytes);
    if (e != cudaSuccess) { cudaFree(q); return e; }
    base = static_cast<__nv_bfloat16*>(q);
    size_t off = 0;
    for (auto& r : reqs) { *r.first = base + off; off += r.second; }
    lo_off = split ? (long long)total : 0;
    return cudaSuccess;
  }
};
struct PlanLoScope {   // plans built inside the scope get the engine's residual-plane offset (plan_gemm)
  gm_ctx* c;
  PlanLoScope(gm_ctx* c_, long long lo) : c(c_) { c->plan_lo = lo; }
  ~PlanLoScope() { c->plan_lo = 0; }
};

// ------------------------------------------------------------------ GAN engine
struct NetLayout {
  int in, hid, out;
  int off_w1, off_b1, off_w2, off_b2, total;
  void init(int in_, int hid_, int out_) {
    in = in_; hid = hid_; out = out_;
    off_w1 = 0; off_b1 = hid * in; off_w2 = off_b1 + hid; off_b2 = off_w2 + out * hid; total = off_b2 + out;
  }
};

struct StepPlans {
  GemmPlan g1, g2, d1_d, d1_g, d1_x, dw1d, dx, dw2g, dhg, dw1g, gp_v, gp_t;
  GemmPlan q1, q2, gq2, dhq, gq1, dfq;   // InfoGAN Q head
  GemmPlan be_enc_d, be_dec_d, be_gwd, be_de_d, be_enc_g, be_dec_g, be_de_g, be_dxg;   // BEGAN autoencoder-discriminator
};

// Bayesian GAN (engine_bayes.inl): the generator GEMMs once per sample (pointer offsets into the stacked operand copies,
// noise, hidden and fake rows), D's over the real and every sample's fake rows at once
constexpr int kBganMaxSamples = 16;
struct BayesPlans {
  GemmPlan g1[kBganMaxSamples], g2[kBganMaxSamples], dw2g[kBganMaxSamples], dhg[kBganMaxSamples], dw1g[kBganMaxSamples];
  GemmPlan d1_d, dw1d, d1_g, dx;
};

struct gm_comm {
  gm_ctx* ctx = nullptr;
  int rank = 0, world = 1, nblocks = 0;
  long long nfloats = 0;
  void* base = nullptr;
  size_t flag_off = 0, stat_off = 0, sflag_off = 0;
  void* peer[kCommMaxWorld] = {};
  bool opened = false;
  unsigned long long seq = 0, seq_stats = 0;
  unsigned long long begun[2] = {0, 0};   // seq of a gm_gan_exchange_begin(net) whose finish half has not run yet (0: none)
};


struct CustomPlans {   // custom-loss path (engine_custom.inl): per-slot D forward / backward, G output kept in DA2
  GemmPlan d1[4], dw1[4], dx[4], g2;
  GemmPlan ae_enc[2], ae_dec[2], ae_gwd[2], ae_de[2];   // BEGAN: the autoencoder D on the real / fake row regions
};
// InfoGAN's per-call Q (engine_custom.inl): each of kQSlots calls keeps its input and hidden rows until its backward ran;
// the backward scratch (DINF, DHQ, the split-K partials PQ1 / PQ2) is the fused Q step's
constexpr int kQSlots = 2;
struct QCallBufs {
  __nv_bfloat16 *X = nullptr, *H = nullptr;   // [x | 1], [relu(h) | 1]
};
struct QCallPlans {
  GemmPlan q1[kQSlots], q2[kQSlots], gq2[kQSlots], dhq[kQSlots], gq1[kQSlots], dx[kQSlots];
};

struct gm_gan {
  gm_ctx* ctx;
  gm_gan_desc d;
  int X, H, Z, XP, HP, ZP, Bmax;
  NetLayout G, D;
  float* par[2] = {nullptr, nullptr};
  float* grd[2] = {nullptr, nullptr};
  float* am[2] = {nullptr, nullptr};
  float* av[2] = {nullptr, nullptr};
  // bf16 activations
  __nv_bfloat16 *Zb = nullptr, *Hg = nullptr, *Xall = nullptr, *Aall = nullptr, *DHall = nullptr, *DA2 = nullptr, *DHg = nullptr;
  // bf16 operand copies of the weight matrices
  __nv_bfloat16 *W1g_s = nullptr, *W2g_s = nullptr, *W2g_t = nullptr, *W1d_s = nullptr, *W1d_t = nullptr;
  float *slots = nullptr, *ds = nullptr, *scores = nullptr, *lossbuf = nullptr, *fisher = nullptr, *dw2p = nullptr;
  float* dw2sum = nullptr;       // [3][HP]: loss path, penalty T path, DRAGAN ds_gp path
  float *dw2p2 = nullptr, *dw2p3 = nullptr, *slots_v = nullptr, *coef = nullptr, *stats = nullptr;
  double *gp_part = nullptr, *mom_part = nullptr;
  // row regions of Xall/Aall/DHall: real, fake (, xhat, R).  Only DRAGAN has the xhat region: WGAN-GP's D layer is linear, so
  // the penalty's hidden pre-activation eps a(x) + (1-eps) a(G(z)) comes from the real / fake rows (gp_hat_kernel)
  int nreg = 2;
  // InfoGAN: auxiliary network Q (image -> hidden -> disc+cont codes), its own Adam state and a
  // SECOND Adam state for G (MI_optimizer spans G and Q, src/info_gan.py:146-148)
  NetLayout Qn;
  int q_out = 0;
  float *parQ = nullptr, *grdQ = nullptr, *amQ = nullptr, *avQ = nullptr, *amG2 = nullptr, *avG2 = nullptr;
  __nv_bfloat16 *Wq1_s = nullptr, *Wq1_t = nullptr, *Wq2_s = nullptr, *Wq2_t = nullptr, *HQ = nullptr, *DINF = nullptr, *DHQ = nullptr;
  float *INF = nullptr, *PQ1 = nullptr, *PQ2 = nullptr;
  double* q_part = nullptr;
  // BEGAN: D is an autoencoder x -> h -> x (src/be_gan.py:63-76)
  __nv_bfloat16 *Wd_s = nullptr, *Wd_t = nullptr, *DR = nullptr, *BT = nullptr;
  float *slots_r = nullptr, *be_state = nullptr, *PWd = nullptr;
  double* be_part = nullptr;
  double* loss_part = nullptr;   // 3 x [loss_blocks][4]
  unsigned int* loss_done = nullptr;
  int loss_blocks = 0;
  float *PD = nullptr, *PG2 = nullptr, *PG1 = nullptr;
  int dh_blocks = 0, dh_rows_per_iter = 0, dh_threads = 0;
  int max_splits = 0;
  int last_rows = 0;
  int region_rows = 0;   // rows per region of Xall/Aall/DHall (3 regions)
  gm_comm* comm = nullptr;   // attached communicator: batch statistics run over the global batch
  // device-step mode (CUDA-graph replay of the step): [0] Adam steps of G, [1] Adam steps of D, [2] train_G calls, [3] train_D calls
  unsigned long long* dstep = nullptr;
  bool dev_step = false;
  int staged_batch = 0;      // > 0: gm_gan_d_stage already staged this many real rows for the next gm_gan_d_grad
  gm_loss_consts lc = {10.f, 1.f, 1.f, 0.f, 1.f, 1.f};   // reference defaults: src/w_gp_gan.py:177, src/dra_gan.py:174, src/ls_gan.py:173,197
  long long pool_n = 0;      // on-device batch sampling over a resident pool of pool_n images (gm_gan_set_sampler)
  uint64_t pool_seed = 0;
  // lazy gradients: *_grad leaves the split-K partials, gm_gan_apply gathers + updates in one kernel
  bool lazy = false;
  bool pend[2] = {false, false};
  GradSegs pend_segs[2];
  std::map<int, StepPlans> plans;
  std::map<int, CustomPlans> cplans;
  QCallBufs qs[kQSlots];     // per-call Q buffers, allocated on the first per-call Q entry
  bool qs_ready = false;
  std::map<int, QCallPlans> qplans;
  std::vector<void*> allocs;
  BfArena arena;
  long long lo = 0;          // arena.lo_off: > 0 in split-operand mode
  // Bayes mode (gm_bgan_create): nsamp > 0 generator samples, stacked in G's flat block g_stride floats apart (a multiple
  // of 4: every sample starts on 16 bytes).  Only the gm_bgan_* entries and the shared ones (bind, sync_shadows,
  // param_count, set_sampler, discriminate, debug_read) serve such an engine.
  int nsamp = 0, g_stride = 0;
  std::map<int, BayesPlans> bplans;
};

// The point-estimate entries (Adam, the fused and per-call steps, data parallelism, device steps, Q and BEGAN) refuse a
// Bayes-mode engine before anything is launched
static int refuse_bayes(gm_gan* g, const char* what) {
  return fail(g->ctx, GM_ERR_ARG, "%s cannot serve a Bayesian GAN engine (use the gm_bgan_* entries)", what);
}
#define REFUSE_BAYES(g, what) do { if ((g) && (g)->nsamp) return refuse_bayes((g), (what)); } while (0)
static int bgan_sync_shadows(gm_gan* g, int net, cudaStream_t s);

// Zeroed device buffers of an engine (gm_gan, gm_vae), freed by its destroy.  bf16 buffers come from the engine's arena
// (finalised at the end of create) unless T is given explicitly, as for the VAE's per-call slot buffers.
template <typename E>
static int dev_alloc(E* g, __nv_bfloat16** p, size_t count) {
  g->arena.request(p, count);
  return GM_OK;
}

template <typename T, typename E>
static int dev_alloc(E* g, T** p, size_t count) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T));
  if (e != cudaSuccess) return fail(g->ctx, GM_ERR_CUDA, "cudaMalloc(%zu) failed: %s", count * sizeof(T), cudaGetErrorString(e));
  g->allocs.push_back(q);
  e = cudaMemset(q, 0, count * sizeof(T));
  if (e != cudaSuccess) return fail(g->ctx, GM_ERR_CUDA, "cudaMemset failed: %s", cudaGetErrorString(e));
  *p = static_cast<T*>(q);
  return GM_OK;
}

extern "C" int gm_gan_destroy(gm_gan* g) {
  if (!g) return GM_OK;
  for (void* p : g->allocs) cudaFree(p);
  delete g;
  return GM_OK;
}

extern "C" int gm_gan_create(gm_ctx* c, const gm_gan_desc* d, gm_gan** out) {
  if (!c || !d || !out) return GM_ERR_ARG;
  *out = nullptr;
  if (!c->encode) return fail(c, GM_ERR_STATE, "context has no device");
  if (d->image_size % 16 || d->hidden_dim % 16 || d->image_size <= 0 || d->hidden_dim <= 0 || d->z_dim <= 0)
    return fail(c, GM_ERR_ARG, "image_size and hidden_dim must be positive multiples of 16 (got %d, %d, z=%d)",
                d->image_size, d->hidden_dim, d->z_dim);
  if (d->max_batch <= 0) return fail(c, GM_ERR_ARG, "max_batch must be positive (got %d)", d->max_batch);
  if (d->dtype_mode != GM_PREC_BF16 && d->dtype_mode != GM_PREC_SPLIT) return fail(c, GM_ERR_ARG, "unknown dtype_mode %d", d->dtype_mode);
  if (d->hidden_dim + 1 > 448 || d->z_dim + 1 > 448)
    return fail(c, GM_ERR_UNSUPPORTED, "hidden_dim <= 447 and generator input width <= 447 in this build (got %d, %d)", d->hidden_dim, d->z_dim);
  gm_gan* g = new gm_gan();
  g->ctx = c;
  g->d = *d;
  g->X = d->image_size; g->H = d->hidden_dim; g->Z = d->z_dim; g->Bmax = d->max_batch;
  g->XP = rup(g->X + 1, 16);
  g->HP = rup(g->H + 1, 16);
  g->ZP = rup(g->Z + 1, 64);
  g->G.init(g->Z, g->H, g->X);
  g->D.init(g->X, g->H, d->variant == GM_BEGAN ? g->X : 1);
  g->region_rows = g->Bmax;
  g->nreg = d->variant == GM_WGP ? 3 : (d->variant == GM_DRA ? 4 : 2);
  // WGAN-GP always runs gp_hat_kernel: every hidden width this function accepts (hidden_dim + 1 <= 448) must fit its lanes
  static_assert(448 <= 64 * kGpHatGroups * 4, "gp_hat_kernel covers at most 64 * kGpHatGroups * 4 hidden columns");
  const size_t B = g->Bmax;
  const size_t NR = g->nreg;
  int rc = GM_OK;
#define TRY(x) do { rc = (x); if (rc) { gm_gan_destroy(g); return rc; } } while (0)
  TRY(dev_alloc(g, &g->Zb, B * g->ZP));
  TRY(dev_alloc(g, &g->Hg, B * g->HP));
  TRY(dev_alloc(g, &g->Xall, NR * B * g->XP));
  TRY(dev_alloc(g, &g->Aall, NR * B * g->HP));
  TRY(dev_alloc(g, &g->DHall, NR * B * g->HP));
  TRY(dev_alloc(g, &g->DA2, B * g->XP));
  TRY(dev_alloc(g, &g->DHg, B * g->HP));
  TRY(dev_alloc(g, &g->W1g_s, size_t(g->H) * g->ZP));
  TRY(dev_alloc(g, &g->W2g_s, size_t(g->X) * g->H));
  TRY(dev_alloc(g, &g->W2g_t, size_t(g->H) * g->X));
  TRY(dev_alloc(g, &g->W1d_s, size_t(g->H) * g->X));
  TRY(dev_alloc(g, &g->W1d_t, size_t(g->X) * g->H));
  const int nslots = 2 * cdiv(g->H, 208);
  TRY(dev_alloc(g, &g->slots, size_t(nslots) * NR * B));
  TRY(dev_alloc(g, &g->ds, NR * B));
  TRY(dev_alloc(g, &g->scores, NR * B));
  TRY(dev_alloc(g, &g->lossbuf, 16));
  TRY(dev_alloc(g, &g->fisher, 4));
  // dh kernel geometry
  const int groups = g->HP / 8;
  g->dh_rows_per_iter = 256 / groups > 0 ? 256 / groups : 1;
  g->dh_threads = groups * g->dh_rows_per_iter;
  g->dh_blocks = c->num_sms * 4;
  TRY(dev_alloc(g, &g->dw2p, size_t(g->dh_blocks) * g->HP));
  TRY(dev_alloc(g, &g->dw2sum, size_t(3) * g->HP));
  if (g->nreg > 2) {
    TRY(dev_alloc(g, &g->dw2p2, size_t(g->dh_blocks) * g->HP));
    TRY(dev_alloc(g, &g->dw2p3, size_t(g->dh_blocks) * g->HP));
    TRY(dev_alloc(g, &g->slots_v, size_t(2 * cdiv(g->X, 208)) * B));
    TRY(dev_alloc(g, &g->coef, B));
    TRY(dev_alloc(g, &g->stats, 4));
    TRY(dev_alloc(g, &g->gp_part, size_t(c->num_sms) * 2 * 4));
    TRY(dev_alloc(g, &g->mom_part, size_t(c->num_sms) * 2 * 2));
  }
  g->loss_blocks = c->num_sms * 2;
  TRY(dev_alloc(g, &g->loss_part, size_t(3) * g->loss_blocks * 4));
  TRY(dev_alloc(g, &g->loss_done, 4));
  // split-K partials
  g->max_splits = c->num_sms;
  const int sp_d = c->num_sms / cdiv(g->X + 1, BM) > 0 ? c->num_sms / cdiv(g->X + 1, BM) : 1;
  const int sp_g2 = c->num_sms / cdiv(g->X, BM) > 0 ? c->num_sms / cdiv(g->X, BM) : 1;
  const int sp_g1 = c->num_sms / cdiv(g->H, BM) > 0 ? c->num_sms / cdiv(g->H, BM) : 1;
  TRY(dev_alloc(g, &g->PD, size_t(sp_d) * g->H * (cdiv(g->X + 1, BM) * BM)));
  TRY(dev_alloc(g, &g->PG2, size_t(sp_g2) * g->X * rup(g->H + 1, 64)));
  TRY(dev_alloc(g, &g->PG1, size_t(sp_g1) * g->H * 64 * cdiv(g->Z + 1, 64)));
  if (d->variant == GM_BEGAN) {
    TRY(dev_alloc(g, &g->Wd_s, size_t(g->X) * g->H));
    TRY(dev_alloc(g, &g->Wd_t, size_t(g->H) * g->X));
    TRY(dev_alloc(g, &g->DR, 2 * B * g->XP));
    TRY(dev_alloc(g, &g->BT, B * g->XP));
    TRY(dev_alloc(g, &g->slots_r, size_t(2 * cdiv(g->X, 208)) * 2 * B));
    TRY(dev_alloc(g, &g->be_state, 16));
    TRY(dev_alloc(g, &g->PWd, size_t(sp_g2) * g->X * rup(g->H + 1, 64)));
    TRY(dev_alloc(g, &g->be_part, size_t(c->num_sms) * 2 * 2));
  }
  if (d->variant == GM_INFO) {
    g->q_out = 20;   // 10 categorical logits + 10 continuous codes (src/info_gan.py:403-407)
    g->Qn.init(g->X, g->H, g->q_out);
    TRY(dev_alloc(g, &g->Wq1_s, size_t(g->H) * g->X));
    TRY(dev_alloc(g, &g->Wq1_t, size_t(g->X) * g->H));
    TRY(dev_alloc(g, &g->Wq2_s, size_t(64) * g->H));
    TRY(dev_alloc(g, &g->Wq2_t, size_t(g->H) * 64));
    TRY(dev_alloc(g, &g->HQ, B * g->HP));
    TRY(dev_alloc(g, &g->DINF, B * 64));
    TRY(dev_alloc(g, &g->DHQ, B * g->HP));
    TRY(dev_alloc(g, &g->INF, B * 32));
    TRY(dev_alloc(g, &g->PQ1, size_t(sp_g1) * g->H * 896));
    TRY(dev_alloc(g, &g->PQ2, size_t(c->num_sms) * 64 * 448));
    TRY(dev_alloc(g, &g->q_part, size_t(c->num_sms) * 2 * 4));
  }
  {
    cudaError_t e = g->arena.finalize(d->dtype_mode == GM_PREC_SPLIT);
    if (e != cudaSuccess) { rc = fail(c, GM_ERR_CUDA, "bf16 arena allocation failed: %s", cudaGetErrorString(e)); gm_gan_destroy(g); return rc; }
    g->allocs.push_back(g->arena.base);
    g->lo = g->arena.lo_off;
  }
#undef TRY
  *out = g;
  return GM_OK;
}

extern "C" int gm_gan_param_count(const gm_gan* g, int net) {
  if (!g) return GM_ERR_ARG;
  if (net == GM_NET_G && g->nsamp) return g->nsamp * g->g_stride;   // the stacked samples (engine_bayes.inl)
  return net == GM_NET_G ? g->G.total : g->D.total;
}

extern "C" int gm_gan_bind(gm_gan* g, int net, float* p, float* gr, float* m, float* v) {
  if (!g || net < 0 || net > 1 || !p || !gr) return g ? fail(g->ctx, GM_ERR_ARG, "gm_gan_bind: bad argument") : GM_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(p) & 15)
    return fail(g->ctx, GM_ERR_ARG, "parameter buffer must be 16-byte aligned");
  g->par[net] = p; g->grd[net] = gr; g->am[net] = m; g->av[net] = v;
  g->plans.clear(); g->cplans.clear(); g->qplans.clear(); g->bplans.clear();
  return GM_OK;
}

static void adam_segs(gm_gan* g, int net, AdamParams& a) {
  a.lo_off = g->lo;
  if (net == GM_NET_G) {
    a.total = g->G.total;
    a.nseg = 2;
    a.seg[0] = {g->G.off_w1, g->H * g->Z, g->Z, g->W1g_s, g->ZP, nullptr, 0};
    a.seg[1] = {g->G.off_w2, g->X * g->H, g->H, g->W2g_s, g->H, g->W2g_t, g->X};
  } else {
    a.total = g->D.total;
    a.nseg = 1;
    a.seg[0] = {g->D.off_w1, g->H * g->X, g->X, g->W1d_s, g->X, g->W1d_t, g->H};
    if (g->d.variant == GM_BEGAN) {   // decoder weight [x, h]: K-major copy + transpose
      a.nseg = 2;
      a.seg[1] = {g->D.off_w2, g->X * g->H, g->H, g->Wd_s, g->H, g->Wd_t, g->X};
      a.lr_scale = g->be_state + 7;
    }
  }
  if (net == GM_NET_G && g->d.variant == GM_BEGAN) a.lr_scale = g->be_state + 7;
}

extern "C" int gm_gan_sync_shadows(gm_gan* g, int net, gm_stream stream) {
  if (!g || net < 0 || net > 1) return GM_ERR_ARG;
  if (!g->par[net]) return fail(g->ctx, GM_ERR_STATE, "net %d not bound", net);
  if (g->nsamp) return bgan_sync_shadows(g, net, static_cast<cudaStream_t>(stream));
  AdamParams a;
  memset(&a, 0, sizeof a);
  a.p = g->par[net];
  a.update = 0;
  adam_segs(g, net, a);
  return launch(g->ctx, "adam_kernel", adam_kernel, cdiv(a.total, 256), 256, 0, static_cast<cudaStream_t>(stream), a);
}

static int flush_pending(gm_gan* g, cudaStream_t s);
static int bump_step(gm_gan* g, int which, cudaStream_t s) {
  if (!g->dev_step) return GM_OK;
  return launch(g->ctx, "bump_step_kernel", bump_step_kernel, 1, 32, 0, s, g->dstep + which);
}


extern "C" int gm_gan_apply(gm_gan* g, int net, const gm_adam_hp* hp, int step, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_apply");
  if (!g || net < 0 || net > 1 || !hp || step <= 0) return g ? fail(g->ctx, GM_ERR_ARG, "gm_gan_apply: bad argument") : GM_ERR_ARG;
  if (!g->par[net] || !g->am[net] || !g->av[net]) return fail(g->ctx, GM_ERR_STATE, "net %d not fully bound", net);
  AdamParams a;
  memset(&a, 0, sizeof a);
  a.p = g->par[net]; a.g = g->grd[net]; a.m = g->am[net]; a.v = g->av[net];
  fill_adam(a, hp, step);
  adam_segs(g, net, a);
  if (g->pend[net]) {   // lazy gradients: gather from the partials inside the update
    a.gather = 1; a.gout = g->grd[net]; a.gsegs = g->pend_segs[net];
    g->pend[net] = false;
  }
  if (g->dev_step) a.step_ptr = g->dstep + net;   // bias corrections from the device counter (`step` is ignored)
  const int rc = launch(g->ctx, "adam_kernel", adam_kernel, cdiv(a.total, 256), 256, 0, static_cast<cudaStream_t>(stream), a);
  return rc ? rc : bump_step(g, net, static_cast<cudaStream_t>(stream));
}

extern "C" int gm_gan_set_lazy_grads(gm_gan* g, int on, gm_stream stream) {
  if (!g) return GM_ERR_ARG;
  int rc;
  if (on) REFUSE_BAYES(g, "gm_gan_set_lazy_grads");
  if (!on && (rc = flush_pending(g, static_cast<cudaStream_t>(stream)))) return rc;
  g->lazy = on != 0;
  return GM_OK;
}
extern "C" int gm_gan_materialize_grads(gm_gan* g, gm_stream stream) {
  if (!g) return GM_ERR_ARG;
  return flush_pending(g, static_cast<cudaStream_t>(stream));
}

// epilogue setters for a plan fresh from plan_gemm (every other field zero)
static void set_bf16_epi(GemmParams& p, __nv_bfloat16* out, int ldo, int out_cols, int pad_one, const float* bias, int act) {
  p.epi = EPI_BF16; p.out = out; p.ldo = ldo; p.out_cols = out_cols; p.pad_one = pad_one; p.bias = bias; p.act = act;
}
static void set_f32_epi(GemmParams& p, float* part, int ldp, long long part_stride, int transpose, const float* bias) {
  p.epi = EPI_F32; p.part = part; p.ldp = ldp; p.part_stride = part_stride; p.transpose = transpose; p.bias = bias;
}
static void set_row_dot(GemmParams& p, int dot, const float* w, float* out, int ld) {
  p.dot = dot; p.dot_w = w; p.dot_out = out; p.dot_ld = ld;
}

static int build_plans(gm_gan* g, int B, StepPlans** out) {
  auto it = g->plans.find(B);
  if (it != g->plans.end()) { *out = &it->second; return GM_OK; }
  gm_ctx* c = g->ctx;
  PlanLoScope lo_scope(c, g->lo);
  StepPlans sp;
  const int X = g->X, H = g->H, Z = g->Z, XP = g->XP, HP = g->HP, ZP = g->ZP;
  const float* pG = g->par[GM_NET_G];
  const float* pD = g->par[GM_NET_D];
  __nv_bfloat16* Xfake = g->Xall + size_t(B) * XP;
  __nv_bfloat16* Afake = g->Aall + size_t(B) * HP;
  __nv_bfloat16* DHfake = g->DHall + size_t(B) * HP;
  const int slot_ld = g->nreg * g->Bmax;
  int rc;
  // G layer 1: Hg = relu(Zb W1g^T + b1g), ones column at H
  if ((rc = plan_gemm(c, &sp.g1, 0, B, H, rup(Z, 16), g->Zb, ZP, g->W1g_s, ZP, HP, 1))) return rc;
  set_bf16_epi(sp.g1.p, g->Hg, HP, HP, 1, pG + g->G.off_b1, ACT_RELU);
  sp.g1.flops = 2.0 * B * H * Z;
  // G layer 2: fake = sigmoid(Hg W2g^T + b2g) -> fake rows of Xall, ones column at X
  if ((rc = plan_gemm(c, &sp.g2, 0, B, X, H, g->Hg, HP, g->W2g_s, H, XP, 1))) return rc;
  set_bf16_epi(sp.g2.p, Xfake, XP, XP, 1, pG + g->G.off_b2, ACT_SIGMOID);
  // D layer 1 (+ fused 400->1 row-dot) on [real; fake] (D step) and on fake only (G step)
  const int nfwd = g->d.variant == GM_DRA ? 3 : 2;      // DRAGAN also scores the interpolated rows
  if ((rc = plan_gemm(c, &sp.d1_d, 0, nfwd * B, H, X, g->Xall, XP, g->W1d_s, X, H, 1))) return rc;
  set_bf16_epi(sp.d1_d.p, g->Aall, HP, H, 0, pD + g->D.off_b1, ACT_RELU);
  // WGAN-GP: the real / fake rows keep their PRE-activations (ReLU inside the row-dot and in dh_kernel): gp_hat_kernel
  // forms a_hat = eps a(x) + (1-eps) a(G(z)) from them
  set_row_dot(sp.d1_d.p, g->d.variant == GM_WGP ? DOT_W_PRE : DOT_W, pD + g->D.off_w2, g->slots, slot_ld);
  if ((rc = plan_gemm(c, &sp.d1_g, 0, B, H, X, Xfake, XP, g->W1d_s, X, H, 1))) return rc;
  set_bf16_epi(sp.d1_g.p, Afake, HP, H, 0, pD + g->D.off_b1, ACT_RELU);
  // the G step does not update D: instead of the hidden activations it stores M = w2 * 1[a1 > 0]
  // (what dL/dfake = ds * (M W1d) needs) and so skips the dh pass over the fake rows
  set_row_dot(sp.d1_g.p, g->d.variant != GM_BEGAN ? DOT_W_MASK : DOT_W, pD + g->D.off_w2, g->slots + B, slot_ld);
  // D layer 1 on the real rows only (inference: gm_gan_discriminate)
  if ((rc = plan_gemm(c, &sp.d1_x, 0, B, H, X, g->Xall, XP, g->W1d_s, X, H, 1))) return rc;
  set_bf16_epi(sp.d1_x.p, g->Aall, HP, H, 0, pD + g->D.off_b1, ACT_RELU);
  set_row_dot(sp.d1_x.p, DOT_W, pD + g->D.off_w2, g->slots, slot_ld);
  // dW1d^T (+ db1 row from the ones column): [X+1, H] = Xall^T DHall over 2B rows
  if ((rc = plan_gemm(c, &sp.dw1d, 1, X + 1, H, g->nreg * B, g->Xall, XP, g->DHall, HP, H, g->max_splits))) return rc;
  {
    const int ldp = sp.dw1d.p.m_tiles * BM;
    set_f32_epi(sp.dw1d.p, g->PD, ldp, (long long)H * ldp, 1, nullptr);
    sp.dw1d.flops = 2.0 * X * H * (double(g->nreg) * B);
  }
  if (g->nreg > 2) {
    // gradient penalty (SURVEY A.2): V = U W1 (+ row sum of squares), T = (R W1^T) * 1[a_hat > 0]
    const size_t rreg = size_t(g->nreg - 1) * B;
    __nv_bfloat16* Rrows = g->Xall + rreg * XP;
    if ((rc = plan_gemm(c, &sp.gp_v, 0, B, X, H, g->DHall + rreg * HP, HP, g->W1d_t, H, X, 1))) return rc;
    set_bf16_epi(sp.gp_v.p, Rrows, XP, X, 0, nullptr, ACT_NONE);
    set_row_dot(sp.gp_v.p, DOT_SQ, nullptr, g->slots_v, g->Bmax);
    if ((rc = plan_gemm(c, &sp.gp_t, 0, B, H, X, Rrows, XP, g->W1d_s, X, H, 1))) return rc;
    set_bf16_epi(sp.gp_t.p, g->DHg, HP, H, 0, nullptr, ACT_NONE);
    // T = coef * (V W1^T) * relu'(a_hat): the per-row factor of R = coef V is applied in the epilogue (R itself is never
    // formed; dGP/dW1 = (coef U)^T V uses the scaled U rows instead), the mask comes from the U rows (nonzero <=> active)
    sp.gp_t.p.aux = g->DHall + rreg * HP; sp.gp_t.p.ld_aux = HP; sp.gp_t.p.aux_mode = AUX_NONZERO_MASK;
    sp.gp_t.p.row_vec = g->coef;
  }
  // dX of D w.r.t. fake, times sigmoid'(fake): DA2 = (DHfake W1d) * fake(1-fake)
  if ((rc = plan_gemm(c, &sp.dx, 0, B, X, H, Afake, HP, g->W1d_t, H, X, 1))) return rc;
  set_bf16_epi(sp.dx.p, g->DA2, XP, X, 0, nullptr, ACT_NONE);
  sp.dx.p.aux = Xfake; sp.dx.p.ld_aux = XP; sp.dx.p.aux_mode = AUX_SIGMOID_GRAD;
  sp.dx.p.row_vec = g->ds + B;     // dL/ds of the fake rows (launch_loss, G step)
  // [dW2g | db2g] = DA2^T [Hg | 1]
  if ((rc = plan_gemm(c, &sp.dw2g, 1, X, H + 1, B, g->DA2, XP, g->Hg, HP, H + 1, g->max_splits))) return rc;
  set_f32_epi(sp.dw2g.p, g->PG2, rup(H + 1, 64), (long long)X * rup(H + 1, 64), 0, nullptr);
  sp.dw2g.flops = 2.0 * X * H * B;
  // DHg = (DA2 W2g) * 1[Hg > 0]
  if ((rc = plan_gemm(c, &sp.dhg, 0, B, H, X, g->DA2, XP, g->W2g_t, X, H, 1))) return rc;
  set_bf16_epi(sp.dhg.p, g->DHg, HP, H, 0, nullptr, ACT_NONE);
  sp.dhg.p.aux = g->Hg; sp.dhg.p.ld_aux = HP; sp.dhg.p.aux_mode = AUX_RELU_MASK;
  // [dW1g | db1g] = DHg^T [Zb | 1]
  if ((rc = plan_gemm(c, &sp.dw1g, 1, H, Z + 1, B, g->DHg, HP, g->Zb, ZP, Z + 1, g->max_splits))) return rc;
  set_f32_epi(sp.dw1g.p, g->PG1, rup(Z + 1, 64), (long long)H * rup(Z + 1, 64), 0, nullptr);
  sp.dw1g.flops = 2.0 * H * Z * B;
  if (g->d.variant == GM_BEGAN) {
    const int slr = 2 * g->Bmax;
    auto l1 = [&](GemmPlan& pl, const __nv_bfloat16* aux, float* slots, const float* rs, int split) {
      pl.p.aux = aux; pl.p.ld_aux = XP; pl.p.aux_mode = AUX_L1; pl.p.dot_out = slots; pl.p.dot_ld = slr;
      pl.p.row_scale = rs; pl.p.row_split = split;
    };
    // D step: encode / decode real and fake rows together, L1 error + its sign fused in the decoder epilogue
    if ((rc = plan_gemm(c, &sp.be_enc_d, 0, 2 * B, H, X, g->Xall, XP, g->W1d_s, X, HP, 1))) return rc;
    set_bf16_epi(sp.be_enc_d.p, g->Aall, HP, HP, 1, pD + g->D.off_b1, ACT_RELU);
    if ((rc = plan_gemm(c, &sp.be_dec_d, 0, 2 * B, X, H, g->Aall, HP, g->Wd_s, H, X, 1))) return rc;
    set_bf16_epi(sp.be_dec_d.p, g->DR, XP, X, 0, pD + g->D.off_b2, ACT_NONE);
    l1(sp.be_dec_d, g->Xall, g->slots_r, g->be_state + 1, B);
    if ((rc = plan_gemm(c, &sp.be_gwd, 1, X, H + 1, 2 * B, g->DR, XP, g->Aall, HP, H + 1, g->max_splits))) return rc;
    set_f32_epi(sp.be_gwd.p, g->PWd, rup(H + 1, 64), (long long)X * rup(H + 1, 64), 0, nullptr);
    sp.be_gwd.flops = 2.0 * X * H * 2.0 * B;
    if ((rc = plan_gemm(c, &sp.be_de_d, 0, 2 * B, H, X, g->DR, XP, g->Wd_t, X, H, 1))) return rc;
    set_bf16_epi(sp.be_de_d.p, g->DHall, HP, H, 0, nullptr, ACT_NONE);
    sp.be_de_d.p.aux = g->Aall; sp.be_de_d.p.ld_aux = HP; sp.be_de_d.p.aux_mode = AUX_RELU_MASK;
    // G step: the same on the fake rows only, then back through the encoder to the images
    if ((rc = plan_gemm(c, &sp.be_enc_g, 0, B, H, X, Xfake, XP, g->W1d_s, X, HP, 1))) return rc;
    set_bf16_epi(sp.be_enc_g.p, Afake, HP, HP, 1, pD + g->D.off_b1, ACT_RELU);
    if ((rc = plan_gemm(c, &sp.be_dec_g, 0, B, X, H, Afake, HP, g->Wd_s, H, X, 1))) return rc;
    set_bf16_epi(sp.be_dec_g.p, g->DR + size_t(B) * XP, XP, X, 0, pD + g->D.off_b2, ACT_NONE);
    l1(sp.be_dec_g, Xfake, g->slots_r + B, g->be_state + 8, 0);
    if ((rc = plan_gemm(c, &sp.be_de_g, 0, B, H, X, g->DR + size_t(B) * XP, XP, g->Wd_t, X, H, 1))) return rc;
    set_bf16_epi(sp.be_de_g.p, DHfake, HP, H, 0, nullptr, ACT_NONE);
    sp.be_de_g.p.aux = Afake; sp.be_de_g.p.ld_aux = HP; sp.be_de_g.p.aux_mode = AUX_RELU_MASK;
    if ((rc = plan_gemm(c, &sp.be_dxg, 0, B, X, H, DHfake, HP, g->W1d_t, H, X, 1))) return rc;
    set_bf16_epi(sp.be_dxg.p, g->BT, XP, X, 0, nullptr, ACT_NONE);
  }
  if (g->d.variant == GM_INFO && g->parQ != nullptr) {
    const float* pQ = g->parQ;
    const int QO = g->q_out;
    if ((rc = plan_gemm(c, &sp.q1, 0, B, H, X, Xfake, XP, g->Wq1_s, X, HP, 1))) return rc;
    set_bf16_epi(sp.q1.p, g->HQ, HP, HP, 1, pQ + g->Qn.off_b1, ACT_RELU);
    if ((rc = plan_gemm(c, &sp.q2, 0, B, QO, H, g->HQ, HP, g->Wq2_s, H, QO, 1))) return rc;
    set_f32_epi(sp.q2.p, g->INF, 32, 0, 0, pQ + g->Qn.off_b2);
    if ((rc = plan_gemm(c, &sp.gq2, 1, QO, H + 1, B, g->DINF, 64, g->HQ, HP, H + 1, g->max_splits))) return rc;
    set_f32_epi(sp.gq2.p, g->PQ2, 448, (long long)64 * 448, 0, nullptr);
    sp.gq2.flops = 2.0 * QO * H * B;
    if ((rc = plan_gemm(c, &sp.dhq, 0, B, H, rup(QO, 16), g->DINF, 64, g->Wq2_t, 64, H, 1))) return rc;
    set_bf16_epi(sp.dhq.p, g->DHQ, HP, H, 0, nullptr, ACT_NONE);
    sp.dhq.p.aux = g->HQ; sp.dhq.p.ld_aux = HP; sp.dhq.p.aux_mode = AUX_RELU_MASK;
    sp.dhq.flops = 2.0 * B * H * QO;
    if ((rc = plan_gemm(c, &sp.gq1, 1, H, X + 1, B, g->DHQ, HP, Xfake, XP, X + 1, g->max_splits))) return rc;
    set_f32_epi(sp.gq1.p, g->PQ1, rup(X + 1, 64), (long long)H * rup(X + 1, 64), 0, nullptr);
    sp.gq1.flops = 2.0 * H * X * B;
    if ((rc = plan_gemm(c, &sp.dfq, 0, B, X, H, g->DHQ, HP, g->Wq1_t, H, X, 1))) return rc;
    set_bf16_epi(sp.dfq.p, g->DA2, XP, X, 0, nullptr, ACT_NONE);
    sp.dfq.p.aux = Xfake; sp.dfq.p.ld_aux = XP; sp.dfq.p.aux_mode = AUX_SIGMOID_GRAD;
  }
  g->plans[B] = sp;
  *out = &g->plans[B];
  return GM_OK;
}

static int check_step_args(gm_gan* g, int batch) {
  if (!g) return GM_ERR_ARG;
  if (batch <= 0 || batch > g->Bmax)
    return fail(g->ctx, GM_ERR_ARG, "batch must be in (0, %d] (got %d)", g->Bmax, batch);
  if (!g->par[0] || !g->par[1] || !g->grd[0] || !g->grd[1]) return fail(g->ctx, GM_ERR_STATE, "bind both nets first");
  return GM_OK;
}

static int run_generator(gm_gan* g, StepPlans* sp, int B, const float* noise, uint64_t seed, uint64_t stream_id, cudaStream_t s,
                         const unsigned long long* step_ptr = nullptr) {
  int rc;
  if ((rc = launch(g->ctx, "stage_noise_kernel", stage_noise_kernel, cdiv(B * ((g->Z + 8) / 8), 256), 256, 0, s, noise, g->Zb, B, g->Z, g->ZP, seed, stream_id, g->lo, step_ptr))) return rc;
  if ((rc = launch_plan(g->ctx, sp->g1, s))) return rc;
  return launch_plan(g->ctx, sp->g2, s);
}

// replace per-block partial sums by their sum over all ranks (no-op without an attached communicator)
static int exchange_stats(gm_gan* g, double* part, int nblk, int stride, int nvals, cudaStream_t s) {
  gm_comm* m = g->comm;
  if (!m || m->world <= 1) return GM_OK;
  CommStats cs;
  memset(&cs, 0, sizeof cs);
  for (int r = 0; r < m->world; ++r) {
    cs.v[r] = reinterpret_cast<double*>(static_cast<char*>(m->peer[r]) + m->stat_off);
    cs.f[r] = reinterpret_cast<unsigned long long*>(static_cast<char*>(m->peer[r]) + m->sflag_off);
  }
  cs.rank = m->rank; cs.world = m->world; cs.seq = ++m->seq_stats;
  return launch(g->ctx, "stats_exchange_kernel", stats_exchange_kernel, 1, 256, 0, s, part, nblk, stride, nvals, cs);
}
static int stat_world(const gm_gan* g) { return (g->comm && g->comm->world > 1) ? g->comm->world : 1; }

static int launch_loss(gm_gan* g, int B, int g_step, float inv_b, cudaStream_t s) {
  LossParams lp;
  lp.slots = g->slots + (g_step ? B : 0);
  lp.nslots = 2 * cdiv(g->H, 208);
  lp.slot_ld = g->nreg * g->Bmax;
  lp.b2 = g->par[GM_NET_D] + g->D.off_b2;
  lp.Bstat = B * stat_world(g);
  lp.done = g->loss_done;
  lp.B = B; lp.g_step = g_step; lp.variant = g->d.variant; lp.out_act = g->d.d_out_act; lp.inv_b = inv_b;
  lp.ds = g->ds + (g_step ? B : 0);
  lp.d_out = g->scores + (g_step ? B : 0);
  lp.loss = g->lossbuf;
  lp.fisher = g->fisher;
  lp.ls_a = g->lc.ls_a; lp.ls_b = g->lc.ls_b; lp.ls_c = g->lc.ls_c;
  const int rows = g_step ? B : 2 * B;
  lp.nblk = cdiv(rows, kLossThreads) < g->loss_blocks ? cdiv(rows, kLossThreads) : g->loss_blocks;
  lp.partA = g->loss_part;
  lp.partB = g->loss_part + size_t(g->loss_blocks) * 4;
  lp.partR = g->loss_part + size_t(g->loss_blocks) * 8;
  const int v = g->d.variant;
  int rc;
  if (!g_step && (v == V_RA || v == V_FISHER)) {
    if ((rc = launch(g->ctx, "loss_pass_kernel<0>", loss_pass_kernel<0>, lp.nblk, kLossThreads, 0, s, lp))) return rc;
    if ((rc = exchange_stats(g, lp.partA, lp.nblk, 4, 4, s))) return rc;       // sum d, d^2 per branch over all ranks
    if (v == V_RA) {
      if ((rc = launch(g->ctx, "loss_pass_kernel<1>", loss_pass_kernel<1>, lp.nblk, kLossThreads, 0, s, lp))) return rc;
      if ((rc = exchange_stats(g, lp.partB, lp.nblk, 4, 1, s))) return rc;     // sum q(1-q)/(q+eps) over all ranks' real rows
    }
  }
  return launch(g->ctx, "loss_pass_kernel<2>", loss_pass_kernel<2>, lp.nblk, kLossThreads, 0, s, lp);   // its last block writes loss[0..1]
}

// The flat gradient of `net` from its partials: now (finalize kernel), or - with lazy gradients -
// inside the next gm_gan_apply(net).
static int emit_grads(gm_gan* g, int net, const GradSegs& gs, cudaStream_t s, bool force_now = false) {
  if (g->lazy && !force_now) {
    g->pend_segs[net] = gs;
    g->pend[net] = true;
    return GM_OK;
  }
  const int rc = launch(g->ctx, "finalize_grads_kernel", finalize_grads_kernel, cdiv(gs.total, 256), 256, 0, s, gs, g->grd[net]);
  if (!rc) g->pend[net] = false;
  return rc;
}
// Partials are only valid until the next *_grad call reuses the buffers: form pending gradients first.
static int flush_pending(gm_gan* g, cudaStream_t s) {
  int rc;
  for (int net = 0; net < 2; ++net)
    if (g->pend[net] && (rc = emit_grads(g, net, g->pend_segs[net], s, true))) return rc;
  return GM_OK;
}

// ---- BEGAN (src/be_gan.py:212-258): D = autoencoder, L1 reconstruction losses ----
static int began_finalize_g(gm_gan* g, StepPlans* sp, cudaStream_t s, bool force_now = false) {
  GradSegs gs;
  memset(&gs, 0, sizeof gs);
  const GemmParams& p2 = sp->dw2g.p;
  const GemmParams& p1 = sp->dw1g.p;
  gs.nseg = 4;
  gs.total = g->G.total;
  gs.s[0] = {g->G.off_w1, g->H * g->Z, 0, g->Z, p1.ldp, 0, p1.splits, p1.part_stride, g->PG1};
  gs.s[1] = {g->G.off_b1, g->H, 2, 0, p1.ldp, g->Z, p1.splits, p1.part_stride, g->PG1};
  gs.s[2] = {g->G.off_w2, g->X * g->H, 0, g->H, p2.ldp, 0, p2.splits, p2.part_stride, g->PG2};
  gs.s[3] = {g->G.off_b2, g->X, 2, 0, p2.ldp, g->H, p2.splits, p2.part_stride, g->PG2};
  return emit_grads(g, GM_NET_G, gs, s, force_now);
}

static int began_d_grad(gm_gan* g, StepPlans* sp, int B, float* loss_dev, cudaStream_t s) {
  gm_ctx* c = g->ctx;
  int rc;
  if ((rc = launch_plan(c, sp->be_enc_d, s))) return rc;
  if ((rc = launch_plan(c, sp->be_dec_d, s))) return rc;   // DR = scaled sign(D(.) - .), row L1 sums -> slots_r
  const int nb = c->num_sms;
  const int ns = 2 * cdiv(g->X, 208);
  if ((rc = launch(c, "vae_rowsum_kernel", vae_rowsum_kernel, nb, 256, 0, s, g->slots_r, ns, 2 * g->Bmax, B, g->be_part))) return rc;
  if ((rc = launch(c, "vae_rowsum_kernel", vae_rowsum_kernel, nb, 256, 0, s, g->slots_r + B, ns, 2 * g->Bmax, B, g->be_part + nb))) return rc;
  if ((rc = exchange_stats(g, g->be_part, nb, 1, 1, s))) return rc;          // DX, DG of the K controller over the global batch
  if ((rc = exchange_stats(g, g->be_part + nb, nb, 1, 1, s))) return rc;
  if ((rc = launch(c, "began_loss_final_kernel", began_loss_final_kernel, 1, 256, 0, s, g->be_part, g->be_part + nb, nb, B * stat_world(g), 0, g->be_state, g->lossbuf))) return rc;
  if ((rc = launch_plan(c, sp->be_gwd, s))) return rc;
  if ((rc = launch_plan(c, sp->be_de_d, s))) return rc;
  if ((rc = launch_plan(c, sp->dw1d, s))) return rc;
  GradSegs gs;
  memset(&gs, 0, sizeof gs);
  const GemmParams& pe = sp->dw1d.p;
  const GemmParams& pd = sp->be_gwd.p;
  gs.nseg = 4;
  gs.total = g->D.total;
  gs.s[0] = {g->D.off_w1, g->H * g->X, 0, g->X, pe.ldp, 0, pe.splits, pe.part_stride, g->PD};
  gs.s[1] = {g->D.off_b1, g->H, 2, 0, pe.ldp, g->X, pe.splits, pe.part_stride, g->PD};
  gs.s[2] = {g->D.off_w2, g->X * g->H, 0, g->H, pd.ldp, 0, pd.splits, pd.part_stride, g->PWd};
  gs.s[3] = {g->D.off_b2, g->X, 2, 0, pd.ldp, g->H, pd.splits, pd.part_stride, g->PWd};
  if ((rc = emit_grads(g, GM_NET_D, gs, s))) return rc;
  if (loss_dev) CU_OK(c, cudaMemcpyAsync(loss_dev, g->lossbuf, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return GM_OK;
}

static int began_g_grad(gm_gan* g, StepPlans* sp, int B, float* loss_dev, cudaStream_t s) {
  gm_ctx* c = g->ctx;
  int rc;
  if ((rc = launch_plan(c, sp->be_enc_g, s))) return rc;
  if ((rc = launch_plan(c, sp->be_dec_g, s))) return rc;
  const int nb = c->num_sms;
  if ((rc = launch(c, "vae_rowsum_kernel", vae_rowsum_kernel, nb, 256, 0, s, g->slots_r + B, 2 * cdiv(g->X, 208), 2 * g->Bmax, B, g->be_part + nb))) return rc;
  if ((rc = launch(c, "began_loss_final_kernel", began_loss_final_kernel, 1, 256, 0, s, g->be_part, g->be_part + nb, nb, B, 1, g->be_state, g->lossbuf))) return rc;
  if ((rc = launch_plan(c, sp->be_de_g, s))) return rc;
  if ((rc = launch_plan(c, sp->be_dxg, s))) return rc;
  if ((rc = launch(c, "began_da2_kernel", began_da2_kernel, c->num_sms * 8, 256, 0, s, g->BT, g->DR + size_t(B) * g->XP, g->Xall + size_t(B) * g->XP, g->DA2, B, g->X, g->XP, g->lo))) return rc;
  if ((rc = launch_plan(c, sp->dw2g, s))) return rc;
  if ((rc = launch_plan(c, sp->dhg, s))) return rc;
  if ((rc = launch_plan(c, sp->dw1g, s))) return rc;
  if ((rc = began_finalize_g(g, sp, s))) return rc;
  if (loss_dev) CU_OK(c, cudaMemcpyAsync(loss_dev, g->lossbuf, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return GM_OK;
}

// BEGAN device state: host get/set of [K, inv_b, -K inv_b, DX, DG, best, bad, lr_scale, inv_b, inv_b, convergence]
extern "C" int gm_gan_began_state(gm_gan* g, float* host11, int set, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_began_state");
  if (!g || !host11) return GM_ERR_ARG;
  if (g->d.variant != GM_BEGAN) return fail(g->ctx, GM_ERR_STATE, "not a BEGAN engine");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (set) CU_OK(g->ctx, cudaMemcpyAsync(g->be_state, host11, 11 * sizeof(float), cudaMemcpyHostToDevice, s));
  else {
    CU_OK(g->ctx, cudaMemcpyAsync(host11, g->be_state, 11 * sizeof(float), cudaMemcpyDeviceToHost, s));
    CU_OK(g->ctx, cudaStreamSynchronize(s));
  }
  return GM_OK;
}
// K <- clip(K + LAMBDA (GAMMA DX - DG), 0, 1) and the plateau schedulers (src/be_gan.py:186-195)
extern "C" int gm_gan_began_control(gm_gan* g, float gamma, float lambda, float patience, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_began_control");
  if (!g) return GM_ERR_ARG;
  if (g->d.variant != GM_BEGAN) return fail(g->ctx, GM_ERR_STATE, "not a BEGAN engine");
  return launch(g->ctx, "began_control_kernel", began_control_kernel, 1, 1, 0, static_cast<cudaStream_t>(stream), g->be_state, gamma, lambda, patience);
}

// real rows -> Xall[0:B] (bf16, ones column); with a sampler pool and no gather_idx the kernel draws the batch rows itself
static int stage_real_rows(gm_gan* g, const void* images, int img_fmt, const int* gather_idx, int B, uint64_t step, cudaStream_t s) {
  gm_ctx* c = g->ctx;
  Sampler smp = kNoSampler;
  if (!gather_idx && g->pool_n > 0) {
    if (B > g->pool_n) return fail(c, GM_ERR_ARG, "batch (%d) exceeds the sampler's pool (%lld)", B, g->pool_n);
    smp = make_sampler(g->pool_n, g->pool_seed, step, 0, g->dev_step ? g->dstep + 3 : nullptr);     // a fresh permutation every step (src/ns_gan.py:224)
  }
  return launch(c, "stage_images_kernel", stage_images_kernel, c->num_sms * 8, 256, 0, s, images, img_fmt, gather_idx, g->Xall, B, g->X, g->XP, smp, g->lo);
}

// process_batch of the NEXT train_D (src/ns_gan.py:222-226) ahead of time: stages the real rows now; the following gm_gan_d_grad
// with the same batch skips its own staging.  Nothing of a G step reads those rows, so a data-parallel host enqueues this
// between gm_gan_exchange_begin(G) and gm_gan_apply_allreduce(G).  `step` = the step argument the later gm_gan_d_grad gets.
extern "C" int gm_gan_d_stage(gm_gan* g, const void* images, int img_fmt, const int* gather_idx, int batch, uint64_t step, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_d_stage");
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  if (!images) return fail(g->ctx, GM_ERR_ARG, "images is null");
  if (g->dev_step) return fail(g->ctx, GM_ERR_STATE, "gm_gan_d_stage is not available in device-step mode");
  if ((rc = stage_real_rows(g, images, img_fmt, gather_idx, batch, step, static_cast<cudaStream_t>(stream)))) return rc;
  g->staged_batch = batch;
  return GM_OK;
}

extern "C" int gm_gan_d_grad(gm_gan* g, const void* images, int img_fmt, const int* gather_idx, int batch,
                             const float* noise, const float* aux, float inv_global_batch, uint64_t seed,
                             uint64_t step, float* loss_dev, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_d_grad");
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  if (!images) return fail(g->ctx, GM_ERR_ARG, "images is null");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StepPlans* sp;
  if ((rc = build_plans(g, batch, &sp))) return rc;
  const int B = batch;
  gm_ctx* c = g->ctx;
  if ((rc = flush_pending(g, s))) return rc;
  // real rows -> Xall[0:B] (bf16, ones column)
  if (g->staged_batch == B) {
    g->staged_batch = 0;       // the real rows are already in place (gm_gan_d_stage)
  } else {
    if ((rc = stage_real_rows(g, images, img_fmt, gather_idx, B, step, s))) return rc;
  }
  const unsigned long long* dptr = g->dev_step ? g->dstep + 3 : nullptr;   // device-step mode: the train_D call counter
  if ((rc = run_generator(g, sp, B, noise, seed, g->dev_step ? 0 : 2 * step, s, dptr))) return rc;
  if (g->d.variant == GM_BEGAN) return (rc = began_d_grad(g, sp, B, loss_dev, s)) ? rc : bump_step(g, 3, s);
  const bool gp = g->nreg > 2;
  const int H = g->H, HP = g->HP, X = g->X, XP = g->XP;
  const float* w2 = g->par[GM_NET_D] + g->D.off_w2;
  const size_t dh_smem = size_t(g->dh_rows_per_iter) * HP * sizeof(float);
  const bool dra = g->d.variant == GM_DRA;
  if (dra) {
    // interpolated rows (region 2) around the real data
    if ((rc = launch(c, "moments_kernel", moments_kernel, c->num_sms * 2, 256, 0, s, g->Xall, B, X, XP, g->mom_part))) return rc;
    if ((rc = exchange_stats(g, g->mom_part, c->num_sms * 2, 2, 2, s))) return rc;     // images.std() over the global batch
    if ((rc = launch(c, "moments_final_kernel", moments_final_kernel, 1, 256, 0, s, g->mom_part, c->num_sms * 2, float(double(B) * X * stat_world(g)), g->stats))) return rc;
    // xhat_kernel takes no programmatic serialisation: launched early behind the generator's output GEMM its CTAs would
    // pile up on the first SMs that GEMM frees instead of spreading over the whole chip
    if ((rc = launch(c, {"xhat_kernel", false}, xhat_kernel, c->num_sms * 8, 256, 0, s, g->Xall, g->Xall + size_t(2) * B * XP, B, X, XP,
                     aux, g->stats, seed, g->dev_step ? 0 : 2 * step, g->lc.dra_c, g->lo, dptr))) return rc;
  }
  if ((rc = launch_plan(c, sp->d1_d, s))) return rc;
  if (g->d.variant == GM_WGP) {
    // U = w2 * relu'(a_hat) and the logit part of s(x_hat) from the pre-activations of the real / fake rows
    if ((rc = launch(c, "gp_hat_kernel", gp_hat_kernel, c->num_sms * 8, 256, 0, s, g->Aall, g->Aall + size_t(B) * HP, w2, g->DHall + size_t(2) * B * HP,
               g->slots + 2 * B, 2 * cdiv(H, 208), g->nreg * g->Bmax, B, H, HP, aux, seed, g->dev_step ? 0 : 2 * step, g->lo, dptr))) return rc;
  }
  if ((rc = launch_loss(g, B, 0, inv_global_batch, s))) return rc;
  if ((rc = launch(c, "dh_kernel", dh_kernel, g->dh_blocks, g->dh_threads, dh_smem, s, g->Aall, g->ds, w2, g->DHall, g->dw2p, 2 * B, H, HP, g->dh_rows_per_iter, g->lo,
             g->d.variant == GM_WGP ? 1 : 0))) return rc;
  if ((rc = launch(c, "colsum_kernel", colsum_kernel, cdiv(HP * 32, 256), 256, 0, s, g->dw2p, g->dh_blocks, HP, HP, g->dw2sum))) return rc;
  if (gp) {
    const size_t rreg = size_t(g->nreg - 1) * B;
    if (dra) {   // DRAGAN keeps a_hat (its penalty back-propagates through s(x_hat) too): U = 1[a_hat > 0] * w2 by a pass
      if ((rc = launch(c, "dh_kernel", dh_kernel, g->dh_blocks, g->dh_threads, dh_smem, s, g->Aall + size_t(2) * B * HP, nullptr, w2, g->DHall + rreg * HP, nullptr,
                                                            B, H, HP, g->dh_rows_per_iter, g->lo, 0))) return rc;
    }
    if ((rc = launch_plan(c, sp->gp_v, s))) return rc;          // V = U W1 -> R region of Xall, ||V||^2 -> slots_v
    {
      // dW1d's bias row sums DHall against Xall's ones column over all nreg regions, and the penalty has no b1 gradient:
      // the R rows' ones column must be 0, but a larger earlier batch leaves its real rows' 1.0 there (V fills [0, X))
      __nv_bfloat16* col = g->Xall + rreg * XP + X;
      CU_OK(c, cudaMemset2DAsync(col, size_t(XP) * sizeof(__nv_bfloat16), 0, sizeof(__nv_bfloat16), B, s));
      if (g->lo) CU_OK(c, cudaMemset2DAsync(col + g->lo, size_t(XP) * sizeof(__nv_bfloat16), 0, sizeof(__nv_bfloat16), B, s));
    }
    GpParams gpp;
    gpp.slots_s = g->slots + 2 * B; gpp.nslots_s = 2 * cdiv(H, 208); gpp.slot_ld = g->nreg * g->Bmax;
    gpp.slots_v = g->slots_v; gpp.nslots_v = 2 * cdiv(X, 208); gpp.slotv_ld = g->Bmax;
    gpp.b2 = g->par[GM_NET_D] + g->D.off_b2;
    gpp.rows = B; gpp.out_act = g->d.d_out_act;
    gpp.lam = g->lc.gp_lambda; gpp.K = g->lc.gp_k; gpp.inv_b = inv_global_batch;
    gpp.coef = g->coef; gpp.ds_gp = g->ds + 2 * B;
    gpp.part = g->gp_part; gpp.nblk = cdiv(B, kLossThreads) < c->num_sms * 2 ? cdiv(B, kLossThreads) : c->num_sms * 2;
    gpp.loss = g->lossbuf;
    if ((rc = launch(c, "gp_rows_kernel", gp_rows_kernel, gpp.nblk, kLossThreads, 0, s, gpp))) return rc;
    if ((rc = launch(c, "gp_final_kernel", gp_final_kernel, 1, kLossThreads, 0, s, gpp))) return rc;
    if ((rc = launch(c, "scale_rows_kernel", scale_rows_kernel, c->num_sms * 4, 256, 0, s, g->DHall + rreg * HP, g->coef, B, HP, g->lo))) return rc;   // U <- coef * U
    if ((rc = launch_plan(c, sp->gp_t, s))) return rc;          // T = coef (V W1^T) * mask -> DHg
    // dGP/dw2 = column sums of T (block partials; no output rows)
    if ((rc = launch(c, "dh_kernel", dh_kernel, g->dh_blocks, g->dh_threads, dh_smem, s, g->DHg, nullptr, w2, static_cast<__nv_bfloat16*>(nullptr), g->dw2p2, B, H, HP, g->dh_rows_per_iter, g->lo, 0))) return rc;
    if ((rc = launch(c, "colsum_kernel", colsum_kernel, cdiv(HP * 32, 256), 256, 0, s, g->dw2p2, g->dh_blocks, HP, HP, g->dw2sum + HP))) return rc;
    if (dra) {   // DRAGAN: the penalty also back-propagates through s(xhat)
      if ((rc = launch(c, "dh_kernel", dh_kernel, g->dh_blocks, g->dh_threads, dh_smem, s, g->Aall + size_t(2) * B * HP, g->ds + 2 * B, w2,
                                                            g->DHall + size_t(2) * B * HP, g->dw2p3, B, H, HP, g->dh_rows_per_iter, g->lo, 0))) return rc;
      if ((rc = launch(c, "colsum_kernel", colsum_kernel, cdiv(HP * 32, 256), 256, 0, s, g->dw2p3, g->dh_blocks, HP, HP, g->dw2sum + 2 * HP))) return rc;
    }
  }
  if ((rc = launch_plan(c, sp->dw1d, s))) return rc;
  GradSegs gs;
  memset(&gs, 0, sizeof gs);
  const GemmParams& pw = sp->dw1d.p;
  gs.nseg = 4;
  gs.total = g->D.total;
  gs.s[0] = {g->D.off_w1, g->H * g->X, 0, g->X, pw.ldp, 0, pw.splits, pw.part_stride, g->PD};
  gs.s[1] = {g->D.off_b1, g->H, 2, 0, pw.ldp, g->X, pw.splits, pw.part_stride, g->PD};
  gs.s[2] = {g->D.off_w2, g->H, 3, 0, 0, 0, gp ? g->nreg - 1 : 1, (long long)HP, g->dw2sum};
  gs.s[3] = {g->D.off_b2, 1, 3, 0, 0, 0, gp ? 2 : 1, 2, g->lossbuf + 1};
  if ((rc = emit_grads(g, GM_NET_D, gs, s))) return rc;
  if (loss_dev) CU_OK(c, cudaMemcpyAsync(loss_dev, g->lossbuf, sizeof(float), cudaMemcpyDeviceToDevice, s));
  g->last_rows = 2 * B;
  return bump_step(g, 3, s);
}

// train_G + backward; `staged`: the generator forward of this step was already enqueued by
// gm_gan_g_forward_stage (it does not depend on the D update, so a data-parallel host can run it
// while the D-gradient exchange is still in flight on another stream)
static int g_grad_impl(gm_gan* g, int batch, const float* noise, float inv_global_batch, uint64_t seed, uint64_t step,
                       float* loss_dev, gm_stream stream, bool staged) {
  REFUSE_BAYES(g, "gm_gan_g_grad");
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StepPlans* sp;
  if ((rc = build_plans(g, batch, &sp))) return rc;
  const int B = batch;
  gm_ctx* c = g->ctx;
  if ((rc = flush_pending(g, s))) return rc;
  if (!staged && (rc = run_generator(g, sp, B, noise, seed, g->dev_step ? 1 : 2 * step + 1, s, g->dev_step ? g->dstep + 2 : nullptr))) return rc;
  if (g->d.variant == GM_BEGAN) return (rc = began_g_grad(g, sp, B, loss_dev, s)) ? rc : bump_step(g, 2, s);
  if ((rc = launch_plan(c, sp->d1_g, s))) return rc;
  if ((rc = launch_loss(g, B, 1, inv_global_batch, s))) return rc;
  if ((rc = launch_plan(c, sp->dx, s))) return rc;
  if ((rc = launch_plan(c, sp->dw2g, s))) return rc;
  if ((rc = launch_plan(c, sp->dhg, s))) return rc;
  if ((rc = launch_plan(c, sp->dw1g, s))) return rc;
  GradSegs gs;
  memset(&gs, 0, sizeof gs);
  const GemmParams& p2 = sp->dw2g.p;
  const GemmParams& p1 = sp->dw1g.p;
  gs.nseg = 4;
  gs.total = g->G.total;
  gs.s[0] = {g->G.off_w1, g->H * g->Z, 0, g->Z, p1.ldp, 0, p1.splits, p1.part_stride, g->PG1};
  gs.s[1] = {g->G.off_b1, g->H, 2, 0, p1.ldp, g->Z, p1.splits, p1.part_stride, g->PG1};
  gs.s[2] = {g->G.off_w2, g->X * g->H, 0, g->H, p2.ldp, 0, p2.splits, p2.part_stride, g->PG2};
  gs.s[3] = {g->G.off_b2, g->X, 2, 0, p2.ldp, g->H, p2.splits, p2.part_stride, g->PG2};
  if ((rc = emit_grads(g, GM_NET_G, gs, s))) return rc;
  if (loss_dev) CU_OK(c, cudaMemcpyAsync(loss_dev, g->lossbuf, sizeof(float), cudaMemcpyDeviceToDevice, s));
  g->last_rows = B;
  return bump_step(g, 2, s);
}

extern "C" int gm_gan_g_grad(gm_gan* g, int batch, const float* noise, float inv_global_batch, uint64_t seed,
                             uint64_t step, float* loss_dev, gm_stream stream) {
  return g_grad_impl(g, batch, noise, inv_global_batch, seed, step, loss_dev, stream, false);
}
extern "C" int gm_gan_g_forward_stage(gm_gan* g, int batch, const float* noise, uint64_t seed, uint64_t step, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_g_forward_stage");
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  StepPlans* sp;
  if ((rc = build_plans(g, batch, &sp))) return rc;
  if ((rc = run_generator(g, sp, batch, noise, seed, 2 * step + 1, static_cast<cudaStream_t>(stream)))) return rc;
  return GM_OK;
}
extern "C" int gm_gan_g_grad_staged(gm_gan* g, int batch, float inv_global_batch, float* loss_dev, gm_stream stream) {
  return g_grad_impl(g, batch, nullptr, inv_global_batch, 0, 0, loss_dev, stream, true);
}

// ---- InfoGAN: auxiliary network Q and the mutual-information step (src/info_gan.py:269-304,196-205)
extern "C" int gm_gan_bind_q(gm_gan* g, float* q_params, float* q_grads, float* q_m, float* q_v, float* g_mi_m, float* g_mi_v) {
  REFUSE_BAYES(g, "gm_gan_bind_q");
  if (!g || !q_params || !q_grads) return g ? fail(g->ctx, GM_ERR_ARG, "gm_gan_bind_q: bad argument") : GM_ERR_ARG;
  if (g->d.variant != GM_INFO) return fail(g->ctx, GM_ERR_STATE, "gm_gan_bind_q: engine was not created with GM_INFO");
  g->parQ = q_params; g->grdQ = q_grads; g->amQ = q_m; g->avQ = q_v; g->amG2 = g_mi_m; g->avG2 = g_mi_v;
  g->plans.clear(); g->cplans.clear(); g->qplans.clear();
  return GM_OK;
}
extern "C" int gm_gan_q_param_count(const gm_gan* g) { return (g && g->d.variant == GM_INFO) ? g->Qn.total : GM_ERR_ARG; }

static void q_adam_segs(gm_gan* g, AdamParams& a) {
  a.lo_off = g->lo;
  a.total = g->Qn.total;
  a.nseg = 2;
  a.seg[0] = {g->Qn.off_w1, g->H * g->X, g->X, g->Wq1_s, g->X, g->Wq1_t, g->H};
  a.seg[1] = {g->Qn.off_w2, g->q_out * g->H, g->H, g->Wq2_s, g->H, g->Wq2_t, 64};
}
extern "C" int gm_gan_sync_shadows_q(gm_gan* g, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_sync_shadows_q");
  if (!g || !g->parQ) return g ? fail(g->ctx, GM_ERR_STATE, "Q not bound") : GM_ERR_ARG;
  AdamParams a;
  memset(&a, 0, sizeof a);
  a.p = g->parQ; a.update = 0;
  q_adam_segs(g, a);
  return launch(g->ctx, "adam_kernel", adam_kernel, cdiv(a.total, 256), 256, 0, static_cast<cudaStream_t>(stream), a);
}

// train_Q + MI_loss.backward(): writes the flat G gradient (G's grad buffer), the flat Q
// gradient and loss_dev[0].  noise_dev [batch, z_total] fp32 is required (structured noise:
// z, one-hot code at [zd, zd+10), continuous code at [zd+10, zd+20)).
extern "C" int gm_gan_q_grad(gm_gan* g, int batch, const float* noise, int zd, float inv_global_batch, float* loss_dev,
                             gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_q_grad");
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  if (g->d.variant != GM_INFO || !g->parQ) return fail(g->ctx, GM_ERR_STATE, "bind Q first (GM_INFO engines only)");
  if (!noise) return fail(g->ctx, GM_ERR_ARG, "the Q step needs the structured noise tensor");
  if (zd + g->q_out != g->Z) return fail(g->ctx, GM_ERR_ARG, "z_dim (%d) + codes (%d) != generator input (%d)", zd, g->q_out, g->Z);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((rc = flush_pending(g, s))) return rc;
  StepPlans* sp;
  if ((rc = build_plans(g, batch, &sp))) return rc;
  const int B = batch;
  gm_ctx* c = g->ctx;
  if ((rc = run_generator(g, sp, B, noise, 0, 0, s))) return rc;
  if ((rc = launch_plan(c, sp->q1, s))) return rc;
  if ((rc = launch_plan(c, sp->q2, s))) return rc;
  const int nb = cdiv(B, kLossThreads) < c->num_sms * 2 ? cdiv(B, kLossThreads) : c->num_sms * 2;
  if ((rc = launch(c, "info_loss_kernel", info_loss_kernel, nb, kLossThreads, 0, s, g->INF, 32, noise, g->Z, zd, 10, 10, B, inv_global_batch, g->DINF, 64, g->q_part, g->lo))) return rc;
  if ((rc = launch(c, "info_loss_final_kernel", info_loss_final_kernel, 1, kLossThreads, 0, s, g->q_part, nb, B, 10, g->lossbuf))) return rc;
  if ((rc = launch_plan(c, sp->gq2, s))) return rc;
  if ((rc = launch_plan(c, sp->dhq, s))) return rc;
  if ((rc = launch_plan(c, sp->gq1, s))) return rc;
  if ((rc = launch_plan(c, sp->dfq, s))) return rc;
  if ((rc = launch_plan(c, sp->dw2g, s))) return rc;
  if ((rc = launch_plan(c, sp->dhg, s))) return rc;
  if ((rc = launch_plan(c, sp->dw1g, s))) return rc;
  GradSegs gs;
  memset(&gs, 0, sizeof gs);
  const GemmParams& p2 = sp->dw2g.p;
  const GemmParams& p1 = sp->dw1g.p;
  gs.nseg = 4;
  gs.total = g->G.total;
  gs.s[0] = {g->G.off_w1, g->H * g->Z, 0, g->Z, p1.ldp, 0, p1.splits, p1.part_stride, g->PG1};
  gs.s[1] = {g->G.off_b1, g->H, 2, 0, p1.ldp, g->Z, p1.splits, p1.part_stride, g->PG1};
  gs.s[2] = {g->G.off_w2, g->X * g->H, 0, g->H, p2.ldp, 0, p2.splits, p2.part_stride, g->PG2};
  gs.s[3] = {g->G.off_b2, g->X, 2, 0, p2.ldp, g->H, p2.splits, p2.part_stride, g->PG2};
  if ((rc = emit_grads(g, GM_NET_G, gs, s, true))) return rc;   // consumed by gm_gan_apply_mi, which reads the flat buffer
  GradSegs qs;
  memset(&qs, 0, sizeof qs);
  const GemmParams& q1 = sp->gq1.p;
  const GemmParams& q2 = sp->gq2.p;
  qs.nseg = 4;
  qs.total = g->Qn.total;
  qs.s[0] = {g->Qn.off_w1, g->H * g->X, 0, g->X, q1.ldp, 0, q1.splits, q1.part_stride, g->PQ1};
  qs.s[1] = {g->Qn.off_b1, g->H, 2, 0, q1.ldp, g->X, q1.splits, q1.part_stride, g->PQ1};
  qs.s[2] = {g->Qn.off_w2, g->q_out * g->H, 0, g->H, q2.ldp, 0, q2.splits, q2.part_stride, g->PQ2};
  qs.s[3] = {g->Qn.off_b2, g->q_out, 2, 0, q2.ldp, g->H, q2.splits, q2.part_stride, g->PQ2};
  if ((rc = launch(c, "finalize_grads_kernel", finalize_grads_kernel, cdiv(qs.total, 256), 256, 0, s, qs, g->grdQ))) return rc;
  if (loss_dev) CU_OK(c, cudaMemcpyAsync(loss_dev, g->lossbuf, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return GM_OK;
}

// MI_optimizer.step(): Adam over G (with its OWN moment buffers, separate from G_optimizer's)
// and over Q (src/info_gan.py:146-148,205); refreshes both nets' operand copies.
extern "C" int gm_gan_apply_mi(gm_gan* g, const gm_adam_hp* hp, int step, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_apply_mi");
  if (!g || !hp || step <= 0) return g ? fail(g->ctx, GM_ERR_ARG, "gm_gan_apply_mi: bad argument") : GM_ERR_ARG;
  if (!g->parQ || !g->amQ || !g->avQ || !g->amG2 || !g->avG2) return fail(g->ctx, GM_ERR_STATE, "Q / MI optimizer state not bound");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  if ((rc = flush_pending(g, s))) return rc;
  AdamParams a;
  memset(&a, 0, sizeof a);
  a.p = g->par[GM_NET_G]; a.g = g->grd[GM_NET_G]; a.m = g->amG2; a.v = g->avG2;
  fill_adam(a, hp, step);
  adam_segs(g, GM_NET_G, a);
  if ((rc = launch(g->ctx, "adam_kernel", adam_kernel, cdiv(a.total, 256), 256, 0, s, a))) return rc;
  AdamParams q;
  memset(&q, 0, sizeof q);
  q.p = g->parQ; q.g = g->grdQ; q.m = g->amQ; q.v = g->avQ;
  fill_adam(q, hp, step);
  q_adam_segs(g, q);
  return launch(g->ctx, "adam_kernel", adam_kernel, cdiv(q.total, 256), 256, 0, s, q);
}

extern "C" int gm_gan_scores(gm_gan* g, float* dst, int n, gm_stream stream) {
  if (!g || !dst || n <= 0) return GM_ERR_ARG;
  if (n > g->nreg * g->Bmax) return fail(g->ctx, GM_ERR_ARG, "n too large");
  CU_OK(g->ctx, cudaMemcpyAsync(dst, g->scores, size_t(n) * sizeof(float), cudaMemcpyDeviceToDevice,
                                static_cast<cudaStream_t>(stream)));
  return GM_OK;
}

__global__ void bf16_rows_to_f32_kernel(const __nv_bfloat16* __restrict__ src, int ld, float* __restrict__ dst, int rows, int cols,
                                        long long lo_off) {
  griddep_sync();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)rows * cols) return;
  const int r = int(i / cols), cidx = int(i % cols);
  float v = __bfloat162float(src[(long long)r * ld + cidx]);
  if (lo_off) v += __bfloat162float(src[(long long)r * ld + cidx + lo_off]);
  dst[i] = v;
}

extern "C" int gm_gan_generate(gm_gan* g, const float* noise, int n, float* images, gm_stream stream) {
  REFUSE_BAYES(g, "gm_gan_generate");
  if (!g || !images || n <= 0) return GM_ERR_ARG;
  if (!g->par[0]) return fail(g->ctx, GM_ERR_STATE, "bind G first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int B = n;
  if (B > g->Bmax) return fail(g->ctx, GM_ERR_ARG, "n (%d) exceeds max_batch", n);
  if (!g->par[1]) return fail(g->ctx, GM_ERR_STATE, "bind D too (plans cover the whole step)");
  StepPlans* sp;
  int rc;
  if ((rc = build_plans(g, B, &sp))) return rc;
  // stage n noise rows (rows n..B-1 keep whatever they held; their outputs are not read)
  if ((rc = launch(g->ctx, "stage_noise_kernel", stage_noise_kernel, cdiv(n * ((g->Z + 8) / 8), 256), 256, 0, s, noise, g->Zb, n, g->Z, g->ZP, 0, 0, g->lo, static_cast<const unsigned long long*>(nullptr)))) return rc;
  if ((rc = launch_plan(g->ctx, sp->g1, s))) return rc;
  if ((rc = launch_plan(g->ctx, sp->g2, s))) return rc;
  const long long tot = (long long)n * g->X;
  return launch(g->ctx, "bf16_rows_to_f32_kernel", bf16_rows_to_f32_kernel, unsigned((tot + 255) / 256), 256, 0, s, g->Xall + size_t(B) * g->XP, g->XP, images, n, g->X, g->lo);
}

extern "C" int gm_gan_discriminate(gm_gan* g, const void* images, int img_fmt, int n, float* scores, gm_stream stream) {
  if (!g || !images || !scores || n <= 0) return GM_ERR_ARG;
  if (n > g->Bmax) return fail(g->ctx, GM_ERR_ARG, "n (%d) exceeds max_batch", n);
  if (!g->par[0] || !g->par[1]) return fail(g->ctx, GM_ERR_STATE, "bind both nets first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StepPlans* sp;
  int rc;
  if ((rc = build_plans(g, n, &sp))) return rc;
  if ((rc = launch(g->ctx, "stage_images_kernel", stage_images_kernel, g->ctx->num_sms * 8, 256, 0, s, images, img_fmt, nullptr, g->Xall, n, g->X, g->XP, kNoSampler, g->lo))) return rc;
  if ((rc = launch_plan(g->ctx, sp->d1_x, s))) return rc;
  return launch(g->ctx, "scores_kernel", scores_kernel, cdiv(n, 256), 256, 0, s, g->slots, 2 * cdiv(g->H, 208), g->nreg * g->Bmax, g->par[GM_NET_D] + g->D.off_b2,
                                            g->d.d_out_act, scores, n);
}

// On-device batch sampling: with a pool set (and gather_idx == NULL) gm_gan_d_grad reads row
// perm_{seed,step}(r) of images_dev for batch row r - the first `batch` entries of a fresh pseudo-random
// permutation of the pool per step, i.e. next(iter(DataLoader(shuffle=True))) (src/ns_gan.py:222-226).
// Loss constants the reference passes as train_D / train_G keyword arguments: LAMBDA of the gradient penalty
// (src/w_gp_gan.py:177; DRAGAN also K and C, src/dra_gan.py:174), LSGAN's targets a, b, c (src/ls_gan.py:173,197).
// Device-step mode: the per-step scalars the host normally passes - Adam's step count (bias correction), the Philox
// stream of train_D / train_G, the sampler's round - live in device counters that the step's own kernels advance, so one
// captured CUDA graph of (gm_gan_d_grad, gm_gan_apply(D), gm_gan_g_grad, gm_gan_apply(G)) replays as successive train
// steps (the launch-bound small-batch regime, BASELINE configs[0]).  counters4 = {Adam steps done on G, on D, train_G
// calls, train_D calls}; the `step` arguments of those entry points are ignored while the mode is on.
extern "C" int gm_gan_use_device_step(gm_gan* g, int on, const unsigned long long* counters4_host, gm_stream stream) {
  if (!g) return GM_ERR_ARG;
  if (on) REFUSE_BAYES(g, "gm_gan_use_device_step");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (on) {
    if (!g->dstep) {
      void* q = nullptr;
      CU_OK(g->ctx, cudaMalloc(&q, 4 * sizeof(unsigned long long)));
      g->allocs.push_back(q);
      g->dstep = static_cast<unsigned long long*>(q);
    }
    unsigned long long zero[4] = {0, 0, 0, 0};
    CU_OK(g->ctx, cudaMemcpyAsync(g->dstep, counters4_host ? counters4_host : zero, sizeof zero, cudaMemcpyHostToDevice, s));
    CU_OK(g->ctx, cudaStreamSynchronize(s));
  }
  g->dev_step = on != 0;
  return GM_OK;
}
extern "C" int gm_gan_device_steps(gm_gan* g, unsigned long long* counters4_host, gm_stream stream) {
  if (!g || !counters4_host || !g->dstep) return g ? fail(g->ctx, GM_ERR_STATE, "device-step mode was never enabled") : GM_ERR_ARG;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CU_OK(g->ctx, cudaMemcpyAsync(counters4_host, g->dstep, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  CU_OK(g->ctx, cudaStreamSynchronize(s));
  return GM_OK;
}
// programmatic dependent launch on / off at run time (stream capture on drivers that reject programmatic edges)
extern "C" int gm_ctx_set_pdl(gm_ctx* c, int on) {
  if (!c) return GM_ERR_ARG;
  c->pdl = on != 0;
  return GM_OK;
}

extern "C" int gm_gan_set_loss_consts(gm_gan* g, const gm_loss_consts* lc) {
  if (!g || !lc) return GM_ERR_ARG;
  g->lc = *lc;
  return GM_OK;
}

extern "C" int gm_gan_set_sampler(gm_gan* g, long long n_pool, uint64_t seed) {
  if (!g || n_pool < 0 || n_pool > 0x7FFFFFFFll) return g ? fail(g->ctx, GM_ERR_ARG, "gm_gan_set_sampler: bad pool size") : GM_ERR_ARG;
  g->pool_n = n_pool; g->pool_seed = seed;
  return GM_OK;
}
// host evaluation of the same permutation (CPU tests of the sampler; no device needed)
extern "C" int gm_sampler_indices_host(long long n_pool, uint64_t seed, uint64_t round, uint64_t offset, int count, int* out_host) {
  if (n_pool <= 0 || n_pool > 0x7FFFFFFFll || count < 0 || !out_host) return GM_ERR_ARG;
  const Sampler sp = make_sampler(n_pool, seed, round, offset);
  for (int r = 0; r < count; ++r) out_host[r] = int(sampler_index(sp, sp.offset + (unsigned long long)r));
  return GM_OK;
}
// the source-row indices gm_gan_d_grad(step) draws for a batch (tests / logging)
extern "C" int gm_gan_sample_indices(gm_gan* g, int batch, uint64_t step, int* idx_dev, gm_stream stream) {
  if (!g || !idx_dev || batch <= 0) return GM_ERR_ARG;
  if (g->pool_n > 0 && batch > g->pool_n) return fail(g->ctx, GM_ERR_ARG, "batch exceeds the pool");
  const Sampler smp = g->pool_n > 0 ? make_sampler(g->pool_n, g->pool_seed, step, 0) : kNoSampler;
  return launch(g->ctx, "sample_indices_kernel", sample_indices_kernel, cdiv(batch, 256), 256, 0, static_cast<cudaStream_t>(stream), smp, batch, idx_dev);
}
// the generator noise of a step as the train step draws it (net_step = 2*step for train_D, 2*step+1 for
// train_G): Philox N(0,1) rounded to the bf16 operand the GEMM reads -> out_dev [batch, z] fp32
extern "C" int gm_gan_debug_noise(gm_gan* g, int batch, uint64_t seed, uint64_t step, int g_step, float* out_dev, gm_stream stream) {
  int rc = check_step_args(g, batch);
  if (rc) return rc;
  if (!out_dev) return GM_ERR_ARG;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((rc = launch(g->ctx, "stage_noise_kernel", stage_noise_kernel, cdiv(batch * ((g->Z + 8) / 8), 256), 256, 0, s, static_cast<const float*>(nullptr), g->Zb, batch, g->Z, g->ZP,
                                                   (unsigned long long)seed, (unsigned long long)(2 * step + (g_step ? 1 : 0)), g->lo, static_cast<const unsigned long long*>(nullptr)))) return rc;
  const long long tot = (long long)batch * g->Z;
  return launch(g->ctx, "bf16_rows_to_f32_kernel", bf16_rows_to_f32_kernel, unsigned((tot + 255) / 256), 256, 0, s, g->Zb, g->ZP, out_dev, batch, g->Z, g->lo);
}

// debug / test aid: an internal bf16 activation buffer as fp32 (hi + lo in split mode), out_dev [rows, cols];
// which: 0 Zb, 1 Hg, 2 Xall, 3 Aall, 4 DHall, 5 DA2, 6 DHg; row0 = first row
extern "C" int gm_gan_debug_read(gm_gan* g, int which, int row0, int rows, int cols, float* out_dev, gm_stream stream) {
  if (!g || !out_dev || rows <= 0 || cols <= 0 || row0 < 0) return GM_ERR_ARG;
  const int plane = which / 16;   // 0: hi + lo, 1: hi plane only, 2: lo plane only
  which %= 16;
  const __nv_bfloat16* src[9] = {g->Zb, g->Hg, g->Xall, g->Aall, g->DHall, g->DA2, g->DHg, g->qs[0].H, g->qs[1].H};
  const int ld[9] = {g->ZP, g->HP, g->XP, g->HP, g->HP, g->XP, g->HP, g->HP, g->HP};
  // a Bayes-mode engine holds num_g x max_batch noise, G hidden and dL/dG rows and (1 + num_g) x max_batch image / D rows
  const long long J = g->nsamp ? g->nsamp : 1, nr = g->nsamp ? 1 + J : g->nreg;
  const long long nrow[9] = {J * g->Bmax, J * g->Bmax, nr * g->Bmax, nr * g->Bmax, nr * g->Bmax, J * g->Bmax, g->Bmax, g->Bmax, g->Bmax};
  static_assert(kQSlots == 2, "debug buffers 7, 8 are the Q call slots' hidden rows");
  if (which < 0 || which > 8 || cols > ld[which] || !src[which]) return fail(g->ctx, GM_ERR_ARG, "gm_gan_debug_read: bad buffer / extent");
  if ((long long)row0 + rows > nrow[which])
    return fail(g->ctx, GM_ERR_ARG, "gm_gan_debug_read: rows [%d, %lld) run past the buffer's %lld rows", row0, (long long)row0 + rows, nrow[which]);
  const long long tot = (long long)rows * cols;
  return launch(g->ctx, "bf16_rows_to_f32_kernel", bf16_rows_to_f32_kernel, unsigned((tot + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream),
             src[which] + size_t(row0) * ld[which] + (plane == 2 ? g->lo : 0), ld[which], out_dev, rows, cols, plane == 0 ? g->lo : 0ll);
}

extern "C" int gm_gan_fisher_state(gm_gan* g, float* lambda_rho_host, int set, gm_stream stream) {
  if (!g || !lambda_rho_host) return GM_ERR_ARG;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (set) CU_OK(g->ctx, cudaMemcpyAsync(g->fisher, lambda_rho_host, 2 * sizeof(float), cudaMemcpyHostToDevice, s));
  else {
    CU_OK(g->ctx, cudaMemcpyAsync(lambda_rho_host, g->fisher, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
    CU_OK(g->ctx, cudaStreamSynchronize(s));
  }
  return GM_OK;
}

#include "engine_custom.inl"
#include "engine_comm.inl"
#include "engine_vae.inl"
#include "engine_conv.inl"
#include "engine_bayes.inl"
