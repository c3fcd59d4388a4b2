// Persistent, warp-specialised wgmma GEMM for sm_90a (hand-written).
//
//   C[M,N] = sum_k A(m,k) * B(n,k)        bf16 operands, fp32 accumulation in registers
//
// Operand memory forms (row-major bf16 matrices in HBM, leading dim multiple of 8):
//   K-major  : matrix [MN rows, K cols]  (activations [batch, feat] as A; nn.Linear
//              weights [out, in] as B)            -> forward and dX GEMMs
//   MN-major : matrix [K rows, MN cols]  (contraction over the batch rows)
//                                                   -> dW GEMMs (A^T * B)
// Tiles: 128 x BN x 64, 128-byte TMA / wgmma swizzle, one m64nBNk16 wgmma per warpgroup and k-step.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected lane of warp 0 issues; the
// warpgroup gives its registers away with setmaxnreg), warpgroups 1..2 = consumers.
// Consumer warpgroup g accumulates rows [64 g, 64 g + 64) of the tile in registers and runs the
// fused epilogue straight from them: each consumer warp owns the 16 rows its fragments hold and
// walks the tile in 64-column steps.  Per step the warp writes its fragments to a private 4 KB
// fp32 scratch tile, and lane L takes row L & 15 and the 32-column block of parity L >> 4 through
// the per-row epilogue; the scratch is then reused as the bf16 staging of the store.  Meanwhile
// the producer keeps filling the smem ring with the next tile's operands.  Pipelines: smem ring
// full/empty mbarriers (TMA <-> wgmma), static round-robin tile scheduler (grid = #SMs).  The 128 x 208
// K-major kernel runs as 2-CTA clusters that share the B tile (kGemmCluster).  Its PINGPONG instances, launched for
// short-K GEMMs with a plain bias + activation epilogue, run the two consumer warpgroups in ping-pong: each runs its 64
// rows of a tile as a half-item of its own, the mainloops take turns through two named barriers, and each warpgroup's
// epilogue runs under the other one's wgmma.  A ring stage then holds one half-item's 64 A rows and the whole B tile.
// The 128 x 208 MN-major kernel (split-K weight gradients of the 400- and 401-wide layers) takes B as three 64-column
// boxes and a 16-column tail box and runs as 2-CTA clusters over n-tile pairs that share the A tile.
#pragma once
#include "ptx.cuh"

namespace gm {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kMmaK = 16;
constexpr int kProducerThreads = 128;                               // warpgroup 0: TMA producer
constexpr int kConsumerWarps = 8;                                   // warpgroups 1..2: wgmma, then the epilogue
constexpr int kGemmThreads = kProducerThreads + kConsumerWarps * 32;
// named barriers of the ping-pong mainloop handoff (0 is __syncthreads'; the kernel uses no other)
constexpr int kBarWg0Issued = 1;
constexpr int kBarWg1Issued = 2;
// setmaxnreg budget: 384 threads launch with 168 registers each; the producer drops to 40 so the consumers can hold a
// 128 x 208 (or 256) fp32 accumulator next to the epilogue's registers
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(kProducerThreads * kProducerRegs + kConsumerWarps * 32 * kConsumerRegs <= 65536, "register file");
constexpr int kSmemBudget = 227 * 1024;                             // H100: opt-in dynamic shared memory per block

enum : int { EPI_BF16 = 0, EPI_F32 = 1 };
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2, ACT_LRELU = 3 };   // LeakyReLU(act_slope): universal epilogue only
// AUX_NONZERO_MASK: like AUX_RELU_MASK for an aux that holds the SIGNED mask form w2 * relu'(a) (nonzero <=> active unit)
enum : int { AUX_NONE = 0, AUX_SIGMOID_GRAD = 1, AUX_RELU_MASK = 2, AUX_VAE_OUT = 3, AUX_L1 = 4, AUX_NONZERO_MASK = 5 };
// Row-dot of the stored values v into dot_out: DOT_W sum v * dot_w[n], DOT_SQ sum v * v.  DOT_W_MASK: as DOT_W, but
// stores dot_w[n] * 1[v > 0] instead of v (the G step needs only M = w2 * relu'(a1) of D's hidden layer: dL/dx =
// ds * (M W1), src/ns_gan.py:57-60 backward).  DOT_W_PRE: sum relu(v) * dot_w[n], and the PRE-activation v is stored
// (WGAN-GP's D forward, which never forms the x_hat rows: the penalty's mask is 1[eps pre_real + (1-eps) pre_fake > 0])
enum : int { DOT_NONE = 0, DOT_W = 1, DOT_SQ = 2, DOT_W_MASK = 3, DOT_W_PRE = 4 };
__host__ __device__ constexpr bool dot_has_w(int dot) { return dot == DOT_W || dot == DOT_W_MASK || dot == DOT_W_PRE; }

// Epilogue signature: (act, aux, bias, dot) packed into one int.  It is the kernel's EPI template argument, which fixes
// the fused epilogue at compile time (small code: the whole kernel must stay inside the instruction cache);
// kEpiUniversal selects the universal instance, which reads the epilogue from GemmParams at run time.
constexpr int kEpiUniversal = -1;
__host__ __device__ constexpr int epi_sig(int act, int aux, bool bias, int dot) { return act | aux << 2 | int(bias) << 5 | dot << 6; }
constexpr int kEpiSigBits = 9;
__host__ __device__ constexpr int epi_act(int sig) { return sig & 3; }
__host__ __device__ constexpr int epi_aux(int sig) { return (sig >> 2) & 7; }
__host__ __device__ constexpr bool epi_bias(int sig) { return (sig >> 5) & 1; }
__host__ __device__ constexpr int epi_dot(int sig) { return sig >> 6; }
// plain epilogues (no aux input, no row-dot) may store their bf16 output through the TMA-store path
__host__ __device__ constexpr bool epi_plain(int aux, int dot) { return aux == AUX_NONE && dot == DOT_NONE; }

struct GemmParams {
  int M, N, K;          // logical extents; K counts contraction elements
  int m_tiles, n_tiles;
  int splits, kblocks, kb_per_split;
  int epi;
  // ---- EPI_BF16: out[m, n] = bf16( f(acc + bias[n]) * g(aux[m,n]) ), row-major, ld = ldo
  __nv_bfloat16* out;
  int ldo;
  int out_cols;         // columns [N, out_cols) are padding: zero, except col N = 1 if pad_one
  int pad_one;
  const float* bias;    // nullable
  int act;
  const __nv_bfloat16* aux;  // nullable, same [m, n] indexing, ld = ld_aux
  int ld_aux;
  int aux_mode;
  // AUX_L1 (BEGAN): out = sign(v - aux) * (row < row_split ? row_scale[0] : row_scale[1]), dot_out = sum |v - aux|
  const float* row_scale;
  int row_split;
  int dot;              // DOT_*: row-dot of the stored values
  const float* dot_w;   // its weights (DOT_W, DOT_W_MASK, DOT_W_PRE)
  // tma_store: full 32-column blocks of the bf16 output leave through the output tensor map
  // (cp.async.bulk.tensor store of the warp's swizzled staging tile) instead of LDS + STG
  int tma_store;
  // row_vec (AUX_SIGMOID_GRAD): additional per-row factor, out = v * row_vec[m] * aux (1 - aux)
  const float* row_vec;
  float* dot_out;       // partial slots [(n_tile*2 + half) * dot_ld + m]
  int dot_ld;
  // ---- EPI_F32: part[split*part_stride + (transpose ? n*ldp + m : m*ldp + n)] = acc
  float* part;
  long long part_stride;
  int ldp;
  int transpose;
  int f32_vec;          // set at launch: every row of every split starts on 16 bytes, so 16 columns leave as 4 float4
  // ---- split-bf16 operands (SPLIT kernels, gm_prec GM_PREC_SPLIT): A = A_hi + A_lo, B = B_hi + B_lo as bf16 planes
  // lo_off elements apart; the contraction runs over nparts = 3 operand pairs (hi,hi), (hi,lo), (lo,hi) of kb_part
  // k-blocks each into the same accumulator (kblocks = 3 kb_part; the dropped lo*lo term is below fp32 resolution).
  // bf16 outputs and aux inputs carry their residual plane at the same offset.
  int nparts, kb_part;
  long long lo_off;
  float act_slope;      // ACT_LRELU
};

inline int epi_sig(const GemmParams& p) { return epi_sig(p.act, p.aux_mode, p.bias != nullptr, p.dot); }

// Epilogue of one consumer warp: 16 rows (its fragments) x 64-column steps, one 32-column block per lane and step.
// Its scratch tile holds a step's fp32 fragments (16-byte chunks of row r XOR-swizzled by frag_swz(r): conflict-free
// 8-byte fragment stores and 16-byte row reads), then the step's bf16 staging: 16 rows x (128 B data + 16 B pad) for
// LDS + STG, or two 16 x 32 TMA-store boxes (64-byte rows, 64B swizzle) at 0 and 1 KB.
constexpr int kEpiRows = 16;
constexpr int kEpiStep = 64;
constexpr int kEpiCols = 32;                           // columns of one lane's block (the TMA-store box width)
constexpr int kEpiScratchBytes = kEpiRows * kEpiStep * 4;
constexpr int kEpiPitch = 144;
constexpr int kEpiVecBlocks = 8;                       // 32-column blocks of a tile the bias/dot staging holds
constexpr int kEpiVecBytes = kEpiVecBlocks * kEpiCols * 4 * 2;   // bias + row-dot weights
static_assert(kEpiRows * kEpiPitch <= kEpiScratchBytes && 2 * kEpiRows * kEpiCols * 2 <= kEpiScratchBytes, "staging");
__device__ __forceinline__ uint32_t frag_swz(int r) { return uint32_t(((r & 3) << 1) | ((r >> 2) & 1)); }

// K-major A tiles of the 128 x 208 kernel arrive as 64-row TMA boxes: one per stage in ping-pong, two otherwise
template <int BN, bool A_MN>
constexpr int kGemmABoxRows = (BN == 208 && !A_MN) ? BM / 2 : BM;

template <int BN_, bool STAGED_EPI = true, bool PINGPONG_ = false>
struct GemmCfg {
  static constexpr int BN = BN_;
  // ping-pong (128 x 208 K-major only): a stage holds the A rows of one 64-row half of the tile
  static constexpr bool PINGPONG = PINGPONG_;
  static_assert(!PINGPONG || (STAGED_EPI && BN == 208), "ping-pong: 128 x 208 K-major kernel only");
  static constexpr int A_ROWS = PINGPONG ? BM / 2 : BM;
  static constexpr int A_BYTES = A_ROWS * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // per-warp scratch / staging tile (+ per-warp copies of the tile's bias / row-dot weights in the K-major kernels)
  static constexpr int EPI_BYTES = kConsumerWarps * (kEpiScratchBytes + (STAGED_EPI ? kEpiVecBytes : 0));
  static_assert(!STAGED_EPI || (BN + kEpiCols - 1) / kEpiCols <= kEpiVecBlocks, "bias/dot staging too small");
  static constexpr int FIXED_BYTES = 1024 + 512 + EPI_BYTES;   // 1024: alignment slack; 512: barriers
  static constexpr int STAGES_RAW = (kSmemBudget - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;   // scratch tiles stay 512-B aligned (TMA 64B swizzle)
  static constexpr int BOXN = BN;   // K-major B: one box of BN rows
  static_assert(BN % 16 == 0 && BN <= 256, "wgmma N constraint (and 16-column epilogue chunks)");
  static_assert(STAGES >= 2, "need a pipeline");
  static_assert(BN < 208 || STAGES >= 4, "the 208- and 256-wide kernels need a 4-stage ring to hide TMA latency");
  // 5 x 34 816 + 50 688 = 224 768 B
  static_assert(!PINGPONG || (STAGES == 5 && SMEM_BYTES <= kSmemBudget), "ping-pong ring");
};

// CTAs per cluster (the default of the kernel's CL).  The 128 x 208 K-major kernel runs as 2-CTA clusters on adjacent
// m-tiles of one n-tile: both read the same B tile (a slice of the weight matrix), so each CTA loads BN / 2 of its rows
// and multicasts them into both CTAs' stage.  That cuts the bytes L2 feeds each CTA per k-block from 43 008 to 29 696,
// which bound the long-K mainloop.  The 128 x 208 MN-major kernel is launched with CL = 2 when its n-tile count is even:
// the two n-tiles of one (split, m-tile) read the same A tile (128 columns of the same batch rows), so each CTA loads
// one 64-column box of it and multicasts it into both CTAs' stage (49 152 -> 34 816 bytes per CTA and k-block with the
// 208-wide B).
template <int BN, bool A_MN, bool B_MN>
constexpr int kGemmCluster = (BN == 208 && !A_MN && !B_MN) ? 2 : 1;
// MN-major 208-wide B tile: three 64-column boxes (128-byte swizzle) and the last 16 columns as a box of their own
// (32-byte swizzle, tensor map tmBt) behind them, read by an m64n192 and an m64n16 wgmma
constexpr int kTnTail = 16;

// EPI: the fused epilogue's signature (epi_sig), or kEpiUniversal.
// PINGPONG: the consumer warpgroups run the 64-row halves of each tile as half-items of their own (see the consumer loop)
// CL: CTAs per cluster; with MN-major operands the cluster's CTAs take adjacent n-tiles of one m-tile.
// tmBt / tmB2t: the 16-column tail boxes of tmB / tmB2 (MN-major 208-wide kernel only)
template <int BN, bool A_MN, bool B_MN, int EPI = kEpiUniversal, bool SPLIT = false, bool PINGPONG = false,
          int CL = kGemmCluster<BN, A_MN, B_MN>>
// 384 threads, one block per SM: 168 registers per thread at launch, redistributed by setmaxnreg
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmA2,
                  const __grid_constant__ CUtensorMap tmB2, const __grid_constant__ CUtensorMap tmBt,
                  const __grid_constant__ CUtensorMap tmB2t, const GemmParams p) {
  constexpr bool kUniversal = EPI == kEpiUniversal;
  static_assert(!SPLIT || kUniversal, "split operands: universal epilogue only");
  using Cfg = GemmCfg<BN, !A_MN, PINGPONG>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr bool PP = PINGPONG;
  constexpr int A_BOX = kGemmABoxRows<BN, A_MN>;
  static_assert(Cfg::A_ROWS % A_BOX == 0, "A tile in whole boxes");
  // MN-major B: whole 64-column atoms, or (208) three of them and the 16-column tail
  constexpr bool kTail = B_MN && BN == 208;
  constexpr int B_BOXES = BN / 64;   // 64-column B boxes
  static_assert(!B_MN || BN % 64 == 0 || kTail, "MN-major B needs 64-wide atoms");
  static_assert(A_MN == B_MN, "one operand form per kernel");
  // K-major: each CTA's share of the B tile starts on a 1024-byte swizzle atom, so the B descriptor is the same as for
  // one box.  MN-major: each CTA's share of the A tile is one whole 64-column box, so the A descriptor is unchanged.
  static_assert(CL == 1 || CL == 2, "cluster size");
  static_assert(CL == 1 || (!B_MN && (BN / CL) % 8 == 0 && (Cfg::B_BYTES / CL) % 1024 == 0) || (B_MN && kTail && BM / CL == 64),
                "multicast share");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t epi_base = bar_base + 512u;   // per-warp scratch tiles, then bias / row-dot slices

  const int warp = __shfl_sync(0xffffffffu, int(threadIdx.x >> 5), 0);   // provably warp-uniform (wgmma issue)
  const int lane = threadIdx.x & 31;

  griddep_launch();   // the next grid may start its prologue as soon as SMs free up
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (SPLIT) { tma_prefetch_desc(&tmA2); tma_prefetch_desc(&tmB2); }
    if constexpr (kTail) { tma_prefetch_desc(&tmBt); if constexpr (SPLIT) tma_prefetch_desc(&tmB2t); }
    if (p.tma_store) tma_prefetch_desc(&tmC);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      // every consumer warp that reads the slot, in every CTA of the cluster, releases it: the peers' multicasts also
      // write it.  In ping-pong one warpgroup per CTA reads a slot.
      mbar_init(empty_bar(s), CL * (PP ? kConsumerWarps / 2 : kConsumerWarps));
    }
    fence_mbar_init();
  }
  // the barriers are initialised in every CTA of the cluster before any peer arrives on them or multicasts into them
  if constexpr (CL > 1) cluster_sync();
  else __syncthreads();
  griddep_wait();     // barrier init above overlapped the previous grid's tail

  // Work items walk (split, m-group, n-group) with one item per cluster.  K-major: CTA rank r of a cluster takes m-tile
  // CL * group + r of the item's n-tile; m-tiles are rounded up to whole groups: a CTA on a tile past M loads its share
  // of B, computes on zero-filled A rows and stores nothing (every store is guarded by row < M or clipped at the tensor
  // extent), so both CTAs walk the same k-blocks through the ring.  MN-major (n_tiles a multiple of CL): rank r takes
  // n-tile CL * group + r of the item's m-tile; both CTAs share split and m-tile, so they walk the same k-blocks too.
  constexpr bool kPairN = CL > 1 && B_MN;
  const int rank = CL > 1 ? int(cluster_ctarank()) : 0;
  const int n_groups = kPairN ? p.n_tiles / CL : p.n_tiles;
  const int tiles = (kPairN ? p.m_tiles : (p.m_tiles + CL - 1) / CL) * n_groups;
  auto m0_of = [&](int rem) { return ((rem / n_groups) * (kPairN ? 1 : CL) + (kPairN ? 0 : rank)) * BM; };
  auto n_tile_of = [&](int rem) { return (rem % n_groups) * (kPairN ? CL : 1) + (kPairN ? rank : 0); };
  const int total = tiles * p.splits;
  const int first = blockIdx.x / CL, stride = gridDim.x / CL;
  // Ping-pong: an item is two half-items, rows [0, 64) for consumer warpgroup 0 and [64, 128) for warpgroup 1, whose
  // k-blocks enter the ring one half after the other.  The second half is skipped in both CTAs of the cluster when rank
  // 0's first row of it is past M (rank 1's rows are higher still), so the peers keep walking the same k-blocks.
  auto halves_of = [&](int rem) -> int {
    if constexpr (PP) return (rem / p.n_tiles) * CL * BM + Cfg::A_ROWS < p.M ? 2 : 1;
    else return 1;
  };
  // A k-block's stage and phase follow from the running count `it` of k-blocks issued, in (item, half-item, k-block)
  // order: stage it % STAGES, phase (it / STAGES) & 1.  Ping-pong consumers derive them from the count at each item,
  // which they also advance past the other warpgroup's half; the cooperative consumers read every k-block and just carry
  // stage and phase along.
  auto stage_of = [](uint32_t it) { return int(it % STAGES); };
  auto phase_of = [](uint32_t it) { return (it / STAGES) & 1u; };

  if (warp < kProducerThreads / 32) {
    // =========================== TMA producer ===========================
    // Warp 0 walks the loop (warp-uniform control flow and addresses keep the TMA operands in
    // uniform registers); one elected lane issues.  Warps 1..3 only release their registers.
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      uint32_t it = 0;
      const bool leader = elect_one();
      for (int item = first; item < total; item += stride) {
        const int split = item / tiles;
        const int rem = item - split * tiles;
        const int m0 = m0_of(rem);
        const int n0 = n_tile_of(rem) * BN;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, p.kblocks);
        const int nh = halves_of(rem);
        for (int h = 0; h < nh; ++h)
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int stage = stage_of(it);
          mbar_wait(empty_bar(stage), phase_of(it) ^ 1u);
          if (leader) {
            const uint32_t a_dst = smem_base + stage * Cfg::STAGE_BYTES;
            const uint32_t b_dst = a_dst + Cfg::A_BYTES;
            int kk = kb, opart = 0;
            if constexpr (SPLIT) { opart = kb / p.kb_part; kk = kb - opart * p.kb_part; }
            const CUtensorMap* const ta = (SPLIT && opart == 2) ? &tmA2 : &tmA;   // (hi,hi), (hi,lo), (lo,hi)
            const CUtensorMap* const tb = (SPLIT && opart == 1) ? &tmB2 : &tmB;
            const int k0 = kk * BK;
            mbar_arrive_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
            if constexpr (!A_MN) {
#pragma unroll
              for (int a = 0; a < Cfg::A_ROWS / A_BOX; ++a)
                tma_load_2d(a_dst + a * (A_BOX * BK * 2), ta, full_bar(stage), k0, m0 + h * Cfg::A_ROWS + a * A_BOX);
            } else if constexpr (CL > 1) {   // A box r into this and the peer CTA; the full barrier expects both boxes
              tma_load_2d_multicast(a_dst + rank * (BK * 128), ta, full_bar(stage), m0 + rank * 64, k0, (1u << CL) - 1);
            } else {
#pragma unroll
              for (int a = 0; a < BM / 64; ++a)
                tma_load_2d(a_dst + a * (BK * 128), ta, full_bar(stage), m0 + a * 64, k0);
            }
            if constexpr (CL > 1 && !B_MN) {   // rows [n0 + r BN/CL, +BN/CL) into this and the peer CTA; the full barrier expects both shares
              tma_load_2d_multicast(b_dst + rank * (Cfg::B_BYTES / CL), tb, full_bar(stage), k0, n0 + rank * (BN / CL), (1u << CL) - 1);
            } else if constexpr (!B_MN) {
              tma_load_2d(b_dst, tb, full_bar(stage), k0, n0);
            } else {
#pragma unroll
              for (int b = 0; b < B_BOXES; ++b)
                tma_load_2d(b_dst + b * (BK * 128), tb, full_bar(stage), n0 + b * 64, k0);
              if constexpr (kTail)
                tma_load_2d(b_dst + B_BOXES * (BK * 128), (SPLIT && opart == 1) ? &tmB2t : &tmBt, full_bar(stage), n0 + B_BOXES * 64, k0);
            }
          }
          __syncwarp();
        }
      }
    }
  } else {
    // ====================== consumers: wgmma, then the epilogue ======================
    setmaxnreg_inc<kConsumerRegs>();
    const int cw = warp - kProducerThreads / 32;   // consumer warp 0..7
    const int wg = cw >> 2;                        // warpgroup: rows [64 wg, 64 wg + 64) of the tile
    const int er = lane & 15;                      // epilogue: this lane's row of the warp's 16
    const int par = lane >> 4;                     // epilogue: parity of this lane's 32-column block in a 64-column step
    const uint32_t scratch_s = epi_base + uint32_t(cw) * kEpiScratchBytes;
    const uint32_t vec_s = epi_base + kConsumerWarps * kEpiScratchBytes + uint32_t(cw) * kEpiVecBytes;   // K-major kernels
    const int act = kUniversal ? p.act : epi_act(EPI);
    const int aux_mode = kUniversal ? p.aux_mode : epi_aux(EPI);
    const bool has_bias = kUniversal ? p.bias != nullptr : epi_bias(EPI);
    const int dot_mode = kUniversal ? p.dot : epi_dot(EPI);
    const bool has_dot = dot_has_w(dot_mode);
    const bool store_pre = dot_mode == DOT_W_PRE;   // ReLU only inside the row-dot
    const bool mask_all = dot_mode == DOT_W_MASK;
    const bool has_sq = dot_mode == DOT_SQ;
    // The bulk store serves the plain-activation epilogues only (launch_plan), so it is compiled out of the aux / row-dot
    // instances, and out of the universal 208-wide one, which those plain epilogues never reach.  Where the store path is
    // compiled in, ptxas keeps the consumers at the launch register count (168) despite setmaxnreg: those instances spill
    // 300-370 bytes with it and none without it.
    constexpr bool kTmaStore = !A_MN && !SPLIT && (kUniversal ? BN != 208 : epi_plain(epi_aux(EPI), epi_dot(EPI)));
    const bool tma_st = kTmaStore && p.tma_store != 0;
    bool st_pending = false;   // a bulk store may still be reading this warp's scratch tile
    auto stage_acquire = [&]() {
      if (st_pending) {
        if (er == 0) bulk_wait_read();   // lanes 0 and 16 issue the stores
        __syncwarp();
        st_pending = false;
      }
    };
    // descriptor strides: K-major: SBO = 8 rows * 128 B (LBO unused); MN-major: LBO = atom stride
    // (BK*128 B), SBO = 8 k-rows * 128 B.  Per k-step (16) advance: K-major 32 B, MN-major 16 rows * 128 B.
    constexpr uint32_t A_LBO = A_MN ? BK * 128 : 16, A_KADV = A_MN ? kMmaK * 128 : kMmaK * 2;
    constexpr uint32_t B_LBO = B_MN ? BK * 128 : 16, B_KADV = B_MN ? kMmaK * 128 : kMmaK * 2;
    constexpr uint32_t A_WG_OFF = A_MN ? BK * 128 : 64 * 128;   // this warpgroup's 64 rows of the A tile
    constexpr uint32_t DESC_HI = (1024u >> 4) | (1u << 30);      // SBO, 128B swizzle
    // MN-major 16-column tail box: 32-byte rows, 32B swizzle; SBO = 8 k-rows * 32 B, LBO (next 16-column atom) unused
    constexpr uint32_t TAIL_LBO = BK * kTnTail * 2, TAIL_KADV = kMmaK * kTnTail * 2;
    constexpr uint32_t TAIL_DESC_HI = ((8u * kTnTail * 2) >> 4) | (3u << 30);
    constexpr int kSteps = (BN + kEpiStep - 1) / kEpiStep;
    float acc[BN / 2];
    // step s's fragments (columns [64 s, 64 s + 64), rows (lane >> 2) + {0, 8}) -> the scratch tile.  The acc index must
    // be a compile-time constant, so every step has its own unrolled copy of the stores and s selects one of them.
    auto frag_to_scratch = [&](int s) {
#pragma unroll
      for (int t = 0; t < kSteps; ++t) {
        if (t == s) {
#pragma unroll
          for (int jj = 0; jj < kEpiStep / 8; ++jj) {
            const int j = t * (kEpiStep / 8) + jj;
            if (j < BN / 8) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = (lane >> 2) + 8 * h, c = 8 * jj + 2 * (lane & 3);
                const uint32_t a = scratch_s + uint32_t(r) * (kEpiStep * 4) + ((uint32_t(c >> 2) ^ frag_swz(r)) << 4) + uint32_t(c & 3) * 4;
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1]) : "memory");
              }
            }
          }
        }
      }
    };
    // 16 fp32 columns [c, c + 16) of this lane's row of the scratch tile
    auto scratch_ld16 = [&](int c, uint32_t (&r)[16]) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint4 v = lds128(scratch_s + uint32_t(er) * (kEpiStep * 4) + ((uint32_t((c >> 2) + i) ^ frag_swz(er)) << 4));
        r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
      }
    };
    // a stage this warp has finished reading is released in this CTA and in its cluster peer (whose producer multicasts into it)
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(empty_bar(s));
        if constexpr (CL > 1) mbar_arrive_cluster(mapa_shared(empty_bar(s), uint32_t(rank ^ 1)));
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    uint32_t it = 0;   // ping-pong: the producer's running k-block count, advanced past the other warpgroup's halves too
#pragma unroll 1
    for (int item = first; item < total; item += stride) {
      const int split = item / tiles;
      const int rem = item - split * tiles;
      const int n_tile = n_tile_of(rem);
      const int m0 = m0_of(rem);
      const int n0 = n_tile * BN;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, p.kblocks);
      const int nh = halves_of(rem);
      if constexpr (PP) {
        // Warpgroup g runs half-item g of every item.  The mainloops take turns: warpgroup 1 issues its first wgmma of an
        // item only after warpgroup 0 has issued all of its wgmmas of that item (named barrier kBarWg0Issued), and
        // warpgroup 0 starts the next item only after warpgroup 1 has issued its half (kBarWg1Issued), so each
        // warpgroup's epilogue runs while the other warpgroup's mainloop keeps the tensor pipe busy.  A skipped second
        // half passes the turn straight back.  Every item's turn is handed over exactly once each way, except that
        // warpgroup 0 waits for none before this CTA's first item and warpgroup 1 hands none back after its last.
        if (wg == 1 || it != 0) named_bar_sync(wg == 1 ? kBarWg0Issued : kBarWg1Issued, kConsumerWarps * 32);
        if (wg == 1 && nh == 1) {
          it += uint32_t(kb1 - kb0);
          if (item + stride < total) named_bar_arrive(kBarWg1Issued, kConsumerWarps * 32);
          continue;
        }
      }
      // ---------------- mainloop: one wgmma group in flight, the slot it read is released one k-block later
      int prev = -1;
      if constexpr (PP) {
        const uint32_t it0 = it + (wg == 1 ? uint32_t(kb1 - kb0) : 0u);
        stage = stage_of(it0);
        phase = phase_of(it0);
        it += uint32_t(nh * (kb1 - kb0));
      }
#pragma unroll 1
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_src = smem_base + stage * Cfg::STAGE_BYTES + (PP ? 0u : wg * A_WG_OFF);
        const uint32_t b_src = smem_base + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES;
        const uint32_t a_lo = ((a_src >> 4) & 0x3FFFu) | ((A_LBO >> 4) << 16);
        const uint32_t b_lo = ((b_src >> 4) & 0x3FFFu) | ((B_LBO >> 4) << 16);
        const uint32_t t_lo = (((b_src + B_BOXES * (BK * 128)) >> 4) & 0x3FFFu) | ((TAIL_LBO >> 4) << 16);
        wgmma_pin(acc);
        wgmma_fence();
        // all four k-steps, also in a ragged last k-block: TMA zero-fills the operands past K
#pragma unroll
        for (int k = 0; k < BK / kMmaK; ++k) {
          const uint64_t da = (uint64_t(DESC_HI) << 32) | (a_lo + k * (A_KADV >> 4));
          const uint64_t db = (uint64_t(DESC_HI) << 32) | (b_lo + k * (B_KADV >> 4));
          const uint32_t sc = (kb > kb0 || k > 0) ? 1u : 0u;
          if constexpr (BN == 256) wgmma_bf16_n256<A_MN, B_MN>(acc, da, db, sc);
          else if constexpr (kTail) {   // columns [0, 192) from the three boxes, [192, 208) from the tail box
            const uint64_t dt = (uint64_t(TAIL_DESC_HI) << 32) | (t_lo + k * (TAIL_KADV >> 4));
            wgmma_bf16_n192<A_MN, B_MN, 0>(acc, da, db, sc);
            wgmma_bf16_n16<A_MN, B_MN, 96>(acc, da, dt, sc);
          } else if constexpr (BN == 208) wgmma_bf16_n208<A_MN, B_MN>(acc, da, db, sc);
          else wgmma_bf16_n64<A_MN, B_MN>(acc, da, db, sc);
        }
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_pin(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      if constexpr (PP) {
        if (wg == 0 || item + stride < total) named_bar_arrive(wg == 0 ? kBarWg0Issued : kBarWg1Issued, kConsumerWarps * 32);
      }
      wgmma_wait<0>();
      wgmma_pin(acc);
      if (prev >= 0) release(prev);
      const int wrow0 = m0 + wg * 64 + (cw & 3) * 16;   // first row of this warp
      const int row = wrow0 + er;
      const bool row_ok = row < p.M;
      if (!A_MN && !(kUniversal && p.epi == EPI_F32)) {
        // ================= bf16 epilogue (K-major kernels) =================
        // coalesced lane mapping for aux reads / output writes: 8 lanes x 16 B = one 128-byte
        // row segment (a whole step), 4 rows per pass, 4 passes
        const int lr = lane >> 3, lc = lane & 7;
        constexpr int kBlocks = (BN + kEpiCols - 1) / kEpiCols;
        // aux tile (16 rows x 64 columns of the warp's next step):
        //  * kernels without bias / row-dot (dX, dHg, penalty T): cp.async straight into the
        //    warp's (otherwise unused) bias staging area, 128-byte rows with the 16-byte chunks
        //    XOR-swizzled by row & 7 so that the row-per-lane reads are conflict-free.
        //    No registers held across the step, no STS;
        //  * otherwise: coalesced LDG into registers, transposed through the scratch tile.
        constexpr bool kAuxAsync = !kUniversal && epi_aux(EPI) != AUX_NONE && epi_dot(EPI) == DOT_NONE && !epi_bias(EPI);
        const uint32_t auxt_s = vec_s;   // 16 rows x 128 B, chunks XOR-swizzled
        uint4 pre[kAuxAsync ? 1 : 4];
        auto aux_fetch = [&](int cs) {   // columns [cs, cs + 64) of the tile
          const int c = n0 + cs + lc * 8;
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rl = it * 4 + lr;
            const int r = wrow0 + rl;
            const bool ok = r < p.M && c < p.out_cols && cs + lc * 8 < BN;
            if constexpr (kAuxAsync) {
              const __nv_bfloat16* src = ok ? p.aux + size_t(r) * p.ld_aux + c : p.aux;
              cp_async16_zfill(auxt_s + rl * 128 + ((lc ^ (rl & 7)) << 4), src, ok ? 16u : 0u);
            } else {
              pre[it] = make_uint4(0, 0, 0, 0);
              if (ok) pre[it] = __ldg(reinterpret_cast<const uint4*>(p.aux + size_t(r) * p.ld_aux + c));
            }
          }
          if constexpr (kAuxAsync) cp_async_commit();
        };
        // bias / row-dot weights of the tile's column blocks -> smem and the first aux tile ->
        // registers before the fragments are read: no global-load latency after them
        if (has_bias || has_dot) {
#pragma unroll
          for (int pass = 0; pass < kEpiVecBlocks / 4; ++pass) {
            const int blk = pass * 4 + (lane >> 3), c4 = (lane & 7) * 4;   // 4 blocks x 8 float4 per pass
            const int c = n0 + blk * kEpiCols + c4;
            uint4 bz = make_uint4(0, 0, 0, 0), wz = bz;
            if (blk < kBlocks && c < p.N) {
              if (has_bias) {
                bz = __ldg(reinterpret_cast<const uint4*>(p.bias + c));
                if (act == ACT_SIGMOID) {   // sigmoid(x + b) = 0.5 tanh(0.5 x + 0.5 b) + 0.5: stage 0.5 b, one FFMA later
                  bz.x = __float_as_uint(0.5f * __uint_as_float(bz.x)); bz.y = __float_as_uint(0.5f * __uint_as_float(bz.y));
                  bz.z = __float_as_uint(0.5f * __uint_as_float(bz.z)); bz.w = __float_as_uint(0.5f * __uint_as_float(bz.w));
                }
              }
              if (has_dot) wz = __ldg(reinterpret_cast<const uint4*>(p.dot_w + c));
            }
            if (has_bias) sts128(vec_s + (blk * kEpiCols + c4) * 4, bz);
            if (has_dot) sts128(vec_s + kEpiVecBytes / 2 + (blk * kEpiCols + c4) * 4, wz);
          }
          __syncwarp();
        }
        if (aux_mode != AUX_NONE) {
          aux_fetch(0);
          // pull the aux tile of the NEXT tile this warp will process (same rows of the tile)
          // into L2 now: its loads are otherwise HBM-latency-bound
          const int nitem = item + stride;
          if (nitem < total) {
            const int nrem = nitem - (nitem / tiles) * tiles;
            const int nm0 = m0_of(nrem) + wg * 64 + (cw & 3) * 16;
            const int nn0 = n_tile_of(nrem) * BN;
            // 16 rows x 416 B: four 128-byte lines per row
            for (int t = lane; t < kEpiRows * 4; t += 32) {
              const int r = nm0 + (t >> 2), c = nn0 + (t & 3) * 64;
              if (r < p.M && c < p.out_cols)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(p.aux + size_t(r) * p.ld_aux + c));
            }
          }
        }
        float dot = 0.f;
        float l1_scale = 0.f;
        if (aux_mode == AUX_L1) l1_scale = __ldg(p.row_scale + (row < p.row_split ? 0 : 1));
        if (aux_mode == AUX_SIGMOID_GRAD || aux_mode == AUX_RELU_MASK || aux_mode == AUX_NONZERO_MASK) l1_scale = (p.row_vec != nullptr && row_ok) ? __ldg(p.row_vec + row) : 1.f;
#pragma unroll 1
        for (int s = 0; s < kSteps; ++s) {
          const int cs = s * kEpiStep;
          if (n0 + cs >= p.out_cols) break;
          const int bi = 2 * s + par;            // this lane's 32-column block of the tile
          const int cb = bi * kEpiCols;
          const int col0 = n0 + cb;
          const int nch = (cb >= BN || col0 >= p.out_cols) ? 0 : (BN - cb) >= kEpiCols ? 2 : (BN - cb) / 16;
          const bool last_step = (cs + kEpiStep >= BN) || (n0 + cs + kEpiStep >= p.out_cols);
          // full 64-column step -> one bulk tensor store per 32-column block of the (64-byte rows, XOR-swizzled) staging
          const bool step_tma = tma_st && BN - cs >= kEpiStep && wrow0 < p.M;
          // accumulator fragments -> scratch -> this lane's row: both chunks in flight, one wait
          stage_acquire();
          frag_to_scratch(s);
          __syncwarp();
          uint32_t raw[2][16];
#pragma unroll
          for (int q = 0; q < 2; ++q)
            if (q < nch && col0 + q * 16 < p.N) scratch_ld16(par * kEpiCols + q * 16, raw[q]);
          __syncwarp();
          uint4 ax[4];
          if (aux_mode != AUX_NONE) {   // prefetched aux (coalesced mapping) -> smem -> own row
            if constexpr (kAuxAsync) {
              cp_async_wait_all();
              __syncwarp();
#pragma unroll
              for (int q = 0; q < 4; ++q) ax[q] = lds128(auxt_s + er * 128 + (((4 * par + q) ^ (er & 7)) << 4));
            } else {
#pragma unroll
              for (int it = 0; it < 4; ++it) sts128(scratch_s + (it * 4 + lr) * kEpiPitch + lc * 16, pre[it]);
              __syncwarp();
#pragma unroll
              for (int q = 0; q < 4; ++q) ax[q] = lds128(scratch_s + er * kEpiPitch + par * 64 + q * 16);
            }
            __syncwarp();
            if (!last_step) aux_fetch(cs + kEpiStep);   // overlaps with this step's math + stores
          }
          uint4 axl[4] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
          if constexpr (SPLIT) {   // residual plane of the aux values of this lane's row (plain loads: the split kernels are not tuned)
            if (p.lo_off != 0 && aux_mode != AUX_NONE && aux_mode != AUX_RELU_MASK && aux_mode != AUX_NONZERO_MASK && row_ok) {
#pragma unroll
              for (int q = 0; q < 4; ++q)
                if (q < 2 * nch && col0 + q * 8 < p.out_cols)
                  axl[q] = __ldg(reinterpret_cast<const uint4*>(p.aux + p.lo_off + size_t(row) * p.ld_aux + col0 + q * 8));
            }
          }
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            if (q < nch) {
              const int c0 = col0 + q * 16;
              float v[16];
              if (c0 < p.N) {
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(raw[q][j]);
                if (has_bias) {
#pragma unroll
                  for (int k4 = 0; k4 < 4; ++k4) {
                    const uint4 b = lds128(vec_s + (bi * kEpiCols + q * 16 + k4 * 4) * 4);
                    if (act == ACT_SIGMOID) {   // staged bias is 0.5 b: v = 0.5 (acc + b), exact
                      v[4 * k4 + 0] = fmaf(v[4 * k4 + 0], 0.5f, __uint_as_float(b.x)); v[4 * k4 + 1] = fmaf(v[4 * k4 + 1], 0.5f, __uint_as_float(b.y));
                      v[4 * k4 + 2] = fmaf(v[4 * k4 + 2], 0.5f, __uint_as_float(b.z)); v[4 * k4 + 3] = fmaf(v[4 * k4 + 3], 0.5f, __uint_as_float(b.w));
                    } else {
                      v[4 * k4 + 0] += __uint_as_float(b.x); v[4 * k4 + 1] += __uint_as_float(b.y);
                      v[4 * k4 + 2] += __uint_as_float(b.z); v[4 * k4 + 3] += __uint_as_float(b.w);
                    }
                  }
                }
                if (act == ACT_RELU) {
                  if (!store_pre) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
                  }
                } else if (kUniversal && act == ACT_LRELU) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) v[j] = v[j] > 0.f ? v[j] : p.act_slope * v[j];
                } else if (act == ACT_SIGMOID) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) {
                    if constexpr (SPLIT) v[j] = 1.f / (1.f + __expf(has_bias ? -2.f * v[j] : -v[j]));   // fp32-grade (tanh.approx is 2^-11)
                    else v[j] = has_bias ? fast_sigmoid_half(v[j]) : fast_sigmoid(v[j]);
                  }
                }
                if (aux_mode != AUX_NONE) {
                  const uint32_t w[8] = {ax[2 * q].x, ax[2 * q].y, ax[2 * q].z, ax[2 * q].w,
                                         ax[2 * q + 1].x, ax[2 * q + 1].y, ax[2 * q + 1].z, ax[2 * q + 1].w};
                  const uint32_t wl[8] = {axl[2 * q].x, axl[2 * q].y, axl[2 * q].z, axl[2 * q].w,
                                          axl[2 * q + 1].x, axl[2 * q + 1].y, axl[2 * q + 1].z, axl[2 * q + 1].w};
#pragma unroll
                  for (int k2 = 0; k2 < 8; ++k2) {
                    float a_lo = bf16_lo(w[k2]), a_hi = bf16_hi(w[k2]);
                    if constexpr (SPLIT) { a_lo += bf16_lo(wl[k2]); a_hi += bf16_hi(wl[k2]); }
                    if (aux_mode == AUX_SIGMOID_GRAD) {
                      v[2 * k2] *= (l1_scale * a_lo) * (1.f - a_lo);
                      v[2 * k2 + 1] *= (l1_scale * a_hi) * (1.f - a_hi);
                    } else if (aux_mode == AUX_L1) {
                      // BEGAN: L1 reconstruction error of the autoencoder-discriminator and its
                      // (scaled) subgradient sign(r - x)   (src/be_gan.py:225-236)
                      const float d0 = v[2 * k2] - a_lo, d1 = v[2 * k2 + 1] - a_hi;
                      dot += fabsf(d0) + fabsf(d1);
                      v[2 * k2] = d0 > 0.f ? l1_scale : (d0 < 0.f ? -l1_scale : 0.f);
                      v[2 * k2 + 1] = d1 > 0.f ? l1_scale : (d1 < 0.f ? -l1_scale : 0.f);
                    } else if (aux_mode == AUX_VAE_OUT) {
                      // v = decoder output, aux = target x: accumulate (x-v)^2 and emit
                      // d/d(pre-sigmoid) of sum (x-v)^2 = -2 (x-v) v (1-v)   (src/vae.py:203)
                      const float d0 = a_lo - v[2 * k2], d1 = a_hi - v[2 * k2 + 1];
                      dot = fmaf(d0, d0, dot); dot = fmaf(d1, d1, dot);
                      v[2 * k2] = -2.f * d0 * v[2 * k2] * (1.f - v[2 * k2]);
                      v[2 * k2 + 1] = -2.f * d1 * v[2 * k2 + 1] * (1.f - v[2 * k2 + 1]);
                    } else {
                      // aux > 0 (post-ReLU activation), or aux != 0 for the signed mask form w2 * relu'(a)
                      const bool on0 = aux_mode == AUX_NONZERO_MASK ? a_lo != 0.f : a_lo > 0.f;
                      const bool on1 = aux_mode == AUX_NONZERO_MASK ? a_hi != 0.f : a_hi > 0.f;
                      v[2 * k2] = on0 ? v[2 * k2] * l1_scale : 0.f;
                      v[2 * k2 + 1] = on1 ? v[2 * k2 + 1] * l1_scale : 0.f;
                    }
                  }
                }
                if (has_sq) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) dot = fmaf(v[j], v[j], dot);
                }
                if (has_dot) {
#pragma unroll
                  for (int k4 = 0; k4 < 4; ++k4) {
                    const uint4 w = lds128(vec_s + kEpiVecBytes / 2 + (bi * kEpiCols + q * 16 + k4 * 4) * 4);
                    if (store_pre) {   // v holds pre-activations: the activation enters the dot product only
                      dot = fmaf(fmaxf(v[4 * k4 + 0], 0.f), __uint_as_float(w.x), dot); dot = fmaf(fmaxf(v[4 * k4 + 1], 0.f), __uint_as_float(w.y), dot);
                      dot = fmaf(fmaxf(v[4 * k4 + 2], 0.f), __uint_as_float(w.z), dot); dot = fmaf(fmaxf(v[4 * k4 + 3], 0.f), __uint_as_float(w.w), dot);
                    } else {
                      dot = fmaf(v[4 * k4 + 0], __uint_as_float(w.x), dot); dot = fmaf(v[4 * k4 + 1], __uint_as_float(w.y), dot);
                      dot = fmaf(v[4 * k4 + 2], __uint_as_float(w.z), dot); dot = fmaf(v[4 * k4 + 3], __uint_as_float(w.w), dot);
                    }
                    if (mask_all) {
                      v[4 * k4 + 0] = v[4 * k4 + 0] > 0.f ? __uint_as_float(w.x) : 0.f;
                      v[4 * k4 + 1] = v[4 * k4 + 1] > 0.f ? __uint_as_float(w.y) : 0.f;
                      v[4 * k4 + 2] = v[4 * k4 + 2] > 0.f ? __uint_as_float(w.z) : 0.f;
                      v[4 * k4 + 3] = v[4 * k4 + 3] > 0.f ? __uint_as_float(w.w) : 0.f;
                    }
                  }
                }
              } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] = 0.f;
                if (c0 == p.N && p.pad_one) v[0] = 1.f;
              }
              {
                const uint4 lo = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
                const uint4 hi = make_uint4(pack_bf16x2(v[8], v[9]), pack_bf16x2(v[10], v[11]), pack_bf16x2(v[12], v[13]), pack_bf16x2(v[14], v[15]));
                if constexpr (SPLIT) {   // residual plane of the output: v - bf16(v), straight from registers
                  if (p.lo_off != 0 && p.out != nullptr && row_ok && c0 < p.out_cols) {
                    uint4* ol = reinterpret_cast<uint4*>(p.out + size_t(row) * p.ldo + p.lo_off + c0);
                    ol[0] = make_uint4(pack_bf16x2_residual(v[0], v[1], lo.x), pack_bf16x2_residual(v[2], v[3], lo.y),
                                       pack_bf16x2_residual(v[4], v[5], lo.z), pack_bf16x2_residual(v[6], v[7], lo.w));
                    ol[1] = make_uint4(pack_bf16x2_residual(v[8], v[9], hi.x), pack_bf16x2_residual(v[10], v[11], hi.y),
                                       pack_bf16x2_residual(v[12], v[13], hi.z), pack_bf16x2_residual(v[14], v[15], hi.w));
                  }
                }
                if (step_tma) {
                  const uint32_t sw = (er >> 1) & 3, rowb = scratch_s + par * (kEpiRows * kEpiCols * 2) + er * 64;
                  sts128(rowb + (((2 * q) ^ sw) << 4), lo);
                  sts128(rowb + (((2 * q + 1) ^ sw) << 4), hi);
                } else {
                  sts128(scratch_s + er * kEpiPitch + par * 64 + q * 32, lo);
                  sts128(scratch_s + er * kEpiPitch + par * 64 + q * 32 + 16, hi);
                }
              }
            }
          }
          if (step_tma) {
            fence_proxy_async_smem();
            __syncwarp();
            if (er == 0 && nch == 2) {
              tma_store_2d(&tmC, scratch_s + par * (kEpiRows * kEpiCols * 2), col0, wrow0);
              bulk_commit();
            }
            st_pending = true;
          } else {
            __syncwarp();
            // coalesced store: 8 lanes cover the step's 128 contiguous bytes of one row, 4 rows per pass
            const int oc = n0 + cs + lc * 8;
            if (p.out != nullptr && cs + lc * 8 < BN && oc < p.out_cols) {
              __nv_bfloat16* o = p.out + size_t(wrow0 + lr) * p.ldo + oc;
              const uint32_t sa = scratch_s + lr * kEpiPitch + lc * 16;
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const int rr = wrow0 + it * 4 + lr;
                if (rr < p.M) {
                  __nv_bfloat16* dst = o + size_t(it * 4) * p.ldo;
                  *reinterpret_cast<uint4*>(dst) = lds128(sa + it * 4 * kEpiPitch);
                }
              }
            }
            __syncwarp();
          }
        }
        if ((has_dot || has_sq || aux_mode == AUX_VAE_OUT || aux_mode == AUX_L1) && p.dot_out != nullptr && row_ok)
          p.dot_out[size_t(n_tile * 2 + par) * p.dot_ld + row] = dot;
      } else {
        // ====== fp32 epilogue: split-K partials (MN-major kernels) or biased fp32 output ======
        float* base = p.part + size_t(split) * p.part_stride;
#pragma unroll 1
        for (int s = 0; s < kSteps; ++s) {
          if (n0 + s * kEpiStep >= p.N) break;
          frag_to_scratch(s);
          __syncwarp();
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int c = s * kEpiStep + par * kEpiCols + q * 16;   // tile column of this lane's 16-column chunk
            const int col0 = n0 + c;
            if (c >= BN || col0 >= p.N) continue;
            float v[16];
            {
              uint32_t raw[16];
              scratch_ld16(par * kEpiCols + q * 16, raw);
#pragma unroll
              for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(raw[j]);
            }
            if (p.bias != nullptr) {
#pragma unroll
              for (int j = 0; j < 16; ++j)
                if (col0 + j < p.N) v[j] += __ldg(p.bias + col0 + j);
            }
            if (row_ok) {
              if (p.transpose) {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                  if (col0 + j < p.N) base[size_t(col0 + j) * p.ldp + row] = v[j];
              } else if (p.f32_vec && col0 + 16 <= p.N) {
                float4* o = reinterpret_cast<float4*>(base + size_t(row) * p.ldp + col0);
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) o[k4] = make_float4(v[4 * k4], v[4 * k4 + 1], v[4 * k4 + 2], v[4 * k4 + 3]);
              } else {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                  if (col0 + j < p.N) base[size_t(row) * p.ldp + col0 + j] = v[j];
              }
            }
          }
          __syncwarp();
        }
      }
    }
    stage_acquire();   // the last bulk store has read its staging tile before shared memory goes away
  }
  // no CTA exits while a peer may still arrive on its barriers (its multicasts have all landed: every stage was consumed)
  if constexpr (CL > 1) cluster_sync();
  else __syncthreads();
}

}  // namespace gm
