// Non-GEMM kernels of the train step: input staging, per-variant loss + upstream
// gradient, hidden-layer backward, gradient finalisation, fused Adam (+ bf16
// operand shadows).  All HBM-bound or tiny; 128-bit accesses where it matters.
#pragma once
#include <curand_kernel.h>

#include "ptx.cuh"

namespace gm {

// ---------------------------------------------------------------- variants
// Order is the ABI (include/gm_b200.h: gm_variant).
enum : int {
  V_NS = 0, V_MM, V_W, V_WGP, V_LS, V_DRA, V_RA, V_FISHER,
  V_F_TV, V_F_FKL, V_F_RKL, V_F_PEARSON, V_F_HELLINGER, V_F_JS, V_INFO, V_BEGAN
};
enum : int { OUT_SIGMOID = 0, OUT_RELU = 1, OUT_NONE = 2 };
constexpr float kEps = 1e-8f;  // the reference's log stabiliser (src/ns_gan.py:191)

// ---------------------------------------------------------------- staging
// images (fp32 | u8 | 1-bit packed, {0,1}) -> bf16 rows [n, ld] with a ones column at
// `x` (bias-gradient trick: dW GEMMs then produce db as one extra row) and zero pad.
// Optional row gather (idx != nullptr): row r reads source row idx[r].
enum : int { IMG_F32 = 0, IMG_U8 = 1, IMG_BITS = 2, IMG_BF16PAD = 3 };

// On-device batch sampling (the DataLoader shuffle of src/ns_gan.py:222-226, src/vae.py:150): row r of
// the batch reads source row perm_key(offset + r), perm_key a pseudo-random PERMUTATION of [0, n) - a
// 4-round Feistel network over the next even power of two, cycle-walked back into range - so the rows
// of one batch are distinct, exactly like the first batch of a freshly shuffled DataLoader (GANs: a new
// key every step, offset 0) or like batch k of one epoch's permutation (VAE: key per epoch, offset k*B).
// n == 0 switches sampling off.
struct Sampler {
  unsigned int n, half_bits;
  unsigned long long key, offset;
  // device-step mode (CUDA-graph replay): the permutation's round comes from a device counter, key = f(seed_mix, *step_ptr)
  const unsigned long long* step_ptr;
  unsigned long long seed_mix;
};
__host__ __device__ __forceinline__ unsigned long long splitmix64_hd(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ unsigned long long sampler_key(unsigned long long seed_mix, unsigned long long round) {
  return splitmix64_hd(seed_mix ^ (round * 0xD1342543DE82EF95ull + 0x2545F4914F6CDD1Dull));
}
__host__ __device__ __forceinline__ unsigned int sampler_mix(unsigned int x, unsigned int k) {
  x ^= k; x *= 0x9E3779B1u; x ^= x >> 15; x *= 0x85EBCA77u; x ^= x >> 13; x *= 0xC2B2AE3Du; x ^= x >> 16;
  return x;
}
__host__ __device__ __forceinline__ unsigned int sampler_index(const Sampler& sp, unsigned long long pos) {
  const unsigned int mask = (1u << sp.half_bits) - 1u;
  const unsigned int k0 = (unsigned int)sp.key, k1 = (unsigned int)(sp.key >> 32);
  unsigned int i = (unsigned int)(pos % sp.n);
  do {
    unsigned int L = i >> sp.half_bits, R = i & mask;
#pragma unroll
    for (int rnd = 0; rnd < 4; ++rnd) {
      const unsigned int F = sampler_mix(R, (rnd & 1 ? k1 : k0) + 0x632BE5ABu * (unsigned int)(rnd + 1)) & mask;
      const unsigned int t = L ^ F;
      L = R; R = t;
    }
    i = (L << sp.half_bits) | R;
  } while (i >= sp.n);
  return i;
}

__global__ void stage_images_kernel(const void* __restrict__ src, int fmt, const int* __restrict__ idx,
                                    __nv_bfloat16* __restrict__ dst, int rows, int x, int ld, const Sampler smp_in, long long lo_off) {
  griddep_sync();
  const int groups = ld / 8;
  const long long total = (long long)rows * groups;
  Sampler smp = smp_in;
  if (smp.step_ptr) smp.key = sampler_key(smp.seed_mix, *smp.step_ptr);
  if (lo_off) {   // split mode: {0,1} pixels are exact in bf16 -> the rows' residual plane is zero (it may hold a previous tenant's values)
    uint4* lo = reinterpret_cast<uint4*>(dst + lo_off);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
      lo[i] = make_uint4(0, 0, 0, 0);
  }
  auto src_row = [&](int r) -> long long {
    if (idx) return (long long)idx[r];
    if (smp.n) return (long long)sampler_index(smp, smp.offset + (unsigned long long)r);
    return (long long)r;
  };
  if (fmt == IMG_BITS && (x & 7) == 0) {
    // One warp per row: lanes walk the row's 8-pixel groups (one packed byte, MSB first, expands
    // to 8 bf16 = one 16-byte store), 4 passes in flight; no index divisions, the gather index
    // of the next row is fetched while this row is expanded.  Bound by the 16-byte stores.
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int xb = x >> 3;   // source bytes per row; group xb holds the ones column
    long long sr_next = w < rows ? src_row(w) : 0;
    for (int r = w; r < rows; r += nwarps) {
      const long long sr = sr_next;
      if (r + nwarps < rows) sr_next = src_row(r + nwarps);
      const uint8_t* srow = reinterpret_cast<const uint8_t*>(src) + sr * xb;
      uint4* drow = reinterpret_cast<uint4*>(dst) + (long long)r * groups;
      for (int g0 = 0; g0 < groups; g0 += 128) {
        uint32_t byte[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int g = g0 + u * 32 + lane;
          byte[u] = g < xb ? uint32_t(__ldg(srow + g)) : (g == xb ? 0x80u : 0u);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int g = g0 + u * 32 + lane;
          if (g >= groups) break;
          const uint32_t b = byte[u];
          // bf16 1.0 = 0x3F80: build the four packed pairs without float conversions
          auto pr = [&](int hi_bit, int lo_bit) { return ((b >> lo_bit) & 1u ? 0x3F80u : 0u) | ((b >> hi_bit) & 1u ? 0x3F800000u : 0u); };
          drow[g] = make_uint4(pr(6, 7), pr(4, 5), pr(2, 3), pr(0, 1));
        }
      }
    }
    return;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = int(i / groups), g = int(i % groups);
    const long long sr = src_row(r);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = g * 8 + j;
      float f = 0.f;
      if (c < x) {
        if (fmt == IMG_F32) f = reinterpret_cast<const float*>(src)[sr * x + c];
        else if (fmt == IMG_U8) f = reinterpret_cast<const uint8_t*>(src)[sr * x + c] ? 1.f : 0.f;
        else if (fmt == IMG_BITS) {
          const long long bit = sr * x + c;  // np.packbits order: MSB first
          f = (reinterpret_cast<const uint8_t*>(src)[bit >> 3] >> (7 - (bit & 7))) & 1 ? 1.f : 0.f;
        } else f = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(src)[sr * ld + c]);
      } else if (c == x) f = 1.f;
      v[j] = f;
    }
    store_bf16x8(dst + i * 8, v, lo_off);     // grey-level fp32 inputs keep their residuals in split mode
  }
}

// the batch's source-row indices as the staging kernel draws them (tests, gm_sample_indices)
__global__ void sample_indices_kernel(const Sampler smp_in, int rows, int* __restrict__ out) {
  griddep_sync();
  Sampler smp = smp_in;
  if (smp.step_ptr) smp.key = sampler_key(smp.seed_mix, *smp.step_ptr);
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) out[r] = smp.n ? int(sampler_index(smp, smp.offset + (unsigned long long)r)) : r;
}

// noise fp32 [rows, z] (or Philox N(0,1) when src == nullptr) -> bf16 [rows, ld], ones col at z.
// One thread per (row, 8-column group); the Philox subsequence is the group index, the
// offset the step stream, so every step / rank / group draws disjoint numbers.
__global__ void stage_noise_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int rows,
                                   int z, int ld, unsigned long long seed, unsigned long long stream_id, long long lo_off,
                                   const unsigned long long* __restrict__ step_ptr) {
  griddep_sync();
  if (step_ptr) stream_id += 2ull * (*step_ptr);      // device-step mode: stream = 2 * step (+ 1 for train_G)
  // One thread per (row, 8-column group that holds noise): every lane runs the Philox /
  // Box-Muller path (a thread per group of the padded row left 5 of 8 lanes idle in it).
  // The thread also writes its share of the row's zero padding groups.
  const int groups = ld / 8, gz = (z + 8) / 8;   // gz: groups holding noise or the ones column
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)rows * gz) return;
  const int r = int(t / gz), g = int(t % gz), c0 = g * 8;
  const long long i = (long long)r * groups + g;   // cell index = Philox subsequence
  float v[8];
  if (c0 < z) {
    if (src == nullptr) {
      curandStatePhilox4_32_10_t st;
      curand_init(seed, (unsigned long long)i, stream_id * 2ull, &st);
      const float4 a = curand_normal4(&st), b = curand_normal4(&st);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c0 + j < z) ? src[(long long)r * z + c0 + j] : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    if (c >= z) v[j] = (c == z) ? 1.f : 0.f;
  }
  uint4* row = reinterpret_cast<uint4*>(dst) + (long long)r * groups;
  store_bf16x8(dst + ((long long)r * groups + g) * 8, v, lo_off);
  for (int pg = gz + g; pg < groups; pg += gz) {
    row[pg] = make_uint4(0, 0, 0, 0);
    if (lo_off) reinterpret_cast<uint4*>(dst + lo_off)[(long long)r * groups + pg] = make_uint4(0, 0, 0, 0);
  }
}

// ---------------------------------------------------------------- block reduction (deterministic)
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < NT / 32; ++i) t += sh[i];
  return t;
}

// ---------------------------------------------------------------- loss + upstream gradient
// Reads the row-dot partial slots the D-layer GEMM epilogue wrote, forms the
// logit s = sum(slots) + b2, D's output d (sigmoid / relu / id) and, per variant
// (SURVEY.md A.1), the loss and dL/ds for each row.  D step: rows [0,B) real,
// [B,2B) fake.  G step: B fake rows.  `inv_b` = 1/(global batch) so data-parallel
// ranks can SUM gradients.  Loss means are over the local batch.
struct LossParams {
  const float* slots; int nslots; int slot_ld;   // slots[k*slot_ld + row]
  const float* b2;
  int B;                 // local batch
  int Bstat;             // batch the statistics (RaNS mean, Fisher moments) run over: B x world when ranks exchange them
  int g_step;            // 0: D step (2B rows), 1: G step (B rows, all fake)
  int variant, out_act;
  float inv_b;
  float* ds;             // out: dL/ds per row
  float* d_out;          // out (nullable): D output per row
  float* loss;           // out: [0] loss  [1] sum(ds) (= db2 grad)  [2..] variant scratch
  float* fisher;         // [0] LAMBDA  [1] RHO  (device state, V_FISHER only)
  float ls_a, ls_b, ls_c;   // LSGAN targets: fake (a), real (b) in train_D, c in train_G (src/ls_gan.py:173,197)
  double* partA; double* partB; double* partR;   // per-block partials [nblk][4]
  int nblk;
  unsigned int* done;    // block-completion counter of PASS 2 (self-resetting): the last block finalises
};

__device__ __forceinline__ float act_out(float s, int a) {
  return a == OUT_SIGMOID ? 1.f / (1.f + expf(-s)) : (a == OUT_RELU ? fmaxf(s, 0.f) : s);
}
__device__ __forceinline__ float act_grad(float s, float d, int a) {
  return a == OUT_SIGMOID ? d * (1.f - d) : (a == OUT_RELU ? (s > 0.f ? 1.f : 0.f) : 1.f);
}

// Multi-block passes.  Every pass writes per-block partial sums (doubles, fixed tree ->
// deterministic); a later pass re-reduces the earlier partials redundantly per block.
//   PASS 0 (RA, Fisher): sum d, d^2 per branch            -> partA[blk][4]
//   PASS 1 (RA):         sum q(1-q)/(q+eps) over real rows -> partB[blk][4] (slot 0)
//   PASS 2 (all):        per-row loss term + dL/ds         -> partR[blk][4] (loss, sum ds)
// The last PASS 2 block to finish (loss_finalize) reduces partR into loss[0..1] and applies the Fisher
// lambda update (src/fisher_gan.py:155).
constexpr int kLossThreads = 256;

__device__ __forceinline__ double reduce_partials4(const double* part, int nblk, int slot, double* sh) {
  double t = 0.0;
  for (int i = threadIdx.x; i < nblk; i += kLossThreads) t += part[(long long)i * 4 + slot];
  return block_sum<kLossThreads>(t, sh);
}

// loss[0..1] from the PASS 2 partials (+ the Fisher lambda update, src/fisher_gan.py:155); one block
__device__ __forceinline__ void loss_finalize(const LossParams& p, double* sh) {
  const double lsum = reduce_partials4(p.partR, p.nblk, 0, sh);
  const double dssum = reduce_partials4(p.partR, p.nblk, 1, sh);
  double s2 = 0, s3 = 0;
  const bool fisher = !p.g_step && p.variant == V_FISHER;
  if (fisher) { s2 = reduce_partials4(p.partA, p.nblk, 2, sh); s3 = reduce_partials4(p.partA, p.nblk, 3, sh); }
  if (threadIdx.x == 0) {
    float L = float(lsum / p.B);
    if (fisher) {
      const float lam = p.fisher[0], rho = p.fisher[1];
      const float omega = 1.f - (0.5f * float(s2 / p.Bstat) + 0.5f * float(s3 / p.Bstat));
      L = L - lam * omega + 0.5f * rho * omega * omega;   // src/fisher_gan.py:221-223
      p.fisher[0] = lam + rho * (-omega);                 // src/fisher_gan.py:155: lambda += rho * dL/dlambda
      p.loss[2] = omega;
    }
    p.loss[0] = L;
    p.loss[1] = float(dssum);
  }
}

template <int PASS>
__global__ void __launch_bounds__(kLossThreads) loss_pass_kernel(const LossParams p) {
  griddep_sync();
  __shared__ double sh[kLossThreads / 32];
  const int rows = p.g_step ? p.B : 2 * p.B;
  const float b2 = p.b2[0];
  auto logit = [&](int r) {
    float s = 0.f;
    for (int k = 0; k < p.nslots; ++k) s += p.slots[(long long)k * p.slot_ld + r];
    return s + b2;
  };
  float mg = 0.f, gq_mean = 0.f, c_f = 0.f;
  if (PASS >= 1 && !p.g_step && (p.variant == V_RA || p.variant == V_FISHER)) {
    const double s1 = reduce_partials4(p.partA, p.nblk, 1, sh);
    mg = float(s1 / p.Bstat);
    if (p.variant == V_FISHER) {
      const double s2 = reduce_partials4(p.partA, p.nblk, 2, sh), s3 = reduce_partials4(p.partA, p.nblk, 3, sh);
      const float omega = 1.f - (0.5f * float(s2 / p.Bstat) + 0.5f * float(s3 / p.Bstat));
      c_f = p.fisher[0] - p.fisher[1] * omega;
    } else if (PASS == 2) {
      gq_mean = float(reduce_partials4(p.partB, p.nblk, 0, sh) / p.Bstat);
    }
  }
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  const float ib = p.inv_b;
  for (int r = blockIdx.x * kLossThreads + threadIdx.x; r < rows; r += gridDim.x * kLossThreads) {
    const float s = logit(r), d = act_out(s, p.out_act);
    const bool fake = p.g_step || r >= p.B;
    if (PASS == 0) {
      if (!fake) { a0 += d; a2 += (double)d * d; } else { a1 += d; a3 += (double)d * d; }
      continue;
    }
    if (PASS == 1) {
      if (!fake) { const float q = 1.f / (1.f + expf(-(d - mg))); a0 += q * (1.f - q) / (q + kEps); }
      continue;
    }
    float l = 0.f, g = 0.f;  // per-row loss term (to be averaged) and dL/dd * B
    if (p.g_step) {
      switch (p.variant) {
        case V_NS: case V_DRA: case V_RA: case V_INFO: l = -logf(d + kEps); g = -1.f / (d + kEps); break;
        case V_MM: l = logf((1.f - d) + kEps); g = -1.f / ((1.f - d) + kEps); break;
        case V_W: case V_WGP: case V_FISHER: l = -d; g = -1.f; break;
        case V_LS: l = 0.5f * (d - p.ls_c) * (d - p.ls_c); g = d - p.ls_c; break;
        case V_F_TV: { const float t = tanhf(d); l = -0.5f * t; g = -0.5f * (1.f - t * t); } break;
        case V_F_FKL: { const float e = expf(d - 1.f); l = -e; g = -e; } break;
        case V_F_RKL: l = 1.f + d; g = 1.f; break;
        case V_F_PEARSON: l = -(0.25f * d * d + d); g = -(0.5f * d + 1.f); break;
        case V_F_HELLINGER: { const float e = expf(-d); l = -(e - 1.f); g = e; } break;
        case V_F_JS: { const float e = expf(d); l = 2.f - e; g = -e; } break;
      }
    } else if (!fake) {
      switch (p.variant) {
        case V_NS: case V_MM: case V_DRA: case V_INFO: l = -logf(d + kEps); g = -1.f / (d + kEps); break;
        case V_W: case V_WGP: l = -d; g = -1.f; break;
        case V_LS: l = 0.5f * (d - p.ls_b) * (d - p.ls_b); g = d - p.ls_b; break;
        case V_RA: { const float q = 1.f / (1.f + expf(-(d - mg)));
                     l = -0.5f * logf(q + kEps); g = -0.5f * q * (1.f - q) / (q + kEps); } break;
        case V_FISHER: l = -d; g = -(1.f - c_f * d); break;   // lambda/rho terms added once in loss_final
        case V_F_TV: { const float t = tanhf(d); l = -0.5f * t; g = -0.5f * (1.f - t * t); } break;
        case V_F_FKL: l = -d; g = -1.f; break;
        case V_F_RKL: { const float e = expf(d); l = e; g = e; } break;
        case V_F_PEARSON: l = -d; g = -1.f; break;
        case V_F_HELLINGER: { const float e = expf(d); l = -(1.f - e); g = e; } break;
        case V_F_JS: { const float e = expf(-d); l = -(1.f - e); g = -e; } break;
      }
    } else {
      switch (p.variant) {
        case V_NS: case V_MM: case V_DRA: case V_INFO: l = -logf((1.f - d) + kEps); g = 1.f / ((1.f - d) + kEps); break;
        case V_W: case V_WGP: l = d; g = 1.f; break;
        case V_LS: l = 0.5f * (d - p.ls_a) * (d - p.ls_a); g = d - p.ls_a; break;
        case V_RA: { const float q = 1.f / (1.f + expf(-(1.f - d)));
                     l = -0.5f * logf(q + kEps); g = 0.5f * (gq_mean + q * (1.f - q) / (q + kEps)); } break;
        case V_FISHER: l = d; g = 1.f + c_f * d; break;
        case V_F_TV: { const float t = tanhf(d); l = 0.5f * t; g = 0.5f * (1.f - t * t); } break;
        case V_F_FKL: { const float e = expf(d - 1.f); l = e; g = e; } break;
        case V_F_RKL: l = -1.f - d; g = -1.f; break;
        case V_F_PEARSON: l = 0.25f * d * d + d; g = 0.5f * d + 1.f; break;
        case V_F_HELLINGER: { const float e = expf(-d); l = e - 1.f; g = -e; } break;
        case V_F_JS: { const float e = expf(d); l = -(2.f - e); g = e; } break;
      }
    }
    const float dsr = g * ib * act_grad(s, d, p.out_act);
    p.ds[r] = dsr;
    if (p.d_out) p.d_out[r] = d;
    a0 += l;
    a1 += dsr;
  }
  a0 = block_sum<kLossThreads>(a0, sh); a1 = block_sum<kLossThreads>(a1, sh);
  a2 = block_sum<kLossThreads>(a2, sh); a3 = block_sum<kLossThreads>(a3, sh);
  if (threadIdx.x == 0) {
    double* out = (PASS == 0 ? p.partA : (PASS == 1 ? p.partB : p.partR)) + (long long)blockIdx.x * 4;
    out[0] = a0; out[1] = a1; out[2] = a2; out[3] = a3;
  }
  if (PASS == 2) {
    // the last block to finish reduces every block's partials (fixed order -> deterministic) instead
    // of a separate one-block launch
    __shared__ bool last;
    if (threadIdx.x == 0) {
      __threadfence();
      last = atomicAdd(p.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last) {
      __threadfence();
      loss_finalize(p, sh);
      if (threadIdx.x == 0) *p.done = 0u;
    }
  }
}

// D's output for inference: d[r] = act(sum(slots[:, r]) + b2)
__global__ void scores_kernel(const float* __restrict__ slots, int nslots, int slot_ld, const float* __restrict__ b2,
                              int out_act, float* __restrict__ out, int rows) {
  griddep_sync();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float s = 0.f;
  for (int k = 0; k < nslots; ++k) s += slots[(long long)k * slot_ld + r];
  out[r] = act_out(s + b2[0], out_act);
}

// out[c] = sum_p part[p*ld + c]: one warp per column (deterministic shuffle tree)
__global__ void colsum_kernel(const float* __restrict__ part, int nparts, int ld, int cols, float* __restrict__ out) {
  griddep_sync();
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= cols) return;
  float t = 0.f;
  for (int i = lane; i < nparts; i += 32) t += part[(long long)i * ld + c];
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (lane == 0) out[c] = t;
}

// ---------------------------------------------------------------- hidden-layer backward of D
// dh[r,n] = ds[r] * w2[n] * 1[a[r,n] > 0] (bf16), and (optionally) per-block partial
// column sums dw2p[block, n] = sum_r ds[r] * a[r,n].  One uint4 (8 bf16) per thread;
// blockDim = (ld/8) * rows_per_iter so a thread always owns the same 8 columns.
__global__ void dh_kernel(const __nv_bfloat16* __restrict__ a, const float* __restrict__ ds,
                          const float* __restrict__ w2, __nv_bfloat16* __restrict__ dh, float* __restrict__ dw2p,
                          int rows, int h, int ld, int rows_per_iter, long long lo_off, int pre) {
  // pre != 0: `a` holds PRE-activations (WGAN-GP's D forward, GemmParams.dot == DOT_W_PRE): relu is applied here
  griddep_sync();
  extern __shared__ float sh_acc[];  // [rows_per_iter][ld]
  const int groups = ld / 8;
  const int g = threadIdx.x % groups, rl = threadIdx.x / groups;
  float w[8], acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    w[j] = c < h ? w2[c] : 0.f;
    acc[j] = 0.f;
  }
  // 4 independent rows in flight per thread (memory-level parallelism: this kernel is HBM-bound)
  const long long stride = (long long)gridDim.x * rows_per_iter;
  for (long long r0 = (long long)blockIdx.x * rows_per_iter + rl; r0 < rows; r0 += 4 * stride) {
    uint4 av[4], al[4];
    float dv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * stride;
      av[u] = make_uint4(0, 0, 0, 0);
      al[u] = make_uint4(0, 0, 0, 0);
      dv[u] = 0.f;
      if (r < rows) {
        av[u] = __ldg(reinterpret_cast<const uint4*>(a + r * ld) + g);
        if (lo_off) al[u] = __ldg(reinterpret_cast<const uint4*>(a + lo_off + r * ld) + g);
        dv[u] = ds ? ds[r] : 1.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * stride;
      if (r >= rows) break;
      const float d = dv[u];
      const uint32_t w4[4] = {av[u].x, av[u].y, av[u].z, av[u].w};
      const uint32_t l4[4] = {al[u].x, al[u].y, al[u].z, al[u].w};
      float o[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float lo = bf16_lo(w4[q]), hi = bf16_hi(w4[q]);   // the sign of the hi part is the sign of the value
        o[2 * q] = lo > 0.f ? d * w[2 * q] : 0.f;
        o[2 * q + 1] = hi > 0.f ? d * w[2 * q + 1] : 0.f;
        const float a0 = (pre && !(lo > 0.f)) ? 0.f : lo + bf16_lo(l4[q]);
        const float a1 = (pre && !(hi > 0.f)) ? 0.f : hi + bf16_hi(l4[q]);
        acc[2 * q] = fmaf(d, a0, acc[2 * q]);
        acc[2 * q + 1] = fmaf(d, a1, acc[2 * q + 1]);
      }
      if (dh != nullptr) store_bf16x8(dh + r * ld + g * 8, o, lo_off);
    }
  }
  if (dw2p == nullptr) return;
#pragma unroll
  for (int j = 0; j < 8; ++j) sh_acc[rl * ld + g * 8 + j] = acc[j];
  __syncthreads();
  for (int c = threadIdx.x; c < ld; c += blockDim.x) {
    float t = 0.f;
    for (int i = 0; i < rows_per_iter; ++i) t += sh_acc[i * ld + c];
    dw2p[(long long)blockIdx.x * ld + c] = t;
  }
}

// ---------------------------------------------------------------- gradient penalty (WGAN-GP, DRAGAN)
// DRAGAN's xhat rows (src/dra_gan.py:200-205, bf16, ld, zero pad, ones column at x: they carry a true backward path):
//   xhat = delta*x + (1-delta)*(x + std*u), delta per row, u per element
// rnd == nullptr: on-device Philox (row stream), else caller tensors: delta[rows] followed by u[rows*x].
// stats: [0] sum x, [1] sum x^2, [2] count over the real rows.
__global__ void xhat_kernel(const __nv_bfloat16* __restrict__ xr, __nv_bfloat16* __restrict__ out, int rows, int x, int ld,
                            const float* __restrict__ rnd, const float* __restrict__ stats,
                            unsigned long long seed, unsigned long long stream_id, float dra_c, long long lo_off,
                            const unsigned long long* __restrict__ step_ptr) {
  griddep_sync();
  if (step_ptr) stream_id += 2ull * (*step_ptr);
  // One warp per row, lanes walk the row's 16-byte groups (coalesced, unlike a thread-per-row
  // mapping).  Philox: the row's delta comes from subsequence r (lane-uniform), the per-element
  // u from subsequence rows + r * groups + g.
  const int groups = ld / 8;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const double n = stats[2], s1 = stats[0], s2 = stats[1];
  const float sd = dra_c * float(sqrt(fmax((s2 - s1 * s1 / n) / (n - 1.0), 0.0)));   // C * images.std(): unbiased, global (src/dra_gan.py:204-205)
  for (int r = w; r < rows; r += nwarps) {
    float e;
    if (rnd) e = rnd[r];
    else {
      curandStatePhilox4_32_10_t st;
      curand_init(seed ^ 0x9E3779B97F4A7C15ull, (unsigned long long)r, stream_id * 256ull, &st);
      e = curand_uniform(&st);   // (0,1]; the reference's rand is [0,1)
    }
    for (int g = lane; g < groups; g += 32) {
      const int c0 = g * 8;
      float va[8], v[8], u[8];
      load_bf16x8(xr + (long long)r * ld + c0, va, lo_off);
      if (rnd == nullptr && c0 < x) {
        curandStatePhilox4_32_10_t su;
        curand_init(seed ^ 0x9E3779B97F4A7C15ull, (unsigned long long)rows + (unsigned long long)r * groups + g, stream_id * 256ull, &su);
        const float4 a = curand_uniform4(&su), b = curand_uniform4(&su);
        u[0] = a.x; u[1] = a.y; u[2] = a.z; u[3] = a.w; u[4] = b.x; u[5] = b.y; u[6] = b.z; u[7] = b.w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        float o = c == x ? 1.f : 0.f;
        if (c < x) {
          const float uu = rnd ? rnd[rows + (long long)r * x + c] : u[j];
          o = e * va[j] + (1.f - e) * (va[j] + sd * uu);
        }
        v[j] = o;
      }
      store_bf16x8(out + (long long)r * ld + c0, v, lo_off);
    }
  }
}

// WGAN-GP without materialised x_hat rows.  D's first layer is linear, so for x_hat = eps x + (1 - eps) G(z)
// (src/w_gp_gan.py:197-201) the hidden pre-activation is  a_hat = eps a(x) + (1 - eps) a(G(z))  - the interpolated rows and
// their share of the D-layer GEMM are never formed.  From the stored pre-activations of the real and fake rows (bf16, or
// hi + lo planes in split mode) one warp per row writes what the penalty needs (SURVEY A.2): U = w2 * relu'(a_hat) (the first
// gradient's operand, bf16 [+ residual plane]) and the logit part s = sum_n w2[n] relu(a_hat[n]) into slot 0 of the row's
// logit slots (the other slots are zeroed; b2 is added by the reader).  eps: rnd[r], or curand_uniform from Philox
// subsequence r of seed ^ 0x9E3779B97F4A7C15 at offset stream_id * 256.
constexpr int kGpHatGroups = 2;    // 16-byte column groups per lane: ld <= 512 columns
__global__ void gp_hat_kernel(const __nv_bfloat16* __restrict__ pre_r, const __nv_bfloat16* __restrict__ pre_f, const float* __restrict__ w2,
                              __nv_bfloat16* __restrict__ U, float* __restrict__ slots, int nslots, int slot_ld, int rows, int h, int ld,
                              const float* __restrict__ rnd, unsigned long long seed, unsigned long long stream_id, long long lo_off,
                              const unsigned long long* __restrict__ step_ptr) {
  griddep_sync();
  if (step_ptr) stream_id += 2ull * (*step_ptr);
  const int groups = ld / 8;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  // this lane's columns (the same for every row): w2 stays in registers
  float wv[kGpHatGroups][8];
#pragma unroll
  for (int k = 0; k < kGpHatGroups; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = (lane + 32 * k) * 8 + j;
      wv[k][j] = (lane + 32 * k < groups && c < h) ? w2[c] : 0.f;
    }
  // two rows per pass, raw 16-byte loads first (predicated, no branches between them): 8 (16 in split mode) loads in
  // flight per lane - the kernel is HBM-bound
  const uint4 z4 = make_uint4(0, 0, 0, 0);
  for (int r0 = w; r0 < rows; r0 += 2 * nwarps) {
    uint4 ra[2][kGpHatGroups], rb[2][kGpHatGroups], la[2][kGpHatGroups], lb[2][kGpHatGroups];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int r = r0 + t * nwarps;
#pragma unroll
      for (int k = 0; k < kGpHatGroups; ++k) {
        const int g = lane + 32 * k;
        const bool ok = r < rows && g < groups;
        const long long off = (long long)(ok ? r : 0) * ld + (ok ? g : 0) * 8;
        ra[t][k] = z4; rb[t][k] = z4; la[t][k] = z4; lb[t][k] = z4;
        if (ok) ra[t][k] = __ldg(reinterpret_cast<const uint4*>(pre_r + off));
        if (ok) rb[t][k] = __ldg(reinterpret_cast<const uint4*>(pre_f + off));
        if (ok && lo_off) la[t][k] = __ldg(reinterpret_cast<const uint4*>(pre_r + lo_off + off));
        if (ok && lo_off) lb[t][k] = __ldg(reinterpret_cast<const uint4*>(pre_f + lo_off + off));
      }
    }
    float e[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int r = r0 + t * nwarps;
      e[t] = 0.f;
      if (r < rows) {
        if (rnd) e[t] = rnd[r];
        else {
          curandStatePhilox4_32_10_t st;
          curand_init(seed ^ 0x9E3779B97F4A7C15ull, (unsigned long long)r, stream_id * 256ull, &st);
          e[t] = curand_uniform(&st);   // (0,1]; the reference's rand is [0,1)
        }
      }
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int r = r0 + t * nwarps;
      if (r >= rows) break;
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < kGpHatGroups; ++k) {
        const int g = lane + 32 * k;
        if (g >= groups) continue;
        const uint32_t a4[4] = {ra[t][k].x, ra[t][k].y, ra[t][k].z, ra[t][k].w}, b4[4] = {rb[t][k].x, rb[t][k].y, rb[t][k].z, rb[t][k].w};
        const uint32_t c4[4] = {la[t][k].x, la[t][k].y, la[t][k].z, la[t][k].w}, d4[4] = {lb[t][k].x, lb[t][k].y, lb[t][k].z, lb[t][k].w};
        float u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float pa = ((j & 1) ? bf16_hi(a4[j >> 1]) : bf16_lo(a4[j >> 1])) + ((j & 1) ? bf16_hi(c4[j >> 1]) : bf16_lo(c4[j >> 1]));
          const float pb = ((j & 1) ? bf16_hi(b4[j >> 1]) : bf16_lo(b4[j >> 1])) + ((j & 1) ? bf16_hi(d4[j >> 1]) : bf16_lo(d4[j >> 1]));
          const float ah = e[t] * pa + (1.f - e[t]) * pb;
          u[j] = ah > 0.f ? wv[k][j] : 0.f;
          dot = fmaf(fmaxf(ah, 0.f), wv[k][j], dot);
        }
        store_bf16x8(U + (long long)r * ld + g * 8, u, lo_off);
      }
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      if (lane < nslots) slots[(long long)lane * slot_ld + r] = lane == 0 ? dot : 0.f;
    }
  }
}

// sum and sum of squares of the first x columns of `rows` bf16 rows -> per-block partials [nblk][2]
__global__ void moments_kernel(const __nv_bfloat16* __restrict__ a, int rows, int x, int ld, double* __restrict__ part) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  const int groups = ld / 8;
  double s1 = 0, s2 = 0;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < (long long)rows * groups; i += gridDim.x * 256ll) {
    const int g = int(i % groups);
    const uint4 v = reinterpret_cast<const uint4*>(a)[i];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float lo = bf16_lo(u[q]), hi = bf16_hi(u[q]);
      if (g * 8 + 2 * q < x) { s1 += lo; s2 += (double)lo * lo; }
      if (g * 8 + 2 * q + 1 < x) { s1 += hi; s2 += (double)hi * hi; }
    }
  }
  s1 = block_sum<256>(s1, sh);
  s2 = block_sum<256>(s2, sh);
  if (threadIdx.x == 0) { part[blockIdx.x * 2] = s1; part[blockIdx.x * 2 + 1] = s2; }
}
__global__ void moments_final_kernel(const double* __restrict__ part, int nblk, float count, float* __restrict__ stats) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double s1 = 0, s2 = 0;
  for (int i = threadIdx.x; i < nblk; i += 256) { s1 += part[2 * i]; s2 += part[2 * i + 1]; }
  s1 = block_sum<256>(s1, sh);
  s2 = block_sum<256>(s2, sh);
  if (threadIdx.x == 0) { stats[0] = float(s1); stats[1] = float(s2); stats[2] = count; }   // count: elements behind the sums
}

// Per xhat row: nv = ||V|| from the sum-of-squares slots of the V GEMM, q = 1[s>0] (ReLU D)
// or p(1-p) (sigmoid D), n = q*nv, r = 2*lam*inv_b*(n-K); writes coef = r*q/nv (0 at nv=0:
// torch's norm subgradient), ds_gp = r*nv*dq/ds, and block partials (sum (n-K)^2, sum ds_gp).
struct GpParams {
  const float* slots_s; int nslots_s; int slot_ld;   // logit slots of the xhat rows (+ b2)
  const float* slots_v; int nslots_v; int slotv_ld;  // sum-of-squares slots of V
  const float* b2;
  int rows, out_act;
  float lam, K, inv_b;
  float* coef; float* ds_gp;
  double* part; int nblk;
  float* loss;   // [0] += lam * sum (n-K)^2 / rows ;  [3] = sum ds_gp
};
__global__ void __launch_bounds__(kLossThreads) gp_rows_kernel(const GpParams p) {
  griddep_sync();
  __shared__ double sh[kLossThreads / 32];
  double a0 = 0, a1 = 0;
  for (int r = blockIdx.x * kLossThreads + threadIdx.x; r < p.rows; r += gridDim.x * kLossThreads) {
    float s = p.b2[0], sq = 0.f;
    for (int k = 0; k < p.nslots_s; ++k) s += p.slots_s[(long long)k * p.slot_ld + r];
    for (int k = 0; k < p.nslots_v; ++k) sq += p.slots_v[(long long)k * p.slotv_ld + r];
    const float nv = sqrtf(sq);
    float q, dq;
    if (p.out_act == OUT_RELU) { q = s > 0.f ? 1.f : 0.f; dq = 0.f; }
    else { const float pr = 1.f / (1.f + expf(-s)); q = pr * (1.f - pr); dq = q * (1.f - 2.f * pr); }
    const float n = q * nv;
    const float rr = 2.f * p.lam * p.inv_b * (n - p.K);
    p.coef[r] = nv > 0.f ? rr * q / nv : 0.f;
    const float dsg = rr * nv * dq;
    p.ds_gp[r] = dsg;
    a0 += (double)(n - p.K) * (n - p.K);
    a1 += dsg;
  }
  a0 = block_sum<kLossThreads>(a0, sh);
  a1 = block_sum<kLossThreads>(a1, sh);
  if (threadIdx.x == 0) { p.part[blockIdx.x * 4] = a0; p.part[blockIdx.x * 4 + 1] = a1; }
}
__global__ void __launch_bounds__(kLossThreads) gp_final_kernel(const GpParams p) {
  griddep_sync();
  __shared__ double sh[kLossThreads / 32];
  const double s0 = reduce_partials4(p.part, p.nblk, 0, sh);
  const double s1 = reduce_partials4(p.part, p.nblk, 1, sh);
  if (threadIdx.x == 0) {
    p.loss[0] += float(p.lam * s0 / p.rows);   // after loss_final wrote the base loss
    p.loss[3] = float(s1);
  }
}

// rows[r, :] *= coef[r]  (bf16, in place)
__global__ void scale_rows_kernel(__nv_bfloat16* __restrict__ a, const float* __restrict__ coef, int rows, int ld, long long lo_off) {
  griddep_sync();
  const int groups = ld / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)rows * groups;
       i += (long long)gridDim.x * blockDim.x) {
    const float c = coef[i / groups];
    float v[8];
    load_bf16x8(a + i * 8, v, lo_off);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= c;
    store_bf16x8(a + i * 8, v, lo_off);
  }
}

// ---------------------------------------------------------------- VAE (src/vae.py:94-106,193-212)
// mulv fp32 [rows, ldm]: columns [0,z) = mu, [z,2z) = log_var.  z = mu + eps*exp(lv/2)
// -> bf16 [rows, ldz] with a ones column at z; eps (caller tensor or Philox) is kept in
// eps_out for the backward; per-block partial of kl = sum 0.5(mu^2 + e^lv - lv - 1).
__global__ void vae_reparam_kernel(const float* __restrict__ mulv, int ldm, const float* __restrict__ eps_in,
                                   float* __restrict__ eps_out, __nv_bfloat16* __restrict__ zb, int ldz, int rows,
                                   int z, unsigned long long seed, unsigned long long stream_id,
                                   double* __restrict__ part, long long lo_off) {
  griddep_sync();
  // One thread per (row, 8-column group of the latent row): 32-byte reads of mu / log_var / eps, one 16-byte store of z
  // (a thread-per-row mapping would read 256-byte-strided rows).  Philox subsequence = cell.
  __shared__ double sh[256 / 32];
  const int groups = ldz / 8, gz = (z + 8) / 8;
  const long long t = blockIdx.x * 256ll + threadIdx.x;
  double kl = 0.0;
  if (t < (long long)rows * gz) {
    const int r = int(t / gz), g = int(t % gz), c0 = g * 8;
    float v[8], e[8];
    if (eps_in == nullptr && c0 < z) {
      curandStatePhilox4_32_10_t st;
      curand_init(seed ^ 0x5851F42D4C957F2Dull, (unsigned long long)r * groups + g, stream_id * 64ull, &st);
      const float4 a = curand_normal4(&st), b = curand_normal4(&st);
      e[0] = a.x; e[1] = a.y; e[2] = a.z; e[3] = a.w; e[4] = b.x; e[5] = b.y; e[6] = b.z; e[7] = b.w;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      float o = (c == z) ? 1.f : 0.f;
      if (c < z) {
        const float mu = mulv[(long long)r * ldm + c], lv = mulv[(long long)r * ldm + z + c];
        const float ee = eps_in ? eps_in[(long long)r * z + c] : e[j];
        eps_out[(long long)r * z + c] = ee;
        o = mu + ee * expf(0.5f * lv);
        kl += 0.5 * ((double)mu * mu + exp((double)lv) - lv - 1.0);
      }
      v[j] = o;
    }
    store_bf16x8(zb + (long long)r * ldz + c0, v, lo_off);
    for (int pg = gz + g; pg < groups; pg += gz) {      // this thread's share of the row's zero padding
      reinterpret_cast<uint4*>(zb)[(long long)r * groups + pg] = make_uint4(0, 0, 0, 0);
      if (lo_off) reinterpret_cast<uint4*>(zb + lo_off)[(long long)r * groups + pg] = make_uint4(0, 0, 0, 0);
    }
  }
  kl = block_sum<256>(kl, sh);
  if (threadIdx.x == 0 && part) part[blockIdx.x] = kl;
}

// dmu = mu + dz ; dlv = 0.5(e^lv - 1) + dz * eps * e^{lv/2} * 0.5  -> bf16 [rows, ld]: [dmu | dlv | 0]
// One thread per (row, 8 output columns): a group never straddles the mu / log_var boundary when z % 8 == 0;
// otherwise the per-element branch below handles it.
__global__ void vae_dlatent_kernel(const float* __restrict__ mulv, int ldm, const float* __restrict__ dz, int lddz,
                                   const float* __restrict__ eps, __nv_bfloat16* __restrict__ out, int ld, int rows,
                                   int z, float scale, long long lo_off) {
  griddep_sync();
  const int groups = ld / 8;
  const long long t = blockIdx.x * 256ll + threadIdx.x;
  if (t >= (long long)rows * groups) return;
  const int r = int(t / groups), c0 = int(t % groups) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    float o = 0.f;
    if (c < z) {
      o = scale * (mulv[(long long)r * ldm + c] + dz[(long long)r * lddz + c]);
    } else if (c < 2 * z) {
      const int k = c - z;
      const float lv = mulv[(long long)r * ldm + z + k];
      o = scale * (0.5f * (expf(lv) - 1.f) + dz[(long long)r * lddz + k] * eps[(long long)r * z + k] * expf(0.5f * lv) * 0.5f);
    }
    v[j] = o;
  }
  store_bf16x8(out + (long long)r * ld + c0, v, lo_off);
}

// recon = sum over rows of the per-row slots (sum (x-out)^2); losses[0] = recon, [1] = kl
__global__ void vae_rowsum_kernel(const float* __restrict__ slots, int nslots, int slot_ld, int rows,
                                  double* __restrict__ part) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double t = 0.0;
  for (int r = blockIdx.x * 256 + threadIdx.x; r < rows; r += gridDim.x * 256)
    for (int k = 0; k < nslots; ++k) t += slots[(long long)k * slot_ld + r];
  t = block_sum<256>(t, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}
__global__ void vae_losses_final_kernel(const double* __restrict__ part_r, int nr, const double* __restrict__ part_k,
                                        int nk, float* __restrict__ losses) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double a = 0, b = 0;
  for (int i = threadIdx.x; i < nr; i += 256) a += part_r[i];
  for (int i = threadIdx.x; i < nk; i += 256) b += part_k[i];
  a = block_sum<256>(a, sh);
  b = block_sum<256>(b, sh);
  if (threadIdx.x == 0) { losses[0] = float(a); losses[1] = float(b); }
}

// ---------------------------------------------------------------- InfoGAN Q head (src/info_gan.py:290-302)
// inf fp32 [rows, ldi]: [0,nd) categorical logits, [nd, nd+nc) continuous code.  noise fp32
// [rows, ldn]: columns [zd, zd+nd) one-hot target, [zd+nd, zd+nd+nc) continuous target.
// loss = mean_r CE(logits_r, argmax onehot_r) + mean_{r,c} (cont - target)^2; writes
// d loss / d inf (x inv_b-style scaling for data parallel) as bf16 [rows, ldo] (zero padded).
__global__ void __launch_bounds__(kLossThreads) info_loss_kernel(const float* __restrict__ inf, int ldi,
                                                                  const float* __restrict__ noise, int ldn, int zd, int nd,
                                                                  int nc, int rows, float inv_b,
                                                                  __nv_bfloat16* __restrict__ dinf, int ldo,
                                                                  double* __restrict__ part, long long lo_off) {
  griddep_sync();
  __shared__ double sh[kLossThreads / 32];
  double ce = 0, mse = 0;
  for (int r = blockIdx.x * kLossThreads + threadIdx.x; r < rows; r += gridDim.x * kLossThreads) {
    const float* v = inf + (long long)r * ldi;
    const float* t = noise + (long long)r * ldn;
    int tgt = 0;
    float best = t[zd];
    for (int c = 1; c < nd; ++c) if (t[zd + c] > best) { best = t[zd + c]; tgt = c; }   // torch.max: first maximum
    float m = v[0];
    for (int c = 1; c < nd; ++c) m = fmaxf(m, v[c]);
    float se = 0.f;
    for (int c = 0; c < nd; ++c) se += expf(v[c] - m);
    const float lse = m + logf(se);
    ce += lse - v[tgt];
    __nv_bfloat16* o = dinf + (long long)r * ldo;
    auto put = [&](int c, float val) {
      const __nv_bfloat16 hi = __float2bfloat16_rn(val);
      o[c] = hi;
      if (lo_off) o[c + lo_off] = __float2bfloat16_rn(val - __bfloat162float(hi));
    };
    for (int c = 0; c < nd; ++c) put(c, (expf(v[c] - lse) - (c == tgt ? 1.f : 0.f)) * inv_b);
    for (int c = 0; c < nc; ++c) {
      const float d = v[nd + c] - t[zd + nd + c];
      mse += (double)d * d;
      put(nd + c, 2.f * d * inv_b / nc);
    }
    for (int c = nd + nc; c < ldo; ++c) put(c, 0.f);
  }
  ce = block_sum<kLossThreads>(ce, sh);
  mse = block_sum<kLossThreads>(mse, sh);
  if (threadIdx.x == 0) { part[blockIdx.x * 4] = ce; part[blockIdx.x * 4 + 1] = mse; }
}
__global__ void __launch_bounds__(kLossThreads) info_loss_final_kernel(const double* __restrict__ part, int nblk, int rows,
                                                                        int nc, float* __restrict__ loss) {
  griddep_sync();
  __shared__ double sh[kLossThreads / 32];
  const double ce = reduce_partials4(part, nblk, 0, sh), mse = reduce_partials4(part, nblk, 1, sh);
  if (threadIdx.x == 0) loss[0] = float(ce / rows + mse / ((double)rows * nc));
}

// ---------------------------------------------------------------- BEGAN (src/be_gan.py)
// device state: [0] K  [1] scale of real rows (= inv_b)  [2] scale of fake rows (= -K inv_b)
// [3] DX  [4] DG  [5] plateau best  [6] plateau bad count  [7] lr scale  [8],[9] inv_b (G step)
// D step: DX = mean_i sum_k |D(x)-x|, DG likewise on fakes, loss = DX - K DG (src/be_gan.py:225-236);
// G step: loss = DG (src/be_gan.py:256).  part_x / part_g: per-block partial row sums.
__global__ void began_loss_final_kernel(const double* __restrict__ part_x, const double* __restrict__ part_g, int nblk,
                                        int B, int g_step, float* __restrict__ state, float* __restrict__ loss) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double a = 0, b = 0;
  for (int i = threadIdx.x; i < nblk; i += 256) { if (!g_step) a += part_x[i]; b += part_g[i]; }
  a = block_sum<256>(a, sh);
  b = block_sum<256>(b, sh);
  if (threadIdx.x == 0) {
    const float DX = float(a / B), DG = float(b / B);
    if (g_step) loss[0] = DG;
    else { loss[0] = DX - state[0] * DG; state[3] = DX; state[4] = DG; }
  }
}
// proportional control of K (src/be_gan.py:189-191) and the two identical ReduceLROnPlateau
// schedulers (factor 0.5, rel threshold 0.01, patience given; src/be_gan.py:133-136,194-195)
__global__ void began_control_kernel(float* __restrict__ state, float gamma, float lambda, float patience) {
  griddep_sync();
  const float DX = state[3], DG = state[4];
  const float K = fminf(fmaxf(state[0] + lambda * (gamma * DX - DG), 0.f), 1.f);
  const float conv = DX + fabsf(gamma * DX - DG);
  state[0] = K;
  state[2] = -K * state[1];
  if (conv < state[5] * (1.f - 0.01f)) { state[5] = conv; state[6] = 0.f; }
  else state[6] += 1.f;
  if (state[6] > patience) { state[7] *= 0.5f; state[6] = 0.f; }
  state[10] = conv;
}
// DA2 = (T - DRg) * fake (1 - fake): dL/d(pre-sigmoid) of G for BEGAN's G loss, whose gradient
// reaches G(z) through D (T) and directly (-DRg)   (src/be_gan.py:256)
__global__ void began_da2_kernel(const __nv_bfloat16* __restrict__ T, const __nv_bfloat16* __restrict__ DRg,
                                 const __nv_bfloat16* __restrict__ fake, __nv_bfloat16* __restrict__ out, int rows, int x,
                                 int ld, long long lo_off) {
  griddep_sync();
  const int groups = ld / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)rows * groups;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = int(i % groups) * 8;
    float t[8], d[8], f[8], o[8];
    load_bf16x8(T + i * 8, t, lo_off);
    load_bf16x8(DRg + i * 8, d, lo_off);
    load_bf16x8(fake + i * 8, f, lo_off);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (c0 + j < x) ? (t[j] - d[j]) * f[j] * (1.f - f[j]) : 0.f;
    store_bf16x8(out + i * 8, o, lo_off);
  }
}

// ---------------------------------------------------------------- gradient finalisation
// flat_grad[dst_off + i] = sum over `nsplit` partial copies of src[map(i)]:
//   kind 0 (matrix, rows x cols):  src[r*ld + c]        (partial stored as [rows][ld])
//   kind 1 (matrix, transposed) :  src[r*ld + c] with i = r*cols + c, same formula —
//          the GEMM epilogue already wrote the torch layout; kept for clarity
//   kind 2 (bias from the ones-column trick): src[i*ld + col]
//   kind 3 (plain vector): src[i]
struct GradSeg {
  int dst_off, n, kind, cols, ld, col, nsplit;
  long long split_stride;
  const float* src;
};
struct GradSegs { GradSeg s[8]; int nseg; int total; };

// element i of the flat gradient: sum of its split-K partials (fixed order -> deterministic)
__device__ __forceinline__ float gather_grad(const GradSegs& segs, int i) {
#pragma unroll 1
  for (int k = 0; k < segs.nseg; ++k) {
    const GradSeg& s = segs.s[k];
    const int j = i - s.dst_off;
    if (j < 0 || j >= s.n) continue;
    long long off;
    if (s.kind <= 1) off = (long long)(j / s.cols) * s.ld + (j % s.cols);
    else if (s.kind == 2) off = (long long)j * s.ld + s.col;
    else off = j;
    // four independent partial sums, combined in a fixed order -> deterministic; the partials are fetched eight at a
    // time (all loads issued before the first add: the kernel is a chain of dependent memory round trips otherwise)
    float t0 = 0.f, t1 = 0.f, t2 = 0.f, t3 = 0.f;
    const float* src = s.src + off;
    int q = 0;
    for (; q + 8 <= s.nsplit; q += 8) {
      float a[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = src[(long long)(q + u) * s.split_stride];
      t0 += a[0]; t1 += a[1]; t2 += a[2]; t3 += a[3];
      t0 += a[4]; t1 += a[5]; t2 += a[6]; t3 += a[7];
    }
    {                                   // tail of up to 7 partials: predicated loads, same accumulator pattern
      float a[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = (q + u < s.nsplit) ? src[(long long)(q + u) * s.split_stride] : 0.f;
      t0 += a[0]; t1 += a[1]; t2 += a[2]; t3 += a[3];
      t0 += a[4]; t1 += a[5]; t2 += a[6]; t3 += a[7];
    }
    return (t0 + t1) + (t2 + t3);
  }
  return 0.f;
}

__global__ void finalize_grads_kernel(const GradSegs segs, float* __restrict__ flat) {
  griddep_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= segs.total) return;
  flat[i] = gather_grad(segs, i);
}

// ---------------------------------------------------------------- fused Adam + operand shadows
// torch.optim.Adam semantics (src/ns_gan.py:107-110; coupled weight decay for
// src/vae.py:139-142; optional clamp = WGAN clipping src/w_gan.py:158).  After the
// update each weight matrix element is also written as bf16 into the GEMM operand
// copies: `shadow` [rows, ld_s] (K-major, zero-padded) and `shadow_t` [cols, ld_t].
struct AdamSeg {
  int off, n, cols;              // flat range, matrix column count (0 for vectors)
  __nv_bfloat16* shadow; int ld_s;
  __nv_bfloat16* shadow_t; int ld_t;
};
struct AdamParams {
  float* p; const float* g; float* m; float* v;
  int total;
  float lr, b1, b2, eps, wd, bc1, bc2_sqrt, clamp;   // clamp <= 0: off
  int update;                                        // 0: only refresh shadows
  const float* lr_scale;                             // nullable device scalar multiplying lr (BEGAN's plateau scheduler)
  AdamSeg seg[6]; int nseg;
  long long lo_off;                                  // split mode: operand copies also get their residual plane
  const unsigned long long* step_ptr;                // device-step mode: bias corrections from the device step counter (+1)
  // lazy gradients (gm_gan_set_lazy_grads): the flat gradient has not been formed yet; the
  // update gathers each element from the split-K partials itself and stores it to gout
  int gather; float* gout; GradSegs gsegs;
};

// one element of the update: p, m, v and the bf16 operand copies
__device__ __forceinline__ void adam_element(const AdamParams& a, int i, float g) {
  float p = a.p[i];
  if (a.update) {
    float bc1 = a.bc1, bc2_sqrt = a.bc2_sqrt;
    if (a.step_ptr) {   // the host's formulas (fill_adam) on the device counter
      const double t = double(*a.step_ptr + 1ull);
      bc1 = float(1.0 - pow(double(a.b1), t));
      bc2_sqrt = float(sqrt(1.0 - pow(double(a.b2), t)));
    }
    if (a.wd != 0.f) g = fmaf(a.wd, p, g);
    const float m = a.b1 * a.m[i] + (1.f - a.b1) * g;
    const float v = a.b2 * a.v[i] + (1.f - a.b2) * g * g;
    a.m[i] = m;
    a.v[i] = v;
    const float denom = sqrtf(v) / bc2_sqrt + a.eps;
    const float lr = a.lr_scale ? a.lr * a.lr_scale[0] : a.lr;
    p = p - (lr / bc1) * (m / denom);
    if (a.clamp > 0.f) p = fminf(fmaxf(p, -a.clamp), a.clamp);
    a.p[i] = p;
  }
#pragma unroll 1
  for (int k = 0; k < a.nseg; ++k) {
    const AdamSeg& s = a.seg[k];
    const int j = i - s.off;
    if (j < 0 || j >= s.n) continue;
    if (s.cols > 0) {
      const int r = j / s.cols, c = j % s.cols;
      const __nv_bfloat16 b = __float2bfloat16_rn(p);
      if (s.shadow) s.shadow[(long long)r * s.ld_s + c] = b;
      if (s.shadow_t) s.shadow_t[(long long)c * s.ld_t + r] = b;
      if (a.lo_off) {
        const __nv_bfloat16 bl = __float2bfloat16_rn(p - __bfloat162float(b));
        if (s.shadow) s.shadow[(long long)r * s.ld_s + c + a.lo_off] = bl;
        if (s.shadow_t) s.shadow_t[(long long)c * s.ld_t + r + a.lo_off] = bl;
      }
    }
    return;
  }
}

// device-step mode: counter += 1 after the kernels that read it (stream order)
__global__ void bump_step_kernel(unsigned long long* __restrict__ ctr) {
  griddep_sync();
  if (threadIdx.x == 0 && blockIdx.x == 0) *ctr += 1ull;
}

__global__ void adam_kernel(const AdamParams a) {
  griddep_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.total) return;
  float g = 0.f;
  if (a.update) {
    if (a.gather) { g = gather_grad(a.gsegs, i); a.gout[i] = g; }
    else g = a.g[i];
  }
  adam_element(a, i, g);
}

// ---------------------------------------------------------------- gradient all-reduce fused into Adam
// Data-parallel optimizer step in ONE kernel per rank (SURVEY.md 8e: the only exchange of the
// path is the SUM of the flat D / G gradient): block b
//   1. forms its 1024-element chunk of the local gradient (split-K gather or the flat buffer)
//      and stores it in this rank's exchange buffer (peer-mapped device memory, CUDA IPC);
//   2. publishes "chunk b of step seq is in place" into every peer's flag array (release.sys
//      stores through NVLink peer mappings);
//   3. waits until every peer's chunk b has arrived (local polling, acquire.sys);
//   4. reads chunk b of every rank through the peer mappings, sums in rank order (bitwise the
//      same on every rank) and applies Adam + the bf16 operand refresh.
// No grid-wide or cross-rank barrier: a block only ever waits for the same-numbered block of its
// peers, whose steps 1-2 never block.  Exchange buffers are double-buffered by seq parity.
constexpr int kCommMaxWorld = 16;
constexpr int kCommChunk = 1024;
constexpr int kCommStatVals = 4;
struct CommDev {
  float* x[kCommMaxWorld];                    // exchange regions [2][kCommMaxWorld][nfloats] of every rank (own = local pointer)
  unsigned long long* f[kCommMaxWorld];       // flag arrays [2][kCommMaxWorld][nblocks] of every rank
  int rank, world, nblocks;
  long long nfloats;
  unsigned long long seq;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_relaxed_sys(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

// Batch statistics over the GLOBAL batch (SURVEY.md 8e caveats: RaNS mean(DG) and sum q(1-q)/(q+eps),
// Fisher moments, DRAGAN images.std(), BEGAN DX / DG): one block reduces the per-block partial sums
// part[blk*stride + v] (v < nvals <= 4), pushes them into every peer's statistics area, waits for the
// peers' values, and replaces the partials by the rank-ordered global sums (entry 0 = sum, rest 0), so
// the passes that re-reduce `part` afterwards see global statistics without knowing about ranks.
struct CommStats {
  double* v[kCommMaxWorld];                   // [2][kCommMaxWorld][kCommStatVals] per rank
  unsigned long long* f[kCommMaxWorld];       // [2][kCommMaxWorld] per rank
  int rank, world;
  unsigned long long seq;
};
__global__ void __launch_bounds__(256) stats_exchange_kernel(double* __restrict__ part, int nblk, int stride, int nvals,
                                                             const CommStats cs) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  __shared__ double tot[kCommStatVals];
  const int tid = threadIdx.x, par = int(cs.seq & 1ull);
  for (int v = 0; v < nvals; ++v) {
    double t = 0.0;
    for (int i = tid; i < nblk; i += 256) t += part[(long long)i * stride + v];
    t = block_sum<256>(t, sh);
    if (tid == 0) tot[v] = t;
  }
  __syncthreads();
  if (tid < cs.world && tid != cs.rank) {
    double* dst = cs.v[tid] + ((long long)par * kCommMaxWorld + cs.rank) * kCommStatVals;
    for (int v = 0; v < nvals; ++v) asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(dst + v), "d"(tot[v]) : "memory");
    st_release_sys(cs.f[tid] + par * kCommMaxWorld + cs.rank, cs.seq);
  }
  if (tid < cs.world && tid != cs.rank) {
    const unsigned long long* flag = cs.f[cs.rank] + par * kCommMaxWorld + tid;
    const long long t0 = clock64();
    while (ld_acquire_sys(flag) < cs.seq) {
      if (clock64() - t0 > 40000000000ll) __trap();
    }
  }
  __syncthreads();
  if (tid < nvals) {
    double g = 0.0;
    for (int r = 0; r < cs.world; ++r) {
      if (r == cs.rank) { g += tot[tid]; continue; }
      const double* src = cs.v[cs.rank] + ((long long)par * kCommMaxWorld + r) * kCommStatVals + tid;
      double x;
      asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(x) : "l"(src) : "memory");
      g += x;
    }
    tot[tid] = g;
  }
  __syncthreads();
  for (int i = tid; i < nblk; i += 256)
    for (int v = 0; v < nvals; ++v) part[(long long)i * stride + v] = (i == 0) ? tot[v] : 0.0;
}

// PUSH protocol, 128-bit accesses: every thread owns 4 consecutive gradient elements (one float4).  It forms them
// (split-K gather or the flat buffer), keeps them in registers and WRITES them into slot [parity][own rank] of every
// peer's exchange region (posted NVLink stores, no round trip); after a system fence the block raises "chunk b of
// step seq" in every peer's flag array; it then waits for its peers' flags on LOCAL memory and reads their chunks from
// its OWN region (local HBM / L2, not over the link), sums in rank order - bitwise identical on every rank - and
// applies Adam.  Exchange region of a rank: [2 parities][kCommMaxWorld source ranks][nfloats].
__device__ __forceinline__ void st_relaxed_sys_v4(float* p, float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_relaxed_sys_v4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__global__ void __launch_bounds__(256) adam_allreduce_kernel(const AdamParams a, const CommDev cm) {
  griddep_sync();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int par = int(cm.seq & 1ull);
  const int i0 = b * kCommChunk + tid * 4;            // this thread's 4 elements (nfloats is a multiple of the chunk)
  float g[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = i0 + j;
    g[j] = i < a.total ? (a.gather ? gather_grad(a.gsegs, i) : a.g[i]) : 0.f;
  }
  const long long slot = ((long long)par * kCommMaxWorld + cm.rank) * cm.nfloats + i0;
  const float4 mine = make_float4(g[0], g[1], g[2], g[3]);
  for (int r = 0; r < cm.world; ++r)
    if (r != cm.rank) st_relaxed_sys_v4(cm.x[r] + slot, mine);
  __threadfence_system();
  __syncthreads();
  if (tid < cm.world && tid != cm.rank) {
    st_release_sys(cm.f[tid] + ((long long)par * kCommMaxWorld + cm.rank) * cm.nblocks + b, cm.seq);
    const unsigned long long* flag = cm.f[cm.rank] + ((long long)par * kCommMaxWorld + tid) * cm.nblocks + b;
    const long long t0 = clock64();
    while (ld_acquire_sys(flag) < cm.seq) {
      if (clock64() - t0 > 40000000000ll) __trap();   // ~20 s: a peer died
    }
  }
  __syncthreads();
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < cm.world; ++r) {
    const float4 v = (r == cm.rank) ? mine
                                    : ld_relaxed_sys_v4(cm.x[cm.rank] + ((long long)par * kCommMaxWorld + r) * cm.nfloats + i0);
    sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
  }
  const float out[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = i0 + j;
    if (i >= a.total) break;
    a.gout[i] = out[j];
    adam_element(a, i, out[j]);
  }
}


// The same exchange in two kernels, so that work which does not depend on the update can run between them (the G step's
// generator forward under the D exchange; the next step's image staging under the G exchange): `push` forms the gradient
// chunk, stores it in its OWN slot and in every peer's, fences and raises the flags - it never waits; `finish` waits for
// the peers' flags, sums all slots of its own region in rank order and applies Adam.
__global__ void __launch_bounds__(256) adam_exchange_push_kernel(const AdamParams a, const CommDev cm) {
  griddep_sync();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int par = int(cm.seq & 1ull);
  const int i0 = b * kCommChunk + tid * 4;
  float g[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = i0 + j;
    g[j] = i < a.total ? (a.gather ? gather_grad(a.gsegs, i) : a.g[i]) : 0.f;
  }
  const long long slot = ((long long)par * kCommMaxWorld + cm.rank) * cm.nfloats + i0;
  const float4 mine = make_float4(g[0], g[1], g[2], g[3]);
  for (int r = 0; r < cm.world; ++r) st_relaxed_sys_v4(cm.x[r] + slot, mine);      // own region included
  __threadfence_system();
  __syncthreads();
  if (tid < cm.world && tid != cm.rank)
    st_release_sys(cm.f[tid] + ((long long)par * kCommMaxWorld + cm.rank) * cm.nblocks + b, cm.seq);
}
__global__ void __launch_bounds__(256) adam_exchange_finish_kernel(const AdamParams a, const CommDev cm) {
  griddep_sync();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int par = int(cm.seq & 1ull);
  const int i0 = b * kCommChunk + tid * 4;
  if (tid < cm.world && tid != cm.rank) {
    const unsigned long long* flag = cm.f[cm.rank] + ((long long)par * kCommMaxWorld + tid) * cm.nblocks + b;
    const long long t0 = clock64();
    while (ld_acquire_sys(flag) < cm.seq) {
      if (clock64() - t0 > 40000000000ll) __trap();   // ~20 s: a peer died
    }
  }
  __syncthreads();
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < cm.world; ++r) {
    const float4 v = ld_relaxed_sys_v4(cm.x[cm.rank] + ((long long)par * kCommMaxWorld + r) * cm.nfloats + i0);
    sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
  }
  const float out[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = i0 + j;
    if (i >= a.total) break;
    a.gout[i] = out[j];
    adam_element(a, i, out[j]);
  }
}

}  // namespace gm
