// Building blocks of the DCGAN conv path (BASELINE configs[4]; the reference only recommends DCGAN, README.md:68,96 —
// there is no reference implementation, see DESIGN.md §6b): NHWC bf16 activations as row-major matrices [B*H*W, C], so
// that every convolution / transposed convolution is one wgmma GEMM (gemm_wgmma.cuh) between an im2col / col2im pass:
//   conv   (k4 s2 p1): col = im2col(x) [B*Ho*Wo, 16*Cin];  y = col W^T        (W [Cout, (kh,kw,ci)])
//   convT  (k4 s2 p1): col = x Wm^T    [B*Hi*Wi, 16*Cout]; y = col2im(col)    (Wm [(kh,kw,co), Cin])
// and their gradients are the same two data movements with the roles swapped.  BatchNorm (training mode, batch
// statistics) and the activations are column-statistics + elementwise kernels over the same matrices.  All HBM-bound:
// 16-byte accesses, grids sized in multiples of the SM count, deterministic two-stage reductions.
#pragma once
#include <curand_kernel.h>
#include "ptx.cuh"

namespace gm {

// ---------------------------------------------------------------- im2col / col2im (kernel 4, stride 2, pad 1)
// Both are pure HBM-bound data movements (the column matrix is 4x the activation it comes from, up to 537 MB at B = 1024),
// so the kernels are written for memory-level parallelism and cheap index arithmetic (the first versions ran at ~40 % of
// the HBM rate: one 16-byte access in flight per thread behind a chain of 64-bit divisions):
// 32-bit indices (the host checks the extents), divisions by the grid extents as shifts when they are powers of two, kUnroll
// independent items per thread with all loads issued before the first store.
struct FastDiv {            // x / d and x % d for 32-bit x; shift >= 0 when d is a power of two
  uint32_t d;
  int shift;
};
__host__ __device__ inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  f.d = d;
  f.shift = -1;
  for (int s = 0; s < 32; ++s)
    if ((1u << s) == d) f.shift = s;
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t x, const FastDiv f) { return f.shift >= 0 ? (x >> f.shift) : (x / f.d); }
__device__ __forceinline__ void fdivmod(uint32_t x, const FastDiv f, uint32_t& q, uint32_t& r) {
  q = fdiv(x, f);
  r = x - q * f.d;
}
constexpr int kConvUnroll = 4;

// x [B, H, W, C] (row pitch ldx elements per pixel) -> col [(b, ho, wo), (kh, kw, c)] with Ho = H/2, Wo = W/2.
// VEC: C % 8 == 0, one item = (output pixel, tap, 8-channel group) = one 16-byte copy (consecutive items are consecutive
// 16-byte chunks of the column matrix: the dominant stream, the writes, is perfectly linear); else one item = (output pixel,
// tap) with a scalar channel loop (the 3-channel image layer).
template <bool VEC>
__global__ void __launch_bounds__(256) im2col_k4s2_kernel(const __nv_bfloat16* __restrict__ x, int H, int W, int C, int ldx,
                                                          __nv_bfloat16* __restrict__ col, int ldc, uint32_t total, FastDiv dcg,
                                                          FastDiv dwo, FastDiv dho) {
  griddep_sync();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x; t0 < total; t0 += stride * kConvUnroll) {
    const __nv_bfloat16* src[kConvUnroll];
    __nv_bfloat16* dst[kConvUnroll];
    bool ok[kConvUnroll], live[kConvUnroll];
#pragma unroll
    for (int u = 0; u < kConvUnroll; ++u) {
      const uint32_t t = t0 + u * stride;
      live[u] = t < total && t >= t0;                 // t >= t0: no wrap-around past 2^32
      uint32_t r, g = 0;
      if (VEC) fdivmod(t, dcg, r, g); else r = t;
      const uint32_t tap = r & 15u;
      r >>= 4;                                        // output pixel index (b, ho, wo)
      uint32_t q, wo, b, ho;
      fdivmod(r, dwo, q, wo);
      fdivmod(q, dho, b, ho);
      const int kh = int(tap >> 2), kw = int(tap & 3u);
      const int iy = 2 * int(ho) - 1 + kh, ix = 2 * int(wo) - 1 + kw;
      ok[u] = live[u] && iy >= 0 && iy < H && ix >= 0 && ix < W;
      dst[u] = col + size_t(r) * ldc + tap * C + g * 8;
      src[u] = x + ((size_t(b) * H + iy) * W + ix) * ldx + g * 8;
    }
    if (VEC) {
      uint4 v[kConvUnroll];
#pragma unroll
      for (int u = 0; u < kConvUnroll; ++u) {
        v[u] = make_uint4(0, 0, 0, 0);
        if (ok[u]) v[u] = __ldg(reinterpret_cast<const uint4*>(src[u]));
      }
#pragma unroll
      for (int u = 0; u < kConvUnroll; ++u)
        if (live[u]) *reinterpret_cast<uint4*>(dst[u]) = v[u];
    } else {
#pragma unroll
      for (int u = 0; u < kConvUnroll; ++u)
        if (live[u])
          for (int c = 0; c < C; ++c) dst[u][c] = ok[u] ? src[u][c] : __float2bfloat16_rn(0.f);
    }
  }
}

// col [(b, iy, ix), (kh, kw, c)] over an Hi x Wi grid -> y [B, 2Hi, 2Wi, C] (gather form: every output pixel sums the
// <= 4 taps that reach it; deterministic, no atomics).  Fused tail, by `mode`:
//   0: y = sum                       1: y = sigmoid(sum)                  (generator output, src/ns_gan.py:45-46)
//   2: y = sum * lrelu'(aux)         3: y = sum * aux (1 - aux)           (gradients through a LeakyReLU / sigmoid output)
// VEC: one item = (output pixel, 8-channel group): four predicated 16-byte loads (+ one of aux) in flight, 2 items per thread.
enum : int { C2I_NONE = 0, C2I_SIGMOID = 1, C2I_LRELU_GRAD = 2, C2I_SIGMOID_GRAD = 3 };
template <bool VEC>
__global__ void __launch_bounds__(256) col2im_k4s2_kernel(const __nv_bfloat16* __restrict__ col, int ldc, int Hi, int Wi, int C,
                                                          __nv_bfloat16* __restrict__ y, int ldy, int mode,
                                                          const __nv_bfloat16* __restrict__ aux, int ld_aux, float slope, uint32_t total,
                                                          FastDiv dcg, FastDiv dwo, FastDiv dho) {
  griddep_sync();
  constexpr int U = 2;
  const uint32_t stride = gridDim.x * blockDim.x;
  if constexpr (VEC) {
    for (uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x; t0 < total; t0 += stride * U) {
      uint4 v[U][4], av[U];
      uint32_t pix[U], g[U];
      bool live[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t t = t0 + u * stride;
        live[u] = t < total && t >= t0;
        fdivmod(t, dcg, pix[u], g[u]);
        uint32_t q, ox, b, oy;
        fdivmod(pix[u], dwo, q, ox);
        fdivmod(q, dho, b, oy);
        // taps with (oy + 1 - kh) even and in range: kh in {(oy + 1) & 1, ((oy + 1) & 1) + 2}
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int kh = int((oy + 1) & 1u) + 2 * a, iy = (int(oy) + 1 - kh) >> 1;
#pragma unroll
          for (int bb = 0; bb < 2; ++bb) {
            const int kw = int((ox + 1) & 1u) + 2 * bb, ix = (int(ox) + 1 - kw) >> 1;
            const bool ok = live[u] && iy >= 0 && iy < Hi && ix >= 0 && ix < Wi;
            uint4 w = make_uint4(0, 0, 0, 0);
            if (ok) w = __ldg(reinterpret_cast<const uint4*>(col + ((size_t(b) * Hi + iy) * Wi + ix) * ldc + (kh * 4 + kw) * C + g[u] * 8));
            v[u][a * 2 + bb] = w;
          }
        }
        av[u] = make_uint4(0, 0, 0, 0);
        if (mode >= C2I_LRELU_GRAD && live[u]) av[u] = __ldg(reinterpret_cast<const uint4*>(aux + size_t(pix[u]) * ld_aux + g[u] * 8));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!live[u]) continue;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {                    // summation order: (kh, kw) ascending
          const uint32_t w[4] = {v[u][k].x, v[u][k].y, v[u][k].z, v[u][k].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) { acc[2 * q] += bf16_lo(w[q]); acc[2 * q + 1] += bf16_hi(w[q]); }
        }
        const uint32_t aw[4] = {av[u].x, av[u].y, av[u].z, av[u].w};
        float o[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          float val = acc[c];
          const float a = (c & 1) ? bf16_hi(aw[c >> 1]) : bf16_lo(aw[c >> 1]);
          if (mode == C2I_SIGMOID) val = 1.f / (1.f + __expf(-val));
          else if (mode == C2I_LRELU_GRAD) val = a > 0.f ? val : slope * val;
          else if (mode == C2I_SIGMOID_GRAD) val = val * a * (1.f - a);
          o[c] = val;
        }
        store_bf16x8(y + size_t(pix[u]) * ldy + g[u] * 8, o, 0);
      }
    }
  } else {
    // C < 8 (the 3-channel image layer): one thread per output pixel, scalar channels
    for (uint32_t pix = blockIdx.x * blockDim.x + threadIdx.x; pix < total; pix += stride) {
      uint32_t q, ox, b, oy;
      fdivmod(pix, dwo, q, ox);
      fdivmod(q, dho, b, oy);
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int kh = int((oy + 1) & 1u) + 2 * a, iy = (int(oy) + 1 - kh) >> 1;
        if (iy < 0 || iy >= Hi) continue;
#pragma unroll
        for (int bb = 0; bb < 2; ++bb) {
          const int kw = int((ox + 1) & 1u) + 2 * bb, ix = (int(ox) + 1 - kw) >> 1;
          if (ix < 0 || ix >= Wi) continue;
          const __nv_bfloat16* src = col + ((size_t(b) * Hi + iy) * Wi + ix) * ldc + (kh * 4 + kw) * C;
#pragma unroll
          for (int c = 0; c < 8; ++c)
            if (c < C) acc[c] += __bfloat162float(src[c]);
        }
      }
      const __nv_bfloat16* ap = aux + size_t(pix) * ld_aux;
      __nv_bfloat16* dst = y + size_t(pix) * ldy;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c < C) {
          float val = acc[c];
          if (mode == C2I_SIGMOID) val = 1.f / (1.f + __expf(-val));
          else if (mode >= C2I_LRELU_GRAD) {
            const float a = __bfloat162float(ap[c]);
            val = mode == C2I_LRELU_GRAD ? (a > 0.f ? val : slope * val) : val * a * (1.f - a);
          }
          dst[c] = __float2bfloat16_rn(val);
        }
      }
    }
  }
}

// ---------------------------------------------------------------- BatchNorm2d, training mode (batch statistics)
// x [rows, C] bf16 (rows = B*H*W).  Pass 1: per-block partial column sums (sum, sum of squares; fp32 per thread over a
// slab of rows, double across the block) -> part [nblk][2][C].  Pass 2 (a warp per channel): mean, invstd (+ running
// statistics, momentum 0.1, unbiased variance like torch).  Pass 3: y = act(gamma * (x - mean) * invstd + beta).
// act: 0 none, 1 ReLU, 2 LeakyReLU(slope).  Thread mapping of every pass: thread = (8-channel group g, row lane rl), the
// block walks rpi = 256 / groups rows per iteration - no division in the loops, per-channel constants in registers, and
// kBnUnroll rows per thread in flight (HBM-bound: the first versions had one 16-byte load in flight per thread and re-read
// gamma / beta / mean / invstd from global memory for every element, 25-45 % of the HBM rate).
constexpr int kBnThreads = 256;
constexpr int kBnUnroll = 4;
constexpr int kBnStatUnroll = 8;
// The double-precision running sums of a thread live in ITS slots of the block's shared array (the same array the final
// cross-row reduction reads), not in registers: 32 fewer registers per thread = more resident warps with loads in flight.
__global__ void __launch_bounds__(kBnThreads) bn_partial_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C, int ld,
                                                                 double* __restrict__ part) {
  griddep_sync();
  extern __shared__ double bn_sh[];                  // [rows_per_iter][2][C]
  const int groups = C / 8;
  const int g = threadIdx.x % groups, rl = threadIdx.x / groups, rpi = kBnThreads / groups;
  if (rl < rpi) {
    double* const my1 = bn_sh + (rl * 2 + 0) * C + g * 8;
    double* const my2 = bn_sh + (rl * 2 + 1) * C + g * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) { my1[j] = 0.0; my2[j] = 0.0; }
    float s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
    int since = 0;
    const long long rstep = (long long)gridDim.x * rpi;
    for (long long r0 = (long long)blockIdx.x * rpi + rl; r0 < rows; r0 += rstep * kBnStatUnroll) {
      uint4 v[kBnStatUnroll];
#pragma unroll
      for (int u = 0; u < kBnStatUnroll; ++u) {
        const long long r = r0 + u * rstep;
        v[u] = make_uint4(0, 0, 0, 0);                // zero rows add nothing to either sum
        if (r < rows) v[u] = __ldg(reinterpret_cast<const uint4*>(x + r * ld) + g);
      }
#pragma unroll
      for (int u = 0; u < kBnStatUnroll; ++u) {
        const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float a = bf16_lo(w[q]), b = bf16_hi(w[q]);
          s1[2 * q] += a; s2[2 * q] = fmaf(a, a, s2[2 * q]);
          s1[2 * q + 1] += b; s2[2 * q + 1] = fmaf(b, b, s2[2 * q + 1]);
        }
      }
      if (++since == 64 / kBnStatUnroll) {   // flush the fp32 running sums into doubles every 64 rows (B*H*W up to 8 M rows)
#pragma unroll
        for (int j = 0; j < 8; ++j) { my1[j] += s1[j]; my2[j] += s2[j]; s1[j] = 0.f; s2[j] = 0.f; }
        since = 0;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { my1[j] += s1[j]; my2[j] += s2[j]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kBnThreads) {
    const int which = c / C, ch = c % C;
    double t = 0.0;
    for (int i = 0; i < rpi; ++i) t += bn_sh[(i * 2 + which) * C + ch];
    part[((long long)blockIdx.x * 2 + which) * C + ch] = t;
  }
}
// stats[0][C] = mean, stats[1][C] = invstd; running[0] mean, running[1] var (nullable).  One WARP per channel: the lanes
// stride over the per-block partials (a thread per channel would walk all ~600 partials serially).
__global__ void bn_finalize_kernel(const double* __restrict__ part, int nblk, int C, double count, float eps,
                                   float* __restrict__ stats, float* __restrict__ running, float momentum) {
  griddep_sync();
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
  for (int i0 = lane; i0 < nblk; i0 += 32 * 8) {          // 16 loads in flight per lane (was a serial chain of ~19 round trips)
    double a1[8], a2[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + 32 * u;
      a1[u] = i < nblk ? part[((long long)i * 2) * C + c] : 0.0;
      a2[u] = i < nblk ? part[((long long)i * 2 + 1) * C + c] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) { s1 += a1[u]; s2 += a2[u]; }
  }
  for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  if (lane != 0) return;
  const double mean = s1 / count;
  const double var = fmax(s2 / count - mean * mean, 0.0);       // biased, as torch normalises with
  stats[c] = float(mean);
  stats[C + c] = float(1.0 / sqrt(var + double(eps)));
  if (running) {
    running[c] = (1.f - momentum) * running[c] + momentum * float(mean);
    running[C + c] = (1.f - momentum) * running[C + c] + momentum * float(var * count / fmax(count - 1.0, 1.0));
  }
}
// y = act(x * sc + sh) with sc = gamma invstd, sh = beta - mean sc (two registers per channel)
__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C, int ld,
                                                               const float* __restrict__ stats, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int act, float slope,
                                                               __nv_bfloat16* __restrict__ y, int ldy) {
  griddep_sync();
  const int groups = C / 8;
  const int g = threadIdx.x % groups, rl = threadIdx.x / groups, rpi = kBnThreads / groups;
  if (rl >= rpi) return;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    sc[j] = gamma[c] * stats[C + c];
    sh[j] = fmaf(-stats[c], sc[j], beta[c]);
  }
  const long long rstep = (long long)gridDim.x * rpi;
  for (long long r0 = (long long)blockIdx.x * rpi + rl; r0 < rows; r0 += rstep * kBnUnroll) {
    uint4 v[kBnUnroll];
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long long r = r0 + u * rstep;
      if (r < rows) v[u] = __ldg(reinterpret_cast<const uint4*>(x + r * ld) + g);
    }
#pragma unroll
    for (int u = 0; u < kBnUnroll; ++u) {
      const long long r = r0 + u * rstep;
      if (r >= rows) break;
      const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xv = (j & 1) ? bf16_hi(w[j >> 1]) : bf16_lo(w[j >> 1]);
        float t = fmaf(xv, sc[j], sh[j]);
        if (act == 1) t = fmaxf(t, 0.f);
        else if (act == 2) t = t > 0.f ? t : slope * t;
        o[j] = t;
      }
      store_bf16x8(y + r * ldy + g * 8, o, 0);
    }
  }
}

// backward: g = dy * act'(gamma xhat + beta); dbeta = sum g; dgamma = sum g xhat;
//           dx = gamma invstd / N * (N g - dbeta - xhat dgamma)            (torch.nn.functional.batch_norm backward)
// Pass 1: partial sums (dbeta, dgamma) with the bn_partial layout; pass 2: finalise into dgb [2][C] fp32; pass 3: dx.
constexpr int kBnBwdUnroll = 4;                       // two operands per row: 8 loads in flight
__global__ void __launch_bounds__(kBnThreads, 2) bn_bwd_partial_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                        long long rows, int C, int ld, const float* __restrict__ stats,
                                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                        int act, float slope, double* __restrict__ part) {
  griddep_sync();
  extern __shared__ double bn_sh[];
  const int groups = C / 8;
  const int g = threadIdx.x % groups, rl = threadIdx.x / groups, rpi = kBnThreads / groups;
  if (rl < rpi) {
    float mu[8], is[8], ga[8], be[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { const int c = g * 8 + j; mu[j] = stats[c]; is[j] = stats[C + c]; ga[j] = gamma[c]; be[j] = beta[c]; }
    double* const my1 = bn_sh + (rl * 2 + 0) * C + g * 8;
    double* const my2 = bn_sh + (rl * 2 + 1) * C + g * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) { my1[j] = 0.0; my2[j] = 0.0; }
    float s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
    int since = 0;
    const long long rstep = (long long)gridDim.x * rpi;
    for (long long r0 = (long long)blockIdx.x * rpi + rl; r0 < rows; r0 += rstep * kBnBwdUnroll) {
      uint4 vx[kBnBwdUnroll], vg[kBnBwdUnroll];
#pragma unroll
      for (int u = 0; u < kBnBwdUnroll; ++u) {
        const long long r = r0 + u * rstep;
        vx[u] = make_uint4(0, 0, 0, 0); vg[u] = make_uint4(0, 0, 0, 0);   // dy = 0 rows add nothing
        if (r < rows) {
          vx[u] = __ldg(reinterpret_cast<const uint4*>(x + r * ld) + g);
          vg[u] = __ldg(reinterpret_cast<const uint4*>(dy + r * ld) + g);
        }
      }
#pragma unroll
      for (int u = 0; u < kBnBwdUnroll; ++u) {
        const uint32_t wx[4] = {vx[u].x, vx[u].y, vx[u].z, vx[u].w}, wg[4] = {vg[u].x, vg[u].y, vg[u].z, vg[u].w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xv = (j & 1) ? bf16_hi(wx[j >> 1]) : bf16_lo(wx[j >> 1]);
          float gg = (j & 1) ? bf16_hi(wg[j >> 1]) : bf16_lo(wg[j >> 1]);
          const float xh = (xv - mu[j]) * is[j];
          const float pre = ga[j] * xh + be[j];
          if (act == 1) gg = pre > 0.f ? gg : 0.f;
          else if (act == 2) gg = pre > 0.f ? gg : slope * gg;
          s1[j] += gg;
          s2[j] = fmaf(gg, xh, s2[j]);
        }
      }
      if (++since == 64 / kBnBwdUnroll) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { my1[j] += s1[j]; my2[j] += s2[j]; s1[j] = 0.f; s2[j] = 0.f; }
        since = 0;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { my1[j] += s1[j]; my2[j] += s2[j]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kBnThreads) {
    const int which = c / C, ch = c % C;
    double t = 0.0;
    for (int i = 0; i < rpi; ++i) t += bn_sh[(i * 2 + which) * C + ch];
    part[((long long)blockIdx.x * 2 + which) * C + ch] = t;
  }
}
// dgb[0][C] = dbeta, dgb[1][C] = dgamma; one warp per output value
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ part, int nblk, int C, float* __restrict__ dgb) {
  griddep_sync();
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= 2 * C) return;
  const int which = c / C, ch = c % C;
  double t = 0.0;
  for (int i0 = lane; i0 < nblk; i0 += 32 * 8) {
    double a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + 32 * u;
      a[u] = i < nblk ? part[((long long)i * 2 + which) * C + ch] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) t += a[u];
  }
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (lane == 0) dgb[c] = float(t);
}
__global__ void __launch_bounds__(kBnThreads, 2) bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                   long long rows, int C, int ld, const float* __restrict__ stats,
                                                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                   int act, float slope, const float* __restrict__ dgb, float inv_count,
                                                                   __nv_bfloat16* __restrict__ dx, int lddx) {
  griddep_sync();
  const int groups = C / 8;
  const int g = threadIdx.x % groups, rl = threadIdx.x / groups, rpi = kBnThreads / groups;
  if (rl >= rpi) return;
  float mu[8], is[8], ga[8], be[8], db[8], dg[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    mu[j] = stats[c]; is[j] = stats[C + c]; ga[j] = gamma[c]; be[j] = beta[c]; db[j] = dgb[c]; dg[j] = dgb[C + c];
  }
  const long long rstep = (long long)gridDim.x * rpi;
  for (long long r0 = (long long)blockIdx.x * rpi + rl; r0 < rows; r0 += rstep * kBnBwdUnroll) {
    uint4 vx[kBnBwdUnroll], vg[kBnBwdUnroll];
#pragma unroll
    for (int u = 0; u < kBnBwdUnroll; ++u) {
      const long long r = r0 + u * rstep;
      if (r < rows) {
        vx[u] = __ldg(reinterpret_cast<const uint4*>(x + r * ld) + g);
        vg[u] = __ldg(reinterpret_cast<const uint4*>(dy + r * ld) + g);
      }
    }
#pragma unroll
    for (int u = 0; u < kBnBwdUnroll; ++u) {
      const long long r = r0 + u * rstep;
      if (r >= rows) break;
      const uint32_t wx[4] = {vx[u].x, vx[u].y, vx[u].z, vx[u].w}, wg[4] = {vg[u].x, vg[u].y, vg[u].z, vg[u].w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xv = (j & 1) ? bf16_hi(wx[j >> 1]) : bf16_lo(wx[j >> 1]);
        float gg = (j & 1) ? bf16_hi(wg[j >> 1]) : bf16_lo(wg[j >> 1]);
        const float xh = (xv - mu[j]) * is[j];
        const float pre = ga[j] * xh + be[j];
        if (act == 1) gg = pre > 0.f ? gg : 0.f;
        else if (act == 2) gg = pre > 0.f ? gg : slope * gg;
        o[j] = ga[j] * is[j] * (gg - inv_count * (db[j] + xh * dg[j]));
      }
      store_bf16x8(dx + r * lddx + g * 8, o, 0);
    }
  }
}

// ---------------------------------------------------------------- small helpers
// fp32 [R, C] -> bf16 copy [R, ld] and (optionally) its transpose [C, ld_t] (GEMM operand forms of a weight matrix)
__global__ void cast_bf16_kernel(const float* __restrict__ src, int R, int C, __nv_bfloat16* __restrict__ dst, int ld,
                                 __nv_bfloat16* __restrict__ dst_t, int ld_t) {
  griddep_sync();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)R * C) return;
  const int r = int(i / C), c = int(i % C);
  const __nv_bfloat16 b = __float2bfloat16_rn(src[i]);
  if (dst) dst[(long long)r * ld + c] = b;
  if (dst_t) dst_t[(long long)c * ld_t + r] = b;
}
// out [rows, ld] bf16: column 0 = v[r], the rest 0 (the upstream gradient of a 1-channel output as a GEMM operand)
__global__ void pack_col0_kernel(const float* __restrict__ v, int rows, __nv_bfloat16* __restrict__ out, int ld) {
  griddep_sync();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ld) return;
  out[i] = __float2bfloat16_rn((i % ld) == 0 ? v[i / ld] : 0.f);
}

// ---------------------------------------------------------------- WGAN-GP on the batch-norm-free conv critic (DESIGN.md §6b)
// The critic is piecewise linear, so the penalty's double backward is closed form: an input-gradient chain at x_hat, a
// per-image norm, a forward-mode (tangent) pass under the same LeakyReLU masks, and one weight-gradient GEMM per layer.
// The kernels below are the parts of that which are not already an im2col / col2im / GEMM.

// per-image eps: the caller's eps_in[b], else Philox U(0,1] with subsequence b of stream (seed, stream_id)
__device__ __forceinline__ float gp_eps(const float* __restrict__ eps_in, uint32_t b, unsigned long long seed, unsigned long long stream_id) {
  if (eps_in) return eps_in[b];
  curandStatePhilox4_32_10_t st;
  curand_init(seed ^ 0x9E3779B97F4A7C15ull, (unsigned long long)b, stream_id * 256ull, &st);
  return curand_uniform(&st);   // (0,1]; torch.rand is [0,1)
}

// x_hat = eps x + (1 - eps) fake per image (src/w_gp_gan.py:197-201) over NHWC rows [B*HW, C].  The two products and the sum
// are rounded separately (no FMA contraction): bit-identical to torch's eps * x + (1 - eps) * fake in fp32, then bf16.
// eps_out[b] (nullable) receives the eps used.  One thread per value, grid-stride.
__global__ void __launch_bounds__(256) gp_interp_kernel(const __nv_bfloat16* __restrict__ xr, int ldr, const __nv_bfloat16* __restrict__ xf,
                                                        int ldf, uint32_t HW, uint32_t C, uint32_t total, const float* __restrict__ eps_in,
                                                        float* __restrict__ eps_out, unsigned long long seed, unsigned long long stream_id,
                                                        __nv_bfloat16* __restrict__ out, int ldo) {
  griddep_sync();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const uint32_t pix = i / C, c = i - pix * C, b = pix / HW;
    const float e = gp_eps(eps_in, b, seed, stream_id);
    const float a = __bfloat162float(xr[size_t(pix) * ldr + c]), f = __bfloat162float(xf[size_t(pix) * ldf + c]);
    out[size_t(pix) * ldo + c] = __float2bfloat16_rn(__fadd_rn(__fmul_rn(e, a), __fmul_rn(__fsub_rn(1.f, e), f)));
    if (eps_out && c == 0 && pix == b * HW) eps_out[b] = e;
  }
}

// One block per image b of the image gradient g [B*HW, C]: norm_b = ||g_b||_2 (fp32 per thread, fixed reduction tree),
// k_b = 2 lambda inv_grad (norm_b - 1) / norm_b, or 0 when norm_b == 0 (torch's subgradient, DESIGN.md §4), and the tangent
// seed r_b = k_b g_b = dP/dg_b in bf16.  norm_out[b] = norm_b.
constexpr int kGpThreads = 256;
__global__ void __launch_bounds__(kGpThreads) gp_penalty_kernel(const __nv_bfloat16* __restrict__ g, int ldg, int HW, int C, float lambda,
                                                                float inv_grad, __nv_bfloat16* __restrict__ r, int ldr, float* __restrict__ norm_out) {
  griddep_sync();
  __shared__ double sh[kGpThreads / 32];
  const int n = HW * C;
  const __nv_bfloat16* gb = g + size_t(blockIdx.x) * HW * ldg;
  __nv_bfloat16* rb = r + size_t(blockIdx.x) * HW * ldr;
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += kGpThreads) {
    const int pix = i / C, c = i - pix * C;
    const float v = __bfloat162float(gb[size_t(pix) * ldg + c]);
    ss = fmaf(v, v, ss);
  }
  const float norm = sqrtf(float(block_sum<kGpThreads>(double(ss), sh)));
  const float k = norm > 0.f ? 2.f * lambda * inv_grad * (norm - 1.f) / norm : 0.f;
  for (int i = threadIdx.x; i < n; i += kGpThreads) {
    const int pix = i / C, c = i - pix * C;
    rb[size_t(pix) * ldr + c] = __float2bfloat16_rn(k * __bfloat162float(gb[size_t(pix) * ldg + c]));
  }
  if (threadIdx.x == 0) norm_out[blockIdx.x] = norm;
}
// loss[0] += lambda inv_loss sum_b (norm_b - 1)^2 (src/w_gp_gan.py:215,218); one block, fixed order
__global__ void __launch_bounds__(kGpThreads) gp_loss_kernel(const float* __restrict__ norms, int B, float lambda, float inv_loss,
                                                             float* __restrict__ loss) {
  griddep_sync();
  __shared__ double sh[kGpThreads / 32];
  double t = 0.0;
  for (int b = threadIdx.x; b < B; b += kGpThreads) {
    const double d = double(norms[b]) - 1.0;
    t += d * d;
  }
  t = block_sum<kGpThreads>(t, sh);
  if (threadIdx.x == 0) loss[0] += float(double(lambda) * double(inv_loss) * t);
}

// ---- DRAGAN on the sigmoid conv critic (src/dra_gan.py:174-225, DESIGN.md §6b)
// (sum x, sum x^2) of the per-block partials of moments_kernel -> out[2] (doubles, fixed order): the local sums of
// images.std() that data-parallel ranks add before xhat_kernel reads them
__global__ void __launch_bounds__(256) moments_sum_kernel(const double* __restrict__ part, int nblk, double* __restrict__ out) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double s1 = 0, s2 = 0;
  for (int i = threadIdx.x; i < nblk; i += 256) { s1 += part[2 * i]; s2 += part[2 * i + 1]; }
  s1 = block_sum<256>(s1, sh);
  s2 = block_sum<256>(s2, sh);
  if (threadIdx.x == 0) { out[0] = s1; out[1] = s2; }
}

// ---- BEGAN's L1 reconstruction loss (src/be_gan.py:225,233,256) on the autoencoder D of the conv path
// r, x: `groups` 16-byte groups of bf16 (NHWC image rows back to back).  grad = sign(r - x) * inv * (coef ? coef[0] : 1) as
// bf16 (sign(0) = 0, torch's abs backward; coef is a device scalar so that K never crosses to the host), and the block's
// partial of sum |r - x| in double (r - x of two bf16 values is exact in double).  Each of r and x is read once.
constexpr int kL1Unroll = 2;
__global__ void __launch_bounds__(256) l1_rows_kernel(const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ x,
                                                      uint32_t groups, float inv, const float* __restrict__ coef,
                                                      __nv_bfloat16* __restrict__ grad, double* __restrict__ part) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  const float k = coef ? inv * coef[0] : inv;
  const uint32_t stride = gridDim.x * blockDim.x;
  double acc = 0.0;
  for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < groups; i0 += stride * kL1Unroll) {
    uint4 rv[kL1Unroll], xv[kL1Unroll];
#pragma unroll
    for (int u = 0; u < kL1Unroll; ++u) {
      const uint32_t i = i0 + u * stride;
      rv[u] = xv[u] = make_uint4(0, 0, 0, 0);
      if (i < groups && i >= i0) {
        rv[u] = __ldg(reinterpret_cast<const uint4*>(r) + i);
        xv[u] = __ldg(reinterpret_cast<const uint4*>(x) + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kL1Unroll; ++u) {
      const uint32_t i = i0 + u * stride;
      if (i >= groups || i < i0) continue;
      const uint32_t a[4] = {rv[u].x, rv[u].y, rv[u].z, rv[u].w}, b[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
      float o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float rr = (q & 1) ? bf16_hi(a[q >> 1]) : bf16_lo(a[q >> 1]);
        const float xx = (q & 1) ? bf16_hi(b[q >> 1]) : bf16_lo(b[q >> 1]);
        const double d = double(rr) - double(xx);
        acc += fabs(d);
        o[q] = d > 0.0 ? k : (d < 0.0 ? -k : 0.f);
      }
      store_bf16x8(grad + size_t(i) * 8, o, 0);
    }
  }
  acc = block_sum<256>(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}
// sum of the per-block partials of l1_rows_kernel -> out[0] (one block, fixed order)
__global__ void __launch_bounds__(256) l1_sum_kernel(const double* __restrict__ part, int nblk, double* __restrict__ out) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  double s = 0;
  for (int i = threadIdx.x; i < nblk; i += 256) s += part[i];
  s = block_sum<256>(s, sh);
  if (threadIdx.x == 0) out[0] = s;
}

// ---- The VAE's reconstruction loss (src/vae.py:203) through the conv decoder's sigmoid output
// out = sigmoid(pre) and x: `groups` 16-byte groups of bf16 (NHWC image rows back to back; out as col2im's C2I_SIGMOID mode
// stores it).  grad = 2 scale (out - x) out (1 - out) = d(scale sum (x - out)^2)/d(pre) as bf16, and the block's partial of
// sum (x - out)^2 in double (x - out of two bf16 values is exact in double); l1_sum_kernel adds the partials in fixed order.
constexpr int kSseUnroll = 2;
__global__ void __launch_bounds__(256) sse_sigmoid_rows_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ x,
                                                               uint32_t groups, float scale, __nv_bfloat16* __restrict__ grad,
                                                               double* __restrict__ part) {
  griddep_sync();
  __shared__ double sh[256 / 32];
  const float k = 2.f * scale;
  const uint32_t stride = gridDim.x * blockDim.x;
  double acc = 0.0;
  for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < groups; i0 += stride * kSseUnroll) {
    uint4 ov[kSseUnroll], xv[kSseUnroll];
#pragma unroll
    for (int u = 0; u < kSseUnroll; ++u) {
      const uint32_t i = i0 + u * stride;
      ov[u] = xv[u] = make_uint4(0, 0, 0, 0);
      if (i < groups && i >= i0) {
        ov[u] = __ldg(reinterpret_cast<const uint4*>(out) + i);
        xv[u] = __ldg(reinterpret_cast<const uint4*>(x) + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kSseUnroll; ++u) {
      const uint32_t i = i0 + u * stride;
      if (i >= groups || i < i0) continue;
      const uint32_t a[4] = {ov[u].x, ov[u].y, ov[u].z, ov[u].w}, b[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
      float o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float oo = (q & 1) ? bf16_hi(a[q >> 1]) : bf16_lo(a[q >> 1]);
        const float xx = (q & 1) ? bf16_hi(b[q >> 1]) : bf16_lo(b[q >> 1]);
        const double d = double(oo) - double(xx);
        acc = fma(d, d, acc);
        o[q] = k * (oo - xx) * oo * (1.f - oo);
      }
      store_bf16x8(grad + size_t(i) * 8, o, 0);
    }
  }
  acc = block_sum<256>(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// ---- The autoencoder's ReLU code (src/ae.py:38-39) between the encoder head's fp32 rows h [rows, ldm] and the decoder.
// One thread per (row, 8-column group of the output row), one 16-byte store; columns past z are the constant part of the
// layout: the ones column at z and zeros (ae_latent_kernel), zeros only (ae_dlatent_kernel).
__global__ void __launch_bounds__(256) ae_latent_kernel(const float* __restrict__ h, int ldm, __nv_bfloat16* __restrict__ zb, int ldz,
                                                        int rows, int z) {
  griddep_sync();
  const int groups = ldz / 8;
  const long long t = blockIdx.x * 256ll + threadIdx.x;
  if (t >= (long long)rows * groups) return;
  const int r = int(t / groups), c0 = int(t % groups) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    v[j] = c < z ? fmaxf(h[(long long)r * ldm + c], 0.f) : (c == z ? 1.f : 0.f);
  }
  store_bf16x8(zb + (long long)r * ldz + c0, v, 0);
}

// dh = dz 1[h > 0] (0 at h == 0 and for NaN h, as torch's threshold backward) -> bf16 [rows, ld], zeros past z
__global__ void __launch_bounds__(256) ae_dlatent_kernel(const float* __restrict__ h, int ldm, const float* __restrict__ dz, int lddz,
                                                         __nv_bfloat16* __restrict__ out, int ld, int rows, int z) {
  griddep_sync();
  const int groups = ld / 8;
  const long long t = blockIdx.x * 256ll + threadIdx.x;
  if (t >= (long long)rows * groups) return;
  const int r = int(t / groups), c0 = int(t % groups) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    v[j] = (c < z && h[(long long)r * ldm + c] > 0.f) ? dz[(long long)r * lddz + c] : 0.f;
  }
  store_bf16x8(out + (long long)r * ld + c0, v, 0);
}

// Inference-mode BatchNorm2d's (mean, invstd) from the running statistics: stats[c] = running[0][c], stats[C + c] =
// 1 / sqrt(running[1][c] + eps), in bn_finalize_kernel's layout and precision, for bn_apply_kernel
__global__ void bn_eval_stats_kernel(const float* __restrict__ running, int C, float eps, float* __restrict__ stats) {
  griddep_sync();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  stats[c] = running[c];
  stats[C + c] = float(1.0 / sqrt(double(running[C + c]) + double(eps)));
}

// ---- InfoGAN's structured generator input (compute_noise, src/info_gan.py:306-325) drawn on the device
// Row r of the bf16 GEMM operand out [rows, ld] is [z (zd) | one-hot (nd) | continuous code (nc) | 1 | 0 ...], and codes
// [rows, K = zd + nd + nc] fp32 holds the same K values (the MI loss's targets).  The N(0, 1) values are rounded to bf16
// before both stores, so the two copies agree bit for bit.  One thread per (row, 8-column group holding draws or the ones
// column), 16-byte stores; the thread also writes its share of the row's zero padding groups (stage_noise_kernel's mapping).
// Philox is keyed by seed; the counter's high 64 bits are stream_id, the low 64 bits a block index unique within the
// stream: row r owns blocks [r (2 gz + 1), (r + 1)(2 gz + 1)).  Its first block draws the category, (w nd) >> 32 of one
// 32-bit word w (uniform over [0, nd) to 2^-32, never nd), so every thread of the row computes the same index; group g
// draws its 8 normals from blocks 2g + 1 and 2g + 2.
__global__ void __launch_bounds__(256) info_noise_kernel(__nv_bfloat16* __restrict__ out, int ld, float* __restrict__ codes, int rows,
                                                         int zd, int nd, int nc, unsigned long long seed, unsigned long long stream_id) {
  griddep_sync();
  const int K = zd + nd + nc, groups = ld / 8, gz = (K + 8) / 8;
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)rows * gz) return;
  const int r = int(t / gz), g = int(t % gz), c0 = g * 8;
  const unsigned long long blk0 = (unsigned long long)r * (2 * gz + 1);
  float v[8];
  if (c0 < K) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, stream_id, 4ull * (blk0 + 1 + 2 * g), &st);
    const float4 a = curand_normal4(&st), b = curand_normal4(&st);
    const float nrm[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    int cat = -1;
    if (c0 < zd + nd && c0 + 8 > zd) {
      curand_init(seed, stream_id, 4ull * blk0, &st);
      cat = int((unsigned long long)curand(&st) * (unsigned)nd >> 32);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      if (c >= zd && c < zd + nd) v[j] = c - zd == cat ? 1.f : 0.f;
      else v[j] = c < K ? __bfloat162float(__float2bfloat16_rn(nrm[j])) : (c == K ? 1.f : 0.f);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c0 + j < K) codes[(long long)r * K + c0 + j] = v[j];
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = c0 + j == K ? 1.f : 0.f;
  }
  store_bf16x8(out + ((long long)r * groups + g) * 8, v, 0);
  uint4* row = reinterpret_cast<uint4*>(out) + (long long)r * groups;
  for (int pg = gz + g; pg < groups; pg += gz) row[pg] = make_uint4(0, 0, 0, 0);
}

// One block per x_hat image b.  J [HW*C] = image gradient of the logit s_b (the beta chain seeded with 1), xh the image.
// sigma = sigmoid(s_b), sigma' = sigma (1 - sigma), ||g|| = sigma' ||J|| (the gradient of D's sigmoid output),
// k = 2 lambda inv_grad (||g|| - K); the tangent seed of the penalty's double backward is
//   r = k sigma' [J / ||J|| + (1 - 2 sigma) ||J|| xh]      (0 when ||J|| = 0)
// whose tangent pass carries both sigma'' ||J|| ds/dtheta (the forward activations of xh are its own tangent: no biases,
// LeakyReLU positively homogeneous) and sigma' (J/||J||) dJ/dtheta.  norm_out[b] = ||g||, r in bf16.
__global__ void __launch_bounds__(kGpThreads) dra_penalty_kernel(const __nv_bfloat16* __restrict__ J, int ldj, const __nv_bfloat16* __restrict__ xh,
                                                                 int ldx, const float* __restrict__ logits, int HW, int C, float lambda, float K,
                                                                 float inv_grad, __nv_bfloat16* __restrict__ r, int ldr, float* __restrict__ norm_out) {
  griddep_sync();
  __shared__ double sh[kGpThreads / 32];
  const int n = HW * C;
  const __nv_bfloat16* jb = J + size_t(blockIdx.x) * HW * ldj;
  const __nv_bfloat16* xb = xh + size_t(blockIdx.x) * HW * ldx;
  __nv_bfloat16* rb = r + size_t(blockIdx.x) * HW * ldr;
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += kGpThreads) {
    const int pix = i / C, c = i - pix * C;
    const float v = __bfloat162float(jb[size_t(pix) * ldj + c]);
    ss = fmaf(v, v, ss);
  }
  const float nj = sqrtf(float(block_sum<kGpThreads>(double(ss), sh)));
  const float sg = 1.f / (1.f + expf(-logits[blockIdx.x])), sp = sg * (1.f - sg);
  const float ng = sp * nj;
  const float k = 2.f * lambda * inv_grad * (ng - K) * sp;
  const float a = nj > 0.f ? k / nj : 0.f, b = nj > 0.f ? k * (1.f - 2.f * sg) * nj : 0.f;
  for (int i = threadIdx.x; i < n; i += kGpThreads) {
    const int pix = i / C, c = i - pix * C;
    const float jv = __bfloat162float(jb[size_t(pix) * ldj + c]), xv = __bfloat162float(xb[size_t(pix) * ldx + c]);
    rb[size_t(pix) * ldr + c] = __float2bfloat16_rn(fmaf(a, jv, b * xv));
  }
  if (threadIdx.x == 0) norm_out[blockIdx.x] = ng;
}
// loss[0] += lambda inv_loss sum_b (norm_b - K)^2 (src/dra_gan.py:219); one block, fixed order
__global__ void __launch_bounds__(kGpThreads) dra_loss_kernel(const float* __restrict__ norms, int B, float lambda, float K, float inv_loss,
                                                              float* __restrict__ loss) {
  griddep_sync();
  __shared__ double sh[kGpThreads / 32];
  double t = 0.0;
  for (int b = threadIdx.x; b < B; b += kGpThreads) {
    const double d = double(norms[b]) - double(K);
    t += d * d;
  }
  t = block_sum<kGpThreads>(t, sh);
  if (threadIdx.x == 0) loss[0] += float(double(lambda) * double(inv_loss) * t);
}

// im2col of the masked tensor x * LeakyReLU'(m) (m: the layer's activation, whose sign is the mask): the tangent
// t_l = phi'_l(y_l) * u_l of the penalty's forward-mode pass, gathered straight into the column matrix that both the next
// tangent GEMM and the penalty's weight-gradient GEMM read.  C % 8 == 0; the item mapping is im2col_k4s2_kernel<true>'s
// plus one 16-byte load of m per item.  The product is rounded once (fp32 -> bf16).
__global__ void __launch_bounds__(256) im2col_k4s2_lrelu_mask_kernel(const __nv_bfloat16* __restrict__ x, int H, int W, int C, int ldx,
                                                                     const __nv_bfloat16* __restrict__ m, int ldm, float slope,
                                                                     __nv_bfloat16* __restrict__ col, int ldc, uint32_t total, FastDiv dcg,
                                                                     FastDiv dwo, FastDiv dho) {
  griddep_sync();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x; t0 < total; t0 += stride * kConvUnroll) {
    uint4 v[kConvUnroll], mv[kConvUnroll];
    __nv_bfloat16* dst[kConvUnroll];
    bool live[kConvUnroll];
#pragma unroll
    for (int u = 0; u < kConvUnroll; ++u) {
      const uint32_t t = t0 + u * stride;
      live[u] = t < total && t >= t0;
      uint32_t r, g;
      fdivmod(t, dcg, r, g);
      const uint32_t tap = r & 15u;
      r >>= 4;
      uint32_t q, wo, b, ho;
      fdivmod(r, dwo, q, wo);
      fdivmod(q, dho, b, ho);
      const int iy = 2 * int(ho) - 1 + int(tap >> 2), ix = 2 * int(wo) - 1 + int(tap & 3u);
      const bool ok = live[u] && iy >= 0 && iy < H && ix >= 0 && ix < W;
      const size_t p = (size_t(b) * H + iy) * W + ix;
      dst[u] = col + size_t(r) * ldc + tap * C + g * 8;
      v[u] = make_uint4(0, 0, 0, 0);
      mv[u] = make_uint4(0, 0, 0, 0);
      if (ok) {
        v[u] = __ldg(reinterpret_cast<const uint4*>(x + p * ldx + g * 8));
        mv[u] = __ldg(reinterpret_cast<const uint4*>(m + p * ldm + g * 8));
      }
    }
#pragma unroll
    for (int u = 0; u < kConvUnroll; ++u) {
      if (!live[u]) continue;
      const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w}, mw[4] = {mv[u].x, mv[u].y, mv[u].z, mv[u].w};
      float o[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        o[2 * q] = bf16_lo(mw[q]) > 0.f ? bf16_lo(w[q]) : slope * bf16_lo(w[q]);
        o[2 * q + 1] = bf16_hi(mw[q]) > 0.f ? bf16_hi(w[q]) : slope * bf16_hi(w[q]);
      }
      store_bf16x8(dst[u], o, 0);
    }
  }
}

// out = x * LeakyReLU'(m) over rows [rows, C], C % 8 == 0 (the 4x4 layer in front of the 1-logit conv, where the masked
// im2col degenerates to an elementwise mask).  out may alias x or m: every thread reads its 16 bytes before writing them.
__global__ void __launch_bounds__(256) lrelu_mask_rows_kernel(const __nv_bfloat16* x, int ldx, const __nv_bfloat16* m, int ldm, uint32_t groups,
                                                              uint32_t total, float slope, __nv_bfloat16* out, int ldo) {
  griddep_sync();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const uint32_t r = i / groups, g = i - r * groups;
    const uint4 v = *reinterpret_cast<const uint4*>(x + size_t(r) * ldx + g * 8);
    const uint4 mv = *reinterpret_cast<const uint4*>(m + size_t(r) * ldm + g * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w}, mw[4] = {mv.x, mv.y, mv.z, mv.w};
    float o[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      o[2 * q] = bf16_lo(mw[q]) > 0.f ? bf16_lo(w[q]) : slope * bf16_lo(w[q]);
      o[2 * q + 1] = bf16_hi(mw[q]) > 0.f ? bf16_hi(w[q]) : slope * bf16_hi(w[q]);
    }
    store_bf16x8(out + size_t(r) * ldo + g * 8, o, 0);
  }
}

// ---------------------------------------------------------------- device-resident dataset pool (DESIGN.md §6b)
// The pool keeps each image as row_vals one-byte codes in NHWC order, and a 256-entry table of bf16 bit patterns maps a
// code to the value stage_images would write.  Batch row r reads pool row sampler_index(smp, smp.offset + r) (kernels.cuh:
// Sampler) and becomes bf16 NHWC row r of out [rows, row_vals].  One block walks one row: each thread issues its 16-byte
// code loads (16 values each) before it looks them up in the shared table and writes two 16-byte stores per load; the
// next row's pool index is computed while this row is in flight.  row_vals % 16 == 0 and 16-byte aligned rows (host checks).
constexpr int kPoolThreads = 256, kPoolUnroll = 4;
__global__ void __launch_bounds__(kPoolThreads) stage_pool_rows_kernel(const uint8_t* __restrict__ codes, int row_vals,
                                                                       const uint16_t* __restrict__ table, const Sampler smp, int rows,
                                                                       __nv_bfloat16* __restrict__ out, int* __restrict__ idx_out) {
  __shared__ uint16_t lut[256];
  griddep_sync();
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = table[i];
  __syncthreads();
  const int groups = row_vals >> 4;
  unsigned int src_next = blockIdx.x < rows ? sampler_index(smp, smp.offset + blockIdx.x) : 0u;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const unsigned int src = src_next;
    if (r + gridDim.x < rows) src_next = sampler_index(smp, smp.offset + (unsigned long long)(r + gridDim.x));
    if (idx_out && threadIdx.x == 0) idx_out[r] = int(src);
    const uint4* crow = reinterpret_cast<const uint4*>(codes + size_t(src) * row_vals);
    uint4* orow = reinterpret_cast<uint4*>(out + size_t(r) * row_vals);
    for (int g0 = threadIdx.x; g0 < groups; g0 += kPoolThreads * kPoolUnroll) {
      uint4 v[kPoolUnroll];
#pragma unroll
      for (int u = 0; u < kPoolUnroll; ++u) {
        const int g = g0 + u * kPoolThreads;
        v[u] = g < groups ? __ldg(crow + g) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < kPoolUnroll; ++u) {
        const int g = g0 + u * kPoolThreads;
        if (g >= groups) break;
        const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
        uint32_t o[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {      // byte j of a word is value 4q + j; bf16 pairs pack the lower-addressed value low
          o[2 * q] = uint32_t(lut[w[q] & 0xFFu]) | (uint32_t(lut[(w[q] >> 8) & 0xFFu]) << 16);
          o[2 * q + 1] = uint32_t(lut[(w[q] >> 16) & 0xFFu]) | (uint32_t(lut[w[q] >> 24]) << 16);
        }
        orow[2 * g] = make_uint4(o[0], o[1], o[2], o[3]);
        orow[2 * g + 1] = make_uint4(o[4], o[5], o[6], o[7]);
      }
    }
  }
}

// ---------------------------------------------------------------- the image layout at the autograd boundary
// The drop-in classes see images as NCHW-flattened fp32 [n, ch*64*64]; the kernels take NHWC bf16 rows [n*4096, ch].  One
// block converts kLayoutPix pixels of one image: the ch planes go through a shared tile [ch][kLayoutPix] so that both
// sides move 16 bytes per access (float4 per plane, 8 bf16 of the interleaved rows).  ch <= 4, 16-byte aligned pointers
// (host checks).
constexpr int kLayoutPix = 1024, kLayoutThreads = 256, kLayoutTiles = 4096 / kLayoutPix;

// dst = bf16_rn(x), or bf16_rn((x * f) * (1 - f)) with f = aux (NHWC bf16, the generator's stored sigmoid output): the
// upstream of the pre-sigmoid output from dL/dG(z), rounded once, in the order torch evaluates g * f * (1 - f)
__global__ void __launch_bounds__(kLayoutThreads) image_to_rows_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ aux,
                                                                       int ch, __nv_bfloat16* __restrict__ dst) {
  __shared__ float tile[4 * kLayoutPix];
  griddep_sync();
  const int b = blockIdx.x / kLayoutTiles, p0 = (blockIdx.x % kLayoutTiles) * kLayoutPix;
  for (int i = threadIdx.x; i < ch * (kLayoutPix / 4); i += kLayoutThreads) {
    const int c = i / (kLayoutPix / 4), q = i % (kLayoutPix / 4);
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + (size_t(b) * ch + c) * 4096 + p0) + q);
    *reinterpret_cast<float4*>(tile + c * kLayoutPix + 4 * q) = v;
  }
  __syncthreads();
  const size_t base = (size_t(b) * 4096 + p0) * ch;
  for (int k = threadIdx.x; k < kLayoutPix * ch / 8; k += kLayoutThreads) {
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = 8 * k + j, p = e / ch;
      f[j] = tile[(e - p * ch) * kLayoutPix + p];
    }
    if (aux) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(aux + base) + k);
      const __nv_bfloat162* s = reinterpret_cast<const __nv_bfloat162*>(&a);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 sf = __bfloat1622float2(s[j]);
        f[2 * j] = __fmul_rn(__fmul_rn(f[2 * j], sf.x), __fsub_rn(1.f, sf.x));
        f[2 * j + 1] = __fmul_rn(__fmul_rn(f[2 * j + 1], sf.y), __fsub_rn(1.f, sf.y));
      }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);     // .x (the lower address) = f[2j]
      ow[j] = *reinterpret_cast<const uint32_t*>(&h);
    }
    reinterpret_cast<uint4*>(dst + base)[k] = o;
  }
}

// dst = float(src): NHWC bf16 rows -> NCHW-flattened fp32, exact
__global__ void __launch_bounds__(kLayoutThreads) rows_to_image_kernel(const __nv_bfloat16* __restrict__ src, int ch, float* __restrict__ dst) {
  __shared__ float tile[4 * kLayoutPix];
  griddep_sync();
  const int b = blockIdx.x / kLayoutTiles, p0 = (blockIdx.x % kLayoutTiles) * kLayoutPix;
  const size_t base = (size_t(b) * 4096 + p0) * ch;
  for (int k = threadIdx.x; k < kLayoutPix * ch / 8; k += kLayoutThreads) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + base) + k);
    const __nv_bfloat162* s = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 sf = __bfloat1622float2(s[j]);
      const int e = 8 * k + 2 * j, p = e / ch, q = (e + 1) / ch;
      tile[(e - p * ch) * kLayoutPix + p] = sf.x;
      tile[(e + 1 - q * ch) * kLayoutPix + q] = sf.y;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ch * (kLayoutPix / 4); i += kLayoutThreads) {
    const int c = i / (kLayoutPix / 4), q = i % (kLayoutPix / 4);
    reinterpret_cast<float4*>(dst + (size_t(b) * ch + c) * 4096 + p0)[q] = *reinterpret_cast<const float4*>(tile + c * kLayoutPix + 4 * q);
  }
}

}  // namespace gm
