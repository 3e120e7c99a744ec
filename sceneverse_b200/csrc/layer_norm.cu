// Fused dropout + residual add + LayerNorm, forward and backward, for the post-norm transformer blocks of the GPS stack
//   y = LayerNorm(residual + dropout(x)) * gamma + beta
// (reference: modules/layers/transformers.py:145-154 `tgt = self.norm1(tgt + self.dropout1(tgt2))`, :311-315 for the
// spatial layers, modules/utils.py:18-25 for the plain LayerNorm of get_mlp_head; the BERT blocks upstream have the same
// form).  The reference runs it as 3-5 ATen kernels per block (dropout, add, dtype casts, layer_norm) plus a slow
// gamma/beta-gradient reduction in the backward; here it is one HBM-bound pass per direction:
//   forward : one warp per row, the row lives in registers (two-pass mean / variance), the dropout mask is the counter
//             hash of csrc/attn_common.cuh (nothing stored), the pre-norm sum s is written once for the backward;
//   backward: one warp per row for ds (and dx = ds o mask / (1 - p)); the gamma / beta gradients come from a second,
//             column-owning pass over g and s (L2-resident right after the first) whose per-CTA partial sums are
//             finished by a small fixed-order reduction — deterministic, no atomics.
// Algorithmic bytes per row (bf16 I/O, D columns): forward 2D (x) + 2D (residual) + 2D (s) + 2D (y) = 8D;
// backward 2D (g) + 2D (s) + 2D (ds) [+ 2D (dx)].
#include <cuda_bf16.h>

#include "attn_common.cuh"
#include "svgps.h"

namespace {

using attn::drop_pair_hash;
using attn::drop_row_key;

struct LnArgs {
  const void *x, *res, *g, *s_in;  // forward: x, res;  backward: g, s_in
  void *y, *s_out, *ds, *dx;
  const float *gamma, *beta;
  float *mean, *rstd;
  float *partials;                 // backward: [gridDim.x][2][D]
  int R, D;
  float eps;
  uint32_t t16;
  float inv_keep;
  unsigned long long seed;
  const unsigned long long *seed_offset;  // device counter added to the seed at run time (or null)
  int key_stride;                  // row r draws its dropout mask with the row key r * key_stride
};

template <typename T>
struct Chunk;  // 8 consecutive elements
template <>
struct Chunk<__nv_bfloat16> {
  static __device__ __forceinline__ void load(const void *base, size_t idx8, float (&v)[8]) {
    const uint4 u = __ldg(reinterpret_cast<const uint4 *>(base) + idx8);
    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
  static __device__ __forceinline__ void store(void *base, size_t idx8, const float (&v)[8]) {
    uint4 u;
    __nv_bfloat162 *h = reinterpret_cast<__nv_bfloat162 *>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    reinterpret_cast<uint4 *>(base)[idx8] = u;
  }
  static __device__ __forceinline__ float round(float f) { return __bfloat162float(__float2bfloat16_rn(f)); }
};
template <>
struct Chunk<float> {
  static __device__ __forceinline__ void load(const void *base, size_t idx8, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4 *>(base) + 2 * idx8);
    const float4 b = __ldg(reinterpret_cast<const float4 *>(base) + 2 * idx8 + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void store(void *base, size_t idx8, const float (&v)[8]) {
    reinterpret_cast<float4 *>(base)[2 * idx8] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4 *>(base)[2 * idx8 + 1] = make_float4(v[4], v[5], v[6], v[7]);
  }
  static __device__ __forceinline__ float round(float f) { return f; }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// keep-scale of the 8 elements of chunk c (columns 8c .. 8c+7) of a row with key rk
__device__ __forceinline__ void drop_scale8(uint32_t rk, int c, uint32_t t16, float inv_keep, float (&m)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t hh = drop_pair_hash(rk, (uint32_t)(c * 4 + i));
    m[2 * i] = (hh & 0xFFFFu) >= t16 ? inv_keep : 0.f;
    m[2 * i + 1] = (hh >> 16) >= t16 ? inv_keep : 0.f;
  }
}

template <typename T, int MAXCH, bool HAS_RES, bool DROP>
__global__ void __launch_bounds__(256) ln_fwd_kernel(const LnArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = a.D >> 3;
  const float invD = 1.0f / (float)a.D;
  for (int row = blockIdx.x * 8 + warp; row < a.R; row += gridDim.x * 8) {
    const size_t base8 = (size_t)row * nch;
    float v[MAXCH][8];
    uint32_t rk = 0;
    if (DROP) rk = drop_row_key(attn::effective_seed(a.seed, a.seed_offset), (unsigned long long)row * a.key_stride);
    float sum = 0.f;
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        Chunk<T>::load(a.x, base8 + c, v[ch]);
        if (DROP) {
          float m[8];
          drop_scale8(rk, c, a.t16, a.inv_keep, m);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[ch][i] *= m[i];
        }
        if (HAS_RES) {
          float r[8];
          Chunk<T>::load(a.res, base8 + c, r);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[ch][i] += r[i];
        }
        if (HAS_RES || DROP) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[ch][i] = Chunk<T>::round(v[ch][i]);  // the statistics see exactly what is stored
          Chunk<T>::store(a.s_out, base8 + c, v[ch]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += v[ch][i];
      }
    }
    const float mean = warp_sum(sum) * invD;
    float sq = 0.f;
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = v[ch][i] - mean;
          sq = fmaf(d, d, sq);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) * invD + a.eps);
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        float o[8], gam[8], bet[8];  // gamma / beta come from L1 per row: keeping them resident costs 48 registers
        Chunk<float>::load(a.gamma, c, gam);
        Chunk<float>::load(a.beta, c, bet);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = fmaf((v[ch][i] - mean) * rstd, gam[i], bet[i]);
        Chunk<T>::store(a.y, base8 + c, o);
      }
    }
    if (lane == 0) {
      a.mean[row] = mean;
      a.rstd[row] = rstd;
    }
  }
}

// backward, parts 1 + 2 in one pass over (g, s): ds (and dx) — one warp per row, gamma re-read from L1 per row — AND the
// per-CTA partial sums of dgamma = sum_rows g * xhat, dbeta = sum_rows g (a separate column-sum kernel re-read both
// tensors: 0.32 ms per step).
// At most 2 CTAs per SM keep the partial-sum scratch at BWD_MAX_BLOCKS rows; lane l of every warp owns the same columns,
// so a thread carries its 8 * MAXCH column sums in registers across its rows and the 8 warps meet once in shared memory.
template <typename T, int MAXCH, bool DROP>
__global__ void __launch_bounds__(256, 2) ln_bwd_fused_kernel(const LnArgs a) {
  extern __shared__ float wsum[];  // [8 warps][2][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = a.D >> 3;
  const float invD = 1.0f / (float)a.D;
  float pg[MAXCH][8], pb[MAXCH][8];
#pragma unroll
  for (int ch = 0; ch < MAXCH; ++ch)
#pragma unroll
    for (int i = 0; i < 8; ++i) pg[ch][i] = pb[ch][i] = 0.f;
  for (int row = blockIdx.x * 8 + warp; row < a.R; row += gridDim.x * 8) {
    const size_t base8 = (size_t)row * nch;
    const float mean = a.mean[row], rstd = a.rstd[row];
    float gy[MAXCH][8], xh[MAXCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        float g[8], s[8], gam[8];
        Chunk<T>::load(a.g, base8 + c, g);
        Chunk<T>::load(a.s_in, base8 + c, s);
        Chunk<float>::load(a.gamma, c, gam);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          xh[ch][i] = (s[i] - mean) * rstd;
          gy[ch][i] = g[i] * gam[i];
          s1 += gy[ch][i];
          s2 = fmaf(gy[ch][i], xh[ch][i], s2);
          pg[ch][i] = fmaf(g[i], xh[ch][i], pg[ch][i]);
          pb[ch][i] += g[i];
        }
      }
    }
    s1 = warp_sum(s1) * invD;
    s2 = warp_sum(s2) * invD;
    uint32_t rk = 0;
    if (DROP) rk = drop_row_key(attn::effective_seed(a.seed, a.seed_offset), (unsigned long long)row * a.key_stride);
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        float d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = rstd * (gy[ch][i] - fmaf(xh[ch][i], s2, s1));
        Chunk<T>::store(a.ds, base8 + c, d);
        if (DROP) {
          float m[8];
          drop_scale8(rk, c, a.t16, a.inv_keep, m);
#pragma unroll
          for (int i = 0; i < 8; ++i) d[i] *= m[i];
          Chunk<T>::store(a.dx, base8 + c, d);
        }
      }
    }
  }
#pragma unroll
  for (int ch = 0; ch < MAXCH; ++ch) {
    const int c = lane + 32 * ch;
    if (c < nch) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        wsum[(warp * 2) * a.D + c * 8 + i] = pg[ch][i];
        wsum[(warp * 2 + 1) * a.D + c * 8 + i] = pb[ch][i];
      }
    }
  }
  __syncthreads();
  float *out = a.partials + (size_t)blockIdx.x * 2 * a.D;
  for (int d = threadIdx.x; d < 2 * a.D; d += 256) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += wsum[w * 2 * a.D + d];
    out[d] = v;
  }
}

// backward, part 3: fixed-order sum of the per-CTA partials; one CTA per 32 columns, the 8 warps split the partial rows
__global__ void __launch_bounds__(256) ln_bwd_reduce_kernel(const float *partials, int nblk, int D, float *dgamma, float *dbeta,
                                                           int accumulate) {
  __shared__ float red[8][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (d < 2 * D)
    for (int b = warp; b < nblk; b += 8) s += partials[(size_t)b * 2 * D + d];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && d < 2 * D) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    float *dst = d < D ? dgamma + d : dbeta + (d - D);
    *dst = accumulate ? *dst + t : t;   // accumulate: straight into the flat gradient buffer (one writer per element)
  }
}

// ---- row-wise L2 normalisation (the contrastive heads: F.normalize(x, dim=-1, p=2) of optim/loss/contra_loss.py:29-30, 59-60, 86-87
// 60-61 and its autograd: ~9 ATen kernels per call, six calls per step) -------------------------------------------------
//   y = x / max(||x||_2, eps)          dx = (g - y (y . g)) / ||x||   (||x|| >= eps),   g / eps   (clamped rows)
template <typename T, int MAXCH>
__global__ void __launch_bounds__(256) l2norm_fwd_kernel(const void *x, void *y, float *norm, int R, int D, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = D >> 3;
  for (int row = blockIdx.x * 8 + warp; row < R; row += gridDim.x * 8) {
    const size_t base8 = (size_t)row * nch;
    float v[MAXCH][8];
    float ss = 0.f;
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        Chunk<T>::load(x, base8 + c, v[ch]);
#pragma unroll
        for (int i = 0; i < 8; ++i) ss = fmaf(v[ch][i], v[ch][i], ss);
      }
    }
    const float nrm = sqrtf(warp_sum(ss));
    const float inv = 1.0f / fmaxf(nrm, eps);
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[ch][i] *= inv;
        Chunk<T>::store(y, base8 + c, v[ch]);
      }
    }
    if (lane == 0) norm[row] = nrm;
  }
}
template <typename T, int MAXCH>
__global__ void __launch_bounds__(256) l2norm_bwd_kernel(const void *g, const void *y, const float *norm, void *dx, int R, int D,
                                                        float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = D >> 3;
  for (int row = blockIdx.x * 8 + warp; row < R; row += gridDim.x * 8) {
    const size_t base8 = (size_t)row * nch;
    const float nrm = norm[row];
    const bool clamped = nrm < eps;
    const float inv = 1.0f / fmaxf(nrm, eps);
    float gg[MAXCH][8], yy[MAXCH][8];
    float dot = 0.f;
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        Chunk<T>::load(g, base8 + c, gg[ch]);
        Chunk<T>::load(y, base8 + c, yy[ch]);
#pragma unroll
        for (int i = 0; i < 8; ++i) dot = fmaf(gg[ch][i], yy[ch][i], dot);
      }
    }
    dot = clamped ? 0.f : warp_sum(dot);
#pragma unroll
    for (int ch = 0; ch < MAXCH; ++ch) {
      const int c = lane + 32 * ch;
      if (c < nch) {
        float d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = (gg[ch][i] - yy[ch][i] * dot) * inv;
        Chunk<T>::store(dx, base8 + c, d);
      }
    }
  }
}
template <typename T, int MAXCH>
int launch_l2norm(bool bwd, const void *a, const void *b, float *norm, void *out, int R, int D, float eps, cudaStream_t st) {
  int grid = (R + 7) / 8;
  if (grid > 132 * 8) grid = 132 * 8;
  if (bwd) l2norm_bwd_kernel<T, MAXCH><<<grid, 256, 0, st>>>(a, b, norm, out, R, D, eps);
  else l2norm_fwd_kernel<T, MAXCH><<<grid, 256, 0, st>>>(a, out, norm, R, D, eps);
  return sv::after_launch();
}
int run_l2norm(bool bwd, const void *a, const void *b, float *norm, void *out, int io_bf16, int R, int D, float eps, void *stream) {
  if (R < 0 || D < 8 || (D % 8) || D > 1024 || !(eps > 0.f)) return SV_ERR_INVALID_ARG;
  if (R == 0) return SV_OK;
  if (!a || !norm || !out || (bwd && !b)) return SV_ERR_INVALID_ARG;
  auto al = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!al(a) || !al(out) || (b && !al(b))) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int maxch = (D + 255) / 256;
  if (io_bf16) {
    switch (maxch) {
      case 1: return launch_l2norm<__nv_bfloat16, 1>(bwd, a, b, norm, out, R, D, eps, st);
      case 2: return launch_l2norm<__nv_bfloat16, 2>(bwd, a, b, norm, out, R, D, eps, st);
      case 3: return launch_l2norm<__nv_bfloat16, 3>(bwd, a, b, norm, out, R, D, eps, st);
      default: return launch_l2norm<__nv_bfloat16, 4>(bwd, a, b, norm, out, R, D, eps, st);
    }
  }
  switch (maxch) {
    case 1: return launch_l2norm<float, 1>(bwd, a, b, norm, out, R, D, eps, st);
    case 2: return launch_l2norm<float, 2>(bwd, a, b, norm, out, R, D, eps, st);
    case 3: return launch_l2norm<float, 3>(bwd, a, b, norm, out, R, D, eps, st);
    default: return launch_l2norm<float, 4>(bwd, a, b, norm, out, R, D, eps, st);
  }
}

constexpr int BWD_MAX_BLOCKS = 296;

template <typename T, int MAXCH>
int launch_fwd(const LnArgs &a, bool has_res, bool drop, cudaStream_t st) {
  int grid = (a.R + 7) / 8;
  if (grid > 132 * 8) grid = 132 * 8;
  if (has_res && drop) ln_fwd_kernel<T, MAXCH, true, true><<<grid, 256, 0, st>>>(a);
  else if (has_res) ln_fwd_kernel<T, MAXCH, true, false><<<grid, 256, 0, st>>>(a);
  else if (drop) ln_fwd_kernel<T, MAXCH, false, true><<<grid, 256, 0, st>>>(a);
  else ln_fwd_kernel<T, MAXCH, false, false><<<grid, 256, 0, st>>>(a);
  return sv::after_launch();
}
template <typename T, int MAXCH>
int launch_bwd(const LnArgs &a, bool drop, float *dgamma, float *dbeta, int accumulate, cudaStream_t st) {
  int grid = (a.R + 7) / 8;
  if (grid > BWD_MAX_BLOCKS) grid = BWD_MAX_BLOCKS;
  const size_t smem = (size_t)8 * 2 * a.D * sizeof(float);   // <= 64 KB at D = 1024
  static bool configured = false;
  if (!configured) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(ln_bwd_fused_kernel<T, MAXCH, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
    if (!rc) rc = sv::cuda_status(cudaFuncSetAttribute(ln_bwd_fused_kernel<T, MAXCH, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
    if (rc) return rc;
    configured = true;
  }
  if (drop) ln_bwd_fused_kernel<T, MAXCH, true><<<grid, 256, smem, st>>>(a);
  else ln_bwd_fused_kernel<T, MAXCH, false><<<grid, 256, smem, st>>>(a);
  int rc = sv::after_launch();
  if (rc) return rc;
  ln_bwd_reduce_kernel<<<(2 * a.D + 31) / 32, 256, 0, st>>>(a.partials, grid, a.D, dgamma, dbeta, accumulate);
  return sv::after_launch();
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int sv_layer_norm_scratch_floats(int D) { return D > 0 ? BWD_MAX_BLOCKS * 2 * D : 0; }

extern "C" int sv_layer_norm_fwd_rows(const void *x, const void *residual, int io_bf16, int R, int D, const float *gamma,
                                      const float *beta, float eps, float dropout_p, unsigned long long seed, void *y,
                                      void *s, float *mean, float *rstd, int row_key_stride, void *stream) {
  if (R < 0 || D < 8 || (D % 8) || D > 1024 || !(dropout_p >= 0.f) || dropout_p >= 1.f || row_key_stride < 1)
    return SV_ERR_INVALID_ARG;
  if (R == 0) return SV_OK;
  const bool drop = dropout_p > 0.f, has_res = residual != nullptr;
  if (!x || !gamma || !beta || !y || !mean || !rstd || ((drop || has_res) && !s)) return SV_ERR_INVALID_ARG;
  if (!aligned16(x) || !aligned16(y) || !aligned16(gamma) || !aligned16(beta) || (residual && !aligned16(residual)) ||
      (s && !aligned16(s)))
    return SV_ERR_INVALID_ARG;
  LnArgs a{};
  a.x = x; a.res = residual; a.y = y; a.s_out = s; a.gamma = gamma; a.beta = beta; a.mean = mean; a.rstd = rstd;
  a.R = R; a.D = D; a.eps = eps; a.t16 = attn::drop_threshold(dropout_p); a.inv_keep = 1.0f / (1.0f - dropout_p);
  a.seed = seed; a.seed_offset = sv::g_seed_offset; a.key_stride = row_key_stride;
  cudaStream_t st = (cudaStream_t)stream;
  const int maxch = (D + 255) / 256;
  const bool d = a.t16 != 0;
  if (io_bf16) {
    switch (maxch) {
      case 1: return launch_fwd<__nv_bfloat16, 1>(a, has_res, d, st);
      case 2: return launch_fwd<__nv_bfloat16, 2>(a, has_res, d, st);
      case 3: return launch_fwd<__nv_bfloat16, 3>(a, has_res, d, st);
      default: return launch_fwd<__nv_bfloat16, 4>(a, has_res, d, st);
    }
  }
  switch (maxch) {
    case 1: return launch_fwd<float, 1>(a, has_res, d, st);
    case 2: return launch_fwd<float, 2>(a, has_res, d, st);
    case 3: return launch_fwd<float, 3>(a, has_res, d, st);
    default: return launch_fwd<float, 4>(a, has_res, d, st);
  }
}

extern "C" int sv_layer_norm_bwd_rows(const void *g, const void *s, int io_bf16, int R, int D, const float *gamma,
                                      const float *mean, const float *rstd, float dropout_p, unsigned long long seed,
                                      void *ds, void *dx, float *dgamma, float *dbeta, int accumulate, float *scratch,
                                      int row_key_stride, void *stream) {
  if (R < 1 || D < 8 || (D % 8) || D > 1024 || !(dropout_p >= 0.f) || dropout_p >= 1.f || row_key_stride < 1)
    return SV_ERR_INVALID_ARG;
  const bool drop = dropout_p > 0.f;
  if (!g || !s || !gamma || !mean || !rstd || !ds || !dgamma || !dbeta || !scratch || (drop && !dx)) return SV_ERR_INVALID_ARG;
  if (!aligned16(g) || !aligned16(s) || !aligned16(gamma) || !aligned16(ds) || (dx && !aligned16(dx))) return SV_ERR_INVALID_ARG;
  LnArgs a{};
  a.g = g; a.s_in = s; a.ds = ds; a.dx = dx; a.gamma = gamma; a.mean = const_cast<float *>(mean);
  a.rstd = const_cast<float *>(rstd); a.partials = scratch;
  a.R = R; a.D = D; a.t16 = attn::drop_threshold(dropout_p); a.inv_keep = 1.0f / (1.0f - dropout_p); a.seed = seed; a.seed_offset = sv::g_seed_offset;
  a.key_stride = row_key_stride;
  cudaStream_t st = (cudaStream_t)stream;
  const int maxch = (D + 255) / 256;
  const bool d = a.t16 != 0;
  if (io_bf16) {
    switch (maxch) {
      case 1: return launch_bwd<__nv_bfloat16, 1>(a, d, dgamma, dbeta, accumulate, st);
      case 2: return launch_bwd<__nv_bfloat16, 2>(a, d, dgamma, dbeta, accumulate, st);
      case 3: return launch_bwd<__nv_bfloat16, 3>(a, d, dgamma, dbeta, accumulate, st);
      default: return launch_bwd<__nv_bfloat16, 4>(a, d, dgamma, dbeta, accumulate, st);
    }
  }
  switch (maxch) {
    case 1: return launch_bwd<float, 1>(a, d, dgamma, dbeta, accumulate, st);
    case 2: return launch_bwd<float, 2>(a, d, dgamma, dbeta, accumulate, st);
    case 3: return launch_bwd<float, 3>(a, d, dgamma, dbeta, accumulate, st);
    default: return launch_bwd<float, 4>(a, d, dgamma, dbeta, accumulate, st);
  }
}

extern "C" int sv_layer_norm_fwd(const void *x, const void *residual, int io_bf16, int R, int D, const float *gamma,
                                 const float *beta, float eps, float dropout_p, unsigned long long seed, void *y,
                                 void *s, float *mean, float *rstd, void *stream) {
  return sv_layer_norm_fwd_rows(x, residual, io_bf16, R, D, gamma, beta, eps, dropout_p, seed, y, s, mean, rstd, 1, stream);
}

extern "C" int sv_layer_norm_bwd_acc(const void *g, const void *s, int io_bf16, int R, int D, const float *gamma,
                                     const float *mean, const float *rstd, float dropout_p, unsigned long long seed, void *ds,
                                     void *dx, float *dgamma, float *dbeta, int accumulate, float *scratch, void *stream) {
  return sv_layer_norm_bwd_rows(g, s, io_bf16, R, D, gamma, mean, rstd, dropout_p, seed, ds, dx, dgamma, dbeta, accumulate,
                                scratch, 1, stream);
}

extern "C" int sv_l2norm_fwd(const void *x, int io_bf16, int R, int D, float eps, void *y, float *norm, void *stream) {
  return run_l2norm(false, x, nullptr, norm, y, io_bf16, R, D, eps, stream);
}

extern "C" int sv_l2norm_bwd(const void *g, const void *y, const float *norm, int io_bf16, int R, int D, float eps, void *dx,
                             void *stream) {
  return run_l2norm(true, g, y, const_cast<float *>(norm), dx, io_bf16, R, D, eps, stream);
}
