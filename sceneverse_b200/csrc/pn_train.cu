// Train-mode set abstraction of PointNet++ in channels-LAST form (SURVEY.md §8 row a7, config C2 — `ObjCls` pre-training with
// a trainable backbone; reference: pointnet2_utils.py:291-373 QueryAndGroup, pytorch_utils.py:11-36,67-120 SharedMLP =
// Conv2d(1x1, no bias) + BatchNorm2d (batch statistics) + ReLU, pointnet2_modules.py:70-73 max over nsample).
//
// The reference keeps (B, C, npoint, nsample) fp32 tensors and runs cuDNN 1x1 convolutions + cuDNN BatchNorm + ReLU + max_pool2d.
// Here a grouped tensor is a ROW matrix X[(b, centre, sample)][channel] in bf16, so that
//   * the 1x1 convolution is the native wgmma GEMM family of csrc/gemm.cu in all three directions (no bias: BN follows),
//   * BatchNorm2d in training mode is a COLUMN statistic over the rows: two HBM passes forward (moments, then normalise +
//     ReLU), two backward (d gamma / d beta sums, then dY) — the kernels below,
//   * the neighbourhood max is a max over `ns` consecutive rows.
// Kernels: group_rows (+grad), col_moments, bn_relu_apply, bn_relu_bwd_sums, bn_relu_bwd_apply, rowgroup_max (+grad).
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"
#include "sm90.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4 u, float (&v)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __uint_as_float(w[i] << 16);
    v[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
  return make_uint4(sm90::pack_bf16(v[0], v[1]), sm90::pack_bf16(v[2], v[3]), sm90::pack_bf16(v[4], v[5]), sm90::pack_bf16(v[6], v[7]));
}

// ---- grouping: X[(b, j, s)][0:3] = xyz[b, idx] - centre[b, j] (raw xyz when centre == null: GroupAll), X[..][3:3+C] = feat[b, idx],
// zero pad up to Cp.  feat: (B, N, C) point-major f32 | bf16.  One thread per (row, 8-column chunk). -------------------------------
template <typename TF>
__global__ void __launch_bounds__(256) group_rows_kernel(const float *xyz, const float *centre, const TF *feat, const int *idx, int N,
                                                        int C, int np, int ns, int Cp, long long rows, __nv_bfloat16 *X) {
  const int chunks = Cp >> 3;
  const long long total = rows * chunks;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const long long r = t / chunks;
    const int c0 = (int)(t % chunks) * 8;
    const long long bj = r / ns;                   // (b, centre)
    const int b = (int)(bj / np);
    const int k = idx != nullptr ? idx[r] : (int)(r % ((long long)np * ns));   // GroupAll: every point in order
    const float *p = xyz + ((size_t)b * N + k) * 3;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c0 + e;
      float x = 0.f;
      if (c < 3) x = p[c] - (centre != nullptr ? centre[(size_t)bj * 3 + c] : 0.f);
      else if (c < 3 + C) x = (float)feat[((size_t)b * N + k) * C + (c - 3)];
      v[e] = x;
    }
    *reinterpret_cast<uint4 *>(X + (size_t)r * Cp + c0) = pack8(v);
  }
}
// gradient w.r.t. feat: dfeat[b, idx][c] += dX[r][3 + c] (fp32 atomics; xyz carries no gradient)
__global__ void __launch_bounds__(256) group_rows_grad_kernel(const __nv_bfloat16 *dX, const int *idx, int N, int C, int np, int ns,
                                                             int Cp, long long rows, float *dfeat) {
  const long long total = rows * C;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const long long r = t / C;
    const int c = (int)(t % C);
    const int b = (int)(r / ((long long)np * ns));
    const int k = idx != nullptr ? idx[r] : (int)(r % ((long long)np * ns));
    atomicAdd(dfeat + ((size_t)b * N + k) * C + c, __bfloat162float(dX[(size_t)r * Cp + 3 + c]));
  }
}

// ---- column statistics: thread (tx, ty) owns 8 columns and a stripe of rows; MODE 0: sum y, sum y^2;
// MODE 1 (BN + ReLU backward): sum g', sum g' * xhat with g' = dout where the forward output was positive ----------------------------
constexpr int TX = 32, TY = 8, MAX_SLABS = 128;

template <int MODE>
__device__ __forceinline__ void col_sums_block(const __nv_bfloat16 *__restrict__ y, const __nv_bfloat16 *__restrict__ dout,
                                               const float *__restrict__ mean, const float *__restrict__ rstd,
                                               const float *__restrict__ gamma, const float *__restrict__ beta, long long R, int C,
                                               float *__restrict__ partials) {
  __shared__ float acc[2][TY][TX * 8 + 8];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int col = (blockIdx.x * TX + tx) * 8;
  const long long per = (R + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * per, r1 = r0 + per < R ? r0 + per : R;
  float s0[8], s1[8], mu[8], rs[8], ga[8], be[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s0[i] = s1[i] = 0.f;
  if (col < C) {
    if (MODE == 1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mu[i] = mean[col + i]; rs[i] = rstd[col + i]; ga[i] = gamma[col + i]; be[i] = beta[col + i];
      }
    }
    for (long long r = r0 + ty; r < r1; r += TY) {
      float v[8];
      unpack8(__ldg(reinterpret_cast<const uint4 *>(y + (size_t)r * C + col)), v);
      if (MODE == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s0[i] += v[i];
          s1[i] = fmaf(v[i], v[i], s1[i]);
        }
      } else {
        float g[8];
        unpack8(__ldg(reinterpret_cast<const uint4 *>(dout + (size_t)r * C + col)), g);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = (v[i] - mu[i]) * rs[i];
          const float gg = fmaf(xh, ga[i], be[i]) > 0.f ? g[i] : 0.f;
          s0[i] += gg;
          s1[i] = fmaf(gg, xh, s1[i]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[0][ty][tx * 8 + i] = s0[i];
    acc[1][ty][tx * 8 + i] = s1[i];
  }
  __syncthreads();
  const int t = ty * TX + tx;
  const int c = blockIdx.x * TX * 8 + t;
  if (c < C) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int r = 0; r < TY; ++r) {
      a += acc[0][r][t];
      b += acc[1][r][t];
    }
    partials[((size_t)blockIdx.y * 2) * C + c] = a;
    partials[((size_t)blockIdx.y * 2 + 1) * C + c] = b;
  }
}
template <int MODE>
__global__ void __launch_bounds__(TX * TY) col_sums_kernel(const __nv_bfloat16 *__restrict__ y, const __nv_bfloat16 *__restrict__ dout,
                                                          const float *__restrict__ mean, const float *__restrict__ rstd,
                                                          const float *__restrict__ gamma, const float *__restrict__ beta, long long R,
                                                          int C, float *__restrict__ partials) {
  col_sums_block<MODE>(y, dout, mean, rstd, gamma, beta, R, C, partials);
}

// ---- cross-rank column statistics (SyncBatchNorm).  Exchange buffer of every rank, allocated for `cap` >= C channels:
// [2 parities][world][2*cap+1] doubles (slot of rank r: [sum0 (C) | sum1 (C) | R]) followed by `world` uint32 flags (flag[r] =
// the last epoch rank r published into this buffer).  push: col_sums as above, then the last CTA reduces the slab partials to
// fp64 and stores them into this rank's slot of EVERY rank's buffer, then raises its flag on every rank.  finish (a separate
// launch): waits for every rank's flag, sums the slots in rank order 0..world-1 (so every rank computes bit-identical
// statistics) and stores the epoch back.  The epoch is device-resident (*epoch_dev + 1) so a captured graph can replay the
// pair.  Parity double-buffering is safe because a rank only pushes exchange e + 2 after its finish of e + 1 saw every peer's
// flag e + 1, and a peer raises that flag only after its own finish of e has read its buffer (one stream per rank).
struct SyncArgs {
  double *const *peer_bufs;   // [world] device pointers
  int cap, world, rank;
};
__device__ __forceinline__ size_t sync_slot(int cap, int world, unsigned parity, int r) {
  return ((size_t)parity * world + r) * (size_t)(2 * cap + 1);
}
__device__ __forceinline__ volatile unsigned *sync_flags(double *buf, int cap, int world) {
  return reinterpret_cast<volatile unsigned *>(buf + (size_t)2 * world * (2 * cap + 1));
}

template <int MODE>
__global__ void __launch_bounds__(TX * TY) col_sums_push_kernel(const __nv_bfloat16 *__restrict__ y, const __nv_bfloat16 *__restrict__ dout,
                                                               const float *__restrict__ mean, const float *__restrict__ rstd,
                                                               const float *__restrict__ gamma, const float *__restrict__ beta,
                                                               long long R, int C, float *__restrict__ partials, const SyncArgs s,
                                                               unsigned *done_counter, const unsigned *epoch_dev) {
  __shared__ unsigned is_last;
  col_sums_block<MODE>(y, dout, mean, rstd, gamma, beta, R, C, partials);
  __threadfence();
  __syncthreads();
  const int t = threadIdx.y * TX + threadIdx.x;
  if (t == 0) is_last = (atomicAdd(done_counter, 1u) == gridDim.x * gridDim.y - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const unsigned epoch = *reinterpret_cast<const volatile unsigned *>(epoch_dev) + 1u;
  const size_t slot = sync_slot(s.cap, s.world, epoch & 1u, s.rank);
  for (int c = t; c < C; c += TX * TY) {
    double a = 0.0, b = 0.0;    // the slab order of col_sums_final_kernel: world 1 reproduces the single-GPU statistics bitwise
    for (int sl = 0; sl < (int)gridDim.y; ++sl) {
      a += __ldcg(partials + ((size_t)sl * 2) * C + c);
      b += __ldcg(partials + ((size_t)sl * 2 + 1) * C + c);
    }
    for (int p = 0; p < s.world; ++p) {
      double *dst = s.peer_bufs[p] + slot;
      dst[c] = a;
      dst[C + c] = b;
    }
  }
  if (t < s.world) s.peer_bufs[t][slot + 2 * C] = (double)R;
  // every thread's peer stores must be visible system-wide before any flag
  __threadfence_system();
  __syncthreads();
  if (t < s.world) *(sync_flags(s.peer_bufs[t], s.cap, s.world) + s.rank) = epoch;
  if (t == 0) *done_counter = 0u;
}

// One CTA: waits for the epoch's flags, then per channel the rank-ordered fp64 sums (and R_total).  MODE 0: mean, rstd, unbiased
// variance over R_total.  MODE 1: out0 = global sum g', out1 = global sum g' * xhat, out2[0] = 1 / R_total (for the dY kernel);
// loc0 (+)= this rank's sum g' (d beta), loc1 (+)= this rank's sum g' * xhat (d gamma), as torch's SyncBatchNorm leaves the
// parameter gradients local (the data-parallel gradient mean averages them).
template <int MODE>
__global__ void __launch_bounds__(256) sync_finish_kernel(const SyncArgs s, int C, float eps, unsigned *epoch_dev, float *out0, float *out1,
                                                          float *out2, float *loc0, float *loc1, int accumulate) {
  __shared__ unsigned s_epoch;
  double *buf = s.peer_bufs[s.rank];
  if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned *>(epoch_dev) + 1u;
  __syncthreads();
  const unsigned epoch = s_epoch;
  if ((int)threadIdx.x < s.world) {
    volatile unsigned *flag = sync_flags(buf, s.cap, s.world) + threadIdx.x;
    while (*flag < epoch) {
    }
  }
  __threadfence_system();
  __syncthreads();
  const volatile double *slots = buf + sync_slot(s.cap, s.world, epoch & 1u, 0);
  const size_t stride = (size_t)(2 * s.cap + 1);
  double n = 0.0;
  for (int r = 0; r < s.world; ++r) n += slots[r * stride + 2 * C];
  const long long Rt = (long long)n;
  if (MODE == 1 && threadIdx.x == 0) out2[0] = Rt > 0 ? 1.0f / (float)Rt : 0.f;
  for (int c = threadIdx.x; c < C; c += 256) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < s.world; ++r) {
      a += slots[r * stride + c];
      b += slots[r * stride + C + c];
    }
    if (MODE == 0) {
      const double m = Rt > 0 ? a / (double)Rt : 0.0;
      double var = Rt > 0 ? b / (double)Rt - m * m : 0.0;
      if (var < 0.0) var = 0.0;
      out0[c] = (float)m;
      out1[c] = (float)(1.0 / sqrt(var + (double)eps));
      if (out2 != nullptr) out2[c] = (float)(Rt > 1 ? var * (double)Rt / (double)(Rt - 1) : var);
    } else {
      out0[c] = (float)a;
      out1[c] = (float)b;
      const float la = (float)slots[s.rank * stride + c], lb = (float)slots[s.rank * stride + C + c];
      loc0[c] = accumulate ? loc0[c] + la : la;
      loc1[c] = accumulate ? loc1[c] + lb : lb;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *epoch_dev = epoch;
}
// MODE 0: mean, rstd (biased variance, as BatchNorm normalises with) + var_unbiased for the running estimate;
// MODE 1: out0 (+)= dbeta, out1 (+)= dgamma
__global__ void __launch_bounds__(256) col_sums_final_kernel(const float *partials, int slabs, int C, long long R, float eps, int mode,
                                                            int accumulate, float *out0, float *out1, float *out2) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int s = 0; s < slabs; ++s) {
    a += partials[((size_t)s * 2) * C + c];
    b += partials[((size_t)s * 2 + 1) * C + c];
  }
  if (mode == 0) {
    const double m = a / (double)R;
    double var = b / (double)R - m * m;
    if (var < 0.0) var = 0.0;
    out0[c] = (float)m;
    out1[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (out2 != nullptr) out2[c] = (float)(R > 1 ? var * (double)R / (double)(R - 1) : var);
  } else {
    out0[c] = accumulate ? out0[c] + (float)a : (float)a;
    out1[c] = accumulate ? out1[c] + (float)b : (float)b;
  }
}

// out = relu((y - mean) * rstd * gamma + beta), bf16
__global__ void __launch_bounds__(256) bn_relu_apply_kernel(const __nv_bfloat16 *y, const float *mean, const float *rstd,
                                                           const float *gamma, const float *beta, long long R, int C,
                                                           __nv_bfloat16 *out) {
  const int chunks = C >> 3;
  const long long total = R * chunks;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const int c0 = (int)(t % chunks) * 8;
    float v[8];
    unpack8(__ldg(reinterpret_cast<const uint4 *>(y) + t), v);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      v[i] = fmaxf(fmaf((v[i] - mean[c0 + i]) * rstd[c0 + i], gamma[c0 + i], beta[c0 + i]), 0.f);
    reinterpret_cast<uint4 *>(out)[t] = pack8(v);
  }
}
// dY = gamma * rstd * (g' - dbeta / R - xhat * dgamma / R); with SyncBatchNorm dbeta, dgamma are the sums over all ranks and
// 1 / R_total is read from the device (inv_count), since only the finish kernel knows R_total
__global__ void __launch_bounds__(256) bn_relu_bwd_apply_kernel(const __nv_bfloat16 *y, const __nv_bfloat16 *dout, const float *mean,
                                                               const float *rstd, const float *gamma, const float *beta,
                                                               const float *dbeta, const float *dgamma, const float *inv_count,
                                                               long long R, int C, __nv_bfloat16 *dy) {
  const int chunks = C >> 3;
  const long long total = R * chunks;
  const float invR = inv_count != nullptr ? *inv_count : 1.0f / (float)R;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const int c0 = (int)(t % chunks) * 8;
    float v[8], g[8];
    unpack8(__ldg(reinterpret_cast<const uint4 *>(y) + t), v);
    unpack8(__ldg(reinterpret_cast<const uint4 *>(dout) + t), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c0 + i;
      const float xh = (v[i] - mean[c]) * rstd[c];
      const float gg = fmaf(xh, gamma[c], beta[c]) > 0.f ? g[i] : 0.f;
      v[i] = gamma[c] * rstd[c] * (gg - dbeta[c] * invR - xh * dgamma[c] * invR);
    }
    reinterpret_cast<uint4 *>(dy)[t] = pack8(v);
  }
}

// max over `ns` consecutive rows (the neighbourhood): out[g][c] = max_s x[g * ns + s][c], arg = first maximal s (int8)
__global__ void __launch_bounds__(256) rowgroup_max_kernel(const __nv_bfloat16 *x, long long G, int ns, int C, __nv_bfloat16 *out,
                                                          unsigned char *arg) {
  const int chunks = C >> 3;
  const long long total = G * chunks;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const long long gi = t / chunks;
    const int c0 = (int)(t % chunks) * 8;
    float m[8];
    unsigned char a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { m[i] = -INFINITY; a[i] = 0; }
    for (int s = 0; s < ns; ++s) {
      float v[8];
      unpack8(__ldg(reinterpret_cast<const uint4 *>(x + ((size_t)gi * ns + s) * C + c0)), v);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (v[i] > m[i]) { m[i] = v[i]; a[i] = (unsigned char)s; }
    }
    *reinterpret_cast<uint4 *>(out + (size_t)gi * C + c0) = pack8(m);
    *reinterpret_cast<uint2 *>(arg + (size_t)gi * C + c0) =
        make_uint2(a[0] | (a[1] << 8) | (a[2] << 16) | ((unsigned)a[3] << 24), a[4] | (a[5] << 8) | (a[6] << 16) | ((unsigned)a[7] << 24));
  }
}
__global__ void __launch_bounds__(256) rowgroup_max_grad_kernel(const __nv_bfloat16 *gout, const unsigned char *arg, long long G, int ns,
                                                               int C, __nv_bfloat16 *gx) {
  const int chunks = C >> 3;
  const long long total = G * ns * chunks;
  for (long long t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (long long)gridDim.x * 256) {
    const long long r = t / chunks;
    const int c0 = (int)(t % chunks) * 8;
    const long long gi = r / ns;
    const int s = (int)(r % ns);
    float g[8];
    unpack8(__ldg(reinterpret_cast<const uint4 *>(gout + (size_t)gi * C + c0)), g);
    const uint2 aa = *reinterpret_cast<const uint2 *>(arg + (size_t)gi * C + c0);
    const unsigned au[2] = {aa.x, aa.y};
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((int)((au[i >> 2] >> ((i & 3) * 8)) & 0xFFu) != s) g[i] = 0.f;
    reinterpret_cast<uint4 *>(gx)[t] = pack8(g);
  }
}

inline int grid_for(long long total) {
  long long g = (total + 255) / 256;
  return (int)(g < 132 * 16 ? (g > 0 ? g : 1) : 132 * 16);
}
bool al16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int sv_pn_group_rows(const float *xyz, const float *centre, const void *feat, int feat_bf16, const int *idx, int B, int N,
                                int C, int np, int ns, int Cp, void *X, void *stream) {
  if (B < 0 || N < 1 || C < 0 || np < 1 || ns < 1 || Cp < 3 + C || (Cp % 8)) return SV_ERR_INVALID_ARG;
  if (B == 0) return SV_OK;
  if (!xyz || (C > 0 && !feat) || !X || !al16(X)) return SV_ERR_INVALID_ARG;
  const long long rows = (long long)B * np * ns;
  cudaStream_t st = (cudaStream_t)stream;
  if (feat_bf16)
    group_rows_kernel<__nv_bfloat16><<<grid_for(rows * (Cp / 8)), 256, 0, st>>>(xyz, centre, (const __nv_bfloat16 *)feat, idx, N, C, np, ns,
                                                                                Cp, rows, (__nv_bfloat16 *)X);
  else
    group_rows_kernel<float><<<grid_for(rows * (Cp / 8)), 256, 0, st>>>(xyz, centre, (const float *)feat, idx, N, C, np, ns, Cp, rows,
                                                                        (__nv_bfloat16 *)X);
  return sv::after_launch();
}

extern "C" int sv_pn_group_rows_grad(const void *dX, const int *idx, int B, int N, int C, int np, int ns, int Cp, float *dfeat,
                                     void *stream) {
  if (B < 0 || N < 1 || C < 0 || np < 1 || ns < 1 || Cp < 3 + C || (Cp % 8)) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if ((long long)B * N * C > 0) {
    if (!dfeat) return SV_ERR_INVALID_ARG;
    int rc = sv::cuda_status(cudaMemsetAsync(dfeat, 0, (size_t)B * N * C * sizeof(float), st));
    if (rc) return rc;
  }
  if (B == 0 || C == 0) return SV_OK;
  if (!dX) return SV_ERR_INVALID_ARG;
  const long long rows = (long long)B * np * ns;
  group_rows_grad_kernel<<<grid_for(rows * C), 256, 0, st>>>((const __nv_bfloat16 *)dX, idx, N, C, np, ns, Cp, rows, dfeat);
  return sv::after_launch();
}

extern "C" int sv_pn_scratch_floats(int C) { return C > 0 ? MAX_SLABS * 2 * C : 0; }

extern "C" int sv_pn_bn_relu_fwd(const void *y, long long R, int C, const float *gamma, const float *beta, float eps, float *mean,
                                 float *rstd, float *var_unbiased, void *out, float *scratch, void *stream) {
  if (R < 1 || C < 8 || (C % 8)) return SV_ERR_INVALID_ARG;
  if (!y || !gamma || !beta || !mean || !rstd || !out || !scratch || !al16(y) || !al16(out)) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int slabs = (int)((R + 255) / 256 < MAX_SLABS ? (R + 255) / 256 : MAX_SLABS);
  const dim3 grid((unsigned)((C / 8 + TX - 1) / TX), (unsigned)slabs), block(TX, TY);
  col_sums_kernel<0><<<grid, block, 0, st>>>((const __nv_bfloat16 *)y, nullptr, nullptr, nullptr, nullptr, nullptr, R, C, scratch);
  int rc = sv::after_launch();
  if (rc) return rc;
  col_sums_final_kernel<<<(C + 255) / 256, 256, 0, st>>>(scratch, slabs, C, R, eps, 0, 0, mean, rstd, var_unbiased);
  rc = sv::after_launch();
  if (rc) return rc;
  bn_relu_apply_kernel<<<grid_for(R * (C / 8)), 256, 0, st>>>((const __nv_bfloat16 *)y, mean, rstd, gamma, beta, R, C, (__nv_bfloat16 *)out);
  return sv::after_launch();
}

extern "C" int sv_pn_bn_relu_bwd(const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta,
                                 const float *mean, const float *rstd, void *dy, float *dgamma, float *dbeta, int accumulate,
                                 float *scratch, void *stream) {
  if (R < 1 || C < 8 || (C % 8)) return SV_ERR_INVALID_ARG;
  if (!y || !dout || !gamma || !beta || !mean || !rstd || !dy || !dgamma || !dbeta || !scratch || !al16(y) || !al16(dout) || !al16(dy))
    return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int slabs = (int)((R + 255) / 256 < MAX_SLABS - 1 ? (R + 255) / 256 : MAX_SLABS - 1);   // the last slab slot holds this launch's sums
  const dim3 grid((unsigned)((C / 8 + TX - 1) / TX), (unsigned)slabs), block(TX, TY);
  col_sums_kernel<1><<<grid, block, 0, st>>>((const __nv_bfloat16 *)y, (const __nv_bfloat16 *)dout, mean, rstd, gamma, beta, R, C, scratch);
  int rc = sv::after_launch();
  if (rc) return rc;
  // this launch's own sums (the apply kernel needs them un-accumulated): scratch tail [2][C]
  float *own = scratch + (size_t)MAX_SLABS * 2 * C - 2 * C;
  col_sums_final_kernel<<<(C + 255) / 256, 256, 0, st>>>(scratch, slabs, C, R, 0.f, 1, 0, own, own + C, nullptr);
  rc = sv::after_launch();
  if (rc) return rc;
  bn_relu_bwd_apply_kernel<<<grid_for(R * (C / 8)), 256, 0, st>>>((const __nv_bfloat16 *)y, (const __nv_bfloat16 *)dout, mean, rstd, gamma,
                                                                  beta, own, own + C, nullptr, R, C, (__nv_bfloat16 *)dy);
  rc = sv::after_launch();
  if (rc) return rc;
  col_sums_final_kernel<<<(C + 255) / 256, 256, 0, st>>>(scratch, slabs, C, R, 0.f, 1, accumulate, dbeta, dgamma, nullptr);
  return sv::after_launch();
}

namespace {
constexpr int SYNC_MAX_WORLD = 64;
bool al8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
bool sync_args_ok(int C, int cap, int world, int rank, void *const *peer_bufs, const unsigned *epoch_dev) {
  return C >= 8 && C % 8 == 0 && C <= cap && world >= 1 && world <= SYNC_MAX_WORLD && rank >= 0 && rank < world && peer_bufs &&
         al8(peer_bufs) && epoch_dev && (reinterpret_cast<uintptr_t>(epoch_dev) & 3) == 0;
}
}  // namespace

extern "C" int sv_pn_sync_floats(int C, int world) {
  if (C < 8 || C % 8 || world < 1 || world > SYNC_MAX_WORLD) return 0;
  return 2 * 2 * world * (2 * C + 1) + (world + 1) / 2 * 2;   // doubles as float pairs, then the flags (8-byte multiple)
}

extern "C" int sv_pn_bn_sync_push(int mode, const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta,
                                  const float *mean, const float *rstd, float *scratch, void *const *peer_bufs, int cap,
                                  unsigned *done_counter, int world, int rank, const unsigned *epoch_dev, void *stream) {
  if ((mode != 0 && mode != 1) || R < 0 || !sync_args_ok(C, cap, world, rank, peer_bufs, epoch_dev)) return SV_ERR_INVALID_ARG;
  if (!scratch || !done_counter || (reinterpret_cast<uintptr_t>(done_counter) & 3)) return SV_ERR_INVALID_ARG;
  if (R > 0 && (!y || !al16(y))) return SV_ERR_INVALID_ARG;
  if (mode == 1 && (!gamma || !beta || !mean || !rstd || (R > 0 && (!dout || !al16(dout))))) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long cap_slabs = mode == 0 ? MAX_SLABS : MAX_SLABS - 1;    // the slab counts of sv_pn_bn_relu_fwd / _bwd
  long long slabs = (R + 255) / 256 < cap_slabs ? (R + 255) / 256 : cap_slabs;
  if (slabs < 1) slabs = 1;                                              // an empty shard still pushes zeros
  const dim3 grid((unsigned)((C / 8 + TX - 1) / TX), (unsigned)slabs), block(TX, TY);
  const SyncArgs s{(double *const *)peer_bufs, cap, world, rank};
  if (mode == 0)
    col_sums_push_kernel<0><<<grid, block, 0, st>>>((const __nv_bfloat16 *)y, nullptr, nullptr, nullptr, nullptr, nullptr, R, C, scratch, s,
                                                    done_counter, epoch_dev);
  else
    col_sums_push_kernel<1><<<grid, block, 0, st>>>((const __nv_bfloat16 *)y, (const __nv_bfloat16 *)dout, mean, rstd, gamma, beta, R, C,
                                                    scratch, s, done_counter, epoch_dev);
  return sv::after_launch();
}

extern "C" int sv_pn_bn_sync_finish_fwd(const void *y, long long R, int C, const float *gamma, const float *beta, float eps, float *mean,
                                        float *rstd, float *var_unbiased, void *out, void *const *peer_bufs, int cap, int world, int rank,
                                        unsigned *epoch_dev, void *stream) {
  if (R < 0 || !sync_args_ok(C, cap, world, rank, peer_bufs, epoch_dev)) return SV_ERR_INVALID_ARG;
  if (!gamma || !beta || !mean || !rstd || (R > 0 && (!y || !out || !al16(y) || !al16(out)))) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const SyncArgs s{(double *const *)peer_bufs, cap, world, rank};
  sync_finish_kernel<0><<<1, 256, 0, st>>>(s, C, eps, epoch_dev, mean, rstd, var_unbiased, nullptr, nullptr, 0);
  int rc = sv::after_launch();
  if (rc || R == 0) return rc;
  bn_relu_apply_kernel<<<grid_for(R * (C / 8)), 256, 0, st>>>((const __nv_bfloat16 *)y, mean, rstd, gamma, beta, R, C, (__nv_bfloat16 *)out);
  return sv::after_launch();
}

extern "C" int sv_pn_bn_sync_finish_bwd(const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta,
                                        const float *mean, const float *rstd, void *dy, float *dgamma, float *dbeta, int accumulate,
                                        float *gsum, void *const *peer_bufs, int cap, int world, int rank, unsigned *epoch_dev,
                                        void *stream) {
  if (R < 0 || !sync_args_ok(C, cap, world, rank, peer_bufs, epoch_dev)) return SV_ERR_INVALID_ARG;
  if (!gamma || !beta || !mean || !rstd || !dgamma || !dbeta || !gsum) return SV_ERR_INVALID_ARG;
  if (R > 0 && (!y || !dout || !dy || !al16(y) || !al16(dout) || !al16(dy))) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const SyncArgs s{(double *const *)peer_bufs, cap, world, rank};
  sync_finish_kernel<1><<<1, 256, 0, st>>>(s, C, 0.f, epoch_dev, gsum, gsum + C, gsum + 2 * C, dbeta, dgamma, accumulate);
  int rc = sv::after_launch();
  if (rc || R == 0) return rc;
  bn_relu_bwd_apply_kernel<<<grid_for(R * (C / 8)), 256, 0, st>>>((const __nv_bfloat16 *)y, (const __nv_bfloat16 *)dout, mean, rstd, gamma,
                                                                  beta, gsum, gsum + C, gsum + 2 * C, R, C, (__nv_bfloat16 *)dy);
  return sv::after_launch();
}

extern "C" int sv_pn_rowgroup_max(const void *x,long long G, int ns, int C, void *out, unsigned char *arg, void *stream) {
  if (G < 0 || ns < 1 || ns > 255 || C < 8 || (C % 8)) return SV_ERR_INVALID_ARG;
  if (G == 0) return SV_OK;
  if (!x || !out || !arg || !al16(x) || !al16(out) || (reinterpret_cast<uintptr_t>(arg) & 7)) return SV_ERR_INVALID_ARG;
  rowgroup_max_kernel<<<grid_for(G * (C / 8)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)x, G, ns, C, (__nv_bfloat16 *)out, arg);
  return sv::after_launch();
}

extern "C" int sv_pn_rowgroup_max_grad(const void *gout, const unsigned char *arg, long long G, int ns, int C, void *gx, void *stream) {
  if (G < 0 || ns < 1 || ns > 255 || C < 8 || (C % 8)) return SV_ERR_INVALID_ARG;
  if (G == 0) return SV_OK;
  if (!gout || !arg || !gx || !al16(gout) || !al16(gx)) return SV_ERR_INVALID_ARG;
  rowgroup_max_grad_kernel<<<grid_for(G * ns * (C / 8)), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)gout, arg, G, ns, C,
                                                                                         (__nv_bfloat16 *)gx);
  return sv::after_launch();
}
