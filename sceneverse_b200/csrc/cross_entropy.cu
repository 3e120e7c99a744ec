// Fused softmax cross-entropy (forward + gradient in one launch) for wide-vocabulary logits — the masked-LM loss of
// the GPS pre-training step (reference: optim/loss/loss.py:56-61 `lm_cls_loss`: F.cross_entropy over (B,30522,L) with
// ignore_index=-1, and loss.py:8-9 `og3d_loss`).  One CTA per row: rows whose label is `ignore_index` (85 % of the
// masked-LM positions) cost nothing but a zero-fill of their gradient row; the others are read twice from L2
// (max / sum-exp, then gradient) instead of the reference path's fp32 copy + log_softmax + nll + two backward passes
// over the whole (rows x vocab) tensor.  -inf logits (padded objects in og3d) are handled (p = 0).
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"

namespace {

__device__ __forceinline__ float ld(const float *p, long long i) { return p[i]; }
__device__ __forceinline__ float ld(const __nv_bfloat16 *p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void st(float *p, long long i, float v) { p[i] = v; }
__device__ __forceinline__ void st(__nv_bfloat16 *p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }

__device__ __forceinline__ float block_reduce(float v, float *red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

template <typename T>
__global__ void __launch_bounds__(256) ce_fwd_bwd_kernel(const T *__restrict__ logits, long long row_stride,
                                                         const long long *__restrict__ labels, int V,
                                                         long long ignore_index, float *__restrict__ loss_rows,
                                                         T *__restrict__ grad, long long grad_stride) {
  __shared__ float red[8];
  const long long r = blockIdx.x;
  const long long label = labels[r];
  const T *x = logits + r * row_stride;
  T *g = grad ? grad + r * grad_stride : nullptr;
  if (g)  // padding columns of a padded-vocabulary gradient (grad_stride > V) are always zero
    for (int j = V + threadIdx.x; j < grad_stride; j += 256) st(g, j, 0.f);
  if (label == ignore_index || label < 0 || label >= V) {
    if (threadIdx.x == 0) loss_rows[r] = 0.f;
    if (g)
      for (int j = threadIdx.x; j < V; j += 256) st(g, j, 0.f);
    return;
  }
  float m = -INFINITY;
  for (int j = threadIdx.x; j < V; j += 256) m = fmaxf(m, ld(x, j));
  m = block_reduce(m, red, true);
  float s = 0.f;
  for (int j = threadIdx.x; j < V; j += 256) s += __expf(ld(x, j) - m);
  s = block_reduce(s, red, false);
  const float lse = __logf(s) + m;
  if (threadIdx.x == 0) loss_rows[r] = lse - ld(x, label);
  if (g) {
    const float inv = 1.0f / s;
    for (int j = threadIdx.x; j < V; j += 256) st(g, j, __expf(ld(x, j) - m) * inv - (j == label ? 1.f : 0.f));
  }
}

}  // namespace

extern "C" int sv_cross_entropy_fwd_bwd_strided(const void *logits, long long row_stride, int is_bf16,
                                                const long long *labels, int R, int V, long long ignore_index,
                                                float *loss_rows, void *grad_logits, long long grad_row_stride,
                                                void *stream) {
  if (R < 0 || V < 1 || grad_row_stride < V) return SV_ERR_INVALID_ARG;
  if (R == 0) return SV_OK;
  if (!logits || !labels || !loss_rows) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (is_bf16)
    ce_fwd_bwd_kernel<__nv_bfloat16><<<R, 256, 0, st>>>((const __nv_bfloat16 *)logits, row_stride, labels, V,
                                                        ignore_index, loss_rows, (__nv_bfloat16 *)grad_logits, grad_row_stride);
  else
    ce_fwd_bwd_kernel<float><<<R, 256, 0, st>>>((const float *)logits, row_stride, labels, V, ignore_index, loss_rows,
                                                (float *)grad_logits, grad_row_stride);
  return sv::after_launch();
}
