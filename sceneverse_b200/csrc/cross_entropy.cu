// Fused softmax cross-entropy (forward + gradient in one launch) for wide-vocabulary logits — the masked-LM loss of
// the GPS pre-training step (reference: optim/loss/loss.py:56-61 `lm_cls_loss`: F.cross_entropy over (B,30522,L) with
// ignore_index=-1, and loss.py:8-9 `og3d_loss`).  One CTA per row: rows whose label is `ignore_index` (85 % of the
// masked-LM positions) cost nothing but a zero-fill of their gradient row; the others are read twice from L2
// (max / sum-exp, then gradient) instead of the reference path's fp32 copy + log_softmax + nll + two backward passes
// over the whole (rows x vocab) tensor.  -inf logits (padded objects in og3d) are handled (p = 0).
//
// masked_ce_fwd_bwd_kernel: the same row body behind the per-object weight of the object-classification losses
// (loss.py:26-47, 64-94: cross-entropy * obj_masks [* (~)obj_sem_masks], summed, divided by the weight sum).  A row of
// weight 0 is handled like an ignored row; the last CTA to finish adds the row losses and the weights in a fixed order
// and writes the normalised loss, so no host read and no second launch are needed.
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float ld(const float *p, long long i) { return p[i]; }
__device__ __forceinline__ float ld(const __nv_bfloat16 *p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void st(float *p, long long i, float v) { p[i] = v; }
__device__ __forceinline__ void st(__nv_bfloat16 *p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }

// max or sum over the CTA in a fixed order (warp butterfly, then the 8 warp values in warp order)
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
  for (int w = 1; w < kThreads / 32; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// One row, run by the whole CTA (`live` must be the same on every thread): the padding columns [V, grad_stride) of the
// gradient row are zeroed; a row that is not live zeroes its gradient columns [0, V) without reading the logits and
// returns 0; a live row returns logsumexp(x) - x[label] on every thread and writes softmax(x) - onehot(label).
template <typename T>
__device__ __forceinline__ float ce_row(const T *__restrict__ x, long long label, int V, bool live, T *__restrict__ g,
                                        long long grad_stride, float *red) {
  if (g)  // padding columns of a padded-vocabulary gradient (grad_stride > V) are always zero
    for (long long j = V + threadIdx.x; j < grad_stride; j += kThreads) st(g, j, 0.f);
  if (!live) {
    if (g)
      for (int j = threadIdx.x; j < V; j += kThreads) st(g, j, 0.f);
    return 0.f;
  }
  float m = -INFINITY;
  for (int j = threadIdx.x; j < V; j += kThreads) m = fmaxf(m, ld(x, j));
  m = block_reduce(m, red, true);
  float s = 0.f;
  for (int j = threadIdx.x; j < V; j += kThreads) s += __expf(ld(x, j) - m);
  s = block_reduce(s, red, false);
  const float lse = __logf(s) + m;
  if (g) {
    const float inv = 1.0f / s;
    for (int j = threadIdx.x; j < V; j += kThreads) st(g, j, __expf(ld(x, j) - m) * inv - (j == label ? 1.f : 0.f));
  }
  return lse - ld(x, label);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) ce_fwd_bwd_kernel(const T *__restrict__ logits, long long row_stride,
                                                              const long long *__restrict__ labels, int V,
                                                              long long ignore_index, float *__restrict__ loss_rows,
                                                              T *__restrict__ grad, long long grad_stride) {
  __shared__ float red[kThreads / 32];
  const long long r = blockIdx.x;
  const long long label = labels[r];
  const bool live = !(label == ignore_index || label < 0 || label >= V);
  const float loss = ce_row(logits + r * row_stride, label, V, live, grad ? grad + r * grad_stride : nullptr, grad_stride,
                            red);
  if (threadIdx.x == 0) loss_rows[r] = loss;
}

// w_r of the object-classification losses: obj_masks, obj_masks & ~obj_sem_masks, obj_masks & obj_sem_masks
__device__ __forceinline__ bool row_weight(const unsigned char *__restrict__ obj_mask,
                                           const unsigned char *__restrict__ sem_mask, int mode, long long r) {
  if (!obj_mask[r]) return false;
  return mode == 0 ? true : (mode == 1 ? !sem_mask[r] : sem_mask[r] != 0);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) masked_ce_fwd_bwd_kernel(
    const T *__restrict__ logits, long long row_stride, const long long *__restrict__ labels, int V,
    const unsigned char *__restrict__ obj_mask, const unsigned char *__restrict__ sem_mask, int mode, int R,
    float *__restrict__ loss_rows, float *__restrict__ sums, float *__restrict__ loss_out, unsigned *__restrict__ counter,
    T *__restrict__ grad, long long grad_stride) {
  __shared__ float red[kThreads / 32];
  __shared__ bool last;
  const long long r = blockIdx.x;
  const long long label = labels[r];
  // torch's ignore_index = -100 lies outside [0, V): a padded slot, like any out-of-range label, contributes nothing
  const bool live = row_weight(obj_mask, sem_mask, mode, r) && label >= 0 && label < V;
  const float loss = ce_row(logits + r * row_stride, label, V, live, grad ? grad + r * grad_stride : nullptr, grad_stride,
                            red);
  if (threadIdx.x == 0) {
    loss_rows[r] = loss;
    __threadfence();
    last = atomicAdd(counter, 1u) == (unsigned)(R - 1);
  }
  __syncthreads();
  if (!last) return;
  // last CTA: every row's loss is visible (fence before the counter); add the losses and the weights in row order per
  // thread, then the fixed block reduction — the result does not depend on which CTA came last
  __threadfence();
  float s = 0.f, n = 0.f;
  for (int i = threadIdx.x; i < R; i += kThreads) {
    s += __ldcg(loss_rows + i);
    n += row_weight(obj_mask, sem_mask, mode, i) ? 1.f : 0.f;
  }
  s = block_reduce(s, red, false);
  n = block_reduce(n, red, false);
  if (threadIdx.x == 0) {
    sums[0] = s;
    sums[1] = n;
    *loss_out = s / n;  // n = 0: 0 / 0 = NaN, as the reference's division
    *counter = 0u;      // ready for the next call (and the next replay of a captured graph)
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
    ce_fwd_bwd_kernel<__nv_bfloat16><<<R, kThreads, 0, st>>>((const __nv_bfloat16 *)logits, row_stride, labels, V,
                                                             ignore_index, loss_rows, (__nv_bfloat16 *)grad_logits,
                                                             grad_row_stride);
  else
    ce_fwd_bwd_kernel<float><<<R, kThreads, 0, st>>>((const float *)logits, row_stride, labels, V, ignore_index, loss_rows,
                                                     (float *)grad_logits, grad_row_stride);
  return sv::after_launch();
}

extern "C" int sv_masked_cross_entropy_fwd_bwd(const void *logits, long long row_stride, int is_bf16,
                                               const long long *labels, const unsigned char *obj_mask,
                                               const unsigned char *sem_mask, int mode, int R, int V, float *loss_rows,
                                               float *sums, float *loss_out, unsigned *counter, void *grad_logits,
                                               long long grad_row_stride, void *stream) {
  if (R < 1 || V < 1 || row_stride < V || (grad_logits && grad_row_stride < V)) return SV_ERR_INVALID_ARG;
  if (mode < 0 || mode > 2 || (mode != 0 && !sem_mask)) return SV_ERR_INVALID_ARG;
  if (!logits || !labels || !obj_mask || !loss_rows || !sums || !loss_out || !counter) return SV_ERR_INVALID_ARG;
  const uintptr_t esz = is_bf16 ? 2 : 4;
  if (((uintptr_t)logits % esz) || (grad_logits && ((uintptr_t)grad_logits % esz)) || ((uintptr_t)labels % 8) ||
      ((uintptr_t)loss_rows % 4) || ((uintptr_t)sums % 4) || ((uintptr_t)loss_out % 4) || ((uintptr_t)counter % 4))
    return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (is_bf16)
    masked_ce_fwd_bwd_kernel<__nv_bfloat16><<<R, kThreads, 0, st>>>(
        (const __nv_bfloat16 *)logits, row_stride, labels, V, obj_mask, sem_mask, mode, R, loss_rows, sums, loss_out,
        counter, (__nv_bfloat16 *)grad_logits, grad_row_stride);
  else
    masked_ce_fwd_bwd_kernel<float><<<R, kThreads, 0, st>>>((const float *)logits, row_stride, labels, V, obj_mask,
                                                            sem_mask, mode, R, loss_rows, sums, loss_out, counter,
                                                            (float *)grad_logits, grad_row_stride);
  return sv::after_launch();
}
