// Question-answering head kernels of the ScanQA / SQA3D fine-tune (reference: modules/heads/qa_head.py:42-90 `AttFlat`,
// `QAHeadV1`; optim/loss/loss.py:50-53 `answer_loss`; optim/loss/contra_loss.py:33-34, the masked-BCE form of
// `TextObjWithinBatch` for task ScanQA).
//
// * bce_fwd_bwd_kernel: binary cross-entropy with logits, loss and gradient in one launch, one CTA per row.  The logits are
//   read in place from padded-vocabulary rows, the int64 multi-hot labels are read as they come from the dataset (the
//   reference's `.float()` costs nothing here) and the optional bool weight is the object mask.  The last CTA to finish adds
//   the per-row losses in a fixed order, so the loss is bitwise reproducible.
// * attn_pool_fwd_kernel / attn_pool_bwd_kernel: the masked soft-attention pooling of AttFlat for one glimpse, one CTA per
//   batch row: the score column of the N = 1 linear (padded rows), masked to exactly -1e9 as in the reference, fp32
//   softmax over the tokens and the weighted sum of the token features with fp32 accumulation.
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float ld(const float *p, long long i) { return p[i]; }
__device__ __forceinline__ float ld(const __nv_bfloat16 *p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void st(float *p, long long i, float v) { p[i] = v; }
__device__ __forceinline__ void st(__nv_bfloat16 *p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }

// sum over the CTA in a fixed order (warp butterfly, then the 8 warp sums in warp order): the same bits on every run
__device__ __forceinline__ float block_sum(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) r += red[w];
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bce_fwd_bwd_kernel(const T *__restrict__ logits, long long row_stride,
                                                               const long long *__restrict__ labels,
                                                               const unsigned char *__restrict__ weight, int R, int C,
                                                               float scale, float *__restrict__ loss_rows,
                                                               float *__restrict__ loss_out, unsigned *__restrict__ counter,
                                                               T *__restrict__ grad, long long grad_stride) {
  __shared__ float red[kThreads / 32];
  __shared__ bool last;
  const long long r = blockIdx.x;
  const T *x = logits + r * row_stride;
  const long long *y = labels + r * (long long)C;
  const unsigned char *w = weight ? weight + r * (long long)C : nullptr;
  T *g = grad ? grad + r * grad_stride : nullptr;
  float acc = 0.f;
  for (int j = threadIdx.x; j < C; j += kThreads) {
    const float v = ld(x, j);
    const float t = (float)y[j];
    const float wt = w ? (w[j] ? 1.f : 0.f) : 1.f;
    const float e = expf(-fabsf(v));                     // in (0, 1]: no overflow for any |v|
    acc += wt * (fmaxf(v, 0.f) - v * t + log1pf(e));     // torch's stable form of BCE-with-logits
    if (g) {
      const float sig = v >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
      st(g, j, wt * (sig - t));
    }
  }
  if (g)  // pad columns of a padded-vocabulary row are zero in the gradient
    for (long long j = C + threadIdx.x; j < grad_stride; j += kThreads) st(g, j, 0.f);
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) {
    loss_rows[r] = acc;
    __threadfence();
    last = atomicAdd(counter, 1u) == (unsigned)(R - 1);
  }
  __syncthreads();
  if (!last) return;
  // last CTA: every row's loss is visible (fence before the counter); add them in row order per thread, then the fixed
  // block reduction — the result does not depend on which CTA came last
  __threadfence();
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += kThreads) s += __ldcg(loss_rows + i);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    *loss_out = s * scale;
    *counter = 0u;  // ready for the next call (and the next replay of a captured graph)
  }
}

__device__ __forceinline__ void bf16x8_to_f32(const uint4 &u, float *f) {
  const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ uint4 f32_to_bf16x8(const float *f) {
  uint4 u;
  __nv_bfloat162 *h = reinterpret_cast<__nv_bfloat162 *>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// p (B, L) = softmax over l of (mask[b,l] ? -1e9 : score[b*L+l][0]); pooled (B, D) = sum_l p_l x[b,l,:]
__global__ void __launch_bounds__(kThreads) attn_pool_fwd_kernel(const __nv_bfloat16 *__restrict__ score, int score_rs,
                                                                 const __nv_bfloat16 *__restrict__ x, long long x_bs,
                                                                 int x_rs, const unsigned char *__restrict__ mask, int L,
                                                                 int D, float *__restrict__ p,
                                                                 __nv_bfloat16 *__restrict__ pooled) {
  extern __shared__ float sp[];  // L floats: the attention weights of this row
  __shared__ float red[kThreads / 32];
  const int b = blockIdx.x;
  float m = -INFINITY;
  for (int l = threadIdx.x; l < L; l += kThreads) {
    const long long i = (long long)b * L + l;
    const float s = (mask && mask[i]) ? -1e9f : __bfloat162float(score[i * score_rs]);
    sp[l] = s;
    m = fmaxf(m, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) m = fmaxf(m, red[w]);
  float z = 0.f;
  for (int l = threadIdx.x; l < L; l += kThreads) {
    const float e = expf(sp[l] - m);
    sp[l] = e;
    z += e;
  }
  z = block_sum(z, red);  // also orders the sp[] writes before the reads below
  const float inv = 1.f / z;
  for (int l = threadIdx.x; l < L; l += kThreads) {
    const float pl = sp[l] * inv;
    sp[l] = pl;
    p[(long long)b * L + l] = pl;
  }
  __syncthreads();
  const __nv_bfloat16 *xb = x + (long long)b * x_bs;
  for (int v = threadIdx.x; v < D / 8; v += kThreads) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int l = 0; l < L; ++l) {
      float f[8];
      bf16x8_to_f32(*reinterpret_cast<const uint4 *>(xb + (long long)l * x_rs + 8 * v), f);
      const float pl = sp[l];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = fmaf(pl, f[k], acc[k]);
    }
    *reinterpret_cast<uint4 *>(pooled + (long long)b * D + 8 * v) = f32_to_bf16x8(acc);
  }
}

// dx[b,l,:] = p_l dpooled[b,:];  dscore[b*L+l][0] = p_l (<dpooled, x_l> - sum_l' p_l' <dpooled, x_l'>), 0 where masked;
// dscore columns 1..score_rs-1 = 0 (the padded layout the N = 1 linear's backward reads)
__global__ void __launch_bounds__(kThreads) attn_pool_bwd_kernel(const __nv_bfloat16 *__restrict__ dpooled, int dp_rs,
                                                                 const float *__restrict__ p,
                                                                 const __nv_bfloat16 *__restrict__ x, long long x_bs,
                                                                 int x_rs, const unsigned char *__restrict__ mask, int L,
                                                                 int D, __nv_bfloat16 *__restrict__ dx,
                                                                 __nv_bfloat16 *__restrict__ dscore, int score_rs) {
  extern __shared__ float sdot[];  // L floats: <dpooled, x_l>
  __shared__ float red[kThreads / 32];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __nv_bfloat16 *xb = x + (long long)b * x_bs;
  const __nv_bfloat16 *g = dpooled + (long long)b * dp_rs;
  const float *pb = p + (long long)b * L;
  for (int l = warp; l < L; l += kThreads / 32) {
    float d = 0.f;
    for (int v = lane; v < D / 8; v += 32) {
      float fx[8], fg[8];
      bf16x8_to_f32(*reinterpret_cast<const uint4 *>(xb + (long long)l * x_rs + 8 * v), fx);
      bf16x8_to_f32(*reinterpret_cast<const uint4 *>(g + 8 * v), fg);
#pragma unroll
      for (int k = 0; k < 8; ++k) d = fmaf(fx[k], fg[k], d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) sdot[l] = d;
  }
  __syncthreads();
  float c = 0.f;
  for (int l = threadIdx.x; l < L; l += kThreads) c += pb[l] * sdot[l];
  c = block_sum(c, red);
  for (int l = threadIdx.x; l < L; l += kThreads) {
    const long long i = (long long)b * L + l;
    const float ds = (mask && mask[i]) ? 0.f : pb[l] * (sdot[l] - c);
    __nv_bfloat16 *row = dscore + i * score_rs;
    row[0] = __float2bfloat16_rn(ds);
    for (int k = 1; k < score_rs; ++k) row[k] = __float2bfloat16_rn(0.f);
  }
  __nv_bfloat16 *dxb = dx + (long long)b * L * D;
  const int nv = D / 8;
  for (long long t = threadIdx.x; t < (long long)L * nv; t += kThreads) {
    const int l = (int)(t / nv), v = (int)(t % nv);
    float fg[8];
    bf16x8_to_f32(*reinterpret_cast<const uint4 *>(g + 8 * v), fg);
    const float pl = pb[l];
#pragma unroll
    for (int k = 0; k < 8; ++k) fg[k] *= pl;
    *reinterpret_cast<uint4 *>(dxb + (long long)l * D + 8 * v) = f32_to_bf16x8(fg);
  }
}

constexpr int kMaxPoolTokens = 8192;  // the per-row weights live in shared memory (32 KB)

bool aligned16(const void *ptr) { return ((uintptr_t)ptr & 15u) == 0; }

}  // namespace

extern "C" int sv_bce_logits_fwd_bwd(const void *logits, long long row_stride, int is_bf16, const long long *labels,
                                     const unsigned char *weight, int R, int C, float *loss_rows, float *loss_out,
                                     unsigned *counter, void *grad_logits, long long grad_row_stride, void *stream) {
  if (R < 1 || C < 1 || row_stride < C || (grad_logits && grad_row_stride < C)) return SV_ERR_INVALID_ARG;
  if (!logits || !labels || !loss_rows || !loss_out || !counter) return SV_ERR_INVALID_ARG;
  const uintptr_t esz = is_bf16 ? 2 : 4;
  if (((uintptr_t)logits % esz) || (grad_logits && ((uintptr_t)grad_logits % esz)) || ((uintptr_t)labels % 8) ||
      ((uintptr_t)loss_rows % 4) || ((uintptr_t)loss_out % 4) || ((uintptr_t)counter % 4))
    return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const float scale = 1.0f / (float)R;
  if (is_bf16)
    bce_fwd_bwd_kernel<__nv_bfloat16><<<R, kThreads, 0, st>>>((const __nv_bfloat16 *)logits, row_stride, labels, weight, R,
                                                              C, scale, loss_rows, loss_out, counter,
                                                              (__nv_bfloat16 *)grad_logits, grad_row_stride);
  else
    bce_fwd_bwd_kernel<float><<<R, kThreads, 0, st>>>((const float *)logits, row_stride, labels, weight, R, C, scale,
                                                      loss_rows, loss_out, counter, (float *)grad_logits, grad_row_stride);
  return sv::after_launch();
}

static int attn_pool_check(const void *score, int score_rs, const void *x, long long x_bs, int x_rs, int B, int L, int D) {
  if (B < 1 || L < 1 || L > kMaxPoolTokens || D < 8 || D % 8 || score_rs < 1) return SV_ERR_INVALID_ARG;
  if (!score || !x || ((uintptr_t)score % 2) || !aligned16(x)) return SV_ERR_INVALID_ARG;
  if (x_rs < D || x_rs % 8 || x_bs % 8 || x_bs < (long long)(L - 1) * x_rs + D) return SV_ERR_INVALID_ARG;
  return SV_OK;
}

extern "C" int sv_attn_pool_fwd(const void *score, int score_rs, const void *x, long long x_bs, int x_rs,
                                const unsigned char *pad_mask, int B, int L, int D, float *p, void *pooled, void *stream) {
  const int s = attn_pool_check(score, score_rs, x, x_bs, x_rs, B, L, D);
  if (s != SV_OK) return s;
  if (!p || !pooled || ((uintptr_t)p % 4) || !aligned16(pooled)) return SV_ERR_INVALID_ARG;
  attn_pool_fwd_kernel<<<B, kThreads, L * sizeof(float), (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)score, score_rs, (const __nv_bfloat16 *)x, x_bs, x_rs, pad_mask, L, D, p,
      (__nv_bfloat16 *)pooled);
  return sv::after_launch();
}

extern "C" int sv_attn_pool_bwd(const void *dpooled, int dp_rs, const float *p, const void *x, long long x_bs, int x_rs,
                                const unsigned char *pad_mask, int B, int L, int D, void *dx, void *dscore, int score_rs,
                                void *stream) {
  const int s = attn_pool_check(dscore, score_rs, x, x_bs, x_rs, B, L, D);
  if (s != SV_OK) return s;
  if (!dpooled || !p || !dx || !aligned16(dpooled) || dp_rs < D || dp_rs % 8 || ((uintptr_t)p % 4) || !aligned16(dx))
    return SV_ERR_INVALID_ARG;
  attn_pool_bwd_kernel<<<B, kThreads, L * sizeof(float), (cudaStream_t)stream>>>(
      (const __nv_bfloat16 *)dpooled, dp_rs, p, (const __nv_bfloat16 *)x, x_bs, x_rs, pad_mask, L, D,
      (__nv_bfloat16 *)dx, (__nv_bfloat16 *)dscore, score_rs);
  return sv::after_launch();
}
