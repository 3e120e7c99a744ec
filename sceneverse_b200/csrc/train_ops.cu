// Small HBM-bound training-side kernels of the GPS step that have no contraction in them:
//   * act_bwd_kernel       — dL/dpre = dL/dy x act'(.) for a linear + activation that is NOT followed by a second linear
//                            (the FFN form fuses this into the dgrad GEMM epilogue, csrc/gemm.cu);
//   * embedding_bwd_kernel — scatter-add of the token gradients into the embedding table gradient (reference: the autograd
//                            of nn.Embedding inside HF BertEmbeddings, modules/language/bert.py:21-26; ATen runs it as a
//                            radix sort + segmented reduction, 8 kernels);
//   * adamw_flat_kernel    — clip + AdamW + bf16 shadow refresh over the FLAT parameter / gradient buffers in one pass
//                            (reference: trainer/build.py:135-145 clip_grad_norm_ + optimizer.step, optim/utils.py:1-18
//                            parameter groups), with a per-segment table for lr / weight decay.
#include <cuda_bf16.h>

#include "attn_common.cuh"
#include "svcommon.h"
#include "svgps.h"

namespace {

__device__ __forceinline__ void gelu_parts(float x, float &cdf, float &e) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  const float p = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  e = attn::ex2f(-z * z * 1.4426950408889634f);
  const float h = 0.5f * p * e;
  cdf = x >= 0.f ? 1.0f - h : h;
}

// g, aux, out: (M, N) bf16, leading dimensions % 8 == 0, N % 8 == 0; thread = 8 consecutive columns of one row
__global__ void __launch_bounds__(256) act_bwd_kernel(const __nv_bfloat16 *g, int ldg, const __nv_bfloat16 *aux, int lda,
                                                     __nv_bfloat16 *out, int ldo, int M, int N, int mode) {
  const int n8 = N >> 3;
  const long long total = (long long)M * n8;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int r = (int)(i / n8), c = (int)(i % n8) * 8;
    const uint4 gv = *reinterpret_cast<const uint4 *>(g + (size_t)r * ldg + c);
    const uint4 av = *reinterpret_cast<const uint4 *>(aux + (size_t)r * lda + c);
    const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w}, aw[4] = {av.x, av.y, av.z, av.w};
    uint32_t ow[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float g0 = __uint_as_float(gw[k] << 16), g1 = __uint_as_float(gw[k] & 0xFFFF0000u);
      const float a0 = __uint_as_float(aw[k] << 16), a1 = __uint_as_float(aw[k] & 0xFFFF0000u);
      if (mode == 1) {  // relu, aux = forward output
        g0 = a0 > 0.f ? g0 : 0.f;
        g1 = a1 > 0.f ? g1 : 0.f;
      } else {          // gelu(erf), aux = pre-activation
        float c0, e0, c1, e1;
        gelu_parts(a0, c0, e0);
        gelu_parts(a1, c1, e1);
        g0 *= fmaf(a0 * e0, 0.3989422804014327f, c0);
        g1 *= fmaf(a1 * e1, 0.3989422804014327f, c1);
      }
      ow[k] = sm90::pack_bf16(g0, g1);
    }
    *reinterpret_cast<uint4 *>(out + (size_t)r * ldo + c) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  }
}

// one warp per token row: dW[ids[t]][:] += g[t][:]  (fp32 atomics; rows with ids == padding_idx are skipped)
template <typename T>
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const T *g, long long ldg, const long long *ids, float *dw, int ntok,
                                                           int D, long long vocab, long long padding_idx) {
  const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= ntok) return;
  const long long id = ids[warp];
  if (id == padding_idx || id < 0 || id >= vocab) return;
  const T *src = g + (size_t)warp * ldg;
  float *dst = dw + (size_t)id * D;
  for (int c = lane * 4; c < D; c += 128) {
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = c + e < D ? (float)src[c + e] : 0.f;
    if (c + 4 <= D && (reinterpret_cast<uintptr_t>(dst + c) & 15) == 0) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3])
                   : "memory");
    } else {
      for (int e = 0; e < 4 && c + e < D; ++e) atomicAdd(dst + c + e, v[e]);
    }
  }
}

// x *= *scale (device scalar), 8 bf16 / 4 f32 per thread: the in-place 1/count scaling of the cross-entropy gradient
template <typename T>
__global__ void __launch_bounds__(256) scale_inplace_kernel(T *x, long long n16, const float *scale) {
  const float s = __ldg(scale);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n16; i += (long long)gridDim.x * 256) {
    uint4 v = reinterpret_cast<uint4 *>(x)[i];
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (sizeof(T) == 2) {
        w[k] = sm90::pack_bf16(__uint_as_float(w[k] << 16) * s, __uint_as_float(w[k] & 0xFFFF0000u) * s);
      } else {
        w[k] = __float_as_uint(__uint_as_float(w[k]) * s);
      }
    }
    reinterpret_cast<uint4 *>(x)[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

struct AdamSeg {          // one parameter group slice of the flat buffer: [begin, end) in elements (multiples of 4)
  long long begin, end;
  float lr_scale;         // base lr of the group / reference lr (the device lr word holds the schedule factor)
  float weight_decay;
};

// sum of squares of the flat gradient: per-CTA partials (fixed order), reduced by the consumer
__global__ void __launch_bounds__(512) sqnorm_partial_kernel(const float *g, long long n, float *partials) {
  __shared__ float red[16];
  float s = 0.f;
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * 512ll + threadIdx.x; i < n4; i += (long long)gridDim.x * 512) {
    const float4 v = reinterpret_cast<const float4 *>(g)[i];
    s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s))));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = g[(n4 << 2) + threadIdx.x];
    s = fmaf(v, v, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 16 ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
  }
}

struct AdamArgs {
  float *p, *m, *v;
  const float *g;
  __nv_bfloat16 *shadow;          // bf16 copy of p, same layout (may be null)
  const AdamSeg *segs;
  int nseg;
  const float *partials;          // squared-norm partials of g
  int npart;
  float max_norm;                 // <= 0: no clipping
  const float *lr_factor;         // device: schedule factor of this step
  const long long *step;          // device: 1-based step count (bias correction)
  float base_lr, beta1, beta2, eps;
  float *norm_out;                // device: total gradient norm (may be null)
};

// torch.optim.AdamW (decoupled weight decay, bias-corrected, eps outside the sqrt of the corrected second moment):
//   p *= 1 - lr wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)
// with g pre-scaled by the clip_grad_norm_ coefficient min(1, max_norm / (||g|| + 1e-6)).
__global__ void __launch_bounds__(256) adamw_flat_kernel(const AdamArgs a) {
  __shared__ float s_clip, s_bc1, s_bc2s, s_lrf;
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < a.npart; ++i) tot += a.partials[i];   // fixed order: deterministic
    const float nrm = sqrtf(tot);
    // not fminf: it would turn a NaN norm into 1 and apply an unclipped update; clamp(max=1) in clip_grad_norm_ keeps the NaN
    const float c = a.max_norm / (nrm + 1e-6f);
    s_clip = a.max_norm > 0.f ? (c > 1.0f ? 1.0f : c) : 1.0f;
    const double st = (double)*a.step;
    s_bc1 = (float)(1.0 - pow((double)a.beta1, st));
    s_bc2s = (float)sqrt(1.0 - pow((double)a.beta2, st));
    s_lrf = *a.lr_factor;
    if (blockIdx.x == 0 && a.norm_out != nullptr) *a.norm_out = nrm;
  }
  __syncthreads();
  const float clip = s_clip, bc1 = s_bc1, bc2s = s_bc2s;
  for (int sg = blockIdx.y; sg < a.nseg; sg += gridDim.y) {
    const AdamSeg seg = a.segs[sg];
    const float lr = a.base_lr * seg.lr_scale * s_lrf;
    const float decay = 1.0f - lr * seg.weight_decay, step_size = lr / bc1;
    const long long b4 = seg.begin >> 2, e4 = seg.end >> 2;
    for (long long i = b4 + blockIdx.x * 256ll + threadIdx.x; i < e4; i += (long long)gridDim.x * 256) {
      float4 p = reinterpret_cast<float4 *>(a.p)[i], m = reinterpret_cast<float4 *>(a.m)[i], v = reinterpret_cast<float4 *>(a.v)[i];
      const float4 g = reinterpret_cast<const float4 *>(a.g)[i];
      float pp[4] = {p.x, p.y, p.z, p.w}, mm[4] = {m.x, m.y, m.z, m.w}, vv[4] = {v.x, v.y, v.z, v.w};
      const float gg[4] = {g.x * clip, g.y * clip, g.z * clip, g.w * clip};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        pp[e] *= decay;
        mm[e] = fmaf(a.beta1, mm[e], (1.0f - a.beta1) * gg[e]);
        vv[e] = fmaf(a.beta2, vv[e], (1.0f - a.beta2) * gg[e] * gg[e]);
        pp[e] -= step_size * mm[e] / (sqrtf(vv[e]) / bc2s + a.eps);
      }
      reinterpret_cast<float4 *>(a.p)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
      reinterpret_cast<float4 *>(a.m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
      reinterpret_cast<float4 *>(a.v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
      if (a.shadow != nullptr)
        reinterpret_cast<uint2 *>(a.shadow)[i] = make_uint2(sm90::pack_bf16(pp[0], pp[1]), sm90::pack_bf16(pp[2], pp[3]));
    }
  }
}

}  // namespace

extern "C" int sv_act_bwd_bf16(const void *g, int ldg, const void *aux, int ld_aux, int mode, int M, int N, void *out, int ldo,
                               void *stream) {
  if (M < 0 || N < 0 || (N % 8) || (ldg % 8) || (ld_aux % 8) || (ldo % 8) || (mode != 1 && mode != 2)) return SV_ERR_INVALID_ARG;
  if (M == 0 || N == 0) return SV_OK;
  if (!g || !aux || !out) return SV_ERR_INVALID_ARG;
  const long long total = (long long)M * (N / 8);
  const int grid = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);
  act_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)g, ldg, (const __nv_bfloat16 *)aux, ld_aux,
                                                          (__nv_bfloat16 *)out, ldo, M, N, mode);
  return sv::after_launch();
}

extern "C" int sv_embedding_bwd(const void *grad_out, long long ldg, int is_bf16, const long long *ids, int ntok, int D,
                                long long vocab, long long padding_idx, float *dw, void *stream) {
  if (ntok < 0 || D < 1 || vocab < 1) return SV_ERR_INVALID_ARG;
  if (ntok == 0) return SV_OK;
  if (!grad_out || !ids || !dw) return SV_ERR_INVALID_ARG;
  const int grid = (ntok + 7) / 8;
  if (is_bf16)
    embedding_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)grad_out, ldg, ids, dw, ntok,
                                                                                D, vocab, padding_idx);
  else
    embedding_bwd_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float *)grad_out, ldg, ids, dw, ntok, D, vocab,
                                                                        padding_idx);
  return sv::after_launch();
}

extern "C" int sv_scale_inplace(void *x, long long n, int is_bf16, const float *scale, void *stream) {
  if (n < 0 || !scale) return SV_ERR_INVALID_ARG;
  if (n == 0) return SV_OK;
  const long long per = is_bf16 ? 8 : 4;
  if (!x || (n % per) || (reinterpret_cast<uintptr_t>(x) & 15)) return SV_ERR_INVALID_ARG;
  const long long n16 = n / per;
  const int grid = (int)((n16 + 255) / 256 < 132 * 16 ? (n16 + 255) / 256 : 132 * 16);
  if (is_bf16) scale_inplace_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16 *)x, n16, scale);
  else scale_inplace_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((float *)x, n16, scale);
  return sv::after_launch();
}

extern "C" int sv_adamw_scratch_floats(void) { return 1024; }

extern "C" int sv_adamw_flat(float *params, float *exp_avg, float *exp_avg_sq, const float *grads, void *shadow_bf16,
                             long long n, const void *segments, int nseg, float max_norm, const float *lr_factor,
                             const long long *step, float base_lr, float beta1, float beta2, float eps, float *scratch,
                             float *norm_out, void *stream) {
  if (n < 0 || nseg < 0) return SV_ERR_INVALID_ARG;
  if (n == 0 || nseg == 0) return SV_OK;
  if (!params || !exp_avg || !exp_avg_sq || !grads || !segments || !lr_factor || !step || !scratch) return SV_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(params) & 15) || (reinterpret_cast<uintptr_t>(grads) & 15) ||
      (reinterpret_cast<uintptr_t>(exp_avg) & 15) || (reinterpret_cast<uintptr_t>(exp_avg_sq) & 15) ||
      (reinterpret_cast<uintptr_t>(shadow_bf16) & 7) || (reinterpret_cast<uintptr_t>(segments) & 7))
    return SV_ERR_INVALID_ARG;   // the shadow is written as uint2, the segment records are read as 8-byte fields
  cudaStream_t st = (cudaStream_t)stream;
  const int npart = 528;  // 132 SMs (H100 SXM) x 4
  sqnorm_partial_kernel<<<npart, 512, 0, st>>>(grads, n, scratch);
  int rc = sv::after_launch();
  if (rc) return rc;
  AdamArgs a{params, exp_avg, exp_avg_sq, grads, (__nv_bfloat16 *)shadow_bf16, (const AdamSeg *)segments, nseg, scratch, npart,
             max_norm, lr_factor, step, base_lr, beta1, beta2, eps, norm_out};
  dim3 grid(132 * 2, nseg < 8 ? nseg : 8);
  adamw_flat_kernel<<<grid, 256, 0, st>>>(a);
  return sv::after_launch();
}
