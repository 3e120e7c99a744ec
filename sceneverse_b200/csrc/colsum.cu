// Column sums of a row-major (R, N) matrix — the bias gradient of every linear layer (db = sum over tokens of dL/dy).
// The reference gets it from ATen's generic strided reduction inside AddmmBackward (~100 launches, 2 ms per step);
// here: thread (tx, ty) owns 8 consecutive columns and walks the rows of its slab, fully coalesced 16-byte loads, fp32
// accumulation, per-slab partials finished by a second tiny kernel in a fixed order (deterministic, no atomics).
// HBM-bound: algorithmic bytes = R * N * sizeof(T).
// The batched entry runs the same two passes over B matrices batch_stride elements apart (blockIdx.z = matrix) and writes
// each matrix's sums in the input's dtype: the backward of ops.scene_broadcast, a fixed-order sum over the U utterance
// copies of every scene's object features.  Algorithmic bytes = B * R * N * sizeof(T) read + B * N * sizeof(T) written.
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"

namespace {

template <typename T>
__device__ __forceinline__ void load8(const T *p, float (&v)[8]);
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16 *p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4 *>(p));
  const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
template <>
__device__ __forceinline__ void load8<float>(const float *p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4 *>(p)), b = __ldg(reinterpret_cast<const float4 *>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

constexpr int TX = 32, TY = 8;  // 32 chunk columns (256 matrix columns) x 8 row lanes per CTA

template <typename T>
__global__ void __launch_bounds__(TX * TY) colsum_partial_kernel(const T *__restrict__ x, long long row_stride, long long batch_stride,
                                                                 int R, int N, float *__restrict__ partials) {
  __shared__ float acc[TY][TX * 8 + 8];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int col = (blockIdx.x * TX + tx) * 8;
  const int rows_per_slab = (R + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per_slab, r1 = min(R, r0 + rows_per_slab);
  x += (size_t)blockIdx.z * batch_stride;
  partials += (size_t)blockIdx.z * gridDim.y * N;
  float s[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = 0.f;
  if (col < N) {
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += TY) {
      float v[8];
      load8<T>(x + (size_t)r * row_stride + col, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[ty][tx * 8 + i] = s[i];
  __syncthreads();
  const int t = ty * TX + tx;  // 256 threads <-> 256 columns of this CTA
  const int c = blockIdx.x * TX * 8 + t;
  if (c < N) {
    float v = 0.f;
#pragma unroll
    for (int r = 0; r < TY; ++r) v += acc[r][t];
    partials[(size_t)blockIdx.y * N + c] = v;
  }
}

__device__ __forceinline__ void store1(float *p, float v) { *p = v; }
__device__ __forceinline__ void store1(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }

// blockIdx.y = matrix: its `slabs` partial rows summed in slab order, rounded once to OutT
template <typename OutT>
__global__ void __launch_bounds__(256) colsum_final_kernel(const float *__restrict__ partials, int slabs, int N,
                                                           OutT *__restrict__ out) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= N) return;
  partials += (size_t)blockIdx.y * slabs * N;
  float v = 0.f;
  for (int s = 0; s < slabs; ++s) v += partials[(size_t)s * N + c];
  store1(out + (size_t)blockIdx.y * N + c, v);
}

constexpr int MAX_SLABS = 64;

int slabs_of(int R) { return R > 64 * MAX_SLABS ? MAX_SLABS : (R + 63) / 64; }

}  // namespace

extern "C" int sv_colsum_scratch_floats(int N) { return N > 0 ? MAX_SLABS * N : 0; }

extern "C" long long sv_colsum_batched_scratch_floats(int B, int R, int N) {
  return (B > 0 && R > 0 && N > 0) ? (long long)B * slabs_of(R) * N : 0;
}

extern "C" int sv_colsum(const void *x, long long row_stride, int is_bf16, int R, int N, float *out, float *scratch,
                         void *stream) {
  if (R < 0 || N < 8 || (N % 8) || (row_stride % 8) || row_stride < N) return SV_ERR_INVALID_ARG;
  if (!x || !out || !scratch || (reinterpret_cast<uintptr_t>(x) & 15)) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (R == 0) return sv::cuda_status(cudaMemsetAsync(out, 0, (size_t)N * sizeof(float), st));
  const int slabs = slabs_of(R);
  const dim3 grid((unsigned)((N / 8 + TX - 1) / TX), (unsigned)slabs), block(TX, TY);
  if (is_bf16) colsum_partial_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16 *)x, row_stride, 0, R, N, scratch);
  else colsum_partial_kernel<float><<<grid, block, 0, st>>>((const float *)x, row_stride, 0, R, N, scratch);
  int rc = sv::after_launch();
  if (rc) return rc;
  colsum_final_kernel<float><<<(N + 255) / 256, 256, 0, st>>>(scratch, slabs, N, out);
  return sv::after_launch();
}

extern "C" int sv_colsum_batched(const void *x, long long row_stride, long long batch_stride, int is_bf16, int B, int R,
                                 int N, void *out, float *scratch, void *stream) {
  if (B < 0 || B > 65535 || R < 0 || N < 8 || (N % 8) || (row_stride % 8) || row_stride < N || (batch_stride % 8) ||
      batch_stride < 0)
    return SV_ERR_INVALID_ARG;
  if (B == 0) return 0;
  if (!out) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t elem = is_bf16 ? sizeof(__nv_bfloat16) : sizeof(float);
  if (R == 0) return sv::cuda_status(cudaMemsetAsync(out, 0, (size_t)B * N * elem, st));
  if (!x || !scratch || (reinterpret_cast<uintptr_t>(x) & 15)) return SV_ERR_INVALID_ARG;
  const int slabs = slabs_of(R);
  const dim3 grid((unsigned)((N / 8 + TX - 1) / TX), (unsigned)slabs, (unsigned)B), block(TX, TY);
  const dim3 fgrid((unsigned)((N + 255) / 256), (unsigned)B);
  if (is_bf16) {
    colsum_partial_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16 *)x, row_stride, batch_stride, R, N,
                                                                 scratch);
    int rc = sv::after_launch();
    if (rc) return rc;
    colsum_final_kernel<__nv_bfloat16><<<fgrid, 256, 0, st>>>(scratch, slabs, N, (__nv_bfloat16 *)out);
  } else {
    colsum_partial_kernel<float><<<grid, block, 0, st>>>((const float *)x, row_stride, batch_stride, R, N, scratch);
    int rc = sv::after_launch();
    if (rc) return rc;
    colsum_final_kernel<float><<<fgrid, 256, 0, st>>>(scratch, slabs, N, (float *)out);
  }
  return sv::after_launch();
}
