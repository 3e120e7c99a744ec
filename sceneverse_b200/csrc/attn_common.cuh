// Shared pieces of the attention forward / backward kernels (csrc/attention.cu, csrc/attention_bwd.cu).
//
// Operand staging: every global operand (Q, K, V, dO head slices: rows x 64 bf16 = 128-byte rows) arrives by TMA
// (cp.async.bulk.tensor.3d over a (columns, rows, scenes) view with box 64 x 16 x 1, CU_TENSOR_MAP_SWIZZLE_128B), so a
// staged tile is always the natural [rows][64] matrix in the 128-byte-swizzle layout; rows past the sequence end are
// zero-filled by the hardware.  The same staged tile serves as
//   * a K-major operand (contraction over the 64 head dims):   sm90::desc_sw128(addr, 16), K step = +32 B;
//   * an MN-major B operand (contraction over the ROWS, N = 64 head dims, e.g. P.V, dS.K): sm90::desc_sw128 read with
//     the wgmma transpose flag, K step of 16 rows = +2048 B — no transposed copy is ever built.
// Thread-written A operands (P, dS, P^T, dS^T) use the canonical no-swizzle K-major layout tile[K/8][64][8]
// (sm90::tile_off, sm90::desc_noswz).
//
// Work unit: one (scene, head, 64-row tile) per CTA of one warpgroup; several CTAs share an SM and run independently, so
// one unit's element-wise stage overlaps another's wgmma chains.  The column dimension is swept in blocks of 64; the
// element-wise work and the backward's output chains of the last block stop at the column count rounded up to 16 (the
// TMA box and the k16 step).  Every output element keeps the chain of k16 steps it had with whole 64-column blocks: the
// skipped steps only ever added products with exact zeros.
//
// Block skipping: a 64-key block in which every key is masked (key-padding mask or past Lk) is never visited — its
// logits are all -inf, so it only ever added P = 0 and dS = 0 products and -inf to the row maximum.  The forward and the
// backward's query-row pass sweep the live key blocks only (the forward loads K / V up to the last live one), and a
// key-row unit of the backward whose 64 keys are all masked writes zero dK / dV rows without loading anything.  The
// visited blocks keep their order and their chains, so every result is bit-for-bit the one of the full sweep, up to the
// sign of a zero.  sv_attention_visit_all_blocks(1) switches skipping off (tests compare both paths).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "sm90.cuh"
#include "svcommon.h"

namespace attn {

using namespace sm90;

constexpr int DH = 64;
constexpr int RESIDENT_MAX = 384;   // keys of the resident forward; Lq and Lk of the sv_attention_*_rows_bf16 entries
constexpr int STREAM_MAX = 2048;     // Lq and Lk of the sv_attention_*_long_bf16 entries: 32 blocks of 64 = one 32-bit mask
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;
constexpr float LOG2_CLAMP = -19.931568569324174f;  // log2(1e-6): the reference clamps sigmoid(.) at 1e-6 before the log

// ---- TMA ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// rows [r0, r0 + 16 * nbox) of head h of scene b -> consecutive 2 KB boxes at dst (the 128-byte swizzle pattern repeats
// every 8 rows, so stacked boxes form one tile); boxes starting past `L` are skipped, rows past `L` inside a box are
// zero-filled.  The caller arms the barrier ONCE per phase with the sum of rows_bytes() of everything it issues on it.
constexpr int BOX_ROWS = 16;
constexpr uint32_t BOX_BYTES = BOX_ROWS * 128;
__device__ __forceinline__ uint32_t rows_bytes(int r0, int nbox, int L) {
  int n = (L - r0 + BOX_ROWS - 1) / BOX_ROWS;
  n = n < 0 ? 0 : (n > nbox ? nbox : n);
  return (uint32_t)n * BOX_BYTES;
}
__device__ __forceinline__ void tma_rows(uint8_t *dst, const CUtensorMap *map, int h, int r0, int nbox, int L, int b,
                                         uint64_t *bar) {
#pragma unroll 1
  for (int i = 0; i < nbox; ++i)
    if (r0 + i * BOX_ROWS < L) tma_load_3d(dst + i * BOX_BYTES, map, h * DH, r0 + i * BOX_ROWS, b, bar);
}

// ---- math -----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2f(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// spatial gate of one (query, key) pair in the log2 domain: log2(clamp(sigmoid(z), 1e-6)), z = b + w . loc.
// `w` holds the six weights pre-multiplied by -log2(e), so t = 2^(w . loc) = exp(-z) and sigmoid = 1 / (1 + t).
struct GateW {
  float b, w0, w1, w2, w3, w4;
  __device__ __forceinline__ void load(const float *p) {
    b = -LOG2E * p[0]; w0 = -LOG2E * p[1]; w1 = -LOG2E * p[2]; w2 = -LOG2E * p[3]; w3 = -LOG2E * p[4]; w4 = -LOG2E * p[5];
  }
  __device__ __forceinline__ float log2gate(float l0, float l1, float l2, float l3, float l4) const {
    const float t = ex2f(fmaf(w4, l4, fmaf(w3, l3, fmaf(w2, l2, fmaf(w1, l1, fmaf(w0, l0, b))))));
    return fmaxf(-lg2f(1.0f + t), LOG2_CLAMP);
  }
};

// ---- wgmma chains of one 64-row unit -----------------------------------------------------------------------------------
// the first n column blocks (1 <= n <= 32): a mask of every block without the undefined shift by 32 at n = 32
__device__ __forceinline__ uint32_t first_blocks(int n) { return 0xffffffffu >> (32 - n); }
// index of the i-th set bit of `live` (the i-th visited column block), -1 past the last
__device__ __forceinline__ int nth_block(uint32_t live, int i) {
  for (; i > 0 && live; --i) live &= live - 1u;
  return live ? __ffs(live) - 1 : -1;
}
// width of column block `blk` of a sweep over `n16` columns (a multiple of 16): 64, the last one 16, 32, 48 or 64
__device__ __forceinline__ int block_cols(int blk, int n16) {
  const int rest = n16 - blk * 64;
  return rest < 64 ? rest : 64;
}
// acc[64 rows x 64] = A[64 rows x 64] . B[64 x 64]^T, both K-major 128-byte-swizzle tiles (contraction over the head dims).
// A last block narrower than 64 is still computed whole: a narrower wgmma form for it makes ptxas serialize the chains,
// and its columns past the block width (products with stale staging rows) are never read.
__device__ __forceinline__ void mma_kk(float (&d)[32], uint32_t aA, uint32_t aB) {
#pragma unroll
  for (int ks = 0; ks < DH / 16; ++ks) wgmma_n64<0, 0>(d, desc_sw128(aA + ks * 32, 16), desc_sw128(aB + ks * 32, 16), ks > 0);
}
// acc[64 rows x 64] (+)= G[64 rows x n] . C[n x 64]: G thread-written in the no-swizzle K-major tile[8][64][8], C a staged
// [n][64] 128-byte-swizzle block read MN-major (contraction over its rows); n / 16 k16 steps
__device__ __forceinline__ void mma_gc(float (&d)[32], uint32_t aG, uint32_t aC, int n, bool accumulate) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    if (ks * 16 < n)
      wgmma_n64<0, 1>(d, desc_noswz(aG + ks * 2048, 1024, 128), desc_sw128(aC + ks * 2048, 8192),
                      (accumulate || ks > 0) ? 1u : 0u);
}

// ---- dropout mask ----------------------------------------------------------------------------------------------------------
// keep(b, h, i, j) is a pure function of (seed, b, h, i, j): one 64-bit mix per (scene, head, query) row gives a 32-bit
// row key; one 32-bit mix per key PAIR gives two 16-bit uniforms; weight j is kept iff its uniform >= round(p * 65536).
// The backward regenerates exactly the forward's mask (the reference draws it inside nn.MultiheadAttention,
// transformers.py:22-24,69-74,118-120).
__host__ __device__ __forceinline__ uint32_t drop_row_key(unsigned long long seed, unsigned long long row) {
  unsigned long long x = seed + row * 0x9E3779B97F4A7C15ull;
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return (uint32_t)x;
}
// seed actually used by a launch: the by-value seed plus the run-time device counter (fresh masks on every replay of a
// captured CUDA graph, whose kernel arguments are frozen)
__device__ __forceinline__ unsigned long long effective_seed(unsigned long long seed, const unsigned long long *offset) {
  return offset != nullptr ? seed + __ldg(offset) * 0xD1B54A32D192ED03ull : seed;
}
__host__ __device__ __forceinline__ uint32_t drop_pair_hash(uint32_t row_key, uint32_t jpair) {
  uint32_t h = row_key ^ (jpair * 0x9E3779B1u);
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}
__host__ __device__ __forceinline__ bool drop_keep(uint32_t pair_hash, uint32_t j, uint32_t t16) {
  return ((pair_hash >> ((j & 1u) * 16u)) & 0xFFFFu) >= t16;
}

// ---- host: tensor map over a (B, L, H*64) bf16 view with row / scene strides (elements) --------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
inline int make_map(CUtensorMap *map, const void *ptr, int B, int L, int H, int row_stride, long long scene_stride) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return SV_ERR_CUDA;
  if (B == 1 && scene_stride < (long long)L * row_stride) scene_stride = (long long)L * row_stride;  // unused dimension
  cuuint64_t dims[3] = {(cuuint64_t)H * DH, (cuuint64_t)L, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)scene_stride * 2};
  cuuint32_t box[3] = {64, 16, 1};  // BOX_ROWS rows of one head slice
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SV_OK : SV_ERR_INVALID_ARG;
}
// sv_attention_visit_all_blocks: 1 = sweep every key block and run every key-row unit (no block skipping)
extern int g_visit_all_blocks;

inline uint32_t drop_threshold(float p) {
  if (!(p > 0.f)) return 0u;
  unsigned t = (unsigned)((double)p * 65536.0 + 0.5);
  return t > 65535u ? 65535u : t;
}

}  // namespace attn
