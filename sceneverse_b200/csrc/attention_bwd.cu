// Backward of the fused attention (csrc/attention.cu) on wgmma: ONE kernel template, launched twice per call.
//   SIDE 0 (tile rows = queries): S = Q K^T, dP = dO V^T -> dS = P o (dP o mask - D) -> dQ = scale * dS K,
//                                 D = rowsum(dO o O), gradients of the 6 spatial-gate weights of each (query, head)
//   SIDE 1 (tile rows = keys):    S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T -> dV = (P o mask)^T dO, dK = scale * dS^T Q
// P is recomputed from Q, K, the gate and the saved log-sum-exp; the dropout mask is regenerated from (seed, indices);
// no (B,H,L,T) tensor is ever stored.  Reference math: autograd of modules/layers/transformers.py:188-237 and of
// nn.MultiheadAttention's core (transformers.py:22-24,69-74,118-120).
// Structure (both sides): the "row" operand pair (Q,dO | K,V) is a 64-row TMA tile owned by the CTA's one warpgroup; the
// "column" operand pair (K,V | Q,dO) is streamed in blocks of 64 rows through a two-deep TMA ring.  Per block: two wgmma
// chains give S and dP in registers (32 + 32 per thread), the element-wise stage writes the bf16 dS / P tiles, and the
// output wgmma chains accumulate over the blocks in registers, reading the SAME staged block MN-major.
#include "attn_common.cuh"
#include "svgps.h"

namespace {

using namespace attn;

struct BwdArgs {
  const __nv_bfloat16 *o, *d_o;      // (B,Lq,H*64) contiguous
  const unsigned char *kpm;          // (B,Lk) or null
  const float *sw, *locs, *lse;      // (B,Lq,H*6) | (B,Lq,Lk,5) | (B,H,Lq)
  int B, H, Lq, Lk;
  float scale;
  __nv_bfloat16 *dq, *dk, *dv;       // dq (B,seq_rows,*), dk / dv (B,Lk,*): rows d_rs elements apart, scenes rows * d_rs
  int d_rs;
  int seq_rows;                      // the queries are the first Lq of seq_rows rows: dq rows [Lq, seq_rows) are zero and
                                     // query i of (b, h) has the dropout row key (b H + h) seq_rows + i
  float *dsw;                        // (B,Lq,H*6) or null
  float *dvec;                       // (B,H,Lq)   D, written by SIDE 0, read by SIDE 1
  uint32_t t16;
  float inv_keep;
  unsigned long long seed;
  const unsigned long long *seed_offset;  // device counter added to the seed at run time (or null)
  int all_blocks;                    // 1 = no block skipping (sv_attention_visit_all_blocks)
};

// 64 columns of a row from the accumulator fragment (row r_lo + 8 r) -> bf16 row of `dst`
__device__ __forceinline__ void store_row_frag(const float (&d)[32], int r, __nv_bfloat16 *dst, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t *>(dst + 8 * j + cq) = pack_bf16(d[4 * j + 2 * r], d[4 * j + 2 * r + 1]);
}
// this thread's 16 columns of a zero row
__device__ __forceinline__ void store_row_zero(__nv_bfloat16 *dst, int cq) {
#pragma unroll
  for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t *>(dst + 8 * j + cq) = 0u;
}

constexpr int BWD_STAGES = 2;   // column-block ring: block j + 1 lands while block j is processed

template <int SIDE>
constexpr size_t bwd_smem_bytes(int NC, bool gated) {
  return 1024 + 16384 + (size_t)BWD_STAGES * 16384 + (SIDE == 1 ? 16384 : 8192) +
         (size_t)(SIDE == 0 ? NC : (gated ? 9 : 3) * NC) * 4 + 8 * (BWD_STAGES + 1) + 16;
}

// One CTA = one warpgroup = one unit (scene, head, 64 rows of the row operand), CTAs ordered by (scene, head) first so
// that the units of one head share its column operand in L2.  Per column block: S and dP wgmma chains; once they are
// complete the staging buffer of the block two ahead is free (its output chain, issued one block earlier, completed with
// them) and the TMA load of the next block is issued; the element-wise stage writes the bf16 dS (and P) tile; the output
// chains are issued and left in flight behind the next block's S / dP chains.
template <int SIDE, bool GATED, bool DROP>
__global__ void __launch_bounds__(128, 3)
attn_bwd_kernel(const __grid_constant__ CUtensorMap mR1, const __grid_constant__ CUtensorMap mR2,
                const __grid_constant__ CUtensorMap mC1, const __grid_constant__ CUtensorMap mC2, const BwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int Lr = SIDE == 0 ? a.Lq : a.Lk;    // rows of the tiles
  const int Lc = SIDE == 0 ? a.Lk : a.Lq;    // columns swept in blocks of 64
  const int NC = (Lc + 15) & ~15;            // columns rounded to the 16-column granule
  uint8_t *sR1 = smem;                       // [64][64] sw128   Q  | K
  uint8_t *sR2 = sR1 + 8192;                 // [64][64] sw128   dO | V
  uint8_t *sC = sR2 + 8192;                  // BWD_STAGES x { [64][64] sw128 K | Q block, [64][64] sw128 V | dO block }
  uint8_t *sG1 = sC + BWD_STAGES * 16384;    // [8][64][8] K-major   scale * dS (^T)
  uint8_t *sG2 = sG1 + 8192;                 // [8][64][8] K-major   dropped P^T (SIDE 1)
  float *vec = reinterpret_cast<float *>(sG2 + (SIDE == 1 ? 8192 : 0));
  // SIDE 0: vec = kb[NC]      SIDE 1: vec = lse2[NC] | Dv[NC] | rk[NC] | W[NC][6] (GATED)
  float *kb = vec;
  float *lse2s = vec, *Dv = vec + NC;
  uint32_t *rks = reinterpret_cast<uint32_t *>(vec + 2 * NC);
  float *Ws = vec + 3 * NC;
  // barriers [0, BWD_STAGES): column block landed in that buffer, BWD_STAGES: row tile landed
  uint64_t *bars = reinterpret_cast<uint64_t *>(vec + (SIDE == 0 ? NC : (GATED ? 9 : 3) * NC));
  // [4] per warp: SIDE 0: bit blk = key block blk holds a live key; SIDE 1: one of the tile's keys is live
  uint32_t *wlive = reinterpret_cast<uint32_t *>(bars + BWD_STAGES + 1);

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int rl = w * 16 + (lane >> 2);             // this thread's first row in the tile (second: rl + 8)
  const int cq = 2 * (lane & 3);                   // its first column in every 8-column group
  const int ntile = (Lr + 63) >> 6;
  const int bh = blockIdx.x / ntile, r0 = (blockIdx.x % ntile) * 64;
  const int b = bh / a.H, h = bh % a.H;
  const int E = a.H * DH;
  const int nblk = (NC + 63) >> 6;
  // dq rows [Lq, seq_rows) of this head: zeros, written by the last query tile (a packed gradient whose queries are a
  // prefix of its rows then feeds one dgrad / wgrad GEMM over all of them)
  if (SIDE == 0 && r0 + 64 >= a.Lq)
    for (int i = a.Lq * 8 + tid; i < a.seq_rows * 8; i += 128)
      reinterpret_cast<uint4 *>(a.dq + ((size_t)b * a.seq_rows + (i >> 3)) * a.d_rs + h * DH)[i & 7] = make_uint4(0, 0, 0, 0);
  uint32_t live = 0u;   // the column blocks visited (attn_common.cuh, block skipping)
  // column block blk, the i-th visited one -> ring buffer i % BWD_STAGES
  auto load_cblock = [&](int i, int blk) {
    const int buf = i % BWD_STAGES;
    mbar_expect_tx(&bars[buf], 2 * rows_bytes(blk * 64, 4, Lc));
    tma_rows(sC + buf * 16384, &mC1, h, blk * 64, 4, Lc, b, &bars[buf]);
    tma_rows(sC + buf * 16384 + 8192, &mC2, h, blk * 64, 4, Lc, b, &bars[buf]);
  };

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i <= BWD_STAGES; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
    tma_prefetch_desc(&mR1);
    tma_prefetch_desc(&mR2);
    tma_prefetch_desc(&mC1);
    tma_prefetch_desc(&mC2);
  }
  // row-tile rows past the sequence end are never written by TMA: start from zeros so that they only ever hold finite
  // values.  Column-block rows past the last box only reach S / dP columns the element-wise stage never reads.
  for (int i = tid; i < 16384 / 16; i += 128) reinterpret_cast<uint4 *>(smem)[i] = make_uint4(0, 0, 0, 0);
  // per-column vectors
  uint32_t lm = 0u;
  if (SIDE == 1 && tid < 64) lm = r0 + tid < a.Lk && !(a.kpm != nullptr && a.kpm[(size_t)b * a.Lk + r0 + tid]);
  for (int c = tid; c < NC; c += 128) {
    if (SIDE == 0) {
      const bool lc = c < a.Lk && !(a.kpm != nullptr && a.kpm[(size_t)b * a.Lk + c]);
      kb[c] = lc ? 0.f : -INFINITY;
      lm |= (uint32_t)lc << (c >> 6);
    } else {
      const bool live = c < a.Lq;
      const size_t r = ((size_t)b * a.H + h) * a.Lq + c;
      lse2s[c] = live ? a.lse[r] * LOG2E : INFINITY;
      Dv[c] = live ? a.dvec[r] : 0.f;
      rks[c] = DROP ? drop_row_key(attn::effective_seed(a.seed, a.seed_offset), ((size_t)b * a.H + h) * a.seq_rows + c) : 0u;
      if (GATED) {
        const float *wp = a.sw + ((size_t)b * a.Lq + (live ? c : 0)) * (a.H * 6) + h * 6;
#pragma unroll
        for (int k = 0; k < 6; ++k) Ws[c * 6 + k] = live ? -LOG2E * wp[k] : 0.f;
      }
    }
  }
  lm = __reduce_or_sync(0xffffffffu, lm);
  if (lane == 0) wlive[w] = lm;
  fence_proxy_async_smem();
  __syncthreads();
  live = wlive[0] | wlive[1] | wlive[2] | wlive[3];
  if (a.all_blocks || (SIDE == 1 && live)) live = first_blocks(nblk);
  const int nlive = __popc(live);
  if (tid == 0 && nlive > 0) {
    mbar_expect_tx(&bars[BWD_STAGES], 2 * rows_bytes(r0, 4, Lr));
    tma_rows(sR1, &mR1, h, r0, 4, Lr, b, &bars[BWD_STAGES]);
    tma_rows(sR2, &mR2, h, r0, 4, Lr, b, &bars[BWD_STAGES]);
    for (int i = 0; i < BWD_STAGES - 1 && i < nlive; ++i) load_cblock(i, nth_block(live, i));
  }
  const float c2 = a.scale * LOG2E;
  const uint32_t aR1 = smem_u32(sR1), aR2 = smem_u32(sR2);
  const uint32_t aG1 = smem_u32(sG1), aG2 = smem_u32(sG2);

  // ---- per-row state (rows rl and rl + 8 of the tile) ----------------------------------------------------------------
  int ri[2];
  bool rlive[2], klive[2];
  float lse2[2] = {INFINITY, INFINITY}, D[2] = {0.f, 0.f};   // SIDE 0
  GateW gw[2];
  const float *loc[2] = {nullptr, nullptr};
  uint32_t rk[2] = {0u, 0u};
  float gg[2][6];                                            // SIDE 0, GATED: d/d(bias, w1..w5) partial sums
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int k = 0; k < 6; ++k) gg[r][k] = 0.f;
    ri[r] = r0 + rl + 8 * r;
    rlive[r] = ri[r] < Lr;
    klive[r] = false;
    if (SIDE == 0) {
      if (rlive[r]) {
        const size_t rr = ((size_t)b * a.H + h) * a.Lq + ri[r];
        lse2[r] = a.lse[rr] * LOG2E;
        const uint4 *po = reinterpret_cast<const uint4 *>(a.o + ((size_t)b * a.Lq + ri[r]) * E + h * DH);
        const uint4 *pd = reinterpret_cast<const uint4 *>(a.d_o + ((size_t)b * a.Lq + ri[r]) * E + h * DH);
        float dd = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const uint4 x = __ldg(po + c), y = __ldg(pd + c);
          const __nv_bfloat162 *xa = reinterpret_cast<const __nv_bfloat162 *>(&x);
          const __nv_bfloat162 *ya = reinterpret_cast<const __nv_bfloat162 *>(&y);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 u = __bfloat1622float2(xa[i]), v = __bfloat1622float2(ya[i]);
            dd = fmaf(u.x, v.x, fmaf(u.y, v.y, dd));
          }
        }
        D[r] = dd;
        if ((lane & 3) == 0) a.dvec[rr] = dd;
        if (GATED) {
          gw[r].load(a.sw + ((size_t)b * a.Lq + ri[r]) * (a.H * 6) + h * 6);
          loc[r] = a.locs + ((size_t)b * a.Lq + ri[r]) * (size_t)a.Lk * 5;
        }
        if (DROP) rk[r] = drop_row_key(attn::effective_seed(a.seed, a.seed_offset), ((size_t)b * a.H + h) * a.seq_rows + ri[r]);
      }
    } else {
      klive[r] = rlive[r] && !(a.kpm != nullptr && a.kpm[(size_t)b * a.Lk + ri[r]]);
    }
  }
  if (nlive == 0) {
    // SIDE 0: every key masked (dQ and the gate-weight gradients are 0); SIDE 1: every key of the tile masked (dK = dV
    // = 0).  Nothing was loaded.  (The accumulators below are only ever written by wgmma: defining them here would
    // serialize the chains.)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (!rlive[r]) continue;
      if (SIDE == 0) {
        store_row_zero(a.dq + ((size_t)b * a.seq_rows + ri[r]) * a.d_rs + h * DH, cq);
        if (GATED && (lane & 3) == 0 && a.dsw != nullptr) {
          float *g = a.dsw + ((size_t)b * a.Lq + ri[r]) * (a.H * 6) + h * 6;
#pragma unroll
          for (int k = 0; k < 6; ++k) g[k] = 0.f;
        }
      } else {
        store_row_zero(a.dk + ((size_t)b * a.Lk + ri[r]) * a.d_rs + h * DH, cq);
        store_row_zero(a.dv + ((size_t)b * a.Lk + ri[r]) * a.d_rs + h * DH, cq);
      }
    }
    return;
  }
  mbar_wait(&bars[BWD_STAGES], 0);

  float o1[32], o2[32];
  int it = 0;
  do {
    const int blk = nth_block(live, it), buf = it % BWD_STAGES;
    // n is CTA-uniform; the shuffle lets ptxas see that too (a width it takes for divergent serializes the output chains)
    const int n = __shfl_sync(0xffffffffu, block_cols(blk, NC), 0);
    const int pre = nth_block(live, it + BWD_STAGES - 1);   // the block loaded once this one's S / dP are done, or -1
    mbar_wait(&bars[buf], (uint32_t)(it / BWD_STAGES) & 1u);
    const uint32_t aC1 = smem_u32(sC) + buf * 16384, aC2 = aC1 + 8192;
    // ---- S_blk, dP_blk (queued behind the previous block's output chains) ---------------------------------------------
    float sa[32], dp[32];
    wgmma_fence();
    mma_kk(sa, aR1, aC1);
    mma_kk(dp, aR2, aC2);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sa);
    fence_regs(dp);
    // every warp's chains are complete: the buffer of visited block it - 1 and the dS / P tiles are free
    __syncthreads();
    if (tid == 0 && pre >= 0) load_cblock(it + BWD_STAGES - 1, pre);

    // ---- element-wise stage over this thread's fragment: rows rl + 8 r, columns 8 j + cq + e of the block ------------
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (8 * j >= n) break;
      const int cl = 8 * j + cq;             // column inside the block
      const int c0 = blk * 64 + cl;          // global column (key for SIDE 0, query for SIDE 1)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float ds[2], pd[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = c0 + e;
          const float sv = sa[4 * j + 2 * r + e];
          float dpi = dp[4 * j + 2 * r + e];
          float p, m = 1.f;
          if (SIDE == 0) {
            float gli = 0.f;
            float l5[5];
            const bool have = GATED && loc[r] != nullptr && c < a.Lk;
            if (have) {
              const float *lp = loc[r] + (size_t)c * 5;
#pragma unroll
              for (int k = 0; k < 5; ++k) l5[k] = __ldg(lp + k);
              gli = gw[r].log2gate(l5[0], l5[1], l5[2], l5[3], l5[4]);
            }
            p = ex2f(fmaf(sv, c2, kb[c]) - lse2[r] + gli);
            if (DROP) {
              const uint32_t hh = drop_pair_hash(rk[r], (uint32_t)c >> 1);
              m = drop_keep(hh, (uint32_t)c, a.t16) ? a.inv_keep : 0.f;
              dpi *= m;
            }
            const float dsi = p * (dpi - D[r]);
            if (GATED && have && gli > LOG2_CLAMP) {                 // clamp(sigmoid, 1e-6) inactive
              const float dz = dsi * (1.0f - ex2f(gli));            // d log(sigmoid(z)) / dz = 1 - sigmoid(z)
              gg[r][0] += dz;
#pragma unroll
              for (int k = 0; k < 5; ++k) gg[r][1 + k] = fmaf(dz, l5[k], gg[r][1 + k]);
            }
            ds[e] = dsi * a.scale;
            pd[e] = p * m;
          } else {
            float gl = 0.f;
            if (GATED && klive[r] && c < a.Lq) {
              const float *wv = Ws + c * 6;
              const GateW g{wv[0], wv[1], wv[2], wv[3], wv[4], wv[5]};
              const float *l = a.locs + (((size_t)b * a.Lq + c) * a.Lk + ri[r]) * 5;
              gl = g.log2gate(__ldg(l), __ldg(l + 1), __ldg(l + 2), __ldg(l + 3), __ldg(l + 4));
            }
            p = klive[r] ? ex2f(fmaf(sv, c2, -lse2s[c]) + gl) : 0.f;
            if (DROP) {
              const uint32_t hh = drop_pair_hash(rks[c], (uint32_t)ri[r] >> 1);
              m = drop_keep(hh, (uint32_t)ri[r], a.t16) ? a.inv_keep : 0.f;
              dpi *= m;
            }
            ds[e] = p * (dpi - Dv[c]) * a.scale;
            pd[e] = p * m;
          }
        }
        const uint32_t off = tile_off(64, rl + 8 * r, cl);
        *reinterpret_cast<uint32_t *>(sG1 + off) = pack_bf16(ds[0], ds[1]);
        if (SIDE == 1) *reinterpret_cast<uint32_t *>(sG2 + off) = pack_bf16(pd[0], pd[1]);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();   // the tile's dS (and P) are complete

    // ---- accumulate the outputs over this block's columns (column operand read MN-major), left in flight ---------------
    wgmma_fence();
    mma_gc(o1, aG1, aC1, n, it > 0);
    if (SIDE == 1) mma_gc(o2, aG2, aC2, n, it > 0);
    wgmma_commit();
  } while (++it < nlive);
  wgmma_wait<0>();
  fence_regs(o1);
  if (SIDE == 1) fence_regs(o2);

  // ---- epilogue ----------------------------------------------------------------------------------------------------------
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (SIDE == 0 && GATED) {
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        gg[r][k] += __shfl_xor_sync(0xffffffffu, gg[r][k], 1);
        gg[r][k] += __shfl_xor_sync(0xffffffffu, gg[r][k], 2);
      }
    }
    if (!rlive[r]) continue;
    if (SIDE == 0) {
      store_row_frag(o1, r, a.dq + ((size_t)b * a.seq_rows + ri[r]) * a.d_rs + h * DH, cq);
      if (GATED && (lane & 3) == 0 && a.dsw != nullptr) {
        float *g = a.dsw + ((size_t)b * a.Lq + ri[r]) * (a.H * 6) + h * 6;
#pragma unroll
        for (int k = 0; k < 6; ++k) g[k] = gg[r][k];
      }
    } else {
      store_row_frag(o1, r, a.dk + ((size_t)b * a.Lk + ri[r]) * a.d_rs + h * DH, cq);
      store_row_frag(o2, r, a.dv + ((size_t)b * a.Lk + ri[r]) * a.d_rs + h * DH, cq);
    }
  }
}

template <int SIDE, bool GATED, bool DROP>
int launch_side(const CUtensorMap &r1, const CUtensorMap &r2, const CUtensorMap &c1, const CUtensorMap &c2,
                const BwdArgs &a, cudaStream_t st) {
  const int Lr = SIDE == 0 ? a.Lq : a.Lk, Lc = SIDE == 0 ? a.Lk : a.Lq;
  const size_t smem = bwd_smem_bytes<SIDE>((Lc + 15) & ~15, GATED);
  // the kernel's dynamic shared-memory limit: the one of 384 columns until a launch needs more (the long entry), then the
  // one of STREAM_MAX columns
  constexpr size_t SMEM_RESIDENT = bwd_smem_bytes<SIDE>(RESIDENT_MAX, GATED);
  constexpr size_t SMEM_LONG = bwd_smem_bytes<SIDE>(STREAM_MAX, GATED);
  auto kern = attn_bwd_kernel<SIDE, GATED, DROP>;
  static size_t configured[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return SV_ERR_INVALID_ARG;
  if (configured[dev] < smem) {
    const size_t limit = smem <= SMEM_RESIDENT ? SMEM_RESIDENT : SMEM_LONG;
    int rc = sv::cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
    if (rc) return rc;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    configured[dev] = limit;
  }
  kern<<<a.B * a.H * ((Lr + 63) >> 6), 128, smem, st>>>(r1, r2, c1, c2, a);
  return sv::after_launch();
}

template <bool GATED, bool DROP>
int launch_both(const CUtensorMap &mq, const CUtensorMap &mk, const CUtensorMap &mv, const CUtensorMap &mo,
                const BwdArgs &a, cudaStream_t st) {
  int rc = launch_side<0, GATED, DROP>(mq, mo, mk, mv, a, st);
  if (rc) return rc;
  return launch_side<1, GATED, DROP>(mk, mv, mq, mo, a, st);
}

// argument checks and launches of both backward entries (Lq, Lk <= max_len)
int attention_bwd(int max_len, const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                  const void *v, long long v_bs, int v_rs, const void *o, const void *d_o, const unsigned char *key_padding_mask,
                  const float *spatial_w, const float *pairwise_locs, const float *lse, int B, int H, int Lq, int Lk,
                  float scale, void *dq, void *dk, void *dv, int d_rs, float *d_spatial_w, float *dvec, float dropout_p,
                  unsigned long long seed, int seq_rows, void *stream) {
  if (d_rs < H * attn::DH || (d_rs % 8)) return SV_ERR_INVALID_ARG;
  if (!(dropout_p >= 0.f) || dropout_p >= 1.f) return SV_ERR_INVALID_ARG;
  if (B < 0 || H < 1 || Lq < 1 || Lk < 1 || Lq > max_len || Lk > max_len || seq_rows < Lq) return SV_ERR_INVALID_ARG;
  if (B == 0) return SV_OK;
  if (!q || !k || !v || !o || !d_o || !lse || !dq || !dk || !dv || !dvec) return SV_ERR_INVALID_ARG;
  if ((q_rs % 8) || (k_rs % 8) || (v_rs % 8) || (q_bs % 8) || (k_bs % 8) || (v_bs % 8)) return SV_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(q) & 15) || (reinterpret_cast<uintptr_t>(k) & 15) ||
      (reinterpret_cast<uintptr_t>(v) & 15) || (reinterpret_cast<uintptr_t>(o) & 15) ||
      (reinterpret_cast<uintptr_t>(d_o) & 15) || (reinterpret_cast<uintptr_t>(dq) & 15) ||
      (reinterpret_cast<uintptr_t>(dk) & 15) || (reinterpret_cast<uintptr_t>(dv) & 15))
    return SV_ERR_INVALID_ARG;
  if (spatial_w && (!pairwise_locs || !d_spatial_w)) return SV_ERR_INVALID_ARG;
  if (spatial_w && dropout_p > 0.f) return SV_ERR_INVALID_ARG;
  BwdArgs a;
  a.o = (const __nv_bfloat16 *)o; a.d_o = (const __nv_bfloat16 *)d_o;
  a.kpm = key_padding_mask; a.sw = spatial_w; a.locs = pairwise_locs; a.lse = lse;
  a.B = B; a.H = H; a.Lq = Lq; a.Lk = Lk; a.scale = scale;
  a.dq = (__nv_bfloat16 *)dq; a.dk = (__nv_bfloat16 *)dk; a.dv = (__nv_bfloat16 *)dv;
  a.d_rs = d_rs;
  a.seq_rows = seq_rows;
  a.dsw = d_spatial_w; a.dvec = dvec;
  a.t16 = drop_threshold(dropout_p);
  a.inv_keep = 1.0f / (1.0f - dropout_p);
  a.seed = seed; a.seed_offset = sv::g_seed_offset;
  a.all_blocks = attn::g_visit_all_blocks;
  CUtensorMap mq, mk, mv, mo;
  int rc = make_map(&mq, q, B, Lq, H, q_rs, q_bs);
  if (rc) return rc;
  rc = make_map(&mk, k, B, Lk, H, k_rs, k_bs);
  if (rc) return rc;
  rc = make_map(&mv, v, B, Lk, H, v_rs, v_bs);
  if (rc) return rc;
  rc = make_map(&mo, d_o, B, Lq, H, H * DH, (long long)Lq * H * DH);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (spatial_w) return launch_both<true, false>(mq, mk, mv, mo, a, st);
  if (a.t16) return launch_both<false, true>(mq, mk, mv, mo, a, st);
  return launch_both<false, false>(mq, mk, mv, mo, a, st);
}

}  // namespace

extern "C" int sv_attention_bwd_rows_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                          const void *v, long long v_bs, int v_rs, const void *o, const void *d_o,
                                          const unsigned char *key_padding_mask, const float *spatial_w,
                                          const float *pairwise_locs, const float *lse, int B, int H, int Lq, int Lk,
                                          float scale, void *dq, void *dk, void *dv, int d_rs, float *d_spatial_w,
                                          float *dvec, float dropout_p, unsigned long long seed, int seq_rows,
                                          void *stream) {
  return attention_bwd(RESIDENT_MAX, q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, o, d_o, key_padding_mask, spatial_w,
                       pairwise_locs, lse, B, H, Lq, Lk, scale, dq, dk, dv, d_rs, d_spatial_w, dvec, dropout_p, seed,
                       seq_rows, stream);
}

extern "C" int sv_attention_bwd_long_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                          const void *v, long long v_bs, int v_rs, const void *o, const void *d_o,
                                          const unsigned char *key_padding_mask, const float *spatial_w,
                                          const float *pairwise_locs, const float *lse, int B, int H, int Lq, int Lk,
                                          float scale, void *dq, void *dk, void *dv, int d_rs, float *d_spatial_w,
                                          float *dvec, float dropout_p, unsigned long long seed, int seq_rows,
                                          void *stream) {
  return attention_bwd(STREAM_MAX, q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, o, d_o, key_padding_mask, spatial_w,
                       pairwise_locs, lse, B, H, Lq, Lk, scale, dq, dk, dv, d_rs, d_spatial_w, dvec, dropout_p, seed,
                       seq_rows, stream);
}

extern "C" int sv_attention_bwd_strided_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs,
                                             int k_rs, const void *v, long long v_bs, int v_rs, const void *o,
                                             const void *d_o, const unsigned char *key_padding_mask,
                                             const float *spatial_w, const float *pairwise_locs, const float *lse, int B,
                                             int H, int Lq, int Lk, float scale, void *dq, void *dk, void *dv, int d_rs,
                                             float *d_spatial_w, float *dvec, float dropout_p, unsigned long long seed,
                                             void *stream) {
  return sv_attention_bwd_rows_bf16(q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, o, d_o, key_padding_mask, spatial_w,
                                    pairwise_locs, lse, B, H, Lq, Lk, scale, dq, dk, dv, d_rs, d_spatial_w, dvec, dropout_p,
                                    seed, Lq, stream);
}
