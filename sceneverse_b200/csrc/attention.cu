// Fused attention forward on wgmma for the GPS shapes (<= 384 keys, head dim 64):
//   O = dropout(softmax( Q K^T / sqrt(64) + spatial_log_bias + key_padding_mask )) V          per (scene, head)
// Replaces the attention core of
//   * MultiHeadAttentionSpatial, 'cond' fusion (modules/layers/transformers.py:188-237): the per-(head, query)
//     spatial gate  log(clamp(sigmoid(w . pairwise_loc + b), 1e-6))  is computed on the fly from the 5-dim pairwise
//     geometry and the 6 language-conditioned weights — the (H,B,L,T) attention / loc_attn / mask tensors of the
//     reference are never materialised;
//   * nn.MultiheadAttention's scaled-dot-product core incl. its attention-weight dropout (joint self-attention of
//     UnifiedSpatialCrossEncoderV2, self/cross attention of the V1 / Entity decoders; transformers.py:22-24,69-74,118-120).
// One CTA = one warpgroup = one unit (scene, head, 64 query rows); Q / K / V head slices arrive by TMA (128-byte swizzle,
// zero-filled past the sequence end).  The softmax takes two passes over 64-key blocks of S = Q K^T, each block one wgmma
// chain into 32 registers per thread: pass 1 finds the row maximum, pass 2 recomputes the block, exponentiates, sums and
// writes the block's unnormalised bf16 probabilities P to shared memory (two buffers, even / odd blocks) as the K-major A
// operand of O += P V, whose B operand is the SAME staged V tile read MN-major (no transposed copy); that chain is left in
// flight behind the next block's S chain.  1 / sum is applied to the fp32 output row.  Exactly the two-pass arithmetic of a
// full-row softmax: no online rescaling.
#include <climits>

#include "attn_common.cuh"
#include "svgps.h"

namespace {

using namespace attn;

struct FwdArgs {
  __nv_bfloat16 *out;              // (B,Lq,*) head h at columns [h*64, h*64+64)
  long long o_bs;
  int o_rs;
  const unsigned char *kpm;        // (B,Lk) 1 = masked key, or null
  const float *sw;                 // (B,Lq,SH*6) [bias, w1..w5] per spatial head (GATED)
  const float *locs;               // (B,Lq,Lk,5)
  int B, H, SH, Lq, Lk;
  float scale;
  float *lse;                      // (B,H,Lq) natural-log log-sum-exp of the logits per query, or null
  uint32_t t16;                    // dropout threshold (DROP)
  float inv_keep;
  unsigned long long seed;
  const unsigned long long *seed_offset;  // device counter added to the seed at run time (or null)
  int all_blocks;                  // 1 = visit every key block (sv_attention_visit_all_blocks)
  int seq_rows;                    // dropout row key of query i: (b H + h) seq_rows + i (the queries are the first Lq rows)
};

template <bool GATED, bool DROP>
__global__ void __launch_bounds__(128, 3)
attn_fwd_kernel(const __grid_constant__ CUtensorMap mq, const __grid_constant__ CUtensorMap mk,
                const __grid_constant__ CUtensorMap mv, const FwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int NK = (a.Lk + 15) & ~15;          // keys rounded to the TMA box
  const int NK64 = (a.Lk + 63) & ~63;        // keys rounded to the 64-key blocks
  const int nkbox = NK >> 4;                 // 16-row TMA boxes of K / V
  const int nblk = NK64 >> 6;                // 64-key blocks, the element-wise work of the last one NK - 64 (nblk - 1) wide
  uint8_t *sQ = smem;                        // [64][64] sw128
  uint8_t *sK = sQ + 8192;                   // [NK][64] sw128 (the S columns of keys past NK are never read)
  uint8_t *sV = sK + NK * 128;               // [NK64][64] sw128 (read MN-major)
  uint8_t *sP = sV + NK64 * 128;             // 2 x [8][64][8] K-major, no swizzle: P of the even / odd key blocks
  float *kb = reinterpret_cast<float *>(sP + 16384);        // [nblk * 64] additive key bias: 0 or -inf
  uint64_t *bar = reinterpret_cast<uint64_t *>(kb + 384);  // Q, K and V landed
  uint32_t *wlive = reinterpret_cast<uint32_t *>(bar + 1);  // [4] per warp: bit blk = key block blk holds a live key

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int rl = w * 16 + (lane >> 2);             // this thread's first row in the tile (second: rl + 8)
  const int cq = 2 * (lane & 3);                   // its first column in every 8-column group
  const int nqt = (a.Lq + 63) >> 6;
  const int bh = blockIdx.x / nqt, q0 = (blockIdx.x % nqt) * 64;
  const int b = bh / a.H, h = bh % a.H;

  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  // V rows [NK, NK64) are never written by TMA: zero them so that the P V terms of the padded keys are exact zeros
  for (int i = tid; i < (NK64 - NK) * 8; i += 128) reinterpret_cast<uint4 *>(sV + NK * 128)[i] = make_uint4(0, 0, 0, 0);
  uint32_t lm = 0u;
  for (int j = tid; j < NK64; j += 128) {
    const bool live = j < a.Lk && !(a.kpm != nullptr && a.kpm[(size_t)b * a.Lk + j]);
    kb[j] = live ? 0.f : -INFINITY;
    lm |= (uint32_t)live << (j >> 6);
  }
  lm = __reduce_or_sync(0xffffffffu, lm);
  if (lane == 0) wlive[w] = lm;
  fence_proxy_async_smem();
  __syncthreads();
  // the key blocks visited: those holding a live key (attn_common.cuh, block skipping); K / V are loaded up to the last
  const uint32_t live = a.all_blocks ? (1u << nblk) - 1u : wlive[0] | wlive[1] | wlive[2] | wlive[3];
  const int nlive = __popc(live);
  const int kvbox = live ? min(nkbox, 4 * (32 - __clz(live))) : 0;
  if (tid == 0) {
    mbar_expect_tx(bar, rows_bytes(q0, 4, a.Lq) + 2 * rows_bytes(0, kvbox, a.Lk));
    tma_rows(sQ, &mq, h, q0, 4, a.Lq, b, bar);
    tma_rows(sK, &mk, h, 0, kvbox, a.Lk, b, bar);
    tma_rows(sV, &mv, h, 0, kvbox, a.Lk, b, bar);
  }
  const float c2 = a.scale * LOG2E;
  const uint32_t aQ = smem_u32(sQ), aK = smem_u32(sK), aV = smem_u32(sV), aP = smem_u32(sP);
  const unsigned long long seed = DROP ? attn::effective_seed(a.seed, a.seed_offset) : 0ull;
  int qi[2];
  bool qlive[2];
  GateW gw[2];
  const float *loc[2] = {nullptr, nullptr};
  uint32_t rk[2] = {0u, 0u};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    qi[r] = q0 + rl + 8 * r;
    qlive[r] = qi[r] < a.Lq;
    if (GATED && qlive[r]) {
      gw[r].load(a.sw + ((size_t)b * a.Lq + qi[r]) * (a.SH * 6) + (a.SH == 1 ? 0 : h) * 6);
      loc[r] = a.locs + ((size_t)b * a.Lq + qi[r]) * (size_t)a.Lk * 5;
    }
    if (DROP) rk[r] = drop_row_key(seed, ((unsigned long long)b * a.H + h) * a.seq_rows + qi[r]);
  }
  mbar_wait(bar, 0);

  // S block blk = Q . K[64 blk, 64 blk + 64)^T, issued behind whatever chain is still in flight and waited on
  auto s_block = [&](float (&s)[32], int blk) {
    wgmma_fence();
    mma_kk(s, aQ, aK + blk * 8192);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
  };
  float s[32];

  // ---- pass 1: row maximum of the scaled, masked logits (the gate is <= 0, so this bounds the gated logits too) ------
  float m2[2] = {-INFINITY, -INFINITY};
  auto row_max = [&](int blk) {
    const int n = block_cols(blk, NK);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (8 * j >= n) break;
      const float2 k2 = *reinterpret_cast<const float2 *>(kb + blk * 64 + 8 * j + cq);
#pragma unroll
      for (int r = 0; r < 2; ++r)
        m2[r] = fmaxf(m2[r], fmaxf(fmaf(s[4 * j + 2 * r], c2, k2.x), fmaf(s[4 * j + 2 * r + 1], c2, k2.y)));
    }
  };
  for (int it = 0; it < nlive; ++it) {
    const int blk = nth_block(live, it);
    s_block(s, blk);
    row_max(blk);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 1));
    m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 2));
    if (m2[r] == -INFINITY) m2[r] = 0.f;  // every key masked: all weights 0, output row 0
  }

  // ---- pass 2: p = 2^(x - max), row sum, dropout, bf16 P block, O += P V -------------------------------------------------
  float sum[2] = {0.f, 0.f};
  float o[32];   // written by wgmma only; never read when no block is visited
  for (int it = 0; it < nlive; ++it) {
    const int blk = nth_block(live, it), n = block_cols(blk, NK);
    // completes the P V chain of visited block it - 1 too; every warp passed its wait for the chain of block it - 2
    // before the barrier that ended block it - 1, so this block's P buffer is free
    s_block(s, blk);
    uint8_t *P = sP + (it & 1) * 8192;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (8 * j >= n) {   // keys past NK: zero weights (the P V chain runs over the whole block)
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl, 8 * j + cq)) = 0u;
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl + 8, 8 * j + cq)) = 0u;
        continue;
      }
      const int col = blk * 64 + 8 * j + cq;
      const float2 k2 = *reinterpret_cast<const float2 *>(kb + col);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float x0 = fmaf(s[4 * j + 2 * r], c2, k2.x) - m2[r], x1 = fmaf(s[4 * j + 2 * r + 1], c2, k2.y) - m2[r];
        if (GATED && loc[r] != nullptr) {
          if (col < a.Lk) {
            const float *l = loc[r] + (size_t)col * 5;
            x0 += gw[r].log2gate(__ldg(l), __ldg(l + 1), __ldg(l + 2), __ldg(l + 3), __ldg(l + 4));
          }
          if (col + 1 < a.Lk) {
            const float *l = loc[r] + (size_t)(col + 1) * 5;
            x1 += gw[r].log2gate(__ldg(l), __ldg(l + 1), __ldg(l + 2), __ldg(l + 3), __ldg(l + 4));
          }
        }
        float p0 = ex2f(x0), p1 = ex2f(x1);
        sum[r] += p0 + p1;
        if (DROP) {
          const uint32_t hh = drop_pair_hash(rk[r], (uint32_t)col >> 1);
          p0 = (hh & 0xFFFFu) >= a.t16 ? p0 * a.inv_keep : 0.f;
          p1 = (hh >> 16) >= a.t16 ? p1 * a.inv_keep : 0.f;
        }
        // unnormalised probabilities -> bf16 A operand; 1 / sum is applied to the fp32 output row
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl + 8 * r, 8 * j + cq)) = pack_bf16(p0, p1);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();   // the block's P is complete
    wgmma_fence();
    // V staged once, read MN-major; all four k16 steps (a chain cut short at the last block makes ptxas serialize it);
    // left in flight behind the next S chain
    mma_gc(o, aP + (it & 1) * 8192, aV + blk * 8192, 64, it > 0);
    wgmma_commit();
  }
  wgmma_wait<0>();
  fence_regs(o);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!qlive[r]) continue;
    const float tot = sum[r];
    const float inv = tot > 0.f ? 1.0f / tot : 0.f;
    if (lane % 4 == 0 && a.lse != nullptr)
      a.lse[((size_t)b * a.H + h) * a.Lq + qi[r]] = tot > 0.f ? (m2[r] + lg2f(tot)) * LN2 : INFINITY;
    __nv_bfloat16 *op = a.out + (size_t)b * a.o_bs + (size_t)qi[r] * a.o_rs + h * DH + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)   // every key masked (no block visited): output row 0
      *reinterpret_cast<uint32_t *>(op + 8 * j) =
          nlive == 0 ? 0u : pack_bf16(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
  }
}

template <bool GATED, bool DROP>
int launch_fwd(const CUtensorMap &mq, const CUtensorMap &mk, const CUtensorMap &mv, const FwdArgs &a, cudaStream_t st) {
  const int NK = (a.Lk + 15) & ~15, NK64 = (a.Lk + 63) & ~63;
  const size_t smem = 1024 + 8192 + (size_t)(NK + NK64) * 128 + 16384 + 384 * 4 + 8 + 16;
  constexpr size_t SMEM_MAX = 1024 + 8192 + 384 * 128 * 2 + 16384 + 384 * 4 + 8 + 16;
  auto kern = attn_fwd_kernel<GATED, DROP>;
  static bool configured[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return SV_ERR_INVALID_ARG;
  if (!configured[dev]) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
    if (rc) return rc;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    configured[dev] = true;
  }
  kern<<<a.B * a.H * ((a.Lq + 63) >> 6), 128, smem, st>>>(mq, mk, mv, a);
  return sv::after_launch();
}

// ---- streamed forward (sv_attention_fwd_long_bf16): up to STREAM_MAX keys -------------------------------------------------
// The resident kernel above with K / V streamed instead of staged whole.  The 64-row Q tile stays resident; the key blocks
// pass through a FWD_STAGES-deep TMA ring twice, in the resident kernel's block order: pass 1 loads the K block of every
// visited block (S, row maximum), pass 2 its K and V blocks (S again, exp2, row sum, P, O += P V).  Every element is
// computed by the same code on the same operands in the same order, so the results equal the resident kernel's bit for
// bit wherever both run.  Ring item i (i < nlive: pass 1, K of visited block i; else pass 2, K | V of visited block
// i - nlive) lands in buffer i % FWD_STAGES.  A pass-1 buffer is free once every warp's S chain on it completed; a pass-2
// buffer once its P V chain did too, i.e. at the next block's S wait.
constexpr int FWD_STAGES = 2;

constexpr size_t fwd_stream_smem_bytes(int NK64) {
  return 1024 + 8192 + (size_t)FWD_STAGES * 16384 + 16384 + (size_t)NK64 * 4 + 8 * (FWD_STAGES + 1) + 16;
}

template <bool GATED, bool DROP>
__global__ void __launch_bounds__(128, 3)
attn_fwd_stream_kernel(const __grid_constant__ CUtensorMap mq, const __grid_constant__ CUtensorMap mk,
                       const __grid_constant__ CUtensorMap mv, const FwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int NK = (a.Lk + 15) & ~15;          // keys rounded to the TMA box
  const int NK64 = (a.Lk + 63) & ~63;        // keys rounded to the 64-key blocks
  const int nblk = NK64 >> 6;
  uint8_t *sQ = smem;                        // [64][64] sw128
  uint8_t *sC = sQ + 8192;                   // FWD_STAGES x { K block [64][64] sw128, V block [64][64] sw128 }
  uint8_t *sP = sC + FWD_STAGES * 16384;     // 2 x [8][64][8] K-major, no swizzle: P of the even / odd visited blocks
  float *kb = reinterpret_cast<float *>(sP + 16384);              // [NK64] additive key bias: 0 or -inf
  uint64_t *bars = reinterpret_cast<uint64_t *>(kb + NK64);       // [0, FWD_STAGES): ring, FWD_STAGES: Q landed
  uint32_t *wlive = reinterpret_cast<uint32_t *>(bars + FWD_STAGES + 1);  // [4] per warp: bit blk = block blk is live

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int rl = w * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int nqt = (a.Lq + 63) >> 6;
  const int bh = blockIdx.x / nqt, q0 = (blockIdx.x % nqt) * 64;
  const int b = bh / a.H, h = bh % a.H;

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i <= FWD_STAGES; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
    tma_prefetch_desc(&mq);
    tma_prefetch_desc(&mk);
    tma_prefetch_desc(&mv);
  }
  uint32_t lm = 0u;
  for (int j = tid; j < NK64; j += 128) {
    const bool live = j < a.Lk && !(a.kpm != nullptr && a.kpm[(size_t)b * a.Lk + j]);
    kb[j] = live ? 0.f : -INFINITY;
    lm |= (uint32_t)live << (j >> 6);
  }
  lm = __reduce_or_sync(0xffffffffu, lm);
  if (lane == 0) wlive[w] = lm;
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t live = a.all_blocks ? first_blocks(nblk) : wlive[0] | wlive[1] | wlive[2] | wlive[3];
  const int nlive = __popc(live), nitems = 2 * nlive;
  auto load_item = [&](int i) {
    const int buf = i % FWD_STAGES, pass2 = i >= nlive;
    const int blk = nth_block(live, pass2 ? i - nlive : i);
    uint8_t *dst = sC + buf * 16384;
    mbar_expect_tx(&bars[buf], (pass2 ? 2 : 1) * rows_bytes(blk * 64, 4, a.Lk));
    tma_rows(dst, &mk, h, blk * 64, 4, a.Lk, b, &bars[buf]);
    if (pass2) tma_rows(dst + 8192, &mv, h, blk * 64, 4, a.Lk, b, &bars[buf]);
  };
  int issued = min(FWD_STAGES, nitems);   // ring items issued so far (the same count in every thread; thread 0 issues)
  if (tid == 0 && nlive > 0) {
    mbar_expect_tx(&bars[FWD_STAGES], rows_bytes(q0, 4, a.Lq));
    tma_rows(sQ, &mq, h, q0, 4, a.Lq, b, &bars[FWD_STAGES]);
    for (int i = 0; i < issued; ++i) load_item(i);
  }
  // every warp is done with the S chain of item i (and with all chains of the items before it): issue what the freed
  // buffers can take
  auto refill = [&](int i) {
    const int lim = min(nitems, (i < nlive ? i + 1 : i) + FWD_STAGES);
    for (; issued < lim; ++issued)
      if (tid == 0) load_item(issued);
  };
  const float c2 = a.scale * LOG2E;
  const uint32_t aQ = smem_u32(sQ), aC = smem_u32(sC), aP = smem_u32(sP);
  const unsigned long long seed = DROP ? attn::effective_seed(a.seed, a.seed_offset) : 0ull;
  int qi[2];
  bool qlive[2];
  GateW gw[2];
  const float *loc[2] = {nullptr, nullptr};
  uint32_t rk[2] = {0u, 0u};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    qi[r] = q0 + rl + 8 * r;
    qlive[r] = qi[r] < a.Lq;
    if (GATED && qlive[r]) {
      gw[r].load(a.sw + ((size_t)b * a.Lq + qi[r]) * (a.SH * 6) + (a.SH == 1 ? 0 : h) * 6);
      loc[r] = a.locs + ((size_t)b * a.Lq + qi[r]) * (size_t)a.Lk * 5;
    }
    if (DROP) rk[r] = drop_row_key(seed, ((unsigned long long)b * a.H + h) * a.seq_rows + qi[r]);
  }
  if (nlive > 0) mbar_wait(&bars[FWD_STAGES], 0);

  // S block = Q . K_blk^T from ring item i, issued behind whatever chain is still in flight and waited on; then every
  // warp's chains are complete
  auto s_block = [&](float (&s)[32], int i) {
    mbar_wait(&bars[i % FWD_STAGES], (uint32_t)(i / FWD_STAGES) & 1u);
    wgmma_fence();
    mma_kk(s, aQ, aC + (i % FWD_STAGES) * 16384);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    __syncthreads();
    refill(i);
  };
  float s[32];

  // ---- pass 1: row maximum of the scaled, masked logits (the gate is <= 0, so this bounds the gated logits too) ------
  float m2[2] = {-INFINITY, -INFINITY};
  for (int it = 0; it < nlive; ++it) {
    const int blk = nth_block(live, it), n = block_cols(blk, NK);
    s_block(s, it);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (8 * j >= n) break;
      const float2 k2 = *reinterpret_cast<const float2 *>(kb + blk * 64 + 8 * j + cq);
#pragma unroll
      for (int r = 0; r < 2; ++r)
        m2[r] = fmaxf(m2[r], fmaxf(fmaf(s[4 * j + 2 * r], c2, k2.x), fmaf(s[4 * j + 2 * r + 1], c2, k2.y)));
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 1));
    m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 2));
    if (m2[r] == -INFINITY) m2[r] = 0.f;  // every key masked: all weights 0, output row 0
  }

  // ---- pass 2: p = 2^(x - max), row sum, dropout, bf16 P block, O += P V -------------------------------------------------
  float sum[2] = {0.f, 0.f};
  float o[32];   // written by wgmma only; never read when no block is visited
  for (int it = 0; it < nlive; ++it) {
    const int i = nlive + it, blk = nth_block(live, it), n = block_cols(blk, NK);
    s_block(s, i);
    uint8_t *P = sP + (it & 1) * 8192;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (8 * j >= n) {   // keys past NK: zero weights (the P V chain runs over the whole block)
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl, 8 * j + cq)) = 0u;
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl + 8, 8 * j + cq)) = 0u;
        continue;
      }
      const int col = blk * 64 + 8 * j + cq;
      const float2 k2 = *reinterpret_cast<const float2 *>(kb + col);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float x0 = fmaf(s[4 * j + 2 * r], c2, k2.x) - m2[r], x1 = fmaf(s[4 * j + 2 * r + 1], c2, k2.y) - m2[r];
        if (GATED && loc[r] != nullptr) {
          if (col < a.Lk) {
            const float *l = loc[r] + (size_t)col * 5;
            x0 += gw[r].log2gate(__ldg(l), __ldg(l + 1), __ldg(l + 2), __ldg(l + 3), __ldg(l + 4));
          }
          if (col + 1 < a.Lk) {
            const float *l = loc[r] + (size_t)(col + 1) * 5;
            x1 += gw[r].log2gate(__ldg(l), __ldg(l + 1), __ldg(l + 2), __ldg(l + 3), __ldg(l + 4));
          }
        }
        float p0 = ex2f(x0), p1 = ex2f(x1);
        sum[r] += p0 + p1;
        if (DROP) {
          const uint32_t hh = drop_pair_hash(rk[r], (uint32_t)col >> 1);
          p0 = (hh & 0xFFFFu) >= a.t16 ? p0 * a.inv_keep : 0.f;
          p1 = (hh >> 16) >= a.t16 ? p1 * a.inv_keep : 0.f;
        }
        *reinterpret_cast<uint32_t *>(P + tile_off(64, rl + 8 * r, 8 * j + cq)) = pack_bf16(p0, p1);
      }
    }
    // V rows past NK (the last block only) are never written by TMA: zero them so that the P V terms of the padded keys
    // are exact zeros, as in the resident kernel (the buffer may hold an earlier block's rows)
    uint8_t *V = sC + (i % FWD_STAGES) * 16384 + 8192;
    for (int e = n * 8 + tid; e < 64 * 8; e += 128) reinterpret_cast<uint4 *>(V)[e] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
    __syncthreads();   // the block's P is complete
    wgmma_fence();
    mma_gc(o, aP + (it & 1) * 8192, smem_u32(V), 64, it > 0);
    wgmma_commit();
  }
  wgmma_wait<0>();
  fence_regs(o);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!qlive[r]) continue;
    const float tot = sum[r];
    const float inv = tot > 0.f ? 1.0f / tot : 0.f;
    if (lane % 4 == 0 && a.lse != nullptr)
      a.lse[((size_t)b * a.H + h) * a.Lq + qi[r]] = tot > 0.f ? (m2[r] + lg2f(tot)) * LN2 : INFINITY;
    __nv_bfloat16 *op = a.out + (size_t)b * a.o_bs + (size_t)qi[r] * a.o_rs + h * DH + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)   // every key masked (no block visited): output row 0
      *reinterpret_cast<uint32_t *>(op + 8 * j) =
          nlive == 0 ? 0u : pack_bf16(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
  }
}

template <bool GATED, bool DROP>
int launch_fwd_stream(const CUtensorMap &mq, const CUtensorMap &mk, const CUtensorMap &mv, const FwdArgs &a,
                      cudaStream_t st) {
  const size_t smem = fwd_stream_smem_bytes((a.Lk + 63) & ~63);
  constexpr size_t SMEM_MAX = fwd_stream_smem_bytes(STREAM_MAX);
  auto kern = attn_fwd_stream_kernel<GATED, DROP>;
  static bool configured[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return SV_ERR_INVALID_ARG;
  if (!configured[dev]) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
    if (rc) return rc;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    configured[dev] = true;
  }
  kern<<<a.B * a.H * ((a.Lq + 63) >> 6), 128, smem, st>>>(mq, mk, mv, a);
  return sv::after_launch();
}

// argument checks and kernel arguments of both forward entries: Lk <= max_lk, Lq <= max_lq.  Returns -1 when the checks
// pass and there is work to do, else the status to return.
int prepare_fwd(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs, const void *v,
                long long v_bs, int v_rs, void *out, long long o_bs, int o_rs, const unsigned char *key_padding_mask,
                const float *spatial_w, int spatial_heads, const float *pairwise_locs, int B, int H, int Lq, int Lk,
                float scale, float *lse, float dropout_p, unsigned long long seed, int seq_rows, int max_lq, int max_lk,
                FwdArgs *a, CUtensorMap *mq, CUtensorMap *mk, CUtensorMap *mv) {
  if (!(dropout_p >= 0.f) || dropout_p >= 1.f) return SV_ERR_INVALID_ARG;
  if (B < 0 || H < 1 || Lq < 0 || Lq > max_lq || Lk < 1 || Lk > max_lk || seq_rows < Lq) return SV_ERR_INVALID_ARG;
  if (B == 0 || Lq == 0) return SV_OK;
  if (!q || !k || !v || !out) return SV_ERR_INVALID_ARG;
  if ((q_rs % 8) || (k_rs % 8) || (v_rs % 8) || (o_rs % 8) || (q_bs % 8) || (k_bs % 8) || (v_bs % 8) || (o_bs % 8))
    return SV_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(q) & 15) || (reinterpret_cast<uintptr_t>(k) & 15) ||
      (reinterpret_cast<uintptr_t>(v) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return SV_ERR_INVALID_ARG;
  if (spatial_w && (!pairwise_locs || (spatial_heads != 1 && spatial_heads != H))) return SV_ERR_INVALID_ARG;
  if (spatial_w && dropout_p > 0.f) return SV_ERR_INVALID_ARG;  // the reference's spatial attention has no weight dropout
  a->out = (__nv_bfloat16 *)out; a->o_bs = o_bs; a->o_rs = o_rs;
  a->kpm = key_padding_mask; a->sw = spatial_w; a->locs = pairwise_locs;
  a->B = B; a->H = H; a->SH = spatial_heads; a->Lq = Lq; a->Lk = Lk; a->scale = scale;
  a->lse = lse;
  a->t16 = drop_threshold(dropout_p);
  a->inv_keep = 1.0f / (1.0f - dropout_p);
  a->seed = seed; a->seed_offset = sv::g_seed_offset;
  a->all_blocks = g_visit_all_blocks;
  a->seq_rows = seq_rows;
  int rc = make_map(mq, q, B, Lq, H, q_rs, q_bs);
  if (rc) return rc;
  rc = make_map(mk, k, B, Lk, H, k_rs, k_bs);
  if (rc) return rc;
  rc = make_map(mv, v, B, Lk, H, v_rs, v_bs);
  if (rc) return rc;
  return -1;
}

}  // namespace

int attn::g_visit_all_blocks = 0;

extern "C" int sv_attention_visit_all_blocks(int on) {
  attn::g_visit_all_blocks = on ? 1 : 0;
  return SV_OK;
}

extern "C" int sv_attention_fwd_rows_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                          const void *v, long long v_bs, int v_rs, void *out, long long o_bs, int o_rs,
                                          const unsigned char *key_padding_mask, const float *spatial_w, int spatial_heads,
                                          const float *pairwise_locs, int B, int H, int Lq, int Lk, float scale, float *lse,
                                          float dropout_p, unsigned long long seed, int seq_rows, void *stream) {
  FwdArgs a;
  CUtensorMap mq, mk, mv;
  const int rc = prepare_fwd(q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, out, o_bs, o_rs, key_padding_mask, spatial_w,
                             spatial_heads, pairwise_locs, B, H, Lq, Lk, scale, lse, dropout_p, seed, seq_rows, INT_MAX,
                             RESIDENT_MAX, &a, &mq, &mk, &mv);
  if (rc >= 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (spatial_w) return launch_fwd<true, false>(mq, mk, mv, a, st);
  if (a.t16) return launch_fwd<false, true>(mq, mk, mv, a, st);
  return launch_fwd<false, false>(mq, mk, mv, a, st);
}

extern "C" int sv_attention_fwd_long_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                          const void *v, long long v_bs, int v_rs, void *out, long long o_bs, int o_rs,
                                          const unsigned char *key_padding_mask, const float *spatial_w, int spatial_heads,
                                          const float *pairwise_locs, int B, int H, int Lq, int Lk, float scale, float *lse,
                                          float dropout_p, unsigned long long seed, int seq_rows, void *stream) {
  FwdArgs a;
  CUtensorMap mq, mk, mv;
  const int rc = prepare_fwd(q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, out, o_bs, o_rs, key_padding_mask, spatial_w,
                             spatial_heads, pairwise_locs, B, H, Lq, Lk, scale, lse, dropout_p, seed, seq_rows, STREAM_MAX,
                             STREAM_MAX, &a, &mq, &mk, &mv);
  if (rc >= 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (spatial_w) return launch_fwd_stream<true, false>(mq, mk, mv, a, st);
  if (a.t16) return launch_fwd_stream<false, true>(mq, mk, mv, a, st);
  return launch_fwd_stream<false, false>(mq, mk, mv, a, st);
}

extern "C" int sv_attention_fwd_dropout_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs,
                                             int k_rs, const void *v, long long v_bs, int v_rs, void *out, long long o_bs,
                                             int o_rs, const unsigned char *key_padding_mask, const float *spatial_w,
                                             int spatial_heads, const float *pairwise_locs, int B, int H, int Lq, int Lk,
                                             float scale, float *lse, float dropout_p, unsigned long long seed,
                                             void *stream) {
  return sv_attention_fwd_rows_bf16(q, q_bs, q_rs, k, k_bs, k_rs, v, v_bs, v_rs, out, o_bs, o_rs, key_padding_mask,
                                    spatial_w, spatial_heads, pairwise_locs, B, H, Lq, Lk, scale, lse, dropout_p, seed,
                                    Lq, stream);
}
