// Persistent, warp-specialised wgmma GEMM with fused epilogues — the dense-contraction workhorse of the GPS path:
// every nn.Linear of the attention stack / BERT / heads in all three directions (forward, dgrad, wgrad) and the
// SA3 + fc stage of PointNet++ (reference: F.linear / 1x1 Conv2d call sites and their autograd, SURVEY.md §2.3,
// e.g. modules/layers/transformers.py:115-154,188-192,285-316).
//
//   C[M,N] = epilogue( A[M,K] x B[N,K]^T ),  bf16 operands, fp32 accumulation in registers
//
// Roles (384 threads): warp 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers: each issues the wgmma chain
// for 64 rows of the 128-row tile and runs the epilogue of those rows straight from its accumulator registers.  The staged
// forward and dgrad kernels at 64- and 128-column tiles have 640 threads instead: warpgroups 3 and 4 run the epilogues of
// warpgroups 1 and 2, fed through shared memory, so the MMAs of the next tile overlap each tile's epilogue (see gemm_kernel).
// Operand tiles travel global -> shared by TMA (cp.async.bulk.tensor.2d, 128-byte rows, SWIZZLE_128B) through an
// mbarrier ring of up to 8 stages that keeps loading the next tiles while the consumers run an epilogue; either operand
// may be stored transposed in memory ([K][rows]) and is then staged as 64-column slabs and read MN-major by wgmma —
// the dgrad / wgrad forms of a linear layer need no transposed copy.  Out-of-bounds rows / columns / K are zero-filled
// by TMA.  The epilogue stages its results in shared memory, one 64-row x 128-byte box at a time, and writes each box with
// one TMA store (WGRAD: TMA reduce-add), which clips it at the tensor edge and drains while the warpgroup goes on to the
// next box or the next tile's main loop; the last columns of a row that does not end on a 16-byte unit are copied out of the
// box per element.  Outputs that cannot take such boxes (the SA3 row max, the residual add, pitches that are not whole
// 16-byte units) keep per-element stores masked at the edge (template parameter OUT_TMA).
//
// Epilogue families (template parameter EPI):
//   EPI_FWD   + bias -> (store pre-activation copy) -> relu | gelu(erf) -> dropout (counter hash, nothing stored)
//             -> + residual -> bf16 | f32 store, or max over 16-row groups (PointNet++ SA3 neighbourhood max)
//   EPI_DGRAD x activation derivative: relu+dropout from the saved forward OUTPUT (h > 0 ? 1/keep : 0), or gelu' from the
//             saved pre-activation with the dropout mask regenerated from (seed, row, column)
//   EPI_WGRAD fp32 result, split-K over the work list, reduce-adds into the (flat) gradient buffer; the bias
//             gradient (column sums of dL/dy) comes out of the SAME main loop: one extra N = 8 wgmma per K step against a
//             constant tile of ones (first column-tile only)
#include <cstdio>
#include <cstdlib>
#include <cuda.h>
#include <cuda_bf16.h>

#include "attn_common.cuh"
#include "sm90.cuh"
#include "svcommon.h"
#include "svgps.h"

namespace {

using namespace sm90;

constexpr int BM = 128, BK = 64;
constexpr int EPI_FWD = 0, EPI_DGRAD = 1, EPI_WGRAD = 2;

struct GemmArgs {
  int M, N, K;
  int dbg = 0;              // profiling switches (sv_gemm_force_ctas bits 8..): 1 = epilogue skips its body, 2 = producer skips TMA
  long long *prof = nullptr;  // profiling (sv_gemm_profile): [gridDim.x][16] cycle counters of the consumer threads, or null
  const float *bias;        // [N] or null (FWD)
  const void *residual;     // [M,N] same dtype as out, or null (FWD; added after activation / dropout)
  void *out;                // [M,N] (or [M/rowmax,N] when rowmax > 0)
  int act;                  // FWD: 0 none, 1 relu, 2 gelu(erf);  DGRAD: 0 none, 1 relu(+dropout) from output, 2 gelu(+dropout) from pre-activation
  int out_f32;              // 0 bf16, 1 f32
  int rowmax;               // 0, or 16: max over groups of 16 consecutive rows (SA3 neighbourhood max)
  int ldo;                  // leading dimension of out / residual / out2 (elements)
  void *out2;               // FWD: bf16 [M,N] (ld = ldo) copy of the pre-activation (acc + bias), or null
  const void *aux;          // DGRAD: bf16 [M,N] saved forward tensor (act 1: output, act 2: pre-activation)
  int ld_aux;
  uint32_t t16;             // dropout threshold (0 = no dropout): keep iff 16-bit uniform >= t16
  float inv_keep;
  unsigned long long seed;
  const unsigned long long *seed_offset;
  int n_fast;               // tile order of the work list: 1 = column tiles vary fastest (A panels stream once, B stays in
                            // L2), 0 = row tiles vary fastest (the reverse); chosen by operand size
  int splits;               // split-K factor (>= 1); > 1 only with red_out
  int red_out;              // WGRAD: accumulate into out with atomic adds instead of storing
  float *bias_grad;         // WGRAD: [M] += row sums of A (the bias gradient), or null
  int n_tma;                // OUT_TMA: columns [0, n_tma) go out by TMA, the rest of [0, N) per element (see run_gemm)
  int aux_tma;              // DGRAD with OUT_TMA and bf16 out: aux is loaded by TMA through mapO2 (see run_gemm)
};

// Phi(x) = 0.5 (1 + erf(x / sqrt 2)) and e = exp(-x^2 / 2) with two MUFU ops: erf by Abramowitz-Stegun 7.1.26
// (|error| < 1.5e-7, far below the bf16 / fp32-accumulation noise of the GEMM it follows); gelu = x Phi,
// gelu' = Phi + x e / sqrt(2 pi) — the exact (erf) GELU the reference uses (F.gelu default, HF "gelu").
__device__ __forceinline__ void gelu_parts(float x, float &cdf, float &e) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  const float p = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  e = attn::ex2f(-z * z * 1.4426950408889634f);
  const float h = 0.5f * p * e;          // = 0.5 (1 - erf|z|)
  cdf = x >= 0.f ? 1.0f - h : h;
}
__device__ __forceinline__ float gelu_erf(float x) {
  float c, e;
  gelu_parts(x, c, e);
  return x * c;
}
__device__ __forceinline__ float gelu_grad(float x) {
  float c, e;
  gelu_parts(x, c, e);
  return fmaf(x * e, 0.3989422804014327f, c);
}

// the two adjacent columns (col, col + 1) of one row: col is even, col + 1 may lie past N
__device__ __forceinline__ void store_pair_bf16(__nv_bfloat16 *o, bool two, bool vec, float v0, float v1) {
  if (two && vec) *reinterpret_cast<uint32_t *>(o) = pack_bf16(v0, v1);
  else {
    o[0] = __float2bfloat16_rn(v0);
    if (two) o[1] = __float2bfloat16_rn(v1);
  }
}

// A staged output box: 64 rows (one consumer warpgroup's share of the tile) x 128 bytes (64 bf16 or 32 fp32 columns),
// SWIZZLE_128B.  Each consumer warpgroup owns a ring of two, so one box can be written while the previous one drains.
constexpr int OUT_BOX = 64 * 128;
constexpr int OUT_RING = 2 * OUT_BOX;
constexpr int SMEM_OPTIN = 232448;   // 227 KB: the sm_90 per-block opt-in limit

template <int BN, int EPI, int OUT_TMA>
struct GemmCfg {
  // EW: the staged forward / dgrad epilogue runs in two warpgroups of its own (see gemm_kernel), fed the accumulators through a
  // shared-memory hand-off of 64 x BN fp32 per MMA warpgroup.  Not at BN = 192: the hand-off (96 KB) would leave 2 stages.
  // OUT_TMA = 2 selects it; run_gemm takes it only where a CTA gets enough tiles for the overlap to pay (pick_tile).
  static constexpr bool EW = OUT_TMA == 2;
  static_assert(!EW || (BN <= 128 && EPI != EPI_WGRAD), "epilogue warpgroups: staged forward / dgrad at BN <= 128 only");
  static constexpr int THREADS = EW ? 640 : 384;
  // Register split (setmaxnreg, NREG): the producer warpgroup gives most of its launch share to the warpgroups that hold the
  // 64 x BN fp32 accumulators.  EW: 640 threads launch with 96 each, 128 x (24 + 2 x 96 epilogue + 2 x 128) = 60416 <= 640 x 96.
  // The cooperative staged kernels: 384 threads launch with 168, 128 x (40 + 2 x 232) = 64512 = 384 x 168 (the 192-wide
  // epilogue spills at a flat 168).  The per-element kernels keep one register count for all their threads.
  static constexpr bool NREG = OUT_TMA != 0;
  static constexpr int REG_LAUNCH = EW ? 96 : 168, REG_PRODUCER = EW ? 24 : 40, REG_EPI = 96, REG_MMA = EW ? 128 : 232;
  static_assert(128 * (REG_PRODUCER + (EW ? 2 * REG_EPI : 0) + 2 * REG_MMA) <= THREADS * REG_LAUNCH,
                "setmaxnreg split exceeds the launch allocation");
  static constexpr int A_STAGE = BM * BK * 2, B_STAGE = BN * BK * 2;
  static constexpr int OUT = OUT_TMA ? 2 * OUT_RING : 0;   // the output rings of the two epilogue-running warpgroups
  static constexpr int HAND = EW ? 2 * 64 * BN * 4 : 0;    // [2 MMA warpgroups][BN / 8][128 threads][4] fp32
  static constexpr int BARS = 2 * 8 + 4 + 4;               // full / empty of at most 8 stages, 2 x 2 aux-box barriers,
                                                           // 2 x (hand-off full, hand-off empty)
  // OUT_TMA: operand stages fill what is left after the output rings, the hand-off, 1 KB alignment slack, the 1 KB tile of
  // ones (WGRAD bias-gradient operand) and the barriers.  The per-element kernels keep their 200 KB operand budget.
  static constexpr int STAGES_RAW =
      OUT_TMA ? (SMEM_OPTIN - OUT - HAND - 1024 - 1024 - BARS * 8) / (A_STAGE + B_STAGE) : (200 * 1024) / (A_STAGE + B_STAGE);
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr size_t SMEM = (size_t)STAGES * (A_STAGE + B_STAGE) + OUT + HAND + 1024 + 1024 + BARS * 8;
  static_assert(SMEM <= SMEM_OPTIN, "gemm_kernel shared memory exceeds the opt-in limit");
};

// Columns [n_tma, N) of a staged box (64 rows from row cm, 8 box_j columns from column cn): they lie past the last whole
// 16-byte unit of a row, and a TMA store clips only to whole units, so they are copied out per element, from the box after
// the warpgroup barrier that completed it.  out2 comes from the box at `pre` (ring slot 0).
__device__ __forceinline__ void store_tail(const uint8_t *box, const uint8_t *pre, const GemmArgs &g, bool red, bool f32,
                                           int cn, int cm, int t) {
  const int r = t >> 1, row = cm + r;   // two threads per box row, alternate columns
  if (row >= g.M) return;
  const int sh = f32 ? 2 : 1;           // log2 of the element size
  const int end = min(g.N - cn, 128 >> sh);
  for (int cc = max(g.n_tma - cn, 0) + (t & 1); cc < end; cc += 2) {
    const int byte = cc << sh;
    const int off = r * 128 + ((((byte >> 4) ^ (r & 7)) << 4) | (byte & 15));
    const size_t o = (size_t)row * g.ldo + cn + cc;
    if (red) atomicAdd(reinterpret_cast<float *>(g.out) + o, *reinterpret_cast<const float *>(box + off));
    else if (f32) reinterpret_cast<float *>(g.out)[o] = *reinterpret_cast<const float *>(box + off);
    else {
      reinterpret_cast<uint16_t *>(g.out)[o] = *reinterpret_cast<const uint16_t *>(box + off);
      if (g.out2 != nullptr) reinterpret_cast<uint16_t *>(g.out2)[o] = *reinterpret_cast<const uint16_t *>(pre + off);
    }
  }
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void mma(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 64) wgmma_n64<TA, TB>(d, da, db, scale_d);
  else if constexpr (BN == 128) wgmma_n128<TA, TB>(d, da, db, scale_d);
  else wgmma_n192<TA, TB>(d, da, db, scale_d);
}

// OUT_TMA = 1 or 2: the epilogue stages out (and out2) in shared memory and writes them by TMA store (WGRAD: TMA reduce-add)
// through mapO / mapO2; 0: per-element stores (the maps are unused).  With g.aux_tma, mapO2 is the DGRAD saved activation,
// whose boxes are loaded into the ring slots the same columns go out through.
//
// Schedules.  Cooperative (384 threads): warpgroups 1 and 2 each run the main loop of 64 rows of the tile, then the epilogue of
// those rows from their accumulator registers, and only then the next tile's main loop.  Epilogue warpgroups (OUT_TMA = 2,
// 640 threads: the staged forward / dgrad at BN <= 128): MMA warpgroup 1 + c copies its accumulator fragment into hand-off
// buffer c ([BN / 8][128 threads][4] fp32: thread t's column group j at (j * 128 + t) * 16 bytes, conflict-free v4 accesses),
// arrives on hand-off barrier "full" and goes straight on to the next tile's main loop; epilogue warpgroup 3 + c, thread t,
// reads back exactly the fragment thread t of the MMA warpgroup held, runs the same epilogue body, and arrives on "empty".
// An MMA warpgroup waits for "empty" only when an epilogue takes longer than a main loop.
template <int BN, int EPI, int TA, int TB, int OUT_TMA>
__global__ void __launch_bounds__(GemmCfg<BN, EPI, OUT_TMA>::THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
            const __grid_constant__ CUtensorMap mapO, const __grid_constant__ CUtensorMap mapO2, const GemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  using Cfg = GemmCfg<BN, EPI, OUT_TMA>;
  constexpr bool EW = Cfg::EW;
  constexpr int A_STAGE = Cfg::A_STAGE, B_STAGE = Cfg::B_STAGE, STAGES = Cfg::STAGES;
  uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B tiles: 1024-byte aligned
  uint8_t *sA = smem;
  uint8_t *sB = smem + STAGES * A_STAGE;
  uint8_t *sOut = sB + STAGES * B_STAGE;                       // [2 epilogue-running warpgroups][OUT_RING] staged output boxes
  float4 *sHand = reinterpret_cast<float4 *>(sOut + Cfg::OUT); // EW: [2][BN / 8][128] accumulator hand-off
  uint8_t *sOnes = sOut + Cfg::OUT + Cfg::HAND;                // [8][64] bf16 ones (1 KB), WGRAD bias-gradient operand
  uint64_t *full = reinterpret_cast<uint64_t *>(sOnes + 1024);
  uint64_t *empty = full + STAGES;
  uint64_t *auxb = empty + STAGES;                             // [2 epilogue-running warpgroups][2 ring slots]: aux box landed
  uint64_t *hfull = auxb + 4, *hempty = hfull + 2;             // EW: [2] hand-off written / read

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int tiles_m = (g.M + BM - 1) / BM, tiles_n = (g.N + BN - 1) / BN;
  const int n_tiles = tiles_m * tiles_n;
  const int k_steps = (g.K + BK - 1) / BK;
  const int kps = (k_steps + g.splits - 1) / g.splits;   // K steps per split (host guarantees every split is non-empty)
  const int n_items = n_tiles * g.splits;                // work list: item i = (tile i % n_tiles, split i / n_tiles)
  const bool with_bias_grad = EPI == EPI_WGRAD && g.bias_grad != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, 2);   // one arrival per MMA warpgroup
    }
    for (int i = 0; i < 4; ++i) mbar_init(auxb + i, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(hfull + i, 128);
      mbar_init(hempty + i, 128);
    }
    mbar_fence_init();
  }
  if (EPI == EPI_WGRAD) {
    for (int i = threadIdx.x; i < 256; i += Cfg::THREADS) reinterpret_cast<uint32_t *>(sOnes)[i] = 0x3F803F80u;  // bf16 1.0 pairs
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------- TMA producer -------------------------------
    if constexpr (Cfg::NREG) setmaxnreg_dec<Cfg::REG_PRODUCER>();
    if (warp == 0 && lane == 0) {
      uint32_t s = 0, ph = 1;   // waiting on parity 1 of a fresh barrier returns at once: the first pass finds every slot free
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int t = item % n_tiles, sp = item / n_tiles;
        const int tmi = g.n_fast ? t / tiles_n : t % tiles_m, tni = g.n_fast ? t % tiles_n : t / tiles_m;
        const int m0 = tmi * BM, n0 = tni * BN;
        const int ks0 = sp * kps, ks1 = min(k_steps, ks0 + kps);
        for (int ks = ks0; ks < ks1; ++ks) {
          mbar_wait(empty + s, ph);
          const int k0 = ks * BK;
          const uint32_t da = smem_u32(sA + s * A_STAGE), db = smem_u32(sB + s * B_STAGE);
          if (g.dbg & 2) {   // profiling: no loads, the MMAs chew on whatever the slot holds
            mbar_arrive(full + s);
          } else {
            mbar_expect_tx(full + s, A_STAGE + B_STAGE);
            if (TA) {  // [K][M] storage: one [BK x 64] box per 64 rows of the tile
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(da + j * (BK * 128), &mapA, m0 + j * 64, k0, full + s);
            } else {
              tma_load_2d(da, &mapA, k0, m0, full + s);
            }
            if (TB) {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(db + j * (BK * 128), &mapB, n0 + j * 64, k0, full + s);
            } else {
              tma_load_2d(db, &mapB, k0, n0, full + s);
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ---------------- MMA warpgroups (wgmma main loop of 64 rows) and the warpgroups that run the epilogue of those rows ----------------
  const bool epi_wg = EW && wg >= 3;    // an epilogue warpgroup (EW); otherwise an MMA warpgroup, which in the cooperative
                                        // schedule runs its own epilogue
  const int c = epi_wg ? wg - 3 : wg - 1;   // rows [64 c, 64 c + 64) of the tile
  const int t = threadIdx.x & 127, w = t >> 5;
  const int r_lo = c * 64 + w * 16 + (lane >> 2);   // this thread's first accumulator row in the tile (second: + 8)
  const int cq = 2 * (lane & 3);                    // its first column inside every 8-column group
  const unsigned long long seed = (EPI != EPI_WGRAD && g.t16) ? attn::effective_seed(g.seed, g.seed_offset) : 0ull;
  // staged output: a box holds box_j 8-column groups.  Without out2, box k of this warpgroup goes to ring slot k % 2; with
  // out2, every box step fills both slots (slot 0 the pre-activation, slot 1 the output).
  constexpr bool tma_out = OUT_TMA != 0;
  const bool f32_out = EPI == EPI_WGRAD || g.out_f32;
  const int box_j = f32_out ? 4 : 8;
  const uint32_t ring = smem_u32(sOut) + (uint32_t)c * OUT_RING;
  // DGRAD with a TMA-loadable saved activation: box k's aux tile is loaded into the ring slot box k is staged in, all of a
  // tile's boxes (at most two: the ring) before its main loop.  Not at BN = 192: three boxes would not fit the ring, and with
  // both aux paths in one kernel its epilogue spills, so it keeps the per-element loads.
  const bool aux_tma = tma_out && EPI == EPI_DGRAD && BN <= 128 && g.aux_tma && !(g.dbg & 1);
  uint64_t *my_auxb = auxb + 2 * c;
  uint32_t aux_ph = 0;   // bit k: parity of ring slot k's next aux load
  // this lane's byte offsets inside a box: stmatrix / ldmatrix row addresses (bf16), or its two fp32 columns of row r_lo - 64 c
  const uint32_t sm_row = (uint32_t)(w * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * 128u, sm_x = lane & 7, sm_j = lane >> 4;
  const uint32_t f_row = (uint32_t)(w * 16 + (lane >> 2)) * 128u, f_hi = (lane >> 1) & 1, f_x = lane >> 2, f_lo = (lane & 1) * 8u;
  float4 *hand = sHand + (size_t)c * (BN / 8) * 128;   // EW: this warpgroup pair's hand-off buffer
  uint32_t nbox = 0;
  uint32_t s = 0, ph = 0, hph = 0;
  long long p_full = 0, p_t0 = g.prof ? clock64() : 0, nks = 0, p_hand = 0;
  unsigned long long p_ns0 = 0;
  if (g.prof) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(p_ns0));

  // the aux boxes of the tile at (m0, n0) land while its main loop runs; the ring is free once every thread has read the last
  // tile's boxes (the per-element tail) and the last stores have read them
  auto load_aux = [&](int m0, int n0) {
    wg_sync(1 + c);
    if (t == 0) {
      bulk_wait_read<0>();
      for (int b = 0; b < BN / 64 && n0 + 64 * b < g.N; ++b) {
        const uint32_t slot = (nbox + (uint32_t)b) & 1u;
        mbar_expect_tx(my_auxb + slot, OUT_BOX);
        tma_load_2d(ring + slot * OUT_BOX, &mapO2, n0 + 64 * b, m0 + 64 * c, my_auxb + slot);
      }
    }
  };

  // ---- epilogue of this thread's elements of the tile at (m0, n0): element (row r_lo + 8 h, column 8 j + cq + e) is
  // q[2 h + e] after fetch(j, q) ----
  auto epilogue = [&](int m0, int n0, auto &&fetch) {
    uint32_t rk[2] = {0u, 0u};
    if (EPI != EPI_WGRAD && g.t16) {
      rk[0] = attn::drop_row_key(seed, (unsigned long long)(m0 + r_lo));
      rk[1] = attn::drop_row_key(seed, (unsigned long long)(m0 + r_lo + 8));
    }
    // The operands the epilogue reads (bias, the saved activation of a dgrad) are loaded for JB column groups at once, before
    // any arithmetic uses them, at indices clamped into the tensor instead of behind bounds branches: a load behind a branch
    // cannot be issued early, so every one of them used to wait out its full latency.  Elements past the edge compute on the
    // clamped values and are never stored.
    constexpr int JB = 4;
#pragma unroll
    for (int jc = 0; jc < BN / 8; jc += JB) {
      // boxes that start at or past N are not staged, so the box holding column N - 1 is the last one of the tile
      if (tma_out && n0 + 8 * (jc - jc % box_j) >= g.N) break;
      if (tma_out && jc % box_j == 0) {
        if (aux_tma) {
          // this box's aux tile has landed in its slot (the slot was free when it was loaded)
          const uint32_t slot = nbox & 1u;
          mbar_wait(my_auxb + slot, (aux_ph >> slot) & 1u);
          aux_ph ^= 1u << slot;
        } else {
          // the slot(s) this box is staged in must have been read out by the TMA store that last used them
          if (t == 0) {
            if (g.out2 != nullptr) bulk_wait_read<0>();
            else bulk_wait_read<1>();
          }
          wg_sync(1 + c);
        }
      }
      const uint32_t box = ring + (g.out2 != nullptr ? (uint32_t)OUT_BOX : (nbox & 1u) * OUT_BOX);
      float bv[2 * JB], xv[2 * JB][2];
      uint32_t pre[2 * JB];   // tma_out with out2: the packed bf16 pre-activation of (jj, h)
      if (EPI == EPI_FWD && g.bias != nullptr) {
#pragma unroll
        for (int jj = 0; jj < JB; ++jj) {
          const int col = n0 + 8 * (jc + jj) + cq;
          bv[2 * jj] = __ldg(g.bias + min(col, g.N - 1));
          bv[2 * jj + 1] = __ldg(g.bias + min(col + 1, g.N - 1));
        }
      }
      if (EPI == EPI_DGRAD && g.act != 0) {
        if (aux_tma) {
          // the aux box has the layout the output box is written in: ldmatrix returns the accumulator's fragments
#pragma unroll
          for (int jj = 0; jj < JB; jj += 2) {
            const uint32_t a = sm_row + (((((uint32_t)(jc + jj) + sm_j) & 7u) ^ sm_x) << 4);
            uint32_t r[4];
            ldmatrix_x4(box + a, r[0], r[1], r[2], r[3]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {   // r[i] = (h i % 2, column group jj + i / 2)
              xv[2 * jj + i][0] = __uint_as_float(r[i] << 16);
              xv[2 * jj + i][1] = __uint_as_float(r[i] & 0xFFFF0000u);
            }
          }
        } else {
          const __nv_bfloat16 *ax = reinterpret_cast<const __nv_bfloat16 *>(g.aux);
#pragma unroll
          for (int jj = 0; jj < JB; ++jj) {
            const int col = n0 + 8 * (jc + jj) + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const size_t r = (size_t)min(m0 + r_lo + 8 * h, g.M - 1) * g.ld_aux;
              xv[2 * jj + h][0] = __bfloat162float(ax[r + min(col, g.N - 1)]);
              xv[2 * jj + h][1] = __bfloat162float(ax[r + min(col + 1, g.N - 1)]);
            }
          }
        }
      }
      float v[JB][4];   // the accumulators of column groups jc .. jc + JB - 1, then the values staged
#pragma unroll
      for (int jj = 0; jj < JB; ++jj) fetch(jc + jj, v[jj]);
#pragma unroll
      for (int jj = 0; jj < JB; ++jj) {
        const int j = jc + jj;
        const int col = n0 + 8 * j + cq;
        const bool c_ok = col < g.N, two = col + 1 < g.N;
        float mx0 = -INFINITY, mx1 = -INFINITY;   // rowmax: this thread's two rows
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + r_lo + 8 * h;
          float v0 = v[jj][2 * h], v1 = v[jj][2 * h + 1];
          if (EPI == EPI_FWD) {
            if (g.bias != nullptr) {
              v0 += bv[2 * jj];
              v1 += bv[2 * jj + 1];
            }
            if (g.out2 != nullptr) {
              if (tma_out) pre[2 * jj + h] = pack_bf16(v0, v1);
              else if (c_ok && row < g.M)
                store_pair_bf16(reinterpret_cast<__nv_bfloat16 *>(g.out2) + (size_t)row * g.ldo + col, two, (g.ldo & 1) == 0, v0, v1);
            }
            if (g.act == 1) {
              v0 = fmaxf(v0, 0.f);
              v1 = fmaxf(v1, 0.f);
            } else if (g.act == 2) {
              v0 = gelu_erf(v0);
              v1 = gelu_erf(v1);
            }
            if (g.t16) {
              const uint32_t hh = attn::drop_pair_hash(rk[h], (uint32_t)col >> 1);
              v0 = (hh & 0xFFFFu) >= g.t16 ? v0 * g.inv_keep : 0.f;
              v1 = (hh >> 16) >= g.t16 ? v1 * g.inv_keep : 0.f;
            }
            if (g.rowmax == 16) {
              mx0 = fmaxf(mx0, v0);
              mx1 = fmaxf(mx1, v1);
              continue;
            }
          } else if (EPI == EPI_DGRAD) {
            if (g.act != 0) {
              // multiply by the activation (+ dropout) derivative read from the saved forward tensor
              const float x0 = xv[2 * jj + h][0], x1 = xv[2 * jj + h][1];
              if (g.act == 1) {
                v0 = x0 > 0.f ? v0 * g.inv_keep : 0.f;
                v1 = x1 > 0.f ? v1 * g.inv_keep : 0.f;
              } else {
                float m0_ = 1.f, m1_ = 1.f;
                if (g.t16) {
                  const uint32_t hh = attn::drop_pair_hash(rk[h], (uint32_t)col >> 1);
                  m0_ = (hh & 0xFFFFu) >= g.t16 ? g.inv_keep : 0.f;
                  m1_ = (hh >> 16) >= g.t16 ? g.inv_keep : 0.f;
                }
                v0 *= gelu_grad(x0) * m0_;
                v1 *= gelu_grad(x1) * m1_;
              }
            }
          }
          if (tma_out) {   // staged below
            v[jj][2 * h] = v0;
            v[jj][2 * h + 1] = v1;
            continue;
          }
          if (!c_ok || row >= g.M) continue;
          if (EPI == EPI_WGRAD || g.out_f32) {
            float *o = reinterpret_cast<float *>(g.out) + (size_t)row * g.ldo + col;
            if (EPI == EPI_WGRAD && g.red_out) {
              atomicAdd(o, v0);
              if (two) atomicAdd(o + 1, v1);
            } else {
              const float *res = EPI == EPI_FWD ? reinterpret_cast<const float *>(g.residual) : nullptr;
              if (res != nullptr) {
                v0 += res[(size_t)row * g.ldo + col];
                if (two) v1 += res[(size_t)row * g.ldo + col + 1];
              }
              o[0] = v0;
              if (two) o[1] = v1;
            }
          } else {
            const __nv_bfloat16 *res = EPI == EPI_FWD ? reinterpret_cast<const __nv_bfloat16 *>(g.residual) : nullptr;
            if (res != nullptr) {
              v0 += __bfloat162float(res[(size_t)row * g.ldo + col]);
              if (two) v1 += __bfloat162float(res[(size_t)row * g.ldo + col + 1]);
            }
            store_pair_bf16(reinterpret_cast<__nv_bfloat16 *>(g.out) + (size_t)row * g.ldo + col, two, (g.ldo & 1) == 0, v0, v1);
          }
        }
        if (EPI == EPI_FWD && g.rowmax == 16) {
          // the 16 rows of a warp (r_lo and r_lo + 8 over the 8 lane quads) are one group of 16 consecutive rows = the 16
          // points of one cloud: max over this thread's two rows, then over the lane quads
          float a0 = mx0, a1 = mx1;
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            a0 = fmaxf(a0, __shfl_xor_sync(0xffffffffu, a0, o));
            a1 = fmaxf(a1, __shfl_xor_sync(0xffffffffu, a1, o));
          }
          const int grow0 = m0 + c * 64 + w * 16;   // first row of the group
          if (lane < 4 && c_ok && grow0 < g.M) {
            const size_t orow = (size_t)(grow0 >> 4);
            if (g.out_f32) {
              float *o = reinterpret_cast<float *>(g.out) + orow * g.ldo + col;
              o[0] = a0;
              if (two) o[1] = a1;
            } else {
              __nv_bfloat16 *o = reinterpret_cast<__nv_bfloat16 *>(g.out) + orow * g.ldo + col;
              o[0] = __float2bfloat16_rn(a0);
              if (two) o[1] = __float2bfloat16_rn(a1);
            }
          }
        }
      }
      if (tma_out) {
        if (f32_out) {
#pragma unroll
          for (int jj = 0; jj < JB; ++jj) {
            const int j = jc + jj;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t a = box + f_row + h * 1024u + ((((uint32_t)(2 * (j & 3)) + f_hi) ^ f_x) << 4) + f_lo;
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v[jj][2 * h]), "f"(v[jj][2 * h + 1]) : "memory");
            }
          }
        } else {
          // columns 8 j .. 8 j + 15 of the warp's 16 rows are four 8x8 matrices: (h 0, j), (h 1, j), (h 0, j + 1), (h 1, j + 1)
#pragma unroll
          for (int jj = 0; jj < JB; jj += 2) {
            const int j = jc + jj;
            const uint32_t a = sm_row + (((((uint32_t)j + sm_j) & 7u) ^ sm_x) << 4);
            stmatrix_x4(box + a, pack_bf16(v[jj][0], v[jj][1]), pack_bf16(v[jj][2], v[jj][3]),
                        pack_bf16(v[jj + 1][0], v[jj + 1][1]), pack_bf16(v[jj + 1][2], v[jj + 1][3]));
            if (EPI == EPI_FWD && g.out2 != nullptr)
              stmatrix_x4(ring + a, pre[2 * jj], pre[2 * jj + 1], pre[2 * jj + 2], pre[2 * jj + 3]);
          }
        }
        if ((jc + JB) % box_j == 0) {
          fence_proxy_async_smem();
          wg_sync(1 + c);
          const int cn = n0 + 8 * (jc + JB - box_j), cm = m0 + 64 * c;
          if (t == 0) {
            if (cn < g.n_tma && cm < g.M) {
              if (EPI == EPI_WGRAD) {
                tma_reduce_add_2d(&mapO, box, cn, cm);
              } else {
                tma_store_2d(&mapO, box, cn, cm);
                if (g.out2 != nullptr) tma_store_2d(&mapO2, ring, cn, cm);
              }
            }
            bulk_commit();
          }
          ++nbox;
        }
      }
    }
    if (tma_out && n0 + BN > g.n_tma && g.n_tma < g.N && m0 + 64 * c < g.M) {
      // columns [n_tma, N) are in the last box staged (still intact: the next acquire comes after a barrier)
      const int cn = n0 + ((g.N - 1 - n0) / (8 * box_j)) * 8 * box_j;
      const uint32_t last = ring + (g.out2 != nullptr ? (uint32_t)OUT_BOX : ((nbox - 1) & 1u) * OUT_BOX);
      store_tail(sOut + (last - smem_u32(sOut)), sOut + (ring - smem_u32(sOut)), g, EPI == EPI_WGRAD, f32_out, cn, m0 + 64 * c, t);
    }
  };

  if (epi_wg) {
    // ------------------------------- epilogue warpgroup c (EW) -------------------------------
    if constexpr (EW) {
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tt = item % n_tiles;
        const int tmi = g.n_fast ? tt / tiles_n : tt % tiles_m, tni = g.n_fast ? tt % tiles_n : tt / tiles_m;
        const int m0 = tmi * BM, n0 = tni * BN;
        if (m0 + 64 * c >= g.M) continue;   // no rows of this warpgroup: the MMA warpgroup hands nothing over
        if (aux_tma) load_aux(m0, n0);
        mbar_wait(hfull + c, hph);
        hph ^= 1u;
        const long long c0 = g.prof ? clock64() : 0;
        if (!(g.dbg & 1))
          epilogue(m0, n0, [&](int j, float (&q)[4]) {
            const float4 x = hand[j * 128 + t];
            q[0] = x.x; q[1] = x.y; q[2] = x.z; q[3] = x.w;
          });
        mbar_arrive(hempty + c);   // every read of the hand-off lies before this release
        if (g.prof) p_hand += clock64() - c0;
      }
      if (t == 0) bulk_wait_all();   // the staged boxes must stay readable until the last store has read them
      if (g.prof && t == 0 && c == 0) g.prof[(size_t)blockIdx.x * 16 + 10] = p_hand;
    }
    return;
  }

  if constexpr (Cfg::NREG) setmaxnreg_inc<Cfg::REG_MMA>();
  // A: 64 rows further into a K-major tile is 8 groups of 1024 B; in MN-major slabs it is the next slab (BK * 128 B)
  const uint32_t a_off = (uint32_t)c * 8192u;
  const uint32_t a_lbo = TA ? BK * 128 : 16, b_lbo = TB ? BK * 128 : 16;
  const uint32_t a_step = TA ? 2048u : 32u, b_step = TB ? 2048u : 32u;
  float acc[BN / 2];
  float accb[4];
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int tt = item % n_tiles, sp = item / n_tiles;
    const int tmi = g.n_fast ? tt / tiles_n : tt % tiles_m, tni = g.n_fast ? tt % tiles_n : tt / tiles_m;
    const int m0 = tmi * BM, n0 = tni * BN;
    const int ks0 = sp * kps, ks1 = min(k_steps, ks0 + kps);
    const bool bias_tile = with_bias_grad && n0 == 0;
    if (!EW && aux_tma && m0 + 64 * c < g.M) load_aux(m0, n0);
    uint32_t prev = 0;
    for (int ks = ks0; ks < ks1; ++ks, ++nks) {
      long long c0 = g.prof ? clock64() : 0;
      mbar_wait(full + s, ph);
      if (g.prof) p_full += clock64() - c0;
      const uint32_t a0 = smem_u32(sA + s * A_STAGE) + a_off, b0 = smem_u32(sB + s * B_STAGE);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint64_t da = desc_sw128(a0 + kk * a_step, a_lbo);
        const uint32_t sc = (ks > ks0 || kk > 0) ? 1u : 0u;
        mma<BN, TA, TB>(acc, da, desc_sw128(b0 + kk * b_step, b_lbo), sc);
        if (EPI == EPI_WGRAD) wgmma_n8<TA, 0>(accb, da, desc_sw128(smem_u32(sOnes) + kk * 32, 16), sc);
      }
      wgmma_commit();
      wgmma_wait<1>();      // the previous k-step's MMAs have read their slot: hand it back to the producer
      if (ks > ks0 && t == 0) mbar_arrive(empty + prev);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (EPI == EPI_WGRAD) fence_regs(accb);
    if (t == 0) mbar_arrive(empty + prev);
    if (m0 + 64 * c >= g.M) continue;   // no rows of this warpgroup to write
    if constexpr (EW) {
      // hand the fragment to epilogue warpgroup c once it has read the previous one (a fresh barrier passes parity 1 at once)
      const long long c0 = g.prof ? clock64() : 0;
      mbar_wait(hempty + c, hph ^ 1u);
      if (g.prof) p_hand += clock64() - c0;
      hph ^= 1u;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) hand[j * 128 + t] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
      mbar_arrive(hfull + c);
      continue;
    }
    if (g.dbg & 1) continue;
    epilogue(m0, n0, [&](int j, float (&q)[4]) {
#pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = acc[4 * j + i];
    });
    if (EPI == EPI_WGRAD && bias_tile && (lane & 3) == 0) {
      // every column of the N = 8 ones-product equals sum_k A[row][k]: the bias gradient of output feature `row`
      if (m0 + r_lo < g.M) atomicAdd(g.bias_grad + m0 + r_lo, accb[0]);
      if (m0 + r_lo + 8 < g.M) atomicAdd(g.bias_grad + m0 + r_lo + 8, accb[2]);
    }
  }
  if (!EW && tma_out && t == 0) bulk_wait_all();   // the staged boxes must stay readable until the last store has read them
  if (g.prof && t == 0 && c == 0) {
    // issue-loop cycles, of which waiting for operands, k-steps, start, end, ns, epilogue (0 per element, 1 staged), schedule
    // (0 cooperative, 1 epilogue warpgroups), cycles waiting for an empty hand-off; slot 10: the epilogue warpgroup's busy cycles
    long long *pp = g.prof + (size_t)blockIdx.x * 16;
    const long long t1 = clock64();
    unsigned long long ns1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns1));
    pp[0] = t1 - p_t0; pp[1] = p_full; pp[2] = 0; pp[3] = nks; pp[4] = p_t0; pp[5] = t1; pp[6] = (long long)(ns1 - p_ns0);
    pp[7] = OUT_TMA != 0; pp[8] = EW; pp[9] = p_hand;
  }
}

using attn::EncodeTiledFn;
using attn::encode_fn;

// row-major [rows, K] bf16 with leading dimension ld (elements); box = [box_rows x 64 elements], 128-byte swizzle
int make_map(CUtensorMap *map, const void *ptr, int rows, int K, int ld, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return SV_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};  // 64 bf16 = one 128-byte swizzle row
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SV_OK : SV_ERR_INVALID_ARG;
}

// [K, rows] bf16 row-major with leading dimension ld (the operand's rows are the contiguous direction): box = [BK x 64]
int make_map_mn(CUtensorMap *map, const void *ptr, int rows, int K, int ld) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return SV_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)rows, (cuuint64_t)K};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)BK};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SV_OK : SV_ERR_INVALID_ARG;
}

// row-major [rows, cols] output (bf16 or fp32) with leading dimension ld (elements): box = [64 rows x 128 bytes], the
// staging layout of the epilogue.  TMA writes nothing outside [rows, cols].
int make_out_map(CUtensorMap *map, void *ptr, int rows, int cols, int ld, bool f32) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return SV_ERR_CUDA;
  const int esz = f32 ? 4 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esz};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esz), 64};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, dims, strides, box,
                  es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SV_OK : SV_ERR_INVALID_ARG;
}

int device_sms(int *dev_out) {
  static int sms_of_dev[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 0;
  if (sms_of_dev[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    sms_of_dev[dev] = n;
  }
  *dev_out = dev;
  return sms_of_dev[dev];
}

template <int BN, int EPI, int TA, int TB, int OUT_TMA>
int launch_gemm(const CUtensorMap &ma, const CUtensorMap &mb, const CUtensorMap &mo, const CUtensorMap &mo2, const GemmArgs &g,
                cudaStream_t st) {
  using Cfg = GemmCfg<BN, EPI, OUT_TMA>;
  constexpr size_t smem = Cfg::SMEM;
  auto kern = gemm_kernel<BN, EPI, TA, TB, OUT_TMA>;
  static bool configured[64] = {false};
  int dev = 0;
  const int sms = device_sms(&dev);
  if (sms == 0) return SV_ERR_INVALID_ARG;
  if (!configured[dev]) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (rc) return rc;
    configured[dev] = true;
  }
  const int units = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN) * g.splits;
  const int grid = units < sms ? units : sms;
  kern<<<grid, Cfg::THREADS, smem, st>>>(ma, mb, mo, mo2, g);
  return sv::after_launch();
}

// Tile selection: the persistent grid runs ceil(tiles / SMs) waves of 128 x BN tiles, and one tile costs BN times a relative
// cost per output column measured for each width, direction and schedule (scripts/time_gemm_shapes.py at every forced width on
// the GPS step's shapes, one H100 80GB HBM3 at 700 W, DESIGN.md §4.1), relative to the cooperative 192-wide tile.  The 64-wide
// tiles re-load the 128-row A panel for every 64 columns; the weight gradient's 128-wide tiles leave less of their reduce-add
// epilogue exposed.  A staged forward or dgrad at 64 or 128 columns may run its epilogue in warpgroups of its own (ew) under the
// next tile's MMAs.  That hides every epilogue but a CTA's last, at the price of a shorter operand ring (the hand-off takes 32
// / 64 KB), so it is offered only where a CTA gets at least three tiles, and at K > 1024 (where an epilogue is a small share
// of a tile) only at 128 columns with at least six: elsewhere the cooperative kernel measured faster (the spatial-80, joint-130
// and BERT-50 ffn2 forwards and the joint-130 qkv / ffn1 dgrads, K = 2048-3072; the spatial-80 ffn1 dgrad with two tiles per
// CTA).
struct TilePick {
  int bn;
  bool ew;
};

float tile_cost(int epi, int bn, bool ew) {
  static const float rel[3][3] = {{1.18f, 1.02f, 1.0f}, {1.02f, 1.0f, 1.0f}, {1.52f, 0.76f, 1.0f}};   // [epi][64, 128, 192]
  static const float rel_ew[2][2] = {{0.85f, 0.75f}, {0.99f, 0.97f}};                                 // [fwd, dgrad][64, 128]
  return (ew ? rel_ew[epi][bn / 64 - 1] : rel[epi][bn / 64 - 1]) * (float)bn;
}

TilePick pick_tile(int M, int N, int K, int sms, int epi, bool staged, int force_bn, int force_sched) {
  const int ew_min_waves = K <= 1024 ? 3 : 6;
  const int cand[3] = {192, 128, 64};
  float best_cost = 1e30f;
  TilePick best{64, false};
  const int tm = (M + BM - 1) / BM;
  for (int i = 0; i < 3; ++i) {
    const int bn = cand[i];
    if (force_bn ? bn != force_bn : (bn > 64 && bn - 64 >= ((N + 63) / 64) * 64)) continue;   // wider than the problem
    const int tiles = tm * ((N + bn - 1) / bn), waves = (tiles + sms - 1) / sms;
    for (int ew = 1; ew >= 0; --ew) {
      if (ew && !(staged && epi != EPI_WGRAD && bn <= 128)) continue;
      if (force_sched ? (force_sched == 2) != (ew == 1) : (ew && (waves < ew_min_waves || (K > 1024 && bn == 64)))) continue;
      const float cost = (float)waves * tile_cost(epi, bn, ew != 0);
      if (cost < best_cost * 0.999f) {
        best_cost = cost;
        best = {bn, ew != 0};
      }
    }
  }
  if (best_cost == 1e30f) best = {force_bn ? force_bn : 64, false};   // a forced schedule the width cannot run
  return best;
}

template <int EPI, int TA, int TB>
int dispatch(TilePick tp, bool tma, const CUtensorMap &ma, const CUtensorMap &mb, const CUtensorMap &mo, const CUtensorMap &mo2,
             const GemmArgs &g, cudaStream_t st) {
  const int bn = tp.bn;
  if constexpr (EPI != EPI_WGRAD) {
    if (tma && tp.ew) {
      if (bn == 128) return launch_gemm<128, EPI, TA, TB, 2>(ma, mb, mo, mo2, g, st);
      if (bn == 64) return launch_gemm<64, EPI, TA, TB, 2>(ma, mb, mo, mo2, g, st);
    }
  }
  if (tma) {
    if (bn == 192) return launch_gemm<192, EPI, TA, TB, 1>(ma, mb, mo, mo2, g, st);
    if (bn == 128) return launch_gemm<128, EPI, TA, TB, 1>(ma, mb, mo, mo2, g, st);
    return launch_gemm<64, EPI, TA, TB, 1>(ma, mb, mo, mo2, g, st);
  }
  if (bn == 192) return launch_gemm<192, EPI, TA, TB, 0>(ma, mb, mo, mo2, g, st);
  if (bn == 128) return launch_gemm<128, EPI, TA, TB, 0>(ma, mb, mo, mo2, g, st);
  return launch_gemm<64, EPI, TA, TB, 0>(ma, mb, mo, mo2, g, st);
}

int g_force_bn = 0;     // tests / benchmarks: 1, 2 or 4 forces 64-, 128- or 192-column tiles, 0 = heuristic
int g_force_sched = 0;  // tests / benchmarks: staged forward / dgrad schedule, 1 cooperative, 2 epilogue warpgroups, 0 = heuristic
int g_gemm_dbg = 0;     // profiling only (bits 8.. of sv_gemm_force_ctas): results are garbage when set
long long *g_gemm_prof = nullptr;

int run_gemm(int epi, const void *A, int lda, int a_t, const void *B, int ldb, int b_t, GemmArgs &g, cudaStream_t st) {
  const int M = g.M, N = g.N, K = g.K;
  if (M < 0 || N < 0 || K < 0) return SV_ERR_INVALID_ARG;
  if (M == 0 || N == 0) return SV_OK;
  if (!A || !B || !g.out || K < 1 || (lda % 8) || (ldb % 8)) return SV_ERR_INVALID_ARG;
  if (a_t ? lda < M : lda < K) return SV_ERR_INVALID_ARG;   // K itself may be anything: TMA zero-fills past the extent
  if (b_t ? ldb < N : ldb < K) return SV_ERR_INVALID_ARG;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return SV_ERR_INVALID_ARG;
  int dev = 0;
  const int sms = device_sms(&dev);
  if (sms == 0) return SV_ERR_INVALID_ARG;
  // the operand with the SMALLER footprint is the one re-read across the in-flight tiles (it stays in L2); the larger one
  // is streamed from HBM exactly once
  g.n_fast = (long long)N <= (long long)M ? 1 : 0;
  g.dbg = g_gemm_dbg;
  g.prof = g_gemm_prof;
  // The epilogue goes out through shared memory by TMA whenever the output rows can take 16-byte-aligned boxes.  The output
  // maps span only the columns that fill whole 16-byte units (n_tma); the last few columns of a width like 607 or 30522 are
  // stored per element by the epilogue itself.  A TMA store clips a box at the map's inner dim only to 16-byte granularity
  // (on H100, N = 607 in bf16 wrote column 607), so a map of width N would write into the pad columns.  The SA3 row max, the
  // residual add and odd pitches keep the per-element stores.
  const int esz = epi == EPI_WGRAD || g.out_f32 ? 4 : 2;
  g.n_tma = (int)(((size_t)N * esz / 16) * 16 / esz);
  auto al16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool tma = g.rowmax == 0 && g.residual == nullptr && g.ldo >= N && ((size_t)g.ldo * esz) % 16 == 0 && g.n_tma > 0 &&
                   al16(g.out) && (g.out2 == nullptr || (esz == 2 && al16(g.out2)));
  const TilePick tp = pick_tile(M, N, K, sms, epi, tma, g_force_bn == 1 ? 64 : g_force_bn == 2 ? 128 : g_force_bn == 4 ? 192 : 0,
                                g_force_sched);
  const int bn = tp.bn;
  g.splits = 1;
  if (epi == EPI_WGRAD && g.red_out) {
    // split-K: the output of a weight gradient is small (a few dozen tiles), the contraction runs over every token
    const int tiles = ((M + BM - 1) / BM) * ((N + bn - 1) / bn), k_steps = (K + BK - 1) / BK;
    float best_eff = 0.f;
    for (int s = 1; s <= 32 && s * 4 <= k_steps; ++s) {
      const int kps = (k_steps + s - 1) / s;
      if ((s - 1) * kps >= k_steps) continue;  // an empty split
      const int items = tiles * s;
      const float eff = (float)items / (float)(((items + sms - 1) / sms) * sms) - 0.005f * s;
      if (eff > best_eff) {
        best_eff = eff;
        g.splits = s;
      }
    }
  }
  CUtensorMap ma, mb;
  int rc = a_t ? make_map_mn(&ma, A, M, K, lda) : make_map(&ma, A, M, K, lda, BM);
  if (rc) return rc;
  rc = b_t ? make_map_mn(&mb, B, N, K, ldb) : make_map(&mb, B, N, K, ldb, bn);
  if (rc) return rc;
  CUtensorMap mo{}, mo2{};
  if (tma) {
    rc = make_out_map(&mo, g.out, M, g.n_tma, g.ldo, esz == 4);
    if (rc) return rc;
    if (g.out2 != nullptr) {
      rc = make_out_map(&mo2, g.out2, M, g.n_tma, g.ldo, false);
      if (rc) return rc;
    }
    // A dgrad's saved activation is loaded by TMA into the bf16 output box its columns go out through, when its rows take
    // 16-byte-aligned boxes; loads zero-fill past [M, N], so its map spans all N columns.  Other pitches keep the loads per
    // element.
    g.aux_tma = epi == EPI_DGRAD && g.act != 0 && esz == 2 && al16(g.aux) && g.ld_aux >= N && ((size_t)g.ld_aux * 2) % 16 == 0;
    if (g.aux_tma) {
      rc = make_out_map(&mo2, const_cast<void *>(g.aux), M, N, g.ld_aux, false);
      if (rc) return rc;
    }
  }
  if (epi == EPI_FWD) {
    if (a_t)
      return b_t ? dispatch<EPI_FWD, 1, 1>(tp, tma, ma, mb, mo, mo2, g, st) : dispatch<EPI_FWD, 1, 0>(tp, tma, ma, mb, mo, mo2, g, st);
    return b_t ? dispatch<EPI_FWD, 0, 1>(tp, tma, ma, mb, mo, mo2, g, st) : dispatch<EPI_FWD, 0, 0>(tp, tma, ma, mb, mo, mo2, g, st);
  }
  if (epi == EPI_DGRAD && !a_t && b_t) return dispatch<EPI_DGRAD, 0, 1>(tp, tma, ma, mb, mo, mo2, g, st);
  if (epi == EPI_WGRAD && a_t && b_t) return dispatch<EPI_WGRAD, 1, 1>(tp, tma, ma, mb, mo, mo2, g, st);
  return SV_ERR_INVALID_ARG;
}

void set_dropout(GemmArgs &g, float p, unsigned long long seed) {
  g.t16 = attn::drop_threshold(p);
  g.inv_keep = 1.0f / (1.0f - p);
  g.seed = seed;
  g.seed_offset = sv::g_seed_offset;
}

}  // namespace

extern "C" int sv_gemm_profile(long long *buf) {
  g_gemm_prof = buf;
  return SV_OK;
}

extern "C" int sv_gemm_force_ctas(int ctas) {
  g_force_bn = ctas & 7;
  g_force_sched = (ctas >> 3) & 3;
  g_gemm_dbg = ctas >> 8;
  return SV_OK;
}

extern "C" int sv_gemm_bf16(const void *A, int lda, const void *B, int ldb, int M, int N, int K, const float *bias,
                            int act, const void *residual, void *out, int ldo, int out_f32, int rowmax, void *stream) {
  return sv_gemm_bf16_ex(A, lda, 0, B, ldb, 0, M, N, K, bias, act, residual, out, ldo, out_f32, rowmax, stream);
}

extern "C" int sv_gemm_bf16_ex(const void *A, int lda, int a_transposed, const void *B, int ldb, int b_transposed, int M,
                               int N, int K, const float *bias, int act, const void *residual, void *out, int ldo,
                               int out_f32, int rowmax, void *stream) {
  if (act < 0 || act > 2 || (rowmax != 0 && rowmax != 16) || (rowmax && residual)) return SV_ERR_INVALID_ARG;
  if (rowmax && (M % 16)) return SV_ERR_INVALID_ARG;
  GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.bias = bias; g.residual = residual; g.out = out; g.act = act; g.out_f32 = out_f32;
  g.rowmax = rowmax; g.ldo = ldo; g.inv_keep = 1.f;
  return run_gemm(EPI_FWD, A, lda, a_transposed, B, ldb, b_transposed, g, (cudaStream_t)stream);
}

extern "C" int sv_linear_fwd_bf16(const void *x, int ldx, const void *w, int ldw, int M, int N, int K, const float *bias,
                                  int act, float dropout_p, unsigned long long seed, void *out, int ldo, int out_f32,
                                  void *pre_out, void *stream) {
  if (act < 0 || act > 2 || !(dropout_p >= 0.f) || dropout_p >= 1.f) return SV_ERR_INVALID_ARG;
  GemmArgs g{};
  g.M = M; g.N = N; g.K = K; g.bias = bias; g.out = out; g.act = act; g.out_f32 = out_f32; g.ldo = ldo; g.out2 = pre_out;
  set_dropout(g, dropout_p, seed);
  return run_gemm(EPI_FWD, x, ldx, 0, w, ldw, 0, g, (cudaStream_t)stream);
}

extern "C" int sv_linear_dgrad_bf16(const void *gy, int ldg, const void *w, int ldw, int M, int N, int Kin, int dact,
                                    const void *aux, int ld_aux, float dropout_p, unsigned long long seed, void *dx, int ldx,
                                    int out_f32, void *stream) {
  // dx[M,Kin] = gy[M,N] . w[N,Kin]: contraction over N, the weight is the transposed (MN-major) B operand
  if (dact < 0 || dact > 2 || (dact && !aux) || !(dropout_p >= 0.f) || dropout_p >= 1.f) return SV_ERR_INVALID_ARG;
  GemmArgs g{};
  g.M = M; g.N = Kin; g.K = N; g.out = dx; g.act = dact; g.out_f32 = out_f32; g.ldo = ldx; g.aux = aux; g.ld_aux = ld_aux;
  set_dropout(g, dropout_p, seed);
  return run_gemm(EPI_DGRAD, gy, ldg, 0, w, ldw, 1, g, (cudaStream_t)stream);
}

extern "C" int sv_linear_wgrad_bf16(const void *gy, int ldg, const void *x, int ldx, int M, int N, int Kin, float *dw,
                                    int ld_dw, float *db, int accumulate, void *stream) {
  // dw[N,Kin] (+)= gy[M,N]^T . x[M,Kin]: contraction over the M tokens, both operands transposed in memory; db[N] (+)= column
  // sums of gy.  accumulate = 0: dw / db are overwritten (zero-filled here first, then reduced into by the split-K work list)
  if (M < 0 || N < 0 || Kin < 0) return SV_ERR_INVALID_ARG;
  if (N == 0 || Kin == 0) return SV_OK;
  if (!dw) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (!accumulate) {
    int rc = sv::cuda_status(cudaMemsetAsync(dw, 0, (size_t)N * ld_dw * sizeof(float), st));
    if (rc) return rc;
    if (db) {
      rc = sv::cuda_status(cudaMemsetAsync(db, 0, (size_t)N * sizeof(float), st));
      if (rc) return rc;
    }
  }
  if (M == 0) return SV_OK;
  GemmArgs g{};
  g.M = N; g.N = Kin; g.K = M; g.out = dw; g.out_f32 = 1; g.ldo = ld_dw; g.red_out = 1; g.bias_grad = db; g.inv_keep = 1.f;
  return run_gemm(EPI_WGRAD, gy, ldg, 1, x, ldx, 1, g, st);
}
