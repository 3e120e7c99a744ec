// L2-normalise + all-gather in ONE kernel over NVLink peer memory — the exchange step of the batch-contrastive losses
// (reference: optim/loss/contra_loss.py:58-64,86-91: F.normalize on both embedding sets, then common/dist_utils.py
// all_gather = 2 x ncclAllGather of (B,768) + list allocations + torch.cat).
// Each rank normalises its rows and stores them straight into EVERY rank's symmetric buffer (P2P stores through
// NVLink / NVSwitch, slot = rank-major like the reference's concat order); the last CTA to finish publishes an epoch flag
// on every peer's signal pad and waits until all peers' flags reached the epoch, so when the kernel completes the
// gathered (world*B, D) matrices are resident locally — no NCCL call, no intermediate copies.
// Buffers are double-buffered by epoch parity (a rank can run at most one exchange ahead of the slowest one).
#include "svcommon.h"
#include "svgps.h"

namespace {

struct NagArgs {
  const float *a, *b;        // local rows (n, D) each
  float *const *peer_bufs;   // [world] device pointers: each buffer is [2 parities][2 tensors][world*n][D] floats
  unsigned *const *peer_sig; // [world] device pointers to signal words (flag[src_rank] at index src_rank)
  unsigned *done_counter;    // local, zero-initialised, reset by the last CTA
  int n, D, world, rank;
  unsigned *epoch_dev;       // device-resident epoch: this launch uses *epoch_dev + 1 and stores it back when done
};

__global__ void __launch_bounds__(256) norm_allgather_kernel(const NagArgs g) {
  __shared__ float red[8];
  __shared__ unsigned is_last, s_epoch;
  // a captured CUDA graph freezes by-value arguments, so the epoch can live on the device: every CTA reads it before it
  // arrives on the done counter, the last CTA advances it after the exchange
  if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned *>(g.epoch_dev) + 1u;
  __syncthreads();
  const unsigned epoch = s_epoch;
  const int row = blockIdx.x % g.n, t = blockIdx.x / g.n;  // t = 0: tensor a, 1: tensor b
  const float *x = (t ? g.b : g.a) + (size_t)row * g.D;
  float ss = 0.f;
  for (int j = threadIdx.x; j < g.D; j += 256) {
    const float v = x[j];
    ss += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);  // F.normalize(p=2, eps=1e-12)
  const size_t slot = (((size_t)(epoch & 1u) * 2 + t) * ((size_t)g.world * g.n) + (size_t)g.rank * g.n + row) * g.D;
  for (int p = 0; p < g.world; ++p) {
    float *dst = g.peer_bufs[p] + slot;
    for (int j = threadIdx.x; j < g.D; j += 256) dst[j] = x[j] * inv;
  }
  // publish: every thread's peer stores must be visible system-wide before the flag
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(g.done_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!is_last) return;
  if (threadIdx.x < g.world) {
    __threadfence_system();
    volatile unsigned *flag = g.peer_sig[threadIdx.x] + g.rank;
    *flag = epoch;  // my data for this epoch is in peer threadIdx.x's buffer
    volatile unsigned *mine = g.peer_sig[g.rank] + threadIdx.x;
    while (*mine < epoch) {
    }
    __threadfence_system();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *g.done_counter = 0u;
    *g.epoch_dev = epoch;
  }
}

}  // namespace

extern "C" int sv_normalize_allgather_dev_f32(const float *a, const float *b, int n, int D, void *const *peer_bufs,
                                              void *const *peer_signals, unsigned *done_counter, int world, int rank,
                                              unsigned *epoch_dev, void *stream) {
  if (n < 0 || D < 1 || world < 1 || world > 64 || rank < 0 || rank >= world) return SV_ERR_INVALID_ARG;
  if (n == 0) return SV_OK;
  if (!a || !b || !peer_bufs || !peer_signals || !done_counter || !epoch_dev) return SV_ERR_INVALID_ARG;
  NagArgs g{a, b, (float *const *)peer_bufs, (unsigned *const *)peer_signals, done_counter, n, D, world, rank, epoch_dev};
  norm_allgather_kernel<<<2 * n, 256, 0, (cudaStream_t)stream>>>(g);
  return sv::after_launch();
}
