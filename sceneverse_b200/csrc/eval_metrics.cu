// Evaluation metrics reduced on the GPU (reference: evaluator/scanrefer_eval.py, referit3d_eval.py, scanqa_eval.py,
// sqa3d_eval.py, objcls_eval.py, pretrain_eval.py `batch_metrics`), and the per-step train-log write.  Every kernel ADDS into one device
// counter vector per evaluator (float64 words, layouts in include/svgps.h), so an epoch of batches — a captured CUDA graph
// replayed once per batch — needs no host synchronisation; `record()` reads the vector once.  Counts are integers held
// exactly in float64 (below 2^53).  An item whose `valid` byte is 0 (padding of the last batch) counts nothing.
//
// argmax is torch's: the first maximum, NaN greater than every number (the first NaN wins).  The top-10 hit of a row is
// decided by rank: among equal scores the lower index ranks first (torch.topk leaves the order of ties unspecified).
#include <cuda_bf16.h>

#include "svcommon.h"
#include "svgps.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ float ld(const float *p, long long i) { return p[i]; }
__device__ __forceinline__ float ld(const __nv_bfloat16 *p, long long i) { return __bfloat162float(p[i]); }

// does (a, i) rank before (b, j)?  NaN first, then larger values, then the lower index
__device__ __forceinline__ bool before(float a, int i, float b, int j) {
  const bool na = isnan(a), nb = isnan(b);
  if (na || nb) return na && (!nb || i < j);
  return a > b || (a == b && i < j);
}

__device__ __forceinline__ void warp_best(float &v, int &i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    if (before(v2, i2, v, i)) {
      v = v2;
      i = i2;
    }
  }
}

// argmax of one row by one warp (the same index on every lane); n >= 1
template <typename T>
__device__ __forceinline__ int warp_argmax(const T *row, int n, int lane, long long stride = 1) {
  float v = -INFINITY;
  int i = 0x7fffffff;
  for (int j = lane; j < n; j += 32) {
    const float x = ld(row, j * stride);
    if (before(x, j, v, i)) {
      v = x;
      i = j;
    }
  }
  warp_best(v, i);
  return i;
}

__device__ __forceinline__ unsigned block_count(unsigned v, unsigned *red) {
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned r = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) r += red[w];
  return r;
}

struct GroundingArgs {
  const void *og;
  long long og_rs, og_cs;
  const long long *tgt_id;
  const long long *iou25, *iou50;
  long long iou_rs;
  const void *txt;
  long long txt_rs;
  int txt_c;
  const long long *tgt_label;
  const unsigned char *is_multiple, *is_hard, *is_view_dep, *valid;
  int B, O;
};

// one warp per item; per-CTA sums, then one atomic per counter
template <typename T, typename TT>
__global__ void __launch_bounds__(kThreads) grounding_kernel(GroundingArgs a, double *__restrict__ ctr) {
  __shared__ unsigned red[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kWarps + warp;
  unsigned c[SV_EVG_TXT_ACC + 1] = {};
  if (b < a.B && (!a.valid || a.valid[b])) {
    const int p = warp_argmax((const T *)a.og + b * a.og_rs, a.O, lane, a.og_cs);
    const bool mult = a.is_multiple && a.is_multiple[b], hard = a.is_hard && a.is_hard[b];
    const bool vdep = a.is_view_dep && a.is_view_dep[b];
    const bool ok = a.tgt_id[b] == p;
    c[SV_EVG_ITEMS] = 1;
    c[SV_EVG_MULTIPLE] = mult;
    c[SV_EVG_HARD] = hard;
    c[SV_EVG_VIEW_DEP] = vdep;
    c[SV_EVG_OG_ACC] = ok;
    c[SV_EVG_OG_ACC_HARD] = ok && hard;
    c[SV_EVG_OG_ACC_VIEW_DEP] = ok && vdep;
    if (a.iou25) {
      const bool h25 = a.iou25[b * a.iou_rs + p] != 0, h50 = a.iou50[b * a.iou_rs + p] != 0;
      c[SV_EVG_IOU25] = h25;
      c[SV_EVG_IOU50] = h50;
      c[SV_EVG_IOU25_MULTIPLE] = h25 && mult;
      c[SV_EVG_IOU50_MULTIPLE] = h50 && mult;
    }
    if (a.txt) c[SV_EVG_TXT_ACC] = warp_argmax((const TT *)a.txt + b * a.txt_rs, a.txt_c, lane) == a.tgt_label[b];
  }
#pragma unroll
  for (int k = 0; k <= SV_EVG_TXT_ACC; ++k) {
    const unsigned s = block_count(lane == 0 ? c[k] : 0u, red);
    if (threadIdx.x == 0 && s) atomicAdd(ctr + k, (double)s);
  }
}

struct ObjClsArgs {
  const void *logits[3];
  int bf16[3];
  long long row_stride[3], item_stride[3];
  int n, B, O, C;
  const long long *labels;
  const unsigned char *masks, *split, *valid;
};

// one warp per (item, object) row.  Without a split mask: hits of tensor t -> ctr[2t], masked rows -> ctr[2t + 1].  With
// one: tensor t owns ctr[6t .. 6t + 5], the (hits, rows) pairs over obj_masks, obj_masks & split, obj_masks & !split.
__global__ void __launch_bounds__(kThreads) obj_cls_kernel(ObjClsArgs a, double *__restrict__ ctr) {
  __shared__ unsigned red[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kWarps + warp;
  const int b = (int)(r / a.O), o = (int)(r % a.O);
  const bool live = r < (long long)a.B * a.O && a.masks[r] && (!a.valid || a.valid[b]);
  const bool in_split = live && a.split && a.split[r];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    if (t >= a.n) break;
    unsigned hit = 0;
    if (live) {
      const long long off = b * a.item_stride[t] + o * a.row_stride[t];
      const int p = a.bf16[t] ? warp_argmax((const __nv_bfloat16 *)a.logits[t] + off, a.C, lane)
                              : warp_argmax((const float *)a.logits[t] + off, a.C, lane);
      hit = lane == 0 && a.labels[r] == p;
    }
    const unsigned h = block_count(hit, red);
    const unsigned m = block_count(lane == 0 && live, red);
    if (!a.split) {
      if (threadIdx.x == 0) {
        if (h) atomicAdd(ctr + 2 * t, (double)h);
        if (m) atomicAdd(ctr + 2 * t + 1, (double)m);
      }
      continue;
    }
    const unsigned hs = block_count(hit && in_split, red);
    const unsigned ms = block_count(lane == 0 && in_split, red);
    if (threadIdx.x == 0) {
      double *c = ctr + 6 * t;
      const unsigned v[6] = {h, m, hs, ms, h - hs, m - ms};
#pragma unroll
      for (int k = 0; k < 6; ++k)
        if (v[k]) atomicAdd(c + k, (double)v[k]);
    }
  }
}

// masked-LM accuracy: one CTA per token row of (R, V) logits; rows whose label is -1 leave at once.  Labelled rows: hit when
// the argmax over the V real columns equals the label (pad columns past V are never read).  The first row of every valid
// item adds one item.  VEC: 16-byte loads (row pitch and base 16-byte aligned); the columns past V of the last vector are
// skipped, so a padded row's pad columns never take part.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads) lm_acc_kernel(const T *__restrict__ logits, long long rs, int V, int L,
                                                          const long long *__restrict__ labels,
                                                          const unsigned char *__restrict__ valid,
                                                          double *__restrict__ ctr) {
  __shared__ float sv[kWarps];
  __shared__ int si[kWarps];
  const long long r = blockIdx.x;
  if (valid && !valid[r / L]) return;
  if (threadIdx.x == 0 && r % L == 0) atomicAdd(ctr + SV_EVP_ITEMS, 1.0);
  const long long label = labels[r];
  if (label == -1) return;
  const T *row = logits + r * rs;
  float v = -INFINITY;
  int i = 0x7fffffff;
  if constexpr (VEC) {
    constexpr int W = 16 / sizeof(T);
    for (int j0 = threadIdx.x * W; j0 < V; j0 += kThreads * W) {
      const uint4 q = __ldg(reinterpret_cast<const uint4 *>(row + j0));
      float x[W];
      if constexpr (W == 8) {
        const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&q);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(h[k]);
          x[2 * k] = f.x, x[2 * k + 1] = f.y;
        }
      } else {
        x[0] = __uint_as_float(q.x), x[1] = __uint_as_float(q.y), x[2] = __uint_as_float(q.z), x[3] = __uint_as_float(q.w);
      }
#pragma unroll
      for (int k = 0; k < W; ++k)
        if (j0 + k < V && before(x[k], j0 + k, v, i)) v = x[k], i = j0 + k;
    }
  } else {
    for (int j = threadIdx.x; j < V; j += kThreads) {
      const float x = ld(row, j);
      if (before(x, j, v, i)) v = x, i = j;
    }
  }
  warp_best(v, i);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sv[warp] = v, si[warp] = i;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < kWarps; ++w)
      if (before(sv[w], si[w], v, i)) v = sv[w], i = si[w];
    if (i == label) atomicAdd(ctr + SV_EVP_LM_HIT, 1.0);
    atomicAdd(ctr + SV_EVP_LM_COUNT, 1.0);
  }
}

// one CTA per row of answer scores: top-1 and top-10 hits against the multi-hot label, per-type counts
template <typename T>
__global__ void __launch_bounds__(kThreads) answers_kernel(const T *__restrict__ scores, long long rs, int A,
                                                           const long long *__restrict__ label,
                                                           const long long *__restrict__ qtype,
                                                           const unsigned char *__restrict__ valid,
                                                           double *__restrict__ ctr) {
  __shared__ float sv[2][kWarps];
  __shared__ int si[2][kWarps];
  __shared__ unsigned red[kWarps];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (valid && !valid[b]) return;
  const T *row = scores + b * rs;
  const long long *lab = label + (long long)b * A;
  float va = -INFINITY, vp = -INFINITY;  // best of the row, best answer labelled 1
  int ia = 0x7fffffff, ip = 0x7fffffff;
  for (int j = threadIdx.x; j < A; j += kThreads) {
    const float x = ld(row, j);
    if (before(x, j, va, ia)) {
      va = x;
      ia = j;
    }
    if (lab[j] == 1 && before(x, j, vp, ip)) {
      vp = x;
      ip = j;
    }
  }
  warp_best(va, ia);
  warp_best(vp, ip);
  if (lane == 0) {
    sv[0][warp] = va, si[0][warp] = ia, sv[1][warp] = vp, si[1][warp] = ip;
  }
  __syncthreads();
  for (int w = 0; w < kWarps; ++w) {
    if (before(sv[0][w], si[0][w], va, ia)) va = sv[0][w], ia = si[0][w];
    if (before(sv[1][w], si[1][w], vp, ip)) vp = sv[1][w], ip = si[1][w];
  }
  const bool any = ip != 0x7fffffff;
  // rank of the best labelled answer = the answers ranked before it
  unsigned ahead = 0;
  if (any)
    for (int j = threadIdx.x; j < A; j += kThreads) ahead += before(ld(row, j), j, vp, ip);
  ahead = block_count(ahead, red);
  if (threadIdx.x == 0) {
    const bool h1 = any && ia == ip, h10 = any && ahead < 10;
    atomicAdd(ctr + SV_EVA_ITEMS, 1.0);
    if (h1) atomicAdd(ctr + SV_EVA_ANS1, 1.0);
    if (h10) atomicAdd(ctr + SV_EVA_ANS10, 1.0);
    if (qtype) {
      const long long t = qtype[b];
      if (t >= 0 && t < SV_EVA_NTYPES) {
        atomicAdd(ctr + SV_EVA_TYPE_ITEMS + t, 1.0);
        if (h1) atomicAdd(ctr + SV_EVA_TYPE_ANS1 + t, 1.0);
      }
    }
  }
}

// SQA3DEval.update after one batch, in its float64 arithmetic and order: the batch is the difference of the integer
// counters and their snapshot.  One thread: the sums run in batch order, as Python's sum() does.
__global__ void sqa3d_batch_kernel(double *__restrict__ ctr) {
  double *snap = ctr + SV_EVA_SNAPSHOT;
  const double n = ctr[SV_EVA_ITEMS] - snap[SV_EVA_ITEMS];
  if (n > 0.0) {
    const double c1 = ctr[SV_EVA_ANS1] - snap[SV_EVA_ANS1], c10 = ctr[SV_EVA_ANS10] - snap[SV_EVA_ANS10];
    const double hit = ctr[SV_EVA_OBJ_HIT] - snap[SV_EVA_OBJ_HIT], cnt = ctr[SV_EVA_OBJ_COUNT] - snap[SV_EVA_OBJ_COUNT];
    // metrics[k] * batch_count, summed over batches
    ctr[SV_EVA_Q_ANS1] = __dadd_rn(ctr[SV_EVA_Q_ANS1], __dmul_rn(__ddiv_rn(c1, n), n));
    ctr[SV_EVA_Q_ANS10] = __dadd_rn(ctr[SV_EVA_Q_ANS10], __dmul_rn(__ddiv_rn(c10, n), n));
    if (cnt > 0.0) ctr[SV_EVA_Q_OBJ] = __dadd_rn(ctr[SV_EVA_Q_OBJ], __dmul_rn(__ddiv_rn(hit, cnt), n));
    for (int t = 0; t < SV_EVA_NTYPES; ++t) {
      const double nt = ctr[SV_EVA_TYPE_ITEMS + t] - snap[SV_EVA_TYPE_ITEMS + t];
      const double ct = ctr[SV_EVA_TYPE_ANS1 + t] - snap[SV_EVA_TYPE_ANS1 + t];
      double count = 1e-10;  // count_type starts at 1e-10 and adds 1 per item
      for (double i = 0.0; i < nt; i += 1.0) count = __dadd_rn(count, 1.0);
      ctr[SV_EVA_Q_TYPE + t] = __dadd_rn(ctr[SV_EVA_Q_TYPE + t], __dmul_rn(__ddiv_rn(ct, count), count));
      ctr[SV_EVA_Q_TYPE_COUNT + t] = __dadd_rn(ctr[SV_EVA_Q_TYPE_COUNT + t], count);
    }
  }
  for (int k = 0; k < SV_EVA_SNAPSHOT; ++k) snap[k] = ctr[k];
}

// PretrainEval.batch_metrics + update for the batch just added, in its float64 arithmetic and order: og_acc = hits / items,
// every other accuracy hits / (count + 1e-8); target_metric = their sum in key order / their number; each sum gains
// metric x items.  The batch is the difference of the integer counters and their snapshot.  One thread.
__global__ void pretrain_batch_kernel(double *__restrict__ ctr, int present) {
  double *snap = ctr + SV_EVP_SNAPSHOT, *q = ctr + SV_EVP_Q;
  const double n = ctr[SV_EVP_ITEMS] - snap[SV_EVP_ITEMS];
  if (n > 0.0) {
    double sum = 0.0;
    int keys = 0;
    auto put = [&](int k, double v) {
      q[k] = __dadd_rn(q[k], __dmul_rn(v, n));
      sum = __dadd_rn(sum, v);
      ++keys;
    };
    auto acc = [&](int hit) {
      return __ddiv_rn(ctr[hit] - snap[hit], __dadd_rn(ctr[hit + 1] - snap[hit + 1], 1e-8));
    };
    if (present & SV_EVP_HAS_OG)
      put(SV_EVP_Q_OG, __ddiv_rn(ctr[SV_EVP_OG + SV_EVG_OG_ACC] - snap[SV_EVP_OG + SV_EVG_OG_ACC], n));
    put(SV_EVP_Q_LM, acc(SV_EVP_LM_HIT));
    int t = SV_EVP_OBJ;
    if (present & SV_EVP_HAS_POST) {
      put(SV_EVP_Q_POST, acc(t));
      put(SV_EVP_Q_POST_UNMASK, acc(t + 2));
      put(SV_EVP_Q_POST_MASK, acc(t + 4));
      t += 6;
    }
    if (present & SV_EVP_HAS_RAW) {
      put(SV_EVP_Q_RAW, acc(t));
      t += 6;
    }
    if (present & SV_EVP_HAS_PRE) {
      put(SV_EVP_Q_PRE, acc(t));
      put(SV_EVP_Q_PRE_UNMASK, acc(t + 2));
      put(SV_EVP_Q_PRE_MASK, acc(t + 4));
    }
    q[SV_EVP_Q_TARGET] = __dadd_rn(q[SV_EVP_Q_TARGET], __dmul_rn(__ddiv_rn(sum, (double)keys), n));
  }
  for (int k = 0; k < SV_EVP_SNAPSHOT; ++k) snap[k] = ctr[k];
}

struct LogValues {
  const float *v[SV_TRAIN_LOG_MAX_VALUES];
};

// one train-log entry: ring row (step % slots) = [step, values..., counters...]
__global__ void train_log_kernel(LogValues vals, int nv, const double *__restrict__ ctr, int nc, long long *step, int advance,
                                 double *__restrict__ ring, int slots) {
  __shared__ long long s;
  if (threadIdx.x == 0) {
    long long k = *step;
    if (advance) *step = ++k;
    s = k;
  }
  __syncthreads();
  double *row = ring + (s % slots) * (long long)(1 + nv + nc);
  if (threadIdx.x == 0) row[0] = (double)s;
#pragma unroll
  for (int k = 0; k < SV_TRAIN_LOG_MAX_VALUES; ++k)
    if (k < nv && threadIdx.x == k) row[1 + k] = (double)*vals.v[k];
  for (int j = threadIdx.x; j < nc; j += blockDim.x) row[1 + nv + j] = ctr[j];
}

bool al(const void *p, uintptr_t a) { return ((uintptr_t)p % a) == 0; }

}  // namespace

extern "C" int sv_eval_counters_size(int kind) {
  switch (kind) {
    case SV_EVAL_GROUNDING: return SV_EVG_SIZE;
    case SV_EVAL_OBJ_CLS: return SV_EVO_SIZE;
    case SV_EVAL_ANSWERS: return SV_EVA_SIZE;
    case SV_EVAL_PRETRAIN: return SV_EVP_SIZE;
    default: return 0;
  }
}

extern "C" int sv_eval_grounding(const void *og3d_logits, int og_bf16, long long og_row_stride, long long og_col_stride,
                                 int B, int O,
                                 const long long *tgt_object_id, const long long *iou25, const long long *iou50,
                                 long long iou_row_stride, const void *txt_cls_logits, int txt_bf16, long long txt_row_stride,
                                 int txt_classes, const long long *tgt_object_label, const unsigned char *is_multiple,
                                 const unsigned char *is_hard, const unsigned char *is_view_dependent,
                                 const unsigned char *valid, double *counters, void *stream) {
  if (B < 1 || O < 1 || og_col_stride < 1 || og_row_stride < (long long)(O - 1) * og_col_stride + 1 || !og3d_logits || !tgt_object_id || !counters) return SV_ERR_INVALID_ARG;
  if (!iou25 != !iou50 || (iou25 && iou_row_stride < O)) return SV_ERR_INVALID_ARG;
  if (txt_cls_logits && (txt_classes < 1 || txt_row_stride < txt_classes || !tgt_object_label)) return SV_ERR_INVALID_ARG;
  const uintptr_t oe = og_bf16 ? 2 : 4, te = txt_bf16 ? 2 : 4;
  if (!al(og3d_logits, oe) || !al(txt_cls_logits, te) || !al(tgt_object_id, 8) || !al(iou25, 8) || !al(iou50, 8) ||
      !al(tgt_object_label, 8) || !al(counters, 8))
    return SV_ERR_INVALID_ARG;
  GroundingArgs a{og3d_logits, og_row_stride, og_col_stride, tgt_object_id, iou25, iou50, iou_row_stride, txt_cls_logits, txt_row_stride,
                  txt_classes, tgt_object_label, is_multiple, is_hard, is_view_dependent, valid, B, O};
  const int grid = (B + kWarps - 1) / kWarps;
  cudaStream_t st = (cudaStream_t)stream;
  if (og_bf16 && txt_bf16) grounding_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, kThreads, 0, st>>>(a, counters);
  else if (og_bf16) grounding_kernel<__nv_bfloat16, float><<<grid, kThreads, 0, st>>>(a, counters);
  else if (txt_bf16) grounding_kernel<float, __nv_bfloat16><<<grid, kThreads, 0, st>>>(a, counters);
  else grounding_kernel<float, float><<<grid, kThreads, 0, st>>>(a, counters);
  return sv::after_launch();
}

extern "C" int sv_eval_obj_cls(int n_logits, const void *const *logits, const int *is_bf16, const long long *row_stride,
                               const long long *item_stride, int B, int O, int C, const long long *obj_labels,
                               const unsigned char *obj_masks, const unsigned char *split_mask, const unsigned char *valid,
                               double *counters, void *stream) {
  if (n_logits < 1 || n_logits > 3 || B < 1 || O < 1 || C < 1 || !logits || !is_bf16 || !row_stride || !item_stride ||
      !obj_labels || !obj_masks || !counters || !al(obj_labels, 8) || !al(counters, 8))
    return SV_ERR_INVALID_ARG;
  ObjClsArgs a{};
  for (int t = 0; t < n_logits; ++t) {
    if (!logits[t] || !al(logits[t], is_bf16[t] ? 2 : 4) || row_stride[t] < C ||
        item_stride[t] < (long long)(O - 1) * row_stride[t] + C)
      return SV_ERR_INVALID_ARG;
    a.logits[t] = logits[t];
    a.bf16[t] = is_bf16[t] != 0;
    a.row_stride[t] = row_stride[t];
    a.item_stride[t] = item_stride[t];
  }
  a.n = n_logits, a.B = B, a.O = O, a.C = C, a.labels = obj_labels, a.masks = obj_masks, a.split = split_mask, a.valid = valid;
  const long long rows = (long long)B * O;
  obj_cls_kernel<<<(unsigned)((rows + kWarps - 1) / kWarps), kThreads, 0, (cudaStream_t)stream>>>(a, counters);
  return sv::after_launch();
}

extern "C" int sv_eval_answers(const void *answer_scores, int is_bf16, long long row_stride, int B, int A,
                               const long long *answer_label, const long long *sqa_type, const unsigned char *valid,
                               double *counters, void *stream) {
  if (B < 1 || A < 1 || row_stride < A || !answer_scores || !answer_label || !counters) return SV_ERR_INVALID_ARG;
  if (!al(answer_scores, is_bf16 ? 2 : 4) || !al(answer_label, 8) || !al(sqa_type, 8) || !al(counters, 8))
    return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (is_bf16)
    answers_kernel<__nv_bfloat16><<<B, kThreads, 0, st>>>((const __nv_bfloat16 *)answer_scores, row_stride, A, answer_label,
                                                          sqa_type, valid, counters);
  else
    answers_kernel<float><<<B, kThreads, 0, st>>>((const float *)answer_scores, row_stride, A, answer_label, sqa_type, valid,
                                                  counters);
  return sv::after_launch();
}

extern "C" int sv_eval_sqa3d_batch(double *counters, void *stream) {
  if (!counters || !al(counters, 8)) return SV_ERR_INVALID_ARG;
  sqa3d_batch_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counters);
  return sv::after_launch();
}

extern "C" int sv_eval_lm_acc(const void *logits, int is_bf16, long long row_stride, long long R, int V, int L,
                              const long long *masked_lm_labels, const unsigned char *valid, double *counters, void *stream) {
  if (R < 1 || V < 1 || L < 1 || R % L || row_stride < V || !logits || !masked_lm_labels || !counters) return SV_ERR_INVALID_ARG;
  if (R > 0x7fffffffLL || !al(logits, is_bf16 ? 2 : 4) || !al(masked_lm_labels, 8) || !al(counters, 8)) return SV_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int es = is_bf16 ? 2 : 4;
  const bool vec = al(logits, 16) && (row_stride * es) % 16 == 0;
  const unsigned grid = (unsigned)R;
  if (is_bf16) {
    const __nv_bfloat16 *p = (const __nv_bfloat16 *)logits;
    if (vec) lm_acc_kernel<__nv_bfloat16, true><<<grid, kThreads, 0, st>>>(p, row_stride, V, L, masked_lm_labels, valid, counters);
    else lm_acc_kernel<__nv_bfloat16, false><<<grid, kThreads, 0, st>>>(p, row_stride, V, L, masked_lm_labels, valid, counters);
  } else {
    const float *p = (const float *)logits;
    if (vec) lm_acc_kernel<float, true><<<grid, kThreads, 0, st>>>(p, row_stride, V, L, masked_lm_labels, valid, counters);
    else lm_acc_kernel<float, false><<<grid, kThreads, 0, st>>>(p, row_stride, V, L, masked_lm_labels, valid, counters);
  }
  return sv::after_launch();
}

extern "C" int sv_eval_pretrain_batch(double *counters, int present, void *stream) {
  if (!counters || !al(counters, 8) || (present & ~(SV_EVP_HAS_OG | SV_EVP_HAS_POST | SV_EVP_HAS_RAW | SV_EVP_HAS_PRE)))
    return SV_ERR_INVALID_ARG;
  pretrain_batch_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counters, present);
  return sv::after_launch();
}

extern "C" int sv_train_log_write(int n_values, const float *const *values, const double *counters, int n_counters,
                                  long long *step, int advance_step, double *ring, int slots, void *stream) {
  if (n_values < 0 || n_values > SV_TRAIN_LOG_MAX_VALUES || n_counters < 0 || slots < 1 || !step || !ring ||
      (n_values && !values) || (n_counters && !counters) || !al(step, 8) || !al(ring, 8) || !al(counters, 8))
    return SV_ERR_INVALID_ARG;
  LogValues v{};
  for (int k = 0; k < n_values; ++k) {
    if (!values[k] || !al(values[k], 4)) return SV_ERR_INVALID_ARG;
    v.v[k] = values[k];
  }
  train_log_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(v, n_values, counters, n_counters, step, advance_step, ring, slots);
  return sv::after_launch();
}
