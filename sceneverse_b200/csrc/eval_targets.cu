// Evaluation targets of the grounding datasets (reference: data/datasets/base.py:387-454 with data/data_utils.py:63-72
// `convert_pc_to_box`, 194-234 `box3d_iou`, 266-277 `construct_bbox_corners`), one CTA per item.
//
// Box of an object: min / max of all its raw points (f32), centre = f32 (min + max) then halved, size = f32 (max - min).
// The IoU follows the reference's pinned numpy 1.26: every scalar step after the f32 sum and difference promotes to float64
// (np.float32 combined with a Python int or float), so the halving, the corners c +- s/2, the intersection, the volumes and
// the `+ 1e-8` are float64, each rounded once (__d*_rn: no contraction into an FMA).  Flags: iou >= 0.25, iou >= 0.5.
//
// Target = the LAST candidate with an IoU-25 hit (the reference's loop overwrites it), none if there is no hit.  gt mode
// (gt_index given): the caller's candidate is the target and its only hit, no IoU.
// Crop when n > O: (1) the IoU-25 hits (the last O of them if there are more), (2) candidates with the target label in
// index order until O are kept, (3) the rest drawn by a keyed permutation of the remaining candidates (hash of seed, item,
// candidate).  Kept candidates take slots in ascending candidate order; "no target" becomes tgt_object_id = n_kept.
#include "counter_hash.cuh"
#include "svcommon.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCand = 4096;  // per item; 6 bytes of shared memory each

__device__ __forceinline__ void warp_minmax(float *mn, float *mx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
      mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    }
}

__device__ __forceinline__ void range_minmax(const float *pts, long long beg, long long end, int lane, int stride,
                                             float *mn, float *mx) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    mn[k] = INFINITY;
    mx[k] = -INFINITY;
  }
  for (long long i = beg + lane; i < end; i += stride) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float v = pts[i * 6 + k];
      mn[k] = fminf(mn[k], v);
      mx[k] = fmaxf(mx[k], v);
    }
  }
}

// convert_pc_to_box -> construct_bbox_corners -> get_box3d_min_max, numpy 1.26 dtypes
__device__ __forceinline__ void corner_box(const float *mn, const float *mx, double *lo, double *hi) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double c = (double)__fadd_rn(mn[k], mx[k]) * 0.5;   // f32 sum; `/2` promotes, exact
    const double h = (double)__fsub_rn(mx[k], mn[k]) * 0.5;   // f32 size; `sx/2` promotes, exact
    const double a = __dadd_rn(h, c), b = __dadd_rn(-h, c);   // corners[k,:] + center[k]
    lo[k] = fmin(a, b);
    hi[k] = fmax(a, b);
  }
}

__device__ __forceinline__ double box_iou(const double *lo1, const double *hi1, const double *lo2, const double *hi2) {
  double inter = 1.0, v1 = 1.0, v2 = 1.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double d = fmax(__dsub_rn(fmin(hi1[k], hi2[k]), fmax(lo1[k], lo2[k])), 0.0);
    inter = k == 0 ? d : __dmul_rn(inter, d);
    v1 = k == 0 ? __dsub_rn(hi1[k], lo1[k]) : __dmul_rn(v1, __dsub_rn(hi1[k], lo1[k]));
    v2 = k == 0 ? __dsub_rn(hi2[k], lo2[k]) : __dmul_rn(v2, __dsub_rn(hi2[k], lo2[k]));
  }
  return __ddiv_rn(inter, __dadd_rn(__dsub_rn(__dadd_rn(v1, v2), inter), 1e-8));
}

constexpr unsigned char kHit25 = 1, kHit50 = 2, kKept = 4;

__global__ void __launch_bounds__(kThreads) grounding_targets_kernel(
    const float *__restrict__ pts, const long long *__restrict__ cand_off, const long long *__restrict__ item_off,
    const float *__restrict__ gt_pts, const long long *__restrict__ gt_off, const long long *__restrict__ gt_index,
    const long long *__restrict__ cand_labels, const long long *__restrict__ tgt_label, int O, int max_cand,
    unsigned long long seed, int *__restrict__ slot_map, long long *__restrict__ tgt_id, long long *__restrict__ iou25,
    long long *__restrict__ iou50, float *__restrict__ iou_out) {
  extern __shared__ unsigned char smem[];
  unsigned *skey = reinterpret_cast<unsigned *>(smem);
  unsigned char *sflag = smem + 4 * (size_t)max_cand;
  unsigned char *spick = sflag + max_cand;
  __shared__ float rmn[kWarps][3], rmx[kWarps][3];
  __shared__ double glo[3], ghi[3];
  __shared__ int s_tgt, s_need;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long c0 = item_off[b];
  const int n = (int)(item_off[b + 1] - c0);
  int *smap = slot_map + (long long)b * O;
  long long *r25 = iou25 + (long long)b * O, *r50 = iou50 + (long long)b * O;
  if (n < 0 || n > max_cand) {  // the caller's bound was wrong: an empty item, never stale memory
    for (int s = threadIdx.x; s < O; s += kThreads) {
      smap[s] = -1;
      r25[s] = r50[s] = 0;
    }
    if (threadIdx.x == 0) tgt_id[b] = 0;
    return;
  }
  if (!gt_index) {
    float mn[3], mx[3];
    range_minmax(gt_pts, gt_off[b], gt_off[b + 1], threadIdx.x, kThreads, mn, mx);
    warp_minmax(mn, mx);
    if (lane == 0)
      for (int k = 0; k < 3; ++k) {
        rmn[warp][k] = mn[k];
        rmx[warp][k] = mx[k];
      }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kWarps; ++w)
        for (int k = 0; k < 3; ++k) {
          rmn[0][k] = fminf(rmn[0][k], rmn[w][k]);
          rmx[0][k] = fmaxf(rmx[0][k], rmx[w][k]);
        }
      corner_box(rmn[0], rmx[0], glo, ghi);
    }
  }
  for (int c = threadIdx.x; c < n; c += kThreads) spick[c] = 0;
  __syncthreads();
  for (int c = warp; c < n; c += kWarps) {
    if (gt_index) {
      if (lane == 0) sflag[c] = c == gt_index[b] ? (kHit25 | kHit50) : 0;
      continue;
    }
    float mn[3], mx[3];
    range_minmax(pts, cand_off[c0 + c], cand_off[c0 + c + 1], lane, 32, mn, mx);
    warp_minmax(mn, mx);
    if (lane == 0) {
      double lo[3], hi[3];
      corner_box(mn, mx, lo, hi);
      const double iou = box_iou(lo, hi, glo, ghi);
      sflag[c] = (iou >= 0.25 ? kHit25 : 0) | (iou >= 0.5 ? kHit50 : 0);
      if (iou_out) iou_out[c0 + c] = (float)iou;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int tgt = -1, nhit = 0;
    for (int c = 0; c < n; ++c)
      if (sflag[c] & kHit25) {
        tgt = c;
        ++nhit;
      }
    int need = 0;
    if (n <= O) {
      for (int c = 0; c < n; ++c) sflag[c] |= kKept;
    } else {
      int kept = 0, skip = nhit > O ? nhit - O : 0;
      for (int c = 0; c < n; ++c)
        if (sflag[c] & kHit25) {
          if (skip > 0) {
            --skip;
          } else {
            sflag[c] |= kKept;
            ++kept;
          }
        }
      const long long tl = tgt_label[b];
      for (int c = 0; c < n && kept < O; ++c)
        if (!(sflag[c] & kKept) && cand_labels[c0 + c] == tl) {
          sflag[c] |= kKept;
          ++kept;
        }
      need = O - kept;
    }
    s_tgt = tgt;
    s_need = need;
  }
  __syncthreads();
  const int need = s_need;
  if (need > 0) {
    for (int c = threadIdx.x; c < n; c += kThreads) skey[c] = sv::hash_u32(seed, (unsigned long long)b, (unsigned long long)c);
    __syncthreads();
    for (int c = threadIdx.x; c < n; c += kThreads) {
      if (sflag[c] & kKept) continue;
      const unsigned kc = skey[c];
      int rank = 0;
      for (int d = 0; d < n && rank < need; ++d)
        if (!(sflag[d] & kKept) && (skey[d] < kc || (skey[d] == kc && d < c))) ++rank;
      spick[c] = rank < need;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int tgt = s_tgt;
    int s = 0;
    long long tslot = -1;
    for (int c = 0; c < n; ++c) {
      if (!((sflag[c] & kKept) || spick[c])) continue;
      if (c == tgt) tslot = s;
      smap[s] = c;
      r25[s] = (sflag[c] & kHit25) ? 1 : 0;
      r50[s] = (sflag[c] & kHit50) ? 1 : 0;
      ++s;
    }
    tgt_id[b] = tslot >= 0 ? tslot : s;
    for (int t = s; t < O; ++t) {
      smap[t] = -1;
      r25[t] = r50[t] = 0;
    }
  }
}

}  // namespace

extern "C" int sv_grounding_targets_f32(const float *points, const long long *cand_offsets, const long long *item_offsets,
                                        const float *gt_points, const long long *gt_offsets, const long long *gt_index,
                                        const long long *cand_labels, const long long *tgt_label, int B, int O, int max_cand,
                                        unsigned long long seed, int *slot_map, long long *tgt_object_id,
                                        long long *iou25, long long *iou50, float *iou_out, void *stream) {
  if (B < 1 || O < 1 || max_cand < 0 || max_cand > kMaxCand) return SV_ERR_INVALID_ARG;
  if (!cand_offsets || !item_offsets || !cand_labels || !tgt_label || !slot_map || !tgt_object_id || !iou25 || !iou50)
    return SV_ERR_INVALID_ARG;
  if (max_cand > 0 && !points) return SV_ERR_INVALID_ARG;
  if (!gt_index && (!gt_points || !gt_offsets)) return SV_ERR_INVALID_ARG;
  if (((uintptr_t)points % 4) || ((uintptr_t)gt_points % 4) || ((uintptr_t)cand_offsets % 8) ||
      ((uintptr_t)item_offsets % 8) || ((uintptr_t)gt_offsets % 8) || ((uintptr_t)gt_index % 8) ||
      ((uintptr_t)cand_labels % 8) || ((uintptr_t)tgt_label % 8) || ((uintptr_t)slot_map % 4) ||
      ((uintptr_t)tgt_object_id % 8) || ((uintptr_t)iou25 % 8) || ((uintptr_t)iou50 % 8) || ((uintptr_t)iou_out % 4))
    return SV_ERR_INVALID_ARG;
  const size_t smem = 6 * (size_t)(max_cand > 0 ? max_cand : 1);
  grounding_targets_kernel<<<B, kThreads, smem, (cudaStream_t)stream>>>(
      points, cand_offsets, item_offsets, gt_points, gt_offsets, gt_index, cand_labels, tgt_label, O, max_cand, seed,
      slot_map, tgt_object_id, iou25, iou50, iou_out);
  return sv::after_launch();
}
