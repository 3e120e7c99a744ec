// Device-side input pipeline of the GPS data path (SURVEY.md §8 f2): what the reference does per object and per token in
// numpy / Python loops on the dataloader workers, as two kernels that build the model's `data_dict` tensors on the GPU
// from ragged raw scene data.
//   scene_prep_kernel  (reference: data/datasets/base.py:697-741 `_obj_processing_post` + dataset_wrapper.py:62-72 padding)
//     per object slot: obj_locs = [mean xyz, max - min] of the RAW points; subsample to P points — without replacement when
//     the object has >= P points, with replacement otherwise (np.random.choice(n, P, replace=n < P)); centre the SAMPLED
//     points on their mean, divide by their max norm (1 when < 1e-6); colours pass through; empty slots become all-ones
//     points, zero locs, mask 0.
//   token_mask_kernel  (reference: data/data_utils.py:76-121 `random_word`, `random_point_cloud`)
//     BERT masked-LM corruption of the caption (15 %: 80 % [MASK], 10 % random id, 10 % kept; label = original id, else -1)
//     and the object "semantic mask" coin flips.
// Randomness is a counter hash of (seed, slot / token, k): reproducible, order-independent, nothing stored.  Sampling
// without replacement is a keyed bijection of [0, 2^b) (xor / odd-multiply / xorshift rounds) with cycle walking onto [0, n):
// the first P images of 0..P-1 are P distinct uniform indices — no sort, no rejection table.
#include "counter_hash.cuh"
#include "svcommon.h"

namespace {

using sv::hash_u32;
// bijection of [0, 2^bits) keyed by (k1, k2, k3); bits >= 1
__device__ __forceinline__ unsigned perm_pow2(unsigned x, int bits, unsigned k1, unsigned k2, unsigned k3) {
  const unsigned mask = bits >= 32 ? 0xffffffffu : ((1u << bits) - 1u);
  const int sh = bits > 1 ? bits / 2 : 1;
  x = ((x ^ k1) * 0x9E3779B1u) & mask;
  x ^= x >> sh;
  x = ((x ^ k2) * 0x85EBCA6Bu) & mask;
  x ^= x >> sh;
  x = ((x ^ k3) * 0xC2B2AE35u) & mask;
  x ^= x >> sh;
  return x & mask;
}

struct PrepArgs {
  const float *raw;            // (total, 6) xyz rgb
  const long long *offsets;    // (S + 1) CSR over object slots; an empty range = padded slot
  int S, P;
  unsigned long long seed;
  float *fts;                  // (S, P, 6)
  float *locs;                 // (S, 6)
  unsigned char *masks;        // (S) 1 = real object
  int *sample_idx;             // (S, P) or null: the chosen raw indices (tests)
  int slots_per_item;
  const int *quarter_turns;    // (S / slots_per_item) or null: x @ R^T per item, theta = k pi / 2
  const int *index_in;         // (S, P) or null: given raw indices instead of drawn ones
  float *boxes;                // (S, 6) or null
};

__device__ __forceinline__ double block_sum(double v, double *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}
__device__ __forceinline__ float block_max(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmaxf(t, red[w]);
  return t;
}

// x @ R^T for R = [[c, -s, 0], [s, c, 0], [0, 0, 1]] in f32, summed in the order of numpy's matmul loop
struct QuarterTurn {
  float c, s;
  __device__ __forceinline__ void apply(float &x, float &y, float &z) const {
    const float x0 = x, y0 = y, z0 = z;
    x = __fadd_rn(__fadd_rn(__fmul_rn(x0, c), __fmul_rn(y0, -s)), __fmul_rn(z0, 0.f));
    y = __fadd_rn(__fadd_rn(__fmul_rn(x0, s), __fmul_rn(y0, c)), __fmul_rn(z0, 0.f));
    z = __fadd_rn(__fadd_rn(__fmul_rn(x0, 0.f), __fmul_rn(y0, 0.f)), __fmul_rn(z0, 1.f));
  }
};
// data/data_utils.py:168-176: theta from [0, pi/2, pi, 3 pi/2], np.cos / np.sin of the f64 angle rounded to f32 (so the
// "zero" entries are +-6.1e-17 / 1.2e-16 / -1.8e-16, as in the reference's matrix)
__device__ __forceinline__ QuarterTurn quarter_turn(int k) {
  return k == 1 ? QuarterTurn{(float)6.123233995736766e-17, 1.f}
       : k == 2 ? QuarterTurn{-1.f, (float)1.2246467991473532e-16}
                : QuarterTurn{(float)-1.8369701987210297e-16, -1.f};
}

// `_obj_processing_post` per object slot, with an optional per-item quarter turn of the raw points, optional given indices and
// optional boxes.
__global__ void __launch_bounds__(256) scene_prep_kernel(const PrepArgs a) {
  extern __shared__ __align__(16) float pts[];   // [P][6] sampled points
  __shared__ double redd[8];
  __shared__ float redf[8];
  const int s = blockIdx.x, tid = threadIdx.x;
  const long long beg = a.offsets[s], n = a.offsets[s + 1] - beg;
  float *out = a.fts + (size_t)s * a.P * 6;
  if (n <= 0) {   // padded slot: all-ones points (dataset_wrapper.py:62-64), zero locs, mask 0
    for (int i = tid; i < a.P * 6; i += 256) out[i] = 1.0f;
    if (tid < 6) a.locs[(size_t)s * 6 + tid] = 0.f;
    if (a.boxes != nullptr && tid < 6) a.boxes[(size_t)s * 6 + tid] = 0.f;
    if (tid == 0) a.masks[s] = 0;
    if (a.sample_idx != nullptr)
      for (int i = tid; i < a.P; i += 256) a.sample_idx[(size_t)s * a.P + i] = -1;
    return;
  }
  const float *raw = a.raw + (size_t)beg * 6;
  bool rot = false;
  QuarterTurn R{1.f, 0.f};
  if (a.quarter_turns != nullptr) {
    const int k = a.quarter_turns[s / a.slots_per_item] & 3;
    rot = k != 0;   // theta = 0: build_rotate_mat returns None, the points are left as they are
    if (rot) R = quarter_turn(k);
  }
  // ---- obj_locs from ALL raw points: centre = mean, size = max - min --------------------------------------------------------
  double sx = 0, sy = 0, sz = 0;
  float mnx = INFINITY, mny = INFINITY, mnz = INFINITY, mxx = -INFINITY, mxy = -INFINITY, mxz = -INFINITY;
  for (long long i = tid; i < n; i += 256) {
    float x = raw[i * 6], y = raw[i * 6 + 1], z = raw[i * 6 + 2];
    if (rot) R.apply(x, y, z);
    sx += x; sy += y; sz += z;
    mnx = fminf(mnx, x); mny = fminf(mny, y); mnz = fminf(mnz, z);
    mxx = fmaxf(mxx, x); mxy = fmaxf(mxy, y); mxz = fmaxf(mxz, z);
  }
  sx = block_sum(sx, redd); sy = block_sum(sy, redd); sz = block_sum(sz, redd);
  mxx = block_max(mxx, redf); mxy = block_max(mxy, redf); mxz = block_max(mxz, redf);
  mnx = -block_max(-mnx, redf); mny = -block_max(-mny, redf); mnz = -block_max(-mnz, redf);
  if (tid == 0) {
    float *l = a.locs + (size_t)s * 6;
    l[0] = (float)(sx / (double)n); l[1] = (float)(sy / (double)n); l[2] = (float)(sz / (double)n);
    l[3] = mxx - mnx; l[4] = mxy - mny; l[5] = mxz - mnz;
    if (a.boxes != nullptr) {   // base.py:714-718: box centre = (max + min) / 2, size = max - min
      float *bx = a.boxes + (size_t)s * 6;
      bx[0] = (mxx + mnx) / 2; bx[1] = (mxy + mny) / 2; bx[2] = (mxz + mnz) / 2;
      bx[3] = l[3]; bx[4] = l[4]; bx[5] = l[5];
    }
    a.masks[s] = 1;
  }
  // ---- subsample P points --------------------------------------------------------------------------------------------------
  int bits = 1;
  while ((1ll << bits) < n) ++bits;
  const unsigned k1 = hash_u32(a.seed, (unsigned long long)s, 1), k2 = hash_u32(a.seed, (unsigned long long)s, 2),
                 k3 = hash_u32(a.seed, (unsigned long long)s, 3);
  double cx = 0, cy = 0, cz = 0;
  for (int k = tid; k < a.P; k += 256) {
    long long idx;
    if (a.index_in != nullptr) {
      idx = a.index_in[(size_t)s * a.P + k];
    } else if (n < a.P) {   // with replacement
      idx = (long long)(((unsigned long long)hash_u32(a.seed, (unsigned long long)s, 16 + (unsigned long long)k) * (unsigned long long)n) >> 32);
    } else {         // without replacement: image of k under a keyed permutation of [0, n)
      unsigned x = perm_pow2((unsigned)k, bits, k1, k2, k3);
      while ((long long)x >= n) x = perm_pow2(x, bits, k1, k2, k3);
      idx = x;
    }
    if (a.sample_idx != nullptr) a.sample_idx[(size_t)s * a.P + k] = (int)idx;
    const float *p = raw + idx * 6;
#pragma unroll
    for (int c = 0; c < 6; ++c) pts[k * 6 + c] = p[c];
    if (rot) {
      R.apply(pts[k * 6], pts[k * 6 + 1], pts[k * 6 + 2]);
      cx += pts[k * 6]; cy += pts[k * 6 + 1]; cz += pts[k * 6 + 2];
    } else {
      cx += p[0]; cy += p[1]; cz += p[2];
    }
  }
  cx = block_sum(cx, redd) / a.P; cy = block_sum(cy, redd) / a.P; cz = block_sum(cz, redd) / a.P;
  const float fx = (float)cx, fy = (float)cy, fz = (float)cz;
  // ---- centre on the sample mean, scale by the max norm ----------------------------------------------------------------------
  float md = 0.f;
  for (int k = tid; k < a.P; k += 256) {
    const float x = pts[k * 6] - fx, y = pts[k * 6 + 1] - fy, z = pts[k * 6 + 2] - fz;
    pts[k * 6] = x; pts[k * 6 + 1] = y; pts[k * 6 + 2] = z;
    md = fmaxf(md, sqrtf(x * x + y * y + z * z));
  }
  md = block_max(md, redf);
  const float inv = md < 1e-6f ? 1.0f : 1.0f / md;   // tiny clouds keep their coordinates (base.py:727-728)
  __syncthreads();
  for (int i = tid; i < a.P * 6; i += 256) {
    const int c = i % 6;
    out[i] = c < 3 ? pts[i] * inv : pts[i];
  }
}

// ---- training-split object augmentation (data_augmentor.py + base.py:742-776) ------------------------------------------------
// Uniforms in (0, 1) from one hash; standard normals by Box-Muller.
__device__ __forceinline__ double u01d(unsigned h) { return ((double)h + 0.5) * (1.0 / 4294967296.0); }
__device__ __forceinline__ float u01f(unsigned h) { return ((float)(h >> 8) + 0.5f) * (1.0f / 16777216.0f); }

// Counter stream of one item / object of the draw kernel: every draw takes the next counter.
struct DrawStream {
  unsigned long long seed, key, ctr;
  __device__ __forceinline__ unsigned next() { return hash_u32(seed, key, ctr++); }
  __device__ __forceinline__ double uniform() { return u01d(next()); }
  __device__ __forceinline__ double normal() {
    const double u1 = uniform(), u2 = uniform();
    return sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
  }
  __device__ __forceinline__ int below(int m) { return (int)(((unsigned long long)next() * (unsigned long long)m) >> 32); }
};

// data_augmentor.py scene_aug / obj_aug rotation: rx, ry, rz from three angles, multiplied in a random order with shuffle
__device__ void draw_rotation(DrawStream &st, int axis_align, const double *value, int shuffle, double *r) {
  double th[3];
  for (int i = 0; i < 3; ++i) {
    if (axis_align) {
      const int q = st.below(4);
      const double ang = q == 0 ? 0.0 : q == 1 ? M_PI / 2 : q == 2 ? M_PI : M_PI * 3 / 2;
      th[i] = ang * value[i];
    } else {
      th[i] = (st.uniform() * 2 * M_PI - M_PI) * value[i];
    }
  }
  double m[3][9];
  const double cx = cos(th[0]), sx = sin(th[0]), cy = cos(th[1]), sy = sin(th[1]), cz = cos(th[2]), sz = sin(th[2]);
  const double rx[9] = {1, 0, 0, 0, cx, -sx, 0, sx, cx};
  const double ry[9] = {cy, 0, sy, 0, 1, 0, -sy, 0, cy};
  const double rz[9] = {cz, sz, 0, -sz, cz, 0, 0, 0, 1};
  int order[3] = {0, 1, 2};
  if (shuffle) {   // np.random.shuffle of three matrices: one of the 6 orders, uniformly
    const int p = st.below(6);
    const int perms[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
    order[0] = perms[p][0]; order[1] = perms[p][1]; order[2] = perms[p][2];
  }
  for (int j = 0; j < 3; ++j) {
    const double *src = order[j] == 0 ? rx : order[j] == 1 ? ry : rz;
    for (int e = 0; e < 9; ++e) m[j][e] = src[e];
  }
  double t[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) t[i * 3 + j] = m[0][i * 3] * m[1][j] + m[0][i * 3 + 1] * m[1][3 + j] + m[0][i * 3 + 2] * m[1][6 + j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[i * 3 + j] = t[i * 3] * m[2][j] + t[i * 3 + 1] * m[2][3 + j] + t[i * 3 + 2] * m[2][6 + j];
}

__device__ __forceinline__ void set_identity(double *r) {
  for (int e = 0; e < 9; ++e) r[e] = (e % 4 == 0) ? 1.0 : 0.0;
}

// one thread per item (item table), then one per object slot (object table)
__global__ void __launch_bounds__(128) aug_draw_kernel(const sv_aug_params p, int n_items, int n_slots, unsigned long long seed,
                                                       double *item_tab, double *obj_tab) {
  const int t = blockIdx.x * 128 + threadIdx.x;
  if (t < n_items) {
    double *it = item_tab + (size_t)t * SV_AUG_ITEM_STRIDE;
    DrawStream st{seed, (1ull << 40) + (unsigned long long)t, 0};
    set_identity(it);
    if (p.flags & SV_AUG_FLIP) {   // np.random.choice(4): flip x, flip y, flip x and y, none
      const int f = st.below(4);
      if (f == 0 || f == 2) it[0] = -1.0;
      if (f == 1 || f == 2) it[4] = -1.0;
    }
    it[9] = (p.flags & SV_AUG_SCALE) ? st.uniform() * (p.scale_hi - p.scale_lo) + p.scale_lo : 1.0;
    for (int i = 0; i < 3; ++i) it[10 + i] = (p.flags & SV_AUG_SCENE_TRANS) ? st.normal() * p.scene_trans[i] : 0.0;
    if (p.flags & SV_AUG_SCENE_ROT) draw_rotation(st, p.scene_rot_axis_align, p.scene_rot, p.scene_rot_shuffle, it + 13);
    else set_identity(it + 13);
    for (int i = 0; i < 3; ++i) it[22 + i] = (p.flags & SV_AUG_COLOR) ? st.normal() * 0.1 : 0.0;
  } else if (t < n_items + n_slots) {
    const int s = t - n_items;
    double *ot = obj_tab + (size_t)s * SV_AUG_OBJ_STRIDE;
    DrawStream st{seed, (2ull << 40) + (unsigned long long)s, 0};
    for (int i = 0; i < 3; ++i) ot[i] = (p.flags & SV_AUG_OBJ_TRANS) ? st.normal() * p.obj_trans[i] : 0.0;
    if (p.flags & SV_AUG_OBJ_ROT) draw_rotation(st, p.obj_rot_axis_align, p.obj_rot, p.obj_rot_shuffle, ot + 3);
    else set_identity(ot + 3);
  }
}

__global__ void __launch_bounds__(128) quarter_turn_draw_kernel(int n_items, unsigned long long seed, int *k) {
  const int t = blockIdx.x * 128 + threadIdx.x;
  if (t < n_items) k[t] = (int)(hash_u32(seed, (3ull << 40) + (unsigned long long)t, 0) >> 30);
}

// v @ M in f64 (numpy's matmul loop order, no contraction), rounded to f32 like the reference's f32 storage
__device__ __forceinline__ void mat_apply(float &x, float &y, float &z, const double *M) {
  const double a = x, b = y, c = z;
  double o[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) o[j] = __dadd_rn(__dadd_rn(__dmul_rn(a, M[j]), __dmul_rn(b, M[3 + j])), __dmul_rn(c, M[6 + j]));
  x = (float)o[0]; y = (float)o[1]; z = (float)o[2];
}

struct AugArgs {
  const float *raw;
  const long long *offsets;
  int S, O, P;
  sv_aug_params p;
  const double *item_tab, *obj_tab;
  const int *index_in;
  const float *noise_in;
  unsigned long long seed;
  float *fts, *locs, *boxes;
  unsigned char *masks;
  int *index_out;
  float *noise_out;
};

__device__ __forceinline__ void block_minmax3(float *mn, float *mx, float *redf) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    mx[c] = block_max(mx[c], redf);
    mn[c] = -block_max(-mn[c], redf);
  }
}

__global__ void __launch_bounds__(256) scene_prep_aug_kernel(const AugArgs a) {
  extern __shared__ __align__(16) float pts[];   // [P][6] the augmented points, in output order
  __shared__ double redd[8];
  __shared__ float redf[8];
  const int s = blockIdx.x, tid = threadIdx.x, P = a.P, fl = a.p.flags;
  const long long beg = a.offsets[s], n = a.offsets[s + 1] - beg;
  float *out = a.fts + (size_t)s * P * 6;
  if (n <= 0) {   // padded slot (dataset_wrapper.py:62-72)
    for (int i = tid; i < P * 6; i += 256) out[i] = 1.0f;
    if (tid < 6) a.locs[(size_t)s * 6 + tid] = 0.f;
    if (a.boxes != nullptr && tid < 6) a.boxes[(size_t)s * 6 + tid] = 0.f;
    if (tid == 0) a.masks[s] = 0;
    if (a.index_out != nullptr)
      for (int i = tid; i < P; i += 256) a.index_out[(size_t)s * P + i] = -1;
    if (a.noise_out != nullptr && (fl & SV_AUG_JITTER))
      for (int i = tid; i < P * 3; i += 256) a.noise_out[(size_t)s * P * 3 + i] = 0.f;
    return;
  }
  const float *raw = a.raw + (size_t)beg * 6;
  const double *it = a.item_tab + (size_t)(s / a.O) * SV_AUG_ITEM_STRIDE, *ot = a.obj_tab + (size_t)s * SV_AUG_OBJ_STRIDE;
  // ---- scene scaling needs the mean of ALL (flipped) raw points: the only pass over the whole object -----------------------
  float mu[3] = {0.f, 0.f, 0.f};
  const float sc = (float)it[9];   // a Python float times an f32 array: f32 arithmetic
  if (fl & SV_AUG_SCALE) {
    double sm[3] = {0, 0, 0};
    for (long long i = tid; i < n; i += 256) {
      float x = raw[i * 6], y = raw[i * 6 + 1], z = raw[i * 6 + 2];
      if (fl & SV_AUG_FLIP) mat_apply(x, y, z, it);
      sm[0] += x; sm[1] += y; sm[2] += z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) mu[c] = (float)(block_sum(sm[c], redd) / (double)n);
  }
  // ---- gather the P rows in output order: flip, scale, jitter, size, translations, scene rotation, colour ----------------------
  int bits = 1;
  while ((1ll << bits) < n) ++bits;
  int pbits = 1;
  while ((1 << pbits) < P) ++pbits;
  const unsigned k1 = hash_u32(a.seed, (unsigned long long)s, 1), k2 = hash_u32(a.seed, (unsigned long long)s, 2),
                 k3 = hash_u32(a.seed, (unsigned long long)s, 3), k4 = hash_u32(a.seed, (unsigned long long)s, 4),
                 k5 = hash_u32(a.seed, (unsigned long long)s, 5), k6 = hash_u32(a.seed, (unsigned long long)s, 6);
  const double jit = a.p.jitter;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int k = tid; k < P; k += 256) {
    long long idx;
    if (a.index_in != nullptr) {
      idx = a.index_in[(size_t)s * P + k];
    } else {
      unsigned j = (unsigned)k;   // pts_shuffle: output position k holds subsample position perm(k)
      if (fl & SV_AUG_PTS_SHUFFLE) {
        j = perm_pow2(j, pbits, k4, k5, k6);
        while ((int)j >= P) j = perm_pow2(j, pbits, k4, k5, k6);
      }
      if (n < P) {
        idx = (long long)(((unsigned long long)hash_u32(a.seed, (unsigned long long)s, 16 + (unsigned long long)j) * (unsigned long long)n) >> 32);
      } else {
        unsigned x = perm_pow2(j, bits, k1, k2, k3);
        while ((long long)x >= n) x = perm_pow2(x, bits, k1, k2, k3);
        idx = x;
      }
    }
    if (a.index_out != nullptr) a.index_out[(size_t)s * P + k] = (int)idx;
    const float *p = raw + idx * 6;
    float v[3] = {p[0], p[1], p[2]};
    if (fl & SV_AUG_FLIP) mat_apply(v[0], v[1], v[2], it);
    if (fl & SV_AUG_SCALE) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(__fmul_rn(__fsub_rn(v[c], mu[c]), sc), mu[c]);
    }
    if (fl & SV_AUG_JITTER) {   // x + (g - 0.5) * value, the -0.5 bias kept (data_augmentor.py jitter_fn)
      float g[3];
      if (a.noise_in != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) g[c] = a.noise_in[((size_t)s * P + k) * 3 + c];
      } else {
        const unsigned long long b = (1ull << 32) + 4ull * (unsigned long long)k;
        float sn, cs;
        const float r0 = sqrtf(-2.f * logf(u01f(hash_u32(a.seed, (unsigned long long)s, b))));
        sincospif(2.f * u01f(hash_u32(a.seed, (unsigned long long)s, b + 1)), &sn, &cs);
        g[0] = r0 * cs; g[1] = r0 * sn;
        const float r1 = sqrtf(-2.f * logf(u01f(hash_u32(a.seed, (unsigned long long)s, b + 2))));
        g[2] = r1 * cospif(2.f * u01f(hash_u32(a.seed, (unsigned long long)s, b + 3)));
      }
      if (a.noise_out != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) a.noise_out[((size_t)s * P + k) * 3 + c] = g[c];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = (float)__dadd_rn((double)v[c], __dmul_rn((double)g[c] - 0.5, jit));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { mn[c] = fminf(mn[c], v[c]); mx[c] = fmaxf(mx[c], v[c]); }
    if (fl & SV_AUG_SCENE_TRANS) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = (float)__dadd_rn((double)v[c], it[10 + c]);
    }
    if (fl & SV_AUG_OBJ_TRANS) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = (float)__dadd_rn((double)v[c], ot[c]);
    }
    if (fl & SV_AUG_SCENE_ROT) mat_apply(v[0], v[1], v[2], it + 13);
    pts[k * 6] = v[0]; pts[k * 6 + 1] = v[1]; pts[k * 6 + 2] = v[2];
#pragma unroll
    for (int c = 0; c < 3; ++c)
      pts[k * 6 + 3 + c] = (fl & SV_AUG_COLOR) ? (float)__dadd_rn((double)p[3 + c], it[22 + c]) : p[3 + c];
  }
  block_minmax3(mn, mx, redf);   // the size: after the jitter, before translation and rotation (data_augmentor.py)
  // ---- object rotation about the mean of the P points: (x - c) @ R + c -----------------------------------------------------------
  if (fl & SV_AUG_OBJ_ROT) {
    double sm[3] = {0, 0, 0};
    for (int k = tid; k < P; k += 256) { sm[0] += pts[k * 6]; sm[1] += pts[k * 6 + 1]; sm[2] += pts[k * 6 + 2]; }
    float c[3];
#pragma unroll
    for (int e = 0; e < 3; ++e) c[e] = (float)(block_sum(sm[e], redd) / P);
    for (int k = tid; k < P; k += 256) {
      const double x = __fsub_rn(pts[k * 6], c[0]), y = __fsub_rn(pts[k * 6 + 1], c[1]), z = __fsub_rn(pts[k * 6 + 2], c[2]);
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double o = __dadd_rn(__dadd_rn(__dmul_rn(x, ot[3 + j]), __dmul_rn(y, ot[6 + j])), __dmul_rn(z, ot[9 + j]));
        pts[k * 6 + j] = (float)__dadd_rn(o, (double)c[j]);
      }
    }
  }
  // ---- base.py:753-769: centre = mean, box = (min + max) / 2, fts = (x - centre) / max(max norm, 1e-6) ------------------------
  double sm[3] = {0, 0, 0};
  float bmn[3] = {INFINITY, INFINITY, INFINITY}, bmx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int k = tid; k < P; k += 256) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = pts[k * 6 + c];
      sm[c] += x; bmn[c] = fminf(bmn[c], x); bmx[c] = fmaxf(bmx[c], x);
    }
  }
  float ctr[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) ctr[c] = (float)(block_sum(sm[c], redd) / P);
  block_minmax3(bmn, bmx, redf);
  if (tid == 0) {
    float *l = a.locs + (size_t)s * 6;
#pragma unroll
    for (int c = 0; c < 3; ++c) { l[c] = ctr[c]; l[3 + c] = mx[c] - mn[c]; }
    if (a.boxes != nullptr) {
      float *bx = a.boxes + (size_t)s * 6;
#pragma unroll
      for (int c = 0; c < 3; ++c) { bx[c] = (bmn[c] + bmx[c]) / 2; bx[3 + c] = mx[c] - mn[c]; }
    }
    a.masks[s] = 1;
  }
  float md = 0.f;
  for (int k = tid; k < P; k += 256) {
    const float x = __fsub_rn(pts[k * 6], ctr[0]), y = __fsub_rn(pts[k * 6 + 1], ctr[1]), z = __fsub_rn(pts[k * 6 + 2], ctr[2]);
    pts[k * 6] = x; pts[k * 6 + 1] = y; pts[k * 6 + 2] = z;
    md = fmaxf(md, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z))));
  }
  md = fmaxf(block_max(md, redf), 1e-6f);   // clamp_(min=1e-6)
  __syncthreads();
  for (int i = tid; i < P * 6; i += 256) {
    const int c = i % 6;
    out[i] = c < 3 ? __fdiv_rn(pts[i], md) : pts[i];
  }
}

struct MaskArgs {
  const long long *ids;            // (T) token ids
  const long long *attn;           // (T) attention mask 0/1
  long long *out_ids, *labels;     // (T)
  long long T;
  float ratio;
  long long mask_id, vocab;
  unsigned long long seed;
};
__global__ void __launch_bounds__(256) token_mask_kernel(const MaskArgs a) {
  const long long t = blockIdx.x * 256ll + threadIdx.x;
  if (t >= a.T) return;
  const long long tok = a.ids[t];
  long long out = tok, lab = -1;
  if (a.attn[t] != 0) {
    float u = (hash_u32(a.seed, (unsigned long long)t, 7) >> 8) * (1.0f / 16777216.0f);
    if (u < a.ratio) {
      u /= a.ratio;
      if (u < 0.8f) out = a.mask_id;
      else if (u < 0.9f) out = (long long)(((unsigned long long)hash_u32(a.seed, (unsigned long long)t, 11) * (unsigned long long)a.vocab) >> 32);
      lab = tok;
    }
  }
  a.out_ids[t] = out;
  a.labels[t] = lab;
}
__global__ void __launch_bounds__(256) coin_mask_kernel(const unsigned char *valid, unsigned char *out, long long n, float ratio,
                                                       unsigned long long seed) {
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= n) return;
  const float u = (hash_u32(seed, (unsigned long long)i, 13) >> 8) * (1.0f / 16777216.0f);
  out[i] = (valid[i] != 0 && !(u < ratio)) ? 1 : 0;
}

}  // namespace

extern "C" int sv_scene_prep_rot_f32(const float *raw_points, const long long *slot_offsets, int n_slots, int slots_per_item,
                                     int P, unsigned long long seed, const int *quarter_turns, const int *index_in,
                                     float *obj_fts, float *obj_locs, float *obj_boxes, unsigned char *obj_masks,
                                     int *sample_idx, void *stream) {
  if (n_slots < 0 || P < 1 || P > 8192 || slots_per_item < 1 || n_slots % slots_per_item != 0) return SV_ERR_INVALID_ARG;
  if (n_slots == 0) return SV_OK;
  if (!raw_points || !slot_offsets || !obj_fts || !obj_locs || !obj_masks) return SV_ERR_INVALID_ARG;
  const size_t smem = (size_t)P * 6 * sizeof(float);
  if (smem > 48 * 1024) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(scene_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (rc) return rc;
  }
  PrepArgs a{raw_points, slot_offsets, n_slots, P, seed, obj_fts, obj_locs, obj_masks, sample_idx, slots_per_item, quarter_turns,
             index_in, obj_boxes};
  scene_prep_kernel<<<n_slots, 256, smem, (cudaStream_t)stream>>>(a);
  return sv::after_launch();
}

extern "C" int sv_quarter_turn_draw(int n_items, unsigned long long seed, int *quarter_turns, void *stream) {
  if (n_items < 0) return SV_ERR_INVALID_ARG;
  if (n_items == 0) return SV_OK;
  if (!quarter_turns) return SV_ERR_INVALID_ARG;
  quarter_turn_draw_kernel<<<(unsigned)((n_items + 127) / 128), 128, 0, (cudaStream_t)stream>>>(n_items, seed, quarter_turns);
  return sv::after_launch();
}

static bool aug_params_ok(const sv_aug_params *p) {
  if (!p || (p->flags & ~511) != 0) return false;
  if ((p->flags & SV_AUG_SCALE) && !(isfinite(p->scale_lo) && isfinite(p->scale_hi))) return false;
  if ((p->flags & SV_AUG_JITTER) && !(p->jitter >= 0.0 && isfinite(p->jitter))) return false;
  return true;
}

extern "C" int sv_aug_draw(const sv_aug_params *params, int n_items, int slots_per_item, unsigned long long seed,
                           double *item_tab, double *obj_tab, void *stream) {
  if (!aug_params_ok(params) || n_items < 0 || slots_per_item < 1) return SV_ERR_INVALID_ARG;
  if (n_items == 0) return SV_OK;
  if (!item_tab || !obj_tab) return SV_ERR_INVALID_ARG;
  const long long total = (long long)n_items * (slots_per_item + 1);
  if (total > 0x7fffffffll) return SV_ERR_INVALID_ARG;
  aug_draw_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>(*params, n_items, n_items * slots_per_item,
                                                                                     seed, item_tab, obj_tab);
  return sv::after_launch();
}

extern "C" int sv_scene_prep_aug_f32(const float *raw_points, const long long *slot_offsets, int n_items, int slots_per_item,
                                     int P, const sv_aug_params *params, const double *item_tab, const double *obj_tab,
                                     const int *index_in, const float *noise_in, unsigned long long seed, float *obj_fts,
                                     float *obj_locs, float *obj_boxes, unsigned char *obj_masks, int *index_out,
                                     float *noise_out, void *stream) {
  if (!aug_params_ok(params) || n_items < 0 || slots_per_item < 1 || P < 1 || P > 8192) return SV_ERR_INVALID_ARG;
  const long long n_slots = (long long)n_items * slots_per_item;
  if (n_slots > 0x7fffffffll) return SV_ERR_INVALID_ARG;
  if (n_slots == 0) return SV_OK;
  if (!raw_points || !slot_offsets || !item_tab || !obj_tab || !obj_fts || !obj_locs || !obj_masks) return SV_ERR_INVALID_ARG;
  const size_t smem = (size_t)P * 6 * sizeof(float);
  if (smem > 48 * 1024) {
    int rc = sv::cuda_status(cudaFuncSetAttribute(scene_prep_aug_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (rc) return rc;
  }
  AugArgs a{raw_points, slot_offsets, (int)n_slots, slots_per_item, P, *params, item_tab, obj_tab, index_in, noise_in, seed,
            obj_fts, obj_locs, obj_boxes, obj_masks, index_out, noise_out};
  scene_prep_aug_kernel<<<(unsigned)n_slots, 256, smem, (cudaStream_t)stream>>>(a);
  return sv::after_launch();
}

extern "C" int sv_token_mask(const long long *ids, const long long *attention_mask, long long n_tokens, float mask_ratio,
                             long long mask_token_id, long long vocab_size, unsigned long long seed, long long *out_ids,
                             long long *labels, void *stream) {
  if (n_tokens < 0 || !(mask_ratio >= 0.f) || mask_ratio > 1.f || vocab_size < 1) return SV_ERR_INVALID_ARG;
  if (n_tokens == 0) return SV_OK;
  if (!ids || !attention_mask || !out_ids || !labels) return SV_ERR_INVALID_ARG;
  MaskArgs a{ids, attention_mask, out_ids, labels, n_tokens, mask_ratio, mask_token_id, vocab_size, seed};
  token_mask_kernel<<<(unsigned)((n_tokens + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
  return sv::after_launch();
}

extern "C" int sv_coin_mask(const unsigned char *valid, long long n, float drop_ratio, unsigned long long seed,
                            unsigned char *out, void *stream) {
  if (n < 0 || !(drop_ratio >= 0.f) || drop_ratio > 1.f) return SV_ERR_INVALID_ARG;
  if (n == 0) return SV_OK;
  if (!valid || !out) return SV_ERR_INVALID_ARG;
  coin_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(valid, out, n, drop_ratio, seed);
  return sv::after_launch();
}
