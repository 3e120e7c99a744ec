/*
 * libsvpointops — C-ABI of the H100 (sm_90a) PointNet++ point operators.
 *
 * This is the drop-in boundary for the reference's pybind extension `pointnet2._ext`
 * (reference: modules/third_party/pointnet2/_ext_src/src/bindings.cpp:6-19).  Every entry point
 * takes raw DEVICE pointers + sizes + a cudaStream_t (passed as void*), enqueues on that stream,
 * does not synchronise, does not allocate, and returns an int status (0 = OK).  Output buffers are
 * fully overwritten (no pre-zeroing needed; the *_grad entry points zero their output themselves,
 * matching the reference's torch::zeros allocation).  All tensors are contiguous fp32 / int32, the
 * same preconditions the reference asserts (include/utils.h:5-25).
 *
 * Index results (fps / ball_query / three_nn idx) are bit-exact with the reference kernels;
 * copies (gather / group) are exact; *_grad use fp32 atomics like the reference (order not fixed).
 */
#ifndef SVPOINTOPS_H
#define SVPOINTOPS_H

#ifdef __cplusplus
extern "C" {
#endif

#define SV_OK 0
#define SV_ERR_INVALID_ARG 1   /* null pointer, negative size, unsupported shape */
#define SV_ERR_CUDA 2          /* launch failed; see sv_last_cuda_error() */

/* library identification */
int sv_version(void);
const char *sv_status_string(int status);
/* cudaError_t of the last failing launch in this thread (0 if none), and its string */
int sv_last_cuda_error(void);
const char *sv_last_cuda_error_string(void);
/* number of kernel launches this library has enqueued so far in this process (bench bookkeeping) */
unsigned long long sv_launch_count(void);

/* replaces furthest_point_sampling (src/sampling.cpp:66-87, kernel src/sampling_gpu.cu:69-173).
 * xyz (B,N,3) -> idx (B,m) i32.  new_xyz may be NULL; when given receives xyz[idx] as (B,m,3)
 * (fuses the gather_points call that always follows, pointnet2_modules.py:54-58). */
int sv_fps_f32(const float *xyz, int B, int N, int m, int *idx, float *new_xyz, void *stream);

/* replaces gather_points (src/sampling.cpp:15-38, src/sampling_gpu.cu:8-20).
 * points (B,C,N), idx (B,M) -> out (B,C,M) */
int sv_gather_points_f32(const float *points, const int *idx, int B, int C, int N, int M,
                         float *out, void *stream);

/* replaces gather_points_grad (src/sampling.cpp:40-65, src/sampling_gpu.cu:34-47).
 * grad_out (B,C,M), idx (B,M) -> grad_points (B,C,N) (zeroed here, then atomic scatter-add) */
int sv_gather_points_grad_f32(const float *grad_out, const int *idx, int B, int C, int N, int M,
                              float *grad_points, void *stream);

/* replaces ball_query (src/ball_query.cpp:8-32, src/ball_query_gpu.cu:9-44).
 * new_xyz (B,M,3), xyz (B,N,3) -> idx (B,M,nsample) i32 */
int sv_ball_query_f32(const float *new_xyz, const float *xyz, int B, int N, int M, float radius,
                      int nsample, int *idx, void *stream);

/* replaces group_points (src/group_points.cpp:12-36, src/group_points_gpu.cu:8-28).
 * points (B,C,N), idx (B,NP,NS) -> out (B,C,NP,NS) */
int sv_group_points_f32(const float *points, const int *idx, int B, int C, int N, int NP, int NS,
                        float *out, void *stream);

/* replaces group_points_grad (src/group_points.cpp:38-62, src/group_points_gpu.cu:43-64).
 * grad_out (B,C,NP,NS), idx (B,NP,NS) -> grad_points (B,C,N) (zeroed here) */
int sv_group_points_grad_f32(const float *grad_out, const int *idx, int B, int C, int N, int NP,
                             int NS, float *grad_points, void *stream);

/* replaces three_nn (src/interpolate.cpp:14-40, src/interpolate_gpu.cu:9-59).
 * unknown (B,n,3), known (B,m,3) -> dist2 (B,n,3) f32, idx (B,n,3) i32 */
int sv_three_nn_f32(const float *unknown, const float *known, int B, int n, int m, float *dist2,
                    int *idx, void *stream);

/* replaces three_interpolate (src/interpolate.cpp:42-70, src/interpolate_gpu.cu:72-101).
 * points (B,c,m), idx (B,n,3), weight (B,n,3) -> out (B,c,n) */
int sv_three_interpolate_f32(const float *points, const int *idx, const float *weight, int B, int c,
                             int m, int n, float *out, void *stream);

/* replaces three_interpolate_grad (src/interpolate.cpp:71-99, src/interpolate_gpu.cu:116-143).
 * grad_out (B,c,n), idx, weight (B,n,3) -> grad_points (B,c,m) (zeroed here) */
int sv_three_interpolate_grad_f32(const float *grad_out, const int *idx, const float *weight, int B,
                                  int c, int n, int m, float *grad_points, void *stream);

/* Fused sample+query used by the new set-abstraction path (one pass over xyz): equals
 * sv_fps_f32(xyz -> fps_idx,new_xyz) followed by sv_ball_query_f32(new_xyz, xyz -> ball_idx).
 * fps_idx (B,m) i32, new_xyz (B,m,3) f32, ball_idx (B,m,nsample) i32. Requires N <= 1024. */
int sv_fps_ballquery_f32(const float *xyz, int B, int N, int m, float radius, int nsample,
                         int *fps_idx, float *new_xyz, int *ball_idx, void *stream);

/* Two-level fused sampling for a PointNet++ set-abstraction stack, one pass over xyz (32 <= N <= 1024):
 * level 1 = sv_fps_ballquery_f32(xyz, m, radius, nsample); level 2 (m2 > 0, requires m == 32) = the
 * same on the (B,32,3) centres of level 1 with (m2, radius_2, nsample2).  Replaces the reference's
 * furthest_point_sample + gather_operation + ball_query of two consecutive PointnetSAModules
 * (pointnet2_modules.py:54-58, pointnet2_utils.py:331); the ball-query distances are taken from the
 * FPS sweep (bit-identical).  Outputs as in sv_fps_ballquery_f32, per level. */
int sv_sa_sample_f32(const float *xyz, int B, int N, int m, float radius, int nsample, int *fps_idx,
                     float *new_xyz, int *ball_idx, int m2, float radius_2, int nsample2, int *fps_idx2,
                     float *new_xyz2, int *ball_idx2, void *stream);

/* ---- device-side input pipeline (SURVEY.md §8 f2) -----------------------------------------------------------------------
 * Builds the model's per-object tensors from ragged raw scene data on the GPU: replaces the per-object numpy loop of
 * data/datasets/base.py:697-741 (`_obj_processing_post`) and the padding of data/datasets/dataset_wrapper.py:62-72.
 * raw_points (total,6) f32 [xyz rgb]; slot_offsets (n_slots+1) int64 CSR over the B*O object slots (empty range = padded
 * slot).  Per slot: obj_locs (6) = [mean xyz, max-min] of the raw points; P points sampled uniformly (without replacement
 * when the object has >= P points, with replacement otherwise), centred on the SAMPLE mean, divided by the sample's max norm
 * (1 when < 1e-6), colours untouched; empty slots: all-ones points, zero locs, mask 0.  sample_idx (n_slots,P) i32 may be
 * NULL (receives the chosen raw indices, -1 for empty slots).  Randomness = counter hash of (seed, slot, k).
 * `rot_aug` (data/data_utils.py:163-178 `build_rotate_mat`): with quarter_turns (n_slots / slots_per_item) i32 in 0..3, the
 * raw xyz of every object of item b are first rotated x @ R^T, R = [[c, -s, 0], [s, c, 0], [0, 0, 1]] in f32 with theta =
 * quarter_turns[b] * pi / 2 (0 = not rotated); NULL = no rotation.  obj_boxes (n_slots, 6) = [(min + max) / 2, max - min] of
 * the rotated raw points, may be NULL.  index_in (n_slots, P) i32 may be NULL (drawn from the seed) or give the sampled raw
 * indices.  sv_quarter_turn_draw fills quarter_turns (n_items) uniformly from the seed. */
int sv_scene_prep_rot_f32(const float *raw_points, const long long *slot_offsets, int n_slots, int slots_per_item, int P,
                          unsigned long long seed, const int *quarter_turns, const int *index_in, float *obj_fts,
                          float *obj_locs, float *obj_boxes, unsigned char *obj_masks, int *sample_idx, void *stream);
int sv_quarter_turn_draw(int n_items, unsigned long long seed, int *quarter_turns, void *stream);
/* Training-split object augmentation (the `data_aug` configs): restates data/datasets/data_augmentor.py
 * `DataAugmentor.update_data_dict` followed by data/datasets/base.py:742-776 `_obj_processing_aug`, per object slot, in this
 * order: scene flip of all raw xyz; scene scaling about the raw mean (taken after the flip); subsample P points (without
 * replacement when n >= P); jitter x + (g - 0.5) * jitter; size = max - min HERE (after the jitter, before translation and
 * rotation, so a 90 degree scene rotation does not swap the sizes); + scene translation, + object translation; x @ R_scene;
 * object rotation (x - c) @ R_obj + c about the mean of the P points; + rgb_delta on the colours; point shuffle.  Outputs:
 * obj_locs = [mean xyz, size], obj_boxes = [(min + max) / 2, size], obj_fts xyz = (x - mean) / max(max norm, 1e-6).
 * Padded slots (empty range): all-ones points, zero locs / boxes, mask 0.
 *
 * Which transforms run is `params->flags` (SV_AUG_*); their random values come from two tables:
 *   item_tab (n_items, SV_AUG_ITEM_STRIDE) f64 = [flip 3x3 | scale | scene translation 3 | scene rotation 3x3 | rgb delta 3]
 *   obj_tab  (n_items * slots_per_item, SV_AUG_OBJ_STRIDE) f64 = [object translation 3 | object rotation 3x3]
 * (matrices row-major, applied as x @ M like the reference).  sv_aug_draw fills them from a seed; a caller may fill them itself
 * (replaying recorded draws).  Per output point: index_in (n_slots, P) i32 = the raw index of output position k (subsample
 * composed with the shuffle) and noise_in (n_slots, P, 3) f32 = the standard normals of its jitter.  Either may be NULL: it is
 * then drawn from (seed, slot, k); noise_in is read only with SV_AUG_JITTER.  index_out / noise_out (same layouts, NULL-able)
 * receive what was used (-1 / 0 on padded slots), so feeding them back as index_in / noise_in with the same tables reproduces
 * the output bit for bit.  obj_boxes (n_slots, 6) may be NULL.  All raw points are read only with SV_AUG_SCALE (the raw mean);
 * otherwise just the P gathered rows.  1 <= P <= 8192. */
#define SV_AUG_FLIP 1
#define SV_AUG_SCALE 2
#define SV_AUG_SCENE_TRANS 4
#define SV_AUG_SCENE_ROT 8
#define SV_AUG_COLOR 16
#define SV_AUG_OBJ_TRANS 32
#define SV_AUG_OBJ_ROT 64
#define SV_AUG_JITTER 128
#define SV_AUG_PTS_SHUFFLE 256
#define SV_AUG_ITEM_STRIDE 25
#define SV_AUG_OBJ_STRIDE 12
typedef struct {
  int flags;                       /* SV_AUG_* */
  int scene_rot_axis_align, scene_rot_shuffle, obj_rot_axis_align, obj_rot_shuffle;
  double scale_lo, scale_hi;       /* scene scaling s ~ U[lo, hi] */
  double scene_trans[3];           /* scene translation N(0,1) * value[i] */
  double scene_rot[3];             /* rotation value[i] (scales each angle) */
  double obj_trans[3];
  double obj_rot[3];
  double jitter;                   /* random_jitter value */
} sv_aug_params;
/* Fills item_tab / obj_tab (layouts above) from (seed, item / slot): flip type uniform over {x, y, x and y, none}; s = U * (hi -
 * lo) + lo; translations N(0,1) * value; rotations built as data_augmentor.py builds rx, ry, rz (angle = choice of {0, pi/2, pi,
 * 3 pi/2} * value with axis_align, else (U * 2 pi - pi) * value), multiplied in a uniformly random order with shuffle; rgb delta
 * N(0,1) * 0.1.  Entries of disabled transforms are identity / zero. */
int sv_aug_draw(const sv_aug_params *params, int n_items, int slots_per_item, unsigned long long seed, double *item_tab,
                double *obj_tab, void *stream);
int sv_scene_prep_aug_f32(const float *raw_points, const long long *slot_offsets, int n_items, int slots_per_item, int P,
                          const sv_aug_params *params, const double *item_tab, const double *obj_tab, const int *index_in,
                          const float *noise_in, unsigned long long seed, float *obj_fts, float *obj_locs, float *obj_boxes,
                          unsigned char *obj_masks, int *index_out, float *noise_out, void *stream);
/* BERT masked-LM corruption (data/data_utils.py:76-104 `random_word`): for tokens with attention_mask != 0, with probability
 * mask_ratio the label is the original id and the token becomes [MASK] (80 %), a uniform random id (10 %) or stays (10 %);
 * every other label is -1.  ids / attention_mask / out_ids / labels: (n_tokens) int64. */
int sv_token_mask(const long long *ids, const long long *attention_mask, long long n_tokens, float mask_ratio,
                  long long mask_token_id, long long vocab_size, unsigned long long seed, long long *out_ids,
                  long long *labels, void *stream);
/* random_point_cloud (data/data_utils.py:107-121): out[i] = valid[i] && u_i >= drop_ratio (bytes). */
int sv_coin_mask(const unsigned char *valid, long long n, float drop_ratio, unsigned long long seed, unsigned char *out,
                 void *stream);

/* Evaluation targets of the grounding datasets (csrc/eval_targets.cu; reference: data/datasets/base.py:387-454), one CTA per
 * item.  points (total, 6) f32 [xyz rgb]; cand_offsets: CSR over points, one range per candidate object (each >= 1 point);
 * item_offsets (B + 1): the candidates of item b are cand_offsets ranges item_offsets[b] .. item_offsets[b+1]-1, at most
 * max_cand (<= 4096) of them.  pred mode (gt_index NULL): gt_points / gt_offsets (B + 1) hold each item's ground-truth object;
 * IoU of the numpy-1.26 box round trip, hits at >= 0.25 / >= 0.5, target = the last IoU-25 hit.  gt mode: gt_index (B) int64
 * is the target candidate (local index) and its only hit.  cand_labels (n_cand) int64, tgt_label (B) int64.
 * Outputs: slot_map (B, O) int32 = local candidate index per slot in ascending order, -1 = empty; tgt_object_id (B) int64 = the
 * target's slot or the kept count when there is none; iou25 / iou50 (B, O) int64 flags per slot; iou_out (n_cand) f32 or NULL. */
int sv_grounding_targets_f32(const float *points, const long long *cand_offsets, const long long *item_offsets,
                             const float *gt_points, const long long *gt_offsets, const long long *gt_index,
                             const long long *cand_labels, const long long *tgt_label, int B, int O, int max_cand,
                             unsigned long long seed, int *slot_map, long long *tgt_object_id, long long *iou25,
                             long long *iou50, float *iou_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SVPOINTOPS_H */
