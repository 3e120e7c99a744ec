/*
 * libsvgps — C-ABI of the tensor-core (wgmma, sm_90a) kernels of the GPS object encoder and attention stack.
 * Raw device pointers + sizes + cudaStream_t (void*), int status (codes in svpointops.h), no
 * allocation, no synchronisation.  bf16 tensors are passed as void* (device, 2-byte elements).
 */
#ifndef SVGPS_H
#define SVGPS_H
#include "svpointops.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bookkeeping of this library (separate counters from libsvpointops) */
unsigned long long svgps_launch_count(void);
int svgps_last_cuda_error(void);
const char *svgps_last_cuda_error_string(void);

/* ---- PointNet++ set-abstraction MLP (inference form: eval-mode BatchNorm folded), wgmma -------------------
 * Replaces QueryAndGroup + SharedMLP(3 x Conv2d1x1+BN+ReLU) + max_pool2d of one PointnetSAModule
 * (reference: pointnet2_modules.py:34-75, pointnet2_utils.py:314-373, pytorch_utils.py:11-36).
 * `params` = packed device buffer of sv_sa_mlp_param_bytes(level) bytes built by
 * sceneverse_b200.modules.pointnet.pack_sa_params: [W1|W2|W3] bf16 in wgmma K-major layout with the BN
 * scale folded in, then shift1|shift2|shift3 (f32).  Outputs are point-major bf16 (B,npoint,C). */
int sv_sa_mlp_param_bytes(int level);
/* level 1: pts (B,P,6) f32 [xyz rgb], new_xyz (B,32,3), ball_idx (B,32,nsample) -> out (B,32,128) bf16
 * (mlp 6->64->64->128) */
int sv_sa1_mlp_bf16(const float *pts, const float *new_xyz, const int *ball_idx, const void *params, int B, int P,
                    int nsample, void *out_feat, void *stream);
/* level 2: xyz (B,P,3) f32, feat (B,P,128) bf16, new_xyz (B,16,3), ball_idx (B,16,nsample) -> out (B,16,256) bf16
 * (mlp 131->128->128->256) */
int sv_sa2_mlp_bf16(const float *xyz, const void *feat, const float *new_xyz, const int *ball_idx, const void *params,
                    int B, int P, int nsample, void *out_feat, void *stream);

/* ---- dense contraction with fused epilogue (wgmma, TMA, persistent) ----------------------------------------------
 * out[M,N] = epilogue(A[M,K] x B[N,K]^T): A, B bf16 row-major with leading dimensions lda, ldb (elements, % 8 == 0,
 * K % 8 == 0, 16-byte aligned) — B is the nn.Linear weight layout, so this replaces F.linear / 1x1 Conv2d
 * (reference call sites: SURVEY.md §2.3).  epilogue: + bias[N] (f32, may be NULL) -> act (0 none, 1 relu, 2 gelu-erf)
 * -> + residual[M,N] (same dtype / ld as out, may be NULL) -> store bf16 (out_f32 = 0) or f32 (1).
 * rowmax = 16: instead store max over each group of 16 consecutive rows into out[M/16,N] (PointNet++ SA3 max-pool). */
int sv_gemm_bf16(const void *A, int lda, const void *B, int ldb, int M, int N, int K, const float *bias, int act,
                 const void *residual, void *out, int ldo, int out_f32, int rowmax, void *stream);
/* Same GEMM with either operand given TRANSPOSED in memory (the two backward GEMMs of a linear layer without any copy):
 * a_transposed = 1: A is stored (K, M) row-major, lda >= M;  b_transposed = 1: B is stored (K, N) row-major, ldb >= N.
 * The staged tiles are then read by the tensor core as MN-major operands.  dgrad of y = x W^T: dx = g . W  ->
 * sv_gemm_bf16_ex(g, N, 0, W, Kin, 1, M, Kin, N, ...);  wgrad: dW = g^T . x -> sv_gemm_bf16_ex(g, N, 1, x, Kin, 1, N, Kin, M,
 * ..., out_f32 = 1).  (reference: autograd of every nn.Linear of the stack, e.g. modules/layers/transformers.py:122-134) */
int sv_gemm_bf16_ex(const void *A, int lda, int a_transposed, const void *B, int ldb, int b_transposed, int M, int N, int K,
                    const float *bias, int act, const void *residual, void *out, int ldo, int out_f32, int rowmax,
                    void *stream);

/* Kernel selection of the GEMM family (tests / benchmarks): 0 = heuristic (default), 1 / 2 / 4 = tiles of 64 / 128 / 192
 * output columns (128 rows each).
 * Bits 8.. are profiling switches that make the RESULT GARBAGE (timing only): 1 = the epilogue skips its body,
 * 2 = the producer skips its TMA loads. */
int sv_gemm_force_ctas(int ctas);

/* Profiling: while `buf` (device, [grid][16] int64) is non-null every GEMM launch writes, per CTA, the first consumer
 * warpgroup's {loop cycles, cycles waiting for operands, 0, k-steps issued, clock at start, at end, loop nanoseconds
 * (globaltimer), epilogue: 1 = staged in shared memory and written by TMA, 0 = per-element stores}. */
int sv_gemm_profile(long long *buf);

/* ---- the three GEMMs of a linear layer y = x W^T + b with their fused epilogues (same wgmma kernel family) --------
 * Replace F.linear and its autograd (AddmmBackward: mm, mm, sum) for every nn.Linear of the attention stack, BERT and the
 * heads (reference: modules/layers/transformers.py:115-154,188-192,285-316; modules/language/bert.py:21-26).
 * x (M,K) bf16 ld ldx; w (N,K) bf16 ld ldw (nn.Linear layout); all leading dimensions % 8 == 0, 16-byte aligned bases.
 * forward:  out = dropout_p(act(x w^T + bias)) -> (M,N) bf16 | f32, ld ldo; act 0 none / 1 relu / 2 gelu(erf);
 *           pre_out (bf16, ld ldo, may be NULL) receives x w^T + bias before the activation (saved for the gelu backward);
 *           the dropout mask is the counter hash of csrc/attn_common.cuh keyed by (seed, row, column): nothing is stored. */
int sv_linear_fwd_bf16(const void *x, int ldx, const void *w, int ldw, int M, int N, int K, const float *bias, int act,
                       float dropout_p, unsigned long long seed, void *out, int ldo, int out_f32, void *pre_out,
                       void *stream);
/* dgrad:    dx (M,Kin) = (gy (M,N) . w (N,Kin)) x f, the weight read as a transposed (MN-major) operand, no copy.
 *           dact 0: f = 1.  dact 1: aux = the forward OUTPUT of a relu(+dropout) layer of shape (M,Kin): f = aux > 0 ? 1/(1-p) : 0.
 *           dact 2: aux = the saved PRE-activation of a gelu(+dropout) layer: f = gelu'(aux) x mask(seed,row,col)/(1-p).
 *           (the activation sits on the INPUT side of this linear: h = dropout(act(pre)), y = h w^T) */
int sv_linear_dgrad_bf16(const void *gy, int ldg, const void *w, int ldw, int M, int N, int Kin, int dact, const void *aux,
                         int ld_aux, float dropout_p, unsigned long long seed, void *dx, int ldx, int out_f32, void *stream);
/* wgrad:    dw (N,Kin) f32 (ld ld_dw) (+)= gy^T . x and db (N) f32 (+)= column sums of gy (db may be NULL), contraction over
 *           the M tokens split across the grid, results reduced with atomic adds — accumulate = 1 adds straight into an
 *           existing gradient buffer (the flat fp32 buffer the data-parallel all-reduce runs on), 0 overwrites.  The bias
 *           gradient costs one extra N = 8 MMA per K step against a tile of ones in the same main loop. */
int sv_linear_wgrad_bf16(const void *gy, int ldg, const void *x, int ldx, int M, int N, int Kin, float *dw, int ld_dw,
                         float *db, int accumulate, void *stream);

/* ---- fused attention (wgmma): O = softmax(Q K^T * scale + spatial gate + key mask) V, head dim 64 ------------------
 * q (B,Lq,*), k/v (B,Lk,*) bf16 with batch strides *_bs and row strides *_rs (elements, % 8 == 0); head h uses columns
 * [64h, 64h+64).  key_padding_mask (B,Lk) bytes, 1 = ignore (may be NULL).  spatial_w (B,Lq,spatial_heads*6) f32 =
 * [bias, w1..w5] per head and pairwise_locs (B,Lq,Lk,5) f32 enable the MultiHeadAttentionSpatial 'cond' gate
 * log(clamp(sigmoid(w . loc + b), 1e-6)) (reference: modules/layers/transformers.py:206-232); NULL = plain attention
 * (nn.MultiheadAttention core).  Lk <= 384.  out (B,Lq,H*64) bf16.  lse (B,H,Lq) f32 (may be NULL) receives the
 * log-sum-exp of each query's logits, which the backward needs.
 * Dropout on the attention weights (nn.MultiheadAttention in training, reference transformers.py:22-24,69-74,118-120;
 * dropout_p = 0: none): weight (b,h,i,j) is kept iff its 16-bit counter-based uniform (csrc/attn_common.cuh: one 64-bit
 * mix per (b,h,i) row, one 32-bit mix per key pair) >= round(p * 65536), and scaled by 1/(1-p); the backward regenerates
 * the same mask from (dropout_p, seed).  Not combinable with the spatial gate (the reference's spatial attention has no
 * weight dropout). */
int sv_attention_fwd_dropout_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                  const void *v, long long v_bs, int v_rs, void *out, long long o_bs, int o_rs,
                                  const unsigned char *key_padding_mask, const float *spatial_w, int spatial_heads,
                                  const float *pairwise_locs, int B, int H, int Lq, int Lk, float scale, float *lse,
                                  float dropout_p, unsigned long long seed, void *stream);
/* The same attention for queries that are the first Lq rows of a sequence of seq_rows (>= Lq) rows, e.g. q = the first
 * row of each scene of a packed (B, seq_rows, 3E) projection, k / v all of its rows: query i of (b, h) draws the dropout
 * mask of row (b H + h) seq_rows + i, exactly the mask it has in the launch over all seq_rows queries.
 * sv_attention_fwd_dropout_bf16 is this call with seq_rows = Lq. */
int sv_attention_fwd_rows_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                               const void *v, long long v_bs, int v_rs, void *out, long long o_bs, int o_rs,
                               const unsigned char *key_padding_mask, const float *spatial_w, int spatial_heads,
                               const float *pairwise_locs, int B, int H, int Lq, int Lk, float scale, float *lse,
                               float dropout_p, unsigned long long seed, int seq_rows, void *stream);

/* Backward of the fused attention (one wgmma kernel template launched twice: dQ + gate-weight gradients with tile rows
 * == queries, dK/dV with tile rows == keys; both recompute P from Q, K, the gate and lse).  q/k/v, dropout_p and seed as in
 * the forward; o, d_o (B,Lq,H*64) bf16 contiguous; dq (B,Lq,*), dk, dv (B,Lk,*) bf16 with rows d_rs (>= H*64) elements
 * apart (scene stride L * d_rs): d_rs = H*64 gives contiguous gradients, d_rs = 3E lets the three be the column slices
 * [0,E) [E,2E) [2E,3E) of ONE packed (B,L,3E) buffer — the gradient of a packed QKV projection, consumed by a single
 * dgrad / wgrad GEMM (requires Lq == Lk; see sv_attention_bwd_rows_bf16 otherwise).  d_spatial_w (B,Lq,H*6) f32 (NULL without gate; gate requires
 * spatial_heads == H); dvec (B,H,Lq) f32 scratch.  Lq, Lk <= 384. */
int sv_attention_bwd_strided_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                                  const void *v, long long v_bs, int v_rs, const void *o, const void *d_o,
                                  const unsigned char *key_padding_mask, const float *spatial_w,
                                  const float *pairwise_locs, const float *lse, int B, int H, int Lq, int Lk, float scale,
                                  void *dq, void *dk, void *dv, int d_rs, float *d_spatial_w, float *dvec, float dropout_p,
                                  unsigned long long seed, void *stream);
/* Backward of sv_attention_fwd_rows_bf16 (same seq_rows): dq is (B, seq_rows, *) with scene stride seq_rows * d_rs, its
 * rows [Lq, seq_rows) are written as zeros, and the dropout masks are those of the forward.  With seq_rows = Lk and
 * d_rs = 3E, dq | dk | dv are the column slices of one packed (B, Lk, 3E) gradient even when only its first Lq rows are
 * queries.  sv_attention_bwd_strided_bf16 is this call with seq_rows = Lq. */
int sv_attention_bwd_rows_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                               const void *v, long long v_bs, int v_rs, const void *o, const void *d_o,
                               const unsigned char *key_padding_mask, const float *spatial_w, const float *pairwise_locs,
                               const float *lse, int B, int H, int Lq, int Lk, float scale, void *dq, void *dk, void *dv,
                               int d_rs, float *d_spatial_w, float *dvec, float dropout_p, unsigned long long seed,
                               int seq_rows, void *stream);

/* The same forward and backward for sequences of up to 2048 queries and 2048 keys (scenes of more than 384 objects, the
 * joint text + object sequence, captions up to BERT's 512 positions).  Parameters, results, dropout masks and the other
 * checks are those of sv_attention_fwd_rows_bf16 / sv_attention_bwd_rows_bf16; 1 <= Lk <= 2048 and Lq <= 2048 (the
 * backward: 1 <= Lq), anything larger is rejected.  The forward streams K and V through a two-stage TMA ring instead of
 * keeping them resident (at most 66 KB of shared memory per CTA); every element is computed as in the resident forward,
 * so on shapes both entries take (<= 384) the results are the same bits.  The backward is the same kernel pair as
 * sv_attention_bwd_rows_bf16, with its per-column arrays sized for the call. */
int sv_attention_fwd_long_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                               const void *v, long long v_bs, int v_rs, void *out, long long o_bs, int o_rs,
                               const unsigned char *key_padding_mask, const float *spatial_w, int spatial_heads,
                               const float *pairwise_locs, int B, int H, int Lq, int Lk, float scale, float *lse,
                               float dropout_p, unsigned long long seed, int seq_rows, void *stream);
int sv_attention_bwd_long_bf16(const void *q, long long q_bs, int q_rs, const void *k, long long k_bs, int k_rs,
                               const void *v, long long v_bs, int v_rs, const void *o, const void *d_o,
                               const unsigned char *key_padding_mask, const float *spatial_w, const float *pairwise_locs,
                               const float *lse, int B, int H, int Lq, int Lk, float scale, void *dq, void *dk, void *dv,
                               int d_rs, float *d_spatial_w, float *dvec, float dropout_p, unsigned long long seed,
                               int seq_rows, void *stream);

/* Both attention directions skip every 64-key block whose keys are all masked (key_padding_mask or past Lk): such a block
 * only adds zero weights, so the results are the full sweep's bit for bit, up to the sign of a zero.  Tests: on = 1 makes
 * every launch sweep all blocks again, on = 0 (default) restores skipping. */
int sv_attention_visit_all_blocks(int on);

/* Fused dropout + residual add + LayerNorm:  y = LayerNorm(residual + dropout(x)) * gamma + beta  (reference: the post-norm
 * blocks of modules/layers/transformers.py:145-154,311-315; plain LayerNorm of modules/utils.py:18-25 with residual = NULL,
 * dropout_p = 0).  x, residual, y, s: (R,D) contiguous, bf16 (io_bf16 = 1) or f32; D % 8 == 0, D <= 1024; gamma, beta (D)
 * f32; s receives the pre-norm sum (required when residual != NULL or dropout_p > 0; the backward's input — with neither,
 * pass x itself to the backward); mean, rstd (R) f32.  The dropout mask is the counter hash of csrc/attn_common.cuh keyed
 * by (seed, row, column): nothing is stored, the backward regenerates it. */
int sv_layer_norm_fwd(const void *x, const void *residual, int io_bf16, int R, int D, const float *gamma, const float *beta,
                      float eps, float dropout_p, unsigned long long seed, void *y, void *s, float *mean, float *rstd,
                      void *stream);
/* Backward: g = dL/dy (R,D) same dtype; ds = dL/d(residual) (= dL/dx without dropout); dx = ds o mask / (1 - p) (required
 * iff dropout_p > 0); dgamma, dbeta (D) f32, overwritten (accumulate = 0) or added into (accumulate = 1: the flat gradient
 * buffer); scratch: sv_layer_norm_scratch_floats(D) floats (per-CTA partial sums, reduced in a fixed order by a second small
 * kernel). */
int sv_layer_norm_bwd_acc(const void *g, const void *s, int io_bf16, int R, int D, const float *gamma, const float *mean,
                          const float *rstd, float dropout_p, unsigned long long seed, void *ds, void *dx, float *dgamma,
                          float *dbeta, int accumulate, float *scratch, void *stream);
/* The same two calls for rows taken every row_key_stride (>= 1) rows of a larger tensor: row r draws the dropout mask of
 * row r * row_key_stride, so LayerNorm over the first token of each of B sequences of L tokens (R = B, row_key_stride = L)
 * drops exactly what the call over all B * L rows drops there.  The calls above are these with row_key_stride = 1. */
int sv_layer_norm_fwd_rows(const void *x, const void *residual, int io_bf16, int R, int D, const float *gamma,
                           const float *beta, float eps, float dropout_p, unsigned long long seed, void *y, void *s,
                           float *mean, float *rstd, int row_key_stride, void *stream);
int sv_layer_norm_bwd_rows(const void *g, const void *s, int io_bf16, int R, int D, const float *gamma, const float *mean,
                           const float *rstd, float dropout_p, unsigned long long seed, void *ds, void *dx, float *dgamma,
                           float *dbeta, int accumulate, float *scratch, int row_key_stride, void *stream);

/* Row-wise L2 normalisation y = x / max(||x||_2, eps) over the last dimension and its backward
 * dx = (g - y (y . g)) / ||x|| (rows with ||x|| < eps: g / eps) — F.normalize(x, dim=-1, p=2) of the contrastive heads
 * (optim/loss/contra_loss.py:29-30, 59-60, 86-87 in the reference) and its autograd in one kernel per direction.
 * x / y / g / dx: (R, D) bf16 (io_bf16 = 1) or fp32, 16-byte aligned, D % 8 == 0, 8 <= D <= 1024; norm: (R) fp32. */
int sv_l2norm_fwd(const void *x, int io_bf16, int R, int D, float eps, void *y, float *norm, void *stream);
int sv_l2norm_bwd(const void *g, const void *y, const float *norm, int io_bf16, int R, int D, float eps, void *dx,
                  void *stream);
int sv_layer_norm_scratch_floats(int D);

/* Every in-kernel dropout mask (attention weights, fused LayerNorm) is a pure function of (seed, indices).  A captured
 * CUDA graph freezes the by-value seed, so a process may register ONE device counter: each dropout launch then uses
 * seed + *device_counter * odd_constant, read on the device at run time — increment the counter once per step (inside the
 * graph) and every replay draws fresh masks while forward and backward of the same step still agree.  NULL unregisters. */
int sv_dropout_seed_offset(const unsigned long long *device_counter);

/* Column sums out[c] = sum_r x[r][c] of a row-major (R, N) bf16 / f32 matrix (rows row_stride elements apart, N % 8 == 0),
 * fp32 accumulation, deterministic: the bias gradient of a linear layer (reference: autograd of every nn.Linear of the
 * stack, e.g. modules/layers/transformers.py:122-134).  scratch: sv_colsum_scratch_floats(N) floats. */
int sv_colsum(const void *x, long long row_stride, int is_bf16, int R, int N, float *out, float *scratch, void *stream);
int sv_colsum_scratch_floats(int N);

/* Batched column sums out[b][c] = sum_r x[b][r][c] of B row-major (R, N) matrices batch_stride elements apart (rows
 * row_stride apart, N % 8 == 0, both strides % 8 == 0), written to a contiguous (B, N) out in x's dtype (is_bf16) after fp32
 * accumulation in the fixed order of sv_colsum: the backward of the per-scene broadcast (reference:
 * model/openvocab.py:170-173 `repeat` of the object features over the U utterances of a scene), the U-sum of the (B, U, O*D)
 * gradient.  scratch: sv_colsum_batched_scratch_floats(B, R, N) floats. */
int sv_colsum_batched(const void *x, long long row_stride, long long batch_stride, int is_bf16, int B, int R, int N, void *out,
                      float *scratch, void *stream);
long long sv_colsum_batched_scratch_floats(int B, int R, int N);

/* calc_pairwise_locs, 'center' relation (reference: modules/utils.py:38-87): centers (B,O,*) f32 with row stride
 * row_stride (>= 3 floats; xyz first) -> out (B,O,O,5) f32 = [dist/max_dist, dz/dist, dist2d/dist, dy/dist2d, dx/dist2d];
 * dist_norm = 0 keeps the raw distance in slot 0.  eps sits inside the square roots (1e-10 in the reference). */
int sv_pairwise_locs_f32(const float *centers, int row_stride, int B, int O, float eps, int dist_norm, float *out,
                         void *stream);

/* Fused softmax cross-entropy, forward + gradient (reference: optim/loss/loss.py:8-9,56-61 — F.cross_entropy with
 * ignore_index): logits (R,V) bf16 (is_bf16 = 1) or f32, rows row_stride elements apart; labels (R) int64.
 * loss_rows[r] = logsumexp(row) - row[label] (0 for ignored rows); grad_logits (R, grad_row_stride >= V, same dtype, may be
 * NULL) = softmax(row) - onehot(label) (zero rows for ignored labels), columns [V, grad_row_stride) written as zeros — the
 * gradient of a vocabulary padded to 16-byte rows (BERT LM head, V = 30522 -> 30528) feeds the backward GEMMs directly.
 * The caller divides by the number of valid rows. */
int sv_cross_entropy_fwd_bwd_strided(const void *logits, long long row_stride, int is_bf16, const long long *labels, int R,
                                     int V, long long ignore_index, float *loss_rows, void *grad_logits,
                                     long long grad_row_stride, void *stream);

/* Binary cross-entropy with logits, forward + gradient in one launch (reference: optim/loss/loss.py:50-53 `answer_loss`, and
 * the ScanQA form of optim/loss/contra_loss.py:33-34 — F.binary_cross_entropy_with_logits(x, y.float(), weight=w,
 * reduction='sum') / R).  logits (R, row_stride >= C) bf16 (is_bf16 = 1) or f32, columns [0, C) used; labels (R, C) int64
 * contiguous; weight (R, C) bytes (bool: nonzero = 1) or NULL.
 * loss_rows[r] = sum_c w (max(x,0) - x y + log1p(exp(-|x|)));  *loss_out = (sum_r loss_rows[r]) / R, the rows added in a fixed
 * order (bitwise reproducible).  counter: a zero-initialised device word, left at zero on completion (one per stream).
 * grad_logits (may be NULL): w (sigmoid(x) - y), same dtype, rows grad_row_stride (>= C) elements apart, columns
 * [C, grad_row_stride) written as zeros — NOT yet scaled by dL/dloss / R (sv_scale_inplace does that in the backward). */
int sv_bce_logits_fwd_bwd(const void *logits, long long row_stride, int is_bf16, const long long *labels,
                          const unsigned char *weight, int R, int C, float *loss_rows, float *loss_out, unsigned *counter,
                          void *grad_logits, long long grad_row_stride, void *stream);

/* Masked soft-attention pooling of one glimpse (reference: modules/heads/qa_head.py:42-70 AttFlat with flat_glimpses = 1).
 * score: the (B*L, score_rs) bf16 output of the N = 1 score linear (column 0 used; score_rs = 8 for the padded rows of the
 * native linear); x (B, L, D) bf16 with batch stride x_bs and row stride x_rs (elements, % 8 == 0, 16-byte aligned base),
 * D % 8 == 0; pad_mask (B, L) bytes, nonzero = masked (may be NULL); 1 <= L <= 8192.
 * forward:  s = pad_mask ? -1e9 : score (exactly the reference's fp32 fill: a fully masked row gets weights 1/L);
 *           p (B, L) f32 = softmax over L of s (saved for the backward); pooled (B, D) bf16 = sum_l p_l x_l (fp32 accumulation).
 * backward: dpooled (B, D) bf16, row stride dp_rs; dx (B, L, D) bf16 contiguous = p_l dpooled;
 *           dscore (B*L, score_rs) bf16: column 0 = p_l (<dpooled, x_l> - sum_l' p_l' <dpooled, x_l'>), 0 at masked positions,
 *           columns 1.. zero — the padded gradient the score linear's backward reads. */
int sv_attn_pool_fwd(const void *score, int score_rs, const void *x, long long x_bs, int x_rs, const unsigned char *pad_mask,
                     int B, int L, int D, float *p, void *pooled, void *stream);
int sv_attn_pool_bwd(const void *dpooled, int dp_rs, const float *p, const void *x, long long x_bs, int x_rs,
                     const unsigned char *pad_mask, int B, int L, int D, void *dx, void *dscore, int score_rs, void *stream);

/* Backward of a stand-alone activation behind a linear layer (the FFN form fuses this into sv_linear_dgrad_bf16):
 * out = g x act'(.), (M,N) bf16, N % 8 == 0.  mode 1: relu, aux = forward output; mode 2: gelu(erf), aux = pre-activation. */
int sv_act_bwd_bf16(const void *g, int ldg, const void *aux, int ld_aux, int mode, int M, int N, void *out, int ldo,
                    void *stream);

/* x[0..n) *= *scale (device scalar) in place, bf16 | f32, n % (8 | 4) == 0, 16-byte aligned: the 1/count scaling of the fused
 * cross-entropy gradient without a second (R, V) tensor. */
int sv_scale_inplace(void *x, long long n, int is_bf16, const float *scale, void *stream);

/* Gradient of an embedding lookup: dw[ids[t]][:] += grad_out[t][:] (fp32 red.add; rows with ids == padding_idx skipped).
 * grad_out (ntok, D) bf16 | f32 with row stride ldg; dw (vocab, D) f32 contiguous, NOT zeroed here (accumulates).
 * (reference: autograd of the three nn.Embedding tables of HF BertEmbeddings, modules/language/bert.py:21-26) */
int sv_embedding_bwd(const void *grad_out, long long ldg, int is_bf16, const long long *ids, int ntok, int D, long long vocab,
                     long long padding_idx, float *dw, void *stream);

/* clip_grad_norm_ + AdamW + bf16 shadow refresh over FLAT buffers in two launches (squared-norm partials, then the update;
 * reference: trainer/build.py:135-145, optim/utils.py:1-18).  params / exp_avg / exp_avg_sq / grads: n f32, 16-byte aligned;
 * shadow_bf16: n bf16, 8-byte aligned (may be NULL).  segments: DEVICE array of nseg records {long long begin, end; float
 * lr_scale, weight_decay} (element ranges, multiples of 4), 8-byte aligned — lr of a segment = base_lr * lr_scale * *lr_factor.
 * step: device 1-based step counter (bias correction).  scratch: sv_adamw_scratch_floats() floats.  norm_out (may be NULL)
 * receives ||g||.  max_norm <= 0 disables clipping.  A non-finite norm poisons the update as it does in clip_grad_norm_: NaN
 * makes every updated element NaN, inf gives a clip factor of 0. */
int sv_adamw_scratch_floats(void);
int sv_adamw_flat(float *params, float *exp_avg, float *exp_avg_sq, const float *grads, void *shadow_bf16, long long n,
                  const void *segments, int nseg, float max_norm, const float *lr_factor, const long long *step, float base_lr,
                  float beta1, float beta2, float eps, float *scratch, float *norm_out, void *stream);

/* ---- train-mode PointNet++ set abstraction in channels-last form (config C2: ObjCls pre-training with a trainable backbone) ----
 * A grouped tensor is the row matrix X[(b, centre, sample)][channel] in bf16: the 1x1 convolutions are sv_linear_*_bf16 (no bias),
 * BatchNorm2d with BATCH statistics is a column statistic over the rows, the neighbourhood max is a max over ns consecutive rows.
 * Reference: pointnet2_utils.py:291-373 (QueryAndGroup / GroupAll), pytorch_utils.py:11-36,67-120 (SharedMLP: Conv2d + BatchNorm2d +
 * ReLU), pointnet2_modules.py:70-73 (max_pool2d over nsample).
 * group_rows: X (B*np*ns, Cp) bf16, Cp % 8 == 0, Cp >= 3 + C: [xyz[idx] - centre | feat[idx] | 0]; centre NULL = raw xyz (GroupAll);
 * idx (B,np,ns) i32 or NULL (GroupAll: every point in order, np = 1, ns = N); feat (B,N,C) point-major f32 | bf16.
 * group_rows_grad: dfeat (B,N,C) f32 (zeroed here) += dX[:, 3:3+C] scattered by idx. */
int sv_pn_group_rows(const float *xyz, const float *centre, const void *feat, int feat_bf16, const int *idx, int B, int N, int C,
                     int np, int ns, int Cp, void *X, void *stream);
int sv_pn_group_rows_grad(const void *dX, const int *idx, int B, int N, int C, int np, int ns, int Cp, float *dfeat, void *stream);
/* BatchNorm (batch statistics over the R rows, biased variance) + ReLU: y, out (R,C) bf16; mean, rstd (C) f32 out; var_unbiased (C)
 * f32 out (may be NULL; for the running estimate); scratch: sv_pn_scratch_floats(C).  Backward: dy = d(out)/d(y) applied to dout,
 * dgamma / dbeta (C) f32 overwritten or accumulated. */
int sv_pn_scratch_floats(int C);
int sv_pn_bn_relu_fwd(const void *y, long long R, int C, const float *gamma, const float *beta, float eps, float *mean, float *rstd,
                      float *var_unbiased, void *out, float *scratch, void *stream);
int sv_pn_bn_relu_bwd(const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta, const float *mean,
                      const float *rstd, void *dy, float *dgamma, float *dbeta, int accumulate, float *scratch, void *stream);
/* The same layer with SyncBatchNorm statistics over `world` ranks (reference: model/objcls.py:33-34 convert_sync_batchnorm;
 * torch.nn.SyncBatchNorm semantics: mean / variance over the rows of all ranks, d gamma / d beta stay this rank's sums, dY uses
 * the global sums and 1 / R_total).  Each BatchNorm pass is two launches, push then finish, so that ranks exchange their column
 * sums in between:
 *   push (mode 0: sum y, sum y^2; mode 1: sum g', sum g' * xhat with the global mean / rstd) reduces this rank's R rows (R = 0
 *   allowed) to fp64 and stores [sum0 (C) | sum1 (C) | R] into this rank's slot of every rank's exchange buffer, then raises
 *   this rank's flag on every rank;
 *   finish waits for every rank's flag, sums the slots in rank order (bit-identical on every rank) and applies the layer.
 * peer_bufs: DEVICE array of `world` device pointers to the ranks' exchange buffers (8-byte aligned), each
 * sv_pn_sync_floats(cap, world) floats, zero-initialised, with C <= cap; one buffer serves every layer on one stream.
 * epoch_dev: zero-initialised device word of this rank: push uses *epoch_dev + 1, finish stores it back (CUDA-graph replay).
 * done_counter: zero-initialised device word, reset by push.  scratch: sv_pn_scratch_floats(C).  gsum: (2C + 1) f32 out, the
 * global sums and 1 / R_total that the dY kernel reads.  Returns 0 floats for an invalid C or world. */
int sv_pn_sync_floats(int C, int world);
int sv_pn_bn_sync_push(int mode, const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta,
                       const float *mean, const float *rstd, float *scratch, void *const *peer_bufs, int cap, unsigned *done_counter,
                       int world, int rank, const unsigned *epoch_dev, void *stream);
int sv_pn_bn_sync_finish_fwd(const void *y, long long R, int C, const float *gamma, const float *beta, float eps, float *mean,
                             float *rstd, float *var_unbiased, void *out, void *const *peer_bufs, int cap, int world, int rank,
                             unsigned *epoch_dev, void *stream);
int sv_pn_bn_sync_finish_bwd(const void *y, const void *dout, long long R, int C, const float *gamma, const float *beta,
                             const float *mean, const float *rstd, void *dy, float *dgamma, float *dbeta, int accumulate, float *gsum,
                             void *const *peer_bufs, int cap, int world, int rank, unsigned *epoch_dev, void *stream);
/* out[g][c] = max over the ns rows of group g, arg = index of the first maximum (bytes, ns <= 255); grad: gx[g*ns+s][c] = gout[g][c]
 * where s == arg, else 0. */
int sv_pn_rowgroup_max(const void *x, long long G, int ns, int C, void *out, unsigned char *arg, void *stream);
int sv_pn_rowgroup_max_grad(const void *gout, const unsigned char *arg, long long G, int ns, int C, void *gx, void *stream);

/* L2-normalise + all-gather fused over NVLink peer memory (reference: contra_loss.py:58-64,86-91 + dist_utils.py:131-149).
 * a, b: local (n,D) f32.  peer_bufs[world] / peer_signals[world]: DEVICE arrays of device pointers into a symmetric
 * allocation mapped on every rank: buffer = [2 parities][2 tensors][world*n][D] f32, signal = >= world uint32 words
 * (zero-initialised).  The epoch is kept in device memory (*epoch_dev, zero-initialised, one word per exchange object): the
 * launch uses epoch = *epoch_dev + 1 and stores it back on completion, so a captured CUDA graph (frozen arguments) can replay
 * it.  When the kernel completes the local buffer holds, for parity epoch&1, normalize(a) and normalize(b) of all ranks in
 * rank-major order. */
int sv_normalize_allgather_dev_f32(const float *a, const float *b, int n, int D, void *const *peer_bufs,
                                   void *const *peer_signals, unsigned *done_counter, int world, int rank,
                                   unsigned *epoch_dev, void *stream);

/* Evaluation metrics (csrc/eval_metrics.cu; reference: evaluator/*.py `batch_metrics`).  Each evaluator owns one zeroed device
 * vector of sv_eval_counters_size(kind) doubles; the kernels ADD one batch into it (atomics, CUDA-graph replay safe).  Counts
 * are integers held exactly in float64.  Logits are bf16 (is_bf16 != 0) or f32 rows with a row stride in elements (padded
 * vocabularies are read in place).  valid: (B,) bytes or NULL (all valid); an item with valid 0 counts nothing. */
enum { SV_EVAL_GROUNDING = 0, SV_EVAL_OBJ_CLS = 1, SV_EVAL_ANSWERS = 2, SV_EVAL_PRETRAIN = 3 };
/* ScanReferEval / ReferIt3DEval: items; is_multiple / is_hard / is_view_dependent items; og_pred == tgt_object_id (all, hard,
 * view-dependent); IoU-25 / IoU-50 flag at og_pred (all, multiple); txt_acc; then up to three (hits, masked objects) pairs of
 * sv_eval_obj_cls at SV_EVG_OBJ. */
enum {
  SV_EVG_ITEMS = 0, SV_EVG_MULTIPLE, SV_EVG_HARD, SV_EVG_VIEW_DEP, SV_EVG_OG_ACC, SV_EVG_OG_ACC_HARD, SV_EVG_OG_ACC_VIEW_DEP,
  SV_EVG_IOU25, SV_EVG_IOU50, SV_EVG_IOU25_MULTIPLE, SV_EVG_IOU50_MULTIPLE, SV_EVG_TXT_ACC, SV_EVG_OBJ, SV_EVG_SIZE = SV_EVG_OBJ + 6
};
/* PretrainObjEval: one (hits, masked objects) pair */
enum { SV_EVO_HIT = 0, SV_EVO_COUNT = 1, SV_EVO_SIZE = 2 };
/* ScanQAEval / SQA3DEval: items, top-1 and top-10 hits, items and top-1 hits per sqa_type (6 types), the (hits, masked
 * objects) pair of obj_cls_raw; then SQA3DEval's state: a snapshot of those integers at the end of the previous batch and its
 * float64 sums of per-batch ratio x batch size (ans1 = target_metric, ans10, obj_cls_raw, type k) and of the type counts. */
enum {
  SV_EVA_NTYPES = 6,
  SV_EVA_ITEMS = 0, SV_EVA_ANS1 = 1, SV_EVA_ANS10 = 2, SV_EVA_TYPE_ITEMS = 3, SV_EVA_TYPE_ANS1 = 9, SV_EVA_OBJ_HIT = 15,
  SV_EVA_OBJ_COUNT = 16, SV_EVA_SNAPSHOT = 17, SV_EVA_Q_ANS1 = 34, SV_EVA_Q_ANS10 = 35, SV_EVA_Q_OBJ = 36, SV_EVA_Q_TYPE = 37,
  SV_EVA_Q_TYPE_COUNT = 43, SV_EVA_SIZE = 49
};
/* PretrainEval: the grounding words SV_EVG_ITEMS..SV_EVG_TXT_ACC at SV_EVP_OG (of them only og_acc is reported); items;
 * masked-LM hits and labelled tokens; then, for each object logits tensor present in the order post, raw, pre (the
 * SV_EVP_HAS_* bits), six words: (hits, rows) over obj_masks, obj_masks & obj_sem_masks, obj_masks & !obj_sem_masks.  Then
 * a snapshot of those SV_EVP_SNAPSHOT integers at the end of the previous batch, and the float64 sums of per-batch metric x
 * items at SV_EVP_Q + SV_EVP_Q_*, in the reference's eval_dict order. */
enum {
  SV_EVP_OG = 0, SV_EVP_ITEMS = SV_EVG_OBJ, SV_EVP_LM_HIT, SV_EVP_LM_COUNT, SV_EVP_OBJ, SV_EVP_SNAPSHOT = SV_EVP_OBJ + 18,
  SV_EVP_Q = 2 * SV_EVP_SNAPSHOT, SV_EVP_SIZE = SV_EVP_Q + 10,
  SV_EVP_Q_TARGET = 0, SV_EVP_Q_OG, SV_EVP_Q_LM, SV_EVP_Q_POST, SV_EVP_Q_PRE, SV_EVP_Q_RAW, SV_EVP_Q_PRE_UNMASK,
  SV_EVP_Q_PRE_MASK, SV_EVP_Q_POST_UNMASK, SV_EVP_Q_POST_MASK,
  SV_EVP_HAS_OG = 1, SV_EVP_HAS_POST = 2, SV_EVP_HAS_RAW = 4, SV_EVP_HAS_PRE = 8
};
int sv_eval_counters_size(int kind);
/* og_pred = argmax of og3d_logits (B, O) (torch's rule: first maximum, NaN above everything), element (b, o) at
 * b * og_row_stride + o * og_col_stride (the grounding head writes it as column 0 of padded rows).  tgt_object_id (B) int64.
 * iou25 / iou50: (B, >= O) int64 rows or both NULL (ReferIt3D).  txt_cls_logits (B, txt_classes) rows or NULL, against
 * tgt_object_label (B) int64.  Flags: (B) bytes or NULL (= 0). */
int sv_eval_grounding(const void *og3d_logits, int og_bf16, long long og_row_stride, long long og_col_stride, int B, int O,
                      const long long *tgt_object_id, const long long *iou25, const long long *iou50, long long iou_row_stride,
                      const void *txt_cls_logits, int txt_bf16, long long txt_row_stride, int txt_classes,
                      const long long *tgt_object_label, const unsigned char *is_multiple, const unsigned char *is_hard,
                      const unsigned char *is_view_dependent, const unsigned char *valid, double *counters, void *stream);
/* Up to three (B, O, C) logits tensors (host arrays of device pointers / dtypes / strides in elements): for tensor t,
 * counters[2t] += #{masked objects whose argmax over C equals obj_labels}, counters[2t + 1] += #{masked objects}.
 * obj_labels (B, O) int64, obj_masks (B, O) bytes.  split_mask (B, O) bytes or NULL: tensor t then adds into
 * counters[6t .. 6t + 5] the (hits, masked objects) pairs over obj_masks, obj_masks & split_mask, obj_masks & !split_mask. */
int sv_eval_obj_cls(int n_logits, const void *const *logits, const int *is_bf16, const long long *row_stride,
                    const long long *item_stride, int B, int O, int C, const long long *obj_labels,
                    const unsigned char *obj_masks, const unsigned char *split_mask, const unsigned char *valid,
                    double *counters, void *stream);
/* answer_scores (B, A) rows; answer_label (B, A) int64 multi-hot (a 1 marks a correct answer).  Top-1 hit: the argmax is
 * labelled 1.  Top-10 hit: a labelled answer ranks among the first 10 (scores descending, NaN first, ties: lower index first).
 * sqa_type (B) int64 in 0..5 or NULL.  Adds into the SV_EVA_* words. */
int sv_eval_answers(const void *answer_scores, int is_bf16, long long row_stride, int B, int A, const long long *answer_label,
                    const long long *sqa_type, const unsigned char *valid, double *counters, void *stream);
/* SQA3DEval.update's float64 bookkeeping for the batch just added (after sv_eval_answers and sv_eval_obj_cls of that batch). */
int sv_eval_sqa3d_batch(double *counters, void *stream);
/* Masked-LM accuracy: logits (R, V) rows (row_stride >= V elements; a padded vocabulary is read in place, its pad columns
 * never), R = B * L token rows, masked_lm_labels (R) int64 with -1 = not labelled.  counters[SV_EVP_LM_HIT] += #{labelled rows
 * whose argmax equals the label}, counters[SV_EVP_LM_COUNT] += #{labelled rows}, counters[SV_EVP_ITEMS] += #{valid items};
 * row r belongs to item r / L. */
int sv_eval_lm_acc(const void *logits, int is_bf16, long long row_stride, long long R, int V, int L,
                   const long long *masked_lm_labels, const unsigned char *valid, double *counters, void *stream);
/* PretrainEval.update's float64 bookkeeping for the batch just added; present = the SV_EVP_HAS_* bits of that batch. */
int sv_eval_pretrain_batch(double *counters, int present, void *stream);
/* One train-log entry: if advance_step, *step += 1 first; then row (*step % slots) of ring ((slots, 1 + n_values +
 * n_counters) doubles) = [*step, *values[0..n_values), counters[0..n_counters)].  values: host array of device pointers to
 * one float each (n_values <= SV_TRAIN_LOG_MAX_VALUES). */
enum { SV_TRAIN_LOG_MAX_VALUES = 32 };
int sv_train_log_write(int n_values, const float *const *values, const double *counters, int n_counters, long long *step,
                       int advance_step, double *ring, int slots, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SVGPS_H */
