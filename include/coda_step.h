/*
 * coda_step.h -- C ABI of the step-glue kernels: what sits between the tensor-core contractions of one
 * CoDA training step and what closes it (global-norm clip + AdamW on the flat parameter buffer).
 *
 * In the reference these are ATen launches issued by Python:
 *   - `src + self.dropout1(src2)` style residual connections and nn.Dropout
 *       (models/transformer.py:461-479, :556-580; models/helpers.py:45-112 dropout=0.3 in the heads)
 *   - nn.BatchNorm1d (+ ReLU + Dropout) of GenericMLP (models/helpers.py:82-99) on (B, C, L) conv maps
 *   - torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW.step (engine.py:161-164, optimizer.py:4-36)
 *   - BoxProcessor (models/model_3detr.py:56-127) + the corner builders (utils/box_util.py:383-490)
 *   - the fp64 corner projection of the CLIP crop pipeline (models/model_3detr.py:912-968,
 *     datasets/sunrgbd_utils.py:611-635)
 *
 * Conventions as in coda_pointnet2.h: raw device pointers, dense row-major fp32 unless stated, `void *stream`
 * is a cudaStream_t, int status (0 = ok).  Nothing allocates or synchronises.
 *
 * Dropout masks are counter-based: element i of a call is kept iff hash(seed[0] + salt, i) >= p * 2^32, where
 * `seed` is a device uint32 that the step advances once per iteration (inside the CUDA graph) and `salt`
 * identifies the call site.  The backward regenerates the mask; nothing is stored.
 */
#ifndef CODA_STEP_H
#define CODA_STEP_H

#ifdef __cplusplus
extern "C" {
#endif

/* out[i] = (resid ? resid[i] : 0) + keep(i) * x[i] / (1 - p);  p == 0 -> plain add.  n % 4 == 0 is NOT required. */
int coda_dropout_add_fwd(long long n, const float *x, const float *resid, float p, unsigned salt,
                         const unsigned *seed, float *out, void *stream);
/* dx[i] = keep(i) * dout[i] / (1 - p)  (the residual branch's gradient is dout itself) */
int coda_dropout_bwd(long long n, const float *dout, float p, unsigned salt, const unsigned *seed, float *dx,
                     void *stream);

/*
 * BatchNorm (given batch statistics, see coda_bn_rows_stats in coda_sa_mlp.h) + optional ReLU + optional dropout
 * on channels-last rows (rows, c):  out = drop( relu( (y - mean) * invstd * gamma + beta ) ).
 * Channel rule as in coda_sa_mlp.h (c % 4 == 0, 256 % (c / 4) == 0).
 */
int coda_bn_act_rows_fwd(long long rows, int c, const float *y, const float *mean, const float *invstd,
                         const float *gamma, const float *beta, int relu, float p, unsigned salt,
                         const unsigned *seed, float *out, void *stream);
/* s1[c] = sum_r dz, s2[c] = sum_r dz * xhat with dz = dout * dropmask * relumask  (= dbeta, dgamma);
 * scratch: coda_bn_rows_scratch_floats(c) floats. */
int coda_bn_act_rows_bwd_reduce(long long rows, int c, const float *y, const float *dout, const float *mean,
                                const float *invstd, const float *gamma, const float *beta, int relu, float p,
                                unsigned salt, const unsigned *seed, float *s1, float *s2, float *scratch,
                                void *stream);
/* dy = gamma * invstd * (dz - s1 / rows - xhat * s2 / rows), fp32 (rows, c) */
int coda_bn_act_rows_bwd(long long rows, int c, const float *y, const float *dout, const float *mean,
                         const float *invstd, const float *gamma, const float *beta, int relu, float p,
                         unsigned salt, const unsigned *seed, const float *s1, const float *s2, float *dy,
                         void *stream);

/*
 * out[i] = srcs[0][i] + ... + srcs[count - 1][i], 1 <= count <= 16; `srcs` is a HOST array of device pointers
 * (16-byte aligned).  The gradient fan-in of a tensor consumed by several branches (the six prediction heads of
 * models/model_3detr.py:1634-1660 on the decoder output, the 2 x dec_nlayers uses of the query embedding in
 * models/transformer.py:556-580) in one pass -- autograd's own accumulation runs count - 1 binary adds.
 * out may alias any of the sources.
 */
int coda_sum_n(long long n, int count, const float *const *srcs, float *out, void *stream);

/*
 * Masked L1 between the heads' 512-d embedding and the CLIP embedding of the boxes' image crops
 * (criterion.py:924-943 loss_predicted_region_embed_l1):
 *   out[l] = sum_{r, k} | pred[l][r][k] * w[r] - target[r][k] * w[r] |,  pred (layers, rows, d), target (rows, d),
 *   w (rows), d % 4 == 0; the target is broadcast over the layers, not repeated.  Deterministic two-stage sum;
 *   scratch: coda_masked_l1_scratch_floats(layers) floats.
 *   backward: dpred[l][r][k] = g[l] * sgn(pred * w - target * w) * w[r]
 */
long long coda_masked_l1_scratch_floats(int layers);
int coda_masked_l1_fwd(int layers, long long rows, int d, const float *pred, const float *target, const float *w,
                       float *out, float *scratch, void *stream);
int coda_masked_l1_bwd(int layers, long long rows, int d, const float *pred, const float *target, const float *w,
                       const float *g, float *dpred, void *stream);

/*
 * Row-wise cross-entropy of the stage-2 contrastive loss over a shared text matrix (criterion.py
 * loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi, reference criterion.py:598-644), on raw logits
 * S = e T^T that a GEMM has already written:
 *   S     (rows, ld) fp32, columns [0, c) used, ld % 4 == 0, ld >= c;  e (rows, d) fp32 the un-normalised embeddings,
 *   d % 4 == 0;  label (rows) int64;  w (rows) fp32 the per-row weights;  scale one device fp32 (logit scale, clipped).
 * Forward, per row r:
 *   inv[r] = 1 / (||e_r|| + 1e-32),  z_rc = scale * inv[r] * S_rc,  lse[r] = log sum_c exp(z_rc),
 *   loss[r] = w[r] * (lse[r] - z_{r, label[r]});  label -100 -> loss 0 (ignore_index); any other label outside
 *   [0, c) -> NaN.
 * Backward, with g (rows) = dL / dloss and G_rc = g[r] * w[r] * (softmax_rc - [c == label[r]]):
 *   dS_rc = scale * inv[r] * G_rc for c < c, 0 for c <= col < ld;
 *   dnorm[r] = coef_r * e_r with coef_r = -(inv[r] / ||e_r||) * sum_c G_rc z_rc  (0 for a zero row): the
 *   gradient through the normalisation, which the caller adds to the GEMM's dS T.  A label -100 row gets zeros,
 *   an out-of-range label NaN.
 * One warp per row, fixed lane-strided order and shuffle trees: the same bits on every run.  No atomics, no
 * allocation, no synchronisation.
 */
int coda_text_ce_fwd(long long rows, int c, int ld, int d, const float *S, const float *e, const long long *label,
                     const float *w, const float *scale, float *loss, float *lse, float *inv, void *stream);
int coda_text_ce_bwd(long long rows, int c, int ld, int d, const float *S, const float *e, const long long *label,
                     const float *w, const float *scale, const float *lse, const float *inv, const float *g,
                     float *dS, float *dnorm, void *stream);

/*
 * Global-norm gradient clip + AdamW over ONE flat fp32 parameter buffer.
 *
 * coda_grad_norm: state[1] = ||grad * grad_scale||_2 over the `n` elements (deterministic two-stage sum, fp64
 *   final stage), state[2] = clip coefficient min(1, max_norm / (norm + 1e-6)) (1 if max_norm <= 0) --
 *   torch.nn.utils.clip_grad_norm_ -- and advances the step counter state[0] by one, caching the bias
 *   corrections state[3] = 1 - beta1^t, state[4] = sqrt(1 - beta2^t).
 *   scratch: coda_grad_norm_scratch_floats() floats.  state: 8 floats, zero-initialised by the caller once.
 * coda_adamw_update: torch.optim.AdamW (decoupled weight decay, no amsgrad) with the clipped, scaled gradient
 *   g = grad * grad_scale * state[2]:
 *       p *= 1 - lr * wd;  m += (g - m)(1 - beta1);  v = beta2 v + (1 - beta2) g^2;
 *       p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
 *   over a table of chunks (device array): each chunk is a run of elements of one parameter tensor with its own
 *   weight decay; elements not covered by any chunk are left untouched (parameters that receive no gradient:
 *   the reference's optimizer skips `grad is None` parameters).  lr is read from the device (`lr_dev`).
 */
typedef struct {
  long long offset;   /* first element in the flat buffers */
  int len;            /* number of elements (<= 65536) */
  float weight_decay;
} coda_opt_chunk;

long long coda_grad_norm_scratch_floats(void);
int coda_grad_norm(long long n, const float *grad, float grad_scale, float max_norm, float beta1, float beta2,
                   float *scratch, float *state, void *stream);
int coda_adamw_update(int nchunks, const coda_opt_chunk *chunks, float *param, const float *grad, float *exp_avg,
                      float *exp_avg_sq, const float *lr_dev, float grad_scale, float beta1, float beta2, float eps,
                      const float *state, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_STEP_H */
