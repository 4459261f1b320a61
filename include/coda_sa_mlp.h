/*
 * coda_sa_mlp.h -- C ABI of the row-streaming kernels that sit between the tensor-core GEMMs of the
 * PointNet++ set-abstraction shared MLP (1x1 Conv2d -> BatchNorm2d -> ReLU, three times, then a max
 * over the `nsample` neighbours of every seed).
 *
 * Replaces, on the training-step path,
 *   third_party_pointnet2/pointnet2/pytorch_utils.py:8-33   (SharedMLP = Conv2d + BatchNorm2d + ReLU blocks)
 *   third_party_pointnet2/pointnet2/pointnet2_modules.py:248-254 (PointnetSAModuleVotes: F.max_pool2d over nsample)
 * which the reference runs as cuDNN convolution + ATen batch-norm / ReLU / pooling kernels, one full
 * pass over the (B * npoint * nsample, C) activation each.  Here the activation is kept channels-last
 * ("rows" = B * npoint * nsample, C channels), the convolutions are the split-bf16 wgmma GEMMs of
 * coda_gemm.h, and everything between two GEMMs is ONE pass: normalise + ReLU + split into the bf16
 * operand planes the next GEMM reads (no fp32 intermediate is written), the last block folds the max
 * over neighbours in as well, and the backward mirrors it (mask + BatchNorm backward + operand planes
 * of the gradient in one pass).
 *
 * All pointers are device pointers, all matrices row-major fp32 unless stated, `stream` is a
 * cudaStream_t.  Channel counts must satisfy c % 4 == 0 and 256 % (c / 4) == 0 (c = 4 .. 1024, powers
 * of two times 4); the plane-writing entry points additionally need c % 64 == 0 (GEMM K granularity).
 * Returns 0 or a coda_status code (coda_pointnet2.h).  Nothing synchronises or allocates.
 */
#ifndef CODA_SA_MLP_H
#define CODA_SA_MLP_H

#ifdef __cplusplus
extern "C" {
#endif

/* floats of scratch the statistics / reduction entry points need for `c` channels */
long long coda_bn_rows_scratch_floats(int c);

/*
 * y (rows, cout) = x (rows, cin) @ w (cout, cin)^T for a tiny cin (<= 8: the xyz(+feature) input of the
 * first shared-MLP layer), exact fp32 FMAs on the CUDA cores -- a K = 3 contraction is not tensor-core work.
 */
int coda_rows_linear_small_k(long long rows, int cin, int cout, const float *x, const float *w, float *y,
                             void *stream);

/*
 * Batch statistics of y (rows, c) over rows (BatchNorm training mode): mean[c], invstd[c] =
 * 1 / sqrt(biased var + eps); if running_mean / running_var are non-NULL they are updated in place with
 * `momentum` (unbiased variance), as nn.BatchNorm2d does.  Deterministic two-stage reduction.
 */
int coda_bn_rows_stats(long long rows, int c, const float *y, float eps, float momentum, float *running_mean,
                       float *running_var, float *mean, float *invstd, float *scratch, void *stream);

/* As coda_bn_rows_stats, plus the folded affine map scale = gamma * invstd, shift = beta - mean * scale
 * (zero-padded to a multiple of 64 entries) for the next GEMM's CODA_A32_AFFINE_RELU prologue. */
int coda_bn_rows_stats_affine(long long rows, int c, const float *y, float eps, float momentum, float *running_mean,
                               float *running_var, const float *gamma, const float *beta, float *mean, float *invstd,
                               float *scale, float *shift, float *scratch, void *stream);

/*
 * The same statistics from per-CTA partial column sums partial[nblocks][2][c] (sum | sum of squares) that a GEMM
 * epilogue wrote (coda_gemm_a32 `col_stats`): no pass over the activation at all.  Optionally also emits the folded
 * affine map of BatchNorm, scale[c] = gamma * invstd, shift[c] = beta - mean * scale (zero-padded to a multiple of
 * 64 entries), which the next GEMM applies in its A prologue (CODA_A32_AFFINE_RELU).
 */
int coda_bn_stats_finalize(int nblocks, long long rows, int c, const float *partial, float eps, float momentum,
                           float *running_mean, float *running_var, const float *gamma, const float *beta,
                           float *mean, float *invstd, float *scale, float *shift, void *stream);
/*
 * Synchronised BatchNorm (reference main.py:993, torch.nn.SyncBatchNorm.convert_sync_batchnorm): the statistics of a
 * layer are taken over the batches of ALL ranks.  Per rank: sums[0..c) = column sums, sums[c..2c) = column sums of
 * squares, in fp64, from a pass over y (coda_bn_rows_sums) or from the partials a GEMM epilogue wrote
 * (coda_bn_partials_sums).  The caller all-reduces `sums` (ONE 16*c-byte collective per layer) and finishes with
 * coda_bn_stats_finalize_sums(rows = global row count): mean, invstd, running buffers (unbiased variance over the
 * global count) and optionally the folded affine map (scale / shift padded to a multiple of 64).
 * Backward: the (s1, s2) sums of coda_*_bwd_reduce are all-reduced the same way (averaged: the kernels divide by
 * the local row count); dgamma / dbeta stay the local sums, as in torch's SyncBatchNorm.
 */
int coda_bn_rows_sums(long long rows, int c, const float *y, double *sums, float *scratch, void *stream);
int coda_bn_partials_sums(int nblocks, int c, const float *partial, double *sums, void *stream);
int coda_bn_stats_finalize_sums(long long rows, int c, const double *sums, float eps, float momentum,
                                float *running_mean, float *running_var, const float *gamma, const float *beta,
                                float *mean, float *invstd, float *scale, float *shift, void *stream);

/*
 * Per-channel coefficients of the BatchNorm(+ReLU) backward as a GEMM prologue (CODA_A32_BN_BWD*):
 *   dy = [y * scale + shift > 0] * scale * d + alpha * y + beta,
 *   alpha = -scale * invstd * s2 / rows,  beta = -scale * s1 / rows - alpha * mean   (padded to a multiple of 64)
 */
int coda_bn_bwd_coefs(int c, long long rows, const float *mean, const float *invstd, const float *gamma,
                      const float *s1, const float *s2, float *alpha, float *beta, void *stream);

/*
 * out[c] = sum over rows of x (rows, c): the bias gradient of a Linear (db = column sums of dY); deterministic
 * two-stage reduction; scratch as for coda_bn_rows_stats.   replaces `dy.sum(dim=0)` in the Linear backward.
 */
int coda_rows_colsum(long long rows, int c, const float *x, float *out, float *scratch, void *stream);

/*
 * planes = split_bf16( relu( (y - mean) * invstd * gamma + beta ) ): bf16 [nsplit][rows][c], the A operand of
 * the next coda_gemm_nt (and the row operand of coda_gemm_tn for its weight gradient).
 */
int coda_bn_relu_pack_rows(long long rows, int c, int nsplit, const float *y, const float *mean,
                           const float *invstd, const float *gamma, const float *beta, void *planes,
                           void *stream);

/*
 * Last block: pooled (groups, c) = max over the `group` consecutive rows of each group of
 * relu(bn(y)); argmax (groups, c) uint8 = row within the group (first maximum), group <= 256.
 */
int coda_bn_relu_maxpool_rows(long long groups, int group, int c, const float *y, const float *mean,
                              const float *invstd, const float *gamma, const float *beta, float *pooled,
                              unsigned char *argmax, void *stream);

/*
 * Backward of relu(bn(y)) given the gradient of its output, first half: s1[c] = sum_r dz_masked,
 * s2[c] = sum_r dz_masked * xhat  (= dbeta, dgamma), dz_masked = dz where bn(y) > 0 else 0.
 *   dense form  : dz (rows, c);
 *   pooled form : the output was max-pooled; dpooled (groups, c) + argmax (groups, c) stand for dz.  dprime
 *                 (groups, c), or NULL: receives [bn(y) > 0 at the arg-max row] * gamma * invstd * dpooled, the operand
 *                 of the CODA_A32_BN_BWD_POOLED_PRE prologue of coda_gemm_a32 / coda_gemm_tn32.
 */
int coda_bn_relu_bwd_reduce(long long rows, int c, const float *y, const float *dz, const float *mean,
                            const float *invstd, const float *gamma, const float *beta, float *s1, float *s2,
                            float *scratch, void *stream);
int coda_bn_relu_bwd_reduce_pooled(long long groups, int group, int c, const float *y, const float *dpooled,
                                   const unsigned char *argmax, const float *mean, const float *invstd,
                                   const float *gamma, const float *beta, float *s1, float *s2, float *scratch,
                                   float *dprime, void *stream);

/*
 * Second half: dy = gamma * invstd * (dz_masked - s1 / rows - xhat * s2 / rows), written directly as the
 * split-bf16 planes [nsplit][rows][c] that the input-gradient GEMM (coda_gemm_nt) and the weight-gradient GEMM
 * (coda_gemm_tn) consume.  Pass dz for the dense form, or dz == NULL with dpooled / argmax / group for the
 * pooled form.
 */
int coda_bn_relu_bwd_pack(long long rows, int c, int nsplit, const float *y, const float *dz,
                          const float *dpooled, const unsigned char *argmax, int group, const float *mean,
                          const float *invstd, const float *gamma, const float *beta, const float *s1,
                          const float *s2, void *planes, void *stream);

/*
 * Second half for the first layer (tiny cin): dy is not stored at all; dw (cout, cin) = sum_r dy[r, :]^T x[r, :]
 * is accumulated in the same pass.  scratch: gridDim * cout * cin floats, see coda_bn_rows_small_k_scratch_floats.
 */
long long coda_bn_rows_small_k_scratch_floats(int cin, int cout);
int coda_bn_relu_bwd_small_k(long long rows, int cin, int cout, const float *y, const float *dz, const float *mean,
                             const float *invstd, const float *gamma, const float *beta, const float *s1,
                             const float *s2, const float *x, float *dw, float *scratch, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_SA_MLP_H */
