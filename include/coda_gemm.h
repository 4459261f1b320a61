/*
 * coda_gemm.h -- C-ABI of the wgmma / TMA GEMM used for every dense layer on
 * the path (Linear / 1x1-Conv of the 3DETR encoder, decoder and heads, the SA
 * shared MLP, and the CLIP ViT blocks).  In the reference these are
 * nn.Linear / nn.Conv1d / nn.Conv2d(1x1) calls into cuBLAS / cuDNN
 * (models/helpers.py:45-112, models/transformer.py, pytorch_utils.py:8-33,
 * CLIP/clip/model.py:295-316).
 *
 * The GEMM is "NT": C[b][m][n] = sum_k A[b][m][k] * B[b][n][k] (+ bias[n]) (ReLU),
 * both operands K-contiguous 16-bit planes whose K extent is padded to a multiple
 * of 64.  fp32 tensors are first split into nsplit bf16 planes by
 * coda_pack_split_bf16 (x = p0 + p1 (+ p2), each the bf16 rounding of what the
 * previous planes left over); the GEMM accumulates the 1 / 3 / 6 significant
 * cross products in fp32 registers.  nsplit = 2 carries ~16 mantissa
 * bits per operand, nsplit = 3 the full 24.
 */
#ifndef CODA_GEMM_H
#define CODA_GEMM_H

#ifdef __cplusplus
extern "C" {
#endif

/*
 * src: fp32 matrix of `rows` x `k` addressed as src[r * src_row_stride + c * src_k_stride]
 *      (one of the two strides must be 1: plain or transposed source); every element is
 *      multiplied by `scale` before splitting.
 * planes: bf16 [nsplit][rows][kpad], zero-padded for k <= c < kpad.  kpad % 64 == 0.
 */
int coda_pack_split_bf16(long long rows, int k, int kpad, long long src_row_stride,
                         long long src_k_stride, const float *src, float scale, int nsplit,
                         void *planes, void *stream);

/* Same, with an explicit distance (elements) between consecutive planes, so that several
 * batch entries can be packed into one [nsplit][batch][rows][kpad] buffer. */
int coda_pack_split_bf16_strided(long long rows, int k, int kpad, long long src_row_stride,
                                 long long src_k_stride, const float *src, float scale, int nsplit,
                                 void *planes, long long plane_stride, void *stream);

/*
 * a: [nsplit planes][batch][m][kpad], plane / batch strides in ELEMENTS; b likewise with n rows;
 * b_batch_stride == 0 means one B shared by every batch entry (weights).
 * is_fp16: operands are IEEE fp16 instead of bf16 (requires nsplit == 1).
 * c: fp32, row stride ldc, batch stride c_batch_stride (elements).  bias may be NULL.
 */
int coda_gemm_nt(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                 long long a_plane_stride, long long a_batch_stride, const void *b,
                 long long b_plane_stride, long long b_batch_stride, const float *bias, int relu,
                 float *c, long long ldc, long long c_batch_stride, void *stream);

/* Extended form: `act` 0 none / 1 ReLU / 2 QuickGELU (x * sigmoid(1.702 x), CLIP/clip/model.py:263-265);
 * out_half != 0 writes C as IEEE fp16 (the CLIP ViT path keeps activations in fp16). */
int coda_gemm_nt_ex(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                    long long a_plane_stride, long long a_batch_stride, const void *b,
                    long long b_plane_stride, long long b_batch_stride, const float *bias, int act,
                    int out_half, void *c, long long ldc, long long c_batch_stride, void *stream);

/* As coda_gemm_nt_ex, plus a fused residual connection on the fp16 path: C = act(A B^T + bias) + residual,
 * residual (m, n) IEEE half with row stride ldr (multiple of 8), batch == 1, fp16 operands and output
 * (the `x + proj(...)` of the CLIP residual blocks, CLIP/clip/model.py:283-288).  NULL = no residual. */
int coda_gemm_nt_res(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                     long long a_plane_stride, long long a_batch_stride, const void *b,
                     long long b_plane_stride, long long b_batch_stride, const float *bias, int act,
                     int out_half, const void *residual, long long ldr, void *c, long long ldc,
                     long long c_batch_stride, void *stream);

/*
 * "TN" form for weight gradients: C[m][n] = sum_{r < mc} A[r][m] * B[r][n], with A planes
 * [nsplit][mc][lda] and B planes [nsplit][mc][ldb] (row-major, lda / ldb multiples of 64), i.e. the
 * contraction runs over ROWS of both stored operands (MN-major tensor-core operands): dW = dY^T X
 * straight from the row-packed dY and X, no transposed copies.  Split-K over mc when m x n is small.
 */
int coda_gemm_tn(int nsplit, int mc, int m, int n, const void *a, long long a_plane_stride, int lda,
                 const void *b, long long b_plane_stride, int ldb, float *c, long long ldc, void *stream);

/*
 * GEMM with an FP32 A operand and an in-kernel prologue (csrc/gemm_a32_sm90.cu):
 *
 *     C (m, n) fp32 = T(A) (m, k) @ B^T  (+ bias) (ReLU)
 *
 * A is read as fp32 rows (row stride lda, multiple of 4 elements, 16-byte aligned base) by TMA, transformed
 * element-wise by T, split into `nsplit` (2 or 3) bf16 planes and handed to the tensor cores as register
 * operands -- no packed copy of A exists in HBM.  T (`a_mode`), with per-k vectors padded to a multiple of 64 (the
 * element formulas, shared with coda_gemm_tn32, are in csrc/a32_prologue.cuh):
 *   CODA_A32_PLAIN          T = a                                   (every nn.Linear / 1x1 conv on the path)
 *   CODA_A32_AFFINE_RELU    T = relu(a * scale[k] + shift[k])       (BatchNorm(batch stats) + ReLU of the previous
 *                                                                    layer: pytorch_utils.py:8-33 SharedMLP blocks)
 *   CODA_A32_BN_BWD         T = [a * scale + shift > 0] * scale * a2 + a * alpha + beta
 *                               a = pre-BN activation, a2 (m, k) = gradient of relu(bn(a)): the BatchNorm+ReLU
 *                               backward folded into the input-gradient GEMM  dX = dY W
 *   CODA_A32_BN_BWD_POOLED  same, the gradient comes from a max-pooled output: a2 = dpooled (m / group, k),
 *                               argmax (m / group, k) uint8 = row within the group that produced the maximum
 * B: bf16 planes as produced by coda_pack_split_bf16, either K-major [n][b_ld] (b_mn = 0, b_ld >= pad64(k)) or
 * "MN-major" [k][b_ld] (b_mn = 1, b_ld >= n: the forward weight planes reused for the input gradient).
 * col_stats: NULL, or a ZERO-INITIALISED [coda_gemm_a32_grid(m, n)][2][n] float buffer that receives per-CTA partial
 * column sums and sums of squares of C (BatchNorm statistics of the layer just computed; n <= 512), to be finalised by
 * coda_bn_stats_finalize (coda_sa_mlp.h).
 */
#define CODA_A32_PLAIN 0
#define CODA_A32_AFFINE_RELU 1
#define CODA_A32_BN_BWD 2
#define CODA_A32_BN_BWD_POOLED 3
/* as _POOLED, but a2 already holds [bn(y) > 0 at the arg-max row] * scale * dpooled (coda_bn_relu_bwd_reduce_pooled's
 * `dprime`): the prologue is  T = [argmax == row] * a2 + a * alpha + beta  -- no ReLU test, no multiply per element */
#define CODA_A32_BN_BWD_POOLED_PRE 4
int coda_gemm_a32_grid(int m, int n);
int coda_gemm_a32(int nsplit, int m, int n, int k, const float *a, long long lda, int a_mode, const float *a_scale,
                  const float *a_shift, const float *a_alpha, const float *a_beta, const float *a2, long long lda2,
                  const unsigned char *a_argmax, int a_group, const void *b_planes, long long b_plane_stride,
                  int b_ld, int b_mn, const float *bias, int act, float *c, long long ldc, float *col_stats,
                  void *stream);

/*
 * Weight-gradient form on fp32 rows with in-kernel prologues (csrc/gemm_tn32_sm90.cu):
 *
 *     C (m, n) fp32 = sum_r TA(A)[r][:m]^T TB(B)[r][:n],   A (rows, m) with row stride lda, B (rows, n) with ldb
 *
 * TA: CODA_A32_PLAIN | CODA_A32_BN_BWD (a2 (rows, m) = gradient of relu(bn(a)), per-column scale / shift / alpha /
 * beta) | CODA_A32_BN_BWD_POOLED (a2 = dpooled (rows / group, m), argmax);  TB: CODA_A32_PLAIN |
 * CODA_A32_AFFINE_RELU (relu(b * b_scale + b_shift): the BatchNorm + ReLU that produced this layer's input).
 * Two bf16 planes per operand (gradient precision).  m, n, lda, ldb, ldc multiples of 4; per-column vectors have
 * at least m (resp. n) entries.  Split-K over all SMs; C is fully overwritten.
 * a_colsum (m floats, or NULL): overwritten with the column sums of TA(A) -- the bias gradient sum_r dY[r][:]
 * of the layer (torch.nn.Linear / Conv1d backward), accumulated by the transform warps from the values they already
 * hold instead of a second pass over dY.
 * Replaces, for dW = dY^T X of every 1x1 conv of the shared MLP (pytorch_utils.py:8-33 backward), the chain
 * "BatchNorm backward -> packed dY planes; packed X planes; packed TN GEMM".
 */
int coda_gemm_tn32(long long rows, int m, int n, const float *a, long long lda, int a_mode, const float *a_scale,
                   const float *a_shift, const float *a_alpha, const float *a_beta, const float *a2, long long lda2,
                   const unsigned char *a_argmax, int a_group, const float *b, long long ldb, int b_mode,
                   const float *b_scale, const float *b_shift, float *c, long long ldc, float *a_colsum, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_GEMM_H */
