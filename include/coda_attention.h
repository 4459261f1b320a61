/*
 * coda_attention.h -- C-ABI of the fused wgmma multi-head attention (forward and backward).
 *
 * Replaces the attention core of torch.nn.MultiheadAttention as the reference calls it
 * in TransformerEncoderLayer / TransformerDecoderLayer (models/transformer.py:461-479,
 * :556-580: q scaled by 1/sqrt(hd), softmax(q k^T) with dropout on the probabilities,
 * times v; with need_weights=True the reference also materialises and head-averages
 * the (B*H, Lq, Lk) probabilities -- a result it then discards) and in CLIP's
 * ResidualAttentionBlock (CLIP/clip/model.py:295-316).  The in/out projections stay
 * separate GEMMs (coda_gemm.h).
 *
 * q (lq, b, h*hd), k / v (lk, b, h*hd): fp32, sequence-first, contiguous (the layout the
 * reference's modules use);  out (lq, b, h*hd) fp32;  lse (b*h, lq) fp32 log-sum-exp of
 * the scaled scores (for the backward pass), may be NULL.
 * hd in {64, 128}.  nsplit in {1, 2, 3}: bf16 planes per fp32 operand (see coda_gemm.h).
 * dropout_p in [0, 1): a counter-based mask, so the backward regenerates it without storing it.  One strong
 * hash per (row i, 64-key tile t) seeds a 32-bit LCG that is stepped along the keys of the tile:
 *   s   = mix32(seed + bh*0x9E3779B1 + i*0x85EBCA77 + t*0xC2B2AE3D)      t = j / 64
 *   x_c = A^(c+1) s + C (A^c + ... + 1)  (mod 2^32),  c = j % 64,  A = 747796405, C = 2891336453
 *   element (bh, i, j) is kept iff x_c >= floor(p * 2^32);  kept probabilities are scaled by 1/(1-p)
 * with mix32(h): h ^= h>>15; h *= 0x2C1B3C6D; h ^= h>>12; h *= 0x297A2D39; h ^= h>>15 (32-bit wrap-around);
 * the effective seed is `seed` + *seed_dev when seed_dev, a device counter, is given.
 * (coda_neurips2023_b200/attention_launch.py:dropout_keep restates the formula for the tests.)
 * workspace: coda_attention_workspace_bytes(...) bytes of device scratch (packed operand planes).
 */
#ifndef CODA_ATTENTION_H
#define CODA_ATTENTION_H

#ifdef __cplusplus
extern "C" {
#endif

long long coda_attention_workspace_bytes(int b, int h, int lq, int lk, int hd, int nsplit);

int coda_attention_fwd(int b, int h, int lq, int lk, int hd, int nsplit, float scale,
                       const float *q, const float *k, const float *v, float *out, float *lse,
                       float dropout_p, unsigned int seed, const unsigned int *seed_dev,
                       void *workspace, void *stream);

/* The two halves of coda_attention_fwd, separately: operand packing (fp32 -> scaled, split bf16
 * planes in `workspace`) and the fused kernel on already-packed operands (what the roofline
 * measurement times). */
int coda_attention_pack(int b, int h, int lq, int lk, int hd, int nsplit, float scale, const float *q,
                        const float *k, const float *v, void *workspace, void *stream);
/* Packing from fp32 or IEEE-half sources with a row stride: q / k / v may be slices of one fused (l, b, 3*h*hd)
 * projection (ld = 3*h*hd) and, for the fp16 CLIP tower, are read as half without an fp32 copy.
 * ld_* in elements, multiples of 4; is_half selects the element type of all three. */
int coda_attention_pack_strided(int b, int h, int lq, int lk, int hd, int nsplit, float scale, const void *q,
                                const void *k, const void *v, long long ld_q, long long ld_k, long long ld_v,
                                int is_half, void *workspace, void *stream);
int coda_attention_fwd_packed(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                              float *out, float *lse, float dropout_p, unsigned int seed,
                              const unsigned int *seed_dev, void *stream);

/* As coda_attention_fwd_packed; out_half != 0 writes `out` as IEEE half (lk <= 64, hd == 64, nsplit <= 2 only:
 * the CLIP image tower, whose activations are fp16). */
int coda_attention_fwd_packed_ex(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                                 void *out, int out_half, float *lse, float dropout_p, unsigned int seed,
                                 const unsigned int *seed_dev, void *stream);

/*
 * fp16 self-attention with at most 64 tokens and head dim 64 (the CLIP ViT image tower, CLIP/clip/model.py:295-316 --
 * nn.MultiheadAttention on fp16 activations): q, k, v (l, b, h*64) IEEE half with row strides ld_* (slices of the fused
 * in-projection), out (l, b, h*64) half.  Operands stay half: one plane, one wgmma per product.
 * workspace: 3 * b*h*l*64 halves + 256 bytes.
 */
int coda_attention_fwd_half(int b, int h, int l, int hd, const void *q, const void *k, const void *v, long long ld_q,
                            long long ld_k, long long ld_v, void *out, void *workspace, void *stream);

/*
 * Attention masks (reference: MaskedTransformerEncoder, models/transformer.py:146-211 -- the radius masks of
 * `--enc_type masked`; nn.MultiheadAttention's boolean attn_mask in general).  Masks are bit-packed:
 * bits[b][row][tile] is one 64-bit word per 64 columns, bit c set = column 64*tile + c is NOT visible from the row.
 * bits_q is indexed by query row (forward, dQ kernel), bits_k by key row (dK/dV kernel: the transposed packing).
 *   coda_attention_mask_pack: from a byte mask (nonzero = masked) addressed mask[b*stride_b + q*stride_q + k*stride_k]
 *     (stride_b = 0 broadcasts one mask over the batch); bits_q has b*lq*ceil(lk/64) words, bits_k b*lk*ceil(lq/64).
 *   coda_attention_mask_radius: masked iff |xyz_i - xyz_j| >= radius (torch.cdist(xyz, xyz) >= radius) for one set of
 *     points xyz (b, l, 3) fp32; the mask is symmetric, `bits` (b*l*ceil(l/64) words) serves as bits_q and bits_k.
 *   coda_attention_fwd_packed_masked: coda_attention_fwd_packed_ex with mask_q (NULL = no mask).  A query row with
 *     no visible key yields NaN, as softmax over an all -inf row does in the reference.
 */
int coda_attention_mask_pack(int b, int lq, int lk, const unsigned char *mask, long long stride_b, long long stride_q,
                             long long stride_k, unsigned long long *bits_q, unsigned long long *bits_k, void *stream);
int coda_attention_mask_radius(int b, int l, const float *xyz, float radius, unsigned long long *bits, void *stream);
int coda_attention_fwd_packed_masked(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                                     void *out, int out_half, float *lse, const unsigned long long *mask_q,
                                     float dropout_p, unsigned int seed, const unsigned int *seed_dev, void *stream);

/*
 * Backward of coda_attention_fwd (hd 64 or 128): two fused wgmma kernels (dQ row-wise; dK, dV
 * column-wise) that recompute the probabilities from `lse`, regenerate the dropout mask from the same
 * counter stream, and never write an (Lq x Lk) tensor.
 *   q, k, v, out, dout as in the forward ((l, b, h*hd) fp32); lse (b*h, lq) from the forward;
 *   dq (lq, b, h*hd), dk / dv (lk, b, h*hd) fully written.  Operands are split into 2 bf16 planes.
 *   workspace: coda_attention_bwd_workspace_bytes(b, h, lq, lk, hd) bytes.
 */
long long coda_attention_bwd_workspace_bytes(int b, int h, int lq, int lk, int hd);
int coda_attention_bwd(int b, int h, int lq, int lk, int hd, float scale, const float *q, const float *k,
                       const float *v, const float *out, const float *dout, const float *lse, float *dq,
                       float *dk, float *dv, float dropout_p, unsigned int seed,
                       const unsigned int *seed_dev, void *workspace, void *stream);

/* As coda_attention_bwd with row strides and masks: q / k / v may be slices of one fused projection (ld_* = elements
 * between consecutive (l, b) rows, multiples of 4), dq / dk / dv may be slices of one packed gradient buffer (the
 * gradient of a fused q/k/v projection is then written in place, no concatenation), mask_q / mask_k as above (both
 * NULL or both given). */
int coda_attention_bwd_ex(int b, int h, int lq, int lk, int hd, float scale, const float *q, const float *k,
                          const float *v, long long ld_q, long long ld_k, long long ld_v, const float *out,
                          const float *dout, const float *lse, float *dq, float *dk, float *dv, long long ld_dq,
                          long long ld_dk, long long ld_dv, const unsigned long long *mask_q,
                          const unsigned long long *mask_k, float dropout_p, unsigned int seed,
                          const unsigned int *seed_dev, void *workspace, void *stream);

/* mult[bh][q][k] = keep(bh, q, k) ? 1/(1-p) : 0 -- the dropout factor the forward kernel applied,
 * regenerated from the counter hash (for a backward pass that materialises the probabilities). */
int coda_attention_dropout_mult(int bh, int lq, int lk, float dropout_p, unsigned int seed,
                                const unsigned int *seed_dev, float *mult, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_ATTENTION_H */
