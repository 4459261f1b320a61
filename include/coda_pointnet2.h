/*
 * coda_pointnet2.h -- C-ABI of the H100-native PointNet++ set-abstraction ops.
 *
 * Drop-in boundary for the reference's pybind module `pointnet2._ext`
 * (third_party_pointnet2/pointnet2/_ext_src/src/bindings.cpp:9-22).  Every
 * entry point below replaces one `*_kernel_wrapper` the reference's C++ host
 * functions call; the cited file:line is the reference declaration it stands
 * in for.  The ABI is plain C: raw DEVICE pointers, sizes, a CUDA stream passed
 * as an opaque `void*` (a `cudaStream_t`), `int` status return
 * (0 == cudaSuccess, otherwise the `cudaError_t` value, or a negative
 * CODA_E* code for argument errors).  Nothing here allocates, synchronises
 * the device, or touches torch types.  All tensors are dense row-major
 * ("contiguous" in the reference's CHECK_CONTIGUOUS sense), fp32 / int32.
 *
 * Unlike the reference launchers (which print and exit(-1) on a launch error,
 * include/cuda_utils.h:32-41) these return the error to the caller.
 */
#ifndef CODA_POINTNET2_H
#define CODA_POINTNET2_H

#ifdef __cplusplus
extern "C" {
#endif

#define CODA_OK 0
#define CODA_EINVAL (-1)      /* bad shape / null pointer                     */
#define CODA_ETOOLARGE (-2)   /* problem exceeds what the resident path holds */

/* Library/ABI version; bumped whenever a signature changes. */
int coda_abi_version(void);

/* Human-readable text for a status returned by any coda_* call. */
const char *coda_status_string(int status);

/*
 * Furthest point sampling.
 *   replaces furthest_point_sampling_kernel_wrapper  (_ext_src/include/sampling.h:9,
 *            _ext_src/src/sampling_gpu.cu:178-232; host caller sampling.cpp:67-88)
 *   xyz  (b, n, 3) fp32      idx (b, m) int32 (every element is written)
 * Bit-exact with the reference kernel including its tie rule (halving tree =>
 * lexicographic min of (bitrev(k mod bs), k) among equal maxima), the
 * |p|^2 <= 1e-3 skip, and FMA contraction order.  The reference's (b, n) `temp`
 * scratch is held in registers here, so no scratch pointer is part of the ABI.
 */
int coda_furthest_point_sampling(int b, int n, int m, const float *xyz,
                                 int *idx, void *stream);

/*
 * gather_points / gather_points_grad
 *   replaces gather_points_kernel_wrapper / gather_points_grad_kernel_wrapper
 *            (_ext_src/include/sampling.h:7-8, src/sampling_gpu.cu:25-60)
 *   points (b, c, n) fp32, idx (b, m) int32 -> out (b, c, m)
 *   grad:  grad_out (b, c, m), idx (b, m) -> grad_points (b, c, n), which the
 *          CALLER must have zeroed (the reference host code allocates zeros).
 */
int coda_gather_points(int b, int c, int n, int m, const float *points,
                       const int *idx, float *out, void *stream);
int coda_gather_points_grad(int b, int c, int n, int m, const float *grad_out,
                            const int *idx, float *grad_points, void *stream);

/*
 * ball_query
 *   replaces query_ball_point_kernel_wrapper (_ext_src/include/ball_query.h:6-7,
 *            src/ball_query_gpu.cu:48-57)
 *   new_xyz (b, m, 3), xyz (b, n, 3) -> idx (b, m, nsample) int32.
 *   First `nsample` indices k (ascending) with d2 < radius*radius; the first
 *   hit pads the tail; no hit -> zeros.  Every element of idx is written.
 */
int coda_ball_query(int b, int n, int m, float radius, int nsample,
                    const float *new_xyz, const float *xyz, int *idx,
                    void *stream);

/*
 * group_points / group_points_grad
 *   replaces group_points_kernel_wrapper / group_points_grad_kernel_wrapper
 *            (_ext_src/include/group_points.h:7-8, src/group_points_gpu.cu:32-78)
 *   points (b, c, n), idx (b, npoints, nsample) -> out (b, c, npoints, nsample)
 *   grad: grad_points (b, c, n) must be zeroed by the caller.
 */
int coda_group_points(int b, int c, int n, int npoints, int nsample,
                      const float *points, const int *idx, float *out,
                      void *stream);
int coda_group_points_grad(int b, int c, int n, int npoints, int nsample,
                           const float *grad_out, const int *idx,
                           float *grad_points, void *stream);

/*
 * three_nn
 *   replaces three_nn_kernel_wrapper (_ext_src/include/interpolate.h:8,
 *            src/interpolate_gpu.cu:64-70)
 *   unknown (b, n, 3), known (b, m, 3) -> dist2 (b, n, 3) SQUARED distances,
 *   idx (b, n, 3) int32.  Unfilled slots (m < 3): idx 0, dist2 +inf.
 */
int coda_three_nn(int b, int n, int m, const float *unknown, const float *known,
                  float *dist2, int *idx, void *stream);

/*
 * three_interpolate / three_interpolate_grad
 *   replaces three_interpolate_kernel_wrapper / ..._grad_kernel_wrapper
 *            (_ext_src/include/interpolate.h:9-12, src/interpolate_gpu.cu:106-157)
 *   points (b, c, m), idx (b, n, 3), weight (b, n, 3) -> out (b, c, n)
 *   grad: grad_out (b, c, n) -> grad_points (b, c, m), zeroed by the caller.
 */
int coda_three_interpolate(int b, int c, int m, int n, const float *points,
                           const int *idx, const float *weight, float *out,
                           void *stream);
int coda_three_interpolate_grad(int b, int c, int n, int m,
                                const float *grad_out, const int *idx,
                                const float *weight, float *grad_points,
                                void *stream);

/*
 * Fused QueryAndGroup for the xyz-only set-abstraction layer
 *   replaces the op SEQUENCE in QueryAndGroup.forward
 *   (pointnet2_utils.py:331-349): ball_query -> grouping_operation(xyz^T) ->
 *   "-= new_xyz" -> "/= radius" (normalize_xyz).
 *   xyz (b, n, 3), new_xyz (b, m, 3) ->
 *     idx (b, m, nsample) int32 (same contract as coda_ball_query)
 *     grouped (b, 3, m, nsample) fp32 = (xyz[idx] - new_xyz) [/ radius if normalize]
 *   The subtraction and IEEE division are done exactly as the torch ops do, so
 *   the result is bit-identical to the unfused sequence.
 */
int coda_query_and_group_xyz(int b, int n, int m, float radius, int nsample,
                             int normalize, const float *xyz,
                             const float *new_xyz, int *idx, float *grouped,
                             void *stream);

/*
 * Test/benchmark knob (not part of the reference surface): force the FPS
 * cluster width (1, 2, 4, 8; 0 = automatic).  Returns the previous value.
 */
int coda_fps_set_cluster(int cluster_ctas);

#ifdef __cplusplus
}
#endif
#endif /* CODA_POINTNET2_H */
