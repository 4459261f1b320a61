/*
 * coda_data.h -- C-ABI of the device-side data layer (SURVEY.md section 8 row f4): the per-scene numpy pipeline of
 * the reference's SUN RGB-D dataset __getitem__ (datasets/sunrgbd_anonymous_aligned_image.py:618-795,
 * utils/random_cuboid.py, utils/pc_util.py:24-32) and of its ScanNet item (datasets/scannet_anonymous_aligned_image.py
 * :373-702, which crops and samples the raw scene first and transforms the sampled rows last, see
 * coda_sample_points_ex and coda_points_flip2_rotate_scale) for a batch of raw scenes resident in HBM.  Conventions as in
 * coda_pointnet2.h.  Scenes are padded: points (b, nmax, stride) fp32 with npts (b) valid rows (columns 0-2 = xyz,
 * the others -- colour, height -- travel along); boxes (b, gmax, box_stride) fp32 rows [cx, cy, cz, ...] with
 * nbox (b) valid rows.  All randomness comes in as small device arrays drawn by the caller.
 *
 * The `_f64` entry points are the same kernels on float64 points and boxes (dims, stats and samples in float64 too),
 * for SUN RGB-D, whose `_pc.npz` / `_bbox.npy` arrays are float64: there the reference's flip, rotation, scale,
 * RandomCuboid and sampling all run in float64 (datasets/sunrgbd_anonymous_aligned_image.py:660-771).  The float32
 * entry points are unchanged by them.
 */
#ifndef CODA_DATA_H
#define CODA_DATA_H

#include "coda_pointnet2.h" /* status codes */

#ifdef __cplusplus
extern "C" {
#endif

/*
 * In place: xyz <- ((flip * x, y, z) @ rot^T) * scale with flip (b) = +-1, rot (b, 3, 3), scale (b)
 *   replaces :663-700 (flip about the YZ plane, pc_util.rotz rotation, 0.85-1.15 scaling) on the points; float32
 *   products / sums rounded separately in numpy's order.
 */
int coda_scene_transform(int b, int nmax, int stride, const int *npts, const float *flip, const float *rot,
                         const float *scale, float *points, void *stream);

/* dims (b, 6) = [min xyz | max xyz] of the valid points (npts may be NULL: all nmax rows). */
int coda_points_extent(int b, int nmax, int stride, const int *npts, const float *points, float *dims, void *stream);

/* float64 twin: replaces RandomCuboid's range_xyz (random_cuboid.py:39-41) on the float64 SUN RGB-D cloud. */
int coda_points_extent_f64(int b, int nmax, int stride, const int *npts, const double *points, double *dims,
                           void *stream);

/*
 * RandomCuboid (utils/random_cuboid.py:39-116) with all `ncand` attempts of a scene evaluated at once.
 *   range_xyz (b, 3) = extent of the cloud; crop_range (b, ncand, 3) fp64 in [min_crop, max_crop] (the reference's
 *   random numbers are doubles and so are the bounds they produce); center_u (b, ncand) in [0, 1) selects the centre
 *   point floor(u * npts).  Attempt c crops to centre +- range_xyz * crop_range / 2 (inclusive, evaluated in fp64).  chosen (b) = first attempt with (i) an aspect ratio >= aspect_min in some plane, (ii) >= min_points
 *   points inside, (iii) -- if the scene has ground truth -- at least one box centre within the extent of the points
 *   inside; -1 = none (the scene is kept whole).  crop (b, 6) = the chosen bounds (+-inf when -1);
 *   box_keep (b, gmax) = boxes that stay (centre inside that extent).  stats_scratch: b * ncand * 8 floats.
 */
int coda_random_cuboid(int b, int nmax, int stride, int ncand, int gmax, int box_stride, int min_points,
                       float aspect_min, const int *npts, const float *points, const float *range_xyz,
                       const double *crop_range, const float *center_u, const float *boxes, const int *nbox,
                       float *stats_scratch, int *chosen, double *crop, unsigned char *box_keep, void *stream);

/*
 * float64 twin (points, range_xyz, boxes, stats_scratch in float64): replaces the SUN RGB-D item's RandomCuboid call
 *   (datasets/sunrgbd_anonymous_aligned_image.py:714-717) on its float64 cloud and boxes; `target_boxes.sum() > 0` is
 *   summed in float64.
 */
int coda_random_cuboid_f64(int b, int nmax, int stride, int ncand, int gmax, int box_stride, int min_points,
                           float aspect_min, const int *npts, const double *points, const double *range_xyz,
                           const double *crop_range, const float *center_u, const double *boxes, const int *nbox,
                           double *stats_scratch, int *chosen, double *crop, unsigned char *box_keep, void *stream);

/*
 * pc_util.random_sampling (:24-32) of the points inside crop (b, 6): out (b, nsample, stride), choice (b, nsample)
 *   = row of the raw scene each sample came from, count (b) = points inside, dims (b, 6) = extent of the sample
 *   (point_cloud_dims_min / max, :748-749).  Without replacement when count >= nsample (a keyed Feistel permutation
 *   with cycle walking instead of a sort), hashed draws with replacement otherwise.  list_scratch: b * nmax ints.
 */
int coda_sample_points(int b, int nmax, int stride, int nsample, const int *npts, const float *points,
                       const double *crop, const unsigned int *seed, int *list_scratch, int *count, float *out,
                       int *choice, float *dims, void *stream);

/*
 * float64 twin (points, out, dims in float64), same sampler and same positions: replaces the SUN RGB-D item's
 *   random_sampling and point_cloud_dims_min / max (:763-771), which stay float64 there.
 */
int coda_sample_points_f64(int b, int nmax, int stride, int nsample, const int *npts, const double *points,
                           const double *crop, const unsigned int *seed, int *list_scratch, int *count, double *out,
                           int *choice, double *dims, void *stream);

/*
 * coda_sample_points plus the ScanNet item's gathers (datasets/scannet_anonymous_aligned_image.py:507-532), in the same
 *   pass and with the same draws, so out / choice / count / dims are those coda_sample_points gives:
 *   list_pos (b, nsample) = position of each sample in the cropped cloud (the reference's `choices`; choice is the
 *   raw-scene row, out[i] = points[choice[i]]); rgb_out (b, nsample, rgb_stride) = the first rgb_stride <= stride
 *   columns of the RAW scene's row list_pos[i] -- the reference's point_clouds_rgb / pcl_color index the uncropped
 *   scene with the cropped cloud's choices, and this reproduces it.  rgb_out may be NULL when rgb_stride is 0.
 */
int coda_sample_points_ex(int b, int nmax, int stride, int nsample, int rgb_stride, const int *npts,
                          const float *points, const double *crop, const unsigned int *seed, int *list_scratch,
                          int *count, float *out, int *choice, int *list_pos, float *rgb_out, float *dims,
                          void *stream);

/*
 * In place on (b, nmax, stride) fp32 rows, npts (b) valid (NULL: all nmax): the ScanNet item's augmentation of the
 *   sampled points (:545-604): x <- flip_yz * x, y <- flip_xz * y (flip_* (b) = +-1, exact), then xyz <- xyz @ rot^T
 *   with rot (b, 3, 3) fp64, then xyz <- xyz * scale with scale (b) fp64; columns 3 and up are untouched.  Rounding
 *   as numpy does it on a float32 cloud: the product with the float64 matrix is formed in fp64 as
 *   fma(z, r2, fma(y, r1, x * r0)) (BLAS dgemm's order) and stored as float32; the scale product is formed in fp64
 *   and stored as float32.  The extents come after this, from coda_points_extent.
 */
int coda_points_flip2_rotate_scale(int b, int nmax, int stride, const int *npts, const float *flip_yz,
                                   const float *flip_xz, const double *rot, const double *scale, float *points,
                                   void *stream);

/*
 * float64 twin on (b, nmax, stride) fp64 rows: the same fused chain with no rounding to float32 anywhere.  Replaces the
 *   SUN RGB-D item's flip about YZ, np.dot with rotz and float64 scale (:664-709, flip_xz = +1) on the whole raw
 *   scene and on the boxes' centres, and the np.dot(rotz(-heading), corners) of my_compute_box_3d (:288-298; one
 *   "scene" per box, 8 rows, scale 1).
 */
int coda_points_flip2_rotate_scale_f64(int b, int nmax, int stride, const int *npts, const float *flip_yz,
                                       const float *flip_xz, const double *rot, const double *scale, double *points,
                                       void *stream);

/*
 * Image augmentation of :624-655 on uint8 HWC images: horizontal flip (flip (b) != 0), per-channel gain (b, 3) and
 * shift (b, 3), per-pixel jitter in [-0.025, 0.025) from a counter hash of seed (b), clip to [0, 1], truncation to
 * uint8.  `out` must not alias `in`.
 */
int coda_image_augment(int b, int h, int w, const unsigned char *in, const unsigned char *flip, const float *gain,
                       const float *shift, const unsigned int *seed, unsigned char *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_DATA_H */
