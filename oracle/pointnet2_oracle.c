/*
 * pointnet2_oracle.c -- CPU restatement of the reference's PointNet++ CUDA ops.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (the package
 * coda_neurips2023_b200/) may import, link or call this file; only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * do, and there only as the checker or as the stated CPU baseline.
 *
 * Parity pinning: the reference ships NO golden vectors for these ops
 * (SURVEY.md section 4); this restatement is pinned instead against the
 * reference's own CUDA extension compiled unmodified from /root/reference
 * (oracle/build_ref_ext.py -> oracle/_ref/) and run on the GPU
 * (tests/test_pointnet2_gpu.py::test_*_vs_reference_ext), and the outputs of
 * that run are committed as fixtures under tests/golden/.
 *
 * Each function simulates the reference kernel thread by thread, so that the
 * tie rules, the skip rule and the fp32 rounding (explicit fmaf in the order
 * nvcc's default --fmad=true contraction produces -- read off the SASS of the
 * reference objects, oracle/_ref/obj/ (one .o per source): for a*a + b*b + c*c it is
 * FMUL(b,b), FFMA(a,a,.), FFMA(c,c,.)) are those of the reference, not of a
 * "clean" algorithm.
 * Compile with -ffp-contract=off so the host compiler adds no contraction of
 * its own.
 *
 * All paths cited are relative to
 *   /root/reference/third_party_pointnet2/pointnet2/_ext_src/
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* include/cuda_utils.h:17-21  opt_n_threads */
int oracle_opt_n_threads(int work_size) {
  const int pow_2 = (int)(log((double)work_size) / log(2.0));
  int t = 1 << pow_2;
  if (t > 512) t = 512;
  if (t < 1) t = 1;
  return t;
}

static float sqdist_pt_minus_ref(float x2, float y2, float z2, float x1,
                                 float y1, float z1) {
  /* src/sampling_gpu.cu:106-107: (x2-x1)*(x2-x1)+(y2-y1)*(y2-y1)+(z2-z1)*(z2-z1).
   * nvcc (--fmad=true) contracts a*a + b*b + c*c as FMUL(b,b); FFMA(a,a,.);
   * FFMA(c,c,.) -- read off the SASS of the reference build
   * (cuobjdump -sass oracle/_ref/obj/sampling_gpu.cu.o): the SECOND product is
   * the plain multiply. */
  const float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
  return fmaf(dz, dz, fmaf(dx, dx, dy * dy));
}

/*
 * src/sampling_gpu.cu:72-176 furthest_point_sampling_kernel<block_size>,
 * launched by :178-232 with block_size = opt_n_threads(n), one block per batch
 * element; temp initialised to 1e10 by src/sampling.cpp:75-77.
 * dataset (b,n,3) -> idxs (b,m) (zero-initialised by the host code).
 */
void oracle_furthest_point_sampling(int b, int n, int m, const float *dataset,
                                    int *idxs) {
  memset(idxs, 0, sizeof(int) * (size_t)b * (size_t)(m > 0 ? m : 0));
  if (m <= 0 || n <= 0) return; /* :76 */
  const int bs = oracle_opt_n_threads(n);
  float *temp = (float *)malloc(sizeof(float) * (size_t)n);
  float *dists = (float *)malloc(sizeof(float) * (size_t)bs);
  int *dists_i = (int *)malloc(sizeof(int) * (size_t)bs);
  for (int bi = 0; bi < b; ++bi) {
    const float *ds = dataset + (size_t)bi * n * 3;
    int *out = idxs + (size_t)bi * m;
    for (int k = 0; k < n; ++k) temp[k] = 1e10f;
    int old = 0;
    out[0] = old; /* :89 */
    for (int j = 1; j < m; ++j) {
      const float x1 = ds[old * 3 + 0], y1 = ds[old * 3 + 1],
                  z1 = ds[old * 3 + 2];
      for (int tid = 0; tid < bs; ++tid) { /* :93-115 per-thread strided scan */
        int besti = 0;
        float best = -1.0f;
        for (int k = tid; k < n; k += bs) {
          const float x2 = ds[k * 3 + 0], y2 = ds[k * 3 + 1],
                      z2 = ds[k * 3 + 2];
          const float mag = fmaf(z2, z2, fmaf(x2, x2, y2 * y2)); /* :103, same contraction */
          if ((double)mag <= 1e-3) continue;                   /* :104 */
          const float d = sqdist_pt_minus_ref(x2, y2, z2, x1, y1, z1);
          const float d2 = fminf(d, temp[k]); /* :109 */
          temp[k] = d2;
          besti = d2 > best ? k : besti; /* :111 */
          best = d2 > best ? d2 : best;  /* :112 */
        }
        dists[tid] = best;
        dists_i[tid] = besti;
      }
      /* :118-171 halving tree; __update (:62-68): keep idx1 unless v2 > v1 */
      for (int s = bs / 2; s >= 1; s >>= 1) {
        for (int tid = 0; tid < s; ++tid) {
          const float v1 = dists[tid], v2 = dists[tid + s];
          const int i1 = dists_i[tid], i2 = dists_i[tid + s];
          dists[tid] = fmaxf(v1, v2);
          dists_i[tid] = v2 > v1 ? i2 : i1;
        }
      }
      old = dists_i[0]; /* :173 */
      out[j] = old;
    }
  }
  free(temp);
  free(dists);
  free(dists_i);
}

/* src/sampling_gpu.cu:11-23 gather_points_kernel */
void oracle_gather_points(int b, int c, int n, int m, const float *points,
                          const int *idx, float *out) {
  for (int i = 0; i < b; ++i)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < m; ++j) {
        const int a = idx[i * m + j];
        out[((size_t)i * c + l) * m + j] = points[((size_t)i * c + l) * n + a];
      }
}

/* src/sampling_gpu.cu:37-49 gather_points_grad_kernel (atomicAdd; here the
 * sum is taken in ascending j, the GPU order is unspecified) */
void oracle_gather_points_grad(int b, int c, int n, int m,
                               const float *grad_out, const int *idx,
                               float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * n);
  for (int i = 0; i < b; ++i)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < m; ++j) {
        const int a = idx[i * m + j];
        grad_points[((size_t)i * c + l) * n + a] +=
            grad_out[((size_t)i * c + l) * m + j];
      }
}

/* src/ball_query_gpu.cu:12-46 query_ball_point_kernel; idx zero-initialised by
 * src/ball_query.cpp:21-23 */
void oracle_ball_query(int b, int n, int m, float radius, int nsample,
                       const float *new_xyz, const float *xyz, int *idx) {
  memset(idx, 0, sizeof(int) * (size_t)b * m * nsample);
  const float radius2 = radius * radius; /* :24 */
  for (int bi = 0; bi < b; ++bi) {
    const float *X = xyz + (size_t)bi * n * 3;
    const float *C = new_xyz + (size_t)bi * m * 3;
    int *I = idx + (size_t)bi * m * nsample;
    for (int j = 0; j < m; ++j) {
      const float nx = C[j * 3 + 0], ny = C[j * 3 + 1], nz = C[j * 3 + 2];
      for (int k = 0, cnt = 0; k < n && cnt < nsample; ++k) {
        const float x = X[k * 3 + 0], y = X[k * 3 + 1], z = X[k * 3 + 2];
        /* :34-35 (new_x-x)^2+(new_y-y)^2+(new_z-z)^2 -> FMUL(dy), FFMA(dx), FFMA(dz) */
        const float dx = nx - x, dy = ny - y, dz = nz - z;
        const float d2 = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
        if (d2 < radius2) {
          if (cnt == 0)
            for (int l = 0; l < nsample; ++l) I[j * nsample + l] = k; /* :37-41 */
          I[j * nsample + cnt] = k;
          ++cnt;
        }
      }
    }
  }
}

/* src/group_points_gpu.cu:11-30 group_points_kernel */
void oracle_group_points(int b, int c, int n, int npoints, int nsample,
                         const float *points, const int *idx, float *out) {
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < npoints; ++j)
        for (int k = 0; k < nsample; ++k) {
          const int ii = idx[((size_t)bi * npoints + j) * nsample + k];
          out[(((size_t)bi * c + l) * npoints + j) * nsample + k] =
              points[((size_t)bi * c + l) * n + ii];
        }
}

/* src/group_points_gpu.cu:46-66 group_points_grad_kernel */
void oracle_group_points_grad(int b, int c, int n, int npoints, int nsample,
                              const float *grad_out, const int *idx,
                              float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * n);
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < npoints; ++j)
        for (int k = 0; k < nsample; ++k) {
          const int ii = idx[((size_t)bi * npoints + j) * nsample + k];
          grad_points[((size_t)bi * c + l) * n + ii] +=
              grad_out[(((size_t)bi * c + l) * npoints + j) * nsample + k];
        }
}

/* src/interpolate_gpu.cu:12-62 three_nn_kernel (double-typed running bests,
 * fp32 distance, strict <) */
void oracle_three_nn(int b, int n, int m, const float *unknown,
                     const float *known, float *dist2, int *idx) {
  for (int bi = 0; bi < b; ++bi) {
    const float *U = unknown + (size_t)bi * n * 3;
    const float *K = known + (size_t)bi * m * 3;
    float *D = dist2 + (size_t)bi * n * 3;
    int *I = idx + (size_t)bi * n * 3;
    for (int j = 0; j < n; ++j) {
      const float ux = U[j * 3 + 0], uy = U[j * 3 + 1], uz = U[j * 3 + 2];
      double best1 = 1e40, best2 = 1e40, best3 = 1e40;
      int besti1 = 0, besti2 = 0, besti3 = 0;
      for (int k = 0; k < m; ++k) {
        const float x = K[k * 3 + 0], y = K[k * 3 + 1], z = K[k * 3 + 2];
        const float dx = ux - x, dy = uy - y, dz = uz - z;
        const float d = fmaf(dz, dz, fmaf(dx, dx, dy * dy)); /* :36 */
        if (d < best1) {
          best3 = best2; besti3 = besti2;
          best2 = best1; besti2 = besti1;
          best1 = d; besti1 = k;
        } else if (d < best2) {
          best3 = best2; besti3 = besti2;
          best2 = d; besti2 = k;
        } else if (d < best3) {
          best3 = d; besti3 = k;
        }
      }
      D[j * 3 + 0] = (float)best1; D[j * 3 + 1] = (float)best2;
      D[j * 3 + 2] = (float)best3;
      I[j * 3 + 0] = besti1; I[j * 3 + 1] = besti2; I[j * 3 + 2] = besti3;
    }
  }
}

/* src/interpolate_gpu.cu:75-104 three_interpolate_kernel:
 * p1*w1 + p2*w2 + p3*w3 -> FMUL(p2,w2); FFMA(p1,w1,.); FFMA(p3,w3,.) (SASS) */
void oracle_three_interpolate(int b, int c, int m, int n, const float *points,
                              const int *idx, const float *weight, float *out) {
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < n; ++j) {
        const float *w = weight + ((size_t)bi * n + j) * 3;
        const int *ii = idx + ((size_t)bi * n + j) * 3;
        const float *p = points + ((size_t)bi * c + l) * m;
        out[((size_t)bi * c + l) * n + j] =
            fmaf(p[ii[2]], w[2], fmaf(p[ii[0]], w[0], p[ii[1]] * w[1]));
      }
}

/* src/interpolate_gpu.cu:119-146 three_interpolate_grad_kernel */
void oracle_three_interpolate_grad(int b, int c, int n, int m,
                                   const float *grad_out, const int *idx,
                                   const float *weight, float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * m);
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < n; ++j) {
        const float *w = weight + ((size_t)bi * n + j) * 3;
        const int *ii = idx + ((size_t)bi * n + j) * 3;
        float *g = grad_points + ((size_t)bi * c + l) * m;
        const float go = grad_out[((size_t)bi * c + l) * n + j];
        g[ii[0]] += go * w[0];
        g[ii[1]] += go * w[1];
        g[ii[2]] += go * w[2];
      }
}

/*
 * Op sequence of QueryAndGroup.forward for the xyz-only layer
 * (../pointnet2_utils.py:331-349): ball_query, group xyz^T, subtract the
 * centre, optionally "/= radius".  On a CUDA tensor torch evaluates a division
 * by a Python scalar as a multiplication by the fp32 reciprocal
 * (ATen/native/cuda/BinaryDivTrueKernel.cu, is_cpu_scalar branch), and the
 * reference only ever runs this on the GPU, so that is what is restated here.
 */
void oracle_query_and_group_xyz(int b, int n, int m, float radius, int nsample,
                                int normalize, const float *xyz,
                                const float *new_xyz, int *idx,
                                float *grouped) {
  oracle_ball_query(b, n, m, radius, nsample, new_xyz, xyz, idx);
  for (int bi = 0; bi < b; ++bi)
    for (int c = 0; c < 3; ++c)
      for (int j = 0; j < m; ++j)
        for (int s = 0; s < nsample; ++s) {
          const int k = idx[((size_t)bi * m + j) * nsample + s];
          float v = xyz[((size_t)bi * n + k) * 3 + c] -
                    new_xyz[((size_t)bi * m + j) * 3 + c];
          if (normalize) v = v * (1.0f / radius);
          grouped[(((size_t)bi * 3 + c) * m + j) * nsample + s] = v;
        }
}
