// Batched crop + white-pad + antialiased bicubic resize + normalise for the CLIP
// crops (include/coda_image.h).  One thread per output pixel (all 3 channels);
// the source canvas is virtual: pixels outside the pasted crop read as 255.
#include <cuda_fp16.h>
#include <math.h>

#include "../../include/coda_image.h"
#include "coda_common.cuh"

using namespace coda;

namespace {

constexpr int MAX_TAPS = 40;

// ATen upsample_antialias: cubic convolution filter with a = -0.5
__device__ __forceinline__ float cubic_aa(float x) {
  const float a = -0.5f;
  x = fabsf(x);
  if (x < 1.0f) return ((a + 2.0f) * x - (a + 3.0f)) * x * x + 1.0f;
  if (x < 2.0f) return (((x - 5.0f) * x + 8.0f) * x - 4.0f) * a;
  return 0.0f;
}

// ---------------------------------------------------------------------------------------------------------------
// Separable form.  The antialiased resize is a tensor product: out[oy][ox] = sum_iy wy[oy][iy] * (sum_ix wx[ox][ix] *
// canvas[ylo + iy][xlo + ix]).  A CTA owns `tr` output rows of one crop:
//   0. the x weights of all `res` columns and the y weights of its rows go to shared memory once (not once per pixel);
//   1. horizontal pass: every source row the tile touches is resampled to `res` columns into shared memory
//      (fp32, 3 channels) -- one 32-bit load per tap from the RGBX copy of the images instead of three byte loads;
//   2. vertical pass over the shared rows, rounding / normalisation, store (NCHW or patch-major).
// The sums run in the order of the direct form (x taps ascending, then y taps ascending), so the result is the same
// to the bit.  Load count per crop at scale 3.3: 29.5 M byte loads (direct) -> 3.9 M word loads + 2.1 M shared loads.
constexpr int CR_THREADS = 1024;
constexpr size_t CR_SMEM_LIMIT = 220 * 1024;

__global__ void __launch_bounds__(256)
rgb_to_rgbx_kernel(long long npix, const unsigned char *__restrict__ rgb, uchar4 *__restrict__ rgbx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const unsigned char *p = rgb + i * 3;
  rgbx[i] = make_uchar4(p[0], p[1], p[2], 255);
}

// byte k of `word` as a float without a conversion instruction (I2F issues at a fraction of the FMA rate and was what
// bound the tap loop): the byte becomes the low mantissa bits of 2^23, and 2^23 + b - 2^23 is exact.
__device__ __forceinline__ float byte_f32(unsigned word, unsigned selector) {
  return __uint_as_float(__byte_perm(word, 0x4B000000u, selector)) - 8388608.0f;
}

// _compute_indices_span + _compute_weights of ATen/native/cuda/UpSample.cuh; the (normalised) weights are written
// to `w` (shared memory), at most `cap` taps
__device__ __forceinline__ void aa_weights_to(float scale, int out_idx, int in_size, int cap, int &lo, int &n,
                                              float *w) {
  const float support = scale >= 1.0f ? 2.0f * scale : 2.0f;
  const float invscale = scale >= 1.0f ? 1.0f / scale : 1.0f;
  const float center = scale * (out_idx + 0.5f);
  lo = max((int)(center - support + 0.5f), 0);
  n = min((int)(center + support + 0.5f), in_size) - lo;
  n = min(n, cap);
  float total = 0.f;
  for (int j = 0; j < n; ++j) {
    const float v = cubic_aa((j + lo - center + 0.5f) * invscale);
    w[j] = v;
    total += v;
  }
  if (total != 0.f)
    for (int j = 0; j < n; ++j) w[j] /= total;
}

template <typename OutT>
__global__ void __launch_bounds__(CR_THREADS)
crop_resize_sep_kernel(int h, int w, int res, int tr, int rmax, int xt, int yt, int patch,
                       const uchar4 *__restrict__ rgbx, const int *__restrict__ scene,
                       const int *__restrict__ boxes, const unsigned char *__restrict__ valid, float m0, float m1,
                       float m2, float s0, float s1, float s2, OutT *__restrict__ out) {
  extern __shared__ __align__(16) unsigned char cr_smem[];
  float *rowbuf = reinterpret_cast<float *>(cr_smem);      // [rmax][res][3]
  float *wx_s = rowbuf + (size_t)rmax * res * 3;             // [res][xt]
  float *wy_s = wx_s + (size_t)res * xt;                     // [tr][yt]
  int *xlo_s = reinterpret_cast<int *>(wy_s + (size_t)tr * yt);
  int *xn_s = xlo_s + res;
  int *ylo_s = xn_s + res;
  int *yn_s = ylo_s + tr;
  const int crop = blockIdx.y;
  const int oy0 = blockIdx.x * tr;
  const int nrow = min(tr, res - oy0);
  const int tid = threadIdx.x;
  const size_t plane = (size_t)res * res;
  const int g = patch > 0 ? res / patch : 0;
  auto store = [&](int oy, int ox, float v0, float v1, float v2) {
    if (patch > 0) {
      OutT *o = out + ((((size_t)crop * g + oy / patch) * g + ox / patch) * 3) * patch * patch +
                (size_t)(oy % patch) * patch + ox % patch;
      o[0] = OutT(v0); o[(size_t)patch * patch] = OutT(v1); o[(size_t)2 * patch * patch] = OutT(v2);
    } else {
      OutT *o = out + (size_t)crop * 3 * plane + (size_t)oy * res + ox;
      o[0] = OutT(v0); o[plane] = OutT(v1); o[2 * plane] = OutT(v2);
    }
  };
  if (!valid[crop]) {
    for (int idx = tid; idx < nrow * res; idx += CR_THREADS) store(oy0 + idx / res, idx % res, 0.f, 0.f, 0.f);
    return;
  }
  const int xmin = boxes[crop * 4 + 0], ymin = boxes[crop * 4 + 1];
  const int wc = boxes[crop * 4 + 2] - xmin, hc = boxes[crop * 4 + 3] - ymin;
  const int edge = max(wc, hc);
  const int y_begin = (edge - hc) / 2, x_begin = (edge - wc) / 2;
  const uchar4 *img = rgbx + (size_t)scene[crop] * h * w;
  const float scale = (float)edge / (float)res;
  for (int ox = tid; ox < res; ox += CR_THREADS) {
    int lo, n;
    aa_weights_to(scale, ox, edge, xt, lo, n, wx_s + (size_t)ox * xt);
    xlo_s[ox] = lo; xn_s[ox] = n;
  }
  for (int r = tid; r < nrow; r += CR_THREADS) {
    int lo, n;
    aa_weights_to(scale, oy0 + r, edge, yt, lo, n, wy_s + (size_t)r * yt);
    ylo_s[r] = lo; yn_s[r] = n;
  }
  __syncthreads();
  const int y_lo = ylo_s[0];
  const int nsrc = ylo_s[nrow - 1] + yn_s[nrow - 1] - y_lo;      // source rows of the tile (ylo is monotonic in oy)
  auto finish = [&](int oy, int ox, float a0, float a1, float a2) {
    // back to what the uint8 tensor would hold, then /255 and Normalize
    a0 = rintf(fminf(fmaxf(a0, 0.f), 255.f));
    a1 = rintf(fminf(fmaxf(a1, 0.f), 255.f));
    a2 = rintf(fminf(fmaxf(a2, 0.f), 255.f));
    store(oy, ox, (a0 / 255.0f - m0) / s0, (a1 / 255.0f - m1) / s1, (a2 / 255.0f - m2) / s2);
  };
  // one source row resampled at column ox
  auto hrow = [&](int canvas_y, int ox, float &r0, float &r1, float &r2) {
    const int cy = canvas_y - y_begin;            // row inside the crop
    const bool yin = cy >= 0 && cy < hc;
    const uchar4 *row = img + (yin ? (size_t)(ymin + cy) * w + xmin : 0);
    const float *wx = wx_s + (size_t)ox * xt;
    const int xlo = xlo_s[ox], xn = xn_s[ox];
    r0 = 0.f; r1 = 0.f; r2 = 0.f;
    const int c0 = xlo - x_begin;
    if (yin && c0 >= 0 && c0 + xn <= wc) {
      // every tap inside the pasted crop (the common case): unconditional loads, several in flight per thread
      const unsigned *src = reinterpret_cast<const unsigned *>(row + c0);
#pragma unroll 5
      for (int ix = 0; ix < xn; ++ix) {
        const unsigned p = __ldg(src + ix);
        const float wv = wx[ix];
        r0 += wv * byte_f32(p, 0x7540u); r1 += wv * byte_f32(p, 0x7541u); r2 += wv * byte_f32(p, 0x7542u);
      }
    } else if (!yin) {
      for (int ix = 0; ix < xn; ++ix) {            // a row of the white canvas
        r0 += wx[ix] * 255.f; r1 += wx[ix] * 255.f; r2 += wx[ix] * 255.f;
      }
    } else {
      for (int ix = 0; ix < xn; ++ix) {
        const int cx = c0 + ix;
        float p0 = 255.f, p1 = 255.f, p2 = 255.f;   // white canvas
        if (cx >= 0 && cx < wc) {
          const uchar4 p = __ldg(row + cx);
          p0 = (float)p.x; p1 = (float)p.y; p2 = (float)p.z;
        }
        r0 += wx[ix] * p0; r1 += wx[ix] * p1; r2 += wx[ix] * p2;
      }
    }
  };
  if (nsrc <= rmax) {
    for (int idx = tid; idx < nsrc * res; idx += CR_THREADS) {
      const int ry = idx / res, ox = idx - ry * res;
      float r0, r1, r2;
      hrow(y_lo + ry, ox, r0, r1, r2);
      float *dst = rowbuf + (size_t)idx * 3;
      dst[0] = r0; dst[1] = r1; dst[2] = r2;
    }
    __syncthreads();
    for (int idx = tid; idx < nrow * res; idx += CR_THREADS) {
      const int r = idx / res, ox = idx - r * res;
      const float *wy = wy_s + (size_t)r * yt;
      const float *src = rowbuf + ((size_t)(ylo_s[r] - y_lo) * res + ox) * 3;
      const int yn = yn_s[r];
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll 5
      for (int iy = 0; iy < yn; ++iy) {
        const float *q = src + (size_t)iy * res * 3;
        a0 += wy[iy] * q[0]; a1 += wy[iy] * q[1]; a2 += wy[iy] * q[2];
      }
      finish(oy0 + r, ox, a0, a1, a2);
    }
  } else {
    // a tile whose source rows do not fit the shared buffer (cannot happen for boxes inside the image the launcher
    // sized the buffer for): direct form, same arithmetic
    for (int idx = tid; idx < nrow * res; idx += CR_THREADS) {
      const int r = idx / res, ox = idx - r * res;
      const float *wy = wy_s + (size_t)r * yt;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int iy = 0; iy < yn_s[r]; ++iy) {
        float r0, r1, r2;
        hrow(ylo_s[r] + iy, ox, r0, r1, r2);
        a0 += wy[iy] * r0; a1 += wy[iy] * r1; a2 += wy[iy] * r2;
      }
      finish(oy0 + r, ox, a0, a1, a2);
    }
  }
}

struct CropPlan {
  int tr, rmax, xt, yt;
  size_t smem;
};
// tile height and shared-memory carve-up for the largest box an (h, w) image can hold
bool crop_plan(int h, int w, int res, int tile_rows, CropPlan &p) {
  const float ms = fmaxf((float)(h > w ? h : w) / (float)res, 1.0f);
  const int taps = 2 * (int)ceilf(2.0f * ms) + 1;
  if (taps > MAX_TAPS) return false;
  constexpr size_t LIMIT = CR_SMEM_LIMIT;
  for (int tr = tile_rows > 0 ? tile_rows : 16; tr >= 1; tr >>= 1) {
    p.tr = tr;
    p.xt = p.yt = taps;
    p.rmax = (int)ceilf(tr * ms) + 2 * (int)ceilf(2.0f * ms) + 3;
    p.smem = ((size_t)p.rmax * res * 3 + (size_t)res * p.xt + (size_t)tr * p.yt) * sizeof(float) +
             (size_t)(2 * res + 2 * tr) * sizeof(int);
    if (p.smem <= LIMIT) return true;
  }
  return false;
}

template <typename OutT>
int launch_crop(const CropPlan &p, int h, int w, int ncrops, int res, int patch, const uchar4 *rgbx, const int *scene,
                const int *boxes, const unsigned char *valid, const float *mean, const float *std, OutT *out,
                cudaStream_t s) {
  constexpr auto kern = crop_resize_sep_kernel<OutT>;
  // crop_plan keeps every launch within CR_SMEM_LIMIT
  if (const int st = raise_smem_limit<kern>((int)CR_SMEM_LIMIT)) return st;
  const dim3 grid((res + p.tr - 1) / p.tr, ncrops);
  kern<<<grid, CR_THREADS, p.smem, s>>>(h, w, res, p.tr, p.rmax, p.xt, p.yt, patch, rgbx, scene, boxes, valid, mean[0],
                                        mean[1], mean[2], std[0], std[1], std[2], out);
  return launch_status();
}

}  // namespace

extern "C" {

long long coda_crop_resize_workspace_bytes(int nimg, int h, int w) {
  return nimg > 0 && h > 0 && w > 0 ? (long long)nimg * h * w * 4 : 0;
}

int coda_crop_resize_normalize_ex(int nimg, int h, int w, int ncrops, int res, const unsigned char *images,
                                  const int *scene, const int *boxes, const unsigned char *valid, const float *mean,
                                  const float *std, int out_half, int patch, int tile_rows, void *workspace,
                                  void *out, void *stream) {
  if (nimg < 0 || h <= 0 || w <= 0 || ncrops < 0 || res <= 0 || patch < 0 || (patch > 0 && res % patch != 0) ||
      tile_rows < 0 || tile_rows > 64)
    return CODA_EINVAL;
  if (ncrops == 0) return CODA_OK;
  if (!images || !scene || !boxes || !valid || !mean || !std || !out || !workspace || ncrops > 65535 ||
      ((uintptr_t)workspace & 3))
    return CODA_EINVAL;
  CropPlan plan;
  // taps per axis = 2 * ceil(2 * scale) + 1 with scale <= max(h, w) / res
  if (!crop_plan(h, w, res, tile_rows, plan)) return CODA_ETOOLARGE;
  cudaStream_t s = (cudaStream_t)stream;
  const long long npix = (long long)nimg * h * w;
  uchar4 *rgbx = (uchar4 *)workspace;
  rgb_to_rgbx_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>(npix, images, rgbx);
  int st = launch_status();
  if (st != CODA_OK) return st;
  if (out_half)
    return launch_crop<__half>(plan, h, w, ncrops, res, patch, rgbx, scene, boxes, valid, mean, std, (__half *)out, s);
  return launch_crop<float>(plan, h, w, ncrops, res, patch, rgbx, scene, boxes, valid, mean, std, (float *)out, s);
}

}  // extern "C"
