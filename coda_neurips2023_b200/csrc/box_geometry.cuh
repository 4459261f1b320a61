// Ground-plane polygon geometry of 3-D boxes that are rotated about the up axis: Sutherland-Hodgman clip of two
// quadrilaterals (reference utils/box_util.py:34-112 polygon_clip / :540-578 polygon_clip_unnest).  Shared by the
// matcher's generalised IoU (detr_kernels.cu) and the evaluation IoU (eval_kernels.cu).
#pragma once

namespace coda {

struct P2 { float x, y; };

__device__ __forceinline__ bool sh_inside(P2 cp1, P2 cp2, P2 p) {
  return (cp2.x - cp1.x) * (p.y - cp1.y) > (cp2.y - cp1.y) * (p.x - cp1.x);
}
__device__ __forceinline__ P2 sh_intersect(P2 cp1, P2 cp2, P2 s, P2 e) {
  const float dcx = cp1.x - cp2.x, dcy = cp1.y - cp2.y;
  const float dpx = s.x - e.x, dpy = s.y - e.y;
  const float n1 = cp1.x * cp2.y - cp1.y * cp2.x;
  const float n2 = s.x * e.y - s.y * e.x;
  const float n3 = 1.0f / (dcx * dpy - dcy * dpx);
  return P2{(n1 * dpx - n2 * dcx) * n3, (n1 * dpy - n2 * dcy) * n3};
}

// Sutherland-Hodgman clip of quadrilateral `subj` by convex quadrilateral `clip`
// (utils/box_util.py:540-578); returns twice-unsigned-area / 2 of the result.
// The area does not depend on where the pair stands, but sh_intersect and the shoelace sum multiply coordinates and
// subtract the products, so their rounding error grows with |coordinate|^2: all eight points are first taken relative
// to clip[0] (differences of nearby fp32 numbers, exact or correctly rounded at the scale of the pair), which keeps
// the error a property of the two boxes wherever in the scene they are.
__device__ inline float clipped_area(const P2 *subj, const P2 *clip) {
  P2 a[10], bq[10], cl[4];
  int na = 4;
  const P2 org = clip[0];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    a[i] = P2{subj[i].x - org.x, subj[i].y - org.y};
    cl[i] = P2{clip[i].x - org.x, clip[i].y - org.y};
  }
  P2 cp1 = cl[3];
  for (int ci = 0; ci < 4; ++ci) {
    const P2 cp2 = cl[ci];
    int nb = 0;
    P2 s = a[na - 1];
    for (int i = 0; i < na; ++i) {
      const P2 e = a[i];
      const bool ein = sh_inside(cp1, cp2, e);
      if (ein) {
        if (!sh_inside(cp1, cp2, s) && nb < 10) bq[nb++] = sh_intersect(cp1, cp2, s, e);
        if (nb < 10) bq[nb++] = e;
      } else if (sh_inside(cp1, cp2, s)) {
        if (nb < 10) bq[nb++] = sh_intersect(cp1, cp2, s, e);
      }
      s = e;
    }
    cp1 = cp2;
    na = nb;
    for (int i = 0; i < nb; ++i) a[i] = bq[i];
    if (na == 0) return 0.f;
  }
  // |dot(xs, roll(ys, 1)) - dot(ys, roll(xs, 1))| * 0.5
  float s1 = 0.f, s2 = 0.f;
  for (int i = 0; i < na; ++i) {
    const int j = (i + na - 1) % na;
    s1 += a[i].x * a[j].y;
    s2 += a[i].y * a[j].x;
  }
  return fabsf(s1 - s2) * 0.5f;
}

}  // namespace coda
