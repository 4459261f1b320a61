/*
 * box_oracle.c -- CPU restatement of the reference's rotated-rectangle intersection
 * (Sutherland-Hodgman clip + shoelace area).  TEST INFRASTRUCTURE ONLY (see
 * pointnet2_oracle.c).  Follows reference utils/box_util.py:524-578
 * (helper_computeIntersection, helper_inside, polygon_clip_unnest) and the area
 * formula of :726-733, in fp32 like the TorchScript path the reference falls back
 * to when its Cython module is not compiled (utils/box_util.py:855-868).
 *
 * rect1 (b, k1, 4, 2), rect2 (b, k2, 4, 2), non_rot (b, k1, k2), nums_k2 (b)
 * -> inter_areas (b, k1, k2); pairs with non_rot == 0, k2 >= nums_k2[b] or
 *    k2 >= k2_limit keep 0.
 */
#include <math.h>
#include <string.h>

typedef struct { float x, y; } P2;

static int inside(P2 cp1, P2 cp2, P2 p) {
  return (cp2.x - cp1.x) * (p.y - cp1.y) > (cp2.y - cp1.y) * (p.x - cp1.x);
}
static P2 intersect(P2 cp1, P2 cp2, P2 s, P2 e) {
  const float dcx = cp1.x - cp2.x, dcy = cp1.y - cp2.y;
  const float dpx = s.x - e.x, dpy = s.y - e.y;
  const float n1 = cp1.x * cp2.y - cp1.y * cp2.x;
  const float n2 = s.x * e.y - s.y * e.x;
  const float n3 = 1.0f / (dcx * dpy - dcy * dpx);
  P2 r = {(n1 * dpx - n2 * dcx) * n3, (n1 * dpy - n2 * dcy) * n3};
  return r;
}

/* like the kernel (csrc/box_geometry.cuh), on the eight points taken relative to clip[0] */
static float clipped_area(const P2 *subj, const P2 *clip) {
  P2 a[16], b[16], cl[4];
  int na = 4;
  const P2 org = clip[0];
  for (int i = 0; i < 4; ++i) {
    a[i].x = subj[i].x - org.x; a[i].y = subj[i].y - org.y;
    cl[i].x = clip[i].x - org.x; cl[i].y = clip[i].y - org.y;
  }
  P2 cp1 = cl[3];
  for (int ci = 0; ci < 4; ++ci) {
    const P2 cp2 = cl[ci];
    int nb = 0;
    P2 s = a[na - 1];
    for (int i = 0; i < na; ++i) {
      const P2 e = a[i];
      if (inside(cp1, cp2, e)) {
        if (!inside(cp1, cp2, s)) b[nb++] = intersect(cp1, cp2, s, e);
        b[nb++] = e;
      } else if (inside(cp1, cp2, s)) {
        b[nb++] = intersect(cp1, cp2, s, e);
      }
      s = e;
    }
    cp1 = cp2;
    na = nb;
    memcpy(a, b, sizeof(P2) * nb);
    if (na == 0) return 0.f;
  }
  float s1 = 0.f, s2 = 0.f;
  for (int i = 0; i < na; ++i) {
    const int j = (i + na - 1) % na;
    s1 += a[i].x * a[j].y;
    s2 += a[i].y * a[j].x;
  }
  return fabsf(s1 - s2) * 0.5f;
}

void oracle_rotated_inter_areas(int b, int k1, int k2, int k2_limit, const float *rect1,
                                const float *rect2, const float *non_rot, const int *nums_k2,
                                float *inter_areas) {
  memset(inter_areas, 0, sizeof(float) * (size_t)b * k1 * k2);
  for (int bi = 0; bi < b; ++bi)
    for (int i = 0; i < k1; ++i)
      for (int j = 0; j < k2; ++j) {
        if (j >= nums_k2[bi] || j >= k2_limit) break;
        const size_t o = ((size_t)bi * k1 + i) * k2 + j;
        if (non_rot[o] == 0.f) continue;
        inter_areas[o] = clipped_area((const P2 *)(rect1 + ((size_t)bi * k1 + i) * 8),
                                      (const P2 *)(rect2 + ((size_t)bi * k2 + j) * 8));
      }
}
