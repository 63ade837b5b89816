// Point-triangle closest points shared by the mesh search of csrc/fit.cu and the depth-map search of csrc/depth_partial.cu.
// Every arithmetic step is rounded on its own (no FMA contraction, IEEE division), so oracle/fit_oracle.py's
// closest_on_triangles reproduces the points bit for bit.
#pragma once
#include <cuda_runtime.h>

namespace mdb {
namespace geom {

struct V3 { float x, y, z; };

__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
// a + s d
__device__ __forceinline__ V3 axpy3(V3 a, float s, V3 d) {
  return {__fadd_rn(a.x, __fmul_rn(s, d.x)), __fadd_rn(a.y, __fmul_rn(s, d.y)), __fadd_rn(a.z, __fmul_rn(s, d.z))};
}
// (a.x b.x + a.y b.y) + a.z b.z
__device__ __forceinline__ float dot3(V3 a, V3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ bool finite3(V3 a) { return isfinite(a.x) && isfinite(a.y) && isfinite(a.z); }

// Closest point to p on segment a -> b: a + clamp(ap.ab / ab.ab, 0, 1) ab, a itself when a == b.
__device__ __forceinline__ V3 closest_on_segment(V3 p, V3 a, V3 b) {
  const V3 ab = sub3(b, a);
  const float den = dot3(ab, ab);
  float t = den > 0.f ? __fdiv_rn(dot3(sub3(p, a), ab), den) : 0.f;
  t = fminf(fmaxf(t, 0.f), 1.f);
  return axpy3(a, t, ab);
}

// Closest point to p on triangle abc by its Voronoi regions (vertices, edges, interior) in the order of Ericson, Real-Time
// Collision Detection, 5.1.5. A degenerate triangle, whose regions do not resolve to a finite point, takes the nearest of its
// three edges ab, bc, ca (the first on ties).
__device__ __forceinline__ V3 closest_on_triangle(V3 p, V3 a, V3 b, V3 c) {
  const V3 ab = sub3(b, a), ac = sub3(c, a), ap = sub3(p, a);
  const float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
  if (d1 <= 0.f && d2 <= 0.f) return a;
  const V3 bp = sub3(p, b);
  const float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
  if (d3 >= 0.f && d4 <= d3) return b;
  V3 r;
  const float vc = __fsub_rn(__fmul_rn(d1, d4), __fmul_rn(d3, d2));
  if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
    r = axpy3(a, __fdiv_rn(d1, __fsub_rn(d1, d3)), ab);
  } else {
    const V3 cp = sub3(p, c);
    const float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.f && d5 <= d6) return c;
    const float vb = __fsub_rn(__fmul_rn(d5, d2), __fmul_rn(d1, d6));
    const float va = __fsub_rn(__fmul_rn(d3, d6), __fmul_rn(d5, d4));
    const float e43 = __fsub_rn(d4, d3), e56 = __fsub_rn(d5, d6);
    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
      r = axpy3(a, __fdiv_rn(d2, __fsub_rn(d2, d6)), ac);
    } else if (va <= 0.f && e43 >= 0.f && e56 >= 0.f) {
      r = axpy3(b, __fdiv_rn(e43, __fadd_rn(e43, e56)), sub3(c, b));
    } else {
      const float den = __fadd_rn(__fadd_rn(va, vb), vc);
      r = den > 0.f ? axpy3(axpy3(a, __fdiv_rn(vb, den), ab), __fdiv_rn(vc, den), ac) : V3{NAN, NAN, NAN};
    }
  }
  if (finite3(r)) return r;
  const V3 s0 = closest_on_segment(p, a, b), s1 = closest_on_segment(p, b, c), s2 = closest_on_segment(p, c, a);
  const V3 e0 = sub3(p, s0), e1 = sub3(p, s1), e2 = sub3(p, s2);
  const float q0 = dot3(e0, e0), q1 = dot3(e1, e1), q2 = dot3(e2, e2);
  r = s0;
  float q = q0;
  if (q1 < q) { r = s1; q = q1; }
  if (q2 < q) r = s2;
  return r;
}

// dist2 = (dx dx + dy dy) + dz dz of d = p - c
__device__ __forceinline__ float dist2(V3 p, V3 c) { const V3 d = sub3(p, c); return dot3(d, d); }

}  // namespace geom
}  // namespace mdb
