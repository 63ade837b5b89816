// Partial DMTets from observed depth maps (`--mode=partial_from_depth`, geometry/depth_partial.py): what one camera sees
// of a surface, turned into the buffers the carving and fitting kernels consume.
//
// * mdb_depth_unproject: one thread per pixel. From a camera depth map it writes the z / w buffer and a face-id-like
//   validity buffer (the layout mdb_raster_depth gives mdb_carve_vertices), the back-projected world point of every pixel
//   centre, and a flag for pixels beside a depth discontinuity (a silhouette, not a surface).
// * mdb_depth_closest_points: one thread per query. The closest point on the observed surface, searched in image space:
//   the query is projected, and the two triangles of every 2 x 2 pixel block of a window around it are tested exactly. No
//   mesh is materialized; blocks are scanned in pixel order and a later triangle wins only when strictly nearer, so there
//   are no atomics and the result is deterministic.
//
// Every arithmetic step is rounded on its own (no FMA contraction, IEEE division), so a float32 numpy restatement
// (oracle/depth_oracle.py) reproduces the buffers, flags, distances and points bit for bit.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <string>

#include "closest_point.cuh"

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

using namespace mdb::geom;

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(std::string(what) + ": " + cudaGetErrorString(e));
}

constexpr float kEmptyDepth = 100.f;  // the rasterizer's empty z / w
constexpr int kMaxHalf = 31;          // window half-width in blocks: at most 2 * 31 + 2 = 64 pixels a side
constexpr int kThreads = 256;

// Row i of a row-major 4 x 4 matrix times [x, y, z, 1]: ((m0 x + m1 y) + m2 z) + m3 (as csrc/raster.cu).
__device__ __forceinline__ float mvp_row(const float* m, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
}

__device__ __forceinline__ bool observed(float d) { return isfinite(d) && d > 0.f; }

__global__ void __launch_bounds__(kThreads) unproject_kernel(const float* __restrict__ depth, int res, const float* __restrict__ proj,
                                                             const float* __restrict__ inv_mv, float max_jump, float* __restrict__ zbuf,
                                                             int* __restrict__ valid, float* __restrict__ points,
                                                             unsigned char* __restrict__ edge) {
  const int obs = blockIdx.y;
  const long long n = (long long)res * res;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const int r = (int)(i / res), c = (int)(i % res);
  const float* D = depth + obs * n;
  const long long k = obs * n + i;
  const float d = D[i];
  if (!observed(d)) {
    zbuf[k] = kEmptyDepth;
    valid[k] = -1;
    points[3 * k] = 0.f;
    points[3 * k + 1] = 0.f;
    points[3 * k + 2] = 0.f;
    edge[k] = 0;
    return;
  }
  const float* P = proj + 16 * obs;
  const float fres = (float)res;
  // pixel centre -> NDC: (c + 0.5) / res * 2 - 1; camera x = d (x_ndc + p02) / p00, y likewise, z = -d
  const float xn = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)c, 0.5f), fres), 2.f), 1.f);
  const float yn = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)r, 0.5f), fres), 2.f), 1.f);
  const float xc = __fdiv_rn(__fmul_rn(d, __fadd_rn(xn, P[2])), P[0]);
  const float yc = __fdiv_rn(__fmul_rn(d, __fadd_rn(yn, P[6])), P[5]);
  const float zc = -d;
  const float* M = inv_mv + 16 * obs;
  points[3 * k] = mvp_row(M, xc, yc, zc);
  points[3 * k + 1] = mvp_row(M + 4, xc, yc, zc);
  points[3 * k + 2] = mvp_row(M + 8, xc, yc, zc);
  // z / w = (A z_cam + B) / d = (B - A d) / d
  zbuf[k] = __fdiv_rn(__fsub_rn(P[11], __fmul_rn(P[10], d)), d);
  valid[k] = 0;
  bool e = false;
  if (c > 0 && observed(D[i - 1])) e |= fabsf(__fsub_rn(d, D[i - 1])) > max_jump;
  if (c + 1 < res && observed(D[i + 1])) e |= fabsf(__fsub_rn(d, D[i + 1])) > max_jump;
  if (r > 0 && observed(D[i - res])) e |= fabsf(__fsub_rn(d, D[i - res])) > max_jump;
  if (r + 1 < res && observed(D[i + res])) e |= fabsf(__fsub_rn(d, D[i + res])) > max_jump;
  edge[k] = e ? 1 : 0;
}

__device__ __forceinline__ bool usable(const int* valid, const unsigned char* edge, long long k) {
  return valid[k] == 0 && edge[k] == 0;
}

__device__ __forceinline__ V3 point_at(const float* __restrict__ p, long long k) { return {p[3 * k], p[3 * k + 1], p[3 * k + 2]}; }

// One thread per query, CTA row blockIdx.y = observation.
__global__ void __launch_bounds__(kThreads) depth_closest_kernel(const float* __restrict__ queries, const long long* __restrict__ query_off,
                                                                 int res, const float* __restrict__ mvp, const float* __restrict__ proj,
                                                                 float radius, const float* __restrict__ points,
                                                                 const int* __restrict__ valid, const unsigned char* __restrict__ edge,
                                                                 float* __restrict__ out_d2, float* __restrict__ out_cp,
                                                                 unsigned char* __restrict__ out_found) {
  const int obs = blockIdx.y;
  const long long q0 = query_off[obs], nq = query_off[obs + 1] - q0;
  const long long qi = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (qi >= nq) return;
  const long long qk = q0 + qi;
  const V3 p{queries[3 * qk], queries[3 * qk + 1], queries[3 * qk + 2]};
  const float* m = mvp + 16 * obs;
  const float* P = proj + 16 * obs;
  const float fres = (float)res;
  float best = __int_as_float(0x7f800000);
  V3 best_c{NAN, NAN, NAN};
  bool found = false;
  const float w = mvp_row(m + 12, p.x, p.y, p.z);
  if (w > 0.f) {
    const float X = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(mvp_row(m, p.x, p.y, p.z), w), 0.5f), 0.5f), fres);
    const float Y = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(mvp_row(m + 4, p.x, p.y, p.z), w), 0.5f), 0.5f), fres);
    // pixels per world unit at camera depth w: max(|p00|, |p11|) * res / 2 / w; the window spans `radius` either side
    const float scale = __fmul_rn(__fmul_rn(fmaxf(fabsf(P[0]), fabsf(P[5])), 0.5f), fres);
    const float hp = __fdiv_rn(__fmul_rn(radius, scale), w);
    if (X > -64.f && X < fres + 64.f && Y > -64.f && Y < fres + 64.f) {
      const int half = hp >= (float)kMaxHalf ? kMaxHalf : (int)ceilf(hp);
      // block (r, c) has its corners at the centres of pixels (r, c) .. (r + 1, c + 1); the query's block holds X, Y
      const int cq = (int)floorf(__fsub_rn(X, 0.5f)), rq = (int)floorf(__fsub_rn(Y, 0.5f));
      const long long base = (long long)obs * res * res;
      const int r0 = max(rq - half, 0), r1 = min(rq + half, res - 2);
      const int c0 = max(cq - half, 0), c1 = min(cq + half, res - 2);
      for (int r = r0; r <= r1; ++r)
        for (int c = c0; c <= c1; ++c) {
          const long long k00 = base + (long long)r * res + c, k10 = k00 + res;
          if (!(usable(valid, edge, k00) && usable(valid, edge, k00 + 1) && usable(valid, edge, k10) &&
                usable(valid, edge, k10 + 1)))
            continue;
          const V3 a = point_at(points, k00), b = point_at(points, k00 + 1);
          const V3 cc = point_at(points, k10 + 1), dd = point_at(points, k10);
          // triangles (00, 01, 11) then (00, 11, 10); strict: ties keep the lower pixel, then the first triangle
          const V3 t0 = closest_on_triangle(p, a, b, cc);
          const float e0 = dist2(p, t0);
          if (e0 < best) { best = e0; best_c = t0; found = true; }
          const V3 t1 = closest_on_triangle(p, a, cc, dd);
          const float e1 = dist2(p, t1);
          if (e1 < best) { best = e1; best_c = t1; found = true; }
        }
    }
  }
  out_d2[qk] = best;
  out_cp[3 * qk] = best_c.x;
  out_cp[3 * qk + 1] = best_c.y;
  out_cp[3 * qk + 2] = best_c.z;
  out_found[qk] = found ? 1 : 0;
}

int check_obs(const char* what, int n_obs, int res) {
  if (n_obs < 0 || n_obs > 65535) return fail(std::string(what) + ": 0 to 65535 observations per call");
  if (res < 2 || res > 4096) return fail(std::string(what) + ": the image side must be in [2, 4096]");
  return 0;
}

}  // namespace

extern "C" {

int mdb_depth_unproject(const float* depth, int n_obs, int res, const float* proj, const float* inv_mv, float max_jump,
                        float* zbuf, int* valid, float* points, unsigned char* edge, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_obs("mdb_depth_unproject", n_obs, res)) return 1;
  if (!(max_jump >= 0.f)) return fail("mdb_depth_unproject: max_jump must be a non-negative number");
  if (n_obs == 0) return 0;
  const long long n = (long long)res * res;
  unproject_kernel<<<dim3((unsigned)((n + kThreads - 1) / kThreads), (unsigned)n_obs), kThreads, 0, s>>>(
      depth, res, proj, inv_mv, max_jump, zbuf, valid, points, edge);
  return check_launch("mdb_depth_unproject");
}

int mdb_depth_closest_points(const float* queries, const long long* query_off, int n_obs, long long max_queries, int res,
                             const float* mvp, const float* proj, float radius, const float* points, const int* valid,
                             const unsigned char* edge, float* dist2, float* closest, unsigned char* found, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_obs("mdb_depth_closest_points", n_obs, res)) return 1;
  if (max_queries < 0 || (max_queries + kThreads - 1) / kThreads > 0x7fffffffLL)
    return fail("mdb_depth_closest_points: max_queries out of range");
  if (!(radius >= 0.f)) return fail("mdb_depth_closest_points: radius must be a non-negative number");
  if (n_obs == 0 || max_queries == 0) return 0;
  depth_closest_kernel<<<dim3((unsigned)((max_queries + kThreads - 1) / kThreads), (unsigned)n_obs), kThreads, 0, s>>>(
      queries, query_off, res, mvp, proj, radius, points, valid, edge, dist2, closest, found);
  return check_launch("mdb_depth_closest_points");
}

}  // extern "C"
