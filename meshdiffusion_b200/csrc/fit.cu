// Geometry-only fit of DMTet training grids to triangle meshes (`--mode=fit_grids`, geometry/fit.py). The reference fits
// its grids by rendering (nvdiffrec/fit_dmtets.py); here the sign comes from multi-view space carving and the deformation
// from a point-to-mesh fit through the differentiable marching tets.
//
// * mdb_carve_vertices: a tet vertex is outside when one of the depth buffers mdb_raster_depth made sees it (the window
//   around its pixel is empty or deeper than the vertex). One thread per (mesh, vertex) loops over the views: no atomics.
// * mdb_closest_points: brute-force closest point on a packed triangle mesh for packed queries, triangles staged through
//   shared memory.
// * mdb_nearest_vertex: brute-force nearest point of a packed point set, points staged through shared memory.
// * mdb_segment_sum: the deterministic gather that takes the nearest-vertex gradient back to the vertices (CSR rows summed
//   in order, no float atomics).
//
// Every arithmetic step is rounded on its own (no FMA contraction, IEEE division), so a float32 numpy restatement
// (oracle/fit_oracle.py) reproduces the flags, distances, indices and closest points bit for bit.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <algorithm>
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

constexpr int kThreads = 256;  // queries per CTA of the brute-force searches
constexpr int kTile = 256;     // triangles or points per shared-memory tile

// Row i of a row-major 4 x 4 matrix times [x, y, z, 1]: ((m0 x + m1 y) + m2 z) + m3 (as csrc/raster.cu).
__device__ __forceinline__ float mvp_row(const float* m, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
}

// One thread per (vertex, mesh): the views are looped inside the thread, so the OR over views needs no atomics.
__global__ void __launch_bounds__(256) carve_kernel(const float* __restrict__ pts, int n_pts, const float* __restrict__ mvp,
                                                    int n_views, int res, int window, const float* __restrict__ depth,
                                                    const int* __restrict__ face_id, unsigned char* __restrict__ outside) {
  const int mesh = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts) return;
  unsigned char* out = outside + (long long)mesh * n_pts + i;
  if (*out) return;  // seen in an earlier call
  const float px = pts[3 * i], py = pts[3 * i + 1], pz = pts[3 * i + 2];
  const float fres = (float)res;
  bool seen = false;
  for (int v = 0; v < n_views && !seen; ++v) {
    const float* m = mvp + 16 * v;
    const float w = mvp_row(m + 12, px, py, pz);
    if (!(w > 0.f)) continue;
    const float X = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(mvp_row(m, px, py, pz), w), 0.5f), 0.5f), fres);
    const float Y = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(mvp_row(m + 4, px, py, pz), w), 0.5f), 0.5f), fres);
    const float z = __fdiv_rn(mvp_row(m + 8, px, py, pz), w);
    if (!(X >= 0.f && X < fres && Y >= 0.f && Y < fres)) continue;
    const int col = (int)X, row = (int)Y;  // pixel c spans [c, c + 1)
    const long long base = ((long long)mesh * n_views + v) * res * res;
    bool clear = true;
    for (int r = max(row - window, 0); r <= min(row + window, res - 1) && clear; ++r)
      for (int c = max(col - window, 0); c <= min(col + window, res - 1); ++c) {
        const long long k = base + (long long)r * res + c;
        if (face_id[k] >= 0 && !(depth[k] > z)) { clear = false; break; }
      }
    seen = clear;
  }
  if (seen) *out = 1;
}

// One thread per query, CTA row blockIdx.y = mesh; the mesh's triangles stream through shared memory in tiles.
__global__ void __launch_bounds__(kThreads) closest_points_kernel(const float* __restrict__ queries, const long long* __restrict__ query_off,
                                                                  const float* __restrict__ verts, const long long* __restrict__ faces,
                                                                  const long long* __restrict__ vert_off, const long long* __restrict__ face_off,
                                                                  float* __restrict__ out_d2, long long* __restrict__ out_face,
                                                                  float* __restrict__ out_cp) {
  __shared__ float tri[9][kTile];
  const int mesh = blockIdx.y;
  const long long q0 = query_off[mesh], nq = query_off[mesh + 1] - q0;
  if ((long long)blockIdx.x * kThreads >= nq) return;  // the whole CTA is past this mesh's queries
  const long long qi = (long long)blockIdx.x * kThreads + threadIdx.x;
  const bool active = qi < nq;
  V3 p{0.f, 0.f, 0.f};
  if (active) p = {queries[3 * (q0 + qi)], queries[3 * (q0 + qi) + 1], queries[3 * (q0 + qi) + 2]};
  const float* v = verts + 3 * vert_off[mesh];
  const long long f0 = face_off[mesh], nf = face_off[mesh + 1] - f0;
  float best = __int_as_float(0x7f800000);
  long long best_f = -1;
  V3 best_c{NAN, NAN, NAN};
  for (long long t0 = 0; t0 < nf; t0 += kTile) {
    const int n = (int)min((long long)kTile, nf - t0);
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const long long* f = faces + 3 * (f0 + t0 + j);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float* q = v + 3 * f[k];
        tri[3 * k][j] = q[0];
        tri[3 * k + 1][j] = q[1];
        tri[3 * k + 2][j] = q[2];
      }
    }
    __syncthreads();
    if (!active) continue;
    for (int j = 0; j < n; ++j) {
      const V3 c = closest_on_triangle(p, {tri[0][j], tri[1][j], tri[2][j]}, {tri[3][j], tri[4][j], tri[5][j]},
                                       {tri[6][j], tri[7][j], tri[8][j]});
      const float d = dist2(p, c);
      if (d < best) { best = d; best_f = t0 + j; best_c = c; }  // strict: ties keep the lower face index
    }
  }
  if (!active) return;
  out_d2[q0 + qi] = best;
  out_face[q0 + qi] = best_f;
  out_cp[3 * (q0 + qi)] = best_c.x;
  out_cp[3 * (q0 + qi) + 1] = best_c.y;
  out_cp[3 * (q0 + qi) + 2] = best_c.z;
}

__global__ void __launch_bounds__(kThreads) nearest_vertex_kernel(const float* __restrict__ queries, const long long* __restrict__ query_off,
                                                                  const float* __restrict__ points, const long long* __restrict__ point_off,
                                                                  float* __restrict__ out_d2, long long* __restrict__ out_idx) {
  __shared__ float pt[3][kTile];
  const int mesh = blockIdx.y;
  const long long q0 = query_off[mesh], nq = query_off[mesh + 1] - q0;
  if ((long long)blockIdx.x * kThreads >= nq) return;
  const long long qi = (long long)blockIdx.x * kThreads + threadIdx.x;
  const bool active = qi < nq;
  V3 p{0.f, 0.f, 0.f};
  if (active) p = {queries[3 * (q0 + qi)], queries[3 * (q0 + qi) + 1], queries[3 * (q0 + qi) + 2]};
  const long long p0 = point_off[mesh], np_ = point_off[mesh + 1] - p0;
  float best = __int_as_float(0x7f800000);
  long long best_i = -1;
  for (long long t0 = 0; t0 < np_; t0 += kTile) {
    const int n = (int)min((long long)kTile, np_ - t0);
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      const float* q = points + 3 * (p0 + t0 + j);
      pt[0][j] = q[0];
      pt[1][j] = q[1];
      pt[2][j] = q[2];
    }
    __syncthreads();
    if (!active) continue;
    for (int j = 0; j < n; ++j) {
      const float d = dist2(p, {pt[0][j], pt[1][j], pt[2][j]});
      if (d < best) { best = d; best_i = t0 + j; }
    }
  }
  if (!active) return;
  out_d2[q0 + qi] = best;
  out_idx[q0 + qi] = best_i;
}

// out[r][c] = sum over k in [row_off[r], row_off[r + 1]) of src[perm[k]][c], added in k order.
__global__ void segment_sum_kernel(const float* __restrict__ src, int width, const long long* __restrict__ perm,
                                   const long long* __restrict__ row_off, long long n_rows, float* __restrict__ out) {
  const long long n = n_rows * width;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / width;
    const int c = (int)(i % width);
    float acc = 0.f;
    for (long long k = row_off[r]; k < row_off[r + 1]; ++k) acc = __fadd_rn(acc, src[perm[k] * width + c]);
    out[i] = acc;
  }
}

int check_search(const char* what, int n_meshes, long long max_queries) {
  if (n_meshes < 0 || n_meshes > 65535) return fail(std::string(what) + ": 0 to 65535 meshes per call");
  if (max_queries < 0 || (max_queries + kThreads - 1) / kThreads > 0x7fffffffLL)
    return fail(std::string(what) + ": max_queries out of range");
  return 0;
}

}  // namespace

extern "C" {

int mdb_carve_vertices(const float* pts, int n_pts, const float* mvp, int n_views, int n_meshes, int res, int window,
                       const float* depth, const int* face_id, unsigned char* outside, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n_pts < 0 || n_views < 0) return fail("mdb_carve_vertices: negative vertex or view count");
  if (n_meshes < 0 || n_meshes > 65535) return fail("mdb_carve_vertices: 0 to 65535 meshes per call");
  if (res < 1 || res > 16384) return fail("mdb_carve_vertices: resolution must be in [1, 16384]");
  if (window < 0 || window > 64) return fail("mdb_carve_vertices: window must be in [0, 64]");
  if (n_pts == 0 || n_views == 0 || n_meshes == 0) return 0;
  carve_kernel<<<dim3((unsigned)((n_pts + 255) / 256), (unsigned)n_meshes), 256, 0, s>>>(pts, n_pts, mvp, n_views, res, window,
                                                                                         depth, face_id, outside);
  return check_launch("mdb_carve_vertices");
}

int mdb_closest_points(const float* queries, const long long* query_off, int n_meshes, long long max_queries, const float* verts,
                       const long long* faces, const long long* vert_off, const long long* face_off, float* dist2,
                       long long* face, float* closest, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_search("mdb_closest_points", n_meshes, max_queries)) return 1;
  if (n_meshes == 0 || max_queries == 0) return 0;
  closest_points_kernel<<<dim3((unsigned)((max_queries + kThreads - 1) / kThreads), (unsigned)n_meshes), kThreads, 0, s>>>(
      queries, query_off, verts, faces, vert_off, face_off, dist2, face, closest);
  return check_launch("mdb_closest_points");
}

int mdb_nearest_vertex(const float* queries, const long long* query_off, int n_meshes, long long max_queries, const float* points,
                       const long long* point_off, float* dist2, long long* index, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_search("mdb_nearest_vertex", n_meshes, max_queries)) return 1;
  if (n_meshes == 0 || max_queries == 0) return 0;
  nearest_vertex_kernel<<<dim3((unsigned)((max_queries + kThreads - 1) / kThreads), (unsigned)n_meshes), kThreads, 0, s>>>(
      queries, query_off, points, point_off, dist2, index);
  return check_launch("mdb_nearest_vertex");
}

int mdb_segment_sum(const float* src, int width, const long long* perm, const long long* row_off, long long n_rows, float* out,
                    void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (width < 1 || n_rows < 0) return fail("mdb_segment_sum: width must be positive and n_rows non-negative");
  if (n_rows == 0) return 0;
  const long long n = n_rows * width;
  const long long blocks = std::min<long long>((n + 255) / 256, 65535);
  segment_sum_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, width, perm, row_off, n_rows, out);
  return check_launch("mdb_segment_sum");
}

}  // extern "C"
