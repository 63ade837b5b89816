// Single-view visibility of a DMTet, for the partial DMTets `--mode=cond_gen` conditions on (the tail of
// nvdiffrec/fit_singleview.py:783-827 over nvdiffrec/lib/render/render.py:335-407).
//
// * mdb_raster_depth: first-layer depth / face-id rasterization of a batch of (mesh, view) jobs. No shading, MSAA, depth
//   peeling or near-plane clipping. Every arithmetic step is rounded on its own (no FMA contraction, IEEE division), so
//   a float32 numpy restatement (oracle/raster_oracle.py) reproduces the buffers bit for bit, and the depth test is an
//   atomicMin on (depth key, face index): the result does not depend on scheduling.
// * mdb_visible_tets: the reference's visible-tet test (a tet centre in front of the minimum depth, or over empty pixels,
//   of the 15 x 15 window around its pixel) fused into one pass, plus the flags of the tets that own a rasterized face.
// * mdb_render_shade: the diffuse, environment-lit preview of nvdiffrec/eval.py on the face ids of a supersampled
//   mdb_raster_depth pass: perspective-correct interpolation, nvdiffrec's two-sided shading normal, 9-term SH irradiance,
//   a box resolve in linear space and an sRGB encode by threshold table. Rounded step by step like the rasterizer
//   (oracle/render_oracle.py).
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <algorithm>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(std::string(what) + ": " + cudaGetErrorString(e));
}

constexpr float kEmptyDepth = 100.f;  // render.py:375
constexpr int kWindow = 7;            // render.py:386, depth_search_range
constexpr int kRasterWarps = 8;

// Row i of a row-major 4 x 4 matrix times [x, y, z, 1]: ((m0 x + m1 y) + m2 z) + m3.
__device__ __forceinline__ float mvp_row(const float* m, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
}

// Edge function of a -> b at p: (bx - ax)(py - ay) - (by - ay)(px - ax).
__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float px, float py) {
  return __fsub_rn(__fmul_rn(__fsub_rn(bx, ax), __fsub_rn(py, ay)), __fmul_rn(__fsub_rn(by, ay), __fsub_rn(px, ax)));
}

struct Tri {
  float x[3], y[3], z[3];  // screen x, y in pixels, z / w
  float area;              // edge_fn(v0, v1, v2)
  float xmin, xmax, ymin, ymax;
};

// Screen position of the face's vertices. Returns false when the face is not drawn; `behind` is set when a vertex has
// w <= 0 (or NaN). A face with a non-finite screen coordinate or a zero or non-finite area is not drawn either.
__device__ __forceinline__ bool setup_tri(const float* __restrict__ v, const long long* __restrict__ f, const float* m,
                                          float res, Tri& t, bool& behind) {
  behind = false;
  bool finite = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = v + 3 * f[k];
    const float px = p[0], py = p[1], pz = p[2];
    const float cx = mvp_row(m, px, py, pz), cy = mvp_row(m + 4, px, py, pz);
    const float cz = mvp_row(m + 8, px, py, pz), cw = mvp_row(m + 12, px, py, pz);
    if (!(cw > 0.f)) behind = true;
    t.x[k] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(cx, cw), 0.5f), 0.5f), res);
    t.y[k] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(cy, cw), 0.5f), 0.5f), res);
    t.z[k] = __fdiv_rn(cz, cw);
    finite = finite && isfinite(t.x[k]) && isfinite(t.y[k]) && isfinite(t.z[k]);
  }
  if (behind || !finite) return false;
  t.area = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  if (!isfinite(t.area) || t.area == 0.f) return false;
  t.xmin = fminf(fminf(t.x[0], t.x[1]), t.x[2]);
  t.xmax = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]);
  t.ymin = fminf(fminf(t.y[0], t.y[1]), t.y[2]);
  t.ymax = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]);
  return true;
}

// The fragment of a drawn face at pixel centre (px, py). Covered when the centre is inside the face's bounding box and
// every edge function has the sign of the area or is zero; depth = ((e0 z0 + e1 z1) + e2 z2) / area is kept when it is
// in [-1, 1].
__device__ __forceinline__ bool fragment(const Tri& t, float px, float py, float& depth) {
  if (!(px >= t.xmin && px <= t.xmax && py >= t.ymin && py <= t.ymax)) return false;
  const float e0 = edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], px, py);
  const float e1 = edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], px, py);
  const float e2 = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], px, py);
  const bool in = t.area > 0.f ? (e0 >= 0.f && e1 >= 0.f && e2 >= 0.f) : (e0 <= 0.f && e1 <= 0.f && e2 <= 0.f);
  if (!in) return false;
  depth = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(e0, t.z[0]), __fmul_rn(e1, t.z[1])), __fmul_rn(e2, t.z[2])), t.area);
  return depth >= -1.f && depth <= 1.f;
}

// Order-preserving map of a float's bits to an unsigned key (negative floats reversed, positive ones above them).
__device__ __forceinline__ unsigned depth_key(float d) {
  const unsigned u = __float_as_uint(d);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_depth(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// One warp per (face, job): the lanes walk the pixels of the face's clipped bounding box.
__global__ void __launch_bounds__(32 * kRasterWarps) raster_kernel(const float* __restrict__ verts, const long long* __restrict__ faces,
                                                                   const long long* __restrict__ vert_off,
                                                                   const long long* __restrict__ face_off, const int* __restrict__ job_mesh,
                                                                   const float* __restrict__ mvps, int res,
                                                                   unsigned long long* __restrict__ zbuf, int* __restrict__ n_behind) {
  const int job = blockIdx.y, lane = threadIdx.x % 32;
  const int mesh = job_mesh[job];
  const long long f0 = face_off[mesh], nf = face_off[mesh + 1] - f0;
  const float* v = verts + 3 * vert_off[mesh];
  float m[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) m[i] = mvps[16 * job + i];
  const float fres = (float)res;
  unsigned long long* zb = zbuf + (long long)job * res * res;
  for (long long f = (long long)blockIdx.x * kRasterWarps + threadIdx.x / 32; f < nf; f += (long long)gridDim.x * kRasterWarps) {
    Tri t;
    bool behind;
    const bool drawn = setup_tri(v, faces + 3 * (f0 + f), m, fres, t, behind);
    if (behind && lane == 0) atomicAdd(n_behind + job, 1);
    if (!drawn) continue;
    // pixel c has its centre at c + 0.5: columns floor(xmin) - 1 .. ceil(xmax) hold every centre in [xmin, xmax]
    const float c_lo = fmaxf(floorf(t.xmin) - 1.f, 0.f), c_hi = fminf(ceilf(t.xmax), fres - 1.f);
    const float r_lo = fmaxf(floorf(t.ymin) - 1.f, 0.f), r_hi = fminf(ceilf(t.ymax), fres - 1.f);
    if (c_lo > c_hi || r_lo > r_hi) continue;
    const int c0 = (int)c_lo, r0 = (int)r_lo, w = (int)c_hi - c0 + 1;
    const long long n = (long long)w * ((int)r_hi - r0 + 1);
    for (long long i = lane; i < n; i += 32) {
      const int r = r0 + (int)(i / w), c = c0 + (int)(i % w);
      float d;
      if (fragment(t, (float)c + 0.5f, (float)r + 0.5f, d))
        atomicMin(zb + (long long)r * res + c, ((unsigned long long)depth_key(d) << 32) | (unsigned long long)(unsigned)f);
    }
  }
}

__global__ void resolve_kernel(const unsigned long long* __restrict__ zbuf, long long n, float* __restrict__ depth, int* __restrict__ face_id) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = zbuf[i];
    const bool empty = k == ~0ull;
    depth[i] = empty ? kEmptyDepth : key_depth((unsigned)(k >> 32));
    face_id[i] = empty ? -1 : (int)(unsigned)(k & 0xffffffffull);
  }
}

// One thread per (tet, job): render.py:346-407 without the max_pool2d temporaries.
__global__ void __launch_bounds__(256) visible_tets_kernel(const float* __restrict__ pos, long long pos_stride, const int* __restrict__ tets,
                                                           int n_tets, const int* __restrict__ job_mesh, const float* __restrict__ mvps,
                                                           int res, const float* __restrict__ depth, const int* __restrict__ face_id,
                                                           unsigned char* __restrict__ visible) {
  const int job = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tets) return;
  const float* p = pos + (long long)job_mesh[job] * pos_stride;
  const float* m = mvps + 16 * job;
  const int4 tv = reinterpret_cast<const int4*>(tets)[t];
  float c[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)  // getTetCenters (dmtet.py:253-257)
    c[k] = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(p[3 * tv.x + k], p[3 * tv.y + k]), p[3 * tv.z + k]), p[3 * tv.w + k]), 0.25f);
  const float hw = mvp_row(m + 12, c[0], c[1], c[2]);
  float n[3], q[3];
  const float top = (float)(res - 1);
  bool in_view = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    n[k] = __fdiv_rn(mvp_row(m + 4 * k, c[0], c[1], c[2]), hw);
    q[k] = rintf(__fmul_rn(__fadd_rn(__fmul_rn(n[k], 0.5f), 0.5f), top));  // torch.round: half to even
    in_view = in_view && q[k] >= 0.f && q[k] <= top;
  }
  unsigned char vis = 0;
  if (in_view) {
    const int row = (int)q[1], col = (int)q[0];  // the reference swaps x and y before indexing [row, col]
    const float* d = depth + (long long)job * res * res;
    const int* id = face_id + (long long)job * res * res;
    float dmin = __int_as_float(0x7f800000);
    bool empty = true;
    for (int r = max(row - kWindow, 0); r <= min(row + kWindow, res - 1); ++r)
      for (int cc = max(col - kWindow, 0); cc <= min(col + kWindow, res - 1); ++cc) {
        dmin = fminf(dmin, d[(long long)r * res + cc]);
        empty = empty && id[(long long)r * res + cc] < 0;
      }
    vis = (dmin >= n[2] || empty) ? 1 : 0;
  }
  visible[(long long)job * n_tets + t] = vis;
}

// rast[job][f2t[face]] = 1 for every face id in the job's buffer
__global__ void rast_tets_kernel(const int* __restrict__ face_id, long long pixels, const int* __restrict__ job_mesh,
                                 const long long* __restrict__ f2t, const long long* __restrict__ face_off, int n_tets,
                                 unsigned char* __restrict__ rast) {
  const int job = blockIdx.y;
  const long long base = face_off[job_mesh[job]];
  const int* id = face_id + (long long)job * pixels;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pixels; i += (long long)gridDim.x * blockDim.x) {
    const int f = id[i];
    if (f >= 0) rast[(long long)job * n_tets + f2t[base + f]] = 1;
  }
}

// ---- shading ---------------------------------------------------------------------------------------------------------

constexpr int kShadeThreads = 256;
constexpr int kShadeJobChunk = 4096;  // jobs per launch (blockIdx.y)
constexpr int kSrgbLevels = 255;      // thresholds between the 256 output codes
constexpr float kNormalThreshold = 0.1f;  // NORMAL_THRESHOLD of nvdiffrec's renderutils (bsdf.py, normal.cu)

struct V3 { float x, y, z; };

__device__ __forceinline__ V3 v3_load(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ V3 v3_sub(V3 a, V3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
__device__ __forceinline__ V3 v3_neg(V3 a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ float v3_dot(V3 a, V3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ V3 v3_cross(V3 a, V3 b) {
  return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
          __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// x / sqrt(max(x . x, 1e-20)): nvdiffrec's safe_normalize
__device__ __forceinline__ V3 v3_safe_normalize(V3 a) {
  const float l = __fsqrt_rn(fmaxf(v3_dot(a, a), 1e-20f));
  return {__fdiv_rn(a.x, l), __fdiv_rn(a.y, l), __fdiv_rn(a.z, l)};
}
// (b0 a0 + b1 a1) + b2 a2
__device__ __forceinline__ V3 v3_interp(const float b[3], V3 a0, V3 a1, V3 a2) {
  return {__fadd_rn(__fadd_rn(__fmul_rn(b[0], a0.x), __fmul_rn(b[1], a1.x)), __fmul_rn(b[2], a2.x)),
          __fadd_rn(__fadd_rn(__fmul_rn(b[0], a0.y), __fmul_rn(b[1], a1.y)), __fmul_rn(b[2], a2.y)),
          __fadd_rn(__fadd_rn(__fmul_rn(b[0], a0.z), __fmul_rn(b[1], a1.z)), __fmul_rn(b[2], a2.z))};
}

// Linear RGB of face f at supersampled pixel centre (px, py); false when the face is not drawn (then the pixel is
// background, as it would be had the rasterizer not drawn it).
__device__ __forceinline__ bool shade_fragment(const float* __restrict__ v, const float* __restrict__ vn,
                                               const long long* __restrict__ f, const float* m, float fres, float px, float py,
                                               V3 cam, const float* sh, const float* kd, float col[3]) {
  Tri t;
  bool behind;
  if (!setup_tri(v, f, m, fres, t, behind)) return false;
  // barycentrics from the edge functions, then perspective-correct with each vertex's clip w
  const float e[3] = {edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], px, py), edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], px, py),
                      edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], px, py)};
  V3 p[3], n[3];
  float q[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    p[k] = v3_load(v + 3 * f[k]);
    n[k] = v3_load(vn + 3 * f[k]);
    q[k] = __fdiv_rn(__fdiv_rn(e[k], t.area), mvp_row(m + 12, p[k].x, p[k].y, p[k].z));
  }
  const float qs = __fadd_rn(__fadd_rn(q[0], q[1]), q[2]);
  const float b[3] = {__fdiv_rn(q[0], qs), __fdiv_rn(q[1], qs), __fdiv_rn(q[2], qs)};
  const V3 pos = v3_interp(b, p[0], p[1], p[2]);
  // bsdf_prepare_shading_normal: two-sided, no normal map, no tangents
  V3 smooth = v3_safe_normalize(v3_interp(b, n[0], n[1], n[2]));
  const V3 view = v3_safe_normalize(v3_sub(cam, pos));
  V3 geom = v3_safe_normalize(v3_cross(v3_sub(p[1], p[0]), v3_sub(p[2], p[0])));
  if (!(v3_dot(geom, view) > 0.f)) {
    smooth = v3_neg(smooth);
    geom = v3_neg(geom);
  }
  const float tb = fminf(fmaxf(__fdiv_rn(v3_dot(view, smooth), kNormalThreshold), 0.f), 1.f);
  const V3 s = v3_sub(smooth, geom);
  const float x = __fadd_rn(geom.x, __fmul_rn(tb, s.x)), y = __fadd_rn(geom.y, __fmul_rn(tb, s.y));
  const float z = __fadd_rn(geom.z, __fmul_rn(tb, s.z));
  // real SH basis, l <= 2, in the order Y00, Y1-1, Y10, Y11, Y2-2, Y2-1, Y20, Y21, Y22
  const float Y[9] = {0.28209479177387814f,
                      __fmul_rn(0.4886025119029199f, y),
                      __fmul_rn(0.4886025119029199f, z),
                      __fmul_rn(0.4886025119029199f, x),
                      __fmul_rn(__fmul_rn(1.0925484305920792f, x), y),
                      __fmul_rn(__fmul_rn(1.0925484305920792f, y), z),
                      __fmul_rn(0.31539156525252005f, __fsub_rn(__fmul_rn(3.f, __fmul_rn(z, z)), 1.f)),
                      __fmul_rn(__fmul_rn(1.0925484305920792f, x), z),
                      __fmul_rn(0.5462742152960396f, __fsub_rn(__fmul_rn(x, x), __fmul_rn(y, y)))};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float E = __fmul_rn(sh[c], Y[0]);
#pragma unroll
    for (int i = 1; i < 9; ++i) E = __fadd_rn(E, __fmul_rn(sh[3 * i + c], Y[i]));
    col[c] = __fmul_rn(kd[c], fmaxf(E, 0.f));
  }
  return true;
}

// One thread per (output pixel, job): shade the ssaa x ssaa sub-pixels, average them in row-major order, encode to sRGB.
__global__ void __launch_bounds__(kShadeThreads) shade_kernel(const float* __restrict__ verts, const float* __restrict__ v_nrm,
                                                              const long long* __restrict__ faces, const long long* __restrict__ vert_off,
                                                              const long long* __restrict__ face_off, const int* __restrict__ job_mesh,
                                                              const float* __restrict__ mvps, const float* __restrict__ campos, int job0,
                                                              int res, int ssaa, const int* __restrict__ face_id,
                                                              const float* __restrict__ sh_coef, const float* __restrict__ kd,
                                                              const float* __restrict__ bg, const float* __restrict__ thresholds,
                                                              unsigned char* __restrict__ rgb) {
  __shared__ float s_thr[kSrgbLevels], s_sh[27], s_kd[3], s_bg[3];
  for (int i = threadIdx.x; i < kSrgbLevels; i += blockDim.x) s_thr[i] = thresholds[i];
  if (threadIdx.x < 27) s_sh[threadIdx.x] = sh_coef[threadIdx.x];
  if (threadIdx.x < 3) {
    s_kd[threadIdx.x] = kd[threadIdx.x];
    s_bg[threadIdx.x] = bg[threadIdx.x];
  }
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)res * res) return;
  const int job = job0 + blockIdx.y;
  const int r = (int)(pix / res), c = (int)(pix % res);
  const int mesh = job_mesh[job];
  const long long* f = faces + 3 * face_off[mesh];
  const float* v = verts + 3 * vert_off[mesh];
  const float* vn = v_nrm + 3 * vert_off[mesh];
  float m[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) m[i] = mvps[16 * job + i];
  const V3 cam = v3_load(campos + 3 * job);
  const int sres = res * ssaa;
  const float fres = (float)sres;
  const int* id = face_id + (long long)job * sres * sres;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int a = 0; a < ssaa; ++a)
    for (int b = 0; b < ssaa; ++b) {
      const int sr = r * ssaa + a, sc = c * ssaa + b;
      const int fi = id[(long long)sr * sres + sc];
      float col[3];
      if (fi < 0 || !shade_fragment(v, vn, f + 3LL * fi, m, fres, (float)sc + 0.5f, (float)sr + 0.5f, cam, s_sh, s_kd, col)) {
        col[0] = s_bg[0];
        col[1] = s_bg[1];
        col[2] = s_bg[2];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k] = __fadd_rn(acc[k], col[k]);
    }
  const float n_sub = (float)(ssaa * ssaa);
  unsigned char* out = rgb + ((long long)job * res * res + pix) * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float x = __fdiv_rn(acc[k], n_sub);
    // the number of thresholds x reaches (the table is ascending; a NaN reaches none)
    int code = 0;
#pragma unroll
    for (int step = 128; step > 0; step >>= 1)
      if (code + step <= kSrgbLevels && x >= s_thr[code + step - 1]) code += step;
    out[k] = (unsigned char)code;
  }
}

int sm_count(int* n) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return fail("cannot query the device");
  return 0;
}

int check_sizes(const char* what, int n_jobs, int res) {
  if (n_jobs < 0 || n_jobs > 65535) return fail(std::string(what) + ": 0 to 65535 jobs per call");
  if (res < 1 || res > 16384) return fail(std::string(what) + ": resolution must be in [1, 16384]");
  return 0;
}

}  // namespace

extern "C" {

int mdb_raster_depth(const float* verts, const long long* faces, const long long* vert_off, const long long* face_off,
                     const int* job_mesh, const float* mvp, int n_jobs, int res, unsigned long long* scratch, float* depth,
                     int* face_id, int* n_behind, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_sizes("mdb_raster_depth", n_jobs, res)) return 1;
  if (n_jobs == 0) return 0;
  int sms = 0;
  if (sm_count(&sms)) return 1;
  const long long pixels = (long long)n_jobs * res * res;
  if (cudaMemsetAsync(scratch, 0xff, (size_t)pixels * sizeof(unsigned long long), s) != cudaSuccess ||
      cudaMemsetAsync(n_behind, 0, (size_t)n_jobs * sizeof(int), s) != cudaSuccess)
    return fail("mdb_raster_depth: cudaMemsetAsync failed");
  const int gx = std::min(1024, std::max(1, (8 * sms + n_jobs - 1) / n_jobs));
  raster_kernel<<<dim3((unsigned)gx, (unsigned)n_jobs), 32 * kRasterWarps, 0, s>>>(verts, faces, vert_off, face_off, job_mesh, mvp,
                                                                                   res, scratch, n_behind);
  if (check_launch("mdb_raster_depth")) return 1;
  const long long blocks = std::min<long long>((pixels + 255) / 256, 32LL * sms);
  resolve_kernel<<<(unsigned)blocks, 256, 0, s>>>(scratch, pixels, depth, face_id);
  return check_launch("mdb_raster_depth (resolve)");
}

int mdb_visible_tets(const float* pos, long long pos_stride, const int* tets, int n_tets, const long long* face_to_tet,
                     const long long* face_off, const int* job_mesh, const float* mvp, int n_jobs, int res, const float* depth,
                     const int* face_id, unsigned char* visible, unsigned char* rast, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_sizes("mdb_visible_tets", n_jobs, res)) return 1;
  if (n_tets < 0) return fail("mdb_visible_tets: negative tet count");
  if (n_jobs == 0 || n_tets == 0) return 0;
  int sms = 0;
  if (sm_count(&sms)) return 1;
  visible_tets_kernel<<<dim3((unsigned)((n_tets + 255) / 256), (unsigned)n_jobs), 256, 0, s>>>(pos, pos_stride, tets, n_tets, job_mesh, mvp,
                                                                                              res, depth, face_id, visible);
  if (check_launch("mdb_visible_tets")) return 1;
  if (cudaMemsetAsync(rast, 0, (size_t)n_jobs * n_tets, s) != cudaSuccess) return fail("mdb_visible_tets: cudaMemsetAsync failed");
  const long long pixels = (long long)res * res;
  const int gx = (int)std::min<long long>((pixels + 255) / 256, std::max(1, (8 * sms + n_jobs - 1) / n_jobs));
  rast_tets_kernel<<<dim3((unsigned)gx, (unsigned)n_jobs), 256, 0, s>>>(face_id, pixels, job_mesh, face_to_tet, face_off, n_tets, rast);
  return check_launch("mdb_visible_tets (rasterized tets)");
}

int mdb_render_shade(const float* verts, const float* v_nrm, const long long* faces, const long long* vert_off,
                     const long long* face_off, const int* job_mesh, const float* mvp, const float* campos, int n_jobs, int res,
                     int ssaa, const int* face_id, const float* sh_coef, const float* kd, const float* bg,
                     const float* srgb_thresholds, unsigned char* rgb, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (check_sizes("mdb_render_shade", n_jobs, res)) return 1;
  if (ssaa < 1 || ssaa > 4) return fail("mdb_render_shade: ssaa must be in [1, 4]");
  if ((long long)res * ssaa > 16384) return fail("mdb_render_shade: res * ssaa must be at most 16384");
  if (n_jobs == 0) return 0;
  const unsigned gx = (unsigned)(((long long)res * res + kShadeThreads - 1) / kShadeThreads);
  for (int j0 = 0; j0 < n_jobs; j0 += kShadeJobChunk) {
    const int nj = std::min(kShadeJobChunk, n_jobs - j0);
    shade_kernel<<<dim3(gx, (unsigned)nj), kShadeThreads, 0, s>>>(verts, v_nrm, faces, vert_off, face_off, job_mesh, mvp, campos, j0,
                                                                  res, ssaa, face_id, sh_coef, kd, bg, srgb_thresholds, rgb);
    if (check_launch("mdb_render_shade")) return 1;
  }
  return 0;
}

}  // extern "C"
