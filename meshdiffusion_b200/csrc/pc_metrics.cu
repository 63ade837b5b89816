// Point-cloud metrics of generated shapes (no reference counterpart: the reference's fitting code calls kaolin's
// sample_points / chamfer_distance, nvdiffrec/lib/geometry/dmtet.py:455-457, and ships no evaluation code).
//
// * mdb_mesh_sample_points: area-weighted surface sampling of a packed batch of marching-tet meshes. Face areas and their
//   per-mesh inclusive prefix sum are fp64 in face order (the same sums as np.cumsum), so the face a uniform selects is
//   the one a host restatement selects.
// * mdb_chamfer_matrix: all-pairs Chamfer distance CD(X,Y) = mean_x min_y d + mean_y min_x d, d the squared Euclidean
//   distance in fp32 on the CUDA cores. One CTA per cloud pair computes both directions in one pass; the minima are exact,
//   so the result is bitwise reproducible, batch-invariant and symmetric in (X, Y).
// * mdb_chamfer_pairs: the same distance over a list of (a, b) pairs of one cloud set (shape completion's block-diagonal
//   pairs), with the a->b half and the largest a->b minimum (the squared one-sided Hausdorff distance). Both kernels run
//   the same device function for the minima and the same fixed-order sums, so a listed pair's CD is bitwise its matrix
//   entry.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <curand_kernel.h>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(std::string(what) + ": " + cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------------------------
// Surface sampling

// 0.5 |(b - a) x (c - a)| in fp64 from fp32 corners, without contraction: bitwise what the numpy restatement computes.
__device__ __forceinline__ double face_area(const float* __restrict__ v, const long long* __restrict__ f) {
  const long long i0 = f[0], i1 = f[1], i2 = f[2];
  const double ax = v[3 * i0], ay = v[3 * i0 + 1], az = v[3 * i0 + 2];
  const double e1x = __dsub_rn(v[3 * i1], ax), e1y = __dsub_rn(v[3 * i1 + 1], ay), e1z = __dsub_rn(v[3 * i1 + 2], az);
  const double e2x = __dsub_rn(v[3 * i2], ax), e2y = __dsub_rn(v[3 * i2 + 1], ay), e2z = __dsub_rn(v[3 * i2 + 2], az);
  const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz));
  return 0.5 * __dsqrt_rn(n2);
}

// One warp per mesh: lanes compute 32 consecutive areas, then every lane runs the same sequential fp64 sum over them
// (the face-order sum np.cumsum does) and keeps the value at its own position.
constexpr int kCdfWarps = 4;
__global__ void __launch_bounds__(32 * kCdfWarps) face_cdf_kernel(const float* __restrict__ verts, const long long* __restrict__ faces,
                                                                  const long long* __restrict__ vert_off,
                                                                  const long long* __restrict__ face_off, int n_meshes,
                                                                  double* __restrict__ cdf) {
  const int b = blockIdx.x * kCdfWarps + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= n_meshes) return;
  const long long f0 = face_off[b], f1 = face_off[b + 1];
  const float* v = verts + 3 * vert_off[b];
  double run = 0.0;
  for (long long base = f0; base < f1; base += 32) {
    const long long f = base + lane;
    const double a = f < f1 ? face_area(v, faces + 3 * f) : 0.0;  // +0.0 past the end leaves the running sum unchanged
    double mine = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      run = __dadd_rn(run, __shfl_sync(0xffffffffu, a, i));
      if (i == lane) mine = run;
    }
    if (f < f1) cdf[f] = mine;
  }
}

__global__ void sample_points_kernel(const float* __restrict__ verts, const long long* __restrict__ faces,
                                     const long long* __restrict__ vert_off, const long long* __restrict__ face_off,
                                     const double* __restrict__ cdf, int n_points, const float* __restrict__ uniforms,
                                     unsigned long long seed, long long first_id, float* __restrict__ points, int* __restrict__ n_written) {
  const int b = blockIdx.y;
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long f0 = face_off[b], f1 = face_off[b + 1];
  const double total = f1 > f0 ? cdf[f1 - 1] : 0.0;
  const bool empty = !(total > 0.0);  // no faces, zero total area (or a non-finite one): nothing to sample from
  if (j == 0) n_written[b] = empty ? 0 : n_points;
  if (empty || j >= n_points) return;
  const long long row = (long long)b * n_points + j;
  float u, r1, r2;
  if (uniforms) {
    u = uniforms[3 * row]; r1 = uniforms[3 * row + 1]; r2 = uniforms[3 * row + 2];
  } else {
    // the key depends on the mesh's own id and the point index only, never on the batch the mesh was launched in
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)(first_id + b) * (unsigned long long)n_points + (unsigned long long)j, 0, &st);
    const uint4 r = curand4(&st);
    u = (float)(r.x >> 8) * 0x1p-24f;  // 24 random bits: exactly representable, in [0, 1)
    r1 = (float)(r.y >> 8) * 0x1p-24f;
    r2 = (float)(r.z >> 8) * 0x1p-24f;
  }
  // smallest k with cdf[k] > u * total; it exists because u < 1 and cdf[f1 - 1] = total > 0
  const double t = (double)u * total;
  long long lo = f0, hi = f1 - 1;
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (cdf[mid] > t) hi = mid; else lo = mid + 1;
  }
  const float* v = verts + 3 * vert_off[b];
  const long long* f = faces + 3 * lo;
  const float* pa = v + 3 * f[0];
  const float* pb = v + 3 * f[1];
  const float* pc = v + 3 * f[2];
  const float s = sqrtf(r1);
  const float wa = 1.0f - s, wb = s * (1.0f - r2), wc = s * r2;
  float* out = points + 3 * row;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = wa * pa[c] + wb * pb[c] + wc * pc[c];
}

// ------------------------------------------------------------------------------------------------------------------
// Chamfer matrix
//
// CTA = 8 warps; a warp is 8 x-lanes x 4 y-lanes. A thread holds kTX x points in registers and, per step, kTY y points
// read from the shared-memory y tile: kTX * kTY distances of 8 FP32-pipe instructions each (3 FADD, 1 FMUL, 2 FFMA,
// 2 FMNMX). Row minima stay in registers over the whole y range of an x chunk and are reduced over the 4 y-lanes at its
// end. Column minima are reduced over the 8 x-lanes by shuffles after every step and merged across warps and x chunks by
// an integer atomicMin on the float bits in shared memory (exact for non-negative floats). Padded points are NaN:
// fminf ignores NaN, so they never win a minimum.
constexpr int kCdThreads = 256, kXL = 8, kYL = 4, kTX = 16, kTY = 4;
constexpr int kXChunk = (kCdThreads / 32) * kXL * kTX;  // 1024 x points per pass
constexpr int kYStep = kYL * kTY;                        // 16 y points per warp step
constexpr int kYTile = 512;                              // y points per shared-memory tile
static_assert(kXL * kYL == 32 && kYTile % kYStep == 0, "warp layout");

__host__ __device__ constexpr long long round_up(long long n, long long m) { return (n + m - 1) / m * m; }

size_t chamfer_smem_bytes(int N, int M) {
  return (size_t)kYTile * sizeof(float4) + (size_t)kCdThreads * sizeof(double) +
         (size_t)(round_up(N, kXChunk) + round_up(M, kYTile)) * sizeof(float);
}

// Sum of v[0..n) in fp64, in an order that depends on n alone: thread t sums t, t + 256, ... sequentially, then a fixed
// halving tree. Both directions go through it, so CD(X, Y) and CD(Y, X) add the same numbers in the same order.
__device__ double fixed_order_sum(const float* v, int n, double* red) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kCdThreads) s += (double)v[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = kCdThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// Row minima of X (min over y of d) -> rowmin[0..N), column minima (min over x of d) -> colmin[0..M), both in shared
// memory (laid out by chamfer_smem_bytes), then a barrier. Every CTA of both kernels runs exactly this code, so a pair's
// minima do not depend on which kernel or launch computed them.
__device__ __forceinline__ void chamfer_minima(const float* __restrict__ X, int N, const float* __restrict__ Y, int M,
                                               float4* ytile, float* rowmin, float* colmin) {
  unsigned* colbits = reinterpret_cast<unsigned*>(colmin);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, xl = lane % kXL, yl = lane / kXL;
  const float kNaN = __int_as_float(0x7fc00000), kInf = __int_as_float(0x7f800000);
  const int Mt = (int)round_up(M, kYTile);
  for (int k = threadIdx.x; k < Mt; k += kCdThreads) colbits[k] = 0x7f800000u;

  for (int x0 = 0; x0 < N; x0 += kXChunk) {
    float px[kTX], py[kTX], pz[kTX], rmin[kTX];
#pragma unroll
    for (int k = 0; k < kTX; ++k) {
      const int x = x0 + k * (kCdThreads / 32) * kXL + warp * kXL + xl;
      const bool in = x < N;
      px[k] = in ? X[3LL * x] : kNaN;
      py[k] = in ? X[3LL * x + 1] : kNaN;
      pz[k] = in ? X[3LL * x + 2] : kNaN;
      rmin[k] = kInf;
    }
    for (int y0 = 0; y0 < M; y0 += kYTile) {
      __syncthreads();  // the previous tile is no longer read (and colmin is initialised)
      for (int k = threadIdx.x; k < kYTile; k += kCdThreads) {
        const int y = y0 + k;
        ytile[k] = y < M ? make_float4(Y[3LL * y], Y[3LL * y + 1], Y[3LL * y + 2], 0.f) : make_float4(kNaN, kNaN, kNaN, 0.f);
      }
      __syncthreads();
      const int steps = (int)(min(kYTile, (int)round_up(M - y0, kYStep)) / kYStep);
      for (int s = 0; s < steps; ++s) {
        float4 q[kTY];
        float cmin[kTY];
#pragma unroll
        for (int t = 0; t < kTY; ++t) { q[t] = ytile[s * kYStep + t * kYL + yl]; cmin[t] = kInf; }
#pragma unroll
        for (int k = 0; k < kTX; ++k) {
#pragma unroll
          for (int t = 0; t < kTY; ++t) {
            const float dx = px[k] - q[t].x, dy = py[k] - q[t].y, dz = pz[k] - q[t].z;
            const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            rmin[k] = fminf(rmin[k], d);
            cmin[t] = fminf(cmin[t], d);
          }
        }
#pragma unroll
        for (int t = 0; t < kTY; ++t) {
          float c = cmin[t];
          c = fminf(c, __shfl_xor_sync(0xffffffffu, c, 1));
          c = fminf(c, __shfl_xor_sync(0xffffffffu, c, 2));
          c = fminf(c, __shfl_xor_sync(0xffffffffu, c, 4));
          if (xl == t) atomicMin(colbits + y0 + s * kYStep + t * kYL + yl, __float_as_uint(c));
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kTX; ++k) {
      float r = rmin[k];
      r = fminf(r, __shfl_xor_sync(0xffffffffu, r, 8));
      r = fminf(r, __shfl_xor_sync(0xffffffffu, r, 16));
      const int x = x0 + k * (kCdThreads / 32) * kXL + warp * kXL + xl;
      if (yl == 0 && x < N) rowmin[x] = r;
    }
  }
  __syncthreads();
}

// The shared-memory regions of chamfer_smem_bytes.
struct ChamferSmem {
  float4* ytile;
  double* red;
  float* rowmin;
  float* colmin;
  __device__ ChamferSmem(unsigned char* smem, int N) {
    ytile = reinterpret_cast<float4*>(smem);
    red = reinterpret_cast<double*>(ytile + kYTile);
    rowmin = reinterpret_cast<float*>(red + kCdThreads);
    colmin = rowmin + round_up(N, kXChunk);
  }
};

__global__ void __launch_bounds__(kCdThreads, 2) chamfer_pair_kernel(const float* __restrict__ A, int N, const float* __restrict__ B,
                                                                    int M, int nB, int self, double* __restrict__ out) {
  const int i = blockIdx.y, j = blockIdx.x;
  if (self && j < i) return;  // the mirror of (j, i)
  if (self && j == i) {
    if (threadIdx.x == 0) out[(long long)i * nB + j] = 0.0;
    return;
  }
  extern __shared__ __align__(16) unsigned char smem[];
  const ChamferSmem sm(smem, N);
  chamfer_minima(A + (long long)i * N * 3, N, B + (long long)j * M * 3, M, sm.ytile, sm.rowmin, sm.colmin);
  const double sx = fixed_order_sum(sm.rowmin, N, sm.red);
  const double sy = fixed_order_sum(sm.colmin, M, sm.red);
  if (threadIdx.x == 0) {
    const double cd = sx / (double)N + sy / (double)M;
    out[(long long)i * nB + j] = cd;
    if (self) out[(long long)j * nB + i] = cd;
  }
}

// Max of v[0..n) (non-negative floats; exact in any order). Thread-strided, then the same halving tree as fixed_order_sum.
__device__ float block_max(const float* v, int n, double* red) {
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += kCdThreads) m = fmaxf(m, v[i]);
  red[threadIdx.x] = (double)m;
  __syncthreads();
  for (int h = kCdThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  const float r = (float)red[0];
  __syncthreads();
  return r;
}

// One CTA per listed pair (a, b) of clouds of one size N: the matrix kernel's minima and sums, plus the largest row minimum.
// A pair the host would refuse (a == b, an index out of range) gets NaN in all three outputs rather than a stray read.
__global__ void __launch_bounds__(kCdThreads, 2) chamfer_list_kernel(const float* __restrict__ clouds, int n_clouds, int N,
                                                                    const int* __restrict__ pairs, double* __restrict__ cd,
                                                                    double* __restrict__ mean_ab, float* __restrict__ max_ab) {
  const int p = blockIdx.x;
  const int a = pairs[2 * p], b = pairs[2 * p + 1];
  if (a == b || a < 0 || b < 0 || a >= n_clouds || b >= n_clouds) {
    if (threadIdx.x == 0) {
      cd[p] = mean_ab[p] = __longlong_as_double(0x7ff8000000000000LL);
      max_ab[p] = __int_as_float(0x7fc00000);
    }
    return;
  }
  extern __shared__ __align__(16) unsigned char smem[];
  const ChamferSmem sm(smem, N);
  chamfer_minima(clouds + (long long)a * N * 3, N, clouds + (long long)b * N * 3, N, sm.ytile, sm.rowmin, sm.colmin);
  const double sx = fixed_order_sum(sm.rowmin, N, sm.red);
  const double sy = fixed_order_sum(sm.colmin, N, sm.red);
  const float mx = block_max(sm.rowmin, N, sm.red);
  if (threadIdx.x == 0) {
    cd[p] = sx / (double)N + sy / (double)N;
    mean_ab[p] = sx / (double)N;
    max_ab[p] = mx;
  }
}

}  // namespace

extern "C" {

int mdb_mesh_sample_points(const float* verts, const long long* faces, const long long* vert_off, const long long* face_off,
                           int n_meshes, int n_points, const float* uniforms, unsigned long long seed, long long first_id,
                           double* cdf, float* points, int* n_written, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n_meshes < 0 || n_points < 0 || first_id < 0) return fail("mdb_mesh_sample_points: negative size or id");
  if (n_meshes > 65535) return fail("mdb_mesh_sample_points: at most 65535 meshes per call");
  if (n_meshes == 0) return 0;
  face_cdf_kernel<<<(n_meshes + kCdfWarps - 1) / kCdfWarps, 32 * kCdfWarps, 0, s>>>(verts, faces, vert_off, face_off, n_meshes, cdf);
  const dim3 grid((unsigned)((n_points + 255) / 256 > 0 ? (n_points + 255) / 256 : 1), (unsigned)n_meshes);
  sample_points_kernel<<<grid, 256, 0, s>>>(verts, faces, vert_off, face_off, cdf, n_points, uniforms, seed, first_id, points, n_written);
  return check_launch("mdb_mesh_sample_points");
}

int mdb_chamfer_matrix(const float* A, int nA, int N, const float* B, int nB, int M, double* out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int self = B == nullptr;
  if (self) { B = A; nB = nA; M = N; }
  if (nA < 0 || nB < 0) return fail("mdb_chamfer_matrix: negative cloud count");
  if (N < 1 || M < 1) return fail("mdb_chamfer_matrix: every cloud needs at least one point");
  if (nA > 65535) return fail("mdb_chamfer_matrix: at most 65535 clouds in A");
  if (nA == 0 || nB == 0) return 0;
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return fail("mdb_chamfer_matrix: cannot query the device");
  const size_t smem = chamfer_smem_bytes(N, M);
  if (smem > (size_t)optin)
    return fail("mdb_chamfer_matrix: the per-point minima of N + M = " + std::to_string((long long)N + M) +
                " points do not fit in shared memory");
  if (cudaFuncSetAttribute(chamfer_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("mdb_chamfer_matrix: cudaFuncSetAttribute failed");
  chamfer_pair_kernel<<<dim3((unsigned)nB, (unsigned)nA), kCdThreads, smem, s>>>(A, N, B, M, nB, self, out);
  return check_launch("mdb_chamfer_matrix");
}

int mdb_chamfer_pairs(const float* clouds, int n_clouds, int N, const int* pairs, int P, double* cd, double* mean_ab,
                      float* max_ab, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n_clouds < 2) return fail("mdb_chamfer_pairs: a pair needs two distinct clouds, got n_clouds = " + std::to_string(n_clouds));
  if (N < 1) return fail("mdb_chamfer_pairs: every cloud needs at least one point");
  if (P < 0) return fail("mdb_chamfer_pairs: negative pair count");
  if (P == 0) return 0;
  if (!clouds || !pairs || !cd || !mean_ab || !max_ab) return fail("mdb_chamfer_pairs: null pointer");
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return fail("mdb_chamfer_pairs: cannot query the device");
  const size_t smem = chamfer_smem_bytes(N, N);
  if (smem > (size_t)optin)
    return fail("mdb_chamfer_pairs: the per-point minima of 2N = " + std::to_string(2LL * N) +
                " points do not fit in shared memory");
  if (cudaFuncSetAttribute(chamfer_list_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("mdb_chamfer_pairs: cudaFuncSetAttribute failed");
  chamfer_list_kernel<<<(unsigned)P, kCdThreads, smem, s>>>(clouds, n_clouds, N, pairs, cd, mean_ab, max_ab);
  return check_launch("mdb_chamfer_pairs");
}

}  // extern "C"
