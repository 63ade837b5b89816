// Light field distance (Chen et al., "On Visual Similarity Based 3D Model Retrieval", Eurographics 2003) for
// `--mode=eval_metrics` (geometry/lfd.py). Two kernels:
// * mdb_lfd_descriptors: one CTA of 256 threads per silhouette (face_id >= 0 of an mdb_raster_depth pass). 35 Zernike
//   magnitudes (n <= 10) and 10 Fourier magnitudes of a 64-ray radial signature, quantized to 8 bits. Every fp32 and fp64
//   operation is rounded on its own, pixels are accumulated per thread in a fixed order and combined by a fixed tree, so
//   the float32 / fp64 numpy restatement (oracle/lfd_oracle.py) reproduces every byte.
// * mdb_lfd_matrix: one CTA per shape pair. The 100 x 100 table of view L1 distances (uint16, from __vsadu4 on 4-byte
//   words), then the 10 x 10 x 60 alignment sums as table lookups and a min. Exact integers: order-independent and
//   batch-invariant.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <cstdint>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(std::string(what) + ": " + cudaGetErrorString(e));
}

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxRes = 256;
constexpr int kMaskWords = kMaxRes * kMaxRes / 32;
constexpr int kZernike = 35;
constexpr int kZValues = 2 * kZernike;  // re, im
constexpr int kRedGroup = 14;           // accumulators combined per pass of the tree
static_assert(kZValues % kRedGroup == 0, "whole groups");
constexpr int kRays = 64;
constexpr int kRayPhases = kThreads / kRays;  // threads that share a ray, taking every kRayPhases-th sample
constexpr int kFourier = 10;
constexpr int kDescBytes = 48;
constexpr int kViews = 10;
constexpr int kShapeViews = 100;  // 10 light fields x 10 views
constexpr int kShapeBytes = kShapeViews * kDescBytes;
constexpr int kRotations = 60;
constexpr double kPi = 3.141592653589793;

// Term k of the descriptor has order n = zn(k) and m = zm(k) (n = 1 .. 10, m = n mod 2 .. n in steps of 2).
__host__ __device__ constexpr int zn(int k) {
  int n = 1;
  while (k >= n / 2 + 1) k -= n / 2 + 1, ++n;
  return n;
}
__host__ __device__ constexpr int zm(int k) {
  int n = 1;
  while (k >= n / 2 + 1) k -= n / 2 + 1, ++n;
  return n % 2 + 2 * k;
}
__host__ __device__ constexpr long long fact(int x) {
  long long r = 1;
  for (int i = 2; i <= x; ++i) r *= i;
  return r;
}
// P_nm(s) = R_n^m(rho) / rho^m is a polynomial in s = rho^2: its integer coefficient of s^j
__host__ __device__ constexpr float zcoef(int n, int m, int j) {
  const int k = (n - m) / 2 - j;
  return (float)((k % 2 ? -1 : 1) * (fact(n - k) / (fact(k) * fact((n + m) / 2 - k) * fact((n - m) / 2 - k))));
}
static_assert(zn(34) == 10 && zm(34) == 10 && zn(35) == 11, "35 terms up to n = 10");
static_assert(zcoef(10, 0, 5) == 252.f && zcoef(10, 0, 0) == -1.f && zcoef(4, 2, 0) == -3.f, "radial polynomials");

// Horner from the highest power: poly = fl(fl(poly s) + c_j) for j = J .. 0
template <int N, int M, int J>
__device__ __forceinline__ float horner(float poly, float s) {
  if constexpr (J < 0) {
    return poly;
  } else {
    constexpr float c = zcoef(N, M, J);
    return horner<N, M, J - 1>(__fadd_rn(__fmul_rn(poly, s), c), s);
  }
}

// acc[2k], acc[2k + 1] += P_nm(s) z^m for terms K .. 34
template <int K>
__device__ __forceinline__ void zernike_add(double* acc, float s, const float* zr, const float* zi) {
  if constexpr (K < kZernike) {
    constexpr int n = zn(K), m = zm(K), d = (n - m) / 2;
    constexpr float top = zcoef(n, m, d);
    const float poly = horner<n, m, d - 1>(top, s);
    acc[2 * K] = __dadd_rn(acc[2 * K], (double)__fmul_rn(poly, zr[m]));
    acc[2 * K + 1] = __dadd_rn(acc[2 * K + 1], (double)__fmul_rn(poly, zi[m]));
    zernike_add<K + 1>(acc, s, zr, zi);
  }
}

__device__ __forceinline__ unsigned char quantize(double v, double scale) {
  return (unsigned char)fmin(255.0, floor(__dadd_rn(__dmul_rn(v, scale), 0.5)));
}

__device__ __forceinline__ bool inside(const unsigned* mask, int p) { return (mask[p >> 5] >> (p & 31)) & 1u; }

// One CTA per image. Pixel p (row-major) belongs to thread p mod 256, which visits its pixels in increasing order.
__global__ void __launch_bounds__(kThreads) lfd_descriptor_kernel(const int* __restrict__ face_id, int res,
                                                                  const float* __restrict__ ray_cs, const double* __restrict__ dft,
                                                                  unsigned char* __restrict__ desc, int* __restrict__ n_inside) {
  __shared__ unsigned s_mask[kMaskWords];
  __shared__ double s_red[kRedGroup * kThreads];
  __shared__ double s_z[kZValues];
  __shared__ double s_fmag[kFourier + 1];
  __shared__ long long s_n[kWarps], s_sx[kWarps], s_sy[kWarps];
  __shared__ int s_last[kRays];
  __shared__ unsigned s_r2;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long img = blockIdx.x;
  const int P = res * res;
  const int* id = face_id + img * P;
  unsigned char* out = desc + img * kDescBytes;
  if (t < kRays) s_last[t] = -1;
  if (t == 0) s_r2 = 0u;

  // 1. inside mask (one ballot word per warp and pass), pixel count and exact sums of 2c + 1 and 2r + 1
  long long n = 0, sx = 0, sy = 0;
  for (int base = 0; base < P; base += kThreads) {
    const int p = base + t;
    const bool in = p < P && id[p] >= 0;
    const unsigned word = __ballot_sync(0xffffffffu, in);
    if (lane == 0) s_mask[(base >> 5) + warp] = word;
    if (in) {
      n += 1;
      sx += 2 * (p % res) + 1;
      sy += 2 * (p / res) + 1;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n += __shfl_down_sync(0xffffffffu, n, o);
    sx += __shfl_down_sync(0xffffffffu, sx, o);
    sy += __shfl_down_sync(0xffffffffu, sy, o);
  }
  if (lane == 0) {
    s_n[warp] = n;
    s_sx[warp] = sx;
    s_sy[warp] = sy;
  }
  __syncthreads();
  n = sx = sy = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    n += s_n[w];
    sx += s_sx[w];
    sy += s_sy[w];
  }
  if (t == 0) n_inside[img] = (int)n;
  if (n == 0) {
    if (t < kDescBytes) out[t] = 0;
    return;
  }
  const double two_n = (double)(2 * n);
  const float cx = __double2float_rn(__ddiv_rn((double)sx, two_n)), cy = __double2float_rn(__ddiv_rn((double)sy, two_n));

  // 2. radius: the largest centre distance, plus half a pixel
  float r2 = 0.f;
  for (int p = t; p < P; p += kThreads)
    if (inside(s_mask, p)) {
      const float dx = __fsub_rn((float)(p % res) + 0.5f, cx), dy = __fsub_rn((float)(p / res) + 0.5f, cy);
      r2 = fmaxf(r2, __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    }
  atomicMax(&s_r2, __float_as_uint(r2));  // non-negative floats order as their bits
  __syncthreads();
  const float rad = __fadd_rn(__fsqrt_rn(__uint_as_float(s_r2)), 0.5f);

  // 3. Zernike sums: V*_nm = P_nm(s) (u - i w)^m per inside pixel, fp32 products added into fp64 in pixel order
  double acc[kZValues];
#pragma unroll
  for (int k = 0; k < kZValues; ++k) acc[k] = 0.0;
  for (int p = t; p < P; p += kThreads) {
    if (!inside(s_mask, p)) continue;
    const float dx = __fsub_rn((float)(p % res) + 0.5f, cx), dy = __fsub_rn((float)(p / res) + 0.5f, cy);
    const float u = __fdiv_rn(dx, rad), w = __fdiv_rn(dy, rad);
    const float s = __fadd_rn(__fmul_rn(u, u), __fmul_rn(w, w));
    float zr[11], zi[11];
    zr[0] = 1.f;
    zi[0] = 0.f;
#pragma unroll
    for (int m = 1; m <= 10; ++m) {  // z^m = z^(m-1) * (u, -w)
      zr[m] = __fsub_rn(__fmul_rn(zr[m - 1], u), __fmul_rn(zi[m - 1], -w));
      zi[m] = __fadd_rn(__fmul_rn(zr[m - 1], -w), __fmul_rn(zi[m - 1], u));
    }
    zernike_add<0>(acc, s, zr, zi);
  }
  // part[t] += part[t + s] for s = 128, 64, ..., 1, kRedGroup accumulators at a time
#pragma unroll
  for (int g0 = 0; g0 < kZValues; g0 += kRedGroup) {
#pragma unroll
    for (int g = 0; g < kRedGroup; ++g) s_red[g * kThreads + t] = acc[g0 + g];
    __syncthreads();
    for (int st = kThreads / 2; st > 0; st >>= 1) {
      for (int i = t; i < kRedGroup * st; i += kThreads) {
        const int g = i / st, k = i % st;
        s_red[g * kThreads + k] = __dadd_rn(s_red[g * kThreads + k], s_red[g * kThreads + k + st]);
      }
      __syncthreads();
    }
    if (t < kRedGroup) s_z[g0 + t] = s_red[t * kThreads];
    __syncthreads();
  }

  // 4. radial signature: the last sample j of each ray (at cx + 0.5 j cos, cy + 0.5 j sin) whose pixel is inside
  {
    const int k = t % kRays;
    const float c = ray_cs[2 * k], sn = ray_cs[2 * k + 1], fres = (float)res;
    int last = -1;
    for (int j = t / kRays;; j += kRayPhases) {
      const float h = __fmul_rn(0.5f, (float)j);
      const float x = __fadd_rn(cx, __fmul_rn(h, c)), y = __fadd_rn(cy, __fmul_rn(h, sn));
      if (!(x >= 0.f && x < fres && y >= 0.f && y < fres)) break;  // monotone in j: the ray does not come back
      if (inside(s_mask, (int)floorf(y) * res + (int)floorf(x))) last = j;
    }
    atomicMax(&s_last[k], last);
  }
  __syncthreads();
  if (t <= kFourier) {
    double re = 0.0, im = 0.0;
    for (int k = 0; k < kRays; ++k) {
      const double rk = s_last[k] > 0 ? __dmul_rn(0.5, (double)s_last[k]) : 0.0;
      re = __dadd_rn(re, __dmul_rn(rk, dft[2 * (t * kRays + k)]));
      im = __dsub_rn(im, __dmul_rn(rk, dft[2 * (t * kRays + k) + 1]));
    }
    s_fmag[t] = __dsqrt_rn(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));
  }
  __syncthreads();

  // 5. the 48 bytes
  if (t < kZernike) {
    const double re = s_z[2 * t], im = s_z[2 * t + 1];
    const double mag = __dmul_rn((double)(zn(t) + 1), __dsqrt_rn(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im))));
    out[t] = quantize(__ddiv_rn(mag, __dmul_rn(__dmul_rn(kPi, (double)rad), (double)rad)), 256.0);
  } else if (t < kZernike + kFourier) {
    const double f0 = s_fmag[0];
    out[t] = f0 > 0.0 ? quantize(__ddiv_rn(s_fmag[t - kZernike + 1], f0), 512.0) : (unsigned char)0;
  } else if (t < kDescBytes) {
    out[t] = 0;
  }
}

// One CTA per (A shape i, B shape j). B == A (self): only i < j, mirrored; the diagonal is 0.
__global__ void __launch_bounds__(kThreads) lfd_matrix_kernel(const unsigned char* __restrict__ A, const unsigned char* __restrict__ B,
                                                              int nB, const signed char* __restrict__ perms, int self,
                                                              int* __restrict__ out) {
  __shared__ uint4 s_a[kShapeBytes / 16], s_b[kShapeBytes / 16];
  __shared__ unsigned short s_d[kShapeViews * kShapeViews];
  __shared__ unsigned char s_p[kRotations * kViews];
  __shared__ int s_min[kWarps];
  const int i = blockIdx.y, j = blockIdx.x, t = threadIdx.x;
  if (self && j <= i) {
    if (j == i && t == 0) out[(long long)i * nB + i] = 0;
    return;
  }
  const uint4* a4 = reinterpret_cast<const uint4*>(A + (long long)i * kShapeBytes);
  const uint4* b4 = reinterpret_cast<const uint4*>(B + (long long)j * kShapeBytes);
  for (int k = t; k < kShapeBytes / 16; k += kThreads) {
    s_a[k] = a4[k];
    s_b[k] = b4[k];
  }
  for (int k = t; k < kRotations * kViews; k += kThreads) s_p[k] = (unsigned char)min((int)(unsigned char)perms[k], kViews - 1);
  __syncthreads();

  // view distance table: thread (ag, bg) owns A views 4 ag .. 4 ag + 3 against B views 10 bg .. 10 bg + 9
  if (t < 250) {
    const int ag = t / 10, bg = t % 10;
    uint4 a[4][3];
#pragma unroll
    for (int v = 0; v < 4; ++v)
#pragma unroll
      for (int q = 0; q < 3; ++q) a[v][q] = s_a[(4 * ag + v) * 3 + q];
#pragma unroll 2
    for (int bv = 0; bv < 10; ++bv) {
      const int b = 10 * bg + bv;
      const uint4 b0 = s_b[b * 3], b1 = s_b[b * 3 + 1], b2 = s_b[b * 3 + 2];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        unsigned d = __vsadu4(a[v][0].x, b0.x) + __vsadu4(a[v][0].y, b0.y) + __vsadu4(a[v][0].z, b0.z) + __vsadu4(a[v][0].w, b0.w);
        d += __vsadu4(a[v][1].x, b1.x) + __vsadu4(a[v][1].y, b1.y) + __vsadu4(a[v][1].z, b1.z) + __vsadu4(a[v][1].w, b1.w);
        d += __vsadu4(a[v][2].x, b2.x) + __vsadu4(a[v][2].y, b2.y) + __vsadu4(a[v][2].z, b2.z) + __vsadu4(a[v][2].w, b2.w);
        s_d[(4 * ag + v) * kShapeViews + b] = (unsigned short)d;
      }
    }
  }
  __syncthreads();

  // alignments (light field s of A, light field u of B, rotation g): sum over i of d(A[s][i], B[u][pi_g(i)])
  int best = 0x7fffffff;
  for (int k = t; k < kViews * kViews * kRotations; k += kThreads) {
    const int g = k % kRotations, su = k / kRotations;
    const unsigned short* row = s_d + (su / kViews) * kViews * kShapeViews + (su % kViews) * kViews;
    const unsigned char* p = s_p + g * kViews;
    int sum = 0;
#pragma unroll
    for (int v = 0; v < kViews; ++v) sum += row[v * kShapeViews + p[v]];
    best = min(best, sum);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_down_sync(0xffffffffu, best, o));
  if ((t & 31) == 0) s_min[t >> 5] = best;
  __syncthreads();
  if (t == 0) {
#pragma unroll
    for (int w = 1; w < kWarps; ++w) best = min(best, s_min[w]);
    out[(long long)i * nB + j] = best;
    if (self) out[(long long)j * nB + i] = best;
  }
}

}  // namespace

extern "C" {

int mdb_lfd_descriptors(const int* face_id, int n_images, int res, const float* ray_cs, const double* dft,
                        unsigned char* desc, int* n_inside, void* stream) {
  if (n_images < 0) return fail("mdb_lfd_descriptors: negative image count");
  if (res < 1 || res > kMaxRes) return fail("mdb_lfd_descriptors: res must be in [1, 256]");
  if (n_images == 0) return 0;
  if (!face_id || !ray_cs || !dft || !desc || !n_inside) return fail("mdb_lfd_descriptors: null pointer");
  lfd_descriptor_kernel<<<(unsigned)n_images, kThreads, 0, (cudaStream_t)stream>>>(face_id, res, ray_cs, dft, desc, n_inside);
  return check_launch("mdb_lfd_descriptors");
}

int mdb_lfd_matrix(const unsigned char* A, int nA, const unsigned char* B, int nB, const signed char* perms, int* out,
                   void* stream) {
  const bool self = B == nullptr;
  if (self) nB = nA;
  if (nA < 0 || nA > 65535 || nB < 0 || nB > 65535) return fail("mdb_lfd_matrix: shape counts must be in [0, 65535]");
  if (nA == 0 || nB == 0) return 0;
  if (!A || !perms || !out) return fail("mdb_lfd_matrix: null pointer");
  if (reinterpret_cast<uintptr_t>(A) % 16 || reinterpret_cast<uintptr_t>(B) % 16)
    return fail("mdb_lfd_matrix: descriptor sets must be 16-byte aligned");
  lfd_matrix_kernel<<<dim3((unsigned)nB, (unsigned)nA), kThreads, 0, (cudaStream_t)stream>>>(A, self ? A : B, nB, perms, self ? 1 : 0,
                                                                                            out);
  return check_launch("mdb_lfd_matrix");
}

}  // extern "C"
