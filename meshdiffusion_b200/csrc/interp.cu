// Spherical interpolation of endpoint pairs for `--mode=uncond_gen_interp` (diffusion/interp.py), over the whole tensor
// with no grid mask, as the reference's `slerp` (lib/diffusion/evaler.py:63-71) does. Three launches per call:
//   1. fp64 partial sums of a.b, a.a, b.b: pair p is cut into kChunks contiguous ranges whatever the pair count, each
//      reduced by a fixed-shape block tree (the pattern of likelihood.cu), so the sums are bitwise reproducible and a
//      pair's sums do not depend on the launch it shares;
//   2. one block per pair sums its chunk partials in a fixed tree and computes the weights of every frame in fp64;
//   3. one thread per 16-byte vector (or per element when rows are not 16-byte aligned) reads a and b once and writes all
//      frames as fl(fl(w_a a) + fl(w_b b)).
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <cmath>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }

constexpr int kThreads = 256;   // phase 1 and 3 block size
constexpr int kChunks = 1024;   // reduction chunks per pair
constexpr int kFinish = 256;    // phase 2 block size: each thread folds kChunks / kFinish partials in order
constexpr int kAlphas = 128;    // frames whose weights one phase-2 launch computes
static_assert(kChunks % kFinish == 0, "phase 2 folds whole rows of partials");

struct Alphas { double v[kAlphas]; };

// fixed-order sum of one double over the block (shuffle tree, then the warps' results in warp order); thread 0 has it
template <int NT>
__device__ double block_sum(double v, double* red) {
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < NT / 32; ++i) t += red[i];
  __syncthreads();
  return t;
}

// grid (kChunks, pairs): block j of pair p owns elements [j*chunk, (j+1)*chunk) of a[p] and b[p]
__global__ void __launch_bounds__(kThreads) slerp_dots_kernel(const float* __restrict__ za, const float* __restrict__ zb,
                                                              long long n, long long chunk, double* __restrict__ partial) {
  __shared__ double red[kThreads / 32];
  const int p = blockIdx.y;
  const long long e0 = (long long)blockIdx.x * chunk;
  const long long e1 = e0 + chunk < n ? e0 + chunk : n;
  const float* a = za + (long long)p * n;
  const float* b = zb + (long long)p * n;
  double ab = 0.0, aa = 0.0, bb = 0.0;
  for (long long e = e0 + threadIdx.x; e < e1; e += kThreads) {
    const double av = (double)__ldg(a + e), bv = (double)__ldg(b + e);
    ab += av * bv;
    aa += av * av;
    bb += bv * bv;
  }
  ab = block_sum<kThreads>(ab, red);
  aa = block_sum<kThreads>(aa, red);
  bb = block_sum<kThreads>(bb, red);
  if (threadIdx.x == 0) {
    double* out = partial + ((long long)p * kChunks + blockIdx.x) * 3;
    out[0] = ab;
    out[1] = aa;
    out[2] = bb;
  }
}

// grid (pairs), kFinish threads: the pair's sums, then the weights of frames f0 .. f0 + count - 1
__global__ void __launch_bounds__(kFinish) slerp_coef_kernel(const double* __restrict__ partial, Alphas alphas, int f0, int count,
                                                             int frames, double* __restrict__ sums, float* __restrict__ coef) {
  __shared__ double red[kFinish / 32];
  __shared__ double s[3];
  const int p = blockIdx.x;
  const double* part = partial + (long long)p * kChunks * 3;
  for (int k = 0; k < 3; ++k) {
    double v = 0.0;
    for (int j = threadIdx.x; j < kChunks; j += kFinish) v += part[j * 3 + k];
    v = block_sum<kFinish>(v, red);
    if (threadIdx.x == 0) s[k] = v;
  }
  __syncthreads();
  const double ab = s[0], aa = s[1], bb = s[2];
  if (f0 == 0 && threadIdx.x < 3) sums[p * 3 + threadIdx.x] = s[threadIdx.x];
  if (threadIdx.x >= count) return;
  const double alpha = alphas.v[threadIdx.x];
  double wa = 1.0 - alpha, wb = alpha;  // lerp: an endpoint is zero, or the endpoints are (anti)parallel
  if (aa > 0.0 && bb > 0.0) {
    double c = ab / sqrt(aa * bb);
    c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c);
    const double theta = acos(c);
    const double st = sin(theta);
    if (st >= 1e-6) {
      wa = sin((1.0 - alpha) * theta) / st;
      wb = sin(alpha * theta) / st;
    }
  }
  float* out = coef + ((long long)p * frames + f0 + threadIdx.x) * 2;
  out[0] = (float)wa;
  out[1] = (float)wb;
}

__device__ __forceinline__ float mix(float wa, float a, float wb, float b) {
  return __fadd_rn(__fmul_rn(wa, a), __fmul_rn(wb, b));
}

// grid (ceil(n4 / kThreads), pairs): n4 = n / 4 vectors per row; rows are 16-byte aligned (n % 4 == 0)
__global__ void __launch_bounds__(kThreads) slerp_frames_vec_kernel(const float4* __restrict__ za, const float4* __restrict__ zb,
                                                                    long long n4, const float2* __restrict__ coef, int frames,
                                                                    float4* __restrict__ out) {
  const int p = blockIdx.y;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n4) return;
  const float4 a = __ldg(za + (long long)p * n4 + i), b = __ldg(zb + (long long)p * n4 + i);
  const float2* w = coef + (long long)p * frames;
  float4* o = out + (long long)p * frames * n4 + i;
  for (int f = 0; f < frames; ++f) {
    const float2 c = __ldg(w + f);
    __stcs(o + (long long)f * n4, make_float4(mix(c.x, a.x, c.y, b.x), mix(c.x, a.y, c.y, b.y), mix(c.x, a.z, c.y, b.z),
                                              mix(c.x, a.w, c.y, b.w)));
  }
}

// the same one element per thread, for rows that are not 16-byte aligned
__global__ void __launch_bounds__(kThreads) slerp_frames_kernel(const float* __restrict__ za, const float* __restrict__ zb,
                                                                long long n, const float2* __restrict__ coef, int frames,
                                                                float* __restrict__ out) {
  const int p = blockIdx.y;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float a = __ldg(za + (long long)p * n + i), b = __ldg(zb + (long long)p * n + i);
  const float2* w = coef + (long long)p * frames;
  float* o = out + (long long)p * frames * n + i;
  for (int f = 0; f < frames; ++f) {
    const float2 c = __ldg(w + f);
    __stcs(o + (long long)f * n, mix(c.x, a, c.y, b));
  }
}

bool aligned16(const void* q) { return ((unsigned long long)q & 15ull) == 0; }

}  // namespace

extern "C" {

int mdb_slerp_chunks(void) { return kChunks; }

int mdb_slerp_frames(const float* za, const float* zb, long long n, int pairs, const double* alphas, int frames,
                     double* partial, double* sums, float* coef, float* out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n < 1 || pairs < 1 || frames < 2) return fail("mdb_slerp_frames: need n >= 1, pairs >= 1 and frames >= 2");
  if (pairs > 65535) return fail("mdb_slerp_frames: at most 65535 pairs");
  if (!za || !zb || !alphas || !partial || !sums || !coef || !out) return fail("mdb_slerp_frames: null argument");
  if (((unsigned long long)coef & 7ull) != 0) return fail("mdb_slerp_frames: coef must be 8-byte aligned");
  for (int f = 0; f < frames; ++f)
    if (!std::isfinite(alphas[f])) return fail("mdb_slerp_frames: alphas must be finite");
  const long long chunk = (n + kChunks - 1) / kChunks;
  slerp_dots_kernel<<<dim3(kChunks, (unsigned)pairs), kThreads, 0, s>>>(za, zb, n, chunk, partial);
  for (int f0 = 0; f0 < frames; f0 += kAlphas) {
    Alphas a{};
    const int count = frames - f0 < kAlphas ? frames - f0 : kAlphas;
    for (int k = 0; k < count; ++k) a.v[k] = alphas[f0 + k];
    slerp_coef_kernel<<<pairs, kFinish, 0, s>>>(partial, a, f0, count, frames, sums, coef);
  }
  const float2* w = reinterpret_cast<const float2*>(coef);
  if (n % 4 == 0 && aligned16(za) && aligned16(zb) && aligned16(out)) {
    const long long n4 = n / 4;
    slerp_frames_vec_kernel<<<dim3((unsigned)((n4 + kThreads - 1) / kThreads), (unsigned)pairs), kThreads, 0, s>>>(
        reinterpret_cast<const float4*>(za), reinterpret_cast<const float4*>(zb), n4, w, frames,
        reinterpret_cast<float4*>(out));
  } else {
    slerp_frames_kernel<<<dim3((unsigned)((n + kThreads - 1) / kThreads), (unsigned)pairs), kThreads, 0, s>>>(
        za, zb, n, w, frames, out);
  }
  const cudaError_t err = cudaGetLastError();
  return err == cudaSuccess ? 0 : fail(std::string("mdb_slerp_frames: ") + cudaGetErrorString(err));
}

}  // extern "C"
