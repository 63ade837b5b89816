// Probability-flow ODE right-hand side of the likelihood driver (diffusion/likelihood.py), one pass over [B][C][V].
//
// VPSDE.sde + reverse(probability_flow=True) with the continuous-time VP score  score = -e / std(t):
//   drift = mask * (-0.5 beta) (x - e / std)
// and the Hutchinson-Skilling estimate of its divergence, with g = J_e^T (h * mask) from mdb_unet_backward_input:
//   div[b] = -0.5 beta ( sum_masked h^2 - (1/std) sum_masked h g )
// The sums are fp64 and reduced in a fixed order: every sample is cut into the same kBlocks voxel chunks whatever the
// batch, each chunk is reduced by a fixed tree, and the chunks by another. So `div` is bitwise reproducible and a
// sample's value does not depend on the batch it was launched in.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }

constexpr int kThreads = 256, kBlocks = 128;

// fixed-order sum of one double over the block (shuffle tree, then the warps' results in warp order)
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

// grid (kBlocks, B): block j of sample b owns voxels [j*chunk, (j+1)*chunk) of every channel
__global__ void __launch_bounds__(kThreads) pflow_drift_div_kernel(const float* __restrict__ x, const float* __restrict__ e,
                                                                   const float* __restrict__ h, const float* __restrict__ g,
                                                                   const float* __restrict__ mask, float coef, float stdv,
                                                                   float* __restrict__ drift, double* __restrict__ part,
                                                                   int C, long long V, long long chunk) {
  __shared__ double red[kThreads / 32];
  const int b = blockIdx.y;
  const long long v0 = (long long)blockIdx.x * chunk;
  const long long v1 = v0 + chunk < V ? v0 + chunk : V;
  double s1 = 0.0, s2 = 0.0;
  for (long long v = v0 + threadIdx.x; v < v1; v += kThreads) {
    const float m = mask ? __ldg(mask + v) : 1.f;
    for (int c = 0; c < C; ++c) {
      const long long i = ((long long)b * C + c) * V + v;
      drift[i] = m * (coef * (__ldg(x + i) - __ldg(e + i) / stdv));
      const double hv = (double)__ldg(h + i);
      s1 += (double)m * hv * hv;
      s2 += (double)m * hv * (double)__ldg(g + i);
    }
  }
  s1 = block_sum<kThreads>(s1, red);
  s2 = block_sum<kThreads>(s2, red);
  if (threadIdx.x == 0) {
    part[((long long)b * kBlocks + blockIdx.x) * 2] = s1;
    part[((long long)b * kBlocks + blockIdx.x) * 2 + 1] = s2;
  }
}

__global__ void __launch_bounds__(kBlocks) pflow_div_finish_kernel(const double* __restrict__ part, double coef, double stdv,
                                                                   double* __restrict__ div) {
  __shared__ double red[kBlocks / 32];
  const int b = blockIdx.x;
  const double s1 = block_sum<kBlocks>(part[((long long)b * kBlocks + threadIdx.x) * 2], red);
  const double s2 = block_sum<kBlocks>(part[((long long)b * kBlocks + threadIdx.x) * 2 + 1], red);
  if (threadIdx.x == 0) div[b] = coef * (s1 - s2 / stdv);
}

}  // namespace

extern "C" {

int mdb_pflow_drift_div(const float* x, const float* e, const float* h, const float* g, const float* mask, float beta,
                        float stdv, float* drift, double* div, int batch, int channels, long long voxels, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (batch < 0 || channels < 1 || voxels < 1) return fail("mdb_pflow_drift_div: bad shape");
  if (batch > 65535) return fail("mdb_pflow_drift_div: at most 65535 samples");
  if (!(stdv > 0.f) || !(stdv < 3.0e38f)) return fail("mdb_pflow_drift_div: std must be positive and finite");
  if (!x || !e || !h || !g || !drift || !div) return fail("mdb_pflow_drift_div: null argument");
  if (batch == 0) return 0;
  double* part = nullptr;
  cudaError_t err = cudaMallocAsync(&part, (size_t)batch * kBlocks * 2 * sizeof(double), s);
  if (err != cudaSuccess) return fail(std::string("mdb_pflow_drift_div: ") + cudaGetErrorString(err));
  const long long chunk = (voxels + kBlocks - 1) / kBlocks;
  pflow_drift_div_kernel<<<dim3(kBlocks, (unsigned)batch), kThreads, 0, s>>>(x, e, h, g, mask, -0.5f * beta, stdv, drift, part,
                                                                           channels, voxels, chunk);
  pflow_div_finish_kernel<<<batch, kBlocks, 0, s>>>(part, -0.5 * (double)beta, (double)stdv, div);
  err = cudaGetLastError();
  cudaFreeAsync(part, s);
  return err == cudaSuccess ? 0 : fail(std::string("mdb_pflow_drift_div: ") + cudaGetErrorString(err));
}

}  // extern "C"
