// One entry of a solver table (diffusion/sampling.py): a DPM-Solver++(2M) step (Lu et al. 2022) or, in a RePaint
// resampling schedule (Lugmayr et al., CVPR 2022; `--mode=edit`), a forward-diffusion jump back up the label grid, then
// the replacement of a kept region on a set of channels. The few-step samplers, the inverter and shape editing all run
// their tables through this one kernel. One HBM pass per entry.
//
// Every product and sum is rounded on its own (no FMA contraction), in this order:
//   denoise: x0 = (x - sigma*eps) * inv_alpha
//            x' = ((c_x*x + c_0*x0) + c_1*x0_prev) + c_z*z   (c_1 term only if c_1 != 0, c_z term only if c_z != 0)
//            x' = x' * g;  x0_hist <- x0
//   renoise: x' = (c_x*x + c_z*z) * g
//   channel c in `channels`: s = coef*known_c + std*z';  x' = (x'*(1-m) + s*m) * g
// The eager torch update in diffusion/sampling.py (_update_eager) does the same operations in the same order, so given
// the same eps and noise the two are bit-identical.
#include "elementwise.cuh"
#include <curand_kernel.h>
#include <algorithm>

namespace mdb {

int sm_count();  // gemm_host.cu

__device__ __forceinline__ float philox_normal(unsigned long long seed, unsigned long long element, unsigned long long offset) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, element, offset, &st);
  return curand_normal(&st);
}

// blockIdx.y = b * C + c (one channel row of one sample), grid-stride over its voxels; element index i = (b C + c) V + v
// keys the Philox draws, so the grid shape does not change the result
__global__ void __launch_bounds__(256) solver_update_kernel(SolverEntryArgs a) {
  const long long bc = blockIdx.y;
  const int ch = (int)(bc % a.C);
  const long long b = bc / a.C;
  const long long row = bc * a.V;
  const bool replace = a.known != nullptr && ((a.channels >> ch) & 1u);
  const float* known = replace ? a.known + b * a.known_bs + (long long)ch * a.V : nullptr;
  const float* kmask = replace ? a.kmask + b * a.kmask_bs : nullptr;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < a.V; v += (long long)gridDim.x * blockDim.x) {
    const long long i = row + v;
    const float g = __ldg(a.mask + v);
    const float xv = a.x[i];
    float xn;
    if (a.renoise) {
      const float z = a.noise ? a.noise[i] : philox_normal(a.seed, (unsigned long long)i, a.offset);
      xn = __fmul_rn(__fadd_rn(__fmul_rn(a.c_x, xv), __fmul_rn(a.c_z, z)), g);
    } else {
      const float x0 = __fmul_rn(__fsub_rn(xv, __fmul_rn(a.sigma, a.eps[i])), a.inv_alpha);
      xn = __fadd_rn(__fmul_rn(a.c_x, xv), __fmul_rn(a.c_0, x0));
      if (a.c_1 != 0.f) xn = __fadd_rn(xn, __fmul_rn(a.c_1, a.x0_hist[i]));
      if (a.c_z != 0.f) {
        const float z = a.noise ? a.noise[i] : philox_normal(a.seed, (unsigned long long)i, a.offset);
        xn = __fadd_rn(xn, __fmul_rn(a.c_z, z));
      }
      xn = __fmul_rn(xn, g);
      a.x0_hist[i] = x0;
    }
    if (replace) {
      const float m = __ldg(kmask + v);
      const float kv = __ldg(known + v);
      const float z2 = a.known_noise ? a.known_noise[i] : philox_normal(a.seed, (unsigned long long)i, a.offset + 2);
      const float sampled = __fadd_rn(__fmul_rn(a.coef, kv), __fmul_rn(a.std, z2));
      xn = __fmul_rn(__fadd_rn(__fmul_rn(xn, __fsub_rn(1.f, m)), __fmul_rn(sampled, m)), g);
    }
    a.x[i] = xn;
  }
}

void launch_solver_entry(const SolverEntryArgs& a, int B, cudaStream_t s) {
  const long long rows = (long long)B * a.C;
  if (rows > 65535) throw std::runtime_error("mdb: a solver entry takes at most 65535 (sample, channel) rows");
  // 32 blocks per SM of the current device over the whole launch, whatever the batch: four waves of 8 resident blocks, so
  // the partial last wave is a short tail (one wave rounded up per row spills a few blocks into a mostly idle second
  // wave: about 20% slower at batch 32, R = 64)
  long long gx = (a.V + 255) / 256;
  const long long cap = std::max(1LL, (long long)sm_count() * 32 / rows);
  if (gx > cap) gx = cap;
  solver_update_kernel<<<dim3((unsigned)gx, (unsigned)rows), 256, 0, s>>>(a);
  MDB_LAUNCH_CHECK();
}

}  // namespace mdb
