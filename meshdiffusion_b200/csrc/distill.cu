// Progressive distillation (Salimans & Ho, ICLR 2022; `--mode=distill`, diffusion/distill.py): the teacher's two DDIM
// steps s -> m -> e of one student step s -> e, and the noise prediction that makes the student's single DDIM step from
// z_s land on the teacher's z_e. Every sample b reads its own row rows[step_idx[b]], so a batch can mix student steps.
//
// Every product and sum is rounded on its own (no FMA contraction), in this order:
//   phase 0: x0 = (z_s - sigma_s eps) inv_alpha_s;  z_mid = (c_x_s z_s + c_0_s x0) g;  labels[b] = m
//   phase 1: x0 = (z_mid - sigma_m eps) inv_alpha_m;  z_e = (c_x_m z_mid + c_0_m x0) g;
//            out = ((z_e - r z_s) inv_d) g;  labels[b] = s
// Phase 0 is the first-order (c_1 = 0, c_z = 0) path of solver_update_kernel, so with equal indices the two agree bit for
// bit. The eager torch phases in diffusion/distill.py (distill_step_eager) do the same operations in the same order.
// A sample whose index lies outside [0, n_rows) reads no row: its outputs and its label are NaN.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <cmath>
#include <stdexcept>
#include <string>

namespace mdb {

void set_last_error(const std::string& msg);

// blockIdx.y = sample b, grid-stride over its C * V elements
__global__ void __launch_bounds__(256) distill_step_kernel(const float* __restrict__ eps, const float* __restrict__ z_s,
                                                           float* z_mid, float* __restrict__ out,
                                                           const float* __restrict__ mask, const int* __restrict__ step_idx,
                                                           const mdb_distill_row* __restrict__ rows, int n_rows, int phase,
                                                           float* __restrict__ labels, long long V, int C) {
  const long long b = blockIdx.y;
  const long long per = V * C;
  const int k = step_idx[b];
  const bool valid = k >= 0 && k < n_rows;
  const float nan = __int_as_float(0x7fc00000);
  float sigma = nan, inv_alpha = nan, c_x = nan, c_0 = nan, r = nan, inv_d = nan, label = nan;
  if (valid) {
    const mdb_distill_row& w = rows[k];
    if (phase == 0) {
      sigma = w.sigma_s; inv_alpha = w.inv_alpha_s; c_x = w.c_x_s; c_0 = w.c_0_s; label = w.label_m;
    } else {
      sigma = w.sigma_m; inv_alpha = w.inv_alpha_m; c_x = w.c_x_m; c_0 = w.c_0_m; r = w.r; inv_d = w.inv_d;
      label = w.label_s;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) labels[b] = label;
  const long long base = b * per;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < per; j += (long long)gridDim.x * blockDim.x) {
    const long long i = base + j;
    const float g = __ldg(mask + j % V);
    if (!valid) {
      (phase == 0 ? z_mid : out)[i] = nan;
      continue;
    }
    const float xv = phase == 0 ? z_s[i] : z_mid[i];
    const float x0 = __fmul_rn(__fsub_rn(xv, __fmul_rn(sigma, eps[i])), inv_alpha);
    float xn = __fadd_rn(__fmul_rn(c_x, xv), __fmul_rn(c_0, x0));
    xn = __fmul_rn(xn, g);
    if (phase == 0) {
      z_mid[i] = xn;
    } else {
      out[i] = __fmul_rn(__fmul_rn(__fsub_rn(xn, __fmul_rn(r, z_s[i])), inv_d), g);
    }
  }
}

void launch_distill_step(const float* eps, const float* z_s, float* z_mid, float* out, const float* mask,
                         const int* step_idx, const mdb_distill_row* rows, int n_rows, int phase, float* labels,
                         long long V, int C, int B, cudaStream_t s) {
  if (phase != 0 && phase != 1) throw std::runtime_error("mdb: distill phase must be 0 (teacher step s -> m) or 1 (m -> e and the target)");
  if (V <= 0 || C <= 0 || B <= 0) throw std::runtime_error("mdb: mdb_distill_step needs positive voxels, channels, batch");
  if (B > 65535) throw std::runtime_error("mdb: mdb_distill_step takes at most 65535 samples");
  if (n_rows < 1) throw std::runtime_error("mdb: mdb_distill_step needs at least one row");
  if (!eps || !z_s || !z_mid || !mask || !step_idx || !rows || !labels || (phase == 1 && !out))
    throw std::runtime_error("mdb: mdb_distill_step: null argument");
  // about 8 resident blocks per SM of the current device over the whole launch, whatever the batch
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1)
    throw std::runtime_error("mdb: mdb_distill_step could not read the device's SM count");
  long long gx = (V * C + 255) / 256;
  const long long cap = ((long long)sms * 8 + B - 1) / B;
  if (gx > cap) gx = cap;
  distill_step_kernel<<<dim3((unsigned)gx, (unsigned)B), 256, 0, s>>>(eps, z_s, z_mid, out, mask, step_idx, rows, n_rows,
                                                                      phase, labels, V, C);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("mdb launch: ") + cudaGetErrorString(e));
}

}  // namespace mdb

extern "C" {

int mdb_distill_step(const float* eps, const float* z_s, float* z_mid, float* out, const float* mask, const int* step_idx,
                     const mdb_distill_row* rows, int n_rows, int phase, float* labels, long long voxels, int channels,
                     int batch, void* stream) {
  try {
    mdb::launch_distill_step(eps, z_s, z_mid, out, mask, step_idx, rows, n_rows, phase, labels, voxels, channels, batch,
                             (cudaStream_t)stream);
  } catch (const std::exception& e) {
    mdb::set_last_error(e.what());
    return 1;
  }
  return 0;
}

}  // extern "C"
