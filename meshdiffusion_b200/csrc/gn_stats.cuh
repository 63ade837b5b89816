// GroupNorm statistics record shared by the GEMM epilogue (producer) and the GroupNorm kernels (consumers).
//
// Per (sample, channel): kStatWords = 4 signed 64-bit integers
//   w0, w1 : sum x      = w0 * 2^-24 + w1 * 2^16
//   w2, w3 : sum x^2    = w2 * 2^-24 + w3 * 2^16
// Every partial p is split EXACTLY into hi = rint(p / 2^16) and lo = p - hi * 2^16 (|lo| <= 2^15), lo is added to the
// low word as a 2^-24 fixed-point integer and hi (almost always 0) to the high word. Integer atomics commute, so the
// totals do not depend on the order tiles finish in -- the statistics, and with them the whole forward pass, are bitwise
// reproducible -- and the pair cannot overflow for any finite bf16/fp32 activation tensor (a single 2^-24 word wraps once
// sum x^2 exceeds 5.5e11, i.e. an rms of 1450 over a 64^3 grid: reached after four Adam steps in the full-size
// training test).
#pragma once
#include <cuda_runtime.h>

namespace mdb {

constexpr int kStatWords = 4;

__device__ __forceinline__ void stat_add(long long* lo_word, float partial) {
  const double v = (double)partial;
  const double hi = rint(v * (1.0 / 65536.0));
  const double lo = v - hi * 65536.0;
  atomicAdd(reinterpret_cast<unsigned long long*>(lo_word), (unsigned long long)__double2ll_rn(lo * 16777216.0));
  if (hi != 0.0) atomicAdd(reinterpret_cast<unsigned long long*>(lo_word) + 1, (unsigned long long)__double2ll_rn(hi));
}

// exact integer accumulation over several records (the channels of a group), combined once
struct StatAcc {
  long long s_lo = 0, s_hi = 0, q_lo = 0, q_hi = 0;
  __device__ __forceinline__ void add(const long long* rec) { s_lo += rec[0]; s_hi += rec[1]; q_lo += rec[2]; q_hi += rec[3]; }
  __device__ __forceinline__ double sum() const { return (double)s_lo * (1.0 / 16777216.0) + (double)s_hi * 65536.0; }
  __device__ __forceinline__ double sumsq() const { return (double)q_lo * (1.0 / 16777216.0) + (double)q_hi * 65536.0; }
};

// nn.GroupNorm(32, C, eps=1e-6) statistics (layers.py:589,652,660; ddpm_res64.py:120): mean and rstd (biased variance) of
// group g (cpg channels) of sample b over the channel concatenation of stats0 (C0 channels) and stats1 (C1 channels)
__device__ __forceinline__ void gn_group_stats(const long long* stats0, int C0, const long long* stats1, int C1, int b, int g,
                                               int cpg, long long voxels, float eps, float& mean, float& rstd) {
  StatAcc acc;
  for (int i = 0; i < cpg; ++i) {
    const int cc = g * cpg + i;
    acc.add((cc < C0) ? stats0 + ((long long)b * C0 + cc) * kStatWords : stats1 + ((long long)b * C1 + (cc - C0)) * kStatWords);
  }
  const double n = (double)voxels * cpg;
  const double m = acc.sum() / n;
  double var = acc.sumsq() / n - m * m;
  if (var < 0) var = 0;
  mean = (float)m;
  rstd = (float)(1.0 / sqrt(var + (double)eps));
}

}  // namespace mdb
