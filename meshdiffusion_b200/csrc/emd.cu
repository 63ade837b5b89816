// Earth Mover's distance matrices of point clouds (no reference counterpart; the reference ships no evaluation code).
//
// EMD(X, Y) = min over bijections pi of (1/N) sum_i |x_i - y_pi(i)|, Euclidean, for clouds of equal size N. One CTA per
// cloud pair solves the N x N assignment with Bertsekas' forward auction and epsilon-scaling, in Jacobi rounds: X points
// bid for Y points, every unassigned bidder at once. The Y cloud, the prices, the owners and the per-object bid slots stay
// in shared memory. Every decision of a round is order-independent (exact minima, lowest-index ties, a 64-bit atomicMax
// on (bid bits, ~bidder)), so the result is bitwise reproducible and does not depend on the other pairs of the launch.
// oracle/emd_oracle.py's emd_auction restates the algorithm in float32 numpy with the same rounding and tie rules.
//
// Per pair the kernel returns the mean cost of its final assignment and a certified gap: that mean minus the dual bound
// (sum_i min_j (c_ij + p_j) - sum_j p_j) / N, which is a lower bound on the optimum for any prices p.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

namespace {

int fail(const std::string& m) { mdb::set_last_error(m); return 1; }

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr float kEpsFactor = 5.0f;        // epsilon divides by this between phases
constexpr float kStartFraction = 0.25f;   // first phase: C_max / 4
constexpr float kFloor = 0x1p-18f;        // eps below kFloor * C_max is refused: fp32 prices cannot resolve it
constexpr float kMargin = 0x1p-19f;       // the last phase runs at eps - kMargin * C_max (absorbs the bids' rounding)
constexpr int kMaxRounds = 1 << 18;       // a pair that needs more rounds gets NaN and an infinite gap

size_t emd_smem_bytes(int N) {
  return (size_t)N * (sizeof(float4) + sizeof(unsigned long long) + sizeof(float) + sizeof(int) + sizeof(unsigned short) + 1) +
         kThreads * sizeof(double) + 64;
}

// c = sqrt((dx*dx + dy*dy) + dz*dz), every operation rounded on its own (no contraction): what numpy's float32 computes
__device__ __forceinline__ float cost(float x, float y, float z, float4 q) {
  const float dx = __fsub_rn(x, q.x), dy = __fsub_rn(y, q.y), dz = __fsub_rn(z, q.z);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}

// Sum over threads' partials in a fixed halving tree: with partials taken over t, t + kThreads, ... the order depends on n only
__device__ double tree_sum(double s, double* red) {
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__device__ float block_reduce(float v, bool is_max, float* redf) {
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : fminf(v, w);
  }
  if (threadIdx.x % 32 == 0) redf[threadIdx.x / 32] = v;
  __syncthreads();
  float r = redf[0];
  for (int k = 1; k < kWarps; ++k) r = is_max ? fmaxf(r, redf[k]) : fminf(r, redf[k]);
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kThreads, 3) emd_pair_kernel(const float* __restrict__ A, const float* __restrict__ B, int N,
                                                               int nB, int self, float eps, double* __restrict__ out,
                                                               double* __restrict__ gap) {
  const int pi = blockIdx.y, pj = blockIdx.x;
  const long long o = (long long)pi * nB + pj;
  if (self && pj < pi) return;  // the mirror of (pj, pi)
  if (self && pj == pi) {
    if (threadIdx.x == 0) { out[o] = 0.0; gap[o] = 0.0; }
    return;
  }
  extern __shared__ __align__(16) unsigned char smem[];
  float4* Y = reinterpret_cast<float4*>(smem);
  unsigned long long* slot = reinterpret_cast<unsigned long long*>(Y + N);  // bids; reused for the dual pass's row minima
  double* red = reinterpret_cast<double*>(slot + N);
  float* price = reinterpret_cast<float*>(red + kThreads);
  int* owner = reinterpret_cast<int*>(price + N);
  unsigned short* list = reinterpret_cast<unsigned short*>(owner + N);
  unsigned char* unas = reinterpret_cast<unsigned char*>(list + N);
  float* redf = reinterpret_cast<float*>(red);  // scratch for float reductions (not live at the same time as red)
  __shared__ int s_count;

  const float* X = A + (long long)pi * N * 3;
  const float* Yg = B + (long long)pj * N * 3;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const float kInf = __int_as_float(0x7f800000);

  float lo[3] = {kInf, kInf, kInf}, hi[3] = {-kInf, -kInf, -kInf};
  for (int k = tid; k < N; k += kThreads) {
    const float4 q = make_float4(Yg[3LL * k], Yg[3LL * k + 1], Yg[3LL * k + 2], 0.f);
    Y[k] = q;
    price[k] = 0.f;
    const float xs[3] = {X[3LL * k], X[3LL * k + 1], X[3LL * k + 2]}, ys[3] = {q.x, q.y, q.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      lo[c] = fminf(lo[c], fminf(xs[c], ys[c]));
      hi[c] = fmaxf(hi[c], fmaxf(xs[c], ys[c]));
    }
  }
  float ext[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) ext[c] = __fsub_rn(block_reduce(hi[c], true, redf), block_reduce(lo[c], false, redf));
  const float cmax = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(ext[0], ext[0]), __fmul_rn(ext[1], ext[1])), __fmul_rn(ext[2], ext[2])));
  if (!(eps >= cmax * kFloor)) {  // the host refuses such eps before the launch; this keeps the kernel bounded regardless
    if (tid == 0) {
      const double nan = __longlong_as_double(0x7ff8000000000000LL);
      out[o] = nan; gap[o] = nan;
      if (self) { out[(long long)pj * nB + pi] = nan; gap[(long long)pj * nB + pi] = nan; }
    }
    return;
  }
  const float last = __fsub_rn(eps, cmax * kMargin);

  int rounds = 0;
  bool capped = false;
  float e = cmax * kStartFraction;
  for (bool final_phase = false; !final_phase && !capped; e = __fdiv_rn(e, kEpsFactor)) {
    if (!(e > last)) { e = last; final_phase = true; }
    // phase start: prices shift by their minimum (the auction is invariant under a common shift), assignment cleared
    float pmin = kInf;
    for (int k = tid; k < N; k += kThreads) pmin = fminf(pmin, price[k]);
    pmin = block_reduce(pmin, false, redf);
    for (int k = tid; k < N; k += kThreads) {
      price[k] = __fsub_rn(price[k], pmin);
      owner[k] = -1;
      unas[k] = 1;
      slot[k] = 0ull;
    }
    while (true) {
      // 1. compact the unassigned bidders (their order in the list does not change any decision)
      if (tid == 0) s_count = 0;
      __syncthreads();
      for (int base = 0; base < N; base += kThreads) {
        const int i = base + tid;
        const bool u = i < N && unas[i];
        const unsigned m = __ballot_sync(0xffffffffu, u);
        int at = 0;
        if (lane == 0 && m) at = atomicAdd(&s_count, __popc(m));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (u) list[at + __popc(m & ((1u << lane) - 1u))] = (unsigned short)i;
      }
      __syncthreads();
      const int n_un = s_count;
      if (n_un == 0) break;
      if (rounds >= kMaxRounds) { capped = true; break; }
      ++rounds;
      // 2. one warp per bidder: best and second-best c_ij + p_j, ties to the lowest j; 3. bid
      for (int k = warp; k < n_un; k += kWarps) {
        const int i = list[k];
        const float x = X[3LL * i], y = X[3LL * i + 1], z = X[3LL * i + 2];
        float best = kInf, second = kInf;
        int bj = 0x7fffffff;
        for (int j = lane; j < N; j += 32) {
          const float v = __fadd_rn(cost(x, y, z, Y[j]), price[j]);
          const bool lt = v < best;
          second = lt ? best : fminf(second, v);
          bj = lt ? j : bj;
          best = lt ? v : best;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, off);
          const float os = __shfl_xor_sync(0xffffffffu, second, off);
          const int oj = __shfl_xor_sync(0xffffffffu, bj, off);
          const bool take = ob < best || (ob == best && oj < bj);
          second = take ? fminf(os, best) : fminf(second, ob);
          bj = take ? oj : bj;
          best = take ? ob : best;
        }
        if (lane == 0) {
          if (second == kInf) second = best;  // N = 1: no second object
          const float bid = __fadd_rn(__fadd_rn(price[bj], __fsub_rn(second, best)), e);
          // highest bid wins, equal bids go to the lowest bidder; non-negative float bits order as integers
          atomicMax(slot + bj, ((unsigned long long)__float_as_uint(bid) << 32) | (unsigned)(~i));
        }
      }
      __syncthreads();
      // 4. objects that received a bid change owner; the displaced owner bids again next round
      for (int j = tid; j < N; j += kThreads) {
        const unsigned long long key = slot[j];
        if (key) {
          const int i = (int)~(unsigned)key, prev = owner[j];
          if (prev >= 0) unas[prev] = 1;
          owner[j] = i;
          unas[i] = 0;
          price[j] = __uint_as_float((unsigned)(key >> 32));
          slot[j] = 0ull;
        }
      }
      __syncthreads();
    }
  }
  if (capped) {
    if (tid == 0) {
      const double nan = __longlong_as_double(0x7ff8000000000000LL), inf = __longlong_as_double(0x7ff0000000000000LL);
      out[o] = nan; gap[o] = inf;
      if (self) { out[(long long)pj * nB + pi] = nan; gap[(long long)pj * nB + pi] = inf; }
    }
    return;
  }

  // the assignment's cost, and the dual bound: row minima of c_ij + p_j in fp64 (exact for fp32 operands)
  double sc = 0.0, sp = 0.0;
  for (int j = tid; j < N; j += kThreads) {
    const int i = owner[j];
    sc += (double)cost(X[3LL * i], X[3LL * i + 1], X[3LL * i + 2], Y[j]);
    sp += (double)price[j];
  }
  double* rowmin = reinterpret_cast<double*>(slot);
  for (int i = warp; i < N; i += kWarps) {
    const float x = X[3LL * i], y = X[3LL * i + 1], z = X[3LL * i + 2];
    double m = __longlong_as_double(0x7ff0000000000000LL);
    for (int j = lane; j < N; j += 32) m = fmin(m, __dadd_rn((double)cost(x, y, z, Y[j]), (double)price[j]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) rowmin[i] = m;
  }
  __syncthreads();
  double sr = 0.0;
  for (int i = tid; i < N; i += kThreads) sr += rowmin[i];
  const double sum_c = tree_sum(sc, red), sum_p = tree_sum(sp, red), sum_r = tree_sum(sr, red);
  if (tid == 0) {
    const double emd = sum_c / (double)N, g = emd - (sum_r - sum_p) / (double)N;
    out[o] = emd; gap[o] = g;
    if (self) { out[(long long)pj * nB + pi] = emd; gap[(long long)pj * nB + pi] = g; }
  }
}

}  // namespace

extern "C" {

int mdb_emd_matrix(const float* A, int nA, const float* B, int nB, int N, float eps, double* out, double* gap, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int self = B == nullptr;
  if (self) { B = A; nB = nA; }
  if (nA < 0 || nB < 0) return fail("mdb_emd_matrix: negative cloud count");
  if (N < 1) return fail("mdb_emd_matrix: every cloud needs at least one point");
  if (N > 65535) return fail("mdb_emd_matrix: at most 65535 points per cloud");
  if (!(eps > 0.0f) || !(eps < 3.0e38f)) return fail("mdb_emd_matrix: eps must be positive and finite");
  if (nA > 65535) return fail("mdb_emd_matrix: at most 65535 clouds in A");
  if (nA == 0 || nB == 0) return 0;
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return fail("mdb_emd_matrix: cannot query the device");
  const size_t smem = emd_smem_bytes(N);
  if (smem > (size_t)optin)
    return fail("mdb_emd_matrix: the auction state of N = " + std::to_string(N) + " points does not fit in shared memory");
  if (cudaFuncSetAttribute(emd_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("mdb_emd_matrix: cudaFuncSetAttribute failed");
  emd_pair_kernel<<<dim3((unsigned)nB, (unsigned)nA), kThreads, smem, s>>>(A, B, N, nB, self, eps, out, gap);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(std::string("mdb_emd_matrix: ") + cudaGetErrorString(e));
}

}  // extern "C"
