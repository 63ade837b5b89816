// Bandwidth-bound training kernels around the score network (reference: lib/diffusion/losses.py:38-85,
// lib/diffusion/models/ema.py:43-64): the masked DDPM loss with its gradient, global-norm gradient clipping, and a
// single multi-tensor pass that applies clipping + Adam + the EMA update (the reference makes ~5 separate passes over
// the 364 M parameters per step: clip_grad_norm_, Adam's foreach ops, EMA).
// These are the optimiser-side building blocks of the training step (the network backward is unet_train.cu).
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdint.h>
#include <stdexcept>
#include <string>

namespace mdb { void set_last_error(const std::string& msg); }

#define TR_API_BEGIN try {
#define TR_API_END                                                              \
  }                                                                             \
  catch (const std::exception& e) { mdb::set_last_error(e.what()); return 1; }  \
  return 0;
#define TR_CHECK(expr)                                                                                         \
  do {                                                                                                         \
    cudaError_t _e = (expr);                                                                                   \
    if (_e != cudaSuccess) throw std::runtime_error(std::string("mdb train: ") + cudaGetErrorString(_e) + " (" #expr ")"); \
  } while (0)

namespace {

__device__ __forceinline__ double block_sum(double v, double* sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  __syncthreads();
  return t;  // valid in thread 0
}

// losses = (pred - noise)^2 * mask; loss = mean_b(mean_{c,v}(losses)) * V / sum(mask)   (losses.py:69-78)
// d loss / d pred = 2 (pred - noise) mask * coef,  coef = 1 / (B C V) * V / sum(mask)
__global__ void ddpm_loss_kernel(const float* __restrict__ pred, const float* __restrict__ noise, const float* __restrict__ mask,
                                 double coef, double* __restrict__ acc, float* __restrict__ grad, long long V, long long total) {
  __shared__ double sh[32];
  double s = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float m = __ldg(mask + (i % V));
    const float d = pred[i] - noise[i];
    s += (double)(d * d * m);
    if (grad) grad[i] = (float)(2.0 * coef) * d * m;
  }
  const double t = block_sum(s, sh);
  if (threadIdx.x == 0) atomicAdd(acc, t * coef);
}
__global__ void store_scalar_kernel(const double* acc, float* out) { *out = (float)*acc; }

// perturbed_data = (sqrt(abar_t) x_0 + sqrt(1 - abar_t) eps) * mask (losses.py:63-66), same op order as the eager torch
// expression (no FMA contraction), so the network input is bit-identical to the reference's
__global__ void ddpm_perturb_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const float* __restrict__ mask,
                                    const float* __restrict__ sa, const float* __restrict__ sb, float* __restrict__ out,
                                    long long V, long long per, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / per;
    const float v = __fadd_rn(__fmul_rn(__ldg(sa + b), x0[i]), __fmul_rn(__ldg(sb + b), noise[i]));
    out[i] = __fmul_rn(v, __ldg(mask + (i % V)));
  }
}

// ---- multi-tensor passes over the parameter set. The work list is a table of fixed-size chunks {tensor, chunk index}
// built once by the host (494 tensors from 4 to 14 M elements: one block per 8192-element chunk keeps every SM streaming
// whatever the size mix), 16-byte vector accesses whenever the tensor's four streams are 16-byte aligned.
constexpr int kChunkElems = 8192;
constexpr int kChunkThreads = 256;

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// per-chunk sums of squares (no atomics: the final reduction below runs in a fixed order, so the clip coefficient is
// bitwise reproducible)
__global__ void __launch_bounds__(kChunkThreads) sq_norm_chunks_kernel(const float* const* __restrict__ grads, const long long* __restrict__ numels,
                                                                        const int2* __restrict__ chunks, double* __restrict__ part) {
  __shared__ double sh[32];
  const int2 ck = chunks[blockIdx.x];
  const float* g = grads[ck.x];
  const long long n = numels[ck.x];
  const long long i0 = (long long)ck.y * kChunkElems;
  const long long i1 = i0 + kChunkElems < n ? i0 + kChunkElems : n;
  float s = 0.f;
  double sd = 0;
  if (aligned16(g) && i1 - i0 == kChunkElems) {
#pragma unroll
    for (int k = 0; k < kChunkElems / (4 * kChunkThreads); ++k) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(g + i0) + threadIdx.x + k * kChunkThreads);
      s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    sd = s;
  } else {
    for (long long i = i0 + threadIdx.x; i < i1; i += kChunkThreads) { const float v = g[i]; sd += (double)v * v; }
  }
  const double t = block_sum(sd, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}
// clip_grad_norm_: coef = min(1, max_norm / (total_norm + 1e-6)); fixed-order sum of the chunk partials (one block)
__global__ void __launch_bounds__(1024) clip_coef_kernel(const double* __restrict__ part, int n_chunks, float max_norm, float* coef, float* total_norm) {
  __shared__ double sh[32];
  double s = 0;
  for (int i = threadIdx.x; i < n_chunks; i += blockDim.x) s += part[i];
  const double t = block_sum(s, sh);
  if (threadIdx.x == 0) {
    const float tn = (float)sqrt(t);
    if (total_norm) *total_norm = tn;
    const float c = max_norm / (tn + 1e-6f);
    if (coef) *coef = c < 1.f ? c : 1.f;
  }
}

struct AdamArgs {
  float* const* params; const float* const* grads; float* const* exp_avg; float* const* exp_avg_sq; float* const* ema;
  const long long* numels; const int2* chunks;
  float beta1, beta2, eps, step_size, inv_bc2_sqrt, one_minus_decay, weight_decay;
  const float* clip_coef;
};
__device__ __forceinline__ void adam_one(float& pi, float gi, float& mi, float& vi, const AdamArgs& a, float cc) {
  gi = gi * cc;
  if (a.weight_decay != 0.f) gi = gi + a.weight_decay * pi;  // grad.add(param, alpha=weight_decay)
  mi = mi + (gi - mi) * (1.f - a.beta1);                     // exp_avg.lerp_(grad, 1 - beta1)
  vi = vi * a.beta2 + (1.f - a.beta2) * gi * gi;             // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
  const float denom = sqrtf(vi) * a.inv_bc2_sqrt + a.eps;
  pi = pi - a.step_size * (mi / denom);                      // param.addcdiv_(exp_avg, denom, value=-step_size)
}
// torch.optim.Adam (no amsgrad) followed by ExponentialMovingAverage.update, one read-modify-write pass:
// 20 B read + 16 B written per parameter
template <bool EMA>
__global__ void __launch_bounds__(kChunkThreads) adam_ema_kernel(AdamArgs a) {
  const int2 ck = a.chunks[blockIdx.x];
  const int t = ck.x;
  float* p = a.params[t]; const float* g = a.grads[t]; float* m = a.exp_avg[t]; float* v = a.exp_avg_sq[t];
  float* e = EMA ? a.ema[t] : nullptr;
  const long long n = a.numels[t];
  const long long i0 = (long long)ck.y * kChunkElems;
  const long long i1 = i0 + kChunkElems < n ? i0 + kChunkElems : n;
  const float cc = a.clip_coef ? __ldg(a.clip_coef) : 1.f;
  if (i1 - i0 == kChunkElems && aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v) && (!EMA || aligned16(e))) {
    constexpr int K = 4;  // float4 per stream in flight per thread (5 streams: 80 registers of payload)
#pragma unroll 1
    for (int k0 = 0; k0 < kChunkElems / (4 * kChunkThreads); k0 += K) {
      float4 pv[K], gv[K], mv[K], vv[K], ev[K];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const long long o = threadIdx.x + (k0 + k) * kChunkThreads;
        gv[k] = __ldg(reinterpret_cast<const float4*>(g + i0) + o);
        pv[k] = reinterpret_cast<const float4*>(p + i0)[o];
        mv[k] = reinterpret_cast<const float4*>(m + i0)[o];
        vv[k] = reinterpret_cast<const float4*>(v + i0)[o];
        if (EMA) ev[k] = reinterpret_cast<const float4*>(e + i0)[o];
      }
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const long long o = threadIdx.x + (k0 + k) * kChunkThreads;
        adam_one(pv[k].x, gv[k].x, mv[k].x, vv[k].x, a, cc);
        adam_one(pv[k].y, gv[k].y, mv[k].y, vv[k].y, a, cc);
        adam_one(pv[k].z, gv[k].z, mv[k].z, vv[k].z, a, cc);
        adam_one(pv[k].w, gv[k].w, mv[k].w, vv[k].w, a, cc);
        reinterpret_cast<float4*>(p + i0)[o] = pv[k];
        reinterpret_cast<float4*>(m + i0)[o] = mv[k];
        reinterpret_cast<float4*>(v + i0)[o] = vv[k];
        if (EMA) {
          ev[k].x -= a.one_minus_decay * (ev[k].x - pv[k].x); ev[k].y -= a.one_minus_decay * (ev[k].y - pv[k].y);
          ev[k].z -= a.one_minus_decay * (ev[k].z - pv[k].z); ev[k].w -= a.one_minus_decay * (ev[k].w - pv[k].w);
          reinterpret_cast<float4*>(e + i0)[o] = ev[k];
        }
      }
    }
    return;
  }
  for (long long i = i0 + threadIdx.x; i < i1; i += kChunkThreads) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_one(pi, g[i], mi, vi, a, cc);
    p[i] = pi; m[i] = mi; v[i] = vi;
    if (EMA) { const float s = e[i]; e[i] = s - a.one_minus_decay * (s - pi); }
  }
}

// ExponentialMovingAverage.update alone (micro-steps that do not update the parameters): s -= (1 - decay) (s - p)
__global__ void __launch_bounds__(kChunkThreads) ema_kernel(float* const* __restrict__ ema, const float* const* __restrict__ params,
                                                             const long long* __restrict__ numels, const int2* __restrict__ chunks, float omd) {
  const int2 ck = chunks[blockIdx.x];
  float* e = ema[ck.x]; const float* p = params[ck.x];
  const long long n = numels[ck.x];
  const long long i0 = (long long)ck.y * kChunkElems;
  const long long i1 = i0 + kChunkElems < n ? i0 + kChunkElems : n;
  if (i1 - i0 == kChunkElems && aligned16(e) && aligned16(p)) {
#pragma unroll
    for (int k = 0; k < kChunkElems / (4 * kChunkThreads); ++k) {
      const long long o = threadIdx.x + k * kChunkThreads;
      float4 s = reinterpret_cast<const float4*>(e + i0)[o];
      const float4 q = __ldg(reinterpret_cast<const float4*>(p + i0) + o);
      s.x -= omd * (s.x - q.x); s.y -= omd * (s.y - q.y); s.z -= omd * (s.z - q.z); s.w -= omd * (s.w - q.w);
      reinterpret_cast<float4*>(e + i0)[o] = s;
    }
    return;
  }
  for (long long i = i0 + threadIdx.x; i < i1; i += kChunkThreads) { const float s = e[i]; e[i] = s - omd * (s - p[i]); }
}

}  // namespace

extern "C" {

int mdb_ddpm_loss(const float* pred, const float* noise, const float* mask, double mask_sum, float* loss_out,
                  float* grad_pred, double* scratch, int B, int C, long long V, void* stream) {
  TR_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  const long long total = (long long)B * C * V;
  const double coef = 1.0 / ((double)B * C * V) * ((double)V / mask_sum);
  TR_CHECK(cudaMemsetAsync(scratch, 0, sizeof(double), s));
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  ddpm_loss_kernel<<<(unsigned)blocks, 256, 0, s>>>(pred, noise, mask, coef, scratch, grad_pred, V, total);
  store_scalar_kernel<<<1, 1, 0, s>>>(scratch, loss_out);
  TR_CHECK(cudaGetLastError());
  TR_API_END
}

int mdb_ddpm_perturb(const float* x0, const float* noise, const float* mask, const float* sqrt_ac, const float* sqrt_1mac,
                     float* out, int B, int C, long long V, void* stream) {
  TR_API_BEGIN
  const long long total = (long long)B * C * V;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  ddpm_perturb_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x0, noise, mask, sqrt_ac, sqrt_1mac, out, V, (long long)C * V, total);
  TR_CHECK(cudaGetLastError());
  TR_API_END
}

int mdb_chunk_elems(void) { return kChunkElems; }

int mdb_grad_clip_coef(const float* const* grads_dev, const long long* numels_dev, const int* chunks_dev, int n_chunks,
                       float max_norm, float* coef_out, float* total_norm_out, double* scratch, void* stream) {
  TR_API_BEGIN
  if (n_chunks < 1) throw std::runtime_error("mdb: empty chunk table");
  cudaStream_t s = (cudaStream_t)stream;
  sq_norm_chunks_kernel<<<n_chunks, kChunkThreads, 0, s>>>(grads_dev, numels_dev, reinterpret_cast<const int2*>(chunks_dev), scratch);
  clip_coef_kernel<<<1, 1024, 0, s>>>(scratch, n_chunks, max_norm, coef_out, total_norm_out);
  TR_CHECK(cudaGetLastError());
  TR_API_END
}

int mdb_adam_ema_step(float* const* params_dev, const float* const* grads_dev, float* const* exp_avg_dev,
                      float* const* exp_avg_sq_dev, float* const* ema_dev, const long long* numels_dev,
                      const int* chunks_dev, int n_chunks, float lr, float beta1, float beta2, float eps,
                      float weight_decay, int step, const float* clip_coef_dev, float ema_decay, void* stream) {
  TR_API_BEGIN
  if (step < 1) throw std::runtime_error("mdb: Adam step counter starts at 1");
  if (n_chunks < 1) throw std::runtime_error("mdb: empty chunk table");
  AdamArgs a{};
  a.params = params_dev; a.grads = grads_dev; a.exp_avg = exp_avg_dev; a.exp_avg_sq = exp_avg_sq_dev; a.ema = ema_dev;
  a.numels = numels_dev; a.chunks = reinterpret_cast<const int2*>(chunks_dev);
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  const double bc1 = 1.0 - pow((double)beta1, step), bc2 = 1.0 - pow((double)beta2, step);
  a.step_size = (float)(lr / bc1);
  a.inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
  a.one_minus_decay = 1.f - ema_decay;
  a.clip_coef = clip_coef_dev;
  if (ema_dev) adam_ema_kernel<true><<<n_chunks, kChunkThreads, 0, (cudaStream_t)stream>>>(a);
  else adam_ema_kernel<false><<<n_chunks, kChunkThreads, 0, (cudaStream_t)stream>>>(a);
  TR_CHECK(cudaGetLastError());
  TR_API_END
}

int mdb_ema_update(float* const* ema_dev, const float* const* params_dev, const long long* numels_dev,
                   const int* chunks_dev, int n_chunks, float ema_decay, void* stream) {
  TR_API_BEGIN
  if (n_chunks < 1) throw std::runtime_error("mdb: empty chunk table");
  ema_kernel<<<n_chunks, kChunkThreads, 0, (cudaStream_t)stream>>>(ema_dev, params_dev, numels_dev,
                                                                     reinterpret_cast<const int2*>(chunks_dev), 1.f - ema_decay);
  TR_CHECK(cudaGetLastError());
  TR_API_END
}

// ---- data-parallel gradient exchange over a caller-owned NCCL communicator. NCCL is resolved at call time from the
// library already loaded in the process (the host created the communicator with it), so this shared object carries no
// link-time dependency on a particular libnccl.
__global__ void scale_kernel(float* p, float f, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] *= f;
}

int mdb_allreduce_grads(void* nccl_comm, float* grads, long long numel, int world_size, void* stream) {
  TR_API_BEGIN
  if (!nccl_comm || world_size < 1) throw std::runtime_error("mdb: mdb_allreduce_grads needs a communicator and its size");
  typedef int (*allreduce_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
  static allreduce_fn fn = nullptr;
  if (!fn) {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) throw std::runtime_error("mdb: libnccl.so.2 is not loadable");
    fn = reinterpret_cast<allreduce_fn>(dlsym(h, "ncclAllReduce"));
    if (!fn) throw std::runtime_error("mdb: ncclAllReduce not found");
  }
  const int ncclFloat32 = 7, ncclSum = 0;  // nccl.h enums (stable since NCCL 2.0)
  const int rc = fn(grads, grads, (size_t)numel, ncclFloat32, ncclSum, nccl_comm, (cudaStream_t)stream);
  if (rc != 0) throw std::runtime_error("mdb: ncclAllReduce failed with code " + std::to_string(rc));
  if (world_size > 1) {
    scale_kernel<<<132 * 8, 256, 0, (cudaStream_t)stream>>>(grads, 1.f / (float)world_size, numel);
    TR_CHECK(cudaGetLastError());
  }
  TR_API_END
}

}  // extern "C"
