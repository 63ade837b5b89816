// Decisions every kernel that reads or writes activations must share bit for bit: the operand mode and its row format,
// the dropout mask, the SiLU forms, and the launch plumbing of the bandwidth kernels. Forward and backward, the fused
// GEMM epilogues and the two-pass kernels all call these definitions, so they cannot drift apart.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <cmath>
#include <stdexcept>
#include <string>
#include <type_traits>

namespace mdb {

// ------------------------------------------------------------------ operand mode and row format
// kBF16X3 ("split bf16"): every fp32 value v is carried as a bf16 pair hi = bf16(v), lo = bf16(v - hi) and every product
// is evaluated as hi*hi + hi*lo + lo*hi into the same fp32 accumulator (three bf16 MMAs per k-step; the
// dropped lo*lo term is 2^-16 relative) -- fp32-class results (the mode that meets the 1e-3 parity contract) at
// one third of the bf16 tensor rate. An X3 tensor with a logical row pitch of `ld` channels occupies 2*ld bf16 per
// voxel: hi parts at [0, ld), lo parts at [ld, 2*ld). All pitches handed to GemmOp / Act and to the launchers stay
// LOGICAL. kTF32 tensors are fp32, rounded to tf32 (rna) wherever a kernel stores an operand: tensor cores truncate fp32
// inputs to 10 mantissa bits, and rounding to nearest instead removes that systematic bias (full res64 net: rel-L2 vs
// fp32 2.5e-3 -> 1.5e-3).
enum Precision { kBF16 = 0, kTF32 = 1, kBF16X3 = 2 };
constexpr int esize(Precision p) { return p == kTF32 ? 4 : 2; }
constexpr int parts(Precision p) { return p == kBF16X3 ? 2 : 1; }
inline Precision precision_from_int(int v) {
  if (v < 0 || v > 2) throw std::runtime_error("mdb: precision must be 0 (bf16), 1 (tf32) or 2 (bf16x3)");
  return static_cast<Precision>(v);
}

__device__ __forceinline__ float to_tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// element type of an activation tensor in mode P
template <Precision P> using ActElem = std::conditional_t<P == kTF32, float, __nv_bfloat16>;
// scalar load / store in the activation format of mode P: tf32 (rounded on store) and bf16 ignore lo_off, split bf16 has
// its lo part lo_off elements behind the hi part
template <Precision P>
__device__ __forceinline__ float load_split(const ActElem<P>* hi, long long lo_off) {
  if constexpr (P == kTF32) {
    return hi[0];
  } else {
    float x = __bfloat162float(hi[0]);
    if constexpr (P == kBF16X3) x += __bfloat162float(hi[lo_off]);
    return x;
  }
}
template <Precision P>
__device__ __forceinline__ void store_split(ActElem<P>* hi, long long lo_off, float v) {
  if constexpr (P == kTF32) {
    hi[0] = to_tf32_rna(v);
  } else {
    const __nv_bfloat16 hb = __float2bfloat16(v);
    hi[0] = hb;
    if constexpr (P == kBF16X3) hi[lo_off] = __float2bfloat16(v - __bfloat162float(hb));  // what the bf16 rounding lost
  }
}

// 8 bf16 in a 16-byte vector
__device__ __forceinline__ void bf16x8_decode(const uint4& raw, float* x) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); x[2 * j] = f.x; x[2 * j + 1] = f.y; }
}
__device__ __forceinline__ void bf16x8_decode_add(const uint4& raw, float* x) {
  float l[8];
  bf16x8_decode(raw, l);
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] += l[j];
}
__device__ __forceinline__ uint4 bf16x8_encode(const float* x) {
  uint4 t;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(x[2 * j], x[2 * j + 1]);
  return t;
}
// lo vector of a split store whose hi vector is `hi` (= bf16x8_encode(x))
__device__ __forceinline__ uint4 bf16x8_encode_lo(const uint4& hi, const float* x) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&hi);
  uint4 t;
  __nv_bfloat162* l = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __bfloat1622float2(h[j]);
    l[j] = __floats2bfloat162_rn(x[2 * j] - f.x, x[2 * j + 1] - f.y);
  }
  return t;
}

// One 16-byte row vector in mode P: 4 fp32 (kTF32) or 8 bf16 values; X3 adds the lo vector lo_bytes after the hi one.
template <Precision P> constexpr int kVecElems = P == kTF32 ? 4 : 8;
// decode of vectors the kernel has already loaded (`lo` is ignored unless X3)
template <Precision P>
__device__ __forceinline__ void decode_vec(const uint4& hi, const uint4& lo, float* x) {
  if constexpr (P == kTF32) {
    x[0] = __uint_as_float(hi.x); x[1] = __uint_as_float(hi.y); x[2] = __uint_as_float(hi.z); x[3] = __uint_as_float(hi.w);
  } else {
    bf16x8_decode(hi, x);
    if constexpr (P == kBF16X3) bf16x8_decode_add(lo, x);
  }
}
template <Precision P>
__device__ __forceinline__ void load_vec(const void* hi, long long lo_bytes, float* x) {
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi));
  uint4 l = h;
  if constexpr (P == kBF16X3) l = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(hi) + lo_bytes));
  decode_vec<P>(h, l, x);
}
template <Precision P>
__device__ __forceinline__ void store_vec(void* hi, long long lo_bytes, const float* x) {
  if constexpr (P == kTF32) {
    *reinterpret_cast<float4*>(hi) = make_float4(to_tf32_rna(x[0]), to_tf32_rna(x[1]), to_tf32_rna(x[2]), to_tf32_rna(x[3]));
  } else {
    const uint4 h = bf16x8_encode(x);
    *reinterpret_cast<uint4*>(hi) = h;
    if constexpr (P == kBF16X3) *reinterpret_cast<uint4*>(reinterpret_cast<char*>(hi) + lo_bytes) = bf16x8_encode_lo(h, x);
  }
}

// ------------------------------------------------------------------ dropout mask
// nn.Dropout after a GroupNorm(+SiLU) (layers.py:661,682). Element e = ((b*V + voxel)*C + channel) is kept iff the 16-bit
// field e%4 of drop_hash64(seed, e/4) is >= thresh, and a kept value is scaled by 1/(1-p). The forward GroupNorm-apply
// kernel, the two-pass GroupNorm backward and the GroupNorm-backward GEMM epilogue all draw the mask from here.
__device__ __forceinline__ unsigned long long drop_hash64(unsigned long long seed, unsigned long long idx) {
  unsigned long long z = idx + seed * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// x[j], j < 4*K: the elements 4*e4 + j
template <int K>
__device__ __forceinline__ void apply_dropout(float* x, unsigned long long seed, unsigned long long e4, int thresh, float scale) {
  unsigned long long h[K];
#pragma unroll
  for (int i = 0; i < K; ++i) h[i] = drop_hash64(seed, e4 + i);
#pragma unroll
  for (int j = 0; j < 4 * K; ++j) {
    const unsigned r16 = (unsigned)((h[j >> 2] >> (16 * (j & 3))) & 0xFFFFu);
    x[j] = r16 >= (unsigned)thresh ? x[j] * scale : 0.f;
  }
}
// host side: probability -> (threshold, scale), and the seed of dropout layer `layer` (each layer draws its own mask)
struct DropoutParams { int thresh; float scale; };
inline DropoutParams dropout_params(float p) { return {(int)std::lround((double)p * 65536.0), p > 0.f ? 1.f / (1.f - p) : 1.f}; }
inline unsigned long long dropout_layer_seed(unsigned long long seed, int layer) {
  return seed + 0x632BE59BD9B4E019ull * (unsigned long long)(layer + 1);
}

// ------------------------------------------------------------------ SiLU
// sigmoid(x) = 1 / (1 + 2^(-x log2 e)) as ex2.approx + rcp.approx (~2^-22 each; the IEEE division and __frcp_rn expand to
// a MUFU plus Newton steps -- ncu showed the bf16x3 GroupNorm pass issue-bound at 32 instructions per element with them,
// profiles/r02_ncu_norm_act_x3.txt). The tf32 / split-bf16 forward, the time embedding and the split-bf16 backward use it.
__device__ __forceinline__ float sigmoid_ex2(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return r;
}
__device__ __forceinline__ float silu_ex2(float x) { return x * sigmoid_ex2(x); }
// silu'(y) = s (1 + y (1 - s)), s = sigmoid(y) -- tanh.approx's 2^-11 error alone would cap the split-bf16 gradient
// accuracy near 5e-4
__device__ __forceinline__ float dsilu_ex2(float y) {
  const float s = sigmoid_ex2(y);
  return s * fmaf(y, 1.f - s, 1.f);
}
// silu'(2h) in the instruction form of the split-bf16 GroupNorm-backward GEMM epilogue: the same value as dsilu_ex2(2h)
// (the constant is exactly 2 float(log2 e)), but ptxas schedules that form differently inside the register-tuned kernel
__device__ __forceinline__ float dsilu_ex2_half(float h) {
  float e, s;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(h * -2.8853900817779268f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(s) : "f"(1.f + e));
  return s * fmaf(2.f * h, 1.f - s, 1.f);
}
// x*sigmoid(x) = 0.5x(1 + tanh(x/2)) with the single-MUFU tanh.approx (rel. error 2^-11: below bf16 resolution);
// halves the MUFU pressure of the bf16 GroupNorm+SiLU pass, which otherwise co-limits with HBM bandwidth.
__device__ __forceinline__ float silu_tanh(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  const float h = 0.5f * x;
  return fmaf(h, t, h);
}
// bf16 backward: silu'(y) from h = y/2 as t + 0.5*h*q with t = (1 + tanh h)/2, q = 1 - tanh^2 h
__device__ __forceinline__ float dsilu_tanh_half(float h) {
  float th;
  asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(h));
  return fmaf(0.5f, h * fmaf(-th, th, 1.f), fmaf(0.5f, th, 0.5f));
}
// IEEE-division form of the time-embedding backward
__device__ __forceinline__ float sigmoid_expf(float x) { return 1.f / (1.f + __expf(-x)); }

// ------------------------------------------------------------------ launch plumbing of the bandwidth kernels
#define MDB_LAUNCH_CHECK()                                                                              \
  do {                                                                                                  \
    cudaError_t _e = cudaGetLastError();                                                                \
    if (_e != cudaSuccess) throw std::runtime_error(std::string("mdb launch: ") + cudaGetErrorString(_e)); \
  } while (0)

// grid-stride launches: at most 8 blocks per SM of the H100 SXM's 132
inline int grid_for(long long work_items, int threads) {
  long long b = (work_items + threads - 1) / threads;
  const long long cap = 132LL * 8;
  if (b > cap) b = cap;
  return b < 1 ? 1 : (int)b;
}

}  // namespace mdb
