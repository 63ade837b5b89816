#include "elementwise.cuh"
#include "gn_stats.cuh"
#include <curand_kernel.h>
#include <stdexcept>
#include <string>

namespace mdb {

// ------------------------------------------------------------------ GroupNorm apply (+SiLU), concat-aware
// blockIdx.y = sample. Every thread owns ONE 16-byte channel vector for the whole kernel (block = k voxels x C/VEC
// vectors): its scale/shift live in registers, its source pointer is selected once, and the loop body is
// load -> fma -> silu -> store with 4 voxels in flight. No div/mod or table lookups in the loop: the kernel is
// HBM-bound instead of issue-bound.
// X3: a channel vector is a 16-byte hi part and a 16-byte lo part one logical row apart, on the input as on the output.
// GroupNorm finalize is fused into the prologue: each thread derives mean / rstd of the group(s) of ITS channels from the
// per-channel sums the producing GEMM left behind (cpg channels x 2 values, L2-resident) -- 80 fewer launches.
template <Precision P>
__global__ void __launch_bounds__(256, P == kTF32 ? 4 : 3) norm_act_kernel(NormActArgs a, int cv, int k) {
  constexpr int VEC = kVecElems<P>;  // 16 bytes
  constexpr int UNROLL = 4;
  const int C = a.C0 + a.C1;
  const int b = blockIdx.y;
  const int cvi = threadIdx.x % cv, vl = threadIdx.x / cv;
  const int c = cvi * VEC;
  float sc[VEC], sh[VEC];
  {
    const int cpg = C / a.groups;
    int cur_g = -1;
    float mean = 0.f, rstd = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const int ch = c + j, g = ch / cpg;
      if (g != cur_g) {
        cur_g = g;
        gn_group_stats(a.stats0, a.C0, a.stats1, a.C1, b, g, cpg, a.voxels, a.eps, mean, rstd);
      }
      sc[j] = a.gamma[ch] * rstd;
      sh[j] = a.beta[ch] - mean * sc[j];
    }
  }
  const int es = esize(P);
  constexpr int PARTS = P == kBF16X3 ? 2 : 1;
  const bool first = c < a.C0;
  const char* src = first ? (const char*)a.x0 + ((long long)b * a.voxels * a.ld0 * PARTS + c) * es
                          : (const char*)a.x1 + ((long long)b * a.voxels * a.ld1 * PARTS + (c - a.C0)) * es;
  const long long src_stride = (first ? a.ld0 : a.ld1) * es * PARTS;  // bytes per voxel
  const long long src_lo = (first ? a.ld0 : a.ld1) * es;              // X3: hi -> lo distance in bytes
  char* dst = (char*)a.y + ((long long)b * a.voxels * C * PARTS + c) * es;
  const long long dst_stride = (long long)C * es * PARTS;
  const long long dst_lo = (long long)C * es;
  const long long step = (long long)gridDim.x * k;
  for (long long v0 = (long long)blockIdx.x * k + vl; v0 < a.voxels; v0 += step * UNROLL) {
    uint4 raw[UNROLL], rawl[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const long long v = v0 + u * step;
      if (v < a.voxels) {
        raw[u] = __ldg((const uint4*)(src + v * src_stride));
        if constexpr (P == kBF16X3) rawl[u] = __ldg((const uint4*)(src + v * src_stride + src_lo));
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const long long v = v0 + u * step;
      if (v >= a.voxels) continue;
      float x[VEC];
      decode_vec<P>(raw[u], rawl[u], x);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        float y = fmaf(x[j], sc[j], sh[j]);
        if (a.silu) y = P == kBF16 ? silu_tanh(y) : silu_ex2(y);
        x[j] = y;
      }
      if (P != kTF32 && a.drop_thresh > 0)  // training engines (bf16 and split bf16)
        apply_dropout<VEC / 4>(x, a.seed, (unsigned long long)((((long long)b * a.voxels + v) * C + c) >> 2), a.drop_thresh,
                               a.drop_scale);
      store_vec<P>(dst + v * dst_stride, dst_lo, x);
    }
  }
}
void launch_norm_act(const NormActArgs& a, int B, cudaStream_t s) {
  const int vec = a.prec == kTF32 ? 4 : 8;
  const int C = a.C0 + a.C1;
  const int cv = C / vec;
  if (cv > 256 || cv < 1 || a.C0 % vec != 0) throw std::runtime_error("mdb: unsupported channel count in norm_act");
  const int k = 256 / cv;  // voxels per block pass
  const int threads = cv * k;
  long long gx = (a.voxels + (long long)k * 4 - 1) / ((long long)k * 4);
  const long long cap = (132LL * 8 + B - 1) / B;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  dim3 grid((unsigned)gx, (unsigned)B);
  if (a.prec == kTF32) norm_act_kernel<kTF32><<<grid, threads, 0, s>>>(a, cv, k);
  else if (a.prec == kBF16X3) norm_act_kernel<kBF16X3><<<grid, threads, 0, s>>>(a, cv, k);
  else norm_act_kernel<kBF16><<<grid, threads, 0, s>>>(a, cv, k);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ nearest 2x upsample (layers.py:620)
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int B, int Z, int Y, int X, int cv) {
  const long long total = (long long)B * (2 * Z) * (2 * Y) * (2 * X) * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int c = (int)(r % cv); r /= cv;
    const int xo = (int)(r % (2 * X)); r /= (2 * X);
    const int yo = (int)(r % (2 * Y)); r /= (2 * Y);
    const int zo = (int)(r % (2 * Z)); r /= (2 * Z);
    const long long src = ((((long long)r * Z + (zo >> 1)) * Y + (yo >> 1)) * X + (xo >> 1)) * cv + c;
    y[i] = __ldg(x + src);
  }
}
void launch_upsample2x(const void* x, void* y, int B, int Z, int Y, int X, int C, int elem_bytes, cudaStream_t s) {
  const int cv = C * elem_bytes / 16;
  const long long total = (long long)B * 8 * Z * Y * X * cv;
  upsample2x_kernel<<<grid_for(total, 256), 256, 0, s>>>((const uint4*)x, (uint4*)y, B, Z, Y, X, cv);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ stem im2col
// One block per (sample, z, group of YB y-rows): the k x (k+YB-1) input rows it needs are staged in shared memory once
// (a warp per row, no per-element div/mod), then every thread emits 16-byte vectors of the [voxel][Kpad] operand
// matrix (column = cin*k^3 + tap) through a per-column slab-offset table.
constexpr int kIm2colYB = 4;
template <Precision P>  // split bf16: row = [Kpad hi | Kpad lo]
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, void* __restrict__ a, int Cin, int R, int k, int Kpad) {
  constexpr int VEC = kVecElems<P>;
  constexpr int YB = kIm2colYB;
  extern __shared__ float slab[];  // [Cin][k][k+YB-1][R + 2*pad]
  const int pad = k / 2, W = R + 2 * pad, T = k * k * k, KH = k + YB - 1;
  const int yblocks = R / YB;
  const int y0 = (blockIdx.x % yblocks) * YB, z0 = (blockIdx.x / yblocks) % R, b = blockIdx.x / (yblocks * R);
  const long long V = (long long)R * R * R;
  const int n_rows = Cin * k * KH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = warp; row < n_rows; row += 8) {
    const int khh = row % KH, kd = (row / KH) % k, ci = row / (KH * k);
    const int zi = z0 + kd - pad, yi = y0 + khh - pad;
    const bool row_ok = zi >= 0 && zi < R && yi >= 0 && yi < R;
    const float* src = x + ((long long)b * Cin + ci) * V + ((long long)zi * R + yi) * R;
    for (int xw = lane; xw < W; xw += 32) {
      const int xi = xw - pad;
      slab[row * W + xw] = (row_ok && xi >= 0 && xi < R) ? __ldg(src + xi) : 0.f;
    }
  }
  int* coloff = reinterpret_cast<int*>(slab + n_rows * W);
  for (int col = threadIdx.x; col < Kpad; col += blockDim.x) {
    int off = -1;
    if (col < Cin * T) {
      const int ci = col / T, tap = col % T;
      const int kd = tap / (k * k), kh = (tap / k) % k, kw = tap % k;
      off = ((ci * k + kd) * KH + kh) * W + kw;
    }
    coloff[col] = off;
  }
  __syncthreads();
  const int kv = Kpad / VEC;
  for (int yb = 0; yb < YB; ++yb) {
    const long long row0 = (((long long)b * R + z0) * R + y0 + yb) * R;
    const int ybase = yb * W;
    for (int i = threadIdx.x; i < R * kv; i += blockDim.x) {
      const int xo = i / kv, col0 = (i - xo * kv) * VEC;
      float v[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const int off = coloff[col0 + j];
        v[j] = off >= 0 ? slab[off + ybase + xo] : 0.f;
      }
      store_vec<P>((char*)a + ((row0 + xo) * parts(P) * Kpad + col0) * esize(P), (long long)Kpad * esize(P), v);
    }
  }
}
void launch_im2col(const float* x, void* a, int B, int Cin, int R, int k, int Kpad, Precision prec, cudaStream_t s) {
  if (R % kIm2colYB != 0) throw std::runtime_error("mdb: im2col needs a grid size divisible by 4");
  const size_t smem = (size_t)Cin * k * (k + kIm2colYB - 1) * (R + 2 * (k / 2)) * sizeof(float) + (size_t)Kpad * sizeof(int);
  static bool configured[64] = {};  // per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 64 || !configured[dev]) {
    cudaFuncSetAttribute(im2col_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(im2col_kernel<kTF32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(im2col_kernel<kBF16X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    if (dev < 64) configured[dev] = true;
  }
  if (smem > 100 * 1024) throw std::runtime_error("mdb: im2col slab too large");
  const unsigned grid = (unsigned)(B * R * (R / kIm2colYB));
  if (prec == kTF32) im2col_kernel<kTF32><<<grid, 256, smem, s>>>(x, a, Cin, R, k, Kpad);
  else if (prec == kBF16X3) im2col_kernel<kBF16X3><<<grid, 256, smem, s>>>(x, a, Cin, R, k, Kpad);
  else im2col_kernel<kBF16><<<grid, 256, smem, s>>>(x, a, Cin, R, k, Kpad);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ row softmax (layers.py:604)
template <Precision P>  // split bf16: hi parts in the first L bf16 of the row, lo parts in the next L
__global__ void softmax_rows_kernel(float* __restrict__ s, long long rows, int L) {
  __shared__ float red[32];
  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
    float* p = s + row * L;
    float vals[16];  // L <= 16 * blockDim.x; fully unrolled so the array stays in registers
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int i = threadIdx.x + j * 256;
      vals[j] = i < L ? p[i] : -INFINITY;
      m = fmaxf(m, vals[j]);
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
    __syncthreads();
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) { vals[j] = __expf(vals[j] - m); sum += vals[j]; }
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += red[w];
    const float inv = 1.f / sum;
    __syncthreads();  // every thread has consumed its fp32 logits before anyone overwrites the row
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int i = threadIdx.x + j * 256;
      if (i < L) {
        store_split<P>(reinterpret_cast<ActElem<P>*>(p) + i, L, vals[j] * inv);
      }
    }
  }
}
void launch_softmax_rows(float* s, long long rows, int L, Precision prec, cudaStream_t st) {
  if (L > 16 * 256) throw std::runtime_error("mdb: softmax row too long");
  const int grid = (int)(rows < 132LL * 16 ? rows : 132LL * 16);
  if (prec == kTF32) softmax_rows_kernel<kTF32><<<grid, 256, 0, st>>>(s, rows, L);
  else if (prec == kBF16X3) softmax_rows_kernel<kBF16X3><<<grid, 256, 0, st>>>(s, rows, L);
  else softmax_rows_kernel<kBF16><<<grid, 256, 0, st>>>(s, rows, L);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ V transpose: out[b][c][v] = in[b][v][c0+c]
template <typename T>
__global__ void transpose_vc_kernel(const T* __restrict__ in, long long ld, int c0, T* __restrict__ out, int V, int C, long long ldo) {
  __shared__ T tile[32][33];
  const int b = blockIdx.z;
  const int v0 = blockIdx.x * 32, cb = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int v = v0 + j, c = cb + threadIdx.x;
    if (v < V && c < C) tile[j][threadIdx.x] = in[((long long)b * V + v) * ld + c0 + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = cb + j, v = v0 + threadIdx.x;
    if (v < V && c < C) out[((long long)b * C + c) * ldo + v] = tile[threadIdx.x][j];
  }
}
// bf16 fast path: 64x64 tiles, two elements (4 bytes) per thread on both the read and the write side, so every warp
// moves full 128-byte rows (the 32x32 / 2-byte version touched half-used sectors in both directions)
__global__ void __launch_bounds__(256) transpose_vc_bf16x2_kernel(const __nv_bfloat16* __restrict__ in, long long ld, int c0,
                                                                  __nv_bfloat16* __restrict__ out, int V, int C, long long ldo) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int b = blockIdx.z;
  const int v0 = blockIdx.x * 64, cb = blockIdx.y * 64;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int j = ty; j < 64; j += 8) {
    const int v = v0 + j, c = cb + 2 * tx;
    if (v < V && c + 1 < C) {
      const __nv_bfloat162 t = *reinterpret_cast<const __nv_bfloat162*>(in + ((long long)b * V + v) * ld + c0 + c);
      tile[j][2 * tx] = t.x; tile[j][2 * tx + 1] = t.y;
    }
  }
  __syncthreads();
  for (int j = ty; j < 64; j += 8) {
    const int c = cb + j, v = v0 + 2 * tx;
    if (c < C && v + 1 < V) {
      __nv_bfloat162 t;
      t.x = tile[2 * tx][j]; t.y = tile[2 * tx + 1][j];
      *reinterpret_cast<__nv_bfloat162*>(out + ((long long)b * C + c) * ldo + v) = t;
    }
  }
}

void launch_transpose_vc(const void* in, long long ld, int c0, void* out, int B, int V, int C, int elem_bytes, cudaStream_t s,
                         long long ld_out) {
  const long long ldo = ld_out ? ld_out : V;
  if (elem_bytes == 2 && V % 64 == 0 && C % 64 == 0 && ld % 2 == 0 && c0 % 2 == 0 && ldo % 2 == 0) {
    dim3 grid(V / 64, C / 64, B), block(32, 8);
    transpose_vc_bf16x2_kernel<<<grid, block, 0, s>>>((const __nv_bfloat16*)in, ld, c0, (__nv_bfloat16*)out, V, C, ldo);
    MDB_LAUNCH_CHECK();
    return;
  }
  dim3 grid((V + 31) / 32, (C + 31) / 32, B), block(32, 8);
  if (elem_bytes == 4) transpose_vc_kernel<float><<<grid, block, 0, s>>>((const float*)in, ld, c0, (float*)out, V, C, ldo);
  else transpose_vc_kernel<__nv_bfloat16><<<grid, block, 0, s>>>((const __nv_bfloat16*)in, ld, c0, (__nv_bfloat16*)out, V, C, ldo);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ time embedding MLP
// get_timestep_embedding (layers.py:542-556): half = nf/2, freq_k = exp(-ln(1e4) * k / (half-1)), [sin, cos];
// then Linear(nf,4nf) -> SiLU -> Linear(4nf,4nf) (ddpm_res64.py:132-136); ResnetBlockDDPM applies act(temb) before
// Dense_0 (layers.py:680), so act(temb) is what every consumer needs and is what we store.
__global__ void temb_kernel(const float* __restrict__ labels, const float* __restrict__ w0, const float* __restrict__ b0,
                            const float* __restrict__ w1, const float* __restrict__ b1, float* __restrict__ out, int nf) {
  extern __shared__ float sm[];
  float* emb = sm;            // nf
  float* h1 = sm + nf;        // 4nf
  const int b = blockIdx.x;
  const int half = nf / 2;
  const float t = labels[b];
  for (int i = threadIdx.x; i < nf; i += blockDim.x) {
    const int k = i < half ? i : i - half;
    const float coef = logf(10000.f) / (float)(half - 1);
    const float f = expf((float)k * -coef);
    const float arg = t * f;
    emb[i] = i < half ? sinf(arg) : cosf(arg);
  }
  __syncthreads();
  const int H = 4 * nf;
  for (int n = threadIdx.x; n < H; n += blockDim.x) {
    float acc = b0[n];
    for (int k = 0; k < nf; ++k) acc += w0[(long long)n * nf + k] * emb[k];
    h1[n] = silu_ex2(acc);
  }
  __syncthreads();
  for (int n = threadIdx.x; n < H; n += blockDim.x) {
    float acc = b1[n];
    for (int k = 0; k < H; ++k) acc += w1[(long long)n * H + k] * h1[k];
    out[(long long)b * H + n] = silu_ex2(acc);
  }
}
void launch_temb(const float* labels, const float* w0, const float* b0, const float* w1, const float* b1, float* out,
                 int B, int nf, cudaStream_t s) {
  temb_kernel<<<B, 256, 5 * nf * sizeof(float), s>>>(labels, w0, b0, w1, b1, out, nf);
  MDB_LAUNCH_CHECK();
}

__global__ void dense_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                             float* __restrict__ out, int B, int K, int N) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int o = warp; o < B * N; o += nwarps) {
    const int b = o / N, n = o % N;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc += w[(long long)n * K + k] * x[(long long)b * K + k];
    for (int s = 16; s; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if (lane == 0) out[(long long)b * N + n] = acc + bias[n];
  }
}
void launch_dense(const float* x, const float* w, const float* bias, float* out, int B, int K, int N, cudaStream_t s) {
  dense_kernel<<<grid_for((long long)B * N * 32, 256), 256, 0, s>>>(x, w, bias, out, B, K, N);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ head conv phase 2: tap shift-sum (Cout == 4)
template <bool PFP32>
__global__ void __launch_bounds__(256) tap_shift_sum_kernel(const void* __restrict__ P, long long ldp, const float* __restrict__ bias,
                                                           float* __restrict__ out, int R, int k) {
  const int pad = k / 2;
  const long long V = (long long)R * R * R;
  const int b = blockIdx.y;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % R), y = (int)((v / R) % R), z = (int)(v / ((long long)R * R));
    float acc0 = bias[0], acc1 = bias[1], acc2 = bias[2], acc3 = bias[3];
    int tap = 0;
    for (int dz = -pad; dz <= pad; ++dz)
      for (int dy = -pad; dy <= pad; ++dy)
        for (int dx = -pad; dx <= pad; ++dx, ++tap) {
          const int zz = z + dz, yy = y + dy, xx = x + dx;
          if ((unsigned)zz >= (unsigned)R || (unsigned)yy >= (unsigned)R || (unsigned)xx >= (unsigned)R) continue;
          const long long row = ((long long)b * V + ((long long)zz * R + yy) * R + xx) * ldp + tap * 4;
          if (PFP32) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(P) + row));
            acc0 += t.x; acc1 += t.y; acc2 += t.z; acc3 += t.w;
          } else {
            const uint2 t = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(P) + row));
            const float2 f0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
            const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
            acc0 += f0.x; acc1 += f0.y; acc2 += f1.x; acc3 += f1.y;
          }
        }
    float* o = out + (long long)b * 4 * V + v;
    o[0] = acc0; o[V] = acc1; o[2 * V] = acc2; o[3 * V] = acc3;
  }
}
void launch_tap_shift_sum(const void* P, long long ldp, int p_fp32, const float* bias, float* out, int B, int R, int k,
                          int Cout, cudaStream_t s) {
  if (Cout != 4) throw std::runtime_error("mdb: tap_shift_sum supports 4 output channels");
  const long long V = (long long)R * R * R;
  long long gx = (V + 255) / 256;
  const long long cap = (132LL * 16 + B - 1) / B;
  if (gx > cap) gx = cap;
  dim3 grid((unsigned)gx, (unsigned)B);
  if (p_fp32) tap_shift_sum_kernel<true><<<grid, 256, 0, s>>>(P, ldp, bias, out, R, k);
  else tap_shift_sum_kernel<false><<<grid, 256, 0, s>>>(P, ldp, bias, out, R, k);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ split-K reduction
// blockIdx.y = sample, blockIdx.x = chunk of voxels; thread = output channel (coalesced rows). Each thread owns a
// channel for its chunk, so its statistics are accumulated in a fixed order (deterministic) and published with one
// integer atomic per (block, channel).
template <Precision P>  // split bf16: out / res rows are [N hi | N lo]
__global__ void __launch_bounds__(256) split_reduce_kernel(SplitReduceArgs a, int vchunk) {
  const int b = blockIdx.y;
  const long long v0 = (long long)blockIdx.x * vchunk;
  const long long v1 = v0 + vchunk < a.voxels ? v0 + vchunk : a.voxels;
  for (int n = threadIdx.x; n < a.N; n += blockDim.x) {
    float add = a.bias ? a.bias[n] : 0.f;
    if (a.rowbias) add += a.rowbias[(long long)b * a.rowbias_ld + n];
    float s1 = 0.f, s2 = 0.f;
    for (long long v = v0; v < v1; ++v) {
      const long long idx = ((long long)b * a.voxels + v) * a.N + n;
      float acc = add;
      for (int sp = 0; sp < a.splits; ++sp) acc += a.partial[sp * a.split_stride + idx];
      if (a.res)
        acc += load_split<P>((const ActElem<P>*)a.res + parts(P) * ((long long)b * a.res_batch_stride + v * a.N) + n, a.N);
      s1 += acc; s2 += acc * acc;
      store_split<P>((ActElem<P>*)a.out + parts(P) * (idx - n) + n, a.N, acc);
    }
    if (a.stats) {
      long long* dst = a.stats + ((long long)b * a.N + n) * kStatWords;
      stat_add(dst, s1);
      stat_add(dst + 2, s2);
    }
  }
}
void launch_split_reduce(const SplitReduceArgs& a, int B, cudaStream_t s) {
  const int vchunk = 8;
  dim3 grid((unsigned)((a.voxels + vchunk - 1) / vchunk), (unsigned)B);
  const int threads = a.N < 256 ? ((a.N + 31) / 32) * 32 : 256;
  if (a.prec == kTF32) split_reduce_kernel<kTF32><<<grid, threads, 0, s>>>(a, vchunk);
  else if (a.prec == kBF16X3) split_reduce_kernel<kBF16X3><<<grid, threads, 0, s>>>(a, vchunk);
  else split_reduce_kernel<kBF16><<<grid, threads, 0, s>>>(a, vchunk);
  MDB_LAUNCH_CHECK();
}

__global__ void add_vec_kernel(const float* a, const float* b, float* out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = a[i] + (b ? b[i] : 0.f);
}
void launch_add_vec(const float* a, const float* b, float* out, int n, cudaStream_t s) {
  add_vec_kernel<<<grid_for(n, 256), 256, 0, s>>>(a, b, out, n);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ sub-pixel upsample-conv weights
__global__ void upconv_weights_kernel(const float* __restrict__ w, float* __restrict__ w8, long long pairs) {
  const long long total = pairs * 64;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i & 7), par = (int)((i >> 3) & 7);
    const long long oc = i >> 6;  // (co, ci) pair
    const int ez = e >> 2, ey = (e >> 1) & 1, ex = e & 1;
    const int pz = par >> 2, py = (par >> 1) & 1, px = par & 1;
    // original taps folded into effective tap (parity q, e): q=0: e0 <- {0}, e1 <- {1,2}; q=1: e0 <- {0,1}, e1 <- {2}
    auto lo = [](int q, int t) { return q == 0 ? (t == 0 ? 0 : 1) : (t == 0 ? 0 : 2); };
    auto hi = [](int q, int t) { return q == 0 ? (t == 0 ? 0 : 2) : (t == 0 ? 1 : 2); };
    float acc = 0.f;
    for (int dz = lo(pz, ez); dz <= hi(pz, ez); ++dz)
      for (int dy = lo(py, ey); dy <= hi(py, ey); ++dy)
        for (int dx = lo(px, ex); dx <= hi(px, ex); ++dx) acc += w[oc * 27 + (dz * 3 + dy) * 3 + dx];
    w8[((long long)par * pairs + oc) * 8 + e] = acc;
  }
}
void launch_upconv_weights(const float* w, float* w8, int Cout, int Cin, cudaStream_t s) {
  const long long pairs = (long long)Cout * Cin;
  upconv_weights_kernel<<<grid_for(pairs * 64, 256), 256, 0, s>>>(w, w8, pairs);
  MDB_LAUNCH_CHECK();
}

// ------------------------------------------------------------------ ancestral sampling update
// Same operation order as the reference's eager fp32 ops (no FMA contraction) so that, given identical eps and
// noise, x and x_mean are bit-identical: score = -eps/std; x_mean = (x + beta*score)/sqrt(1-beta);
// x = x_mean + sqrt(beta)*z; both multiplied by grid_mask (sampling.py:222-230, 476-478).
__global__ void sampler_update_kernel(SamplerUpdateArgs a, int B, float sqrt_1m_beta, float sqrt_beta, float stdv) {
  const long long per = a.V * a.C;
  const long long total = per * B;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long v = i % a.V;
    const float m = __ldg(a.mask + v);
    const float score = __fdiv_rn(-a.eps[i], stdv);
    const float xm = __fdiv_rn(__fadd_rn(a.x[i], __fmul_rn(a.beta, score)), sqrt_1m_beta);
    float z;
    if (a.noise) {
      z = a.noise[i];
    } else {
      curandStatePhilox4_32_10_t st;
      curand_init(a.seed, (unsigned long long)i, a.offset, &st);
      z = curand_normal(&st);
    }
    const float xn = __fadd_rn(xm, __fmul_rn(sqrt_beta, z));
    float xo = __fmul_rn(xn, m), xmo = __fmul_rn(xm, m);
    if (a.cond_partial) {
      const long long bc = i / a.V;
      const int ch = (int)(bc % a.C);
      if (ch == a.cond_channel) {
        const long long b = bc / a.C;
        const float pm = __ldg(a.cond_pmask + b * a.cond_pmask_bs + v);
        const float pv = __ldg(a.cond_partial + b * a.cond_partial_bs + v);
        const float keep = __fsub_rn(1.f, pm);
        const float x1 = __fmul_rn(__fadd_rn(__fmul_rn(xo, keep), __fmul_rn(pv, pm)), m);
        float z2;
        if (a.cond_noise) {
          z2 = a.cond_noise[b * a.V + v];
        } else {
          curandStatePhilox4_32_10_t st;
          curand_init(a.seed, (unsigned long long)i, a.offset + 2, &st);
          z2 = curand_normal(&st);
        }
        const float sampled = __fadd_rn(__fmul_rn(a.cond_coef, x1), __fmul_rn(a.cond_std, z2));
        xo = __fmul_rn(__fadd_rn(__fmul_rn(x1, keep), __fmul_rn(sampled, pm)), m);
        xmo = xo;
      }
    }
    a.x[i] = xo;
    a.x_mean[i] = xmo;
  }
}
void launch_sampler_update(const SamplerUpdateArgs& a, int B, cudaStream_t s) {
  const float one_m = 1.f - a.beta;
  const float sq1m = sqrtf(one_m), sqb = sqrtf(a.beta);
  sampler_update_kernel<<<grid_for(a.V * a.C * B, 256), 256, 0, s>>>(a, B, sq1m, sqb, a.stdv);
  MDB_LAUNCH_CHECK();
}

}  // namespace mdb
