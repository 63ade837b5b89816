// wgmma weight-gradient kernel for sm_90a (training path: the dW half of nn.Conv3d / NIN / Linear backward,
// i.e. what autograd computes for the reference's `loss.backward()` in lib/diffusion/losses.py:104-139).
//
//   G[tap][m][n] = sum over positions p of  dY[p][m] * X[p + off(tap)][n]
//
// Both operands are NDHWC activations, so the contraction index (the voxel) is the SLOW axis of both tiles: the tiles
// are fed to the tensor cores as MN-major operands (wgmma descriptors with the 64-channel block stride in LBO and the
// 8-voxel group stride in SBO, transpose flags set) -- no transposed copy of any activation exists. A CTA owns ONE
// (Cout tile, Cin tile, tap) and a contiguous range of voxel tiles; its 128x128 fp32 accumulator stays in registers for
// the whole range -- each consumer warpgroup holds 64 of the 128 rows -- and is written once, as a split-K partial, at the
// end. (One tap per CTA: three taps sharing a halo load of X would need 192 accumulator registers per thread, more than a
// thread can hold next to its addressing.) Partials are summed in a fixed order by wgrad_reduce_kernel (deterministic
// gradients), which also scatters into the reference's OIDHW layout.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (warp 0), warpgroups 1-2 = MMA + drain.
#pragma once
#include "gemm_tc.cuh"

namespace mdb {

constexpr int kWgThreads = 384;
constexpr int kWgStages = 3;
constexpr int kWgYChunkBytes = 128 * kRowBytes;           // 64 channels x 128 voxels
constexpr int kWgStageBytes = 4 * kWgYChunkBytes;         // dY and X: two 64-channel chunks each
constexpr int kWgSmemBytes = 1024 + kWgStages * kWgStageBytes + 2 * kWgStages * 8;
constexpr int kWgMaxGroups = 27;
constexpr int kWgMaxXMaps = 8;

struct WgradGroup {
  int8_t xmap;        // which X tensor map (stride-2 convs: the parity sub-grid of this tap)
  int8_t dx, dy, dz;  // coordinate offset of the X box relative to the dY tile origin
  int8_t tap;         // output tap index
  int8_t pad[3];
};
static_assert(sizeof(WgradGroup) == 8, "WgradGroup must be 8 bytes");

struct WgradParams {
  CUtensorMap ymap;
  CUtensorMap xmap[kWgMaxXMaps];
  WgradGroup groups[kWgMaxGroups];
  int n_groups;
  int bx, by, bz, bb;   // voxel tile (product 128)
  int tx, ty, tz, tb;   // voxel tile counts
  int m_tiles, n_tiles;
  int splits;           // CTAs sharing one (m tile, n tile, group): contiguous ranges of voxel tiles
  int taps;             // taps of the whole operation (partial layout)
  int Mp, Np;           // padded extents (multiples of 128)
  float* partial;       // [splits][taps][Mp][Np]
};

#ifdef MDB_WGRAD_KERNEL_IMPL  // the kernel itself is compiled in wgrad_host.cu only
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStageBytes);
  const uint32_t stage0 = smem_u32(smem);
  const uint32_t full = smem_u32(bars), empty = full + 8 * kWgStages;
  // (broadcast from lane 0, so the compiler can treat the warpgroup branches as warp-uniform)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  // work item of this CTA
  int w = blockIdx.x;
  const int split = w % p.splits; w /= p.splits;
  const int gi = w % p.n_groups; w /= p.n_groups;
  const int nt = w % p.n_tiles;
  const int mt = w / p.n_tiles;
  const WgradGroup grp = p.groups[gi];
  const int tiles = p.tx * p.ty * p.tz * p.tb;
  const int t_lo = (int)((long long)tiles * split / p.splits);
  const int t_hi = (int)((long long)tiles * (split + 1) / p.splits);
  const int m0 = mt * 128, n0 = nt * 128;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.ymap);
    tma_prefetch_desc(&p.xmap[grp.xmap]);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kWgStages; ++i) { mbar_init(full + 8 * i, 1); mbar_init(empty + 8 * i, 2); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<kRegsProducer>();
    if (warp == 0) {
      // ------------------------------------------------------------------ TMA producer
      uint32_t st = 0, ph = 0;
      const uint32_t bytes = kWgStageBytes;
      for (int t = t_lo; t < t_hi; ++t) {
        int r = t;
        const int x0 = (r % p.tx) * p.bx; r /= p.tx;
        const int y0 = (r % p.ty) * p.by; r /= p.ty;
        const int z0 = (r % p.tz) * p.bz; r /= p.tz;
        const int b0 = r * p.bb;
        mbar_wait(empty + 8 * st, ph ^ 1);
        if (elect_one()) {
          const uint32_t bar = full + 8 * st;
          const uint32_t sbase = stage0 + st * kWgStageBytes;
          mbar_expect_tx(bar, bytes);
          tma_load_5d(&p.ymap, bar, sbase, m0, x0, y0, z0, b0);
          tma_load_5d(&p.ymap, bar, sbase + kWgYChunkBytes, m0 + 64, x0, y0, z0, b0);
          const uint32_t xb = sbase + 2 * kWgYChunkBytes;
          tma_load_5d(&p.xmap[grp.xmap], bar, xb, n0, x0 + grp.dx, y0 + grp.dy, z0 + grp.dz, b0);
          tma_load_5d(&p.xmap[grp.xmap], bar, xb + kWgYChunkBytes, n0 + 64, x0 + grp.dx, y0 + grp.dy, z0 + grp.dz, b0);
        }
        __syncwarp();
        if (++st == kWgStages) { st = 0; ph ^= 1; }
      }
    }
  } else {
    setmaxnreg_inc<kRegsConsumer>();
    // ------------------------------------------------------------------ MMA: warpgroup wg owns rows [64*wg, 64*wg + 64)
    const int wg = (warp - 4) >> 2, wt = threadIdx.x & 127;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    uint32_t st = 0, ph = 0;
    int prev = -1;
    for (int t = t_lo; t < t_hi; ++t) {
      mbar_wait(full + 8 * st, ph);
      const uint32_t sbase = stage0 + st * kWgStageBytes;
      // A = this warpgroup's 64-channel dY block (one MN block); B = both 64-channel X blocks, LBO apart
      const uint64_t a0 = make_wgmma_desc(sbase + wg * kWgYChunkBytes, kWgYChunkBytes, 1024);
      const uint64_t b0 = make_wgmma_desc(sbase + 2 * kWgYChunkBytes, kWgYChunkBytes, 1024);
      fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 8; ++c)  // 16 voxels (two 8-row swizzle groups = 2048 B) per instruction
        wgmma_m64n128k16_bf16<1, 1>(acc, a0 + c * 128, b0 + c * 128, 1u);
      wgmma_commit();
      fence_operands(acc);
      wgmma_wait<1>();
      if (prev >= 0 && wt == 0) mbar_arrive(empty + 8 * prev);
      prev = (int)st;
      if (++st == kWgStages) { st = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    fence_operands(acc);
    // ------------------------------------------------------------------ drain: registers -> fp32 partial
    // register 4i+{0,1} = (row l/4, cols 8i + 2(l%4) + {0,1}), 4i+{2,3} = the same columns 8 rows further down
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2), col = 2 * (lane & 3);
    float* dst = p.partial + (((long long)split * p.taps + grp.tap) * p.Mp + m0 + row) * p.Np + n0 + col;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(dst + 8 * p.Np + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
}

#endif  // MDB_WGRAD_KERNEL_IMPL

}  // namespace mdb
