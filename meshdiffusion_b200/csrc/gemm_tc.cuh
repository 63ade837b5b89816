// Persistent, warp-specialised wgmma implicit-GEMM kernel for sm_90a.
//
// One kernel serves every dense contraction on the score-network path (reference: nn.Conv3d call sites
// lib/diffusion/models/layers.py:118-132, NIN layers.py:573-582, attention einsums layers.py:602-606):
//
//   D[m, n] = alpha * sum_{k-steps} A_step[m, :] . B[n, kcol(step) : +KB]  (+ bias, + per-sample bias, + residual)
//
// * M indexes output voxels. An M-tile is a (bx,by,bz,bb) box of 128 voxels of the NDHWC activation tensor.
//   A tiles are fetched by TMA straight from the activation tensor as shifted 5-D boxes (zero-filled out of
//   bounds) -- no im2col buffer exists anywhere.  One A load may carry a halo along the slowest box axis so that
//   several filter taps (k-steps) reuse the same shared-memory tile through an advanced wgmma descriptor.
// * B is the packed weight matrix [N][Ktot] (K-major) whose K order is exactly the k-step order of the load
//   table, fetched by TMA as (KB x BLOCK_N) tiles.
// * Accumulators live in registers: each of the two consumer warpgroups owns 64 rows of the tile (wgmma m64nNk16 /
//   m64nNk8). After the last k-step they are staged through shared memory, and the same 256 threads read them back one
//   row per thread to add bias / time-embedding bias / residual, store NDHWC output and reduce per-(sample, channel)
//   sum and sum-of-squares for the GroupNorm that follows (warp-shuffle butterfly + shared + one atomic per channel).
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (warp 0), warpgroups 1-2 = MMA + epilogue.
#pragma once
#include "ptx.cuh"
#include "gn_stats.cuh"

namespace mdb {

constexpr int kBlockM = 128;
constexpr int kRowBytes = 128;                       // bytes of K per row per k-step (one 128B swizzle atom)
constexpr int kAStageRows = 160;                     // 128 + up to 32 halo rows (5-tap reuse)
constexpr int kAStageBytes = kAStageRows * kRowBytes;  // 20480, multiple of 1024
constexpr int kMaxLoads = 2048;
constexpr int kMaxAMaps = 16;  // X3 doubles the maps (hi + lo parts): 8 parity sub-grids x 2
constexpr int kGemmThreads = 384;   // producer warpgroup + 2 MMA / epilogue warpgroups
constexpr int kEpiThreads = 256;

struct __align__(16) LoadEntry {
  uint8_t tmap;   // index of the A tensor map
  uint8_t nk;     // k-steps that reuse this A load
  uint8_t rows;   // rows in the A box (128 or 144)
  uint8_t jrows;  // smem row advance between consecutive k-steps of this load
  int8_t dx, dy, dz;  // coordinate offsets added to the tile origin
  uint8_t wsrc;   // (weight packer) source weight tensor
  uint16_t c0;    // channel coordinate in the A tensor
  uint16_t wc0;   // (weight packer) input-channel offset in the weight tensor; with GemmParams::b_explicit_k the
                  // K coordinate of this entry's first B tile (activation-B operands of the X3 mode)
  uint8_t tap0;   // (weight packer) tap index of k-step 0
  uint8_t tapj;   // (weight packer) tap increment per k-step
  uint16_t wpart; // (weight packer, X3) 0 = hi part bf16(w), 1 = lo part bf16(w - hi)
};
static_assert(sizeof(LoadEntry) == 16, "LoadEntry must be 16 bytes");

// A run of identical pipeline groups. One group = one shared-memory stage = one full/empty mbarrier pair:
// one A box and the nk weight tiles it is multiplied with. All fields are
// warp-uniform kernel parameters, so the MMA warp's control flow and descriptor arithmetic never touch memory.
struct GemmSeg {
  int n_groups;
  int nk;        // k-steps per entry
  int a_bytes;   // bytes of one A box (rows * 128) -- the TMA transaction size
  int a_stride;  // distance between the group's A boxes in the stage (multiple of 1024)
  int jbytes;    // A-descriptor advance between the k-steps of one entry (halo reuse)
};
constexpr int kMaxSegs = 8;

struct GemmParams {
  CUtensorMap amap[kMaxAMaps];
  CUtensorMap bmap;
  const LoadEntry* loads;
  int n_loads;
  int n_segs;
  GemmSeg segs[kMaxSegs];
  int bx, by, bz, bb;  // M-tile box (product 128)
  int X, Y, Z, Bn;     // output extents
  int tx, ty, tz, tb;  // tile counts per axis
  int n_tiles_n;
  int N;               // valid output columns
  int b_batched;       // B tensor map has a batch coordinate following the tile's sample
  int splits;          // split-K: each tile's group sequence is cut into `splits` ranges handled by different CTAs
  int total_groups;    // sum of segs[].n_groups
  float* partial;      // [splits][same layout as out] fp32 partial sums (splits > 1)
  long long split_stride;
  int batch_fastest;   // enumerate the batch axis first among M-tiles (residual shared by all samples stays in L2)
  int kb_elems;        // K elements per k-step (64 bf16 / 32 tf32)
  int b_explicit_k;    // B tile K coordinates come from LoadEntry::wc0 instead of the running k column
  int n_stages, stage_bytes;  // shared-memory operand ring: as many stages as fit next to the epilogue scratch
  // X3 (split bf16) epilogue: the lo parts of the output / residual rows sit this many elements behind the hi parts
  long long out_lo_off, res_lo_off;
  // epilogue
  void* out;
  long long osx, osy, osz, osb;  // output element strides per voxel axis
  long long ocs;                 // output column stride (1 = channels contiguous; else scalar store path)
  int out_fp32;
  int round_out;  // TF32 operands: round stored activations to tf32 (rna) so downstream MMAs do not truncate them
  const float* bias;
  int bias_on_m;
  const float* rowbias;  // [Bn][rowbias_ld] per-sample bias (time embedding projection) or null
  long long rowbias_ld;
  const void* res;       // residual, same dtype as activations unless res_fp32
  long long rsx, rsy, rsz, rsb;
  int res_fp32;
  float alpha;
  long long* stats;  // [Bn][N][kStatWords] (sum, sum of squares) as split fixed-point integers (gn_stats.cuh) or null
  // ---- GroupNorm-backward fusion (GNB instantiations; training data gradients). The accumulator is dL/da of a
  // GroupNorm(+SiLU)(+dropout) output a = drop(act(gamma*xhat+beta)); `res` holds the GroupNorm INPUT x (columns
  // >= res_c0 come from res1: the second source of a channel concatenation). The epilogue stores
  // dy = da*drop*act'(y) and per-tile column partials of (sum dy, sum dy*xhat) for the GroupNorm backward.
  const void* res1;
  long long r1sx, r1sy, r1sz, r1sb;
  int res_c0;
  const float4* gnb_c;  // [Bn][N] {hsc, hsh, rs, nm}: y/2 = x*hsc + hsh, xhat = x*rs + nm
  int gnb_silu;
  int gnb_drop_thresh; float gnb_drop_scale; unsigned long long gnb_seed;
  float* gnb_part;      // [tiles_m * bb][N][2]
};

constexpr int kMaxStages = 6;
constexpr int kMaxDynSmem = 232448;  // 227 KB: the opt-in limit of dynamic shared memory per block on sm_90
template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kBTileBytes = BLOCK_N * kRowBytes;  // weight tile bytes per k-step
  static constexpr int kStatsFloats = 24 * BLOCK_N;  // 2 x [4 warps][sum,sumsq][N] column partials + 2 x [4 segs][N] bias
  // accumulator staging [128 rows][kAccPitch]: the 4-float pad keeps the row-per-lane float4 reads conflict-free
  static constexpr int kAccPitch = BLOCK_N + 4;
  static constexpr int kAccFloats = kBlockM * kAccPitch;
  // everything but the operand ring: alignment slack, accumulator staging, epilogue scratch, mbarriers (kMaxStages)
  static constexpr int kFixedBytes = 1024 + kAccFloats * 4 + kStatsFloats * 4 + 2 * kMaxStages * 8;
};
constexpr int kRegsProducer = 40, kRegsConsumer = 232;  // 128 x 40 + 256 x 232 <= 65 536

// dropout hash shared with the GroupNorm kernels (backward.cuh::drop_hash64)
__device__ __forceinline__ unsigned long long gn_drop_hash64(unsigned long long seed, unsigned long long idx) {
  unsigned long long z = idx + seed * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// K-major 128B-swizzled operand at `saddr` (SBO = 1024 B)
__device__ __forceinline__ uint64_t kdesc(uint32_t saddr) { return make_wgmma_desc(saddr, 16, 1024); }

// GNB: GroupNorm-backward epilogue (see GemmParams::gnb_c) -- a separate instantiation, so the inference kernels'
// code is untouched.
// X3: split-bf16 operands (see Precision::kBF16X3): the main loop is unchanged (the three partial products are extra
// k-steps of the load table); the epilogue reads residuals and stores outputs as (hi, lo) bf16 pairs.
template <int BLOCK_N, bool TF32, bool GNB = false, bool X3 = false>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  using Cfg = GemmCfg<BLOCK_N>;
  const int NS = p.n_stages;
  const uint32_t kStageBytesRt = (uint32_t)p.stage_bytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* s_acc = reinterpret_cast<float*>(smem + NS * p.stage_bytes);
  float* s_stats = s_acc + Cfg::kAccFloats;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stats + Cfg::kStatsFloats);

  const uint32_t stage0 = smem_u32(smem);
  const uint32_t full = smem_u32(bars), empty = full + 8 * kMaxStages;

  // (broadcast from lane 0, so the compiler can treat the warpgroup branches as warp-uniform)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < kMaxAMaps; ++i) tma_prefetch_desc(&p.amap[i]);
    tma_prefetch_desc(&p.bmap);
  }
  if (warp == 1 && lane == 0) {
    // full: the producer's expect_tx arrival; empty: one arrival per consumer warpgroup
    for (int i = 0; i < NS; ++i) { mbar_init(full + 8 * i, 1); mbar_init(empty + 8 * i, 2); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  const int tiles_m = p.tx * p.ty * p.tz * p.tb;
  const int splits = p.splits > 1 ? p.splits : 1;
  const int total_tiles = tiles_m * p.n_tiles_n * splits;
  const int first_tile = (int)blockIdx.x;
  const int tile_step = (int)gridDim.x;

  // split-K range of a work item: groups [lo, hi) of the tile's group sequence
  auto split_range = [&](int item, int& lo, int& hi) {
    const int sidx = item % splits;
    lo = (int)((long long)p.total_groups * sidx / splits);
    hi = (int)((long long)p.total_groups * (sidx + 1) / splits);
  };
  int mt_of_tile = 0;  // M-tile index of the last decoded work item (GNB partial rows)
  auto decode = [&](int tile, int& x0, int& y0, int& z0, int& b0, int& n0) {
    tile /= splits;
    int nt = tile % p.n_tiles_n;
    int mt = tile / p.n_tiles_n;
    mt_of_tile = mt;
    n0 = nt * BLOCK_N;
    int bt = 0;
    if (p.batch_fastest) { bt = mt % p.tb; mt /= p.tb; }
    int xt = mt % p.tx; mt /= p.tx;
    int yt = mt % p.ty; mt /= p.ty;
    int zt = mt % p.tz; mt /= p.tz;
    if (!p.batch_fastest) bt = mt;
    x0 = xt * p.bx; y0 = yt * p.by; z0 = zt * p.bz; b0 = bt * p.bb;
  };

  if (warp < 4) {
    setmaxnreg_dec<kRegsProducer>();
    if (warp == 0) {
      // ------------------------------------------------------------------ TMA producer
      uint32_t st = 0, ph = 0;
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        int x0, y0, z0, b0, n0;
        decode(tile, x0, y0, z0, b0, n0);
        int kcol = 0, l = 0, gi = 0, g_lo, g_hi;
        split_range(tile, g_lo, g_hi);
        const int bcoord = p.b_batched ? b0 : 0;
        for (int sg = 0; sg < p.n_segs; ++sg) {
          const GemmSeg& seg = p.segs[sg];
          const uint32_t group_bytes = seg.a_bytes + seg.nk * Cfg::kBTileBytes;
          for (int g = 0; g < seg.n_groups; ++g, ++gi) {
            if (gi < g_lo || gi >= g_hi) {  // another CTA's share of this tile's K range
              kcol += seg.nk * p.kb_elems;
              ++l;
              continue;
            }
            // the table entry of this group is fetched before blocking on the stage
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(p.loads + l));
            mbar_wait(empty + 8 * st, ph ^ 1);
            if (elect_one()) {
              const uint32_t sbase = stage0 + st * kStageBytesRt;
              int kc = kcol;
              const uint32_t bar = full + 8 * st;
              mbar_expect_tx(bar, group_bytes);
              const LoadEntry& en = reinterpret_cast<const LoadEntry&>(raw);
              if (X3 && p.b_explicit_k) kc = en.wc0;
              tma_load_5d(&p.amap[en.tmap], bar, sbase, en.c0, x0 + en.dx, y0 + en.dy, z0 + en.dz, b0);
              for (int j = 0; j < seg.nk; ++j) {
                tma_load_3d(&p.bmap, bar, sbase + seg.a_stride + j * Cfg::kBTileBytes, kc, n0, bcoord);
                kc += p.kb_elems;
              }
            }
            __syncwarp();
            kcol += seg.nk * p.kb_elems;
            ++l;
            if (++st == (uint32_t)NS) { st = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<kRegsConsumer>();
    const int wg = (warp - 4) >> 2;  // consumer warpgroup: accumulator rows [64*wg, 64*wg + 64)
    const int wt = threadIdx.x & 127;
    // ------------------------------------------------------------------ epilogue (row-per-thread view of the tile)
    // 8 warps: warp w reads accumulator rows 32*(w%4).. and owns the column chunks {half, half+2, ...}
    const int q = warp & 3;
    const int half = (warp - 4) >> 2;
    constexpr int kChunks = BLOCK_N / 32;
    constexpr int kChunkStep = kChunks >= 2 ? 2 : 1;
    const int row = q * 32 + lane;
    const int et = threadIdx.x - 128;  // 0..255
    const int rows_per_b = p.bx * p.by * p.bz;
    const int seg = row / rows_per_b;  // which sample of the tile this row belongs to (warp-uniform by construction)
    int it = 0;
    int staged_n0 = -1, staged_b0 = -1, bias_buf = 0;
    // GNB: whether column sums are wanted is decided once and pinned in a register instead of re-reading two pointers of
    // the parameter block in front of every chunk's reduction
    int want_cols = 0;
    if constexpr (GNB) {
      want_cols = (p.stats != nullptr || p.gnb_part != nullptr) ? 1 : 0;
      asm volatile("" : "+r"(want_cols));
    }
    uint32_t st = 0, ph = 0;
    for (int tile = first_tile; tile < total_tiles; tile += tile_step, ++it) {
      const int vit = it;
      // ---------------------------------------------------------------- main loop: wgmma over the k-step groups
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      {
        int gi = 0, g_lo, g_hi;
        split_range(tile, g_lo, g_hi);
        int prev = -1;  // stage whose wgmmas may still be reading it
        const uint32_t a_row0 = (uint32_t)wg * 64 * kRowBytes;
        for (int sg = 0; sg < p.n_segs; ++sg) {
          // (by reference: the segment stays in parameter space, where the compiler can see its fields are uniform)
          const GemmSeg& sgm = p.segs[sg];
          for (int g = 0; g < sgm.n_groups; ++g, ++gi) {
            if (gi < g_lo || gi >= g_hi) continue;
            mbar_wait(full + 8 * st, ph);
            const uint32_t sbase = stage0 + st * kStageBytesRt;
            for (int j = 0; j < sgm.nk; ++j) {
              const uint64_t ad = kdesc(sbase + j * sgm.jbytes + a_row0);
              const uint64_t bd = kdesc(sbase + sgm.a_stride + j * Cfg::kBTileBytes);
              wgmma_fence();  // directly in front of the straight-line wgmmas: no branch between the fence and them
#pragma unroll
              for (int k = 0; k < kRowBytes / 32; ++k) wgmma_kmajor<BLOCK_N, TF32>(acc, ad + 2 * k, bd + 2 * k, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous group's wgmmas have retired: hand its stage back to the producer
            if (prev >= 0 && wt == 0) mbar_arrive(empty + 8 * prev);
            prev = (int)st;
            if (++st == (uint32_t)NS) { st = 0; ph ^= 1; }
          }
        }
        wgmma_wait<0>();
        fence_operands(acc);
        if (prev >= 0 && wt == 0) mbar_arrive(empty + 8 * prev);
      }
      int x0, y0, z0, b0, n0;
      decode(tile, x0, y0, z0, b0, n0);
      int r = row;
      const int xl = r % p.bx; r /= p.bx;
      const int yl = r % p.by; r /= p.by;
      const int zl = r % p.bz; r /= p.bz;
      const int xg = x0 + xl, yg = y0 + yl, zg = z0 + zl, bg = b0 + r;
      const bool valid = (xg < p.X) && (yg < p.Y) && (zg < p.Z) && (bg < p.Bn);
      const long long ooff = xg * p.osx + yg * p.osy + zg * p.osz + bg * p.osb;
      const long long roff = xg * p.rsx + yg * p.rsy + zg * p.rsz + bg * p.rsb;

      // accumulators -> shared staging (the previous tile's epilogue must be done reading it first). wgmma layout:
      // register 4j+{0,1} = (row l/4, cols 8j + 2(l%4) + {0,1}), 4j+{2,3} = the same columns 8 rows further down.
      named_bar_sync(2, kEpiThreads);
      {
        const int w4 = (warp & 3), srow = wg * 64 + w4 * 16 + (lane >> 2), scol = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(s_acc + srow * Cfg::kAccPitch + 8 * j + scol) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(s_acc + (srow + 8) * Cfg::kAccPitch + 8 * j + scol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }

      // stage bias + per-sample (time-embedding) bias of this tile's columns, s_bias[seg][col] -- only when the tile's
      // (column block, first sample) differs from what is already staged (for a conv that is once per sample)
      const int bkey = p.rowbias ? b0 : 0;  // without a per-sample bias the staged values do not depend on the sample
      if (n0 != staged_n0 || bkey != staged_b0) {
        staged_n0 = n0; staged_b0 = bkey;
        bias_buf ^= 1;  // the other buffer may still be read by warps finishing the previous tile
        float* wb = s_stats + 16 * BLOCK_N + bias_buf * 4 * BLOCK_N;
        for (int i = et; i < p.bb * BLOCK_N; i += kEpiThreads) {
          const int sg = i / BLOCK_N, c = i % BLOCK_N;
          const int n = n0 + c, bgl = b0 + sg;
          float bv = 0.f;
          if (n < p.N) {
            if (p.bias && !p.bias_on_m) bv += __ldg(p.bias + n);
            if (p.rowbias && bgl < p.Bn) bv += __ldg(p.rowbias + static_cast<long long>(bgl) * p.rowbias_ld + n);
          }
          wb[i] = bv;
        }
      }
      const float* s_bias = s_stats + 16 * BLOCK_N + bias_buf * 4 * BLOCK_N;
      float* s_part = s_stats + (vit & 1) * 8 * BLOCK_N;  // column partials, double-buffered across tiles
      // residual rows do not depend on the accumulator: fetch the first chunk before the staging barrier, and every
      // next chunk while the current one is being stored, so the (L2/HBM) latency is never exposed
      uint4 rbuf[8];
      auto prefetch_res = [&](int ch) {
        const int nbp = n0 + ch * 32;
        if (!(p.res && valid && p.ocs == 1 && nbp + 32 <= p.N)) return;
        if constexpr (GNB) {
          // the GroupNorm input x: first or second source of the channel concatenation (32-column chunks never straddle)
          const bool second = p.res1 && nbp >= p.res_c0;
          const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(second ? p.res1 : p.res);
          const long long off = second ? xg * p.r1sx + yg * p.r1sy + zg * p.r1sz + bg * p.r1sb + (nbp - p.res_c0) : roff + nbp;
          const uint4* rp = reinterpret_cast<const uint4*>(base + off);
#pragma unroll
          for (int i = 0; i < 4; ++i) rbuf[i] = __ldg(rp + i);
          return;
        }
        if (TF32 || p.res_fp32) {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.res) + roff + nbp);
#pragma unroll
          for (int i = 0; i < 8; ++i) rbuf[i] = __ldg(rp + i);
        } else {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + roff + nbp);
#pragma unroll
          for (int i = 0; i < 4; ++i) rbuf[i] = __ldg(rp + i);
          if constexpr (X3) {
            const uint4* rl = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + roff + nbp + p.res_lo_off);
#pragma unroll
            for (int i = 0; i < 4; ++i) rbuf[4 + i] = __ldg(rl + i);
          }
        }
      };
      const int ch0 = kChunkStep == 2 ? half : 0;
      const bool active = kChunkStep == 2 || half == 0;  // BLOCK_N == 32: one chunk, the second warp of a quarter idles
      if (active) prefetch_res(ch0);
      named_bar_sync(2, kEpiThreads);  // staged accumulators (and bias) visible to every epilogue thread

#pragma unroll 1
      for (int ch = ch0; ch < kChunks && active; ch += kChunkStep) {
        uint32_t rr[32];
        {
          const float4* src = reinterpret_cast<const float4*>(s_acc + row * Cfg::kAccPitch + ch * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 t = src[i];
            rr[4 * i] = __float_as_uint(t.x); rr[4 * i + 1] = __float_as_uint(t.y);
            rr[4 * i + 2] = __float_as_uint(t.z); rr[4 * i + 3] = __float_as_uint(t.w);
          }
        }
        const int nb = n0 + ch * 32;
        if (nb >= p.N) continue;  // warp-uniform
        if (splits > 1) {
          // split-K: raw fp32 partial sums; bias / residual / statistics are applied by the reduction kernel
          if (valid) {
            // (X3: ooff is in physical bf16 elements, twice the logical row pitch the fp32 partials use)
            float* pp = p.partial + (long long)(tile % splits) * p.split_stride + (X3 ? (ooff >> 1) : ooff) + nb;
            if (nb + 32 <= p.N) {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                reinterpret_cast<float4*>(pp)[i] = make_float4(__uint_as_float(rr[4 * i]), __uint_as_float(rr[4 * i + 1]),
                                                               __uint_as_float(rr[4 * i + 2]), __uint_as_float(rr[4 * i + 3]));
            } else {
              for (int i = 0; i < 32; ++i) if (nb + i < p.N) pp[i] = __uint_as_float(rr[i]);
            }
          }
          continue;
        }
        const bool full = (nb + 32 <= p.N) && (p.ocs == 1);
        float v[32];
        const float mbias = (p.bias && p.bias_on_m && valid) ? __ldg(p.bias + xg) : 0.f;
        const float* sb = s_bias + (seg < 4 ? seg : 0) * BLOCK_N + ch * 32;
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(rr[i]) * p.alpha + mbias + sb[i];
        float q2[GNB ? 32 : 1];  // dy * xhat (GNB)
        if constexpr (GNB) {
          if (valid) {
            const float4* cc = p.gnb_c + static_cast<long long>(bg) * p.N + nb;
            unsigned long long hsh[8];
            if (p.gnb_drop_thresh > 0) {
              // same element index as the forward GroupNorm-apply kernel: ((b*V + voxel)*C + channel)
              const unsigned long long e4 = (unsigned long long)((((static_cast<long long>(bg) * p.Z + zg) * p.Y + yg) * p.X + xg) * p.N + nb) >> 2;
#pragma unroll
              for (int i = 0; i < 8; ++i) hsh[i] = gn_drop_hash64(p.gnb_seed, e4 + i);
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const float4 kc = __ldg(cc + i);
              const __nv_bfloat16 xb = reinterpret_cast<const __nv_bfloat16*>(rbuf)[i];
              const float xv = __bfloat162float(xb);
              float d = v[i];
              if (p.gnb_drop_thresh > 0) {
                const unsigned r16 = (unsigned)((hsh[i >> 2] >> (16 * (i & 3))) & 0xFFFFu);
                d = r16 >= (unsigned)p.gnb_drop_thresh ? d * p.gnb_drop_scale : 0.f;
              }
              if (p.gnb_silu) {
                const float h = fmaf(xv, kc.x, kc.y);
                float th;
                asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(h));
                d *= fmaf(0.5f, h * fmaf(-th, th, 1.f), fmaf(0.5f, th, 0.5f));
              }
              v[i] = d;
              q2[i] = d * fmaf(xv, kc.z, kc.w);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) q2[i] = 0.f;
          }
        }
        if (!GNB && p.res && valid) {
          if (TF32 || p.res_fp32) {
            if (full) {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 t = *reinterpret_cast<const float4*>(&rbuf[i]);
                v[4 * i] += t.x; v[4 * i + 1] += t.y; v[4 * i + 2] += t.z; v[4 * i + 3] += t.w;
              }
            } else {
              const float* rp = reinterpret_cast<const float*>(p.res) + roff + nb;
              for (int i = 0; i < 32; ++i) if (nb + i < p.N) v[i] += rp[i];
            }
          } else {
            if (full) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&rbuf[i]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  float2 f = __bfloat1622float2(h[j]);
                  if constexpr (X3) {
                    const float2 l = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(&rbuf[4 + i])[j]);
                    f.x += l.x; f.y += l.y;
                  }
                  v[8 * i + 2 * j] += f.x; v[8 * i + 2 * j + 1] += f.y;
                }
              }
            } else {
              const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.res) + roff + nb;
              for (int i = 0; i < 32; ++i)
                if (nb + i < p.N) v[i] += __bfloat162float(rp[i]) + (X3 ? __bfloat162float(rp[i + p.res_lo_off]) : 0.f);
            }
          }
        }
        if (ch + kChunkStep < kChunks) prefetch_res(ch + kChunkStep);  // lands while this chunk is stored / reduced
        if (valid) {
          if (TF32 || p.out_fp32) {
            float* op = reinterpret_cast<float*>(p.out) + ooff + nb;
            if (full) {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                float4 t = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
                if (p.round_out) { t.x = to_tf32_rna(t.x); t.y = to_tf32_rna(t.y); t.z = to_tf32_rna(t.z); t.w = to_tf32_rna(t.w); }
                reinterpret_cast<float4*>(op)[i] = t;
              }
            } else {
              for (int i = 0; i < 32; ++i) if (nb + i < p.N) op[i * p.ocs] = v[i];
            }
          } else {
            __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + ooff + nb;
            if (full) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                uint4 t;
                __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
                for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[8 * i + 2 * j], v[8 * i + 2 * j + 1]);
                reinterpret_cast<uint4*>(op)[i] = t;
                if constexpr (X3) {  // lo parts: what the bf16 rounding of the hi parts lost
                  uint4 tl;
                  __nv_bfloat162* l = reinterpret_cast<__nv_bfloat162*>(&tl);
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    const float2 f = __bfloat1622float2(h[j]);
                    l[j] = __floats2bfloat162_rn(v[8 * i + 2 * j] - f.x, v[8 * i + 2 * j + 1] - f.y);
                  }
                  reinterpret_cast<uint4*>(op + p.out_lo_off)[i] = tl;
                }
              }
            } else {
              for (int i = 0; i < 32; ++i)
                if (nb + i < p.N) {
                  const __nv_bfloat16 hb = __float2bfloat16(v[i]);
                  op[i * p.ocs] = hb;
                  if constexpr (X3) op[i * p.ocs + p.out_lo_off] = __float2bfloat16(v[i] - __bfloat162float(hb));
                }
            }
          }
        }
        if (GNB ? (want_cols != 0) : (p.stats != nullptr)) {  // (never reached in split-K mode)
          // Column sums over the warp's 32 rows: butterfly transpose-reduce (31 shuffles per quantity);
          // afterwards lane i holds the sum of column i.
          float s[32], ss[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float t = valid ? v[i] : 0.f;
            s[i] = t; ss[i] = GNB ? q2[GNB ? i : 0] : t * t;
          }
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            const bool hi = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < off; ++i) {
              const float send_s = hi ? s[i] : s[i + off];
              const float send_q = hi ? ss[i] : ss[i + off];
              const float keep_s = hi ? s[i + off] : s[i];
              const float keep_q = hi ? ss[i + off] : ss[i];
              s[i] = keep_s + __shfl_xor_sync(0xffffffffu, send_s, off);
              ss[i] = keep_q + __shfl_xor_sync(0xffffffffu, send_q, off);
            }
          }
          // per-warp slot, no atomics: the cross-warp sum below runs in a fixed order (deterministic results)
          s_part[(q * 2 + 0) * BLOCK_N + ch * 32 + lane] = s[0];
          s_part[(q * 2 + 1) * BLOCK_N + ch * 32 + lane] = ss[0];
        }
      }
      if constexpr (GNB) {
        if (p.gnb_part && splits == 1) {
          // per-tile column partials, one row per (M-tile, sample of the tile): summed in a fixed order by
          // gnb_tile_reduce_kernel (deterministic gradients; no atomics)
          named_bar_sync(1, kEpiThreads);
          const int warps_per_seg = rows_per_b >= 128 ? 4 : rows_per_b / 32;
          for (int i = et; i < p.bb * BLOCK_N; i += kEpiThreads) {
            const int sg = i / BLOCK_N, c = i % BLOCK_N;
            const int n = n0 + c;
            if (mt_of_tile < tiles_m && n < p.N) {
              float ts = 0.f, tq = 0.f;
              for (int w = sg * warps_per_seg; w < (sg + 1) * warps_per_seg; ++w) {
                ts += s_part[(w * 2 + 0) * BLOCK_N + c];
                tq += s_part[(w * 2 + 1) * BLOCK_N + c];
              }
              float* dst = p.gnb_part + ((static_cast<long long>(mt_of_tile) * p.bb + sg) * p.N + n) * 2;
              dst[0] = ts; dst[1] = tq;
            }
          }
        }
      }
      if (!GNB && p.stats && splits == 1) {
        // the only barrier per tile: partials of tile i+1 go to the other buffer, and a buffer is rewritten two tiles
        // later, after every warp has passed this barrier once more
        named_bar_sync(1, kEpiThreads);
        const int warps_per_seg = rows_per_b >= 128 ? 4 : rows_per_b / 32;
        // the same trip count in every thread: a per-thread loop bound here left the warp possibly diverged at the top of
        // the next tile, and the compiler then serialised that tile's wgmmas
        for (int i0 = 0; i0 < p.bb * BLOCK_N; i0 += kEpiThreads) {
          const int i = i0 + et;
          const int sg = i / BLOCK_N, c = i % BLOCK_N;
          const int bgl = b0 + sg, n = n0 + c;
          if (i < p.bb * BLOCK_N && bgl < p.Bn && n < p.N) {
            float ts = 0.f, tq = 0.f;
            for (int w = sg * warps_per_seg; w < (sg + 1) * warps_per_seg; ++w) {
              ts += s_part[(w * 2 + 0) * BLOCK_N + c];
              tq += s_part[(w * 2 + 1) * BLOCK_N + c];
            }
            long long* dst = p.stats + (static_cast<long long>(bgl) * p.N + n) * kStatWords;
            stat_add(dst, ts);
            stat_add(dst + 2, tq);
          }
        }
      }
    }
  }
}

}  // namespace mdb
