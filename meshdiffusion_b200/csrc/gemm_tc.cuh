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
//   m64nNk8). After the last k-step they are staged through shared memory (64 columns at a time), and the same 256
//   threads read them back one row per thread to add bias / time-embedding bias / residual, store NDHWC output and
//   reduce per-(sample, channel) sum and sum-of-squares for the GroupNorm that follows (warp-shuffle butterfly + shared
//   + one atomic per channel). In the bf16 / split-bf16 inference kernels with 128-column tiles (GemmParams::epi_tma)
//   each 64-column round borrows the next B slot: the producer TMA-loads the residual box into it, the threads
//   overwrite it with the output box and one thread stores that with TMA. Other launches store row by row.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (warp 0), warpgroups 1-2 = MMA + epilogue.
#pragma once
#include "ptx.cuh"
#include "act_format.cuh"
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
  uint8_t tmap_lo;  // X3: index of the A tensor map of the lo parts (same box, loaded next to the hi parts)
  uint8_t pad;
};
static_assert(sizeof(LoadEntry) == 16, "LoadEntry must be 16 bytes");

// A run of identical pipeline groups. One group = one load-table entry: one A box (X3: its hi and lo parts) in an A slot,
// multiplied with the weight tiles of its nk k-steps, one B slot per k-step (X3: the W_hi and W_lo tiles of the k-step).
// All fields are warp-uniform kernel parameters, so the MMA warp's control flow and descriptor arithmetic never touch
// memory.
struct GemmSeg {
  int n_groups;
  int nk;        // k-steps per entry
  int a_bytes;   // bytes of one A box (rows * 128) -- the TMA transaction size
  int a_stride;  // X3: distance from the hi to the lo box in the A slot (multiple of 1024)
  int jbytes;    // A-descriptor advance between the k-steps of one entry (halo reuse)
};
constexpr int kMaxSegs = 8;

struct GemmParams {
  CUtensorMap amap[kMaxAMaps];
  CUtensorMap bmap;
  // TMA epilogue (epi_tma != 0): each 64-column staging round takes the next B slot; the producer loads the residual box
  // into it, the epilogue threads overwrite it with the output box and one thread stores that with TMA. Boxes are
  // (kStageCols channels, bx, by, bz, bb), 128B-swizzled; [0] = the tensor / the hi parts, [1] = the split-bf16 lo parts.
  CUtensorMap omap[2];
  CUtensorMap rmap[2];
  int epi_tma;
#ifdef MDB_EPI_TRACE
  unsigned long long* trace;  // [kTraceCtas][kTraceTiles][kTraceStamps] globaltimer stamps (instrumented build only)
#endif
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
  int b_kstep;         // K coordinate advance of the B tiles per k-step (X3 packed weights: 2 * kb_elems, hi + lo)
  int b_lo_k;          // X3: K distance from a k-step's W_hi tile to its W_lo tile
  // shared-memory operand rings (as many slots as fit next to the epilogue scratch): A slots hold one entry's A box,
  // B slots the weight tiles of one k-step
  int n_aslots, a_slot_bytes, n_bslots, b_slot_bytes;
  // X3 (split bf16) epilogue: the lo parts of the output / residual rows sit this many elements behind the hi parts
  long long out_lo_off, res_lo_off;
  // epilogue
  void* out;
  long long osx, osy, osz, osb;  // output element strides per voxel axis
  long long ocs;                 // output column stride (1 = channels contiguous; else scalar store path)
  int out_fp32;  // plain fp32 output (attention logits, head projection, stem field); else the activation format
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
  long long res1_lo_off;  // X3: lo parts of the res1 rows (res rows: res_lo_off)
  int res_c0;
  const float4* gnb_c;  // [Bn][N] {hsc, hsh, rs, nm}: y/2 = x*hsc + hsh, xhat = x*rs + nm
  int gnb_silu;
  int gnb_drop_thresh; float gnb_drop_scale; unsigned long long gnb_seed;
  float* gnb_part;      // [tiles_m * bb][N][2]
};

constexpr int kMaxSlots = 8;  // per ring
constexpr int kMaxDynSmem = 232448;  // 227 KB: the opt-in limit of dynamic shared memory per block on sm_90
// kWholeTile: stage all BLOCK_N columns in one round (the GroupNorm-backward epilogues: the split-bf16 one spills
// registers when round 1's accumulators stay live through round 0, the bf16 one runs slower)
template <int BLOCK_N, bool kWholeTile = false>
struct GemmCfg {
  static constexpr int kBTileBytes = BLOCK_N * kRowBytes;  // weight tile bytes per k-step
  static constexpr int kStatsFloats = 24 * BLOCK_N;  // 2 x [4 warps][sum,sumsq][N] column partials + 2 x [4 segs][N] bias
  // accumulator staging [128 rows][kAccPitch], in kStageRounds rounds of kStageCols columns: 64-column rounds leave the
  // operand rings 32 KB more than staging all 128 columns at once would. The 4-float pad keeps the row-per-lane float4
  // reads conflict-free.
  static constexpr int kStageCols = (kWholeTile || BLOCK_N < 64) ? BLOCK_N : 64;
  static constexpr int kStageRounds = BLOCK_N / kStageCols;
  static_assert(kStageRounds <= 2, "the epilogue stages at most two rounds");
  static constexpr int kAccPitch = kStageCols + 4;
  static constexpr int kAccFloats = kBlockM * kAccPitch;
  // everything but the operand rings: alignment slack, accumulator staging, epilogue scratch, mbarriers (full / empty of
  // both rings)
  static constexpr int kFixedBytes = 1024 + kAccFloats * 4 + kStatsFloats * 4 + 4 * kMaxSlots * 8;
};
constexpr int kRegsProducer = 40, kRegsConsumer = 232;  // 128 x 40 + 256 x 232 <= 65 536

// The TMA epilogue exists in the inference instantiations with 128-column tiles of bf16 rows: there one round's output box
// (64 channels x 128 rows x 2 B) is exactly one weight tile, and a split-bf16 B slot holds its hi and lo boxes.
template <int BLOCK_N, Precision P, bool GNB>
constexpr bool kHasTmaEpi = !GNB && BLOCK_N == 128 && P != kTF32;
constexpr int kEpiBoxBytes = 64 * 2 * kBlockM;  // one part of one round's output / residual box
static_assert(kEpiBoxBytes == GemmCfg<128>::kBTileBytes, "an epilogue box is one weight tile");

#ifdef MDB_EPI_TRACE
// Instrumented build (-DMDB_EPI_TRACE): the first kTraceTiles tiles of the first kTraceCtas CTAs record globaltimer
// stamps, taken by epilogue thread 0: 0 = last wgmma_wait<0>, 1 = round 0 staged, 2 = round 0's chunks done (TMA
// epilogue: its store issued), 3 = the same for round 1, 4 = statistics atomics done, 5 = the tile's first k-step has its
// operands (the previous tile's epilogue ends at the next tile's stamp 5).
constexpr int kTraceCtas = 16, kTraceTiles = 64, kTraceStamps = 6;
#define MDB_STAMP(k) do { if (trace_row && et == 0) trace_row[k] = globaltimer(); } while (0)
#else
#define MDB_STAMP(k) do { } while (0)
#endif

// K-major 128B-swizzled operand at `saddr` (SBO = 1024 B)
__device__ __forceinline__ uint64_t kdesc(uint32_t saddr) { return make_wgmma_desc(saddr, 16, 1024); }

// Column sums over a warp's 32 rows, two quantities at once: butterfly transpose-reduce (31 shuffles per quantity); on
// return lane i holds the sums of column i in s[0] / ss[0]. Level OFF halves the live columns [0, 2 OFF): a lane sends the
// half its partner keeps and adds the received values to the half it keeps. The levels are template recursion so that
// every array index is a compile-time constant and the lane select is a select between two registers: nvcc leaves an
// inner loop bounded by an outer loop's OFF rolled, and its lane-dependent indices put both arrays in local memory
// (build.py fails a build that gives this kernel a stack frame).
template <int OFF>
__device__ __forceinline__ void colsum_butterfly(float (&s)[32], float (&ss)[32], int lane) {
  const bool hi = (lane & OFF) != 0;
#pragma unroll
  for (int i = 0; i < OFF; ++i) {
    const float send_s = hi ? s[i] : s[i + OFF];
    const float send_q = hi ? ss[i] : ss[i + OFF];
    const float keep_s = hi ? s[i + OFF] : s[i];
    const float keep_q = hi ? ss[i + OFF] : ss[i];
    s[i] = keep_s + __shfl_xor_sync(0xffffffffu, send_s, OFF);
    ss[i] = keep_q + __shfl_xor_sync(0xffffffffu, send_q, OFF);
  }
  if constexpr (OFF > 1) colsum_butterfly<OFF / 2>(s, ss, lane);
}

// v[0, 32) += the residual chunk prefetched as 16-byte vectors in mode P (split bf16: hi vectors in buf[0, 4), lo in [4, 8))
template <Precision P>
__device__ __forceinline__ void add_res_chunk(const uint4 (&buf)[8], float (&v)[32]) {
  constexpr int E = kVecElems<P>, NV = 32 / E;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float r[E];
    decode_vec<P>(buf[i], buf[P == kBF16X3 ? NV + i : i], r);
#pragma unroll
    for (int j = 0; j < E; ++j) v[E * i + j] += r[j];
  }
}

// P: the operand mode (act_format.cuh); the epilogue reads residuals and stores outputs in its row format.
// GNB: GroupNorm-backward epilogue (see GemmParams::gnb_c) -- a separate instantiation, so the inference kernels'
// code is untouched.
// kBF16X3 (split bf16): an entry loads the hi and lo parts of its A box, a k-step the W_hi and W_lo tiles. Per k16 step,
// A_hi . [W_hi; W_lo] is one m64n(2 BLOCK_N) wgmma into acc[0, BLOCK_N) (first half: the W_hi columns, second half: W_lo),
// then A_lo . W_hi an m64nBLOCK_N one into acc[0, BLOCK_N / 2); after the last k-step the second half is folded into the
// first. GNB with kBF16X3 reads the GroupNorm input as hi + lo, stores dy as (hi, lo) and takes the SiLU derivative from
// ex2/rcp (tanh.approx's 2^-11 would cap the gradient accuracy near 5e-4).
template <int BLOCK_N, Precision P, bool GNB>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  static_assert(!(GNB && P == kTF32), "the GroupNorm-backward epilogue is built for bf16 / split-bf16 operands");
  using Cfg = GemmCfg<BLOCK_N, GNB>;
  constexpr int kParts = parts(P);  // operand parts per A box / per k-step of weights
  const int NA = p.n_aslots, NB = p.n_bslots;
  const uint32_t a_slot = (uint32_t)p.a_slot_bytes, b_slot = (uint32_t)p.b_slot_bytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* s_acc = reinterpret_cast<float*>(smem + NA * p.a_slot_bytes + NB * p.b_slot_bytes);
  float* s_stats = s_acc + Cfg::kAccFloats;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stats + Cfg::kStatsFloats);

  const uint32_t a_ring = smem_u32(smem), b_ring = a_ring + NA * a_slot;
  const uint32_t a_full = smem_u32(bars), a_empty = a_full + 8 * kMaxSlots;
  const uint32_t b_full = a_empty + 8 * kMaxSlots, b_empty = b_full + 8 * kMaxSlots;

  // (broadcast from lane 0, so the compiler can treat the warpgroup branches as warp-uniform)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < kMaxAMaps; ++i) tma_prefetch_desc(&p.amap[i]);
    tma_prefetch_desc(&p.bmap);
  }
  if (warp == 1 && lane == 0) {
    // full: the producer's expect_tx arrival; empty: one arrival per consumer warpgroup
    for (int i = 0; i < NA; ++i) { mbar_init(a_full + 8 * i, 1); mbar_init(a_empty + 8 * i, 2); }
    for (int i = 0; i < NB; ++i) { mbar_init(b_full + 8 * i, 1); mbar_init(b_empty + 8 * i, 2); }
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
      uint32_t as = 0, aph = 0, bs = 0, bph = 0;
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        int x0, y0, z0, b0, n0;
        decode(tile, x0, y0, z0, b0, n0);
        int kcol = 0, l = 0, gi = 0, g_lo, g_hi;
        split_range(tile, g_lo, g_hi);
        const int bcoord = p.b_batched ? b0 : 0;
        for (int sg = 0; sg < p.n_segs; ++sg) {
          const GemmSeg& seg = p.segs[sg];
          for (int g = 0; g < seg.n_groups; ++g, ++gi) {
            if (gi < g_lo || gi >= g_hi) {  // another CTA's share of this tile's K range
              kcol += seg.nk * p.b_kstep;
              ++l;
              continue;
            }
            // the table entry of this group is fetched before blocking on the slot
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(p.loads + l));
            const LoadEntry& en = reinterpret_cast<const LoadEntry&>(raw);
            mbar_wait(a_empty + 8 * as, aph ^ 1);
            if (elect_one()) {
              const uint32_t abase = a_ring + as * a_slot, bar = a_full + 8 * as;
              mbar_expect_tx(bar, kParts * seg.a_bytes);
              tma_load_5d(&p.amap[en.tmap], bar, abase, en.c0, x0 + en.dx, y0 + en.dy, z0 + en.dz, b0);
              if constexpr (P == kBF16X3) tma_load_5d(&p.amap[en.tmap_lo], bar, abase + seg.a_stride, en.c0, x0 + en.dx, y0 + en.dy, z0 + en.dz, b0);
            }
            __syncwarp();
            if (++as == (uint32_t)NA) { as = 0; aph ^= 1; }
            int kc = (P == kBF16X3 && p.b_explicit_k) ? (int)en.wc0 : kcol;
            for (int j = 0; j < seg.nk; ++j) {
              mbar_wait(b_empty + 8 * bs, bph ^ 1);
              if (elect_one()) {
                const uint32_t bbase = b_ring + bs * b_slot, bar = b_full + 8 * bs;
                mbar_expect_tx(bar, kParts * Cfg::kBTileBytes);
                tma_load_3d(&p.bmap, bar, bbase, kc, n0, bcoord);
                if constexpr (P == kBF16X3) tma_load_3d(&p.bmap, bar, bbase + Cfg::kBTileBytes, kc + p.b_lo_k, n0, bcoord);
              }
              __syncwarp();
              kc += p.b_kstep;
              if (++bs == (uint32_t)NB) { bs = 0; bph ^= 1; }
            }
            kcol += seg.nk * p.b_kstep;
            ++l;
          }
        }
        if constexpr (kHasTmaEpi<BLOCK_N, P, GNB>) {
          // the tile's epilogue slots, one per staging round: the residual box(es) of the round's columns, loaded while
          // the last k-steps run, or (no residual / no valid column) a plain arrival
          if (p.epi_tma) {
            for (int rnd = 0; rnd < Cfg::kStageRounds; ++rnd) {
              mbar_wait(b_empty + 8 * bs, bph ^ 1);
              if (elect_one()) {
                const uint32_t bbase = b_ring + bs * b_slot, bar = b_full + 8 * bs;
                const int c = n0 + rnd * Cfg::kStageCols;
                if (p.res && c < p.N) {
                  mbar_expect_tx(bar, kParts * kEpiBoxBytes);
                  tma_load_5d(&p.rmap[0], bar, bbase, c, x0, y0, z0, b0);
                  if constexpr (P == kBF16X3) tma_load_5d(&p.rmap[1], bar, bbase + kEpiBoxBytes, c, x0, y0, z0, b0);
                } else {
                  mbar_arrive(bar);
                }
              }
              __syncwarp();
              if (++bs == (uint32_t)NB) { bs = 0; bph ^= 1; }
            }
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
    uint32_t as = 0, aph = 0, bs = 0, bph = 0;
    // TMA epilogue: the slot of the tile's last round, handed back once its store has read it (epilogue thread 0 only)
    int epi_pend = -1;
    for (int tile = first_tile; tile < total_tiles; tile += tile_step, ++it) {
      const int vit = it;
#ifdef MDB_EPI_TRACE
      unsigned long long* trace_row = (p.trace && (int)blockIdx.x < kTraceCtas && it < kTraceTiles)
                                          ? p.trace + ((long long)blockIdx.x * kTraceTiles + it) * kTraceStamps : nullptr;
      bool first_k = true;
#endif
      if constexpr (kHasTmaEpi<BLOCK_N, P, GNB>) {
        if (et == 0 && epi_pend >= 0) {
          bulk_wait_read<0>();
          mbar_arrive(b_empty + 8 * epi_pend);
          mbar_arrive(b_empty + 8 * epi_pend);
          epi_pend = -1;
        }
      }
      // ---------------------------------------------------------------- main loop: wgmma over the k-step groups
      constexpr int kAccRegs = kParts * BLOCK_N / 2;  // split bf16: [W_hi columns | W_lo columns] until the fold
      float acc[kAccRegs];
      float (&acc_hi)[BLOCK_N / 2] = *reinterpret_cast<float (*)[BLOCK_N / 2]>(acc);
#pragma unroll
      for (int i = 0; i < kAccRegs; ++i) acc[i] = 0.f;
      {
        int gi = 0, g_lo, g_hi;
        split_range(tile, g_lo, g_hi);
        // slots whose wgmmas may still be reading them: each is handed back once the next k-step's wait shows them retired
        int prev_b = -1, prev_a = -1;
        const uint32_t a_row0 = (uint32_t)wg * 64 * kRowBytes;
        for (int sg = 0; sg < p.n_segs; ++sg) {
          // (by reference: the segment stays in parameter space, where the compiler can see its fields are uniform)
          const GemmSeg& sgm = p.segs[sg];
          for (int g = 0; g < sgm.n_groups; ++g, ++gi) {
            if (gi < g_lo || gi >= g_hi) continue;
            mbar_wait(a_full + 8 * as, aph);
            const uint32_t abase = a_ring + as * a_slot + a_row0;
            for (int j = 0; j < sgm.nk; ++j) {
              mbar_wait(b_full + 8 * bs, bph);
#ifdef MDB_EPI_TRACE
              if (first_k) { MDB_STAMP(5); first_k = false; }
#endif
              const uint64_t ad = kdesc(abase + j * sgm.jbytes);
              const uint64_t bd = kdesc(b_ring + bs * b_slot);
              wgmma_fence();  // directly in front of the straight-line wgmmas: no branch between the fence and them
              if constexpr (P == kBF16X3) {
                const uint64_t adl = kdesc(abase + sgm.a_stride + j * sgm.jbytes);
#pragma unroll
                for (int k = 0; k < kRowBytes / 32; ++k) wgmma_kmajor<2 * BLOCK_N, false>(acc, ad + 2 * k, bd + 2 * k, 1u);
                wgmma_fence();  // the next wgmmas have another shape: order their accumulator accesses after these
#pragma unroll
                for (int k = 0; k < kRowBytes / 32; ++k) wgmma_kmajor<BLOCK_N, false>(acc_hi, adl + 2 * k, bd + 2 * k, 1u);
              } else {
#pragma unroll
                for (int k = 0; k < kRowBytes / 32; ++k) wgmma_kmajor<BLOCK_N, P == kTF32>(acc, ad + 2 * k, bd + 2 * k, 1u);
              }
              wgmma_commit();
              wgmma_wait<1>();  // the previous k-step's wgmmas have retired: hand its slots back to the producer
              if (wt == 0) {
                if (prev_b >= 0) mbar_arrive(b_empty + 8 * prev_b);
                if (prev_a >= 0) mbar_arrive(a_empty + 8 * prev_a);
              }
              prev_b = (int)bs;
              prev_a = j + 1 == sgm.nk ? (int)as : -1;
              if (++bs == (uint32_t)NB) { bs = 0; bph ^= 1; }
            }
            if (++as == (uint32_t)NA) { as = 0; aph ^= 1; }
          }
        }
        wgmma_wait<0>();
        fence_operands(acc);
        MDB_STAMP(0);
        if (wt == 0) {
          if (prev_b >= 0) mbar_arrive(b_empty + 8 * prev_b);
          if (prev_a >= 0) mbar_arrive(a_empty + 8 * prev_a);
        }
        if constexpr (P == kBF16X3) {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] += acc[BLOCK_N / 2 + i];
        }
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

      // accumulators -> shared staging, one round of kStageCols columns at a time. wgmma layout: register 4j+{0,1} =
      // (row l/4, cols 8j + 2(l%4) + {0,1}), 4j+{2,3} = the same columns 8 rows further down, so the columns of round r
      // are acc[kRoundRegs * r, kRoundRegs * (r + 1)).
      constexpr int kRoundRegs = Cfg::kStageCols / 2;
      auto stage = [&]() {
        const int w4 = (warp & 3), srow = wg * 64 + w4 * 16 + (lane >> 2), scol = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < Cfg::kStageCols / 8; ++j) {
          *reinterpret_cast<float2*>(s_acc + srow * Cfg::kAccPitch + 8 * j + scol) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(s_acc + (srow + 8) * Cfg::kAccPitch + 8 * j + scol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      };
      named_bar_sync(2, kEpiThreads);  // the previous tile's epilogue is done reading the staging
      stage();
      // round 1's registers take the place of round 0's, so that the (rolled) round loop below stages the same registers
      if constexpr (Cfg::kStageRounds > 1) {
#pragma unroll
        for (int i = 0; i < kRoundRegs; ++i) acc[i] = acc[kRoundRegs + i];
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
          if constexpr (P == kBF16X3) {
            const uint4* rl = reinterpret_cast<const uint4*>(base + off + (second ? p.res1_lo_off : p.res_lo_off));
#pragma unroll
            for (int i = 0; i < 4; ++i) rbuf[4 + i] = __ldg(rl + i);
          }
          return;
        }
        if (P == kTF32 || p.res_fp32) {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.res) + roff + nbp);
#pragma unroll
          for (int i = 0; i < 8; ++i) rbuf[i] = __ldg(rp + i);
        } else {
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + roff + nbp);
#pragma unroll
          for (int i = 0; i < 4; ++i) rbuf[i] = __ldg(rp + i);
          if constexpr (P == kBF16X3) {
            const uint4* rl = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + roff + nbp + p.res_lo_off);
#pragma unroll
            for (int i = 0; i < 4; ++i) rbuf[4 + i] = __ldg(rl + i);
          }
        }
      };
      // TMA epilogue (residual, when there is one, from the round's slot; output into it): decided by the launch's
      // parameters, the same for every thread and for the producer
      const bool tma_epi = kHasTmaEpi<BLOCK_N, P, GNB> && p.epi_tma != 0;
      const int ch0 = kChunkStep == 2 ? half : 0;
      const bool active = kChunkStep == 2 || half == 0;  // BLOCK_N == 32: one chunk, the second warp of a quarter idles
      if (active && !tma_epi) prefetch_res(ch0);

      // the chunks of round r are [kRoundChunks * r, kRoundChunks * (r + 1)); each warp takes its own in the same order
      // (half, half + 2, ...) as from a single round
      constexpr int kRoundChunks = Cfg::kStageCols / 32;
#pragma unroll 1
      for (int rnd = 0; rnd < Cfg::kStageRounds; ++rnd) {
        if (rnd > 0) {
          named_bar_sync(2, kEpiThreads);  // every warp is done reading the previous round
          stage();
        }
        named_bar_sync(2, kEpiThreads);  // staged accumulators (and bias) visible to every epilogue thread
        if (rnd == 0) MDB_STAMP(1);
        // TMA epilogue: the round's slot, in the producer's ring order; 128B-swizzled rows of 128 B (64 bf16 channels),
        // the 16-byte vector c of row r at r * 128 + 16 (c ^ r % 8), so the row-per-lane accesses are conflict-free
        int eslot_i = 0;
        uint8_t* eslot = nullptr;
        if constexpr (kHasTmaEpi<BLOCK_N, P, GNB>) {
          if (tma_epi) {
            eslot_i = (int)bs;
            eslot = smem + NA * p.a_slot_bytes + bs * p.b_slot_bytes;
            mbar_wait(b_full + 8 * bs, bph);
            if (++bs == (uint32_t)NB) { bs = 0; bph ^= 1; }
          }
        }

#pragma unroll 1
        for (int ch = ch0 + rnd * kRoundChunks; ch < (rnd + 1) * kRoundChunks && active; ch += kChunkStep) {
          uint32_t rr[32];
          {
            const float4* src = reinterpret_cast<const float4*>(s_acc + row * Cfg::kAccPitch + (ch - rnd * kRoundChunks) * 32);
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
              // (split bf16: ooff is in physical bf16 elements, twice the logical row pitch the fp32 partials use)
              float* pp = p.partial + (long long)(tile % splits) * p.split_stride + (P == kBF16X3 ? (ooff >> 1) : ooff) + nb;
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
              // dropout mask of act_format.cuh (apply_dropout, interleaved with the loop below: the helper's separate pass
              // changes this instantiation's register allocation)
              unsigned long long hsh[8];
              if (p.gnb_drop_thresh > 0) {
                const unsigned long long e4 = (unsigned long long)((((static_cast<long long>(bg) * p.Z + zg) * p.Y + yg) * p.X + xg) * p.N + nb) >> 2;
#pragma unroll
                for (int i = 0; i < 8; ++i) hsh[i] = drop_hash64(p.gnb_seed, e4 + i);
              }
#pragma unroll
              for (int i = 0; i < 32; ++i) {
                const float4 kc = __ldg(cc + i);
                const __nv_bfloat16 xb = reinterpret_cast<const __nv_bfloat16*>(rbuf)[i];
                float xv = __bfloat162float(xb);
                if constexpr (P == kBF16X3) xv += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(rbuf + 4)[i]);
                float d = v[i];
                if (p.gnb_drop_thresh > 0) {
                  const unsigned r16 = (unsigned)((hsh[i >> 2] >> (16 * (i & 3))) & 0xFFFFu);
                  d = r16 >= (unsigned)p.gnb_drop_thresh ? d * p.gnb_drop_scale : 0.f;
                }
                if (p.gnb_silu) {
                  const float h = fmaf(xv, kc.x, kc.y);
                  d *= P == kBF16X3 ? dsilu_ex2_half(h) : dsilu_tanh_half(h);
                }
                v[i] = d;
                q2[i] = d * fmaf(xv, kc.z, kc.w);
              }
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i) q2[i] = 0.f;
            }
          }
          // byte offset of this chunk's 16-byte vector i in the round's slot (TMA epilogue)
          const int chr = ch - rnd * kRoundChunks;
          auto eoff = [&](int i) { return row * 128 + (((4 * chr + i) ^ (row & 7)) << 4); };
          if (!GNB && p.res && valid && tma_epi) {
            // (columns past N were zero-filled by TMA and are not stored)
            uint4 buf[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              buf[i] = *reinterpret_cast<const uint4*>(eslot + eoff(i));
              buf[4 + i] = P == kBF16X3 ? *reinterpret_cast<const uint4*>(eslot + kEpiBoxBytes + eoff(i)) : buf[i];
            }
            add_res_chunk<P>(buf, v);
          } else if (!GNB && p.res && valid) {
            if (P == kTF32 || p.res_fp32) {  // plain fp32 (also the tf32 activation format, whose loads need no rounding)
              if (full) {
                add_res_chunk<kTF32>(rbuf, v);
              } else {
                const float* rp = reinterpret_cast<const float*>(p.res) + roff + nb;
                for (int i = 0; i < 32; ++i) if (nb + i < p.N) v[i] += rp[i];
              }
            } else {
              if (full) {
                add_res_chunk<P>(rbuf, v);
              } else {
                const ActElem<P>* rp = reinterpret_cast<const ActElem<P>*>(p.res) + roff + nb;
                for (int i = 0; i < 32; ++i) if (nb + i < p.N) v[i] += load_split<P>(rp + i, p.res_lo_off);
              }
            }
          }
          if (!tma_epi && ch + kChunkStep < kChunks) prefetch_res(ch + kChunkStep);  // lands while this chunk is stored / reduced
          if (tma_epi) {
            // over the residual bytes this thread has read; rows outside the grid are clipped by the store
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const uint4 h = bf16x8_encode(v + 8 * i);
              *reinterpret_cast<uint4*>(eslot + eoff(i)) = h;
              if constexpr (P == kBF16X3) *reinterpret_cast<uint4*>(eslot + kEpiBoxBytes + eoff(i)) = bf16x8_encode_lo(h, v + 8 * i);
            }
          } else if (valid) {
            if (p.out_fp32) {
              float* op = reinterpret_cast<float*>(p.out) + ooff + nb;
              if (full) {
#pragma unroll
                for (int i = 0; i < 8; ++i) reinterpret_cast<float4*>(op)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
              } else {
                for (int i = 0; i < 32; ++i) if (nb + i < p.N) op[i * p.ocs] = v[i];
              }
            } else {
              ActElem<P>* op = reinterpret_cast<ActElem<P>*>(p.out) + ooff + nb;
              if (full) {
                constexpr int E = kVecElems<P>;
#pragma unroll
                for (int i = 0; i < 32 / E; ++i) store_vec<P>(op + E * i, p.out_lo_off * (long long)sizeof(ActElem<P>), v + E * i);
              } else {
                for (int i = 0; i < 32; ++i) if (nb + i < p.N) store_split<P>(op + i * p.ocs, p.out_lo_off, v[i]);
              }
            }
          }
          if (GNB ? (want_cols != 0) : (p.stats != nullptr)) {  // (never reached in split-K mode)
            float s[32], ss[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const float t = valid ? v[i] : 0.f;
              s[i] = t; ss[i] = GNB ? q2[GNB ? i : 0] : t * t;
            }
            colsum_butterfly<16>(s, ss, lane);
            // per-warp slot, no atomics: the cross-warp sum below runs in a fixed order (deterministic results)
            s_part[(q * 2 + 0) * BLOCK_N + ch * 32 + lane] = s[0];
            s_part[(q * 2 + 1) * BLOCK_N + ch * 32 + lane] = ss[0];
          }
        }
        if constexpr (kHasTmaEpi<BLOCK_N, P, GNB>) {
          if (tma_epi) {
            fence_proxy_async();  // this thread's output bytes, visible to the TMA store
            named_bar_sync(2, kEpiThreads);
            if (et == 0) {
              // TMA clips the box at the grid and at N (a round wholly past N stores nothing)
              const int c = n0 + rnd * Cfg::kStageCols;
              const uint32_t src = b_ring + eslot_i * b_slot;
              if (c < p.N) {
                tma_store_5d(&p.omap[0], src, c, x0, y0, z0, b0);
                if constexpr (P == kBF16X3) tma_store_5d(&p.omap[1], src + kEpiBoxBytes, c, x0, y0, z0, b0);
              }
              bulk_commit();
              // the previous round's slot goes back to the producer once its store has read it; nothing waits for the
              // global writes
              if (epi_pend >= 0) {
                bulk_wait_read<1>();
                mbar_arrive(b_empty + 8 * epi_pend);
                mbar_arrive(b_empty + 8 * epi_pend);
              }
              epi_pend = eslot_i;
            }
          }
        }
        MDB_STAMP(2 + rnd);
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
      MDB_STAMP(4);
    }
    if constexpr (kHasTmaEpi<BLOCK_N, P, GNB>) {
      if (et == 0 && epi_pend >= 0) bulk_wait<0>();  // the shared memory outlives the last store
    }
  }
}

}  // namespace mdb
