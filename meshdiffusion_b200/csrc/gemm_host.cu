// Host-side builders for the wgmma implicit-GEMM kernel (see gemm_tc.cuh).
#include "gemm_host.h"
#include "elementwise.cuh"
#include <cstring>
#include <cstdlib>
#include <mutex>

namespace mdb {

// ------------------------------------------------------------------ driver entry point (no libcuda link dependency)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !f)
      throw std::runtime_error("mdb: cuTensorMapEncodeTiled not available (needs an sm_90+ driver)");
    fn = reinterpret_cast<PFN_encodeTiled>(f);
  });
  return fn;
}

void encode_map(CUtensorMap* m, Precision prec, const MapDesc& d) {
  cuuint64_t gd[5], gs[4];
  cuuint32_t bd[5], es[5];
  for (int i = 0; i < d.rank; ++i) { gd[i] = d.dims[i]; bd[i] = d.box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < d.rank; ++i) gs[i] = d.strides[i];
  CUtensorMapDataType dt = prec == kTF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = get_encode()(m, dt, d.rank, d.base, gd, gs, bd, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::string msg = "mdb: cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ") rank " +
                      std::to_string(d.rank) + " dims";
    for (int i = 0; i < d.rank; ++i) msg += " " + std::to_string(d.dims[i]);
    msg += " box";
    for (int i = 0; i < d.rank; ++i) msg += " " + std::to_string(d.box[i]);
    throw std::runtime_error(msg);
  }
}

// ------------------------------------------------------------------ kernel instantiations
template <int BN, Precision P, bool GNB>
static void launch_impl(const GemmParams& p, int grid, int smem, cudaStream_t stream) {
  static bool configured[64] = {};  // the attribute is per device
  auto kern = gemm_tc_kernel<BN, P, GNB>;
  int dev = 0;
  MDB_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !configured[dev]) {
    MDB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    if (dev < 64) configured[dev] = true;
  }
  kern<<<grid, kGemmThreads, smem, stream>>>(p);
  MDB_CUDA_CHECK(cudaGetLastError());
}

struct GemmVariant {
  void (*launch)(const GemmParams&, int grid, int smem, cudaStream_t);
  int fixed_bytes;  // GemmCfg::kFixedBytes: the shared memory next to the operand rings
};
template <int BN, Precision P, bool GNB>
static GemmVariant variant() { return {launch_impl<BN, P, GNB>, GemmCfg<BN, GNB>::kFixedBytes}; }
template <int BN>
static GemmVariant variant(Precision prec, bool gnb) {
  if (gnb) {
    if (prec == kTF32) throw std::runtime_error("mdb: the GroupNorm-backward epilogue is built for bf16 / split-bf16 operands");
    return prec == kBF16X3 ? variant<BN, kBF16X3, true>() : variant<BN, kBF16, true>();
  }
  return prec == kTF32 ? variant<BN, kTF32, false>() : prec == kBF16X3 ? variant<BN, kBF16X3, false>() : variant<BN, kBF16, false>();
}
// the one choice of kernel instantiation for (BLOCK_N, operand mode, GroupNorm-backward epilogue)
static GemmVariant gemm_variant(int block_n, Precision prec, bool gnb) {
  return block_n == 32 ? variant<32>(prec, gnb) : variant<128>(prec, gnb);
}

int GemmOp::pick_slots(GemmParams& q) const {
  // Operand rings of this op in the shared memory left next to the epilogue scratch: two slots of each at least (one
  // filling while one is read). Then B slots are added until they cover the k-steps of every A slot in flight, and A slots
  // (entries in flight) up to MDB_MAX_STAGES (default 4), whichever is behind and still fits. MDB_MAX_BSLOTS caps the B
  // slots (weight lookahead) the same way; both change timing only, never results.
  const int fixed = gemm_variant(block_n, prec, gnb).fixed_bytes;
  const int budget = kMaxDynSmem - fixed;
  q.a_slot_bytes = (a_slot_need + 1023) / 1024 * 1024;
  q.b_slot_bytes = parts(prec) * block_n * kRowBytes;
  auto env_cap = [](const char* name, int def) {
    int cap = def;
    if (const char* e = getenv(name)) { const int c = atoi(e); if (c >= 2) cap = c; }
    return cap < kMaxSlots ? cap : kMaxSlots;
  };
  const int cap = env_cap("MDB_MAX_STAGES", 4), bcap = env_cap("MDB_MAX_BSLOTS", kMaxSlots);
  int na = 2, nb = 2;
  int used = na * q.a_slot_bytes + nb * q.b_slot_bytes;
  if (used > budget) throw std::runtime_error("mdb: operand rings need at least two slots each");
  for (;;) {
    if (nb < na * nk_max && nb < bcap && used + q.b_slot_bytes <= budget) { ++nb; used += q.b_slot_bytes; }
    else if (na < cap && used + q.a_slot_bytes <= budget) { ++na; used += q.a_slot_bytes; }
    else break;
  }
  q.n_aslots = na;
  q.n_bslots = nb;
  return fixed + used;
}

void GemmOp::slots(int& a_slots, int& b_slots, int& smem_bytes) const {
  GemmParams q = p;
  smem_bytes = pick_slots(q);
  a_slots = q.n_aslots;
  b_slots = q.n_bslots;
}

double GemmOp::fill_bytes(int B) const {
  // bytes TMA writes into shared memory for one launch: every entry's A box(es) and weight tiles, once per output tile
  // (split-K only divides the entries between CTAs)
  double per_tile = 0;
  for (const auto& e : loads) per_tile += parts(prec) * ((double)e.rows * kRowBytes + (double)e.nk * block_n * kRowBytes);
  const int tb = B > 0 ? (B + p.bb - 1) / p.bb : p.tb;
  return per_tile * p.tx * p.ty * p.tz * tb * p.n_tiles_n;
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    MDB_CUDA_CHECK(cudaGetDevice(&dev));
    MDB_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}

Geometry pick_geometry(int X, int Y, int Z) {
  if (Y == 1 && Z == 1) return {128, 1, 1, 1};
  int bx = X < 8 ? X : 8;
  int by = 128 / bx;
  if (by > 16) by = 16;
  if (by > Y) by = Y;
  int rem = 128 / (bx * by);
  int bz = rem < Z ? rem : Z;
  int bb = rem / bz;
  return {bx, by, bz, bb};
}

int plan_splits(int X, int Y, int Z, int B, int N, int cin_total, int taps, Precision prec) {
  const Geometry g = pick_geometry(X, Y, Z);
  const int tiles_m = ((X + g.bx - 1) / g.bx) * ((Y + g.by - 1) / g.by) * ((Z + g.bz - 1) / g.bz) * ((B + g.bb - 1) / g.bb);
  const int block_n = N <= 32 ? 32 : 128;
  const int tiles = tiles_m * ((N + block_n - 1) / block_n);
  // work per tile in k-step products: a split-bf16 k-step is three of them (hi.hi, hi.lo, lo.hi)
  const int kprod = ((cin_total + kb_elems(prec) - 1) / kb_elems(prec)) * taps * (prec == kBF16X3 ? 3 : 1);
  if (tiles > 49 || kprod < 48) return 1;
  int S = kPlanSMs / tiles;
  if (S > 16) S = 16;
  if (S > kprod / 8) S = kprod / 8;
  return S < 2 ? 1 : S;
}

void GemmOp::enable_splits(int S, float* scratch) {
  if (S <= 1) return;
  if (p.ocs != 1 || p.out_fp32 || p.bias_on_m || p.alpha != 1.f || p.res_fp32)
    throw std::runtime_error("mdb: split-K is only wired for plain NDHWC conv outputs");
  if (p.osx != (long long)p.N * parts(prec) || (p.rsx && p.rsx != (long long)p.N * parts(prec)))
    throw std::runtime_error("mdb: split-K needs dense [B][V][N] output / residual");
  splits = S;
  p.splits = S;
  p.partial = scratch;
  p.split_stride = (long long)p.Bn * p.X * p.Y * p.Z * p.N;
}

#ifdef MDB_EPI_TRACE
std::vector<const GemmOp*>& trace_registry() {
  static std::vector<const GemmOp*> ops;
  return ops;
}
// Instrumented build only (not part of the C ABI): the epilogue stamps of the last launch of uploaded op i, as
// [kTraceCtas][kTraceTiles][kTraceStamps] nanoseconds (0 = not reached), and its name. Returns -1 past the last op.
extern "C" int mdb_epi_trace_read(int i, char* name, int name_cap, unsigned long long* out) {
  auto& ops = trace_registry();
  if (i < 0 || i >= (int)ops.size()) return -1;
  snprintf(name, name_cap, "%s", ops[i]->name.c_str());
  if (cudaMemcpy(out, ops[i]->d_trace, sizeof(unsigned long long) * kTraceCtas * kTraceTiles * kTraceStamps,
                 cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
  return kTraceCtas * kTraceTiles * kTraceStamps;
}
extern "C" int mdb_epi_trace_dims(int* ctas, int* tiles, int* stamps) {
  *ctas = kTraceCtas; *tiles = kTraceTiles; *stamps = kTraceStamps;
  return 0;
}
#endif

GemmOp::~GemmOp() {
#ifdef MDB_EPI_TRACE
  auto& ops = trace_registry();
  for (size_t i = 0; i < ops.size(); ++i) if (ops[i] == this) { ops.erase(ops.begin() + i); break; }
  if (d_trace) cudaFree(d_trace);
#endif
  if (d_loads) cudaFree(d_loads);
  if (d_ks0) cudaFree(d_ks0);
  if (d_wpacked && owns_w) cudaFree(d_wpacked);
}

// Logical element strides (sx, sy, sz, sb) of an epilogue tensor -> physical ones; returns the offset of the lo parts.
// Split-bf16 rows are (hi, lo) pairs: physical pitches twice the logical ones, lo parts lo_off (logical) elements behind.
static long long physical_strides(bool split, long long lo_off, long long& sx, long long& sy, long long& sz, long long& sb) {
  if (!split) return 0;
  sx *= 2; sy *= 2; sz *= 2; sb *= 2;
  return lo_off;
}

void GemmOp::set_output_strided(Precision pr, int X, int Y, int Z, int B, int N, void* out, long long osx,
                                long long osy, long long osz, long long osb, bool out_fp32, long long lo_off) {
  prec = pr;
  geo = pick_geometry(X, Y, Z);
  if (geo.bx * geo.by * geo.bz * geo.bb != kBlockM) throw std::runtime_error("mdb: unsupported tile geometry");
  if (geo.bb > 1 && (geo.bx * geo.by * geo.bz) % 32 != 0)
    throw std::runtime_error("mdb: multi-sample tiles need a multiple of 32 rows per sample");
  if (geo.bb > 4) throw std::runtime_error("mdb: at most 4 samples per tile");
  p.bx = geo.bx; p.by = geo.by; p.bz = geo.bz; p.bb = geo.bb;
  p.X = X; p.Y = Y; p.Z = Z; p.Bn = B;
  p.tx = (X + geo.bx - 1) / geo.bx; p.ty = (Y + geo.by - 1) / geo.by;
  p.tz = (Z + geo.bz - 1) / geo.bz; p.tb = (B + geo.bb - 1) / geo.bb;
  p.N = N;
  block_n = N <= 32 ? 32 : 128;
  p.n_tiles_n = (N + block_n - 1) / block_n;
  p.out = out;
  p.osx = osx; p.osy = osy; p.osz = osz; p.osb = osb;
  p.out_fp32 = out_fp32 ? 1 : 0;
  p.out_lo_off = physical_strides(prec == kBF16X3 && !out_fp32, lo_off >= 0 ? lo_off : osx, p.osx, p.osy, p.osz, p.osb);
  p.alpha = 1.f;
  p.ocs = 1;
  p.kb_elems = kb_elems(prec);
}

void GemmOp::set_output(Precision pr, int X, int Y, int Z, int B, int N, void* out, long long ldc, bool out_fp32) {
  set_output_strided(pr, X, Y, Z, B, N, out, ldc, ldc * X, ldc * X * Y, ldc * X * Y * Z, out_fp32);
}

MapDesc act_map(const Act& a, Precision prec, int part, Geometry box, int sub, int px, int py, int pz) {
  const long long es = esize(prec);
  const long long sx = a.row() * parts(prec) * es, sy = sx * a.X, sz = sy * a.Y, sb = sz * a.Z;  // physical, bytes
  MapDesc m;
  m.rank = 5;
  m.base = static_cast<char*>(a.ptr) + (long long)part * a.row() * es + px * sx + py * sy + pz * sz;
  m.dims[0] = a.C; m.dims[1] = (a.X - px + sub - 1) / sub; m.dims[2] = (a.Y - py + sub - 1) / sub;
  m.dims[3] = (a.Z - pz + sub - 1) / sub; m.dims[4] = a.B;
  m.strides[0] = sx * sub; m.strides[1] = sy * sub; m.strides[2] = sz * sub; m.strides[3] = sb;
  m.box[0] = kb_elems(prec); m.box[1] = box.bx; m.box[2] = box.by; m.box[3] = box.bz; m.box[4] = box.bb;
  return m;
}

int GemmOp::add_amap(const Act& a, int halo, int sub, int px, int py, int pz, int part) {
  if ((int)amaps_.size() >= kMaxAMaps) throw std::runtime_error("mdb: too many A tensor maps");
  if (halo > 0 && (geo.bz != 1 || geo.bb != 1)) throw std::runtime_error("mdb: halo needs a (bx,by,1,1) tile");
  amaps_.push_back(act_map(a, prec, part, {geo.bx, geo.by + halo, geo.bz, geo.bb}, sub, px, py, pz));
  return (int)amaps_.size() - 1;
}

void GemmOp::add_load_x(int tm_hi, int tm_lo, int nk, int rows, int jrows, int dx, int dy, int dz, int c0, int wsrc,
                        int wc0, int tap0, int tapj) {
  if ((int)loads.size() >= kMaxLoads) throw std::runtime_error("mdb: load table overflow");
  if (rows > kAStageRows) throw std::runtime_error("mdb: A box exceeds the stage size");
  LoadEntry e{};
  e.tmap = (uint8_t)tm_hi; e.tmap_lo = (uint8_t)(prec == kBF16X3 ? tm_lo : tm_hi);
  e.nk = (uint8_t)nk; e.rows = (uint8_t)rows; e.jrows = (uint8_t)jrows;
  e.dx = (int8_t)dx; e.dy = (int8_t)dy; e.dz = (int8_t)dz; e.wsrc = (uint8_t)wsrc;
  e.c0 = (uint16_t)c0; e.wc0 = (uint16_t)wc0; e.tap0 = (uint8_t)tap0; e.tapj = (uint8_t)tapj;
  loads.push_back(e);
  ksteps += nk;
}

void GemmOp::add_conv(const std::vector<Act>& srcs, const float* w, int k, int stride) {
  int ctot = 0;
  for (auto& s : srcs) ctot += s.C;
  const int T = k * k * k;
  add_conv_w(srcs, WSrc{w, 1LL * ctot * T, (long long)T, 1, ctot}, k, stride);
}

// Data gradient of a stride-1 k^3 convolution = the same convolution over dY with the weight transposed (Cout <-> Cin)
// and every tap mirrored: W'[ci][co][tap] = W[co][ci][T-1-tap].
void GemmOp::add_conv_dgrad(const Act& dy, const float* w_oidhw, int cin_total, int k) {
  const int T = k * k * k;
  add_conv_w({dy}, WSrc{w_oidhw + (T - 1), (long long)T, 1LL * cin_total * T, -1, dy.C}, k, 1);
}

void GemmOp::add_conv_w(const std::vector<Act>& srcs, const WSrc& wsrc, int k, int stride) {
  const int KB = kb_elems(prec);
  int ctot = 0;
  for (auto& s : srcs) ctot += s.C;
  const int T = k * k * k;
  const int ws = add_wsrc(wsrc);
  const int pad = k / 2;
  flops += 2.0 * p.X * p.Y * p.Z * p.Bn * (double)p.N * ctot * T;
  int coff = 0;
  if (stride == 1) {
    const bool reuse = geo.bz == 1 && geo.bb == 1 && geo.bx * (geo.by + k - 1) <= kAStageRows && p.Y >= geo.by;
    const bool x3 = prec == kBF16X3;
    for (auto& s : srcs) {
      const int tm = add_amap(s, reuse ? k - 1 : 0);
      const int tl = x3 ? add_amap(s, reuse ? k - 1 : 0, 1, 0, 0, 0, 1) : tm;
      for (int c0 = 0; c0 < s.C; c0 += KB) {
        if (reuse) {
          for (int dz = 0; dz < k; ++dz)
            for (int dx = 0; dx < k; ++dx)
              add_load_x(tm, tl, k, geo.bx * (geo.by + k - 1), geo.bx, dx - pad, -pad, dz - pad, c0, ws, coff + c0,
                         (dz * k) * k + dx, k);
        } else {
          for (int dz = 0; dz < k; ++dz)
            for (int dy = 0; dy < k; ++dy)
              for (int dx = 0; dx < k; ++dx)
                add_load_x(tm, tl, 1, kBlockM, 0, dx - pad, dy - pad, dz - pad, c0, ws, coff + c0, (dz * k + dy) * k + dx, 0);
        }
      }
      coff += s.C;
    }
  } else if (stride == 2) {
    // layers.py:626-643: pad one voxel on the high side only, then stride-2 VALID conv: in = 2*o + d.
    // Tap d reads the parity-(d&1) sub-grid at coordinate o + (d>>1); coordinate == sub-grid size -> zero fill = pad.
    if (k != 3) throw std::runtime_error("mdb: stride-2 conv supports k=3 only");
    const bool x3 = prec == kBF16X3;
    for (auto& s : srcs) {
      int tm[8], tl[8];
      for (int par = 0; par < 8; ++par) tm[par] = add_amap(s, 0, 2, par & 1, (par >> 1) & 1, (par >> 2) & 1);
      for (int par = 0; par < 8; ++par) tl[par] = x3 ? add_amap(s, 0, 2, par & 1, (par >> 1) & 1, (par >> 2) & 1, 1) : tm[par];
      for (int c0 = 0; c0 < s.C; c0 += KB)
        for (int dz = 0; dz < 3; ++dz)
          for (int dy = 0; dy < 3; ++dy)
            for (int dx = 0; dx < 3; ++dx) {
              const int par = (dx & 1) | ((dy & 1) << 1) | ((dz & 1) << 2);
              add_load_x(tm[par], tl[par], 1, kBlockM, 0, dx >> 1, dy >> 1, dz >> 1, c0, ws, coff + c0, (dz * 3 + dy) * 3 + dx, 0);
            }
      coff += s.C;
    }
  } else {
    throw std::runtime_error("mdb: unsupported stride");
  }
}

void GemmOp::add_conv_up2(const Act& s, const float* w8, int px, int py, int pz) {
  const int KB = kb_elems(prec);
  const int ws = add_wsrc(WSrc{w8, 8LL * s.C, 8, 1, s.C});
  flops += 2.0 * p.X * p.Y * p.Z * p.Bn * (double)p.N * s.C * 8;
  const bool x3 = prec == kBF16X3;
  // effective tap e in {0,1} of an axis with output parity q reads the input at offset e - 1 + q
  const bool reuse = geo.bz == 1 && geo.bb == 1 && geo.bx * (geo.by + 1) <= kAStageRows && p.Y >= geo.by;
  const int tm = add_amap(s, reuse ? 1 : 0);
  const int tl = x3 ? add_amap(s, reuse ? 1 : 0, 1, 0, 0, 0, 1) : tm;
  for (int c0 = 0; c0 < s.C; c0 += KB) {
    for (int ez = 0; ez < 2; ++ez)
      for (int ex = 0; ex < 2; ++ex) {
        if (reuse) {  // the two y-taps share one box with a 1-row halo
          add_load_x(tm, tl, 2, geo.bx * (geo.by + 1), geo.bx, ex - 1 + px, -1 + py, ez - 1 + pz, c0, ws, c0, (ez * 2) * 2 + ex, 2);
        } else {
          for (int ey = 0; ey < 2; ++ey)
            add_load_x(tm, tl, 1, kBlockM, 0, ex - 1 + px, ey - 1 + py, ez - 1 + pz, c0, ws, c0, (ez * 2 + ey) * 2 + ex, 0);
        }
      }
  }
}

void GemmOp::add_pointwise(const std::vector<Act>& srcs, const float* w, bool w_in_out) {
  int ctot = 0;
  for (auto& s : srcs) ctot += s.C;
  WSrc ws = w_in_out ? WSrc{w, 1, (long long)p.N, 0, ctot} : WSrc{w, (long long)ctot, 1, 0, ctot};
  add_pointwise_w(srcs, &ws);
}

void GemmOp::add_pointwise_w(const std::vector<Act>& srcs, const WSrc* w) {
  const int KB = kb_elems(prec);
  int ctot = 0;
  for (auto& s : srcs) ctot += s.C;
  int ws = 0;
  if (w) ws = add_wsrc(*w);
  flops += 2.0 * p.X * p.Y * p.Z * p.Bn * (double)p.N * ctot;
  int coff = 0;
  for (auto& s : srcs) {
    const int tm = add_amap(s, 0);
    const int tl = prec == kBF16X3 ? add_amap(s, 0, 1, 0, 0, 0, 1) : tm;
    for (int c0 = 0; c0 < s.C; c0 += KB) add_load_x(tm, tl, 1, kBlockM, 0, 0, 0, 0, c0, ws, coff + c0, 0, 0);
    coff += s.C;
  }
}

void GemmOp::set_residual(const void* res, long long ldr, long long batch_stride, bool fp32) {
  p.res = res;
  p.batch_fastest = batch_stride == 0 ? 1 : 0;  // a residual shared by every sample: keep its slice L2-resident
  p.rsx = ldr; p.rsy = ldr * p.X; p.rsz = ldr * p.X * p.Y; p.rsb = batch_stride;
  p.res_fp32 = fp32 ? 1 : 0;
  p.res_lo_off = physical_strides(prec == kBF16X3 && !fp32, ldr, p.rsx, p.rsy, p.rsz, p.rsb);
}

void GemmOp::set_gn_backward(const void* x0, long long ld0, int c0, const void* x1, long long ld1, const void* consts, int silu,
                             float* part) {
  if (prec == kTF32 || p.out_fp32 || p.ocs != 1)
    throw std::runtime_error("mdb: the GroupNorm-backward epilogue is built for bf16 / split-bf16 NDHWC outputs");
  if (p.N % 32 != 0 || (ld1 > 0 && c0 % 32 != 0)) throw std::runtime_error("mdb: GroupNorm-backward epilogue needs 32-channel aligned sources");
  if (splits > 1) throw std::runtime_error("mdb: GroupNorm-backward epilogue cannot be combined with split-K");
  gnb = true;
  p.res = x0; p.res_fp32 = 0; p.batch_fastest = 0;
  p.rsx = ld0; p.rsy = ld0 * p.X; p.rsz = ld0 * p.X * p.Y; p.rsb = ld0 * p.X * p.Y * p.Z;
  p.res1 = x1; p.res_c0 = ld1 > 0 ? c0 : p.N;
  p.r1sx = ld1; p.r1sy = ld1 * p.X; p.r1sz = ld1 * p.X * p.Y; p.r1sb = ld1 * p.X * p.Y * p.Z;
  p.res_lo_off = physical_strides(prec == kBF16X3, ld0, p.rsx, p.rsy, p.rsz, p.rsb);
  p.res1_lo_off = physical_strides(prec == kBF16X3, ld1, p.r1sx, p.r1sy, p.r1sz, p.r1sb);
  p.gnb_c = reinterpret_cast<const float4*>(consts);
  p.gnb_silu = silu;
  p.gnb_part = part;
}

MapDesc GemmOp::b_desc(void* ptr, long long K, int N, int batch, long long rsb, long long bsb) const {
  MapDesc m;
  m.base = ptr; m.rank = 3;
  m.dims[0] = (uint64_t)K; m.dims[1] = (uint64_t)N; m.dims[2] = (uint64_t)batch;
  m.strides[0] = (uint64_t)rsb; m.strides[1] = (uint64_t)bsb;
  m.box[0] = (uint32_t)kb_elems(prec); m.box[1] = (uint32_t)block_n; m.box[2] = 1;
  return m;
}

void GemmOp::set_b_activation(void* ptr, int K, int N, int batch, long long rs, long long bs) {
  b_from_act = true;
  p.b_batched = 1;
  const long long es = esize(prec);
  if (prec == kBF16X3) {
    // rows are (hi, lo) pairs: the lo parts are addressed as K coordinates [rs, rs + K) of the same map
    if (K % kb_elems(prec) != 0) throw std::runtime_error("mdb: X3 activation-B operands need K to be a multiple of 64");
    b_lo_off = rs;
    bmap_ = b_desc(ptr, (int)(rs + K), N, batch, 2 * rs * es, 2 * bs * es);
    return;
  }
  bmap_ = b_desc(ptr, K, N, batch, rs * es, bs * es);
}

// ------------------------------------------------------------------ weight packing (device gather)
struct PackWSrc { const float* ptr; long long sn, sc, st; int cvalid; int ndiv; long long sn_hi; int cdiv; long long sc_hi; };
struct PackArgs { PackWSrc w[4]; };

// split bf16: every k-step is packed as its hi = bf16(w) tile followed by its lo = bf16(w - hi) tile (K columns
// [2 ks KB, 2 ks KB + KB) and [2 ks KB + KB, 2 (ks + 1) KB)).
// One thread = 8 consecutive K elements (one 16- / 32-byte store) of EVERY k-step of one load entry for one output row: the
// entry / source / offset arithmetic is done once per 8 * nk outputs. (The first version, one thread per packed element with
// two 64-bit divisions and a table walk each, made the per-optimiser-step re-pack of the training engine instruction-bound:
// 6-8 ms for 2.9 GB of traffic.)
template <Precision P>
__global__ void __launch_bounds__(256) pack_weights_kernel(const LoadEntry* __restrict__ loads, const int* __restrict__ load_ks0,
                                                         int n_loads, const __grid_constant__ PackArgs args, int N, int ksteps,
                                                         int KB, void* __restrict__ out) {
  const int vpk = KB >> 3;  // 8-element vectors per k-step
  const long long total = 1LL * N * n_loads * vpk;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int v8 = (int)(idx % vpk);
    const long long t = idx / vpk;
    const int l = (int)(t % n_loads);
    const int n = (int)(t / n_loads);
    const LoadEntry e = loads[l];
    const PackWSrc& w = args.w[e.wsrc];
    const long long noff = w.ndiv ? (long long)(n % w.ndiv) * w.sn + (long long)(n / w.ndiv) * w.sn_hi : (long long)n * w.sn;
    const int c0 = e.wc0 + v8 * 8;
    long long coff[8];  // (may be negative: mirrored sources point at their last tap and walk backwards)
    unsigned valid = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c0 + i;
      if (c < w.cvalid) valid |= 1u << i;
      coff[i] = noff + (w.cdiv ? (long long)(c % w.cdiv) * w.sc + (long long)(c / w.cdiv) * w.sc_hi : (long long)c * w.sc);
    }
    const long long obase = ((long long)n * ksteps + load_ks0[l]) * parts(P) * KB + v8 * 8;
    for (int j = 0; j < e.nk; ++j) {
      const long long toff = (long long)(e.tap0 + j * e.tapj) * w.st;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = (valid >> i) & 1u ? __ldg(w.ptr + coff[i] + toff) : 0.f;
      ActElem<P>* op = reinterpret_cast<ActElem<P>*>(out) + obase + (long long)j * parts(P) * KB;
      constexpr int E = kVecElems<P>;
#pragma unroll
      for (int i = 0; i < 8 / E; ++i) store_vec<P>(op + E * i, (long long)KB * sizeof(ActElem<P>), v + E * i);
    }
  }
}

void GemmOp::repack(cudaStream_t stream) {
  if (b_from_act) return;
  if (!d_ks0) {  // first k-step of every load entry: built once, reused by every re-pack
    std::vector<int> ks0;
    int run = 0;
    for (size_t l = 0; l < loads.size(); ++l) { ks0.push_back(run); run += loads[l].nk; }
    if (run != ksteps) throw std::runtime_error("mdb: load table does not cover the packed K extent");
    MDB_CUDA_CHECK(cudaMalloc(&d_ks0, ks0.size() * sizeof(int)));
    MDB_CUDA_CHECK(cudaMemcpy(d_ks0, ks0.data(), ks0.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  if (wsrcs.size() > 4) throw std::runtime_error("mdb: too many weight sources");
  PackArgs args{};
  for (size_t i = 0; i < wsrcs.size(); ++i) args.w[i] = {wsrcs[i].ptr, wsrcs[i].sn, wsrcs[i].sc, wsrcs[i].st, wsrcs[i].cvalid, wsrcs[i].ndiv, wsrcs[i].sn_hi, wsrcs[i].cdiv, wsrcs[i].sc_hi};
  const int KB = kb_elems(prec), n_loads = (int)loads.size();
  const long long total = 1LL * p.N * n_loads * (KB / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > kPlanSMs * 16) blocks = kPlanSMs * 16;
  if (prec == kTF32)
    pack_weights_kernel<kTF32><<<blocks, 256, 0, stream>>>(d_loads, d_ks0, n_loads, args, p.N, ksteps, KB, d_wpacked);
  else if (prec == kBF16X3)
    pack_weights_kernel<kBF16X3><<<blocks, 256, 0, stream>>>(d_loads, d_ks0, n_loads, args, p.N, ksteps, KB, d_wpacked);
  else
    pack_weights_kernel<kBF16><<<blocks, 256, 0, stream>>>(d_loads, d_ks0, n_loads, args, p.N, ksteps, KB, d_wpacked);
  MDB_CUDA_CHECK(cudaGetLastError());
}

void GemmOp::finalize() {
  if (loads.empty()) throw std::runtime_error("mdb: GemmOp without loads");
  p.b_explicit_k = 0;
  p.b_kstep = kb_elems(prec) * parts(prec);  // packed weights: a k-step's tiles sit side by side (X3: hi, lo)
  p.b_lo_k = kb_elems(prec);
  if (b_from_act) p.b_kstep = kb_elems(prec);
  if (b_from_act && prec == kBF16X3) {
    // activation-B operand in the split layout: every entry names the K coordinate of its B hi tile itself (wc0); the
    // lo parts of the rows are the K coordinates b_lo_off further on
    p.b_explicit_k = 1;
    p.b_lo_k = (int)b_lo_off;
  }
  if (!b_from_act) p.b_batched = 0;
  p.n_loads = (int)loads.size();
  if (p.splits < 1) p.splits = 1;
  // pipeline segments: runs of identical entries. An entry's A box (X3: both parts) takes an A slot, the weight tiles of
  // each of its k-steps a B slot; the A slot size is the largest box of this op.
  {
    a_slot_need = 0;
    nk_max = 0;
    p.n_segs = 0;
    p.total_groups = 0;
    size_t i = 0;
    while (i < loads.size()) {
      size_t j = i;
      while (j < loads.size() && loads[j].nk == loads[i].nk && loads[j].rows == loads[i].rows && loads[j].jrows == loads[i].jrows) ++j;
      if (p.n_segs >= kMaxSegs) throw std::runtime_error("mdb: too many pipeline segments");
      GemmSeg sg{};
      sg.n_groups = (int)(j - i); sg.nk = loads[i].nk;
      sg.a_bytes = loads[i].rows * kRowBytes;
      sg.a_stride = (sg.a_bytes + 1023) / 1024 * 1024;
      sg.jbytes = loads[i].jrows * kRowBytes;
      const int need = parts(prec) * sg.a_stride;
      if (sg.a_stride > kAStageBytes) throw std::runtime_error("mdb: A box exceeds the slot size");
      if (need > a_slot_need) a_slot_need = need;
      if (sg.nk > nk_max) nk_max = sg.nk;
      p.segs[p.n_segs++] = sg;
      p.total_groups += sg.n_groups;
      i = j;
    }
  }
  if (p.splits > p.total_groups) { p.splits = p.total_groups; splits = p.splits; }
}

// The TMA epilogue needs 128-column tiles of bf16 / split-bf16 rows stored whole (no split-K partials, no scalar column
// stride, no fp32 output), a residual in the same format with its own rows per sample, and tensor-map-compatible
// addresses: 16-byte aligned bases and strides. Every other launch keeps the per-thread stores.
bool GemmOp::epi_tma_ok(const GemmParams& p) const {
  if (gnb || block_n != 128 || prec == kTF32 || p.splits > 1 || p.ocs != 1 || p.out_fp32) return false;
  if (p.res && (p.res_fp32 || p.batch_fastest)) return false;
  const long long es = esize(prec);
  auto aligned = [&](const void* base, long long lo_off, long long sx, long long sy, long long sz, long long sb) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(base);
    return a % 16 == 0 && (lo_off * es) % 16 == 0 && (sx * es) % 16 == 0 && (sy * es) % 16 == 0 && (sz * es) % 16 == 0 &&
           (sb * es) % 16 == 0;
  };
  if (!aligned(p.out, prec == kBF16X3 ? p.out_lo_off : 0, p.osx, p.osy, p.osz, p.osb)) return false;
  if (p.res && !aligned(p.res, prec == kBF16X3 ? p.res_lo_off : 0, p.rsx, p.rsy, p.rsz, p.rsb)) return false;
  return true;
}

// Output and residual maps of the TMA epilogue at batch B: (N channels, X, Y, Z, B) over the (physical) element strides
// of the epilogue, boxes of one staging round (64 channels) by the M-tile; part 1 = the split-bf16 lo parts.
static MapDesc epi_map(const void* base, Precision prec, int part, long long lo_off, const GemmParams& q, int B, long long sx,
                       long long sy, long long sz, long long sb) {
  const long long es = esize(prec);
  MapDesc m;
  m.rank = 5;
  m.base = const_cast<char*>(static_cast<const char*>(base)) + (long long)part * lo_off * es;
  m.dims[0] = q.N; m.dims[1] = q.X; m.dims[2] = q.Y; m.dims[3] = q.Z; m.dims[4] = B;
  const long long st[4] = {sx * es, sy * es, sz * es, sb * es};
  // an axis of extent 1 is only ever addressed at 0: its stride (0 in some callers' views) is replaced by a valid one
  long long prev = es * q.N;
  for (int i = 0; i < 4; ++i) {
    m.strides[i] = (uint64_t)(m.dims[i + 1] == 1 ? prev : st[i]);
    prev = (long long)m.strides[i] * (long long)m.dims[i + 1];
  }
  m.box[0] = kRowBytes / es; m.box[1] = q.bx; m.box[2] = q.by; m.box[3] = q.bz; m.box[4] = q.bb;
  return m;
}

void GemmOp::encode_epi_maps(GemmParams& q, int B) const {
  for (int part = 0; part < parts(prec); ++part) {
    encode_map(&q.omap[part], prec, epi_map(q.out, prec, part, q.out_lo_off, q, B, q.osx, q.osy, q.osz, q.osb));
    if (q.res) encode_map(&q.rmap[part], prec, epi_map(q.res, prec, part, q.res_lo_off, q, B, q.rsx, q.rsy, q.rsz, q.rsb));
  }
}

void GemmOp::upload(cudaStream_t stream) {
  for (size_t i = 0; i < amaps_.size(); ++i) encode_map(&p.amap[i], prec, amaps_[i]);
  p.epi_tma = epi_tma_ok(p) ? 1 : 0;
  if (p.epi_tma && p.out) encode_epi_maps(p, p.Bn);
#ifdef MDB_EPI_TRACE
  // (instrumented build only: time the per-thread stores on the same launches)
  if (getenv("MDB_EPI_TRACE_PER_THREAD")) p.epi_tma = 0;
  MDB_CUDA_CHECK(cudaMalloc(&d_trace, sizeof(unsigned long long) * kTraceCtas * kTraceTiles * kTraceStamps));
  MDB_CUDA_CHECK(cudaMemset(d_trace, 0, sizeof(unsigned long long) * kTraceCtas * kTraceTiles * kTraceStamps));
  p.trace = d_trace;
  trace_registry().push_back(this);
#endif
  MDB_CUDA_CHECK(cudaMalloc(&d_loads, loads.size() * sizeof(LoadEntry)));
  MDB_CUDA_CHECK(cudaMemcpyAsync(d_loads, loads.data(), loads.size() * sizeof(LoadEntry), cudaMemcpyHostToDevice, stream));
  p.loads = d_loads;
  if (!b_from_act) {
    const long long ktot = 1LL * ksteps * kb_elems(prec) * parts(prec);
    const long long bytes = ktot * p.N * esize(prec);
    MDB_CUDA_CHECK(cudaMalloc(&d_wpacked, bytes));
    owns_w = true;
    bmap_ = b_desc(d_wpacked, ktot, p.N, 1, ktot * esize(prec), bytes);
  }
  encode_map(&p.bmap, prec, bmap_);
  MDB_CUDA_CHECK(cudaStreamSynchronize(stream));
}

void GemmOp::launch(cudaStream_t stream, int B, void* out_override) const {
  GemmParams p = this->p;
  const int smem = pick_slots(p);
  if (B > 0) {
    if (B > this->p.Bn) throw std::runtime_error("mdb: batch exceeds the batch the op was built for");
    p.Bn = B;
    p.tb = (B + p.bb - 1) / p.bb;
  }
  if (out_override) p.out = out_override;
  // the epilogue's maps clip at the launch's batch and address the launch's output
  if (p.epi_tma && (out_override || p.Bn != this->p.Bn)) {
    p.epi_tma = epi_tma_ok(p) ? 1 : 0;
    if (p.epi_tma) encode_epi_maps(p, p.Bn);
  }
  const int tiles_m = p.tx * p.ty * p.tz * p.tb;
  const int total = tiles_m * p.n_tiles_n * (p.splits > 1 ? p.splits : 1);
  const int grid = total < sm_count() ? total : sm_count();
  if (gnb) {
    if (p.splits > 1) throw std::runtime_error("mdb: GroupNorm-backward epilogue: no split-K");
    p.gnb_drop_thresh = rt_drop_thresh; p.gnb_drop_scale = rt_drop_scale; p.gnb_seed = rt_seed;
  }
  gemm_variant(block_n, prec, gnb).launch(p, grid, smem, stream);
  if (p.splits > 1) {
    SplitReduceArgs a{};
    a.partial = p.partial; a.split_stride = p.split_stride; a.splits = p.splits;
    a.bias = p.bias; a.rowbias = p.rowbias; a.rowbias_ld = p.rowbias_ld;
    a.res = p.res; a.res_batch_stride = p.rsb;
    a.out = p.out; a.stats = p.stats; a.voxels = (long long)p.X * p.Y * p.Z; a.N = p.N; a.prec = prec;
    if (prec == kBF16X3) a.res_batch_stride = p.rsb / 2;  // the reduction kernel takes logical strides
    launch_split_reduce(a, p.Bn, stream);
  }
}

}  // namespace mdb
