// Host-side construction of wgmma implicit-GEMM operations: TMA tensor maps, load tables, packed weights.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <stdexcept>
#include "gemm_tc.cuh"

namespace mdb {

#define MDB_CUDA_CHECK(expr)                                                                         \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      throw std::runtime_error(std::string("CUDA error ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" + \
                               std::to_string(__LINE__) + " (" #expr ")");                           \
  } while (0)

// kBF16X3 ("split bf16"): every fp32 value v is carried as a bf16 pair hi = bf16(v), lo = bf16(v - hi) and every product
// is evaluated as hi*hi + hi*lo + lo*hi into the same fp32 accumulator (three bf16 MMAs per k-step; the
// dropped lo*lo term is 2^-16 relative) -- fp32-class results (the mode that meets the 1e-3 parity contract) at
// one third of the bf16 tensor rate. An X3 tensor with a logical row pitch of `ld` channels occupies 2*ld bf16 per
// voxel: hi parts at [0, ld), lo parts at [ld, 2*ld). All pitches handed to GemmOp / Act stay LOGICAL.
enum Precision { kBF16 = 0, kTF32 = 1, kBF16X3 = 2 };
inline int esize(Precision p) { return p == kTF32 ? 4 : 2; }
inline int kb_elems(Precision p) { return kRowBytes / esize(p); }
inline int parts(Precision p) { return p == kBF16X3 ? 2 : 1; }
inline Precision precision_from_int(int v) {
  if (v < 0 || v > 2) throw std::runtime_error("mdb: precision must be 0 (bf16), 1 (tf32) or 2 (bf16x3)");
  return static_cast<Precision>(v);
}

// A dense NDHWC activation tensor (channels innermost).
struct Act {
  void* ptr = nullptr;
  int C = 0, X = 0, Y = 0, Z = 0, B = 0;
  long long ld = 0;  // (logical) elements between consecutive voxels (0 = dense, i.e. C)
  long long row() const { return ld ? ld : C; }
  long long voxels() const { return 1LL * X * Y * Z; }
  long long elems() const { return voxels() * B * C; }
};

// A weight tensor addressed as W[n*sn + c*sc + tap*st]; channels >= cvalid read as zero (K padding).
struct WSrc {
  const float* ptr = nullptr;
  long long sn = 0, sc = 0, st = 0;
  int cvalid = 0;
  // optional split of the output index: n -> (n / ndiv, n % ndiv) addressed with strides (sn_hi, sn)
  int ndiv = 0;
  long long sn_hi = 0;
  // optional split of the channel index: c -> (c / cdiv, c % cdiv) addressed with strides (sc_hi, sc)
  int cdiv = 0;
  long long sc_hi = 0;
};

struct Geometry { int bx, by, bz, bb; };
Geometry pick_geometry(int X, int Y, int Z);

class GemmOp {
 public:
  GemmParams p{};
  Precision prec = kBF16;
  int block_n = 128;
  int splits = 1;     // split-K factor (small problems: few tiles, long K)
  std::vector<LoadEntry> loads;
  std::vector<WSrc> wsrcs;
  int n_amaps = 0;
  int ksteps = 0;
  // device-owned
  LoadEntry* d_loads = nullptr;
  int* d_ks0 = nullptr;      // (weight packer) first k-step of every load entry
  void* d_wpacked = nullptr;  // [N][ksteps*KB] in activation dtype
  bool owns_w = false;
  double flops = 0;  // algorithmic FLOPs of one launch (2*M*N*K over valid taps, counted densely)
  std::string name;

  ~GemmOp();
  GemmOp() = default;
  GemmOp(const GemmOp&) = delete;
  GemmOp& operator=(const GemmOp&) = delete;

  // output geometry; must be called first
  void set_output(Precision prec, int X, int Y, int Z, int B, int N, void* out, long long ldc, bool out_fp32);
  // lo_off (X3 only): logical distance from the hi to the lo parts of an output row; default = osx (dense rows)
  void set_output_strided(Precision prec, int X, int Y, int Z, int B, int N, void* out, long long osx, long long osy,
                          long long osz, long long osb, bool out_fp32, long long lo_off = -1);
  // adds a 5-D A tensor map over `a` (optionally a stride-2 parity sub-grid) with a (KB, bx, by+halo, bz, bb) box.
  // part: 0 = the tensor itself / the hi parts of an X3 tensor, 1 = its lo parts
  int add_amap(const Act& a, int halo_rows_y, int sub_stride = 1, int px = 0, int py = 0, int pz = 0, int part = 0);
  void add_load(int tmap, int nk, int rows, int jrows, int dx, int dy, int dz, int c0, int wsrc, int wc0, int tap0,
                int tapj, int wpart = 0);
  // one logical A load -> 1 table entry (bf16 / tf32) or the 3 entries of the split product (X3): (A hi, W hi),
  // (A hi, W lo), (A lo, W hi); tm_lo is the tensor map of the lo parts
  void add_load_x(int tm_hi, int tm_lo, int nk, int rows, int jrows, int dx, int dy, int dz, int c0, int wsrc, int wc0,
                  int tap0, int tapj);
  int add_wsrc(const WSrc& w) { wsrcs.push_back(w); return (int)wsrcs.size() - 1; }

  // Dense k^3 convolution (cross-correlation, zero padding k/2, stride 1 or 2 [pad-high variant]) over the channel
  // concatenation of `srcs`; weight OIDHW fp32 [N][sum C][k^3].
  void add_conv(const std::vector<Act>& srcs, const float* w_oidhw, int ksize, int stride);
  void add_conv_w(const std::vector<Act>& srcs, const WSrc& w, int ksize, int stride);
  // One output-parity class of Upsample (nearest x2, layers.py:611-623) followed by its 3^3 convolution, evaluated on the
  // LOW-resolution input: output voxel 2h+p sees only two distinct input voxels per axis (h-1, h for p = 0; h, h+1 for
  // p = 1), so the 27 taps collapse to a 2^3 kernel whose weights are sums of the original ones (w8: [N][C][2][2][2] fp32,
  // built by launch_upconv_weights). The op's output geometry must be the low-resolution grid with strides into the
  // high-resolution tensor (set_output_strided). 8/27 of the FLOPs, and the 8x larger tensor is never materialised.
  void add_conv_up2(const Act& src, const float* w8, int px, int py, int pz);
  // conv data gradient: N = cin_total of the forward conv, A = dY (C = forward Cout), weight fp32 OIDHW of the forward
  void add_conv_dgrad(const Act& dy, const float* w_oidhw, int cin_total, int ksize);
  // 1x1x1 projection of the channel concatenation of `srcs` with W[in][out] (NIN layout) or [out][in] (Linear/conv).
  void add_pointwise(const std::vector<Act>& srcs, const float* w, bool w_in_out);
  // same with an explicit weight view (nullptr = no packed weights: B comes from set_b_activation)
  void add_pointwise_w(const std::vector<Act>& srcs, const WSrc* w);

  // B operand taken from a runtime activation matrix instead of packed weights: Bm[batch][N][K] (K-major).
  // (X3: logical strides; the lo parts of a row sit row_stride_elems behind its hi parts)
  void set_b_activation(void* ptr, int K, int N, int batch, long long row_stride_elems, long long batch_stride_elems);

  void set_bias(const float* bias, bool on_m = false) { p.bias = bias; p.bias_on_m = on_m ? 1 : 0; }
  void set_rowbias(const float* rb, long long ld) { p.rowbias = rb; p.rowbias_ld = ld; }
  void set_out_col_stride(long long ocs) { p.ocs = ocs; }
  void set_residual(const void* res, long long ldr, long long batch_stride, bool fp32);
  void set_stats(long long* stats) { p.stats = stats; }
  // GroupNorm-backward epilogue (training data gradients, bf16): the GEMM result is dL/da of a GroupNorm(+SiLU)(+dropout)
  // whose INPUT is the channel concatenation of x0 (c0 channels, row pitch ld0) and x1; `consts` = [B][N] float4 from
  // launch_gn_consts; `part` = [gnb_rows()][N][2] per-tile partials for launch_gnb_tile_reduce. Dropout of the layer is
  // supplied per launch through rt_drop_*.
  void set_gn_backward(const void* x0, long long ld0, int c0, const void* x1, long long ld1, const void* consts, int silu, float* part);
  long long gnb_rows() const { return 1LL * p.tx * p.ty * p.tz * p.tb * p.bb; }
  int gnb_tiles_per_batch_tile() const { return p.tx * p.ty * p.tz; }
  int gnb_bb() const { return p.bb; }
  bool gnb = false;
  int rt_drop_thresh = 0; float rt_drop_scale = 1.f; unsigned long long rt_seed = 0;
  void set_alpha(float a) { p.alpha = a; }
  // Split-K over `S` CTAs per tile; `scratch` holds S fp32 copies of the output ([B][V][N] each). Call before finalize.
  void enable_splits(int S, float* scratch);

  // Packs weights (device gather kernel), uploads the table, encodes the B map. Call after all add_* calls.
  void finalize(cudaStream_t stream, bool pack = true);
  // Re-pack weights only (after a weight reload into the same source buffers).
  void repack(cudaStream_t stream);
  // B <= the batch the op was built for; out_override replaces the output pointer (user buffers).
  void launch(cudaStream_t stream, int B = -1, void* out_override = nullptr) const;

 private:
  Geometry geo{};
  bool b_from_act = false;
  int stage_need = 0;  // bytes of the largest pipeline group (decides the stage size / count at launch)
  long long b_lo_off = 0;  // X3 activation-B: K coordinate of the lo parts
  void encode_bmap(void* ptr, int K, int N, int batch, long long row_stride_bytes, long long batch_stride_bytes);
};

int sm_count();
// SMs the split-K plans and grid caps are sized for (the H100 SXM's 132). A constant (not the device query) so that the
// GPU-less sizing pass and the real pass agree on every scratch size.
constexpr int kPlanSMs = 132;
void encode_map(CUtensorMap* m, Precision prec, int rank, void* base, const uint64_t* dims,
                const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box);
// Split-K factor for a conv-like op (pure function of the shapes, so the dry planning pass and the real pass agree).
int plan_splits(int X, int Y, int Z, int B, int N, int cin_total, int taps, Precision prec);

}  // namespace mdb
