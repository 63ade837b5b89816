// Host-side builders for the wgmma weight-gradient kernel (see wgrad_tc.cuh) and its split-K reduction.
#define MDB_WGRAD_KERNEL_IMPL
#include "wgrad_host.h"
#include <cstdlib>

namespace mdb {

// X3 stages carry hi and lo parts of half the voxels: the forward tile with its slowest axis of extent > 1 halved
static Geometry half_geometry(Geometry g) {
  if (g.bb > 1) g.bb /= 2;
  else if (g.bz > 1) g.bz /= 2;
  else if (g.by > 1) g.by /= 2;
  else g.bx /= 2;
  return g;
}

WgradPlan plan_wgrad(int X, int Y, int Z, int B, int M, int N, int ksize, int stride, Precision prec) {
  WgradPlan pl;
  if (ksize != 1 && ksize != 3) throw std::runtime_error("mdb: wgrad supports 1x1x1 and 3x3x3 kernels");
  pl.flat = ksize == 1;
  const int vox = 128 / parts(prec);
  long long tiles;
  if (pl.flat) {
    pl.geo = {vox, 1, 1, 1};
    pl.n_groups = 1; pl.taps = 1;
    tiles = ((long long)B * X * Y * Z + vox - 1) / vox;
  } else {
    pl.geo = pick_geometry(X, Y, Z);
    if (prec == kBF16X3) pl.geo = half_geometry(pl.geo);
    if (pl.geo.bx * pl.geo.by * pl.geo.bz * pl.geo.bb != vox) throw std::runtime_error("mdb: unsupported wgrad tile geometry");
    pl.n_groups = 27;
    pl.taps = 27;
    tiles = 1LL * ((X + pl.geo.bx - 1) / pl.geo.bx) * ((Y + pl.geo.by - 1) / pl.geo.by) * ((Z + pl.geo.bz - 1) / pl.geo.bz) *
            ((B + pl.geo.bb - 1) / pl.geo.bb);
  }
  pl.m_tiles = (M + 127) / 128;
  pl.n_tiles = (N + 127) / 128;
  const long long items = 1LL * pl.m_tiles * pl.n_tiles * pl.n_groups;
  long long S = kPlanSMs / items;
  if (S < 1) S = 1;
  if (S > tiles) S = tiles;
  pl.max_splits = (int)S;
  pl.scratch_bytes = (size_t)S * pl.taps * pl.m_tiles * 128 * pl.n_tiles * 128 * sizeof(float);
  return pl;
}

void WgradOp::init(const Act& dy, const Act& x, int ksize, int stride, const WgradOut& out, float* scratch, Precision prec) {
  if (prec == kTF32) throw std::runtime_error("mdb: weight gradients are built for bf16 or split-bf16 operands");
  dy_ = dy; x_ = x; ksize_ = ksize; stride_ = stride; out_ = out;
  prec_ = prec;
  M_ = dy.C; N_ = x.C;
  plan_ = plan_wgrad(dy.X, dy.Y, dy.Z, dy.B, M_, N_, ksize, stride, prec);
  if (ksize == 3 && stride == 1 && (x.X != dy.X || x.Y != dy.Y || x.Z != dy.Z)) throw std::runtime_error("mdb: wgrad extent mismatch");
  if (ksize == 3 && stride == 2 && (x.X != 2 * dy.X || x.Y != 2 * dy.Y || x.Z != 2 * dy.Z)) throw std::runtime_error("mdb: stride-2 wgrad extent mismatch");
  if (ksize == 1 && x.voxels() != dy.voxels()) throw std::runtime_error("mdb: pointwise wgrad extent mismatch");
  WgradParams& p = base_;
  p.bx = plan_.geo.bx; p.by = plan_.geo.by; p.bz = plan_.geo.bz; p.bb = plan_.geo.bb;
  p.m_tiles = plan_.m_tiles; p.n_tiles = plan_.n_tiles;
  p.taps = plan_.taps;
  p.Mp = plan_.m_tiles * 128; p.Np = plan_.n_tiles * 128;
  p.partial = scratch;
  p.n_groups = plan_.n_groups;
  int g = 0;
  if (plan_.flat) {
    p.groups[g++] = WgradGroup{0, 0, 0, 0, 0, {0, 0, 0}};
  } else {
    for (int kz = 0; kz < 3; ++kz)
      for (int ky = 0; ky < 3; ++ky)
        for (int kx = 0; kx < 3; ++kx) {
          const int8_t tap = (int8_t)((kz * 3 + ky) * 3 + kx);
          if (stride == 1) p.groups[g++] = WgradGroup{0, (int8_t)(kx - 1), (int8_t)(ky - 1), (int8_t)(kz - 1), tap, {0, 0, 0}};
          else p.groups[g++] = WgradGroup{(int8_t)((kx & 1) | ((ky & 1) << 1) | ((kz & 1) << 2)), (int8_t)(kx >> 1), (int8_t)(ky >> 1), (int8_t)(kz >> 1), tap, {0, 0, 0}};
        }
  }
  flops = 2.0 * dy.voxels() * dy.B * (double)M_ * N_ * plan_.taps;
}

const WgradParams& WgradOp::params_for(int B) {
  auto it = cache_.find(B);
  if (it != cache_.end()) return it->second;
  WgradParams p = base_;
  Act dy = dy_, x = x_;
  if (plan_.flat) {
    // one row axis over the voxels of every sample (pointwise: stride 1)
    const long long rows = (long long)B * dy_.voxels();
    p.tx = (int)((rows + p.bx - 1) / p.bx); p.ty = p.tz = p.tb = 1;
    dy.X = x.X = (int)rows;
    dy.Y = dy.Z = dy.B = x.Y = x.Z = x.B = 1;
  } else {
    p.tx = (dy_.X + p.bx - 1) / p.bx; p.ty = (dy_.Y + p.by - 1) / p.by; p.tz = (dy_.Z + p.bz - 1) / p.bz;
    p.tb = (B + p.bb - 1) / p.bb;
    dy.B = x.B = B;
  }
  auto enc = [&](CUtensorMap* m, const Act& a, int part, int sub = 1, int par = 0) {
    encode_map(m, prec_, act_map(a, prec_, part, plan_.geo, sub, par & 1, (par >> 1) & 1, (par >> 2) & 1));
  };
  for (int part = 0; part < parts(prec_); ++part) {
    enc(part ? &p.ymap_lo : &p.ymap, dy, part);
    CUtensorMap* xm = part ? p.xmap_lo : p.xmap;
    if (stride_ == 1) {
      enc(&xm[0], x, part);
    } else {
      for (int par = 0; par < 8; ++par) enc(&xm[par], x, part, 2, par);
    }
  }
  const long long tiles = 1LL * p.tx * p.ty * p.tz * p.tb;
  const long long items = 1LL * p.m_tiles * p.n_tiles * p.n_groups;
  long long S = kPlanSMs / items;
  if (S < 1) S = 1;
  if (S > tiles) S = tiles;
  if (S > plan_.max_splits) S = plan_.max_splits;
  p.splits = (int)S;
  return cache_.emplace(B, p).first->second;
}

// ------------------------------------------------------------------ split reduction + scatter to the parameter layout
// One thread per (tap, m, n): the split partials of that element are summed in split order (deterministic) and the
// result goes to its slot of the parameter layout. (A thread per (m, n) looping over the taps left 16 K threads with
// 432 dependent loads each: 38 us per launch, 5.6 ms per backward pass.)
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(WgradReduceArgs a) {
  const long long per_tap = (long long)a.M * a.N;
  const long long total = per_tap * a.taps;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / per_tap);
    const long long r = i - (long long)t * per_tap;
    const int m = (int)(r / a.N), n = (int)(r % a.N);
    float acc = 0.f;
    for (int s = 0; s < a.splits; ++s) acc += __ldg(a.partial + (((long long)s * a.taps + t) * a.Mp + m) * a.Np + n);
    const long long noff = a.ndiv ? (long long)(n % a.ndiv) * a.sn + (long long)(n / a.ndiv) * a.sn_hi : (long long)n * a.sn;
    float* o = a.out + m * a.sm + noff + t * a.st;
    *o = a.accumulate ? *o + acc : acc;
  }
}

void launch_wgrad_reduce(const WgradReduceArgs& a, cudaStream_t s) {
  const long long total = (long long)a.M * a.N * a.taps;
  long long blocks = (total + 255) / 256;
  if (blocks > kPlanSMs * 16) blocks = kPlanSMs * 16;
  wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, s>>>(a);
  MDB_CUDA_CHECK(cudaGetLastError());
}

void WgradOp::launch(cudaStream_t s, int B, bool accumulate, float* out_ptr) {
  if (B < 1 || B > dy_.B) throw std::runtime_error("mdb: wgrad batch out of range");
  const WgradParams& p = params_for(B);
  static bool configured_dev[64] = {};  // the attribute is per device
  int dev = 0;
  MDB_CUDA_CHECK(cudaGetDevice(&dev));
  bool& configured = configured_dev[dev < 64 ? dev : 63];
  if (!configured || dev >= 63) {
    MDB_CUDA_CHECK(cudaFuncSetAttribute(wgrad_tc_kernel<kBF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmemBytes));
    MDB_CUDA_CHECK(cudaFuncSetAttribute(wgrad_tc_kernel<kBF16X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmemBytes));
    configured = true;
  }
  const int grid = p.m_tiles * p.n_tiles * p.n_groups * p.splits;
  if (prec_ == kBF16X3) wgrad_tc_kernel<kBF16X3><<<grid, kWgThreads, kWgSmemBytes, s>>>(p);
  else wgrad_tc_kernel<kBF16><<<grid, kWgThreads, kWgSmemBytes, s>>>(p);
  MDB_CUDA_CHECK(cudaGetLastError());
  WgradReduceArgs r{};
  r.partial = p.partial; r.splits = p.splits; r.taps = p.taps; r.Mp = p.Mp; r.Np = p.Np; r.M = out_.m_valid ? out_.m_valid : M_; r.N = out_.n_valid ? out_.n_valid : N_;
  r.out = out_ptr ? out_ptr : out_.ptr; r.sm = out_.sm; r.sn = out_.sn; r.st = out_.st; r.ndiv = out_.ndiv; r.sn_hi = out_.sn_hi;
  r.accumulate = accumulate ? 1 : 0;
  launch_wgrad_reduce(r, s);
}

}  // namespace mdb
