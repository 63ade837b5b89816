// Batched marching tetrahedra with the reference's exact output ordering (nvdiffrec/lib/geometry/dmtet.py:105-163).
//
// The reference builds, per call, the lexicographically sorted unique edge list of the *valid* tets with
// torch.unique and numbers the crossing edges by their rank in that list. The set of crossing edges of valid tets
// equals the set of crossing edges of the whole grid (a tet owning a crossing edge has mixed occupancy, hence is
// valid), and ranks inside a sorted subsequence are preserved, so the same numbering is obtained from a STATIC
// sorted edge table of the tet grid built once in mdb_marching_tets_prepare:
//     vertex id of edge e  =  exclusive prefix sum of crossing flags over the globally sorted edge table.
// Faces follow the reference's order: all 1-triangle tets in tet order, then all 2-triangle tets in tet order.
// Per call the work is 7 kernels for the whole batch (blockIdx.y = sample): flags + tile sums of the edge and tet segments in
// one grid, tile sums of the valid-vertex flags, one scan of all tile sums; then -- once the host has sized the outputs from
// the counts -- three emitters that finish the exclusive scan of their segment inside each 2048-element tile and write
// vertices / faces / valid vertices straight from it (no flag or scan array is kept except the 1-byte flags and the
// edge -> vertex-id map the face emitter gathers from). ~7 MB / sample at R=64 (tets 2.5 MB + tet->edge table 3.8 MB +
// sdf/pos 0.5 MB); the exact-size outputs of the reference API force one host read of the counts per batch.
#include "../../include/meshdiff_b200.h"
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>

namespace mdbmt {

#define MT_CHECK(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) throw std::runtime_error(std::string("mdb MT: ") + cudaGetErrorString(_e) + " (" #expr ")"); \
  } while (0)

// dmtet.py:34-53
__constant__ int8_t c_tri_table[16][6] = {
    {-1, -1, -1, -1, -1, -1}, {1, 0, 2, -1, -1, -1}, {4, 0, 3, -1, -1, -1}, {1, 4, 2, 1, 3, 4},
    {3, 1, 5, -1, -1, -1},    {2, 3, 0, 2, 5, 3},    {1, 4, 0, 1, 5, 4},    {4, 2, 5, -1, -1, -1},
    {4, 5, 2, -1, -1, -1},    {4, 1, 0, 4, 5, 1},    {3, 2, 0, 3, 5, 2},    {1, 3, 5, -1, -1, -1},
    {4, 1, 2, 4, 3, 1},       {3, 0, 4, -1, -1, -1}, {2, 0, 1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1}};
__constant__ int8_t c_num_tri[16] = {0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0};

struct Handle {
  int F = 0, Nv = 0, E = 0, max_batch = 0;
  int tE = 0, tF = 0, tV = 0;  // scan tiles per segment (edges, tets, vertices)
  int* d_tets = nullptr;      // [F][4]
  int2* d_edges = nullptr;    // [E] sorted (a<b), lexicographic
  int* d_tet_edges = nullptr; // [F][6] edge ids in base_tet_edges order
  int* d_vadj_off = nullptr;  // [Nv + 1] CSR of the edges incident to every grid vertex (backward pass)
  int* d_vadj = nullptr;      // [2 E]   2 * edge id + (0: the vertex is the edge's first endpoint, 1: its second)
  // per-call workspace (sized for max_batch)
  uint8_t* d_eflag = nullptr;    // [B][E]  edge crosses the surface
  uint32_t* d_escan = nullptr;   // [B][E]  vertex id of a crossing edge (exclusive prefix sum of eflag)
  uint8_t* d_tetidx = nullptr;   // [B][F]  occupancy code of the tet (-> 0 / 1 / 2 triangles)
  uint8_t* d_vflag = nullptr;    // [B][Nv] vertex belongs to a tet with >= 1 triangle
  uint32_t* d_partials = nullptr;  // [B][tE + 2 tF + tV] tile sums -> exclusive tile offsets, segments (E | n1 | n2 | V)
  int* d_counts = nullptr;       // [B][4]: nverts, n1, n2, nvalidverts
  long long* d_offs = nullptr;   // [3][B]: packed output offsets of every sample (verts, faces, valid verts)
  int* h_counts = nullptr;       // pinned
  int last_batch = 0;
};

constexpr int SCAN_TILE = 2048;   // elements per block (256 threads x 8)

// exclusive prefix of `v` over the 256 threads of a block (+ the block total in *total); sh: 9 words
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* sh, uint32_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) sh[w] = inc;
  __syncthreads();
  if (threadIdx.x < 8) {
    uint32_t x = sh[threadIdx.x], xi = x;
    for (int o = 1; o < 8; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffu, xi, o); if ((int)threadIdx.x >= o) xi += t; }
    sh[threadIdx.x] = xi - x;          // exclusive warp offsets
    if (threadIdx.x == 7) sh[8] = xi;  // block total
  }
  __syncthreads();
  const uint32_t ex = sh[w] + inc - v;
  if (total) *total = sh[8];
  __syncthreads();
  return ex;
}
__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t* sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t t = 0;
  if (threadIdx.x == 0) for (int w = 0; w < 8; ++w) t += sh[w];
  __syncthreads();
  return t;  // valid in thread 0
}

// ---------------------------------------------------------------- pass 1: flags + tile sums, one launch
// blockIdx.x < tE: a tile of the sorted edge table (crossing flags); else a tile of tets (occupancy code, 1- / 2-triangle
// counts, scatter of the valid-vertex flags). blockIdx.y = sample. occ = sdf > 0 (dmtet.py:107).
__global__ void __launch_bounds__(256) mt_flags_kernel(const int2* __restrict__ edges, const int* __restrict__ tets,
                                                      const float* __restrict__ sdf, uint8_t* __restrict__ eflag,
                                                      uint8_t* __restrict__ tetidx, uint8_t* __restrict__ vflag,
                                                      uint32_t* __restrict__ partials, int E, int F, int Nv, int tE, int tF, int tV) {
  __shared__ uint32_t sh[9];
  const int b = blockIdx.y;
  const float* s = sdf + (size_t)b * Nv;
  uint32_t* part = partials + (size_t)b * (tE + 2 * tF + tV);
  if ((int)blockIdx.x < tE) {
    const int base = blockIdx.x * SCAN_TILE;
    uint32_t n = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = base + i * 256 + threadIdx.x;
      if (e < E) {
        const int2 ab = __ldg(edges + e);
        const uint32_t f = ((s[ab.x] > 0.f) != (s[ab.y] > 0.f)) ? 1u : 0u;
        eflag[(size_t)b * E + e] = (uint8_t)f;
        n += f;
      }
    }
    const uint32_t t = block_sum(n, sh);
    if (threadIdx.x == 0) part[blockIdx.x] = t;
  } else {
    const int tile = blockIdx.x - tE;
    const int base = tile * SCAN_TILE;
    uint8_t* vf = vflag + (size_t)b * Nv;
    uint32_t n = 0;  // low 16 bits: 1-triangle tets, high 16 bits: 2-triangle tets
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = base + i * 256 + threadIdx.x;
      if (t < F) {
        const int4 v = __ldg(reinterpret_cast<const int4*>(tets) + t);
        const int idx = (s[v.x] > 0.f ? 1 : 0) | (s[v.y] > 0.f ? 2 : 0) | (s[v.z] > 0.f ? 4 : 0) | (s[v.w] > 0.f ? 8 : 0);
        const int nt = c_num_tri[idx];
        tetidx[(size_t)b * F + t] = (uint8_t)idx;
        n += (nt == 1 ? 1u : 0u) + (nt == 2 ? 0x10000u : 0u);
        if (nt > 0) { vf[v.x] = 1; vf[v.y] = 1; vf[v.z] = 1; vf[v.w] = 1; }  // valid_vert_idx (dmtet.py:161)
      }
    }
    const uint32_t t = block_sum(n, sh);
    if (threadIdx.x == 0) { part[tE + tile] = t & 0xffffu; part[tE + tF + tile] = t >> 16; }
  }
}

__global__ void __launch_bounds__(256) mt_vflag_sums_kernel(const uint8_t* __restrict__ vflag, uint32_t* __restrict__ partials,
                                                           int Nv, int tE, int tF, int tV) {
  __shared__ uint32_t sh[9];
  const int b = blockIdx.y;
  const int base = blockIdx.x * SCAN_TILE;
  uint32_t n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const int v = base + i * 256 + threadIdx.x; if (v < Nv) n += vflag[(size_t)b * Nv + v]; }
  const uint32_t t = block_sum(n, sh);
  if (threadIdx.x == 0) partials[(size_t)b * (tE + 2 * tF + tV) + tE + 2 * tF + blockIdx.x] = t;
}

// ---------------------------------------------------------------- pass 2: exclusive scan of the tile sums, 4 segments per sample
__global__ void __launch_bounds__(1024) mt_scan_partials_kernel(uint32_t* partials, int tE, int tF, int tV, int* counts) {
  __shared__ uint32_t sh[1024];
  __shared__ uint32_t carry;
  const int seg = blockIdx.x, b = blockIdx.y;
  const int tiles = seg == 0 ? tE : (seg == 3 ? tV : tF);
  const int base0 = seg == 0 ? 0 : (seg == 1 ? tE : (seg == 2 ? tE + tF : tE + 2 * tF));
  uint32_t* p = partials + (size_t)b * (tE + 2 * tF + tV) + base0;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < tiles; base += 1024) {
    const int k = base + threadIdx.x;
    const uint32_t v = k < tiles ? p[k] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const uint32_t t = (int)threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    const uint32_t incl = sh[threadIdx.x];
    if (k < tiles) p[k] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[b * 4 + seg] = (int)carry;
}

// packed output offsets of the batch: exclusive sums over the samples of (nverts, n1 + 2 n2, nvalidverts)
__global__ void mt_offsets_kernel(const int* __restrict__ counts, long long* __restrict__ offs, int B, int stride) {
  if (threadIdx.x < 3) {
    long long run = 0;
    for (int b = 0; b < B; ++b) {
      offs[(size_t)threadIdx.x * stride + b] = run;
      run += threadIdx.x == 0 ? counts[b * 4] : (threadIdx.x == 1 ? counts[b * 4 + 1] + 2 * counts[b * 4 + 2] : counts[b * 4 + 3]);
    }
  }
}

// ---------------------------------------------------------------- pass 3: in-tile scans fused with the emitters
// verts[vid] = (p_a * (-s_b) + p_b * s_a) / (s_a - s_b) in the reference's operation order (dmtet.py:125-132);
// vid = rank of the edge among the crossing edges of the sorted table. Also leaves escan for the face emitter.
__global__ void __launch_bounds__(256) mt_emit_verts_kernel(const int2* __restrict__ edges, const uint8_t* __restrict__ eflag,
                                                           const uint32_t* __restrict__ partials, uint32_t* __restrict__ escan,
                                                           const float* __restrict__ pos, long long pos_bstride,
                                                           const float* __restrict__ sdf, float* __restrict__ verts,
                                                           const long long* __restrict__ vert_off, int E, int Nv, int ptiles) {
  __shared__ uint32_t sh[9];
  const int b = blockIdx.y;
  const float* s = sdf + (size_t)b * Nv;
  const float* p = pos + (size_t)b * pos_bstride;
  float* out = verts + vert_off[b] * 3;
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * 8;
  uint8_t f[8];
  uint32_t n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { f[i] = (base + i < E) ? eflag[(size_t)b * E + base + i] : 0; n += f[i]; }
  uint32_t run = partials[(size_t)b * ptiles + blockIdx.x] + block_excl_scan(n, sh, nullptr);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int e = base + i;
    if (e >= E) break;
    escan[(size_t)b * E + e] = run;
    if (f[i]) {
      const int2 ab = __ldg(edges + e);
      const float sa = s[ab.x], sb = -s[ab.y];
      const float den = __fadd_rn(sa, sb);
      const float wa = __fdiv_rn(sb, den), wb = __fdiv_rn(sa, den);  // flip: weight of a is (-s_b)/den
#pragma unroll
      for (int k = 0; k < 3; ++k)
        out[(size_t)run * 3 + k] = __fadd_rn(__fmul_rn(p[(size_t)ab.x * 3 + k], wa), __fmul_rn(p[(size_t)ab.y * 3 + k], wb));
      ++run;
    }
  }
}

// faces: all 1-triangle tets in tet order, then all 2-triangle tets in tet order (dmtet.py:136-144); uv_idx / face_to_tet
// as map_uv (dmtet.py:70-99, 156-159)
__global__ void __launch_bounds__(256) mt_emit_faces_kernel(const int* __restrict__ tet_edges, const uint8_t* __restrict__ tetidx,
                                                           const uint32_t* __restrict__ partials, const uint32_t* __restrict__ escan,
                                                           const int* __restrict__ counts, long long* __restrict__ faces,
                                                           long long* __restrict__ uv_idx, long long* __restrict__ f2t,
                                                           const long long* __restrict__ face_off, int F, int E, int tE, int tF,
                                                           int ptiles) {
  __shared__ uint32_t sh[9];
  const int b = blockIdx.y;
  const int n1 = counts[b * 4 + 1];
  long long* fo = faces + face_off[b] * 3;
  long long* uo = uv_idx + face_off[b] * 3;
  long long* to = f2t + face_off[b];
  const uint32_t* es = escan + (size_t)b * E;
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * 8;
  uint8_t code[8];
  uint32_t n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    code[i] = (base + i < F) ? tetidx[(size_t)b * F + base + i] : 0;
    const int nt = c_num_tri[code[i]];
    n += (nt == 1 ? 1u : 0u) + (nt == 2 ? 0x10000u : 0u);
  }
  const uint32_t ex = block_excl_scan(n, sh, nullptr);
  uint32_t r1 = partials[(size_t)b * ptiles + tE + blockIdx.x] + (ex & 0xffffu);
  uint32_t r2 = partials[(size_t)b * ptiles + tE + tF + blockIdx.x] + (ex >> 16);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int t = base + i;
    const int idx = code[i];
    const int nt = c_num_tri[idx];
    if (nt == 0) continue;
    const long long f0 = nt == 1 ? (long long)r1 : (long long)n1 + 2LL * r2;
    if (nt == 1) ++r1; else ++r2;
    int eid[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) eid[k] = __ldg(tet_edges + (size_t)t * 6 + k);
    for (int j = 0; j < nt; ++j) {
      const long long f = f0 + j;
#pragma unroll
      for (int k = 0; k < 3; ++k) fo[f * 3 + k] = (long long)es[eid[c_tri_table[idx][j * 3 + k]]];
      // map_uv (dmtet.py:70-99): face_gidx = 2*t + j -> tet cell t, triangle j
      uo[f * 3 + 0] = 4LL * t;
      uo[f * 3 + 1] = 4LL * t + j + 1;
      uo[f * 3 + 2] = 4LL * t + j + 2;
      to[f] = t;
    }
  }
}

__global__ void __launch_bounds__(256) mt_emit_valid_verts_kernel(const uint8_t* __restrict__ vflag, const uint32_t* __restrict__ partials,
                                                                 long long* __restrict__ out, const long long* __restrict__ vv_off,
                                                                 int Nv, int tE, int tF, int ptiles) {
  __shared__ uint32_t sh[9];
  const int b = blockIdx.y;
  long long* o = out + vv_off[b];
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * 8;
  uint8_t f[8];
  uint32_t n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { f[i] = (base + i < Nv) ? vflag[(size_t)b * Nv + base + i] : 0; n += f[i]; }
  uint32_t run = partials[(size_t)b * ptiles + tE + 2 * tF + blockIdx.x] + block_excl_scan(n, sh, nullptr);
#pragma unroll
  for (int i = 0; i < 8; ++i) if (f[i]) o[run++] = base + i;
}

// ---------------------------------------------------------------- backward of the vertex interpolation
// What torch autograd computes for dmtet.py:125-132: with s_a = sdf[a], t = -sdf[b], den = s_a + t, the surface vertex of a
// crossing edge (a, b) is v = p_a * (t / den) + p_b * (s_a / den). For g = dL/dv:
//     dL/dp_a = g * t / den          dL/dp_b = g * s_a / den
//     dL/dsdf[a] = g.(p_b - p_a) * t / den^2       dL/dsdf[b] = g.(p_b - p_a) * s_a / den^2   (= own weight / den)
// One thread per grid vertex GATHERS over its incident edges (static CSR), in table order: no atomics, the sums are
// bitwise reproducible. vid = the crossing edge's output row (the exclusive scan the forward pass left / the caller kept).
__global__ void __launch_bounds__(256) mt_grad_kernel(const int2* __restrict__ edges, const int* __restrict__ vadj_off,
                                                     const int* __restrict__ vadj, const uint32_t* __restrict__ vid,
                                                     const float* __restrict__ pos, long long pos_bstride,
                                                     const float* __restrict__ sdf, const float* __restrict__ gverts,
                                                     const long long* __restrict__ vert_off, float* __restrict__ gpos,
                                                     float* __restrict__ gsdf, int E, int Nv) {
  const int b = blockIdx.y;
  const int v = blockIdx.x * 256 + threadIdx.x;
  if (v >= Nv) return;
  const float* s = sdf + (size_t)b * Nv;
  const float* p = pos + (size_t)b * pos_bstride;
  const float* g = gverts + vert_off[b] * 3;
  const uint32_t* id = vid + (size_t)b * E;
  const float sv = s[v];
  const bool occ = sv > 0.f;
  float gx = 0.f, gy = 0.f, gz = 0.f, gs = 0.f;
  const int k1 = __ldg(vadj_off + v + 1);
  for (int k = __ldg(vadj_off + v); k < k1; ++k) {
    const int code = __ldg(vadj + k);
    const int e = code >> 1;
    const int2 ab = __ldg(edges + e);
    const int other = (code & 1) ? ab.x : ab.y;
    const float so = s[other];
    if ((so > 0.f) == occ) continue;  // not a crossing edge
    const float sa = (code & 1) ? so : sv, t = (code & 1) ? -sv : -so;
    const float den = sa + t;
    const float w = ((code & 1) ? sa : t) / den;  // interpolation weight of THIS endpoint; d v / d sdf[this] = (p_b - p_a) * w / den
    const float* gr = g + (size_t)id[e] * 3;
    const float g0 = gr[0], g1 = gr[1], g2 = gr[2];
    gx = fmaf(g0, w, gx); gy = fmaf(g1, w, gy); gz = fmaf(g2, w, gz);
    const float* pa = p + (size_t)ab.x * 3;
    const float* pb = p + (size_t)ab.y * 3;
    const float dot = g0 * (pb[0] - pa[0]) + g1 * (pb[1] - pa[1]) + g2 * (pb[2] - pa[2]);
    gs = fmaf(dot, w / den, gs);
  }
  if (gpos) {
    float* o = gpos + ((size_t)b * Nv + v) * 3;
    o[0] = gx; o[1] = gy; o[2] = gz;
  }
  if (gsdf) gsdf[(size_t)b * Nv + v] = gs;
}

static int grid1d(int n) { int g = (n + 255) / 256; return g > 132 * 4 ? 132 * 4 : (g < 1 ? 1 : g); }

}  // namespace mdbmt

using namespace mdbmt;

namespace mdb { void set_last_error(const std::string& msg); }  // api.cu

#define MT_API_BEGIN try {
#define MT_API_END                                                              \
  }                                                                             \
  catch (const std::exception& e) { mdb::set_last_error(e.what()); return 1; }  \
  return 0;

// map_uv's static atlas (dmtet.py:70-88): N = ceil(sqrt(F)) cells, 4 corners per cell.
__global__ void uvs_kernel(float* __restrict__ uvs, int N) {
  const float start = 0.f, end = 1.f - (1.f / (float)N);
  const float step = (end - start) / (float)(N - 1);
  const float pad = 0.9f / (float)N;
  const long long total = (long long)N * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int yi = (int)(i / N), xi = (int)(i % N);
    // torch.linspace evaluates symmetrically from both ends
    const float tx = xi < N / 2 ? start + step * (float)xi : end - step * (float)(N - 1 - xi);
    const float ty = yi < N / 2 ? start + step * (float)yi : end - step * (float)(N - 1 - yi);
    float* o = uvs + i * 8;
    o[0] = tx;       o[1] = ty;
    o[2] = tx + pad; o[3] = ty;
    o[4] = tx + pad; o[5] = ty + pad;
    o[6] = tx;       o[7] = ty + pad;
  }
}

extern "C" {

int mdb_marching_tets_prepare(const int* tets_host, int F, int Nv, int max_batch, void** handle) {
  MT_API_BEGIN
  auto* h = new Handle;
  h->F = F; h->Nv = Nv; h->max_batch = max_batch;
  // static sorted unique edge table + tet -> edge ids (base_tet_edges = [0,1, 0,2, 0,3, 1,2, 1,3, 2,3], dmtet.py:54)
  static const int be[12] = {0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3};
  std::vector<uint64_t> keys((size_t)F * 6);
  for (int t = 0; t < F; ++t)
    for (int k = 0; k < 6; ++k) {
      uint32_t a = (uint32_t)tets_host[t * 4 + be[2 * k]], b = (uint32_t)tets_host[t * 4 + be[2 * k + 1]];
      if (a > b) std::swap(a, b);
      keys[(size_t)t * 6 + k] = ((uint64_t)a << 32) | b;
    }
  std::vector<uint64_t> uniq(keys);
  std::sort(uniq.begin(), uniq.end());
  uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
  h->E = (int)uniq.size();
  std::vector<int2> edges(h->E);
  for (int e = 0; e < h->E; ++e) edges[e] = make_int2((int)(uniq[e] >> 32), (int)(uniq[e] & 0xffffffffu));
  std::vector<int> te((size_t)F * 6);
  for (size_t i = 0; i < keys.size(); ++i)
    te[i] = (int)(std::lower_bound(uniq.begin(), uniq.end(), keys[i]) - uniq.begin());
  // vertex -> incident edges (CSR, edges in table order): the gather form of the backward pass
  std::vector<int> adj_off((size_t)Nv + 1, 0), adj((size_t)2 * h->E);
  for (int e = 0; e < h->E; ++e) { adj_off[edges[e].x + 1]++; adj_off[edges[e].y + 1]++; }
  for (int v = 0; v < Nv; ++v) adj_off[v + 1] += adj_off[v];
  {
    std::vector<int> fill(adj_off.begin(), adj_off.end() - 1);
    for (int e = 0; e < h->E; ++e) { adj[fill[edges[e].x]++] = 2 * e; adj[fill[edges[e].y]++] = 2 * e + 1; }
  }
  const size_t B = max_batch;
  MT_CHECK(cudaMalloc(&h->d_vadj_off, ((size_t)Nv + 1) * 4));
  MT_CHECK(cudaMalloc(&h->d_vadj, (size_t)2 * h->E * 4 + 4));
  MT_CHECK(cudaMemcpy(h->d_vadj_off, adj_off.data(), ((size_t)Nv + 1) * 4, cudaMemcpyHostToDevice));
  MT_CHECK(cudaMemcpy(h->d_vadj, adj.data(), (size_t)2 * h->E * 4, cudaMemcpyHostToDevice));
  MT_CHECK(cudaMalloc(&h->d_tets, (size_t)F * 16));
  MT_CHECK(cudaMalloc(&h->d_edges, (size_t)h->E * 8));
  MT_CHECK(cudaMalloc(&h->d_tet_edges, (size_t)F * 24));
  MT_CHECK(cudaMemcpy(h->d_tets, tets_host, (size_t)F * 16, cudaMemcpyHostToDevice));
  MT_CHECK(cudaMemcpy(h->d_edges, edges.data(), (size_t)h->E * 8, cudaMemcpyHostToDevice));
  MT_CHECK(cudaMemcpy(h->d_tet_edges, te.data(), (size_t)F * 24, cudaMemcpyHostToDevice));
  h->tE = (h->E + SCAN_TILE - 1) / SCAN_TILE; h->tF = (F + SCAN_TILE - 1) / SCAN_TILE; h->tV = (Nv + SCAN_TILE - 1) / SCAN_TILE;
  MT_CHECK(cudaMalloc(&h->d_eflag, B * h->E)); MT_CHECK(cudaMalloc(&h->d_escan, B * h->E * 4));
  MT_CHECK(cudaMalloc(&h->d_vflag, B * Nv));
  MT_CHECK(cudaMalloc(&h->d_tetidx, B * F));
  MT_CHECK(cudaMalloc(&h->d_partials, B * (size_t)(h->tE + 2 * h->tF + h->tV) * 4));
  MT_CHECK(cudaMalloc(&h->d_counts, B * 4 * sizeof(int)));
  MT_CHECK(cudaMalloc(&h->d_offs, 3 * B * sizeof(long long)));
  MT_CHECK(cudaMallocHost(&h->h_counts, B * 4 * sizeof(int)));
  *handle = h;
  MT_API_END
}

void mdb_marching_tets_destroy(void* handle) {
  auto* h = static_cast<Handle*>(handle);
  if (!h) return;
  cudaFree(h->d_tets); cudaFree(h->d_edges); cudaFree(h->d_tet_edges); cudaFree(h->d_vadj_off); cudaFree(h->d_vadj);
  cudaFree(h->d_eflag); cudaFree(h->d_escan); cudaFree(h->d_vflag);
  cudaFree(h->d_tetidx); cudaFree(h->d_partials); cudaFree(h->d_counts); cudaFree(h->d_offs); cudaFreeHost(h->h_counts);
  delete h;
}

int mdb_marching_tets_info(void* handle, int* n_edges, int* uv_grid_n) {
  auto* h = static_cast<Handle*>(handle);
  if (n_edges) *n_edges = h->E;
  if (uv_grid_n) *uv_grid_n = (int)std::ceil(std::sqrt((double)((2LL * h->F + 1) / 2)));
  return 0;
}

/* uvs fp32 [N*N*4][2] (N from mdb_marching_tets_info) */
int mdb_marching_tets_uvs(void* handle, float* uvs, void* stream) {
  MT_API_BEGIN
  auto* h = static_cast<Handle*>(handle);
  const int N = (int)std::ceil(std::sqrt((double)((2LL * h->F + 1) / 2)));
  uvs_kernel<<<grid1d(N * N), 256, 0, (cudaStream_t)stream>>>(uvs, N);
  MT_CHECK(cudaGetLastError());
  MT_API_END
}

/* Phase 1: occupancy flags + scans for `batch` samples (sdf [B][Nv]); counts_host[b] = {nverts, nfaces, nvalidverts}.
 * Synchronises the stream (the caller needs the counts to size the outputs). */
int mdb_marching_tets_count(void* handle, const float* sdf, int batch, int* counts_host, void* stream) {
  MT_API_BEGIN
  auto* h = static_cast<Handle*>(handle);
  cudaStream_t s = (cudaStream_t)stream;
  if (batch < 1 || batch > h->max_batch) throw std::runtime_error("mdb MT: batch out of range");
  const int E = h->E, F = h->F, Nv = h->Nv;
  // 4 launches: vertex-flag clear, flags + tile sums (edges and tets in one grid), vertex-flag tile sums (they depend on the
  // tets' scatter), scan of the tile sums of all four segments
  MT_CHECK(cudaMemsetAsync(h->d_vflag, 0, (size_t)batch * Nv, s));
  mt_flags_kernel<<<dim3(h->tE + h->tF, batch), 256, 0, s>>>(h->d_edges, h->d_tets, sdf, h->d_eflag, h->d_tetidx, h->d_vflag,
                                                             h->d_partials, E, F, Nv, h->tE, h->tF, h->tV);
  mt_vflag_sums_kernel<<<dim3(h->tV, batch), 256, 0, s>>>(h->d_vflag, h->d_partials, Nv, h->tE, h->tF, h->tV);
  mt_scan_partials_kernel<<<dim3(4, batch), 1024, 0, s>>>(h->d_partials, h->tE, h->tF, h->tV, h->d_counts);
  mt_offsets_kernel<<<1, 32, 0, s>>>(h->d_counts, h->d_offs, batch, h->max_batch);
  MT_CHECK(cudaGetLastError());
  MT_CHECK(cudaMemcpyAsync(h->h_counts, h->d_counts, (size_t)batch * 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
  MT_CHECK(cudaStreamSynchronize(s));
  for (int b = 0; b < batch; ++b) {
    counts_host[b * 3 + 0] = h->h_counts[b * 4 + 0];
    counts_host[b * 3 + 1] = h->h_counts[b * 4 + 1] + 2 * h->h_counts[b * 4 + 2];
    counts_host[b * 3 + 2] = h->h_counts[b * 4 + 3];
  }
  h->last_batch = batch;
  MT_API_END
}

/* Phase 2: emit. pos [B][Nv][3] (pos_batch_stride = 0 shares one vertex array), sdf as in phase 1.
 * Outputs are packed per sample at the element offsets given (device arrays of `batch` int64):
 *   verts fp32 [sum nverts][3], faces / uv_idx int64 [sum nfaces][3], face_to_tet int64 [sum nfaces],
 *   valid_vert_idx int64 [sum nvalidverts]. */
int mdb_marching_tets_extract(void* handle, const float* pos, long long pos_batch_stride, const float* sdf, int batch,
                              float* verts, long long* faces, long long* uv_idx, long long* face_to_tet,
                              long long* valid_vert_idx, const long long* vert_off, const long long* face_off,
                              const long long* vv_off, void* stream) {
  MT_API_BEGIN
  auto* h = static_cast<Handle*>(handle);
  cudaStream_t s = (cudaStream_t)stream;
  if (batch != h->last_batch) throw std::runtime_error("mdb MT: call mdb_marching_tets_count first with the same batch");
  const int E = h->E, F = h->F, Nv = h->Nv;
  // NULL offsets: outputs packed back to back in sample order -- the offsets the count pass left on the device
  if (!vert_off) vert_off = h->d_offs;
  if (!face_off) face_off = h->d_offs + h->max_batch;
  if (!vv_off) vv_off = h->d_offs + 2 * (size_t)h->max_batch;
  // 3 launches: each finishes the exclusive scan of its segment inside the tile and emits straight from it
  const int pt = h->tE + 2 * h->tF + h->tV;
  mt_emit_verts_kernel<<<dim3(h->tE, batch), 256, 0, s>>>(h->d_edges, h->d_eflag, h->d_partials, h->d_escan, pos, pos_batch_stride,
                                                          sdf, verts, vert_off, E, Nv, pt);
  mt_emit_faces_kernel<<<dim3(h->tF, batch), 256, 0, s>>>(h->d_tet_edges, h->d_tetidx, h->d_partials, h->d_escan, h->d_counts, faces,
                                                          uv_idx, face_to_tet, face_off, F, E, h->tE, h->tF, pt);
  mt_emit_valid_verts_kernel<<<dim3(h->tV, batch), 256, 0, s>>>(h->d_vflag, h->d_partials, valid_vert_idx, vv_off, Nv, h->tE, h->tF, pt);
  MT_CHECK(cudaGetLastError());
  MT_API_END
}

/* Copies the crossing-edge -> output-row map of the last mdb_marching_tets_extract ([batch][n_edges] uint32) so that a
 * backward pass can run after the handle has been used for another batch. */
int mdb_marching_tets_vertex_ids(void* handle, int batch, unsigned* out, void* stream) {
  MT_API_BEGIN
  auto* h = static_cast<Handle*>(handle);
  if (batch != h->last_batch) throw std::runtime_error("mdb MT: vertex ids are those of the last extract; batch differs");
  MT_CHECK(cudaMemcpyAsync(out, h->d_escan, (size_t)batch * h->E * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  MT_API_END
}

/* Backward of the vertex interpolation (what autograd does for dmtet.py:125-132). */
int mdb_marching_tets_backward(void* handle, const float* pos, long long pos_batch_stride, const float* sdf, int batch,
                               const unsigned* vertex_ids, const float* grad_verts, const long long* vert_off,
                               float* grad_pos, float* grad_sdf, void* stream) {
  MT_API_BEGIN
  auto* h = static_cast<Handle*>(handle);
  if (batch < 1 || batch > h->max_batch) throw std::runtime_error("mdb MT: batch out of range");
  if (!vertex_ids || !vert_off) {
    if (batch != h->last_batch) throw std::runtime_error("mdb MT: backward without saved vertex ids needs the batch of the last extract");
    if (!vertex_ids) vertex_ids = h->d_escan;
    if (!vert_off) vert_off = h->d_offs;
  }
  mt_grad_kernel<<<dim3((h->Nv + 255) / 256, batch), 256, 0, (cudaStream_t)stream>>>(
      h->d_edges, h->d_vadj_off, h->d_vadj, vertex_ids, pos, pos_batch_stride, sdf, grad_verts, vert_off, grad_pos, grad_sdf,
      h->E, h->Nv);
  MT_CHECK(cudaGetLastError());
  MT_API_END
}

}  // extern "C"
