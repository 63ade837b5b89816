// extern "C" boundary (include/meshdiff_b200.h). Exceptions never cross it: they become error codes + a message.
#include "../../include/meshdiff_b200.h"
#include "unet.h"
#include <cstring>
#include <cmath>

using namespace mdb;

static thread_local std::string g_err;
namespace mdb { void set_last_error(const std::string& msg) { g_err = msg; } }

#define MDB_API_BEGIN try {
#define MDB_API_END                         \
  }                                         \
  catch (const std::exception& e) {         \
    g_err = e.what();                       \
    return 1;                               \
  }                                         \
  catch (...) {                             \
    g_err = "mdb: unknown error";           \
    return 2;                               \
  }                                         \
  return 0;

struct mdb_unet { UNet* net; };

namespace mdb {
void launch_distill_step(const float* eps, const float* z_s, float* z_mid, float* out, const float* mask,
                         const int* step_idx, const mdb_distill_row* rows, int n_rows, int phase, float* labels,
                         long long V, int C, int B, cudaStream_t s);
}  // csrc/distill.cu

extern "C" {

const char* mdb_last_error(void) { return g_err.c_str(); }
int mdb_version(void) { return 100; }

static int create_impl(const mdb_unet_config* c, mdb_unet** out, bool dry) {
  MDB_API_BEGIN
  if (!c || !out) throw std::runtime_error("mdb: null argument");
  UNetConfig u;
  u.image_size = c->image_size; u.nf = c->nf; u.n_levels = c->n_levels;
  for (int i = 0; i < 8; ++i) u.ch_mult[i] = c->ch_mult[i];
  u.num_res_blocks = c->num_res_blocks; u.level0_blocks = c->level0_blocks;
  u.n_attn = c->n_attn;
  for (int i = 0; i < 4; ++i) u.attn_resolutions[i] = c->attn_resolutions[i];
  u.num_channels = c->num_channels; u.stem_ksize = c->stem_ksize; u.use_pos_bias = c->use_pos_bias;
  u.max_batch = c->max_batch; u.precision = c->precision; u.training = c->training; u.num_classes = c->num_classes;
  auto* h = new mdb_unet;
  h->net = nullptr;
  try { h->net = new UNet(u, dry); } catch (...) { delete h; throw; }
  *out = h;
  MDB_API_END
}

int mdb_unet_create(const mdb_unet_config* c, mdb_unet** out) { return create_impl(c, out, false); }
int mdb_unet_create_dry(const mdb_unet_config* c, mdb_unet** out) { return create_impl(c, out, true); }

void mdb_unet_destroy(mdb_unet* n) {
  if (!n) return;
  delete n->net;
  delete n;
}

int mdb_unet_num_params(mdb_unet* n) { return n ? (int)n->net->params().size() : -1; }

int mdb_unet_param_info(mdb_unet* n, int idx, const char** name, long long* numel, int* ndim, long long* shape8) {
  MDB_API_BEGIN
  const auto& ps = n->net->params();
  if (idx < 0 || idx >= (int)ps.size()) throw std::runtime_error("mdb: parameter index out of range");
  if (name) *name = ps[idx].name.c_str();
  if (numel) *numel = ps[idx].numel;
  if (ndim) *ndim = (int)ps[idx].shape.size();
  if (shape8) for (size_t i = 0; i < ps[idx].shape.size() && i < 8; ++i) shape8[i] = ps[idx].shape[i];
  MDB_API_END
}

int mdb_unet_set_param(mdb_unet* n, const char* name, const float* src, long long numel, int dev, void* stream) {
  MDB_API_BEGIN
  n->net->set_param(name, src, numel, dev != 0, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_set_params(mdb_unet* n, int count, const char* const* names, const float* const* srcs, const long long* numels,
                        void* stream) {
  MDB_API_BEGIN
  for (int i = 0; i < count; ++i) n->net->set_param(names[i], srcs[i], numels[i], true, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_get_param(mdb_unet* n, const char* name, float* dst, long long numel, int dev, void* stream) {
  MDB_API_BEGIN
  n->net->get_param(name, dst, numel, dev != 0, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_commit(mdb_unet* n, void* stream) {
  MDB_API_BEGIN
  n->net->commit((cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_forward(mdb_unet* n, const float* x, const float* labels, float* out, int B, void* stream) {
  MDB_API_BEGIN
  n->net->forward(x, labels, out, B, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_info(mdb_unet* n, double* flops, long long* arena, int* ngemm, int* nsteps) {
  MDB_API_BEGIN
  if (flops) *flops = n->net->flops_per_sample();
  if (arena) *arena = (long long)n->net->arena_bytes();
  if (ngemm) *ngemm = n->net->num_gemm_launches();
  if (nsteps) *nsteps = n->net->num_steps();
  MDB_API_END
}

int mdb_unet_gemm_ops(mdb_unet* n, int i, const char** name, double* flops, double* fill_bytes) {
  MDB_API_BEGIN
  if (i < 0 || i >= n->net->num_gemm_launches()) throw std::runtime_error("mdb: GEMM launch index out of range");
  const GemmOp& g = n->net->gemm(i);
  if (name) *name = g.name.c_str();
  if (flops) *flops = g.flops;
  if (fill_bytes) *fill_bytes = g.fill_bytes();
  MDB_API_END
}

int mdb_unet_gemm_slots(mdb_unet* n, int i, int* a_slots, int* b_slots, int* smem_bytes) {
  MDB_API_BEGIN
  if (i < 0 || i >= n->net->num_gemm_launches()) throw std::runtime_error("mdb: GEMM launch index out of range");
  int a = 0, b = 0, sm = 0;
  n->net->gemm(i).slots(a, b, sm);
  if (a_slots) *a_slots = a;
  if (b_slots) *b_slots = b;
  if (smem_bytes) *smem_bytes = sm;
  MDB_API_END
}

int mdb_unet_gemm_tiles(mdb_unet* n, int i, int* work_items, int* splits, int* ksteps, int* entry_ksteps, int* block_n) {
  MDB_API_BEGIN
  if (i < 0 || i >= n->net->num_gemm_launches()) throw std::runtime_error("mdb: GEMM launch index out of range");
  const GemmOp& g = n->net->gemm(i);
  const int s = g.p.splits > 1 ? g.p.splits : 1;
  int nk = 0;
  for (const LoadEntry& e : g.loads) nk = e.nk > nk ? e.nk : nk;
  if (work_items) *work_items = g.p.tx * g.p.ty * g.p.tz * g.p.tb * g.p.n_tiles_n * s;
  if (splits) *splits = s;
  if (ksteps) *ksteps = g.ksteps;
  if (entry_ksteps) *entry_ksteps = nk;
  if (block_n) *block_n = g.block_n;
  MDB_API_END
}

int mdb_unet_profile(mdb_unet* n, const float* x, const float* labels, float* out, int B, void* stream, char* names,
                     int names_len, float* ms, int max_steps, int* nsteps) {
  MDB_API_BEGIN
  auto r = n->net->profile(x, labels, out, B, (cudaStream_t)stream);
  std::string all;
  int k = 0;
  for (auto& p : r) {
    if (k >= max_steps) break;
    all += p.first; all += "\n";
    ms[k++] = p.second;
  }
  if ((int)all.size() + 1 > names_len) throw std::runtime_error("mdb: names buffer too small");
  std::memcpy(names, all.c_str(), all.size() + 1);
  if (nsteps) *nsteps = k;
  MDB_API_END
}

int mdb_unet_set_dropout(mdb_unet* n, float p, unsigned long long seed) {
  MDB_API_BEGIN
  n->net->set_dropout(p, seed);
  MDB_API_END
}

int mdb_unet_set_classes(mdb_unet* n, const int* classes, int B, void* stream) {
  MDB_API_BEGIN
  n->net->set_classes(classes, B, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_backward(mdb_unet* n, const float* dout, float* grads, long long grads_numel, int B, int accumulate, void* stream) {
  MDB_API_BEGIN
  if (grads_numel != n->net->total_param_numel()) throw std::runtime_error("mdb: gradient buffer has the wrong size");
  n->net->backward(dout, grads, B, accumulate != 0, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_backward_marked(mdb_unet* n, const float* dout, float* grads, long long grads_numel, int B, int accumulate,
                             const int* mark_steps, void* const* mark_events, int n_marks, void* stream) {
  MDB_API_BEGIN
  if (grads_numel != n->net->total_param_numel()) throw std::runtime_error("mdb: gradient buffer has the wrong size");
  if (n_marks > 0 && (!mark_steps || !mark_events)) throw std::runtime_error("mdb: null mark arrays");
  n->net->backward(dout, grads, B, accumulate != 0, (cudaStream_t)stream, mark_steps, mark_events, n_marks);
  MDB_API_END
}

int mdb_unet_backward_input(mdb_unet* n, const float* dout, float* dx, float* grads, long long grads_numel, int B, int accumulate,
                            void* stream) {
  MDB_API_BEGIN
  if (grads && grads_numel != n->net->total_param_numel()) throw std::runtime_error("mdb: gradient buffer has the wrong size");
  n->net->backward_input(dout, dx, grads, B, accumulate != 0, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_unet_grad_ready(mdb_unet* n, const char* name, int* step) {
  MDB_API_BEGIN
  *step = n->net->grad_ready_step(name);
  MDB_API_END
}

int mdb_unet_grad_offset(mdb_unet* n, const char* name, long long* off) {
  MDB_API_BEGIN
  *off = n->net->grad_offset(name);
  MDB_API_END
}

int mdb_unet_debug_stats(mdb_unet* n, long long* host_out, long long capacity, long long* count) {
  MDB_API_BEGIN
  const long long c = (long long)n->net->stats_count();
  if (count) *count = c;
  if (host_out) {
    if (capacity < c) throw std::runtime_error("mdb: stats buffer too small");
    MDB_CUDA_CHECK(cudaMemcpy(host_out, n->net->stats_ptr(), (size_t)c * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  MDB_API_END
}

int mdb_unet_train_info(mdb_unet* n, double* bwd_flops, int* nsteps, long long* numel) {
  MDB_API_BEGIN
  if (bwd_flops) *bwd_flops = n->net->bwd_flops_per_sample();
  if (nsteps) *nsteps = n->net->num_bwd_steps();
  if (numel) *numel = n->net->total_param_numel();
  MDB_API_END
}

int mdb_unet_profile_backward(mdb_unet* n, const float* dout, float* grads, int B, void* stream, char* names, int names_len,
                              float* ms, int max_steps, int* nsteps) {
  MDB_API_BEGIN
  auto r = n->net->profile_backward(dout, grads, B, (cudaStream_t)stream);
  std::string all;
  int k = 0;
  for (auto& p : r) {
    if (k >= max_steps) break;
    all += p.first; all += "\n";
    ms[k++] = p.second;
  }
  if ((int)all.size() + 1 > names_len) throw std::runtime_error("mdb: names buffer too small");
  std::memcpy(names, all.c_str(), all.size() + 1);
  if (nsteps) *nsteps = k;
  MDB_API_END
}

static void set_cond(SamplerUpdateArgs& a, const mdb_sampler_cond* c, float coef, float stdv) {
  if (!c || !c->partial) return;
  if (!c->partial_mask) throw std::runtime_error("mdb: conditional sampling needs partial_mask");
  if (c->channel < 0 || c->channel >= a.C) throw std::runtime_error("mdb: partial_channel out of range");
  a.cond_partial = c->partial; a.cond_partial_bs = c->partial_bstride;
  a.cond_pmask = c->partial_mask; a.cond_pmask_bs = c->mask_bstride;
  a.cond_channel = c->channel; a.cond_coef = coef; a.cond_std = stdv; a.cond_noise = c->noise;
}

int mdb_sampler_update(const float* eps, float* x, float* x_mean, const float* noise, const float* mask, float beta,
                       float stdv, long long V, int C, int B, unsigned long long seed, unsigned long long offset,
                       const mdb_sampler_cond* cond, void* stream) {
  MDB_API_BEGIN
  SamplerUpdateArgs a{};
  a.eps = eps; a.x = x; a.x_mean = x_mean; a.noise = noise; a.mask = mask; a.beta = beta; a.stdv = stdv;
  a.V = V; a.C = C; a.seed = seed; a.offset = offset;
  if (cond) set_cond(a, cond, cond->mean_coef, cond->std);
  launch_sampler_update(a, B, (cudaStream_t)stream);
  MDB_API_END
}

// Order-independent 64-bit fingerprint of fp32 tensors (position-weighted sum of the raw words, integer atomics).
// The Python shell uses it to notice parameter edits that bypass autograd's version counters (`p.data[...] = ...`,
// which is how the reference's trainer writes the grid mask and how its EMA copies weights).
__global__ void fingerprint_kernel(const unsigned int* const* ptrs, const long long* numels, unsigned long long* out) {
  const int t = blockIdx.y;
  const unsigned int* p = ptrs[t];
  const long long n = numels[t];
  unsigned long long h = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    h += (unsigned long long)p[i] * (0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1) | 1ull);
  for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if ((threadIdx.x & 31) == 0 && h) atomicAdd(out + t, h);
}

int mdb_fingerprint(const void* const* ptrs_dev, const long long* numels_dev, int n, unsigned long long* out_dev, void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  MDB_CUDA_CHECK(cudaMemsetAsync(out_dev, 0, (size_t)n * 8, s));
  fingerprint_kernel<<<dim3(64, n), 256, 0, s>>>(reinterpret_cast<const unsigned int* const*>(ptrs_dev), numels_dev, out_dev);
  MDB_CUDA_CHECK(cudaGetLastError());
  MDB_API_END
}

__global__ void fill_kernel(float* p, float v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// eps_buf <- network(x) at `label` for every sample of the batch (labels_buf: device scratch [B])
static void forward_at(mdb_unet* n, const float* x, float label, float* labels_buf, float* eps_buf, int B, cudaStream_t s) {
  fill_kernel<<<(B + 127) / 128, 128, 0, s>>>(labels_buf, label, B);
  n->net->forward(x, labels_buf, eps_buf, B, s, /*allow_graph=*/true);
}

int mdb_sampler_run(mdb_unet* n, float* x, float* x_mean, const float* mask, const float* labels, const float* betas,
                    const float* stds, int n_steps, int B, unsigned long long seed, float* eps_buf, float* labels_buf,
                    int step0, const mdb_sampler_cond* cond, const float* cond_mean_coefs, const float* cond_stds,
                    int cond_until, void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  const UNetConfig& c = n->net->cfg();
  const long long V = (long long)c.image_size * c.image_size * c.image_size;
  if (cond && cond->partial && (!cond_mean_coefs || !cond_stds)) throw std::runtime_error("mdb: conditional run needs the marginal_prob tables");
  if (cond && cond->noise) throw std::runtime_error("mdb: mdb_sampler_run draws its noise in-kernel (cond->noise must be NULL)");
  for (int i = 0; i < n_steps; ++i) {
    forward_at(n, x, labels[i], labels_buf, eps_buf, B, s);
    SamplerUpdateArgs a{};
    a.eps = eps_buf; a.x = x; a.x_mean = x_mean; a.noise = nullptr; a.mask = mask; a.beta = betas[i]; a.stdv = stds[i];
    // curand_normal consumes two 32-bit Philox outputs and `offset` counts single outputs: 4*i gives every step its own
    // 128-bit counter block, so the noise of consecutive steps is independent
    a.V = V; a.C = c.num_channels; a.seed = seed; a.offset = 4ull * (unsigned long long)(step0 + i);
    if (cond && step0 + i < cond_until) set_cond(a, cond, cond_mean_coefs[i], cond_stds[i]);
    launch_sampler_update(a, B, s);
  }
  MDB_API_END
}

int mdb_distill_targets(mdb_unet* n, const float* z_s, const int* step_idx, const mdb_distill_row* rows, int n_rows,
                        const float* mask, float* eps_target, float* labels, float* z_mid, float* eps_buf, int B,
                        void* stream) {
  MDB_API_BEGIN
  if (!n || !n->net) throw std::runtime_error("mdb: mdb_distill_targets needs the teacher network");
  if (n_rows < 1) throw std::runtime_error("mdb: mdb_distill_targets needs at least one row");
  if (!z_s || !step_idx || !rows || !mask || !eps_target || !labels || !z_mid || !eps_buf)
    throw std::runtime_error("mdb: mdb_distill_targets: null argument");
  if (B <= 0 || B > 65535) throw std::runtime_error("mdb: mdb_distill_targets needs a batch in [1, 65535]");
  cudaStream_t s = (cudaStream_t)stream;
  const UNetConfig& c = n->net->cfg();
  const long long V = (long long)c.image_size * c.image_size * c.image_size;
  // no CUDA graph: z_s, z_mid, eps_buf and labels are new buffers on every training micro-step, and graphs are keyed by
  // the buffer addresses
  n->net->forward(z_s, labels, eps_buf, B, s, /*allow_graph=*/false);
  launch_distill_step(eps_buf, z_s, z_mid, nullptr, mask, step_idx, rows, n_rows, 0, labels, V, c.num_channels, B, s);
  n->net->forward(z_mid, labels, eps_buf, B, s, /*allow_graph=*/false);
  launch_distill_step(eps_buf, z_s, z_mid, eps_target, mask, step_idx, rows, n_rows, 1, labels, V, c.num_channels, B, s);
  MDB_API_END
}

static SolverEntryArgs entry_args(const float* eps, float* x, float* x0_hist, const float* mask, const mdb_solver_entry& e,
                                  long long V, int C, const mdb_solver_known* k) {
  if (e.kind != 0 && e.kind != 1) throw std::runtime_error("mdb: solver entry kind must be 0 (denoise) or 1 (renoise)");
  SolverEntryArgs a{};
  a.renoise = e.kind; a.eps = eps; a.x = x; a.x0_hist = x0_hist; a.mask = mask;
  a.sigma = e.sigma; a.inv_alpha = e.inv_alpha; a.c_x = e.c_x; a.c_0 = e.c_0; a.c_1 = e.c_1; a.c_z = e.c_z;
  a.V = V; a.C = C;
  if (k && k->known && k->channels) {
    if (!k->mask) throw std::runtime_error("mdb: the kept region needs its mask");
    if (C > 32 || (C < 32 && (k->channels >> C) != 0u)) throw std::runtime_error("mdb: kept channel set outside the channels");
    a.known = k->known; a.known_bs = k->known_bstride; a.kmask = k->mask; a.kmask_bs = k->mask_bstride;
    a.channels = k->channels; a.coef = e.known_coef; a.std = e.known_std; a.known_noise = k->noise;
  }
  return a;
}

int mdb_solver_update(const float* eps, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entry,
                      long long V, int C, int B, const float* noise, unsigned long long seed, unsigned long long offset,
                      const mdb_solver_known* known, void* stream) {
  MDB_API_BEGIN
  if (!entry) throw std::runtime_error("mdb: mdb_solver_update needs an entry");
  if (V <= 0 || C <= 0 || B <= 0) throw std::runtime_error("mdb: mdb_solver_update needs positive voxels, channels, batch");
  SolverEntryArgs a = entry_args(eps, x, x0_hist, mask, *entry, V, C, known);
  if (!a.renoise && !eps) throw std::runtime_error("mdb: a denoise entry needs the network output");
  a.noise = noise; a.seed = seed; a.offset = offset;
  launch_solver_entry(a, B, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_solver_update_guided(const float* eps_c, const float* eps_u, float w, float* x, float* x0_hist, const float* mask,
                             const mdb_solver_entry* entry, long long V, int C, int B, const float* noise,
                             unsigned long long seed, unsigned long long offset, const mdb_solver_known* known, void* stream) {
  MDB_API_BEGIN
  if (!entry) throw std::runtime_error("mdb: mdb_solver_update_guided needs an entry");
  if (V <= 0 || C <= 0 || B <= 0) throw std::runtime_error("mdb: mdb_solver_update_guided needs positive voxels, channels, batch");
  SolverEntryArgs a = entry_args(eps_c, x, x0_hist, mask, *entry, V, C, known);
  if (!a.renoise && (!eps_c || !eps_u)) throw std::runtime_error("mdb: a guided denoise entry needs both network outputs");
  if (!a.renoise) { a.eps_u = eps_u; a.w = w; }
  a.noise = noise; a.seed = seed; a.offset = offset;
  launch_solver_entry(a, B, (cudaStream_t)stream);
  MDB_API_END
}

int mdb_solver_run_guided(mdb_unet* n, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entries,
                          int n_entries, int B, unsigned long long seed, const int* classes, float w, float* eps_buf,
                          float* eps_u_buf, float* labels_buf, int step0, const mdb_solver_known* known, int replace_until,
                          void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  UNet& net = *n->net;
  const UNetConfig& c = net.cfg();
  const long long V = (long long)c.image_size * c.image_size * c.image_size;
  if (c.num_classes == 0) throw std::runtime_error("mdb: mdb_solver_run_guided needs a class-conditional network (num_classes > 0)");
  if (!classes) throw std::runtime_error("mdb: mdb_solver_run_guided needs the class ids");
  if (w != 1.f && !eps_u_buf) throw std::runtime_error("mdb: mdb_solver_run_guided needs eps_u_buf unless w == 1");
  if (n_entries > 0 && !entries) throw std::runtime_error("mdb: mdb_solver_run_guided needs the entry table");
  if (known && known->noise) throw std::runtime_error("mdb: mdb_solver_run_guided draws its noise in-kernel (known->noise must be NULL)");
  net.set_classes(classes, B, s);  // copies and checks the ids once
  try {
    for (int i = 0; i < n_entries; ++i) {
      SolverEntryArgs a = entry_args(eps_buf, x, x0_hist, mask, entries[i], V, c.num_channels,
                                     step0 + i < replace_until ? known : nullptr);
      if (!a.renoise) {
        net.use_null_class(false);
        forward_at(n, x, entries[i].label, labels_buf, eps_buf, B, s);
        if (w != 1.f) {
          net.use_null_class(true);
          n->net->forward(x, labels_buf, eps_u_buf, B, s, /*allow_graph=*/true);
          a.eps_u = eps_u_buf; a.w = w;
        }
      }
      // mdb_solver_run's Philox counter blocks
      a.noise = nullptr; a.seed = seed; a.offset = 4ull * (unsigned long long)(step0 + i);
      launch_solver_entry(a, B, s);
    }
  } catch (...) {
    net.use_null_class(false);
    throw;
  }
  net.use_null_class(false);
  MDB_API_END
}

int mdb_solver_run(mdb_unet* n, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entries,
                   int n_entries, int B, unsigned long long seed, float* eps_buf, float* labels_buf, int step0,
                   const mdb_solver_known* known, int replace_until, void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  const UNetConfig& c = n->net->cfg();
  const long long V = (long long)c.image_size * c.image_size * c.image_size;
  if (n_entries > 0 && !entries) throw std::runtime_error("mdb: mdb_solver_run needs the entry table");
  if (known && known->noise) throw std::runtime_error("mdb: mdb_solver_run draws its noise in-kernel (known->noise must be NULL)");
  for (int i = 0; i < n_entries; ++i) {
    SolverEntryArgs a = entry_args(eps_buf, x, x0_hist, mask, entries[i], V, c.num_channels,
                                   step0 + i < replace_until ? known : nullptr);
    if (!a.renoise) forward_at(n, x, entries[i].label, labels_buf, eps_buf, B, s);
    // mdb_sampler_run's Philox counter blocks, keyed by the global entry: 4 outputs per entry, the replacement draw at +2
    a.noise = nullptr; a.seed = seed; a.offset = 4ull * (unsigned long long)(step0 + i);
    launch_solver_entry(a, B, s);
  }
  MDB_API_END
}

int mdb_conv3d(const void* x, int B, int cin, int z, int y_, int x_, const float* w, const float* bias, int cout,
               int ksize, int stride, void* out, const float* rowbias, const void* residual, long long* stats,
               int precision, void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  const Precision pr = precision_from_int(precision);
  const int xo = x_ / stride, yo = y_ / stride, zo = z / stride;
  GemmOp g;
  g.set_output(pr, xo, yo, zo, B, cout, out, cout, false);
  Act a; a.ptr = const_cast<void*>(x); a.C = cin; a.X = x_; a.Y = y_; a.Z = z; a.B = B;
  if (ksize == 1) g.add_pointwise({a}, w, false);
  else g.add_conv({a}, w, ksize, stride);
  if (bias) g.set_bias(bias);
  if (rowbias) g.set_rowbias(rowbias, cout);
  if (residual) g.set_residual(residual, cout, (long long)xo * yo * zo * cout, false);
  if (stats) g.set_stats(stats);
  g.finalize();
  g.upload(s);
  g.repack(s);
  g.launch(s);
  MDB_CUDA_CHECK(cudaStreamSynchronize(s));
  MDB_API_END
}

int mdb_groupnorm_act(const void* x, const long long* stats, const float* gamma, const float* beta, void* y, int B,
                      long long V, int C, int silu, int precision, void* stream) {
  MDB_API_BEGIN
  if (!stats) throw std::runtime_error("mdb: GroupNorm needs the per-channel statistics of x (stats)");
  cudaStream_t s = (cudaStream_t)stream;
  NormActArgs na{};
  na.x0 = x; na.C0 = C; na.ld0 = C; na.x1 = nullptr; na.C1 = 0; na.ld1 = 0;
  na.y = y; na.voxels = V; na.silu = silu; na.prec = precision_from_int(precision);
  na.stats0 = stats; na.stats1 = nullptr; na.gamma = gamma; na.beta = beta; na.groups = 32; na.eps = 1e-6f;
  launch_norm_act(na, B, s);
  MDB_CUDA_CHECK(cudaStreamSynchronize(s));
  MDB_API_END
}

int mdb_conv3d_backward(const void* dy, const void* x, const float* w, int B, int cin, int cout, int z, int y_, int x_,
                        int ksize, int stride, float* dw, void* dx, void* stream) {
  return mdb_conv3d_backward_prec(dy, x, w, B, cin, cout, z, y_, x_, ksize, stride, dw, dx, 0, stream);
}

int mdb_conv3d_backward_prec(const void* dy, const void* x, const float* w, int B, int cin, int cout, int z, int y_, int x_,
                             int ksize, int stride, float* dw, void* dx, int precision, void* stream) {
  MDB_API_BEGIN
  cudaStream_t s = (cudaStream_t)stream;
  const Precision pr = precision_from_int(precision);
  if (pr == kTF32) throw std::runtime_error("mdb: conv3d backward takes bf16 (0) or bf16x3 (2) operands");
  const int xo = x_ / stride, yo = y_ / stride, zo = z / stride;
  Act ady; ady.ptr = const_cast<void*>(dy); ady.C = cout; ady.X = xo; ady.Y = yo; ady.Z = zo; ady.B = B;
  Act ax; ax.ptr = const_cast<void*>(x); ax.C = cin; ax.X = x_; ax.Y = y_; ax.Z = z; ax.B = B;
  if (dw) {
    const int T = ksize * ksize * ksize;
    const WgradPlan pl = plan_wgrad(xo, yo, zo, B, cout, cin, ksize, stride, pr);
    float* scratch = nullptr;
    MDB_CUDA_CHECK(cudaMalloc(&scratch, pl.scratch_bytes));
    WgradOut o; o.ptr = dw; o.sm = (long long)cin * T; o.sn = T; o.st = 1;
    WgradOp op;
    op.init(ady, ax, ksize, stride, o, scratch, pr);
    op.launch(s, B, false);
    MDB_CUDA_CHECK(cudaStreamSynchronize(s));
    cudaFree(scratch);
  }
  if (dx) {
    if (stride != 1) throw std::runtime_error("mdb: conv3d data gradient entry point supports stride 1");
    GemmOp g;
    g.set_output(pr, x_, y_, z, B, cin, dx, cin, false);
    if (ksize == 1) { WSrc ws{w, 1, (long long)cin, 0, cout}; g.add_pointwise_w({ady}, &ws); }
    else g.add_conv_dgrad(ady, w, cin, ksize);
    g.finalize();
    g.upload(s);
    g.repack(s);
    g.launch(s);
    MDB_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  MDB_API_END
}

int mdb_groupnorm_act_backward(const void* x, const long long* stats, const float* gamma, const float* beta, void* da,
                               const void* add, void* dx, float* dgamma, float* dbeta, int B, long long V, int C, int silu,
                               float dropout_p, unsigned long long seed, void* stream) {
  return mdb_groupnorm_act_backward_prec(x, stats, gamma, beta, da, add, dx, dgamma, dbeta, B, V, C, silu, dropout_p, seed, 0, stream);
}

int mdb_groupnorm_act_backward_prec(const void* x, const long long* stats, const float* gamma, const float* beta, void* da,
                                    const void* add, void* dx, float* dgamma, float* dbeta, int B, long long V, int C, int silu,
                                    float dropout_p, unsigned long long seed, int precision, void* stream) {
  MDB_API_BEGIN
  if (!stats) throw std::runtime_error("mdb: GroupNorm backward needs the forward statistics of x (stats)");
  cudaStream_t s = (cudaStream_t)stream;
  const Precision pr = precision_from_int(precision);
  if (pr == kTF32) throw std::runtime_error("mdb: GroupNorm backward takes bf16 (0) or bf16x3 (2) operands");
  float *part = nullptr, *sums = nullptr;
  MDB_CUDA_CHECK(cudaMalloc(&part, (size_t)kBwdPartRows(B) * C * 2 * sizeof(float)));
  MDB_CUDA_CHECK(cudaMalloc(&sums, (size_t)B * C * 2 * sizeof(float)));
  GnBwdArgs a{};
  a.x0 = x; a.C0 = C; a.ld0 = C; a.stats0 = stats; a.gamma = gamma; a.beta = beta; a.da = da;
  a.voxels = V; a.silu = silu; a.groups = 32; a.eps = 1e-6f;
  const DropoutParams d = dropout_params(dropout_p);
  a.drop_thresh = d.thresh; a.drop_scale = d.scale; a.seed = seed;
  a.part = part; a.sums = sums; a.dgamma = dgamma; a.dbeta = dbeta; a.accumulate = 0;
  a.dx = dx; a.add0 = add; a.add0_ld = C;
  a.prec = pr;
  launch_gn_bwd_reduce(a, B, s);
  launch_gn_bwd_apply(a, B, s);
  MDB_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(part); cudaFree(sums);
  MDB_API_END
}

}  // extern "C"
