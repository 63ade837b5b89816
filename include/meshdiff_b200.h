/* meshdiff_b200 -- C ABI of the H100-native MeshDiffusion hot path.
 *
 * The reference (lzzcd001/MeshDiffusion) has no FFI on this path: its seam is a set of Python callables
 * (SURVEY.md section 8b). Each entry point below names the reference callable it replaces. All pointers are raw
 * device pointers unless stated otherwise; `stream` is a cudaStream_t passed as void*. Every function returns 0 on
 * success and a non-zero code on failure, with a message available from mdb_last_error(). Nothing here
 * synchronises the stream except where stated, and nothing allocates caller-visible memory.
 */
#ifndef MESHDIFF_B200_H
#define MESHDIFF_B200_H

#ifdef __cplusplus
extern "C" {
#endif

const char* mdb_last_error(void);
int mdb_version(void);

/* ------------------------------------------------------------------------------------------------------------
 * Score network. Replaces DDPMRes64 / DDPMRes128 construction + forward
 * (lib/diffusion/models/ddpm_res64.py:41-199, ddpm_res128.py:43-215) as created by
 * mutils.create_model (lib/diffusion/models/utils.py:88-96).
 */
typedef struct mdb_unet mdb_unet;

typedef struct mdb_unet_config {
  int image_size;          /* config.data.image_size */
  int nf;                  /* config.model.nf */
  int n_levels;            /* len(config.model.ch_mult) */
  int ch_mult[8];          /* config.model.ch_mult */
  int num_res_blocks;      /* config.model.num_res_blocks */
  int level0_blocks;       /* ddpm_res128.py:98 forces 2 at level 0; -1 = num_res_blocks */
  int n_attn;
  int attn_resolutions[4]; /* config.model.attn_resolutions */
  int num_channels;        /* config.data.num_channels */
  int stem_ksize;          /* 3 = ddpm_conv3x3 (res64), 5 = ddpm_conv5x5 (res128) */
  int use_pos_bias;        /* 1: stem adds pos_layer(coords*0) = its bias (ddpm_res64.py:148) */
  int max_batch;
  int precision;           /* 0 = bf16 operands, 1 = tf32 operands, 2 = split bf16 ("bf16x3": every value is a (hi, lo)
                              bf16 pair and every product hi*hi + hi*lo + lo*hi -- fp32-class results, the mode that
                              meets the 1e-3 parity contract); fp32 accumulation in all three */
  int training;            /* 1 = also build the backward plan and keep what it needs; precision 0 (bf16) or 2 (split bf16:
                              fp32-class gradients at about a third of the tensor rate); tf32 is refused */
  int num_classes;         /* config.model.num_classes: 0 = unconditional (the reference's network). K > 0 adds
                              label_embed.weight [K+1][4nf], last in the parameter table; row K is the null class of
                              classifier-free guidance: act(temb) = silu(Linear1(silu(Linear0(emb(t)))) + E[y]) */
} mdb_unet_config;

int mdb_unet_create(const mdb_unet_config* cfg, mdb_unet** out);
/* Plan only, no GPU needed: built by the same code as mdb_unet_create, so it answers the parameter table, arena size,
 * step and GEMM counts, mdb_unet_gemm_ops, mdb_unet_gemm_slots, mdb_unet_gemm_tiles, FLOPs, mdb_unet_train_info and mdb_unet_grad_ready. It cannot run:
 * set/get_param, commit, forward, backward* and profile* return an error. */
int mdb_unet_create_dry(const mdb_unet_config* cfg, mdb_unet** out);
void mdb_unet_destroy(mdb_unet* net);

/* Parameter table == the reference state_dict without the DataParallel `module.` prefix
 * (lib/diffusion/utils.py:23-30). Shapes are the reference's (OIDHW conv weights, [in,out] NIN.W, ...). */
int mdb_unet_num_params(mdb_unet* net);
int mdb_unet_param_info(mdb_unet* net, int idx, const char** name, long long* numel, int* ndim, long long* shape8);
/* load_state_dict: copy one tensor in (src on host if src_is_device == 0). */
int mdb_unet_set_param(mdb_unet* net, const char* name, const float* src, long long numel, int src_is_device,
                       void* stream);
/* The same for `count` DEVICE tensors in one call (the training step re-uploads all ~500 master parameters after every
 * optimiser step, losses.py:26-52: one host call instead of 500). */
int mdb_unet_set_params(mdb_unet* net, int count, const char* const* names, const float* const* srcs, const long long* numels,
                        void* stream);
/* state_dict: copy one tensor out; synchronises the stream. */
int mdb_unet_get_param(mdb_unet* net, const char* name, float* dst, long long numel, int dst_is_device, void* stream);
/* Re-derive packed weights / constant stem field after parameters changed; synchronises the stream. */
int mdb_unet_commit(mdb_unet* net, void* stream);
/* score_model(x, labels): x fp32 NCDHW [B][C][R][R][R], labels fp32 [B], out fp32 NCDHW (ddpm_res64.py:126-199). */
int mdb_unet_forward(mdb_unet* net, const float* x, const float* labels, float* out, int batch, void* stream);
int mdb_unet_info(mdb_unet* net, double* flops_per_sample, long long* arena_bytes, int* n_gemm_launches, int* n_steps);
/* Forward GEMM launch i (0 <= i < n_gemm_launches) at the engine's max batch: its step name (valid while the engine
 * lives), executed FLOPs and the bytes TMA writes into shared memory (A boxes + weight tiles, summed over output tiles). */
int mdb_unet_gemm_ops(mdb_unet* net, int i, const char** name, double* flops, double* fill_bytes);
/* Operand ring depth of forward GEMM launch i: the A slots (entries in flight) and B slots (k-steps of weight tiles in
 * flight) it takes under the current MDB_MAX_STAGES / MDB_MAX_BSLOTS, and the dynamic shared memory it requests. */
int mdb_unet_gemm_slots(mdb_unet* net, int i, int* a_slots, int* b_slots, int* smem_bytes);
/* Tile shape of forward GEMM launch i at the engine's max batch: the work items its persistent CTAs share (output tiles
 * times the split-K factor), the split-K factor, the k-steps of one output tile, the most k-steps of one load-table entry
 * (3 or 5 for a halo convolution) and the tile width BLOCK_N. A launch runs on min(work items, SMs) CTAs. */
int mdb_unet_gemm_tiles(mdb_unet* net, int i, int* work_items, int* splits, int* ksteps, int* entry_ksteps, int* block_n);
/* One profiled forward: per-step device milliseconds. names_buf receives '\n'-separated step names. Synchronises. */
int mdb_unet_profile(mdb_unet* net, const float* x, const float* labels, float* out, int batch, void* stream,
                     char* names_buf, int names_len, float* ms, int max_steps, int* n_steps);

/* ---- training (engines created with cfg.training = 1). Replaces `loss.backward()` through score_model
 * (lib/diffusion/losses.py:104-139 -> torch autograd over ddpm_res64.py:126-199).
 * Dropout of the next forward/backward pair (nn.Dropout(p) after GroupNorm_1+SiLU, layers.py:661,682); p = 0 is
 * model.eval(). The same (p, seed) must be in force for a forward and its backward. */
int mdb_unet_set_dropout(mdb_unet* net, float p, unsigned long long seed);
/* Class ids (device int32 [batch], each in 0..K with K = num_classes the null class; NULL = the null class for every
 * sample) of the following forward/backward pairs, which must run at this batch; in force until the next call, like
 * mdb_unet_set_dropout. The ids are copied on `stream` into a buffer the engine owns and checked there; the check copies
 * them back to the host and synchronises `stream`. The caller's array may be freed when the call returns. Each forward
 * copies the ids in force, on its stream, into a second engine buffer at a fixed address, which is what its CUDA graphs
 * read. An engine with num_classes = 0 refuses a non-NULL pointer; an id outside 0..K is an error (no ids are then in
 * force: the null class). */
int mdb_unet_set_classes(mdb_unet* net, const int* classes, int batch, void* stream);
/* dout = dL/d(out) of the immediately preceding mdb_unet_forward (same x, labels, batch; x and labels must still be
 * alive). grads: ONE flat fp32 buffer of grads_numel = sum of all parameter numels, parameter i at the offset
 * mdb_unet_grad_offset gives (table order); slots of non-trainable tensors (mask, coords, sigmas, pos_layer.weight,
 * whose input is coords*0) are not written. accumulate != 0: grads += (micro-batching, losses.py:111-113). */
int mdb_unet_backward(mdb_unet* net, const float* dout, float* grads, long long grads_numel, int batch, int accumulate,
                      void* stream);
int mdb_unet_grad_offset(mdb_unet* net, const char* name, long long* offset);
/* dx = dL/dx fp32 NCDHW [B][C][R][R][R] of the immediately preceding mdb_unet_forward (same contract as mdb_unet_backward;
 * engines with 4 input channels). grads == NULL: input gradient only -- launches whose only outputs are parameter gradients
 * are not enqueued. grads != NULL: the full mdb_unet_backward (same grads / accumulate semantics) plus dx. dx is bitwise the
 * same either way. Vector-Jacobian products of the score network for the probability-flow likelihood (no reference
 * counterpart: the reference differentiates with torch autograd, lib/diffusion/likelihood.py:26-37). */
int mdb_unet_backward_input(mdb_unet* net, const float* dout, float* dx, float* grads, long long grads_numel, int batch,
                            int accumulate, void* stream);
/* Data-parallel overlap (replaces the gradient gather of nn.DataParallel, lib/diffusion/models/utils.py:95): the backward
 * plan is a fixed launch list; mdb_unet_grad_ready gives, per parameter, the number of launches after which its gradient
 * is final (0 = never written). mdb_unet_backward_marked is mdb_unet_backward that additionally records the caller's CUDA
 * events (cudaEvent_t as void*) on `stream` once mark_steps[j] launches (ascending) have been enqueued, so the host can
 * all-reduce a finished range of the flat buffer on another stream while the remaining launches run. */
int mdb_unet_grad_ready(mdb_unet* net, const char* name, int* n_launches);
int mdb_unet_backward_marked(mdb_unet* net, const float* dout, float* grads, long long grads_numel, int batch,
                             int accumulate, const int* mark_steps, void* const* mark_events, int n_marks, void* stream);
/* Diagnostics: copies the raw GroupNorm statistics of the last forward to the host (split fixed-point records (sum lo, sum hi,
 * sumsq lo, sumsq hi), per tensor [B][C][4] in plan order); synchronises. count receives the number of int64 values. */
int mdb_unet_debug_stats(mdb_unet* net, long long* host_out, long long capacity, long long* count);
int mdb_unet_train_info(mdb_unet* net, double* bwd_flops_per_sample, int* n_bwd_steps, long long* total_param_numel);
/* One profiled backward (same contract as mdb_unet_profile). */
int mdb_unet_profile_backward(mdb_unet* net, const float* dout, float* grads, int batch, void* stream, char* names_buf,
                              int names_len, float* ms, int max_steps, int* n_steps);

/* Position-weighted 64-bit fingerprints of n fp32 device tensors (ptrs_dev / numels_dev / out_dev are device
 * arrays of n entries). Host plumbing for load_state_dict-style change detection; no reference counterpart. */
int mdb_fingerprint(const void* const* ptrs_dev, const long long* numels_dev, int n, unsigned long long* out_dev,
                    void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sampler. Replaces AncestralSamplingPredictor.vpsde_update_fn + get_score_fn + the two grid_mask multiplies of
 * pc_sampler (lib/diffusion/sampling.py:222-230, 469-478; lib/diffusion/models/utils.py:191-198).
 * eps = network output, x / x_mean fp32 NCDHW [B][C][V], mask [V]; noise may be NULL (then Philox(seed, offset)).
 */
/* Replacement conditioning of pc_sampler's partial branch (`cond_gen`; lib/diffusion/sampling.py:453-467), fused into the
 * same update kernel. After the masked predictor update, on channel `channel` only (g = grid mask, pm = partial_mask):
 *   x_c <- (x_c (1 - pm) + partial pm) g;   s = mean_coef x_c + std z';   x_c <- (x_c (1 - pm) + s pm) g;   x_mean_c <- x_c
 * with (mean_coef, std) = VPSDE.marginal_prob(., t_i) (sde_lib.py:210-214). partial / partial_mask point at channel
 * `channel` of sample 0 ([V] floats); *_bstride is the element distance to the next sample (0 = one grid shared by the
 * whole batch, the (1,1,R,R,R) tensors evaler.py:181-201 builds). noise: z' [B][V], or NULL for Philox(seed, offset + 2). */
typedef struct mdb_sampler_cond {
  const float* partial;
  long long partial_bstride;
  const float* partial_mask;
  long long mask_bstride;
  int channel;
  float mean_coef, std; /* mdb_sampler_update only (mdb_sampler_run takes per-step tables) */
  const float* noise;
} mdb_sampler_cond;

/* Philox: element e of step i draws its predictor noise from counter block (seed, subsequence e, offset); `offset` counts
 * 32-bit outputs and a normal consumes two, so callers stepping a loop pass offset = 4 * i (mdb_sampler_run does). */
int mdb_sampler_update(const float* eps, float* x, float* x_mean, const float* noise, const float* mask, float beta,
                       float std, long long voxels, int channels, int batch, unsigned long long seed,
                       unsigned long long offset, const mdb_sampler_cond* cond /* nullable */, void* stream);
/* Whole predictor loop of pc_sampler (unconditional branch sampling.py:469-478; partial branch :441-467 when `cond` is
 * given) without host round trips: for i < n_steps: labels[i] -> network -> update [-> replacement conditioning while
 * step0 + i < cond_until, i.e. min(freeze_iters, N - 1)]. labels/betas/stds (and cond_mean_coefs/cond_stds) are HOST
 * arrays of n_steps floats for the global steps step0 .. step0 + n_steps - 1. eps_buf: device scratch [B][C][V];
 * labels_buf: device scratch [B]. Noise is in-kernel Philox at offset 4 * (step0 + i). The call only enqueues work. */
int mdb_sampler_run(mdb_unet* net, float* x, float* x_mean, const float* mask, const float* labels,
                    const float* betas, const float* stds, int n_steps, int batch, unsigned long long seed,
                    float* eps_buf, float* labels_buf, int step0, const mdb_sampler_cond* cond /* nullable */,
                    const float* cond_mean_coefs, const float* cond_stds, int cond_until, void* stream);

/* Solver tables: few-step sampling with DPM-Solver++(2M) (Lu et al. 2022), ODE or SDE form, on the same noise prediction
 * as the sampler above, its inverse (a grid's latent), the distilled student's DDIM grid, and RePaint resampling
 * (Lugmayr et al. 2022) for shape editing (`--mode=edit`). diffusion/sampling.py computes every table in float64 on the
 * host (dpm_solver_schedule, dpm_solver_inversion_schedule, ddim_table, repaint_schedule). An entry is one of two kinds,
 * on x fp32 [B][C][V] with the grid mask g [V]:
 *   denoise (kind 0): the network runs at `label`, then one DPM-Solver++(2M) step from that label to the next:
 *            x0 = (x - sigma eps) inv_alpha;  x' = (c_x x + c_0 x0 + c_1 x0_prev + c_z z) g;  x0_prev <- x0
 *            c_1 = 0 marks a first-order step (x0_prev is not read); c_z = 0 one without noise.
 *   renoise (kind 1): a jump up the label grid by forward diffusion, no network: x' = (c_x x + c_z z) g with
 *            c_x = alpha_hi / alpha_lo and c_z = sqrt(1 - c_x^2); x0_prev is not touched (sigma, inv_alpha, c_0, c_1 unused)
 * With a kept region, both kinds then replace it on every channel c in `known->channels`:
 *   x_c <- (x_c (1 - m) + (known_coef known_c + known_std z'_c) m) g
 * with (known_coef, known_std) = alpha, sigma of the label the entry lands on. The conditional sampler (`cond_gen`) keeps
 * one channel of a partial grid and stops replacing before its last step; a RePaint table ends with (1, 0), which makes
 * the kept region of the output equal `known`. */
typedef struct mdb_solver_entry {
  int kind;                      /* 0 = denoise, 1 = renoise */
  float label;                   /* denoise: network label; renoise: the label it jumps to */
  float sigma, inv_alpha;        /* x0 = (x - sigma*eps) * inv_alpha */
  float c_x, c_0, c_1, c_z;      /* x' = c_x*x + c_0*x0 + c_1*x0_prev + c_z*z */
  float known_coef, known_std;   /* replacement after the entry */
} mdb_solver_entry;

/* The kept region. known: channel 0 of sample 0 of a [B][C][V] fp32 tensor; known_bstride is the element distance to the
 * next sample (0 = one grid for the whole batch). mask: m [V] of sample 0, mask_bstride likewise. channels: bit c set =
 * channel c is replaced (channels < 2^C). noise: z' [B][C][V], or NULL for Philox(seed, element, offset + 2). */
typedef struct mdb_solver_known {
  const float* known;
  long long known_bstride;
  const float* mask;
  long long mask_bstride;
  unsigned channels;
  const float* noise;
} mdb_solver_known;

/* One entry, in place on x and x0_hist ([batch][channels][voxels] fp32; mask [voxels]). eps: the network output (denoise;
 * ignored by renoise). noise: z [batch][channels][voxels], or NULL for Philox(seed, element, offset) with element the
 * index in x, as in mdb_sampler_update (a loop passes offset = 4 * e for global entry e). known: nullable (no
 * replacement). */
int mdb_solver_update(const float* eps, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entry,
                      long long voxels, int channels, int batch, const float* noise /* nullable */,
                      unsigned long long seed, unsigned long long offset, const mdb_solver_known* known /* nullable */,
                      void* stream);
/* The whole table without host round trips: for i < n_entries: denoise entries run entries[i].label -> network
 * (eps_buf) -> update, renoise entries the update alone, with in-kernel Philox at offset 4 * (step0 + i), and the
 * replacement while step0 + i < replace_until. `entries` is a HOST array of n_entries entries for the global entries
 * step0 .. step0 + n_entries - 1. eps_buf: device scratch [B][C][V]; labels_buf: device scratch [B]. known->noise must be
 * NULL. The call only enqueues work. */
int mdb_solver_run(mdb_unet* net, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entries,
                   int n_entries, int batch, unsigned long long seed, float* eps_buf, float* labels_buf, int step0,
                   const mdb_solver_known* known /* nullable */, int replace_until, void* stream);

/* Classifier-free guidance (Ho & Salimans 2022) of a class-conditional network. A guided denoise entry reads the
 * conditional output eps_c and the null-class output eps_u and uses, in the same single pass over HBM,
 *   eps = eps_u + w (eps_c - eps_u)     (each operation rounded on its own)
 * in place of eps; the rest is mdb_solver_update's arithmetic, unchanged. Renoise entries ignore both outputs. */
int mdb_solver_update_guided(const float* eps_c, const float* eps_u, float w, float* x, float* x0_hist, const float* mask,
                             const mdb_solver_entry* entry, long long voxels, int channels, int batch,
                             const float* noise /* nullable */, unsigned long long seed, unsigned long long offset,
                             const mdb_solver_known* known /* nullable */, void* stream);
/* mdb_solver_run with guidance: each denoise entry runs the network twice at `batch`, with `classes` (device int32
 * [batch], checked as mdb_unet_set_classes checks them) into eps_buf and with the null class into eps_u_buf (device
 * scratch [B][C][V]), then the guided entry. w == 1 runs the conditional forward and the plain entry only (eps_u_buf may
 * be NULL): bitwise mdb_unet_set_classes(classes) followed by mdb_solver_run. After the call `classes` are the ids in
 * force, as after mdb_unet_set_classes. */
int mdb_solver_run_guided(mdb_unet* net, float* x, float* x0_hist, const float* mask, const mdb_solver_entry* entries,
                          int n_entries, int batch, unsigned long long seed, const int* classes, float w, float* eps_buf,
                          float* eps_u_buf, float* labels_buf, int step0, const mdb_solver_known* known /* nullable */,
                          int replace_until, void* stream);

/* Progressive distillation (Salimans & Ho 2022; `--mode=distill`, diffusion/distill.py, with the rows computed in float64
 * on the host by diffusion/sampling.py: distill_rows). A student step i moves z from label s = l_{2i} to e = l_{2i+2} of
 * the teacher's DDIM grid l (ddim_grid); the teacher takes two first-order ODE (DDIM) steps s -> m = l_{2i+1} -> e, each
 * in the form of mdb_solver_update's denoise entry with c_1 = c_z = 0:  x0 = (z - sigma eps) inv_alpha;
 *   z' = (c_x z + c_0 x0) g.
 * The student's target is the noise prediction whose single DDIM step from z_s lands on the teacher's z_e:
 *   eps~ = (z_e - r z_s) inv_d   with r = alpha_e / alpha_s and inv_d = 1 / (sigma_e - alpha_e sigma_s / alpha_s). */
typedef struct mdb_distill_row {
  float label_s, label_m, label_e;                    /* network labels of the three grid points */
  float sigma_s, inv_alpha_s, c_x_s, c_0_s;           /* teacher step s -> m */
  float sigma_m, inv_alpha_m, c_x_m, c_0_m;           /* teacher step m -> e */
  float r, inv_d;                                     /* target coefficients */
} mdb_distill_row;

/* One phase on fp32 [batch][channels][voxels] tensors (mask g [voxels]). step_idx: DEVICE int [batch], sample b uses
 * rows[step_idx[b]]; rows: DEVICE array of n_rows entries. An index outside [0, n_rows) reads no row: that sample's
 * outputs and label are NaN.
 *   phase 0 (teacher step s -> m, eps = teacher(z_s, s)): z_mid = (c_x_s z_s + c_0_s x0) g, bitwise mdb_solver_update's
 *           first-order denoise entry; labels[b] = m (the next forward's labels). out is not touched (may be NULL).
 *   phase 1 (teacher step m -> e, eps = teacher(z_mid, m)): z_e as above from z_mid, then out = ((z_e - r z_s) inv_d) g;
 *           labels[b] = s (the student's labels). z_mid is read only.
 * Every product and sum is rounded on its own. The call only enqueues work. */
int mdb_distill_step(const float* eps, const float* z_s, float* z_mid, float* out, const float* mask, const int* step_idx,
                     const mdb_distill_row* rows, int n_rows, int phase, float* labels, long long voxels, int channels,
                     int batch, void* stream);
/* The student's targets on the teacher's inference engine, without host round trips: teacher(z_s, labels) -> phase 0 ->
 * teacher(z_mid, labels) -> phase 1 -> eps_target. labels: device fp32 [batch] holding s = rows[step_idx[b]].label_s on
 * entry (the perturbation and the student's forward use them too); it holds them again on return. z_mid, eps_buf: device
 * scratch [batch][C][V]. Rows and indices as in mdb_distill_step. The call only enqueues work. */
int mdb_distill_targets(mdb_unet* teacher, const float* z_s, const int* step_idx, const mdb_distill_row* rows, int n_rows,
                        const float* mask, float* eps_target, float* labels, float* z_mid, float* eps_buf, int batch,
                        void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Training-step kernels (optimiser side). Replace get_ddpm_loss_fn's elementwise tail (lib/diffusion/losses.py:69-78),
 * torch.nn.utils.clip_grad_norm_ + torch.optim.Adam.step (losses.py:45-50, 26-35) and
 * ExponentialMovingAverage.update (lib/diffusion/models/ema.py:43-64). Pointer tables / numels are DEVICE arrays of
 * n entries (one per parameter tensor). The multi-tensor passes walk a CHUNK TABLE the host builds once: a device array of
 * n_chunks (tensor index, chunk index) int32 pairs covering every tensor in pieces of mdb_chunk_elems() elements.
 */
/* loss = mean_b[mean_{c,v}((pred-noise)^2 mask[v])] * V / mask_sum -> *loss_out; grad_pred (nullable) = dloss/dpred.
 * scratch: one device double. */
int mdb_ddpm_loss(const float* pred, const float* noise, const float* mask, double mask_sum, float* loss_out,
                  float* grad_pred, double* scratch, int batch, int channels, long long voxels, void* stream);
/* x_t = (sqrt_ac[b] x_0 + sqrt_1mac[b] eps) * mask[v] (losses.py:63-66), fp32 NCDHW [B][C][V]; coefficient arrays [B] on
 * the device; same rounding as the eager torch expression. */
int mdb_ddpm_perturb(const float* x0, const float* noise, const float* mask, const float* sqrt_ac,
                     const float* sqrt_1mac, float* out, int batch, int channels, long long voxels, void* stream);
int mdb_chunk_elems(void);
/* clip_grad_norm_ (losses.py:49): coef = min(1, max_norm / (||g||_2 + 1e-6)) over all tensors -> *coef_out (and the norm
 * in *total_norm_out); the gradients themselves are NOT rescaled (mdb_adam_ema_step applies the coefficient on the fly).
 * scratch: n_chunks device doubles (per-chunk partials, summed in a fixed order: reproducible). */
int mdb_grad_clip_coef(const float* const* grads_dev, const long long* numels_dev, const int* chunks_dev, int n_chunks,
                       float max_norm, float* coef_out, float* total_norm_out, double* scratch, void* stream);
/* g *= *clip_coef (nullable); torch.optim.Adam(lr, beta1, beta2, eps, weight_decay) update number `step` >= 1 (losses.py:26-35);
 * then, when ema_dev != NULL, ExponentialMovingAverage.update: ema -= (1 - ema_decay)(ema - p) (ema.py:43-64). One pass. */
int mdb_adam_ema_step(float* const* params_dev, const float* const* grads_dev, float* const* exp_avg_dev,
                      float* const* exp_avg_sq_dev, float* const* ema_dev, const long long* numels_dev,
                      const int* chunks_dev, int n_chunks, float lr, float beta1, float beta2, float eps,
                      float weight_decay, int step, const float* clip_coef_dev, float ema_decay, void* stream);
/* ExponentialMovingAverage.update on its own (micro-steps that accumulate gradients without an optimiser step). */
int mdb_ema_update(float* const* ema_dev, const float* const* params_dev, const long long* numels_dev,
                   const int* chunks_dev, int n_chunks, float ema_decay, void* stream);

/* Data-parallel training: mean all-reduce of the flat gradient buffer (what mdb_unet_backward filled) over the caller's
 * NCCL communicator (ncclComm_t passed as void*), in place, on `stream`; replaces nn.DataParallel's gradient gather
 * (lib/diffusion/models/utils.py:95). NCCL is taken from the libnccl.so.2 already loaded in the process. The Python
 * host of this repository uses torch.distributed.all_reduce on the same buffer instead (torch owns its communicator). */
int mdb_allreduce_grads(void* nccl_comm, float* grads, long long numel, int world_size, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Operator-level entry points (parity tests call these like the reference's renderutils tests call its ops).
 * Activations are NDHWC in the operand dtype of `precision` (bf16 or fp32).
 */
/* nn.Conv3d k in {1,3,5}, stride 1 (padding k/2) or stride 2 (Downsample: pad-high + VALID, layers.py:626-643).
 * x: [B][Z][Y][X][Cin] (input extents), w: fp32 OIDHW, y: [B][Zo][Yo][Xo][Cout]. Optional: bias [Cout],
 * rowbias [B][Cout], residual (same layout as y), stats [B][Cout][4] int64 = (sum, sum of squares) of the result as
 * split fixed-point pairs, value = w_lo * 2^-24 + w_hi * 2^16 (csrc/gn_stats.cuh: exact, order-independent, cannot
 * overflow), accumulated with integer atomics (must be zeroed by the caller). */
int mdb_conv3d(const void* x, int batch, int cin, int z, int y_, int x_, const float* w, const float* bias, int cout,
               int ksize, int stride, void* out, const float* rowbias, const void* residual, long long* stats,
               int precision, void* stream);
/* GroupNorm(32, eps=1e-6) [+ SiLU] from channel statistics: x [B][V][C], stats [B][C][4] (split fixed point, as above),
 * y [B][V][C]. */
int mdb_groupnorm_act(const void* x, const long long* stats, const float* gamma, const float* beta, void* y, int batch,
                      long long voxels, int channels, int silu, int precision, void* stream);

/* Backward of mdb_conv3d for bf16 operands (k = 3 stride 1 | 2, or k = 1): what autograd's conv3d backward returns.
 * dy: [B][Zo][Yo][Xo][Cout], x: [B][Z][Y][X][Cin] (both bf16 NDHWC), w: fp32 OIDHW. dw (nullable): fp32 OIDHW;
 * dx (nullable, stride 1 only): bf16 [B][Z][Y][X][Cin]. Synchronises. */
int mdb_conv3d_backward(const void* dy, const void* x, const float* w, int batch, int cin, int cout, int z, int y_,
                        int x_, int ksize, int stride, float* dw, void* dx, void* stream);
/* The same with an operand mode: precision 0 = bf16 (= mdb_conv3d_backward), 2 = split bf16 (dy, x and dx rows of 2C
 * bf16: the hi parts of the C channels, then their lo parts, as in mdb_conv3d). */
int mdb_conv3d_backward_prec(const void* dy, const void* x, const float* w, int batch, int cin, int cout, int z, int y_,
                             int x_, int ksize, int stride, float* dw, void* dx, int precision, void* stream);
/* Backward of mdb_groupnorm_act (bf16): da = dL/dy [B][V][C] -> dx [B][V][C], dgamma / dbeta fp32 [C]. `add`
 * (nullable, [B][V][C]) is summed into dx. Dropout (p, seed) as in mdb_unet_set_dropout. `da` is used as scratch
 * (overwritten with the pre-activation gradient). Synchronises. */
int mdb_groupnorm_act_backward(const void* x, const long long* stats, const float* gamma, const float* beta,
                               void* da, const void* add, void* dx, float* dgamma, float* dbeta, int batch,
                               long long voxels, int channels, int silu, float dropout_p, unsigned long long seed,
                               void* stream);
/* The same with an operand mode: precision 0 = bf16 (= mdb_groupnorm_act_backward), 2 = split bf16 (x, da, add and dx
 * rows of 2C bf16, hi parts then lo parts). */
int mdb_groupnorm_act_backward_prec(const void* x, const long long* stats, const float* gamma, const float* beta,
                                    void* da, const void* add, void* dx, float* dgamma, float* dbeta, int batch,
                                    long long voxels, int channels, int silu, float dropout_p, unsigned long long seed,
                                    int precision, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Implicit-GEMM test entry points: one GemmOp (or one of the engine's multi-launch composites) built from a description
 * with the builder calls the engine uses, so a test can compare a single variant with a reference of that operation.
 * Activations are NDHWC rows in the operand format of `precision` (split bf16: the hi parts of a row's channels, then
 * their lo parts, `lo_off` logical elements further on). All of them synchronise the stream.
 */
/* One A source: [batch_plan][z][y][x] voxels of `channels` channels, `ld` logical elements apart (0 = channels). */
typedef struct mdb_gemm_src {
  const void* ptr;
  int channels, x, y, z;
  long long ld;
} mdb_gemm_src;
enum { MDB_PROBE_CONV = 0, MDB_PROBE_CONV_UP2 = 1, MDB_PROBE_CONV_DGRAD = 2, MDB_PROBE_POINTWISE = 3, MDB_PROBE_ACT_B = 4 };
typedef struct mdb_gemm_probe_desc {
  int precision;          /* 0 bf16, 1 tf32, 2 split bf16 */
  int kind;               /* MDB_PROBE_*: add_conv, add_conv_up2, add_conv_dgrad, add_pointwise, add_pointwise_w(NULL) */
  int ksize, stride;      /* conv: k in {1,3,5}, stride 1 | 2; dgrad: k */
  int parity;             /* conv_up2: px | py << 1 | pz << 2 */
  int n_src;              /* 1 or 2 (the channel concatenation) */
  mdb_gemm_src src[2];
  /* conv: OIDHW [n][sum C][k^3]; conv_up2: the 3^3 OIDHW weight [n][C][27], folded by launch_upconv_weights;
   * dgrad: the forward conv's OIDHW [C of src 0][n][k^3]; pointwise: [in][out] (w_in_out) or [out][in]. fp32. */
  const float* w;
  int w_in_out;
  /* activation B (MDB_PROBE_ACT_B): B[batch][n][k], rows b_row_stride and samples b_batch_stride logical elements apart */
  const void* b_ptr;
  int b_k, b_n;
  long long b_row_stride, b_batch_stride;
  /* extra pointwise k-steps in the same accumulator (the NIN shortcut of a resblock's Conv_1): W_extra [in][out] */
  int n_extra;
  mdb_gemm_src extra[2];
  const float* w_extra;
  /* output (set_output_strided): grid x, y, z of the planned batch, n columns, logical strides */
  int x, y, z, n;
  void* out;
  long long osx, osy, osz, osb, lo_off;  /* lo_off < 0: osx */
  int out_fp32;
  /* epilogue */
  const float* bias;
  const float* rowbias;
  long long rowbias_ld;
  const void* residual;   /* in the operand format */
  long long res_ld, res_batch_stride;
  long long* stats;
  float alpha;            /* 0 = 1 */
  int splits;             /* 0 = none, -1 = plan_splits as the engine calls it, > 1 = forced (clamped to the k-groups) */
  int batch_plan, batch;  /* built for batch_plan samples, launched at batch (<= batch_plan; <= 0: batch_plan) */
  int dry;                /* 1: describe only (no CUDA call; pointers may be NULL) and fill the report */
  /* GroupNorm(32, eps 1e-6) backward (bf16 / split bf16; the training plan's data-gradient GEMMs): the GEMM result `out`
   * (dense, n = gn_c0 + gn_c1 channels) is dL/da of a = dropout(act(GroupNorm(x))) over the concatenation x = {gn_x0,
   * gn_x1} (dense rows, forward statistics as mdb_conv3d writes them). gnb = 1: the fused epilogue (set_gn_backward,
   * after launch_gn_consts; then launch_gnb_tile_reduce and launch_gn_bwd_apply), as the training plan builds it;
   * gnb = 2: the same GEMM without it, then launch_gn_bwd_reduce and launch_gn_bwd_apply (the two-pass path). Both
   * overwrite `out` with dL/dy and write gn_dx [batch][voxels][n] and gn_dgamma / gn_dbeta [n] (fp32). */
  int gnb;
  const void* gn_x0; int gn_c0;
  const void* gn_x1; int gn_c1;
  const long long* gn_stats0; const long long* gn_stats1;
  const float* gn_gamma; const float* gn_beta;
  int gn_silu;
  float gn_dropout;                /* p of the dropout after the activation (0 = none) */
  unsigned long long gn_seed;      /* the layer's dropout seed */
  void* gn_dx; float* gn_dgamma; float* gn_dbeta;
} mdb_gemm_probe_desc;
/* What mdb_unet_gemm_tiles and mdb_unet_gemm_ops report for a launch at its planned batch. */
typedef struct mdb_gemm_probe_report {
  int work_items, splits, ksteps, entry_ksteps, block_n;
  double flops, fill_bytes;
} mdb_gemm_probe_report;
int mdb_gemm_probe(const mdb_gemm_probe_desc* desc, mdb_gemm_probe_report* report, void* stream);
/* The inference plan's sub-pixel Upsample + conv3^3 (the engine's own construction): x [batch_plan][r^3][C] -> out
 * [batch_plan][(2r)^3][C]; w fp32 OIDHW [C][C][27], bias [C], stats as in mdb_conv3d (nullable). w8: caller scratch of
 * 64 C^2 floats that receives the fold [8 parities][C][C][2][2][2]. parity_mask: bit p launches parity class p.
 * reports (nullable): the 8 parity ops. dry: describe only. */
int mdb_upsample_conv(const void* x, const float* w, const float* bias, float* w8, void* out, long long* stats, int r,
                      int C, int batch_plan, int batch, int parity_mask, int precision, int dry,
                      mdb_gemm_probe_report* reports, void* stream);
/* The attention core of the engine's AttnBlock over qkv rows [batch_plan][V][3C] (q | k | v): stage bit 0 = v^T into
 * vT [batch_plan][C][V], bit 1 = logits S = q k^T / sqrt(C) (fp32 [batch_plan][V][V]), bit 2 = softmax of the rows of S
 * in place (probabilities in the operand format at the start of each fp32 row), bit 3 = O = P v ([batch_plan][V][C]).
 * reports (nullable): the qk and pv ops. */
int mdb_attention_core(const void* qkv, void* vT, float* S, void* O, int V, int C, int batch_plan, int batch, int stages,
                       int precision, int dry, mdb_gemm_probe_report* reports, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Marching tetrahedra. Replaces DMTet.__call__ (nvdiffrec/lib/geometry/dmtet.py:105-163; tables :34-54, map_uv
 * :70-99) for a batch of samples over one static tet grid. Integer outputs (faces, uv_idx, face_to_tet,
 * valid_vert_idx; all int64 like the reference's torch.long) are bit-exact with the reference ordering.
 */
/* tets: HOST int32 [F][4] (the npz `indices`); builds the static sorted edge table on the device. */
int mdb_marching_tets_prepare(const int* tets_host, int n_tets, int n_verts, int max_batch, void** handle);
void mdb_marching_tets_destroy(void* handle);
int mdb_marching_tets_info(void* handle, int* n_edges, int* uv_grid_n);
/* uvs: device fp32 [uv_grid_n^2 * 4][2] */
int mdb_marching_tets_uvs(void* handle, float* uvs, void* stream);
/* Phase 1 (synchronises): sdf device fp32 [B][n_verts]; counts_host[b] = {n_verts_out, n_faces, n_valid_verts}. */
int mdb_marching_tets_count(void* handle, const float* sdf, int batch, int* counts_host, void* stream);
/* Phase 2: pos device fp32 [B][n_verts][3] (pos_batch_stride in floats; 0 = shared). Outputs packed per sample at
 * the given element offsets (device int64 [B]); NULL offsets = samples packed back to back in batch order (the exclusive
 * sums of the phase-1 counts, which the library keeps on the device: no upload needed). */
int mdb_marching_tets_extract(void* handle, const float* pos, long long pos_batch_stride, const float* sdf, int batch,
                              float* verts, long long* faces, long long* uv_idx, long long* face_to_tet,
                              long long* valid_vert_idx, const long long* vert_off, const long long* face_off,
                              const long long* vv_off, void* stream);
/* Backward of the vertex interpolation: what torch autograd computes for DMTet.__call__'s `verts` with respect to `pos_nx3`
 * and `sdf_n` (nvdiffrec/lib/geometry/dmtet.py:125-132 under loss.backward(); every other output is an integer tensor).
 * grad_verts fp32 packed like `verts`; vert_off device int64 [B] (NULL = the offsets of the last phase 1); vertex_ids device
 * uint32 [B][n_edges] = crossing edge -> output row, as copied by mdb_marching_tets_vertex_ids after the forward extract
 * (NULL = the last extract's, still held by the handle). grad_pos fp32 [B][n_verts][3] and grad_sdf fp32 [B][n_verts] are
 * overwritten (either may be NULL). A gather per grid vertex over its incident edges: no atomics, bitwise reproducible. */
int mdb_marching_tets_vertex_ids(void* handle, int batch, unsigned* out, void* stream);
int mdb_marching_tets_backward(void* handle, const float* pos, long long pos_batch_stride, const float* sdf, int batch,
                               const unsigned* vertex_ids, const float* grad_verts, const long long* vert_off,
                               float* grad_pos, float* grad_sdf, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Mesh post-ops after marching tets (SURVEY 8f-1). Scatter-adds run as 2^-40 fixed-point integer atomics: results are
 * independent of face order (bitwise reproducible).
 */
/* auto_normals (nvdiffrec/lib/render/mesh.py:200-227): v_pos fp32 [Nv][3], faces int64 [F][3] -> v_nrm fp32 [Nv][3]
 * (sum of unnormalised face normals, degenerate -> (0,0,1), safe_normalize), f_nrm fp32 [F][3] (nullable).
 * scratch: device int64 [Nv][3]. */
int mdb_mesh_auto_normals(const float* v_pos, const long long* faces, int n_verts, int n_faces, float* v_nrm, float* f_nrm,
                          long long* scratch, void* stream);
/* compute_tangents (mesh.py:233-277): per-face tangent from positions and texture coordinates, averaged per normal
 * index, Gram-Schmidt against v_nrm. v_tex fp32 [Nt][2]; index arrays int64 [F][3]; v_nrm fp32 [Nn][3] -> v_tng [Nn][3].
 * scratch: device bytes Nn*3*8 + Nn*4. */
int mdb_mesh_compute_tangents(const float* v_pos, const long long* t_pos_idx, const float* v_tex, const long long* t_tex_idx,
                              const float* v_nrm, const long long* t_nrm_idx, int n_nrm, int n_faces, float* v_tng,
                              long long* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Point-cloud metrics of generated shapes (MMD / COV / 1-NNA over the Chamfer distance). No reference counterpart: the
 * reference's fitting code calls kaolin's sample_points / chamfer_distance (nvdiffrec/lib/geometry/dmtet.py:455-457).
 */
/* Area-weighted surface sampling of n_meshes meshes packed like mdb_marching_tets_extract's output: verts fp32 [V][3],
 * faces int64 [F][3] with indices local to their mesh (not checked here: the caller validates them), vert_off device int64
 * [n_meshes], face_off device int64 [n_meshes + 1] (exclusive sums, face_off[n_meshes] = F). Face areas
 * 0.5 |(b-a) x (c-a)| and their per-mesh inclusive prefix sum (the CDF) are fp64 in face order; cdf: device scratch of F
 * doubles. Point j of mesh b takes uniforms (u, r1, r2) in [0, 1) from uniforms [n_meshes][n_points][3] or, when it is NULL,
 * from Philox(seed, subsequence (first_id + b) * n_points + j, offset 0) (24 high bits of each of the first three outputs
 * times 2^-24); its face is the smallest k with cdf[k] > u * total and its position
 * (1 - sqrt r1) a + sqrt r1 (1 - r2) b + sqrt r1 r2 c -> points fp32 [n_meshes][n_points][3]. A mesh with no faces or zero
 * total area gets n_written[b] = 0 (device int32 [n_meshes]; n_points otherwise) and none of its points are written. */
int mdb_mesh_sample_points(const float* verts, const long long* faces, const long long* vert_off, const long long* face_off,
                           int n_meshes, int n_points, const float* uniforms, unsigned long long seed, long long first_id,
                           double* cdf, float* points, int* n_written, void* stream);
/* out[i][j] = CD(A_i, B_j) fp64 [nA][nB] for A fp32 [nA][N][3], B fp32 [nB][M][3]:
 * CD(X, Y) = mean_x min_y d(x, y) + mean_y min_x d(x, y), d = fmaf(dz, dz, fmaf(dy, dy, dx * dx)) in fp32 (the
 * squared-distance, sum-of-two-means convention of kaolin's chamfer_distance). Bitwise reproducible and batch-invariant;
 * CD(X, Y) and CD(Y, X) are bitwise equal. B == NULL: self matrix of A (nB, M ignored), only i < j computed and mirrored,
 * diagonal exactly 0. The N + M per-point minima of a pair live in shared memory: N + M up to about 50 000 points. */
int mdb_chamfer_matrix(const float* A, int nA, int N, const float* B, int nB, int M, double* out, void* stream);
/* Paired Chamfer distances for shape completion. clouds fp32 [n_clouds][N][3] (one size N); pairs: DEVICE int32 [P][2] of
 * cloud indices (a, b). Per pair p, one CTA computes, with mdb_chamfer_matrix's distance, minima and fixed-order sums:
 *   cd[p]      = CD(clouds[a], clouds[b]), bitwise mdb_chamfer_matrix's entry for the same two clouds;
 *   mean_ab[p] = mean over x in a of min over y in b of d (the a->b half of cd[p]);
 *   max_ab[p]  = max over x in a of min over y in b of d (fp32; sqrt of it is the one-sided Hausdorff distance a->b).
 * Bitwise reproducible; an entry does not depend on the other pairs of the launch. Callers check the list on the host:
 * a pair with a == b or an index outside [0, n_clouds) is not an error here but gets NaN in all three outputs. 2N
 * per-point minima live in shared memory, as in mdb_chamfer_matrix. The call only enqueues work. */
int mdb_chamfer_pairs(const float* clouds, int n_clouds, int N, const int* pairs, int P, double* cd, double* mean_ab,
                      float* max_ab, void* stream);
/* out[i][j] = EMD(A_i, B_j) fp64 [nA][nB] for A fp32 [nA][N][3], B fp32 [nB][N][3] (equal sizes):
 * EMD(X, Y) = min over bijections pi of (1/N) sum_i |x_i - y_pi(i)| (Euclidean, not squared), with
 * |d| = sqrt((dx*dx + dy*dy) + dz*dz) in fp32, each operation rounded. Forward auction with epsilon-scaling, one CTA per
 * pair: every entry is the mean cost of a bijection, at most eps above the optimum over those fp32 costs.
 * gap[i][j] = out[i][j] minus the dual lower bound (sum_i min_j (c_ij + p_j) - sum_j p_j) / N of the final prices: a
 * certificate that out[i][j] - optimum <= gap[i][j] <= eps. eps must be at least 2^-18 times the diagonal of the pair's
 * joint bounding box (fp32 prices resolve it); a pair below that floor gets NaN in both outputs, a pair that needs more than
 * 2^18 auction rounds gets out = NaN and gap = +inf. Coordinates must be finite (not checked here: the caller checks them).
 * Bitwise reproducible and batch-invariant. B == NULL: self matrix of A (nB ignored), only i < j computed and mirrored,
 * diagonal exactly 0 with gap 0. About 35 N bytes of shared memory per pair: N up to about 6000 points. */
int mdb_emd_matrix(const float* A, int nA, const float* B, int nB, int N, float eps, double* out, double* gap, void* stream);
/* Light field descriptors (Chen et al. 2003 structure; geometry/lfd.py). face_id int32 [n_images][res][res] (res in
 * [1, 256]); the silhouette is face_id >= 0. One CTA of 256 threads per image; pixel p (row-major, centre (c + 0.5, r + 0.5))
 * belongs to thread p mod 256, visited in increasing order. n = inside pixels, cx = fp32(fp64(sum 2c + 1) / 2n), cy
 * likewise; dx = x - cx, dy = y - cy, radius r = sqrt(max (dx dx + dy dy)) + 0.5. Zernike n = 1..10, m = n mod 2..n step 2
 * (35 terms): per inside pixel u = dx / r, w = dy / r, s = u u + w w, V* = P_nm(s) (u - i w)^m (P_nm = R_n^m / rho^m by
 * Horner in s, powers by repeated complex products), fp32 products added into fp64 per-thread sums, combined by the tree
 * part[t] += part[t + s], s = 128..1; |A| = ((n + 1) |sum|) / ((pi r) r), byte min(255, floor(256 |A| + 0.5)). Fourier:
 * ray k of 64 (ray_cs device fp32 [64][2], cos and sin), sample j at (cx + (0.5 j) cos, cy + (0.5 j) sin) while inside
 * [0, res)^2; r_k = 0.5 x the last j whose pixel (floor y, floor x) is inside (else 0); F_m = sum_k r_k e^(-2 pi i m k / 64)
 * in k order with dft device fp64 [11][64][2] (cos, sin); byte min(255, floor(512 |F_m| / |F_0| + 0.5)), m = 1..10 (0 when
 * F_0 = 0). desc uint8 [n_images][48]: 35 Zernike, 10 Fourier, 3 zero bytes (all zero for an empty image); n_inside int32
 * [n_images]. Every operation rounded on its own: oracle/lfd_oracle.py reproduces the bytes. */
int mdb_lfd_descriptors(const int* face_id, int n_images, int res, const float* ray_cs, const double* dft,
                        unsigned char* desc, int* n_inside, void* stream);
/* Light field distance matrix. A uint8 [nA][10][10][48], B uint8 [nB][10][10][48] (light field, view, descriptor; 16-byte
 * aligned); perms device int8 [60][10], the view permutation pi_g of each rotation of the dodecahedron (values outside
 * 0..9 are clamped to 9). out int32 [nA][nB] = min over light fields s of A, t of B and g of
 * sum_i sum_c |A[s][i][c] - B[t][pi_g(i)][c]|: one CTA per pair builds the 100 x 100 view-distance table in shared memory
 * (__vsadu4) and takes the 6000 alignment sums as lookups. Exact integers: batch-invariant, and symmetric when perms is
 * a group. B == NULL: self matrix of A (nB ignored), only i < j computed and mirrored, diagonal 0. nA, nB <= 65535. */
int mdb_lfd_matrix(const unsigned char* A, int nA, const unsigned char* B, int nB, const signed char* perms, int* out,
                   void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Probability-flow ODE likelihood (lib/diffusion/likelihood.py:26-113 with the continuous VP score -e / std(t)).
 * One evaluation of the ODE right-hand side between the network's forward and its input-only backward:
 *   drift = mask * (-0.5 beta) (x - e / std)                       (VPSDE.sde + reverse(probability_flow=True))
 *   div[b] = -0.5 beta * ( sum_masked h^2  -  (1/std) sum_masked h * g )   g = J_e^T (h * mask), from mdb_unet_backward_input
 * x, e, h, g, drift fp32 [B][C][V]; mask [V] shared by the batch, or NULL (all ones); h = Hutchinson noise.
 * div: fp64 per sample, fixed-order reduction (bitwise reproducible, batch-invariant). */
int mdb_pflow_drift_div(const float* x, const float* e, const float* h, const float* g, const float* mask, float beta, float std,
                        float* drift, double* div, int batch, int channels, long long voxels, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Single-view visibility for partial DMTets (nvdiffrec/lib/render/render.py:335-407, fit_singleview.py:783-827): a
 * first-layer depth / face-id rasterization and the reference's visible-tet test on top of it. Every product, sum and
 * quotient is rounded on its own (no FMA contraction), so a float32 restatement reproduces both bit for bit.
 */
/* Rasterizes n_jobs (mesh, view) jobs into res x res buffers. Meshes are packed like mdb_marching_tets_extract's output:
 * verts fp32 [V][3], faces int64 [F][3] local to their mesh, vert_off device int64 [n_meshes], face_off device int64
 * [n_meshes + 1]. job_mesh device int32 [n_jobs] (mesh of each job, not range-checked here), mvp device fp32 [n_jobs][16]
 * (row-major). Per vertex clip = mvp [x, y, z, 1] (each row ((m0 x + m1 y) + m2 z) + m3); a face with a vertex at
 * w <= 0 is not drawn and is counted in n_behind (device int32 [n_jobs], overwritten); so is a face with a non-finite
 * screen coordinate or a zero area, uncounted. Screen X = (x / w * 0.5 + 0.5) * res (likewise Y); pixel (r, c) has its
 * centre at (c + 0.5, r + 0.5), so row 0 is clip y = -1. A pixel is covered when its centre lies in the face's bounding
 * box and every edge function has the sign of the area or is zero (both windings); depth = z / w interpolated with the
 * edge-function weights, dropped outside [-1, 1]. The nearest fragment wins, ties to the lower face index (a 64-bit
 * atomicMin on (depth key, face)). depth fp32 [n_jobs][res][res] (100 where empty), face_id int32 (-1 where empty; else
 * the face's index within its mesh). scratch: device uint64 [n_jobs][res][res]. */
int mdb_raster_depth(const float* verts, const long long* faces, const long long* vert_off, const long long* face_off,
                     const int* job_mesh, const float* mvp, int n_jobs, int res, unsigned long long* scratch, float* depth,
                     int* face_id, int* n_behind, void* stream);
/* For every tet t and job j: centre c = (((p0 + p1) + p2) + p3) * 0.25 over pos + job_mesh[j] * pos_stride (fp32 [Nv][3];
 * pos_stride in floats, 0 = shared), h = mvp c, n = h.xyz / h.w, q = rint((n * 0.5 + 0.5) * (res - 1)) (half to even).
 * visible[j][t] = 1 when q is in [0, res - 1] in all three components and, over rows q.y +- 7 and columns q.x +- 7
 * clipped to the image, the minimum depth is >= n.z or every pixel is empty. rast[j][t] = 1 when
 * face_to_tet[face_off[job_mesh[j]] + id] == t for an id in the job's face_id buffer. tets device int32 [n_tets][4]
 * (16-byte aligned); depth / face_id as mdb_raster_depth wrote them; visible, rast uint8 [n_jobs][n_tets], overwritten. */
int mdb_visible_tets(const float* pos, long long pos_stride, const int* tets, int n_tets, const long long* face_to_tet,
                     const long long* face_off, const int* job_mesh, const float* mvp, int n_jobs, int res, const float* depth,
                     const int* face_id, unsigned char* visible, unsigned char* rast, void* stream);
/* The diffuse preview image of nvdiffrec/eval.py (kd material, environment light, white background) on the face ids of an
 * mdb_raster_depth pass at res * ssaa (ssaa in 1..4, res * ssaa <= 16384). Meshes, job_mesh and mvp as in
 * mdb_raster_depth; v_nrm fp32 [V][3] smooth vertex normals packed like verts; campos device fp32 [n_jobs][3] (world-space
 * camera position, the translation of the inverse model-view); face_id [n_jobs][res * ssaa][res * ssaa]. Per sub-pixel
 * centre (c + 0.5, r + 0.5): empty -> bg; else barycentrics e_k / area made perspective-correct (b_k / w_k renormalised),
 * interpolated position p and smooth normal, and bsdf_prepare_shading_normal with two-sided shading (safe-normalised smooth
 * normal and view campos - p, face normal (v1 - v0) x (v2 - v0) normalised, both flipped unless face . view > 0, lerp
 * geom + t (smooth - geom) with t = clamp(view . smooth / 0.1, 0, 1)); colour kd * max(E(n), 0) with E the 9-term real SH
 * sum_i sh_coef[i][c] Y_i(n) (order Y00, Y1-1, Y10, Y11, Y2-2, Y2-1, Y20, Y21, Y22; sh_coef device fp32 [9][3], the SH
 * coefficients of irradiance / pi). Per output pixel: the ssaa^2 sub-pixel colours summed in row-major order, divided by
 * ssaa^2, and each channel encoded as the number of srgb_thresholds (device fp32 [255], ascending) it reaches. kd, bg:
 * device fp32 [3], linear. rgb uint8 [n_jobs][res][res][3], row 0 = buffer row 0. Every step rounded on its own. */
int mdb_render_shade(const float* verts, const float* v_nrm, const long long* faces, const long long* vert_off,
                     const long long* face_off, const int* job_mesh, const float* mvp, const float* campos, int n_jobs, int res,
                     int ssaa, const int* face_id, const float* sh_coef, const float* kd, const float* bg,
                     const float* srgb_thresholds, unsigned char* rgb, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Geometry-only fit of DMTet training grids to triangle meshes (`--mode=fit_grids`; the reference fits them by rendering,
 * nvdiffrec/fit_dmtets.py). Every product, sum and quotient is rounded on its own (no FMA contraction), so a float32
 * restatement reproduces the flags, distances, indices and closest points bit for bit.
 */
/* Space carving. pts fp32 [n_pts][3] (shared by the meshes); mvp device fp32 [n_views][16] (row-major); depth / face_id
 * [n_meshes][n_views][res][res] as mdb_raster_depth wrote them. Per vertex and view: clip = mvp [p, 1] (rows as in
 * mdb_raster_depth), skipped unless w > 0; X = (x / w * 0.5 + 0.5) * res, Y likewise, z = z / w; skipped unless X and Y
 * are in [0, res); pixel (floor Y, floor X). The view sees the vertex when every pixel of rows floor Y +- window and
 * columns floor X +- window, clipped to the image, is empty (face_id < 0) or has depth > z. outside uint8
 * [n_meshes][n_pts]: set to 1 where a view sees the vertex, left as it is elsewhere (zero it before the first call, so
 * that views can be carved in several calls). */
int mdb_carve_vertices(const float* pts, int n_pts, const float* mvp, int n_views, int n_meshes, int res, int window,
                       const float* depth, const int* face_id, unsigned char* outside, void* stream);
/* Closest point of a triangle mesh for every query point. Queries fp32 [Q][3] packed by mesh: query_off device int64
 * [n_meshes + 1] (exclusive sums), max_queries >= the largest per-mesh count. Meshes packed as in mdb_raster_depth
 * (verts, faces int64 local to their mesh, vert_off [n_meshes], face_off [n_meshes + 1]). Brute force over the mesh's
 * faces by Voronoi region (Ericson, Real-Time Collision Detection 5.1.5); a degenerate face whose regions give no finite
 * point takes the nearest of its edges ab, bc, ca. dist2 fp32 [Q] = (dx dx + dy dy) + dz dz of query - closest; face int64
 * [Q] = the nearest face's index within its mesh, ties to the lower index; closest fp32 [Q][3]. A mesh without faces gives
 * dist2 = +inf, face = -1 and NaN points. */
int mdb_closest_points(const float* queries, const long long* query_off, int n_meshes, long long max_queries, const float* verts,
                       const long long* faces, const long long* vert_off, const long long* face_off, float* dist2,
                       long long* face, float* closest, void* stream);
/* Nearest point of a point set for every query: queries packed as in mdb_closest_points, points fp32 [P][3] packed by
 * point_off device int64 [n_meshes + 1]. dist2 fp32 [Q] as in mdb_closest_points; index int64 [Q] within the mesh's
 * points, ties to the lower index; -1 (and dist2 = +inf) when the set is empty. */
int mdb_nearest_vertex(const float* queries, const long long* query_off, int n_meshes, long long max_queries, const float* points,
                       const long long* point_off, float* dist2, long long* index, void* stream);
/* out fp32 [n_rows][width] (overwritten): row r = sum of src[perm[k]] (fp32 [*][width]) over k in
 * [row_off[r], row_off[r + 1]), added in k order. With perm a stable sort of the rows' keys this is a deterministic
 * scatter-add (no float atomics). perm, row_off device int64. */
int mdb_segment_sum(const float* src, int width, const long long* perm, const long long* row_off, long long n_rows, float* out,
                    void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Partial DMTets from observed depth maps (`--mode=partial_from_depth`). Every product, sum and quotient is rounded on its
 * own (no FMA contraction), so a float32 restatement reproduces the buffers, flags, distances and points bit for bit.
 */
/* depth fp32 [n_obs][res][res]: camera depth along -z_cam, row 0 = clip y = -1; 0 or non-finite = no surface. proj,
 * inv_mv device fp32 [n_obs][16] (row-major): the perspective matrix (rows [p00 0 p02 0], [0 p11 p12 0], [0 0 A B],
 * [0 0 -1 0]) and the inverse of the model-view. Per observed pixel (r, c): x_ndc = (c + 0.5) / res * 2 - 1 (y_ndc from
 * r), camera point (d (x_ndc + p02) / p00, d (y_ndc + p12) / p11, -d), world point = rows 0-2 of inv_mv times it (rows as
 * in mdb_raster_depth), z / w = (B - A d) / d. Outputs [n_obs][res][res]: zbuf fp32 (100 where empty), valid int32 (0
 * surface, -1 empty; with zbuf the buffers mdb_carve_vertices reads), points fp32 [..][3] (0 where empty), edge uint8 (1
 * where an observed 4-neighbour's depth differs by more than max_jump). res in [2, 4096]. */
int mdb_depth_unproject(const float* depth, int n_obs, int res, const float* proj, const float* inv_mv, float max_jump,
                        float* zbuf, int* valid, float* points, unsigned char* edge, void* stream);
/* Closest point on the observed surface for every query: queries fp32 [Q][3] packed by observation (query_off device
 * int64 [n_obs + 1], max_queries >= the largest count); mvp, proj device fp32 [n_obs][16]; points, valid, edge as
 * mdb_depth_unproject wrote them. The query is projected like mdb_carve_vertices (skipped unless w > 0 and X, Y lie within
 * 64 px of the image); the window half-width is min(31, ceil(radius max(|p00|, |p11|) 0.5 res / w)) blocks around block
 * (floor(Y - 0.5), floor(X - 0.5)), clipped to the image. Block (r, c) with all four corner pixels valid and not edges
 * gives triangles (r c, r c+1, r+1 c+1) and (r c, r+1 c+1, r+1 c), tested as in mdb_closest_points; blocks in row-major
 * order, the nearest wins, ties to the first. dist2 fp32 [Q] (+inf if none), closest fp32 [Q][3] (NaN if none), found
 * uint8 [Q]. */
int mdb_depth_closest_points(const float* queries, const long long* query_off, int n_obs, long long max_queries, int res,
                             const float* mvp, const float* proj, float radius, const float* points, const int* valid,
                             const unsigned char* edge, float* dist2, float* closest, unsigned char* found, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Shape interpolation (`--mode=uncond_gen_interp`). Replaces `slerp` of lib/diffusion/evaler.py:63-71 (which the
 * reference's uncond_gen_interp, :73-130, applies to two prior noises): spherical interpolation over the whole tensor, no
 * grid mask.
 */
/* Number of reduction chunks per pair (the second extent of `partial`). */
int mdb_slerp_chunks(void);
/* P = pairs endpoint pairs za, zb fp32 [P][n]; alphas: HOST fp64 [frames] (any finite values; frames >= 2).
 * Phase 1: pair p is cut into mdb_slerp_chunks() contiguous ranges of ceil(n / chunks) elements whatever P; each range's
 *   fp64 sums of a*b, a*a, b*b (per thread in element order, then a fixed block tree) -> partial [P][chunks][3] (device
 *   scratch, overwritten).
 * Phase 2: the chunk sums in a fixed tree -> sums fp64 [P][3] = (a.b, a.a, b.b); bitwise reproducible and independent of P.
 *   In fp64: cos t = a.b / sqrt(a.a b.b) clamped to [-1, 1], t = acos, w_a = sin((1 - alpha) t) / sin t,
 *   w_b = sin(alpha t) / sin t; when a.a or b.b is 0 or sin t < 1e-6 (parallel or antiparallel endpoints) the weights
 *   are lerp's (1 - alpha, alpha). Rounded to fp32 -> coef [P][frames][2] (8-byte aligned). alpha = 0 and 1 give exactly
 *   (1, 0) and (0, 1).
 * Phase 3: out fp32 [P][frames][n], frame f of pair p = fl(fl(w_a a) + fl(w_b b)) per element, each operation rounded on
 *   its own. The call only enqueues work. */
int mdb_slerp_frames(const float* za, const float* zb, long long n, int pairs, const double* alphas, int frames,
                     double* partial, double* sums, float* coef, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
