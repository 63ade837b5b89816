// Bandwidth-bound kernels around the wgmma contractions: GroupNorm finalize/apply (+SiLU), nearest 2x upsample,
// stem im2col, attention softmax / V transpose, time-embedding MLP, ancestral-sampling and DPM-Solver updates.
// All of these are HBM-roofline kernels: 16-byte vector accesses, grid-stride loops sized to the SM count.
#pragma once
#include "act_format.cuh"

namespace mdb {

// y[b][v][c] = act(GroupNorm(x)[b][v][c]) over the channel concatenation of up to 2 sources, in operand mode `prec`.
struct NormActArgs {
  const void* x0; int C0; long long ld0;
  const void* x1; int C1; long long ld1;
  void* y;                                 // [B][V][C0+C1] dense
  long long voxels; int silu; Precision prec;
  // per-channel (sum, sumsq) records of the two sources (gn_stats.cuh), affine parameters
  const long long* stats0; const long long* stats1;
  const float* gamma; const float* beta;
  int groups; float eps;
  // training: nn.Dropout after the activation (act_format.cuh: apply_dropout)
  int drop_thresh; float drop_scale; unsigned long long seed;
};
void launch_norm_act(const NormActArgs& a, int B, cudaStream_t s);

// moves whole rows: elem_bytes = 2 (bf16; a split-bf16 row is passed as 2C channels) or 4 (fp32)
void launch_upsample2x(const void* x, void* y, int B, int Z, int Y, int X, int C, int elem_bytes, cudaStream_t s);

// x fp32 NCDHW [B][Cin][R^3] -> A[b][voxel][Kpad], column = cin*k^3 + tap (tap = (kd*k+kh)*k+kw), zero padded.
void launch_im2col(const float* x, void* a, int B, int Cin, int R, int ksize, int Kpad, Precision prec, cudaStream_t s);

// in-place row softmax: rows of L fp32 logits (row stride L floats); writes probabilities in the activation dtype
// at the start of each row (bf16 rows keep the fp32 row pitch).
void launch_softmax_rows(float* s, long long rows, int L, Precision prec, cudaStream_t st);

// out[b][c][v] = in[b][v][c0 + c], elements of elem_bytes = 2 or 4 bytes
void launch_transpose_vc(const void* in, long long ld_in, int c0, void* out, int B, int V, int C, int elem_bytes,
                         cudaStream_t s, long long ld_out = 0);

// temb path (ddpm_res64.py:132-136 + layers.py:542-556,680): act(temb)[B][4nf]
void launch_temb(const float* labels, const float* w0, const float* b0, const float* w1, const float* b1, float* out,
                 int B, int nf, cudaStream_t s);
// out[b][n] = W[n][:] . x[b][:] + bias[n]   (all Dense_0 projections at once)
void launch_dense(const float* x, const float* w, const float* bias, float* out, int B, int K, int N, cudaStream_t s);

// Head convolution, second phase: out[b][co][v] = bias[co] + sum_taps P[b][v + off(tap)][tap*Cout + co] (zero outside the
// grid). P holds the per-tap projections of the normalised activations ([B][V][ldp], activation dtype or fp32).
void launch_tap_shift_sum(const void* P, long long ldp, int p_fp32, const float* bias, float* out, int B, int R, int k,
                          int Cout, cudaStream_t s);

// Split-K reduction + the GEMM epilogue terms: out[b][v][n] = sum_s partial[s][b][v][n] + bias[n] + rowbias[b][n] +
// res[b][v][n], stored in the activation dtype, with the per-(sample, channel) GroupNorm statistics.
struct SplitReduceArgs {
  const float* partial; long long split_stride; int splits;
  const float* bias; const float* rowbias; long long rowbias_ld;
  const void* res; long long res_batch_stride;  // same [V][N] layout as out (activation dtype)
  void* out; long long* stats; long long voxels; int N; Precision prec;
};
void launch_split_reduce(const SplitReduceArgs& a, int B, cudaStream_t s);

void launch_add_vec(const float* a, const float* b, float* out, int n, cudaStream_t s);

// Sub-pixel form of Upsample(nearest x2) + conv3^3 (layers.py:611-623): w OIDHW [Cout][Cin][3][3][3] -> w8
// [8 parities (pz,py,px)][Cout][Cin][2][2][2] with, per axis, parity 0: {W0, W1+W2}, parity 1: {W0+W1, W2}.
void launch_upconv_weights(const float* w, float* w8, int Cout, int Cin, cudaStream_t s);

// Ancestral-sampling predictor update fused with the score scaling and both mask multiplies
// (sampling.py:222-230,476-478; models/utils.py:191-198). All fp32, NCDHW [B][4][V]; mask [V].
struct SamplerUpdateArgs {
  const float* eps;    // network output
  float* x;            // in/out state
  float* x_mean;       // out
  const float* noise;  // z ~ N(0,1) or null (then Philox below)
  const float* mask;   // [V]
  float beta, stdv;    // beta_t, sqrt(1-alpha_bar_t)
  long long V; int C;
  unsigned long long seed, offset;  // Philox stream for in-kernel noise
  // replacement conditioning of pc_sampler's partial branch (sampling.py:453-467), applied to channel cond_channel after
  // the masked predictor update when cond_partial != nullptr:
  //   x_c <- (x_c (1-pm) + partial pm) g;  s = coef x_c + std z';  x_c <- (x_c (1-pm) + s pm) g;  x_mean_c <- x_c
  const float* cond_partial; long long cond_partial_bs;  // channel c of sample 0, sample stride (0 = shared grid)
  const float* cond_pmask; long long cond_pmask_bs;
  int cond_channel;
  float cond_coef, cond_std;     // marginal_prob(x, t_i): exp(log_mean_coeff), sqrt(1 - exp(2 log_mean_coeff))
  const float* cond_noise;       // z' [B][V] or null (then Philox(seed, element, offset + 2))
};
void launch_sampler_update(const SamplerUpdateArgs& a, int B, cudaStream_t s);

// One entry of a solver table (csrc/solver.cu), in place, fp32 NCDHW [B][C][V]; mask g [V]:
//   denoise: x0 = (x - sigma eps) inv_alpha;  x' = (c_x x + c_0 x0 [+ c_1 x0_prev] [+ c_z z]) g;  x0_hist <- x0
//            (the c_1 term is skipped when c_1 == 0, a first-order step that does not read x0_hist; the noise term when
//            c_z == 0)
//   renoise: x' = (c_x x + c_z z) g   (c_x = alpha_hi / alpha_lo, c_z = sqrt(1 - c_x^2); x0_hist untouched)
// then, when known != nullptr, on every channel c with bit c of `channels` set:
//   x_c <- (x_c (1 - m) + (coef known_c + std z'_c) m) g
struct SolverEntryArgs {
  int renoise;
  const float* eps;    // network output (denoise)
  float* x;            // in/out state
  float* x0_hist;      // denoise: in x0 of the previous step, out x0 of this step
  const float* mask;   // g [V]
  float sigma, inv_alpha, c_x, c_0, c_1, c_z;
  long long V; int C;
  const float* noise;               // z [B][C][V] or null (then Philox(seed, element, offset))
  unsigned long long seed, offset;
  const float* known; long long known_bs;  // [C][V] of sample 0, sample stride (0 = shared)
  const float* kmask; long long kmask_bs;  // m [V] of sample 0, sample stride (0 = shared)
  unsigned channels;
  float coef, std;                  // alpha, sigma of the label the entry lands on
  const float* known_noise;         // z' [B][C][V] or null (then Philox(seed, element, offset + 2))
};
void launch_solver_entry(const SolverEntryArgs& a, int B, cudaStream_t s);

}  // namespace mdb
