// Bandwidth-bound kernels of the score-network backward pass (what torch autograd runs for the reference's
// loss.backward(), lib/diffusion/losses.py:104-139): GroupNorm(+SiLU, +dropout) backward, bias / time-embedding
// column sums, the data movement of Down/Upsample backward, attention softmax backward and the time-embedding MLP.
// Every reduction is staged (per-thread -> per-block partial -> fixed-order final sum): gradients are bitwise
// reproducible run to run.
// Activation-dtype tensors are bf16 or split bf16 (Precision kBF16 / kBF16X3, act_format.cuh): a row of logical
// pitch ld holds the hi parts of its channels at [0, ld) and their lo parts at [ld, 2 ld). Pointers and pitches passed
// here stay logical; the kernels decode hi + lo, compute in fp32 and store (hi, lo) again.
#pragma once
#include "act_format.cuh"

namespace mdb {

// total block budget of the staged reductions: grid = (ceil(kBwdTargetBlocks / B), B). Partial buffers hold
// kBwdPartRows(B) rows of C (or 2C) floats.
constexpr int kBwdTargetBlocks = 592;
inline int kBwdPartRows(int B) { return kBwdTargetBlocks + B; }

// GroupNorm(32, eps 1e-6) [+SiLU] [+dropout] backward over the channel concatenation of up to two sources.
//   forward:  y = gamma*xhat + beta, a = drop(act(y));   given da = dL/da  [B][V][C] dense
//   pass 1 (reduce): S1[b][c] = sum_v dy, S2[b][c] = sum_v dy*xhat           (dy = da * act'(y) * drop)
//   pass 2 (apply):  dx = rstd*(gamma*dy - mean_g(gamma*dy) - xhat*mean_g(gamma*dy*xhat)) + add0 + add1
//   Pass 1 stores dy over da, so the activation derivative and the dropout hash are evaluated once per element.
struct GnBwdArgs {
  const void* x0; int C0; long long ld0;   // forward input (raw), first source
  const void* x1; int C1; long long ld1;   // second (concatenated) source or null
  const long long* stats0; const long long* stats1;  // forward statistics of the sources ([B][Ci][kStatWords], gn_stats.cuh)
  const float* gamma; const float* beta;
  const void* da;          // [B][V][C] dense, activation dtype; OVERWRITTEN with dy by pass 1 (pass 2 reads dy from it)
  long long voxels; int silu; int groups; float eps;
  // dropout that followed the activation in the forward pass (act_format.cuh: apply_dropout)
  int drop_thresh; float drop_scale; unsigned long long seed;
  // pass 1 output / pass 2 input
  float* part;             // [gx][B][C][2] block partials (scratch)
  float* sums;             // [B][C][2]
  float* dgamma; float* dbeta; int accumulate;  // parameter gradients (+= when accumulate)
  // pass 2
  void* dx;                // [B][V][C] dense
  const void* add0; long long add0_ld;
  const void* add1; long long add1_ld;
  // optional by-product of pass 2: cs_per[b][c] = sum_v dx[b][v][c] (cs_part: [rows][C] block partials)
  float* cs_part; float* cs_per;
  Precision prec;          // of x0 / x1 / da / dx / add0 / add1: kBF16 or kBF16X3
};
void launch_gn_bwd_reduce(const GnBwdArgs& a, int B, cudaStream_t s);  // part -> sums -> dgamma/dbeta
void launch_gn_bwd_apply(const GnBwdArgs& a, int B, cudaStream_t s);

// Fused variant: the data-gradient GEMM that produces `da` applies dy = da*drop*act'(y) in its epilogue (gemm_tc.cuh,
// GNB) and leaves per-tile column partials; pass 1 above is then replaced by these two small kernels.
// consts[b][c] = {0.5*rstd*gamma, 0.5*(beta - mean*rstd*gamma), rstd, -mean*rstd}
void launch_gn_consts(const GnBwdArgs& a, float* consts4, int B, cudaStream_t s);
// sums[b][c][2] = sum over the T tiles of sample b of part[((b/bb*T + t)*bb + b%bb)][c][2]; then dgamma / dbeta
void launch_gnb_tile_reduce(const GnBwdArgs& a, const float* tile_part, int T, int bb, int B, cudaStream_t s);

// colsum: per[b][c] = sum_v t[b][v][c]; total[c] (+)= sum_b per[b][c]. `per` (nullable) is written with row pitch
// per_ld; up to three `total` outputs receive the same values (conv bias + folded shortcut bias, stem biases).
struct ColsumArgs {
  const void* t; long long ld; int C; long long voxels;
  float* part;                // [gx][B][C] scratch
  float* per; long long per_ld;
  float* total0; float* total1; float* total2; int accumulate;
  const float* from_per; long long from_ld;  // per-sample sums already computed by the producing kernel ([B][from_ld])
  Precision prec;             // of t: kBF16 or kBF16X3
};
void launch_colsum(const ColsumArgs& a, int B, cudaStream_t s);

// Downsample backward helper: z[b][2i+1 (each axis)][c] = dy[b][i][c], zero elsewhere (z has twice the extents).
// Moves whole rows, so a split-bf16 tensor is passed as 2C channels.
void launch_zero_stuff2x(const void* dy, void* z, int B, int R, int C, cudaStream_t s);
// Upsample backward: dx[b][i][c] = sum over the 2x2x2 block of d_up (R = extents of dx).
void launch_downsum2x(const void* dup, void* dx, int B, int R, int C, Precision prec, cudaStream_t s);
// out[v][c] = sum_b t[b][v][c]  (VC = voxels x C; split bf16: rows of C channels)
void launch_batch_sum(const void* t, void* out, int B, long long VC, int C, Precision prec, cudaStream_t s);
// out[c] (+)= sum_{b,v} t[b][c][v]  (fp32 NCDHW, e.g. the head bias gradient)
void launch_rowsum_nc(const float* t, float* out, int B, int C, long long V, int accumulate, cudaStream_t s);

// Attention softmax backward, in place: row r holds dP (fp32, L values); P holds the probabilities written by the
// forward softmax (bf16 at the start of rows of L fp32 slots; split bf16: L hi parts followed by L lo parts, filling the slots).
// Writes dS = P*(dP - sum(P*dP)) in the same convention over each dP row.
void launch_softmax_bwd_rows(const float* P, float* dP, long long rows, int L, Precision prec, cudaStream_t s);

// dW[n][k] (+)= sum_b dy[b][n] x[b][k];  db[n] (+)= sum_b dy[b][n]      (fp32, small)
void launch_outer_sum(const float* dy, long long dy_ld, const float* x, long long x_ld, float* dW, float* db, int B, int N, int K,
                      int accumulate, cudaStream_t s);
// dx[b][k] = sum_n dy[b][n] W[n][k]
void launch_dense_bwd_input(const float* dy, long long dy_ld, const float* W, float* dx, int B, int N, int K, cudaStream_t s);
// time-embedding MLP backward (recomputes the forward from labels): given d(act(temb)) [B][4nf] produces
// dt2, h1 [B][4nf] and dt1 [B][4nf], emb [B][nf] for the outer-product weight gradients.
void launch_temb_bwd(const float* labels, const float* w0, const float* b0, const float* w1, const float* b1, const float* dact,
                     float* dt2, float* h1, float* dt1, float* emb, int B, int nf, cudaStream_t s, const int* classes = nullptr,
                     const float* label_w = nullptr);
// gradient of label_embed.weight [K+1][H]: dE[k][n] (+)= sum over b = 0 .. B-1 in order with classes[b] == k of dt2[b][n]
// (one thread per (k, n), no atomics: the same bits on every run)
void launch_label_embed_grad(const int* classes, const float* dt2, float* dE, int B, int K1, int H, int accumulate, cudaStream_t s);

}  // namespace mdb
