// Score-network engine: builds the DDPM 3-D U-Net (reference lib/diffusion/models/ddpm_res64.py:41-199,
// ddpm_res128.py:43-215, layers.py:573-689) as a static plan of wgmma GEMM ops + bandwidth kernels over a
// liveness-packed HBM arena, and replays it per denoising step.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include "gemm_host.h"
#include "wgrad_host.h"
#include "elementwise.cuh"
#include "backward.cuh"

namespace mdb {

struct UNetConfig {
  int image_size = 64;
  int nf = 128;
  int n_levels = 5;
  int ch_mult[8] = {1, 1, 2, 4, 4, 0, 0, 0};
  int num_res_blocks = 3;
  int level0_blocks = -1;  // ddpm_res128.py:98 uses 2 blocks at level 0; -1 = num_res_blocks
  int n_attn = 1;
  int attn_resolutions[4] = {16, 0, 0, 0};
  int num_channels = 4;
  int stem_ksize = 3;   // 3 (res64) or 5 (res128)
  int use_pos_bias = 1; // ddpm_res64.py:148 adds pos_layer(coords*0) == its bias; res128 does not
  int max_batch = 1;
  int precision = 0;    // 0 = bf16 operands, 1 = tf32 operands, 2 = split bf16 (fp32 accumulate in all three)
  int training = 0;     // 1: keep the activations backward needs and build the backward plan (bf16 or split bf16)
  int num_classes = 0;  // K > 0: class-conditional, label_embed.weight [K+1][4nf] (row K = the null class)
};

struct ParamInfo {
  std::string name;
  std::vector<long long> shape;
  long long numel = 0;
  float* d = nullptr;
  bool external = false;  // storage is a slice of a larger buffer
};

class Arena {
 public:
  size_t alloc(size_t bytes);
  void release(size_t off);
  size_t peak() const { return peak_; }
  size_t in_use() const { size_t n = 0; for (auto& b : blocks_) if (!b.free) n += b.size; return n; }
  void reset() { blocks_.clear(); end_ = 0; peak_ = 0; }
 private:
  struct Block { size_t off, size; bool free; };
  std::vector<Block> blocks_;
  size_t end_ = 0, peak_ = 0;
};

// A gradient buffer in the arena, shared by the views handed to the tensors it is the gradient of (the two halves of
// a channel concatenation); returned to the arena when the last view is dropped.
struct GradBuf { size_t off = 0; int refs = 0; bool has_cs = false; size_t cs_off = 0; };
struct GradView {
  std::shared_ptr<GradBuf> buf;
  void* ptr = nullptr;
  long long ld = 0;
  int C = 0;
  float* colsum = nullptr;  // [B][cs_ld] per-sample column sums of this view's channels (left by gn_bwd_apply), or null
  long long cs_ld = 0;
  bool valid() const { return buf != nullptr; }
};

struct Tens {
  size_t off = 0, bytes = 0;
  int C = 0, R = 0;
  long long* stats = nullptr;
  void* ptr = nullptr;
  bool live = true;   // arena block still held
  GradView grad;      // training: dL/d(this), set by the backward of its consumers
};
typedef std::shared_ptr<Tens> TensP;

// Multi-launch composites of the forward plan. The engine and the test entry points (api.cu) both build them here, so a
// test of one runs the engine's construction.
// Sub-pixel Upsample + conv3^3, output-parity class par = px | py << 1 | pz << 2: a 2^3 convolution over the
// low-resolution x ([x.B][r^3][C]) with that class's share of the folded weights w8 (launch_upconv_weights), writing its
// strided sites of out, the high-resolution [x.B][(2r)^3][C] tensor; stats summed over the 8 classes.
void build_upconv_parity(GemmOp& g, Precision prec, const Act& x, void* out, const float* w8, const float* bias,
                         long long* stats, int par);
// AttnBlock core over qkv rows [mb][V][3C] (q | k | v): v^T [mb][C][V] (the K-major B operand of P.v), the fp32 logits
// S = q.k^T / sqrt(C) [mb][V][V], their row softmax in place, O = P.v [mb][V][C].
void launch_attn_vT(Precision prec, const void* qkv, void* vT, int B, int V, int C, cudaStream_t s);
void build_attn_qk(GemmOp& g, Precision prec, int V, int C, int mb, void* qkv, float* S);
void launch_attn_softmax(Precision prec, float* S, int B, int V, cudaStream_t s);
void build_attn_pv(GemmOp& g, Precision prec, int V, int C, int mb, float* S, void* vT, void* O);

class UNet {
 public:
  // The plan is built twice by the same code: a dry pass without the GPU (it sizes the arena; the pointers it records
  // are null) and, unless dry_only, a real pass over the allocated arena that must reproduce the dry pass exactly.
  // A dry_only plan answers every host-side query (parameters, arena, steps, GEMM ops, FLOPs, grad_ready) but cannot run.
  explicit UNet(const UNetConfig& cfg, bool dry_only = false);
  ~UNet();
  const std::vector<ParamInfo>& params() const { return params_; }
  // copies `numel` floats into the named parameter (src on host or device)
  void set_param(const std::string& name, const float* src, long long numel, bool src_device, cudaStream_t s);
  void get_param(const std::string& name, float* dst, long long numel, bool dst_device, cudaStream_t s);
  // after (re)loading parameters: derived vectors, constant stem field, weight packing
  void commit(cudaStream_t s);
  // x: fp32 NCDHW [B][Cin][R^3]; labels: fp32 [B]; out: fp32 NCDHW [B][Cin][R^3]
  // allow_graph: the caller promises that (x, labels, out) are the SAME buffers call after call (the sampler loop): for
  // small batches, where the ~200 launches of a step are launch-latency bound, the whole step is then captured once
  // into a CUDA graph (on a private capture stream) and replayed on `s`
  void forward(const float* x, const float* labels, float* out, int B, cudaStream_t s, bool allow_graph = false);
  // training engines only. Dropout of the next forward()/backward() pair (p = 0 disables; same seed in both).
  void set_dropout(float p, unsigned long long seed);
  // class-conditional engines: the class ids (device int32 [B], each in 0..K; nullptr = the null class K for every sample)
  // of the following forward()/backward() pairs, which must run at batch B. The ids are copied on `s` into a buffer the
  // engine owns and checked there (the copy back to the host synchronises `s`), so the caller's array may be freed as
  // soon as the call returns. Every forward copies the ids in force into a second engine buffer at a fixed address,
  // on its own stream, which is what the captured forward graphs read. K = 0 refuses a non-null pointer.
  void set_classes(const int* classes, int B, cudaStream_t s);
  // the following forwards run the null class (true) or the ids set last (false); mdb_solver_run_guided alternates
  void use_null_class(bool on) { null_forward_ = on; }
  // dout: fp32 NCDHW dL/d(out) of the preceding forward() (same x, labels, B). grads: flat fp32 buffer holding the
  // gradient of every parameter in table order (params()[i] at the sum of the numels before it); entries of
  // non-trainable tensors (mask, coords, pos_layer.weight) are left untouched. accumulate: += instead of =.
  // marks (optional): after `mark_steps[j]` backward launches have been enqueued (ascending), the CUDA event
  // mark_events[j] is recorded on `s` -- the hook a data-parallel host uses to start all-reducing a gradient bucket while
  // the rest of the backward pass still runs (grad_ready_step tells it after which launch a parameter's gradient is final)
  void backward(const float* dout, float* grads, int B, bool accumulate, cudaStream_t s, const int* mark_steps = nullptr,
                void* const* mark_events = nullptr, int n_marks = 0);
  // backward() that also writes dx = dL/dx (fp32 NCDHW, like the forward's x). grads == nullptr: the input gradient only --
  // launches whose only outputs are parameter gradients are skipped, and dx is bitwise the same as with grads
  void backward_input(const float* dout, float* dx, float* grads, int B, bool accumulate, cudaStream_t s);
  int grad_ready_step(const std::string& name) const;
  long long grad_offset(const std::string& name) const;
  long long total_param_numel() const;
  int num_bwd_steps() const { return (int)bwd_steps_.size(); }
  // diagnostics: raw GroupNorm statistics of the last forward ([tensor][B][C][2] int64, 2^-24 fixed point)
  size_t stats_count() const { return stats_doubles_; }
  const long long* stats_ptr() const { return stats_base_; }
  double bwd_flops_per_sample() const { return bwd_flops_ / cfg_.max_batch; }
  std::vector<std::pair<std::string, float>> profile_backward(const float* dout, float* grads, int B, cudaStream_t s);
  double flops_per_sample() const { return flops_ / cfg_.max_batch; }
  size_t arena_bytes() const { return arena_bytes_; }
  int num_gemm_launches() const { return (int)gemms_.size(); }
  const GemmOp& gemm(int i) const { return *gemms_.at(i); }
  int num_steps() const { return (int)steps_.size(); }
  const UNetConfig& cfg() const { return cfg_; }
  // per-GEMM timing breakdown of one forward (ms), for profiling
  std::vector<std::pair<std::string, float>> profile(const float* x, const float* labels, float* out, int B, cudaStream_t s);

 private:
  UNetConfig cfg_;
  Precision prec_;
  bool dry_ = true;
  std::vector<ParamInfo> params_;
  std::map<std::string, int> pindex_;
  std::vector<void*> owned_;  // cudaMalloc'd buffers
  Arena arena_;
  char* arena_base_ = nullptr;
  size_t arena_bytes_ = 0;
  long long* stats_base_ = nullptr;
  size_t stats_doubles_ = 0, stats_cursor_ = 0;
  std::vector<std::unique_ptr<GemmOp>> gemms_;
  std::vector<std::unique_ptr<GemmOp>> commit_gemms_;
  // kind (backward plan): which outputs a launch has, so a pass that does not want them can skip it
  enum StepKind { kAlways = 0, kParamGradOnly = 1, kInputGradOnly = 2 };
  struct Step { std::string name; std::function<void(cudaStream_t, int)> fn; int kind = kAlways; };
  std::vector<Step> steps_, commit_steps_;
  bool committed_ = false;
  double flops_ = 0;
  // CUDA-graph replay of the forward plan (allow_graph): one instantiated graph per (x, labels, out, B)
  struct FwdGraph { const float* x; const float* labels; float* out; int B; int uses; cudaGraphExec_t exec; };
  std::vector<FwdGraph> graphs_;
  cudaStream_t capture_stream_ = nullptr;
  int graph_max_batch_ = 8;
  void drop_graphs();
  // runtime pointers
  const float* rt_x_ = nullptr;
  const float* rt_labels_ = nullptr;
  float* rt_out_ = nullptr;
  // temb
  float* temb_act_ = nullptr;
  float* dense_w_ = nullptr; float* dense_b_ = nullptr; float* dense_out_ = nullptr;
  int dense_total_ = 0, dense_cursor_ = 0;
  // class conditioning: label_embed.weight, the ids the forward reads ([max_batch], fixed address), K repeated
  float* label_w_ = nullptr;
  int* classes_buf_ = nullptr;
  int* null_ids_ = nullptr;
  int* ids_set_ = nullptr;      // copy of the ids given to set_classes
  bool have_ids_ = false, null_forward_ = false;
  int ids_B_ = 0;
  void stage_classes(int B, cudaStream_t s);

  void build();
  void check_runnable() const { if (dry_) throw std::runtime_error("mdb: a dry plan cannot run"); }
  // external: the storage is `slice`, a part of a larger buffer (null in the dry pass), instead of a buffer of its own
  float* P(const std::string& name, std::vector<long long> shape, bool external = false, float* slice = nullptr);
  // the allocation layer is the only code that knows the pass: in the dry pass both return nullptr
  void* dmalloc(size_t bytes, bool zero = true);
  char* at(size_t arena_off) const { return dry_ ? nullptr : arena_base_ + arena_off; }
  TensP new_act(int C, int R, bool stats);
  void release(TensP& t);
  Act act_of(const TensP& t) const;
  GemmOp* new_gemm(const std::string& name, bool commit_time = false);
  void add_step(const std::string& name, std::function<void(cudaStream_t, int)> fn) { steps_.push_back({name, fn}); }
  // finalizes g, uploads it (real pass), and appends its launch (fn, default g->launch(s, B)) to `steps` under its name
  void gemm_step(std::vector<Step>& steps, GemmOp* g, std::function<void(cudaStream_t, int)> fn = {}, int kind = kAlways);
  struct Scratch { int S = 1; size_t off = 0; float* ptr = nullptr; bool active = false; };
  Scratch split_begin(int R, int N, int cin_total, int taps);
  void split_end(Scratch& s);
  TensP gn(const std::string& pname, const std::vector<TensP>& ins, bool silu, int drop_layer = -1);
  // ---- training plan (unet_train.cu)
  bool train_ = false;
  std::vector<std::function<void()>> tape_;  // backward emitters, pushed in forward order, run in reverse
  std::vector<Step> bwd_steps_;
  std::vector<std::unique_ptr<GemmOp>> bwd_gemms_;
  std::vector<std::unique_ptr<WgradOp>> wgrads_;
  double bwd_flops_ = 0;
  std::map<std::string, long long> goff_;
  mutable std::vector<std::string> touched_;  // parameters whose gradient offset the running backward emitter asked for
  std::map<std::string, int> grad_ready_;     // parameter -> number of backward launches after which its gradient is final
  float* rt_grads_ = nullptr; const float* rt_dout_ = nullptr; bool rt_accum_ = false;
  float* rt_dx_ = nullptr;
  bool has_input_grad_ = false;  // the plan carries the stem's data gradient (4 input channels, as the head's shift-sum)
  int rt_drop_thresh_ = 0; float rt_drop_scale_ = 1.f; unsigned long long rt_seed_ = 0;
  float* d_dense_out_ = nullptr;  // [mb][dense_total] gradient of the time-embedding projections
  void add_bwd(const std::string& name, std::function<void(cudaStream_t, int)> fn, int kind = kAlways) {
    bwd_steps_.push_back({name, fn, kind});
  }
  void run_backward(const float* dout, float* grads, float* dx, int B, bool accumulate, cudaStream_t s, const int* mark_steps,
                    void* const* mark_events, int n_marks);
  void free_act(const TensP& t);
  GradView new_grad(int C, int R);
  GradView grad_view(const GradView& g, int c0, int C);
  void unref(GradView& g);
  Act act_of_grad(const GradView& g, int R) const;
  long long G(const std::string& name) const;  // offset of a parameter's gradient in the flat buffer
  struct Tmp { size_t off = 0; void* ptr = nullptr; };
  // GroupNorm backward fused into the epilogue of the data-gradient GEMM that produces dL/d(GroupNorm output):
  // filled in by the caller (which layer), completed by emit_conv_dgrad / emit_pointwise (whether it could be fused)
  struct GnFuse {
    std::string pname; std::vector<TensP> ins; bool silu = false; int drop_layer = -1;
    bool on = false; Tmp consts, part; int T = 0, bb = 1;
  };
  void gn_fuse_attach(GnFuse& f, GemmOp* g, int N, int R);
  Tmp tmp_alloc(size_t bytes);
  void tmp_free(Tmp& t);
  GemmOp* new_bwd_gemm(const std::string& name);
  void emit_colsum(const std::string& name, const GradView& t, int R, float* per, long long per_ld, long long g0, long long g1, long long g2);
  void emit_wgrad(const std::string& name, const Act& dy, const Act& x, int ksize, int stride, long long goff, const WgradOut& layout);
  GradView emit_conv_dgrad(const std::string& name, const GradView& dy, int R, const float* w, int cin_total, const GradView* addend, GnFuse* fuse = nullptr);
  GradView emit_pointwise(const std::string& name, const std::vector<Act>& srcs, const std::vector<WSrc>& ws, int N, int R, const GradView* addend, GnFuse* fuse = nullptr);
  GradView emit_gn_backward(const std::string& pname, const std::vector<TensP>& ins, const GradView& da, bool silu, int drop_layer,
                            const GradView* add0, const GradView* add1, GnFuse* fuse = nullptr);
  void tape_resblock(const std::vector<TensP>& ins, TensP a, TensP h, TensP a2, TensP out, int out_ch, int midx, int doff);
  void tape_attn(TensP x, TensP hn, TensP qkv, TensP S, TensP O, TensP out, int midx);
  void tape_downsample(TensP x, TensP out, int midx);
  void tape_upsample(TensP x, TensP up, TensP out, int midx);
  void tape_stem(TensP h0, void* Am, int Kpad, int Kpad_m);
  void tape_head(TensP h, TensP a, const std::string& gn_name, const std::string& conv_name);
  void tape_temb();
  TensP resblock(const std::vector<TensP>& ins, int out_ch, int midx);
  TensP attn(const TensP& x, int midx);
  TensP downsample(const TensP& x, int midx);
  TensP upsample(const TensP& x, int midx);
};

}  // namespace mdb
