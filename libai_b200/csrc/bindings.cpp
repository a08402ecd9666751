// torch.ops.libai_b200.* : thin argument-checking wrappers around the extern "C" kernel launchers.
// Registered with TORCH_LIBRARY so the in-tree `_C.so` is loaded by torch.ops.load_library (no
// python ABI dependency).
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <cstring>
#include <mutex>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <tuple>

extern "C" {
int lb_gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo, int layout,
                 int epi, const void* bias, int act, void* pre_out, int force_bn, int force_splits, cudaStream_t s);
int lb_gemm_set_schedule(int schedule);
int lb_norm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd, int rows, int H,
                float eps, int rms, int dtype, int wdtype, cudaStream_t s);
int lb_gemm_bf16_bias_residual(const void* x, const void* w, void* out, int M, int N, int K, int lda, int ldb,
                               const void* bias, const void* residual, cudaStream_t s);
int lb_gemm_fp8(const void* xq, const void* wq, void* out, int M, int N, int K, const void* bias, int act, void* pre_out,
                const void* residual, const float* deq_x, const float* deq_w, int force_bn, cudaStream_t s);
int lb_quant_e4m3(const void* x, void* q, void* amax_scratch, float* deq, long n, cudaStream_t s);
int lb_norm_bwd_workspace_rows(int rows);
int lb_norm_bwd_supports_gadd(int H);
int lb_norm_bwd(const void* gy, const void* x, const void* gamma, const float* mean, const float* rstd, void* gx,
                float* dgamma, float* dbeta, float* workspace, int rows, int H, int rms, int dtype, int wdtype,
                int accumulate, const void* gadd, cudaStream_t s);
int lb_bias_act_fwd(const void* x, const void* bias, void* y, long rows, int N, int act, cudaStream_t s);
int lb_gemm_bf16_actgrad(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo,
                         int layout, int act, const void* pre_in, float* colsum, cudaStream_t stream);
int lb_bias_act_bwd(const void* gy, const void* x, const void* bias, void* gx, long rows, int N, int act,
                    cudaStream_t s);
int lb_bias_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N, cudaStream_t s);
int lb_swiglu_fwd(const void* gate, const void* up, void* y, long n, cudaStream_t s);
int lb_swiglu_bwd(const void* gy, const void* gate, const void* up, void* dgate, void* dup, long n, cudaStream_t s);
int lb_swiglu_packed_fwd(const void* gu, void* y, long rows, long F, cudaStream_t s);
int lb_swiglu_packed_bwd(const void* gy, const void* gu, void* dgu, long rows, long F, cudaStream_t s);
int lb_rope_qkv(const void* x, const float* cosv, const float* sinv, void* y, long groups, int S, int G, int r, int D,
                int pos_offset, const int* positions, int npos, int backward, cudaStream_t s);
int lb_rope(const void* x, const float* cosv, const float* sinv, void* y, long rows, int S, int D, int backward,
            cudaStream_t s);
int lb_colsum_workspace_rows(int M, int N);
int lb_colsum(const void* x, float* out, int M, int N, int accumulate, float* workspace, cudaStream_t s);
int lb_embedding_fwd(const int64_t* ids, const void* table, void* out, long T, int H, long vocab_start, long rows, cudaStream_t s);
int lb_embedding_bwd(const int64_t* sorted_ids, const int64_t* order, const void* gy, float* grad, long T, int H,
                     long vocab_start, long rows, cudaStream_t s);
int lb_ce_stats(const void* logits, const int64_t* labels, float* mx, float* se, float* tgt, int T, int V,
                long vocab_start, int dtype, cudaStream_t s);
int lb_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* gloss, void* dlogits, int T,
              int V, long vocab_start, int dtype, cudaStream_t s);
int lb_adamw(float* master, const float* grad, float* m, float* v, void* lp_out, int lp_dtype, const float* scale, long n,
             float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, int decoupled, cudaStream_t s);
int lb_sqnorm_workspace(long n);
int lb_sqnorm(const float* x, float* out, long n, float* workspace, cudaStream_t s);
int lb_gemm_bf16_comm(const void* a, const void* b, void* out, int M, int N, int K, int layout, int epi,
                      const void* bias, int act, void* pre_out, const void* pre_in, float* colsum, int mode,
                      int world, int rank, const long* peer_buf, const long* peer_flags, const long* peer_done,
                      void* state, const void* local_shard, int fill_local, const void* residual, void* rs_out,
                      long staging_parity_off, int n_comm, cudaStream_t stream);
int lb_zero_reduce_scatter(const long* grad_ptrs, const long* flag_ptrs, float* red, float* sqnorm, long lo, long n,
                           float scale, int world, int rank, unsigned epoch, long mc_grad, cudaStream_t s);
int lb_zero_adam_allgather(float* master, const float* red, float* m, float* v, const long* param_ptrs,
                           const long* flag_ptrs, unsigned* done_counter, const float* clip, long lo, long n, float lr,
                           float b1, float b2, float eps, float wd, float bc1, float bc2, int decoupled, int world,
                           int rank, unsigned epoch, long mc_param, cudaStream_t s);
int lb_device_barrier(const long* flag_ptrs, int world, int rank, int slot, unsigned epoch, cudaStream_t s);
int lb_p2p_allgather(const void* shard, const long* out_ptrs, const long* flag_ptrs, unsigned* done_counter,
                     long nbytes, int world, int rank, unsigned epoch, cudaStream_t s);
// mirror of lb::RngArgs (common.cuh)
struct LbRngArgs {
  unsigned long long seed_val, offset_val;
  const long long* seed_ptr;
  const long long* offset_ptr;
  unsigned int offset_intragraph;
  int captured;
  unsigned long long salt;
};
int lb_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int A, int G, int Sq, int Sk,
                int D, const long* q_strides, const long* k_strides, const long* v_strides, int causal, float scale,
                const int* kv_lens, const int* kv_start, const int* doc_start, const void* bias,
                const long* bias_strides, const float* alibi_slopes, float p_drop, const LbRngArgs* rng,
                long long* rng_out, cudaStream_t s);
int lb_attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* o, const float* lse,
                void* dq, void* dk, void* dv, const long* dq_strides, const long* dkv_strides, float* delta,
                float* dq_accum, int B, int A, int G, int Sq, int Sk, int D, const long* q_strides, const long* k_strides,
                const long* v_strides, const long* do_strides, int causal, float scale, const int* kv_lens,
                const int* kv_start, const int* doc_start, const void* bias, const long* bias_strides,
                const float* alibi_slopes, float* dbias, float p_drop, const long long* rng_state, unsigned* dq_order,
                cudaStream_t s);
long lb_attn_bwd_accum_floats(int B, int A, int Sq, int D);
int lb_bias_dropout_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N, float p,
                             const LbRngArgs* rng, const long long* rng_in, long long* rng_out, cudaStream_t s);
int lb_spin_timeout_report(char* buf, int n);
int lb_decode_splits(int B, int blocks, int C, int D);
int lb_decode_attn(const void* q, const long* q_strides, const void* k, const void* v, void* o, float* part_o,
                   float* part_ml, const int* seqlens, const int* kv_start, int B, int Sq, int A, int G, int C, int D,
                   float scale, int nsplit, cudaStream_t s);
int lb_kv_append(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_cache, void* v_cache,
                 const int* seqlens, int B, int Sq, int G, int r, int C, int D, cudaStream_t s);
int lb_window_attn_groups(int B, int H, int W, int ws, int heads);
int lb_window_attn_fwd(const void* qkv, void* out, float* lse, const float* table, const float* tau, int B, int H, int W,
                       int ws, int shift, int heads, int d, float scale, cudaStream_t s);
int lb_window_attn_bwd(const void* dout, const void* qkv, const float* lse, const float* table,
                       const float* tau, void* dqkv, float* dtable, float* dtau, float* dt_part, float* dtau_part, int B,
                       int H, int W, int ws, int shift, int heads, int d, float scale, cudaStream_t s);
}

namespace {

using at::Tensor;

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// description of the device flag wait that timed out and trapped in this process, or "" when none did
std::string spin_timeout_report() {
  char buf[256];
  return std::string(buf, lb_spin_timeout_report(buf, sizeof(buf)));
}

void check(int code, const char* what) {
  if (code == 0) return;
  const std::string timeout = spin_timeout_report();
  TORCH_CHECK(false, "libai_b200 kernel '", what, "' failed with code ", code,
              code > 0 ? std::string(" (") + cudaGetErrorString(static_cast<cudaError_t>(code)) + ")" : std::string(),
              timeout.empty() ? std::string() : "; " + timeout);
}

int dtype_code(const Tensor& t) {
  if (t.scalar_type() == at::kBFloat16) return 0;
  if (t.scalar_type() == at::kFloat) return 1;
  TORCH_CHECK(false, "libai_b200: unsupported dtype ", t.scalar_type());
}

// ---- GEMM -----------------------------------------------------------------------------------------
// layout 0: a[M,K] b[N,K]; 1: a[M,K] b[K,N]; 2: a[K,M] b[K,N].  Returns out (allocated when not given).
Tensor gemm(const Tensor& a, const Tensor& b, int64_t layout, const c10::optional<Tensor>& bias,
            const c10::optional<Tensor>& out_opt, bool accumulate, at::ScalarType out_dtype) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2, "gemm: 2-D CUDA tensors expected");
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm: bf16 operands expected");
  TORCH_CHECK(a.stride(1) == 1 && b.stride(1) == 1, "gemm: operands must be row-major");
  c10::cuda::CUDAGuard guard(a.device());
  int64_t M, N, K;
  if (layout == 0) { M = a.size(0); K = a.size(1); N = b.size(0); TORCH_CHECK(b.size(1) == K, "gemm NT: K mismatch"); }
  else if (layout == 1) { M = a.size(0); K = a.size(1); N = b.size(1); TORCH_CHECK(b.size(0) == K, "gemm NN: K mismatch"); }
  else { K = a.size(0); M = a.size(1); N = b.size(1); TORCH_CHECK(b.size(0) == K, "gemm TN: K mismatch"); }
  Tensor out;
  int epi;
  if (out_opt.has_value()) {
    out = out_opt.value();
    TORCH_CHECK(out.dim() == 2 && out.size(0) == M && out.size(1) == N && out.stride(1) == 1, "gemm: bad out shape");
  } else {
    auto opts = a.options().dtype(out_dtype);
    out = (accumulate || (layout == 2 && out_dtype == at::kFloat)) ? at::zeros({M, N}, opts) : at::empty({M, N}, opts);
  }
  if (out.scalar_type() == at::kBFloat16) {
    TORCH_CHECK(!accumulate, "gemm: accumulate needs an fp32 output");
    epi = 0;
  } else {
    TORCH_CHECK(out.scalar_type() == at::kFloat, "gemm: out must be bf16 or fp32");
    // a freshly zeroed wgrad output takes the accumulating epilogue too; a given `out` is added to only on request
    epi = (accumulate || (layout == 2 && !out_opt.has_value())) ? 2 : 1;
  }
  const void* bias_ptr = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(epi == 0 && bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "gemm: bias must be bf16 [N]");
    bias_ptr = bias->data_ptr();
  }
  check(lb_gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, (int)a.stride(0),
                     (int)b.stride(0), (int)out.stride(0), (int)layout, epi, bias_ptr, 0, nullptr, 0, 0, cur_stream()),
        "gemm");
  return out;
}

// dpre = (gy @ w) * act'(pre): the dgrad GEMM of the layer that consumed act(pre), with the activation backward
// applied in its epilogue (gy [M,N], w [N,K] row-major, pre [M,K]).
// With `bias_grad` (fp32 [N], e.g. the bias' slice of main_grad) the column sums of the result are accumulated into it
// by the GEMM epilogue.
Tensor dgrad_actgrad(const Tensor& gy, const Tensor& w, const Tensor& pre, int64_t act, const c10::optional<Tensor>& bias_grad) {
  TORCH_CHECK(gy.is_cuda() && gy.dim() == 2 && w.dim() == 2 && pre.dim() == 2, "dgrad_actgrad: 2-D CUDA tensors");
  TORCH_CHECK(gy.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && pre.scalar_type() == at::kBFloat16,
              "dgrad_actgrad: bf16 expected");
  TORCH_CHECK(gy.stride(1) == 1 && w.stride(1) == 1 && pre.is_contiguous(), "dgrad_actgrad: row-major operands");
  const int64_t M = gy.size(0), K = gy.size(1), N = w.size(1);
  TORCH_CHECK(w.size(0) == K && pre.size(0) == M && pre.size(1) == N, "dgrad_actgrad: shape mismatch");
  c10::cuda::CUDAGuard guard(gy.device());
  Tensor out = at::empty({M, N}, gy.options());
  float* colsum = nullptr;
  if (bias_grad.has_value() && bias_grad->defined()) {
    TORCH_CHECK(bias_grad->scalar_type() == at::kFloat && bias_grad->is_contiguous() && bias_grad->numel() == N && bias_grad->is_cuda(),
                "dgrad_actgrad: bias_grad must be a contiguous fp32 CUDA tensor [N]");
    colsum = bias_grad->data_ptr<float>();
  }
  check(lb_gemm_bf16_actgrad(gy.data_ptr(), w.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, (int)gy.stride(0),
                             (int)w.stride(0), (int)N, 1, (int)act, pre.data_ptr(), nullptr, cur_stream()),
        "dgrad_actgrad");
  // the bias gradient = column sums of the stored output, in a fixed summation order (the GEMM epilogue's per-tile
  // reductions would arrive in scheduling order)
  if (colsum != nullptr) {
    Tensor ws = at::empty({(int64_t)lb_colsum_workspace_rows((int)M, (int)N) * N}, gy.options().dtype(at::kFloat));
    check(lb_colsum(out.data_ptr(), colsum, (int)M, (int)N, 1, ws.data_ptr<float>(), cur_stream()), "dgrad_actgrad colsum");
  }
  return out;
}

// y = x @ w^T + bias + residual (one kernel)
Tensor linear_bias_residual(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& bias, const Tensor& residual) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "linear_bias_residual: shape mismatch");
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && residual.scalar_type() == at::kBFloat16,
              "linear_bias_residual: bf16 expected");
  TORCH_CHECK(x.stride(1) == 1 && w.stride(1) == 1 && residual.is_contiguous(), "linear_bias_residual: row-major operands");
  const int64_t M = x.size(0), K = x.size(1), N = w.size(0);
  TORCH_CHECK(residual.dim() == 2 && residual.size(0) == M && residual.size(1) == N, "linear_bias_residual: residual must be [M, N]");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({M, N}, x.options());
  const void* bias_ptr = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "linear_bias_residual: bias must be bf16 [N]");
    bias_ptr = bias->data_ptr();
  }
  check(lb_gemm_bf16_bias_residual(x.data_ptr(), w.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, (int)x.stride(0),
                                   (int)w.stride(0), bias_ptr, residual.data_ptr(), cur_stream()),
        "linear_bias_residual");
  return y;
}

// y = act(x @ w^T + bias); optionally also returns the pre-activation (for backward)
std::tuple<Tensor, Tensor> linear_fwd(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& bias, int64_t act,
                                      bool need_pre) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "linear_fwd: shape mismatch");
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16, "linear_fwd: bf16 expected");
  TORCH_CHECK(x.stride(1) == 1 && w.stride(1) == 1, "linear_fwd: row-major operands expected");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), K = x.size(1), N = w.size(0);
  Tensor y = at::empty({M, N}, x.options());
  Tensor pre;
  if (need_pre && act != 0) pre = at::empty({M, N}, x.options());
  const void* bias_ptr = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "linear_fwd: bias must be bf16 [N]");
    bias_ptr = bias->data_ptr();
  }
  check(lb_gemm_bf16(x.data_ptr(), w.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, (int)x.stride(0),
                     (int)w.stride(0), (int)N, 0, 0, bias_ptr, (int)act, pre.defined() ? pre.data_ptr() : nullptr, 0, 0,
                     cur_stream()),
        "linear_fwd");
  return std::make_tuple(y, pre.defined() ? pre : at::empty({0}, x.options()));
}

// per-tensor E4M3 quantisation of a contiguous bf16 tensor: returns (q [same shape, float8_e4m3fn], deq fp32 [1]) with
// x ≈ q * deq (deq = amax / 448); two kernels, no host synchronisation
std::tuple<Tensor, Tensor> quantize_e4m3(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.scalar_type() == at::kBFloat16, "quantize_e4m3: contiguous bf16 CUDA tensor");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = at::empty(x.sizes(), x.options().dtype(at::kFloat8_e4m3fn));
  Tensor scratch = at::zeros({2}, x.options().dtype(at::kFloat));   // [0] = dequantisation scale, [1] = amax bits (zeroed)
  check(lb_quant_e4m3(x.data_ptr(), q.data_ptr(), scratch.data_ptr<float>() + 1, scratch.data_ptr<float>(), (long)x.numel(),
                      cur_stream()),
        "quantize_e4m3");
  return std::make_tuple(q, scratch.narrow(0, 0, 1));
}

// fp8 forward: y = act((xq @ wqᵀ) * deq_x * deq_w + bias) in bf16, optional bf16 pre-activation copy; with a residual
// y = (xq @ wqᵀ) * deq_x * deq_w + bias + residual (no activation, no pre-activation copy).  bn: tile width (0 = the
// heuristic; 64 / 128 / 192 / 256 for tests and tuning)
std::tuple<Tensor, Tensor> linear_fp8_fwd(const Tensor& xq, const Tensor& wq, const Tensor& deq_x, const Tensor& deq_w,
                                          const c10::optional<Tensor>& bias, int64_t act, bool want_pre,
                                          const c10::optional<Tensor>& residual, int64_t bn) {
  TORCH_CHECK(bn == 0 || bn == 64 || bn == 128 || bn == 192 || bn == 256, "linear_fp8_fwd: bn must be 0, 64, 128, 192 or 256");
  const bool has_res = residual.has_value() && residual->defined();
  TORCH_CHECK(!has_res || (act == 0 && !want_pre),
              "linear_fp8_fwd: a residual epilogue takes no activation and no pre-activation copy");
  TORCH_CHECK(xq.is_cuda() && xq.dim() == 2 && wq.dim() == 2 && xq.size(1) == wq.size(1), "linear_fp8_fwd: shape mismatch");
  TORCH_CHECK(xq.scalar_type() == at::kFloat8_e4m3fn && wq.scalar_type() == at::kFloat8_e4m3fn, "linear_fp8_fwd: e4m3 operands");
  TORCH_CHECK(xq.is_contiguous() && wq.is_contiguous(), "linear_fp8_fwd: contiguous operands");
  TORCH_CHECK(deq_x.scalar_type() == at::kFloat && deq_w.scalar_type() == at::kFloat && deq_x.is_cuda() && deq_w.is_cuda(),
              "linear_fp8_fwd: fp32 device scales");
  const int64_t M = xq.size(0), K = xq.size(1), N = wq.size(0);
  TORCH_CHECK(K % 16 == 0 && N % 8 == 0, "linear_fp8_fwd: K % 16 == 0 and N % 8 == 0 required");
  c10::cuda::CUDAGuard guard(xq.device());
  auto opts = xq.options().dtype(at::kBFloat16);
  Tensor y = at::empty({M, N}, opts);
  Tensor pre = want_pre ? at::empty({M, N}, opts) : Tensor();
  const void* bias_ptr = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "linear_fp8_fwd: bias must be bf16 [N]");
    bias_ptr = bias->data_ptr();
  }
  const void* res_ptr = nullptr;
  if (residual.has_value() && residual->defined()) {
    TORCH_CHECK(residual->scalar_type() == at::kBFloat16 && residual->is_contiguous() && residual->numel() == M * N,
                "linear_fp8_fwd: residual must be contiguous bf16 [M, N]");
    res_ptr = residual->data_ptr();
  }
  check(lb_gemm_fp8(xq.data_ptr(), wq.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, bias_ptr, (int)act,
                    pre.defined() ? pre.data_ptr() : nullptr, res_ptr, deq_x.data_ptr<float>(), deq_w.data_ptr<float>(),
                    (int)bn, cur_stream()),
        "linear_fp8_fwd");
  return std::make_tuple(y, pre.defined() ? pre : at::empty({0}, opts));
}

// raw entry used by tests / autotuning: explicit tile-N and split-K
Tensor gemm_tuned(const Tensor& a, const Tensor& b, int64_t layout, int64_t bn, int64_t splits, bool fp32_out) {
  c10::cuda::CUDAGuard guard(a.device());
  int64_t M, N, K;
  if (layout == 0) { M = a.size(0); K = a.size(1); N = b.size(0); }
  else if (layout == 1) { M = a.size(0); K = a.size(1); N = b.size(1); }
  else { K = a.size(0); M = a.size(1); N = b.size(1); }
  const bool atomic = splits != 1;
  Tensor out = atomic ? at::zeros({M, N}, a.options().dtype(at::kFloat))
                      : at::empty({M, N}, a.options().dtype(fp32_out ? at::kFloat : at::kBFloat16));
  const int epi = atomic ? 2 : (fp32_out ? 1 : 0);
  check(lb_gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, (int)a.stride(0),
                     (int)b.stride(0), (int)N, (int)layout, epi, nullptr, 0, nullptr, (int)bn, (int)splits,
                     cur_stream()),
        "gemm_tuned");
  return out;
}

// GEMM schedule of later calls, for comparing the kernels in one process: 0 = automatic (the ping-pong kernel for bf16
// outputs of NT / NN GEMMs with a 128-wide or heuristic tile), 1 = the 288-thread kernel only.  Returns the previous one.
int64_t gemm_schedule(int64_t schedule) {
  TORCH_CHECK(schedule == 0 || schedule == 1, "gemm_schedule: 0 (automatic) or 1 (288-thread kernel only)");
  return lb_gemm_set_schedule((int)schedule);
}

// gx = gy * act'(pre)
Tensor act_bwd(const Tensor& gy, const Tensor& pre, int64_t act) {
  c10::cuda::CUDAGuard guard(gy.device());
  Tensor gx = at::empty_like(gy);
  check(lb_bias_act_bwd(gy.data_ptr(), pre.data_ptr(), nullptr, gx.data_ptr(), gy.size(0), (int)gy.size(1), (int)act,
                        cur_stream()),
        "act_bwd");
  return gx;
}

// column sums of a bf16 [M, N] tensor.  With `accum` (fp32 [N], e.g. a bias' slice of the flat main-grad buffer) the
// sums are added into it and an empty tensor is returned; otherwise a fresh bf16 [N] tensor.
// embedding lookup on a (vocabulary shard of a) bf16 table; ids int64 (any shape) -> [ids.numel(), H]
Tensor embedding_fwd(const Tensor& ids, const Tensor& table, int64_t vocab_start) {
  c10::cuda::CUDAGuard guard(table.device());
  TORCH_CHECK(ids.scalar_type() == at::kLong && ids.is_contiguous() && ids.is_cuda(), "embedding_fwd: contiguous int64 CUDA ids");
  TORCH_CHECK(table.dim() == 2 && table.is_contiguous() && table.scalar_type() == at::kBFloat16, "embedding_fwd: contiguous bf16 table");
  const int64_t T = ids.numel(), H = table.size(1);
  Tensor out = at::empty({T, H}, table.options());
  check(lb_embedding_fwd(ids.data_ptr<int64_t>(), table.data_ptr(), out.data_ptr(), (long)T, (int)H, (long)vocab_start,
                         (long)table.size(0), cur_stream()),
        "embedding_fwd");
  return out;
}
// grad[ids - vocab_start] += gy   (grad: the parameter's fp32 main-grad view, same shape as the table)
void embedding_bwd(const Tensor& ids, const Tensor& gy, Tensor grad, int64_t vocab_start) {
  c10::cuda::CUDAGuard guard(gy.device());
  TORCH_CHECK(ids.scalar_type() == at::kLong && ids.is_contiguous(), "embedding_bwd: contiguous int64 ids");
  TORCH_CHECK(gy.is_cuda() && ids.device() == gy.device() && grad.device() == gy.device(),
              "embedding_bwd: ids, gy and grad must be on one CUDA device");
  TORCH_CHECK(gy.dim() == 2 && gy.is_contiguous() && gy.scalar_type() == at::kBFloat16 && gy.size(0) == ids.numel(),
              "embedding_bwd: gy must be contiguous bf16 [ids.numel(), H]");
  TORCH_CHECK(grad.dim() == 2 && grad.is_contiguous() && grad.scalar_type() == at::kFloat && grad.size(1) == gy.size(1),
              "embedding_bwd: grad must be contiguous fp32 [rows, H]");
  const auto sorted = at::sort(ids.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
  check(lb_embedding_bwd(std::get<0>(sorted).data_ptr<int64_t>(), std::get<1>(sorted).data_ptr<int64_t>(), gy.data_ptr(),
                         grad.data_ptr<float>(), (long)ids.numel(), (int)gy.size(1), (long)vocab_start, (long)grad.size(0),
                         cur_stream()),
        "embedding_bwd");
}

Tensor colsum(const Tensor& x, const c10::optional<Tensor>& accum) {
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.dim() == 2 && x.is_contiguous() && x.scalar_type() == at::kBFloat16, "colsum: contiguous bf16 [M,N]");
  if (accum.has_value() && accum->defined()) {
    TORCH_CHECK(accum->scalar_type() == at::kFloat && accum->numel() == x.size(1) && accum->is_contiguous(),
                "colsum: accum must be contiguous fp32 [N]");
    Tensor ws = at::empty({(int64_t)lb_colsum_workspace_rows((int)x.size(0), (int)x.size(1)) * x.size(1)},
                          x.options().dtype(at::kFloat));
    check(lb_colsum(x.data_ptr(), accum->data_ptr<float>(), (int)x.size(0), (int)x.size(1), 1, ws.data_ptr<float>(),
                    cur_stream()),
          "colsum");
    return at::empty({0}, x.options());
  }
  Tensor out = at::empty({x.size(1)}, x.options().dtype(at::kFloat));
  Tensor ws = at::empty({(int64_t)lb_colsum_workspace_rows((int)x.size(0), (int)x.size(1)) * x.size(1)},
                        x.options().dtype(at::kFloat));
  check(lb_colsum(x.data_ptr(), out.data_ptr<float>(), (int)x.size(0), (int)x.size(1), 0, ws.data_ptr<float>(), cur_stream()),
        "colsum");
  return out.to(at::kBFloat16);
}

// ---- norms ----------------------------------------------------------------------------------------
// The kernels read H elements of γ (and β) with no bounds of their own and are built for the (x, γ) dtype pairs
// (bf16, bf16), (bf16, fp32) and (fp32, fp32).
void check_norm_params(const char* what, const Tensor& x, const Tensor& gamma, const Tensor* beta) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous(), what, ": x must be a contiguous CUDA tensor [rows, H]");
  const bool pair_ok = (x.scalar_type() == at::kBFloat16 &&
                        (gamma.scalar_type() == at::kBFloat16 || gamma.scalar_type() == at::kFloat)) ||
                       (x.scalar_type() == at::kFloat && gamma.scalar_type() == at::kFloat);
  TORCH_CHECK(pair_ok, what, ": unsupported dtypes x ", x.scalar_type(), " with gamma ", gamma.scalar_type(),
              " (supported: bf16/bf16, bf16/fp32, fp32/fp32)");
  TORCH_CHECK(gamma.is_contiguous() && gamma.numel() == x.size(1) && gamma.device() == x.device(), what,
              ": gamma must be contiguous with H = ", x.size(1), " elements on x's device");
  if (beta != nullptr) {
    TORCH_CHECK(beta->scalar_type() == gamma.scalar_type(), what, ": beta must have gamma's dtype");
    TORCH_CHECK(beta->is_contiguous() && beta->numel() == x.size(1) && beta->device() == x.device(), what,
                ": beta must be contiguous with H = ", x.size(1), " elements on x's device");
  }
}

std::tuple<Tensor, Tensor, Tensor> norm_fwd(const Tensor& x, const Tensor& gamma, const c10::optional<Tensor>& beta,
                                            double eps, bool rms) {
  c10::cuda::CUDAGuard guard(x.device());
  const bool has_beta = beta.has_value() && beta->defined();
  check_norm_params("norm_fwd", x, gamma, has_beta ? &beta.value() : nullptr);
  const int rows = (int)x.size(0), H = (int)x.size(1);
  Tensor y = at::empty_like(x);
  Tensor mean = rms ? at::empty({0}, x.options().dtype(at::kFloat)) : at::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = at::empty({rows}, x.options().dtype(at::kFloat));
  const void* b = has_beta ? beta->data_ptr() : nullptr;
  check(lb_norm_fwd(x.data_ptr(), gamma.data_ptr(), b, y.data_ptr(), rms ? nullptr : mean.data_ptr<float>(),
                    rstd.data_ptr<float>(), rows, H, (float)eps, rms ? 1 : 0, dtype_code(x), dtype_code(gamma),
                    cur_stream()),
        "norm_fwd");
  return std::make_tuple(y, mean, rstd);
}

std::tuple<Tensor, Tensor, Tensor> norm_bwd(const Tensor& gy, const Tensor& x, const Tensor& gamma, const Tensor& mean,
                                            const Tensor& rstd, bool rms, bool has_bias,
                                            const c10::optional<Tensor>& dgamma_accum,
                                            const c10::optional<Tensor>& dbeta_accum,
                                            const c10::optional<Tensor>& gadd) {
  c10::cuda::CUDAGuard guard(x.device());
  check_norm_params("norm_bwd", x, gamma, nullptr);
  TORCH_CHECK(gy.sizes() == x.sizes() && gy.scalar_type() == x.scalar_type() && gy.is_contiguous() &&
                  gy.device() == x.device(),
              "norm_bwd: gy must be contiguous with x's shape, dtype and device");
  const int rows = (int)x.size(0), H = (int)x.size(1);
  TORCH_CHECK(rstd.numel() == rows && (rms || mean.numel() == rows), "norm_bwd: mean / rstd must hold one value per row");
  Tensor gx = at::empty_like(x);
  auto fopt = x.options().dtype(at::kFloat);
  // accumulate mode: dgamma / dbeta are added straight into the fp32 main-grad slices of the parameters
  const bool acc = dgamma_accum.has_value() && dgamma_accum->defined();
  if (acc) {
    TORCH_CHECK(dgamma_accum->scalar_type() == at::kFloat && dgamma_accum->numel() == H && dgamma_accum->is_contiguous(),
                "norm_bwd: dgamma_accum must be contiguous fp32 [H]");
    TORCH_CHECK(!has_bias || (dbeta_accum.has_value() && dbeta_accum->defined() &&
                              dbeta_accum->scalar_type() == at::kFloat && dbeta_accum->numel() == H &&
                              dbeta_accum->is_contiguous()),
                "norm_bwd: dbeta_accum must be contiguous fp32 [H]");
  }
  Tensor dgamma = acc ? dgamma_accum.value() : at::empty({H}, fopt);
  Tensor dbeta = !has_bias ? at::empty({0}, fopt) : (acc ? dbeta_accum.value() : at::empty({H}, fopt));
  const int wrows = lb_norm_bwd_workspace_rows(rows);
  Tensor ws = at::empty({2 * (int64_t)wrows * H}, fopt);
  // optional gradient of the skip connection around this norm: added to gx inside the kernel when supported
  const bool has_add = gadd.has_value() && gadd->defined();
  const bool fuse_add = has_add && lb_norm_bwd_supports_gadd(H) && gadd->is_contiguous() && gadd->scalar_type() == x.scalar_type();
  check(lb_norm_bwd(gy.data_ptr(), x.data_ptr(), gamma.data_ptr(), rms ? nullptr : mean.data_ptr<float>(),
                    rstd.data_ptr<float>(), gx.data_ptr(), dgamma.data_ptr<float>(),
                    has_bias ? dbeta.data_ptr<float>() : nullptr, ws.data_ptr<float>(), rows, H, rms ? 1 : 0,
                    dtype_code(x), dtype_code(gamma), acc ? 1 : 0, fuse_add ? gadd->data_ptr() : nullptr, cur_stream()),
        "norm_bwd");
  if (has_add && !fuse_add) gx.add_(gadd->to(gx.scalar_type()));
  if (acc) return std::make_tuple(gx, at::empty({0}, fopt), at::empty({0}, fopt));
  return std::make_tuple(gx, dgamma, dbeta);
}

// ---- elementwise ------------------------------------------------------------------------------------
Tensor bias_act_fwd(const Tensor& x, const c10::optional<Tensor>& bias, int64_t act) {
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty_like(x);
  const void* b = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  check(lb_bias_act_fwd(x.data_ptr(), b, y.data_ptr(), x.size(0), (int)x.size(1), (int)act, cur_stream()), "bias_act_fwd");
  return y;
}
Tensor bias_act_bwd(const Tensor& gy, const Tensor& x, const c10::optional<Tensor>& bias, int64_t act) {
  c10::cuda::CUDAGuard guard(x.device());
  Tensor gx = at::empty_like(x);
  const void* b = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  check(lb_bias_act_bwd(gy.data_ptr(), x.data_ptr(), b, gx.data_ptr(), x.size(0), (int)x.size(1), (int)act, cur_stream()),
        "bias_act_bwd");
  return gx;
}
Tensor bias_residual_fwd(const Tensor& x, const c10::optional<Tensor>& bias, const c10::optional<Tensor>& res) {
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty_like(x);
  const void* b = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  const void* r = (res.has_value() && res->defined()) ? res->data_ptr() : nullptr;
  check(lb_bias_residual(x.data_ptr(), b, r, y.data_ptr(), x.size(0), (int)x.size(1), cur_stream()), "bias_residual");
  return y;
}
Tensor swiglu_fwd(const Tensor& gate, const Tensor& up) {
  c10::cuda::CUDAGuard guard(gate.device());
  Tensor y = at::empty_like(gate);
  check(lb_swiglu_fwd(gate.data_ptr(), up.data_ptr(), y.data_ptr(), gate.numel(), cur_stream()), "swiglu_fwd");
  return y;
}
std::tuple<Tensor, Tensor> swiglu_bwd(const Tensor& gy, const Tensor& gate, const Tensor& up) {
  c10::cuda::CUDAGuard guard(gate.device());
  Tensor dg = at::empty_like(gate), du = at::empty_like(up);
  check(lb_swiglu_bwd(gy.data_ptr(), gate.data_ptr(), up.data_ptr(), dg.data_ptr(), du.data_ptr(), gate.numel(),
                      cur_stream()),
        "swiglu_bwd");
  return std::make_tuple(dg, du);
}
// gu [T, 2F] = [gate | up] (one GEMM against the stacked gate / up weights) -> silu(gate) * up  [T, F]
Tensor swiglu_packed_fwd(const Tensor& gu) {
  c10::cuda::CUDAGuard guard(gu.device());
  TORCH_CHECK(gu.dim() == 2 && gu.is_contiguous() && gu.scalar_type() == at::kBFloat16 && gu.size(1) % 16 == 0,
              "swiglu_packed_fwd: contiguous bf16 [T, 2F] with F % 8 == 0");
  Tensor y = at::empty({gu.size(0), gu.size(1) / 2}, gu.options());
  check(lb_swiglu_packed_fwd(gu.data_ptr(), y.data_ptr(), gu.size(0), gu.size(1) / 2, cur_stream()), "swiglu_packed_fwd");
  return y;
}
Tensor swiglu_packed_bwd(const Tensor& gy, const Tensor& gu) {
  c10::cuda::CUDAGuard guard(gu.device());
  TORCH_CHECK(gy.is_contiguous() && gu.is_contiguous() && gy.dim() == 2 && gu.size(1) == 2 * gy.size(1) &&
                  gy.scalar_type() == at::kBFloat16, "swiglu_packed_bwd: gy [T, F], gu [T, 2F] contiguous bf16");
  Tensor dgu = at::empty_like(gu);
  check(lb_swiglu_packed_bwd(gy.data_ptr(), gu.data_ptr(), dgu.data_ptr(), gu.size(0), gy.size(1), cur_stream()),
        "swiglu_packed_bwd");
  return dgu;
}
// Geometry of a packed projection: [b, s, a, 3d] (per-head [q|k|v], G = a, r = 1) or the grouped [b, s, g, r + 2, d]
// (per K/V group q_0 .. q_{r-1}, k, v).
struct PackedQKV {
  int B, S, G, r, D;
};
PackedQKV packed_qkv(const Tensor& qkv, const char* what) {
  TORCH_CHECK(qkv.dim() == 4 || qkv.dim() == 5, what, ": packed projection [b, s, a, 3d] or [b, s, g, r + 2, d] expected");
  PackedQKV g;
  g.B = (int)qkv.size(0);
  g.S = (int)qkv.size(1);
  g.G = (int)qkv.size(2);
  if (qkv.dim() == 4) {
    g.r = 1;
    g.D = (int)qkv.size(3) / 3;
    TORCH_CHECK(qkv.size(3) == 3 * g.D, what, ": last dim must be 3*d");
  } else {
    g.r = (int)qkv.size(3) - 2;
    g.D = (int)qkv.size(4);
    TORCH_CHECK(g.r >= 1, what, ": a group holds r >= 1 query heads, k and v");
  }
  return g;
}

// per-token int32 [B, S] tensor of a packed batch (rope positions, attention doc_start) → device pointer or nullptr
const int* token_index(const c10::optional<Tensor>& t, const Tensor& like, int B, int S, const char* what) {
  if (!(t.has_value() && t->defined())) return nullptr;
  TORCH_CHECK(t->scalar_type() == at::kInt, what, ": int32 expected, got ", t->scalar_type());
  TORCH_CHECK(t->dim() == 2 && t->size(0) == B && t->size(1) == S, what, ": [", B, ", ", S, "] expected, got shape ",
              t->sizes());
  TORCH_CHECK(t->is_cuda() && t->device() == like.device(), what, ": must be on ", like.device(), ", got ", t->device());
  TORCH_CHECK(t->is_contiguous(), what, ": must be contiguous");
  return t->data_ptr<int>();
}

// packed projection [b, s, a, 3d] or [b, s, g, r + 2, d]; rotates every q and k (v copied).  inplace=true rewrites qkv
// itself.  positions (optional, int32 [b, s]): the position of every token (packed sequences), instead of
// s + pos_offset; values outside the tables are clamped to them.
Tensor rope_qkv(const Tensor& qkv, const Tensor& cosv, const Tensor& sinv, int64_t pos_offset, bool backward,
                bool inplace, const c10::optional<Tensor>& positions) {
  c10::cuda::CUDAGuard guard(qkv.device());
  TORCH_CHECK(qkv.is_contiguous() && qkv.scalar_type() == at::kBFloat16, "rope_qkv: contiguous bf16 packed projection");
  const PackedQKV g = packed_qkv(qkv, "rope_qkv");
  const int S = g.S, D = g.D;
  TORCH_CHECK(D % 2 == 0, "rope_qkv: head dim must be even");
  const int* pos = token_index(positions, qkv, g.B, S, "rope_qkv: positions");
  TORCH_CHECK(cosv.scalar_type() == at::kFloat && sinv.scalar_type() == at::kFloat && cosv.is_contiguous() &&
                  sinv.is_contiguous() && cosv.size(0) >= (pos != nullptr ? 1 : S + pos_offset) && cosv.size(1) == D &&
                  sinv.sizes() == cosv.sizes(),
              "rope_qkv: cos/sin fp32 [>=S+offset, D]");
  TORCH_CHECK(cosv.device() == qkv.device() && sinv.device() == qkv.device(), "rope_qkv: cos/sin must be on qkv's device");
  Tensor y = inplace ? qkv : at::empty_like(qkv);
  check(lb_rope_qkv(qkv.data_ptr(), cosv.data_ptr<float>(), sinv.data_ptr<float>(), y.data_ptr(),
                    qkv.numel() / ((g.r + 2) * D), S, g.G, g.r, D, (int)pos_offset, pos, (int)cosv.size(0),
                    backward ? 1 : 0, cur_stream()),
        "rope_qkv");
  return y;
}

Tensor rope(const Tensor& x, const Tensor& cosv, const Tensor& sinv, bool backward) {
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.dim() == 4 && x.is_contiguous() && x.scalar_type() == at::kBFloat16, "rope: contiguous bf16 [b,a,s,d]");
  const int S = (int)x.size(2), D = (int)x.size(3);
  TORCH_CHECK(cosv.scalar_type() == at::kFloat && sinv.scalar_type() == at::kFloat && cosv.is_contiguous() &&
                  sinv.is_contiguous() && cosv.dim() == 2 && cosv.size(0) >= S && cosv.size(1) == D &&
                  sinv.sizes() == cosv.sizes(),
              "rope: cos/sin fp32 contiguous [>=S, D] of one shape");
  TORCH_CHECK(cosv.device() == x.device() && sinv.device() == x.device(), "rope: cos/sin must be on x's device");
  Tensor y = at::empty_like(x);
  check(lb_rope(x.data_ptr(), cosv.data_ptr<float>(), sinv.data_ptr<float>(), y.data_ptr(), x.numel() / D, S, D,
                backward ? 1 : 0, cur_stream()),
        "rope");
  return y;
}

// ---- cross entropy ------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor> ce_stats(const Tensor& logits, const Tensor& labels, int64_t vocab_start) {
  c10::cuda::CUDAGuard guard(logits.device());
  TORCH_CHECK(logits.dim() == 2 && logits.is_contiguous() && labels.scalar_type() == at::kLong, "ce_stats: bad args");
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  auto fopt = logits.options().dtype(at::kFloat);
  Tensor mx = at::empty({T}, fopt), se = at::empty({T}, fopt), tgt = at::empty({T}, fopt);
  check(lb_ce_stats(logits.data_ptr(), labels.data_ptr<int64_t>(), mx.data_ptr<float>(), se.data_ptr<float>(),
                    tgt.data_ptr<float>(), T, V, (long)vocab_start, dtype_code(logits), cur_stream()),
        "ce_stats");
  return std::make_tuple(mx, se, tgt);
}
Tensor ce_bwd(const Tensor& logits, const Tensor& labels, const Tensor& lse, const Tensor& gloss, int64_t vocab_start) {
  c10::cuda::CUDAGuard guard(logits.device());
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  // in place: the saved logits buffer becomes dlogits (no second [T, V] allocation)
  Tensor d = logits;
  check(lb_ce_bwd(logits.data_ptr(), labels.data_ptr<int64_t>(), lse.data_ptr<float>(), gloss.data_ptr<float>(),
                  d.data_ptr(), T, V, (long)vocab_start, dtype_code(logits), cur_stream()),
        "ce_bwd");
  return d;
}

// ---- optimizer ------------------------------------------------------------------------------------------
void fused_adamw(Tensor master, const Tensor& grad, Tensor m, Tensor v, const c10::optional<Tensor>& lp_out,
                 const Tensor& scale, double lr, double b1, double b2, double eps, double wd, double bc1, double bc2,
                 bool decoupled) {
  // float4 loads and stores over master.numel() elements of every buffer
  const auto dev = master.device();
  for (const Tensor* t : {static_cast<const Tensor*>(&master), &grad, static_cast<const Tensor*>(&m),
                          static_cast<const Tensor*>(&v)}) {
    TORCH_CHECK(t->is_cuda() && t->device() == dev && t->scalar_type() == at::kFloat && t->is_contiguous() &&
                    t->numel() == master.numel(),
                "fused_adamw: master, grad, m and v must be contiguous fp32 tensors of one size on one CUDA device");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "fused_adamw: buffers must be 16-byte aligned");
  }
  TORCH_CHECK(master.numel() % 4 == 0, "fused_adamw: numel must be a multiple of 4");
  TORCH_CHECK(scale.is_cuda() && scale.device() == dev && scale.scalar_type() == at::kFloat && scale.numel() == 1,
              "fused_adamw: scale must be a one-element fp32 tensor on the buffers' device");
  void* lp = nullptr;
  int lp_dtype = 0;
  if (lp_out.has_value() && lp_out->defined()) {
    TORCH_CHECK(lp_out->scalar_type() == at::kBFloat16 || lp_out->scalar_type() == at::kHalf,
                "fused_adamw: lp_out must be bf16 or fp16");
    TORCH_CHECK(lp_out->is_cuda() && lp_out->device() == dev && lp_out->is_contiguous() &&
                    lp_out->numel() == master.numel() && reinterpret_cast<uintptr_t>(lp_out->data_ptr()) % 8 == 0,
                "fused_adamw: lp_out must be contiguous, 8-byte aligned, of master's size and on its device");
    lp = lp_out->data_ptr();
    lp_dtype = lp_out->scalar_type() == at::kHalf ? 1 : 0;
  }
  c10::cuda::CUDAGuard guard(dev);
  check(lb_adamw(master.data_ptr<float>(), grad.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), lp, lp_dtype,
                 scale.data_ptr<float>(), master.numel(), (float)lr, (float)b1, (float)b2, (float)eps, (float)wd,
                 (float)bc1, (float)bc2, decoupled ? 1 : 0, cur_stream()),
        "fused_adamw");
}
Tensor sqnorm(const Tensor& x) {
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::zeros({1}, x.options().dtype(at::kFloat));
  Tensor ws = at::empty({(int64_t)lb_sqnorm_workspace(x.numel())}, x.options().dtype(at::kFloat));
  check(lb_sqnorm(x.data_ptr<float>(), out.data_ptr<float>(), x.numel(), ws.data_ptr<float>(), cur_stream()), "sqnorm");
  return out;
}

// ---- dropout RNG ---------------------------------------------------------------------------------------------
// (seed, offset) of the default CUDA generator, advanced by `increment`; graph-capture aware (pointers + intra-graph
// offset while capturing — PyTorch refreshes the pointed-to values before every replay).  `salt` != 0 decorrelates
// tensor-parallel ranks in sharded regions.
LbRngArgs next_rng(int64_t salt, uint64_t increment = 4) {
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(c10::nullopt, at::cuda::detail::getDefaultCUDAGenerator());
  at::PhiloxCudaState st;
  {
    std::lock_guard<std::mutex> lock(gen->mutex_);
    st = gen->philox_cuda_state(increment);
  }
  LbRngArgs a;
  std::memset(&a, 0, sizeof(a));
  a.captured = st.captured_ ? 1 : 0;
  if (st.captured_) {
    a.seed_ptr = reinterpret_cast<const long long*>(st.seed_.ptr);
    a.offset_ptr = reinterpret_cast<const long long*>(st.offset_.ptr);
    a.offset_intragraph = st.offset_intragraph_;
  } else {
    a.seed_val = st.seed_.val;
    a.offset_val = st.offset_.val;
  }
  a.salt = static_cast<unsigned long long>(salt);
  return a;
}

// y = residual + dropout(x + bias, p); returns (y, rng_state int64[2]) — the backward is the same op on the output
// gradient with `rng_state` passed back in (bias = residual = None)
std::tuple<Tensor, Tensor> bias_dropout_residual(const Tensor& x, const c10::optional<Tensor>& bias,
                                                 const c10::optional<Tensor>& res, double p, int64_t salt,
                                                 const c10::optional<Tensor>& rng_state) {
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.is_contiguous() && x.dim() == 2, "bias_dropout_residual: bf16 contiguous 2-D");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "dropout probability must be in [0, 1)");
  Tensor y = at::empty_like(x);
  const void* bptr = (bias.has_value() && bias->defined()) ? bias->data_ptr() : nullptr;
  const void* rptr = (res.has_value() && res->defined()) ? res->data_ptr() : nullptr;
  if (rng_state.has_value() && rng_state->defined()) {
    check(lb_bias_dropout_residual(x.data_ptr(), bptr, rptr, y.data_ptr(), x.size(0), (int)x.size(1), (float)p, nullptr,
                                   reinterpret_cast<const long long*>(rng_state->data_ptr<int64_t>()), nullptr, cur_stream()),
          "bias_dropout_residual");
    return std::make_tuple(y, *rng_state);
  }
  Tensor st = at::empty({2}, x.options().dtype(at::kLong));
  LbRngArgs a = next_rng(salt);
  check(lb_bias_dropout_residual(x.data_ptr(), bptr, rptr, y.data_ptr(), x.size(0), (int)x.size(1), (float)p, &a, nullptr,
                                 reinterpret_cast<long long*>(st.data_ptr<int64_t>()), cur_stream()),
        "bias_dropout_residual");
  return std::make_tuple(y, st);
}

// ---- attention ----------------------------------------------------------------------------------------------
// q: [B, A, Sq, D] or, grouped, [B, G, r, Sq, D]; k, v: [B, G, Sk, D] with A = G * r (grouped-query attention: query
// head h reads K/V head h / r) and head dim D a multiple of 8 in [8, 128]; views with arbitrary batch/head/seq strides
// (D contiguous).  Output o is allocated as [B, Sq, A, D] and returned as the [B, A, Sq, D] view, lse fp32 [B, A, Sq].
// Key j is visible to query i of sample b iff kv_start[b] <= j < kv_lens[b] (defaults 0 and Sk) and, when causal,
// j <= i + Sk - Sq.
struct BiasDesc {
  const void* ptr = nullptr;
  long strides[3] = {0, 0, 0};
};
// bias [Bb, Ab, Sq, Sk] (Bb in {1, B}, Ab in {1, A}), bf16, key dimension contiguous; broadcast dims get stride 0
BiasDesc bias_desc(const c10::optional<Tensor>& bias, int B, int A, int Sq, int Sk) {
  BiasDesc d;
  if (!(bias.has_value() && bias->defined())) return d;
  const Tensor& b = *bias;
  TORCH_CHECK(b.dim() == 4 && b.scalar_type() == at::kBFloat16 && b.stride(3) == 1 && b.size(2) == Sq && b.size(3) == Sk,
              "attention bias: bf16 [B|1, A|1, Sq, Sk] with contiguous keys");
  TORCH_CHECK((b.size(0) == 1 || b.size(0) == B) && (b.size(1) == 1 || b.size(1) == A), "attention bias: bad broadcast shape");
  d.ptr = b.data_ptr();
  d.strides[0] = b.size(0) == 1 ? 0 : b.stride(0);
  d.strides[1] = b.size(1) == 1 ? 0 : b.stride(1);
  d.strides[2] = b.stride(2);
  return d;
}

// shapes of an attention call: q [B, A, Sq, D] / [B, G, r, Sq, D] against k, v [B, G, Sk, D]; qs = q's {batch, group,
// in-group, seq} strides
struct QGeom {
  int B, A, G, Sq, Sk, D;
  long qs[4];
};
QGeom q_geom(const Tensor& q, const Tensor& k, const Tensor& v, const char* what) {
  TORCH_CHECK(q.dim() == 4 || q.dim() == 5, what, ": q must be [B, A, S, D] or [B, G, r, S, D]");
  TORCH_CHECK(k.dim() == 4 && k.sizes() == v.sizes(), what, ": k, v must be [B, G, S, D] of one shape");
  TORCH_CHECK(q.stride(-1) == 1 && k.stride(3) == 1 && v.stride(3) == 1, what, ": D must be contiguous");
  QGeom g;
  g.B = (int)q.size(0);
  g.G = (int)k.size(1);
  g.Sq = (int)q.size(-2);
  g.Sk = (int)k.size(2);
  g.D = (int)q.size(-1);
  if (q.dim() == 4) {
    g.A = (int)q.size(1);
    TORCH_CHECK(g.G > 0 && g.A % g.G == 0, what, ": the query heads must be a multiple of the K/V heads");
    const long r = g.A / g.G;
    g.qs[0] = q.stride(0);
    g.qs[1] = r * q.stride(1);
    g.qs[2] = q.stride(1);
    g.qs[3] = q.stride(2);
  } else {
    TORCH_CHECK(q.size(1) == g.G, what, ": grouped q [B, G, r, S, D] must have the K/V heads' G");
    g.A = g.G * (int)q.size(2);
    g.qs[0] = q.stride(0);
    g.qs[1] = q.stride(1);
    g.qs[2] = q.stride(2);
    g.qs[3] = q.stride(3);
  }
  TORCH_CHECK(k.size(0) == g.B && k.size(3) == g.D, what, ": k, v do not match q");
  TORCH_CHECK(g.D % 8 == 0 && g.D >= 8 && g.D <= 128, what, ": head dim must be a multiple of 8 in [8, 128], got ", g.D);
  TORCH_CHECK(g.Sq >= 1 && g.Sk >= 1, what, ": empty query or key sequence");
  return g;
}

// optional per-sample key bound (kv_lens: end, kv_start: start of the visible keys) → device pointer or nullptr
const int* key_bound(const c10::optional<Tensor>& t, const Tensor& q, int B, const char* what) {
  if (!(t.has_value() && t->defined())) return nullptr;
  TORCH_CHECK(t->scalar_type() == at::kInt, what, ": int32 expected, got ", t->scalar_type());
  TORCH_CHECK(t->numel() == B, what, ": ", B, " elements (one per sample) expected, got shape ", t->sizes());
  TORCH_CHECK(t->is_cuda() && t->device() == q.device(), what, ": must be on ", q.device(), ", got ", t->device());
  TORCH_CHECK(t->is_contiguous(), what, ": must be contiguous");
  return t->data_ptr<int>();
}

// doc_start (optional, int32 [B, S]): packed sequences, query i sees keys doc_start[b, i] <= j <= i (clamped to [0, i])
const int* doc_starts(const c10::optional<Tensor>& doc_start, const Tensor& q, const QGeom& g, bool causal,
                      bool other_masks, double p_drop, const char* what) {
  const int* ds = token_index(doc_start, q, g.B, g.Sq, what);
  TORCH_CHECK(ds == nullptr || (causal && g.Sq == g.Sk && !other_masks && p_drop == 0.0), what,
              ": supported for causal self-attention (Sq == Sk) without kv_lens, kv_start, bias, ALiBi or dropout");
  return ds;
}

// returns (o, lse, rng_state): rng_state int64[2] = (seed, offset) of the dropout mask (empty without dropout)
std::tuple<Tensor, Tensor, Tensor> attn_fwd(const Tensor& q, const Tensor& k, const Tensor& v, bool causal, double scale,
                                            const c10::optional<Tensor>& kv_lens, const c10::optional<Tensor>& bias,
                                            const c10::optional<Tensor>& alibi_slopes, double p_drop, int64_t salt,
                                            const c10::optional<Tensor>& kv_start, const c10::optional<Tensor>& doc_start) {
  c10::cuda::CUDAGuard guard(q.device());
  const QGeom g = q_geom(q, k, v, "attn_fwd");
  const int B = g.B, A = g.A, Sq = g.Sq, Sk = g.Sk, D = g.D;
  const bool has_alibi = alibi_slopes.has_value() && alibi_slopes->defined();
  const int* dst = doc_starts(doc_start, q, g, causal,
                              (kv_lens.has_value() && kv_lens->defined()) || (kv_start.has_value() && kv_start->defined()) ||
                                  (bias.has_value() && bias->defined()) || has_alibi,
                              p_drop, "attn_fwd: doc_start");
  Tensor o = at::empty({B, Sq, A, D}, q.options());
  Tensor lse = at::empty({B, A, Sq}, q.options().dtype(at::kFloat));
  const long* qs = g.qs;
  long ks[3] = {k.stride(0), k.stride(1), k.stride(2)};
  long vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  const int* kvl = key_bound(kv_lens, q, B, "attn_fwd: kv_lens");
  const int* kvs = key_bound(kv_start, q, B, "attn_fwd: kv_start");
  BiasDesc bd = bias_desc(bias, B, A, Sq, Sk);
  const float* slopes = nullptr;
  if (alibi_slopes.has_value() && alibi_slopes->defined()) {
    TORCH_CHECK(alibi_slopes->scalar_type() == at::kFloat && alibi_slopes->numel() == A && alibi_slopes->is_cuda(), "alibi_slopes: fp32 cuda [A]");
    slopes = alibi_slopes->data_ptr<float>();
  }
  Tensor rng_state;
  LbRngArgs a;
  const bool drop = p_drop > 0.0;
  if (drop) {
    TORCH_CHECK(p_drop < 1.0, "dropout probability must be in [0, 1)");
    rng_state = at::empty({2}, q.options().dtype(at::kLong));
    a = next_rng(salt);
  } else {
    rng_state = at::empty({0}, q.options().dtype(at::kLong));
  }
  check(lb_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), B, A, g.G, Sq, Sk, D, qs,
                    ks, vs, causal ? 1 : 0, (float)scale, kvl, kvs, dst, bd.ptr, bd.strides, slopes, (float)p_drop,
                    drop ? &a : nullptr,
                    drop ? reinterpret_cast<long long*>(rng_state.data_ptr<int64_t>()) : nullptr, cur_stream()),
        "attn_fwd");
  return std::make_tuple(o.permute({0, 2, 1, 3}), lse, rng_state);
}

// ---- KV-cache decoding ------------------------------------------------------------------------------
// The cache capacity C (rows per head) cannot be checked against the device-side lengths without a host sync: the
// caller (libai_b200.inference.kv_cache.StaticKVCache) guarantees cache_seqlens[b] + Sq <= C before every call.
void check_cache(const Tensor& k_cache, const Tensor& v_cache, const char* what) {
  TORCH_CHECK(k_cache.is_cuda() && k_cache.scalar_type() == at::kBFloat16 && v_cache.scalar_type() == at::kBFloat16,
              what, ": bf16 CUDA cache expected");
  TORCH_CHECK(k_cache.dim() == 4 && k_cache.sizes() == v_cache.sizes() && k_cache.is_contiguous() && v_cache.is_contiguous(),
              what, ": K and V caches must be contiguous [B, G, C, D] of the same shape");
  TORCH_CHECK(k_cache.size(3) == 64 || k_cache.size(3) == 128, what, ": head dim must be 64 or 128");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(k_cache.data_ptr()) % 16 == 0 &&
              reinterpret_cast<uintptr_t>(v_cache.data_ptr()) % 16 == 0, what, ": caches must be 16-byte aligned");
}
void check_lengths(const Tensor& t, int64_t B, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kInt && t.dim() == 1 && t.size(0) == B && t.is_contiguous(), what,
              ": int32 CUDA [B] expected");
}

// k, v of the packed projection qkv ([B, Sq, A, 3D] or grouped [B, Sq, G, r + 2, D]) go to rows cache_seqlens[b] + i
// of the caches [B, G, C, D]; with cos/sin (fp32 [>= positions, D]) q and k are rotated first.  Returns the (rotated) q
// as [B, Sq, G * r, D] when write_q, else empty.
Tensor kv_append(const Tensor& qkv, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cache_seqlens,
                 const c10::optional<Tensor>& cosv, const c10::optional<Tensor>& sinv, bool write_q) {
  c10::cuda::CUDAGuard guard(qkv.device());
  check_cache(k_cache, v_cache, "kv_append");
  const int B = (int)k_cache.size(0), G = (int)k_cache.size(1), C = (int)k_cache.size(2), D = (int)k_cache.size(3);
  TORCH_CHECK(qkv.is_cuda() && qkv.scalar_type() == at::kBFloat16 && qkv.is_contiguous(),
              "kv_append: contiguous bf16 packed projection expected");
  const PackedQKV g = packed_qkv(qkv, "kv_append");
  TORCH_CHECK(g.B == B && g.G == G && g.D == D, "kv_append: qkv does not match the cache");
  const int Sq = g.S, A = G * g.r;
  TORCH_CHECK(Sq >= 1 && Sq <= C, "kv_append: 1 <= Sq <= capacity");
  check_lengths(cache_seqlens, B, "kv_append: cache_seqlens");
  const float* cp = nullptr;
  const float* sp = nullptr;
  if (cosv.has_value() && cosv->defined()) {
    TORCH_CHECK(sinv.has_value() && sinv->defined(), "kv_append: cos and sin go together");
    TORCH_CHECK(cosv->scalar_type() == at::kFloat && sinv->scalar_type() == at::kFloat && cosv->is_contiguous() &&
                sinv->is_contiguous() && cosv->dim() == 2 && cosv->size(1) == D && cosv->sizes() == sinv->sizes() &&
                cosv->is_cuda(), "kv_append: cos/sin fp32 contiguous [positions, D]");
    // like the capacity, the rows of the tables (positions up to cache_seqlens[b] + Sq - 1) are the caller's guarantee
    cp = cosv->data_ptr<float>();
    sp = sinv->data_ptr<float>();
  }
  Tensor q_out = write_q ? at::empty({B, Sq, A, D}, qkv.options()) : at::empty({0}, qkv.options());
  check(lb_kv_append(qkv.data_ptr(), cp, sp, write_q ? q_out.data_ptr() : nullptr, k_cache.data_ptr(),
                     v_cache.data_ptr(), cache_seqlens.data_ptr<int>(), B, Sq, G, g.r, C, D, cur_stream()),
        "kv_append");
  return q_out;
}

// q [B, Sq, A, D] (any strides with D contiguous, e.g. a view of the packed projection) against the caches [B, G, C, D]
// (query head h reads cache head h / (A / G)); query i of sample b sees keys kv_start[b] .. cache_seqlens[b] + i.
// Returns o [B, Sq, A, D] contiguous.  splits = 0: automatic.
Tensor decode_attn(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cache_seqlens,
                   const Tensor& kv_start, double scale, int64_t splits) {
  c10::cuda::CUDAGuard guard(q.device());
  check_cache(k_cache, v_cache, "decode_attn");
  const int B = (int)k_cache.size(0), G = (int)k_cache.size(1), C = (int)k_cache.size(2), D = (int)k_cache.size(3);
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kBFloat16 && q.dim() == 4 && q.stride(3) == 1,
              "decode_attn: bf16 q [B, Sq, A, D] with D contiguous expected");
  const int A = (int)q.size(2);
  TORCH_CHECK(q.size(0) == B && A % G == 0 && q.size(3) == D, "decode_attn: q does not match the cache");
  const int Sq = (int)q.size(1);
  TORCH_CHECK(Sq >= 1 && Sq <= 16, "decode_attn: 1 <= Sq <= 16 new queries");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(q.data_ptr()) % 16 == 0 && q.stride(0) % 8 == 0 && q.stride(1) % 8 == 0 &&
              q.stride(2) % 8 == 0, "decode_attn: q must be 16-byte aligned with strides that are multiples of 8");
  check_lengths(cache_seqlens, B, "decode_attn: cache_seqlens");
  check_lengths(kv_start, B, "decode_attn: kv_start");
  const int row_blocks = ((A / G) * Sq + 15) / 16;   // (query head, token) rows of one cache head, 16 per CTA
  const int nsplit = splits > 0 ? (int)std::min<int64_t>(splits, 32) : lb_decode_splits(B, G * row_blocks, C, D);
  Tensor o = at::empty({B, Sq, A, D}, q.options());
  Tensor part_o, part_ml;
  if (nsplit > 1) {
    part_o = at::empty({(int64_t)B * A * nsplit * Sq * D}, q.options().dtype(at::kFloat));
    part_ml = at::empty({(int64_t)B * A * nsplit * Sq * 2}, q.options().dtype(at::kFloat));
  }
  long qs[3] = {q.stride(0), q.stride(1), q.stride(2)};
  check(lb_decode_attn(q.data_ptr(), qs, k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(),
                       nsplit > 1 ? part_o.data_ptr<float>() : nullptr, nsplit > 1 ? part_ml.data_ptr<float>() : nullptr,
                       cache_seqlens.data_ptr<int>(), kv_start.data_ptr<int>(), B, Sq, A, G, C, D, (float)scale, nsplit,
                       cur_stream()),
        "decode_attn");
  return o;
}

// ---- shifted-window attention -----------------------------------------------------------------------
// qkv [B, H*W, 3*C] in image order (per token [3, heads, d]), an H x W map of ws x ws windows cyclically shifted by
// `shift`; table fp32 [(2ws - 1)^2, heads]; tau fp32 [heads] selects cosine attention (SwinV2).  Returns the head dim.
int64_t check_window_args(const Tensor& qkv, int64_t H, int64_t W, int64_t ws, int64_t shift, int64_t heads,
                          const Tensor& table, const c10::optional<Tensor>& tau, const char* what) {
  TORCH_CHECK(qkv.is_cuda() && qkv.scalar_type() == at::kBFloat16 && qkv.dim() == 3 && qkv.is_contiguous(), what,
              ": contiguous bf16 CUDA qkv [B, H*W, 3*C] expected");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 16 == 0, what, ": qkv must be 16-byte aligned");
  TORCH_CHECK(heads >= 1 && heads <= 65535 && qkv.size(2) % (3 * heads) == 0, what, ": qkv width ", qkv.size(2),
              " is not 3 * heads * d for ", heads, " heads");
  const int64_t d = qkv.size(2) / (3 * heads);
  TORCH_CHECK(d % 8 == 0 && d >= 8 && d <= 64, what, ": head dim ", d,
              " not supported (supported: multiples of 8 from 8 to 64)");
  TORCH_CHECK(ws >= 1 && ws <= 16, what, ": window ", ws, " not supported (supported: 1 to 16)");
  TORCH_CHECK(H >= 1 && W >= 1 && H % ws == 0 && W % ws == 0, what, ": the ", H, " x ", W,
              " map must be a whole number of ", ws, " x ", ws, " windows");
  TORCH_CHECK(qkv.size(1) == H * W, what, ": qkv has ", qkv.size(1), " tokens, the map ", H * W);
  TORCH_CHECK(qkv.size(0) * H * W <= INT32_MAX, what, ": more than 2^31 - 1 tokens");
  TORCH_CHECK(shift >= 0 && shift < ws, what, ": shift ", shift, " not supported (supported: 0 <= shift < window)");
  TORCH_CHECK(table.is_cuda() && table.scalar_type() == at::kFloat && table.is_contiguous() && table.dim() == 2 &&
                  table.size(0) == (2 * ws - 1) * (2 * ws - 1) && table.size(1) == heads,
              what, ": table must be contiguous fp32 CUDA [(2 * window - 1)^2, heads]");
  if (tau.has_value() && tau->defined())
    TORCH_CHECK(tau->is_cuda() && tau->scalar_type() == at::kFloat && tau->is_contiguous() && tau->numel() == heads,
                what, ": tau must be contiguous fp32 CUDA [heads]");
  return d;
}

std::tuple<Tensor, Tensor> window_attn_fwd(const Tensor& qkv, int64_t H, int64_t W, int64_t window, int64_t shift,
                                           int64_t heads, double scale, const Tensor& table,
                                           const c10::optional<Tensor>& tau) {
  c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t d = check_window_args(qkv, H, W, window, shift, heads, table, tau, "window_attn_fwd");
  const int64_t B = qkv.size(0), nwin = B * (H / window) * (W / window);
  Tensor o = at::empty({B, H * W, heads * d}, qkv.options());
  Tensor lse = at::empty({nwin, heads, window * window}, qkv.options().dtype(at::kFloat));
  const bool cos = tau.has_value() && tau->defined();
  check(lb_window_attn_fwd(qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), table.data_ptr<float>(),
                           cos ? tau->data_ptr<float>() : nullptr, (int)B, (int)H, (int)W, (int)window, (int)shift,
                           (int)heads, (int)d, (float)scale, cur_stream()),
        "window_attn_fwd");
  return {o, lse};
}

// returns (dqkv [B, H*W, 3*C] bf16, dtable fp32 like table, dtau fp32 [heads] (empty without tau))
std::tuple<Tensor, Tensor, Tensor> window_attn_bwd(const Tensor& dout, const Tensor& qkv, const Tensor& lse, int64_t H, int64_t W, int64_t window,
                                                   int64_t shift, int64_t heads, double scale, const Tensor& table,
                                                   const c10::optional<Tensor>& tau) {
  c10::cuda::CUDAGuard guard(qkv.device());
  const int64_t d = check_window_args(qkv, H, W, window, shift, heads, table, tau, "window_attn_bwd");
  const int64_t B = qkv.size(0), N = window * window, nwin = B * (H / window) * (W / window);
  TORCH_CHECK(dout.is_cuda() && dout.scalar_type() == at::kBFloat16 && dout.is_contiguous() &&
                  dout.sizes() == at::IntArrayRef({B, H * W, heads * d}) &&
                  reinterpret_cast<uintptr_t>(dout.data_ptr()) % 16 == 0,
              "window_attn_bwd: dout must be a contiguous 16-byte aligned bf16 [B, H*W, C]");
  TORCH_CHECK(lse.is_cuda() && lse.scalar_type() == at::kFloat && lse.is_contiguous() &&
                  lse.sizes() == at::IntArrayRef({nwin, heads, N}),
              "window_attn_bwd: lse must be the forward's fp32 [windows, heads, window^2]");
  const bool cos = tau.has_value() && tau->defined();
  const int G = lb_window_attn_groups((int)B, (int)H, (int)W, (int)window, (int)heads);
  Tensor dqkv = at::empty_like(qkv);
  Tensor dtable = at::empty_like(table);
  Tensor dtau = at::empty({cos ? heads : 0}, table.options());
  Tensor part = at::empty({std::max<int64_t>(G, 1) * heads * N * N}, table.options());
  Tensor tau_part = at::empty({cos ? std::max<int64_t>(G, 1) * heads : 0}, table.options());
  check(lb_window_attn_bwd(dout.data_ptr(), qkv.data_ptr(), lse.data_ptr<float>(),
                           table.data_ptr<float>(), cos ? tau->data_ptr<float>() : nullptr, dqkv.data_ptr(),
                           dtable.data_ptr<float>(), cos ? dtau.data_ptr<float>() : nullptr, part.data_ptr<float>(),
                           cos ? tau_part.data_ptr<float>() : nullptr, (int)B, (int)H, (int)W, (int)window, (int)shift,
                           (int)heads, (int)d, (float)scale, cur_stream()),
        "window_attn_bwd");
  if (nwin == 0) {
    dtable.zero_();
    dtau.zero_();
  }
  return {dqkv, dtable, dtau};
}

// `dbias` (optional, fp32, same shape as `bias`): the gradient of a learned bias is accumulated into it
std::tuple<Tensor, Tensor, Tensor, Tensor> attn_bwd(const Tensor& dout, const Tensor& q, const Tensor& k, const Tensor& v,
                                            const Tensor& o, const Tensor& lse, bool causal, double scale,
                                            const c10::optional<Tensor>& kv_lens, const c10::optional<Tensor>& bias,
                                            const c10::optional<Tensor>& alibi_slopes, c10::optional<Tensor> dbias,
                                            double p_drop, const c10::optional<Tensor>& rng_state,
                                            const c10::optional<Tensor>& kv_start,
                                            const c10::optional<Tensor>& doc_start) {
  c10::cuda::CUDAGuard guard(q.device());
  const QGeom g = q_geom(q, k, v, "attn_bwd");
  const int B = g.B, A = g.A, G = g.G, Sq = g.Sq, Sk = g.Sk, D = g.D, r = A / G;
  const int* dst = doc_starts(doc_start, q, g, causal,
                              (kv_lens.has_value() && kv_lens->defined()) || (kv_start.has_value() && kv_start->defined()) ||
                                  (bias.has_value() && bias->defined()) ||
                                  (alibi_slopes.has_value() && alibi_slopes->defined()),
                              p_drop, "attn_bwd: doc_start");
  // Sq == Sk: gradients are produced in the packed [B, S, G, r + 2, D] layout (r = 1: [B, S, A, 3, D]) so that the QKV
  // dgrad/wgrad GEMMs read them directly; dq comes back in q's shape (a copy only for a 4-D q with r > 1).
  // Sq != Sk: dq is [B, Sq, G, r, D] and dk, dv are packed as [B, Sk, G, 2, D]; the returned dqkv is empty.
  Tensor dqkv, dq5, dk, dv;
  if (Sq == Sk) {
    dqkv = at::empty({B, Sq, G, r + 2, D}, q.options());
    dq5 = dqkv.narrow(3, 0, r).permute({0, 2, 3, 1, 4});
    dk = dqkv.select(3, r).permute({0, 2, 1, 3});
    dv = dqkv.select(3, r + 1).permute({0, 2, 1, 3});
  } else {
    dqkv = at::empty({0}, q.options());
    dq5 = at::empty({B, Sq, G, r, D}, q.options()).permute({0, 2, 3, 1, 4});
    Tensor dkv = at::empty({B, Sk, G, 2, D}, q.options());
    dk = dkv.select(3, 0).permute({0, 2, 1, 3});
    dv = dkv.select(3, 1).permute({0, 2, 1, 3});
  }
  const long dqs[4] = {dq5.stride(0), dq5.stride(1), dq5.stride(2), dq5.stride(3)};
  const long dkvs[3] = {dk.stride(0), dk.stride(1), dk.stride(2)};
  Tensor delta = at::empty({B, A, Sq}, q.options().dtype(at::kFloat));
  // fp32 dQ tiles, cleared by the delta kernel
  Tensor dq_acc = at::empty({lb_attn_bwd_accum_floats(B, A, Sq, D)}, q.options().dtype(at::kFloat));
  // per (batch, head, 64-query block): key blocks that have added their dQ contribution
  Tensor dq_order = at::zeros({B * A * ((Sq + 63) / 64)}, q.options().dtype(at::kInt));
  TORCH_CHECK(o.stride(3) == 1, "attn_bwd: o must have contiguous D");
  Tensor dout_c = dout;
  if (dout.strides() != o.strides()) {  // bring dout into the [B, S, A, D]-backed layout of o
    dout_c = at::empty_strided(o.sizes(), o.strides(), o.options());
    dout_c.copy_(dout);
  }
  const long* qs = g.qs;
  long ks[3] = {k.stride(0), k.stride(1), k.stride(2)};
  long vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  long ds[3] = {dout_c.stride(0), dout_c.stride(1), dout_c.stride(2)};
  BiasDesc bd = bias_desc(bias, B, A, Sq, Sk);
  const int* kvl = key_bound(kv_lens, q, B, "attn_bwd: kv_lens");
  const int* kvs = key_bound(kv_start, q, B, "attn_bwd: kv_start");
  float* dbp = nullptr;
  if (dbias.has_value() && dbias->defined()) {
    TORCH_CHECK(bd.ptr != nullptr && dbias->scalar_type() == at::kFloat && dbias->sizes() == bias->sizes() &&
                    dbias->strides() == bias->strides(), "attn_bwd: dbias must be fp32 with the shape/strides of bias");
    dbp = dbias->data_ptr<float>();
  }
  const bool has_rng = p_drop > 0.0 && rng_state.has_value() && rng_state->defined() && rng_state->numel() == 2;
  check(lb_attn_bwd(dout_c.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr<float>(),
                    dq5.data_ptr(), dk.data_ptr(), dv.data_ptr(), dqs, dkvs, delta.data_ptr<float>(),
                    dq_acc.data_ptr<float>(), B, A, G, Sq, Sk, D, qs, ks, vs, ds, causal ? 1 : 0, (float)scale, kvl, kvs,
                    dst, bd.ptr, bd.strides,
                    (alibi_slopes.has_value() && alibi_slopes->defined()) ? alibi_slopes->data_ptr<float>() : nullptr, dbp,
                    (float)(has_rng ? p_drop : 0.0),
                    has_rng ? reinterpret_cast<const long long*>(rng_state->data_ptr<int64_t>()) : nullptr,
                    reinterpret_cast<unsigned*>(dq_order.data_ptr<int>()), cur_stream()),
        "attn_bwd");
  Tensor dq = q.dim() == 5 ? dq5 : dq5.reshape({B, A, Sq, D});   // after the kernel: for r > 1 this copies
  return std::make_tuple(dq, dk, dv, dqkv);
}

// ---- fused collectives ---------------------------------------------------------------------------------------
std::vector<long> to_longs(at::IntArrayRef v) { return std::vector<long>(v.begin(), v.end()); }

const void* opt_ptr(const c10::optional<Tensor>& t) { return (t.has_value() && t->defined()) ? t->data_ptr() : nullptr; }

// all-gather -> GEMM: y [M, N] = epilogue(all_gather(shard) @ op(w)); `gathered` is the local symmetric buffer [M, K]
// whose remote rows the peers' copy CTAs fill during the kernel.  Epilogue: + bias, activation (returning the
// pre-activation as second tensor when `need_pre`), or `* act'(pre_in)` (dgrad fused with the activation backward) and
// optional column sums into `colsum` (fp32 [N]).
std::tuple<Tensor, Tensor> ag_gemm(const Tensor& gathered, const Tensor& shard, const Tensor& w, int64_t layout,
                                   const c10::optional<Tensor>& bias, int64_t act, bool need_pre,
                                   const c10::optional<Tensor>& pre_in, c10::optional<Tensor> colsum, bool fill_local,
                                   int64_t world, int64_t rank, at::IntArrayRef peer_buf, at::IntArrayRef peer_flags,
                                   at::IntArrayRef peer_done, Tensor state, int64_t n_comm) {
  c10::cuda::CUDAGuard guard(gathered.device());
  TORCH_CHECK(gathered.dim() == 2 && shard.dim() == 2 && w.dim() == 2 && gathered.is_contiguous() && shard.is_contiguous() &&
                  w.is_contiguous(), "ag_gemm: contiguous 2-D operands");
  TORCH_CHECK(layout == 0 || layout == 1, "ag_gemm: layout 0 (w [N,K]) or 1 (w [K,N])");
  const int64_t M = gathered.size(0), K = gathered.size(1), N = layout == 0 ? w.size(0) : w.size(1);
  TORCH_CHECK((layout == 0 ? w.size(1) : w.size(0)) == K && shard.size(1) == K && shard.size(0) * world == M, "ag_gemm: shape mismatch");
  auto pb = to_longs(peer_buf), pf = to_longs(peer_flags), pd = to_longs(peer_done);
  Tensor out = at::empty({M, N}, gathered.options());
  Tensor pre = need_pre ? at::empty({M, N}, gathered.options()) : Tensor();
  float* cs = (colsum.has_value() && colsum->defined()) ? colsum->data_ptr<float>() : nullptr;
  check(lb_gemm_bf16_comm(gathered.data_ptr(), w.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, (int)layout, 0,
                          opt_ptr(bias), (int)act, need_pre ? pre.data_ptr() : nullptr, opt_ptr(pre_in), cs, 1, (int)world,
                          (int)rank, pb.data(), pf.data(), pd.data(), state.data_ptr(), shard.data_ptr(), fill_local ? 1 : 0,
                          nullptr, nullptr, 0, (int)n_comm, cur_stream()),
        "ag_gemm");
  return {out, need_pre ? pre : out};
}

// wgrad with the all-gather inside: out [Nl, K] (fp32) (+)= gyᵀ [Nl, T] @ all_gather(shard) [T, K]; the shards lie
// along the reduction dimension, partitions of the local shard run first while the remote ones arrive.
void ag_wgrad(const Tensor& gy, const Tensor& gathered, const Tensor& shard, Tensor out, bool accumulate, int64_t world,
              int64_t rank, at::IntArrayRef peer_buf, at::IntArrayRef peer_flags, at::IntArrayRef peer_done, Tensor state,
              int64_t n_comm) {
  c10::cuda::CUDAGuard guard(gy.device());
  TORCH_CHECK(gy.dim() == 2 && gathered.dim() == 2 && gy.is_contiguous() && gathered.is_contiguous() && shard.is_contiguous(),
              "ag_wgrad: contiguous 2-D operands");
  const int64_t T = gy.size(0), Nl = gy.size(1), K = gathered.size(1);
  TORCH_CHECK(gathered.size(0) == T && shard.size(1) == K && shard.size(0) * world == T, "ag_wgrad: shape mismatch");
  TORCH_CHECK(out.scalar_type() == at::kFloat && out.dim() == 2 && out.size(0) == Nl && out.size(1) == K && out.is_contiguous(),
              "ag_wgrad: out must be contiguous fp32 [N_local, K]");
  if (!accumulate) out.zero_();
  auto pb = to_longs(peer_buf), pf = to_longs(peer_flags), pd = to_longs(peer_done);
  check(lb_gemm_bf16_comm(gy.data_ptr(), gathered.data_ptr(), out.data_ptr(), (int)Nl, (int)K, (int)T, 2, 2, nullptr, 0,
                          nullptr, nullptr, nullptr, 1, (int)world, (int)rank, pb.data(), pf.data(), pd.data(),
                          state.data_ptr(), shard.data_ptr(), 0, nullptr, nullptr, 0, (int)n_comm, cur_stream()),
        "ag_wgrad");
}

// GEMM -> reduce-scatter: returns [M / world, N] = sum over ranks of (x @ op(w)) rows owned by this rank (+bias +residual)
Tensor gemm_rs(const Tensor& x, const Tensor& w, int64_t layout, const c10::optional<Tensor>& bias,
               const c10::optional<Tensor>& residual, int64_t world, int64_t rank, at::IntArrayRef peer_buf,
               at::IntArrayRef peer_flags, at::IntArrayRef peer_done, Tensor state, int64_t staging_parity_off) {
  c10::cuda::CUDAGuard guard(x.device());
  TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.is_contiguous() && w.is_contiguous(), "gemm_rs: contiguous 2-D operands");
  TORCH_CHECK(layout == 0 || layout == 1, "gemm_rs: layout 0 (w [N,K]) or 1 (w [K,N])");
  const int64_t M = x.size(0), K = x.size(1), N = layout == 0 ? w.size(0) : w.size(1);
  TORCH_CHECK((layout == 0 ? w.size(1) : w.size(0)) == K, "gemm_rs: K mismatch");
  auto pb = to_longs(peer_buf), pf = to_longs(peer_flags), pd = to_longs(peer_done);
  Tensor out = at::empty({M / world, N}, x.options());
  check(lb_gemm_bf16_comm(x.data_ptr(), w.data_ptr(), out.data_ptr(), (int)M, (int)N, (int)K, (int)layout, 0, opt_ptr(bias),
                          0, nullptr, nullptr, nullptr, 2, (int)world, (int)rank, pb.data(), pf.data(), pd.data(),
                          state.data_ptr(), nullptr, 0, opt_ptr(residual), out.data_ptr(), (long)staging_parity_off, 0,
                          cur_stream()),
        "gemm_rs");
  return out;
}

void zero_reduce_scatter(at::IntArrayRef grad_ptrs, at::IntArrayRef flag_ptrs, Tensor red, Tensor sqnorm, int64_t lo,
                         int64_t n, double scale, int64_t world, int64_t rank, int64_t epoch, int64_t mc_grad) {
  c10::cuda::CUDAGuard guard(red.device());
  auto g = to_longs(grad_ptrs), f = to_longs(flag_ptrs);
  check(lb_zero_reduce_scatter(g.data(), f.data(), red.data_ptr<float>(), sqnorm.data_ptr<float>(), (long)lo, (long)n,
                               (float)scale, (int)world, (int)rank, (unsigned)epoch, (long)mc_grad, cur_stream()),
        "zero_reduce_scatter");
}

void zero_adam_allgather(Tensor master, const Tensor& red, Tensor m, Tensor v, at::IntArrayRef param_ptrs,
                         at::IntArrayRef flag_ptrs, Tensor done_counter, const Tensor& clip, int64_t lo, int64_t n,
                         double lr, double b1, double b2, double eps, double wd, double bc1, double bc2, bool decoupled,
                         int64_t world, int64_t rank, int64_t epoch, int64_t mc_param) {
  c10::cuda::CUDAGuard guard(master.device());
  auto pp = to_longs(param_ptrs), f = to_longs(flag_ptrs);
  check(lb_zero_adam_allgather(master.data_ptr<float>(), red.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                               pp.data(), f.data(), reinterpret_cast<unsigned*>(done_counter.data_ptr()),
                               clip.data_ptr<float>(), (long)lo, (long)n, (float)lr, (float)b1, (float)b2, (float)eps,
                               (float)wd, (float)bc1, (float)bc2, decoupled ? 1 : 0, (int)world, (int)rank,
                               (unsigned)epoch, (long)mc_param, cur_stream()),
        "zero_adam_allgather");
}

void device_barrier(at::IntArrayRef flag_ptrs, int64_t world, int64_t rank, int64_t slot, int64_t epoch) {
  auto f = to_longs(flag_ptrs);
  check(lb_device_barrier(f.data(), (int)world, (int)rank, (int)slot, (unsigned)epoch, cur_stream()), "device_barrier");
}

void p2p_allgather(const Tensor& shard, at::IntArrayRef out_ptrs, at::IntArrayRef flag_ptrs, Tensor done_counter,
                   int64_t world, int64_t rank, int64_t epoch) {
  c10::cuda::CUDAGuard guard(shard.device());
  auto o = to_longs(out_ptrs), f = to_longs(flag_ptrs);
  check(lb_p2p_allgather(shard.data_ptr(), o.data(), f.data(), reinterpret_cast<unsigned*>(done_counter.data_ptr()),
                         (long)(shard.numel() * shard.element_size()), (int)world, (int)rank, (unsigned)epoch,
                         cur_stream()),
        "p2p_allgather");
}

}  // namespace

TORCH_LIBRARY(libai_b200, m) {
  m.def("spin_timeout_report() -> str", &spin_timeout_report);
  m.def("ag_gemm(Tensor gathered, Tensor shard, Tensor w, int layout, Tensor? bias, int act, bool need_pre, Tensor? pre_in, Tensor(a!)? colsum, bool fill_local, int world, int rank, int[] peer_buf, int[] peer_flags, int[] peer_done, Tensor(b!) state, int n_comm) -> (Tensor, Tensor)", &ag_gemm);
  m.def("ag_wgrad(Tensor gy, Tensor gathered, Tensor shard, Tensor(a!) out, bool accumulate, int world, int rank, int[] peer_buf, int[] peer_flags, int[] peer_done, Tensor(b!) state, int n_comm) -> ()", &ag_wgrad);
  m.def("gemm_rs(Tensor x, Tensor w, int layout, Tensor? bias, Tensor? residual, int world, int rank, int[] peer_buf, int[] peer_flags, int[] peer_done, Tensor(a!) state, int staging_parity_off) -> Tensor", &gemm_rs);
  m.def("zero_reduce_scatter(int[] grad_ptrs, int[] flag_ptrs, Tensor(a!) red, Tensor(b!) sqnorm, int lo, int n, float scale, int world, int rank, int epoch, int mc_grad=0) -> ()", &zero_reduce_scatter);
  m.def("zero_adam_allgather(Tensor(a!) master, Tensor red, Tensor(b!) m, Tensor(c!) v, int[] param_ptrs, int[] flag_ptrs, Tensor(d!) done_counter, Tensor clip, int lo, int n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, bool decoupled, int world, int rank, int epoch, int mc_param=0) -> ()", &zero_adam_allgather);
  m.def("device_barrier(int[] flag_ptrs, int world, int rank, int slot, int epoch) -> ()", &device_barrier);
  m.def("p2p_allgather(Tensor shard, int[] out_ptrs, int[] flag_ptrs, Tensor(a!) done_counter, int world, int rank, int epoch) -> ()", &p2p_allgather);
  m.def("gemm(Tensor a, Tensor b, int layout, Tensor? bias, Tensor? out, bool accumulate, ScalarType out_dtype) -> Tensor", &gemm);
  m.def("linear_bias_residual(Tensor x, Tensor w, Tensor? bias, Tensor residual) -> Tensor", &linear_bias_residual);
  m.def("embedding_fwd(Tensor ids, Tensor table, int vocab_start) -> Tensor", &embedding_fwd);
  m.def("embedding_bwd(Tensor ids, Tensor gy, Tensor(a!) grad, int vocab_start) -> ()", &embedding_bwd);
  m.def("gemm_tuned(Tensor a, Tensor b, int layout, int bn, int splits, bool fp32_out) -> Tensor", &gemm_tuned);
  m.def("gemm_schedule(int schedule) -> int", &gemm_schedule);
  m.def("linear_fwd(Tensor x, Tensor w, Tensor? bias, int act, bool need_pre) -> (Tensor, Tensor)", &linear_fwd);
  m.def("quantize_e4m3(Tensor x) -> (Tensor, Tensor)", &quantize_e4m3);
  m.def("linear_fp8_fwd(Tensor xq, Tensor wq, Tensor deq_x, Tensor deq_w, Tensor? bias, int act, bool need_pre, Tensor? residual=None, int bn=0) -> (Tensor, Tensor)", &linear_fp8_fwd);
  m.def("act_bwd(Tensor gy, Tensor pre, int act) -> Tensor", &act_bwd);
  m.def("colsum(Tensor x, Tensor(a!)? accum=None) -> Tensor", &colsum);
  m.def("norm_fwd(Tensor x, Tensor gamma, Tensor? beta, float eps, bool rms) -> (Tensor, Tensor, Tensor)", &norm_fwd);
  m.def("norm_bwd(Tensor gy, Tensor x, Tensor gamma, Tensor mean, Tensor rstd, bool rms, bool has_bias, Tensor(a!)? dgamma_accum=None, Tensor(b!)? dbeta_accum=None, Tensor? gadd=None) -> (Tensor, Tensor, Tensor)", &norm_bwd);
  m.def("bias_act_fwd(Tensor x, Tensor? bias, int act) -> Tensor", &bias_act_fwd);
  m.def("bias_act_bwd(Tensor gy, Tensor x, Tensor? bias, int act) -> Tensor", &bias_act_bwd);
  m.def("bias_residual_fwd(Tensor x, Tensor? bias, Tensor? res) -> Tensor", &bias_residual_fwd);
  m.def("swiglu_fwd(Tensor gate, Tensor up) -> Tensor", &swiglu_fwd);
  m.def("swiglu_bwd(Tensor gy, Tensor gate, Tensor up) -> (Tensor, Tensor)", &swiglu_bwd);
  m.def("swiglu_packed_fwd(Tensor gu) -> Tensor", &swiglu_packed_fwd);
  m.def("swiglu_packed_bwd(Tensor gy, Tensor gu) -> Tensor", &swiglu_packed_bwd);
  m.def("dgrad_actgrad(Tensor gy, Tensor w, Tensor pre, int act, Tensor(a!)? bias_grad=None) -> Tensor", &dgrad_actgrad);
  m.def("rope(Tensor x, Tensor cos, Tensor sin, bool backward) -> Tensor", &rope);
  m.def("rope_qkv(Tensor(a!) qkv, Tensor cos, Tensor sin, int pos_offset, bool backward, bool inplace, Tensor? positions=None) -> Tensor(a!)", &rope_qkv);
  m.def("ce_stats(Tensor logits, Tensor labels, int vocab_start) -> (Tensor, Tensor, Tensor)", &ce_stats);
  m.def("ce_bwd(Tensor(a!) logits, Tensor labels, Tensor lse, Tensor gloss, int vocab_start) -> Tensor(a!)", &ce_bwd);
  m.def("fused_adamw(Tensor(a!) master, Tensor grad, Tensor(b!) m, Tensor(c!) v, Tensor? lp_out, Tensor scale, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, bool decoupled) -> ()", &fused_adamw);
  m.def("sqnorm(Tensor x) -> Tensor", &sqnorm);
  m.def("attn_fwd(Tensor q, Tensor k, Tensor v, bool causal, float scale, Tensor? kv_lens, Tensor? bias=None, Tensor? alibi_slopes=None, float p_drop=0.0, int salt=0, Tensor? kv_start=None, Tensor? doc_start=None) -> (Tensor, Tensor, Tensor)", &attn_fwd);
  m.def("attn_bwd(Tensor dout, Tensor q, Tensor k, Tensor v, Tensor o, Tensor lse, bool causal, float scale, Tensor? kv_lens, Tensor? bias=None, Tensor? alibi_slopes=None, Tensor(a!)? dbias=None, float p_drop=0.0, Tensor? rng_state=None, Tensor? kv_start=None, Tensor? doc_start=None) -> (Tensor, Tensor, Tensor, Tensor)", &attn_bwd);
  m.def("kv_append(Tensor qkv, Tensor(a!) k_cache, Tensor(b!) v_cache, Tensor cache_seqlens, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append);
  m.def("window_attn_fwd(Tensor qkv, int H, int W, int window, int shift, int heads, float scale, Tensor table, Tensor? tau) -> (Tensor, Tensor)", &window_attn_fwd);
  m.def("window_attn_bwd(Tensor dout, Tensor qkv, Tensor lse, int H, int W, int window, int shift, int heads, float scale, Tensor table, Tensor? tau) -> (Tensor, Tensor, Tensor)", &window_attn_bwd);
  m.def("decode_attn(Tensor q, Tensor k_cache, Tensor v_cache, Tensor cache_seqlens, Tensor kv_start, float scale, int splits=0) -> Tensor", &decode_attn);
  m.def("bias_dropout_residual(Tensor x, Tensor? bias, Tensor? res, float p, int salt, Tensor? rng_state=None) -> (Tensor, Tensor)", &bias_dropout_residual);
}
