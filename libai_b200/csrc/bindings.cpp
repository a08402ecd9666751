// torch.ops.libai_b200.* : thin argument-checking wrappers around the extern "C" kernel launchers.
// Registered with TORCH_LIBRARY so the in-tree `_C.so` is loaded by torch.ops.load_library (no
// python ABI dependency).
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <cmath>
#include <cstring>
#include <mutex>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <tuple>

#include "launchers.h"

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


bool given(const c10::optional<Tensor>& t) { return t.has_value() && t->defined(); }

// ---- argument checks ------------------------------------------------------------------------------------
// The kernels get raw pointers, so every tensor argument of an op is checked by one call that states its dtype, its
// sizes (kAny: a free dimension), its layout and, where the kernel vector-loads it, its alignment.  Those rules run
// first, for every argument; guard() then requires every argument on the first one's device and that device to be a
// CUDA device, and returns the guard for it.  The guard and every allocation come after the checks, and no check
// syncs the host or allocates.
constexpr int64_t kAny = -1;
constexpr at::ScalarType kAnyDtype = at::ScalarType::Undefined;
enum class Layout { Contiguous, LastDimContiguous, Strided };

// one dtype, or either of two (kAnyDtype: any)
struct Dtypes {
  Dtypes(at::ScalarType t) : a(t), b(t) {}
  Dtypes(at::ScalarType t, at::ScalarType u) : a(t), b(u) {}
  at::ScalarType a, b;
};

const char* dtype_name(at::ScalarType t) {
  switch (t) {
    case at::kBFloat16: return "bf16";
    case at::kHalf: return "fp16";
    case at::kFloat: return "fp32";
    case at::kDouble: return "fp64";
    case at::kInt: return "int32";
    case at::kLong: return "int64";
    case at::kFloat8_e4m3fn: return "float8_e4m3fn";
    case at::kByte: return "uint8";
    default: return c10::toString(t);
  }
}

struct Rule {
  Dtypes dtypes;
  at::IntArrayRef sizes;
  Layout layout;
  int align;
};
std::ostream& operator<<(std::ostream& os, const Rule& r) {
  if (r.align != 0) os << r.align << "-byte aligned ";
  if (r.layout == Layout::Contiguous) os << "contiguous ";
  if (r.dtypes.a != kAnyDtype) os << dtype_name(r.dtypes.a) << " ";
  if (r.dtypes.b != r.dtypes.a) os << "or " << dtype_name(r.dtypes.b) << " ";
  os << "[";
  for (size_t i = 0; i < r.sizes.size(); ++i) {
    if (i > 0) os << ", ";
    if (r.sizes[i] == kAny) os << "*";
    else os << r.sizes[i];
  }
  os << "]";
  if (r.layout == Layout::LastDimContiguous) os << " with a contiguous last dim";
  return os;
}
struct Got {
  const Tensor& t;
};
std::ostream& operator<<(std::ostream& os, const Got& g) {
  return os << dtype_name(g.t.scalar_type()) << " " << g.t.sizes() << " on " << g.t.device();
}

class Args {
 public:
  explicit Args(const char* op) : op_(op) {}
  const char* op() const { return op_; }

  // Checks one argument now and its device in guard().  The first argument checked is the reference: the op runs on
  // its device.
  const Tensor& operator()(const char* name, const Tensor& t, Dtypes dtypes, at::IntArrayRef sizes,
                           Layout layout = Layout::Contiguous, int align = 0) {
    const Rule rule{dtypes, sizes, layout, align};
    TORCH_CHECK(fits(t, rule), op_, ": ", name, " must be ", rule, ", got ", Got{t});
    TORCH_INTERNAL_ASSERT(n_ < kMaxArgs, op_, ": too many tensor arguments");
    seen_[n_++] = {name, &t};
    return t;
  }
  // an optional argument: its data pointer, or nullptr for None
  template <typename T = const void>
  T* opt(const char* name, const c10::optional<Tensor>& t, Dtypes dtypes, at::IntArrayRef sizes,
         Layout layout = Layout::Contiguous, int align = 0) {
    if (!given(t)) return nullptr;
    return static_cast<T*>((*this)(name, *t, dtypes, sizes, layout, align).data_ptr());
  }

  c10::cuda::CUDAGuard guard() const {
    const auto& [ref_name, ref] = seen_[0];
    for (int i = 1; i < n_; ++i)
      TORCH_CHECK(seen_[i].second->device() == ref->device(), op_, ": ", seen_[i].first, " must be on ", ref_name,
                  "'s device ", ref->device(), ", got ", Got{*seen_[i].second});
    TORCH_CHECK(ref->is_cuda(), op_, ": ", ref_name, " must be a CUDA tensor, got ", Got{*ref});
    return c10::cuda::CUDAGuard(ref->device());
  }

 private:
  static bool fits(const Tensor& t, const Rule& r) {
    if (r.dtypes.a != kAnyDtype && t.scalar_type() != r.dtypes.a && t.scalar_type() != r.dtypes.b) return false;
    if (t.dim() != (int64_t)r.sizes.size()) return false;
    for (int64_t i = 0; i < t.dim(); ++i)
      if (r.sizes[i] != kAny && t.size(i) != r.sizes[i]) return false;
    if (r.layout == Layout::Contiguous && !t.is_contiguous()) return false;
    if (r.layout == Layout::LastDimContiguous && t.dim() > 0 && t.stride(-1) != 1) return false;
    return r.align == 0 || reinterpret_cast<uintptr_t>(t.data_ptr()) % r.align == 0;
  }

  static constexpr int kMaxArgs = 16;
  const char* op_;
  std::pair<const char*, const Tensor*> seen_[kMaxArgs];
  int n_ = 0;
};

// ---- GEMM -----------------------------------------------------------------------------------------
struct GemmDims {
  int64_t M, N, K;
};
// the bf16 operands of layout 0: a [M, K] b [N, K]; 1: a [M, K] b [K, N]; 2: a [K, M] b [K, N] (row-major, any row
// stride)
GemmDims gemm_operands(Args& args, const Tensor& a, const Tensor& b, int64_t layout) {
  TORCH_CHECK(layout >= 0 && layout <= 2, args.op(), ": layout must be 0, 1 or 2, got ", layout);
  args("a", a, at::kBFloat16, {kAny, kAny}, Layout::LastDimContiguous);
  GemmDims d;
  d.M = layout == 2 ? a.size(1) : a.size(0);
  d.K = layout == 2 ? a.size(0) : a.size(1);
  if (layout == 0) args("b", b, at::kBFloat16, {kAny, d.K}, Layout::LastDimContiguous);
  else args("b", b, at::kBFloat16, {d.K, kAny}, Layout::LastDimContiguous);
  d.N = layout == 0 ? b.size(0) : b.size(1);
  return d;
}

// Returns out (allocated when not given).
Tensor gemm(const Tensor& a, const Tensor& b, int64_t layout, const c10::optional<Tensor>& bias,
            const c10::optional<Tensor>& out_opt, bool accumulate, at::ScalarType out_dtype) {
  Args args("gemm");
  const auto [M, N, K] = gemm_operands(args, a, b, layout);
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  args.opt("out", out_opt, {at::kBFloat16, at::kFloat}, {M, N}, Layout::LastDimContiguous);
  const at::ScalarType odt = given(out_opt) ? out_opt->scalar_type() : out_dtype;
  TORCH_CHECK(odt == at::kBFloat16 || odt == at::kFloat, "gemm: out must be bf16 or fp32");
  TORCH_CHECK(odt == at::kFloat || !accumulate, "gemm: accumulate needs an fp32 output");
  // a freshly zeroed wgrad output takes the accumulating epilogue too; a given `out` is added to only on request
  const int epi = odt == at::kBFloat16 ? 0 : (accumulate || (layout == 2 && !given(out_opt))) ? 2 : 1;
  TORCH_CHECK(bias_ptr == nullptr || epi == 0, "gemm: a bias needs a bf16 output");
  const auto guard = args.guard();
  const auto opts = a.options().dtype(odt);
  const Tensor out = given(out_opt) ? *out_opt : epi == 2 ? at::zeros({M, N}, opts) : at::empty({M, N}, opts);
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
  Args args("dgrad_actgrad");
  args("gy", gy, at::kBFloat16, {kAny, kAny}, Layout::LastDimContiguous);
  const int64_t M = gy.size(0), K = gy.size(1);
  args("w", w, at::kBFloat16, {K, kAny}, Layout::LastDimContiguous);
  const int64_t N = w.size(1);
  args("pre", pre, at::kBFloat16, {M, N});
  float* colsum = args.opt<float>("bias_grad", bias_grad, at::kFloat, {N});
  const auto guard = args.guard();
  Tensor out = at::empty({M, N}, gy.options());
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

// x [M, K] and w [N, K] of a forward GEMM (bf16, row-major with any row stride); returns (M, N, K)
GemmDims linear_operands(Args& args, const Tensor& x, const Tensor& w) {
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::LastDimContiguous);
  args("w", w, at::kBFloat16, {kAny, x.size(1)}, Layout::LastDimContiguous);
  return {x.size(0), w.size(0), x.size(1)};
}

// y = x @ w^T + bias + residual (one kernel)
Tensor linear_bias_residual(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& bias, const Tensor& residual) {
  Args args("linear_bias_residual");
  const auto [M, N, K] = linear_operands(args, x, w);
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  args("residual", residual, at::kBFloat16, {M, N});
  const auto guard = args.guard();
  Tensor y = at::empty({M, N}, x.options());
  check(lb_gemm_bf16_bias_residual(x.data_ptr(), w.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, (int)x.stride(0),
                                   (int)w.stride(0), bias_ptr, residual.data_ptr(), cur_stream()),
        "linear_bias_residual");
  return y;
}

// y = act(x @ w^T + bias); optionally also returns the pre-activation (for backward)
std::tuple<Tensor, Tensor> linear_fwd(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& bias, int64_t act,
                                      bool need_pre) {
  Args args("linear_fwd");
  const auto [M, N, K] = linear_operands(args, x, w);
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  const auto guard = args.guard();
  Tensor y = at::empty({M, N}, x.options());
  Tensor pre;
  if (need_pre && act != 0) pre = at::empty({M, N}, x.options());
  check(lb_gemm_bf16(x.data_ptr(), w.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, (int)x.stride(0),
                     (int)w.stride(0), (int)N, 0, 0, bias_ptr, (int)act, pre.defined() ? pre.data_ptr() : nullptr, 0, 0,
                     cur_stream()),
        "linear_fwd");
  return std::make_tuple(y, pre.defined() ? pre : at::empty({0}, x.options()));
}

// FP8 (E4M3) weights with per-output-channel scales: w float8_e4m3fn [N, K] (16-byte aligned, K % 16 == 0) and
// w_scale fp32 [N]
void fp8_weight_args(Args& args, const Tensor& w, const Tensor& w_scale) {
  args("w", w, at::kFloat8_e4m3fn, {kAny, kAny}, Layout::Contiguous, 16);
  TORCH_CHECK(w.size(0) >= 1 && w.size(1) >= 16 && w.size(1) % 16 == 0, args.op(),
              ": K must be a positive multiple of 16, got ", w.sizes());
  TORCH_CHECK(w.size(0) <= INT32_MAX && w.size(1) <= INT32_MAX, args.op(), ": N and K must fit in int32");
  args("w_scale", w_scale, at::kFloat, {w.size(0)});
}

// y [M, N] = act((x [M, K] · float(w)ᵀ) · w_scale + bias): the weight-streaming kernel for 1 <= M <= 64 (x bf16
// contiguous and 16-byte aligned, bias bf16 [N] or None, act one of the ACT_* ids without the residual add)
Tensor linear_fp8w(const Tensor& x, const Tensor& w, const Tensor& w_scale, const c10::optional<Tensor>& bias,
                   int64_t act) {
  Args args("linear_fp8w");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  fp8_weight_args(args, w, w_scale);
  const int64_t M = x.size(0), K = x.size(1), N = w.size(0);
  TORCH_CHECK(w.size(1) == K, "linear_fp8w: x [M, K] and w [N, K] disagree on K: ", x.sizes(), " vs ", w.sizes());
  TORCH_CHECK(M >= 1 && M <= 64, "linear_fp8w: 1 <= M <= 64 rows, got ", M);
  TORCH_CHECK(act >= 0 && act <= 5, "linear_fp8w: act must be an activation id in [0, 5], got ", act);
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  const auto guard = args.guard();
  Tensor y = at::empty({M, N}, x.options());
  const long ws = lb_linear_fp8w_workspace((int)M, (int)N, (int)K);
  Tensor part = ws > 0 ? at::empty({ws}, x.options().dtype(at::kFloat)) : Tensor();
  check(lb_linear_fp8w(x.data_ptr(), w.data_ptr(), w_scale.data_ptr<float>(), bias_ptr, y.data_ptr(),
                       ws > 0 ? part.data_ptr<float>() : nullptr, (int)M, (int)N, (int)K, (int)act, cur_stream()),
        "linear_fp8w");
  return y;
}

// bf16 [N, K] = bf16_rn(float(w) · w_scale[:, None]) (the weight the prefill GEMM of an FP8 linear multiplies)
Tensor dequant_e4m3_rows(const Tensor& w, const Tensor& w_scale) {
  Args args("dequant_e4m3_rows");
  fp8_weight_args(args, w, w_scale);
  const auto guard = args.guard();
  Tensor out = at::empty(w.sizes(), w.options().dtype(at::kBFloat16));
  check(lb_dequant_e4m3_rows(w.data_ptr(), w_scale.data_ptr<float>(), out.data_ptr(), (long)w.size(0), (int)w.size(1),
                             cur_stream()),
        "dequant_e4m3_rows");
  return out;
}

// Group-wise INT4 weights: w uint8 [N, K/2] (two 4-bit values per byte, 16-byte aligned), w_scale bf16 and w_zero uint8
// [N, K/128], K % 128 == 0; returns (N, K)
std::pair<int64_t, int64_t> int4_weight_args(Args& args, const Tensor& w, const Tensor& w_scale, const Tensor& w_zero) {
  args("w", w, at::kByte, {kAny, kAny}, Layout::Contiguous, 16);
  const int64_t N = w.size(0), K = 2 * w.size(1);
  TORCH_CHECK(N >= 1 && K >= 128 && K % 128 == 0, args.op(), ": w [N, K/2] needs K a positive multiple of 128, got ",
              w.sizes());
  TORCH_CHECK(N <= INT32_MAX && K <= INT32_MAX, args.op(), ": N and K must fit in int32");
  args("w_scale", w_scale, at::kBFloat16, {N, K / 128});
  args("w_zero", w_zero, at::kByte, {N, K / 128});
  return {N, K};
}

// y [M, N] = act(x [M, K] · Ŵᵀ + bias), Ŵ = bf16_rn((q − w_zero) · w_scale) per group of 128 columns: the
// weight-streaming kernel for 1 <= M <= 64 (x bf16 contiguous and 16-byte aligned, bias bf16 [N] or None, act one of
// the ACT_* ids without the residual add)
Tensor linear_int4w(const Tensor& x, const Tensor& w, const Tensor& w_scale, const Tensor& w_zero,
                    const c10::optional<Tensor>& bias, int64_t act) {
  Args args("linear_int4w");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  const auto [N, K] = int4_weight_args(args, w, w_scale, w_zero);
  const int64_t M = x.size(0);
  TORCH_CHECK(x.size(1) == K, "linear_int4w: x [M, K] and w [N, K/2] disagree on K: ", x.sizes(), " vs ", w.sizes());
  TORCH_CHECK(M >= 1 && M <= 64, "linear_int4w: 1 <= M <= 64 rows, got ", M);
  TORCH_CHECK(act >= 0 && act <= 5, "linear_int4w: act must be an activation id in [0, 5], got ", act);
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  const auto guard = args.guard();
  Tensor y = at::empty({M, N}, x.options());
  const long ws = lb_linear_int4w_workspace((int)M, (int)N, (int)K);
  Tensor part = ws > 0 ? at::empty({ws}, x.options().dtype(at::kFloat)) : Tensor();
  check(lb_linear_int4w(x.data_ptr(), w.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(), bias_ptr, y.data_ptr(),
                        ws > 0 ? part.data_ptr<float>() : nullptr, (int)M, (int)N, (int)K, (int)act, cur_stream()),
        "linear_int4w");
  return y;
}

// bf16 [N, K] = Ŵ (the weight the prefill GEMM of an INT4 linear multiplies)
Tensor dequant_int4_rows(const Tensor& w, const Tensor& w_scale, const Tensor& w_zero) {
  Args args("dequant_int4_rows");
  const auto [N, K] = int4_weight_args(args, w, w_scale, w_zero);
  const auto guard = args.guard();
  Tensor out = at::empty({N, K}, w.options().dtype(at::kBFloat16));
  check(lb_dequant_int4_rows(w.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(), out.data_ptr(), (long)N, (int)K,
                             cur_stream()),
        "dequant_int4_rows");
  return out;
}

// The verify step's arguments of both acceptance ops: logits bf16 or fp32 [b, R, V] (contiguous, R = k + 1 <= 16),
// draft int64 [b, R - 1] and unfinished int64 [b].  Returns (b, R, V).
std::tuple<int64_t, int64_t, int64_t> spec_verify_args(Args& args, const Tensor& logits, const Tensor& draft,
                                                       const Tensor& unfinished) {
  args("logits", logits, Dtypes(at::kBFloat16, at::kFloat), {kAny, kAny, kAny});
  const int64_t B = logits.size(0), R = logits.size(1), V = logits.size(2);
  TORCH_CHECK(B >= 1 && R >= 1 && R <= 16 && V >= 1 && V <= INT32_MAX, args.op(), ": logits [b, k + 1, V] needs ",
              "b >= 1, 1 <= k + 1 <= 16 and V >= 1, got ", logits.sizes());
  args("draft", draft, at::kLong, {B, R - 1});
  args("unfinished", unfinished, at::kLong, {B});
  return {B, R, V};
}

// The output of both acceptance ops, out int64 [b, 2R + 3], followed in its allocation by `scratch` int32 entries for
// the kernel and its block counter, which the launcher zeroes on the stream.
struct SpecOut {
  Tensor out;
  int64_t* data;
  int* scratch;   // nullptr when scratch = 0
  unsigned int* counter;
};
SpecOut spec_out(const Tensor& like, int64_t B, int64_t R, int64_t scratch) {
  const int64_t n = B * (2 * R + 3), words = (scratch + 1) / 2;
  Tensor buf = at::empty({n + words + 1}, like.options().dtype(at::kLong));
  int64_t* data = buf.data_ptr<int64_t>();
  return {buf.narrow(0, 0, n).view({B, 2 * R + 3}), data, scratch > 0 ? reinterpret_cast<int*>(data + n) : nullptr,
          reinterpret_cast<unsigned int*>(data + n + words)};
}

// One speculative-decoding iteration's greedy acceptance (speculative_sm90.cu): logits bf16 or fp32 [b, R, V]
// (contiguous), draft int64 [b, R - 1], unfinished int64 [b] (updated in place); eos < 0: no EOS.  Returns out int64
// [b, 2R + 3]: the argmaxes, the emitted tokens, a_b, n and the updated unfinished.
Tensor spec_accept(const Tensor& logits, const Tensor& draft, Tensor unfinished, int64_t eos, int64_t pad) {
  Args args("spec_accept");
  const auto [B, R, V] = spec_verify_args(args, logits, draft, unfinished);
  const auto guard = args.guard();
  const SpecOut o = spec_out(draft, B, R, 0);
  check(lb_spec_accept(logits.data_ptr(), logits.scalar_type() == at::kFloat ? 1 : 0, draft.data_ptr<int64_t>(),
                       unfinished.data_ptr<int64_t>(), o.data, o.counter, (int)B, (int)R, (int)V, (long long)eos,
                       (long long)pad, cur_stream()),
        "spec_accept");
  return o.out;
}

// The warp arguments of speculative sampling: temperature > 0 (finite), top_k >= 0 (0: off), 0 < top_p <= 1.
static void check_warp(const char* op, double temperature, int64_t top_k, double top_p) {
  TORCH_CHECK(std::isfinite(temperature) && temperature > 0, op, ": temperature must be a finite float > 0, got ",
              temperature);
  TORCH_CHECK(top_k >= 0 && top_k <= INT32_MAX, op, ": top_k must be >= 0 (0: off), got ", top_k);
  TORCH_CHECK(top_p > 0 && top_p <= 1, op, ": top_p must be in (0, 1], got ", top_p);
}

// One draft step of speculative sampling (speculative_sm90.cu): logits bf16 or fp32 [b, V] (contiguous) is kept in
// q[:, j] (q [b, K, V], the same dtype) and proposals[:, j] (int64 [b, J]) is drawn from its warped distribution with
// the uniforms u[:, j] (fp32 [b, J]).
void spec_sample(const Tensor& logits, Tensor q, int64_t j, const Tensor& u, Tensor proposals, double temperature,
                 int64_t top_k, double top_p) {
  Args args("spec_sample");
  args("logits", logits, Dtypes(at::kBFloat16, at::kFloat), {kAny, kAny});
  const int64_t B = logits.size(0), V = logits.size(1);
  TORCH_CHECK(B >= 1 && V >= 1 && V <= INT32_MAX, "spec_sample: logits [b, V] needs b >= 1 and V >= 1, got ",
              logits.sizes());
  args("q", q, logits.scalar_type(), {B, kAny, V});
  args("proposals", proposals, at::kLong, {B, kAny});
  const int64_t K = q.size(1), J = proposals.size(1);
  args("u", u, at::kFloat, {B, J});
  TORCH_CHECK(j >= 0 && j < K && j < J, "spec_sample: column j = ", j, " must be below q's ", K, " and proposals' ", J);
  check_warp("spec_sample", temperature, top_k, top_p);
  const auto guard = args.guard();
  check(lb_spec_sample(logits.data_ptr(), q.data_ptr(), logits.scalar_type() == at::kFloat ? 1 : 0, u.data_ptr<float>(),
                       proposals.data_ptr<int64_t>(), (int)B, (int)V, (int)K, (int)J, (int)j, (float)temperature,
                       (int)top_k, (float)top_p, cur_stream()),
        "spec_sample");
}

// One speculative-sampling iteration's acceptance (speculative_sm90.cu): logits bf16 or fp32 [b, R, V], q bf16 or
// fp32 [b, K, V] (the draft's rows, K >= R - 1), draft int64 [b, R - 1], u fp32 [b, R, 2], unfinished int64 [b]
// (updated in place), scores (optional) fp32 [b, R, V], written with the target's warped logits.  Returns out int64
// [b, 2R + 3] laid out as spec_accept's; the kernel keeps the per-row decisions in out's scratch.
Tensor spec_accept_sample(const Tensor& logits, const Tensor& q, const Tensor& draft, const Tensor& u,
                          Tensor unfinished, double temperature, int64_t top_k, double top_p, int64_t eos, int64_t pad,
                          c10::optional<Tensor> scores) {
  Args args("spec_accept_sample");
  const auto [B, R, V] = spec_verify_args(args, logits, draft, unfinished);
  args("q", q, Dtypes(at::kBFloat16, at::kFloat), {B, kAny, V});
  TORCH_CHECK(q.size(1) >= R - 1, "spec_accept_sample: q holds ", q.size(1), " draft rows, the iteration needs ", R - 1);
  args("u", u, at::kFloat, {B, R, 2});
  float* scores_ptr = args.opt<float>("scores", scores, at::kFloat, {B, R, V});
  check_warp("spec_accept_sample", temperature, top_k, top_p);
  const auto guard = args.guard();
  const SpecOut o = spec_out(draft, B, R, B * R);
  check(lb_spec_accept_sample(logits.data_ptr(), logits.scalar_type() == at::kFloat ? 1 : 0, q.data_ptr(),
                              q.scalar_type() == at::kFloat ? 1 : 0, draft.data_ptr<int64_t>(), u.data_ptr<float>(),
                              unfinished.data_ptr<int64_t>(), o.data, o.scratch, o.counter, scores_ptr, (int)B,
                              (int)R, (int)V, (int)q.size(1), (float)temperature, (int)top_k, (float)top_p,
                              (long long)eos, (long long)pad, cur_stream()),
        "spec_accept_sample");
  return o.out;
}

// per-tensor E4M3 quantisation of a contiguous bf16 tensor: returns (q [same shape, float8_e4m3fn], deq fp32 [1]) with
// x ≈ q * deq (deq = amax / 448); two kernels, no host synchronisation
std::tuple<Tensor, Tensor> quantize_e4m3(const Tensor& x) {
  Args args("quantize_e4m3");
  args("x", x, at::kBFloat16, x.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
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
  TORCH_CHECK(!given(residual) || (act == 0 && !want_pre),
              "linear_fp8_fwd: a residual epilogue takes no activation and no pre-activation copy");
  Args args("linear_fp8_fwd");
  args("xq", xq, at::kFloat8_e4m3fn, {kAny, kAny});
  args("wq", wq, at::kFloat8_e4m3fn, {kAny, xq.size(1)});
  args("deq_x", deq_x, at::kFloat, {1});
  args("deq_w", deq_w, at::kFloat, {1});
  const int64_t M = xq.size(0), K = xq.size(1), N = wq.size(0);
  TORCH_CHECK(K % 16 == 0 && N % 8 == 0, "linear_fp8_fwd: K % 16 == 0 and N % 8 == 0 required");
  const void* bias_ptr = args.opt("bias", bias, at::kBFloat16, {N});
  const void* res_ptr = args.opt("residual", residual, at::kBFloat16, {M, N});
  const auto guard = args.guard();
  auto opts = xq.options().dtype(at::kBFloat16);
  Tensor y = at::empty({M, N}, opts);
  Tensor pre = want_pre ? at::empty({M, N}, opts) : Tensor();
  check(lb_gemm_fp8(xq.data_ptr(), wq.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, bias_ptr, (int)act,
                    pre.defined() ? pre.data_ptr() : nullptr, res_ptr, deq_x.data_ptr<float>(), deq_w.data_ptr<float>(),
                    (int)bn, cur_stream()),
        "linear_fp8_fwd");
  return std::make_tuple(y, pre.defined() ? pre : at::empty({0}, opts));
}

// raw entry used by tests / autotuning: explicit tile-N and split-K
Tensor gemm_tuned(const Tensor& a, const Tensor& b, int64_t layout, int64_t bn, int64_t splits, bool fp32_out) {
  Args args("gemm_tuned");
  const auto [M, N, K] = gemm_operands(args, a, b, layout);
  const auto guard = args.guard();
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
  Args args("act_bwd");
  args("gy", gy, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  args("pre", pre, at::kBFloat16, gy.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor gx = at::empty_like(gy);
  check(lb_bias_act_bwd(gy.data_ptr(), pre.data_ptr(), nullptr, gx.data_ptr(), gy.size(0), (int)gy.size(1), (int)act,
                        cur_stream()),
        "act_bwd");
  return gx;
}

// embedding lookup on a (vocabulary shard of a) bf16 table; ids int64 (any shape) -> [ids.numel(), H]
Tensor embedding_fwd(const Tensor& ids, const Tensor& table, int64_t vocab_start) {
  Args args("embedding_fwd");
  args("table", table, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  args("ids", ids, at::kLong, ids.sizes());
  const auto guard = args.guard();
  const int64_t T = ids.numel(), H = table.size(1);
  Tensor out = at::empty({T, H}, table.options());
  check(lb_embedding_fwd(ids.data_ptr<int64_t>(), table.data_ptr(), out.data_ptr(), (long)T, (int)H, (long)vocab_start,
                         (long)table.size(0), cur_stream()),
        "embedding_fwd");
  return out;
}
// grad[ids - vocab_start] += gy   (grad: the parameter's fp32 main-grad view, same shape as the table)
void embedding_bwd(const Tensor& ids, const Tensor& gy, Tensor grad, int64_t vocab_start) {
  Args args("embedding_bwd");
  args("gy", gy, at::kBFloat16, {ids.numel(), kAny}, Layout::Contiguous, 16);
  args("ids", ids, at::kLong, ids.sizes());
  args("grad", grad, at::kFloat, {kAny, gy.size(1)}, Layout::Contiguous, 16);
  const auto guard = args.guard();
  const auto sorted = at::sort(ids.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
  check(lb_embedding_bwd(std::get<0>(sorted).data_ptr<int64_t>(), std::get<1>(sorted).data_ptr<int64_t>(), gy.data_ptr(),
                         grad.data_ptr<float>(), (long)ids.numel(), (int)gy.size(1), (long)vocab_start, (long)grad.size(0),
                         cur_stream()),
        "embedding_bwd");
}

// column sums of a bf16 [M, N] tensor.  With `accum` (fp32 [N], e.g. a bias' slice of the flat main-grad buffer) the
// sums are added into it and an empty tensor is returned; otherwise a fresh bf16 [N] tensor.
Tensor colsum(const Tensor& x, const c10::optional<Tensor>& accum) {
  Args args("colsum");
  args("x", x, at::kBFloat16, {kAny, kAny});
  const int64_t M = x.size(0), N = x.size(1);
  float* acc = args.opt<float>("accum", accum, at::kFloat, {N});
  const auto guard = args.guard();
  Tensor out = acc != nullptr ? Tensor() : at::empty({N}, x.options().dtype(at::kFloat));
  Tensor ws = at::empty({(int64_t)lb_colsum_workspace_rows((int)M, (int)N) * N}, x.options().dtype(at::kFloat));
  check(lb_colsum(x.data_ptr(), acc != nullptr ? acc : out.data_ptr<float>(), (int)M, (int)N, acc != nullptr ? 1 : 0,
                  ws.data_ptr<float>(), cur_stream()),
        "colsum");
  return acc != nullptr ? at::empty({0}, x.options()) : out.to(at::kBFloat16);
}

// ---- norms ----------------------------------------------------------------------------------------
// The kernels read H elements of γ (and β) with no bounds of their own and are built for the (x, γ) dtype pairs
// (bf16, bf16), (bf16, fp32) and (fp32, fp32).
void norm_args(Args& args, const Tensor& x, const Tensor& gamma, const Tensor* beta) {
  const char* what = args.op();
  args("x", x, {at::kBFloat16, at::kFloat}, {kAny, kAny});
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
  Args args("norm_fwd");
  norm_args(args, x, gamma, given(beta) ? &beta.value() : nullptr);
  const auto guard = args.guard();
  const int rows = (int)x.size(0), H = (int)x.size(1);
  Tensor y = at::empty_like(x);
  Tensor mean = rms ? at::empty({0}, x.options().dtype(at::kFloat)) : at::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = at::empty({rows}, x.options().dtype(at::kFloat));
  const void* b = given(beta) ? beta->data_ptr() : nullptr;
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
  Args args("norm_bwd");
  norm_args(args, x, gamma, nullptr);
  const int rows = (int)x.size(0), H = (int)x.size(1);
  args("gy", gy, x.scalar_type(), x.sizes());
  if (!rms) args("mean", mean, at::kFloat, {rows});
  args("rstd", rstd, at::kFloat, {rows});
  // accumulate mode: dgamma / dbeta are added straight into the fp32 main-grad slices of the parameters
  const bool acc = given(dgamma_accum);
  if (acc) {
    args("dgamma_accum", *dgamma_accum, at::kFloat, {H});
    TORCH_CHECK(!has_bias || given(dbeta_accum), "norm_bwd: dbeta_accum must be given with dgamma_accum when has_bias");
    if (has_bias) args("dbeta_accum", *dbeta_accum, at::kFloat, {H});
  }
  // optional gradient of the skip connection around this norm: added to gx inside the kernel when supported
  args.opt("gadd", gadd, kAnyDtype, x.sizes(), Layout::Strided);
  const bool fuse_add = given(gadd) && lb_norm_bwd_supports_gadd(H) && gadd->is_contiguous() &&
                        gadd->scalar_type() == x.scalar_type();
  const auto guard = args.guard();
  Tensor gx = at::empty_like(x);
  auto fopt = x.options().dtype(at::kFloat);
  Tensor dgamma = acc ? dgamma_accum.value() : at::empty({H}, fopt);
  Tensor dbeta = !has_bias ? at::empty({0}, fopt) : (acc ? dbeta_accum.value() : at::empty({H}, fopt));
  const int wrows = lb_norm_bwd_workspace_rows(rows);
  Tensor ws = at::empty({2 * (int64_t)wrows * H}, fopt);
  check(lb_norm_bwd(gy.data_ptr(), x.data_ptr(), gamma.data_ptr(), rms ? nullptr : mean.data_ptr<float>(),
                    rstd.data_ptr<float>(), gx.data_ptr(), dgamma.data_ptr<float>(),
                    has_bias ? dbeta.data_ptr<float>() : nullptr, ws.data_ptr<float>(), rows, H, rms ? 1 : 0,
                    dtype_code(x), dtype_code(gamma), acc ? 1 : 0, fuse_add ? gadd->data_ptr() : nullptr, cur_stream()),
        "norm_bwd");
  if (given(gadd) && !fuse_add) gx.add_(gadd->to(gx.scalar_type()));
  if (acc) return std::make_tuple(gx, at::empty({0}, fopt), at::empty({0}, fopt));
  return std::make_tuple(gx, dgamma, dbeta);
}

// ---- elementwise ------------------------------------------------------------------------------------
// The kernels load 8 bf16 values at a time from every operand: each is 16-byte aligned and, but for the [N] bias,
// contiguous [rows, N] (N % 8 == 0, which the launchers check).
Tensor bias_act_fwd(const Tensor& x, const c10::optional<Tensor>& bias, int64_t act) {
  Args args("bias_act_fwd");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  const void* b = args.opt("bias", bias, at::kBFloat16, {x.size(1)}, Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor y = at::empty_like(x);
  check(lb_bias_act_fwd(x.data_ptr(), b, y.data_ptr(), x.size(0), (int)x.size(1), (int)act, cur_stream()), "bias_act_fwd");
  return y;
}
Tensor bias_act_bwd(const Tensor& gy, const Tensor& x, const c10::optional<Tensor>& bias, int64_t act) {
  Args args("bias_act_bwd");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  args("gy", gy, at::kBFloat16, x.sizes(), Layout::Contiguous, 16);
  const void* b = args.opt("bias", bias, at::kBFloat16, {x.size(1)}, Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor gx = at::empty_like(x);
  check(lb_bias_act_bwd(gy.data_ptr(), x.data_ptr(), b, gx.data_ptr(), x.size(0), (int)x.size(1), (int)act, cur_stream()),
        "bias_act_bwd");
  return gx;
}
Tensor bias_residual_fwd(const Tensor& x, const c10::optional<Tensor>& bias, const c10::optional<Tensor>& res) {
  Args args("bias_residual_fwd");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  const void* b = args.opt("bias", bias, at::kBFloat16, {x.size(1)}, Layout::Contiguous, 16);
  const void* r = args.opt("res", res, at::kBFloat16, x.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor y = at::empty_like(x);
  check(lb_bias_residual(x.data_ptr(), b, r, y.data_ptr(), x.size(0), (int)x.size(1), cur_stream()), "bias_residual");
  return y;
}
Tensor swiglu_fwd(const Tensor& gate, const Tensor& up) {
  Args args("swiglu_fwd");
  args("gate", gate, at::kBFloat16, gate.sizes(), Layout::Contiguous, 16);
  args("up", up, at::kBFloat16, gate.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor y = at::empty_like(gate);
  check(lb_swiglu_fwd(gate.data_ptr(), up.data_ptr(), y.data_ptr(), gate.numel(), cur_stream()), "swiglu_fwd");
  return y;
}
std::tuple<Tensor, Tensor> swiglu_bwd(const Tensor& gy, const Tensor& gate, const Tensor& up) {
  Args args("swiglu_bwd");
  args("gate", gate, at::kBFloat16, gate.sizes(), Layout::Contiguous, 16);
  args("up", up, at::kBFloat16, gate.sizes(), Layout::Contiguous, 16);
  args("gy", gy, at::kBFloat16, gate.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor dg = at::empty_like(gate), du = at::empty_like(up);
  check(lb_swiglu_bwd(gy.data_ptr(), gate.data_ptr(), up.data_ptr(), dg.data_ptr(), du.data_ptr(), gate.numel(),
                      cur_stream()),
        "swiglu_bwd");
  return std::make_tuple(dg, du);
}
// gu [T, 2F] = [gate | up] (one GEMM against the stacked gate / up weights) -> silu(gate) * up  [T, F]
void swiglu_packed_args(Args& args, const Tensor& gu) {
  args("gu", gu, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  TORCH_CHECK(gu.size(1) % 16 == 0, args.op(), ": gu [T, 2F] needs F % 8 == 0, got ", gu.sizes());
}
Tensor swiglu_packed_fwd(const Tensor& gu) {
  Args args("swiglu_packed_fwd");
  swiglu_packed_args(args, gu);
  const auto guard = args.guard();
  Tensor y = at::empty({gu.size(0), gu.size(1) / 2}, gu.options());
  check(lb_swiglu_packed_fwd(gu.data_ptr(), y.data_ptr(), gu.size(0), gu.size(1) / 2, cur_stream()), "swiglu_packed_fwd");
  return y;
}
Tensor swiglu_packed_bwd(const Tensor& gy, const Tensor& gu) {
  Args args("swiglu_packed_bwd");
  swiglu_packed_args(args, gu);
  args("gy", gy, at::kBFloat16, {gu.size(0), gu.size(1) / 2}, Layout::Contiguous, 16);
  const auto guard = args.guard();
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

// the cos / sin tables of a rotary embedding: fp32 [>= min_rows, D] of one shape
void rope_tables(Args& args, const Tensor& cosv, const Tensor& sinv, int64_t min_rows, int64_t D) {
  args("cos/sin", cosv, at::kFloat, {kAny, D});
  args("cos/sin", sinv, at::kFloat, cosv.sizes());
  TORCH_CHECK(cosv.size(0) >= min_rows, args.op(), ": cos/sin must have at least ", min_rows, " rows, got ",
              cosv.sizes());
}

// packed projection [b, s, a, 3d] or [b, s, g, r + 2, d]; rotates every q and k (v copied).  inplace=true rewrites qkv
// itself.  positions (optional, int32 [b, s]): the position of every token (packed sequences), instead of
// s + pos_offset; values outside the tables are clamped to them.
Tensor rope_qkv(const Tensor& qkv, const Tensor& cosv, const Tensor& sinv, int64_t pos_offset, bool backward,
                bool inplace, const c10::optional<Tensor>& positions) {
  Args args("rope_qkv");
  args("qkv", qkv, at::kBFloat16, qkv.sizes());
  const PackedQKV g = packed_qkv(qkv, "rope_qkv");
  const int S = g.S, D = g.D;
  TORCH_CHECK(D % 2 == 0, "rope_qkv: head dim must be even");
  const int* pos = args.opt<const int>("positions", positions, at::kInt, {g.B, S});
  rope_tables(args, cosv, sinv, pos != nullptr ? 1 : S + pos_offset, D);
  const auto guard = args.guard();
  Tensor y = inplace ? qkv : at::empty_like(qkv);
  check(lb_rope_qkv(qkv.data_ptr(), cosv.data_ptr<float>(), sinv.data_ptr<float>(), y.data_ptr(),
                    qkv.numel() / ((g.r + 2) * D), S, g.G, g.r, D, (int)pos_offset, pos, (int)cosv.size(0),
                    backward ? 1 : 0, cur_stream()),
        "rope_qkv");
  return y;
}

// ChatGLM rotary: the fused projection [b, s, (a + 2g) * d] <-> the packed layouts the attention kernels read (grouped
// [b, s, g, a/g + 2, d] or per-head [b, s, a, 3d]).  `name` names the input in the errors.
struct GlmRotary {
  int B, S, A, G, D;
  const int* positions;
};
GlmRotary glm_rotary_args(Args& args, const char* name, const Tensor& t, int64_t B, int64_t S, int64_t heads,
                          int64_t kv_heads, int64_t D, const Tensor& table, int64_t pos_offset,
                          const c10::optional<Tensor>& position_ids) {
  const char* what = args.op();
  TORCH_CHECK(t.scalar_type() == at::kBFloat16, what, ": bf16 input expected, got ", t.scalar_type());
  TORCH_CHECK(t.is_contiguous(), what, ": contiguous input expected");
  args(name, t, at::kBFloat16, t.sizes());
  TORCH_CHECK(heads > 0 && kv_heads > 0 && heads % kv_heads == 0, what, ": heads (", heads,
              ") must be a positive multiple of kv_heads (", kv_heads, ")");
  TORCH_CHECK(D > 0 && D % 4 == 0, what, ": head dim must be a positive multiple of 4, got ", D);
  TORCH_CHECK(S > 0, what, ": empty sequence");
  args("table", table, at::kFloat, {kAny, D / 4, 2});
  TORCH_CHECK(!given(position_ids) || position_ids->scalar_type() == at::kInt, what, ": int32 position_ids expected, got ",
              position_ids->scalar_type());
  GlmRotary g{(int)B, (int)S, (int)heads, (int)kv_heads, (int)D, nullptr};
  g.positions = args.opt<const int>("position_ids", position_ids, at::kInt, {B, S});
  const int64_t P = table.size(0);
  TORCH_CHECK(g.positions != nullptr || (pos_offset >= 0 && pos_offset + S <= P), what, ": positions [", pos_offset,
              ", ", pos_offset + S, ") exceed the table's ", P, " rows");
  return g;
}
// every sample takes the positions of the first row (one host sync, after the other checks)
void check_glm_positions(const char* what, const c10::optional<Tensor>& position_ids, int64_t P) {
  if (!given(position_ids)) return;
  const auto [lo, hi] = at::aminmax(position_ids->select(0, 0));
  const int64_t mn = lo.item<int64_t>(), mx = hi.item<int64_t>();
  TORCH_CHECK(mn >= 0 && mx < P, what, ": position_ids must lie in [0, ", P, "), got [", mn, ", ", mx, "]");
}

// pos_base (optional, int32 [>= 1], not with position_ids): token i sits at pos_base[0] + pos_offset + i, read on the
// device (a decoding step's cache length, e.g. cache_seqlens; a captured step then replays at the current length).
// Like the lengths of kv_append, those positions are the caller's guarantee.
Tensor glm_rotary_qkv(const Tensor& mixed, int64_t heads, int64_t kv_heads, const Tensor& table, int64_t pos_offset,
                      const c10::optional<Tensor>& position_ids, bool grouped, const c10::optional<Tensor>& pos_base) {
  TORCH_CHECK(mixed.dim() == 3, "glm_rotary_qkv: fused projection [b, s, (a + 2g) * d] expected, got ", mixed.sizes());
  TORCH_CHECK(heads > 0 && kv_heads > 0 && mixed.size(2) % (heads + 2 * kv_heads) == 0, "glm_rotary_qkv: last dim ",
              mixed.size(2), " is not (heads + 2 * kv_heads) * d");
  TORCH_CHECK(!(given(pos_base) && given(position_ids)),
              "glm_rotary_qkv: position_ids and pos_base exclude each other");
  const int64_t B = mixed.size(0), S = mixed.size(1), D = mixed.size(2) / (heads + 2 * kv_heads);
  Args args("glm_rotary_qkv");
  // (the host-side range check of pos_offset does not apply to a device-side base)
  const GlmRotary g = glm_rotary_args(args, "mixed", mixed, B, S, heads, kv_heads, D, table,
                                      given(pos_base) ? 0 : pos_offset, position_ids);
  const int* base = args.opt<const int>("pos_base", pos_base, at::kInt, {kAny});
  TORCH_CHECK(base == nullptr || pos_base->numel() >= 1, "glm_rotary_qkv: pos_base must hold at least one element");
  const auto guard = args.guard();
  check_glm_positions("glm_rotary_qkv", position_ids, table.size(0));
  Tensor out = grouped ? at::empty({B, S, kv_heads, heads / kv_heads + 2, D}, mixed.options())
                       : at::empty({B, S, heads, 3 * D}, mixed.options());
  check(lb_glm_rotary_qkv(mixed.data_ptr(), table.data_ptr<float>(), out.data_ptr(), B * S, g.S, g.A, g.G, g.D,
                          (int)pos_offset, g.positions, base, grouped ? 1 : 0, 0, cur_stream()),
        "glm_rotary_qkv");
  return out;
}

// grad: the gradient of glm_rotary_qkv's output (its rank tells the layout) -> the gradient of the fused projection
Tensor glm_rotary_qkv_bwd(const Tensor& grad, int64_t heads, int64_t kv_heads, const Tensor& table, int64_t pos_offset,
                          const c10::optional<Tensor>& position_ids, const c10::optional<Tensor>& pos_base) {
  const bool grouped = grad.dim() == 5;
  TORCH_CHECK(heads > 0 && kv_heads > 0 && heads % kv_heads == 0, "glm_rotary_qkv_bwd: heads (", heads,
              ") must be a positive multiple of kv_heads (", kv_heads, ")");
  TORCH_CHECK(grad.dim() == 4 || grad.dim() == 5, "glm_rotary_qkv_bwd: gradient [b, s, g, a/g + 2, d] or [b, s, a, 3d] "
              "expected, got ", grad.sizes());
  TORCH_CHECK((grouped && grad.size(2) == kv_heads && grad.size(3) == heads / kv_heads + 2) ||
                  (grad.dim() == 4 && grad.size(2) == heads && grad.size(3) % 3 == 0),
              "glm_rotary_qkv_bwd: gradient [b, s, g, a/g + 2, d] or [b, s, a, 3d] expected, got ", grad.sizes());
  TORCH_CHECK(!(given(pos_base) && given(position_ids)),
              "glm_rotary_qkv_bwd: position_ids and pos_base exclude each other");
  const int64_t B = grad.size(0), S = grad.size(1), D = grouped ? grad.size(4) : grad.size(3) / 3;
  Args args("glm_rotary_qkv_bwd");
  const GlmRotary g = glm_rotary_args(args, "grad", grad, B, S, heads, kv_heads, D, table,
                                      given(pos_base) ? 0 : pos_offset, position_ids);
  const int* base = args.opt<const int>("pos_base", pos_base, at::kInt, {kAny});
  TORCH_CHECK(base == nullptr || pos_base->numel() >= 1, "glm_rotary_qkv_bwd: pos_base must hold at least one element");
  const auto guard = args.guard();
  check_glm_positions("glm_rotary_qkv_bwd", position_ids, table.size(0));
  Tensor dmixed = at::empty({B, S, (heads + 2 * kv_heads) * D}, grad.options());
  check(lb_glm_rotary_qkv(grad.data_ptr(), table.data_ptr<float>(), dmixed.data_ptr(), B * S, g.S, g.A, g.G, g.D,
                          (int)pos_offset, g.positions, base, grouped ? 1 : 0, 1, cur_stream()),
        "glm_rotary_qkv_bwd");
  return dmixed;
}

// ---- cross entropy ------------------------------------------------------------------------------------
// logits bf16 or fp32 [T, V], labels int64 [T]
void ce_args(Args& args, const Tensor& logits, const Tensor& labels) {
  args("logits", logits, {at::kBFloat16, at::kFloat}, {kAny, kAny});
  args("labels", labels, at::kLong, {logits.size(0)});
}
std::tuple<Tensor, Tensor, Tensor> ce_stats(const Tensor& logits, const Tensor& labels, int64_t vocab_start) {
  Args args("ce_stats");
  ce_args(args, logits, labels);
  const auto guard = args.guard();
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  auto fopt = logits.options().dtype(at::kFloat);
  Tensor mx = at::empty({T}, fopt), se = at::empty({T}, fopt), tgt = at::empty({T}, fopt);
  check(lb_ce_stats(logits.data_ptr(), labels.data_ptr<int64_t>(), mx.data_ptr<float>(), se.data_ptr<float>(),
                    tgt.data_ptr<float>(), T, V, (long)vocab_start, dtype_code(logits), cur_stream()),
        "ce_stats");
  return std::make_tuple(mx, se, tgt);
}
Tensor ce_bwd(const Tensor& logits, const Tensor& labels, const Tensor& lse, const Tensor& gloss, int64_t vocab_start) {
  Args args("ce_bwd");
  ce_args(args, logits, labels);
  const int T = (int)logits.size(0), V = (int)logits.size(1);
  args("lse", lse, at::kFloat, {T});
  args("gloss", gloss, at::kFloat, {T});
  const auto guard = args.guard();
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
  Args args("fused_adamw");
  args("master", master, at::kFloat, master.sizes(), Layout::Contiguous, 16);
  args("grad", grad, at::kFloat, master.sizes(), Layout::Contiguous, 16);
  args("m", m, at::kFloat, master.sizes(), Layout::Contiguous, 16);
  args("v", v, at::kFloat, master.sizes(), Layout::Contiguous, 16);
  TORCH_CHECK(master.numel() % 4 == 0, "fused_adamw: numel must be a multiple of 4");
  args("scale", scale, at::kFloat, {1});
  void* lp = args.opt<void>("lp_out", lp_out, {at::kBFloat16, at::kHalf}, master.sizes(), Layout::Contiguous, 8);
  const int lp_dtype = lp != nullptr && lp_out->scalar_type() == at::kHalf ? 1 : 0;
  const auto guard = args.guard();
  check(lb_adamw(master.data_ptr<float>(), grad.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), lp, lp_dtype,
                 scale.data_ptr<float>(), master.numel(), (float)lr, (float)b1, (float)b2, (float)eps, (float)wd,
                 (float)bc1, (float)bc2, decoupled ? 1 : 0, cur_stream()),
        "fused_adamw");
}
Tensor sqnorm(const Tensor& x) {
  Args args("sqnorm");
  args("x", x, at::kFloat, x.sizes(), Layout::Contiguous, 16);
  const auto guard = args.guard();
  Tensor out = at::zeros({1}, x.options().dtype(at::kFloat));
  Tensor ws = at::empty({(int64_t)lb_sqnorm_workspace(x.numel())}, x.options().dtype(at::kFloat));
  check(lb_sqnorm(x.data_ptr<float>(), out.data_ptr<float>(), x.numel(), ws.data_ptr<float>(), cur_stream()), "sqnorm");
  return out;
}

// ---- dropout RNG ---------------------------------------------------------------------------------------------
// (seed, offset) of the default CUDA generator, advanced by `increment`; graph-capture aware (pointers + intra-graph
// offset while capturing — PyTorch refreshes the pointed-to values before every replay).  `salt` != 0 decorrelates
// tensor-parallel ranks in sharded regions.
lb::RngArgs next_rng(int64_t salt, uint64_t increment = 4) {
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(c10::nullopt, at::cuda::detail::getDefaultCUDAGenerator());
  at::PhiloxCudaState st;
  {
    std::lock_guard<std::mutex> lock(gen->mutex_);
    st = gen->philox_cuda_state(increment);
  }
  lb::RngArgs a;
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
  Args args("bias_dropout_residual");
  args("x", x, at::kBFloat16, {kAny, kAny}, Layout::Contiguous, 16);
  const void* bptr = args.opt("bias", bias, at::kBFloat16, {x.size(1)}, Layout::Contiguous, 16);
  const void* rptr = args.opt("res", res, at::kBFloat16, x.sizes(), Layout::Contiguous, 16);
  const auto* rng_in = args.opt<const long long>("rng_state", rng_state, at::kLong, {2});
  TORCH_CHECK(p >= 0.0 && p < 1.0, "dropout probability must be in [0, 1)");
  const auto guard = args.guard();
  Tensor y = at::empty_like(x);
  if (rng_in != nullptr) {
    check(lb_bias_dropout_residual(x.data_ptr(), bptr, rptr, y.data_ptr(), x.size(0), (int)x.size(1), (float)p, nullptr,
                                   rng_in, nullptr, cur_stream()),
          "bias_dropout_residual");
    return std::make_tuple(y, *rng_state);
  }
  Tensor st = at::empty({2}, x.options().dtype(at::kLong));
  lb::RngArgs a = next_rng(salt);
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
// j <= i + Sk - Sq or j < prefix_lens[b].

// One flash-attention problem, validated: q, k, v as above, bf16; kv_lens / kv_start / prefix_lens int32 [B]; doc_start
// int32 [B, Sq] (packed sequences); bias bf16 [B|1, A|1, Sq, Sk] with contiguous keys (broadcast dims get stride 0);
// alibi_slopes fp32 [A]; p_drop in [0, 1).
lb::AttnArgs attn_args(Args& args, const Tensor& q, const Tensor& k, const Tensor& v, bool causal, double scale,
                       const c10::optional<Tensor>& kv_lens, const c10::optional<Tensor>& kv_start,
                       const c10::optional<Tensor>& doc_start, const c10::optional<Tensor>& bias,
                       const c10::optional<Tensor>& alibi_slopes, double p_drop,
                       const c10::optional<Tensor>& prefix_lens) {
  const char* what = args.op();
  TORCH_CHECK(q.dim() == 4 || q.dim() == 5, what, ": q must be [B, A, S, D] or [B, G, r, S, D]");
  args("q", q, at::kBFloat16, q.sizes(), Layout::LastDimContiguous);
  args("k", k, at::kBFloat16, {q.size(0), kAny, kAny, q.size(-1)}, Layout::LastDimContiguous);
  args("v", v, at::kBFloat16, k.sizes(), Layout::LastDimContiguous);
  lb::AttnArgs a{};
  a.B = (int)q.size(0);
  a.G = (int)k.size(1);
  a.Sq = (int)q.size(-2);
  a.Sk = (int)k.size(2);
  a.d = (int)q.size(-1);
  if (q.dim() == 4) {
    a.A = (int)q.size(1);
    TORCH_CHECK(a.G > 0 && a.A % a.G == 0, what, ": the query heads must be a multiple of the K/V heads");
    const long r = a.A / a.G;
    a.q_strides[0] = q.stride(0);
    a.q_strides[1] = r * q.stride(1);
    a.q_strides[2] = q.stride(1);
    a.q_strides[3] = q.stride(2);
  } else {
    TORCH_CHECK(q.size(1) == a.G, what, ": grouped q [B, G, r, S, D] must have the K/V heads' G");
    a.A = a.G * (int)q.size(2);
    for (int i = 0; i < 4; ++i) a.q_strides[i] = q.stride(i);
  }
  TORCH_CHECK(a.d % 8 == 0 && a.d >= 8 && a.d <= 128, what, ": head dim must be a multiple of 8 in [8, 128], got ", a.d);
  TORCH_CHECK(a.Sq >= 1 && a.Sk >= 1, what, ": empty query or key sequence");
  for (int i = 0; i < 3; ++i) {
    a.k_strides[i] = k.stride(i);
    a.v_strides[i] = v.stride(i);
  }
  a.causal = causal;
  a.scale = (float)scale;
  // per-sample key bound (kv_lens: end, kv_start: start of the visible keys)
  a.kv_lens = args.opt<const int>("kv_lens", kv_lens, at::kInt, {a.B});
  a.kv_start = args.opt<const int>("kv_start", kv_start, at::kInt, {a.B});
  a.doc_start = args.opt<const int>("doc_start", doc_start, at::kInt, {a.B, a.Sq});
  a.prefix_lens = args.opt<const int>("prefix_lens", prefix_lens, at::kInt, {a.B});
  if (given(bias)) {
    const Tensor& b = args("bias", *bias, at::kBFloat16, {kAny, kAny, a.Sq, a.Sk}, Layout::LastDimContiguous);
    TORCH_CHECK((b.size(0) == 1 || b.size(0) == a.B) && (b.size(1) == 1 || b.size(1) == a.A), what,
                ": attention bias: bad broadcast shape");
    a.bias = b.data_ptr();
    a.bias_strides[0] = b.size(0) == 1 ? 0 : b.stride(0);
    a.bias_strides[1] = b.size(1) == 1 ? 0 : b.stride(1);
    a.bias_strides[2] = b.stride(2);
  }
  a.alibi_slopes = args.opt<const float>("alibi_slopes", alibi_slopes, at::kFloat, {a.A});
  TORCH_CHECK(p_drop < 1.0, "dropout probability must be in [0, 1)");
  a.p_drop = (float)p_drop;
  TORCH_CHECK(a.doc_start == nullptr || lb::attn_doc_start_supported(a), what,
              ": doc_start: supported for causal self-attention (Sq == Sk) without kv_lens, kv_start, bias, ALiBi or "
              "dropout");
  TORCH_CHECK(a.prefix_lens == nullptr || lb::attn_prefix_supported(a), what,
              ": prefix_lens: supported for causal attention, with kv_lens, kv_start, grouped-query heads and dropout, "
              "without bias, ALiBi or doc_start");
  return a;
}

// returns (o, lse, rng_state): rng_state int64[2] = (seed, offset) of the dropout mask (empty without dropout)
std::tuple<Tensor, Tensor, Tensor> attn_fwd(const Tensor& q, const Tensor& k, const Tensor& v, bool causal, double scale,
                                            const c10::optional<Tensor>& kv_lens, const c10::optional<Tensor>& bias,
                                            const c10::optional<Tensor>& alibi_slopes, double p_drop, int64_t salt,
                                            const c10::optional<Tensor>& kv_start, const c10::optional<Tensor>& doc_start,
                                            const c10::optional<Tensor>& prefix_lens) {
  Args args("attn_fwd");
  const lb::AttnArgs a = attn_args(args, q, k, v, causal, scale, kv_lens, kv_start, doc_start, bias, alibi_slopes, p_drop,
                                   prefix_lens);
  const auto guard = args.guard();
  Tensor o = at::empty({a.B, a.Sq, a.A, a.d}, q.options());
  Tensor lse = at::empty({a.B, a.A, a.Sq}, q.options().dtype(at::kFloat));
  const bool drop = p_drop > 0.0;
  Tensor rng_state = at::empty({drop ? 2 : 0}, q.options().dtype(at::kLong));
  lb::RngArgs rng{};
  if (drop) rng = next_rng(salt);
  check(lb_attn_fwd(&a, q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr<float>(),
                    drop ? &rng : nullptr, drop ? reinterpret_cast<long long*>(rng_state.data_ptr<int64_t>()) : nullptr,
                    cur_stream()),
        "attn_fwd");
  return std::make_tuple(o.permute({0, 2, 1, 3}), lse, rng_state);
}

// Causal flash attention of q [B, Sq, A, D] (the new tokens, appended already; any strides with D contiguous) over the
// logical rows [0, past + Sq) of a paged cache: contiguous bf16 pools [P, G, 64, D] (D 64 or 128, A a multiple of G)
// read through block_table int32 [B, max_pages] (max_pages * 64 >= past + Sq).  kv_start int32 [B] (left padding) and
// alibi_slopes fp32 [A] as in attn_fwd.  The table entries of those rows are the caller's guarantee (an entry outside
// [0, P) reads as zero rows).  Returns o [B, Sq, A, D] contiguous.
Tensor attn_fwd_paged(const Tensor& q, const Tensor& k_pool, const Tensor& v_pool, const Tensor& block_table,
                      int64_t past, double scale, const c10::optional<Tensor>& kv_start,
                      const c10::optional<Tensor>& alibi_slopes) {
  Args args("attn_fwd_paged");
  args("q", q, at::kBFloat16, {kAny, kAny, kAny, kAny}, Layout::LastDimContiguous, 16);
  const int64_t D = q.size(3);
  TORCH_CHECK(D == 64 || D == 128, "attn_fwd_paged: head dim must be 64 or 128, got ", D);
  args("k_pool", k_pool, at::kBFloat16, {kAny, kAny, 64, D});
  args("v_pool", v_pool, at::kBFloat16, k_pool.sizes());
  args("block_table", block_table, at::kInt, {q.size(0), kAny});
  lb::AttnArgs a{};
  a.B = (int)q.size(0);
  a.Sq = (int)q.size(1);
  a.A = (int)q.size(2);
  a.G = (int)k_pool.size(1);
  a.d = (int)D;
  TORCH_CHECK(a.G > 0 && a.A % a.G == 0, "attn_fwd_paged: the query heads must be a multiple of the K/V heads");
  TORCH_CHECK(k_pool.size(0) >= 1 && k_pool.size(0) <= INT32_MAX, "attn_fwd_paged: 1 <= pages <= INT32_MAX");
  TORCH_CHECK(past >= 0 && a.Sq >= 1 && past + a.Sq <= block_table.size(1) * 64, "attn_fwd_paged: the rows [0, past + ",
              "Sq) must fit the block table's ", block_table.size(1), " pages, got past = ", past, ", Sq = ", a.Sq);
  a.Sk = (int)(past + a.Sq);
  const long r = a.A / a.G;
  a.q_strides[0] = q.stride(0);
  a.q_strides[1] = r * q.stride(2);
  a.q_strides[2] = q.stride(2);
  a.q_strides[3] = q.stride(1);
  for (int i = 0; i < 3; ++i) a.k_strides[i] = a.v_strides[i] = k_pool.stride(i);
  a.causal = true;
  a.scale = (float)scale;
  a.kv_start = args.opt<const int>("kv_start", kv_start, at::kInt, {a.B});
  a.alibi_slopes = args.opt<const float>("alibi_slopes", alibi_slopes, at::kFloat, {a.A});
  const auto guard = args.guard();
  Tensor o = at::empty({a.B, a.Sq, a.A, a.d}, q.options());
  Tensor lse = at::empty({a.B, a.A, a.Sq}, q.options().dtype(at::kFloat));
  check(lb_attn_fwd_paged(&a, q.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), (int)k_pool.size(0),
                          block_table.data_ptr<int>(), (int)block_table.size(1), o.data_ptr(), lse.data_ptr<float>(),
                          cur_stream()),
        "attn_fwd_paged");
  return o;
}

// The causal flash attention of N ragged sequences packed in q [T, A, D] (any strides with D contiguous) over their
// logical rows of a paged cache's bf16 pools [P, G, 64, D]: sequence n owns the rows cu_q[n] .. cu_q[n + 1] of q and
// holds past[n] rows before them in row n of block_table int32 [N, max_pages] (cu_q int32 [N + 1], past int32 [N]).
// tiles int32 [n_tiles, 2] lists (n, 128-query block) once for every block of every sequence (built on the host, which
// knows the lengths).  Those device values are the caller's guarantee: cu_q non-decreasing from 0 to at most T,
// past[n] + Sq_n <= max_pages * 64, and the table entries of the rows each sequence reads (an entry outside [0, P)
// reads as zero rows).  alibi_slopes fp32 [A] as in attn_fwd.  Returns o [T, A, D]; rows of no sequence are left
// uninitialised.
// With k_scale and v_scale (fp32 [P, G, 64], contiguous) the pools are FP8 (E4M3, contiguous, 16-byte aligned): each
// sequence's output is the bf16 op's over the dequantized pools bf16_rn(float(e) * s), bit for bit, whatever the pools
// hold outside the windows.
Tensor attn_fwd_paged_varlen_any(const char* op, const Tensor& q, const Tensor& k_pool, const Tensor& v_pool,
                                 const Tensor* k_scale, const Tensor* v_scale, const Tensor& block_table,
                                 const Tensor& cu_q, const Tensor& past, const Tensor& tiles, double scale,
                                 const c10::optional<Tensor>& alibi_slopes) {
  Args args(op);
  args("q", q, at::kBFloat16, {kAny, kAny, kAny}, Layout::LastDimContiguous, 16);
  const int64_t D = q.size(2);
  TORCH_CHECK(D == 64 || D == 128, op, ": head dim must be 64 or 128, got ", D);
  if (k_scale != nullptr) {
    args("k_pool", k_pool, at::kFloat8_e4m3fn, {kAny, kAny, 64, D}, Layout::Contiguous, 16);
    args("v_pool", v_pool, at::kFloat8_e4m3fn, k_pool.sizes(), Layout::Contiguous, 16);
    args("k_scale", *k_scale, at::kFloat, k_pool.sizes().slice(0, 3), Layout::Contiguous, 16);
    args("v_scale", *v_scale, at::kFloat, k_pool.sizes().slice(0, 3), Layout::Contiguous, 16);
  } else {
    args("k_pool", k_pool, at::kBFloat16, {kAny, kAny, 64, D});
    args("v_pool", v_pool, at::kBFloat16, k_pool.sizes());
  }
  args("block_table", block_table, at::kInt, {kAny, kAny});
  const int64_t N = block_table.size(0);
  args("cu_q", cu_q, at::kInt, {N + 1});
  args("past", past, at::kInt, {N});
  args("tiles", tiles, at::kInt, {kAny, 2}, Layout::Contiguous, 8);
  lb::AttnArgs a{};
  a.B = 1;
  a.Sq = (int)q.size(0);
  a.A = (int)q.size(1);
  a.G = (int)k_pool.size(1);
  a.d = (int)D;
  TORCH_CHECK(a.G > 0 && a.A % a.G == 0, op, ": the query heads must be a multiple of the K/V heads");
  TORCH_CHECK(k_pool.size(0) >= 1 && k_pool.size(0) <= INT32_MAX, op, ": 1 <= pages <= INT32_MAX");
  TORCH_CHECK(a.Sq >= 1 && N >= 1 && block_table.size(1) >= 1, op, ": at least one token, one sequence and one table "
              "column");
  TORCH_CHECK(tiles.size(0) <= INT32_MAX / 2, op, ": too many tiles");
  const long r = a.A / a.G;
  a.q_strides[0] = (long)q.size(0) * q.stride(0);
  a.q_strides[1] = r * q.stride(1);
  a.q_strides[2] = q.stride(1);
  a.q_strides[3] = q.stride(0);
  for (int i = 0; i < 3; ++i) a.k_strides[i] = a.v_strides[i] = k_pool.stride(i);
  a.causal = true;
  a.scale = (float)scale;
  a.alibi_slopes = args.opt<const float>("alibi_slopes", alibi_slopes, at::kFloat, {a.A});
  const auto guard = args.guard();
  Tensor o = at::empty({a.Sq, a.A, a.d}, q.options());
  Tensor lse = at::empty({(int64_t)a.Sq * a.A}, q.options().dtype(at::kFloat));
  const int P = (int)k_pool.size(0), mp = (int)block_table.size(1), n_tiles = (int)tiles.size(0);
  if (k_scale != nullptr)
    check(lb_attn_fwd_paged_varlen_fp8(&a, q.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(),
                                       k_scale->data_ptr<float>(), v_scale->data_ptr<float>(), P,
                                       block_table.data_ptr<int>(), mp, cu_q.data_ptr<int>(), past.data_ptr<int>(),
                                       tiles.data_ptr<int>(), n_tiles, o.data_ptr(), lse.data_ptr<float>(),
                                       cur_stream()),
          op);
  else
    check(lb_attn_fwd_paged_varlen(&a, q.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), P,
                                   block_table.data_ptr<int>(), mp, cu_q.data_ptr<int>(), past.data_ptr<int>(),
                                   tiles.data_ptr<int>(), n_tiles, o.data_ptr(), lse.data_ptr<float>(), cur_stream()),
          op);
  return o;
}
Tensor attn_fwd_paged_varlen(const Tensor& q, const Tensor& k_pool, const Tensor& v_pool, const Tensor& block_table,
                             const Tensor& cu_q, const Tensor& past, const Tensor& tiles, double scale,
                             const c10::optional<Tensor>& alibi_slopes) {
  return attn_fwd_paged_varlen_any("attn_fwd_paged_varlen", q, k_pool, v_pool, nullptr, nullptr, block_table, cu_q,
                                   past, tiles, scale, alibi_slopes);
}
Tensor attn_fwd_paged_varlen_fp8(const Tensor& q, const Tensor& k_pool, const Tensor& v_pool, const Tensor& k_scale,
                                 const Tensor& v_scale, const Tensor& block_table, const Tensor& cu_q,
                                 const Tensor& past, const Tensor& tiles, double scale,
                                 const c10::optional<Tensor>& alibi_slopes) {
  return attn_fwd_paged_varlen_any("attn_fwd_paged_varlen_fp8", q, k_pool, v_pool, &k_scale, &v_scale, block_table,
                                   cu_q, past, tiles, scale, alibi_slopes);
}

// ---- KV-cache decoding ------------------------------------------------------------------------------
// K and V caches [B, G, C, D], bf16 or (with row scales k_scale, v_scale fp32 [B, G, C]) FP8 (E4M3), D 64 or 128.  An
// FP8 cache's capacity is a multiple of 4: the decode kernel loads the scales of a tile from a 16-byte boundary.  The
// capacity C cannot be checked against the device-side lengths without a host sync: the caller
// (libai_b200.inference.kv_cache.StaticKVCache) guarantees cache_seqlens[b] + Sq <= C before every call.
void cache_args(Args& args, const Tensor& k_cache, const Tensor& v_cache, const Tensor* k_scale, const Tensor* v_scale,
                at::IntArrayRef sizes) {
  const at::ScalarType dtype = k_scale != nullptr ? at::kFloat8_e4m3fn : at::kBFloat16;
  args("k_cache", k_cache, dtype, sizes, Layout::Contiguous, 16);
  args("v_cache", v_cache, dtype, k_cache.sizes(), Layout::Contiguous, 16);
  TORCH_CHECK(k_cache.size(3) == 64 || k_cache.size(3) == 128, args.op(), ": head dim must be 64 or 128");
  if (k_scale != nullptr) {
    TORCH_CHECK(k_cache.size(2) % 4 == 0, args.op(), ": an FP8 cache's capacity must be a multiple of 4");
    args("k_scale", *k_scale, at::kFloat, k_cache.sizes().slice(0, 3), Layout::Contiguous, 16);
    args("v_scale", *v_scale, at::kFloat, k_cache.sizes().slice(0, 3), Layout::Contiguous, 16);
  }
}

// k, v of the packed projection qkv ([B, Sq, A, 3D] or grouped [B, Sq, G, r + 2, D]) go to rows cache_seqlens[b] + i
// of the caches [B, G, C, D]; with cos/sin (fp32 [>= positions, D]) q and k are rotated first.  Returns the (rotated) q
// as [B, Sq, G * r, D] when write_q, else empty.  With k_scale and v_scale the caches are FP8 (E4M3): the bf16 k row
// before quantization is that of a bf16 cache, and each k and v row x is stored as the bytes e4m3_rn_satfinite(x / s)
// with s = amax|x| / 448 (1 for a zero row).  With a block table (int32 [B, max_pages]) the caches are paged: pools of
// 64-row pages [P, G, 64, D] (scales [P, G, 64]), logical row j of sample b at row j % 64 of page table[b][j / 64];
// like the lengths, page ids in [0, P) for the rows written are the caller's guarantee.
Tensor kv_append_any(const char* op, const Tensor& qkv, const Tensor& k_cache, const Tensor& v_cache,
                     const Tensor* k_scale, const Tensor* v_scale, const Tensor& cache_seqlens,
                     const c10::optional<Tensor>& cosv, const c10::optional<Tensor>& sinv, bool write_q,
                     const Tensor* table = nullptr) {
  Args args(op);
  args("qkv", qkv, at::kBFloat16, qkv.sizes());
  const PackedQKV g = packed_qkv(qkv, op);
  if (table != nullptr)
    cache_args(args, k_cache, v_cache, k_scale, v_scale, {kAny, g.G, 64, g.D});
  else
    cache_args(args, k_cache, v_cache, k_scale, v_scale, {g.B, g.G, kAny, g.D});
  if (table != nullptr) args("block_table", *table, at::kInt, {g.B, kAny});
  const int max_pages = table != nullptr ? (int)table->size(1) : 0;
  const int B = g.B, G = g.G, C = table != nullptr ? max_pages * 64 : (int)k_cache.size(2), D = g.D, Sq = g.S,
            A = G * g.r;
  TORCH_CHECK(Sq >= 1 && Sq <= C, op, ": 1 <= Sq <= capacity");
  args("cache_seqlens", cache_seqlens, at::kInt, {B});
  TORCH_CHECK(given(cosv) == given(sinv), op, ": cos and sin go together");
  // like the capacity, the rows of the tables (positions up to cache_seqlens[b] + Sq - 1) are the caller's guarantee
  if (given(cosv)) rope_tables(args, *cosv, *sinv, 0, D);
  const auto guard = args.guard();
  Tensor q_out = write_q ? at::empty({B, Sq, A, D}, qkv.options()) : at::empty({0}, qkv.options());
  const float* cp = given(cosv) ? cosv->data_ptr<float>() : nullptr;
  const float* sp = given(sinv) ? sinv->data_ptr<float>() : nullptr;
  void* qp = write_q ? q_out.data_ptr() : nullptr;
  const int* tp = table != nullptr ? table->data_ptr<int>() : nullptr;
  if (k_scale != nullptr && table != nullptr)
    check(lb_kv_append_fp8_paged(qkv.data_ptr(), cp, sp, qp, k_cache.data_ptr(), v_cache.data_ptr(),
                                 k_scale->data_ptr<float>(), v_scale->data_ptr<float>(), cache_seqlens.data_ptr<int>(),
                                 tp, max_pages, B, Sq, G, g.r, D, cur_stream()),
          op);
  else if (k_scale != nullptr)
    check(lb_kv_append_fp8(qkv.data_ptr(), cp, sp, qp, k_cache.data_ptr(), v_cache.data_ptr(), k_scale->data_ptr<float>(),
                           v_scale->data_ptr<float>(), cache_seqlens.data_ptr<int>(), B, Sq, G, g.r, C, D, cur_stream()),
          op);
  else if (table != nullptr)
    check(lb_kv_append_paged(qkv.data_ptr(), cp, sp, qp, k_cache.data_ptr(), v_cache.data_ptr(),
                             cache_seqlens.data_ptr<int>(), tp, max_pages, B, Sq, G, g.r, D, cur_stream()),
          op);
  else
    check(lb_kv_append(qkv.data_ptr(), cp, sp, qp, k_cache.data_ptr(), v_cache.data_ptr(), cache_seqlens.data_ptr<int>(),
                       B, Sq, G, g.r, C, D, cur_stream()),
          op);
  return q_out;
}
Tensor kv_append(const Tensor& qkv, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cache_seqlens,
                 const c10::optional<Tensor>& cosv, const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_any("kv_append", qkv, k_cache, v_cache, nullptr, nullptr, cache_seqlens, cosv, sinv, write_q);
}
Tensor kv_append_fp8(const Tensor& qkv, const Tensor& k_cache, const Tensor& v_cache, const Tensor& k_scale,
                     const Tensor& v_scale, const Tensor& cache_seqlens, const c10::optional<Tensor>& cosv,
                     const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_any("kv_append_fp8", qkv, k_cache, v_cache, &k_scale, &v_scale, cache_seqlens, cosv, sinv, write_q);
}
Tensor kv_append_paged(const Tensor& qkv, const Tensor& k_pool, const Tensor& v_pool, const Tensor& block_table,
                       const Tensor& cache_seqlens, const c10::optional<Tensor>& cosv,
                       const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_any("kv_append_paged", qkv, k_pool, v_pool, nullptr, nullptr, cache_seqlens, cosv, sinv, write_q,
                       &block_table);
}
Tensor kv_append_fp8_paged(const Tensor& qkv, const Tensor& k_pool, const Tensor& v_pool, const Tensor& k_scale,
                           const Tensor& v_scale, const Tensor& block_table, const Tensor& cache_seqlens,
                           const c10::optional<Tensor>& cosv, const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_any("kv_append_fp8_paged", qkv, k_pool, v_pool, &k_scale, &v_scale, cache_seqlens, cosv, sinv,
                       write_q, &block_table);
}

// k, v of the packed projection qkv [1, T, A, 3D] or [1, T, G, r + 2, D] of N ragged sequences go to their pages: token
// t of sequence n (cu_q[n] <= t < cu_q[n + 1]) to logical row past[n] + t - cu_q[n] of row n of block_table int32
// [N, max_pages], rotated at that position with cos/sin; bf16 pools [P, G, 64, D].  Like the lengths of
// kv_append_paged, cu_q (int32 [N + 1], from 0 to T, non-decreasing), past (int32 [N]) and the page ids of the rows
// written are the caller's guarantee.  Returns q [1, T, G * r, D] when write_q, else empty.
Tensor kv_append_paged_varlen_any(const char* op, const Tensor& qkv, const Tensor& k_pool, const Tensor& v_pool,
                                  const Tensor* k_scale, const Tensor* v_scale, const Tensor& block_table,
                                  const Tensor& cu_q, const Tensor& past, const c10::optional<Tensor>& cosv,
                                  const c10::optional<Tensor>& sinv, bool write_q) {
  Args args(op);
  args("qkv", qkv, at::kBFloat16, qkv.sizes());
  const PackedQKV g = packed_qkv(qkv, op);
  TORCH_CHECK(g.B == 1, op, ": the sequences are packed along dim 1 of a batch of 1, got batch ", g.B);
  cache_args(args, k_pool, v_pool, k_scale, v_scale, {kAny, g.G, 64, g.D});
  args("block_table", block_table, at::kInt, {kAny, kAny});
  const int64_t N = block_table.size(0);
  TORCH_CHECK(N >= 1 && N <= INT32_MAX && block_table.size(1) >= 1, op, ": at least one sequence and table column");
  args("cu_q", cu_q, at::kInt, {N + 1});
  args("past", past, at::kInt, {N});
  TORCH_CHECK(given(cosv) == given(sinv), op, ": cos and sin go together");
  if (given(cosv)) rope_tables(args, *cosv, *sinv, 0, g.D);
  const auto guard = args.guard();
  const int T = g.S, A = g.G * g.r;
  Tensor q_out = write_q ? at::empty({1, T, A, g.D}, qkv.options()) : at::empty({0}, qkv.options());
  const float* cp = given(cosv) ? cosv->data_ptr<float>() : nullptr;
  const float* sp = given(sinv) ? sinv->data_ptr<float>() : nullptr;
  void* qp = write_q ? q_out.data_ptr() : nullptr;
  if (k_scale != nullptr)
    check(lb_kv_append_fp8_paged_varlen(qkv.data_ptr(), cp, sp, qp, k_pool.data_ptr(), v_pool.data_ptr(),
                                        k_scale->data_ptr<float>(), v_scale->data_ptr<float>(), cu_q.data_ptr<int>(),
                                        past.data_ptr<int>(), (int)N, block_table.data_ptr<int>(),
                                        (int)block_table.size(1), T, g.G, g.r, g.D, cur_stream()),
          op);
  else
    check(lb_kv_append_paged_varlen(qkv.data_ptr(), cp, sp, qp, k_pool.data_ptr(), v_pool.data_ptr(),
                                    cu_q.data_ptr<int>(), past.data_ptr<int>(), (int)N, block_table.data_ptr<int>(),
                                    (int)block_table.size(1), T, g.G, g.r, g.D, cur_stream()),
          op);
  return q_out;
}
Tensor kv_append_paged_varlen(const Tensor& qkv, const Tensor& k_pool, const Tensor& v_pool, const Tensor& block_table,
                              const Tensor& cu_q, const Tensor& past, const c10::optional<Tensor>& cosv,
                              const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_paged_varlen_any("kv_append_paged_varlen", qkv, k_pool, v_pool, nullptr, nullptr, block_table, cu_q,
                                    past, cosv, sinv, write_q);
}
// kv_append_paged_varlen into FP8 (E4M3) pools with row scales k_scale, v_scale fp32 [P, G, 64]: each sequence's
// bytes, scales and q are kv_append_fp8_paged's on that sequence alone
Tensor kv_append_fp8_paged_varlen(const Tensor& qkv, const Tensor& k_pool, const Tensor& v_pool, const Tensor& k_scale,
                                  const Tensor& v_scale, const Tensor& block_table, const Tensor& cu_q,
                                  const Tensor& past, const c10::optional<Tensor>& cosv,
                                  const c10::optional<Tensor>& sinv, bool write_q) {
  return kv_append_paged_varlen_any("kv_append_fp8_paged_varlen", qkv, k_pool, v_pool, &k_scale, &v_scale,
                                    block_table, cu_q, past, cosv, sinv, write_q);
}

// Copies page src to page dst of every array of `arrays` (the K and V pools, and the FP8 scales, of every layer of a
// paged cache: contiguous, on one device, with the same number of pages P and pages of a multiple of 16 bytes) for
// each row (src, dst) of `pairs` (int32 [n, 2], on the host, ids in [0, P): checked here).  One launch.
void kv_page_copy(at::TensorList arrays, const Tensor& pairs) {
  TORCH_CHECK(pairs.device().is_cpu() && pairs.scalar_type() == at::kInt && pairs.dim() == 2 && pairs.size(1) == 2,
              "kv_page_copy: pairs must be a host int32 [n, 2] tensor, got ", Got{pairs});
  TORCH_CHECK(!arrays.empty(), "kv_page_copy: no arrays");
  const int64_t n = pairs.size(0), P = arrays[0].size(0), A = (int64_t)arrays.size();
  TORCH_CHECK(A <= 65535, "kv_page_copy: at most 65535 arrays");
  std::vector<long> desc(2 * n + 2 * A);
  const Tensor pc = pairs.contiguous();
  const int* pp = pc.data_ptr<int>();
  for (int64_t i = 0; i < 2 * n; ++i) {
    TORCH_CHECK(pp[i] >= 0 && pp[i] < P, "kv_page_copy: page ids must be in [0, ", P, "), got ", pp[i]);
    desc[i] = pp[i];
  }
  for (int64_t a = 0; a < A; ++a) {
    const Tensor& t = arrays[a];
    TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.dim() >= 2 && t.size(0) == P && t.device() == arrays[0].device(),
                "kv_page_copy: every array must be a contiguous CUDA tensor of ", P, " pages on ", arrays[0].device(),
                ", got ", Got{t});
    const int64_t bytes = t.numel() / P * t.element_size();
    TORCH_CHECK(bytes % 16 == 0 && reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0,
                "kv_page_copy: pages must be multiples of 16 bytes, 16-byte aligned");
    desc[2 * n + 2 * a] = reinterpret_cast<long>(t.data_ptr());
    desc[2 * n + 2 * a + 1] = bytes;
  }
  if (n == 0) return;
  const c10::cuda::CUDAGuard guard(arrays[0].device());
  Tensor d = at::from_blob(desc.data(), {(int64_t)desc.size()}, at::kLong)
                 .to(arrays[0].device(), /*non_blocking=*/false, /*copy=*/true);
  check(lb_kv_page_copy(reinterpret_cast<const long*>(d.data_ptr()), (int)n, (int)A, cur_stream()), "kv_page_copy");
}

// q [B, Sq, A, D] (any strides with D contiguous, e.g. a view of the packed projection) against the caches [B, G, C, D]
// (query head h reads cache head h / (A / G)); query i of sample b sees keys kv_start[b] .. cache_seqlens[b] + i.
// Returns o [B, Sq, A, D] contiguous.  splits = 0: automatic.  alibi_slopes (fp32 [A]): ALiBi, each visible score gets
// slope_h * (j - cache_seqlens[b] - i).  rel_bias (fp32 [A, R]): T5's relative-position bias, each visible score gets
// rel_bias[h, min(cache_seqlens[b] + i - j, R - 1)].  causal = false: every query sees kv_start[b] <= j < cache_seqlens[b]
// (cross-attention; the new tokens are not in this cache), without a bias.  k_scale, v_scale (fp32 [B, G, C]): the row
// scales of FP8 (E4M3) caches, required for those and rejected otherwise; the scores and outputs are those over the
// dequantized rows float(e) * s.
// With a block table (int32 [B, max_pages]) the caches are paged (see kv_append_any; no rel_bias, causal only): the
// kernel runs the same tiles as over a contiguous cache of capacity max_pages * 64, and the same splits.
Tensor decode_attn_any(const char* op, const Tensor& q, const Tensor& k_cache, const Tensor& v_cache,
                       const Tensor& cache_seqlens, const Tensor& kv_start, double scale, int64_t splits,
                       const c10::optional<Tensor>& alibi_slopes, const c10::optional<Tensor>& rel_bias, bool causal,
                       const c10::optional<Tensor>& k_scale, const c10::optional<Tensor>& v_scale,
                       const Tensor* table) {
  Args args(op);
  args("q", q, at::kBFloat16, {kAny, kAny, kAny, kAny}, Layout::LastDimContiguous, 16);
  TORCH_CHECK(q.stride(0) % 8 == 0 && q.stride(1) % 8 == 0 && q.stride(2) % 8 == 0,
              op, ": q must be 16-byte aligned with strides that are multiples of 8");
  const bool fp8 = k_cache.scalar_type() == at::kFloat8_e4m3fn;
  TORCH_CHECK(!fp8 || (given(k_scale) && given(v_scale)), op, ": an FP8 cache needs k_scale and v_scale");
  TORCH_CHECK(fp8 || (!given(k_scale) && !given(v_scale)), op, ": k_scale and v_scale belong to an FP8 cache");
  if (table != nullptr)
    cache_args(args, k_cache, v_cache, fp8 ? &*k_scale : nullptr, fp8 ? &*v_scale : nullptr,
               {kAny, kAny, 64, q.size(3)});
  else
    cache_args(args, k_cache, v_cache, fp8 ? &*k_scale : nullptr, fp8 ? &*v_scale : nullptr,
               {q.size(0), kAny, kAny, q.size(3)});
  if (table != nullptr) args("block_table", *table, at::kInt, {q.size(0), kAny});
  const int max_pages = table != nullptr ? (int)table->size(1) : 0;
  const int B = (int)q.size(0), G = (int)k_cache.size(1), D = (int)k_cache.size(3);
  const int C = table != nullptr ? max_pages * 64 : (int)k_cache.size(2);
  const int Sq = (int)q.size(1), A = (int)q.size(2);
  TORCH_CHECK(A % G == 0, op, ": the query heads must be a multiple of the cache heads");
  TORCH_CHECK(Sq >= 1 && Sq <= 16, op, ": 1 <= Sq <= 16 new queries");
  args("cache_seqlens", cache_seqlens, at::kInt, {B});
  args("kv_start", kv_start, at::kInt, {B});
  const float* slopes = args.opt<const float>("alibi_slopes", alibi_slopes, at::kFloat, {A});
  const float* rel = nullptr;
  int R = 0;
  if (given(rel_bias)) {
    const Tensor& r = *rel_bias;
    TORCH_CHECK(r.scalar_type() == at::kFloat && r.dim() == 2 && r.size(0) == A && r.size(1) >= 1 &&
                    r.device() == q.device() && r.is_contiguous(),
                op, ": rel_bias: contiguous fp32 [A, R] with R >= 1 on q's device, got ", r.scalar_type(), " ",
                r.sizes(), " on ", r.device());
    TORCH_CHECK(r.size(1) <= INT32_MAX, op, ": rel_bias: R fits in int32");
    TORCH_CHECK(slopes == nullptr, op, ": alibi_slopes or rel_bias, not both");
    rel = r.data_ptr<float>();
    R = (int)r.size(1);
  }
  TORCH_CHECK(causal || (slopes == nullptr && rel == nullptr),
              op, ": causal=False takes no score bias (neither alibi_slopes nor rel_bias)");
  TORCH_CHECK(table == nullptr || (rel == nullptr && causal), op, ": a paged cache takes no rel_bias and no causal=False");
  const auto guard = args.guard();
  const int row_blocks = ((A / G) * Sq + 15) / 16;   // (query head, token) rows of one cache head, 16 per CTA
  const int nsplit = splits > 0 ? (int)std::min<int64_t>(splits, 32) : lb_decode_splits(B, G * row_blocks, C, D, fp8);
  Tensor o = at::empty({B, Sq, A, D}, q.options());
  Tensor part_o, part_ml;
  if (nsplit > 1) {
    part_o = at::empty({(int64_t)B * A * nsplit * Sq * D}, q.options().dtype(at::kFloat));
    part_ml = at::empty({(int64_t)B * A * nsplit * Sq * 2}, q.options().dtype(at::kFloat));
  }
  long qs[3] = {q.stride(0), q.stride(1), q.stride(2)};
  check(lb_decode_attn(q.data_ptr(), qs, k_cache.data_ptr(), v_cache.data_ptr(), o.data_ptr(),
                       nsplit > 1 ? part_o.data_ptr<float>() : nullptr, nsplit > 1 ? part_ml.data_ptr<float>() : nullptr,
                       cache_seqlens.data_ptr<int>(), kv_start.data_ptr<int>(), slopes, rel, R, causal,
                       fp8 ? k_scale->data_ptr<float>() : nullptr, fp8 ? v_scale->data_ptr<float>() : nullptr,
                       table != nullptr ? table->data_ptr<int>() : nullptr, max_pages, B, Sq, A, G, C, D, (float)scale,
                       nsplit, cur_stream()),
        op);
  return o;
}

Tensor decode_attn(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cache_seqlens,
                   const Tensor& kv_start, double scale, int64_t splits, const c10::optional<Tensor>& alibi_slopes,
                   const c10::optional<Tensor>& rel_bias, bool causal, const c10::optional<Tensor>& k_scale,
                   const c10::optional<Tensor>& v_scale) {
  return decode_attn_any("decode_attn", q, k_cache, v_cache, cache_seqlens, kv_start, scale, splits, alibi_slopes,
                         rel_bias, causal, k_scale, v_scale, nullptr);
}
Tensor decode_attn_paged(const Tensor& q, const Tensor& k_pool, const Tensor& v_pool, const Tensor& block_table,
                         const Tensor& cache_seqlens, const Tensor& kv_start, double scale, int64_t splits,
                         const c10::optional<Tensor>& alibi_slopes, const c10::optional<Tensor>& k_scale,
                         const c10::optional<Tensor>& v_scale) {
  return decode_attn_any("decode_attn_paged", q, k_pool, v_pool, cache_seqlens, kv_start, scale, splits, alibi_slopes,
                         c10::nullopt, true, k_scale, v_scale, &block_table);
}

// ---- shifted-window attention -----------------------------------------------------------------------
// qkv [B, H*W, 3*C] in image order (per token [3, heads, d]), an H x W map of ws x ws windows cyclically shifted by
// `shift`; table fp32 [(2ws - 1)^2, heads]; tau fp32 [heads] selects cosine attention (SwinV2).  Returns the head dim.
int64_t window_args(Args& args, const Tensor& qkv, int64_t H, int64_t W, int64_t ws, int64_t shift, int64_t heads,
                    const Tensor& table, const c10::optional<Tensor>& tau) {
  const char* what = args.op();
  args("qkv", qkv, at::kBFloat16, {kAny, kAny, kAny}, Layout::Contiguous, 16);
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
  args("table", table, at::kFloat, {(2 * ws - 1) * (2 * ws - 1), heads});
  args.opt("tau", tau, at::kFloat, {heads});
  return d;
}

std::tuple<Tensor, Tensor> window_attn_fwd(const Tensor& qkv, int64_t H, int64_t W, int64_t window, int64_t shift,
                                           int64_t heads, double scale, const Tensor& table,
                                           const c10::optional<Tensor>& tau) {
  Args args("window_attn_fwd");
  const int64_t d = window_args(args, qkv, H, W, window, shift, heads, table, tau);
  const auto guard = args.guard();
  const int64_t B = qkv.size(0), nwin = B * (H / window) * (W / window);
  Tensor o = at::empty({B, H * W, heads * d}, qkv.options());
  Tensor lse = at::empty({nwin, heads, window * window}, qkv.options().dtype(at::kFloat));
  const bool cos = given(tau);
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
  Args args("window_attn_bwd");
  const int64_t d = window_args(args, qkv, H, W, window, shift, heads, table, tau);
  const int64_t B = qkv.size(0), N = window * window, nwin = B * (H / window) * (W / window);
  args("dout", dout, at::kBFloat16, {B, H * W, heads * d}, Layout::Contiguous, 16);
  args("lse", lse, at::kFloat, {nwin, heads, N});
  const auto guard = args.guard();
  const bool cos = given(tau);
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
                                            const c10::optional<Tensor>& doc_start,
                                            const c10::optional<Tensor>& prefix_lens) {
  Args args("attn_bwd");
  const lb::AttnArgs a = attn_args(args, q, k, v, causal, scale, kv_lens, kv_start, doc_start, bias, alibi_slopes, p_drop,
                                   prefix_lens);
  const int B = a.B, A = a.A, G = a.G, Sq = a.Sq, Sk = a.Sk, D = a.d, r = A / G;
  args("o", o, at::kBFloat16, {B, A, Sq, D}, Layout::LastDimContiguous);
  args("dout", dout, kAnyDtype, {B, A, Sq, D}, Layout::Strided);
  args("lse", lse, at::kFloat, {B, A, Sq});
  const bool drop = p_drop > 0.0;
  TORCH_CHECK(!drop || given(rng_state), "attn_bwd: p_drop > 0 needs the forward's rng_state");
  const auto* rng_in = drop ? args.opt<const long long>("rng_state", rng_state, at::kLong, {2}) : nullptr;
  float* dbp = nullptr;
  if (given(dbias)) {
    TORCH_CHECK(given(bias), "attn_bwd: dbias needs bias");
    dbp = args.opt<float>("dbias", dbias, at::kFloat, bias->sizes(), Layout::Strided);
    TORCH_CHECK(dbias->strides() == bias->strides(), "attn_bwd: dbias must have the strides of bias");
  }
  const auto guard = args.guard();
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
  Tensor dout_c = dout;
  if (dout.strides() != o.strides() || dout.scalar_type() != at::kBFloat16) {   // into the [B, S, A, D]-backed layout of o
    dout_c = at::empty_strided(o.sizes(), o.strides(), o.options());
    dout_c.copy_(dout);
  }
  const long ds[3] = {dout_c.stride(0), dout_c.stride(1), dout_c.stride(2)};
  check(lb_attn_bwd(&a, dout_c.data_ptr(), ds, q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                    lse.data_ptr<float>(), dq5.data_ptr(), dk.data_ptr(), dv.data_ptr(), dqs, dkvs,
                    delta.data_ptr<float>(), dq_acc.data_ptr<float>(), dbp, rng_in,
                    reinterpret_cast<unsigned*>(dq_order.data_ptr<int>()), cur_stream()),
        "attn_bwd");
  Tensor dq = q.dim() == 5 ? dq5 : dq5.reshape({B, A, Sq, D});   // after the kernel: for r > 1 this copies
  return std::make_tuple(dq, dk, dv, dqkv);
}

// ---- fused collectives ---------------------------------------------------------------------------------------
std::vector<long> to_longs(at::IntArrayRef v) { return std::vector<long>(v.begin(), v.end()); }

const void* opt_ptr(const c10::optional<Tensor>& t) { return given(t) ? t->data_ptr() : nullptr; }

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
  float* cs = given(colsum) ? colsum->data_ptr<float>() : nullptr;
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
  m.def("linear_fp8w(Tensor x, Tensor w, Tensor w_scale, Tensor? bias, int act) -> Tensor", &linear_fp8w);
  m.def("dequant_e4m3_rows(Tensor w, Tensor w_scale) -> Tensor", &dequant_e4m3_rows);
  m.def("linear_int4w(Tensor x, Tensor w, Tensor w_scale, Tensor w_zero, Tensor? bias, int act) -> Tensor",
        &linear_int4w);
  m.def("dequant_int4_rows(Tensor w, Tensor w_scale, Tensor w_zero) -> Tensor", &dequant_int4_rows);
  m.def("spec_accept(Tensor logits, Tensor draft, Tensor(a!) unfinished, int eos, int pad) -> Tensor", &spec_accept);
  m.def("spec_sample(Tensor logits, Tensor(a!) q, int j, Tensor u, Tensor(b!) proposals, float temperature, int top_k, "
        "float top_p) -> ()", &spec_sample);
  m.def("spec_accept_sample(Tensor logits, Tensor q, Tensor draft, Tensor u, Tensor(a!) unfinished, float temperature, "
        "int top_k, float top_p, int eos, int pad, Tensor(b!)? scores=None) -> Tensor", &spec_accept_sample);
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
  m.def("rope_qkv(Tensor(a!) qkv, Tensor cos, Tensor sin, int pos_offset, bool backward, bool inplace, Tensor? positions=None) -> Tensor(a!)", &rope_qkv);
  m.def("glm_rotary_qkv(Tensor mixed, int heads, int kv_heads, Tensor table, int pos_offset, Tensor? position_ids, bool grouped, Tensor? pos_base=None) -> Tensor", &glm_rotary_qkv);
  m.def("glm_rotary_qkv_bwd(Tensor grad, int heads, int kv_heads, Tensor table, int pos_offset, Tensor? position_ids, Tensor? pos_base=None) -> Tensor", &glm_rotary_qkv_bwd);
  m.def("ce_stats(Tensor logits, Tensor labels, int vocab_start) -> (Tensor, Tensor, Tensor)", &ce_stats);
  m.def("ce_bwd(Tensor(a!) logits, Tensor labels, Tensor lse, Tensor gloss, int vocab_start) -> Tensor(a!)", &ce_bwd);
  m.def("fused_adamw(Tensor(a!) master, Tensor grad, Tensor(b!) m, Tensor(c!) v, Tensor? lp_out, Tensor scale, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, bool decoupled) -> ()", &fused_adamw);
  m.def("sqnorm(Tensor x) -> Tensor", &sqnorm);
  m.def("attn_fwd(Tensor q, Tensor k, Tensor v, bool causal, float scale, Tensor? kv_lens, Tensor? bias=None, Tensor? alibi_slopes=None, float p_drop=0.0, int salt=0, Tensor? kv_start=None, Tensor? doc_start=None, Tensor? prefix_lens=None) -> (Tensor, Tensor, Tensor)", &attn_fwd);
  m.def("attn_bwd(Tensor dout, Tensor q, Tensor k, Tensor v, Tensor o, Tensor lse, bool causal, float scale, Tensor? kv_lens, Tensor? bias=None, Tensor? alibi_slopes=None, Tensor(a!)? dbias=None, float p_drop=0.0, Tensor? rng_state=None, Tensor? kv_start=None, Tensor? doc_start=None, Tensor? prefix_lens=None) -> (Tensor, Tensor, Tensor, Tensor)", &attn_bwd);
  m.def("attn_fwd_paged(Tensor q, Tensor k_pool, Tensor v_pool, Tensor block_table, int past, float scale, Tensor? kv_start=None, Tensor? alibi_slopes=None) -> Tensor", &attn_fwd_paged);
  m.def("attn_fwd_paged_varlen(Tensor q, Tensor k_pool, Tensor v_pool, Tensor block_table, Tensor cu_q, Tensor past, Tensor tiles, float scale, Tensor? alibi_slopes=None) -> Tensor", &attn_fwd_paged_varlen);
  m.def("attn_fwd_paged_varlen_fp8(Tensor q, Tensor k_pool, Tensor v_pool, Tensor k_scale, Tensor v_scale, Tensor block_table, Tensor cu_q, Tensor past, Tensor tiles, float scale, Tensor? alibi_slopes=None) -> Tensor", &attn_fwd_paged_varlen_fp8);
  m.def("kv_append_fp8_paged_varlen(Tensor qkv, Tensor(a!) k_pool, Tensor(b!) v_pool, Tensor(c!) k_scale, Tensor(d!) v_scale, Tensor block_table, Tensor cu_q, Tensor past, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append_fp8_paged_varlen);
  m.def("kv_append_paged_varlen(Tensor qkv, Tensor(a!) k_pool, Tensor(b!) v_pool, Tensor block_table, Tensor cu_q, Tensor past, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append_paged_varlen);
  m.def("kv_append(Tensor qkv, Tensor(a!) k_cache, Tensor(b!) v_cache, Tensor cache_seqlens, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append);
  m.def("kv_append_fp8(Tensor qkv, Tensor(a!) k_cache, Tensor(b!) v_cache, Tensor(c!) k_scale, Tensor(d!) v_scale, Tensor cache_seqlens, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append_fp8);
  m.def("window_attn_fwd(Tensor qkv, int H, int W, int window, int shift, int heads, float scale, Tensor table, Tensor? tau) -> (Tensor, Tensor)", &window_attn_fwd);
  m.def("window_attn_bwd(Tensor dout, Tensor qkv, Tensor lse, int H, int W, int window, int shift, int heads, float scale, Tensor table, Tensor? tau) -> (Tensor, Tensor, Tensor)", &window_attn_bwd);
  m.def("kv_append_paged(Tensor qkv, Tensor(a!) k_pool, Tensor(b!) v_pool, Tensor block_table, Tensor cache_seqlens, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append_paged);
  m.def("kv_append_fp8_paged(Tensor qkv, Tensor(a!) k_pool, Tensor(b!) v_pool, Tensor(c!) k_scale, Tensor(d!) v_scale, Tensor block_table, Tensor cache_seqlens, Tensor? cos, Tensor? sin, bool write_q) -> Tensor", &kv_append_fp8_paged);
  m.def("kv_page_copy(Tensor(a!)[] arrays, Tensor pairs) -> ()", &kv_page_copy);
  m.def("decode_attn_paged(Tensor q, Tensor k_pool, Tensor v_pool, Tensor block_table, Tensor cache_seqlens, Tensor kv_start, float scale, int splits=0, Tensor? alibi_slopes=None, Tensor? k_scale=None, Tensor? v_scale=None) -> Tensor", &decode_attn_paged);
  m.def("decode_attn(Tensor q, Tensor k_cache, Tensor v_cache, Tensor cache_seqlens, Tensor kv_start, float scale, int splits=0, Tensor? alibi_slopes=None, Tensor? rel_bias=None, bool causal=True, Tensor? k_scale=None, Tensor? v_scale=None) -> Tensor", &decode_attn);
  m.def("bias_dropout_residual(Tensor x, Tensor? bias, Tensor? res, float p, int salt, Tensor? rng_state=None) -> (Tensor, Tensor)", &bias_dropout_residual);
}
