// Greedy acceptance of speculative decoding, in one launch: the token decisions of one iteration of
// Generator.speculative_search.
//
// Inputs: the verify step's logits [b, R, V] (R = k + 1 rows per sample: the rows after x, d_1, ..., d_k; bf16 or
// fp32, read in place), the proposals draft [b, k] (int64) and unfinished [b] (int64, 1 = the sample has not emitted
// EOS), updated in place.  Per sample, with t_j the argmax of row j (the lowest index among equal maxima):
//
//   a_b  = the length of the longest prefix with draft[b, j] == t_j;
//   n    = min over the samples unfinished on entry of a_b, where a sample that emits EOS among t_0 .. t_{a_b} counts as
//          k (what follows its EOS is padding whatever the target chose); k when no sample is unfinished;
//   e_j  = t_j for j <= n while the sample is unfinished, pad once it is (it becomes finished after emitting eos); -1
//          for j > n.
//
// out [b, 2R + 3] (int64): columns [0, R) t, [R, 2R) e, 2R a_b, 2R + 1 n, 2R + 2 the updated unfinished.  eos < 0:
// no EOS (unfinished stays as it is, pad unused).
//
// Phase 1 is one block per row: a strided scan of V and a block reduction of (value, index) pairs.  The pair order
// (larger value, then smaller index) is a total order on finite and −inf values, so the result does not depend on
// the order of the comparisons: the reduction is deterministic.  V needs no alignment (scalar, coalesced loads).
//
// Phase 2 (emit(), shared with spec_accept_sample) runs in the last block to finish, over the b·R tokens t in
// out[:, 0:R) and a predicate that says whether row (b, j)'s proposal is accepted (here draft[b, j] == t_j): it
// computes a_b, writes draft[b, j] over t_j for j < a_b (for greedy acceptance the value already there), then n, e and
// the updated unfinished.  The block finds that it is last through a counter that the launcher zeroes on the stream
// before the kernel (cudaMemsetAsync): every launch has its own, so launches on other streams never share one and a
// launch that did not complete leaves nothing behind.
#include <climits>

#include "common.cuh"

namespace lb {
namespace spec {

constexpr int kThreads = 512;

__device__ __forceinline__ float load(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float load(const float* p) { return *p; }

// (v, i) beats (w, j): a larger value, or an equal one at a smaller index
__device__ __forceinline__ bool beats(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// Called by every thread once thread 0 has written its block's results: whether this block is the last of the launch
// to finish, in which case every block's results are visible to it.
__device__ __forceinline__ bool last_block(unsigned int* counter) {
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  return true;
}

// Phase 2 of both acceptance kernels, in the last block, from the tokens t in out[:, 0:R) and accepted(b, j), whether
// row j's proposal draft[b, j] is accepted (j < k).
template <typename Accepted>
__device__ __forceinline__ void emit(Accepted accepted, const int64_t* __restrict__ draft,
                                     int64_t* __restrict__ unfinished, int64_t* out, int B, int R, long long eos,
                                     long long pad) {
  __shared__ int s_n;
  const int k = R - 1, cols = 2 * R + 3;
  if (threadIdx.x == 0) s_n = k;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    volatile int64_t* t = out + (size_t)b * cols;
    int a = 0;
    while (a < k && accepted(b, a)) ++a;
    for (int j = 0; j < a; ++j) t[j] = draft[(size_t)b * k + j];
    t[2 * R] = a;
    if (unfinished[b] != 0) {
      bool ends = false;
      for (int j = 0; j <= a && eos >= 0; ++j) ends |= t[j] == eos;
      atomicMin(&s_n, ends ? k : a);
    }
  }
  __syncthreads();
  const int n = s_n;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int64_t* o = out + (size_t)b * cols;
    const volatile int64_t* t = o;
    int64_t u = unfinished[b];
    for (int j = 0; j < R; ++j) {
      int64_t e = -1;
      if (j <= n) {
        e = t[j];
        if (eos >= 0) {
          if (u == 0) e = pad;
          if (e == eos) u = 0;
        }
      }
      o[R + j] = e;
    }
    o[2 * R + 1] = n;
    o[2 * R + 2] = u;
    unfinished[b] = u;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) accept_kernel(const T* __restrict__ logits, const int64_t* __restrict__ draft,
                                                          int64_t* __restrict__ unfinished, int64_t* __restrict__ out,
                                                          unsigned int* __restrict__ counter, int B, int R, int V,
                                                          long long eos, long long pad) {
  __shared__ float s_val[kThreads / 32];
  __shared__ int s_idx[kThreads / 32];
  const int row = blockIdx.x;   // b * R + j
  const int cols = 2 * R + 3;
  const T* p = logits + (size_t)row * V;

  float best = -INFINITY;
  int idx = INT_MAX;
  for (int i = threadIdx.x; i < V; i += kThreads) {
    const float v = load(p + i);
    if (beats(v, i, best, idx)) best = v, idx = i;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, best, off);
    const int j = __shfl_xor_sync(0xffffffffu, idx, off);
    if (beats(w, j, best, idx)) best = w, idx = j;
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) s_val[warp] = best, s_idx[warp] = idx;
  __syncthreads();
  if (warp == 0) {
    best = lane < kThreads / 32 ? s_val[lane] : -INFINITY;
    idx = lane < kThreads / 32 ? s_idx[lane] : INT_MAX;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, best, off);
      const int j = __shfl_xor_sync(0xffffffffu, idx, off);
      if (beats(w, j, best, idx)) best = w, idx = j;
    }
    // a row of −inf only: every index ties, the lowest is 0 (as torch.argmax); idx is INT_MAX only when V == 0
    if (lane == 0) out[(size_t)(row / R) * cols + row % R] = idx == INT_MAX ? 0 : idx;
  }
  if (!last_block(counter)) return;
  const volatile int64_t* t = out;
  const int k = R - 1;
  emit([=](int b, int j) { return draft[(size_t)b * k + j] == t[(size_t)b * cols + j]; }, draft, unfinished, out, B,
       R, eos, pad);
}

}  // namespace spec
}  // namespace lb

extern "C" {

int lb_spec_accept(const void* logits, int logits_fp32, const int64_t* draft, int64_t* unfinished, int64_t* out,
                   unsigned int* counter, int B, int R, int V, long long eos, long long pad, cudaStream_t s) {
  using namespace lb::spec;
  if (B < 1 || R < 1 || V < 1 || (long long)B * R > 0x7fffffffLL) return static_cast<int>(cudaErrorInvalidValue);
  const cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned int), s);
  if (e != cudaSuccess) return static_cast<int>(e);
  const unsigned grid = (unsigned)(B * R);
  if (logits_fp32)
    accept_kernel<float><<<grid, kThreads, 0, s>>>(static_cast<const float*>(logits), draft, unfinished, out, counter,
                                                   B, R, V, eos, pad);
  else
    accept_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>(static_cast<const __nv_bfloat16*>(logits), draft,
                                                           unfinished, out, counter, B, R, V, eos, pad);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Speculative sampling (Leviathan et al. 2023; Chen et al. 2023): the draft samples its proposals from its warped
// distribution q, the target accepts d with probability min(1, p(d) / q(d)) and replaces the first rejected proposal
// by a draw from norm(max(0, p − q)).  The warp rule (temperature, top-k, top-p, fixed-point masses, the inverse-CDF
// pick) is sampling.cuh's, one CTA per row.
//
// spec_sample: after draft step j, per sample b: q_j[b] = the step's logits row, kept in qbuf[b, j] (q itself is never
// materialised), and d_{j+1} = pick(floor(u[b, j] · Σe)) over q_j's masses, written to proposals[b, j].
//
// spec_accept_sample, phase 1, one CTA per row (b, j) of the verify step's logits [B, R, V] (R = k + 1):
//   accept_j = u[b, j, 0] · q_j(d_{j+1}) < p_j(d_{j+1})                         (j < k, in fp64 from the masses)
//   c_j      = pick(floor(u[b, j, 1] · Σr)) over r_i = 2^40 · max(0, p_j(i) − q_j(i)), rounded (j < k, Σr > 0);
//              pick over p_j's masses when Σr = 0 or j = k (the bonus token)
// phase 2, spec_accept's emit() over t_j = c_j and accepted(b, j) = accept_j: a_b = the first rejected j (k if none);
// t_j = d_{j+1} for j < a_b; then n, e and unfinished from t.  scores (optional, fp32 [B, R, V]): the target's warped
// logits, z on the kept set and −inf elsewhere.
#include "sampling.cuh"

namespace lb {
namespace spec {

using samp::Row;
using samp::Warped;

template <typename T>
__global__ void __launch_bounds__(samp::kThreads, 1) sample_kernel(const T* __restrict__ logits, T* __restrict__ qbuf,
                                                                const float* __restrict__ u,
                                                                int64_t* __restrict__ proposals, int V, int K, int J,
                                                                int j, float temperature, int top_k, float top_p) {
  __shared__ samp::Shared sh;
  const int b = blockIdx.x;
  const T* x = logits + (size_t)b * V;
  T* q = qbuf + ((size_t)b * K + j) * V;
  for (int i = threadIdx.x; i < V; i += samp::kThreads) q[i] = x[i];
  const Row<T> row{x, temperature};
  const Warped w = samp::warp_row(row, V, top_k, top_p, sh);
  const int d = samp::pick([row, w](int i) { return samp::mass_of(row, w, i); }, V,
                           samp::draw(u[(size_t)b * J + j], w.total), sh);
  if (threadIdx.x == 0) proposals[(size_t)b * J + j] = d;
}

template <typename TP, typename TQ>
__global__ void __launch_bounds__(samp::kThreads, 1) accept_sample_kernel(
    const TP* __restrict__ logits, const TQ* __restrict__ qbuf, const int64_t* __restrict__ draft,
    const float* __restrict__ u, int64_t* __restrict__ unfinished, int64_t* __restrict__ out, int* __restrict__ accepted,
    unsigned int* __restrict__ counter, float* __restrict__ scores, int B, int R, int V, int K, float temperature,
    int top_k, float top_p, long long eos, long long pad) {
  __shared__ samp::Shared sh;
  const int row_id = blockIdx.x;   // b * R + j
  const int b = row_id / R, j = row_id % R, k = R - 1;
  const int cols = 2 * R + 3;
  const Row<TP> p_row{logits + (size_t)row_id * V, temperature};
  const Warped pw = samp::warp_row(p_row, V, top_k, top_p, sh);
  const float u0 = u[(size_t)row_id * 2], u1 = u[(size_t)row_id * 2 + 1];
  int cand;
  if (j < k) {
    const Row<TQ> q_row{qbuf + ((size_t)b * K + j) * V, temperature};
    const Warped qw = samp::warp_row(q_row, V, top_k, top_p, sh);
    const double inv_p = 1.0 / (double)pw.total, inv_q = 1.0 / (double)qw.total;
    if (threadIdx.x == 0) {
      const int64_t d = draft[(size_t)b * k + j];
      bool acc = false;
      if (d >= 0 && d < V) {
        const double pd = (double)samp::mass_of(p_row, pw, (int)d) * inv_p;
        const double qd = (double)samp::mass_of(q_row, qw, (int)d) * inv_q;
        acc = (double)u0 * qd < pd;
      }
      accepted[row_id] = acc;
    }
    auto resid = [&](int i) {
      const double r = (double)samp::mass_of(p_row, pw, i) * inv_p - (double)samp::mass_of(q_row, qw, i) * inv_q;
      return r > 0.0 ? __double2ull_rn(r * samp::kOneD) : 0ull;
    };
    unsigned long long s = 0;
    for (int i = threadIdx.x; i < V; i += samp::kThreads) s += resid(i);
    const unsigned long long total = samp::block_sum(s, sh);
    if (total > 0)
      cand = samp::pick(resid, V, samp::draw(u1, total), sh);
    else
      cand = samp::pick([&](int i) { return samp::mass_of(p_row, pw, i); }, V, samp::draw(u1, pw.total), sh);
  } else {
    if (threadIdx.x == 0) accepted[row_id] = 0;
    cand = samp::pick([&](int i) { return samp::mass_of(p_row, pw, i); }, V, samp::draw(u1, pw.total), sh);
  }
  if (scores != nullptr) {
    float* o = scores + (size_t)row_id * V;
    for (int i = threadIdx.x; i < V; i += samp::kThreads) {
      const float z = p_row.z(i);
      o[i] = samp::key_of(z) >= pw.keep ? z : -INFINITY;
    }
  }
  if (threadIdx.x == 0) out[(size_t)b * cols + j] = cand;
  if (!last_block(counter)) return;
  const volatile int* acc = accepted;
  emit([=](int bb, int jj) { return acc[(size_t)bb * R + jj] != 0; }, draft, unfinished, out, B, R, eos, pad);
}

}  // namespace spec
}  // namespace lb

extern "C" {

int lb_spec_sample(const void* logits, void* qbuf, int fp32, const float* u, int64_t* proposals, int B, int V, int K,
                   int J, int j, float temperature, int top_k, float top_p, cudaStream_t s) {
  using namespace lb::spec;
  if (B < 1 || V < 1 || K < 1 || J < 1 || j < 0 || j >= K || j >= J) return static_cast<int>(cudaErrorInvalidValue);
  if (fp32)
    sample_kernel<float><<<B, lb::samp::kThreads, 0, s>>>(static_cast<const float*>(logits), static_cast<float*>(qbuf),
                                                          u, proposals, V, K, J, j, temperature, top_k, top_p);
  else
    sample_kernel<__nv_bfloat16><<<B, lb::samp::kThreads, 0, s>>>(
        static_cast<const __nv_bfloat16*>(logits), static_cast<__nv_bfloat16*>(qbuf), u, proposals, V, K, J, j,
        temperature, top_k, top_p);
  return static_cast<int>(cudaGetLastError());
}

int lb_spec_accept_sample(const void* logits, int logits_fp32, const void* qbuf, int q_fp32, const int64_t* draft,
                          const float* u, int64_t* unfinished, int64_t* out, int* accepted, unsigned int* counter,
                          float* scores, int B, int R, int V, int K, float temperature, int top_k, float top_p,
                          long long eos, long long pad, cudaStream_t s) {
  using namespace lb::spec;
  if (B < 1 || R < 1 || V < 1 || K < R - 1 || (long long)B * R > 0x7fffffffLL)
    return static_cast<int>(cudaErrorInvalidValue);
  const cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned int), s);
  if (e != cudaSuccess) return static_cast<int>(e);
  const unsigned grid = (unsigned)(B * R);
  constexpr int nt = lb::samp::kThreads;
#define LB_ACCEPT_SAMPLE(TP, TQ)                                                                                       \
  accept_sample_kernel<TP, TQ><<<grid, nt, 0, s>>>(static_cast<const TP*>(logits), static_cast<const TQ*>(qbuf), draft, \
                                                   u, unfinished, out, accepted, counter, scores, B, R, V, K,           \
                                                   temperature, top_k, top_p, eos, pad)
  if (logits_fp32 && q_fp32) LB_ACCEPT_SAMPLE(float, float);
  else if (logits_fp32) LB_ACCEPT_SAMPLE(float, __nv_bfloat16);
  else if (q_fp32) LB_ACCEPT_SAMPLE(__nv_bfloat16, float);
  else LB_ACCEPT_SAMPLE(__nv_bfloat16, __nv_bfloat16);
#undef LB_ACCEPT_SAMPLE
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
