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
// the order of the comparisons: the reduction is deterministic.  V needs no alignment (scalar, coalesced loads).  The
// last block to finish runs phase 2 over the b·R argmaxes.  It finds that it is last through a counter that the launcher
// zeroes on the stream before the kernel (cudaMemsetAsync): every launch has its own, so launches on other streams
// never share one and a launch that did not complete leaves nothing behind.
#include <climits>

#include "common.cuh"

namespace lb {
namespace spec {

constexpr int kThreads = 512;

__device__ __forceinline__ float load(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float load(const float* p) { return *p; }

// (v, i) beats (w, j): a larger value, or an equal one at a smaller index
__device__ __forceinline__ bool beats(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

template <typename T>
__global__ void __launch_bounds__(kThreads) accept_kernel(const T* __restrict__ logits, const int64_t* __restrict__ draft,
                                                          int64_t* __restrict__ unfinished, int64_t* __restrict__ out,
                                                          unsigned int* __restrict__ counter, int B, int R, int V,
                                                          long long eos, long long pad) {
  __shared__ float s_val[kThreads / 32];
  __shared__ int s_idx[kThreads / 32];
  __shared__ bool s_last;
  __shared__ int s_n;
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
    if (lane == 0) {
      // a row of −inf only: every index ties, the lowest is 0 (as torch.argmax); idx is INT_MAX only when V == 0
      out[(size_t)(row / R) * cols + row % R] = idx == INT_MAX ? 0 : idx;
      __threadfence();
      s_last = atomicAdd(counter, 1u) == (unsigned)(gridDim.x - 1);
    }
  }
  __syncthreads();
  if (!s_last) return;

  // phase 2: the last block sees every row's argmax
  __threadfence();
  const int k = R - 1;
  if (threadIdx.x == 0) s_n = k;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += kThreads) {
    const volatile int64_t* t = out + (size_t)b * cols;
    int a = 0;
    while (a < k && draft[(size_t)b * k + a] == t[a]) ++a;
    out[(size_t)b * cols + 2 * R] = a;
    if (unfinished[b] != 0) {
      bool ends = false;
      for (int j = 0; j <= a && eos >= 0; ++j) ends |= t[j] == eos;
      atomicMin(&s_n, ends ? k : a);
    }
  }
  __syncthreads();
  const int n = s_n;
  for (int b = threadIdx.x; b < B; b += kThreads) {
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
