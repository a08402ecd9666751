// The warp rule of speculative sampling (speculative_sm90.cu), one CTA per logits row.  Everything a row's decisions
// depend on is computed from that row alone, in a fixed way, so the results are bit-identical across launches, streams
// and batch compositions:
//
//   z_i     = logit_i / T                                   an IEEE fp32 division (__fdiv_rn: the build uses
//                                                           --use_fast_math, which would make `/` approximate)
//   top-k   keep z_i >= the k'-th largest z (k' = min(top_k, V), counting duplicates; off when top_k is 0 or >= V):
//           a radix select over order-preserving uint32 keys, four 8-bit passes with a shared count histogram (one
//           atomic per bin and warp: __match_any_sync groups a warp's keys by bin)
//   e_i     = 2^40 · exp(z_i − z_max), rounded to an integer (a 64-bit fixed-point mass; e = 2^40 where z_i == z_max,
//           so a row of −inf only is uniform); 0 for a token that is not kept
//   top-p   over the top-k set: keep i iff the mass of kept tokens with z strictly greater than z_i is
//           <= floor(top_p · Σe) (off when top_p >= 1): a radix select over the same keys whose histograms hold
//           masses, walking each level's bins from the top while the mass above stays within the limit
//   p_i     = e_i / Σe over the final kept set
//   pick(t) = the smallest index i whose inclusive prefix sum of the weights exceeds t, the weights summed in index
//           order over a hierarchy of contiguous segments (16 per level, one per warp), then one warp scan
//
// Masses are integers, so every histogram, sum and prefix is exact and independent of the order of the atomics and
// of the reduction; the one float reduction, the maximum, is order-independent too.
#pragma once
#include "common.cuh"

namespace lb {
namespace samp {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr unsigned long long kOne = 1ull << 40;   // the fixed-point mass of the row's maximum
constexpr double kOneD = 1099511627776.0;           // 2^40

struct Shared {
  unsigned long long hist[256];
  unsigned long long part[kWarps];
  float fpart[kWarps];
  unsigned long long b0, b1;
  unsigned u0;
  int i0;
};

__device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float ld(const float* p) { return *p; }

// one logits row and its temperature: z_i
template <typename T>
struct Row {
  const T* x;
  float temperature;
  __device__ __forceinline__ float z(int i) const { return __fdiv_rn(ld(x + i), temperature); }
};

// order-preserving key of a float (−0 and +0 share one key: they are equal logits)
__device__ __forceinline__ unsigned key_of(float z) {
  const unsigned u = z == 0.0f ? 0u : __float_as_uint(z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ unsigned long long fixed_mass(float z, float zmax) {
  return z == zmax ? kOne : __float2ull_rn(__expf(z - zmax) * 0x1p40f);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// the block's sum of v (every thread gets it)
__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, Shared& sh) {
  v = warp_sum(v);
  if (threadIdx.x % 32 == 0) sh.part[threadIdx.x / 32] = v;
  __syncthreads();
  unsigned long long s = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) s += sh.part[w];
  __syncthreads();
  return s;
}

__device__ __forceinline__ float block_max(float v, Shared& sh) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
  if (threadIdx.x % 32 == 0) sh.fpart[threadIdx.x / 32] = v;
  __syncthreads();
  float m = -INFINITY;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) m = fmaxf(m, sh.fpart[w]);
  __syncthreads();
  return m;
}

// a warped row: keep token i iff key_of(z_i) >= keep; total = Σ e_i over the kept tokens
struct Warped {
  float zmax;
  unsigned keep;
  unsigned long long total;
};

template <typename T>
__device__ __forceinline__ unsigned long long mass_of(const Row<T>& row, const Warped& w, int i) {
  const float z = row.z(i);
  return key_of(z) >= w.keep ? fixed_mass(z, w.zmax) : 0ull;
}

// the key of the k-th largest z (1 <= k <= V), counting duplicates
template <typename T>
__device__ unsigned topk_key(const Row<T>& row, int V, int k, Shared& sh) {
  unsigned prefix = 0, mask = 0;
  int remaining = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kThreads) sh.hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += kThreads) {
      const unsigned key = key_of(row.z(i));
      const bool in = (key & mask) == prefix;
      // most keys share a few bins: one atomic per bin and warp (the lowest lane of the bin's peers adds their count)
      const unsigned peers = __match_any_sync(__activemask(), in ? (key >> shift) & 255u : 256u);
      if (in && (threadIdx.x & 31) == __ffs(peers) - 1)
        atomicAdd(&sh.hist[(key >> shift) & 255u], (unsigned long long)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int d = 255;
      for (; d > 0; --d) {
        const int c = (int)sh.hist[d];
        if (remaining <= c) break;
        remaining -= c;
      }
      sh.u0 = prefix | ((unsigned)d << shift);
      sh.i0 = remaining;
    }
    __syncthreads();
    prefix = sh.u0;
    remaining = sh.i0;
    mask |= 255u << shift;
  }
  return prefix;
}

// top-p over the tokens with key >= w.keep: raises w.keep to the smallest kept key whose mass above is within
// floor(top_p · Σe), and sets w.total to the mass of the tokens it keeps
template <typename T>
__device__ void topp_key(const Row<T>& row, int V, float top_p, Warped& w, Shared& sh) {
  unsigned prefix = 0, mask = 0;
  unsigned long long above = 0, limit = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kThreads) sh.hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += kThreads) {
      const float z = row.z(i);
      const unsigned key = key_of(z);
      const bool in = key >= w.keep && (key & mask) == prefix;
      const unsigned long long m = in ? fixed_mass(z, w.zmax) : 0ull;
      // one atomic per bin and warp: the bin's peers sum their masses (m <= 2^40) in two exact 32-bit reductions of
      // 21 and 20 bits
      const unsigned peers = __match_any_sync(__activemask(), in ? (key >> shift) & 255u : 256u);
      const unsigned lo = __reduce_add_sync(peers, (unsigned)(m & 0x1fffffull));
      const unsigned hi = __reduce_add_sync(peers, (unsigned)(m >> 21));
      const unsigned long long sum = lo + ((unsigned long long)hi << 21);
      if (in && sum && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&sh.hist[(key >> shift) & 255u], sum);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (shift == 24) {
        unsigned long long s = 0;
        for (int d = 0; d < 256; ++d) s += sh.hist[d];
        limit = (unsigned long long)((double)top_p * (double)s);
      }
      // the lowest non-empty bin whose mass above is within the limit holds the answer (the mass above a bin grows
      // as the bins go down; the row's maximum has none above it, so the top bin always qualifies)
      int sel = 255;
      unsigned long long a = above, sel_above = above;
      for (int d = 255; d >= 0; --d) {
        const unsigned long long h = sh.hist[d];
        if (!h) continue;
        if (a > limit) break;
        sel = d, sel_above = a;
        a += h;
      }
      sh.u0 = prefix | ((unsigned)sel << shift);
      sh.b0 = sel_above;
      sh.b1 = sel_above + sh.hist[sel];   // at the last level: the kept mass
    }
    __syncthreads();
    prefix = sh.u0;
    above = sh.b0;
    mask |= 255u << shift;
    if (shift == 0) w.total = sh.b1;
    __syncthreads();
  }
  w.keep = prefix;
}

// the warp rule of one row
template <typename T>
__device__ Warped warp_row(const Row<T>& row, int V, int top_k, float top_p, Shared& sh) {
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += kThreads) m = fmaxf(m, row.z(i));
  Warped w;
  w.zmax = block_max(m, sh);
  w.keep = 0;
  w.total = 0;
  if (top_k > 0 && top_k < V) w.keep = topk_key(row, V, top_k, sh);
  if (top_p < 1.0f) {
    topp_key(row, V, top_p, w, sh);
  } else {
    unsigned long long s = 0;
    for (int i = threadIdx.x; i < V; i += kThreads) s += mass_of(row, w, i);
    w.total = block_sum(s, sh);
  }
  return w;
}

// pick(t) over weights wt(i), 0 <= t < Σ wt (every thread gets the index)
template <class W>
__device__ int pick(const W& wt, int V, unsigned long long t, Shared& sh) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  int lo = 0, hi = V;
  unsigned long long base = 0;
  while (hi - lo > 32) {
    const int seg = (hi - lo + kWarps - 1) / kWarps;
    const int s0 = lo + warp * seg, s1 = min(s0 + seg, hi);
    unsigned long long s = 0;
    for (int i = s0 + lane; i < s1; i += 32) s += wt(i);
    s = warp_sum(s);
    if (lane == 0) sh.part[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long b = base;
      int sel = 0;
      for (; sel < kWarps - 1; ++sel) {
        if (b + sh.part[sel] > t) break;
        b += sh.part[sel];
      }
      sh.b0 = b;
      sh.i0 = sel;
    }
    __syncthreads();
    base = sh.b0;
    lo += sh.i0 * seg;
    hi = min(lo + seg, hi);
    __syncthreads();
  }
  if (warp == 0) {
    const int i = lo + lane;
    unsigned long long v = i < hi ? wt(i) : 0ull;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const unsigned long long o = __shfl_up_sync(0xffffffffu, v, off);
      if (lane >= off) v += o;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, i < hi && base + v > t);
    if (lane == 0) sh.i0 = hit ? lo + __ffs(hit) - 1 : max(hi - 1, 0);
  }
  __syncthreads();
  const int idx = sh.i0;
  __syncthreads();
  return idx;
}

// t = floor(u · total) for a uniform u in [0, 1): below total
__device__ __forceinline__ unsigned long long draw(float u, unsigned long long total) {
  const unsigned long long t = (unsigned long long)((double)u * (double)total);
  return t < total ? t : total - 1;
}

}  // namespace samp
}  // namespace lb
