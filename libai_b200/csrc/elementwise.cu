// Bandwidth-bound fused kernels for sm_90a: bias+activation (fwd/bwd), bias+residual, SwiGLU,
// RoPE, column sums (bias gradients), vocab-parallel softmax cross entropy (stats + backward),
// fused AdamW over flat buffers, squared-norm reduction.  All use 128-bit accesses and grid-stride
// loops sized to the SM count.
//
// Reference call sites replaced: fused_bias_add_gelu (libai/layers/mlp.py:95), fused_bias_add_dropout
// (mlp.py:104, attention.py:265; p = 0 path), silu(gate)*up (projects/Llama/llama.py:111-113),
// apply_rotary_pos_emb (projects/Llama/llama.py:31-43), sparse_softmax_cross_entropy
// (libai/layers/cross_entropy.py:44), flow.optim.AdamW multi-tensor update (configs/common/optim.py).
#include "common.cuh"
#include <cuda_fp8.h>

namespace lb {

LB_DEVICE void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  uint4 q = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16(q.x), b = unpack_bf16(q.y), c = unpack_bf16(q.z), d = unpack_bf16(q.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
LB_DEVICE void st8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) =
      make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}

// y = act(x + bias)            (N % 8 == 0)
__global__ void bias_act_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ bias,
                                    __nv_bfloat16* __restrict__ y, size_t total_vec, int nvec_per_row, int act) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float v[8];
    ld8(x + i * 8, v);
    if (bias != nullptr) {
      float b[8];
      ld8(bias + (i % nvec_per_row) * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += b[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = act_fwd(v[j], act);
    st8(y + i * 8, v);
  }
}

// gx = gy * act'(x + bias)
__global__ void bias_act_bwd_kernel(const __nv_bfloat16* __restrict__ gy, const __nv_bfloat16* __restrict__ x,
                                    const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ gx,
                                    size_t total_vec, int nvec_per_row, int act) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float v[8], g[8];
    ld8(x + i * 8, v);
    ld8(gy + i * 8, g);
    if (bias != nullptr) {
      float b[8];
      ld8(bias + (i % nvec_per_row) * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += b[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= act_grad(v[j], act);
    st8(gx + i * 8, g);
  }
}

// y = x + bias + residual
__global__ void bias_residual_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ bias,
                                     const __nv_bfloat16* __restrict__ res, __nv_bfloat16* __restrict__ y,
                                     size_t total_vec, int nvec_per_row) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float v[8];
    ld8(x + i * 8, v);
    if (bias != nullptr) {
      float b[8];
      ld8(bias + (i % nvec_per_row) * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += b[j];
    }
    if (res != nullptr) {
      float r[8];
      ld8(res + i * 8, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += r[j];
    }
    st8(y + i * 8, v);
  }
}

// y = residual + dropout(x + bias) * 1/(1-p)     (reference: flow._C.fused_bias_add_dropout + the residual add,
// libai/layers/mlp.py:104, attention.py:265).  One Philox call (128 bits) decides 8 elements with 16 bits each:
// keep <=> u16 >= thresh, p_eff = thresh / 65536, scale = 65536 / (65536 - thresh) (exactly unbiased).  The mask is a
// function of (seed, offset, element index) only: the backward is the same kernel on the output gradient (bias =
// residual = nullptr) with the (seed, offset) pair the forward stored in `rng_out`.
__global__ void __launch_bounds__(256)
bias_dropout_residual_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ bias,
                             const __nv_bfloat16* __restrict__ res, __nv_bfloat16* __restrict__ y, size_t total_vec,
                             int nvec_per_row, uint32_t thresh, float scale, RngArgs rng, const long long* rng_in,
                             long long* rng_out) {
  unsigned long long seed, offset;
  if (rng_in != nullptr) {
    seed = static_cast<unsigned long long>(rng_in[0]);
    offset = static_cast<unsigned long long>(rng_in[1]);
  } else {
    rng_resolve(rng, seed, offset);
    if (rng_out != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
      rng_out[0] = static_cast<long long>(seed);
      rng_out[1] = static_cast<long long>(offset);
    }
  }
  const uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  const uint32_t o0 = static_cast<uint32_t>(offset), o1 = static_cast<uint32_t>(offset >> 32);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float v[8];
    ld8(x + i * 8, v);
    if (bias != nullptr) {
      float b[8];
      ld8(bias + (i % nvec_per_row) * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += b[j];
    }
    const uint4 rnd = philox4x32_7(static_cast<uint32_t>(i), static_cast<uint32_t>(i >> 32), o0, o1, k0, k1);
    const uint32_t w[4] = {rnd.x, rnd.y, rnd.z, rnd.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t u = (w[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu;
      v[j] = u >= thresh ? v[j] * scale : 0.f;
    }
    if (res != nullptr) {
      float r[8];
      ld8(res + i * 8, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += r[j];
    }
    st8(y + i * 8, v);
  }
}

__global__ void swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gate, const __nv_bfloat16* __restrict__ up,
                                  __nv_bfloat16* __restrict__ y, size_t total_vec) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float g[8], u[8];
    ld8(gate + i * 8, g);
    ld8(up + i * 8, u);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = g[j] / (1.0f + __expf(-g[j])) * u[j];
    st8(y + i * 8, g);
  }
}

// packed form: gu [T, 2F] = [gate | up] (the output of ONE GEMM against the stacked gate/up weights) -> y [T, F]
__global__ void swiglu_packed_fwd_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ y, size_t rows,
                                         size_t fvec /* F / 8 */) {
  const size_t total = rows * fvec;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / fvec, c = i % fvec;
    float g[8], u[8];
    ld8(gu + (r * 2 * fvec + c) * 8, g);
    ld8(gu + (r * 2 * fvec + fvec + c) * 8, u);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = g[j] / (1.0f + __expf(-g[j])) * u[j];
    st8(y + i * 8, g);
  }
}
// dgu [T, 2F] = [d gate | d up] from gy [T, F] and the saved gu
__global__ void swiglu_packed_bwd_kernel(const __nv_bfloat16* __restrict__ gy, const __nv_bfloat16* __restrict__ gu,
                                         __nv_bfloat16* __restrict__ dgu, size_t rows, size_t fvec) {
  const size_t total = rows * fvec;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / fvec, c = i % fvec;
    float g[8], u[8], d[8], dg[8], du[8];
    ld8(gu + (r * 2 * fvec + c) * 8, g);
    ld8(gu + (r * 2 * fvec + fvec + c) * 8, u);
    ld8(gy + i * 8, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.0f / (1.0f + __expf(-g[j]));
      du[j] = d[j] * g[j] * sg;
      dg[j] = d[j] * u[j] * sg * (1.0f + g[j] * (1.0f - sg));
    }
    st8(dgu + (r * 2 * fvec + c) * 8, dg);
    st8(dgu + (r * 2 * fvec + fvec + c) * 8, du);
  }
}

__global__ void swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ gy, const __nv_bfloat16* __restrict__ gate,
                                  const __nv_bfloat16* __restrict__ up, __nv_bfloat16* __restrict__ dgate,
                                  __nv_bfloat16* __restrict__ dup, size_t total_vec) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total_vec; i += (size_t)gridDim.x * blockDim.x) {
    float g[8], u[8], d[8], dg[8], du[8];
    ld8(gate + i * 8, g);
    ld8(up + i * 8, u);
    ld8(gy + i * 8, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = 1.0f / (1.0f + __expf(-g[j]));
      du[j] = d[j] * g[j] * s;
      dg[j] = d[j] * u[j] * s * (1.0f + g[j] * (1.0f - s));
    }
    st8(dgate + i * 8, dg);
    st8(dup + i * 8, du);
  }
}

// RoPE ("rotate_half" convention): x [B, A, S, D] contiguous, cos/sin fp32 [S, D]
//   fwd: y = x*cos + rot(x)*sin, rot(x) = cat(-x2, x1);   bwd: gx = g*cos + rot^T(g*sin) = g*cos - rot(g*sin) ... (below)
__global__ void rope_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ cosv,
                            const float* __restrict__ sinv, __nv_bfloat16* __restrict__ y, size_t rows, int S, int D,
                            int backward) {
  const int half = D / 2;
  const size_t total = rows * half;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / half;
    const int c = static_cast<int>(i % half);
    const int s = static_cast<int>(row % S);
    const float x1 = __bfloat162float(x[row * D + c]), x2 = __bfloat162float(x[row * D + c + half]);
    const float c1 = cosv[s * D + c], c2 = cosv[s * D + c + half];
    const float s1 = sinv[s * D + c], s2 = sinv[s * D + c + half];
    float y1, y2;
    if (!backward) {
      y1 = x1 * c1 - x2 * s1;
      y2 = x2 * c2 + x1 * s2;
    } else {
      y1 = x1 * c1 + x2 * s2;
      y2 = x2 * c2 - x1 * s1;
    }
    y[row * D + c] = __float2bfloat16(y1);
    y[row * D + c + half] = __float2bfloat16(y2);
  }
}

// Rotary embedding on the grouped packed QKV projection [tokens(b*s), G, r + 2, D] (per K/V group q_0 .. q_{r-1}, k, v;
// r = 1 is the per-head [q|k|v] layout): the r + 1 q/k slots are rotated with the position (s + pos_offset), v is
// copied.  `y` may alias `x` (in-place, used by the backward).
__global__ void rope_qkv_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ cosv,
                                const float* __restrict__ sinv, __nv_bfloat16* __restrict__ y, size_t groups, int S,
                                int G, int r, int D, int pos_offset, int backward, int copy_v) {
  const int half = D / 2;
  const int parts = copy_v ? r + 2 : r + 1;
  const size_t total = groups * parts * half;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = static_cast<int>(i % half);
    const int part = static_cast<int>((i / half) % parts);
    const size_t head = i / (static_cast<size_t>(half) * parts);   // token * G + group
    const size_t base = head * (r + 2) * D + static_cast<size_t>(part) * D;
    const float x1 = __bfloat162float(x[base + c]), x2 = __bfloat162float(x[base + c + half]);
    if (part == r + 1) {
      y[base + c] = x[base + c];
      y[base + c + half] = x[base + c + half];
      continue;
    }
    const int s = static_cast<int>((head / G) % S) + pos_offset;
    const float c1 = cosv[s * D + c], c2 = cosv[s * D + c + half];
    const float s1 = sinv[s * D + c], s2 = sinv[s * D + c + half];
    float y1, y2;
    if (!backward) {
      y1 = x1 * c1 - x2 * s1;
      y2 = x2 * c2 + x1 * s2;
    } else {
      y1 = x1 * c1 + x2 * s2;
      y2 = x2 * c2 - x1 * s1;
    }
    y[base + c] = __float2bfloat16(y1);
    y[base + c + half] = __float2bfloat16(y2);
  }
}

// part[blockIdx.y, c] = sum over the block's rows of x[r, c]: block = 32 column lanes (8 columns each, 16-byte loads) x
// 8 row stripes combined in shared memory.  The partials are summed in a fixed order by colsum_partials_kernel, so the
// result does not depend on the order in which blocks finish.
__global__ void __launch_bounds__(256) colsum_vec_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part,
                                                         int M, int N, int rows_per_block) {
  __shared__ float sm[8][32][9];
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  const int c8 = (blockIdx.x * 32 + tx) * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c8 < N) {
    int r = r0 + ty;
    for (; r + 24 < r1; r += 32) {  // four independent 16-byte loads in flight
      uint4 q[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) q[j] = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(r + j * 8) * N + c8);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = unpack_bf16(q[j].x), b = unpack_bf16(q[j].y), c = unpack_bf16(q[j].z), d = unpack_bf16(q[j].w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      }
    }
    for (; r < r1; r += 8) {
      const uint4 q = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(r) * N + c8);
      const float2 a = unpack_bf16(q.x), b = unpack_bf16(q.y), c = unpack_bf16(q.z), d = unpack_bf16(q.w);
      acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
      acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[ty][tx][j] = acc[j];
  __syncthreads();
  // 256 threads <-> 256 columns of the block
  const int col = threadIdx.x;
  const int gcol = blockIdx.x * 256 + col;
  if (gcol < N) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += sm[j][col / 8][col % 8];
    part[static_cast<size_t>(blockIdx.y) * N + gcol] = t;
  }
}

// part[blockIdx.y, c] = sum over the block's rows of x[r, c]  (any even N)
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part, int M, int N,
                              int rows_per_block) {
  const int c2 = blockIdx.x * blockDim.x + threadIdx.x;  // pair of columns
  if (c2 * 2 >= N) return;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float a0 = 0.f, a1 = 0.f;
  for (int r = r0; r < r1; ++r) {
    const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(x + static_cast<size_t>(r) * N + c2 * 2));
    a0 += v.x;
    a1 += v.y;
  }
  part[static_cast<size_t>(blockIdx.y) * N + c2 * 2] = a0;
  part[static_cast<size_t>(blockIdx.y) * N + c2 * 2 + 1] = a1;
}

// out[c] (+)= sum_b part[b, c], b in increasing order (one thread per column: coalesced, deterministic)
__global__ void __launch_bounds__(256) colsum_partials_kernel(const float* __restrict__ part, float* __restrict__ out,
                                                              int nparts, int N, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  float t = 0.f;
  for (int b = 0; b < nparts; ++b) t += part[static_cast<size_t>(b) * N + c];
  out[c] = accumulate ? out[c] + t : t;
}

// out[0] += sum of part[0, n): each lane sums a fixed stride, then a fixed shuffle tree (one warp)
__global__ void sum_partials_kernel(const float* __restrict__ part, int n, float* __restrict__ out) {
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += 32) acc += part[i];
  acc = warp_sum(acc);
  if (threadIdx.x == 0) out[0] += acc;
}

// ------------------------------------------------------------------------------------------------
// vocab-parallel cross entropy
// ------------------------------------------------------------------------------------------------
template <typename T>
LB_DEVICE float ld_logit(const T* p);
template <>
LB_DEVICE float ld_logit<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <>
LB_DEVICE float ld_logit<float>(const float* p) { return *p; }

// load 8 consecutive logits as floats (16-byte / 32-byte vector access)
template <typename T>
LB_DEVICE void ld_logits8(const T* p, float (&v)[8]);
template <>
LB_DEVICE void ld_logits8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) { ld8(p, v); }
template <>
LB_DEVICE void ld_logits8<float>(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <typename T>
LB_DEVICE void st_logits8(T* p, const float (&v)[8]);
template <>
LB_DEVICE void st_logits8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) { st8(p, v); }
template <>
LB_DEVICE void st_logits8<float>(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// per row: local max, sum exp(x - max), target logit (0 if the label lives on another rank)
template <typename T>
__global__ void __launch_bounds__(256) ce_stats_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                                                       float* __restrict__ mx_out, float* __restrict__ se_out,
                                                       float* __restrict__ tgt_out, int V, int64_t vocab_start) {
  __shared__ float sm[8], ss[8];
  const int row = blockIdx.x;
  const T* lr = logits + static_cast<size_t>(row) * V;
  float m = -INFINITY, s = 0.f;
  if (V % 8 == 0) {
    for (int c = threadIdx.x * 8; c < V; c += blockDim.x * 8) {
      float x[8];
      ld_logits8<T>(lr + c, x);
      float cm = x[0];
#pragma unroll
      for (int j = 1; j < 8; ++j) cm = fmaxf(cm, x[j]);
      if (cm == -INFINITY) continue;  // adds exp(-inf) = 0; with m = -inf the update below would add exp(-inf + inf)
      if (cm > m) {
        s *= __expf(m - cm);
        m = cm;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += __expf(x[j] - m);
    }
  } else {
    for (int c = threadIdx.x; c < V; c += blockDim.x) {
      const float x = ld_logit<T>(lr + c);
      if (x == -INFINITY) continue;
      if (x > m) {
        s = s * __expf(m - x) + 1.0f;
        m = x;
      } else {
        s += __expf(x - m);
      }
    }
  }
  const float wm = warp_max(m);
  s = (m == -INFINITY) ? 0.f : s * __expf(m - wm);
  s = warp_sum(s);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) {
    sm[warp] = wm;
    ss[warp] = s;
  }
  __syncthreads();
  if (warp == 0) {
    float m2 = lane < 8 ? sm[lane] : -INFINITY;
    float s2 = lane < 8 ? ss[lane] : 0.f;
    const float bm = warp_max(m2);
    s2 = (m2 == -INFINITY) ? 0.f : s2 * __expf(m2 - bm);
    s2 = warp_sum(s2);
    if (lane == 0) {
      mx_out[row] = bm;
      se_out[row] = s2;
      const int64_t local = labels[row] - vocab_start;
      tgt_out[row] = (local >= 0 && local < V) ? ld_logit<T>(lr + local) : 0.f;
    }
  }
}

// dlogits = (exp(x - lse) - onehot) * g[row]
template <typename T>
__global__ void __launch_bounds__(256) ce_bwd_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                                                     const float* __restrict__ lse, const float* __restrict__ gloss,
                                                     T* __restrict__ dlogits, int V, int64_t vocab_start) {
  const int row = blockIdx.x;
  const T* lr = logits + static_cast<size_t>(row) * V;
  T* dr = dlogits + static_cast<size_t>(row) * V;
  const float l = lse[row], g = gloss[row];
  const int64_t local = labels[row] - vocab_start;
  if (V % 8 == 0) {
    for (int c = threadIdx.x * 8; c < V; c += blockDim.x * 8) {
      float x[8];
      ld_logits8<T>(lr + c, x);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float p = __expf(x[j] - l);
        if (c + j == local) p -= 1.0f;
        x[j] = p * g;
      }
      st_logits8<T>(dr + c, x);
    }
  } else {
    for (int c = threadIdx.x; c < V; c += blockDim.x) {
      float p = __expf(ld_logit<T>(lr + c) - l);
      if (c == local) p -= 1.0f;
      dr[c] = static_cast<T>(p * g);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fused AdamW over flat fp32 buffers (+ optional low-precision parameter copy)
// ------------------------------------------------------------------------------------------------
__global__ void adamw_kernel(float* __restrict__ master, const float* __restrict__ grad, float* __restrict__ m,
                             float* __restrict__ v, __nv_bfloat16* __restrict__ lp_out,
                             const float* __restrict__ scale_ptr, size_t n, float lr, float b1, float b2, float eps,
                             float wd, float bc1, float bc2, int decoupled) {
  const float scale = scale_ptr != nullptr ? *scale_ptr : 1.0f;
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float4 p4 = reinterpret_cast<float4*>(master)[i];
    const float4 g4 = reinterpret_cast<const float4*>(grad)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i];
    float4 v4 = reinterpret_cast<float4*>(v)[i];
    float pp[4] = {p4.x, p4.y, p4.z, p4.w}, gg[4] = {g4.x, g4.y, g4.z, g4.w};
    float mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float g = gg[j] * scale;
      if (!decoupled) g += wd * pp[j];
      mm[j] = b1 * mm[j] + (1.0f - b1) * g;
      vv[j] = b2 * vv[j] + (1.0f - b2) * g * g;
      float upd = (mm[j] / bc1) / (sqrtf(vv[j] / bc2) + eps);
      if (decoupled) upd += wd * pp[j];
      pp[j] -= lr * upd;
    }
    reinterpret_cast<float4*>(master)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (lp_out != nullptr) {
      reinterpret_cast<uint2*>(lp_out)[i] = make_uint2(pack_bf16(pp[0], pp[1]), pack_bf16(pp[2], pp[3]));
    }
  }
}

// out[0] += sum x^2
// part[blockIdx.x] = sum of x[i]^2 over the block's grid-stride slice (summed in order by sum_partials_kernel)
__global__ void sqnorm_kernel(const float* __restrict__ x, float* __restrict__ part, size_t n) {
  __shared__ float sm[32];
  float acc = 0.f;
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const float4 q = reinterpret_cast<const float4*>(x)[i];
    acc += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // the n % 4 tail
    for (size_t i = nvec * 4; i < n; ++i) acc += x[i] * x[i];
  }
  acc = warp_sum(acc);
  if (threadIdx.x % 32 == 0) sm[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < blockDim.x / 32 ? sm[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) part[blockIdx.x] = t;
  }
}

// ---- embedding ---------------------------------------------------------------------------------------------------
// out[t, :] = table[ids[t] - vocab_start, :]  (zero row when the id belongs to another vocabulary shard)
__global__ void __launch_bounds__(128) embedding_fwd_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                                                            __nv_bfloat16* __restrict__ out, int H, long vocab_start, long rows) {
  const long t = blockIdx.x;
  const long r = ids[t] - vocab_start;
  const bool inside = r >= 0 && r < rows;
  const uint4* src = reinterpret_cast<const uint4*>(table + (inside ? r : 0) * H);
  uint4* dst = reinterpret_cast<uint4*>(out + t * H);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) dst[i] = inside ? src[i] : make_uint4(0, 0, 0, 0);
}

// grad_table[ids[t] - vocab_start, :] += gy[t, :]   (fp32 main-grad buffer; the tied LM-head wgrad accumulates into the
// same buffer).  The ids arrive sorted (stable) with their token positions: the block of the first token of every run
// of equal ids sums the run in token order and is the only writer of that row, so the result is deterministic.
__global__ void __launch_bounds__(128) embedding_bwd_kernel(const int64_t* __restrict__ sorted_ids,
                                                            const int64_t* __restrict__ order,
                                                            const __nv_bfloat16* __restrict__ gy, float* __restrict__ grad,
                                                            long T, int H, long vocab_start, long rows) {
  const long t = blockIdx.x;
  const int64_t id = sorted_ids[t];
  if (t > 0 && sorted_ids[t - 1] == id) return;
  const long r = id - vocab_start;
  if (r < 0 || r >= rows) return;
  float* dst = grad + r * H;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long u = t; u < T && sorted_ids[u] == id; ++u) {
      const uint4 q = reinterpret_cast<const uint4*>(gy + order[u] * H)[i];
      const float2 a = unpack_bf16(q.x), b = unpack_bf16(q.y), c = unpack_bf16(q.z), d = unpack_bf16(q.w);
      acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
      acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
    }
    float4* d4 = reinterpret_cast<float4*>(dst + i * 8);
    const float4 o0 = d4[0], o1 = d4[1];
    d4[0] = make_float4(o0.x + acc[0], o0.y + acc[1], o0.z + acc[2], o0.w + acc[3]);
    d4[1] = make_float4(o1.x + acc[4], o1.y + acc[5], o1.z + acc[6], o1.w + acc[7]);
  }
}

}  // namespace lb

namespace {
int ew_grid(size_t work, int block) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  size_t need = (work + block - 1) / block;
  size_t cap = (size_t)sms * 8;
  return (int)(need < cap ? (need == 0 ? 1 : need) : cap);
}
}  // namespace

using bf16 = __nv_bfloat16;

extern "C" int lb_bias_act_fwd(const void* x, const void* bias, void* y, long rows, int N, int act, cudaStream_t s) {
  if (N % 8) return -1;
  const size_t tv = (size_t)rows * N / 8;
  if (tv == 0) return 0;
  lb::bias_act_fwd_kernel<<<ew_grid(tv, 256), 256, 0, s>>>((const bf16*)x, (const bf16*)bias, (bf16*)y, tv, N / 8, act);
  return (int)cudaGetLastError();
}
extern "C" int lb_bias_act_bwd(const void* gy, const void* x, const void* bias, void* gx, long rows, int N, int act,
                               cudaStream_t s) {
  if (N % 8) return -1;
  const size_t tv = (size_t)rows * N / 8;
  if (tv == 0) return 0;
  lb::bias_act_bwd_kernel<<<ew_grid(tv, 256), 256, 0, s>>>((const bf16*)gy, (const bf16*)x, (const bf16*)bias,
                                                           (bf16*)gx, tv, N / 8, act);
  return (int)cudaGetLastError();
}
extern "C" int lb_bias_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N,
                                cudaStream_t s) {
  if (N % 8) return -1;
  const size_t tv = (size_t)rows * N / 8;
  if (tv == 0) return 0;
  lb::bias_residual_kernel<<<ew_grid(tv, 256), 256, 0, s>>>((const bf16*)x, (const bf16*)bias, (const bf16*)res,
                                                            (bf16*)y, tv, N / 8);
  return (int)cudaGetLastError();
}
// p in [0, 1): drop probability.  rng_in != nullptr: reuse a stored (seed, offset) pair (backward); else resolve `rng`
// and store the pair into rng_out (if given).
extern "C" int lb_bias_dropout_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N, float p,
                                        const lb::RngArgs* rng, const long long* rng_in, long long* rng_out,
                                        cudaStream_t s) {
  if (N % 8) return -1;
  const size_t tv = (size_t)rows * N / 8;
  if (tv == 0) return 0;
  uint32_t thresh = (uint32_t)(p * 65536.0f + 0.5f);
  if (thresh > 65535u) thresh = 65535u;
  const float scale = 65536.0f / (65536.0f - (float)thresh);
  lb::RngArgs r{};
  if (rng != nullptr) r = *rng;
  lb::bias_dropout_residual_kernel<<<ew_grid(tv, 256), 256, 0, s>>>((const bf16*)x, (const bf16*)bias, (const bf16*)res,
                                                                    (bf16*)y, tv, N / 8, thresh, scale, r, rng_in, rng_out);
  return (int)cudaGetLastError();
}
extern "C" int lb_swiglu_fwd(const void* gate, const void* up, void* y, long n, cudaStream_t s) {
  if (n % 8) return -1;
  if (n == 0) return 0;
  lb::swiglu_fwd_kernel<<<ew_grid(n / 8, 256), 256, 0, s>>>((const bf16*)gate, (const bf16*)up, (bf16*)y, n / 8);
  return (int)cudaGetLastError();
}
extern "C" int lb_swiglu_bwd(const void* gy, const void* gate, const void* up, void* dgate, void* dup, long n,
                             cudaStream_t s) {
  if (n % 8) return -1;
  if (n == 0) return 0;
  lb::swiglu_bwd_kernel<<<ew_grid(n / 8, 256), 256, 0, s>>>((const bf16*)gy, (const bf16*)gate, (const bf16*)up,
                                                            (bf16*)dgate, (bf16*)dup, n / 8);
  return (int)cudaGetLastError();
}
extern "C" int lb_swiglu_packed_fwd(const void* gu, void* y, long rows, long F, cudaStream_t s) {
  if (F % 8) return -1;
  if (rows == 0) return 0;
  lb::swiglu_packed_fwd_kernel<<<ew_grid(rows * F / 8, 256), 256, 0, s>>>((const bf16*)gu, (bf16*)y, (size_t)rows, (size_t)(F / 8));
  return (int)cudaGetLastError();
}
extern "C" int lb_swiglu_packed_bwd(const void* gy, const void* gu, void* dgu, long rows, long F, cudaStream_t s) {
  if (F % 8) return -1;
  if (rows == 0) return 0;
  lb::swiglu_packed_bwd_kernel<<<ew_grid(rows * F / 8, 256), 256, 0, s>>>((const bf16*)gy, (const bf16*)gu, (bf16*)dgu,
                                                                         (size_t)rows, (size_t)(F / 8));
  return (int)cudaGetLastError();
}
extern "C" int lb_rope(const void* x, const float* cosv, const float* sinv, void* y, long rows, int S, int D,
                       int backward, cudaStream_t s) {
  if (rows == 0) return 0;
  lb::rope_kernel<<<ew_grid((size_t)rows * D / 2, 256), 256, 0, s>>>((const bf16*)x, cosv, sinv, (bf16*)y,
                                                                     (size_t)rows, S, D, backward);
  return (int)cudaGetLastError();
}
// groups = tokens * G; r query heads per group
extern "C" int lb_rope_qkv(const void* x, const float* cosv, const float* sinv, void* y, long groups, int S, int G, int r,
                           int D, int pos_offset, int backward, cudaStream_t s) {
  if (groups == 0) return 0;
  const int copy_v = (x != y);
  lb::rope_qkv_kernel<<<ew_grid((size_t)groups * (copy_v ? r + 2 : r + 1) * D / 2, 256), 256, 0, s>>>(
      (const bf16*)x, cosv, sinv, (bf16*)y, (size_t)groups, S, G, r, D, pos_offset, backward, copy_v);
  return (int)cudaGetLastError();
}
// rows per block of the column-sum pass; the number of row blocks is the row count of its fp32 workspace [.., N]
static int colsum_rows_per_block(int M, int N) {
  if (N % 8) return 128;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int col_blocks = (N + 255) / 256;
  int row_blocks = (2 * sms + col_blocks - 1) / col_blocks;  // ~2 blocks per SM
  if (row_blocks > (M + 63) / 64) row_blocks = (M + 63) / 64;
  if (row_blocks < 1) row_blocks = 1;
  return (M + row_blocks - 1) / row_blocks;
}
extern "C" int lb_colsum_workspace_rows(int M, int N) {
  if (M <= 0) return 1;
  const int rpb = colsum_rows_per_block(M, N);
  return (M + rpb - 1) / rpb;
}
// out[c] (+)= sum_r x[r, c]; workspace: fp32 [lb_colsum_workspace_rows(M, N), N]
extern "C" int lb_colsum(const void* x, float* out, int M, int N, int accumulate, float* workspace, cudaStream_t s) {
  if (N % 2) return -1;
  if (M == 0) {
    if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float) * N, s);
    return 0;
  }
  const int rpb = colsum_rows_per_block(M, N);
  const int row_blocks = (M + rpb - 1) / rpb;
  if (N % 8 == 0) {
    lb::colsum_vec_kernel<<<dim3((N + 255) / 256, row_blocks), 256, 0, s>>>((const bf16*)x, workspace, M, N, rpb);
  } else {
    lb::colsum_kernel<<<dim3((N / 2 + 127) / 128, row_blocks), 128, 0, s>>>((const bf16*)x, workspace, M, N, rpb);
  }
  lb::colsum_partials_kernel<<<(N + 255) / 256, 256, 0, s>>>(workspace, out, row_blocks, N, accumulate);
  return (int)cudaGetLastError();
}
extern "C" int lb_ce_stats(const void* logits, const int64_t* labels, float* mx, float* se, float* tgt, int T, int V,
                           long vocab_start, int dtype, cudaStream_t s) {
  if (T == 0) return 0;
  if (dtype == 0)
    lb::ce_stats_kernel<bf16><<<T, 256, 0, s>>>((const bf16*)logits, labels, mx, se, tgt, V, vocab_start);
  else
    lb::ce_stats_kernel<float><<<T, 256, 0, s>>>((const float*)logits, labels, mx, se, tgt, V, vocab_start);
  return (int)cudaGetLastError();
}
extern "C" int lb_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* gloss, void* dlogits,
                         int T, int V, long vocab_start, int dtype, cudaStream_t s) {
  if (T == 0) return 0;
  if (dtype == 0)
    lb::ce_bwd_kernel<bf16><<<T, 256, 0, s>>>((const bf16*)logits, labels, lse, gloss, (bf16*)dlogits, V, vocab_start);
  else
    lb::ce_bwd_kernel<float><<<T, 256, 0, s>>>((const float*)logits, labels, lse, gloss, (float*)dlogits, V,
                                               vocab_start);
  return (int)cudaGetLastError();
}
extern "C" int lb_adamw(float* master, const float* grad, float* m, float* v, void* lp_out, const float* scale,
                        long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, int decoupled,
                        cudaStream_t s) {
  if (n % 4) return -1;
  if (n == 0) return 0;
  lb::adamw_kernel<<<ew_grid(n / 4, 256), 256, 0, s>>>(master, grad, m, v, (bf16*)lp_out, scale, (size_t)n, lr, b1, b2,
                                                       eps, wd, bc1, bc2, decoupled);
  return (int)cudaGetLastError();
}
extern "C" int lb_embedding_fwd(const int64_t* ids, const void* table, void* out, long T, int H, long vocab_start, long rows,
                                cudaStream_t s) {
  if (T == 0) return 0;
  if (H % 8) return -1;
  lb::embedding_fwd_kernel<<<(unsigned)T, 128, 0, s>>>(ids, (const bf16*)table, (bf16*)out, H, vocab_start, rows);
  return (int)cudaGetLastError();
}
// sorted_ids / order: the ids sorted stably and their token positions
extern "C" int lb_embedding_bwd(const int64_t* sorted_ids, const int64_t* order, const void* gy, float* grad, long T, int H,
                                long vocab_start, long rows, cudaStream_t s) {
  if (T == 0) return 0;
  if (H % 8) return -1;
  lb::embedding_bwd_kernel<<<(unsigned)T, 128, 0, s>>>(sorted_ids, order, (const bf16*)gy, grad, T, H, vocab_start, rows);
  return (int)cudaGetLastError();
}
extern "C" int lb_sqnorm_workspace(long n) { return ew_grid(n / 4, 256); }
// out[0] += sum x^2; workspace: fp32 [lb_sqnorm_workspace(n)]
extern "C" int lb_sqnorm(const float* x, float* out, long n, float* workspace, cudaStream_t s) {
  if (n == 0) return 0;  // (the kernel handles the n % 4 tail)
  const int grid = ew_grid(n / 4, 256);
  lb::sqnorm_kernel<<<grid, 256, 0, s>>>(x, workspace, (size_t)n);
  lb::sum_partials_kernel<<<1, 32, 0, s>>>(workspace, grid, out);
  return (int)cudaGetLastError();
}


// ---------------------------------------------------------------------------------------------------------------
// fp8 (E4M3) per-tensor quantisation for the fp8 forward GEMM: amax pass + cast pass, no host synchronisation
//   amax : max |x| over the tensor (atomicMax on the bit pattern: non-negative floats order like unsigned ints)
//   cast : q = sat_e4m3(x * 448 / amax); deq[0] = amax / 448
// ---------------------------------------------------------------------------------------------------------------
namespace {
__global__ void amax_bf16_kernel(const uint4* __restrict__ x, long n8, const __nv_bfloat16* __restrict__ tail, int ntail,
                                 unsigned* __restrict__ amax_bits) {
  float m = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // |bf16| pairs: clear both sign bits, the larger half decides
      const unsigned a = w[j] & 0x7FFF7FFFu;
      m = fmaxf(m, __uint_as_float(a << 16));
      m = fmaxf(m, __uint_as_float(a & 0xFFFF0000u));
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < ntail) m = fmaxf(m, fabsf(__bfloat162float(tail[threadIdx.x])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));
}

__global__ void quant_e4m3_kernel(const uint4* __restrict__ x, long n8, const __nv_bfloat16* __restrict__ tail, int ntail,
                                  const unsigned* __restrict__ amax_bits, uint2* __restrict__ q, uint8_t* __restrict__ qtail,
                                  float* __restrict__ deq) {
  const float amax = fmaxf(__uint_as_float(*amax_bits), 1e-12f);
  const float scale = 448.0f / amax;
  if (blockIdx.x == 0 && threadIdx.x == 0) deq[0] = amax / 448.0f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    unsigned short h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = make_float2(__uint_as_float(w[j] << 16) * scale, __uint_as_float(w[j] & 0xFFFF0000u) * scale);
      h[j] = __nv_cvt_float2_to_fp8x2(f, __NV_SATFINITE, __NV_E4M3);
    }
    q[i] = make_uint2((unsigned)h[0] | ((unsigned)h[1] << 16), (unsigned)h[2] | ((unsigned)h[3] << 16));
  }
  if (blockIdx.x == 0 && threadIdx.x < ntail)
    qtail[threadIdx.x] = __nv_cvt_float_to_fp8(__bfloat162float(tail[threadIdx.x]) * scale, __NV_SATFINITE, __NV_E4M3);
}
}  // namespace

// x: bf16 [n] (16-byte aligned), q: e4m3 bytes [n] (8-byte aligned), amax_scratch: one uint32 the caller has zeroed
// (a kernel-node fill rather than a memset node keeps captured graphs homogeneous),
// deq: one float (the dequantisation scale).
extern "C" int lb_quant_e4m3(const void* x, void* q, void* amax_scratch, float* deq, long n, cudaStream_t s) {
  if (n <= 0) return 0;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(q) & 7)) return -1;
  const long n8 = n / 8;
  const int ntail = (int)(n - n8 * 8);
  const __nv_bfloat16* tail = reinterpret_cast<const __nv_bfloat16*>(x) + n8 * 8;
  long blocks = (n8 + 255) / 256;
  if (blocks < 1) blocks = 1;
  const long cap = ew_grid(~size_t(0) >> 1, 1);   // 8 blocks per SM
  if (blocks > cap) blocks = cap;
  amax_bf16_kernel<<<(int)blocks, 256, 0, s>>>(reinterpret_cast<const uint4*>(x), n8, tail, ntail,
                                              reinterpret_cast<unsigned*>(amax_scratch));
  quant_e4m3_kernel<<<(int)blocks, 256, 0, s>>>(reinterpret_cast<const uint4*>(x), n8, tail, ntail,
                                               reinterpret_cast<const unsigned*>(amax_scratch),
                                               reinterpret_cast<uint2*>(q), reinterpret_cast<uint8_t*>(q) + n8 * 8, deq);
  return (int)cudaGetLastError();
}
