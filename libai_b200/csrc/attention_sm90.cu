// Flash attention for sm_90a on wgmma / TMA / mbarrier (head dim 64 or 128, causal or full, bf16).
//
// Replaces the score GEMM + fused_scale_(tril_)softmax(_mask)_dropout + context GEMM sequence of the
// reference (libai/layers/attention.py:211-253): no [b, a, s, s] tensor and no materialised mask.
// Q/K/V are read straight out of the packed QKV projection through strided 4-D TMA tensor maps
// ([B, A, S, D] views), O is written in [B, S, A, D] so the output projection consumes it as-is.
//
// Forward, one CTA per (batch, head, 128-query block), 384 threads:
//   warpgroup 0  TMA producer (one elected thread): Q once, then K/V tiles of 128 keys (double buffered); it gives
//                its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2  consumers, 64 query rows each: S = Q·K_jᵀ (wgmma, accumulators in registers) →
//                online softmax (exp2) in registers → P (bf16) stays in registers as the A operand of O += P·V_j
#include "common.cuh"

#include <cstdlib>
#include <cstring>

namespace lb {

constexpr int ATT_BM = 128;   // queries per CTA (forward)
constexpr int ATT_BN = 128;   // keys per tile (forward)
constexpr int ATT_FWD_THREADS = 384;
constexpr int ATT_BWD_BN = 64;   // keys per CTA (backward)
constexpr int ATT_BWD_BM = 64;   // queries per step (backward)
constexpr int ATT_BWD_THREADS = 160;

struct AttnFwdParams {
  __nv_bfloat16* o;   // [B, S, A, D]
  float* lse;         // [B, A, S]
  int B, A, S;
  int causal;
  float scale_log2;   // scale * log2(e)
  float scale;
  const int* kv_lens; // optional [B]: number of valid keys per sample (right-padded batches)
  // additive score bias (v2 kernel): dense bf16 [.., S, S] with (batch, head, query) strides in elements (0 = broadcast;
  // T5 relative-position bias, Swin/BERT style masks) or ALiBi slopes per head (bias = slope * (key - query))
  const __nv_bfloat16* bias;
  long bias_strides[3];
  const float* alibi_slopes;
  // attention dropout on P (v2 kernel): keep <=> philox byte >= drop_thresh; O is scaled by inv_keep
  uint32_t drop_thresh;
  float inv_keep;
  RngArgs rng;
  long long* rng_out;   // [2]: the (seed, offset) pair used, for the backward
};

enum AttnBias : int { BIAS_NONE = 0, BIAS_DENSE = 1, BIAS_ALIBI = 2 };

// 16 random bytes for keys [16 g, 16 g + 16) of query row q_idx of (batch, head) slice bh
LB_DEVICE uint4 attn_dropout_bytes(uint32_t q_idx, uint32_t g, uint32_t bh, unsigned long long seed, unsigned long long offset) {
  return philox4x32_7(q_idx, g, bh ^ (static_cast<uint32_t>(offset >> 32) << 20), static_cast<uint32_t>(offset),
                      static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
}
LB_DEVICE uint32_t rnd_byte(const uint4& r, int i) {   // i in [0, 16)
  const uint32_t w = (i < 4) ? r.x : (i < 8 ? r.y : (i < 12 ? r.z : r.w));
  return (w >> ((i & 3) * 8)) & 0xFFu;
}
// bf16 pair of an fp32 accumulator fragment: the m64nN accumulator layout of columns [16 kk, 16 kk + 16) is exactly the
// A-operand register layout of an m64k16 wgmma, so P (or dSᵀ) feeds the next MMA without a trip through shared memory
LB_DEVICE void acc_to_a_frag(const float* d, uint32_t (&a)[4]) {
  a[0] = pack_bf16(d[0], d[1]);
  a[1] = pack_bf16(d[2], d[3]);
  a[2] = pack_bf16(d[4], d[5]);
  a[3] = pack_bf16(d[6], d[7]);
}

template <int D>
struct AttnFwdCfg {
  static constexpr int CHUNKS = D / 64;                    // 64-element (128B) chunks of a row
  static constexpr int TILE_BYTES = ATT_BN * D * 2;        // one Q / K / V tile
  static constexpr int SMEM_BYTES = 5 * TILE_BYTES + 1024 + 256;   // Q + 2 x (K, V)
};

template <int D, int BIAS, bool DROP>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, AttnFwdParams p) {
  using Cfg = AttnFwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::TILE_BYTES;
  uint8_t* sV = sK + 2 * Cfg::TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * Cfg::TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;   // 2
  uint64_t* k_empty = bars + 3;  // 2
  uint64_t* v_full = bars + 5;   // 2
  uint64_t* v_empty = bars + 7;  // 2

  const int warp_idx = threadIdx.x / 32;
  // heavy (late) query blocks first: better tail behaviour under the causal mask
  const int q_blk = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);
  const int head = blockIdx.y, batch = blockIdx.z;
  const int q0 = q_blk * ATT_BM;
  const int kv_len = p.kv_lens != nullptr ? max(1, min(p.S, p.kv_lens[batch])) : p.S;
  int nkv = (kv_len + ATT_BN - 1) / ATT_BN;
  if (p.causal) nkv = min(nkv, q_blk + 1);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 256);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 256);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp_idx < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp_idx == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, Cfg::TILE_BYTES);
#pragma unroll
      for (int c = 0; c < Cfg::CHUNKS; ++c)
        tma_load_4d(sQ + c * (ATT_BM * 128), &tmap_q, q_full, c * 64, q0, head, batch);
      for (int j = 0; j < nkv; ++j) {
        const int b = j & 1;
        const uint32_t par = ((j >> 1) & 1) ^ 1;
        mbar_wait(&k_empty[b], par);
        mbar_arrive_expect_tx(&k_full[b], Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c)
          tma_load_4d(sK + b * Cfg::TILE_BYTES + c * (ATT_BN * 128), &tmap_k, &k_full[b], c * 64, j * ATT_BN, head, batch);
        mbar_wait(&v_empty[b], par);
        mbar_arrive_expect_tx(&v_full[b], Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c)
          tma_load_4d(sV + b * Cfg::TILE_BYTES + c * (ATT_BN * 128), &tmap_v, &v_full[b], c * 64, j * ATT_BN, head, batch);
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
  const int wg = warp_idx / 4 - 1;
  const int t = threadIdx.x % 128;
  const int r_loc = 64 * wg + 16 * (t / 32) + (t % 32) / 4;   // this thread's rows: r_loc and r_loc + 8
  const int cq = 2 * (t % 4);                                  // its columns inside every 8-column group: cq, cq + 1
  int q_idx[2], key_lim[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    q_idx[h] = q0 + r_loc + 8 * h;
    key_lim[h] = p.causal ? min(kv_len, q_idx[h] + 1) : kv_len;   // keys [0, key_lim) are visible to this row
  }
  constexpr float LOG2E = 1.4426950408889634f;
  unsigned long long rng_seed = 0, rng_offset = 0;
  if constexpr (DROP) {
    rng_resolve(p.rng, rng_seed, rng_offset);
    if (p.rng_out != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 128) {
      p.rng_out[0] = static_cast<long long>(rng_seed);
      p.rng_out[1] = static_cast<long long>(rng_offset);
    }
  }
  const uint32_t bh = static_cast<uint32_t>(batch * p.A + head);
  const __nv_bfloat16* bias_row[2] = {nullptr, nullptr};
  float slope2 = 0.f;
  if constexpr (BIAS == BIAS_DENSE) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      bias_row[h] = p.bias + batch * p.bias_strides[0] + head * p.bias_strides[1] +
                    static_cast<long>(min(q_idx[h], p.S - 1)) * p.bias_strides[2];
  }
  if constexpr (BIAS == BIAS_ALIBI) slope2 = p.alibi_slopes[head] * LOG2E;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
  mbar_wait(q_full, 0);

  for (int j = 0; j < nkv; ++j) {
    const int b = j & 1;
    const uint32_t par = (j >> 1) & 1;
    // ---- S = Q·K_jᵀ (64 x 128 per warpgroup)
    float s[ATT_BN / 2];
    mbar_wait(&k_full[b], par);
    const uint32_t k_addr = smem_u32(sK + b * Cfg::TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t off = (kk / 4) * (ATT_BM * 128) + (kk % 4) * 32;
      wgmma_bf16_ss<ATT_BN, 0, 0>(s, make_smem_desc_sw128(q_addr + off, 0, 1024),
                                  make_smem_desc_sw128(k_addr + (kk / 4) * (ATT_BN * 128) + (kk % 4) * 32, 0, 1024),
                                  kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    mbar_arrive(&k_empty[b]);

    // ---- scores in the log2 domain, masked
    const int kbase = j * ATT_BN;
    const bool need_mask = (p.causal && j == q_blk) || (kbase + ATT_BN > kv_len);
#pragma unroll
    for (int jj = 0; jj < ATT_BN / 8; ++jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int kidx = kbase + 8 * jj + cq + c;
          float x = s[4 * jj + 2 * h + c] * p.scale_log2;
          if constexpr (BIAS == BIAS_DENSE) {
            const int kb = kbase + 8 * jj + cq;
            const float2 f = kb < p.S ? unpack_bf16(*reinterpret_cast<const uint32_t*>(bias_row[h] + kb)) : make_float2(0.f, 0.f);
            x = fmaf(c ? f.y : f.x, LOG2E, x);
          } else if constexpr (BIAS == BIAS_ALIBI) {
            x = fmaf(slope2, static_cast<float>(kidx - q_idx[h]), x);
          }
          if (need_mask && kidx >= key_lim[h]) x = -INFINITY;
          s[4 * jj + 2 * h + c] = x;
        }
      }
    }
    // ---- online softmax: row max over the 4 lanes sharing a row, rescale O and the running sum
    float m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < ATT_BN / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = fast_exp2(m_run[h] - m_use[h]);   // 0 on the first block
      m_run[h] = m_new;
      l_run[h] *= alpha;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj) {
        o[4 * jj + 2 * h] *= alpha;
        o[4 * jj + 2 * h + 1] *= alpha;
      }
    }
    // ---- P = exp2(s - m): the normaliser sums the UNdropped probabilities, P·V takes the dropped ones
    uint32_t pa[ATT_BN / 16][4];
#pragma unroll
    for (int g = 0; g < ATT_BN / 16; ++g) {
      uint4 rnd[2];
      if constexpr (DROP) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          rnd[h] = attn_dropout_bytes(static_cast<uint32_t>(q_idx[h]), static_cast<uint32_t>((kbase >> 4) + g), bh, rng_seed, rng_offset);
      }
      float e[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        // u = 4 * (jj - 2 g) + 2 h + c: key 16 g + 8 (jj - 2 g) + cq + c of row h
        const int h = (u >> 1) & 1, c = u & 1, half8 = u >> 2;
        float v = fast_exp2(s[8 * g + u] - m_use[h]);
        l_run[h] += v;
        if constexpr (DROP) {
          if (rnd_byte(rnd[h], 8 * half8 + cq + c) < p.drop_thresh) v = 0.f;
        }
        e[u] = v;
      }
      acc_to_a_frag(e, pa[g]);
    }
    // ---- O += P·V_j
    mbar_wait(&v_full[b], par);
    const uint32_t v_addr = smem_u32(sV + b * Cfg::TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      wgmma_bf16_rs<D, 1>(o, pa[kk], make_smem_desc_sw128(v_addr + kk * (16 * 128), ATT_BN * 128, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    mbar_arrive(&v_empty[b]);
  }

  // ---- epilogue: O / l  →  [B, S, A, D]; lse in natural log
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? (DROP ? p.inv_keep : 1.0f) / l : 0.f;
    if (q_idx[h] < p.S) {
      __nv_bfloat16* orow = p.o + ((static_cast<size_t>(batch) * p.S + q_idx[h]) * p.A + head) * D;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + cq) = pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      if (t % 4 == 0)
        p.lse[(static_cast<size_t>(batch) * p.A + head) * p.S + q_idx[h]] =
            (m_run[h] == -INFINITY) ? -INFINITY : (m_run[h] + log2f(l)) * 0.6931471805599453f;
    }
  }
}

}  // namespace lb

namespace {
// dims innermost first: {D, S, A, B}; st = {batch, head, seq} strides in elements; boxes of 64 columns x `rows` rows
bool make_qkv_tmap(CUtensorMap* m, const void* ptr, int B, int A, int S, int D, const long* st, int rows) {
  uint64_t dims[4] = {(uint64_t)D, (uint64_t)S, (uint64_t)A, (uint64_t)B};
  uint64_t strides[4] = {2, (uint64_t)st[2] * 2, (uint64_t)st[1] * 2, (uint64_t)st[0] * 2};
  uint32_t box[4] = {64, (uint32_t)rows, 1, 1};
  return lb_host::make_tmap_bf16(m, ptr, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int D, int BIAS, bool DROP>
cudaError_t launch_fwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const lb::AttnFwdParams& p,
                         cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = lb::attn_fwd_kernel<D, BIAS, DROP>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid((p.S + lb::ATT_BM - 1) / lb::ATT_BM, p.A, p.B);
  kern<<<grid, lb::ATT_FWD_THREADS, Cfg::SMEM_BYTES, s>>>(tq, tk, tv, p);
  return cudaGetLastError();
}

template <int D>
cudaError_t launch_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const lb::AttnFwdParams& p,
                       cudaStream_t s) {
  const int bias = p.bias != nullptr ? lb::BIAS_DENSE : (p.alibi_slopes != nullptr ? lb::BIAS_ALIBI : lb::BIAS_NONE);
  const bool drop = p.drop_thresh > 0;
  if (bias == lb::BIAS_NONE) return drop ? launch_fwd_t<D, lb::BIAS_NONE, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_NONE, false>(tq, tk, tv, p, s);
  if (bias == lb::BIAS_DENSE) return drop ? launch_fwd_t<D, lb::BIAS_DENSE, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_DENSE, false>(tq, tk, tv, p, s);
  return drop ? launch_fwd_t<D, lb::BIAS_ALIBI, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_ALIBI, false>(tq, tk, tv, p, s);
}
}  // namespace
// p_drop in [0, 1): attention dropout probability (quantised to 1/256 like the byte-threshold test of the kernel);
// bias (optional, bf16): dense additive score bias with (batch, head, query-row) strides in elements, key stride 1;
// alibi_slopes (optional, fp32 [A]).
extern "C" int lb_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int A, int S, int D,
                           const long* q_strides, const long* k_strides, const long* v_strides, int causal, float scale,
                           const int* kv_lens, const void* bias, const long* bias_strides, const float* alibi_slopes,
                           float p_drop, const lb::RngArgs* rng, long long* rng_out, cudaStream_t s) {
  if (D != 64 && D != 128) return -1;
  for (int i = 0; i < 3; ++i)
    if ((q_strides[i] % 8) || (k_strides[i] % 8) || (v_strides[i] % 8)) return -3;
  CUtensorMap tq, tk, tv;
  if (!make_qkv_tmap(&tq, q, B, A, S, D, q_strides, 128)) return -2;
  if (!make_qkv_tmap(&tk, k, B, A, S, D, k_strides, 128)) return -2;
  if (!make_qkv_tmap(&tv, v, B, A, S, D, v_strides, 128)) return -2;
  lb::AttnFwdParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.B = B;
  p.A = A;
  p.S = S;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.kv_lens = kv_lens;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  for (int i = 0; i < 3; ++i) p.bias_strides[i] = (bias != nullptr && bias_strides != nullptr) ? bias_strides[i] : 0;
  if (bias != nullptr && ((p.bias_strides[0] | p.bias_strides[1] | p.bias_strides[2]) % 8 || (reinterpret_cast<uintptr_t>(bias) & 15)))
    return -3;
  p.alibi_slopes = bias != nullptr ? nullptr : alibi_slopes;
  uint32_t thr = (uint32_t)(p_drop * 256.0f + 0.5f);
  if (thr > 255u) thr = 255u;
  p.drop_thresh = (p_drop > 0.f && rng != nullptr) ? (thr == 0 ? 1u : thr) : 0u;
  p.inv_keep = 256.0f / (256.0f - (float)p.drop_thresh);
  memset(&p.rng, 0, sizeof(p.rng));
  if (rng != nullptr) p.rng = *rng;
  p.rng_out = rng_out;
  cudaError_t e = (D == 64) ? launch_fwd<64>(tq, tk, tv, p, s) : launch_fwd<128>(tq, tk, tv, p, s);
  return (int)e;
}
// =================================================================================================
// Backward.  One CTA per (batch, head, 64-key block); one consumer warpgroup loops over the 64-query blocks that
// attend to it (warp 4 = TMA producer, Q / dO double buffered):
//   Sᵀ = K·Q_iᵀ , dPᵀ = V·dO_iᵀ                  (wgmma, registers)
//   Pᵀ = exp(Sᵀ·scale − lse) , dSᵀ = Pᵀ ∘ (dPᵀ − δ) · scale
//   dV += Pᵀ·dO_i , dK += dSᵀ·Q_i                 (A operands straight from the registers, accumulators stay in
//                                                  registers for the whole CTA)
//   dQ_i += dS·K                                  (dSᵀ through shared memory, read as a transposed A operand; fp32
//                                                  red.add into dq_accum, key block after key block in decreasing
//                                                  order: a per-query-block counter orders the CTAs, so the sums are
//                                                  deterministic.  CTA kb at step `it` needs what kb + 1 added at step
//                                                  it - 1, so the CTAs do not stall each other, and the highest key
//                                                  blocks are launched first so that a waiter's predecessor is resident)
// Forward progress of that wait relies on the hardware dispatching the CTAs of a grid in increasing linear block index
// (the waited-for CTA always has the lower index), the same assumption as FlashAttention-3's deterministic backward.
// Should it ever fail, the bounded spin wait traps after its timeout instead of hanging.
// δ = rowsum(dO ∘ O) is produced by attn_delta_kernel, dq_accum is converted to bf16 afterwards.
// =================================================================================================
namespace lb {

template <int D>
struct AttnBwdCfg {
  static constexpr int CHUNKS = D / 64;
  static constexpr int TILE_BYTES = 64 * D * 2;   // 64 rows of K / V / Q / dO
  static constexpr int DS_BYTES = 64 * 64 * 2;
  static constexpr int SMEM_BYTES = 2 * TILE_BYTES /*K,V*/ + 4 * TILE_BYTES /*Q,dO x2*/ + DS_BYTES + 1024 + 256;
};

struct AttnBwdParams {
  const float* lse;     // [B, A, S]
  const float* delta;   // [B, A, S]
  float* dq_accum;      // [B, A, S, D] fp32
  __nv_bfloat16* dk;    // strided [B, A, S, D] views
  __nv_bfloat16* dv;
  long g_strides[3];    // batch, head, seq strides (elements) of dk / dv
  int B, A, S;
  int causal;
  float scale, scale_log2;
  const int* kv_lens;   // optional [B]
  // same additive bias / dropout description as the forward; `rng_state` = the (seed, offset) pair the forward used
  const __nv_bfloat16* bias;
  long bias_strides[3];
  const float* alibi_slopes;
  float* dbias;         // optional fp32, same strides as `bias`: += P ∘ (dP − δ) (gradient of a learned bias)
  uint32_t drop_thresh;
  float inv_keep;
  const long long* rng_state;
  unsigned* dq_order;   // [B * A * query blocks]: key blocks whose dQ contribution has landed (zeroed by the caller)
};

template <int D, int BIAS, bool DROP>
__global__ void __launch_bounds__(ATT_BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do, AttnBwdParams p) {
  using Cfg = AttnBwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + Cfg::TILE_BYTES;
  uint8_t* sQ = sV + Cfg::TILE_BYTES;      // 2 stages
  uint8_t* sDO = sQ + 2 * Cfg::TILE_BYTES;  // 2 stages
  uint8_t* sDS = sDO + 2 * Cfg::TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sDS + Cfg::DS_BYTES);
  uint64_t* kv_full = bars;
  uint64_t* qdo_full = bars + 1;    // 2
  uint64_t* qdo_empty = bars + 3;   // 2

  const int warp_idx = threadIdx.x / 32;
  const int kv_blk = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);
  const int head = blockIdx.y, batch = blockIdx.z;
  const int k0 = kv_blk * ATT_BWD_BN;
  const int kv_len = p.kv_lens != nullptr ? max(1, min(p.S, p.kv_lens[batch])) : p.S;
  const int nq = (p.S + ATT_BWD_BM - 1) / ATT_BWD_BM;
  const int i_begin = p.causal ? (k0 / ATT_BWD_BM) : 0;
  const int iters = nq - i_begin;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    tma_prefetch_desc(&tmap_do);
    mbar_init(kv_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&qdo_full[i], 1);
      mbar_init(&qdo_empty[i], 128);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp_idx == 4) {
    if (elect_one()) {
      mbar_arrive_expect_tx(kv_full, 2 * Cfg::TILE_BYTES);
#pragma unroll
      for (int c = 0; c < Cfg::CHUNKS; ++c) {
        tma_load_4d(sK + c * (64 * 128), &tmap_k, kv_full, c * 64, k0, head, batch);
        tma_load_4d(sV + c * (64 * 128), &tmap_v, kv_full, c * 64, k0, head, batch);
      }
      for (int it = 0; it < iters; ++it) {
        const int st = it & 1;
        const int q0 = (i_begin + it) * ATT_BWD_BM;
        mbar_wait(&qdo_empty[st], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&qdo_full[st], 2 * Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c) {
          tma_load_4d(sQ + st * Cfg::TILE_BYTES + c * (64 * 128), &tmap_q, &qdo_full[st], c * 64, q0, head, batch);
          tma_load_4d(sDO + st * Cfg::TILE_BYTES + c * (64 * 128), &tmap_do, &qdo_full[st], c * 64, q0, head, batch);
        }
      }
    }
    return;
  }

  const int t = threadIdx.x;                              // 0..127
  const int r_loc = 16 * (t / 32) + (t % 32) / 4;         // fragment rows r_loc, r_loc + 8
  const int cq = 2 * (t % 4);
  const size_t bh = static_cast<size_t>(batch) * p.A + head;
  constexpr float LOG2E = 1.4426950408889634f;
  unsigned long long rng_seed = 0, rng_offset = 0;
  if constexpr (DROP) {
    rng_seed = static_cast<unsigned long long>(p.rng_state[0]);
    rng_offset = static_cast<unsigned long long>(p.rng_state[1]);
  }
  float slope2 = 0.f;
  if constexpr (BIAS == BIAS_ALIBI) slope2 = p.alibi_slopes[head] * LOG2E;
  const long bias_bh = batch * p.bias_strides[0] + head * p.bias_strides[1];
  const float inv_scale = 1.0f / p.scale;
  const uint32_t k_addr = smem_u32(sK), v_addr = smem_u32(sV), ds_addr = smem_u32(sDS);

  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) {
    dv[i] = 0.f;
    dk[i] = 0.f;
  }
  mbar_wait(kv_full, 0);

  for (int it = 0; it < iters; ++it) {
    const int st = it & 1;
    const int q0 = (i_begin + it) * ATT_BWD_BM;
    const uint32_t q_addr = smem_u32(sQ + st * Cfg::TILE_BYTES), do_addr = smem_u32(sDO + st * Cfg::TILE_BYTES);
    mbar_wait(&qdo_full[st], (it >> 1) & 1);
    // ---- Sᵀ = K·Q_iᵀ, dPᵀ = V·dO_iᵀ (64 keys x 64 queries each)
    float sT[32], dpT[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t off = (kk / 4) * (64 * 128) + (kk % 4) * 32;
      wgmma_bf16_ss<64, 0, 0>(sT, make_smem_desc_sw128(k_addr + off, 0, 1024), make_smem_desc_sw128(q_addr + off, 0, 1024),
                              kk > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t off = (kk / 4) * (64 * 128) + (kk % 4) * 32;
      wgmma_bf16_ss<64, 0, 0>(dpT, make_smem_desc_sw128(v_addr + off, 0, 1024), make_smem_desc_sw128(do_addr + off, 0, 1024),
                              kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sT);
    wgmma_fence_regs(dpT);

    // ---- Pᵀ (as it multiplied V in the forward, i.e. dropped and rescaled) into sT, dSᵀ into dpT
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int q_idx = q0 + 8 * jj + cq + c;
        const bool q_ok = q_idx < p.S;
        const float lse2 = q_ok ? p.lse[bh * p.S + q_idx] * LOG2E : 0.f;
        const float delta_s = q_ok ? p.delta[bh * p.S + q_idx] * p.scale : 0.f;
        const int key_lim = !q_ok ? 0 : (p.causal ? min(kv_len, q_idx + 1) : kv_len);
        uint4 rnd;
        if constexpr (DROP)   // both rows of this thread lie in the same 16-key group
          rnd = attn_dropout_bytes(static_cast<uint32_t>(q_idx), static_cast<uint32_t>((k0 + 16 * (t / 32)) >> 4),
                                   static_cast<uint32_t>(bh), rng_seed, rng_offset);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int kidx = k0 + r_loc + 8 * h;
          const int i = 4 * jj + 2 * h + c;
          float x = sT[i] * p.scale_log2;
          long boff = 0;
          if constexpr (BIAS == BIAS_DENSE) {
            boff = bias_bh + static_cast<long>(min(q_idx, p.S - 1)) * p.bias_strides[2] + min(kidx, p.S - 1);
            x = fmaf(__bfloat162float(p.bias[boff]), LOG2E, x);
          } else if constexpr (BIAS == BIAS_ALIBI) {
            x = fmaf(slope2, static_cast<float>(kidx - q_idx), x);
          }
          const float pv = kidx < key_lim ? fast_exp2(x - lse2) : 0.f;
          float g = dpT[i], pd = pv;   // dP w.r.t. the dropped, rescaled P; what multiplied V in the forward
          if constexpr (DROP) {
            const bool keep = rnd_byte(rnd, (r_loc + 8 * h) & 15) >= p.drop_thresh;
            g = keep ? g * p.inv_keep : 0.f;
            pd = keep ? pv * p.inv_keep : 0.f;
          }
          const float ds = pv * fmaf(g, p.scale, -delta_s);
          if constexpr (BIAS == BIAS_DENSE) {
            // d bias = P ∘ (dP − δ): fp32 reductions (broadcast dims sum over CTAs)
            if (p.dbias != nullptr && q_ok && kidx < p.S) atomicAdd(p.dbias + boff, ds * inv_scale);
          }
          sT[i] = pd;
          dpT[i] = ds;
        }
      }
    }
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      acc_to_a_frag(&sT[8 * g], pa[g]);
      acc_to_a_frag(&dpT[8 * g], da[g]);
    }
    // dSᵀ -> shared memory (64 key rows x 128 B, 128-byte swizzle) for the dQ product
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r_loc + 8 * h;
        *reinterpret_cast<uint32_t*>(sDS + row * 128 + ((jj ^ (row & 7)) << 4) + cq * 2) =
            pack_bf16(dpT[4 * jj + 2 * h], dpT[4 * jj + 2 * h + 1]);
      }
    }
    fence_proxy_async();
    warpgroup_sync(0);
    // ---- dV += Pᵀ·dO_i, dK += dSᵀ·Q_i (B operands: the [query, D] tiles read MN-major)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma_bf16_rs<D, 1>(dv, pa[kk], make_smem_desc_sw128(do_addr + kk * (16 * 128), 64 * 128, 1024), 1u);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma_bf16_rs<D, 1>(dk, da[kk], make_smem_desc_sw128(q_addr + kk * (16 * 128), 64 * 128, 1024), 1u);
    wgmma_commit();
    // ---- dQ_i is accumulated by the key blocks in decreasing order: wait until the key blocks above this one that
    // contribute to query block i (all of them, or those up to i under the causal mask) have added theirs
    const int q_blk = i_begin + it;
    unsigned* order = p.dq_order + bh * nq + q_blk;
    const int last_kb = p.causal ? q_blk : static_cast<int>(gridDim.x) - 1;
    if (t == 0) spin_wait_ge_sys(order, static_cast<uint32_t>(last_kb - kv_blk), 0, /*what=*/5, kv_blk);
    warpgroup_sync(0);
    // ---- dQ_i = dS·K, 64 columns at a time: A = dSᵀ read transposed, B = the K tile read MN-major
#pragma unroll
    for (int n = 0; n < D / 64; ++n) {
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_bf16_ss<64, 1, 1>(dq, make_smem_desc_sw128(ds_addr + kk * (16 * 128), 64 * 128, 1024),
                                make_smem_desc_sw128(k_addr + n * (64 * 128) + kk * (16 * 128), 64 * 128, 1024),
                                kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int q_idx = q0 + r_loc + 8 * h;
        if (q_idx < p.S) {
          float* dq_row = p.dq_accum + (bh * p.S + q_idx) * D + n * 64;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};\n" ::"l"(dq_row + 8 * jj + cq), "f"(dq[4 * jj + 2 * h]),
                         "f"(dq[4 * jj + 2 * h + 1])
                         : "memory");
        }
      }
    }
    __threadfence();
    warpgroup_sync(0);
    if (t == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(order) : "memory");
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    mbar_arrive(&qdo_empty[st]);
  }

  // ---- dV / dK: fragment rows = key rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k_idx = k0 + r_loc + 8 * h;
    if (k_idx >= p.S) continue;
    const long off = batch * p.g_strides[0] + head * p.g_strides[1] + static_cast<long>(k_idx) * p.g_strides[2];
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj) {
      *reinterpret_cast<uint32_t*>(p.dv + off + 8 * jj + cq) = pack_bf16(dv[4 * jj + 2 * h], dv[4 * jj + 2 * h + 1]);
      *reinterpret_cast<uint32_t*>(p.dk + off + 8 * jj + cq) = pack_bf16(dk[4 * jj + 2 * h], dk[4 * jj + 2 * h + 1]);
    }
  }
}

// delta[b, a, s] = sum_d dO[b, a, s, d] * O[b, a, s, d]
// D / 8 lanes per row, 16-byte loads; rows are visited in (b, s, a) order = memory order of the [b, s, a, d] tensors, so
// a warp reads 32 x 16 contiguous bytes per tensor, and every thread keeps 4 rows (8 loads) in flight.
template <int D>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ o, float* __restrict__ delta,
                  int B, int A, int S, long sb, long sa, long ss, float4* __restrict__ zero_fill, long zero_n4) {
  constexpr int LPR = D / 8;  // lanes per row
  const long total = static_cast<long>(B) * A * S;
  const long gid = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  // the fp32 dQ accumulator of the main kernel is cleared here (one launch and one pass less than a memset in front)
  for (long z = gid; z < zero_n4; z += static_cast<long>(gridDim.x) * blockDim.x) zero_fill[z] = make_float4(0.f, 0.f, 0.f, 0.f);
  const long gstride = static_cast<long>(gridDim.x) * blockDim.x / LPR;
  const int sub = static_cast<int>(gid % LPR);
  const long warp_r0 = (gid - (threadIdx.x % 32)) / LPR;  // loop bound is warp-uniform (the shuffles below need all lanes)
  for (long base = 0; warp_r0 + base < total; base += 4 * gstride) {
    const long r0 = gid / LPR + base;
    uint4 x[4], y[4];
    long drow[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long r = r0 + u * gstride;
      const bool ok = r < total;
      const long rr = ok ? r : 0;
      const int a = static_cast<int>(rr % A), sq = static_cast<int>((rr / A) % S);
      const long b = rr / (static_cast<long>(A) * S);
      const long off = b * sb + a * sa + sq * ss + sub * 8;
      drow[u] = ok ? (b * A + a) * static_cast<long>(S) + sq : -1;
      x[u] = ok ? *reinterpret_cast<const uint4*>(dout + off) : make_uint4(0, 0, 0, 0);
      y[u] = ok ? *reinterpret_cast<const uint4*>(o + off) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float2 a0 = unpack_bf16(x[u].x), a1 = unpack_bf16(x[u].y), a2 = unpack_bf16(x[u].z), a3 = unpack_bf16(x[u].w);
      const float2 b0 = unpack_bf16(y[u].x), b1 = unpack_bf16(y[u].y), b2 = unpack_bf16(y[u].z), b3 = unpack_bf16(y[u].w);
      float acc = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y + a3.x * b3.x + a3.y * b3.y;
#pragma unroll
      for (int m = LPR / 2; m >= 1; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
      if (sub == 0 && drow[u] >= 0) delta[drow[u]] = acc;
    }
  }
}

// dq (strided bf16) = dq_accum (fp32 [B, A, S, D]); 8 elements per thread (two 16-byte loads, one 16-byte store)
__global__ void __launch_bounds__(256)
attn_dq_convert_kernel(const float* __restrict__ acc, __nv_bfloat16* __restrict__ dq, int B, int A, int S, int D, long sb,
                       long sa, long ss) {
  const long nvec = static_cast<long>(B) * A * S * D / 8;
  const long stride = static_cast<long>(gridDim.x) * blockDim.x;
  for (long i0 = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i0 < nvec; i0 += 2 * stride) {
    float4 lo[2], hi[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long i = i0 + u * stride;
      if (i < nvec) {
        lo[u] = reinterpret_cast<const float4*>(acc)[2 * i];
        hi[u] = reinterpret_cast<const float4*>(acc)[2 * i + 1];
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long i = i0 + u * stride;
      if (i < nvec) {
        const long e = i * 8;
        const int d = static_cast<int>(e % D);
        const long row = e / D;
        const int sq = static_cast<int>(row % S), a = static_cast<int>((row / S) % A);
        const long b = row / (static_cast<long>(S) * A);
        *reinterpret_cast<uint4*>(dq + b * sb + a * sa + sq * ss + d) =
            make_uint4(pack_bf16(lo[u].x, lo[u].y), pack_bf16(lo[u].z, lo[u].w), pack_bf16(hi[u].x, hi[u].y), pack_bf16(hi[u].z, hi[u].w));
      }
    }
  }
}

}  // namespace lb

namespace {
int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

template <int D, int BIAS, bool DROP>
cudaError_t launch_bwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                         const lb::AttnBwdParams& p, cudaStream_t s) {
  using Cfg = lb::AttnBwdCfg<D>;
  auto kern = lb::attn_bwd_kernel<D, BIAS, DROP>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid((p.S + lb::ATT_BWD_BN - 1) / lb::ATT_BWD_BN, p.A, p.B);
  kern<<<grid, lb::ATT_BWD_THREADS, Cfg::SMEM_BYTES, s>>>(tq, tk, tv, tdo, p);
  return cudaGetLastError();
}
template <int D>
cudaError_t launch_bwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                       const lb::AttnBwdParams& p, cudaStream_t s) {
  const int bias = p.bias != nullptr ? lb::BIAS_DENSE : (p.alibi_slopes != nullptr ? lb::BIAS_ALIBI : lb::BIAS_NONE);
  const bool drop = p.drop_thresh > 0;
  if (bias == lb::BIAS_NONE) return drop ? launch_bwd_t<D, lb::BIAS_NONE, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_NONE, false>(tq, tk, tv, tdo, p, s);
  if (bias == lb::BIAS_DENSE) return drop ? launch_bwd_t<D, lb::BIAS_DENSE, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_DENSE, false>(tq, tk, tv, tdo, p, s);
  return drop ? launch_bwd_t<D, lb::BIAS_ALIBI, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_ALIBI, false>(tq, tk, tv, tdo, p, s);
}
}  // namespace
extern "C" int lb_attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* o,
                           const float* lse, void* dq, void* dk, void* dv, float* delta, float* dq_accum, int B, int A,
                           int S, int D, const long* q_strides, const long* k_strides, const long* v_strides,
                           const long* do_strides, int causal, float scale, const int* kv_lens, const void* bias,
                           const long* bias_strides, const float* alibi_slopes, float* dbias, float p_drop,
                           const long long* rng_state, unsigned* dq_order, cudaStream_t s) {
  if (D != 64 && D != 128) return -1;
  for (int i = 0; i < 3; ++i)
    if ((q_strides[i] % 8) || (k_strides[i] % 8) || (v_strides[i] % 8) || (do_strides[i] % 8)) return -3;
  CUtensorMap tq, tk, tv, tdo;
  if (!make_qkv_tmap(&tq, q, B, A, S, D, q_strides, 64)) return -2;
  if (!make_qkv_tmap(&tk, k, B, A, S, D, k_strides, 64)) return -2;
  if (!make_qkv_tmap(&tv, v, B, A, S, D, v_strides, 64)) return -2;
  if (!make_qkv_tmap(&tdo, dout, B, A, S, D, do_strides, 64)) return -2;
  const long rows = (long)B * A * S;
  {
    // 4 rows per thread-group and iteration; cap the grid at a few waves
    const long groups = (rows + 3) / 4;
    const long lpr = D / 8;
    long blocks = (groups * lpr + 255) / 256;
    if (blocks > sm_count() * 16L) blocks = sm_count() * 16L;
    if (D == 64)
      lb::attn_delta_kernel<64><<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)o, delta, B,
                                                                   A, S, do_strides[0], do_strides[1], do_strides[2],
                                                                   reinterpret_cast<float4*>(dq_accum), rows * D / 4);
    else
      lb::attn_delta_kernel<128><<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)o, delta, B,
                                                                    A, S, do_strides[0], do_strides[1], do_strides[2],
                                                                    reinterpret_cast<float4*>(dq_accum), rows * D / 4);
  }
  lb::AttnBwdParams p;
  p.lse = lse;
  p.delta = delta;
  p.dq_accum = dq_accum;
  p.dk = (__nv_bfloat16*)dk;
  p.dv = (__nv_bfloat16*)dv;
  // dq / dk / dv are views of one packed [B, S, A, 3, D] tensor: same strides as the packed q view
  p.g_strides[0] = (long)S * A * 3 * D;
  p.g_strides[1] = 3L * D;
  p.g_strides[2] = (long)A * 3 * D;
  p.B = B;
  p.A = A;
  p.S = S;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.kv_lens = kv_lens;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  for (int i = 0; i < 3; ++i) p.bias_strides[i] = (bias != nullptr && bias_strides != nullptr) ? bias_strides[i] : 0;
  p.alibi_slopes = bias != nullptr ? nullptr : alibi_slopes;
  p.dbias = bias != nullptr ? dbias : nullptr;
  uint32_t thr = (uint32_t)(p_drop * 256.0f + 0.5f);
  if (thr > 255u) thr = 255u;
  p.drop_thresh = (p_drop > 0.f && rng_state != nullptr) ? (thr == 0 ? 1u : thr) : 0u;
  p.inv_keep = 256.0f / (256.0f - (float)p.drop_thresh);
  p.rng_state = rng_state;
  p.dq_order = dq_order;
  cudaError_t e = (D == 64) ? launch_bwd<64>(tq, tk, tv, tdo, p, s) : launch_bwd<128>(tq, tk, tv, tdo, p, s);
  if (e != cudaSuccess) return (int)e;
  const long nvec = rows * D / 8;
  int blocks = (int)((nvec + 511) / 512);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  lb::attn_dq_convert_kernel<<<blocks, 256, 0, s>>>(dq_accum, (__nv_bfloat16*)dq, B, A, S, D, p.g_strides[0],
                                                    p.g_strides[1], p.g_strides[2]);
  return (int)cudaGetLastError();
}
