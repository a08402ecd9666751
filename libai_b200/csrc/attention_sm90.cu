// Flash attention for sm_90a on wgmma / TMA / mbarrier (bf16, causal or full, head dim d a multiple of 8 in [8, 128]).
//
// Head dim: d runs on a tile of D = 64 (d <= 64) or D = 128 (64 < d <= 128) columns.  The Q/K/V/dO tensor maps have
// d columns, so TMA fills columns d .. D of every 64-column box with zeros (the transaction byte counts stay at the full
// box): the padded columns add nothing to S = Q·Kᵀ or dPᵀ = V·dOᵀ and stay zero in the O, dK, dV and dQ accumulators.
// Every store stops at column d: in the packed projections the columns past a q slot's d are the k slot of the head.
//
// Replaces the score GEMM + fused_scale_(tril_)softmax(_mask)_dropout + context GEMM sequence of the
// reference (libai/layers/attention.py:211-253): no [b, a, s, s] tensor and no materialised mask.
// Q/K/V are read straight out of the packed QKV projection through strided TMA tensor maps, O is written in
// [B, S, A, D] so the output projection consumes it as-is.
//
// Grouped-query attention: A query heads share G = A / r key/value heads, query head h reading K/V head h / r.  Q is
// described by (batch, group, in-group, seq) strides and read through a 5-D map ({D, S, r, G, B}), so both a plain
// [B, A, S, D] q and the q slots of the grouped packed projection [B, S, G, r + 2, D] (per group q_0 .. q_{r-1}, k, v;
// r = 1 is the per-head [q|k|v] layout) are read without a copy.  K/V use 4-D maps over the G heads.  Everything else
// (O, lse, bias, ALiBi slope, dropout stream, kv_lens) stays per query head.
//
// Rectangular problems: Sq queries against Sk keys.  Key j is visible to query i of sample b iff
// kv_start[b] <= j < kv_lens[b] (defaults 0 and Sk; kv_lens is clamped to >= 1 as it always was) and, when causal,
// j <= i + (Sk - Sq) (bottom-right alignment, as in decode attention).  A query without a visible key gets O = 0,
// lse = 0 and dQ = 0, and adds nothing to dK / dV.
//
// Packed sequences (DOC instances, causal self-attention only): doc_start [B, S] gives the first key of each query's
// document, so query i of sample b sees key j iff doc_start[b, i] <= j <= i (doc_start clamped to [0, i]: every query
// sees itself).  Nothing assumes doc_start to be non-decreasing along a row: which key tiles a forward CTA loads and
// which (key block, query block) visits the backward skips come from the minimum over the rows of the query block.
//
// Forward, one CTA per (batch, query head, 128-query block), 384 threads:
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
constexpr int ATT_BWD_BN = 64;   // keys per consumer warpgroup (backward)
constexpr int ATT_BWD_BM = 64;   // queries per step (backward)

struct AttnFwdParams {
  __nv_bfloat16* o;   // [B, Sq, A, d]
  float* lse;         // [B, A, Sq]
  int B, A, Sq, Sk;
  int d;              // head dim (d <= D, a multiple of 8)
  int r;              // query heads per K/V head
  int causal;
  float scale_log2;   // scale * log2(e)
  float scale;
  const int* kv_lens; // optional [B]: end of the visible keys per sample (right-padded batches)
  const int* kv_start;   // optional [B]: start of the visible keys per sample (left-padded batches)
  const int* doc_start;  // [B, Sq] in the DOC instances: first key of each query's document
  // additive score bias (v2 kernel): dense bf16 [.., Sq, Sk] with (batch, head, query) strides in elements (0 = broadcast;
  // T5 relative-position bias, Swin/BERT style masks) or ALiBi slopes per head (bias = slope * (key - query - (Sk - Sq)))
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
// column c (a compile-time constant in the unrolled store loops) of a D-wide tile lies inside head dim d; the 128-wide
// tile runs d > 64 only, so its first 64 columns need no run-time test
template <int D>
LB_DEVICE bool col_in_head(int c, int d) {
  return (D == 128 && c < 64) || c < d;
}
// first visible key of query row i (< S) of a packed sample: its doc_start, clamped to [0, i]
LB_DEVICE int doc_begin(const int* doc_start, int S, int batch, int i) {
  return min(max(doc_start[static_cast<size_t>(batch) * S + i], 0), i);
}

template <int D>
struct AttnFwdCfg {
  static constexpr int CHUNKS = D / 64;                    // 64-element (128B) chunks of a row
  static constexpr int TILE_BYTES = ATT_BN * D * 2;        // one Q / K / V tile
  static constexpr int SMEM_BYTES = 5 * TILE_BYTES + 1024 + 256;   // Q + 2 x (K, V)
};

// the forward of one CTA; tmap_* and p are the kernel's __grid_constant__ parameters (inlined: no call in the kernel)
template <int D, int BIAS, bool DROP, bool DOC>
LB_DEVICE void attn_fwd_cta(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k, const CUtensorMap& tmap_v,
                            const AttnFwdParams& p) {
  static_assert(!DOC || (BIAS == BIAS_NONE && !DROP), "packed sequences run without bias and dropout");
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
  int* doc_min = reinterpret_cast<int*>(bars + 9);   // 4 (DOC): per-warp minima of the block's document starts

  const int warp_idx = threadIdx.x / 32;
  // heavy (late) query blocks first: better tail behaviour under the causal mask
  const int q_blk = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / p.r;
  const int q0 = q_blk * ATT_BM;
  const int kv_len = p.kv_lens != nullptr ? max(1, min(p.Sk, p.kv_lens[batch])) : p.Sk;
  const int kv_beg = p.kv_start != nullptr ? min(max(p.kv_start[batch], 0), p.Sk) : 0;
  const int off = p.Sk - p.Sq;   // causal offset: query i sees keys j <= i + off
  // key tiles j0 .. j0 + nkv - 1 hold every key some row of this block can see; the others are not loaded
  const int key_end = p.causal ? min(kv_len, min(q0 + ATT_BM, p.Sq) + off) : kv_len;
  if constexpr (DOC) {   // warpgroup 0 reads one row each (rows past Sq repeat the last row)
    if (warp_idx < 4) {
      const int m = __reduce_min_sync(0xffffffffu, doc_begin(p.doc_start, p.Sq, batch, min(q0 + static_cast<int>(threadIdx.x), p.Sq - 1)));
      if (threadIdx.x % 32 == 0) doc_min[warp_idx] = m;
    }
  }

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
  // the first tile holds the earliest key any row of the block sees
  const int j0 = (DOC ? min(min(doc_min[0], doc_min[1]), min(doc_min[2], doc_min[3])) : kv_beg) / ATT_BN;
  const int nkv = max(0, (key_end + ATT_BN - 1) / ATT_BN - j0);

  if (warp_idx < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp_idx == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, Cfg::TILE_BYTES);
#pragma unroll
      for (int c = 0; c < Cfg::CHUNKS; ++c)
        tma_load_5d(sQ + c * (ATT_BM * 128), &tmap_q, q_full, c * 64, q0, head - kv_head * p.r, kv_head, batch);
      for (int it = 0; it < nkv; ++it) {
        const int j = j0 + it, b = it & 1;
        const uint32_t par = ((it >> 1) & 1) ^ 1;
        mbar_wait(&k_empty[b], par);
        mbar_arrive_expect_tx(&k_full[b], Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c)
          tma_load_4d(sK + b * Cfg::TILE_BYTES + c * (ATT_BN * 128), &tmap_k, &k_full[b], c * 64, j * ATT_BN, kv_head, batch);
        mbar_wait(&v_empty[b], par);
        mbar_arrive_expect_tx(&v_full[b], Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c)
          tma_load_4d(sV + b * Cfg::TILE_BYTES + c * (ATT_BN * 128), &tmap_v, &v_full[b], c * 64, j * ATT_BN, kv_head, batch);
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
  const int wg = warp_idx / 4 - 1;
  const int t = threadIdx.x % 128;
  const int r_loc = 64 * wg + 16 * (t / 32) + (t % 32) / 4;   // this thread's rows: r_loc and r_loc + 8
  const int cq = 2 * (t % 4);                                  // its columns inside every 8-column group: cq, cq + 1
  // keys row_beg + [0, vis_len) are visible to row h: one unsigned comparison of key - row_beg per element tests both
  // ends (row_beg = kv_beg, or the row's document start in the DOC instances)
  int q_idx[2], vis_len[2], row_beg[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    q_idx[h] = q0 + r_loc + 8 * h;
    row_beg[h] = DOC ? doc_begin(p.doc_start, p.Sq, batch, min(q_idx[h], p.Sq - 1)) : kv_beg;
    vis_len[h] = max(0, (p.causal ? min(kv_len, q_idx[h] + off + 1) : kv_len) - row_beg[h]);
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
                    static_cast<long>(min(q_idx[h], p.Sq - 1)) * p.bias_strides[2];
  }
  if constexpr (BIAS == BIAS_ALIBI) slope2 = p.alibi_slopes[head] * LOG2E;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
  mbar_wait(q_full, 0);

  for (int it = 0; it < nkv; ++it) {
    const int j = j0 + it, b = it & 1;
    const uint32_t par = (it >> 1) & 1;
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
    const int kbase = j * ATT_BN, krel = kbase - kv_beg;
    // (per thread in the DOC instances: a tile may start before one of its rows' documents only)
    const bool need_mask = kbase < (DOC ? max(row_beg[0], row_beg[1]) : kv_beg) || kbase + ATT_BN > kv_len ||
                           (p.causal && kbase + ATT_BN - 1 > q0 + off);
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
            // a pair load never reads past the row's last key (Sk may be odd)
            const float2 f = kb + 1 < p.Sk ? unpack_bf16(*reinterpret_cast<const uint32_t*>(bias_row[h] + kb))
                             : make_float2(kb < p.Sk ? __bfloat162float(bias_row[h][kb]) : 0.f, 0.f);
            x = fmaf(c ? f.y : f.x, LOG2E, x);
          } else if constexpr (BIAS == BIAS_ALIBI) {
            x = fmaf(slope2, static_cast<float>(kidx - q_idx[h] - off), x);
            // (ALiBi keeps the test inline: the separate pass below costs the head-dim-128 dropout variant a spill)
            if (need_mask && static_cast<unsigned>(krel + 8 * jj + cq + c) >= static_cast<unsigned>(vis_len[h])) x = -INFINITY;
          }
          s[4 * jj + 2 * h + c] = x;
        }
      }
    }
    if (BIAS != BIAS_ALIBI && need_mask) {   // uniform per tile: tiles inside every row's window skip the element test
#pragma unroll
      for (int jj = 0; jj < ATT_BN / 8; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int c = 0; c < 2; ++c)
            if (static_cast<unsigned>((DOC ? kbase - row_beg[h] : krel) + 8 * jj + cq + c) >= static_cast<unsigned>(vis_len[h]))
              s[4 * jj + 2 * h + c] = -INFINITY;
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

  // ---- epilogue: O / l  →  [B, Sq, A, d]; lse in natural log (0 for a row without a visible key)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? (DROP ? p.inv_keep : 1.0f) / l : 0.f;
    if (q_idx[h] < p.Sq) {
      __nv_bfloat16* orow = p.o + ((static_cast<size_t>(batch) * p.Sq + q_idx[h]) * p.A + head) * p.d;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        if (col_in_head<D>(8 * jj, p.d))
          *reinterpret_cast<uint32_t*>(orow + 8 * jj + cq) = pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      if (t % 4 == 0)
        p.lse[(static_cast<size_t>(batch) * p.A + head) * p.Sq + q_idx[h]] =
            (m_run[h] == -INFINITY) ? 0.f : (m_run[h] + log2f(l)) * 0.6931471805599453f;
    }
  }
}

template <int D, int BIAS, bool DROP>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnFwdParams p) {
  attn_fwd_cta<D, BIAS, DROP, false>(tmap_q, tmap_k, tmap_v, p);
}
// packed sequences (doc_start): causal self-attention without bias or dropout
template <int D>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_doc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnFwdParams p) {
  attn_fwd_cta<D, BIAS_NONE, false, true>(tmap_q, tmap_k, tmap_v, p);
}

}  // namespace lb

namespace {
// the tile width a head dim runs on: 64 or 128, 0 for an unsupported head dim
int head_dim_tile(int d) {
  if (d % 8 || d < 8 || d > 128) return 0;
  return d <= 64 ? 64 : 128;
}
// dims innermost first: {d, S, A, B}; st = {batch, head, seq} strides in elements; boxes of 64 columns x `rows` rows
// (columns past d are zero-filled)
bool make_qkv_tmap(CUtensorMap* m, const void* ptr, int B, int A, int S, int D, const long* st, int rows) {
  uint64_t dims[4] = {(uint64_t)D, (uint64_t)S, (uint64_t)A, (uint64_t)B};
  uint64_t strides[4] = {2, (uint64_t)st[2] * 2, (uint64_t)st[1] * 2, (uint64_t)st[0] * 2};
  uint32_t box[4] = {64, (uint32_t)rows, 1, 1};
  return lb_host::make_tmap_bf16(m, ptr, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
// query-head tensors of grouped-query attention, dims innermost first {d, S, r, G, B}; st = {batch, group, in-group,
// seq} strides in elements
bool make_q_tmap(CUtensorMap* m, const void* ptr, int B, int G, int r, int S, int D, const long* st, int rows) {
  uint64_t dims[5] = {(uint64_t)D, (uint64_t)S, (uint64_t)r, (uint64_t)G, (uint64_t)B};
  uint64_t strides[5] = {2, (uint64_t)st[3] * 2, (uint64_t)st[2] * 2, (uint64_t)st[1] * 2, (uint64_t)st[0] * 2};
  uint32_t box[5] = {64, (uint32_t)rows, 1, 1, 1};
  return lb_host::make_tmap_bf16(m, ptr, 5, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int D, int BIAS, bool DROP, bool DOC = false>
cudaError_t launch_fwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const lb::AttnFwdParams& p,
                         cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = DOC ? lb::attn_fwd_doc_kernel<D> : lb::attn_fwd_kernel<D, BIAS, DROP>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid((p.Sq + lb::ATT_BM - 1) / lb::ATT_BM, p.A, p.B);
  kern<<<grid, lb::ATT_FWD_THREADS, Cfg::SMEM_BYTES, s>>>(tq, tk, tv, p);
  return cudaGetLastError();
}

template <int D>
cudaError_t launch_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const lb::AttnFwdParams& p,
                       cudaStream_t s) {
  if (p.doc_start != nullptr) return launch_fwd_t<D, lb::BIAS_NONE, false, true>(tq, tk, tv, p, s);
  const int bias = p.bias != nullptr ? lb::BIAS_DENSE : (p.alibi_slopes != nullptr ? lb::BIAS_ALIBI : lb::BIAS_NONE);
  const bool drop = p.drop_thresh > 0;
  if (bias == lb::BIAS_NONE) return drop ? launch_fwd_t<D, lb::BIAS_NONE, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_NONE, false>(tq, tk, tv, p, s);
  if (bias == lb::BIAS_DENSE) return drop ? launch_fwd_t<D, lb::BIAS_DENSE, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_DENSE, false>(tq, tk, tv, p, s);
  return drop ? launch_fwd_t<D, lb::BIAS_ALIBI, true>(tq, tk, tv, p, s) : launch_fwd_t<D, lb::BIAS_ALIBI, false>(tq, tk, tv, p, s);
}
}  // namespace
// A query heads in G groups (A % G == 0); Sq queries, Sk keys; head dim D a multiple of 8 in [8, 128]; q_strides =
// {batch, group, in-group, seq}, k/v_strides = {batch, head, seq} over the G K/V heads (elements).  kv_lens / kv_start
// (optional, int32 [B], device): per-sample key window.
// p_drop in [0, 1): attention dropout probability (quantised to 1/256 like the byte-threshold test of the kernel);
// bias (optional, bf16): dense additive score bias with (batch, head, query-row) strides in elements, key stride 1;
// alibi_slopes (optional, fp32 [A]); doc_start (optional, int32 [B, Sq], device): packed sequences, causal Sq == Sk
// only, without kv_lens, kv_start, bias or dropout.
extern "C" int lb_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int A, int G, int Sq,
                           int Sk, int D, const long* q_strides, const long* k_strides, const long* v_strides, int causal,
                           float scale, const int* kv_lens, const int* kv_start, const int* doc_start, const void* bias,
                           const long* bias_strides, const float* alibi_slopes, float p_drop, const lb::RngArgs* rng,
                           long long* rng_out, cudaStream_t s) {
  const int tile = head_dim_tile(D);
  if (tile == 0) return -1;
  if (Sq <= 0 || Sk <= 0) return -5;
  if (G <= 0 || A % G) return -4;
  if (doc_start != nullptr && (!causal || Sq != Sk || kv_lens != nullptr || kv_start != nullptr || bias != nullptr ||
                               alibi_slopes != nullptr || p_drop > 0.f))
    return -6;
  for (int i = 0; i < 3; ++i)
    if ((q_strides[i] % 8) || (k_strides[i] % 8) || (v_strides[i] % 8)) return -3;
  if (q_strides[3] % 8) return -3;
  CUtensorMap tq, tk, tv;
  if (!make_q_tmap(&tq, q, B, G, A / G, Sq, D, q_strides, 128)) return -2;
  if (!make_qkv_tmap(&tk, k, B, G, Sk, D, k_strides, 128)) return -2;
  if (!make_qkv_tmap(&tv, v, B, G, Sk, D, v_strides, 128)) return -2;
  lb::AttnFwdParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.B = B;
  p.A = A;
  p.r = A / G;
  p.Sq = Sq;
  p.Sk = Sk;
  p.d = D;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.kv_lens = kv_lens;
  p.kv_start = kv_start;
  p.doc_start = doc_start;
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
  cudaError_t e = (tile == 64) ? launch_fwd<64>(tq, tk, tv, p, s) : launch_fwd<128>(tq, tk, tv, p, s);
  return (int)e;
}
// =================================================================================================
// Backward.  One CTA per (batch, K/V head, NWG consecutive 64-key blocks).  Consumer warpgroup w (warpgroups 1 ..
// NWG) owns key block kb = NWG * cta + w and loops over the r query heads of the group and, for each, over the
// 64-query blocks that attend to it; warpgroup 0 holds the TMA producer (warp 0) and the dQ writer (warp 1).  With
// NWG = 2 the producer warpgroup gives its registers to the consumers (setmaxnreg), and one warpgroup's exp / dS math
// overlaps the other's wgmmas (attn_bwd_wgs says which instances run two).
// Which query blocks a key block visits depends on the shapes only (Sq, Sk, causal): under the causal mask query block
// i and key block kb meet iff 64 kb <= 64 i + 63 + (Sk - Sq).  Keys outside a sample's kv_start / kv_lens window are
// masked element-wise, so every visit happens and the dQ ordering below counts the same visits on both sides.
// The warpgroups of a CTA step through one sequence of (query head, query block) visits, from the first query block
// its lowest key block meets; the producer loads Q_i, dO_i and the block's lse and δ once for all of them, and a
// warpgroup whose key block does not meet query block i (a higher block under the causal mask) lets that visit pass
// without an MMA.
// Packed sequences (DOC): a visit in which every query row's document starts after the key block is skipped by its
// warpgroup (no MMA), and by the producer (no Q / dO load) when every key block of the CTA skips it; skips are taken
// from the same minimum over the rows everywhere.  A skipped visit does not touch the dQ order counter: whether a
// visit is skipped is monotone in the key block (skipped blocks lie below every contributing one), so a contributing
// key block waits for exactly the contributing blocks above it, and the contributions land in decreasing key-block
// order.
//   Sᵀ = K·Q_iᵀ , dPᵀ = V·dO_iᵀ                  (wgmma, registers)
//   Pᵀ = exp(Sᵀ·scale − lse) , dSᵀ = Pᵀ ∘ (dPᵀ − δ) · scale
//   dV += Pᵀ·dO_i , dK += dSᵀ·Q_i                 (A operands straight from the registers, accumulators stay in
//                                                  registers for the whole CTA: the group's sum is formed in a fixed
//                                                  order and written once, no atomics)
//   dQ_i += dS·K                                  (dSᵀ through shared memory, read as a transposed A operand; the fp32
//                                                  partial goes to a shared staging buffer and the consumer moves on)
// The dQ writer warp adds the staged partials to dq_accum (one cp.reduce.async.bulk add.f32 per partial), key block
// after key block in decreasing order: a per-(query head, query block) counter in global memory orders the CTAs, and
// within a CTA the writer takes the partials of a visit from the highest key block down, so every element of dq_accum
// receives the same additions in the same order as with one key block per CTA, and the sums are deterministic.  Key block kb adds to query block
// i once the counter shows the last_kb - kb blocks above it that visit i; the writer then fences its additions and
// releases the counter.  Key block kb at step `it` needs what kb + 1 added at an earlier step, so the CTAs do not
// stall each other, and the highest key blocks are launched first so that a waiter's predecessor is resident.
// Forward progress of that wait relies on the hardware dispatching the CTAs of a grid in increasing linear block index:
// a writer waits either for its own CTA's higher key block, whose partial it added itself just before, or for a CTA
// of lower linear index, whose writer in turn waits only for lower indices (the same assumption as FlashAttention-3's
// deterministic backward).  Inside a CTA nothing waits for the writer except a consumer whose staging buffers are all
// full, so the writer's progress is all the consumers need.  Should the assumption ever fail, the bounded spin wait
// traps after its timeout instead of hanging.
// δ = rowsum(dO ∘ O) is produced by attn_delta_kernel, dq_accum is converted to bf16 afterwards.
// =================================================================================================
namespace lb {

// consumer warpgroups (64-key blocks) per CTA of an instance.  Two share the register file with the producer
// warpgroup at 224 registers each (the producer keeps 56), which the dropout and head-dim-128 consumers exceed: those
// keep one consumer warpgroup and all 255 registers.
template <int D, int BIAS, bool DROP>
constexpr int attn_bwd_wgs() {
  return D == 64 && !DROP ? 2 : 1;
}

template <int D, int NWG>
struct AttnBwdCfg {
  static constexpr int CHUNKS = D / 64;
  static constexpr int THREADS = 128 * (NWG + 1);
  static constexpr int TILE_BYTES = 64 * D * 2;      // 64 rows of K / V / Q / dO
  static constexpr int DS_BYTES = 64 * 64 * 2;       // one warpgroup's dSᵀ
  static constexpr int DQ_BYTES = 64 * D * 4;        // one staged fp32 dQ partial
  static constexpr int DQ_BUFS = 2;                  // staging buffers per warpgroup
  static constexpr int ROW_BYTES = 2 * 64 * 4;       // lse and δ of a query block
  static constexpr int BAR_BYTES = 512;
  static constexpr int FIXED = 2 * NWG * TILE_BYTES /*K, V*/ + NWG * DS_BYTES + NWG * DQ_BUFS * DQ_BYTES;
  static constexpr int STAGE_BYTES = 2 * TILE_BYTES /*Q, dO*/ + ROW_BYTES;
  // as many Q / dO stages as the 227 KB of shared memory per block hold: 6 with two consumer warpgroups at D = 64,
  // 10 with one, 3 at D = 128
  static constexpr int STAGES = (227 * 1024 - 1024 - BAR_BYTES - FIXED) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = FIXED + STAGES * STAGE_BYTES + BAR_BYTES + 1024;
  static_assert(STAGES >= 2, "the Q / dO ring needs two stages");
  static_assert((1 + 2 * STAGES + 2 * NWG * DQ_BUFS) * 8 <= BAR_BYTES, "barriers");
};

struct AttnBwdParams {
  const float* lse;     // [B, A, Sq]
  const float* delta;   // [B, A, Sq]
  float* dq_accum;      // [B, A, query blocks] tiles of [64][D] fp32 (dq_tile_index)
  __nv_bfloat16* dk;    // strided [B, G, Sk, d] views
  __nv_bfloat16* dv;
  long g_strides[3];    // batch, head, seq strides (elements) of dk / dv
  int B, A, Sq, Sk;
  int d;                // head dim (d <= D, a multiple of 8)
  int r;                // query heads per K/V head (G = A / r)
  int causal;
  float scale, scale_log2;
  const int* kv_lens;   // optional [B]
  const int* kv_start;  // optional [B]
  const int* doc_start; // [B, Sq] in the DOC instances
  // same additive bias / dropout description as the forward; `rng_state` = the (seed, offset) pair the forward used
  const __nv_bfloat16* bias;
  long bias_strides[3];
  const float* alibi_slopes;
  float* dbias;         // optional fp32, same strides as `bias`: += P ∘ (dP − δ) (gradient of a learned bias)
  uint32_t drop_thresh;
  float inv_keep;
  const long long* rng_state;
  unsigned* dq_order;   // [B * A * query blocks]: key blocks whose dQ contribution has landed (zeroed by the caller)
  SpinTimeout* timeout_rec;  // where a timed-out dq_order wait leaves its diagnostic (host-mapped)
};

// DOC: true when no row of the query block [q0, q0 + 64) sees a key of the block [k0, k0 + 64), i.e. every row's
// document starts after it.  Called by a whole warp; rows past Sq repeat the last row.
LB_DEVICE bool doc_visit_empty(const int* doc_start, int S, int batch, int q0, int k0) {
  const int lane = threadIdx.x % 32;
  const int m = min(doc_begin(doc_start, S, batch, min(q0 + lane, S - 1)),
                    doc_begin(doc_start, S, batch, min(q0 + 32 + lane, S - 1)));
  return __reduce_min_sync(0xffffffffu, m) >= k0 + ATT_BWD_BN;
}
// first query block whose last row (64 i + 63) sees key block kb: floor((64 kb - (Sk - Sq)) / 64), at least 0 (C
// division truncates a negative quotient towards 0, which the max turns into the same 0).  At most nq - 1, since
// 64 kb <= Sk - 1.
LB_DEVICE int bwd_first_qblock(const AttnBwdParams& p, int kb) {
  return p.causal ? max(0, (kb * ATT_BWD_BN - (p.Sk - p.Sq)) / ATT_BWD_BM) : 0;
}
// dq_accum holds each (batch, query head, 64-query block) as one [64][D] fp32 tile, stored as the backward stages its
// dQ partials so that the writer adds a partial with one bulk operation: row-major, the 16-byte chunks of a row
// swizzled with the row (chunk c at c ^ (row % 8)), which keeps the consumers' fragment stores free of bank conflicts.
// Rows past Sq and columns past d are padding: the accumulator holds B·A·⌈Sq/64⌉·64·D floats against B·A·Sq·d for
// a dense one, e.g. 2.7x at d = 24 and 1.6x at d = 80 (both cleared by the delta kernel).  Returns the float index of
// (row, col) inside a tile.
template <int D>
LB_DEVICE int dq_tile_index(int row, int col) {
  return row * D + ((((col >> 2) ^ row) & 7) | ((col >> 2) & ~7)) * 4 + (col & 3);
}
// whether key block kb (of nkb) visits query block qb; called by a whole warp (DOC)
template <bool DOC>
LB_DEVICE bool bwd_visits(const AttnBwdParams& p, int batch, int nkb, int kb, int qb) {
  if (kb >= nkb || qb < bwd_first_qblock(p, kb)) return false;
  return !DOC || !doc_visit_empty(p.doc_start, p.Sq, batch, qb * ATT_BWD_BM, kb * ATT_BWD_BN);
}

template <int D, int BIAS, bool DROP, bool DOC>
__global__ void __launch_bounds__(AttnBwdCfg<D, attn_bwd_wgs<D, BIAS, DROP>()>::THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do, AttnBwdParams p) {
  static_assert(!DOC || (BIAS == BIAS_NONE && !DROP), "packed sequences run without bias and dropout");
  constexpr int NWG = attn_bwd_wgs<D, BIAS, DROP>();
  using Cfg = AttnBwdCfg<D, NWG>;
  constexpr int STAGES = Cfg::STAGES, DQ_BUFS = Cfg::DQ_BUFS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;                               // NWG tiles
  uint8_t* sV = sK + NWG * Cfg::TILE_BYTES;         // NWG tiles
  uint8_t* sQ = sV + NWG * Cfg::TILE_BYTES;         // STAGES
  uint8_t* sDO = sQ + STAGES * Cfg::TILE_BYTES;     // STAGES
  uint8_t* sDS = sDO + STAGES * Cfg::TILE_BYTES;    // NWG
  float* sDQ = reinterpret_cast<float*>(sDS + NWG * Cfg::DS_BYTES);   // NWG x DQ_BUFS partials [64][D], 16-byte swizzle
  float* sRow = sDQ + NWG * DQ_BUFS * 64 * D;       // STAGES x {lse[64], δ[64]}
  uint64_t* bars = reinterpret_cast<uint64_t*>(sRow + STAGES * 128);
  uint64_t* kv_full = bars;
  uint64_t* qdo_full = bars + 1;                    // STAGES
  uint64_t* qdo_empty = qdo_full + STAGES;          // STAGES
  uint64_t* dq_full = qdo_empty + STAGES;           // NWG x DQ_BUFS
  uint64_t* dq_empty = dq_full + NWG * DQ_BUFS;     // NWG x DQ_BUFS

  const int warp_idx = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int cta = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);   // highest keys first
  const int kv_head = blockIdx.y, batch = blockIdx.z;
  const int nkb = (p.Sk + ATT_BWD_BN - 1) / ATT_BWD_BN;
  const int kb0 = NWG * cta;                        // the CTA's lowest key block
  const int off = p.Sk - p.Sq;
  const int nq = (p.Sq + ATT_BWD_BM - 1) / ATT_BWD_BM;
  const int i_begin = bwd_first_qblock(p, kb0);
  const int iters = nq - i_begin;   // query blocks per query head
  const int steps = p.r * iters;    // step = (query head in group) * iters + query block - i_begin

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    tma_prefetch_desc(&tmap_do);
    mbar_init(kv_full, 1);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&qdo_full[i], 1);
      mbar_init(&qdo_empty[i], NWG * 128);
    }
    for (int i = 0; i < NWG * DQ_BUFS; ++i) {
      mbar_init(&dq_full[i], 128);
      mbar_init(&dq_empty[i], 1);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp_idx < 4) {
    if constexpr (NWG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 56;\n" ::: "memory");
    if (warp_idx == 0) {   // ---- producer: K / V once, then Q_i, dO_i, lse_i, δ_i per visit some warpgroup makes
      if (lane == 0) {
        const int nblk = min(NWG, nkb - kb0);
        mbar_arrive_expect_tx(kv_full, 2 * nblk * Cfg::TILE_BYTES);
        for (int w = 0; w < nblk; ++w) {
#pragma unroll
          for (int c = 0; c < Cfg::CHUNKS; ++c) {
            tma_load_4d(sK + w * Cfg::TILE_BYTES + c * (64 * 128), &tmap_k, kv_full, c * 64, (kb0 + w) * ATT_BWD_BN, kv_head, batch);
            tma_load_4d(sV + w * Cfg::TILE_BYTES + c * (64 * 128), &tmap_v, kv_full, c * 64, (kb0 + w) * ATT_BWD_BN, kv_head, batch);
          }
        }
      }
      int ld = 0;   // visits loaded so far: the Q / dO ring position
      for (int step = 0; step < steps; ++step) {
        const int hi = step / iters;
        const int qb = i_begin + step - hi * iters;
        bool need = false;
#pragma unroll
        for (int w = 0; w < NWG; ++w) need = need || bwd_visits<DOC>(p, batch, nkb, kb0 + w, qb);
        if (!need) continue;
        const int st = ld % STAGES;
        mbar_wait(&qdo_empty[st], ((ld / STAGES) & 1) ^ 1);
        const int q0 = qb * ATT_BWD_BM;
        const size_t bh = static_cast<size_t>(batch) * p.A + kv_head * p.r + hi;
        for (int i = lane; i < ATT_BWD_BM; i += 32) {   // rows past Sq are never read
          const int q = min(q0 + i, p.Sq - 1);
          sRow[st * 128 + i] = p.lse[bh * p.Sq + q];
          sRow[st * 128 + 64 + i] = p.delta[bh * p.Sq + q];
        }
        __syncwarp();
        if (lane == 0) {
          mbar_arrive_expect_tx(&qdo_full[st], 2 * Cfg::TILE_BYTES);
#pragma unroll
          for (int c = 0; c < Cfg::CHUNKS; ++c) {
            tma_load_5d(sQ + st * Cfg::TILE_BYTES + c * (64 * 128), &tmap_q, &qdo_full[st], c * 64, q0, hi, kv_head, batch);
            tma_load_5d(sDO + st * Cfg::TILE_BYTES + c * (64 * 128), &tmap_do, &qdo_full[st], c * 64, q0, hi, kv_head, batch);
          }
        }
        ++ld;
      }
    } else if (warp_idx == 1) {   // ---- dQ writer: the staged partials into dq_accum, in decreasing key-block order
      int staged[NWG];
#pragma unroll
      for (int w = 0; w < NWG; ++w) staged[w] = 0;
      for (int step = 0; step < steps; ++step) {
        const int hi = step / iters;
        const int qb = i_begin + step - hi * iters;
        bool makes[NWG];
#pragma unroll
        for (int w = 0; w < NWG; ++w) makes[w] = bwd_visits<DOC>(p, batch, nkb, kb0 + w, qb);
        if (lane == 0) {
          const size_t blk = (static_cast<size_t>(batch) * p.A + kv_head * p.r + hi) * nq + qb;
          unsigned* order = p.dq_order + blk;
          // the key blocks above kb that visit query block qb: all of them, or under the causal mask
          // kb' <= (64 qb + 63 + off) / 64 (a non-negative quotient, since kb visits qb)
          const int last_kb = p.causal ? min(nkb - 1, (qb * ATT_BWD_BM + ATT_BWD_BM - 1 + off) / ATT_BWD_BN) : nkb - 1;
          uint32_t landed = 0;   // partials of this visit added so far
#pragma unroll
          for (int w = NWG - 1; w >= 0; --w) {
            if (!makes[w]) continue;
            const int kb = kb0 + w, b = staged[w] % DQ_BUFS;
            const uint32_t par = (staged[w] / DQ_BUFS) & 1;
            ++staged[w];
            // after the partial of the key block above, added by this thread, the counter is at this block's target
            if (landed == 0) {
              spin_wait_ge_gpu(order, static_cast<uint32_t>(last_kb - kb), 0, p.timeout_rec, /*what=*/5, kb);
              asm volatile("fence.proxy.async.global;\n" ::: "memory");   // the acquire orders the bulk addition below
            }
            mbar_wait(&dq_full[w * DQ_BUFS + b], par);
            bulk_reduce_add_f32(p.dq_accum + blk * (64 * D), sDQ + (w * DQ_BUFS + b) * (64 * D), 64 * D * 4);
            tma_store_commit();
            tma_store_wait<0>();   // performed: the next partial of this query block adds on top of it
            mbar_arrive(&dq_empty[w * DQ_BUFS + b]);
            ++landed;
          }
          if (landed) {
            __threadfence();
            asm volatile("red.release.gpu.global.add.u32 [%0], %1;\n" ::"l"(order), "r"(landed) : "memory");
          }
        }
        __syncwarp();
      }
    }
    return;
  }
  if constexpr (NWG == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 224;\n" ::: "memory");

  // ---- consumer warpgroup w: key block kb0 + w
  const int w = NWG == 1 ? 0 : warp_idx / 4 - 1;   // (a constant with one warpgroup: fewer address registers)
  const int kb = kb0 + w;
  const int k0 = kb * ATT_BWD_BN;
  const int kv_len = p.kv_lens != nullptr ? max(1, min(p.Sk, p.kv_lens[batch])) : p.Sk;
  const int kv_beg = p.kv_start != nullptr ? min(max(p.kv_start[batch], 0), p.Sk) : 0;
  const int t = threadIdx.x % 128;
  const int r_loc = 16 * (t / 32) + (t % 32) / 4;         // fragment rows r_loc, r_loc + 8
  const int cq = 2 * (t % 4);
  constexpr float LOG2E = 1.4426950408889634f;
  unsigned long long rng_seed = 0, rng_offset = 0;
  if constexpr (DROP) {
    rng_seed = static_cast<unsigned long long>(p.rng_state[0]);
    rng_offset = static_cast<unsigned long long>(p.rng_state[1]);
  }
  const float inv_scale = 1.0f / p.scale;
  const uint32_t k_addr = smem_u32(sK + w * Cfg::TILE_BYTES), v_addr = smem_u32(sV + w * Cfg::TILE_BYTES);
  uint8_t* my_ds = sDS + w * Cfg::DS_BYTES;
  const uint32_t ds_addr = smem_u32(my_ds);
  // this thread's key rows are fixed for the CTA: a row before kv_start is never visible, which folds into the one
  // comparison against key_lim per element (INT_MAX is never below it)
  int kvis[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) kvis[h] = k0 + r_loc + 8 * h >= kv_beg ? k0 + r_loc + 8 * h : INT_MAX;

  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) {
    dv[i] = 0.f;
    dk[i] = 0.f;
  }
  mbar_wait(kv_full, 0);

  int ld = 0;       // visits loaded so far (the producer's ring position)
  int staged = 0;   // dQ partials staged so far
  for (int step = 0; step < steps; ++step) {
    const int hi = step / iters;
    const int it = step - hi * iters;
    const int qb = i_begin + it;
    const bool mine = bwd_visits<DOC>(p, batch, nkb, kb, qb);
    bool need = mine;
#pragma unroll
    for (int u = 0; u < NWG; ++u)
      if (u != w) need = need || bwd_visits<DOC>(p, batch, nkb, kb0 + u, qb);
    if (!need) continue;   // not loaded
    const int st = ld % STAGES;
    mbar_wait(&qdo_full[st], (ld / STAGES) & 1);
    ++ld;
    if (mine) {
      const int head = kv_head * p.r + hi;   // query head
      const size_t bh = static_cast<size_t>(batch) * p.A + head;
      float slope2 = 0.f;
      if constexpr (BIAS == BIAS_ALIBI) slope2 = p.alibi_slopes[head] * LOG2E;
      const long bias_bh = batch * p.bias_strides[0] + head * p.bias_strides[1];
      const int q0 = qb * ATT_BWD_BM;
      const float* s_lse = sRow + st * 128;
      const float* s_delta = s_lse + 64;
      const uint32_t q_addr = smem_u32(sQ + st * Cfg::TILE_BYTES), do_addr = smem_u32(sDO + st * Cfg::TILE_BYTES);
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
          const bool q_ok = q_idx < p.Sq;
          const float lse2 = q_ok ? s_lse[8 * jj + cq + c] * LOG2E : 0.f;
          const float delta_s = q_ok ? s_delta[8 * jj + cq + c] * p.scale : 0.f;
          const int key_lim = !q_ok ? 0 : (p.causal ? min(kv_len, q_idx + off + 1) : kv_len);
          const int key_lo = DOC && q_ok ? doc_begin(p.doc_start, p.Sq, batch, q_idx) : 0;   // the query's document
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
              boff = bias_bh + static_cast<long>(min(q_idx, p.Sq - 1)) * p.bias_strides[2] + min(kidx, p.Sk - 1);
              x = fmaf(__bfloat162float(p.bias[boff]), LOG2E, x);
            } else if constexpr (BIAS == BIAS_ALIBI) {
              x = fmaf(slope2, static_cast<float>(kidx - q_idx - off), x);
            }
            const float pv = kvis[h] < key_lim && (!DOC || kvis[h] >= key_lo) ? fast_exp2(x - lse2) : 0.f;
            float g = dpT[i], pd = pv;   // dP w.r.t. the dropped, rescaled P; what multiplied V in the forward
            if constexpr (DROP) {
              const bool keep = rnd_byte(rnd, (r_loc + 8 * h) & 15) >= p.drop_thresh;
              g = keep ? g * p.inv_keep : 0.f;
              pd = keep ? pv * p.inv_keep : 0.f;
            }
            const float ds = pv * fmaf(g, p.scale, -delta_s);
            if constexpr (BIAS == BIAS_DENSE) {
              // d bias = P ∘ (dP − δ): fp32 reductions (broadcast dims sum over CTAs)
              if (p.dbias != nullptr && q_ok && kidx < p.Sk) atomicAdd(p.dbias + boff, ds * inv_scale);
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
          *reinterpret_cast<uint32_t*>(my_ds + row * 128 + ((jj ^ (row & 7)) << 4) + cq * 2) =
              pack_bf16(dpT[4 * jj + 2 * h], dpT[4 * jj + 2 * h + 1]);
        }
      }
      fence_proxy_async();
      warpgroup_sync(w);
      // ---- dV += Pᵀ·dO_i, dK += dSᵀ·Q_i (B operands: the [query, D] tiles read MN-major)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_bf16_rs<D, 1>(dv, pa[kk], make_smem_desc_sw128(do_addr + kk * (16 * 128), 64 * 128, 1024), 1u);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_bf16_rs<D, 1>(dk, da[kk], make_smem_desc_sw128(q_addr + kk * (16 * 128), 64 * 128, 1024), 1u);
      wgmma_commit();
      // ---- dQ_i = dS·K, 64 columns at a time (A = dSᵀ read transposed, B = the K tile read MN-major), staged for the
      // writer in the layout of a dq_accum tile
      const int b = staged % DQ_BUFS;
      const uint32_t dpar = (staged / DQ_BUFS) & 1;
      ++staged;
      float* stage = sDQ + (w * DQ_BUFS + b) * (64 * D);
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
        if (n == 0) mbar_wait(&dq_empty[w * DQ_BUFS + b], dpar ^ 1);
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r_loc + 8 * h;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int col = n * 64 + 8 * jj + cq;
            *reinterpret_cast<float2*>(stage + dq_tile_index<D>(row, col)) = make_float2(dq[4 * jj + 2 * h], dq[4 * jj + 2 * h + 1]);
          }
        }
      }
      fence_proxy_async();   // the writer's bulk addition reads the tile through the async proxy
      mbar_arrive(&dq_full[w * DQ_BUFS + b]);
      wgmma_fence_regs(dv);
      wgmma_fence_regs(dk);
    }
    mbar_arrive(&qdo_empty[st]);
  }

  // ---- dV / dK: fragment rows = key rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k_idx = k0 + r_loc + 8 * h;
    if (k_idx >= p.Sk) continue;
    const long off = batch * p.g_strides[0] + kv_head * p.g_strides[1] + static_cast<long>(k_idx) * p.g_strides[2];
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj) {
      if (!col_in_head<D>(8 * jj, p.d)) continue;
      *reinterpret_cast<uint32_t*>(p.dv + off + 8 * jj + cq) = pack_bf16(dv[4 * jj + 2 * h], dv[4 * jj + 2 * h + 1]);
      *reinterpret_cast<uint32_t*>(p.dk + off + 8 * jj + cq) = pack_bf16(dk[4 * jj + 2 * h], dk[4 * jj + 2 * h + 1]);
    }
  }
}

// delta[b, a, s] = sum_d dO[b, a, s, d] * O[b, a, s, d] over the head dim d <= D
// D / 8 lanes per row (lanes past d add zeros), 16-byte loads; rows are visited in (b, s, a) order = memory order of the
// [b, s, a, d] tensors, so a warp reads contiguous bytes per tensor, and every thread keeps 4 rows (8 loads) in flight.
template <int D>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ o, float* __restrict__ delta,
                  int B, int A, int S, int d, long sb, long sa, long ss, float4* __restrict__ zero_fill, long zero_n4) {
  constexpr int LPR = D / 8;  // lanes per row
  const long total = static_cast<long>(B) * A * S;
  const long gid = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  // the fp32 dQ accumulator of the main kernel is cleared here (one launch and one pass less than a memset in front)
  for (long z = gid; z < zero_n4; z += static_cast<long>(gridDim.x) * blockDim.x) zero_fill[z] = make_float4(0.f, 0.f, 0.f, 0.f);
  const long gstride = static_cast<long>(gridDim.x) * blockDim.x / LPR;
  const int sub = static_cast<int>(gid % LPR);
  const bool col_ok = sub * 8 < d;
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
      x[u] = ok && col_ok ? *reinterpret_cast<const uint4*>(dout + off) : make_uint4(0, 0, 0, 0);
      y[u] = ok && col_ok ? *reinterpret_cast<const uint4*>(o + off) : make_uint4(0, 0, 0, 0);
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

// dq (strided bf16, query head a = group a / r, slot a % r) = dq_accum (tiles of [64][D] fp32, dq_tile_index); 8
// columns per thread (two 16-byte loads, one 16-byte store)
template <int D>
__global__ void __launch_bounds__(256)
attn_dq_convert_kernel(const float* __restrict__ acc, __nv_bfloat16* __restrict__ dq, int B, int A, int S, int d, int r,
                       long sb, long sg, long si, long ss) {
  const int vpr = d / 8;   // 8-column groups per row
  const long nvec = static_cast<long>(B) * A * S * vpr;
  const long nq = (S + ATT_BWD_BM - 1) / ATT_BWD_BM;
  const long stride = static_cast<long>(gridDim.x) * blockDim.x;
  for (long i0 = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i0 < nvec; i0 += 2 * stride) {
    float4 lo[2], hi[2];
    long row[2];
    int col[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long i = i0 + u * stride;
      row[u] = i / vpr;
      col[u] = static_cast<int>(i - row[u] * vpr) * 8;
      if (i < nvec) {
        const int sq = static_cast<int>(row[u] % S);
        const float* tile = acc + ((row[u] / S) * nq + sq / ATT_BWD_BM) * (ATT_BWD_BM * D);
        lo[u] = *reinterpret_cast<const float4*>(tile + dq_tile_index<D>(sq % ATT_BWD_BM, col[u]));
        hi[u] = *reinterpret_cast<const float4*>(tile + dq_tile_index<D>(sq % ATT_BWD_BM, col[u] + 4));
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (i0 + u * stride < nvec) {
        const int sq = static_cast<int>(row[u] % S), a = static_cast<int>((row[u] / S) % A);
        const long b = row[u] / (static_cast<long>(S) * A);
        *reinterpret_cast<uint4*>(dq + b * sb + (a / r) * sg + (a % r) * si + sq * ss + col[u]) =
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

template <int D, int BIAS, bool DROP, bool DOC = false>
cudaError_t launch_bwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                         const lb::AttnBwdParams& p, cudaStream_t s) {
  constexpr int NWG = lb::attn_bwd_wgs<D, BIAS, DROP>();
  using Cfg = lb::AttnBwdCfg<D, NWG>;
  auto kern = lb::attn_bwd_kernel<D, BIAS, DROP, DOC>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  const int nkb = (p.Sk + lb::ATT_BWD_BN - 1) / lb::ATT_BWD_BN;   // 64-key blocks, NWG per CTA
  dim3 grid((nkb + NWG - 1) / NWG, p.A / p.r, p.B);
  kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, s>>>(tq, tk, tv, tdo, p);
  return cudaGetLastError();
}
template <int D>
cudaError_t launch_bwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                       const lb::AttnBwdParams& p, cudaStream_t s) {
  if (p.doc_start != nullptr) return launch_bwd_t<D, lb::BIAS_NONE, false, true>(tq, tk, tv, tdo, p, s);
  const int bias = p.bias != nullptr ? lb::BIAS_DENSE : (p.alibi_slopes != nullptr ? lb::BIAS_ALIBI : lb::BIAS_NONE);
  const bool drop = p.drop_thresh > 0;
  if (bias == lb::BIAS_NONE) return drop ? launch_bwd_t<D, lb::BIAS_NONE, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_NONE, false>(tq, tk, tv, tdo, p, s);
  if (bias == lb::BIAS_DENSE) return drop ? launch_bwd_t<D, lb::BIAS_DENSE, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_DENSE, false>(tq, tk, tv, tdo, p, s);
  return drop ? launch_bwd_t<D, lb::BIAS_ALIBI, true>(tq, tk, tv, tdo, p, s) : launch_bwd_t<D, lb::BIAS_ALIBI, false>(tq, tk, tv, tdo, p, s);
}
}  // namespace
// floats of the backward's dQ accumulator (fp32 [64][tile] per batch, query head and 64-query block)
extern "C" long lb_attn_bwd_accum_floats(int B, int A, int Sq, int D) {
  return (long)B * A * ((Sq + lb::ATT_BWD_BM - 1) / lb::ATT_BWD_BM) * lb::ATT_BWD_BM * head_dim_tile(D);
}
// A query heads in G groups; q_strides = {batch, group, in-group, seq}, k/v_strides = {batch, head, seq} over the G K/V
// heads, do_strides = {batch, head, seq} over the A query heads.  dq is written with dq_strides = {batch, group,
// in-group, seq}, dk and dv with dkv_strides = {batch, head, seq} (for Sq == Sk the caller passes views of one packed
// [B, S, G, r + 2, D] gradient).
extern "C" int lb_attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* o,
                           const float* lse, void* dq, void* dk, void* dv, const long* dq_strides, const long* dkv_strides,
                           float* delta, float* dq_accum, int B, int A, int G, int Sq, int Sk, int D, const long* q_strides,
                           const long* k_strides, const long* v_strides, const long* do_strides, int causal, float scale,
                           const int* kv_lens, const int* kv_start, const int* doc_start, const void* bias,
                           const long* bias_strides, const float* alibi_slopes, float* dbias, float p_drop,
                           const long long* rng_state, unsigned* dq_order, cudaStream_t s) {
  const int tile = head_dim_tile(D);
  if (tile == 0) return -1;
  if (Sq <= 0 || Sk <= 0) return -5;
  if (G <= 0 || A % G) return -4;
  if (doc_start != nullptr && (!causal || Sq != Sk || kv_lens != nullptr || kv_start != nullptr || bias != nullptr ||
                               alibi_slopes != nullptr || p_drop > 0.f))
    return -6;
  const int r = A / G;
  for (int i = 0; i < 3; ++i)
    if ((q_strides[i] % 8) || (k_strides[i] % 8) || (v_strides[i] % 8) || (do_strides[i] % 8)) return -3;
  if (q_strides[3] % 8) return -3;
  const long do_strides4[4] = {do_strides[0], r * do_strides[1], do_strides[1], do_strides[2]};
  CUtensorMap tq, tk, tv, tdo;
  if (!make_q_tmap(&tq, q, B, G, r, Sq, D, q_strides, 64)) return -2;
  if (!make_qkv_tmap(&tk, k, B, G, Sk, D, k_strides, 64)) return -2;
  if (!make_qkv_tmap(&tv, v, B, G, Sk, D, v_strides, 64)) return -2;
  if (!make_q_tmap(&tdo, dout, B, G, r, Sq, D, do_strides4, 64)) return -2;
  const long rows = (long)B * A * Sq;
  {
    // 4 rows per thread-group and iteration; cap the grid at a few waves
    const long groups = (rows + 3) / 4;
    const long lpr = tile / 8;
    long blocks = (groups * lpr + 255) / 256;
    if (blocks > sm_count() * 16L) blocks = sm_count() * 16L;
    if (tile == 64)
      lb::attn_delta_kernel<64><<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)o, delta, B,
                                                                   A, Sq, D, do_strides[0], do_strides[1], do_strides[2],
                                                                   reinterpret_cast<float4*>(dq_accum), lb_attn_bwd_accum_floats(B, A, Sq, D) / 4);
    else
      lb::attn_delta_kernel<128><<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)o, delta, B,
                                                                    A, Sq, D, do_strides[0], do_strides[1], do_strides[2],
                                                                    reinterpret_cast<float4*>(dq_accum), lb_attn_bwd_accum_floats(B, A, Sq, D) / 4);
  }
  lb::AttnBwdParams p;
  p.lse = lse;
  p.delta = delta;
  p.dq_accum = dq_accum;
  p.dk = (__nv_bfloat16*)dk;
  p.dv = (__nv_bfloat16*)dv;
  for (int i = 0; i < 3; ++i) p.g_strides[i] = dkv_strides[i];
  p.B = B;
  p.A = A;
  p.r = r;
  p.Sq = Sq;
  p.Sk = Sk;
  p.d = D;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.kv_lens = kv_lens;
  p.kv_start = kv_start;
  p.doc_start = doc_start;
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
  p.timeout_rec = lb_host::spin_timeout_record(s);
  cudaError_t e = (tile == 64) ? launch_bwd<64>(tq, tk, tv, tdo, p, s) : launch_bwd<128>(tq, tk, tv, tdo, p, s);
  if (e != cudaSuccess) return (int)e;
  const long nvec = rows * D / 8;
  int blocks = (int)((nvec + 511) / 512);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  auto convert = tile == 64 ? lb::attn_dq_convert_kernel<64> : lb::attn_dq_convert_kernel<128>;
  convert<<<blocks, 256, 0, s>>>(dq_accum, (__nv_bfloat16*)dq, B, A, Sq, D, r, dq_strides[0], dq_strides[1],
                                 dq_strides[2], dq_strides[3]);
  return (int)cudaGetLastError();
}
