// The split-KV decode attention kernel (documented in decode_attention_sm90.cu) and its launch.  Four translation units
// instantiate it: decode_attention_sm90.cu without a score bias, decode_attention_alibi_sm90.cu with ALiBi slopes,
// decode_attention_t5_sm90.cu with T5's relative-position bias or a non-causal key window, and
// decode_attention_fp8_sm90.cu every score kind over an FP8 (E4M3) cache.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace lb {
namespace dec {

constexpr int kTile = 64;                  // keys per pipeline stage
constexpr int kWarps = 4;                  // consumer warps, 16 keys of every tile each
constexpr int kThreads = (kWarps + 1) * 32;
constexpr int kMaxQ = 16;                  // rows of the m16n8k16 MMA: (query head, new token) pairs
constexpr int kMaxSplits = 32;

template <int D>
struct Cfg {
  static constexpr int kRow = D + 8;                       // padded smem row (elements): rows start 4 banks apart
  static constexpr int kStages = D == 128 ? 3 : 4;         // 104 / 74 KB: two or three CTAs per SM
  static constexpr int kStageElems = 2 * kTile * kRow;     // K tile, then V tile
  static constexpr int kRingBytes = kStages * kStageElems * 2;
  static constexpr int kMergeBytes = kWarps * kMaxQ * (D + 2) * 4;   // per-warp O, m, l for the merge
  static constexpr int kSmem = (kRingBytes > kMergeBytes ? kRingBytes : kMergeBytes) + 2 * kStages * 8;
};

// FP8 (E4M3) caches: K, V bytes [B, G, C, D] and one fp32 scale per row, [B, G, C] (C a multiple of 4, so every
// 4-row group of scales is 16-byte aligned).  A stage holds the window rows of one 64-key tile, each array loaded with
// one bulk copy: K, V, and their scales from the 16-byte boundary at or below the tile's first row.  Each consumer
// warp widens its own 16 keys of K and V to bf16 (exact) into a padded staging area of its own, read by the same
// ldmatrix code as the bf16 ring.  Four / six stages: 100 / 69 KB, two / three CTAs per SM at D = 128 / 64.
template <int D>
struct Cfg8 {
  static constexpr int kRow = D + 8;                                  // padded bf16 staging row (elements)
  static constexpr int kStages = D == 128 ? 4 : 6;
  static constexpr int kScales = kTile + 4;                           // floats of one scale array in a stage
  static constexpr int kStageBytes = 2 * kTile * D + 2 * kScales * 4;  // K, V bytes, then K, V scales
  static constexpr int kStagingBytes = kWarps * 2 * 16 * kRow * 2;    // per consumer warp: 16 keys of K, then of V
  static constexpr int kRingBytes = kStages * kStageBytes + kStagingBytes;
  static constexpr int kMergeBytes = Cfg<D>::kMergeBytes;
  static constexpr int kSmem = (kRingBytes > kMergeBytes ? kRingBytes : kMergeBytes) + 2 * kStages * 8;
};

struct Params {
  const __nv_bfloat16* q;      // [B, Sq, A, D] view: strides below (elements), D contiguous
  long q_sb, q_si, q_sh;
  const __nv_bfloat16* k;      // [B, G, C, D] contiguous
  const __nv_bfloat16* v;
  __nv_bfloat16* o;            // [B, Sq, A, D] contiguous
  float* part_o;               // [B, G, splits, r * Sq, D] (splits > 1)
  float2* part_ml;             // [B, G, splits, r * Sq]: (max, sum) in log2 units
  const int* seqlens;          // [B]
  const int* kv_start;         // [B]
  int A, G, C, Sq;
  int rows;                    // r * Sq
  int row_blocks;              // ceil(rows / 16)
  float scale_log2;
  int R;                       // Score::kRelBias: columns of the bias (in former padding: the layout is unchanged)
  const float* bias;           // Score::kAlibi: the slopes [A]; Score::kRelBias: the relative bias [A, R]
};

// What a visible score gets besides q·k·scale, and which keys are visible.  kNone, kAlibi, kRelBias: query i of sample b
// sees kv_start[b] <= j <= cache_seqlens[b] + i (causal); kWindow: every query sees kv_start[b] <= j < cache_seqlens[b].
enum class Score { kNone, kAlibi, kRelBias, kWindow };

LB_DEVICE void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// FP8: p.k / p.v point at the E4M3 bytes and k_scale / v_scale at their row scales; key j's score is
// scale·s^k_j·(q·ê_j), and P·V runs on P_j·s^v_j while the softmax sums P_j.
// PAGED (decode_attention_paged_sm90.cu): p.k, p.v (and the FP8 scales) are pools of pages [P, G, kTile, D]
// ([P, G, kTile]), logical row j of sample b is row j % kTile of page block_table[b * max_pages + j / kTile], and
// p.C = max_pages * kTile.  Only the producer's addresses change: the tiles still start at kv_start[b], not at page
// boundaries, so every sum runs in the order of the contiguous kernel and the result is bit-identical to it over the
// same logical rows.  (The table is not a field of Params: a larger Params changes the code of every other instance.)
template <int D, Score S, bool FP8 = false, bool PAGED = false>
__device__ __forceinline__ void decode_attn_body(const Params& p, const float* k_scale = nullptr,
                                                 const float* v_scale = nullptr, const int* block_table = nullptr,
                                                 int max_pages = 0) {
  constexpr bool ALIBI = S == Score::kAlibi;
  using C = std::conditional_t<FP8, Cfg8<D>, Cfg<D>>;
  extern __shared__ __align__(128) unsigned char smem[];
  __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(smem);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (C::kRingBytes > C::kMergeBytes ? C::kRingBytes : C::kMergeBytes));
  uint64_t* empty = full + C::kStages;

  const int split = blockIdx.x, nsplit = gridDim.x, b = blockIdx.z;
  const int kvh = blockIdx.y / p.row_blocks;                  // cache head
  const int row0 = (blockIdx.y - kvh * p.row_blocks) * kMaxQ; // first (query head in group, token) row of this CTA
  const int nrows = min(kMaxQ, p.rows - row0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long head_off = ((long)b * p.G + kvh) * p.C * D;
  const int len = p.seqlens[b];
  const int lo = max(p.kv_start[b], 0);
  // exclusive; the cache object keeps len + Sq <= C, this only guards memory
  const int hi = S == Score::kWindow ? min(len, p.C) : min(len + p.Sq, p.C);
  const int ntiles = hi > lo ? (hi - lo + kTile - 1) / kTile : 0;
  const int per = (ntiles + nsplit - 1) / nsplit;
  const int t0 = split * per;
  const int my = max(0, min(ntiles, t0 + per) - t0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // merge state of the consumer warps (rows r0 and r0 + 8 of the 16 query rows)
  float o[D / 8][4];
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int n = 0; n < D / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  const int r0 = lane >> 2, c0 = (lane & 3) * 2;

  if (warp == kWarps) {
    if constexpr (FP8) {
      // producer: the window rows of each tile (clipped at hi) and their scales; nothing past the window is copied
      const uint8_t* kg = reinterpret_cast<const uint8_t*>(p.k) + head_off;
      const uint8_t* vg = reinterpret_cast<const uint8_t*>(p.v) + head_off;
      const long srow = ((long)b * p.G + kvh) * p.C;
      const int soff = lo & 3;   // first row of every tile past its 16-byte scale boundary
      for (int t = 0; t < my && lane == 0; ++t) {
        const int st = t % C::kStages;
        if (t >= C::kStages) mbar_wait(&empty[st], ((t / C::kStages) & 1) ^ 1);
        const int base = lo + (t0 + t) * kTile;
        const int n = min(kTile, hi - base), ns = (soff + n + 3) & ~3;
        unsigned char* sk = smem + st * C::kStageBytes;
        mbar_arrive_expect_tx(&full[st], 2 * n * D + 2 * ns * 4);
        if constexpr (PAGED) {
          // A tile spans at most two pages: one piece of each array per page.  The scales start at the 4-row boundary
          // base - soff, in the page of base (page boundaries are multiples of 4 rows), and end at the 4-row boundary
          // at or past base + n, which passes the page boundary only when the rows do: every piece of bytes and of
          // scales starts and ends on a 16-byte boundary, as in the contiguous layout.
          const int* table = block_table + (long)b * max_pages;
          for (int r = base - soff; r < base - soff + ns;) {
            const int end = min((r / kTile + 1) * kTile, base - soff + ns);
            const long pg = ((long)table[r / kTile] * p.G + kvh) * kTile;
            const int b0 = max(r, base), b1 = min(end, base + n);   // the rows of the piece
            if (b1 > b0) {
              bulk_load(sk + (b0 - base) * D, reinterpret_cast<const uint8_t*>(p.k) + (pg + b0 % kTile) * D,
                        (b1 - b0) * D, &full[st]);
              bulk_load(sk + kTile * D + (b0 - base) * D,
                        reinterpret_cast<const uint8_t*>(p.v) + (pg + b0 % kTile) * D, (b1 - b0) * D, &full[st]);
            }
            const int s0 = r - (base - soff);
            bulk_load(sk + 2 * kTile * D + s0 * 4, k_scale + pg + r % kTile, (end - r) * 4, &full[st]);
            bulk_load(sk + 2 * kTile * D + C::kScales * 4 + s0 * 4, v_scale + pg + r % kTile, (end - r) * 4,
                      &full[st]);
            r = end;
          }
        } else {
          bulk_load(sk, kg + (long)base * D, n * D, &full[st]);
          bulk_load(sk + kTile * D, vg + (long)base * D, n * D, &full[st]);
          bulk_load(sk + 2 * kTile * D, k_scale + srow + base - soff, ns * 4, &full[st]);
          bulk_load(sk + 2 * kTile * D + C::kScales * 4, v_scale + srow + base - soff, ns * 4, &full[st]);
        }
      }
    } else {
      // producer: rows past the window repeat its last row (finite data; those keys get zero weight)
      const __nv_bfloat16* kg = p.k + head_off;
      const __nv_bfloat16* vg = p.v + head_off;
      for (int t = 0; t < my; ++t) {
        const int st = t % C::kStages;
        if (t >= C::kStages) mbar_wait(&empty[st], ((t / C::kStages) & 1) ^ 1);
        if (lane == 0) mbar_arrive_expect_tx(&full[st], 2 * kTile * D * 2);
        __syncwarp();
        __nv_bfloat16* sk = ring + st * C::kStageElems;
        __nv_bfloat16* sv = sk + kTile * C::kRow;
        const int base = lo + (t0 + t) * kTile;
  #pragma unroll
        for (int r = lane; r < kTile; r += 32) {
          const long row = min(base + r, hi - 1);
          if constexpr (PAGED) {
            const long at = (((long)block_table[(long)b * max_pages + row / kTile] * p.G + kvh) * kTile +
                             row % kTile) * D;
            bulk_load(sk + r * C::kRow, p.k + at, D * 2, &full[st]);
            bulk_load(sv + r * C::kRow, p.v + at, D * 2, &full[st]);
          } else {
            bulk_load(sk + r * C::kRow, kg + row * D, D * 2, &full[st]);
            bulk_load(sv + r * C::kRow, vg + row * D, D * 2, &full[st]);
          }
        }
      }
    }
  } else if (my > 0) {
    // Q fragments (A operand, rows = (query head, new token) pairs; rows past the last pair are zero), loaded once.
    // lim: the last visible key of each of this thread's two rows (causal among the new tokens; the whole window
    // for kWindow)
    uint32_t qf[D / 16][4];
    int lim[2];
    float slope2[2] = {0.f, 0.f};   // ALiBi slope of each row's query head, times log2(e)
    const float* rb[2] = {nullptr, nullptr};   // kRelBias: the bias row of each row's query head
    {
      const int hr = kvh * (p.rows / p.Sq);   // first query head of the group
      const bool v0 = r0 < nrows, v1 = r0 + 8 < nrows;
      const int t0 = (row0 + r0) % p.Sq, t1 = (row0 + r0 + 8) % p.Sq;
      lim[0] = S == Score::kWindow ? hi - 1 : len + t0;
      lim[1] = S == Score::kWindow ? hi - 1 : len + t1;
      if constexpr (S == Score::kRelBias) {   // rows past the last pair read head 0's row (their scores are unused)
        rb[0] = p.bias + (v0 ? (long)(hr + (row0 + r0) / p.Sq) * p.R : 0);
        rb[1] = p.bias + (v1 ? (long)(hr + (row0 + r0 + 8) / p.Sq) * p.R : 0);
      }
      if constexpr (ALIBI) {
        constexpr float kLog2e = 1.4426950408889634f;
        slope2[0] = v0 ? p.bias[hr + (row0 + r0) / p.Sq] * kLog2e : 0.f;
        slope2[1] = v1 ? p.bias[hr + (row0 + r0 + 8) / p.Sq] * kLog2e : 0.f;
      }
      const __nv_bfloat16* qb = p.q + (long)b * p.q_sb + c0;
      const uint32_t* q0 = reinterpret_cast<const uint32_t*>(
          qb + (long)t0 * p.q_si + (long)(hr + (row0 + r0) / p.Sq) * p.q_sh);
      const uint32_t* q1 = reinterpret_cast<const uint32_t*>(
          qb + (long)t1 * p.q_si + (long)(hr + (row0 + r0 + 8) / p.Sq) * p.q_sh);
#pragma unroll
      for (int ks = 0; ks < D / 16; ++ks) {
        qf[ks][0] = v0 ? q0[ks * 8] : 0u;
        qf[ks][1] = v1 ? q1[ks * 8] : 0u;
        qf[ks][2] = v0 ? q0[ks * 8 + 4] : 0u;
        qf[ks][3] = v1 ? q1[ks * 8 + 4] : 0u;
      }
    }
    const int kw = warp * 16;
    const int kr = FP8 ? 0 : kw;   // the first of this warp's keys among the rows ldmatrix reads (FP8: its staging)
    // ldmatrix lane addresses: K (non-transposed: keys = rows of the B fragment), V (transposed)
    const int k_row = kr + (lane & 7) + ((lane >> 4) << 3), k_col = ((lane >> 3) & 1) * 8;
    const int v_row = kr + (lane & 7) + (((lane >> 3) & 1) << 3), v_col = (lane >> 4) * 8;
    for (int t = 0; t < my; ++t) {
      const int st = t % C::kStages;
      mbar_wait(&full[st], (t / C::kStages) & 1);
      const __nv_bfloat16* sk;
      const __nv_bfloat16* sv;
      float ksc[2][2], vsc[2][2];   // FP8: the scales of this thread's keys kw + n * 8 + c0 + e (0 past the window)
      if constexpr (FP8) {
        const unsigned char* stage = smem + st * C::kStageBytes;
        __nv_bfloat16* stg = reinterpret_cast<__nv_bfloat16*>(smem + C::kStages * C::kStageBytes) +
                             warp * 2 * 16 * C::kRow;
        const int first = lo + (t0 + t) * kTile + kw;   // this warp's first key
        __syncwarp();   // the previous tile's ldmatrix reads of the staging area are done
        // widen 16 bytes per lane and step: rows past the window become zeros (the bytes there were not copied)
#pragma unroll
        for (int c = lane; c < D; c += 32) {   // 16 rows of D / 16 chunks
          const int r = c / (D / 16), col = (c % (D / 16)) * 16;
          const bool in = first + r < hi;
          const uint4 kx = in ? *reinterpret_cast<const uint4*>(stage + (kw + r) * D + col) : make_uint4(0, 0, 0, 0);
          const uint4 vx = in ? *reinterpret_cast<const uint4*>(stage + kTile * D + (kw + r) * D + col)
                              : make_uint4(0, 0, 0, 0);
          uint4* dk = reinterpret_cast<uint4*>(stg + r * C::kRow + col);
          uint4* dv = reinterpret_cast<uint4*>(stg + (16 + r) * C::kRow + col);
          const uint2 k0 = e4m3x4_to_bf16x4(kx.x), k1 = e4m3x4_to_bf16x4(kx.y), k2 = e4m3x4_to_bf16x4(kx.z),
                      k3 = e4m3x4_to_bf16x4(kx.w);
          dk[0] = make_uint4(k0.x, k0.y, k1.x, k1.y);
          dk[1] = make_uint4(k2.x, k2.y, k3.x, k3.y);
          const uint2 v0 = e4m3x4_to_bf16x4(vx.x), v1 = e4m3x4_to_bf16x4(vx.y), v2 = e4m3x4_to_bf16x4(vx.z),
                      v3 = e4m3x4_to_bf16x4(vx.w);
          dv[0] = make_uint4(v0.x, v0.y, v1.x, v1.y);
          dv[1] = make_uint4(v2.x, v2.y, v3.x, v3.y);
        }
        const float* ks = reinterpret_cast<const float*>(stage + 2 * kTile * D) + (lo & 3) + kw;
        const float* vs = ks + C::kScales;
#pragma unroll
        for (int n = 0; n < 2; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = n * 8 + c0 + e;
            ksc[n][e] = first + k < hi ? ks[k] : 0.f;
            vsc[n][e] = first + k < hi ? vs[k] : 0.f;
          }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);   // this warp is done with the stage: the producer may refill it
        sk = stg;
        sv = stg + 16 * C::kRow;
      } else {
        sk = ring + st * C::kStageElems;
        sv = sk + kTile * C::kRow;
      }
      float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int ks = 0; ks < D / 16; ++ks) {
        uint32_t bk[4];
        ldsm_x4(bk, sk + k_row * C::kRow + ks * 16 + k_col);
        mma_bf16(s[0], qf[ks], bk[0], bk[1]);
        mma_bf16(s[1], qf[ks], bk[2], bk[3]);
      }
      // mask + online softmax (log2 domain); the two rows of this thread are r0 and r0 + 8
      const int key0 = lo + (t0 + t) * kTile + kw + c0;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int n = 0; n < 2; ++n)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int key = key0 + n * 8 + (j & 1);
          const bool vis = key < hi && key <= lim[j >> 1];
          if constexpr (FP8) s[n][j] *= ksc[n][j & 1];
          if constexpr (ALIBI) {   // key − lim is a non-positive integer of at most the capacity: exact in fp32
            s[n][j] = vis ? fmaf(slope2[j >> 1], static_cast<float>(key - lim[j >> 1]), s[n][j] * p.scale_log2)
                          : -INFINITY;
          } else if constexpr (S == Score::kRelBias) {
            // bias of the distance lim − key = cache_seqlens[b] + i − j, constant from R − 1 on; a few hundred bytes
            // per head, read through L1 (the clamp below 0 only keeps the address of an invisible key in the row)
            constexpr float kLog2e = 1.4426950408889634f;
            const float bias = __ldg(rb[j >> 1] + min(max(lim[j >> 1] - key, 0), p.R - 1));
            s[n][j] = vis ? fmaf(bias, kLog2e, s[n][j] * p.scale_log2) : -INFINITY;
          } else {
            s[n][j] = vis ? s[n][j] * p.scale_log2 : -INFINITY;
          }
          mx[j >> 1] = fmaxf(mx[j >> 1], s[n][j]);
        }
      float alpha[2], base[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m[r], mx[r]);
        base[r] = mn == -INFINITY ? 0.f : mn;
        alpha[r] = fast_exp2(m[r] - base[r]);
        m[r] = mn;
        l[r] *= alpha[r];
      }
      uint32_t pa[4];
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        const float p0 = fast_exp2(s[n][0] - base[0]), p1 = fast_exp2(s[n][1] - base[0]);
        const float p2 = fast_exp2(s[n][2] - base[1]), p3 = fast_exp2(s[n][3] - base[1]);
        l[0] += p0 + p1;
        l[1] += p2 + p3;
        if constexpr (FP8) {
          pa[2 * n] = pack_bf16(p0 * vsc[n][0], p1 * vsc[n][1]);
          pa[2 * n + 1] = pack_bf16(p2 * vsc[n][0], p3 * vsc[n][1]);
        } else {
          pa[2 * n] = pack_bf16(p0, p1);
          pa[2 * n + 1] = pack_bf16(p2, p3);
        }
      }
#pragma unroll
      for (int n = 0; n < D / 8; ++n) {
        o[n][0] *= alpha[0];
        o[n][1] *= alpha[0];
        o[n][2] *= alpha[1];
        o[n][3] *= alpha[1];
      }
#pragma unroll
      for (int j = 0; j < D / 16; ++j) {
        uint32_t bv[4];
        ldsm_x4_t(bv, sv + v_row * C::kRow + j * 16 + v_col);
        mma_bf16(o[2 * j], pa, bv[0], bv[1]);
        mma_bf16(o[2 * j + 1], pa, bv[2], bv[3]);
      }
      if constexpr (!FP8) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
  }
  __syncthreads();   // every stage has been consumed: the ring becomes the merge buffer

  float* mo = reinterpret_cast<float*>(smem);                 // [warp][16][D]
  float* mm = mo + kWarps * kMaxQ * D;                        // [warp][16]
  float* ml = mm + kWarps * kMaxQ;                            // [warp][16]
  if (warp < kWarps) {
    float* w = mo + warp * kMaxQ * D;
#pragma unroll
    for (int n = 0; n < D / 8; ++n) {
      *reinterpret_cast<float2*>(w + r0 * D + n * 8 + c0) = make_float2(o[n][0], o[n][1]);
      *reinterpret_cast<float2*>(w + (r0 + 8) * D + n * 8 + c0) = make_float2(o[n][2], o[n][3]);
    }
    if ((lane & 3) == 0) {
      mm[warp * kMaxQ + r0] = m[0];
      mm[warp * kMaxQ + r0 + 8] = m[1];
      ml[warp * kMaxQ + r0] = l[0];
      ml[warp * kMaxQ + r0 + 8] = l[1];
    }
  }
  __syncthreads();

  const long bg = (long)b * p.G + kvh;
  for (int e = threadIdx.x; e < nrows * D; e += kThreads) {
    const int i = e / D, d = e % D;   // row row0 + i: query head kvh * r + (row0 + i) / Sq, token (row0 + i) % Sq
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) M = fmaxf(M, mm[w * kMaxQ + i]);
    const float base = M == -INFINITY ? 0.f : M;
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const float f = fast_exp2(mm[w * kMaxQ + i] - base);
      L += ml[w * kMaxQ + i] * f;
      O += mo[(w * kMaxQ + i) * D + d] * f;
    }
    if (nsplit == 1) {
      const int row = row0 + i, tok = row % p.Sq;
      const int h = kvh * (p.rows / p.Sq) + row / p.Sq;
      p.o[(((long)b * p.Sq + tok) * p.A + h) * D + d] = __float2bfloat16(L > 0.f ? O / L : 0.f);
    } else {
      const long row = (bg * nsplit + split) * p.rows + row0 + i;
      p.part_o[row * D + d] = O;
      if (d == 0) p.part_ml[row] = make_float2(M, L);
    }
  }
}

// The row of a cache that holds logical row pos of sample b, cache head g: [B, G, C, D] caches, or (PAGED) pools of
// pages [P, G, kTile, D] through the block table [B, max_pages]
template <bool PAGED>
__device__ __forceinline__ size_t cache_row(const int* table, int max_pages, int b, int g, int G, int C, int pos) {
  if constexpr (PAGED)
    return ((size_t)table[(size_t)b * max_pages + pos / kTile] * G + g) * kTile + pos % kTile;
  else
    return ((size_t)b * G + g) * C + pos;
}

// the bf16 cache append (kv_append_kernel, and its paged instances): one thread per (b, i, group, c < D/2).
// RAGGED (paged, B = 1): token i belongs to the sequence n with cu_q[n] <= i < cu_q[n + 1] (nseq sequences, found by
// binary search) and goes to its logical row seqlens[n] + i - cu_q[n] through table row n.
template <bool PAGED, bool RAGGED = false>
__device__ __forceinline__ void kv_append_body(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv,
                                               const float* __restrict__ sinv, __nv_bfloat16* __restrict__ q_out,
                                               __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc,
                                               const int* __restrict__ seqlens, const int* __restrict__ table,
                                               int max_pages, int B, int Sq, int G, int r, int C, int D,
                                               const int* __restrict__ cu_q = nullptr, int nseq = 0) {
  static_assert(!RAGGED || PAGED, "ragged sequences append to pages");
  const int half = D / 2;
  const size_t total = (size_t)B * Sq * G * half;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = static_cast<int>(idx % half);
    const size_t grp = idx / half;               // (b * Sq + i) * G + g
    const int g = static_cast<int>(grp % G);
    const int i = static_cast<int>((grp / G) % Sq);
    const int b = static_cast<int>(grp / ((size_t)G * Sq));
    int seq = b, pos;
    if constexpr (RAGGED) {
      int lo = 0, hi = nseq - 1;   // the last n with cu_q[n] <= i
      while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (cu_q[mid] <= i) lo = mid; else hi = mid - 1;
      }
      seq = lo;
      pos = seqlens[seq] + i - cu_q[seq];
    } else {
      pos = seqlens[b] + i;
    }
    const size_t in = grp * (r + 2) * D;
    const size_t crow = cache_row<PAGED>(table, max_pages, seq, g, G, C, pos) * D;
    RopePair t{1.f, 1.f, 0.f, 0.f};
    if (cosv != nullptr) t = RopePair::load(cosv, sinv, pos, c, D);
    for (int j = 0; j <= r; ++j) {   // slots 0 .. r - 1: q of query head g * r + j; slot r: k
      const size_t src = in + (size_t)j * D;
      const float x1 = __bfloat162float(qkv[src + c]), x2 = __bfloat162float(qkv[src + c + half]);
      const float2 y = cosv != nullptr ? t.rotate(x1, x2, false) : make_float2(x1, x2);
      if (j == r) {
        kc[crow + c] = __float2bfloat16(y.x);
        kc[crow + c + half] = __float2bfloat16(y.y);
      } else if (q_out != nullptr) {
        const size_t qrow = (grp * r + j) * D;    // [B, Sq, A, D] with A = G * r
        q_out[qrow + c] = __float2bfloat16(y.x);
        q_out[qrow + c + half] = __float2bfloat16(y.y);
      }
    }
    vc[crow + c] = qkv[in + (size_t)(r + 1) * D + c];
    vc[crow + c + half] = qkv[in + (size_t)(r + 1) * D + c + half];
  }
}

// IEEE round-to-nearest division, also under --use_fast_math (no flush of subnormals)
__device__ __forceinline__ float div_rn(float a, float b) {
  float r;
  asm("div.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// one row of an FP8 cache: the scale s = amax / 448 (1 for a zero row) and the bytes e4m3_rn_satfinite(x / s) of the
// bf16 values x[p], x[p + 1] (columns lane * 2 + 64 * p' and D / 2 past them, see kv_append_fp8_kernel)
template <int P>
__device__ __forceinline__ void quantize_row(const float (&x)[2 * P], uint8_t* row, float* scale, int lane) {
  float amax = 0.f;
#pragma unroll
  for (int e = 0; e < 2 * P; ++e) amax = fmaxf(amax, fabsf(x[e]));
  amax = warp_max(amax);
  const float s = amax == 0.f ? 1.f : div_rn(amax, 448.f);
#pragma unroll
  for (int e = 0; e < 2 * P; ++e)
    row[(e & 1) * (P * 32) + (e >> 1) * 32 + lane] =
        __nv_cvt_float_to_fp8(div_rn(x[e], s), __NV_SATFINITE, __NV_E4M3);
  if (lane == 0) *scale = s;
}

// the FP8 cache append (kv_append_fp8_kernel, and its paged instances); see kv_append_fp8_kernel.
// RAGGED (paged, B = 1): token i goes to its sequence's row as in kv_append_body's RAGGED instance.
template <int D, bool PAGED, bool RAGGED = false>
__device__ __forceinline__ void kv_append_fp8_body(
    const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv, const float* __restrict__ sinv,
    __nv_bfloat16* __restrict__ q_out, uint8_t* __restrict__ kc, uint8_t* __restrict__ vc, float* __restrict__ ks,
    float* __restrict__ vs, const int* __restrict__ seqlens, const int* __restrict__ table, int max_pages, int B,
    int Sq, int G, int r, int C, const int* __restrict__ cu_q = nullptr, int nseq = 0) {
  static_assert(!RAGGED || PAGED, "ragged sequences append to pages");
  constexpr int half = D / 2, P = half / 32;
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)B * Sq * G;
  const size_t stride = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t grp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; grp < total; grp += stride) {
    const int g = static_cast<int>(grp % G);
    const int i = static_cast<int>((grp / G) % Sq);
    const int b = static_cast<int>(grp / ((size_t)G * Sq));
    int seq = b, pos;
    if constexpr (RAGGED) {
      int lo = 0, hi = nseq - 1;   // the last n with cu_q[n] <= i
      while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (cu_q[mid] <= i) lo = mid; else hi = mid - 1;
      }
      seq = lo;
      pos = seqlens[seq] + i - cu_q[seq];
    } else {
      pos = seqlens[b] + i;
    }
    const size_t in = grp * (r + 2) * D;
    const size_t crow = cache_row<PAGED>(table, max_pages, seq, g, G, C, pos);
    RopePair t[P];
#pragma unroll
    for (int p = 0; p < P; ++p) {
      t[p] = RopePair{1.f, 1.f, 0.f, 0.f};
      if (cosv != nullptr) t[p] = RopePair::load(cosv, sinv, pos, lane + 32 * p, D);
    }
    float kx[2 * P], vx[2 * P];   // the bf16 k and v values of this lane: [2p] column c, [2p + 1] column c + D/2
    for (int j = 0; j <= r; ++j) {   // slots 0 .. r - 1: q of query head g * r + j; slot r: k
      const size_t src = in + (size_t)j * D;
#pragma unroll
      for (int p = 0; p < P; ++p) {
        const int c = lane + 32 * p;
        const float x1 = __bfloat162float(qkv[src + c]), x2 = __bfloat162float(qkv[src + c + half]);
        const float2 y = cosv != nullptr ? t[p].rotate(x1, x2, false) : make_float2(x1, x2);
        if (j == r) {
          kx[2 * p] = __bfloat162float(__float2bfloat16(y.x));
          kx[2 * p + 1] = __bfloat162float(__float2bfloat16(y.y));
        } else if (q_out != nullptr) {
          const size_t qrow = (grp * r + j) * D;
          q_out[qrow + c] = __float2bfloat16(y.x);
          q_out[qrow + c + half] = __float2bfloat16(y.y);
        }
      }
    }
#pragma unroll
    for (int p = 0; p < P; ++p) {
      vx[2 * p] = __bfloat162float(qkv[in + (size_t)(r + 1) * D + lane + 32 * p]);
      vx[2 * p + 1] = __bfloat162float(qkv[in + (size_t)(r + 1) * D + lane + 32 * p + half]);
    }
    quantize_row<P>(kx, kc + crow * D, ks + crow, lane);
    quantize_row<P>(vx, vc + crow * D, vs + crow, lane);
  }
}

template <int D, bool ALIBI>
__global__ void __launch_bounds__(kThreads) decode_attn_kernel(const Params p) {
  decode_attn_body<D, ALIBI ? Score::kAlibi : Score::kNone>(p);
}

// S = kRelBias or kWindow (decode_attention_t5_sm90.cu)
template <int D, Score S>
__global__ void __launch_bounds__(kThreads) decode_attn_t5_kernel(const Params p) {
  decode_attn_body<D, S>(p);
}

template <int D, Score S>
constexpr auto decode_kernel() {
  if constexpr (S == Score::kNone || S == Score::kAlibi)
    return decode_attn_kernel<D, S == Score::kAlibi>;
  else
    return decode_attn_t5_kernel<D, S>;
}

// opts the kernel into its dynamic shared memory once; returns how many of its CTAs one SM holds (0 on error)
template <int D, Score S>
int configure_decode() {
  static int resident = 0;
  if (resident == 0) {
    auto kern = decode_kernel<D, S>();
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<D>::kSmem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, kThreads, Cfg<D>::kSmem) != cudaSuccess)
      resident = 0;
  }
  return resident;
}

// the attention kernel over the (split) key ranges; the partials of nsplit > 1 are reduced by decode_combine_kernel
template <int D, Score S>
cudaError_t launch_decode_attn(const Params& p, int B, int nsplit, cudaStream_t s) {
  if (configure_decode<D, S>() == 0) return cudaErrorInvalidConfiguration;   // the shared memory opt-in failed
  decode_kernel<D, S>()<<<dim3(nsplit, p.G * p.row_blocks, B), kThreads, Cfg<D>::kSmem, s>>>(p);
  return cudaGetLastError();
}

// the ALIBI instances (decode_attention_alibi_sm90.cu); D is 64 or 128
cudaError_t launch_decode_attn_alibi(const Params& p, int D, int B, int nsplit, cudaStream_t s);
// the T5 instances (decode_attention_t5_sm90.cu): S is kRelBias or kWindow, D is 64 or 128
cudaError_t launch_decode_attn_t5(const Params& p, Score S, int D, int B, int nsplit, cudaStream_t s);
// the FP8 instances (decode_attention_fp8_sm90.cu): every score kind, D is 64 or 128
cudaError_t launch_decode_attn_fp8(const Params& p, const float* k_scale, const float* v_scale, Score S, int D, int B,
                                   int nsplit, cudaStream_t s);
// CTAs per SM of the FP8 instances at head dim D (0 when the shared memory opt-in failed)
int decode_fp8_resident(int D);
// the paged instances (decode_attention_paged_sm90.cu): S is kNone or kAlibi, bf16 or (k_scale given) FP8, D 64 or 128
cudaError_t launch_decode_attn_paged(const Params& p, const float* k_scale, const float* v_scale,
                                     const int* block_table, int max_pages, Score S, int D, int B, int nsplit,
                                     cudaStream_t s);

}  // namespace dec
}  // namespace lb
