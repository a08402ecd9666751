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
// Prefix LM (PREFIX instances, causal only, without bias or doc_start): prefix_lens [B] makes the first prefix_lens[b]
// keys visible to every query, so the causal condition becomes j <= i + (Sk - Sq) or j < prefix_lens[b] (GLM: a
// bidirectional context followed by a causal generated part).  A row's key limit is max(i + Sk - Sq + 1, prefix),
// clipped to kv_lens; with a prefix of 0 the instances compute what the causal kernel does, with a prefix >= Sk what
// the non-causal one does, bit for bit.
//
// Packed sequences (DOC instances, causal self-attention only): doc_start [B, S] gives the first key of each query's
// document, so query i of sample b sees key j iff doc_start[b, i] <= j <= i (doc_start clamped to [0, i]: every query
// sees itself).  Nothing assumes doc_start to be non-decreasing along a row: which key tiles a forward CTA loads and
// which (key block, query block) visits the backward skips come from the minimum over the rows of the query block.
//
// Paged K/V (PAGED instances, forward only, causal, no bias or ALiBi, D = 64 and 128): the keys are the logical rows of
// a paged KV cache, read through its block table; each 128-key tile is two 64-row pages (see AttnPages).
//
// Ragged paged K/V (RAGGED instances, attn_fwd_paged_varlen_kernel): N sequences packed along the token axis, each with
// its own rows already held and its own block-table row; one CTA per (128-query tile of a sequence, query head), the
// tiles listed by the host (see AttnRagged).
//
// FP8 ragged paged K/V (RAGGED FP8 instances, attn_fwd_paged_varlen_fp8_kernel): the same over E4M3 pools with fp32 row
// scales; the producer warpgroup dequantizes the pages into the bf16 tiles (see AttnFp8Pages).
//
// Forward, one CTA per (batch, query head, 128-query block), 384 threads:
//   warpgroup 0  TMA producer (one elected thread): Q once, then K/V tiles of 128 keys (double buffered); it gives
//                its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2  consumers, 64 query rows each: S = Q·K_jᵀ (wgmma, accumulators in registers) →
//                online softmax (exp2) in registers → P (bf16) stays in registers as the A operand of O += P·V_j
#include "common.cuh"

#include <cstdlib>
#include <cstring>
#include <type_traits>

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
  const int* prefix_lens;   // [B] in the PREFIX instances: keys below it are visible to every query (last: the older
                            // members keep their offsets)
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
  // the FP8 instances' staging buffer after the barriers: K and V bytes of one key tile, and their scales
  static constexpr int FP8_SMEM_BYTES = SMEM_BYTES + 2 * ATT_BN * D + 2 * ATT_BN * 4;
};

// Paged K/V (PAGED instances, attn_fwd_paged_kernel): the keys are the logical rows [0, Sk) of pools [P, G, 64, D],
// row j of sample b being row j % 64 of page table[b * max_pages + j / 64].  tmap_k / tmap_v cover the pools as
// {D, 64, G, P}; tail_k / tail_v the same pools with only the first Sk % 64 rows of each page (Sk % 64 != 0).
constexpr int ATT_PAGE_ROWS = 64;   // a key tile (ATT_BN) is two pages
struct AttnPages {
  const int* table;   // [B, max_pages]
  int max_pages;
  int num_pages;      // P
};
// The coordinates (row, page) of the box that fills page slot `slot` of sample `batch`, and whether it reads the tail
// map.  A slot at or past the window end, or whose table entry is not a page of the pool, gets a box wholly below the
// page's 64 rows: TMA fills it with zeros, as the contiguous kernel's rows past Sk, reads no memory and still counts the
// box's bytes, so no V row outside the window (uninitialised, or another sequence's, NaN included) reaches P·V.  The
// rows of the last, partial page past Sk read through the tail map, whose row extent ends at Sk % 64, so they are
// zero-filled too.
LB_DEVICE void attn_page_box(const AttnPages& pg, int batch, int slot, int Sk, int& row, int& page, bool& tail) {
  const int rows = Sk - slot * ATT_PAGE_ROWS;
  row = ATT_PAGE_ROWS;
  page = 0;
  tail = false;
  if (rows > 0) {
    const int id = pg.table[static_cast<size_t>(batch) * pg.max_pages + slot];
    if (id >= 0 && id < pg.num_pages) {
      row = 0;
      page = id;
      tail = rows < ATT_PAGE_ROWS;
    }
  }
}

// Ragged paged K/V (RAGGED instances): sequence n owns the query rows cu_q[n] .. cu_q[n + 1] of a packed q [T, A, D]
// and holds past[n] rows before them in block-table row n; its query i sees its logical rows [0, past[n] + i].  A
// tile is (n, 128-query block of n), listed heaviest first by the host, which knows every length.  Each CTA runs the
// paged forward of its sequence alone (Sq = its length, Sk = past + Sq), so its output is that of the PAGED kernel
// called on the sequence by itself, bit for bit.
struct AttnRagged {
  const int* cu_q;    // [N + 1]
  const int* past;    // [N]
  const int2* tiles;  // [n_tiles]: (sequence, query block)
};

// FP8 ragged paged K/V (RAGGED FP8 instances): pools of E4M3 bytes [P, G, 64, D] and fp32 row scales [P, G, 64].  No
// TMA reads them: the producer warpgroup's 128 threads copy a tile's window rows of both pools (cp.async, 16 bytes each)
// and their scales into one staging buffer, then write each element as bf16_rn(float(e) * s) into the K / V tile, laid
// out exactly as the 128B-swizzled TMA box lays out a bf16 page, with zeros for rows at or past the window and for
// pages whose table entry is outside the pool (what the bf16 kernel's tail map and out-of-page boxes load).  So the
// tiles, and the output, are those of the bf16 RAGGED kernel over the dequantized pools, bit for bit.
struct AttnFp8Pages {
  const uint8_t* k;
  const uint8_t* v;
  const float* k_scale;
  const float* v_scale;
  int G;
};
// the rows of page slot `slot` (of a RAGGED sequence, whose table row pg.table is) inside the window [0, Sk), 0 when
// there are none or the entry is outside the pool; `page` its id
LB_DEVICE int attn_page_rows(const AttnPages& pg, int slot, int Sk, int& page) {
  const int rows = Sk - slot * ATT_PAGE_ROWS;
  page = 0;
  if (rows <= 0) return 0;
  const int id = pg.table[slot];
  if (id < 0 || id >= pg.num_pages) return 0;
  page = id;
  return min(rows, ATT_PAGE_ROWS);
}
// shared-memory accesses by shared-space address (smem_u32): the tile pointers are computed through an integer, from
// which the compiler cannot tell the space, and the producer has no registers for generic addressing
LB_DEVICE void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
}
LB_DEVICE void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(dst), "l"(src) : "memory");
}
LB_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
LB_DEVICE void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
LB_DEVICE void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};\n" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
LB_DEVICE void sts32(uint32_t a, uint32_t x) { asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(a), "r"(x) : "memory"); }
LB_DEVICE uint2 lds64(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
  return v;
}
LB_DEVICE float lds32f(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];\n" : "=f"(v) : "r"(a) : "memory");
  return v;
}
// the producer warpgroup's barrier (the consumers' is 1)
LB_DEVICE void producer_sync() { asm volatile("bar.sync 2, 128;\n" ::: "memory"); }
// IEEE round-to-nearest product, also under --use_fast_math (no flush of subnormal products)
LB_DEVICE float mul_rn(float a, float b) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// the two E4M3 bytes of x's low half, dequantized with scale s: bf16_rn(float(e) * s) each, low byte first
LB_DEVICE uint32_t e4m3x2_dequant(uint32_t x, float s) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(x & 0xffffu), __NV_E4M3);
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
  return pack_bf16(mul_rn(f.x, s), mul_rn(f.y, s));
}
// thread t (of 128) stages its part of one pool's key tile j (page slots 2j and 2j + 1 of the sequence's table row)
// into st [128, D] bytes and st_s [128] scales (shared addresses), as one commit group: the window rows' bytes and
// scales by cp.async, zero bytes and a zero scale for every other row (which then dequantize to +0, the bits of TMA's
// zero fill)
template <int D>
LB_DEVICE void fp8_tile_stage(uint32_t st, uint32_t st_s, const uint8_t* pool, const float* scale, const AttnPages& pg,
                              int j, int Sk, int G, int kv_head, int t) {
  constexpr int PIECES = D / 16;   // 16-byte pieces of a row
  int page0, page1;
  const int n0 = attn_page_rows(pg, 2 * j, Sk, page0), n1 = attn_page_rows(pg, 2 * j + 1, Sk, page1);
#pragma unroll 1
  for (int i = 0; i < ATT_BN * PIECES / 128; ++i) {
    const int e = t + 128 * i;
    const int row = e / PIECES, h = row / ATT_PAGE_ROWS, rr = row % ATT_PAGE_ROWS;
    if (rr < (h ? n1 : n0))
      cp_async16(st + e * 16, pool + ((static_cast<size_t>(h ? page1 : page0) * G + kv_head) * ATT_PAGE_ROWS + rr) * D +
                                  (e % PIECES) * 16);
    else
      sts128(st + e * 16, 0u, 0u, 0u, 0u);
  }
  const int h = t / ATT_PAGE_ROWS, rr = t % ATT_PAGE_ROWS;   // thread t: the scale of row t
  if (rr < (h ? n1 : n0))
    cp_async4(st_s + 4 * t, scale + (static_cast<size_t>(h ? page1 : page0) * G + kv_head) * ATT_PAGE_ROWS + rr);
  else
    sts32(st_s + 4 * t, 0u);
  cp_async_commit();
}
// thread t writes its part of the bf16 tile (2 x 64-row pages, CHUNKS 64-column boxes; shared address `tile`) from the
// staged rows, one 16-byte unit (8 columns) at a time
template <int D>
LB_DEVICE void fp8_tile_fill(uint32_t tile, uint32_t st, uint32_t st_s, int t) {
  constexpr int UNITS = D / 8;   // 16-byte bf16 units of a row
#pragma unroll 1
  for (int i = 0; i < ATT_BN * UNITS / 128; ++i) {
    const int e = t + 128 * i;
    const int row = e / UNITS, c = e % UNITS;
    const uint2 x = lds64(st + e * 8);
    const float s = lds32f(st_s + 4 * row);
    // columns 8c .. 8c + 7: unit c % 8 of row `row` of 64-column box c / 8, at its 128B-swizzled place (unit u of
    // row r at u ^ (r % 8))
    sts128(tile + (c / 8) * (ATT_BN * 128) + row * 128 + (((c % 8) ^ (row % 8)) * 16), e4m3x2_dequant(x.x, s),
           e4m3x2_dequant(x.x >> 16, s), e4m3x2_dequant(x.y, s), e4m3x2_dequant(x.y >> 16, s));
  }
}

// the forward of one CTA; tmap_* and p are the kernel's __grid_constant__ parameters (inlined: no call in the kernel).
// PAGED: K/V through the block table `pages` (tail: the maps tail_k, tail_v; see AttnPages); only the producer's
// addresses change, so the shared-memory tiles, and the output, are those of the contiguous kernel over the gathered
// rows [0, Sk).
// RAGGED (with PAGED; see AttnRagged): p, pages are the sequence's own (p.o, p.lse and the table at its rows), q_blk its
// query block and q_row its first row in q.  One tail map cannot end at every sequence's window, so the tail maps are
// the full ones and the last page's rows past Sk arrive as they are in the pool (anything, NaN included).  Their
// scores are masked by assignment, so K needs nothing; V's rows at or past Sk in the window's last tile are zeroed in
// shared memory before P·V (the consumers' generic stores, a proxy fence, then a barrier of the 256 consumer threads),
// so that tile holds what the tail map would have loaded.
// FP8 (with RAGGED; see AttnFp8Pages): K/V come from the FP8 pools `f8`, dequantized by the producer warpgroup; the
// tiles hold zeros past the window, so V needs no zeroing, and tmap_k / tmap_v are not read.
template <int D, int BIAS, bool DROP, bool DOC, bool PREFIX = false, bool PAGED = false, bool RAGGED = false,
          bool FP8 = false>
LB_DEVICE void attn_fwd_cta(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k, const CUtensorMap& tmap_v,
                            const AttnFwdParams& p, const CUtensorMap* tail_k = nullptr,
                            const CUtensorMap* tail_v = nullptr, const AttnPages* pages = nullptr, int rg_blk = 0,
                            int rg_row = 0, const AttnFp8Pages* f8 = nullptr) {
  static_assert(!PAGED || (!DROP && !DOC && !PREFIX && BIAS != BIAS_DENSE), "paged K/V: no dropout, dense bias, "
                "packed sequences or prefix");
  static_assert(!RAGGED || PAGED, "ragged sequences read paged K/V");
  static_assert(!FP8 || RAGGED, "FP8 pools are read by the ragged instances");
  static_assert(!DOC || (BIAS == BIAS_NONE && !DROP), "packed sequences run without bias and dropout");
  static_assert(!PREFIX || (BIAS == BIAS_NONE && !DOC), "a prefix runs without bias and packed sequences");
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
  const int q_blk = RAGGED ? rg_blk : static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);
  const int head = blockIdx.y, batch = RAGGED ? 0 : blockIdx.z;
  const int kv_head = head / p.r;
  const int q0 = q_blk * ATT_BM;
  const int kv_len = p.kv_lens != nullptr ? max(1, min(p.Sk, p.kv_lens[batch])) : p.Sk;
  const int kv_beg = p.kv_start != nullptr ? min(max(p.kv_start[batch], 0), p.Sk) : 0;
  const int off = p.Sk - p.Sq;   // causal offset: query i sees keys j <= i + off
  // keys below `pre` are visible to every row (PREFIX; 0 otherwise)
  const int pre = PREFIX ? min(max(p.prefix_lens[batch], 0), p.Sk) : 0;
  // key tiles j0 .. j0 + nkv - 1 hold every key some row of this block can see; the others are not loaded
  const int key_end = p.causal ? min(kv_len, PREFIX ? max(min(q0 + ATT_BM, p.Sq) + off, pre) : min(q0 + ATT_BM, p.Sq) + off)
                               : kv_len;
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
    if constexpr (FP8) {
      // the TMA producer's 24 registers: the consumers' setmaxnreg.inc to 240 takes exactly the registers the
      // producer warpgroup releases from the kernel's 168 (128 * 24 + 256 * 240 = 168 * 384), so the 128 threads
      // filling tiles must fit in 24 as well
      asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
      if (warp_idx == 0 && elect_one()) {
        mbar_arrive_expect_tx(q_full, Cfg::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < Cfg::CHUNKS; ++c)
          tma_load_5d(sQ + c * (ATT_BM * 128), &tmap_q, q_full, c * 64, rg_row + q0, head - kv_head * p.r, kv_head, 0);
      }
      const int t = threadIdx.x;
      // staging: K bytes [128, D], V bytes [128, D], K scales [128], V scales [128]
      const uint32_t st_k = smem_u32(bars) + 256, st_v = st_k + ATT_BN * D;
      const uint32_t ss_k = st_v + ATT_BN * D, ss_v = ss_k + ATT_BN * 4;
      // each half of the staging buffer is refilled with the next tile as soon as it has been read, so the copies
      // land while the other half is dequantized and the consumers run
      if (nkv > 0) {
        fp8_tile_stage<D>(st_k, ss_k, f8->k, f8->k_scale, *pages, j0, p.Sk, f8->G, kv_head, t);
        fp8_tile_stage<D>(st_v, ss_v, f8->v, f8->v_scale, *pages, j0, p.Sk, f8->G, kv_head, t);
      }
      for (int it = 0; it < nkv; ++it) {
        const int j = j0 + it, b = it & 1;
        const uint32_t par = ((it >> 1) & 1) ^ 1;
        cp_async_wait<1>();   // this thread's K copies (its V copies may be in flight)
        producer_sync();      // everyone's
        mbar_wait(&k_empty[b], par);
        fp8_tile_fill<D>(smem_u32(sK) + b * Cfg::TILE_BYTES, st_k, ss_k, t);
        fence_proxy_async();   // the generic stores, before the wgmma reads the tile through the async proxy
        cp_async_wait<0>();
        producer_sync();       // the K tile written, every V copy landed, the K staging free
        if (t == 0) mbar_arrive(&k_full[b]);
        if (it + 1 < nkv) fp8_tile_stage<D>(st_k, ss_k, f8->k, f8->k_scale, *pages, j + 1, p.Sk, f8->G, kv_head, t);
        mbar_wait(&v_empty[b], par);
        fp8_tile_fill<D>(smem_u32(sV) + b * Cfg::TILE_BYTES, st_v, ss_v, t);
        fence_proxy_async();
        producer_sync();       // the V tile written, the V staging free
        if (t == 0) mbar_arrive(&v_full[b]);
        if (it + 1 < nkv) fp8_tile_stage<D>(st_v, ss_v, f8->v, f8->v_scale, *pages, j + 1, p.Sk, f8->G, kv_head, t);
      }
      return;
    }
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp_idx == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, Cfg::TILE_BYTES);
#pragma unroll
      for (int c = 0; c < Cfg::CHUNKS; ++c)
        tma_load_5d(sQ + c * (ATT_BM * 128), &tmap_q, q_full, c * 64, RAGGED ? rg_row + q0 : q0, head - kv_head * p.r,
                    kv_head, batch);
      for (int it = 0; it < nkv; ++it) {
        const int j = j0 + it, b = it & 1;
        const uint32_t par = ((it >> 1) & 1) ^ 1;
        if constexpr (PAGED) {
          // page slot 2j + h fills rows 64h .. 64h + 63 of the tile: one 64-row box per page and 64-column chunk, at
          // a 1024-byte (8-row) boundary, so the 128B swizzle lays the rows out as one 128-row box does
          int row[2], page[2];
          bool tail[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) attn_page_box(*pages, batch, 2 * j + h, p.Sk, row[h], page[h], tail[h]);
          mbar_wait(&k_empty[b], par);
          mbar_arrive_expect_tx(&k_full[b], Cfg::TILE_BYTES);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < Cfg::CHUNKS; ++c)
              tma_load_4d(sK + b * Cfg::TILE_BYTES + c * (ATT_BN * 128) + h * (ATT_PAGE_ROWS * 128),
                          tail[h] ? tail_k : &tmap_k, &k_full[b], c * 64, row[h], kv_head, page[h]);
          mbar_wait(&v_empty[b], par);
          mbar_arrive_expect_tx(&v_full[b], Cfg::TILE_BYTES);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < Cfg::CHUNKS; ++c)
              tma_load_4d(sV + b * Cfg::TILE_BYTES + c * (ATT_BN * 128) + h * (ATT_PAGE_ROWS * 128),
                          tail[h] ? tail_v : &tmap_v, &v_full[b], c * 64, row[h], kv_head, page[h]);
        } else {
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
    vis_len[h] = max(0, (p.causal ? min(kv_len, PREFIX ? max(q_idx[h] + off + 1, pre) : q_idx[h] + off + 1) : kv_len) -
                            row_beg[h]);
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
    // (PREFIX: a tile inside the prefix is visible to every row whatever the causal bound)
    const bool need_mask = kbase < (DOC ? max(row_beg[0], row_beg[1]) : kv_beg) || kbase + ATT_BN > kv_len ||
                           (p.causal && kbase + ATT_BN - 1 > q0 + off && (!PREFIX || kbase + ATT_BN > pre));
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
    if constexpr (RAGGED && !FP8) {
      // the window's last tile: rows kv_len - kbase .. 127 of every 64-column chunk (the 128B swizzle permutes the
      // 16-byte pieces inside a row, so a chunk's rows from r0 on are one contiguous range)
      const int r0 = kv_len - kbase;
      if (r0 < ATT_BN) {
        for (int c = 0; c < Cfg::CHUNKS; ++c) {
          uint4* z = reinterpret_cast<uint4*>(sV + b * Cfg::TILE_BYTES + c * (ATT_BN * 128) + r0 * 128);
          for (int e = threadIdx.x - 128; e < (ATT_BN - r0) * 8; e += 256) z[e] = make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();   // the generic stores, before the wgmma reads the tile through the async proxy
        asm volatile("bar.sync 1, 256;\n" ::: "memory");
      }
    }
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
// prefix LM (prefix_lens): causal attention without bias, with or without dropout
template <int D, bool DROP>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_prefix_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnFwdParams p) {
  attn_fwd_cta<D, BIAS_NONE, DROP, false, true>(tmap_q, tmap_k, tmap_v, p);
}
// paged K/V (AttnPages): causal attention of the new tokens over a paged cache, without bias or with ALiBi
template <int D, int BIAS>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_paged_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnFwdParams p,
                      const __grid_constant__ CUtensorMap tail_k, const __grid_constant__ CUtensorMap tail_v,
                      const __grid_constant__ AttnPages pages) {
  attn_fwd_cta<D, BIAS, false, false, false, true>(tmap_q, tmap_k, tmap_v, p, &tail_k, &tail_v, &pages);
}
// ragged paged K/V (AttnRagged): the sequences of one packed q, each causal over its own pages, without bias or with
// ALiBi; p holds the shapes shared by every sequence (A, d, r, scale, slopes), p.o [T, A, d] and p.lse [T * A], whose
// sequence n part is [A, Sq_n] at A * cu_q[n]; pages.table is [N, max_pages]
template <int D, int BIAS>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_paged_varlen_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                             const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnFwdParams p,
                             const __grid_constant__ AttnPages pages, const __grid_constant__ AttnRagged rg) {
  const int2 tile = rg.tiles[blockIdx.x];
  const int n = tile.x, row0 = rg.cu_q[n];
  AttnFwdParams sp = p;
  sp.Sq = rg.cu_q[n + 1] - row0;
  sp.Sk = rg.past[n] + sp.Sq;
  sp.o = p.o + static_cast<size_t>(row0) * p.A * p.d;
  sp.lse = p.lse + static_cast<size_t>(row0) * p.A;
  AttnPages pg = pages;
  pg.table = pages.table + static_cast<size_t>(n) * pages.max_pages;
  attn_fwd_cta<D, BIAS, false, false, false, true, true>(tmap_q, tmap_k, tmap_v, sp, &tmap_k, &tmap_v, &pg, tile.y,
                                                         row0);
}
// attn_fwd_paged_varlen_kernel over FP8 pools (AttnFp8Pages): the same tiles, shapes and outputs
template <int D, int BIAS>
__global__ void __launch_bounds__(ATT_FWD_THREADS, 1)
attn_fwd_paged_varlen_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ AttnFwdParams p,
                                 const __grid_constant__ AttnPages pages, const __grid_constant__ AttnRagged rg,
                                 const __grid_constant__ AttnFp8Pages f8) {
  const int2 tile = rg.tiles[blockIdx.x];
  const int n = tile.x, row0 = rg.cu_q[n];
  AttnFwdParams sp = p;
  sp.Sq = rg.cu_q[n + 1] - row0;
  sp.Sk = rg.past[n] + sp.Sq;
  sp.o = p.o + static_cast<size_t>(row0) * p.A * p.d;
  sp.lse = p.lse + static_cast<size_t>(row0) * p.A;
  AttnPages pg = pages;
  pg.table = pages.table + static_cast<size_t>(n) * pages.max_pages;
  attn_fwd_cta<D, BIAS, false, false, false, true, true, true>(tmap_q, tmap_q, tmap_q, sp, nullptr, nullptr, &pg,
                                                               tile.y, row0, &f8);
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

template <int D, int BIAS, bool DROP, bool DOC, bool PREFIX>
cudaError_t launch_fwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const lb::AttnFwdParams& p,
                         cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = DOC ? lb::attn_fwd_doc_kernel<D> : PREFIX ? lb::attn_fwd_prefix_kernel<D, DROP> : lb::attn_fwd_kernel<D, BIAS, DROP>;
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

// the launcher-level conditions both directions share: the tile width (64 or 128) of the head dim, or -1 (head dim),
// -5 (empty sequence), -4 (A % G), -6 (doc_start outside causal self-attention), -7 (prefix_lens without the causal
// mask, or with bias, ALiBi or doc_start), -3 (strides or bias not 16-byte aligned)
int check_attn_args(const lb::AttnArgs& a) {
  const int tile = head_dim_tile(a.d);
  if (tile == 0) return -1;
  if (a.Sq <= 0 || a.Sk <= 0) return -5;
  if (a.G <= 0 || a.A % a.G) return -4;
  if (a.doc_start != nullptr && !lb::attn_doc_start_supported(a)) return -6;
  if (a.prefix_lens != nullptr && !lb::attn_prefix_supported(a)) return -7;
  for (int i = 0; i < 3; ++i)
    if ((a.q_strides[i] % 8) || (a.k_strides[i] % 8) || (a.v_strides[i] % 8)) return -3;
  if (a.q_strides[3] % 8) return -3;
  if (a.bias != nullptr && ((a.bias_strides[0] | a.bias_strides[1] | a.bias_strides[2]) % 8 ||
                            (reinterpret_cast<uintptr_t>(a.bias) & 15)))
    return -3;
  return tile;
}

// the fields AttnFwdParams and AttnBwdParams share (each keeps its own member order: the kernels sit at their register
// limit, so the layout is part of their performance).  `dropout`: a dropout stream is given; a dense bias takes
// precedence over ALiBi slopes.
template <class P>
void fill_score_params(P& p, const lb::AttnArgs& a, bool dropout) {
  p.B = a.B;
  p.A = a.A;
  p.r = a.A / a.G;
  p.Sq = a.Sq;
  p.Sk = a.Sk;
  p.d = a.d;
  p.causal = a.causal;
  p.scale = a.scale;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.kv_lens = a.kv_lens;
  p.kv_start = a.kv_start;
  p.doc_start = a.doc_start;
  p.prefix_lens = a.prefix_lens;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(a.bias);
  for (int i = 0; i < 3; ++i) p.bias_strides[i] = a.bias != nullptr ? a.bias_strides[i] : 0;
  p.alibi_slopes = a.bias != nullptr ? nullptr : a.alibi_slopes;
  // keep a key iff its random byte >= drop_thresh: p quantised to 1/256, a positive p drops at least 1/256
  uint32_t thr = (uint32_t)(a.p_drop * 256.0f + 0.5f);
  if (thr > 255u) thr = 255u;
  p.drop_thresh = (a.p_drop > 0.f && dropout) ? (thr == 0 ? 1u : thr) : 0u;
  p.inv_keep = 256.0f / (256.0f - (float)p.drop_thresh);
}

template <int V>
using int_c = std::integral_constant<int, V>;
template <bool V>
using bool_c = std::integral_constant<bool, V>;
// calls launch(D, BIAS, DROP, DOC, PREFIX) with the compile-time parameters of the kernel instance that runs p: the
// tile width, the bias kind, dropout, packed sequences (whose instances run without bias and dropout) and a prefix
// (whose instances run without bias)
template <class P, class F>
cudaError_t launch_instance(int tile, const P& p, F&& launch) {
  auto with_tile = [&](auto D) {
    if (p.doc_start != nullptr) return launch(D, int_c<lb::BIAS_NONE>{}, bool_c<false>{}, bool_c<true>{}, bool_c<false>{});
    if (p.prefix_lens != nullptr)
      return p.drop_thresh > 0 ? launch(D, int_c<lb::BIAS_NONE>{}, bool_c<true>{}, bool_c<false>{}, bool_c<true>{})
                               : launch(D, int_c<lb::BIAS_NONE>{}, bool_c<false>{}, bool_c<false>{}, bool_c<true>{});
    auto with_bias = [&](auto BIAS) {
      return p.drop_thresh > 0 ? launch(D, BIAS, bool_c<true>{}, bool_c<false>{}, bool_c<false>{})
                               : launch(D, BIAS, bool_c<false>{}, bool_c<false>{}, bool_c<false>{});
    };
    if (p.bias == nullptr && p.alibi_slopes == nullptr) return with_bias(int_c<lb::BIAS_NONE>{});
    if (p.bias != nullptr) return with_bias(int_c<lb::BIAS_DENSE>{});
    return with_bias(int_c<lb::BIAS_ALIBI>{});
  };
  return tile == 64 ? with_tile(int_c<64>{}) : with_tile(int_c<128>{});
}
}  // namespace
// o [B, Sq, A, d], lse [B, A, Sq]; see launchers.h
extern "C" int lb_attn_fwd(const lb::AttnArgs* a, const void* q, const void* k, const void* v, void* o, float* lse,
                           const lb::RngArgs* rng, long long* rng_out, cudaStream_t s) {
  const int tile = check_attn_args(*a);
  if (tile < 0) return tile;
  CUtensorMap tq, tk, tv;
  if (!make_q_tmap(&tq, q, a->B, a->G, a->A / a->G, a->Sq, a->d, a->q_strides, 128)) return -2;
  if (!make_qkv_tmap(&tk, k, a->B, a->G, a->Sk, a->d, a->k_strides, 128)) return -2;
  if (!make_qkv_tmap(&tv, v, a->B, a->G, a->Sk, a->d, a->v_strides, 128)) return -2;
  lb::AttnFwdParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  fill_score_params(p, *a, rng != nullptr);
  memset(&p.rng, 0, sizeof(p.rng));
  if (rng != nullptr) p.rng = *rng;
  p.rng_out = rng_out;
  return (int)launch_instance(tile, p, [&](auto tile_c, auto bias, auto drop, auto doc, auto prefix) {
    return launch_fwd_t<decltype(tile_c)::value, decltype(bias)::value, decltype(drop)::value, decltype(doc)::value,
                        decltype(prefix)::value>(tq, tk, tv, p, s);
  });
}

namespace {
template <int D, int BIAS>
cudaError_t launch_fwd_paged_t(const CUtensorMap (&maps)[5], const lb::AttnFwdParams& p, const lb::AttnPages& pages,
                               cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = lb::attn_fwd_paged_kernel<D, BIAS>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dim3 grid((p.Sq + lb::ATT_BM - 1) / lb::ATT_BM, p.A, p.B);
  kern<<<grid, lb::ATT_FWD_THREADS, Cfg::SMEM_BYTES, s>>>(maps[0], maps[1], maps[2], p, maps[3], maps[4], pages);
  return cudaGetLastError();
}
}  // namespace
// o [B, Sq, A, d], lse [B, A, Sq] over the paged pools [num_pages, G, 64, d]; see launchers.h.  Returns -8 for a problem
// the paged instances do not run (d not 64 or 128, not causal, kv_lens, dense bias, doc_start, prefix_lens, dropout)
// and -9 when the block table has fewer than Sk / 64 slots.
extern "C" int lb_attn_fwd_paged(const lb::AttnArgs* a, const void* q, const void* k_pool, const void* v_pool,
                                 int num_pages, const int* block_table, int max_pages, void* o, float* lse,
                                 cudaStream_t s) {
  const int tile = check_attn_args(*a);
  if (tile < 0) return tile;
  if (a->d != tile || !a->causal || a->kv_lens != nullptr || a->bias != nullptr || a->doc_start != nullptr ||
      a->prefix_lens != nullptr || a->p_drop > 0.f)
    return -8;
  if (num_pages <= 0 || (long)max_pages * lb::ATT_PAGE_ROWS < a->Sk) return -9;
  const int P = lb::ATT_PAGE_ROWS, tail_rows = a->Sk % P == 0 ? P : a->Sk % P;
  const long pool_strides[3] = {(long)a->G * P * a->d, (long)P * a->d, a->d};   // {page, head, row}
  CUtensorMap maps[5];   // q, k, v, tail_k, tail_v
  if (!make_q_tmap(&maps[0], q, a->B, a->G, a->A / a->G, a->Sq, a->d, a->q_strides, 128)) return -2;
  if (!make_qkv_tmap(&maps[1], k_pool, num_pages, a->G, P, a->d, pool_strides, P)) return -2;
  if (!make_qkv_tmap(&maps[2], v_pool, num_pages, a->G, P, a->d, pool_strides, P)) return -2;
  if (!make_qkv_tmap(&maps[3], k_pool, num_pages, a->G, tail_rows, a->d, pool_strides, P)) return -2;
  if (!make_qkv_tmap(&maps[4], v_pool, num_pages, a->G, tail_rows, a->d, pool_strides, P)) return -2;
  lb::AttnFwdParams p;
  fill_score_params(p, *a, false);
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  memset(&p.rng, 0, sizeof(p.rng));
  p.rng_out = nullptr;
  const lb::AttnPages pages{block_table, max_pages, num_pages};
  const bool alibi = p.alibi_slopes != nullptr;
  if (tile == 64)
    return (int)(alibi ? launch_fwd_paged_t<64, lb::BIAS_ALIBI>(maps, p, pages, s)
                       : launch_fwd_paged_t<64, lb::BIAS_NONE>(maps, p, pages, s));
  return (int)(alibi ? launch_fwd_paged_t<128, lb::BIAS_ALIBI>(maps, p, pages, s)
                     : launch_fwd_paged_t<128, lb::BIAS_NONE>(maps, p, pages, s));
}

namespace {
template <int D, int BIAS>
cudaError_t launch_fwd_paged_varlen_t(const CUtensorMap (&maps)[3], const lb::AttnFwdParams& p,
                                      const lb::AttnPages& pages, const lb::AttnRagged& rg, int n_tiles,
                                      cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = lb::attn_fwd_paged_varlen_kernel<D, BIAS>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<dim3(n_tiles, p.A), lb::ATT_FWD_THREADS, Cfg::SMEM_BYTES, s>>>(maps[0], maps[1], maps[2], p, pages, rg);
  return cudaGetLastError();
}
}  // namespace
namespace {
// what both ragged launchers share: the checks of q, the problem and the pool, q's tensor map and the parameters.
// Returns the tile width, 0 when there is nothing to launch, or the launcher's error code.
int varlen_setup(const lb::AttnArgs* a, const void* q, int num_pages, int max_pages, int n_tiles, void* o, float* lse,
                 CUtensorMap& tq, lb::AttnFwdParams& p) {
  lb::AttnArgs full = *a;
  full.Sk = a->Sq;   // check_attn_args looks at the shapes of q; the key windows are per sequence
  const int tile = check_attn_args(full);
  if (tile < 0) return tile;
  if (a->B != 1 || a->d != tile || !a->causal || a->kv_lens != nullptr || a->kv_start != nullptr ||
      a->bias != nullptr || a->doc_start != nullptr || a->prefix_lens != nullptr || a->p_drop > 0.f)
    return -8;
  if (num_pages <= 0 || max_pages <= 0) return -9;
  if (n_tiles == 0) return 0;
  if (!make_q_tmap(&tq, q, 1, a->G, a->A / a->G, a->Sq, a->d, a->q_strides, 128)) return -2;
  fill_score_params(p, full, false);
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  memset(&p.rng, 0, sizeof(p.rng));
  p.rng_out = nullptr;
  return tile;
}
}  // namespace
// o [T, A, d] and lse [T * A] of the N ragged sequences of q [T, A, d] (a->B = 1, a->Sq = T) over the paged pools
// [num_pages, G, 64, d]; see launchers.h.  Returns -8 for a problem the paged instances do not run (as
// lb_attn_fwd_paged, kv_start included) and -9 for an empty pool or table.
extern "C" int lb_attn_fwd_paged_varlen(const lb::AttnArgs* a, const void* q, const void* k_pool, const void* v_pool,
                                        int num_pages, const int* block_table, int max_pages, const int* cu_q,
                                        const int* past, const int* tiles, int n_tiles, void* o, float* lse,
                                        cudaStream_t s) {
  CUtensorMap maps[3];   // q, k, v
  lb::AttnFwdParams p;
  const int tile = varlen_setup(a, q, num_pages, max_pages, n_tiles, o, lse, maps[0], p);
  if (tile <= 0) return tile;
  const int P = lb::ATT_PAGE_ROWS;
  const long pool_strides[3] = {(long)a->G * P * a->d, (long)P * a->d, a->d};   // {page, head, row}
  if (!make_qkv_tmap(&maps[1], k_pool, num_pages, a->G, P, a->d, pool_strides, P)) return -2;
  if (!make_qkv_tmap(&maps[2], v_pool, num_pages, a->G, P, a->d, pool_strides, P)) return -2;
  const lb::AttnPages pages{block_table, max_pages, num_pages};
  const lb::AttnRagged rg{cu_q, past, reinterpret_cast<const int2*>(tiles)};
  const bool alibi = p.alibi_slopes != nullptr;
  if (tile == 64)
    return (int)(alibi ? launch_fwd_paged_varlen_t<64, lb::BIAS_ALIBI>(maps, p, pages, rg, n_tiles, s)
                       : launch_fwd_paged_varlen_t<64, lb::BIAS_NONE>(maps, p, pages, rg, n_tiles, s));
  return (int)(alibi ? launch_fwd_paged_varlen_t<128, lb::BIAS_ALIBI>(maps, p, pages, rg, n_tiles, s)
                     : launch_fwd_paged_varlen_t<128, lb::BIAS_NONE>(maps, p, pages, rg, n_tiles, s));
}

namespace {
template <int D, int BIAS>
cudaError_t launch_fwd_paged_varlen_fp8_t(const CUtensorMap& tq, const lb::AttnFwdParams& p,
                                          const lb::AttnPages& pages, const lb::AttnRagged& rg,
                                          const lb::AttnFp8Pages& f8, int n_tiles, cudaStream_t s) {
  using Cfg = lb::AttnFwdCfg<D>;
  auto kern = lb::attn_fwd_paged_varlen_fp8_kernel<D, BIAS>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::FP8_SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<dim3(n_tiles, p.A), lb::ATT_FWD_THREADS, Cfg::FP8_SMEM_BYTES, s>>>(tq, p, pages, rg, f8);
  return cudaGetLastError();
}
}  // namespace
// lb_attn_fwd_paged_varlen over FP8 pools; see launchers.h.  Returns the codes of lb_attn_fwd_paged_varlen, and -3
// for pools or scales not 16-byte aligned.
extern "C" int lb_attn_fwd_paged_varlen_fp8(const lb::AttnArgs* a, const void* q, const void* k_pool,
                                            const void* v_pool, const float* k_scale, const float* v_scale,
                                            int num_pages, const int* block_table, int max_pages, const int* cu_q,
                                            const int* past, const int* tiles, int n_tiles, void* o, float* lse,
                                            cudaStream_t s) {
  if (((reinterpret_cast<uintptr_t>(k_pool) | reinterpret_cast<uintptr_t>(v_pool) |
        reinterpret_cast<uintptr_t>(k_scale) | reinterpret_cast<uintptr_t>(v_scale)) & 15))
    return -3;
  CUtensorMap tq;
  lb::AttnFwdParams p;
  const int tile = varlen_setup(a, q, num_pages, max_pages, n_tiles, o, lse, tq, p);
  if (tile <= 0) return tile;
  const lb::AttnPages pages{block_table, max_pages, num_pages};
  const lb::AttnRagged rg{cu_q, past, reinterpret_cast<const int2*>(tiles)};
  const lb::AttnFp8Pages f8{static_cast<const uint8_t*>(k_pool), static_cast<const uint8_t*>(v_pool), k_scale, v_scale,
                            a->G};
  const bool alibi = p.alibi_slopes != nullptr;
  if (tile == 64)
    return (int)(alibi ? launch_fwd_paged_varlen_fp8_t<64, lb::BIAS_ALIBI>(tq, p, pages, rg, f8, n_tiles, s)
                       : launch_fwd_paged_varlen_fp8_t<64, lb::BIAS_NONE>(tq, p, pages, rg, f8, n_tiles, s));
  return (int)(alibi ? launch_fwd_paged_varlen_fp8_t<128, lb::BIAS_ALIBI>(tq, p, pages, rg, f8, n_tiles, s)
                     : launch_fwd_paged_varlen_fp8_t<128, lb::BIAS_NONE>(tq, p, pages, rg, f8, n_tiles, s));
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
// Prefix LM (PREFIX): query block i and key block kb of sample b meet iff 64 kb <= 64 i + 63 + (Sk - Sq) or
// 64 kb < prefix_lens[b] (the shapes and that one number per sample).  A key block inside the prefix meets every query
// block, so a CTA whose lowest key block lies in the prefix starts its visits at query block 0.  Meeting stays monotone
// in the key block (if kb meets i, every lower key block does), so the dQ counter rule below keeps its form: key block
// kb adds to query block i after exactly last_kb - kb additions, where last_kb = min(nkb - 1, max(the causal last
// block (64 i + 63 + Sk - Sq) / 64, ceil(min(prefix_lens[b], Sk) / 64) - 1)).  Keys outside kv_start / kv_lens stay
// masked element-wise, with every visit made.  Forward progress rests on the same dispatch-order assumption as
// without a prefix (below): a waiter only waits for higher key blocks, which live in its own CTA or in CTAs of lower
// linear index.
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
  const int* prefix_lens;    // [B] in the PREFIX instances (last: the older members keep their offsets)
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
// 64 kb <= Sk - 1.  PREFIX: 0 for a key block that starts inside the prefix `pre` (every query sees it).
template <bool PREFIX>
LB_DEVICE int bwd_first_qblock(const AttnBwdParams& p, int kb, int pre) {
  if (PREFIX && kb * ATT_BWD_BN < pre) return 0;
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
template <bool DOC, bool PREFIX>
LB_DEVICE bool bwd_visits(const AttnBwdParams& p, int batch, int nkb, int kb, int qb, int pre) {
  if (kb >= nkb || qb < bwd_first_qblock<PREFIX>(p, kb, pre)) return false;
  return !DOC || !doc_visit_empty(p.doc_start, p.Sq, batch, qb * ATT_BWD_BM, kb * ATT_BWD_BN);
}

// the backward of one CTA; the tensor maps and p are the kernel's parameters (inlined: no call in the kernel)
template <int D, int BIAS, bool DROP, bool DOC, bool PREFIX>
LB_DEVICE void attn_bwd_cta(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k, const CUtensorMap& tmap_v,
                            const CUtensorMap& tmap_do, const AttnBwdParams& p) {
  static_assert(!DOC || (BIAS == BIAS_NONE && !DROP), "packed sequences run without bias and dropout");
  static_assert(!PREFIX || (BIAS == BIAS_NONE && !DOC), "a prefix runs without bias and packed sequences");
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
  const int pre = PREFIX ? min(max(p.prefix_lens[batch], 0), p.Sk) : 0;   // keys every query sees
  const int i_begin = bwd_first_qblock<PREFIX>(p, kb0, pre);
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
        for (int w = 0; w < NWG; ++w) need = need || bwd_visits<DOC, PREFIX>(p, batch, nkb, kb0 + w, qb, pre);
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
        for (int w = 0; w < NWG; ++w) makes[w] = bwd_visits<DOC, PREFIX>(p, batch, nkb, kb0 + w, qb, pre);
        if (lane == 0) {
          const size_t blk = (static_cast<size_t>(batch) * p.A + kv_head * p.r + hi) * nq + qb;
          unsigned* order = p.dq_order + blk;
          // the key blocks above kb that visit query block qb: all of them, or under the causal mask
          // kb' <= (64 qb + 63 + off) / 64 (a non-negative quotient, since kb visits qb) or, with a prefix, the blocks
          // that start inside it
          int last_kb = p.causal ? min(nkb - 1, (qb * ATT_BWD_BM + ATT_BWD_BM - 1 + off) / ATT_BWD_BN) : nkb - 1;
          if (PREFIX && p.causal) last_kb = min(nkb - 1, max(last_kb, (pre + ATT_BWD_BN - 1) / ATT_BWD_BN - 1));
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
    const bool mine = bwd_visits<DOC, PREFIX>(p, batch, nkb, kb, qb, pre);
    bool need = mine;
#pragma unroll
    for (int u = 0; u < NWG; ++u)
      if (u != w) need = need || bwd_visits<DOC, PREFIX>(p, batch, nkb, kb0 + u, qb, pre);
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
          const int key_lim = !q_ok ? 0 : (p.causal ? min(kv_len, PREFIX ? max(q_idx + off + 1, pre) : q_idx + off + 1) : kv_len);
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

template <int D, int BIAS, bool DROP, bool DOC>
__global__ void __launch_bounds__(AttnBwdCfg<D, attn_bwd_wgs<D, BIAS, DROP>()>::THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do, AttnBwdParams p) {
  attn_bwd_cta<D, BIAS, DROP, DOC, false>(tmap_q, tmap_k, tmap_v, tmap_do, p);
}
// prefix LM (prefix_lens): causal attention without bias, with or without dropout
template <int D, bool DROP>
__global__ void __launch_bounds__(AttnBwdCfg<D, attn_bwd_wgs<D, BIAS_NONE, DROP>()>::THREADS, 1)
attn_bwd_prefix_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                       AttnBwdParams p) {
  attn_bwd_cta<D, BIAS_NONE, DROP, false, true>(tmap_q, tmap_k, tmap_v, tmap_do, p);
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
template <int D, int BIAS, bool DROP, bool DOC, bool PREFIX>
cudaError_t launch_bwd_t(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                         const lb::AttnBwdParams& p, cudaStream_t s) {
  constexpr int NWG = lb::attn_bwd_wgs<D, BIAS, DROP>();
  using Cfg = lb::AttnBwdCfg<D, NWG>;
  auto kern = PREFIX ? lb::attn_bwd_prefix_kernel<D, DROP> : lb::attn_bwd_kernel<D, BIAS, DROP, DOC>;
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
}  // namespace
// floats of the backward's dQ accumulator (fp32 [64][tile] per batch, query head and 64-query block)
extern "C" long lb_attn_bwd_accum_floats(int B, int A, int Sq, int D) {
  return (long)B * A * ((Sq + lb::ATT_BWD_BM - 1) / lb::ATT_BWD_BM) * lb::ATT_BWD_BM * head_dim_tile(D);
}
// see launchers.h; for Sq == Sk the caller passes views of one packed [B, S, G, r + 2, D] gradient as dq, dk and dv
extern "C" int lb_attn_bwd(const lb::AttnArgs* a, const void* dout, const long* do_strides, const void* q, const void* k,
                           const void* v, const void* o, const float* lse, void* dq, void* dk, void* dv,
                           const long* dq_strides, const long* dkv_strides, float* delta, float* dq_accum, float* dbias,
                           const long long* rng_state, unsigned* dq_order, cudaStream_t s) {
  const int tile = check_attn_args(*a);
  if (tile < 0) return tile;
  const int B = a->B, A = a->A, G = a->G, Sq = a->Sq, Sk = a->Sk, D = a->d, r = A / G;
  for (int i = 0; i < 3; ++i)
    if (do_strides[i] % 8) return -3;
  const long do_strides4[4] = {do_strides[0], r * do_strides[1], do_strides[1], do_strides[2]};
  CUtensorMap tq, tk, tv, tdo;
  if (!make_q_tmap(&tq, q, B, G, r, Sq, D, a->q_strides, 64)) return -2;
  if (!make_qkv_tmap(&tk, k, B, G, Sk, D, a->k_strides, 64)) return -2;
  if (!make_qkv_tmap(&tv, v, B, G, Sk, D, a->v_strides, 64)) return -2;
  if (!make_q_tmap(&tdo, dout, B, G, r, Sq, D, do_strides4, 64)) return -2;
  const long rows = (long)B * A * Sq;
  {
    // 4 rows per thread-group and iteration; cap the grid at a few waves
    const long groups = (rows + 3) / 4;
    const long lpr = tile / 8;
    long blocks = (groups * lpr + 255) / 256;
    if (blocks > lb_host::num_sms() * 16L) blocks = lb_host::num_sms() * 16L;
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
  fill_score_params(p, *a, rng_state != nullptr);
  p.dbias = a->bias != nullptr ? dbias : nullptr;
  p.rng_state = rng_state;
  p.dq_order = dq_order;
  p.timeout_rec = lb_host::spin_timeout_record(s);
  cudaError_t e = launch_instance(tile, p, [&](auto tile_c, auto bias, auto drop, auto doc, auto prefix) {
    return launch_bwd_t<decltype(tile_c)::value, decltype(bias)::value, decltype(drop)::value, decltype(doc)::value,
                        decltype(prefix)::value>(tq, tk, tv, tdo, p, s);
  });
  if (e != cudaSuccess) return (int)e;
  const long nvec = rows * D / 8;
  int blocks = (int)((nvec + 511) / 512);
  if (blocks > lb_host::num_sms() * 8) blocks = lb_host::num_sms() * 8;
  auto convert = tile == 64 ? lb::attn_dq_convert_kernel<64> : lb::attn_dq_convert_kernel<128>;
  convert<<<blocks, 256, 0, s>>>(dq_accum, (__nv_bfloat16*)dq, B, A, Sq, D, r, dq_strides[0], dq_strides[1],
                                 dq_strides[2], dq_strides[3]);
  return (int)cudaGetLastError();
}
