// KV-cache decoding on sm_90a: the cache append (with rotary embedding) and split-KV ("flash-decoding") attention.
//
// Grouped-query attention: the A query heads share G = A / r cache heads.  The packed projection is grouped,
// [B, Sq, G, r + 2, D] with q_0 .. q_{r-1}, k, v per group (r = 1: per-head [q|k|v]), and the caches hold the G heads.
//
// lb_kv_append: one pass over the packed projection.  q and k are rotated with the fp32 cos/sin tables in the
//   rotate-half convention of rope_qkv_kernel (same expressions, so the rotated values are bit-identical), k and v are
//   written into the layer's cache K, V [B, G, C, D] at rows cache_seqlens[b] + i, and the rotated q goes to
//   q_out [B, Sq, A, D].  Without tables (GPT-2) the values are copied unrotated.
//
// lb_decode_attn: o [B, Sq, A, D] for 1 <= Sq <= 16 new queries per (sample, head).  Query i of sample b sees exactly the
//   keys j with kv_start[b] <= j <= cache_seqlens[b] + i (kv_start = left padding, cache_seqlens = length before this
//   step's append); every other key is excluded outright, and a query without a visible key writes zeros.
//   The MMA rows of a CTA are (query head in group, new token) pairs of one cache head: row = j * Sq + i for query head
//   g * r + j and token i, r * Sq rows cut into blocks of 16.  A group with r * Sq <= 16 therefore reads each K/V tile
//   once for all its query heads.
//   Grid (splits, G * row blocks, B), 160 threads: the key window of each (b, g) is cut into `splits` contiguous ranges
//   of 64-key tiles so that small batches still fill the SMs.  Warp 4 streams the K/V tiles of its range through a ring of
//   shared-memory stages with cp.async.bulk (one bulk copy per key row, into rows padded by 16 bytes so the ldmatrix
//   reads below are free of bank conflicts; the non-tensor bulk copy has no swizzle), completion on mbarriers.  Warps
//   0-3 each take 16 keys of every tile: S = Q·Kᵀ and O += P·V on mma.sync m16n8k16 (bf16 in, fp32 accumulators), the
//   16 rows of the MMA being (query head, new token) pairs, and keep their own online-softmax state.  The four warps are
//   merged in warp order in shared memory; with one split that is the output, otherwise the CTA writes its fp32 partial
//   (m, l, O) and decode_combine_kernel reduces the partials in split order.  No atomics: results are bit-identical from
//   run to run.
//   mma.sync rather than wgmma: the kernel moves ~2 bytes of K/V per multiply-add, so it is bound by HBM bandwidth, not
//   by the tensor cores; wgmma's 64-row minimum M would be 4-64x wasted work for Sq <= 16 and would need swizzled
//   (TMA tensor-map) tiles, while mma.sync's M = 16 matches Sq exactly and reads plain row-major tiles.
//   Lengths are read on the device and the grid depends only on (B, G, r, Sq, splits): one captured launch replays correctly
//   after cache_seqlens has been bumped on the device.
//   Known limit (docs/source/tutorials/get_started/Benchmark.md, "Decoding"): at large batches the kernel tops out near
//   the same rate of key rows per second at both head dims (about 2.1 TB/s at 128, 1.0 TB/s at 64 on an H100), which
//   points to the one bulk copy per row, not to HBM (not confirmed with a profiler).  Whole-tile TMA tensor-map loads
//   with a 128-byte swizzle (and the matching XOR in the ldmatrix addresses) are the planned change.
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
};

LB_DEVICE void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
template <int D>
__global__ void __launch_bounds__(kThreads) decode_attn_kernel(const Params p) {
  using C = Cfg<D>;
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
  const int hi = min(len + p.Sq, p.C);   // exclusive; the cache object keeps len + Sq <= C, this only guards memory
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
        bulk_load(sk + r * C::kRow, kg + row * D, D * 2, &full[st]);
        bulk_load(sv + r * C::kRow, vg + row * D, D * 2, &full[st]);
      }
    }
  } else if (my > 0) {
    // Q fragments (A operand, rows = (query head, new token) pairs; rows past the last pair are zero), loaded once.
    // lim: the last visible key of each of this thread's two rows (causal among the new tokens)
    uint32_t qf[D / 16][4];
    int lim[2];
    {
      const int hr = kvh * (p.rows / p.Sq);   // first query head of the group
      const bool v0 = r0 < nrows, v1 = r0 + 8 < nrows;
      const int t0 = (row0 + r0) % p.Sq, t1 = (row0 + r0 + 8) % p.Sq;
      lim[0] = len + t0;
      lim[1] = len + t1;
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
    // ldmatrix lane addresses: K (non-transposed: keys = rows of the B fragment), V (transposed)
    const int k_row = kw + (lane & 7) + ((lane >> 4) << 3), k_col = ((lane >> 3) & 1) * 8;
    const int v_row = kw + (lane & 7) + (((lane >> 3) & 1) << 3), v_col = (lane >> 4) * 8;
    for (int t = 0; t < my; ++t) {
      const int st = t % C::kStages;
      mbar_wait(&full[st], (t / C::kStages) & 1);
      const __nv_bfloat16* sk = ring + st * C::kStageElems;
      const __nv_bfloat16* sv = sk + kTile * C::kRow;
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
          s[n][j] = vis ? s[n][j] * p.scale_log2 : -INFINITY;
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
        pa[2 * n] = pack_bf16(p0, p1);
        pa[2 * n + 1] = pack_bf16(p2, p3);
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
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
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

// o[b, i, h, :] from the per-split partials, summed in split order; one CTA per (cache head, row block, sample)
template <int D>
__global__ void __launch_bounds__(128) decode_combine_kernel(const Params p, int nsplit) {
  const int b = blockIdx.y;
  const int kvh = blockIdx.x / p.row_blocks;
  const int row0 = (blockIdx.x - kvh * p.row_blocks) * kMaxQ;
  const int nrows = min(kMaxQ, p.rows - row0);
  const long bg = (long)b * p.G + kvh;
  for (int e = threadIdx.x; e < nrows * D; e += blockDim.x) {
    const int i = row0 + e / D, d = e % D;
    float M = -INFINITY;
    for (int s = 0; s < nsplit; ++s) M = fmaxf(M, p.part_ml[(bg * nsplit + s) * p.rows + i].x);
    const float base = M == -INFINITY ? 0.f : M;
    float L = 0.f, O = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const long row = (bg * nsplit + s) * p.rows + i;
      const float2 ml = p.part_ml[row];
      const float f = fast_exp2(ml.x - base);
      L += ml.y * f;
      O += p.part_o[row * D + d] * f;
    }
    const int h = kvh * (p.rows / p.Sq) + i / p.Sq;
    p.o[(((long)b * p.Sq + i % p.Sq) * p.A + h) * D + d] = __float2bfloat16(L > 0.f ? O / L : 0.f);
  }
}

// one thread per (b, i, group, c < D/2): the r q pairs and the k pair (c, c + D/2) rotated exactly like rope_qkv_kernel,
// v copied
__global__ void kv_append_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv,
                                 const float* __restrict__ sinv, __nv_bfloat16* __restrict__ q_out,
                                 __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc,
                                 const int* __restrict__ seqlens, int B, int Sq, int G, int r, int C, int D) {
  const int half = D / 2;
  const size_t total = (size_t)B * Sq * G * half;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = static_cast<int>(idx % half);
    const size_t grp = idx / half;               // (b * Sq + i) * G + g
    const int g = static_cast<int>(grp % G);
    const int i = static_cast<int>((grp / G) % Sq);
    const int b = static_cast<int>(grp / ((size_t)G * Sq));
    const int pos = seqlens[b] + i;
    const size_t in = grp * (r + 2) * D;
    const size_t crow = (((size_t)b * G + g) * C + pos) * D;
    float c1 = 1.f, c2 = 1.f, s1 = 0.f, s2 = 0.f;
    if (cosv != nullptr) {
      c1 = cosv[pos * D + c], c2 = cosv[pos * D + c + half];
      s1 = sinv[pos * D + c], s2 = sinv[pos * D + c + half];
    }
    for (int j = 0; j <= r; ++j) {   // slots 0 .. r - 1: q of query head g * r + j; slot r: k
      const size_t src = in + (size_t)j * D;
      const float x1 = __bfloat162float(qkv[src + c]), x2 = __bfloat162float(qkv[src + c + half]);
      float y1 = x1, y2 = x2;
      if (cosv != nullptr) {
        y1 = x1 * c1 - x2 * s1;
        y2 = x2 * c2 + x1 * s2;
      }
      if (j == r) {
        kc[crow + c] = __float2bfloat16(y1);
        kc[crow + c + half] = __float2bfloat16(y2);
      } else if (q_out != nullptr) {
        const size_t qrow = (grp * r + j) * D;    // [B, Sq, A, D] with A = G * r
        q_out[qrow + c] = __float2bfloat16(y1);
        q_out[qrow + c + half] = __float2bfloat16(y2);
      }
    }
    vc[crow + c] = qkv[in + (size_t)(r + 1) * D + c];
    vc[crow + c + half] = qkv[in + (size_t)(r + 1) * D + c + half];
  }
}

}  // namespace dec
}  // namespace lb

namespace {
// opts the kernel into its dynamic shared memory once; returns how many of its CTAs one SM holds (0 on error)
template <int D>
int configure_decode() {
  static int resident = 0;
  if (resident == 0) {
    using Cfg = lb::dec::Cfg<D>;
    auto kern = lb::dec::decode_attn_kernel<D>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, lb::dec::kThreads, Cfg::kSmem) != cudaSuccess)
      resident = 0;
  }
  return resident;
}

template <int D>
cudaError_t launch_decode(const lb::dec::Params& p, int B, int nsplit, cudaStream_t s) {
  using Cfg = lb::dec::Cfg<D>;
  auto kern = lb::dec::decode_attn_kernel<D>;
  if (configure_decode<D>() == 0) return cudaErrorInvalidConfiguration;   // the shared memory opt-in failed
  kern<<<dim3(nsplit, p.G * p.row_blocks, B), lb::dec::kThreads, Cfg::kSmem, s>>>(p);
  if (nsplit > 1) lb::dec::decode_combine_kernel<D><<<dim3(p.G * p.row_blocks, B), 128, 0, s>>>(p, nsplit);
  return cudaGetLastError();
}
}  // namespace

// Number of key-range splits per (sample, cache head, row block): as many as fill the resident CTA slots of the GPU in
// one wave (a second, partial wave would only add a tail), at most one split per 128 keys of the capacity.  `blocks` =
// G * ceil(r * Sq / 16) CTAs per sample and split.  Depends on the shapes only, never on the current lengths.
extern "C" int lb_decode_splits(int B, int blocks, int C, int D) {
  const int resident = D == 64 ? configure_decode<64>() : configure_decode<128>();
  int n = lb_host::num_sms() * (resident > 0 ? resident : 1) / (B * blocks);
  n = n < (C + 127) / 128 ? n : (C + 127) / 128;
  n = n < lb::dec::kMaxSplits ? n : lb::dec::kMaxSplits;
  return n > 1 ? n : 1;
}

extern "C" int lb_decode_attn(const void* q, const long* q_strides, const void* k, const void* v, void* o,
                              float* part_o, float* part_ml, const int* seqlens, const int* kv_start, int B, int Sq,
                              int A, int G, int C, int D, float scale, int nsplit, cudaStream_t s) {
  if (B == 0 || A == 0) return 0;
  if (G <= 0 || A % G) return -4;
  lb::dec::Params p;
  p.q = static_cast<const __nv_bfloat16*>(q);
  p.q_sb = q_strides[0];
  p.q_si = q_strides[1];
  p.q_sh = q_strides[2];
  p.k = static_cast<const __nv_bfloat16*>(k);
  p.v = static_cast<const __nv_bfloat16*>(v);
  p.o = static_cast<__nv_bfloat16*>(o);
  p.part_o = part_o;
  p.part_ml = reinterpret_cast<float2*>(part_ml);
  p.seqlens = seqlens;
  p.kv_start = kv_start;
  p.A = A;
  p.G = G;
  p.C = C;
  p.Sq = Sq;
  p.rows = (A / G) * Sq;
  p.row_blocks = (p.rows + lb::dec::kMaxQ - 1) / lb::dec::kMaxQ;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaError_t e = D == 64 ? launch_decode<64>(p, B, nsplit, s) : launch_decode<128>(p, B, nsplit, s);
  return (int)e;
}

extern "C" int lb_kv_append(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_cache,
                            void* v_cache, const int* seqlens, int B, int Sq, int G, int r, int C, int D, cudaStream_t s) {
  const size_t total = (size_t)B * Sq * G * (D / 2);
  if (total == 0) return 0;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < 4096 ? (total + threads - 1) / threads : 4096);
  lb::dec::kv_append_kernel<<<blocks, threads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(qkv), cosv, sinv, static_cast<__nv_bfloat16*>(q_out),
      static_cast<__nv_bfloat16*>(k_cache), static_cast<__nv_bfloat16*>(v_cache), seqlens, B, Sq, G, r, C, D);
  return (int)cudaGetLastError();
}
