// KV-cache decoding on sm_90a: the cache append (with rotary embedding) and split-KV ("flash-decoding") attention.
//
// Grouped-query attention: the A query heads share G = A / r cache heads.  The packed projection is grouped,
// [B, Sq, G, r + 2, D] with q_0 .. q_{r-1}, k, v per group (r = 1: per-head [q|k|v]), and the caches hold the G heads.
//
// lb_kv_append: one pass over the packed projection.  q and k are rotated with the fp32 cos/sin tables in the
//   rotate-half convention (RopePair, as rope_qkv_kernel rotates them), k and v are written into the layer's cache
//   K, V [B, G, C, D] at rows cache_seqlens[b] + i, and the rotated q goes to q_out [B, Sq, A, D].  Without tables
//   (GPT-2) the values are copied unrotated.
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
//   ALiBi (BLOOM): with alibi_slopes (fp32 [A]) every visible score gets slope_h·(j − (cache_seqlens[b] + i)), which is
//   the flash kernel's slope·(j − i − (Sk − Sq)) with Sk = cache_seqlens[b] + Sq, so a continuation scores the same
//   through either kernel.
//   T5 (decode_attention_t5_sm90.cu): with rel_bias (fp32 [A, R]) every visible score gets
//   rel_bias[h, min(cache_seqlens[b] + i − j, R − 1)], T5's unidirectional bucketed relative-position bias, which is
//   constant past max_distance; with causal = false (cross-attention) every new token sees kv_start[b] <= j <
//   cache_seqlens[b], the new tokens not being in that cache.
//   The kernel template lives in decode_attention_sm90.cuh; its ALiBi instances are compiled in
//   decode_attention_alibi_sm90.cu and its T5 instances in decode_attention_t5_sm90.cu.
//   Paged caches (decode_attention_paged_sm90.cu, with their appends): pools of 64-row pages and a block table per
//   sample; the same tiles, so the same output bit for bit.
//   FP8 (E4M3) caches (decode_attention_fp8_sm90.cu, with their quantizing append): K, V bytes with one fp32 scale per
//   row; every score kind at both head dims, one bulk copy per tile and array, the scales folded into the scores and
//   probabilities (Cfg8 and decode_attn_body in decode_attention_sm90.cuh).
//   Known limit (docs/source/tutorials/get_started/Benchmark.md, "Decoding"): at large batches the kernel tops out near
//   the same rate of key rows per second at both head dims (about 2.1 TB/s at 128, 1.0 TB/s at 64 on an H100), which
//   points to the one bulk copy per row, not to HBM (not confirmed with a profiler).  Whole-tile TMA tensor-map loads
//   with a 128-byte swizzle (and the matching XOR in the ldmatrix addresses) are the planned change.
#include "decode_attention_sm90.cuh"

namespace lb {
namespace dec {

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

// one thread per (b, i, group, c < D/2): the r q pairs and the k pair (c, c + D/2) rotated (RopePair), v copied
__global__ void kv_append_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv,
                                 const float* __restrict__ sinv, __nv_bfloat16* __restrict__ q_out,
                                 __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc,
                                 const int* __restrict__ seqlens, int B, int Sq, int G, int r, int C, int D) {
  kv_append_body<false>(qkv, cosv, sinv, q_out, kc, vc, seqlens, nullptr, 0, B, Sq, G, r, C, D);
}

}  // namespace dec
}  // namespace lb

namespace {
template <int D>
cudaError_t launch_decode(const lb::dec::Params& p, const float* k_scale, const float* v_scale, const int* block_table,
                          int max_pages, int B, int nsplit, lb::dec::Score score, cudaStream_t s) {
  using lb::dec::Score;
  cudaError_t e = block_table != nullptr ? lb::dec::launch_decode_attn_paged(p, k_scale, v_scale, block_table,
                                                                             max_pages, score, D, B, nsplit, s)
                  : k_scale != nullptr     ? lb::dec::launch_decode_attn_fp8(p, k_scale, v_scale, score, D, B, nsplit, s)
                  : score == Score::kAlibi ? lb::dec::launch_decode_attn_alibi(p, D, B, nsplit, s)
                  : score == Score::kNone  ? lb::dec::launch_decode_attn<D, Score::kNone>(p, B, nsplit, s)
                                           : lb::dec::launch_decode_attn_t5(p, score, D, B, nsplit, s);
  if (e != cudaSuccess) return e;
  if (nsplit > 1) lb::dec::decode_combine_kernel<D><<<dim3(p.G * p.row_blocks, B), 128, 0, s>>>(p, nsplit);
  return cudaGetLastError();
}
}  // namespace

// Number of key-range splits per (sample, cache head, row block): as many as fill the resident CTA slots of the GPU in
// one wave (a second, partial wave would only add a tail), at most one split per 128 keys of the capacity.  `blocks` =
// G * ceil(r * Sq / 16) CTAs per sample and split, of the FP8 instances when `fp8`.  Depends on the shapes only, never
// on the current lengths.
extern "C" int lb_decode_splits(int B, int blocks, int C, int D, bool fp8) {
  // (the ALiBi and T5 instances hold as many CTAs per SM: the same shared memory, and registers that do not limit it)
  using lb::dec::Score;
  const int resident = fp8        ? lb::dec::decode_fp8_resident(D)
                       : D == 64 ? lb::dec::configure_decode<64, Score::kNone>()
                                 : lb::dec::configure_decode<128, Score::kNone>();
  int n = lb_host::num_sms() * (resident > 0 ? resident : 1) / (B * blocks);
  n = n < (C + 127) / 128 ? n : (C + 127) / 128;
  n = n < lb::dec::kMaxSplits ? n : lb::dec::kMaxSplits;
  return n > 1 ? n : 1;
}

extern "C" int lb_decode_attn(const void* q, const long* q_strides, const void* k, const void* v, void* o,
                              float* part_o, float* part_ml, const int* seqlens, const int* kv_start,
                              const float* alibi_slopes, const float* rel_bias, int R, bool causal,
                              const float* k_scale, const float* v_scale, const int* block_table, int max_pages, int B,
                              int Sq, int A, int G, int C, int D, float scale, int nsplit, cudaStream_t s) {
  if (B == 0 || A == 0) return 0;
  if (G <= 0 || A % G) return -4;
  // the four kinds: no bias or ALiBi or T5's relative bias (causal), no bias (non-causal)
  if ((alibi_slopes != nullptr) + (rel_bias != nullptr) + !causal > 1 || (rel_bias != nullptr && R < 1)) return -5;
  if ((k_scale != nullptr) != (v_scale != nullptr) || (k_scale != nullptr && C % 4)) return -6;
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
  p.bias = alibi_slopes != nullptr ? alibi_slopes : rel_bias;
  p.R = R;
  using lb::dec::Score;
  const Score score = alibi_slopes != nullptr ? Score::kAlibi
                      : rel_bias != nullptr   ? Score::kRelBias
                      : !causal               ? Score::kWindow
                                              : Score::kNone;
  cudaError_t e = D == 64 ? launch_decode<64>(p, k_scale, v_scale, block_table, max_pages, B, nsplit, score, s)
                          : launch_decode<128>(p, k_scale, v_scale, block_table, max_pages, B, nsplit, score, s);
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
