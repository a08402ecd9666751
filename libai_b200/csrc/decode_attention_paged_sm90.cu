// Paged KV caches: the split-KV decode attention kernel and the cache appends over pools of 64-row pages, and the page
// copy of copy-on-write.  Kept in their own translation unit so that the objects of the contiguous kernels hold exactly
// the kernels they held before them.
//
// A paged cache holds, per layer, a K and a V pool [P, G, kTile, D] (bf16, or E4M3 bytes with fp32 row scales
// [P, G, kTile]) and one block table int32 [B, max_pages] for every layer: logical row j of sample b is row j % kTile of
// page block_table[b][j / kTile].  A page is one tile of the decode kernel (kTile = 64 rows).  The kernels read the
// pages of the rows they touch and nothing else of the table; that those page ids are in [0, P) is the caller's
// guarantee, like the lengths (libai_b200.inference.kv_cache.PagedKVCache maps the pages of a step's rows before it).
//
// decode attention: decode_attn_body<..., PAGED = true>.  Its tiles start at kv_start[b] as in the contiguous kernel,
//   not at page boundaries, so a tile may span two pages; every sum then runs in the contiguous kernel's order and the
//   output is bit-identical to it over the same logical rows and the same number of splits.  bf16 issues one bulk copy
//   per row as before (only the address changes); FP8 issues one bulk copy per page piece and array, at most two.
//   Instances: no score bias and ALiBi, bf16 and FP8, D = 64 and 128.
// appends: kv_append_body / kv_append_fp8_body with the row address taken through the table; bytes and scales are
//   those of the contiguous appends.  The ragged appends (the RAGGED flag of kv_append_body and kv_append_fp8_body)
//   write the tokens of N sequences packed along one axis, each at its own rows; their bytes (and FP8 scales) are
//   those of the paged append per sequence.
// page copy: the (src, dst) page pairs of every array of a list (K, V and the FP8 scales of every layer) in one
//   launch.
#include "decode_attention_sm90.cuh"

namespace lb {
namespace dec {

template <int D, Score S, bool FP8>
__global__ void __launch_bounds__(kThreads) decode_attn_paged_kernel(const Params p, const float* k_scale,
                                                                     const float* v_scale, const int* block_table,
                                                                     int max_pages) {
  decode_attn_body<D, S, FP8, true>(p, k_scale, v_scale, block_table, max_pages);
}

template <int D, Score S, bool FP8>
cudaError_t launch_paged(const Params& p, const float* k_scale, const float* v_scale, const int* block_table,
                         int max_pages, int B, int nsplit, cudaStream_t s) {
  constexpr int smem = FP8 ? Cfg8<D>::kSmem : Cfg<D>::kSmem;
  static bool configured = false;
  auto kern = decode_attn_paged_kernel<D, S, FP8>;
  if (!configured) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return cudaErrorInvalidConfiguration;   // the shared memory opt-in failed
    configured = true;
  }
  kern<<<dim3(nsplit, p.G * p.row_blocks, B), kThreads, smem, s>>>(p, k_scale, v_scale, block_table, max_pages);
  return cudaGetLastError();
}

template <int D, bool FP8>
cudaError_t launch_paged(const Params& p, const float* k_scale, const float* v_scale, const int* table, int max_pages,
                         Score S, int B, int nsplit, cudaStream_t s) {
  return S == Score::kAlibi ? launch_paged<D, Score::kAlibi, FP8>(p, k_scale, v_scale, table, max_pages, B, nsplit, s)
                            : launch_paged<D, Score::kNone, FP8>(p, k_scale, v_scale, table, max_pages, B, nsplit, s);
}

cudaError_t launch_decode_attn_paged(const Params& p, const float* k_scale, const float* v_scale, const int* table,
                                     int max_pages, Score S, int D, int B, int nsplit, cudaStream_t s) {
  if (S != Score::kNone && S != Score::kAlibi) return cudaErrorInvalidValue;
  const bool fp8 = k_scale != nullptr;
  if (D == 64)
    return fp8 ? launch_paged<64, true>(p, k_scale, v_scale, table, max_pages, S, B, nsplit, s)
               : launch_paged<64, false>(p, k_scale, v_scale, table, max_pages, S, B, nsplit, s);
  return fp8 ? launch_paged<128, true>(p, k_scale, v_scale, table, max_pages, S, B, nsplit, s)
             : launch_paged<128, false>(p, k_scale, v_scale, table, max_pages, S, B, nsplit, s);
}

__global__ void kv_append_paged_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv,
                                       const float* __restrict__ sinv, __nv_bfloat16* __restrict__ q_out,
                                       __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc,
                                       const int* __restrict__ seqlens, const int* __restrict__ table, int max_pages,
                                       int B, int Sq, int G, int r, int D) {
  kv_append_body<true>(qkv, cosv, sinv, q_out, kc, vc, seqlens, table, max_pages, B, Sq, G, r, kTile, D);
}

// the append of N ragged sequences packed along the token axis (kv_append_body's RAGGED flag)
__global__ void kv_append_paged_varlen_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv,
                                              const float* __restrict__ sinv, __nv_bfloat16* __restrict__ q_out,
                                              __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc,
                                              const int* __restrict__ cu_q, const int* __restrict__ past, int nseq,
                                              const int* __restrict__ table, int max_pages, int T, int G, int r,
                                              int D) {
  kv_append_body<true, true>(qkv, cosv, sinv, q_out, kc, vc, past, table, max_pages, 1, T, G, r, kTile, D, cu_q, nseq);
}

template <int D>
__global__ void __launch_bounds__(256) kv_append_fp8_paged_kernel(
    const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv, const float* __restrict__ sinv,
    __nv_bfloat16* __restrict__ q_out, uint8_t* __restrict__ kc, uint8_t* __restrict__ vc, float* __restrict__ ks,
    float* __restrict__ vs, const int* __restrict__ seqlens, const int* __restrict__ table, int max_pages, int B,
    int Sq, int G, int r) {
  kv_append_fp8_body<D, true>(qkv, cosv, sinv, q_out, kc, vc, ks, vs, seqlens, table, max_pages, B, Sq, G, r, kTile);
}

// the FP8 append of N ragged sequences packed along the token axis (kv_append_fp8_body's RAGGED flag)
template <int D>
__global__ void __launch_bounds__(256) kv_append_fp8_paged_varlen_kernel(
    const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv, const float* __restrict__ sinv,
    __nv_bfloat16* __restrict__ q_out, uint8_t* __restrict__ kc, uint8_t* __restrict__ vc, float* __restrict__ ks,
    float* __restrict__ vs, const int* __restrict__ cu_q, const int* __restrict__ past, int nseq,
    const int* __restrict__ table, int max_pages, int T, int G, int r) {
  kv_append_fp8_body<D, true, true>(qkv, cosv, sinv, q_out, kc, vc, ks, vs, past, table, max_pages, 1, T, G, r, kTile,
                                    cu_q, nseq);
}

// one CTA per (pair, array): the page src of array a to its page dst, 16 bytes per thread and step
__global__ void __launch_bounds__(256) kv_page_copy_kernel(const long* __restrict__ desc, int npairs) {
  // desc: npairs (src, dst) pairs, then per array its address and its page bytes (a multiple of 16)
  const int i = blockIdx.x, a = blockIdx.y;
  const long src = desc[2 * i], dst = desc[2 * i + 1];
  unsigned char* base = reinterpret_cast<unsigned char*>(desc[2 * npairs + 2 * a]);
  const long bytes = desc[2 * npairs + 2 * a + 1];
  const uint4* from = reinterpret_cast<const uint4*>(base + src * bytes);
  uint4* to = reinterpret_cast<uint4*>(base + dst * bytes);
  for (long e = threadIdx.x; e < bytes / 16; e += blockDim.x) to[e] = from[e];
}

}  // namespace dec
}  // namespace lb

extern "C" int lb_kv_append_paged(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool,
                                  void* v_pool, const int* seqlens, const int* block_table, int max_pages, int B,
                                  int Sq, int G, int r, int D, cudaStream_t s) {
  const size_t total = (size_t)B * Sq * G * (D / 2);
  if (total == 0) return 0;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < 4096 ? (total + threads - 1) / threads : 4096);
  lb::dec::kv_append_paged_kernel<<<blocks, threads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(qkv), cosv, sinv, static_cast<__nv_bfloat16*>(q_out),
      static_cast<__nv_bfloat16*>(k_pool), static_cast<__nv_bfloat16*>(v_pool), seqlens, block_table, max_pages, B, Sq,
      G, r, D);
  return (int)cudaGetLastError();
}

extern "C" int lb_kv_append_paged_varlen(const void* qkv, const float* cosv, const float* sinv, void* q_out,
                                         void* k_pool, void* v_pool, const int* cu_q, const int* past, int nseq,
                                         const int* block_table, int max_pages, int T, int G, int r, int D,
                                         cudaStream_t s) {
  const size_t total = (size_t)T * G * (D / 2);
  if (total == 0 || nseq == 0) return 0;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < 4096 ? (total + threads - 1) / threads : 4096);
  lb::dec::kv_append_paged_varlen_kernel<<<blocks, threads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(qkv), cosv, sinv, static_cast<__nv_bfloat16*>(q_out),
      static_cast<__nv_bfloat16*>(k_pool), static_cast<__nv_bfloat16*>(v_pool), cu_q, past, nseq, block_table,
      max_pages, T, G, r, D);
  return (int)cudaGetLastError();
}

extern "C" int lb_kv_append_fp8_paged(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool,
                                      void* v_pool, float* k_scale, float* v_scale, const int* seqlens,
                                      const int* block_table, int max_pages, int B, int Sq, int G, int r, int D,
                                      cudaStream_t s) {
  const size_t warps = (size_t)B * Sq * G;
  if (warps == 0) return 0;
  if (D != 64 && D != 128) return -4;
  const int threads = 256;
  const int blocks = (int)((warps * 32 + threads - 1) / threads < 4096 ? (warps * 32 + threads - 1) / threads : 4096);
  auto kern = D == 64 ? lb::dec::kv_append_fp8_paged_kernel<64> : lb::dec::kv_append_fp8_paged_kernel<128>;
  kern<<<blocks, threads, 0, s>>>(static_cast<const __nv_bfloat16*>(qkv), cosv, sinv,
                                  static_cast<__nv_bfloat16*>(q_out), static_cast<uint8_t*>(k_pool),
                                  static_cast<uint8_t*>(v_pool), k_scale, v_scale, seqlens, block_table, max_pages, B,
                                  Sq, G, r);
  return (int)cudaGetLastError();
}

extern "C" int lb_kv_append_fp8_paged_varlen(const void* qkv, const float* cosv, const float* sinv, void* q_out,
                                             void* k_pool, void* v_pool, float* k_scale, float* v_scale,
                                             const int* cu_q, const int* past, int nseq, const int* block_table,
                                             int max_pages, int T, int G, int r, int D, cudaStream_t s) {
  const size_t warps = (size_t)T * G;
  if (warps == 0 || nseq == 0) return 0;
  if (D != 64 && D != 128) return -4;
  const int threads = 256;
  const int blocks = (int)((warps * 32 + threads - 1) / threads < 4096 ? (warps * 32 + threads - 1) / threads : 4096);
  auto kern = D == 64 ? lb::dec::kv_append_fp8_paged_varlen_kernel<64> : lb::dec::kv_append_fp8_paged_varlen_kernel<128>;
  kern<<<blocks, threads, 0, s>>>(static_cast<const __nv_bfloat16*>(qkv), cosv, sinv,
                                  static_cast<__nv_bfloat16*>(q_out), static_cast<uint8_t*>(k_pool),
                                  static_cast<uint8_t*>(v_pool), k_scale, v_scale, cu_q, past, nseq, block_table,
                                  max_pages, T, G, r);
  return (int)cudaGetLastError();
}

extern "C" int lb_kv_page_copy(const long* desc, int npairs, int narrays, cudaStream_t s) {
  if (npairs == 0 || narrays == 0) return 0;
  lb::dec::kv_page_copy_kernel<<<dim3(npairs, narrays), 256, 0, s>>>(desc, npairs);
  return (int)cudaGetLastError();
}
