// FP8 (E4M3) KV caches: the quantizing cache append, and the instances of the split-KV decode attention kernel for
// every score kind at head dims 64 and 128.  Kept in their own translation unit so that the objects of the bf16
// kernels hold exactly the kernels they held before them.  The format, the scale folding and the shared-memory layout are described
// at Cfg8 and decode_attn_body in decode_attention_sm90.cuh; the partials go through the same decode_combine_kernel.
#include "decode_attention_sm90.cuh"

namespace lb {
namespace dec {

// the FP8 cache append: one warp per (b, i, group); lane c < D/2 handles the pairs (c + 32 p, c + 32 p + D/2) of the
// r q rows and of k (rotated, RopePair) and of v, then each of the k and v rows is quantized (quantize_row) at row
// cache_seqlens[b] + i
template <int D>
__global__ void __launch_bounds__(256) kv_append_fp8_kernel(
    const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ cosv, const float* __restrict__ sinv,
    __nv_bfloat16* __restrict__ q_out, uint8_t* __restrict__ kc, uint8_t* __restrict__ vc, float* __restrict__ ks,
    float* __restrict__ vs, const int* __restrict__ seqlens, int B, int Sq, int G, int r, int C) {
  kv_append_fp8_body<D, false>(qkv, cosv, sinv, q_out, kc, vc, ks, vs, seqlens, nullptr, 0, B, Sq, G, r, C);
}

template <int D, Score S>
__global__ void __launch_bounds__(kThreads) decode_attn_fp8_kernel(const Params p, const float* k_scale,
                                                                   const float* v_scale) {
  decode_attn_body<D, S, true>(p, k_scale, v_scale);
}

template <int D, Score S>
int configure_decode_fp8() {
  static int resident = 0;
  if (resident == 0) {
    auto kern = decode_attn_fp8_kernel<D, S>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg8<D>::kSmem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, kThreads, Cfg8<D>::kSmem) != cudaSuccess)
      resident = 0;
  }
  return resident;
}

template <int D, Score S>
cudaError_t launch_fp8(const Params& p, const float* k_scale, const float* v_scale, int B, int nsplit,
                       cudaStream_t s) {
  if (configure_decode_fp8<D, S>() == 0) return cudaErrorInvalidConfiguration;   // the shared memory opt-in failed
  decode_attn_fp8_kernel<D, S><<<dim3(nsplit, p.G * p.row_blocks, B), kThreads, Cfg8<D>::kSmem, s>>>(p, k_scale,
                                                                                                      v_scale);
  return cudaGetLastError();
}

template <int D>
cudaError_t launch_fp8(const Params& p, const float* k_scale, const float* v_scale, Score S, int B, int nsplit,
                       cudaStream_t s) {
  switch (S) {
    case Score::kNone: return launch_fp8<D, Score::kNone>(p, k_scale, v_scale, B, nsplit, s);
    case Score::kAlibi: return launch_fp8<D, Score::kAlibi>(p, k_scale, v_scale, B, nsplit, s);
    case Score::kRelBias: return launch_fp8<D, Score::kRelBias>(p, k_scale, v_scale, B, nsplit, s);
    default: return launch_fp8<D, Score::kWindow>(p, k_scale, v_scale, B, nsplit, s);
  }
}

cudaError_t launch_decode_attn_fp8(const Params& p, const float* k_scale, const float* v_scale, Score S, int D, int B,
                                   int nsplit, cudaStream_t s) {
  return D == 64 ? launch_fp8<64>(p, k_scale, v_scale, S, B, nsplit, s)
                 : launch_fp8<128>(p, k_scale, v_scale, S, B, nsplit, s);
}

// (the other score kinds hold as many CTAs per SM: the same shared memory, and registers that do not limit it)
int decode_fp8_resident(int D) {
  return D == 64 ? configure_decode_fp8<64, Score::kNone>() : configure_decode_fp8<128, Score::kNone>();
}

}  // namespace dec
}  // namespace lb

extern "C" int lb_kv_append_fp8(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_cache,
                                void* v_cache, float* k_scale, float* v_scale, const int* seqlens, int B, int Sq, int G,
                                int r, int C, int D, cudaStream_t s) {
  const size_t warps = (size_t)B * Sq * G;
  if (warps == 0) return 0;
  if (D != 64 && D != 128) return -4;
  const int threads = 256;
  const int blocks = (int)((warps * 32 + threads - 1) / threads < 4096 ? (warps * 32 + threads - 1) / threads : 4096);
  auto kern = D == 64 ? lb::dec::kv_append_fp8_kernel<64> : lb::dec::kv_append_fp8_kernel<128>;
  kern<<<blocks, threads, 0, s>>>(static_cast<const __nv_bfloat16*>(qkv), cosv, sinv,
                                  static_cast<__nv_bfloat16*>(q_out), static_cast<uint8_t*>(k_cache),
                                  static_cast<uint8_t*>(v_cache), k_scale, v_scale, seqlens, B, Sq, G, r, C);
  return (int)cudaGetLastError();
}
