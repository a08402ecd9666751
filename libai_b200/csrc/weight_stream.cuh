// What the weight-streaming linear kernels (linear_fp8w_sm90.cu, linear_int4w_sm90.cu) share: the K-split policy, the
// streaming load, the bias/activation epilogue and the kernel that sums the fp32 partials of the K ranges.
//
// A CTA is 4 warps = 64 weight rows over one K range.  The number of K ranges (splits) is chosen from (N, K) alone, so
// that about 4 · 132 CTAs are in flight even at N = 4096; with more than one range the fp32 partials [splits, M, N] go
// to a workspace and combine() sums them in range order.  Neither the splits nor any summation order depend on M: a
// token's output row is the same bits whether it is computed alone or among 63 others.
#pragma once

#include "common.cuh"

namespace lb {
namespace wstream {

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kRows = kWarps * 16;     // weight rows per CTA
constexpr int kMinRange = 256;         // K columns of a range at least
constexpr int kTargetCtas = 4 * 132;   // CTAs to keep in flight: four per SM of an H100 SXM

struct Split {
  int splits, range;   // range: K columns per split (a multiple of the kernel's step; the last split may hold fewer)
};

// step: the K columns a warp consumes per step; every range but the last is a multiple of it
inline Split split_of(int N, int K, int step) {
  const int row_blocks = (N + kRows - 1) / kRows;
  const int max_splits = (K + kMinRange - 1) / kMinRange;
  const int want = (kTargetCtas + row_blocks - 1) / row_blocks;
  const int splits = want < 1 ? 1 : (want > max_splits ? max_splits : want);
  const int range = ((K + splits - 1) / splits + step - 1) / step * step;
  return {(K + range - 1) / range, range};
}

// 16 bytes that are read once: no L1 allocation, and the rest of the 256-byte L2 block is prefetched (the next steps
// of the same rows read it)
LB_DEVICE uint4 ld_stream(const void* p) {
  uint4 r;
  asm("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];\n"
      : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
      : "l"(p));
  return r;
}

LB_DEVICE uint32_t word(const uint4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

// act(acc · scale[n] + bias[n]) of a finished fp32 sum; kRowScale false: act(acc + bias[n]) (scale unused)
template <bool kRowScale>
LB_DEVICE float epilogue(float acc, int n, const float* scale, const __nv_bfloat16* bias, int act) {
  float v = acc;
  if constexpr (kRowScale) v = acc * scale[n];
  if (bias != nullptr) v += __bfloat162float(bias[n]);
  return act_fwd(v, act);
}

// y = epilogue(sum over the splits of part [splits, M, N]), summed in split order
template <bool kRowScale>
__global__ void combine(const float* __restrict__ part, const float* __restrict__ scale,
                        const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int MN, int N,
                        int splits, int act) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < MN; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < splits; ++p) s += part[(long)p * MN + i];
    y[i] = __float2bfloat16(epilogue<kRowScale>(s, i % N, scale, bias, act));
  }
}

template <bool kRowScale>
cudaError_t launch_combine(const float* part, const float* scale, const void* bias, void* y, int M, int N, int splits,
                           int act, cudaStream_t s) {
  const int MN = M * N, blocks = (MN + 255) / 256;
  combine<kRowScale><<<blocks, 256, 0, s>>>(part, scale, static_cast<const __nv_bfloat16*>(bias),
                                            static_cast<__nv_bfloat16*>(y), MN, N, splits, act);
  return cudaGetLastError();
}

}  // namespace wstream
}  // namespace lb
