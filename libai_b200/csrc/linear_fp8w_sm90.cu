// Linear layers over FP8 (E4M3) weights with one fp32 scale per output channel, for the decode steps of generate():
//
//   y [M, N] (bf16) = act((x [M, K] · float(W [N, K])ᵀ) · s [N] + bias [N]),  x bf16, W E4M3, fp32 accumulation.
//
// With M = 1 .. 64 tokens the product is a stream over the N·K weight bytes, and the kernel exists to read them at HBM
// bandwidth.  The operands are swapped: weight rows are the M dimension of mma.sync m16n8k16 (16 output channels per
// fragment, one per warp) and tokens its N dimension (one n8 tile per 8 tokens).  Each lane quad holds 64 bytes of a
// row pair per step, loaded straight into registers with 16-byte streaming loads; the lanes widen them to bf16 (exact)
// and feed them to the MMA as the A fragment.  The K positions of a step are permuted: lane q's four columns of k-step
// j are bytes q·16 + j·4 .. + 3 of the 64, so one 16-byte load covers the lane's A operands of all four k-steps and two
// 16-byte loads of x its B operands.  Every sum runs over the same K positions, in a fixed order.  The loads of the
// next steps are in flight while the current ones are multiplied.
//
// The split policy, the streaming load, the epilogue and the sum over the K ranges are weight_stream.cuh's.  The
// per-row scale, the bias and the activation are applied once, to the finished fp32 sum.
#include "weight_stream.cuh"

namespace lb {
namespace fp8w {

using namespace wstream;

constexpr int kStep = 64;              // K columns per warp step: 16 bytes of each row per lane of a quad

// NT: n8 tiles of tokens (M <= 8 * NT); U: steps whose weight loads are issued together
template <int NT, int U>
__global__ void __launch_bounds__(kThreads) linear_fp8w_kernel(const __nv_bfloat16* __restrict__ x,
                                                              const uint8_t* __restrict__ w,
                                                              const float* __restrict__ scale,
                                                              const __nv_bfloat16* __restrict__ bias,
                                                              __nv_bfloat16* __restrict__ y, float* __restrict__ part,
                                                              int M, int N, int K, int range, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = lane & 3, g = lane >> 2;
  const int row = blockIdx.x * kRows + warp * 16 + g;   // this lane's rows: row and row + 8
  const int k0 = blockIdx.y * range, k1 = min(K, k0 + range);
  const bool v0 = row < N, v1 = row + 8 < N;
  const uint8_t* w0 = w + (long)(v0 ? row : 0) * K + q * 16;
  const uint8_t* w1 = w + (long)(v1 ? row + 8 : 0) * K + q * 16;

  float acc[NT][4];
#pragma unroll
  for (int t = 0; t < NT; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;

  // columns past k1 (K % 64 may be 16, 32 or 48) and rows past N load zeros
  uint4 cur[U][2], nxt[U][2];
  auto load = [&](uint4 (&dst)[U][2], int kb) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = kb + u * kStep + q * 16;
      dst[u][0] = v0 && k < k1 ? ld_stream(w0 + kb + u * kStep) : make_uint4(0, 0, 0, 0);
      dst[u][1] = v1 && k < k1 ? ld_stream(w1 + kb + u * kStep) : make_uint4(0, 0, 0, 0);
    }
  };
  load(cur, k0);
  for (int kb = k0; kb < k1; kb += U * kStep) {
    load(nxt, kb + U * kStep);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = kb + u * kStep + q * 16;
      if (kb + u * kStep >= k1) break;
      uint32_t a[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint2 lo = e4m3x4_to_bf16x4(word(cur[u][0], j)), hi = e4m3x4_to_bf16x4(word(cur[u][1], j));
        a[j][0] = lo.x;
        a[j][1] = hi.x;
        a[j][2] = lo.y;
        a[j][3] = hi.y;
      }
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int tok = t * 8 + g;
        uint4 xa = make_uint4(0, 0, 0, 0), xb = make_uint4(0, 0, 0, 0);
        if (tok < M && k < k1) {
          const uint4* xp = reinterpret_cast<const uint4*>(x + (long)tok * K + k);
          xa = __ldg(xp);
          xb = __ldg(xp + 1);
        }
        mma_bf16(acc[t], a[0], xa.x, xa.y);
        mma_bf16(acc[t], a[1], xa.z, xa.w);
        mma_bf16(acc[t], a[2], xb.x, xb.y);
        mma_bf16(acc[t], a[3], xb.z, xb.w);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      cur[u][0] = nxt[u][0];
      cur[u][1] = nxt[u][1];
    }
  }

  // acc[t]: (row, token t·8 + 2q), (row, t·8 + 2q + 1), (row + 8, t·8 + 2q), (row + 8, t·8 + 2q + 1)
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int tok = t * 8 + 2 * q + (e & 1), n = row + (e >> 1) * 8;
      if (tok >= M || n >= N) continue;
      if (gridDim.y == 1)
        y[(long)tok * N + n] = __float2bfloat16(epilogue<true>(acc[t][e], n, scale, bias, act));
      else
        part[((long)blockIdx.y * M + tok) * N + n] = acc[t][e];
    }
}

// out [rows, K] bf16 = bf16_rn(float(w) · scale[row]); 16 weight bytes per thread and step
__global__ void dequant_e4m3_rows(const uint8_t* __restrict__ w, const float* __restrict__ scale,
                                  __nv_bfloat16* __restrict__ out, long chunks, int K) {
  const int per_row = K / 16;
  for (long c = blockIdx.x * (long)blockDim.x + threadIdx.x; c < chunks; c += (long)gridDim.x * blockDim.x) {
    const float s = scale[c / per_row];
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(w) + c);
    uint32_t o[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t b = word(v, i);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __half2_raw r =
            __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(b >> (16 * h)), __NV_E4M3);
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&r));
        o[2 * i + h] = pack_bf16(__fmul_rn(f.x, s), __fmul_rn(f.y, s));
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(out) + 2 * c;
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

template <int NT, int U>
cudaError_t launch(const void* x, const void* w, const float* scale, const void* bias, void* y, float* part, int M,
                   int N, int K, int act, cudaStream_t s) {
  const Split sp = split_of(N, K, kStep);
  linear_fp8w_kernel<NT, U><<<dim3((N + kRows - 1) / kRows, sp.splits), kThreads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const uint8_t*>(w), scale,
      static_cast<const __nv_bfloat16*>(bias), static_cast<__nv_bfloat16*>(y), part, M, N, K, sp.range, act);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || sp.splits == 1) return e;
  return launch_combine<true>(part, scale, bias, y, M, N, sp.splits, act, s);
}

}  // namespace fp8w
}  // namespace lb

extern "C" {

long lb_linear_fp8w_workspace(int M, int N, int K) {
  const lb::wstream::Split sp = lb::wstream::split_of(N, K, lb::fp8w::kStep);
  return sp.splits > 1 ? (long)sp.splits * M * N : 0;
}

int lb_linear_fp8w(const void* x, const void* w, const float* w_scale, const void* bias, void* y, float* part, int M,
                   int N, int K, int act, cudaStream_t s) {
  using namespace lb::fp8w;
  if (M < 1 || M > 64 || N < 1 || K < 16 || K % 16 != 0) return static_cast<int>(cudaErrorInvalidValue);
  cudaError_t e;
  if (M <= 8)
    e = launch<1, 4>(x, w, w_scale, bias, y, part, M, N, K, act, s);
  else if (M <= 16)
    e = launch<2, 4>(x, w, w_scale, bias, y, part, M, N, K, act, s);
  else if (M <= 32)
    e = launch<4, 2>(x, w, w_scale, bias, y, part, M, N, K, act, s);
  else
    e = launch<8, 2>(x, w, w_scale, bias, y, part, M, N, K, act, s);
  return static_cast<int>(e);
}

int lb_dequant_e4m3_rows(const void* w, const float* scale, void* out, long rows, int K, cudaStream_t s) {
  if (rows < 1 || K < 16 || K % 16 != 0) return static_cast<int>(cudaErrorInvalidValue);
  const long chunks = rows * (K / 16);
  const long blocks = (chunks + 255) / 256;
  lb::fp8w::dequant_e4m3_rows<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, s>>>(
      static_cast<const uint8_t*>(w), scale, static_cast<__nv_bfloat16*>(out), chunks, K);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
