// Linear layers over group-wise INT4 weights, for the decode steps of generate():
//
//   y [M, N] (bf16) = act(x [M, K] · Ŵᵀ + bias [N]),  Ŵ[n, k] = bf16_rn((q[n, k] − z[n, k/128]) · s[n, k/128]),
//
// x bf16, fp32 accumulation.  q is packed two per byte (byte j of row n: column 2j in the low nibble, 2j + 1 in the
// high one), s is bf16 and z a uint8 in 0..15, one pair per row and group of 128 columns.  q − z is an integer in
// [−15, 15] and s has an 8-bit significand, so the product is exact and Ŵ is one rounding: the bf16 the MMA multiplies
// is the weight dequant_int4_rows writes and OF.int4_dequant_ref computes.
//
// With M = 1 .. 64 tokens the product is a stream over the N·K/2 weight bytes.  The layout is linear_fp8w's: weight
// rows are the M dimension of mma.sync m16n8k16 (one 16-row fragment per warp) and tokens its N dimension (one n8 tile
// per 8 tokens), and the weight bytes go from 16-byte streaming loads straight into registers.  A warp step is one
// group: lane q of a quad loads columns q·32 .. q·32 + 31 of the group (16 bytes) for each of its two rows, so a load
// needs one (s, z) per row.  A nibble becomes bf16 128 + q with one lop3 into the mantissa of 128.0; one bf16x2
// subtract of 128 + z and one bf16x2 multiply by s then give Ŵ with the rounding above.  The K positions are permuted:
// a 32-bit word holds columns c0 .. c7, and the four bf16x2 values (c0, c4), (c1, c5), (c2, c6), (c3, c7) come from
// shifts of it by 0, 4, 8 and 12 bits, so they are the A operands of two k-steps as they are; x's columns are paired
// the same way with byte permutes.  Every sum runs over the same K positions, in a fixed order.  The loads of the next
// steps (weights, scales and zeros) are in flight while the current ones are multiplied.
//
// The split policy (ranges of whole groups), the streaming load, the epilogue and the sum over the K ranges are
// weight_stream.cuh's; the bias and the activation are applied once, to the finished fp32 sum.
#include "weight_stream.cuh"

namespace lb {
namespace int4w {

using namespace wstream;

constexpr int kGroup = 128;   // K columns per (s, z)
constexpr int kStep = 128;    // K columns per warp step: one group, 16 bytes of each row per lane of a quad

LB_DEVICE uint32_t sub_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("sub.rn.bf16x2 %0, %1, %2;\n" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

LB_DEVICE uint32_t mul_bf16x2(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;\n" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

// The bf16x2 (128 + z, 128 + z) and (s, s) of a (scale, zero) pair: the second operands of the subtract and multiply
struct GroupCoef {
  uint32_t zz, ss;
  LB_DEVICE static GroupCoef of(uint16_t s_bits, uint8_t z) {
    return {0x43004300u | z | (uint32_t(z) << 16), s_bits | (uint32_t(s_bits) << 16)};
  }
};

// Ŵ of the eight columns c0 .. c7 of a packed word (bytes c0|c1, c2|c3, c4|c5, c6|c7): r[i] = bf16x2 (c_i, c_i+4)
LB_DEVICE void dequant_word(uint32_t v, const GroupCoef& c, uint32_t (&r)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t biased = ((v >> (4 * i)) & 0x000F000Fu) | 0x43004300u;   // bf16x2 (128 + c_i, 128 + c_i+4)
    r[i] = mul_bf16x2(sub_bf16x2(biased, c.zz), c.ss);
  }
}

// NT: n8 tiles of tokens (M <= 8 * NT); U: steps whose weight loads are issued together
template <int NT, int U>
__global__ void __launch_bounds__(kThreads) linear_int4w_kernel(const __nv_bfloat16* __restrict__ x,
                                                               const uint8_t* __restrict__ w,
                                                               const uint16_t* __restrict__ scale,
                                                               const uint8_t* __restrict__ zero,
                                                               const __nv_bfloat16* __restrict__ bias,
                                                               __nv_bfloat16* __restrict__ y, float* __restrict__ part,
                                                               int M, int N, int K, int range, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = lane & 3, g = lane >> 2;
  const int row = blockIdx.x * kRows + warp * 16 + g;   // this lane's rows: row and row + 8
  const int k0 = blockIdx.y * range, k1 = min(K, k0 + range);
  const bool v0 = row < N, v1 = row + 8 < N;
  const int groups = K / kGroup;
  const long r0 = v0 ? row : 0, r1 = v1 ? row + 8 : 0;
  const uint8_t* w0 = w + r0 * (K / 2) + q * 16;
  const uint8_t* w1 = w + r1 * (K / 2) + q * 16;

  float acc[NT][4];
#pragma unroll
  for (int t = 0; t < NT; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;

  // ranges hold whole groups, so a step is inside [k0, k1) or past it; rows past N load zeros (Ŵ = 0)
  uint4 cur[U][2], nxt[U][2];
  uint16_t cs[U][2], ns[U][2];
  uint8_t cz[U][2], nz[U][2];
  auto load = [&](uint4 (&dst)[U][2], uint16_t (&ds)[U][2], uint8_t (&dz)[U][2], int kb) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = kb + u * kStep;
      const bool in = k < k1;
      const int grp = k / kGroup;
      dst[u][0] = v0 && in ? ld_stream(w0 + k / 2) : make_uint4(0, 0, 0, 0);
      dst[u][1] = v1 && in ? ld_stream(w1 + k / 2) : make_uint4(0, 0, 0, 0);
      ds[u][0] = v0 && in ? __ldg(scale + r0 * groups + grp) : uint16_t(0);
      ds[u][1] = v1 && in ? __ldg(scale + r1 * groups + grp) : uint16_t(0);
      dz[u][0] = v0 && in ? __ldg(zero + r0 * groups + grp) : uint8_t(0);
      dz[u][1] = v1 && in ? __ldg(zero + r1 * groups + grp) : uint8_t(0);
    }
  };
  load(cur, cs, cz, k0);
  for (int kb = k0; kb < k1; kb += U * kStep) {
    load(nxt, ns, nz, kb + U * kStep);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = kb + u * kStep + q * 32;   // this lane's first column of the step
      if (kb + u * kStep >= k1) break;
      const GroupCoef c0 = GroupCoef::of(cs[u][0], cz[u][0]), c1 = GroupCoef::of(cs[u][1], cz[u][1]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {   // columns k + 8j .. + 7: two k-steps
        uint32_t lo[4], hi[4];
        dequant_word(word(cur[u][0], j), c0, lo);
        dequant_word(word(cur[u][1], j), c1, hi);
        const uint32_t a0[4] = {lo[0], hi[0], lo[1], hi[1]};   // k-step of columns (c0, c4 | c1, c5)
        const uint32_t a1[4] = {lo[2], hi[2], lo[3], hi[3]};   // (c2, c6 | c3, c7)
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          const int tok = t * 8 + g;
          uint4 xv = make_uint4(0, 0, 0, 0);
          if (tok < M) xv = __ldg(reinterpret_cast<const uint4*>(x + (long)tok * K + k + 8 * j));
          mma_bf16(acc[t], a0, __byte_perm(xv.x, xv.z, 0x5410), __byte_perm(xv.x, xv.z, 0x7632));
          mma_bf16(acc[t], a1, __byte_perm(xv.y, xv.w, 0x5410), __byte_perm(xv.y, xv.w, 0x7632));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      cur[u][0] = nxt[u][0];
      cur[u][1] = nxt[u][1];
      cs[u][0] = ns[u][0];
      cs[u][1] = ns[u][1];
      cz[u][0] = nz[u][0];
      cz[u][1] = nz[u][1];
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
        y[(long)tok * N + n] = __float2bfloat16(epilogue<false>(acc[t][e], n, nullptr, bias, act));
      else
        part[((long)blockIdx.y * M + tok) * N + n] = acc[t][e];
    }
}

// out [rows, K] bf16 = Ŵ; 16 packed bytes (32 columns of one group) per thread and step
__global__ void dequant_int4_rows(const uint8_t* __restrict__ w, const uint16_t* __restrict__ scale,
                                  const uint8_t* __restrict__ zero, __nv_bfloat16* __restrict__ out, long chunks,
                                  int K) {
  const int per_group = kGroup / 32;
  for (long c = blockIdx.x * (long)blockDim.x + threadIdx.x; c < chunks; c += (long)gridDim.x * blockDim.x) {
    const long grp = c / per_group;   // row-major over [rows, K / 128]
    const GroupCoef coef = GroupCoef::of(__ldg(scale + grp), __ldg(zero + grp));
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(w) + c);
    uint4* dst = reinterpret_cast<uint4*>(out) + 4 * c;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t r[4];   // (c0, c4), (c1, c5), (c2, c6), (c3, c7)
      dequant_word(word(v, i), coef, r);
      dst[i] = make_uint4(__byte_perm(r[0], r[1], 0x5410), __byte_perm(r[2], r[3], 0x5410),
                          __byte_perm(r[0], r[1], 0x7632), __byte_perm(r[2], r[3], 0x7632));
    }
  }
}

template <int NT, int U>
cudaError_t launch(const void* x, const void* w, const void* scale, const void* zero, const void* bias, void* y,
                   float* part, int M, int N, int K, int act, cudaStream_t s) {
  const Split sp = split_of(N, K, kStep);
  linear_int4w_kernel<NT, U><<<dim3((N + kRows - 1) / kRows, sp.splits), kThreads, 0, s>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const uint8_t*>(w), static_cast<const uint16_t*>(scale),
      static_cast<const uint8_t*>(zero), static_cast<const __nv_bfloat16*>(bias), static_cast<__nv_bfloat16*>(y), part,
      M, N, K, sp.range, act);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || sp.splits == 1) return e;
  return launch_combine<false>(part, nullptr, bias, y, M, N, sp.splits, act, s);
}

}  // namespace int4w
}  // namespace lb

extern "C" {

long lb_linear_int4w_workspace(int M, int N, int K) {
  const lb::wstream::Split sp = lb::wstream::split_of(N, K, lb::int4w::kStep);
  return sp.splits > 1 ? (long)sp.splits * M * N : 0;
}

int lb_linear_int4w(const void* x, const void* w, const void* w_scale, const void* w_zero, const void* bias, void* y,
                    float* part, int M, int N, int K, int act, cudaStream_t s) {
  using namespace lb::int4w;
  if (M < 1 || M > 64 || N < 1 || K < kGroup || K % kGroup != 0) return static_cast<int>(cudaErrorInvalidValue);
  cudaError_t e;
  if (M <= 8)
    e = launch<1, 4>(x, w, w_scale, w_zero, bias, y, part, M, N, K, act, s);
  else if (M <= 16)
    e = launch<2, 4>(x, w, w_scale, w_zero, bias, y, part, M, N, K, act, s);
  else if (M <= 32)
    e = launch<4, 2>(x, w, w_scale, w_zero, bias, y, part, M, N, K, act, s);
  else
    e = launch<8, 2>(x, w, w_scale, w_zero, bias, y, part, M, N, K, act, s);
  return static_cast<int>(e);
}

int lb_dequant_int4_rows(const void* w, const void* w_scale, const void* w_zero, void* out, long rows, int K,
                         cudaStream_t s) {
  using namespace lb::int4w;
  if (rows < 1 || K < kGroup || K % kGroup != 0) return static_cast<int>(cudaErrorInvalidValue);
  const long chunks = rows * (K / 32);
  const long blocks = (chunks + 255) / 256;
  dequant_int4_rows<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, s>>>(
      static_cast<const uint8_t*>(w), static_cast<const uint16_t*>(w_scale), static_cast<const uint8_t*>(w_zero),
      static_cast<__nv_bfloat16*>(out), chunks, K);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
