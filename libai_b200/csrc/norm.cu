// Fused LayerNorm / RMSNorm forward + backward for sm_90a (bandwidth-bound: one warp per row,
// 128-bit vector accesses, statistics in fp32, row cached in registers between the passes).
// Replaces flow._C.layer_norm_affine / rms_norm (reference libai/layers/layer_norm.py:78-131).
//
//   fwd : y = (x - mean) * rstd * gamma + beta          (rms: y = x * rstd * gamma, mean := 0)
//   bwd : dx = rstd * (g·γ - mean_h(g·γ) - x̂ · mean_h(g·γ·x̂))   (rms: no mean_h(g·γ) term)
//         dγ = Σ_rows g·x̂ ,  dβ = Σ_rows g        (two-stage: per-CTA partials, then column reduce)
#include "common.cuh"
#include <type_traits>

namespace lb {

constexpr int NORM_WARPS = 8;

template <typename T>
struct Vec8;
template <>
struct Vec8<__nv_bfloat16> {
  static LB_DEVICE void load(const __nv_bfloat16* p, float (&v)[8]) {
    uint4 q = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16(q.x), b = unpack_bf16(q.y), c = unpack_bf16(q.z), d = unpack_bf16(q.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
  static LB_DEVICE void store(__nv_bfloat16* p, const float (&v)[8]) {
    *reinterpret_cast<uint4*>(p) =
        make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
  }
};
template <>
struct Vec8<float> {
  static LB_DEVICE void load(const float* p, float (&v)[8]) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static LB_DEVICE void store(float* p, const float (&v)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
};

// H = VPL * 256 elements per row (each lane owns VPL vectors of 8, interleaved for coalescing)
template <typename T, typename W, int VPL, bool RMS>
__global__ void __launch_bounds__(NORM_WARPS * 32)
norm_fwd_kernel(const T* __restrict__ x, const W* __restrict__ gamma, const W* __restrict__ beta, T* __restrict__ y,
                float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, float eps) {
  constexpr int H = VPL * 256;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int row = blockIdx.x * NORM_WARPS + warp; row < rows; row += gridDim.x * NORM_WARPS) {
    const T* xr = x + static_cast<size_t>(row) * H;
    float v[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      Vec8<T>::load(xr + (i * 32 + lane) * 8, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
    float mean = 0.f;
    if (!RMS) mean = warp_sum(s) * (1.0f / H);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        sq += d * d;
      }
    const float rstd = rsqrtf(warp_sum(sq) * (1.0f / H) + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      rstd_out[row] = rstd;
    }
    T* yr = y + static_cast<size_t>(row) * H;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      float g[8], b[8], o[8];
      Vec8<W>::load(gamma + (i * 32 + lane) * 8, g);
      if (beta != nullptr) Vec8<W>::load(beta + (i * 32 + lane) * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = (v[i][j] - mean) * rstd * g[j];
        if (beta != nullptr) o[j] += b[j];
      }
      Vec8<T>::store(yr + (i * 32 + lane) * 8, o);
    }
  }
}

template <typename T, typename W, int VPL, bool RMS>
__global__ void __launch_bounds__(NORM_WARPS * 32)
norm_bwd_kernel(const T* __restrict__ gy, const T* __restrict__ x, const W* __restrict__ gamma,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in, T* __restrict__ gx,
                float* __restrict__ part_dgamma, float* __restrict__ part_dbeta, int rows,
                const T* __restrict__ gadd /* optional [rows, H]: gradient of the residual path, added to gx */) {
  constexpr int H = VPL * 256;
  __shared__ float red[NORM_WARPS][32 * 8 + 8];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  float dg[VPL][8], db[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dg[i][j] = db[i][j] = 0.f;
  float gam[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i) Vec8<W>::load(gamma + (i * 32 + lane) * 8, gam[i]);

  for (int row = blockIdx.x * NORM_WARPS + warp; row < rows; row += gridDim.x * NORM_WARPS) {
    const float mean = RMS ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    const T* xr = x + static_cast<size_t>(row) * H;
    const T* gr = gy + static_cast<size_t>(row) * H;
    float xh[VPL][8], gw[VPL][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      float xv[8], gv[8];
      Vec8<T>::load(xr + (i * 32 + lane) * 8, xv);
      Vec8<T>::load(gr + (i * 32 + lane) * 8, gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[i][j] = (xv[j] - mean) * rstd;
        gw[i][j] = gv[j] * gam[i][j];
        s1 += gw[i][j];
        s2 += gw[i][j] * xh[i][j];
        dg[i][j] += gv[j] * xh[i][j];
        db[i][j] += gv[j];
      }
    }
    s1 = RMS ? 0.f : warp_sum(s1) * (1.0f / H);
    s2 = warp_sum(s2) * (1.0f / H);
    T* gxr = gx + static_cast<size_t>(row) * H;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (gw[i][j] - s1 - xh[i][j] * s2);
      if (gadd != nullptr) {  // the skip connection's gradient rides along: saves autograd's separate add kernel
        float a[8];
        Vec8<T>::load(gadd + static_cast<size_t>(row) * H + (i * 32 + lane) * 8, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += a[j];
      }
      Vec8<T>::store(gxr + (i * 32 + lane) * 8, o);
    }
  }
  // block-level reduction of the per-warp column partials, one vector slot at a time
  for (int i = 0; i < VPL; ++i) {
    for (int which = 0; which < (part_dbeta != nullptr ? 2 : 1); ++which) {
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = which == 0 ? dg[i][j] : db[i][j];
      __syncthreads();
      for (int c = threadIdx.x; c < 256; c += NORM_WARPS * 32) {
        float acc = 0.f;
#pragma unroll
        for (int w = 0; w < NORM_WARPS; ++w) acc += red[w][c];
        float* dst = (which == 0 ? part_dgamma : part_dbeta) + static_cast<size_t>(blockIdx.x) * H + i * 256 + c;
        *dst = acc;
      }
    }
  }
}

// bf16 activations, bandwidth-oriented variant of the kernel above (same maths, same outputs).  The first version kept
// x̂ and g·γ of a row as 2 x VPL x 8 floats across the two warp reductions and fetched the residual gradient afterwards:
// 191 registers → one 8-warp block per SM, and three dependent memory phases per row, about twice the time its memory
// traffic needs.  Here a row's x, gy and residual gradient are
// fetched together as raw 16-byte vectors (3 x VPL x 4 registers), unpacked twice (before and after the reductions:
// ALU is free here), and blocks are 4 warps at <= 168 registers → 12 warps per SM with 12 loads each in flight.
constexpr int NORM_BWD_WARPS = 4;

template <typename W, int VPL, bool RMS>
__global__ void __launch_bounds__(NORM_BWD_WARPS * 32, 3)
norm_bwd_bf16_kernel(const __nv_bfloat16* __restrict__ gy, const __nv_bfloat16* __restrict__ x, const W* __restrict__ gamma,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in, __nv_bfloat16* __restrict__ gx,
                     float* __restrict__ part_dgamma, float* __restrict__ part_dbeta, int rows,
                     const __nv_bfloat16* __restrict__ gadd) {
  constexpr int H = VPL * 256;
  __shared__ float red[NORM_BWD_WARPS][32 * 8 + 8];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  float dg[VPL][8], db[VPL][8];
#pragma unroll
  for (int i = 0; i < VPL; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dg[i][j] = db[i][j] = 0.f;
  // (γ is re-read from L1 in both passes instead of living in VPL x 8 registers)
  auto unpack8 = [](const uint4& q, float (&v)[8]) {
    const float2 a = unpack_bf16(q.x), b = unpack_bf16(q.y), c = unpack_bf16(q.z), d = unpack_bf16(q.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  };

  for (int row = blockIdx.x * NORM_BWD_WARPS + warp; row < rows; row += gridDim.x * NORM_BWD_WARPS) {
    const size_t base = static_cast<size_t>(row) * H;
    uint4 xq[VPL], gq[VPL], aq[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      xq[i] = *reinterpret_cast<const uint4*>(x + base + (i * 32 + lane) * 8);
      gq[i] = *reinterpret_cast<const uint4*>(gy + base + (i * 32 + lane) * 8);
    }
    if (gadd != nullptr) {
#pragma unroll
      for (int i = 0; i < VPL; ++i) aq[i] = *reinterpret_cast<const uint4*>(gadd + base + (i * 32 + lane) * 8);
    }
    const float mean = RMS ? 0.f : mean_in[row];
    const float rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      float xv[8], gv[8], gm[8];
      unpack8(xq[i], xv);
      unpack8(gq[i], gv);
      Vec8<W>::load(gamma + (i * 32 + lane) * 8, gm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (xv[j] - mean) * rstd;
        const float gw = gv[j] * gm[j];
        s1 += gw;
        s2 += gw * xh;
        dg[i][j] += gv[j] * xh;
        db[i][j] += gv[j];
      }
    }
    s1 = RMS ? 0.f : warp_sum(s1) * (1.0f / H);
    s2 = warp_sum(s2) * (1.0f / H);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      float xv[8], gv[8], gm[8], o[8];
      unpack8(xq[i], xv);
      unpack8(gq[i], gv);
      Vec8<W>::load(gamma + (i * 32 + lane) * 8, gm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (xv[j] - mean) * rstd;
        o[j] = rstd * (gv[j] * gm[j] - s1 - xh * s2);
      }
      if (gadd != nullptr) {  // the skip connection's gradient rides along: saves autograd's separate add kernel
        float a[8];
        unpack8(aq[i], a);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += a[j];
      }
      Vec8<__nv_bfloat16>::store(gx + base + (i * 32 + lane) * 8, o);
    }
  }
  // block-level reduction of the per-warp column partials, one vector slot at a time
  for (int i = 0; i < VPL; ++i) {
    for (int which = 0; which < (part_dbeta != nullptr ? 2 : 1); ++which) {
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = which == 0 ? dg[i][j] : db[i][j];
      __syncthreads();
      for (int c = threadIdx.x; c < 256; c += NORM_BWD_WARPS * 32) {
        float acc = 0.f;
#pragma unroll
        for (int w = 0; w < NORM_BWD_WARPS; ++w) acc += red[w][c];
        float* dst = (which == 0 ? part_dgamma : part_dbeta) + static_cast<size_t>(blockIdx.x) * H + i * 256 + c;
        *dst = acc;
      }
    }
  }
}

// out[c] = sum_r part[r, c]   (block = 32 columns x 8 row stripes, smem tree over the stripes)
// blockIdx.y selects (part0 -> out0) / (part1 -> out1): dgamma and dbeta in one launch; `accumulate` adds into `out`
// (each column is owned by exactly one thread, so the fp32 main-grad buffer is updated with a plain read-modify-write)
__global__ void __launch_bounds__(256) colreduce_kernel(const float* __restrict__ part0, float* __restrict__ out0,
                                                        const float* __restrict__ part1, float* __restrict__ out1,
                                                        int nrows, int H, int accumulate) {
  const float* __restrict__ part = blockIdx.y == 0 ? part0 : part1;
  float* __restrict__ out = blockIdx.y == 0 ? out0 : out1;
  __shared__ float sm[8][33];
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  const int c = blockIdx.x * 32 + tx;
  float acc = 0.f;
  if (c < H) {
    int r = ty;
    for (; r + 24 < nrows; r += 32) {
      const float a0 = part[static_cast<size_t>(r) * H + c], a1 = part[static_cast<size_t>(r + 8) * H + c];
      const float a2 = part[static_cast<size_t>(r + 16) * H + c], a3 = part[static_cast<size_t>(r + 24) * H + c];
      acc += (a0 + a1) + (a2 + a3);
    }
    for (; r < nrows; r += 8) acc += part[static_cast<size_t>(r) * H + c];
  }
  sm[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < H) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += sm[j][tx];
    out[c] = accumulate ? out[c] + t : t;
  }
}

// ---------------- generic (any H) fallbacks: one warp per row, strided scalar access ----------------
template <typename T, typename W, bool RMS>
__global__ void norm_fwd_generic(const T* __restrict__ x, const W* __restrict__ gamma, const W* __restrict__ beta,
                                 T* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                 int rows, int H, float eps) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int row = blockIdx.x * (blockDim.x / 32) + warp;
  if (row >= rows) return;
  const T* xr = x + static_cast<size_t>(row) * H;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) s += static_cast<float>(xr[c]);
  const float mean = RMS ? 0.f : warp_sum(s) / H;
  float sq = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float d = static_cast<float>(xr[c]) - mean;
    sq += d * d;
  }
  const float rstd = rsqrtf(warp_sum(sq) / H + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
  T* yr = y + static_cast<size_t>(row) * H;
  for (int c = lane; c < H; c += 32) {
    float o = (static_cast<float>(xr[c]) - mean) * rstd * static_cast<float>(gamma[c]);
    if (beta != nullptr) o += static_cast<float>(beta[c]);
    yr[c] = static_cast<T>(o);
  }
}

// gx only; dγ / dβ come from norm_bwd_colpart_generic + colreduce_kernel
template <typename T, typename W, bool RMS>
__global__ void norm_bwd_generic(const T* __restrict__ gy, const T* __restrict__ x, const W* __restrict__ gamma,
                                 const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                 T* __restrict__ gx, int rows, int H) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int row = blockIdx.x * (blockDim.x / 32) + warp;
  if (row >= rows) return;
  const float mean = RMS ? 0.f : mean_in[row], rstd = rstd_in[row];
  const T* xr = x + static_cast<size_t>(row) * H;
  const T* gr = gy + static_cast<size_t>(row) * H;
  float s1 = 0.f, s2 = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float xh = (static_cast<float>(xr[c]) - mean) * rstd;
    const float gw = static_cast<float>(gr[c]) * static_cast<float>(gamma[c]);
    s1 += gw;
    s2 += gw * xh;
  }
  s1 = RMS ? 0.f : warp_sum(s1) / H;
  s2 = warp_sum(s2) / H;
  T* gxr = gx + static_cast<size_t>(row) * H;
  for (int c = lane; c < H; c += 32) {
    const float xh = (static_cast<float>(xr[c]) - mean) * rstd;
    const float gw = static_cast<float>(gr[c]) * static_cast<float>(gamma[c]);
    gxr[c] = static_cast<T>(rstd * (gw - s1 - xh * s2));
  }
}

// part_dgamma[blockIdx.y, c] = Σ g·x̂ and part_dbeta[blockIdx.y, c] = Σ g over rows [blockIdx.y * rows_per_block, +
// rows_per_block): one thread per column, rows in increasing order, so the sums colreduce_kernel makes of the partials
// do not depend on scheduling (atomics would make dγ / dβ differ from run to run in the last bits)
template <typename T, bool RMS>
__global__ void __launch_bounds__(256)
norm_bwd_colpart_generic(const T* __restrict__ gy, const T* __restrict__ x, const float* __restrict__ mean_in,
                         const float* __restrict__ rstd_in, float* __restrict__ part_dgamma,
                         float* __restrict__ part_dbeta, int rows, int H, int rows_per_block) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(rows, r0 + rows_per_block);
  float dg = 0.f, db = 0.f;
  for (int r = r0; r < r1; ++r) {
    const float mean = RMS ? 0.f : mean_in[r];
    const float g = static_cast<float>(gy[static_cast<size_t>(r) * H + c]);
    dg += g * ((static_cast<float>(x[static_cast<size_t>(r) * H + c]) - mean) * rstd_in[r]);
    db += g;
  }
  part_dgamma[static_cast<size_t>(blockIdx.y) * H + c] = dg;
  if (part_dbeta != nullptr) part_dbeta[static_cast<size_t>(blockIdx.y) * H + c] = db;
}

}  // namespace lb

namespace {
int norm_grid(int rows) {
  const int need = (rows + lb::NORM_WARPS - 1) / lb::NORM_WARPS;
  const int cap = lb_host::num_sms() * 2;
  return need < cap ? need : cap;
}
// forward: 64 registers → four 8-warp blocks per SM
int norm_fwd_grid(int rows) {
  const int need = (rows + lb::NORM_WARPS - 1) / lb::NORM_WARPS;
  const int cap = lb_host::num_sms() * 4;
  return need < cap ? need : cap;
}
// bf16 backward: three 4-warp blocks per SM (one wave; every block leaves one row of column partials)
int norm_bwd_bf16_grid(int rows) {
  const int need = (rows + lb::NORM_BWD_WARPS - 1) / lb::NORM_BWD_WARPS;
  const int cap = lb_host::num_sms() * 3;
  return need < cap ? need : cap;
}

template <typename T, typename W, bool RMS>
bool fwd_dispatch(int vpl, const T* x, const W* g, const W* b, T* y, float* mean, float* rstd, int rows, float eps,
                  cudaStream_t s) {
  const int grid = norm_fwd_grid(rows);
#define LB_CASE(V)                                                                                             \
  case V:                                                                                                      \
    lb::norm_fwd_kernel<T, W, V, RMS><<<grid, lb::NORM_WARPS * 32, 0, s>>>(x, g, b, y, mean, rstd, rows, eps); \
    return true;
  switch (vpl) {
    LB_CASE(1) LB_CASE(2) LB_CASE(3) LB_CASE(4) LB_CASE(5) LB_CASE(6) LB_CASE(8) LB_CASE(10) LB_CASE(12) LB_CASE(16)
    LB_CASE(20) LB_CASE(32)
    default:
      return false;
  }
#undef LB_CASE
}

template <typename W, bool RMS>
bool bwd_dispatch_bf16(int vpl, const __nv_bfloat16* gy, const __nv_bfloat16* x, const W* g, const float* mean,
                       const float* rstd, __nv_bfloat16* gx, float* pdg, float* pdb, int rows, int grid, cudaStream_t s,
                       const __nv_bfloat16* gadd) {
#define LB_CASE(V)                                                                                                        \
  case V:                                                                                                                 \
    lb::norm_bwd_bf16_kernel<W, V, RMS><<<grid, lb::NORM_BWD_WARPS * 32, 0, s>>>(gy, x, g, mean, rstd, gx, pdg, pdb, rows, gadd); \
    return true;
  switch (vpl) {
    LB_CASE(1) LB_CASE(2) LB_CASE(3) LB_CASE(4)
    default:
      return false;
  }
#undef LB_CASE
}
// H <= 1024 with bf16 activations takes the bandwidth-oriented kernel (wider rows would spill at 168 registers)
bool norm_bwd_uses_bf16_kernel(int H, int dtype) { return dtype == 0 && H % 256 == 0 && H / 256 <= 4; }

template <typename T, typename W, bool RMS>
bool bwd_dispatch(int vpl, const T* gy, const T* x, const W* g, const float* mean, const float* rstd, T* gx, float* pdg,
                  float* pdb, int rows, int grid, cudaStream_t s, const T* gadd) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    if (norm_bwd_uses_bf16_kernel(vpl * 256, 0))
      return bwd_dispatch_bf16<W, RMS>(vpl, gy, x, g, mean, rstd, gx, pdg, pdb, rows, grid, s, gadd);
  }
#define LB_CASE(V)                                                                                                   \
  case V:                                                                                                            \
    lb::norm_bwd_kernel<T, W, V, RMS><<<grid, lb::NORM_WARPS * 32, 0, s>>>(gy, x, g, mean, rstd, gx, pdg, pdb, rows, gadd); \
    return true;
  switch (vpl) {
    LB_CASE(1) LB_CASE(2) LB_CASE(3) LB_CASE(4) LB_CASE(5) LB_CASE(6) LB_CASE(8) LB_CASE(10) LB_CASE(12) LB_CASE(16)
    default:
      return false;
  }
#undef LB_CASE
}
}  // namespace

// dtype codes: 0 = bf16 activations, 1 = fp32 activations; wdtype: 0 = bf16 params, 1 = fp32 params
extern "C" int lb_norm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                           int rows, int H, float eps, int rms, int dtype, int wdtype, cudaStream_t s) {
  if (rows == 0) return 0;
  const bool fast = (H % 256 == 0);
  bool done = false;
#define LB_GO(T, W)                                                                                                   \
  {                                                                                                                   \
    if (fast) {                                                                                                       \
      done = rms ? fwd_dispatch<T, W, true>(H / 256, (const T*)x, (const W*)gamma, (const W*)beta, (T*)y, mean, rstd, \
                                            rows, eps, s)                                                             \
                 : fwd_dispatch<T, W, false>(H / 256, (const T*)x, (const W*)gamma, (const W*)beta, (T*)y, mean,      \
                                             rstd, rows, eps, s);                                                     \
    }                                                                                                                 \
    if (!done) {                                                                                                      \
      const int wpb = 8;                                                                                              \
      const int grid = (rows + wpb - 1) / wpb;                                                                        \
      if (rms)                                                                                                        \
        lb::norm_fwd_generic<T, W, true><<<grid, wpb * 32, 0, s>>>((const T*)x, (const W*)gamma, (const W*)beta,      \
                                                                   (T*)y, mean, rstd, rows, H, eps);                  \
      else                                                                                                            \
        lb::norm_fwd_generic<T, W, false><<<grid, wpb * 32, 0, s>>>((const T*)x, (const W*)gamma, (const W*)beta,     \
                                                                    (T*)y, mean, rstd, rows, H, eps);                 \
    }                                                                                                                 \
  }
  if (dtype == 0 && wdtype == 0) LB_GO(__nv_bfloat16, __nv_bfloat16)
  else if (dtype == 0 && wdtype == 1) LB_GO(__nv_bfloat16, float)
  else if (dtype == 1 && wdtype == 1) LB_GO(float, float)
  else return -1;
#undef LB_GO
  return (int)cudaGetLastError();
}

// workspace: float[2 * grid_cap * H] where grid_cap = lb_norm_bwd_workspace_rows(); dgamma/dbeta fp32 [H]
extern "C" int lb_norm_bwd_workspace_rows(int rows) {
  const int a = norm_grid(rows), b = norm_bwd_bf16_grid(rows);
  return a > b ? a : b;
}
// the fused "+ residual gradient" is implemented by the register-cached kernel only (H = 256 * {1..6, 8, 10, 12, 16})
extern "C" int lb_norm_bwd_supports_gadd(int H) {
  if (H % 256 != 0) return 0;
  const int v = H / 256;
  return (v >= 1 && v <= 6) || v == 8 || v == 10 || v == 12 || v == 16;
}

extern "C" int lb_norm_bwd(const void* gy, const void* x, const void* gamma, const float* mean, const float* rstd,
                           void* gx, float* dgamma, float* dbeta, float* workspace, int rows, int H, int rms, int dtype,
                           int wdtype, int accumulate, const void* gadd, cudaStream_t s) {
  if (rows == 0) return 0;
  const bool fast = (H % 256 == 0) && (H / 256 <= 16);
  if (gadd != nullptr && !lb_norm_bwd_supports_gadd(H)) return -3;  // caller adds the residual gradient itself
  const int grid = norm_bwd_uses_bf16_kernel(H, dtype) ? norm_bwd_bf16_grid(rows) : norm_grid(rows);
  bool done = false;
  float* pdg = workspace;
  float* pdb = dbeta != nullptr ? workspace + static_cast<size_t>(grid) * H : nullptr;
#define LB_GO(T, W)                                                                                                  \
  {                                                                                                                  \
    if (fast) {                                                                                                      \
      done = rms ? bwd_dispatch<T, W, true>(H / 256, (const T*)gy, (const T*)x, (const W*)gamma, mean, rstd, (T*)gx, \
                                            pdg, pdb, rows, grid, s, (const T*)gadd)           \
                 : bwd_dispatch<T, W, false>(H / 256, (const T*)gy, (const T*)x, (const W*)gamma, mean, rstd,        \
                                             (T*)gx, pdg, pdb, rows, grid, s, (const T*)gadd); \
      if (done) {                                                                            \
        lb::colreduce_kernel<<<dim3((H + 31) / 32, dbeta != nullptr ? 2 : 1), 256, 0, s>>>(pdg, dgamma, pdb, dbeta, grid, \
                                                                                           H, accumulate);           \
      }                                                                                                              \
    }                                                                                                                \
    if (!done) {                                                                                                     \
      const int wpb = 8;                                                                                             \
      const int g2 = (rows + wpb - 1) / wpb;                                                                         \
      /* column partials over `grid` (<= workspace rows) fixed row blocks */                                         \
      const int rpb = (rows + grid - 1) / grid;                                                                      \
      const int nparts = (rows + rpb - 1) / rpb;                                                                     \
      const dim3 pgrid((H + 255) / 256, nparts);                                                                     \
      if (rms) {                                                                                                     \
        lb::norm_bwd_generic<T, W, true><<<g2, wpb * 32, 0, s>>>((const T*)gy, (const T*)x, (const W*)gamma, mean,   \
                                                                 rstd, (T*)gx, rows, H);                             \
        lb::norm_bwd_colpart_generic<T, true><<<pgrid, 256, 0, s>>>((const T*)gy, (const T*)x, mean, rstd, pdg, pdb, \
                                                                    rows, H, rpb);                                   \
      } else {                                                                                                       \
        lb::norm_bwd_generic<T, W, false><<<g2, wpb * 32, 0, s>>>((const T*)gy, (const T*)x, (const W*)gamma, mean,  \
                                                                  rstd, (T*)gx, rows, H);                            \
        lb::norm_bwd_colpart_generic<T, false><<<pgrid, 256, 0, s>>>((const T*)gy, (const T*)x, mean, rstd, pdg,     \
                                                                     pdb, rows, H, rpb);                             \
      }                                                                                                              \
      lb::colreduce_kernel<<<dim3((H + 31) / 32, dbeta != nullptr ? 2 : 1), 256, 0, s>>>(pdg, dgamma, pdb, dbeta,    \
                                                                                         nparts, H, accumulate);     \
    }                                                                                                                \
  }
  if (dtype == 0 && wdtype == 0) LB_GO(__nv_bfloat16, __nv_bfloat16)
  else if (dtype == 0 && wdtype == 1) LB_GO(__nv_bfloat16, float)
  else if (dtype == 1 && wdtype == 1) LB_GO(float, float)
  else return -1;
#undef LB_GO
  return (int)cudaGetLastError();
}
