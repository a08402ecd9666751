// Shifted-window attention (Swin, SwinV2) on sm_90a, read straight from the image-ordered qkv projection.
//
// qkv [B, H*W, 3, heads, d] (the qkv Linear applied to the image-ordered tokens), O [B, H*W, heads, d].  Local position
// (i, j) of window (wy, wx) is the token ((wy*ws + i + s) mod H, (wx*ws + j + s) mod W): this is roll(-s) -> window
// partition -> attention -> window reverse -> roll(+s), with no copy of the activations.
//
// Score of query p against key q of one window and head h:
//   z = sc * <q_p, k_q> + T[rel(p, q), h] + m(p, q)
//   rel = (y_p - y_q + ws - 1) * (2ws - 1) + (x_p - x_q + ws - 1) from the local coordinates (relative_position_index);
//   m = -100 when the shift is on and the two tokens' region labels differ (shifted_window_mask).  The label of rolled-
//   frame row r = wy*ws + i is 0 if r < H - ws, 1 if r < H - s and 2 otherwise; columns alike; label = 3*row + col.
//   Plain mode: sc = scale.  Cosine mode (SwinV2): q and k are normalised in fp32 (x / max(|x|, 1e-12), F.normalize),
//   sc = tau_h, and <q^, k^> is formed from bf16 hi/lo splits (hi*hi + hi*lo + lo*hi, fp32 accumulation): a single bf16
//   product would move logits scaled by tau up to 100 by about tau * 2^-8.
// No bias or mask tensor exists: the table column of the head lives in shared memory, labels are computed per token.
//
// One CTA of min(NP / 16, 4) warps per (window, head) in the forward.  The window's q/k/v rows (d <= 64 columns,
// zero-padded to DP, a multiple of 16) are gathered with 16-byte loads into padded shared-memory rows (rows wrap at the
// shift, so TMA boxes do not fit); N = ws^2 rows are padded to NP, a multiple of 16.  Each warp takes 16-row blocks
// and runs mma.sync m16n8k16 over 64-key chunks with an online softmax (one chunk, so no rescaling, for ws <= 8).  P is
// rounded to bf16 for P.V.  The lse (log2 units) is saved for the backward.
//
// Backward, per (window, head), recomputing P from the lse:
//   delta, warps own query rows:  delta_i = sum_j P_ij dP_ij with dP = dO V^T, from the same fp32 P and dP as dS below,
//                                 so that sum_j dS_ij = 0 holds to fp32 rounding (rowsum(dO * O) of the bf16 O would
//                                 leave a per-row bias that the table and tau gradients, sums of dS, accumulate)
//   pass A, warps own key rows:   dV = P^T dO, dK = sc * dS^T Q   with dS = P * (dP - delta)
//   pass B, warps own query rows: dQ = sc * dS K, and dS itself for the table gradient (and dtau = sum dS <q^, k^>)
// In cosine mode dQ and dK then go through the normalisation Jacobian, (g - x^ <x^, g>) / |x| (or g / 1e-12 when the
// norm is clamped).  Every element of dqkv is written exactly once: no zero-fill, no atomics.
// Table gradient: a CTA walks a fixed contiguous range of windows for one head and keeps sum dS per (i, j), each
// element owned by one thread, then writes it to a fp32 partial [G, heads, N, N]; window_dt_sum_kernel adds the G
// partials in order and window_dt_fold_kernel folds (i, j) into table entries in order.  G depends only on (windows,
// heads), so the result is bit-identical from run to run and on any device.
//
// Bandwidth: one (window, head) at N = 49, d = 32 moves ~12.5 KB of q/k/v/o for ~0.5 MFLOP of padded MMA work, far
// below the bf16 ridge of the H100, so mma.sync on plain row-major shared-memory tiles is enough (no wgmma).
#include "common.cuh"

namespace lb {
namespace wa {

// One warp per 16-row block of the padded window, at most kFwdWarps / kBwdWarps (NP / 16 is 1, 4, 9 or 16 for windows
// up to 4, 8, 12 and 16).  The forward keeps 4 warps and ~100 registers so that several CTAs share an SM; the backward
// holds one CTA per SM at ws >= 12 (registers, shared memory), where 9 warps give every block of ws 12 its own warp.
constexpr int kFwdWarps = 4;
constexpr int kBwdWarps = 9;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kMaskValue = -100.f;
constexpr float kNormEps = 1e-12f;

struct Params {
  const __nv_bfloat16* qkv;    // [B, H*W, 3, heads, d]
  const __nv_bfloat16* dout;   // [B, H*W, heads, d]
  __nv_bfloat16* out;          // forward: O
  __nv_bfloat16* dqkv;         // backward: [B, H*W, 3, heads, d]
  float* lse;                  // [nwin, heads, N], log2 units
  const float* table;          // [(2ws - 1)^2, heads]
  const float* tau;            // [heads] (cosine mode) or null
  float* dt_part;              // [G, heads, N, N]
  float* dtau_part;            // [G, heads]
  int H, W, ws, shift, heads, d, N, NP, nWx, nW, nwin, per, tbl;
  float scale;
};

// The backward keeps its running sum of dS over the windows of the CTA in shared memory up to ws = 12 ([N][N] fp32, at
// most 81 KB) and in its global partial slice beyond.
__host__ __device__ inline bool smem_dt(int NP) { return NP <= 144; }

// shared memory: bf16 row buffers Q, K, V (then Q lo, K lo in cosine mode, then dO in the backward), each [NP][DP + 8]
// (rows start 4 banks apart: ldmatrix is conflict-free), then the fp32 table column [tbl], six [NP] arrays and
// (backward, smem_dt) the dS sum.
template <int DP, bool COS>
struct Layout {
  static constexpr int kRow = DP + 8;
  __host__ __device__ static int bufs(bool bwd) { return 3 + (COS ? 2 : 0) + (bwd ? 1 : 0); }
  __host__ __device__ static int bytes(int NP, int tbl, bool bwd) {
    return bufs(bwd) * NP * kRow * 2 + (tbl + 6 * NP) * 4 + (bwd && smem_dt(NP) ? NP * NP * 4 : 0);
  }
};

template <int DP, bool COS>
struct Smem {
  __nv_bfloat16 *q, *k, *v, *qlo, *klo, *dout;
  float* T;
  int* meta;     // rel-position coordinate | region label << 16 of each local index
  int* tok;      // token of each local index (-1: padding row)
  float *delta, *lse, *nq, *nk;
  LB_DEVICE Smem(unsigned char* base, int NP, int tbl, bool bwd) {
    constexpr int R = Layout<DP, COS>::kRow;
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(base);
    q = b;
    k = b + NP * R;
    v = b + 2 * NP * R;
    qlo = COS ? b + 3 * NP * R : q;
    klo = COS ? b + 4 * NP * R : k;
    dout = b + (COS ? 5 : 3) * NP * R;
    T = reinterpret_cast<float*>(b + Layout<DP, COS>::bufs(bwd) * NP * R);
    meta = reinterpret_cast<int*>(T + tbl);
    tok = meta + NP;
    delta = reinterpret_cast<float*>(tok + NP);
    lse = delta + NP;
    nq = lse + NP;
    nk = nq + NP;
  }
};

// Gathers window w of head h into shared memory (and, in the backward, dO and the lse); cosine mode replaces Q
// and K by the hi parts of the normalised rows and fills the lo buffers.  Ends with a CTA barrier.
template <int DP, bool COS, bool BWD>
LB_DEVICE void load_window(const Params& p, const Smem<DP, COS>& s, int w, int h) {
  constexpr int R = Layout<DP, COS>::kRow;
  const int b = w / p.nW, wi = w - b * p.nW, wy = wi / p.nWx, wx = wi - wy * p.nWx;
  for (int i = threadIdx.x; i < p.NP; i += blockDim.x) {
    int t = -1, meta = 0;
    if (i < p.N) {
      const int yi = i / p.ws, xi = i - yi * p.ws;
      const int ry = wy * p.ws + yi, rx = wx * p.ws + xi;   // rolled frame
      const int y = ry + p.shift < p.H ? ry + p.shift : ry + p.shift - p.H;
      const int x = rx + p.shift < p.W ? rx + p.shift : rx + p.shift - p.W;
      t = (b * p.H + y) * p.W + x;
      const int ly = ry < p.H - p.ws ? 0 : (ry < p.H - p.shift ? 1 : 2);
      const int lx = rx < p.W - p.ws ? 0 : (rx < p.W - p.shift ? 1 : 2);
      meta = (yi * (2 * p.ws - 1) + xi) | ((3 * ly + lx) << 16);
    }
    s.tok[i] = t;
    s.meta[i] = meta;
  }
  __syncthreads();
  constexpr int nch = DP / 8;
  const int dch = p.d / 8;
  const long C = (long)p.heads * p.d;
  for (int e = threadIdx.x; e < p.NP * nch; e += blockDim.x) {
    const int r = e / nch, c = e - r * nch;
    const int t = s.tok[r];
    const bool ok = t >= 0 && c < dch;
    const long base = (long)t * 3 * C + (long)h * p.d + c * 8;
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(s.q + r * R + c * 8) = ok ? *reinterpret_cast<const uint4*>(p.qkv + base) : z;
    *reinterpret_cast<uint4*>(s.k + r * R + c * 8) = ok ? *reinterpret_cast<const uint4*>(p.qkv + base + C) : z;
    *reinterpret_cast<uint4*>(s.v + r * R + c * 8) = ok ? *reinterpret_cast<const uint4*>(p.qkv + base + 2 * C) : z;
    if (BWD)
      *reinterpret_cast<uint4*>(s.dout + r * R + c * 8) =
          ok ? *reinterpret_cast<const uint4*>(p.dout + (long)t * C + (long)h * p.d + c * 8) : z;
  }
  if (BWD) {
    for (int r = threadIdx.x; r < p.NP; r += blockDim.x) {
      const int t = s.tok[r];
      s.lse[r] = t >= 0 ? p.lse[((long)w * p.heads + h) * p.N + r] : 0.f;
    }
  }
  __syncthreads();
  if (COS) {
    for (int task = threadIdx.x; task < 2 * p.NP; task += blockDim.x) {
      const int r = task % p.NP;
      __nv_bfloat16* x = (task < p.NP ? s.q : s.k) + r * R;
      __nv_bfloat16* xl = (task < p.NP ? s.qlo : s.klo) + r * R;
      float ss = 0.f;
      for (int c = 0; c < p.d; ++c) {
        const float f = __bfloat162float(x[c]);
        ss = fmaf(f, f, ss);
      }
      const float n = sqrtf(ss);
      const float inv = 1.f / fmaxf(n, kNormEps);
      for (int c = 0; c < DP; ++c) {
        const float f = __bfloat162float(x[c]) * inv;
        const __nv_bfloat16 hi = __float2bfloat16(f);
        x[c] = hi;
        xl[c] = __float2bfloat16(f - __bfloat162float(hi));
      }
      if (BWD) (task < p.NP ? s.nq : s.nk)[r] = n;
    }
    __syncthreads();
  }
}

// A fragments (16 rows from row0, all DP columns) of a row buffer
template <int DP>
LB_DEVICE void load_a(uint32_t (&a)[DP / 16][4], const __nv_bfloat16* buf, int row0, int lane) {
  constexpr int R = DP + 8;
#pragma unroll
  for (int ks = 0; ks < DP / 16; ++ks) ldsm_x4(a[ks], buf + (row0 + (lane & 15)) * R + ks * 16 + (lane >> 4) * 8);
}

// acc[n] += A(16 rows) . B(rows col0 + 8n ..)^T over DP: B rows are the columns of the product.  COS adds the hi*lo and
// lo*hi products.  Columns at or past NP are skipped (their accumulators stay as they were).
template <int DP, int NT, bool COS>
LB_DEVICE void mma_abt(float (&acc)[NT][4], const uint32_t (&ah)[DP / 16][4], const uint32_t (&al)[DP / 16][4],
                       const __nv_bfloat16* bh, const __nv_bfloat16* bl, int col0, int NP, int lane) {
  constexpr int R = DP + 8;
  const int br = (lane & 7) + ((lane >> 4) << 3), bc = ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int t = 0; t < NT / 2; ++t) {
    if (col0 + 16 * t < NP) {
#pragma unroll
      for (int ks = 0; ks < DP / 16; ++ks) {
        uint32_t b[4];
        ldsm_x4(b, bh + (col0 + 16 * t + br) * R + ks * 16 + bc);
        mma_bf16(acc[2 * t], ah[ks], b[0], b[1]);
        mma_bf16(acc[2 * t + 1], ah[ks], b[2], b[3]);
        if (COS) {
          mma_bf16(acc[2 * t], al[ks], b[0], b[1]);
          mma_bf16(acc[2 * t + 1], al[ks], b[2], b[3]);
          ldsm_x4(b, bl + (col0 + 16 * t + br) * R + ks * 16 + bc);
          mma_bf16(acc[2 * t], ah[ks], b[0], b[1]);
          mma_bf16(acc[2 * t + 1], ah[ks], b[2], b[3]);
        }
      }
    }
  }
}

// o += P(16 rows x 16 keys from key0, A fragment) . V(rows key0 .., all DP columns)
template <int DP>
LB_DEVICE void mma_pv(float (&o)[DP / 8][4], const uint32_t (&pa)[4], const __nv_bfloat16* vb, int key0, int lane) {
  constexpr int R = DP + 8;
  const int vr = key0 + (lane & 7) + (((lane >> 3) & 1) << 3), vc = (lane >> 4) * 8;
#pragma unroll
  for (int j = 0; j < DP / 16; ++j) {
    uint32_t b[4];
    ldsm_x4_t(b, vb + vr * R + j * 16 + vc);
    mma_bf16(o[2 * j], pa, b[0], b[1]);
    mma_bf16(o[2 * j + 1], pa, b[2], b[3]);
  }
}

// A fragment of columns 16t .. 16t + 15 of a C-fragment array (rows r0 and r0 + 8)
template <int NT>
LB_DEVICE void pack_a(uint32_t (&a)[4], const float (&c)[NT][4], int t) {
  a[0] = pack_bf16(c[2 * t][0], c[2 * t][1]);
  a[1] = pack_bf16(c[2 * t][2], c[2 * t][3]);
  a[2] = pack_bf16(c[2 * t + 1][0], c[2 * t + 1][1]);
  a[3] = pack_bf16(c[2 * t + 1][2], c[2 * t + 1][3]);
}

// z (natural units) of query meta mq against key meta mk
LB_DEVICE float score(float acc, float sc, int mq, int mk, const float* T, int rel0, bool shifted) {
  float z = fmaf(sc, acc, T[(mq & 0xffff) - (mk & 0xffff) + rel0]);
  if (shifted && (mq >> 16) != (mk >> 16)) z += kMaskValue;
  return z;
}

// Writes sc * g (rows row0 + r0 and row0 + r0 + 8 of a [16 x DP] C-fragment array) to slot `slot` of dqkv; cosine mode
// applies the normalisation Jacobian with x^ = hi + lo and the row norms `nrm`.
template <int DP, bool COS>
LB_DEVICE void store_grad(const Params& p, const int* tok, float (&g)[DP / 8][4], float sc,
                          const __nv_bfloat16* hi, const __nv_bfloat16* lo, const float* nrm, int row0, int slot, int h,
                          int lane) {
  constexpr int R = DP + 8;
  const int r0 = lane >> 2, c0 = (lane & 3) * 2;
  const long C = (long)p.heads * p.d;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int row = row0 + r0 + 8 * half;
    float dot = 0.f;
    if (COS) {
#pragma unroll
      for (int n = 0; n < DP / 8; ++n) {
        const int col = n * 8 + c0;
        const float x0 = __bfloat162float(hi[row * R + col]) + __bfloat162float(lo[row * R + col]);
        const float x1 = __bfloat162float(hi[row * R + col + 1]) + __bfloat162float(lo[row * R + col + 1]);
        dot = fmaf(g[n][2 * half], x0, fmaf(g[n][2 * half + 1], x1, dot));
      }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    }
    if (row < p.N) {
      const int t = tok[row];
      const float n = COS ? nrm[row] : 1.f;
      const bool clamped = COS && !(n > kNormEps);
      const float rn = COS ? 1.f / fmaxf(n, kNormEps) : 1.f;
      __nv_bfloat16* dst = p.dqkv + (long)t * 3 * C + slot * C + (long)h * p.d;
#pragma unroll
      for (int nn = 0; nn < DP / 8; ++nn) {
        const int col = nn * 8 + c0;
        if (col < p.d) {
          float v0 = sc * g[nn][2 * half], v1 = sc * g[nn][2 * half + 1];
          if (COS) {
            if (!clamped) {
              const float x0 = __bfloat162float(hi[row * R + col]) + __bfloat162float(lo[row * R + col]);
              const float x1 = __bfloat162float(hi[row * R + col + 1]) + __bfloat162float(lo[row * R + col + 1]);
              v0 = fmaf(-sc * dot, x0, v0);
              v1 = fmaf(-sc * dot, x1, v1);
            }
            v0 *= rn;
            v1 *= rn;
          }
          *reinterpret_cast<uint32_t*>(dst + col) = pack_bf16(v0, v1);
        }
      }
    }
  }
}

template <int DP, bool COS>
__global__ void __launch_bounds__(kFwdWarps * 32, 1) window_attn_fwd_kernel(const Params p) {
  extern __shared__ __align__(16) unsigned char smem[];
  const Smem<DP, COS> s(smem, p.NP, p.tbl, false);
  const int w = blockIdx.x, h = blockIdx.y;
  for (int e = threadIdx.x; e < p.tbl; e += blockDim.x) s.T[e] = p.table[e * p.heads + h];
  load_window<DP, COS, false>(p, s, w, h);
  const float sc = COS ? p.tau[h] : p.scale;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int r0 = lane >> 2, c0 = (lane & 3) * 2;
  const bool shifted = p.shift > 0;
  const int rel0 = (p.ws - 1) * 2 * p.ws;
  const long C = (long)p.heads * p.d;
  for (int rb = warp * 16; rb < p.NP; rb += nwarps * 16) {
    uint32_t ah[DP / 16][4], al[DP / 16][4];
    load_a<DP>(ah, s.q, rb, lane);
    if (COS) load_a<DP>(al, s.qlo, rb, lane);
    const int mq[2] = {s.meta[rb + r0], s.meta[rb + r0 + 8]};
    float o[DP / 8][4];
#pragma unroll
    for (int n = 0; n < DP / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    for (int kc = 0; kc < p.NP; kc += 64) {
      float sa[8][4];
#pragma unroll
      for (int n = 0; n < 8; ++n) sa[n][0] = sa[n][1] = sa[n][2] = sa[n][3] = 0.f;
      mma_abt<DP, 8, COS>(sa, ah, al, s.k, s.klo, kc, p.NP, lane);
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = kc + n * 8 + c0 + (j & 1);
          const float z = col < p.N ? score(sa[n][j], sc, mq[j >> 1], s.meta[col], s.T, rel0, shifted) * kLog2e
                                    : -INFINITY;
          sa[n][j] = z;
          mx[j >> 1] = fmaxf(mx[j >> 1], z);
        }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m[r], mx[r]);   // finite: every chunk holds at least one real key
        alpha[r] = fast_exp2(m[r] - mn);
        m[r] = mn;
        l[r] *= alpha[r];
      }
#pragma unroll
      for (int n = 0; n < DP / 8; ++n) {
        o[n][0] *= alpha[0];
        o[n][1] *= alpha[0];
        o[n][2] *= alpha[1];
        o[n][3] *= alpha[1];
      }
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          sa[n][j] = fast_exp2(sa[n][j] - m[j >> 1]);
          l[j >> 1] += sa[n][j];
        }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (kc + 16 * t < p.NP) {
          uint32_t pa[4];
          pack_a<8>(pa, sa, t);
          mma_pv<DP>(o, pa, s.v, kc + 16 * t, lane);
        }
      }
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      float L = l[half];
      L += __shfl_xor_sync(0xffffffffu, L, 1);
      L += __shfl_xor_sync(0xffffffffu, L, 2);
      const int row = rb + r0 + 8 * half;
      if (row < p.N) {
        const int t = s.tok[row];
        const float inv = 1.f / L;
        __nv_bfloat16* dst = p.out + (long)t * C + (long)h * p.d;
#pragma unroll
        for (int n = 0; n < DP / 8; ++n) {
          const int col = n * 8 + c0;
          if (col < p.d)
            *reinterpret_cast<uint32_t*>(dst + col) = pack_bf16(o[n][2 * half] * inv, o[n][2 * half + 1] * inv);
        }
        if ((lane & 3) == 0) p.lse[((long)w * p.heads + h) * p.N + row] = m[half] + __log2f(L);
      }
    }
  }
}

template <int DP, bool COS>
__global__ void __launch_bounds__(kBwdWarps * 32, 1) window_attn_bwd_kernel(const Params p) {
  extern __shared__ __align__(16) unsigned char smem[];
  const Smem<DP, COS> s(smem, p.NP, p.tbl, true);
  __shared__ float red[kBwdWarps];
  constexpr int NT = DP >= 48 ? 2 : 4;   // key / query columns per step, in 8-column MMA tiles (registers at DP >= 48)
  const int g = blockIdx.x, h = blockIdx.y;
  for (int e = threadIdx.x; e < p.tbl; e += blockDim.x) s.T[e] = p.table[e * p.heads + h];
  const float sc = COS ? p.tau[h] : p.scale;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int r0 = lane >> 2, c0 = (lane & 3) * 2;
  const bool shifted = p.shift > 0;
  const int rel0 = (p.ws - 1) * 2 * p.ws;
  const int w0 = g * p.per, w1 = min(w0 + p.per, p.nwin);
  float* part = p.dt_part + ((long)g * p.heads + h) * p.N * p.N;
  float* dsum = smem_dt(p.NP) ? s.nk + p.NP : part;   // [N][N]: each element read and written by one thread only
  float dtau = 0.f;
  for (int w = w0; w < w1; ++w) {
    __syncthreads();   // the previous window's shared memory has been read
    load_window<DP, COS, true>(p, s, w, h);

    // delta of every query row
    for (int rb = warp * 16; rb < p.NP; rb += nwarps * 16) {
      uint32_t qh[DP / 16][4], ql[DP / 16][4], of[DP / 16][4];
      load_a<DP>(qh, s.q, rb, lane);
      if (COS) load_a<DP>(ql, s.qlo, rb, lane);
      load_a<DP>(of, s.dout, rb, lane);
      const int mq[2] = {s.meta[rb + r0], s.meta[rb + r0 + 8]};
      const float lr[2] = {s.lse[rb + r0], s.lse[rb + r0 + 8]};
      float dl[2] = {0.f, 0.f};
      for (int kc = 0; kc < p.NP; kc += NT * 8) {
        float sa[NT][4], dp[NT][4];
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) sa[n][j] = dp[n][j] = 0.f;
        mma_abt<DP, NT, COS>(sa, qh, ql, s.k, s.klo, kc, p.NP, lane);
        mma_abt<DP, NT, false>(dp, of, of, s.v, s.v, kc, p.NP, lane);
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = kc + n * 8 + c0 + (j & 1);
            if (col < p.N) {
              const float z = score(sa[n][j], sc, mq[j >> 1], s.meta[col], s.T, rel0, shifted);
              dl[j >> 1] = fmaf(fast_exp2(z * kLog2e - lr[j >> 1]), dp[n][j], dl[j >> 1]);
            }
          }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        dl[r] += __shfl_xor_sync(0xffffffffu, dl[r], 1);
        dl[r] += __shfl_xor_sync(0xffffffffu, dl[r], 2);
      }
      if ((lane & 3) == 0) {
        s.delta[rb + r0] = dl[0];
        s.delta[rb + r0 + 8] = dl[1];
      }
    }
    __syncthreads();

    // pass A: warps own key rows -> dK, dV
    for (int rb = warp * 16; rb < p.NP; rb += nwarps * 16) {
      uint32_t kh[DP / 16][4], kl[DP / 16][4], vf[DP / 16][4];
      load_a<DP>(kh, s.k, rb, lane);
      if (COS) load_a<DP>(kl, s.klo, rb, lane);
      load_a<DP>(vf, s.v, rb, lane);
      const int mk[2] = {s.meta[rb + r0], s.meta[rb + r0 + 8]};
      float dk[DP / 8][4], dv[DP / 8][4];
#pragma unroll
      for (int n = 0; n < DP / 8; ++n)
#pragma unroll
        for (int j = 0; j < 4; ++j) dk[n][j] = dv[n][j] = 0.f;
      for (int qc = 0; qc < p.NP; qc += NT * 8) {
        float st[NT][4], dp[NT][4];
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) st[n][j] = dp[n][j] = 0.f;
        mma_abt<DP, NT, COS>(st, kh, kl, s.q, s.qlo, qc, p.NP, lane);
        mma_abt<DP, NT, false>(dp, vf, vf, s.dout, s.dout, qc, p.NP, lane);
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = qc + n * 8 + c0 + (j & 1);   // query
            float pr = 0.f, ds = 0.f;
            if (col < p.N) {
              const float z = score(st[n][j], sc, s.meta[col], mk[j >> 1], s.T, rel0, shifted);
              pr = fast_exp2(z * kLog2e - s.lse[col]);
              ds = pr * (dp[n][j] - s.delta[col]);
            }
            st[n][j] = pr;
            dp[n][j] = ds;
          }
#pragma unroll
        for (int t = 0; t < NT / 2; ++t) {
          if (qc + 16 * t < p.NP) {
            uint32_t a[4];
            pack_a<NT>(a, st, t);
            mma_pv<DP>(dv, a, s.dout, qc + 16 * t, lane);
            pack_a<NT>(a, dp, t);
            mma_pv<DP>(dk, a, s.q, qc + 16 * t, lane);
          }
        }
      }
      store_grad<DP, false>(p, s.tok, dv, 1.f, nullptr, nullptr, nullptr, rb, 2, h, lane);
      store_grad<DP, COS>(p, s.tok, dk, sc, s.k, s.klo, s.nk, rb, 1, h, lane);
    }

    // pass B: warps own query rows -> dQ, dS for the table gradient and dtau
    for (int rb = warp * 16; rb < p.NP; rb += nwarps * 16) {
      uint32_t qh[DP / 16][4], ql[DP / 16][4], of[DP / 16][4];
      load_a<DP>(qh, s.q, rb, lane);
      if (COS) load_a<DP>(ql, s.qlo, rb, lane);
      load_a<DP>(of, s.dout, rb, lane);
      const int mq[2] = {s.meta[rb + r0], s.meta[rb + r0 + 8]};
      const float lr[2] = {s.lse[rb + r0], s.lse[rb + r0 + 8]};
      const float dr[2] = {s.delta[rb + r0], s.delta[rb + r0 + 8]};
      const bool live[2] = {rb + r0 < p.N, rb + r0 + 8 < p.N};
      float dq[DP / 8][4];
#pragma unroll
      for (int n = 0; n < DP / 8; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;
      for (int kc = 0; kc < p.NP; kc += NT * 8) {
        float sa[NT][4], dp[NT][4];
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) sa[n][j] = dp[n][j] = 0.f;
        mma_abt<DP, NT, COS>(sa, qh, ql, s.k, s.klo, kc, p.NP, lane);
        mma_abt<DP, NT, false>(dp, of, of, s.v, s.v, kc, p.NP, lane);
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = kc + n * 8 + c0 + (j & 1);   // key
            const int r = j >> 1;
            float ds = 0.f;
            if (col < p.N) {
              const float z = score(sa[n][j], sc, mq[r], s.meta[col], s.T, rel0, shifted);
              ds = fast_exp2(z * kLog2e - lr[r]) * (dp[n][j] - dr[r]);
              if (live[r]) {
                float* a = dsum + (rb + r0 + 8 * r) * p.N + col;
                *a = w == w0 ? ds : *a + ds;
                if (COS) dtau = fmaf(ds, sa[n][j], dtau);
              }
            }
            sa[n][j] = ds;
          }
#pragma unroll
        for (int t = 0; t < NT / 2; ++t) {
          if (kc + 16 * t < p.NP) {
            uint32_t a[4];
            pack_a<NT>(a, sa, t);
            mma_pv<DP>(dq, a, s.k, kc + 16 * t, lane);
          }
        }
      }
      store_grad<DP, COS>(p, s.tok, dq, sc, s.q, s.qlo, s.nq, rb, 0, h, lane);
    }
  }
  if (dsum != part) {
    __syncthreads();
    for (int e = threadIdx.x; e < p.N * p.N; e += blockDim.x) part[e] = dsum[e];
  }
  if (COS) {
    dtau = warp_sum(dtau);
    if (lane == 0) red[warp] = dtau;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < nwarps; ++i) t += red[i];
      p.dtau_part[(long)g * p.heads + h] = t;
    }
  }
}

// part[0 .. n) = sum over g of part[g * n + e], in g order (in place into the g = 0 slice)
__global__ void window_dt_sum_kernel(float* part, int G, long n) {
  for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < n; e += (long)gridDim.x * blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int g = 0;
    for (; g + 8 <= G; g += 8)
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] += part[(long)(g + u) * n + e];
    for (int u = 0; g < G; ++g, ++u) acc[u] += part[(long)g * n + e];
    part[e] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
  }
}

// dtable[e, h] = sum over query i (in order) of S[h, i, j(i, e)], S = the summed partial [heads, N, N]; dtau[h] = sum
// over g of dtau_part[g, h]
__global__ void window_dt_fold_kernel(const float* S, const float* dtau_part, float* dtable, float* dtau, int G,
                                      int heads, int ws, int N, int tbl) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= tbl * heads) return;
  const int e = idx / heads, h = idx - e * heads;
  const int span = 2 * ws - 1;
  const int dy = e / span - (ws - 1), dx = e % span - (ws - 1);
  float acc = 0.f;
  for (int i = 0; i < N; ++i) {
    const int yi = i / ws, xi = i - yi * ws;
    const int yj = yi - dy, xj = xi - dx;
    if (yj >= 0 && yj < ws && xj >= 0 && xj < ws) acc += S[((long)h * N + i) * N + yj * ws + xj];
  }
  dtable[idx] = acc;
  if (dtau != nullptr && e == 0) {
    float t = 0.f;
    for (int g = 0; g < G; ++g) t += dtau_part[(long)g * heads + h];
    dtau[h] = t;
  }
}

}  // namespace wa
}  // namespace lb

namespace {
using lb::wa::Params;

Params window_params(int B, int H, int W, int ws, int shift, int heads, int d, float scale) {
  Params p{};
  p.H = H;
  p.W = W;
  p.ws = ws;
  p.shift = shift;
  p.heads = heads;
  p.d = d;
  p.N = ws * ws;
  p.NP = (p.N + 15) / 16 * 16;
  p.nWx = W / ws;
  p.nW = (H / ws) * p.nWx;
  p.nwin = B * p.nW;
  p.tbl = (2 * ws - 1) * (2 * ws - 1);
  p.scale = scale;
  return p;
}

// windows per backward CTA: about 2048 CTAs over all heads, from the shape alone
int window_per(int nwin, int heads) {
  int g0 = 2048 / heads;
  g0 = g0 < 1 ? 1 : (g0 > nwin ? nwin : g0);
  return (nwin + g0 - 1) / g0;
}

template <int DP, bool COS>
cudaError_t launch_window(const Params& p, bool bwd, cudaStream_t s) {
  using L = lb::wa::Layout<DP, COS>;
  const int bytes = L::bytes(p.NP, p.tbl, bwd);
  static int configured[2] = {0, 0};   // the dynamic shared memory each kernel has been opted into
  auto fwd_kern = lb::wa::window_attn_fwd_kernel<DP, COS>;
  auto bwd_kern = lb::wa::window_attn_bwd_kernel<DP, COS>;
  if (bytes > configured[bwd]) {
    cudaError_t e = bwd ? cudaFuncSetAttribute(bwd_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)
                        : cudaFuncSetAttribute(fwd_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    configured[bwd] = bytes;
  }
  const int most = bwd ? lb::wa::kBwdWarps : lb::wa::kFwdWarps;
  const int threads = 32 * (p.NP / 16 < most ? p.NP / 16 : most);
  if (bwd) {
    const int G = (p.nwin + p.per - 1) / p.per;
    bwd_kern<<<dim3(G, p.heads), threads, bytes, s>>>(p);
  } else {
    fwd_kern<<<dim3(p.nwin, p.heads), threads, bytes, s>>>(p);
  }
  return cudaGetLastError();
}

cudaError_t dispatch_window(const Params& p, bool bwd, cudaStream_t s) {
  const bool cos = p.tau != nullptr;
  switch ((p.d + 15) / 16) {
    case 1: return cos ? launch_window<16, true>(p, bwd, s) : launch_window<16, false>(p, bwd, s);
    case 2: return cos ? launch_window<32, true>(p, bwd, s) : launch_window<32, false>(p, bwd, s);
    case 3: return cos ? launch_window<48, true>(p, bwd, s) : launch_window<48, false>(p, bwd, s);
    case 4: return cos ? launch_window<64, true>(p, bwd, s) : launch_window<64, false>(p, bwd, s);
    default: return cudaErrorInvalidValue;
  }
}
}  // namespace

// number of fp32 [heads, N, N] table-gradient partials the backward of this shape writes
extern "C" int lb_window_attn_groups(int B, int H, int W, int ws, int heads) {
  const int nwin = B * (H / ws) * (W / ws);
  if (nwin == 0) return 0;
  const int per = window_per(nwin, heads);
  return (nwin + per - 1) / per;
}

extern "C" int lb_window_attn_fwd(const void* qkv, void* out, float* lse, const float* table, const float* tau, int B,
                                  int H, int W, int ws, int shift, int heads, int d, float scale, cudaStream_t s) {
  Params p = window_params(B, H, W, ws, shift, heads, d, scale);
  if (p.nwin == 0) return 0;
  p.qkv = static_cast<const __nv_bfloat16*>(qkv);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.lse = lse;
  p.table = table;
  p.tau = tau;
  return (int)dispatch_window(p, false, s);
}

extern "C" int lb_window_attn_bwd(const void* dout, const void* qkv, const float* lse, const float* table,
                                  const float* tau, void* dqkv, float* dtable, float* dtau, float* dt_part,
                                  float* dtau_part, int B, int H, int W, int ws, int shift, int heads, int d,
                                  float scale, cudaStream_t s) {
  Params p = window_params(B, H, W, ws, shift, heads, d, scale);
  if (p.nwin == 0) return 0;
  p.dout = static_cast<const __nv_bfloat16*>(dout);
  p.qkv = static_cast<const __nv_bfloat16*>(qkv);
  p.lse = const_cast<float*>(lse);
  p.table = table;
  p.tau = tau;
  p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
  p.dt_part = dt_part;
  p.dtau_part = dtau_part;
  p.per = window_per(p.nwin, heads);
  const int G = (p.nwin + p.per - 1) / p.per;
  cudaError_t e = dispatch_window(p, true, s);
  if (e != cudaSuccess) return (int)e;
  const long n = (long)heads * p.N * p.N;
  const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  lb::wa::window_dt_sum_kernel<<<blocks, 256, 0, s>>>(dt_part, G, n);
  const int cells = p.tbl * heads;
  lb::wa::window_dt_fold_kernel<<<(cells + 127) / 128, 128, 0, s>>>(dt_part, dtau_part, dtable, tau ? dtau : nullptr, G,
                                                                    heads, ws, p.N, p.tbl);
  return (int)cudaGetLastError();
}
