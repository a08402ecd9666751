// Shared device helpers for the sm_90a kernels: mbarrier, TMA, wgmma PTX wrappers.
// Everything is inline PTX (no CUTLASS dependency) so the kernels compile in seconds.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace lb {

#define LB_DEVICE __device__ __forceinline__

// ---------------------------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------------------------
LB_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

LB_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// cross-GPU flag waits (NVLink peer memory).  Every wait is BOUNDED: a dead or wedged peer must not hang the GPU
// forever — after `timeout_ns` the waiter records who/what it was waiting for and traps, which surfaces
// as a CUDA error on the host (the trainer's emergency path / the launcher's restart then take over).
//
// The timeout path makes no function call (no printf, no assert, no __noinline__ helper): a call anywhere in a kernel
// that issues wgmma makes ptxas wait for every wgmma to complete before the next one issues (warning C7510), which
// the build treats as an error.  The diagnostic goes to a record in host-mapped pinned memory instead, which the host
// can still read after the trap has destroyed the context (lb_host::spin_timeout_record, read by lb_spin_timeout_report).
// ---------------------------------------------------------------------------------------------
struct SpinTimeout {
  uint32_t claimed;            // the first waiter to time out owns the record
  uint32_t set;                // the fields below are complete
  int kind, who, block;
  uint32_t value, target;
  unsigned long long flag;     // address of the flag that was waited on
};
LB_DEVICE unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
  return t;
}
LB_DEVICE uint32_t ld_acquire_sys_u32(const uint32_t* a) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(a) : "memory");
  return v;
}
LB_DEVICE uint32_t ld_acquire_gpu_u32(const uint32_t* a) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(a) : "memory");
  return v;
}
template <bool SYS>
LB_DEVICE uint32_t ld_acquire_u32(const uint32_t* a) {
  return SYS ? ld_acquire_sys_u32(a) : ld_acquire_gpu_u32(a);
}
constexpr unsigned long long kDefaultSpinTimeoutNs = 120ull * 1000ull * 1000ull * 1000ull;  // 2 min
// wait until *addr >= target (wrap-safe signed distance), polling with system-scope (SYS: flags written by a peer GPU)
// or GPU-scope acquire loads; `what`/`who` only label the diagnostic written to `rec` (may be null: then the waiter
// traps without a record)
template <bool SYS>
LB_DEVICE void spin_wait_ge(const uint32_t* addr, uint32_t target, unsigned long long timeout_ns, SpinTimeout* rec,
                            int what, int who) {
  if (static_cast<int32_t>(ld_acquire_u32<SYS>(addr) - target) >= 0) return;
  const unsigned long long t0 = globaltimer_ns();
  const unsigned long long budget = timeout_ns ? timeout_ns : kDefaultSpinTimeoutNs;
  uint32_t polls = 0;
  while (static_cast<int32_t>(ld_acquire_u32<SYS>(addr) - target) < 0) {
    if ((++polls & 1023u) == 0 && globaltimer_ns() - t0 > budget) {
      if (rec != nullptr && atomicCAS(&rec->claimed, 0u, 1u) == 0u) {
        rec->kind = what;
        rec->who = who;
        rec->block = static_cast<int>(blockIdx.x);
        rec->value = ld_acquire_u32<SYS>(addr);
        rec->target = target;
        rec->flag = reinterpret_cast<unsigned long long>(addr);
        __threadfence_system();
        *reinterpret_cast<volatile uint32_t*>(&rec->set) = 1u;
        __threadfence_system();
      }
      asm volatile("trap;");
    }
  }
}
LB_DEVICE void spin_wait_ge_sys(const uint32_t* addr, uint32_t target, unsigned long long timeout_ns, SpinTimeout* rec,
                                int what, int who) {
  spin_wait_ge<true>(addr, target, timeout_ns, rec, what, who);
}
LB_DEVICE void spin_wait_ge_gpu(const uint32_t* addr, uint32_t target, unsigned long long timeout_ns, SpinTimeout* rec,
                                int what, int who) {
  spin_wait_ge<false>(addr, target, timeout_ns, rec, what, who);
}

// ---------------------------------------------------------------------------------------------
// counter-based RNG for dropout: Philox4x32 (7 rounds — passes BigCrush, Salmon et al. 2011) keyed by the PyTorch CUDA
// generator's (seed, offset) and indexed by ELEMENT POSITION, so forward, backward and any re-tiling regenerate the
// same mask.  The (seed, offset) pair comes from `at::CUDAGeneratorImpl::philox_cuda_state`: plain values in eager
// mode, device pointers + an intra-graph offset while a CUDA graph is being captured (PyTorch rewrites the pointed-to
// values before every replay) — so captured transformer blocks draw fresh masks on every replay.
// `salt` distinguishes tensor-parallel ranks in sharded regions (0 in replicated regions: identical masks).
// ---------------------------------------------------------------------------------------------
struct RngArgs {
  unsigned long long seed_val, offset_val;   // eager: the values
  const long long* seed_ptr;                 // capture: where PyTorch keeps them
  const long long* offset_ptr;
  unsigned int offset_intragraph;
  int captured;
  unsigned long long salt;
};
LB_DEVICE void rng_resolve(const RngArgs& a, unsigned long long& seed, unsigned long long& offset) {
  if (a.captured) {
    seed = static_cast<unsigned long long>(*a.seed_ptr);
    offset = static_cast<unsigned long long>(*a.offset_ptr) + a.offset_intragraph;
  } else {
    seed = a.seed_val;
    offset = a.offset_val;
  }
  seed ^= a.salt * 0x9E3779B97F4A7C15ull;
}
LB_DEVICE uint4 philox4x32_7(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
LB_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
LB_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
LB_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

LB_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
LB_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
LB_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
LB_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) – 2D / 3D tiled loads into shared memory, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
LB_DEVICE void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
LB_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
LB_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
LB_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2,
                           int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
LB_DEVICE void tma_load_5d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1, int32_t c2,
                           int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
      "[%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// shared -> global tiled store (bulk async group completion)
LB_DEVICE void tma_store_2d(const CUtensorMap* map, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
LB_DEVICE void tma_store_4d(const CUtensorMap* map, const void* smem_src, int32_t c0, int32_t c1, int32_t c2,
                            int32_t c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// global[dst .. dst + bytes) += shared[src ..] (fp32 element-wise adds, one bulk operation; 16-byte aligned, bytes a
// multiple of 16), bulk async group completion
LB_DEVICE void bulk_reduce_add_f32(float* dst, const float* src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;\n" ::"l"(dst),
               "r"(smem_u32(src)), "r"(bytes)
               : "memory");
}
LB_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
template <int N>
LB_DEVICE void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
template <int N>
LB_DEVICE void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, accumulators in registers)
// ---------------------------------------------------------------------------------------------
LB_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
LB_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
LB_DEVICE void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
LB_DEVICE void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over the 128 threads of one warpgroup (ids 1..4 are reserved for this)
LB_DEVICE void warpgroup_sync(int wg) { asm volatile("bar.sync %0, 128;\n" ::"r"(wg + 1) : "memory"); }

// shared-memory matrix descriptor for wgmma, 128-byte swizzle (bit layout: PTX ISA "Matrix Descriptor Format"):
//   start address [0,14) (>>4), LBO [16,30) (>>4), SBO [32,46) (>>4), layout = 1 (128B swizzle) [62,64)
// K-major tiles (rows of 64 bf16 = 128 bytes): SBO = 1024 (8-row groups), advance 32 bytes per 16 elements of K.
// MN-major tiles (64-element MN atoms, one 128-byte row per k): LBO = distance between MN atoms, SBO = 1024.
LB_DEVICE uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ---------------------------------------------------------------------------------------------
// mma.sync m16n8k16 (bf16 in, fp32 accumulators) and its ldmatrix operand loads
// ---------------------------------------------------------------------------------------------
LB_DEVICE void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
LB_DEVICE void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
LB_DEVICE void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------------
// numeric helpers
// ---------------------------------------------------------------------------------------------
LB_DEVICE uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
LB_DEVICE float2 unpack_bf16(uint32_t u) {
  // a bf16 is the upper half of an fp32: one shift for the low element, one mask for the high one (the intrinsic
  // compiled to PRMT + IMAD for the high half)
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

// one Adam step of one element, shared by fused_adamw and the ZeRO update: g = grad * scale (+ wd * p when the weight
// decay is coupled), fp32 moments m, v, bias corrections bc1, bc2; decoupled weight decay adds wd * p to the update
LB_DEVICE void adam_element(float& p, float& m, float& v, float grad, float scale, float lr, float b1, float b2, float eps,
                            float wd, float bc1, float bc2, int decoupled) {
  float g = grad * scale;
  if (!decoupled) g += wd * p;
  m = b1 * m + (1.0f - b1) * g;
  v = b2 * v + (1.0f - b2) * g * g;
  float upd = (m / bc1) / (sqrtf(v / bc2) + eps);
  if (decoupled) upd += wd * p;
  p -= lr * upd;
}

enum Act : int { ACT_NONE = 0, ACT_GELU = 1, ACT_GELU_TANH = 2, ACT_RELU = 3, ACT_SILU = 4, ACT_QUICK_GELU = 5,
                 ACT_RESADD = 6 /* GEMM epilogue only: out = acc (+ bias) + pre_in, i.e. the residual add */ };

// erfc(|x|/sqrt2) and exp(-x^2/2) from one MUFU.EX2 + one MUFU.RCP (Abramowitz-Stegun 7.1.26, |err(erf)| < 1.5e-7 -
// three orders of magnitude below bf16 resolution).  The libm erff costs ~60 instructions with a divergent branch,
// which made the 4-warp GEMM epilogue (one thread per accumulator row) the bottleneck of the h->4h projection.
LB_DEVICE void gelu_terms(float x, float& erfc_abs, float& gauss) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.72134752044448170f));  // exp(-x^2/2)
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  erfc_abs = poly * t * e;
  gauss = e;
}
LB_DEVICE float gelu_fast(float x) {
  float q, e;
  gelu_terms(x, q, e);
  const float h = 0.5f * q;                 // 0.5 * erfc(|x|/sqrt2)
  return x * (x >= 0.f ? 1.0f - h : h);     // no cancellation on the negative side
}
LB_DEVICE float gelu_grad_fast(float x) {
  float q, e;
  gelu_terms(x, q, e);
  const float h = 0.5f * q;
  const float cdf = x >= 0.f ? 1.0f - h : h;
  return fmaf(x * 0.3989422804014327f, e, cdf);
}
// 2^x on the SFU without the denormal-range fix-up branch that exp2f() compiles to (one BSSY/BRA/BSYNC triple per
// element in the softmax loops); ex2.approx(-inf) = +0.
LB_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
LB_DEVICE float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

LB_DEVICE float act_fwd(float x, int act) {
  switch (act) {
    case ACT_GELU:
      return gelu_fast(x);
    case ACT_GELU_TANH: {
      float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
      return 0.5f * x * (1.0f + tanh_fast(u));
    }
    case ACT_RELU:
      return x > 0.f ? x : 0.f;
    case ACT_SILU:
      return x / (1.0f + __expf(-x));
    case ACT_QUICK_GELU:
      return x / (1.0f + __expf(-1.702f * x));
    default:
      return x;
  }
}
// d act(x) / dx
LB_DEVICE float act_grad(float x, int act) {
  switch (act) {
    case ACT_GELU:
      return gelu_grad_fast(x);
    case ACT_GELU_TANH: {
      float x2 = x * x;
      float u = 0.7978845608028654f * (x + 0.044715f * x * x2);
      float t = tanh_fast(u);
      float du = 0.7978845608028654f * (1.0f + 3.0f * 0.044715f * x2);
      return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
    }
    case ACT_RELU:
      return x > 0.f ? 1.f : 0.f;
    case ACT_SILU: {
      float s = 1.0f / (1.0f + __expf(-x));
      return s * (1.0f + x * (1.0f - s));
    }
    case ACT_QUICK_GELU: {
      float s = 1.0f / (1.0f + __expf(-1.702f * x));
      return s * (1.0f + 1.702f * x * (1.0f - s));
    }
    default:
      return 1.f;
  }
}

LB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
LB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace lb

// ---------------------------------------------------------------------------------------------
// host: tensor-map creation through the driver entry point (no -lcuda link dependency)
// ---------------------------------------------------------------------------------------------
namespace lb_host {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_tiled();
// rank-`rank` bf16 tensor; dims/strides innermost first (strides in bytes, strides[0] implied = 2)
bool make_tmap_typed(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle);
bool make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, CUtensorMapSwizzle swizzle);
// the process-wide lb::SpinTimeout record (host-mapped pinned memory, allocated on first use); null when it does not
// exist yet and `s` is being captured into a CUDA graph, or when the allocation failed
lb::SpinTimeout* spin_timeout_record(cudaStream_t s);
}  // namespace lb_host
