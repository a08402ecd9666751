// In-kernel NVLink collectives over peer-mapped (symmetric) memory, fused with the adjacent compute.
//
//   zero_reduce_scatter : each rank pulls its slice of the fp32 gradient bucket from every peer
//                         (P2P loads over NVLink), sums, scales, writes the reduced slice and the
//                         partial squared norm (for global-norm clipping)            [K3, first half]
//   zero_adam_allgather : AdamW on the owned slice (fp32 master, m, v) and the bf16 parameter slice is
//                         pushed straight into every peer's parameter buffer (P2P stores)  [K3 + K4]
//   NVLS                : when the buffers are bound to an NVSwitch multicast object (parallel/symm_mem.py), the reduce-
//                         scatter is ONE `multimem.ld_reduce` per 16 bytes — the switch adds the eight ranks' values and
//                         returns the sum, 1/8 of the inbound NVLink traffic of the pull form — and the parameter
//                         all-gather is ONE `multimem.st` per vector, replicated by the switch to every rank
//   device barrier      : release/acquire flag exchange at .sys scope with monotonically increasing
//                         epochs (no host synchronisation, survives CUDA-graph replay as long as the
//                         epoch is advanced per launch)
//
// These replace NCCL reduce-scatter -> multi-tensor Adam -> NCCL all-gather of the reference's ZeRO
// path (libai/models/utils/graph_base.py:69-70 + flow.optim.AdamW).
#include "common.cuh"

namespace lb {

constexpr int MAX_RANKS = 8;

struct PeerPtrs {
  void* p[MAX_RANKS];
};

// streaming 128-bit load (peer or local memory); NOT volatile so that several loads per thread stay in flight
LB_DEVICE float4 ld_stream_f4(const float4* p) {
  float4 v;
  // "memory": must not be hoisted above the barrier that follows the flag wait (it reads data other ranks publish)
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];\n"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// in-switch reduction of 4 floats over every device bound to the multicast object (NVLS)
LB_DEVICE float4 multimem_ld_reduce_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];\n"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
// one store, replicated by the switch into every bound device's memory (4 bf16 values)
LB_DEVICE void multimem_st_bf16x4(__nv_bfloat16* mc, uint2 v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.bf16x2 [%0], {%1, %2};\n" ::"l"(mc), "r"(v.x), "r"(v.y) : "memory");
}

LB_DEVICE void st_release_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(addr), "r"(v) : "memory");
}
LB_DEVICE uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(addr) : "memory");
  return v;
}

// Signal "rank reached epoch" into every peer's flag row and wait until every peer did the same.
// flags[q] points to rank q's flag array; slot `slot*world + r` holds the epoch last published by rank r.
LB_DEVICE void signal_peers(const PeerPtrs& flags, int world, int rank, int slot, uint32_t epoch) {
  __threadfence_system();
  for (int q = 0; q < world; ++q)
    st_release_sys(reinterpret_cast<uint32_t*>(flags.p[q]) + slot * world + rank, epoch);
}
LB_DEVICE void wait_peers(const PeerPtrs& flags, int world, int rank, int slot, uint32_t epoch, SpinTimeout* rec) {
  const uint32_t* mine = reinterpret_cast<const uint32_t*>(flags.p[rank]) + slot * world;
  // bounded (common.cuh): a dead peer turns into a device trap with a diagnostic instead of a hung GPU
  for (int q = 0; q < world; ++q) spin_wait_ge_sys(mine + q, epoch, 0ull, rec, /*what=*/10 + slot, q);
}

// ------------------------------------------------------------------------------------------------
// ZeRO reduce-scatter: red[i] = scale * sum_q grad_q[lo + i]   for i in [0, n)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
zero_reduce_scatter_kernel(PeerPtrs grads, PeerPtrs flags, float* __restrict__ red, float* __restrict__ sqnorm,
                           size_t lo, size_t n, float scale, int world, int rank, uint32_t epoch,
                           const float* __restrict__ mc_grad /* multicast address of the gradient buffers, or null */,
                           SpinTimeout* timeout_rec) {
  __shared__ float sm[8];
  if (blockIdx.x == 0 && threadIdx.x == 0) signal_peers(flags, world, rank, /*slot=*/0, epoch);
  if (threadIdx.x == 0) wait_peers(flags, world, rank, 0, epoch, timeout_rec);
  __syncthreads();
  const size_t nvec = n / 4;
  float acc_sq = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mc_grad != nullptr) {
      s = multimem_ld_reduce_f4(mc_grad + lo + i * 4);   // the switch returns the sum over all ranks
    } else {
      float4 part[MAX_RANKS];
#pragma unroll
      for (int q = 0; q < MAX_RANKS; ++q) {
        if (q < world) {
          // rotate the start so that the ranks do not all hammer the same peer at the same time
          const int src = (rank + q) % world;
          part[q] = ld_stream_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grads.p[src]) + lo) + i);
        }
      }
#pragma unroll
      for (int q = 0; q < MAX_RANKS; ++q) {
        if (q < world) {
          s.x += part[q].x; s.y += part[q].y; s.z += part[q].z; s.w += part[q].w;
        }
      }
    }
    s.x *= scale; s.y *= scale; s.z *= scale; s.w *= scale;
    reinterpret_cast<float4*>(red)[i] = s;
    acc_sq += s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w;
  }
  acc_sq = warp_sum(acc_sq);
  if (threadIdx.x % 32 == 0) sm[threadIdx.x / 32] = acc_sq;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? sm[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0 && sqnorm != nullptr) atomicAdd(sqnorm, t);
  }
}

// ------------------------------------------------------------------------------------------------
// AdamW on the owned slice + all-gather of the low-precision parameters by P2P stores
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
zero_adam_allgather_kernel(float* __restrict__ master, const float* __restrict__ red, float* __restrict__ m,
                           float* __restrict__ v, PeerPtrs params /* bf16 flat buffers */, PeerPtrs flags,
                           unsigned int* __restrict__ done_counter, const float* __restrict__ clip_ptr, size_t lo,
                           size_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2,
                           int decoupled, int world, int rank, uint32_t epoch,
                           __nv_bfloat16* __restrict__ mc_param /* multicast address of the parameter buffers, or null */,
                           SpinTimeout* timeout_rec) {
  const float clip = clip_ptr != nullptr ? *clip_ptr : 1.0f;
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float4 p4 = reinterpret_cast<float4*>(master)[i];
    const float4 g4 = reinterpret_cast<const float4*>(red)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i];
    float4 v4 = reinterpret_cast<float4*>(v)[i];
    float pp[4] = {p4.x, p4.y, p4.z, p4.w}, gg[4] = {g4.x, g4.y, g4.z, g4.w};
    float mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) adam_element(pp[j], mm[j], vv[j], gg[j], clip, lr, b1, b2, eps, wd, bc1, bc2, decoupled);
    reinterpret_cast<float4*>(master)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    const uint2 lp = make_uint2(pack_bf16(pp[0], pp[1]), pack_bf16(pp[2], pp[3]));
    if (mc_param != nullptr) {
      multimem_st_bf16x4(mc_param + lo + i * 4, lp);    // replicated to every rank (this one included) by the switch
    } else {
#pragma unroll 8
      for (int q = 0; q < world; ++q) {
        const int dst = (rank + q) % world;
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(params.p[dst]) + lo)[i] = lp;
      }
    }
  }
  // all CTAs done -> publish completion to every peer, then wait for theirs: when this kernel retires,
  // the local parameter buffer holds the updated slices of ALL ranks.
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      *done_counter = 0;
      signal_peers(flags, world, rank, /*slot=*/1, epoch);
      wait_peers(flags, world, rank, 1, epoch, timeout_rec);
    }
  }
}

// plain device-side barrier (used by tests and between phases that have no data dependency flag)
__global__ void device_barrier_kernel(PeerPtrs flags, int world, int rank, int slot, uint32_t epoch, SpinTimeout* timeout_rec) {
  if (threadIdx.x == 0) {
    signal_peers(flags, world, rank, slot, epoch);
    wait_peers(flags, world, rank, slot, epoch, timeout_rec);
  }
}

// all-gather by P2P stores: every rank pushes its shard into slot `rank` of every peer's buffer
__global__ void __launch_bounds__(256)
p2p_allgather_push_kernel(const uint4* __restrict__ shard, PeerPtrs outs, PeerPtrs flags, unsigned int* done_counter,
                          size_t nvec, int world, int rank, uint32_t epoch, SpinTimeout* timeout_rec) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = shard[i];
#pragma unroll 8
    for (int q = 0; q < world; ++q) {
      const int dst = (rank + q) % world;
      (reinterpret_cast<uint4*>(outs.p[dst]) + (size_t)rank * nvec)[i] = v;
    }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      *done_counter = 0;
      signal_peers(flags, world, rank, 2, epoch);
      wait_peers(flags, world, rank, 2, epoch, timeout_rec);
    }
  }
}

}  // namespace lb

namespace {
int comm_grid(size_t work) {
  size_t need = (work + 255) / 256;
  size_t cap = (size_t)lb_host::num_sms() * 4;
  return (int)(need < cap ? (need == 0 ? 1 : need) : cap);
}
lb::PeerPtrs to_peers(const long* ptrs, int world) {
  lb::PeerPtrs pp;
  for (int i = 0; i < lb::MAX_RANKS; ++i) pp.p[i] = i < world ? reinterpret_cast<void*>(ptrs[i]) : nullptr;
  return pp;
}
}  // namespace

extern "C" int lb_zero_reduce_scatter(const long* grad_ptrs, const long* flag_ptrs, float* red, float* sqnorm, long lo,
                                      long n, float scale, int world, int rank, unsigned epoch, long mc_grad,
                                      cudaStream_t s) {
  if (world > lb::MAX_RANKS || (n % 4) || (lo % 4)) return -1;
  lb::zero_reduce_scatter_kernel<<<comm_grid(n / 4), 256, 0, s>>>(to_peers(grad_ptrs, world), to_peers(flag_ptrs, world),
                                                                 red, sqnorm, (size_t)lo, (size_t)n, scale, world, rank,
                                                                 epoch, reinterpret_cast<const float*>(mc_grad),
                                                                 lb_host::spin_timeout_record(s));
  return (int)cudaGetLastError();
}

extern "C" int lb_zero_adam_allgather(float* master, const float* red, float* m, float* v, const long* param_ptrs,
                                      const long* flag_ptrs, unsigned* done_counter, const float* clip, long lo, long n,
                                      float lr, float b1, float b2, float eps, float wd, float bc1, float bc2,
                                      int decoupled, int world, int rank, unsigned epoch, long mc_param, cudaStream_t s) {
  if (world > lb::MAX_RANKS || (n % 4) || (lo % 4)) return -1;
  lb::zero_adam_allgather_kernel<<<comm_grid(n / 4), 256, 0, s>>>(
      master, red, m, v, to_peers(param_ptrs, world), to_peers(flag_ptrs, world), done_counter, clip, (size_t)lo,
      (size_t)n, lr, b1, b2, eps, wd, bc1, bc2, decoupled, world, rank, epoch,
      reinterpret_cast<__nv_bfloat16*>(mc_param), lb_host::spin_timeout_record(s));
  return (int)cudaGetLastError();
}

extern "C" int lb_device_barrier(const long* flag_ptrs, int world, int rank, int slot, unsigned epoch, cudaStream_t s) {
  lb::device_barrier_kernel<<<1, 32, 0, s>>>(to_peers(flag_ptrs, world), world, rank, slot, epoch,
                                             lb_host::spin_timeout_record(s));
  return (int)cudaGetLastError();
}

extern "C" int lb_p2p_allgather(const void* shard, const long* out_ptrs, const long* flag_ptrs, unsigned* done_counter,
                                long nbytes, int world, int rank, unsigned epoch, cudaStream_t s) {
  if (nbytes % 16) return -1;
  lb::p2p_allgather_push_kernel<<<comm_grid(nbytes / 16), 256, 0, s>>>(
      (const uint4*)shard, to_peers(out_ptrs, world), to_peers(flag_ptrs, world), done_counter, (size_t)(nbytes / 16),
      world, rank, epoch, lb_host::spin_timeout_record(s));
  return (int)cudaGetLastError();
}
