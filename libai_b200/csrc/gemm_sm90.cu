// Persistent warp-specialised bf16 GEMM for sm_90a: TMA -> shared (128B swizzle) -> wgmma (accumulators in
// registers) -> epilogue with fused bias / activation straight from the accumulator registers.
//
//   D[M,N] = A · Bᵀ   with three operand layouts (all row-major tensors in global memory):
//     NT: A[M,K], B[N,K]   (forward  : y  = x · Wᵀ)
//     NN: A[M,K], B[K,N]   (dgrad    : dx = dy · W,   B is "MN-major")
//     TN: A[K,M], B[K,N]   (wgrad    : dW = dyᵀ · x,  both "MN-major"; split-K + fp32 red.add)
//
// Replaces the cuBLAS matmuls behind libai/layers/linear.py:123-157 and the separate
// fused_bias_add_gelu kernel (libai/layers/mlp.py:95) of the reference.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (rows [0, 64) and [64, 128) of the 128-row tile; each
// issues m64nBLOCK_Nk16 wgmma over the shared stage and runs the epilogue of its rows), warp 8 = TMA producer.  One CTA
// per SM, static round-robin tile scheduler over (m_blk, n_blk, k_split).
//
// The bf16-output NT / NN GEMMs without a collective run gemm_pingpong_kernel below instead (384 threads, whole tiles
// per consumer warpgroup, TMA-store epilogue); gemm_impl decides which kernel a call takes.
#include "common.cuh"

#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <cstring>
#include <mutex>

namespace lb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;  // bf16 elements (= 32 bytes, also the 32 e4m3 elements of one fp8 wgmma)
constexpr int NUM_CONSUMER_THREADS = 256;
constexpr int NUM_THREADS = NUM_CONSUMER_THREADS + 32;
constexpr int PRODUCER_WARP = NUM_CONSUMER_THREADS / 32;

enum Epi : int { EPI_BF16 = 0, EPI_F32 = 1, EPI_ATOMIC_F32 = 2 };

struct GemmParams {
  int M, N, K;
  int k_splits;        // number of K partitions (atomic epilogue only when > 1)
  int k_per_split;     // in units of BLOCK_K blocks
  const __nv_bfloat16* bias;  // [N] or nullptr
  int act;                    // Act enum
  void* out;                  // bf16 or fp32 [M, ldo]
  __nv_bfloat16* pre_out;     // optional pre-activation copy (bf16)
  const __nv_bfloat16* pre_in;  // optional [M, ldo]: out = acc * act'(pre_in)  (dgrad fused with the activation backward)
  int ldo;                    // leading dimension of out (elements)
  int rmw;                    // EPI_F32: out += acc (plain read-modify-write; a tile is owned by one CTA)
  // fp8 (E4M3) operands, K-major only.  The byte layout of a [rows, K] e4m3 matrix equals that of a [rows, K/2] bf16
  // matrix, so the TMA maps, the 128-byte swizzle rows and the 32-byte descriptor advance per MMA are unchanged (K
  // above is in bf16-equivalent units = bytes / 2); only the MMA kind (kind::f8f6f4, 32 elements of K per instruction)
  // and the dequantisation scale in the epilogue differ.
  // optional fp32 [N] vector receiving the column sums of the bf16 output (`red.add`): the bias gradient of the layer
  // whose output gradient this GEMM produces (dgrad fused with the activation backward), without a second pass
  float* colsum;
  int fp8;
  const float* deq_a;         // per-tensor dequantisation scales (device scalars): out = acc * deq_a[0] * deq_b[0]
  const float* deq_b;
};

// Fused collective modes (tensor parallel): peer pointers refer to NVLink peer-mapped symmetric memory.
//   COMM_AG : all-gather -> GEMM.  One operand is the concatenation over ranks of [rows_per_rank, K] shards along its
//             row dimension: A for NT/NN (row blocks of the output), B for TN (`gathered_is_b`: the shards lie along
//             the REDUCTION dimension of the wgrad dW = dyᵀ · all_gather(x)).  Tiles / k-blocks that only need the local
//             shard read it through its own tensor map and start at once; `n_comm` dedicated CTAs push the local shard
//             into every peer's gathered buffer (TMA bulk copies over NVLink) meanwhile; per-row-block arrival counters
//             (bumped by the pushing peer) gate the TMA loads of the remote rows.
//   COMM_RS : GEMM -> reduce-scatter.  Each rank computes the full [M, N] partial product; the epilogue stores
//             row block tiles straight into the owner's staging slot (P2P stores) and bumps the owner's arrival
//             counter; after its tiles every CTA helps reducing the local rows (sum over sources + bias + residual).
// All handshake state lives in DEVICE memory and is advanced by the kernel itself (`state[0]` = number of completed
// calls on this buffer set): the launch parameters of a call site never change, so transformer blocks containing these
// kernels are captured into CUDA graphs and replayed.  Write-after-read safety of the symmetric buffers does not rely
// on any call-order convention: a rank publishes "finished call c" into every peer's `done` row when its kernel
// retires, and nobody writes call c+1 data into a peer's buffer before having seen that peer's "finished call c".
enum CommMode : int { COMM_NONE = 0, COMM_AG = 1, COMM_RS = 2 };
struct CommParams {
  int mode, world, rank;
  int rows_per_rank;            // rows of one shard, multiple of BLOCK_M
  int n_comm;                   // COMM_AG: number of copy CTAs
  int gathered_is_b;            // COMM_AG with the TN layout: the gathered operand is B, gated per k-block
  int fill_local;               // COMM_AG: the copy CTAs also write the local shard into the local gathered buffer
  int copy_rings;               // COMM_AG: independent copy engines (threads with their own smem ring) per copy CTA
  uint32_t arrivals;            // arrivals per row block and call (AG: 1; RS: world * n_blocks)
  uint32_t* state;              // local: [0] completed calls on this buffer set, [1] CTA exit counter
  __nv_bfloat16* peer_buf[8];   // AG: gathered buffers of all ranks; RS: staging buffers of all ranks
  uint32_t* peer_flags[8];      // per-row-block arrival counters of all ranks (AG: M/128 entries; RS: rows_per_rank/128)
  uint32_t* peer_done[8];       // [world] words on every rank: peer_done[q][r] = calls rank r has finished (written by r)
  const __nv_bfloat16* local_shard;  // AG: this rank's shard [rows_per_rank, K] (source of the pushes)
  const __nv_bfloat16* residual;  // RS: optional [rows_per_rank, N]
  __nv_bfloat16* rs_out;        // RS: [rows_per_rank, N]
  long staging_parity_off;      // RS: element offset of the staging half used by this call
  unsigned long long timeout_ns;  // bound of every cross-GPU flag wait (0 = default)
  SpinTimeout* timeout_rec;       // where a timed-out wait leaves its diagnostic (host-mapped)
};

// streaming (non-volatile, L1 no-allocate) 128-bit load: many of these stay in flight per thread over NVLink
LB_DEVICE uint4 ld_stream_u4(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

template <int BLOCK_N>
struct StageCfg {
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int NUM_STAGES = (BLOCK_N == 256) ? 4 : (BLOCK_N == 192 ? 5 : (BLOCK_N == 128 ? 6 : 8));
  static constexpr int AUX_BYTES = 1024;  // COMM_AG copy CTAs: the mbarriers of their copy rings
  static constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + AUX_BYTES;
};

template <int BLOCK_N, bool A_MN, bool B_MN, int EPI, bool FP8 = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_g /* COMM_AG: the local shard of the gathered operand */, GemmParams p,
            CommParams cp) {
  using Cfg = StageCfg<BLOCK_N>;
  constexpr int NS = Cfg::NUM_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NS * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + NS;
  uint8_t* aux = smem + NS * Cfg::STAGE_BYTES + 256;

  const int warp_idx = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

  const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int k_blocks_total = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int num_tiles = m_blocks * n_blocks * p.k_splits;
  // CTAs [0, n_comm) are copy CTAs in COMM_AG mode; the rest run the GEMM roles
  const int n_comm = (cp.mode == COMM_AG) ? cp.n_comm : 0;
  const int cta = static_cast<int>(blockIdx.x) - n_comm;
  const int cta_stride = static_cast<int>(gridDim.x) - n_comm;
  const int mbpr = cp.mode != COMM_NONE ? cp.rows_per_rank / BLOCK_M : m_blocks;
  const bool ag_b = cp.mode == COMM_AG && cp.gathered_is_b != 0;   // TN wgrad: shards along the reduction dimension
  // row blocks are visited owner by owner: AG starts with the local rows (already resident), RS ends with them
  auto map_m = [&](int m_seq) -> int {
    if (cp.mode == COMM_NONE || ag_b) return m_seq;
    const int shift = (cp.mode == COMM_AG) ? 0 : 1;
    const int owner = (cp.rank + shift + m_seq / mbpr) % cp.world;
    return owner * mbpr + m_seq % mbpr;
  };

  // work item -> (output tile, K partition).  Default: partitions of one tile are neighbours (their red.adds hit L2
  // together).  Gathered-B wgrad: partition-major, starting with the partitions that lie in the local shard (the host
  // makes k_splits a multiple of world and partitions never straddle a shard boundary), so every CTA has local work
  // while the remote shards are still in flight.
  const int mn_tiles = m_blocks * n_blocks;
  auto decode_tile = [&](int tile, int& mn, int& split) {
    if (ag_b) {
      mn = tile % mn_tiles;
      split = (tile / mn_tiles + cp.rank * (p.k_splits / cp.world)) % p.k_splits;
    } else {
      mn = tile / p.k_splits;
      split = tile % p.k_splits;
    }
  };
  // handshake epoch of this call: number of calls already completed on this buffer set (identical on all ranks; the
  // last CTA to leave advances it, i.e. nobody modifies it while any CTA of this launch may still read it)
  const uint32_t call_idx = cp.mode != COMM_NONE ? *reinterpret_cast<volatile const uint32_t*>(cp.state) : 0u;
  const uint32_t arrive_target = (call_idx + 1u) * cp.arrivals;


  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (cp.mode == COMM_AG) tma_prefetch_desc(&tmap_g);
#pragma unroll
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMER_THREADS);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (n_comm > 0 && static_cast<int>(blockIdx.x) < n_comm) {
    // ======================= COMM_AG copy CTA: push the local row blocks to the peers over NVLink ==============
    // Push, not pull: P2P stores are posted (no NVLink round trip per request) and the data is ready by stream
    // order, so no "shard ready" handshake is needed.  The copy itself is done by the TMA engine: one thread streams
    // 32 KB chunks  local global -> smem ring (cp.async.bulk + mbarrier)  ->  peer global (cp.async.bulk store),
    // keeping the whole ring (6 x 32 KB = the GEMM pipeline's smem, idle in this CTA) in flight, instead of
    // 16-byte register round trips.  Row blocks (128 rows x K, contiguous in both buffers) are taken round-robin,
    // destination by destination in the order the peers consume them (the peer right "below" needs our rows
    // first); after a row block has fully landed the peer's arrival counter is bumped with a system-scope release.
    // WAR safety: the gathered buffers are double-buffered by call parity; a peer only finishes call n-1 after our
    // pushes of call n-1, which we issue after our call n-2 kernel ended, so nobody still reads parity (n-2).
    // `copy_rings` independent engines per copy CTA (lane 0 of the first warps), each with its own slice of the
    // (otherwise idle) pipeline smem as a 6-slot ring and its own mbarriers: one engine alone is latency bound.
    const int n_rings = cp.copy_rings > 0 ? cp.copy_rings : 1;
    if (lane == 0 && warp_idx < n_rings) {
      // 12 slots; at most LOADS_AHEAD loads (local, L2-resident source: fast) and up to NSLOT - LOADS_AHEAD stores (the
      // slow side: remote writes) are in flight
      constexpr int NSLOT = 12, LOADS_AHEAD = 3, STORES_PENDING = NSLOT - LOADS_AHEAD;
      const int ring = warp_idx;
      const uint32_t ring_bytes = static_cast<uint32_t>(NS * Cfg::STAGE_BYTES) / n_rings;
      const uint32_t CHUNK = (ring_bytes / NSLOT) & ~1023u;
      uint8_t* ring_smem = smem + ring * ring_bytes;
      uint64_t* bars = reinterpret_cast<uint64_t*>(aux) + ring * 16;
#pragma unroll
      for (int b = 0; b < NSLOT; ++b) mbar_init(&bars[b], 1);
      fence_barrier_init();
      fence_proxy_async();
      const size_t blk_bytes = static_cast<size_t>(BLOCK_M) * (ag_b ? p.N : p.K) * 2;  // 128 rows of the gathered operand
      const int n_chunks = static_cast<int>((blk_bytes + CHUNK - 1) / CHUNK);
      // destinations in the order the peers consume our rows (the rank right "below" first); with `fill_local` the
      // local gathered buffer is one more destination, served last (q / mbpr == world - 1 -> dst == rank)
      const int n_remote = (cp.world - 1 + (cp.fill_local ? 1 : 0)) * mbpr;
      auto dst_of = [&](int q) { return (cp.rank - 1 - q / mbpr + 2 * cp.world) % cp.world; };
      auto blk_of = [&](int q) { return cp.rank * mbpr + q % mbpr; };
      // write-after-read: before the first byte of this call goes into peer d's buffer, d must have retired its
      // previous call on this buffer (it read what we pushed then).  Checked once per destination.
      uint32_t dst_ok_mask = 1u << cp.rank;
      auto chunk_bytes = [&](int c) {
        const size_t off = static_cast<size_t>(c) * CHUNK;
        return static_cast<uint32_t>(blk_bytes - off < CHUNK ? blk_bytes - off : CHUNK);
      };
      auto signal = [&](uint32_t* flag) {
        // the bulk stores of the row block have completed (wait_group): order them (async proxy) before the
        // generic-proxy release that publishes the arrival
        asm volatile("fence.proxy.async.global;\n" ::: "memory");
        asm volatile("red.release.sys.global.add.u32 [%0], 1;\n" ::"l"(flag) : "memory");
      };
      // One flat stream of chunks over all row blocks of this engine: the load cursor runs up to NSLOT-1 chunks ahead
      // of the store cursor, and a finished row block is signalled two stores later (so the completion wait never
      // drains the pipe).
      const int engine = static_cast<int>(blockIdx.x) * n_rings + ring, n_engines = n_comm * n_rings;
      int q_ld = engine, c_ld = 0, q_st = engine, c_st = 0;
      uint32_t issued = 0, stored = 0, pend_at = 0;
      uint32_t* pend_flag = nullptr;
      while (q_st < n_remote) {
        while (q_ld < n_remote && issued - stored < static_cast<uint32_t>(LOADS_AHEAD)) {
          const uint32_t slot = issued % NSLOT;
          // the slot was last read by store #(issued - NSLOT); at least STORES_PENDING newer stores exist (fill bound)
          if (issued >= static_cast<uint32_t>(NSLOT)) tma_store_wait_read<STORES_PENDING>();
          const uint8_t* sp = reinterpret_cast<const uint8_t*>(cp.local_shard) +
                              static_cast<size_t>(q_ld % mbpr) * blk_bytes + static_cast<size_t>(c_ld) * CHUNK;
          const uint32_t bytes = chunk_bytes(c_ld);
          mbar_arrive_expect_tx(&bars[slot], bytes);
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                           smem_u32(ring_smem + slot * CHUNK)),
                       "l"(sp), "r"(bytes), "r"(smem_u32(&bars[slot]))
                       : "memory");
          ++issued;
          if (++c_ld == n_chunks) {
            c_ld = 0;
            q_ld += n_engines;
          }
        }
        const uint32_t slot = stored % NSLOT;
        mbar_wait(&bars[slot], (stored / NSLOT) & 1);
        const int dst = dst_of(q_st);
        if (!((dst_ok_mask >> dst) & 1u)) {
          spin_wait_ge_sys(cp.peer_done[cp.rank] + dst, call_idx, cp.timeout_ns, cp.timeout_rec, /*what=*/3, dst);
          dst_ok_mask |= 1u << dst;
        }
        uint8_t* dp = reinterpret_cast<uint8_t*>(cp.peer_buf[dst]) + static_cast<size_t>(blk_of(q_st)) * blk_bytes +
                      static_cast<size_t>(c_st) * CHUNK;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(dp),
                     "r"(smem_u32(ring_smem + slot * CHUNK)), "r"(chunk_bytes(c_st))
                     : "memory");
        tma_store_commit();
        ++stored;
        if (++c_st == n_chunks) {
          if (pend_flag != nullptr) {  // (tiny row blocks) the previous one is still unsignalled: complete everything
            tma_store_wait<0>();
            signal(pend_flag);
          }
          // (the local fill needs no arrival: its consumers are later kernels of this stream)
          pend_flag = dst == cp.rank ? nullptr : cp.peer_flags[dst] + blk_of(q_st);
          pend_at = stored + 6;
          c_st = 0;
          q_st += n_engines;
        }
        if (pend_flag != nullptr && stored >= pend_at) {
          tma_store_wait<6>();  // all but the six newest stores are complete -> the pending row block has landed
          signal(pend_flag);
          pend_flag = nullptr;
        }
      }
      tma_store_wait<0>();   // nothing may still read the ring (or be in flight to the local buffer) when the CTA exits
      if (pend_flag != nullptr) signal(pend_flag);
    }
  } else if (warp_idx == PRODUCER_WARP) {
    // ======================= TMA producer =======================
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int waited_blk = -1;
      for (int tile = cta; tile < num_tiles; tile += cta_stride) {
        int split, mn;
        decode_tile(tile, mn, split);
        const int m_blk = map_m(mn / n_blocks), n_blk = mn % n_blocks;
        // gathered A: rows of the local shard come straight from the shard's own tensor map, rows owned by a peer
        // from the gathered buffer once that peer's copy CTAs have pushed the row block (arrival counter)
        const bool a_local = cp.mode == COMM_AG && !ag_b && m_blk / mbpr == cp.rank;
        if (cp.mode == COMM_AG && !ag_b && !a_local) {
          spin_wait_ge_sys(cp.peer_flags[cp.rank] + m_blk, arrive_target, cp.timeout_ns, cp.timeout_rec, /*what=*/1, m_blk / mbpr);
          asm volatile("fence.proxy.async.global;\n" ::: "memory");
        }
        const CUtensorMap* map_a = a_local ? &tmap_g : &tmap_a;
        const int m_row = a_local ? (m_blk - cp.rank * mbpr) * BLOCK_M : m_blk * BLOCK_M;
        const int kb0 = split * p.k_per_split;
        const int kb1 = min(kb0 + p.k_per_split, k_blocks_total);
        for (int kb = kb0; kb < kb1; ++kb) {
          // gathered B (TN): k-block kb = token rows [64 kb, 64 kb + 64) = half of row block kb / 2
          bool b_local = false;
          if (ag_b) {
            const int blk = (kb * BLOCK_K) / BLOCK_M;
            b_local = blk / mbpr == cp.rank;
            if (!b_local && blk != waited_blk) {
              spin_wait_ge_sys(cp.peer_flags[cp.rank] + blk, arrive_target, cp.timeout_ns, cp.timeout_rec, /*what=*/1, blk / mbpr);
              asm volatile("fence.proxy.async.global;\n" ::: "memory");
              waited_blk = blk;
            }
          }
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          const CUtensorMap* map_b = b_local ? &tmap_g : &tmap_b;
          const int k_row = b_local ? kb * BLOCK_K - cp.rank * cp.rows_per_rank : kb * BLOCK_K;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          if constexpr (!A_MN) {
            tma_load_2d(sa, map_a, &full_bar[stage], kb * BLOCK_K, m_row);
          } else {
#pragma unroll
            for (int a = 0; a < BLOCK_M / 64; ++a)
              tma_load_2d(sa + a * (BLOCK_K * 128), &tmap_a, &full_bar[stage], m_blk * BLOCK_M + a * 64, kb * BLOCK_K);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          } else {
#pragma unroll
            for (int a = 0; a < BLOCK_N / 64; ++a)
              tma_load_2d(sb + a * (BLOCK_K * 128), map_b, &full_bar[stage], n_blk * BLOCK_N + a * 64, k_row);
          }
          if (++stage == NS) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ======================= consumers: wgmma main loop + epilogue (two warpgroups) =======================
    const int wg = warp_idx / 4;                 // rows [64 wg, 64 wg + 64) of the tile
    const int t = threadIdx.x % 128;
    const int row_in_tile = 64 * wg + 16 * (t / 32) + (t % 32) / 4;   // and row_in_tile + 8
    const int col_in_8 = 2 * (t % 4);
    float alpha = 1.0f;
    if constexpr (FP8) alpha = __ldg(p.deq_a) * __ldg(p.deq_b);
    if (cp.mode == COMM_RS) {
      // write-after-read on the owners' staging buffers: every owner must have retired its previous call on this
      // buffer set (its reduce phase read what we stored then) before the first partial tile of this call lands
      if (lane == 0) {
        for (int q = 0; q < cp.world; ++q)
          if (q != cp.rank) spin_wait_ge_sys(cp.peer_done[cp.rank] + q, call_idx, cp.timeout_ns, cp.timeout_rec, /*what=*/4, q);
      }
      __syncwarp();
    }
    int stage = 0;
    uint32_t phase = 0;
    float acc[BLOCK_N / 2];
    for (int tile = cta; tile < num_tiles; tile += cta_stride) {
      int split, mn;
      decode_tile(tile, mn, split);
      const int m_blk = map_m(mn / n_blocks), n_blk = mn % n_blocks;
      const int kb0 = split * p.k_per_split;
      const int kb1 = min(kb0 + p.k_per_split, k_blocks_total);
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          // K-major: 8-row groups are 1024B apart (SBO), advance 32B per WGMMA_K inside the swizzle row; this
          //          warpgroup's 64 rows of A start 64 x 128 B into the tile.
          // MN-major: 64-element MN atoms are BLOCK_K*128B apart (LBO), 8-k-row groups 1024B apart (SBO),
          //           advance 16 k-rows = 2048B per WGMMA_K; this warpgroup's rows of A are the atom `wg`.
          const uint64_t da = A_MN ? make_smem_desc_sw128(sa + wg * (BLOCK_K * 128) + k * (WGMMA_K * 128), BLOCK_K * 128, 1024)
                                   : make_smem_desc_sw128(sa + wg * (64 * 128) + k * (WGMMA_K * 2), 0, 1024);
          const uint64_t db = B_MN ? make_smem_desc_sw128(sb + k * (WGMMA_K * 128), BLOCK_K * 128, 1024)
                                   : make_smem_desc_sw128(sb + k * (WGMMA_K * 2), 0, 1024);
          const uint32_t accumulate = (kb > kb0 || k > 0) ? 1u : 0u;
          if constexpr (FP8) wgmma_e4m3_ss<BLOCK_N>(acc, da, db, accumulate);
          else wgmma_bf16_ss<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accumulate);
        }
        wgmma_commit();
        // one k-block stays in flight: the stage of the previous one is free once its group has retired
        wgmma_wait<1>();
        if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == NS) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);

      const int col_base = n_blk * BLOCK_N + col_in_8;
      if constexpr (EPI == EPI_BF16) {
        const bool use_bias = p.bias != nullptr && cp.mode != COMM_RS;  // RS: bias added once, in the reduce phase
        const bool use_pre = p.pre_in != nullptr;
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        size_t ld = static_cast<size_t>(p.ldo);
        if (cp.mode == COMM_RS) {
          // partial tile -> this rank's OWN partial-product buffer [M, N] (peer-mapped): the epilogue runs at local
          // HBM speed; the owners pull the rows they own during their reduce phase
          out = cp.peer_buf[cp.rank] + cp.staging_parity_off;
          ld = static_cast<size_t>(p.N);
        }
        float* colsum = (p.colsum != nullptr && cp.mode != COMM_RS) ? p.colsum : nullptr;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = col_base + 8 * j;
          const bool col_ok = col < p.N;   // N % 8 == 0: col + 1 is valid too
          float2 b2 = make_float2(0.f, 0.f);
          if (use_bias && col_ok) b2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
          float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m_blk * BLOCK_M + row_in_tile + 8 * h;
            if (!col_ok || row >= p.M) continue;
            float v0 = acc[4 * j + 2 * h] * alpha + b2.x;
            float v1 = acc[4 * j + 2 * h + 1] * alpha + b2.y;
            if (p.pre_out != nullptr)
              *reinterpret_cast<uint32_t*>(p.pre_out + static_cast<size_t>(row) * p.ldo + col) = pack_bf16(v0, v1);
            if (use_pre) {
              const float2 a = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.pre_in + static_cast<size_t>(row) * p.ldo + col));
              if (p.act == ACT_RESADD) {  // row-parallel output projection: y = x·Wᵀ + bias + residual in one pass
                v0 += a.x;
                v1 += a.y;
              } else if (p.act == ACT_GELU) {
                v0 *= gelu_grad_fast(a.x);
                v1 *= gelu_grad_fast(a.y);
              } else {
                v0 *= act_grad(a.x, p.act);
                v1 *= act_grad(a.y, p.act);
              }
            } else if (p.act == ACT_GELU) {
              v0 = gelu_fast(v0);
              v1 = gelu_fast(v1);
            } else if (p.act != ACT_NONE) {
              v0 = act_fwd(v0, p.act);
              v1 = act_fwd(v1, p.act);
            }
            const uint32_t packed = pack_bf16(v0, v1);
            *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(row) * ld + col) = packed;
            const float2 r = unpack_bf16(packed);   // the column sums are those of the stored (bf16) values
            cs0 += r.x;
            cs1 += r.y;
          }
          if (colsum != nullptr) {   // uniform over the CTA
#pragma unroll
            for (int off = 4; off < 32; off <<= 1) {
              cs0 += __shfl_xor_sync(0xffffffffu, cs0, off);
              cs1 += __shfl_xor_sync(0xffffffffu, cs1, off);
            }
            if (lane < 4 && col_ok)
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};\n" ::"l"(colsum + col), "f"(cs0), "f"(cs1) : "memory");
          }
        }
      } else {
        // fp32 outputs (wgrad: plain store / read-modify-write into main_grad, or red.add for split-K)
        float* out = reinterpret_cast<float*>(p.out);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = col_base + 8 * j;
          if (col >= p.N) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m_blk * BLOCK_M + row_in_tile + 8 * h;
            if (row >= p.M) continue;
            float* dst = out + static_cast<size_t>(row) * p.ldo + col;
            float2 o2 = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            if constexpr (EPI == EPI_F32) {
              if (p.rmw) {
                const float2 old = *reinterpret_cast<const float2*>(dst);
                o2.x += old.x;
                o2.y += old.y;
              }
              *reinterpret_cast<float2*>(dst) = o2;
            } else {
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};\n" ::"l"(dst), "f"(o2.x), "f"(o2.y) : "memory");
            }
          }
        }
      }
      if (cp.mode == COMM_RS) {
        // all 256 consumer threads have issued their stores -> one release-increment on the owner's counter
        asm volatile("bar.sync 1, 256;\n" ::: "memory");
        if (threadIdx.x == 0) {
          // (release at system scope is cumulative over the stores of all 256 consumer threads ordered before it by
          // the bar.sync above)
          const int owner = m_blk / mbpr;
          // one arrival per (source rank, column tile): world * n_blocks per row block and call
          asm volatile("red.release.sys.global.add.u32 [%0], 1;\n" ::"l"(cp.peer_flags[owner] + (m_blk % mbpr)) : "memory");
        }
      }
    }
  }

  if (cp.mode == COMM_RS) {
    // ---------------- reduce phase: out[r, :] = sum_src staging[src][r, :] (+ bias) (+ residual) ----------------
    // Bandwidth bound (world + 2 streams of rows_per_rank x N bf16), one CTA per SM: every thread keeps UNR row
    // vectors x (sources + residual) 16-byte loads in flight — with one vector at a time this phase was latency bound
    // and cost more than the GEMM it follows.
    constexpr int UNR = 4;
    const int col_groups = (p.N + 255) / 256;
    const int units = mbpr * col_groups;
    auto acc_add = [](float (&a)[8], const uint4& q) {
      const float2 x = unpack_bf16(q.x), y = unpack_bf16(q.y), z = unpack_bf16(q.z), w = unpack_bf16(q.w);
      a[0] += x.x; a[1] += x.y; a[2] += y.x; a[3] += y.y; a[4] += z.x; a[5] += z.y; a[6] += w.x; a[7] += w.y;
    };
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      const int lm = u / col_groups, cg = u % col_groups;
      if (threadIdx.x == 0) spin_wait_ge_sys(cp.peer_flags[cp.rank] + lm, arrive_target, cp.timeout_ns, cp.timeout_rec, /*what=*/2, lm);
      __syncthreads();
      const int c_lo = cg * 256;
      const int c_n = min(256, p.N - c_lo) / 8;  // vectors of 8 per row in this column group
      const int total_v = BLOCK_M * c_n;
      for (int v0 = threadIdx.x; v0 < total_v; v0 += NUM_THREADS * UNR) {
        float acc8[UNR][8];
        size_t off[UNR];
        int cc[UNR];
        bool ok[UNR];
#pragma unroll
        for (int j = 0; j < UNR; ++j) {
          const int v = v0 + j * NUM_THREADS;
          ok[j] = v < total_v;
          const int vv = ok[j] ? v : 0;
          cc[j] = c_lo + (vv % c_n) * 8;
          off[j] = static_cast<size_t>(lm * BLOCK_M + vv / c_n) * p.N + cc[j];
#pragma unroll
          for (int e = 0; e < 8; ++e) acc8[j][e] = 0.f;
        }
        uint4 q[UNR], rq[UNR], bq[UNR];
        if (cp.residual != nullptr) {
#pragma unroll
          for (int j = 0; j < UNR; ++j) rq[j] = ld_stream_u4(reinterpret_cast<const uint4*>(cp.residual + off[j]));
        }
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < UNR; ++j) bq[j] = *reinterpret_cast<const uint4*>(p.bias + cc[j]);
        }
        for (int s0 = 0; s0 < cp.world; ++s0) {
          // every rank's partial product of MY rows (peers over NVLink, starting with the next rank so that the ranks
          // do not all pull from the same peer at the same time)
          const int src = (cp.rank + 1 + s0) % cp.world;
          const __nv_bfloat16* sp = cp.peer_buf[src] + cp.staging_parity_off + static_cast<size_t>(cp.rank) * cp.rows_per_rank * p.N;
#pragma unroll
          for (int j = 0; j < UNR; ++j) q[j] = ld_stream_u4(reinterpret_cast<const uint4*>(sp + off[j]));
#pragma unroll
          for (int j = 0; j < UNR; ++j) acc_add(acc8[j], q[j]);
        }
#pragma unroll
        for (int j = 0; j < UNR; ++j) {
          if (p.bias != nullptr) acc_add(acc8[j], bq[j]);
          if (cp.residual != nullptr) acc_add(acc8[j], rq[j]);
          if (ok[j])
            *reinterpret_cast<uint4*>(cp.rs_out + off[j]) =
                make_uint4(pack_bf16(acc8[j][0], acc8[j][1]), pack_bf16(acc8[j][2], acc8[j][3]),
                           pack_bf16(acc8[j][4], acc8[j][5]), pack_bf16(acc8[j][6], acc8[j][7]));
        }
      }
      __syncthreads();
    }
  }

  __syncthreads();
  if (cp.mode != COMM_NONE && threadIdx.x == 0) {
    // retire: the last CTA to get here advances the call counter and tells every peer that this rank is done reading
    // (AG: its gathered buffer, RS: its staging buffer) for call `call_idx`
    __threadfence();
    const uint32_t prev = atomicAdd(cp.state + 1, 1u);
    if (prev == gridDim.x - 1) {
      cp.state[1] = 0;
      cp.state[0] = call_idx + 1u;
      __threadfence_system();
      for (int q = 0; q < cp.world; ++q) {
        if (q == cp.rank) continue;
        asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(cp.peer_done[q] + cp.rank), "r"(call_idx + 1u) : "memory");
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Ping-pong schedule for bf16 outputs (NT forward and NN dgrad, one K partition, no collective).
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected thread; registers lowered with setmaxnreg),
// warpgroups 1 and 2 = consumers, each owning WHOLE 128 x 128 output tiles (two m64n128k16 wgmmas per k-step, 128 fp32
// accumulators per thread).  The CTA's tiles cta + k * stride go to consumer k % 2.  Two named barriers hand the
// tensor cores from one consumer to the other: consumer A's k-loop of tile k issues before consumer B's k-loop of
// tile k + 1, and A's epilogue runs under B's k-loop.  With short K (1024: most forward and dgrad GEMMs of a
// transformer) the epilogue of the 288-thread kernel above took as long as the main loop with the tensor cores idle.
//
// Epilogue: the bf16 tile goes through a per-consumer 32 KB shared staging buffer (two 64-column boxes, 128-byte
// swizzle) and leaves with TMA stores, which clip at M and N.  The store completes while the consumer runs its next
// k-loop; it waits for the read of the staging buffer only before the buffer is written again.  `pre_out` uses the same
// buffer first.  `pre_in` (GELU' input, or the residual of ACT_RESADD) is loaded by the producer with TMA into the
// staging buffer when the tile's k-loop starts, and each thread overwrites its own elements with the result.
//
// Numerics are those of gemm_kernel<.., EPI_BF16>: the same k-blocks in increasing order, the same wgmma k16 steps,
// the same epilogue arithmetic and RNE rounding, so every output element is bit-identical.
constexpr int PP_BLOCK_N = 128;
constexpr int PP_THREADS = 384;
constexpr int PP_STAGES = 5;
constexpr int PP_STAGE_BYTES = (BLOCK_M + PP_BLOCK_N) * BLOCK_K * 2;       // 32 KB
constexpr int PP_STAGING_BYTES = BLOCK_M * PP_BLOCK_N * 2;                 // 32 KB per consumer
constexpr int PP_BOX_BYTES = BLOCK_M * 64 * 2;                             // one 64-column box of the staging tile
constexpr int PP_SMEM_BYTES = PP_STAGES * PP_STAGE_BYTES + 2 * PP_STAGING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(PP_SMEM_BYTES <= 227 * 1024, "ping-pong GEMM exceeds the shared memory of an SM");

// named barriers: 1, 2 = warpgroup_sync of consumer 0 / 1; 3, 4 = "consumer 0 / 1 may issue its k-loop"
LB_DEVICE void pp_order_wait(int c) { asm volatile("bar.sync %0, 256;\n" ::"r"(3 + c) : "memory"); }
LB_DEVICE void pp_order_signal(int c) { asm volatile("bar.arrive %0, 256;\n" ::"r"(3 + c) : "memory"); }

// last epilogue pass of the ping-pong kernel for one activation: act(acc) or acc * act'(pre_in) or acc + residual, in
// the arithmetic of gemm_kernel's bf16 epilogue (act_fwd(GELU) is gelu_fast, act_grad(GELU) is gelu_grad_fast), packed
// to bf16 into the staging tile.  `row0`: this thread's slot in row 16 * warp + r, column 0; r = lane / 4 is also the
// row's swizzle phase.  With PRE_IN the slot holds the pre_in element on entry.
template <int ACT, bool PRE_IN>
LB_DEVICE void pp_finish(float (&acc)[2][PP_BLOCK_N / 2], uint32_t row0, int r) {
#pragma unroll
  for (int j = 0; j < PP_BLOCK_N / 8; ++j) {
    const uint32_t col_off = (j / 8) * PP_BOX_BYTES + (((j % 8) ^ r) << 4);
#pragma unroll
    for (int hm = 0; hm < 2; ++hm)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t addr = row0 + (64 * hm + 8 * h) * 128 + col_off;
        float v0 = acc[hm][4 * j + 2 * h], v1 = acc[hm][4 * j + 2 * h + 1];
        if constexpr (PRE_IN) {
          uint32_t u;
          asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(u) : "r"(addr) : "memory");
          const float2 a = unpack_bf16(u);
          if constexpr (ACT == ACT_RESADD) {
            v0 += a.x;
            v1 += a.y;
          } else {
            v0 *= act_grad(a.x, ACT);
            v1 *= act_grad(a.y, ACT);
          }
        } else if constexpr (ACT != ACT_NONE) {
          v0 = act_fwd(v0, ACT);
          v1 = act_fwd(v1, ACT);
        }
        asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(addr), "r"(pack_bf16(v0, v1)) : "memory");
      }
  }
}

template <bool B_MN>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_pre_out,
                     const __grid_constant__ CUtensorMap tmap_pre_in, GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* staging = smem + PP_STAGES * PP_STAGE_BYTES;   // [2][PP_STAGING_BYTES]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + 2 * PP_STAGING_BYTES);
  uint64_t* empty_bar = full_bar + PP_STAGES;
  uint64_t* pre_full = empty_bar + PP_STAGES;    // [2] pre_in tile of consumer c landed in its staging buffer
  uint64_t* stg_free = pre_full + 2;             // [2] consumer c's previous TMA store has read its staging buffer

  const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_blocks = (p.N + PP_BLOCK_N - 1) / PP_BLOCK_N;
  const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int num_tiles = m_blocks * n_blocks;
  const int cta = blockIdx.x, cta_stride = gridDim.x;
  const bool use_pre = p.pre_in != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
#pragma unroll
    for (int i = 0; i < PP_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 128);
    }
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      mbar_init(&pre_full[c], 1);
      mbar_init(&stg_free[c], 1);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  const int wg = threadIdx.x / 128;
  if (wg == 0) {
    // ======================= TMA producer: tiles in the consumers' interleaved order =======================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (threadIdx.x < 32 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int k = 0, tile = cta; tile < num_tiles; ++k, tile += cta_stride) {
        const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
        if (use_pre) {
          const int c = k & 1;
          mbar_wait(&stg_free[c], (k >> 1) & 1);
          uint8_t* dst = staging + c * PP_STAGING_BYTES;
          mbar_arrive_expect_tx(&pre_full[c], PP_STAGING_BYTES);
          tma_load_2d(dst, &tmap_pre_in, &pre_full[c], n_blk * PP_BLOCK_N, m_blk * BLOCK_M);
          tma_load_2d(dst + PP_BOX_BYTES, &tmap_pre_in, &pre_full[c], n_blk * PP_BLOCK_N + 64, m_blk * BLOCK_M);
        }
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * PP_STAGE_BYTES;
          uint8_t* sb = sa + BLOCK_M * BLOCK_K * 2;
          mbar_arrive_expect_tx(&full_bar[stage], PP_STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * PP_BLOCK_N);
          } else {
#pragma unroll
            for (int a = 0; a < PP_BLOCK_N / 64; ++a)
              tma_load_2d(sb + a * (BLOCK_K * 128), &tmap_b, &full_bar[stage], n_blk * PP_BLOCK_N + a * 64, kb * BLOCK_K);
          }
          if (++stage == PP_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // ======================= consumers: whole tiles, alternately =======================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int c = wg - 1;
  const int t = threadIdx.x % 128;
  const int warp = t / 32, lane = t % 32;
  uint8_t* stg = staging + c * PP_STAGING_BYTES;
  const uint32_t stg_u32 = smem_u32(stg);
  // this thread's 4-byte slot of (m64 half hm, 8-column group j, row offset 8h) in the swizzled staging tile
  auto stg_off = [&](int hm, int j, int h) -> uint32_t {
    const int row = 64 * hm + 16 * warp + lane / 4 + 8 * h;
    return (j / 8) * PP_BOX_BYTES + row * 128 + (((j % 8) ^ (lane / 4)) << 4) + 4 * (lane % 4);
  };
  auto tile_of = [&](int k) { return cta + k * cta_stride; };
  // consumer 1's first k-loop waits for consumer 0's; consumer 0 goes first
  if (c == 1) pp_order_signal(0);

  float acc[2][PP_BLOCK_N / 2];
  for (int k = c; tile_of(k) < num_tiles; k += 2) {
    const int tile = tile_of(k);
    const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
    if (use_pre && t == 0) {
      // the producer loads this tile's pre_in into the staging buffer once the previous store has read it
      tma_store_wait_read<0>();
      mbar_arrive(&stg_free[c]);
    }
    pp_order_wait(c);
    const long g0 = static_cast<long>(k) * k_blocks;   // k-blocks the ring delivered before this tile
    int stage = static_cast<int>(g0 % PP_STAGES);
    uint32_t phase = static_cast<uint32_t>((g0 / PP_STAGES) & 1);
    int prev_stage = -1;
    for (int kb = 0; kb < k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * PP_STAGE_BYTES);
      const uint32_t sb = sa + BLOCK_M * BLOCK_K * 2;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BLOCK_K / WGMMA_K; ++kk) {
        const uint64_t db = B_MN ? make_smem_desc_sw128(sb + kk * (WGMMA_K * 128), BLOCK_K * 128, 1024)
                                 : make_smem_desc_sw128(sb + kk * (WGMMA_K * 2), 0, 1024);
        const uint32_t accumulate = (kb > 0 || kk > 0) ? 1u : 0u;
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
          const uint64_t da = make_smem_desc_sw128(sa + hm * (64 * 128) + kk * (WGMMA_K * 2), 0, 1024);
          wgmma_bf16_ss<PP_BLOCK_N, 0, B_MN ? 1 : 0>(acc[hm], da, db, accumulate);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == PP_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    // the other consumer's next tile may issue now (its wgmmas queue behind ours)
    if (tile_of(k + 1) < num_tiles) pp_order_signal(c ^ 1);
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);

    // ---------------- epilogue ----------------
    if (use_pre) {
      mbar_wait(&pre_full[c], (k >> 1) & 1);
    } else {
      if (t == 0) tma_store_wait_read<0>();
      warpgroup_sync(c);
    }
    const int col_base = n_blk * PP_BLOCK_N + 2 * (lane % 4);
    // bias (and the pre-activation copy, which passes through the staging buffer first)
#pragma unroll
    for (int j = 0; j < PP_BLOCK_N / 8; ++j) {
      const int col = col_base + 8 * j;
      float2 b2 = make_float2(0.f, 0.f);
      if (p.bias != nullptr && col < p.N) b2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          acc[hm][4 * j + 2 * h] += b2.x;
          acc[hm][4 * j + 2 * h + 1] += b2.y;
          if (p.pre_out != nullptr)
            asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(stg_u32 + stg_off(hm, j, h)),
                         "r"(pack_bf16(acc[hm][4 * j + 2 * h], acc[hm][4 * j + 2 * h + 1]))
                         : "memory");
        }
    }
    if (p.pre_out != nullptr) {
      fence_proxy_async();
      warpgroup_sync(c);
      if (t == 0) {
        tma_store_2d(&tmap_pre_out, stg, n_blk * PP_BLOCK_N, m_blk * BLOCK_M);
        tma_store_2d(&tmap_pre_out, stg + PP_BOX_BYTES, n_blk * PP_BLOCK_N + 64, m_blk * BLOCK_M);
        tma_store_commit();
        tma_store_wait_read<0>();
      }
      warpgroup_sync(c);
    }
    // one unrolled pass per (activation, pre_in) pair: a runtime switch inside the 64 unrolled steps would spread the
    // executed instructions over a code region that evicts the other consumer's k-loop from the instruction cache
    const uint32_t row0 = stg_u32 + (16 * warp + lane / 4) * 128 + 4 * (lane % 4);   // row 16 warp + lane / 4, column 0
    const int r = lane / 4;
    switch (p.act) {
      case ACT_GELU:
        use_pre ? pp_finish<ACT_GELU, true>(acc, row0, r) : pp_finish<ACT_GELU, false>(acc, row0, r);
        break;
      case ACT_GELU_TANH:
        use_pre ? pp_finish<ACT_GELU_TANH, true>(acc, row0, r) : pp_finish<ACT_GELU_TANH, false>(acc, row0, r);
        break;
      case ACT_RELU:
        use_pre ? pp_finish<ACT_RELU, true>(acc, row0, r) : pp_finish<ACT_RELU, false>(acc, row0, r);
        break;
      case ACT_SILU:
        use_pre ? pp_finish<ACT_SILU, true>(acc, row0, r) : pp_finish<ACT_SILU, false>(acc, row0, r);
        break;
      case ACT_QUICK_GELU:
        use_pre ? pp_finish<ACT_QUICK_GELU, true>(acc, row0, r) : pp_finish<ACT_QUICK_GELU, false>(acc, row0, r);
        break;
      case ACT_RESADD:
        pp_finish<ACT_RESADD, true>(acc, row0, r);
        break;
      default:
        use_pre ? pp_finish<ACT_NONE, true>(acc, row0, r) : pp_finish<ACT_NONE, false>(acc, row0, r);
    }
    fence_proxy_async();
    warpgroup_sync(c);
    if (t == 0) {
      tma_store_2d(&tmap_out, stg, n_blk * PP_BLOCK_N, m_blk * BLOCK_M);
      tma_store_2d(&tmap_out, stg + PP_BOX_BYTES, n_blk * PP_BLOCK_N + 64, m_blk * BLOCK_M);
      tma_store_commit();
    }
  }
  if (t == 0) tma_store_wait<0>();
}

}  // namespace lb

// =================================================================================================
// host side
// =================================================================================================
namespace lb_host {

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

bool make_tmap_typed(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_tiled();
  if (fn == nullptr) return false;
  // the driver entry point needs a current context: threads that have not touched the runtime yet (the autograd
  // engine's) bind the primary context once (otherwise the first call returns CUDA_ERROR_INVALID_CONTEXT — handled by
  // the retry below, but reported as an API error by compute-sanitizer)
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstride[5];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstride[i - 1] = strides_bytes[i];
  }
  CUresult r = fn(out, dtype, rank, const_cast<void*>(base), gdim, gstride, gbox, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // driver entry point called on a thread (e.g. the autograd engine's) that has not touched the runtime yet:
    // bind the primary context to this thread and retry
    cudaFree(nullptr);
    r = fn(out, dtype, rank, const_cast<void*>(base), gdim, gstride, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[libai_b200] cuTensorMapEncodeTiled failed (%d): base=%p rank=%d dims=", (int)r, base, rank);
    for (int i = 0; i < rank; ++i) fprintf(stderr, "%llu ", (unsigned long long)gdim[i]);
    fprintf(stderr, "strides(B)=");
    for (int i = 0; i + 1 < rank; ++i) fprintf(stderr, "%llu ", (unsigned long long)gstride[i]);
    fprintf(stderr, "box=");
    for (int i = 0; i < rank; ++i) fprintf(stderr, "%u ", gbox[i]);
    fprintf(stderr, "\n");
  }
  return r == CUDA_SUCCESS;
}

bool make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, CUtensorMapSwizzle swizzle) {
  return make_tmap_typed(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box, swizzle);
}

static lb::SpinTimeout* g_spin_timeout = nullptr;

lb::SpinTimeout* spin_timeout_record(cudaStream_t s) {
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (g_spin_timeout != nullptr) return g_spin_timeout;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) return nullptr;
  void* host = nullptr;
  if (cudaHostAlloc(&host, sizeof(lb::SpinTimeout), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  memset(host, 0, sizeof(lb::SpinTimeout));
  void* dev = nullptr;
  if (cudaHostGetDevicePointer(&dev, host, 0) != cudaSuccess) {
    cudaGetLastError();
    cudaFreeHost(host);
    return nullptr;
  }
  g_spin_timeout = static_cast<lb::SpinTimeout*>(dev);
  return g_spin_timeout;
}

}  // namespace lb_host

// Writes a one-line description of the flag wait that timed out into buf (n bytes) and returns its length, or 0 when
// no wait has timed out.  Reads host memory only, so it works after the trap has left the CUDA context unusable.
extern "C" int lb_spin_timeout_report(char* buf, int n) {
  const volatile lb::SpinTimeout* r = lb_host::g_spin_timeout;
  if (r == nullptr || r->set == 0u || n <= 0) return 0;
  const int len = snprintf(buf, n,
                           "device flag wait timed out: kind=%d rank/peer=%d flag=0x%llx value=%u target=%u (block %d)",
                           r->kind, r->who, r->flag, r->value, r->target, r->block);
  return len < n ? len : n - 1;
}

namespace {

int g_num_sms = 0;
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_num_sms;
}

// operand tensor map: K-major [rows, K] -> box {64, rows_box}; MN-major [K, cols] -> box {64, 64}
bool operand_tmap(CUtensorMap* m, const void* ptr, bool mn_major, int rows_or_cols, int K, int ld, int block_mn) {
  if (!mn_major) {
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)rows_or_cols};
    uint64_t strides[2] = {2, (uint64_t)ld * 2};
    uint32_t box[2] = {(uint32_t)lb::BLOCK_K, (uint32_t)block_mn};
    return lb_host::make_tmap_bf16(m, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  }
  uint64_t dims[2] = {(uint64_t)rows_or_cols, (uint64_t)K};
  uint64_t strides[2] = {2, (uint64_t)ld * 2};
  uint32_t box[2] = {64u, (uint32_t)lb::BLOCK_K};
  return lb_host::make_tmap_bf16(m, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}


template <int BN, bool AMN, bool BMN, int EPI, bool FP8 = false>
cudaError_t launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tg, const lb::GemmParams& p,
                       const lb::CommParams& cp, int grid, cudaStream_t stream) {
  using Cfg = lb::StageCfg<BN>;
  auto kern = lb::gemm_kernel<BN, AMN, BMN, EPI, FP8>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<grid, lb::NUM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, tg, p, cp);
  return cudaGetLastError();
}

template <bool AMN, bool BMN, int EPI, bool FP8 = false>
cudaError_t launch_bn(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tg, const lb::GemmParams& p,
                      const lb::CommParams& cp, int grid, cudaStream_t s) {
  switch (bn) {
    case 256:
      return launch_cfg<256, AMN, BMN, EPI, FP8>(ta, tb, tg, p, cp, grid, s);
    case 192:
      return launch_cfg<192, AMN, BMN, EPI, FP8>(ta, tb, tg, p, cp, grid, s);
    case 128:
      return launch_cfg<128, AMN, BMN, EPI, FP8>(ta, tb, tg, p, cp, grid, s);
    default:
      return launch_cfg<64, AMN, BMN, EPI, FP8>(ta, tb, tg, p, cp, grid, s);
  }
}

// bf16 [M, N] matrix with row stride ld, in 64-column x 128-row boxes (128-byte swizzle): the ping-pong kernel's
// epilogue stores (out, pre_out) and pre_in loads
bool epilogue_tmap(CUtensorMap* m, const void* ptr, int M, int N, int ld) {
  uint64_t dims[2] = {(uint64_t)N, (uint64_t)M};
  uint64_t strides[2] = {2, (uint64_t)ld * 2};
  uint32_t box[2] = {64u, (uint32_t)lb::BLOCK_M};
  return lb_host::make_tmap_bf16(m, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <bool BMN>
cudaError_t launch_pingpong(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& tpo,
                            const CUtensorMap& tpi, const lb::GemmParams& p, int grid, cudaStream_t stream) {
  auto kern = lb::gemm_pingpong_kernel<BMN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lb::PP_SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<grid, lb::PP_THREADS, lb::PP_SMEM_BYTES, stream>>>(ta, tb, to, tpo, tpi, p);
  return cudaGetLastError();
}

// 0: the ping-pong kernel where it applies (bf16 output, NT / NN, no collective); 1: always the 288-thread kernel
std::atomic<int> g_gemm_schedule{0};

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

}  // namespace

// Selects the GEMM schedule of later calls (0 = automatic, 1 = the 288-thread kernel only) and returns the previous
// one: for in-process comparisons of the two kernels.  Decided on the host at launch, so a CUDA graph keeps the kernel
// that was selected when it was captured.
extern "C" int lb_gemm_set_schedule(int schedule) { return g_gemm_schedule.exchange(schedule == 1 ? 1 : 0); }

// layout: 0 = NT (A[M,K], B[N,K]); 1 = NN (A[M,K], B[K,N]); 2 = TN (A[K,M], B[K,N])
// epi:    0 = bf16 store (+bias, act, optional pre-activation copy); 1 = fp32 store; 2 = fp32 atomic accumulate
// Returns 0 on success, a negative code for unsupported arguments, or a cudaError_t (> 0).
static bool wgrad_rmw() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("LIBAI_B200_WGRAD_RMW");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

static int gemm_impl(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo, int layout,
                     int epi, const void* bias, int act, void* pre_out, const void* pre_in, int force_bn,
                     int force_splits, const lb::CommParams& cp_in, cudaStream_t stream, const float* deq_a = nullptr,
                     const float* deq_b = nullptr, float* colsum = nullptr) {
  lb::CommParams cp = cp_in;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (N % 8) || (ldo % 4)) return -1;
  const bool a_mn = (layout == 2);
  const bool b_mn = (layout != 0);
  const int sms = num_sms();
  const int m_blocks = (M + lb::BLOCK_M - 1) / lb::BLOCK_M;
  // ---- ping-pong schedule: bf16 output of NT / NN without a collective, 128 x 128 tiles.  Its epilogue goes through
  // TMA (16-byte aligned bases, ldo % 8 == 0); pre_out and pre_in share its staging buffer, so not both at once; the
  // column-sum epilogue stays with the 288-thread kernel.  Explicit tile widths other than 128 select that kernel too.
  const bool pingpong = g_gemm_schedule.load(std::memory_order_relaxed) == 0 && cp.mode == lb::COMM_NONE && epi == 0 &&
                        deq_a == nullptr && layout != 2 && colsum == nullptr && !(pre_out != nullptr && pre_in != nullptr) &&
                        (force_bn == 0 || force_bn == lb::PP_BLOCK_N) && ldo % 8 == 0 && aligned16(out) &&
                        aligned16(pre_out) && aligned16(pre_in);
  if (pingpong) {
    lb::GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M;
    p.N = N;
    p.K = K;
    p.k_splits = 1;
    p.k_per_split = (K + lb::BLOCK_K - 1) / lb::BLOCK_K;
    p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
    p.act = act;
    p.out = out;
    p.pre_out = reinterpret_cast<__nv_bfloat16*>(pre_out);
    p.pre_in = reinterpret_cast<const __nv_bfloat16*>(pre_in);
    p.ldo = ldo;
    CUtensorMap ta, tb, to, tpo, tpi;
    if (!operand_tmap(&ta, a, false, M, K, lda, lb::BLOCK_M)) return -2;
    if (!operand_tmap(&tb, b, b_mn, N, K, ldb, lb::PP_BLOCK_N)) return -2;
    if (!epilogue_tmap(&to, out, M, N, ldo)) return -2;
    tpo = to;
    tpi = to;
    if (pre_out != nullptr && !epilogue_tmap(&tpo, pre_out, M, N, ldo)) return -2;
    if (pre_in != nullptr && !epilogue_tmap(&tpi, pre_in, M, N, ldo)) return -2;
    const long tiles = (long)m_blocks * ((N + lb::PP_BLOCK_N - 1) / lb::PP_BLOCK_N);
    const int grid = (int)(tiles < sms ? tiles : sms);
    return (int)(b_mn ? launch_pingpong<true>(ta, tb, to, tpo, tpi, p, grid, stream)
                      : launch_pingpong<false>(ta, tb, to, tpo, tpi, p, grid, stream));
  }
  // ---- tile-N heuristic: least estimated time (waves x per-tile time), ties -> wider tile
  int bn = force_bn;
  if (bn == 0 && epi == 2 && cp.mode == lb::COMM_AG && cp.gathered_is_b) {
    // gathered-B wgrad: split-K fills the machine, so take the widest tile that fits N
    bn = N >= 192 ? 256 : (N >= 96 ? 128 : 64);
  }
  if (bn == 0) {
    double best = 1e30;
    const int cands[4] = {256, 192, 128, 64};
    const double k_blocks = (double)((K + lb::BLOCK_K - 1) / lb::BLOCK_K);
    for (int c : cands) {
      if (c > 64 && N <= c / 2) continue;
      const long tiles = (long)m_blocks * ((N + c - 1) / c);
      const long waves = (tiles + sms - 1) / sms;
      // cost ~ waves * per-tile time in microseconds = main loop (c * k-blocks * per-column cost: narrower tiles pay
      // more shared-memory traffic per flop) + epilogue.  The bf16 epilogue grows faster than the tile width, so with
      // a short K (1024: the forward and most dgrad GEMMs of a transformer) narrow tiles win and only a long K pays
      // for a wide one; the fp32 epilogues (wgrad) are cheap at every width.  Fitted to dev/gemm_sweep.py on an
      // H100 SXM (700 W).
      const double per_col = c == 256 ? 0.00286 : (c == 192 ? 0.00272 : (c == 128 ? 0.00332 : 0.00414));
      const double epilogue = epi != 0 ? 4.0 : (c == 256 ? 54.0 : (c == 192 ? 24.4 : (c == 128 ? 11.6 : 4.2)));
      const double cost = (double)waves * (c * k_blocks * per_col + epilogue);
      if (cost < best - 1e-9) {
        best = cost;
        bn = c;
      }
    }
  }
  const int n_blocks = (N + bn - 1) / bn;
  const int k_blocks = (K + lb::BLOCK_K - 1) / lb::BLOCK_K;
  int splits = 1;
  if (epi == 2) {
    splits = force_splits;
    const bool ag_b = cp.mode == lb::COMM_AG && cp.gathered_is_b;
    if (ag_b) {
      // gathered-B wgrad: the partitions must not straddle a shard boundary and their number must be a multiple of the
      // group size (the kernel starts every rank on the partitions of its own shard)
      const int kb_per_rank = cp.rows_per_rank / lb::BLOCK_K;
      const long tiles = (long)m_blocks * n_blocks;
      const int gemm_ctas = sms - cp.n_comm;
      double best = 1e30;
      splits = cp.world;
      for (int j = 1; j <= 16 && j <= kb_per_rank; ++j) {
        if (kb_per_rank % j) continue;
        if (j > 1 && kb_per_rank / j < 4) break;
        const int c = cp.world * j;
        const long rounds = (tiles * c + gemm_ctas - 1) / gemm_ctas;
        const double cost = (double)rounds * (kb_per_rank / j + 6.0);
        if (cost < best - 1e-9) {
          best = cost;
          splits = c;
        }
      }
    } else if (splits <= 0) {
      // One K partition per tile: then every output element receives exactly one addition per call and the result does
      // not depend on the order in which partitions finish.  The tile width is chosen to fill the machine instead.
      splits = 1;
    }
    if (splits > k_blocks) splits = k_blocks;
  }
  lb::GemmParams p;
  p.M = M;
  p.N = N;
  p.K = K;
  p.k_splits = splits;
  p.k_per_split = (k_blocks + splits - 1) / splits;
  p.k_splits = (k_blocks + p.k_per_split - 1) / p.k_per_split;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.rmw = 0;
  if (epi == 2 && p.k_splits == 1 && wgrad_rmw()) {
    // a single K partition owns the whole tile: accumulate with a plain read-modify-write instead of L2 atomics.
    // Off by default since the epilogue became coalesced: `red.add.v4` is fire-and-forget, while the read of the old
    // tile sits exposed at the end of a one-tile-per-CTA GEMM.  LIBAI_B200_WGRAD_RMW=1 restores it.
    epi = 1;
    p.rmw = 1;
  }
  p.act = act;
  p.out = out;
  p.pre_out = reinterpret_cast<__nv_bfloat16*>(pre_out);
  p.pre_in = reinterpret_cast<const __nv_bfloat16*>(pre_in);
  p.ldo = ldo;
  p.colsum = (epi == 0) ? colsum : nullptr;
  p.fp8 = (deq_a != nullptr && deq_b != nullptr) ? 1 : 0;
  p.deq_a = deq_a;
  p.deq_b = deq_b;

  CUtensorMap ta, tb, tg;
  if (!operand_tmap(&ta, a, a_mn, M, K, lda, lb::BLOCK_M)) return -2;
  if (!operand_tmap(&tb, b, b_mn, N, K, ldb, bn)) return -2;
  tg = ta;
  if (cp.mode == lb::COMM_AG) {
    // tensor map of the local shard of the gathered operand: [rows_per_rank, K] rows of A (NT/NN), or rows_per_rank
    // reduction rows of B (TN)
    const bool ok = cp.gathered_is_b ? operand_tmap(&tg, cp.local_shard, true, N, cp.rows_per_rank, ldb, bn)
                                     : operand_tmap(&tg, cp.local_shard, false, cp.rows_per_rank, K, lda, lb::BLOCK_M);
    if (!ok) return -2;
    cp.arrivals = 1;
  } else if (cp.mode == lb::COMM_RS) {
    cp.arrivals = (uint32_t)(cp.world * n_blocks);
  }
  const long num_tiles = (long)m_blocks * n_blocks * p.k_splits;
  int grid = (int)(num_tiles < sms ? num_tiles : sms);
  if (cp.mode == lb::COMM_AG) {
    const long g = num_tiles < (sms - cp.n_comm) ? num_tiles : (sms - cp.n_comm);
    grid = (int)g + cp.n_comm;
  }

  cudaError_t e;
  if (p.fp8) {
    if (layout != 0 || epi != 0 || cp.mode != lb::COMM_NONE) return -7;
    e = launch_bn<false, false, lb::EPI_BF16, true>(bn, ta, tb, tg, p, cp, grid, stream);
  } else if (layout == 0) {
    if (epi == 0) e = launch_bn<false, false, lb::EPI_BF16>(bn, ta, tb, tg, p, cp, grid, stream);
    else if (epi == 1) e = launch_bn<false, false, lb::EPI_F32>(bn, ta, tb, tg, p, cp, grid, stream);
    else e = launch_bn<false, false, lb::EPI_ATOMIC_F32>(bn, ta, tb, tg, p, cp, grid, stream);
  } else if (layout == 1) {
    if (epi == 0) e = launch_bn<false, true, lb::EPI_BF16>(bn, ta, tb, tg, p, cp, grid, stream);
    else if (epi == 1) e = launch_bn<false, true, lb::EPI_F32>(bn, ta, tb, tg, p, cp, grid, stream);
    else e = launch_bn<false, true, lb::EPI_ATOMIC_F32>(bn, ta, tb, tg, p, cp, grid, stream);
  } else {
    if (epi == 0) e = launch_bn<true, true, lb::EPI_BF16>(bn, ta, tb, tg, p, cp, grid, stream);
    else if (epi == 1) e = launch_bn<true, true, lb::EPI_F32>(bn, ta, tb, tg, p, cp, grid, stream);
    else e = launch_bn<true, true, lb::EPI_ATOMIC_F32>(bn, ta, tb, tg, p, cp, grid, stream);
  }
  return (int)e;
}

extern "C" int lb_gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo,
                            int layout, int epi, const void* bias, int act, void* pre_out, int force_bn,
                            int force_splits, cudaStream_t stream) {
  lb::CommParams cp;
  memset(&cp, 0, sizeof(cp));
  return gemm_impl(a, b, out, M, N, K, lda, ldb, ldo, layout, epi, bias, act, pre_out, nullptr, force_bn, force_splits, cp,
                   stream);
}

// fp8 forward GEMM: y[M,N] (bf16) = act((xq[M,K] · wq[N,K]ᵀ) * deq_x * deq_w + bias); xq / wq hold E4M3 bytes, K % 16 == 0.
// The operands are handed to the kernel as bf16 matrices with K/2 columns (identical bytes, see GemmParams::fp8).
// With `residual` ([M, N] bf16) the epilogue is bias + residual add instead of an activation, and neither an activation
// nor a pre-activation copy may be asked for.  force_bn: tile width 64 / 128 / 192 / 256, or 0 for the heuristic.
extern "C" int lb_gemm_fp8(const void* xq, const void* wq, void* out, int M, int N, int K, const void* bias, int act,
                           void* pre_out, const void* residual, const float* deq_x, const float* deq_w, int force_bn,
                           cudaStream_t stream) {
  if ((K % 16) != 0 || deq_x == nullptr || deq_w == nullptr) return -7;
  if (residual != nullptr && (act != lb::ACT_NONE || pre_out != nullptr)) return -7;
  lb::CommParams cp;
  memset(&cp, 0, sizeof(cp));
  if (residual != nullptr) act = lb::ACT_RESADD;
  return gemm_impl(xq, wq, out, M, N, K / 2, K / 2, K / 2, N, 0, 0, bias, act, pre_out, residual, force_bn, 0, cp, stream,
                   deq_x, deq_w);
}

// dgrad fused with the activation backward: out[M,N] = (A·B) * act'(pre_in[M,N])   (bf16 output, ldo = row stride
// of both `out` and `pre_in`)
// `colsum` (optional, fp32 [N], 16-byte aligned): += column sums of `out` = the bias gradient of the layer that produced
// `pre_in`, accumulated by the epilogue (no separate pass over the [M, N] tensor).
extern "C" int lb_gemm_bf16_actgrad(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb,
                                    int ldo, int layout, int act, const void* pre_in, float* colsum, cudaStream_t stream) {
  lb::CommParams cp;
  memset(&cp, 0, sizeof(cp));
  if (colsum != nullptr && (reinterpret_cast<uintptr_t>(colsum) & 15)) return -8;
  return gemm_impl(a, b, out, M, N, K, lda, ldb, ldo, layout, 0, nullptr, act, nullptr, pre_in, 0, 0, cp, stream, nullptr,
                   nullptr, colsum);
}

// y[M,N] = x[M,K]·w[N,K]ᵀ + bias[N] + residual[M,N]   (bias+residual add of the transformer block in the GEMM epilogue;
// the residual tile is read by the epilogue straight from global memory)
extern "C" int lb_gemm_bf16_bias_residual(const void* x, const void* w, void* out, int M, int N, int K, int lda, int ldb,
                                          const void* bias, const void* residual, cudaStream_t stream) {
  lb::CommParams cp;
  memset(&cp, 0, sizeof(cp));
  return gemm_impl(x, w, out, M, N, K, lda, ldb, N, 0, 0, bias, lb::ACT_RESADD, nullptr, residual, 0, 0, cp, stream);
}

// Tensor-parallel fused collective GEMMs.
//   mode 1 (AG->GEMM), layout 0/1: a = local gathered buffer [M, K] (remote rows are pushed into it by the peers' copy
//           CTAs), local_shard = this rank's [M/world, K] rows, out [M, N] bf16 (+bias, +act with pre-activation copy,
//           or x act'(pre_in) for a dgrad fused with the activation backward, + column sums for the bias gradient)
//   mode 1, layout 2 (gathered-B wgrad): a = dy [T, M] (T tokens), b = local gathered buffer [T, N], local_shard =
//           this rank's [T/world, N] rows of it, out [M, N] fp32: epi 2 accumulates (red.add), epi 1 stores
//   mode 2 (GEMM->RS), layout 0/1: a = local [M, K_shard]; partial tiles go to the owners' staging buffers;
//           rs_out [M/world, N] = sum over ranks (+bias +residual)
static unsigned long long spin_timeout_ns() {
  static unsigned long long v = ~0ull;
  if (v == ~0ull) {
    const char* e = getenv("LIBAI_B200_SPIN_TIMEOUT_MS");
    v = (e != nullptr && atoll(e) > 0) ? (unsigned long long)atoll(e) * 1000000ull : 0ull;
  }
  return v;
}

extern "C" int lb_gemm_bf16_comm(const void* a, const void* b, void* out, int M, int N, int K, int layout, int epi,
                                 const void* bias, int act, void* pre_out, const void* pre_in, float* colsum, int mode,
                                 int world, int rank, const long* peer_buf, const long* peer_flags, const long* peer_done,
                                 void* state, const void* local_shard, int fill_local, const void* residual, void* rs_out,
                                 long staging_parity_off, int n_comm, cudaStream_t stream) {
  if (world > 8 || world < 2 || state == nullptr) return -4;
  const int gathered_rows = (mode == 1 && layout == 2) ? K : M;   // extent of the dimension that is split over ranks
  if (gathered_rows % (lb::BLOCK_M * world) != 0) return -4;
  if (layout < 0 || layout > 2 || (layout == 2 && mode != 1)) return -6;
  lb::CommParams cp;
  memset(&cp, 0, sizeof(cp));
  cp.mode = mode;
  cp.world = world;
  cp.rank = rank;
  cp.rows_per_rank = gathered_rows / world;
  cp.n_comm = mode == 1 ? n_comm : 0;
  cp.gathered_is_b = (mode == 1 && layout == 2) ? 1 : 0;
  cp.fill_local = fill_local;
  cp.state = reinterpret_cast<uint32_t*>(state);
  for (int i = 0; i < world; ++i) {
    cp.peer_buf[i] = reinterpret_cast<__nv_bfloat16*>(peer_buf[i]);
    cp.peer_flags[i] = reinterpret_cast<uint32_t*>(peer_flags[i]);
    cp.peer_done[i] = reinterpret_cast<uint32_t*>(peer_done[i]);
  }
  cp.local_shard = reinterpret_cast<const __nv_bfloat16*>(local_shard);
  cp.residual = reinterpret_cast<const __nv_bfloat16*>(residual);
  cp.rs_out = reinterpret_cast<__nv_bfloat16*>(rs_out);
  cp.staging_parity_off = staging_parity_off;
  cp.timeout_ns = spin_timeout_ns();
  cp.timeout_rec = lb_host::spin_timeout_record(stream);
  {
    static int rings = -1;
    if (rings < 0) {
      const char* e = getenv("LIBAI_B200_COPY_RINGS");
      rings = (e != nullptr && atoi(e) >= 1 && atoi(e) <= 8) ? atoi(e) : 1;
    }
    cp.copy_rings = rings;
  }
  // timing experiments only (results are WRONG with these set): keep the handshake but take the NVLink payload out
  {
    static int dbg = -1;
    if (dbg < 0) {
      const char* e = getenv("LIBAI_B200_DEBUG_COMM_NO_PAYLOAD");
      dbg = (e != nullptr && e[0] == '1') ? 1 : 0;
    }
    if (dbg == 1) {
      for (int i = 0; i < world; ++i) cp.peer_buf[i] = cp.peer_buf[rank];   // AG pushes / RS partial tiles stay local
    }
  }
  if (mode == 1 && local_shard == nullptr) return -4;
  if (colsum != nullptr && (reinterpret_cast<uintptr_t>(colsum) & 15)) return -8;
  int lda, ldb, ldo;
  if (layout == 0) { lda = K; ldb = K; ldo = N; }
  else if (layout == 1) { lda = K; ldb = N; ldo = N; }
  else { lda = M; ldb = N; ldo = N; }
  if (mode == 2) epi = 0;
  // the RS epilogue writes into the staging buffers; `out` is unused there (pass any valid pointer)
  return gemm_impl(a, b, mode == 2 ? rs_out : out, M, N, K, lda, ldb, ldo, layout, epi, bias, act, pre_out, pre_in, 0,
                   mode == 1 && layout == 2 ? 0 : 1, cp, stream, nullptr, nullptr, colsum);
}
