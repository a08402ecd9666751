// The native C boundary: every extern "C" kernel launcher of the extension, declared once.  Each .cu file sees these
// declarations through common.cuh and bindings.cpp includes them, so a definition that disagrees with its declaration
// fails to compile ("conflicting declaration of C function") instead of being called with the wrong arguments.
// Host-only: no device code, so g++ compiles it as well as nvcc.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lb {

// (seed, offset) of the PyTorch CUDA generator for a dropout mask (see rng_resolve in common.cuh): the values in eager
// mode, device pointers and an intra-graph offset while a CUDA graph is being captured; `salt` distinguishes
// tensor-parallel ranks in sharded regions
struct RngArgs {
  unsigned long long seed_val, offset_val;   // eager: the values
  const long long* seed_ptr;                 // capture: where PyTorch keeps them
  const long long* offset_ptr;
  unsigned int offset_intragraph;
  int captured;
  unsigned long long salt;
};

// One flash-attention problem, shared by lb_attn_fwd and lb_attn_bwd.  A query heads in G groups (query head h reads
// K/V head h / (A / G)); Sq queries against Sk keys; head dim d a multiple of 8 in [8, 128].  Strides are in elements.
// Key j is visible to query i of sample b iff kv_start[b] <= j < kv_lens[b] (defaults 0 and Sk) and, when causal,
// j <= i + (Sk - Sq) or j < prefix_lens[b] (prefix LM: the first prefix_lens[b] keys are visible to every query).
struct AttnArgs {
  int B, A, G, Sq, Sk, d;
  long q_strides[4];   // {batch, group, in-group, seq}
  long k_strides[3];   // {batch, head, seq} over the G K/V heads
  long v_strides[3];
  bool causal;
  float scale;
  const int* kv_lens;     // optional int32 [B]: end of the visible keys per sample
  const int* kv_start;    // optional int32 [B]: start of the visible keys per sample
  const int* doc_start;   // optional int32 [B, Sq]: packed sequences, query i sees keys doc_start[b, i] <= j <= i
  const void* bias;       // optional bf16 additive score bias, key stride 1
  long bias_strides[3];   // {batch, head, query} of bias, 0 for a broadcast dimension
  const float* alibi_slopes;   // optional fp32 [A]; ignored when `bias` is given
  float p_drop;           // attention dropout probability in [0, 1), quantised to 1/256
  const int* prefix_lens; // optional int32 [B] (causal only): keys j < prefix_lens[b] are visible to every query
};

// packed sequences (doc_start) run as causal self-attention only, without kv_lens, kv_start, bias, ALiBi or dropout
inline bool attn_doc_start_supported(const AttnArgs& a) {
  return a.causal && a.Sq == a.Sk && a.kv_lens == nullptr && a.kv_start == nullptr && a.bias == nullptr &&
         a.alibi_slopes == nullptr && !(a.p_drop > 0.f);
}

// a prefix (prefix_lens) runs with the causal mask only, combined with kv_start, kv_lens, grouped-query heads and
// dropout, without bias, ALiBi or doc_start
inline bool attn_prefix_supported(const AttnArgs& a) {
  return a.causal && a.bias == nullptr && a.alibi_slopes == nullptr && a.doc_start == nullptr;
}

}  // namespace lb

extern "C" {
int lb_gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo, int layout,
                 int epi, const void* bias, int act, void* pre_out, int force_bn, int force_splits, cudaStream_t s);
int lb_gemm_set_schedule(int schedule);
int lb_norm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd, int rows, int H,
                float eps, int rms, int dtype, int wdtype, cudaStream_t s);
int lb_gemm_bf16_bias_residual(const void* x, const void* w, void* out, int M, int N, int K, int lda, int ldb,
                               const void* bias, const void* residual, cudaStream_t s);
int lb_gemm_fp8(const void* xq, const void* wq, void* out, int M, int N, int K, const void* bias, int act, void* pre_out,
                const void* residual, const float* deq_x, const float* deq_w, int force_bn, cudaStream_t s);
int lb_quant_e4m3(const void* x, void* q, void* amax_scratch, float* deq, long n, cudaStream_t s);
int lb_norm_bwd_workspace_rows(int rows);
int lb_norm_bwd_supports_gadd(int H);
int lb_norm_bwd(const void* gy, const void* x, const void* gamma, const float* mean, const float* rstd, void* gx,
                float* dgamma, float* dbeta, float* workspace, int rows, int H, int rms, int dtype, int wdtype,
                int accumulate, const void* gadd, cudaStream_t s);
int lb_bias_act_fwd(const void* x, const void* bias, void* y, long rows, int N, int act, cudaStream_t s);
int lb_gemm_bf16_actgrad(const void* a, const void* b, void* out, int M, int N, int K, int lda, int ldb, int ldo,
                         int layout, int act, const void* pre_in, float* colsum, cudaStream_t stream);
int lb_bias_act_bwd(const void* gy, const void* x, const void* bias, void* gx, long rows, int N, int act,
                    cudaStream_t s);
int lb_bias_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N, cudaStream_t s);
int lb_swiglu_fwd(const void* gate, const void* up, void* y, long n, cudaStream_t s);
int lb_swiglu_bwd(const void* gy, const void* gate, const void* up, void* dgate, void* dup, long n, cudaStream_t s);
int lb_swiglu_packed_fwd(const void* gu, void* y, long rows, long F, cudaStream_t s);
int lb_swiglu_packed_bwd(const void* gy, const void* gu, void* dgu, long rows, long F, cudaStream_t s);
int lb_rope_qkv(const void* x, const float* cosv, const float* sinv, void* y, long groups, int S, int G, int r, int D,
                int pos_offset, const int* positions, int npos, int backward, cudaStream_t s);
// ChatGLM rotary between the fused projection [tokens, (A + 2G) * D] and a packed layout (grouped [tokens, G, A/G + 2,
// D] or per-head [tokens, A, 3D]): forward packs (in = fused, out = packed), backward unpacks the gradient (in =
// packed, out = fused); table fp32 [npos, D/4, 2], positions optional int32 [S], pos_base optional int32 (its first
// element is added to i + pos_offset on the device)
int lb_glm_rotary_qkv(const void* in, const float* table, void* out, long tokens, int S, int A, int G, int D,
                      int pos_offset, const int* positions, const int* pos_base, int grouped, int backward,
                      cudaStream_t s);
int lb_colsum_workspace_rows(int M, int N);
int lb_colsum(const void* x, float* out, int M, int N, int accumulate, float* workspace, cudaStream_t s);
int lb_embedding_fwd(const int64_t* ids, const void* table, void* out, long T, int H, long vocab_start, long rows, cudaStream_t s);
int lb_embedding_bwd(const int64_t* sorted_ids, const int64_t* order, const void* gy, float* grad, long T, int H,
                     long vocab_start, long rows, cudaStream_t s);
int lb_ce_stats(const void* logits, const int64_t* labels, float* mx, float* se, float* tgt, int T, int V,
                long vocab_start, int dtype, cudaStream_t s);
int lb_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* gloss, void* dlogits, int T,
              int V, long vocab_start, int dtype, cudaStream_t s);
int lb_adamw(float* master, const float* grad, float* m, float* v, void* lp_out, int lp_dtype, const float* scale, long n,
             float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, int decoupled, cudaStream_t s);
int lb_sqnorm_workspace(long n);
int lb_sqnorm(const float* x, float* out, long n, float* workspace, cudaStream_t s);
int lb_gemm_bf16_comm(const void* a, const void* b, void* out, int M, int N, int K, int layout, int epi,
                      const void* bias, int act, void* pre_out, const void* pre_in, float* colsum, int mode,
                      int world, int rank, const long* peer_buf, const long* peer_flags, const long* peer_done,
                      void* state, const void* local_shard, int fill_local, const void* residual, void* rs_out,
                      long staging_parity_off, int n_comm, cudaStream_t stream);
int lb_zero_reduce_scatter(const long* grad_ptrs, const long* flag_ptrs, float* red, float* sqnorm, long lo, long n,
                           float scale, int world, int rank, unsigned epoch, long mc_grad, cudaStream_t s);
int lb_zero_adam_allgather(float* master, const float* red, float* m, float* v, const long* param_ptrs,
                           const long* flag_ptrs, unsigned* done_counter, const float* clip, long lo, long n, float lr,
                           float b1, float b2, float eps, float wd, float bc1, float bc2, int decoupled, int world,
                           int rank, unsigned epoch, long mc_param, cudaStream_t s);
int lb_device_barrier(const long* flag_ptrs, int world, int rank, int slot, unsigned epoch, cudaStream_t s);
int lb_p2p_allgather(const void* shard, const long* out_ptrs, const long* flag_ptrs, unsigned* done_counter,
                     long nbytes, int world, int rank, unsigned epoch, cudaStream_t s);
// forward: o [B, Sq, A, d] bf16, lse fp32 [B, A, Sq]; with dropout, `rng` is the stream and rng_out [2] receives the
// (seed, offset) pair it resolved to, for the backward
int lb_attn_fwd(const lb::AttnArgs* a, const void* q, const void* k, const void* v, void* o, float* lse,
                const lb::RngArgs* rng, long long* rng_out, cudaStream_t s);
// the forward over a paged cache: q (a->q_strides) holds the Sq new tokens, appended already; k_pool and v_pool are
// contiguous bf16 pools [num_pages, G, 64, d] (d = 64 or 128) whose logical row j of sample b is row j % 64 of page
// block_table[b * max_pages + j / 64], and the keys are the rows [0, a->Sk) (Sk = past + Sq), causal, with kv_start and
// ALiBi slopes (no kv_lens, dense bias, doc_start, prefix_lens or dropout).  Rows at or past Sk, and table entries
// outside [0, num_pages), are never read: they count as zero rows.  o [B, Sq, A, d] bf16, lse fp32 [B, A, Sq].
int lb_attn_fwd_paged(const lb::AttnArgs* a, const void* q, const void* k_pool, const void* v_pool, int num_pages,
                      const int* block_table, int max_pages, void* o, float* lse, cudaStream_t s);
// the forward of N ragged sequences over a paged cache: q [T, A, d] (a->B = 1, a->Sq = T, a->q_strides) packs them,
// sequence n owning rows cu_q[n] .. cu_q[n + 1] and holding past[n] rows before them in table row n
// (block_table [N, max_pages]); its query i sees its logical rows [0, past[n] + i], causal, with ALiBi slopes (no
// kv_start, kv_lens, dense bias, doc_start, prefix_lens or dropout).  tiles int32 [n_tiles, 2]: (n, 128-query block),
// one CTA per tile and query head.  Each sequence's output is lb_attn_fwd_paged's on that sequence alone, bit for bit;
// rows past its window, and table entries outside [0, num_pages), never reach P·V.  o [T, A, d] bf16 (rows of no
// sequence are not written), lse fp32 [T * A] (sequence n's [A, Sq_n] at A * cu_q[n]).
int lb_attn_fwd_paged_varlen(const lb::AttnArgs* a, const void* q, const void* k_pool, const void* v_pool,
                             int num_pages, const int* block_table, int max_pages, const int* cu_q, const int* past,
                             const int* tiles, int n_tiles, void* o, float* lse, cudaStream_t s);
// lb_attn_fwd_paged_varlen over FP8 (E4M3) pools [num_pages, G, 64, d] with fp32 row scales k_scale, v_scale
// [num_pages, G, 64] (16-byte aligned): the keys and values are the rows bf16_rn(float(e) * s), so each sequence's
// output is lb_attn_fwd_paged_varlen's over the dequantized pools, bit for bit
int lb_attn_fwd_paged_varlen_fp8(const lb::AttnArgs* a, const void* q, const void* k_pool, const void* v_pool,
                                 const float* k_scale, const float* v_scale, int num_pages, const int* block_table,
                                 int max_pages, const int* cu_q, const int* past, const int* tiles, int n_tiles,
                                 void* o, float* lse, cudaStream_t s);
// backward: dout with do_strides = {batch, head, seq} over the A query heads; dq written with dq_strides = {batch,
// group, in-group, seq}, dk and dv with dkv_strides = {batch, head, seq}; delta fp32 [B, A, Sq] and dq_accum
// (lb_attn_bwd_accum_floats) are workspaces, dq_order [B * A * ceil(Sq / 64)] zeroed by the caller; dbias (optional,
// fp32, bias' strides) accumulates the bias gradient; rng_state = the forward's (seed, offset) under dropout
int lb_attn_bwd(const lb::AttnArgs* a, const void* dout, const long* do_strides, const void* q, const void* k,
                const void* v, const void* o, const float* lse, void* dq, void* dk, void* dv, const long* dq_strides,
                const long* dkv_strides, float* delta, float* dq_accum, float* dbias, const long long* rng_state,
                unsigned* dq_order, cudaStream_t s);
long lb_attn_bwd_accum_floats(int B, int A, int Sq, int D);
int lb_bias_dropout_residual(const void* x, const void* bias, const void* res, void* y, long rows, int N, float p,
                             const lb::RngArgs* rng, const long long* rng_in, long long* rng_out, cudaStream_t s);
int lb_spin_timeout_report(char* buf, int n);
int lb_decode_splits(int B, int blocks, int C, int D, bool fp8);
// k_scale, v_scale (fp32 [B, G, C], C a multiple of 4): k and v are an FP8 (E4M3) cache with these row scales.
// block_table (int32 [B, max_pages], or null): k, v (and the scales) are pools of 64-row pages [P, G, 64, D]
// ([P, G, 64]) and C = max_pages * 64; no score bias or ALiBi only
int lb_decode_attn(const void* q, const long* q_strides, const void* k, const void* v, void* o, float* part_o,
                   float* part_ml, const int* seqlens, const int* kv_start, const float* alibi_slopes,
                   const float* rel_bias, int R, bool causal, const float* k_scale, const float* v_scale,
                   const int* block_table, int max_pages, int B, int Sq, int A, int G, int C, int D, float scale,
                   int nsplit, cudaStream_t s);
int lb_kv_append(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_cache, void* v_cache,
                 const int* seqlens, int B, int Sq, int G, int r, int C, int D, cudaStream_t s);
// lb_kv_append into an FP8 (E4M3) cache: each k and v row is stored as bytes [B, G, C, D] and an fp32 scale [B, G, C]
int lb_kv_append_fp8(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_cache, void* v_cache,
                     float* k_scale, float* v_scale, const int* seqlens, int B, int Sq, int G, int r, int C, int D,
                     cudaStream_t s);
// lb_kv_append and lb_kv_append_fp8 into paged caches: pools [P, G, 64, D] (scales [P, G, 64]), logical row
// seqlens[b] + i at row (seqlens[b] + i) % 64 of page block_table[b][(seqlens[b] + i) / 64]
int lb_kv_append_paged(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool, void* v_pool,
                       const int* seqlens, const int* block_table, int max_pages, int B, int Sq, int G, int r, int D,
                       cudaStream_t s);
// lb_kv_append_paged for N ragged sequences packed along Sq (B = 1): token t of sequence n (cu_q[n] <= t <
// cu_q[n + 1], int32 [N + 1] on the device) goes to logical row past[n] + t - cu_q[n] of table row n, rotated at that
// position; bf16 pools only
int lb_kv_append_paged_varlen(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool,
                              void* v_pool, const int* cu_q, const int* past, int nseq, const int* block_table,
                              int max_pages, int T, int G, int r, int D, cudaStream_t s);
int lb_kv_append_fp8_paged(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool,
                           void* v_pool, float* k_scale, float* v_scale, const int* seqlens, const int* block_table,
                           int max_pages, int B, int Sq, int G, int r, int D, cudaStream_t s);
// lb_kv_append_paged_varlen into FP8 pools [P, G, 64, D] with scales [P, G, 64]
int lb_kv_append_fp8_paged_varlen(const void* qkv, const float* cosv, const float* sinv, void* q_out, void* k_pool,
                                  void* v_pool, float* k_scale, float* v_scale, const int* cu_q, const int* past,
                                  int nseq, const int* block_table, int max_pages, int T, int G, int r, int D,
                                  cudaStream_t s);
// desc (device int64): npairs (src, dst) page pairs, then per array its address and page bytes (a multiple of 16);
// copies page src to page dst of every array
int lb_kv_page_copy(const long* desc, int npairs, int narrays, cudaStream_t s);
// y [M, N] bf16 = act((x [M, K] bf16 · float(w [N, K] E4M3)ᵀ) · w_scale [N] + bias [N]) with 1 <= M <= 64 and
// K % 16 == 0; bias (bf16 [N]) may be null.  part: an fp32 workspace of lb_linear_fp8w_workspace(M, N, K) floats (null
// when that is 0).
long lb_linear_fp8w_workspace(int M, int N, int K);
int lb_linear_fp8w(const void* x, const void* w, const float* w_scale, const void* bias, void* y, float* part, int M,
                   int N, int K, int act, cudaStream_t s);
// out [rows, K] bf16 = bf16_rn(float(w [rows, K] E4M3) · scale[row]), K % 16 == 0
int lb_dequant_e4m3_rows(const void* w, const float* scale, void* out, long rows, int K, cudaStream_t s);
// y [M, N] bf16 = act(x [M, K] bf16 · Ŵᵀ + bias [N]) with Ŵ[n, k] = bf16_rn((q[n, k] − zero[n, k/128]) · scale[n, k/128]):
// w uint8 [N, K/2] holds q two per byte (column 2j in the low nibble of byte j), scale bf16 and zero uint8 [N, K/128].
// 1 <= M <= 64, K % 128 == 0; bias may be null.  part: an fp32 workspace of lb_linear_int4w_workspace(M, N, K) floats
// (null when that is 0).
long lb_linear_int4w_workspace(int M, int N, int K);
int lb_linear_int4w(const void* x, const void* w, const void* w_scale, const void* w_zero, const void* bias, void* y,
                    float* part, int M, int N, int K, int act, cudaStream_t s);
// out [rows, K] bf16 = Ŵ of lb_linear_int4w, K % 128 == 0
int lb_dequant_int4_rows(const void* w, const void* w_scale, const void* w_zero, void* out, long rows, int K,
                         cudaStream_t s);
// Greedy acceptance of one speculative-decoding iteration (speculative_sm90.cu): logits [B, R, V] bf16 (logits_fp32 = 0)
// or fp32, draft int64 [B, R - 1], unfinished int64 [B] (updated in place), out int64 [B, 2R + 3]; counter: a uint32 of
// this launch's own, zeroed on the stream before the kernel.  eos < 0: no EOS.
int lb_spec_accept(const void* logits, int logits_fp32, const int64_t* draft, int64_t* unfinished, int64_t* out,
                   unsigned int* counter, int B, int R, int V, long long eos, long long pad, cudaStream_t s);
// Speculative sampling (speculative_sm90.cu, the warp rule of sampling.cuh).  lb_spec_sample, after draft step j:
// logits [B, V] (bf16, or fp32 with fp32 = 1) is copied to qbuf[:, j] ([B, K, V], the same dtype) and
// proposals[:, j] ([B, J] int64) is drawn from its warped distribution with u[:, j] ([B, J] fp32).
int lb_spec_sample(const void* logits, void* qbuf, int fp32, const float* u, int64_t* proposals, int B, int V, int K,
                   int J, int j, float temperature, int top_k, float top_p, cudaStream_t s);
// The acceptance of one speculative-sampling iteration: logits [B, R, V], qbuf [B, K, V] (K >= R - 1; each bf16 or
// fp32), draft int64 [B, R - 1], u fp32 [B, R, 2], unfinished int64 [B] (updated in place), out int64 [B, 2R + 3] as
// lb_spec_accept's; accepted: B·R ints of scratch; counter: a uint32 of this launch's own; scores: fp32 [B, R, V] or
// null.  eos < 0: no EOS.
int lb_spec_accept_sample(const void* logits, int logits_fp32, const void* qbuf, int q_fp32, const int64_t* draft,
                          const float* u, int64_t* unfinished, int64_t* out, int* accepted, unsigned int* counter,
                          float* scores, int B, int R, int V, int K, float temperature, int top_k, float top_p,
                          long long eos, long long pad, cudaStream_t s);
int lb_window_attn_groups(int B, int H, int W, int ws, int heads);
int lb_window_attn_fwd(const void* qkv, void* out, float* lse, const float* table, const float* tau, int B, int H, int W,
                       int ws, int shift, int heads, int d, float scale, cudaStream_t s);
int lb_window_attn_bwd(const void* dout, const void* qkv, const float* lse, const float* table,
                       const float* tau, void* dqkv, float* dtable, float* dtau, float* dt_part, float* dtau_part, int B,
                       int H, int W, int ws, int shift, int heads, int d, float scale, cudaStream_t s);
}
