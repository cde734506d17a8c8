// d9d_b200 native op launchers (plain C++ API, no torch dependency).
// Every launcher enqueues work on `stream` and returns immediately.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace d9d {

// ------------------------------------------------------------------ GEMM (wgmma) -----------------
// Launch codes of the GEMMs, named here once for the bindings and the launchers.  The kernels take them as int template
// parameters, so their values are part of the kernels' symbol names.
namespace gemm {

enum Mode : int { DENSE = 0, GROUPED_M = 1, GROUPED_K = 2 };
enum Epi : int {
  EPI_BF16 = 0,       // D(bf16) = acc
  EPI_F32 = 1,        // D(f32) = acc
  EPI_F32_ACC = 2,    // D(f32) += acc
  EPI_BF16_ACC = 3,   // D(bf16) += acc   TMA path: rn(D + rn_bf16(acc)), the add done in bf16 in L2;
                      //                  direct-store path: rn(D + acc) with the add in fp32
  EPI_CE_LSE = 4,     // fused linear-CE forward: per (row, n_tile) running max / sum-exp / target logit
  EPI_CE_DLOGITS = 5, // fused linear-CE backward: D(bf16) = g[row] * (exp(acc - lse[row]) - [col == target[row]])
  // regularised linear-CE (label smoothing eps, z-loss zeta over V classes in all):
  EPI_CE_LSE_SUM = 6,    // EPI_CE_LSE + per (row, n_tile) sum of the tile's logits
  EPI_CE_DLOGITS_REG = 7 // D(bf16) = g[row] * ((1 + 2 zeta lse[row]) p - (1 - eps) [col == target[row]] - eps / V)
};

// Tensor-parallel communication fused into the GEMM (operands / outputs living in NVLink peer memory):
//   COMM_AG_A   A's rows (the M dim) are sharded over the peers: every m-tile is TMA-loaded straight from the owner's
//               shard                                   => all-gather -> GEMM without a gathered copy of A
//   COMM_RS_D   every output tile is TMA reduce-added into the shard of the peer that owns those rows
//                                                        => GEMM -> reduce-scatter without a partial-sum buffer
//   COMM_AG_KA / COMM_AG_KB   A / B (MN-major) is sharded along the *reduction* dim (wgrad of a sequence-parallel
//               layer): every k-block is loaded from the owner's shard
// Row index -> (owner, local row):  blk = idx / comm_block_rows; owner = blk % comm_world;
//                                   local = (blk / comm_world) * comm_block_rows + idx % comm_block_rows
// (covers both "tokens sharded as one contiguous block per rank" and "[batch, seq/W] per rank, batch-major").
//   COMM_WAIT_A A is a *local* gathered buffer that is being filled shard by shard (peer copies running concurrently on
//               the copy engines / another stream); the producer waits on the owner's arrival flag before the first
//               load of an m-tile and tiles are visited starting with the local shard  => all-gather overlapped with
//               the GEMM tile by tile while every remote byte crosses NVLink exactly once
enum Comm : int { COMM_NONE = 0, COMM_AG_A = 1, COMM_RS_D = 2, COMM_AG_KA = 3, COMM_AG_KB = 4, COMM_WAIT_A = 5 };

}  // namespace gemm

struct GemmArgs {
  gemm::Mode mode = gemm::DENSE;
  gemm::Epi epi = gemm::EPI_BF16;
  bool a_mn = false;   // A stored [K, M] (M contiguous) instead of [M, K]
  bool b_mn = false;   // B stored [K, N] (N contiguous) instead of [N, K]
  const void* A = nullptr;
  const void* B = nullptr;
  void* D = nullptr;
  long long lda = 0, ldb = 0, ldd = 0;  // leading dims in elements
  long long b_group_stride = 0;         // GROUPED_M: elements between experts in B (0 => dense packing)
  long long d_group_stride = 0;         // GROUPED_K: elements between experts in D
  int M = 0, N = 0, K = 0;
  int num_groups = 1;
  long long k_total = 0;               // GROUPED_K: total rows of the grouped reduction dim
  const int* tile_group = nullptr;     // GROUPED_M
  const int* group_offsets = nullptr;  // GROUPED_K
  int block_n = 0;                     // 0 => heuristic
  int ctas = 0;                        // 1: one CTA per tile, 2: CTA pairs (cta_group::2, 256-row tiles), 0: process-wide policy
  int k_splits = 0;                    // dense fp32-accumulate epilogue only: 0 => heuristic, 1 => off
  // fused tensor-parallel communication (gemm::Comm); the sharded operand / output is described by its peers
  gemm::Comm comm = gemm::COMM_NONE;
  int comm_world = 1;
  int comm_block_rows = 0;                     // rows per (rank, block) of the sharded dim
  const void* const* comm_peer_ptrs = nullptr; // host array [comm_world]: base pointer of every peer's shard
  long long comm_rows_local = 0;               // rows of one shard
  long long comm_ld = 0;                       // leading dim (elements) of the shards
  int comm_rank = 0;                           // COMM_WAIT_A: this rank
  const int* comm_flags = nullptr;             // COMM_WAIT_A: device array [comm_world] of shard arrival flags
  int comm_spare_sms = 0;                      // COMM_WAIT_A: SMs left free for the concurrent copy kernels
  // fused linear cross entropy
  const long long* ce_target = nullptr;
  const float* ce_lse = nullptr;
  const float* ce_grad = nullptr;
  float* ce_part_max = nullptr;
  float* ce_part_sum = nullptr;
  float* ce_tgt_logit = nullptr;
  long long ce_ignore_index = -100;
  float ce_softcap = 0.f;              // logits -> softcap * tanh(logits / softcap); 0 = off
  const float* ce_bias = nullptr;      // [N] fp32 logit bias
  long long ce_col_offset = 0;         // B is a row slice of the classifier starting at this class id
  float* ce_part_zsum = nullptr;       // [n_tiles, M] per-tile logit sums (regularised forward)
  float ce_z_loss = 0.f;               // regularised backward: z-loss coefficient zeta
  float ce_smoothing = 0.f;            // regularised backward: label smoothing eps
  int ce_num_classes = 0;              // regularised backward: classes over all slices of the classifier
};

void gemm_dense(const GemmArgs& a, cudaStream_t stream);
void gemm_dense_pair(const GemmArgs& a, cudaStream_t stream);  // CTA-pair kernels (gemm_dense_pair.cu)
// process-wide policy for GemmArgs::ctas == 0: 0 = single-CTA kernels, 1 = CTA pairs for eligible dense / fused-CE shapes.
// Default 1 (D9D_GEMM_PAIR=0 switches it off); returns the previous value.
int gemm_set_pair_mode(int mode);
int gemm_pair_mode();
bool gemm_pair_eligible(const GemmArgs& a);
void gemm_grouped(const GemmArgs& a, cudaStream_t stream);
void gemm_ce(const GemmArgs& a, cudaStream_t stream);
void gemm_comm(const GemmArgs& a, cudaStream_t stream);  // dense GEMM with a.comm != 0 (gemm_comm_*.cu)
int gemm_ce_block_n();
// (part_max, part_sum)[n_tiles, M] + tgt_logit[M] -> lse[M], nll[M] (0 where target == ignore_index)
void ce_finalize(const float* part_max, const float* part_sum, const float* tgt_logit, const long long* target,
                 long long ignore_index, int n_tiles, int M, float* lse, float* nll, cudaStream_t stream);
// ce_finalize + part_zsum[n_tiles, M] -> zsum[M], summed over the tiles in order
void ce_finalize_zsum(const float* part_max, const float* part_sum, const float* part_zsum, const float* tgt_logit,
                      const long long* target, long long ignore_index, int n_tiles, int M, float* lse, float* nll,
                      float* zsum, cudaStream_t stream);

// ------------------------------------------------------------------ fp8 GEMM (wgmma e4m3, MX block scales) -----
namespace fp8 {
enum Scaling : int { ROWCOL = 0, MX = 1, BLOCKWISE = 2 };
}  // namespace fp8

struct Fp8GemmArgs {
  gemm::Mode mode = gemm::DENSE;  // DENSE, GROUPED_M (MoE forward / dgrad), GROUPED_K (MoE wgrad)
  gemm::Epi epi = gemm::EPI_BF16; // bf16 store (dense); GROUPED_M: + bf16 accumulate; GROUPED_K: fp32 / bf16 store / accumulate;
                                  // BLOCKWISE: bf16 or fp32 store
  // ROWCOL: row / column scales in the epilogue; MX: UE8M0 scale per 32 K-elements (DENSE); BLOCKWISE: scale_a / scale_b
  // are [ceil(K/128), round_up(M / N, 128)] per (k-block, row) scales (DENSE; GROUPED_M: scale_b [E, ceil(K/128),
  // round_up(N, 128)]; GROUPED_K: both [k_total/128, round_up(M / N, 128)], one k-block per 128-token group)
  fp8::Scaling scaling = fp8::ROWCOL;
  const void* A = nullptr;   // [M, K] e4m3, K contiguous (row pitch lda bytes); GROUPED_K: [M, k_total]
  const void* B = nullptr;   // [N, K] e4m3; GROUPED_M: [E, N, K] (expert pitch b_group_stride bytes); GROUPED_K: [N, k_total]
  void* D = nullptr;         // [M, N] bf16; GROUPED_K: [E, M, N] (expert pitch d_group_stride elements)
  long long lda = 0, ldb = 0, ldd = 0;
  long long b_group_stride = 0, d_group_stride = 0;
  int M = 0, N = 0, K = 0;
  int num_groups = 1;
  long long k_total = 0;               // GROUPED_K: rows of the grouped reduction dim
  const int* tile_group = nullptr;     // GROUPED_M: [M/128] expert per m-tile or -1
  const int* group_offsets = nullptr;  // GROUPED_K: [E+1] row offsets, multiples of 128
  const float* scale_a = nullptr;     // [M] or nullptr; GROUPED_K: [E, M]
  const float* scale_b = nullptr;     // [N] or nullptr; grouped: [E, N]
  float scale_scalar = 1.f;
  const uint8_t* sfa = nullptr;       // [ceil(M/128), K/128, 512]
  const uint8_t* sfb = nullptr;       // [ceil(N/128), K/128, 512]
};
void gemm_fp8(const Fp8GemmArgs& a, cudaStream_t stream);
void quantize_rowwise_e4m3(const void* x, void* q, float* scale, long long M, int K, long long ldx, cudaStream_t stream);
// qt[e, C, R] (row pitch ldq bytes, planes C * ldq apart) = e4m3(x[e, R, C]^T / scale[e, c]) for E planes of x
// (R * ldx elements apart); amax_scratch: [E, C] fp32
void quantize_colwise_t_e4m3(const void* x, void* qt, float* scale, float* amax_scratch, long long R, int C, long long ldx,
                             long long ldq, cudaStream_t stream, int E = 1);
// x[R, C] with R a multiple of 128 (the MoE layout's capacity) -> qt[C, R] (row pitch ldq bytes), scale[E, C]:
// expert e's rows [seg_offsets[e], seg_offsets[e] + counts[e]) are quantised with one scale per (e, c) over them (1 when
// they are all zero or there are none); every other row of qt is zero.  No host synchronisation.
void quantize_segments_t_e4m3(const void* x, void* qt, float* scale, float* amax_scratch, const int* tile_group,
                              const int* seg_offsets, const int* counts, int E, long long R, int C, long long ldx, long long ldq,
                              cudaStream_t stream);
// sf must be zero-initialised by the caller when M is not a multiple of 256 (pad blocks)
void quantize_mx_e4m3(const void* x, void* q, void* sf, long long M, int K, long long ldx, cudaStream_t stream);
// x[R, C] bf16 -> e4m3 with one fp32 scale (amax / 448, 1 for all-zero groups) per group: GROUP_ROW = 1 x 128 row groups
// (q[R, C], s[ceil(C/128), lds]), GROUP_COL = 128 x 1 column groups (transposed qT[C, R] with pitch ldq >= R, zero pad
// columns, s[ceil(R/128), lds]), GROUP_BLOCK = 128 x 128 blocks (plain: s[ceil(C/128), lds] per row, transposed:
// s[ceil(R/128), lds] per column of qT's rows).  lds is the scale row pitch, a multiple of 128 at least the scaled dimension.
enum BlockGroup : int { GROUP_ROW = 0, GROUP_COL = 1, GROUP_BLOCK = 2 };
void quantize_blockwise_e4m3(const void* x, void* q, float* scale, long long R, int C, long long ldx, long long ldq, long long lds,
                             BlockGroup group, bool transpose, cudaStream_t stream);
// The 128 x 128 blocks of every expert's weight w[e, R, C] (contiguous): plain q[e, R, C] with s[e, ceil(C/128), lds] per row,
// or transposed qt[e, C, R] with s[e, ceil(R/128), lds] per column; lds as above.
void quantize_expert_blocks_e4m3(const void* w, void* q, float* scale, int E, long long R, int C, long long lds, bool transpose,
                                 cudaStream_t stream);
// x[R, C] in the MoE layout (R a multiple of 128): 128-row tiles with tile_group -1 are skipped.  Plain: GROUP_ROW codes
// q[R, C] (row pitch ldq) and s[ceil(C/128), lds]; transposed: GROUP_COL codes qt[C, R] (pitch ldq >= R) and s[R/128, lds],
// the token groups of expert g ending at row seg_offsets[g] + counts[g] (later rows of its tiles are zeros).
void quantize_blockwise_tiles_e4m3(const void* x, void* q, float* scale, const int* tile_group, const int* seg_offsets,
                                   const int* counts, long long R, int C, long long ldx, long long ldq, long long lds, bool transpose,
                                   cudaStream_t stream);

// ------------------------------------------------------------------ normalisation ----------------
// element type of the normalisation, activation and grad-utility launchers
enum DType : int { DTYPE_BF16 = 0, DTYPE_F32 = 1, DTYPE_F16 = 2 };
void rms_norm_fwd(const void* x, const void* w, void* out, float* inv_rms, long long M, int N, float eps,
                  bool zero_centered, DType dtype, cudaStream_t stream);
// dw_partial: [rms_norm_bwd_num_partials(), N] fp32 scratch; dw: [N] in dtype
int rms_norm_bwd_num_partials();
void rms_norm_bwd(const void* dout, const void* x, const void* w, const float* inv_rms, void* dx, void* dw,
                  float* dw_partial, long long M, int N, bool zero_centered, DType dtype, cudaStream_t stream);

// ------------------------------------------------------------------ activations ------------------
void silu_mul_fwd(const void* x, const void* y, void* out, long long n, DType dtype, cudaStream_t stream);
void silu_mul_bwd(const void* dout, const void* x, const void* y, void* dx, void* dy, long long n, DType dtype,
                  cudaStream_t stream);
// MoE variant: out[r, :] = silu(x) * y * probs[r];  bwd also yields dprobs[r]
void silu_mul_probs_fwd(const void* x, const void* y, const float* probs, void* out, long long rows, int cols,
                        const int* valid_rows, cudaStream_t s);
// valid_rows (device scalar or nullptr): rows >= *valid_rows are skipped (unused tail of a static-capacity buffer)
void silu_mul_probs_bwd(const void* dout, const void* x, const void* y, const float* probs, void* dx, void* dy,
                        float* dprobs, long long rows, int cols, const int* valid_rows, cudaStream_t s);

// ------------------------------------------------------------------ stochastic rounding ----------
void sr_copy_f32_to_bf16(const float* src, void* dst, long long n, uint64_t seed, cudaStream_t stream);

struct AdamTensorMeta {
  void* p;        // bf16
  const void* g;  // bf16 or fp32
  void* m;        // bf16 or fp32
  void* v;        // bf16 or fp32
  long long n;
  long long rng_base;  // element offset into the launch-wide philox stream
};
// metas / block_map live in device memory. block_map[b] = {tensor index, chunk index}; chunk = ADAM_CHUNK elements.
constexpr int ADAM_CHUNK = 8192;
void adamw_sr_multi(const AdamTensorMeta* metas, const int2* block_map, int num_blocks, float lr, float beta1,
                    float beta2, float eps, float weight_decay, float bias_corr1, float bias_corr2, uint64_t seed,
                    const float* grad_scale /*device scalar or null*/, bool grad_bf16, bool state_bf16,
                    cudaStream_t stream);

// ------------------------------------------------------------------ RoPE (+ fused q/k RMSNorm) ---
// x: [T, H, D] (row stride = ldx elements per token), cos/sin cache: [max_pos, rope_dim] fp32 or bf16 (as float here),
// pos: [T] int64. style 0 = HALF, 1 = INTERLEAVED. inverse => apply the transposed rotation (backward).
void rope_apply(const void* x, void* out, const float* cos_cache, const float* sin_cache, const long long* pos,
                long long T, int H, int D, int rope_dim, long long ldx, long long ldo, int style, bool inverse,
                cudaStream_t stream);

// ------------------------------------------------------------------ MoE routing / permutation ----
// Builds the 128-row-aligned expert-sorted layout fully on device (no host sync):
//   topk_ids [T, k] int64 (ids outside [0, E) are dropped)
//   -> counts[E], seg_offsets[E+1] (aligned to `align`), row_map[T*k] (dest row or -1),
//      tile_group[cap/128] (expert per 128-row tile or -1), total_rows[1]
long long moe_layout_scratch_ints(long long n_entries, int E);
void moe_build_layout(const long long* topk_ids, long long T, int k, int E, int align, long long capacity_rows,
                      int* counts, int* seg_offsets, int* row_map, int* tile_group, int* chunk_scratch,
                      cudaStream_t stream);
// zero the pad rows [seg_offsets[e] + counts[e], seg_offsets[e+1]) of xp (and pp if given)
void moe_zero_pad(void* xp, float* pp, const int* counts, const int* seg_offsets, int E, int H, cudaStream_t stream);
// x[T,H] -> xp[cap,H] (rows not written stay zero: caller zero-fills), probs[T,k] -> pp[cap]
void moe_permute(const void* x, const float* probs, const int* row_map, void* xp, float* pp, long long T, int k,
                 int H, cudaStream_t stream);
// y[T,H] = sum_k yp[row_map[t,k], :]   (fp32 accumulate)
void moe_unpermute(const void* yp, const int* row_map, void* y, long long T, int k, int H, cudaStream_t stream);
// backward of permute: dx[T,H] = sum_k dxp[row_map[t,k]], dprobs[T,k] = dpp[row_map[t,k]]
void moe_permute_bwd(const void* dxp, const float* dpp, const int* row_map, void* dx, float* dprobs, long long T,
                     int k, int H, cudaStream_t stream);

// ------------------------------------------------------------------ grad utilities ---------------
// out[0] += sum(x^2) over a flat fp32/bf16 buffer
void sumsq_accumulate(const void* x, long long n, DType dtype, float* out, cudaStream_t stream);
// x *= *scale (device scalar)
void scale_inplace(void* x, long long n, DType dtype, const float* scale, cudaStream_t stream);

// ------------------------------------------------------------------ flash attention (forward / backward) --
// q / dq [total_q, Hq, Dqk], out / dout [total_q, Hq, Dv], k / dk [total_k, Hk, Dqk], v / dv [total_k, Hk, Dv] bf16
// contiguous, (Dqk, Dv) one of (64, 64), (128, 128), (192, 128), where total = B * S for
// fixed-length batches (cu_q == cu_k == nullptr) or the packed token count (cu_q / cu_k: [B + 1] int32 device arrays, Sq /
// Sk = maximum sequence lengths).  lse / delta: fp32 [B, Hq, Sq] (packed: [Hq, total_q]).
// window: key k is visible to query q iff q + (Sk - Sq) - window_left <= k <= q + (Sk - Sq) + window_right (-1 = unbounded;
// causal = window_right 0).  softcap 0 = off.  sink: per-head logit joining the softmax denominator (or nullptr).
// Packed rows outside every sequence (before cu_q[0] / cu_k[0] or from cu_q[B] / cu_k[B] on) come back with out = dq = dk =
// dv = 0 and lse = -inf.  A query without a visible key gets out = 0, dq = 0 and lse = -inf (with a sink: lse = sink).
struct FlashAttnArgs {
  const void *q, *k, *v;
  void* out;            // forward: written; backward: read
  float* lse;           // forward: written; backward: read
  const void* dout;     // backward
  float* delta;         // backward scratch (written)
  void *dq, *dk, *dv;   // backward outputs
  const float* sink;
  const int *cu_q, *cu_k;
  int B, Sq, Sk, Hq, Hk, Dqk, Dv;
  long long total_q, total_k;
  int window_left, window_right;
  float scale, softcap;
};
void flash_attn_fwd(const FlashAttnArgs& a, cudaStream_t stream);
// backward = delta pre-pass (delta[b,h,q] = sum_d dO*O, written to a.delta) followed by the dK/dV and dQ kernels (which read
// a.delta; the caller may subtract d(lse) from it in between)
void flash_attn_bwd_delta(const FlashAttnArgs& a, cudaStream_t stream);
void flash_attn_bwd(const FlashAttnArgs& a, cudaStream_t stream);

// ------------------------------------------------------------------ fused q/k RMSNorm + RoPE -------------
// q [T, Hq, D] (row stride ldq), k [T, Hk, D] (row stride ldk), cos/sin [T, rope_dim] fp32 (already gathered per token)
int qk_norm_rope_grid(long long T, int Ht);  // number of blocks == rows of dw_partial
void qk_norm_rope_fwd(const void* q, const void* k, const void* wq, const void* wk, const float* cos_t, const float* sin_t,
                      long long T, int Hq, int Hk, int D, int rope_dim, long long ldq, long long ldk, float eps,
                      bool zero_centered, int style, void* q_out, void* k_out, float* inv_rms, cudaStream_t s);
void qk_norm_rope_bwd(const void* dq_out, const void* dk_out, const void* q, const void* k, const void* wq, const void* wk,
                      const float* cos_t, const float* sin_t, const float* inv_rms, long long T, int Hq, int Hk, int D,
                      int rope_dim, long long ldq, long long ldk, bool zero_centered, int style, void* dq, void* dk,
                      float* dw_partial, float* dwq, float* dwk, cudaStream_t s);

// ------------------------------------------------------------------ MoE router -----------------------------
// logits [T, E] bf16 -> scores (fp32 softmax, or sigmoid) -> top-k by (score + bias), optionally only among the
// topk_groups best of num_groups expert groups (group score: sum of its two best keys; dropped experts get key 0) ->
// idx [T, k] int64, probs [T, k] fp32 = scale * score (renormalised over the k when renorm).
// With num_seqs > 0 (a divisor of T) also the auxiliary-loss statistics of the num_seqs sequences of T / num_seqs
// consecutive tokens, deterministic (no atomics): counts [num_seqs, E] int32 (selections per expert),
// score_sum [num_seqs, E] = sum_{t in seq} s[t] (softmax: s = softmax(x_t); sigmoid: s = sigma(x_t) / sum_j sigma(x_t)_j)
// and lse2_sum [num_seqs] = sum_{t in seq} lse_t^2 (softmax; zeros for sigmoid), via part_counts [P, E],
// part_scores [P, E], part_lse2 [P] with P = router_stat_parts(T, num_seqs) (0 when T = 0: zeros are written).
// With num_seqs = 0 the statistics pointers are unused (may be null).
int router_stat_parts(long long T, long long num_seqs);
void router_topk_fwd(const void* logits, const float* bias, long long T, int E, int k, bool renorm, bool sigmoid,
                     int num_groups, int topk_groups, float scale, long long* idx, float* probs, long long num_seqs,
                     int* part_counts, float* part_scores, float* part_lse2, int* counts, float* score_sum,
                     float* lse2_sum, cudaStream_t stream);
// With g != nullptr, plus the balance gradient of g [num_seqs, E] fp32 (num_seqs a divisor of T), row t / (T / num_seqs)
// for token t: softmax dlogits[t, e] += s_e (g_e - s.g) + z_coef lse_t s_e (z_coef = 2 w_tok coef_z); sigmoid
// dlogits[t, e] += sigma_e (1 - sigma_e) (g_e - s.g) / sum_j sigma_j
void router_topk_bwd(const void* logits, const long long* idx, const float* dprobs, long long T, int E, int k,
                     bool renorm, bool sigmoid, float scale, const float* g, long long num_seqs, float z_coef,
                     void* dlogits, cudaStream_t stream);

// ------------------------------------------------------------------ expert-parallel exchange over NVLink ----
// peer_base: device array [world] of symmetric-arena base pointers; off_* are byte offsets of regions inside the arena.
// dest_rank / dest_row: per (token, slot) pair, the owner rank and the row in its buffer (row < 0: dropped pair).
void ep_push(const void* x, const float* probs, const int* dest_rank, const int* dest_row, void* const* peer_base, long long off_x,
             long long off_p, long long n_pairs, int k, int H, cudaStream_t stream);
void ep_pull_sum(void* const* peer_base, long long off_y, long long off_dp, const int* dest_rank, const int* dest_row, void* y,
                 float* dprobs, long long T, int k, int H, cudaStream_t stream);

// ------------------------------------------------------------------ NVLink data-parallel optimizer -----------
// peer_* : device array [world] of per-replica base pointers of the symmetric arena; mc_* : multicast (NVLS) mapping
// of the same arena or nullptr.  [begin, end) is this rank's shard (multiples of 8 elements).
void nvl_reduce_shard(const float* const* peer_grads, const float* mc_grad, float* own_grad, long long begin,
                      long long end, int world, int rank, float* sumsq, cudaStream_t stream);
void nvl_adamw_shard(void* const* peer_params, void* mc_param, void* own_param, const float* own_grad, void* exp_avg,
                     void* exp_avg_sq, long long begin, long long end, int world, int rank, float lr, float beta1,
                     float beta2, float eps, float weight_decay, float bias_corr1, float bias_corr2, uint64_t seed,
                     const float* grad_scale, bool state_bf16, cudaStream_t stream);

}  // namespace d9d
