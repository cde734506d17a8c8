// d9d_b200 — MoE router: fp32 scores over the experts (softmax or element-wise sigmoid) + top-k selection (+ optional
// selection bias, + optional DeepSeek-V3 group-limited selection, + optional renormalisation and scaling of the selected
// scores) in one pass, one warp per token; and its backward.
// Replaces softmax / topk (radix select + sort) / gather / div / sum launches of the eager path.
// The options are template parameters: the plain softmax instantiations (<VPL, false, false, false, false> forward,
// <VPL, false, false, false> backward) compile to the same instructions as before the options existed.
// STATS adds the statistics of the router's auxiliary losses, per sequence of seq_len consecutive tokens (the batch
// losses use one sequence of all T tokens): the per-expert selection counts, sum_t s[t, e] and sum_t lse_t^2.  Each block
// owns a contiguous range of at most `chunk` tokens inside one sequence and writes its partials (per-warp registers ->
// per-block partials in a fixed order), and router_aux_finalize_kernel sums each sequence's partials in a fixed order: no
// atomics, so two passes over the same logits agree bit for bit.  Sigmoid scores enter the statistics normalised over the
// experts (s = sigma / sum_j sigma_j), softmax ones as they are (and with lse^2).
// BALANCE adds the balance and z-loss gradients to dlogits before its bf16 rounding, from the gradient row g[t / seq_len].
#include <stdexcept>

#include "common.cuh"
#include "d9d_ops.h"

namespace d9d {
namespace {

constexpr float RENORM_EPS = 1e-20f;
constexpr int ROUTER_WARPS = 8;  // 256 threads per block

template <int VPL>  // experts per lane: E <= 32 * VPL
__device__ __forceinline__ void load_row_softmax(const __nv_bfloat16* __restrict__ row, int E, int lane, float (&p)[VPL],
                                                 float& mx, float& sum) {
  mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int e = lane + i * 32;  // strided ownership keeps global loads coalesced
    p[i] = (e < E) ? __bfloat162float(row[e]) : -INFINITY;
    mx = fmaxf(mx, p[i]);
  }
  mx = warp_max(mx);
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    p[i] = (lane + i * 32 < E) ? __expf(p[i] - mx) : 0.f;
    sum += p[i];
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < VPL; ++i) p[i] *= inv;
}

// softmax also leaves the row max and the sum of exp(x - max) (lse = max + log(sum)); sigmoid leaves them untouched
template <int VPL, bool SIGMOID>
__device__ __forceinline__ void load_row_scores(const __nv_bfloat16* __restrict__ row, int E, int lane, float (&p)[VPL],
                                                float& mx, float& sum) {
  if constexpr (SIGMOID) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int e = lane + i * 32;
      p[i] = (e < E) ? __bfloat162float(row[e]) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) p[i] = 1.f / (1.f + __expf(-p[i]));  // padding lanes are never selected
  } else {
    load_row_softmax<VPL>(row, E, lane, p, mx, sum);
  }
}

// Group-limited selection (DeepSeek-V3): a group's score is the sum of its min(2, E/G) largest keys, the topk_groups best
// groups (ties: lower group index) stay eligible and every expert of a dropped group gets key 0.0 (not -inf).  `row` is
// this warp's E-float staging area in shared memory; lane g < G ranks group g and zeroes it when it is dropped.
template <int VPL>
__device__ __forceinline__ void mask_dropped_groups(float (&key)[VPL], float* __restrict__ row, int E, int G,
                                                    int topk_groups, int lane) {
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int e = lane + i * 32;
    if (e < E) row[e] = key[i];
  }
  __syncwarp();
  const int S = E / G;
  float gs = -INFINITY;
  if (lane < G) {
    float m1 = -INFINITY, m2 = -INFINITY;
    int j = lane % S;  // start each lane at a different column: fewer bank conflicts, same top-2
    for (int n = 0; n < S; ++n) {
      const float v = row[lane * S + j];
      if (v > m1) { m2 = m1; m1 = v; } else if (v > m2) { m2 = v; }
      if (++j == S) j = 0;
    }
    gs = (S >= 2) ? m1 + m2 : m1;
  }
  unsigned keep = 0u;
  for (int r = 0; r < topk_groups; ++r) {
    float best = gs;
    int best_g = lane;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int og = __shfl_xor_sync(0xffffffffu, best_g, off);
      if (ob > best || (ob == best && og < best_g)) { best = ob; best_g = og; }
    }
    keep |= 1u << best_g;
    if (lane == best_g) gs = -INFINITY;
  }
  if (lane < G && !((keep >> lane) & 1u))
    for (int n = 0; n < S; ++n) row[lane * S + n] = 0.f;
  __syncwarp();
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int e = lane + i * 32;
    if (e < E) key[i] = row[e];
  }
  __syncwarp();  // the next token's keys overwrite the staging row
}

// The new option instantiations declare a minimum of one block per SM: without it ptxas caps some of them at 64 registers
// and spills.  A minimum of 0 is the plain __launch_bounds__(256) of the softmax path.
// STATS: block b covers tokens [q S + c chunk, q S + min(S, (c + 1) chunk)) of sequence q = b / seq_parts,
// c = b % seq_parts (S = seq_len), a warp every ROUTER_WARPS tokens; the grid has (T / S) seq_parts blocks.  It writes
// part_counts[b, E], part_scores[b, E] and part_lse2[b] (sums over its tokens).
template <int VPL, bool SIGMOID, bool GROUPED, bool SCALED, bool STATS>
__global__ void __launch_bounds__(256, (GROUPED || STATS) ? 1 : 0)
    router_fwd_kernel(const __nv_bfloat16* __restrict__ logits, const float* __restrict__ bias, long long T, int E, int k,
                      bool renorm, long long* __restrict__ idx_out, float* __restrict__ probs_out, int G,
                      int topk_groups, float scale, int* __restrict__ part_counts, float* __restrict__ part_scores,
                      float* __restrict__ part_lse2, long long seq_len, int chunk, int seq_parts) {
  const int lane = threadIdx.x & 31;
  long long t_begin = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5, t_end = T;
  long long t_step = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  if constexpr (STATS) {
    const long long first = static_cast<long long>(blockIdx.x / seq_parts) * seq_len;
    const long long c = static_cast<long long>(blockIdx.x % seq_parts) * chunk;
    t_begin = first + c + (threadIdx.x >> 5);
    t_end = first + min(seq_len, c + chunk);
    t_step = ROUTER_WARPS;
  }
  float acc_s[VPL], acc_lse2 = 0.f;  // STATS: lane-owned sum_t s[t, e] and (warp-uniform) sum_t lse_t^2
  int acc_c[VPL];                    // STATS: lane-owned selection counts
  if constexpr (STATS) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) { acc_s[i] = 0.f; acc_c[i] = 0; }
  }
  for (long long t = t_begin; t < t_end; t += t_step) {
    float p[VPL], key[VPL], mx, sum;
    load_row_scores<VPL, SIGMOID>(logits + t * E, E, lane, p, mx, sum);
    if constexpr (STATS && SIGMOID) {  // normalised affinities; padding lanes hold sigma(0) and are left out
      float ssum = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) ssum += (lane + i * 32 < E) ? p[i] : 0.f;
      const float inv = 1.f / warp_sum(ssum);
#pragma unroll
      for (int i = 0; i < VPL; ++i) acc_s[i] += p[i] * inv;
    } else if constexpr (STATS) {
#pragma unroll
      for (int i = 0; i < VPL; ++i) acc_s[i] += p[i];  // padding lanes hold 0
      const float lse = mx + __logf(sum);
      acc_lse2 += lse * lse;
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int e = lane + i * 32;
      key[i] = (e < E) ? (bias ? p[i] + bias[e] : p[i]) : -INFINITY;
    }
    if constexpr (GROUPED) {
      extern __shared__ float router_keys[];  // [ROUTER_WARPS, E]
      mask_dropped_groups<VPL>(key, router_keys + (threadIdx.x >> 5) * E, E, G, topk_groups, lane);
    }
    float sel_p = 0.f;   // lane j keeps the j-th selection
    int sel_e = 0;
    float total = 0.f;
    unsigned picked = 0u;  // STATS: bit i set when this lane's expert lane + 32 i was selected
    for (int j = 0; j < k; ++j) {
      // arg-max over the warp; ties go to the lower expert index
      float best = -INFINITY;
      int best_e = 0x7fffffff;
      float best_p = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int e = lane + i * 32;
        if (key[i] > best || (key[i] == best && e < best_e)) { best = key[i]; best_e = e; best_p = p[i]; }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oe = __shfl_xor_sync(0xffffffffu, best_e, off);
        const float op = __shfl_xor_sync(0xffffffffu, best_p, off);
        if (ob > best || (ob == best && oe < best_e)) { best = ob; best_e = oe; best_p = op; }
      }
      if ((best_e & 31) == lane) {  // owner retires the winner
        key[best_e >> 5] = -INFINITY;
        if constexpr (STATS) picked |= 1u << (best_e >> 5);
      }
      if (lane == j) { sel_p = best_p; sel_e = best_e; }
      total += best_p;
    }
    if (lane < k) {
      idx_out[t * k + lane] = sel_e;
      float w = renorm ? sel_p / (total + RENORM_EPS) : sel_p;
      if constexpr (SCALED) w *= scale;
      probs_out[t * k + lane] = w;
    }
    if constexpr (STATS) {
#pragma unroll
      for (int i = 0; i < VPL; ++i) acc_c[i] += (picked >> i) & 1u;
    }
  }
  if constexpr (STATS) {
    // block reduction in warp order: s_*[e] = ((w0 + w1) + w2) + ...
    __shared__ float s_scores[32 * VPL];
    __shared__ int s_counts[32 * VPL];
    __shared__ float s_lse2[ROUTER_WARPS];
    const int w = threadIdx.x >> 5;
    for (int r = 0; r < ROUTER_WARPS; ++r) {
      if (w == r) {
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
          const int e = lane + i * 32;
          if (e < E) {
            s_scores[e] = r ? s_scores[e] + acc_s[i] : acc_s[i];
            s_counts[e] = r ? s_counts[e] + acc_c[i] : acc_c[i];
          }
        }
      }
      __syncthreads();
    }
    if (lane == 0) s_lse2[w] = acc_lse2;
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      part_scores[static_cast<long long>(blockIdx.x) * E + e] = s_scores[e];
      part_counts[static_cast<long long>(blockIdx.x) * E + e] = s_counts[e];
    }
    if (threadIdx.x == 0) {
      float v = 0.f;
      for (int r = 0; r < ROUTER_WARPS; ++r) v += s_lse2[r];
      part_lse2[blockIdx.x] = v;
    }
  }
}

// Sums one sequence's [parts, E] partials in a fixed order.  Blocks of 32 x 32 threads: block b < ceil(E / 32) owns
// experts 32 b + x, thread row y sums parts y, y + 32, ... and row 0 then adds the 32 row sums in order; the last block
// sums part_lse2 the same way.  With no parts (T = 0) it writes zeros.
__device__ __forceinline__ void router_aux_finalize(const int* __restrict__ part_counts, const float* __restrict__ part_scores,
                                                    const float* __restrict__ part_lse2, int parts, int E,
                                                    int* __restrict__ counts, float* __restrict__ score_sum,
                                                    float* __restrict__ lse2_sum) {
  __shared__ float s_sum[32][33];
  __shared__ int s_cnt[32][33];
  const int x = threadIdx.x, y = threadIdx.y;
  if (static_cast<int>(blockIdx.x) * 32 < E) {  // block-uniform branch
    const int e = blockIdx.x * 32 + x;
    int c = 0;
    float s = 0.f;
    if (e < E) {
      for (int b = y; b < parts; b += 32) {
        c += part_counts[static_cast<long long>(b) * E + e];
        s += part_scores[static_cast<long long>(b) * E + e];
      }
    }
    s_cnt[y][x] = c;
    s_sum[y][x] = s;
    __syncthreads();
    if (y == 0 && e < E) {
      int cc = 0;
      float ss = 0.f;
      for (int r = 0; r < 32; ++r) { cc += s_cnt[r][x]; ss += s_sum[r][x]; }
      counts[e] = cc;
      score_sum[e] = ss;
    }
  } else {
    const int tid = y * 32 + x;
    float v = 0.f;
    for (int b = tid; b < parts; b += 1024) v += part_lse2[b];
    s_sum[y][x] = v;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
      for (int r = 0; r < 32; ++r)
        for (int q = 0; q < 32; ++q) t += s_sum[r][q];
      *lse2_sum = t;
    }
  }
}

// The partials are [seqs, parts, E] / [seqs, parts] and the outputs [seqs, E] / [seqs]; blockIdx.y strides over the
// sequences.
__global__ void __launch_bounds__(1024)
    router_aux_finalize_kernel(const int* __restrict__ part_counts, const float* __restrict__ part_scores,
                               const float* __restrict__ part_lse2, int parts, int E, int* __restrict__ counts,
                               float* __restrict__ score_sum, float* __restrict__ lse2_sum, long long seqs) {
  for (long long q = blockIdx.y; q < seqs; q += gridDim.y) {
    const long long off = q * parts;
    router_aux_finalize(part_counts + off * E, part_scores + off * E, part_lse2 + off, parts, E, counts + q * E,
                        score_sum + q * E, lse2_sum + q);
    __syncthreads();  // the next sequence reuses the shared row sums
  }
}

// r_j = scale * s_j (/ (S + eps) when renorm).  With dr' = scale * dr: ds_j = (dr'_j - sum_i dr'_i r_i) / (S + eps) when
// renorm, else dr'_j; dp = scatter(ds).  softmax: dlogits[e] = p_e * (dp_e - sum_j ds_j s_j); sigmoid: s_e (1 - s_e) dp_e.
// BALANCE: g is [T / seq_len, E] (balance gradient per sequence and expert) and token t uses row t / seq_len.  Softmax:
// dlogits[e] += p_e * (g_e - sum_j p_j g_j) + z_coef * lse * p_e (z_coef = 2 w_tok coef_z), folded in as dp_e += g_e and
// inner += sum_j p_j g_j - z_coef * lse.  Sigmoid (s_e = p_e / sum_j p_j, the balance scores):
// dlogits[e] += p_e (1 - p_e) (g_e - sum_j s_j g_j) / sum_j p_j, folded in as dp_e += (g_e - s.g) / sum_j p_j.
template <int VPL, bool SIGMOID, bool SCALED, bool BALANCE>
__global__ void __launch_bounds__(256, (SIGMOID || SCALED || BALANCE) ? 1 : 0)
    router_bwd_kernel(const __nv_bfloat16* __restrict__ logits, const long long* __restrict__ idx,
                      const float* __restrict__ dprobs, long long T, int E, int k, bool renorm,
                      __nv_bfloat16* __restrict__ dlogits, float scale, const float* __restrict__ g, float z_coef,
                      long long seq_len) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float gv[VPL];  // BALANCE: this lane's g_e, per token from its sequence's row
  for (long long t = warp; t < T; t += warps) {
    float p[VPL], mx, sum;
    load_row_scores<VPL, SIGMOID>(logits + t * E, E, lane, p, mx, sum);
    if constexpr (BALANCE) {
      const float* __restrict__ row = g + (t / seq_len) * E;
#pragma unroll
      for (int i = 0; i < VPL; ++i) gv[i] = (lane + i * 32 < E) ? row[lane + i * 32] : 0.f;
    }
    // lane j < k handles selection j
    const int my_e = (lane < k) ? static_cast<int>(idx[t * k + lane]) : -1;
    float my_dr = (lane < k) ? dprobs[t * k + lane] : 0.f;
    if constexpr (SCALED) my_dr *= scale;
    // s_j = p[my_e]: fetch from the owning lane
    float my_s = 0.f;
    for (int j = 0; j < k; ++j) {
      const int e = __shfl_sync(0xffffffffu, my_e, j);
      float v = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i)
        if ((e >> 5) == i) v = p[i];
      v = __shfl_sync(0xffffffffu, v, e & 31);
      if (lane == j) my_s = v;
    }
    float my_ds = my_dr;
    if (renorm) {
      const float S = warp_sum(my_s) + RENORM_EPS;
      const float r = my_s / S;
      const float dot = warp_sum(my_dr * r);
      my_ds = (lane < k) ? (my_dr - dot) / S : 0.f;
    }
    float inner = 0.f;
    if constexpr (BALANCE && !SIGMOID) {
      float pg = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) pg += p[i] * gv[i];
      inner = warp_sum(my_ds * my_s + pg) - z_coef * (mx + __logf(sum));
    } else if constexpr (!SIGMOID) {
      inner = warp_sum(my_ds * my_s);
    }
    float dp[VPL];
    if constexpr (BALANCE && SIGMOID) {
      float psum = 0.f, pg = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        psum += (lane + i * 32 < E) ? p[i] : 0.f;  // padding lanes hold sigma(0)
        pg += p[i] * gv[i];                         // and g = 0
      }
      const float inv = 1.f / warp_sum(psum);
      const float sg = warp_sum(pg) * inv;
#pragma unroll
      for (int i = 0; i < VPL; ++i) dp[i] = (gv[i] - sg) * inv;
    } else {
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        if constexpr (BALANCE) dp[i] = gv[i];
        else dp[i] = 0.f;
      }
    }
    for (int j = 0; j < k; ++j) {
      const int e = __shfl_sync(0xffffffffu, my_e, j);
      const float d = __shfl_sync(0xffffffffu, my_ds, j);
      if ((e & 31) == lane) {
#pragma unroll
        for (int i = 0; i < VPL; ++i)
          if ((e >> 5) == i) dp[i] += d;
      }
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int e = lane + i * 32;
      if constexpr (SIGMOID) {
        if (e < E) dlogits[t * E + e] = __float2bfloat16_rn(p[i] * (1.f - p[i]) * dp[i]);
      } else {
        if (e < E) dlogits[t * E + e] = __float2bfloat16_rn(p[i] * (dp[i] - inner));
      }
    }
  }
}

inline int sms() {
  static int n = 0;
  if (!n) { int d; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); }
  return n;
}

inline int grid_for(long long T) {
  long long blocks = (T + 7) / 8;
  const long long cap = static_cast<long long>(sms()) * 8;
  return static_cast<int>(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// STATS: tokens per block, a multiple of ROUTER_WARPS giving each warp the token count of a grid-stride walk over
// grid_for(T) blocks, so long sequences get about as many blocks as the plain kernels
inline int seq_chunk(long long T) {
  const long long warps = static_cast<long long>(grid_for(T)) * ROUTER_WARPS;
  return static_cast<int>((T + warps - 1) / warps) * ROUTER_WARPS;
}

// stats: per-sequence statistics with part_* sized [num_seqs * seq_parts, E] / [num_seqs * seq_parts]
template <int VPL>
void launch_fwd(const __nv_bfloat16* logits, const float* bias, long long T, int E, int k, bool renorm, bool sigmoid,
                int G, int topk_groups, float scale, long long* idx, float* probs, bool stats, int* part_counts,
                float* part_scores, float* part_lse2, cudaStream_t stream, long long seq_len, int chunk,
                int seq_parts) {
  const bool grouped = G > 1, scaled = scale != 1.f;
  const size_t smem = grouped ? sizeof(float) * ROUTER_WARPS * E : 0;  // <= 32 KiB for E <= 1024
#define D9D_ROUTER_FWD(SIG, GRP, SCL, STATS)                                                                          \
  if (sigmoid == SIG && grouped == GRP && scaled == SCL && stats == STATS) {                                         \
    const int grid = STATS ? static_cast<int>(T / seq_len) * seq_parts : grid_for(T);                                 \
    router_fwd_kernel<VPL, SIG, GRP, SCL, STATS><<<grid, 256, smem, stream>>>(                                       \
        logits, bias, T, E, k, renorm, idx, probs, G, topk_groups, scale, part_counts, part_scores, part_lse2, seq_len, \
        chunk, seq_parts);                                                                                             \
    return;                                                                                                            \
  }
  D9D_ROUTER_FWD(false, false, false, false) D9D_ROUTER_FWD(false, false, true, false)
  D9D_ROUTER_FWD(false, true, false, false) D9D_ROUTER_FWD(false, true, true, false)
  D9D_ROUTER_FWD(true, false, false, false) D9D_ROUTER_FWD(true, false, true, false)
  D9D_ROUTER_FWD(true, true, false, false) D9D_ROUTER_FWD(true, true, true, false)
  D9D_ROUTER_FWD(false, false, false, true) D9D_ROUTER_FWD(false, false, true, true)
  D9D_ROUTER_FWD(false, true, false, true) D9D_ROUTER_FWD(false, true, true, true)
  D9D_ROUTER_FWD(true, false, false, true) D9D_ROUTER_FWD(true, false, true, true)
  D9D_ROUTER_FWD(true, true, false, true) D9D_ROUTER_FWD(true, true, true, true)
#undef D9D_ROUTER_FWD
}

template <int VPL>
void launch_bwd(const __nv_bfloat16* logits, const long long* idx, const float* dprobs, long long T, int E, int k,
                bool renorm, bool sigmoid, float scale, __nv_bfloat16* dlogits, const float* g, float z_coef,
                cudaStream_t stream, long long seq_len) {
  const bool scaled = scale != 1.f, balance = g != nullptr;
#define D9D_ROUTER_BWD(SIG, SCL, BAL)                                                                             \
  if (sigmoid == SIG && scaled == SCL && balance == BAL) {                                                        \
    router_bwd_kernel<VPL, SIG, SCL, BAL><<<grid_for(T), 256, 0, stream>>>(logits, idx, dprobs, T, E, k, renorm, \
                                                                           dlogits, scale, g, z_coef, seq_len);   \
    return;                                                                                                       \
  }
  D9D_ROUTER_BWD(false, false, false) D9D_ROUTER_BWD(false, true, false)
  D9D_ROUTER_BWD(true, false, false) D9D_ROUTER_BWD(true, true, false)
  D9D_ROUTER_BWD(false, false, true) D9D_ROUTER_BWD(false, true, true)
  D9D_ROUTER_BWD(true, false, true) D9D_ROUTER_BWD(true, true, true)
#undef D9D_ROUTER_BWD
}

}  // namespace

#define D9D_ROUTER_DISPATCH(LAUNCH, ...)      \
  do {                                        \
    if (E <= 32) LAUNCH<1>(__VA_ARGS__);      \
    else if (E <= 64) LAUNCH<2>(__VA_ARGS__); \
    else if (E <= 128) LAUNCH<4>(__VA_ARGS__);  \
    else if (E <= 256) LAUNCH<8>(__VA_ARGS__);  \
    else if (E <= 512) LAUNCH<16>(__VA_ARGS__); \
    else LAUNCH<32>(__VA_ARGS__);             \
  } while (0)

static void check_router_shape(int E, int k) {
  if (E > 1024 || k > 32 || k > E) throw std::runtime_error("d9d router: E <= 1024 and k <= min(32, E) required");
}

static void check_router_groups(int E, int num_groups, int topk_groups) {
  if (num_groups < 1 || num_groups > 32 || E % num_groups != 0 || topk_groups < 1 || topk_groups > num_groups)
    throw std::runtime_error("d9d router: 1 <= num_groups <= 32 dividing E and 1 <= topk_groups <= num_groups required");
}

static void check_num_seqs(long long T, long long num_seqs) {
  if (num_seqs < 1 || T % num_seqs != 0)
    throw std::runtime_error("d9d router: the sequence count must be a positive divisor of the token count");
}

int router_stat_parts(long long T, long long num_seqs) {
  if (num_seqs == 0) return 0;
  check_num_seqs(T, num_seqs);
  if (T == 0) return 0;
  const long long chunk = seq_chunk(T), seq_len = T / num_seqs;
  return static_cast<int>(num_seqs * ((seq_len + chunk - 1) / chunk));
}

void router_topk_fwd(const void* logits, const float* bias, long long T, int E, int k, bool renorm, bool sigmoid,
                     int num_groups, int topk_groups, float scale, long long* idx, float* probs, long long num_seqs,
                     int* part_counts, float* part_scores, float* part_lse2, int* counts, float* score_sum,
                     float* lse2_sum, cudaStream_t stream) {
  if (T == 0 && num_seqs == 0) return;
  check_router_shape(E, k);
  check_router_groups(E, num_groups, topk_groups);
  const int parts = router_stat_parts(T, num_seqs);
  const int seq_parts = num_seqs ? static_cast<int>(parts / num_seqs) : 1;
  if (T > 0)
    D9D_ROUTER_DISPATCH(launch_fwd, static_cast<const __nv_bfloat16*>(logits), bias, T, E, k, renorm, sigmoid,
                        num_groups, topk_groups, scale, idx, probs, num_seqs > 0, part_counts, part_scores, part_lse2,
                        stream, num_seqs ? T / num_seqs : 0, num_seqs ? seq_chunk(T) : 0, seq_parts);
  if (num_seqs > 0)
    router_aux_finalize_kernel<<<dim3((E + 31) / 32 + 1, static_cast<unsigned>(num_seqs < 65535 ? num_seqs : 65535)),
                                 dim3(32, 32), 0, stream>>>(part_counts, part_scores, part_lse2, seq_parts, E, counts,
                                                            score_sum, lse2_sum, num_seqs);
}

void router_topk_bwd(const void* logits, const long long* idx, const float* dprobs, long long T, int E, int k,
                     bool renorm, bool sigmoid, float scale, const float* g, long long num_seqs, float z_coef,
                     void* dlogits, cudaStream_t stream) {
  if (T == 0) return;
  check_router_shape(E, k);
  if (g) check_num_seqs(T, num_seqs);
  D9D_ROUTER_DISPATCH(launch_bwd, static_cast<const __nv_bfloat16*>(logits), idx, dprobs, T, E, k, renorm, sigmoid,
                      scale, static_cast<__nv_bfloat16*>(dlogits), g, z_coef, stream, g ? T / num_seqs : 0);
}

}  // namespace d9d
