// d9d_b200 — MoE router: fp32 scores over the experts (softmax or element-wise sigmoid) + top-k selection (+ optional
// selection bias, + optional DeepSeek-V3 group-limited selection, + optional renormalisation and scaling of the selected
// scores) in one pass, one warp per token; and its backward.
// Replaces softmax / topk (radix select + sort) / gather / div / sum launches of the eager path.
// The options are template parameters: the plain softmax instantiations (<VPL, false, false, false> forward,
// <VPL, false, false> backward) compile to the same instructions as before the options existed.
#include <stdexcept>

#include "common.cuh"
#include "d9d_ops.h"

namespace d9d {
namespace {

constexpr float RENORM_EPS = 1e-20f;
constexpr int ROUTER_WARPS = 8;  // 256 threads per block

template <int VPL>  // experts per lane: E <= 32 * VPL
__device__ __forceinline__ void load_row_softmax(const __nv_bfloat16* __restrict__ row, int E, int lane, float (&p)[VPL]) {
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int e = lane + i * 32;  // strided ownership keeps global loads coalesced
    p[i] = (e < E) ? __bfloat162float(row[e]) : -INFINITY;
    mx = fmaxf(mx, p[i]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
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

template <int VPL, bool SIGMOID>
__device__ __forceinline__ void load_row_scores(const __nv_bfloat16* __restrict__ row, int E, int lane, float (&p)[VPL]) {
  if constexpr (SIGMOID) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int e = lane + i * 32;
      p[i] = (e < E) ? __bfloat162float(row[e]) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < VPL; ++i) p[i] = 1.f / (1.f + __expf(-p[i]));  // padding lanes are never selected
  } else {
    load_row_softmax<VPL>(row, E, lane, p);
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
template <int VPL, bool SIGMOID, bool GROUPED, bool SCALED>
__global__ void __launch_bounds__(256, GROUPED ? 1 : 0)
    router_fwd_kernel(const __nv_bfloat16* __restrict__ logits, const float* __restrict__ bias, long long T, int E, int k,
                      bool renorm, long long* __restrict__ idx_out, float* __restrict__ probs_out, int G,
                      int topk_groups, float scale) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long t = warp; t < T; t += warps) {
    float p[VPL], key[VPL];
    load_row_scores<VPL, SIGMOID>(logits + t * E, E, lane, p);
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
      if ((best_e & 31) == lane) key[best_e >> 5] = -INFINITY;  // owner retires the winner
      if (lane == j) { sel_p = best_p; sel_e = best_e; }
      total += best_p;
    }
    if (lane < k) {
      idx_out[t * k + lane] = sel_e;
      float w = renorm ? sel_p / (total + RENORM_EPS) : sel_p;
      if constexpr (SCALED) w *= scale;
      probs_out[t * k + lane] = w;
    }
  }
}

// r_j = scale * s_j (/ (S + eps) when renorm).  With dr' = scale * dr: ds_j = (dr'_j - sum_i dr'_i r_i) / (S + eps) when
// renorm, else dr'_j; dp = scatter(ds).  softmax: dlogits[e] = p_e * (dp_e - sum_j ds_j s_j); sigmoid: s_e (1 - s_e) dp_e.
template <int VPL, bool SIGMOID, bool SCALED>
__global__ void __launch_bounds__(256, (SIGMOID || SCALED) ? 1 : 0)
    router_bwd_kernel(const __nv_bfloat16* __restrict__ logits, const long long* __restrict__ idx,
                      const float* __restrict__ dprobs, long long T, int E, int k, bool renorm,
                      __nv_bfloat16* __restrict__ dlogits, float scale) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long t = warp; t < T; t += warps) {
    float p[VPL];
    load_row_scores<VPL, SIGMOID>(logits + t * E, E, lane, p);
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
    if constexpr (!SIGMOID) inner = warp_sum(my_ds * my_s);
    float dp[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) dp[i] = 0.f;
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

template <int VPL>
void launch_fwd(const __nv_bfloat16* logits, const float* bias, long long T, int E, int k, bool renorm, bool sigmoid,
                int G, int topk_groups, float scale, long long* idx, float* probs, cudaStream_t stream) {
  const bool grouped = G > 1, scaled = scale != 1.f;
  const size_t smem = grouped ? sizeof(float) * ROUTER_WARPS * E : 0;  // <= 32 KiB for E <= 1024
#define D9D_ROUTER_FWD(SIG, GRP, SCL)                                                                               \
  if (sigmoid == SIG && grouped == GRP && scaled == SCL) {                                                          \
    router_fwd_kernel<VPL, SIG, GRP, SCL><<<grid_for(T), 256, smem, stream>>>(logits, bias, T, E, k, renorm, idx,   \
                                                                              probs, G, topk_groups, scale);        \
    return;                                                                                                         \
  }
  D9D_ROUTER_FWD(false, false, false) D9D_ROUTER_FWD(false, false, true)
  D9D_ROUTER_FWD(false, true, false) D9D_ROUTER_FWD(false, true, true)
  D9D_ROUTER_FWD(true, false, false) D9D_ROUTER_FWD(true, false, true)
  D9D_ROUTER_FWD(true, true, false) D9D_ROUTER_FWD(true, true, true)
#undef D9D_ROUTER_FWD
}

template <int VPL>
void launch_bwd(const __nv_bfloat16* logits, const long long* idx, const float* dprobs, long long T, int E, int k,
                bool renorm, bool sigmoid, float scale, __nv_bfloat16* dlogits, cudaStream_t stream) {
  const bool scaled = scale != 1.f;
#define D9D_ROUTER_BWD(SIG, SCL)                                                                                     \
  if (sigmoid == SIG && scaled == SCL) {                                                                             \
    router_bwd_kernel<VPL, SIG, SCL><<<grid_for(T), 256, 0, stream>>>(logits, idx, dprobs, T, E, k, renorm, dlogits, \
                                                                      scale);                                        \
    return;                                                                                                          \
  }
  D9D_ROUTER_BWD(false, false) D9D_ROUTER_BWD(false, true) D9D_ROUTER_BWD(true, false) D9D_ROUTER_BWD(true, true)
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

void router_topk_fwd(const void* logits, const float* bias, long long T, int E, int k, bool renorm, bool sigmoid,
                     int num_groups, int topk_groups, float scale, long long* idx, float* probs, cudaStream_t stream) {
  if (T == 0) return;
  if (E > 1024 || k > 32 || k > E) throw std::runtime_error("d9d router: E <= 1024 and k <= min(32, E) required");
  if (num_groups < 1 || num_groups > 32 || E % num_groups != 0 || topk_groups < 1 || topk_groups > num_groups)
    throw std::runtime_error("d9d router: 1 <= num_groups <= 32 dividing E and 1 <= topk_groups <= num_groups required");
  D9D_ROUTER_DISPATCH(launch_fwd, static_cast<const __nv_bfloat16*>(logits), bias, T, E, k, renorm, sigmoid,
                      num_groups, topk_groups, scale, idx, probs, stream);
}

void router_topk_bwd(const void* logits, const long long* idx, const float* dprobs, long long T, int E, int k,
                     bool renorm, bool sigmoid, float scale, void* dlogits, cudaStream_t stream) {
  if (T == 0) return;
  if (E > 1024 || k > 32 || k > E) throw std::runtime_error("d9d router: E <= 1024 and k <= min(32, E) required");
  D9D_ROUTER_DISPATCH(launch_bwd, static_cast<const __nv_bfloat16*>(logits), idx, dprobs, T, E, k, renorm, sigmoid,
                      scale, static_cast<__nv_bfloat16*>(dlogits), stream);
}

}  // namespace d9d
