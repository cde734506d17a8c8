// d9d_b200 — per-head RMSNorm of q and k fused with rotary embedding (forward and backward).
// One warp per (token, head); q and k heads share a launch.  Replaces 2 RMSNorm + 2 RoPE launches (forward) and
// 2 x (RMSNorm backward + dW reduce) + 2 RoPE launches (backward), and halves the activation traffic.
#include <stdexcept>

#include "common.cuh"
#include "d9d_ops.h"

namespace d9d {
namespace {

// Thread mapping: a head of D elements is owned by LPH = D / 8 consecutive lanes, 8 contiguous elements (16 bytes) per
// lane, so one warp works on 32 / LPH heads at once; all reductions / exchanges are segmented xor-shuffles.
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    v[2 * i] = f.x; v[2 * i + 1] = f.y;
  }
}

__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]); u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

template <int LPH>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int off = LPH / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// out = R(theta) v on the first rope_dim dims (inverse: R(-theta)); `sub` = lane index inside the head group.
// c / sn hold cos / sin of this lane's 8 elements (loaded once per token and reused for every head).
template <int LPH>
__device__ __forceinline__ void rotate8(const float (&v)[8], float (&o)[8], const float (&c)[8], const float (&sn)[8], int sub,
                                        int rope_dim, int style, bool inverse) {
  const int e0 = sub * 8;
  if (style == 0) {  // HALF: element e pairs with e +/- rope_dim/2, i.e. the lane `half/8` further up / down
    const int half = rope_dim >> 1;
    const int lane_shift = half >> 3;
    const bool low = e0 < half;
    const int lane = threadIdx.x & 31;
    const int src = low ? lane + lane_shift : lane - lane_shift;
    float partner[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) partner[i] = __shfl_sync(0xffffffffu, v[i], src & 31);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float s = inverse ? -sn[i] : sn[i];
      o[i] = (e0 < rope_dim) ? v[i] * c[i] + (low ? -partner[i] : partner[i]) * s : v[i];
    }
  } else {  // INTERLEAVED: pairs (2i, 2i+1) live in the same lane
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
      const float s0 = inverse ? -sn[i] : sn[i], s1 = inverse ? -sn[i + 1] : sn[i + 1];
      o[i] = (e0 < rope_dim) ? v[i] * c[i] - v[i + 1] * s0 : v[i];
      o[i + 1] = (e0 < rope_dim) ? v[i + 1] * c[i + 1] + v[i] * s1 : v[i + 1];
    }
  }
}

__device__ __forceinline__ void load_angles(const float* __restrict__ cos_t, const float* __restrict__ sin_t, long long t,
                                            int rope_dim, int sub, float (&c)[8], float (&sn)[8]) {
  const int e0 = sub * 8;
  if (e0 < rope_dim) {
    const float4 c0 = *reinterpret_cast<const float4*>(cos_t + t * rope_dim + e0);
    const float4 c1 = *reinterpret_cast<const float4*>(cos_t + t * rope_dim + e0 + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(sin_t + t * rope_dim + e0);
    const float4 s1 = *reinterpret_cast<const float4*>(sin_t + t * rope_dim + e0 + 4);
    c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
    sn[0] = s0.x; sn[1] = s0.y; sn[2] = s0.z; sn[3] = s0.w; sn[4] = s1.x; sn[5] = s1.y; sn[6] = s1.z; sn[7] = s1.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i] = 1.f; sn[i] = 0.f; }
  }
}

constexpr int ROWS_IN_FLIGHT = 2;  // independent (token, head) rows per head group per iteration (memory-level parallelism)

// One warp per token: cos / sin of the token are loaded once and reused for all of its q and k heads; the head groups of
// the warp walk the heads ROWS_IN_FLIGHT at a time.
template <int LPH>
__global__ void __launch_bounds__(256) qk_norm_rope_fwd_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ wq,
    const __nv_bfloat16* __restrict__ wk, const float* __restrict__ cos_t, const float* __restrict__ sin_t, long long T,
    int Hq, int Hk, int rope_dim, long long ldq, long long ldk, float eps, bool zero_centered, int style,
    __nv_bfloat16* __restrict__ q_out, __nv_bfloat16* __restrict__ k_out, float* __restrict__ inv_rms) {
  constexpr int D = LPH * 8;
  constexpr int GROUPS = 32 / LPH;
  const int lane = threadIdx.x & 31, sub = lane % LPH, grp = lane / LPH;
  const int Ht = Hq + Hk;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wqv[8], wkv[8];
  load8(wq + sub * 8, wqv);
  load8(wk + sub * 8, wkv);
  if (zero_centered) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { wqv[i] += 1.f; wkv[i] += 1.f; }
  }
  const int head_iters = (Ht + GROUPS * ROWS_IN_FLIGHT - 1) / (GROUPS * ROWS_IN_FLIGHT);  // warp-uniform trip count
  for (long long t = warp; t < T; t += warps) {
    float c[8], sn[8];
    load_angles(cos_t, sin_t, t, rope_dim, sub, c, sn);
    for (int hi = 0; hi < head_iters; ++hi) {
      float v[ROWS_IN_FLIGHT][8];
      int hh[ROWS_IN_FLIGHT];
      bool ok[ROWS_IN_FLIGHT], isk[ROWS_IN_FLIGHT];
#pragma unroll
      for (int u = 0; u < ROWS_IN_FLIGHT; ++u) {
        hh[u] = (hi * ROWS_IN_FLIGHT + u) * GROUPS + grp;
        ok[u] = hh[u] < Ht;
        const int h = ok[u] ? hh[u] : 0;
        isk[u] = h >= Hq;
        const __nv_bfloat16* src = isk[u] ? k + t * ldk + static_cast<long long>(h - Hq) * D : q + t * ldq + static_cast<long long>(h) * D;
        load8(src + sub * 8, v[u]);
      }
#pragma unroll
      for (int u = 0; u < ROWS_IN_FLIGHT; ++u) {
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) ss += v[u][i] * v[u][i];
        ss = group_sum<LPH>(ss);
        const float r = rsqrtf(ss / D + eps);
        float y[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) y[i] = v[u][i] * r * (isk[u] ? wkv[i] : wqv[i]);
        rotate8<LPH>(y, o, c, sn, sub, rope_dim, style, false);
        if (ok[u]) {
          __nv_bfloat16* dst = isk[u] ? k_out + (t * Hk + (hh[u] - Hq)) * D : q_out + (t * Hq + hh[u]) * D;
          store8(dst + sub * 8, o);
          if (sub == 0) inv_rms[t * Ht + hh[u]] = r;
        }
      }
    }
  }
}

template <int LPH>
__global__ void __launch_bounds__(256) qk_norm_rope_bwd_kernel(
    const __nv_bfloat16* __restrict__ dq_out, const __nv_bfloat16* __restrict__ dk_out, const __nv_bfloat16* __restrict__ q,
    const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ wk,
    const float* __restrict__ cos_t, const float* __restrict__ sin_t, const float* __restrict__ inv_rms, long long T, int Hq,
    int Hk, int rope_dim, long long ldq, long long ldk, bool zero_centered, int style, __nv_bfloat16* __restrict__ dq,
    __nv_bfloat16* __restrict__ dk, float* __restrict__ dw_partial /* [grid, 2, D] */) {
  constexpr int D = LPH * 8;
  constexpr int GROUPS = 32 / LPH;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, sub = lane % LPH, grp = lane / LPH;
  const int Ht = Hq + Hk;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wqv[8], wkv[8], accq[8], acck[8];
  load8(wq + sub * 8, wqv);
  load8(wk + sub * 8, wkv);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (zero_centered) { wqv[i] += 1.f; wkv[i] += 1.f; }
    accq[i] = 0.f; acck[i] = 0.f;
  }
  const int head_iters = (Ht + GROUPS * ROWS_IN_FLIGHT - 1) / (GROUPS * ROWS_IN_FLIGHT);
  for (long long t = warp; t < T; t += warps) {
    float c[8], sn[8];
    load_angles(cos_t, sin_t, t, rope_dim, sub, c, sn);
    for (int hi = 0; hi < head_iters; ++hi) {
      float g[ROWS_IN_FLIGHT][8], x[ROWS_IN_FLIGHT][8], rr[ROWS_IN_FLIGHT];
      long long off[ROWS_IN_FLIGHT];
      bool ok[ROWS_IN_FLIGHT], isk[ROWS_IN_FLIGHT];
#pragma unroll
      for (int u = 0; u < ROWS_IN_FLIGHT; ++u) {
        const int hraw = (hi * ROWS_IN_FLIGHT + u) * GROUPS + grp;
        ok[u] = hraw < Ht;
        const int h = ok[u] ? hraw : 0;
        isk[u] = h >= Hq;
        const __nv_bfloat16* xs = isk[u] ? k + t * ldk + static_cast<long long>(h - Hq) * D : q + t * ldq + static_cast<long long>(h) * D;
        off[u] = isk[u] ? (t * Hk + (h - Hq)) * D : (t * Hq + h) * D;
        load8((isk[u] ? dk_out : dq_out) + off[u] + sub * 8, g[u]);
        load8(xs + sub * 8, x[u]);
        rr[u] = inv_rms[t * Ht + h];
      }
#pragma unroll
      for (int u = 0; u < ROWS_IN_FLIGHT; ++u) {
        float dy[8], dx[8];
        rotate8<LPH>(g[u], dy, c, sn, sub, rope_dim, style, true);
        const float r = rr[u];
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xhat = x[u][i] * r;
          const float gw = dy[i] * (isk[u] ? wkv[i] : wqv[i]);
          dot += gw * xhat;
          if (ok[u]) { if (isk[u]) acck[i] += dy[i] * xhat; else accq[i] += dy[i] * xhat; }
          dx[i] = gw;
          x[u][i] = xhat;
        }
        dot = group_sum<LPH>(dot) / D;
#pragma unroll
        for (int i = 0; i < 8; ++i) dx[i] = r * (dx[i] - x[u][i] * dot);
        if (ok[u]) store8((isk[u] ? dk : dq) + off[u] + sub * 8, dx);
      }
    }
  }
  // weight gradients: fold the head groups of a warp, then the 8 warps of the block, into one partial row per block
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int offl = LPH; offl < 32; offl <<= 1) {
      accq[i] += __shfl_xor_sync(0xffffffffu, accq[i], offl);
      acck[i] += __shfl_xor_sync(0xffffffffu, acck[i], offl);
    }
  }
  __shared__ float red[8][2][D];
  if (grp == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      red[wid][0][sub * 8 + i] = accq[i];
      red[wid][1][sub * 8 + i] = acck[i];
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 2 * D; e += blockDim.x) {
    const int which = e / D, d = e - which * D;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][which][d];
    dw_partial[(static_cast<long long>(blockIdx.x) * 2 + which) * D + d] = s;
  }
}

// partial [blocks, 2, D] -> dwq[D], dwk[D]; one block per 32 columns, 8 row-lanes x 32 columns of threads
__global__ void __launch_bounds__(256) qk_dw_reduce_kernel(const float* __restrict__ partial, int blocks, int D,
                                                           float* __restrict__ dwq, float* __restrict__ dwk) {
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);  // column in [0, 2D)
  const int rl = threadIdx.x >> 5;
  float s = 0.f;
  if (col < 2 * D)
    for (int b = rl; b < blocks; b += 8) s += partial[static_cast<long long>(b) * 2 * D + col];
  __shared__ float sm[8][32];
  sm[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && col < 2 * D) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
    if (col < D) dwq[col] = t; else dwk[col - D] = t;
  }
}

inline int sms() {
  static int n = 0;
  if (!n) { int d; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); }
  return n;
}

inline void check_dims(int D, int rope_dim) {
  if ((D != 64 && D != 128 && D != 256) || rope_dim > D || rope_dim % 16 != 0)
    throw std::runtime_error("d9d qk_norm_rope: head_dim must be 64/128/256 and rope_dim a multiple of 16");
}

}  // namespace

int qk_norm_rope_grid(long long T, int Ht) {
  (void)Ht;
  long long blocks = (T + 7) / 8;  // one warp per token
  const long long cap = static_cast<long long>(sms()) * 8;
  if (blocks > cap) blocks = cap;
  return static_cast<int>(blocks > 0 ? blocks : 1);
}

void qk_norm_rope_fwd(const void* q, const void* k, const void* wq, const void* wk, const float* cos_t, const float* sin_t,
                      long long T, int Hq, int Hk, int D, int rope_dim, long long ldq, long long ldk, float eps,
                      bool zero_centered, int style, void* q_out, void* k_out, float* inv_rms, cudaStream_t s) {
  if (T == 0) return;
  check_dims(D, rope_dim);
  const int grid = qk_norm_rope_grid(T, Hq + Hk);
#define D9D_QKF(V)                                                                                                   \
  qk_norm_rope_fwd_kernel<V><<<grid, 256, 0, s>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)wq, \
      (const __nv_bfloat16*)wk, cos_t, sin_t, T, Hq, Hk, rope_dim, ldq, ldk, eps, zero_centered, style,                 \
      (__nv_bfloat16*)q_out, (__nv_bfloat16*)k_out, inv_rms)
  if (D == 64) D9D_QKF(8); else if (D == 128) D9D_QKF(16); else D9D_QKF(32);
#undef D9D_QKF
}

void qk_norm_rope_bwd(const void* dq_out, const void* dk_out, const void* q, const void* k, const void* wq, const void* wk,
                      const float* cos_t, const float* sin_t, const float* inv_rms, long long T, int Hq, int Hk, int D,
                      int rope_dim, long long ldq, long long ldk, bool zero_centered, int style, void* dq, void* dk,
                      float* dw_partial, float* dwq, float* dwk, cudaStream_t s) {
  check_dims(D, rope_dim);
  if (T == 0) {  // no token contributes: the weight gradients are zero (the reduce kernel that writes them does not run)
    cudaMemsetAsync(dwq, 0, static_cast<size_t>(D) * sizeof(float), s);
    cudaMemsetAsync(dwk, 0, static_cast<size_t>(D) * sizeof(float), s);
    return;
  }
  const int grid = qk_norm_rope_grid(T, Hq + Hk);
#define D9D_QKB(V)                                                                                                   \
  qk_norm_rope_bwd_kernel<V><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dq_out, (const __nv_bfloat16*)dk_out,        \
      (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)wq, (const __nv_bfloat16*)wk, cos_t, sin_t, \
      inv_rms, T, Hq, Hk, rope_dim, ldq, ldk, zero_centered, style, (__nv_bfloat16*)dq, (__nv_bfloat16*)dk, dw_partial)
  if (D == 64) D9D_QKB(8); else if (D == 128) D9D_QKB(16); else D9D_QKB(32);
#undef D9D_QKB
  qk_dw_reduce_kernel<<<(2 * D + 31) / 32, 256, 0, s>>>(dw_partial, grid, D, dwq, dwk);
}

}  // namespace d9d
