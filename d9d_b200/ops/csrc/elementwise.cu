// d9d_b200 — bandwidth-bound sm_90a kernels: RMSNorm fwd/bwd, SiLU·mul, stochastic-rounding copy,
// multi-tensor SR-AdamW, RoPE, grad utilities.  All 128-bit vectorised, fp32 math.
#include <stdexcept>

#include "common.cuh"
#include "d9d_ops.h"

namespace d9d {

int rms_norm_bwd_num_partials();

namespace {

// ---------------------------------------------------------------- typed 8-wide vector IO -------
template <typename T>
struct Vec8;  // 8 elements as fp32 in registers

template <>
struct Vec8<__nv_bfloat16> {
  static __device__ __forceinline__ void load(const void* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
  }
  static __device__ __forceinline__ void store(void* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};

template <>
struct Vec8<float> {
  static __device__ __forceinline__ void load(const void* p, float (&f)[8]) {
    const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  static __device__ __forceinline__ void store(void* p, const float (&f)[8]) {
    reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
};

template <>
struct Vec8<__half> {
  static __device__ __forceinline__ void load(const void* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void store(void* p, const float (&f)[8]) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};

inline int num_sms() {
  static int n = 0;
  if (!n) { int d; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); }
  return n;
}

// Persistent kernels (each block loops over rows and owns one partial-dW row) must be launched with exactly as many blocks
// as fit on the device at once: a grid of 1.5 "waves" leaves the last half wave running at half occupancy.
template <typename K>
inline int resident_blocks(K kernel, int threads, size_t smem) {
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
  if (per_sm < 1) per_sm = 1;
  return per_sm * num_sms();
}

// Rows are kept in registers in their *packed* storage type (16 bytes = 8 bf16/fp16 values; fp32: 32 bytes) and unpacked on
// use — half the registers of an fp32 copy, which is what decides how many rows an SM keeps in flight.
template <typename T> struct Raw8 { uint4 v; };
template <> struct Raw8<float> { float4 a, b; };

template <typename T>
__device__ __forceinline__ Raw8<T> raw_load(const T* p) {
  Raw8<T> r;
  r.v = *reinterpret_cast<const uint4*>(p);
  return r;
}
template <>
__device__ __forceinline__ Raw8<float> raw_load<float>(const float* p) {
  Raw8<float> r;
  r.a = reinterpret_cast<const float4*>(p)[0];
  r.b = reinterpret_cast<const float4*>(p)[1];
  return r;
}
template <typename T>
__device__ __forceinline__ void raw_unpack(const Raw8<T>& r, float (&f)[8]) {
  Vec8<T>::load(&r.v, f);
}
template <>
__device__ __forceinline__ void raw_unpack<float>(const Raw8<float>& r, float (&f)[8]) {
  f[0] = r.a.x; f[1] = r.a.y; f[2] = r.a.z; f[3] = r.a.w; f[4] = r.b.x; f[5] = r.b.y; f[6] = r.b.z; f[7] = r.b.w;
}

template <typename T>
__device__ __forceinline__ void load_weight(const T* w, int vi, bool zero_centered, float (&wf)[8]) {
  Vec8<T>::load(w + vi * 8, wf);  // a few KiB shared by every row: stays in L1
  if (zero_centered) {
#pragma unroll
    for (int i = 0; i < 8; ++i) wf[i] += 1.f;
  }
}

// ================================================================= RMSNorm ======================
// A row is owned by G lanes (G in {8,16,32}) each holding VPL 8-wide vectors; N <= G*VPL*8, N % 8 == 0.
// Rows are register-resident: one read of x, one write of out (HBM roofline = 2 B/elt r + 2 B/elt w for bf16).
template <typename T, int G, int VPL>
__global__ void __launch_bounds__(256) rms_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                      T* __restrict__ out, float* __restrict__ inv_rms, long long M,
                                                      int N, float eps, bool zero_centered) {
  constexpr int ROWS_PER_WARP = 32 / G;
  constexpr int U = (VPL <= 2) ? 2 : 1;  // short rows: two row groups in flight per warp
  const int lane = threadIdx.x & 31, sub = lane % G, rsub = lane / G;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nvec = N >> 3;
  for (long long rb = warp_global * ROWS_PER_WARP * U; rb < M; rb += warps_total * ROWS_PER_WARP * U) {
    Raw8<T> xr[U][VPL];
    long long rows[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      rows[u] = rb + u * ROWS_PER_WARP + rsub;
      ok[u] = rows[u] < M;  // trip count is warp-uniform so the shuffles below stay convergent
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int vi = sub + v * G;
        if (vi < nvec && ok[u]) xr[u][v] = raw_load<T>(x + rows[u] * N + vi * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float ss = 0.f;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        if (sub + v * G < nvec && ok[u]) {
          float xf[8];
          raw_unpack<T>(xr[u][v], xf);
#pragma unroll
          for (int i = 0; i < 8; ++i) ss += xf[i] * xf[i];
        }
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float ir = rsqrtf(ss / static_cast<float>(N) + eps);
      if (sub == 0 && inv_rms && ok[u]) inv_rms[rows[u]] = ir;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int vi = sub + v * G;
        if (vi < nvec && ok[u]) {
          float xf[8], wf[8], o[8];
          raw_unpack<T>(xr[u][v], xf);
          load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] = xf[i] * ir * wf[i];
          Vec8<T>::store(out + rows[u] * N + vi * 8, o);
        }
      }
    }
  }
}

// Backward: persistent, register-resident rows; per-lane dw accumulators, block reduce, deterministic partials.
template <typename T, int G, int VPL>
__global__ void __launch_bounds__(256) rms_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ x,
                                                      const T* __restrict__ w, const float* __restrict__ inv_rms,
                                                      T* __restrict__ dx, float* __restrict__ dw_partial, long long M,
                                                      int N, bool zero_centered) {
  constexpr int ROWS_PER_WARP = 32 / G;
  extern __shared__ float red[];  // [warps][N]
  const int lane = threadIdx.x & 31, sub = lane % G, rsub = lane / G, warp = threadIdx.x >> 5;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nvec = N >> 3;
  const int nwarps = blockDim.x >> 5;

  float dwf[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int i = 0; i < 8; ++i) dwf[v][i] = 0.f;
  for (long long rb = warp_global * ROWS_PER_WARP; rb < M; rb += warps_total * ROWS_PER_WARP) {
    const long long row = rb + rsub;
    const bool row_ok = row < M;  // trip count is warp-uniform so the shuffles below stay convergent
    const float ir = row_ok ? inv_rms[row] : 0.f;
    Raw8<T> xr[VPL], gr[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = sub + v * G;
      if (vi < nvec && row_ok) {
        xr[v] = raw_load<T>(x + row * N + vi * 8);
        gr[v] = raw_load<T>(dout + row * N + vi * 8);
      }
    }
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = sub + v * G;
      if (vi < nvec && row_ok) {
        float xf[8], df[8], wf[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = xf[i] * ir;
          dwf[v][i] += df[i] * xh;
          dot += df[i] * wf[i] * xh;
        }
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float mean_dot = dot / static_cast<float>(N);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = sub + v * G;
      if (vi < nvec && row_ok) {
        float xf[8], df[8], wf[8], o[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = ir * (df[i] * wf[i] - xf[i] * ir * mean_dot);
        Vec8<T>::store(dx + row * N + vi * 8, o);
      }
    }
  }
  // combine the ROWS_PER_WARP sub-rows inside the warp, then across warps through smem
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int o = G; o < 32; o <<= 1) dwf[v][i] += __shfl_xor_sync(0xffffffffu, dwf[v][i], o);
  if (rsub == 0) {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = sub + v * G;
      if (vi < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) red[warp * N + vi * 8 + i] = dwf[v][i];
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    float s = 0.f;
    for (int wi = 0; wi < nwarps; ++wi) s += red[wi * N + c];
    dw_partial[static_cast<long long>(blockIdx.x) * N + c] = s;
  }
}

// partial [num_partials, N] -> dw[N]; one block per 32 columns, 8 row lanes x 32 columns of threads (fixed order: deterministic)
template <typename T>
__global__ void __launch_bounds__(256) rms_dw_reduce_kernel(const float* __restrict__ partial, int num_partials, int N,
                                                            T* __restrict__ dw) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  float s = 0.f;
  if (c < N)
    for (int p = rl; p < num_partials; p += 8) s += partial[static_cast<long long>(p) * N + c];
  __shared__ float sm[8][32];
  sm[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && c < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
    dw[c] = static_cast<T>(t);
  }
}

template <typename T, int G, int VPL>
void rms_fwd_launch(const void* x, const void* w, void* out, float* inv_rms, long long M, int N, float eps, bool zc,
                    cudaStream_t s) {
  constexpr int ROWS_PER_WARP = 32 / G;
  const long long warps_needed = (M + ROWS_PER_WARP - 1) / ROWS_PER_WARP;
  long long blocks = (warps_needed + 7) / 8;
  const long long max_blocks = static_cast<long long>(num_sms()) * 8;
  if (blocks > max_blocks) blocks = max_blocks;
  rms_fwd_kernel<T, G, VPL><<<static_cast<int>(blocks), 256, 0, s>>>(
      static_cast<const T*>(x), static_cast<const T*>(w), static_cast<T*>(out), inv_rms, M, N, eps, zc);
}

template <typename T, int G, int VPL>
void rms_bwd_launch(const void* dout, const void* x, const void* w, const float* inv_rms, void* dx, void* dw,
                    float* dw_partial, long long M, int N, bool zc, cudaStream_t s) {
  constexpr int ROWS_PER_WARP = 32 / G;
  const long long warps_needed = (M + ROWS_PER_WARP - 1) / ROWS_PER_WARP;
  long long blocks = (warps_needed + 7) / 8;
  const size_t smem = static_cast<size_t>(8) * N * sizeof(float);
  auto kern = rms_bwd_kernel<T, G, VPL>;
  if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  long long max_blocks = resident_blocks(kern, 256, smem);
  if (max_blocks > rms_norm_bwd_num_partials()) max_blocks = rms_norm_bwd_num_partials();
  if (blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  kern<<<static_cast<int>(blocks), 256, smem, s>>>(static_cast<const T*>(dout), static_cast<const T*>(x),
                                                   static_cast<const T*>(w), inv_rms, static_cast<T*>(dx), dw_partial,
                                                   M, N, zc);
  rms_dw_reduce_kernel<T><<<(N + 31) / 32, 256, 0, s>>>(dw_partial, static_cast<int>(blocks), N, static_cast<T*>(dw));
}


// ---- CTA-per-row variants for wide rows (N up to 256*VPL*8) ----
__device__ __forceinline__ float block_sum_256(float v, float* sm) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[w] = v;
  __syncthreads();
  float t = sm[threadIdx.x & 7];
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

template <typename T, int VPL>
__global__ void __launch_bounds__(256) rms_fwd_block_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                            T* __restrict__ out, float* __restrict__ inv_rms,
                                                            long long M, int N, float eps, bool zero_centered) {
  // 256 threads x VPL vectors cover a row; rows narrower than that simply leave the tail threads idle for the loads,
  // which lets N <= 4096 run with VPL = 2 and therefore few registers / many resident blocks
  __shared__ float sm[8];
  const int nvec = N >> 3;
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    Raw8<T> xr[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) xr[v] = raw_load<T>(x + row * N + vi * 8);
    }
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      if (threadIdx.x + v * 256 < nvec) {
        float xf[8];
        raw_unpack<T>(xr[v], xf);
#pragma unroll
        for (int i = 0; i < 8; ++i) ss += xf[i] * xf[i];
      }
    }
    ss = block_sum_256(ss, sm);
    const float ir = rsqrtf(ss / static_cast<float>(N) + eps);
    if (threadIdx.x == 0 && inv_rms) inv_rms[row] = ir;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        float xf[8], wf[8], o[8];
        raw_unpack<T>(xr[v], xf);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = xf[i] * ir * wf[i];
        Vec8<T>::store(out + row * N + vi * 8, o);
      }
    }
  }
}

template <typename T, int VPL>
__global__ void __launch_bounds__(256, (VPL <= 2) ? 5 : 3) rms_bwd_block_kernel(const T* __restrict__ dout, const T* __restrict__ x,
                                                                                const T* __restrict__ w,
                                                                                const float* __restrict__ inv_rms, T* __restrict__ dx,
                                                                                float* __restrict__ dw_partial, long long M, int N,
                                                                                bool zero_centered) {
  // dW accumulators live in shared memory (thread t owns the same columns for every row, so plain += is race free):
  // registers only hold the packed x / dy vectors, which keeps five blocks resident per SM.
  extern __shared__ float dw_acc[];  // [N]
  __shared__ float sm[8];
  const int nvec = N >> 3;
  for (int c = threadIdx.x; c < N; c += 256) dw_acc[c] = 0.f;
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    const float ir = inv_rms[row];
    Raw8<T> xr[VPL], gr[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        xr[v] = raw_load<T>(x + row * N + vi * 8);
        gr[v] = raw_load<T>(dout + row * N + vi * 8);
      }
    }
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        float xf[8], df[8], wf[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
        float4* acc = reinterpret_cast<float4*>(dw_acc + vi * 8);
        float4 a0 = acc[0], a1 = acc[1];
        const float xh0 = xf[0] * ir, xh1 = xf[1] * ir, xh2 = xf[2] * ir, xh3 = xf[3] * ir;
        const float xh4 = xf[4] * ir, xh5 = xf[5] * ir, xh6 = xf[6] * ir, xh7 = xf[7] * ir;
        a0.x += df[0] * xh0; a0.y += df[1] * xh1; a0.z += df[2] * xh2; a0.w += df[3] * xh3;
        a1.x += df[4] * xh4; a1.y += df[5] * xh5; a1.z += df[6] * xh6; a1.w += df[7] * xh7;
        acc[0] = a0; acc[1] = a1;
        dot += df[0] * wf[0] * xh0 + df[1] * wf[1] * xh1 + df[2] * wf[2] * xh2 + df[3] * wf[3] * xh3 +
               df[4] * wf[4] * xh4 + df[5] * wf[5] * xh5 + df[6] * wf[6] * xh6 + df[7] * wf[7] * xh7;
      }
    }
    dot = block_sum_256(dot, sm);
    const float mean_dot = dot / static_cast<float>(N);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        float xf[8], df[8], wf[8], o[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = ir * (df[i] * wf[i] - xf[i] * ir * mean_dot);
        Vec8<T>::store(dx + row * N + vi * 8, o);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < N; c += 256) dw_partial[static_cast<long long>(blockIdx.x) * N + c] = dw_acc[c];
}

// register-accumulator variant (faster for rows of <= 4096 elements: two vectors per thread)
template <typename T, int VPL>
__global__ void __launch_bounds__(256, (VPL <= 2) ? 4 : 2) rms_bwd_block_reg_kernel(const T* __restrict__ dout, const T* __restrict__ x,
                                                            const T* __restrict__ w, const float* __restrict__ inv_rms,
                                                            T* __restrict__ dx, float* __restrict__ dw_partial,
                                                            long long M, int N, bool zero_centered) {
  __shared__ float sm[8];
  const int nvec = N >> 3;
  float dwf[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int i = 0; i < 8; ++i) dwf[v][i] = 0.f;
  for (long long row = blockIdx.x; row < M; row += gridDim.x) {
    const float ir = inv_rms[row];
    Raw8<T> xr[VPL], gr[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        xr[v] = raw_load<T>(x + row * N + vi * 8);
        gr[v] = raw_load<T>(dout + row * N + vi * 8);
      }
    }
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        float xf[8], df[8], wf[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = xf[i] * ir;
          dwf[v][i] += df[i] * xh;
          dot += df[i] * wf[i] * xh;
        }
      }
    }
    dot = block_sum_256(dot, sm);
    const float mean_dot = dot / static_cast<float>(N);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int vi = threadIdx.x + v * 256;
      if (vi < nvec) {
        float xf[8], df[8], wf[8], o[8];
        raw_unpack<T>(xr[v], xf);
        raw_unpack<T>(gr[v], df);
        load_weight<T>(w, vi, zero_centered, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = ir * (df[i] * wf[i] - xf[i] * ir * mean_dot);
        Vec8<T>::store(dx + row * N + vi * 8, o);
      }
    }
  }
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    const int vi = threadIdx.x + v * 256;
    if (vi < nvec) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dw_partial[static_cast<long long>(blockIdx.x) * N + vi * 8 + i] = dwf[v][i];
    }
  }
}

template <typename T, int VPL>
void rms_fwd_block_launch(const void* x, const void* w, void* out, float* inv_rms, long long M, int N, float eps,
                          bool zc, cudaStream_t s) {
  long long blocks = M;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  rms_fwd_block_kernel<T, VPL><<<static_cast<int>(blocks), 256, 0, s>>>(
      static_cast<const T*>(x), static_cast<const T*>(w), static_cast<T*>(out), inv_rms, M, N, eps, zc);
}

template <typename T, int VPL>
void rms_bwd_block_launch(const void* dout, const void* x, const void* w, const float* inv_rms, void* dx, void* dw,
                          float* dw_partial, long long M, int N, bool zc, cudaStream_t s) {
  long long blocks = M;
  if (blocks < 1) blocks = 1;
  if constexpr (VPL <= 2) {
    long long cap = resident_blocks(rms_bwd_block_reg_kernel<T, VPL>, 256, 0);
    if (cap > rms_norm_bwd_num_partials()) cap = rms_norm_bwd_num_partials();
    if (blocks > cap) blocks = cap;
    rms_bwd_block_reg_kernel<T, VPL><<<static_cast<int>(blocks), 256, 0, s>>>(
        static_cast<const T*>(dout), static_cast<const T*>(x), static_cast<const T*>(w), inv_rms, static_cast<T*>(dx), dw_partial, M,
        N, zc);
    rms_dw_reduce_kernel<T><<<(N + 31) / 32, 256, 0, s>>>(dw_partial, static_cast<int>(blocks), N, static_cast<T*>(dw));
    return;
  }
  auto kern = rms_bwd_block_kernel<T, VPL>;
  const size_t smem = static_cast<size_t>(N) * sizeof(float);
  if (smem > 40 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  long long cap = resident_blocks(kern, 256, smem);
  if (cap > rms_norm_bwd_num_partials()) cap = rms_norm_bwd_num_partials();
  if (blocks > cap) blocks = cap;
  kern<<<static_cast<int>(blocks), 256, smem, s>>>(
      static_cast<const T*>(dout), static_cast<const T*>(x), static_cast<const T*>(w), inv_rms, static_cast<T*>(dx),
      dw_partial, M, N, zc);
  rms_dw_reduce_kernel<T><<<(N + 31) / 32, 256, 0, s>>>(dw_partial, static_cast<int>(blocks), N, static_cast<T*>(dw));
}

#define D9D_RMS_FWD_DISPATCH(T, ...)                                                     \
  do {                                                                                   \
    if (N <= 64) rms_fwd_launch<T, 8, 1>(__VA_ARGS__);                                   \
    else if (N <= 128) rms_fwd_launch<T, 16, 1>(__VA_ARGS__);                            \
    else if (N <= 256) rms_fwd_launch<T, 32, 1>(__VA_ARGS__);                            \
    else if (N <= 512) rms_fwd_launch<T, 32, 2>(__VA_ARGS__);                            \
    else if (N <= 1024) rms_fwd_launch<T, 32, 4>(__VA_ARGS__);                           \
    else if (N <= 2048) rms_fwd_launch<T, 32, 8>(__VA_ARGS__);                           \
    else if (N <= 4096) rms_fwd_block_launch<T, 2>(__VA_ARGS__);                         \
    else if (N <= 8192) rms_fwd_block_launch<T, 4>(__VA_ARGS__);                         \
    else if (N <= 16384) rms_fwd_block_launch<T, 8>(__VA_ARGS__);                        \
    else throw std::runtime_error("d9d rms_norm: N > 16384 not supported");              \
  } while (0)

#define D9D_RMS_BWD_DISPATCH(T, ...)                                                     \
  do {                                                                                   \
    if (N <= 64) rms_bwd_launch<T, 8, 1>(__VA_ARGS__);                                   \
    else if (N <= 128) rms_bwd_launch<T, 16, 1>(__VA_ARGS__);                            \
    else if (N <= 256) rms_bwd_launch<T, 32, 1>(__VA_ARGS__);                            \
    else if (N <= 512) rms_bwd_launch<T, 32, 2>(__VA_ARGS__);                            \
    else if (N <= 1024) rms_bwd_launch<T, 32, 4>(__VA_ARGS__);                           \
    else if (N <= 2048) rms_bwd_block_launch<T, 1>(__VA_ARGS__);                         \
    else if (N <= 4096) rms_bwd_block_launch<T, 2>(__VA_ARGS__);                         \
    else if (N <= 8192) rms_bwd_block_launch<T, 4>(__VA_ARGS__);                         \
    else throw std::runtime_error("d9d rms_norm bwd: N > 8192 not supported");           \
  } while (0)

}  // namespace

int rms_norm_bwd_num_partials() { return num_sms() * 8; }

void rms_norm_fwd(const void* x, const void* w, void* out, float* inv_rms, long long M, int N, float eps,
                  bool zero_centered, DType dtype, cudaStream_t stream) {
  if (M == 0) return;
  if (N % 8 != 0) throw std::runtime_error("d9d rms_norm: N must be a multiple of 8");
  if (dtype == DTYPE_BF16) D9D_RMS_FWD_DISPATCH(__nv_bfloat16, x, w, out, inv_rms, M, N, eps, zero_centered, stream);
  else if (dtype == DTYPE_F32) D9D_RMS_FWD_DISPATCH(float, x, w, out, inv_rms, M, N, eps, zero_centered, stream);
  else D9D_RMS_FWD_DISPATCH(__half, x, w, out, inv_rms, M, N, eps, zero_centered, stream);
}

void rms_norm_bwd(const void* dout, const void* x, const void* w, const float* inv_rms, void* dx, void* dw,
                  float* dw_partial, long long M, int N, bool zero_centered, DType dtype, cudaStream_t stream) {
  if (N % 8 != 0) throw std::runtime_error("d9d rms_norm: N must be a multiple of 8");
  if (dtype == DTYPE_BF16) D9D_RMS_BWD_DISPATCH(__nv_bfloat16, dout, x, w, inv_rms, dx, dw, dw_partial, M, N, zero_centered, stream);
  else if (dtype == DTYPE_F32) D9D_RMS_BWD_DISPATCH(float, dout, x, w, inv_rms, dx, dw, dw_partial, M, N, zero_centered, stream);
  else D9D_RMS_BWD_DISPATCH(__half, dout, x, w, inv_rms, dx, dw, dw_partial, M, N, zero_centered, stream);
}

// ================================================================= SiLU * mul ===================
namespace {

template <typename T>
__global__ void __launch_bounds__(256) silu_mul_fwd_kernel(const T* __restrict__ x, const T* __restrict__ y,
                                                           T* __restrict__ out, long long n) {
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float a[8], b[8], o[8];
    Vec8<T>::load(x + i * 8, a);
    Vec8<T>::load(y + i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-a[j]));
      // silu is rounded to the storage dtype before the product (matches the reference numerics)
      const float silu = static_cast<float>(static_cast<T>(a[j] * sg));
      o[j] = silu * b[j];
    }
    Vec8<T>::store(out + i * 8, o);
  }
  // tail
  const long long tail0 = nvec << 3;
  for (long long i = tail0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float a = static_cast<float>(x[i]), b = static_cast<float>(y[i]);
    const float sg = 1.f / (1.f + __expf(-a));
    out[i] = static_cast<T>(static_cast<float>(static_cast<T>(a * sg)) * b);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) silu_mul_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ x,
                                                           const T* __restrict__ y, T* __restrict__ dx,
                                                           T* __restrict__ dy, long long n) {
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float g[8], a[8], b[8], da[8], db[8];
    Vec8<T>::load(dout + i * 8, g);
    Vec8<T>::load(x + i * 8, a);
    Vec8<T>::load(y + i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-a[j]));
      const float silu = a[j] * sg;
      db[j] = g[j] * silu;
      da[j] = g[j] * b[j] * (sg + silu * (1.f - sg));
    }
    Vec8<T>::store(dx + i * 8, da);
    Vec8<T>::store(dy + i * 8, db);
  }
  const long long tail0 = nvec << 3;
  for (long long i = tail0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float g = static_cast<float>(dout[i]), a = static_cast<float>(x[i]), b = static_cast<float>(y[i]);
    const float sg = 1.f / (1.f + __expf(-a));
    const float silu = a * sg;
    dy[i] = static_cast<T>(g * silu);
    dx[i] = static_cast<T>(g * b * (sg + silu * (1.f - sg)));
  }
}

inline int ew_grid(long long nvec) {
  long long blocks = (nvec + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

// One warp per row chunk: out = silu(x)*y*p[row]; cols % 8 == 0
__global__ void __launch_bounds__(256) silu_mul_probs_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 const __nv_bfloat16* __restrict__ y,
                                                                 const float* __restrict__ probs,
                                                                 __nv_bfloat16* __restrict__ out, long long rows,
                                                                 int cols, const int* __restrict__ valid_rows) {
  if (valid_rows != nullptr) rows = min(rows, static_cast<long long>(*valid_rows));  // rows past the last expert segment are never read
  const int vec_per_row = cols >> 3;
  const long long nvec = rows * vec_per_row;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const long long r = i / vec_per_row;
    const float p = probs[r];
    float a[8], b[8], o[8];
    Vec8<__nv_bfloat16>::load(x + i * 8, a);
    Vec8<__nv_bfloat16>::load(y + i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-a[j]));
      o[j] = a[j] * sg * b[j] * p;
    }
    Vec8<__nv_bfloat16>::store(out + i * 8, o);
  }
}

// one warp per row: needs the row-wise reduction for dprobs
__global__ void __launch_bounds__(256) silu_mul_probs_bwd_kernel(
    const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ y,
    const float* __restrict__ probs, __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dy,
    float* __restrict__ dprobs, long long rows, int cols, const int* __restrict__ valid_rows) {
  if (valid_rows != nullptr) rows = min(rows, static_cast<long long>(*valid_rows));
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int vec_per_row = cols >> 3;
  for (long long r = warp_global; r < rows; r += warps_total) {
    const float p = probs[r];
    float acc = 0.f;
    for (int v = lane; v < vec_per_row; v += 32) {
      const long long off = r * cols + v * 8;
      float g[8], a[8], b[8], da[8], db[8];
      Vec8<__nv_bfloat16>::load(dout + off, g);
      Vec8<__nv_bfloat16>::load(x + off, a);
      Vec8<__nv_bfloat16>::load(y + off, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float sg = 1.f / (1.f + __expf(-a[j]));
        const float silu = a[j] * sg;
        acc += g[j] * silu * b[j];
        const float gp = g[j] * p;
        db[j] = gp * silu;
        da[j] = gp * b[j] * (sg + silu * (1.f - sg));
      }
      Vec8<__nv_bfloat16>::store(dx + off, da);
      Vec8<__nv_bfloat16>::store(dy + off, db);
    }
    acc = warp_sum(acc);
    if (lane == 0) dprobs[r] = acc;
  }
}

}  // namespace

void silu_mul_fwd(const void* x, const void* y, void* out, long long n, DType dtype, cudaStream_t s) {
  if (n == 0) return;
  const int grid = ew_grid(n >> 3);
  if (dtype == DTYPE_BF16) silu_mul_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)y, (__nv_bfloat16*)out, n);
  else if (dtype == DTYPE_F32) silu_mul_fwd_kernel<float><<<grid, 256, 0, s>>>((const float*)x, (const float*)y, (float*)out, n);
  else silu_mul_fwd_kernel<__half><<<grid, 256, 0, s>>>((const __half*)x, (const __half*)y, (__half*)out, n);
}

void silu_mul_bwd(const void* dout, const void* x, const void* y, void* dx, void* dy, long long n, DType dtype,
                  cudaStream_t s) {
  if (n == 0) return;
  const int grid = ew_grid(n >> 3);
  if (dtype == DTYPE_BF16) silu_mul_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)x, (const __nv_bfloat16*)y, (__nv_bfloat16*)dx, (__nv_bfloat16*)dy, n);
  else if (dtype == DTYPE_F32) silu_mul_bwd_kernel<float><<<grid, 256, 0, s>>>((const float*)dout, (const float*)x, (const float*)y, (float*)dx, (float*)dy, n);
  else silu_mul_bwd_kernel<__half><<<grid, 256, 0, s>>>((const __half*)dout, (const __half*)x, (const __half*)y, (__half*)dx, (__half*)dy, n);
}

void silu_mul_probs_fwd(const void* x, const void* y, const float* probs, void* out, long long rows, int cols,
                        const int* valid_rows, cudaStream_t s) {
  if (rows == 0) return;
  if (cols % 8) throw std::runtime_error("d9d silu_mul_probs: cols must be a multiple of 8");
  silu_mul_probs_fwd_kernel<<<ew_grid(rows * (cols >> 3)), 256, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)y, probs, (__nv_bfloat16*)out, rows, cols, valid_rows);
}

void silu_mul_probs_bwd(const void* dout, const void* x, const void* y, const float* probs, void* dx, void* dy,
                        float* dprobs, long long rows, int cols, const int* valid_rows, cudaStream_t s) {
  if (rows == 0) return;
  if (cols % 8) throw std::runtime_error("d9d silu_mul_probs: cols must be a multiple of 8");
  long long blocks = (rows + 7) / 8;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  silu_mul_probs_bwd_kernel<<<static_cast<int>(blocks), 256, 0, s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)x, (const __nv_bfloat16*)y, probs, (__nv_bfloat16*)dx, (__nv_bfloat16*)dy, dprobs, rows, cols, valid_rows);
}

// ================================================================= stochastic rounding ==========
namespace {

__global__ void __launch_bounds__(256) sr_copy_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst,
                                                      long long n, uint64_t seed) {
  // each thread handles 8 elements = 2 philox draws (4x32 bits -> 8x16 bits per draw)
  const long long nvec = (n + 7) >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 r = philox4x32(seed, static_cast<uint64_t>(i));
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
    const long long base = i << 3;
    if (base + 8 <= n) {
      const float4 a = reinterpret_cast<const float4*>(src + base)[0];
      const float4 b = reinterpret_cast<const float4*>(src + base)[1];
      const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t lo = sr_bf16_bits(f[2 * j], rr[j] & 0xFFFF);
        const uint32_t hi = sr_bf16_bits(f[2 * j + 1], rr[j] >> 16);
        o[j] = lo | (hi << 16);
      }
      *reinterpret_cast<uint4*>(dst + base) = make_uint4(o[0], o[1], o[2], o[3]);
    } else {
      for (int j = 0; j < 8 && base + j < n; ++j) {
        const uint32_t rnd = (j & 1) ? (rr[j >> 1] >> 16) : (rr[j >> 1] & 0xFFFF);
        dst[base + j] = sr_bf16_bits(src[base + j], rnd);
      }
    }
  }
}

template <bool GRAD_BF16, bool STATE_BF16>
__global__ void __launch_bounds__(256) adamw_sr_kernel(const AdamTensorMeta* __restrict__ metas,
                                                       const int2* __restrict__ block_map, float lr, float beta1,
                                                       float beta2, float eps, float wd, float bc1, float bc2,
                                                       uint64_t seed, const float* __restrict__ grad_scale) {
  const int2 bm = block_map[blockIdx.x];
  const AdamTensorMeta mt = metas[bm.x];
  const long long chunk0 = static_cast<long long>(bm.y) * ADAM_CHUNK;
  const float gs = grad_scale ? *grad_scale : 1.f;
  uint16_t* p = static_cast<uint16_t*>(mt.p);
  const bool aligned = ((reinterpret_cast<uintptr_t>(mt.p) | reinterpret_cast<uintptr_t>(mt.g) |
                         reinterpret_cast<uintptr_t>(mt.m) | reinterpret_cast<uintptr_t>(mt.v)) & 31) == 0;
#pragma unroll 1
  for (int it = 0; it < ADAM_CHUNK / (256 * 8); ++it) {
    const long long base = chunk0 + (static_cast<long long>(it) * 256 + threadIdx.x) * 8;
    if (base >= mt.n) break;
    const int cnt = (mt.n - base >= 8) ? 8 : static_cast<int>(mt.n - base);
    float pf[8], gf[8], mf[8], vf[8];
    if (cnt == 8 && aligned) {
      Vec8<__nv_bfloat16>::load(p + base, pf);
      if (GRAD_BF16) Vec8<__nv_bfloat16>::load(static_cast<const uint16_t*>(mt.g) + base, gf);
      else Vec8<float>::load(static_cast<const float*>(mt.g) + base, gf);
      if (STATE_BF16) {
        Vec8<__nv_bfloat16>::load(static_cast<const uint16_t*>(mt.m) + base, mf);
        Vec8<__nv_bfloat16>::load(static_cast<const uint16_t*>(mt.v) + base, vf);
      } else {
        Vec8<float>::load(static_cast<const float*>(mt.m) + base, mf);
        Vec8<float>::load(static_cast<const float*>(mt.v) + base, vf);
      }
    } else {
      for (int j = 0; j < 8; ++j) {
        pf[j] = gf[j] = mf[j] = vf[j] = 0.f;
        if (j < cnt) {
          pf[j] = __uint_as_float(static_cast<uint32_t>(p[base + j]) << 16);
          gf[j] = GRAD_BF16 ? __uint_as_float(static_cast<uint32_t>(static_cast<const uint16_t*>(mt.g)[base + j]) << 16)
                            : static_cast<const float*>(mt.g)[base + j];
          if (STATE_BF16) {
            mf[j] = __uint_as_float(static_cast<uint32_t>(static_cast<const uint16_t*>(mt.m)[base + j]) << 16);
            vf[j] = __uint_as_float(static_cast<uint32_t>(static_cast<const uint16_t*>(mt.v)[base + j]) << 16);
          } else {
            mf[j] = static_cast<const float*>(mt.m)[base + j];
            vf[j] = static_cast<const float*>(mt.v)[base + j];
          }
        }
      }
    }
    // three independent 16-bit streams per element: params, exp_avg, exp_avg_sq
    const uint64_t ctr = static_cast<uint64_t>((mt.rng_base + base) >> 3);
    const uint4 rp = philox4x32(seed, ctr);
    uint4 rm = make_uint4(0, 0, 0, 0), rv = make_uint4(0, 0, 0, 0);
    if (STATE_BF16) {
      rm = philox4x32(seed + 42, ctr);
      rv = philox4x32(seed + 67, ctr);
    }
    const uint32_t rpa[4] = {rp.x, rp.y, rp.z, rp.w}, rma[4] = {rm.x, rm.y, rm.z, rm.w},
                   rva[4] = {rv.x, rv.y, rv.z, rv.w};
    uint16_t po[8], mo[8], vo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float g = gf[j] * gs;
      float pw = pf[j] * (1.f - lr * wd);
      const float mn = beta1 * mf[j] + (1.f - beta1) * g;
      const float vn = beta2 * vf[j] + (1.f - beta2) * (g * g);
      const float mh = mn / bc1, vh = vn / bc2;
      pw -= (lr * mh) / (sqrtf(vh) + eps);
      const uint32_t sel = (j & 1) ? 16 : 0;
      po[j] = sr_bf16_bits(pw, (rpa[j >> 1] >> sel) & 0xFFFF);
      mf[j] = mn; vf[j] = vn;
      if (STATE_BF16) {
        mo[j] = sr_bf16_bits(mn, (rma[j >> 1] >> sel) & 0xFFFF);
        vo[j] = sr_bf16_bits(vn, (rva[j >> 1] >> sel) & 0xFFFF);
      }
    }
    if (cnt == 8 && aligned) {
      *reinterpret_cast<uint4*>(p + base) = *reinterpret_cast<const uint4*>(po);
      if (STATE_BF16) {
        *reinterpret_cast<uint4*>(static_cast<uint16_t*>(mt.m) + base) = *reinterpret_cast<const uint4*>(mo);
        *reinterpret_cast<uint4*>(static_cast<uint16_t*>(mt.v) + base) = *reinterpret_cast<const uint4*>(vo);
      } else {
        Vec8<float>::store(static_cast<float*>(mt.m) + base, mf);
        Vec8<float>::store(static_cast<float*>(mt.v) + base, vf);
      }
    } else {
      for (int j = 0; j < cnt; ++j) {
        p[base + j] = po[j];
        if (STATE_BF16) {
          static_cast<uint16_t*>(mt.m)[base + j] = mo[j];
          static_cast<uint16_t*>(mt.v)[base + j] = vo[j];
        } else {
          static_cast<float*>(mt.m)[base + j] = mf[j];
          static_cast<float*>(mt.v)[base + j] = vf[j];
        }
      }
    }
  }
}

}  // namespace

void sr_copy_f32_to_bf16(const float* src, void* dst, long long n, uint64_t seed, cudaStream_t s) {
  if (n == 0) return;
  if ((reinterpret_cast<uintptr_t>(src) & 31) || (reinterpret_cast<uintptr_t>(dst) & 15))
    throw std::runtime_error("d9d sr_copy: buffers must be 32B/16B aligned");
  sr_copy_kernel<<<ew_grid((n + 7) >> 3), 256, 0, s>>>(src, static_cast<uint16_t*>(dst), n, seed);
}

void adamw_sr_multi(const AdamTensorMeta* metas, const int2* block_map, int num_blocks, float lr, float beta1,
                    float beta2, float eps, float weight_decay, float bias_corr1, float bias_corr2, uint64_t seed,
                    const float* grad_scale, bool grad_bf16, bool state_bf16, cudaStream_t s) {
  if (num_blocks == 0) return;
#define D9D_ADAM(GB, SB) \
  adamw_sr_kernel<GB, SB><<<num_blocks, 256, 0, s>>>(metas, block_map, lr, beta1, beta2, eps, weight_decay, bias_corr1, bias_corr2, seed, grad_scale)
  if (grad_bf16 && state_bf16) D9D_ADAM(true, true);
  else if (grad_bf16 && !state_bf16) D9D_ADAM(true, false);
  else if (!grad_bf16 && state_bf16) D9D_ADAM(false, true);
  else D9D_ADAM(false, false);
#undef D9D_ADAM
}

// ================================================================= RoPE =========================
namespace {

// One warp per (token, head). Lane l owns D/32 contiguous elements; the HALF-style partner lives in lane l^16.
template <int VEC>  // VEC = D / 32 in {2, 4, 8}
__global__ void __launch_bounds__(256) rope_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                                   const float* __restrict__ cos_cache,
                                                   const float* __restrict__ sin_cache,
                                                   const long long* __restrict__ pos, long long T, int H, int rope_dim,
                                                   long long ldx, long long ldo, int style, bool inverse) {
  constexpr int D = VEC * 32;
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long total = T * H;
  for (long long idx = warp_global; idx < total; idx += warps_total) {
    const long long t = idx / H;
    const int h = static_cast<int>(idx - t * H);
    const __nv_bfloat16* xp = x + t * ldx + static_cast<long long>(h) * D + lane * VEC;
    __nv_bfloat16* op = out + t * ldo + static_cast<long long>(h) * D + lane * VEC;
    float v[VEC];
#pragma unroll
    for (int i = 0; i < VEC; i += 2) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xp + i));
      v[i] = f.x; v[i + 1] = f.y;
    }
    const long long ps = pos[t];
    const float* cp = cos_cache + ps * rope_dim;
    const float* sp = sin_cache + ps * rope_dim;
    float o[VEC];
    if (style == 0) {
      // HALF: out = x*cos + rotate_half(x)*sin, rotate_half(x) = cat(-x2, x1) over the first rope_dim dims
      const int half = rope_dim >> 1;
      float partner[VEC];
      // exchange with the lane holding index (+/- half). Valid when half is a multiple of VEC.
      const int lane_shift = half / VEC;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int e = lane * VEC + i;
        const int src_lane = (e < half) ? lane + lane_shift : lane - lane_shift;
        partner[i] = __shfl_sync(0xffffffffu, v[i], src_lane & 31);
      }
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int e = lane * VEC + i;
        if (e < rope_dim) {
          const float c = cp[e];
          float s = sp[e];
          if (inverse) s = -s;
          const float rot = (e < half) ? -partner[i] : partner[i];
          o[i] = v[i] * c + rot * s;
        } else {
          o[i] = v[i];
        }
      }
    } else {
      // INTERLEAVED: pairs (2i, 2i+1) rotate together; cos/sin indexed by the element (cache is repeat-interleaved)
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        const int e = lane * VEC + i;
        if (e < rope_dim) {
          const float c0 = cp[e], c1 = cp[e + 1];
          float s0 = sp[e], s1 = sp[e + 1];
          if (inverse) { s0 = -s0; s1 = -s1; }
          o[i] = v[i] * c0 - v[i + 1] * s0;
          o[i + 1] = v[i + 1] * c1 + v[i] * s1;
        } else {
          o[i] = v[i]; o[i + 1] = v[i + 1];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < VEC; i += 2) *reinterpret_cast<uint32_t*>(op + i) = pack_bf16x2(o[i], o[i + 1]);
  }
}

}  // namespace

void rope_apply(const void* x, void* out, const float* cos_cache, const float* sin_cache, const long long* pos,
                long long T, int H, int D, int rope_dim, long long ldx, long long ldo, int style, bool inverse,
                cudaStream_t s) {
  if (T == 0 || H == 0) return;
  long long blocks = (T * H + 7) / 8;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  const int grid = static_cast<int>(blocks);
  const int vec = D / 32;
  // rope_dim a multiple of 2 * vec: an odd rope_dim would rotate an element without its partner
  if (D <= 0 || D % 64 != 0 || rope_dim % (2 * vec) != 0 || rope_dim > D)
    throw std::runtime_error("d9d rope: unsupported head_dim / rope_dim combination");
#define D9D_ROPE(V) \
  rope_kernel<V><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)out, cos_cache, sin_cache, pos, T, H, rope_dim, ldx, ldo, style, inverse)
  if (vec == 2) D9D_ROPE(2);
  else if (vec == 4) D9D_ROPE(4);
  else if (vec == 8) D9D_ROPE(8);
  else throw std::runtime_error("d9d rope: head_dim must be 64, 128 or 256");
#undef D9D_ROPE
}

// ================================================================= grad utilities ===============
namespace {

template <typename T>
__global__ void __launch_bounds__(256) sumsq_kernel(const T* __restrict__ x, long long n, float* __restrict__ out) {
  float acc = 0.f;
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float f[8];
    Vec8<T>::load(x + i * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += f[j] * f[j];
  }
  for (long long i = (nvec << 3) + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float f = static_cast<float>(x[i]);
    acc += f * f;
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = sm[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) scale_kernel(T* __restrict__ x, long long n, const float* __restrict__ scale) {
  const float sc = *scale;
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float f[8];
    Vec8<T>::load(x + i * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= sc;
    Vec8<T>::store(x + i * 8, f);
  }
  for (long long i = (nvec << 3) + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    x[i] = static_cast<T>(static_cast<float>(x[i]) * sc);
}

}  // namespace

void sumsq_accumulate(const void* x, long long n, DType dtype, float* out, cudaStream_t s) {
  if (n == 0) return;
  long long blocks = ((n >> 3) + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (dtype == DTYPE_BF16) sumsq_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, n, out);
  else if (dtype == DTYPE_F32) sumsq_kernel<float><<<(int)blocks, 256, 0, s>>>((const float*)x, n, out);
  else sumsq_kernel<__half><<<(int)blocks, 256, 0, s>>>((const __half*)x, n, out);
}

void scale_inplace(void* x, long long n, DType dtype, const float* scale, cudaStream_t s) {
  if (n == 0) return;
  const int grid = ew_grid(n >> 3);
  if (dtype == DTYPE_BF16) scale_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16*)x, n, scale);
  else if (dtype == DTYPE_F32) scale_kernel<float><<<grid, 256, 0, s>>>((float*)x, n, scale);
  else scale_kernel<__half><<<grid, 256, 0, s>>>((__half*)x, n, scale);
}

}  // namespace d9d
