// d9d_b200 — expert-parallel token exchange over NVLink peer memory (replaces the all-to-all of dispatch / combine).
//
// Every rank knows, for each of its (token, slot) pairs, the rank that owns the chosen expert and the row that pair
// occupies in the owner's 128-row aligned, expert-sorted buffer (computed on the device from the exchanged per-expert
// counts; no host synchronisation, no variable-size collective):
//   ep_push      rows are written straight into the owners' GEMM-ready buffers (dispatch forward, combine backward)
//   ep_pull_sum  each token gathers its k expert outputs from the owners and sums them in fp32
//                (combine forward, dispatch backward — optionally also pulling d(prob))
// Both are one warp per row with 16-byte vector accesses on the mapped peer pointers.
#include <stdexcept>

#include "common.cuh"
#include "d9d_ops.h"

namespace d9d {
namespace {

__device__ __forceinline__ uint4 ld_peer_16(const void* p) {
  uint4 v;
  asm volatile("ld.global.relaxed.sys.v4.b32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void st_peer_16(void* p, uint4 v) {
  asm volatile("st.global.relaxed.sys.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__global__ void __launch_bounds__(256) ep_push_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ probs,
                                                      const int* __restrict__ dest_rank, const int* __restrict__ dest_row,
                                                      uint8_t* const* __restrict__ peer_base, long long off_x, long long off_p,
                                                      long long n_pairs, int k, int H) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nvec = H >> 3;
  for (long long i = warp; i < n_pairs; i += warps) {
    const int row = dest_row[i];
    if (row < 0) continue;  // dropped pair
    uint8_t* base = peer_base[dest_rank[i]];
    const uint4* src = reinterpret_cast<const uint4*>(x + (i / k) * H);
    uint4* dst = reinterpret_cast<uint4*>(base + off_x) + static_cast<long long>(row) * nvec;
    for (int c = lane; c < nvec; c += 32) st_peer_16(dst + c, src[c]);
    if (probs != nullptr && lane == 0) reinterpret_cast<float*>(base + off_p)[row] = probs[i];
  }
}

__global__ void __launch_bounds__(256) ep_pull_sum_kernel(uint8_t* const* __restrict__ peer_base, long long off_y, long long off_dp,
                                                          const int* __restrict__ dest_rank, const int* __restrict__ dest_row,
                                                          __nv_bfloat16* __restrict__ y, float* __restrict__ dprobs, long long T,
                                                          int k, int H) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nvec = H >> 3;
  for (long long t = warp; t < T; t += warps) {
    for (int c0 = 0; c0 < nvec; c0 += 32) {
      const int c = c0 + lane;
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < k; ++j) {
        const int row = dest_row[t * k + j];
        if (row < 0 || c >= nvec) continue;
        const uint8_t* base = peer_base[dest_rank[t * k + j]];
        const uint4 v = ld_peer_16(reinterpret_cast<const uint4*>(base + off_y) + static_cast<long long>(row) * nvec + c);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(w[q]);
          acc[2 * q] += f.x; acc[2 * q + 1] += f.y;
        }
      }
      if (c < nvec) {
        uint4 o;
        o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]); o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
        reinterpret_cast<uint4*>(y + t * H)[c] = o;
      }
    }
    if (dprobs != nullptr && lane < k) {
      const int row = dest_row[t * k + lane];
      float d = 0.f;
      if (row >= 0) {
        const float* src = reinterpret_cast<const float*>(peer_base[dest_rank[t * k + lane]] + off_dp) + row;
        asm volatile("ld.global.relaxed.sys.f32 %0, [%1];\n" : "=f"(d) : "l"(src) : "memory");
      }
      dprobs[t * k + lane] = d;
    }
  }
}

inline int sms() {
  static int n = 0;
  if (!n) { int d; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); }
  return n;
}

}  // namespace

void ep_push(const void* x, const float* probs, const int* dest_rank, const int* dest_row, void* const* peer_base, long long off_x,
             long long off_p, long long n_pairs, int k, int H, cudaStream_t stream) {
  if (n_pairs == 0) return;
  if (H % 8 != 0 || (off_x & 15) != 0) throw std::runtime_error("d9d ep_push: H % 8 == 0 and 16-byte aligned regions required");
  if (probs != nullptr && (off_p & 3) != 0) throw std::runtime_error("d9d ep_push: the probability region must be 4-byte aligned");
  long long blocks = (n_pairs + 7) / 8;
  const long long cap = static_cast<long long>(sms()) * 8;
  if (blocks > cap) blocks = cap;
  ep_push_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), probs, dest_rank, dest_row,
                                                               reinterpret_cast<uint8_t* const*>(peer_base), off_x, off_p, n_pairs, k, H);
}

void ep_pull_sum(void* const* peer_base, long long off_y, long long off_dp, const int* dest_rank, const int* dest_row, void* y,
                 float* dprobs, long long T, int k, int H, cudaStream_t stream) {
  if (T == 0) return;
  if (H % 8 != 0 || k > 32 || (off_y & 15) != 0) throw std::runtime_error("d9d ep_pull_sum: H % 8 == 0, k <= 32, aligned regions required");
  if (dprobs != nullptr && (off_dp & 3) != 0) throw std::runtime_error("d9d ep_pull_sum: the d(prob) region must be 4-byte aligned");
  long long blocks = (T + 7) / 8;
  const long long cap = static_cast<long long>(sms()) * 8;
  if (blocks > cap) blocks = cap;
  ep_pull_sum_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(reinterpret_cast<uint8_t* const*>(peer_base), off_y, off_dp, dest_rank,
                                                                   dest_row, static_cast<__nv_bfloat16*>(y), dprobs, T, k, H);
}

}  // namespace d9d
