// fp8 (e4m3) GEMM launchers + the quantisation kernels that produce their operands.
//   quantize_rowwise     x[M,K] bf16 -> q[M,K] e4m3, scale[M]            (scale = amax / 448 per row)
//   quantize_colwise_t   x[E,R,C] bf16 -> qT[E,C,R] e4m3, scale[E,C]   (transposed copy, scale per column of every x[e])
//   quantize_segments_t  x[cap,C] bf16 -> qT[C,cap] e4m3, scale[E,C]   (transposed copy, scale per column of every expert's
//                                                                      rows; pad rows come out as zeros)
//   quantize_mx          x[M,K] bf16 -> q[M,K] e4m3, UE8M0 scale blocks  (one scale per 32 K-elements, 128-row x 4-group blocks)
//   quantize_blockwise   x[R,C] bf16 -> e4m3 with fp32 scales per 1x128 row group, 128x1 column group (transposed copy) or
//                        128x128 block (either copy), stored k-block-major for the BLOCKWISE GEMM
//   quantize_expert_blocks / quantize_blockwise_tiles  the same blockwise groups for the MoE experts: every expert's weight
//                        blocks (batched over E), and the MoE layout's row / 128-token groups, skipping unused 128-row tiles
//   gemm_fp8 / gemm_mxfp8  D[M,N] bf16 = scaled A·B^T on wgmma e4m3 (MX: per-32-K scales applied in registers), the
//                          grouped expert GEMMs (GROUPED_M / GROUPED_K) and the BLOCKWISE GEMM (bf16 / fp32 D), see
//                          gemm_fp8_sm90.cuh
#include <cuda_fp8.h>

#include "gemm_fp8_sm90.cuh"
#include "gemm_host.cuh"

namespace d9d {
namespace {

constexpr float E4M3_MAX = 448.f;

// Scale of a group with the given amax: amax / 448, at least FLT_MIN (2^-126), and 1 for an all-zero group.  The library
// builds with fast math, where amax / 448 below FLT_MIN flushes to zero and 1 / 0 is inf: every code of the group would
// become NaN or +-448.  With the floor, the reciprocal is at most 2^126 and every code stays finite.
__device__ __forceinline__ float e4m3_scale(float amax) { return amax > 0.f ? fmaxf(amax / E4M3_MAX, 0x1p-126f) : 1.f; }

__device__ __forceinline__ uint16_t cvt_e4m3x2(float lo, float hi) {
  return static_cast<uint16_t>(__nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, __NV_E4M3));
}

__device__ __forceinline__ void load8_bf16(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 raw = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y), c = unpack_bf16x2(raw.z), d = unpack_bf16x2(raw.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}

__device__ __forceinline__ uint2 quant8(const float (&v)[8], float inv) {
  uint2 o;
  o.x = cvt_e4m3x2(v[0] * inv, v[1] * inv) | (static_cast<uint32_t>(cvt_e4m3x2(v[2] * inv, v[3] * inv)) << 16);
  o.y = cvt_e4m3x2(v[4] * inv, v[5] * inv) | (static_cast<uint32_t>(cvt_e4m3x2(v[6] * inv, v[7] * inv)) << 16);
  return o;
}

// ---- row-wise: one warp per row, K % 8 == 0 --------------------------------------------------------------------
__global__ void quant_rowwise_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale,
                                     long long M, int K, long long ldx) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const __nv_bfloat16* xr = x + row * ldx;
  float amax = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    float v[8];
    load8_bf16(xr + k, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(v[i]));
  }
  amax = warp_max(amax);
  const float s = e4m3_scale(amax);
  const float inv = 1.f / s;
  if (lane == 0) scale[row] = s;
  uint8_t* qr = q + row * K;
  for (int k = lane * 8; k < K; k += 256) {
    float v[8];
    load8_bf16(xr + k, v);
    *reinterpret_cast<uint2*>(qr + k) = quant8(v, inv);
  }
}

// ---- column-wise + transpose -----------------------------------------------------------------------------------
// Which rows of x form one scale group ("plane") and where they go in qT:
//   batched  (tile_group == nullptr): plane e = blockIdx.z is x + e * x_plane [R, C] -> qt + e * q_plane [C, R]
//   segments (tile_group != nullptr): one x [R = cap, C] -> qt [C, cap]; row r belongs to expert g = tile_group[r / 128]
//            and is quantised with expert g's scales when r < seg_offsets[g] + counts[g]; every other row is written as
//            a zero (and never read).  Scale groups start on 128-row boundaries, so a 64- or 128-row tile has one expert.
struct ColTPlanes {
  long long x_plane, q_plane;
  const int* tile_group;
  const int* seg_offsets;
  const int* counts;
  int num_planes;  // E: planes of amax / scale ([E, C])
};

// expert of the 128-row-aligned tile starting at row r0 and the end of its valid rows (-1 / r0: no valid rows)
__device__ __forceinline__ int segment_of(const ColTPlanes& pl, long long r0, long long& valid_end) {
  const int g = pl.tile_group[r0 / 128];
  valid_end = g >= 0 ? static_cast<long long>(pl.seg_offsets[g]) + pl.counts[g] : r0;
  return g;
}

// pass 1: amax per column (non-negative floats order like their bit patterns: atomicMax on the int view)
__global__ void col_amax_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ amax, long long R, int C, long long ldx,
                                int rows_per_block, ColTPlanes pl) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long r0 = static_cast<long long>(blockIdx.y) * rows_per_block;
  long long r1 = min(R, r0 + rows_per_block);
  int g = blockIdx.z;
  if (pl.tile_group != nullptr) {
    long long valid_end;
    g = segment_of(pl, r0, valid_end);
    if (g < 0) return;
    r1 = min(r1, valid_end);
  } else {
    x += g * pl.x_plane;
  }
  float m = 0.f;
  for (long long r = r0; r < r1; ++r) m = fmaxf(m, fabsf(__bfloat162float(x[r * ldx + c])));
  atomicMax(reinterpret_cast<int*>(amax) + static_cast<long long>(g) * C + c, __float_as_int(m));
}

// pass 2: 64 x 64 tile through shared memory; amax is turned into the scales by the blocks of the first tile row
__global__ void quant_colwise_t_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ amax, uint8_t* __restrict__ qt,
                                       float* __restrict__ scale, long long R, int C, long long ldx, long long ldq, ColTPlanes pl) {
  __shared__ uint8_t tile[64][64 + 4];
  const int c0 = blockIdx.x * 64;
  const long long r0 = static_cast<long long>(blockIdx.y) * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;  // 256 threads: 64 columns x 4 row phases
  const int c = c0 + tx;
  const bool segments = pl.tile_group != nullptr;
  int g = blockIdx.z;
  long long r_end = R;
  if (segments) {
    g = -1;
    r_end = r0;
    if (r0 < R) g = segment_of(pl, r0, r_end);
  } else {
    x += g * pl.x_plane;
    qt += g * pl.q_plane;
  }
  auto put_scale = [&](int e) {
    scale[static_cast<long long>(e) * C + c] = e4m3_scale(amax[static_cast<long long>(e) * C + c]);
  };
  if (blockIdx.y == 0 && c < C) {
    if (segments) {
      for (int e = ty; e < pl.num_planes; e += 4) put_scale(e);  // every expert's, also of those without rows
    } else if (ty == 0) {
      put_scale(g);
    }
  }
  float inv = 0.f;
  if (c < C && g >= 0) {
    inv = 1.f / e4m3_scale(amax[static_cast<long long>(g) * C + c]);
  }
  for (int i = ty; i < 64; i += 4) {
    const long long r = r0 + i;
    float v = 0.f;
    if (r < r_end && c < C) v = __bfloat162float(x[r * ldx + c]) * inv;
    tile[tx][i] = static_cast<uint8_t>(__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3));
  }
  __syncthreads();
  // write qT[c0 + j, r0 .. r0+63]: 64 bytes per output row, 4 rows per pass
  for (int j = ty; j < 64; j += 4) {
    const long long r = r0 + tx;
    if (c0 + j < C && r < R) qt[static_cast<long long>(c0 + j) * ldq + r] = tile[j][tx];
  }
}

// ---- MX: one thread per 32-element group -----------------------------------------------------------------------
__global__ void quant_mx_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf, long long M,
                                int K, long long ldx) {
  const int groups_per_row = K / 32;
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= M * groups_per_row) return;
  const long long row = t / groups_per_row;
  const int g = static_cast<int>(t - row * groups_per_row);
  const __nv_bfloat16* src = x + row * ldx + g * 32;
  float v[4][8];
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    load8_bf16(src + j * 8, v[j]);
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(v[j][i]));
  }
  // smallest power of two 2^e with amax / 2^e <= 448 = 1.75 * 2^8: with amax = m * 2^x (1 <= m < 2) that is
  // e = x - 8 (+1 if m > 1.75) - exact integer arithmetic on the float's bit pattern
  int e = -127;
  if (amax > 0.f) {
    const uint32_t bits = __float_as_uint(amax);
    e = static_cast<int>((bits >> 23) & 0xFF) - 127 - 8 + ((bits & 0x7FFFFF) > 0x600000 ? 1 : 0);
    e = max(-126, min(126, e));
  }
  const float inv = (e == -127) ? 0.f : __uint_as_float(static_cast<uint32_t>(127 - e) << 23);
  uint8_t* dst = q + row * K + g * 32;
#pragma unroll
  for (int j = 0; j < 4; ++j) *reinterpret_cast<uint2*>(dst + j * 8) = quant8(v[j], inv);
  const long long blk = (row / 128) * (K / 128) + (g / 4);
  const int r = static_cast<int>(row % 128);
  sf[blk * 512 + (r % 32) * 16 + (r / 32) * 4 + (g % 4)] = static_cast<uint8_t>(e + 127);
}

// ---- blockwise: one CTA per 128 x 128 tile of x, single pass ------------------------------------------------------
// Every scale group (1 x 128 row group, 128 x 1 column group, 128 x 128 block) lies inside one tile, so the tile's amax
// needs no second pass, atomics or scratch.  Thread (tx, ty) of 256 holds rows 8 ty .. 8 ty + 7 and columns
// 8 tx .. 8 tx + 7 of the tile; elements past R / C are read as zero (a partial group's scale covers its valid elements).
//   not transposed: q[r, c] row pitch ldq bytes; s[c / 128][r] (ROW: the row group's scale, BLOCK: the block's)
//   transposed:     q[c, r] row pitch ldq bytes, columns r in [R, ldq) written as zeros; s[r / 128][c] (COL / BLOCK)
// GROUP is a BlockGroup (d9d_ops.h).

// quant_blockwise_tile: the tile (row_tile, col_tile) of x, the work of one CTA of 256 threads.
template <int GROUP, bool TRANSPOSE>
__device__ __forceinline__ void quant_blockwise_tile(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ s,
                                                     long long R, int C, long long ldx, long long ldq, long long lds,
                                                     unsigned row_tile, unsigned col_tile) {
  static_assert(GROUP == GROUP_BLOCK || (GROUP == GROUP_ROW) != TRANSPOSE, "row groups: plain copy; column groups: transposed");
  __shared__ float red[8][128];                          // per-warp partial amax (COL: per column, BLOCK: one value)
  __shared__ uint32_t tq[TRANSPOSE ? 128 : 1][33];       // transposed tile: 128 columns x 128 row bytes (+1 word pad)
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = static_cast<long long>(row_tile) * 128;
  const int c0 = col_tile * 128;
  const int cc = c0 + 8 * tx;
  float v[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = r0 + 8 * ty + i;
    if (r < R && cc < C) {
      load8_bf16(x + r * ldx + cc, v[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
  }
  // scales: the ROW group of each of this thread's rows, the COL group of each of its columns, or the BLOCK's
  float inv_r[8], inv_c[8];
  if constexpr (GROUP == GROUP_ROW) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) a = fmaxf(a, fabsf(v[i][j]));
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));  // the 16 threads of the row
      const float sc = e4m3_scale(a);
      inv_r[i] = 1.f / sc;
      const long long r = r0 + 8 * ty + i;
      if (tx == 0 && r < R) s[static_cast<long long>(col_tile) * lds + r] = sc;
    }
  } else if constexpr (GROUP == GROUP_COL) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) a = fmaxf(a, fabsf(v[i][j]));
      a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 16));  // the warp's two row slices
      if (lane < 16) red[warp][8 * tx + j] = a;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) a = fmaxf(a, red[w][8 * tx + j]);
      const float sc = e4m3_scale(a);
      inv_c[j] = 1.f / sc;
      if (ty == 0 && cc + j < C) s[static_cast<long long>(row_tile) * lds + cc + j] = sc;
    }
  } else {
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) a = fmaxf(a, fabsf(v[i][j]));
    a = warp_max(a);
    if (lane == 0) red[warp][0] = a;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < 8; ++w) a = fmaxf(a, red[w][0]);
    const float sc = e4m3_scale(a);
    inv_r[0] = 1.f / sc;
    // one scale per row (plain copy) or per column (transposed copy) of the block: 128 values, 256 threads
    if (threadIdx.x < 128) {
      if constexpr (TRANSPOSE) {
        if (c0 + static_cast<int>(threadIdx.x) < C) s[static_cast<long long>(row_tile) * lds + c0 + threadIdx.x] = sc;
      } else {
        if (r0 + threadIdx.x < R) s[static_cast<long long>(col_tile) * lds + r0 + threadIdx.x] = sc;
      }
    }
  }
  auto inv_of = [&](int i, int j) {
    if constexpr (GROUP == GROUP_ROW) return inv_r[i];
    else if constexpr (GROUP == GROUP_COL) return inv_c[j];
    else return inv_r[0];
  };
  if constexpr (!TRANSPOSE) {
    if (cc >= C) return;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long r = r0 + 8 * ty + i;
      if (r >= R) break;
      float w[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = v[i][j] * inv_of(i, j);
      *reinterpret_cast<uint2*>(q + r * ldq + cc) = quant8(w, 1.f);
    }
  } else {
    // column 8 tx + j of the tile becomes row 8 tx + j of the transposed tile; this thread's 8 rows are its bytes 8 ty ..
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        lo |= static_cast<uint32_t>(__nv_cvt_float_to_fp8(v[i][j] * inv_of(i, j), __NV_SATFINITE, __NV_E4M3)) << (8 * i);
        hi |= static_cast<uint32_t>(__nv_cvt_float_to_fp8(v[i + 4][j] * inv_of(i + 4, j), __NV_SATFINITE, __NV_E4M3)) << (8 * i);
      }
      tq[8 * tx + j][2 * ty] = lo;
      tq[8 * tx + j][2 * ty + 1] = hi;
    }
    __syncthreads();
    // 16 bytes per thread: 8 threads per output row of 128 bytes, 32 rows per pass; pad columns up to ldq get the zeros
    // of the rows past R
#pragma unroll
    for (int pass = 0; pass < 4; ++pass) {
      const int row = pass * 32 + (threadIdx.x >> 3), seg = threadIdx.x & 7;
      const long long col = r0 + 16 * seg;
      if (c0 + row < C && col < ldq) {
        const uint4 w = make_uint4(tq[row][4 * seg], tq[row][4 * seg + 1], tq[row][4 * seg + 2], tq[row][4 * seg + 3]);
        *reinterpret_cast<uint4*>(q + static_cast<long long>(c0 + row) * ldq + col) = w;
      }
    }
  }
}

template <int GROUP, bool TRANSPOSE>
__global__ void __launch_bounds__(256) quant_blockwise_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                                              float* __restrict__ s, long long R, int C, long long ldx, long long ldq,
                                                              long long lds) {
  quant_blockwise_tile<GROUP, TRANSPOSE>(x, q, s, R, C, ldx, ldq, lds, blockIdx.y, blockIdx.x);
}

// The 128x128 blocks of every expert's weight w[e] (blockIdx.z = e): planes of x and q R * C elements apart, of s
// s_plane floats apart.
template <bool TRANSPOSE>
__global__ void __launch_bounds__(256) quant_expert_blocks_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                                                  float* __restrict__ s, long long R, int C, long long ldq,
                                                                  long long lds, long long s_plane) {
  const long long e = blockIdx.z;
  quant_blockwise_tile<GROUP_BLOCK, TRANSPOSE>(x + e * R * C, q + e * R * C, s + e * s_plane, R, C, C, ldq, lds, blockIdx.y, blockIdx.x);
}

// The MoE layout x[cap, C] (cap a multiple of 128) in 128-row tiles: a tile whose tile_group entry is -1 is skipped (its
// codes and scales are left as they were).  Row groups (plain copy) quantise every row of a tile in use; the transposed
// 128-token groups end at the expert's last row, rows past it come out as zeros.
template <int GROUP, bool TRANSPOSE>
__global__ void __launch_bounds__(256) quant_blockwise_tiles_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                                                    float* __restrict__ s, long long R, int C, long long ldx,
                                                                    long long ldq, long long lds, const int* __restrict__ tile_group,
                                                                    const int* __restrict__ seg_offsets, const int* __restrict__ counts) {
  const int g = tile_group[blockIdx.y];
  if (g < 0) return;
  const long long r_end = TRANSPOSE ? static_cast<long long>(seg_offsets[g]) + counts[g] : R;
  quant_blockwise_tile<GROUP, TRANSPOSE>(x, q, s, r_end, C, ldx, ldq, lds, blockIdx.y, blockIdx.x);
}

// 2-D map, or 3-D ([d2, d1, d0], box depth 1) when d2 > 0
CUtensorMap make_tmap_u8(const void* base, uint64_t d0, uint64_t d1, uint64_t stride1_bytes, uint32_t box0, uint32_t box1,
                         uint64_t d2 = 0, uint64_t stride2_bytes = 0) {
  CUtensorMap m;
  const cuuint32_t rank = d2 > 0 ? 3 : 2;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (strides[0] & 15) != 0 || (rank == 3 && (strides[1] & 15) != 0))
    throw std::runtime_error("d9d gemm_fp8: operand base / row pitch must be 16-byte aligned for TMA");
  CUresult r = gemm::get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, rank, const_cast<void*>(base), dims, strides, box, estr,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("d9d gemm_fp8: cuTensorMapEncodeTiled failed: " + std::to_string(r));
  return m;
}

template <int BLOCK_N, int SCALING, int MODE = gemm::DENSE, int EPI = gemm::EPI_BF16>
void launch_fp8(const Fp8GemmArgs& a, cudaStream_t stream) {
  using C = fp8::Cfg<BLOCK_N, SCALING>;
  auto kern = fp8::gemm_fp8_kernel<BLOCK_N, SCALING, MODE, EPI>;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    configured = true;
  }
  // GROUPED_K: A [M, k_total] and B [N, k_total], the reduction over the grouped rows; GROUPED_M: B [E, N, K]
  const uint64_t k_dim = MODE == gemm::GROUPED_K ? static_cast<uint64_t>(a.k_total) : static_cast<uint64_t>(a.K);
  CUtensorMap ta = make_tmap_u8(a.A, k_dim, a.M, a.lda, fp8::BLOCK_K, fp8::BLOCK_M);
  CUtensorMap tb = MODE == gemm::GROUPED_M ? make_tmap_u8(a.B, a.K, a.N, a.ldb, fp8::BLOCK_K, BLOCK_N, a.num_groups, a.b_group_stride)
                                           : make_tmap_u8(a.B, k_dim, a.N, a.ldb, fp8::BLOCK_K, BLOCK_N);
  CUtensorMap td;
  constexpr bool out_bf16 = (EPI == gemm::EPI_BF16 || EPI == gemm::EPI_BF16_ACC);
  const uint64_t groups = MODE == gemm::GROUPED_K ? a.num_groups : 1;
  if (!gemm::make_tmap_out(&td, a.D, out_bf16, a.N, a.M, groups, a.ldd, a.d_group_stride))
    throw std::runtime_error("d9d gemm_fp8: output must be 16-byte aligned with 16-byte row (and expert) pitches");
  fp8::Params p{};
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.scale_a = a.scale_a; p.scale_b = a.scale_b; p.scale_scalar = a.scale_scalar;
  p.sfa = a.sfa; p.sfb = a.sfb;
  p.num_groups = a.num_groups; p.tile_group = a.tile_group; p.group_offsets = a.group_offsets;
  const long long tiles = static_cast<long long>((a.M + fp8::BLOCK_M - 1) / fp8::BLOCK_M) * ((a.N + BLOCK_N - 1) / BLOCK_N) *
                          (MODE == gemm::GROUPED_K ? a.num_groups : 1);
  if (tiles <= 0) return;
  const int grid = static_cast<int>(tiles < gemm::sm_count() ? tiles : gemm::sm_count());
  kern<<<grid, fp8::NUM_THREADS, C::SMEM_BYTES, stream>>>(ta, tb, td, p);
}

}  // namespace

void quantize_rowwise_e4m3(const void* x, void* q, float* scale, long long M, int K, long long ldx, cudaStream_t stream) {
  if (M <= 0) return;
  if (K % 8 != 0) throw std::runtime_error("d9d quantize_rowwise: K must be a multiple of 8");
  const int warps = 4;
  quant_rowwise_kernel<<<static_cast<unsigned>((M + warps - 1) / warps), warps * 32, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q), scale, M, K, ldx);
}

void quantize_colwise_t_e4m3(const void* x, void* qt, float* scale, float* amax_scratch, long long R, int C, long long ldx,
                             long long ldq, cudaStream_t stream, int E) {
  if (R <= 0 || C <= 0 || E <= 0) return;
  cudaMemsetAsync(amax_scratch, 0, sizeof(float) * C * E, stream);
  const ColTPlanes pl{R * ldx, C * ldq, nullptr, nullptr, nullptr, E};
  const int rows_per_block = 256;
  dim3 g1((C + 127) / 128, static_cast<unsigned>((R + rows_per_block - 1) / rows_per_block), E);
  col_amax_kernel<<<g1, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_scratch, R, C, ldx, rows_per_block, pl);
  dim3 g2((C + 63) / 64, static_cast<unsigned>((R + 63) / 64), E);
  quant_colwise_t_kernel<<<g2, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_scratch, static_cast<uint8_t*>(qt),
                                                 scale, R, C, ldx, ldq, pl);
}

void quantize_segments_t_e4m3(const void* x, void* qt, float* scale, float* amax_scratch, const int* tile_group,
                              const int* seg_offsets, const int* counts, int E, long long R, int C, long long ldx, long long ldq,
                              cudaStream_t stream) {
  if (C <= 0 || E <= 0) return;
  cudaMemsetAsync(amax_scratch, 0, sizeof(float) * C * E, stream);
  const ColTPlanes pl{0, 0, tile_group, seg_offsets, counts, E};
  // R (the capacity) is a multiple of 128: one expert per 128-row block of pass 1; pass 2 writes the scales of all E
  // experts from its first tile row, so it runs even when R is 0
  if (R > 0) {
    dim3 g1((C + 127) / 128, static_cast<unsigned>(R / 128));
    col_amax_kernel<<<g1, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_scratch, R, C, ldx, 128, pl);
  }
  dim3 g2((C + 63) / 64, static_cast<unsigned>(R > 0 ? R / 64 : 1));
  quant_colwise_t_kernel<<<g2, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_scratch, static_cast<uint8_t*>(qt),
                                                 scale, R, C, ldx, ldq, pl);
}

void quantize_mx_e4m3(const void* x, void* q, void* sf, long long M, int K, long long ldx, cudaStream_t stream) {
  if (M <= 0) return;
  if (K % 128 != 0) throw std::runtime_error("d9d quantize_mx: K must be a multiple of 128");
  const long long n = M * (K / 32);
  quant_mx_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x),
                                                                             static_cast<uint8_t*>(q), static_cast<uint8_t*>(sf), M, K, ldx);
}

void quantize_blockwise_e4m3(const void* x, void* q, float* scale, long long R, int C, long long ldx, long long ldq, long long lds,
                             BlockGroup group, bool transpose, cudaStream_t stream) {
  if (R <= 0 || C <= 0) return;
  if (C % 8 != 0) throw std::runtime_error("d9d quantize_blockwise: C must be a multiple of 8");
  const dim3 grid(static_cast<unsigned>((C + 127) / 128), static_cast<unsigned>((R + 127) / 128));
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  auto* qb = static_cast<uint8_t*>(q);
  if (group == GROUP_ROW && !transpose)
    quant_blockwise_kernel<GROUP_ROW, false><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds);
  else if (group == GROUP_COL && transpose)
    quant_blockwise_kernel<GROUP_COL, true><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds);
  else if (group == GROUP_BLOCK && !transpose)
    quant_blockwise_kernel<GROUP_BLOCK, false><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds);
  else if (group == GROUP_BLOCK && transpose)
    quant_blockwise_kernel<GROUP_BLOCK, true><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds);
  else
    throw std::runtime_error("d9d quantize_blockwise: row groups give a plain copy, column groups a transposed one");
}

void quantize_expert_blocks_e4m3(const void* w, void* q, float* scale, int E, long long R, int C, long long lds, bool transpose,
                                 cudaStream_t stream) {
  if (E <= 0 || R <= 0 || C <= 0) return;
  if (C % 8 != 0 || (transpose && R % 16 != 0)) throw std::runtime_error("d9d quantize_expert_blocks: C must be a multiple of 8 (R of 16)");
  const dim3 grid(static_cast<unsigned>((C + 127) / 128), static_cast<unsigned>((R + 127) / 128), static_cast<unsigned>(E));
  const auto* xb = static_cast<const __nv_bfloat16*>(w);
  auto* qb = static_cast<uint8_t*>(q);
  if (transpose) {
    const long long s_plane = (R + 127) / 128 * lds;
    quant_expert_blocks_kernel<true><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, R, lds, s_plane);
  } else {
    const long long s_plane = (C + 127) / 128 * lds;
    quant_expert_blocks_kernel<false><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, C, lds, s_plane);
  }
}

void quantize_blockwise_tiles_e4m3(const void* x, void* q, float* scale, const int* tile_group, const int* seg_offsets,
                                   const int* counts, long long R, int C, long long ldx, long long ldq, long long lds, bool transpose,
                                   cudaStream_t stream) {
  if (R <= 0 || C <= 0) return;
  if (R % 128 != 0 || C % 8 != 0) throw std::runtime_error("d9d quantize_blockwise_tiles: R must be a multiple of 128 and C of 8");
  const dim3 grid(static_cast<unsigned>((C + 127) / 128), static_cast<unsigned>(R / 128));
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  auto* qb = static_cast<uint8_t*>(q);
  if (transpose)
    quant_blockwise_tiles_kernel<GROUP_COL, true><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds, tile_group, seg_offsets, counts);
  else
    quant_blockwise_tiles_kernel<GROUP_ROW, false><<<grid, 256, 0, stream>>>(xb, qb, scale, R, C, ldx, ldq, lds, tile_group, seg_offsets, counts);
}

void gemm_fp8(const Fp8GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0) return;
  switch (a.scaling) {
    case fp8::BLOCKWISE:
      if (a.scale_a == nullptr || a.scale_b == nullptr) throw std::runtime_error("d9d gemm_fp8_blockwise: both scale tensors are required");
      switch (a.mode) {
        case gemm::DENSE:
          if (a.epi == gemm::EPI_BF16) launch_fp8<128, fp8::BLOCKWISE, gemm::DENSE, gemm::EPI_BF16>(a, stream);
          else if (a.epi == gemm::EPI_F32) launch_fp8<128, fp8::BLOCKWISE, gemm::DENSE, gemm::EPI_F32>(a, stream);
          else throw std::runtime_error("d9d gemm_fp8_blockwise: bf16 or fp32 store only");
          break;
        case gemm::GROUPED_M:
          if (a.epi == gemm::EPI_BF16) launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_M, gemm::EPI_BF16>(a, stream);
          else if (a.epi == gemm::EPI_BF16_ACC) launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_M, gemm::EPI_BF16_ACC>(a, stream);
          else throw std::runtime_error("d9d gemm_fp8_blockwise: GROUPED_M supports bf16 store / accumulate only");
          break;
        case gemm::GROUPED_K:
          switch (a.epi) {
            case gemm::EPI_BF16: launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_K, gemm::EPI_BF16>(a, stream); break;
            case gemm::EPI_F32: launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_K, gemm::EPI_F32>(a, stream); break;
            case gemm::EPI_F32_ACC: launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_K, gemm::EPI_F32_ACC>(a, stream); break;
            case gemm::EPI_BF16_ACC: launch_fp8<128, fp8::BLOCKWISE, gemm::GROUPED_K, gemm::EPI_BF16_ACC>(a, stream); break;
            default: throw std::runtime_error("d9d gemm_fp8_blockwise: GROUPED_K supports fp32 / bf16 store / accumulate only");
          }
          break;
      }
      break;
    case fp8::MX:
      if (a.K % 128 != 0 || a.sfa == nullptr || a.sfb == nullptr)
        throw std::runtime_error("d9d gemm_mxfp8: K must be a multiple of 128 and both scale-factor tensors are required");
      launch_fp8<128, fp8::MX>(a, stream);
      break;
    case fp8::ROWCOL:
      switch (a.mode) {
        case gemm::GROUPED_M:
          if (a.epi == gemm::EPI_BF16) launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_M, gemm::EPI_BF16>(a, stream);
          else if (a.epi == gemm::EPI_BF16_ACC) launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_M, gemm::EPI_BF16_ACC>(a, stream);
          else throw std::runtime_error("d9d gemm_fp8: GROUPED_M supports bf16 store / accumulate only");
          break;
        case gemm::GROUPED_K:
          switch (a.epi) {
            case gemm::EPI_BF16: launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_K, gemm::EPI_BF16>(a, stream); break;
            case gemm::EPI_F32: launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_K, gemm::EPI_F32>(a, stream); break;
            case gemm::EPI_F32_ACC: launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_K, gemm::EPI_F32_ACC>(a, stream); break;
            case gemm::EPI_BF16_ACC: launch_fp8<128, fp8::ROWCOL, gemm::GROUPED_K, gemm::EPI_BF16_ACC>(a, stream); break;
            default: throw std::runtime_error("d9d gemm_fp8: GROUPED_K supports fp32 / bf16 store / accumulate only");
          }
          break;
        case gemm::DENSE:
          // 128-wide tiles only: a 256-wide fp32 accumulator (128 registers per consumer thread) spills at the kernel's
          // 168-register budget
          launch_fp8<128, fp8::ROWCOL>(a, stream);
          break;
      }
      break;
  }
}

}  // namespace d9d
