// Host-side launcher pieces for the wgmma GEMM: TMA descriptor encoding + dispatch helpers.
#pragma once

#include <mutex>
#include <stdexcept>
#include <string>

#include "d9d_ops.h"
#include "gemm_sm90.cuh"

namespace d9d {
namespace gemm {

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // resolved at run time so the extension has no link-time dependency on libcuda (CPU-only build hosts)
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || p == nullptr) throw std::runtime_error("d9d: cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 3-D bf16 tensor map, 128B swizzle. dims/strides innermost-first; strides in elements for dims 1,2.
inline CUtensorMap make_tmap_bf16_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_elems,
                                     uint64_t stride2_elems, uint32_t box0, uint32_t box1) {
  CUtensorMap m;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_elems * 2, stride2_elems * 2};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (strides[0] & 15) != 0 || (strides[1] & 15) != 0)
    throw std::runtime_error("d9d gemm: operand base/strides must be 16-byte aligned for TMA");
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("d9d gemm: cuTensorMapEncodeTiled failed: " + std::to_string(r));
  return m;
}

// Output tensor map: [groups, rows, cols] row-major, box = 16 rows x 128 bytes, 128B swizzle (matches the epilogue's
// per-warp staging layout).  Returns false when base / pitches do not meet TMA's 16-byte alignment rules, and when a row is
// not a whole number of 16-byte chunks: the swizzled TMA store clips a row at 16-byte granularity, so it would write
// past column `cols` into the row padding.
inline bool make_tmap_out(CUtensorMap* m, void* base, bool bf16, uint64_t cols, uint64_t rows, uint64_t groups,
                          uint64_t row_pitch_elems, uint64_t group_pitch_elems) {
  const uint64_t esz = bf16 ? 2 : 4;
  cuuint64_t dims[3] = {cols, rows, groups};
  cuuint64_t strides[2] = {row_pitch_elems * esz, (groups > 1 ? group_pitch_elems : row_pitch_elems * rows) * esz};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(128 / esz), EPI_BOX_ROWS, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (strides[0] & 15) != 0 || (strides[1] & 15) != 0 || ((cols * esz) & 15) != 0)
    return false;
  CUresult r = get_encode_fn()(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base,
                               dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("d9d gemm: cuTensorMapEncodeTiled (output) failed: " + std::to_string(r));
  return true;
}

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

// number of two-CTA clusters that can be resident at once
template <typename Kern>
int max_active_pairs(Kern kern, int smem_bytes) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(sm_count() / 2 * 2));
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.attrs = &attr; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    n = sm_count() / 2;
  }
  return n;
}

template <int MODE, int BLOCK_N, bool A_MN, bool B_MN, int EPI, int COMM = COMM_NONE, int CTAS = 1>
void launch_one(const GemmArgs& a, cudaStream_t stream) {
  using C = Cfg<BLOCK_N, CTAS>;
  auto kern = gemm_kernel<MODE, BLOCK_N, A_MN, B_MN, EPI, COMM, CTAS>;
  static bool configured = false;
  static int pairs = 0;
  if (!configured) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (CTAS == 2) pairs = max_active_pairs(kern, C::SMEM_BYTES);
    configured = true;
  }
  // ---- tensor maps ----
  CUtensorMap ta, tb;
  typename PeerArg<COMM>::type peers{};
  if constexpr (COMM == COMM_WAIT_A) {
    if (a.comm_flags == nullptr || a.comm_block_rows <= 0 || a.comm_block_rows % BLOCK_M != 0)
      throw std::runtime_error("d9d gemm: flag-gated all-gather GEMM needs arrival flags and tile-aligned shard blocks");
  } else if constexpr (COMM != COMM_NONE) {
    if (a.comm_world < 1 || a.comm_world > MAX_PEERS || a.comm_peer_ptrs == nullptr)
      throw std::runtime_error("d9d gemm: fused communication needs 1..8 peer pointers");
    const int unit = (COMM == COMM_AG_A) ? BLOCK_M : (COMM == COMM_RS_D ? 32 : BLOCK_K);
    if (a.comm_block_rows <= 0 || a.comm_block_rows % unit != 0)
      throw std::runtime_error("d9d gemm: the per-rank block of the sharded dim must be a multiple of the tile size");
    for (int r = 0; r < a.comm_world; ++r) {
      const void* base = a.comm_peer_ptrs[r];
      const uint64_t rows = a.comm_rows_local, ld = a.comm_ld;
      if constexpr (COMM == COMM_AG_A) peers.m[r] = make_tmap_bf16_3d(base, a.K, rows, 1, ld, ld * rows, 64, BLOCK_M);
      else if constexpr (COMM == COMM_AG_KA) peers.m[r] = make_tmap_bf16_3d(base, a.M, rows, 1, ld, ld * rows, 64, BLOCK_K);
      else if constexpr (COMM == COMM_AG_KB) peers.m[r] = make_tmap_bf16_3d(base, a.N, rows, 1, ld, ld * rows, 64, BLOCK_K);
      else if (!make_tmap_out(&peers.m[r], const_cast<void*>(base), EPI == EPI_BF16_ACC, a.N, rows, 1, ld, 0))
        throw std::runtime_error("d9d gemm: reduce-scatter output shards must be 16-byte aligned");
    }
  }
  constexpr bool A_FROM_PEERS = (COMM == COMM_AG_A || COMM == COMM_AG_KA);
  constexpr bool B_FROM_PEERS = (COMM == COMM_AG_KB);
  if (MODE == GROUPED_K) {
    // A: [R, M] (M contiguous), B: [R, N] (N contiguous); reduction over grouped rows
    ta = make_tmap_bf16_3d(a.A, a.M, a.k_total, 1, a.lda, a.lda * a.k_total, 64, BLOCK_K);
    tb = make_tmap_bf16_3d(a.B, a.N, a.k_total, 1, a.ldb, a.ldb * a.k_total, 64, BLOCK_K);
  } else {
    const uint64_t g = (MODE == GROUPED_M) ? a.num_groups : 1;
    if (!B_FROM_PEERS) {
      if (!B_MN) tb = make_tmap_bf16_3d(a.B, a.K, a.N, g, a.ldb, a.b_group_stride ? a.b_group_stride : a.ldb * a.N, 64, C::B_ROWS);
      else       tb = make_tmap_bf16_3d(a.B, a.N, a.K, g, a.ldb, a.b_group_stride ? a.b_group_stride : a.ldb * a.K, 64, BLOCK_K);
    }
    if (!A_FROM_PEERS) {
      if (!A_MN) ta = make_tmap_bf16_3d(a.A, a.K, a.M, 1, a.lda, a.lda * a.M, 64, BLOCK_M);
      else       ta = make_tmap_bf16_3d(a.A, a.M, a.K, 1, a.lda, a.lda * a.K, 64, BLOCK_K);
    } else {
      ta = tb;  // placeholder: the kernel loads A through the peer maps
    }
    if (B_FROM_PEERS) tb = ta;
  }
  Params p{};
  CUtensorMap td = ta;  // placeholder when the direct-store epilogue is used
  if (COMM == COMM_RS_D) {
    p.tma_epilogue = 1;  // output tiles are reduce-added through the peer maps
  } else if (EPI != EPI_CE_LSE && EPI != EPI_CE_LSE_SUM) {
    constexpr bool out_bf16 = (EPI == EPI_BF16 || EPI == EPI_BF16_ACC || EPI == EPI_CE_DLOGITS || EPI == EPI_CE_DLOGITS_REG);
    const uint64_t groups = (MODE == GROUPED_K) ? a.num_groups : 1;
    p.tma_epilogue = make_tmap_out(&td, a.D, out_bf16, a.N, a.M, groups, a.ldd, a.d_group_stride) ? 1 : 0;
  }
  p.k_splits = 1;
  const bool can_split = MODE == DENSE && EPI == EPI_F32_ACC && p.tma_epilogue;
  if (a.k_splits > 1 && !can_split)
    throw std::runtime_error("d9d gemm: split-K needs a dense fp32-accumulate GEMM whose output TMA can address");
  if (can_split) {
    // split-K: reduce-adds from several CTAs land on the same tile (fp32 adds in L2; order is not deterministic).
    // A forced count is honoured exactly: slices past the last k-block are empty and add nothing.
    long long splits = a.k_splits;
    if (splits == 0) {
      const long long mn_tiles = ((a.M + C::TILE_M - 1) / C::TILE_M) * ((a.N + BLOCK_N - 1) / BLOCK_N);
      const long long k_blocks = (a.K + BLOCK_K - 1) / BLOCK_K;
      splits = (sm_count() / CTAS) / mn_tiles;
      const long long max_splits = k_blocks / 8;  // keep >= 8 k-blocks (512 deep) per slice
      if (splits > max_splits) splits = max_splits;
      if (splits < 1) splits = 1;
    }
    p.k_splits = static_cast<int>(splits);
  }
  p.M = a.M; p.N = a.N; p.K = a.K; p.num_groups = a.num_groups;
  p.comm_world = a.comm_world; p.comm_block_rows = a.comm_block_rows;
  p.comm_rank = a.comm_rank; p.comm_flags = a.comm_flags;
  p.comm_m_rot = (COMM == COMM_WAIT_A) ? (a.comm_rank * a.comm_block_rows / BLOCK_M) % static_cast<int>((a.M + BLOCK_M - 1) / BLOCK_M) : 0;
  p.D = a.D; p.ldd = a.ldd; p.d_group_stride = a.d_group_stride;
  p.tile_group = a.tile_group; p.group_offsets = a.group_offsets;
  p.ce_target = a.ce_target; p.ce_lse = a.ce_lse; p.ce_grad = a.ce_grad;
  p.ce_part_max = a.ce_part_max; p.ce_part_sum = a.ce_part_sum; p.ce_tgt_logit = a.ce_tgt_logit;
  p.ce_ignore_index = a.ce_ignore_index; p.ce_softcap = a.ce_softcap; p.ce_bias = a.ce_bias;
  p.ce_col_offset = a.ce_col_offset;
  p.ce_part_zsum = a.ce_part_zsum; p.ce_z_loss = a.ce_z_loss; p.ce_smoothing = a.ce_smoothing;
  p.ce_num_classes = a.ce_num_classes;

  const long long m_tiles = (a.M + C::TILE_M - 1) / C::TILE_M, n_tiles = (a.N + BLOCK_N - 1) / BLOCK_N;
  long long tiles = m_tiles * n_tiles * (MODE == GROUPED_K ? a.num_groups : 1) * p.k_splits;
  if (tiles <= 0) return;
  if constexpr (CTAS == 2) {
    // one CTA pair (cluster of 2) per tile
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(2 * (tiles < pairs ? tiles : pairs)));
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = C::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, td, p, peers);
    if (e != cudaSuccess) throw std::runtime_error(std::string("d9d gemm: CTA-pair launch failed: ") + cudaGetErrorString(e));
    return;
  }
  // COMM_WAIT_A runs next to copy / flag kernels of another stream: leave `comm_spare_sms` SMs to them
  const int usable = sm_count() - ((COMM == COMM_WAIT_A) ? a.comm_spare_sms : 0);
  const int grid = static_cast<int>(tiles < usable ? tiles : usable);
  kern<<<grid, NUM_THREADS, C::SMEM_BYTES, stream>>>(ta, tb, td, p, peers);
}

// pick BLOCK_N minimising (waves x tile cost); ties go to the wider tile
inline int pick_block_n(long long m_tiles_x_groups, int N) {
  const int cands[3] = {256, 192, 128};
  int best = 256;
  double best_cost = 1e30;
  for (int bn : cands) {
    const long long tiles = m_tiles_x_groups * ((N + bn - 1) / bn);
    const long long waves = (tiles + sm_count() - 1) / sm_count();
    const double cost = static_cast<double>(waves) * (bn + 24 /*fixed per-tile overhead*/);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

#define D9D_DISPATCH_BN(MODE, AMN, BMN, EPI, bn, args, stream)                     \
  do {                                                                             \
    if ((bn) == 256) launch_one<MODE, 256, AMN, BMN, EPI>(args, stream);           \
    else if ((bn) == 192) launch_one<MODE, 192, AMN, BMN, EPI>(args, stream);      \
    else if ((bn) == 128) launch_one<MODE, 128, AMN, BMN, EPI>(args, stream);      \
    else throw std::runtime_error("d9d gemm: BLOCK_N must be 128, 192 or 256");   \
  } while (0)

#define D9D_DISPATCH_EPI4(MODE, AMN, BMN, epi, bn, args, stream)                                  \
  do {                                                                                            \
    switch (epi) {                                                                                \
      case EPI_BF16: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_BF16, bn, args, stream); break;          \
      case EPI_F32: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_F32, bn, args, stream); break;            \
      case EPI_F32_ACC: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_F32_ACC, bn, args, stream); break;    \
      case EPI_BF16_ACC: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_BF16_ACC, bn, args, stream); break;  \
      default: throw std::runtime_error("d9d gemm: unsupported epilogue for this mode");          \
    }                                                                                             \
  } while (0)

// CTA-pair (two-CTA cluster, B multicast) variants: 256 x {256, 128} tiles
#define D9D_DISPATCH_PAIR_BN(AMN, BMN, EPI, bn, args, stream)                                        \
  do {                                                                                               \
    if ((bn) == 256) launch_one<DENSE, 256, AMN, BMN, EPI, COMM_NONE, 2>(args, stream);              \
    else if ((bn) == 128) launch_one<DENSE, 128, AMN, BMN, EPI, COMM_NONE, 2>(args, stream);         \
    else throw std::runtime_error("d9d gemm: CTA-pair BLOCK_N must be 128 or 256");                 \
  } while (0)

#define D9D_DISPATCH_PAIR_EPI4(AMN, BMN, epi, bn, args, stream)                                      \
  do {                                                                                               \
    switch (epi) {                                                                                   \
      case EPI_BF16: D9D_DISPATCH_PAIR_BN(AMN, BMN, EPI_BF16, bn, args, stream); break;              \
      case EPI_F32: D9D_DISPATCH_PAIR_BN(AMN, BMN, EPI_F32, bn, args, stream); break;                \
      case EPI_F32_ACC: D9D_DISPATCH_PAIR_BN(AMN, BMN, EPI_F32_ACC, bn, args, stream); break;        \
      case EPI_BF16_ACC: D9D_DISPATCH_PAIR_BN(AMN, BMN, EPI_BF16_ACC, bn, args, stream); break;      \
      default: throw std::runtime_error("d9d gemm: unsupported epilogue for this mode");             \
    }                                                                                                \
  } while (0)

// store-only epilogues (layouts that never receive an accumulate request keep the instantiation count down)
#define D9D_DISPATCH_EPI2(MODE, AMN, BMN, epi, bn, args, stream)                                  \
  do {                                                                                            \
    switch (epi) {                                                                                \
      case EPI_BF16: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_BF16, bn, args, stream); break;          \
      case EPI_F32: D9D_DISPATCH_BN(MODE, AMN, BMN, EPI_F32, bn, args, stream); break;            \
      default: throw std::runtime_error("d9d gemm: accumulate epilogue not built for this operand layout"); \
    }                                                                                             \
  } while (0)

}  // namespace gemm
}  // namespace d9d
