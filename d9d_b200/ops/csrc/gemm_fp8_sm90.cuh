// d9d_b200 — persistent warp-specialised wgmma GEMM for 8-bit floating point operands (sm_90a).
//
//   D[M,N] (bf16) = scale( A[M,K] · B[N,K]^T )       A, B: e4m3, K-major.
// The tensor core sums each MMA chain in a reduced-precision accumulator (the tests model it with a unit roundoff of
// 2^-13); fp32 registers hold only what the kernel adds outside a chain.  ROWCOL / MX DENSE: one chain over all of K (ROWCOL) or per
// 32-deep MMA (MX); BLOCKWISE and the grouped modes: one chain per 128-deep k-block (promoted accumulation).
//
// Two scaling recipes share the mainloop:
//   ROWCOL  D = acc * scale_a[row] * scale_b[col]  (per-token / per-output-channel or per-tensor scales, applied in the
//           epilogue)
//   MX      one UE8M0 scale per 32 K-elements of every row of A and B (OCP MXFP8).  The scale-factor blocks (512 bytes =
//           128 rows x 4 K-groups per operand tile) are bulk-copied into shared memory next to the A/B tiles; every K=32
//           wgmma writes a fresh partial product that is added to the accumulator with its row x column scale
//           (Hopper's tensor core has no block-scaled MMA).
//   BLOCKWISE one fp32 scale per (128-deep k-block, row) of A and of B (DeepSeek-V3's 1x128 activation / 128x128 weight
//           groups; a weight block's scale is repeated on each of its 128 rows), stored k-block-major
//           [ceil(K/128), round_up(rows, 128)].  The k-block's four MMAs go into a fresh accumulator that is added to the
//           fp32 accumulator with its row x column scale (promoted accumulation); bf16 or fp32 output.
// Same structure as the bf16 kernel (gemm_sm90.cuh): warpgroup 0 = TMA producer, warpgroups 1-2 = wgmma + epilogue over
// 64 rows each (registers -> swizzled smem -> TMA store); a stage holds 128 bytes of K (= 128 fp8 elements = 4 MMAs).
//
// Every epilogue applies the row and the column scale one at a time, (acc * sa) * sb, never acc * (sa * sb): the library
// builds with fast math (flush to zero), and the product of two small scales flushes to 0 below 2^-126 even when the result
// is a normal number.  With sb <= 1 (quantiser scales are amax / 448) an intermediate flushes only when the result does.
//
// Three problem shapes (gemm::Mode, with the bf16 kernel's tile walk, gemm::get_tile), all K-major:
//   DENSE      D[M,N] bf16
//   GROUPED_M  MoE forward / input gradient: rows of A and D grouped by expert in 128-row segments (tile_group), B is
//              [E, N, K]; scale_a[row], scale_b[e * N + col]; bf16 store or accumulate
//   GROUPED_K  MoE weight gradient: A [M, R] and B [N, R] with the reduction over expert e's rows
//              [group_offsets[e], group_offsets[e+1]), D is [E, M, N]; scale_a[e * M + row], scale_b[e * N + col];
//              fp32 / bf16 store or accumulate (an expert without rows stores zeros and accumulates nothing)
// The grouped modes promote the accumulation: every 128-deep k-block is summed by the tensor core into a fresh
// accumulator, which is then added to the fp32 register accumulator.  Hopper's e4m3 wgmma keeps a reduced-precision
// accumulator inside one MMA chain, and an expert's weight gradient reduces over thousands of tokens.
// The ROWCOL grouped modes live in grouped_tiles() and BLOCKWISE (DENSE and grouped) in blockwise_tiles(), whose DENSE
// producer keeps its own loop; the ROWCOL / MX DENSE instances keep
// their own body, unchanged, so that they compile to exactly the instructions they compiled to before the other modes
// existed (even an unused local in a shared body changed their schedule).
#pragma once

#include "common.cuh"
#include "d9d_ops.h"  // fp8::Scaling
#include "gemm_sm90.cuh"

namespace d9d {
namespace fp8 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 128;  // fp8 elements = bytes = one 128B swizzle row
constexpr int MMA_K = 32;
constexpr int NUM_THREADS = 384;
constexpr int NUM_CONSUMERS = 2;
constexpr int NUM_EPI_WARPS = 4 * NUM_CONSUMERS;
constexpr int EPI_BOX_ROWS = 16;
constexpr int SF_BLOCK_BYTES = 512;  // 128 rows x 4 K-groups of 32 elements

struct Params {
  int M, N, K;           // GROUPED_M: M = padded row capacity.  GROUPED_K: M, N = per-expert output dims, K unused
  const float* scale_a;  // ROWCOL: [M] or nullptr (=1); GROUPED_K: [E, M]; BLOCKWISE: [ceil(K/128), round_up(M, 128)]
  const float* scale_b;  // ROWCOL: [N] or nullptr (=1); grouped: [E, N]; BLOCKWISE: [ceil(K/128), round_up(N, 128)]
  float scale_scalar;    // ROWCOL: extra scalar factor
  const uint8_t* sfa;    // MX: [ceil(M/128), K/128, 512] UE8M0 blocks, byte (r%32)*16 + (r/32)*4 + kgroup
  const uint8_t* sfb;    // MX: [ceil(N/128), K/128, 512]
  // grouped modes (fields read by gemm::get_tile)
  int num_groups;
  const int* tile_group;     // GROUPED_M: [M/128] expert per m-tile (-1 => unused tile, never written)
  const int* group_offsets;  // GROUPED_K: [E+1] row offsets, multiples of BLOCK_K
};

template <int BLOCK_N, int SCALING>
struct Cfg {
  static constexpr bool IS_MX = (SCALING == MX);
  static constexpr bool IS_BLOCKWISE = (SCALING == BLOCKWISE);
  static_assert(BLOCK_N == 128, "128-wide tiles: wider fp32 accumulators (and MX's second, partial one) spill");
  static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K;
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K;
  static constexpr int SFB_BLOCKS = (BLOCK_N + 127) / 128;
  // BLOCKWISE: the k-block's fp32 scales of the tile's 128 rows of A and BLOCK_N rows of B
  static constexpr int SFA_STAGE_BYTES = IS_MX ? SF_BLOCK_BYTES : IS_BLOCKWISE ? BLOCK_M * 4 : 0;
  static constexpr int SFB_STAGE_BYTES = IS_MX ? SFB_BLOCKS * SF_BLOCK_BYTES : IS_BLOCKWISE ? BLOCK_N * 4 : 0;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES + SFA_STAGE_BYTES + SFB_STAGE_BYTES;
  static constexpr int EPI_BUFS = 2;
  static constexpr int EPI_STAGING_BYTES = NUM_EPI_WARPS * EPI_BUFS * EPI_BOX_ROWS * 128;
  static constexpr int SMEM_BUDGET = 227 * 1024 - 2048 - 256 - EPI_STAGING_BYTES;
  static constexpr int STAGES_RAW = SMEM_BUDGET / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static_assert(STAGES >= 3, "need at least 3 operand stages");
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_STAGING_BYTES + 2048 /*two alignments*/ + 256 /*barriers*/;
};

__device__ __forceinline__ void tile_coord(int tile, int m_tiles, int n_tiles, int& m_blk, int& n_blk) {
  constexpr int GROUP_M = 8;  // L2-friendly rasterisation (same as the bf16 kernel)
  const int group_span = GROUP_M * n_tiles;
  const int gid = tile / group_span;
  const int first_m = gid * GROUP_M;
  const int gm = min(m_tiles - first_m, GROUP_M);
  const int r = tile - gid * group_span;
  m_blk = first_m + (r % gm);
  n_blk = r / gm;
}

__device__ __forceinline__ float ue8m0(uint8_t e) { return __uint_as_float(static_cast<uint32_t>(e) << 23); }

// One CTA's work in the grouped modes (ROWCOL scaling, BLOCK_N = 128): the dense kernel's producer / consumer structure
// with the bf16 kernel's tile walk (gemm::get_tile), per-expert scales, promoted accumulation and the store /
// reduce-add epilogues.  scale_a and scale_b are required; scale_scalar is not applied.
template <int BLOCK_N, int MODE, int EPI>
__device__ __forceinline__ void grouped_tiles(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_d,
                                              const Params& p) {
  using C = Cfg<BLOCK_N, ROWCOL>;
  static_assert(MODE == gemm::GROUPED_M || MODE == gemm::GROUPED_K, "grouped modes only");
  static_assert(EPI == gemm::EPI_BF16 || EPI == gemm::EPI_BF16_ACC || (MODE == gemm::GROUPED_K && (EPI == gemm::EPI_F32 || EPI == gemm::EPI_F32_ACC)),
                "GROUPED_M: bf16 store / accumulate; GROUPED_K: fp32 / bf16 store / accumulate");
  constexpr bool OUT_BF16 = (EPI == gemm::EPI_BF16 || EPI == gemm::EPI_BF16_ACC);
  constexpr bool REDUCE = (EPI == gemm::EPI_F32_ACC || EPI == gemm::EPI_BF16_ACC);
  constexpr int CHUNK_COLS = OUT_BF16 ? 64 : 32;  // one 128-byte staging row
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + STAGES * C::A_STAGE_BYTES;
  uint8_t* smem_epi = smem_b + STAGES * C::B_STAGE_BYTES;  // 1024-aligned: both stage sizes are multiples of 1 KiB
  static_assert((C::A_STAGE_BYTES % 1024) == 0 && (C::B_STAGE_BYTES % 1024) == 0, "operand stages keep the 1024-byte swizzle alignment");
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + C::EPI_STAGING_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int total_tiles = gemm::num_tiles<MODE, BLOCK_N, BLOCK_M>(p);

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_d);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================= TMA producer =================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const gemm::TileCoord t = gemm::get_tile<MODE, BLOCK_N, BLOCK_M, BLOCK_K>(p, tile);
        if (!t.valid) continue;  // GROUPED_M: an m-tile past the last expert's segment
        const int m_idx = t.m_blk * BLOCK_M, n_idx = t.n_blk * BLOCK_N;
        for (int kb = 0; kb < t.k_blocks; ++kb) {
          mbar_wait_wg(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          const int k_idx = t.k_begin + kb * BLOCK_K;  // GROUPED_K: the expert's rows start at k_begin
          tma_load_2d(smem_a + stage * C::A_STAGE_BYTES, &tmap_a, &full_bar[stage], k_idx, m_idx);
          if constexpr (MODE == gemm::GROUPED_M)  // B: [E, N, K]
            tma_load_3d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], k_idx, n_idx, t.group);
          else
            tma_load_2d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], k_idx, n_idx);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers: 64 rows each =================
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int lane = lane_id();
    const int cq = (lane & 3) * 2;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t epi_chunk = 0;
    float acc[BLOCK_N / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const gemm::TileCoord t = gemm::get_tile<MODE, BLOCK_N, BLOCK_M, BLOCK_K>(p, tile);
      if (!t.valid) continue;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < t.k_blocks; ++kb) {
        mbar_wait_wg(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem_a + stage * C::A_STAGE_BYTES) + cw * (64 * 128);
        const uint32_t b_addr = smem_u32(smem_b + stage * C::B_STAGE_BYTES);
        // promoted accumulation: the k-block's four MMAs into a fresh accumulator, then one fp32 add per element
        float part[BLOCK_N / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          wgmma_e4m3_ss<BLOCK_N>(part, make_wgmma_desc(a_addr + k * MMA_K, 16, 1024), make_wgmma_desc(b_addr + k * MMA_K, 16, 1024),
                                 k > 0 ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(part);
        if (wq == 0 && lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] += part[i];
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }

      const int rbase = t.m_blk * BLOCK_M + cw * 64 + wq * 16;
      const int col0 = t.n_blk * BLOCK_N;
      // per-expert scale rows: GROUPED_K scale_a [E, M], scale_b [E, N]
      const float* scale_a = p.scale_a + (MODE == gemm::GROUPED_K ? static_cast<long long>(t.group) * p.M : 0);
      const float* scale_b = p.scale_b + static_cast<long long>(t.group) * p.N;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rbase + (lane >> 2) + 8 * h;
        const float row_scale = row < p.M ? scale_a[row] : 0.f;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = col0 + 8 * j + cq + e;
            const float cs = col < p.N ? scale_b[col] : 0.f;
            acc[4 * j + 2 * h + e] = acc[4 * j + 2 * h + e] * row_scale * cs;  // one scale at a time: see the header
          }
        }
      }
      if (REDUCE && t.k_blocks == 0) continue;  // an expert without rows (GROUPED_K) stores zeros but adds nothing
#pragma unroll
      for (int c = 0; c < BLOCK_N / CHUNK_COLS; ++c) {
        const int cbase = col0 + c * CHUNK_COLS;
        if (cbase >= p.N) break;  // warp-uniform
        uint8_t* stage_buf = smem_epi + ((cw * 4 + wq) * C::EPI_BUFS + (epi_chunk % C::EPI_BUFS)) * (EPI_BOX_ROWS * 128);
        ++epi_chunk;
        if (lane == 0) tma_store_wait_read<C::EPI_BUFS - 1>();
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (lane >> 2) + 8 * h;
          if constexpr (OUT_BF16) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = c * 8 + jj;
              *reinterpret_cast<uint32_t*>(stage_buf + r * 128 + ((jj ^ (r & 7)) << 4) + (lane & 3) * 4) =
                  pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          } else {
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = c * 4 + jj;
              const int q = 2 * jj + ((lane & 3) >> 1);
              *reinterpret_cast<float2*>(stage_buf + r * 128 + ((q ^ (r & 7)) << 4) + (lane & 1) * 8) =
                  make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          const int g0 = (MODE == gemm::GROUPED_K) ? t.group : 0;  // D is [E, M, N]
          if constexpr (REDUCE) tma_reduce_add_3d(&tmap_d, stage_buf, cbase, rbase, g0);
          else tma_store_3d(&tmap_d, stage_buf, cbase, rbase, g0);
          tma_store_commit();
        }
      }
    }
    if (lane == 0) tma_store_wait<0>();
  }
}

// The tile at index `tile` of a BLOCKWISE walk: the DENSE rasterisation (tile_coord, every tile valid, all k_blocks) or
// the grouped modes' gemm::get_tile (GROUPED_M: -1 tiles invalid; GROUPED_K: the expert's rows from k_begin).
template <int MODE, int BLOCK_N>
__device__ __forceinline__ gemm::TileCoord blockwise_tile(const Params& p, int tile, int m_tiles, int n_tiles, int k_blocks) {
  if constexpr (MODE == gemm::DENSE) {
    gemm::TileCoord t;
    tile_coord(tile, m_tiles, n_tiles, t.m_blk, t.n_blk);
    t.group = 0;
    t.k_begin = 0;
    t.k_blocks = k_blocks;
    t.valid = true;
    return t;
  } else {
    return gemm::get_tile<MODE, BLOCK_N, BLOCK_M, BLOCK_K>(p, tile);
  }
}

// One CTA's work in the BLOCKWISE scaling (BLOCK_N = 128): every stage carries the k-block's A / B tiles and their
// 128 + 128 fp32 scales; the consumers compute the k-block's four MMAs into a fresh accumulator and add it with
// acc = fma(part, sa[row] * sb[col], acc).  Tails: TMA zero-fills a partial last k-block and the rows / columns of A / B
// past M / N (their scales are never applied to a stored element), and the TMA store clips D to [M, N].
// The scales of k-block kb (all k-block-major, row pitch round_up(rows, 128)):
//   DENSE      scale_a [ceil(K/128), M], scale_b [ceil(K/128), N]: row kb of both
//   GROUPED_M  scale_a [ceil(K/128), M] (M = capacity): row kb; scale_b [E, ceil(K/128), N]: row kb of expert e's plane
//   GROUPED_K  scale_a [R/128, M], scale_b [R/128, N] (128-token groups): row group_offsets[e] / 128 + kb of both
// The consumers raised their register budget (acc + part = 128 fp32 registers), so they wait with mbar_wait_flag and a
// timed-out wait traps after their region (see mbar_wait_flag).
template <int BLOCK_N, int MODE, int EPI>
__device__ __forceinline__ void blockwise_tiles(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_d,
                                                const Params& p) {
  using C = Cfg<BLOCK_N, BLOCKWISE>;
  static_assert(MODE == gemm::DENSE ? (EPI == gemm::EPI_BF16 || EPI == gemm::EPI_F32)
                                    : (EPI == gemm::EPI_BF16 || EPI == gemm::EPI_BF16_ACC ||
                                       (MODE == gemm::GROUPED_K && (EPI == gemm::EPI_F32 || EPI == gemm::EPI_F32_ACC))),
                "BLOCKWISE DENSE: bf16 or fp32 store; GROUPED_M: bf16 store / accumulate; GROUPED_K: fp32 / bf16 store / accumulate");
  constexpr bool OUT_BF16 = (EPI == gemm::EPI_BF16 || EPI == gemm::EPI_BF16_ACC);
  constexpr bool REDUCE = (EPI == gemm::EPI_F32_ACC || EPI == gemm::EPI_BF16_ACC);
  constexpr int CHUNK_COLS = OUT_BF16 ? 64 : 32;  // one 128-byte staging row
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + STAGES * C::A_STAGE_BYTES;
  float* smem_sa = reinterpret_cast<float*>(smem_b + STAGES * C::B_STAGE_BYTES);
  float* smem_sb = smem_sa + STAGES * BLOCK_M;
  uint8_t* smem_epi = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_sb + STAGES * BLOCK_N) + 1023) & ~uintptr_t(1023));
  static_assert((C::A_STAGE_BYTES % 1024) == 0 && (C::B_STAGE_BYTES % 1024) == 0, "operand stages keep the 1024-byte swizzle alignment");
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + C::EPI_STAGING_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M, n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int total_tiles = m_tiles * n_tiles * (MODE == gemm::GROUPED_K ? p.num_groups : 1);
  const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;  // DENSE / GROUPED_M
  // k-block-major scales: rows padded to whole tiles, so a tile's scales are one aligned 512-byte copy inside the tensor
  const long long lds_a = static_cast<long long>(m_tiles) * BLOCK_M, lds_b = static_cast<long long>(n_tiles) * BLOCK_N;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_d);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_EPI_WARPS);  // every consumer warp releases the stage once it has read its scales
    }
    fence_barrier_init();
  }
  __syncthreads();

  bool stuck = false;  // a consumer's mbarrier wait timed out (see mbar_wait_flag)

  if (warp < 4) {
    // ================= TMA producer =================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        if constexpr (MODE == gemm::DENSE) {
          int m_blk, n_blk;
          tile_coord(tile, m_tiles, n_tiles, m_blk, n_blk);
          const int m_idx = m_blk * BLOCK_M, n_idx = n_blk * BLOCK_N;
          for (int kb = 0; kb < k_blocks; ++kb) {
            mbar_wait_wg(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
            tma_load_2d(smem_a + stage * C::A_STAGE_BYTES, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_idx);
            tma_load_2d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_idx);
            bulk_load_1d(smem_sa + stage * BLOCK_M, p.scale_a + kb * lds_a + m_idx, C::SFA_STAGE_BYTES, &full_bar[stage]);
            bulk_load_1d(smem_sb + stage * BLOCK_N, p.scale_b + kb * lds_b + n_idx, C::SFB_STAGE_BYTES, &full_bar[stage]);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        } else {
          const gemm::TileCoord t = gemm::get_tile<MODE, BLOCK_N, BLOCK_M, BLOCK_K>(p, tile);
          if (!t.valid) continue;  // GROUPED_M: an m-tile past the last expert's segment
          const int m_idx = t.m_blk * BLOCK_M, n_idx = t.n_blk * BLOCK_N;
          // the scale rows of k-block kb (see above): GROUPED_M scale_b is one [ceil(K/128), N] plane per expert; GROUPED_K
          // reads the 128-token groups from the expert's first row
          const long long sa_row0 = MODE == gemm::GROUPED_K ? t.k_begin / BLOCK_K : 0;
          const long long sb_row0 = MODE == gemm::GROUPED_K ? t.k_begin / BLOCK_K : static_cast<long long>(t.group) * t.k_blocks;
          for (int kb = 0; kb < t.k_blocks; ++kb) {
            mbar_wait_wg(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
            const int k_idx = t.k_begin + kb * BLOCK_K;  // GROUPED_K: the expert's rows start at k_begin
            tma_load_2d(smem_a + stage * C::A_STAGE_BYTES, &tmap_a, &full_bar[stage], k_idx, m_idx);
            if constexpr (MODE == gemm::GROUPED_M)  // B: [E, N, K]
              tma_load_3d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], k_idx, n_idx, t.group);
            else
              tma_load_2d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], k_idx, n_idx);
            bulk_load_1d(smem_sa + stage * BLOCK_M, p.scale_a + (sa_row0 + kb) * lds_a + m_idx, C::SFA_STAGE_BYTES, &full_bar[stage]);
            bulk_load_1d(smem_sb + stage * BLOCK_N, p.scale_b + (sb_row0 + kb) * lds_b + n_idx, C::SFB_STAGE_BYTES, &full_bar[stage]);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ================= consumers: 64 rows each =================
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int lane = lane_id();
    const int cq = (lane & 3) * 2;
    const int r_loc = cw * 64 + wq * 16 + (lane >> 2);  // tile-local rows r_loc and r_loc + 8 of this thread
    int stage = 0;
    uint32_t phase = 0;
    uint32_t epi_chunk = 0;
    float acc[BLOCK_N / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const gemm::TileCoord t = blockwise_tile<MODE, BLOCK_N>(p, tile, m_tiles, n_tiles, k_blocks);
      if (!t.valid) continue;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < t.k_blocks; ++kb) {
        mbar_wait_flag(&full_bar[stage], phase, stuck);
        const uint32_t a_addr = smem_u32(smem_a + stage * C::A_STAGE_BYTES) + cw * (64 * 128);
        const uint32_t b_addr = smem_u32(smem_b + stage * C::B_STAGE_BYTES);
        float part[BLOCK_N / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          wgmma_e4m3_ss<BLOCK_N>(part, make_wgmma_desc(a_addr + k * MMA_K, 16, 1024), make_wgmma_desc(b_addr + k * MMA_K, 16, 1024),
                                 k > 0 ? 1 : 0);
        wgmma_commit();
        // the scales of this thread's two rows and 32 columns, read while the MMAs run
        const float* sa = smem_sa + stage * BLOCK_M;
        const float* sb = smem_sb + stage * BLOCK_N;
        const float sa0 = sa[r_loc], sa1 = sa[r_loc + 8];
        float2 sbj[BLOCK_N / 8];
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) sbj[j] = *reinterpret_cast<const float2*>(sb + 8 * j + cq);
        wgmma_wait<0>();
        wgmma_fence_regs(part);
        __syncwarp();  // the warp's MMAs and scale reads are done: the stage can be refilled
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          acc[4 * j] = fmaf(part[4 * j] * sa0, sbj[j].x, acc[4 * j]);
          acc[4 * j + 1] = fmaf(part[4 * j + 1] * sa0, sbj[j].y, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(part[4 * j + 2] * sa1, sbj[j].x, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(part[4 * j + 3] * sa1, sbj[j].y, acc[4 * j + 3]);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (REDUCE && t.k_blocks == 0) continue;  // an expert without rows (GROUPED_K) stores zeros but adds nothing

      const int rbase = t.m_blk * BLOCK_M + cw * 64 + wq * 16;
      const int col0 = t.n_blk * BLOCK_N;
#pragma unroll
      for (int c = 0; c < BLOCK_N / CHUNK_COLS; ++c) {
        const int cbase = col0 + c * CHUNK_COLS;
        if (cbase >= p.N) break;  // warp-uniform
        uint8_t* stage_buf = smem_epi + ((cw * 4 + wq) * C::EPI_BUFS + (epi_chunk % C::EPI_BUFS)) * (EPI_BOX_ROWS * 128);
        ++epi_chunk;
        if (lane == 0) tma_store_wait_read<C::EPI_BUFS - 1>();
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (lane >> 2) + 8 * h;
          if constexpr (OUT_BF16) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = c * 8 + jj;
              *reinterpret_cast<uint32_t*>(stage_buf + r * 128 + ((jj ^ (r & 7)) << 4) + (lane & 3) * 4) =
                  pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          } else {
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = c * 4 + jj;
              const int q = 2 * jj + ((lane & 3) >> 1);
              *reinterpret_cast<float2*>(stage_buf + r * 128 + ((q ^ (r & 7)) << 4) + (lane & 1) * 8) =
                  make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          const int g0 = (MODE == gemm::GROUPED_K) ? t.group : 0;  // GROUPED_K: D is [E, M, N]
          if constexpr (REDUCE) tma_reduce_add_3d(&tmap_d, stage_buf, cbase, rbase, g0);
          else tma_store_3d(&tmap_d, stage_buf, cbase, rbase, g0);
          tma_store_commit();
        }
      }
    }
    if (lane == 0) tma_store_wait<0>();
  }
  // A stuck consumer fell through its later waits (it still released every stage and stored its tiles, so the producer
  // does not wait on it forever) and turns the hang into a trap here, outside its raised register budget.
  if (stuck) __trap();
}

template <int BLOCK_N, int SCALING, int MODE = gemm::DENSE, int EPI = gemm::EPI_BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const __grid_constant__ CUtensorMap tmap_d, const Params p) {
  static_assert(MODE == gemm::DENSE || SCALING != MX, "the grouped modes use row / column or blockwise scaling");
  static_assert(MODE != gemm::DENSE || EPI == gemm::EPI_BF16 || (SCALING == BLOCKWISE && EPI == gemm::EPI_F32),
                "the dense kernel stores bf16 (BLOCKWISE: or fp32)");
  if constexpr (SCALING == BLOCKWISE) {
    blockwise_tiles<BLOCK_N, MODE, EPI>(tmap_a, tmap_b, tmap_d, p);
  } else if constexpr (MODE != gemm::DENSE) {
    grouped_tiles<BLOCK_N, MODE, EPI>(tmap_a, tmap_b, tmap_d, p);
  } else {
    using C = Cfg<BLOCK_N, SCALING>;
    constexpr int STAGES = C::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem_a + STAGES * C::A_STAGE_BYTES;
    uint8_t* smem_sfa = smem_b + STAGES * C::B_STAGE_BYTES;
    uint8_t* smem_sfb = smem_sfa + STAGES * C::SFA_STAGE_BYTES;
    // the swizzled epilogue staging boxes must start on a 1024-byte boundary (the scale-factor regions are 512-byte granular)
    uint8_t* smem_epi = reinterpret_cast<uint8_t*>(
        (reinterpret_cast<uintptr_t>(smem_sfb + STAGES * C::SFB_STAGE_BYTES) + 1023) & ~uintptr_t(1023));
    static_assert((C::A_STAGE_BYTES % 1024) == 0 && (C::B_STAGE_BYTES % 1024) == 0, "operand stages keep the 1024-byte swizzle alignment");
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + C::EPI_STAGING_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + STAGES;

    const int warp = threadIdx.x >> 5;
    const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M, n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int total_tiles = m_tiles * n_tiles;
    const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
    const int sf_k_blocks = k_blocks;

    if (warp == 0 && elect_one()) {
      tma_prefetch_desc(&tmap_a);
      tma_prefetch_desc(&tmap_b);
      tma_prefetch_desc(&tmap_d);
      for (int i = 0; i < STAGES; ++i) {
        mbar_init(&full_bar[i], 1);
        mbar_init(&empty_bar[i], NUM_CONSUMERS);
      }
      fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
      // ================= TMA producer =================
      setmaxnreg_dec<40>();
      if (warp == 0 && elect_one()) {
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          int m_blk, n_blk;
          tile_coord(tile, m_tiles, n_tiles, m_blk, n_blk);
          const int m_idx = m_blk * BLOCK_M, n_idx = n_blk * BLOCK_N;
          for (int kb = 0; kb < k_blocks; ++kb) {
            mbar_wait_wg(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
            tma_load_2d(smem_a + stage * C::A_STAGE_BYTES, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_idx);
            tma_load_2d(smem_b + stage * C::B_STAGE_BYTES, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_idx);
            if constexpr (C::IS_MX) {
              bulk_load_1d(smem_sfa + stage * C::SFA_STAGE_BYTES,
                           p.sfa + (static_cast<long long>(m_blk) * sf_k_blocks + kb) * SF_BLOCK_BYTES, SF_BLOCK_BYTES, &full_bar[stage]);
#pragma unroll
              for (int j = 0; j < C::SFB_BLOCKS; ++j)
                bulk_load_1d(smem_sfb + stage * C::SFB_STAGE_BYTES + j * SF_BLOCK_BYTES,
                             p.sfb + (static_cast<long long>(n_blk * C::SFB_BLOCKS + j) * sf_k_blocks + kb) * SF_BLOCK_BYTES,
                             SF_BLOCK_BYTES, &full_bar[stage]);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else {
      // ================= consumers: 64 rows each =================
      setmaxnreg_inc<232>();
      const int cw = (warp >> 2) - 1;
      const int wq = warp & 3;
      const int lane = lane_id();
      const int cq = (lane & 3) * 2;
      const int r_loc = cw * 64 + wq * 16 + (lane >> 2);  // tile-local rows r_loc and r_loc + 8 of this thread
      int stage = 0;
      uint32_t phase = 0;
      uint32_t epi_chunk = 0;
      float acc[BLOCK_N / 2];
      auto release = [&](int s) {
        if (wq == 0 && lane == 0) mbar_arrive(&empty_bar[s]);
      };
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coord(tile, m_tiles, n_tiles, m_blk, n_blk);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
        wgmma_fence_regs(acc);
        int prev = -1;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait_wg(&full_bar[stage], phase);
          const uint32_t a_addr = smem_u32(smem_a + stage * C::A_STAGE_BYTES) + cw * (64 * 128);
          const uint32_t b_addr = smem_u32(smem_b + stage * C::B_STAGE_BYTES);
          if constexpr (C::IS_MX) {
            const uint8_t* sfa = smem_sfa + stage * C::SFA_STAGE_BYTES;
            const uint8_t* sfb = smem_sfb + stage * C::SFB_STAGE_BYTES;
#pragma unroll
            for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
              float part[BLOCK_N / 2];
              wgmma_fence();
              wgmma_e4m3_ss<BLOCK_N>(part, make_wgmma_desc(a_addr + k * MMA_K, 16, 1024), make_wgmma_desc(b_addr + k * MMA_K, 16, 1024), 0);
              wgmma_commit();
              wgmma_wait<0>();
              wgmma_fence_regs(part);
              float sa[2];
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = r_loc + 8 * h;
                sa[h] = ue8m0(sfa[(r % 32) * 16 + (r / 32) * 4 + k]);
              }
#pragma unroll
              for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int n = 8 * j + cq + e;
                  const float sb = ue8m0(sfb[(n / 128) * SF_BLOCK_BYTES + (n % 32) * 16 + ((n % 128) / 32) * 4 + k]);
                  acc[4 * j + e] = fmaf(part[4 * j + e] * sa[0], sb, acc[4 * j + e]);
                  acc[4 * j + 2 + e] = fmaf(part[4 * j + 2 + e] * sa[1], sb, acc[4 * j + 2 + e]);
                }
              }
            }
            release(stage);
          } else {
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / MMA_K; ++k)
              wgmma_e4m3_ss<BLOCK_N>(acc, make_wgmma_desc(a_addr + k * MMA_K, 16, 1024), make_wgmma_desc(b_addr + k * MMA_K, 16, 1024), 1);
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0) release(prev);
            prev = stage;
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if constexpr (!C::IS_MX) {
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
          if (prev >= 0) release(prev);
        }

        const int rbase = m_blk * BLOCK_M + cw * 64 + wq * 16;
        const int col0 = n_blk * BLOCK_N;
        if constexpr (!C::IS_MX) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rbase + (lane >> 2) + 8 * h;
            const float row_scale = (p.scale_a != nullptr && row < p.M) ? p.scale_a[row] : 1.f;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int col = col0 + 8 * j + cq + e;
                const float cs = (p.scale_b != nullptr && col < p.N) ? p.scale_b[col] : 1.f;
                acc[4 * j + 2 * h + e] = acc[4 * j + 2 * h + e] * row_scale * cs * p.scale_scalar;
              }
            }
          }
        }
#pragma unroll
        for (int c = 0; c < BLOCK_N / 64; ++c) {
          const int cbase = col0 + c * 64;
          if (cbase >= p.N) break;  // warp-uniform
          uint8_t* stage_buf = smem_epi + ((cw * 4 + wq) * C::EPI_BUFS + (epi_chunk % C::EPI_BUFS)) * (EPI_BOX_ROWS * 128);
          ++epi_chunk;
          if (lane == 0) tma_store_wait_read<C::EPI_BUFS - 1>();
          __syncwarp();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = (lane >> 2) + 8 * h;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = c * 8 + jj;
              *reinterpret_cast<uint32_t*>(stage_buf + r * 128 + ((jj ^ (r & 7)) << 4) + (lane & 3) * 4) =
                  pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          }
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            tma_store_3d(&tmap_d, stage_buf, cbase, rbase, 0);
            tma_store_commit();
          }
        }
      }
      if (lane == 0) tma_store_wait<0>();
    }
  }
}

}  // namespace fp8
}  // namespace d9d
