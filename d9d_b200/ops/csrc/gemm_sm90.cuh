// d9d_b200 — persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = A[M,K] · B[N,K]^T      bf16 operands, fp32 accumulation in registers.
//
// * operands are staged by TMA (128B swizzle) into a multi-stage smem ring,
// * warpgroup 0 is the TMA producer; warpgroups 1 and 2 each own 64 rows of the 128 x BLOCK_N tile and issue
//   wgmma.mma_async (m64 x BLOCK_N x k16) straight from shared memory, keeping one k-block in flight while the stage of
//   the previous one is released,
// * either operand may be K-major or MN-major (needed for dgrad / wgrad without transposes),
// * three problem shapes share the mainloop:
//     DENSE      plain GEMM
//     GROUPED_M  rows of A/D are grouped by expert (128-row aligned segments, device-side tile->expert table),
//                B is [E, ...]  -> MoE forward / dgrad without any host sync
//     GROUPED_K  the reduction dim is grouped (per-expert weight gradients), D is [E, M, N]
// * epilogues: bf16 store, fp32 store, fp32/bf16 accumulate, and the fused linear-cross-entropy epilogues.
//   Output tiles leave the SM through TMA: registers -> 128B-swizzled smem staging (16 rows x 128 B per warp) ->
//   cp.async.bulk.tensor store, or cp.reduce.async.bulk.tensor (.add) for the accumulate epilogues, so `D += acc` costs
//   no global loads in the SM (the add happens in L2) and partial tiles are clipped by the tensor map.
// * split-K (DENSE, accumulate epilogues): several CTAs reduce-add K-slices of one output tile; used when a wgrad
//   has few output tiles but a long reduction dim.
#pragma once

#include <type_traits>

#include "common.cuh"
#include "d9d_ops.h"  // gemm::Mode, gemm::Epi, gemm::Comm

namespace d9d {
namespace gemm {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int MMA_K = 16;
constexpr int NUM_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue (64 rows each)
constexpr int NUM_CONSUMERS = 2;
constexpr int NUM_EPI_WARPS = 4 * NUM_CONSUMERS;
constexpr int EPI_BOX_ROWS = 16;  // output staging box: one warp's 16 accumulator rows x 128 bytes
// per-thread register budgets (setmaxnreg; 2 x 128 x CONSUMER_REGS + 128 x PRODUCER_REGS <= 64 K).  A consumer holds a
// 64 x BLOCK_N fp32 accumulator, 128 registers at BLOCK_N = 256, and the fused-CE epilogues work on all of it in place.
// The producer's tile walk and peer tensor-map selection spill at 24 and 32 (the fused-communication GEMMs), so 240 / 24
// is not spill-free; at 232 / 40 no instance spills.  The consumers only get this budget because their waits cannot trap
// (see mbar_wait_flag): under a reachable trap ptxas holds them to the launch bound's 168.
constexpr int CONSUMER_REGS = 232;
constexpr int PRODUCER_REGS = 40;

constexpr int MAX_PEERS = 8;
struct PeerMaps { CUtensorMap m[MAX_PEERS]; };
struct NoPeerMaps {};
template <int COMM> struct PeerArg { using type = PeerMaps; };
template <> struct PeerArg<COMM_NONE> { using type = NoPeerMaps; };
template <> struct PeerArg<COMM_WAIT_A> { using type = NoPeerMaps; };

struct Params {
  int M, N, K;            // DENSE: problem dims. GROUPED_M: M = padded row capacity. GROUPED_K: M,N = per-expert out dims
  int num_groups;         // experts (1 for dense)
  int k_splits;           // DENSE + accumulate epilogue: K is cut into this many slices (1 => off)
  int tma_epilogue;       // 1: output through the tmap_d TMA store/reduce path, 0: direct global stores
  int comm_world;         // COMM_*: number of peers
  int comm_block_rows;    // COMM_*: rows per (rank, block) of the sharded dim
  int comm_rank;          // COMM_WAIT_A: this rank (its shard needs no wait)
  int comm_m_rot;         // COMM_WAIT_A: m-blocks are visited starting at this block (the local shard first)
  const int* comm_flags;  // COMM_WAIT_A: [comm_world] arrival flags of the shards (non-zero = landed)
  void* D;                // output
  long long ldd;          // leading dim of D (elements)
  long long d_group_stride;  // GROUPED_K: elements between per-expert outputs
  const int* tile_group;  // GROUPED_M: [M/128] expert id per m-tile (-1 => unused tile)
  const int* group_offsets;  // GROUPED_K: [E+1] row offsets (multiples of BLOCK_K) into the grouped K dimension
  // fused CE
  const long long* ce_target;  // [M] int64 targets (ignore_index allowed)
  const float* ce_lse;         // [M]           (DLOGITS)
  const float* ce_grad;        // [M]           (DLOGITS) upstream grad per row
  float* ce_part_max;          // [n_tiles, M]  (LSE)
  float* ce_part_sum;          // [n_tiles, M]  (LSE)
  float* ce_tgt_logit;         // [M]           (LSE) written by the tile that owns the target column
  long long ce_ignore_index;
  float ce_softcap;            // logits -> softcap * tanh(logits / softcap) (0 = off)
  const float* ce_bias;        // [N] fp32 added to the logits (or nullptr)
  long long ce_col_offset;     // B is a row slice of the classifier: global class id of its first row
  // regularised CE (appended: the fields above keep their offsets, and Params still ends before the next 64-byte
  // boundary, where the peer tensor maps of the fused-communication GEMMs begin)
  float* ce_part_zsum;         // [n_tiles, M]  (LSE_SUM) sum of the tile's logits
  float ce_z_loss;             // (DLOGITS_REG) zeta
  float ce_smoothing;          // (DLOGITS_REG) eps
  int ce_num_classes;          // (DLOGITS_REG) V: classes over all slices of the classifier
};

// logit transform shared by the fused-CE epilogues: z = softcap(acc + bias); returns z and dz/dacc
__device__ __forceinline__ float ce_transform(float acc, float bias, float cap, float inv_cap, float& dz) {
  float z = acc + bias;
  dz = 1.f;
  if (cap > 0.f) {
    const float th = tanhf(z * inv_cap);
    z = cap * th;
    dz = 1.f - th * th;
  }
  return z;
}

// CTAS = 2: a cluster of two CTAs works on a 256 x BLOCK_N tile: every CTA stages its own 128 rows of A and loads half of
// the B tile, multicast into both CTAs, i.e. half the B traffic from L2 per flop.
template <int BLOCK_N, int CTAS = 1>
struct Cfg {
  static_assert(CTAS == 1 || CTAS == 2, "one CTA or a cluster of two");
  static_assert(CTAS == 1 || BLOCK_N % 128 == 0, "a CTA pair splits B into halves of whole 64-column swizzle atoms");
  static constexpr int TILE_M = BLOCK_M * CTAS;
  static constexpr int B_ROWS = BLOCK_N / CTAS;  // rows of B loaded by one CTA
  static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;  // the whole B tile (pair: both halves land in every CTA)
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int EPI_BUFS = 2;
  static constexpr int EPI_STAGING_BYTES = NUM_EPI_WARPS * EPI_BUFS * EPI_BOX_ROWS * 128;
  static constexpr int SMEM_BUDGET = 227 * 1024 - 1024 - 256 - EPI_STAGING_BYTES;
  static constexpr int STAGES_RAW = SMEM_BUDGET / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static_assert(STAGES >= 3, "need at least 3 operand stages");
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_STAGING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

struct TileCoord {
  int m_blk, n_blk, group;
  int k_begin, k_blocks;  // k offset (elements) and number of BLOCK_K chunks
  bool valid;
};

// The tile walk is shared with the fp8 kernel (gemm_fp8_sm90.cuh): BK is the depth of a k-block in elements, and the
// parameter block P needs M, N, K, num_groups, tile_group and group_offsets; the DENSE-only fields (k_splits,
// comm_m_rot) are read in DENSE instances only.
template <int MODE, int BLOCK_N, int TILE_M = BLOCK_M, typename P = Params>
__device__ __forceinline__ int num_tiles(const P& p) {
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int m_tiles = (p.M + TILE_M - 1) / TILE_M;
  if constexpr (MODE == GROUPED_K) return p.num_groups * m_tiles * n_tiles;
  if constexpr (MODE == DENSE) return m_tiles * n_tiles * p.k_splits;
  return m_tiles * n_tiles;
}

template <int MODE, int BLOCK_N, int TILE_M = BLOCK_M, int BK = BLOCK_K, typename P = Params>
__device__ __forceinline__ TileCoord get_tile(const P& p, int tile) {
  TileCoord t;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int m_tiles = (p.M + TILE_M - 1) / TILE_M;
  t.valid = true;
  if constexpr (MODE == GROUPED_K) {
    const int per_group = m_tiles * n_tiles;
    t.group = tile / per_group;
    const int r = tile - t.group * per_group;
    t.m_blk = r / n_tiles;
    t.n_blk = r - t.m_blk * n_tiles;
    const int k0 = p.group_offsets[t.group], k1 = p.group_offsets[t.group + 1];
    t.k_begin = k0;
    t.k_blocks = (k1 - k0 + BK - 1) / BK;
    return t;
  }
  int k_split = 0;
  if constexpr (MODE == DENSE) {
    if (p.k_splits > 1) {  // tile = split * (m_tiles * n_tiles) + mn: one K-slice per wave
      k_split = tile / (m_tiles * n_tiles);
      tile -= k_split * (m_tiles * n_tiles);
    }
  }
  // L2-friendly rasterisation: walk GROUP_M m-blocks for each n-block before moving on.
  constexpr int GROUP_M = 8;
  const int group_span = GROUP_M * n_tiles;
  const int gid = tile / group_span;
  const int first_m = gid * GROUP_M;
  const int gm = min(m_tiles - first_m, GROUP_M);
  const int r = tile - gid * group_span;
  t.m_blk = first_m + (r % gm);
  t.n_blk = r / gm;
  if constexpr (MODE == DENSE) {
    if (p.comm_m_rot != 0) t.m_blk = (t.m_blk + p.comm_m_rot) % m_tiles;
  }
  t.k_begin = 0;
  t.k_blocks = (p.K + BK - 1) / BK;
  if constexpr (MODE == DENSE) {
    if (p.k_splits > 1) {
      const int per_split = (t.k_blocks + p.k_splits - 1) / p.k_splits;
      const int first = k_split * per_split;
      t.k_begin = first * BK;
      t.k_blocks = max(0, min(per_split, t.k_blocks - first));
      t.valid = t.k_blocks > 0;  // an empty slice has nothing to add
    }
  }
  t.group = 0;
  if constexpr (MODE == GROUPED_M) {
    t.group = p.tile_group[t.m_blk];
    t.valid = t.group >= 0;
  }
  return t;
}

__device__ __forceinline__ void comm_locate(const Params& p, int idx, int& owner, int& local) {
  const int blk = idx / p.comm_block_rows;
  owner = blk % p.comm_world;
  local = (blk / p.comm_world) * p.comm_block_rows + (idx - blk * p.comm_block_rows);
}

template <int MODE, int BLOCK_N, bool A_MN, bool B_MN, int EPI, int COMM = COMM_NONE, int CTAS = 1>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_d, const Params p,
            const __grid_constant__ typename PeerArg<COMM>::type peers) {
  static_assert(COMM == COMM_NONE || MODE == DENSE, "fused communication is implemented for dense GEMMs");
  static_assert((COMM != COMM_AG_A && COMM != COMM_WAIT_A) || !A_MN, "COMM_AG_A / COMM_WAIT_A work on a K-major A");
  static_assert(COMM != COMM_AG_KA || A_MN, "COMM_AG_KA gathers an MN-major A along K");
  static_assert(COMM != COMM_AG_KB || B_MN, "COMM_AG_KB gathers an MN-major B along K");
  static_assert(COMM != COMM_RS_D || EPI == EPI_F32_ACC || EPI == EPI_BF16_ACC, "COMM_RS_D needs a reduce-add epilogue");
  static_assert(CTAS == 1 || (MODE == DENSE && COMM == COMM_NONE), "CTA pairs are implemented for plain dense GEMMs");
  using C = Cfg<BLOCK_N, CTAS>;
  constexpr int STAGES = C::STAGES;
  constexpr int TILE_M = C::TILE_M;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * C::A_STAGE_BYTES;
  uint8_t* smem_epi = smem + STAGES * C::STAGE_BYTES;  // 1024-aligned: STAGE_BYTES is a multiple of 8 KiB
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + C::EPI_STAGING_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int total_tiles = num_tiles<MODE, BLOCK_N, TILE_M>(p);
  // persistent loop: one tile per CTA (pair) at a time
  const int pair_rank = (CTAS == 2) ? static_cast<int>(cluster_ctarank()) : 0;
  const int first_tile = static_cast<int>(blockIdx.x) / CTAS;
  const int tile_stride = static_cast<int>(gridDim.x) / CTAS;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.tma_epilogue) tma_prefetch_desc(&tmap_d);
    if constexpr (COMM != COMM_NONE && COMM != COMM_WAIT_A)
      for (int r = 0; r < p.comm_world; ++r) tma_prefetch_desc(&peers.m[r]);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMERS * CTAS);  // pair: a stage is refilled once the consumers of BOTH CTAs are done
    }
    fence_barrier_init();
  }
  if constexpr (CTAS == 2) cluster_sync_all();  // the peer's barriers are initialised before anything is multicast into it
  else __syncthreads();

  bool stuck = false;  // a consumer's mbarrier wait timed out (see mbar_wait_flag)

  if (warp < 4) {
    // ================= TMA producer (one thread of warpgroup 0) =================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      // grouped modes read the tile's expert / row range from global memory: fetch it one whole tile ahead so that the
      // load latency never sits between two tiles on the critical path
      TileCoord t_next = get_tile<MODE, BLOCK_N, TILE_M>(p, first_tile);
      for (int tile = first_tile; tile < total_tiles; tile += tile_stride) {
        const TileCoord t = t_next;
        if (tile + tile_stride < total_tiles) t_next = get_tile<MODE, BLOCK_N, TILE_M>(p, tile + tile_stride);
        if (!t.valid) continue;
        // pair: this CTA's 128 rows of the 256-row tile and its half of the B tile
        const int m_idx = t.m_blk * TILE_M + pair_rank * BLOCK_M, n_idx = t.n_blk * BLOCK_N + pair_rank * C::B_ROWS;
        if constexpr (COMM == COMM_WAIT_A) {  // the shard holding this m-tile may still be in flight
          int owner, unused;
          comm_locate(p, m_idx, owner, unused);
          if (owner != p.comm_rank) {
            const int* flag = p.comm_flags + owner;
            int landed;
            long long spins = 0;
            do {
              asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(landed) : "l"(flag) : "memory");
              if (!landed) {
                __nanosleep(500);
                if (++spins > 8000000LL) __trap();  // ~4 s: the producer of the flag never ran (would otherwise hang the GPU)
              }
            } while (!landed);
            fence_proxy_async_all();  // the copy's generic-proxy writes are ordered before our async-proxy (TMA) reads
          }
        }
        for (int kb = 0; kb < t.k_blocks; ++kb) {
          mbar_wait_wg(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);  // pair: the peer's multicast half lands here too
          const int k_idx = t.k_begin + kb * BLOCK_K;
          uint8_t* sa = smem_a + stage * C::A_STAGE_BYTES;
          uint8_t* sb = smem_b + stage * C::B_STAGE_BYTES;
          if constexpr (COMM == COMM_AG_A) {  // the m-tile lives in its owner's shard: load it over NVLink
            int owner, m_local;
            comm_locate(p, m_idx, owner, m_local);
            tma_load_3d(sa, &peers.m[owner], &full_bar[stage], k_idx, m_local, 0);
          } else if constexpr (COMM == COMM_AG_KA) {
            int owner, k_local;
            comm_locate(p, k_idx, owner, k_local);
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_3d(sa + j * (BLOCK_K * 128), &peers.m[owner], &full_bar[stage], m_idx + j * 64, k_local, 0);
          } else if (!A_MN) {
            tma_load_3d(sa, &tmap_a, &full_bar[stage], k_idx, m_idx, 0);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_3d(sa + j * (BLOCK_K * 128), &tmap_a, &full_bar[stage], m_idx + j * 64, k_idx, 0);
          }
          const int bg = (MODE == GROUPED_M) ? t.group : 0;
          if constexpr (COMM == COMM_AG_KB) {
            int owner, k_local;
            comm_locate(p, k_idx, owner, k_local);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_3d(sb + j * (BLOCK_K * 128), &peers.m[owner], &full_bar[stage], n_idx + j * 64, k_local, 0);
          } else if (!B_MN) {
            uint8_t* dst = sb + pair_rank * C::B_ROWS * 128;
            if constexpr (CTAS == 2) tma_load_3d_multicast(dst, &tmap_b, &full_bar[stage], 0b11, k_idx, n_idx, bg);
            else tma_load_3d(dst, &tmap_b, &full_bar[stage], k_idx, n_idx, bg);
          } else {
#pragma unroll
            for (int j = 0; j < C::B_ROWS / 64; ++j) {
              uint8_t* dst = sb + (pair_rank * (C::B_ROWS / 64) + j) * (BLOCK_K * 128);
              if constexpr (CTAS == 2) tma_load_3d_multicast(dst, &tmap_b, &full_bar[stage], 0b11, n_idx + j * 64, k_idx, bg);
              else tma_load_3d(dst, &tmap_b, &full_bar[stage], n_idx + j * 64, k_idx, bg);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers: wgmma over 64 rows each, then the epilogue of those rows =================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = (warp >> 2) - 1;  // consumer warpgroup: rows [64 cw, 64 cw + 64) of this CTA's 128
    const int wq = warp & 3;         // warp inside the warpgroup: 16 rows
    const int lane = lane_id();
    const int cq = (lane & 3) * 2;   // first of the two accumulator columns this thread holds in every 8-column group
    int stage = 0;
    uint32_t phase = 0;
    uint32_t epi_chunk = 0;  // running count of staged chunks (selects the staging buffer)
    float acc[BLOCK_N / 2];
    // Shared-window address of the stage ring, pinned in a register.  In a cluster kernel a shared address carries the
    // CTA's id, and ptxas rebuilt it from SR_CgaCtaId before every k-block's barrier wait and first wgmma instead of
    // keeping it live.
    uint32_t ring;
    asm volatile("mov.b32 %0, %1;\n" : "=r"(ring) : "r"(smem_u32(smem)));
    const uint32_t ring_b = ring + static_cast<uint32_t>(smem_b - smem);
    const uint32_t ring_full = ring + static_cast<uint32_t>(reinterpret_cast<uint8_t*>(full_bar) - smem);
    const uint32_t ring_empty = ring + static_cast<uint32_t>(reinterpret_cast<uint8_t*>(empty_bar) - smem);
    auto release = [&](int s) {  // one thread per consumer warpgroup frees the stage (in both CTAs of a pair)
      if (wq == 0 && lane == 0) {
        if constexpr (CTAS == 2) {
          mbar_arrive_cluster(ring_empty + s * 8, 0);
          mbar_arrive_cluster(ring_empty + s * 8, 1);
        } else {
          mbar_arrive(&empty_bar[s]);
        }
      }
    };
    TileCoord t_next = get_tile<MODE, BLOCK_N, TILE_M>(p, first_tile);
    for (int tile = first_tile; tile < total_tiles; tile += tile_stride) {
      const TileCoord t = t_next;
      if (tile + tile_stride < total_tiles) t_next = get_tile<MODE, BLOCK_N, TILE_M>(p, tile + tile_stride);
      if (!t.valid) continue;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      wgmma_fence_regs(acc);
      int prev = -1;
      for (int kb = 0; kb < t.k_blocks; ++kb) {
        mbar_wait_flag(ring_full + stage * 8, phase, stuck);
        const uint32_t a_addr = ring + stage * C::A_STAGE_BYTES;
        const uint32_t b_addr = ring_b + stage * C::B_STAGE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
          const uint64_t da = A_MN ? make_wgmma_desc(a_addr + cw * (BLOCK_K * 128) + k * (MMA_K * 128), BLOCK_K * 128, 1024)
                                   : make_wgmma_desc(a_addr + cw * (64 * 128) + k * (MMA_K * 2), 16, 1024);
          const uint64_t db = B_MN ? make_wgmma_desc(b_addr + k * (MMA_K * 128), BLOCK_K * 128, 1024)
                                   : make_wgmma_desc(b_addr + k * (MMA_K * 2), 16, 1024);
          wgmma_bf16_ss<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs are complete: its stage can be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0) release(prev);

      const int rbase = t.m_blk * TILE_M + pair_rank * BLOCK_M + cw * 64 + wq * 16;  // first of this warp's 16 rows
      const int col0 = t.n_blk * BLOCK_N;
      const bool have_acc = t.k_blocks > 0;

      if constexpr (EPI == EPI_CE_LSE || EPI == EPI_CE_LSE_SUM) {
        // softmax statistics of this tile's columns; a row's columns are spread over the 4 threads of a quad.  Accumulator
        // column o = 8 j + e of this thread is class col0 + cq + o: the column loops compare o with per-row bounds only
        const bool ce_xf = (p.ce_bias != nullptr) || (p.ce_softcap > 0.f);  // warp-uniform
        const float ce_inv_cap = p.ce_softcap > 0.f ? 1.f / p.ce_softcap : 0.f;
        const int ncol = p.N - col0 - cq;  // columns o >= ncol lie past the last class
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = rbase + (lane >> 2) + 8 * h;
          const bool row_ok = row < p.M;
          long long tgt = row_ok ? p.ce_target[row] : -1;
          tgt = (tgt == p.ce_ignore_index) ? -1 : tgt - p.ce_col_offset;  // class id relative to this slice of the classifier
          // the target's column o when this thread holds it (o % 8 is 0 or 1), else -1
          const long long tgt_o = tgt - col0 - cq;
          const bool mine = tgt >= 0 && tgt_o >= 0 && tgt_o < BLOCK_N && tgt_o < ncol && (tgt_o & 6) == 0;
          const int trel = mine ? static_cast<int>(tgt_o) : -1;
          float mx = -INFINITY, tgt_logit = 0.f;
          // one loop per transform: a branch on ce_xf inside the unrolled loop keeps both paths' temporaries live
          auto logits = [&](auto xf) {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int o = 8 * j + e;
                float v = acc[4 * j + 2 * h + e];
                if constexpr (decltype(xf)::value) {
                  float dz;
                  const float b = (p.ce_bias != nullptr && o < ncol) ? p.ce_bias[col0 + cq + o] : 0.f;
                  v = ce_transform(v, b, p.ce_softcap, ce_inv_cap, dz);
                }
                v = (o < ncol) ? v : -INFINITY;
                acc[4 * j + 2 * h + e] = v;
                mx = fmaxf(mx, v);
                if (o == trel) tgt_logit = v;
              }
            }
          };
          if (ce_xf) logits(std::true_type{});
          else logits(std::false_type{});
          if (row_ok && trel >= 0) p.ce_tgt_logit[row] = tgt_logit;
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          float sum = 0.f;
          if (mx > -INFINITY) {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
              sum += __expf(acc[4 * j + 2 * h] - mx) + __expf(acc[4 * j + 2 * h + 1] - mx);
          }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          if (row_ok && (lane & 3) == 0) {
            p.ce_part_max[static_cast<long long>(t.n_blk) * p.M + row] = mx;
            p.ce_part_sum[static_cast<long long>(t.n_blk) * p.M + row] = sum;
          }
          if constexpr (EPI == EPI_CE_LSE_SUM) {
            // the row's logit sum over the tile's valid columns, in a pass of its own once max and sum-exp are stored
            // (accumulated inside the logits loop it kept one more register live there, and the single-CTA kernel spilt)
            float zsum = 0.f;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) zsum += (8 * j + e < ncol) ? acc[4 * j + 2 * h + e] : 0.f;
            }
            zsum += __shfl_xor_sync(0xffffffffu, zsum, 1);
            zsum += __shfl_xor_sync(0xffffffffu, zsum, 2);
            if (row_ok && (lane & 3) == 0) p.ce_part_zsum[static_cast<long long>(t.n_blk) * p.M + row] = zsum;
          }
        }
      } else {
        if constexpr (EPI == EPI_CE_DLOGITS || EPI == EPI_CE_DLOGITS_REG) {
          // D(bf16) = g[row] * (softmax - onehot) * dz/dacc, computed in place on the accumulator (column o as in EPI_CE_LSE).
          // DLOGITS_REG: g[row] * ((1 + 2 zeta lse) softmax - (1 - eps) onehot - eps / V) * dz/dacc
          float p_scale = 1.f, hit = 1.f, uniform = 0.f;
          if constexpr (EPI == EPI_CE_DLOGITS_REG) {
            hit = 1.f - p.ce_smoothing;
            uniform = p.ce_smoothing / static_cast<float>(p.ce_num_classes);
          }
          const bool ce_xf = (p.ce_bias != nullptr) || (p.ce_softcap > 0.f);  // warp-uniform
          const float ce_inv_cap = p.ce_softcap > 0.f ? 1.f / p.ce_softcap : 0.f;
          const int ncol = p.N - col0 - cq;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rbase + (lane >> 2) + 8 * h;
            float lse = 0.f, g = 0.f;
            long long tgt = -1;
            if (row < p.M) {
              tgt = p.ce_target[row];
              lse = p.ce_lse[row];
              g = (tgt == p.ce_ignore_index) ? 0.f : p.ce_grad[row];
              tgt = (tgt == p.ce_ignore_index) ? -1 : tgt - p.ce_col_offset;
            }
            const long long tgt_o = tgt - col0 - cq;
            const int trel = (tgt >= 0 && tgt_o >= 0 && tgt_o < BLOCK_N) ? static_cast<int>(tgt_o) : -1;
            if constexpr (EPI == EPI_CE_DLOGITS_REG) p_scale = fmaf(2.f * p.ce_z_loss, lse, 1.f);
            auto dlogits = [&](auto xf) {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int o = 8 * j + e;
                  float z = acc[4 * j + 2 * h + e];
                  float dz = 1.f;
                  if constexpr (decltype(xf)::value) {
                    const float b = (p.ce_bias != nullptr && o < ncol) ? p.ce_bias[col0 + cq + o] : 0.f;
                    z = ce_transform(z, b, p.ce_softcap, ce_inv_cap, dz);
                  }
                  float pr = __expf(z - lse);
                  if constexpr (EPI == EPI_CE_DLOGITS_REG) {
                    pr = fmaf(pr, p_scale, -uniform);
                    if (o == trel) pr -= hit;
                  } else {
                    if (o == trel) pr -= 1.f;
                  }
                  acc[4 * j + 2 * h + e] = pr * g * dz;
                }
              }
            };
            if (ce_xf) dlogits(std::true_type{});
            else dlogits(std::false_type{});
          }
        }
        constexpr bool OUT_BF16 = (EPI == EPI_BF16 || EPI == EPI_BF16_ACC || EPI == EPI_CE_DLOGITS || EPI == EPI_CE_DLOGITS_REG);
        constexpr bool REDUCE = (EPI == EPI_F32_ACC || EPI == EPI_BF16_ACC);
        if (p.tma_epilogue) {
          // ---- TMA epilogue: 128-byte output chunks (32 fp32 / 64 bf16 columns) of the warp's 16 rows, staged swizzled ----
          constexpr int CHUNK_COLS = OUT_BF16 ? 64 : 32;
          static_assert(BLOCK_N % CHUNK_COLS == 0, "BLOCK_N must be a multiple of the epilogue chunk");
          if (have_acc || !REDUCE) {
#pragma unroll
            for (int c = 0; c < BLOCK_N / CHUNK_COLS; ++c) {
              const int cbase = col0 + c * CHUNK_COLS;
              if (cbase >= p.N) break;  // warp-uniform
              uint8_t* stage_buf = smem_epi + ((cw * 4 + wq) * C::EPI_BUFS + (epi_chunk % C::EPI_BUFS)) * (EPI_BOX_ROWS * 128);
              ++epi_chunk;
              if (lane == 0) tma_store_wait_read<C::EPI_BUFS - 1>();  // the store that last read this buffer has drained
              __syncwarp();
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = (lane >> 2) + 8 * h;
                uint8_t* my_row = stage_buf + r * 128;
                // 16-byte chunk q of row r lives at q ^ (r & 7) under the 128B swizzle
                if constexpr (OUT_BF16) {
#pragma unroll
                  for (int jj = 0; jj < 8; ++jj) {
                    const int j = c * 8 + jj;
                    *reinterpret_cast<uint32_t*>(my_row + ((jj ^ (r & 7)) << 4) + (lane & 3) * 4) =
                        pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                  }
                } else {
#pragma unroll
                  for (int jj = 0; jj < 4; ++jj) {
                    const int j = c * 4 + jj;
                    const int q = 2 * jj + ((lane & 3) >> 1);
                    *reinterpret_cast<float2*>(my_row + ((q ^ (r & 7)) << 4) + (lane & 1) * 8) =
                        make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                  }
                }
              }
              fence_proxy_async_smem();
              __syncwarp();
              if (lane == 0) {
                const int g0 = (MODE == GROUPED_K) ? t.group : 0;
                if constexpr (COMM == COMM_RS_D) {  // reduce-add into the shard of the peer that owns these rows
                  int owner, r_local;
                  comm_locate(p, rbase, owner, r_local);
                  tma_reduce_add_3d(&peers.m[owner], stage_buf, cbase, r_local, 0);
                } else if constexpr (REDUCE) tma_reduce_add_3d(&tmap_d, stage_buf, cbase, rbase, g0);
                else tma_store_3d(&tmap_d, stage_buf, cbase, rbase, g0);
                tma_store_commit();
              }
            }
          }
        } else {
          // ---- direct global stores (outputs TMA cannot address) ----
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rbase + (lane >> 2) + 8 * h;
            if (row >= p.M) continue;
            long long d_off = static_cast<long long>(row) * p.ldd;
            if (MODE == GROUPED_K) d_off += static_cast<long long>(t.group) * p.d_group_stride;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
              const int col = col0 + 8 * j + cq;
              if (col >= p.N) continue;
              const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              const bool pair_ok = col + 1 < p.N;
              if constexpr (OUT_BF16) {
                __nv_bfloat16* dptr = reinterpret_cast<__nv_bfloat16*>(p.D) + d_off + col;
                if (pair_ok && (reinterpret_cast<uintptr_t>(dptr) & 3) == 0) {
                  float2 o = make_float2(v0, v1);
                  if constexpr (EPI == EPI_BF16_ACC) {
                    const float2 old = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dptr));
                    o.x += old.x; o.y += old.y;
                  }
                  *reinterpret_cast<uint32_t*>(dptr) = pack_bf16x2(o.x, o.y);
                } else {
                  float o0 = v0, o1 = v1;
                  if constexpr (EPI == EPI_BF16_ACC) {
                    o0 += __bfloat162float(dptr[0]);
                    if (pair_ok) o1 += __bfloat162float(dptr[1]);
                  }
                  dptr[0] = __float2bfloat16_rn(o0);
                  if (pair_ok) dptr[1] = __float2bfloat16_rn(o1);
                }
              } else {
                float* dptr = reinterpret_cast<float*>(p.D) + d_off + col;
                if (pair_ok && (reinterpret_cast<uintptr_t>(dptr) & 7) == 0) {
                  float2 o = make_float2(v0, v1);
                  if constexpr (EPI == EPI_F32_ACC) {
                    const float2 old = *reinterpret_cast<const float2*>(dptr);
                    o.x += old.x; o.y += old.y;
                  }
                  *reinterpret_cast<float2*>(dptr) = o;
                } else {
                  float o0 = v0, o1 = v1;
                  if constexpr (EPI == EPI_F32_ACC) {
                    o0 += dptr[0];
                    if (pair_ok) o1 += dptr[1];
                  }
                  dptr[0] = o0;
                  if (pair_ok) dptr[1] = o1;
                }
              }
            }
          }
        }
      }
    }
    if (lane == 0) tma_store_wait<0>();  // all bulk stores of this warp are complete before smem is released
  }

  // pair: neither CTA leaves while its peer may still multicast into its smem or arrive on its barriers
  if constexpr (CTAS == 2) cluster_sync_all();
  // A stuck consumer fell through its later waits (it still released every stage and stored its tiles, so neither the
  // producer nor the pair's peer waits on it forever) and turns the hang into a trap here, outside the region whose
  // register budget setmaxnreg raised.
  if (stuck) __trap();
}

}  // namespace gemm
}  // namespace d9d
