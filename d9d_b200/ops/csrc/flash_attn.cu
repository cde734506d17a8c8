// d9d_b200 — flash attention forward + backward on wgmma (sm_90a).
//
//   O = softmax(scale * Q K^T + mask [, sink]) V            GQA (Hq = g * Hk), causal / sliding window (left, right),
//                                                           optional tanh soft-cap, optional per-head attention sink,
//                                                           fixed-length batches or packed variable-length sequences.
//
// All tensors are [rows, H, D] row-major views of the projection outputs (rows = B*S, or the packed token count):
// no transposes, TMA 3-D maps (d, h, row) with 128B swizzle.  LSE / delta are fp32 [B, H, S] (packed: [H, total]).
// Q / K / dQ / dK have head dim DQK, V / O / dO / dV head dim DV; the built pairs (DQK, DV) are (64, 64), (128, 128) and
// (192, 128) (multi-head latent attention: 128 nope + 64 rope query / key columns, 128 value columns).
//
// Forward (flash_attn_fwd_kernel): one CTA owns a 128-row query tile of one (batch, head); warpgroup 0 streams K / V tiles
// of 128 keys with TMA, warpgroups 1-2 own 64 query rows each with S, P and O in registers (P is handed to the second
// GEMM as its register A operand).
// Backward = delta pre-pass + two wgmma kernels built from one template (no atomics, deterministic): see
// flash_attn_bwd_kernel.
// Reference parity: d9d/kernel/flash_attn/function.py:72-178 (fwd/bwd, sink gradient), :181-305 (varlen).
#include <stdexcept>
#include <string>
#include <type_traits>

#include "gemm_host.cuh"

namespace d9d {
namespace {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct FaParams {
  int B, Sq, Sk, Hq, Hk;     // Sq / Sk: per-sequence lengths (fixed-length) or maxima (varlen)
  int wl, wr;                // window: key k visible to query q iff q+off-wl <= k <= q+off+wr (off = Sk-Sq); -1 = unbounded
  float scale, softcap;      // softcap == 0 -> off
  const int* cu_q;           // [B+1] or nullptr
  const int* cu_k;
  long long lse_bs, lse_hs;  // lse / delta index = b*lse_bs + h*lse_hs + (varlen ? q_start : 0) + q
  const float* sink;         // [Hq] or nullptr (forward)
  __nv_bfloat16* out;        // forward output / unused
  float* lse;                // forward: written; backward: read
  const float* delta;        // backward
  __nv_bfloat16 *dq, *dk, *dv;
};

struct SeqInfo {
  int q_start, k_start, Sq, Sk, off;
  long long lse_base;  // + h*lse_hs + q
};

__device__ __forceinline__ SeqInfo resolve_seq(const FaParams& p, int b) {
  SeqInfo s;
  if (p.cu_q != nullptr) {
    s.q_start = p.cu_q[b];
    s.Sq = p.cu_q[b + 1] - s.q_start;
    s.k_start = p.cu_k[b];
    s.Sk = p.cu_k[b + 1] - s.k_start;
    s.lse_base = s.q_start;
  } else {
    s.q_start = b * p.Sq;
    s.Sq = p.Sq;
    s.k_start = b * p.Sk;
    s.Sk = p.Sk;
    s.lse_base = static_cast<long long>(b) * p.lse_bs;
  }
  s.off = s.Sk - s.Sq;
  return s;
}

// The grid is one-dimensional (gridDim.z would cap a packed batch at 65535 sequences):
//   blockIdx.x = tile + tiles * (head + H * b), the dispatch order of a (tiles, H, B) grid
struct TileIdx {
  int tile, head, b;
};
__device__ __forceinline__ TileIdx decode_block(int tiles, int H) {
  const int x = static_cast<int>(blockIdx.x), th = tiles * H;
  TileIdx t;
  t.b = x / th;
  t.head = (x - t.b * th) / tiles;
  t.tile = x - t.b * th - t.head * tiles;
  return t;
}

// A streamed tile that runs past the end of its sequence holds rows of the next sequence, batch element or padding.  Masking
// zeroes their P / dS, but 0 * NaN = NaN on the tensor core, so the rows themselves must be zero.  The producer warp lands
// such a tile on a separate barrier, zeroes rows [r_from, box_rows) of its `nbox` [box_rows x 128 B] boxes with this
// function and only then arrives on the consumers' full barrier; whole tiles take the plain TMA path.  The 128B swizzle only
// permutes the 16-byte chunks inside a row: whole rows need no un-swizzling.
__device__ __forceinline__ void zero_tile_rows(uint8_t* tile, int box_rows, int nbox, int r_from, int lane) {
  const int n = (box_rows - r_from) * 8;
  for (int bx = 0; bx < nbox; ++bx) {
    uint8_t* base = tile + bx * box_rows * 128 + r_from * 128;
    for (int i = lane; i < n; i += 32) *reinterpret_cast<uint4*>(base + i * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
  fence_proxy_async_smem();  // generic-proxy zeros before the wgmma (async proxy) reads
  __syncwarp();
}

// ======================================================================================================
// forward
// ======================================================================================================
constexpr int FA_THREADS = 384;  // warpgroup 0: TMA producer; warpgroups 1-2: 64 resident rows each
constexpr int FA_CONSUMERS = 2;

// wgmma operand descriptors of the [rows x 128 B] 128B-swizzled boxes TMA writes (one box per 64 head-dim columns)
//   K-major operand (head dim = reduction):  k-step kk of 16 columns at box kk / 4, byte 32 (kk % 4) of every row
//   MN-major operand (rows = reduction):     k-step kk = rows [16 kk, 16 kk + 16), LBO = distance between the d boxes
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t base, int box_bytes, int kk) {
  return make_wgmma_desc(base + (kk >> 2) * box_bytes + (kk & 3) * 32, 16, 1024);
}
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t base, int box_bytes, int kk) {
  return make_wgmma_desc(base + kk * (16 * 128), box_bytes, 1024);
}

// accumulator columns [16 s, 16 s + 16) of an m64 fragment, rounded to bf16: the A operand of k-step s
template <int R>
__device__ __forceinline__ void pack_a_frag(const float (&d)[R], int s, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * s + 0], d[8 * s + 1]);
  a[1] = pack_bf16x2(d[8 * s + 2], d[8 * s + 3]);
  a[2] = pack_bf16x2(d[8 * s + 4], d[8 * s + 5]);
  a[3] = pack_bf16x2(d[8 * s + 6], d[8 * s + 7]);
}

// select one of two lvalues at compile time (they may have different types)
template <bool FIRST, class A, class B>
__device__ __forceinline__ auto& pick(A& a, B& b) {
  if constexpr (FIRST) return a;
  else return b;
}

template <int DQK, int DV>
struct FwdCfg {
  static constexpr int QK_BYTES = 128 * DQK * 2;  // Q tile and every K tile: 128 rows
  static constexpr int V_BYTES = 128 * DV * 2;    // every V tile
  static constexpr int NSLOT = 2;                 // K and V rings
  static constexpr int SMEM_BYTES = QK_BYTES + NSLOT * (QK_BYTES + V_BYTES) + 1024 + 256;
};

// One CTA owns a 128-row query tile of one (batch, head); each consumer warpgroup owns 64 of its rows and keeps S, P and O
// in registers: S = Q K_j^T (wgmma from shared memory), online softmax on the fragment (a row lives in the 4 threads of a
// quad), P packed to bf16 in place as the register A operand of O += P V_j.  The producer streams K_j / V_j through two
// 2-slot rings, so the loads of tile j+1 run under the math of tile j.
template <int DQK, int DV>
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, const FaParams p) {
  using C = FwdCfg<DQK, DV>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem_q + C::QK_BYTES;               // [NSLOT][QK tile]
  uint8_t* smem_v = smem_k + C::NSLOT * C::QK_BYTES;    // [NSLOT][V tile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + C::NSLOT * C::V_BYTES);
  uint64_t* bar_q = bars;         // 1
  uint64_t* k_full = bars + 1;    // [2]
  uint64_t* k_empty = bars + 3;   // [2]
  uint64_t* v_full = bars + 5;    // [2]
  uint64_t* v_empty = bars + 7;   // [2]
  uint64_t* v_land = bars + 9;    // 1: the partial last V tile, zeroed past Sk before v_full

  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int tiles = (p.Sq + 127) / 128;
  const TileIdx bi = decode_block(tiles, p.Hq);
  const int h = bi.head, b = bi.b;
  const int hk = h / (p.Hq / p.Hk);
  const SeqInfo sq = resolve_seq(p, b);
  const int q0 = (tiles - 1 - bi.tile) * 128;  // heavy (late) query tiles first
  if (q0 >= sq.Sq) return;  // whole CTA exits together (varlen: shorter sequences)

  // kv tile range [jbeg, jend) of the query rows [q0, qb]
  const int qb = min(q0 + 127, sq.Sq - 1);
  const int klo = p.wl < 0 ? 0 : max(0, q0 + sq.off - p.wl);
  const int khi = p.wr < 0 ? sq.Sk - 1 : min(sq.Sk - 1, qb + sq.off + p.wr);
  const int jbeg = klo / 128, jend = (khi >= klo) ? khi / 128 + 1 : jbeg;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(bar_q, 1);
    mbar_init(v_land, 1);
    for (int i = 0; i < C::NSLOT; ++i) {
      mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], FA_CONSUMERS);
      mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], FA_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================= TMA producer =================
    setmaxnreg_dec<40>();
    // a tile without visible keys loads nothing: its consumers never wait on bar_q, and no copy may still be landing in
    // shared memory when the CTA exits
    // shared memory when the CTA exits.  Only the last key tile can run past Sk: its V rows there are zeroed (K rows past
    // Sk only reach masked scores)
    if (warp == 0 && jend > jbeg) {
      if (elect_one()) {
        mbar_arrive_expect_tx(bar_q, C::QK_BYTES);
#pragma unroll
        for (int dc = 0; dc < DQK / 64; ++dc)
          tma_load_3d(smem_q + dc * (128 * 128), &tmap_q, bar_q, dc * 64, h, sq.q_start + q0);
        for (int j = jbeg; j < jend; ++j) {
          const int n = j - jbeg, slot = n % C::NSLOT;
          const uint32_t ph = (n / C::NSLOT) & 1;
          mbar_wait_wg(&k_empty[slot], ph ^ 1);
          mbar_arrive_expect_tx(&k_full[slot], C::QK_BYTES);
#pragma unroll
          for (int dc = 0; dc < DQK / 64; ++dc)
            tma_load_3d(smem_k + slot * C::QK_BYTES + dc * (128 * 128), &tmap_k, &k_full[slot], dc * 64, hk, sq.k_start + j * 128);
          mbar_wait_wg(&v_empty[slot], ph ^ 1);
          uint64_t* vbar = (j * 128 + 128 > sq.Sk) ? v_land : &v_full[slot];
          mbar_arrive_expect_tx(vbar, C::V_BYTES);
#pragma unroll
          for (int dc = 0; dc < DV / 64; ++dc)
            tma_load_3d(smem_v + slot * C::V_BYTES + dc * (128 * 128), &tmap_v, vbar, dc * 64, hk, sq.k_start + j * 128);
        }
      }
      __syncwarp();
      const int jl = jend - 1, k_last = jl * 128;
      if (k_last + 128 > sq.Sk) {
        const int slot = (jl - jbeg) % C::NSLOT;
        mbar_wait_wg(v_land, 0);
        zero_tile_rows(smem_v + slot * C::V_BYTES, 128, DV / 64, sq.Sk - k_last, lane);
        if (lane == 0) mbar_arrive(&v_full[slot]);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ================= consumers: softmax + both GEMMs of 64 query rows =================
    const int cw = (warp >> 2) - 1, wq = warp & 3;
    const int cq = (lane & 3) * 2;
    const int row_l = cw * 64 + wq * 16 + (lane >> 2);  // tile rows row_l and row_l + 8 of this thread
    const bool signal = (wq == 0 && lane == 0);
    int k_lo[2], k_hi[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int qi = q0 + row_l + 8 * r;
      k_lo[r] = p.wl < 0 ? 0 : max(0, qi + sq.off - p.wl);
      k_hi[r] = p.wr < 0 ? sq.Sk - 1 : min(sq.Sk - 1, qi + sq.off + p.wr);
    }
    const bool capped = p.softcap != 0.f;
    const float scale_eff = capped ? kLog2e : p.scale * kLog2e;  // log2-domain multiplier of the (capped) score
    const float cap_in = capped ? p.scale / p.softcap : 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[DV / 2];
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
    const uint32_t q_addr = smem_u32(smem_q) + cw * (64 * 128);
    if (jend > jbeg) mbar_wait_wg(bar_q, 0);
    for (int j = jbeg; j < jend; ++j) {
      const int n = j - jbeg, slot = n % C::NSLOT;
      const uint32_t ph = (n / C::NSLOT) & 1;
      const int k0 = j * 128;
      float s[64];
      mbar_wait_wg(&k_full[slot], ph);
      const uint32_t k_addr = smem_u32(smem_k + slot * C::QK_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DQK / 16; ++kk)
        wgmma_bf16_ss<128, 0, 0>(s, desc_kmajor(q_addr, 128 * 128, kk), desc_kmajor(k_addr, 128 * 128, kk), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      if (signal) mbar_arrive(&k_empty[slot]);
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int lo_rel = k_lo[r] - k0 - cq, hi_rel = k_hi[r] - k0 - cq;
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float x = s[4 * jj + 2 * r + e];
            if (capped) x = p.softcap * tanhf(x * cap_in);
            const int c = 8 * jj + e;  // key k0 + cq + c
            x = (c < lo_rel || c > hi_rel) ? -INFINITY : x;
            s[4 * jj + 2 * r + e] = x;
            mx = fmaxf(mx, x);
          }
        }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[r], mx * scale_eff);
        alpha[r] = (m_new == -INFINITY) ? 1.f : exp2f(m[r] - m_new);
        m[r] = m_new;
        l[r] *= alpha[r];
        const float neg_m = (m_new == -INFINITY) ? 0.f : -m_new;
        float sum = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = exp2f(fmaf(s[4 * jj + 2 * r + e], scale_eff, neg_m));
            s[4 * jj + 2 * r + e] = pv;
            sum += pv;
          }
        }
        l[r] += sum;  // partial over this thread's columns; the quad is summed once at the end
      }
#pragma unroll
      for (int jj = 0; jj < DV / 8; ++jj) {
        o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
        o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
      }
      uint32_t pa[8][4];
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) pack_a_frag(s, ks, pa[ks]);
      mbar_wait_wg(&v_full[slot], ph);
      const uint32_t v_addr = smem_u32(smem_v + slot * C::V_BYTES);
      wgmma_fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) wgmma_bf16_rs<DV, 1>(o, pa[ks], desc_mnmajor(v_addr, 128 * 128, ks), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (signal) mbar_arrive(&v_empty[slot]);
    }
    // ---- epilogue: O / l -> global, LSE (natural log; the sink joins the denominator)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float lr = l[r], m_fin = m[r], o_scale = 1.f;
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      if (p.sink != nullptr) {
        // the sink joins the running max, so that a sink far above every score (or a row without visible keys) cannot
        // overflow l
        const float s2 = p.sink[h] * kLog2e;
        if (s2 > m[r]) {
          o_scale = exp2f(m[r] - s2);
          lr = lr * o_scale + 1.f;
          m_fin = s2;
        } else if (m[r] != -INFINITY) {
          lr += exp2f(s2 - m[r]);
        }
      }
      const float m_safe = (m_fin == -INFINITY) ? 0.f : m_fin;
      const float inv_l = (lr > 0.f) ? o_scale / lr : 0.f;
      const int qi = q0 + row_l + 8 * r;
      if (qi < sq.Sq) {
        __nv_bfloat16* dst = p.out + (static_cast<long long>(sq.q_start + qi) * p.Hq + h) * DV + cq;
#pragma unroll
        for (int jj = 0; jj < DV / 8; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * r] * inv_l, o[4 * jj + 2 * r + 1] * inv_l);
        if ((lane & 3) == 0 && p.lse != nullptr)
          p.lse[sq.lse_base + static_cast<long long>(h) * p.lse_hs + qi] = (lr > 0.f) ? (m_safe + log2f(lr)) * kLn2 : -INFINITY;
      }
    }
  }
}

// ======================================================================================================
// backward
// ======================================================================================================
template <int DQK, int DV, bool DKV>
struct BwdCfg {
  // Streamed tile height SR and ring depth NST.  At (192, 128) the dK/dV consumers hold dK (96 registers) and dV (64): with
  // 64-row streamed tiles S^T, dP^T and their bf16 operands would take another 96, so they stream 32-row tiles (m64n32 S^T
  // and dP^T).  Four 64-row stages of Q + dO (dK/dV) or K + V (dQ) exceed shared memory at DQK = 192: dQ keeps three.
  static constexpr int SR = (DQK == 192 && DKV) ? 32 : 64;
  static constexpr int NST = DQK == 192 ? (DKV ? 6 : 3) : 4;
  static constexpr int R1_BYTES = 128 * DQK * 2;  // resident K (DKV) / Q (DQ)
  static constexpr int R2_BYTES = 128 * DV * 2;   // resident V (DKV) / dO (DQ)
  static constexpr int S1_BYTES = SR * DQK * 2;   // streamed Q (DKV) / K (DQ)
  static constexpr int S2_BYTES = SR * DV * 2;    // streamed dO (DKV) / V (DQ)
  static constexpr int STAGE_BYTES = S1_BYTES + S2_BYTES;
  static constexpr int VEC_BYTES = DKV ? NST * 2 * SR * 4 : 0;
  static constexpr int SMEM_BYTES = R1_BYTES + R2_BYTES + NST * STAGE_BYTES + VEC_BYTES + 1024 + 256;
  // per-thread register budgets (setmaxnreg; 2 x 128 x CONSUMER + 128 x PRODUCER <= 64 K).  The D = 128 consumers hold
  // two 64 x 128 fp32 accumulators, S, dP and the bf16 A operands with wgmma in flight: below 240 ptxas serialises them
  // (C7512).  The D = 64 producer spills at 24.
  static constexpr int CONSUMER_REGS = DQK == 64 ? 232 : 240;
  static constexpr int PRODUCER_REGS = DQK == 64 ? 40 : 24;
};

// Two kernels from one template (no atomics, deterministic):
//   DKV: CTA owns a 128-key tile of one kv head (64 keys per consumer warpgroup), keeps K,V resident, streams SR-row Q/dO
//        tiles of every query head of the group: S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T (registers, bf16 A operands)
//        -> dV += P^T dO, dK += dS^T Q accumulated in registers over the whole loop.
//   DQ : CTA owns a 128-row query tile of one head, keeps Q,dO resident, streams SR-key K/V tiles:
//        S = Q K^T, dP = dO V^T -> dS -> dQ += dS K.
// S and dS reduce over DQK (Q, K), dP over DV (V, dO).
template <int DQK, int DV, bool DKV>
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_r1, const __grid_constant__ CUtensorMap tmap_r2,
                      const __grid_constant__ CUtensorMap tmap_s1, const __grid_constant__ CUtensorMap tmap_s2, const FaParams p) {
  // DKV: r1 = K, r2 = V (128-row boxes), s1 = Q, s2 = dO (SR-row boxes).   DQ: r1 = Q, r2 = dO, s1 = K, s2 = V.
  using C = BwdCfg<DQK, DV, DKV>;
  constexpr int SR = C::SR, NST = C::NST;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_r1 = smem;
  uint8_t* smem_r2 = smem_r1 + C::R1_BYTES;
  uint8_t* smem_s = smem_r2 + C::R2_BYTES;                      // [NST][s1 | s2]
  float* smem_vec = reinterpret_cast<float*>(smem_s + NST * C::STAGE_BYTES);  // DKV: [NST][lse2(SR) | delta(SR)]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(smem_vec) + C::VEC_BYTES);
  uint64_t* r_full = bars;                  // 1
  uint64_t* st_full = bars + 1;             // [NST]
  uint64_t* st_empty = bars + 1 + NST;      // [NST]
  uint64_t* st_land = bars + 1 + 2 * NST;   // 1: a streamed tile past the end of the sequence, zeroed there before st_full

  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int tiles = ((DKV ? p.Sk : p.Sq) + 127) / 128;
  const TileIdx bi = decode_block(tiles, DKV ? p.Hk : p.Hq);
  const int b = bi.b;
  const SeqInfo sq = resolve_seq(p, b);
  const int g = p.Hq / p.Hk;
  // first resident row (key for DKV, query for DQ), sequence-local.  Blocks are dispatched in blockIdx order: under a causal
  // mask the heavy tiles are the early keys (DKV: natural order) and the LATE queries (DQ: reversed order), so that the light
  // tiles fill the tail of the grid
  const int r0 = (DKV ? bi.tile : tiles - 1 - bi.tile) * 128;
  if (r0 >= (DKV ? sq.Sk : sq.Sq)) return;
  const int head = bi.head;         // DKV: kv head; DQ: query head
  const int hk = DKV ? head : head / g;

  // streamed tile range [clo, chi) in units of SR rows
  int clo = 0, chi = 0;
  if constexpr (DKV) {
    const int qa = p.wr < 0 ? 0 : max(0, r0 - sq.off - p.wr);                         // first query seeing key r0
    const int qb = p.wl < 0 ? sq.Sq - 1 : min(sq.Sq - 1, r0 + 127 - sq.off + p.wl);    // last query seeing key r0+127
    if (qb >= qa) { clo = qa / SR; chi = qb / SR + 1; }
  } else {
    const int qb = min(r0 + 127, sq.Sq - 1);
    const int ka = p.wl < 0 ? 0 : max(0, r0 + sq.off - p.wl);
    const int kb = p.wr < 0 ? sq.Sk - 1 : min(sq.Sk - 1, qb + sq.off + p.wr);
    if (kb >= ka) { clo = ka / SR; chi = kb / SR + 1; }
  }
  const int nc = chi - clo;
  const int T = DKV ? g * nc : nc;  // streamed tiles processed by this CTA

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_r1);
    tma_prefetch_desc(&tmap_r2);
    tma_prefetch_desc(&tmap_s1);
    tma_prefetch_desc(&tmap_s2);
    mbar_init(r_full, 1);
    mbar_init(st_land, 1);
    for (int i = 0; i < NST; ++i) { mbar_init(&st_full[i], DKV ? 2 : 1); mbar_init(&st_empty[i], FA_CONSUMERS); }
    fence_barrier_init();
  }
  __syncthreads();
  const float scale_log2 = p.scale * kLog2e;
  bool stuck = false;  // a consumer's mbarrier wait timed out (see mbar_wait_flag)

  if (warp < 4) {
    setmaxnreg_dec<C::PRODUCER_REGS>();
    // ================= producer (warp 0): TMA tiles (+ lse / delta vectors in DKV mode) =================
    if (warp == 0 && T > 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(r_full, C::R1_BYTES + C::R2_BYTES);
        const int rrow = (DKV ? sq.k_start : sq.q_start) + r0;
#pragma unroll
        for (int dc = 0; dc < DQK / 64; ++dc) {
          tma_load_3d(smem_r1 + dc * (128 * 128), &tmap_r1, r_full, dc * 64, head, rrow);
          if (dc < DV / 64) tma_load_3d(smem_r2 + dc * (128 * 128), &tmap_r2, r_full, dc * 64, head, rrow);
        }
      }
      __syncwarp();
      const int s_len = DKV ? sq.Sq : sq.Sk;
      int n_land = 0;
      for (int t = 0; t < T; ++t) {
        const int st = t % NST;
        const int hs = DKV ? head * g + t / nc : hk;   // head of the streamed operand
        const int c0 = (clo + (DKV ? t % nc : t)) * SR;  // first streamed row, sequence-local
        const bool partial = c0 + SR > s_len;
        uint64_t* bar = partial ? st_land : &st_full[st];
        mbar_wait_wg(&st_empty[st], ((t / NST) & 1) ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(bar, C::STAGE_BYTES);
          const int srow = (DKV ? sq.q_start : sq.k_start) + c0;
          uint8_t* dst = smem_s + st * C::STAGE_BYTES;
#pragma unroll
          for (int dc = 0; dc < DQK / 64; ++dc) {
            tma_load_3d(dst + dc * (SR * 128), &tmap_s1, bar, dc * 64, hs, srow);
            if (dc < DV / 64) tma_load_3d(dst + C::S1_BYTES + dc * (SR * 128), &tmap_s2, bar, dc * 64, hs, srow);
          }
        }
        if (partial) {
          // DKV: Q and dO rows past Sq (both feed a second GEMM).  DQ: K rows past Sk; its V rows only reach dP, which the
          // mask selects away.  The stage's boxes are contiguous: Q (K) boxes, then dO (V) boxes
          __syncwarp();
          mbar_wait_wg(st_land, n_land & 1);
          ++n_land;
          zero_tile_rows(smem_s + st * C::STAGE_BYTES, SR, DKV ? DQK / 64 + DV / 64 : DQK / 64, s_len - c0, lane);
          if (lane == 0) mbar_arrive(&st_full[st]);
        }
        if constexpr (DKV) {
          // per-query statistics of this tile: lse in the log2 domain (+inf -> P = 0 for rows outside the sequence).
          // Column c = 8 jj + 2 quad + e of a consumer fragment goes to quad * SR/4 + 2 jj + e: the two columns a consumer
          // thread reads per jj are one 8-byte shared load
          constexpr int PER_LANE = SR / 32;
          float* vec = smem_vec + st * (2 * SR);
          const long long base = sq.lse_base + static_cast<long long>(hs) * p.lse_hs;
#pragma unroll
          for (int e = 0; e < PER_LANE; ++e) {
            const int c = lane * PER_LANE + e, q = c0 + c;
            const int pos = ((c >> 1) & 3) * (SR / 4) + (c >> 3) * 2 + (c & 1);
            float l2 = INFINITY, dl = 0.f;
            if (q < sq.Sq) {
              const float lv = p.lse[base + q];
              l2 = (lv == -INFINITY) ? INFINITY : lv * kLog2e;
              dl = p.delta[base + q];
            }
            vec[pos] = l2;
            vec[SR + pos] = dl;
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&st_full[st]);
        }
        __syncwarp();
      }
    }
  } else {
    setmaxnreg_inc<C::CONSUMER_REGS>();
    // ================= consumers: 64 resident rows each =================
    const int cw = (warp >> 2) - 1, wq = warp & 3;
    const int cq = (lane & 3) * 2;
    const int row_l = cw * 64 + wq * 16 + (lane >> 2);  // resident rows row_l, row_l + 8 of this thread
    const bool signal = (wq == 0 && lane == 0);
    const bool capped = p.softcap != 0.f;
    const float cap_in = capped ? p.scale / p.softcap : 0.f;
    float my_lse2[2] = {INFINITY, INFINITY}, my_delta[2] = {0.f, 0.f};
    if constexpr (!DKV) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int ri = r0 + row_l + 8 * r;
        if (ri < sq.Sq) {
          const long long idx = sq.lse_base + static_cast<long long>(head) * p.lse_hs + ri;
          const float lv = p.lse[idx];
          my_lse2[r] = (lv == -INFINITY) ? INFINITY : lv * kLog2e;
          my_delta[r] = p.delta[idx];
        }
      }
    }
    constexpr int ACC1 = DKV ? DV / 2 : DQK / 2;
    float acc1[ACC1], acc2[DQK / 2];  // DKV: dV, dK.  DQ: dQ, unused
#pragma unroll
    for (int i = 0; i < DQK / 2; ++i) {
      if (i < ACC1) acc1[i] = 0.f;
      acc2[i] = 0.f;
    }
    const uint32_t r1_addr = smem_u32(smem_r1) + cw * (64 * 128), r2_addr = smem_u32(smem_r2) + cw * (64 * 128);
    // Commit groups per streamed tile, in issue order: S, dP, [dV,] dK / dQ.  The exp of P runs while dP is on the tensor
    // cores and dS is formed while dV runs.  The tile's groups all retire before the next one starts: groups still in
    // flight across the loop's back edge make ptxas serialise every wgmma (C7515).
    // DKV: the two consumer warpgroups take turns to issue S and dP (named barriers 1 + cw, FA3's warpgroup ping-pong), so
    // that the tensor cores run one warpgroup's GEMMs while the other computes P and dS, instead of both doing their math
    // at once.  Warpgroup 1 opens the first turn for warpgroup 0 and skips its last hand-over: no arrival is left pending.
    // DQ has no dV GEMM to cover the other warpgroup's math and ran 1-5 % slower with the turns (H100): it takes none.
    if (T > 0) {
      if (DKV && cw == 1) named_barrier_arrive(1, 256);
      mbar_wait_flag(r_full, 0, stuck);
    }
    // this thread's lse2 / delta columns 8 jj + cq + {0, 1} of a DKV stage: 8 bytes at vec_lane + 8 jj (see the producer)
    const uint32_t vec_lane = smem_u32(smem_vec) + (lane & 3) * (SR / 4) * 4;
    for (int t = 0; t < T; ++t) {
      const int st = t % NST;
      const int c0 = (clo + (DKV ? t % nc : t)) * SR;  // first streamed row of this tile
      mbar_wait_flag(&st_full[st], (t / NST) & 1, stuck);
      const uint32_t s1_addr = smem_u32(smem_s + st * C::STAGE_BYTES), s2_addr = s1_addr + C::S1_BYTES;
      float s[SR / 2], dp[SR / 2];            // S (then P times the soft-cap derivative), dP
      uint32_t pf[SR / 16][4], df[SR / 16][4];  // P and dS in bf16: the A operands of the second GEMMs
      if constexpr (DKV) named_barrier_sync(1 + cw, 256);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DQK / 16; ++kk)
        wgmma_bf16_ss<SR, 0, 0>(s, desc_kmajor(r1_addr, 128 * 128, kk), desc_kmajor(s1_addr, SR * 128, kk), kk != 0);
      wgmma_commit();
#pragma unroll
      for (int kk = 0; kk < DV / 16; ++kk)
        wgmma_bf16_ss<SR, 0, 0>(dp, desc_kmajor(r2_addr, 128 * 128, kk), desc_kmajor(s2_addr, SR * 128, kk), kk != 0);
      wgmma_commit();
      if (DKV && (cw == 0 || t + 1 < T)) named_barrier_arrive(2 - cw, 256);
      const uint32_t vec_addr = vec_lane + st * (2 * SR * 4);
      int vlo[2], vhi[2];  // visible streamed columns [vlo, vhi] (relative to c0) of this thread's two rows
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int ri = r0 + row_l + 8 * r;  // sequence-local key (DKV) / query (DQ) index
        if constexpr (DKV) {  // row = key ri, column = query c0 + c
          vlo[r] = p.wr < 0 ? 0 : ri - sq.off - p.wr - c0;
          vhi[r] = p.wl < 0 ? SR - 1 : ri - sq.off + p.wl - c0;
        } else {              // row = query ri, column = key c0 + c
          vlo[r] = p.wl < 0 ? 0 : ri + sq.off - p.wl - c0;
          vhi[r] = min(sq.Sk - 1, p.wr < 0 ? sq.Sk - 1 : ri + sq.off + p.wr) - c0;
        }
      }
      // Only tiles on a mask edge test columns: in the others every column of this thread's rows is visible
      const bool edge = vlo[0] > 0 || vlo[1] > 0 || vhi[0] < SR - 1 || vhi[1] < SR - 1;
      wgmma_wait<1>();  // S
      wgmma_fence_regs(s);
      auto p_tile = [&](auto masked, auto cap) {
#pragma unroll
        for (int jj = 0; jj < SR / 8; ++jj) {
          float2 l2v = make_float2(0.f, 0.f);
          if constexpr (DKV) l2v = lds_f32x2(vec_addr + 8 * jj);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float pv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * jj + cq + e;
              const int i = 4 * jj + 2 * r + e;
              const float l2 = DKV ? (e ? l2v.y : l2v.x) : my_lse2[r];
              float x = s[i], dcap = 1.f;
              if constexpr (cap) {
                const float tcap = tanhf(x * cap_in);
                x = p.softcap * tcap * kLog2e - l2;
                dcap = 1.f - tcap * tcap;
              } else {
                // x * scale - lse with one rounding in every copy of the loop (given as a product and a difference,
                // the compiler may form the product once for all copies and round it separately)
                x = fmaf(x, scale_log2, -l2);
              }
              const bool vis = !masked || ((c >= vlo[r]) && (c <= vhi[r]));
              pv[e] = vis ? exp2f(x) : 0.f;
              s[i] = pv[e] * dcap;
            }
            pf[jj >> 1][2 * (jj & 1) + r] = pack_bf16x2(pv[0], pv[1]);  // = pack_a_frag(P, jj / 2)
          }
        }
      };
      // one copy of the loop per (mask edge, soft-cap) case: a branch on either inside it is taken per element
      if (capped) {
        if (edge) p_tile(std::true_type{}, std::true_type{});
        else p_tile(std::false_type{}, std::true_type{});
      } else {
        if (edge) p_tile(std::true_type{}, std::false_type{});
        else p_tile(std::false_type{}, std::false_type{});
      }
      if constexpr (DKV) {
        wgmma_fence_regs(acc1);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < SR / 16; ++ks) wgmma_bf16_rs<DV, 1>(acc1, pf[ks], desc_mnmajor(s2_addr, SR * 128, ks), 1);  // dV += P^T dO
        wgmma_commit();
      }
      wgmma_wait<DKV ? 1 : 0>();  // dP
      wgmma_fence_regs(dp);
      auto ds_tile = [&](auto masked) {
#pragma unroll
        for (int jj = 0; jj < SR / 8; ++jj) {
          float2 dlv = make_float2(0.f, 0.f);
          if constexpr (DKV) dlv = lds_f32x2(vec_addr + SR * 4 + 8 * jj);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float ds[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * jj + cq + e;
              const int i = 4 * jj + 2 * r + e;
              const float dl = DKV ? (e ? dlv.y : dlv.x) : my_delta[r];
              // dP may be NaN at masked columns (DQ: V rows past the end of the sequence), where dS must be exactly 0
              const bool vis = !masked || ((c >= vlo[r]) && (c <= vhi[r]));
              ds[e] = vis ? s[i] * (dp[i] - dl) : 0.f;
            }
            df[jj >> 1][2 * (jj & 1) + r] = pack_bf16x2(ds[0], ds[1]);
          }
        }
      };
      if (edge) ds_tile(std::true_type{});
      else ds_tile(std::false_type{});
      float(&acc_ds)[DQK / 2] = pick<DKV>(acc2, acc1);
      wgmma_fence_regs(acc_ds);
      wgmma_fence();
      // DKV: dK += dS^T Q.  DQ: dQ += dS K
#pragma unroll
      for (int ks = 0; ks < SR / 16; ++ks) wgmma_bf16_rs<DQK, 1>(acc_ds, df[ks], desc_mnmajor(s1_addr, SR * 128, ks), 1);
      wgmma_commit();
      wgmma_wait<0>();
      if (signal) mbar_arrive(&st_empty[st]);
    }
    wgmma_fence_regs(acc1);
    if constexpr (DKV) wgmma_fence_regs(acc2);
    // ---- epilogue: accumulators -> bf16 -> global.  DKV: dV, dK (scaled); DQ: dQ (scaled)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int ri = r0 + row_l + 8 * r;
      if (ri >= (DKV ? sq.Sk : sq.Sq)) continue;
      if constexpr (DKV) {
        __nv_bfloat16* dv = p.dv + (static_cast<long long>(sq.k_start + ri) * p.Hk + head) * DV + cq;
        __nv_bfloat16* dk = p.dk + (static_cast<long long>(sq.k_start + ri) * p.Hk + head) * DQK + cq;
#pragma unroll
        for (int jj = 0; jj < DQK / 8; ++jj) {
          if (jj < DV / 8)
            *reinterpret_cast<uint32_t*>(dv + 8 * jj) = pack_bf16x2(acc1[4 * jj + 2 * r], acc1[4 * jj + 2 * r + 1]);
          *reinterpret_cast<uint32_t*>(dk + 8 * jj) =
              pack_bf16x2(acc2[4 * jj + 2 * r] * p.scale, acc2[4 * jj + 2 * r + 1] * p.scale);
        }
      } else {
        __nv_bfloat16* dq = p.dq + (static_cast<long long>(sq.q_start + ri) * p.Hq + head) * DQK + cq;
#pragma unroll
        for (int jj = 0; jj < DQK / 8; ++jj)
          *reinterpret_cast<uint32_t*>(dq + 8 * jj) = pack_bf16x2(acc1[4 * jj + 2 * r] * p.scale, acc1[4 * jj + 2 * r + 1] * p.scale);
      }
    }
  }
  if (stuck) __trap();
}

// delta[b, h, q] = sum_d dO[q, h, d] * O[q, h, d] over the DV value columns   (DV/8 lanes per (row, head), 16-byte loads)
template <int DV>
__global__ void flash_attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout,
                                        float* __restrict__ delta, const int* __restrict__ cu_q, int B, int Sq, int Hq,
                                        long long total_rows, long long lse_bs, long long lse_hs) {
  constexpr int LANES = DV / 8;  // lanes cooperating on one (row, head)
  const long long gt = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long item = gt / LANES;
  const int sub = static_cast<int>(gt % LANES);
  const bool ok = item < total_rows * Hq;
  float acc = 0.f;
  if (ok) {
    const uint4 a = *reinterpret_cast<const uint4*>(o + item * DV + sub * 8), c = *reinterpret_cast<const uint4*>(dout + item * DV + sub * 8);
    const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y), a2 = unpack_bf16x2(a.z), a3 = unpack_bf16x2(a.w);
    const float2 c0 = unpack_bf16x2(c.x), c1 = unpack_bf16x2(c.y), c2 = unpack_bf16x2(c.z), c3 = unpack_bf16x2(c.w);
    acc = a0.x * c0.x + a0.y * c0.y + a1.x * c1.x + a1.y * c1.y + a2.x * c2.x + a2.y * c2.y + a3.x * c3.x + a3.y * c3.y;
  }
#pragma unroll
  for (int off = LANES / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (ok && sub == 0) {
    const long long r = item / Hq;
    const int h = static_cast<int>(item % Hq);
    long long idx;
    if (cu_q != nullptr) {
      idx = static_cast<long long>(h) * lse_hs + r;  // packed: [H, total]
    } else {
      const long long b = r / Sq, q = r % Sq;
      idx = b * lse_bs + static_cast<long long>(h) * lse_hs + q;
    }
    delta[idx] = acc;
  }
}

// Packed batches: rows outside every sequence (before cu[0] or from cu[B] on) belong to no kernel above.  Zero them in x0 /
// x1 ([rows, row_elems] bf16, either may be null) and set lse[h, row] = -inf (lse may be null), reading cu on the device.
__global__ void flash_attn_zero_outside_kernel(__nv_bfloat16* __restrict__ x0, __nv_bfloat16* __restrict__ x1, float* __restrict__ lse,
                                               const int* __restrict__ cu, int B, long long rows, int row_elems, int H) {
  const long long head = cu[0], tail_from = cu[B];
  const long long n_out = head + (rows - tail_from);
  const int chunks = row_elems / 8;  // 16-byte chunks per row
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_out * chunks; i += stride) {
    const long long k = i / chunks, row = k < head ? k : tail_from + (k - head);
    const long long off = row * row_elems + (i % chunks) * 8;
    if (x0 != nullptr) *reinterpret_cast<uint4*>(x0 + off) = make_uint4(0u, 0u, 0u, 0u);
    if (x1 != nullptr) *reinterpret_cast<uint4*>(x1 + off) = make_uint4(0u, 0u, 0u, 0u);
  }
  if (lse != nullptr)
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_out * H; i += stride) {
      const long long k = i / H, row = k < head ? k : tail_from + (k - head);
      lse[(i % H) * rows + row] = -INFINITY;
    }
}

void check_launch(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("d9d flash_attn: launch of ") + what + " failed: " + cudaGetErrorString(e));
}

void zero_outside(void* x0, void* x1, float* lse, const int* cu, int B, long long rows, int row_elems, int H, cudaStream_t stream) {
  flash_attn_zero_outside_kernel<<<128, 256, 0, stream>>>(static_cast<__nv_bfloat16*>(x0), static_cast<__nv_bfloat16*>(x1), lse, cu, B,
                                                          rows, row_elems, H);
  check_launch("the packed-batch padding pass");
}

// [rows, H, D] bf16 -> 3-D tensor map (d, h, row), box = 64 x 1 x box_rows, 128B swizzle
CUtensorMap make_tmap_rhd(const void* base, long long rows, int H, int D, int box_rows) {
  CUtensorMap m;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(D) * 2, static_cast<cuuint64_t>(H) * D * 2};
  cuuint32_t box[3] = {64, 1, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[3] = {1, 1, 1};
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) throw std::runtime_error("d9d flash_attn: tensors must be 16-byte aligned");
  CUresult r = gemm::get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("d9d flash_attn: cuTensorMapEncodeTiled failed: " + std::to_string(r));
  return m;
}

// (tiles of 128 rows) x H x B blocks, flattened as decode_block expects
unsigned grid_1d(int S, int H, int B) {
  const long long n = static_cast<long long>((S + 127) / 128) * H * B;
  if (n > 0x7fffffffLL) throw std::runtime_error("d9d flash_attn: more than 2^31 - 1 tiles in one launch");
  return static_cast<unsigned>(n);
}

FaParams make_params(const FlashAttnArgs& a) {
  FaParams p{};
  p.B = a.B; p.Sq = a.Sq; p.Sk = a.Sk; p.Hq = a.Hq; p.Hk = a.Hk;
  p.wl = a.window_left; p.wr = a.window_right;
  p.scale = a.scale; p.softcap = a.softcap;
  p.cu_q = a.cu_q; p.cu_k = a.cu_k;
  if (a.cu_q != nullptr) { p.lse_bs = 0; p.lse_hs = a.total_q; }
  else { p.lse_bs = static_cast<long long>(a.Hq) * a.Sq; p.lse_hs = a.Sq; }
  p.sink = a.sink;
  return p;
}

template <int DQK, int DV>
void launch_fwd(const FlashAttnArgs& a, cudaStream_t stream) {
  using C = FwdCfg<DQK, DV>;
  auto kern = flash_attn_fwd_kernel<DQK, DV>;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    configured = true;
  }
  const CUtensorMap tq = make_tmap_rhd(a.q, a.total_q, a.Hq, DQK, 128), tk = make_tmap_rhd(a.k, a.total_k, a.Hk, DQK, 128),
                    tv = make_tmap_rhd(a.v, a.total_k, a.Hk, DV, 128);
  FaParams p = make_params(a);
  p.out = static_cast<__nv_bfloat16*>(a.out);
  p.lse = a.lse;
  kern<<<grid_1d(a.Sq, a.Hq, a.B), FA_THREADS, C::SMEM_BYTES, stream>>>(tq, tk, tv, p);
  check_launch("the forward kernel");
}

template <int DV>
void launch_delta(const FlashAttnArgs& a, cudaStream_t stream) {
  const long long threads = a.total_q * a.Hq * (DV / 8);
  flash_attn_delta_kernel<DV><<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(a.out), static_cast<const __nv_bfloat16*>(a.dout), a.delta, a.cu_q, a.B, a.Sq, a.Hq,
      a.total_q, static_cast<long long>(a.Hq) * a.Sq, a.cu_q != nullptr ? a.total_q : a.Sq);
  check_launch("the delta kernel");
}

template <int DQK, int DV>
void launch_bwd(const FlashAttnArgs& a, cudaStream_t stream) {
  FaParams p = make_params(a);
  p.lse = a.lse;
  p.delta = a.delta;
  p.dq = static_cast<__nv_bfloat16*>(a.dq);
  p.dk = static_cast<__nv_bfloat16*>(a.dk);
  p.dv = static_cast<__nv_bfloat16*>(a.dv);
  if (a.Sk > 0) {
    using C = BwdCfg<DQK, DV, true>;
    auto kern = flash_attn_bwd_kernel<DQK, DV, true>;
    static bool configured = false;
    if (!configured) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
      configured = true;
    }
    const CUtensorMap tk = make_tmap_rhd(a.k, a.total_k, a.Hk, DQK, 128), tv = make_tmap_rhd(a.v, a.total_k, a.Hk, DV, 128),
                      tq = make_tmap_rhd(a.q, a.total_q, a.Hq, DQK, C::SR), tdo = make_tmap_rhd(a.dout, a.total_q, a.Hq, DV, C::SR);
    kern<<<grid_1d(a.Sk, a.Hk, a.B), FA_THREADS, C::SMEM_BYTES, stream>>>(tk, tv, tq, tdo, p);
    check_launch("the dK/dV kernel");
  }
  if (a.Sq > 0) {
    using C = BwdCfg<DQK, DV, false>;
    auto kern = flash_attn_bwd_kernel<DQK, DV, false>;
    static bool configured = false;
    if (!configured) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
      configured = true;
    }
    const CUtensorMap tq = make_tmap_rhd(a.q, a.total_q, a.Hq, DQK, 128), tdo = make_tmap_rhd(a.dout, a.total_q, a.Hq, DV, 128),
                      tk = make_tmap_rhd(a.k, a.total_k, a.Hk, DQK, C::SR), tv = make_tmap_rhd(a.v, a.total_k, a.Hk, DV, C::SR);
    kern<<<grid_1d(a.Sq, a.Hq, a.B), FA_THREADS, C::SMEM_BYTES, stream>>>(tq, tdo, tk, tv, p);
    check_launch("the dQ kernel");
  }
}

void check_args(const FlashAttnArgs& a) {
  if (a.Hq % a.Hk != 0) throw std::runtime_error("d9d flash_attn: Hq must be a multiple of Hk");
  const bool dims_ok = (a.Dqk == 64 && a.Dv == 64) || (a.Dqk == 128 && a.Dv == 128) || (a.Dqk == 192 && a.Dv == 128);
  if (!dims_ok)
    throw std::runtime_error("d9d flash_attn: (qk, v) head dims must be (64, 64), (128, 128) or (192, 128), got (" +
                             std::to_string(a.Dqk) + ", " + std::to_string(a.Dv) + ")");
  if ((a.cu_q == nullptr) != (a.cu_k == nullptr)) throw std::runtime_error("d9d flash_attn: cu_seqlens_q and cu_seqlens_k go together");
}

}  // namespace

void flash_attn_fwd(const FlashAttnArgs& a, cudaStream_t stream) {
  if (a.B == 0 || a.Hq == 0 || a.total_q == 0) return;
  check_args(a);
  if (a.cu_q != nullptr) zero_outside(a.out, nullptr, a.lse, a.cu_q, a.B, a.total_q, a.Hq * a.Dv, a.Hq, stream);
  if (a.Sq == 0) return;
  if (a.Dqk == 64) launch_fwd<64, 64>(a, stream);
  else if (a.Dqk == 128) launch_fwd<128, 128>(a, stream);
  else launch_fwd<192, 128>(a, stream);
}

void flash_attn_bwd_delta(const FlashAttnArgs& a, cudaStream_t stream) {
  if (a.B == 0 || a.Hq == 0 || a.total_q == 0) return;
  check_args(a);
  if (a.Dv == 64) launch_delta<64>(a, stream);
  else launch_delta<128>(a, stream);
}

void flash_attn_bwd(const FlashAttnArgs& a, cudaStream_t stream) {
  if (a.B == 0 || a.Hq == 0 || a.total_q == 0) return;
  check_args(a);
  if (a.total_k == 0) {  // no key anywhere: dq = 0
    if (cudaMemsetAsync(a.dq, 0, static_cast<size_t>(a.total_q) * a.Hq * a.Dqk * 2, stream) != cudaSuccess)
      throw std::runtime_error("d9d flash_attn: cudaMemsetAsync failed");
    return;
  }
  if (a.cu_q != nullptr) {
    zero_outside(a.dq, nullptr, nullptr, a.cu_q, a.B, a.total_q, a.Hq * a.Dqk, 0, stream);
    if (a.Dqk == a.Dv) {
      zero_outside(a.dk, a.dv, nullptr, a.cu_k, a.B, a.total_k, a.Hk * a.Dqk, 0, stream);
    } else {  // dk and dv rows differ in width
      zero_outside(a.dk, nullptr, nullptr, a.cu_k, a.B, a.total_k, a.Hk * a.Dqk, 0, stream);
      zero_outside(a.dv, nullptr, nullptr, a.cu_k, a.B, a.total_k, a.Hk * a.Dv, 0, stream);
    }
  }
  if (a.Dqk == 64) launch_bwd<64, 64>(a, stream);
  else if (a.Dqk == 128) launch_bwd<128, 128>(a, stream);
  else launch_bwd<192, 128>(a, stream);
}

}  // namespace d9d
