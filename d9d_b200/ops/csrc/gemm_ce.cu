// Fused linear + cross-entropy on the wgmma GEMM (no [T, V] logits tensor in the forward pass).
//   forward : logits tile -> per-(row, n_tile) online-softmax partials + target logit  (EPI_CE_LSE)
//   finalize: partials -> lse[row], nll[row]
//   backward: recompute logits tile, write g*(softmax - onehot) as bf16 chunk          (EPI_CE_DLOGITS)
// The regularised loss (label smoothing, z-loss) has its own instances: EPI_CE_LSE_SUM also writes per-tile logit sums,
// EPI_CE_DLOGITS_REG writes the regularised gradient.  The plain instances are the same code as without them.
#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

constexpr int CE_BN = 256;
int gemm_ce_block_n() { return CE_BN; }

void gemm_ce(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0) return;
  if (a.a_mn || a.b_mn) throw std::runtime_error("d9d gemm_ce: K-major operands required");
  const bool pair = a.ctas == 2 || (a.ctas == 0 && gemm_pair_mode() == 1 && gemm_pair_eligible(a));
  if (a.epi == EPI_CE_LSE) {
    if (pair) launch_one<DENSE, CE_BN, false, false, EPI_CE_LSE, COMM_NONE, 2>(a, stream);
    else launch_one<DENSE, CE_BN, false, false, EPI_CE_LSE>(a, stream);
  } else if (a.epi == EPI_CE_DLOGITS) {
    if (pair) launch_one<DENSE, CE_BN, false, false, EPI_CE_DLOGITS, COMM_NONE, 2>(a, stream);
    else launch_one<DENSE, CE_BN, false, false, EPI_CE_DLOGITS>(a, stream);
  } else if (a.epi == EPI_CE_LSE_SUM) {
    if (pair) launch_one<DENSE, CE_BN, false, false, EPI_CE_LSE_SUM, COMM_NONE, 2>(a, stream);
    else launch_one<DENSE, CE_BN, false, false, EPI_CE_LSE_SUM>(a, stream);
  } else if (a.epi == EPI_CE_DLOGITS_REG) {
    if (pair) launch_one<DENSE, CE_BN, false, false, EPI_CE_DLOGITS_REG, COMM_NONE, 2>(a, stream);
    else launch_one<DENSE, CE_BN, false, false, EPI_CE_DLOGITS_REG>(a, stream);
  } else {
    throw std::runtime_error("d9d gemm_ce: bad epilogue");
  }
}

__device__ __forceinline__ void ce_finalize_row(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                                                const float* __restrict__ tgt_logit, const long long* __restrict__ target,
                                                long long ignore_index, int n_tiles, int M, int row,
                                                float* __restrict__ lse, float* __restrict__ nll) {
  float mx = -INFINITY;
  for (int t = 0; t < n_tiles; ++t) mx = fmaxf(mx, part_max[static_cast<long long>(t) * M + row]);
  float s = 0.f;
  for (int t = 0; t < n_tiles; ++t) {
    const float pm = part_max[static_cast<long long>(t) * M + row];
    if (pm > -INFINITY) s += part_sum[static_cast<long long>(t) * M + row] * __expf(pm - mx);
  }
  const float l = mx + __logf(s);
  lse[row] = l;
  const long long tg = target[row];
  nll[row] = (tg == ignore_index) ? 0.f : (l - tgt_logit[row]);
}

__global__ void ce_finalize_kernel(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                                   const float* __restrict__ tgt_logit, const long long* __restrict__ target,
                                   long long ignore_index, int n_tiles, int M, float* __restrict__ lse,
                                   float* __restrict__ nll) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= M) return;
  ce_finalize_row(part_max, part_sum, tgt_logit, target, ignore_index, n_tiles, M, row, lse, nll);
}

// ce_finalize_kernel + the row's logit sum, accumulated over the tiles in order (deterministic, no atomics)
__global__ void ce_finalize_zsum_kernel(const float* __restrict__ part_max, const float* __restrict__ part_sum,
                                        const float* __restrict__ part_zsum, const float* __restrict__ tgt_logit,
                                        const long long* __restrict__ target, long long ignore_index, int n_tiles, int M,
                                        float* __restrict__ lse, float* __restrict__ nll, float* __restrict__ zsum) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= M) return;
  ce_finalize_row(part_max, part_sum, tgt_logit, target, ignore_index, n_tiles, M, row, lse, nll);
  float s = 0.f;
  for (int t = 0; t < n_tiles; ++t) s += part_zsum[static_cast<long long>(t) * M + row];
  zsum[row] = s;
}

void ce_finalize(const float* part_max, const float* part_sum, const float* tgt_logit, const long long* target,
                 long long ignore_index, int n_tiles, int M, float* lse, float* nll, cudaStream_t stream) {
  if (M <= 0) return;
  ce_finalize_kernel<<<(M + 255) / 256, 256, 0, stream>>>(part_max, part_sum, tgt_logit, target, ignore_index,
                                                          n_tiles, M, lse, nll);
}

void ce_finalize_zsum(const float* part_max, const float* part_sum, const float* part_zsum, const float* tgt_logit,
                      const long long* target, long long ignore_index, int n_tiles, int M, float* lse, float* nll,
                      float* zsum, cudaStream_t stream) {
  if (M <= 0) return;
  ce_finalize_zsum_kernel<<<(M + 255) / 256, 256, 0, stream>>>(part_max, part_sum, part_zsum, tgt_logit, target,
                                                               ignore_index, n_tiles, M, lse, nll, zsum);
}
}  // namespace d9d
