// Grouped wgmma GEMM instantiations for MoE experts:
//   GROUPED_M: Y[r,:] = X[r,:] · W[e(r)]      (forward: B MN-major [E,K,N]; dgrad: B K-major [E,N',K'])
//   GROUPED_K: dW[e]  = X_e^T · dY_e          (both operands MN-major, reduction over the expert's rows)
#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

void gemm_grouped(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0) return;
  const long long m_tiles = (a.M + BLOCK_M - 1) / BLOCK_M;
  if (a.mode == GROUPED_M) {
    const int bn = a.block_n ? a.block_n : pick_block_n(m_tiles, a.N);
    if (a.a_mn) throw std::runtime_error("d9d gemm: GROUPED_M requires K-major A");
    if (a.epi == EPI_BF16_ACC) {
      // D += X W^T (second dgrad of a pair of projections sharing the input: gate / up) - K-major B only
      if (a.b_mn) throw std::runtime_error("d9d gemm: GROUPED_M accumulate is built for K-major B (dgrad) only");
      D9D_DISPATCH_BN(GROUPED_M, false, false, EPI_BF16_ACC, bn, a, stream);
    } else {
      if (a.epi != EPI_BF16) throw std::runtime_error("d9d gemm: GROUPED_M supports bf16 store / accumulate only");
      if (a.b_mn) D9D_DISPATCH_BN(GROUPED_M, false, true, EPI_BF16, bn, a, stream);
      else        D9D_DISPATCH_BN(GROUPED_M, false, false, EPI_BF16, bn, a, stream);
    }
  } else if (a.mode == GROUPED_K) {
    const int bn = a.block_n ? a.block_n : pick_block_n(m_tiles * a.num_groups, a.N);
    if (!a.a_mn || !a.b_mn) throw std::runtime_error("d9d gemm: GROUPED_K requires MN-major A and B");
    D9D_DISPATCH_EPI4(GROUPED_K, true, true, a.epi, bn, a, stream);
  } else {
    throw std::runtime_error("d9d gemm: bad grouped mode");
  }
}
}  // namespace d9d
