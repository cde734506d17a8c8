// Dense wgmma GEMM instantiations (forward NT, dgrad NN-as-MN-major-B, wgrad TN-as-MN/MN).
#include <cstdlib>

#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

namespace {
int& pair_mode_ref() {
  static int mode = [] {
    // CTA pairs (B tile multicast over a two-CTA cluster) are the default for eligible shapes;
    // D9D_GEMM_PAIR=0 restores the single-CTA kernels everywhere
    const char* e = std::getenv("D9D_GEMM_PAIR");
    return (e != nullptr && e[0] == '0') ? 0 : 1;
  }();
  return mode;
}
}  // namespace

int gemm_set_pair_mode(int mode) {
  const int prev = pair_mode_ref();
  pair_mode_ref() = mode ? 1 : 0;
  return prev;
}
int gemm_pair_mode() { return pair_mode_ref(); }

// CTA pairs pay off once there are enough 256-row tiles to fill the 66 SM pairs; tiny problems keep the single-CTA kernels
bool gemm_pair_eligible(const GemmArgs& a) { return a.M >= 512 && a.N >= 128 && a.comm == COMM_NONE; }

void gemm_dense(const GemmArgs& a, cudaStream_t stream) {
  // MN-major A with K-major B has store epilogues only, whichever kernel (single CTA or pair) the shape would pick
  if (a.a_mn && !a.b_mn && (a.epi == EPI_F32_ACC || a.epi == EPI_BF16_ACC))
    throw std::runtime_error("d9d gemm: accumulate epilogue not built for an MN-major A with a K-major B");
  if (a.M <= 0 || a.N <= 0) return;
  if (a.ctas == 2 || (a.ctas == 0 && gemm_pair_mode() == 1 && gemm_pair_eligible(a))) {
    gemm_dense_pair(a, stream);
    return;
  }
  const long long m_tiles = (a.M + BLOCK_M - 1) / BLOCK_M;
  const int bn = a.block_n ? a.block_n : pick_block_n(m_tiles, a.N);
  if (!a.a_mn && !a.b_mn) {
    D9D_DISPATCH_EPI4(DENSE, false, false, a.epi, bn, a, stream);
  } else if (!a.a_mn && a.b_mn) {
    D9D_DISPATCH_EPI4(DENSE, false, true, a.epi, bn, a, stream);  // accumulate: chunked dE of the fused linear-CE
  } else if (a.a_mn && a.b_mn) {
    D9D_DISPATCH_EPI4(DENSE, true, true, a.epi, bn, a, stream);
  } else {
    D9D_DISPATCH_EPI2(DENSE, true, false, a.epi, bn, a, stream);
  }
}
}  // namespace d9d
