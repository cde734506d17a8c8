// Dense wgmma GEMM on CTA pairs: 256 x {256, 128} tiles, one cluster of two CTAs per tile.
// Every CTA stages its own 128 rows of A and loads half of the B tile, multicast into both CTAs.
#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

void gemm_dense_pair(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0) return;
  if (a.comm != COMM_NONE) throw std::runtime_error("d9d gemm: CTA-pair kernels do not implement fused communication");
  // 256-wide tiles unless the problem is narrow or the narrower tile wastes fewer columns of the last n-tile
  int bn = a.block_n ? a.block_n : 256;
  if (a.block_n == 0) {
    const long long w256 = (a.N + 255) / 256 * 256, w128 = (a.N + 127) / 128 * 128;
    if (w128 < w256) bn = 128;
  }
  if (!a.a_mn && !a.b_mn) {
    D9D_DISPATCH_PAIR_EPI4(false, false, a.epi, bn, a, stream);
  } else if (!a.a_mn && a.b_mn) {
    D9D_DISPATCH_PAIR_EPI4(false, true, a.epi, bn, a, stream);
  } else if (a.a_mn && a.b_mn) {
    D9D_DISPATCH_PAIR_EPI4(true, true, a.epi, bn, a, stream);
  } else {
    D9D_DISPATCH_PAIR_EPI4(true, false, a.epi, bn, a, stream);
  }
}
}  // namespace d9d
