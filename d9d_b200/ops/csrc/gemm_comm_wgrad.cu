// Weight gradients of sequence-parallel tensor-parallel layers: one MN-major operand is sharded along the reduction
// (token) dim over the peers and is TMA-loaded k-block by k-block from its owners (COMM_AG_KA / COMM_AG_KB).
#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

template <int COMM>
static void dispatch_epi(const GemmArgs& a, int bn, cudaStream_t stream) {
#define D9D_COMM_W(EPI)                                                       \
  do {                                                                        \
    if (bn == 256) launch_one<DENSE, 256, true, true, EPI, COMM>(a, stream);  \
    else launch_one<DENSE, 128, true, true, EPI, COMM>(a, stream);            \
  } while (0)
  if (bn != 128 && bn != 256) throw std::runtime_error("d9d gemm_comm: BLOCK_N must be 128 or 256");
  switch (a.epi) {
    case EPI_F32_ACC: D9D_COMM_W(EPI_F32_ACC); break;
    case EPI_F32: D9D_COMM_W(EPI_F32); break;
    case EPI_BF16: D9D_COMM_W(EPI_BF16); break;
    default: throw std::runtime_error("d9d gemm_comm: unsupported wgrad epilogue");
  }
#undef D9D_COMM_W
}

void gemm_comm_wgrad(const GemmArgs& a, cudaStream_t stream) {
  if (!a.a_mn || !a.b_mn) throw std::runtime_error("d9d gemm_comm: wgrad needs MN-major operands");
  const long long m_tiles = (a.M + BLOCK_M - 1) / BLOCK_M;
  int bn = a.block_n;
  if (bn == 0) {
    bn = pick_block_n(m_tiles, a.N);
    if (bn == 192) bn = 256;
  }
  if (a.comm == COMM_AG_KA) dispatch_epi<COMM_AG_KA>(a, bn, stream);
  else dispatch_epi<COMM_AG_KB>(a, bn, stream);
}
}  // namespace d9d
