// Tensor-parallel GEMMs with the collective fused in (activations side):
//   all-gather -> GEMM      (COMM_AG_A: A tiles TMA-loaded from the owning peer's shard over NVLink)
//   GEMM -> reduce-scatter  (COMM_RS_D: output tiles TMA reduce-added into the owning peer's shard)
#include "gemm_host.cuh"

namespace d9d {
using namespace gemm;

void gemm_comm_wgrad(const GemmArgs& a, cudaStream_t stream);

template <int COMM, int EPI>
static void dispatch_layout(const GemmArgs& a, int bn, cudaStream_t stream) {
  if (a.a_mn) throw std::runtime_error("d9d gemm_comm: K-major A required");
  if (bn != 128 && bn != 256) throw std::runtime_error("d9d gemm_comm: BLOCK_N must be 128 or 256");
  if (!a.b_mn) {
    if (bn == 256) launch_one<DENSE, 256, false, false, EPI, COMM>(a, stream);
    else launch_one<DENSE, 128, false, false, EPI, COMM>(a, stream);
  } else {
    if (bn == 256) launch_one<DENSE, 256, false, true, EPI, COMM>(a, stream);
    else launch_one<DENSE, 128, false, true, EPI, COMM>(a, stream);
  }
}

void gemm_comm(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0) return;
  const long long m_tiles = (a.M + BLOCK_M - 1) / BLOCK_M;
  int bn = a.block_n;
  if (bn == 0) {
    bn = pick_block_n(m_tiles, a.N);
    if (bn == 192) bn = 256;  // the fused-communication GEMMs are built for 128- and 256-wide tiles only
  }
  switch (a.comm) {
    case COMM_AG_A:
      if (a.epi != EPI_BF16) throw std::runtime_error("d9d gemm_comm: all-gather GEMM stores bf16");
      dispatch_layout<COMM_AG_A, EPI_BF16>(a, bn, stream);
      break;
    case COMM_WAIT_A:
      if (a.epi != EPI_BF16) throw std::runtime_error("d9d gemm_comm: all-gather GEMM stores bf16");
      dispatch_layout<COMM_WAIT_A, EPI_BF16>(a, bn, stream);
      break;
    case COMM_RS_D:
      if (a.epi != EPI_BF16_ACC) throw std::runtime_error("d9d gemm_comm: reduce-scatter GEMM reduce-adds bf16");
      dispatch_layout<COMM_RS_D, EPI_BF16_ACC>(a, bn, stream);
      break;
    case COMM_AG_KA:
    case COMM_AG_KB:
      gemm_comm_wgrad(a, stream);
      break;
    default:
      throw std::runtime_error("d9d gemm_comm: unknown communication mode");
  }
}
}  // namespace d9d
