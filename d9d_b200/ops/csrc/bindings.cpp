// d9d_b200 — torch bindings (TORCH_LIBRARY) for the native sm_90a kernels.
// Compiled with the host compiler only; the kernels live in *.cu translation units that do not include torch.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <cmath>
#include <tuple>
#include <vector>

#include "d9d_ops.h"

using namespace d9d::gemm;  // the GEMM launch codes: Mode, Epi, Comm

namespace {

using at::Tensor;

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

inline d9d::DType dtype_code(const Tensor& t) {
  if (t.scalar_type() == at::kBFloat16) return d9d::DTYPE_BF16;
  if (t.scalar_type() == at::kFloat) return d9d::DTYPE_F32;
  if (t.scalar_type() == at::kHalf) return d9d::DTYPE_F16;
  TORCH_CHECK(false, "d9d_b200: unsupported dtype ", t.scalar_type());
}

#define CHECK_CUDA_CONTIG(t) TORCH_CHECK((t).is_cuda() && (t).is_contiguous(), #t " must be a contiguous CUDA tensor")
// Operands the kernels load or store 16 bytes at a time (uint4 / float4). A contiguous view at an element offset keeps
// is_contiguous() but not the alignment, so it is refused here rather than reaching a misaligned vector access.
#define CHECK_ALIGNED16(t) \
  TORCH_CHECK(reinterpret_cast<uintptr_t>((t).data_ptr()) % 16 == 0, #t " must start on a 16-byte boundary")

// ------------------------------------------------------------------ GEMM ------------------------
Epi epi_for(const Tensor& d, bool accumulate) {
  if (d.scalar_type() == at::kBFloat16) return accumulate ? EPI_BF16_ACC : EPI_BF16;
  TORCH_CHECK(d.scalar_type() == at::kFloat, "gemm output must be bf16 or fp32");
  return accumulate ? EPI_F32_ACC : EPI_F32;
}

// block_n: output tile width (0 = the heuristic's choice). Single-CTA dense and grouped kernels are built for 128, 192 and
// 256; CTA pairs and the fused-communication GEMMs for 128 and 256. Unknown values are rejected, never remapped.
void check_block_n(int64_t block_n, bool allow_192, const std::string& op) {
  if (block_n == 0 || block_n == 128 || block_n == 256 || (allow_192 && block_n == 192)) return;
  throw std::runtime_error(op + ": block_n must be 0, 128, " + (allow_192 ? "192 " : "") + "or 256, got " +
                           std::to_string(block_n));
}

// d[M,N] (+)= op(a) · op(b)^T.  a: [M,K] or (a_mn) [K,M];  b: [N,K] or (b_mn) [K,N].  Row strides may be padded.
// ctas: 1 = single CTA, 2 = CTA pair, 0 = process-wide policy.  k_splits (fp32 accumulate only): number of K slices, 0 = heuristic.
void gemm(const Tensor& a, const Tensor& b, Tensor d, bool a_mn, bool b_mn, bool accumulate, int64_t ctas, int64_t block_n,
          int64_t k_splits) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && d.is_cuda(), "gemm: CUDA tensors required");
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm: bf16 operands required");
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && d.dim() == 2, "gemm: 2-D tensors required");
  TORCH_CHECK(a.stride(1) == 1 && b.stride(1) == 1 && d.stride(1) == 1, "gemm: innermost stride must be 1");
  c10::cuda::CUDAGuard guard(a.device());
  d9d::GemmArgs g;
  g.mode = DENSE;
  g.a_mn = a_mn; g.b_mn = b_mn;
  g.M = static_cast<int>(a_mn ? a.size(1) : a.size(0));
  g.K = static_cast<int>(a_mn ? a.size(0) : a.size(1));
  g.N = static_cast<int>(b_mn ? b.size(1) : b.size(0));
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == g.K, "gemm: K mismatch");
  TORCH_CHECK(d.size(0) == g.M && d.size(1) == g.N, "gemm: output shape mismatch");
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.epi = epi_for(d, accumulate);
  TORCH_CHECK(ctas >= 0 && ctas <= 2, "gemm: ctas must be 0, 1 or 2");
  g.ctas = static_cast<int>(ctas);
  const bool pair = ctas == 2 || (ctas == 0 && d9d::gemm_pair_mode() == 1 && d9d::gemm_pair_eligible(g));
  check_block_n(block_n, !pair, pair ? "gemm (CTA pair)" : "gemm");
  TORCH_CHECK(k_splits >= 0, "gemm: k_splits must be >= 0");
  TORCH_CHECK(k_splits <= 1 || g.epi == EPI_F32_ACC, "gemm: k_splits needs an fp32 output with accumulate=True");
  g.block_n = static_cast<int>(block_n);
  g.k_splits = static_cast<int>(k_splits);
  d9d::gemm_dense(g, cur_stream());
}

int64_t gemm_set_pair_mode(int64_t mode) { return d9d::gemm_set_pair_mode(static_cast<int>(mode)); }

// d[R,N] = a[R,K] · W[e(r)];  b: [E,N,K] (b_mn=false) or [E,K,N] (b_mn=true)
void gemm_grouped_m(const Tensor& a, const Tensor& b, Tensor d, const Tensor& tile_group, bool b_mn, bool accumulate,
                    int64_t block_n) {
  CHECK_CUDA_CONTIG(a); CHECK_CUDA_CONTIG(b); CHECK_CUDA_CONTIG(d); CHECK_CUDA_CONTIG(tile_group);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16 && d.scalar_type() == at::kBFloat16);
  TORCH_CHECK(tile_group.scalar_type() == at::kInt && a.size(0) % 128 == 0 && tile_group.numel() == a.size(0) / 128);
  c10::cuda::CUDAGuard guard(a.device());
  d9d::GemmArgs g;
  g.mode = GROUPED_M; g.epi = accumulate ? EPI_BF16_ACC : EPI_BF16; g.a_mn = false; g.b_mn = b_mn;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1));
  g.N = static_cast<int>(b_mn ? b.size(2) : b.size(1));
  TORCH_CHECK((b_mn ? b.size(1) : b.size(2)) == g.K, "gemm_grouped_m: K mismatch");
  TORCH_CHECK(d.size(0) == g.M && d.size(1) == g.N);
  g.num_groups = static_cast<int>(b.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(1); g.ldd = d.stride(0);
  g.b_group_stride = b.stride(0);
  g.tile_group = tile_group.data_ptr<int>();
  check_block_n(block_n, true, "gemm_grouped_m");
  g.block_n = static_cast<int>(block_n);
  d9d::gemm_grouped(g, cur_stream());
}

// d[E,M,N] (+)= a[rows_e, M]^T · b[rows_e, N] over each expert's row range group_offsets[e]..[e+1]
void gemm_grouped_k(const Tensor& a, const Tensor& b, Tensor d, const Tensor& group_offsets, bool accumulate, int64_t block_n) {
  CHECK_CUDA_CONTIG(a); CHECK_CUDA_CONTIG(b); CHECK_CUDA_CONTIG(d); CHECK_CUDA_CONTIG(group_offsets);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16);
  TORCH_CHECK(group_offsets.scalar_type() == at::kInt && a.size(0) == b.size(0));
  c10::cuda::CUDAGuard guard(a.device());
  d9d::GemmArgs g;
  g.mode = GROUPED_K; g.a_mn = true; g.b_mn = true;
  g.M = static_cast<int>(a.size(1)); g.N = static_cast<int>(b.size(1)); g.K = 0;
  g.k_total = a.size(0);
  g.num_groups = static_cast<int>(d.size(0));
  TORCH_CHECK(group_offsets.numel() == g.num_groups + 1 && d.size(1) == g.M && d.size(2) == g.N);
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(1); g.d_group_stride = d.stride(0);
  g.group_offsets = group_offsets.data_ptr<int>();
  g.epi = epi_for(d, accumulate);
  check_block_n(block_n, true, "gemm_grouped_k");
  g.block_n = static_cast<int>(block_n);
  d9d::gemm_grouped(g, cur_stream());
}

// fused linear-CE forward over a row slice w = C[col_offset : col_offset + V] of the classifier:
// returns (nll[T], lse[T], tgt_logit[T]) fp32; tgt_logit is 0 where the target lies outside the slice (nll is then lse)
std::tuple<Tensor, Tensor, Tensor> ce_forward_ex(const Tensor& h, const Tensor& w, const Tensor& target, int64_t ignore_index,
                                                 const c10::optional<Tensor>& bias, double softcap, int64_t col_offset) {
  CHECK_CUDA_CONTIG(h); CHECK_CUDA_CONTIG(w); CHECK_CUDA_CONTIG(target);
  TORCH_CHECK(h.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && target.scalar_type() == at::kLong);
  c10::cuda::CUDAGuard guard(h.device());
  const int T = static_cast<int>(h.size(0)), K = static_cast<int>(h.size(1)), V = static_cast<int>(w.size(0));
  TORCH_CHECK(w.size(1) == K && target.numel() == T);
  const int bn = d9d::gemm_ce_block_n();
  const int n_tiles = (V + bn - 1) / bn;
  auto fopt = h.options().dtype(at::kFloat);
  Tensor part_max = at::empty({n_tiles, T}, fopt), part_sum = at::empty({n_tiles, T}, fopt);
  Tensor tgt_logit = at::zeros({T}, fopt), lse = at::empty({T}, fopt), nll = at::empty({T}, fopt);
  d9d::GemmArgs g;
  g.mode = DENSE; g.epi = EPI_CE_LSE;
  g.M = T; g.N = V; g.K = K;
  g.A = h.data_ptr(); g.B = w.data_ptr(); g.lda = K; g.ldb = K; g.ldd = V;
  g.ce_target = reinterpret_cast<const long long*>(target.data_ptr<int64_t>());
  g.ce_part_max = part_max.data_ptr<float>(); g.ce_part_sum = part_sum.data_ptr<float>();
  g.ce_tgt_logit = tgt_logit.data_ptr<float>();
  g.ce_ignore_index = ignore_index;
  g.ce_softcap = static_cast<float>(softcap);
  g.ce_col_offset = col_offset;
  if (bias.has_value()) {
    CHECK_CUDA_CONTIG(*bias);
    TORCH_CHECK(bias->scalar_type() == at::kFloat && bias->numel() == V, "ce: bias must be fp32 [V]");
    g.ce_bias = bias->data_ptr<float>();
  }
  d9d::gemm_ce(g, cur_stream());
  d9d::ce_finalize(part_max.data_ptr<float>(), part_sum.data_ptr<float>(), tgt_logit.data_ptr<float>(),
                   reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), ignore_index, n_tiles, T,
                   lse.data_ptr<float>(), nll.data_ptr<float>(), cur_stream());
  return {nll, lse, tgt_logit};
}

// Operand checks of the regularised linear-CE ops, before anything touches the device
void check_ce_reg_operands(const char* op, const Tensor& h, const Tensor& w, const Tensor& target,
                           const c10::optional<Tensor>& bias, double softcap, int64_t col_offset) {
  CHECK_CUDA_CONTIG(h); CHECK_CUDA_CONTIG(w); CHECK_CUDA_CONTIG(target);
  TORCH_CHECK(h.dim() == 2 && w.dim() == 2 && target.dim() == 1, op, ": h [T, K], w [V, K] and target [T] expected");
  TORCH_CHECK(h.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16, op, ": h and w must be bf16");
  TORCH_CHECK(target.scalar_type() == at::kLong, op, ": target must be int64");
  TORCH_CHECK(w.device() == h.device() && target.device() == h.device(), op, ": operands must be on one device");
  TORCH_CHECK(w.size(1) == h.size(1) && target.numel() == h.size(0), op, ": shape mismatch");
  TORCH_CHECK(h.size(1) % 8 == 0 && h.size(1) > 0, op, ": the hidden size must be a positive multiple of 8");
  TORCH_CHECK(h.size(0) < (int64_t(1) << 31) && w.size(0) < (int64_t(1) << 31), op, ": too many rows");
  CHECK_ALIGNED16(h); CHECK_ALIGNED16(w);
  TORCH_CHECK(std::isfinite(softcap) && softcap >= 0.0, op, ": softcap must be finite and >= 0");
  TORCH_CHECK(col_offset >= 0, op, ": col_offset must be >= 0");
  if (bias.has_value()) {
    CHECK_CUDA_CONTIG(*bias);
    TORCH_CHECK(bias->device() == h.device() && bias->scalar_type() == at::kFloat && bias->numel() == w.size(0),
                op, ": bias must be fp32 [V]");
  }
}

// regularised linear-CE forward over a row slice w = C[col_offset : col_offset + V] of the classifier: ce_forward_ex's
// (nll[T], lse[T], tgt_logit[T]) plus zsum[T], the sum of the row's logits over the slice (after bias and soft-cap)
std::tuple<Tensor, Tensor, Tensor, Tensor> ce_forward_reg(const Tensor& h, const Tensor& w, const Tensor& target,
                                                          int64_t ignore_index, const c10::optional<Tensor>& bias,
                                                          double softcap, int64_t col_offset) {
  check_ce_reg_operands("ce_forward_reg", h, w, target, bias, softcap, col_offset);
  c10::cuda::CUDAGuard guard(h.device());
  const int T = static_cast<int>(h.size(0)), K = static_cast<int>(h.size(1)), V = static_cast<int>(w.size(0));
  const int bn = d9d::gemm_ce_block_n();
  const int n_tiles = (V + bn - 1) / bn;
  auto fopt = h.options().dtype(at::kFloat);
  Tensor part_max = at::empty({n_tiles, T}, fopt), part_sum = at::empty({n_tiles, T}, fopt);
  Tensor part_zsum = at::empty({n_tiles, T}, fopt);
  Tensor tgt_logit = at::zeros({T}, fopt), lse = at::empty({T}, fopt), nll = at::empty({T}, fopt);
  Tensor zsum = at::empty({T}, fopt);
  d9d::GemmArgs g;
  g.mode = DENSE; g.epi = EPI_CE_LSE_SUM;
  g.M = T; g.N = V; g.K = K;
  g.A = h.data_ptr(); g.B = w.data_ptr(); g.lda = K; g.ldb = K; g.ldd = V;
  g.ce_target = reinterpret_cast<const long long*>(target.data_ptr<int64_t>());
  g.ce_part_max = part_max.data_ptr<float>(); g.ce_part_sum = part_sum.data_ptr<float>();
  g.ce_part_zsum = part_zsum.data_ptr<float>();
  g.ce_tgt_logit = tgt_logit.data_ptr<float>();
  g.ce_ignore_index = ignore_index;
  g.ce_softcap = static_cast<float>(softcap);
  g.ce_col_offset = col_offset;
  if (bias.has_value()) g.ce_bias = bias->data_ptr<float>();
  d9d::gemm_ce(g, cur_stream());
  d9d::ce_finalize_zsum(part_max.data_ptr<float>(), part_sum.data_ptr<float>(), part_zsum.data_ptr<float>(),
                        tgt_logit.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                        ignore_index, n_tiles, T, lse.data_ptr<float>(), nll.data_ptr<float>(), zsum.data_ptr<float>(),
                        cur_stream());
  return {nll, lse, tgt_logit, zsum};
}

// fused linear-CE forward: returns (nll[T] fp32, lse[T] fp32)
std::tuple<Tensor, Tensor> ce_forward(const Tensor& h, const Tensor& w, const Tensor& target, int64_t ignore_index) {
  auto r = ce_forward_ex(h, w, target, ignore_index, c10::nullopt, 0.0, 0);
  return {std::get<0>(r), std::get<1>(r)};
}

// fused linear-CE backward, one chunk: out[T, V] (bf16) = grad[t] * d nll[t] / d logits[t, col_offset : col_offset + V]
// (w is the matching row slice of the classifier; lse is the log-sum-exp over the WHOLE vocabulary)
void ce_dlogits(const Tensor& h, const Tensor& w, const Tensor& target, const Tensor& lse, const Tensor& grad,
                Tensor out, int64_t ignore_index, const c10::optional<Tensor>& bias, double softcap, int64_t col_offset) {
  CHECK_CUDA_CONTIG(h); CHECK_CUDA_CONTIG(w); CHECK_CUDA_CONTIG(target); CHECK_CUDA_CONTIG(lse);
  CHECK_CUDA_CONTIG(grad);
  TORCH_CHECK(out.is_cuda() && out.dim() == 2 && out.stride(1) == 1, "ce_dlogits: out must be row-major (row pitch may be padded)");
  TORCH_CHECK(out.scalar_type() == at::kBFloat16 && lse.scalar_type() == at::kFloat && grad.scalar_type() == at::kFloat);
  c10::cuda::CUDAGuard guard(h.device());
  const int T = static_cast<int>(h.size(0)), K = static_cast<int>(h.size(1)), V = static_cast<int>(w.size(0));
  TORCH_CHECK(out.size(0) == T && out.size(1) == V);
  d9d::GemmArgs g;
  g.mode = DENSE; g.epi = EPI_CE_DLOGITS;
  g.M = T; g.N = V; g.K = K;
  g.A = h.data_ptr(); g.B = w.data_ptr(); g.D = out.data_ptr(); g.lda = K; g.ldb = K; g.ldd = out.stride(0);
  g.ce_target = reinterpret_cast<const long long*>(target.data_ptr<int64_t>());
  g.ce_lse = lse.data_ptr<float>(); g.ce_grad = grad.data_ptr<float>();
  g.ce_ignore_index = ignore_index;
  g.ce_softcap = static_cast<float>(softcap);
  g.ce_col_offset = col_offset;
  if (bias.has_value()) {
    CHECK_CUDA_CONTIG(*bias);
    TORCH_CHECK(bias->scalar_type() == at::kFloat && bias->numel() == V, "ce: bias must be fp32 [V]");
    g.ce_bias = bias->data_ptr<float>();
  }
  d9d::gemm_ce(g, cur_stream());
}

// regularised linear-CE backward, one chunk: out[T, V] (bf16) = grad[t] * d loss[t] / d logits[t, col_offset : col_offset + V]
// with loss = (1 - eps) (lse - z_y) + eps (lse - sum_j z_j / num_classes) + zeta lse^2, i.e.
// grad[t] * ((1 + 2 zeta lse) softmax - (1 - eps) onehot - eps / num_classes) * dz/dacc  (lse over the WHOLE vocabulary)
void ce_dlogits_reg(const Tensor& h, const Tensor& w, const Tensor& target, const Tensor& lse, const Tensor& grad, Tensor out,
                    int64_t ignore_index, double z_loss_coef, double label_smoothing, int64_t num_classes,
                    const c10::optional<Tensor>& bias, double softcap, int64_t col_offset) {
  check_ce_reg_operands("ce_dlogits_reg", h, w, target, bias, softcap, col_offset);
  CHECK_CUDA_CONTIG(lse); CHECK_CUDA_CONTIG(grad);
  TORCH_CHECK(lse.scalar_type() == at::kFloat && grad.scalar_type() == at::kFloat, "ce_dlogits_reg: lse and grad must be fp32");
  TORCH_CHECK(lse.device() == h.device() && grad.device() == h.device() && out.device() == h.device(),
              "ce_dlogits_reg: operands must be on one device");
  TORCH_CHECK(lse.numel() == h.size(0) && grad.numel() == h.size(0), "ce_dlogits_reg: lse and grad must be [T]");
  TORCH_CHECK(out.is_cuda() && out.dim() == 2 && out.stride(1) == 1 && out.scalar_type() == at::kBFloat16,
              "ce_dlogits_reg: out must be a row-major bf16 matrix (row pitch may be padded)");
  TORCH_CHECK(out.size(0) == h.size(0) && out.size(1) == w.size(0), "ce_dlogits_reg: out must be [T, V]");
  TORCH_CHECK(std::isfinite(z_loss_coef) && z_loss_coef >= 0.0, "ce_dlogits_reg: z_loss_coef must be finite and >= 0");
  TORCH_CHECK(label_smoothing >= 0.0 && label_smoothing <= 1.0, "ce_dlogits_reg: label_smoothing must lie in [0, 1]");
  TORCH_CHECK(num_classes >= col_offset + w.size(0) && num_classes > 0 && num_classes < (int64_t(1) << 31),
              "ce_dlogits_reg: num_classes must cover the slice (num_classes >= col_offset + V) and fit in int32");
  c10::cuda::CUDAGuard guard(h.device());
  const int T = static_cast<int>(h.size(0)), K = static_cast<int>(h.size(1)), V = static_cast<int>(w.size(0));
  d9d::GemmArgs g;
  g.mode = DENSE; g.epi = EPI_CE_DLOGITS_REG;
  g.M = T; g.N = V; g.K = K;
  g.A = h.data_ptr(); g.B = w.data_ptr(); g.D = out.data_ptr(); g.lda = K; g.ldb = K; g.ldd = out.stride(0);
  g.ce_target = reinterpret_cast<const long long*>(target.data_ptr<int64_t>());
  g.ce_lse = lse.data_ptr<float>(); g.ce_grad = grad.data_ptr<float>();
  g.ce_ignore_index = ignore_index;
  g.ce_softcap = static_cast<float>(softcap);
  g.ce_col_offset = col_offset;
  g.ce_z_loss = static_cast<float>(z_loss_coef);
  g.ce_smoothing = static_cast<float>(label_smoothing);
  g.ce_num_classes = static_cast<int>(num_classes);
  if (bias.has_value()) g.ce_bias = bias->data_ptr<float>();
  d9d::gemm_ce(g, cur_stream());
}

// ------------------------------------------------------------------ fp8 GEMM -----------------------
// x[M,K] bf16 -> (q[M,K] e4m3, scale[M] fp32) with x ~= q * scale[:, None]
std::tuple<Tensor, Tensor> quantize_rowwise(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.scalar_type() == at::kBFloat16, "quantize_rowwise: 2-D bf16 CUDA tensor required");
  TORCH_CHECK(x.size(1) % 16 == 0 && x.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0,
              "quantize_rowwise: K must be a multiple of 16 and rows 16-byte aligned");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), K = x.size(1);
  Tensor q = at::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor scale = at::empty({M}, x.options().dtype(at::kFloat));
  d9d::quantize_rowwise_e4m3(x.data_ptr(), q.data_ptr(), scale.data_ptr<float>(), M, static_cast<int>(K), x.stride(0), cur_stream());
  return {q, scale};
}

// x[E,R,C] bf16 (R a multiple of 16) -> (qt[E,C,R] e4m3, scale[E,C] fp32) with x[e,r,c] ~= qt[e,c,r] * scale[e,c]
std::tuple<Tensor, Tensor> quantize_colwise_t_batched(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.is_contiguous() && x.scalar_type() == at::kBFloat16,
              "quantize_colwise_t_batched: contiguous 3-D bf16 CUDA tensor required");
  TORCH_CHECK(x.size(1) % 16 == 0, "quantize_colwise_t_batched: R must be a multiple of 16 (16-byte rows of the transposed copy)");
  TORCH_CHECK(x.size(0) < (int64_t(1) << 16) && x.size(2) < (int64_t(1) << 31), "quantize_colwise_t_batched: too many planes / columns");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t E = x.size(0), R = x.size(1), C = x.size(2);
  Tensor qt = at::empty({E, C, R}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor scale = at::empty({E, C}, x.options().dtype(at::kFloat));
  Tensor amax = at::empty({E, C}, x.options().dtype(at::kFloat));
  d9d::quantize_colwise_t_e4m3(x.data_ptr(), qt.data_ptr(), scale.data_ptr<float>(), amax.data_ptr<float>(), R, static_cast<int>(C),
                               C, R, cur_stream(), static_cast<int>(E));
  return {qt, scale};
}

// x[cap,C] bf16 in the MoE layout (cap a multiple of 128) -> (qt[C,cap] e4m3, scale[E,C] fp32): expert e's rows
// [seg_offsets[e], seg_offsets[e] + counts[e]) with one scale per (e, c) over them; all other rows of qt are zero
std::tuple<Tensor, Tensor> quantize_segments_t(const Tensor& x, const Tensor& tile_group, const Tensor& seg_offsets,
                                               const Tensor& counts) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.scalar_type() == at::kBFloat16,
              "quantize_segments_t: 2-D bf16 CUDA tensor with unit column stride required");
  CHECK_CUDA_CONTIG(tile_group); CHECK_CUDA_CONTIG(seg_offsets); CHECK_CUDA_CONTIG(counts);
  TORCH_CHECK(tile_group.scalar_type() == at::kInt && seg_offsets.scalar_type() == at::kInt && counts.scalar_type() == at::kInt,
              "quantize_segments_t: tile_group, seg_offsets and counts must be int32");
  TORCH_CHECK(tile_group.device() == x.device() && seg_offsets.device() == x.device() && counts.device() == x.device(),
              "quantize_segments_t: operands must be on one device");
  TORCH_CHECK(x.size(0) % 128 == 0 && tile_group.numel() == x.size(0) / 128,
              "quantize_segments_t: rows must be a multiple of 128 with one tile_group entry per 128 rows");
  TORCH_CHECK(counts.numel() > 0 && seg_offsets.numel() == counts.numel() + 1, "quantize_segments_t: seg_offsets must be [E + 1], counts [E]");
  TORCH_CHECK(x.size(0) < (int64_t(1) << 31) && x.size(1) < (int64_t(1) << 31), "quantize_segments_t: too large");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t R = x.size(0), C = x.size(1), E = counts.numel();
  Tensor qt = at::empty({C, R}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor scale = at::empty({E, C}, x.options().dtype(at::kFloat));
  Tensor amax = at::empty({E, C}, x.options().dtype(at::kFloat));
  d9d::quantize_segments_t_e4m3(x.data_ptr(), qt.data_ptr(), scale.data_ptr<float>(), amax.data_ptr<float>(), tile_group.data_ptr<int>(),
                                seg_offsets.data_ptr<int>(), counts.data_ptr<int>(), static_cast<int>(E), R, static_cast<int>(C),
                                x.stride(0), R, cur_stream());
  return {qt, scale};
}

// x[R,C] bf16 -> (qt[C,R] e4m3 (row pitch padded to 16 bytes), scale[C] fp32) with x[r,c] ~= qt[c,r] * scale[c]
std::tuple<Tensor, Tensor> quantize_colwise_t(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.scalar_type() == at::kBFloat16, "quantize_colwise_t: 2-D bf16 CUDA tensor required");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t R = x.size(0), C = x.size(1);
  const int64_t pitch = (R + 15) / 16 * 16;
  Tensor qt = at::zeros({C, pitch}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor scale = at::empty({C}, x.options().dtype(at::kFloat));
  Tensor amax = at::empty({C}, x.options().dtype(at::kFloat));
  d9d::quantize_colwise_t_e4m3(x.data_ptr(), qt.data_ptr(), scale.data_ptr<float>(), amax.data_ptr<float>(), R, static_cast<int>(C),
                               x.stride(0), pitch, cur_stream());
  return {qt.narrow(1, 0, R), scale};
}

// x[M,K] bf16 -> (q[M,K] e4m3, sf uint8 [2*ceil(M/256), K/128, 512]): OCP MXFP8, one UE8M0 scale per 32 elements along K,
// stored in the 128-row x 4-group block layout the MXFP8 GEMM reads
std::tuple<Tensor, Tensor> quantize_mx(const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.scalar_type() == at::kBFloat16, "quantize_mx: 2-D bf16 CUDA tensor required");
  TORCH_CHECK(x.size(1) % 128 == 0 && x.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0,
              "quantize_mx: K must be a multiple of 128 and rows 16-byte aligned");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), K = x.size(1);
  Tensor q = at::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor sf = at::zeros({(M + 255) / 256 * 2, K / 128, 512}, x.options().dtype(at::kByte));
  d9d::quantize_mx_e4m3(x.data_ptr(), q.data_ptr(), sf.data_ptr(), M, static_cast<int>(K), x.stride(0), cur_stream());
  return {q, sf};
}

static void fill_fp8_operands(d9d::Fp8GemmArgs& g, const Tensor& a, const Tensor& b, Tensor& d) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && d.is_cuda() && a.dim() == 2 && b.dim() == 2 && d.dim() == 2, "gemm_fp8: 2-D CUDA tensors required");
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8: e4m3 operands required");
  TORCH_CHECK(d.scalar_type() == at::kBFloat16 && a.stride(1) == 1 && b.stride(1) == 1 && d.stride(1) == 1, "gemm_fp8: bf16 row-major output");
  TORCH_CHECK(a.size(1) == b.size(1) && d.size(0) == a.size(0) && d.size(1) == b.size(0), "gemm_fp8: shape mismatch");
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1)); g.N = static_cast<int>(b.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
}

// d[M,N] bf16 = (a[M,K] · b[N,K]^T) * scale_a[m] * scale_b[n] * scalar
void gemm_fp8(const Tensor& a, const Tensor& b, const c10::optional<Tensor>& scale_a, const c10::optional<Tensor>& scale_b, double scalar,
              Tensor d) {
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  fill_fp8_operands(g, a, b, d);
  if (scale_a.has_value()) {
    CHECK_CUDA_CONTIG(*scale_a);
    TORCH_CHECK(scale_a->scalar_type() == at::kFloat && scale_a->numel() == g.M, "gemm_fp8: scale_a must be fp32 [M]");
    g.scale_a = scale_a->data_ptr<float>();
  }
  if (scale_b.has_value()) {
    CHECK_CUDA_CONTIG(*scale_b);
    TORCH_CHECK(scale_b->scalar_type() == at::kFloat && scale_b->numel() == g.N, "gemm_fp8: scale_b must be fp32 [N]");
    g.scale_b = scale_b->data_ptr<float>();
  }
  g.scale_scalar = static_cast<float>(scalar);
  d9d::gemm_fp8(g, cur_stream());
}

// d[M,N] bf16 = sum_k (a * 2^sfa) (b * 2^sfb): block-scaled (MXFP8) operands from quantize_mx
void gemm_mxfp8(const Tensor& a, const Tensor& sfa, const Tensor& b, const Tensor& sfb, Tensor d) {
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  fill_fp8_operands(g, a, b, d);
  CHECK_CUDA_CONTIG(sfa); CHECK_CUDA_CONTIG(sfb);
  TORCH_CHECK(g.K % 128 == 0, "gemm_mxfp8: K must be a multiple of 128");
  const int64_t kb = g.K / 128;
  TORCH_CHECK(sfa.scalar_type() == at::kByte && sfa.numel() >= (static_cast<int64_t>(g.M) + 127) / 128 * kb * 512, "gemm_mxfp8: sfa too small");
  TORCH_CHECK(sfb.scalar_type() == at::kByte && sfb.numel() >= (static_cast<int64_t>(g.N) + 127) / 128 * kb * 512, "gemm_mxfp8: sfb too small");
  g.scaling = d9d::fp8::MX;
  g.sfa = sfa.data_ptr<uint8_t>(); g.sfb = sfb.data_ptr<uint8_t>();
  d9d::gemm_fp8(g, cur_stream());
}

// Operand checks of the grouped fp8 GEMMs, before anything touches the device: e4m3 K-major operands with 16-byte rows,
// fp32 scales of the stated lengths, int32 tables, one device
void check_fp8_grouped(const char* op, const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, const Tensor& d,
                       const Tensor& table) {
  for (const Tensor* t : {&a, &sa, &b, &sb, &d, &table}) {
    TORCH_CHECK(t->is_cuda() && t->device() == a.device(), op, ": all operands must be CUDA tensors on one device");
    TORCH_CHECK(t->is_contiguous(), op, ": operands must be contiguous");
  }
  CHECK_ALIGNED16(a); CHECK_ALIGNED16(b); CHECK_ALIGNED16(d);
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn, op, ": a and b must be float8_e4m3fn");
  TORCH_CHECK(sa.scalar_type() == at::kFloat && sb.scalar_type() == at::kFloat, op, ": scales must be fp32");
  TORCH_CHECK(table.scalar_type() == at::kInt, op, ": the expert table must be int32");
  TORCH_CHECK(a.dim() == 2 && a.size(1) % 16 == 0 && a.size(1) > 0, op, ": a must be 2-D with rows of a positive multiple of 16 bytes");
  TORCH_CHECK(a.size(0) < (int64_t(1) << 31) && a.size(1) < (int64_t(1) << 31), op, ": a is too large");
}

// d[R,N] (+)= (a[R,K] · b[e(r)]^T) * sa[r] * sb[e(r), n]: the MoE forward / input gradient in fp8.  a: the expert-sorted
// rows (R a multiple of 128), b: [E, N, K], tile_group: [R/128] expert of every 128-row tile (-1: never written)
void gemm_fp8_grouped_m(const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, Tensor d, const Tensor& tile_group,
                        bool accumulate) {
  check_fp8_grouped("gemm_fp8_grouped_m", a, sa, b, sb, d, tile_group);
  TORCH_CHECK(b.dim() == 3 && b.size(2) == a.size(1), "gemm_fp8_grouped_m: b must be [E, N, K] with the K of a");
  TORCH_CHECK(b.size(0) > 0 && b.size(1) > 0 && b.size(1) < (int64_t(1) << 31), "gemm_fp8_grouped_m: b must have experts and N > 0");
  TORCH_CHECK(a.size(0) % 128 == 0 && tile_group.numel() == a.size(0) / 128,
              "gemm_fp8_grouped_m: rows must be a multiple of 128 with one tile_group entry per 128 rows");
  TORCH_CHECK(sa.numel() == a.size(0), "gemm_fp8_grouped_m: sa must be [R]");
  TORCH_CHECK(sb.numel() == b.size(0) * b.size(1), "gemm_fp8_grouped_m: sb must be [E * N]");
  TORCH_CHECK(d.dim() == 2 && d.size(0) == a.size(0) && d.size(1) == b.size(1) && d.scalar_type() == at::kBFloat16,
              "gemm_fp8_grouped_m: d must be bf16 [R, N]");
  TORCH_CHECK(d.size(1) % 8 == 0, "gemm_fp8_grouped_m: N must be a multiple of 8 (16-byte output rows)");
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  g.mode = GROUPED_M; g.epi = accumulate ? EPI_BF16_ACC : EPI_BF16;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1)); g.N = static_cast<int>(b.size(1));
  g.num_groups = static_cast<int>(b.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(1); g.b_group_stride = b.stride(0); g.ldd = d.stride(0);
  g.scale_a = sa.data_ptr<float>(); g.scale_b = sb.data_ptr<float>();
  g.tile_group = tile_group.data_ptr<int>();
  d9d::gemm_fp8(g, cur_stream());
}

// d[e] (+)= (a[:, rows_e] · b[:, rows_e]^T) * sa[e, m] * sb[e, n] over expert e's rows group_offsets[e] .. [e+1]: the MoE
// weight gradient in fp8.  a: [M, R], b: [N, R] (the transposed, per-expert quantised activations / output gradients),
// d: [E, M, N] fp32 or bf16 (an expert without rows: zeros when storing, untouched when accumulating)
void gemm_fp8_grouped_k(const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, Tensor d, const Tensor& group_offsets,
                        bool accumulate) {
  check_fp8_grouped("gemm_fp8_grouped_k", a, sa, b, sb, d, group_offsets);
  TORCH_CHECK(b.dim() == 2 && b.size(1) == a.size(1) && b.size(0) > 0 && b.size(0) < (int64_t(1) << 31),
              "gemm_fp8_grouped_k: b must be [N, R] with the R of a");
  TORCH_CHECK(a.size(1) % 128 == 0, "gemm_fp8_grouped_k: R must be a multiple of 128 (the expert segments' alignment)");
  TORCH_CHECK(d.dim() == 3 && d.size(0) > 0 && d.size(1) == a.size(0) && d.size(2) == b.size(0),
              "gemm_fp8_grouped_k: d must be [E, M, N]");
  TORCH_CHECK(d.scalar_type() == at::kFloat || d.scalar_type() == at::kBFloat16, "gemm_fp8_grouped_k: d must be fp32 or bf16");
  TORCH_CHECK(d.size(2) * d.element_size() % 16 == 0, "gemm_fp8_grouped_k: rows of d must be a multiple of 16 bytes");
  TORCH_CHECK(group_offsets.numel() == d.size(0) + 1, "gemm_fp8_grouped_k: group_offsets must be [E + 1]");
  TORCH_CHECK(sa.numel() == d.size(0) * d.size(1), "gemm_fp8_grouped_k: sa must be [E * M]");
  TORCH_CHECK(sb.numel() == d.size(0) * d.size(2), "gemm_fp8_grouped_k: sb must be [E * N]");
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  g.mode = GROUPED_K; g.epi = epi_for(d, accumulate);
  g.M = static_cast<int>(a.size(0)); g.N = static_cast<int>(b.size(0)); g.K = 0;
  g.k_total = a.size(1);
  g.num_groups = static_cast<int>(d.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(1); g.d_group_stride = d.stride(0);
  g.scale_a = sa.data_ptr<float>(); g.scale_b = sb.data_ptr<float>();
  g.group_offsets = group_offsets.data_ptr<int>();
  d9d::gemm_fp8(g, cur_stream());
}

// ------------------------------------------------------------------ blockwise fp8 (DeepSeek-V3 recipe) ----------------
// Scales are k-block-major: [ceil(K/128), rows] with a row pitch of round_up(rows, 128) (a view of a zero-padded
// allocation), so the GEMM reads a tile's scales as one aligned 512-byte copy inside the tensor.
static int64_t round_up128(int64_t v) { return (v + 127) / 128 * 128; }

static Tensor blockwise_scales(const Tensor& like, int64_t groups, int64_t rows) {
  return at::zeros({groups, round_up128(rows)}, like.options().dtype(at::kFloat)).narrow(1, 0, rows);
}

static void check_blockwise_input(const char* op, const Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && x.scalar_type() == at::kBFloat16, op, ": 2-D bf16 CUDA tensor with unit column stride required");
  TORCH_CHECK(x.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0, op, ": rows must be 16-byte aligned");
  TORCH_CHECK(x.size(0) < (int64_t(1) << 31) && x.size(1) < (int64_t(1) << 31), op, ": too large");
}

// x[M,K] bf16 (K a multiple of 16) -> (q[M,K] e4m3, s[ceil(K/128), M] fp32): one scale per 1 x 128 group of every row
std::tuple<Tensor, Tensor> quantize_blockwise(const Tensor& x) {
  check_blockwise_input("quantize_blockwise", x);
  TORCH_CHECK(x.size(1) % 16 == 0, "quantize_blockwise: K must be a multiple of 16");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), K = x.size(1);
  Tensor q = at::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = blockwise_scales(x, (K + 127) / 128, M);
  d9d::quantize_blockwise_e4m3(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), M, static_cast<int>(K), x.stride(0), K, s.stride(0),
                               d9d::GROUP_ROW, false, cur_stream());
  return {q, s};
}

// x[M,C] bf16 (C a multiple of 16, any M) -> (qt[C,M] e4m3 with a 16-byte row pitch and zero pad columns,
// s[ceil(M/128), C] fp32): one scale per 128 rows of every column, i.e. per 128-token group of a channel
std::tuple<Tensor, Tensor> quantize_blockwise_t(const Tensor& x) {
  check_blockwise_input("quantize_blockwise_t", x);
  TORCH_CHECK(x.size(1) % 16 == 0, "quantize_blockwise_t: C must be a multiple of 16");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), C = x.size(1);
  const int64_t pitch = (M + 15) / 16 * 16;
  Tensor qt = at::empty({C, pitch}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = blockwise_scales(x, (M + 127) / 128, C);
  d9d::quantize_blockwise_e4m3(x.data_ptr(), qt.data_ptr(), s.data_ptr<float>(), M, static_cast<int>(C), x.stride(0), pitch, s.stride(0),
                               d9d::GROUP_COL, true, cur_stream());
  return {qt.narrow(1, 0, M), s};
}

// w[N,K] bf16 (N, K multiples of 16) -> one scale per 128 x 128 block, repeated on each row of the copy the GEMM reads:
//   transpose = false: (q[N,K], s[ceil(K/128), N]);  transpose = true: (qt[K,N], s[ceil(N/128), K])
std::tuple<Tensor, Tensor> quantize_weight_blocks(const Tensor& w, bool transpose) {
  check_blockwise_input("quantize_weight_blocks", w);
  TORCH_CHECK(w.size(0) % 16 == 0 && w.size(1) % 16 == 0, "quantize_weight_blocks: both dims must be multiples of 16");
  c10::cuda::CUDAGuard guard(w.device());
  const int64_t N = w.size(0), K = w.size(1);
  Tensor q = transpose ? at::empty({K, N}, w.options().dtype(at::kFloat8_e4m3fn)) : at::empty({N, K}, w.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = transpose ? blockwise_scales(w, (N + 127) / 128, K) : blockwise_scales(w, (K + 127) / 128, N);
  d9d::quantize_blockwise_e4m3(w.data_ptr(), q.data_ptr(), s.data_ptr<float>(), N, static_cast<int>(K), w.stride(0), q.stride(0),
                               s.stride(0), d9d::GROUP_BLOCK, transpose, cur_stream());
  return {q, s};
}

static void check_blockwise_scales(const char* name, const Tensor& s, const Tensor& like, int64_t groups, int64_t rows) {
  TORCH_CHECK(s.is_cuda() && s.device() == like.device(), "gemm_fp8_blockwise: ", name, " must be on the operands' device");
  TORCH_CHECK(s.scalar_type() == at::kFloat && s.dim() == 2 && s.size(0) == groups && s.size(1) == rows && s.stride(1) == 1,
              "gemm_fp8_blockwise: ", name, " must be fp32 [ceil(K/128), rows] with the K and rows of its operand");
  TORCH_CHECK(s.stride(0) == round_up128(rows), "gemm_fp8_blockwise: ", name, " must have a row pitch of round_up(rows, 128)");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(s.data_ptr()) & 15) == 0, "gemm_fp8_blockwise: ", name, " must start on a 16-byte boundary");
  const int64_t avail = static_cast<int64_t>(s.storage().nbytes()) - s.storage_offset() * 4;
  TORCH_CHECK(avail >= groups * s.stride(0) * 4, "gemm_fp8_blockwise: ", name, "'s storage must hold its padded rows");
}

// d[M,N] (bf16 or fp32) = sum over 128-deep k-blocks kb of (a[:, kb] · b[:, kb]^T) * sa[kb, m] * sb[kb, n]
void gemm_fp8_blockwise(const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, Tensor d) {
  for (const Tensor* t : {&a, &b, static_cast<const Tensor*>(&d)})
    TORCH_CHECK(t->is_cuda() && t->device() == a.device() && t->dim() == 2 && t->stride(1) == 1,
                "gemm_fp8_blockwise: a, b and d must be 2-D CUDA tensors on one device with unit column stride");
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8_blockwise: a and b must be float8_e4m3fn");
  TORCH_CHECK(d.scalar_type() == at::kBFloat16 || d.scalar_type() == at::kFloat, "gemm_fp8_blockwise: d must be bf16 or fp32");
  TORCH_CHECK(a.size(1) == b.size(1) && a.size(1) > 0, "gemm_fp8_blockwise: a and b must share a positive K");
  TORCH_CHECK(d.size(0) == a.size(0) && d.size(1) == b.size(0), "gemm_fp8_blockwise: d must be [M, N]");
  TORCH_CHECK(a.size(0) < (int64_t(1) << 31) && b.size(0) < (int64_t(1) << 31) && a.size(1) < (int64_t(1) << 31), "gemm_fp8_blockwise: too large");
  CHECK_ALIGNED16(a); CHECK_ALIGNED16(b); CHECK_ALIGNED16(d);
  TORCH_CHECK(a.stride(0) % 16 == 0 && b.stride(0) % 16 == 0, "gemm_fp8_blockwise: rows of a and b must be 16-byte aligned");
  TORCH_CHECK(d.stride(0) * d.element_size() % 16 == 0 && d.size(1) * d.element_size() % 16 == 0,
              "gemm_fp8_blockwise: rows of d must be a multiple of 16 bytes");
  const int64_t kb = (a.size(1) + 127) / 128;
  check_blockwise_scales("sa", sa, a, kb, a.size(0));
  check_blockwise_scales("sb", sb, a, kb, b.size(0));
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  g.scaling = d9d::fp8::BLOCKWISE;
  g.epi = d.scalar_type() == at::kBFloat16 ? EPI_BF16 : EPI_F32;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1)); g.N = static_cast<int>(b.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.scale_a = sa.data_ptr<float>(); g.scale_b = sb.data_ptr<float>();
  d9d::gemm_fp8(g, cur_stream());
}

// ------------------------------------------------------------------ blockwise fp8 MoE experts ---------------------------
// w[E, in, out] bf16 (in, out multiples of 16) -> one scale per 128 x 128 block of every w[e], in the copy a grouped GEMM reads:
//   transpose = true (forward):  (qt[E, out, in], s[E, ceil(in/128), out])
//   transpose = false (dgrad):   (q[E, in, out],  s[E, ceil(out/128), in])
// s is a view with a row pitch of round_up(rows, 128) (zero pad)
std::tuple<Tensor, Tensor> quantize_expert_weight_blocks(const Tensor& w, bool transpose) {
  TORCH_CHECK(w.is_cuda() && w.dim() == 3 && w.is_contiguous() && w.scalar_type() == at::kBFloat16,
              "quantize_expert_weight_blocks: contiguous 3-D bf16 CUDA tensor [E, in, out] required");
  TORCH_CHECK(w.size(0) > 0 && w.size(1) % 16 == 0 && w.size(2) % 16 == 0, "quantize_expert_weight_blocks: in and out must be multiples of 16");
  TORCH_CHECK(w.size(0) < (int64_t(1) << 16) && w.size(1) < (int64_t(1) << 31) && w.size(2) < (int64_t(1) << 31),
              "quantize_expert_weight_blocks: too large");
  CHECK_ALIGNED16(w);
  c10::cuda::CUDAGuard guard(w.device());
  const int64_t E = w.size(0), R = w.size(1), C = w.size(2);
  const int64_t groups = transpose ? (R + 127) / 128 : (C + 127) / 128, rows = transpose ? C : R;
  Tensor q = transpose ? at::empty({E, C, R}, w.options().dtype(at::kFloat8_e4m3fn)) : at::empty({E, R, C}, w.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = at::zeros({E, groups, round_up128(rows)}, w.options().dtype(at::kFloat)).narrow(2, 0, rows);
  d9d::quantize_expert_blocks_e4m3(w.data_ptr(), q.data_ptr(), s.data_ptr<float>(), static_cast<int>(E), R, static_cast<int>(C),
                                   s.stride(1), transpose, cur_stream());
  return {q, s};
}

static void check_tiles_input(const char* op, const Tensor& x, const Tensor& tile_group) {
  check_blockwise_input(op, x);
  TORCH_CHECK(x.size(1) % 16 == 0, op, ": C must be a multiple of 16");
  TORCH_CHECK(tile_group.is_cuda() && tile_group.device() == x.device() && tile_group.is_contiguous() && tile_group.scalar_type() == at::kInt,
              op, ": tile_group must be a contiguous int32 tensor on x's device");
  TORCH_CHECK(x.size(0) % 128 == 0 && tile_group.numel() == x.size(0) / 128, op,
              ": rows must be a multiple of 128 with one tile_group entry per 128 rows");
}

// x[cap, C] bf16 in the MoE layout -> (q[cap, C] e4m3, s[ceil(C/128), cap] fp32): one scale per 1 x 128 group of every row
// of the 128-row tiles in use; tiles whose tile_group is -1 are skipped (their codes and scales are never read)
std::tuple<Tensor, Tensor> quantize_blockwise_tiles(const Tensor& x, const Tensor& tile_group) {
  check_tiles_input("quantize_blockwise_tiles", x, tile_group);
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t R = x.size(0), C = x.size(1);
  Tensor q = at::empty({R, C}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = at::empty({(C + 127) / 128, R}, x.options().dtype(at::kFloat));
  d9d::quantize_blockwise_tiles_e4m3(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), tile_group.data_ptr<int>(), nullptr, nullptr, R,
                                     static_cast<int>(C), x.stride(0), C, s.stride(0), false, cur_stream());
  return {q, s};
}

// x[cap, C] bf16 in the MoE layout -> (qt[C, cap] e4m3, s[cap/128, C] fp32): one scale per 128-token group of every channel;
// an expert's groups start at its segment and end at its last row (later rows of its tiles are zeros in qt); tiles whose
// tile_group is -1 are skipped
std::tuple<Tensor, Tensor> quantize_blockwise_t_tiles(const Tensor& x, const Tensor& tile_group, const Tensor& seg_offsets,
                                                      const Tensor& counts) {
  check_tiles_input("quantize_blockwise_t_tiles", x, tile_group);
  for (const Tensor* t : {&seg_offsets, &counts})
    TORCH_CHECK(t->is_cuda() && t->device() == x.device() && t->is_contiguous() && t->scalar_type() == at::kInt,
                "quantize_blockwise_t_tiles: seg_offsets and counts must be contiguous int32 tensors on x's device");
  TORCH_CHECK(counts.numel() > 0 && seg_offsets.numel() == counts.numel() + 1, "quantize_blockwise_t_tiles: seg_offsets must be [E + 1], counts [E]");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t R = x.size(0), C = x.size(1);
  Tensor qt = at::empty({C, R}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = blockwise_scales(x, R / 128, C);
  d9d::quantize_blockwise_tiles_e4m3(x.data_ptr(), qt.data_ptr(), s.data_ptr<float>(), tile_group.data_ptr<int>(), seg_offsets.data_ptr<int>(),
                                     counts.data_ptr<int>(), R, static_cast<int>(C), x.stride(0), R, s.stride(0), true, cur_stream());
  return {qt, s};
}

// Operand checks of the blockwise grouped GEMMs: e4m3 K-major operands with 16-byte rows, int32 table, one device
static void check_blockwise_grouped(const char* op, const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, const Tensor& d,
                                    const Tensor& table) {
  for (const Tensor* t : {&a, &sa, &b, &sb, &d, &table})
    TORCH_CHECK(t->is_cuda() && t->device() == a.device(), op, ": all operands must be CUDA tensors on one device");
  for (const Tensor* t : {&a, &b, &d, &table}) TORCH_CHECK(t->is_contiguous(), op, ": a, b, d and the expert table must be contiguous");
  CHECK_ALIGNED16(a); CHECK_ALIGNED16(b); CHECK_ALIGNED16(d);
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn, op, ": a and b must be float8_e4m3fn");
  TORCH_CHECK(sa.scalar_type() == at::kFloat && sb.scalar_type() == at::kFloat, op, ": scales must be fp32");
  TORCH_CHECK(table.scalar_type() == at::kInt, op, ": the expert table must be int32");
  TORCH_CHECK(a.dim() == 2 && a.size(1) % 16 == 0 && a.size(1) > 0, op, ": a must be 2-D with rows of a positive multiple of 16 bytes");
  TORCH_CHECK(a.size(0) < (int64_t(1) << 31) && a.size(1) < (int64_t(1) << 31), op, ": a is too large");
}

// s: [..., groups, rows] fp32 view with unit column stride, a row pitch of round_up(rows, 128), planes groups * pitch apart
static void check_grouped_scales(const char* op, const char* name, const Tensor& s, std::vector<int64_t> shape) {
  const int64_t rows = shape.back(), pitch = round_up128(rows);
  TORCH_CHECK(s.sizes().vec() == shape, op, ": ", name, " has the wrong shape for its operand");
  TORCH_CHECK(s.stride(-1) == 1 && s.stride(-2) == pitch && (s.dim() == 2 || s.stride(0) == shape[1] * pitch), op, ": ", name,
              " must be k-block-major with a row pitch of round_up(rows, 128)");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(s.data_ptr()) & 15) == 0, op, ": ", name, " must start on a 16-byte boundary");
  int64_t planes = 1;
  for (size_t i = 0; i + 1 < shape.size(); ++i) planes *= shape[i];
  const int64_t avail = static_cast<int64_t>(s.storage().nbytes()) - s.storage_offset() * 4;
  TORCH_CHECK(avail >= planes * pitch * 4, op, ": ", name, "'s storage must hold its padded rows");
}

// d[R, N] (+)= sum_kb (a[R, kb] · b[e(r), :, kb]^T) * sa[kb, r] * sb[e(r), kb, n]: the MoE forward / input gradient under the
// blockwise recipe.  a: expert-sorted rows (R a multiple of 128), b: [E, N, K], tile_group: [R/128] (-1: never read or written)
void gemm_fp8_blockwise_grouped_m(const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, Tensor d, const Tensor& tile_group,
                                  bool accumulate) {
  const char* op = "gemm_fp8_blockwise_grouped_m";
  check_blockwise_grouped(op, a, sa, b, sb, d, tile_group);
  TORCH_CHECK(b.dim() == 3 && b.size(2) == a.size(1), op, ": b must be [E, N, K] with the K of a");
  TORCH_CHECK(b.size(0) > 0 && b.size(1) > 0 && b.size(1) < (int64_t(1) << 31), op, ": b must have experts and N > 0");
  TORCH_CHECK(a.size(0) % 128 == 0 && tile_group.numel() == a.size(0) / 128, op, ": rows must be a multiple of 128 with one tile_group entry per 128 rows");
  TORCH_CHECK(d.dim() == 2 && d.size(0) == a.size(0) && d.size(1) == b.size(1) && d.scalar_type() == at::kBFloat16, op, ": d must be bf16 [R, N]");
  TORCH_CHECK(d.size(1) % 8 == 0, op, ": N must be a multiple of 8 (16-byte output rows)");
  const int64_t kb = (a.size(1) + 127) / 128;
  check_grouped_scales(op, "sa", sa, {kb, a.size(0)});
  check_grouped_scales(op, "sb", sb, {b.size(0), kb, b.size(1)});
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  g.scaling = d9d::fp8::BLOCKWISE;
  g.mode = GROUPED_M; g.epi = accumulate ? EPI_BF16_ACC : EPI_BF16;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1)); g.N = static_cast<int>(b.size(1));
  g.num_groups = static_cast<int>(b.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(1); g.b_group_stride = b.stride(0); g.ldd = d.stride(0);
  g.scale_a = sa.data_ptr<float>(); g.scale_b = sb.data_ptr<float>();
  g.tile_group = tile_group.data_ptr<int>();
  d9d::gemm_fp8(g, cur_stream());
}

// d[e] (+)= sum over expert e's 128-token groups kb of (a[:, kb] · b[:, kb]^T) * sa[kb, m] * sb[kb, n]: the MoE weight gradient
// under the blockwise recipe.  a: [M, R], b: [N, R] from quantize_blockwise_t_tiles, d: [E, M, N] fp32 or bf16 (an expert without
// rows: zeros when storing, untouched when accumulating)
void gemm_fp8_blockwise_grouped_k(const Tensor& a, const Tensor& sa, const Tensor& b, const Tensor& sb, Tensor d, const Tensor& group_offsets,
                                  bool accumulate) {
  const char* op = "gemm_fp8_blockwise_grouped_k";
  check_blockwise_grouped(op, a, sa, b, sb, d, group_offsets);
  TORCH_CHECK(b.dim() == 2 && b.size(1) == a.size(1) && b.size(0) > 0 && b.size(0) < (int64_t(1) << 31), op, ": b must be [N, R] with the R of a");
  TORCH_CHECK(a.size(1) % 128 == 0, op, ": R must be a multiple of 128 (the expert segments' alignment)");
  TORCH_CHECK(d.dim() == 3 && d.size(0) > 0 && d.size(1) == a.size(0) && d.size(2) == b.size(0), op, ": d must be [E, M, N]");
  TORCH_CHECK(d.scalar_type() == at::kFloat || d.scalar_type() == at::kBFloat16, op, ": d must be fp32 or bf16");
  TORCH_CHECK(d.size(2) * d.element_size() % 16 == 0, op, ": rows of d must be a multiple of 16 bytes");
  TORCH_CHECK(group_offsets.numel() == d.size(0) + 1, op, ": group_offsets must be [E + 1]");
  check_grouped_scales(op, "sa", sa, {a.size(1) / 128, a.size(0)});
  check_grouped_scales(op, "sb", sb, {a.size(1) / 128, b.size(0)});
  c10::cuda::CUDAGuard guard(a.device());
  d9d::Fp8GemmArgs g;
  g.scaling = d9d::fp8::BLOCKWISE;
  g.mode = GROUPED_K; g.epi = epi_for(d, accumulate);
  g.M = static_cast<int>(a.size(0)); g.N = static_cast<int>(b.size(0)); g.K = 0;
  g.k_total = a.size(1);
  g.num_groups = static_cast<int>(d.size(0));
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(1); g.d_group_stride = d.stride(0);
  g.scale_a = sa.data_ptr<float>(); g.scale_b = sb.data_ptr<float>();
  g.group_offsets = group_offsets.data_ptr<int>();
  d9d::gemm_fp8(g, cur_stream());
}

// ------------------------------------------------------------------ RMSNorm ---------------------
std::tuple<Tensor, Tensor> rms_norm_fwd(const Tensor& x, const Tensor& w, double eps, bool zero_centered) {
  CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(w); CHECK_ALIGNED16(x); CHECK_ALIGNED16(w);
  TORCH_CHECK(x.scalar_type() == w.scalar_type(), "rms_norm: x and weight dtypes must match");
  c10::cuda::CUDAGuard guard(x.device());
  const int N = static_cast<int>(x.size(-1));
  TORCH_CHECK(N > 0 && w.numel() == N, "rms_norm: weight must have x.size(-1) elements");
  const int64_t M = x.numel() / N;
  Tensor out = at::empty_like(x);
  Tensor inv = at::empty({M}, x.options().dtype(at::kFloat));
  d9d::rms_norm_fwd(x.data_ptr(), w.data_ptr(), out.data_ptr(), inv.data_ptr<float>(), M, N, static_cast<float>(eps),
                    zero_centered, dtype_code(x), cur_stream());
  return {out, inv};
}

std::tuple<Tensor, Tensor> rms_norm_bwd(const Tensor& dout, const Tensor& x, const Tensor& w, const Tensor& inv_rms,
                                        bool zero_centered) {
  CHECK_CUDA_CONTIG(dout); CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(w); CHECK_CUDA_CONTIG(inv_rms);
  CHECK_ALIGNED16(dout); CHECK_ALIGNED16(x); CHECK_ALIGNED16(w);
  TORCH_CHECK(dout.scalar_type() == x.scalar_type() && w.scalar_type() == x.scalar_type() && dout.numel() == x.numel(),
              "rms_norm bwd: dout, x and weight must share a dtype and dout the shape of x");
  c10::cuda::CUDAGuard guard(x.device());
  const int N = static_cast<int>(x.size(-1));
  TORCH_CHECK(N > 0 && w.numel() == N, "rms_norm bwd: weight must have x.size(-1) elements");
  const int64_t M = x.numel() / N;
  TORCH_CHECK(inv_rms.scalar_type() == at::kFloat && inv_rms.numel() == M, "rms_norm bwd: inv_rms must be fp32 with one value per row");
  Tensor dx = at::empty_like(x);
  Tensor dw = at::empty_like(w);
  Tensor partial = at::empty({d9d::rms_norm_bwd_num_partials(), N}, x.options().dtype(at::kFloat));
  d9d::rms_norm_bwd(dout.data_ptr(), x.data_ptr(), w.data_ptr(), inv_rms.data_ptr<float>(), dx.data_ptr(),
                    dw.data_ptr(), partial.data_ptr<float>(), M, N, zero_centered, dtype_code(x), cur_stream());
  return {dx, dw};
}

// ------------------------------------------------------------------ SiLU * mul -------------------
Tensor silu_mul_fwd(const Tensor& x, const Tensor& y) {
  CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(y); CHECK_ALIGNED16(x); CHECK_ALIGNED16(y);
  TORCH_CHECK(x.scalar_type() == y.scalar_type() && x.numel() == y.numel());
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty_like(x);
  d9d::silu_mul_fwd(x.data_ptr(), y.data_ptr(), out.data_ptr(), x.numel(), dtype_code(x), cur_stream());
  return out;
}

std::tuple<Tensor, Tensor> silu_mul_bwd(const Tensor& dout, const Tensor& x, const Tensor& y) {
  CHECK_CUDA_CONTIG(dout); CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(y);
  CHECK_ALIGNED16(dout); CHECK_ALIGNED16(x); CHECK_ALIGNED16(y);
  TORCH_CHECK(dout.scalar_type() == x.scalar_type() && y.scalar_type() == x.scalar_type() && dout.numel() == x.numel() &&
              y.numel() == x.numel(), "silu_mul bwd: dout, x and y must share a dtype and a size");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = at::empty_like(x), dy = at::empty_like(y);
  d9d::silu_mul_bwd(dout.data_ptr(), x.data_ptr(), y.data_ptr(), dx.data_ptr(), dy.data_ptr(), x.numel(),
                    dtype_code(x), cur_stream());
  return {dx, dy};
}

static const int* valid_rows_ptr(const c10::optional<Tensor>& v) {
  if (!v.has_value()) return nullptr;
  TORCH_CHECK(v->is_cuda() && v->scalar_type() == at::kInt && v->numel() >= 1, "valid_rows must be an int32 CUDA scalar");
  return v->data_ptr<int>();
}

Tensor silu_mul_probs_fwd(const Tensor& x, const Tensor& y, const Tensor& probs, const c10::optional<Tensor>& valid_rows) {
  CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(y); CHECK_CUDA_CONTIG(probs); CHECK_ALIGNED16(x); CHECK_ALIGNED16(y);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 && probs.scalar_type() == at::kFloat);
  TORCH_CHECK(x.dim() == 2 && y.sizes() == x.sizes() && probs.numel() == x.size(0),
              "silu_mul_probs: x and y must be [rows, cols] and probs [rows]");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty_like(x);
  d9d::silu_mul_probs_fwd(x.data_ptr(), y.data_ptr(), probs.data_ptr<float>(), out.data_ptr(), x.size(0),
                          static_cast<int>(x.size(1)), valid_rows_ptr(valid_rows), cur_stream());
  return out;
}

std::tuple<Tensor, Tensor, Tensor> silu_mul_probs_bwd(const Tensor& dout, const Tensor& x, const Tensor& y,
                                                      const Tensor& probs, const c10::optional<Tensor>& valid_rows) {
  CHECK_CUDA_CONTIG(dout); CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(y); CHECK_CUDA_CONTIG(probs);
  CHECK_ALIGNED16(dout); CHECK_ALIGNED16(x); CHECK_ALIGNED16(y);
  TORCH_CHECK(dout.scalar_type() == at::kBFloat16 && x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 &&
              probs.scalar_type() == at::kFloat, "silu_mul_probs bwd: bf16 dout / x / y and fp32 probs required");
  TORCH_CHECK(x.dim() == 2 && y.sizes() == x.sizes() && dout.sizes() == x.sizes() && probs.numel() == x.size(0),
              "silu_mul_probs bwd: dout, x and y must be [rows, cols] and probs [rows]");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = at::empty_like(x), dy = at::empty_like(y), dp = at::empty_like(probs);
  d9d::silu_mul_probs_bwd(dout.data_ptr(), x.data_ptr(), y.data_ptr(), probs.data_ptr<float>(), dx.data_ptr(),
                          dy.data_ptr(), dp.data_ptr<float>(), x.size(0), static_cast<int>(x.size(1)), valid_rows_ptr(valid_rows),
                          cur_stream());
  return {dx, dy, dp};
}

// ------------------------------------------------------------------ stochastic rounding ----------
void sr_copy_(Tensor dst, const Tensor& src, int64_t seed) {
  CHECK_CUDA_CONTIG(dst); CHECK_CUDA_CONTIG(src);
  TORCH_CHECK(dst.scalar_type() == at::kBFloat16 && src.scalar_type() == at::kFloat && dst.numel() == src.numel());
  c10::cuda::CUDAGuard guard(src.device());
  d9d::sr_copy_f32_to_bf16(src.data_ptr<float>(), dst.data_ptr(), src.numel(), static_cast<uint64_t>(seed), cur_stream());
}

// metas: int64 [n_tensors, 6] = (p, g, m, v, numel, rng_base) in device memory; block_map: int32 [n_blocks, 2]
void adamw_sr_multi_(const Tensor& metas, const Tensor& block_map, double lr, double beta1, double beta2, double eps,
                     double weight_decay, int64_t step, int64_t seed, const c10::optional<Tensor>& grad_scale,
                     bool grad_bf16, bool state_bf16) {
  CHECK_CUDA_CONTIG(metas); CHECK_CUDA_CONTIG(block_map);
  TORCH_CHECK(metas.scalar_type() == at::kLong && metas.size(1) == 6 && block_map.scalar_type() == at::kInt);
  static_assert(sizeof(d9d::AdamTensorMeta) == 6 * sizeof(int64_t), "meta layout");
  c10::cuda::CUDAGuard guard(metas.device());
  const double bc1 = 1.0 - std::exp(static_cast<double>(step) * std::log(beta1));
  const double bc2 = 1.0 - std::exp(static_cast<double>(step) * std::log(beta2));
  const float* gs = nullptr;
  if (grad_scale.has_value()) {
    TORCH_CHECK(grad_scale->is_cuda() && grad_scale->scalar_type() == at::kFloat && grad_scale->numel() == 1);
    gs = grad_scale->data_ptr<float>();
  }
  d9d::adamw_sr_multi(reinterpret_cast<const d9d::AdamTensorMeta*>(metas.data_ptr<int64_t>()),
                      reinterpret_cast<const int2*>(block_map.data_ptr<int>()), static_cast<int>(block_map.size(0)),
                      static_cast<float>(lr), static_cast<float>(beta1), static_cast<float>(beta2),
                      static_cast<float>(eps), static_cast<float>(weight_decay), static_cast<float>(bc1),
                      static_cast<float>(bc2), static_cast<uint64_t>(seed), gs, grad_bf16, state_bf16, cur_stream());
}

// ------------------------------------------------------------------ RoPE -------------------------
// x: [T, H, D] view (token stride arbitrary, head/dim contiguous); cos/sin: [max_pos, rope_dim] fp32; pos: [T] int64
Tensor rope_apply(const Tensor& x, const Tensor& cos_cache, const Tensor& sin_cache, const Tensor& pos, int64_t style,
                  bool inverse) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.stride(2) == 1 && x.stride(1) == x.size(2), "rope: heads must be contiguous");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 4 == 0 && x.stride(0) % 2 == 0,
              "rope: x and its token stride must be 4-byte aligned (the kernel moves bf16 pairs)");
  CHECK_CUDA_CONTIG(cos_cache); CHECK_CUDA_CONTIG(sin_cache); CHECK_CUDA_CONTIG(pos);
  TORCH_CHECK(cos_cache.scalar_type() == at::kFloat && sin_cache.scalar_type() == at::kFloat && pos.scalar_type() == at::kLong);
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t T = x.size(0);
  const int H = static_cast<int>(x.size(1)), D = static_cast<int>(x.size(2));
  Tensor out = at::empty({T, H, D}, x.options());
  d9d::rope_apply(x.data_ptr(), out.data_ptr(), cos_cache.data_ptr<float>(), sin_cache.data_ptr<float>(),
                  reinterpret_cast<const long long*>(pos.data_ptr<int64_t>()), T, H, D,
                  static_cast<int>(cos_cache.size(1)), x.stride(0), static_cast<int64_t>(H) * D,
                  static_cast<int>(style), inverse, cur_stream());
  return out;
}

// ------------------------------------------------------------------ MoE --------------------------
// -> (counts[E], seg_offsets[E+1], row_map[T*k], tile_group[capacity/128])   all int32, no host sync
std::tuple<Tensor, Tensor, Tensor, Tensor> moe_build_layout(const Tensor& topk_ids, int64_t num_experts, int64_t align,
                                                            int64_t capacity) {
  CHECK_CUDA_CONTIG(topk_ids);
  TORCH_CHECK(topk_ids.scalar_type() == at::kLong && topk_ids.dim() == 2);
  c10::cuda::CUDAGuard guard(topk_ids.device());
  const int64_t T = topk_ids.size(0), k = topk_ids.size(1);
  auto iopt = topk_ids.options().dtype(at::kInt);
  Tensor counts = at::empty({num_experts}, iopt), seg = at::empty({num_experts + 1}, iopt);
  Tensor row_map = at::empty({T * k}, iopt), tile_group = at::empty({capacity / 128}, iopt);
  Tensor scratch = at::empty({std::max<int64_t>(1, d9d::moe_layout_scratch_ints(T * k, static_cast<int>(num_experts)))}, iopt);
  d9d::moe_build_layout(reinterpret_cast<const long long*>(topk_ids.data_ptr<int64_t>()), T, static_cast<int>(k),
                        static_cast<int>(num_experts), static_cast<int>(align), capacity, counts.data_ptr<int>(),
                        seg.data_ptr<int>(), row_map.data_ptr<int>(), tile_group.data_ptr<int>(),
                        scratch.data_ptr<int>(), cur_stream());
  return {counts, seg, row_map, tile_group};
}

// x[T,H] (+ probs[T,k]) -> xp[capacity,H] (+ pp[capacity]); pad rows zeroed, rows past the last segment untouched
std::tuple<Tensor, Tensor> moe_permute(const Tensor& x, const c10::optional<Tensor>& probs, const Tensor& row_map,
                                       const Tensor& counts, const Tensor& seg_offsets, int64_t capacity) {
  CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(row_map); CHECK_ALIGNED16(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.size(1) % 8 == 0, "moe_permute: x must be bf16 [T, H], H % 8 == 0");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t T = x.size(0), H = x.size(1);
  const int k = static_cast<int>(row_map.numel() / std::max<int64_t>(T, 1));
  Tensor xp = at::empty({capacity, H}, x.options());
  Tensor pp;
  const float* pptr = nullptr;
  float* ppout = nullptr;
  if (probs.has_value()) {
    TORCH_CHECK(probs->is_contiguous() && probs->scalar_type() == at::kFloat);
    pp = at::empty({capacity}, x.options().dtype(at::kFloat));
    pptr = probs->data_ptr<float>();
    ppout = pp.data_ptr<float>();
  } else {
    pp = at::empty({0}, x.options().dtype(at::kFloat));
  }
  d9d::moe_permute(x.data_ptr(), pptr, row_map.data_ptr<int>(), xp.data_ptr(), ppout, T, k, static_cast<int>(H), cur_stream());
  d9d::moe_zero_pad(xp.data_ptr(), ppout, counts.data_ptr<int>(), seg_offsets.data_ptr<int>(),
                    static_cast<int>(counts.numel()), static_cast<int>(H), cur_stream());
  return {xp, pp};
}

// zero the pad rows [seg[e] + counts[e], seg[e+1]) of an aligned expert-sorted buffer (and of its per-row fp32 side array)
void moe_zero_pad(Tensor xp, const c10::optional<Tensor>& pp, const Tensor& counts, const Tensor& seg_offsets) {
  TORCH_CHECK(xp.is_cuda() && xp.dim() == 2 && xp.scalar_type() == at::kBFloat16 && xp.stride(1) == 1 && xp.stride(0) == xp.size(1));
  TORCH_CHECK(xp.size(1) % 8 == 0, "moe_zero_pad: xp rows must be a multiple of 8 elements");
  CHECK_ALIGNED16(xp);
  TORCH_CHECK(counts.scalar_type() == at::kInt && seg_offsets.scalar_type() == at::kInt && counts.is_contiguous() && seg_offsets.is_contiguous());
  TORCH_CHECK(seg_offsets.numel() == counts.numel() + 1, "moe_zero_pad: seg_offsets must have one entry more than counts");
  c10::cuda::CUDAGuard guard(xp.device());
  float* p = nullptr;
  if (pp.has_value()) {
    TORCH_CHECK(pp->scalar_type() == at::kFloat && pp->is_contiguous());
    p = pp->data_ptr<float>();
  }
  d9d::moe_zero_pad(xp.data_ptr(), p, counts.data_ptr<int>(), seg_offsets.data_ptr<int>(), static_cast<int>(counts.numel()),
                    static_cast<int>(xp.size(1)), cur_stream());
}

// y[T,H] = sum_j yp[row_map[t,j]];   with dpp: also dprobs[T,k] = dpp[row_map[t,j]]
std::tuple<Tensor, Tensor> moe_gather(const Tensor& yp, const c10::optional<Tensor>& dpp, const Tensor& row_map,
                                      int64_t T, int64_t k) {
  CHECK_CUDA_CONTIG(yp); CHECK_CUDA_CONTIG(row_map); CHECK_ALIGNED16(yp);
  TORCH_CHECK(yp.scalar_type() == at::kBFloat16 && yp.dim() == 2 && row_map.numel() == T * k);
  c10::cuda::CUDAGuard guard(yp.device());
  const int H = static_cast<int>(yp.size(1));
  Tensor y = at::empty({T, H}, yp.options());
  Tensor dprobs;
  if (dpp.has_value()) {
    dprobs = at::empty({T, k}, yp.options().dtype(at::kFloat));
    d9d::moe_permute_bwd(yp.data_ptr(), dpp->data_ptr<float>(), row_map.data_ptr<int>(), y.data_ptr(),
                         dprobs.data_ptr<float>(), T, static_cast<int>(k), H, cur_stream());
  } else {
    dprobs = at::empty({0}, yp.options().dtype(at::kFloat));
    d9d::moe_unpermute(yp.data_ptr(), row_map.data_ptr<int>(), y.data_ptr(), T, static_cast<int>(k), H, cur_stream());
  }
  return {y, dprobs};
}

// ------------------------------------------------------------------ grad utils -------------------
void sumsq_accumulate_(const Tensor& x, Tensor out) {
  CHECK_CUDA_CONTIG(x); CHECK_ALIGNED16(x);
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.numel() == 1);
  c10::cuda::CUDAGuard guard(x.device());
  d9d::sumsq_accumulate(x.data_ptr(), x.numel(), dtype_code(x), out.data_ptr<float>(), cur_stream());
}

void scale_inplace_(Tensor x, const Tensor& scale) {
  CHECK_CUDA_CONTIG(x); CHECK_ALIGNED16(x);
  TORCH_CHECK(scale.is_cuda() && scale.scalar_type() == at::kFloat && scale.numel() == 1);
  c10::cuda::CUDAGuard guard(x.device());
  d9d::scale_inplace(x.data_ptr(), x.numel(), dtype_code(x), scale.data_ptr<float>(), cur_stream());
}

}  // namespace

// ------------------------------------------------------------------ flash attention forward / backward
// q [B, Sq, Hq, Dqk] (or packed [total_q, Hq, Dqk] with cu_seqlens), k likewise with Hk heads, v like k but with Dv columns.
// window_left / window_right: -1 = unbounded.
static d9d::FlashAttnArgs fa_args(const Tensor& q, const Tensor& k, const Tensor& v, double scale, int64_t window_left,
                                  int64_t window_right, double softcap, const c10::optional<Tensor>& sink,
                                  const c10::optional<Tensor>& cu_q, const c10::optional<Tensor>& cu_k, int64_t max_q, int64_t max_k) {
  CHECK_CUDA_CONTIG(q); CHECK_CUDA_CONTIG(k); CHECK_CUDA_CONTIG(v);
  TORCH_CHECK(q.scalar_type() == at::kBFloat16 && k.scalar_type() == at::kBFloat16 && v.scalar_type() == at::kBFloat16,
              "flash_attn: bf16 tensors expected");
  TORCH_CHECK(k.dim() == v.dim() && k.dim() >= 1 && k.sizes().slice(0, k.dim() - 1) == v.sizes().slice(0, v.dim() - 1),
              "flash_attn: k and v must agree in every dimension but the last");
  TORCH_CHECK(q.dim() == k.dim() && q.size(-1) == k.size(-1), "flash_attn: q and k must have the same head dim");
  d9d::FlashAttnArgs a{};
  a.q = q.data_ptr(); a.k = k.data_ptr(); a.v = v.data_ptr();
  const bool varlen = cu_q.has_value();
  TORCH_CHECK(varlen == cu_k.has_value(), "flash_attn: cu_seqlens_q and cu_seqlens_k go together");
  if (varlen) {
    TORCH_CHECK(q.dim() == 3 && k.dim() == 3, "flash_attn (varlen): [total, H, D] tensors expected");
    TORCH_CHECK(cu_q->is_cuda() && cu_k->is_cuda() && cu_q->scalar_type() == at::kInt && cu_k->scalar_type() == at::kInt &&
                cu_q->is_contiguous() && cu_k->is_contiguous() && cu_q->numel() == cu_k->numel() && cu_q->numel() >= 2,
                "flash_attn (varlen): cu_seqlens must be int32 CUDA tensors of length B + 1");
    a.B = static_cast<int>(cu_q->numel() - 1);
    a.Sq = static_cast<int>(max_q); a.Sk = static_cast<int>(max_k);
    a.total_q = q.size(0); a.total_k = k.size(0);
    a.Hq = static_cast<int>(q.size(1)); a.Hk = static_cast<int>(k.size(1));
    a.Dqk = static_cast<int>(q.size(2)); a.Dv = static_cast<int>(v.size(2));
    a.cu_q = cu_q->data_ptr<int>(); a.cu_k = cu_k->data_ptr<int>();
  } else {
    TORCH_CHECK(q.dim() == 4 && k.dim() == 4, "flash_attn: [B, S, H, D] tensors expected");
    TORCH_CHECK(q.size(0) == k.size(0));
    a.B = static_cast<int>(q.size(0)); a.Sq = static_cast<int>(q.size(1)); a.Sk = static_cast<int>(k.size(1));
    a.Hq = static_cast<int>(q.size(2)); a.Hk = static_cast<int>(k.size(2));
    a.Dqk = static_cast<int>(q.size(3)); a.Dv = static_cast<int>(v.size(3));
    a.total_q = static_cast<long long>(a.B) * a.Sq; a.total_k = static_cast<long long>(a.B) * a.Sk;
  }
  a.window_left = static_cast<int>(window_left); a.window_right = static_cast<int>(window_right);
  a.scale = static_cast<float>(scale); a.softcap = static_cast<float>(softcap);
  if (sink.has_value()) {
    TORCH_CHECK(sink->is_cuda() && sink->scalar_type() == at::kFloat && sink->is_contiguous() && sink->numel() == a.Hq,
                "flash_attn: sink must be a contiguous fp32 [Hq] CUDA tensor");
    a.sink = sink->data_ptr<float>();
  }
  return a;
}

// out / dout: q's shape with v's head dim
static std::vector<int64_t> fa_out_shape(const d9d::FlashAttnArgs& a, const Tensor& q) {
  std::vector<int64_t> s = q.sizes().vec();
  s.back() = a.Dv;
  return s;
}

static Tensor fa_stats_like(const d9d::FlashAttnArgs& a, const Tensor& q) {
  return a.cu_q != nullptr ? at::empty({a.Hq, a.total_q}, q.options().dtype(at::kFloat))
                           : at::empty({a.B, a.Hq, a.Sq}, q.options().dtype(at::kFloat));
}

std::tuple<Tensor, Tensor> flash_attn_fwd(const Tensor& q, const Tensor& k, const Tensor& v, double scale, int64_t window_left,
                                          int64_t window_right, double softcap, const c10::optional<Tensor>& sink,
                                          const c10::optional<Tensor>& cu_q, const c10::optional<Tensor>& cu_k, int64_t max_q,
                                          int64_t max_k) {
  c10::cuda::CUDAGuard guard(q.device());
  d9d::FlashAttnArgs a = fa_args(q, k, v, scale, window_left, window_right, softcap, sink, cu_q, cu_k, max_q, max_k);
  Tensor out = at::empty(fa_out_shape(a, q), q.options());
  Tensor lse = fa_stats_like(a, q);
  a.out = out.data_ptr();
  a.lse = lse.data_ptr<float>();
  d9d::flash_attn_fwd(a, cur_stream());
  return {out, lse};
}

std::tuple<Tensor, Tensor, Tensor, Tensor> flash_attn_bwd(const Tensor& dout, const Tensor& q, const Tensor& k, const Tensor& v,
                                                          const Tensor& out, const Tensor& lse, double scale, int64_t window_left,
                                                          int64_t window_right, double softcap, const c10::optional<Tensor>& cu_q,
                                                          const c10::optional<Tensor>& cu_k, int64_t max_q, int64_t max_k,
                                                          const c10::optional<Tensor>& dlse) {
  c10::cuda::CUDAGuard guard(q.device());
  CHECK_CUDA_CONTIG(dout); CHECK_CUDA_CONTIG(out); CHECK_CUDA_CONTIG(lse);
  TORCH_CHECK(dout.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16 && lse.scalar_type() == at::kFloat);
  d9d::FlashAttnArgs a = fa_args(q, k, v, scale, window_left, window_right, softcap, c10::nullopt, cu_q, cu_k, max_q, max_k);
  const std::vector<int64_t> out_shape = fa_out_shape(a, q);
  TORCH_CHECK(dout.sizes() == c10::IntArrayRef(out_shape) && out.sizes() == c10::IntArrayRef(out_shape),
              "flash_attn_bwd: dout / out must have q's shape with v's head dim");
  Tensor delta = fa_stats_like(a, q);
  TORCH_CHECK(lse.numel() == delta.numel(), "flash_attn_bwd: lse has the wrong shape");
  Tensor dq = at::empty_like(q), dk = at::empty_like(k), dv = at::empty_like(v);
  a.out = out.data_ptr();
  a.dout = dout.data_ptr();
  a.lse = lse.data_ptr<float>();
  a.delta = delta.data_ptr<float>();
  a.dq = dq.data_ptr(); a.dk = dk.data_ptr(); a.dv = dv.data_ptr();
  d9d::flash_attn_bwd_delta(a, cur_stream());
  if (dlse.has_value()) delta.sub_(dlse->reshape(delta.sizes()));  // d(lse)/dS = P folds into the row statistic
  d9d::flash_attn_bwd(a, cur_stream());
  return {dq, dk, dv, delta};
}

// ------------------------------------------------------------------ fused q/k RMSNorm + RoPE
static void check_qk(const Tensor& q, const Tensor& k) {
  TORCH_CHECK(q.is_cuda() && k.is_cuda() && q.dim() == 3 && k.dim() == 3 && q.scalar_type() == at::kBFloat16 &&
              k.scalar_type() == at::kBFloat16, "qk_norm_rope: q/k must be bf16 [T, H, D]");
  TORCH_CHECK(q.stride(2) == 1 && k.stride(2) == 1 && q.stride(1) == q.size(2) && k.stride(1) == k.size(2) &&
              q.size(0) == k.size(0) && q.size(2) == k.size(2), "qk_norm_rope: heads must be densely packed");
  CHECK_ALIGNED16(q); CHECK_ALIGNED16(k);
  TORCH_CHECK(q.stride(0) % 8 == 0 && k.stride(0) % 8 == 0, "qk_norm_rope: token strides must be multiples of 8 elements");
}

static void check_qk_params(const Tensor& q, const Tensor& wq, const Tensor& wk, const Tensor& cos_t, const Tensor& sin_t) {
  CHECK_CUDA_CONTIG(wq); CHECK_CUDA_CONTIG(wk); CHECK_CUDA_CONTIG(cos_t); CHECK_CUDA_CONTIG(sin_t);
  CHECK_ALIGNED16(wq); CHECK_ALIGNED16(wk); CHECK_ALIGNED16(cos_t); CHECK_ALIGNED16(sin_t);
  TORCH_CHECK(wq.scalar_type() == at::kBFloat16 && wk.scalar_type() == at::kBFloat16 && cos_t.scalar_type() == at::kFloat &&
              sin_t.scalar_type() == at::kFloat, "qk_norm_rope: bf16 weights and fp32 cos / sin required");
  const int64_t T = q.size(0), D = q.size(2), rope_dim = cos_t.size(-1);
  TORCH_CHECK(cos_t.numel() == T * rope_dim && sin_t.numel() == T * rope_dim, "qk_norm_rope: cos / sin must be [T, rope_dim]");
  TORCH_CHECK(wq.numel() == D && wk.numel() == D, "qk_norm_rope: weights must have head_dim elements");
}

std::tuple<Tensor, Tensor, Tensor> qk_norm_rope_fwd(const Tensor& q, const Tensor& k, const Tensor& wq, const Tensor& wk,
                                                    const Tensor& cos_t, const Tensor& sin_t, double eps, bool zero_centered,
                                                    int64_t style) {
  check_qk(q, k);
  check_qk_params(q, wq, wk, cos_t, sin_t);
  c10::cuda::CUDAGuard guard(q.device());
  const int64_t T = q.size(0), Hq = q.size(1), Hk = k.size(1), D = q.size(2), rope_dim = cos_t.size(-1);
  Tensor qo = at::empty({T, Hq, D}, q.options()), ko = at::empty({T, Hk, D}, k.options());
  Tensor inv = at::empty({T, Hq + Hk}, q.options().dtype(at::kFloat));
  d9d::qk_norm_rope_fwd(q.data_ptr(), k.data_ptr(), wq.data_ptr(), wk.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), T,
                        static_cast<int>(Hq), static_cast<int>(Hk), static_cast<int>(D), static_cast<int>(rope_dim), q.stride(0),
                        k.stride(0), static_cast<float>(eps), zero_centered, static_cast<int>(style), qo.data_ptr(), ko.data_ptr(),
                        inv.data_ptr<float>(), cur_stream());
  return {qo, ko, inv};
}

std::tuple<Tensor, Tensor, Tensor, Tensor> qk_norm_rope_bwd(const Tensor& dq_out, const Tensor& dk_out, const Tensor& q, const Tensor& k,
                                                            const Tensor& wq, const Tensor& wk, const Tensor& cos_t,
                                                            const Tensor& sin_t, const Tensor& inv_rms, bool zero_centered,
                                                            int64_t style) {
  check_qk(q, k);
  check_qk_params(q, wq, wk, cos_t, sin_t);
  CHECK_CUDA_CONTIG(dq_out); CHECK_CUDA_CONTIG(dk_out); CHECK_CUDA_CONTIG(inv_rms);
  CHECK_ALIGNED16(dq_out); CHECK_ALIGNED16(dk_out);
  TORCH_CHECK(dq_out.scalar_type() == at::kBFloat16 && dk_out.scalar_type() == at::kBFloat16 &&
              dq_out.numel() == q.numel() && dk_out.numel() == k.numel(), "qk_norm_rope bwd: dq_out / dk_out must match q / k");
  c10::cuda::CUDAGuard guard(q.device());
  const int64_t T = q.size(0), Hq = q.size(1), Hk = k.size(1), D = q.size(2), rope_dim = cos_t.size(-1);
  TORCH_CHECK(inv_rms.scalar_type() == at::kFloat && inv_rms.numel() == T * (Hq + Hk), "qk_norm_rope bwd: inv_rms must be fp32 [T, Hq + Hk]");
  Tensor dq = at::empty({T, Hq, D}, q.options()), dk = at::empty({T, Hk, D}, k.options());
  const int grid = d9d::qk_norm_rope_grid(T, static_cast<int>(Hq + Hk));
  auto fopt = q.options().dtype(at::kFloat);
  Tensor partial = at::empty({grid, 2, D}, fopt), dwq = at::empty({D}, fopt), dwk = at::empty({D}, fopt);
  d9d::qk_norm_rope_bwd(dq_out.data_ptr(), dk_out.data_ptr(), q.data_ptr(), k.data_ptr(), wq.data_ptr(), wk.data_ptr(),
                        cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), inv_rms.data_ptr<float>(), T, static_cast<int>(Hq),
                        static_cast<int>(Hk), static_cast<int>(D), static_cast<int>(rope_dim), q.stride(0), k.stride(0), zero_centered,
                        static_cast<int>(style), dq.data_ptr(), dk.data_ptr(), partial.data_ptr<float>(), dwq.data_ptr<float>(),
                        dwk.data_ptr<float>(), cur_stream());
  return {dq, dk, dwq, dwk};
}

// ------------------------------------------------------------------ MoE router
static bool router_sigmoid(c10::string_view score_function) {
  TORCH_CHECK(score_function == "softmax" || score_function == "sigmoid", "router: unknown score function ", score_function);
  return score_function == "sigmoid";
}

std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor> router_topk_fwd(const Tensor& logits, const c10::optional<Tensor>& bias,
                                                                   int64_t k, bool renorm, c10::string_view score_function,
                                                                   int64_t num_groups, int64_t topk_groups,
                                                                   double scaling_factor, int64_t num_seqs) {
  CHECK_CUDA_CONTIG(logits);
  TORCH_CHECK(logits.scalar_type() == at::kBFloat16 && logits.dim() == 2);
  const bool sigmoid = router_sigmoid(score_function);
  const int64_t T = logits.size(0), E = logits.size(1);
  TORCH_CHECK(num_seqs == 0 || (num_seqs > 0 && T % num_seqs == 0), "router fwd: the sequence count must be 0 (no "
              "statistics) or a positive divisor of the token count");
  const float* b = nullptr;
  if (bias.has_value()) {
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->scalar_type() == at::kFloat && bias->numel() == E);
    TORCH_CHECK(bias->device() == logits.device(), "router fwd: the bias must be on the logits' device");
    b = bias->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor idx = at::empty({T, k}, logits.options().dtype(at::kLong));
  Tensor probs = at::empty({T, k}, logits.options().dtype(at::kFloat));
  if (num_seqs == 0) {  // no statistics: undefined outputs (None in Python), so the plain call allocates nothing more
    d9d::router_topk_fwd(logits.data_ptr(), b, T, static_cast<int>(E), static_cast<int>(k), renorm, sigmoid,
                         static_cast<int>(num_groups), static_cast<int>(topk_groups), static_cast<float>(scaling_factor),
                         reinterpret_cast<long long*>(idx.data_ptr<int64_t>()), probs.data_ptr<float>(), 0, nullptr,
                         nullptr, nullptr, nullptr, nullptr, nullptr, cur_stream());
    return {idx, probs, Tensor(), Tensor(), Tensor()};
  }
  const int64_t parts = d9d::router_stat_parts(T, num_seqs);
  Tensor part_counts = at::empty({parts, E}, logits.options().dtype(at::kInt));
  Tensor part_scores = at::empty({parts, E}, logits.options().dtype(at::kFloat));
  Tensor part_lse2 = at::empty({parts}, logits.options().dtype(at::kFloat));
  Tensor counts = at::empty({num_seqs, E}, logits.options().dtype(at::kInt));
  Tensor score_sum = at::empty({num_seqs, E}, logits.options().dtype(at::kFloat));
  Tensor lse2_sum = at::empty({num_seqs}, logits.options().dtype(at::kFloat));
  d9d::router_topk_fwd(logits.data_ptr(), b, T, static_cast<int>(E), static_cast<int>(k), renorm, sigmoid,
                       static_cast<int>(num_groups), static_cast<int>(topk_groups), static_cast<float>(scaling_factor),
                       reinterpret_cast<long long*>(idx.data_ptr<int64_t>()), probs.data_ptr<float>(), num_seqs,
                       part_counts.data_ptr<int>(), part_scores.data_ptr<float>(), part_lse2.data_ptr<float>(),
                       counts.data_ptr<int>(), score_sum.data_ptr<float>(), lse2_sum.data_ptr<float>(), cur_stream());
  return {idx, probs, counts, score_sum, lse2_sum};
}

// balance_grad [B, E] (B dividing T): the balance gradient row of each sequence of T / B tokens
Tensor router_topk_bwd(const Tensor& logits, const Tensor& idx, const Tensor& dprobs, bool renorm,
                       c10::string_view score_function, double scaling_factor, const c10::optional<Tensor>& balance_grad,
                       double z_coef) {
  CHECK_CUDA_CONTIG(logits); CHECK_CUDA_CONTIG(idx); CHECK_CUDA_CONTIG(dprobs);
  TORCH_CHECK(logits.scalar_type() == at::kBFloat16 && idx.scalar_type() == at::kLong && dprobs.scalar_type() == at::kFloat);
  const bool sigmoid = router_sigmoid(score_function);
  TORCH_CHECK(logits.dim() == 2 && idx.dim() == 2 && idx.size(0) == logits.size(0) && dprobs.sizes() == idx.sizes(),
              "router bwd: idx and dprobs must be [T, k] for logits [T, E]");
  TORCH_CHECK(idx.device() == logits.device() && dprobs.device() == logits.device(),
              "router bwd: all operands must be on the logits' device");
  const int64_t T = logits.size(0), E = logits.size(1), k = idx.size(1);
  const float* g = nullptr;
  int64_t B = 0;
  if (balance_grad.has_value()) {
    CHECK_CUDA_CONTIG((*balance_grad));
    TORCH_CHECK(balance_grad->scalar_type() == at::kFloat && balance_grad->dim() == 2 && balance_grad->size(1) == E,
                "router bwd: the balance gradient must be fp32 [B, E]");
    TORCH_CHECK(balance_grad->device() == logits.device(), "router bwd: all operands must be on the logits' device");
    B = balance_grad->size(0);
    TORCH_CHECK(B > 0 && T % B == 0, "router bwd: the balance gradient's row count must be a positive divisor of the "
                "token count");
    g = balance_grad->data_ptr<float>();
  }
  TORCH_CHECK(z_coef == 0.0 || (g && !sigmoid), "router bwd: the z-loss is defined for softmax routers only, with a "
              "balance gradient");
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor out = at::empty_like(logits);
  d9d::router_topk_bwd(logits.data_ptr(), reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()), dprobs.data_ptr<float>(),
                       T, static_cast<int>(E), static_cast<int>(k), renorm, sigmoid, static_cast<float>(scaling_factor), g,
                       B, static_cast<float>(z_coef), out.data_ptr(), cur_stream());
  return out;
}

// ------------------------------------------------------------------ tensor-parallel GEMMs with fused communication
// peer pointer lists come from torch.distributed._symmetric_memory (handle.buffer_ptrs) plus a byte offset.
static std::vector<const void*> to_ptrs(at::IntArrayRef v) {
  std::vector<const void*> out;
  out.reserve(v.size());
  for (int64_t p : v) out.push_back(reinterpret_cast<const void*>(p));
  return out;
}

// d[M,N] = all_gather(a_shards)[M,K] · B ; every peer holds a_shard[rows_local, K] (bf16, leading dim lda)
void gemm_ag_a(at::IntArrayRef a_peer_ptrs, int64_t rows_local, int64_t lda, int64_t block_rows, const Tensor& b, Tensor d,
               bool b_mn, int64_t block_n) {
  TORCH_CHECK(b.is_cuda() && d.is_cuda() && b.dim() == 2 && d.dim() == 2 && b.stride(1) == 1 && d.stride(1) == 1);
  TORCH_CHECK(b.scalar_type() == at::kBFloat16 && d.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(d.device());
  auto ptrs = to_ptrs(a_peer_ptrs);
  d9d::GemmArgs g;
  g.mode = DENSE; g.a_mn = false; g.b_mn = b_mn; g.epi = EPI_BF16;
  g.M = static_cast<int>(d.size(0)); g.N = static_cast<int>(d.size(1));
  g.K = static_cast<int>(b_mn ? b.size(0) : b.size(1));
  TORCH_CHECK((b_mn ? b.size(1) : b.size(0)) == g.N, "gemm_ag_a: N mismatch");
  TORCH_CHECK(rows_local * static_cast<int64_t>(ptrs.size()) == g.M, "gemm_ag_a: shards do not add up to M");
  g.B = b.data_ptr(); g.D = d.data_ptr(); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.comm = COMM_AG_A; g.comm_world = static_cast<int>(ptrs.size()); g.comm_block_rows = static_cast<int>(block_rows);
  g.comm_peer_ptrs = ptrs.data(); g.comm_rows_local = rows_local; g.comm_ld = lda;
  check_block_n(block_n, false, "gemm_ag_a");
  g.block_n = static_cast<int>(block_n);
  d9d::gemm_comm(g, cur_stream());
}

// d[M,N] = a[M,K] · B where a is a local buffer whose shards (owner(row) per the block mapping) arrive asynchronously:
// the GEMM starts with this rank's shard and waits on flags[owner] (int32, non-zero = landed) before touching another one
void gemm_wait_a(const Tensor& a, const Tensor& flags, int64_t rank, int64_t block_rows, const Tensor& b, Tensor d, bool b_mn,
                 int64_t spare_sms, int64_t block_n) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && d.is_cuda() && a.dim() == 2 && b.dim() == 2 && d.dim() == 2);
  TORCH_CHECK(a.stride(1) == 1 && b.stride(1) == 1 && d.stride(1) == 1);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16 && d.scalar_type() == at::kBFloat16);
  TORCH_CHECK(flags.is_cuda() && flags.scalar_type() == at::kInt && flags.is_contiguous());
  c10::cuda::CUDAGuard guard(d.device());
  d9d::GemmArgs g;
  g.mode = DENSE; g.a_mn = false; g.b_mn = b_mn; g.epi = EPI_BF16;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1));
  g.N = static_cast<int>(b_mn ? b.size(1) : b.size(0));
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == g.K && d.size(0) == g.M && d.size(1) == g.N, "gemm_wait_a: shape mismatch");
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.D = d.data_ptr();
  g.lda = a.stride(0); g.ldb = b.stride(0); g.ldd = d.stride(0);
  g.comm = COMM_WAIT_A; g.comm_world = static_cast<int>(flags.numel()); g.comm_block_rows = static_cast<int>(block_rows);
  g.comm_rank = static_cast<int>(rank); g.comm_flags = flags.data_ptr<int>();
  g.comm_spare_sms = static_cast<int>(spare_sms);
  check_block_n(block_n, false, "gemm_wait_a");
  g.block_n = static_cast<int>(block_n);
  d9d::gemm_comm(g, cur_stream());
}

// d_shards[owner][rows_local, N] += (a[M,K] · B) rows owned by `owner` (bf16 reduce-add over NVLink)
void gemm_rs_d(const Tensor& a, const Tensor& b, at::IntArrayRef d_peer_ptrs, int64_t rows_local, int64_t ldd, int64_t block_rows,
               bool b_mn, int64_t block_n) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.dim() == 2 && b.dim() == 2 && a.stride(1) == 1 && b.stride(1) == 1);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(a.device());
  auto ptrs = to_ptrs(d_peer_ptrs);
  d9d::GemmArgs g;
  g.mode = DENSE; g.a_mn = false; g.b_mn = b_mn; g.epi = EPI_BF16_ACC;
  g.M = static_cast<int>(a.size(0)); g.K = static_cast<int>(a.size(1));
  g.N = static_cast<int>(b_mn ? b.size(1) : b.size(0));
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == g.K, "gemm_rs_d: K mismatch");
  TORCH_CHECK(rows_local * static_cast<int64_t>(ptrs.size()) == g.M, "gemm_rs_d: shards do not add up to M");
  g.A = a.data_ptr(); g.B = b.data_ptr(); g.lda = a.stride(0); g.ldb = b.stride(0);
  g.comm = COMM_RS_D; g.comm_world = static_cast<int>(ptrs.size()); g.comm_block_rows = static_cast<int>(block_rows);
  g.comm_peer_ptrs = ptrs.data(); g.comm_rows_local = rows_local; g.comm_ld = ldd;
  check_block_n(block_n, false, "gemm_rs_d");
  g.block_n = static_cast<int>(block_n);
  d9d::gemm_comm(g, cur_stream());
}

// d[M,N] (+)= A^T · B over the token dim where one operand ([tokens, M] or [tokens, N], MN-major) is sharded by tokens
void gemm_ag_k(const Tensor& local, at::IntArrayRef peer_ptrs, bool peer_is_a, int64_t rows_local, int64_t peer_ld,
               int64_t block_rows, Tensor d, bool accumulate, int64_t block_n, int64_t k_splits) {
  TORCH_CHECK(local.is_cuda() && d.is_cuda() && local.dim() == 2 && d.dim() == 2 && local.stride(1) == 1 && d.stride(1) == 1);
  TORCH_CHECK(local.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(d.device());
  auto ptrs = to_ptrs(peer_ptrs);
  d9d::GemmArgs g;
  g.mode = DENSE; g.a_mn = true; g.b_mn = true;
  g.M = static_cast<int>(d.size(0)); g.N = static_cast<int>(d.size(1)); g.K = static_cast<int>(local.size(0));
  TORCH_CHECK(rows_local * static_cast<int64_t>(ptrs.size()) == g.K, "gemm_ag_k: shards do not add up to the token dim");
  TORCH_CHECK(local.size(1) == (peer_is_a ? g.N : g.M), "gemm_ag_k: local operand width mismatch");
  if (peer_is_a) { g.B = local.data_ptr(); g.ldb = local.stride(0); }
  else { g.A = local.data_ptr(); g.lda = local.stride(0); }
  g.D = d.data_ptr(); g.ldd = d.stride(0);
  g.epi = epi_for(d, accumulate);
  g.comm = peer_is_a ? COMM_AG_KA : COMM_AG_KB; g.comm_world = static_cast<int>(ptrs.size()); g.comm_block_rows = static_cast<int>(block_rows);
  g.comm_peer_ptrs = ptrs.data(); g.comm_rows_local = rows_local; g.comm_ld = peer_ld;
  check_block_n(block_n, false, "gemm_ag_k");
  TORCH_CHECK(k_splits >= 0, "gemm_ag_k: k_splits must be >= 0");
  TORCH_CHECK(k_splits <= 1 || g.epi == EPI_F32_ACC, "gemm_ag_k: k_splits needs an fp32 output with accumulate=True");
  g.block_n = static_cast<int>(block_n);
  g.k_splits = static_cast<int>(k_splits);
  d9d::gemm_comm(g, cur_stream());
}

// ------------------------------------------------------------------ expert-parallel exchange over NVLink
void ep_push(const Tensor& x, const c10::optional<Tensor>& probs, const Tensor& dest_rank, const Tensor& dest_row, int64_t peer_ptrs_dev,
             int64_t off_x, int64_t off_p, int64_t k) {
  CHECK_CUDA_CONTIG(x); CHECK_CUDA_CONTIG(dest_rank); CHECK_CUDA_CONTIG(dest_row);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && dest_rank.scalar_type() == at::kInt && dest_row.scalar_type() == at::kInt);
  TORCH_CHECK(dest_rank.numel() == x.size(0) * k && dest_row.numel() == x.size(0) * k, "ep_push: one destination per (token, slot) pair");
  c10::cuda::CUDAGuard guard(x.device());
  const float* pr = nullptr;
  if (probs.has_value()) {
    TORCH_CHECK(probs->is_cuda() && probs->is_contiguous() && probs->scalar_type() == at::kFloat && probs->numel() == dest_row.numel());
    pr = probs->data_ptr<float>();
  }
  d9d::ep_push(x.data_ptr(), pr, dest_rank.data_ptr<int>(), dest_row.data_ptr<int>(), reinterpret_cast<void* const*>(peer_ptrs_dev), off_x,
               off_p, dest_row.numel(), static_cast<int>(k), static_cast<int>(x.size(1)), cur_stream());
}

std::tuple<Tensor, Tensor> ep_pull_sum(int64_t peer_ptrs_dev, int64_t off_y, int64_t off_dp, const Tensor& dest_rank, const Tensor& dest_row,
                                       int64_t T, int64_t k, int64_t H, bool with_dprobs) {
  CHECK_CUDA_CONTIG(dest_rank); CHECK_CUDA_CONTIG(dest_row);
  TORCH_CHECK(dest_rank.scalar_type() == at::kInt && dest_row.scalar_type() == at::kInt && dest_row.numel() == T * k);
  c10::cuda::CUDAGuard guard(dest_row.device());
  Tensor y = at::empty({T, H}, dest_row.options().dtype(at::kBFloat16));
  Tensor dprobs = at::empty({with_dprobs ? T : 0, k}, dest_row.options().dtype(at::kFloat));
  d9d::ep_pull_sum(reinterpret_cast<void* const*>(peer_ptrs_dev), off_y, off_dp, dest_rank.data_ptr<int>(), dest_row.data_ptr<int>(),
                   y.data_ptr(), with_dprobs ? dprobs.data_ptr<float>() : nullptr, T, static_cast<int>(k), static_cast<int>(H), cur_stream());
  return {y, dprobs};
}

// ------------------------------------------------------------------ NVLink data-parallel optimizer -----------
// `peer_ptrs_dev` / `multicast_ptr` come from torch.distributed._symmetric_memory (buffer_ptrs_dev, multicast_ptr).
void nvl_reduce_shard_(Tensor own_grad, int64_t peer_ptrs_dev, int64_t multicast_ptr, int64_t begin, int64_t end,
                       int64_t world, int64_t rank, Tensor sumsq) {
  CHECK_CUDA_CONTIG(own_grad); CHECK_CUDA_CONTIG(sumsq);
  TORCH_CHECK(own_grad.scalar_type() == at::kFloat && sumsq.scalar_type() == at::kFloat);
  TORCH_CHECK(0 <= begin && begin <= end && end <= own_grad.numel(), "nvl_reduce_shard_: bad shard bounds");
  c10::cuda::CUDAGuard guard(own_grad.device());
  d9d::nvl_reduce_shard(reinterpret_cast<const float* const*>(peer_ptrs_dev), reinterpret_cast<const float*>(multicast_ptr),
                        own_grad.data_ptr<float>(), begin, end, static_cast<int>(world), static_cast<int>(rank),
                        sumsq.data_ptr<float>(), cur_stream());
}

void nvl_adamw_shard_(Tensor own_param, const Tensor& own_grad, Tensor exp_avg, Tensor exp_avg_sq, int64_t peer_ptrs_dev,
                      int64_t multicast_ptr, int64_t begin, int64_t end, int64_t world, int64_t rank, double lr,
                      double beta1, double beta2, double eps, double weight_decay, double bias_corr1, double bias_corr2,
                      int64_t seed, const c10::optional<Tensor>& grad_scale) {
  CHECK_CUDA_CONTIG(own_param); CHECK_CUDA_CONTIG(own_grad); CHECK_CUDA_CONTIG(exp_avg); CHECK_CUDA_CONTIG(exp_avg_sq);
  TORCH_CHECK(own_param.scalar_type() == at::kBFloat16 && own_grad.scalar_type() == at::kFloat);
  TORCH_CHECK(exp_avg.scalar_type() == exp_avg_sq.scalar_type() &&
              (exp_avg.scalar_type() == at::kBFloat16 || exp_avg.scalar_type() == at::kFloat));
  TORCH_CHECK(0 <= begin && begin <= end && end <= own_param.numel() && end <= own_grad.numel(), "nvl_adamw_shard_: bad shard bounds");
  TORCH_CHECK(exp_avg.numel() >= end - begin && exp_avg_sq.numel() >= end - begin, "nvl_adamw_shard_: state smaller than shard");
  c10::cuda::CUDAGuard guard(own_param.device());
  const float* gs = nullptr;
  if (grad_scale.has_value()) {
    TORCH_CHECK(grad_scale->is_cuda() && grad_scale->scalar_type() == at::kFloat);
    gs = grad_scale->data_ptr<float>();
  }
  d9d::nvl_adamw_shard(reinterpret_cast<void* const*>(peer_ptrs_dev), reinterpret_cast<void*>(multicast_ptr), own_param.data_ptr(),
                       own_grad.data_ptr<float>(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(), begin, end,
                       static_cast<int>(world), static_cast<int>(rank), static_cast<float>(lr), static_cast<float>(beta1),
                       static_cast<float>(beta2), static_cast<float>(eps), static_cast<float>(weight_decay),
                       static_cast<float>(bias_corr1), static_cast<float>(bias_corr2), static_cast<uint64_t>(seed), gs,
                       exp_avg.scalar_type() == at::kBFloat16, cur_stream());
}

TORCH_LIBRARY(d9d_b200, m) {
  m.def("gemm(Tensor a, Tensor b, Tensor(a!) d, bool a_mn, bool b_mn, bool accumulate, int ctas=0, int block_n=0, int k_splits=0) -> ()");
  m.def("gemm_set_pair_mode(int mode) -> int", &gemm_set_pair_mode);
  m.def("gemm_grouped_m(Tensor a, Tensor b, Tensor(a!) d, Tensor tile_group, bool b_mn, bool accumulate=False, int block_n=0) -> ()");
  m.def("gemm_grouped_k(Tensor a, Tensor b, Tensor(a!) d, Tensor group_offsets, bool accumulate, int block_n=0) -> ()");
  m.def("ce_forward(Tensor h, Tensor w, Tensor target, int ignore_index) -> (Tensor, Tensor)");
  m.def("ce_forward_ex(Tensor h, Tensor w, Tensor target, int ignore_index, Tensor? bias=None, float softcap=0.0, int col_offset=0) -> (Tensor, Tensor, Tensor)");
  m.def("ce_dlogits(Tensor h, Tensor w, Tensor target, Tensor lse, Tensor grad, Tensor(a!) out, int ignore_index, Tensor? bias=None, float softcap=0.0, int col_offset=0) -> ()");
  m.def("ce_forward_reg(Tensor h, Tensor w, Tensor target, int ignore_index, Tensor? bias=None, float softcap=0.0, int col_offset=0) -> (Tensor, Tensor, Tensor, Tensor)");
  m.def("ce_dlogits_reg(Tensor h, Tensor w, Tensor target, Tensor lse, Tensor grad, Tensor(a!) out, int ignore_index, float z_loss_coef, float label_smoothing, int num_classes, Tensor? bias=None, float softcap=0.0, int col_offset=0) -> ()");
  m.def("quantize_rowwise(Tensor x) -> (Tensor, Tensor)");
  m.def("quantize_colwise_t(Tensor x) -> (Tensor, Tensor)");
  m.def("quantize_mx(Tensor x) -> (Tensor, Tensor)");
  m.def("gemm_fp8(Tensor a, Tensor b, Tensor? scale_a, Tensor? scale_b, float scalar, Tensor(a!) d) -> ()");
  m.def("gemm_mxfp8(Tensor a, Tensor sfa, Tensor b, Tensor sfb, Tensor(a!) d) -> ()");
  m.def("quantize_colwise_t_batched(Tensor x) -> (Tensor, Tensor)");
  m.def("quantize_segments_t(Tensor x, Tensor tile_group, Tensor seg_offsets, Tensor counts) -> (Tensor, Tensor)");
  m.def("gemm_fp8_grouped_m(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor(a!) d, Tensor tile_group, bool accumulate=False) -> ()");
  m.def("gemm_fp8_grouped_k(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor(a!) d, Tensor group_offsets, bool accumulate) -> ()");
  m.def("quantize_blockwise(Tensor x) -> (Tensor, Tensor)");
  m.def("quantize_blockwise_t(Tensor x) -> (Tensor, Tensor)");
  m.def("quantize_weight_blocks(Tensor w, bool transpose=False) -> (Tensor, Tensor)");
  m.def("gemm_fp8_blockwise(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor(a!) d) -> ()");
  m.def("quantize_expert_weight_blocks(Tensor w, bool transpose) -> (Tensor, Tensor)");
  m.def("quantize_blockwise_tiles(Tensor x, Tensor tile_group) -> (Tensor, Tensor)");
  m.def("quantize_blockwise_t_tiles(Tensor x, Tensor tile_group, Tensor seg_offsets, Tensor counts) -> (Tensor, Tensor)");
  m.def("gemm_fp8_blockwise_grouped_m(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor(a!) d, Tensor tile_group, bool accumulate=False) -> ()");
  m.def("gemm_fp8_blockwise_grouped_k(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor(a!) d, Tensor group_offsets, bool accumulate) -> ()");
  m.def("rms_norm_fwd(Tensor x, Tensor w, float eps, bool zero_centered) -> (Tensor, Tensor)");
  m.def("rms_norm_bwd(Tensor dout, Tensor x, Tensor w, Tensor inv_rms, bool zero_centered) -> (Tensor, Tensor)");
  m.def("silu_mul_fwd(Tensor x, Tensor y) -> Tensor");
  m.def("silu_mul_bwd(Tensor dout, Tensor x, Tensor y) -> (Tensor, Tensor)");
  m.def("silu_mul_probs_fwd(Tensor x, Tensor y, Tensor probs, Tensor? valid_rows=None) -> Tensor");
  m.def("silu_mul_probs_bwd(Tensor dout, Tensor x, Tensor y, Tensor probs, Tensor? valid_rows=None) -> (Tensor, Tensor, Tensor)");
  m.def("sr_copy_(Tensor(a!) dst, Tensor src, int seed) -> ()");
  m.def(
      "adamw_sr_multi_(Tensor metas, Tensor block_map, float lr, float beta1, float beta2, float eps, float "
      "weight_decay, int step, int seed, Tensor? grad_scale, bool grad_bf16, bool state_bf16) -> ()");
  m.def("rope_apply(Tensor x, Tensor cos_cache, Tensor sin_cache, Tensor pos, int style, bool inverse) -> Tensor");
  m.def("moe_build_layout(Tensor topk_ids, int num_experts, int align, int capacity) -> (Tensor, Tensor, Tensor, Tensor)");
  m.def("moe_permute(Tensor x, Tensor? probs, Tensor row_map, Tensor counts, Tensor seg_offsets, int capacity) -> (Tensor, Tensor)");
  m.def("moe_gather(Tensor yp, Tensor? dpp, Tensor row_map, int T, int k) -> (Tensor, Tensor)");
  m.def("sumsq_accumulate_(Tensor x, Tensor(a!) out) -> ()");
  m.def("moe_zero_pad(Tensor(a!) xp, Tensor? pp, Tensor counts, Tensor seg_offsets) -> ()");
  m.def("flash_attn_fwd(Tensor q, Tensor k, Tensor v, float scale, int window_left, int window_right, float softcap, Tensor? sink, Tensor? cu_q, Tensor? cu_k, int max_q, int max_k) -> (Tensor, Tensor)");
  m.def("flash_attn_bwd(Tensor dout, Tensor q, Tensor k, Tensor v, Tensor out, Tensor lse, float scale, int window_left, int window_right, float softcap, Tensor? cu_q, Tensor? cu_k, int max_q, int max_k, Tensor? dlse) -> (Tensor, Tensor, Tensor, Tensor)");
  m.def("qk_norm_rope_fwd(Tensor q, Tensor k, Tensor wq, Tensor wk, Tensor cos_t, Tensor sin_t, float eps, bool zero_centered, "
        "int style) -> (Tensor, Tensor, Tensor)");
  m.def("qk_norm_rope_bwd(Tensor dq_out, Tensor dk_out, Tensor q, Tensor k, Tensor wq, Tensor wk, Tensor cos_t, Tensor sin_t, "
        "Tensor inv_rms, bool zero_centered, int style) -> (Tensor, Tensor, Tensor, Tensor)");
  m.def("router_topk_fwd(Tensor logits, Tensor? bias, int k, bool renorm, str score_function, int num_groups, int topk_groups, "
        "float scaling_factor, int num_seqs) -> (Tensor, Tensor, Tensor, Tensor, Tensor)");
  m.def("router_topk_bwd(Tensor logits, Tensor idx, Tensor dprobs, bool renorm, str score_function, float scaling_factor, "
        "Tensor? balance_grad, float z_coef) -> Tensor");
  m.def("gemm_ag_a(int[] a_peer_ptrs, int rows_local, int lda, int block_rows, Tensor b, Tensor(a!) d, bool b_mn, int block_n=0) -> ()");
  m.def("gemm_wait_a(Tensor a, Tensor flags, int rank, int block_rows, Tensor b, Tensor(a!) d, bool b_mn, int spare_sms=0, "
        "int block_n=0) -> ()");
  m.def("gemm_rs_d(Tensor a, Tensor b, int[] d_peer_ptrs, int rows_local, int ldd, int block_rows, bool b_mn, int block_n=0) -> ()");
  m.def("gemm_ag_k(Tensor local, int[] peer_ptrs, bool peer_is_a, int rows_local, int peer_ld, int block_rows, Tensor(a!) d, "
        "bool accumulate, int block_n=0, int k_splits=0) -> ()");
  m.def("ep_push(Tensor x, Tensor? probs, Tensor dest_rank, Tensor dest_row, int peer_ptrs_dev, int off_x, int off_p, int k) -> ()");
  m.def("ep_pull_sum(int peer_ptrs_dev, int off_y, int off_dp, Tensor dest_rank, Tensor dest_row, int T, int k, int H, bool with_dprobs) "
        "-> (Tensor, Tensor)");
  m.def("nvl_reduce_shard_(Tensor(a!) own_grad, int peer_ptrs_dev, int multicast_ptr, int begin, int end, int world, int rank, "
        "Tensor(b!) sumsq) -> ()");
  m.def("nvl_adamw_shard_(Tensor(a!) own_param, Tensor own_grad, Tensor(b!) exp_avg, Tensor(c!) exp_avg_sq, int peer_ptrs_dev, "
        "int multicast_ptr, int begin, int end, int world, int rank, float lr, float beta1, float beta2, float eps, "
        "float weight_decay, float bias_corr1, float bias_corr2, int seed, Tensor? grad_scale) -> ()");
  m.def("scale_inplace_(Tensor(a!) x, Tensor scale) -> ()");
}

TORCH_LIBRARY_IMPL(d9d_b200, CUDA, m) {
  m.impl("gemm", &gemm);
  m.impl("gemm_grouped_m", &gemm_grouped_m);
  m.impl("gemm_grouped_k", &gemm_grouped_k);
  m.impl("ce_forward", &ce_forward);
  m.impl("ce_forward_ex", &ce_forward_ex);
  m.impl("ce_dlogits", &ce_dlogits);
  m.impl("ce_forward_reg", &ce_forward_reg);
  m.impl("ce_dlogits_reg", &ce_dlogits_reg);
  m.impl("quantize_rowwise", &quantize_rowwise);
  m.impl("quantize_colwise_t", &quantize_colwise_t);
  m.impl("quantize_mx", &quantize_mx);
  m.impl("gemm_fp8", &gemm_fp8);
  m.impl("gemm_mxfp8", &gemm_mxfp8);
  m.impl("quantize_colwise_t_batched", &quantize_colwise_t_batched);
  m.impl("quantize_segments_t", &quantize_segments_t);
  m.impl("gemm_fp8_grouped_m", &gemm_fp8_grouped_m);
  m.impl("gemm_fp8_grouped_k", &gemm_fp8_grouped_k);
  m.impl("quantize_blockwise", &quantize_blockwise);
  m.impl("quantize_blockwise_t", &quantize_blockwise_t);
  m.impl("quantize_weight_blocks", &quantize_weight_blocks);
  m.impl("gemm_fp8_blockwise", &gemm_fp8_blockwise);
  m.impl("quantize_expert_weight_blocks", &quantize_expert_weight_blocks);
  m.impl("quantize_blockwise_tiles", &quantize_blockwise_tiles);
  m.impl("quantize_blockwise_t_tiles", &quantize_blockwise_t_tiles);
  m.impl("gemm_fp8_blockwise_grouped_m", &gemm_fp8_blockwise_grouped_m);
  m.impl("gemm_fp8_blockwise_grouped_k", &gemm_fp8_blockwise_grouped_k);
  m.impl("rms_norm_fwd", &rms_norm_fwd);
  m.impl("rms_norm_bwd", &rms_norm_bwd);
  m.impl("silu_mul_fwd", &silu_mul_fwd);
  m.impl("silu_mul_bwd", &silu_mul_bwd);
  m.impl("silu_mul_probs_fwd", &silu_mul_probs_fwd);
  m.impl("silu_mul_probs_bwd", &silu_mul_probs_bwd);
  m.impl("sr_copy_", &sr_copy_);
  m.impl("adamw_sr_multi_", &adamw_sr_multi_);
  m.impl("rope_apply", &rope_apply);
  m.impl("moe_build_layout", &moe_build_layout);
  m.impl("moe_permute", &moe_permute);
  m.impl("moe_gather", &moe_gather);
  m.impl("sumsq_accumulate_", &sumsq_accumulate_);
  m.impl("moe_zero_pad", &moe_zero_pad);
  m.impl("flash_attn_fwd", &flash_attn_fwd);
  m.impl("flash_attn_bwd", &flash_attn_bwd);
  m.impl("qk_norm_rope_fwd", &qk_norm_rope_fwd);
  m.impl("qk_norm_rope_bwd", &qk_norm_rope_bwd);
  m.impl("router_topk_fwd", &router_topk_fwd);
  m.impl("router_topk_bwd", &router_topk_bwd);
  m.impl("gemm_ag_a", &gemm_ag_a);
  m.impl("gemm_wait_a", &gemm_wait_a);
  m.impl("gemm_rs_d", &gemm_rs_d);
  m.impl("gemm_ag_k", &gemm_ag_k);
  m.impl("ep_push", &ep_push);
  m.impl("ep_pull_sum", &ep_pull_sum);
  m.impl("nvl_reduce_shard_", &nvl_reduce_shard_);
  m.impl("nvl_adamw_shard_", &nvl_adamw_shard_);
  m.impl("scale_inplace_", &scale_inplace_);
}
