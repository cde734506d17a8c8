"""Self-test of the fp64 reference / error bound that the GEMM kernel tests rely on: it must accept correctly rounded
results and reject the faults a broken kernel produces."""

import pytest
import torch

from tests.gemm_reference import Canaried, assert_within, err_ratio, gemm_bound, matmul_ref, padded, shard_rows


def _case(M, N, K, a_mn=False, b_mn=False):
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(K, M, generator=g).bfloat16() if a_mn else torch.randn(M, K, generator=g).bfloat16()
    b = torch.randn(K, N, generator=g).bfloat16() if b_mn else torch.randn(N, K, generator=g).bfloat16()
    return a, b


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (129, 136, 520), (64, 200, 1024)])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_accepts_correctly_rounded(out_dtype, M, N, K, a_mn, b_mn):
    a, b = _case(M, N, K, a_mn, b_mn)
    prod, S = matmul_ref(a, b, a_mn, b_mn)
    ref, bound = gemm_bound(prod, S, K, out_dtype)
    assert err_ratio(ref.to(out_dtype), ref, bound) <= 1.0
    # fp32 accumulation in any order (here: torch's fp32 matmul) stays inside the accumulation term
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    assert_within((A @ B).to(out_dtype), ref, bound)


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_accepts_accumulate_and_split_k(out_dtype):
    M, N, K, splits = 96, 72, 1000, 5
    a, b = _case(M, N, K)
    d0 = torch.randn(M, N).to(out_dtype)
    prod, S = matmul_ref(a, b, False, False)
    ref, bound = gemm_bound(prod, S, K, out_dtype, d0=d0, k_splits=splits)
    if out_dtype == torch.bfloat16:
        got = (d0.float() + prod.float().bfloat16().float()).bfloat16()  # TMA reduce-add: rn(d0 + rn(acc))
    else:  # one fp32 partial per K slice, added to d0 in reverse order
        A, B = a.float(), b.float().t()
        got = d0.clone()
        for s in reversed(range(splits)):
            k0, k1 = s * K // splits, (s + 1) * K // splits
            got += A[:, k0:k1] @ B[k0:k1]
    assert_within(got, ref, bound)


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_rejects_faults(out_dtype):
    M, N, K = 129, 200, 520
    a, b = _case(M, N, K)
    prod, S = matmul_ref(a, b, False, False)
    ref, bound = gemm_bound(prod, S, K, out_dtype)
    good = ref.to(out_dtype)

    # one 64-deep k-block never accumulated
    A, B = a.double(), b.double().t()
    missing = (ref - A[:, 128:192] @ B[128:192]).to(out_dtype)
    assert err_ratio(missing, ref, bound) > 1.0

    # one element off by 3 bf16 ulps
    i, j = divmod(int(ref.abs().argmax()), N)
    off = good.clone()
    x = off[i, j].double()
    ulp = 2.0 ** (torch.floor(torch.log2(x.abs())) - 7)
    off[i, j] = (x + 3 * ulp * torch.sign(x)).to(out_dtype)
    assert err_ratio(off, ref, bound) > 1.0

    # two 8-column groups swapped
    sw = good.clone()
    sw[:, 16:24], sw[:, 40:48] = good[:, 40:48], good[:, 16:24]
    assert err_ratio(sw, ref, bound) > 1.0

    # a NaN
    nan = good.clone()
    nan[5, 7] = float("nan")
    assert err_ratio(nan, ref, bound) == float("inf")
    with pytest.raises(AssertionError):
        assert_within(nan, ref, bound)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("tma", [True, False])
def test_canaried_output_layout(dtype, tma):
    c = Canaried(5, 13, dtype, tma=tma, device="cpu")
    esz = c.buf.element_size()
    aligned = (c.view.data_ptr() % 16 == 0) and (c.view.stride(0) * esz % 16 == 0)
    assert aligned == tma
    c.view.fill_(1.0)
    c.assert_untouched()
    c.buf[0, 0] = 0.0
    with pytest.raises(AssertionError):
        c.assert_untouched()


def test_padded_operand_and_shards():
    x = padded(4, 24, 8, device="cpu")
    assert x.stride(0) == 32 and torch.isfinite(x.float()).all()
    assert torch.isnan(x.as_strided((4, 32), (32, 1))[:, 24:].float()).all()
    owners = shard_rows(torch.empty(12, 1), 3, 2)  # blocks of 2 rows, dealt round-robin to 3 ranks
    assert owners == [[0, 1, 6, 7], [2, 3, 8, 9], [4, 5, 10, 11]]
