"""CPU self-test of the fp8 models in ``tests/fp8_reference.py``: the e4m3 rounding model against torch's float8 cast,
the admissible-code range, the chain-length GEMM bound against a simulated reduced-precision accumulation, and the MX
scale packer against ``fp8.unpack_mx_scales``."""

import math

import pytest
import torch

from d9d_b200.kernel import fp8
from tests.fp8_reference import (
    DELTA, E4M3_MAX, FLT_MIN, U_CHAIN, admissible_codes, assert_codes_admissible, check_scales, code_rank, e4m3_values,
    gemm_bound, pack_mx_scales, rn_e4m3, scale_bounds,
)


def _all_finite_bf16() -> torch.Tensor:
    bits = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32).to(torch.int16)
    x = bits.view(torch.bfloat16)
    return x[torch.isfinite(x)]


def test_code_table():
    v = e4m3_values()
    assert torch.equal(v.float().to(fp8.FP8).view(torch.uint8)[:127], torch.arange(127, dtype=torch.uint8))
    assert float(v[0x7E]) == 448.0 and float(v[1]) == 2.0**-9 and math.isnan(float(v[0x7F])) and math.isnan(float(v[0xFF]))


@pytest.mark.parametrize("scale", [1.0, 2.0**-10, 0.3, 3.7e-3, 1.0 / 448, 2.0**20 / 7])
def test_rounding_model_matches_torch_cast_on_every_bf16_value(scale):
    x = _all_finite_bf16().double() * scale
    x = x[torch.isfinite(x)]
    mine = rn_e4m3(x)
    # torch's cast does not saturate (out-of-range values become NaN): clamp first, as the emulations do
    theirs = x.clamp(-E4M3_MAX, E4M3_MAX).float().to(fp8.FP8).view(torch.uint8).to(torch.int64)
    # the fp64 -> fp32 step above can round once more; compare where fp32 holds x exactly
    exact32 = x.float().double() == x
    assert torch.equal(mine[exact32], theirs[exact32])


def test_rounding_model_ties_saturation_and_signs():
    v = torch.tensor([0.0, -0.0, 2.0**-10, 2.0**-10 + 2.0**-40, 3 * 2.0**-10, 1.0625, 1.1875, 464.0, 1e30, -1e30, -2.0**-11], dtype=torch.float64)
    codes = rn_e4m3(v).tolist()
    assert codes == [0x00, 0x80, 0x00, 0x01, 0x02, 0x38, 0x3A, 0x7E, 0x7E, 0xFE, 0x80]


def test_code_rank_orders_by_value():
    v = e4m3_values()
    finite = torch.isfinite(v)
    codes = torch.arange(256)[finite]
    r = code_rank(codes)
    order = torch.argsort(v[finite], stable=True)
    assert bool((r[order][1:] >= r[order][:-1]).all())
    assert int(code_rank(torch.tensor([0x7F]))) > 126 and int(code_rank(torch.tensor([0xFF]))) < -126


def test_admissible_codes_bracket_the_exact_rounding():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(20000, generator=g) * torch.logspace(-30, 30, 20000)).bfloat16().double()
    s = (x.abs().max() / 448) * torch.rand(20000, generator=g, dtype=torch.float64).add(0.5)
    lo, hi = admissible_codes(x, s)
    r = code_rank(rn_e4m3(x / s))
    assert bool(((lo <= r) & (r <= hi)).all())
    # a perturbation of the quotient by 2^-22 (what rcp.approx and one fp32 rounding can do) stays inside
    for f in (1 - 2.0**-22, 1 + 2.0**-22):
        rp = code_rank(rn_e4m3(x / s * f))
        assert bool(((lo <= rp) & (rp <= hi)).all())
    # and the range is tight: only a handful of values sit within 2^-21 of a rounding boundary
    assert float((hi > lo).double().mean()) < 1e-3
    with pytest.raises(AssertionError):
        assert_codes_admissible(x, rn_e4m3(x / s * 1.07).to(torch.uint8), s, "off by 7 %")
    assert_codes_admissible(x, rn_e4m3(x / s).to(torch.uint8), s, "exact")


def test_flushed_elements_may_be_zero():
    x = torch.tensor([FLT_MIN / 2, -FLT_MIN / 4, FLT_MIN])
    s = torch.full_like(x, FLT_MIN)
    lo, hi = admissible_codes(x, s)
    assert lo[0] <= 0 <= hi[0] and lo[1] <= 0 <= hi[1]
    assert int(lo[2]) == int(hi[2]) == 0x38  # exactly 1.0


def test_scale_model():
    amax = torch.tensor([0.0, 448.0, 1.0, FLT_MIN, 447 * FLT_MIN, 3.3e38])
    lo, hi = scale_bounds(amax)
    assert float(lo[0]) == float(hi[0]) == 1.0
    assert float(lo[1]) <= 1.0 <= float(hi[1])
    assert float(lo[3]) == FLT_MIN and float(lo[4]) == FLT_MIN  # the floor
    s = torch.where(amax > 0, (amax / 448).clamp_min(FLT_MIN), torch.ones_like(amax)).float()
    check_scales(s, amax)
    with pytest.raises(AssertionError):
        check_scales(s * (1 + 2.0**-20), amax)
    with pytest.raises(AssertionError):
        check_scales(torch.tensor([0.0]), torch.tensor([1.0]))  # a flushed scale
    # the emulations follow the same rule
    x = torch.zeros(3, 16, dtype=torch.bfloat16)
    x[1, 3] = 5 * FLT_MIN
    x[2, 0] = 300.0
    _, se = fp8.quantize_rowwise_reference(x)
    check_scales(se, x.double().abs().amax(1))


def test_emulated_quantiser_codes_are_admissible():
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(64, 256, generator=g) * torch.logspace(-3, 3, 64)[:, None]).bfloat16()
    q, s = fp8.quantize_rowwise_reference(x)
    assert_codes_admissible(x, q, s[:, None], "rowwise emulation")


def test_chain_bound_covers_a_simulated_reduced_precision_chain():
    """Sum chains of length L rounding every partial sum to 14 significant bits (unit roundoff U_CHAIN), add the chains
    in fp32, scale: the result stays inside gemm_bound for L = 32, 128 and K."""
    g = torch.Generator().manual_seed(2)

    def rn_bits(v, bits):
        m, e = torch.frexp(v)
        return torch.ldexp(torch.round(m * 2.0**bits) / 2.0**bits, e)

    M, N, K = 8, 8, 1024
    a = rn_e4m3(torch.randn(M, K, generator=g, dtype=torch.float64) * 100)
    b = rn_e4m3(torch.randn(N, K, generator=g, dtype=torch.float64) * 100)
    A, B = e4m3_values()[a], e4m3_values()[b]
    sa, sb = torch.rand(M, 1, generator=g, dtype=torch.float64) + 0.5, torch.rand(1, N, generator=g, dtype=torch.float64) + 0.5
    ref = (A @ B.t()) * sa * sb
    S = (A.abs() @ B.abs().t()) * sa * sb
    for L in (32, 128, K):
        d = torch.zeros(M, N, dtype=torch.float32)
        for k0 in range(0, K, L):
            part = torch.zeros(M, N, dtype=torch.float64)
            for k in range(k0, k0 + L):
                part = rn_bits(part + A[:, k : k + 1] * B[:, k : k + 1].t(), 14)
            d = d + part.float()
        d = (d * sa.float()) * sb.float()
        bound = gemm_bound(ref, S, K, L, torch.float32)
        assert bool(((d.double() - ref).abs() <= bound).all()), L


def test_mx_packer_round_trips():
    g = torch.Generator().manual_seed(3)
    for rows, K in [(1, 128), (128, 256), (300, 512), (129, 128)]:
        e = torch.randint(-127, 128, (rows, K // 32), generator=g)
        sf = pack_mx_scales(e)
        assert sf.shape == ((rows + 127) // 128, K // 128, 512) and sf.dtype == torch.uint8
        assert torch.equal(fp8.unpack_mx_scales(sf, rows, K), e.to(torch.int32))
    # and matches the layout of the native quantiser's emulation: [2 * ceil(rows / 256)] blocks when asked for them
    sf = pack_mx_scales(e, row_blocks=4)
    assert sf.shape[0] == 4 and torch.equal(fp8.unpack_mx_scales(sf, 129, 128), e.to(torch.int32))
