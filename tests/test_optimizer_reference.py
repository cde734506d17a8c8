"""Self-test of the stochastic-rounding model and the AdamW bound that the optimizer kernel tests rely on.  CPU only.

The Philox model must reproduce Random123's published known-answer vectors, the rounding model must be unbiased and
monotone, a torch fp32 emulation of each kernel (also with its divisions and square roots off by their fast-math error)
must pass the checker at the kernel suite's sizes, and every fault a broken kernel could make must fail it."""

from __future__ import annotations

import pytest
import torch

from tests.optimizer_reference import (
    MASK32,
    adam_inputs,
    adamw_bits,
    bias_corrections,
    check_adamw,
    check_sr_exact,
    f32,
    f32_bits,
    from_bf16_bits,
    from_f32_bits,
    philox4x32_10,
    sr_bits,
    sr_copy_bits,
    stream_bits,
    tensor_positions,
)

CHUNK = 8192  # d9d::ADAM_CHUNK
ADAM_SIZES = [1, 7, 8, 9, 8191, 8192, 8193, 3 * CHUNK + 5, 100_003]
H100_SMS = 132
NVL_N = 3 * H100_SMS * 8 * 256 * 8 + 104  # three passes of nvl_adamw_shard's grid on an H100, plus a tail
NVL_BEGIN = 8 * 4099
HYPER = dict(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.1)
SEED = (1 << 33) + 977


# ----------------------------------------------------------------------------- Philox, rounding model
# Random123 kat_vectors, philox4x32 with 10 rounds: (counter words, key words, output words)
PHILOX_KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((MASK32,) * 4, (MASK32, MASK32), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", PHILOX_KAT)
def test_philox_known_answers(ctr, key, want):
    assert philox4x32_10(*ctr, *key).tolist() == list(want)


def _sr_inputs() -> torch.Tensor:
    """fp32 values between bf16 neighbours of every binade, both signs, denormals and zeros."""
    g = torch.Generator().manual_seed(5)
    e = torch.arange(0, 255, dtype=torch.int64)
    mant = torch.randint(0, 1 << 23, (255,), generator=g)
    bits = (e << 23) | mant
    bits = torch.cat([bits, bits | (1 << 31), torch.tensor([0, 1 << 31, 1, 0x7FFFFF, 0x7F7FFFFF, 0x3F808000])])
    return bits


def test_sr_model_exhaustive():
    """Over all 65,536 values of r: bf16-representable values never move, the mean of the outputs is x exactly (where no
    output overflows to inf), the outputs are the two bf16 neighbours of x, and the model is monotone in x."""
    bits = _sr_inputs()
    r = torch.arange(1 << 16, dtype=torch.int64)
    out = sr_bits(bits[:, None], r[None, :])  # [inputs, 65536]
    vals = from_bf16_bits(out).double()
    x = from_f32_bits(bits).double()
    exact = (bits & 0xFFFF) == 0
    assert bool((out[exact] == (bits[exact, None] >> 16)).all()), "a bf16 value moved"
    finite = torch.isfinite(vals).all(1)
    assert bool((vals[finite].mean(1) == x[finite]).all()), "SR is biased"
    assert torch.equal(~finite, (bits & 0x7FFFFFFF) > 0x7F7F0000), "only values above the bf16 maximum may reach inf"
    lo = bits >> 16
    assert bool(((out == lo[:, None]) | (out == lo[:, None] + 1)).all())
    pos = bits[(bits >> 31) == 0]
    order = pos.argsort()
    assert bool((sr_bits(pos[order][:, None], r[None, :]).diff(dim=0) >= 0).all()), "SR is not monotone"


def test_sr_model_nonfinite():
    nan_bits = torch.tensor([0x7F800001, 0xFF800001, 0x7FC00000, 0x7F810000, 0xFFFFFFFF])
    inf_bits = torch.tensor([0x7F800000, 0xFF800000])
    r = torch.full((5,), 0xFFFF)
    assert bool(torch.isnan(from_bf16_bits(sr_bits(nan_bits, r)).float()).all())
    assert sr_bits(inf_bits, r[:2]).tolist() == [0x7F80, 0xFF80]


def test_stream_layout():
    """Element e of a stream: counter e >> 3, word (e & 7) >> 1, low half if even."""
    seed = (1 << 40) + 3
    r = sr_copy_bits(24, seed)
    words = philox4x32_10(torch.arange(3), 0, 0, 0, seed & MASK32, seed >> 32)
    for e in range(24):
        w = int(words[e >> 3, (e & 7) >> 1])
        assert int(r[e]) == (w >> (16 * (e & 1))) & 0xFFFF


# ----------------------------------------------------------------------------- kernel emulations and faults
SR_FAULTS = ["round to nearest", "truncation", "halves swapped", "wrong word", "high seed word dropped",
             "NaN to inf"]
ADAM_FAULTS = ["round to nearest", "truncation", "p and m share a stream", "halves swapped", "wrong word",
               "rng_base ignored", "high counter word dropped", "high seed word dropped", "grad_scale ignored",
               "bias correction at step - 1", "weight decay after the update", "eps inside the square root"]
NVL_FAULTS = ["shard-local counter"]


def _faulty_bits(pos: torch.Tensor, key: int, fault: str | None, rng_base: int = 0) -> torch.Tensor:
    if fault == "truncation":
        return torch.zeros_like(pos)
    if fault == "halves swapped":
        pos = pos ^ 1
    elif fault == "wrong word":
        pos = pos ^ 2
    elif fault in ("rng_base ignored", "shard-local counter"):
        pos = pos - rng_base
    elif fault == "high counter word dropped":
        pos = pos & ((1 << 35) - 1)
    elif fault == "high seed word dropped":
        key &= MASK32
    return stream_bits(pos, key)


def _round(x: torch.Tensor, pos, key, fault, rng_base=0) -> torch.Tensor:
    if fault == "round to nearest":
        return x.bfloat16()
    bits = f32_bits(x)
    out = sr_bits(bits, _faulty_bits(pos, key, fault, rng_base))
    if fault == "NaN to inf":
        out = torch.where(torch.isnan(x), bits >> 16, out)
    return from_bf16_bits(out)


def emulate_sr_copy(src: torch.Tensor, seed: int, fault: str | None = None) -> torch.Tensor:
    return _round(src, torch.arange(src.numel()), seed, fault)


def _perturbed(x: torch.Tensor, gen: torch.Generator | None) -> torch.Tensor:
    """x moved by up to 2 ulp (the fast-math division and square root error) where it is finite and nonzero."""
    if gen is None:
        return x
    d = torch.randint(-2, 3, x.shape, generator=gen, dtype=torch.int32)
    moved = (x.view(torch.int32) + d).view(torch.float32)
    return torch.where((x != 0) & torch.isfinite(x), moved, x)


def emulate_adamw(p, g, m, v, pos, *, seed, lr, beta1, beta2, eps, wd, step, grad_scale=None, fault=None,
                  perturb: torch.Generator | None = None, rng_base: int = 0):
    """fp32 AdamW in the order of adamw_sr_kernel / nvl_adamw_shard_kernel; returns (p, m, v) as the kernel stores them."""
    F = lambda x: torch.tensor(f32(x), dtype=torch.float32)  # noqa: E731
    lr_, b1, b2, eps_, wd_ = F(lr), F(beta1), F(beta2), F(eps), F(wd)
    bc1, bc2 = bias_corrections(beta1, beta2, step - 1 if fault == "bias correction at step - 1" else step)
    gs = F(1.0 if grad_scale is None or fault == "grad_scale ignored" else grad_scale)
    gk = g.float() * gs
    c = 1 - lr_ * wd_
    pw = p.float()
    if fault != "weight decay after the update":
        pw = pw * c
    mn = b1 * m.float() + (1 - b1) * gk
    vn = b2 * v.float() + (1 - b2) * (gk * gk)
    mh = _perturbed(mn / F(bc1), perturb)
    vh = _perturbed(vn / F(bc2), perturb)
    den = _perturbed((vh + eps_).sqrt(), perturb) if fault == "eps inside the square root" \
        else _perturbed(vh.sqrt(), perturb) + eps_
    pw = pw - _perturbed((lr_ * mh) / den, perturb)
    if fault == "weight decay after the update":
        pw = pw * c
    m_key = seed if fault == "p and m share a stream" else seed + 42
    p_out = _round(pw, pos, seed, fault, rng_base)
    if m.dtype == torch.bfloat16:
        return p_out, _round(mn, pos, m_key, fault, rng_base), _round(vn, pos, seed + 67, fault, rng_base)
    return p_out, mn, vn


def _adam_launch(grad_dtype, state_dtype, seed_offset=0):
    """The tensors of one multi-tensor launch at ADAM_SIZES with their rng_base, as the launch plan lays them out; the
    first rng_base is 2^35 so that the high counter word is in use."""
    gen = torch.Generator().manual_seed(17 + seed_offset)
    out, base = [], 1 << 35
    for n in ADAM_SIZES:
        out.append((adam_inputs(n, grad_dtype, state_dtype, gen), base))
        base += (n + 7) // 8 * 8
    return out


def _check_launch(tensors, fault=None, perturb=None, grad_scale=0.37, step=3, **kw):
    hyper = {**HYPER, **kw}
    stats = []
    for (p, g, m, v), base in tensors:
        pos = tensor_positions(p.numel(), base)
        po, mo, vo = emulate_adamw(p, g, m, v, pos, seed=SEED, step=step, grad_scale=grad_scale, fault=fault,
                                   perturb=perturb, rng_base=base, **hyper)
        bc1, bc2 = bias_corrections(hyper["beta1"], hyper["beta2"], step)
        stats.append(check_adamw(po, mo, vo, p, g, m, v, pos, SEED, f"n={p.numel()}", bc1=bc1, bc2=bc2,
                                 grad_scale=grad_scale, **hyper))
    return stats


@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("perturb", [False, True])
def test_adamw_emulation_passes(grad_dtype, state_dtype, perturb):
    stats = _check_launch(_adam_launch(grad_dtype, state_dtype), perturb=torch.Generator().manual_seed(3) if perturb else None)
    n = sum(ADAM_SIZES)
    for k in stats[0]:
        if k.endswith("ambiguous"):
            assert sum(s[k] for s in stats) < n * 2.0**-10, (k, [s[k] for s in stats])


@pytest.mark.parametrize("perturb", [False, True])
def test_adamw_emulation_passes_edges(perturb):
    """beta1 = 0, wd = 0, step 1 and 1000, no grad_scale."""
    tensors = _adam_launch(torch.float32, torch.bfloat16, 1)
    gen = torch.Generator().manual_seed(4) if perturb else None
    _check_launch(tensors, perturb=gen, grad_scale=None, step=1, beta1=0.0)
    _check_launch(tensors, perturb=gen, step=1000, wd=0.0)


def _nvl_case(state_dtype):
    gen = torch.Generator().manual_seed(23)
    return adam_inputs(NVL_N, torch.float32, state_dtype, gen)


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_nvl_adamw_emulation_passes(state_dtype):
    p, g, m, v = _nvl_case(state_dtype)
    pos = NVL_BEGIN + torch.arange(NVL_N)
    bc1, bc2 = bias_corrections(HYPER["beta1"], HYPER["beta2"], 7)
    po, mo, vo = emulate_adamw(p, g, m, v, pos, seed=SEED, step=7, grad_scale=0.37,
                               perturb=torch.Generator().manual_seed(9), **HYPER)
    check_adamw(po, mo, vo, p, g, m, v, pos, SEED, "nvl", bc1=bc1, bc2=bc2, grad_scale=0.37, **HYPER)


def _sr_copy_faulty_source() -> torch.Tensor:
    bits = torch.cat([_sr_inputs(), torch.tensor([0x7F800001, 0xFF800001, 0x7FC00000, 0x7F800000])])
    return from_f32_bits(bits)


@pytest.mark.parametrize("fault", SR_FAULTS)
def test_sr_copy_fault_caught(fault):
    src = _sr_copy_faulty_source()
    seed = (1 << 32) + 5
    r = sr_copy_bits(src.numel(), seed)
    check_sr_exact(emulate_sr_copy(src, seed), src, r, "clean")
    with pytest.raises(AssertionError):
        check_sr_exact(emulate_sr_copy(src, seed, fault), src, r, fault)


@pytest.mark.parametrize("fault", ADAM_FAULTS)
def test_adamw_fault_caught(fault):
    with pytest.raises(AssertionError):
        _check_launch(_adam_launch(torch.float32, torch.bfloat16), fault=fault)


@pytest.mark.parametrize("fault", NVL_FAULTS)
def test_nvl_fault_caught(fault):
    n = 4096
    p, g, m, v = adam_inputs(n, torch.float32, torch.bfloat16, torch.Generator().manual_seed(2))
    pos = NVL_BEGIN + torch.arange(n)
    bc1, bc2 = bias_corrections(HYPER["beta1"], HYPER["beta2"], 7)
    po, mo, vo = emulate_adamw(p, g, m, v, pos, seed=SEED, step=7, fault=fault, rng_base=NVL_BEGIN, **HYPER)
    with pytest.raises(AssertionError):
        check_adamw(po, mo, vo, p, g, m, v, pos, SEED, fault, bc1=bc1, bc2=bc2, **HYPER)


def test_stream_keys_are_64_bit_sums():
    """seed + 42 carries into the key's high word for a seed just under 2^32."""
    seed = (1 << 32) - 20
    pos = torch.arange(64)
    _, rm, _ = adamw_bits(pos, seed)
    assert torch.equal(rm, stream_bits(pos, (1 << 32) + 22))
    assert not torch.equal(rm, stream_bits(pos, 22))
