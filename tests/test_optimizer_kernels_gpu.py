"""The stochastic-rounding copy and AdamW kernels (``ops/csrc/elementwise.cu``, ``ops/csrc/nvlink_optim.cu``) against
the exact model of their Philox streams and the fp64 AdamW reference of ``tests/optimizer_reference.py``.

Every rounding decision is predicted from (seed, counter), so the copy is checked bit for bit and an AdamW output is
checked exactly wherever the fp64 bound leaves one bf16 value possible (all but a small, reported fraction).  The
grid-stride kernels run at sizes computed from the SM count with the launchers' grid caps, so that every thread makes
three passes plus a ragged tail.  The NVLink kernels run with one replica, no peer table and no multicast mapping: that
is their arithmetic and their counter without any peer traffic."""

from __future__ import annotations

import pytest
import torch

from tests.gemm_reference import assert_within
from tests.optimizer_reference import (
    adam_inputs,
    adamw_ref,
    bias_corrections,
    check_adamw,
    check_sr_exact,
    from_f32_bits,
    move_probability,
    sr_copy_bits,
    tensor_positions,
)
from tests.pointwise_reference import sumsq_ref

pytestmark = pytest.mark.gpu

CHUNK = 8192  # d9d::ADAM_CHUNK
ADAM_SIZES = [1, 7, 8, 9, 8191, 8192, 8193, 3 * CHUNK + 5, 100_003]
HYPER = dict(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, wd=0.1)
BIG_SEED = (1 << 33) + 4321
AMBIGUOUS: dict[str, list[int]] = {}  # kernel output -> [ambiguous elements, elements]
WORST: dict[str, float] = {}


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    yield _ops.load()
    if AMBIGUOUS:
        print("\nambiguous fraction per output: " + ", ".join(
            f"{k} {a / max(n, 1):.3g} ({a} of {n})" for k, (a, n) in sorted(AMBIGUOUS.items())))
    if WORST:
        print("worst err/bound per output: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def record(kernel: str, stats: dict[str, float], n: int) -> None:
    for key, val in stats.items():
        name, kind = key.split(".")
        if kind == "ambiguous":
            tally = AMBIGUOUS.setdefault(f"{kernel}.{name}", [0, 0])
            tally[0] += int(val)
            tally[1] += n
        else:
            WORST[f"{kernel}.{name}"] = max(WORST.get(f"{kernel}.{name}", 0.0), val)


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    it = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return torch.equal(a.contiguous().view(it), b.contiguous().view(it))


# ============================================================================ sr_copy_
SPECIAL_BITS = [
    0x7F800001, 0xFF800001, 0x7FC00000, 0xFFC00001, 0x7FFFFFFF, 0x7F810000,  # NaNs: low-only and high payloads
    0x7F800000, 0xFF800000,  # inf
    0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F0000, 0xFF7F0000,  # fp32 and bf16 maxima
    0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00400000, 0x80012345,  # zeros, denormals
]


def sr_copy_persistent_n() -> int:
    # sr_copy_f32_to_bf16: ew_grid caps the grid at num_sms * 16 blocks of 256 threads, 8 elements each
    return 3 * sms() * 16 * 256 * 8 + 13


def sr_source(n: int, gen: torch.Generator) -> torch.Tensor:
    """fp32 bit patterns of every exponent (2^-149 ... 2^127), both signs, with bf16-exact values, denormals and the
    special values of SPECIAL_BITS both at the front and spread over the buffer."""
    dev = "cuda"
    e = torch.randint(0, 255, (n,), device=dev, generator=gen)
    e = torch.where(torch.arange(n, device=dev) % 16 == 5, 0, e)  # denormals (2^-130 lies here)
    bits = (e << 23) | torch.randint(0, 1 << 23, (n,), device=dev, generator=gen)
    bits |= torch.randint(0, 2, (n,), device=dev, generator=gen) << 31
    bits = torch.where(torch.arange(n, device=dev) % 4 == 1, bits & ~0xFFFF, bits)  # bf16-exact
    special = torch.tensor(SPECIAL_BITS, device=dev, dtype=torch.int64)
    k = min(n, special.numel())
    bits[:k] = special[:k]
    if n > 4 * special.numel():
        at = torch.randint(0, n, (8 * special.numel(),), device=dev, generator=gen)
        bits[at] = special.repeat(8)
    return from_f32_bits(bits)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 4097, "persistent"])
@pytest.mark.parametrize("seed", [(1 << 32) + 11, (1 << 62) + 12345])
def test_sr_copy_bit_exact(ops, n, seed):
    if n == "persistent":
        n = sr_copy_persistent_n()
    src = sr_source(n, torch.Generator(device="cuda").manual_seed(n))
    dst = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ops.sr_copy_(dst, src, seed)
    check_sr_exact(dst, src, sr_copy_bits(n, seed, device="cuda"), f"sr_copy n={n}")
    again = torch.empty_like(dst)
    ops.sr_copy_(again, src, seed)
    assert bits_equal(dst, again), "not reproducible for a seed"
    if n > 1000:
        ops.sr_copy_(again, src, seed + 1)
        assert not bits_equal(dst, again), "another seed gave the same bits"


def test_sr_copy_through_wrapper(ops):
    """copy_fp32_to_bf16_stochastic_ draws its seed from the generator and rounds with it."""
    from d9d_b200.kernel.stochastic import copy_fp32_to_bf16_stochastic_
    from d9d_b200.kernel.stochastic._rng import draw_seed

    src = torch.randn(3, 1000, device="cuda")
    dst = torch.empty(3, 1000, device="cuda", dtype=torch.bfloat16)
    gen = torch.Generator().manual_seed(8)
    replay = torch.Generator()
    replay.set_state(gen.get_state())
    copy_fp32_to_bf16_stochastic_(dst, src, generator=gen)
    check_sr_exact(dst, src, sr_copy_bits(src.numel(), draw_seed(replay), device="cuda"), "copy_fp32_to_bf16_stochastic_")


@pytest.mark.parametrize("which", ["src", "dst"])
def test_sr_copy_refuses_misaligned(ops, which):
    n = 4097
    src_buf = torch.randn(n + 8, device="cuda")
    dst_buf = torch.full((n + 8,), 7.0, device="cuda", dtype=torch.bfloat16)
    src = src_buf[1:n + 1] if which == "src" else src_buf[:n]
    dst = dst_buf[1:n + 1] if which == "dst" else dst_buf[:n]
    with pytest.raises(RuntimeError, match="aligned"):
        ops.sr_copy_(dst, src, 3)
    torch.cuda.synchronize()
    assert bool((dst_buf == 7.0).all()), "the refused copy wrote to its destination"


# ============================================================================ adamw_sr_multi_
def make_tensors(sizes, grad_dtype, state_dtype, seed: int):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [adam_inputs(n, grad_dtype, state_dtype, gen, device="cuda") for n in sizes]


def run_multi(tensors, *, seed, step, grad_scale=None, plan=None, **hyper):
    """One adamw_stochastic_bf16_multi_ launch over clones of ``tensors``; returns (plan, outputs)."""
    from d9d_b200.kernel.stochastic import adamw_stochastic_bf16_multi_

    out = [tuple(t.clone() for t in ts) for ts in tensors]
    if plan is not None:  # a plan carries raw pointers: rebuild it for the clones, keeping its rng_base column
        from d9d_b200.kernel.stochastic.adamw_step import AdamWLaunchPlan

        bases = plan.metas[:, 5].clone()
        plan = AdamWLaunchPlan(*zip(*out, strict=True))
        plan.metas[:, 5] = bases
    gs = None if grad_scale is None else torch.tensor([grad_scale], device="cuda")
    h = {**HYPER, **hyper}
    plan = adamw_stochastic_bf16_multi_(*(list(c) for c in zip(*out, strict=True)), lr=h["lr"], beta1=h["beta1"],
                                        beta2=h["beta2"], eps=h["eps"], weight_decay=h["wd"], step=step, seed=seed,
                                        grad_scale=gs, plan=plan)
    return plan, out


def check_multi(tensors, out, plan, *, seed, step, grad_scale=None, what="", **hyper):
    h = {**HYPER, **hyper}
    bc1, bc2 = bias_corrections(h["beta1"], h["beta2"], step)
    for (p, g, m, v), (po, _, mo, vo), base in zip(tensors, out, plan.metas[:, 5].tolist(), strict=True):
        pos = tensor_positions(p.numel(), base, device="cuda")
        stats = check_adamw(po, mo, vo, p, g, m, v, pos, seed, f"{what} n={p.numel()}", bc1=bc1, bc2=bc2,
                            grad_scale=grad_scale, **h)
        record("adamw_sr_multi", stats, p.numel())


@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("grad_scale", [None, 0.37])
@pytest.mark.parametrize("step", [1, 1000])
def test_adamw_sr_multi(ops, grad_dtype, state_dtype, grad_scale, step):
    tensors = make_tensors(ADAM_SIZES, grad_dtype, state_dtype, step)
    seed = BIG_SEED + step
    plan, out = run_multi(tensors, seed=seed, step=step, grad_scale=grad_scale)
    check_multi(tensors, out, plan, seed=seed, step=step, grad_scale=grad_scale)
    for (g0, g1) in ((t[1], o[1]) for t, o in zip(tensors, out, strict=True)):
        assert bits_equal(g0, g1), "the gradient was written"
    _, again = run_multi(tensors, seed=seed, step=step, grad_scale=grad_scale)
    assert all(bits_equal(a[0], b[0]) for a, b in zip(out, again, strict=True)), "not reproducible for a seed"


@pytest.mark.parametrize("edge", [dict(beta1=0.0), dict(wd=0.0)])
def test_adamw_sr_multi_edges(ops, edge):
    tensors = make_tensors(ADAM_SIZES, torch.float32, torch.bfloat16, 5)
    plan, out = run_multi(tensors, seed=BIG_SEED, step=3, grad_scale=0.37, **edge)
    check_multi(tensors, out, plan, seed=BIG_SEED, step=3, grad_scale=0.37, **edge)


def test_adamw_sr_multi_many_tensors(ops):
    """One launch over 300 small tensors: a block map of mostly single-chunk tensors."""
    sizes = torch.randint(1, 3000, (300,), generator=torch.Generator().manual_seed(1)).tolist()
    tensors = make_tensors(sizes, torch.bfloat16, torch.bfloat16, 6)
    plan, out = run_multi(tensors, seed=BIG_SEED, step=2, grad_scale=0.37)
    assert plan.metas.shape[0] == 300
    check_multi(tensors, out, plan, seed=BIG_SEED, step=2, grad_scale=0.37)


@pytest.mark.parametrize("operand", [0, 1, 2, 3], ids=["p", "g", "m", "v"])
@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_adamw_sr_multi_misaligned(ops, operand, grad_dtype, state_dtype):
    """A contiguous view at a one-element storage offset sends the whole tensor down the scalar path, which must give
    the aligned result bit for bit."""
    tensors = make_tensors([7, 8193, 20_005], grad_dtype, state_dtype, 7)
    shifted = []
    for ts in tensors:
        ts = list(ts)
        buf = torch.empty(ts[operand].numel() + 1, device="cuda", dtype=ts[operand].dtype)
        buf[1:].copy_(ts[operand])
        ts[operand] = buf[1:]
        shifted.append(tuple(ts))
    _, ref = run_multi(tensors, seed=BIG_SEED, step=4, grad_scale=0.37)
    from d9d_b200.kernel.stochastic import adamw_stochastic_bf16_multi_

    gs = torch.tensor([0.37], device="cuda")
    adamw_stochastic_bf16_multi_(*(list(c) for c in zip(*shifted, strict=True)), lr=HYPER["lr"], beta1=HYPER["beta1"],
                                 beta2=HYPER["beta2"], eps=HYPER["eps"], weight_decay=HYPER["wd"], step=4,
                                 seed=BIG_SEED, grad_scale=gs)
    for a, b in zip(ref, shifted, strict=True):
        for x, y in zip(a, b, strict=True):
            assert bits_equal(x, y), "the scalar path differs from the vector path"


def test_adamw_sr_multi_counter_above_2_32(ops):
    """rng_base >= 2^35 puts the tensors' counters above 2^32, in the high counter word."""
    from d9d_b200.kernel.stochastic.adamw_step import AdamWLaunchPlan

    tensors = make_tensors([9, 8193, 30_001], torch.float32, torch.bfloat16, 8)
    plan = AdamWLaunchPlan(*zip(*tensors, strict=True))
    plan.metas[:, 5] += (1 << 35) + 8 * 1234567
    plan, out = run_multi(tensors, seed=BIG_SEED, step=2, plan=plan)
    assert int(plan.metas[0, 5]) >> 3 >= 1 << 32
    check_multi(tensors, out, plan, seed=BIG_SEED, step=2, what="rng_base >= 2^35")


def test_adamw_sr_multi_seed_carry(ops):
    """seed = 2^32 - 20: the exp_avg and exp_avg_sq keys, seed + 42 and seed + 67, carry into the key's high word."""
    seed = (1 << 32) - 20
    tensors = make_tensors([8193, 30_001], torch.bfloat16, torch.bfloat16, 9)
    plan, out = run_multi(tensors, seed=seed, step=2)
    check_multi(tensors, out, plan, seed=seed, step=2, what="seed carry")


def test_adamw_sr_regime(ops):
    """Updates of about a tenth of an ulp of p: round-to-nearest would leave every p unchanged, SR moves each with
    probability |update| / ulp.  The number that moved must match the fp64 expectation within 5 sigma."""
    n = 200_003
    gen = torch.Generator(device="cuda").manual_seed(10)
    p = (1 + torch.rand(n, device="cuda", generator=gen)).bfloat16()  # [1, 2): ulp 2^-7
    g = torch.randn(n, device="cuda", generator=gen)
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    hyper = dict(lr=1e-3, wd=0.0)
    plan, out = run_multi([(p, g, m, v)], seed=BIG_SEED, step=1, **hyper)
    po = out[0][0]
    h = {**HYPER, **hyper}
    bc1, bc2 = bias_corrections(h["beta1"], h["beta2"], 1)
    ref = adamw_ref(p, g, m, v, bc1=bc1, bc2=bc2, **h)[0]
    assert float(((ref - p.double()).abs() < 2.0**-9).double().mean()) > 0.99, "updates are not below half an ulp"
    prob = move_probability(ref, p)
    moved = int((po != p).sum())
    mean, sigma = float(prob.sum()), float((prob * (1 - prob)).sum().sqrt())
    assert abs(moved - mean) <= 5 * sigma, (moved, mean, sigma)
    assert moved > 0.05 * n
    check_multi([(p, g, m, v)], out, plan, seed=BIG_SEED, step=1, what="SR regime", **hyper)


# ============================================================================ NVLink shard kernels, one replica
BEGIN = 8 * 37


def reduce_n() -> int:
    # nvl_reduce_shard: at most num_sms * 4 blocks of 512 threads, UNROLL = 4 float4 per thread per pass
    return 3 * sms() * 4 * 512 * 4 * 4 + 104


def adamw_shard_n() -> int:
    # nvl_adamw_shard: at most num_sms * 8 blocks of 256 threads, 8 elements per thread per pass
    return 3 * sms() * 8 * 256 * 8 + 104


def test_nvl_reduce_shard(ops):
    n = reduce_n()
    end = BEGIN + n
    buf = torch.randn(end + 64, device="cuda")
    before = buf.clone()
    sumsq = torch.tensor([3.5], device="cuda")
    ops.nvl_reduce_shard_(buf, 0, 0, BEGIN, end, 1, 0, sumsq)
    assert bits_equal(buf, before), "one replica's reduce changed its gradients or the sentinels"
    blocks = min((n // 4 + 2047) // 2048, sms() * 4)
    ref, bound = sumsq_ref(buf[BEGIN:end], 3.5, adds=blocks)
    r = assert_within(sumsq, torch.tensor([ref], device="cuda", dtype=torch.float64),
                      torch.tensor([bound], device="cuda", dtype=torch.float64), "nvl_reduce_shard sumsq")
    WORST["nvl_reduce_shard.sumsq"] = max(WORST.get("nvl_reduce_shard.sumsq", 0.0), r)

    # exact probe: small integers on every pass boundary and spread over the shard, all sums exact in fp32
    probe = torch.zeros(end + 64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(11)
    per_pass = sms() * 4 * 512 * 4 * 4
    at = [BEGIN + k * per_pass + d for k in range(4) for d in (0, 1, 2, 3, -1, -4, -5, -8) if 0 <= k * per_pass + d < n]
    at += [end - 1, end - 104]
    probe[torch.tensor(at, device="cuda")] = 2.0
    probe[BEGIN:end:997] = torch.randint(-3, 4, (len(range(BEGIN, end, 997)),), device="cuda", generator=gen).float()
    probe[:BEGIN] = 1000.0  # sentinels: would show in the sum
    probe[end:] = 1000.0
    want = 5.0 + float(probe[BEGIN:end].double().square().sum())
    assert want < 2**24
    s = torch.tensor([5.0], device="cuda")
    ops.nvl_reduce_shard_(probe, 0, 0, BEGIN, end, 1, 0, s)
    assert float(s) == want, (float(s), want)


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("grad_scale", [None, 0.37])
def test_nvl_adamw_shard(ops, state_dtype, grad_scale):
    n = adamw_shard_n()
    end = BEGIN + n
    total = end + 64
    gen = torch.Generator(device="cuda").manual_seed(12)
    p, g, m, v = adam_inputs(n, torch.float32, state_dtype, gen, device="cuda")
    param = torch.randn(total, device="cuda").bfloat16()
    grad = torch.randn(total, device="cuda")
    param[BEGIN:end] = p
    grad[BEGIN:end] = g
    step, seed = 5, BIG_SEED + 77
    bc1, bc2 = bias_corrections(HYPER["beta1"], HYPER["beta2"], step)
    gs = None if grad_scale is None else torch.tensor([grad_scale], device="cuda")

    def launch(prm, ma, va, lo, hi):
        ops.nvl_adamw_shard_(prm, grad, ma, va, 0, 0, lo, hi, 1, 0, HYPER["lr"], HYPER["beta1"], HYPER["beta2"],
                             HYPER["eps"], HYPER["wd"], bc1, bc2, seed, gs)

    param0, grad0 = param.clone(), grad.clone()
    out_p, out_m, out_v = param.clone(), m.clone(), v.clone()
    launch(out_p, out_m, out_v, BEGIN, end)
    assert bits_equal(grad, grad0), "the gradient arena was written"
    assert bits_equal(out_p[:BEGIN], param0[:BEGIN]) and bits_equal(out_p[end:], param0[end:]), "a sentinel moved"
    pos = torch.arange(BEGIN, end, device="cuda")
    stats = check_adamw(out_p[BEGIN:end], out_m, out_v, p, g, m, v, pos, seed, "nvl_adamw_shard", lr=HYPER["lr"],
                        beta1=HYPER["beta1"], beta2=HYPER["beta2"], eps=HYPER["eps"], wd=HYPER["wd"], bc1=bc1,
                        bc2=bc2, grad_scale=grad_scale)
    record("nvl_adamw_shard", stats, n)

    # the same range as two shards, each with its own shard-local state: the global counter makes them equal
    mid = BEGIN + 8 * 123_457
    split_p = param0.clone()
    m1, v1, m2, v2 = m[: mid - BEGIN].clone(), v[: mid - BEGIN].clone(), m[mid - BEGIN:].clone(), v[mid - BEGIN:].clone()
    launch(split_p, m1, v1, BEGIN, mid)
    launch(split_p, m2, v2, mid, end)
    assert bits_equal(split_p, out_p), "sharding changed the parameters"
    assert bits_equal(torch.cat([m1, m2]), out_m) and bits_equal(torch.cat([v1, v2]), out_v), "sharding changed the state"


def test_nvl_shard_bounds_refused(ops):
    n = 4096
    grad = torch.randn(n, device="cuda")
    param = torch.randn(n, device="cuda").bfloat16()
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    p0, g0 = param.clone(), grad.clone()
    s = torch.zeros(1, device="cuda")
    for lo, hi in ((4, 1024), (8, 1020)):
        with pytest.raises(RuntimeError, match="multiples of 8"):
            ops.nvl_adamw_shard_(param, grad, m, v, 0, 0, lo, hi, 1, 0, 1e-2, 0.9, 0.95, 1e-8, 0.1, 0.1, 0.05, 1, None)
        with pytest.raises(RuntimeError, match="multiples of 8"):
            ops.nvl_reduce_shard_(grad, 0, 0, lo, hi, 1, 0, s)
    torch.cuda.synchronize()
    assert bits_equal(param, p0) and bits_equal(grad, g0) and float(s) == 0.0
    assert not bool(m.any()) and not bool(v.any())


# ============================================================================ StochasticAdamW
@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_stochastic_adamw_steps(ops, state_dtype, monkeypatch):
    """Three steps of two parameter groups: fp32- and bf16-gradient buckets, a parameter whose gradient goes away after
    step 1 (its state and step count must stay), one that first gets a gradient at step 2 (its own bucket and bias
    correction), and a grad_scale.  Seeds are replayed from a copy of the generator in the documented order, and the
    launch plans must be reused once the buckets stop changing."""
    from d9d_b200.kernel.stochastic import adamw_step
    from d9d_b200.kernel.stochastic._rng import draw_seed
    from d9d_b200.optim.stochastic import StochasticAdamW

    built = []
    init = adamw_step.AdamWLaunchPlan.__init__

    def counting_init(self, *args, **kwargs):
        built.append(self)
        init(self, *args, **kwargs)

    monkeypatch.setattr(adamw_step.AdamWLaunchPlan, "__init__", counting_init)

    def param(*shape):
        return torch.nn.Parameter(torch.randn(*shape, device="cuda").bfloat16())

    A, B, N, C, L = param(300, 70), param(20_001), param(513), param(8193), param(4097)
    for p in (A, N, C, L):
        p.grad_dtype = torch.float32
    when = {A: {1, 2, 3}, B: {1, 2, 3}, N: {1}, C: {1, 2, 3}, L: {2, 3}}
    betas, eps = (0.9, 0.95), 1e-8
    gen = torch.Generator().manual_seed(99)
    opt = StochasticAdamW([{"params": [A, B, N], "lr": 1e-3, "weight_decay": 0.1},
                           {"params": [C, L], "lr": 3e-3, "weight_decay": 0.0}],
                          lr=1e-3, betas=betas, eps=eps, generator=gen, state_dtype=state_dtype)
    opt.grad_scale = torch.tensor([0.37], device="cuda")
    steps = {p: 0 for p in when}
    builds = []
    for t in (1, 2, 3):
        for p, ts in when.items():
            if t not in ts:
                p.grad = None
                continue
            if p.grad is None:
                p.grad = torch.zeros_like(p, dtype=getattr(p, "grad_dtype", p.dtype))
            p.grad.copy_(torch.randn_like(p, dtype=torch.float32) * 0.01)

        def state(p, key):
            st = opt.state[p]
            return st[key].clone() if key in st else torch.zeros_like(p, dtype=state_dtype)

        before = {p: (p.detach().clone(), None if p.grad is None else p.grad.clone(), state(p, "exp_avg"),
                      state(p, "exp_avg_sq")) for p in when}
        replay = torch.Generator()
        replay.set_state(gen.get_state())
        n_built = len(built)
        opt.step()
        builds.append(len(built) - n_built)

        for group in opt.param_groups:
            buckets: dict = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                steps[p] += 1
                buckets.setdefault((steps[p], p.grad.dtype), []).append(p)
            for (step, _), ps in buckets.items():
                seed = draw_seed(replay)
                bc1, bc2 = bias_corrections(*betas, step)
                base = 0
                for p in ps:
                    p0, g0, m0, v0 = before[p]
                    pos = tensor_positions(p.numel(), base, device="cuda")
                    stats = check_adamw(p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], p0, g0, m0,
                                        v0, pos, seed, f"StochasticAdamW step {t}", lr=group["lr"], beta1=betas[0],
                                        beta2=betas[1], eps=eps, wd=group["weight_decay"], bc1=bc1, bc2=bc2,
                                        grad_scale=0.37)
                    record("StochasticAdamW", stats, p.numel())
                    base += (p.numel() + 7) // 8 * 8
        if t > 1:
            assert bits_equal(N.detach(), before[N][0]), "a parameter without a gradient moved"
            assert opt.state[N]["step"] == 1
            assert bits_equal(opt.state[N]["exp_avg"], before[N][2])
            assert bits_equal(opt.state[N]["exp_avg_sq"], before[N][3])
    # step 1: group 0's fp32 bucket [A, N] and bf16 bucket [B], group 1's [C]; step 2: [A] without N and the new [L];
    # step 3: nothing new
    assert builds == [3, 2, 0], builds
