"""Every bf16 wgmma GEMM instance (dense single-CTA and CTA-pair, split-K, grouped by expert, fused linear-CE and the fused
tensor-parallel GEMMs emulated on one GPU) against an fp64 reference with a per-element error bound.

Each case forces the tile width (and split count) it means to test, writes into a canaried view with padded row pitch
(everything outside the view must stay bitwise unchanged) and reads operands whose row padding holds NaN (a read past K,
M or N poisons the result).  The output layout picks the epilogue: a 16-byte aligned base and pitch take the TMA store /
reduce path, a misaligned base or odd pitch the direct-store path.

Set D9D_GEMM_REPORT=<file> to write the worst err/bound per kernel family and the list of launched instances as JSON.
"""

import json
import os

import pytest
import torch

from tests.gemm_reference import CANARY, U_BF16, Canaried, assert_within, ck, gemm_bound, matmul_ref, padded, shard_rows

pytestmark = pytest.mark.gpu

DEV = "cuda"
LAYOUTS = {"NT": (False, False), "NN": (False, True), "TN": (True, True), "TT": (True, False)}  # (a_mn, b_mn)
EPIS = {"bf16": (torch.bfloat16, False), "f32": (torch.float32, False), "f32_acc": (torch.float32, True),
        "bf16_acc": (torch.bfloat16, True)}
STORE_EPIS = ("bf16", "f32")
LAYOUT_EPIS = [(lay, epi) for lay in LAYOUTS for epi in (STORE_EPIS if lay == "TT" else EPIS)]

_worst: dict[str, float] = {}
_instances: set[tuple] = set()


def _record(family, instance, ratio):
    _worst[family] = max(_worst.get(family, 0.0), ratio)
    _instances.add(instance)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("D9D_GEMM_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({"worst_err_over_bound": _worst, "instances": sorted(map(list, _instances)),
                       "num_instances": len(_instances)}, f, indent=1)


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _ceil8(x):
    return (x + 7) // 8 * 8


def _operands(M, N, K, a_mn, b_mn):
    a = padded(K, M, 8, device=DEV) if a_mn else padded(M, K, 8, device=DEV)
    b = padded(K, N, 8, device=DEV) if b_mn else padded(N, K, 8, device=DEV)
    return a, b


def _legal(M, N, a_mn, b_mn):
    """TMA needs 16-byte operand row pitches: an MN-major operand's contiguous dim must be a multiple of 8."""
    return (_ceil8(M) if a_mn else M), (_ceil8(N) if b_mn else N)


def _run_dense(ops, layout, epi, M, N, K, *, tma, ctas, block_n, k_splits=0, family):
    a_mn, b_mn = LAYOUTS[layout]
    out_dtype, acc = EPIS[epi]
    M, N = _legal(M, N, a_mn, b_mn)
    a, b = _operands(M, N, K, a_mn, b_mn)
    d0 = torch.randn(M, N, device=DEV).to(out_dtype) if acc else None
    out = Canaried(M, N, out_dtype, tma=tma, device=DEV, init=d0)
    ops.gemm(a, b, out.view, a_mn, b_mn, acc, ctas=ctas, block_n=block_n, k_splits=k_splits)
    prod, S = matmul_ref(a, b, a_mn, b_mn)
    kb = (K + 63) // 64
    splits = k_splits if k_splits else max(1, kb // 8)
    ref, bound = gemm_bound(prod, S, K, out_dtype, d0=d0, k_splits=splits)
    r = assert_within(out.view, ref, bound, f"{layout} {epi} M={M} N={N} K={K} bn={block_n} ctas={ctas}")
    out.assert_untouched()
    _record(f"{family}/{epi}", ("dense", layout, epi, block_n, ctas, "none"), r)
    return a, b, out


# ----------------------------------------------------------------------------- dense, single CTA
# (M, N, K, 16-byte aligned output base and pitch).  M / N are rounded up to a multiple of 8 where the operand layout needs
# it.  An odd N (K-major B only) takes the direct store even with an aligned pitch: a TMA store would clip the row at
# 16-byte granularity and write into the padding.
SINGLE_SHAPES = [(1, 136, 520, True), (127, 200, 8, False), (129, 8, 72, True), (333, 203, 72, False),
                 (129, 200, 520, True), (333, 136, 8, False), (129, 203, 72, True)]


@pytest.mark.parametrize("block_n", [128, 192, 256])
@pytest.mark.parametrize("layout,epi", LAYOUT_EPIS)
@pytest.mark.parametrize("M,N,K,tma", SINGLE_SHAPES)
def test_dense_single_cta(ops, layout, epi, block_n, M, N, K, tma):
    _run_dense(ops, layout, epi, M, N, K, tma=tma, ctas=1, block_n=block_n, family="dense")


@pytest.mark.parametrize("block_n", [128, 192, 256])
@pytest.mark.parametrize("layout,epi", [("NT", "bf16"), ("TN", "f32_acc")])
def test_dense_single_cta_more_tiles_than_sms(ops, layout, epi, block_n):
    # 18 x 10..20 tiles of 128 x block_n: every CTA walks several tiles and the operand stage ring wraps many times
    _run_dense(ops, layout, epi, 2304, 2560, 4168, tma=True, ctas=1, block_n=block_n, k_splits=1, family="dense")


# ----------------------------------------------------------------------------- dense, CTA pair
PAIR_SHAPES = [(64, 200, 520, True), (200, 203, 72, False), (600, 136, 72, True), (600, 200, 136, False)]


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("layout,epi", LAYOUT_EPIS)
@pytest.mark.parametrize("M,N,K,tma", PAIR_SHAPES)
def test_dense_cta_pair(ops, layout, epi, block_n, M, N, K, tma):
    # M = 64 / 200: the second CTA's 128 rows are wholly / partly out of bounds
    _run_dense(ops, layout, epi, M, N, K, tma=tma, ctas=2, block_n=block_n, k_splits=1, family="pair")


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("epi", STORE_EPIS)
@pytest.mark.parametrize("tma", [True, False])
def test_pair_bitwise_equals_single(ops, layout, epi, block_n, tma):
    # same MMA width and the same k order per element: the pair kernel must reproduce the single-CTA result exactly
    a, b, out = _run_dense(ops, layout, epi, 600, 200, 520, tma=tma, ctas=2, block_n=block_n, family="pair")
    a_mn, b_mn = LAYOUTS[layout]
    single = Canaried(*out.view.shape, out.view.dtype, tma=tma, device=DEV)
    ops.gemm(a, b, single.view, a_mn, b_mn, False, ctas=1, block_n=block_n)
    assert torch.equal(out.view, single.view)
    _record(f"dense/{epi}", ("dense", layout, epi, block_n, 1, "none"), 0.0)


# ----------------------------------------------------------------------------- split-K
@pytest.mark.parametrize("layout", ["NT", "NN", "TN"])
@pytest.mark.parametrize("ctas,block_n", [(1, 128), (1, 192), (1, 256), (2, 128), (2, 256)])
@pytest.mark.parametrize("k_splits", [2, 5, "kb+3"])
def test_split_k_forced(ops, layout, ctas, block_n, k_splits):
    M, N, K = 256, 384, 1000  # 16 k-blocks
    ks = 16 + 3 if k_splits == "kb+3" else k_splits  # more slices than k-blocks: the trailing ones are empty
    _run_dense(ops, layout, "f32_acc", M, N, K, tma=True, ctas=ctas, block_n=block_n, k_splits=ks, family="split_k")


@pytest.mark.parametrize("layout", ["NT", "TN"])
def test_split_k_heuristic_empty_slice(ops, layout):
    # 2 x 3 tiles of 128 x 128 and 167 k-blocks: min(132 / 6, 167 / 8) = 20 slices of 9 k-blocks, the last one empty
    _run_dense(ops, layout, "f32_acc", 256, 384, 10688, tma=True, ctas=1, block_n=128, k_splits=0, family="split_k")


def test_split_k_rejected_where_it_cannot_run(ops):
    a, b = _operands(256, 384, 1000, False, False)
    d = torch.zeros(256, 384, device=DEV)
    with pytest.raises(RuntimeError, match="k_splits"):
        ops.gemm(a, b, d, False, False, False, ctas=1, block_n=128, k_splits=2)  # store epilogue
    direct = Canaried(256, 384, torch.float32, tma=False, device=DEV)
    with pytest.raises(RuntimeError, match="split-K"):
        ops.gemm(a, b, direct.view, False, False, True, ctas=1, block_n=128, k_splits=2)  # output TMA cannot address
    with pytest.raises(RuntimeError, match="k_splits"):
        ops.gemm(a, b, d, False, False, True, ctas=1, block_n=128, k_splits=-1)
    direct.assert_untouched()


def test_block_n_is_validated(ops):
    a, b = _operands(256, 384, 128, False, False)
    d = torch.zeros(256, 384, device=DEV, dtype=torch.bfloat16)
    for ctas, bn in ((1, 64), (1, 200), (2, 192), (2, 64)):
        with pytest.raises(RuntimeError, match="block_n"):
            ops.gemm(a, b, d, False, False, False, ctas=ctas, block_n=bn)
    assert (d == 0).all()


# ----------------------------------------------------------------------------- MN-major A with K-major B: store only
@pytest.mark.parametrize("M", [8, 128, 640])
@pytest.mark.parametrize("ctas", [0, 1, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_tt_accumulate_raises_for_every_shape(ops, M, ctas, dtype):
    a, b = _operands(M, 256, 128, True, False)
    d = torch.zeros(M, 256, device=DEV, dtype=dtype)
    with pytest.raises(RuntimeError, match="accumulate"):
        ops.gemm(a, b, d, True, False, True, ctas=ctas)
    assert (d == 0).all()


# ----------------------------------------------------------------------------- grouped by expert (rows of A / D)
def _flat_out(shape, dtype, tma, init=None):
    """Contiguous output at an offset inside a canaried flat buffer (the grouped bindings need contiguous outputs)."""
    n = 1
    for s in shape:
        n *= s
    off = (16 // torch.empty((), dtype=dtype).element_size()) if tma else 1
    flat = torch.full((n + 2 * off + 8,), CANARY[dtype], device=DEV, dtype=dtype)
    view = flat[off : off + n].view(shape)
    if init is not None:
        view.copy_(init)
    return flat, view, flat.clone(), off, off + n


def _assert_flat_untouched(flat, before, lo, hi):
    int_t = torch.int16 if flat.element_size() == 2 else torch.int32
    assert torch.equal(flat[:lo].view(int_t), before[:lo].view(int_t))
    assert torch.equal(flat[hi:].view(int_t), before[hi:].view(int_t))


@pytest.mark.parametrize("block_n", [128, 192, 256])
@pytest.mark.parametrize("b_mn,acc", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("tma", [True, False])
def test_grouped_m(ops, block_n, b_mn, acc, tma):
    counts = [0, 1, 128, 300]  # rows per expert; every expert's segment is padded to whole 128-row tiles
    E, K, N = len(counts), 136, 200
    tiles = [-(-c // 128) for c in counts]
    tile_group = [e for e, t in enumerate(tiles) for _ in range(t)] + [-1, -1]  # trailing unused tiles
    cap = 128 * len(tile_group)
    a = torch.randn(cap, K, device=DEV).bfloat16()
    w = (torch.randn(E, K, N, device=DEV) if b_mn else torch.randn(E, N, K, device=DEV)).bfloat16()
    tg = torch.tensor(tile_group, dtype=torch.int32, device=DEV)
    d0 = torch.randn(cap, N, device=DEV).bfloat16()
    flat, d, before, lo, hi = _flat_out((cap, N), torch.bfloat16, tma, init=d0)
    ops.gemm_grouped_m(a, w, d, tg, b_mn, acc, block_n=block_n)
    worst = 0.0
    for t, e in enumerate(tile_group):
        rows = slice(128 * t, 128 * t + 128)
        if e < 0:
            assert torch.equal(d[rows], d0[rows]), "an unused tile was written"
            continue
        prod, S = matmul_ref(a[rows], w[e], False, b_mn)
        ref, bound = gemm_bound(prod, S, K, torch.bfloat16, d0=d0[rows] if acc else None)
        worst = max(worst, assert_within(d[rows], ref, bound, f"tile {t} expert {e}"))
    _assert_flat_untouched(flat, before, lo, hi)
    _record("grouped_m/bf16_acc" if acc else "grouped_m/bf16", ("grouped_m", "NN" if b_mn else "NT", "bf16_acc" if acc else "bf16", block_n, 1, "none"), worst)


@pytest.mark.parametrize("block_n", [128, 192, 256])
@pytest.mark.parametrize("epi", list(EPIS))
@pytest.mark.parametrize("tma", [True, False])
def test_grouped_k(ops, block_n, epi, tma):
    # group offsets on 64-row boundaries, empty first and last groups; M = 136: the partial second m-tile must clip at
    # its own group's edge instead of spilling into the next group's output
    offs = [0, 0, 64, 256, 320, 448, 448]
    E, M, N, R = len(offs) - 1, 136, 200, offs[-1]
    out_dtype, acc = EPIS[epi]
    x = torch.randn(R, M, device=DEV).bfloat16()  # the grouped bindings take contiguous operands only
    dy = torch.randn(R, N, device=DEV).bfloat16()
    d0 = torch.randn(E, M, N, device=DEV).to(out_dtype)
    flat, d, before, lo, hi = _flat_out((E, M, N), out_dtype, tma, init=d0)
    ops.gemm_grouped_k(x, dy, d, torch.tensor(offs, dtype=torch.int32, device=DEV), acc, block_n=block_n)
    worst = 0.0
    for e in range(E):
        k0, k1 = offs[e], offs[e + 1]
        prod, S = matmul_ref(x[k0:k1], dy[k0:k1], True, True)
        ref, bound = gemm_bound(prod, S, max(k1 - k0, 1), out_dtype, d0=d0[e] if acc else None)
        worst = max(worst, assert_within(d[e], ref, bound, f"group {e} rows {k0}:{k1}"))
    _assert_flat_untouched(flat, before, lo, hi)
    _record(f"grouped_k/{epi}", ("grouped_k", "TN", epi, block_n, 1, "none"), worst)


# ----------------------------------------------------------------------------- fused linear cross-entropy
def _ce_reference(h, w, tgt, bias, softcap, col_offset, ignore=-100):
    z = h.double() @ w.double().t()
    S = h.double().abs() @ w.double().abs().t()
    if bias is not None:
        z = z + bias.double()
    dz = torch.ones_like(z)
    if softcap > 0:
        th = torch.tanh(z / softcap)
        z, dz = softcap * th, 1 - th * th
    lse = torch.logsumexp(z, -1)
    rel = tgt - col_offset
    inside = (tgt != ignore) & (rel >= 0) & (rel < w.shape[0])
    tl = torch.where(inside, z.gather(1, rel.clamp(0, w.shape[0] - 1)[:, None])[:, 0], torch.zeros_like(lse))
    nll = torch.where(tgt == ignore, torch.zeros_like(lse), lse - tl)
    return z, dz, S, lse, tl, nll, inside


def _check_ce(ops, T, V, K, *, pair_mode, tma, bias=False, softcap=0.0, col_offset=0, all_ignored=False):
    h = (torch.randn(T, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(V, K, device=DEV) * 0.1).bfloat16()
    b = torch.randn(V, device=DEV) * 0.5 if bias else None
    vt = V + col_offset
    tgt = torch.randint(0, vt + (40 if col_offset else 0), (T,), device=DEV)
    for i, c in enumerate([0, V - 1, (V - 1) // 256 * 256 + (V - 1) % 256 // 2]):  # first, last, inside the last tile
        if i < T:
            tgt[i] = c + col_offset
    tgt[4::7] = -100
    if all_ignored:
        tgt[:] = -100
    prev = ops.gemm_set_pair_mode(pair_mode)
    try:
        nll, lse, tl = ops.ce_forward_ex(h, w, tgt, -100, b, softcap, col_offset)
        z, dz, S, rlse, rtl, rnll, inside = _ce_reference(h, w, tgt, b, softcap, col_offset)
        n_tiles = (V + 255) // 256
        e_z = ck(K) * S.max(-1).values + 2.0**-20 * (1 + z.abs().max(-1).values) + (softcap * 2.0**-18 if softcap else 0.0)
        e_lse = e_z + (64 + n_tiles) * 2.0**-23 + 2.0**-19 * (1 + rlse.abs())
        worst_fwd = max(assert_within(lse, rlse, e_lse, "lse"),
                        assert_within(tl, rtl, torch.where(inside, e_z, 0.0), "target logit"),
                        assert_within(nll, rnll, torch.where(tgt == -100, 0.0, e_lse + e_z), "nll"))
        g = torch.rand(T, device=DEV)
        out = Canaried(T, V, torch.bfloat16, tma=tma, device=DEV)
        ops.ce_dlogits(h, w, tgt, rlse.float(), g, out.view, -100, b, softcap, col_offset)
        p = torch.exp(z - rlse.double()[:, None])
        gv = (g.double() * (tgt != -100))[:, None]
        onehot = torch.zeros_like(p)
        rows = inside.nonzero()[:, 0]
        onehot[rows, tgt[rows] - col_offset] = 1
        ref = gv * (p - onehot) * dz
        bound = U_BF16 * ref.abs() + gv * dz * p * (e_z[:, None] + 2.0**-19 * (1 + (z - rlse[:, None]).abs()))
        if softcap:
            bound = bound + gv * p * 2.0**-16
        worst_bwd = assert_within(out.view, ref, bound, "dlogits")
        out.assert_untouched()
    finally:
        ops.gemm_set_pair_mode(prev)
    ctas = 2 if (pair_mode and T >= 512 and V >= 128) else 1
    _record("ce_forward", ("dense", "NT", "ce_lse", 256, ctas, "none"), worst_fwd)
    _record("ce_dlogits", ("dense", "NT", "ce_dlogits", 256, ctas, "none"), worst_bwd)


@pytest.mark.parametrize("pair_mode", [0, 1])
@pytest.mark.parametrize("V", [1, 100, 255, 257, 50257])
@pytest.mark.parametrize("T", [1, 129, 1000])
@pytest.mark.parametrize("tma", [True, False])
def test_linear_ce(ops, pair_mode, V, T, tma):
    _check_ce(ops, T, V, 136, pair_mode=pair_mode, tma=tma)


@pytest.mark.parametrize("pair_mode", [0, 1])
@pytest.mark.parametrize("V", [257, 1500])
def test_linear_ce_bias_softcap_slice(ops, pair_mode, V):
    _check_ce(ops, 1000, V, 128, pair_mode=pair_mode, tma=True, bias=True, softcap=8.0, col_offset=300)


@pytest.mark.parametrize("pair_mode", [0, 1])
def test_linear_ce_all_rows_ignored(ops, pair_mode):
    _check_ce(ops, 600, 300, 64, pair_mode=pair_mode, tma=False, all_ignored=True)


# ----------------------------------------------------------------------------- 64-bit output offsets
@pytest.mark.parametrize("ctas", [1, 2])
def test_output_beyond_2_pow_31_elements(ops, ctas):
    M, N, K = 32769, 65537, 72  # M * N > 2^31; odd N and a misaligned base take the direct store
    a, b = _operands(M, N, K, False, False)
    flat = torch.full((M * N + 2,), CANARY[torch.bfloat16], device=DEV, dtype=torch.bfloat16)
    d = flat[1 : 1 + M * N].view(M, N)
    bn = 256 if ctas == 2 else 192
    ops.gemm(a, b, d, False, False, False, ctas=ctas, block_n=bn)
    assert flat[0].item() == CANARY[torch.bfloat16] and flat[-1].item() == CANARY[torch.bfloat16]
    mid = (1 << 31) // N
    rows = torch.tensor(sorted({0, 1, mid - 1, mid, mid + 1, M - 2, M - 1, *torch.randint(0, M, (8,)).tolist()}), device=DEV)
    prod, S = matmul_ref(a[rows], b, False, False)
    ref, bound = gemm_bound(prod, S, K, torch.bfloat16)
    r = assert_within(d[rows], ref, bound, "sampled rows")
    _record("dense_large", ("dense", "NT", "bf16", bn, ctas, "none"), r)


# ----------------------------------------------------------------------------- fused tensor-parallel GEMMs on one GPU
# W ranks are emulated with W separate buffers: the kernels take every peer's shard as a plain device pointer, so the
# owner / local-row mapping (blocks of block_rows dealt round-robin over the ranks) is exercised exactly as on W GPUs.
WORLDS = [1, 2, 3, 8]


def _shards(full, world, block_rows, pad=8):
    owners = shard_rows(full, world, block_rows)
    shards = []
    for rows in owners:
        s = padded(len(rows), full.shape[1], pad, device=DEV)
        s.copy_(full[rows])
        shards.append(s)
    return owners, shards


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("unit_mult", [1, 2])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_ag_a(ops, world, unit_mult, b_mn, block_n):
    br = 128 * unit_mult
    M, N, K = world * 2 * br, 200, 136  # every rank owns two blocks
    a = padded(M, K, 8, device=DEV)
    _, b = _operands(M, N, K, False, b_mn)
    owners, shards = _shards(a, world, br)
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    ops.gemm_ag_a([s.data_ptr() for s in shards], M // world, shards[0].stride(0), br, b, out.view, b_mn, block_n=block_n)
    prod, S = matmul_ref(a, b, False, b_mn)
    ref, bound = gemm_bound(prod, S, K, torch.bfloat16)
    r = assert_within(out.view, ref, bound, "gemm_ag_a")
    out.assert_untouched()
    plain = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, b, plain, False, b_mn, False, ctas=1, block_n=block_n)
    assert torch.equal(out.view, plain)
    _record("ag_a", ("dense", "NN" if b_mn else "NT", "bf16", block_n, 1, "ag_a"), r)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("unit_mult", [1, 2])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("last_rank,spare_sms", [(False, 0), (True, 8), (True, 0)])
def test_gemm_wait_a(ops, world, unit_mult, b_mn, block_n, last_rank, spare_sms):
    br = 128 * unit_mult
    M, N, K = world * 2 * br, 200, 136
    rank = world - 1 if last_rank else 0
    a = padded(M, K, 8, device=DEV)
    _, b = _operands(M, N, K, False, b_mn)
    # every shard has landed: the kernel must never find a zero flag (it would spin, then trap)
    flags = torch.ones(world, dtype=torch.int32, device=DEV)
    assert bool((flags != 0).all())
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    ops.gemm_wait_a(a, flags, rank, br, b, out.view, b_mn, spare_sms=spare_sms, block_n=block_n)
    prod, S = matmul_ref(a, b, False, b_mn)
    ref, bound = gemm_bound(prod, S, K, torch.bfloat16)
    r = assert_within(out.view, ref, bound, "gemm_wait_a")
    out.assert_untouched()
    plain = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, b, plain, False, b_mn, False, ctas=1, block_n=block_n)
    assert torch.equal(out.view, plain)
    _record("wait_a", ("dense", "NN" if b_mn else "NT", "bf16", block_n, 1, "wait_a"), r)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("unit_mult", [1, 2])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_rs_d(ops, world, unit_mult, b_mn, block_n):
    br = 32 * unit_mult
    M, N, K = world * 3 * br, 200, 136  # three blocks per rank
    rows_local = M // world
    a = padded(M, K, 8, device=DEV)
    _, b = _operands(M, N, K, False, b_mn)
    owners = shard_rows(a, world, br)
    prod, S = matmul_ref(a, b, False, b_mn)
    plain = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, b, plain, False, b_mn, False, ctas=1, block_n=block_n)
    worst = 0.0
    for zero_init in (False, True):
        inits = [torch.zeros(rows_local, N, device=DEV).bfloat16() if zero_init else torch.randn(rows_local, N, device=DEV).bfloat16()
                 for _ in range(world)]
        outs = [Canaried(rows_local, N, torch.bfloat16, tma=True, device=DEV, init=i) for i in inits]
        ops.gemm_rs_d(a, b, [o.view.data_ptr() for o in outs], rows_local, outs[0].view.stride(0), br, b_mn, block_n=block_n)
        for r, (o, init) in enumerate(zip(outs, inits)):
            ref, bound = gemm_bound(prod[owners[r]], S[owners[r]], K, torch.bfloat16, d0=init)
            worst = max(worst, assert_within(o.view, ref, bound, f"gemm_rs_d shard {r}"))
            o.assert_untouched()
            if zero_init:  # 0 + rn(acc) == the plain bf16 store
                assert torch.equal(o.view, plain[owners[r]])
    _record("rs_d", ("dense", "NN" if b_mn else "NT", "bf16_acc", block_n, 1, "rs_d"), worst)


def _run_ag_k(ops, world, br, nb, M, N, peer_is_a, epi, block_n, k_splits=0):
    T = world * nb * br  # token (reduction) dim
    out_dtype, acc = EPIS[epi]
    x = padded(T, M, 8, device=DEV)  # A: [tokens, M], MN-major
    y = padded(T, N, 8, device=DEV)  # B: [tokens, N], MN-major
    _, shards = _shards(x if peer_is_a else y, world, br)
    local = y if peer_is_a else x
    d0 = torch.randn(M, N, device=DEV).to(out_dtype) if acc else None
    out = Canaried(M, N, out_dtype, tma=True, device=DEV, init=d0)
    ops.gemm_ag_k(local, [s.data_ptr() for s in shards], peer_is_a, T // world, shards[0].stride(0), br, out.view, acc,
                  block_n=block_n, k_splits=k_splits)
    prod, S = matmul_ref(x, y, True, True)
    splits = k_splits if k_splits else max(1, T // 64 // 8)
    ref, bound = gemm_bound(prod, S, T, out_dtype, d0=d0, k_splits=splits)
    r = assert_within(out.view, ref, bound, "gemm_ag_k")
    out.assert_untouched()
    _record(f"ag_k/{epi}", ("dense", "TN", epi, block_n, 1, "ag_ka" if peer_is_a else "ag_kb"), r)


@pytest.mark.parametrize("world,unit_mult", [(1, 1), (2, 2), (3, 1), (8, 2)])
@pytest.mark.parametrize("peer_is_a", [False, True])
@pytest.mark.parametrize("epi", ["bf16", "f32", "f32_acc"])
@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_ag_k(ops, world, unit_mult, peer_is_a, epi, block_n):
    _run_ag_k(ops, world, 64 * unit_mult, 2, 136, 200, peer_is_a, epi, block_n)


@pytest.mark.parametrize("peer_is_a", [False, True])
@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("k_splits", [0, 5])
def test_gemm_ag_k_split_over_peer_shards(ops, peer_is_a, block_n, k_splits):
    # few output tiles and 8192 tokens: the fp32-accumulate epilogue splits K, and the slices cross the peers' shards
    _run_ag_k(ops, 8, 64, 16, 256, 256, peer_is_a, "f32_acc", block_n, k_splits)
