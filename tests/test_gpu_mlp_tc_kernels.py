"""mm_mlp_tc, the whole-tower kernel (models_b200/csrc/mlp_tc.cu), at every variant mlp_tc_impl dispatches: the kernel
for each padded layer-1 width N1P (16, 32, ..., 128) with the single-head or the multi-head epilogue, each chain layer's
compile-time (Np, KS) (padded width, 4 or 8 k-steps of its input), ring depths of 4 to 12 slots with a tile's slots
wrapping mid-tile, all seven activations at layer 1 and at a chain layer, and every output: fp32 rows (row stride N or
more, odd N), the fused Dense(N -> 1) head with and without those rows, H <= 8 fused heads, the split-bf16 operand rows
of mm_mlp_tc_operand_out with and without fp32 rows, and the pairs hand-off of mm_mlp_tc_pairs at 1 to 31 DLRM tables.
`plan` restates plan_tower; tests/test_mlp_tc_host.py pins it to the library and checks, without a GPU, that the case
tables below reach every variant.

Each case compares EVERY output element with float64 computed on the device, within the bounds documented in
tests/test_gpu_dense_tc_kernels.py (E = 2^-24, UNIT = 3 * 2^-16 per split-bf16 product, _chain over the layers):
  * a chain layer's A operand is the split of the previous layer's fp32 activations, so every layer is one more step
    of _chain with UNIT, its K the previous layer's true width;
  * a fused head is an fp32 dot of N products plus its bias, each product rounded into the running sum once, and the
    head's activation: one more step of _chain with unit E (N + 1 roundings of the absolute terms);
  * a split-bf16 output row hi + lo is within 2^-16 of its fp32 value, and with fp32 rows it is their split bit for bit.
A dropped cross term, a lost bias, a wrong activation, a swapped head or a lost column moves an element by far more.

The data has rows of exact zeros (with a bias that is zero in every third column, the pre-activation is exactly 0:
relu's mask), rows scaled by 40 (sigmoid and tanh saturate, selu / elu / gelu reach their negative tails) and values on
both sides of 0.  Every output is a view of a NaN buffer with guard rows past M (and, for fp32 rows, guard columns
beside the view); nothing outside the view may be written."""
import ctypes
from collections import namedtuple

import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, blocks, datasets, ops
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import helpers as H
from tests.test_gpu_dense_tc_kernels import ACTS, UNIT, _f32_out, _f32_untouched, padded_k, padded_n
from tests.test_gpu_forward_scale import SPLIT, _chain, _nan_bf16
from tests.test_gpu_mlp_tc_tiles import _tiles_per_cta
from tests.test_gpu_pairs_handoff import _rows_and_guarded_bottom, _same
from tests.test_gpu_train_scale import E, GUARD, _nan, _within

pytestmark = pytest.mark.gpu
SMEM = 227 * 1024
SMS = 132  # SMs of an H100 SXM: the lap case is sized for it (and asserted on the device's own count)
TILE = 64  # rows of one tile: one consumer warpgroup's wgmma M


# ---------------------------------------------------------------------------------------------------------------
# the launcher, restated
# ---------------------------------------------------------------------------------------------------------------
def plan(K, widths, heads=False):
    """plan_tower: padded layer-1 K and width, each chain layer's (Np, Kp, KS) and resident weight bytes, the ring depth
    (4..12 slots of one half k-block each, at most 4 per layer-1 k-block) and whether the tower fits in shared memory.
    heads: the multi-head epilogue's larger head staging."""
    K1p, N1p = padded_k(K), padded_n(widths[0])
    chain, prev = [], widths[0]
    for n in widths[1:]:
        Np, Kp = padded_n(n), padded_k(prev)
        chain.append(dict(Np=Np, Kp=Kp, KS=Kp // 16, w_bytes=2 * (Kp // 64) * Np * 64 * 2))
        prev = n
    w_bytes = sum(c["w_bytes"] for c in chain)
    stage = TILE * 64 * 2 + N1p * 64 * 2
    head_floats = 8 * 128 + 8 if heads else 128
    fixed = 1024 + w_bytes + 40 * 8 + (4 * 128 + head_floats) * 4
    KB = K1p // 64
    stages = min((SMEM - fixed) // stage, 12, 4 * KB)
    return dict(K1p=K1p, N1p=N1p, KB=KB, chain=chain, w_bytes=w_bytes, stages=stages, fits=fixed + 4 * stage <= SMEM)


def supported(K, widths, with_head=0):
    """mm_mlp_tc_supported: 2..4 layers of width 1..128, the last <= 32 under a fused head, and the plan fits."""
    if K <= 0 or not 2 <= len(widths) <= 4 or not all(1 <= w <= 128 for w in widths):
        return False
    if with_head and widths[-1] > 32:
        return False
    return plan(K, widths, heads=with_head > 1)["fits"]


def wraps(p):
    """A tile's 2 KB slots wrap around the ring mid-tile and the next tile starts at another slot."""
    return 2 * p["KB"] > p["stages"] and (2 * p["KB"]) % p["stages"] != 0


def tiles_per_cta(M, sms=SMS):
    """The tile counts of the CTAs (one per SM, 64-row tiles in blockIdx order)."""
    tiles = -(-M // TILE)
    grid = min(tiles, sms)
    return {tiles // grid + (1 if c < tiles % grid else 0) for c in range(grid)}


# ---------------------------------------------------------------------------------------------------------------
# case tables (importable without CUDA)
# ---------------------------------------------------------------------------------------------------------------
Rows = namedtuple("Rows", "M K widths acts bias layout")  # mm_mlp_tc, fp32 rows
Head = namedtuple("Head", "M K widths acts head_act layout")  # mm_mlp_tc, the fused head alone and with fp32 rows
Heads = namedtuple("Heads", "M K widths acts H")  # mm_mlp_tc_heads
Operand = namedtuple("Operand", "M K widths acts layout")  # mm_mlp_tc_operand_out, alone and with fp32 rows
Pairs = namedtuple("Pairs", "M K widths acts layout H")  # mm_mlp_tc_pairs: fp32 rows, a sigmoid head, H heads

LAPS_M = 400 * TILE - 37  # 400 tiles on 132 SMs: 4 CTAs run 4 tiles, 128 run 3

ROWS = [
    Rows(1, 13, (128, 100, 7), ("tanh", "selu", "linear"), True, "dense"),
    Rows(63, 415, (16, 128, 80), ("gelu", "sigmoid", "relu"), True, "vec"),
    Rows(64, 200, (33, 80), ("elu", "gelu"), False, "odd"),
    Rows(65, 129, (80, 96, 112, 63), ("selu", "elu", "tanh", "sigmoid"), True, "off1"),
    Rows(129, 300, (96, 30), ("sigmoid", "tanh"), True, "vec"),
    Rows(LAPS_M, 415, (128, 64, 32), ("relu", "relu", "relu"), True, "odd"),
    Rows(1001, 67, (112, 17), ("linear", "elu"), True, "dense"),
    Rows(300, 560, (64, 127), ("relu", "gelu"), True, "vec"),
    Rows(777, 100, (32, 1), ("tanh", "relu"), True, "off1"),
]

HEAD = [
    Head(1001, 415, (128, 64, 32), ("relu", "relu", "relu"), "sigmoid", "dense"),
    Head(129, 65, (48, 96, 24), ("gelu", "relu", "selu"), "tanh", "odd"),
    Head(63, 1, (16, 16), ("sigmoid", "linear"), "gelu", "vec"),
    Head(65, 250, (112, 80, 9), ("elu", "tanh", "gelu"), "elu", "off1"),
    Head(1, 129, (64, 48, 32, 32), ("linear", "sigmoid", "relu", "tanh"), "selu", "dense"),
    Head(777, 64, (96, 1), ("relu", "selu"), "linear", "vec"),
    Head(300, 200, (80, 20), ("tanh", "elu"), "relu", "odd"),
    Head(129, 100, (32, 112, 31), ("selu", "elu", "linear"), "sigmoid", "off1"),
]

# one case per padded layer-1 width, H = 1, 3 and 8 heads; head h of case i takes ACTS[(i + h) % 7]
HEADS = [
    Heads(129, 64, (10, 20), ("relu", "gelu"), 1),
    Heads(1, 415, (32, 64, 32), ("sigmoid", "relu", "tanh"), 3),
    Heads(1001, 100, (40, 32), ("selu", "elu"), 8),
    Heads(65, 560, (64, 48, 5), ("elu", "linear", "relu"), 1),
    Heads(300, 200, (75, 128, 32), ("gelu", "tanh", "sigmoid"), 3),
    Heads(64, 13, (90, 16), ("tanh", "selu"), 8),
    Heads(777, 129, (100, 48, 32, 24), ("linear", "gelu", "elu", "relu"), 3),
    Heads(63, 300, (128, 32), ("relu", "sigmoid"), 8),
]

# the last width is a multiple of 4; fp32 rows beside the operand need 16-byte aligned rows (dense or vec)
OPERAND = [
    Operand(1000, 13, (128, 64), ("relu", "relu"), "dense"),
    Operand(129, 99, (56, 36), ("selu", "linear"), "vec"),
    Operand(65, 415, (96, 128, 4), ("tanh", "gelu", "elu"), "dense"),
    Operand(1, 64, (20, 100), ("sigmoid", "sigmoid"), "vec"),
    Operand(63, 300, (80, 96, 64, 8), ("elu", "relu", "tanh", "gelu"), "vec"),
]

# K = 64 + F (F - 1) / 2 for F = 2, 3, 9, 27 and 32 features (1, 2, 8, 26 and 31 tables beside the bottom vector)
PAIRS_K = (65, 67, 100, 415, 560)
PAIRS = [
    Pairs(1001, 65, (48, 32), ("relu", "relu"), "odd", 3),
    Pairs(129, 67, (80, 64, 32), ("relu", "relu", "relu"), "dense", 1),
    Pairs(64, 100, (16, 16), ("gelu", "tanh"), "vec", 8),
    Pairs(65, 415, (128, 64, 32), ("relu", "relu", "relu"), "off1", 3),
    Pairs(777, 560, (112, 96, 28), ("selu", "sigmoid", "elu"), "dense", 8),
]


def case_id(c):
    return f"M{c.M}-K{c.K}-{'x'.join(map(str, c.widths))}-{'.'.join(c.acts)}"


def heads_acts(i, H):
    return [ACTS[(i + h) % 7] for h in range(H)]


# ---------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------
def _tower(M, K, widths, seed, device, bias=True):
    """x (M, K) with rows of exact zeros (every 7th) and rows scaled by 40 (every 5th), W_l (k, n) / sqrt(k), b_l zero in
    every third column (or None), and the split operands: (x, Ws, bs, a_split, w_splits)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((M, K), generator=g, device=device)
    r = torch.arange(M, device=device)
    x[r % 7 == 3] = 0.0
    x[r % 5 == 1] *= 40.0
    Ws, bs, k = [], [], K
    for n in widths:
        Ws.append(torch.randn((k, n), generator=g, device=device) / k ** 0.5)
        b = torch.randn(n, generator=g, device=device) * 0.5
        b[1::3] = 0.0
        bs.append(b if bias else None)
        k = n
    return x, Ws, bs, ops.split_rows(x), [ops.split_weights(W) for W in Ws]


def _reference(x, Ws, bs, acts):
    return _chain(x.double(), list(zip(Ws, bs, acts)), unit=UNIT)


def _head_reference(y, ey, hw, hb, act):
    """One fused head over the float64 tower output y (within ey of the device's): an fp32 dot, bias, activation."""
    N = hw.numel()
    h, eh = _chain(y, [(hw.reshape(N, 1), hb.reshape(1), act)], ey, unit=E)
    return h[:, 0], eh[:, 0]


def _head_weights(N, H, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn((N, H), generator=g, device=device) / N ** 0.5, torch.randn(H, generator=g, device=device) * 0.5


def _guarded(n, device):
    """A NaN vector of n + GUARD values: (buffer, its first n)."""
    buf = _nan((n + GUARD,), device)
    return buf, buf[:n]


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------
# 1. mm_mlp_tc: fp32 rows at every layer-1 kernel, chain variant, ring depth and activation
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", ROWS, ids=lambda c: f"{case_id(c)}-{c.layout}")
def test_mlp_tc_rows_match_float64(device, c):
    """fp32 rows in the case's layout, within _chain's bound; a repeat call writes the same bits."""
    if c.M == LAPS_M:
        counts = _tiles_per_cta(c.M)
        assert max(counts) >= 3 and {n % 2 for n in counts} == {0, 1}, f"premise: tiles per CTA {sorted(counts)}"
    N = c.widths[-1]
    x, Ws, bs, a, ws = _tower(c.M, c.K, c.widths, ROWS.index(c), device, bias=c.bias)
    fb, fv, col = _f32_out(c.M, N, c.layout, device)
    ops.mlp_tc(a, c.K, ws, list(c.widths), bs, list(c.acts), out=fv)
    _f32_untouched(fb, c.M, col, N, "out_f32")
    y, ey = _reference(x, Ws, bs, c.acts)
    _within(fv, y, ey, f"out_f32 ({'/'.join(c.acts)})")
    again, av, _ = _f32_out(c.M, N, c.layout, device)
    ops.mlp_tc(a, c.K, ws, list(c.widths), bs, list(c.acts), out=av)
    assert torch.equal(_bits(again), _bits(fb)), "a repeat call is not bit-identical"


# ---------------------------------------------------------------------------------------------------------------
# 2. the fused Dense(N -> 1) head, alone and with the fp32 rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", HEAD, ids=lambda c: f"{case_id(c)}-head_{c.head_act}")
def test_mlp_tc_head_matches_float64(device, c):
    """head_out[m] = head_act(tower(x)[m] . head_w + head_b): with fp32 rows and alone, bit for bit the same."""
    N = c.widths[-1]
    i = HEAD.index(c)
    x, Ws, bs, a, ws = _tower(c.M, c.K, c.widths, 100 + i, device)
    hw, hb = _head_weights(N, 1, 100 + i, device)
    hw, hb32 = hw[:, 0].contiguous(), float(hb[0])
    fb, fv, col = _f32_out(c.M, N, c.layout, device)
    h1b, h1 = _guarded(c.M, device)
    h2b, h2 = _guarded(c.M, device)
    args = (a, c.K, ws, list(c.widths), bs, list(c.acts))
    ops.mlp_tc(*args, out=fv, head_w=hw, head_b=hb32, head_act=c.head_act, head_out=h1)
    ops.mlp_tc(*args, head_w=hw, head_b=hb32, head_act=c.head_act, head_out=h2)
    _f32_untouched(fb, c.M, col, N, "out_f32 beside the head")
    for buf, what in ((h1b, "head with rows"), (h2b, "head alone")):
        assert bool(torch.isnan(buf[c.M:]).all()), f"{what}: a guard element past M was written"
    assert torch.equal(_bits(h2), _bits(h1)), "the head alone differs from the head beside the fp32 rows"
    y, ey = _reference(x, Ws, bs, c.acts)
    _within(fv, y, ey, "out_f32 beside the head")
    h, eh = _head_reference(y, ey, hw, torch.tensor([hb32], device=device), c.head_act)
    _within(h1, h, eh, f"head ({c.head_act})")


# ---------------------------------------------------------------------------------------------------------------
# 3. mm_mlp_tc_heads: the multi-head kernel at every padded layer-1 width
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", HEADS, ids=lambda c: f"{case_id(c)}-H{c.H}")
def test_mlp_tc_heads_matches_float64(device, c):
    """out[h] = heads_act[h](tower(x) @ heads_w[:, h] + heads_b[h]) with mixed activations and the biases read from
    the device, into (H, M) of a NaN buffer with guards past it."""
    N, i = c.widths[-1], HEADS.index(c)
    x, Ws, bs, a, ws = _tower(c.M, c.K, c.widths, 200 + i, device)
    hw, hb = _head_weights(N, c.H, 200 + i, device)
    acts = heads_acts(i, c.H)
    buf, flat = _guarded(c.H * c.M, device)
    out = flat.view(c.H, c.M)
    ops.mlp_tc_heads(a, c.K, ws, list(c.widths), bs, list(c.acts), hw, hb, acts, out)
    assert bool(torch.isnan(buf[c.H * c.M:]).all()), "heads: a guard element past the output was written"
    y, ey = _reference(x, Ws, bs, c.acts)
    for h, act in enumerate(acts):
        want, bound = _head_reference(y, ey, hw[:, h], hb[h], act)
        _within(out[h], want, bound, f"head {h} of {c.H} ({act})")


# ---------------------------------------------------------------------------------------------------------------
# 4. mm_mlp_tc_operand_out: the split-bf16 rows of the next kernel's operand, alone and with fp32 rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", OPERAND, ids=lambda c: f"{case_id(c)}-{c.layout}")
def test_mlp_tc_operand_out_matches_float64(device, c):
    """Rows (M, 2 N) = [hi | lo] at a pitch of 4 N bytes: with fp32 rows, their split bit for bit and hi + lo within
    2^-16 of them; alone, the same bits, within the float64 bound plus 2^-16.  Rows past M stay NaN."""
    N = c.widths[-1]
    x, Ws, bs, a, ws = _tower(c.M, c.K, c.widths, 300 + OPERAND.index(c), device)
    args = (a, c.K, ws, list(c.widths), bs, list(c.acts))
    ob1 = _nan_bf16((c.M + GUARD, 2 * N), device)
    ob2 = _nan_bf16((c.M + GUARD, 2 * N), device)
    fb, fv, col = _f32_out(c.M, N, c.layout, device)
    ops.mlp_tc(*args, out=fv, out_operand=ob1[:c.M])
    ops.mlp_tc(*args, out_operand=ob2[:c.M])
    _f32_untouched(fb, c.M, col, N, "out_f32 beside the operand")
    for ob, what in ((ob1, "operand with rows"), (ob2, "operand alone")):
        assert bool(torch.isnan(ob[c.M:].float()).all()), f"{what}: a guard row past M was written"
    Kp = padded_k(N)
    sp = ops.split_rows(fv.contiguous())
    assert torch.equal(ob1[:c.M, :N], sp[:, :N]) and torch.equal(ob1[:c.M, N:], sp[:, Kp:Kp + N]), \
        "operand rows are not split_rows(out_f32) bit for bit"
    assert torch.equal(_bits(ob2), _bits(ob1)), "the operand alone differs from the operand beside the fp32 rows"
    hilo = ob1[:c.M, :N].double() + ob1[:c.M, N:].double()
    _within(hilo, fv.double(), SPLIT * fv.double().abs(), "hi + lo against the fp32 rows")
    y, ey = _reference(x, Ws, bs, c.acts)
    _within(fv, y, ey, "out_f32 beside the operand")
    _within(hilo, y, ey + SPLIT * (y.abs() + ey), "operand hi + lo")


# ---------------------------------------------------------------------------------------------------------------
# 5. mm_mlp_tc_pairs: k-block 0 from the bottom rows, the rest from the pairs rows
# ---------------------------------------------------------------------------------------------------------------
def _pairs_rows(a, M, K, device):
    """(bottom rows (M, 128) in a buffer with NaN rows past M, pairs rows (M, 2 pairs_cols(K - 64)) with NaN padding
    columns) holding the columns of the concatenated split rows a (M, 2 K1p)."""
    K1p, n = padded_k(K), K - 64
    kq = ops.pairs_cols(n)
    guard = _nan_bf16((M + GUARD, 128), device)
    guard[:M, :64] = a[:, :64]
    guard[:M, 64:] = a[:, K1p:K1p + 64]
    pairs = _nan_bf16((M, 2 * kq), device)
    pairs[:, :n] = a[:, 64:K]
    pairs[:, kq:kq + n] = a[:, K1p + 64:K1p + K]
    return guard[:M], pairs


@pytest.mark.parametrize("c", PAIRS, ids=lambda c: f"{case_id(c)}-{c.layout}-H{c.H}")
def test_mlp_tc_pairs_matches_concatenated_and_float64(device, c):
    """fp32 rows, a fused sigmoid head and H heads from bottom + pairs rows: (a) byte-identical to mm_mlp_tc over the
    concatenated [bottom | pairs] split rows, (b) within the float64 bound."""
    N, i = c.widths[-1], PAIRS.index(c)
    x, Ws, bs, a, ws = _tower(c.M, c.K, c.widths, 400 + i, device)
    bottom, pairs = _pairs_rows(a, c.M, c.K, device)
    args = (c.K, ws, list(c.widths), bs, list(c.acts))
    hw, hb = _head_weights(N, c.H, 400 + i, device)
    acts = heads_acts(i, c.H)
    y, ey = _reference(x, Ws, bs, c.acts)
    got = []
    for src, kw in ((a, {}), (pairs, dict(a_bottom=bottom))):
        fb, fv, col = _f32_out(c.M, N, c.layout, device)
        h1b, h1 = _guarded(c.M, device)
        hsb, hs = _guarded(c.H * c.M, device)
        ops.mlp_tc(src, *args, out=fv, **kw)
        ops.mlp_tc(src, *args, head_w=hw[:, 0].contiguous(), head_b=float(hb[0]), head_act="sigmoid", head_out=h1, **kw)
        ops.mlp_tc_heads(src, *args, hw, hb, acts, hs.view(c.H, c.M), **kw)
        got.append((fb, h1b, hsb))
    for (old, new), what in zip(zip(*got), ("fp32 rows", "head", "heads")):
        assert torch.equal(_bits(new), _bits(old)), f"pairs hand-off {what}: not byte-identical to the concatenated rows"
    fb, h1b, hsb = got[1]
    _f32_untouched(fb, c.M, col, N, "pairs out_f32")
    assert bool(torch.isnan(h1b[c.M:]).all()) and bool(torch.isnan(hsb[c.H * c.M:]).all()), "a guard past M was written"
    _within(fb[:c.M, col:col + N], y, ey, "pairs out_f32")
    h, eh = _head_reference(y, ey, hw[:, 0], hb[0], "sigmoid")
    _within(h1b[:c.M], h, eh, "pairs head")
    for j, act in enumerate(acts):
        h, eh = _head_reference(y, ey, hw[:, j], hb[j], act)
        _within(hsb[j * c.M:(j + 1) * c.M], h, eh, f"pairs head {j} of {c.H} ({act})")


# ---------------------------------------------------------------------------------------------------------------
# 6. DLRMModel takes the hand-off at every table count
# ---------------------------------------------------------------------------------------------------------------
def _dlrm_schema(T, targets):
    cols = [ColumnSchema(f"C{t}", tags=(Tags.CATEGORICAL,), dtype="int64",
                         properties={"domain": {"min": 0, "max": 500 + 37 * t, "name": f"C{t}"}}) for t in range(T)]
    cols += [ColumnSchema(f"I{i}", tags=(Tags.CONTINUOUS,), dtype="float32") for i in range(1, 14)]
    for name, tag in targets:
        cols.append(ColumnSchema(name, tags=(Tags.TARGET, tag), dtype="float32" if tag == Tags.REGRESSION else "int64"))
    return Schema(cols)


# (tables, top tower, multi-task): layer-1 widths 48 and 80 (N1P never reached by the 128-wide default tower)
E2E = [(1, (48, 32), False), (2, (80, 32), False), (8, (48, 16), False), (31, (80, 64, 32), False), (8, (80, 32), True)]


@pytest.mark.parametrize("T,top,multi", E2E, ids=lambda v: str(v))
def test_dlrm_takes_the_pairs_handoff(device, monkeypatch, T, top, multi):
    """DLRMModel(embedding_dim=64) with T tables: its forward hands the tower the bottom rows (a_bottom), and its
    predictions equal the tower over the concatenated [bottom | pairs] rows byte for byte."""
    B = 1001
    targets = [("click", Tags.BINARY_CLASSIFICATION), ("rating", Tags.REGRESSION)] if multi else \
        [("label", Tags.BINARY_CLASSIFICATION)]
    schema = _dlrm_schema(T, targets)
    mm.set_seed(T)
    kw = dict(prediction_tasks=mm.OutputBlock(schema)) if multi else {}
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock(list(top)), **kw)
    feats = datasets.generate_batch(schema.excluding_by_tag(Tags.TARGET), B, seed=T, index_law="uniform")
    inputs = H.device_batch(feats, device)
    model.build(device)
    model(inputs)  # builds the heads
    K = model.body.output_width_before_top()
    assert K == 64 + (T + 1) * T // 2
    _, full, _ = _rows_and_guarded_bottom(model, inputs, B, device)

    seen = []
    for name in ("mlp_tc", "mlp_tc_heads"):
        def wrap(*args, _f=getattr(ops, name), _n=name, **kwargs):
            seen.append((_n, kwargs.get("a_bottom") is not None))
            return _f(*args, **kwargs)
        monkeypatch.setattr(ops, name, wrap)
    got = model(inputs)
    assert seen and seen[-1] == ("mlp_tc_heads" if multi else "mlp_tc", True), f"the top tower did not take the hand-off: {seen}"
    if multi:
        heads = model.prediction
        want = heads.split(blocks.run_dense_chain(None, model.body.top_block.dense_layers, a_split=full, K=K, heads=heads))
        got = got.outputs if isinstance(got, mm.Prediction) else got
        assert list(got) == list(want)
        for k in want:
            _same(got[k], want[k], f"output {k}")
    else:
        layers, _ = model.body.top_block.chain([model.prediction.to_call])
        _same(got, blocks.run_dense_chain(None, layers, a_split=full, K=K), "predictions")


# ---------------------------------------------------------------------------------------------------------------
# 7. M = 0
# ---------------------------------------------------------------------------------------------------------------
def test_mlp_tc_zero_rows_writes_nothing(device):
    """M = 0 through the four C entries with real buffers: every output, fp32 rows, head, heads and operand rows, keeps
    its NaN."""
    K, widths, acts = 100, [48, 32], ["gelu", "relu"]
    x, Ws, bs, a, ws = _tower(GUARD, K, widths, 7, device)
    bottom, pairs = _pairs_rows(a, GUARD, K, device)
    _, n, wp, wd, bp, ac = ops._tower("mlp_tc", a, K, ws, widths, bs, acts)
    hw, hb = _head_weights(32, 3, 7, device)
    ha = (ctypes.c_int * 3)(*[_cabi.ACTIVATIONS[h] for h in ("sigmoid", "tanh", "gelu")])
    fb, hb1, hsb = _nan((GUARD, 32), device), _nan((GUARD,), device), _nan((3 * GUARD,), device)
    ob = _nan_bf16((GUARD, 64), device)
    lib, st = _cabi.load(), torch.cuda.current_stream().cuda_stream
    sig = _cabi.ACTIVATIONS["sigmoid"]
    w0 = hw[:, 0].contiguous()
    _cabi.check(lib.mm_mlp_tc(a.data_ptr(), 0, K, n, wp, wd, bp, ac, fb.data_ptr(), 32, w0.data_ptr(), 0.5, sig,
                              hb1.data_ptr(), st), "mm_mlp_tc")
    _cabi.check(lib.mm_mlp_tc_heads(a.data_ptr(), 0, K, n, wp, wd, bp, ac, 3, hw.data_ptr(), hb.data_ptr(), ha,
                                    hsb.data_ptr(), st), "mm_mlp_tc_heads")
    _cabi.check(lib.mm_mlp_tc_operand_out(a.data_ptr(), 0, K, n, wp, wd, bp, ac, fb.data_ptr(), 32, ob.data_ptr(), st),
                "mm_mlp_tc_operand_out")
    _cabi.check(lib.mm_mlp_tc_pairs(bottom.data_ptr(), pairs.data_ptr(), 0, K, n, wp, wd, bp, ac, fb.data_ptr(), 32,
                                    w0.data_ptr(), 0.5, sig, hb1.data_ptr(), 0, None, None, st), "mm_mlp_tc_pairs")
    _cabi.check(lib.mm_mlp_tc_pairs(bottom.data_ptr(), pairs.data_ptr(), 0, K, n, wp, wd, bp, ac, None, 0,
                                    hw.data_ptr(), 0.0, 0, hsb.data_ptr(), 3, hb.data_ptr(), ha, st), "mm_mlp_tc_pairs (heads)")
    torch.cuda.synchronize()
    for t, what in ((fb, "out_f32"), (hb1, "head_out"), (hsb, "heads_out"), (ob, "out_operand")):
        assert bool(torch.isnan(t.float()).all()), f"M = 0 wrote {what}"
