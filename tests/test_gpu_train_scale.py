"""The training-step kernels at the sizes the benchmark trains with: B = 65 536 for DLRM (full Criteo-shaped tables, packed
1/2/3-byte ids, Adagrad, one CUDA graph) and B = N = 16 384 for the two-tower in-batch soft-max.  At the small batches of
the per-kernel tests every grid-stride loop finishes in one lap; here each kernel runs its steady state (buffers flipped
and refilled, tiles revisited, thousands of duplicate ids per row), and every large-B test asserts that premise from the
launcher's own formula and the device's SM count.

References are float64 on the device, in sample chunks.  Tolerances are per element and derived from the arithmetic:
a 3-pass split-bf16 product is exact to U = 2^-16 of |a b|, an fp32 sum of n terms is within (n - 1) 2^-24 of the sum
of the absolute terms.  A lost or repeated lap changes a result by at least 1 / laps of its scale, far above those
bounds.  Output buffers carry NaN-filled guard rows past B and padding columns; they must stay NaN."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200._cabi import HYPER_BETA1, HYPER_BETA2, HYPER_EPS, HYPER_LR, HYPER_LR_T
from models_b200.graph import HostBatch, _view
from models_b200.train import DENSE_PATH_MAX_ROWS
from tests import twotower_train_oracle as O
from tests.test_gpu_lookup_v2 import pack_ids
from tests.test_gpu_train import _interaction_ref
from tests.test_gpu_train_twotower import _ce_case, allclose

pytestmark = pytest.mark.gpu
U = 2.0 ** -16  # relative accuracy of one 3-pass split-bf16 product
E = 2.0 ** -24  # fp32 unit round-off
BIG = 65536
RAGGED = BIG + 37  # leaves a ragged last lap
GUARD = 8  # NaN rows past the batch in every output buffer
INT_MAX = 2 ** 31 - 1


def _sms(device) -> int:
    return torch.cuda.get_device_properties(device).multi_processor_count


def _nan(shape, device):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=device)


def _within(got, ref, bound, what):
    """|got - ref| <= bound element-wise (NaN anywhere fails)."""
    err = (got.double() - ref.double()).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        ratio = float((err / bound.clamp_min(1e-300)).max())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off (first at flat index {i}: got "
                             f"{float(got.reshape(-1)[i])}, want {float(ref.reshape(-1)[i])}, bound {float(bound.reshape(-1)[i]):.3e}); "
                             f"worst |err| / bound = {ratio:.3g}")


def _untouched(buf, rows, cols, what):
    """Rows >= `rows` and columns >= `cols` of a NaN-filled output buffer were not written."""
    assert bool(torch.isnan(buf[rows:]).all()), f"{what}: a guard row past the batch was written"
    if buf.shape[1] > cols:
        assert bool(torch.isnan(buf[:, cols:]).all()), f"{what}: a padding column was written"


# ---------------------------------------------------------------------------------------------------------------
# 1. mm_dlrm_interact_backward
# ---------------------------------------------------------------------------------------------------------------
def _ibwd_grid(B, D, F, P, operand, sms):
    """(warps per CTA, CTAs) as launch_ibwd / launch_ibwd_ps in train_sparse.cu choose them."""
    OW = P + F * (F - 1) // 2
    stage_floats = ((OW + 3) & ~3) + 4
    if operand:
        stage_off = (256 + (F * (F - 1) // 2) * 2 + 255) & ~255
        buf = (F * 256 + stage_floats * 4 + 2 * 32 * 80 + 15) & ~15
        warps = min((227 * 1024 - stage_off) // buf, 16)
    else:
        stage_off = 32 * (D + 4) * 4
        buf = (stage_off + stage_floats * 4 + 15) & ~15
        warps = min((227 * 1024) // (2 * buf), 8)
    return warps, min(-(-B // warps), sms)


WIDTHS = (1, 2, 3, 4, 8)


def _width_rows(w, t):
    return {1: 200, 2: 5000, 3: 70000, 4: 70000, 8: 70000}[w] + (t if w == 1 else 7 * t)


def _ids_with_oob(rng, rows, w, B):
    """Uniform ids in [0, rows) with ~1 % of them outside the table at the width's range (negative for signed widths)."""
    ids = rng.integers(0, rows, B)
    k = max(1, B // 100)
    at = rng.choice(B, k, replace=False)
    hi = {1: 256, 2: 65536, 3: 1 << 24, 4: 1 << 31, 8: 1 << 40}[w]
    ids[at] = rng.integers(rows, hi, k)
    if w >= 4:
        ids[at[: k // 2]] = -1 - rng.integers(0, 1000, k // 2)
    return ids


@pytest.mark.parametrize("D,operand,B", [(64, False, BIG), (64, False, RAGGED), (64, True, BIG), (64, True, RAGGED),
                                         (16, False, 8192), (16, False, 8192 + 37), (128, False, 8192), (128, False, 8192 + 37)])
def test_interact_backward_at_scale(device, D, operand, B):
    """Criteo shape (26 tables + the bottom vector, P = D), ids of every width (1, 2, 3, 4, 8 bytes) with ~1 % outside the
    table, fp32 rows or (D = 64) the split mirrors, the bottom mask on and off: every slice and d_bottom against float64
    autograd.  Bound per element 4 U (|G| |X|) (+ |dA| of the shortcut for d_bottom): every output is a sum of 27
    split-bf16 products (each within U of |g x|) accumulated in fp32 over six MMA steps (6 * 2^-24 << U); a stale or
    skipped sample is off by O(1) of that scale.  A sample is one warp's work, so the rows of a window launched alone
    must equal the full run's bit for bit."""
    T = 26
    F, P = T + 1, D
    warps, ctas = _ibwd_grid(B, D, F, P, operand, _sms(device))
    laps = -(-B // (warps * ctas))
    assert laps >= 2, f"premise: B = {B} gives {laps} lap(s) of {warps} warps x {ctas} CTAs"
    rng = np.random.default_rng(B + D + operand)
    gen = torch.Generator(device=device).manual_seed(B + D)
    widths = [WIDTHS[t % 5] for t in range(T)]
    rows = [_width_rows(w, t) for t, w in enumerate(widths)]
    tables = [torch.randn((r, D), generator=gen, device=device) * 0.3 for r in rows]
    ids64 = [_ids_with_oob(rng, r, w, B) for r, w in zip(rows, widths)]
    ids = [torch.from_numpy(pack_ids(i, w)).to(device) for i, w in zip(ids64, widths)]
    assert [ops.index_bytes_of(i) for i in ids] == widths
    names = sorted([f"C{t}" for t in range(T)] + ["bottom_block"])
    slot_b = names.index("bottom_block")
    slots = [s for s in range(F) if s != slot_b]
    bottom = torch.randn((B, D), generator=gen, device=device)
    bottom[:, ::3] = 0.0
    OW = P + F * (F - 1) // 2
    dA = torch.randn((B, (OW + 3) // 4 * 4), generator=gen, device=device)[:, :OW]
    w_in = [ops.split_rows(w) for w in tables] if operand else tables
    b_in = ops.split_rows(bottom) if operand else bottom

    gbuf = _nan((T, B + GUARD, D + 4), device)
    dbuf = _nan((B + GUARD, D + 4), device)

    def run(mask, lo=0, hi=B, g=None, db=None):
        g = [gbuf[t, :B, :D] for t in range(T)] if g is None else g
        db = dbuf[:B, :D] if db is None else db
        ops.dlrm_interact_backward(w_in, [i[lo:hi] for i in ids], slots, rows, D, b_in[lo:hi], slot_b, dA[lo:hi], g, db,
                                   mask_bottom=mask, operand_rows=operand)

    # float64 reference in chunks: values and the absolute-value bound
    dev_ids = [torch.from_numpy(i).to(device) for i in ids64]
    ref_rows, ref_bottom, abs_rows, abs_bottom = [], [], [], []
    for s in range(0, B, 8192):
        e = min(B, s + 8192)
        looked = []
        for t in range(T):
            i = dev_ids[t][s:e]
            ok = (i >= 0) & (i < rows[t])
            looked.append(tables[t][i.clamp(0, rows[t] - 1)] * ok.unsqueeze(1))
        r, b = _interaction_ref(looked, bottom[s:e], dA[s:e], slot_b, P)
        ra, ba = _interaction_ref([x.abs() for x in looked], bottom[s:e].abs(), dA[s:e].abs(), slot_b, P)
        ref_rows.append(r)
        ref_bottom.append(b)
        abs_rows.append(ra)
        abs_bottom.append(ba)
    ref_rows = [torch.cat([c[t] for c in ref_rows]) for t in range(T)]
    abs_rows = [torch.cat([c[t] for c in abs_rows]) for t in range(T)]
    ref_bottom, abs_bottom = torch.cat(ref_bottom), torch.cat(abs_bottom)
    on = bottom > 0
    for mask in (False, True):
        gbuf.fill_(float("nan"))
        dbuf.fill_(float("nan"))
        run(mask)
        for t in range(T):
            _within(gbuf[t, :B, :D], ref_rows[t], 4 * U * abs_rows[t], f"slices of table {t} ({widths[t]}-byte ids), mask {mask}")
            _untouched(gbuf[t], B, D, f"slices of table {t}")
        want = ref_bottom * on if mask else ref_bottom
        _within(dbuf[:B, :D], want, 4 * U * abs_bottom, f"d_bottom, mask {mask}")
        _untouched(dbuf, B, D, "d_bottom")
    # position independence: windows (first lap, mid-batch, the ragged end) launched alone, bit for bit
    for lo, w in ((0, 1000), (B // 2 + 3, 777), (B - 901, 901)):
        gw = torch.empty((T, w, D), device=device)
        dw = torch.empty((w, D), device=device)
        run(True, lo, lo + w, [gw[t] for t in range(T)], dw)
        for t in range(T):
            assert torch.equal(gw[t], gbuf[t, lo:lo + w, :D]), f"window [{lo}, {lo + w}): slices of table {t} depend on the position"
        assert torch.equal(dw, dbuf[lo:lo + w, :D]), f"window [{lo}, {lo + w}): d_bottom depends on the position"


# ---------------------------------------------------------------------------------------------------------------
# 2. mm_dense_dgrad / mm_dense_wgrad at the DLRM step's shapes
# ---------------------------------------------------------------------------------------------------------------
STEP_SHAPES = [(415, 128), (128, 64), (64, 32)]


def _dgrad_laps(M, K, sms):
    """Grid-stride laps of dgrad_kernel (launch_dgrad: 8 warps of 16 rows, grid capped at 2 SMs / ky)."""
    ky = -(-K // 128)
    tiles = -(-M // 16)
    gx = min(-(-tiles // 8), max(1, 2 * sms // ky))
    return -(-tiles // (gx * 8))


@pytest.mark.parametrize("store", ["vec4", "vec2", "scalar"])
@pytest.mark.parametrize("K,N", STEP_SHAPES)
@pytest.mark.parametrize("M", [BIG, RAGGED])
def test_dense_dgrad_at_scale(device, M, K, N, store):
    """dX = dZ W^T, without and with the relu mask, at a dX / mask row stride that is a multiple of 4 (16-byte stores
    through the shared-memory stage), even only (8-byte stores) or odd (scalar stores).  Bound per element
    4 U (|dZ| |W|^T): N <= 128 split-bf16 products (within U each), fp32 accumulation over <= 24 MMA steps (< U / 2).
    A 16-row tile is one warp's work, so windows aligned to 16 rows launched alone give the same rows bit for bit."""
    laps = _dgrad_laps(M, K, _sms(device))
    assert laps >= 2, f"premise: M = {M}, K = {K} gives {laps} lap(s)"
    ld = {"vec4": (K + 3) // 4 * 4, "vec2": (K + 3) // 4 * 4 + 2, "scalar": K if K % 2 else K + 1}[store]
    assert (ld % 4 == 0) == (store == "vec4") and (ld % 2 == 0) == (store != "scalar")
    gen = torch.Generator(device=device).manual_seed(M + K + ld)
    mbuf = torch.zeros((M, ld), device=device)
    mbuf[:, :K] = torch.randn((M, K), generator=gen, device=device).clamp_min(0.0)  # the layer input (relu output)
    mask = mbuf[:, :K]
    dz = torch.randn((M, N), generator=gen, device=device)
    W = torch.randn((K, N), generator=gen, device=device) * 0.1
    ref = dz.double() @ W.double().t()
    bound = 4 * U * (dz.double().abs() @ W.double().abs().t())
    buf = _nan((M + GUARD, ld), device)
    dx = buf[:M, :K]
    ops.dense_dgrad(dz, W, dx)
    _within(dx, ref, bound, f"dX (stride {ld})")
    _untouched(buf, M, K, "dX")
    buf.fill_(float("nan"))
    ops.dense_dgrad(dz, W, dx, mask=mask)
    _within(dx, ref * (mask > 0), bound, f"dX masked (stride {ld})")
    _untouched(buf, M, K, "dX masked")
    for lo, w in ((0, 800), (16 * 2049, 1600), ((M - 1600) // 16 * 16, M - (M - 1600) // 16 * 16)):
        wb = _nan((w, ld), device)
        ops.dense_dgrad(dz[lo:lo + w], W, wb[:, :K], mask=mask[lo:lo + w])
        assert torch.equal(wb[:, :K], dx[lo:lo + w]), f"window [{lo}, {lo + w}): dX rows depend on the position"


def _wgrad_launch(M, K, N, sms):
    """(rows per CTA, CTAs along the batch) as launch_wgrad in train_dense.cu chooses them."""
    ks = 128 if K > 64 else 64 if K > 16 else 16
    ns = 128 if N > 64 else 64 if N > 32 else 32
    ctas = max(1, 2 * sms // (-(-K // ks) * -(-N // ns)))
    rows = -(-M // ctas)
    rows = max(256, -(-rows // 32) * 32)
    return rows, -(-M // rows)


@pytest.mark.parametrize("K,N", STEP_SHAPES + [(13, 128)])
@pytest.mark.parametrize("M", [BIG, RAGGED])
def test_dense_wgrad_at_scale(device, M, K, N):
    """dW = X^T dZ and db = column sums of dZ from fp32 X at the trainer's padded stride (416 for the interaction output)
    and from the split operand.  A CTA accumulates `rows` batch rows in 32-row chunks (3 MMA passes per 16 rows), the CTAs
    meet in fp32 atomics: an element of dW is within (U + (3 rows / 16 + CTAs) 2^-24) (|X|^T |dZ|) of the exact sum
    (asserted at twice that), db within (rows + 256 + CTAs) 2^-24 sum |dZ|.  A lost 32-row chunk is 1 / (M / 32) of the
    scale on average, several times the dW bound."""
    rows, gx = _wgrad_launch(M, K, N, _sms(device))
    assert rows // 32 >= 2, f"premise: {rows} rows per CTA is a single chunk"
    gen = torch.Generator(device=device).manual_seed(M + 7 * K + N)
    ld = (K + 3) // 4 * 4
    xb = _nan((M, ld), device)
    xb[:, :K] = torch.randn((M, K), generator=gen, device=device).clamp_min(0.0)
    x = xb[:, :K]
    dz = torch.randn((M, N), generator=gen, device=device)
    xd, zd = x.double(), dz.double()
    ref_w, ref_b = xd.t() @ zd, zd.sum(0)
    bw = 2 * (U + (3 * rows / 16 + gx) * E) * (xd.abs().t() @ zd.abs())
    bb = 2 * (rows + 256 + gx) * E * zd.abs().sum(0)
    for split in (False, True):
        dw = torch.zeros((K, N), device=device)
        db = torch.zeros(N, device=device)
        if split:
            ops.dense_wgrad_split(ops.split_rows(x), K, dz, dw, db)
        else:
            ops.dense_wgrad(x, dz, dw, db)
        _within(dw, ref_w, bw, f"dW (split operand {split})")
        _within(db, ref_b, bb, f"db (split operand {split})")


# ---------------------------------------------------------------------------------------------------------------
# 3. mm_sparse_rows_apply at B = 65 536
# ---------------------------------------------------------------------------------------------------------------
def _rule(opt, w0, s1, s2, g, hyper):
    """Keras update in float64 with the optimizer's fp32 hyper-parameters as the device holds them (lr_t as mm_opt_tick
    computed it for this step): (new w, |d new w / d g| bound at g, the size of the terms the fp32 update rounds)."""
    lr, b1, b2, eps, lr_t = (float(hyper[i]) for i in (HYPER_LR, HYPER_BETA1, HYPER_BETA2, HYPER_EPS, HYPER_LR_T))
    if opt == "sgd":
        return w0 - lr * g, torch.full_like(g, lr), lr * g.abs()
    if opt == "adagrad":
        step = lr * g / ((s1 + g * g).sqrt() + eps)
        return w0 - step, lr / s1.sqrt(), step.abs()
    m = b1 * s2[0] + (1 - b1) * g
    v = b2 * s2[1] + (1 - b2) * g * g
    sv = v.sqrt()
    # d/dg [m / (sqrt(v) + eps)] <= (1 - b1) / (sqrt(v) + eps) + |m| sqrt(1 - b2) / (sqrt(v) + eps)^2
    lip = lr_t * ((1 - b1) / (sv + eps) + m.abs() * (1 - b2) ** 0.5 / (sv + eps) ** 2)
    # m = b1 m0 + (1 - b1) g may cancel: its rounding is relative to the two terms, not to m
    return w0 - lr_t * m / (sv + eps), lip, lr_t * (b1 * s2[0].abs() + (1 - b1) * g.abs()) / (sv + eps)


def _check_sparse_update(opt, what, before, after, ids, values, hyper):
    """after (weights, s1, s2) against the Keras rule applied to the float64 sum of each touched row's slices, from
    `before`; `hyper`: the device's hyper-parameter vector of this step.  A row's fp32 sum of k slices is within
    dg = (k - 1) 2^-24 sum |g| of the exact sum, which moves the update by at most lip * dg (lip from _rule, taken at g
    and at |g| - dg); the update itself rounds a handful of times at the size of its terms (|dw|, and for Adam the two
    terms of m): bound 2 (lip dg + 2^-24 |w| + 8 2^-24 terms).
    Untouched rows and their slots are bit-identical to before."""
    w0, s10, s20 = before
    w1, s11, s21 = after
    rows = w0.shape[0]
    ok = (ids >= 0) & (ids < rows)
    u, inv, cnt = torch.unique(ids[ok], return_inverse=True, return_counts=True)
    g = values[ok].double()
    gs = torch.zeros((len(u), g.shape[1]), dtype=torch.float64, device=g.device).index_add_(0, inv, g)
    ga = torch.zeros_like(gs).index_add_(0, inv, g.abs())
    dg = (cnt - 1).double().unsqueeze(1) * E * ga
    st1 = None if s10 is None else s10[u].double()
    st2 = (s10[u].double(), s20[u].double()) if opt == "adam" else None
    want, lip, terms = _rule(opt, w0[u].double(), st1, st2, gs, hyper)
    if opt == "adam":  # Adam's derivative grows as |g| shrinks: also take it at the smallest |g| within dg
        g_lo = gs.sign() * (gs.abs() - dg).clamp_min(0.0)
        lip = torch.maximum(lip, _rule(opt, w0[u].double(), st1, st2, g_lo, hyper)[1])
    bound = 2 * (lip * dg + E * want.abs() + 8 * E * terms)
    _within(w1[u], want, bound, f"{what}: touched rows")
    keep = torch.ones(rows, dtype=torch.bool, device=w0.device)
    keep[u] = False
    for name, a, b in (("weights", w1, w0), ("state1", s11, s10), ("state2", s21, s20)):
        if a is not None:
            assert torch.equal(a[keep], b[keep]), f"{what}: an untouched row of the {name} changed"
    return cnt


SPARSE_TABLES = [(500, w) for w in (2, 3, 4, 8)] + [(20000, w) for w in (2, 3, 4, 8)] + [(400000, w) for w in (3, 4, 8)]


@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("law", ["uniform", "zipf"])
@pytest.mark.parametrize("B", [BIG, RAGGED])
def test_sparse_rows_apply_at_scale(device, B, law, opt, mirror):
    """Tables of 500 (counting-sort path), 20 000 (vector-red path) and 400 000 rows (election path) in ONE call, ids at
    every width each table allows (~0.5 % outside the table), uniform or zipf (one hot row then takes thousands of
    folds), D = 64 with and without the operand mirror, two steps; the trainer's dense accumulators for the tables up to
    DENSE_PATH_MAX_ROWS.  Each step is checked from the state the device held before it (see _check_sparse_update),
    then the map is idle, the accumulators are zero and the mirror equals split_rows(weights) bit for bit."""
    D, lr = 64, 0.05
    assert SPARSE_TABLES[0][0] <= 1024 < SPARSE_TABLES[4][0] <= DENSE_PATH_MAX_ROWS < SPARSE_TABLES[-1][0]  # one per path
    assert -(-B // 1024) >= 2  # several counting-sort CTAs per small table
    eps = 1e-6 if opt == "adam" else 1e-7
    o = {"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt]
    hyper = torch.from_numpy(o.hyper()).to(device)
    rng = np.random.default_rng(B + len(law) + len(opt) + mirror)
    gen = torch.Generator(device=device).manual_seed(B + mirror)
    n = len(SPARSE_TABLES)
    W = [torch.randn((r, D), generator=gen, device=device) * 0.1 for r, _ in SPARSE_TABLES]
    s1 = [torch.full_like(w, o.initial_accumulator_value) if o.slots >= 1 else None for w in W]
    s2 = [torch.zeros_like(w) if o.slots >= 2 else None for w in W]
    rep = [ops.fill_i32(torch.empty(r, dtype=torch.int32, device=device), INT_MAX) for r, _ in SPARSE_TABLES]
    mir = [ops.split_rows(w) if mirror else None for w in W]
    dense = [torch.zeros_like(w) if r <= DENSE_PATH_MAX_ROWS else None for w, (r, _) in zip(W, SPARSE_TABLES)]
    hottest = 0
    for step in (1, 2):
        ids64 = []
        for r, w in SPARSE_TABLES:
            i = rng.integers(0, r, B) if law == "uniform" else np.minimum(rng.zipf(1.05, B) - 1, r - 1)
            at = rng.choice(B, B // 200, replace=False)
            i[at] = rng.integers(r, {2: 65536, 3: 1 << 24, 4: 1 << 31, 8: 1 << 40}[w], len(at))
            if w >= 4:
                i[at[: len(at) // 2]] = -1
            ids64.append(i)
        vals = [torch.randn((B, D), generator=gen, device=device) for _ in range(n)]
        before = [(w.clone(), None if a is None else a.clone(), None if b is None else b.clone()) for w, a, b in zip(W, s1, s2)]
        tabs = [dict(weights=W[t], indices=torch.from_numpy(pack_ids(ids64[t], SPARSE_TABLES[t][1])).to(device),
                     grad_rows=vals[t].clone(), rep_map=rep[t], state1=s1[t], state2=s2[t], mirror=mir[t], dense_grad=dense[t])
                for t in range(n)]
        ops.opt_tick(hyper)
        ops.sparse_rows_apply(opt, tabs, B, D, hyper)
        hy = hyper.cpu().numpy()
        for t, (r, w) in enumerate(SPARSE_TABLES):
            what = f"{opt} step {step}, {r} rows, {w}-byte {law} ids"
            cnt = _check_sparse_update(opt, what, before[t], (W[t], s1[t], s2[t]), torch.from_numpy(ids64[t]).to(device), vals[t], hy)
            hottest = max(hottest, int(cnt.max()))
            assert int((rep[t] != INT_MAX).sum()) == 0, f"{what}: the representative map is not idle"
            assert dense[t] is None or float(dense[t].abs().max()) == 0.0, f"{what}: the dense accumulator was not cleared"
            if mir[t] is not None:
                assert torch.equal(mir[t], ops.split_rows(W[t])), f"{what}: the mirror is out of step"
    if law == "zipf":
        assert hottest > 1000, hottest  # premise: one row folds thousands of duplicates


# ---------------------------------------------------------------------------------------------------------------
# 4. mm_inbatch_softmax_ce_backward at the two-tower benchmark shape
# ---------------------------------------------------------------------------------------------------------------
def _ce_ref_chunked(q, pos, neg, pid, nid, T, c, chunk=2048):
    """float64 loss and gradients of sum_b c (lse_b - s_b0), s = [q.pos | masked(q neg^T)] / T, in chunks of query rows
    (the rule of test_gpu_train_twotower._ce_ref: a down-scored logit is a constant, its gradient zero)."""
    qd, pd, nd = q.double(), pos.double(), neg.double()
    B = qd.shape[0]
    gq, gp, gn = torch.zeros_like(qd), torch.zeros_like(qd), torch.zeros_like(nd)
    loss = 0.0
    mf = float(np.float32(O.MIN_FLOAT))
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        qc = qd[s:e]
        m = pid[s:e].view(-1, 1) == nid.view(1, -1)
        sn = torch.where(m, torch.full((), mf, dtype=torch.float64, device=qd.device), qc @ nd.T)
        z = torch.cat([(qc * pd[s:e]).sum(-1, keepdim=True), sn], dim=1) / T
        lse = torch.logsumexp(z, 1, keepdim=True)
        loss += float((c * (lse[:, 0] - z[:, 0])).sum())
        p = c * torch.exp(z - lse)
        p[:, 0] -= c
        pn = p[:, 1:].masked_fill(m, 0.0) / T
        gq[s:e] = p[:, :1] / T * pd[s:e] + pn @ nd
        gp[s:e] = p[:, :1] / T * qc
        gn += pn.T @ qc
    return loss, gq, gp, gn


@pytest.mark.parametrize("B,N,D,alias", [(16384, 16384, 128, True), (16384 - 5, 16384 + 77, 64, False)])
def test_ce_backward_at_scale(device, B, N, D, alias):
    """Down-scoring on with duplicated item ids, T = 0.05: dq, dpos, dneg (dpos aliasing dneg writes their sum) and the
    loss against the chunked float64 reference, with the tolerance rule of the small-batch test (allclose, floor = a few
    ulps of one term c p x / T)."""
    T = 0.05
    tiles_n, tiles_b = -(-N // 128), -(-B // 128)
    assert min(tiles_n, tiles_b) > 2 * 4, "premise: every CTA refills each of its <= 4 ring stages at least once"
    q, pos, neg, pid, nid, _ = _ce_case(device, B, N, D, True, False, T, seed=2 if alias else 3)
    assert (neg is pos) == alias and int(torch.unique(pid).numel()) < B // 2
    stats = ops.inbatch_softmax_ce(q, pos, neg, pos_ids=pid, neg_ids=nid, downscore=True, false_neg_score=O.MIN_FLOAT, temperature=T)
    qbuf, nbuf = _nan((B + GUARD, D), device), _nan((N + GUARD, D), device)
    pbuf = nbuf if alias else _nan((B + GUARD, D), device)
    loss = torch.zeros(1, device=device)
    c = torch.full((1,), 1.0 / B, device=device)
    ops.inbatch_softmax_ce_backward(ops.split_rows(q), ops.split_rows(neg), D, stats, q, pos, c, qbuf[:B], pbuf[:B], nbuf[:N],
                                    loss=loss, pos_ids=pid, neg_ids=nid, downscore=True, false_neg_score=O.MIN_FLOAT, temperature=T)
    want_loss, gq, gp, gn = _ce_ref_chunked(q, pos, neg, pid, nid, T, 1.0 / B)
    assert abs(float(loss.item()) - want_loss) <= 1e-4 * max(1.0, abs(want_loss)), (float(loss.item()), want_loss)
    floor = 1e-6 / B / T * max(float(t.abs().max()) for t in (q, pos, neg))
    allclose(qbuf[:B], gq, what="dq", floor=floor)
    if alias:
        allclose(nbuf[:N], gp + gn, what="dpos + dneg (aliased)", floor=floor)
    else:
        allclose(pbuf[:B], gp, what="dpos", floor=floor)
        allclose(nbuf[:N], gn, what="dneg", floor=floor)
        _untouched(pbuf, B, D, "dpos")
    _untouched(qbuf, B, D, "dq")
    _untouched(nbuf, N, D, "dneg")


# ---------------------------------------------------------------------------------------------------------------
# 5. one DLRM training step as bench.py --workload dlrm-train runs it
# ---------------------------------------------------------------------------------------------------------------
CAP = 400000


def _bench_model(device, seed):
    mm.set_seed(seed)
    schema = datasets.criteo_schema({k: min(v, CAP - 1) for k, v in datasets.CRITEO_MAX.items()})
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]))
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    return schema, model


def _variables(tr):
    out = [t.table for t in tr.tables]
    a = tr.arena
    for i in range(len(a.layers)):
        out += [v for v in (a.view(a.w, i, "kernel"), a.view(a.w, i, "bias")) if v is not None]
    return out


def _reference_step(tr, inputs, y, B, chunk=8192, rows_of=None):
    """float64 autograd on the device of the trainer's forward (bottom MLP, lookup, pairwise dots, top MLP, head, mean BCE)
    over the looked-up rows, in sample chunks.  Returns the loss, the dense gradients by variable name, the slices per
    table, and per sample whether a relu unit is on in one implementation and off in the other.  rows_of(t, s, e): the
    float64 rows of table t for samples [s, e) (default: the table's rows at the trainer's ids; a multi-hot feature passes
    its pooled rows)."""
    layers = tr.bottom + tr.top + [tr.head]
    P = [(l.kernel.double().requires_grad_(True), None if l.bias is None else l.bias.double().requires_grad_(True)) for l in layers]
    cont = tr.body.continuous(inputs)
    x0 = torch.cat([cont[k].reshape(B, -1) for k in sorted(cont)], dim=1).double()
    ids = [ops.widen_index(i).long() for i in tr._idx]
    saved = [h[:B] for h in tr.h] + [t[:B] for t in tr.t]  # the trainer's activations
    nb = len(tr.bottom)
    order = [tr.slots[f] for f in tr.feats]
    bslot = tr.slots["bottom_block"]
    F = len(tr.slots)
    triu = torch.triu(torch.ones(F, F, dtype=torch.bool, device=x0.device), diagonal=1)
    loss, slices, flips = 0.0, [[] for _ in ids], []
    yd = y.reshape(-1).double()
    terms = {}  # |X|^T |dZ| and sum |dZ| of every dense gradient: the scale of the fp32 sums that make it

    def dense(h, li, flips_of_chunk, s, e):
        (Wk, bk), l = P[li], layers[li]
        z = h @ Wk + (bk if bk is not None else 0.0)
        z.retain_grad()
        pre.append((li, h.detach(), z))
        if l.activation != "relu":
            return z
        with torch.no_grad():  # on/off differently: only ever a unit within rounding of zero
            flip = (saved[li][s:e] > 0) != (z > 0)
            band = (h.abs() @ Wk.abs() + (bk.abs() if bk is not None else 0.0)) * 2.0 ** -10
            assert bool((z.abs()[flip] <= band[flip]).all()), f"layer {l.name}: a unit far from zero is on/off differently"
        flips_of_chunk.append(flip.any(1))
        return torch.relu(z)

    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        flip, pre = [], []
        h = x0[s:e]
        for li in range(nb):
            h = dense(h, li, flip, s, e)
        rows = [(tr.tables[t].table[ids[t][s:e]].double() if rows_of is None else rows_of(t, s, e)).requires_grad_(True)
                for t in range(len(ids))]
        seq = [None] * F
        for t, sl in enumerate(order):
            seq[sl] = rows[t]
        seq[bslot] = h
        st = torch.stack(seq, dim=1)
        z = torch.bmm(st, st.transpose(1, 2))
        h = torch.cat([h, z[:, triu]], dim=1)
        for li in range(nb, nb + len(tr.top)):
            h = dense(h, li, flip, s, e)
        logit = dense(h, len(layers) - 1, flip, s, e).reshape(-1)
        yy = yd[s:e]
        per = torch.clamp(logit, min=0) - logit * yy + torch.log1p(torch.exp(-logit.abs()))
        part = per.sum() / B
        part.backward()
        loss += float(part)
        for t, r in enumerate(rows):
            slices[t].append(r.grad)
        flips.append(torch.stack(flip).any(0))
        for li, hin, z in pre:
            name = layers[li].name
            terms[f"{name}/kernel"] = terms.get(f"{name}/kernel", 0.0) + hin.abs().t() @ z.grad.abs()
            terms[f"{name}/bias"] = terms.get(f"{name}/bias", 0.0) + z.grad.abs().sum(0)
    grads = {}
    for l, (Wk, bk) in zip(layers, P):
        grads[f"{l.name}/kernel"] = Wk.grad
        if bk is not None:
            grads[f"{l.name}/bias"] = bk.grad
    return loss, grads, {k: terms[k] for k in grads}, [torch.cat(s) for s in slices], torch.cat(flips)


def test_dlrm_train_step_as_the_benchmark_runs_it(device):
    """Criteo schema capped at 400 000 rows (eight tables on the election path with 3-byte ids), embedding_dim 64 with
    the operand mirrors, bottom [128, 64], top [128, 64, 32], Adagrad, B = 65 536, packed ids through HostBatch into one
    CUDA graph.
    (a) two graph replays on packed ids against two eager steps of a twin model on int64 ids: every variable within
        1e-5 of its scale (same kernels; only the order of the fp32 atomics differs), as at B = 512.
    (b) forward_backward against float64 autograd: loss at 1e-5; each dense gradient's Frobenius error under 1e-4 of
        the Frobenius norm of its terms |X|^T |dZ| (sum |dZ| for a bias): at B = 65 536 the first layers' gradients
        are sums of terms of both signs that cancel to a few tenths of a percent of the terms, so their error is set by
        the terms; per element the wgrad arithmetic alone is within 2 (U + depth 2^-24) ~ 7e-5 of them (observed on an
        H100: <= 3.2e-5, growing down the backward chain).  Slices per element within
        1e-3 |ref| + 3e-4 max |ref slices of that sample| (observed: < 7 % of that), leaving out the samples with a
        relu unit on in one implementation and off in the other (its pre-activation within rounding of zero; each such
        unit is asserted to be within 2^-10 of its terms); they must be under 1 % of the batch (observed: 58).
    (c) the Adagrad update of the touched rows against the float64 rule on the summed slices (_check_sparse_update);
        untouched rows unchanged; every mirror equals split_rows of its table."""
    B = BIG
    schema, ma = _bench_model(device, 21)
    _, mb = _bench_model(device, 21)
    widths = ma.id_bytes()
    assert sorted(f for f, w in widths.items() if w == 3) == sorted(
        f for f, v in datasets.CRITEO_MAX.items() if v + 1 > DENSE_PATH_MAX_ROWS) and len([w for w in widths.values() if w == 3]) == 8
    label = schema.select_by_tag(mm.Tags.TARGET).column_names[0]
    hosts = [datasets.generate_batch(schema, B, seed=4321 + i, index_law="uniform", index_dtype=np.int32) for i in range(3)]
    names = ma.input_columns() + [label]
    hbs = [HostBatch.like(h, names, id_bytes=widths) for h in hosts]
    packed = [hb.buffer.to(device) for hb in hbs]
    static = packed[0].clone()
    views = {k: _view(static, hbs[0].offsets[k], shp, dt) for k, (shp, dt) in hbs[0].spec.items()}
    inputs = {k: v for k, v in views.items() if k != label}
    ta, tb = ma.trainer(B), mb.trainer(B)
    assert ta.operand_rows and all(t._mirror is not None for t in ta.tables)
    ta.capture(inputs, views[label], clone=False)
    for i in (0, 1):
        static.copy_(packed[i])
        la = float(ta.replay().item())
        x = {k: torch.from_numpy(np.asarray(hosts[i][k]).astype(np.int64) if np.asarray(hosts[i][k]).dtype.kind in "iu"
                                 else np.asarray(hosts[i][k])).to(device) for k in ma.input_columns()}
        lb = float(tb.step(x, torch.from_numpy(np.asarray(hosts[i][label])).to(device)).item())
        np.testing.assert_allclose(la, lb, rtol=1e-6)
    for i, (va, vb) in enumerate(zip(_variables(ta), _variables(tb))):
        err = float((va - vb).abs().max()) / max(float(vb.abs().max()), 1e-30)
        assert err < 1e-5, f"variable {i}: graph replay on packed ids vs eager on int64 ids differ by {err:.3e} of the scale"
    del tb, mb, x
    torch.cuda.empty_cache()

    # (b)
    static.copy_(packed[2])
    ta.forward_backward(inputs, views[label])
    want_loss, want, terms, ref_slices, flipped = _reference_step(ta, inputs, views[label], B)
    np.testing.assert_allclose(float(ta.loss.item()), want_loss, rtol=1e-5)
    got = ta.gradients()
    assert sorted(got) == sorted(want)
    for k in want:
        fro = float((got[k].double() - want[k]).norm() / terms[k].norm())
        assert fro < 1e-4, f"{k}: Frobenius error {fro:.3e} of the terms' scale"
    n_flip = int(flipped.sum())
    assert n_flip < B // 100, f"{n_flip} samples have a relu unit on/off differently"
    keep = ~flipped
    scale = torch.stack([s.abs().amax(1) for s in ref_slices]).amax(0)[keep].unsqueeze(1)
    for t, f in enumerate(ta.feats):
        r = ref_slices[t][keep]
        _within(ta._slices[t][keep], r, 1e-3 * r.abs() + 3e-4 * scale, f"slices of {f}")

    # (c)
    before = [(t.table.clone(), a.clone(), None) for t, a in zip(ta.tables, ta.tstate1)]
    slices = [s.clone() for s in ta._slices]  # the update folds duplicates into the slices in place
    ids = [ops.widen_index(i).long() for i in ta._idx]
    ta.apply_gradients()
    hy = ta.hyper.cpu().numpy()
    for t, f in enumerate(ta.feats):
        _check_sparse_update("adagrad", f"Adagrad step, table of {f}", before[t], (ta.tables[t].table, ta.tstate1[t], None),
                             ids[t], slices[t], hy)
        assert torch.equal(ta.tables[t]._mirror, ops.split_rows(ta.tables[t].table)), f"mirror of {f} out of step"
