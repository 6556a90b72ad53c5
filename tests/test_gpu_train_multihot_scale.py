"""Multi-hot DLRM training at the sizes tools/train_multihot_bench.py trains with: B = 65 536, D = 64, the Criteo tables,
15 fixed-length bags of MLPerf DLRM-DCNv2's sizes (L from 2 to 100, 203 bag ids per sample), Adagrad, one CUDA graph.
There the pooling kernels take a second grid-stride lap, mm_bag_grad_rows expands 13.3 M rows per step (6.55 M for one
table), and mm_sparse_rows_apply gets B = nnz: 320 counting-sort CTAs for a 72-row table, an election map holding sample
indices in the millions.  Every large-B test asserts that premise from the launcher's formula and the SM count.

Pooling and expansion are bit-exact: gather_seq / gather_bag add rows left to right with __fadd_rn and divide with
__fdiv_rn, bag_grad_rows makes each row with one IEEE division, the library is built without fast-math, so an fp32
reference that adds in the same order (and divides by a device tensor: torch multiplies by the reciprocal of a CPU
scalar) is bit-identical.  The update and the training step are checked against float64 references on the device, with
the tolerances of tests/test_gpu_train_scale.py.  Output buffers carry NaN guard rows (and columns); they must stay NaN."""
import dataclasses

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200.train import DENSE_PATH_MAX_ROWS
from tests.test_gpu_train_scale import CAP, _check_sparse_update, _reference_step, _sms, _untouched, _variables, _within

pytestmark = pytest.mark.gpu
BIG = 65536
RAGGED = BIG + 37
GUARD = 8
INT_MAX = 2 ** 31 - 1
D = 64
# MLPerf DLRM-DCNv2's bag size of C1..C26, as tools/train_multihot_bench.py feeds them (size 1 stays a one-hot column)
BAG_SIZES = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]
BAG = {f"C{i}": L for i, L in enumerate(BAG_SIZES, start=1) if L > 1}
SEQ_FEATURE = {}  # bag size -> the first feature of that size
for _f, _L in BAG.items():
    SEQ_FEATURE.setdefault(_L, _f)


def _rows(f, cap=None):
    r = datasets.CRITEO_MAX[f] + 1
    return r if cap is None else min(r, cap)


def _table(rows, seed, device):
    return ops.init_uniform_hash(torch.empty((rows, D), device=device), seed, -1.0, 1.0)


def _nan(shape, device):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=device)


def _pool_laps(B, sms):
    """Grid-stride laps of gather_seq_kernel / gather_bag_kernel: one warp per sample, 8 warps per block, the grid capped
    at 32 blocks per SM (mm_gather_seq / mm_gather_bag)."""
    blocks = min(-(-B * 32 // 256), 32 * sms)
    return -(-B // (blocks * 8))


def _expand_laps(tasks, sms):
    """Grid-stride laps of bag_grad_rows_kernel: one warp per task, 8 warps per block, at most 64 blocks per SM."""
    blocks = min(-(-tasks // 8), 64 * sms)
    return -(-tasks // (blocks * 8))


def _seq_ref(table, ids, comb):
    """fp32 pooling of (B, L) ids in the kernel's order: from +0.0, add position l's row (a zero where the id is outside
    the table) for l = 0 .. L-1, then (mean) one division by L."""
    rows = table.shape[0]
    acc = torch.zeros((ids.shape[0], table.shape[1]), device=table.device)
    for l in range(ids.shape[1]):
        i = ids[:, l]
        ok = ((i >= 0) & (i < rows)).unsqueeze(1)
        acc = acc + table[i.clamp(0, rows - 1)] * ok
    return acc / torch.full_like(acc, float(ids.shape[1])) if comb == "mean" else acc


def _bag_ref(table, values, offsets):
    """fp32 sum of each ragged bag in the kernel's order (position k added only where its id is in the table: adding a
    zero would turn -0.0 into +0.0) and the number of ids added.  Position k is visited only for the bags longer than k,
    taken as a prefix of the bags sorted by length."""
    rows = table.shape[0]
    lens = offsets[1:] - offsets[:-1]
    order = torch.argsort(lens, descending=True)
    start, lens_s = offsets[:-1][order], lens[order]
    B = lens.numel()
    longer = B - torch.cumsum(torch.bincount(lens, minlength=int(lens.max()) + 1), 0).cpu().numpy()  # bags longer than k
    acc = torch.zeros((B, table.shape[1]), device=table.device)
    cnt = torch.zeros(B, dtype=torch.int64, device=table.device)
    for k in range(int(lens_s[0])):
        n = int(longer[k])
        i = values[start[:n] + k]
        use = (i >= 0) & (i < rows)
        acc[:n] = torch.where(use.unsqueeze(1), acc[:n] + table[i.clamp(0, rows - 1)], acc[:n])
        cnt[:n] += use
    out_acc, out_cnt = torch.empty_like(acc), torch.empty_like(cnt)
    out_acc[order], out_cnt[order] = acc, cnt
    return out_acc, out_cnt


def _bag_combine(acc, cnt, comb):
    """The kernel's last step: mean / sqrtn divide a non-empty bag's sum once (by cnt or sqrtf(cnt))."""
    if comb == "sum":
        return acc
    den = cnt.float() if comb == "mean" else torch.sqrt(cnt.float())
    return torch.where((cnt > 0).unsqueeze(1), acc / den.clamp_min(1.0).unsqueeze(1), acc)


def _den(cnt, comb):
    """bag_grad_rows' divisor of a ragged bag (None: sum, the rows are copies)."""
    return None if comb == "sum" else cnt.float() if comb == "mean" else torch.sqrt(cnt.float())


def _expand_ref(g, seg, ok, den):
    """fp32 on the device: row i = g[seg[i]] / den[seg[i]] (one IEEE division; den None: a copy) where ok[i], else +0."""
    x = g[seg]
    if den is not None:
        x = x / den[seg].unsqueeze(1)
    return torch.where(ok.unsqueeze(1), x, torch.zeros((), device=g.device))


def _check_update_by_rows(opt, what, before, after, ids, values, hyper, part=1 << 20):
    """_check_sparse_update over ranges of `part` rows: rows are updated independently, and a range bounds the float64
    reference's memory for a table of millions of rows.  Returns the number of slices of every touched row."""
    cnts = []
    for r0 in range(0, before[0].shape[0], part):
        r1 = r0 + part
        sel = (ids >= r0) & (ids < r1)

        def cut(state):
            return tuple(None if a is None else a[r0:r1] for a in state)

        cnts.append(_check_sparse_update(opt, f"{what}, rows from {r0}", cut(before), cut(after), ids[sel] - r0, values[sel], hyper))
    return torch.cat(cnts)


def _plant_oob(rng, ids, rows, frac):
    """Replace ~frac of the ids by ids outside [0, rows), half negative, half >= rows (all within int32)."""
    at = rng.random(ids.shape) < frac
    n = int(at.sum())
    bad = np.where(rng.random(n) < 0.5, -1 - rng.integers(0, 1000, n), rows + rng.integers(0, 1 << 20, n))
    ids[at] = bad
    return n


# ---------------------------------------------------------------------------------------------------------------
# 1. pooling: mm_gather_seq and mm_gather_bag, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", sorted(SEQ_FEATURE))
@pytest.mark.parametrize("B", [BIG, RAGGED])
def test_gather_seq_at_scale(device, B, L):
    """(B, L) ids of the bench's feature of bag size L on its table (10 M rows for C1, C10, C20, C22), ~0.5 % outside
    the table, int32 and int64, sum and mean, written at out_col 4 of a NaN-filled buffer: bit-equal to _seq_ref, the
    out-of-range counter equal to the planted count, the guard rows and columns still NaN."""
    assert _pool_laps(B, _sms(device)) == 2, "premise: the pooling grid takes a second lap"
    f = SEQ_FEATURE[L]
    rows = _rows(f)
    table = _table(rows, 100 + L, device)
    rng = np.random.default_rng(B + L)
    ids64 = rng.integers(0, rows, (B, L))
    n_oob = _plant_oob(rng, ids64, rows, 0.005)
    assert n_oob > 0
    ids = torch.from_numpy(ids64).to(device)
    buf = _nan((B + GUARD, D + 8), device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    for comb in ("sum", "mean"):
        want = _seq_ref(table, ids, comb)
        for dt in (torch.int32, torch.int64):
            buf.fill_(float("nan"))
            oob.zero_()
            ops.gather_seq(table, ids.to(dt), comb, buf[:B], out_col=4, oob=oob)
            assert torch.equal(buf[:B, 4:4 + D], want), f"{f} (L = {L}), {comb}, {dt}: pooled rows differ from the fp32 reference"
            assert bool(torch.isnan(buf[:, :4]).all()) and bool(torch.isnan(buf[:, 4 + D:]).all()), f"{f}: a column outside out_col was written"
            _untouched(buf, B, D + 8, f"{f} pooled")
            assert int(oob.item()) == n_oob, f"{f}: {int(oob.item())} out-of-range ids counted, {n_oob} planted"


@pytest.mark.parametrize("id_dt,off_dt", [(torch.int32, torch.int32), (torch.int64, torch.int32), (torch.int32, torch.int64),
                                          (torch.int64, torch.int64)])
@pytest.mark.parametrize("f", ["C15", "C21"])
def test_gather_bag_at_scale(device, f, id_dt, off_dt):
    """Ragged bags of the feature's table at B = 65 573: lengths 0 .. 2L (~2 % empty, one bag of 5 000 ids), ~3 % ids
    negative (pruned, not counted) and ~0.5 % >= rows (counted, not summed); mean, sum and sqrtn bit-equal to _bag_ref
    and _bag_combine, out_col 4 of a NaN-filled buffer."""
    B = RAGGED
    assert _pool_laps(B, _sms(device)) == 2, "premise: the pooling grid takes a second lap"
    L, rows = BAG[f], _rows(f)
    table = _table(rows, 200 + L, device)
    rng = np.random.default_rng(L + 7 * (id_dt == torch.int64) + 13 * (off_dt == torch.int64))
    lens = rng.integers(0, 2 * L + 1, B)
    lens[rng.random(B) < 0.02] = 0
    lens[B // 3] = 5000
    offsets = np.concatenate([[0], np.cumsum(lens)])
    values = rng.integers(0, rows, int(offsets[-1]))
    r = rng.random(values.size)
    values[r < 0.03] = -1 - rng.integers(0, 1000, int((r < 0.03).sum()))
    hi = (r >= 0.03) & (r < 0.035)
    values[hi] = rows + rng.integers(0, 1 << 20, int(hi.sum()))
    n_oob = int(hi.sum())
    vals = torch.from_numpy(values).to(device)
    offs = torch.from_numpy(offsets).to(device)
    acc, cnt = _bag_ref(table, vals, offs)
    assert int((cnt == 0).sum()) > B // 100
    buf = _nan((B + GUARD, D + 8), device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    for comb in ("mean", "sum", "sqrtn"):
        buf.fill_(float("nan"))
        oob.zero_()
        ops.gather_bag(table, vals.to(id_dt), offs.to(off_dt), comb, buf[:B], out_col=4, oob=oob)
        assert torch.equal(buf[:B, 4:4 + D], _bag_combine(acc, cnt, comb)), f"{f}, {comb}: pooled rows differ from the fp32 reference"
        assert bool(torch.isnan(buf[:, :4]).all()) and bool(torch.isnan(buf[:, 4 + D:]).all()), f"{f}: a column outside out_col was written"
        _untouched(buf, B, D + 8, f"{f} pooled")
        assert int(oob.item()) == n_oob, f"{f}: {int(oob.item())} out-of-range ids counted, {n_oob} planted"


# ---------------------------------------------------------------------------------------------------------------
# 2. expansion: mm_bag_grad_rows at nnz in the millions, bit for bit
# ---------------------------------------------------------------------------------------------------------------
EXPAND_B = 135205  # one warp per bag on at most 64 x 8 warps per SM: 3 laps on 132 SMs (the bench's 65 536 takes one)


@pytest.mark.parametrize("B,L,Dx,id_dt", [(EXPAND_B, 100, 16, torch.int64), (EXPAND_B, 27, 64, torch.int32),
                                          (EXPAND_B, 3, 128, torch.int64), (BIG, 100, 64, torch.int32)])
def test_bag_grad_rows_fixed_length_at_scale(device, B, L, Dx, id_dt):
    """Fixed-length bags, ~0.5 % of the ids outside the table, g read at a padded row stride: every row is g[bag] (sum)
    or g[bag] / L (mean) bit for bit, zero with out_ids -1 where the id is outside the table; guard rows stay NaN and
    guard ids untouched.  The last case is the bench's C21 (1.7 GB of rows), whose 65 536 bags take one lap."""
    laps = _expand_laps(B, _sms(device))
    assert laps == (1 if B == BIG else 3), f"premise: B = {B} gives {laps} lap(s)"
    rows = 400000
    rng = np.random.default_rng(B + L + Dx)
    ids64 = rng.integers(0, rows, (B, L))
    _plant_oob(rng, ids64, rows, 0.005)
    ids = torch.from_numpy(ids64).to(device=device, dtype=id_dt)
    gen = torch.Generator(device=device).manual_seed(L + Dx)
    g = torch.randn((B, Dx + 4), generator=gen, device=device)[:, :Dx]
    nnz = B * L
    buf = _nan((nnz + GUARD, Dx), device)
    oi = torch.full((nnz + GUARD,), 77, dtype=id_dt, device=device)
    for comb in ("sum", "mean"):
        buf.fill_(float("nan"))
        ops.bag_grad_rows(g, ids, None, rows, comb, buf[:nnz], out_ids=oi[:nnz])
        den = None if comb == "sum" else torch.full((B,), float(L), device=device)
        for s in range(0, B, 16384):  # in bag chunks: the full reference of the bench case would be another 1.7 GB
            e = min(B, s + 16384)
            i = ids[s:e].reshape(-1).long()
            ok = (i >= 0) & (i < rows)
            seg = torch.arange(s, e, device=device).repeat_interleave(L)
            assert torch.equal(buf[s * L:e * L], _expand_ref(g, seg, ok, den)), f"L = {L}, D = {Dx}, {comb}: rows of bags [{s}, {e}) differ"
            assert torch.equal(oi[s * L:e * L].long(), torch.where(ok, i, -1)), f"L = {L}, D = {Dx}: out_ids of bags [{s}, {e}) differ"
        _untouched(buf, nnz, Dx, f"expanded rows, L = {L}, D = {Dx}, {comb}")
        assert bool((oi[nnz:] == 77).all()), "an id past nnz was written"


@pytest.mark.parametrize("id_dt,off_dt", [(torch.int32, torch.int64), (torch.int64, torch.int32)])
def test_bag_grad_rows_ragged_at_scale(device, id_dt, off_dt):
    """Ragged bags at B = 135 205 (B + 2 tasks, 3 laps) with offsets[0] > 0 and offsets[B] < nnz, lengths 0 .. 18, ~3 %
    ids negative and ~0.5 % >= rows: bag rows are g[bag] / cnt (mean), g[bag] / sqrtf(cnt) (sqrtn) or g[bag] (sum) bit
    for bit where the id is in the table; ids outside it and the uncovered head and tail give zero rows and out_ids -1
    (their ids are in the table)."""
    B, rows, head, tail = EXPAND_B, 400000, 1000, 777
    assert _expand_laps(B + 2, _sms(device)) == 3, "premise: the expansion grid takes three laps"
    rng = np.random.default_rng(3 + (id_dt == torch.int64))
    lens = rng.integers(0, 19, B)
    offsets = head + np.concatenate([[0], np.cumsum(lens)])
    nnz = int(offsets[-1]) + tail
    values = rng.integers(0, rows, nnz)
    r = rng.random(nnz)
    r[:head] = r[nnz - tail:] = 1.0  # the uncovered positions hold ids in the table
    values[r < 0.03] = -1 - rng.integers(0, 1000, int((r < 0.03).sum()))
    hi = (r >= 0.03) & (r < 0.035)
    values[hi] = rows + rng.integers(0, 1 << 20, int(hi.sum()))
    ids = torch.from_numpy(values).to(device=device, dtype=id_dt)
    offs = torch.from_numpy(offsets).to(device=device, dtype=off_dt)
    gen = torch.Generator(device=device).manual_seed(5)
    g = torch.randn((B, D), generator=gen, device=device)
    i = ids.long()
    seg = torch.zeros(nnz, dtype=torch.int64, device=device)
    covered = torch.zeros(nnz, dtype=torch.bool, device=device)
    covered[head:nnz - tail] = True
    seg[head:nnz - tail] = torch.arange(B, device=device).repeat_interleave(torch.from_numpy(lens).to(device))
    ok = covered & (i >= 0) & (i < rows)
    cnt = torch.zeros(B, dtype=torch.int64, device=device).index_add_(0, seg[covered], ok[covered].long())
    buf = _nan((nnz + GUARD, D), device)
    oi = torch.full((nnz + GUARD,), 77, dtype=id_dt, device=device)
    for comb in ("mean", "sum", "sqrtn"):
        buf.fill_(float("nan"))
        ops.bag_grad_rows(g, ids, offs, rows, comb, buf[:nnz], out_ids=oi[:nnz])
        assert torch.equal(buf[:nnz], _expand_ref(g, seg, ok, _den(cnt, comb))), f"{comb}: expanded rows differ"
        assert torch.equal(oi[:nnz].long(), torch.where(ok, i, -1)), f"{comb}: out_ids differ"
        _untouched(buf, nnz, D, f"expanded rows, {comb}")
        assert bool((oi[nnz:] == 77).all()), "an id past nnz was written"


# ---------------------------------------------------------------------------------------------------------------
# 3. the update: mm_sparse_rows_apply with B = nnz
# ---------------------------------------------------------------------------------------------------------------
APPLY_TABLES = [("C16", 72), ("C15", 9780), ("C21", CAP), ("C21", _rows("C21"))]  # counting sort, vector reds, election x2
ZIPF = 1.5  # the hottest row takes 1 / zeta(1.5) = 38 % of the ids: > 100 000 folds on every table


def _apply_ids(rng, law, rows, L, g, device):
    """(flat ids, expanded rows) of one bag table as the trainer hands them to the update: (65 536, L) ids expanded by
    bag_grad_rows (sum), or (law "marked") a ragged batch (lengths 0 .. 2L, ~3 % ids -1) whose ids are bag_grad_rows'
    out_ids."""
    if law == "marked":
        lens = rng.integers(0, 2 * L + 1, BIG)
        offs = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).to(device)
        vals = rng.integers(0, rows, int(lens.sum()))
        vals[rng.random(vals.size) < 0.03] = -1
        vals = torch.from_numpy(vals).to(device=device, dtype=torch.int32)
        out = torch.empty((vals.numel(), D), device=device)
        ids = torch.empty_like(vals)
        ops.bag_grad_rows(g, vals, offs, rows, "sum", out, out_ids=ids)
        return ids, out
    ids = rng.integers(0, rows, (BIG, L)) if law == "uniform" else np.minimum(rng.zipf(ZIPF, (BIG, L)) - 1, rows - 1)
    ids = torch.from_numpy(ids).to(device=device, dtype=torch.int32)
    out = torch.empty((ids.numel(), D), device=device)
    ops.bag_grad_rows(g, ids, None, rows, "sum", out)
    return ids.reshape(-1), out


@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("law", ["uniform", "zipf", "marked"])
@pytest.mark.parametrize("f,rows", APPLY_TABLES)
def test_sparse_rows_apply_bag_table_at_scale(device, f, rows, law, opt, mirror):
    """One call per table with B = nnz = 65 536 L, as apply_gradients makes it for a bag: flat int32 ids, the expanded
    rows, the dense accumulator for tables up to DENSE_PATH_MAX_ROWS; D = 64 with and without the mirror, two steps,
    each checked by _check_sparse_update from the state before it; then the map is idle, the accumulator is zero and the
    mirror equals split_rows(weights)."""
    L = BAG[f]
    nnz = BIG * L
    if rows <= 1024:
        assert -(-nnz // 1024) == 320, "premise: 320 counting-sort CTAs"
    elif rows <= DENSE_PATH_MAX_ROWS:
        assert nnz > 4 * rows, "premise: the vector-red path folds several slices per row"
    elif rows == CAP:
        assert nnz > 16 * rows, "premise: the election path folds ~16 slices per row"
    else:
        assert nnz > rows > DENSE_PATH_MAX_ROWS, "premise: the election map holds sample indices in the millions"
    lr = 0.05
    eps = 1e-6 if opt == "adam" else 1e-7
    o = {"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt]
    hyper = torch.from_numpy(o.hyper()).to(device)
    rng = np.random.default_rng(rows + len(law) + len(opt) + mirror)
    gen = torch.Generator(device=device).manual_seed(rows + mirror)
    W = torch.randn((rows, D), generator=gen, device=device) * 0.1
    s1 = torch.full_like(W, o.initial_accumulator_value) if o.slots >= 1 else None
    s2 = torch.zeros_like(W) if o.slots >= 2 else None
    rep = ops.fill_i32(torch.empty(rows, dtype=torch.int32, device=device), INT_MAX)
    mir = ops.split_rows(W) if mirror else None
    dense = torch.zeros_like(W) if rows <= DENSE_PATH_MAX_ROWS else None
    hottest = 0
    for step in (1, 2):
        g = torch.randn((BIG, D), generator=gen, device=device)
        ids, vals = _apply_ids(rng, law, rows, L, g, device)
        del g
        before = (W.clone(), None if s1 is None else s1.clone(), None if s2 is None else s2.clone())
        want_vals = vals.clone()  # the update folds duplicates into the rows in place
        ops.opt_tick(hyper)
        ops.sparse_rows_apply(opt, [dict(weights=W, indices=ids, grad_rows=vals, rep_map=rep, state1=s1, state2=s2, mirror=mir,
                                         dense_grad=dense)], vals.shape[0], D, hyper)
        what = f"{opt} step {step}, {f} ({rows} rows), {law} ids"
        cnt = _check_update_by_rows(opt, what, before, (W, s1, s2), ids.long(), want_vals, hyper.cpu().numpy())
        hottest = max(hottest, int(cnt.max()))
        assert int((rep != INT_MAX).sum()) == 0, f"{what}: the representative map is not idle"
        assert dense is None or float(dense.abs().max()) == 0.0, f"{what}: the dense accumulator was not cleared"
        if mir is not None:
            assert torch.equal(mir, ops.split_rows(W)), f"{what}: the mirror is out of step"
        del before, want_vals, vals, ids
    if law == "zipf":
        assert hottest > 100000, f"premise: the hottest row folds {hottest} slices"


# ---------------------------------------------------------------------------------------------------------------
# 4. one fixed-length multi-hot step as tools/train_multihot_bench.py runs it;  5. ragged features at scale
# ---------------------------------------------------------------------------------------------------------------
def _multihot_model(device, seed, ragged=None):
    """Criteo schema capped at CAP rows, D = 64 (with the operand mirrors), bottom [128, 64], top [128, 64, 32],
    Adagrad(0.01); bags pooled with `sum`, the features of `ragged` ({feature: combiner}) declared ragged lists."""
    ragged = ragged or {}
    mm.set_seed(seed)
    capped = datasets.criteo_schema({k: min(v, CAP - 1) for k, v in datasets.CRITEO_MAX.items()})
    schema = mm.Schema([dataclasses.replace(c, is_list=True, is_ragged=True) if c.name in ragged else c for c in capped])
    comb = {f: ragged.get(f, "sum") for f in datasets.CRITEO_MAX}
    emb = mm.Embeddings(schema.select_by_tag(mm.Tags.CATEGORICAL), dim=D, sequence_combiner=comb)
    model = mm.DLRMModel(schema, embeddings=emb, bottom_block=mm.MLPBlock([128, D]), top_block=mm.MLPBlock([128, 64, 32]))
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    return model


def _fixed_batch(B, seed, device, ragged=None, mean_len=None, avoid=None):
    """The bench's batch on the capped tables (int32 ids; (B, L) for a bag); the features of `ragged` ({feature: offsets
    dtype}) as `__values` (the offsets' dtype) + `__offsets` with lengths 0 .. 2 mean_len and ~3 % ids -1, drawn below
    rows - avoid[f] when given."""
    ragged, avoid = ragged or {}, avoid or {}
    g = torch.Generator(device=device).manual_seed(seed)
    rng = np.random.default_rng(seed)
    x = {}
    for i, L in enumerate(BAG_SIZES, start=1):
        f = f"C{i}"
        rows = _rows(f, CAP)
        if f in ragged:
            lens = rng.integers(0, 2 * mean_len + 1, B)
            vals = rng.integers(0, rows - avoid.get(f, 0), int(lens.sum()))
            vals[rng.random(vals.size) < 0.03] = -1
            x[f + "__values"] = torch.from_numpy(vals).to(device=device, dtype=ragged[f])
            x[f + "__offsets"] = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).to(device=device, dtype=ragged[f])
        else:
            x[f] = torch.randint(0, rows, (B,) if L == 1 else (B, L), generator=g, device=device, dtype=torch.int32)
    for i in range(1, 14):
        x[f"I{i}"] = torch.rand(B, generator=g, device=device)
    return x, (torch.rand(B, generator=g, device=device) < 0.5).float()


def _long(x):
    return {k: v.long() if not v.is_floating_point() else v for k, v in x.items()}


def _close(ta, tb, what):
    for i, (va, vb) in enumerate(zip(_variables(ta), _variables(tb))):
        err = float((va - vb).abs().max()) / max(float(vb.abs().max()), 1e-30)
        assert err < 1e-5, f"{what}: variable {i} differs by {err:.3e} of its scale"


def _bag_input(x, f):
    """(int64 ids, int64 offsets) of a ragged feature, ((B, L) int64 ids, None) of a fixed-length one."""
    if f + "__values" in x:
        return x[f + "__values"].long(), x[f + "__offsets"].long()
    return x[f].long(), None


def _rows_of(tr, x):
    """rows_of for _reference_step: a bag's pooled rows in float64 from the fp32 table (the combiner over the ids in the
    table), a one-hot feature's rows."""
    onehot = {t: ops.widen_index(i).long() for t, i in enumerate(tr._idx) if t not in tr._bags}

    def rows_of(t, s, e):
        tab = tr.tables[t].table
        if t in onehot:
            return tab[onehot[t][s:e]].double()
        ids, offs = _bag_input(x, tr.feats[t])
        rows = tab.shape[0]
        if offs is None:
            i = ids[s:e]
            ok = (i >= 0) & (i < rows)
            return (tab[i.clamp(0, rows - 1)].double() * ok.unsqueeze(2)).sum(1)
        v = ids[offs[s]:offs[e]]
        seg = torch.arange(e - s, device=v.device).repeat_interleave(offs[s + 1:e + 1] - offs[s:e])
        ok = (v >= 0) & (v < rows)
        acc = torch.zeros((e - s, tab.shape[1]), dtype=torch.float64, device=v.device).index_add_(0, seg[ok], tab[v[ok]].double())
        cnt = torch.zeros(e - s, dtype=torch.float64, device=v.device).index_add_(0, seg, ok.double())
        comb = tr._bags[t]["comb"]
        den = torch.ones_like(cnt) if comb == "sum" else cnt.clamp_min(1.0) if comb == "mean" else cnt.clamp_min(1.0).sqrt()
        return acc / den.unsqueeze(1)

    return rows_of


def _check_gradients(tr, x, y, B):
    """(c) forward_backward (already run) against float64 autograd, bounds of test_dlrm_train_step_as_the_benchmark_runs_it:
    loss to 1e-5, dense gradients' Frobenius error under 1e-4 of their terms, slices (a bag's: the pooled-row gradient)
    per element within 1e-3 |ref| + 3e-4 max |ref slices of the sample|, leaving out the < 1 % relu-flip samples."""
    want_loss, want, terms, ref_slices, flipped = _reference_step(tr, x, y, B, rows_of=_rows_of(tr, x))
    np.testing.assert_allclose(float(tr.loss.item()), want_loss, rtol=1e-5)
    got = tr.gradients()
    assert sorted(got) == sorted(want)
    for k in want:
        fro = float((got[k].double() - want[k]).norm() / terms[k].norm())
        assert fro < 1e-4, f"{k}: Frobenius error {fro:.3e} of the terms' scale"
    n_flip = int(flipped.sum())
    assert n_flip < B // 100, f"{n_flip} samples have a relu unit on/off differently"
    keep = ~flipped
    scale = torch.stack([s.abs().amax(1) for s in ref_slices]).amax(0)[keep].unsqueeze(1)
    for t, f in enumerate(tr.feats):
        r = ref_slices[t][keep]
        _within(tr._slices[t][keep], r, 1e-3 * r.abs() + 3e-4 * scale, f"slices of {f}")


def _check_expansion(tr):
    """(d) every bag's expanded rows and update ids bit-equal to _expand_ref of its pooled-row gradient."""
    for t, bg in tr._bags.items():
        f, rows = tr.feats[t], tr.tables[t].table.shape[0]
        g = tr._slices[t]
        i = bg["ids"].reshape(-1).long()
        ok = (i >= 0) & (i < rows)
        if bg["offsets"] is None:
            L = bg["ids"].shape[1]
            seg = torch.arange(g.shape[0], device=g.device).repeat_interleave(L)
            den = None if bg["comb"] == "sum" else torch.full((g.shape[0],), float(L), device=g.device)
        else:
            offs = bg["offsets"].long()
            assert int(offs[0]) == 0 and int(offs[-1]) == i.numel()
            seg = torch.arange(g.shape[0], device=g.device).repeat_interleave(offs[1:] - offs[:-1])
            den = _den(torch.zeros(g.shape[0], dtype=torch.int64, device=g.device).index_add_(0, seg, ok.long()), bg["comb"])
        assert torch.equal(bg["rows"], _expand_ref(g, seg, ok, den)), f"expanded rows of {f}"
        assert torch.equal(bg["apply_ids"].long(), torch.where(ok, i, -1)), f"update ids of {f}"


def _check_update(tr):
    """(e) apply_gradients: every table against _check_sparse_update (a bag table with its update ids and expanded rows),
    then the map idle, the accumulators zero, the mirrors equal split_rows of their tables."""
    before = [(tb.table.clone(), a.clone(), None) for tb, a in zip(tr.tables, tr.tstate1)]
    grads = []
    for t in range(len(tr.tables)):
        bg = tr._bags.get(t)
        ids, vals = (bg["apply_ids"], bg["rows"]) if bg is not None else (tr._idx[t], tr._slices[t])
        grads.append((ops.widen_index(ids).long().reshape(-1), vals.clone()))  # the update folds duplicates in place
    tr.apply_gradients()
    hy = tr.hyper.cpu().numpy()
    for t, f in enumerate(tr.feats):
        tb = tr.tables[t]
        _check_update_by_rows("adagrad", f"Adagrad step, table of {f}", before[t], (tb.table, tr.tstate1[t], None), *grads[t], hy)
        grads[t] = None
        assert int((tr.rep[t] != INT_MAX).sum()) == 0, f"table of {f}: the representative map is not idle"
        assert tr.tdense[t] is None or float(tr.tdense[t].abs().max()) == 0.0, f"table of {f}: the accumulator was not cleared"
        assert torch.equal(tb._mirror, ops.split_rows(tb.table)), f"mirror of {f} out of step"


def test_multihot_train_step_as_the_benchmark_runs_it(device):
    """The bench's model on tables capped at CAP rows (8 bag tables on the election path, 6 on the dense path, C16 on
    the counting-sort path), B = 65 536, int32 (B, L) ids, one CUDA graph.
    (a) two graph replays against two eager steps of a twin on int64 ids: every variable within 1e-5 of its scale.
    (f) then one eager step of B - 37 on both (the leading rows of the pooled and expanded buffers), within 1e-5.
    (b) the trainer's pooled rows bit-equal to _seq_ref, their split copy to split_rows of them.
    (c) gradients against float64 autograd (_check_gradients); (d) the expansion bit for bit (_check_expansion);
    (e) the Adagrad update of every table (_check_update)."""
    B = BIG
    caps = {f: _rows(f, CAP) for f in BAG}
    assert sum(BAG.values()) == 203, "premise: 203 bag ids per sample"
    assert (sorted(f for f, r in caps.items() if r > DENSE_PATH_MAX_ROWS) == sorted(["C1", "C10", "C11", "C12", "C20", "C21", "C22", "C23"])
            and sorted(f for f, r in caps.items() if 1024 < r <= DENSE_PATH_MAX_ROWS) == sorted(["C2", "C4", "C5", "C14", "C15", "C24"])
            and [f for f, r in caps.items() if r <= 1024] == ["C16"]), "premise: the bag tables' update paths"
    ma, mb = _multihot_model(device, 21), _multihot_model(device, 21)
    ta, tb = ma.trainer(B), mb.trainer(B)
    assert ta.operand_rows and all(t._mirror is not None for t in ta.tables)
    batches = [_fixed_batch(B, 500 + i, device) for i in range(4)]
    ta.capture(*batches[0])
    for i in (0, 1):
        la = float(ta.replay(*batches[i]).item())
        lb = float(tb.step(_long(batches[i][0]), batches[i][1]).item())
        np.testing.assert_allclose(la, lb, rtol=1e-6)
    assert sorted(ta.feats[t] for t in ta._bags) == sorted(BAG)
    _close(ta, tb, "graph replay on int32 ids vs eager on int64 ids")
    # (f)
    x, y = batches[2]
    small = ({k: v[:B - 37] for k, v in x.items()}, y[:B - 37])
    ta.step(*small)
    tb.step(_long(small[0]), small[1])
    _close(ta, tb, f"eager step of {B - 37} samples after the capture")
    del tb, mb
    torch.cuda.empty_cache()

    # (b)
    x, y = batches[3]
    ta.forward_backward(x, y)
    for t, bg in ta._bags.items():
        f = ta.feats[t]
        assert torch.equal(bg["pooled"], _seq_ref(ta.tables[t].table, x[f].long(), "sum")), f"pooled rows of {f}"
        assert torch.equal(bg["split"], ops.split_rows(bg["pooled"])), f"split pooled rows of {f}"
    _check_gradients(ta, x, y, B)
    _check_expansion(ta)
    _check_update(ta)


RAGGED_FEATS = {"C16": ("mean", torch.int32), "C15": ("sqrtn", torch.int64), "C21": ("sum", torch.int32), "C1": ("mean", torch.int64)}


def test_ragged_features_at_scale_grow_then_reuse_their_buffers(device):
    """The model of test_multihot_train_step_as_the_benchmark_runs_it with four bags ragged (mean, sqrtn, sum on the
    counting-sort, vector-red and election paths; int32 offsets and values on two, int64 on the others), three eager steps
    at B = 65 536 with mean bag lengths 5, 9 and 3: the expanded-row and id buffers grow twice, then serve a shorter
    prefix.  Before the third step their tails are NaN rows and ids of rows that no bag of that batch holds; after it
    no NaN has reached a variable and those rows and their slots are unchanged.  The third step is checked as (c) to
    (e) of the fixed-length test."""
    B, free = BIG, 8
    model = _multihot_model(device, 31, {f: c for f, (c, _) in RAGGED_FEATS.items()})
    tr = model.trainer(B)
    dts = {f: dt for f, (_, dt) in RAGGED_FEATS.items()}
    sizes = []
    for step, m in ((1, 5), (2, 9)):
        tr.step(*_fixed_batch(B, 700 + step, device, dts, m))
        sizes.append({t: tr._bag_bufs[t]["rows"].shape[0] for t in tr._bags if tr.feats[t] in RAGGED_FEATS})
    assert len(sizes[0]) == 4 and all(sizes[1][t] > sizes[0][t] for t in sizes[0]), "premise: the buffers grow"
    x, y = _fixed_batch(B, 703, device, dts, 3, avoid={f: free for f in RAGGED_FEATS})
    held = {}
    for t, n in sizes[1].items():
        f = tr.feats[t]
        nnz = x[f + "__values"].numel()
        assert nnz < n, "premise: the third batch uses a prefix of the buffers"
        rows = tr.tables[t].table.shape[0]
        held[t] = torch.arange(rows - free, rows, device=device)
        buf = tr._bag_bufs[t]
        buf["rows"][nnz:] = float("nan")
        buf["ids"][nnz:] = held[t].to(buf["ids"].dtype).repeat(-(-(n - nnz) // free))[:n - nnz]
    kept = {t: (tr.tables[t].table[held[t]].clone(), tr.tstate1[t][held[t]].clone(), tr.tables[t]._mirror[held[t]].clone()) for t in held}
    tr.forward_backward(x, y)
    _check_gradients(tr, x, y, B)
    _check_expansion(tr)
    _check_update(tr)
    for v in _variables(tr) + tr.tstate1:
        assert not bool(torch.isnan(v).any()), "a NaN from a buffer tail reached a variable"
    for t, (w, a, mir) in kept.items():
        f = tr.feats[t]
        assert torch.equal(tr.tables[t].table[held[t]], w) and torch.equal(tr.tstate1[t][held[t]], a), f"{f}: a row no bag holds moved"
        assert torch.equal(tr.tables[t]._mirror[held[t]], mir), f"{f}: the mirror of a row no bag holds moved"
