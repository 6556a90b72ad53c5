"""Training DLRMModel on multi-hot features (ragged `name__values` + `name__offsets`, fixed-length (B, L) ids) on the GPU:
mm_bag_grad_rows against a float64 torch restatement, and whole training steps of models mixing one-hot, ragged and
fixed-length features against tests/multihot_oracle.py (autograd of the restated forward + the Keras update rules) and
against one step of the reference's torch DLRMModel (tests/golden/multihot/ref_torch_dlrm_train_multihot.npz)."""
from pathlib import Path

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200.blocks import set_table_mirror
from models_b200.schema import ColumnSchema, Schema, Tags
from oracle import oracle_train
from tests import helpers as H
from tests import multihot_oracle as MO

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------
def _ref_rows(g, ids, offsets, rows, comb):
    """float64 restatement for well-formed bags: row i = scale(bag(i)) * g[bag(i)], zero for ids outside [0, rows)."""
    g = g.double().cpu()
    if offsets is None:
        B, L = ids.shape
        seg = torch.arange(B).repeat_interleave(L)
        flat = ids.reshape(-1).cpu().long()
        scale = torch.full((B,), 1.0 / L if comb == "mean" else 1.0, dtype=torch.float64)
    else:
        off = offsets.cpu().long()
        B = off.numel() - 1
        seg = torch.arange(B).repeat_interleave(off[1:] - off[:-1])
        flat = ids.cpu().long()
        ok = (flat >= 0) & (flat < rows)
        cnt = torch.zeros(B, dtype=torch.float64).index_add(0, seg, ok.double())
        safe = torch.where(cnt > 0, cnt, torch.ones_like(cnt))
        scale = {"mean": 1.0 / safe, "sum": torch.ones(B, dtype=torch.float64), "sqrtn": 1.0 / safe.sqrt()}[comb]
    ok = ((flat >= 0) & (flat < rows)).double().unsqueeze(1)
    return g[seg] * scale[seg].unsqueeze(1) * ok


def _check_rows(got, g, ids, offsets, rows, comb):
    want = _ref_rows(g, ids, offsets, rows, comb)
    got = got.cpu()
    assert not torch.isnan(got).any(), "an output row was not written"
    if comb == "sum":
        assert torch.equal(got, want.float()), "scale 1: the rows must be copies of g"
    else:
        err = (got.double() - want).abs().max().item() / max(want.abs().max().item(), 1e-30)
        assert err < 1e-6, err


@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("id_dt,off_dt", [(torch.int32, torch.int32), (torch.int64, torch.int32), (torch.int32, torch.int64),
                                          (torch.int64, torch.int64)])
def test_bag_grad_rows_ragged(device, D, id_dt, off_dt):
    rng = np.random.default_rng(D + 7 * (id_dt == torch.int64) + 13 * (off_dt == torch.int64))
    rows = 1000
    lens = rng.integers(0, 12, 300)
    lens[[3, 17, 100]] = 0          # empty bags
    lens[5], lens[6] = 1, 300       # length 1 and a long bag
    offsets = np.concatenate([[0], np.cumsum(lens)])
    values = rng.integers(-3, rows + 3, int(offsets[-1]))  # ids < 0 and >= rows
    values[offsets[7]:offsets[8]] = -1  # a bag whose every id is pruned
    g = torch.from_numpy(rng.standard_normal((300, D)).astype(np.float32)).to(device)
    ids = torch.from_numpy(values).to(device=device, dtype=id_dt)
    offs = torch.from_numpy(offsets).to(device=device, dtype=off_dt)
    for comb in ("mean", "sum", "sqrtn"):
        out = torch.full((ids.numel(), D), float("nan"), device=device)
        ops.bag_grad_rows(g, ids, offs, rows, comb, out)
        _check_rows(out, g, ids, offs, rows, comb)


@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("L", [2, 3, 100])
@pytest.mark.parametrize("id_dt", [torch.int32, torch.int64])
def test_bag_grad_rows_fixed_length(device, D, L, id_dt):
    rng = np.random.default_rng(L * D)
    rows, B = 500, 257
    ids = torch.from_numpy(rng.integers(-2, rows + 2, (B, L))).to(device=device, dtype=id_dt)
    g = torch.from_numpy(rng.standard_normal((B, D)).astype(np.float32)).to(device)
    for comb in ("mean", "sum"):
        out = torch.full((B * L, D), float("nan"), device=device)
        ops.bag_grad_rows(g, ids, None, rows, comb, out)
        _check_rows(out, g, ids, None, rows, comb)
    with pytest.raises(ValueError, match="mm_bag_grad_rows"):
        ops.bag_grad_rows(g, ids, None, rows, "max", torch.empty((B * L, D), device=device))


def test_bag_grad_rows_malformed_offsets_stay_inside_out(device):
    """Decreasing offsets, offsets past nnz and negative offsets: every output row is written, nothing outside `out`."""
    D, nnz, guard = 32, 40, 8
    ids = torch.arange(nnz, dtype=torch.int32, device=device) % 7
    g = torch.randn((6, D), device=device)
    for off in ([5, 3, 20, 10, 60, 2, 1000], [-4, 7, 7, 2, 30, 35, 38], [10, 12, 14, 16, 18, 20, 22]):
        buf = torch.full((nnz + 2 * guard, D), float("nan"), device=device)
        out = buf[guard:guard + nnz]
        offs = torch.tensor(off, dtype=torch.int64, device=device)
        ops.bag_grad_rows(g, ids, offs, 7, "mean", out)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + nnz:]).all(), off
        assert not torch.isnan(out).any(), off
    # well-formed offsets with uncovered head and tail: those rows are zeros
    buf = torch.full((nnz, D), float("nan"), device=device)
    ops.bag_grad_rows(g, ids, torch.tensor([10, 12, 14, 16, 18, 20, 22], device=device), 7, "sum", buf)
    assert torch.equal(buf[:10], torch.zeros_like(buf[:10])) and torch.equal(buf[22:], torch.zeros_like(buf[22:]))


# ---------------------------------------------------------------------------------------------------------------
# whole training steps
# ---------------------------------------------------------------------------------------------------------------
# (name, rows, form, combiner): small tables take the dense accumulator path, C2 / bag_sum the election path
FEATS = [("C1", 300, "onehot", None), ("C2", 140000, "onehot", None), ("bag_mean", 50, "ragged", "mean"),
         ("bag_sum", 140000, "ragged", "sum"), ("bag_sqrtn", 300, "ragged", "sqrtn"), ("seq_mean", 40, 3, "mean"),
         ("seq_sum", 1000, 5, "sum")]


def _schema(feats):
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", is_list=form == "ragged", is_ragged=form == "ragged",
                         properties={"domain": {"min": 0, "max": rows - 1, "name": n}}) for n, rows, form, _ in feats]
    cols += [ColumnSchema(f"I{i}", tags=(Tags.CONTINUOUS,), dtype="float32") for i in (1, 2, 3)]
    cols.append(ColumnSchema("label", tags=(Tags.BINARY_CLASSIFICATION, Tags.TARGET), dtype="int64"))
    return Schema(cols)


def _model(device, feats, D, seed=3, combiners=None):
    mm.set_seed(seed)
    schema = _schema(feats)
    comb = combiners or {n: c for n, _, _, c in feats if c}
    emb = mm.Embeddings(schema.select_by_tag(Tags.CATEGORICAL), dim=D, sequence_combiner=comb)
    model = mm.DLRMModel(schema, embeddings=emb, bottom_block=mm.MLPBlock([32, D]), top_block=mm.MLPBlock([32, 16]))
    model.build(device)
    return schema, model


def _batch(feats, B, seed):
    """Ids repeated within and across bags (small tables), empty bags, ids < 0 in ragged bags."""
    rng = np.random.default_rng(seed)
    out = {}
    for n, rows, form, _ in feats:
        if form == "onehot":
            out[n] = rng.integers(0, rows, B).astype(np.int64)
        elif form == "ragged":
            lens = rng.integers(0, 6, B)
            offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
            vals = rng.integers(0, rows, int(offs[-1])).astype(np.int64)
            vals[rng.random(vals.size) < 0.1] = -1
            out[n + "__values"], out[n + "__offsets"] = vals, offs
        else:
            out[n] = rng.integers(0, rows, (B, form)).astype(np.int64)
    for i in (1, 2, 3):
        out[f"I{i}"] = rng.random(B).astype(np.float32)
    y = (rng.random(B) < 0.5).astype(np.float32)
    return out, y


def _state(model):
    tables, f2t = H.emb_tables(model.body.embeddings)
    return dict(tables={k: v.astype(np.float64) for k, v in tables.items()}, f2t=f2t, cont=model.body.continuous.features,
                bottom=H.mlp_layers(model.body.bottom_block), top=H.mlp_layers(model.body.top_block), head=H.head_layer(model.prediction))


def _flat(model):
    st = _state(model)
    out = [st["tables"][n] for n in sorted(st["tables"])]
    for tag in ("bottom", "top"):
        for l in st[tag]:
            out += [l["kernel"], l["bias"]]
    return out + [st["head"]["kernel"], st["head"]["bias"]]


def _combiners(model):
    return {f: t.sequence_combiner or "mean" for f, t in model.body.embeddings.feature_to_table.items()}


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("D,mirror", [(16, False), (64, True), (64, False)])
def test_multihot_training_steps_match_oracle(device, opt, D, mirror):
    """Three optimizer steps against autograd of the restated forward + the Keras update rules (float64), compared as in
    test_gpu_train.test_training_steps_match_oracle: the update of every variable to 0.1 in the Frobenius norm and 0.5
    of its largest element; rows no batch touched do not move; the staged forward then reads the trained tables."""
    set_table_mirror(mirror)
    try:
        schema, model = _model(device, FEATS, D)
        st = _state(model)
        comb = _combiners(model)
        before = [np.array(v, dtype=np.float64) for v in _flat(model)]
        lr = {"sgd": 1.0, "adagrad": 0.05, "adam": 0.01}[opt]
        eps = 1e-6 if opt == "adam" else 1e-7
        model.compile(optimizer={"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt])

        def slots(shape):
            if opt == "adagrad":
                return {"a": np.full(shape, 0.1)}
            return {"m": np.zeros(shape), "v": np.zeros(shape)} if opt == "adam" else {}

        tslots = {n: slots(t.shape) for n, t in st["tables"].items()}
        dslots = {}
        for step in (1, 2, 3):
            feats, y = _batch(FEATS, 256, seed=100 + step)
            m = model.train_step((H.device_batch(feats, device), torch.from_numpy(y).to(device)))
            loss, _, grads = MO.dlrm_loss_and_grads(feats, st["tables"], st["f2t"], comb, st["cont"], st["bottom"], st["top"], st["head"], y)
            np.testing.assert_allclose(m["loss"].item(), loss, rtol=1e-4)
            kw = dict(beta_1=0.9, beta_2=0.999, epsilon=eps, step=step)
            for f, tname in st["f2t"].items():
                uniq = MO.touched_rows(feats, f, st["tables"][tname].shape[0])
                st["tables"][tname] = oracle_train.sparse_update(opt, st["tables"][tname], uniq, grads[f"table/{tname}"][uniq],
                                                                 tslots[tname], lr, **kw)
            for tag in ("bottom", "top"):
                for i, l in enumerate(st[tag]):
                    for what in ("kernel", "bias"):
                        key = f"{tag}/{what}_{i}"
                        dslots.setdefault(key, slots(l[what].shape))
                        l[what] = oracle_train.dense_update(opt, l[what], grads[key], dslots[key], lr, **kw)
            for what in ("kernel", "bias"):
                key = f"head/{what}"
                dslots.setdefault(key, slots(st["head"][what].shape))
                st["head"][what] = oracle_train.dense_update(opt, st["head"][what], grads[key], dslots[key], lr, **kw)
        want = [st["tables"][n] for n in sorted(st["tables"])]
        for tag in ("bottom", "top"):
            for l in st[tag]:
                want += [l["kernel"], l["bias"]]
        want += [st["head"]["kernel"], st["head"]["bias"]]
        after = _flat(model)
        for i, (a, w, b0) in enumerate(zip(after, want, before)):
            upd_ref = np.asarray(w, dtype=np.float64) - b0
            assert np.max(np.abs(upd_ref)) > 0, i
            upd = np.asarray(a, dtype=np.float64) - b0
            fro = float(np.linalg.norm(upd - upd_ref) / np.linalg.norm(upd_ref))
            assert fro < 0.1, f"update of variable {i} after 3 {opt} steps: relative Frobenius error {fro:.3e}"
            err = float(np.max(np.abs(upd - upd_ref)) / np.max(np.abs(upd_ref)))
            assert err < 0.5, f"update of variable {i} after 3 {opt} steps: max error {err:.3e}"
            untouched = np.all(w == b0, axis=1) if w.ndim == 2 and i < len(st["tables"]) else None
            if untouched is not None:
                assert np.array_equal(np.asarray(a)[untouched], b0[untouched]), f"table {i}: an untouched row moved"
        # the staged forward of the same model reads the trained tables
        feats, y = _batch(FEATS, 200, seed=55)
        got = model(H.device_batch(feats, device)).cpu().numpy().reshape(-1)
        st = _state(model)
        _, logits, _ = MO.dlrm_loss_and_grads(feats, st["tables"], st["f2t"], comb, st["cont"], st["bottom"], st["top"], st["head"], y)
        assert H.rel_err(got, 1.0 / (1.0 + np.exp(-logits))) < 2e-4
    finally:
        set_table_mirror(None)


FIXED = [("C1", 300, "onehot", None), ("C2", 5000, "onehot", None), ("seq_mean", 40, 3, "mean"), ("seq_sum", 1000, 7, "sum")]


def test_graph_replay_equals_eager_steps_with_fixed_length_features(device):
    _, model_a = _model(device, FIXED, 32, seed=11)
    _, model_b = _model(device, FIXED, 32, seed=11)
    B = 512
    batches = []
    for s in range(4):
        f, y = _batch(FIXED, B, seed=s)
        batches.append((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    model_a.compile(optimizer=mm.Adagrad(0.05))
    model_b.compile(optimizer=mm.Adagrad(0.05))
    ta, tb = model_a.trainer(B), model_b.trainer(B)
    tb.capture(*batches[0])
    for i, (va, vb) in enumerate(zip(_flat(model_a), _flat(model_b))):
        assert np.array_equal(va, vb), i  # capture does not train
    for x, y in batches:
        la = ta.step(x, y).item()
        lb = tb.replay(x, y).item()
        np.testing.assert_allclose(la, lb, rtol=1e-6)
    for i, (va, vb) in enumerate(zip(_flat(model_a), _flat(model_b))):
        scale = max(float(np.max(np.abs(va))), 1e-30)
        assert float(np.max(np.abs(va - vb))) / scale < 1e-5, i


def test_capture_rejects_ragged_features(device):
    feats = [("C1", 300, "onehot", None), ("tags", 50, "ragged", "mean")]
    _, model = _model(device, feats, 16)
    model.compile(optimizer="sgd")
    f, y = _batch(feats, 64, seed=1)
    tr = model.trainer(64)
    with pytest.raises(NotImplementedError, match="ragged feature 'tags'"):
        tr.capture(H.device_batch(f, device), torch.from_numpy(y).to(device))


def test_out_of_range_ids_in_bags_are_counted_and_negative_ids_pruned(device):
    feats = [("C1", 300, "onehot", None), ("tags", 50, "ragged", "sum"), ("seq", 40, 3, "mean")]
    _, model = _model(device, feats, 16)
    model.compile(optimizer="sgd")
    f, y = _batch(feats, 64, seed=2)
    f["tags__values"] = f["tags__values"].copy()
    f["tags__values"][:5] = -1  # pruned silently
    model.train_step((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    model._trainer.check_indices()  # no error: ids < 0 in ragged bags are not out of range
    f["tags__values"][0] = 10**6
    f["seq"] = f["seq"].copy()
    f["seq"][2, 1] = 50
    before = {n: t.embeddings.clone() for n, t in model.body.embeddings.tables.items()}
    model.train_step((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    assert torch.isfinite(model._trainer.loss).all()
    with pytest.raises(IndexError, match="2 indices out of range"):
        model._trainer.check_indices()
    for n, t in model.body.embeddings.tables.items():
        assert t.embeddings.shape == before[n].shape


def test_rejections(device):
    feats = [("C1", 300, "onehot", None), ("seq", 40, 3, "max")]
    _, model = _model(device, feats, 16)
    model.compile(optimizer="sgd")
    f, y = _batch(feats, 32, seed=3)
    with pytest.raises(NotImplementedError, match="feature 'seq'.*max"):
        model.train_step((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    import torch.distributed as dist

    feats = [("C1", 300, "onehot", None), ("tags", 50, "ragged", "mean")]
    _, model = _model(device, feats, 16)
    model.compile(optimizer="sgd")
    f, y = _batch(feats, 32, seed=4)
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        tr = model.trainer(32, group=dist.group.WORLD)
        with pytest.raises(NotImplementedError, match="feature 'tags'.*process group"):
            tr.step(H.device_batch(f, device), torch.from_numpy(y).to(device))
    finally:
        dist.destroy_process_group()


def test_fit_on_a_parquet_list_column_learns_a_planted_rule(device, tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    rng = np.random.default_rng(0)
    n = 16000
    feats = [("C1", 50, "onehot", None), ("tags", 30, "ragged", "mean")]
    schema = _schema(feats)
    c1 = rng.integers(0, 50, n)
    lens = rng.integers(1, 6, n)
    offs = np.concatenate([[0], np.cumsum(lens)])
    vals = rng.integers(0, 30, int(offs[-1]))
    frac_low = np.add.reduceat((vals < 10).astype(np.float64), offs[:-1]) / lens  # share of the bag's ids below 10
    cont = {f"I{i}": rng.random(n).astype(np.float32) for i in (1, 2, 3)}
    score = 3.0 * frac_low + (c1 % 2 == 0) * 1.0 - 1.5
    click = (rng.random(n) < 1 / (1 + np.exp(-3 * score))).astype(np.int64)
    tags = pa.ListArray.from_arrays(pa.array(offs.astype(np.int32)), pa.array(vals.astype(np.int64)))
    d = tmp_path / "data"
    d.mkdir()
    ntr = 13000
    pq.write_table(pa.table({"C1": c1[:ntr], "tags": tags.slice(0, ntr), **{k: v[:ntr] for k, v in cont.items()}, "label": click[:ntr]}),
                   d / "train.parquet")
    loader = mm.Loader(str(d), batch_size=1000, shuffle=True, schema=schema, device=device)
    mm.set_seed(5)
    emb = mm.Embeddings(schema.select_by_tag(Tags.CATEGORICAL), dim=16, sequence_combiner="mean")
    model = mm.DLRMModel(schema, embeddings=emb, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    model.compile(optimizer=mm.Adam(0.02))
    hist = model.fit(loader, epochs=6)
    losses = hist.history["loss"]
    assert len(losses) == 6 and losses[-1] < losses[0] - 0.03, losses
    held_offs = (offs[ntr:] - offs[ntr]).astype(np.int32)
    held = {"C1": c1[ntr:], "tags__values": vals[offs[ntr]:], "tags__offsets": held_offs, **{k: v[ntr:] for k, v in cont.items()}}
    p = model(H.device_batch(held, device)).cpu().numpy().reshape(-1)
    y = click[ntr:]
    auc_pairs = (p[y == 1][:, None] > p[y == 0][None, :]).mean()
    assert auc_pairs > 0.6, auc_pairs


def test_bag_grad_rows_out_ids_mark_rows_without_a_gradient(device):
    """out_ids: the id where the row carries a gradient, -1 for positions no bag covers and ids outside [0, rows)."""
    D, rows = 16, 7
    vals = torch.tensor([3, 4, 1, 9, -2, 5, 6, 2, 0, 1], dtype=torch.int64, device=device)
    offs = torch.tensor([2, 5, 5, 8], dtype=torch.int32, device=device)  # positions 0, 1 and 8, 9 lie outside every bag
    g = torch.randn((3, D), device=device)
    out = torch.full((10, D), float("nan"), device=device)
    oi = torch.full((10,), 77, dtype=torch.int64, device=device)
    ops.bag_grad_rows(g, vals, offs, rows, "sum", out, out_ids=oi)
    assert oi.cpu().tolist() == [-1, -1, 1, -1, -1, 5, 6, 2, -1, -1]
    want = torch.zeros((10, D))
    want[2], want[5], want[6], want[7] = g[0].cpu(), g[2].cpu(), g[2].cpu(), g[2].cpu()
    assert torch.equal(out.cpu(), want)


def test_adam_does_not_move_rows_no_bag_holds(device):
    """A ragged batch whose offsets leave values uncovered (offsets[0] > 0): the rows only those values name keep their
    weights and slots under Adam (LazyAdam moves every row it is handed, even with a zero gradient)."""
    feats = [("C1", 300, "onehot", None), ("tags", 50, "ragged", "mean")]
    _, model = _model(device, feats, 16)
    model.compile(optimizer=mm.Adam(0.01))
    f, y = _batch(feats, 64, seed=9)
    held = set(f["tags__values"][f["tags__values"] >= 0].tolist())
    free = [r for r in range(50) if r not in held][:2]
    assert len(free) == 2
    f["tags__values"] = np.concatenate([np.array(free, dtype=np.int64), f["tags__values"]])
    f["tags__offsets"] = (f["tags__offsets"] + 2).astype(np.int32)
    tab = model.body.embeddings.feature_to_table["tags"]
    before = tab.embeddings.clone()
    for _ in range(2):
        model.train_step((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    after = tab.embeddings
    assert torch.equal(after[free], before[free])
    moved = sorted(held)
    assert not torch.equal(after[moved], before[moved])


def test_step_gradients_match_the_reference_torch_backend(device):
    """Loss and every gradient of ONE step against the reference's torch DLRMModel on one-hot columns plus a ragged column
    (tests/golden/make_golden_multihot.py): 3e-4 of each tensor's scale, as test_gpu_train does for one-hot features."""
    from tests.golden import replay

    z = replay.load(Path(__file__).parent / "golden" / "multihot" / "ref_torch_dlrm_train_multihot.npz")
    lists = {str(n) for n in z["list_names"]}
    feats = [(str(n), int(mx) + 1, "ragged" if str(n) in lists else "onehot", str(z["combiner"]) if str(n) in lists else None)
             for n, mx in zip(z["cat_names"], z["cat_max"])]
    cols = [ColumnSchema(n, tags=(Tags.CATEGORICAL,), dtype="int64", is_list=form == "ragged", is_ragged=form == "ragged",
                         properties={"domain": {"min": 0, "max": rows - 1, "name": n}}) for n, rows, form, _ in feats]
    cols += [ColumnSchema(str(n), tags=(Tags.CONTINUOUS,), dtype="float32") for n in z["cont_names"]]
    cols.append(ColumnSchema("click", tags=(Tags.BINARY_CLASSIFICATION, Tags.TARGET), dtype="int64"))
    schema = Schema(cols)
    dim = int(z["dim"])
    emb = mm.Embeddings(schema.select_by_tag(Tags.CATEGORICAL), dim=dim, sequence_combiner=str(z["combiner"]))
    model = mm.DLRMModel(schema, embeddings=emb, bottom_block=mm.MLPBlock([32, dim]), top_block=mm.MLPBlock([24, 8]))
    model.build(device)
    for name, t in model.body.embeddings.tables.items():
        t.table = torch.from_numpy(z[f"table_{name}"]).to(device).contiguous()
        t.built = True
    for blk, tag in ((model.body.bottom_block, "bottom"), (model.body.top_block, "top")):
        for l, w in zip(blk.dense_layers, replay.unpack_layers(z, tag)):
            l.set_weights(w["kernel"], w["bias"])
    h = replay.unpack_layers(z, "head")[0]
    model.prediction.to_call.set_weights(h["kernel"], h["bias"])
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z if k.startswith("batch_")}
    y = torch.from_numpy(z["targets"]).to(device)
    model.compile(optimizer=mm.SGD(0.0))
    tr = model.trainer(len(z["targets"]))
    tr.forward_backward(batch, y)
    np.testing.assert_allclose(tr.loss.item(), float(z["loss"]), rtol=1e-5)
    np.testing.assert_allclose(torch.sigmoid(tr.logits).cpu().numpy(), z["out"].reshape(-1), rtol=2e-4, atol=2e-6)

    def close(got, ref, what):
        got = got.detach().double().cpu().numpy()
        scale = max(float(np.max(np.abs(ref))), 1e-30)
        err = float(np.max(np.abs(got - ref))) / scale
        assert err < 3e-4, f"{what}: max |diff| / max |ref| = {err:.3e}"

    got = tr.gradients()
    for l, (tag, i) in zip(tr.arena.layers, [("bottom", 0), ("bottom", 1), ("top", 0), ("top", 1), ("head", 0)]):
        close(got[f"{l.name}/kernel"], z[f"grad_{tag}_kernel_{i}"], f"{tag} kernel {i}")
        close(got[f"{l.name}/bias"], z[f"grad_{tag}_bias_{i}"], f"{tag} bias {i}")
    for t, f in enumerate(tr.feats):
        rows = z[f"table_{f}"].shape[0]
        bag = tr._bags.get(t)
        ids, vals = (bag["apply_ids"], bag["rows"]) if bag is not None else (tr._idx[t], tr._slices[t])
        ids = ops.widen_index(ids).long().reshape(-1)
        keep = (ids >= 0) & (ids < rows)
        dense = torch.zeros((rows, dim), dtype=torch.float64, device=device).index_add_(0, ids[keep], vals[keep].double())
        close(dense, z[f"grad_table_{f}"], f"table {f}")
    assert f in lists and tr._bags  # the ragged column went through the bag path
