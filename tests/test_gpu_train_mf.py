"""MatrixFactorizationModel training on the GPU: mm_concat_backward_l2 against float64, then TwoTowerTrainer on tower-less
towers (mm.MatrixFactorizationModel compile / train_step / fit) against the reference's torch step
(tests/golden/mf_train/ref_torch_mf_train.npz) and the float64 restatement with the embeddings' L2 term
(tests/mf_train_oracle.py), graph replay, what training leaves in the model, and the configurations it refuses."""
import time

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, datasets, ops
from models_b200.graph import HostBatch, _view
from models_b200.schema import ColumnSchema, Schema
from tests import helpers as H
from tests import mf_train_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = __import__("pathlib").Path(__file__).parent / "golden" / "mf_train" / "ref_torch_mf_train.npz"


def close(got, ref, tol, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale if ref.size else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


# ---------------------------------------------------------------------------------------------------------------
# mm_concat_backward_l2
# ---------------------------------------------------------------------------------------------------------------
def _l2_case(device, B, widths, n_add, seed):
    """x0 (B, d) with a width-1 continuous column before every table (unaligned column offsets), n_add addends, one
    destination per table with NaN guard columns, a factor per table (every third one 0)."""
    g = np.random.default_rng(seed)
    cols, c = [], 0
    for w in widths:
        c += 1
        cols.append(c)
        c += w
    d = c + 1
    x0 = torch.from_numpy(g.standard_normal((B, d)).astype(np.float32)).to(device)
    adds = [torch.from_numpy(g.standard_normal((B, d)).astype(np.float32)).to(device) for _ in range(n_add)]
    dst = [torch.full((B, w + 4), float("nan"), device=device) for w in widths]
    lam = [0.0 if t % 3 == 2 else float(10.0 ** g.uniform(-5, -1)) for t in range(len(widths))]
    return x0, adds, dst, cols, lam


def _l2_run(x0, adds, dst, cols, lam, c0=0.25):
    loss = torch.tensor([c0, 0.0], device=x0.device)
    ws = ops.concat_l2_workspace(len(dst), x0.device)
    ops.concat_backward_l2(adds, [(t[:, :t.shape[1] - 4], c) for t, c in zip(dst, cols)], x0, lam, loss, ws)
    torch.cuda.synchronize()
    return loss


@pytest.mark.parametrize("B,widths,n_add", [
    (1, [4], 1),
    (37, [4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 44, 48, 52, 56, 60, 64, 68, 72, 76, 80, 84, 88, 92, 96, 100, 104, 108, 112,
         116, 120, 124, 128], 2),
    (1000, [64, 64], 1),
    (513, [4 + 4 * (t % 32) for t in range(64)], 3),
    (65536 + 37, [128, 64, 4], 1),
    (65536 + 37, [64], 4),
])
def test_concat_backward_l2_matches_float64(device, B, widths, n_add):
    x0, adds, dst, cols, lam = _l2_case(device, B, widths, n_add, seed=B + len(widths) + n_add)
    laps = (B * max(widths) // 4 + 255) // 256 / min(4 * torch.cuda.get_device_properties(device).multi_processor_count,
                                                      _cabi.CONCAT_L2_CTAS)
    if B > 65536:
        assert laps > 2, "premise: several grid-stride laps"
    loss = _l2_run(x0, adds, dst, cols, lam)
    xd = x0.double().cpu()
    ad = sum(a.double().cpu() for a in adds)
    reg = 0.0
    for t, (w, c, l) in enumerate(zip(widths, cols, lam)):
        want = ad[:, c:c + w] + 2 * l * xd[:, c:c + w]
        got = dst[t][:, :w].double().cpu()
        bound = 4e-7 * (sum(a.double().cpu()[:, c:c + w].abs() for a in adds) + 2 * l * xd[:, c:c + w].abs()) + 1e-30
        assert ((got - want).abs() <= bound).all(), f"slice {t} (width {w}, col {c}, l2 {l})"
        assert torch.isnan(dst[t][:, w:]).all(), f"slice {t}: guard columns written"
        reg += l * float((xd[:, c:c + w] ** 2).sum())
    got_reg, got_total = float(loss[1].item()), float(loss[0].item())
    assert abs(got_reg - reg) <= 1e-5 * reg, (got_reg, reg)
    assert abs(got_total - (0.25 + reg)) <= 1e-6 * (0.25 + reg)
    dst2 = [torch.full_like(t, float("nan")) for t in dst]
    loss2 = _l2_run(x0, adds, dst2, cols, lam)
    assert torch.equal(loss, loss2), "two runs give different bits"
    for a, b in zip(dst, dst2):
        assert torch.equal(a[:, :a.shape[1] - 4], b[:, :b.shape[1] - 4])


def test_concat_backward_l2_rejects_bad_arguments(device):
    x0, adds, dst, cols, lam = _l2_case(device, 8, [8, 8], 1, seed=1)
    loss = torch.zeros(2, device=device)
    sl = [(t[:, :8], c) for t, c in zip(dst, cols)]
    ws = ops.concat_l2_workspace(2, device)
    with pytest.raises(ValueError, match="l2"):
        ops.concat_backward_l2(adds, sl, x0, [1e-3, -1.0], loss, ws)
    with pytest.raises(ValueError, match="partials"):
        ops.concat_backward_l2(adds, sl, x0, lam[:2], loss, ws[:100])
    with pytest.raises(ValueError, match="one l2 factor"):
        ops.concat_backward_l2(adds, sl, x0, [1e-3], loss, ws)
    with pytest.raises(ValueError, match="loss"):
        ops.concat_backward_l2(adds, sl, x0, lam[:2], torch.zeros(1, device=device), ws)
    bad = [(dst[0][:, 1:9], cols[0])]  # not 16-byte aligned: the rule mm_concat_backward has
    with pytest.raises(ValueError, match="16-byte"):
        ops.concat_backward_l2(adds, bad, x0, lam[:1], loss, ws)


# ---------------------------------------------------------------------------------------------------------------
# one step through mm.MatrixFactorizationModel
# ---------------------------------------------------------------------------------------------------------------
def _golden_model(z, device, T, l2_reg=0.0, post=None):
    dim = int(z["dim"])

    def col(name, tag):
        props = {"domain": {"min": 0, "max": int(z[f"{tag}_table_{name}_rows_total"]) - 1, "name": name}}
        tags = ("user", "user_id") if tag == "query" else ("item", "item_id")
        return ColumnSchema(name, tags=("categorical",) + tags, dtype="int64", properties=props)

    schema = Schema([col(str(z["query_cols"][0]), "query"), col(str(z["item_cols"][0]), "item")])
    model = mm.MatrixFactorizationModel(schema, dim, embeddings_l2_reg=l2_reg, post=post, logits_temperature=T)
    for tag, tw in (("query", model.body.query), ("item", model.body.item)):
        for name, table in tw.inputs.embeddings.tables.items():
            full = torch.zeros((int(z[f"{tag}_table_{name}_rows_total"]), dim), dtype=torch.float32)
            full[torch.from_numpy(z[f"{tag}_table_{name}_ids"])] = torch.from_numpy(z[f"{tag}_table_{name}_rows"])
            table.table = full.to(device).contiguous()
            table.built = True
    model.build(device)
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z.files if k.startswith("batch_")}
    return model, batch


def _summed_slices(tr, z, tag, name, dim):
    ids, rows = (t.cpu().numpy() for t in tr.table_gradients()[name])
    ref_ids = z[f"{tag}_table_{name}_ids"]
    summed = np.zeros((len(ref_ids), dim))
    assert np.isin(ids, ref_ids).all()
    np.add.at(summed, np.searchsorted(ref_ids, ids), rows.astype(np.float64))
    return summed


@pytest.mark.parametrize("variant", [0, 1])
def test_one_step_matches_reference(device, variant):
    """The reference's torch step (no L2 term: its torch backend has no add_loss): the loss at rtol 1e-5, each table's
    summed IndexedSlices at 3e-4 of its scale, at T = 1 and T = 0.5; a tower-less step launches no dense update."""
    z = np.load(GOLDEN)
    vt, T = [(f"T{float(t):g}".replace(".", "p"), float(t)) for t in z["temperatures"]][variant]
    model, batch = _golden_model(z, device, T)
    B, dim = int(z["batch_movieId"].shape[0]), int(z["dim"])
    model.compile(optimizer="sgd")
    tr = model.trainer(B)
    assert tr.arena.size == 0 and not tr._tc_layers
    tr.forward_backward(batch)
    torch.cuda.synchronize()
    want = float(z[f"{vt}_loss"])
    assert abs(float(tr.loss[0].item()) - want) <= 1e-5 * abs(want)
    assert float(tr.loss[1].item()) == 0.0
    for tag in ("query", "item"):
        name = str(z[f"{tag}_cols"][0])
        close(_summed_slices(tr, z, tag, name, dim), z[f"{vt}_grad_{tag}_table_{name}_rows"], 3e-4, f"table {name}")


@pytest.mark.parametrize("post", [None, "l2-norm"])
def test_one_step_with_l2_reg_matches_restatement(device, post):
    """embeddings_l2_reg > 0 on the fixture's batch: loss = CE + reg, regularization_loss = reg and both tables'
    IndexedSlices against the float64 restatement."""
    z = np.load(GOLDEN)
    lam = 2e-3
    model, batch = _golden_model(z, device, 0.5, l2_reg=lam, post=post)
    B, dim = int(z["batch_movieId"].shape[0]), int(z["dim"])
    ob, towers, _ = O.golden_inputs(z)
    want, want_reg, _, grads = O.mf_loss_and_grads(ob, towers, "movieId", temperature=0.5, l2=post is not None,
                                                   l2_reg={"query": lam, "item": lam})
    assert want_reg > 0.01 * want, "premise: the L2 term is not negligible"
    model.compile(optimizer="sgd")
    tr = model.trainer(B)
    tr.forward_backward(batch)
    torch.cuda.synchronize()
    assert abs(float(tr.loss[0].item()) - want) <= 1e-5 * want
    assert abs(float(tr.loss[1].item()) - want_reg) <= 1e-5 * want_reg
    for tag in ("query", "item"):
        name = str(z[f"{tag}_cols"][0])
        close(_summed_slices(tr, z, tag, name, dim), grads[f"{tag}/table/{name}"], 3e-4, f"{post} table {name}")
    out = model.train_step((batch,))  # the public step: the same numbers, then the update
    np.testing.assert_allclose([float(out["loss"].item()), float(out["regularization_loss"].item())], [want, want_reg],
                               rtol=1e-5)
    assert float(out["loss_batch"].item()) == float(out["loss"].item())


def _oracle_towers(model):
    out = {}
    for tag, tb in (("query", model.body.query), ("item", model.body.item)):
        emb = tb.inputs.embeddings
        out[tag] = {"tables": {f: H.to_numpy(t.table) for f, t in emb.feature_to_table.items()},
                    "combiner": {f: t.sequence_combiner or "mean" for f, t in emb.feature_to_table.items()},
                    "continuous": list(tb.inputs.continuous.features) if tb.inputs.continuous is not None else [],
                    "layers": H.mlp_layers(tb.mlp) if tb.mlp is not None else []}
    return out


def _oracle_batch(feats, towers):
    b = dict(feats)
    for t in towers.values():
        for f in t["tables"]:
            if f + "__values" in feats:
                b[f] = (feats[f + "__values"], feats[f + "__offsets"])
    return b


def _batch(schema, n, seed):
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, n, seed=seed))
    return feats


def test_twotower_with_l2_reg_matches_restatement(device):
    """A TwoTowerModel with embeddings_l2_reg on ML-1M: towers [64, 32], the ragged genres bag (the term on its pooled
    row, expanded by mm_bag_grad_rows), continuous columns (no term): loss, regularization, every dense gradient and
    every table's gradient."""
    lam = 1e-3
    mm.set_seed(5)
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([64, 32]), logits_temperature=0.5,
                             embedding_options=mm.EmbeddingOptions(embedding_dim_default=16, embeddings_l2_reg=lam))
    feats = _batch(schema, 256, 77)
    model.build(device)
    towers = _oracle_towers(model)
    want, want_reg, _, grads = O.mf_loss_and_grads(_oracle_batch(feats, towers), towers, "movieId", temperature=0.5,
                                                   l2_reg={"query": lam, "item": lam})
    model.compile(optimizer="sgd")
    tr = model.trainer(256)
    tr.forward_backward(H.device_batch(feats, device))
    torch.cuda.synchronize()
    assert abs(float(tr.loss[0].item()) - want) <= 2e-5 * want and abs(float(tr.loss[1].item()) - want_reg) <= 1e-5 * want_reg
    g = tr.gradients()
    for tag, tw in (("query", model.body.query), ("item", model.body.item)):
        for i, l in enumerate(tw.mlp.dense_layers):
            close(g[f"{tw.name}/{l.name}/kernel"], grads[f"{tag}/kernel_{i}"], 3e-4, f"{tag} kernel {i}")
            close(g[f"{tw.name}/{l.name}/bias"], grads[f"{tag}/bias_{i}"], 3e-4, f"{tag} bias {i}")
    for f, (ids, rows) in tr.table_gradients().items():
        tag = "query" if f in towers["query"]["tables"] else "item"
        ref = grads[f"{tag}/table/{f}"]
        dense = np.zeros_like(ref)
        ids, rows = ids.cpu().numpy().astype(np.int64), rows.cpu().numpy().astype(np.float64)
        ok = ids >= 0
        np.add.at(dense, ids[ok], rows[ok])
        close(dense, ref, 3e-4, f"table {f}")


def _mf_ml1m(device, lam, post=None, dim=32, seed=9):
    mm.set_seed(seed)
    schema = datasets.movielens_1m_schema()
    model = mm.MatrixFactorizationModel(schema, dim, embeddings_l2_reg=lam, post=post, logits_temperature=0.5)
    model.build(device)
    return schema, model


def _hyper(opt):
    return dict(beta_1=float(np.float32(0.9)), beta_2=float(np.float32(0.999)), epsilon=float(np.float32(1e-7))) if opt == "adam" else {}


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_match_restatement(device, opt):
    """Three steps with embeddings_l2_reg = 1e-3, the last batch smaller than the compiled one: loss and regularization
    per step, and every table's update, against the restatement with the Keras update rules."""
    lam = 1e-3
    schema, model = _mf_ml1m(device, lam)
    feats = [_batch(schema, n, 300 + i) for i, n in enumerate((256, 256, 200))]
    towers0 = _oracle_towers(model)
    lr = {"sgd": 0.5, "adagrad": 0.05, "adam": 0.002}[opt]
    model.compile(optimizer={"sgd": mm.SGD, "adagrad": mm.Adagrad, "adam": mm.Adam}[opt](learning_rate=lr))
    model.trainer(256)
    got = []
    for f in feats:
        m = model.train_step((H.device_batch(f, device),))
        got.append((float(m["loss"].item()), float(m["regularization_loss"].item())))
    want, towers = O.mf_train_steps([_oracle_batch(f, towers0) for f in feats], towers0, "movieId", opt, lr, temperature=0.5,
                                    l2_reg={"query": lam, "item": lam}, **_hyper(opt))
    np.testing.assert_allclose(np.array(got), np.array(want), rtol=2e-4)
    now = _oracle_towers(model)
    tol = 2e-3 if opt == "adam" else 5e-4
    for tag in ("query", "item"):
        for f in now[tag]["tables"]:
            close(now[tag]["tables"][f] - towers0[tag]["tables"][f], towers[tag]["tables"][f] - towers0[tag]["tables"][f], tol,
                  f"{opt}: {tag} table {f} update")


def test_graph_replay_on_packed_ids_equals_eager(device):
    """Two graph replays on 3-byte packed ids (HostBatch) against two eager steps of a twin model on int64 ids."""
    B, lam = 512, 1e-4
    hosts, results = None, []
    for mode in ("graph", "eager"):
        mm.set_seed(13)
        schema = datasets.retrieval_10m_schema(n_items=50_000, n_users=5_000)
        model = mm.MatrixFactorizationModel(schema, 64, embeddings_l2_reg=lam)
        model.build(device)
        model.compile(optimizer=mm.Adagrad(0.05))
        tr = model.trainer(B)
        names = model.input_columns()
        hosts = hosts or [datasets.generate_batch(schema, B, seed=40 + i, index_dtype=np.int32) for i in range(2)]
        losses = []
        if mode == "graph":
            widths = model.id_bytes()
            assert max(widths.values()) <= 3, widths
            hbs = [HostBatch.like(h, names, id_bytes=widths) for h in hosts]
            packed = [hb.buffer.to(device) for hb in hbs]
            static = packed[0].clone()
            inputs = {k: _view(static, hbs[0].offsets[k], shp, dt) for k, (shp, dt) in hbs[0].spec.items()}
            tr.capture(inputs, clone=False)
            for p in packed:
                static.copy_(p)
                out = tr.replay()
                losses.append((float(out[0].item()), float(out[1].item())))
        else:
            for h in hosts:
                x = {k: torch.from_numpy(np.asarray(h[k]).astype(np.int64)).to(device) for k in names}
                out = tr.step(x, None)
                losses.append((float(out[0].item()), float(out[1].item())))
        torch.cuda.synchronize()
        results.append((losses, {k: np.array(v) for k, v in model.state_dict().items()}))
    (lg, wg), (le, we) = results
    np.testing.assert_allclose(lg, le, rtol=1e-6)
    for k in we:
        np.testing.assert_allclose(wg[k], we[k], rtol=1e-6, atol=1e-7, err_msg=k)


def test_trained_model_forward_evaluate_topk_and_save_load(device, tmp_path):
    schema, model = _mf_ml1m(device, 1e-4, post="l2-norm")
    feats = [_batch(schema, 128, 60 + i) for i in range(3)]
    model.compile(optimizer="adam")
    hist = model.fit([H.device_batch(f, device) for f in feats], batch_size=128, epochs=2)
    assert sorted(hist.history) == ["loss", "regularization_loss"]
    assert len(hist.history["loss"]) == 2 and all(r > 0 for r in hist.history["regularization_loss"])
    assert all(l > r for l, r in zip(hist.history["loss"], hist.history["regularization_loss"]))
    x = H.device_batch(feats[0], device)
    scores = model(x)
    assert tuple(scores.shape) == (128, 1)
    q = O.l2_normalize(torch.from_numpy(H.to_numpy(model.body.query.inputs.embeddings.tables["userId"].table)).double())
    it = O.l2_normalize(torch.from_numpy(H.to_numpy(model.body.item.inputs.embeddings.tables["movieId"].table)).double())
    u, m = feats[0]["userId"].astype(np.int64), feats[0]["movieId"].astype(np.int64)
    close(scores.reshape(-1), (q[u] * it[m]).sum(-1), 1e-5, "scores")
    res = model.evaluate([x], item_corpus={"movieId": feats[1]["movieId"]})
    assert 0.0 <= res["recall_at_10"] <= 1.0
    enc = model.to_top_k_encoder({"movieId": np.arange(100, dtype=np.int64)}, k=5)
    top = enc({"userId": x["userId"][:8]})
    ids = top.identifiers if hasattr(top, "identifiers") else top[1]
    sc = top.scores if hasattr(top, "scores") else top[0]
    want = (q[u[:8]] @ it[:100].T).topk(5, dim=1)
    close(sc, want.values, 1e-5, "top-k scores")
    model.save(str(tmp_path / "mf"))
    back = mm.Model.load(str(tmp_path / "mf"), device=device)
    sd, sd2 = model.state_dict(), back.state_dict()
    assert sd.keys() == sd2.keys() and all(np.array_equal(sd[k], sd2[k]) for k in sd)
    assert torch.equal(back(x), scores)


def test_fit_learns_a_planted_rule(device):
    """Item id = f(user id): in-batch recall@10 rises by at least 0.3."""
    mm.set_seed(11)
    schema = datasets.retrieval_10m_schema(n_items=50_000, n_users=5_000)
    model = mm.MatrixFactorizationModel(schema, 64, embeddings_l2_reg=1e-5)
    g = np.random.default_rng(0)
    n_users = 2000
    rule = g.integers(0, 50_000, n_users)

    def batch(seed):
        r = np.random.default_rng(seed)
        f = _batch(schema, 256, seed)
        f["user_id"] = r.integers(0, n_users, 256).astype(f["user_id"].dtype)
        f["item_id"] = rule[f["user_id"]].astype(f["item_id"].dtype)
        return H.device_batch(f, device)

    train = [batch(1000 + i) for i in range(40)]
    held = [batch(5000 + i) for i in range(4)]
    before = model.evaluate(held)["recall_at_10"]
    model.compile(optimizer=mm.Adam(0.01))
    hist = model.fit(train, batch_size=256, epochs=5)
    after = model.evaluate(held)["recall_at_10"]
    assert hist.history["loss"][-1] < hist.history["loss"][0], hist.history["loss"]
    assert after > before + 0.3, (before, after, hist.history["loss"])


def test_step_at_benchmark_size(device):
    """retrieval_10m_schema (10 M x 64 items, 1 M x 64 users), B = 16 384, embeddings_l2_reg = 1e-4, Adagrad, one captured
    step: the loss, the regularization and the IndexedSlices on 512 sampled rows against float64 (the soft-max over the
    whole batch in float64 on the device)."""
    B, lam = 16384, 1e-4
    mm.set_seed(21)
    schema = datasets.retrieval_10m_schema()
    model = mm.MatrixFactorizationModel(schema, 64, embeddings_l2_reg=lam)
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.01))
    torch.cuda.reset_peak_memory_stats(device)
    t0 = time.perf_counter()
    tr = model.trainer(B)
    host = datasets.generate_batch(schema, B, seed=808, index_law="zipf", index_dtype=np.int32)
    x = {k: torch.from_numpy(np.asarray(host[k])).to(device) for k in model.input_columns()}
    tr.capture(x)
    qi = [x["user_id"].long(), x["item_id"].long()]

    def reference(tables):
        q, it = (tables[t][qi[t]].double() for t in range(2))
        s = q @ it.T
        same = qi[1].view(-1, 1) == qi[1].view(1, -1)
        neg = torch.where(same, torch.full_like(s, float(np.float32(O.MIN_FLOAT))), s)
        logits = torch.cat([s.diagonal().view(-1, 1), neg], 1)
        want_reg = lam * float((q * q).sum() + (it * it).sum())
        want = float((torch.logsumexp(logits, 1) - logits[:, 0]).mean()) + want_reg
        return q, it, torch.softmax(logits, 1) / B, want, want_reg

    tables0 = [t.table.clone() for t in tr.tables]
    tr.replay()  # the captured step: its loss and regularization against the tables it started from
    torch.cuda.synchronize()
    _, _, _, want, want_reg = reference(tables0)
    assert abs(float(tr.loss[1].item()) - want_reg) <= 1e-5 * want_reg and abs(float(tr.loss[0].item()) - want) <= 1e-5 * want
    del tables0
    # the update folds duplicate ids' slices in place, so the IndexedSlices are checked on an eager forward_backward
    tables1 = [t.table.clone() for t in tr.tables]
    tr.forward_backward(x)
    torch.cuda.synchronize()
    q, it, p, want, want_reg = reference(tables1)
    assert abs(float(tr.loss[1].item()) - want_reg) <= 1e-5 * want_reg and abs(float(tr.loss[0].item()) - want) <= 1e-5 * want
    rows = torch.from_numpy(np.random.default_rng(1).choice(B, 512, replace=False)).to(device)
    dq = p[rows, :1] * it[rows] + p[rows, 1:] @ it - it[rows] / B + 2 * lam * q[rows]
    di = p[rows, :1] * q[rows] + p[:, 1:][:, rows].T @ q - q[rows] / B + 2 * lam * it[rows]
    close(tr.slices[0][rows], dq, 3e-4, "user slices")
    close(tr.slices[1][rows], di, 3e-4, "item slices")
    took = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(device) / 2**30
    print(f"MF step at B = {B}: trainer + capture + replay + reference in {took:.1f} s, peak {peak:.2f} GiB")


def test_refused_configurations(device):
    """Each refusal is the trainer's existing message."""
    from models_b200.retrieval import PopularityBasedSamplerV2

    schema = datasets.movielens_1m_schema()
    x = H.device_batch(_batch(schema, 64, 1), device)

    def fails(model, match, group=None):
        model.compile(optimizer="sgd")
        with pytest.raises(NotImplementedError, match=match):
            if group is None:
                model.train_step((x,))
            else:
                model.trainer(64, group=group)

    fails(mm.MatrixFactorizationModel(schema, 16, samplers=[PopularityBasedSamplerV2(max_id=3000)]), "in-batch")
    m = mm.MatrixFactorizationModel(schema, 16)
    m.prediction.scorer.sampled_softmax_mode = True
    fails(m, "sampled_softmax_mode")
    fails(mm.MatrixFactorizationModel(schema, 16), "process group", group=object())
    fails(mm.MatrixFactorizationModel(schema, 6), "multiple of 4")
    fails(mm.MatrixFactorizationModel(schema, 132), "up to 128")
    mm.set_dense_engine("fp32")
    try:
        fails(mm.MatrixFactorizationModel(schema, 16), "fp32")
    finally:
        mm.set_dense_engine("auto")
