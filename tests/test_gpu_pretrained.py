"""Training and serving with pretrained embeddings on the GPU: DCN and sequential (MLP, MMoE) training steps against the
float64 restatement (tests/pretrained_oracle.py) — loss, logits and every dense gradient, the projection's included —,
eager steps equal to CUDA-graph replays, the EmbeddingOperator path bit-equal to a batch that carries the vectors, the
reference's DCN test configuration and notebook flow through fit / evaluate, save / load and the compiled forward, and
one step at B = 65 536, Dp = 768."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import pretrained_oracle as PO

pytestmark = pytest.mark.gpu
TOL = 3e-4
ROWS = 50


def close(got, ref, tol, what):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale if ref.size else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def _schema(rows=ROWS):
    return Schema([
        ColumnSchema("item_category", tags=(Tags.CATEGORICAL,), dtype="int64", properties={"domain": {"min": 0, "max": rows - 1}}),
        ColumnSchema("user_age", tags=(Tags.CONTINUOUS,)),
        ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
    ])


def _setup(dims, device, seed=0, rows=ROWS):
    """Schema with one EmbeddingOperator per (name, Dp), the operators' host matrices and the operators (the caller keeps
    them alive, as a Loader does with its transforms)."""
    rng = np.random.default_rng(seed)
    schema, mats, ops_ = _schema(rows), {}, []
    for name, Dp in dims:
        mats[name] = rng.random((rows, Dp)).astype(np.float32)
        ops_.append(mm.EmbeddingOperator(mats[name], lookup_key="item_category", embedding_name=name, device=device))
        schema = ops_[-1].compute_output_schema(schema)
    return schema, mats, ops_


def _batch(B, device, seed, rows=ROWS):
    rng = np.random.default_rng(seed)
    feats = {"item_category": rng.integers(0, rows, B).astype(np.int32), "user_age": rng.random(B).astype(np.float32)}
    y = (rng.random(B) < 0.4).astype(np.float32)
    return feats, y


def _dev(feats, device):
    return {k: torch.from_numpy(v).to(device) for k, v in feats.items()}


def _model(kind, schema, output_dims, l2):
    pe = mm.PretrainedEmbeddings(schema.select_by_tag(Tags.EMBEDDING), output_dims=output_dims,
                                 normalizer="l2-norm" if l2 else None)
    ib = mm.InputBlockV2(schema, categorical=mm.Embeddings(schema.select_by_tag(Tags.CATEGORICAL), dim=8),
                         pretrained_embeddings=pe)
    if kind == "dcn":
        return mm.DCNModel(schema, depth=2, input_block=ib, deep_block=mm.MLPBlock([32, 16]), prediction_tasks=mm.BinaryOutput("click"))
    if kind == "mlp":
        return mm.Model(ib, mm.MLPBlock([32, 16]), mm.BinaryOutput("click"))
    out = mm.BinaryOutput("click")
    return mm.Model(ib, mm.MLPBlock([32]), mm.MMOEBlock(out, mm.MLPBlock([16]), 3), out)


def _np(t):
    return None if t is None else t.detach().cpu().numpy().astype(np.float64)


def _layers(ls):
    return [{"kernel": _np(l.kernel), "bias": _np(l.bias), "activation": l.activation} for l in ls]


def _restate(model, tr, kind, feats, y, mats, dense):
    """The restatement's loss, logits and gradients, and the trainer's gradients under the same keys."""
    ib = model.body.input_block
    b = len(y)
    emb = ib.embeddings
    tables = {f: _np(emb.feature_to_table[f].table) for f in emb.feature_names}
    pre = []
    got = {}
    a = tr.arena
    for n, br in ib.pretrained.branches.items():
        proj = None
        if br.projection is not None:
            proj = {"name": f"proj_{n}", "kernel": _np(br.projection.kernel), "bias": _np(br.projection.bias)}
            li = a.layers.index(br.projection)
            got[f"proj_{n}/kernel"], got[f"proj_{n}/bias"] = a.view(a.grad, li, "kernel"), a.view(a.grad, li, "bias")
        pre.append({"name": n, "P": mats[n][feats["item_category"]] if dense else mats[n],
                    "ids": None if dense else feats["item_category"], "proj": proj, "l2": br.l2})
    masks, layers = {}, {}
    if kind == "dcn":
        layers = {"cross": _layers([c.dense for c in model.body.cross.cross_layers]), "deep": _layers(tr.deep)}
        masks = {f"deep_{i}": (tr.h[i][:b] > 0).cpu().numpy() for i in range(len(tr.deep))}
        for i, l in enumerate(tr.cross):
            li = a.layers.index(l)
            got[f"cross/kernel_{i}"], got[f"cross/bias_{i}"] = a.view(a.grad, li, "kernel"), a.view(a.grad, li, "bias")
        for i, l in enumerate(tr.deep):
            li = a.layers.index(l)
            got[f"deep/kernel_{i}"], got[f"deep/bias_{i}"] = a.view(a.grad, li, "kernel"), a.view(a.grad, li, "bias")
    else:
        layers["bottom"] = _layers(tr.bottom)
        masks = {f"bottom_{i}": (tr.h[i][:b] > 0).cpu().numpy() for i in range(len(tr.bottom))}
        for i, l in enumerate(tr.bottom):
            got[f"bottom/kernel_{i}"], got[f"bottom/bias_{i}"] = a.view(a.grad, i, "kernel"), a.view(a.grad, i, "bias")
        if kind == "mmoe":
            mo = tr.mmoe
            layers["experts"] = {"kernel": _np(mo.experts.kernel), "bias": _np(mo.experts.bias), "activation": mo.experts.activation,
                                 "E": mo.num_experts}
            layers["gates"] = _np(mo.gates.kernel)
            masks["experts"] = (tr.X[:b] > 0).cpu().numpy()
            got["experts/kernel"], got["experts/bias"] = a.view(a.grad, tr.li_experts, "kernel"), a.view(a.grad, tr.li_experts, "bias")
            got["gates/kernel"] = a.view(a.grad, tr.li_gates, "kernel")
    hi = len(a.layers) - 1
    got["head/kernel"], got["head/bias"] = a.view(a.grad, hi, "kernel"), a.view(a.grad, hi, "bias")
    head = {"kernel": _np(model.prediction.to_call.kernel), "bias": _np(model.prediction.to_call.bias)}
    loss, z, g = PO.loss_and_grads(feats, tables, ["user_age"], pre, kind, layers, head, y, masks=masks)
    return loss, z, g, got


@pytest.mark.parametrize("kind", ["dcn", "mlp", "mmoe"])
@pytest.mark.parametrize("dims,output_dims,l2,dense", [
    ((("pretrained_category_embeddings", 12),), 16, False, False),   # the reference test's configuration
    ((("pre_a", 300), ("pre_b", 16)), {"pre_a": 64}, True, False),
    ((("pre_a", 20),), 8, True, True),                               # the batch carries the vectors
    ((("pre_a", 12),), None, False, False),                          # unprojected
])
def test_training_step_matches_restatement(device, kind, dims, output_dims, l2, dense):
    mm.set_seed(11)
    schema, mats, _ops = _setup(dims, device)
    model = _model(kind, schema, output_dims, l2)
    model.compile(optimizer="adagrad")
    B = 257
    feats, y = _batch(B, device, 3)
    x = _dev(feats, device)
    if dense:
        for n in mats:
            x[n] = torch.from_numpy(mats[n][feats["item_category"]]).to(device)
    model.build(device)
    tr = model.trainer(B)
    tr.forward_backward(x, [torch.from_numpy(y).to(device)])
    loss, z, g, got = _restate(model, tr, kind, feats, y, mats, dense)
    close(tr._loss_all[0], loss, 1e-5, "loss")
    close(tr.logits.view(-1)[:B], z, TOL, "logits")
    for k, v in got.items():
        close(v, g[k], TOL, k)
    # the inference forward (InputBlockV2.call: the in-place l2-norm, the operator's gather) on the same variables
    close(model(x).reshape(-1), 1.0 / (1.0 + np.exp(-z)), TOL, "inference predictions")


def test_ragged_last_batch_trains_the_projection(device):
    """A trainer compiled for 2048 samples trains a projected slot on a last batch of 1100: a size whose backward splits
    into more row chunks than 2048 does, so its workspace must be sized for every batch up to the compiled one."""
    mm.set_seed(12)
    rows = 512
    schema, mats, _ops = _setup((("pre_a", 768),), device, seed=8, rows=rows)
    model = _model("dcn", schema, 64, False)
    model.compile(optimizer="adagrad")
    model.build(device)
    tr = model.trainer(2048)
    for b in (2048, 1100, 1057, 1376):
        feats, y = _batch(b, device, b, rows=rows)
        tr.forward_backward(_dev(feats, device), [torch.from_numpy(y).to(device)])
        loss, z, g, got = _restate(model, tr, "dcn", feats, y, mats, False)
        close(tr._loss_all[0], loss, 1e-5, f"loss at b = {b}")
        for k in ("proj_pre_a/kernel", "proj_pre_a/bias"):
            close(got[k], g[k], TOL, f"{k} at b = {b}")
    # through fit: 2048 + 1100 samples in batches of 2048
    n = 2048 + 1100
    rng = np.random.default_rng(3)
    data = {"item_category": rng.integers(0, rows, n), "user_age": rng.random(n).astype(np.float32),
            "click": (rng.random(n) < 0.5).astype(np.int64)}
    loader = mm.Loader(data, batch_size=2048, schema=schema, device=device)
    hist = model.fit(loader, epochs=2)
    assert len(hist.history["loss"]) == 2 and all(np.isfinite(hist.history["loss"]))


def test_catalog_trainer_refuses_pretrained_features(device):
    schema, _, _ops = _setup((("pre_a", 12),), device)
    s = Schema(list(schema) + [ColumnSchema("next_item", tags=(Tags.TARGET,), dtype="int64",
                                            properties={"domain": {"min": 0, "max": ROWS - 1}})])
    emb = mm.Embeddings(s.select_by_tag(Tags.CATEGORICAL), dim=16)
    pe = mm.PretrainedEmbeddings(s.select_by_tag(Tags.EMBEDDING), output_dims=8)
    out = mm.CategoricalOutput(to_call=emb.tables["item_category"], target_name="next_item")
    model = mm.Model(mm.InputBlockV2(s, categorical=emb, pretrained_embeddings=pe), mm.MLPBlock([16]), out)
    model.compile(optimizer="adagrad")
    model.build(device)
    with pytest.raises(NotImplementedError, match="pretrained embeddings"):
        model.trainer(64)


def test_out_of_range_ids_without_tables_are_reported(device):
    """An input block whose only ids are a pretrained feature's lookup keys still reports out-of-range ids: eagerly, and
    from a CompiledForward's captured graph."""
    schema, _, _ops = _setup((("pre_a", 12),), device)
    ib = mm.InputBlockV2(schema, categorical=Tags.USER_ID, pretrained_embeddings=mm.PretrainedEmbeddings(
        schema.select_by_tag(Tags.EMBEDDING), output_dims=8))
    assert ib.embeddings is None
    model = mm.Model(ib, mm.MLPBlock([8]), mm.BinaryOutput("click"))
    feats, _ = _batch(64, device, 1)
    model(_dev(feats, device))
    bad = dict(feats, item_category=feats["item_category"].copy())
    bad["item_category"][5] = ROWS + 3
    with pytest.raises(IndexError):
        model(_dev(bad, device))
    cf = mm.CompiledForward(model, mm.HostBatch.like(feats))
    cf(mm.HostBatch.like(feats))
    with pytest.raises(IndexError):
        cf(mm.HostBatch.like(bad))


@pytest.mark.parametrize("kind", ["dcn", "mmoe"])
def test_eager_steps_equal_graph_replays(device, kind):
    batches = [_batch(128, device, s) for s in range(3)]

    def run(graph):
        mm.set_seed(5)
        schema, _, _ops = _setup((("pre_a", 24),), device, seed=2)
        model = _model(kind, schema, 16, True)
        model.compile(optimizer="adam")
        model.build(device)
        tr = model.trainer(128)
        losses = []
        for i, (f, y) in enumerate(batches):
            x, yt = _dev(f, device), torch.from_numpy(y).to(device)
            if graph:
                if i == 0:
                    tr.capture(x, [yt])
                losses.append(tr.replay(x, [yt])[0].clone())
            else:
                losses.append(tr.step(x, [yt])[0].clone())
        proj = model.body.input_block.pretrained.branches["pre_a"].projection
        return torch.stack(losses), proj.kernel.clone(), proj.bias.clone()

    eager, graph = run(False), run(True)
    # the dense backward kernels sum with float atomics, so the two engines agree to rounding, not bit for bit
    close(graph[0], eager[0].cpu().numpy(), 1e-5, "losses")
    close(graph[1], eager[1].cpu().numpy(), 2e-4, "projection kernel")
    close(graph[2], eager[2].cpu().numpy(), 2e-4, "projection bias")


def test_operator_path_bit_equal_to_dense_vectors(device):
    mm.set_seed(7)
    schema, mats, _ops = _setup((("pre_a", 36),), device, seed=4)
    model = _model("dcn", schema, 16, True)
    feats, y = _batch(300, device, 9)
    x = _dev(feats, device)
    xd = dict(x, pre_a=torch.from_numpy(mats["pre_a"][feats["item_category"]]).to(device))
    assert torch.equal(model(x), model(xd))
    unproj = _model("mlp", schema, None, False)
    assert torch.equal(unproj(x), unproj(xd))
    model.compile(optimizer="sgd")
    tr = model.trainer(300)
    yt = [torch.from_numpy(y).to(device)]
    tr.forward_backward(x, yt)
    want, logits = tr.arena.grad.clone(), tr.logits.clone()
    tr.arena.grad.zero_()
    tr.forward_backward(xd, yt)
    assert torch.equal(tr.logits, logits), "the training forward differs between the two paths"
    # the dense backward kernels sum with float atomics: equal to rounding
    close(tr.arena.grad, want.cpu().numpy(), 1e-5, "dense gradients")


def test_reference_dcn_configuration_fit_and_evaluate(device):
    """tests/unit/tf/models/test_ranking.py::test_dcn_model_with_pretrained_embeddings: Dp = 12, output_dims=16, depth 1,
    MLPBlock([2]), through fit and evaluate over a Loader with the EmbeddingOperator."""
    mm.set_seed(1)
    rng = np.random.default_rng(0)
    n = 200
    data = {"item_id": rng.integers(0, 30, n), "item_category": rng.integers(0, ROWS, n),
            "user_age": rng.random(n).astype(np.float32), "click": (rng.random(n) < 0.5).astype(np.int64)}
    schema = Schema([ColumnSchema("item_id", tags=(Tags.CATEGORICAL, Tags.ITEM_ID), dtype="int64",
                                  properties={"domain": {"min": 0, "max": 29}})] + list(_schema()))
    loader = mm.Loader(data, batch_size=10, schema=schema, device=device, transforms=[
        mm.EmbeddingOperator(rng.random((ROWS, 12)), lookup_key="item_category", embedding_name="pretrained_category_embeddings")])
    s = loader.output_schema
    pe = mm.PretrainedEmbeddings(s.select_by_tag(Tags.EMBEDDING), output_dims=16)
    ib = mm.InputBlockV2(s, pretrained_embeddings=pe)
    model = mm.DCNModel(s, input_block=ib, depth=1, deep_block=mm.MLPBlock([2]), stacked=True,
                        prediction_tasks=mm.BinaryOutput("click"))
    model.compile(optimizer="adam")
    hist = model.fit(loader, epochs=1)
    assert np.isfinite(hist.history["loss"][0])
    res = model.evaluate(loader, return_dict=True)
    assert np.isfinite(res["loss"])


def test_notebook_flow_on_parquet(device, tmp_path):
    """The entertainment notebook's flow: a parquet file, an EmbeddingOperator over movie vectors, PretrainedEmbeddings,
    DCNModel(depth=2, MLPBlock([64, 32])), adagrad, five epochs: the loss decreases."""
    import pandas as pd

    mm.set_seed(2)
    rng = np.random.default_rng(1)
    n, movies = 4096, 64
    vecs = rng.standard_normal((movies, 48)).astype(np.float32)
    movie = rng.integers(0, movies, n)
    user = rng.integers(0, 20, n)
    w = rng.standard_normal(48)
    rating = ((vecs[movie] @ w + 0.3 * rng.standard_normal(n)) > 0).astype(np.int64)
    pd.DataFrame({"movieId": movie, "userId": user, "rating_binary": rating}).to_parquet(tmp_path / "train.parquet")
    schema = Schema([
        ColumnSchema("movieId", tags=(Tags.CATEGORICAL, Tags.ITEM_ID), dtype="int64", properties={"domain": {"min": 0, "max": movies - 1}}),
        ColumnSchema("userId", tags=(Tags.CATEGORICAL, Tags.USER_ID), dtype="int64", properties={"domain": {"min": 0, "max": 19}}),
        ColumnSchema("rating_binary", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
    ])
    loader = mm.Loader(str(tmp_path / "train.parquet"), batch_size=1024, schema=schema, device=device, transforms=[
        mm.EmbeddingOperator(vecs, lookup_key="movieId", embedding_name="pretrained_movie_embeddings")])
    pretrained = mm.PretrainedEmbeddings(loader.output_schema.select_by_tag(Tags.EMBEDDING))
    embeddings_block = mm.Embeddings(loader.output_schema.select_by_tag(Tags.CATEGORICAL), dim=16)
    input_block = mm.InputBlockV2(loader.output_schema, categorical=embeddings_block, pretrained_embeddings=pretrained)
    model = mm.DCNModel(loader.output_schema, depth=2, input_block=input_block, deep_block=mm.MLPBlock([64, 32]),
                        prediction_tasks=mm.BinaryOutput("rating_binary"))
    model.compile(optimizer=mm.Adagrad(0.05))
    hist = model.fit(loader, epochs=5)
    losses = hist.history["loss"]
    assert losses[-1] < losses[0], losses


def test_save_load_and_compiled_forward(device, tmp_path):
    mm.set_seed(4)
    schema, mats, _ops = _setup((("pre_a", 40),), device, seed=6)
    model = _model("dcn", schema, 16, True)
    model.compile(optimizer="adagrad")
    feats, y = _batch(64, device, 1)
    x = _dev(feats, device)
    model.train_step((x, torch.from_numpy(y).to(device)))
    want = model(x).clone()
    model.save(tmp_path / "m")
    import json

    manifest = json.loads(next((tmp_path / "m").rglob("manifest.json")).read_text())
    stored = [e["shape"] for e in manifest["variables"]]
    assert [ROWS, 40] not in stored, "the pretrained matrix must not be saved"
    loaded = mm.io.load_model(tmp_path / "m", device=device)
    assert torch.equal(loaded(x), want)
    hb = mm.HostBatch.like(feats)
    cf = mm.CompiledForward(model, hb)
    got = cf(hb)
    assert torch.equal(got.reshape(-1).cpu(), want.reshape(-1).cpu())


def test_one_step_at_benchmark_size(device):
    mm.set_seed(8)
    B, rows = 65536, 4096
    schema, mats, _ops = _setup((("pre_a", 768),), device, seed=3, rows=rows)
    model = _model("dcn", schema, 64, False)
    model.compile(optimizer="adagrad")
    feats, y = _batch(B, device, 5, rows=rows)
    x = _dev(feats, device)
    model.build(device)
    tr = model.trainer(B)
    tr.forward_backward(x, [torch.from_numpy(y).to(device)])
    br = model.body.input_block.pretrained.branches["pre_a"]
    li = tr.arena.layers.index(br.projection)
    # dW of the projection against float64 over the slot's input gradient the trainer left in its addends
    ids = torch.from_numpy(feats["item_category"]).to(device).long()
    P = torch.from_numpy(mats["pre_a"]).to(device).double()
    c = tr.inp.cols["pre_a"]
    gsum = sum(t[:B, c:c + 64].double() for t in (tr.g, tr.p, tr.acc))
    close(tr.arena.view(tr.arena.grad, li, "kernel"), (P[ids].t() @ gsum).cpu().numpy(), 1e-4, "dW at B = 65 536")
    close(tr.arena.view(tr.arena.grad, li, "bias"), gsum.sum(0).cpu().numpy(), 1e-4, "db at B = 65 536")
    tr.apply_gradients()
    assert torch.isfinite(tr.loss).all()
