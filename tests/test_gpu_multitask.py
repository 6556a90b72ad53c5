"""Multi-output ranking models on the GPU: mm_heads_fwd_bwd and mm_mlp_tc_heads against float64 torch restatements,
OutputBlock models through the fused and unfused forward paths, and the multi-output training step.

Loss and gradient semantics (Keras): loss_h = sum_i sw_i l_h,i / B, total = sum_h lambda_h loss_h; BinaryOutput heads
use BCE on the logits, RegressionOutput heads (z - y)^2.
"""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200.blocks import last_dense_path, set_dense_engine
from models_b200.schema import ColumnSchema, Schema, Tags
from tests import helpers as H
from tests.multitask_oracle import heads_ref

pytestmark = pytest.mark.gpu
TOL = 3e-4
KINDS = {"b": "binary_crossentropy", "r": "mse"}


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))), 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def _targets(g, M, losses, dtypes, device):
    ys = []
    for h, l in enumerate(losses):
        dt = dtypes[h % len(dtypes)]
        if l == "binary_crossentropy":
            y = (torch.rand(M, generator=g) < 0.4)
        else:  # regression targets, some far from the prediction
            y = torch.randn(M, generator=g) * 3.0
            if dt in (torch.int32, torch.int64):
                y = y.round()
        ys.append(y.to(dt).to(device))
    return ys


@pytest.mark.parametrize("spec", ["b", "r", "br", "bbr", "brbrbrbr"])
@pytest.mark.parametrize("K", [1, 7, 32, 64, 256])
@pytest.mark.parametrize("M", [1, 37, 65536])
def test_heads_fwd_bwd_matches_float64(device, spec, K, M):
    g = torch.Generator().manual_seed(len(spec) * 1000 + K * 7 + M)
    H_ = len(spec)
    losses = [KINDS[c] for c in spec]
    ys = _targets(g, M, losses, [torch.int32, torch.int64, torch.float32, torch.float64], device)
    x = torch.randn((M, K), generator=g).to(device)
    W = (torch.randn((K, H_), generator=g) * 0.3).to(device)
    b = (torch.randn(H_, generator=g) * 0.1).to(device)
    shared = torch.rand(M, generator=g).to(device)
    per_head = [torch.rand(M, generator=g).to(device) if h % 2 == 0 else None for h in range(H_)]
    lws = [0.5 + 0.25 * h for h in range(H_)]
    for sw, mask in ((None, True), (shared, False), (per_head, True)):
        sws = sw if isinstance(sw, list) else [sw] * H_
        logits = torch.zeros((H_, M), device=device)
        loss = torch.zeros(1 + H_, device=device)
        dx = torch.full((M, K), 7.0, device=device)
        dW = torch.zeros((K, H_), device=device)
        db = torch.zeros(H_, device=device)
        ops.heads_fwd_bwd(x, W, b, losses, ys, logits, loss, dx, dW, db, loss_weights=lws, mask_relu=mask, sample_weight=sw)
        tot, per, z, rdx, rdW, rdb = heads_ref(x, W, b, losses, ys, sws, lws, mask)
        np.testing.assert_allclose(loss[0].item(), tot.item(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(loss[1:].cpu().numpy(), per.cpu().numpy(), rtol=1e-5, atol=1e-7)
        close(logits, z, 1e-5, "logits")
        close(dx, rdx, what="dx")
        close(dW, rdW, what="dW")
        close(db, rdb, what="db")


@pytest.mark.parametrize("K", [7, 32])
def test_heads_forward_only_touches_no_gradient_buffer(device, K):
    g = torch.Generator().manual_seed(K)
    M, losses = 1000, ["binary_crossentropy", "mse", "binary_crossentropy"]
    x = torch.randn((M, K), generator=g).to(device)
    W = torch.randn((K, 3), generator=g).to(device)
    b = torch.randn(3, generator=g).to(device)
    out = torch.zeros((3, M), device=device)
    ops.heads_fwd_bwd(x, W, b, losses, None, out)
    z = (x.double() @ W.double() + b.double()).t()
    want = torch.stack([torch.sigmoid(z[0]), z[1], torch.sigmoid(z[2])])
    close(out, want, 1e-5, "predictions")
    # the C entry with gradient buffers given but no targets must leave them untouched
    from models_b200 import _cabi
    import ctypes as C
    loss = torch.full((4,), 5.0, device=device)
    dx = torch.full((M, K), 5.0, device=device)
    dW = torch.full((K, 3), 5.0, device=device)
    db = torch.full((3,), 5.0, device=device)
    kinds = (C.c_int * 3)(0, 1, 0)
    _cabi.check(_cabi.load().mm_heads_fwd_bwd(x.data_ptr(), M, K, K, 3, W.data_ptr(), b.data_ptr(), kinds, None, None, None, None,
                                              out.data_ptr(), loss.data_ptr(), dx.data_ptr(), K, 1, dW.data_ptr(), db.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream), "mm_heads_fwd_bwd")
    torch.cuda.synchronize()
    for t in (loss, dx, dW, db):
        assert float(t.min()) == 5.0 and float(t.max()) == 5.0


@pytest.mark.parametrize("H_", [1, 2, 8])
@pytest.mark.parametrize("widths", [(128, 64, 32), (64, 16), (128, 64, 32, 8)])
def test_mlp_tc_heads_matches_float64(device, H_, widths):
    g = torch.Generator().manual_seed(H_ * 31 + len(widths))
    M, K = 3000, 415
    x = torch.randn((M, K), generator=g).to(device)
    layers, k = [], K
    for n in widths:
        layers.append(((torch.randn((k, n), generator=g) / k ** 0.5).to(device), (torch.randn(n, generator=g) * 0.1).to(device)))
        k = n
    W = (torch.randn((k, H_), generator=g) * 0.3).to(device)
    b = (torch.randn(H_, generator=g) * 0.1).to(device)
    acts = ["sigmoid" if h % 2 == 0 else "linear" for h in range(H_)]
    out = torch.zeros((H_, M), device=device)
    ops.mlp_tc_heads(ops.split_rows(x), K, [ops.split_weights(w) for w, _ in layers], list(widths), [bb for _, bb in layers],
                     ["relu"] * len(widths), W, b, acts, out)
    h = x.double()
    for w, bb in layers:
        h = torch.relu(h @ w.double() + bb.double())
    z = (h @ W.double() + b.double()).t()
    want = torch.stack([torch.sigmoid(z[i]) if a == "sigmoid" else z[i] for i, a in enumerate(acts)])
    close(out, want, 5e-5, "mlp_tc_heads")


# ---------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------
REGRESSION_TARGETS = ("rating", "dwell", "watch_time")  # the other target names are binary


def _mt_schema(cap=200, targets=("click", "conversion", "rating")):
    base = datasets.criteo_schema({k: min(v, cap) for k, v in datasets.CRITEO_MAX.items()})
    cols = [c for c in base if not c.has_tag(Tags.TARGET)]
    for t in targets:
        if t in REGRESSION_TARGETS:
            cols.append(ColumnSchema(t, tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32"))
        else:
            cols.append(ColumnSchema(t, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"))
    return Schema(cols)


def _batch(schema, B, seed):
    batch = datasets.generate_batch(schema.excluding_by_tag(Tags.TARGET), B, seed=seed, index_law="uniform")
    feats, _ = datasets.split_targets(schema.excluding_by_tag(Tags.TARGET), batch)
    rng = np.random.default_rng(seed)
    ys = {}
    for c in schema.select_by_tag(Tags.TARGET):
        ys[c.name] = (rng.random(B) * 5.0).astype(np.float32) if c.has_tag(Tags.REGRESSION) else (rng.random(B) < 0.3).astype(np.int64)
    return feats, ys


def _head_ref(model, x_last):
    """(H, B) float64 predictions of the model's heads on its last tower output."""
    W = model.prediction.to_call.kernel.double()
    b = model.prediction.to_call.bias.double()
    z = (x_last.double() @ W + b).t()
    return torch.stack([torch.sigmoid(z[h]) if a == "sigmoid" else z[h] for h, a in enumerate(model.prediction.activations)])


def _dlrm(schema, top=(64, 32), seed=3):
    mm.set_seed(seed)
    return mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([64, 64]), top_block=mm.MLPBlock(list(top)),
                        prediction_tasks=mm.OutputBlock(schema))


def _heads(model):
    """One oracle head dict per output (a (K, 1) column of the stacked kernel) and its activation."""
    W = H.to_numpy(model.prediction.to_call.kernel)
    b = H.to_numpy(model.prediction.to_call.bias)
    return [{"kernel": W[:, h:h + 1], "bias": b[h:h + 1], "activation": a} for h, a in enumerate(model.prediction.activations)]


def oracle_dlrm_outputs(model, feats):
    from oracle import oracle as O

    body = model.body
    tables, f2t = H.emb_tables(body.embeddings)
    return [O.dlrm_forward(feats, tables, f2t, body.continuous.features, H.mlp_layers(body.bottom_block),
                           H.mlp_layers(body.top_block), hd).reshape(-1) for hd in _heads(model)]


def oracle_dcn_outputs(model, feats):
    from oracle import oracle as O

    body = model.body
    tables, f2t = H.emb_tables(body.input_block.embeddings)
    cont = body.input_block.continuous.features if body.input_block.continuous is not None else []
    cross = [{"kernel": H.to_numpy(l.dense.kernel), "bias": None if l.dense.bias is None else H.to_numpy(l.dense.bias)}
             for l in body.cross.cross_layers]
    return [O.dcn_forward(feats, tables, f2t, cont, cross, H.mlp_layers(body.deep), hd, stacked=body.stacked,
                          branch_order=body.branch_order()).reshape(-1) for hd in _heads(model)]


@pytest.mark.parametrize("top", [(64, 32), (64, 48)])  # last width 32: fused heads (mm_mlp_tc_heads); 48: unfused
@pytest.mark.parametrize("engine", ["auto", "fp32"])
def test_dlrm_output_block_forward_matches_oracle(device, top, engine):
    schema = _mt_schema()
    model = _dlrm(schema, top)
    model.build(device)
    feats, _ = _batch(schema, 700, 5)
    set_dense_engine(engine)
    try:
        out = model(H.device_batch(feats, device))
        path = last_dense_path()
    finally:
        set_dense_engine("auto")
    assert list(out) == model.prediction.names == ["click/binary_output", "conversion/binary_output", "rating/regression_output"]
    if engine == "fp32":
        assert path == "fp32"
    elif top[-1] <= 32:
        assert path == "mlp_tc"  # the heads ran in the tower kernel's epilogue
    for n, want in zip(model.prediction.names, oracle_dlrm_outputs(model, feats)):
        assert tuple(out[n].shape) == (700, 1)
        assert H.rel_err(out[n].cpu().numpy().reshape(-1), want) < 2e-4, n
    assert model.output_schema().column_names == model.prediction.names


@pytest.mark.parametrize("stacked", [True, False])
def test_dcn_output_block_forward_matches_oracle(device, stacked):
    schema = _mt_schema(targets=("click", "rating"))
    mm.set_seed(4)
    model = mm.DCNModel(schema, depth=2, deep_block=mm.MLPBlock([64, 32]), stacked=stacked, embedding_dim=16,
                        prediction_tasks=mm.OutputBlock(schema))
    model.build(device)
    feats, _ = _batch(schema, 500, 6)
    out = model(H.device_batch(feats, device))
    for n, want in zip(model.prediction.names, oracle_dcn_outputs(model, feats)):
        assert H.rel_err(out[n].cpu().numpy().reshape(-1), want) < 2e-4, n


def _train_ref(model, tr, ys, lws):
    """Head loss and gradients restated in float64 on the trainer's saved last tower output."""
    x = tr.t[-1][:tr._b]
    losses = model.prediction.losses if hasattr(model.prediction, "losses") else [model.prediction.loss]
    W = model.prediction.to_call.kernel
    return heads_ref(x, W, model.prediction.to_call.bias, losses, ys, [None] * len(losses), lws,
                     model.body.top_block.dense_layers[-1].activation == "relu")


def test_train_step_multi_output_losses_and_head_gradients(device):
    schema = _mt_schema()
    model = _dlrm(schema)
    model.build(device)
    model.compile(optimizer=mm.SGD(0.0), loss_weights={"rating/regression_output": 0.25})
    feats, ys = _batch(schema, 512, 7)
    x = H.device_batch(feats, device)
    y = {k: torch.from_numpy(v).to(device) for k, v in ys.items()}
    tr = model.trainer(512)
    tr.forward_backward(x, [y[o.target] for o in model.output_blocks()])
    lws = [1.0, 1.0, 0.25]
    tot, per, _, _, rdW, rdb = _train_ref(model, tr, [y[o.target] for o in model.output_blocks()], lws)
    np.testing.assert_allclose(tr.loss[0].item(), tot.item(), rtol=1e-5)
    np.testing.assert_allclose(tr.loss[1:].cpu().numpy(), per.cpu().numpy(), rtol=1e-5)
    g = tr.gradients()
    hl = model.prediction.to_call
    close(g[f"{hl.name}/kernel"], rdW, what="dW heads")
    close(g[f"{hl.name}/bias"], rdb, what="db heads")
    tr.arena.grad.zero_()
    # train_step: step metrics per output (unweighted), a missing target names the column
    m = model.train_step((x, y))
    assert set(m) == {"loss", "loss_batch", "regularization_loss", "click/binary_output_loss",
                      "conversion/binary_output_loss", "rating/regression_output_loss"}
    np.testing.assert_allclose(m["rating/regression_output_loss"].item(), per[2].item(), rtol=1e-5)
    with pytest.raises(ValueError, match="conversion"):
        model.train_step((x, {k: v for k, v in y.items() if k != "conversion"}))


# up to 8 outputs, binary and regression mixed (sorted by name they interleave)
MANY_TARGETS = ("click", "rating", "conversion", "dwell", "like", "watch_time", "share", "follow")


@pytest.mark.parametrize("top", [(64, 32), (64, 48)])  # last width 32: fused heads (mm_mlp_tc_heads); 48: mm_heads_fwd_bwd
@pytest.mark.parametrize("n_out", [4, 5, 6, 7, 8])
def test_four_to_eight_outputs_forward_step_and_served_predictions(device, n_out, top):
    """A DLRM with 4..8 outputs: the forward per output against the oracle, through the kernel _LAST_HEADS names; one
    training step's total and per-output losses and the stacked head's kernel and bias gradients (per column) against
    float64 with unequal loss weights; and the model's forward on the step's batch against the activation of the
    trainer's logits, per output."""
    from models_b200.blocks import _LAST_HEADS

    schema = _mt_schema(targets=MANY_TARGETS[:n_out])
    model = _dlrm(schema, top, seed=40 + n_out)
    model.build(device)
    names = model.prediction.names
    assert len(names) == n_out and {KINDS[c] for c in "br"} == set(model.prediction.losses)
    B = 700
    feats, ys = _batch(schema, B, 50 + n_out)
    x = H.device_batch(feats, device)
    out = model(x)
    assert _LAST_HEADS[0] == ("mlp_tc" if top[-1] <= 32 else "heads")
    for n, want in zip(names, oracle_dlrm_outputs(model, feats)):
        assert tuple(out[n].shape) == (B, 1)
        assert H.rel_err(out[n].cpu().numpy().reshape(-1), want) < 2e-4, n
    lws = [0.25 + 0.25 * h for h in range(n_out)]
    model.compile(optimizer=mm.SGD(0.0), loss_weights=lws)
    yl = [torch.from_numpy(ys[o.target]).to(device) for o in model.output_blocks()]
    tr = model.trainer(B)
    tr.forward_backward(x, yl)
    tot, per, _, _, rdW, rdb = _train_ref(model, tr, yl, lws)
    np.testing.assert_allclose(tr.loss[0].item(), tot.item(), rtol=1e-5)
    np.testing.assert_allclose(tr.loss[1:].cpu().numpy(), per.cpu().numpy(), rtol=1e-5)
    g = tr.gradients()
    hl = model.prediction.to_call
    for h, n in enumerate(names):
        close(g[f"{hl.name}/kernel"][:, h], rdW[:, h], what=f"dW of {n}")
    close(g[f"{hl.name}/bias"], rdb, what="db")
    served = model(x)
    for h, (n, a) in enumerate(zip(names, model.prediction.activations)):
        zl = tr.logits[h].double()
        want = torch.sigmoid(zl) if a == "sigmoid" else zl
        assert H.rel_err(served[n].cpu().numpy().reshape(-1), want.cpu().numpy()) < 2e-4, n


def test_single_regression_output_forward_and_train(device):
    schema = _mt_schema(targets=("rating",))
    mm.set_seed(8)
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([64, 64]), top_block=mm.MLPBlock([64, 32]),
                         prediction_tasks=mm.RegressionOutput("rating"))
    model.build(device)
    feats, ys = _batch(schema, 400, 9)
    x = H.device_batch(feats, device)
    out = model(x)
    assert isinstance(out, torch.Tensor) and tuple(out.shape) == (400, 1)
    model.compile(optimizer=mm.Adagrad(0.05), loss="mse")
    y = torch.from_numpy(ys["rating"]).to(device)
    first = model.train_step((x, y))["loss"].item()
    want = float(((out.double().reshape(-1) - y.double()) ** 2).mean())
    np.testing.assert_allclose(first, want, rtol=1e-4)
    for _ in range(30):
        last = model.train_step((x, y))["loss"].item()
    assert last < first * 0.5, (first, last)


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_graph_replay_equals_eager_multi_output(device, opt):
    schema = _mt_schema()
    ma, mb = _dlrm(schema, seed=12), _dlrm(schema, seed=12)
    ma.build(device), mb.build(device)
    o = {"sgd": lambda: mm.SGD(0.5), "adagrad": lambda: mm.Adagrad(0.05), "adam": lambda: mm.Adam(0.01)}[opt]
    ma.compile(optimizer=o(), loss_weights=[1.0, 2.0, 0.5])
    mb.compile(optimizer=o(), loss_weights=[1.0, 2.0, 0.5])
    B = 256
    batches = []
    for s in range(3):
        f, ys = _batch(schema, B, 20 + s)
        batches.append((H.device_batch(f, device), [torch.from_numpy(ys[o_.target]).to(device) for o_ in ma.output_blocks()]))
    ta, tb = ma.trainer(B), mb.trainer(B)
    tb.capture(*batches[0])
    for x, y in batches:
        la = ta.step(x, y).clone()
        lb = tb.replay(x, y).clone()
        close(la, lb, 1e-5, "losses")
    for (na, va), (nb, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(va, vb, 1e-4, na)


def test_fit_multi_output_parquet(device, tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    rng = np.random.default_rng(0)
    n = 16000
    schema = _mt_schema(cap=50, targets=("click", "rating"))
    feats, _ = _batch(schema, n, 1)
    s1 = (feats["C1"] % 2 == 0).astype(np.float32) * 1.5 + feats["I1"].reshape(-1) * 2.0 - 1.0
    click = (rng.random(n) < 1 / (1 + np.exp(-3 * s1))).astype(np.int64)
    rating = ((feats["C2"] % 3).astype(np.float32) + feats["I2"].reshape(-1)).astype(np.float32)
    cols = {k: np.asarray(v).reshape(-1) for k, v in feats.items()}
    cols["click"], cols["rating"] = click, rating
    d = tmp_path / "data"
    d.mkdir()
    pq.write_table(pa.table(cols), d / "train.parquet")
    loader = mm.Loader(str(d), batch_size=2000, shuffle=True, schema=schema, device=device)
    mm.set_seed(5)
    # one binary target among several keeps a single BinaryOutput by default: ask for an output per target
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]),
                         prediction_tasks=mm.OutputBlock(schema))
    assert isinstance(model.prediction, mm.ParallelOutputs)
    model.compile(optimizer=mm.Adam(0.02))
    hist = model.fit(loader, epochs=6).history
    for k in ("loss", "click/binary_output_loss", "rating/regression_output_loss"):
        assert len(hist[k]) == 6 and hist[k][-1] < hist[k][0], (k, hist[k])


# ---------------------------------------------------------------------------------------------------------------
# the training step against the reference's torch backend and the restatement
# ---------------------------------------------------------------------------------------------------------------
GOLDEN = __import__("pathlib").Path(__file__).parent / "golden" / "multitask" / "ref_torch_dlrm_train_multitask.npz"


def test_train_step_matches_the_reference_torch_backend_multitask(device):
    """Loss, predictions and every gradient of ONE step of the reference's torch DLRMModel with its default output block
    over click / conversion (binary) and rating (regression) (tests/golden/make_golden_multitask.py), at 3e-4 of each
    tensor's scale.  The torch backend averages the per-output losses: loss_weights = 1/H reproduces it."""
    from tests import multitask_oracle as MT
    from tests.golden import replay

    z = replay.load(GOLDEN)
    dim = int(z["dim"])
    cols = [ColumnSchema(str(n), tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": int(mx), "name": str(n)}})
            for n, mx in zip(z["cat_names"], z["cat_max"])]
    cols += [ColumnSchema(str(n), tags=("continuous",), dtype="float32") for n in z["cont_names"]]
    for t, k in zip(z["target_names"], z["target_kinds"]):
        cols.append(ColumnSchema(str(t), tags=("target", "binary_classification" if str(k) == "binary" else "regression"),
                                 dtype="int64" if str(k) == "binary" else "float32"))
    schema = Schema(cols)
    model = mm.DLRMModel(schema, embedding_dim=dim, bottom_block=mm.MLPBlock([32, dim]), top_block=mm.MLPBlock([24, 8]),
                         prediction_tasks=mm.OutputBlock(schema))
    model.build(device)
    for name, t in model.body.embeddings.tables.items():
        t.table = torch.from_numpy(z[f"table_{name}"]).to(device).contiguous()
        t.built = True
    for blk, tag in ((model.body.bottom_block, "bottom"), (model.body.top_block, "top")):
        for l, w in zip(blk.dense_layers, replay.unpack_layers(z, tag)):
            l.set_weights(w["kernel"], w["bias"])
    heads = MT.golden_inputs(z)[6]
    assert [h["name"] for h in heads] == model.prediction.names
    # the per-output Keras names load_weights accepts: prediction/<output name>/dense/{kernel,bias}
    model.load_weights({f"prediction/{h['name']}/dense/{w}": h[w] for h in heads for w in ("kernel", "bias")},
                       name_map=lambda n: n, strict=False)
    H_ = len(heads)
    model.compile(optimizer=mm.SGD(0.0), loss_weights=[1.0 / H_] * H_)
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z if k.startswith("batch_")}
    ys = [torch.from_numpy(z[f"targets_{h['target']}"]).to(device) for h in heads]
    tr = model.trainer(len(ys[0]))
    tr.forward_backward(batch, ys)
    np.testing.assert_allclose(tr.loss[0].item(), float(z["loss"]), rtol=1e-5)
    for h, hd in enumerate(heads):
        zl = tr.logits[h].double()
        pred = torch.sigmoid(zl) if hd["loss"] == MT.BCE else zl
        np.testing.assert_allclose(pred.cpu().numpy(), z[f"out_{hd['target']}"].reshape(-1), rtol=2e-4, atol=2e-6)
    got = tr.gradients()
    layers = tr.arena.layers
    names = [("bottom", 0), ("bottom", 1), ("top", 0), ("top", 1)]
    for l, (tag, i) in zip(layers, names):
        close(got[f"{l.name}/kernel"], z[f"grad_{tag}_kernel_{i}"], what=f"{tag} kernel {i}")
        close(got[f"{l.name}/bias"], z[f"grad_{tag}_bias_{i}"], what=f"{tag} bias {i}")
    hl = layers[-1]
    for h, hd in enumerate(heads):
        close(got[f"{hl.name}/kernel"][:, h:h + 1], z[f"grad_head_{hd['target']}_kernel"], what=f"head {hd['name']} kernel")
        close(got[f"{hl.name}/bias"][h:h + 1], z[f"grad_head_{hd['target']}_bias"], what=f"head {hd['name']} bias")
    for t, f in enumerate(tr.feats):
        ids = ops.widen_index(tr._idx[t]).long()
        dense = torch.zeros(z[f"table_{f}"].shape, dtype=torch.float64, device=device)
        dense.index_add_(0, ids, tr._slices[t].double())
        close(dense, z[f"grad_table_{f}"], what=f"table {f}")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_match_the_restatement(device, opt):
    """Three optimizer steps of a click / conversion / rating DLRM with loss weights against autograd of the restated step
    (tests/multitask_oracle.py) + the Keras update rules in float64; every variable's UPDATE compared as in
    tests/test_gpu_train.py::test_training_steps_match_oracle (0.1 relative Frobenius, 0.5 of the largest element)."""
    from oracle import oracle_train
    from tests import multitask_oracle as MT

    schema = _mt_schema(cap=300)
    mm.set_seed(3)
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([64, 16]), top_block=mm.MLPBlock([64, 32]),
                         prediction_tasks=mm.OutputBlock(schema))
    model.build(device)
    lws = [1.0, 0.5, 0.2]
    tables, f2t = H.emb_tables(model.body.embeddings)
    st = dict(tables={k: v.astype(np.float64) for k, v in tables.items()}, bottom=H.mlp_layers(model.body.bottom_block),
              top=H.mlp_layers(model.body.top_block))
    W0, b0 = H.to_numpy(model.prediction.to_call.kernel).astype(np.float64), H.to_numpy(model.prediction.to_call.bias).astype(np.float64)
    heads = [{"name": n, "kernel": W0[:, h:h + 1].copy(), "bias": b0[h:h + 1].copy(), "loss": l}
             for h, (n, l) in enumerate(zip(model.prediction.names, model.prediction.losses))]

    def flat(m):
        t, _ = H.emb_tables(m.body.embeddings)
        out = [t[n] for n in sorted(t)]
        for blk in (m.body.bottom_block, m.body.top_block):
            for l in H.mlp_layers(blk):
                out += [l["kernel"], l["bias"]]
        return out + [H.to_numpy(m.prediction.to_call.kernel), H.to_numpy(m.prediction.to_call.bias)]

    before = [np.array(v, dtype=np.float64) for v in flat(model)]
    lr = {"sgd": 0.5, "adagrad": 0.05, "adam": 0.01}[opt]
    eps = 1e-6 if opt == "adam" else 1e-7
    model.compile(optimizer={"sgd": mm.SGD(lr), "adagrad": mm.Adagrad(lr), "adam": mm.Adam(lr, epsilon=eps)}[opt], loss_weights=lws)

    def slots(shape):
        if opt == "adagrad":
            return {"a": np.full(shape, 0.1)}
        return {"m": np.zeros(shape), "v": np.zeros(shape)} if opt == "adam" else {}

    tslots = {n: slots(t.shape) for n, t in st["tables"].items()}
    dslots = {}
    B = 300
    for step in (1, 2, 3):
        feats, ys = _batch(schema, B, 100 + step)
        y_dev = {k: torch.from_numpy(v).to(device) for k, v in ys.items()}
        m = model.train_step((H.device_batch(feats, device), y_dev))
        targets = [ys[n.split("/")[0]] for n in model.prediction.names]
        loss, per, _, grads = MT.dlrm_multitask_loss_and_grads(feats, st["tables"], f2t, model.body.continuous.features,
                                                               st["bottom"], st["top"], heads, targets, loss_weights=lws)
        np.testing.assert_allclose(m["loss"].item(), loss, rtol=1e-4)
        for h, n in enumerate(model.prediction.names):
            np.testing.assert_allclose(m[f"{n}_loss"].item(), per[h], rtol=1e-4)
        kw = dict(beta_1=0.9, beta_2=0.999, epsilon=eps, step=step)
        for f, tname in f2t.items():
            uniq = np.unique(np.asarray(feats[f]).reshape(-1))
            st["tables"][tname] = oracle_train.sparse_update(opt, st["tables"][tname], uniq, grads[f"table/{tname}"][uniq], tslots[tname], lr, **kw)
        for tag in ("bottom", "top"):
            for i, l in enumerate(st[tag]):
                for what in ("kernel", "bias"):
                    key = f"{tag}/{what}_{i}"
                    dslots.setdefault(key, slots(l[what].shape))
                    l[what] = oracle_train.dense_update(opt, l[what], grads[key], dslots[key], lr, **kw)
        for hd in heads:
            for what in ("kernel", "bias"):
                key = f"head/{hd['name']}/{what}"
                dslots.setdefault(key, slots(hd[what].shape))
                hd[what] = oracle_train.dense_update(opt, hd[what], grads[key], dslots[key], lr, **kw)
    want = [st["tables"][n] for n in sorted(st["tables"])]
    for tag in ("bottom", "top"):
        for l in st[tag]:
            want += [l["kernel"], l["bias"]]
    want += [np.concatenate([hd["kernel"] for hd in heads], axis=1), np.concatenate([hd["bias"] for hd in heads])]
    after = flat(model)
    assert len(after) == len(want) == len(before)
    for i, (a, w, b0_) in enumerate(zip(after, want, before)):
        upd_ref = np.asarray(w, dtype=np.float64) - b0_
        assert np.max(np.abs(upd_ref)) > 0, i
        upd = np.asarray(a, dtype=np.float64) - b0_
        fro = float(np.linalg.norm(upd - upd_ref) / np.linalg.norm(upd_ref))
        assert fro < 0.1, f"update of variable {i} after 3 {opt} steps: relative Frobenius error {fro:.3e}"
        close(upd, upd_ref, 0.5, f"update of variable {i} after 3 {opt} steps")


def test_save_load_round_trip_and_compiled_forward(device, tmp_path):
    from models_b200.graph import HostBatch

    schema = _mt_schema()
    model = _dlrm(schema, seed=31)
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.05))
    feats, ys = _batch(schema, 256, 3)
    x = H.device_batch(feats, device)
    model.train_step((x, {k: torch.from_numpy(v).to(device) for k, v in ys.items()}))  # the heads live in the arena now
    eager = {k: v.clone() for k, v in model(x).items()}
    # variables named per output, each a (K, 1) / (1,) column of the stacked head
    sd = model.state_dict()
    W = H.to_numpy(model.prediction.to_call.kernel)
    for h, n in enumerate(model.prediction.names):
        np.testing.assert_array_equal(sd[f"prediction/{n}/dense/kernel"], W[:, h:h + 1])
    model.save(tmp_path / "export")
    loaded = mm.Model.load(tmp_path / "export")
    got = loaded(x)
    assert list(got) == list(eager)
    for n in eager:
        assert torch.equal(got[n], eager[n]), n
    # load_weights from the export's per-output names lands in the right columns
    fresh = _dlrm(schema, seed=77)
    fresh.build(device)
    names = dict(zip(fresh.weights(), model.weights()))  # auto layer names differ between two models; order does not
    fresh.load_weights(tmp_path / "export", name_map=names)
    for n, v in fresh(x).items():
        assert torch.equal(v, eager[n]), n
    # CUDA-graph forward: one pinned (H, B) buffer, one D2H copy, a dict of host views equal to the eager outputs
    hb = HostBatch.like(feats, model.input_columns())
    cf = model.compile(hb)
    res = cf(hb)
    assert list(res) == list(eager) and cf.output.shape == (3, 256)
    for n in eager:
        assert torch.equal(res[n], eager[n].cpu()), n
    pf = model.pipeline(hb, depth=2)
    k = pf.submit(hb)
    res = pf.result(k)
    for n in eager:
        assert torch.equal(res[n], eager[n].cpu()), n
