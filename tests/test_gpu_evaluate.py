"""Ranking-model evaluation on the GPU: mm_metrics_update against the NumPy restatement (tests/metrics_oracle.py),
the logits forward of every ranking path against `model(inputs)`, `evaluate` and `fit(validation_data=...)`."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops
from models_b200 import metrics as M
from tests import helpers as H
from tests import metrics_oracle as O

pytestmark = pytest.mark.gpu
KINDS = {"b": "binary_crossentropy", "r": "mse"}
DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]


def gpu_sigmoid(z: torch.Tensor, form: int) -> torch.Tensor:
    """The sigmoid of the forward kernels on z (H, M): mm_heads_fwd_bwd forward-only (PRED_HEAD) on an identity head, or
    mm_dense_fp32's activation epilogue (PRED_ACT) on a 1x1 identity layer.  Both compute z * 1 + 0 = z exactly first."""
    Hh, Mm = z.shape
    if form == _cabi.PRED_HEAD:
        out = torch.empty_like(z)
        eye = torch.eye(Hh, device=z.device)
        x = torch.empty((Mm, Hh), device=z.device).copy_(z.t())  # fresh (Hh, 1) strides, also for Mm = 1
        return ops.heads_fwd_bwd(x, eye, torch.zeros(Hh, device=z.device), ["binary_crossentropy"] * Hh, None, out)
    one = torch.ones((1, 1), device=z.device)
    return torch.stack([ops.dense_fp32(z[h].reshape(-1, 1).contiguous(), one, None, "sigmoid",
                                       torch.empty((Mm, 1), device=z.device)).reshape(-1) for h in range(Hh)])


def _kernel_case(spec, M_, seed, device, weighted, logit_fn=None):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn((len(spec), M_), generator=g) * 2.0)
    if logit_fn is not None:
        z = logit_fn(z)
    z = z.to(device).contiguous()
    ys, sws, mws = [], [], []
    for h, c in enumerate(spec):
        dt = DTYPES[h % 4]
        y = (torch.rand(M_, generator=g) < 0.4).float() if c == "b" else torch.randn(M_, generator=g) * 2
        if c == "r" and dt in (torch.int32, torch.int64):
            y = y.round()
        ys.append(y.to(dt).to(device))
        sws.append(torch.rand(M_, generator=g).to(device) if weighted else None)
        mws.append(torch.rand(M_, generator=g).to(device) if weighted else None)
    return z, ys, sws, mws


def _run(z, spec, ys, sws, mws, T, form, thresholds):
    Hh = len(spec)
    sets = [[None] * Hh] + ([mws] if mws[0] is not None else [])
    state = torch.zeros((Hh, _cabi.METRICS_SCALARS + 4 * T), dtype=torch.float64, device=z.device)
    ws = torch.empty(max(ops.metrics_workspace_bytes(z.shape[1], Hh), 1), dtype=torch.uint8, device=z.device)
    ops.metrics_update(z, [KINDS[c] for c in spec], ys, state, ws, T, [form] * Hh, thresholds, sample_weight=sws, metric_weights=sets)
    return state.cpu().numpy()


def _oracle(z, spec, ys, sws, mws, T, form, thresholds):
    p = gpu_sigmoid(z, form).cpu().numpy()
    zn = z.cpu().numpy()
    heads = [(KINDS[c], p[h], zn[h], ys[h].double().cpu().numpy(), None if sws[h] is None else sws[h].cpu().numpy(),
              None if mws[h] is None else mws[h].cpu().numpy()) for h, c in enumerate(spec)]
    return O.state(heads, T, 2 if mws[0] is not None else 1, thresholds)


def _compare(got, want, spec, T, weighted):
    C = _cabi
    for h, c in enumerate(spec):
        np.testing.assert_allclose(got[h, C.METRICS_LOSS], want[h, C.METRICS_LOSS], rtol=1e-6, atol=1e-9)
        assert got[h, C.METRICS_COUNT] == want[h, C.METRICS_COUNT] and got[h, C.METRICS_INVALID] == 0
        # set 0 is unweighted: counts, bit for bit (squared errors are fp64 sums: 1e-12)
        s0 = slice(C.METRICS_SET0, C.METRICS_SET0 + C.METRICS_SET_STRIDE)
        if c == "b":
            np.testing.assert_array_equal(got[h, s0], want[h, s0])
            np.testing.assert_array_equal(got[h, C.METRICS_SCALARS:C.METRICS_SCALARS + 2 * T],
                                          want[h, C.METRICS_SCALARS:C.METRICS_SCALARS + 2 * T])
            assert abs(M.auc_from_histogram(got[h, C.METRICS_SCALARS:C.METRICS_SCALARS + T],
                                            got[h, C.METRICS_SCALARS + T:C.METRICS_SCALARS + 2 * T])
                       - O.auc(want[h, C.METRICS_SCALARS:C.METRICS_SCALARS + T],
                               want[h, C.METRICS_SCALARS + T:C.METRICS_SCALARS + 2 * T])) < 1e-9
        else:
            np.testing.assert_allclose(got[h, s0], want[h, s0], rtol=1e-12, atol=0)
        if weighted:
            s1 = slice(C.METRICS_SET0 + C.METRICS_SET_STRIDE, C.METRICS_SET0 + 2 * C.METRICS_SET_STRIDE)
            np.testing.assert_allclose(got[h, s1], want[h, s1], rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(got[h, C.METRICS_SCALARS + 2 * T:], want[h, C.METRICS_SCALARS + 2 * T:], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("spec", ["b", "brb", "bbrbbrbb"])
@pytest.mark.parametrize("M_", [1, 37, 65536, 65536 + 37])
@pytest.mark.parametrize("T", [200, 1024])
@pytest.mark.parametrize("weighted", [False, True])
def test_metrics_update_matches_oracle(device, spec, M_, T, weighted):
    z, ys, sws, mws = _kernel_case(spec, M_, M_ + T + len(spec), device, weighted)
    form = _cabi.PRED_HEAD if (M_ + T) % 2 else _cabi.PRED_ACT
    thr = [[0.5, 0.3, 0.9, 0.0] if c == "b" else [] for c in spec]
    got = _run(z, spec, ys, sws, mws, T, form, thr)
    _compare(got, _oracle(z, spec, ys, sws, mws, T, form, thr), spec, T, weighted)


def _edge_logits(T, form, device):
    """fp32 logits whose sigmoid (as the kernel computes it) lands on or next to the bucket edges j/(T-1), plus z = 0."""
    j = np.arange(1, T - 1)
    base = np.log(j / (T - 1)) - np.log1p(-j / (T - 1))
    near = [base.astype(np.float32)]
    for _ in range(4):  # 4 fp32 neighbours on each side
        near = [np.nextafter(near[0], np.float32(-np.inf))] + near + [np.nextafter(near[-1], np.float32(np.inf))]
    z = np.concatenate(near + [np.zeros(64, np.float32)])
    zt = torch.from_numpy(z.astype(np.float32)).to(device).reshape(1, -1)
    p = gpu_sigmoid(zt, form)
    assert (p[0, -64:] == 0.5).all()  # z = 0 gives p = 0.5 exactly
    edges = torch.from_numpy((j / (T - 1)).astype(np.float32)).to(device)
    assert torch.isin(p, edges).any(), "no prediction found exactly on a bucket edge"
    return zt


@pytest.mark.parametrize("T", [200, 1024])
@pytest.mark.parametrize("form", [_cabi.PRED_ACT, _cabi.PRED_HEAD])
def test_bucket_edges_zero_logits_and_one_hot_bucket(device, T, form):
    z = _edge_logits(T, form, device)
    g = torch.Generator().manual_seed(T)
    y = [(torch.rand(z.shape[1], generator=g) < 0.5).to(torch.int64).to(device)]
    thr = [[0.5]]
    got = _run(z, "b", y, [None], [None], T, form, thr)
    _compare(got, _oracle(z, "b", y, [None], [None], T, form, thr), "b", T, False)
    # contention: 65 573 predictions in one bucket, weighted and not
    zc = torch.full((1, 65536 + 37), 1.3, device=device)
    yc = [(torch.rand(zc.shape[1], generator=g) < 0.5).float().to(device)]
    w = [torch.rand(zc.shape[1], generator=g).to(device)]
    got = _run(zc, "b", yc, w, w, T, form, thr)
    assert np.count_nonzero(got[0, _cabi.METRICS_SCALARS:]) == 4  # [pos | neg] of one bucket, in both metric sets
    _compare(got, _oracle(zc, "b", yc, w, w, T, form, thr), "b", T, True)


def test_two_runs_are_bit_identical(device):
    z, ys, sws, mws = _kernel_case("bbr", 65536 + 37, 5, device, False)
    thr = [[0.5], [0.5], []]
    a = _run(z, "bbr", ys, sws, mws, 200, _cabi.PRED_ACT, thr)
    b = _run(z, "bbr", ys, sws, mws, 200, _cabi.PRED_ACT, thr)
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("bad", ["target", "nan"])
def test_invalid_samples_raise(device, bad):
    spec = M.MetricsSpec([mm.BinaryOutput("click")], [1.0])
    st = M.MetricsState(spec, device)
    z = torch.randn((1, 100), device=device)
    y = (torch.rand(100, device=device) < 0.5).float()
    if bad == "target":
        y[7] = 0.3
    else:
        z[0, 9] = float("nan")
    st.update(z, [y], _cabi.PRED_ACT)
    with pytest.raises(ValueError, match="click/binary_output"):
        st.result()


# ---------------------------------------------------------------------------------------------------------------
# through the models
# ---------------------------------------------------------------------------------------------------------------
def _dlrm_onehot():
    from tests.test_gpu_train_dcn import _batch, _schema

    mm.set_seed(3)
    model = mm.DLRMModel(_schema(), embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    return model, lambda B, s: _batch(B, s)


def _dlrm_ragged():
    from tests.test_gpu_train_multihot import _batch, _model

    feats = [("C1", 300, "onehot", None), ("tags", 50, "ragged", "mean")]
    _, model = _model(torch.device("cuda", 0), feats, 16)
    return model, lambda B, s: (lambda f, y: (f, y.astype(np.int64)))(*_batch(feats, B, s))


def _dcn(stacked, deep=(32, 16)):
    from tests.test_gpu_train_dcn import _batch, _dcn as make

    return lambda: (make(stacked=stacked, deep=deep), lambda B, s: _batch(B, s))


def _deepfm():
    from tests.test_gpu_train_deepfm import _batch, _deepfm as make

    return make(), lambda B, s: _batch(B, s)


def _multi():
    from tests.test_gpu_train_dcn import _batch, _schema

    schema = _schema(("click", "like", "rating"))
    mm.set_seed(5)
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]),
                         prediction_tasks=mm.OutputBlock(schema))

    def batch(B, s):
        f, y = _batch(B, s)
        g = np.random.default_rng(s + 1)
        return f, {"click": y, "like": (g.random(B) < 0.3).astype(np.int64), "rating": g.standard_normal(B).astype(np.float32)}

    return model, batch


# deep towers with a first layer wider than 128 units leave the whole-tower kernel: layer by layer on mm_dense_tc, the
# output layer either fused into the last layer's epilogue (mm_dense_tc_head, last width <= 32) or a layer of its own
MODELS = {"dlrm": _dlrm_onehot, "dlrm_ragged": _dlrm_ragged, "dcn_stacked": _dcn(True), "dcn_parallel": _dcn(False),
          "dcn_dense_tc_head": _dcn(True, (256, 32)), "dcn_dense_tc": _dcn(True, (256, 64)), "deepfm": _deepfm, "multi": _multi}


def _device_batches(make_batch, device, sizes=(1000, 1000, 337)):
    out = []
    for i, B in enumerate(sizes):
        f, y = make_batch(B, 100 + i)
        yd = {k: torch.from_numpy(np.asarray(v)).to(device) for k, v in y.items()} if isinstance(y, dict) else torch.from_numpy(y).to(device)
        sw = torch.rand(B, generator=torch.Generator().manual_seed(i)).to(device)
        out.append((H.device_batch(f, device), yd, sw))
    return out


@pytest.fixture(params=["auto", "fp32"])
def engine(request):
    mm.set_dense_engine(request.param)
    yield request.param
    mm.set_dense_engine("auto")


@pytest.mark.parametrize("name", list(MODELS))
def test_evaluate_matches_oracle_on_the_model_predictions(device, engine, name):
    model, make_batch = MODELS[name]()
    model.build(device)
    model.compile(optimizer="adam", weighted_metrics=["auc", "binary_accuracy"] if name != "multi" else None)
    batches = _device_batches(make_batch, device)
    outs = model.output_blocks()
    per_batch = []
    for x, y, sw in batches:
        pred = model(x)
        z, form = model.logits(x)
        preds = [pred[o.name] for o in outs] if isinstance(pred, dict) else [pred]
        for h, o in enumerate(outs):
            if o.loss == "binary_crossentropy":  # the metric's sigmoid is the forward's, bit for bit
                assert torch.equal(gpu_sigmoid(z[h:h + 1].contiguous(), form).reshape(-1), preds[h].reshape(-1)), o.name
            else:
                assert torch.equal(z[h], preds[h].reshape(-1)), o.name
        ys = model._targets_by_output(y)
        per_batch.append([(o.loss, preds[h].reshape(-1).cpu().numpy(), z[h].cpu().numpy(), ys[h].double().cpu().numpy(),
                           sw.cpu().numpy()) for h, o in enumerate(outs)])
    weights = {k: v.clone() for k, v in model.weights().items() if v is not None}
    from models_b200.core import weights_version

    wv = weights_version()
    got = model.evaluate(batches, return_dict=True)
    assert weights_version() == wv
    for k, v in weights.items():
        assert torch.equal(model.weights()[k], v), k
    want = O.evaluate([o.name for o in outs], per_batch, weighted=name != "multi")
    if name != "multi":
        for k in ("weighted_precision", "weighted_recall"):
            want.pop(k)
    assert set(got) == set(want) == set(model.metrics_names)
    for k in want:
        tol = 1e-6 if "loss" in k else 1e-9
        assert abs(got[k] - want[k]) <= tol * max(1.0, abs(want[k])), (k, got[k], want[k])
    # a second pass gives the same dict; weighted AUC buckets are fp64 atomics: the last bits may move
    again = model.evaluate(batches, return_dict=True)
    assert {k: v for k, v in again.items() if not k.startswith("weighted_")} == {k: v for k, v in got.items() if not k.startswith("weighted_")}
    assert all(abs(again[k] - got[k]) < 1e-12 for k in got)
    assert len(model.evaluate(batches)) == len(model.metrics_names)
    # the two full-size batches replayed the captured step; the ragged model's batches cannot be replayed
    assert (getattr(model, "_eval_graph", None) is None) == (name == "dlrm_ragged")
    from models_b200 import models as models_module

    models_module._EVAL_GRAPH[0] = False
    try:
        eager = model.evaluate(batches, return_dict=True)
    finally:
        models_module._EVAL_GRAPH[0] = True
    # the graph path equals the eager path bit for bit (weighted AUC buckets: fp64 atomics)
    assert {k: v for k, v in eager.items() if not k.startswith("weighted_")} == {k: v for k, v in got.items() if not k.startswith("weighted_")}
    assert all(abs(eager[k] - got[k]) < 1e-12 for k in got)


def test_evaluate_graph_state_equals_eager_state_bitwise(device):
    model, make_batch = _multi()
    model.build(device)
    model.compile(optimizer="adam")
    batches = _device_batches(make_batch, device, sizes=(2048, 2048, 2048, 500))
    from models_b200 import models as models_module

    states = []
    for graph in (True, False):
        models_module._EVAL_GRAPH[0] = graph
        try:
            model.evaluate(batches)
        finally:
            models_module._EVAL_GRAPH[0] = True
        states.append(model._eval_state.state.clone())
    assert model._eval_graph is not None and model._eval_graph.launches_per_replay > 0
    assert torch.equal(states[0], states[1])
    # steps=k takes k batches from the iterator, no more
    it = iter(batches)
    model.evaluate(it, steps=2)
    assert next(it) is batches[2]


def test_fit_validation_and_training_metrics(device):
    from tests.test_gpu_train_dcn import _batch, _schema

    mm.set_seed(11)
    model = mm.DLRMModel(_schema(), embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    model.build(device)

    def planted(B, s):
        f, _ = _batch(B, s)
        y = ((f["C1"] % 2 == 0) | (f["C7"] == 3)).astype(np.int64)  # a rule of two categorical features
        return H.device_batch(f, device), torch.from_numpy(y).to(device)

    train = [planted(2048, s) for s in range(8)]
    valid = [planted(2048, 100 + s) for s in range(2)] + [planted(300, 200)]
    model.compile(optimizer=mm.Adam(0.01))
    hist = model.fit(train, epochs=4, validation_data=valid, train_metrics_steps=3).history
    assert hist["val_auc"][-1] > 0.9 and hist["val_auc"][-1] > hist["val_auc"][0]
    assert len(hist["auc"]) == len(hist["loss"]) == 4
    last = model.evaluate(valid, return_dict=True)
    assert {k: v[-1] for k, v in hist.items() if k.startswith("val_")} == {f"val_{k}": v for k, v in last.items()}
    assert set(model.fit(train, epochs=1, train_metrics_steps=0).history) == {"loss"}  # without metrics: what fit reported before
    with pytest.raises(ValueError, match="validation_freq"):
        model.fit(train, epochs=1, validation_data=valid, validation_freq=0)


def test_training_metrics_leave_the_loss_history_alone(device):
    """The same model from the same seed, trained with and without training metrics: the same losses (the training step's
    weight-gradient reductions end in atomics, so agreement is to fp32 rounding, not bit for bit)."""
    from tests.test_gpu_train_dcn import _batch, _schema

    hists = []
    for every in (1, 0):
        mm.set_seed(21)
        model = mm.DLRMModel(_schema(), embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
        model.build(device)
        model.compile(optimizer="adagrad")
        data = []
        for s in range(6):
            f, y = _batch(1024, s)
            data.append((H.device_batch(f, device), torch.from_numpy(y).to(device)))
        hists.append(model.fit(data, epochs=2, train_metrics_steps=every).history)
    assert set(hists[0]) == {"loss", "precision", "recall", "binary_accuracy", "auc"} and set(hists[1]) == {"loss"}
    np.testing.assert_allclose(hists[0]["loss"], hists[1]["loss"], rtol=1e-5)


def test_training_metrics_match_oracle_over_the_step_logits(device):
    from tests.test_gpu_train_dcn import _batch, _schema

    mm.set_seed(12)
    model = mm.DLRMModel(_schema(), embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    model.build(device)
    model.compile(optimizer="adagrad")
    data = []
    for s in range(5):
        f, y = _batch(1024 if s < 4 else 500, s)
        data.append((H.device_batch(f, device), torch.from_numpy(y).to(device)))
    logits, hist = [], None

    class Recording(list):
        def __iter__(self_):
            for i, b in enumerate(data):
                yield b
                if i % 2 == 0:  # train_metrics_steps=2: batches 0, 2, 4
                    n = b[1].numel()
                    logits.append((model._trainer.logits.view(-1)[:n].clone(), b[1].clone()))

    hist = model.fit(Recording(), epochs=1, train_metrics_steps=2).history
    z = torch.cat([l for l, _ in logits]).reshape(1, -1).contiguous()
    y = torch.cat([t for _, t in logits]).cpu().numpy()
    p = gpu_sigmoid(z, _cabi.PRED_HEAD).reshape(-1).cpu().numpy()
    want = O.head_metrics("binary_crossentropy", p, z.reshape(-1).cpu().numpy(), y)
    for k, v in want.items():
        assert abs(hist[k][0] - v) < 1e-9, k


def test_evaluate_leaves_a_captured_training_graph_alone(device):
    from tests.test_gpu_train_dcn import _batch, _schema

    mm.set_seed(13)
    model = mm.DLRMModel(_schema(), embedding_dim=16, bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([32, 16]))
    model.build(device)
    model.compile(optimizer="adam")
    f, y = _batch(1024, 1)
    x, yt = H.device_batch(f, device), torch.from_numpy(y).to(device)
    tr = model.trainer(1024)
    tr.capture(x, yt)
    n = tr.launches_per_step
    snap = tr._snapshot()
    model.evaluate([(x, yt)])
    for k in ("w", "s1", "s2", "hyper"):
        if snap[k] is not None:
            assert torch.equal(snap[k], tr._snapshot()[k]), k
    tr.replay(x, yt)
    assert tr.launches_per_step == n
