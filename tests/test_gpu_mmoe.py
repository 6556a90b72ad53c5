"""The multi-task Model(InputBlockV2, [MLPBlock], [MMOEBlock], output) on the GPU: mm_mmoe_heads_fwd_bwd against float64,
then MMoETrainer against the restatement (tests/mmoe_oracle.py), graph replay, the forward, evaluate, fit, save / load and
the compiled forward.  Tolerances: max |diff| / max |ref| per tensor, as tests/test_gpu_multitask.py."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from models_b200.graph import HostBatch
from tests import helpers as H
from tests.mmoe_oracle import BCE, MSE, gate_mix, heads_loss, mmoe_loss_and_grads, model_arrays
from tests.test_mmoe_host import mmoe_model, schema

pytestmark = pytest.mark.gpu
TOL = 3e-4


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale if ref.size else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


# ---------------------------------------------------------------------------------------------------------------
# mm_mmoe_heads_fwd_bwd against float64
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,E,U,Hn,T,sw,relu", [
    (65536, 4, 64, 3, 1.0, False, True),   # the benchmark shape
    (65536, 4, 64, 3, 1.0, True, False),
    (4099, 16, 256, 8, 0.5, True, True),   # the limits, B not a multiple of the 8-sample CTA tile
    (1001, 16, 256, 1, 2.0, False, True),
    (37, 3, 7, 2, 1.7, True, True),
])
def test_mmoe_heads_kernel_matches_float64(device, B, E, U, Hn, T, sw, relu):
    g = torch.Generator().manual_seed(B + 7 * E + U + Hn)
    losses = [(BCE, MSE)[t % 2] for t in range(Hn)]
    X = torch.randn((B, E * U), generator=g)
    if relu:
        X = X.clamp_min(0)
    L = torch.randn((B, Hn * E), generator=g) * 2
    W = torch.randn((U, Hn), generator=g) * 0.2
    b = torch.randn(Hn, generator=g) * 0.1
    ys = [(torch.rand(B, generator=g) < 0.4).to(torch.int64) if l == BCE else torch.randn(B, generator=g) for l in losses]
    sws = [torch.rand(B, generator=g) if (sw and t % 2 == 0) else None for t in range(Hn)]
    lws = [0.5 + 0.25 * t for t in range(Hn)]
    # float64 restatement
    Xd, Ld, Wd, bd = (t.double().clone().requires_grad_(True) for t in (X, L, W, b))
    zs = [gate_mix(Xd, Ld[:, t * E:(t + 1) * E], E, T) @ Wd[:, t] + bd[t] for t in range(Hn)]
    total, per = heads_loss(zs, losses, [y.numpy() for y in ys], lws, [None if s is None else s.numpy() for s in sws])
    total.backward()
    dX_ref = Xd.grad * (X > 0) if relu else Xd.grad
    dev = device
    Xg, Lg, Wg, bg = X.to(dev), L.to(dev), W.to(dev), b.to(dev)
    out = torch.zeros((Hn, B), device=dev)
    loss = torch.zeros(1 + Hn, device=dev)
    dX = torch.full((B, E * U), float("nan"), device=dev)
    dL = torch.full((B, Hn * E), float("nan"), device=dev)
    dW, db = torch.zeros((U, Hn), device=dev), torch.zeros(Hn, device=dev)
    gl = lambda M: [M[:, t * E:(t + 1) * E] for t in range(Hn)]
    ops.mmoe_heads_fwd_bwd(Xg, E, gl(Lg), T, Wg, bg, losses, [y.to(dev) for y in ys], out, loss, dx=dX, d_gate_logits=gl(dL),
                           dw=dW, db=db, loss_weights=lws, mask_relu=relu,
                           sample_weight=[None if s is None else s.to(dev) for s in sws])
    close(out, torch.stack([z.detach() for z in zs]), TOL, "logits")
    close(loss[0], total.detach(), 1e-5, "total loss")
    close(loss[1:], torch.stack([p.detach() for p in per]), 1e-5, "per-task losses")
    close(dX, dX_ref, TOL, "dX")
    close(dL, Ld.grad, TOL, "dL")
    close(dW, Wd.grad, TOL, "dW")
    close(db, bd.grad, TOL, "db")
    # forward only (null targets): the activated predictions
    pred = torch.zeros((Hn, B), device=dev)
    ops.mmoe_heads_fwd_bwd(Xg, E, gl(Lg), T, Wg, bg, losses, None, pred)
    ref = torch.stack([torch.sigmoid(z.detach()) if l == BCE else z.detach() for z, l in zip(zs, losses)])
    close(pred, ref, TOL, "predictions")


def test_mmoe_heads_kernel_argument_checks(device):
    X = torch.zeros((8, 12), device=device)
    out = torch.zeros((1, 8), device=device)
    W = torch.zeros((4, 1), device=device)
    with pytest.raises(ValueError, match="temperature"):
        ops.mmoe_heads_fwd_bwd(X, 3, [torch.zeros((8, 3), device=device)], 0.0, W, None, [BCE], None, out)
    with pytest.raises(ValueError, match="experts"):
        ops.mmoe_heads_fwd_bwd(X, 5, [torch.zeros((8, 5), device=device)], 1.0, W, None, [BCE], None, out)
    with pytest.raises(ValueError, match="gate_logits"):
        ops.mmoe_heads_fwd_bwd(X, 3, [torch.zeros((8, 4), device=device)], 1.0, W, None, [BCE], None, out)


# ---------------------------------------------------------------------------------------------------------------
# the training step against the restatement
# ---------------------------------------------------------------------------------------------------------------
def _batch(s, B, seed):
    b = datasets.generate_batch(s, B, seed=seed, index_law="uniform")
    feats, targs = datasets.split_targets(s, b)
    return feats, targs


def _targets(model, targs, device):
    return {o.target: torch.from_numpy(np.asarray(targs[o.target])).to(device) for o in model.output_blocks()}


def _check_gradients(model, tr, feats, targs, sample_weight=None):
    """One forward_backward against the restatement (with the device's relu decisions): loss, every dense gradient and the
    tables' dense gradients.  sample_weight: one (B,) numpy array or None per output."""
    arr = model_arrays(model)
    outs = model.output_blocks()
    ys = [np.asarray(targs[o.target]) for o in outs]
    dev = tr.device
    sw = None if sample_weight is None else [None if w is None else torch.from_numpy(w).to(dev) for w in sample_weight]
    tr.forward_backward(H.device_batch(feats, dev), [torch.from_numpy(y).to(dev) for y in ys], sample_weight=sw)
    b = len(ys[0])
    masks = {f"bottom_{i}": (tr.h[i][:b] > 0).cpu().numpy() for i in range(len(tr.bottom))}
    if tr.mmoe is not None:
        masks["experts"] = (tr.X[:b] > 0).cpu().numpy()
    for tag, bufs in (("gate", tr.gbufs), ("tower", tr.tbufs)):
        for t, (h_, _, _) in enumerate(bufs):
            masks.update({f"{tag}_{t}_{i}": (x[:b] > 0).cpu().numpy() for i, x in enumerate(h_)})
    total, per, zs, g = mmoe_loss_and_grads(feats, arr["tables"], arr["continuous"], arr["bottom"], arr["experts"], arr["gates"],
                                            arr["temperature"], arr["heads"], ys, loss_weights=model.loss_weights,
                                            sample_weight=sample_weight, masks=masks, towers=arr["towers"])
    close(tr._loss_all[0], total, 1e-5, "loss")
    if len(outs) > 1:
        close(tr._loss_all[1:], np.array(per), 1e-5, "per-task losses")
    a = tr.arena
    for i in range(len(tr.bottom)):
        close(a.view(a.grad, i, "kernel"), g[f"bottom/kernel_{i}"], TOL, f"bottom kernel {i}")
        close(a.view(a.grad, i, "bias"), g[f"bottom/bias_{i}"], TOL, f"bottom bias {i}")
    nb = len(tr.bottom)
    if tr.mmoe is not None:
        E = tr.mmoe.num_experts
        close(a.view(a.grad, nb, "kernel"), np.concatenate([g[f"expert/kernel_{e}"] for e in range(E)], 1), TOL, "expert kernels")
        close(a.view(a.grad, nb, "bias"), np.concatenate([g[f"expert/bias_{e}"] for e in range(E)]), TOL, "expert biases")
        if tr.mmoe.gates is not None:
            close(a.view(a.grad, nb + 1, "kernel"), np.concatenate([g[f"gate/kernel_{t}"] for t in range(len(outs))], 1), TOL, "gates")
    for tag, li0s, chains in (("gate", tr.gate_li0, tr.gate_chains), ("tower", tr.tower_li0, tr.towers)):
        for t, (li0, c) in enumerate(zip(li0s, chains)):
            for i, l in enumerate(c):
                close(a.view(a.grad, li0 + i, "kernel"), g[f"{tag}_{t}/kernel_{i}"], TOL, f"{tag} {t} kernel {i}")
                if l.bias is not None:
                    close(a.view(a.grad, li0 + i, "bias"), g[f"{tag}_{t}/bias_{i}"], TOL, f"{tag} {t} bias {i}")
    hi = len(a.layers) - 1
    close(a.view(a.grad, hi, "kernel"), np.concatenate([g[f"head/kernel_{t}"] for t in range(len(outs))], 1), TOL, "head kernel")
    close(a.view(a.grad, hi, "bias"), np.concatenate([g[f"head/bias_{t}"] for t in range(len(outs))]), TOL, "head bias")
    tr._bag_grads()
    for t, f in enumerate(tr.feats):
        rows, D = tr.tables[t].table.shape
        dense = torch.zeros((rows, D), dtype=torch.float64, device=dev)
        bag = tr._bags.get(t)
        ids, sl = (bag["apply_ids"], bag["rows"]) if bag is not None else (tr._idx[t], tr._slices[t])
        ids = ops.widen_index(ids).reshape(-1).long()
        ok = (ids >= 0) & (ids < rows)
        dense.index_add_(0, ids[ok], sl.reshape(-1, D)[ok].double())
        close(dense, g[f"table/{f}"], TOL, f"table {f}")
    return total


@pytest.mark.parametrize("case", ["mmoe", "mmoe_bottom", "bottom_only", "single_output", "lists", "towers_gates", "towers_only",
                                  "bottom_towers", "single_towers"])
def test_training_step_gradients_match_the_restatement(device, case):
    mm.set_seed(11)
    lists = [("L_r", 300, True), ("L_f", 260, False)] if case == "lists" else ()  # inferred width 16
    s = schema(lists=lists, targets=(("click", "bin"),) if case in ("single_output", "single_towers") else (("click", "bin"), ("conversion", "bin"),
                                                                                           ("rating", "reg")))
    if case == "bottom_only":
        model = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([32, 16]), mm.OutputBlock(s))
    elif case == "bottom_towers":  # the towers read the shared bottom's output
        model = mm.Model(mm.InputBlockV2(s), mm.MLPBlock([32, 16]), mm.OutputBlock(s, task_blocks=mm.MLPBlock([16, 8])))
    elif case in ("towers_gates", "towers_only", "single_towers"):  # the notebook's configuration (towers, gate blocks)
        model = mmoe_model(s, E=4, U=16, bottom=[32] if case == "towers_gates" else None, T=0.9, towers=[12],
                           gate=None if case == "towers_only" else [8])
    else:
        model = mmoe_model(s, E=3, U=16, bottom=[32] if case in ("mmoe_bottom", "lists") else None, T=0.8)
    model.build(device)
    model.compile(optimizer="sgd", loss_weights=None if case.startswith("single") else [1.0, 0.5, 2.0])
    B = 300
    feats, targs = _batch(s, B, 5)
    if case == "lists":  # the fixed-length list feature as a (B, 3) id matrix
        feats.pop("L_f__values"), feats.pop("L_f__offsets")
        feats["L_f"] = np.random.default_rng(2).integers(0, 261, (B, 3)).astype(np.int32)
    tr = model.trainer(B)
    _check_gradients(model, tr, feats, targs)


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_and_graph_replay_equal_eager(device, opt):
    """Three steps with each optimizer on the notebook's configuration (shared bottom, gate blocks, task towers): the first
    step's gradients against the restatement, and a captured graph replays the same steps as the eager engine."""
    s = schema()
    mk = lambda: {"sgd": mm.SGD(0.5), "adagrad": mm.Adagrad(0.1), "adam": mm.Adam(0.01)}[opt]
    mm.set_seed(21)
    ma = mmoe_model(s, E=4, U=16, bottom=[32], T=1.3, towers=[12], gate=[8])
    mm.set_seed(21)
    mb = mmoe_model(s, E=4, U=16, bottom=[32], T=1.3, towers=[12], gate=[8])
    for m in (ma, mb):
        m.build(device)
        m.compile(optimizer=mk())
    for (na, va), (nb_, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        assert torch.equal(va, vb), na
    B = 256
    batches = [_batch(s, B, 40 + k) for k in range(3)]
    ta, tb = ma.trainer(B), mb.trainer(B)
    _check_gradients(ma, ta, *batches[0])
    ta.apply_gradients()
    ta._after_step()
    tb.capture(H.device_batch(batches[0][0], device), list(_targets(mb, batches[0][1], device).values()))
    tb.replay(H.device_batch(batches[0][0], device), list(_targets(mb, batches[0][1], device).values()))
    losses = []
    for f, t in batches[1:]:
        la = ma.train_step((H.device_batch(f, device), _targets(ma, t, device)))["loss"].clone()
        lb = tb.replay(H.device_batch(f, device), list(_targets(mb, t, device).values()))[0].clone()
        close(lb, la, 1e-5, "replayed loss")
        losses.append(float(la))
    # the two engines sum their atomics in different orders; Adam divides by sqrt(v), which magnifies that in tiny updates
    for (na, va), (nb_, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(vb, va, 2e-4 if opt == "adam" else 1e-5, na)
    assert all(np.isfinite(losses))


def test_benchmark_size_step(device):
    """One step at B = 65 536 on the Criteo schema with click / conversion / rating targets at inferred embedding widths
    (tables capped at 20 000 rows)."""
    mm.set_seed(3)
    base = datasets.criteo_schema({k: min(v, 20000) for k, v in datasets.CRITEO_MAX.items()})
    cols = [c for c in base if c.name != "label"]
    from models_b200.schema import ColumnSchema, Schema, Tags

    cols += [ColumnSchema("click", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
             ColumnSchema("conversion", tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION), dtype="int64"),
             ColumnSchema("rating", tags=(Tags.TARGET, Tags.REGRESSION), dtype="float32")]
    s = Schema(cols)
    model = mmoe_model(s, E=4, U=64)
    model.build(device)
    assert model.body.input_width() > 256  # the input gradient takes the transposed-kernel GEMM at every width
    model.compile(optimizer=mm.Adagrad(0.01))
    feats, targs = _batch(s, 65536, 9)
    tr = model.trainer(65536)
    _check_gradients(model, tr, feats, targs)


# ---------------------------------------------------------------------------------------------------------------
# model-level paths
# ---------------------------------------------------------------------------------------------------------------
def _evaluate_matches_call(model, feats, targs, device):
    """evaluate's loss, per-output losses and binary accuracy against values computed from call's predictions."""
    out = model(H.device_batch(feats, device))
    outs = model.output_blocks()
    preds = out if isinstance(out, dict) else {outs[0].name: out}
    res = model.evaluate([(H.device_batch(feats, device), _targets(model, targs, device))], return_dict=True)
    total = 0.0
    for o in outs:
        p = preds[o.name].double().cpu().numpy().reshape(-1)
        y = np.asarray(targs[o.target], dtype=np.float64)
        if o.loss == BCE:
            pc = np.clip(p, 1e-7, 1 - 1e-7)
            lt = float(np.mean(-(y * np.log(pc) + (1 - y) * np.log(1 - pc))))
            acc = float(np.mean((p > 0.5) == (y > 0.5)))
            key = "binary_accuracy" if len(outs) == 1 else f"{o.name}/binary_accuracy"
            assert abs(res[key] - acc) < 1e-6, (key, res[key], acc)
        else:
            lt = float(np.mean((p - y) ** 2))
        if len(outs) > 1:
            assert abs(res[f"{o.name}_loss"] - lt) < 1e-4 * max(1.0, lt), (o.name, res[f"{o.name}_loss"], lt)
        total += lt
    assert abs(res["loss"] - total) < 1e-4 * max(1.0, total), (res["loss"], total)
    return res


def test_forward_evaluate_fit_save_load_and_compiled_forward(device, tmp_path):
    s = schema()
    mm.set_seed(5)
    model = mmoe_model(s, E=4, U=32, bottom=[32], T=0.9, towers=[16], gate=[8])
    model.build(device)
    model.compile(optimizer=mm.Adagrad(0.05))
    feats, targs = _batch(s, 512, 77)
    out = model(H.device_batch(feats, device))
    assert isinstance(out, dict) and sorted(out) == model.prediction.names
    arr = model_arrays(model)
    outs = model.output_blocks()
    _, _, zs, _ = mmoe_loss_and_grads(feats, arr["tables"], arr["continuous"], arr["bottom"], arr["experts"], arr["gates"],
                                      arr["temperature"], arr["heads"], [np.asarray(targs[o.target]) for o in outs],
                                      towers=arr["towers"])
    for o, z in zip(outs, zs):
        ref = 1.0 / (1.0 + np.exp(-z)) if o.loss == BCE else z
        close(out[o.name].reshape(-1), ref, 2e-4, f"forward {o.name}")
    z, form = model.logits(H.device_batch(feats, device))
    from models_b200._cabi import PRED_HEAD

    assert form == PRED_HEAD
    from models_b200 import models as models_mod

    for graph in (True, False):  # the captured evaluation graph and the eager path
        models_mod._EVAL_GRAPH[0] = graph
        try:
            _evaluate_matches_call(model, feats, targs, device)
        finally:
            models_mod._EVAL_GRAPH[0] = True
    data = [(H.device_batch(feats, device), _targets(model, targs, device))]
    hist = model.fit(data, epochs=2, validation_data=data).history
    for o in outs:
        assert f"{o.name}_loss" in hist and f"val_{o.name}_loss" in hist and len(hist[f"{o.name}_loss"]) == 2
    assert "val_loss" in hist
    # save / load: bit-identical predictions
    after = model(H.device_batch(feats, device))
    model.save(tmp_path / "export")
    loaded = mm.Model.load(tmp_path / "export")
    got = loaded(H.device_batch(feats, device))
    for k in after:
        np.testing.assert_array_equal(got[k].cpu().numpy(), after[k].cpu().numpy())
    names = set(loaded.weights())
    assert any(n.startswith("body/mmoe/expert_3/") for n in names)
    assert {f"body/mmoe/gate_{n}/gate_final/kernel" for n in model.prediction.names} <= names
    # load_weights into a fresh model with the same structure
    fresh = mm.Model.load(tmp_path / "export")
    for v in fresh.weights().values():
        v.zero_()
    fresh.load_weights(tmp_path / "export")
    for k, v in fresh(H.device_batch(feats, device)).items():
        np.testing.assert_array_equal(v.cpu().numpy(), after[k].cpu().numpy())
    # the compiled forward returns the same dict
    hb = HostBatch.like(feats, model.input_columns())
    cf = model.compile(hb)
    res = cf(hb)
    assert isinstance(res, dict)
    for k in after:
        close(np.asarray(res[k]).reshape(-1), after[k].cpu().numpy().reshape(-1), 1e-6, f"compiled {k}")


def test_single_output_evaluate_matches_call(device):
    s = schema(targets=(("click", "bin"),))
    out = mm.BinaryOutput("click")
    model = mm.Model(mm.InputBlockV2(s), mm.MMOEBlock(out, mm.MLPBlock([16]), 3), out)
    model.build(device)
    model.compile(optimizer="adam")
    feats, targs = _batch(s, 200, 3)
    p = model(H.device_batch(feats, device)).reshape(-1)
    z, form = model.logits(H.device_batch(feats, device))
    from models_b200._cabi import PRED_HEAD

    assert form == PRED_HEAD and z.shape == (1, 200)
    zt = z[0].double().cpu().numpy()
    close(p, 1 / (1 + np.exp(-zt)), 1e-6, "sigmoid of the logits")
    _evaluate_matches_call(model, feats, targs, device)
