"""NCFModel on the GPU: mm_ncf_head_fwd_bwd against float64 at every compiled instantiation, one training step against the
reference's torch fixture and the float64 restatement (tests/ncf_train_oracle.py), three optimizer steps eager and as a
CUDA graph, the trained model's forward, evaluate, compiled forward and save / load, fit on a planted rule, the benchmark's
step size and the refusals that need a device."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import ops
from models_b200.schema import ColumnSchema, Schema, Tags
from tests.ncf_train_oracle import golden_inputs, model_params, ncf_loss_and_grads, ncf_train_steps

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "ncf_train" / "ref_torch_ncf_train.npz"
BCE, MSE = "binary_crossentropy", "mse"

# (D, U, H, B, id bytes, l2, relu_h): every (H rounded up to 1/2/4/8, columns per lane of D, of U) pair the launcher
# dispatches, each at one case (tests/test_ncf_host.py checks that the table reaches all 48)
_HS = (1, 2, 3, 8)
_BS, _WS = (1, 37, 4099, 37, 1000), (4, 8, 1, 2, 3)
KERNEL_CASES = []
for _hi, _H in enumerate(_HS):
    for _di, _D in enumerate((16, 64, 128)):
        for _ui, _U in enumerate((8, 48, 100, 256)):
            n = len(KERNEL_CASES)
            D = 4 if (_D == 16 and n % 2) else _D  # D = 4 and 16 share the one-column kernels
            U = 200 if (_U == 256 and n % 8 == 3) else (64 if (_U == 48 and n % 3 == 0) else _U)
            KERNEL_CASES.append((D, U, _H, 65536 if n in (7, 29) else _BS[n % 5], _WS[n % 5], 1e-3 if n % 2 else 0.0, n % 3 != 2))


def _rows_for(width: int) -> int:
    return {1: 200, 2: 3000, 3: 70000}.get(width, 5000)


def _ids(rng, B, rows, width, dev):
    """(ids as the kernel reads them, as int64) with a few out-of-range ids and duplicates."""
    v = rng.integers(0, rows, B).astype(np.int64)
    if B > 4:
        v[1] = v[0]
        v[B // 2] = rows + 3 if width != 1 else rows + 10  # out of range (still fits one byte for width 1)
    if width == 4:
        t = torch.from_numpy(v.astype(np.int32))
    elif width == 8:
        t = torch.from_numpy(v)
    elif width == 1:
        t = torch.from_numpy(v.astype(np.uint8))
    elif width == 2:
        t = torch.from_numpy(v.astype(np.uint16))
    else:
        t = torch.from_numpy(np.stack([v & 255, (v >> 8) & 255, (v >> 16) & 255], 1).astype(np.uint8))
    return t.to(dev), v


def _ref(tu, ti, vu, vi, h, w, b, losses, ys, lws, sws, l2, relu_h):
    """float64 forward and backward of the head on the device."""
    d = torch.float64
    dev = h.device
    ok_u = torch.as_tensor((vu >= 0) & (vu < tu.shape[0]), device=dev)
    ok_i = torch.as_tensor((vi >= 0) & (vi < ti.shape[0]), device=dev)
    iu = torch.as_tensor(np.clip(vu, 0, tu.shape[0] - 1), device=dev)
    ii = torch.as_tensor(np.clip(vi, 0, ti.shape[0] - 1), device=dev)
    u = (tu.to(d)[iu] * ok_u.unsqueeze(1)).requires_grad_(True)
    i = (ti.to(d)[ii] * ok_i.unsqueeze(1)).requires_grad_(True)
    hh = h.to(d).requires_grad_(True)
    W = w.to(d).requires_grad_(True)
    bb = b.to(d).requires_grad_(True)
    z = torch.cat([u * i, hh], 1) @ W + bb
    B = z.shape[0]
    total = torch.zeros((), dtype=d, device=dev)
    per = []
    for t, (l, y) in enumerate(zip(losses, ys)):
        zt, yt = z[:, t], y.to(d)
        term = (zt + zt.abs()) / 2 - zt * yt + torch.log1p(torch.exp(-zt.abs())) if l == BCE else (zt - yt) ** 2
        if sws[t] is not None:
            term = term * sws[t].to(d)
        lt = term.sum() / B
        per.append(lt)
        total = total + lws[t] * lt
    reg = l2 * ((u * u).sum() + (i * i).sum())
    (total + reg).backward()
    dh = hh.grad.clone()
    if relu_h:
        dh[h <= 0] = 0
    return dict(z=z.detach().T, loss=torch.stack([total + reg] + per).detach(), reg=reg.detach(), du=u.grad, di=i.grad, dh=dh,
                dw=W.grad, db=bb.grad, oob=int((~ok_u).sum() + (~ok_i).sum()))


def _close(got, want, what, rtol=2e-4, atol_rel=1e-5):
    got, want = got.double(), want.double()
    scale = max(float(want.abs().max()), 1e-30)
    err = float((got - want).abs().max())
    assert torch.allclose(got, want, rtol=rtol, atol=atol_rel * scale), f"{what}: max |err| {err:.3e} (scale {scale:.3e})"


@pytest.mark.parametrize("D,U,H,B,width,l2,relu_h", KERNEL_CASES)
def test_ncf_head_kernel_matches_float64(D, U, H, B, width, l2, relu_h):
    dev = torch.device("cuda")
    rng = np.random.default_rng(D * 1000 + U * 10 + H + B)
    g = torch.Generator(device="cpu").manual_seed(B + D)
    rows = _rows_for(width)
    tu = (torch.randn((rows, D), generator=g) * 0.3).to(dev)
    ti = (torch.randn((rows + 7, D), generator=g) * 0.3).to(dev)
    ids_u, vu = _ids(rng, B, rows, width, dev)
    ids_i, vi = _ids(rng, B, rows + 7, width, dev)
    h = torch.randn((B, U), generator=g).to(dev)
    if relu_h:
        h = torch.relu(h)
        h[0, 0] = 0.0  # an exact zero at the strict mask
    w = (torch.randn((D + U, H), generator=g) * 0.2).to(dev)
    b = torch.randn(H, generator=g).to(dev)
    losses = [BCE if t % 2 == 0 else MSE for t in range(H)]
    ys = [torch.from_numpy(rng.integers(0, 2, B).astype(np.float32)).to(dev) if l == BCE
          else torch.from_numpy((rng.random(B) * 3).astype(np.float32)).to(dev) for l in losses]
    lws = [1.0 if t == 0 else 0.5 + 0.25 * t for t in range(H)]
    sws = [None if t % 2 == 0 else torch.from_numpy(rng.random(B).astype(np.float32)).to(dev) for t in range(H)]
    if H == 1 and B > 1:
        sws = [torch.from_numpy(rng.random(B).astype(np.float32)).to(dev)]
        sws[0][0] = 0.0
    f32 = dict(dtype=torch.float32, device=dev)
    out = torch.full((H, B), float("nan"), **f32)
    loss = torch.zeros(1 + H, **f32)
    reg = torch.zeros(1, **f32)
    du, di = torch.full((B, D), float("nan"), **f32), torch.full((B, D), float("nan"), **f32)
    dh_buf = torch.full((B, U + 5), float("nan"), **f32)  # strided: 5 guard columns must stay NaN
    dh = dh_buf[:, :U]
    dw, db = torch.zeros((D + U, H), **f32), torch.zeros(H, **f32)
    oob = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.ncf_head_fwd_bwd(tu, ids_u, ti, ids_i, h, w, b, losses, ys, out, loss=loss, reg=reg if l2 else None, l2=l2, du=du, di=di,
                         dh=dh, dw=dw, db=db, loss_weights=lws, relu_h=relu_h, sample_weight=sws, oob=oob)
    ref = _ref(tu, ti, vu, vi, h, w, b, losses, ys, lws, sws, l2, relu_h)
    _close(out, ref["z"], "logits")
    _close(loss, ref["loss"], "loss")
    if l2:
        _close(reg, ref["reg"].reshape(1), "reg")
    _close(du, ref["du"], "du")
    _close(di, ref["di"], "di")
    _close(dh, ref["dh"], "dh")
    assert torch.isnan(dh_buf[:, U:]).all(), "dh's guard columns were written"
    _close(dw, ref["dw"], "dw")
    _close(db, ref["db"], "db")
    assert int(oob.item()) == ref["oob"]
    # the forward-only form: the predictions of the training form's logits, the same reg, nothing else written
    pred = torch.full((H, B), float("nan"), **f32)
    reg2 = torch.zeros(1, **f32)
    oob.zero_()
    ops.ncf_head_fwd_bwd(tu, ids_u, ti, ids_i, h, w, b, losses, None, pred, reg=reg2 if l2 else None, l2=l2, oob=oob)
    want = torch.stack([out[t] if l == MSE else torch.sigmoid(out[t].double()).float() for t, l in enumerate(losses)])
    assert torch.allclose(pred, want, rtol=1e-6, atol=1e-7)
    assert torch.equal(pred[[t for t, l in enumerate(losses) if l == MSE]], out[[t for t, l in enumerate(losses) if l == MSE]])
    if l2:
        _close(reg2, ref["reg"].reshape(1), "forward-only reg")
    assert int(oob.item()) == ref["oob"]


def test_ncf_head_argument_checks():
    dev = torch.device("cuda")
    f32 = dict(dtype=torch.float32, device=dev)
    tu, ti = torch.zeros((10, 8), **f32), torch.zeros((10, 8), **f32)
    ids = torch.zeros(4, dtype=torch.int32, device=dev)
    h, w, b, out = torch.zeros((4, 6), **f32), torch.zeros((14, 1), **f32), torch.zeros(1, **f32), torch.zeros((1, 4), **f32)
    ops.ncf_head_fwd_bwd(tu, ids, ti, ids, h, w, b, [BCE], None, out)
    with pytest.raises(ValueError, match="same width"):
        ops.ncf_head_fwd_bwd(tu, ids, torch.zeros((10, 4), **f32), ids, h, w, b, [BCE], None, out)
    with pytest.raises(ValueError, match="w must be"):
        ops.ncf_head_fwd_bwd(tu, ids, ti, ids, h, torch.zeros((13, 1), **f32), b, [BCE], None, out)
    with pytest.raises(ValueError, match="ids_u"):
        ops.ncf_head_fwd_bwd(tu, ids[:3], ti, ids, h, w, b, [BCE], None, out)
    with pytest.raises(ValueError, match="must be in"):
        big = torch.zeros((10, 132), **f32)
        ops.ncf_head_fwd_bwd(big, ids, big, ids, h, torch.zeros((138, 1), **f32), b, [BCE], None, out)
    with pytest.raises(ValueError, match="l2"):
        ops.ncf_head_fwd_bwd(tu, ids, ti, ids, h, w, b, [BCE], None, out, l2=-1.0)
    with pytest.raises(ValueError, match="training needs"):
        ops.ncf_head_fwd_bwd(tu, ids, ti, ids, h, w, b, [BCE], [torch.zeros(4, **f32)], out, loss=torch.zeros(2, **f32))
    with pytest.raises(ValueError, match="losses"):
        ops.ncf_head_fwd_bwd(tu, ids, ti, ids, h, w, b, ["hinge"], None, out)


# ---- models ----------------------------------------------------------------------------------------------------------
def _schema(users: int, items: int, targets=(("rating", "regression"), ("rating_binary", "binary"))) -> Schema:
    cols = [ColumnSchema("userId", tags=(Tags.CATEGORICAL, Tags.USER, Tags.USER_ID), dtype="int64",
                         properties={"domain": {"min": 0, "max": users - 1, "name": "userId"}}),
            ColumnSchema("movieId", tags=(Tags.CATEGORICAL, Tags.ITEM, Tags.ITEM_ID), dtype="int64",
                         properties={"domain": {"min": 0, "max": items - 1, "name": "movieId"}})]
    for n, k in targets:
        cols.append(ColumnSchema(n, tags=(Tags.TARGET, Tags.BINARY_CLASSIFICATION) if k == "binary" else (Tags.TARGET, Tags.REGRESSION),
                                 dtype="int64" if k == "binary" else "float32"))
    return Schema(cols)


def _set(t: torch.Tensor, v) -> None:
    with torch.no_grad():
        t.copy_(torch.as_tensor(np.asarray(v, dtype=np.float32)))


def _fixture_model(l2: float = 0.0):
    """An NCFModel whose tables are the fixture's touched rows (ids remapped to them) and whose Dense variables are the
    fixture's, and the remapped batch."""
    z = np.load(GOLDEN)
    ids, p, ys, losses = golden_inputs(z)
    dev = torch.device("cuda")
    model = mm.benchmark.NCFModel(_schema(len(z["mf_query_ids"]), len(z["mf_item_ids"])), int(z["dim"]),
                                  mm.MLPBlock([int(u) for u in z["units"]]), embeddings_l2_reg=l2)
    model.build(dev)
    assert [o.name for o in model.output_blocks()] == ["rating/regression_output", "rating_binary/binary_output"]
    body = model.body
    for b in ("mf", "mlp"):
        for s in ("query", "item"):
            _set(body.table(b, s).table, p[f"{b}/{s}"])
    for l, lp in zip(body.mlp.dense_layers, p["layers"]):
        _set(l.kernel, lp["kernel"])
        _set(l.bias, lp["bias"])
    _set(model.prediction.to_call.kernel, p["head_kernel"])
    _set(model.prediction.to_call.bias, p["head_bias"])
    x = {"userId": torch.from_numpy(ids["query"].astype(np.int64)).to(dev), "movieId": torch.from_numpy(ids["item"].astype(np.int64)).to(dev)}
    y = {"rating": torch.from_numpy(ys[0]).to(dev), "rating_binary": torch.from_numpy(ys[1]).to(dev)}
    return z, model, x, y, ids, p, ys, losses


def _table_grad(ids, rows, n):
    g = np.zeros((n, rows.shape[1]))
    np.add.at(g, ids.cpu().numpy().astype(np.int64).reshape(-1), rows.double().cpu().numpy())
    return g


@pytest.mark.parametrize("l2", [0.0, 1e-3])
def test_ncf_step_matches_fixture_and_restatement(l2):
    z, model, x, y, ids, p, ys, losses = _fixture_model(l2)
    model.compile(optimizer=mm.SGD(0.1))
    tr = model.trainer(len(ids["query"]))
    tr.forward_backward(x, [y["rating"], y["rating_binary"]])
    loss, reg, per, Z, grads = ncf_loss_and_grads(ids, p, losses, ys, l2=l2)
    got = tr._loss_all.double().cpu().numpy()
    assert abs(got[1] - loss) < 1e-5 * max(1.0, abs(loss)) and abs(got[0] - reg) < 1e-5 * max(1.0, reg + 1e-3)
    np.testing.assert_allclose(got[2:], per, rtol=2e-5, atol=1e-6)
    if not l2:
        assert abs(got[1] - float(z["loss"])) < 1e-5 * abs(float(z["loss"]))
    tg = tr.table_gradients()
    for b in ("mf", "mlp"):
        for s in ("query", "item"):
            want = grads[f"{b}/{s}"]
            gi, gr = tg[f"{b}/{s}"]
            # h comes out of the tower's split-bf16 (x3) GEMMs, |err| ~ 2^-16 relative: it reaches every table's gradient
            np.testing.assert_allclose(_table_grad(gi, gr, want.shape[0]), want, rtol=1e-4, atol=2e-5 * np.abs(want).max())
            if not l2:
                np.testing.assert_allclose(want[np.unique(ids[s])], z[f"grad_{b}_{s}_rows"], rtol=1e-5, atol=1e-8)
    dg = tr.gradients()
    for i, l in enumerate(model.body.mlp.dense_layers):
        np.testing.assert_allclose(dg[f"{l.name}/kernel"].double().cpu().numpy(), grads[f"kernel_{i}"], rtol=1e-3,
                                   atol=2e-3 * np.abs(grads[f"kernel_{i}"]).max())  # the tower's wgrad reads split-bf16 x
        np.testing.assert_allclose(dg[f"{l.name}/bias"].double().cpu().numpy(), grads[f"bias_{i}"], rtol=1e-3,
                                   atol=2e-3 * np.abs(grads[f"bias_{i}"]).max())
    hd = model.prediction.to_call.name
    np.testing.assert_allclose(dg[f"{hd}/kernel"].double().cpu().numpy(), grads["head_kernel"], rtol=1e-4,
                               atol=1e-5 * np.abs(grads["head_kernel"]).max())
    np.testing.assert_allclose(dg[f"{hd}/bias"].double().cpu().numpy(), grads["head_bias"], rtol=1e-4, atol=1e-6)


def _random_model(seed, users=300, items=500, dim=16, units=(32, 8), l2=1e-3, targets=(("click", "binary"),), opt="adagrad"):
    mm.set_seed(seed)
    model = mm.benchmark.NCFModel(_schema(users, items, targets), dim, mm.MLPBlock(list(units)), embeddings_l2_reg=l2)
    model.build(torch.device("cuda"))
    model.compile(optimizer=opt)
    return model


def _random_batches(n, B, users, items, seed, planted=False):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        u, i = rng.integers(0, users, B), rng.integers(0, items, B)
        y = ((u % 2) == (i % 2)).astype(np.float32) if planted else rng.integers(0, 2, B).astype(np.float32)
        out.append((u.astype(np.int64), i.astype(np.int64), y))
    return out


def _dev_batch(u, i, y):
    dev = torch.device("cuda")
    return {"userId": torch.from_numpy(u).to(dev), "movieId": torch.from_numpy(i).to(dev)}, torch.from_numpy(y).to(dev)


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_ncf_three_steps_per_optimizer_and_graph_replay(opt):
    batches = _random_batches(3, 256, 300, 500, seed=5)
    model = _random_model(11, opt=opt)
    p0 = model_params(model)
    want, p3 = ncf_train_steps([dict(ids={"query": u, "item": i}, targets=[y]) for u, i, y in batches], p0, [BCE], opt,
                               {"sgd": 0.01, "adagrad": 0.001, "adam": 0.001}[opt], l2=1e-3)
    got = [float(model.train_step(_dev_batch(*b))["loss"].item()) for b in batches]
    np.testing.assert_allclose(got, want, rtol=2e-5)
    p_got = model_params(model)
    for k in ("mf/query", "mf/item", "mlp/query", "mlp/item", "head_kernel"):
        np.testing.assert_allclose(p_got[k], p3[k], rtol=1e-4, atol=1e-6)
    # the same three steps as one captured graph on a second, identically initialised model
    g = _random_model(11, opt=opt)
    tr = g.trainer(256)
    x0, y0 = _dev_batch(*batches[0])
    tr.capture(x0, [y0])
    assert tr.launches_per_step > 0
    for b in batches:
        x, y = _dev_batch(*b)
        tr.replay(x, [y])
    p_g = model_params(g)
    for k in ("mf/query", "mf/item", "mlp/query", "mlp/item", "head_kernel", "head_bias"):
        np.testing.assert_allclose(p_g[k], p_got[k], rtol=1e-5, atol=1e-7)


def test_ncf_trained_model_forward_evaluate_compiled_and_save_load(tmp_path):
    model = _random_model(21, targets=(("rating", "regression"), ("click", "binary")), l2=1e-3)
    batches = _random_batches(4, 512, 300, 500, seed=8, planted=True)
    for u, i, y in batches:
        x, yt = _dev_batch(u, i, y)
        m = model.train_step((x, {"rating": yt * 3.0, "click": yt}))
    assert float(m["regularization_loss"].item()) > 0
    names = [o.name for o in model.output_blocks()]  # the heads' column order
    losses = [MSE if n.startswith("rating") else BCE for n in names]
    ys = lambda y: [y * 3.0 if n.startswith("rating") else y for n in names]  # noqa: E731
    u, i, y = batches[-1]
    x, yt = _dev_batch(u, i, y)
    out = model(x)
    p = model_params(model)
    _, reg, _, Z, _ = ncf_loss_and_grads({"query": u, "item": i}, p, losses, ys(y), l2=1e-3)
    for t, n in enumerate(names):
        want = Z[t] if losses[t] == MSE else 1 / (1 + np.exp(-Z[t]))
        np.testing.assert_allclose(out[n].double().cpu().numpy().reshape(-1), want, rtol=1e-3, atol=1e-4)
    data = [(_dev_batch(u, i, y)[0], {"rating": _dev_batch(u, i, y)[1] * 3.0, "click": _dev_batch(u, i, y)[1]})
            for u, i, y in batches]
    res = model.evaluate(data, return_dict=True)
    regs, batch_losses = [], []
    for u, i, y in batches:
        L, r, _, _, _ = ncf_loss_and_grads({"query": u, "item": i}, p, losses, ys(y), l2=1e-3)
        regs.append(r)
        batch_losses.append(L)
    assert abs(res["loss"] - np.mean(batch_losses)) < 1e-3 * abs(np.mean(batch_losses))
    assert abs(res["regularization_loss"] - regs[-1]) < 1e-4 * regs[-1]
    zc = np.concatenate([ncf_loss_and_grads({"query": u, "item": i}, p, losses, ys(y), l2=1e-3)[3][names.index("click/binary_output")]
                         for u, i, y in batches])
    yc = np.concatenate([y for _, _, y in batches])
    assert abs(res["click/binary_output/auc"] - _auc(yc, zc)) < 0.02  # 200 thresholds against the exact rank statistic
    from models_b200 import models as M

    M._EVAL_GRAPH[0] = False
    try:
        eager = model.evaluate(data, return_dict=True)
    finally:
        M._EVAL_GRAPH[0] = True
    for k in res:
        assert abs(res[k] - eager[k]) <= 1e-6 * max(1.0, abs(eager[k])), k
    from models_b200.graph import HostBatch

    hb = HostBatch.like({"userId": u, "movieId": i}, model.input_columns(), id_bytes=model.id_bytes())  # packed ids
    cf = model.compile(hb)
    pred = cf(hb)
    np.testing.assert_allclose(np.asarray(pred["click/binary_output"]).reshape(-1),
                               out["click/binary_output"].cpu().numpy().reshape(-1), rtol=1e-6, atol=1e-7)
    model.save(tmp_path / "ncf")
    loaded = mm.Model.load(tmp_path / "ncf", device=torch.device("cuda"))
    assert sorted(loaded.weights()) == sorted(model.weights())
    out2 = loaded(x)
    for k in out:
        assert torch.equal(out[k], out2[k])


def _auc(y, s):
    r = np.empty(len(s))
    r[np.argsort(s)] = np.arange(1, len(s) + 1)
    P = y.sum()
    return (r[y == 1].sum() - P * (P + 1) / 2) / (P * (len(y) - P))


def test_ncf_fit_learns_a_planted_rule():
    model = _random_model(31, users=64, items=64, dim=8, units=(16, 8), l2=1e-5, opt=mm.Adam(0.01))
    batches = [_dev_batch(*b) for b in _random_batches(16, 1024, 64, 64, seed=12, planted=True)]
    before = model.evaluate(batches, return_dict=True)
    hist = model.fit(batches, epochs=4)
    after = model.evaluate(batches, return_dict=True)
    assert "regularization_loss" in hist.history and len(hist.history["regularization_loss"]) == 4
    assert hist.history["loss"][-1] < hist.history["loss"][0]
    assert after["loss"] < before["loss"] and after["auc"] > max(before["auc"], 0.8)


def test_ncf_step_at_benchmark_size():
    """One step at the benchmark's batch size, embedding width and tower ([256, 64]) on 200 000-row tables: loss and the
    GMF gradients against float64."""
    B = 65536
    model = _random_model(41, users=200_000, items=200_000, dim=64, units=(256, 64), l2=1e-4)
    (u, i, y), = _random_batches(1, B, 200_000, 200_000, seed=3)
    x, yt = _dev_batch(u, i, y)
    tr = model.trainer(B)
    tr.forward_backward(x, [yt])
    loss, reg, _, _, grads = ncf_loss_and_grads({"query": u, "item": i}, model_params(model), [BCE], [y], l2=1e-4)
    got = tr._loss_all.double().cpu().numpy()
    assert abs(got[1] - loss) < 1e-5 * abs(loss) and abs(got[0] - reg) < 1e-4 * reg
    tg = tr.table_gradients()
    for k in ("mf/query", "mf/item"):
        gi, gr = tg[k]
        want = grads[k]
        np.testing.assert_allclose(_table_grad(gi, gr, want.shape[0]), want, rtol=1e-3, atol=1e-5 * np.abs(want).max())


def test_ncf_refusals_on_device():
    from models_b200.blocks import set_dense_engine

    model = _random_model(51)
    u, i, y = _random_batches(1, 64, 300, 500, seed=1)[0]
    x, yt = _dev_batch(u, i, y)
    set_dense_engine("fp32")
    try:
        with pytest.raises(NotImplementedError, match="tensor-core engine"):
            model.train_step((x, yt))
    finally:
        set_dense_engine("auto")
    model._trainer = None
    tr = model.trainer(64)
    offs = torch.arange(0, 65, device=x["userId"].device, dtype=torch.int64)
    ragged = {"userId__values": x["userId"], "userId__offsets": offs, "movieId": x["movieId"]}
    with pytest.raises(NotImplementedError, match="ragged"):
        tr.capture(ragged, [yt])
    with pytest.raises(NotImplementedError, match="multi-hot|one id per sample"):
        tr.step(ragged, [yt])
