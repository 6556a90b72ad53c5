"""WideAndDeepModel on the GPU: mm_wide_deep_head_fwd_bwd and mm_wide_bag_grad (+ mm_wide_rows_apply) against float64
references, then WideAndDeepTrainer against the restatement (tests/wide_deep_train_oracle.py), graph replay, the forward,
evaluate, save / load, the compiled forward and fit.  Tolerances: max |diff| / max |ref| per tensor."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import ops
from tests.test_wide_deep_host import schema
from tests.wide_deep_train_oracle import BCE, MSE, bags_of, encode, wide_deep_forward, wide_deep_loss_and_grads

pytestmark = pytest.mark.gpu
TOL = 3e-4
LISTS = [("L2", 300), ("L4", 260)]  # inferred embedding width 16: the multi-hot deep update takes 16, 32, 64, 128


def close(got, ref, tol=TOL, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale if ref.size else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def packed(ids: np.ndarray, width: int, device) -> torch.Tensor:
    if width == 1:
        return torch.from_numpy(ids.astype(np.uint8)).to(device)
    if width == 2:
        return torch.from_numpy(ids.astype(np.uint16)).to(device)
    if width == 3:
        u = ids.astype(np.uint32)
        return torch.from_numpy(np.stack([u & 255, (u >> 8) & 255, (u >> 16) & 255], 1).astype(np.uint8)).to(device)
    return torch.from_numpy(ids.astype(np.int32 if width == 4 else np.int64)).to(device)


# ---------------------------------------------------------------------------------------------------------------
# mm_wide_deep_head_fwd_bwd against float64
# ---------------------------------------------------------------------------------------------------------------
def _head_case(device, B, n_oh, bag_kinds, mode, loss, use_sw, act_dl, U, seed=0):
    """One-hot features of every id width (about 8 % of the ids out of range), bag features ragged (empty bags,
    duplicates, offsets that leave values uncovered at both ends) or fixed length."""
    g = np.random.default_rng(seed)
    onehot, oh_np, bags, bag_np, off = [], [], [], [], 0
    for f in range(n_oh):
        w = (1, 2, 3, 4, 8)[f % 5]
        rows = int(g.integers(20, 230))
        ids = g.integers(0, rows + rows // 12 + 1, B)
        onehot.append((packed(ids, w, device), rows, off))
        oh_np.append((ids, rows, off))
        off += rows
    for q, kind in enumerate(bag_kinds):
        rows = int(g.integers(5, 40))
        dt = (torch.int32, torch.int64, torch.uint8, torch.uint16)[q % 4]
        if kind == "fixed":
            L = int(g.integers(1, 9))
            v = g.integers(0, rows + 2, (B, L))
            bags.append((torch.from_numpy(v).to(device).to(dt), None, rows, off, mode))
            bag_np.append((v, rows, off))
        else:
            lens = g.integers(0, 12, B)
            lens[::7] = 0
            head = 3  # values before offsets[0] and after offsets[B] belong to no bag
            offs = np.concatenate([[0], np.cumsum(lens)]) + head
            v = g.integers(0, rows + 2, int(offs[-1]) + 2)
            v[head:head + 4] = v[head]  # duplicates in the first bag
            bags.append((torch.from_numpy(v).to(device).to(dt), torch.from_numpy(offs).to(device).to(torch.int32 if q % 2 else torch.int64),
                         rows, off, mode))
            bag_np.append(((v, offs), rows, off))
        off += rows
    W = max(off, 1)
    f32 = lambda *s: torch.from_numpy(g.standard_normal(s).astype(np.float32) * 0.4).to(device)  # noqa: E731
    p = dict(onehot=onehot, oh_np=oh_np, bags=bags, bag_np=bag_np, mode=mode, wide=f32(W) if off else None, bw=f32(1) if off else None,
             h=torch.from_numpy(np.maximum(g.standard_normal((B, U)), 0).astype(np.float32)).to(device) if U else None,
             w_dl=f32(U) if U else None, b_dl=f32(1), act_dl=act_dl, out_w=f32(1) + 1.0, out_b=f32(1), loss=loss)
    p["y"] = torch.from_numpy(g.integers(0, 2, B)).to(device) if loss == BCE else torch.from_numpy(g.standard_normal(B).astype(np.float32)).to(device)
    p["sw"] = torch.from_numpy(g.random(B).astype(np.float32) * 2).to(device) if use_sw else None
    return p


def _head_ref(p, B):
    dev = p["y"].device
    s = torch.zeros(B, dtype=torch.float64, device=dev)
    n_bad = 0
    if p["wide"] is not None:
        wk = p["wide"].double().cpu().numpy()
        w = np.zeros(B)
        for ids, rows, off in p["oh_np"]:
            ok = ids < rows
            n_bad += int((~ok).sum())
            w += np.where(ok, wk[off + np.minimum(ids, rows - 1)], 0.0)
        for x, rows, off in p["bag_np"]:
            w += encode(x, rows, p["mode"]) @ wk[off:off + rows]
            n_bad += sum(int((ids >= rows).sum()) for ids in bags_of(x))
        s += torch.from_numpy(w).to(dev) + p["bw"].double()
    u = None
    if p["h"] is not None:
        u = p["h"].double() @ p["w_dl"].double() + p["b_dl"].double()
        s += torch.relu(u) if p["act_dl"] == "relu" else u
    z = s * p["out_w"].double() + p["out_b"].double()
    y = p["y"].double()
    sw = p["sw"].double() if p["sw"] is not None else torch.ones_like(z)
    if p["loss"] == BCE:
        per, g = torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs())), torch.sigmoid(z) - y
    else:
        per, g = (z - y) ** 2, 2 * (z - y)
    delta = g * sw / B
    ds = delta * p["out_w"].double()
    out = dict(z=z, s=s, ds=ds, delta=delta, loss=(per * sw).sum() / B, n_bad=n_bad)
    if u is not None:
        du = torch.where(u > 0, ds, torch.zeros_like(ds)) if p["act_dl"] == "relu" else ds
        out.update(du=du, dh=du[:, None] * p["w_dl"].double()[None, :] * (p["h"] > 0).double())
    return out


def _run_head(p, B, train=True):
    dev = p["y"].device
    f32 = dict(dtype=torch.float32, device=dev)
    U = 0 if p["h"] is None else p["h"].shape[1]
    r = dict(out=torch.zeros(B, **f32), loss=torch.zeros(2, **f32), ds=torch.zeros(B, **f32),
             dh=torch.zeros((B, U), **f32) if U else None, dw_out=torch.zeros(1, **f32), db_out=torch.zeros(1, **f32),
             dw_dl=torch.zeros(U, **f32) if U else None, db_dl=torch.zeros(1, **f32), dbw=torch.zeros(1, **f32),
             oob=torch.zeros(1, dtype=torch.int32, device=dev))
    kw = dict(loss=p["loss"], targets=p["y"], sample_weight=p["sw"], loss_buf=r["loss"], ds=r["ds"], dh=r["dh"], dw_out=r["dw_out"],
              db_out=r["db_out"], dw_dl=r["dw_dl"], db_dl=r["db_dl"] if U else None, d_wide_bias=r["dbw"] if p["wide"] is not None else None) if train else {}
    ops.wide_deep_head_fwd_bwd(p["onehot"], p["bags"], p["wide"], p["bw"], p["h"], True, p["w_dl"], p["b_dl"] if U else None, p["act_dl"],
                               p["out_w"], p["out_b"], r["out"], out_act="sigmoid", oob=r["oob"], **kw)
    torch.cuda.synchronize()
    return r


def _check_head(p, B):
    ref = _head_ref(p, B)
    r = _run_head(p, B)
    close(r["out"], ref["z"], 1e-5, "z")
    close(r["ds"], ref["ds"], 1e-5, "ds")
    close(r["loss"][0], ref["loss"], 1e-5, "loss")
    close(r["loss"][1], r["loss"][0], 1e-6, "the output's loss")
    close(r["dw_out"][0], (ref["delta"] * ref["s"]).sum(), TOL, "dw_out")
    close(r["db_out"][0], ref["delta"].sum(), TOL, "db_out")
    if p["wide"] is not None:
        close(r["dbw"][0], ref["ds"].sum(), TOL, "d_wide_bias")
    if p["h"] is not None:
        close(r["dh"], ref["dh"], 1e-5, "dh")
        close(r["dw_dl"], ref["du"] @ p["h"].double(), TOL, "dw_dl")
        close(r["db_dl"][0], ref["du"].sum(), TOL, "db_dl")
    assert int(r["oob"]) == ref["n_bad"]
    f = _run_head(p, B, train=False)  # forward only: the activated prediction
    close(f["out"], torch.sigmoid(ref["z"]), 1e-5, "forward")
    assert int(f["oob"]) == ref["n_bad"]


@pytest.mark.parametrize("B", [1, 7, 33, 1000])
@pytest.mark.parametrize("shape", ["onehot", "bags", "both"])
def test_head_matches_float64(device, B, shape):
    n_oh = {"onehot": 7, "bags": 0, "both": 5}[shape]
    bags = {"onehot": [], "bags": ["ragged", "fixed", "ragged", "fixed"], "both": ["fixed", "ragged"]}[shape]
    for mode in ("multi_hot", "count"):
        _check_head(_head_case(device, B, n_oh, bags, mode, BCE, True, "linear", 48, seed=B), B)


@pytest.mark.parametrize("loss,sw,act,U", [(MSE, False, "relu", 64), (BCE, False, "relu", 256), (MSE, True, "linear", 512),
                                           (BCE, True, "linear", 30), (BCE, True, "linear", 0)])
def test_head_losses_deep_logits_and_partial_models(device, loss, sw, act, U):
    B = 517
    _check_head(_head_case(device, B, 3, ["ragged"], "multi_hot", loss, sw, act, U, seed=U), B)
    if U:  # pure deep
        _check_head(_head_case(device, B, 0, [], "multi_hot", loss, sw, act, U, seed=U + 1), B)


# ---------------------------------------------------------------------------------------------------------------
# mm_wide_bag_grad + mm_wide_rows_apply
# ---------------------------------------------------------------------------------------------------------------
def _bag_update(device, B, ragged, mode, opt, seed=0):
    g = np.random.default_rng(seed)
    rows, off, W = 37, 11, 60
    if ragged:
        lens = g.integers(0, 9, B)
        offs = np.concatenate([[0], np.cumsum(lens)]) + 2
        v = g.integers(0, rows + 3, int(offs[-1]) + 3)
        x = (v, offs)
        bag = (torch.from_numpy(v).to(device), torch.from_numpy(offs).to(device), rows, off, mode)
    else:
        v = g.integers(0, rows + 3, (B, 6))
        x = v
        bag = (torch.from_numpy(v).to(device), None, rows, off, mode)
    nnz = v.size
    ds = torch.from_numpy(g.standard_normal(B).astype(np.float32)).to(device)
    ids = torch.empty(nnz, dtype=torch.int64, device=device)
    vals = torch.empty(nnz, dtype=torch.float32, device=device)
    ops.wide_bag_grad(bag, B, ds, ids, vals)
    # the expansion's pairs sum to the encoding's gradient E^T ds
    E = encode(x, rows, mode)
    want = E.T @ ds.double().cpu().numpy()
    got = np.zeros(rows)
    i, vv = ids.cpu().numpy(), vals.double().cpu().numpy()
    np.add.at(got, i[i >= 0], vv[i >= 0])
    close(got, want, 1e-5, "expanded gradient")
    assert np.all(vv[i < 0] == 0)
    w = torch.from_numpy(g.standard_normal(W).astype(np.float32)).to(device)
    w0 = w.clone()
    s1 = torch.full((W,), 0.1, device=device) if opt != "sgd" else None
    s2 = torch.zeros(W, device=device) if opt == "adam" else None
    acc = torch.zeros(W, device=device)
    rep = ops.fill_i32(torch.empty(W, dtype=torch.int32, device=device), 2**31 - 1)
    hyper = torch.from_numpy(mm.train.get_optimizer(opt).hyper()).to(device)
    ops.opt_tick(hyper)
    ops.wide_rows_apply(opt, w, s1, s2, [ids], [rows], [off], vals, acc, rep, [], None, None, None, None, hyper)
    torch.cuda.synchronize()
    touched = np.zeros(W, bool)
    touched[off + i[i >= 0]] = True
    assert torch.equal(w[~torch.from_numpy(touched).to(device)], w0[~torch.from_numpy(touched).to(device)]), "untouched rows moved"
    if opt == "sgd":
        lr = float(hyper[0])
        ref = w0.double().cpu().numpy().copy()
        ref[off:off + rows] -= lr * want
        close(w, ref, 1e-6, "sgd update")
    assert float(acc.abs().sum()) == 0 and int((rep != 2**31 - 1).sum()) == 0


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("mode", ["multi_hot", "count"])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_bag_grad_and_update(device, ragged, mode, opt):
    _bag_update(device, 300, ragged, mode, opt)


@pytest.mark.parametrize("B", [65536, 65536 + 37])
def test_head_and_update_at_scale(device, B):
    p = _head_case(device, B, 13, ["fixed", "fixed", "ragged"], "multi_hot", BCE, True, "linear", 256, seed=5)
    _check_head(p, B)
    _bag_update(device, B, False, "multi_hot", "adagrad", seed=1)


# ---------------------------------------------------------------------------------------------------------------
# WideAndDeepTrainer
# ---------------------------------------------------------------------------------------------------------------
def _model(seed, mode="multi_hot", deep=(16, 8), wide=True, deep_on=True, ragged=False):
    mm.set_seed(seed)
    s = schema(lists=LISTS, ragged=ragged)
    ws = s.select_by_name(["C1", "C3", "L2", "L4", "I1"])
    return mm.WideAndDeepModel(s, deep_block=mm.MLPBlock(list(deep)) if deep_on else None, wide_schema=ws if wide else None,
                               wide_preprocess=mm.CategoryEncoding(ws, output_mode=mode) if wide else None,
                               prediction_tasks=mm.BinaryOutput("click"))


def _batch(B, seed, ragged=False):
    g = np.random.default_rng(seed)
    f = {n: g.integers(0, mx + 1, B).astype(np.int64) for n, mx in [("C1", 30), ("C3", 3), ("C5", 400), ("C7", 7)]}
    for n, mx in LISTS:
        if ragged:
            lens = g.integers(1, 6, B)
            f[n + "__values"] = g.integers(0, mx + 1, int(lens.sum())).astype(np.int64)
            f[n + "__offsets"] = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        else:
            v = g.integers(0, mx + 1, (B, 4)).astype(np.int64)
            v[:, 1] = v[:, 0]  # duplicates in every bag
            f[n] = v
    f["I1"] = g.standard_normal(B).astype(np.float32)
    f["I2"] = g.standard_normal(B).astype(np.float32)
    y = g.integers(0, 2, B).astype(np.int64)
    return f, y


def _dev(f, device):
    return {k: torch.from_numpy(v).to(device) for k, v in f.items()}


def _oracle_batch(f):
    out = {k: v for k, v in f.items() if "__" not in k}
    for n in ("L2", "L4"):
        if n + "__values" in f:
            out[n] = (f[n + "__values"], f[n + "__offsets"])
    return out


def _oracle_state(model):
    t = lambda x: x.detach().cpu().numpy()  # noqa: E731
    b = model.body
    wide = deep = None
    if b.wide is not None:
        wide = {"cards": dict(b.wide.cardinalities), "mode": b.wide.mode, "kernel": t(b.wide.dense.kernel), "bias": t(b.wide.dense.bias)}
    if b.input_block is not None:
        emb, cont = b.input_block.embeddings, b.input_block.continuous
        deep = {"tables": {f: t(emb.feature_to_table[f].table) for f in emb.feature_names} if emb is not None else {},
                "continuous": list(cont.features) if cont is not None else [],
                "layers": [{"kernel": t(l.kernel), "bias": t(l.bias), "activation": l.activation} for l in b.deep.dense_layers],
                "logit": {"kernel": t(b.deep_logit.dense_layers[0].kernel), "bias": t(b.deep_logit.dense_layers[0].bias), "activation": "linear"}}
    d = model.prediction.to_call
    head = {"kernel": t(d.kernel), "bias": t(d.bias), "activation": d.activation, "loss": BCE}
    return wide, deep, head


@pytest.mark.parametrize("case", ["multi_hot", "count", "ragged", "wide_only", "deep_only", "one_hot"])
def test_step_gradients_match_the_restatement(device, case):
    mode = {"count": "count", "one_hot": "one_hot"}.get(case, "multi_hot")
    model = _model(3, mode=mode, wide=case != "deep_only", deep_on=case != "wide_only", ragged=case == "ragged")
    if case == "one_hot":
        s = schema(lists=LISTS, ragged=False)
        model = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([16, 8]), wide_schema=s.select_by_name(["C1", "C7"]),
                                    prediction_tasks=mm.BinaryOutput("click"))
    model.build(device)
    model.compile(optimizer="sgd")
    B = 200
    f, y = _batch(B, 9, ragged=case == "ragged")
    sw = np.random.default_rng(1).random(B).astype(np.float32)
    tr = model.trainer(B)
    tr.forward_backward(_dev(f, device), torch.from_numpy(y).to(device), torch.from_numpy(sw).to(device))
    torch.cuda.synchronize()
    wide, deep, head = _oracle_state(model)
    L, z, g = wide_deep_loss_and_grads(_oracle_batch(f), wide, deep, head, y, sample_weight=sw)
    close(tr.loss[0], L, 1e-5, "loss")
    close(tr.logits[:B], z, 1e-4, "logits")
    grads = tr.gradients()
    close(grads[f"{model.prediction.to_call.name}/kernel"], g["head/kernel"], TOL, "head/kernel")
    close(grads[f"{model.prediction.to_call.name}/bias"], g["head/bias"], TOL, "head/bias")
    if deep is not None:
        for i, l in enumerate(model.body.deep.dense_layers):
            close(grads[f"{l.name}/kernel"], g[f"deep/kernel_{i}"], TOL, f"deep/kernel_{i}")
            close(grads[f"{l.name}/bias"], g[f"deep/bias_{i}"], TOL, f"deep/bias_{i}")
        dl = model.body.deep_logit.dense_layers[0]
        close(grads[f"{dl.name}/kernel"], g["deep_logit/kernel"], TOL, "deep_logit/kernel")
        close(grads[f"{dl.name}/bias"], g["deep_logit/bias"], TOL, "deep_logit/bias")
        for t, name in enumerate(tr.feats):  # one-hot tables: scatter the IndexedSlices
            if tr._idx[t] is None:
                continue
            rows = tr.tables[t].table.shape[0]
            dense = torch.zeros((rows, tr.tables[t].table.shape[1]), dtype=torch.float64, device=device)
            dense.index_add_(0, tr._idx[t].long(), tr._slices[t].double())
            close(dense, g[f"table/{name}"], TOL, f"table/{name}")
    if wide is not None:
        wg = tr.wide_gradients()
        close(wg["wide/kernel"], g["wide/kernel"], TOL, "wide/kernel")
        close(wg["wide/bias"], g["wide/bias"], TOL, "wide/bias")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_update_only_touched_wide_rows(device, opt):
    """Three steps: the loss is finite and falls on a repeated batch, wide rows no batch touches keep their bits, and the
    first SGD step moves the wide kernel by -lr times the restatement's gradient."""
    model = _model(5)
    model.build(device)
    model.compile(optimizer={"sgd": mm.SGD(0.5), "adagrad": mm.Adagrad(0.1), "adam": mm.Adam(0.01)}[opt])
    B = 256
    f, y = _batch(B, 11)
    wk0 = model.body.wide.dense.kernel.clone()
    wide, deep, head = _oracle_state(model)
    _, _, g = wide_deep_loss_and_grads(_oracle_batch(f), wide, deep, head, y)
    losses = []
    for s in range(3):
        losses.append(float(model.train_step((_dev(f, device), torch.from_numpy(y).to(device)))["loss"]))
        if s == 0 and opt == "sgd":
            close(model.body.wide.dense.kernel.double() - wk0.double(), -0.5 * g["wide/kernel"], 1e-4, "first SGD step")
    assert np.all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    untouched = torch.from_numpy(g["wide/kernel"].reshape(-1) == 0).to(device)
    assert torch.equal(model.body.wide.dense.kernel.reshape(-1)[untouched], wk0.reshape(-1)[untouched])


def test_graph_replay_equals_eager_steps(device):
    ma, mb = _model(12), _model(12)
    ma.build(device), mb.build(device)
    ma.compile(optimizer=mm.Adagrad(0.05))
    mb.compile(optimizer=mm.Adagrad(0.05))
    B = 256
    batches = [_batch(B, 20 + s) for s in range(3)]
    ta, tb = ma.trainer(B), mb.trainer(B)
    w0 = mb.body.wide.dense.kernel.clone()
    tb.capture(_dev(batches[0][0], device), torch.from_numpy(batches[0][1]).to(device))
    assert torch.equal(mb.body.wide.dense.kernel, w0), "capture moved the wide kernel"
    for f, y in batches:
        la = ta.step(_dev(f, device), torch.from_numpy(y).to(device)).clone()
        lb = tb.replay(_dev(f, device), torch.from_numpy(y).to(device)).clone()
        close(la, lb, 1e-5, "loss")
    for (na, va), (nb, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(va, vb, 1e-4, na)
    fr, yr = _batch(B, 3, ragged=True)
    mc = _model(13, ragged=True)
    mc.build(device)
    mc.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="ragged"):
        mc.trainer(B).capture(_dev(fr, device), torch.from_numpy(yr).to(device))


def test_trained_model_forward_evaluate_save_load_compile(device, tmp_path):
    from models_b200.graph import HostBatch

    model = _model(4)
    model.compile(optimizer=mm.Adam(0.01))
    for s in range(3):
        f, y = _batch(256, 40 + s)
        model.train_step((_dev(f, device), torch.from_numpy(y).to(device)))
    f, y = _batch(256, 50)
    p = model(_dev(f, device)).reshape(-1)
    wide, deep, head = _oracle_state(model)
    close(p, wide_deep_forward(_oracle_batch(f), wide, deep, head), 2e-4, "forward vs the oracle")
    res = model.evaluate([(_dev(f, device), torch.from_numpy(y).to(device))], return_dict=True)
    zz = wide_deep_forward(_oracle_batch(f), wide, deep, head, logits=True)
    bce = float(np.mean(np.maximum(zz, 0) - zz * y + np.log1p(np.exp(-np.abs(zz)))))
    assert abs(res["loss"] - bce) < 1e-3 * max(1.0, bce), (res, bce)
    hb = HostBatch.like(f, model.input_columns())
    cf = model.compile(hb)
    close(np.asarray(cf(hb)).reshape(-1), p.cpu().numpy(), 1e-5, "compiled forward")
    model.save(tmp_path / "export")
    loaded = mm.Model.load(tmp_path / "export")
    np.testing.assert_array_equal(loaded(_dev(f, device)).cpu().numpy().reshape(-1), p.cpu().numpy())
    mr = _model(4, ragged=True)
    mr.build(device)
    fr, _ = _batch(64, 51, ragged=True)
    close(mr(_dev(fr, device)).reshape(-1), wide_deep_forward(_oracle_batch(fr), *_oracle_state(mr)), 2e-4, "ragged forward")


def test_out_of_range_wide_ids_raise(device):
    """Without a deep part no embedding lookup sees the ids: the wide head alone bumps the counter the forward checks."""
    model = _model(6, deep_on=False)
    model.build(device)
    f, _ = _batch(32, 1)
    model(_dev(f, device))
    f["L4"][3, 2] = 261  # cardinality 261: id 261 is out of range
    with pytest.raises(IndexError):
        model(_dev(f, device))


@pytest.mark.parametrize("mode", ["multi_hot", "count"])
def test_pure_wide_model_trains(device, mode):
    """deep_block=None: eager SGD steps move the wide kernel, its bias and the output layer by -lr times the restatement's
    gradients, and a captured graph replays the same steps."""
    ma, mb = _model(14, mode=mode, deep_on=False), _model(14, mode=mode, deep_on=False)
    for m in (ma, mb):
        m.build(device)
        m.compile(optimizer=mm.SGD(0.5))
    B = 128
    batches = [_batch(B, 60 + s) for s in range(3)]
    tb = mb.trainer(B)
    tb.capture(_dev(batches[0][0], device), torch.from_numpy(batches[0][1]).to(device))
    for f, y in batches:
        wide, _, head = _oracle_state(ma)
        L, _, g = wide_deep_loss_and_grads(_oracle_batch(f), wide, None, head, y)
        la = ma.train_step((_dev(f, device), torch.from_numpy(y).to(device)))["loss"]
        close(la, L, 1e-5, "loss")
        close(ma.body.wide.dense.kernel.double(), wide["kernel"] - 0.5 * g["wide/kernel"], 1e-5, "wide kernel")
        close(ma.body.wide.dense.bias.double(), wide["bias"] - 0.5 * g["wide/bias"], 1e-5, "wide bias")
        d = ma.prediction.to_call
        close(d.kernel.double(), head["kernel"] - 0.5 * g["head/kernel"], 1e-5, "output kernel")
        close(d.bias.double(), head["bias"] - 0.5 * g["head/bias"], 1e-5, "output bias")
        close(tb.replay(_dev(f, device), torch.from_numpy(y).to(device))[0], la, 1e-5, "replayed loss")
    for (na, va), (nb, vb) in zip(sorted(ma.weights().items()), sorted(mb.weights().items())):
        close(va, vb, 1e-5, na)


def test_continuous_only_deep_model(device):
    """A deep part over continuous columns only and no wide part has no ids to count: the forward and a step run."""
    s = schema(lists=LISTS, ragged=False)
    with pytest.warns(UserWarning):
        model = mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), deep_schema=s.select_by_name(["I1", "I2", "click"]),
                                    prediction_tasks=mm.BinaryOutput("click"))
    model.build(device)
    model.compile(optimizer="sgd")
    f, y = _batch(64, 2)
    p = model(_dev(f, device)).reshape(-1)
    close(p, wide_deep_forward(_oracle_batch(f), *_oracle_state(model)), 2e-4, "forward")
    L = model.train_step((_dev(f, device), torch.from_numpy(y).to(device)))["loss"]
    assert np.isfinite(float(L))


def test_fit_learns_a_planted_rule(device):
    """The reference's multi-hot example trains with compile(optimizer="adam") and fit: clicks follow whether a bag holds
    an even id of L4."""
    model = _model(8)
    model.compile(optimizer="adam")
    data = []
    for s in range(20):
        f, _ = _batch(1000, 100 + s)
        rule = (f["L4"] % 2 == 0).any(axis=1)
        y = (np.random.default_rng(s).random(1000) < np.where(rule, 0.9, 0.1)).astype(np.int64)
        data.append((_dev(f, device), torch.from_numpy(y).to(device)))
    hist = model.fit(data, epochs=10).history["loss"]
    assert hist[-1] < 0.75 * hist[0], hist


def test_unsupported_training_configurations(device):
    s = schema(lists=LISTS, ragged=False)
    ws = s.select_by_name(["C1"])
    cases = [(mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, deep_dropout=0.1), "dropout"),
             (mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, wide_dropout=0.1), "wide_dropout"),
             (mm.WideAndDeepModel(s, deep_block=mm.MLPBlock([8]), wide_schema=ws, deep_regularizer="l2"), "regularizers")]
    for m, match in cases:
        m.build(device)
        m.compile(optimizer="sgd")
        with pytest.raises(NotImplementedError, match=match):
            m.trainer(16)
    m = _model(2)
    m.build(device)
    m.compile(optimizer="sgd")
    mm.set_dense_engine("fp32")
    try:
        with pytest.raises(NotImplementedError, match="fp32"):
            m.trainer(16)
    finally:
        mm.set_dense_engine("auto")
