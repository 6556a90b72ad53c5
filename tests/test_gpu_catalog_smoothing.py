"""Label-smoothed full-catalog soft-max cross-entropy on the GPU (mm_catalog_smoothed_ce_backward,
inbatch_flash_kernel<SmoothedCatalogCE, DQ / DN>, mm_catalog_mean_logit): dx, dE, db and the loss against float64 over
the unsmoothed kernels' grid at eps = 0.1 and 0.3, eps = 0 bit-identical to the unsmoothed call, bit-identical repeats,
out-of-range labels, the 10 M x 64 catalog; and the session-based example's model trained with label_smoothing=0.1,
logits_temperature=0.05 and Adam: one step against float64, fit / fit(validation_data) / evaluate / save / load, a
planted next-item rule with dropout=0.2 in the MLP, and evaluate's loss against the float64 smoothed loss of the
materialised logits (dropout is identity outside training)."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops
from oracle import oracle
from tests import catalog_model_oracle as O
from tests.catalog_smoothing_oracle import smoothed_catalog_ce, smoothed_restated_step
from tests.test_gpu_catalog_train import CASES, EPS_SPLIT, bounds, dev

pytestmark = pytest.mark.gpu


def run(device, x, E, b, y, T, sw, eps, label_dtype=torch.int64, oob=None):
    """As test_gpu_catalog_train.run, with label_smoothing = eps."""
    B, D = x.shape
    N = E.shape[0]
    xt = dev((x / np.float32(T)).astype(np.float32) if T != 1.0 else x, device)
    bt = None if b is None else dev((b / np.float32(T)).astype(np.float32) if T != 1.0 else b, device)
    labels = dev(y, device).to(label_dtype)
    e_split = ops.split_rows(dev(E, device))
    stats, _, _ = ops.catalog_score(xt, e_split, N, bias=bt, targets=labels, k=0)
    c = dev((np.ones(B, np.float32) if sw is None else sw.astype(np.float32)) / np.float32(B), device)
    dx = torch.full((B, D), float("nan"), device=device)
    de = torch.full((N, D), float("nan"), device=device)
    db = torch.full((N,), float("nan"), device=device) if b is not None else None
    loss = torch.zeros(1, device=device)
    ops.catalog_softmax_ce_backward(ops.split_rows(xt), e_split, D, stats, labels, c, dx, de, db=db, bias=bt, loss=loss,
                                    temperature=T, oob=oob, label_smoothing=eps)
    return stats, loss, dx, de, db


def smooth_bounds(x, E, b, y, T, sw, eps, lse):
    """The unsmoothed error model (keep <= 1, so its |G| bounds still hold) plus the rank-one terms' own: the column
    sums read the split operands (hi + lo: EPS_SPLIT / 2 of each element) and add in fp32 / double."""
    ex, ee, eb = bounds(x, E, b, y, T, sw, lse)
    B, N = x.shape[0], E.shape[0]
    c = (np.ones(B) if sw is None else sw.astype(np.float64)) / B
    aE, ax = np.abs(E.astype(np.float64)).sum(0), np.abs(x.astype(np.float64))
    ex = ex + 4 * EPS_SPLIT * (eps / N) * np.outer(c, aE) / T + 1e-12
    ee = ee + 4 * EPS_SPLIT * (eps / (N * T)) * (c @ ax)[None, :] + 1e-12
    eb = eb + 4 * 2.0 ** -22 * (eps / (N * T)) * c.sum() + 1e-12
    return ex, ee, eb


@pytest.mark.parametrize("eps", [0.1, 0.3])
@pytest.mark.parametrize("B,N,D,T,use_bias,weights,label_dtype", CASES)
def test_smoothed_backward_against_float64(device, B, N, D, T, use_bias, weights, label_dtype, eps):
    rng = np.random.default_rng(B * 7 + N + D)
    x = (rng.standard_normal((B, D)) * (0.3 if T < 1 else 1.0)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.5 / np.sqrt(D / 16)).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32) if use_bias else None
    y = rng.integers(0, N, B).astype(np.int64)
    y[: min(B, 2)] = [0, N - 1][: min(B, 2)]
    sw = rng.uniform(0.2, 2.0, B).astype(np.float32) if weights else None
    stats, loss, dx, de, db = run(device, x, E, b, y, T, sw, eps, label_dtype)
    lse = stats[:, 1].double().cpu().numpy()
    rl, rdx, rde, rdb = smoothed_catalog_ce(x, E, b, y, T, eps, sw)
    ex, ee, eb = smooth_bounds(x, E, b, y, T, sw, eps, lse)
    for name, got, ref, bound in (("dx", dx, rdx, ex), ("dE", de, rde, ee)):
        err = np.abs(got.double().cpu().numpy() - ref)
        worst = np.unravel_index(np.argmax(err / bound), err.shape)
        assert np.all(err <= bound), f"{name}: |err| {err[worst]:.3e} > bound {bound[worst]:.3e} at {worst}"
    if use_bias:
        err = np.abs(db.double().cpu().numpy() - rdb)
        assert np.all(err <= eb), f"db: max |err| / bound {np.max(err / eb):.3f}"
    assert abs(loss.item() - rl) <= 1e-5 * max(1.0, abs(rl)) + 3e-4 * max(1.0, 1 / T) * np.sqrt(D / 64)


@pytest.mark.parametrize("B,N,D", [(200, 100_003, 64), (4096 + 37, 3000, 128)])
def test_eps_zero_is_the_unsmoothed_call_bit_for_bit(device, B, N, D):
    """label_smoothing=0.0 through ops and through mm_catalog_smoothed_ce_backward give exactly the unsmoothed outputs."""
    rng = np.random.default_rng(13)
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.25).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32)
    y = rng.integers(0, N, B)
    ref = run(device, x, E, b, y, 0.5, None, 0.0)
    from tests.test_gpu_catalog_train import run as run_plain

    plain = run_plain(device, x, E, b, y, 0.5, None)
    for a, c in zip(ref, plain):
        assert torch.equal(a, c)
    # the C entry point with eps = 0 and the unsmoothed workspace
    stats, _, _, _, _ = plain
    xt, bt = dev(x / np.float32(0.5), device), dev(b / np.float32(0.5), device)
    labels = dev(y, device)
    c = torch.full((1,), 1.0 / B, device=device)
    dx, de, db = torch.empty((B, D), device=device), torch.empty((N, D), device=device), torch.empty(N, device=device)
    loss = torch.zeros(1, device=device)
    ws = torch.empty(max(16, ops.catalog_softmax_ce_workspace_bytes(B, N, D)), dtype=torch.uint8, device=device)
    xs, es = ops.split_rows(xt), ops.split_rows(dev(E, device))
    _cabi.check(ops._lib().mm_catalog_smoothed_ce_backward(
        xs.data_ptr(), es.data_ptr(), B, N, D, bt.data_ptr(), labels.data_ptr(), _cabi.MM_I64, 0.5, 0.0, stats.data_ptr(),
        c.data_ptr(), 1, dx.data_ptr(), de.data_ptr(), db.data_ptr(), loss.data_ptr(), None, ws.data_ptr(), ws.numel(),
        ops._stream()), "mm_catalog_smoothed_ce_backward")
    for a, r in zip((loss, dx, de, db), plain[1:]):
        assert torch.equal(a, r)


def test_smoothed_repeats_bit_identical(device):
    """Split dq path, the dn kernel and the column sums: fixed summation order."""
    rng = np.random.default_rng(11)
    B, N, D = 200, 100_003, 64
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.25).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32)
    y = rng.integers(0, N, B)
    sw = rng.uniform(0.2, 2.0, B).astype(np.float32)
    assert ops.catalog_softmax_ce_workspace_bytes(B, N, D) > 0  # the split path
    first = run(device, x, E, b, y, 0.5, sw, 0.1)
    for _ in range(2):
        again = run(device, x, E, b, y, 0.5, sw, 0.1)
        for a, c in zip(first, again):
            assert torch.equal(a, c)


def test_smoothed_out_of_range_labels(device):
    """The unsmoothed rule (no one-hot term, counted once per row, NaN loss) with the uniform term kept."""
    rng = np.random.default_rng(12)
    B, N, D = 130, 500, 64
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.3).astype(np.float32)
    y = rng.integers(0, N, B)
    y[[0, 5, 129]] = [N, -1, 1 << 40]
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    stats, loss, dx, de, db = run(device, x, E, None, y, 1.0, None, 0.2, oob=oob)
    assert oob.item() == 3 and np.isnan(loss.item())
    run(device, x[:1], E, None, y[:1], 1.0, None, 0.2, oob=oob)  # one query tile, the catalog split over several CTAs
    assert oob.item() == 4
    _, rdx, rde, _ = smoothed_catalog_ce(x, E, None, y, 1.0, 0.2)
    ex, ee, _ = smooth_bounds(x, E, None, y, 1.0, None, 0.2, stats[:, 1].double().cpu().numpy())
    assert np.all(np.abs(dx.double().cpu().numpy() - rdx) <= ex)
    assert np.all(np.abs(de.double().cpu().numpy() - rde) <= ee)


@pytest.mark.parametrize("B,N,D,use_bias", [(1, 1, 4, True), (300, 100_003, 60, True), (4133, 3000, 128, False)])
def test_mean_logit_against_float64(device, B, N, D, use_bias):
    rng = np.random.default_rng(B + N)
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32) if use_bias else None
    got = ops.catalog_mean_logit(ops.split_rows(dev(x, device)), ops.split_rows(dev(E, device)), D,
                                 bias=None if b is None else dev(b, device)).double().cpu().numpy()
    xd, Ed = x.astype(np.float64), E.astype(np.float64)
    want = (xd @ Ed.sum(0) + (0.0 if b is None else b.astype(np.float64).sum())) / N
    bound = 4 * EPS_SPLIT * (np.abs(xd) @ np.abs(Ed).sum(0) + (0.0 if b is None else np.abs(b).sum())) / N + 1e-7
    assert np.all(np.abs(got - want) <= bound)


def test_catalog_10m_sampled_rows_smoothed(device):
    """10 M x 64 catalog with B = 4096 (the split dq shape) at eps = 0.1: dE and db of sampled catalog rows and dx of
    sampled queries against float64 over the hash-initialised table, s_E summed over all 10 M rows on the host."""
    I, D, B, eps = 10_000_000, 64, 4096, 0.1
    rng = np.random.default_rng(21)
    E = torch.empty((I, D), dtype=torch.float32, device=device)
    ops.init_uniform_hash(E, 77, -0.5, 0.5)
    bias = torch.empty((I, 1), dtype=torch.float32, device=device)
    ops.init_uniform_hash(bias, 78, -0.2, 0.2)
    bias = bias.reshape(-1)
    x = (rng.standard_normal((B, D)) * 0.5).astype(np.float32)
    y = rng.integers(0, I, B).astype(np.int64)
    rows = np.array([0, 1, 127, 128, 5_000_000, I - 1] + list(y[:4]), dtype=np.int64)
    y[4:6] = [0, I - 1]
    e_split = ops.split_rows(E)
    labels = dev(y, device)
    stats, _, _ = ops.catalog_score(dev(x, device), e_split, I, bias=bias, targets=labels, k=0)
    c = torch.full((1,), 1.0 / B, device=device)
    dx = torch.empty((B, D), device=device)
    de = torch.empty((I, D), device=device)
    db = torch.empty(I, device=device)
    loss = torch.zeros(1, device=device)
    ops.catalog_softmax_ce_backward(ops.split_rows(dev(x, device)), e_split, D, stats, labels, c, dx, de, db=db, bias=bias,
                                    loss=loss, label_smoothing=eps)
    lse = stats[:, 1].double().cpu().numpy()
    xd = x.astype(np.float64)
    Er = oracle.hash_table_rows(rows, D, 77, -0.5, 0.5).astype(np.float64)
    br = bias[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    G = (np.exp(xd @ Er.T + br[None, :] - lse[:, None]) - (1 - eps) * (y[:, None] == rows[None, :])) / B
    r = (eps / I) * xd.mean(0)  # (eps / N) sum_b c_b x_b with c = 1 / B
    ridx = torch.from_numpy(rows).to(device)
    err = np.abs(de[ridx].double().cpu().numpy() - (G.T @ xd - r[None, :]))
    assert np.all(err <= 1e-3 * (np.abs(G).T @ np.abs(xd)) + 1e-3 * np.abs(r)[None, :] + 1e-12)
    err = np.abs(db[ridx].double().cpu().numpy() - (G.sum(axis=0) - eps / I))
    assert np.all(err <= 1e-3 * (np.abs(G).sum(axis=0) + eps / I) + 1e-12)
    qs = [0, 1, 4, 5, 2047, 4095]
    acc, s_E, beta = np.zeros((len(qs), D)), np.zeros(D), 0.0
    bias_h = bias.double().cpu().numpy()
    step = 1_000_000
    for r0 in range(0, I, step):
        rr = np.arange(r0, min(I, r0 + step))
        blk = oracle.hash_table_rows(rr, D, 77, -0.5, 0.5).astype(np.float64)
        p = np.exp(xd[qs] @ blk.T + bias_h[rr][None, :] - lse[qs][:, None])
        acc += p @ blk
        s_E += blk.sum(0)
        beta += bias_h[rr].sum()
    acc -= (1 - eps) * oracle.hash_table_rows(y[qs], D, 77, -0.5, 0.5).astype(np.float64)
    acc -= (eps / I) * s_E[None, :]
    np.testing.assert_allclose(dx[qs].double().cpu().numpy(), acc / B, rtol=0, atol=2e-7)
    tl = stats[:, 2].double().cpu().numpy()
    want_loss = np.mean(lse - (1 - eps) * tl - (eps / I) * (xd @ s_E + beta))
    assert abs(loss.item() - want_loss) <= 1e-4 * max(1.0, abs(want_loss))


# ---------------------------------------------------------------------------------------------------------------
# the session-based example's model
# ---------------------------------------------------------------------------------------------------------------
def dev_batch(feats, labels, device):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in feats.items()}, torch.from_numpy(labels).to(device)


def smoothed(eps):
    return mm.losses.CategoricalCrossEntropy(from_logits=True, label_smoothing=eps)


@pytest.mark.parametrize("tied,T,weights", [("onehot", 0.05, True), ("list", 1.0, False), ("none", 0.05, False)])
def test_step_against_smoothed_restatement(device, tied, T, weights):
    """One CatalogTrainer step with label_smoothing=0.1: the loss, the MLP's gradients, the tied dE and db against
    torch autograd of F.cross_entropy(label_smoothing=0.1) over the float64 restatement."""
    from tests.test_gpu_catalog_model import close

    n_items, D, B, eps = 700, 32, 300, 0.1
    model, s, table = O.build(n_items, D, tied, widths=(48,), T=T)
    model.build(device)
    model.prediction.bias.copy_(torch.randn(n_items, generator=torch.Generator().manual_seed(1)).to(device) * 0.3)
    feats, y = O.batch(s, n_items, B, seed=3, hot=5)
    sw = np.random.default_rng(4).uniform(0.2, 2.0, B).astype(np.float32) if weights else None
    want_loss, want, _ = smoothed_restated_step(model, feats, y, eps, sw)
    model.compile(optimizer=mm.SGD(0.1), loss=smoothed(eps))
    tr = model.trainer(B)
    x, yt = dev_batch(feats, y, device)
    tr.forward_backward(x, [yt], None if sw is None else torch.from_numpy(sw).to(device))
    torch.cuda.synchronize()
    assert abs(tr.loss[0].item() - want_loss) <= 2e-4 * max(1.0, abs(want_loss), 1.0 / T)
    g = tr.gradients()
    for i, l in enumerate(model.mlp.dense_layers):
        close(g[f"{l.name}/kernel"], want[f"mlp/{i}/kernel"], f"mlp {i} kernel")
        close(g[f"{l.name}/bias"], want[f"mlp/{i}/bias"], f"mlp {i} bias")
    close(tr.wk.dE, want["tables/item_id"], "tied dE", rtol=5e-3)
    close(tr.wk.db, want["bias"], "db", rtol=5e-3)


def test_three_steps_graph_replay_bit_identical_smoothed(device):
    """Eager steps and one captured graph's replays from the same state: the column sums and the smoothed kernels are
    fixed-order, so the first step's loss, tied table and bias are bit-identical (the later ones differ by the MLP's
    wgrad atomics only, as without smoothing)."""
    n_items, D, B = 900, 64, 256
    batches = [O.batch(O.schema(n_items, "list", n_users=300_000), n_items, B, seed=10 + i, hot=3) for i in range(3)]
    runs = []
    for graph in (False, True):
        model, s, table = O.build(n_items, D, "list", T=0.05, seed=5, n_users=300_000)
        model.build(device)
        model.compile(optimizer=mm.Adam(0.01, epsilon=1e-3), loss=smoothed(0.1))
        tr = model.trainer(B)
        losses = []
        for i, (f, y) in enumerate(batches):
            x, yt = dev_batch(f, y, device)
            if not graph:
                losses.append(tr.step(x, [yt])[0].clone())
            else:
                if i == 0:
                    tr.capture(x, [yt])
                losses.append(tr.replay(x, [yt])[0].clone())
            if i == 0:
                first = (table.table.clone(), model.prediction.bias.clone())
        runs.append((losses, first, table.table.clone()))
    (la, fa, ea), (lb, fb, eb) = runs
    assert torch.equal(la[0], lb[0]) and torch.equal(fa[0], fb[0]) and torch.equal(fa[1], fb[1])
    for a, b in zip(la, lb):
        assert abs(a.item() - b.item()) <= 1e-6 * abs(a.item())
    assert (ea - eb).abs().max().item() <= 1e-6 * ea.abs().max().item()


def planted(s, n_items, B, seed):
    """Batches whose next item is a fixed function of the last item: next = (3 last + 1) mod n_items."""
    f, _ = O.batch(s, n_items, B, seed=seed)
    return f, ((3 * f["last_item"] + 1) % n_items).astype(np.int64)


def test_example_model_fit_evaluate_save_load(device, tmp_path):
    """The example's Model(InputBlockV2, MLPBlock([128, D], no_activation_last_layer=True, dropout=0.2), CategoricalOutput(table,
    logits_temperature=0.05)) compiled with Adam and CategoricalCrossEntropy(from_logits=True, label_smoothing=0.1):
    fit with validation data learns the planted rule, evaluate's loss is the float64 smoothed loss of the materialised
    logits, and save / load keeps the model."""
    n_items, D, B, eps, T = 400, 32, 256, 0.1, 0.05
    mm.set_seed(3)
    s = O.schema(n_items, "onehot")
    emb = mm.Embeddings(s.select_by_tag(mm.Tags.CATEGORICAL), dim=D)
    ib = mm.InputBlockV2(s, categorical=emb)
    mlp = mm.MLPBlock([128, D], no_activation_last_layer=True, dropout=0.2)
    out = mm.CategoricalOutput(to_call=emb.tables["item_id"], logits_temperature=T, target_name="next_item")
    model = mm.Model(ib, mlp, out)
    model.compile(optimizer=mm.Adam(0.005), loss=smoothed(eps))
    data = [dev_batch(*planted(s, n_items, B, seed=100 + i), device) for i in range(8)]
    val = [dev_batch(*planted(s, n_items, B, seed=200 + i), device) for i in range(2)]
    hist = model.fit(data, epochs=12, validation_data=val)
    h = hist.history
    assert len(h["loss"]) == 12 and h["loss"][-1] < 0.5 * h["loss"][0]
    assert "val_loss" in h and h["val_recall_at_10"][-1] > 0.5, h["val_recall_at_10"]  # chance: 10 / 400
    res = model.evaluate(val, return_dict=True)
    assert res["recall_at_10"] == h["val_recall_at_10"][-1] and abs(res["loss"] - h["val_loss"][-1]) <= 1e-6 * abs(res["loss"])
    # float64 smoothed loss of the materialised logits (the model's call is without the temperature)
    rows, loss = 0, 0.0
    for x, y in val:
        z = model(x).double().cpu().numpy() / T
        yy = y.cpu().numpy()
        m = z.max(1, keepdims=True)
        lse = m[:, 0] + np.log(np.exp(z - m).sum(1))
        loss += float(np.sum(lse - (1 - eps) * z[np.arange(len(yy)), yy] - eps * z.mean(1)))
        rows += len(yy)
    assert abs(res["loss"] - loss / rows) <= 1e-4 * max(1.0, loss / rows)
    x, _ = val[0]
    z0 = model(x)
    model.save(tmp_path / "m")
    loaded = mm.Model.load(tmp_path / "m")
    assert torch.equal(loaded(x), z0)
    loaded.compile(optimizer="adam", loss=smoothed(eps))
    assert loaded.evaluate(val, return_dict=True) == res
    loaded.compile(optimizer="adam")  # unsmoothed: eps (z[y] - mean z) less per row, positive on a confident model
    assert loaded.evaluate(val, return_dict=True)["loss"] < res["loss"]


def test_smoothed_out_of_range_label_raises(device):
    n_items, B = 300, 64
    model, s, _ = O.build(n_items, 16, "onehot")
    model.compile(optimizer="sgd", loss=smoothed(0.1))
    f, y = O.batch(s, n_items, B)
    y[5] = n_items
    with pytest.raises(IndexError):
        model.fit([dev_batch(f, y, device)], epochs=1)
    with pytest.raises(IndexError):
        model.evaluate([dev_batch(f, y, device)])
