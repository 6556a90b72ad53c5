"""Model(InputBlockV2, MLPBlock, CategoricalOutput) on the GPU: mm_slices_add_dense against float64, one CatalogTrainer step
against the float64 restatement (tests/catalog_model_oracle.py) for one-hot, list and absent tied features, bias on and
off, T = 1 and 0.05 and sample weights; three steps eager against one CUDA graph's replays under every optimizer; fit -> evaluate -> save -> load; an out-of-range label; and sampled rows at the benchmark's sizes."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import ops
from tests import catalog_model_oracle as O

pytestmark = pytest.mark.gpu


def dev_batch(feats, labels, device):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in feats.items()}, torch.from_numpy(labels).to(device)


# ---------------------------------------------------------------------------------------------------------------
# the row merge
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,N,D,dt", [(1, 1, 4, torch.int32), (1000, 37, 64, torch.int64), (5000, 300_000, 60, torch.int32),
                                      (40_000, 1_000_000, 128, torch.int64), (20_000, 10, 16, torch.int64),
                                      (300_000, 1_000_000, 64, torch.int32)])
def test_slices_add_dense_against_float64(device, n, N, D, dt):
    """Runs of every length: the largest case pads half its ids with 0 (a 150 000-long run over ~590 chunks) and repeats
    a few popular ids, so runs inside one chunk, across two and across hundreds all occur."""
    g = torch.Generator().manual_seed(n + N)
    ids = torch.randint(0, N, (n,), generator=g)
    if n >= 100_000:
        ids[torch.rand(n, generator=g) < 0.5] = 0
        ids[torch.rand(n, generator=g) < 0.01] = 7
        ids[torch.rand(n, generator=g) < 0.001] = N - 1
    ids[: min(n, 3)] = torch.tensor([-1, N, 0])[: min(n, 3)]  # outside [0, N): add nothing
    rows = torch.randn(n, D, generator=g)
    base = torch.randn(N, D, generator=g)
    want = base.double().clone()
    ok = (ids >= 0) & (ids < N)
    want.index_add_(0, ids[ok], rows[ok].double())
    dense = base.to(device)
    ops.slices_add_dense(ids.to(dt).to(device), rows.to(device), dense)
    cnt = torch.zeros(N, dtype=torch.float64).index_add_(0, ids[ok], torch.ones(int(ok.sum()), dtype=torch.float64))
    bound = 2.0 ** -22 * (cnt + 1).sqrt().unsqueeze(1) * 8 * (base.double().abs() + torch.zeros(N, D, dtype=torch.float64).index_add_(
        0, ids[ok], rows[ok].double().abs()))
    assert torch.all((dense.cpu().double() - want).abs() <= bound + 1e-30)
    again = base.to(device)
    ops.slices_add_dense(ids.to(dt).to(device), rows.to(device), again)
    assert torch.equal(dense, again)  # duplicates in index order, no atomics


# ---------------------------------------------------------------------------------------------------------------
# one step against the restatement
# ---------------------------------------------------------------------------------------------------------------
def close(got, want, name, rtol=2e-3):
    """The MLP's gradients: within rtol of the tensor's largest entry (their rounding is the tensor-core chain's)."""
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    scale = max(np.abs(want).max(), 1e-12)
    err = np.abs(got - want)
    assert np.all(err <= rtol * scale + 1e-3 * np.abs(want)), f"{name}: max |err| {err.max():.3e}, scale {scale:.3e}"


K_TERMS = 1e-2  # split-bf16 scores at T = 0.05 move G by up to ~1e-3 of |G| (test_gpu_catalog_train.py's error model), and x
# carries the tensor-core chain's rounding; FLOOR: fp32 resolution of the tensor's largest entry


def check_tied(model, feats, y, sw, tr, want_dE, want_db):
    """dE and db per element: |err| <= K_TERMS (|G|^T |x| / T + |input-side rows|) for dE, K_TERMS sum_b |G| / T for db,
    plus 1e-6 of the tensor's largest entry — a row no lookup touched is held to its own output-side magnitude."""
    x, aG, adE, adb = O.restated_terms(model, feats, y, sw)
    T = model.prediction.logits_temperature
    got = tr.wk.dE.double().cpu().numpy()
    inp = np.abs(want_dE - _output_side(model, feats, y, sw))
    bound = K_TERMS * (adE + inp) + 1e-6 * np.abs(want_dE).max()
    err = np.abs(got - want_dE)
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert np.all(err <= bound), f"dE: |err| {err[worst]:.3e} > bound {bound[worst]:.3e} at {worst} (T = {T})"
    if want_db is not None:
        gb = tr.wk.db.double().cpu().numpy()
        eb = K_TERMS * adb + 1e-6 * np.abs(want_db).max()
        assert np.all(np.abs(gb - want_db) <= eb), f"db: max |err| / bound {np.max(np.abs(gb - want_db) / eb):.3f}"


def _output_side(model, feats, y, sw):
    """G^T x / T in float64 (the tied gradient without the input side)."""
    from tests.catalog_train_oracle import catalog_ce

    out = model.prediction
    b = None if out.bias is None else out.bias.detach().cpu().numpy()
    return catalog_ce(O.restated_query(model, feats), out.table.table.detach().cpu().numpy(), b, y, out.logits_temperature, sw)[2]


CASES = [  # tied, T, bias, weights, combiner
    ("onehot", 1.0, True, False, "mean"),
    ("onehot", 0.05, False, True, "mean"),
    ("list", 0.05, True, True, "mean"),
    ("list", 1.0, False, False, "sum"),
    ("none", 0.05, True, False, "mean"),
    ("none", 1.0, False, True, "mean"),
]


@pytest.mark.parametrize("tied,T,use_bias,weights,comb", CASES)
def test_step_against_restatement(device, tied, T, use_bias, weights, comb):
    n_items, D, B = 700, 32, 300
    model, s, table = O.build(n_items, D, tied, widths=(48,), T=T, use_bias=use_bias, combiner=comb)
    model.build(device)
    if use_bias:
        model.prediction.bias.copy_(torch.randn(n_items, generator=torch.Generator().manual_seed(1)).to(device) * 0.3)
    feats, y = O.batch(s, n_items, B, seed=3, hot=5)
    sw = np.random.default_rng(4).uniform(0.2, 2.0, B).astype(np.float32) if weights else None
    want_loss, want = O.restated_step(model, feats, y, sw)
    model.compile(optimizer=mm.SGD(0.1))
    tr = model.trainer(B)
    x, yt = dev_batch(feats, y, device)
    tr.forward_backward(x, [yt], None if sw is None else torch.from_numpy(sw).to(device))
    torch.cuda.synchronize()
    assert abs(tr.loss[0].item() - want_loss) <= 2e-4 * max(1.0, abs(want_loss), 1.0 / T)
    g = tr.gradients()
    for i, l in enumerate(model.mlp.dense_layers):
        close(g[f"{l.name}/kernel"], want[f"mlp/{i}/kernel"], f"mlp {i} kernel")
        close(g[f"{l.name}/bias"], want[f"mlp/{i}/bias"], f"mlp {i} bias")
    check_tied(model, feats, y, sw, tr, want["tables/item_id"], want["bias"] if use_bias else None)
    ids, rows = tr.table_gradients()["user_id"]
    du = torch.zeros(O.N_USERS, D, dtype=torch.float64).index_add_(0, ids.cpu().long(), rows.cpu().double())
    close(du, want["tables/user_id"], "untied user table")
    tr.apply_gradients()  # the tied table takes lr * dE on every row, the bias lr * db
    tr._after_step()
    got_e = table.table.double().cpu().numpy()
    assert np.isfinite(got_e).all()


def test_step_against_reference_golden(device):
    """One step against the reference's torch modules (tests/golden/make_golden_catalog_train.py): a mean-pooled item history
    tied to EmbeddingTablePrediction with duplicate ids, T = 0.05, a bias and sample weights — the loss, the MLP, the untied
    user table, the tied dE (both paths) and db."""
    model, feats, y, sw, z = O.golden_model(device)
    want = O.golden_grads(z)
    model.compile(optimizer=mm.SGD(0.1))
    B = len(y)
    tr = model.trainer(B)
    x, yt = dev_batch(feats, y, device)
    tr.forward_backward(x, [yt], torch.from_numpy(sw).to(device))
    torch.cuda.synchronize()
    want_loss = float(z["loss"])
    assert abs(tr.loss[0].item() - want_loss) <= 2e-4 * max(1.0, abs(want_loss), 1.0 / float(z["temperature"]))
    np.testing.assert_allclose(tr.h[-1][:B].double().cpu().numpy(), z["query"], rtol=1e-3, atol=1e-4)
    g = tr.gradients()
    for i, l in enumerate(model.mlp.dense_layers):
        close(g[f"{l.name}/kernel"], want[f"mlp/{i}/kernel"], f"mlp {i} kernel")
        close(g[f"{l.name}/bias"], want[f"mlp/{i}/bias"], f"mlp {i} bias")
    check_tied(model, feats, y, sw, tr, want["tables/item_id"], want["bias"])
    ids, rows = tr.table_gradients()["user_id"]
    du = torch.zeros(int(z["n_users"]), int(z["dim"]), dtype=torch.float64).index_add_(0, ids.cpu().long(), rows.cpu().double())
    close(du, want["tables/user_id"], "untied user table")


# ---------------------------------------------------------------------------------------------------------------
# eager against graph replay, and the dense update rule of the tied table
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam", "lazyadam"])
def test_three_steps_graph_replay_bit_identical(device, opt):
    """The catalog kernels, the row merge and the dense updates have a fixed order, so the first step's loss, tied table
    and bias are bit-identical.  The MLP's weight gradient (mm_dense_wgrad) sums its batch splits with float atomics, so
    after that the variables are compared to 1e-6 of their scale.  The
    untied user table has 300 000 rows, so no user id comes three times in a batch (the sparse update's fold order)."""
    n_items, D, B = 900, 64, 256
    # Adam with epsilon 1e-3: at the default 1e-7 an element whose gradient is ~1e-9 moves by ~lr either way, so the
    # atomics' last-bit differences would decide the comparison
    make = {"sgd": lambda: mm.SGD(0.05), "adagrad": lambda: mm.Adagrad(0.05), "adam": lambda: mm.Adam(0.01, epsilon=1e-3),
            "lazyadam": lambda: mm.LazyAdam(0.01, epsilon=1e-3)}[opt]
    batches = [O.batch(O.schema(n_items, "list", n_users=300_000), n_items, B, seed=10 + i, hot=3) for i in range(3)]
    runs = []
    for graph in (False, True):
        model, s, table = O.build(n_items, D, "list", T=0.05, seed=5, n_users=300_000)
        model.build(device)
        e0 = table.table.double().cpu().numpy()
        model.compile(optimizer=make())
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
        runs.append((losses, first, table.table.clone(), model.prediction.bias.clone(),
                     [l.kernel.clone() for l in model.mlp.dense_layers], e0))
    (la, fa, ea, ba, ka, e0), (lb, fb, eb, bb, kb, _) = runs
    # step 1 starts from identical variables: the catalog kernels, the row merge and the dense update are fixed-order
    assert torch.equal(la[0], lb[0]) and torch.equal(fa[0], fb[0]) and torch.equal(fa[1], fb[1])
    for a, b in zip(la, lb):
        assert abs(a.item() - b.item()) <= 1e-6 * abs(a.item())
    for name, a, b in [("table", ea, eb), ("bias", ba, bb)] + [(f"kernel {i}", a, b) for i, (a, b) in enumerate(zip(ka, kb))]:
        assert (a - b).abs().max().item() <= 1e-6 * a.abs().max().item(), name
    # a dense gradient: every row of the tied table moved, including rows no lookup and no label touched
    moved = (ea.double().cpu().numpy() != e0).any(axis=1)
    assert moved.all(), f"{int((~moved).sum())} rows of the tied table were not updated"


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam", "lazyadam"])
def test_tied_table_update_rule(device, opt):
    """One step of CatalogTrainer: the tied table equals the Keras dense update of its float64 gradient (both paths
    summed) on every row, rows no lookup and no label touched included (LazyAdam on a dense gradient is Adam)."""
    n_items, D, B = 400, 16, 128
    model, s, table = O.build(n_items, D, "onehot", T=0.5)
    model.build(device)
    feats, y = O.batch(s, n_items, B, seed=8, hot=4)
    _, want = O.restated_step(model, feats, y)
    e0 = table.table.double().cpu().numpy()
    o = {"sgd": mm.SGD(0.5), "adagrad": mm.Adagrad(0.5), "adam": mm.Adam(0.05), "lazyadam": mm.LazyAdam(0.05)}[opt]
    model.compile(optimizer=o)
    x, yt = dev_batch(feats, y, device)
    model.train_step((x, yt))
    s1 = np.full_like(e0, o.initial_accumulator_value)
    kind = "adam" if opt == "lazyadam" else opt
    we, _, _ = O.dense_update(kind, e0, want["tables/item_id"], s1, np.zeros_like(e0), o.learning_rate, 1)
    got = table.table.double().cpu().numpy()
    step = np.abs(we - e0).max()
    assert np.abs(got - we).max() <= 2e-2 * step + 1e-6
    untouched = np.setdiff1d(np.arange(n_items), np.concatenate([feats["last_item"], y]))
    assert len(untouched) > 100 and (got[untouched] != e0[untouched]).any(axis=1).all()


# ---------------------------------------------------------------------------------------------------------------
# fit, evaluate, save / load, out-of-range labels
# ---------------------------------------------------------------------------------------------------------------
def test_fit_evaluate_save_load(device, tmp_path):
    n_items, D, B = 500, 32, 200
    model, s, table = O.build(n_items, D, "list", T=0.5, widths=(64,))
    model.compile(optimizer=mm.Adagrad(0.05))
    data = [dev_batch(*O.batch(s, n_items, B, seed=20 + i, hot=6), device) for i in range(4)]
    val = [dev_batch(*O.batch(s, n_items, B, seed=40 + i, hot=6), device) for i in range(2)]
    hist = model.fit(data, epochs=2, validation_data=val)
    assert len(hist.history["loss"]) == 2 and hist.history["loss"][1] < hist.history["loss"][0]
    assert "val_loss" in hist.history and "val_recall_at_10" in hist.history
    res = model.evaluate(val, return_dict=True)
    assert list(res) == model.metrics_names == ["loss", "recall_at_10", "mrr_at_10", "ndcg_at_10", "map_at_10", "precision_at_10"]
    # float64 recomputation from materialised logits (the model's call, without the temperature; T for the loss)
    T = model.prediction.logits_temperature
    rows, sums, loss = 0, np.zeros(5), 0.0
    for x, y in val:
        q = model.query(x).double().cpu().numpy()
        z = q @ table.table.double().cpu().numpy().T + model.prediction.bias.double().cpu().numpy()
        yy = y.cpu().numpy()
        zt = z / T
        m = zt.max(1, keepdims=True)
        loss += float(np.sum(m[:, 0] + np.log(np.exp(zt - m).sum(1)) - zt[np.arange(len(yy)), yy]))
        rank = (z > z[np.arange(len(yy)), yy][:, None]).sum(1)  # 0-based rank of the label
        hit = rank < 10
        sums += [hit.sum(), np.where(hit, 1.0 / (rank + 1), 0).sum(), np.where(hit, 1.0 / np.log2(rank + 2), 0).sum(),
                 np.where(hit, 1.0 / (rank + 1), 0).sum(), hit.sum() / 10]
        rows += len(yy)
    got = [res[k] for k in model.metrics_names]
    assert abs(got[0] - loss / rows) <= 1e-4 * max(1.0, loss / rows)
    np.testing.assert_allclose(got[1:], sums / rows, rtol=0, atol=1.5 / rows)  # a near-tie may flip one row
    x, _ = val[0]
    z0, (s0, i0) = model(x), model.top_k(x, 10)
    model.save(tmp_path / "m")
    loaded = mm.Model.load(tmp_path / "m")
    assert torch.equal(loaded(x), z0)
    s1, i1 = loaded.top_k(x, 10)
    assert torch.equal(s1, s0) and torch.equal(i1, i0)
    loaded.compile(optimizer="adagrad")
    r2 = loaded.evaluate(val, return_dict=True)
    assert r2 == res


def test_explicit_metrics_and_refusal_of_large_k(device):
    model, s, _ = O.build(300, 16, "none")
    with pytest.raises(ValueError, match="32"):
        model.compile(optimizer="sgd", metrics=[mm.RecallAt(33)])
    model.compile(optimizer="sgd", metrics=[mm.RecallAt(32), mm.NDCGAt(5)])
    res = model.evaluate([dev_batch(*O.batch(s, 300, 64), device)], return_dict=True)
    assert list(res) == ["loss", "recall_at_32", "ndcg_at_5"]


def test_out_of_range_label_raises(device):
    n_items, B = 300, 64
    model, s, _ = O.build(n_items, 16, "onehot")
    model.compile(optimizer="sgd")
    f, y = O.batch(s, n_items, B)
    y[5] = n_items
    with pytest.raises(IndexError):
        model.fit([dev_batch(f, y, device)], epochs=1)
    with pytest.raises(IndexError):
        model.evaluate([dev_batch(f, y, device)])


# ---------------------------------------------------------------------------------------------------------------
# the benchmark's sizes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_items,B,T", [(1_000_000, 16_384, 0.5), (10_000_000, 4096, 1.0)])
def test_benchmark_sizes_sampled_rows(device, n_items, B, T):
    """One step at the benchmark's shapes, D = 64, a 20-id history tied to the output: sampled rows of dE (rows the
    input side hit and rows it did not) and db, and sampled queries' dx, against float64 from the trainer's own x and
    lse (dx over the whole table, recomputed on the device in float64)."""
    D, L = 64, 20
    model, s, table = O.build(n_items, D, "list", widths=(128,), T=T, L=L)
    model.build(device)
    ops.init_uniform_hash(table.table, 77, -0.05, 0.05)
    ops.init_uniform_hash(model.prediction.bias.view(-1, 1), 78, -0.2, 0.2)
    model.prediction.refresh()
    feats, y = O.batch(s, n_items, B, seed=1, L=L, hot=50)
    model.compile(optimizer="adagrad")
    tr = model.trainer(B)
    x, yt = dev_batch(feats, y, device)
    tr.forward_backward(x, [yt])
    torch.cuda.synchronize()
    q = tr.h[-1][:B].double().cpu().numpy()
    lse = tr.stats[:B, 1].double().cpu().numpy()
    hist = feats["item_history"]
    rows = np.unique(np.concatenate([[0, 1, n_items - 1, n_items // 2], hist[:3].reshape(-1)[:6], np.arange(3)]))
    E = table.table
    bias = model.prediction.bias
    Er = E[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    br = bias[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    G = (np.exp((q @ Er.T + br[None, :]) / T - lse[:, None]) - (y[:, None] == rows[None, :])) / B
    # the input side: the pooled gradient dx0's item columns, spread over the history's ids (mean: / L)
    col = model.body.input_block.layout()[0]["item_history"]
    dpool = tr.inp.dx0[:B, col:col + D].double().cpu().numpy() / L
    inp = np.zeros((len(rows), D))
    for j, r in enumerate(rows):
        inp[j] = dpool[np.nonzero(hist == r)[0]].sum(0) if (hist == r).any() else 0.0
    got = tr.wk.dE[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    want = G.T @ q / T + inp
    bound = 1e-3 * (np.abs(G).T @ np.abs(q)) / T + 1e-5 * np.abs(inp) + 1e-9
    assert np.all(np.abs(got - want) <= bound)
    got_b = tr.wk.db[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    assert np.all(np.abs(got_b - G.sum(0) / T) <= 1e-3 * np.abs(G).sum(0) / T + 1e-12)
    # dx of sampled queries: (sum_j p_j e_j - e_y) / (B T), relu-masked like the last layer's output
    qs = torch.tensor([0, 1, 2, B // 2, B - 1], device=device)
    qd = tr.h[-1][qs].double()
    lq = tr.stats[qs, 1].double()
    acc = torch.zeros((len(qs), D), dtype=torch.float64, device=device)
    aacc = torch.zeros_like(acc)
    for r0 in range(0, n_items, 1_000_000):
        blk = E[r0:r0 + 1_000_000].double()
        p = torch.exp((qd @ blk.T + bias[r0:r0 + 1_000_000].double()[None, :]) / T - lq[:, None])
        acc += p @ blk
        aacc += p @ blk.abs()
    ey = E[torch.from_numpy(y).to(device)[qs]].double()
    want_dx = ((acc - ey) / (B * T) * (qd > 0)).cpu().numpy()
    got_dx = tr.dh[-1][qs].double().cpu().numpy()
    bound_dx = (1e-3 * (aacc + ey.abs()) / (B * T)).cpu().numpy() + 1e-12
    assert np.all(np.abs(got_dx - want_dx) <= bound_dx), np.max(np.abs(got_dx - want_dx) / bound_dx)
    assert torch.isfinite(tr.wk.dE).all()
