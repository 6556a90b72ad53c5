"""Training-mode dropout of the weight-tied next-item step on the GPU: mm_dense_tc_dropout's masks against the numpy
Philox4x32-10 port bit for bit, the keep fraction over 10^6 elements, masks across steps and layers, rate = 0; one
CatalogTrainer step with dropout (and label smoothing) against the float64 restatement given the masks; eager steps
against CUDA-graph replays bit for bit; and masks that change from step to step in a captured graph."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops
from tests import catalog_model_oracle as O
from tests.catalog_smoothing_oracle import smoothed_restated_step
from tests.dropout_mask import keep_mask

pytestmark = pytest.mark.gpu


def layer(device, M, K, N, act, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(device)
    W = (torch.randn(K, N, generator=g) / K ** 0.5).to(device)
    b = (torch.randn(N, generator=g) * 0.1).to(device)
    return ops.split_rows(x), ops.split_weights(W), b


def run(device, a, w, b, K, N, act, dropout=None):
    M = a.shape[0]
    h = torch.empty((M, N), device=device)
    hs = torch.empty((M, 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=device)
    ops.dense_tc(a, K, w, N, b, act, out_f32=h, out_split=hs, dropout=dropout)
    return h, hs


@pytest.mark.parametrize("M,K,N,rate", [(8192, 64, 128, 0.2), (300, 100, 60, 0.5), (129, 32, 200, 0.1)])
def test_masks_equal_the_numpy_port(device, M, K, N, rate):
    """A linear layer (no exact zeros before dropout): the kept elements are the plain output times 1 / (1 - rate) in
    fp32, the dropped ones exact zeros, the split output the split of the dropped output, and the mask the port's."""
    a, w, b = layer(device, M, K, N, "linear", seed=M)
    plain, _ = run(device, a, w, b, K, N, "linear")
    step = torch.full((1,), 5.0, device=device)
    h, hs = run(device, a, w, b, K, N, "linear", dropout=(rate, 1234567890123, step, 3))
    want = keep_mask(M, N, rate, 1234567890123, 5, 3)
    got = (h != 0).cpu().numpy()
    assert (plain != 0).all() and np.array_equal(got, want)
    scale = np.float32(1.0) / np.float32(1.0 - rate)
    assert torch.equal(h, torch.where(torch.from_numpy(want).to(device), plain * float(scale), torch.zeros_like(plain)))
    assert torch.equal(hs, ops.split_rows(h))
    if M * N >= 10 ** 6:  # binomial: 5 standard deviations
        assert abs(got.mean() - (1 - rate)) <= 5 * np.sqrt(rate * (1 - rate) / got.size)


def test_masks_differ_across_steps_and_layers_and_rate_zero_is_no_dropout(device):
    M, K, N = 1024, 64, 128
    a, w, b = layer(device, M, K, N, "relu")
    step = torch.zeros(1, device=device)
    m0 = run(device, a, w, b, K, N, "linear", dropout=(0.3, 9, step, 0))[0] != 0
    step.fill_(1.0)
    m1 = run(device, a, w, b, K, N, "linear", dropout=(0.3, 9, step, 0))[0] != 0
    m2 = run(device, a, w, b, K, N, "linear", dropout=(0.3, 9, step, 1))[0] != 0
    for x, y in ((m0, m1), (m1, m2), (m0, m2)):
        assert 0.35 < (x != y).float().mean().item() < 0.49  # independent masks: 2 p (1 - p) = 42 %
    plain = run(device, a, w, b, K, N, "relu")
    zero = run(device, a, w, b, K, N, "relu", dropout=(0.0, 9, step, 0))
    assert torch.equal(plain[0], zero[0]) and torch.equal(plain[1], zero[1])


def with_dropout(model, rate, no_act_last):
    """O.build's MLPBlock(widths + [D]) (relu everywhere) as MLPBlock(..., no_activation_last_layer, dropout=rate)."""
    mlp = model.mlp
    mlp.dropout, mlp.no_activation_last_layer = rate, no_act_last
    if no_act_last:
        mlp.dense_layers[-1].activation = "linear"


def dev_batch(feats, labels, device):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in feats.items()}, torch.from_numpy(labels).to(device)


@pytest.mark.parametrize("no_act_last,eps,T", [(True, 0.1, 0.05), (False, 0.0, 1.0), (False, 0.1, 0.05)])
def test_step_with_dropout_against_restatement(device, no_act_last, eps, T):
    """One step with MLPBlock([48, D], no_activation_last_layer, dropout=0.2): the forward activations and every gradient against the float64
    restatement with the port's masks (seed of mm.set_seed, step 0, layer index)."""
    from tests.test_gpu_catalog_model import close

    n_items, D, B, rate = 700, 32, 300, 0.2
    model, s, table = O.build(n_items, D, "onehot", widths=(48,), T=T, seed=7)
    with_dropout(model, rate, no_act_last)
    model.build(device)
    feats, y = O.batch(s, n_items, B, seed=3, hot=5)
    loss = mm.losses.CategoricalCrossEntropy(label_smoothing=eps)
    model.compile(optimizer=mm.SGD(0.1), loss=loss)
    tr = model.trainer(B)
    assert tr.dropout_rates == ([rate, 0.0] if no_act_last else [rate, rate])
    masks = [None if not r else keep_mask(B, l.units, r, 7, 0, i) * float(np.float32(1.0) / np.float32(1.0 - r))
             for i, (l, r) in enumerate(zip(model.mlp.dense_layers, tr.dropout_rates))]
    want_loss, want, x = smoothed_restated_step(model, feats, y, eps, None, drop=masks)
    xd, yt = dev_batch(feats, y, device)
    tr.forward_backward(xd, [yt])
    torch.cuda.synchronize()
    close(tr.h[-1][:B], x, "x (forward)")
    if not no_act_last:  # dropped elements are exact zeros
        assert np.array_equal((tr.h[-1][:B] != 0).cpu().numpy(), x != 0)
    assert abs(tr.loss[0].item() - want_loss) <= 2e-4 * max(1.0, abs(want_loss), 1.0 / T)
    g = tr.gradients()
    for i, l in enumerate(model.mlp.dense_layers):
        close(g[f"{l.name}/kernel"], want[f"mlp/{i}/kernel"], f"mlp {i} kernel")
        close(g[f"{l.name}/bias"], want[f"mlp/{i}/bias"], f"mlp {i} bias")
    close(tr.wk.dE, want["tables/item_id"], "tied dE", rtol=5e-3)
    close(tr.wk.db, want["bias"], "db", rtol=5e-3)
    ids, rows = tr.table_gradients()["user_id"]
    du = torch.zeros(O.N_USERS, D, dtype=torch.float64).index_add_(0, ids.cpu().long(), rows.cpu().double())
    close(du, want["tables/user_id"], "untied user table")


def test_three_steps_eager_and_graph_replay_bit_identical(device):
    """Dropout and label smoothing: three eager steps and three replays of one captured step from the same state give
    the same activations (masks drawn from the device step counter), and the first step's variables bit for bit."""
    n_items, D, B = 900, 64, 256
    batches = [O.batch(O.schema(n_items, "list", n_users=300_000), n_items, B, seed=10 + i, hot=3) for i in range(3)]
    runs = []
    for graph in (False, True):
        model, s, table = O.build(n_items, D, "list", widths=(64,), T=0.05, seed=5, n_users=300_000)
        with_dropout(model, 0.2, False)
        model.build(device)
        model.compile(optimizer=mm.Adam(0.01, epsilon=1e-3), loss=mm.losses.CategoricalCrossEntropy(label_smoothing=0.1))
        tr = model.trainer(B)
        losses, acts = [], []
        for i, (f, y) in enumerate(batches):
            x, yt = dev_batch(f, y, device)
            if not graph:
                losses.append(tr.step(x, [yt])[0].clone())
            else:
                if i == 0:
                    tr.capture(x, [yt])
                losses.append(tr.replay(x, [yt])[0].clone())
            acts.append(tr.h[0][:B].clone())
            if i == 0:
                first = (table.table.clone(), model.prediction.bias.clone())
        runs.append((losses, first, acts))
    (la, fa, aa), (lb, fb, ab) = runs
    assert torch.equal(la[0], lb[0]) and torch.equal(fa[0], fb[0]) and torch.equal(fa[1], fb[1]) and torch.equal(aa[0], ab[0])
    for a, b in zip(la, lb):
        assert abs(a.item() - b.item()) <= 1e-6 * abs(a.item())
    # the masks change from step to step in the replays too (the zero pattern of the first layer's output)
    z = [(a == 0) for a in ab]
    assert (z[0] != z[1]).float().mean().item() > 0.1 and (z[1] != z[2]).float().mean().item() > 0.1
    for a, b in zip(aa, ab):
        assert torch.equal(a == 0, b == 0)


def test_dropout_after_a_linear_inner_layer_is_refused(device):
    model, s, _ = O.build(300, 16, "onehot")
    with_dropout(model, 0.2, False)
    model.mlp.dense_layers[0].activation = "linear"  # its output does not mark the dropped elements
    model.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="relu layers only"):
        model.trainer(64)
