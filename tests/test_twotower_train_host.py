"""CPU checks of the two-tower training restatement (tests/twotower_train_oracle.py) against the reference's torch
two-tower step (tests/golden/twotower_train/ref_torch_twotower_train.npz, written by
tests/golden/make_golden_twotower_train.py), and of the argument checks of mm_inbatch_softmax_ce_backward /
mm_l2_normalize_backward.

The restatement's autograd gradients are checked against the closed forms the CUDA kernels implement
(include/mm_b200.h K16): g[b,0] = c (p[b,0] - 1) / T, g[b,1+n] = c p[b,1+n] / T off the mask, dq = g[:,0] pos + G N,
dpos = g[:,0] q, dneg = G^T q; and the L2Norm backward dx = (dy - y (y . dy)) / n."""
from pathlib import Path

import numpy as np
import pytest
import torch

from models_b200 import _cabi
from tests import twotower_train_oracle as O


def _closed_form(q, pos, neg, pid, nid, T, fns):
    B = q.shape[0]
    s0 = (q * pos).sum(-1) / T
    sn = q @ neg.T
    mask = pid[:, None] == nid[None, :]
    sn = np.where(mask, fns, sn) / T
    s = np.concatenate([s0[:, None], sn], 1)
    lse = np.log(np.exp(s - s.max(1, keepdims=True)).sum(1)) + s.max(1)
    p = np.exp(s - lse[:, None])
    c = 1.0 / B
    g0 = c * (p[:, 0] - 1) / T
    G = np.where(mask, 0.0, c * p[:, 1:] / T)
    return float(c * (lse - s[:, 0]).sum()), g0[:, None] * pos + G @ neg, g0[:, None] * q, G.T @ q


@pytest.mark.parametrize("T", [1.0, 0.25])
def test_restated_loss_and_gradients_match_closed_form(T):
    g = np.random.default_rng(1)
    B, D = 23, 8
    q, it = g.standard_normal((B, D)), g.standard_normal((B, D))
    ids = g.integers(0, 6, B)
    qt, itt = torch.tensor(q, requires_grad=True), torch.tensor(it, requires_grad=True)
    loss = O.inbatch_ce(qt, itt, ids, T)
    loss.backward()
    want, dq, dpos, dneg = _closed_form(q, it, it, ids, ids, T, O.MIN_FLOAT)
    assert abs(float(loss.item()) - want) < 1e-12
    np.testing.assert_allclose(qt.grad.numpy(), dq, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(itt.grad.numpy(), dpos + dneg, rtol=1e-10, atol=1e-12)


def test_restated_l2_backward_matches_closed_form():
    g = np.random.default_rng(2)
    x = g.standard_normal((9, 5))
    x[2] = 0.0
    dy = g.standard_normal(x.shape)
    xt = torch.tensor(x, requires_grad=True)
    (O.l2_normalize(xt) * torch.tensor(dy)).sum().backward()
    s = (x * x).sum(1, keepdims=True)
    n = np.sqrt(np.maximum(s, 1e-12))
    y = x / n
    want = np.where(s >= 1e-12, (dy - y * (y * dy).sum(1, keepdims=True)) / n, dy / 1e-6)
    np.testing.assert_allclose(xt.grad.numpy(), want, rtol=1e-10, atol=1e-12)


def test_restated_step_pools_bags_and_skips_untouched_rows():
    """A ragged mean bag and a one-hot id feed one tower: rows the batch never looked up keep a zero gradient, and the
    SGD step moves exactly the touched rows."""
    g = np.random.default_rng(3)
    towers = {
        "query": {"tables": {"u": g.standard_normal((10, 4))}, "continuous": ["c"],
                  "layers": [{"kernel": g.standard_normal((5, 4)), "bias": np.zeros(4), "activation": "relu"}]},
        "item": {"tables": {"i": g.standard_normal((12, 4)), "tags": g.standard_normal((7, 4))}, "combiner": {"tags": "mean"},
                 "layers": [{"kernel": g.standard_normal((8, 4)), "bias": np.zeros(4), "activation": "linear"}]},
    }
    batch = {"u": np.array([1, 2, 2, 5]), "c": np.array([0.5, -1.0, 2.0, 0.0], np.float32), "i": np.array([3, 4, 3, 11]),
             "tags": (np.array([0, 1, 1, 6, 2]), np.array([0, 2, 3, 3, 5]))}
    _, out, grads = O.twotower_loss_and_grads(batch, towers, "i")
    assert out["query"].shape == (4, 4) and out["item"].shape == (4, 4)
    for key, touched in (("query/table/u", {1, 2, 5}), ("item/table/i", {3, 4, 11}), ("item/table/tags", {0, 1, 2, 6})):
        rows = {int(r) for r in np.nonzero(np.abs(grads[key]).sum(1))[0]}
        assert rows <= touched, (key, rows)
    _, trained = O.train_steps([batch], towers, "i", "sgd", 0.1)
    moved = np.nonzero(np.abs(trained["item"]["tables"]["i"] - towers["item"]["tables"]["i"]).sum(1))[0]
    assert set(moved.tolist()) <= {3, 4, 11}


FIXTURE = Path(__file__).parent / "golden" / "twotower_train" / "ref_torch_twotower_train.npz"


def _close(a, b, tol=2e-5):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    scale = max(1e-30, float(np.abs(b).max()) if b.size else 1.0)
    assert np.abs(a - b).max() <= tol * scale, float(np.abs(a - b).max()) / scale


def test_restatement_matches_reference_step():
    """The reference's torch two-tower step (TabularInputBlock + EmbeddingTables(mean) -> MLPBlock, in-batch
    ContrastiveOutput.contrastive_outputs with false-negative rescoring, LogitsTemperatureScaler, F.cross_entropy against
    class 0, autograd) at T = 1 and T = 0.5: loss, tower outputs, every tower variable's gradient and the touched table rows'
    gradients against the float64 restatement."""
    z = np.load(FIXTURE)
    batch, towers, _ = O.golden_inputs(z)
    variants = O.golden_variants(z)
    assert [t for _, t in variants] == [1.0, 0.5]
    movie = z["batch_movieId"]
    assert (movie[:, None] == movie[None, :]).sum() > len(movie)  # an accidental hit off the diagonal
    for vt, T in variants:
        loss, out, grads = O.twotower_loss_and_grads(batch, towers, "movieId", temperature=T, false_neg_score=float(z["min_float"]))
        assert abs(loss - float(z[f"{vt}_loss"])) <= 1e-5 * abs(loss), (vt, loss, float(z[f"{vt}_loss"]))
        for tag, t in towers.items():
            _close(out[tag], z[f"{vt}_{tag}_out"], 1e-5)
            for i, l in enumerate(t["layers"]):
                _close(grads[f"{tag}/kernel_{i}"], z[f"{vt}_grad_{tag}_kernel_{i}"])
                _close(grads[f"{tag}/bias_{i}"], z[f"{vt}_grad_{tag}_bias_{i}"])
            for f in t["tables"]:
                _close(grads[f"{tag}/table/{f}"], z[f"{vt}_grad_{tag}_table_{f}_rows"])


# ---- argument checks with made-up device addresses (never dereferenced: the calls return before any launch) ----
pytestmark_cpu = pytest.mark.skipif(torch.cuda.is_available(), reason="passes fake device pointers: CPU-only check")
BASE = 0x7F0000000000


def _bwd(D=64, q_split=BASE, T=1.0, stats=BASE + 0x10000, dpos=BASE + 0x50000, dneg=BASE + 0x60000, B=64, N=64, downscore=0,
         ids=None):
    return _cabi.load().mm_inbatch_softmax_ce_backward(q_split, BASE + 0x80000, B, N, D, ids, ids, _cabi.MM_I64, downscore, -1.0, None,
                                                       T, stats, BASE + 0x20000, BASE + 0x30000, BASE + 0x90000, 1, BASE + 0x40000,
                                                       dpos, dneg, None, None)


@pytestmark_cpu
def test_ce_backward_argument_errors_before_launch():
    assert _bwd(D=129) == -2
    assert _bwd(q_split=BASE + 2) == -3
    assert _bwd(T=0.0) == -1 and _bwd(T=-0.5) == -1
    assert _bwd(stats=None) == -1
    assert _bwd(dpos=BASE + 0x50000, dneg=BASE + 0x50000, N=63) == -1
    assert _bwd(downscore=1) == -1
    assert _bwd(B=1 << 31) == -2


@pytestmark_cpu
def test_l2_backward_argument_errors():
    lib = _cabi.load()
    assert lib.mm_l2_normalize_backward(None, BASE, 4, 8, 8, 8, BASE, 8, None) == -1
    assert lib.mm_l2_normalize_backward(BASE, BASE, 4, 8, 7, 8, BASE, 8, None) == -1
