"""Label-smoothed full-catalog soft-max cross-entropy without a GPU: the float64 restatement (catalog_smoothing_oracle.py)
against torch autograd of F.cross_entropy(label_smoothing=eps) and central finite differences, its eps = 0 case against
the unsmoothed restatement, the loss classes, CatalogModel.compile's acceptance and refusals, and the argument rules of
ops.catalog_softmax_ce_backward(label_smoothing=...) and the C entry points that hold before any CUDA call."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops
from tests import catalog_model_oracle as O
from tests.catalog_smoothing_oracle import smoothed_by_autograd, smoothed_catalog_ce
from tests.catalog_train_oracle import catalog_ce


@pytest.mark.parametrize("T,bias,weights,eps", [(1.0, True, False, 0.1), (0.5, False, True, 0.3), (0.05, True, True, 0.1),
                                                (1.0, True, True, 0.9)])
def test_restatement_matches_autograd(T, bias, weights, eps):
    rng = np.random.default_rng(5)
    B, N, D = 7, 11, 5
    x = rng.standard_normal((B, D))
    E = rng.standard_normal((N, D)) * 0.5
    b = rng.standard_normal(N) * 0.3 if bias else None
    y = rng.integers(0, N, B)
    y[:2] = [0, N - 1]
    sw = rng.uniform(0.2, 2.0, B) if weights else None
    got = smoothed_catalog_ce(x, E, b, y, T, eps, sw)
    ref = smoothed_by_autograd(x, E, b, y, T, eps, sw)
    assert abs(got[0] - ref[0]) <= 1e-12 * max(1.0, abs(ref[0]))
    for g, r in zip(got[1:3], ref[1:3]):
        np.testing.assert_allclose(g, r, rtol=1e-10, atol=1e-12)
    if bias:
        np.testing.assert_allclose(got[3], ref[3], rtol=1e-10, atol=1e-12)


def test_restatement_against_finite_differences():
    rng = np.random.default_rng(6)
    B, N, D, T, eps = 5, 9, 4, 0.5, 0.2
    x, E, b = rng.standard_normal((B, D)), rng.standard_normal((N, D)) * 0.5, rng.standard_normal(N) * 0.3
    y, sw = rng.integers(0, N, B), rng.uniform(0.5, 1.5, B)
    _, dx, dE, db = smoothed_catalog_ce(x, E, b, y, T, eps, sw)
    h = 1e-6
    for arr, grad in ((x, dx), (E, dE), (b, db)):
        for idx in [tuple(int(rng.integers(0, n)) for n in arr.shape) for _ in range(5)]:
            vals = []
            for sgn in (1, -1):
                a = arr.copy()
                a[idx] += sgn * h
                args = [a if arr is v else v for v in (x, E, b)]
                vals.append(smoothed_catalog_ce(*args, y, T, eps, sw)[0])
            fd = (vals[0] - vals[1]) / (2 * h)
            assert abs(fd - grad[idx]) <= 1e-6 * max(1.0, abs(fd)), (idx, fd, grad[idx])


def test_eps_zero_is_the_unsmoothed_restatement():
    rng = np.random.default_rng(7)
    x, E, b = rng.standard_normal((6, 4)), rng.standard_normal((10, 4)), rng.standard_normal(10)
    y = rng.integers(0, 10, 6)
    for g, r in zip(smoothed_catalog_ce(x, E, b, y, 0.5, 0.0), catalog_ce(x, E, b, y, 0.5)):
        np.testing.assert_allclose(g, r, rtol=1e-13, atol=1e-15)


def test_out_of_range_label_keeps_the_uniform_term():
    """No one-hot term and a NaN loss entry (the unsmoothed rule), but the row still pulls toward eps / N everywhere."""
    rng = np.random.default_rng(8)
    x, E = rng.standard_normal((3, 4)), rng.standard_normal((5, 4))
    eps = 0.25
    loss, dx, dE, db = smoothed_catalog_ce(x, E, None, [5, -1, 2], 1.0, eps)
    assert np.isnan(loss)
    z = x @ E.T
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    np.testing.assert_allclose(dx[0], (p[0] @ E - eps / 5 * E.sum(0)) / 3, rtol=1e-12)
    # sum_j of a row's gradient: c (1 - (1 - eps) [label in range] - eps): two out-of-range rows, one in range
    np.testing.assert_allclose(db.sum(), 2 * (1 - eps) / 3, rtol=1e-12, atol=1e-15)


def test_loss_classes():
    ce = mm.losses.CategoricalCrossEntropy(label_smoothing=0.1)
    assert ce.from_logits and ce.label_smoothing == 0.1  # the reference's default: from_logits=True
    assert not mm.losses.CategoricalCrossentropy().from_logits  # Keras' default
    assert mm.losses.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1) == ce
    assert "label_smoothing=0.1" in repr(ce)
    with pytest.raises(NotImplementedError, match="retrieval"):  # not a retrieval model's loss
        mm.losses.get(ce)


def test_compile_accepts_the_smoothed_loss():
    model, _, _ = O.build(40, 8, "onehot")
    for loss, eps in ((None, 0.0), ("categorical_crossentropy", 0.0), ("CategoricalCrossentropy", 0.0),
                      (mm.losses.CategoricalCrossEntropy(), 0.0),
                      (mm.losses.CategoricalCrossEntropy(from_logits=True, label_smoothing=0.1), 0.1),
                      (mm.losses.CategoricalCrossentropy(from_logits=True, label_smoothing=0.3), 0.3)):
        model.compile(optimizer="adam", loss=loss)
        assert model.label_smoothing == eps
        assert model.metrics_names[0] == "loss" and len(model.metrics_names) == 6  # the top-k metrics are unchanged


def test_compile_refusals():
    model, _, _ = O.build(40, 8, "onehot")
    for loss, match in ((mm.losses.CategoricalCrossentropy(label_smoothing=0.1), "from_logits"),
                        (mm.losses.CategoricalCrossEntropy(from_logits=False), "from_logits"),
                        (mm.losses.CategoricalCrossEntropy(label_smoothing=1.0), r"\[0, 1\)"),
                        (mm.losses.CategoricalCrossEntropy(label_smoothing=-0.1), r"\[0, 1\)"),
                        (mm.losses.CategoricalCrossEntropy(label_smoothing=float("nan")), r"\[0, 1\)"),
                        (mm.losses.BPRLoss(), "categorical_crossentropy"),
                        ("bpr", "categorical_crossentropy")):
        with pytest.raises(NotImplementedError, match=match):
            model.compile(optimizer="adam", loss=loss)


def test_python_argument_errors_before_launch():
    t = torch.zeros(4, 4)
    for eps in (-0.1, 1.0, float("nan")):
        with pytest.raises(ValueError, match="label_smoothing"):
            ops.catalog_softmax_ce_backward(t, t, 4, t, t, t, t, t, label_smoothing=eps)
    with pytest.raises(RuntimeError, match="CUDA"):  # no CPU fallback
        ops.catalog_softmax_ce_backward(t, t, 4, t, t, t, t, t, label_smoothing=0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.catalog_mean_logit(t, t, 4)


def test_c_entry_points_reject_bad_arguments():
    """mm_catalog_smoothed_ce_backward and mm_catalog_mean_logit return an error code before any CUDA call (fake,
    aligned, non-null pointers)."""
    lib = _cabi.load()
    P = 1 << 20

    def bwd(eps=0.1, D=64, T=1.0, N=8, labels=P, stats=P, dx=P + 4096, de=P + 8192, x_split=P, ws=None, ws_bytes=0):
        return lib.mm_catalog_smoothed_ce_backward(x_split, P, 8, N, D, None, labels, _cabi.MM_I64, T, eps, stats, P, 1, dx, de, None,
                                                   None, None, ws, ws_bytes, None)

    assert bwd(eps=-0.1) == -1 and bwd(eps=1.0) == -1 and bwd(eps=float("nan")) == -1
    assert bwd(labels=None) == -1 and bwd(stats=None) == -1 and bwd(T=0.0) == -1 and bwd(N=0) == -1
    assert bwd(de=P + 4096) == -1  # dx aliases de
    assert bwd(D=129) == -2
    assert bwd(x_split=P + 2) == -3

    def mean(D=64, N=8, x=P, out=P + 4096, ws=P + 8192, ws_bytes=1 << 20):
        return lib.mm_catalog_mean_logit(x, P, 8, N, D, None, out, ws, ws_bytes, None)

    assert mean(x=None) == -1 and mean(out=None) == -1 and mean(N=0) == -1
    assert mean(D=129) == -2 and mean(x=P + 2) == -3 and mean(out=P + 4098) == -3
