"""Host-side checks of the full-catalog soft-max cross-entropy backward: the float64 oracle against autograd, and the
argument rules of ops.catalog_softmax_ce_backward and mm_catalog_softmax_ce_backward that hold before any CUDA call."""
import numpy as np
import pytest
import torch

from models_b200 import _cabi, ops
from tests.catalog_train_oracle import catalog_ce, closed_form_grads_by_autograd


@pytest.mark.parametrize("T,bias,weights", [(1.0, True, False), (0.5, False, True), (0.05, True, True)])
def test_oracle_matches_autograd(T, bias, weights):
    rng = np.random.default_rng(3)
    B, N, D = 7, 11, 5
    x = rng.standard_normal((B, D))
    E = rng.standard_normal((N, D)) * 0.5
    b = rng.standard_normal(N) * 0.3 if bias else None
    y = rng.integers(0, N, B)
    y[:2] = [0, N - 1]
    sw = rng.uniform(0.2, 2.0, B) if weights else None
    got = catalog_ce(x, E, b, y, T, sw)
    ref = closed_form_grads_by_autograd(x, E, b, y, T, sw)
    assert abs(got[0] - ref[0]) <= 1e-12 * max(1.0, abs(ref[0]))
    for g, r in zip(got[1:3], ref[1:3]):
        np.testing.assert_allclose(g, r, rtol=1e-10, atol=1e-12)
    if bias:
        np.testing.assert_allclose(got[3], ref[3], rtol=1e-10, atol=1e-12)


def test_oracle_tiny_closed_form():
    """One query, two classes, no bias: G = c (softmax - onehot) / T by hand."""
    x = np.array([[1.0, 0.0]])
    E = np.array([[2.0, 0.0], [0.0, 1.0]])
    T = 0.5
    z = np.array([4.0, 0.0])  # x E^T / T
    p = np.exp(z) / np.exp(z).sum()
    loss, dx, dE, db = catalog_ce(x, E, None, [1], T)
    assert loss == pytest.approx(np.log(np.exp(z).sum()) - z[1], rel=1e-14)
    g = (p - np.array([0.0, 1.0])) / T
    np.testing.assert_allclose(dx[0], g @ E, rtol=1e-14)
    np.testing.assert_allclose(dE, np.outer(g, x[0]), rtol=1e-14)
    np.testing.assert_allclose(db, g, rtol=1e-14)


def test_oracle_out_of_range_label_keeps_the_softmax_only():
    rng = np.random.default_rng(4)
    x, E = rng.standard_normal((3, 4)), rng.standard_normal((5, 4))
    loss, dx, dE, db = catalog_ce(x, E, None, [5, -1, 2])
    _, dx_in, _, _ = catalog_ce(x[2:], E, None, [2])
    assert np.isnan(loss)
    np.testing.assert_allclose(db.sum(), (2 / 3), rtol=1e-12)  # rows 0, 1: sum_j c p = 1/3 each, row 2: 0
    np.testing.assert_allclose(dx[2], dx_in[0] / 3, rtol=1e-12)  # c = 1/3 instead of 1


def test_python_argument_errors_before_launch():
    t = torch.zeros(4, 4)
    with pytest.raises(RuntimeError, match="CUDA"):  # no CPU fallback
        ops.catalog_softmax_ce_backward(t, t, 4, t, t, t, t, t)


def test_c_entry_point_rejects_bad_arguments():
    """mm_catalog_softmax_ce_backward returns an error code before any CUDA call (fake, aligned, non-null pointers)."""
    lib = _cabi.load()
    P = 1 << 20

    def bwd(D=64, T=1.0, N=8, labels=P, dt=_cabi.MM_I64, stats=P, dx=P + 4096, de=P + 8192, x_split=P, db=None):
        return lib.mm_catalog_softmax_ce_backward(x_split, P, 8, N, D, None, labels, dt, T, stats, P, 1, dx, de, db, None, None, None, 0,
                                                  None)

    assert bwd(labels=None) == -1 and bwd(stats=None) == -1 and bwd(dx=None) == -1 and bwd(de=None) == -1
    assert bwd(T=0.0) == -1 and bwd(N=0) == -1 and bwd(dt=7) == -1
    assert bwd(de=P + 4096) == -1  # dx aliases de
    assert bwd(D=129) == -2  # MM_ERR_UNSUPPORTED
    assert bwd(dx=P + 2) == -3 and bwd(x_split=P + 2) == -3 and bwd(db=P + 1) == -3  # MM_ERR_ALIGN
