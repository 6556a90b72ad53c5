"""The pairwise ranking losses without a GPU: the float64 restatement (tests/pairwise_oracle.py) against hand-evaluated
values and finite differences, the loss registry and compile(loss=...), the argument checks of ops.inbatch_pairwise /
inbatch_pairwise_backward and of the C entry points (made before any launch), and the kernel cases of
tests/test_gpu_pairwise.py reaching every kernel instantiation."""
import math

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, datasets, ops
from tests import pairwise_oracle as O


def sig(x):
    return 1.0 / (1.0 + math.exp(-x))


def _scores():
    sp = torch.tensor([[0.7], [-0.3]], dtype=torch.float64)
    sn = torch.tensor([[0.2, -1.1, 1.5], [0.4, -0.3 - 0.25, 2.0]], dtype=torch.float64)
    return sp, sn


def _by_hand(kind, sp, sn, lam=1.0):
    out = []
    for b in range(sn.shape[0]):
        p = float(sp[b, 0])
        neg = [float(v) for v in sn[b]]
        w = np.exp(np.array(neg) - max(neg))
        w = w / w.sum()
        row = []
        for j, n in enumerate(neg):
            if kind == "bpr":
                row.append(-math.log(sig(p - n)))
            elif kind == "bpr-max":
                row.append(-math.log(sig(p - n) * w[j]) + lam * n * n * w[j])
            elif kind in ("top1", "top1_v2"):
                row.append(sig(n - p) + sig(n * n))
            elif kind == "top1-max":
                row.append((sig(n - p) + sig(n * n)) * w[j])
            elif kind == "logistic":
                row.append(max(n - p, 0.0) + math.log1p(math.exp(-abs(n - p))))
            else:
                row.append(max(1.0 + n - p, 0.0))
        if kind == "top1_v2":
            row = [sum(row) / len(row) - sig(p * p) / len(row)]
        out.append(row)
    return np.array(out)


@pytest.mark.parametrize("kind", O.KINDS)
def test_element_losses_match_hand_values(kind):
    sp, sn = _scores()
    got = O.element_losses(sp, sn, kind, reg_lambda=0.5).numpy()
    np.testing.assert_allclose(got, _by_hand(kind, sp, sn, lam=0.5), rtol=1e-12)


def test_downscored_column_constants():
    """T = 1, down-scoring: the row's own column scores MIN_FLOAT = -655.04.  TOP1 adds sigmoid(655^2) = 1 for it (and
    sigmoid(-655 - sp) = 0); BPR-max adds -log(1e-24) = 55.26, because its soft-max weight is 0 in float32 (a float64
    product would give exp(-655) and a loss near 656)."""
    q = torch.tensor([[0.3, -0.2], [0.1, 0.5]], dtype=torch.float64)
    it = torch.tensor([[0.4, 0.1], [-0.2, 0.3]], dtype=torch.float64)
    ids = np.array([5, 9])
    sp, sn = O.inbatch_scores(q, it, it, ids, ids, 1.0, True)
    assert float(sn[0, 0]) == float(np.float32(O.MIN_FLOAT)) and float(sn[1, 1]) == float(np.float32(O.MIN_FLOAT))
    top1 = O.element_losses(sp, sn, "top1")
    assert float(top1[0, 0]) == 1.0 and float(top1[1, 1]) == 1.0
    bprmax = O.element_losses(sp, sn, "bpr-max")
    np.testing.assert_allclose([float(bprmax[0, 0]), float(bprmax[1, 1])], [O.EPS0_LOSS] * 2, rtol=1e-12)
    assert abs(O.EPS0_LOSS - 55.262042231857095) < 1e-9
    # the unmasked column follows the formula; without down-scoring the own column is an ordinary negative (BPR: log 2)
    np.testing.assert_allclose(float(bprmax[0, 1]), _by_hand("bpr-max", sp, sn)[0, 1], rtol=1e-12)
    sp2, sn2 = O.inbatch_scores(q, it, it, ids, ids, 1.0, False)
    np.testing.assert_allclose(float(O.element_losses(sp2, sn2, "bpr")[0, 0]), math.log(2.0), rtol=1e-12)
    # the down-scored column's element is a constant: no gradient reaches the scores through it
    qd = q.clone().requires_grad_(True)
    sp, sn = O.inbatch_scores(qd, it, it, ids, ids, 1.0, True)
    O.element_losses(sp, sn, "top1")[0, 0].backward()
    assert float(qd.grad.abs().max()) < 1e-200


def test_eps0_is_decided_in_float32():
    """A weight that underflows float32 takes the eps0 branch; a subnormal float32 weight does not."""
    sp = torch.tensor([[0.0]], dtype=torch.float64)
    sn = torch.tensor([[0.0, -110.0]], dtype=torch.float64)  # exp(-110) < the smallest float32 subnormal
    el = O.element_losses(sp, sn, "bpr-max", reg_lambda=0.0)
    np.testing.assert_allclose(float(el[0, 1]), O.EPS0_LOSS, rtol=1e-12)
    sn = torch.tensor([[0.0, -95.0]], dtype=torch.float64)  # exp(-95): a float32 subnormal
    el = O.element_losses(sp, sn, "bpr-max", reg_lambda=0.0)
    assert float(el[0, 1]) > 90.0
    el = O.element_losses(torch.tensor([[-120.0]], dtype=torch.float64), torch.tensor([[0.0]], dtype=torch.float64), "bpr")
    np.testing.assert_allclose(float(el[0, 0]), O.EPS0_LOSS, rtol=1e-12)


@pytest.mark.parametrize("kind", O.KINDS)
def test_gradients_match_finite_differences(kind):
    g = np.random.default_rng(3)
    sp = torch.tensor(g.standard_normal((5, 1)), dtype=torch.float64, requires_grad=True)
    sn = torch.tensor(g.standard_normal((5, 7)), dtype=torch.float64, requires_grad=True)
    # away from the kinks: hinge at sn - sp = -1, logistic at sn = sp
    with torch.no_grad():
        u = sn - sp
        assert float((u + 1).abs().min()) > 1e-3 and float(u.abs().min()) > 1e-3
    loss = O.element_losses(sp, sn, kind, reg_lambda=0.7).mean()
    loss.backward()
    h = 1e-6
    for t in (sp, sn):
        num = np.zeros(tuple(t.shape))
        for idx in np.ndindex(*t.shape):
            with torch.no_grad():
                t[idx] += h
                up = float(O.element_losses(sp, sn, kind, reg_lambda=0.7).mean())
                t[idx] -= 2 * h
                dn = float(O.element_losses(sp, sn, kind, reg_lambda=0.7).mean())
                t[idx] += h
            num[idx] = (up - dn) / (2 * h)
        np.testing.assert_allclose(t.grad.numpy(), num, rtol=1e-6, atol=1e-9)


def test_registry():
    assert sorted(mm.losses.REGISTRY) == sorted(_cabi.PAIRWISE_KINDS) == sorted(O.KINDS)
    for name, cls in mm.losses.REGISTRY.items():
        obj = mm.losses.get(name)
        assert type(obj) is cls and obj.kind == name and mm.losses.get(obj) is obj
    assert mm.losses.get("bpr-max").reg_lambda == 1.0
    assert mm.losses.get(mm.losses.BPRmaxLoss(reg_lambda=0.25)).reg_lambda == 0.25
    assert mm.losses.BPRmaxLoss(0.5) == mm.losses.BPRmaxLoss(0.5) != mm.losses.BPRmaxLoss(1.0)
    assert mm.losses.get(None) is None and mm.losses.get("categorical_crossentropy") is None
    assert isinstance(mm.losses.get("top1_v2"), mm.losses.TOP1v2Loss) and isinstance(mm.losses.get("top1-max"), mm.losses.TOP1maxLoss)
    assert isinstance(mm.losses.get("logistic"), mm.losses.LogisticLoss) and isinstance(mm.losses.get("hinge"), mm.losses.HingeLoss)


def test_compile_accepts_pairwise_losses_on_retrieval_models_only():
    schema = datasets.movielens_1m_schema()
    for model in (mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32])), mm.MatrixFactorizationModel(schema, 16)):
        for name in O.KINDS:
            model.compile(optimizer="sgd", loss=name)
            assert model.pairwise_loss.kind == name
        model.compile(optimizer="sgd", loss=mm.losses.BPRmaxLoss(reg_lambda=0.3))
        assert model.pairwise_loss.reg_lambda == 0.3
        model.compile(optimizer="sgd", loss="categorical_crossentropy")
        assert model.pairwise_loss is None
        model.compile(optimizer="sgd")
        assert model.pairwise_loss is None
        for bad in ("mse", "binary_crossentropy", "bpr_max", "warp"):
            with pytest.raises(NotImplementedError, match="loss"):
                model.compile(optimizer="sgd", loss=bad)
    ranking = mm.DLRMModel(datasets.criteo_schema({k: min(v, 50) for k, v in datasets.CRITEO_MAX.items()}), embedding_dim=16,
                           bottom_block=mm.MLPBlock([32, 16]), top_block=mm.MLPBlock([16]))
    for bad in ("bpr", mm.losses.BPRLoss(), "top1-max"):
        with pytest.raises(NotImplementedError):
            ranking.compile(optimizer="sgd", loss=bad)


def test_python_argument_errors_before_launch():
    """Loss kind and reg_lambda are checked before any tensor is touched (these tensors are on the CPU)."""
    t = torch.zeros(4, 4)
    with pytest.raises(ValueError, match="kind"):
        ops.inbatch_pairwise(t, t, 4, t, t, "bpr_max")
    with pytest.raises(ValueError, match="reg_lambda"):
        ops.inbatch_pairwise(t, t, 4, t, t, "bpr-max", reg_lambda=float("nan"))
    with pytest.raises(ValueError, match="kind"):
        ops.inbatch_pairwise_backward(t, t, 4, t, t, t, t, t, t, t, "mse")
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.inbatch_pairwise(t, t, 4, t, t, "bpr")  # then the device: no CPU fallback


def test_c_entry_points_reject_bad_arguments():
    """The C entry points return an error code before any CUDA call (fake, aligned, non-null pointers)."""
    lib = _cabi.load()
    P = 1 << 20

    def fwd(kind=0, lam=1.0, D=64, T=1.0, stats=P, q_split=P, N=8, downscore=0, ids=None):
        return lib.mm_inbatch_pairwise_fwd(q_split, P, 8, N, D, ids, ids, _cabi.MM_I64, downscore, -655.04, T, kind, lam, P, stats,
                                           None, None)

    def bwd(dpos=P + 4096, dneg=P + 8192, dq=P + 16384, N=8):
        return lib.mm_inbatch_pairwise_bwd(P, P, 8, N, 64, None, None, _cabi.MM_I64, 0, -655.04, 1.0, 0, 1.0, P, P, P, P, dq, dpos,
                                           dneg, None)

    assert fwd(kind=7) == -1 and fwd(kind=-1) == -1
    assert fwd(lam=float("nan")) == -1 and fwd(lam=float("inf")) == -1
    assert fwd(T=0.0) == -1 and fwd(N=0) == -1
    assert fwd(stats=None) == -1 and fwd(downscore=1) == -1  # down-scoring needs ids
    assert fwd(D=129) == -2  # MM_ERR_UNSUPPORTED
    assert fwd(stats=P + 4) == -3 and fwd(q_split=P + 2) == -3  # MM_ERR_ALIGN
    assert bwd(dpos=P + 4096, dneg=P + 4096, N=7) == -1  # dpos aliases dneg only when N == B
    assert bwd(dq=P + 4096) == -1  # dq aliases dpos
    assert bwd(dpos=None) == -1


def test_kernel_cases_reach_every_instantiation():
    """tests/test_gpu_pairwise.py's kernel cases run every kind at both padded widths (64, 128) the forward, dq and dn
    kernels are compiled for, with and without down-scoring, at both temperatures, with ragged tiles, in-batch and not."""
    from tests.test_gpu_pairwise import KERNEL_CASES, KINDS

    assert sorted(KINDS) == sorted(_cabi.PAIRWISE_KINDS)
    widths = {64 if D <= 64 else 128 for _, _, D, *_ in KERNEL_CASES}
    assert widths == {64, 128}
    assert {c[3] for c in KERNEL_CASES} == {True, False} and {c[4] for c in KERNEL_CASES} == {1.0, 0.05}
    assert any(B % 128 and N % 128 and B > 128 for B, N, *_ in KERNEL_CASES)  # ragged last tiles, several tiles
    assert any(B == N == 1 for B, N, *_ in KERNEL_CASES)
    # the in-batch layout (own column down-scored, dpos aliasing dneg) at a single row, a ragged size and several tiles,
    # with and without down-scoring, at both widths
    in_batch = {(B, 64 if D <= 64 else 128, ds) for B, N, D, ds, T, ib in KERNEL_CASES if ib}
    assert all(B == N for B, N, *_, ib in KERNEL_CASES if ib)
    assert {(B, w, ds) for B in (1, 37, 1024) for w in (64, 128) for ds in (True, False)} <= in_batch
