"""mm_opt_tick_schedule (include/mm_b200.h K25): every schedule kind over 300 ticks, the learning rate and Adam's
bias-corrected rate read back against the float64 restatement, and the argument checks of ops.opt_tick_schedule."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, ops
from tests.test_optimizer_schedules_host import CASES, keras_lr

pytestmark = pytest.mark.gpu

FP32 = 2.0 ** -23


@pytest.mark.parametrize("kind,cfg", CASES + [("PiecewiseConstantDecay", dict(boundaries=[0, 1, 2, 150, 299],
                                                                              values=[6.0, 5.0, 4.0, 3.0, 2.0, 1.0]))],
                         ids=[f"{k}-{i}" for i, (k, _) in enumerate(CASES + [("PiecewiseConstantDecay", {})])])
def test_schedule_tick_matches_float64(device, kind, cfg):
    sch = getattr(mm.schedules, kind)(**cfg)
    opt = mm.Adam(sch, beta_1=0.9, beta_2=0.999)
    hyper = torch.from_numpy(opt.hyper()).to(device)
    sched = torch.from_numpy(sch.device_params()).to(device)
    n = 300
    got = torch.zeros((n, 3), dtype=torch.float32, device=device)
    for s in range(n):
        ops.opt_tick_schedule(hyper, sched)
        got[s] = hyper[[_cabi.HYPER_LR, _cabi.HYPER_LR_T, _cabi.HYPER_STEP]]
    got = got.double().cpu().numpy()
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    for s in range(n):
        lr = keras_lr(kind, cfg, s)
        lr_t = lr * np.sqrt(1 - b2 ** (s + 1)) / (1 - b1 ** (s + 1))
        # fp32 evaluation of s / decay_steps, pow and cos: a few ulp of the result (and of the exponent for pow)
        tol = 64 * FP32 * max(abs(lr), 1e-30) + 1e-12
        assert abs(got[s, 0] - lr) <= tol, (kind, s, got[s, 0], lr)
        # lr_t: mm_opt_tick's fp32 1 - b2^t loses up to ~1e-4 of itself at small t
        assert abs(got[s, 1] - lr_t) <= 1e-4 * abs(lr_t) + tol, (kind, s, got[s, 1], lr_t)
        assert got[s, 2] == s + 1
    # the exactly representable cases are exact
    if kind == "PiecewiseConstantDecay":
        assert all(got[s, 0] == np.float32(keras_lr(kind, cfg, s)) for s in range(n))


def test_tick_without_schedule_is_unchanged(device):
    """A float learning rate keeps mm_opt_tick: one launch, lr untouched."""
    opt = mm.Adagrad(0.25)
    h = torch.from_numpy(opt.hyper()).to(device)
    n0 = ops.launch_count()
    ops.opt_tick(h)
    assert ops.launch_count() - n0 == 1 and float(h[_cabi.HYPER_LR]) == 0.25 and float(h[_cabi.HYPER_STEP]) == 1


def test_opt_tick_schedule_argument_checks(device):
    h = torch.zeros(_cabi.HYPER_COUNT, device=device)
    s = torch.from_numpy(mm.schedules.CosineDecay(0.1, 10).device_params()).to(device)
    with pytest.raises(ValueError, match="hyper must hold"):
        ops.opt_tick_schedule(h[:4], s)
    with pytest.raises(ValueError, match="sched must hold"):
        ops.opt_tick_schedule(h, s[:-1])
    with pytest.raises(ValueError, match="sched must hold"):
        ops.opt_tick_schedule(h, torch.zeros((_cabi.SCHED_COUNT, 2), device=device)[:, 0])
    with pytest.raises(TypeError, match="float32"):
        ops.opt_tick_schedule(h, s.double())
    with pytest.raises(TypeError, match="float32"):
        ops.opt_tick_schedule(h.half(), s)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.opt_tick_schedule(h, s.cpu())
    n0 = ops.launch_count()
    ops.opt_tick_schedule(h, s)
    assert ops.launch_count() - n0 == 1 and float(h[_cabi.HYPER_LR]) == pytest.approx(0.1)
