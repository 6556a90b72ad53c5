"""Learning-rate schedules: the five built-in schedules of tf.keras.optimizers.schedules (TF 2.9-2.12), with Keras'
argument names and defaults.  `SGD`, `Adagrad` and `Adam` take one as `learning_rate`; the training step evaluates it
on the device from the optimizer's step counter (include/mm_b200.h K25, mm_opt_tick_schedule), so a captured CUDA graph
follows the schedule without host work.  `step` below is the optimizer's `iterations` before the update: 0 on the first
step, as Keras' OptimizerV2._decayed_lr.  `__call__` is a float64 evaluation on the host."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np


class LearningRateSchedule:
    """Base of the built-in schedules.  Only the built-in classes themselves train: a subclass would need a host
    evaluation per step, which a captured graph cannot do."""

    def __call__(self, step) -> float:  # pragma: no cover - abstract
        raise NotImplementedError

    def get_config(self) -> dict:  # pragma: no cover - abstract
        raise NotImplementedError

    @classmethod
    def from_config(cls, config: dict) -> "LearningRateSchedule":
        return cls(**config)

    def device_params(self) -> np.ndarray:
        """The K25 device array (ops.schedule_params) of this schedule."""
        raise NotImplementedError  # pragma: no cover - abstract

    def __eq__(self, other) -> bool:
        return type(other) is type(self) and other.get_config() == self.get_config()

    def __repr__(self) -> str:
        return f"{type(self).__name__}({self.get_config()})"


def _decay_steps(v) -> float:
    if not float(v) > 0:
        raise ValueError(f"decay_steps must be > 0, got {v}")
    return v


class ExponentialDecay(LearningRateSchedule):
    """initial_learning_rate * decay_rate ** (step / decay_steps), the exponent floored when staircase."""

    def __init__(self, initial_learning_rate: float, decay_steps, decay_rate: float, staircase: bool = False,
                 name: Optional[str] = None):
        self.initial_learning_rate, self.decay_steps = initial_learning_rate, _decay_steps(decay_steps)
        self.decay_rate, self.staircase, self.name = decay_rate, bool(staircase), name

    def __call__(self, step) -> float:
        p = float(step) / float(self.decay_steps)
        if self.staircase:
            p = math.floor(p)
        return float(self.initial_learning_rate) * float(self.decay_rate) ** p

    def get_config(self) -> dict:
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "decay_rate": self.decay_rate, "staircase": self.staircase, "name": self.name}

    def device_params(self) -> np.ndarray:
        from .ops import schedule_params

        return schedule_params("ExponentialDecay", self.initial_learning_rate, self.decay_steps, self.decay_rate,
                               flag=self.staircase)


class PiecewiseConstantDecay(LearningRateSchedule):
    """values[0] up to and including boundaries[0], values[i] on (boundaries[i-1], boundaries[i]], values[-1] after."""

    def __init__(self, boundaries: Sequence, values: Sequence, name: Optional[str] = None):
        if len(boundaries) != len(values) - 1:
            raise ValueError("The length of boundaries should be 1 less than the length of values")
        self.boundaries, self.values, self.name = list(boundaries), list(values), name
        self.device_params()  # the device schedule's limits, refused here rather than at the first step

    def __call__(self, step) -> float:
        s = float(step)
        for b, v in zip(self.boundaries, self.values):
            if s <= float(b):
                return float(v)
        return float(self.values[-1])

    def get_config(self) -> dict:
        return {"boundaries": self.boundaries, "values": self.values, "name": self.name}

    def device_params(self) -> np.ndarray:
        from .ops import schedule_params

        return schedule_params("PiecewiseConstantDecay", boundaries=self.boundaries, values=self.values)


class PolynomialDecay(LearningRateSchedule):
    """(initial - end) * (1 - step' / D) ** power + end: without cycle step' = min(step, decay_steps), D = decay_steps;
    with cycle step' = step, D = decay_steps * max(1, ceil(step / decay_steps))."""

    def __init__(self, initial_learning_rate: float, decay_steps, end_learning_rate: float = 0.0001, power: float = 1.0,
                 cycle: bool = False, name: Optional[str] = None):
        self.initial_learning_rate, self.decay_steps = initial_learning_rate, _decay_steps(decay_steps)
        self.end_learning_rate, self.power, self.cycle, self.name = end_learning_rate, power, bool(cycle), name

    def __call__(self, step) -> float:
        s, ds = float(step), float(self.decay_steps)
        if self.cycle:
            d = ds * max(1.0, math.ceil(s / ds))
        else:
            s, d = min(s, ds), ds
        init, end = float(self.initial_learning_rate), float(self.end_learning_rate)
        return (init - end) * (1.0 - s / d) ** float(self.power) + end

    def get_config(self) -> dict:
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "end_learning_rate": self.end_learning_rate, "power": self.power, "cycle": self.cycle, "name": self.name}

    def device_params(self) -> np.ndarray:
        from .ops import schedule_params

        return schedule_params("PolynomialDecay", self.initial_learning_rate, self.decay_steps, self.end_learning_rate,
                               self.power, self.cycle)


class InverseTimeDecay(LearningRateSchedule):
    """initial_learning_rate / (1 + decay_rate * step / decay_steps), the quotient floored when staircase."""

    def __init__(self, initial_learning_rate: float, decay_steps, decay_rate: float, staircase: bool = False,
                 name: Optional[str] = None):
        self.initial_learning_rate, self.decay_steps = initial_learning_rate, _decay_steps(decay_steps)
        self.decay_rate, self.staircase, self.name = decay_rate, bool(staircase), name

    def __call__(self, step) -> float:
        p = float(step) / float(self.decay_steps)
        if self.staircase:
            p = math.floor(p)
        return float(self.initial_learning_rate) / (1.0 + float(self.decay_rate) * p)

    def get_config(self) -> dict:
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "decay_rate": self.decay_rate, "staircase": self.staircase, "name": self.name}

    def device_params(self) -> np.ndarray:
        from .ops import schedule_params

        return schedule_params("InverseTimeDecay", self.initial_learning_rate, self.decay_steps, self.decay_rate,
                               flag=self.staircase)


class CosineDecay(LearningRateSchedule):
    """initial * ((1 - alpha) * 0.5 * (1 + cos(pi * min(step, decay_steps) / decay_steps)) + alpha)."""

    def __init__(self, initial_learning_rate: float, decay_steps, alpha: float = 0.0, name: Optional[str] = None):
        self.initial_learning_rate, self.decay_steps = initial_learning_rate, _decay_steps(decay_steps)
        self.alpha, self.name = alpha, name

    def __call__(self, step) -> float:
        frac = min(float(step), float(self.decay_steps)) / float(self.decay_steps)
        a = float(self.alpha)
        return float(self.initial_learning_rate) * ((1.0 - a) * 0.5 * (1.0 + math.cos(math.pi * frac)) + a)

    def get_config(self) -> dict:
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "alpha": self.alpha, "name": self.name}

    def device_params(self) -> np.ndarray:
        from .ops import schedule_params

        return schedule_params("CosineDecay", self.initial_learning_rate, self.decay_steps, self.alpha)


_BUILT_IN = {c.__name__: c for c in (ExponentialDecay, PiecewiseConstantDecay, PolynomialDecay, InverseTimeDecay,
                                     CosineDecay)}


def serialize(schedule: LearningRateSchedule) -> dict:
    """Keras' serialised form {"class_name": ..., "config": ...}."""
    return {"class_name": type(schedule).__name__, "config": schedule.get_config()}


def deserialize(config: dict) -> LearningRateSchedule:
    cls = _BUILT_IN.get(config.get("class_name"))
    if cls is None:
        raise ValueError(f"unknown learning-rate schedule {config.get('class_name')!r}; supported: {sorted(_BUILT_IN)}")
    return cls.from_config(dict(config["config"]))


def check_trainable(lr) -> None:
    """Refuse a learning rate the device cannot follow: a callable or a LearningRateSchedule other than the built-ins."""
    if type(lr) not in _BUILT_IN.values():
        raise NotImplementedError(f"learning_rate={type(lr).__name__}: only a float or one of the built-in schedules "
                                  f"{sorted(_BUILT_IN)} is implemented (the device evaluates the schedule each step; another "
                                  "callable would need a host evaluation per step, which a captured CUDA graph cannot do)")
