"""Block plumbing for the H100 hot path: lazy device weights, Keras-style initialisers, the
reference's dict-of-features conventions (sorted-name aggregation, `__values`/`__offsets` ragged
pairs) and a Prediction record.

This is deliberately NOT the reference's block algebra (merlin/models/tf/core/, 3.7 kLoC of Keras
layer composition): a model here is a short list of blocks that launch fused kernels through
models_b200.ops.  What is kept are the names, constructor arguments, call protocol and error
messages a user of the hot path sees.
"""
from __future__ import annotations

import itertools
import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import ops

TabularData = Dict[str, torch.Tensor]

_SEED = [0x5EED]
_NAME_COUNTER: Dict[str, itertools.count] = {}


def set_seed(seed: int) -> None:
    """Seed for weight initialisation (each variable draws from its own derived generator)."""
    _SEED[0] = int(seed)
    _NAME_COUNTER.clear()


def unique_name(base: str) -> str:
    """Keras-style auto names: base, base_1, base_2, ..."""
    c = _NAME_COUNTER.setdefault(base, itertools.count())
    i = next(c)
    return base if i == 0 else f"{base}_{i}"


# Cached scratch buffers (e.g. the split-bf16 operand buffers of the dense layers) are keyed by a
# namespace so that two CUDA graphs of the same model that may run concurrently never share scratch.
_BUFFER_NS = [0]
_NEXT_NS = itertools.count(1)


_WEIGHTS_VERSION = [0]


def weights_version() -> int:
    """Bumped whenever a variable is reassigned (load_weights / set_weights).  Derived state — BatchNorm-folded
    layers, captured CUDA graphs (graph.CompiledForward re-captures when it changes) — is keyed by it."""
    return _WEIGHTS_VERSION[0]


def bump_weights_version() -> int:
    _WEIGHTS_VERSION[0] += 1
    return _WEIGHTS_VERSION[0]


def buffer_namespace() -> int:
    return _BUFFER_NS[0]


def new_buffer_namespace() -> int:
    return next(_NEXT_NS)


def set_buffer_namespace(ns: int) -> int:
    old = _BUFFER_NS[0]
    _BUFFER_NS[0] = int(ns)
    return old


def default_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(
            "models_b200 needs a CUDA device: the hot path is hand-written sm_90a kernels and has no "
            "CPU fallback (the CPU restatement lives in oracle/ and is test infrastructure only)"
        )
    return torch.device("cuda", torch.cuda.current_device())


# ------------------------------------------------------------------------------------------------
# initialisers (Keras names used by the reference: "uniform" inputs/embedding.py:205,
# "glorot_uniform"/"zeros" blocks/mlp.py:39-40, "truncated_normal" blocks/cross.py:34,
# TruncatedNormal(0, 0.05) inputs/embedding.py:1050)
# ------------------------------------------------------------------------------------------------
InitializerType = Union[str, Callable, np.ndarray, torch.Tensor]


def _generator(device, salt: str) -> torch.Generator:
    g = torch.Generator(device=device)
    h = 1469598103934665603
    for ch in salt.encode():
        h = ((h ^ ch) * 1099511628211) & (2**63 - 1)
    g.manual_seed((_SEED[0] * 1000003 + h) & (2**63 - 1))
    return g


def create_variable(shape: Tuple[int, ...], initializer: InitializerType, device, name: str) -> torch.Tensor:
    shape = tuple(int(s) for s in shape)
    if isinstance(initializer, (np.ndarray, torch.Tensor)):
        if isinstance(initializer, np.ndarray):
            initializer = np.array(initializer, dtype=np.float32)  # private writable copy (frames can be read-only)
        t = torch.as_tensor(initializer, dtype=torch.float32)
        if tuple(t.shape) != shape:
            raise ValueError(f"{name}: initial value has shape {tuple(t.shape)}, expected {shape}")
        return t.to(device).contiguous()
    if callable(initializer):
        t = torch.as_tensor(initializer(shape), dtype=torch.float32)
        return t.to(device).contiguous()
    if isinstance(initializer, dict) and "hash_seed" in initializer:
        # bit-reproducible on the host (oracle.hash_table_rows): used for multi-GiB tables
        w = torch.empty(shape, dtype=torch.float32, device=device)
        return ops.init_uniform_hash(w, initializer["hash_seed"], initializer.get("lo", -0.05),
                                     initializer.get("hi", 0.05))
    init = (initializer or "zeros").lower() if isinstance(initializer, str) or initializer is None else initializer
    g = _generator(device, name)
    w = torch.empty(shape, dtype=torch.float32, device=device)
    if init == "zeros":
        return w.zero_()
    if init == "ones":
        return w.fill_(1.0)
    if init in ("uniform", "random_uniform"):
        return w.uniform_(-0.05, 0.05, generator=g)
    if init == "glorot_uniform":
        fan_in, fan_out = (shape[0], shape[1]) if len(shape) == 2 else (shape[0], shape[0])
        limit = math.sqrt(6.0 / (fan_in + fan_out))
        return w.uniform_(-limit, limit, generator=g)
    if init == "glorot_normal":
        fan_in, fan_out = (shape[0], shape[1]) if len(shape) == 2 else (shape[0], shape[0])
        std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
        return torch.nn.init.trunc_normal_(w, 0.0, std, -2 * std, 2 * std, generator=g)
    if init in ("truncated_normal", "random_normal", "normal"):
        std = 0.05
        if init == "truncated_normal":
            return torch.nn.init.trunc_normal_(w, 0.0, std, -2 * std, 2 * std, generator=g)
        return w.normal_(0.0, std, generator=g)
    raise ValueError(f"Unknown initializer {initializer!r}")


# ------------------------------------------------------------------------------------------------
# feature dict helpers
# ------------------------------------------------------------------------------------------------
def as_device_tensor(v, device) -> torch.Tensor:
    if isinstance(v, torch.Tensor):
        return v if v.device == device else v.to(device, non_blocking=True)
    return torch.as_tensor(np.asarray(v)).to(device, non_blocking=True)


def to_device(batch: Dict[str, object], device=None) -> TabularData:
    device = device or default_device()
    return {k: as_device_tensor(v, device) for k, v in batch.items()}


def batch_size_of(inputs: TabularData) -> int:
    for k, v in inputs.items():
        if k.endswith("__offsets"):
            return int(v.numel()) - 1
        if not k.endswith("__values"):
            return int(v.shape[0])
    raise ValueError("cannot infer the batch size from an empty / values-only feature dict")


def get_feature(inputs: TabularData, name: str):
    """Scalar/dense feature tensor, or the ragged pair (values, offsets) for a list feature given as
    `name__values` + `name__offsets` (merlin/models/tf/transforms/features.py:190-210)."""
    if name in inputs:
        return inputs[name]
    if name + "__values" in inputs:
        if name + "__offsets" not in inputs:
            raise ValueError(f"feature {name!r}: `{name}__values` given without `{name}__offsets`")
        return (inputs[name + "__values"], inputs[name + "__offsets"])
    raise KeyError(name)


def has_feature(inputs: TabularData, name: str) -> bool:
    return name in inputs or (name + "__values") in inputs


def concat_sorted(d: TabularData, device=None) -> torch.Tensor:
    """ConcatFeatures (core/aggregation.py:54-66): pieces in sorted(name) order, cast to fp32 —
    one mm_concat_columns launch writing the (B, sum k_i) matrix."""
    keys = sorted(d)
    pieces = [d[k] for k in keys]
    B = pieces[0].shape[0]
    width = sum(1 if p.dim() == 1 else p.shape[1] for p in pieces)
    out = torch.empty((B, width), dtype=torch.float32, device=pieces[0].device)
    return ops.concat_columns(pieces, out)


# ------------------------------------------------------------------------------------------------
# blocks
# ------------------------------------------------------------------------------------------------
class Block:
    """Callable unit with lazily created device weights (Keras `build` on first call)."""

    # attribute -> value restored when the block is pickled (models_b200/io.py): caches and device scratch
    # derived from the variables are rebuilt on demand instead of being written to disk
    _TRANSIENT: Dict[str, object] = {}

    def __init__(self, name: Optional[str] = None):
        self.name = name or unique_name(_snake(type(self).__name__))
        self.built = False

    def __getstate__(self):
        import copy as _copy

        state = dict(self.__dict__)
        for klass in type(self).__mro__:
            for k, v in vars(klass).get("_TRANSIENT", {}).items():
                if k in state:
                    state[k] = _copy.copy(v)
        return state

    def build(self, device=None) -> "Block":
        self.built = True
        return self

    def __call__(self, inputs, **kwargs):
        return self.call(inputs, **kwargs)

    def call(self, inputs, **kwargs):  # pragma: no cover - abstract
        raise NotImplementedError

    def weights(self) -> Dict[str, torch.Tensor]:
        """name -> device tensor (Keras-style variable names)."""
        return {}

    def connect(self, *blocks: "Block") -> "SequentialBlock":
        layers = list(self.layers) if isinstance(self, SequentialBlock) else [self]
        for b in blocks:
            layers.extend(b.layers if isinstance(b, SequentialBlock) else [b])
        return SequentialBlock(layers)

    def copy(self) -> "Block":
        """Keras `copy()` goes through from_config: the copy gets fresh layer names and therefore independently
        initialised variables.  Here variables are seeded from the layer name (create_variable), so a plain deepcopy
        of an unbuilt block would initialise, e.g., the default item tower identically to the query tower: every Block
        inside the copy gets a new unique name."""
        import copy as _copy
        import re as _re

        new = _copy.deepcopy(self)

        def rename(o, depth=0, seen=None):
            seen = set() if seen is None else seen
            if id(o) in seen or depth > 8:
                return
            seen.add(id(o))
            if isinstance(o, Block):
                base = _re.sub(r"_\d+$", "", o.name.split("/")[-1]) or "block"
                o.name = unique_name(base)
                for v in vars(o).values():
                    rename(v, depth + 1, seen)
            elif isinstance(o, (list, tuple)):
                for v in o:
                    rename(v, depth + 1, seen)
            elif isinstance(o, dict):
                for v in o.values():
                    rename(v, depth + 1, seen)

        rename(new)
        return new


class SequentialBlock(Block):
    def __init__(self, layers: Sequence[Block], name: Optional[str] = None, block_name: Optional[str] = None):
        super().__init__(name or unique_name("sequential_block"))
        self.layers: List[Block] = [l for l in layers if l is not None]
        self.block_name = block_name

    def call(self, inputs, **kwargs):
        x = inputs
        for layer in self.layers:
            x = layer(x, **kwargs)
        return x

    def weights(self):
        out = {}
        for l in self.layers:
            for k, v in l.weights().items():
                out[f"{l.name}/{k}"] = v
        return out

    def __len__(self):
        return len(self.layers)

    def __iter__(self):
        return iter(self.layers)

    def __getitem__(self, i):
        return self.layers[i]


class Prediction:
    """merlin/models/tf/core/prediction.py:25-86 — (outputs, targets[, negative ids])."""

    def __init__(self, outputs, targets=None, negative_candidate_ids=None, **extra):
        self.outputs = outputs
        self.targets = targets
        self.negative_candidate_ids = negative_candidate_ids
        self.extra = extra

    @property
    def predictions(self):
        return self.outputs

    def __iter__(self):
        return iter((self.outputs, self.targets))


PredictionOutput = Prediction


def _snake(name: str) -> str:
    out = []
    for i, ch in enumerate(name):
        if ch.isupper() and i and (not name[i - 1].isupper() or (i + 1 < len(name) and name[i + 1].islower())):
            out.append("_")
        out.append(ch.lower())
    return "".join(out).lstrip("_")
