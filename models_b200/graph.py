"""Host-side runtime for the hot path: packed pinned host batches and CUDA-graph replay.

At B = 65 536 a DLRM forward is ~0.3 ms of GPU work spread over ~10 kernels; launching them one
by one from Python (argument checks, ctypes, tensor-map encodes, allocator calls) costs more host
time than that.  `CompiledForward` captures the whole forward once into a CUDA graph over static
device buffers and replays it: one H2D copy of a packed pinned batch, one graph launch, one D2H copy
of the predictions.  This is the reference-facing "call a user makes" for serving: host buffers in,
host predictions out (`Model.compile(example_batch)`), and what bench.py reports as `e2e`.
"""
from __future__ import annotations

import contextlib
import gc
from typing import Dict, Optional

import numpy as np
import torch

from .core import Prediction, default_device, new_buffer_namespace, set_buffer_namespace

_ALIGN = 256


@contextlib.contextmanager
def graph_capture(graph: torch.cuda.CUDAGraph):
    """torch.cuda.graph(graph) with Python's cyclic garbage collector kept out of the capture.  A CUDA graph that sits in
    an unreachable reference cycle (a dropped model, trainer or compiled forward) is destroyed whenever the collector
    runs; destroying a graph while a stream is capturing invalidates that capture.  So pending garbage is collected
    first and the collector stays off until the capture ends."""
    enabled = gc.isenabled()
    gc.collect()
    gc.disable()
    try:
        with torch.cuda.graph(graph):
            yield
    finally:
        if enabled:
            gc.enable()


class HostBatch:
    """All input columns of one batch inside ONE pinned host allocation (so the H2D transfer is a
    single cudaMemcpyAsync), exposed as per-column NumPy / torch views."""

    def __init__(self, spec: Dict[str, tuple]):
        """spec: name -> (shape tuple, numpy dtype)."""
        self.spec = {k: (tuple(int(x) for x in shp), np.dtype(dt)) for k, (shp, dt) in spec.items()}
        self.offsets: Dict[str, int] = {}
        off = 0
        for name, (shp, dt) in self.spec.items():
            self.offsets[name] = off
            nbytes = int(np.prod(shp, dtype=np.int64)) * dt.itemsize
            off += (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        self.nbytes = off
        self.buffer = torch.empty(max(off, _ALIGN), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
        self.columns: Dict[str, torch.Tensor] = {name: _view(self.buffer, self.offsets[name], shp, dt)
                                                 for name, (shp, dt) in self.spec.items()}

    @classmethod
    def like(cls, batch: Dict[str, np.ndarray], names=None, id_bytes: Optional[Dict[str, int]] = None) -> "HostBatch":
        """Layout for batches shaped like `batch`.  `id_bytes` (`Model.id_bytes()`): integer id columns listed
        there travel packed — 1 -> uint8 (B,), 2 -> uint16 (B,), 3 -> uint8 (B,3) little-endian — instead
        of int32/int64; `fill` narrows them (ids must lie in [0, 2^(8*width)))."""
        names = list(batch) if names is None else list(names)
        spec = {}
        for k in names:
            a = np.asarray(batch[k])
            w = (id_bytes or {}).get(k)
            if w in (1, 2, 3) and a.dtype.kind in "iu" and (a.ndim == 1 or (a.ndim == 2 and a.shape[1] == 1)):
                spec[k] = ((a.shape[0],), np.uint8) if w == 1 else ((a.shape[0],), np.uint16) if w == 2 else ((a.shape[0], 3), np.uint8)
            else:
                spec[k] = (a.shape, a.dtype)
        hb = cls(spec)
        hb.fill(batch)
        return hb

    def fill(self, batch: Dict[str, np.ndarray]) -> "HostBatch":
        for name, (shp, dt) in self.spec.items():
            src = np.asarray(batch[name])
            dst = self.columns[name].numpy()
            if src.shape == shp and src.dtype == dt:
                dst[...] = src
                continue
            width = {(1, 1): 1, (1, 2): 2, (2, 1): 3}.get((len(shp), dt.itemsize)) if dt.kind == "u" else None
            if width is None or src.dtype.kind not in "iu" or src.size != shp[0]:
                raise ValueError(f"column {name!r}: expected {shp} {dt}, got {src.shape} {src.dtype}")
            flat = src.reshape(-1)
            if flat.size and (int(flat.min()) < 0 or int(flat.max()) >= (1 << (8 * width))):
                raise ValueError(f"column {name!r}: ids outside [0, 2^{8 * width}) cannot travel as {width}-byte ids")
            if width == 3:
                dst[...] = flat.astype("<u4").view(np.uint8).reshape(-1, 4)[:, :3]
            else:
                dst[...] = flat.astype(dt)
        return self

    def payload_bytes(self) -> int:
        return sum(int(np.prod(shp, dtype=np.int64)) * dt.itemsize for shp, dt in self.spec.values())


def _view(buf: torch.Tensor, off: int, shape, dt: np.dtype) -> torch.Tensor:
    n = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
    tdt = torch.from_numpy(np.empty(0, dtype=dt)).dtype
    return buf[off: off + n].view(tdt).view(*shape) if n else torch.empty(shape, dtype=tdt, device=buf.device)


class CompiledForward:
    """A model forward captured into a CUDA graph over static device buffers."""

    def __init__(self, model, example: HostBatch, device=None, **call_kwargs):
        self.model = model
        self.device = device or default_device()
        self.spec = example.spec
        self.offsets = example.offsets
        self.call_kwargs = call_kwargs
        self.dev_buffer = torch.empty(example.buffer.numel(), dtype=torch.uint8, device=self.device)
        self.inputs = {name: _view(self.dev_buffer, example.offsets[name], shp, dt) for name, (shp, dt) in self.spec.items()}
        self.dev_buffer.copy_(example.buffer, non_blocking=True)
        self._oob = model.index_error_counter(self.device)
        self.namespace = new_buffer_namespace()  # private scratch buffers: graphs may run concurrently
        self._capture()
        self.output_host = torch.empty(self.output.shape, dtype=self.output.dtype, pin_memory=True)
        self.host_result = self._as_result(self.output_host)
        self._oob_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self.check_indices(sync=True)

    def _capture(self) -> None:
        """Warm-up + capture over the static buffers.  Runs at construction and again whenever a model variable was
        reassigned since the last capture (core.weights_version): the graph holds raw pointers to derived buffers
        (split-bf16 kernels, folded layers) and scalar arguments (the fused head's bias) that a reassignment frees or
        changes, so replaying the old graph would read stale or freed memory."""
        from . import ops
        from .core import weights_version

        model = self.model
        model.defer_index_check(True)
        old_ns = set_buffer_namespace(self.namespace)
        try:
            # warm-up on a side stream (builds weights, split kernels, zeroed operand buffers, smem
            # attributes) — nothing lazy may remain for the capture
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._run()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count()
            with graph_capture(self.graph):
                out = self._run()
            self.launches_per_replay = ops.launch_count() - n0  # kernels of libmm_b200.so inside the graph
            names = None
            if isinstance(out, dict):  # several outputs: (B, 1) views of ONE (H, B) buffer -> one D2H copy
                names, out = list(out), _stacked_outputs(out)
            if getattr(self, "output", None) is not None and (out.shape != self.output.shape or out.dtype != self.output.dtype
                                                              or names != self.output_names):
                raise RuntimeError("re-capture changed the output layout")
            self.output, self.output_names = out, names
            self.device_result = self._as_result(out)
            self._wv = weights_version()
        finally:
            model.defer_index_check(False)
            set_buffer_namespace(old_ns)

    def _ensure_current(self) -> None:
        from .core import weights_version

        if weights_version() != self._wv:
            torch.cuda.synchronize()
            self._capture()

    def _run(self) -> torch.Tensor:
        out = self.model(self.inputs, **self.call_kwargs)
        return out.outputs if isinstance(out, Prediction) else out

    def _as_result(self, buf: torch.Tensor):
        """The output tensor of a single-output model; {name: (B, 1) view of row h} of the (H, B) buffer otherwise."""
        if self.output_names is None:
            return buf
        return {n: buf[h].view(-1, 1) for h, n in enumerate(self.output_names)}

    def check_indices(self, sync: bool = False) -> None:
        if self._oob is None:
            return
        if sync:
            n = int(self._oob.item())
        else:
            n = int(self._oob_host.item())
        if n:
            self._oob.zero_()
            raise IndexError(f"{n} indices out of range for the embedding tables "
                             "(TF raises InvalidArgumentError: indices[...] is not in [0, rows))")

    # ---- device-resident inputs: copy into the static buffer and replay ---------------------------
    def replay(self) -> torch.Tensor:
        self._ensure_current()
        self.graph.replay()
        return self.device_result

    def load_device(self, packed: torch.Tensor) -> None:
        """Device-to-device refresh of the static input buffer (packed layout of `HostBatch`)."""
        self.dev_buffer.copy_(packed, non_blocking=True)

    # ---- host in / host out ---------------------------------------------------------------------------
    def __call__(self, batch: HostBatch) -> torch.Tensor:
        """One H2D copy of the packed pinned batch, one graph launch, one D2H copy; returns the pinned
        host predictions (valid until the next call): a tensor, or {output name: (B, 1)} views of one pinned (H, B) buffer
        for a model with several outputs."""
        if batch.spec != self.spec:
            raise ValueError("batch layout differs from the one this forward was compiled for")
        self._ensure_current()
        self.dev_buffer.copy_(batch.buffer, non_blocking=True)
        self.graph.replay()
        self.output_host.copy_(self.output, non_blocking=True)
        if self._oob is not None:
            self._oob_host.copy_(self._oob, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.check_indices()
        return self.host_result


def _stacked_outputs(out: Dict[str, torch.Tensor]) -> torch.Tensor:
    """The (H, B) buffer behind a multi-output forward's {name: (B, 1)} views (models.ParallelOutputs.split)."""
    vals = list(out.values())
    base = vals[0]._base
    if base is None or base.dim() != 2 or base.shape[0] != len(vals) or not base.is_contiguous() or any(
            v._base is not base or v.data_ptr() != base[h].data_ptr() for h, v in enumerate(vals)):
        raise RuntimeError("a multi-output forward must return views of one (H, B) buffer, in output order")
    return base


class PipelinedForward:
    """`depth` CompiledForward instances on their own streams: while one batch computes, the next
    one's pinned H2D copy is already in flight (PCIe and the SMs overlap).  submit() returns a
    ticket, result(ticket) waits for that batch's pinned host predictions."""

    def __init__(self, model, example: HostBatch, depth: int = 2, **call_kwargs):
        if depth < 1:
            raise ValueError("depth must be >= 1")
        self.slots = [CompiledForward(model, example, **call_kwargs) for _ in range(depth)]
        dev = self.slots[0].device
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(depth)]
        self.done = [torch.cuda.Event() for _ in range(depth)]
        self.busy = [False] * depth
        self.n = 0

    def submit(self, batch: HostBatch) -> int:
        k = self.n % len(self.slots)
        if self.busy[k]:
            raise RuntimeError("pipeline slot still holds an uncollected result: call result() first")
        cf, st = self.slots[k], self.streams[k]
        if batch.spec != cf.spec:
            raise ValueError("batch layout differs from the one this forward was compiled for")
        cf._ensure_current()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            cf.dev_buffer.copy_(batch.buffer, non_blocking=True)
            cf.graph.replay()
            cf.output_host.copy_(cf.output, non_blocking=True)
            if cf._oob is not None:
                cf._oob_host.copy_(cf._oob, non_blocking=True)
            self.done[k].record(st)
        self.busy[k] = True
        self.n += 1
        return k

    def submit_device(self, packed: torch.Tensor) -> int:
        """Same as submit() for a batch that is already resident on the device (packed HostBatch layout):
        D2D refresh of the slot's static input buffer + graph replay on the slot's stream; no D2H."""
        k = self.n % len(self.slots)
        cf, st = self.slots[k], self.streams[k]
        cf._ensure_current()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            cf.dev_buffer.copy_(packed, non_blocking=True)
            cf.graph.replay()
            self.done[k].record(st)
        self.n += 1
        return k

    def join(self) -> None:
        """Make the current stream wait for everything submitted so far."""
        for st in self.streams:
            torch.cuda.current_stream().wait_stream(st)

    def output(self, ticket: int) -> torch.Tensor:
        return self.slots[ticket].device_result

    def result(self, ticket: int) -> torch.Tensor:
        self.done[ticket].synchronize()
        self.busy[ticket] = False
        self.slots[ticket].check_indices()
        return self.slots[ticket].host_result


def _uniq_clones(ts):
    """Clones of a list of tensors (entries may be None or repeat: a repeated tensor is cloned once)."""
    seen = {}
    return [None if t is None else seen.setdefault(id(t), t.clone()) for t in ts]


class EvalGraph:
    """One evaluation step of a ranking model — the logits forward (RankingModel.logits) and the metric update
    (metrics.MetricsState.update) — captured into a CUDA graph over static device buffers, for batches of one layout.
    `replay` refreshes the static buffers (device-to-device, all columns in a few multi-tensor copies) and launches the graph.  Re-captured when a
    model variable was reassigned or trained since the capture (core.weights_version), as CompiledForward is."""

    def __init__(self, model, state, inputs: Dict[str, torch.Tensor], targets, sample_weight):
        self.model, self.state = model, state
        self.key = self.layout(inputs, targets, sample_weight, state.device)
        self.inputs = {k: v.clone() for k, v in inputs.items()}
        self.targets = _uniq_clones(targets)
        self.sample_weight = None if sample_weight is None else _uniq_clones(sample_weight)
        self.namespace = new_buffer_namespace()  # private scratch buffers of the captured forward
        self._capture()

    @staticmethod
    def layout(inputs, targets, sample_weight, device) -> Optional[tuple]:
        """Shapes and dtypes of a batch, or None when it cannot be replayed: a ragged feature (its number of ids changes from
        batch to batch) or a column that is not a tensor on `device`."""
        cols = list(inputs.items()) + [(f"#y{h}", t) for h, t in enumerate(targets)]
        cols += [(f"#w{h}", w) for h, w in enumerate(sample_weight or []) if w is not None]
        key = []
        for k, v in cols:
            if not isinstance(v, torch.Tensor) or v.device != device or k.endswith("__values") or k.endswith("__offsets"):
                return None
            key.append((k, tuple(v.shape), v.dtype))
        shared = list(targets) + list(sample_weight or [])  # which entries are one tensor (one static copy)
        key.append(tuple(next(i for i, u in enumerate(shared) if u is t) for t in shared if t is not None))
        return tuple(key)

    def _step(self) -> None:
        self.model._eval_step(self.state, self.inputs, self.targets, self.sample_weight)

    def _capture(self) -> None:
        from . import ops
        from .core import weights_version

        st = self.state
        saved = (st.state.clone(), st.before_last.clone(), None if st.reg is None else st.reg.clone())
        old_ns = set_buffer_namespace(self.namespace)
        try:
            # warm-up on a side stream (split kernels, scratch buffers, the fused head's host bias, the metric workspace);
            # it adds two batches into the state, which is restored afterwards
            s = torch.cuda.Stream(device=st.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._step()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            st.state.copy_(saved[0])
            st.before_last.copy_(saved[1])
            if st.reg is not None:  # created by the warm-up when the model has an L2 term
                st.reg.copy_(saved[2]) if saved[2] is not None else st.reg.zero_()
            self.workspace = st.workspace  # the graph holds its address: keep it alive
            self.graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count()
            with graph_capture(self.graph):
                self._step()
            self.launches_per_replay = ops.launch_count() - n0
            self._wv = weights_version()
        finally:
            set_buffer_namespace(old_ns)

    def replay(self, inputs: Dict[str, torch.Tensor], targets, sample_weight) -> None:
        from .core import weights_version

        if weights_version() != self._wv:
            torch.cuda.synchronize()
            self._capture()
        dst, src, done = list(self.inputs.values()), [inputs[k] for k in self.inputs], set()
        for mine, theirs in zip(self.targets + (self.sample_weight or []), list(targets) + list(sample_weight or [])):
            if mine is not None and id(mine) not in done:
                dst.append(mine)
                src.append(theirs)
                done.add(id(mine))
        groups: Dict[torch.dtype, tuple] = {}
        for d, s_ in zip(dst, src):
            g = groups.setdefault(d.dtype, ([], []))
            g[0].append(d)
            g[1].append(s_)
        for d, s_ in groups.values():  # one multi-tensor copy per dtype instead of one launch per column
            torch._foreach_copy_(d, s_, non_blocking=True)
        self.graph.replay()
