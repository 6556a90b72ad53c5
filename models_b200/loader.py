"""The step before the hot path (SURVEY §8f-3): parquet / DataFrame / dict-of-arrays -> device batches in the
reference's input convention.

Reference: `mm.Loader` (merlin/models/tf/loader.py:135-365, on top of merlin.dataloader) and
`sample_batch` (:367-420).  What is kept is what the model sees: `(inputs, targets)` per batch, `inputs` a
dict keyed by schema column names, scalar features `(B,)`, list features as the ragged pair `name__values` +
`name__offsets` (int32 offsets of length B+1, transforms/features.py:190-210), targets split off by the TARGET
tag; `shuffle`, `drop_last`, `global_size` / `global_rank` sharding (one loader per GPU process, as Horovod
does), `peek()`, `len()`, `output_schema`.

H100 hand-off: every batch is packed on the host into ONE pinned allocation (HostBatch) and moved with ONE
cudaMemcpyAsync on a copy stream; a background thread packs batch i+1 while batch i is consumed, and an event
orders the consumer's stream after the copy — so parquet decode, host packing and H2D all overlap the forward.
Categorical ids are narrowed to int32 when the schema's domain allows (halves the index traffic of the gather).
"""
from __future__ import annotations

import os
import queue
import threading
from typing import Dict, Iterator, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .core import default_device
from .graph import HostBatch, _view
from .schema import Schema, Tags

Batch = Tuple[Dict[str, torch.Tensor], Optional[Union[torch.Tensor, Dict[str, torch.Tensor]]]]


# ------------------------------------------------------------------------------------------------
# sources -> column arrays
# ------------------------------------------------------------------------------------------------
class _Columns:
    """Column store on the host: scalar columns as 1-D arrays, list columns as (values, offsets int64)."""

    def __init__(self):
        self.scalar: Dict[str, np.ndarray] = {}
        self.ragged: Dict[str, Tuple[np.ndarray, np.ndarray]] = {}
        self.rows = 0

    def names(self) -> List[str]:
        return list(self.scalar) + list(self.ragged)


def _find_schema(path: str) -> Optional[Schema]:
    d = path if os.path.isdir(path) else os.path.dirname(path)
    for name in ("schema.pbtxt", "schema.json", os.path.join(".merlin", "schema.json")):
        p = os.path.join(d, name)
        if os.path.exists(p):
            return Schema.load(p)
    return None


def _from_arrow_table(table) -> _Columns:
    import pyarrow as pa

    cols = _Columns()
    cols.rows = table.num_rows
    for name in table.column_names:
        col = table.column(name).combine_chunks()
        if pa.types.is_list(col.type) or pa.types.is_large_list(col.type):
            if col.null_count:
                raise ValueError(f"column {name!r}: null lists are not supported")
            offsets = np.asarray(col.offsets.to_numpy(zero_copy_only=False), dtype=np.int64)
            values = col.values.to_numpy(zero_copy_only=False)
            base = int(offsets[0])
            cols.ragged[name] = (np.ascontiguousarray(values[base:int(offsets[-1])]), offsets - base)
        else:
            if col.null_count:
                raise ValueError(f"column {name!r} has {col.null_count} nulls: fill them in preprocessing (NVTabular FillMissing)")
            cols.scalar[name] = np.ascontiguousarray(col.to_numpy(zero_copy_only=False))
    return cols


def _from_mapping(data: Dict[str, np.ndarray]) -> _Columns:
    cols = _Columns()
    for k, v in data.items():
        if k.endswith("__values"):
            continue
        if k.endswith("__offsets"):
            base = k[: -len("__offsets")]
            cols.ragged[base] = (np.asarray(data[base + "__values"]), np.asarray(v, dtype=np.int64))
            cols.rows = len(v) - 1
        else:
            a = np.asarray(v)
            cols.scalar[k] = a.reshape(a.shape[0], -1)[:, 0] if a.ndim == 2 and a.shape[1] == 1 else a
            cols.rows = a.shape[0]
    return cols


def _read_source(src, columns: Optional[Sequence[str]]) -> Tuple[_Columns, Optional[Schema]]:
    schema = None
    if isinstance(src, dict):
        return _from_mapping(src), None
    if hasattr(src, "to_dict") and hasattr(src, "columns"):  # pandas DataFrame
        import pyarrow as pa

        return _from_arrow_table(pa.Table.from_pandas(src, preserve_index=False)), None
    import pyarrow.parquet as pq

    paths = [src] if isinstance(src, (str, os.PathLike)) else list(src)
    files: List[str] = []
    for p in paths:
        p = str(p)
        if os.path.isdir(p):
            files.extend(sorted(os.path.join(p, f) for f in os.listdir(p) if f.endswith(".parquet")))
            schema = schema or _find_schema(p)
        else:
            files.append(p)
            schema = schema or _find_schema(p)
    if not files:
        raise ValueError(f"no parquet files under {paths}")
    import pyarrow as pa

    tables = [pq.read_table(f, columns=list(columns) if columns else None) for f in files]
    return _from_arrow_table(pa.concat_tables(tables) if len(tables) > 1 else tables[0]), schema


# ------------------------------------------------------------------------------------------------
# the loader
# ------------------------------------------------------------------------------------------------
class Loader:
    """Iterates `(inputs, targets)` device batches over a parquet dataset / DataFrame / dict of arrays.

    Signature follows merlin/models/tf/loader.py:247-270; arguments that only configure the dask/NVTabular
    machinery of the reference (`engine`, `buffer_size`, `parts_per_chunk`, `reader_kwargs`, `sparse_*`) are
    accepted and ignored."""

    def __init__(self, paths_or_dataset, batch_size: int, label_names: Optional[Sequence[str]] = None,
                 feature_columns: Optional[Sequence[str]] = None, cat_names: Optional[Sequence[str]] = None,
                 cont_names: Optional[Sequence[str]] = None, engine=None, shuffle: bool = True, seed_fn=None,
                 buffer_size=0.1, device=None, parts_per_chunk: int = 1, reader_kwargs=None,
                 global_size: Optional[int] = None, global_rank: Optional[int] = None, drop_last: bool = False,
                 sparse_names=None, sparse_max=None, sparse_as_dense: bool = False, schema: Optional[Schema] = None,
                 index_dtype: str = "int32", prefetch: int = 2, id_bytes: Optional[Dict[str, int]] = None,
                 transforms: Optional[Sequence] = None, **loader_kwargs):
        if batch_size is None or int(batch_size) <= 0:
            raise ValueError("`batch_size` must be a positive integer")
        self.batch_size = int(batch_size)
        cols, found = _read_source(paths_or_dataset, None)
        self.schema = schema or found
        have = set(cols.names())
        if self.schema is not None:
            tagged_cat = [c.name for c in self.schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)]
            tagged_cont = [c.name for c in self.schema.select_by_tag(Tags.CONTINUOUS).excluding_by_tag(Tags.TARGET)]
            tagged_label = [c.name for c in self.schema.select_by_tag(Tags.TARGET)]
        else:
            tagged_cat = tagged_cont = tagged_label = []
        self.label_names = list(label_names) if label_names is not None else [n for n in tagged_label if n in have]
        if feature_columns is not None:
            feats = list(feature_columns)
        elif cat_names is not None or cont_names is not None:
            feats = list(cat_names or []) + list(cont_names or [])
        elif self.schema is not None:
            feats = [n for n in tagged_cat + tagged_cont if n in have]
        else:
            feats = [n for n in cols.names() if n not in self.label_names]
        missing = [n for n in feats + self.label_names if n not in have]
        if missing:
            raise ValueError(f"columns {missing} are not in the dataset (has {sorted(have)})")
        # EmbeddingOperator transforms: their vectors stay on the device and are looked up by the model, so a batch
        # only has to carry each operator's lookup ids
        self.transforms = list(transforms or [])
        for op in self.transforms:
            from .pretrained import EmbeddingOperator

            if not isinstance(op, EmbeddingOperator):
                raise NotImplementedError(f"Loader transform {type(op).__name__} is not implemented (EmbeddingOperator only)")
            if op.lookup_key not in have:
                raise ValueError(f"EmbeddingOperator {op.embedding_name!r}: lookup key {op.lookup_key!r} is not in the dataset")
            if op.lookup_key not in feats:
                feats.append(op.lookup_key)
        self.feature_names = feats
        self.cat_names = [n for n in feats if n in (cat_names or tagged_cat)]
        self._cols = cols
        self.shuffle = bool(shuffle)
        self.drop_last = bool(drop_last)
        self.seed_fn = seed_fn
        self.global_size = int(global_size or 1)
        self.global_rank = int(global_rank or 0)
        if not 0 <= self.global_rank < self.global_size:
            raise ValueError("`global_rank` must be in [0, global_size)")
        self.device = torch.device(device) if device is not None else (default_device() if torch.cuda.is_available() else torch.device("cpu"))
        self.prefetch = max(1, int(prefetch))
        self._index_dtype = np.dtype(index_dtype)
        self._epoch = 0
        # `Model.id_bytes()`: scalar id columns listed here travel packed (1/2/3-byte unsigned) over PCIe
        self.id_bytes = {k: int(v) for k, v in (id_bytes or {}).items() if int(v) in (1, 2, 3)}
        self._casts = self._plan_casts()
        self._copy_stream = torch.cuda.Stream(device=self.device) if self.device.type == "cuda" else None

    # -- dtype policy -----------------------------------------------------------------------------
    def _plan_casts(self) -> Dict[str, np.dtype]:
        """Categorical ids -> int32 when they fit (schema domain, else the data's own range); continuous
        features and targets -> float32 unless integer targets are wanted as is."""
        casts: Dict[str, np.dtype] = {}
        for n in self.feature_names + self.label_names:
            arr = self._cols.scalar[n] if n in self._cols.scalar else self._cols.ragged[n][0]
            if np.issubdtype(arr.dtype, np.integer):
                hi = None
                cs = self.schema.get(n) if self.schema is not None else None
                if cs is not None and cs.int_domain is not None and cs.int_domain.max is not None:
                    hi = int(cs.int_domain.max)
                elif arr.size:
                    hi = int(arr.max())
                fits = hi is not None and hi < np.iinfo(self._index_dtype).max and (arr.size == 0 or int(arr.min()) >= np.iinfo(self._index_dtype).min)
                casts[n] = self._index_dtype if (fits and n not in self.label_names) else np.dtype(arr.dtype)
            elif np.issubdtype(arr.dtype, np.floating):
                casts[n] = np.dtype(np.float32)
            else:
                raise TypeError(f"column {n!r}: dtype {arr.dtype} is not numeric (encode strings with NVTabular Categorify first)")
        return casts

    # -- schema -----------------------------------------------------------------------------------
    @property
    def output_schema(self) -> Optional[Schema]:
        if self.schema is None:
            return None
        out = self.schema.select_by_name(self.feature_names + self.label_names)
        for op in self.transforms:
            out = op.compute_output_schema(out)
        return out

    @property
    def input_schema(self) -> Optional[Schema]:
        return self.schema

    # -- iteration --------------------------------------------------------------------------------
    def _my_rows(self) -> np.ndarray:
        n = self._cols.rows
        order = np.arange(n, dtype=np.int64)
        if self.shuffle:
            seed = int(self.seed_fn()) if self.seed_fn is not None else 1234 + self._epoch
            order = np.random.default_rng(seed).permutation(n)
        if self.global_size > 1:  # every rank sees a disjoint, equally sized (+-1) slice of the same permutation
            order = order[self.global_rank::self.global_size]
        return order

    def __len__(self) -> int:
        n = len(range(self.global_rank, self._cols.rows, self.global_size))
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def _pack(self, rows: np.ndarray, contiguous: bool) -> Tuple[HostBatch, Dict[str, tuple]]:
        """Host side of one batch: gather the rows of every column into one pinned HostBatch."""
        arrays: Dict[str, np.ndarray] = {}
        lo, hi = (int(rows[0]), int(rows[-1]) + 1) if len(rows) else (0, 0)
        for n in self.feature_names + self.label_names:
            dt = self._casts[n]
            if n in self._cols.scalar:
                src = self._cols.scalar[n]
                arrays[n] = (src[lo:hi] if contiguous else src[rows]).astype(dt, copy=False)
            else:
                vals, off = self._cols.ragged[n]
                if contiguous:
                    v, o = vals[int(off[lo]):int(off[hi])], off[lo:hi + 1] - off[lo]
                else:
                    lens = off[rows + 1] - off[rows]
                    o = np.concatenate([[0], np.cumsum(lens)])
                    v = vals[np.repeat(off[rows] - o[:-1], lens) + np.arange(int(o[-1]))]
                arrays[n + "__values"] = v.astype(dt, copy=False)
                arrays[n + "__offsets"] = o.astype(np.int32)
        packed = {k: w for k, w in self.id_bytes.items() if k in self._cols.scalar and k in arrays and k not in self.label_names}
        hb = HostBatch.like(arrays, id_bytes=packed)
        return hb, hb.spec

    def _to_device(self, hb: HostBatch) -> Tuple[Dict[str, torch.Tensor], Optional[torch.cuda.Event]]:
        if self.device.type != "cuda":
            return {k: v.clone() for k, v in hb.columns.items()}, None
        with torch.cuda.stream(self._copy_stream):
            dev = torch.empty(hb.buffer.numel(), dtype=torch.uint8, device=self.device)
            dev.copy_(hb.buffer, non_blocking=True)  # ONE H2D for the whole batch
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        return {name: _view(dev, hb.offsets[name], shp, dt) for name, (shp, dt) in hb.spec.items()}, ev

    def _split(self, tensors: Dict[str, torch.Tensor]) -> Batch:
        inputs = {k: v for k, v in tensors.items() if k.split("__")[0] not in self.label_names or k in self.feature_names}
        targets = {n: tensors[n] for n in self.label_names if n in tensors}
        if not targets:
            return inputs, None
        return inputs, (next(iter(targets.values())) if len(targets) == 1 else targets)

    def _batches(self) -> Iterator[Tuple[np.ndarray, bool]]:
        order = self._my_rows()
        contiguous = not self.shuffle and self.global_size == 1
        stop = len(order) - (len(order) % self.batch_size if self.drop_last else 0)
        for s in range(0, stop, self.batch_size):
            yield order[s:min(stop, s + self.batch_size)], contiguous

    def __iter__(self) -> Iterator[Batch]:
        q: "queue.Queue" = queue.Queue(maxsize=self.prefetch)
        done = object()
        failure: List[BaseException] = []

        def producer():
            try:
                if self.device.type == "cuda":
                    torch.cuda.set_device(self.device)
                for rows, contiguous in self._batches():
                    hb, _ = self._pack(rows, contiguous)
                    q.put((hb,) + self._to_device(hb))
            except BaseException as e:  # surfaced in the consumer
                failure.append(e)
            finally:
                q.put(done)

        t = threading.Thread(target=producer, daemon=True, name="mm-loader")
        t.start()
        try:
            while True:
                item = q.get()
                if item is done:
                    break
                hb, tensors, ev = item
                if ev is not None:
                    torch.cuda.current_stream(self.device).wait_event(ev)  # consumer stream ordered after the H2D
                    for v in tensors.values():
                        v.record_stream(torch.cuda.current_stream(self.device))
                yield self._split(tensors)
        finally:
            self._epoch += 1
            while t.is_alive():  # drain so the producer can exit if the consumer stopped early
                try:
                    q.get(timeout=0.05)
                except queue.Empty:
                    pass
        if failure:
            raise failure[0]

    def peek(self) -> Batch:
        """First batch (loader.py `peek`), without advancing the epoch."""
        rows, contiguous = next(self._batches())
        hb, _ = self._pack(rows, contiguous)
        tensors, ev = self._to_device(hb)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
        return self._split(tensors)

    def host_batches(self) -> Iterator[HostBatch]:
        """Packed pinned batches without the H2D (feeds `CompiledForward` / `PipelinedForward`, which own the copy)."""
        for rows, contiguous in self._batches():
            yield self._pack(rows, contiguous)[0]


def sample_batch(dataset_or_loader, batch_size: Optional[int] = None, shuffle: Optional[bool] = False,
                 include_targets: Optional[bool] = True, prepare_features: Optional[bool] = True, **loader_kwargs):
    """merlin/models/tf/loader.py:367-420: one batch of input tensors (and targets).  `prepare_features` is
    accepted for parity: the blocks here consume the loader's convention directly (core.get_feature)."""
    if isinstance(dataset_or_loader, Loader):
        loader = dataset_or_loader
    else:
        if not batch_size:
            raise ValueError("Either use 'Loader' or specify 'batch_size'")
        loader = Loader(dataset_or_loader, batch_size=batch_size, shuffle=bool(shuffle), **loader_kwargs)
    inputs, targets = loader.peek()
    return (inputs, targets) if include_targets else inputs
