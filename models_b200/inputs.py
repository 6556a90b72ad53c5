"""Input blocks: EmbeddingTable / Embeddings / ContinuousFeatures / InputBlock(V2).

Mirrors the constructor surface of merlin/models/tf/inputs/embedding.py:65-714,
inputs/continuous.py:73-204 and inputs/base.py:40-341 for the one-hot / multi-hot / dense
sequence lookups on the hot path.  Execution differs by design: ALL one-hot features of a block
are gathered by ONE fused kernel (ops.gather_multi) straight into the layout the consumer wants —
(B, sum D) for concat, (B, F, D) for stack — instead of one gather per table plus tf.concat/stack.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import ops
from .core import (Block, InitializerType, TabularData, batch_size_of, create_variable, default_device,
                   get_feature, has_feature, unique_name)
from .schema import ColumnSchema, Schema, Tags


def infer_embedding_dim(col_schema: ColumnSchema, multiplier: float = 2.0, ensure_multiple_of_8: bool = True) -> int:
    """merlin/models/utils/schema_utils.py:169-207."""
    cardinality = col_schema.int_domain.max + 1
    size = int(math.ceil(math.pow(cardinality, 0.25) * multiplier))
    if ensure_multiple_of_8:
        size = int(math.ceil(size / 8) * 8)
    return size


@dataclass
class EmbeddingOptions:
    """inputs/embedding.py:931-942."""

    embedding_dims: Optional[Dict[str, int]] = None
    embedding_dim_default: Optional[int] = 64
    infer_embedding_sizes: bool = False
    infer_embedding_sizes_multiplier: float = 2.0
    infer_embeddings_ensure_dim_multiple_of_8: bool = False
    embeddings_initializers: Optional[Union[Dict[str, InitializerType], InitializerType]] = None
    embeddings_l2_reg: float = 0.0
    combiner: Optional[str] = "mean"


class EmbeddingTable(Block):
    """One embedding matrix shared by one or more features (inputs/embedding.py:153-582).

    input_dim = int_domain.max + 1 (:92-93); table name = int_domain.name or column name (:96-97).
    """

    def __init__(self, dim: int, *col_schemas: ColumnSchema, embeddings_initializer: InitializerType = "uniform",
                 sequence_combiner: Optional[str] = None, trainable: bool = True, name: Optional[str] = None,
                 table_name: Optional[str] = None, **kwargs):
        if not col_schemas:
            raise ValueError("At least one col_schema must be provided to the embedding table.")
        first = col_schemas[0]
        if first.int_domain is None or first.int_domain.max is None:
            raise ValueError(f"`col_schema` {first.name!r} needs to have an int-domain")
        self.dim = int(dim)
        self.col_schema = first
        self.features: Dict[str, ColumnSchema] = {}
        self.input_dim = int(first.int_domain.max) + 1
        self.table_name = table_name or first.int_domain.name or first.name
        super().__init__(name or self.table_name)
        for c in col_schemas:
            self.add_feature(c)
        if sequence_combiner is not None and sequence_combiner not in ("mean", "sum", "sqrtn", "max"):
            raise ValueError(f"Unsupported sequence_combiner {sequence_combiner!r}")
        self.sequence_combiner = sequence_combiner
        self.embeddings_initializer = embeddings_initializer
        self.trainable = trainable
        self.table: Optional[torch.Tensor] = None
        self._mirror: Optional[torch.Tensor] = None
        self._mirror_src = None

    _TRANSIENT = {"_mirror": None, "_mirror_src": None}

    def operand_mirror(self) -> torch.Tensor:
        """The table as bf16 split rows (rows, 2*dim) = [hi | lo] (ops.split_rows; dim a multiple of 64): a second,
        same-size copy in HBM that removes the per-sample bf16 split from the fused lookup + interaction kernel.  Built on
        first use; rebuilt when the table tensor was replaced; call `_weights_changed()` after modifying the table in place."""
        t = self.embeddings
        key = (t.data_ptr(), tuple(t.shape))
        if self._mirror is None or self._mirror_src != key:
            reuse = self._mirror is not None and self._mirror.shape[0] == t.shape[0]
            self._mirror = ops.split_rows(t.contiguous(), out=self._mirror if reuse else None)
            self._mirror_src = key
        return self._mirror

    def _weights_changed(self) -> None:
        from .core import bump_weights_version

        if self._mirror is not None and self.table is not None and self._mirror.shape[0] == self.table.shape[0]:
            ops.split_rows(self.table.contiguous(), out=self._mirror)  # refresh in place: captured graphs keep valid pointers
        else:
            self._mirror = None
        bump_weights_version()

    def add_feature(self, col_schema: ColumnSchema) -> None:
        """inputs/embedding.py:99-130: all features of a table must share the domain."""
        if not col_schema.int_domain:
            raise ValueError("`col_schema` needs to have an int-domain")
        dom, mine = col_schema.int_domain, self.col_schema.int_domain
        if (dom.name or col_schema.name) != (mine.name or self.col_schema.name) and col_schema is not self.col_schema:
            raise ValueError(
                f"`col_schema` int-domain name {dom.name!r} does not match table domain {mine.name!r}")
        if dom.max != mine.max:
            raise ValueError("`col_schema.int_domain.max` does not match other column schemas of this table")
        self.features[col_schema.name] = col_schema

    @classmethod
    def from_pretrained(cls, data, col_schema: Optional[ColumnSchema] = None, trainable: bool = True,
                        name: Optional[str] = None, **kwargs) -> "EmbeddingTable":
        """inputs/embedding.py:283-345 (array form): rows x dim matrix as the table."""
        import numpy as np

        if hasattr(data, "to_numpy") and not isinstance(data, torch.Tensor):  # pandas / cudf DataFrame (df_to_tensor)
            data = data.to_numpy()
        arr = data.detach().cpu().numpy() if isinstance(data, torch.Tensor) else np.asarray(data, dtype=np.float32)
        rows, dim = arr.shape
        if col_schema is None:
            if not name:
                raise ValueError("`name` is required when not using a ColumnSchema")
            col_schema = ColumnSchema(name, tags=(Tags.CATEGORICAL,), dtype="int64",
                                      properties={"domain": {"min": 0, "max": rows - 1, "name": name}})
        return cls(dim, col_schema, embeddings_initializer=arr, trainable=trainable, name=name, **kwargs)

    def build(self, device=None) -> "EmbeddingTable":
        if self.table is None:
            device = device or default_device()
            self.table = create_variable((self.input_dim, self.dim), self.embeddings_initializer, device,
                                         f"{self.table_name}/embeddings")
        self.built = True
        return self

    @property
    def embeddings(self) -> torch.Tensor:
        return self.build().table

    def weights(self):
        return {"embeddings": self.embeddings}

    def to_df(self, gpu=None):
        """inputs/embedding.py:363-379: the table as a DataFrame with one column per embedding dimension
        (pandas; `gpu` is accepted for signature parity — cudf is not a dependency here)."""
        import pandas as pd

        return pd.DataFrame(self.embeddings.detach().cpu().numpy())

    @classmethod
    def from_dataset(cls, data, trainable=True, name=None, col_schema=None, **kwargs) -> "EmbeddingTable":
        """inputs/embedding.py:327-349."""
        return cls.from_pretrained(data, col_schema=col_schema, trainable=trainable, name=name, **kwargs)

    # -- execution --------------------------------------------------------------------------------
    def lookup_kind(self, feat) -> str:
        if isinstance(feat, tuple):
            return "bag"
        if feat.dtype == torch.uint8 and feat.dim() == 2 and feat.shape[1] == 3:
            return "onehot"  # packed 24-bit ids (graph.HostBatch id_bytes)
        if feat.dim() == 1 or (feat.dim() == 2 and feat.shape[1] == 1):
            return "onehot"
        if feat.dim() == 2 or (feat.dim() == 3 and feat.shape[2] == 1):
            return "seq"
        raise ValueError(f"unsupported categorical input shape {tuple(feat.shape)}")

    def lookup_into(self, feat, out: torch.Tensor, out_col: int, oob=None) -> None:
        """_call_table (inputs/embedding.py:424-471) writing into out[:, out_col:out_col+dim]."""
        self.build(out.device)
        kind = self.lookup_kind(feat)
        if kind == "bag":  # ragged + combiner -> safe_embedding_lookup_sparse (:432-441)
            values, offsets = feat
            ops.gather_bag(self.table, ops.as_index(values).reshape(-1), ops.as_index(offsets), self.sequence_combiner or "mean",
                           out, out_col, oob)
        elif kind == "onehot":
            ops.gather_multi([self.table], [ops.as_index(feat).reshape(-1)], [out_col], out, oob)
        else:  # dense (B, L): gather then combiner over axis 1, padding not masked (:457-461)
            ids = ops.as_index(feat).reshape(feat.shape[0], -1).contiguous()
            comb = self.sequence_combiner or "mean"
            if comb == "sqrtn":
                raise ValueError("sequence_combiner 'sqrtn' is only defined for ragged inputs")
            ops.gather_seq(self.table, ids, comb, out, out_col, oob)

    def call(self, inputs, **kwargs):
        """inputs/embedding.py:401-422: dict -> dict over this table's features; tensor -> tensor."""
        if isinstance(inputs, dict):
            out = {}
            for fname in self.features:
                if has_feature(inputs, fname):
                    out[fname] = self._call_one(get_feature(inputs, fname))
            return out
        return self._call_one(inputs)

    def _call_one(self, feat) -> torch.Tensor:
        B = (feat[1].numel() - 1) if isinstance(feat, tuple) else feat.shape[0]
        dev = feat[0].device if isinstance(feat, tuple) else feat.device
        out = torch.empty((B, self.dim), dtype=torch.float32, device=dev)
        oob = torch.zeros(1, dtype=torch.int32, device=dev)
        self.lookup_into(feat, out, 0, oob)
        _raise_on_oob(oob, self.table_name)
        return out


def _raise_on_oob(oob: torch.Tensor, what: str) -> None:
    n = int(oob.item())
    if n:
        oob.zero_()
        raise IndexError(f"{n} indices out of range for embedding table(s) {what} "
                         "(TF raises InvalidArgumentError: indices[...] is not in [0, rows))")


class EmbeddingsBlock(Block):
    """Result of `Embeddings(schema, ...)`: a ParallelBlock of EmbeddingTables keyed by table name
    (inputs/embedding.py:681-683), executed as ONE fused gather."""

    def __init__(self, tables: Dict[str, EmbeddingTable], schema: Schema, name: str = "embeddings",
                 check_indices: bool = True):
        super().__init__(name)
        self.tables = tables
        self.schema = schema
        self.feature_to_table: Dict[str, EmbeddingTable] = {}
        for t in tables.values():
            for f in t.features:
                self.feature_to_table[f] = t
        self.check_indices = check_indices
        self.oob_counter: Optional[torch.Tensor] = None  # persistent device int32[1]
        self.defer_check = False  # CUDA-graph capture: the owner checks the counter after replay

    _TRANSIENT = {"oob_counter": None, "defer_check": False}

    def counter(self, device) -> Optional[torch.Tensor]:
        if not self.check_indices:
            return None
        if self.oob_counter is None or self.oob_counter.device != device:
            self.oob_counter = torch.zeros(1, dtype=torch.int32, device=device)
        return self.oob_counter

    def finish_check(self, oob: Optional[torch.Tensor]) -> None:
        if oob is not None and not self.defer_check:
            _raise_on_oob(oob, ",".join(self.tables) or self.name)

    @property
    def feature_names(self) -> List[str]:
        return list(self.feature_to_table.keys())

    def select_by_names(self, names) -> List[EmbeddingTable]:
        return [self.feature_to_table[n] for n in names]

    def build(self, device=None):
        for t in self.tables.values():
            t.build(device)
        self.built = True
        return self

    def weights(self):
        return {f"{n}/embeddings": t.embeddings for n, t in self.tables.items()}

    def output_dims(self) -> Dict[str, int]:
        return {f: t.dim for f, t in self.feature_to_table.items()}

    def lookup_all_into(self, inputs: TabularData, out: torch.Tensor, out_cols: Dict[str, int]) -> None:
        """Every feature of this block into out[:, out_cols[f] : +dim_f]; one-hot features share one
        launch (chunks of 64 tables), bag / sequence features one launch each."""
        self.build(out.device)
        oob = self.counter(out.device)
        one_w, one_i, one_c = [], [], []
        for fname, table in self.feature_to_table.items():
            if not has_feature(inputs, fname):
                raise ValueError(f"missing input feature {fname!r}")
            feat = get_feature(inputs, fname)
            if table.lookup_kind(feat) == "onehot":
                one_w.append(table.table)
                one_i.append(ops.as_index(feat).reshape(-1))
                one_c.append(out_cols[fname])
            else:
                table.lookup_into(feat, out, out_cols[fname], oob)
        if one_w:
            if len({i.dtype for i in one_i}) > 1:
                one_i = [i.to(torch.int64) for i in one_i]
            ops.gather_multi(one_w, one_i, one_c, out, oob)
        self.finish_check(oob)

    def call(self, inputs: TabularData, **kwargs) -> TabularData:
        """dict feature -> (B, dim_f) views of one (B, sum dim) buffer (iteration order = schema order)."""
        dims = self.output_dims()
        cols, c = {}, 0
        for f in self.feature_to_table:
            cols[f] = c
            c += dims[f]
        B = batch_size_of({k: v for k, v in inputs.items() if any(k == f or k.startswith(f + "__") for f in dims)})
        dev = next(iter(inputs.values())).device
        buf = torch.empty((B, c), dtype=torch.float32, device=dev)
        self.lookup_all_into(inputs, buf, cols)
        return {f: buf[:, cols[f]: cols[f] + dims[f]] for f in dims}


def _get_dim(col: ColumnSchema, dim, infer_dim_fn) -> int:
    """inputs/embedding.py:704-714."""
    if isinstance(dim, dict):
        d = dim.get(col.name)
        return int(d) if d else int(infer_dim_fn(col))
    if dim:
        return int(dim)
    return int(infer_dim_fn(col))


def Embeddings(schema: Schema, dim: Optional[Union[Dict[str, int], int]] = None,
               infer_dim_fn: Callable[[ColumnSchema], int] = infer_embedding_dim,
               sequence_combiner: Optional[Union[str, Dict[str, str]]] = "mean",
               embeddings_initializer: Optional[Union[InitializerType, Dict[str, InitializerType]]] = None,
               trainable: Optional[Dict[str, bool]] = None, name: str = "embeddings", **kwargs) -> EmbeddingsBlock:
    """inputs/embedding.py:585-683: one table per `int_domain.name or col.name`; columns sharing a
    domain share the table (:668-679)."""
    if trainable:
        kwargs["trainable"] = trainable
    tables: Dict[str, EmbeddingTable] = {}
    for col in schema:
        if col.int_domain is None or col.int_domain.max is None:
            continue
        table_name = col.int_domain.name or col.name
        if table_name in tables:
            tables[table_name].add_feature(col)
            continue
        tkw = {}
        for k, v in dict(sequence_combiner=sequence_combiner, embeddings_initializer=embeddings_initializer,
                         **kwargs).items():
            if isinstance(v, dict) and not ("hash_seed" in v):
                v = v.get(table_name, v.get(col.name))
            if v is not None:
                tkw[k] = v
        if isinstance(tkw.get("embeddings_initializer"), dict) and "hash_seed" in tkw["embeddings_initializer"]:
            # derive an independent stream per table from the shared seed
            spec = dict(tkw["embeddings_initializer"])
            spec["hash_seed"] = (spec["hash_seed"] * 1000003 + _stable_hash(table_name)) & (2**63 - 1)
            tkw["embeddings_initializer"] = spec
        tkw.setdefault("embeddings_initializer", "uniform")
        tables[table_name] = EmbeddingTable(_get_dim(col, dim, infer_dim_fn), col, name=table_name, **tkw)
    return EmbeddingsBlock(tables, schema, name=name)


def _stable_hash(s: str) -> int:
    h = 1469598103934665603
    for ch in s.encode():
        h = ((h ^ ch) * 1099511628211) & (2**63 - 1)
    return h


class ContinuousFeatures(Block):
    """inputs/continuous.py:73-204: select continuous columns; (B,) -> (B,1).  The fp32 cast and
    the concat happen in the consumer's concat kernel."""

    def __init__(self, features: Sequence[str], name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("continuous_features"))
        self.features = list(features)

    @classmethod
    def from_schema(cls, schema: Schema, tags=None, **kwargs) -> "ContinuousFeatures":
        if tags is not None:
            schema = schema.select_by_tag(tags)
        return cls(schema.column_names, **kwargs)

    def call(self, inputs: TabularData, **kwargs) -> TabularData:
        out = {}
        for n in self.features:
            if n not in inputs:
                raise ValueError(f"missing continuous feature {n!r}")
            v = inputs[n]
            out[n] = v.view(-1, 1) if v.dim() == 1 else v
        return out


class InputBlockV2(Block):
    """inputs/base.py:216-341 with the default aggregation="concat": embeddings (inferred dims
    unless `categorical`/`dim` given) + continuous features, concatenated in sorted(name) order.
    The embeddings are gathered directly at their concat offsets (no intermediate tensors)."""

    def __init__(self, schema: Schema, categorical: Union[Tags, EmbeddingsBlock] = Tags.CATEGORICAL,
                 continuous: Union[Tags, ContinuousFeatures] = Tags.CONTINUOUS, pretrained_embeddings=Tags.EMBEDDING,
                 aggregation: Optional[str] = "concat", name: Optional[str] = None, **embedding_kwargs):
        super().__init__(name or unique_name("input_block"))
        if aggregation not in ("concat", None):
            raise ValueError(f"InputBlockV2: unsupported aggregation {aggregation!r} (concat or None)")
        self.schema = schema
        self.aggregation = aggregation
        if isinstance(categorical, EmbeddingsBlock):
            self.embeddings: Optional[EmbeddingsBlock] = categorical
        else:
            cat = schema.select_by_tag(categorical).excluding_by_tag(Tags.TARGET)
            self.embeddings = Embeddings(cat, **embedding_kwargs) if len(cat) else None
        if isinstance(continuous, ContinuousFeatures):
            self.continuous: Optional[ContinuousFeatures] = continuous
        else:
            con = schema.select_by_tag(continuous).excluding_by_tag(Tags.TARGET)
            self.continuous = ContinuousFeatures.from_schema(con) if len(con) else None
        from .pretrained import PretrainedEmbeddings, PretrainedEmbeddingsBlock

        if isinstance(pretrained_embeddings, PretrainedEmbeddingsBlock):
            self.pretrained: Optional[PretrainedEmbeddingsBlock] = pretrained_embeddings
        else:
            pre = schema.select_by_tag(pretrained_embeddings).excluding_by_tag(Tags.TARGET)
            self.pretrained = PretrainedEmbeddings(pre) if len(pre) else None
        if self.embeddings is None and self.continuous is None and self.pretrained is None:
            raise ValueError("InputBlockV2: the schema has neither categorical, continuous nor pretrained features")
        # the pretrained lookups count out-of-range ids in the tables' counter; without tables an EmbeddingsBlock without
        # tables owns it, so the model's checks (fit, CompiledForward) find it as they find the tables'
        self.pretrained_ids: Optional[EmbeddingsBlock] = (
            EmbeddingsBlock({}, Schema([]), name="pretrained_ids") if self.pretrained is not None and self.embeddings is None
            else None)

    def __setstate__(self, state):
        self.__dict__.update(state)
        for k in ("pretrained", "pretrained_ids"):  # a model saved before input blocks had pretrained features
            self.__dict__.setdefault(k, None)

    def build(self, device=None):
        if self.embeddings is not None:
            self.embeddings.build(device)
        if self.pretrained is not None:
            self.pretrained.build(device)
        self.built = True
        return self

    def weights(self):
        out = {} if self.embeddings is None else {f"embeddings/{k}": v for k, v in self.embeddings.weights().items()}
        if self.pretrained is not None:
            out.update({f"{self.pretrained.name}/{k}": v for k, v in self.pretrained.weights().items()})
        return out

    def layout(self) -> Tuple[Dict[str, int], Dict[str, int], int]:
        """(column offset, width) of every feature in the sorted-name concat, and the total width."""
        widths: Dict[str, int] = {}
        if self.embeddings is not None:
            widths.update(self.embeddings.output_dims())
        if self.pretrained is not None:
            widths.update(self.pretrained.output_dims())
        if self.continuous is not None:
            widths.update({n: 1 for n in self.continuous.features})
        cols, c = {}, 0
        for n in sorted(widths):
            cols[n] = c
            c += widths[n]
        return cols, widths, c

    def call(self, inputs: TabularData, **kwargs):
        cols, widths, total = self.layout()
        if self.aggregation is None:
            out = {}
            if self.embeddings is not None:
                out.update(self.embeddings(inputs))
            if self.continuous is not None:
                out.update(self.continuous(inputs))
            if self.pretrained is not None:
                out.update(self.pretrained(inputs))
            return out
        B = batch_size_of(inputs)
        dev = next(iter(inputs.values())).device
        buf = torch.empty((B, total), dtype=torch.float32, device=dev)
        if self.pretrained is not None:
            # the tables' counter, checked after their own gathers below; without tables pretrained_ids', checked here
            owner = self.embeddings if self.embeddings is not None else self.pretrained_ids
            oob = owner.counter(dev)
            self.pretrained.write_into(inputs, buf, cols, oob)
            if owner is self.pretrained_ids:
                owner.finish_check(oob)
        if self.embeddings is not None:
            self.embeddings.lookup_all_into(inputs, buf, cols)
        if self.continuous is not None:
            con = self.continuous(inputs)
            names = sorted(con)
            ops.concat_columns([con[n] for n in names], buf, [cols[n] for n in names])
        return buf


class InputBlock(Block):
    """Legacy InputBlock (inputs/base.py:40-206) as TwoTowerBlock uses it: aggregation=None, output
    = dict {continuous features..., categorical features...}; embeddings via EmbeddingOptions
    (EmbeddingFeatures.from_schema, inputs/embedding.py:1005-1094: default initialiser
    TruncatedNormal(0, 0.05), default dim 64, combiner "mean")."""

    def __init__(self, schema: Schema, embedding_options: EmbeddingOptions = EmbeddingOptions(),
                 aggregation: Optional[str] = None, name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("input_block"))
        self.schema = schema
        opts = self.embedding_options = embedding_options  # the training step reads embeddings_l2_reg from it
        cat = schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)
        con = schema.select_by_tag(Tags.CONTINUOUS).excluding_by_tag(Tags.TARGET)
        dims = dict(opts.embedding_dims or {})
        if opts.infer_embedding_sizes:
            for c in cat:
                dims.setdefault(c.name, infer_embedding_dim(c, opts.infer_embedding_sizes_multiplier,
                                                            opts.infer_embeddings_ensure_dim_multiple_of_8))
        for c in cat:
            dims.setdefault(c.name, opts.embedding_dim_default)
        init = opts.embeddings_initializers or "truncated_normal"
        self.embeddings = (Embeddings(cat, dim=dims, sequence_combiner=opts.combiner, embeddings_initializer=init)
                           if len(cat) else None)
        self.continuous = ContinuousFeatures.from_schema(con) if len(con) else None
        self._v2 = InputBlockV2(schema, categorical=self.embeddings if self.embeddings is not None else Tags.CATEGORICAL,
                                continuous=self.continuous if self.continuous is not None else Tags.CONTINUOUS,
                                aggregation=aggregation) if (self.embeddings or self.continuous) else None
        self.aggregation = aggregation

    def build(self, device=None):
        if self.embeddings is not None:
            self.embeddings.build(device)
        self.built = True
        return self

    def weights(self):
        return {} if self.embeddings is None else self.embeddings.weights()

    def layout(self):
        return self._v2.layout()

    def call(self, inputs: TabularData, **kwargs):
        return self._v2(inputs)

    def concat(self, inputs: TabularData) -> torch.Tensor:
        """The sorted-name concat the first _Dense of a tower applies to this block's dict output
        (blocks/mlp.py:275-277) — produced directly, without materialising the dict."""
        agg = self._v2.aggregation
        self._v2.aggregation = "concat"
        try:
            return self._v2(inputs)
        finally:
            self._v2.aggregation = agg
