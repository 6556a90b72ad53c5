"""Pretrained embeddings: a vector per id from outside the model (text or image embeddings of an item, a vector from another
model), fed through the input block's concat.

Reference: `merlin.dataloader.ops.embeddings.EmbeddingOperator` (a Loader transform that adds the looked-up vectors to each
batch), `mm.PretrainedEmbeddings` (merlin/models/tf/inputs/embedding.py:717-800: one branch per column, an optional
Dense(new_dim) projection and L2Norm) and `mm.TensorInitializer`.

Execution differs by design.  The operator copies its matrix to the device once and batches keep the lookup ids: no (B, Dp)
block is packed on the host or copied host-to-device.  The input block finds the operator by the column name it was given
(`embedding_name`) and gathers the rows straight into their slot of x0, or projects them in the same pass
(include/mm_b200.h K24).  A batch that carries the (B, Dp) vectors itself under that name is read row by row instead.
"""
from __future__ import annotations

import weakref
from typing import Dict, List, Optional, Union

import numpy as np
import torch

from . import ops
from .blocks import _Dense
from .core import Block, TabularData, default_device
from .schema import ColumnSchema, Schema, Tags

# embedding_name -> the live EmbeddingOperator that serves it (the last one constructed under that name).  Weak: the
# loader that owns an operator, and every block that has read from it, keep it alive; the registry alone does not.
_OPERATORS: "weakref.WeakValueDictionary[str, EmbeddingOperator]" = weakref.WeakValueDictionary()


def registered_operator(name: str) -> Optional["EmbeddingOperator"]:
    return _OPERATORS.get(name)


class EmbeddingOperator:
    """`EmbeddingOperator(embeddings, lookup_key="id", embedding_name="embeddings")`: a `Loader(transforms=[...])` transform
    whose output schema gains the fp32 column `embedding_name`, tagged EMBEDDING, of shape (B, Dp).  `embeddings` (N, Dp)
    (array or tensor) is copied to the device once as fp32; the vectors are looked up on the device by the batch's
    `lookup_key` ids when the model reads them."""

    def __init__(self, embeddings, lookup_key: str = "id", embedding_name: str = "embeddings", device=None):
        if isinstance(embeddings, torch.Tensor):
            emb = embeddings.detach().to(torch.float32)
        else:
            if hasattr(embeddings, "to_numpy"):
                embeddings = embeddings.to_numpy()
            emb = torch.from_numpy(np.array(embeddings, dtype=np.float32))
        if emb.dim() != 2 or emb.shape[0] < 1 or emb.shape[1] < 1:
            raise ValueError(f"embeddings must be a non-empty (N, Dp) matrix, got shape {tuple(emb.shape)}")
        self.lookup_key = str(lookup_key)
        self.embedding_name = str(embedding_name)
        self.device = torch.device(device) if device is not None else default_device()
        self.embeddings = emb.to(self.device).contiguous()
        _OPERATORS[self.embedding_name] = self

    @property
    def dim(self) -> int:
        return int(self.embeddings.shape[1])

    def column_schema(self) -> ColumnSchema:
        return ColumnSchema(self.embedding_name, tags=(Tags.EMBEDDING,), dtype="float32", is_list=True,
                            properties={"value_count": {"min": self.dim, "max": self.dim}, "lookup_key": self.lookup_key})

    def compute_output_schema(self, input_schema: Optional[Schema]) -> Schema:
        cols = list(input_schema) if input_schema is not None else []
        return Schema([c for c in cols if c.name != self.embedding_name] + [self.column_schema()])


def TensorInitializer(weights):
    """`mm.TensorInitializer(weights)`: an `embeddings_initializer` that loads the (rows, dim) array into the table."""
    if isinstance(weights, torch.Tensor):
        return weights.detach().cpu().numpy().astype(np.float32)
    if hasattr(weights, "to_numpy"):
        weights = weights.to_numpy()
    return np.array(weights, dtype=np.float32)


class PretrainedBranch:
    """One pretrained column: its width Dp, the lookup key, the optional Dense(new_dim) projection and L2Norm."""

    def __init__(self, name: str, dim: int, lookup_key: Optional[str], projection: Optional[_Dense], l2: bool):
        self.name, self.dim, self.lookup_key, self.projection, self.l2 = name, int(dim), lookup_key, projection, bool(l2)

    @property
    def width(self) -> int:
        """Columns of the concat this branch fills."""
        return self.projection.units if self.projection is not None else self.dim


class PretrainedEmbeddingsBlock(Block):
    """Result of `PretrainedEmbeddings(schema, ...)`: a branch per column, keyed by column name."""

    def __init__(self, branches: Dict[str, PretrainedBranch], name: str = "pretrained_embeddings"):
        super().__init__(name)
        self.branches = branches
        # column -> the operator this block first read it from: kept for the block's life, so a later operator under the
        # same name does not change what it reads, and a captured graph's pointer to the matrix stays valid.  Not saved:
        # a loaded model binds again to the live operator of that name.
        self._bound: Dict[str, EmbeddingOperator] = {}

    _TRANSIENT = {"_bound": {}}

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.__dict__.setdefault("_bound", {})

    def build(self, device=None):
        for br in self.branches.values():
            if br.projection is not None:
                br.projection.build(br.dim, device or default_device())
        self.built = True
        return self

    def output_dims(self) -> Dict[str, int]:
        return {n: br.width for n, br in self.branches.items()}

    def weights(self):
        out = {}
        for n, br in self.branches.items():
            if br.projection is not None:
                out.update({f"{n}/{br.projection.name}/{k}": v for k, v in br.projection.weights().items()})
        return out

    def source(self, inputs: TabularData, name: str):
        """(P, ids) of column `name` in this batch: the batch's own (B, Dp) vectors with ids None, or the registered
        operator's matrix and the batch's lookup ids."""
        br = self.branches[name]
        if name in inputs:
            v = inputs[name]
            if v.dim() != 2 or v.shape[1] != br.dim:
                raise ValueError(f"pretrained feature {name!r}: expected (B, {br.dim}) vectors, got {tuple(v.shape)}")
            if v.dtype != torch.float32:
                raise TypeError(f"pretrained feature {name!r} must be float32, got {v.dtype}")
            return v, None
        op = self._bound.get(name) or registered_operator(name)
        if op is None:
            raise ValueError(f"pretrained feature {name!r}: the batch carries no vectors under that name and no "
                             "EmbeddingOperator serves it")
        if op.dim != br.dim:
            raise ValueError(f"pretrained feature {name!r}: the EmbeddingOperator's vectors are {op.dim} wide, the block "
                             f"was built for {br.dim}")
        key = br.lookup_key or op.lookup_key
        if key not in inputs:
            raise ValueError(f"pretrained feature {name!r}: the batch has no lookup key column {key!r}")
        self._bound[name] = op
        return op.embeddings, ops.as_index(inputs[key]).reshape(-1).contiguous()

    def write_into(self, inputs: TabularData, out: torch.Tensor, cols: Dict[str, int], oob: Optional[torch.Tensor]) -> None:
        """Every branch into out[:, cols[name] : + width] (inference: the l2-norm is applied in place)."""
        self.build(out.device)
        for n, br in self.branches.items():
            P, ids = self.source(inputs, n)
            slot = out[:, cols[n]: cols[n] + br.width]
            if br.projection is None:
                ops.pretrained_gather(P, ids, slot, oob)
            else:
                ops.pretrained_project(P, ids, br.projection.kernel, br.projection.bias, slot, oob)
            if br.l2:
                ops.l2_normalize(slot, out=slot)

    def call(self, inputs: TabularData, **kwargs) -> TabularData:
        from .core import batch_size_of

        B = batch_size_of(inputs)
        dims = self.output_dims()
        dev = next(iter(inputs.values())).device
        cols, c = {}, 0
        for n, w in dims.items():
            cols[n] = c
            c += w
        buf = torch.empty((B, c), dtype=torch.float32, device=dev)
        self.write_into(inputs, buf, cols, None)
        return {n: buf[:, cols[n]: cols[n] + dims[n]] for n in dims}


def _pretrained_dim(col: ColumnSchema) -> int:
    vc = col.value_count
    if vc is not None and vc.max is not None and vc.min == vc.max:
        return int(vc.max)
    op = registered_operator(col.name)
    if op is not None:
        return op.dim
    raise ValueError(f"pretrained column {col.name!r}: its width is unknown (no fixed value_count in the schema and no "
                     "EmbeddingOperator by that name)")


def PretrainedEmbeddings(schema: Schema, output_dims: Optional[Union[Dict[str, int], int]] = None,
                         sequence_combiner: Optional[str] = "mean", normalizer: Optional[str] = None, pre=None, post=None,
                         aggregation=None, block_name: str = "pretrained_embeddings", **kwargs) -> PretrainedEmbeddingsBlock:
    """inputs/embedding.py:717-800: a branch per column of `schema` (typically `schema.select_by_tag(Tags.EMBEDDING)`),
    each an optional `MLPBlock([new_dim], activation=None)` projection (`output_dims`: an int for every column or a dict by
    column) followed by the normalizer ("l2-norm").  `sequence_combiner` only acts on 3-D (sequence) inputs."""
    for what, v in (("pre", pre), ("post", post), ("aggregation", aggregation)):
        if v is not None:
            raise NotImplementedError(f"PretrainedEmbeddings: `{what}` is not implemented")
    if kwargs.get("id_lookup_table") is not None:
        raise NotImplementedError("PretrainedEmbeddings: `id_lookup_table` is not implemented")
    if normalizer is not None and normalizer != "l2-norm":
        raise NotImplementedError(f"PretrainedEmbeddings: normalizer {normalizer!r} is not implemented (only 'l2-norm')")
    from ._cabi import PRETRAINED_MAX_DIM, PRETRAINED_MAX_OUT

    branches: Dict[str, PretrainedBranch] = {}
    for col in schema:
        if col.is_ragged or (col.value_count is not None and col.value_count.min != col.value_count.max) \
                or col.properties.get("is_sequence"):
            raise NotImplementedError(f"pretrained column {col.name!r}: 3-D (sequence) pretrained inputs are not implemented")
        dim = _pretrained_dim(col)
        if not 1 <= dim <= PRETRAINED_MAX_DIM:
            raise NotImplementedError(f"pretrained column {col.name!r}: width {dim} outside the kernels' 1..{PRETRAINED_MAX_DIM}")
        new_dim = output_dims.get(col.name) if isinstance(output_dims, dict) else output_dims
        proj = None
        if new_dim:
            if not 1 <= int(new_dim) <= PRETRAINED_MAX_OUT:
                raise NotImplementedError(f"pretrained column {col.name!r}: output_dims {new_dim} outside the kernels' "
                                          f"1..{PRETRAINED_MAX_OUT}")
            proj = _Dense(int(new_dim), activation=None)
        branches[col.name] = PretrainedBranch(col.name, dim, col.properties.get("lookup_key"), proj, normalizer == "l2-norm")
    return PretrainedEmbeddingsBlock(branches, name=block_name)
