"""Top-k retrieval and the evaluation step (SURVEY §8f-2), forward only.

Reference: `TopKIndexBlock` (merlin/models/tf/core/index.py:170-284), `BruteForce` / `TopKLayer`
(outputs/topk.py:33-243), `TopKEncoder` (core/encoder.py:427-665), `RetrievalModel.evaluate(item_corpus=...)`
(models/base.py:2266-2351) and the ranking metrics of metrics/topk.py:48-190.

The reference materialises `scores = matmul(queries, candidates^T)` (B, N) and runs `tf.math.top_k` over it;
here query x catalog scoring and the top-k selection are ONE kernel (`mm_catalog_score`, csrc/catalog_tc.cu,
k <= 32): the (B, N) matrix never exists, which is what makes a 10 M-item corpus usable.  k > 32 falls back
to the tensor-core GEMM + a sort of the materialised scores for small corpora.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, List, NamedTuple, Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from .core import Block, Prediction, TabularData, default_device, to_device, unique_name
from .schema import Tags

MIN_FLOAT = -655.04  # utils/constants.py:19 (float16-safe "minus infinity" of the reference)
_FUSED_MAX_K = 32


class TopKPrediction(NamedTuple):
    """outputs/topk.py: (scores, identifiers) of the k best candidates per query."""

    scores: torch.Tensor
    identifiers: torch.Tensor


def _as_device(x, device, dtype=None) -> torch.Tensor:
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.array(x))  # private copy (frames can be read-only)
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    return t.to(device)


def _topk_scores(queries: torch.Tensor, e_split: torch.Tensor, values: torch.Tensor, k: int):
    """(scores (B,k) descending, row indices (B,k) int64) of queries against the candidate matrix."""
    n = values.shape[0]
    if k > n:
        raise ValueError(f"k = {k} exceeds the number of candidates ({n})")
    if queries.dim() != 2 or queries.shape[1] != values.shape[1]:
        raise ValueError(
            "Query and candidates vectors must have the same embedding size "
            f"(got query dimension of {queries.shape[-1]} and candidates dimension of {values.shape[1]})")
    if k <= _FUSED_MAX_K:
        _, scores, idx = ops.catalog_score(queries.contiguous(), e_split, n, k=k, want_stats=False)
        return scores, idx
    B = queries.shape[0]
    if B * n > (1 << 28):
        raise NotImplementedError(f"top-{k} over {n} candidates: k > {_FUSED_MAX_K} needs the scores materialised "
                                  f"({B} x {n} floats); use k <= {_FUSED_MAX_K} (fused kernel) or smaller batches")
    w = ops.split_weights(values.t().contiguous())
    full = torch.empty((B, n), dtype=torch.float32, device=queries.device)
    ops.dense_tc(ops.split_rows(queries.contiguous()), queries.shape[1], w, n, None, "linear", out_f32=full)
    return torch.topk(full, k, dim=1)


class _CandidateIndex(Block):
    """Shared storage of the two index flavours: candidate embeddings (N, D) fp32 + identifiers (N,)."""

    _TRANSIENT = {"_e_split": None}

    def __init__(self, k: int, name: Optional[str] = None):
        super().__init__(name or unique_name(type(self).__name__.lower()))
        self._k = int(k)
        self.values: Optional[torch.Tensor] = None
        self.ids: Optional[torch.Tensor] = None
        self._e_split: Optional[torch.Tensor] = None

    def _set(self, values, ids, device=None) -> None:
        device = device or (values.device if isinstance(values, torch.Tensor) and values.is_cuda else default_device())
        v = _as_device(values, device, torch.float32)
        if v.dim() != 2:
            raise ValueError(f"The candidates embeddings tensor must be 2D (got {tuple(v.shape)}).")
        i = torch.arange(v.shape[0], device=device, dtype=torch.int64) if ids is None else _as_device(ids, device).reshape(-1).to(torch.int64)
        if i.shape[0] != v.shape[0]:
            raise ValueError("The candidates and identifiers tensors must have the same number of rows "
                             f"(got {v.shape[0]} candidates rows and {i.shape[0]} identifier rows).")
        self.values, self.ids, self._e_split = v.contiguous(), i, None
        self.built = True

    def _split(self) -> torch.Tensor:
        if self._e_split is None:
            self._e_split = ops.split_rows(self.values)  # (N, 2*Kp) split-bf16 catalog, once per index
        return self._e_split

    def _weights_changed(self) -> None:
        from .core import bump_weights_version

        self._e_split = None
        bump_weights_version()

    def weights(self):
        return {} if self.values is None else {"candidates": self.values}

    def _search(self, queries: torch.Tensor, k: Optional[int]):
        if self.values is None:
            raise ValueError("You should call the `index` method first to set the _candidates index.")
        k = self._k if k is None else int(k)
        scores, idx = _topk_scores(queries, self._split() if k <= _FUSED_MAX_K else None, self.values, k)
        return scores, self.ids[idx]

    @staticmethod
    def extract_ids_embeddings(data, check_unique_ids: bool = True):
        """A DataFrame of embeddings indexed by candidate id (outputs/topk.py:88-107, core/index.py:84-100),
        or an (ids, embeddings) pair."""
        if isinstance(data, (tuple, list)) and len(data) == 2:
            ids, values = data
        elif hasattr(data, "index") and hasattr(data, "to_numpy"):
            if check_unique_ids and data.index.to_series().nunique() != data.shape[0]:
                raise ValueError("Please make sure that `data` contains unique indices")
            ids, values = data.index.to_numpy(), data.to_numpy(dtype=np.float32)
        else:
            ids, values = None, data
        return ids, values


class TopKIndexBlock(_CandidateIndex):
    """core/index.py:170-284: `index(queries, k=None) -> (top_scores, top_ids)`."""

    def __init__(self, k, values, ids=None, **kwargs):
        super().__init__(k, kwargs.get("name"))
        self._set(values, ids)
        self.false_negatives_score = MIN_FLOAT

    @classmethod
    def from_block(cls, block: Block, data: Dict[str, np.ndarray], k: int = 20, id_column: Optional[str] = None,
                   batch_size: int = 65536, **kwargs) -> "TopKIndexBlock":
        """Candidate embeddings = `block` (the item tower) applied to the unique item rows `data`
        (core/index.py:59-82, :200-230)."""
        ids, values = encode_candidates(block, data, id_column, batch_size)
        return cls(k, values, ids, **kwargs)

    def update(self, values, ids=None) -> "TopKIndexBlock":
        self._set(values, ids)
        return self

    def update_from_block(self, block: Block, data, id_column: Optional[str] = None, check_unique_ids: bool = True,
                          batch_size: int = 65536):
        ids, values = encode_candidates(block, data, id_column, batch_size, check_unique_ids)
        return self.update(values, ids)

    def call(self, inputs: torch.Tensor, k=None, **kwargs):
        return self._search(inputs, k)

    def call_outputs(self, positive_item_ids: torch.Tensor, queries: torch.Tensor, **kwargs) -> Prediction:
        """core/index.py:252-284: scores of the top-k candidates per query, one-hot targets marking where the
        positive item sits among them, label_relevant_counts = 1."""
        n = positive_item_ids.shape[0]
        scores, top_ids = self(queries[:n], k=self._k)
        targets = (positive_item_ids.reshape(-1, 1).to(torch.int64) == top_ids).to(torch.float32)
        return Prediction(scores, targets, label_relevant_counts=torch.ones(n, dtype=torch.float32, device=scores.device),
                          top_ids=top_ids)

    def to_df(self):
        import pandas as pd

        return pd.DataFrame(self.values.cpu().numpy(), index=self.ids.cpu().numpy())


class BruteForce(_CandidateIndex):
    """outputs/topk.py:129-243 ("brute-force-topk")."""

    def __init__(self, k: int = 10, name: Optional[str] = None, **kwargs):
        super().__init__(k, name)

    def index(self, candidates, identifiers=None) -> "BruteForce":
        c = candidates if isinstance(candidates, torch.Tensor) else torch.from_numpy(np.array(candidates))
        if c.dim() != 2:
            raise ValueError(f"candidates must be 2-D tensor (got {tuple(c.shape)})")
        self._set(c, identifiers)
        return self

    def index_from_dataset(self, data, check_unique_ids: bool = True) -> "BruteForce":
        ids, values = self.extract_ids_embeddings(data, check_unique_ids)
        return self.index(values, ids)

    def call(self, inputs: torch.Tensor, targets: Optional[torch.Tensor] = None, testing: bool = False, k: Optional[int] = None,
             **kwargs) -> Union[Prediction, TopKPrediction]:
        top_scores, top_ids = self._search(inputs, k)
        if testing:
            if targets is None:
                raise ValueError("Targets should be provided during the evaluation mode")
            t = targets.reshape(-1, 1).to(device=top_ids.device, dtype=torch.int64)
            return Prediction(top_scores, (t == top_ids).to(torch.float32))
        return TopKPrediction(top_scores, top_ids)


def _np(v) -> np.ndarray:
    return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def take_rows(data: Dict[str, np.ndarray], idx: np.ndarray) -> Dict[str, np.ndarray]:
    """Rows `idx` of a feature dict; ragged pairs (`name__values`, `name__offsets`) are re-packed."""
    out = {}
    for k, v in data.items():
        if k.endswith("__values"):
            continue
        if k.endswith("__offsets"):
            base = k[: -len("__offsets")]
            off, vals = _np(v).astype(np.int64), _np(data[base + "__values"])
            lens = off[idx + 1] - off[idx]
            new_off = np.concatenate([[0], np.cumsum(lens)])
            # position j of output row r reads vals[off[idx[r]] + j]
            src = np.repeat(off[idx] - new_off[:-1], lens) + np.arange(int(new_off[-1]))
            out[base + "__values"] = vals[src]
            out[k] = new_off.astype(_np(v).dtype)
        else:
            out[k] = _np(v)[idx]
    return out


def slice_rows(data: Dict[str, np.ndarray], start: int, stop: int) -> Dict[str, np.ndarray]:
    out = {}
    for k, v in data.items():
        if k.endswith("__values"):
            continue
        if k.endswith("__offsets"):
            base = k[: -len("__offsets")]
            off = _np(v)
            out[base + "__values"] = _np(data[base + "__values"])[int(off[start]):int(off[stop])]
            out[k] = (off[start:stop + 1] - off[start]).astype(off.dtype)
        else:
            out[k] = v[start:stop]
    return out


def _num_rows(data) -> int:
    for k, v in data.items():
        if k.endswith("__offsets"):
            return int(v.shape[0]) - 1
        if not k.endswith("__values"):
            return int(v.shape[0])
    raise ValueError("empty feature dict")


def encode_candidates(block: Block, data, id_column: Optional[str] = None, batch_size: int = 65536,
                      check_unique_ids: bool = True):
    """(ids, embeddings) of the rows of `data` (dict name -> array) through `block` in batches of
    `batch_size` — `IndexBlock.get_candidates_dataset` (core/index.py:59-82) without dask."""
    if isinstance(data, (tuple, list)) or hasattr(data, "to_numpy"):
        return _CandidateIndex.extract_ids_embeddings(data, check_unique_ids)
    if not id_column:
        schema = getattr(getattr(block, "inputs", None), "schema", None) or getattr(block, "schema", None)
        if schema is not None:
            tagged = schema.select_by_tag(Tags.ITEM_ID)
            if tagged:
                id_column = tagged.first.name
    if not id_column or id_column not in data:
        raise ValueError("`id_column` is required (the block's schema has no item-id tagged column present in `data`)")
    ids = np.asarray(data[id_column]).reshape(-1)
    if check_unique_ids and np.unique(ids).shape[0] != ids.shape[0]:
        raise ValueError("Please make sure that `data` contains unique indices")
    device = default_device()
    n = ids.shape[0]
    outs = []
    for s in range(0, n, batch_size):
        outs.append(block(to_device(slice_rows(data, s, min(n, s + batch_size)), device)))
    return ids, torch.cat(outs, dim=0) if len(outs) > 1 else outs[0]


class TowerEncoder(Block):
    """One tower of a two-tower model as an encoder: feature dict -> (B, D), with the model's `post`
    (e.g. L2Norm) applied to the single embedding (core/encoder.py `Encoder` of the V2 API)."""

    def __init__(self, tower: Block, post: Optional[Block] = None):
        super().__init__(unique_name("tower_encoder"))
        self.tower, self.post = tower, post
        self.inputs = getattr(tower, "inputs", None)

    def weights(self):
        return self.tower.weights()

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        if not self.tower.built:
            self.tower.build(next(iter(inputs.values())).device)
        x = self.tower(inputs)
        return self.post(x) if self.post is not None else x


def encode_rows(block: Block, data: Dict[str, np.ndarray], id_column: Optional[str], batch_size: int = 65536):
    """(ids or None, embeddings) of all rows of `data` through `block`, `batch_size` rows at a time."""
    dev = default_device()
    n = _num_rows(data)
    outs = []
    for s in range(0, n, batch_size):
        outs.append(block(to_device(slice_rows(data, s, min(n, s + batch_size)), dev)))
    ids = None if not id_column or id_column not in data else np.asarray(data[id_column]).reshape(-1)
    return ids, torch.cat(outs, dim=0) if len(outs) > 1 else outs[0]


def unique_rows_by_features(data: Dict[str, np.ndarray], id_column: str) -> Dict[str, np.ndarray]:
    """utils/dataset.py `unique_rows_by_features`: the first occurrence of every distinct item id
    (ragged list features are re-packed)."""
    ids = _np(data[id_column]).reshape(-1)
    _, first = np.unique(ids, return_index=True)
    first.sort()
    return take_rows(data, first)


class TopKEncoder(Block):
    """core/encoder.py:427-665: query encoder -> top-k layer over an indexed candidate set."""

    def __init__(self, query_encoder: Block, topk_layer: Union[str, BruteForce] = "brute-force-topk", candidates=None,
                 candidate_encoder: Optional[Block] = None, k: int = 10, pre: Optional[Block] = None,
                 post: Optional[Block] = None, target: Optional[str] = None, **kwargs):
        super().__init__(unique_name("top_k_encoder"))
        if isinstance(topk_layer, str):
            if topk_layer != "brute-force-topk":
                raise ValueError(f"Unknown top-k layer {topk_layer!r}; supported: ['brute-force-topk']")
            if candidates is None:
                raise ValueError("`candidates` is required when `topk_layer` is given by name")
            topk_layer = BruteForce(k=k)
        self.query_encoder, self.topk_layer, self.candidate_encoder = query_encoder, topk_layer, candidate_encoder
        self.pre, self.post, self.target, self.k = pre, post, target, int(k)
        if candidates is not None:
            ids, values = _CandidateIndex.extract_ids_embeddings(candidates)
            self.topk_layer.index(values, ids)

    @classmethod
    def from_candidate_dataset(cls, query_encoder: Block, candidate_encoder: Block, candidates: Dict[str, np.ndarray],
                               candidate_id: Optional[str] = None, k: int = 10, batch_size: int = 65536, **kwargs):
        """core/encoder.py:484-540: index = `candidate_encoder` applied to the item features."""
        ids, values = encode_candidates(candidate_encoder, candidates, candidate_id, batch_size)
        return cls(query_encoder, candidates=(ids, values), candidate_encoder=candidate_encoder, k=k, **kwargs)

    def index_candidates(self, candidates, candidate_id: Optional[str] = None, batch_size: int = 65536) -> "TopKEncoder":
        if isinstance(candidates, dict):
            if self.candidate_encoder is None:
                raise ValueError("raw item features need a `candidate_encoder`")
            candidates = encode_candidates(self.candidate_encoder, candidates, candidate_id, batch_size)
        ids, values = _CandidateIndex.extract_ids_embeddings(candidates)
        self.topk_layer.index(values, ids)
        return self

    def weights(self):
        out = {f"query_encoder/{k}": v for k, v in self.query_encoder.weights().items()}
        out.update({f"topk/{k}": v for k, v in self.topk_layer.weights().items()})
        return out

    def encode(self, inputs: TabularData) -> torch.Tensor:
        x = self.pre(inputs) if self.pre is not None else inputs
        return self.query_encoder(x)

    def call(self, inputs: TabularData, targets=None, testing: bool = False, k: Optional[int] = None, **kwargs):
        out = self.topk_layer(self.encode(inputs), targets=targets, testing=testing, k=k if k is not None else self.k)
        return self.post(out) if self.post is not None else out

    def batch_predict(self, batches: Iterable[Dict[str, np.ndarray]], k: Optional[int] = None):
        """(scores, ids) for every batch of query features (host arrays in, host arrays out)."""
        dev = default_device()
        scores, ids = [], []
        for b in batches:
            p = self(to_device(b, dev), k=k)
            scores.append(p.scores.cpu().numpy())
            ids.append(p.identifiers.cpu().numpy())
        return np.concatenate(scores), np.concatenate(ids)

    def evaluate(self, batches, target: Optional[str] = None, metrics: Optional[Sequence["TopKMetric"]] = None) -> Dict[str, float]:
        """Ranking metrics of the positive item `target` (default: the item-id column) against the index."""
        target = target or self.target
        if target is None:
            raise ValueError("`target` (name of the positive item-id column) is required")
        return evaluate_topk(lambda b: self(b, targets=b[target], testing=True, k=_max_k(metrics, self.k)), batches, metrics)


# ------------------------------------------------------------------------------------------------
# ranking metrics (metrics/topk.py:48-190) on pre-sorted (B, k) relevance matrices
# ------------------------------------------------------------------------------------------------
class TopKMetric:
    name = "metric"

    def __init__(self, k: int = 10):
        self.k = int(k)

    def __call__(self, y_true: torch.Tensor, label_relevant_counts: Optional[torch.Tensor] = None) -> torch.Tensor:
        if y_true.shape[1] < self.k:
            raise ValueError(f"{self.label}: needs the top {self.k} predictions, got {y_true.shape[1]}")
        if label_relevant_counts is None:
            label_relevant_counts = y_true.sum(dim=1)
        return self.compute(y_true.to(torch.float32), label_relevant_counts.to(torch.float32))

    @property
    def label(self) -> str:
        return f"{self.name}_{self.k}"

    def compute(self, y_true, rel):  # pragma: no cover - abstract
        raise NotImplementedError


def _div_no_nan(a, b):
    return torch.where(b != 0, a / torch.where(b != 0, b, torch.ones_like(b)), torch.zeros_like(a))


def _dcg(y_true, k):
    pos = torch.arange(k, device=y_true.device, dtype=torch.float32)
    disc = 1.0 / (torch.log(pos + 2.0) / math.log(2.0))
    return (y_true[:, :k] * disc).sum(dim=1)


class RecallAt(TopKMetric):
    name = "recall_at"

    def compute(self, y_true, rel):
        return _div_no_nan(y_true[:, :self.k].sum(dim=1), rel.clamp(1, float(self.k)))


class PrecisionAt(TopKMetric):
    name = "precision_at"

    def compute(self, y_true, rel):
        return y_true[:, :self.k].mean(dim=1)


class AvgPrecisionAt(TopKMetric):
    name = "map_at"

    def compute(self, y_true, rel):
        k = self.k
        ranks = torch.arange(1, k + 1, device=y_true.device, dtype=torch.float32)
        precisions = y_true[:, :k].cumsum(dim=1) / ranks
        return _div_no_nan((precisions * y_true[:, :k]).sum(dim=1), rel.clamp(1, float(k)))


class NDCGAt(TopKMetric):
    name = "ndcg_at"

    def compute(self, y_true, rel):
        k = self.k
        ideal = (torch.arange(k, device=y_true.device, dtype=torch.float32).unsqueeze(0) < rel.unsqueeze(1)).to(torch.float32)
        return _div_no_nan(_dcg(y_true, k), _dcg(ideal, k))


class MRRAt(TopKMetric):
    name = "mrr_at"

    def compute(self, y_true, rel):
        first = (y_true.argmax(dim=1) + 1).to(torch.float32)
        hit = y_true[:, :self.k].max(dim=1).values
        return _div_no_nan(torch.ones_like(first), first * hit)


def _max_k(metrics, default: int) -> int:
    return max([m.k for m in metrics]) if metrics else default


def evaluate_topk(predict, batches, metrics: Optional[Sequence[TopKMetric]] = None) -> Dict[str, float]:
    """Mean of every metric over all rows of all batches; `predict(device batch) -> Prediction(scores, targets)`
    with rows already sorted by score (top-k kernels return them sorted).  Dict batches are moved to the device first;
    other batches (a model's (inputs, targets) tuples) reach `predict` as they are."""
    metrics = list(metrics) if metrics else [RecallAt(10), NDCGAt(10)]
    if isinstance(batches, dict):
        batches = [batches]
    dev = default_device()
    sums = {m.label: 0.0 for m in metrics}
    rows = 0
    for b in batches:
        pred = predict(to_device(b, dev) if isinstance(b, dict) else b)
        rel = pred.extra.get("label_relevant_counts") if isinstance(pred, Prediction) else None
        for m in metrics:
            sums[m.label] += float(m(pred.targets, rel).sum().item())
        rows += pred.targets.shape[0]
    if rows == 0:
        raise ValueError("evaluate: no rows")
    return {k: v / rows for k, v in sums.items()}
