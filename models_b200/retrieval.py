"""Two-tower retrieval: TwoTowerBlock, in-batch sampler, ItemRetrievalScorer / ItemRetrievalTask
(v1 API used by mm.TwoTowerModel) and ContrastiveOutput (v2 API).

Reference: merlin/models/tf/blocks/retrieval/{two_tower,base}.py, blocks/sampling/in_batch.py,
prediction_tasks/retrieval.py, outputs/contrastive.py, outputs/sampling/{in_batch,popularity}.py,
utils/tf_utils.py:126-154.  The scorer is one fused kernel: Q.N^T + false-negative mask + logQ +
[pos | neg] layout + temperature, writing the (B, 1+N) logits exactly once.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import ops
from .blocks import MLP, dense_engine
from .core import Block, Prediction, TabularData, unique_name
from .inputs import EmbeddingOptions, InputBlock
from .schema import Schema, Tags

MIN_FLOAT = float(np.finfo(np.float16).min) / 100.0  # merlin/models/utils/constants.py:19


class L2Norm(Block):
    """transforms/regularization.py:27-82."""

    def call(self, inputs, **kwargs):
        if isinstance(inputs, dict):
            return {k: ops.l2_normalize(v) for k, v in inputs.items()}
        return ops.l2_normalize(inputs)


class TowerBlock(Block):
    """One tower: legacy InputBlock(schema subset) -> tower MLP (two_tower.py:98-118).  The
    sorted-name concat that the first _Dense applies to the InputBlock's dict is produced directly
    by the fused gather (embeddings land at their concat offsets).  mlp=None: the tower is the concat
    of its embeddings (QueryItemIdsEmbeddingsBlock)."""

    def __init__(self, inputs: InputBlock, mlp: Optional[MLP], name: str):
        super().__init__(name)
        self.inputs = inputs
        self.mlp = mlp

    def build(self, device=None):
        self.inputs.build(device)
        if self.mlp is not None:
            _, _, width = self.inputs.layout()
            self.mlp.build_from_width(width, device)
        self.built = True
        return self

    def weights(self):
        out = {f"inputs/{k}": v for k, v in self.inputs.weights().items()}
        if self.mlp is not None:
            out.update({f"mlp/{k}": v for k, v in self.mlp.weights().items()})
        return out

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        x = self.inputs.concat(inputs)
        return x if self.mlp is None else self.mlp(x, **kwargs)


class TwoTowerBlock(Block):
    """blocks/retrieval/two_tower.py:32-118 / DualEncoderBlock (retrieval/base.py:59-129)."""

    def __init__(self, schema: Schema, query_tower: MLP, item_tower: Optional[MLP] = None,
                 query_tower_tag=Tags.USER, item_tower_tag=Tags.ITEM,
                 embedding_options: EmbeddingOptions = EmbeddingOptions(embedding_dims=None, embedding_dim_default=64,
                                                                        infer_embedding_sizes=False,
                                                                        infer_embedding_sizes_multiplier=2.0),
                 post: Optional[Block] = None, **kwargs):
        if schema is None:
            raise ValueError("The schema is required by TwoTower")
        if query_tower is None:
            raise ValueError("The query_tower is required by TwoTower")
        super().__init__(unique_name("two_tower_block"))
        _item_tower = item_tower or query_tower.copy()
        if isinstance(_item_tower, TowerBlock):
            self.item = _item_tower
        else:
            item_schema = schema.select_by_tag(item_tower_tag) if item_tower_tag else schema
            if not item_schema:
                raise ValueError(
                    f"The schema should contain features with the tag `{item_tower_tag}`,"
                    "required by item-tower"
                )
            self.item = TowerBlock(InputBlock(item_schema, embedding_options=embedding_options), _item_tower, "item")
        if isinstance(query_tower, TowerBlock):
            self.query = query_tower
        else:
            query_schema = schema.select_by_tag(query_tower_tag) if query_tower_tag else schema
            if not query_schema:
                raise ValueError(
                    f"The schema should contain features with the tag `{query_schema}`,"
                    "required by query-tower"
                )
            self.query = TowerBlock(InputBlock(query_schema, embedding_options=embedding_options), query_tower, "query")
        if isinstance(post, str):
            if post not in ("l2-norm", "l2_norm"):
                raise ValueError(f"Unknown post block {post!r}")
            post = L2Norm()
        self.post = post
        self.schema = schema

    def build(self, device=None):
        self.query.build(device)
        self.item.build(device)
        self.built = True
        return self

    def weights(self):
        out = {f"query/{k}": v for k, v in self.query.weights().items()}
        out.update({f"item/{k}": v for k, v in self.item.weights().items()})
        return out

    def call(self, inputs: TabularData, **kwargs) -> Dict[str, torch.Tensor]:
        out = {"query": self.query(inputs, **kwargs), "item": self.item(inputs, **kwargs)}
        if self.post is not None:
            out = self.post(out)
        return out


class QueryItemIdsEmbeddingsBlock(TwoTowerBlock):
    """blocks/retrieval/matrix_factorization.py:31-112: a dual encoder whose towers are the id embeddings themselves
    (no MLP): the query tower embeds the columns tagged `query_id_tag`, the item tower those tagged `item_id_tag`, each
    table `dim` wide, with EmbeddingOptions(embedding_dim_default=dim, embeddings_l2_reg=...).  The training step adds
    embeddings_l2_reg * sum ||e||^2 over the batch's looked-up embeddings to the loss, as the reference does."""

    def __init__(self, schema: Schema, dim: int, query_id_tag=Tags.USER_ID, item_id_tag=Tags.ITEM_ID,
                 embeddings_initializers=None, embeddings_l2_reg: float = 0.0, post: Optional[Block] = None, **kwargs):
        if schema is None:
            raise ValueError("The schema is required by QueryItemIdsEmbeddingsBlock")
        if embeddings_l2_reg < 0:
            raise ValueError(f"embeddings_l2_reg must be >= 0, got {embeddings_l2_reg}")
        opts = EmbeddingOptions(embedding_dim_default=int(dim), embeddings_l2_reg=float(embeddings_l2_reg),
                                embeddings_initializers=embeddings_initializers or None)
        towers = []
        for tag, name in ((query_id_tag, "query"), (item_id_tag, "item")):
            sub = schema.select_by_tag(tag)
            if not sub:
                raise ValueError(f"The schema should contain features with the tag `{tag}`, required by the {name} embeddings")
            towers.append(TowerBlock(InputBlock(sub, embedding_options=opts), None, name))
        super().__init__(schema, towers[0], towers[1], post=post)
        self.dim = int(dim)


# ------------------------------------------------------------------------------------------------
# samplers
# ------------------------------------------------------------------------------------------------
class InBatchSampler:
    """blocks/sampling/in_batch.py:25-113 / outputs/sampling/in_batch.py:25-100: the negatives are
    the batch's own item embeddings and ids (identity)."""

    def __init__(self, batch_size: Optional[int] = None, **kwargs):
        self.batch_size = batch_size

    def sample(self, item_embeddings: torch.Tensor, item_ids: Optional[torch.Tensor]):
        return item_embeddings, item_ids, None


InBatchSamplerV2 = InBatchSampler


class PopularityBasedSamplerV2:
    """outputs/sampling/popularity.py:24-195: negatives for sampled softmax drawn over the WHOLE catalog from the
    log-uniform (Zipfian) law of tf.random.log_uniform_candidate_sampler — P(k) = (log(k+2) - log(k+1)) / log(R+1) on
    k = 0..R-1, R = max_id - min_id, shifted by min_id — assuming ids are sorted by decreasing frequency.  It returns ids
    only (the output layer looks their embeddings up) and provides the sampling probabilities of positives and negatives
    for the logQ correction (`sampling_dist`, the formula of :141-165: for unique=True the probability of being drawn at
    least once in max_num_samples trials).
    The random draw runs as a few torch ops on the device: it is data preparation (the reference's sampler is a TF random
    op whose stream cannot be reproduced bit-wise), not part of the scored path; `seed` makes it reproducible here."""

    def __init__(self, max_id: int, min_id: int = 0, max_num_samples: int = 10, unique: Optional[bool] = True,
                 seed: Optional[int] = None, **kwargs):
        assert max_num_samples <= max_id, (f"Number of items to sample `{max_num_samples}`"
                                           f"should be less than total number of ids `{max_id}`")
        self.max_id, self.min_id, self.max_num_samples = int(max_id), int(min_id), int(max_num_samples)
        self.unique, self.seed = bool(unique), seed
        self.sampling_dist = self.get_sampling_distribution()
        self._dist_dev: Dict[str, torch.Tensor] = {}
        self._gen: Dict[str, torch.Generator] = {}

    def get_sampling_distribution(self) -> np.ndarray:
        return log_uniform_sampling_probs(self.max_id, self.min_id, self.max_num_samples, unique=self.unique)

    def _generator(self, device) -> torch.Generator:
        g = self._gen.get(str(device))
        if g is None:
            g = torch.Generator(device=device)
            g.manual_seed(0x5EED if self.seed is None else int(self.seed))
            self._gen[str(device)] = g
        return g

    def sample_ids(self, device) -> torch.Tensor:
        """(max_num_samples,) int64 ids in [min_id, max_id)."""
        R, n = self.max_id - self.min_id, self.max_num_samples
        g = self._generator(device)
        log_r1 = float(np.log(R + 1.0))

        def draw(m):
            u = torch.rand(m, device=device, generator=g, dtype=torch.float64)
            return torch.clamp((torch.exp(u * log_r1) - 1.0).floor().to(torch.int64), 0, R - 1)

        if not self.unique:
            return draw(n) + self.min_id
        got = torch.unique(draw(2 * n))
        while got.numel() < n:  # rejection until n distinct ids (as the TF sampler does)
            got = torch.unique(torch.cat([got, draw(2 * n)]))
        # torch.unique sorts: keep a random subset so that the kept set is not biased to small ids
        keep = torch.randperm(got.numel(), device=device, generator=g)[:n]
        return got[keep] + self.min_id

    def sampling_probs(self, ids: torch.Tensor) -> torch.Tensor:
        """with_sampling_probs (:167-185): gather of the sampling distribution by id."""
        key = str(ids.device)
        d = self._dist_dev.get(key)
        if d is None:
            d = torch.from_numpy(self.sampling_dist).to(ids.device)
            self._dist_dev[key] = d
        return d[ids.reshape(-1).long()].contiguous()

    def sample(self, item_embeddings=None, item_ids=None):
        """(embeddings=None, ids, probabilities): the caller looks the embeddings up."""
        dev = item_embeddings.device if item_embeddings is not None else item_ids.device
        ids = self.sample_ids(dev)
        return None, ids, self.sampling_probs(ids)


def log_uniform_sampling_probs(max_id: int, min_id: int = 0, max_num_samples: int = 0, unique: bool = True) -> np.ndarray:
    """PopularityBasedSamplerV2 sampling probabilities (outputs/sampling/popularity.py:141-165)."""
    R = max_id - min_id
    k = np.arange(R + 1, dtype=np.float64)
    p = (np.log(k + 2.0) - np.log(k + 1.0)) / np.log(R + 2.0)
    if unique:
        p = -np.expm1(max_num_samples * np.log1p(-p))
    return np.concatenate([np.zeros(min_id), p]).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# scorer (v1) and contrastive output (v2)
# ------------------------------------------------------------------------------------------------
_TARGET_ROWS: Dict[tuple, torch.Tensor] = {}


def _target_row(width: int, device) -> torch.Tensor:
    """[1, 0, 0, ...] (cached per width/device; built without host scalars so it is graph-capturable)."""
    key = (width, str(device))
    row = _TARGET_ROWS.get(key)
    if row is None:
        row = torch.zeros(width, dtype=torch.float32, device=device)
        row[:1].fill_(1.0)
        if len(_TARGET_ROWS) > 16:
            _TARGET_ROWS.clear()
        _TARGET_ROWS[key] = row
    return row


def _score(query, pos_item, neg_items, pos_ids, neg_ids, downscore, false_neg_score, temperature,
           pos_prob=None, neg_prob=None, fused_loss: bool = False) -> Prediction:
    B, N = query.shape[0], neg_items.shape[0]
    if fused_loss:
        # soft-max cross-entropy against the one-hot target on column 0, straight from the GEMM epilogue: the
        # (B, 1+N) logits (1.07 GB at B = 16 384) are never written.  outputs = (B,3) [max, log-sum-exp, positive logit]
        if dense_engine() == "fp32":
            raise NotImplementedError("fused_loss runs on the tensor-core engine")
        stats = ops.inbatch_softmax_ce(query.contiguous(), pos_item.contiguous(), neg_items.contiguous(), pos_ids=pos_ids,
                                       neg_ids=neg_ids, downscore=downscore, false_neg_score=false_neg_score,
                                       pos_prob=pos_prob, neg_prob=neg_prob, temperature=temperature)
        return Prediction(stats, None, negative_candidate_ids=neg_ids, kind="softmax_ce_stats")
    # (B, 1+N) logits as a view into a (B, 4+Nr) buffer starting at physical column 3: the negatives
    # (logical columns 1..N) then start 16-byte aligned in every row, so the GEMM epilogue can use
    # 128-bit stores; Nr = N rounded up to 4 keeps the row stride a multiple of 16 bytes
    Nr = (N + 3) // 4 * 4
    out = torch.empty((B, 4 + Nr), dtype=torch.float32, device=query.device)[:, 3:4 + N]
    ops.inbatch_scores(query.contiguous(), pos_item.contiguous(), neg_items.contiguous(), out, pos_ids=pos_ids,
                       neg_ids=neg_ids, downscore=downscore, false_neg_score=false_neg_score, pos_prob=pos_prob,
                       neg_prob=neg_prob, temperature=temperature, tensor_cores=dense_engine() != "fp32")
    # targets: one-hot on column 0 (retrieval/base.py:413-422) as a broadcast view — the reference
    # materialises a second (B, 1+N) tensor; nothing downstream needs it resident
    return Prediction(out, _target_row(1 + N, query.device).unsqueeze(0).expand(B, 1 + N), negative_candidate_ids=neg_ids)


class ItemRetrievalScorer(Block):
    """blocks/retrieval/base.py:134-502 (in-batch / sampled negatives mode)."""

    def _sampled_softmax(self, query: torch.Tensor, targets: torch.Tensor, temperature: float, fused_loss: bool) -> Prediction:
        pos = _lookup_rows(self.item_table, targets)
        neg, nid, _, _ = _sampled_negatives(self.samplers, self.item_table, pos, targets, logq=False)
        return _score(query, pos, neg, targets, nid, self.downscore_false_negatives and nid is not None, self.false_negatives_score,
                      temperature, fused_loss=fused_loss)

    def __init__(self, samplers: Sequence = (), sampling_downscore_false_negatives: bool = True,
                 sampling_downscore_false_negatives_value: float = MIN_FLOAT, item_id_feature_name: str = "item_id",
                 item_domain: str = "item_id", query_name: str = "query", item_name: str = "item",
                 cache_query: bool = False, sampled_softmax_mode: bool = False, store_negative_ids: bool = False,
                 **kwargs):
        super().__init__(unique_name("item_retrieval_scorer"))
        self.samplers = list(samplers) if samplers else [InBatchSampler()]
        self.downscore_false_negatives = sampling_downscore_false_negatives
        self.false_negatives_score = sampling_downscore_false_negatives_value
        self.item_id_feature_name = item_id_feature_name
        self.query_name, self.item_name = query_name, item_name
        self.store_negative_ids = store_negative_ids
        self.sampled_softmax_mode = bool(sampled_softmax_mode)
        # sampled_softmax_mode (retrieval/base.py:274,313,431-453) reads the item embedding table from the model
        # context in the reference; here it is handed over explicitly
        self.item_table = kwargs.pop("item_table", None)
        if self.sampled_softmax_mode and self.item_table is None:
            raise ValueError("sampled_softmax_mode=True needs `item_table=` (the EmbeddingTable of the item-id domain)")
        if cache_query:
            raise NotImplementedError("cache_query is outside the forward hot path")

    def _check_input_from_two_tower(self, inputs):
        if set(inputs.keys()) != {self.query_name, self.item_name}:
            raise ValueError(
                f"Wrong input-names, expected: {[self.query_name, self.item_name]} "
                f"but got: {inputs.keys()}"
            )

    def call(self, inputs: Dict[str, torch.Tensor], training: bool = False, testing: bool = False, **kwargs):
        """Inference: (B,1) positive scores (retrieval/base.py:277-281); sampled_softmax_mode: the (B, N_I) logits
        of the whole catalog, x @ E^T (:431-438)."""
        if training or testing:
            return inputs
        if self.sampled_softmax_mode:
            if not isinstance(inputs, torch.Tensor):
                raise ValueError(f"Inputs to the Sampled Softmax block should be tensors, got {type(inputs)}")
            self.item_table.build(inputs.device)
            E = self.item_table.embeddings
            out = torch.empty((inputs.shape[0], E.shape[0]), dtype=torch.float32, device=inputs.device)
            ops.dense_tc(ops.split_rows(inputs.contiguous()), inputs.shape[1], ops.split_weights(E.t().contiguous()), E.shape[0], None,
                         "linear", out_f32=out)
            return out
        self._check_input_from_two_tower(inputs)
        q, it = inputs[self.query_name], inputs[self.item_name]
        out = torch.empty((q.shape[0], 1), dtype=torch.float32, device=q.device)
        return ops.rowwise_dot(q, it, out)

    def call_outputs(self, predictions: Dict[str, torch.Tensor], features: TabularData, temperature: float = 1.0,
                     fused_loss: bool = False, **kwargs) -> Prediction:
        """Training / testing logits (retrieval/base.py:283-429); `fused_loss=True`: the cross-entropy statistics
        of those logits instead of the logits (see _score)."""
        assert len(self.samplers) > 0, "At least one sampler is required by ItemRetrievalScorer for negative sampling"
        if self.sampled_softmax_mode:
            # positives: rows of the item table at the target ids (:440-453); negatives: sampled ids -> rows
            targets = kwargs.get("targets")
            if targets is None or not isinstance(predictions, torch.Tensor):
                raise ValueError("sampled_softmax_mode needs the query tensor as predictions and `targets` = positive item ids")
            return self._sampled_softmax(predictions, targets.reshape(-1), temperature, fused_loss)
        self._check_input_from_two_tower(predictions)
        q, items = predictions[self.query_name], predictions[self.item_name]
        pos_ids = None
        if self.downscore_false_negatives or self.store_negative_ids:
            if self.item_id_feature_name not in features:
                raise ValueError(f"the item id feature {self.item_id_feature_name!r} is required to "
                                 "downscore false negatives")
            pos_ids = features[self.item_id_feature_name].reshape(-1)
        neg_e, neg_i = [], []
        for s in self.samplers:
            e, i, _ = s.sample(items, pos_ids)
            if e.shape[0] > 0:
                neg_e.append(e)
                neg_i.append(i)
        if not neg_e:
            raise Exception(f"No negative items where sampled from samplers {self.samplers}")
        neg = neg_e[0] if len(neg_e) == 1 else torch.cat(neg_e, dim=0)
        nid = None
        if pos_ids is not None:
            nid = neg_i[0] if len(neg_i) == 1 else torch.cat(neg_i, dim=0)
        return _score(q, items, neg, pos_ids, nid, self.downscore_false_negatives, self.false_negatives_score,
                      temperature, fused_loss=fused_loss)


def _lookup_rows(table, ids: torch.Tensor) -> torch.Tensor:
    """(n, D) rows of an EmbeddingTable (mm_gather_multi)."""
    table.build(ids.device)
    out = torch.empty((ids.numel(), table.dim), dtype=torch.float32, device=ids.device)
    ops.gather_multi([table.embeddings], [ids.reshape(-1).contiguous()], [0], out)
    return out


def _sampled_negatives(samplers, table, pos_emb, pos_ids, logq: bool):
    """Negatives from `samplers` (in-batch and / or popularity-based): embeddings, ids, and — for the logQ correction,
    which the reference allows with exactly one sampler — the sampling probabilities of positives and negatives."""
    neg_e, neg_i = [], []
    pos_prob = neg_prob = None
    if logq and len(samplers) > 1:
        raise ValueError("It is only possible to apply logQ sampling correction "
                         "(logq_sampling_correction=True) when only one negative sampler is provided.")
    for s in samplers:
        e, i, p = s.sample(pos_emb, pos_ids)
        if e is None:  # id-only sampler: look the rows up in the candidate table
            if table is None:
                raise ValueError(f"{type(s).__name__} samples ids: the output layer needs the candidate EmbeddingTable to embed them")
            e = _lookup_rows(table, i)
        if logq:
            if not hasattr(s, "sampling_probs"):
                raise ValueError(f"{type(s).__name__} does not provide sampling probabilities (with_sampling_probs) for logQ")
            pos_prob, neg_prob = s.sampling_probs(pos_ids), (p if p is not None else s.sampling_probs(i))
        if e.shape[0] > 0:
            neg_e.append(e)
            neg_i.append(i)
    if not neg_e:
        raise Exception(f"No negative items where sampled from samplers {samplers}")
    neg = neg_e[0] if len(neg_e) == 1 else torch.cat(neg_e, dim=0)
    nid = None
    if all(i is not None for i in neg_i):
        nid = neg_i[0] if len(neg_i) == 1 else torch.cat([i.reshape(-1) for i in neg_i], dim=0)
    return neg, nid, pos_prob, neg_prob


class ItemRetrievalTask(Block):
    """prediction_tasks/retrieval.py:33-191: ItemRetrievalScorer (+ LogitsTemperatureScaler when
    T != 1, applied only in training/testing — transforms/bias.py:44-52).  Its loss is the v1 default,
    CategoricalCrossentropy(from_logits=True) against the one-hot on column 0 (:69)."""

    loss = "categorical_crossentropy"

    def __init__(self, schema: Schema, samplers: Sequence = (), target_name: Optional[str] = None,
                 task_name: Optional[str] = None, post_logits=None, logits_temperature: float = 1.0,
                 cache_query: bool = False, store_negative_ids: bool = False, **kwargs):
        super().__init__(task_name or unique_name("item_retrieval_task"))
        if post_logits is not None:
            raise NotImplementedError("post_logits blocks are outside the hot path")
        ids = schema.select_by_tag(Tags.ITEM_ID).column_names
        if not ids:
            raise ValueError("ItemRetrievalTask needs a column tagged ITEM_ID in the schema")
        self.schema = schema
        self.item_id_feature_name = ids[0]
        self.logits_temperature = float(logits_temperature)
        self.scorer = ItemRetrievalScorer(samplers=samplers, item_id_feature_name=self.item_id_feature_name,
                                          cache_query=cache_query, store_negative_ids=store_negative_ids)
        self.target_name = target_name

    def call(self, inputs, features: Optional[TabularData] = None, training: bool = False, testing: bool = False,
             fused_loss: bool = False, **kwargs):
        if training or testing:
            return self.scorer.call_outputs(inputs, features, temperature=self.logits_temperature, fused_loss=fused_loss)
        return self.scorer(inputs)


class ContrastiveOutput(Block):
    """outputs/contrastive.py:47-453 (DotProduct to_call, in-batch / provided negatives).

    call({query_name: (B,D), candidate_name: (B,D)}, candidate_ids, training|testing) -> Prediction
    with logits (B, 1+N); inference -> (B,1) row-wise dot (outputs/base.py:291-322)."""

    def __init__(self, to_call=None, negative_samplers="in-batch", target_name: Optional[str] = None,
                 logits_temperature: float = 1.0, name: Optional[str] = None, downscore_false_negatives: bool = True,
                 false_negative_score: float = MIN_FLOAT, query_name: str = "query", candidate_name: str = "candidate",
                 store_negative_ids: bool = False, logq_sampling_correction: Optional[bool] = False, **kwargs):
        super().__init__(name or unique_name("contrastive_output"))
        self.to_call = to_call
        if isinstance(negative_samplers, (str, InBatchSampler, PopularityBasedSamplerV2)):
            negative_samplers = [negative_samplers]
        self.negative_samplers = [InBatchSampler() if s in ("in-batch", "in_batch") else s for s in negative_samplers]
        if not self.negative_samplers:
            raise ValueError("At least one negative sampler is required")
        self.logits_temperature = float(logits_temperature)
        self.downscore_false_negatives = downscore_false_negatives
        self.false_negative_score = false_negative_score
        self.query_name, self.candidate_name = query_name, candidate_name
        self.store_negative_ids = store_negative_ids
        self.logq_sampling_correction = logq_sampling_correction

    @property
    def has_candidate_weights(self) -> bool:
        """to_call is an item EmbeddingTable (LookUpProtocol, contrastive.py:420-425): positives are rows of it at the
        target ids and sampled negative ids are embedded by it — the sampled-softmax set-up."""
        from .inputs import EmbeddingTable

        return isinstance(self.to_call, EmbeddingTable)

    def call(self, inputs, candidate_ids: Optional[torch.Tensor] = None, training: bool = False, testing: bool = False,
             sampling_probs: Optional[torch.Tensor] = None, fused_loss: bool = False, targets: Optional[torch.Tensor] = None,
             **kwargs):
        """call_contrastive (contrastive.py:223-274) + outputs (:276-344)."""
        if isinstance(inputs, dict) and self.query_name in inputs:
            q = inputs[self.query_name]
        elif isinstance(inputs, torch.Tensor):
            q = inputs
        else:
            raise ValueError("Couldn't infer query embedding")
        table = self.to_call if self.has_candidate_weights else None
        if not (training or testing):
            if table is not None:  # inference over the whole catalog: x @ E^T
                table.build(q.device)
                E = table.embeddings
                out = torch.empty((q.shape[0], E.shape[0]), dtype=torch.float32, device=q.device)
                ops.dense_tc(ops.split_rows(q.contiguous()), q.shape[1], ops.split_weights(E.t().contiguous()), E.shape[0], None,
                             "linear", out_f32=out)
                return out
            c = inputs[self.candidate_name]
            out = torch.empty((q.shape[0], 1), dtype=torch.float32, device=q.device)
            return ops.rowwise_dot(q, c, out)
        if table is not None:
            if targets is None:
                raise ValueError("ContrastiveOutput over an EmbeddingTable needs `targets` (the positive item ids)")
            ids = targets.reshape(-1)
            c = _lookup_rows(table, ids)
        else:
            c = inputs[self.candidate_name]
            if self.downscore_false_negatives and candidate_ids is None:
                raise ValueError("candidate ids are required to downscore false negatives")
            ids = None if candidate_ids is None else candidate_ids.reshape(-1)
        use_sampler_probs = self.logq_sampling_correction and sampling_probs is None
        neg, nid, pos_prob, neg_prob = _sampled_negatives(self.negative_samplers, table, c, ids, logq=use_sampler_probs)
        if self.logq_sampling_correction and not use_sampler_probs:
            # explicit probability table over item ids (contrastive.py:309-319 with the probabilities gathered by id)
            pos_prob = sampling_probs[ids.long()].contiguous()
            neg_prob = sampling_probs[nid.long()].contiguous()
        downscore = self.downscore_false_negatives and ids is not None and nid is not None
        return _score(q, c, neg, ids, nid, downscore, self.false_negative_score, self.logits_temperature, pos_prob, neg_prob,
                      fused_loss=fused_loss)


# ------------------------------------------------------------------------------------------------
# full-catalog scoring (a14)
# ------------------------------------------------------------------------------------------------
class CategoricalOutput(Block):
    """outputs/classification.py:127-216 with the weight-tied `EmbeddingTablePrediction` to_call
    (:311-382): logits = x @ E^T + bias over the whole item table E (N_I, D).

    call(x)                      -> (B, N_I) logits, materialised (what the reference returns; only
                                    sensible for small catalogs)
    softmax_ce_stats(x, targets) -> (B, 3) [row max, log-sum-exp, logit[target]] — everything
                                    CategoricalCrossEntropy(from_logits=True) needs
                                    (losses/listwise.py:38-50): loss = lse - logit[target]
    top_k(x, k)                  -> (scores, ids) in tf.math.top_k order (outputs/topk.py:221-223)
    The last two stream the catalog through one wgmma GEMM without ever writing (B, N_I).
    `Model(InputBlockV2, MLPBlock, CategoricalOutput)` trains it (models.CatalogModel, train.CatalogTrainer) on the
    `target_name` column."""

    loss = "categorical_crossentropy"

    def __init__(self, to_call, logits_temperature: float = 1.0, use_bias: bool = True, name: Optional[str] = None,
                 target_name: Optional[str] = None, **kwargs):
        from .inputs import EmbeddingTable

        super().__init__(name or unique_name("categorical_output"))
        if not isinstance(to_call, EmbeddingTable):
            raise NotImplementedError("CategoricalOutput(to_call=...) supports a weight-tied EmbeddingTable")
        self.table = to_call
        # the target column: class ids in [0, N_I) (classification.py:190-196 takes the table's column by default and a
        # `target=` keyword over it)
        target = kwargs.pop("target", None)
        if target is not None and target_name is not None and target != target_name:
            raise ValueError(f"CategoricalOutput: target={target!r} and target_name={target_name!r} name different columns")
        self.target_name = target_name or target or to_call.col_schema.name
        self.target = self.target_name
        self.num_classes = to_call.input_dim
        self.logits_temperature = float(logits_temperature)
        self.use_bias = use_bias
        self.bias: Optional[torch.Tensor] = None
        self._e_split: Optional[torch.Tensor] = None
        self._w_split: Optional[torch.Tensor] = None

    def build(self, device=None):
        self.table.build(device)
        if self.use_bias and self.bias is None:
            self.bias = torch.zeros(self.num_classes, dtype=torch.float32, device=self.table.table.device)
        self.built = True
        return self

    def weights(self):
        out = {"embeddings": self.table.embeddings}
        if self.bias is not None:
            out["bias"] = self.bias
        return out

    _TRANSIENT = {"_e_split": None, "_w_split": None, "_t_key": None, "_t_vec": None, "_t_bias": None}

    def refresh(self) -> None:
        """Drop the cached split-bf16 copies (call after changing the table)."""
        from .core import bump_weights_version

        self._e_split = self._w_split = None
        self._t_key = None
        bump_weights_version()

    _weights_changed = refresh

    def _catalog_split(self) -> torch.Tensor:
        if self._e_split is None:
            self._e_split = ops.split_rows(self.table.embeddings)  # (N_I, 2*Kp), once per catalog
        return self._e_split

    def _tempered(self, x: torch.Tensor):
        """LogitsTemperatureScaler (transforms/bias.py:44-52, applied to the logits in training and testing):
        (x E^T + b) / T = (x / T) E^T + b / T — the query is scaled by mm_scale_shift, the bias copy is cached."""
        T = self.logits_temperature
        if T == 1.0:
            return x, self.bias
        key = (str(x.device), x.shape[1])
        if getattr(self, "_t_key", None) != key:
            self._t_vec = (torch.full((x.shape[1],), 1.0 / T, dtype=torch.float32, device=x.device),
                           torch.zeros(x.shape[1], dtype=torch.float32, device=x.device))
            self._t_bias = None if self.bias is None else (self.bias / T).contiguous()
            self._t_key = key
        return ops.scale_shift(x.contiguous(), *self._t_vec), self._t_bias

    def call(self, x: torch.Tensor, training: bool = False, testing: bool = False, **kwargs) -> torch.Tensor:
        self.build(x.device)
        bias = self.bias
        if training or testing:
            x, bias = self._tempered(x)
        if self._w_split is None:
            self._w_split = ops.split_weights(self.table.embeddings.t().contiguous())
        out = torch.empty((x.shape[0], self.num_classes), dtype=torch.float32, device=x.device)
        ops.dense_tc(ops.split_rows(x), x.shape[1], self._w_split, self.num_classes, bias, "linear", out_f32=out)
        return out

    def softmax_ce_stats(self, x: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        """[max, log-sum-exp, logit[target]] of the TRAINING logits, i.e. with the temperature applied."""
        self.build(x.device)
        x, bias = self._tempered(x)
        stats, _, _ = ops.catalog_score(x, self._catalog_split(), self.num_classes, bias=bias, targets=targets, k=0)
        return stats

    def top_k(self, x: torch.Tensor, k: int):
        self.build(x.device)
        _, scores, ids = ops.catalog_score(x, self._catalog_split(), self.num_classes, bias=self.bias, k=k, want_stats=False)
        return scores, ids


# ------------------------------------------------------------------------------------------------
# V2 API: Encoder towers + RetrievalModelV2 (models/retrieval.py:409-486, core/encoder.py:41-260)
# ------------------------------------------------------------------------------------------------
class Encoder(Block):
    """core/encoder.py:41-110: `Encoder(schema_or_input_block, *blocks, pre=None, post=None)` — InputBlockV2 (sorted-name
    concat of embeddings and continuous columns) followed by the blocks; feature dict -> (B, D)."""

    def __init__(self, inputs, *blocks, pre: Optional[Block] = None, post: Optional[Block] = None, **kwargs):
        from .inputs import InputBlockV2

        super().__init__(unique_name("encoder"))
        if pre is not None:
            raise NotImplementedError("Encoder(pre=...) is outside the hot path")
        if isinstance(inputs, Schema):
            self._schema = inputs
            inputs = InputBlockV2(inputs, **kwargs)
        else:
            self._schema = getattr(inputs, "schema", None)
        self.inputs = inputs
        self.blocks = list(blocks)
        self.post = L2Norm() if post in ("l2-norm", "l2_norm") else post

    @property
    def schema(self) -> Schema:
        return self._schema

    def build(self, device=None):
        self.inputs.build(device)
        width = self.inputs.layout()[2]
        for b in self.blocks:
            if isinstance(b, MLP):
                b.build_from_width(width, device)
                width = b.dense_layers[-1].units
        self.built = True
        return self

    def weights(self):
        out = {f"inputs/{k}": v for k, v in self.inputs.weights().items()}
        for i, b in enumerate(self.blocks):
            out.update({f"block_{i}/{k}": v for k, v in b.weights().items()})
        return out

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        x = self.inputs(inputs)
        for b in self.blocks:
            x = b(x)
        return self.post(x) if self.post is not None else x
