"""The reference's pairwise ranking losses for retrieval models (losses/pairwise.py:44-395), by their registry names.

    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([128, 64]))
    model.compile(optimizer="adam", loss="bpr")                      # or loss=mm.losses.BPRmaxLoss(reg_lambda=0.5)

Each class only names a loss (its kind and, for BPR-max, reg_lambda): the retrieval training step
(models_b200/train.py: TwoTowerTrainer) computes it over the in-batch scores with mm_inbatch_pairwise_fwd / _bwd.  The
positive is column 0 of the scores, the negatives the batch's items (false negatives down-scored to a constant), and the
loss is the mean over the (B, N) per-element losses (Keras' SUM_OVER_BATCH_SIZE; top1_v2: the mean of its (B, 1) rows).

CategoricalCrossEntropy / CategoricalCrossentropy name the full-catalog soft-max cross-entropy of a CategoricalOutput
model with its label smoothing (models_b200/train.py: CatalogTrainer):

    model.compile(optimizer="adam", loss=mm.losses.CategoricalCrossEntropy(from_logits=True, label_smoothing=0.1))
"""
from __future__ import annotations

from typing import Dict, Optional, Type


class PairwiseLoss:
    """A pairwise ranking loss of the retrieval step: `kind` is its registry name."""

    kind: str = ""

    def get_config(self) -> dict:
        return {}

    def __repr__(self) -> str:
        args = ", ".join(f"{k}={v!r}" for k, v in self.get_config().items())
        return f"{type(self).__name__}({args})"

    def __eq__(self, other) -> bool:
        return type(other) is type(self) and other.get_config() == self.get_config()

    def __hash__(self) -> int:
        return hash((self.kind, tuple(sorted(self.get_config().items()))))


class BPRLoss(PairwiseLoss):
    """-log(sigmoid(s_p - s_n)) (Rendle et al., BPR)."""

    kind = "bpr"


class BPRmaxLoss(PairwiseLoss):
    """-log(sigmoid(s_p - s_n) softmax(s_neg)_n) + reg_lambda s_n^2 softmax(s_neg)_n (Hidasi & Karatzoglou, BPR-max)."""

    kind = "bpr-max"

    def __init__(self, reg_lambda: float = 1.0):
        self.reg_lambda = float(reg_lambda)

    def get_config(self) -> dict:
        return {"reg_lambda": self.reg_lambda}


class TOP1Loss(PairwiseLoss):
    """sigmoid(s_n - s_p) + sigmoid(s_n^2) (Hidasi et al., TOP1)."""

    kind = "top1"


class TOP1v2Loss(PairwiseLoss):
    """mean_n(sigmoid(s_n - s_p) + sigmoid(s_n^2)) - sigmoid(s_p^2) / N, one value per row (GRU4Rec's TOP1)."""

    kind = "top1_v2"


class TOP1maxLoss(PairwiseLoss):
    """(sigmoid(s_n - s_p) + sigmoid(s_n^2)) softmax(s_neg)_n (Hidasi & Karatzoglou, TOP1-max)."""

    kind = "top1-max"


class LogisticLoss(PairwiseLoss):
    """relu(s_n - s_p) + log1p(exp(-|s_n - s_p|))."""

    kind = "logistic"


class HingeLoss(PairwiseLoss):
    """relu(1 + s_n - s_p)."""

    kind = "hinge"


class CategoricalCrossentropy:
    """Keras CategoricalCrossentropy(from_logits, label_smoothing) as a loss of a CategoricalOutput model
    (CatalogModel.compile): the soft-max cross-entropy of the tempered logits against (1 - label_smoothing) onehot(y) +
    label_smoothing / N_I.  Only from_logits=True with label_smoothing in [0, 1) trains (CatalogModel refuses the rest);
    Keras' default is from_logits=False."""

    def __init__(self, from_logits: bool = False, label_smoothing: float = 0.0):
        self.from_logits = bool(from_logits)
        self.label_smoothing = float(label_smoothing)

    def get_config(self) -> dict:
        return {"from_logits": self.from_logits, "label_smoothing": self.label_smoothing}

    def __repr__(self) -> str:
        args = ", ".join(f"{k}={v!r}" for k, v in self.get_config().items())
        return f"{type(self).__name__}({args})"

    def __eq__(self, other) -> bool:
        return isinstance(other, CategoricalCrossentropy) and other.get_config() == self.get_config()

    def __hash__(self) -> int:
        return hash(tuple(sorted(self.get_config().items())))


class CategoricalCrossEntropy(CategoricalCrossentropy):
    """The reference's CategoricalCrossEntropy (losses/listwise.py): Keras' CategoricalCrossentropy with
    from_logits=True by default."""

    def __init__(self, from_logits: bool = True, label_smoothing: float = 0.0):
        super().__init__(from_logits=from_logits, label_smoothing=label_smoothing)


REGISTRY: Dict[str, Type[PairwiseLoss]] = {c.kind: c for c in (BPRLoss, BPRmaxLoss, TOP1Loss, TOP1v2Loss, TOP1maxLoss,
                                                                LogisticLoss, HingeLoss)}


def get(loss) -> Optional[PairwiseLoss]:
    """The pairwise loss `loss` names (a registry name or a PairwiseLoss), or None for the retrieval task's default
    in-batch soft-max cross-entropy (None or "categorical_crossentropy").  Anything else raises NotImplementedError."""
    if loss is None or (isinstance(loss, str) and loss == "categorical_crossentropy"):
        return None
    if isinstance(loss, PairwiseLoss):
        if loss.kind not in REGISTRY:
            raise NotImplementedError(f"loss {loss!r}: not a registered pairwise loss")
        return loss
    if isinstance(loss, str) and loss in REGISTRY:
        return REGISTRY[loss]()
    raise NotImplementedError(f"loss {loss!r} for a retrieval model: categorical_crossentropy or one of the pairwise losses "
                              f"{sorted(REGISTRY)} is implemented")
