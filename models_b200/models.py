"""Model factories behind the reference constructors: DLRMModel, DCNModel, TwoTowerModel.

Reference: merlin/models/tf/models/ranking.py:23-168, models/retrieval.py:106-203,
models/base.py:1805-1854 (Model.call protocol), outputs/classification.py:72-123 (BinaryOutput),
prediction_tasks/classification.py:59-116 (BinaryClassificationTask).  Construction, the forward call, compile / fit /
train_step (models_b200/train.py) and, for ranking models, evaluate and the compiled metrics (models_b200/metrics.py).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from .blocks import (FM, MLP, CategoryEncoding, CrossBlock, CrossBlockSeq, DLRM, DLRMBlock, FMBlock, MLPBlock, WideLinear, _Dense,
                     dense_engine, run_dense_chain, tower_kernel_applies)
from .core import Block, Prediction, TabularData, batch_size_of, default_device, to_device, unique_name
from .inputs import EmbeddingOptions, EmbeddingsBlock, InputBlockV2
from .retrieval import ItemRetrievalTask, QueryItemIdsEmbeddingsBlock, TwoTowerBlock
from .schema import Schema, Tags


class BinaryOutput(Block):
    """outputs/classification.py:72-123: Dense(1, activation="sigmoid") on the body output."""

    activation, loss, suffix = "sigmoid", "binary_crossentropy", "binary_output"

    def __init__(self, target: Optional[Union[str, object]] = None, name: Optional[str] = None, **kwargs):
        tname = getattr(target, "name", target)
        super().__init__(name or (f"{tname}/{self.suffix}" if tname else unique_name(self.suffix)))
        self.target = tname
        self.to_call = _Dense(1, activation=self.activation, name=f"{self.name}/dense")

    task_blocks = None  # {name: tower} when OutputBlock(task_blocks=...) gave this output a tower

    def build(self, width: Optional[int] = None, device=None):
        if self.task_blocks and width is not None:
            tower = self.task_blocks[self.name]
            tower.build_from_width(width, device)
            width = tower.dense_layers[-1].units
        self.to_call.build(width, device)
        self.built = True
        return self

    def weights(self):
        out = {f"dense/{k}": v for k, v in self.to_call.weights().items()}
        if self.task_blocks:
            out.update({f"task_block/{k}": v for k, v in self.task_blocks[self.name].weights().items()})
        return out

    def call(self, inputs: torch.Tensor, logits: bool = False, **kwargs) -> torch.Tensor:
        return self.to_call(inputs, activation="linear" if logits else None)


class BinaryClassificationTask(BinaryOutput):
    """prediction_tasks/classification.py:59-116 (v1): Dense(1, linear) followed by an fp32 sigmoid —
    the same function as BinaryOutput, fused in the layer epilogue here."""

    def __init__(self, target: Optional[str] = None, task_name: Optional[str] = None, **kwargs):
        super().__init__(target, name=task_name or (f"{target}/binary_classification_task" if target else None))


class RegressionOutput(BinaryOutput):
    """outputs/regression.py:35-58: Dense(1, activation="linear") on the body output, mean squared error."""

    activation, loss, suffix = "linear", "mse", "regression_output"


def _is_regression(out) -> bool:
    return isinstance(out, RegressionOutput)


class ParallelOutputs(Block):
    """The ParallelBlock of ModelOutputs that OutputBlock builds for several targets (outputs/block.py:32-131): outputs keyed
    by name ("<target>/binary_output", "<target>/regression_output"), in the order tf.nest flattens that dict (sorted by
    name).  Owns the stacked head `to_call` = Dense(K -> H) (kernel (K, H), bias (H,)) that the fused kernels read; each
    output's own Dense is only its initialiser.  The forward returns {name: (B, 1)}."""

    def __init__(self, outputs: Sequence[Block], name: Optional[str] = None):
        super().__init__(name or unique_name("parallel_outputs"))
        outs = list(outputs)
        for o in outs:
            if not isinstance(o, BinaryOutput):
                raise NotImplementedError(f"{getattr(o, 'name', o)!r}: only BinaryOutput / RegressionOutput heads can be combined")
        names = [o.name for o in outs]
        if len(set(names)) != len(names):
            raise ValueError(f"output names must be unique, got {names}")
        if not 2 <= len(outs) <= 8:
            raise NotImplementedError(f"2..8 outputs are supported, got {len(outs)}")
        self.outputs = sorted(outs, key=lambda o: o.name)
        self.to_call = _Dense(len(outs), activation="linear", name=f"{self.name}/dense")
        self.task_blocks: Optional[Dict[str, MLP]] = None  # {output name: tower} (OutputBlock(task_blocks=...))

    @property
    def names(self) -> List[str]:
        return [o.name for o in self.outputs]

    @property
    def losses(self) -> List[str]:
        return [o.loss for o in self.outputs]

    @property
    def activations(self) -> List[str]:
        return [o.activation for o in self.outputs]

    def build(self, width: Optional[int] = None, device=None):
        if self.task_blocks and width is not None and self.to_call.kernel is None:
            for o in self.outputs:
                self.task_blocks[o.name].build_from_width(width, device)
            width = self.task_blocks[self.outputs[0].name].dense_layers[-1].units
        if width is not None and width > 256:  # mm_heads_fwd_bwd / mm_mlp_tc_heads read the body vector from registers
            raise NotImplementedError(f"{self.name}: several outputs need a body output of at most 256 units, got {width}")
        if self.to_call.kernel is None:
            for o in self.outputs:
                o.build(width, device)
            self.to_call.build(width, device)
            self.to_call.kernel.copy_(torch.cat([o.to_call.kernel for o in self.outputs], dim=1))
            self.to_call.bias.copy_(torch.cat([o.to_call.bias for o in self.outputs]))
            for o in self.outputs:  # the stacked kernel is the one variable
                o.to_call.kernel = o.to_call.bias = None
        self.built = True
        return self

    def weights(self):
        """Each output's (K, 1) kernel and (1,) bias as a view of the stacked head: `<output name>/dense/{kernel,bias}`."""
        out = {}
        if self.to_call.kernel is None:
            return out
        for h, o in enumerate(self.outputs):
            out[f"{o.name}/dense/kernel"] = self.to_call.kernel[:, h:h + 1]
            out[f"{o.name}/dense/bias"] = self.to_call.bias[h:h + 1]
            if self.task_blocks:
                out.update({f"{o.name}/task_block/{k}": v for k, v in self.task_blocks[o.name].weights().items()})
        return out

    def split(self, stacked: torch.Tensor) -> Dict[str, torch.Tensor]:
        """(H, B) predictions -> {name: (B, 1) view}."""
        return {n: stacked[h].view(-1, 1) for h, n in enumerate(self.names)}

    def stacked_forward(self, x: torch.Tensor, out: torch.Tensor, logits: bool = False) -> torch.Tensor:
        """out (H, B) = the heads on the body output x by mm_heads_fwd_bwd (forward only): the activated predictions, or with
        logits=True the logits (every head run as a linear regression head)."""
        from .blocks import _LAST_HEADS

        _LAST_HEADS[0] = "heads"
        return ops.heads_fwd_bwd(x.contiguous(), self.to_call.kernel, self.to_call.bias,
                                 ["mse"] * len(self.outputs) if logits else self.losses, None, out)

    def call(self, inputs: torch.Tensor, logits: bool = False, **kwargs) -> Dict[str, torch.Tensor]:
        self.build(inputs.shape[1], inputs.device)
        out = torch.empty((len(self.outputs), inputs.shape[0]), dtype=torch.float32, device=inputs.device)
        return self.split(self.stacked_forward(inputs, out, logits=logits))


def OutputBlock(schema: Schema, model_outputs=None, task_blocks=None) -> Block:
    """outputs/block.py:32-131: one BinaryOutput / RegressionOutput per target column of the schema (continuous /
    regression-tagged targets first, then binary ones; a categorical target with int_domain.max == 1 is binary).  One target:
    that output itself; several: ParallelOutputs.  `model_outputs` (list or dict by name) replaces the outputs it names.
    `task_blocks` (outputs/block.py:133-190): one MLPBlock cloned for every output, or a dict keyed by output name or target
    column; output t then reads Dense(1)(task_block_t(body)).  The towers must end in the same width (the outputs' heads stay
    one stacked (K, H) Dense)."""
    targets = schema.select_by_tag(Tags.TARGET)
    if not len(targets):
        raise ValueError("No targets found in schema. Please tag your targets or provide them as branches.")
    given: Dict[str, Block] = {}
    if model_outputs is not None:
        if isinstance(model_outputs, dict):
            given = dict(model_outputs)
        elif isinstance(model_outputs, (list, tuple)):
            given = {m.name: m for m in model_outputs}
        elif isinstance(model_outputs, Block):
            given = {model_outputs.name: model_outputs}
        else:
            raise ValueError("If provided model_outputs should be either a dict or list of ModelOutput")
    outputs = dict(given)
    covered = {getattr(o, "target", None) for o in given.values()}
    for col in targets:
        if col.name in covered:  # a given output predicts this target, whatever its name
            continue
        if col.has_tag(Tags.CONTINUOUS) or col.has_tag(Tags.REGRESSION):
            cls = RegressionOutput
        elif col.has_tag(Tags.BINARY_CLASSIFICATION) or col.has_tag(Tags.BINARY):
            cls = BinaryOutput
        elif col.has_tag(Tags.CATEGORICAL) or col.has_tag(Tags.MULTI_CLASS_CLASSIFICATION):
            dom = col.int_domain
            if dom is None or dom.max != 1:
                raise NotImplementedError(f"target {col.name!r}: CategoricalOutput (multi-class training) is not implemented")
            cls = BinaryOutput
        else:
            raise ValueError(f"target {col.name!r}: tag it as regression, binary or categorical")
        name = f"{col.name}/{cls.suffix}"
        if name not in outputs:
            outputs[name] = cls(col.name)
    out = next(iter(outputs.values())) if len(outputs) == 1 else ParallelOutputs(list(outputs.values()))
    if task_blocks is not None:
        _attach_towers(out, task_blocks)
    return out


def _attach_towers(out: Block, task_blocks) -> None:
    """out.task_blocks = {output name: its tower} from task_blocks (a Layer cloned per output, or a dict by output name or
    target column)."""
    outs = out.outputs if isinstance(out, ParallelOutputs) else [out]
    towers = {}
    for o in outs:
        if isinstance(task_blocks, dict):
            blk = task_blocks.get(o.name, task_blocks.get(o.target))
            if blk is None:
                continue
        else:
            blk = task_blocks.copy()  # an independent copy per output
        if not isinstance(blk, MLP) or blk.has_normalization:
            raise NotImplementedError(f"task block of {o.name!r}: MLPBlock towers without normalization are implemented, got "
                                      f"{type(blk).__name__}")
        towers[o.name] = blk
    if isinstance(task_blocks, dict):
        unknown = sorted(set(task_blocks) - {o.name for o in outs} - {o.target for o in outs})
        if unknown:
            raise ValueError(f"task_blocks names unknown outputs / targets {unknown}")
    if towers and len(towers) != len(outs):
        raise NotImplementedError("OutputBlock(task_blocks=...): every output needs a tower (the heads read towers of one width)")
    widths = {t.dense_layers[-1].units for t in towers.values()}
    if len(widths) > 1:
        raise NotImplementedError(f"OutputBlock(task_blocks=...): the towers must end in the same width, got {sorted(widths)}")
    if widths and widths.pop() > 256:
        raise NotImplementedError("OutputBlock(task_blocks=...): a tower's last layer must be at most 256 wide")
    out.task_blocks = towers or None


def output_towers(prediction: Block) -> Optional[List[MLP]]:
    """The output towers of an output block in output order, or None."""
    towers = getattr(prediction, "task_blocks", None)
    if not towers:
        return None
    outs = prediction.outputs if isinstance(prediction, ParallelOutputs) else [prediction]
    return [towers[o.name] for o in outs]


def parse_prediction_blocks(schema: Schema, prediction_blocks=None) -> Block:
    """models/utils.py:12-31 / outputs/block.py:79-128: default = BinaryOutput for the (single)
    binary-classification target of the schema.  A schema with several binary targets, or several targets none of them
    binary, gets OutputBlock(schema).  A schema with exactly one binary target among several keeps that one BinaryOutput
    (the reference would build an output per target there)."""
    if prediction_blocks is None:
        targets = schema.select_by_tag(Tags.BINARY_CLASSIFICATION)
        if not len(targets):
            targets = schema.select_by_tag(Tags.TARGET)
        if not len(targets):
            raise ValueError("The schema has no target column: pass `prediction_tasks` explicitly")
        if len(targets) > 1:
            binary = [c.name for c in targets if c.has_tag(Tags.BINARY_CLASSIFICATION)]
            if len(binary) != 1:
                return OutputBlock(schema)
            return BinaryOutput(binary[0])
        return BinaryOutput(targets.first.name)
    for b in (prediction_blocks if isinstance(prediction_blocks, (list, tuple)) else [prediction_blocks]):
        if getattr(b, "task_blocks", None):
            raise NotImplementedError("per-task towers (OutputBlock(task_blocks=...)) are implemented for the sequential "
                                      "Model(InputBlockV2, ..., output) only")
    if isinstance(prediction_blocks, (list, tuple)):
        if len(prediction_blocks) > 1:
            return ParallelOutputs(prediction_blocks)
        if not prediction_blocks:
            raise ValueError("prediction_tasks is empty")
        prediction_blocks = prediction_blocks[0]
    if not isinstance(prediction_blocks, Block):
        raise ValueError(f"Unsupported prediction task {prediction_blocks!r}")
    return prediction_blocks


_LOSS_ALIASES = {"binary_crossentropy": "binary_crossentropy", "mse": "mse", "mean_squared_error": "mse",
                 "categorical_crossentropy": "categorical_crossentropy"}


def resolve_loss_weights(outputs: Sequence[Block], loss=None, loss_weights=None) -> List[float]:
    """Keras `compile(loss=..., loss_weights=...)` over the model's outputs: `loss` None (each output's default), one name
    valid for every output or a dict by output name; `loss_weights` a list in output order or a dict by output name
    (default 1).  Returns the loss weights in output order."""
    names = [o.name for o in outputs]
    if isinstance(loss, dict):
        unknown = sorted(set(loss) - set(names))
        if unknown:
            raise ValueError(f"loss names unknown outputs {unknown}; outputs are {names}")
        per = [loss.get(n) for n in names]
    else:
        per = [loss] * len(outputs)
    for o, l in zip(outputs, per):
        if l is None:
            continue
        if not isinstance(l, str) or _LOSS_ALIASES.get(l) != o.loss:
            raise NotImplementedError(f"loss {l!r} for output {o.name!r}: only its default ({o.loss!r}) is implemented")
    if loss_weights is None:
        return [1.0] * len(outputs)
    if isinstance(loss_weights, dict):
        unknown = sorted(set(loss_weights) - set(names))
        if unknown:
            raise ValueError(f"loss_weights names unknown outputs {unknown}; outputs are {names}")
        return [float(loss_weights.get(n, 1.0)) for n in names]
    lw = [float(v) for v in loss_weights]
    if len(lw) != len(outputs):
        raise ValueError(f"loss_weights has {len(lw)} entries for {len(outputs)} outputs")
    return lw


def expected_input_columns(schema: Schema) -> List[str]:
    """models/base.py:1730-1749: non-target columns; list columns as `__values` + `__offsets`.  Pretrained (EMBEDDING)
    columns are optional: an EmbeddingOperator serves them from the batch's lookup ids when the batch does not carry them."""
    cols = []
    for c in schema.excluding_by_tag(Tags.TARGET):
        if c.has_tag(Tags.EMBEDDING):
            continue
        if c.is_list and c.is_ragged:
            cols += [c.name + "__values", c.name + "__offsets"]
        else:
            cols.append(c.name)
    return cols


def _is_sequential(args, kwargs) -> bool:
    """Model(*blocks) (the reference's form) rather than Model(body, prediction, schema): no Schema argument and an
    InputBlockV2 first."""
    return (not kwargs and len(args) >= 2 and isinstance(args[0], InputBlockV2)
            and not any(isinstance(a, Schema) for a in args))


def _sequential_model(*blocks) -> "RankingModel":
    """Model(InputBlockV2, [MLPBlock], [MMOEBlock], output): the concatenating input block, optionally one MLPBlock as a
    shared bottom, optionally one MMOEBlock, then a BinaryOutput / RegressionOutput or the result of OutputBlock."""
    from .blocks import MLP
    from .experts import MMOEBlock

    from .retrieval import CategoricalOutput

    ib, mid, out = blocks[0], list(blocks[1:-1]), blocks[-1]
    order = "Model(*blocks) takes InputBlockV2, then optionally one MLPBlock, then optionally one MMOEBlock, then the output"
    if ib.aggregation != "concat":
        raise NotImplementedError("Model(*blocks): the input block must concatenate its features (aggregation='concat')")
    if isinstance(out, CategoricalOutput):
        return _catalog_model(ib, mid, out)
    if not isinstance(out, (BinaryOutput, ParallelOutputs)):
        raise NotImplementedError(f"{order} (BinaryOutput, RegressionOutput or OutputBlock(schema)); got {type(out).__name__} last")
    bottom = mmoe = None
    for blk in mid:
        if isinstance(blk, MLP) and bottom is None and mmoe is None:
            bottom = blk
        elif isinstance(blk, MMOEBlock) and mmoe is None:
            mmoe = blk
        else:
            raise NotImplementedError(f"{order}; got {[type(b).__name__ for b in blocks]}")
    if bottom is None and mmoe is None and not getattr(out, "task_blocks", None):
        raise NotImplementedError(f"{order}: an MLPBlock, an MMOEBlock or task towers are needed between the input and the output")
    if mmoe is not None:
        mmoe.bind(out.names if isinstance(out, ParallelOutputs) else [out.name])
    return RankingModel(MMoEBody(ib, bottom, mmoe), out, ib.schema)


def _catalog_model(ib: InputBlockV2, mid: list, out) -> "CatalogModel":
    """Model(InputBlockV2, MLPBlock, CategoricalOutput(to_call=EmbeddingTable)): the weight-tied next-item classifier
    (outputs/classification.py:127-216, :311-382).  The MLP's last width must be the table's width."""
    from .experts import MMOEBlock

    if any(isinstance(b, MMOEBlock) for b in mid) or getattr(out, "task_blocks", None):
        raise NotImplementedError("Model(*blocks): an MMOEBlock or task towers before a CategoricalOutput are not implemented")
    if len(mid) != 1 or not isinstance(mid[0], MLP):
        raise NotImplementedError("Model(*blocks) with a CategoricalOutput takes InputBlockV2, exactly one MLPBlock and the output; "
                                  f"got {[type(b).__name__ for b in [ib] + mid + [out]]}")
    mlp = mid[0]
    last, D = mlp.dense_layers[-1].units, out.table.dim
    if last != D:
        raise ValueError(f"the MLPBlock ends in {last} units but the CategoricalOutput's table {out.table.table_name!r} is "
                         f"{D} wide: the query must have the table's width")
    return CatalogModel(MMoEBody(ib, mlp, None), out, ib.schema)


class _ModelMeta(type):
    """`Model(*blocks)` (the reference's sequential form) builds through _sequential_model; every other call constructs the
    class as usual, so `Model(body, prediction, schema)` keeps its exact signature."""

    def __call__(cls, *args, **kwargs):
        if cls is Model and _is_sequential(args, kwargs):
            return _sequential_model(*args)
        return super().__call__(*args, **kwargs)


class Model(Block, metaclass=_ModelMeta):
    """models/base.py:1621-2245: model(inputs, targets=None, training=False, testing=False) with `inputs` a dict keyed by
    schema column names; `compile(optimizer)` / `fit` / `train_step` for the DLRM path (models_b200/train.py).

    `Model(body, prediction, schema)` wraps a body and its prediction block; `Model(InputBlockV2, *blocks)` (no schema
    argument) is the reference's sequential form and returns a RankingModel (_sequential_model)."""

    def __init__(self, body: Block, prediction: Block, schema: Schema):
        super().__init__(unique_name("model"))
        self.body = body
        self.prediction = prediction
        self.schema = schema
        self._pinned: Dict[str, torch.Tensor] = {}

    _TRANSIENT = {"_pinned": {}, "_trainer": None}

    @property
    def blocks(self) -> List[Block]:
        return [self.body, self.prediction]

    # -- checkpoint boundary (models_b200/io.py; reference: models/base.py:1687-1728) -----------
    def save(self, export_path, include_optimizer: bool = True, save_traces: bool = True) -> None:
        """Variables (Keras layouts, one .npy each), block structure and `.merlin` schema metadata.
        `include_optimizer` / `save_traces` are accepted for signature parity (forward path only)."""
        from . import io as _io

        _io.save_model(self, export_path)

    @classmethod
    def load(cls, export_path, device=None) -> "Model":
        from . import io as _io

        return _io.load_model(export_path, device)

    def load_weights(self, source, name_map=None, strict: bool = True):
        """Assign variables from an export directory or a {name: array} mapping (e.g. a Keras checkpoint
        exported as `{v.name: v.numpy()}`); see io.load_weights."""
        from . import io as _io

        return _io.load_weights(self, source, name_map=name_map, strict=strict)

    def state_dict(self) -> Dict[str, np.ndarray]:
        from . import io as _io

        return _io.state_dict(self)

    def output_schema(self) -> Schema:
        """One float column per prediction task (what `get_output_schema` records for the reference)."""
        from .schema import ColumnSchema

        if isinstance(self.prediction, ParallelOutputs):
            return Schema([ColumnSchema(n, dtype="float32") for n in self.prediction.names])
        target = getattr(self.prediction, "target", None) or getattr(self.prediction, "target_name", None)
        name = f"{target}/{self.prediction.name}" if target else self.prediction.name
        return Schema([ColumnSchema(name, dtype="float32")])

    def weights(self):
        out = {f"body/{k}": v for k, v in self.body.weights().items()}
        out.update({f"prediction/{k}": v for k, v in self.prediction.weights().items()})
        return out

    def _check_inputs(self, inputs: TabularData) -> None:
        if not isinstance(inputs, dict):
            raise ValueError(f"Model inputs must be a dict of features, got {type(inputs).__name__}")
        missing = [c for c in self.input_columns() if c not in inputs]
        if missing:
            raise ValueError(f"Missing input features: {missing}")

    def input_columns(self) -> List[str]:
        return expected_input_columns(self.schema)

    def id_bytes(self) -> Dict[str, int]:
        """Narrowest id width (1, 2 or 3 bytes) each scalar categorical input column can travel at from the
        host: its table has <= 2^8 / 2^16 / 2^24 rows.  `HostBatch.like(batch, names, id_bytes=...)` packs
        the pinned batch accordingly (the loader hand-off is PCIe-bound: a Criteo sample shrinks from 156 to
        104 bytes); the fused lookup kernel reads packed ids natively, other paths widen them on the device."""
        out: Dict[str, int] = {}
        for emb in self.embedding_blocks():
            for f, table in emb.feature_to_table.items():
                col = self.schema.get(f)
                if col is None or col.is_list:
                    continue
                rows = table.input_dim
                if rows <= (1 << 8):
                    out[f] = 1
                elif rows <= (1 << 16):
                    out[f] = 2
                elif rows <= (1 << 24):
                    out[f] = 3
        return out

    def call(self, inputs: TabularData, targets=None, training: bool = False, testing: bool = False, **kwargs):
        self._check_inputs(inputs)
        x = self.body(inputs, training=training, testing=testing)
        return self.prediction(x, features=inputs, targets=targets, training=training, testing=testing)

    # -- training (models_b200/train.py; reference: models/base.py:1121-1231) ------------------
    def output_blocks(self) -> List[Block]:
        """The model's outputs in output order (one for a single-output model)."""
        return list(self.prediction.outputs) if isinstance(self.prediction, ParallelOutputs) else [self.prediction]

    def _compile_training(self, optimizer, loss=None, loss_weights=None, metrics=None, weighted_metrics=None) -> None:
        from .train import get_optimizer

        self.loss_weights = resolve_loss_weights(self.output_blocks(), loss, loss_weights)
        self.optimizer = get_optimizer(optimizer)
        self._trainer = None

    def _targets_by_output(self, y) -> list:
        """Targets as given to train_step / evaluate (a tensor, or a dict keyed by target column) -> one per output."""
        outs = self.output_blocks()
        if y is None:
            raise ValueError("targets are needed")
        if isinstance(y, dict):
            if len(outs) == 1 and len(y) == 1:
                return [next(iter(y.values()))]
            missing = [o.target for o in outs if o.target not in y]
            if missing:
                raise ValueError(f"no targets for {missing} (got keys {sorted(y)})")
            return [y[o.target] for o in outs]
        if len(outs) > 1:
            raise ValueError(f"this model has {len(outs)} outputs: pass the targets as a dict keyed by target column")
        return [y]

    def trainer(self, batch_size: int, group=None):
        """The static-buffer training engine for batches of (up to) `batch_size` samples (train.trainer_for picks it by
        the body: DLRMTrainer, DCNTrainer or DeepFMTrainer)."""
        from .train import trainer_for

        if getattr(self, "optimizer", None) is None:
            raise RuntimeError("compile() the model with an optimizer before training it")
        tr = getattr(self, "_trainer", None)
        if tr is not None:
            if group is not None and tr.group is not group:
                raise ValueError("this model already trains with another process group")
            if tr.B < batch_size:
                raise NotImplementedError("the training batch size grew after the first step: create the engine for the largest "
                                          "batch first (model.trainer(batch_size) before the first train_step)")
            return tr
        tr = self._trainer = trainer_for(self, self.optimizer, batch_size, group=group)
        return tr

    def train_step(self, data) -> Dict[str, torch.Tensor]:
        """One optimizer step on `data` = (inputs, targets[, sample_weight]); returns the reference's step metrics
        {"loss", "loss_batch", "regularization_loss"} as device scalars (models/base.py:1121-1177).  The loss scalars are
        views of the engine's loss buffer: valid until the next step (clone to keep)."""
        if getattr(self, "optimizer", None) is None:
            raise RuntimeError("compile() the model with an optimizer before training it")
        if not isinstance(data, (tuple, list)) or len(data) < 2:
            raise ValueError("train_step expects (inputs, targets) or (inputs, targets, sample_weight)")
        x, y = data[0], data[1]
        sw = data[2] if len(data) > 2 else None
        outs = self.output_blocks()
        if y is None:
            raise ValueError("train_step needs targets")
        try:
            y = self._targets_by_output(y)
        except ValueError as e:
            raise ValueError(f"train_step: {e}") from None
        if isinstance(sw, dict):
            sw = [sw.get(o.name) for o in outs]
        self._check_inputs(x)
        tr = self.trainer(batch_size_of(x))
        loss = tr.step(x, y, sw)
        reg = getattr(tr, "regularization", None)  # the embeddings' L2 term, part of the total (NCF)
        out = {"loss": loss[0], "loss_batch": loss[0],
               "regularization_loss": torch.zeros((), device=loss.device) if reg is None else reg}
        if len(outs) > 1:
            out.update({f"{o.name}_loss": loss[1 + h] for h, o in enumerate(outs)})
        return out

    # train_step entries that fit does not average into the History besides "loss" (a ranking model's regularization_loss
    # is always 0)
    _fit_skip = ("loss", "loss_batch", "regularization_loss")

    def fit(self, x=None, y=None, batch_size: Optional[int] = None, epochs: int = 1, steps_per_epoch: Optional[int] = None,
            verbose: int = 0, **kwargs):
        """Keras `fit` over a models_b200.Loader (or any iterable of (inputs, targets)): returns a History-like object
        whose `.history["loss"]` holds the mean batch loss of every epoch."""
        if x is None:
            raise ValueError("fit needs a loader / iterable of (inputs, targets) batches")
        if y is not None:
            raise NotImplementedError("fit(x, y): pass a Loader or an iterable of (inputs, targets) batches")
        bs = batch_size or getattr(x, "batch_size", None)
        history = {"loss": []}
        train_metrics, every = self._fit_train_metrics(kwargs)
        for epoch in range(int(epochs)):
            total, n = None, 0
            if train_metrics is not None:
                train_metrics.reset()
            for inputs, targets in x:
                if getattr(self, "_trainer", None) is None and bs:
                    self._check_inputs(inputs)
                    self.trainer(int(bs))
                m = self.train_step((inputs, targets))
                if train_metrics is not None and n % every == 0:
                    self._update_train_metrics(train_metrics, targets)
                # the loss-buffer views are valid until the next step: [loss_batch, per-output losses...] summed on the device
                vec = torch.stack([m["loss_batch"]] + [v for k, v in m.items() if k not in self._fit_skip])
                total = vec.clone() if total is None else total + vec
                n += 1
                if steps_per_epoch and n >= steps_per_epoch:
                    break
            if n == 0:
                raise ValueError("fit: the loader produced no batches")
            means = (total / n).tolist()
            history["loss"].append(float(total[0].item()) / n)
            for i, k in enumerate([k for k in m if k not in self._fit_skip]):
                history.setdefault(k, []).append(means[1 + i])
            self._trainer.check_indices()
            self._fit_epoch_end(epoch, history, train_metrics, kwargs)
        from .train import History

        self.history = History(history)
        return self.history

    def _fit_train_metrics(self, fit_kwargs):
        """(state, every): the device state of the training metrics and the batch interval of their updates (None: off)."""
        return None, 0

    def _fit_epoch_end(self, epoch: int, history: Dict[str, List[float]], train_metrics, fit_kwargs) -> None:
        pass

    # -- CUDA-graph runtime (models_b200/graph.py) ---------------------------------------------
    def embedding_blocks(self) -> List[EmbeddingsBlock]:
        """Every EmbeddingsBlock of the model (they share one out-of-range index counter)."""
        found: List[EmbeddingsBlock] = []

        def walk(o, depth=0):
            if isinstance(o, EmbeddingsBlock):
                if o not in found:
                    found.append(o)
                return
            if depth > 6 or not isinstance(o, Block):
                return
            for v in vars(o).values():
                if isinstance(v, Block):
                    walk(v, depth + 1)
                elif isinstance(v, (list, tuple)):
                    for e in v:
                        walk(e, depth + 1)

        walk(self)
        return found

    def index_error_counter(self, device) -> Optional[torch.Tensor]:
        blocks = [b for b in self.embedding_blocks() if b.check_indices]
        if not blocks:
            return None
        c = blocks[0].counter(device)
        for b in blocks[1:]:
            b.oob_counter = c
        return c

    def defer_index_check(self, flag: bool) -> None:
        for b in self.embedding_blocks():
            b.defer_check = bool(flag)

    def compile(self, example: Union[Dict[str, np.ndarray], "HostBatch", str, None] = None, *, optimizer=None, loss=None,
                metrics=None, run_eagerly=None, **call_kwargs):
        """Two uses, told apart by the argument:

        * `compile(optimizer="adam")` / `compile("adagrad")` / `compile(optimizer=mm.Adagrad(0.01))` — Keras `compile`
          (models/base.py: the reference's models are compiled before `fit`): picks the optimizer of the training step
          (models_b200/train.py), or a MultiOptimizer of one optimizer per block (models_b200/optimizer.py).  The loss is the prediction task's default (binary cross-entropy for BinaryOutput).
          Ranking models take `metrics` / `weighted_metrics` (models_b200/metrics.py: None = each output's reference
          defaults) for `evaluate` and `fit`; `run_eagerly` is accepted for signature parity.
        * `compile(example_batch, **call_kwargs)` — capture this model's forward for `example`'s batch layout into a CUDA
          graph; the result maps a packed pinned HostBatch to pinned host predictions with one H2D, one graph launch and
          one D2H (models_b200/graph.py)."""
        from .graph import CompiledForward, HostBatch
        from .optimizer import MultiOptimizer
        from .train import Optimizer

        if optimizer is not None or isinstance(example, (str, Optimizer, MultiOptimizer)) or example is None:
            if example is not None and optimizer is not None:
                raise ValueError("compile(): pass either an example batch (graph capture) or an optimizer (training)")
            return self._compile_training(optimizer if optimizer is not None else (example or "adam"), loss,
                                          call_kwargs.pop("loss_weights", None), metrics, call_kwargs.pop("weighted_metrics", None))
        if not isinstance(example, HostBatch):
            example = HostBatch.like(example, self.input_columns())
        return CompiledForward(self, example, **call_kwargs)

    def pipeline(self, example: Union[Dict[str, np.ndarray], "HostBatch"], depth: int = 2, **call_kwargs) -> "PipelinedForward":
        """`depth` graph instances on separate streams so that the H2D copy of batch i+1 overlaps the
        forward of batch i (models_b200/graph.py)."""
        from .graph import HostBatch, PipelinedForward

        if not isinstance(example, HostBatch):
            example = HostBatch.like(example, self.input_columns())
        return PipelinedForward(self, example, depth=depth, **call_kwargs)

    # -- host-buffer entry point (the e2e path of bench.py) -----------------------------------
    def forward_host(self, batch: Dict[str, np.ndarray], stream: Optional[torch.cuda.Stream] = None, **kwargs):
        """Host numpy batch -> pinned staging -> H2D -> forward -> D2H of the predictions."""
        dev = default_device()
        dev_inputs = {}
        for k in self.input_columns():
            src = torch.from_numpy(np.ascontiguousarray(batch[k]))
            pin = self._pinned.get(k)
            if pin is None or pin.shape != src.shape or pin.dtype != src.dtype:
                pin = torch.empty(src.shape, dtype=src.dtype, pin_memory=True)
                self._pinned[k] = pin
            pin.copy_(src)
            dev_inputs[k] = pin.to(dev, non_blocking=True)
        out = self.call(dev_inputs, **kwargs)
        pred = out.outputs if isinstance(out, Prediction) else out
        return pred.cpu()


_EVAL_GRAPH = [True]  # evaluate replays full-size fixed-shape batches as a CUDA graph (tests switch it off for the eager path)


class RankingModel(Model):
    """DLRM / DCN / DeepFM: body -> (B, h) -> BinaryOutput (B,1) (or an OutputBlock's heads).  `evaluate` and
    `fit(validation_data=...)` report the compiled metrics (models_b200/metrics.py), accumulated on the device."""

    _TRANSIENT = {"_pinned": {}, "_trainer": None, "_eval_state": None, "_fit_state": None, "_eval_graph": None}

    @property
    def _fit_skip(self):
        # an NCF model's History records its regularization_loss, as matrix factorization's does
        return ("loss", "loss_batch") if isinstance(self.body, NCFBody) else Model._fit_skip

    def _eval_regularization(self, device) -> Optional[torch.Tensor]:
        """The device float the forward leaves the batch's embeddings L2 term in (None: the model has none)."""
        if isinstance(self.body, NCFBody) and self.body.embeddings_l2_reg:
            return self.body.regularization(device)
        return None

    def _eval_step(self, state, inputs: TabularData, targets, sample_weight) -> None:
        """One batch of evaluate: the logits forward and the metric update (with the batch's L2 term, if any)."""
        z, form = self.logits(inputs)
        state.update(z, targets, form, sample_weight, regularization=self._eval_regularization(z.device))

    def _distributed(self) -> bool:
        """Row-sharded tables or a data-parallel training engine: each rank sees only its share of the data."""
        return getattr(self.body, "sharded", None) is not None or getattr(getattr(self, "_trainer", None), "group", None) is not None

    def _compile_training(self, optimizer, loss=None, loss_weights=None, metrics=None, weighted_metrics=None) -> None:
        from .metrics import MetricsSpec

        super()._compile_training(optimizer, loss, loss_weights)
        self.metrics_spec = MetricsSpec(self.output_blocks(), self.loss_weights, metrics, weighted_metrics)
        self._eval_state = self._fit_state = None

    @property
    def metrics_names(self) -> List[str]:
        """The keys of `evaluate(return_dict=True)`, in the order of `evaluate`'s list."""
        return self._compiled_metrics().result_names()

    def _compiled_metrics(self):
        spec = getattr(self, "metrics_spec", None)
        if spec is None:
            raise RuntimeError("You must compile your model before training/testing. Use `model.compile(optimizer, loss)`.")
        return spec

    def _metrics_state(self, attr: str, device):
        from .metrics import MetricsState

        st = getattr(self, attr, None)
        if st is None or st.spec is not self.metrics_spec or st.device != device:
            st = MetricsState(self.metrics_spec, device)
            setattr(self, attr, st)
        st.reset()
        return st

    def predict(self, *args, **kwargs):
        raise NotImplementedError("predict is not implemented: call the model on a batch, or compile(example_batch) for a "
                                  "CUDA-graph forward")

    def evaluate(self, x, y=None, batch_size: Optional[int] = None, steps: Optional[int] = None, return_dict: bool = False,
                 verbose: int = 0, callbacks=None, **kwargs):
        """Keras `evaluate` (models/base.py:1176-1310) over a Loader or an iterable of (inputs, targets[, sample_weight])
        batches; targets a tensor or a dict keyed by target column, sample_weight a tensor or a dict by output name.  Each
        batch is the forward up to the logits (RankingModel.logits) plus one mm_metrics_update launch.  Batches of the first
        batch's size whose columns all have a fixed shape replay that step as one CUDA graph over static buffers
        (graph.EvalGraph); a smaller last batch and ragged features run eagerly.  Nothing is read back until the end: then
        one copy of the metric state and one read of the out-of-range id counter.  Returns the values in `metrics_names`
        order, or a dict with return_dict=True.  Variables, optimizer slots and captured training graphs are not touched."""
        from .graph import EvalGraph

        spec = self._compiled_metrics()
        if y is not None:
            raise NotImplementedError("evaluate(x, y): pass a Loader or an iterable of (inputs, targets[, sample_weight]) batches")
        if callbacks:
            raise NotImplementedError("evaluate(callbacks=...) is not implemented")
        if self._distributed():
            raise NotImplementedError("evaluate of a sharded or data-parallel model is not implemented (each rank would need "
                                      "the metric states of every other rank)")
        outs = self.output_blocks()
        for o in outs:
            if not isinstance(o, BinaryOutput):
                raise NotImplementedError(f"evaluate: output {o.name!r} is not a BinaryOutput / RegressionOutput")
        state, n, dev, oob, full = None, 0, None, None, None
        it = iter(x)
        self.defer_index_check(True)
        try:
            while steps is None or n < int(steps):
                try:
                    batch = next(it)
                except StopIteration:
                    break
                if not isinstance(batch, (tuple, list)) or len(batch) < 2:
                    raise ValueError("evaluate expects batches of (inputs, targets) or (inputs, targets, sample_weight)")
                inputs, targets = batch[0], batch[1]
                sw = batch[2] if len(batch) > 2 else None
                self._check_inputs(inputs)
                if state is None:
                    dev = next(iter(inputs.values())).device
                    state = self._metrics_state("_eval_state", dev)
                    oob = self.index_error_counter(dev)  # one counter shared by every table, read once at the end
                    full = batch_size_of(inputs)
                ys = [torch.as_tensor(t, device=dev) for t in self._targets_by_output(targets)]
                if isinstance(sw, dict):
                    sw = [sw.get(o.name) for o in outs]
                elif sw is not None and not isinstance(sw, (list, tuple)):
                    sw = [sw] * len(outs)
                key = EvalGraph.layout(inputs, ys, sw, dev) if _EVAL_GRAPH[0] and batch_size_of(inputs) == full else None
                if key is None:
                    self._eval_step(state, inputs, ys, sw)
                else:
                    g = getattr(self, "_eval_graph", None)
                    if g is None or g.key != key or g.state is not state:
                        g = self._eval_graph = None  # drop the old graph before capturing the new one
                        g = self._eval_graph = EvalGraph(self, state, inputs, ys, sw)
                    g.replay(inputs, ys, sw)
                n += 1
        finally:
            self.defer_index_check(False)
        if n == 0:
            raise ValueError("evaluate: the data produced no batches")
        res = state.result()
        if oob is not None:
            from .inputs import _raise_on_oob

            _raise_on_oob(oob, "evaluate")
        return res if return_dict else [res[k] for k in spec.result_names()]

    def fit(self, x=None, y=None, batch_size: Optional[int] = None, epochs: int = 1, steps_per_epoch: Optional[int] = None,
            verbose: int = 0, validation_data=None, validation_steps: Optional[int] = None, validation_freq=1,
            train_metrics_steps: int = 1, callbacks=None, **kwargs):
        """Model.fit plus the compiled metrics: on the training batches (from the step's logits, on the first batch and
        every `train_metrics_steps` batches of each epoch, 0: off) under their own names, and with `validation_data`
        `evaluate` after every epoch that `validation_freq` names (an interval, or a list of 1-based epochs) under
        `val_<name>`.  The metric launches happen between steps, outside the training step and its captured graph."""
        if callbacks:
            raise NotImplementedError("fit(callbacks=...) is not implemented")
        freqs = list(validation_freq) if isinstance(validation_freq, (list, tuple, set, range)) else [validation_freq]
        if any(int(f) < 1 for f in freqs):
            raise ValueError(f"validation_freq must be a positive interval or a list of positive epochs, got {validation_freq!r}")
        return super().fit(x, y, batch_size=batch_size, epochs=epochs, steps_per_epoch=steps_per_epoch, verbose=verbose,
                           validation_data=validation_data, validation_steps=validation_steps, validation_freq=validation_freq,
                           train_metrics_steps=train_metrics_steps, **kwargs)

    def _fit_train_metrics(self, fit_kwargs):
        every = int(fit_kwargs.get("train_metrics_steps", 1))
        if every < 0:
            raise ValueError("train_metrics_steps must be >= 0")
        # with sharded tables or a data-parallel engine each rank would report its own, unaveraged metrics: off
        if (every == 0 or getattr(self, "metrics_spec", None) is None or not self._compiled_metrics().metric_keys()
                or self._distributed()):
            return None, 0
        return self._metrics_state("_fit_state", default_device()), every

    def _update_train_metrics(self, state, targets) -> None:
        from ._cabi import PRED_HEAD

        tr = self._trainer
        ys = [t if isinstance(t, torch.Tensor) and t.device == state.device else torch.as_tensor(t, device=state.device)
              for t in self._targets_by_output(targets)]
        b = ys[0].numel()
        state.update(tr.logits.view(-1)[:tr.H * b].view(tr.H, b), ys, PRED_HEAD)

    def _fit_epoch_end(self, epoch: int, history, train_metrics, fit_kwargs) -> None:
        if train_metrics is not None:
            res = train_metrics.result()
            for k in self.metrics_spec.metric_keys():
                history.setdefault(k, []).append(res[k])
        data = fit_kwargs.get("validation_data")
        if data is None:
            return
        freq = fit_kwargs.get("validation_freq", 1)
        due = (epoch + 1) in freq if isinstance(freq, (list, tuple, set, range)) else (epoch + 1) % int(freq) == 0
        if due:
            res = self.evaluate(data, steps=fit_kwargs.get("validation_steps"), return_dict=True)
            for k, v in res.items():
                history.setdefault(f"val_{k}", []).append(v)

    def build(self, device=None):
        self.body.build(device)
        self.prediction.build(self.body_width(), device)
        self.built = True
        return self

    def _all_onehot(self, inputs: TabularData) -> bool:
        from .core import get_feature

        emb = self.body.embeddings
        return all(emb.feature_to_table[f].lookup_kind(get_feature(inputs, f)) == "onehot" for f in emb.feature_names)

    def body_width(self) -> int:
        if isinstance(self.body, DLRM):
            if self.body.top_block is not None:
                return self.body.top_block.dense_layers[-1].units
            return self.body.output_width_before_top()
        return self.body.output_width()

    def call(self, inputs: TabularData, targets=None, training: bool = False, testing: bool = False, **kwargs):
        return self._forward(inputs, training=training)

    def logits(self, inputs: TabularData):
        """The forward of `call` stopped before the output activation: (z, pred_form) with z the (H, B) logits of the H
        outputs (output order) and pred_form the _cabi.PRED_* form in which that forward applies the sigmoid (the
        multi-head kernel mm_heads_fwd_bwd has its own), so that a metric recomputing sigmoid(z) gets `call`'s
        predictions bit for bit."""
        from ._cabi import PRED_ACT, PRED_HEAD
        from .blocks import _LAST_HEADS

        _LAST_HEADS[0] = "none"
        out = self._forward(inputs, logits=True)
        if isinstance(out, dict):
            from .graph import _stacked_outputs

            return _stacked_outputs(out), PRED_HEAD if _LAST_HEADS[0] == "heads" else PRED_ACT
        return out.reshape(1, -1), PRED_HEAD if _LAST_HEADS[0] == "heads" else PRED_ACT

    def _forward(self, inputs: TabularData, training: bool = False, logits: bool = False):
        self._check_inputs(inputs)
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        heads = self.prediction if isinstance(self.prediction, ParallelOutputs) else None
        extra = [] if heads is not None else [self.prediction.to_call]
        if heads is not None and not self.prediction.built:
            self.prediction.build(self.body_width(), next(iter(inputs.values())).device)

        def chain(x, layers, **kw):
            if heads is None:
                return run_dense_chain(x, layers, logits=logits, **kw)
            return heads.split(run_dense_chain(x, layers, heads=heads, logits=logits, **kw))

        if isinstance(self.body, DLRM) and self.body.top_block is not None:
            # top MLP + output layer as ONE dense chain (no fp32 round trip between them)
            # top MLP (+ its normalizations, folded) + the output Dense as one chain
            layers, tail = self.body.top_block.chain(extra)
            assert tail is None
            if dense_engine() != "fp32" and self.body.can_emit_split():
                # production path: bottom vector and table rows in the interaction kernel's operand format when the
                # mirrors are on (no bf16 split inside the hot loop); split-bf16 row straight into the top tower
                op = self.body.use_operand_rows() and self._all_onehot(inputs)
                K = self.body.output_width_before_top()
                bottom = self.body.bottom_forward(inputs, operand_out=op)
                # the whole-tower kernel reads the bottom vector from the bottom tower's own rows: the interaction
                # kernel then writes the pairs alone (the row sharded tables feed keeps [bottom | pairs])
                pairs = op and self.body.sharded is None and tower_kernel_applies(layers, K, heads)
                a = self.body.interaction_forward(inputs, bottom, as_split=True, operand_rows=op, pairs_only=pairs)
                return chain(None, layers, a_split=a, K=K, a_bottom=bottom if pairs else None)
            bottom = self.body.bottom_forward(inputs)
            x = self.body.interaction_forward(inputs, bottom)
            return chain(x, layers)
        if isinstance(self.body, DeepFMBody):
            return self.body.forward(inputs, out_layer=self.prediction.to_call, logits=logits)
        if isinstance(self.body, WideAndDeepBody):
            return self.body.forward(inputs, out_layer=self.prediction.to_call, logits=logits)
        if isinstance(self.body, NCFBody):
            out = self.body.forward(inputs, self.output_blocks(), self.prediction.to_call, logits=logits)
            return heads.split(out) if heads is not None else out.view(-1, 1)
        if isinstance(self.body, MMoEBody) and (self.body.mmoe is not None or output_towers(self.prediction)):
            out = self.body.forward(inputs, self.output_blocks(), self.prediction.to_call, output_towers(self.prediction),
                                    logits=logits)
            return heads.split(out) if heads is not None else out.view(-1, 1)
        if isinstance(self.body, MMoEBody):
            x = self.body.input_block(inputs)
            layers, tail = self.body.bottom.chain(extra)
            assert tail is None
            return chain(x, layers)
        if isinstance(self.body, DCNBody) and self.body.stacked:
            x = self.body.cross(self.body.input_block(inputs))
            layers, tail = self.body.deep.chain(extra)
            assert tail is None
            return chain(x, layers)
        x = self.body(inputs, training=training)
        return self.prediction(x, logits=True) if logits else self.prediction(x)


class CatalogModel(Model):
    """Model(InputBlockV2, MLPBlock, CategoricalOutput(to_call=EmbeddingTable)): the reference's weight-tied next-item
    classifier.  The input block and the MLP make the query x (B, D); the output scores it against the item table E
    (N_I, D) that an input feature may also read.  Calling the model returns CategoricalOutput's (B, N_I) logits without
    the temperature; `top_k` streams the table without them.  `compile` / `fit` / `train_step` train it with
    CategoricalCrossentropy(from_logits=True), optionally label-smoothed (losses.CategoricalCrossEntropy(label_smoothing=
    eps)), on the tempered logits (train.CatalogTrainer); `evaluate` reports that loss
    and top-k metrics of the label among the whole table (default_categorical_prediction_metrics(k=10))."""

    _TRANSIENT = {"_pinned": {}, "_trainer": None}

    @property
    def mlp(self) -> MLP:
        return self.body.bottom

    def build(self, device=None):
        self.body.build(device)
        self.prediction.build(device)
        self.built = True
        return self

    def query(self, inputs: TabularData) -> torch.Tensor:
        """(B, D): the MLP's output, what the output layer scores against the table."""
        self._check_inputs(inputs)
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        return run_dense_chain(self.body.input_block(inputs), self.mlp.dense_layers)

    def call(self, inputs: TabularData, targets=None, training: bool = False, testing: bool = False, **kwargs):
        return self.prediction(self.query(inputs))

    def top_k(self, inputs: TabularData, k: int):
        """(scores, ids) (B, k) of the whole table, in tf.math.top_k order."""
        return self.prediction.top_k(self.query(inputs), k)

    def _compile_training(self, optimizer, loss=None, loss_weights=None, metrics=None, weighted_metrics=None) -> None:
        from .losses import CategoricalCrossentropy
        from .topk import TopKMetric, _FUSED_MAX_K

        if isinstance(loss, CategoricalCrossentropy):
            if not loss.from_logits:
                raise NotImplementedError(f"loss {loss!r}: a CategoricalOutput trains on its logits (from_logits=True)")
            if not 0.0 <= loss.label_smoothing < 1.0:
                raise NotImplementedError(f"loss {loss!r}: label_smoothing in [0, 1) is implemented")
            label_smoothing = loss.label_smoothing
        elif isinstance(loss, str) and loss in ("categorical_crossentropy", "CategoricalCrossentropy") or loss is None:
            label_smoothing = 0.0
        else:
            raise NotImplementedError(f"loss {loss!r}: a CategoricalOutput trains with its default, categorical_crossentropy, "
                                      "or CategoricalCrossEntropy(from_logits=True, label_smoothing=...)")
        if loss_weights is not None or weighted_metrics:
            raise NotImplementedError("loss_weights / weighted_metrics: a CategoricalOutput model has one output and unweighted "
                                      "top-k metrics")
        metrics = list(metrics) if metrics else default_categorical_metrics()
        for m in metrics:
            if not isinstance(m, TopKMetric):
                raise NotImplementedError(f"metric {m!r}: a CategoricalOutput model evaluates top-k metrics (RecallAt, MRRAt, "
                                          "NDCGAt, AvgPrecisionAt, PrecisionAt)")
            if not 1 <= m.k <= _FUSED_MAX_K:
                raise ValueError(f"{m.label}: k must be in [1, {_FUSED_MAX_K}] (the fused top-k's limit)")
        super()._compile_training(optimizer, None, None)
        self.topk_metrics = metrics
        self.label_smoothing = label_smoothing

    @property
    def metrics_names(self) -> List[str]:
        return ["loss"] + [m.label for m in self._compiled_topk()]

    def _compiled_topk(self):
        metrics = getattr(self, "topk_metrics", None)
        if metrics is None:
            raise RuntimeError("You must compile your model before training/testing. Use `model.compile(optimizer, loss)`.")
        return metrics

    def evaluate(self, x, y=None, batch_size: Optional[int] = None, steps: Optional[int] = None, return_dict: bool = False,
                 verbose: int = 0, callbacks=None, **kwargs):
        """Keras `evaluate` over an iterable of (inputs, targets[, sample_weight]) batches (targets: the class ids, or a
        dict holding them under `target_name`): `loss` is the catalog soft-max cross-entropy of the tempered logits (as in
        testing mode), weighted by sample_weight and averaged over the rows; each top-k metric has the label as the one
        relevant item among the top k of the whole table.  One mm_catalog_score pass per batch gives both (no (B, N_I)
        logits); with the compiled loss' label_smoothing eps the loss is against the smoothed target, whose uniform part
        takes the rows' mean logit from mm_catalog_mean_logit.  Returns the values in `metrics_names` order, or a dict with return_dict=True.  A label outside [0, N_I)
        is counted on the device and raises IndexError at the end."""
        from .topk import evaluate_topk

        metrics = self._compiled_topk()
        if y is not None:
            raise NotImplementedError("evaluate(x, y): pass an iterable of (inputs, targets[, sample_weight]) batches")
        if callbacks:
            raise NotImplementedError("evaluate(callbacks=...) is not implemented")
        out, N = self.prediction, self.prediction.num_classes
        eps = float(getattr(self, "label_smoothing", 0.0))
        kmax = max(m.k for m in metrics)
        acc = {"loss": None, "rows": 0, "bad": None}

        def batches():
            for n, batch in enumerate(x):
                if steps is not None and n >= int(steps):
                    return
                if not isinstance(batch, (tuple, list)) or len(batch) < 2:
                    raise ValueError("evaluate expects batches of (inputs, targets) or (inputs, targets, sample_weight)")
                yield batch

        def predict(batch):
            inputs, targets = batch[0], batch[1]
            dev = next(iter(inputs.values())).device
            yv = torch.as_tensor(self._targets_by_output(targets)[0], device=dev).reshape(-1)
            if yv.dtype not in (torch.int32, torch.int64):
                raise ValueError(f"targets must be int32 / int64 class ids, got {yv.dtype}")
            bad = ((yv < 0) | (yv >= N)).sum()
            acc["bad"] = bad if acc["bad"] is None else acc["bad"] + bad
            # one pass over the table: the statistics of the tempered logits and their top-k (T > 0 keeps the order)
            xt, bt = out._tempered(self.query(inputs))
            stats, _, ids = ops.catalog_score(xt, out._catalog_split(), N, bias=bt, targets=yv, k=kmax)
            # an out-of-range label's target logit is NaN: counted above, raised below
            if eps:  # the smoothed target: lse - (1 - eps) z[y] - eps mean_j z[j]
                mean = ops.catalog_mean_logit(ops.split_rows(xt), out._catalog_split(), xt.shape[1], bias=bt)
                per = stats[:, 1] - (1.0 - eps) * stats[:, 2] - eps * mean
            else:
                per = stats[:, 1] - stats[:, 2]
            if len(batch) > 2 and batch[2] is not None:
                sw = batch[2][out.name] if isinstance(batch[2], dict) else batch[2]
                per = per * torch.as_tensor(sw, device=dev, dtype=torch.float32).reshape(-1)
            acc["loss"] = per.sum() if acc["loss"] is None else acc["loss"] + per.sum()
            acc["rows"] += yv.numel()
            return Prediction(None, (ids == yv.view(-1, 1).to(ids.dtype)).to(torch.float32),
                              label_relevant_counts=torch.ones(yv.numel(), device=dev))

        res = evaluate_topk(predict, batches(), metrics)
        bad = int(acc["bad"].item())
        if bad:
            raise IndexError(f"evaluate: {bad} labels out of range for the {N} classes of {out.table.table_name!r}")
        res = {"loss": float(acc["loss"].item()) / acc["rows"], **res}
        return res if return_dict else [res[k] for k in self.metrics_names]

    def _fit_epoch_end(self, epoch: int, history, train_metrics, fit_kwargs) -> None:
        data = fit_kwargs.get("validation_data")
        if data is None:
            return
        freq = fit_kwargs.get("validation_freq", 1)
        due = (epoch + 1) in freq if isinstance(freq, (list, tuple, set, range)) else (epoch + 1) % int(freq) == 0
        if due:
            res = self.evaluate(data, steps=fit_kwargs.get("validation_steps"), return_dict=True)
            for k, v in res.items():
                history.setdefault(f"val_{k}", []).append(v)


def default_categorical_metrics(k: int = 10) -> list:
    """metrics/topk.py default_categorical_prediction_metrics(k=10): RecallAt, MRRAt, NDCGAt, AvgPrecisionAt, PrecisionAt."""
    from .topk import AvgPrecisionAt, MRRAt, NDCGAt, PrecisionAt, RecallAt

    return [RecallAt(k), MRRAt(k), NDCGAt(k), AvgPrecisionAt(k), PrecisionAt(k)]


class MMoEBody(Block):
    """The body of Model(InputBlockV2, [MLPBlock], [MMOEBlock], output): input block -> shared bottom -> experts and gates.
    Without an MMOEBlock the output heads read the bottom's output as in the other ranking models; with one, the gates,
    the mixture and the heads are one kernel (ops.mmoe_heads_fwd_bwd) after the stacked expert and gate layers."""

    def __init__(self, input_block: InputBlockV2, bottom: Optional[MLP], mmoe):
        super().__init__(unique_name("mmoe_body"))
        self.input_block, self.bottom, self.mmoe = input_block, bottom, mmoe
        if bottom is not None and bottom.has_normalization and mmoe is not None:
            raise NotImplementedError("Model(*blocks): normalization in the shared bottom before an MMOEBlock is not implemented")

    def input_width(self) -> int:
        """Width of what the experts and gates (or the heads) read."""
        return self.bottom.dense_layers[-1].units if self.bottom is not None else self.input_block.layout()[2]

    def build(self, device=None):
        self.input_block.build(device)
        _, _, d = self.input_block.layout()
        if self.bottom is not None:
            self.bottom.build_from_width(d, device)
        if self.mmoe is not None:
            self.mmoe.build(self.input_width(), device)
        self.built = True
        return self

    def output_width(self) -> int:
        return self.mmoe.units if self.mmoe is not None else self.input_width()

    def weights(self):
        out = {f"input/{k}": v for k, v in self.input_block.weights().items()}
        if self.bottom is not None:
            out.update({f"bottom/{k}": v for k, v in self.bottom.weights().items()})
        if self.mmoe is not None:
            out.update({f"mmoe/{k}": v for k, v in self.mmoe.weights().items()})
        return out

    def forward(self, inputs: TabularData, outputs: Sequence[Block], head: _Dense, towers: Optional[List[MLP]],
                logits: bool = False) -> torch.Tensor:
        """(H, B): the activated predictions of the outputs, or their logits with logits=True (each head run as a linear
        regression head, as ParallelOutputs.stacked_forward does).  Without towers the gates, the mixture and the heads are
        mm_mmoe_heads_fwd_bwd; with towers mm_mmoe_mix_fwd, one tower chain per output and mm_mmoe_task_heads_fwd_bwd."""
        from .blocks import _LAST_HEADS

        if not self.built:
            self.build(next(iter(inputs.values())).device)
        mo = self.mmoe
        x = self.input_block(inputs)
        if self.bottom is not None:
            x = run_dense_chain(x, self.bottom.dense_layers)
        B, K = x.shape
        H = len(outputs)
        dev = x.device
        out = torch.empty((H, B), dtype=torch.float32, device=dev)
        losses = ["mse"] * H if logits else [o.loss for o in outputs]
        _LAST_HEADS[0] = "heads"
        if mo is None:  # towers on the shared vector
            ts = [run_dense_chain(x, t.dense_layers) for t in towers]
            return ops.mmoe_task_heads_fwd_bwd(ts, head.kernel, head.bias, losses, None, out)
        xs = ops.split_rows(x)
        X = torch.empty((B, mo.experts.units), dtype=torch.float32, device=dev)
        ops.dense_tc(xs, K, mo.experts.split_kernel(), mo.experts.units, mo.experts.bias, mo.experts.activation, out_f32=X)
        if mo.gates is not None:
            L = torch.empty((B, mo.gates.units), dtype=torch.float32, device=dev)
            ops.dense_tc(xs, K, mo.gates.split_kernel(), mo.gates.units, None, "linear", out_f32=L)
            gl = mo.gate_logits(L)
        else:
            gl = [run_dense_chain(x, mo.gate_chain(t)) for t in range(H)]
        if towers is None:
            return ops.mmoe_heads_fwd_bwd(X, mo.num_experts, gl, mo.temperature, head.kernel, head.bias, losses, None, out)
        U = mo.units
        m = torch.empty((H, B, U), dtype=torch.float32, device=dev)
        m_split = torch.empty((H, B, 2 * ops.tc_padded_k(U)), dtype=torch.bfloat16, device=dev)
        p = torch.empty((B, H * mo.num_experts), dtype=torch.float32, device=dev)
        ops.mmoe_mix_fwd(X, mo.num_experts, gl, mo.temperature, p, m, m_split)
        ts = [run_dense_chain(None, t.dense_layers, a_split=m_split[i], K=U) for i, t in enumerate(towers)]
        return ops.mmoe_task_heads_fwd_bwd(ts, head.kernel, head.bias, losses, None, out)

    def call(self, inputs: TabularData, **kwargs):
        raise NotImplementedError("MMoEBody runs inside its RankingModel (the output heads are fused with the mixture)")


def DLRMModel(schema: Schema, *, embeddings: Optional[EmbeddingsBlock] = None, embedding_dim: Optional[int] = None,
              embedding_options: Optional[EmbeddingOptions] = None, bottom_block: Optional[MLP] = None,
              top_block: Optional[MLP] = None, prediction_tasks=None) -> RankingModel:
    """models/ranking.py:23-92."""
    prediction = parse_prediction_blocks(schema, prediction_tasks)
    body = DLRMBlock(schema, embedding_dim=embedding_dim, embedding_options=embedding_options, embeddings=embeddings,
                     bottom_block=bottom_block, top_block=top_block)
    return RankingModel(body, prediction, schema)


class DCNBody(Block):
    """input_block.connect(CrossBlock(depth), deep_block) (stacked) or connect_branch(..., "concat")."""

    def __init__(self, input_block: InputBlockV2, cross: CrossBlockSeq, deep: MLP, stacked: bool):
        super().__init__(unique_name("dcn_body"))
        self.input_block, self.cross, self.deep, self.stacked = input_block, cross, deep, stacked

    def build(self, device=None):
        self.input_block.build(device)
        _, _, d = self.input_block.layout()
        for l in self.cross.cross_layers:
            l.build(d, device)
        self.deep.build_from_width(d, device)
        self.built = True
        return self

    def output_width(self) -> int:
        _, _, d = self.input_block.layout()
        last = self.deep.dense_layers[-1].units
        return last if self.stacked else d + last

    def weights(self):
        out = {f"input/{k}": v for k, v in self.input_block.weights().items()}
        for l in self.cross.cross_layers:
            out.update({f"{l.name}/{k}": v for k, v in l.weights().items()})
        out.update({f"deep/{k}": v for k, v in self.deep.weights().items()})
        return out

    def call(self, inputs: TabularData, **kwargs):
        x0 = self.input_block(inputs)
        c = self.cross(x0)
        if self.stacked:
            return self.deep(c)
        d = self.deep(x0)
        out = torch.empty((x0.shape[0], c.shape[1] + d.shape[1]), dtype=torch.float32, device=x0.device)
        return ops.concat_columns([c, d] if self.branch_order() == ("cross", "deep") else [d, c], out)

    def branch_order(self):
        """Column order of the non-stacked concat.  The reference's `connect_branch(CrossBlock(depth), deep_block,
        aggregation="concat")` builds a ParallelBlock keyed by the two layers' auto names and ConcatFeatures sorts the
        keys (core/combinators.py, core/aggregation.py:54-66): both are `sequential_block[_N]`, the deep block is created
        first, so the order is normally [deep | cross] — by STRING comparison of the names (`..._10` < `..._9`).  The same
        rule is applied to this package's Keras-style names; set `body.concat_order = ("cross", "deep")` (or the reverse)
        to pin the layout of an imported checkpoint's output kernel explicitly."""
        forced = getattr(self, "concat_order", None)
        if forced is not None:
            if tuple(forced) not in (("cross", "deep"), ("deep", "cross")):
                raise ValueError("concat_order must be ('cross', 'deep') or ('deep', 'cross')")
            return tuple(forced)
        return ("cross", "deep") if self.cross.name < self.deep.name else ("deep", "cross")


class DeepFMBody(Block):
    """ParallelBlock({"fm": FMBlock, "deep": input_block -> deep_block -> deep_logit_block}, "element-wise-sum")
    (models/ranking.py:250-274): (B, 1).  The deep tower is the usual concat + dense chain; the FM pairwise term, the wide
    part, the sum with the deep logit and (from RankingModel) the output layer are ONE kernel (ops.deepfm_head)."""

    def __init__(self, input_block: InputBlockV2, fm: FM, deep: MLP, deep_logit: MLP):
        super().__init__(unique_name("deepfm_body"))
        self.input_block, self.fm, self.deep, self.deep_logit = input_block, fm, deep, deep_logit
        if deep.has_normalization or deep_logit.has_normalization:
            raise NotImplementedError("DeepFMModel: normalization inside deep_block / deep_logit_block is not implemented")
        if deep_logit.dense_layers[-1].units != 1:
            raise ValueError("The last dimension of deep_logit_block needs to be 1")

    def build(self, device=None):
        self.input_block.build(device)
        _, _, d = self.input_block.layout()
        self.deep.build_from_width(d, device)
        self.deep_logit.build_from_width(self.deep.dense_layers[-1].units, device)
        self.fm.build(device)
        self.built = True
        return self

    def output_width(self) -> int:
        return 1

    def weights(self):
        out = {f"input/{k}": v for k, v in self.input_block.weights().items()}
        out.update({f"fm/{k}": v for k, v in self.fm.weights().items()})
        out.update({f"deep/{k}": v for k, v in self.deep.weights().items()})
        out.update({f"deep_logit/{k}": v for k, v in self.deep_logit.weights().items()})
        return out

    def forward(self, inputs: TabularData, out_layer: Optional[_Dense] = None, logits: bool = False) -> torch.Tensor:
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        x0 = self.input_block(inputs)
        deep = run_dense_chain(x0, self.deep.dense_layers + self.deep_logit.dense_layers)
        return self.fm.head(inputs, addend=deep, out_layer=out_layer, logits=logits)

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        return self.forward(inputs)


def DeepFMModel(schema: Schema, embedding_dim: Optional[int] = None, deep_block: Optional[MLP] = None,
                input_block: Optional[InputBlockV2] = None, wide_input_block=None, wide_logit_block=None,
                deep_logit_block: Optional[MLP] = None, prediction_tasks=None, **kwargs) -> RankingModel:
    """models/ranking.py:171-279: sigmoid(Dense(1)(FM(x) + deep(x))) with FM = wide + pairwise (blocks.FM), deep =
    MLP over the concatenated embeddings and continuous features followed by MLPBlock([1], linear).  Defaults as the
    reference: deep_block = MLPBlock([64]); one embedding dimension for every categorical feature (`embedding_dim`)."""
    if input_block is None:
        if embedding_dim is None:
            raise ValueError("DeepFMModel needs `embedding_dim` (the FM term stacks the embeddings: one dimension for all tables)")
        from .inputs import Embeddings

        cat = schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)
        input_block = InputBlockV2(schema, categorical=Embeddings(cat, dim=embedding_dim), **kwargs)
    fm = FMBlock(schema, fm_input_block=input_block, wide_input_block=wide_input_block, wide_logit_block=wide_logit_block)
    deep_block = deep_block if deep_block is not None else MLPBlock([64])
    deep_logit_block = deep_logit_block if deep_logit_block is not None else MLPBlock([1], activation="linear", use_bias=True)
    prediction = parse_prediction_blocks(schema, prediction_tasks)
    if isinstance(prediction, ParallelOutputs):
        raise NotImplementedError("DeepFMModel with several outputs is not implemented: pass one BinaryOutput")
    return RankingModel(DeepFMBody(input_block, fm, deep_block, deep_logit_block), prediction, schema)


class WideAndDeepBody(Block):
    """ParallelBlock({"deep": input_block -> deep_block -> MLPBlock([1]), "wide": CategoryEncoding -> Dense(1)},
    "element-wise-sum") (models/ranking.py:504-570): (B, 1).  The deep tower's hidden layers are the usual dense chain;
    the deep logit's Dense(1), the wide Dense(1) over the encoded wide features, the sum and (from RankingModel) the output
    layer are ONE kernel (ops.wide_deep_head_fwd_bwd).  Either branch may be absent (input_block / wide None)."""

    def __init__(self, input_block: Optional[InputBlockV2], deep: Optional[MLP], deep_logit: Optional[MLP], wide: Optional[WideLinear],
                 regularized: bool = False):
        super().__init__(unique_name("wide_and_deep_body"))
        self.input_block, self.deep, self.deep_logit, self.wide = input_block, deep, deep_logit, wide
        self.regularized = regularized  # a deep / wide regularizer was given (it only changes training)
        if deep is not None:
            if deep.has_normalization:
                raise NotImplementedError("WideAndDeepModel: normalization inside deep_block is not implemented")
            if deep.dense_layers[-1].units > 512:
                raise NotImplementedError(f"WideAndDeepModel: the head kernel reads at most 512 units of the deep block's last "
                                          f"layer, got {deep.dense_layers[-1].units}")

    def build(self, device=None):
        if self.input_block is not None:
            self.input_block.build(device)
            _, _, d = self.input_block.layout()
            self.deep.build_from_width(d, device)
            self.deep_logit.build_from_width(self.deep.dense_layers[-1].units, device)
        if self.wide is not None:
            self.wide.build(device)
        self.built = True
        return self

    def output_width(self) -> int:
        return 1

    def weights(self):
        out = {}
        if self.input_block is not None:
            out.update({f"input/{k}": v for k, v in self.input_block.weights().items()})
            out.update({f"deep/{k}": v for k, v in self.deep.weights().items()})
            out.update({f"deep_logit/{k}": v for k, v in self.deep_logit.weights().items()})
        if self.wide is not None:
            out.update({f"wide/{k}": v for k, v in self.wide.weights().items()})
        return out

    def oob_counter(self, device):
        """The out-of-range id counter of the model's tables and wide features (one shared counter) and its owner; (None,
        None) for a model without ids (a deep branch over continuous columns only and no wide branch)."""
        if self.input_block is not None and self.input_block.embeddings is not None:
            owner = self.input_block.embeddings
        elif self.wide is not None:
            owner = self.wide.ids
        else:
            return None, None
        return owner.counter(device), owner

    def forward(self, inputs: TabularData, out_layer: _Dense, logits: bool = False) -> torch.Tensor:
        dev = next(iter(inputs.values())).device
        if not self.built:
            self.build(dev)
        B = batch_size_of(inputs)
        h = dl = None
        if self.input_block is not None:
            h = run_dense_chain(self.input_block(inputs), self.deep.dense_layers)
            dl = self.deep_logit.dense_layers[-1]
        onehot, bags = self.wide.blocks(inputs) if self.wide is not None else ([], [])
        wd = self.wide.dense if self.wide is not None else None
        out_layer.build(1, dev)
        out = torch.empty((B, 1), dtype=torch.float32, device=dev)
        oob, owner = self.oob_counter(dev)
        ops.wide_deep_head_fwd_bwd(onehot, bags, None if wd is None else wd.kernel.reshape(-1), None if wd is None else wd.bias, h, False,
                                   None if dl is None else dl.kernel.reshape(-1), None if dl is None else dl.bias,
                                   "linear" if dl is None else dl.activation, out_layer.kernel.reshape(-1), out_layer.bias,
                                   out.reshape(-1), out_act="linear" if logits else out_layer.activation, oob=oob)
        if owner is not None:
            owner.finish_check(oob)
        return out

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        raise NotImplementedError("WideAndDeepBody runs inside its RankingModel (the output layer is fused into its head)")


def WideAndDeepModel(schema: Schema, deep_block: Optional[MLP] = None, wide_schema: Optional[Schema] = None,
                     deep_schema: Optional[Schema] = None, wide_preprocess=None, deep_input_block: Optional[InputBlockV2] = None,
                     wide_input_block=None, deep_regularizer=None, wide_regularizer=None, deep_dropout: Optional[float] = None,
                     wide_dropout: Optional[float] = None, prediction_tasks=None, pre=None, **wide_body_kwargs) -> RankingModel:
    """models/ranking.py:276-570: Dense(1)(deep(x)) + Dense(1)(CategoryEncoding(wide features)), then the prediction task.

    deep   deep_input_block, default InputBlockV2(deep_schema, categorical=Embeddings(categorical part of deep_schema,
           sequence_combiner="mean")) at inferred widths, deep_schema defaulting to schema; then deep_block and
           MLPBlock([1], no_activation_last_layer=True).  No deep part when deep_block is None or deep_schema has no
           input features (the reference needs a deep_block).
    wide   wide_preprocess (a CategoryEncoding; default CategoryEncoding(wide_schema, output_mode="one_hot")) over the
           categorical columns of wide_schema in sorted-name order, then Dense(1) with bias.  Continuous columns of
           wide_schema add nothing (CategoryEncoding emits categorical columns only).  No wide_schema: pure deep, with the
           reference's warning.
    A list feature given ragged (`__values` / `__offsets`) contributes only its own ids to the wide term; the reference
    pads it to a dense (B, L) matrix with id 0 first (ToDense).  Dropout is the identity in the forward; regularizers do
    not change the forward."""
    import warnings

    if pre is not None:
        raise NotImplementedError("WideAndDeepModel(pre=...) is not implemented")
    if wide_input_block is not None:
        raise NotImplementedError("WideAndDeepModel: a custom wide_input_block is not implemented (pass wide_schema and a "
                                  "CategoryEncoding as wide_preprocess)")
    if wide_body_kwargs:
        raise NotImplementedError(f"WideAndDeepModel: options {sorted(wide_body_kwargs)} of the wide Dense are not implemented")
    prediction = parse_prediction_blocks(schema, prediction_tasks)
    if isinstance(prediction, ParallelOutputs):
        raise NotImplementedError("WideAndDeepModel with several outputs is not implemented: pass one BinaryOutput or RegressionOutput")
    if not wide_schema:
        warnings.warn("If not specify wide_schema, NO feature would be sent to wide model")
    if not deep_schema:
        deep_schema = schema
    deep = deep_logit = None
    if deep_block is not None:
        if deep_input_block is None:
            feats = deep_schema.excluding_by_tag(Tags.TARGET)
            if len(feats):
                from .inputs import Embeddings

                cat = feats.select_by_tag(Tags.CATEGORICAL)
                deep_input_block = InputBlockV2(feats, categorical=Embeddings(cat, sequence_combiner="mean")) if len(cat) else InputBlockV2(feats)
        if deep_input_block is not None:
            deep = deep_block
            deep_logit = MLPBlock([1], no_activation_last_layer=True, dropout=deep_dropout)
    else:
        deep_input_block = None
    wide = None
    if wide_schema is not None and len(wide_schema) > 0:
        enc = wide_preprocess if wide_preprocess is not None else CategoryEncoding(wide_schema, output_mode="one_hot", sparse=True)
        if isinstance(enc, (tuple, list)) and len(enc) == 1:
            enc = enc[0]
        if not isinstance(enc, CategoryEncoding):
            raise NotImplementedError(f"WideAndDeepModel: wide_preprocess {type(enc).__name__} is not implemented (CategoryEncoding only)")
        outside = [n for n in enc.cardinalities if n not in wide_schema.column_names]
        if outside:
            raise ValueError(f"wide_preprocess encodes {outside}, which are not in wide_schema")
        wide = WideLinear(enc, exclude=wide_schema.select_by_tag(Tags.TARGET).column_names)
        wide.dropout = wide_dropout
    if deep is None and wide is None:
        raise ValueError("At least the deep part (deep_schema/deep_input_block) or wide part (wide_schema/wide_input_block) must be provided.")
    body = WideAndDeepBody(deep_input_block, deep, deep_logit, wide, regularized=deep_regularizer is not None or wide_regularizer is not None)
    return RankingModel(body, prediction, schema)


class NCFBody(Block):
    """ParallelBlock({"mf": MatrixFactorizationBlock(aggregation=ElementWiseMultiply()), "mlp":
    QueryItemIdsEmbeddingsBlock -> mlp_block}, aggregation="concat") (models/benchmark.py:32-100): (B, D + U) = [u_mf * i_mf |
    h], h = mlp_block([i_mlp | u_mlp]) (the first Dense concatenates the dict {"query", "item"} in sorted-key order: item
    first).  Four tables, each `dim` wide: the GMF product never reaches memory, because the GMF rows are gathered by the
    output-head kernel itself (ops.ncf_head_fwd_bwd), which also runs the output heads."""

    def __init__(self, mf: QueryItemIdsEmbeddingsBlock, mlp_ids: QueryItemIdsEmbeddingsBlock, mlp: MLP, embeddings_l2_reg: float):
        super().__init__(unique_name("ncf_body"))
        self.mf, self.mlp_ids, self.mlp = mf, mlp_ids, mlp
        self.embeddings_l2_reg = float(embeddings_l2_reg)
        self.dim = mf.dim
        for branch, blk in (("mf", mf), ("mlp", mlp_ids)):
            for side in ("query", "item"):
                ib = getattr(blk, side).inputs
                cols = ib.schema.excluding_by_tag(Tags.TARGET)
                if len(cols) != 1 or ib.embeddings is None or cols.first.is_list:
                    raise NotImplementedError(f"NCFModel: the {branch} branch's {side} side needs exactly one non-list id column, "
                                              f"got {cols.column_names}")
        if self.dim % 4 or not 4 <= self.dim <= ops.NCF_MAX_WIDTH:
            raise NotImplementedError(f"NCFModel: embedding_dim {self.dim} is not supported (it needs a multiple of 4 no larger "
                                      f"than {ops.NCF_MAX_WIDTH})")
        if not mlp.dense_layers or mlp.dense_layers[-1].units > ops.NCF_MAX_UNITS:
            raise NotImplementedError(f"NCFModel: the head kernel reads at most {ops.NCF_MAX_UNITS} units of mlp_block's last layer")
        # [item | query]: the first Dense of mlp_block concatenates {"query", "item"} in sorted-key order
        self.mlp_columns = {self.feature("mlp", "item"): 0, self.feature("mlp", "query"): self.dim}
        self.mlp_embeddings = EmbeddingsBlock({t.table_name: t for t in (self.table("mlp", "item"), self.table("mlp", "query"))},
                                              mlp_ids.schema, name="mlp_embeddings")
        # the training step's input block over the same two tables (its columns at mlp_columns, not in sorted-name order)
        self.mlp_input_block = InputBlockV2(mlp_ids.schema.select_by_name(list(self.mlp_columns)), categorical=self.mlp_embeddings)
        self._reg: Optional[torch.Tensor] = None

    _TRANSIENT = {"_reg": None}

    def feature(self, branch: str, side: str) -> str:
        """The id column of one side ("query" / "item") of one branch ("mf" / "mlp")."""
        return getattr(self.mf if branch == "mf" else self.mlp_ids, side).inputs.embeddings.feature_names[0]

    def table(self, branch: str, side: str):
        blk = self.mf if branch == "mf" else self.mlp_ids
        emb = getattr(blk, side).inputs.embeddings
        return emb.feature_to_table[emb.feature_names[0]]

    def build(self, device=None):
        from .core import create_variable

        for side in ("query", "item"):  # the mlp branch's own initial values, not a copy of the mf table of the same name
            t = self.table("mlp", side)
            if t.table is None:
                t.table = create_variable((t.input_dim, t.dim), t.embeddings_initializer, device or default_device(),
                                          f"mlp/{t.table_name}/embeddings")
        self.mf.build(device)
        self.mlp_ids.build(device)
        self.mlp.build_from_width(2 * self.dim, device)
        self.built = True
        return self

    def output_width(self) -> int:
        return self.dim + self.mlp.dense_layers[-1].units

    def weights(self):
        out = {f"mf/{k}": v for k, v in self.mf.weights().items()}
        out.update({f"mlp/{k}": v for k, v in self.mlp_ids.weights().items()})
        out.update({f"mlp/mlp/{k}": v for k, v in self.mlp.weights().items()})
        return out

    def ids(self, inputs: TabularData, side: str) -> torch.Tensor:
        """The GMF id column of one side, as the head kernel reads it (packed host-batch ids at their own width)."""
        from .core import get_feature

        f = self.feature("mf", side)
        x = get_feature(inputs, f)
        if isinstance(x, tuple) or self.table("mf", side).lookup_kind(x) != "onehot":
            raise NotImplementedError(f"NCFModel: feature {f!r} must be one id per sample (ragged / multi-hot ids are not "
                                      "implemented)")
        return ops.fused_ids(x)

    def mlp_input(self, inputs: TabularData) -> torch.Tensor:
        """(B, 2 D) = [i_mlp | u_mlp], through the embeddings' concat path."""
        B = batch_size_of(inputs)
        x0 = torch.empty((B, 2 * self.dim), dtype=torch.float32, device=next(iter(inputs.values())).device)
        self.mlp_embeddings.lookup_all_into(inputs, x0, self.mlp_columns)
        return x0

    def regularization(self, device) -> torch.Tensor:
        """One device float: the embeddings' L2 term of the last forward (with embeddings_l2_reg > 0)."""
        if self._reg is None or self._reg.device != device:
            self._reg = torch.zeros(1, dtype=torch.float32, device=device)
        return self._reg

    def forward(self, inputs: TabularData, outputs: Sequence[Block], head: _Dense, logits: bool = False) -> torch.Tensor:
        """(H, B): the activated predictions of the outputs, or their logits with logits=True.  With embeddings_l2_reg > 0
        the batch's L2 term over the four tables' looked-up rows lands in regularization()."""
        from .blocks import _LAST_HEADS

        dev = next(iter(inputs.values())).device
        if not self.built:
            self.build(dev)
        x0 = self.mlp_input(inputs)
        h = run_dense_chain(x0, self.mlp.dense_layers)
        B, H = x0.shape[0], len(outputs)
        out = torch.empty((H, B), dtype=torch.float32, device=dev)
        losses = ["mse"] * H if logits else [o.loss for o in outputs]
        l2 = self.embeddings_l2_reg
        reg = None
        if l2:
            reg = self.regularization(dev)
            reg.zero_()
        emb = self.mf.query.inputs.embeddings
        oob = emb.counter(dev)
        _LAST_HEADS[0] = "heads"
        ops.ncf_head_fwd_bwd(self.table("mf", "query").embeddings, self.ids(inputs, "query"), self.table("mf", "item").embeddings,
                             self.ids(inputs, "item"), h, head.kernel, head.bias, losses, None, out, reg=reg, l2=l2,
                             relu_h=False, x_reg=x0 if l2 else None, oob=oob)
        emb.finish_check(oob)
        return out

    def call(self, inputs: TabularData, **kwargs):
        raise NotImplementedError("NCFBody runs inside its RankingModel (the output heads are fused with the GMF branch)")


def DCNModel(schema: Schema, depth: int, deep_block: Optional[MLP] = None, stacked: bool = True,
             input_block: Optional[InputBlockV2] = None, prediction_tasks=None, **kwargs) -> RankingModel:
    """models/ranking.py:95-168 (default deep_block = MLPBlock([512, 256]))."""
    deep_block = deep_block if deep_block is not None else MLPBlock([512, 256])
    input_block = input_block or InputBlockV2(schema, **kwargs)
    prediction = parse_prediction_blocks(schema, prediction_tasks)
    body = DCNBody(input_block, CrossBlock(depth), deep_block, stacked)
    return RankingModel(body, prediction, schema)


def _brute_force(k: int):
    from .topk import BruteForce

    return BruteForce(k=k)


class RetrievalModel(Model):
    """models/base.py:2259-2489.  `compile(optimizer=...)` / `train_step` / `fit` train a v1 TwoTowerModel or a
    MatrixFactorizationModel with its ItemRetrievalTask's in-batch soft-max cross-entropy plus the embeddings' L2 term
    (models_b200/train.py: TwoTowerTrainer)."""

    _TRANSIENT = {"pre_eval_topk": None}
    _fit_skip = ("loss", "loss_batch")  # History: "loss" and "regularization_loss"

    def _compile_training(self, optimizer, loss=None, loss_weights=None, metrics=None, weighted_metrics=None) -> None:
        """As Model's, and `loss` may also name one of the reference's pairwise losses (models_b200/losses.py): "bpr",
        "bpr-max", "top1", "top1_v2", "top1-max", "logistic", "hinge" or a loss object.  `pairwise_loss` keeps it (None:
        the in-batch soft-max cross-entropy)."""
        from .losses import get

        pairwise = None if isinstance(loss, dict) else get(loss)
        super()._compile_training(optimizer, None if pairwise is not None else loss, loss_weights, metrics, weighted_metrics)
        self.pairwise_loss = pairwise

    def train_step(self, data) -> Dict[str, torch.Tensor]:
        """One optimizer step on `data` = (inputs,) or (inputs, targets); the targets are ignored, because the retrieval task
        builds its own one-hot targets (the positive item on column 0).  Returns {"loss", "loss_batch",
        "regularization_loss"} as device scalars, views of the engine's loss buffer valid until the next step."""
        if getattr(self, "optimizer", None) is None:
            raise RuntimeError("compile() the model with an optimizer before training it")
        if isinstance(data, dict):
            data = (data,)
        if not isinstance(data, (tuple, list)) or not data:
            raise ValueError("train_step expects (inputs,) or (inputs, targets)")
        if len(data) > 2 and data[2] is not None:
            raise NotImplementedError("sample_weight is not implemented in the two-tower training step")
        x = data[0]
        self._check_inputs(x)
        tr = self.trainer(batch_size_of(x))
        loss = tr.step(x, None)  # [total, regularization]: the embeddings' L2 term is part of the total
        return {"loss": loss[0], "loss_batch": loss[0], "regularization_loss": loss[1]}

    def fit(self, x=None, y=None, batch_size: Optional[int] = None, epochs: int = 1, steps_per_epoch: Optional[int] = None,
            verbose: int = 0, **kwargs):
        """Keras `fit` over a Loader or an iterable of batches, each a feature dict or (inputs, targets) (targets ignored)."""
        if x is None:
            raise ValueError("fit needs a loader / iterable of batches")
        bs = batch_size or getattr(x, "batch_size", None)

        class _Pairs:
            def __iter__(self_):
                for item in x:
                    yield (item, None) if isinstance(item, dict) else (item[0], None)

        return super().fit(_Pairs(), y, batch_size=bs, epochs=epochs, steps_per_epoch=steps_per_epoch, verbose=verbose, **kwargs)

    def build(self, device=None):
        self.body.build(device)
        self.built = True
        return self

    def input_columns(self) -> List[str]:
        tb: TwoTowerBlock = self.body
        used = Schema(list(tb.query.inputs.schema) + [c for c in tb.item.inputs.schema
                                                      if c.name not in tb.query.inputs.schema])
        return expected_input_columns(used)

    def call(self, inputs: TabularData, targets=None, training: bool = False, testing: bool = False, **kwargs):
        self._check_inputs(inputs)
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        emb = self.body(inputs, training=False)
        # fused_loss=True (training/testing): Prediction.outputs = (B,3) [max, log-sum-exp, positive logit] of the in-batch
        # logits — loss = outputs[:,1] - outputs[:,2] — instead of the (B, 1+B) logits themselves
        return self.prediction(emb, features=inputs, training=training, testing=testing, **kwargs)

    # -- top-k retrieval / evaluation (SURVEY §8f-2; models/base.py:2266-2489) ---------------------
    @property
    def retrieval_block(self) -> TwoTowerBlock:
        return self.body

    def query_encoder(self) -> Block:
        """Query tower (+ the model's `post`, e.g. L2 normalisation) as a feature-dict -> (B, D) block."""
        from .topk import TowerEncoder

        return TowerEncoder(self.body.query, self.body.post)

    def candidate_encoder(self) -> Block:
        from .topk import TowerEncoder

        return TowerEncoder(self.body.item, self.body.post)

    def _item_id_column(self) -> str:
        tagged = self.schema.select_by_tag(Tags.ITEM_ID)
        if not tagged:
            raise ValueError("the schema has no column tagged ITEM_ID")
        return tagged.first.name

    def query_embeddings(self, data: Dict[str, np.ndarray], batch_size: int = 65536, query_id: Optional[str] = None):
        """models/base.py:2354-2385: (ids, embeddings) of the query tower over `data`."""
        from .topk import encode_rows

        query_id = query_id or (self.schema.select_by_tag(Tags.USER_ID).first.name if self.schema.select_by_tag(Tags.USER_ID) else None)
        return encode_rows(self.query_encoder(), data, query_id, batch_size)

    def item_embeddings(self, data: Dict[str, np.ndarray], batch_size: int = 65536, item_id: Optional[str] = None):
        """models/base.py:2387-2418: (ids, embeddings) of the item tower over `data`."""
        from .topk import encode_rows

        return encode_rows(self.candidate_encoder(), data, item_id or self._item_id_column(), batch_size)

    def to_top_k_encoder(self, candidates, candidate_id: Optional[str] = None, k: int = 10, batch_size: int = 65536,
                         **kwargs):
        """models/base.py `to_top_k_encoder`: query tower -> brute-force top-k over `candidates` — raw item
        features (dict, encoded by the item tower) or precomputed (ids, embeddings) / a DataFrame indexed by id."""
        from .topk import TopKEncoder

        enc = TopKEncoder(self.query_encoder(), candidates=None if isinstance(candidates, dict) else candidates,
                          candidate_encoder=self.candidate_encoder(), k=k, target=self._item_id_column(),
                          topk_layer=kwargs.pop("topk_layer", None) or _brute_force(k), **kwargs)
        if isinstance(candidates, dict):
            enc.index_candidates(candidates, candidate_id or self._item_id_column(), batch_size)
        return enc

    def evaluate(self, x, item_corpus=None, metrics=None, batch_size: int = 65536, return_dict: bool = True, **kwargs):
        """models/base.py:2266-2351.  `x`: one feature-dict batch or an iterable of them (host arrays or device
        tensors).  With `item_corpus` (a TopKIndexBlock, or the item features of the corpus as a dict: deduplicated
        by item id and encoded by the item tower) every query is ranked against the whole corpus by the fused
        score + top-k kernel; without it the batch's own items are the candidates (in-batch evaluation)."""
        from .topk import (NDCGAt, RecallAt, TopKIndexBlock, evaluate_topk, unique_rows_by_features)

        metrics = list(metrics) if metrics else [RecallAt(10), NDCGAt(10)]
        kmax = max(m.k for m in metrics)
        item_id = self._item_id_column()
        if item_corpus is not None:
            if isinstance(item_corpus, TopKIndexBlock):
                index = item_corpus
                if index._k < kmax:
                    raise ValueError(f"the index returns {index._k} candidates, the metrics need {kmax}")
            elif isinstance(item_corpus, dict):
                corpus = unique_rows_by_features(item_corpus, item_id)
                if not self.built:
                    self.build(default_device())
                index = TopKIndexBlock.from_block(self.candidate_encoder(), corpus, k=kmax, id_column=item_id,
                                                  batch_size=batch_size)
            else:
                raise ValueError(f"`item_corpus` must be either a `TopKIndexBlock` or a dict of item features. Got {type(item_corpus)}")
            self.pre_eval_topk = index
            q = self.query_encoder()

            def predict(b):
                if not self.built:
                    self.build(next(iter(b.values())).device)
                return index.call_outputs(b[item_id].reshape(-1), q(b))
        else:
            def predict(b):
                out = self(b, testing=True)
                k = min(kmax, out.outputs.shape[1])
                scores, order = torch.topk(out.outputs, k, dim=1)
                return Prediction(scores, torch.gather(out.targets, 1, order))
        return evaluate_topk(predict, x, metrics)


class RetrievalModelV2(Model):
    """models/base.py RetrievalModelV2 (forward): query Encoder, candidate Encoder, one output layer.
    Inference: output({"query": q, "candidate": c}) -> (B,1); training/testing: [positive | negatives] logits from the
    output's samplers (or their soft-max CE statistics with fused_loss=True)."""

    def __init__(self, query, candidate, output, schema: Optional[Schema] = None, candidate_id_tag=Tags.ITEM_ID):
        from .retrieval import Encoder

        if schema is None:
            cols = list(query.schema) + [c for c in candidate.schema if c.name not in query.schema]
            schema = Schema(cols)
        super().__init__(query, output, schema)
        self.query_encoder_block, self.candidate_encoder_block = query, candidate
        ids = candidate.schema.select_by_tag(candidate_id_tag).column_names
        if not ids:
            raise ValueError(f"the candidate tower has no column tagged {candidate_id_tag}")
        self.candidate_id_name = ids[0]

    @property
    def blocks(self) -> List[Block]:
        return [self.query_encoder_block, self.candidate_encoder_block, self.prediction]

    def weights(self):
        out = {f"query/{k}": v for k, v in self.query_encoder_block.weights().items()}
        out.update({f"candidate/{k}": v for k, v in self.candidate_encoder_block.weights().items()})
        return out

    def build(self, device=None):
        self.query_encoder_block.build(device)
        self.candidate_encoder_block.build(device)
        self.built = True
        return self

    def input_columns(self) -> List[str]:
        return expected_input_columns(self.schema)

    def query_encoder(self) -> Block:
        return self.query_encoder_block

    def candidate_encoder(self) -> Block:
        return self.candidate_encoder_block

    def call(self, inputs: TabularData, targets=None, training: bool = False, testing: bool = False, **kwargs):
        self._check_inputs(inputs)
        if not self.built:
            self.build(next(iter(inputs.values())).device)
        out = self.prediction
        enc = {out.query_name: self.query_encoder_block(inputs), out.candidate_name: self.candidate_encoder_block(inputs)}
        return out(enc, candidate_ids=inputs[self.candidate_id_name], training=training, testing=testing, **kwargs)


def TwoTowerModelV2(query_tower, candidate_tower, candidate_id_tag=Tags.ITEM_ID, outputs=None, logits_temperature: float = 1.0,
                    negative_samplers=None, schema: Optional[Schema] = None, **kwargs) -> RetrievalModelV2:
    """models/retrieval.py:409-486: two Encoder towers + ContrastiveOutput(DotProduct, in-batch negatives by default)."""
    from .retrieval import ContrastiveOutput, Encoder

    assert isinstance(query_tower, Encoder), ValueError("The query tower should be an instance of `Encoder` class")
    assert isinstance(candidate_tower, Encoder), ValueError("The query tower should be an instance of `Encoder` class")
    if not outputs:
        if not negative_samplers:
            negative_samplers = ["in-batch"]
        outputs = ContrastiveOutput(to_call=None, negative_samplers=negative_samplers, logits_temperature=logits_temperature,
                                    **kwargs)
    if isinstance(outputs, (list, tuple)):
        if len(outputs) != 1:
            raise NotImplementedError("multi-task outputs are outside the hot path")
        outputs = outputs[0]
    return RetrievalModelV2(query_tower, candidate_tower, outputs, schema=schema, candidate_id_tag=candidate_id_tag)


def TwoTowerModel(schema: Schema, query_tower: MLP, item_tower: Optional[MLP] = None, query_tower_tag=Tags.USER,
                  item_tower_tag=Tags.ITEM,
                  embedding_options: EmbeddingOptions = EmbeddingOptions(embedding_dims=None, embedding_dim_default=64,
                                                                         infer_embedding_sizes=False,
                                                                         infer_embedding_sizes_multiplier=2.0),
                  post: Optional[Block] = None, prediction_tasks=None, logits_temperature: float = 1.0,
                  samplers: Sequence = (), **kwargs) -> RetrievalModel:
    """models/retrieval.py:106-203."""
    if not prediction_tasks:
        prediction_tasks = ItemRetrievalTask(schema, logits_temperature=logits_temperature, samplers=list(samplers))
    if isinstance(prediction_tasks, (list, tuple)):
        prediction_tasks = prediction_tasks[0]
    two_tower = TwoTowerBlock(schema=schema, query_tower=query_tower, item_tower=item_tower,
                              query_tower_tag=query_tower_tag, item_tower_tag=item_tower_tag,
                              embedding_options=embedding_options, post=post)
    return RetrievalModel(two_tower, prediction_tasks, schema)


def MatrixFactorizationModel(schema: Schema, dim: int, query_id_tag=Tags.USER_ID, item_id_tag=Tags.ITEM_ID,
                             embeddings_initializers=None, embeddings_l2_reg: float = 0.0, post: Optional[Block] = None,
                             prediction_tasks=None, logits_temperature: float = 1.0, samplers: Sequence = (),
                             **kwargs) -> RetrievalModel:
    """models/retrieval.py:27-103: a RetrievalModel over QueryItemIdsEmbeddingsBlock (user-id and item-id embeddings
    of width `dim`, no MLP) with an ItemRetrievalTask (in-batch negatives by default).  embeddings_l2_reg adds
    embeddings_l2_reg * sum ||e||^2 over the batch's looked-up embeddings to the training loss."""
    if not prediction_tasks:
        prediction_tasks = ItemRetrievalTask(schema, logits_temperature=logits_temperature, samplers=list(samplers), **kwargs)
    if isinstance(prediction_tasks, (list, tuple)):
        prediction_tasks = prediction_tasks[0]
    mf = QueryItemIdsEmbeddingsBlock(schema=schema, dim=dim, query_id_tag=query_id_tag, item_id_tag=item_id_tag,
                                     embeddings_initializers=embeddings_initializers, embeddings_l2_reg=embeddings_l2_reg,
                                     post=post)
    return RetrievalModel(mf, prediction_tasks, schema)
