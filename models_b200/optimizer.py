"""Per-block optimizers (blocks/optimizer.py:42-340, 461-485): `OptimizerBlocks`, `MultiOptimizer` and
`split_embeddings_on_size`.  A block's variables are the Dense layers, embedding tables and CategoricalOutput biases
reachable from it; the training step gives every optimizer its own device hyper-parameters (step counter, learning
rate, schedule) and slots, and updates each variable with its optimizer's rule (models_b200/train.py)."""
from __future__ import annotations

import warnings
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple, Union

from .core import Block

# the reference's default; RMSprop is not implemented, so it is refused only when a variable falls to it
_RMSPROP = "rmsprop"


@dataclass
class OptimizerBlocks:
    """An optimizer (a name or an instance) and the block or blocks it applies to."""

    optimizer: object
    blocks: Union[Block, Sequence[Block]]

    def get_config(self) -> tuple:
        """(serialised optimizer, [serialised block, ...]), the reference's layout."""
        return _serialize_optimizer(self.optimizer), [{"class_name": type(b).__name__, "config": {"name": b.name}}
                                                      for b in _as_list(self.blocks)]


def _as_list(blocks) -> List[Block]:
    return [blocks] if isinstance(blocks, Block) else list(blocks)


def _serialize_optimizer(opt) -> Union[str, dict]:
    return opt if isinstance(opt, str) else {"class_name": type(opt).__name__, "config": opt.get_config()}


def _get_optimizer(spec, default: bool = False):
    """An Optimizer instance; as the default, the unimplemented "rmsprop" is kept as its name (refused when used)."""
    from .train import Optimizer, get_optimizer

    if default and isinstance(spec, str) and spec.lower() == _RMSPROP:
        return _RMSPROP
    if not isinstance(spec, (str, Optimizer)):
        raise TypeError(f"optimizers must be a name or a models_b200 Optimizer, got {type(spec).__name__}")
    return get_optimizer(spec)


def variable_name(v) -> str:
    from .inputs import EmbeddingTable
    from .retrieval import CategoricalOutput

    if isinstance(v, EmbeddingTable):
        return f"{v.table_name}/embeddings"
    if isinstance(v, CategoricalOutput):
        return f"{v.name}/bias"
    return v.name


def block_variables(block) -> List[object]:
    """The variables reachable from `block`, each once: Dense layers (kernel and bias), EmbeddingTables, and
    CategoricalOutputs with a bias (the bias; its weight-tied table is reached as a table)."""
    from .blocks import _Dense
    from .inputs import EmbeddingTable
    from .pretrained import PretrainedBranch
    from .retrieval import CategoricalOutput

    found: List[object] = []
    seen = set()

    def walk(o, depth: int) -> None:
        if id(o) in seen or depth > 24:
            return
        seen.add(id(o))
        if isinstance(o, (_Dense, EmbeddingTable)):
            found.append(o)
            return
        if isinstance(o, CategoricalOutput) and o.use_bias:
            found.append(o)
        if isinstance(o, (Block, PretrainedBranch)):
            for v in vars(o).values():
                walk(v, depth + 1)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v, depth + 1)
        elif isinstance(o, dict):
            for v in o.values():
                walk(v, depth + 1)

    walk(block, 0)
    return found


def stacked_layers(model) -> Dict[int, tuple]:
    """id(stacked Dense) -> (stacked Dense, [its parts]) for the layers that hold several variables of the reference as
    views: MMOEBlock's experts and stacked gates, ParallelOutputs' stacked heads."""
    from .experts import MMOEBlock
    from .models import ParallelOutputs

    out: Dict[int, tuple] = {}
    for b in block_variables_owners(model, (MMOEBlock, ParallelOutputs)):
        if isinstance(b, MMOEBlock):
            out[id(b.experts)] = (b.experts, [b.expert_blocks[n].dense_layers[0] for n in b.expert_names])
            if b.gates is not None:
                out[id(b.gates)] = (b.gates, [b.gate_finals[n] for n in b.output_names])
        else:
            out[id(b.to_call)] = (b.to_call, [o.to_call for o in b.outputs])
    return out


def block_variables_owners(root, types: tuple) -> List[Block]:
    """Every block of the given types reachable from root."""
    found: List[Block] = []
    seen = set()

    def walk(o, depth: int) -> None:
        if id(o) in seen or depth > 24:
            return
        seen.add(id(o))
        if isinstance(o, types):
            found.append(o)
        if isinstance(o, Block):
            for v in vars(o).values():
                walk(v, depth + 1)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v, depth + 1)
        elif isinstance(o, dict):
            for v in o.values():
                walk(v, depth + 1)

    walk(root, 0)
    return found


class MultiOptimizer:
    """Different optimizers for different blocks (blocks/optimizer.py:63-340): each OptimizerBlocks entry's optimizer
    updates the variables reachable from its blocks, `default_optimizer` every other variable.  The entries must be
    disjoint; entries given through `update()` are resolved afterwards and override.  Every optimizer keeps its own step
    counter, learning rate (or schedule) and slots.  The default "rmsprop" is the reference's; RMSprop is not implemented,
    so training refuses it only when some variable actually falls to it."""

    def __init__(self, optimizers_and_blocks: Sequence[OptimizerBlocks], default_optimizer="rmsprop",
                 name: str = "MultiOptimizer", **kwargs):
        if not optimizers_and_blocks:
            raise ValueError("`optimizers_and_blocks` can't be empty")
        self.name = name
        self.default_optimizer = _get_optimizer(default_optimizer, default=True)
        self.optimizers_and_blocks: List[OptimizerBlocks] = []
        self.update_optimizers_and_blocks: List[OptimizerBlocks] = []
        for pair in optimizers_and_blocks:
            self.add(pair)

    @staticmethod
    def _resolved(pair: OptimizerBlocks) -> OptimizerBlocks:
        if not isinstance(pair, OptimizerBlocks):
            raise TypeError(f"expected OptimizerBlocks, got {type(pair).__name__}")
        pair.optimizer = _get_optimizer(pair.optimizer)
        pair.blocks = _as_list(pair.blocks)
        return pair

    def add(self, optimizer_blocks: OptimizerBlocks) -> None:
        """Another optimizer and the blocks it applies to (disjoint from the other entries)."""
        self.optimizers_and_blocks.append(self._resolved(optimizer_blocks))

    def update(self, optimizer_blocks: OptimizerBlocks) -> None:
        """Give the blocks this optimizer whatever they had before (kept apart, resolved after the other entries)."""
        self.update_optimizers_and_blocks.append(self._resolved(optimizer_blocks))

    @property
    def optimizers(self) -> list:
        """The optimizers in order, the default last."""
        return [p.optimizer for p in self.optimizers_and_blocks] + [self.default_optimizer]

    def get_config(self) -> dict:
        return {"default_optimizer": _serialize_optimizer(self.default_optimizer), "name": self.name,
                "optimizers_and_blocks": [p.get_config() for p in self.optimizers_and_blocks],
                "update_optimizers_and_blocks": [p.get_config() for p in self.update_optimizers_and_blocks]}

    def assignments(self, model) -> Dict[int, object]:
        """id(variable) -> optimizer for every variable an entry covers (not the default's).  A variable reachable from
        two optimizers_and_blocks entries raises ValueError; part of a stacked layer (MMoE experts / gates, stacked
        output heads) under another optimizer than the rest of it raises NotImplementedError."""
        assign: Dict[int, object] = {}
        where: Dict[int, str] = {}
        for pair in self.optimizers_and_blocks:
            mine = {}
            for blk in pair.blocks:
                for v in block_variables(blk):
                    mine[id(v)] = v
            for k, v in mine.items():
                if k in assign:
                    raise ValueError(f"The set of variables handled by each optimizer should be disjoint, but variable "
                                     f"{variable_name(v)!r} is handled both by {where[k]} and {_describe(pair.optimizer)}")
                assign[k], where[k] = pair.optimizer, _describe(pair.optimizer)
        for pair in self.update_optimizers_and_blocks:
            for blk in pair.blocks:
                for v in block_variables(blk):
                    assign[id(v)] = pair.optimizer
        for k, (layer, parts) in stacked_layers(model).items():
            whole = assign.get(k, self.default_optimizer)
            opts = {id(assign.get(id(p), whole)): assign.get(id(p), whole) for p in parts}
            if len(opts) > 1:
                raise NotImplementedError(f"{layer.name}: its parts are assigned to different optimizers "
                                          f"({', '.join(_describe(o) for o in opts.values())}); they are views of one "
                                          "stacked layer, which trains under one optimizer")
            assign[k] = next(iter(opts.values()))
        return assign


def _describe(opt) -> str:
    return repr(opt) if isinstance(opt, str) else f"{type(opt).__name__}(learning_rate={opt.learning_rate!r})"


def split_embeddings_on_size(embeddings, threshold: int) -> Tuple[List[Block], List[Block]]:
    """(large, small): the tables of an embeddings block with input_dim >= threshold, and the others."""
    from .inputs import EmbeddingsBlock

    if not isinstance(embeddings, EmbeddingsBlock):
        raise TypeError(f"split_embeddings_on_size takes an embeddings block, got {type(embeddings).__name__}")
    large, small = [], []
    for t in embeddings.tables.values():
        (large if t.input_dim >= threshold else small).append(t)
    if not large:
        warnings.warn(f"All embedding tables in given ParallelBlock {embeddings.name} have smaller input dim than threshold "
                      f"{threshold}, thus return empty list.")
    return large, small
