"""Training steps (SURVEY §8(f)-4): forward with saved activations, loss, backward and optimizer update as hand-written
CUDA (include/mm_b200.h K14), behind the reference's `compile` / `fit` / `train_step`
(merlin/models/tf/models/base.py:1121-1231; optimizers: tf.keras.optimizers.{SGD, Adagrad, Adam}, LazyAdam
blocks/optimizer.py:342).  One trainer per model (DLRMTrainer, DCNTrainer, TwoTowerTrainer, DeepFMTrainer,
WideAndDeepTrainer, MMoETrainer, NCFTrainer; trainer_for picks) holds what is particular to it; the parts they share are methods of
_StepTrainer (the construction checks, the dense arena, the table checks and optimizer state, a chain of Dense layers forward
and backward, multi-hot pooling, the output heads, the step's prologue, the update (apply_gradients), snapshot / restore,
capture / replay) and two parts a trainer owns: the concatenating input block (_ConcatInput) and a wide kernel trained
outside the arena (_WideKernel).

What a step launches (DLRM, bottom [.., D], top [...], BinaryOutput):

    forward   concat+split -> dense_tc per bottom layer (fp32 activation saved + operand of the next layer) -> fused
              lookup + interaction -> dense_tc per top layer.  D = 64 with table mirrors: the kernel reads operand-format
              rows and writes the top tower's split operand directly; otherwise fp32 rows + one split pass
    loss      mm_heads_fwd_bwd: the output heads (BinaryOutput: Dense(1) + sigmoid + BCE; RegressionOutput: Dense(1) + MSE;
              up to 8 of them with loss weights) forward AND backward in one pass
    backward  per Dense layer mm_dense_wgrad[_split] (dW, db) + mm_dense_dgrad (input gradient, relu mask fused);
              mm_dlrm_interact_backward: pair gradients -> IndexedSlices per table + bottom-vector gradient
    update    mm_opt_tick, [DP: all-reduce of the dense gradient arena, all-gather of the slices], mm_dense_apply over the flat
              parameter arena, mm_sparse_rows_apply (duplicate ids summed, one update per touched row), mm_split_weights
              refresh of the tensor-core operand copies (in place)

Multi-hot features (ragged `name__values` + `name__offsets`, or (B, L) id matrices; combiners mean / sum / sqrtn) are pooled
by mm_gather_bag / mm_gather_seq (_pool_bag), in DLRM into a (B, D) buffer that the lookup + interaction kernels read as one
more table of B rows at ids 0..B-1, so those kernels serve them unchanged; the backward's slice of that "table" is the
pooled-row gradient, which mm_bag_grad_rows expands to one scaled row per id for one mm_sparse_rows_apply call per multi-hot
table.  Ragged features are trained eagerly (their number of ids changes per batch); fixed-length ones can be captured like
one-hot features.

DCNModel trains through DCNTrainer (below): the cross network's backward (mm_cross_backward per layer), the input block's
backward straight into per-table slices (mm_concat_backward) and one sparse update per distinct embedding width.
The v1 TwoTowerModel trains through TwoTowerTrainer: both towers as DCN's input block + deep tower, the in-batch soft-max
cross-entropy forward and backward without the (B, 1+B) logits (mm_inbatch_softmax_ce[_backward]).  MatrixFactorizationModel
trains there too, with towers that are the id embeddings themselves; the embeddings' L2 term (embeddings_l2_reg) is fused
into the input block's backward (mm_concat_backward_l2).
DeepFMModel trains through DeepFMTrainer: DCN's input block and deep tower, the FM / wide / output head forward and
backward in one kernel (mm_deepfm_head_fwd_bwd), the FM term's input gradient (mm_fm_concat_backward) and the wide
kernel's sparse update (mm_wide_rows_apply).
NCFModel trains through NCFTrainer: the mlp branch's rows and tower as DCN's input block and deep tower, and the GMF branch,
the output heads and their loss forward and backward in one kernel that gathers the GMF rows itself (mm_ncf_head_fwd_bwd).

All Dense variables of the model are re-homed into ONE flat fp32 arena (gradients and optimizer slots mirror its layout), so
the dense update is one launch and data-parallel training needs one all-reduce.  Every buffer is static: a step can be
captured into a CUDA graph (`capture()` / `replay()`), the learning rate lives in device memory.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _cabi, ops, schedules
from .blocks import DLRM, MLP, _Dense
from .core import batch_size_of, default_device, get_feature
from .graph import graph_capture

INT32_MAX = 2**31 - 1
DENSE_PATH_MAX_ROWS = 131072  # tables up to this size accumulate duplicate ids in a dense (rows, D) gradient
SPARSE_MAX_TABLES = 32  # tables per mm_sparse_rows_apply call (MM_LOOKUP_MAX_ROWS)
CONCAT_MAX_SLICES = 64  # tables per mm_concat_backward call


class History:
    """What Keras `fit` returns: `.history["loss"]` = mean batch loss of every epoch."""

    def __init__(self, history: Dict[str, List[float]]):
        self.history = history
        self.epoch = list(range(len(history.get("loss", []))))


class Optimizer:
    """Hyper-parameters of one of the update rules in include/mm_b200.h (Keras argument names and defaults).
    learning_rate: a float, or one of the built-in schedules of models_b200.schedules (evaluated on the device each step
    from the optimizer's step counter, K25)."""

    kind = "sgd"

    def __init__(self, learning_rate, beta_1: float = 0.0, beta_2: float = 0.0, epsilon: float = 1e-7,
                 initial_accumulator_value: float = 0.0):
        if callable(learning_rate) or isinstance(learning_rate, schedules.LearningRateSchedule):
            schedules.check_trainable(learning_rate)
            self.learning_rate = learning_rate
        else:
            if learning_rate < 0:
                raise ValueError("learning_rate must be >= 0")
            self.learning_rate = float(learning_rate)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)
        self.initial_accumulator_value = float(initial_accumulator_value)

    @property
    def schedule(self) -> Optional[schedules.LearningRateSchedule]:
        return self.learning_rate if isinstance(self.learning_rate, schedules.LearningRateSchedule) else None

    def hyper(self) -> np.ndarray:
        """The device hyper-parameters before the first step; a schedule's lr(0) as the learning rate."""
        h = np.zeros(_cabi.HYPER_COUNT, dtype=np.float32)
        lr = self.learning_rate if self.schedule is None else self.schedule(0)
        h[_cabi.HYPER_LR], h[_cabi.HYPER_BETA1], h[_cabi.HYPER_BETA2] = lr, self.beta_1, self.beta_2
        h[_cabi.HYPER_EPS] = self.epsilon
        return h

    @property
    def slots(self) -> int:
        return {"sgd": 0, "adagrad": 1, "adam": 2}[self.kind]

    def get_config(self) -> dict:
        lr = self.learning_rate if self.schedule is None else schedules.serialize(self.schedule)
        return {"name": type(self).__name__, "learning_rate": lr, "beta_1": self.beta_1, "beta_2": self.beta_2,
                "epsilon": self.epsilon, "initial_accumulator_value": self.initial_accumulator_value}


class SGD(Optimizer):
    """tf.keras.optimizers.SGD(learning_rate=0.01) without momentum."""

    kind = "sgd"

    def __init__(self, learning_rate=0.01, momentum: float = 0.0, **kwargs):
        if momentum:
            raise NotImplementedError("SGD momentum is not implemented")
        super().__init__(learning_rate)


class Adagrad(Optimizer):
    """tf.keras.optimizers.Adagrad(learning_rate=0.001, initial_accumulator_value=0.1, epsilon=1e-7)."""

    kind = "adagrad"

    def __init__(self, learning_rate=0.001, initial_accumulator_value: float = 0.1, epsilon: float = 1e-7, **kwargs):
        if initial_accumulator_value < 0:
            raise ValueError("initial_accumulator_value must be non-negative")
        super().__init__(learning_rate, epsilon=epsilon, initial_accumulator_value=initial_accumulator_value)


class Adam(Optimizer):
    """tf.keras.optimizers.Adam(0.001, 0.9, 0.999, 1e-7).  Embedding rows are updated lazily (only the rows a batch looked
    up, from the summed duplicate gradients) — the reference's LazyAdam (blocks/optimizer.py:342)."""

    kind = "adam"

    def __init__(self, learning_rate=0.001, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7, **kwargs):
        super().__init__(learning_rate, beta_1, beta_2, epsilon)


LazyAdam = Adam

_BY_NAME = {"sgd": SGD, "adagrad": Adagrad, "adam": Adam, "lazyadam": Adam, "lazy_adam": Adam}


def get_optimizer(spec):
    """An Optimizer (or a MultiOptimizer) from a name or an instance."""
    from .optimizer import MultiOptimizer

    if isinstance(spec, (Optimizer, MultiOptimizer)):
        return spec
    if isinstance(spec, str):
        if spec.lower() not in _BY_NAME:
            raise ValueError(f"Unknown optimizer {spec!r}; supported: {sorted(_BY_NAME)}")
        return _BY_NAME[spec.lower()]()
    raise TypeError(f"optimizer must be a name or a models_b200.train.Optimizer, got {type(spec).__name__}")


def _align(n: int, a: int = 64) -> int:
    return (n + a - 1) // a * a


def _ld4(d: int) -> int:
    """Row stride (a multiple of 4) of the fp32 buffer behind a (B, d) view."""
    return (d + 3) // 4 * 4


class DenseArena:
    """All Dense variables of a chain of layers in one flat fp32 buffer (kernel then bias per layer, 256-byte aligned);
    `grad`, `state1`, `state2` share the layout.  The layers' `kernel` / `bias` become views of it.  optimizer: one
    optimizer for every layer, or one per layer (anything with `slots` and `initial_accumulator_value`); `runs` holds
    (start, end, optimizer) per contiguous run of layers with the same optimizer, in arena order."""

    def __init__(self, layers: Sequence[_Dense], optimizer, device):
        self.layers = list(layers)
        opts = list(optimizer) if isinstance(optimizer, (list, tuple)) else [optimizer] * len(self.layers)
        off = 0
        self.kernel_off, self.bias_off = [], []
        for l in self.layers:
            if l.kernel is None:
                raise RuntimeError(f"{l.name}: build the model before compiling it for training")
            self.kernel_off.append(off)
            off = _align(off + l.kernel.numel())
            self.bias_off.append(off if l.bias is not None else None)
            if l.bias is not None:
                off = _align(off + l.bias.numel())
        self.size = off
        self.runs: List[tuple] = []
        for i, o in enumerate(opts):
            if self.runs and self.runs[-1][2] is o:
                continue
            if self.runs:
                self.runs[-1] = (self.runs[-1][0], self.kernel_off[i], self.runs[-1][2])
            self.runs.append((self.kernel_off[i], off, o))
        self.w = torch.zeros(off, dtype=torch.float32, device=device)
        self.grad = torch.zeros_like(self.w)
        slots = max((o.slots for o in (opts or ([] if isinstance(optimizer, (list, tuple)) else [optimizer]))), default=0)
        self.state1 = torch.zeros_like(self.w) if slots >= 1 else None
        self.state2 = torch.zeros_like(self.w) if slots >= 2 else None
        for s, e, o in self.runs:
            if o.slots >= 1:
                self.state1[s:e] = o.initial_accumulator_value
        for i, l in enumerate(self.layers):
            k = self.view(self.w, i, "kernel")
            k.copy_(l.kernel)
            l.kernel = k
            if l.bias is not None:
                b = self.view(self.w, i, "bias")
                b.copy_(l.bias)
                l.bias = b
            l._weights_changed()

    def view(self, buf: torch.Tensor, i: int, what: str) -> Optional[torch.Tensor]:
        l = self.layers[i]
        if what == "kernel":
            K, N = l.kernel.shape
            return buf[self.kernel_off[i]: self.kernel_off[i] + K * N].view(K, N)
        if self.bias_off[i] is None:
            return None
        return buf[self.bias_off[i]: self.bias_off[i] + l.units]


class _OptGroup:
    """One optimizer of a training step: its update rule, its device hyper-parameters (own step counter, lr, Adam's
    lr_t) and, with a learning-rate schedule, the K25 schedule array its tick evaluates."""

    def __init__(self, opt: Optimizer, device):
        self.opt, self.kind, self.slots = opt, opt.kind, opt.slots
        self.initial_accumulator_value = opt.initial_accumulator_value
        self.hyper = torch.from_numpy(opt.hyper()).to(device)
        sch = opt.schedule
        self.sched = None if sch is None else torch.from_numpy(sch.device_params()).to(device)

    def tick(self) -> None:
        if self.sched is None:
            ops.opt_tick(self.hyper)
        else:
            ops.opt_tick_schedule(self.hyper, self.sched)


class _OptGroups:
    """The optimizer groups of a trainer, created in order of first use: one for a plain optimizer; for a MultiOptimizer
    one per optimizer that some variable of the model resolves to."""

    def __init__(self, optimizer, model, device):
        from .optimizer import MultiOptimizer

        self.device = device
        self.multi = optimizer if isinstance(optimizer, MultiOptimizer) else None
        self.single = None if self.multi is not None else optimizer
        self._assign = self.multi.assignments(model) if self.multi is not None else {}
        self.groups: List[_OptGroup] = []
        self._by_opt: Dict[int, _OptGroup] = {}

    def of(self, var) -> _OptGroup:
        """The group of a variable (a _Dense, an EmbeddingTable or a CategoricalOutput's bias)."""
        opt = self.single if self.multi is None else self._assign.get(id(var), self.multi.default_optimizer)
        if isinstance(opt, str):
            from .optimizer import variable_name

            raise NotImplementedError(f"{variable_name(var)}: no OptimizerBlocks entry covers it and the MultiOptimizer's "
                                      f"default_optimizer {opt!r} (RMSprop) is not implemented: cover every variable or pass "
                                      "another default_optimizer")
        g = self._by_opt.get(id(opt))
        if g is None:
            g = self._by_opt[id(opt)] = _OptGroup(opt, self.device)
            self.groups.append(g)
        return g


def _by_group(items: Sequence, group_of) -> List[tuple]:
    """[(group, [items...])] in order of first appearance: one entry when every item shares a group."""
    out: List[tuple] = []
    for it in items:
        g = group_of(it)
        for og, lst in out:
            if og is g:
                lst.append(it)
                break
        else:
            out.append((g, [it]))
    return out


def gather_slices(ids: torch.Tensor, slices: torch.Tensor, group) -> tuple:
    """Data-parallel embedding gradients: Horovod all-gathers IndexedSlices (values and indices concatenated over the ranks,
    values divided by the world size; models/base.py:476-508).  ids (T, B) int32, slices (T, B, D) ->
    (T, world*B) ids and (T, world*B, D) slices, identical on every rank."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    T, B = ids.shape
    all_ids = torch.empty((world, T, B), dtype=ids.dtype, device=ids.device)
    all_sl = torch.empty((world,) + tuple(slices.shape), dtype=slices.dtype, device=slices.device)
    dist.all_gather([all_ids[r] for r in range(world)], ids.contiguous(), group=group)
    dist.all_gather([all_sl[r] for r in range(world)], slices.contiguous(), group=group)
    return (all_ids.permute(1, 0, 2).reshape(T, world * B).contiguous(),
            all_sl.permute(1, 0, 2, 3).reshape(T, world * B, slices.shape[2]).contiguous())


class _StepTrainer:
    """What every static-buffer training step shares: the dense arena and its operand copies, the table checks and
    optimizer state, a chain of Dense layers forward and backward, the concatenating input block forward and backward,
    multi-hot pooling and its gradient expansion, the output heads, the update, CUDA-graph capture / replay, and the
    host-side bookkeeping.  A subclass sets the attributes below in its __init__ (through the _init_* methods) and
    implements forward_backward, which starts with _begin_step and leaves _idx / _slices / _bags / _b for apply_gradients:
      model, body, opt, device, B, group, world, arena, hyper, head, outputs, H, losses, loss_weights,
      _tc_layers / _wsplit (Dense layers whose split operand copies follow the updates), _wide (see _init_wide),
      feats / tables / tstate1 / tstate2 / rep / tdense / slices, oob, logits / _loss_all / loss, wk (_WideKernel)."""

    head: Optional[_Dense] = None  # the output layer; a trainer whose task builds its own targets has none
    _model_name = "this model"  # how the construction checks' messages name the model
    _onehot_only = False  # the model's input block trains one-hot features only
    # a variable trained outside the arena: a wide kernel (DeepFM, Wide&Deep) or the weight-tied item table (_TiedTable)
    wk: Optional["_WideKernel"] = None

    # ---- construction checks ------------------------------------------------------------------------------------------
    def _refuse_group(self, group) -> None:
        if group is not None:
            raise NotImplementedError(f"training {self._model_name} with a process group is not implemented")

    def _require_tc_engine(self) -> None:
        from .blocks import dense_engine

        if dense_engine() == "fp32":
            raise NotImplementedError(f"training {self._model_name} runs on the tensor-core engine (dense_engine() == 'fp32')")

    def _refuse_sharded(self, owner) -> None:
        """owner: the embeddings (or the body) that would hold a row-sharded placement."""
        if getattr(owner, "sharded", None) is not None:
            raise NotImplementedError(f"training {self._model_name} with row-sharded tables is not implemented")

    def _check_mlps(self, blocks, allow_dropout: bool = False) -> None:
        for blk in blocks:
            if not isinstance(blk, MLP) or blk.has_normalization or (blk.dropout and not allow_dropout):
                raise NotImplementedError(f"{blk.name}: training {self._model_name} supports MLPBlocks without normalization / "
                                          "dropout")

    @staticmethod
    def _check_activations(layers: Sequence[_Dense]) -> None:
        for l in layers:
            if l.activation not in ("relu", "linear"):
                raise NotImplementedError(f"{l.name}: training supports relu / linear activations, got {l.activation!r}")

    def _init_common(self, model, optimizer: Optimizer, batch_size: int, device, group) -> None:
        self.model, self.body, self.opt = model, model.body, optimizer
        self.device = torch.device(device) if device is not None else default_device()
        if not model.built:
            model.build(self.device)
        self._groups = _OptGroups(optimizer, model, self.device)
        self.B = int(batch_size)
        self.group = group
        self.world = 1
        if group is not None:
            import torch.distributed as dist

            self.world = dist.get_world_size(group)

    @property
    def hyper(self) -> torch.Tensor:
        """The first optimizer group's device hyper-parameters (every group's step counter moves together)."""
        return self._groups.groups[0].hyper

    def _init_heads(self) -> None:
        self.head = self.model.prediction.to_call
        self.outputs = self.model.output_blocks()
        self.H = len(self.outputs)
        self.losses = [o.loss for o in self.outputs]
        self.loss_weights = list(getattr(self.model, "loss_weights", None) or [1.0] * self.H)

    def _init_wide(self, needs_dgrad, dz_split_given=lambda li: False) -> None:
        """Layers wider than mm_dense_dgrad's 128 units take dX = dZ W^T through the tensor-core forward GEMM on the
        transposed kernel: per such layer of _tc_layers (index li with needs_dgrad(li)) a transposed copy, its split
        operand and, unless the caller passes dZ's split to _dgrad (dz_split_given(li)), the split of dZ."""
        self._wide: Dict[int, dict] = {}
        for li, l in enumerate(self._tc_layers):
            if l.units > 128 and needs_dgrad(li):
                K, N = l.kernel.shape
                wT = torch.empty((N, K), dtype=torch.float32, device=self.device)
                dzs = None if dz_split_given(li) else torch.zeros((self.B, 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=self.device)
                self._wide[li] = dict(wT=wT, wT_split=torch.zeros((ops.tc_padded_n(K), 2 * ops.tc_padded_k(N)), dtype=torch.bfloat16, device=self.device),
                                      dz_split=dzs)

    def _init_dense(self, tc_layers: Sequence[_Dense], fused_layers: Sequence[_Dense]) -> None:
        """One arena over tc_layers (run by mm_dense_tc: each gets a split operand copy that follows the updates) and
        fused_layers (read as fp32 by a fused kernel), and the optimizer's hyper-parameters in device memory."""
        layers = list(tc_layers) + list(fused_layers)
        self.arena = DenseArena(layers, [self._groups.of(l) for l in layers], self.device)
        self._tc_layers = list(tc_layers)
        self._wsplit = [ops.split_weights(l.kernel) for l in self._tc_layers]
        for l, ws in zip(self._tc_layers, self._wsplit):
            l._w_split = ws  # the model's forward keeps reading the refreshed operand copies

    def _init_tables(self, feats: Sequence[str], tables: Sequence, check_width: bool = True) -> None:
        """feats / tables (one table per feature, by position) after the checks every sparse update needs, their
        optimizer state, and the table positions of every embedding width."""
        seen = set()
        for f, t in zip(feats, tables):
            if id(t) in seen:
                raise NotImplementedError(f"feature {f!r}: training with a table shared between features is not implemented")
            seen.add(id(t))
            if not t.trainable:
                raise NotImplementedError(f"feature {f!r}: frozen embedding tables are not implemented in the training step")
            D = t.table.shape[1]
            if check_width and (D % 4 or D > 128):
                raise NotImplementedError(f"table {t.table_name!r}: embedding width {D} is not supported by the sparse update "
                                          "(it needs a multiple of 4 no larger than 128)")
        self.feats, self.tables = list(feats), list(tables)
        self.tgroup = [self._groups.of(t) for t in self.tables]
        self.rep = [ops.fill_i32(torch.empty(t.table.shape[0], dtype=torch.int32, device=self.device), INT32_MAX) for t in self.tables]
        self.tstate1 = [torch.full_like(t.table, g.initial_accumulator_value) if g.slots >= 1 else None
                        for t, g in zip(self.tables, self.tgroup)]
        self.tstate2 = [torch.zeros_like(t.table) if g.slots >= 2 else None for t, g in zip(self.tables, self.tgroup)]
        # tables with few rows (every id repeats many times per batch) sum their slices into a dense accumulator
        self.tdense = [torch.zeros_like(t.table) if t.table.shape[0] <= DENSE_PATH_MAX_ROWS else None for t in self.tables]
        self._by_width: Dict[int, List[int]] = {}
        for t, tb in enumerate(self.tables):
            self._by_width.setdefault(tb.table.shape[1], []).append(t)
        # multi-hot features (ragged bags, (B, L) id matrices), by table position: the expanded row gradients and the
        # update's ids, created on the first batch that carries the feature as a bag (see _pool_bag)
        self._bag_bufs: Dict[int, dict] = {}
        self._bags: Dict[int, dict] = {}

    def _init_inputs(self, parts: Sequence["_ConcatInput"]) -> None:
        """_init_tables over the features of the input parts, in order (each part learns its features' table
        positions), and every table's (B, D) IndexedSlices buffer."""
        feats, tables = [], []
        for p in parts:
            p.tidx = list(range(len(feats), len(feats) + len(p.feats)))
            feats += p.feats
            tables += [p.emb.feature_to_table[f] for f in p.feats]
        self._init_tables(feats, tables)
        self.slices = [torch.zeros((self.B, t.table.shape[1]), dtype=torch.float32, device=self.device) for t in self.tables]

    def _chain_buffers(self, layers: Sequence[_Dense], split_last: bool = False) -> tuple:
        """(h, h_split, dh) of a chain of Dense layers: the fp32 activations, the split operand every layer but the last
        (split_last: every layer) emits for the layer that reads it, and the pre-activation gradients."""
        f32 = dict(dtype=torch.float32, device=self.device)
        h = [torch.zeros((self.B, l.units), **f32) for l in layers]
        h_split = [torch.zeros((self.B, 2 * ops.tc_padded_k(l.units)), dtype=torch.bfloat16, device=self.device)
                   for l in (layers if split_last else layers[:-1])]
        dh = [torch.zeros((self.B, l.units), **f32) for l in layers]
        return h, h_split, dh

    def _init_loss(self, B: int) -> None:
        f32 = dict(dtype=torch.float32, device=self.device)
        self.logits = torch.zeros((self.H, B) if self.H > 1 else B, **f32)  # z of each output; (B,) for one
        # [total, loss_0 .. loss_{H-1}]; `loss` is the (1,) total alone for one output, the whole vector for several
        self._loss_all = torch.zeros(1 + self.H, **f32)
        self.loss = self._loss_all if self.H > 1 else self._loss_all[:1]
        self.steps = 0
        self._graph = None
        self._static: Optional[Dict[str, torch.Tensor]] = None
        self._static_y: Optional[List[torch.Tensor]] = None

    def _check_batch(self, b: int) -> None:
        if b > self.B or b < 1:
            raise ValueError(f"this trainer was compiled for batches of up to {self.B} samples, got {b}")

    def _check_targets(self, targets, b: int) -> list:
        self._check_batch(b)
        targets = list(targets) if isinstance(targets, (list, tuple)) else [targets]
        if len(targets) != self.H:
            raise ValueError(f"{self.H} target tensors expected (one per output), got {len(targets)}")
        for o, t in zip(self.outputs, targets):
            if t.numel() != b:
                raise ValueError(f"targets of {o.name!r} must hold {b} values, got {tuple(t.shape)}")
        return targets

    def _begin_step(self, inputs, targets, sample_weight) -> tuple:
        """What every forward_backward starts with: the loss zeroed, the batch size b checked (and the targets against it,
        unless the task builds its own), the step's ids / slices / bags reset.  Returns (b, targets as a list,
        sample_weight), a single output's sample_weight taken out of its list."""
        self._loss_all.zero_()
        b = batch_size_of(inputs)
        if self.head is None:
            self._check_batch(b)
        else:
            targets = self._check_targets(targets, b)
        if self.H == 1 and isinstance(sample_weight, (list, tuple)):
            sample_weight = sample_weight[0]
        self._idx: List[Optional[torch.Tensor]] = [None] * len(self.tables)
        self._slices = [s[:b] for s in self.slices]
        self._bags = {}
        return b, targets, sample_weight

    def _heads(self, x: torch.Tensor, targets, dx: torch.Tensor, mask_relu: bool, sample_weight, b: int) -> None:
        """The output heads' forward, loss and backward: logits, loss, dx and the head's gradients in the arena."""
        a, hi = self.arena, len(self.arena.layers) - 1
        ops.heads_fwd_bwd(x, self.head.kernel, self.head.bias, self.losses, [t.reshape(-1) for t in targets],
                          self.logits.view(-1)[:self.H * b].view(self.H, b),
                          self._loss_all, dx, a.view(a.grad, hi, "kernel"), a.view(a.grad, hi, "bias"), loss_weights=self.loss_weights,
                          mask_relu=mask_relu, sample_weight=sample_weight)

    def _dgrad(self, li: int, layer: _Dense, dz: torch.Tensor, dx: torch.Tensor, mask: Optional[torch.Tensor],
               dz_split: Optional[torch.Tensor] = None) -> None:
        """dx = dz W^T (zeroed where mask <= 0) for layer `li` of _tc_layers.  dz_split: dz's split operand when it exists
        already (wide layers only)."""
        wide = self._wide.get(li)
        if wide is None:
            ops.dense_dgrad(dz, layer.kernel, dx, mask=mask)
            return
        K, N = layer.kernel.shape
        b = dz.shape[0]
        wide["wT"].copy_(layer.kernel.t())
        ops.split_weights(wide["wT"], out=wide["wT_split"])
        if dz_split is None:
            dz_split = wide["dz_split"][:b]
            ops.split_rows(dz, out=dz_split)
        ops.dense_tc(dz_split, N, wide["wT_split"], K, None, None, out_f32=dx)
        if mask is not None:
            ops.relu_mask(dx, mask)

    def _table_args(self, t: int, indices: torch.Tensor, grad_rows: torch.Tensor) -> dict:
        tb = self.tables[t]
        mirror = tb._mirror if (tb._mirror is not None and tb._mirror.shape[0] == tb.table.shape[0]) else None
        return dict(weights=tb.table, indices=indices, grad_rows=grad_rows, rep_map=self.rep[t], state1=self.tstate1[t],
                    state2=self.tstate2[t], mirror=mirror, dense_grad=self.tdense[t])

    # ---- a chain of Dense layers (layers li0 .. of _tc_layers) on b-row views of _chain_buffers -----------------------
    def _chain_forward(self, op: torch.Tensor, K: int, li0: int, layers, h, h_split, drop=None) -> None:
        """The chain on the split operand `op` of its (b, K) input: fp32 activations into h, each layer's split output
        (where h_split has one) into the operand of the next.  drop: per layer None or ops.dense_tc's dropout tuple."""
        for i, l in enumerate(layers):
            nxt = h_split[i] if i < len(h_split) else None
            ops.dense_tc(op, K, self._wsplit[li0 + i], l.units, l.bias, l.activation, out_f32=h[i], out_split=nxt,
                         dropout=None if drop is None else drop[i])
            op, K = nxt, l.units

    def _chain_backward(self, li0: int, layers, h, dh, first_in, dx: Optional[torch.Tensor], drop_scale=None) -> None:
        """From dh[-1] (the pre-activation gradient of the last layer) down: per layer dW, db into the arena and the input
        gradient with the relu mask of the layer below.  first_in: the chain's input, as (split operand, K) or as an fp32
        matrix; dx: where the first layer's input gradient goes (None: nothing below needs it).  drop_scale: per layer
        None or the (units,) vector 1 / (1 - rate) of a relu layer with dropout: its saved output is zero where the mask
        dropped, so the relu mask applies the dropout mask too and only the scale is left (dh[-1] comes scaled)."""
        a = self.arena
        for i in range(len(layers) - 1, 0, -1):
            ops.dense_wgrad(h[i - 1], dh[i], a.view(a.grad, li0 + i, "kernel"), a.view(a.grad, li0 + i, "bias"))
            self._dgrad(li0 + i, layers[i], dh[i], dh[i - 1], h[i - 1] if layers[i - 1].activation == "relu" else None)
            if drop_scale is not None and drop_scale[i - 1] is not None:
                ops.scale_shift(dh[i - 1], drop_scale[i - 1], self._drop_zero[: dh[i - 1].shape[1]], out=dh[i - 1])
        if isinstance(first_in, tuple):
            ops.dense_wgrad_split(first_in[0], first_in[1], dh[0], a.view(a.grad, li0, "kernel"), a.view(a.grad, li0, "bias"))
        else:
            ops.dense_wgrad(first_in, dh[0], a.view(a.grad, li0, "kernel"), a.view(a.grad, li0, "bias"))
        if dx is not None:
            self._dgrad(li0, layers[0], dh[0], dx, None)

    # ---- multi-hot features -----------------------------------------------------------------------------------------
    def _pool_bag(self, t: int, f: str, x, kind: str, out: torch.Tensor, col: int) -> None:
        """The forward's combiner over the rows of multi-hot feature f (table t) into out[:, col:col+D], and in _bags[t]
        what the backward needs: the ids, the buffer of the expanded row gradients and the update's ids."""
        tb = self.tables[t]
        D = tb.table.shape[1]
        comb = tb.sequence_combiner or "mean"
        if comb == "max":
            raise NotImplementedError(f"feature {f!r}: training with the 'max' sequence combiner is not implemented")
        buf = self._bag_bufs.setdefault(t, dict(rows=None, ids=None))
        if kind == "bag":
            values, offsets = x
            ids, offs = ops.as_index(values).reshape(-1), ops.as_index(offsets)
            ops.gather_bag(tb.table, ids, offs, comb, out, col, self.oob)
        else:
            if comb == "sqrtn":
                raise ValueError(f"feature {f!r}: sequence_combiner 'sqrtn' is only defined for ragged inputs")
            ids, offs = ops.as_index(x).reshape(x.shape[0], -1).contiguous(), None
            ops.gather_seq(tb.table, ids, comb, out, col, self.oob)
        nnz = ids.numel()
        if buf["rows"] is None or buf["rows"].shape[0] < nnz:  # ragged: grows to the largest batch; fixed length: b * L
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"feature {f!r}: the expanded gradient buffer cannot grow during graph capture")
            buf["rows"] = torch.empty((nnz, D), dtype=torch.float32, device=self.device)
        if kind == "bag" and (buf["ids"] is None or buf["ids"].shape[0] < nnz or buf["ids"].dtype != ids.dtype):
            # the update's indices: a ragged batch's offsets need not cover every value (offsets[0] > 0, offsets[B] < nnz);
            # the expansion marks such positions -1 so that no row the batch does not hold is updated
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"feature {f!r}: the expanded id buffer cannot grow during graph capture")
            buf["ids"] = torch.empty(max(nnz, 1), dtype=ids.dtype, device=self.device)
        self._bags[t] = dict(ids=ids, offsets=offs, comb=comb, rows=buf["rows"][:nnz],
                             apply_ids=buf["ids"][:nnz] if kind == "bag" else ids.reshape(-1))

    def _bag_grads(self) -> None:
        """Pooled-row gradient (the feature's slice of the backward) -> one scaled row per id."""
        for t, bg in self._bags.items():
            ops.bag_grad_rows(self._slices[t], bg["ids"], bg["offsets"], self.tables[t].table.shape[0], bg["comb"], bg["rows"],
                              out_ids=bg["apply_ids"] if bg["offsets"] is not None else None)

    # ---- the update ---------------------------------------------------------------------------------------------------
    def _gradients_to_apply(self) -> tuple:
        """(ids per table, slices per table, rows per slice, scale of the dense gradient) of the last forward_backward."""
        return self._idx, self._slices, self._b, 1.0

    def apply_gradients(self) -> None:
        """Each optimizer group's tick, then mm_dense_apply per run of the arena that one group owns (the whole arena for
        one optimizer), mm_sparse_rows_apply per (embedding width, group), the wide kernel or tied table."""
        a = self.arena
        for g in self._groups.groups:
            g.tick()
        idx, slices, rows, scale = self._gradients_to_apply()
        for s, e, g in a.runs:  # a model without Dense layers (matrix factorization) has an empty arena
            ops.dense_apply(g.kind, a.w[s:e], a.grad[s:e], a.state1[s:e] if g.slots >= 1 else None,
                            a.state2[s:e] if g.slots >= 2 else None, g.hyper, grad_scale=scale)
        for D, ts in self._by_width.items():
            for g, onehot in _by_group([t for t in ts if t not in self._bags], lambda t: self.tgroup[t]):
                for s in range(0, len(onehot), SPARSE_MAX_TABLES):
                    chunk = onehot[s:s + SPARSE_MAX_TABLES]
                    ops.sparse_rows_apply(g.kind, [self._table_args(t, idx[t], slices[t]) for t in chunk], rows, D, g.hyper)
            for t in ts:
                bag = self._bags.get(t)
                if bag is not None and bag["rows"].shape[0] > 0:  # a multi-hot table: its own call over the nnz expanded rows
                    g = self.tgroup[t]
                    tab = self._table_args(t, bag["apply_ids"], bag["rows"])
                    ops.sparse_rows_apply(g.kind, [tab], bag["rows"].shape[0], D, g.hyper)
        if self.wk is not None:
            self.wk.apply()
        self._refresh_operands()

    def _refresh_operands(self) -> None:
        for l, ws in zip(self._tc_layers, self._wsplit):
            ops.split_weights(l.kernel, out=ws)

    def step(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> torch.Tensor:
        """One eager training step; returns [total loss, per-output losses...] as a (1 + H,) device tensor (valid until the
        next step)."""
        self.forward_backward(inputs, targets, sample_weight)
        self.apply_gradients()
        self._after_step()
        return self.loss

    def _after_step(self) -> None:
        from .core import bump_weights_version

        self.steps += 1
        if self.head is not None:
            self.head._bias_host = None
        bump_weights_version()  # forward graphs captured earlier hold scalars / operand copies of the old variables

    # ---- CUDA-graph replay over static input buffers ------------------------------------------------------------
    def capture(self, inputs: Dict[str, torch.Tensor], targets: torch.Tensor, clone: bool = True) -> None:
        """Capture forward + backward + update into ONE CUDA graph over copies of `inputs` / `targets` (single GPU; with a
        process group the collectives stay eager between two graphs).  clone=False: the given tensors ARE the static
        buffers (e.g. views of one packed device buffer that a single H2D copy refreshes before replay())."""
        if self.world > 1:
            raise NotImplementedError("graph capture of the data-parallel step is not implemented")
        for f in self.feats:
            if isinstance(get_feature(inputs, f), tuple):
                raise NotImplementedError(f"graph capture with the ragged feature {f!r} is not implemented: its number of ids "
                                          "changes from batch to batch (train it eagerly, or feed it as a fixed-length (B, L) matrix)")
        self._static = {k: (v.clone() if clone else v) for k, v in inputs.items()}
        ys = list(targets) if isinstance(targets, (list, tuple)) else [targets]
        self._static_y = [y.clone() if clone else y for y in ys]
        self.model.defer_index_check(True)
        try:
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            # warm-up steps DO train: snapshot and restore every variable so that capture has no side effect
            snap = self._snapshot()
            with torch.cuda.stream(s):
                for _ in range(2):
                    self.forward_backward(self._static, self._static_y)
                    self.apply_gradients()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self._graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count()
            with graph_capture(self._graph):
                self.forward_backward(self._static, self._static_y)
                self.apply_gradients()
            self.launches_per_step = ops.launch_count() - n0
            self._restore(snap)
        finally:
            self.model.defer_index_check(False)

    def _state(self) -> Dict[str, Optional[torch.Tensor]]:
        """Every variable a step changes, by name: the arena's w / s1 / s2, the hyper-parameters (the step counter), each
        table and its optimizer slots, and the wide kernel's; None where an optimizer has no such slot."""
        a = self.arena
        state = dict(w=a.w, s1=a.state1, s2=a.state2, hyper=self.hyper)
        state.update({f"hyper{i}": g.hyper for i, g in enumerate(self._groups.groups) if i})
        for t, (tb, s1, s2) in enumerate(zip(self.tables, self.tstate1, self.tstate2)):
            state.update({f"table{t}": tb.table, f"table{t}/s1": s1, f"table{t}/s2": s2})
        if self.wk is not None:
            state.update(self.wk.state())
        return state

    def _snapshot(self) -> Dict[str, Optional[torch.Tensor]]:
        return {k: None if v is None else v.clone() for k, v in self._state().items()}

    def _restore(self, snap) -> None:
        for k, dst in self._state().items():
            if dst is not None:
                dst.copy_(snap[k])
        self.arena.grad.zero_()
        if self.wk is not None:
            self.wk.grad.zero_()
        for t in self.tables:
            if t._mirror is not None and t._mirror.shape[0] == t.table.shape[0]:
                ops.split_rows(t.table, out=t._mirror)
        self._refresh_operands()

    def replay(self, inputs: Optional[Dict[str, torch.Tensor]] = None, targets: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self._graph is None:
            raise RuntimeError("capture() first")
        if inputs is not None:
            for k, v in self._static.items():
                v.copy_(inputs[k], non_blocking=True)
        if targets is not None:
            ys = list(targets) if isinstance(targets, (list, tuple)) else [targets]
            for s, y in zip(self._static_y, ys):
                s.copy_(y.reshape(s.shape), non_blocking=True)
        self._graph.replay()
        self._after_step()
        return self.loss

    def check_indices(self) -> None:
        """Raise IndexError if any batch since the last check carried an id outside its table (the forward read a zero
        row for it and its gradient was dropped).  One device-to-host read: `fit` calls it once per epoch, not per step."""
        if self.oob is None:
            return
        n = int(self.oob.item())
        if n:
            self.oob.zero_()
            raise IndexError(f"{n} indices out of range for the embedding tables "
                             "(TF raises InvalidArgumentError: indices[...] is not in [0, rows))")

    def set_learning_rate(self, lr: float) -> None:
        if len(self._groups.groups) > 1 or self._groups.groups[0].sched is not None:
            raise NotImplementedError("set_learning_rate: the learning rates of a MultiOptimizer or a schedule are set by "
                                      "their optimizers (schedules move on the device)")
        self.opt.learning_rate = float(lr)
        self.hyper[_cabi.HYPER_LR] = float(lr)

    def gradients(self) -> Dict[str, torch.Tensor]:
        """Dense gradients by variable name (after forward_backward, before apply_gradients) — for parity tests."""
        out = {}
        for i, l in enumerate(self.arena.layers):
            out[f"{l.name}/kernel"] = self.arena.view(self.arena.grad, i, "kernel")
            b = self.arena.view(self.arena.grad, i, "bias")
            if b is not None:
                out[f"{l.name}/bias"] = b
        return out


class _ConcatInput:
    """A trainer's concatenating input block (InputBlockV2): x0 (B, d) = [embedding rows | continuous columns] at their
    sorted-name offsets `cols`, its split operand xs and, for a caller that needs the input gradient, dx0 (None without
    tables).  feats: the features it gathers, by default every feature of the block's embeddings, at the trainer's table
    positions tidx (set by _init_inputs); cont: its continuous columns, by default in sorted-name order; cols: the
    features' column offsets, by default the block's sorted-name layout."""

    def __init__(self, tr: _StepTrainer, ib, dx0: bool = False, feats: Optional[Sequence[str]] = None,
                 cont: Optional[Sequence[str]] = None, cols: Optional[Dict[str, int]] = None, pretrained_ok: bool = False):
        self.tr = tr
        self.emb = ib.embeddings
        self.cols, _, self.d = ib.layout()
        # pretrained features (PretrainedEmbeddings): gathered, or gathered and projected, into their slots of x0
        self.pre = getattr(ib, "pretrained", None)
        self.pslots = list(self.pre.branches.values()) if self.pre is not None else []
        if self.pslots and not pretrained_ok:
            raise NotImplementedError(f"training {tr._model_name} with pretrained embeddings (PretrainedEmbeddings) is not "
                                      "implemented")
        self.proj_layers = [br.projection for br in self.pslots if br.projection is not None]
        if cols is not None:  # an explicit column offset per feature instead of the sorted-name concat (NCF's [item | query])
            dims = self.emb.output_dims()
            self.cols, self.d = dict(cols), max(c + dims[f] for f, c in cols.items())
        if feats is None:
            feats = self.emb.feature_names if self.emb is not None else []
        if cont is None:
            cont = sorted(ib.continuous.features) if ib.continuous is not None else []
        self.feats, self.cont = list(feats), list(cont)
        self.tidx: List[int] = []
        # embeddings_l2_reg per feature (set by a trainer that applies it) and mm_concat_backward_l2's partials
        self.l2_reg: List[float] = [0.0] * len(self.feats)
        self.l2_ws: Optional[torch.Tensor] = None
        ids_owner = self.emb if self.emb is not None else getattr(ib, "pretrained_ids", None)
        self.oob = ids_owner.counter(tr.device) if ids_owner is not None else None
        f32 = dict(dtype=torch.float32, device=tr.device)
        self.x0 = torch.zeros((tr.B, _ld4(self.d)), **f32)
        self.xs = torch.zeros((tr.B, 2 * ops.tc_padded_k(self.d)), dtype=torch.bfloat16, device=tr.device)
        self.dx0 = torch.zeros((tr.B, _ld4(self.d)), **f32) if dx0 and (self.feats or self.proj_layers) else None
        # per projected slot: the pre-norm projection (l2-normalised slots) and the backward's workspace
        self.ypre = [torch.zeros((tr.B, br.width), **f32) if br.projection is not None and br.l2 else None for br in self.pslots]
        self.pws = [ops.pretrained_backward_workspace(tr.B, br.dim, br.width, tr.device) if br.projection is not None else None
                    for br in self.pslots]
        self._psrc: List[tuple] = [None] * len(self.pslots)

    def check_multihot_widths(self, schema) -> None:
        """Refuse a list feature whose table the multi-hot gradient expansion (mm_bag_grad_rows) cannot serve."""
        for f in self.feats:
            col, t = schema.get(f), self.emb.feature_to_table[f]
            if col is not None and col.is_list and t.dim not in (16, 32, 64, 128):
                raise NotImplementedError(f"feature {f!r}: training a multi-hot feature needs an embedding width of 16, 32, 64 "
                                          f"or 128, got {t.dim} (give its table one with Embeddings(dim=...))")

    def views(self, b: int) -> tuple:
        """(x0, xs, dx0) on the leading b rows."""
        return self.x0[:b, :self.d], self.xs[:b], None if self.dx0 is None else self.dx0[:b, :self.d]

    def forward(self, inputs, b: int) -> tuple:
        """The features' rows and the continuous columns into x0, and x0's split operand xs; returns views(b).  One-hot
        features share one mm_gather_multi, a multi-hot feature is pooled straight into its columns (_pool_bag).  Leaves
        the update's ids in the trainer's _idx (None for a multi-hot feature)."""
        tr = self.tr
        x0, xs, dx0 = self.views(b)
        ts, ids = [], []
        for t, f in zip(self.tidx, self.feats):
            x = get_feature(inputs, f)
            kind = tr.tables[t].lookup_kind(x)
            if kind == "onehot":
                ts.append(t)
                ids.append(ops.as_index(x).reshape(-1))
            elif tr._onehot_only:
                raise NotImplementedError(f"feature {f!r}: training {tr._model_name} on multi-hot / ragged features "
                                          "is not implemented")
            else:
                tr._pool_bag(t, f, x, kind, x0, self.cols[f])
        if ts:
            if len({i.dtype for i in ids}) > 1:  # one launch reads one index dtype
                ids = [i.to(torch.int64) for i in ids]
            ops.gather_multi([tr.tables[t].table for t in ts], ids, [self.cols[tr.feats[t]] for t in ts], x0, tr.oob)
            for t, i in zip(ts, ids):
                tr._idx[t] = i
        if self.cont:
            ops.concat_columns([inputs[n] for n in self.cont], x0, [self.cols[n] for n in self.cont])
        for i, br in enumerate(self.pslots):
            P, ids = self._psrc[i] = self.pre.source(inputs, br.name)
            slot = x0[:, self.cols[br.name]:self.cols[br.name] + br.width]
            if br.projection is None:
                ops.pretrained_gather(P, ids, slot, self.oob)
            else:
                y = slot if self.ypre[i] is None else self.ypre[i][:b]
                ops.pretrained_project(P, ids, br.projection.kernel, br.projection.bias, y, self.oob)
                if y is not slot:
                    ops.l2_normalize(y, out=slot)
                continue
            if br.l2:
                ops.l2_normalize(slot, out=slot)
        ops.split_rows(x0, out=xs)
        return x0, xs, dx0

    def set_l2_reg(self, l2: float) -> None:
        """Apply embeddings_l2_reg = l2 to every table of the block: its gradient joins the backward, the term the loss."""
        self.l2_reg = [float(l2)] * len(self.feats)
        if l2 and self.l2_ws is None:
            self.l2_ws = ops.concat_l2_workspace(min(len(self.feats), CONCAT_MAX_SLICES), self.tr.device)

    def backward(self, addends, b: int, fm: Optional[torch.Tensor] = None) -> None:
        """The tables' columns of the summed (b, d) addends into each table's slice of the trainer's _slices; fm: the FM
        term's ds (b,), whose input gradient from x0 is added (mm_fm_concat_backward).  Tables with an L2 factor also get
        2 l2 x0 (mm_concat_backward_l2), and the term goes into the trainer's loss vector [total, regularization]."""
        tr = self.tr
        slices = [(tr._slices[t], self.cols[f]) for t, f in zip(self.tidx, self.feats)]
        for s in range(0, len(slices), CONCAT_MAX_SLICES):
            l2 = self.l2_reg[s:s + CONCAT_MAX_SLICES]
            if fm is not None:
                ops.fm_concat_backward(addends, self.x0[:b, :self.d], fm, slices[s:s + CONCAT_MAX_SLICES])
            elif any(l2):
                ops.concat_backward_l2(addends, slices[s:s + CONCAT_MAX_SLICES], self.x0[:b, :self.d], l2, tr._loss_all[:2],
                                       self.l2_ws)
            else:
                ops.concat_backward(addends, slices[s:s + CONCAT_MAX_SLICES])
        a = tr.arena
        for i, br in enumerate(self.pslots):  # a projection's dW, db from its slot's columns; nothing flows into P
            if br.projection is None:
                continue
            c, li = self.cols[br.name], a.layers.index(br.projection)
            P, ids = self._psrc[i]
            ops.pretrained_project_backward(P, ids, [x[:, c:c + br.width] for x in addends], a.view(a.grad, li, "kernel"),
                                            a.view(a.grad, li, "bias"), ypre=None if self.ypre[i] is None else self.ypre[i][:b],
                                            workspace=self.pws[i])


class _WideKernel:
    """A wide Dense(1) (DeepFM's FM wide term, Wide&Deep's wide branch) trained outside the arena: its kernel (W, 1) stays
    where it is, one row per category of every feature (and per continuous column), with its bias' and its own optimizer
    slots beside it, the accumulator and representative map of mm_wide_rows_apply, and `grad` = [the continuous rows'
    gradients..., the bias' gradient] that the head kernel accumulates.  The trainer's forward_backward leaves in `calls`
    the step's gradient as (ids per block, rows per block, kernel offset per block, gradient values) groups."""

    def __init__(self, tr: _StepTrainer, dense: _Dense, cont_offsets: Sequence[int] = ()):
        self.tr, self.dense = tr, dense
        self.cont_offsets = list(cont_offsets)
        self.group = opt = tr._groups.of(dense)
        f32 = dict(dtype=torch.float32, device=tr.device)
        W = dense.kernel.numel()
        nb = 1 if dense.bias is not None else 0
        self.wk_s1 = torch.full((W,), opt.initial_accumulator_value, **f32) if opt.slots >= 1 else None
        self.wk_s2 = torch.zeros(W, **f32) if opt.slots >= 2 else None
        self.wb_s1 = torch.full((nb,), opt.initial_accumulator_value, **f32) if opt.slots >= 1 and nb else None
        self.wb_s2 = torch.zeros(nb, **f32) if opt.slots >= 2 and nb else None
        self.acc = torch.zeros(W, **f32)
        self.rep = ops.fill_i32(torch.empty(W, dtype=torch.int32, device=tr.device), INT32_MAX)
        self.grad = torch.zeros(len(self.cont_offsets) + nb, **f32)
        self.calls: List[tuple] = []

    def state(self) -> Dict[str, Optional[torch.Tensor]]:
        return {"wide/kernel": self.dense.kernel, "wide/bias": self.dense.bias, "wide/kernel/s1": self.wk_s1,
                "wide/kernel/s2": self.wk_s2, "wide/bias/s1": self.wb_s1, "wide/bias/s2": self.wb_s2}

    def apply(self) -> None:
        """One mm_wide_rows_apply per group of `calls`; the continuous rows and the bias take their step with the first."""
        wk, bias = self.dense.kernel.reshape(-1), self.dense.bias
        for i, (ids, rows, offs, g) in enumerate(self.calls):
            first = i == 0
            ops.wide_rows_apply(self.group.kind, wk, self.wk_s1, self.wk_s2, ids, rows, offs, g, self.acc, self.rep,
                                self.cont_offsets if first else [], self.grad if first and self.grad.numel() else None,
                                bias.reshape(-1) if first and bias is not None else None, self.wb_s1 if first else None,
                                self.wb_s2 if first else None, self.group.hyper)

    def gradients(self) -> Dict[str, torch.Tensor]:
        """The kernel's gradient (W, 1) and the bias' (after forward_backward, before apply_gradients), assembled in float64
        from `calls` and `grad` — for parity tests."""
        W = self.dense.kernel.numel()
        g = torch.zeros(W, dtype=torch.float64, device=self.tr.device)
        for ids, rows, offs, vals in self.calls:
            v = vals.double()
            for i, r, o in zip(ids, rows, offs):
                i = ops.widen_index(i).reshape(-1).long()
                ok = (i >= 0) & (i < r)
                g.index_add_(0, i[ok] + o, v[ok])
        nc = len(self.cont_offsets)
        for c, o in enumerate(self.cont_offsets):
            g[o] += self.grad[c].double()
        out = {"wide/kernel": g.reshape(W, 1)}
        if self.dense.bias is not None:
            out["wide/bias"] = self.grad[nc:].double().clone()
        return out


class DLRMTrainer(_StepTrainer):
    """Static-buffer training step of a DLRM RankingModel at one batch size."""

    _model_name = "DLRMModel"

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import BinaryOutput, ParallelOutputs

        body = model.body
        if not isinstance(body, DLRM) or body.top_block is None or body.bottom_block is None:
            raise NotImplementedError("train_step is implemented for DLRMModel with bottom and top blocks")
        if not isinstance(model.prediction, (BinaryOutput, ParallelOutputs)):
            raise NotImplementedError("train_step needs BinaryOutput / RegressionOutput heads or an OutputBlock of them")
        if group is not None and isinstance(model.prediction, ParallelOutputs):
            raise NotImplementedError("training several outputs with a process group is not implemented")
        self._refuse_sharded(body)
        if not body.can_emit_split():
            raise NotImplementedError("training needs <= 32 interaction features and embedding_dim in {16, 32, 64, 128}")
        self._init_common(model, optimizer, batch_size, device, group)
        self._check_mlps((body.bottom_block, body.top_block))
        self.bottom = body.bottom_block.dense_layers
        self.top = body.top_block.dense_layers
        self._init_heads()
        self._check_activations(self.bottom + self.top)
        if self.head.input_dim > 256:
            raise NotImplementedError("the output layer's input must be <= 256 wide")
        self._init_dense(self.bottom + self.top, [self.head])
        self._init_wide(lambda li: li != 0)  # the first bottom layer needs no input gradient

        # ---- tables (their width is one of can_emit_split's)
        emb = body.embeddings
        self.slots = body.slots()
        self.D = body.embedding_dim
        self._init_tables(emb.feature_names, [emb.feature_to_table[f] for f in emb.feature_names], check_width=False)
        T, B, D = len(self.tables), self.B, self.D
        self.slices = torch.zeros((T, B, D), dtype=torch.float32, device=self.device)

        # ---- activations and gradients
        # operand-format rows for the lookup + interaction kernels (forward and backward) (D = 64, mirrors enabled): the tables' mirrors (the
        # optimizer kernels keep them in step) and the bottom vector as the last bottom layer's split output
        from .blocks import table_mirror

        self.operand_rows = bool(D == 64 and table_mirror())
        if self.operand_rows:
            for t in self.tables:
                t.operand_mirror()
        f32 = dict(dtype=torch.float32, device=self.device)
        self.K0 = len(body.continuous.features)
        self.x0_split = torch.zeros((B, 2 * ops.tc_padded_k(self.K0)), dtype=torch.bfloat16, device=self.device)
        self.h, self.h_split, self.dh = self._chain_buffers(self.bottom, split_last=self.operand_rows)
        F = len(self.slots)
        self.OW = D + F * (F - 1) // 2
        self.ldA = _ld4(self.OW)
        self.A = None if self.operand_rows else torch.zeros((B, self.ldA), **f32)
        self.dA = torch.zeros((B, self.ldA), **f32)
        self.A_split = torch.zeros((B, 2 * ops.tc_padded_k(self.OW)), dtype=torch.bfloat16, device=self.device)
        self.t, self.t_split, self.dt = self._chain_buffers(self.top)
        self._init_loss(B)
        self.oob = emb.counter(self.device)
        # multi-hot features, by table position: the pooled rows and their operand copy, created with the first bag
        self._pooled: Dict[int, dict] = {}
        self._iota: Optional[torch.Tensor] = None

    # ---- one step on device tensors ------------------------------------------------------------------------------
    def _indices(self, inputs, b: Optional[int] = None) -> List[torch.Tensor]:
        """Ids the lookup + interaction kernels read per table.  A multi-hot feature is pooled first (_pool_bag, the
        forward's combiner) into a (B, D) buffer that those kernels then read as one more table of b rows at ids 0..b-1;
        its backward returns the pooled-row gradient, which _bag_grads expands to one row per id."""
        idx: List[torch.Tensor] = []
        self._bags = {}
        for t, f in enumerate(self.feats):
            x = get_feature(inputs, f)
            kind = self.tables[t].lookup_kind(x)
            if kind == "onehot":
                idx.append(ops.fused_ids(x))
                continue
            if self.group is not None:  # gather_slices exchanges (T, B, D) slices: one row per sample and table
                raise NotImplementedError(f"feature {f!r}: training multi-hot features with a process group is not implemented")
            if b is None:  # the pooled rows and the ids that read them must agree on the batch size
                b = batch_size_of(inputs)
            buf = self._pooled.get(t)
            if buf is None:
                if self._iota is None:
                    self._iota = torch.arange(self.B, dtype=torch.int32, device=self.device)
                buf = self._pooled[t] = dict(
                    pooled=torch.zeros((self.B, self.D), dtype=torch.float32, device=self.device),
                    split=torch.zeros((self.B, 2 * ops.tc_padded_k(self.D)), dtype=torch.bfloat16, device=self.device) if self.operand_rows else None)
            pooled, split = buf["pooled"][:b], None
            self._pool_bag(t, f, x, kind, pooled, 0)
            if self.operand_rows:
                split = buf["split"][:b]
                ops.split_rows(pooled, out=split)
            self._bags[t].update(pooled=pooled, split=split)
            idx.append(self._iota[:b])
        return idx

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena and the IndexedSlices.  Batches smaller
        than the compiled size run in the leading rows of the same buffers.  targets: one tensor per output (a bare tensor
        for a single output); sample_weight: one (b,) tensor for every output, or a list with one per output."""
        nb = len(self.bottom)
        D = self.D
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)
        cont = self.body.continuous(inputs)
        pieces = [cont[k] for k in sorted(cont)]
        h, t_, dt, dh = ([x[:b] for x in bufs] for bufs in (self.h, self.t, self.dt, self.dh))
        h_split, x0_split, A_split = [x[:b] for x in self.h_split], self.x0_split[:b], self.A_split[:b]
        ops.concat_split(pieces, out=x0_split)  # the concatenated continuous columns exist only as this operand
        # -- bottom tower (operand_rows: its last layer emits the split bottom vector too)
        self._chain_forward(x0_split, self.K0, 0, self.bottom, h, h_split)
        # -- lookup + interaction (fp32 rows)
        idx = self._indices(inputs, b)
        tabs = [self._bags[t]["pooled"] if t in self._bags else tb.table for t, tb in enumerate(self.tables)]
        mirrors = [self._bags[t]["split"] if t in self._bags else tb._mirror for t, tb in enumerate(self.tables)]
        rows = [t.shape[0] for t in tabs]
        tslots = [self.slots[f] for f in self.feats]
        bslot = self.slots["bottom_block"]
        dA_view = self.dA[:b, :self.OW]
        if self.operand_rows:
            # operand-format rows in, split-bf16 operand of the top tower out: no fp32 copy of [bottom | interactions] exists
            A_view = None
            ops.dlrm_lookup_interact(mirrors, idx, tslots, rows, D, h_split[-1], bslot, A_split, self.oob, operand_rows=True)
        else:
            A_view = self.A[:b, :self.OW]
            ops.dlrm_lookup_interact(tabs, idx, tslots, rows, D, h[-1], bslot, A_view, self.oob)
            ops.split_rows(A_view, out=A_split)
        # -- top tower
        self._chain_forward(A_split, self.OW, nb, self.top, t_, [x[:b] for x in self.t_split])
        # -- output layer + loss, forward and backward
        self._heads(t_[-1], targets, dt[-1], self.top[-1].activation == "relu", sample_weight, b)
        # -- top tower backward: its input exists as fp32 only without operand_rows
        self._chain_backward(nb, self.top, t_, dt, (A_split, self.OW) if A_view is None else A_view, dA_view)
        # -- interaction + lookup backward
        if self.operand_rows:
            ops.dlrm_interact_backward(mirrors, idx, tslots, rows, D, h_split[-1], bslot, dA_view,
                                       self._slices, dh[-1], mask_bottom=self.bottom[-1].activation == "relu", operand_rows=True)
        else:
            ops.dlrm_interact_backward(tabs, idx, tslots, rows, D, h[-1], bslot, dA_view, self._slices, dh[-1],
                                       mask_bottom=self.bottom[-1].activation == "relu")
        self._bag_grads()
        # -- bottom tower backward
        self._chain_backward(0, self.bottom, h, dh, (x0_split, self.K0), None)
        self._idx, self._b = idx, b

    def _gradients_to_apply(self) -> tuple:
        """Data parallel: the dense gradients are summed over the ranks (and scaled by 1 / world in the update), every
        rank applies every rank's IndexedSlices."""
        if self.world == 1:
            return super()._gradients_to_apply()
        import torch.distributed as dist

        dist.all_reduce(self.arena.grad, group=self.group)
        scale = 1.0 / self.world
        ids32 = torch.stack([ops.widen_index(i).to(torch.int32) for i in self._idx])
        all_ids, all_sl = gather_slices(ids32, torch.stack(self._slices), self.group)
        all_sl.mul_(scale)
        return list(all_ids), list(all_sl), self._b * self.world, scale


class DCNTrainer(_StepTrainer):
    """Static-buffer training step of a DCN-v2 RankingModel (DCNModel, stacked or parallel body) at one batch size.

    forward   gather of every table's rows + the continuous columns into x0 (B, d) at their sorted-name offsets, its split
              operand; per cross layer mm_dense_tc (z_l = x_l W_l + b_l, fp32 saved) -> mm_cross_combine
              (x_{l+1} = x0 z_l + x_l) -> mm_split_rows (the next operand); the deep tower as in DLRM's towers
    loss      mm_heads_fwd_bwd on the deep output (stacked) or on [cross | deep] in DCNBody.branch_order() (parallel)
    backward  deep tower as DLRM's towers; per cross layer (top down) mm_cross_backward (g += p, dz = g x0 fp32 + split,
              acc += g z_l), mm_dense_wgrad_split on x_l's saved operand, p = dz W_l^T (transposed-kernel mm_dense_tc for
              d > 128); mm_concat_backward sums g + p + acc (+ the deep branch's input gradient) = dx0 into each table's
              (B, D_t) IndexedSlices buffer
    update    mm_opt_tick, mm_dense_apply over the arena [cross layers, deep layers, head], one mm_sparse_rows_apply per
              distinct embedding width, mm_split_weights refresh of the operand copies the model's forward reads."""

    _model_name = "DCNModel"
    _onehot_only = True

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .blocks import Cross
        from .models import BinaryOutput, DCNBody, ParallelOutputs

        body = model.body
        if not isinstance(body, DCNBody):
            raise NotImplementedError("DCNTrainer trains DCNModel bodies")
        if not isinstance(model.prediction, (BinaryOutput, ParallelOutputs)):
            raise NotImplementedError("train_step needs BinaryOutput / RegressionOutput heads or an OutputBlock of them")
        self._refuse_group(group)
        cross_layers = body.cross.cross_layers
        for c in cross_layers:
            if not isinstance(c, Cross) or c.low_rank_dim is not None:
                raise NotImplementedError(f"{c.name}: training a low-rank cross layer (low_rank_dim) is not implemented")
        if body.cross.inputs is not None:
            raise NotImplementedError("training a CrossBlock with its own `inputs` block is not implemented")
        self._check_mlps([body.deep])
        ib = body.input_block
        if getattr(ib, "aggregation", "concat") != "concat":
            raise NotImplementedError("training DCNModel needs the concatenating input block")
        self._init_common(model, optimizer, batch_size, device, None)
        self.stacked = bool(body.stacked)
        self.cross = [c.dense for c in cross_layers]
        self.deep = body.deep.dense_layers
        self._init_heads()
        self._check_activations(self.deep)
        self.inp = _ConcatInput(self, ib, pretrained_ok=True)
        self._init_inputs([self.inp])
        d = self.inp.d

        self._init_dense(self.cross + self.deep, self.inp.proj_layers + [self.head])
        # every layer needs its input gradient (x0 is the tables' rows); mm_cross_backward writes the split of a cross
        # layer's dz itself
        L = len(self.cross)
        self._init_wide(lambda li: True, dz_split_given=lambda li: li < L)

        # ---- activations and gradients (fp32 (B, d) buffers with a row stride that is a multiple of 4)
        B = self.B
        f32 = dict(dtype=torch.float32, device=self.device)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        Kp = ops.tc_padded_k(d)

        def mat():
            return torch.zeros((B, _ld4(d)), **f32)

        # operands of x_0 (the input block's) .. x_L
        self.xs = [self.inp.xs] + [torch.zeros((B, 2 * Kp), **bf) for _ in range(L - 1 + (1 if self.stacked else 0))]
        self.z = [mat() for _ in range(L)]
        self.xf = [mat() for _ in range(min(L, 2))]  # fp32 x_1 .. x_L, alternating (only the residual of the next layer)
        self.h, self.h_split, self.dh = self._chain_buffers(self.deep)
        self.g, self.p, self.acc, self.dz = mat(), mat(), mat(), mat()
        self.dz_split = torch.zeros((B, 2 * Kp), **bf)
        if not self.stacked:
            # the head reads [cross | deep] (or [deep | cross]): x_L and the deep output are written straight into it
            u = self.deep[-1].units
            self.order = body.branch_order()
            self.coff, self.doff = (0, d) if self.order == ("cross", "deep") else (u, 0)
            self.cat = torch.zeros((B, d + u), **f32)
            self.dcat = torch.zeros((B, d + u), **f32)
            self.ddeep = mat()  # input gradient of the deep branch (an addend of dx0)
        # mm_heads_fwd_bwd reads at most 256 inputs per row.  A wider head input (a parallel body's [cross | deep] at
        # realistic d, or a wide last deep layer) takes its logits from the tensor-core GEMM; the loss kernel then runs on
        # those logits with an identity kernel (dz out, db accumulated), and dW / dX come from mm_dense_wgrad_split /
        # mm_dense_dgrad on dz.
        self.wide_head = self.head.input_dim > 256
        if self.wide_head:
            Kh = self.head.input_dim
            self._head_x_split = torch.zeros((B, 2 * ops.tc_padded_k(Kh)), **bf)
            self._head_w_split = torch.zeros((ops.tc_padded_n(self.H), 2 * ops.tc_padded_k(Kh)), **bf)
            self._head_z = torch.zeros((B, self.H), **f32)
            self._head_dz = torch.zeros((B, self.H), **f32)
            self._head_eye = torch.eye(self.H, **f32)
        self._init_loss(B)
        self.oob = self.inp.oob

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena and the IndexedSlices.  Batches smaller
        than the compiled size run in the leading rows of the same buffers."""
        a = self.arena
        d, L = self.inp.d, len(self.cross)
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)

        def v(t):
            return t[:b]

        def vd(t):
            return t[:b, :d]

        # -- input block: x0 = [embeddings | continuous] in sorted-name order, its operand xs[0]
        x0, _, _ = self.inp.forward(inputs, b)
        # -- cross network
        x = x0
        cat = v(self.cat) if not self.stacked else None
        for l, layer in enumerate(self.cross):
            ops.dense_tc(v(self.xs[l]), d, self._wsplit[l], d, layer.bias, "linear", out_f32=vd(self.z[l]))
            last = l == L - 1
            out = cat[:, self.coff:self.coff + d] if (last and cat is not None) else vd(self.xf[l % len(self.xf)])
            ops.cross_combine(x0, vd(self.z[l]), x, out)
            if l + 1 < len(self.xs):
                ops.split_rows(out, out=v(self.xs[l + 1]))
            x = out
        # -- deep tower on x_L (stacked) or x0 (parallel)
        op0 = v(self.xs[L] if self.stacked else self.xs[0])
        h, dh = [v(t) for t in self.h], [v(t) for t in self.dh]
        if cat is not None:
            h[-1] = cat[:, self.doff:self.doff + self.deep[-1].units]
        self._chain_forward(op0, d, L, self.deep, h, [v(t) for t in self.h_split])
        # -- output layer + loss, forward and backward
        relu_last = self.deep[-1].activation == "relu"
        g = vd(self.g)
        if cat is None:
            self._dcn_heads(h[-1], targets, dh[-1], relu_last, sample_weight, b)
        else:
            dcat = v(self.dcat)
            self._dcn_heads(cat, targets, dcat, False, sample_weight, b)
            dh[-1] = dcat[:, self.doff:self.doff + self.deep[-1].units]
            if relu_last:
                ops.relu_mask(dh[-1], h[-1])
            ops.concat_columns([dcat[:, self.coff:self.coff + d]], g, [0])  # the cross branch's output gradient
        # -- deep tower backward: its input gradient adds to x_L's (stacked) or is an addend of dx0 (parallel)
        self._chain_backward(L, self.deep, h, dh, (op0, d), g if self.stacked else vd(self.ddeep))
        # -- cross network backward (g: gradient into x_{l+1}; p: dgrad of the layer above)
        p, acc, dz, dzs = vd(self.p), vd(self.acc), vd(self.dz), v(self.dz_split)
        for l in range(L - 1, -1, -1):
            ops.cross_backward(x0, vd(self.z[l]), g, p if l < L - 1 else None, acc, l == L - 1, dz, dzs)
            ops.dense_wgrad_split(v(self.xs[l]), d, dz, a.view(a.grad, l, "kernel"), a.view(a.grad, l, "bias"))
            self._dgrad(l, self.cross[l], dz, p, None, dz_split=dzs)
        # -- input block backward: dx0 = g_1 + p_0 + acc (+ the deep branch's input gradient), the tables' columns only
        addends = [g, p, acc] + ([vd(self.ddeep)] if not self.stacked else [])
        self.inp.backward(addends, b)
        self._b = b

    def _dcn_heads(self, x: torch.Tensor, targets, dx: torch.Tensor, mask_relu: bool, sample_weight, b: int) -> None:
        """The output heads on x (b, K): the fused loss kernel for K <= 256, otherwise the wide-head composition."""
        if not self.wide_head:
            self._heads(x, targets, dx, mask_relu, sample_weight, b)
            return
        a, hi, K = self.arena, len(self.arena.layers) - 1, x.shape[1]
        xs, z, dz = self._head_x_split[:b], self._head_z[:b], self._head_dz[:b]
        ops.split_rows(x, out=xs)
        ops.split_weights(self.head.kernel, out=self._head_w_split)
        ops.dense_tc(xs, K, self._head_w_split, self.H, None, "linear", out_f32=z)  # x W: the logits without the bias
        ops.heads_fwd_bwd(z, self._head_eye, self.head.bias, self.losses, [t.reshape(-1) for t in targets],
                          self.logits.view(-1)[:self.H * b].view(self.H, b), self._loss_all, dz, None,
                          a.view(a.grad, hi, "bias"), loss_weights=self.loss_weights, mask_relu=False, sample_weight=sample_weight)
        ops.dense_wgrad_split(xs, K, dz, a.view(a.grad, hi, "kernel"), None)
        ops.dense_dgrad(dz, self.head.kernel, dx, mask=x if mask_relu else None)


class TwoTowerTrainer(_StepTrainer):
    """Static-buffer training step of a v1 TwoTowerModel (RetrievalModel over a TwoTowerBlock, ItemRetrievalTask with
    in-batch negatives and false negatives down-scored by the item-id column) at one batch size; a smaller batch b runs in
    the leading rows with its own b items as the negatives.  A MatrixFactorizationModel trains here too: its towers have
    no Dense layers, so a tower's output is its input block's x0 (and, without post, x0's split operand xs is what the
    in-batch kernels read), the arena is empty and neither mm_dense_apply nor mm_split_weights runs.

    The loss vector is [total, regularization]: with embeddings_l2_reg > 0 in a tower's EmbeddingOptions, the tower's
    mm_concat_backward becomes mm_concat_backward_l2, which adds 2 l2 e to the tables' IndexedSlices and l2 sum ||e||^2
    over the batch's looked-up (pooled) embeddings to both entries (the reference's EmbeddingFeatures.add_loss).

    forward   per tower: gather of its tables' rows (mm_gather_multi; ragged bags mm_gather_bag, (B, L) ids mm_gather_seq)
              and its continuous columns (mm_concat_columns) into x0 at their sorted-name offsets, its split operand, one
              mm_dense_tc per layer (fp32 activation saved + the next layer's operand); mm_l2_normalize (post="l2-norm");
              mm_split_rows of both outputs; mm_positive_scores + mm_inbatch_softmax_ce (no (b, 1+b) logits)
    backward  mm_inbatch_softmax_ce_backward (c = 1/b: Keras' mean; dpos and dneg summed into one item gradient, the loss
              accumulated on the device) — or, compiled with a pairwise loss (models_b200/losses.py), mm_inbatch_pairwise_fwd
              + mm_inbatch_pairwise_bwd in place of mm_inbatch_softmax_ce and its backward; mm_l2_normalize_backward; per tower mm_dense_wgrad[_split] + mm_dense_dgrad down to
              x0; mm_concat_backward into each table's (b, D) IndexedSlices buffer; mm_bag_grad_rows for multi-hot features
    update    mm_opt_tick, mm_dense_apply over ONE arena holding both towers, one mm_sparse_rows_apply per embedding width
              (and per multi-hot table), mm_split_weights refresh of the operand copies the model's forward reads."""

    _model_name = "a TwoTowerModel"

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import RetrievalModel
        from .retrieval import InBatchSampler, ItemRetrievalTask, L2Norm, TwoTowerBlock

        if not isinstance(model, RetrievalModel) or not isinstance(model.body, TwoTowerBlock):
            raise NotImplementedError("TwoTowerTrainer trains the v1 TwoTowerModel (a RetrievalModel over a TwoTowerBlock)")
        task = model.prediction
        if not isinstance(task, ItemRetrievalTask):
            raise NotImplementedError("training a TwoTowerModel needs the default ItemRetrievalTask")
        scorer = task.scorer
        if scorer.sampled_softmax_mode:
            raise NotImplementedError("training with sampled_softmax_mode is not implemented")
        if len(scorer.samplers) != 1 or not isinstance(scorer.samplers[0], InBatchSampler):
            raise NotImplementedError("training supports the in-batch sampler only (other samplers are not implemented)")
        if getattr(task, "logq_sampling_correction", False):
            raise NotImplementedError("the logQ sampling correction is not implemented in the training step")
        self._refuse_group(group)
        self._require_tc_engine()
        body = model.body
        if body.post is not None and not isinstance(body.post, L2Norm):
            raise NotImplementedError(f"post block {type(body.post).__name__}: only post='l2-norm' is implemented in training")
        self._init_common(model, optimizer, batch_size, device, None)
        self.task = task
        self.temperature = float(task.logits_temperature)
        self.downscore = bool(scorer.downscore_false_negatives)
        self.false_neg_score = float(scorer.false_negatives_score)
        self.item_id = scorer.item_id_feature_name
        self.l2 = body.post is not None
        self.H = 1
        self.towers, self.inps = [], []  # per tower: its layers and buffers, its input block
        for tb in (body.query, body.item):
            layers = [] if tb.mlp is None else tb.mlp.dense_layers
            if tb.mlp is not None:
                self._check_mlps([tb.mlp])
                self._check_activations(layers)
            self.towers.append(dict(name=tb.name, layers=layers))
            # a tower without tables has nothing below x0; a tower without layers hands its output gradient to the input block
            self.inps.append(_ConcatInput(self, tb.inputs, dx0=bool(layers)))
        out_w = {t["layers"][-1].units if t["layers"] else inp.d for t, inp in zip(self.towers, self.inps)}
        if len(out_w) != 1:
            raise ValueError(f"the query and item towers must end in the same width, got {sorted(out_w)}")
        self.D = out_w.pop()
        if ops.tc_padded_k(self.D) > 128:
            raise NotImplementedError(f"tower output width {self.D}: the in-batch soft-max kernels take up to 128")

        self._init_inputs(self.inps)
        for tb, inp in zip((body.query, body.item), self.inps):
            inp.set_l2_reg(getattr(getattr(tb.inputs, "embedding_options", None), "embeddings_l2_reg", 0.0))
        self._init_dense([l for t in self.towers for l in t["layers"]], [])
        first_layer = {}
        li = 0
        for t, inp in zip(self.towers, self.inps):
            t["li0"] = li
            if t["layers"]:
                first_layer[li] = bool(inp.feats)  # the first layer needs its input gradient only when the tower has tables
            li += len(t["layers"])
        self._init_wide(lambda i: first_layer.get(i, True))

        # ---- activations and gradients
        B = self.B
        f32 = dict(dtype=torch.float32, device=self.device)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        for t in self.towers:
            t["h"], t["h_split"], t["dh"] = self._chain_buffers(t["layers"])
            t["dout"] = t["dh"][-1] if t["layers"] else torch.zeros((B, self.D), **f32)  # the gradient of the tower's output
            t["y"] = torch.zeros((B, self.D), **f32) if self.l2 else None  # the normalised output
            # the in-batch kernels' operand of the output; a tower without layers or post hands them x0's split xs
            t["split"] = torch.zeros((B, 2 * ops.tc_padded_k(self.D)), **bf) if (t["layers"] or self.l2) else None
        self.pos_logit = torch.zeros(B, **f32)
        # the compiled loss: None = the soft-max cross-entropy, else a models_b200.losses.PairwiseLoss
        self.pairwise = getattr(model, "pairwise_loss", None)
        if self.pairwise is None:
            self.stats = torch.zeros((B, 3), **f32)
            ws = max(ops.catalog_workspace_bytes(min(128 * m, B), min(128 * m, B)) for m in range(1, (B + 127) // 128 + 1))
            self.ws = torch.zeros(ws, dtype=torch.uint8, device=self.device)
        else:
            self.stats = torch.zeros((B, 4), **f32)  # [row loss, dloss/dsp, lse, A] of mm_inbatch_pairwise_fwd
        self._inv_b: Dict[int, torch.Tensor] = {}  # c = 1/b per batch size, one device float each
        self._init_loss(B)
        self.loss = self._loss_all  # [total, regularization]
        self.logits = self.stats  # per row of the last step: CE [max, log-sum-exp, positive logit]; pairwise as above
        # one counter for both towers (every gather receives it), so check_indices sees every table
        self.oob = next((p.oob for p in self.inps if p.oob is not None), None)

    # ---- the parts of _StepTrainer that concern output heads do not apply: the retrieval task builds its own targets
    def capture(self, inputs: Dict[str, torch.Tensor], targets=None, clone: bool = True) -> None:
        """As _StepTrainer.capture; the targets are ignored (the task's targets are the one-hot column 0)."""
        super().capture(inputs, [], clone=clone)

    def replay(self, inputs: Optional[Dict[str, torch.Tensor]] = None, targets=None) -> torch.Tensor:
        return super().replay(inputs, None)

    def gradients(self) -> Dict[str, torch.Tensor]:
        """Dense gradients by tower-qualified variable name (after forward_backward, before apply_gradients)."""
        out = {}
        for t in self.towers:
            for j, l in enumerate(t["layers"]):
                i = t["li0"] + j
                out[f"{t['name']}/{l.name}/kernel"] = self.arena.view(self.arena.grad, i, "kernel")
                bv = self.arena.view(self.arena.grad, i, "bias")
                if bv is not None:
                    out[f"{t['name']}/{l.name}/bias"] = bv
        return out

    def table_gradients(self) -> Dict[str, tuple]:
        """{feature: (ids, rows)} of the last forward_backward: the IndexedSlices of every table before duplicates are
        summed (multi-hot features: one row per id)."""
        out = {}
        for t, f in enumerate(self.feats):
            bag = self._bags.get(t)
            if bag is None:
                out[f] = (self._idx[t], self._slices[t])
            else:
                out[f] = (bag["apply_ids"], bag["rows"])
        return out

    # ---- one step on device tensors ------------------------------------------------------------------------------
    def _scale(self, b: int) -> torch.Tensor:
        c = self._inv_b.get(b)
        if c is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("the loss scale of a new batch size cannot be created during graph capture")
            c = self._inv_b[b] = torch.full((1,), 1.0 / b, dtype=torch.float32, device=self.device)
        return c

    def _tower_forward(self, tw: dict, inp: _ConcatInput, inputs, b: int) -> tuple:
        """(the tower's (normalised) output, its split operand)."""
        x0, xs, _ = inp.forward(inputs, b)
        if not tw["layers"] and not self.l2:
            return x0, xs
        out = x0
        if tw["layers"]:
            h = [x[:b] for x in tw["h"]]
            self._chain_forward(xs, inp.d, tw["li0"], tw["layers"], h, [x[:b] for x in tw["h_split"]])
            out = h[-1]
        if self.l2:
            out = ops.l2_normalize(out, out=tw["y"][:b])
        ops.split_rows(out, out=tw["split"][:b])
        return out, tw["split"][:b]

    def _tower_backward(self, tw: dict, inp: _ConcatInput, dout: torch.Tensor, b: int) -> None:
        """dout: gradient of the tower's (normalised) output, overwritten by the pre-activation gradient of the last layer
        (without layers: by the gradient of x0)."""
        h, dh, layers = [x[:b] for x in tw["h"]], [x[:b] for x in tw["dh"]], tw["layers"]
        if not layers:
            x0, _, _ = inp.views(b)
            if self.l2:
                ops.l2_normalize_backward(x0, dout, dout)
            inp.backward([dout], b)
            return
        if self.l2:
            ops.l2_normalize_backward(h[-1], dout, dout)
        if layers[-1].activation == "relu":
            ops.relu_mask(dout, h[-1])
        dh[-1] = dout
        _, xs, dx0 = inp.views(b)
        self._chain_backward(tw["li0"], layers, h, dh, (xs, inp.d), dx0)
        if dx0 is not None:
            inp.backward([dx0], b)

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets=None, sample_weight=None) -> None:
        """Forward (activations saved), in-batch soft-max cross-entropy and backward: fills the gradient arena and the
        IndexedSlices.  `targets` are ignored: the task's target is the positive on column 0 of every row."""
        if sample_weight is not None and not (isinstance(sample_weight, (list, tuple)) and all(s is None for s in sample_weight)):
            raise NotImplementedError("sample_weight is not implemented in the two-tower training step")
        b, _, _ = self._begin_step(inputs, targets, sample_weight)
        (q, qs), (it, its) = (self._tower_forward(tw, inp, inputs, b) for tw, inp in zip(self.towers, self.inps))
        ids = ops.as_index(inputs[self.item_id]).reshape(-1) if self.downscore else None  # packed host-batch ids widened
        T = self.temperature
        ops.positive_scores(q, it, self.pos_logit[:b], temperature=T)
        # dq -> the query tower's last dh, d_item = dpos + dneg (the negatives are the positives) -> the item tower's
        dq, di = self.towers[0]["dout"][:b], self.towers[1]["dout"][:b]
        pw = self.pairwise
        if pw is None:
            ops.inbatch_softmax_ce_split(qs, its, self.D, self.pos_logit[:b], self.stats[:b], self.ws, pos_ids=ids, neg_ids=ids,
                                         downscore=self.downscore, false_neg_score=self.false_neg_score, temperature=T)
            ops.inbatch_softmax_ce_backward(qs, its, self.D, self.stats[:b], q, it, self._scale(b), dq, di, di, loss=self._loss_all[:1],
                                            pos_ids=ids, neg_ids=ids, downscore=self.downscore,
                                            false_neg_score=self.false_neg_score, temperature=T)
        else:
            kw = dict(pos_ids=ids, neg_ids=ids, downscore=self.downscore, false_neg_score=self.false_neg_score, temperature=T,
                      reg_lambda=getattr(pw, "reg_lambda", 1.0))
            ops.inbatch_pairwise(qs, its, self.D, self.pos_logit[:b], self.stats[:b], pw.kind, loss=self._loss_all[:1], **kw)
            ops.inbatch_pairwise_backward(qs, its, self.D, self.pos_logit[:b], self.stats[:b], q, it, dq, di, di, pw.kind, **kw)
        for tw, inp, dout in zip(self.towers, self.inps, (dq, di)):
            self._tower_backward(tw, inp, dout, b)
        self._bag_grads()
        self._b = b


class DeepFMTrainer(_StepTrainer):
    """Static-buffer training step of a DeepFMModel (one BinaryOutput or RegressionOutput) at one batch size.

    forward   mm_gather_multi of every table's rows + mm_concat_columns of the continuous columns into x0 (B, d) at their
              sorted-name offsets, its split operand; mm_dense_tc per deep layer and per deep-logit layer but the last
    head      mm_deepfm_head_fwd_bwd: FM pairwise term from x0, wide lookup, the last Dense(1) of the deep logit, the output
              layer and the loss, forward and backward: logits, ds = dloss/ds (B,), dh, and the gradients of the deep logit,
              the output layer (arena), the wide bias and the continuous rows of the wide kernel
    backward  mm_dense_wgrad[_split] + dgrad per tower layer down to dx0; mm_fm_concat_backward: dx0 + ds (S_f - e_f) into
              each table's (B, D) IndexedSlices buffer
    update    mm_opt_tick, mm_dense_apply over the arena [deep, deep logit, output layer], mm_sparse_rows_apply (tables),
              mm_wide_rows_apply (the wide kernel's rows: one (B,) gradient vector for every feature block; continuous rows
              and bias by the dense rule), mm_split_weights refresh of the operand copies the model's forward reads.
    The wide kernel (one row per category of every feature) stays where it is, its optimizer slots beside it."""

    _model_name = "DeepFMModel"
    _onehot_only = True

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import BinaryOutput, DeepFMBody

        body = model.body
        if not isinstance(body, DeepFMBody):
            raise NotImplementedError("DeepFMTrainer trains DeepFMModel bodies")
        if not isinstance(model.prediction, BinaryOutput):
            raise NotImplementedError("training DeepFMModel needs one BinaryOutput or RegressionOutput")
        self._refuse_group(group)
        self._require_tc_engine()
        ib, fm = body.input_block, body.fm
        self._refuse_sharded(ib.embeddings)
        if fm.embeddings is not ib.embeddings:
            raise NotImplementedError("training DeepFMModel needs the FM term to read the input block's tables")
        self._check_mlps((body.deep, body.deep_logit))
        self._init_common(model, optimizer, batch_size, device, None)
        self._init_heads()
        self.chain = body.deep.dense_layers + body.deep_logit.dense_layers[:-1]  # tower layers run by mm_dense_tc
        self.last = body.deep_logit.dense_layers[-1]  # Dense(1), fused into the head kernel
        self._check_activations(self.chain + [self.last])
        self.U = self.chain[-1].units
        if self.U > 512:
            raise NotImplementedError(f"{self.chain[-1].name}: the head kernel reads at most 512 units of the last deep layer, got {self.U}")

        # ---- input block, tables (the FM term's features, in its order), wide kernel
        if len(fm.cat_names) > 32 or len(fm.cont_names) > 32:
            raise NotImplementedError("the DeepFM head kernel takes up to 32 categorical and 32 continuous features")
        self.inp = _ConcatInput(self, ib, dx0=True, feats=fm.cat_names, cont=fm.cont_names)
        self._init_inputs([self.inp])
        self.D = fm.dim
        self.woff = [fm.wide_offsets[f] for f in self.feats]
        self.coff = [fm.wide_offsets[n] for n in self.inp.cont]

        # the step reads self.last as fp32 (the head kernel); its operand copy is what the model's forward reads
        self._init_dense(self.chain + [self.last], [self.head])
        n = len(self.chain)
        self._init_wide(lambda li: li < n)
        self.wk = _WideKernel(self, fm.wide, self.coff)  # _Dense(1) over [one-hot | continuous]: kernel (W, 1), bias (1,)

        # ---- activations and gradients
        B = self.B
        self.h, self.h_split, self.dh = self._chain_buffers(self.chain)
        self.ds = torch.zeros(B, dtype=torch.float32, device=self.device)
        self._init_loss(B)
        self.oob = self.inp.oob

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena, the IndexedSlices of the tables, ds (the
        wide kernel's gradient values) and the gradients of the wide kernel's continuous rows and bias.  Batches smaller
        than the compiled size run in the leading rows of the same buffers."""
        a = self.arena
        d, n = self.inp.d, len(self.chain)
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)
        x0, xs, dx0 = self.inp.forward(inputs, b)
        # the head kernel and the updates read the ids at the width they came in (packed host-batch ids are not widened)
        fidx = [ops.fused_ids(get_feature(inputs, f)) for f in self.feats]
        conts = [inputs[c] for c in self.inp.cont]
        h, dh = [t[:b] for t in self.h], [t[:b] for t in self.dh]
        self._chain_forward(xs, d, 0, self.chain, h, [t[:b] for t in self.h_split])
        # -- FM + wide + deep logit + output layer + loss, forward and backward
        hi = len(a.layers) - 1
        ds = self.ds[:b]
        nc = len(self.coff)
        rows = [tb.table.shape[0] for tb in self.tables]
        wk, wg = self.wk.dense, self.wk.grad
        ops.deepfm_head_fwd_bwd(
            x0, [self.inp.cols[f] for f in self.feats], self.D, fidx, rows, self.woff, conts,
            self.coff, wk.kernel.reshape(-1), wk.bias, h[-1], self.chain[-1].activation == "relu", self.last.kernel.reshape(-1),
            self.last.bias, self.last.activation, self.head.kernel.reshape(-1), self.head.bias, self.losses[0], targets[0].reshape(-1),
            sample_weight, self.logits[:b], self._loss_all, ds, dh[-1], dw_out=a.view(a.grad, hi, "kernel"), db_out=a.view(a.grad, hi, "bias"),
            dw_dl=a.view(a.grad, n, "kernel"), db_dl=a.view(a.grad, n, "bias"),
            d_wide_bias=wg[nc:] if wk.bias is not None else None, d_cont=wg[:nc] if nc else None, oob=self.oob)
        # -- deep tower backward down to dx0
        self._chain_backward(0, self.chain, h, dh, (xs, d), dx0)
        # -- input block backward: the deep tower's dx0 + the FM term, the tables' columns only
        self.inp.backward([dx0], b, fm=ds)
        self.wk.calls = [(fidx, rows, self.woff, ds)]  # one gradient value per sample for every feature's block
        self._fidx, self._b = fidx, b

    def _gradients_to_apply(self) -> tuple:
        return self._fidx, self._slices, self._b, 1.0

    def wide_gradients(self) -> Dict[str, torch.Tensor]:
        """The wide kernel's gradient (W, 1) and its bias' (after forward_backward, before apply_gradients) — for parity tests."""
        return self.wk.gradients()


class WideAndDeepTrainer(_StepTrainer):
    """Static-buffer training step of a WideAndDeepModel (one BinaryOutput or RegressionOutput) at one batch size.

    forward   the deep input block as DCN's (one-hot features gathered, multi-hot features pooled by their combiner) into x0
              and its split operand; mm_dense_tc per deep layer
    head      mm_wide_deep_head_fwd_bwd: the wide term over the one-hot and bag features, the deep logit's Dense(1), the
              sum, the output layer and the loss, forward and backward: logits, ds = dloss/ds (B,), dh and the gradients of
              the deep logit, the output layer (arena) and the wide bias; mm_wide_bag_grad per wide bag feature
    backward  mm_dense_wgrad[_split] + dgrad per deep layer down to dx0; mm_concat_backward into each table's IndexedSlices
              buffer, mm_bag_grad_rows for multi-hot deep features
    update    mm_opt_tick, mm_dense_apply over the arena [deep, deep logit, output layer], mm_sparse_rows_apply (tables),
              mm_wide_rows_apply over the wide kernel's one-hot blocks (gradient values ds, with the bias) and once per wide
              bag feature (its nnz expanded pairs), mm_split_weights refresh of the operand copies the model's forward reads.
    The wide kernel stays where it is, its optimizer slots beside it.  Fixed-length list features can be captured into one
    CUDA graph; ragged ones train eagerly (their number of ids changes from batch to batch)."""

    _model_name = "WideAndDeepModel"

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import BinaryOutput, WideAndDeepBody

        body = model.body
        if not isinstance(body, WideAndDeepBody):
            raise NotImplementedError("WideAndDeepTrainer trains WideAndDeepModel bodies")
        if not isinstance(model.prediction, BinaryOutput):
            raise NotImplementedError("training WideAndDeepModel needs one BinaryOutput or RegressionOutput")
        self._refuse_group(group)
        self._require_tc_engine()
        if body.regularized:
            raise NotImplementedError("training WideAndDeepModel with deep / wide regularizers is not implemented")
        if body.wide is not None and getattr(body.wide, "dropout", None):
            raise NotImplementedError("training WideAndDeepModel with wide_dropout is not implemented")
        ib = body.input_block
        self.deep = ib is not None
        if self.deep:
            self._refuse_sharded(ib.embeddings)
            self._check_mlps((body.deep, body.deep_logit))
        self._init_common(model, optimizer, batch_size, device, None)
        self._init_heads()
        B = self.B
        self.chain, self.last, self.inp = [], None, None
        if self.deep:
            self.chain = body.deep.dense_layers  # run by mm_dense_tc
            self.last = body.deep_logit.dense_layers[-1]  # Dense(1), fused into the head kernel
            self._check_activations(self.chain + [self.last])
            self.inp = _ConcatInput(self, ib, dx0=True)
            self.inp.check_multihot_widths(model.schema)
        self._init_inputs([self.inp] if self.deep else [])
        self._init_dense(self.chain + ([self.last] if self.deep else []), [self.head])
        n = len(self.chain)
        self._init_wide(lambda li: li < n)
        if self.deep:
            self.h, self.h_split, self.dh = self._chain_buffers(self.chain)
        # ---- the wide kernel (W, 1) and its bias, outside the arena
        self.wl = body.wide
        self.ds = torch.zeros(B, dtype=torch.float32, device=self.device)
        if self.wl is not None:
            self.wk = _WideKernel(self, self.wl.dense)
        self._wbag_bufs: Dict[int, dict] = {}
        self._init_loss(B)
        self.oob = body.oob_counter(self.device)[0]

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena, the tables' IndexedSlices, ds and the
        expanded (id, value) pairs of the wide bag features, and the wide bias' gradient.  Batches smaller than the
        compiled size run in the leading rows of the same buffers."""
        a = self.arena
        n = len(self.chain)
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)  # no tables without a deep part
        h = dh = None
        if self.deep:
            _, xs, dx0 = self.inp.forward(inputs, b)
            h, dh = [t[:b] for t in self.h], [t[:b] for t in self.dh]
            self._chain_forward(xs, self.inp.d, 0, self.chain, h, [t[:b] for t in self.h_split])
        onehot, bags = self.wl.blocks(inputs) if self.wl is not None else ([], [])
        ds = self.ds[:b]
        hi = len(a.layers) - 1
        wk = self.wk.dense if self.wk is not None else None
        ops.wide_deep_head_fwd_bwd(
            onehot, bags, None if wk is None else wk.kernel.reshape(-1), None if wk is None else wk.bias, None if h is None else h[-1],
            self.deep and self.chain[-1].activation == "relu", None if not self.deep else self.last.kernel.reshape(-1),
            None if not self.deep else self.last.bias, "linear" if not self.deep else self.last.activation, self.head.kernel.reshape(-1),
            self.head.bias, self.logits[:b], loss=self.losses[0], targets=targets[0].reshape(-1), sample_weight=sample_weight,
            loss_buf=self._loss_all, ds=ds, dh=None if dh is None else dh[-1], dw_out=a.view(a.grad, hi, "kernel"),
            db_out=a.view(a.grad, hi, "bias"), dw_dl=a.view(a.grad, n, "kernel") if self.deep else None,
            db_dl=a.view(a.grad, n, "bias") if self.deep else None, d_wide_bias=None if wk is None else self.wk.grad, oob=self.oob)
        # the wide kernel's gradient: ds for the one-hot blocks, each bag feature's as (id, value) pairs
        calls = [([i for i, _, _ in onehot], [r for _, r, _ in onehot], [o for _, _, o in onehot], ds)] if onehot else []
        for q, bag in enumerate(bags):
            nnz = bag[0].numel()
            buf = self._wbag_bufs.setdefault(q, dict(ids=None, vals=None))
            if buf["ids"] is None or buf["ids"].shape[0] < nnz:
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("the wide bag gradient buffers cannot grow during graph capture")
                buf["ids"] = torch.empty(max(nnz, 1), dtype=torch.int64, device=self.device)
                buf["vals"] = torch.empty(max(nnz, 1), dtype=torch.float32, device=self.device)
            ids, vals = buf["ids"][:nnz], buf["vals"][:nnz]
            ops.wide_bag_grad(bag, b, ds, ids, vals)
            calls.append(([ids], [bag[2]], [bag[3]], vals))
        if self.wk is not None:
            self.wk.calls = calls
        if self.deep:
            self._chain_backward(0, self.chain, h, dh, (xs, self.inp.d), dx0)
            if self.tables:
                self.inp.backward([dx0], b)
                self._bag_grads()
        self._b = b

    def wide_gradients(self) -> Dict[str, torch.Tensor]:
        """The wide kernel's gradient (W, 1) and its bias' (after forward_backward, before apply_gradients) — for parity tests."""
        return self.wk.gradients()

    def capture(self, inputs: Dict[str, torch.Tensor], targets: torch.Tensor, clone: bool = True) -> None:
        for f in (self.wl.names if self.wl is not None else []):
            if isinstance(get_feature(inputs, f), tuple):
                raise NotImplementedError(f"graph capture with the ragged wide feature {f!r} is not implemented: its number of ids "
                                          "changes from batch to batch (train it eagerly, or feed it as a fixed-length (B, L) matrix)")
        super().capture(inputs, targets, clone)


class MMoETrainer(_StepTrainer):
    """Static-buffer training step of Model(InputBlockV2, [MLPBlock], [MMOEBlock], output) at one batch size, the output
    optionally with per-task towers (OutputBlock(task_blocks=...)).

    forward   the input block as DCN's (one-hot features gathered, multi-hot features pooled by their combiner) into x0 and
              its split operand; mm_dense_tc per shared-bottom layer (the last one emits its split operand too); with an
              MMOEBlock, mm_dense_tc of the stacked expert layer (B, E U) and the gates on that same operand (one stacked
              bias-free layer, or one chain per gate with a gate_block)
    head      without towers mm_mmoe_heads_fwd_bwd: gate soft-max, mixture, heads and loss, forward and backward; with
              towers mm_mmoe_mix_fwd (the mixtures and their split operands) -> one tower chain per output ->
              mm_mmoe_task_heads_fwd_bwd -> each tower's backward down to dm -> mm_mmoe_mix_bwd; without an MMOEBlock the
              towers (or, without them, mm_heads_fwd_bwd) read the bottom's output
    backward  every layer that reads the shared vector (experts, gates or towers) writes its pre-activation gradient into
              its columns of one buffer G; mm_dense_wgrad_split per such layer, then their summed input gradient as ONE
              transposed-kernel GEMM G [W_0 | W_1 | ..]^T; the bottom's backward; mm_concat_backward into each table's
              IndexedSlices buffer, mm_bag_grad_rows for multi-hot features
    update    mm_opt_tick, mm_dense_apply over the arena, mm_sparse_rows_apply per embedding width, mm_split_weights refresh
              of the operand copies the model's forward reads.
    Fixed-length list features can be captured into one CUDA graph; ragged ones train eagerly."""

    _model_name = "a multi-task Model(*blocks)"

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import BinaryOutput, MMoEBody, ParallelOutputs, output_towers

        body = model.body
        if not isinstance(body, MMoEBody):
            raise NotImplementedError("MMoETrainer trains Model(InputBlockV2, [MLPBlock], [MMOEBlock], output) bodies")
        if not isinstance(model.prediction, (BinaryOutput, ParallelOutputs)):
            raise NotImplementedError("train_step needs BinaryOutput / RegressionOutput heads or an OutputBlock of them")
        self._refuse_group(group)
        self._require_tc_engine()
        ib, mo = body.input_block, body.mmoe
        self._refuse_sharded(ib.embeddings)
        towers = output_towers(model.prediction) or []
        # the bottom, the task towers and the gate blocks
        self._check_mlps(([body.bottom] if body.bottom is not None else []) + towers
                         + (list(mo.gate_blocks.values()) if mo is not None and mo.gate_blocks else []))
        if mo is not None and mo.dropout:
            raise NotImplementedError("training MMOEBlock experts with dropout is not implemented")
        self._init_common(model, optimizer, batch_size, device, None)
        self._init_heads()
        self.bottom = body.bottom.dense_layers if body.bottom is not None else []
        self.mmoe = mo
        self.towers = [t.dense_layers for t in towers]
        self.gate_chains = [mo.gate_chain(t) for t in range(mo.num_gates)] if mo is not None and mo.gate_blocks else []
        chain_layers = [l for c in self.gate_chains + self.towers for l in c]
        self._check_activations(self.bottom + chain_layers + ([mo.experts] if mo is not None else []))
        if self.head.input_dim > 256:
            raise NotImplementedError("the output layer's input must be <= 256 wide")
        self.inp = _ConcatInput(self, ib, dx0=True, pretrained_ok=True)
        self.inp.check_multihot_widths(model.schema)
        self._init_inputs([self.inp])
        # arena order: bottom, [experts, stacked gates], gate chains, towers, heads; li0 of each chain
        tc = list(self.bottom)
        if mo is not None:
            self.li_experts = len(tc)
            tc.append(mo.experts)
            if mo.gates is not None:
                self.li_gates = len(tc)
                tc.append(mo.gates)
        self.gate_li0 = []
        for c in self.gate_chains:
            self.gate_li0.append(len(tc))
            tc += c
        self.tower_li0 = []
        for c in self.towers:
            self.tower_li0.append(len(tc))
            tc += c
        self._init_dense(tc, self.inp.proj_layers + [self.head])
        nb = len(self.bottom)
        firsts = set(self.gate_li0) | (set() if mo is not None else set(self.tower_li0))
        # layers whose input gradient _dgrad computes (> 128 units: through the transposed kernel); the layers reading the
        # shared vector take theirs together, and a tower's first layer reading the mixture takes it alone
        self._init_wide(lambda li: (li < nb and (li > 0 or self.inp.dx0 is not None)) or (li >= nb + (2 if mo is not None and mo.gates is not None else 1 if mo is not None else 0) and li not in firsts))

        B = self.B
        f32 = dict(dtype=torch.float32, device=self.device)
        bf = dict(dtype=torch.bfloat16, device=self.device)
        fanout = mo is not None or bool(self.towers)
        if nb:
            self.h, self.h_split, self.dh = self._chain_buffers(self.bottom, split_last=fanout)
        # the layers that read the shared vector, and their columns in G
        readers = ([mo.experts] + ([mo.gates] if mo.gates is not None else [c[0] for c in self.gate_chains])) if mo is not None \
            else [c[0] for c in self.towers]
        self.readers = readers
        self.G = self.G_split = self.wT = self.wT_split = None
        if fanout:
            K = body.input_width()
            N = sum(l.units for l in readers)
            self.G = torch.zeros((B, N), **f32)
            self.G_split = torch.zeros((B, 2 * ops.tc_padded_k(N)), **bf)
            self.wT = torch.zeros((N, K), **f32)  # [W_0 | W_1 | ..]^T
            self.wT_split = torch.zeros((ops.tc_padded_n(K), 2 * ops.tc_padded_k(N)), **bf)
            self.G_cols, c = [], 0
            for l in readers:
                self.G_cols.append((c, c + l.units))
                c += l.units
        if mo is not None:
            self.EU = mo.experts.units
            self.X = torch.zeros((B, self.EU), **f32)
            if mo.gates is not None:
                self.L = torch.zeros((B, mo.gates.units), **f32)
        self.gbufs = [self._chain_buffers(c) for c in self.gate_chains]
        self.tbufs = [self._chain_buffers(c) for c in self.towers]
        if self.towers and mo is not None:
            H, U = self.H, mo.units
            self.P = torch.zeros((B, H * mo.num_experts), **f32)
            self.M = torch.zeros((H, B, U), **f32)
            self.M_split = torch.zeros((H, B, 2 * ops.tc_padded_k(U)), **bf)
            self.dM = torch.zeros((H, B, U), **f32)
        self._init_loss(B)
        self.oob = self.inp.oob

    def _g(self, i: int, b: int) -> torch.Tensor:
        """Reader i's columns of G (its pre-activation gradient)."""
        c0, c1 = self.G_cols[i]
        return self.G[:b, c0:c1]

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena and the tables' IndexedSlices.  Batches
        smaller than the compiled size run in the leading rows of the same buffers."""
        a = self.arena
        nb, d, mo = len(self.bottom), self.inp.d, self.mmoe
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)
        ys = [t.reshape(-1) for t in targets]
        hi = len(a.layers) - 1
        logits = self.logits.view(-1)[:self.H * b].view(self.H, b)
        v = lambda ts: [t[:b] for t in ts]
        _, xs, dx0 = self.inp.forward(inputs, b)  # dx0: None without tables
        op, K = xs, d
        if nb:
            h, h_split, dh = v(self.h), v(self.h_split), v(self.dh)
            self._chain_forward(xs, d, 0, self.bottom, h, h_split)
            if self.G is not None:
                op, K = h_split[-1], self.bottom[-1].units
        heads_kw = dict(loss_weights=self.loss_weights, sample_weight=sample_weight)
        if self.G is None:  # shared bottom -> heads
            self._heads(h[-1], targets, dh[-1], self.bottom[-1].activation == "relu", sample_weight, b)
        elif mo is None:  # towers on the shared vector
            tb = [[v(x) for x in bufs] for bufs in self.tbufs]
            for i, (c, (th, ths, tdh)) in enumerate(zip(self.towers, tb)):
                tdh[0] = self._g(i, b)
                self._chain_forward(op, K, self.tower_li0[i], c, th, ths)
            ops.mmoe_task_heads_fwd_bwd([t[0][-1] for t in tb], self.head.kernel, self.head.bias, self.losses, ys, logits,
                                        self._loss_all, [t[2][-1] for t in tb], a.view(a.grad, hi, "kernel"), a.view(a.grad, hi, "bias"),
                                        mask_relu=self.towers[0][-1].activation == "relu", **heads_kw)
            for i, (c, (th, ths, tdh)) in enumerate(zip(self.towers, tb)):
                self._chain_backward(self.tower_li0[i], c, th, tdh, (op, K), None)
        else:
            X = self.X[:b]
            ops.dense_tc(op, K, self._wsplit[self.li_experts], self.EU, mo.experts.bias, mo.experts.activation, out_f32=X)
            gb = [[v(x) for x in bufs] for bufs in self.gbufs]
            if mo.gates is not None:
                L = self.L[:b]
                ops.dense_tc(op, K, self._wsplit[self.li_gates], mo.gates.units, None, "linear", out_f32=L)
                gl, dgl = mo.gate_logits(L), mo.gate_logits(self._g(1, b))
            else:
                for i, (c, (gh, ghs, gdh)) in enumerate(zip(self.gate_chains, gb)):
                    gdh[0] = self._g(1 + i, b)
                    self._chain_forward(op, K, self.gate_li0[i], c, gh, ghs)
                gl, dgl = [g[0][-1] for g in gb], [g[2][-1] for g in gb]
            dX = self._g(0, b)
            relu_x = mo.experts.activation == "relu"
            if not self.towers:
                ops.mmoe_heads_fwd_bwd(X, mo.num_experts, gl, mo.temperature, self.head.kernel, self.head.bias, self.losses, ys,
                                       logits, self._loss_all, dx=dX, d_gate_logits=dgl, dw=a.view(a.grad, hi, "kernel"),
                                       db=a.view(a.grad, hi, "bias"), mask_relu=relu_x, **heads_kw)
            else:
                U = mo.units
                H = self.H
                # (H, b, ...) views of the leading H b rows, contiguous like the kernels write them
                M, Ms, dM = (t.view(-1)[:H * b * t.shape[2]].view(H, b, t.shape[2]) for t in (self.M, self.M_split, self.dM))
                P = self.P[:b]
                ops.mmoe_mix_fwd(X, mo.num_experts, gl, mo.temperature, P, M, Ms)
                tb = [[v(x) for x in bufs] for bufs in self.tbufs]
                for i, (c, (th, ths, tdh)) in enumerate(zip(self.towers, tb)):
                    self._chain_forward(Ms[i], U, self.tower_li0[i], c, th, ths)
                ops.mmoe_task_heads_fwd_bwd([t[0][-1] for t in tb], self.head.kernel, self.head.bias, self.losses, ys, logits,
                                            self._loss_all, [t[2][-1] for t in tb], a.view(a.grad, hi, "kernel"),
                                            a.view(a.grad, hi, "bias"), mask_relu=self.towers[0][-1].activation == "relu", **heads_kw)
                for i, (c, (th, ths, tdh)) in enumerate(zip(self.towers, tb)):
                    self._chain_backward(self.tower_li0[i], c, th, tdh, (Ms[i], U), dM[i])
                ops.mmoe_mix_bwd(X, mo.num_experts, P, mo.temperature, dM, dX, dgl, mask_relu=relu_x)
            ops.dense_wgrad_split(op, K, dX, a.view(a.grad, self.li_experts, "kernel"), a.view(a.grad, self.li_experts, "bias"))
            if mo.gates is not None:
                ops.dense_wgrad_split(op, K, self._g(1, b), a.view(a.grad, self.li_gates, "kernel"), None)
            else:
                for i, (c, (gh, ghs, gdh)) in enumerate(zip(self.gate_chains, gb)):
                    self._chain_backward(self.gate_li0[i], c, gh, gdh, (op, K), None)
        dx_in = dh[-1] if nb else dx0
        if self.G is not None and dx_in is not None:  # G [W_0 | W_1 | ..]^T: the readers' input gradients summed by one GEMM
            for (c0, c1), l in zip(self.G_cols, self.readers):
                self.wT[c0:c1].copy_(l.kernel.t())
            ops.split_weights(self.wT, out=self.wT_split)
            Gs = self.G_split[:b]
            ops.split_rows(self.G[:b], out=Gs)
            ops.dense_tc(Gs, self.G.shape[1], self.wT_split, K, None, None, out_f32=dx_in)
            if nb and self.bottom[-1].activation == "relu":
                ops.relu_mask(dx_in, h[-1])
        if nb:
            self._chain_backward(0, self.bottom, h, dh, (xs, d), dx0)
        if dx0 is not None:
            self.inp.backward([dx0], b)
            self._bag_grads()
        self._b = b


class NCFTrainer(_StepTrainer):
    """Static-buffer training step of an NCFModel (RankingModel over NCFBody; 1..8 BinaryOutput / RegressionOutput heads)
    at one batch size.

    forward   the mlp branch's rows [i_mlp | u_mlp] into x0 (mm_gather_multi) and its split operand; mm_dense_tc per
              mlp_block layer (fp32 activation saved + the next layer's operand)
    head      mm_ncf_head_fwd_bwd: the GMF rows gathered by id, u * i next to the tower's output h, the heads, their losses
              and the backward in one pass: the GMF tables' IndexedSlices values (du, di, with 2 l2 e), dh (relu-masked),
              the heads' dW / db in the arena, and the GMF part of the L2 term
    backward  mm_dense_wgrad[_split] + mm_dense_dgrad per layer down to dx0; mm_concat_backward (mm_concat_backward_l2 with
              embeddings_l2_reg > 0) into the mlp tables' IndexedSlices values
    update    mm_opt_tick, mm_dense_apply over the arena, mm_sparse_rows_apply per embedding width (all four tables),
              mm_split_weights refresh of the operand copies the model's forward reads.

    The loss vector is [regularization, total, loss_0 ..]: `loss` is its tail, the vector of the other ranking steps, and
    mm_concat_backward_l2 adds the mlp tables' term to its first two entries.  Fixed-shape ids capture into one CUDA graph."""

    _model_name = "an NCFModel"
    _onehot_only = True

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import NCFBody

        body = model.body
        if not isinstance(body, NCFBody):
            raise NotImplementedError("NCFTrainer trains NCFModel bodies")
        self._refuse_group(group)
        self._require_tc_engine()
        self._refuse_sharded(body)
        for emb in model.embedding_blocks():
            self._refuse_sharded(emb)
        self._check_mlps([body.mlp])
        self.layers = body.mlp.dense_layers
        self._check_activations(self.layers)
        self._init_common(model, optimizer, batch_size, device, None)
        self._init_heads()
        self.inp = _ConcatInput(self, body.mlp_input_block, dx0=True, cols=body.mlp_columns)
        # table positions: the mlp branch's (the input block's order), then the GMF user and item tables
        gmf = [(body.feature("mf", s), body.table("mf", s)) for s in ("query", "item")]
        self.inp.tidx = list(range(len(self.inp.feats)))
        self._init_tables(self.inp.feats + [f for f, _ in gmf], [self.inp.emb.feature_to_table[f] for f in self.inp.feats]
                          + [t for _, t in gmf])
        self.slices = [torch.zeros((self.B, t.table.shape[1]), dtype=torch.float32, device=self.device) for t in self.tables]
        self.t_u, self.t_i = len(self.inp.feats), len(self.inp.feats) + 1
        self.l2 = body.embeddings_l2_reg
        self.inp.set_l2_reg(self.l2)
        self._init_dense(self.layers, [self.head])
        self._init_wide(lambda li: True)
        self.h, self.h_split, self.dh = self._chain_buffers(self.layers)
        self._init_loss(self.B)
        self._loss_all = torch.zeros(2 + self.H, dtype=torch.float32, device=self.device)  # [regularization, total, loss_0 ..]
        self.loss = self._loss_all[1:] if self.H > 1 else self._loss_all[1:2]
        self.regularization = self._loss_all[0]
        self.oob = self.inp.oob

    def table_gradients(self) -> Dict[str, tuple]:
        """{"mf/query" | "mf/item" | "mlp/query" | "mlp/item": (ids, rows)} of the last forward_backward: each table's
        IndexedSlices before duplicates are summed."""
        body = self.body
        out = {f"mf/{s}": (self._idx[t], self._slices[t]) for s, t in (("query", self.t_u), ("item", self.t_i))}
        for s in ("query", "item"):
            t = self.inp.tidx[self.inp.feats.index(body.feature("mlp", s))]
            out[f"mlp/{s}"] = (self._idx[t], self._slices[t])
        return out

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), loss and backward: fills the gradient arena and the four tables' IndexedSlices.
        Batches smaller than the compiled size run in the leading rows of the same buffers."""
        a, body = self.arena, self.body
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)
        hi = len(a.layers) - 1
        _, xs, dx0 = self.inp.forward(inputs, b)
        h, h_split, dh = ([x[:b] for x in bufs] for bufs in (self.h, self.h_split, self.dh))
        self._chain_forward(xs, self.inp.d, 0, self.layers, h, h_split)
        ids_u, ids_i = body.ids(inputs, "query"), body.ids(inputs, "item")
        self._idx[self.t_u], self._idx[self.t_i] = ids_u, ids_i
        ops.ncf_head_fwd_bwd(self.tables[self.t_u].table, ids_u, self.tables[self.t_i].table, ids_i, h[-1], self.head.kernel,
                             self.head.bias, self.losses, [t.reshape(-1) for t in targets],
                             self.logits.view(-1)[:self.H * b].view(self.H, b), loss=self._loss_all[1:],
                             reg=self._loss_all[:1] if self.l2 else None, l2=self.l2, du=self._slices[self.t_u],
                             di=self._slices[self.t_i], dh=dh[-1], dw=a.view(a.grad, hi, "kernel"), db=a.view(a.grad, hi, "bias"),
                             loss_weights=self.loss_weights, relu_h=self.layers[-1].activation == "relu",
                             sample_weight=sample_weight, oob=self.oob)
        self._chain_backward(0, self.layers, h, dh, (xs, self.inp.d), dx0)
        self.inp.backward([dx0], b)
        self._b = b


class _TiedTable:
    """The weight-tied item table E (N_I, D) of a CategoricalOutput and its bias (N_I,), trained outside the arena on
    DENSE gradients: grad = [dE | db], where dE is the output side's G^T x / T (every row) plus the input side's
    IndexedSlices (mm_slices_add_dense), as TensorFlow sums a gather's and a matmul's gradient of one variable.  So every
    optimizer (LazyAdam too) updates every row of E every step.  E's optimizer slots are the trainer's table slots when an
    input feature reads E, its own otherwise; e_split and bt are the operands the catalog kernels read (E's split rows and
    b / T), refreshed after each update."""

    def __init__(self, tr: "_StepTrainer", out, t: Optional[int]):
        dev = tr.device
        self.tr, self.out, self.t = tr, out, t
        self.E, self.bias = out.table.table, out.bias
        # E trains with its table's optimizer group, the bias with the CategoricalOutput's
        self.gE = opt = tr._groups.of(out.table)
        self.gb = tr._groups.of(out) if self.bias is not None else None
        N, D = self.E.shape
        self.T = float(out.logits_temperature)
        nb = N if self.bias is not None else 0
        self.grad = torch.zeros(_align(N * D) + nb, dtype=torch.float32, device=dev)
        self.dE = self.grad[:N * D].view(N, D)
        self.db = self.grad[_align(N * D):] if nb else None
        if t is None:  # no input feature reads E: its own slots
            self.s1 = torch.full_like(self.E, opt.initial_accumulator_value) if opt.slots >= 1 else None
            self.s2 = torch.zeros_like(self.E) if opt.slots >= 2 else None
        else:
            self.s1, self.s2 = tr.tstate1[t], tr.tstate2[t]
        gb = self.gb
        self.b_s1 = torch.full((nb,), gb.initial_accumulator_value, dtype=torch.float32, device=dev) if nb and gb.slots >= 1 else None
        self.b_s2 = torch.zeros(nb, dtype=torch.float32, device=dev) if nb and gb.slots >= 2 else None
        self.e_split = ops.split_rows(self.E)
        self.bt = None
        if self.bias is not None:
            self.bt = self.bias if self.T == 1.0 else torch.zeros_like(self.bias)
            self._inv_t = torch.full((1,), 1.0 / self.T, dtype=torch.float32, device=dev)
            self._zero = torch.zeros(1, dtype=torch.float32, device=dev)
        self.refresh()

    def state(self) -> Dict[str, Optional[torch.Tensor]]:
        """The variables a step changes that the trainer's table state does not already hold."""
        st = {"tied/bias": self.bias, "tied/bias/s1": self.b_s1, "tied/bias/s2": self.b_s2}
        if self.t is None:
            st.update({"tied/embeddings": self.E, "tied/embeddings/s1": self.s1, "tied/embeddings/s2": self.s2})
        return st

    def apply(self) -> None:
        ops.dense_apply(self.gE.kind, self.E.view(-1), self.dE.view(-1), None if self.s1 is None else self.s1.view(-1),
                        None if self.s2 is None else self.s2.view(-1), self.gE.hyper)
        if self.bias is not None:
            ops.dense_apply(self.gb.kind, self.bias, self.db, self.b_s1, self.b_s2, self.gb.hyper)

    def refresh(self) -> None:
        """The catalog kernels' operands (E's split rows, b / T) and E's lookup mirror, if it has one, from the variables."""
        ops.split_rows(self.E, out=self.e_split)
        if self.bt is not None and self.bt is not self.bias:
            N = self.bias.numel()
            ops.scale_shift(self.bias.view(N, 1), self._inv_t, self._zero, out=self.bt.view(N, 1))
        m = self.out.table._mirror
        if m is not None and m.shape[0] == self.E.shape[0]:
            ops.split_rows(self.E, out=m)


class CatalogTrainer(_StepTrainer):
    """Static-buffer training step of Model(InputBlockV2, MLPBlock, CategoricalOutput(to_call=EmbeddingTable)) — the
    weight-tied next-item classifier — at one batch size, with Keras CategoricalCrossentropy(from_logits=True) on
    z = (x E^T + b) / T: loss = sum_b c_b (lse_b - z_b[y_b]), c = sample_weight / B (1 / B without weights).  With the
    compiled loss' label_smoothing eps the target is (1 - eps) onehot(y) + eps / N_I: loss = sum_b c_b (lse_b - (1 - eps)
    z_b[y_b] - eps mean_j z_b[j]) (mm_catalog_smoothed_ce_backward).  The MLPBlock's dropout trains here (and only here):
    mm_dense_tc_dropout draws each layer's mask in its epilogue, and the backward scales the relu-masked gradient.

    forward   the input block as MMoETrainer's (one-hot features gathered, multi-hot features pooled) into x0 and its split
              operand; mm_dense_tc per MLP layer (the last one emits x's split operand when T = 1); x / T by mm_scale_shift
              and its split (T != 1); mm_catalog_score's soft-max statistics against the trainer's split copy of E with
              b / T, without the (B, N_I) logits
    backward  mm_catalog_softmax_ce_backward: dx, dE (N_I, D) over every row, db and the loss; the MLP's backward down to
              dx0; mm_concat_backward into the tables' IndexedSlices, mm_bag_grad_rows for multi-hot features; the tied
              table's input-side slices added into dE by mm_slices_add_dense (duplicates in index order, one writer per row)
    update    mm_opt_tick, mm_dense_apply over the arena, over E (flat N_I D) and over the bias, mm_sparse_rows_apply for
              the untied tables; then E's split copy, b / T and the MLP's split weights are refreshed, and after the step
              CategoricalOutput.refresh() drops its cached operands, so a later forward, top_k or evaluate sees the update.
    A label outside [0, N_I) is never used as an address: it adds one to the gathers' out-of-range counter, which
    check_indices (once per `fit` epoch) turns into an IndexError.  Fixed-length list features can be captured into one
    CUDA graph; ragged ones train eagerly."""

    _model_name = "a Model(InputBlockV2, MLPBlock, CategoricalOutput)"

    def __init__(self, model, optimizer: Optimizer, batch_size: int, device=None, group=None):
        from .models import CatalogModel

        if not isinstance(model, CatalogModel):
            raise NotImplementedError("CatalogTrainer trains Model(InputBlockV2, MLPBlock, CategoricalOutput)")
        self._refuse_group(group)
        self._require_tc_engine()
        ib, out = model.body.input_block, model.prediction
        self._refuse_sharded(ib.embeddings)
        self._check_mlps([model.body.bottom], allow_dropout=True)
        D = out.table.dim
        if D > 128 or D % 4:
            raise NotImplementedError(f"table {out.table.table_name!r}: training a CategoricalOutput needs an item table width "
                                      f"that is a multiple of 4 no larger than 128 (the catalog kernels'), got {D}")
        if not out.table.trainable:
            raise NotImplementedError(f"table {out.table.table_name!r}: a frozen CategoricalOutput table is not implemented")
        self._init_common(model, optimizer, batch_size, device, None)
        self.layers = model.body.bottom.dense_layers
        self._check_activations(self.layers)
        # Keras Dropout(rate) in training after the MLP's layers (blocks/mlp.py:97-131), drawn in mm_dense_tc's epilogue:
        # the mask hashes (seed of mm.set_seed, the optimizer's device step counter, layer, row, column), so eager steps
        # and graph replays from one state draw the same masks and every step draws new ones
        rates = model.body.bottom.dropout_rates()
        for l, r in zip(self.layers, rates):
            if r and l.activation != "relu":
                raise NotImplementedError(f"{l.name}: dropout in training after a {l.activation!r} layer is not implemented "
                                          "(relu layers only)")
        self.dropout_rates = rates
        self.outputs, self.H, self.losses, self.loss_weights = [out], 1, [out.loss], [1.0]
        self.inp = _ConcatInput(self, ib, dx0=True)
        self.inp.check_multihot_widths(model.schema)
        self._init_inputs([self.inp])
        tt = next((t for t, tb in enumerate(self.tables) if tb is out.table), None)
        if tt is not None:  # the tied table's gradient is dense: it leaves the sparse updates
            self._by_width = {w: [t for t in ts if t != tt] for w, ts in self._by_width.items()}
        self._init_dense(self.layers, [])
        self._init_wide(lambda li: li > 0 or bool(self.tables))
        self.T = float(out.logits_temperature)
        self.D, self.N = D, out.num_classes
        B = self.B
        f32 = dict(dtype=torch.float32, device=self.device)
        self.h, self.h_split, self.dh = self._chain_buffers(self.layers, split_last=self.T == 1.0)
        if self.T != 1.0:
            self.xt = torch.zeros((B, D), **f32)
            self.xt_split = torch.zeros((B, 2 * ops.tc_padded_k(D)), dtype=torch.bfloat16, device=self.device)
            self._t_vec = (torch.full((D,), 1.0 / self.T, **f32), torch.zeros(D, **f32))
        self.stats = torch.zeros((B, 3), **f32)
        # workspaces for every batch size up to B (their sizes need not grow with it)
        self.ws_stats = torch.zeros(max(16, max(ops.catalog_workspace_bytes(m, self.N) for m in range(1, B + 1))),
                                    dtype=torch.uint8, device=self.device)
        self.eps = float(getattr(model, "label_smoothing", 0.0))
        ws_bytes = ops.catalog_smoothed_ce_workspace_bytes if self.eps else ops.catalog_softmax_ce_workspace_bytes
        self.ws_bwd = torch.zeros(max(16, max(ws_bytes(m, self.N, D) for m in range(1, B + 1))), dtype=torch.uint8,
                                  device=self.device)
        self.c = torch.zeros(B, **f32)  # per-row loss weights c = sample_weight / b
        self._inv_b: Dict[int, torch.Tensor] = {}
        self._zero = torch.zeros(1, **f32)
        self.ws_merge: Optional[torch.Tensor] = None  # mm_slices_add_dense's workspace, sized by the first batch
        self.tt = tt
        self.wk = _TiedTable(self, out, tt)
        self._init_loss(B)
        from .core import _SEED

        step = self.hyper[_cabi.HYPER_STEP:_cabi.HYPER_STEP + 1]
        self._drop = [None if not r else (r, _SEED[0], step, i) for i, r in enumerate(rates)]
        self._drop_scale = [None if not r else torch.full((l.units,), 1.0 / (1.0 - r), **f32) for l, r in zip(self.layers, rates)]
        self._drop_zero = torch.zeros(max(l.units for l in self.layers), **f32)
        self.logits = self.stats  # per row of the last step: [max, log-sum-exp, target logit] of the tempered logits
        self.oob = self.inp.oob if self.inp.oob is not None else torch.zeros(1, dtype=torch.int32, device=self.device)

    def _scale(self, b: int) -> torch.Tensor:
        c = self._inv_b.get(b)
        if c is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("the loss scale of a new batch size cannot be created during graph capture")
            c = self._inv_b[b] = torch.full((1,), 1.0 / b, dtype=torch.float32, device=self.device)
        return c

    def _labels(self, targets, b: int) -> torch.Tensor:
        ys = list(targets) if isinstance(targets, (list, tuple)) else [targets]
        if len(ys) != 1:
            raise ValueError(f"one target tensor expected (the class ids), got {len(ys)}")
        y = ys[0].reshape(-1)
        if y.numel() != b or y.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"targets must hold {b} int32 / int64 class ids, got {tuple(ys[0].shape)} {ys[0].dtype}")
        return y

    def table_gradients(self) -> Dict[str, tuple]:
        """{feature: (ids, rows)} of the last forward_backward: every input table's IndexedSlices before duplicates are
        summed (multi-hot features: one row per id); the tied table's are already in `gradients()['tied/embeddings']`."""
        out = {}
        for t, f in enumerate(self.feats):
            bag = self._bags.get(t)
            out[f] = (self._idx[t], self._slices[t]) if bag is None else (bag["apply_ids"], bag["rows"])
        return out

    def gradients(self) -> Dict[str, torch.Tensor]:
        """The MLP's gradients by variable name, the tied table's dense dE (both sides) and the bias' db (after
        forward_backward, before apply_gradients)."""
        out = super().gradients()
        out["tied/embeddings"] = self.wk.dE
        if self.wk.db is not None:
            out["tied/bias"] = self.wk.db
        return out

    def forward_backward(self, inputs: Dict[str, torch.Tensor], targets, sample_weight=None) -> None:
        """Forward (activations saved), the catalog soft-max cross-entropy and the backward: fills the arena's gradients,
        the tables' IndexedSlices and the tied table's [dE | db].  Batches smaller than the compiled size run in the
        leading rows of the same buffers."""
        b, targets, sample_weight = self._begin_step(inputs, targets, sample_weight)
        y = self._labels(targets, b)
        wk, D = self.wk, self.D
        _, xs, dx0 = self.inp.forward(inputs, b)
        h, h_split, dh = ([t[:b] for t in bufs] for bufs in (self.h, self.h_split, self.dh))
        self._chain_forward(xs, self.inp.d, 0, self.layers, h, h_split, drop=self._drop)
        x = h[-1]
        if self.T == 1.0:
            x_split = h_split[-1]
        else:
            ops.scale_shift(x, *self._t_vec, out=self.xt[:b])
            x_split = ops.split_rows(self.xt[:b], out=self.xt_split[:b])
        stats = self.stats[:b]
        ops.catalog_stats_split(x_split, D, wk.e_split, stats, y, self.ws_stats, bias=wk.bt)
        if sample_weight is None:
            c = self._scale(b)
        else:
            sw = sample_weight.reshape(-1)
            if sw.numel() != b or sw.dtype != torch.float32:
                raise ValueError(f"sample_weight must hold {b} float32 values, got {tuple(sample_weight.shape)} {sample_weight.dtype}")
            c = self.c[:b]
            ops.scale_shift(sw.contiguous().view(b, 1), self._scale(b), self._zero, out=c.view(b, 1))
        ops.catalog_softmax_ce_backward(x_split, wk.e_split, D, stats, y, c, dh[-1], wk.dE, db=wk.db, bias=wk.bt,
                                        loss=self._loss_all[:1], temperature=self.T, workspace=self.ws_bwd, oob=self.oob,
                                        label_smoothing=self.eps)
        if self.layers[-1].activation == "relu":
            ops.relu_mask(dh[-1], x)
        if self._drop_scale[-1] is not None:
            ops.scale_shift(dh[-1], self._drop_scale[-1], self._drop_zero[:D], out=dh[-1])
        self._chain_backward(0, self.layers, h, dh, (xs, self.inp.d), dx0, drop_scale=self._drop_scale)
        if self.tables:
            self.inp.backward([dx0], b)
            self._bag_grads()
        if self.tt is not None:  # the tied table's input side: its IndexedSlices added into dE
            bag = self._bags.get(self.tt)
            ids, rows = (self._idx[self.tt], self._slices[self.tt]) if bag is None else (bag["apply_ids"], bag["rows"])
            need = max(16, ops.slices_add_dense_workspace_bytes(ids.numel()))
            if self.ws_merge is None or self.ws_merge.numel() < need:
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("the row-merge workspace cannot grow during graph capture")
                self.ws_merge = torch.empty(need, dtype=torch.uint8, device=self.device)
            ops.slices_add_dense(ids, rows, wk.dE, workspace=self.ws_merge)
        self._b = b

    def _refresh_operands(self) -> None:
        super()._refresh_operands()
        self.wk.refresh()

    def _after_step(self) -> None:
        super()._after_step()
        self.model.prediction.refresh()  # CategoricalOutput's cached split copies and b / T


def trainer_for(model, optimizer: Optimizer, batch_size: int, group=None):
    """The training engine of `model`: DLRMTrainer, DCNTrainer, DeepFMTrainer, WideAndDeepTrainer, MMoETrainer or
    NCFTrainer by the ranking body, TwoTowerTrainer for a RetrievalModel, CatalogTrainer for a CatalogModel."""
    from .models import CatalogModel, DCNBody, DeepFMBody, MMoEBody, NCFBody, RetrievalModel, RetrievalModelV2, WideAndDeepBody

    if isinstance(model, CatalogModel):
        return CatalogTrainer(model, optimizer, batch_size, group=group)
    if isinstance(model, RetrievalModelV2):
        raise NotImplementedError("training TwoTowerModelV2 / ContrastiveOutput is not implemented: train the v1 TwoTowerModel")
    if isinstance(model, RetrievalModel):
        return TwoTowerTrainer(model, optimizer, batch_size, group=group)
    by_body = {DCNBody: DCNTrainer, DeepFMBody: DeepFMTrainer, WideAndDeepBody: WideAndDeepTrainer, MMoEBody: MMoETrainer,
               NCFBody: NCFTrainer}
    body = getattr(model, "body", None)
    cls = next((c for t, c in by_body.items() if isinstance(body, t)), DLRMTrainer)
    return cls(model, optimizer, batch_size, group=group)
