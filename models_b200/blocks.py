"""Body blocks of the hot path: MLPBlock, DotProductInteraction, CrossBlock, DLRMBlock.

Constructor surface and error messages follow merlin/models/tf/blocks/{mlp,interaction,cross,dlrm}.py;
execution is a handful of fused kernel launches (models_b200.ops), not a Keras layer graph.
"""
from __future__ import annotations

import os

from typing import Dict, List, Optional, Sequence, Union

import torch

from . import ops
from ._cabi import ACTIVATIONS
from .core import (Block, InitializerType, SequentialBlock, TabularData, batch_size_of, buffer_namespace,
                   concat_sorted, create_variable, default_device, unique_name)
from .inputs import (ContinuousFeatures, EmbeddingOptions, Embeddings, EmbeddingsBlock, InputBlock, InputBlockV2,
                     infer_embedding_dim)
from .schema import Schema, Tags

# dense-layer engine: "fp32" = exact CUDA-core kernel (mm_dense_fp32); "tc" = wgmma split-bf16
_DENSE_ENGINE = ["auto"]


def set_dense_engine(engine: str) -> None:
    if engine not in ("auto", "fp32", "tc"):
        raise ValueError("engine must be 'auto', 'fp32' or 'tc'")
    _DENSE_ENGINE[0] = engine


def dense_engine() -> str:
    return _DENSE_ENGINE[0]


def _use_tc() -> bool:
    return _DENSE_ENGINE[0] in ("auto", "tc")


_MLP_FUSION = [os.environ.get("MM_MLP_FUSION", "1") != "0"]
_LAST_PATH = ["none"]


def set_mlp_fusion(on: bool) -> None:
    """Whole-tower kernel (mm_mlp_tc) for towers whose widths are all <= 128; off = one launch per layer."""
    _MLP_FUSION[0] = bool(on)


def last_dense_path() -> str:
    """"mlp_tc" | "dense_tc" | "fp32": which kernels the most recent run_dense_chain used (tests / notes)."""
    return _LAST_PATH[0]


_SMALL_TOWER = [True]  # mm_tower2_small for narrow-input two-layer towers (tests switch it off to reach the TMA tower kernel)
_TABLE_MIRROR = [None]  # None: decide from MM_TABLE_MIRROR (default on); True / False: forced


def set_table_mirror(on: Optional[bool]) -> None:
    """Split-bf16 mirrors of the embedding tables for the fused DLRM kernel (D = 64): a second copy of every table in
    HBM; the kernel then loads MMA fragments with ldmatrix instead of splitting fp32 rows per sample.
    None = environment default (MM_TABLE_MIRROR, on unless it is '0')."""
    _TABLE_MIRROR[0] = on


def table_mirror() -> bool:
    if _TABLE_MIRROR[0] is not None:
        return bool(_TABLE_MIRROR[0])
    import os

    return os.environ.get("MM_TABLE_MIRROR", "1") != "0"


def run_dense_chain(x: Optional[torch.Tensor], layers: "List[_Dense]", a_split: Optional[torch.Tensor] = None,
                    K: Optional[int] = None, operand_out: bool = False) -> torch.Tensor:
    """A chain of Dense layers on one input matrix.  operand_out=True: the result rows come back as bf16 split rows
    (B, 2*Kp) = [hi | lo] (the interaction kernel's operand format) — directly from the whole-tower kernel's last
    epilogue when it applies, by one mm_split_rows pass over the fp32 result otherwise.

    tensor-core engine ("auto"/"tc"): x is split once into bf16 (hi, lo); every layer is one
    wgmma launch whose epilogue (bias + activation) directly emits the NEXT layer's split-bf16
    operand, so intermediate activations never exist in fp32 in HBM; the last layer writes fp32.
    "fp32" engine: exact CUDA-core kernels (parity anchor)."""
    if a_split is not None:  # producer (interaction kernel) already emitted the split-bf16 operand
        device, B, a = a_split.device, a_split.shape[0], a_split
    else:
        device, B, K = x.device, x.shape[0], x.shape[1]
    width = K
    for l in layers:
        l.build(width, device)
        width = l.units
    if not _use_tc():
        if x is None:
            raise ValueError("the fp32 dense engine needs an fp32 input")
        for l in layers:
            x = l(x)
        _LAST_PATH[0] = "fp32"
        return ops.split_rows(x.contiguous()) if operand_out else x
    if a_split is None:
        a = ops.split_rows(x)
    out = None
    # a trailing Dense(N -> 1) (BinaryOutput) after a layer with N <= 32 units is evaluated inside that
    # layer's GEMM epilogue: one launch and one HBM round trip fewer
    fuse_head = (len(layers) >= 2 and layers[-1].units == 1 and layers[-2].units <= 32
                 and layers[-1].input_dim == layers[-2].units)
    if fuse_head:
        head, layers = layers[-1], layers[:-1]
    if K != layers[0].input_dim:
        raise ValueError(f"{layers[0].name}: input width {K} != kernel rows {layers[0].input_dim}")
    widths = [l.units for l in layers]
    if _MLP_FUSION[0] and ops.mlp_tc_supported(K, widths, head=fuse_head):
        # whole tower in one launch: layers 2..n run on chip, activations stay in registers
        _LAST_PATH[0] = "mlp_tc"
        kw = {}
        if fuse_head:
            out = torch.empty((B, 1), dtype=torch.float32, device=device)
            kw = dict(head_w=head.kernel.reshape(-1), head_b=head.bias_value(), head_act=head.activation, head_out=out)
        elif operand_out and widths[-1] % 64 == 0:
            out = torch.empty((B, 2 * widths[-1]), dtype=torch.bfloat16, device=device)  # split rows [hi | lo]
            kw = dict(out_operand=out)
            operand_out = False  # done by the kernel
        else:
            out = torch.empty((B, widths[-1]), dtype=torch.float32, device=device)
            kw = dict(out=out)
        ops.mlp_tc(a, K, [l.split_kernel() for l in layers], widths, [l.bias for l in layers],
                   [l.activation for l in layers], **kw)
        return ops.split_rows(out) if operand_out else out
    _LAST_PATH[0] = "dense_tc"
    for i, l in enumerate(layers):
        last = i == len(layers) - 1
        if K != l.input_dim:
            raise ValueError(f"{l.name}: input width {K} != kernel rows {l.input_dim}")
        nxt = None
        if last and fuse_head:
            out = torch.empty((B, 1), dtype=torch.float32, device=device)
            ops.dense_tc_head(a, K, l.split_kernel(), l.units, l.bias, l.activation, head.kernel.reshape(-1),
                              head.bias_value(), head.activation, out)
            return out
        if last:
            out = torch.empty((B, l.units), dtype=torch.float32, device=device)
        else:
            nxt = l.split_buffer(B, device)
        ops.dense_tc(a, K, l.split_kernel(), l.units, l.bias, l.activation, passes=3, out_f32=out, out_split=nxt)
        a, K = nxt, l.units
    return ops.split_rows(out) if operand_out else out


class _Dense(Block):
    """Keras Dense as wrapped by blocks/mlp.py:210-300: dict inputs are concat-aggregated in
    sorted-key order first (:275-277), then act(x @ kernel + bias) with kernel (in, units)."""

    def __init__(self, units: int, activation: Optional[str] = None, use_bias: bool = True,
                 kernel_initializer: InitializerType = "glorot_uniform", bias_initializer: InitializerType = "zeros",
                 name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("dense"))
        if activation not in ACTIVATIONS:
            raise ValueError(f"Unknown activation function: {activation!r}")
        self.units = int(units)
        self.activation = activation or "linear"
        self.use_bias = use_bias
        self.kernel_initializer = kernel_initializer
        self.bias_initializer = bias_initializer
        self.kernel: Optional[torch.Tensor] = None
        self.bias: Optional[torch.Tensor] = None
        self.input_dim: Optional[int] = None
        self._w_split: Optional[torch.Tensor] = None
        self._split_bufs: Dict[tuple, torch.Tensor] = {}

    _TRANSIENT = {"_w_split": None, "_split_bufs": {}, "_bias_host": None}

    def _weights_changed(self) -> None:
        """Variables were assigned (load_weights): drop everything derived from them.  Captured CUDA graphs hold raw
        pointers to the derived buffers (and the fused head's bias as a scalar argument): the bumped weights version
        makes graph.CompiledForward re-capture before its next replay."""
        from .core import bump_weights_version

        self._w_split = None
        self._bias_host = None
        bump_weights_version()

    def split_kernel(self) -> torch.Tensor:
        """(Np, 2*Kp) split-bf16 K-major copy of the kernel for the tensor-core path (built once)."""
        if self._w_split is None:
            self._w_split = ops.split_weights(self.kernel)
        return self._w_split

    def split_buffer(self, B: int, device) -> torch.Tensor:
        """Cached (B, 2*Kp(units)) bf16 buffer receiving this layer's output as the next layer's
        operand; its padding columns are zeroed once and never written again."""
        key = (B, buffer_namespace())
        buf = self._split_bufs.get(key)
        if buf is None or buf.device != device:
            if len(self._split_bufs) > 8:
                self._split_bufs = {k: v for k, v in self._split_bufs.items() if k[1] != 0}  # keep graph-owned buffers
            buf = torch.zeros((B, 2 * ops.tc_padded_k(self.units)), dtype=torch.bfloat16, device=device)
            self._split_bufs[key] = buf
        return buf

    def bias_value(self) -> float:
        """Scalar bias of a 1-unit layer (cached on the host: it is a kernel argument of the fused head)."""
        if self.bias is None:
            return 0.0
        if getattr(self, "_bias_host", None) is None:
            self._bias_host = float(self.bias.reshape(-1)[0].item())
        return self._bias_host

    def build(self, input_dim: Optional[int] = None, device=None) -> "_Dense":
        if self.kernel is None:
            if input_dim is None:
                raise ValueError(f"{self.name}: cannot build without the input width")
            device = device or default_device()
            self.input_dim = int(input_dim)
            self.kernel = create_variable((input_dim, self.units), self.kernel_initializer, device, f"{self.name}/kernel")
            if self.use_bias:
                self.bias = create_variable((self.units,), self.bias_initializer, device, f"{self.name}/bias")
        self.built = True
        return self

    def set_weights(self, kernel, bias=None) -> None:
        dev = default_device()
        self.kernel = torch.as_tensor(kernel, dtype=torch.float32).to(dev).contiguous()
        self.input_dim = self.kernel.shape[0]
        if self.kernel.shape[1] != self.units:
            raise ValueError(f"{self.name}: kernel has {self.kernel.shape[1]} columns, expected {self.units}")
        self.bias = None if bias is None else torch.as_tensor(bias, dtype=torch.float32).to(dev).contiguous()
        self.use_bias = bias is not None
        self._weights_changed()
        self.built = True

    def weights(self):
        out = {"kernel": self.kernel}
        if self.bias is not None:
            out["bias"] = self.bias
        return out

    def call(self, inputs, x0: Optional[torch.Tensor] = None, **kwargs) -> torch.Tensor:
        x = concat_sorted(inputs) if isinstance(inputs, dict) else inputs
        if x.dim() != 2:
            raise ValueError(f"{self.name}: expected a 2-D input, got shape {tuple(x.shape)}")
        self.build(x.shape[1], x.device)
        if x.shape[1] != self.input_dim:
            raise ValueError(f"{self.name}: input width {x.shape[1]} != kernel rows {self.input_dim}")
        out = torch.empty((x.shape[0], self.units), dtype=torch.float32, device=x.device)
        if x0 is None and not _use_tc():
            return ops.dense_fp32(x, self.kernel, self.bias, self.activation, out)
        if x0 is None:
            ops.dense_tc(ops.split_rows(x), self.input_dim, self.split_kernel(), self.units, self.bias, self.activation,
                         out_f32=out)
            return out
        return ops.dense_fp32(x, self.kernel, self.bias, self.activation, out, x0=x0)


class BatchNormalization(Block):
    """tf.keras.layers.BatchNormalization as MLPBlock(normalization="batch_norm") appends it after every Dense
    (blocks/mlp.py:131-135), INFERENCE semantics: y = (x - moving_mean) / sqrt(moving_var + eps) * gamma + beta,
    eps = 1e-3, fresh variables gamma = 1, beta = 0, moving_mean = 0, moving_var = 1.  On the forward path it never
    runs as a layer of its own when a Dense follows: MLP.chain() folds it into that Dense's kernel and bias."""

    def __init__(self, axis: int = -1, momentum: float = 0.99, epsilon: float = 1e-3, center: bool = True, scale: bool = True,
                 name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("batch_normalization"))
        if axis not in (-1, 1):
            raise ValueError("BatchNormalization: only the feature axis (-1) is supported")
        self.epsilon, self.momentum, self.center, self.scale = float(epsilon), float(momentum), center, scale
        self.gamma = self.beta = self.moving_mean = self.moving_variance = None
        self._st = None

    _TRANSIENT = {"_st": None}

    def build(self, width: Optional[int] = None, device=None) -> "BatchNormalization":
        if self.gamma is None:
            if width is None:
                raise ValueError(f"{self.name}: cannot build without the input width")
            device = device or default_device()
            self.gamma = torch.ones(width, dtype=torch.float32, device=device)
            self.beta = torch.zeros(width, dtype=torch.float32, device=device)
            self.moving_mean = torch.zeros(width, dtype=torch.float32, device=device)
            self.moving_variance = torch.ones(width, dtype=torch.float32, device=device)
        self.built = True
        return self

    def set_weights(self, gamma=None, beta=None, moving_mean=None, moving_variance=None) -> None:
        dev = default_device()
        for name, v in (("gamma", gamma), ("beta", beta), ("moving_mean", moving_mean), ("moving_variance", moving_variance)):
            if v is not None:
                setattr(self, name, torch.as_tensor(v, dtype=torch.float32).to(dev).contiguous())
        self._weights_changed()
        self.built = True

    def _weights_changed(self) -> None:
        from .core import bump_weights_version

        self._st = None
        bump_weights_version()

    def weights(self):
        return {"gamma": self.gamma, "beta": self.beta, "moving_mean": self.moving_mean, "moving_variance": self.moving_variance}

    def scale_shift(self):
        """(scale, shift) with y = x * scale + shift (set-up time torch arithmetic, cached)."""
        if self._st is None:
            s = self.gamma / torch.sqrt(self.moving_variance + self.epsilon)
            self._st = (s.contiguous(), (self.beta - self.moving_mean * s).contiguous())
        return self._st

    def call(self, inputs, training: bool = False, **kwargs):
        if training:
            raise NotImplementedError("BatchNormalization with batch statistics (training=True) is outside the forward hot path")
        self.build(inputs.shape[1], inputs.device)
        s, t = self.scale_shift()
        return ops.scale_shift(inputs, s, t)


class MLP(SequentialBlock):
    """The SequentialBlock MLPBlock() returns; `.layers` are the _Dense layers (each optionally followed by a
    BatchNormalization, blocks/mlp.py:108-135; dropout is identity at inference and is not a layer here)."""

    def __init__(self, layers: Sequence[_Dense], filter_names: Optional[List[str]] = None, block_name: str = "MLPBlock",
                 dropout: Optional[float] = None):
        super().__init__(layers, block_name=block_name)
        self.filter_names = filter_names
        self.dropout = dropout

    @property
    def dense_layers(self) -> List[_Dense]:
        return [l for l in self.layers if isinstance(l, _Dense)]

    def build_from_width(self, width: int, device=None) -> "MLP":
        for l in self.layers:
            if isinstance(l, _Dense):
                l.build(width, device)
                width = l.units
            elif isinstance(l, BatchNormalization):
                l.build(width, device)
        self.built = True
        return self

    @property
    def has_normalization(self) -> bool:
        return any(isinstance(l, BatchNormalization) for l in self.layers)

    def chain(self, extra: Sequence[_Dense] = ()):
        """(dense layers to run, trailing normalization or None) for this block followed by the Dense layers `extra`
        (e.g. the output head).  Every BatchNormalization that is followed by a Dense is folded into it:
        (x * s + t) W + b = x (diag(s) W) + (b + t W) — the folded layers are cached shadow _Dense objects, rebuilt when
        any variable is reassigned.  The block must be built."""
        if not self.has_normalization:
            return self.dense_layers + list(extra), None
        from .core import weights_version

        key = (weights_version(), tuple(id(e) for e in extra))
        if getattr(self, "_chain_key", None) == key:
            return self._chain
        out, pending = [], None
        for l in list(self.layers) + list(extra):
            if isinstance(l, BatchNormalization):
                if pending is not None:
                    raise NotImplementedError("two normalizations in a row")
                pending = l
            elif isinstance(l, _Dense):
                if pending is None:
                    out.append(l)
                    continue
                if l.kernel is None or pending.gamma is None:
                    raise RuntimeError("MLP.chain(): build the block first")
                s, t = pending.scale_shift()
                f = _Dense(l.units, activation=l.activation, use_bias=True, name=f"{l.name}/folded_bn")
                # assigned directly: a derived layer is not a variable assignment (no weights-version bump)
                f.kernel = (s.unsqueeze(1) * l.kernel).contiguous()
                f.bias = (t @ l.kernel if l.bias is None else l.bias + t @ l.kernel).contiguous()
                f.input_dim, f.built = l.kernel.shape[0], True
                out.append(f)
                pending = None
        self._chain, self._chain_key = (out, pending), key
        return self._chain

    _TRANSIENT = {"_chain": None, "_chain_key": None}

    def call(self, inputs, training: bool = False, operand_out: bool = False, **kwargs):
        if self.dropout and training:
            raise NotImplementedError("dropout in training mode is outside the forward hot path")
        if self.has_normalization and training:
            raise NotImplementedError("BatchNormalization with batch statistics (training=True) is outside the forward hot path")
        x = inputs
        a = K = None
        if isinstance(x, dict):
            if self.filter_names is not None:
                x = {k: v for k, v in x.items() if k in self.filter_names}
            pieces = [x[k] for k in sorted(x)]
            if _use_tc() and _SMALL_TOWER[0] and batch_size_of(x) > 0:
                # narrow-input two-layer tower (the DLRM bottom tower): columns -> layer 1 -> layer 2 in one launch
                K_in = sum(1 if t.dim() == 1 else int(t.shape[1]) for t in pieces)
                self.build_from_width(K_in, pieces[0].device)
                layers, tail = self.chain()
                if (tail is None and len(layers) == 2 and layers[0].input_dim == K_in
                        and ops.tower2_small_supported(pieces, layers[0].units, layers[1].units)):
                    B = batch_size_of(x)
                    l1, l2 = layers
                    _LAST_PATH[0] = "tower2_small"
                    if operand_out:
                        out = torch.empty((B, 2 * l2.units), dtype=torch.bfloat16, device=pieces[0].device)
                        ops.tower2_small(pieces, l1.split_kernel(), l1.units, l1.bias, l1.activation, l2.split_kernel(), l2.units,
                                         l2.bias, l2.activation, out_split=out)
                    else:
                        out = torch.empty((B, l2.units), dtype=torch.float32, device=pieces[0].device)
                        ops.tower2_small(pieces, l1.split_kernel(), l1.units, l1.bias, l1.activation, l2.split_kernel(), l2.units,
                                         l2.bias, l2.activation, out=out)
                    return out
            if _use_tc() and ops.concat_split_supported(pieces) and batch_size_of(x) > 0:
                # ConcatFeatures straight into the split-bf16 operand of the first tensor-core layer
                a, K = ops.concat_split(pieces)
                x = None
            else:
                x = concat_sorted(x)
        width = K if x is None else x.shape[1]
        self.build_from_width(width, a.device if x is None else x.device)
        layers, tail = self.chain()
        if tail is not None:  # a trailing normalization runs on fp32 rows
            out = tail(run_dense_chain(x, layers, a_split=a, K=K) if x is None else run_dense_chain(x, layers))
            return ops.split_rows(out) if operand_out else out
        return (run_dense_chain(x, layers, a_split=a, K=K, operand_out=operand_out) if x is None
                else run_dense_chain(x, layers, operand_out=operand_out))

    def oracle_layers(self):
        return [{"kernel": l.kernel.cpu().numpy(), "bias": None if l.bias is None else l.bias.cpu().numpy(),
                 "activation": l.activation} for l in self.dense_layers]


def MLPBlock(dimensions: List[int], activation: Union[str, List[str]] = "relu", use_bias: bool = True,
             kernel_initializer: InitializerType = "glorot_uniform", bias_initializer: InitializerType = "zeros",
             kernel_regularizer=None, bias_regularizer=None, activity_regularizer=None, dropout: Optional[float] = None,
             normalization=None, filter: Optional[Union[Schema, Tags, List[str]]] = None,
             no_activation_last_layer: bool = False, block_name: str = "MLPBlock", **kwargs) -> MLP:
    """blocks/mlp.py:35-139.  Activation is applied on every layer including the last unless
    `no_activation_last_layer` (:99-106).  Regularizers only matter for training and are accepted
    and ignored.  `normalization="batch_norm"` (or a BatchNormalization instance, deep-copied per layer) follows every
    Dense as in the reference (:131-135); at inference it is folded into the next Dense."""
    if isinstance(activation, list) and len(activation) != len(dimensions):
        raise ValueError(
            f"Activation and Dimensions length mismatch. \
        Activation length: {len(activation)}, Dimensions length: {len(dimensions)}"
        )
    if normalization is not None and normalization != "batch_norm" and not isinstance(normalization, BatchNormalization):
        raise ValueError("Normalization needs to be an instance `Layer` or " "`batch_norm`")
    layers = []
    for idx, dim in enumerate(dimensions):
        act = activation or "linear"
        act_i = act if isinstance(act, str) else act[idx]
        if no_activation_last_layer and idx == len(dimensions) - 1:
            act_i = "linear"
        layers.append(_Dense(dim, activation=act_i, use_bias=use_bias, kernel_initializer=kernel_initializer,
                             bias_initializer=bias_initializer))
        if normalization == "batch_norm":
            layers.append(BatchNormalization())
        elif normalization is not None:
            layers.append(BatchNormalization(epsilon=normalization.epsilon, momentum=normalization.momentum))
    names = None
    if filter is not None:
        if isinstance(filter, Schema):
            names = filter.column_names
        elif isinstance(filter, (list, tuple)):
            names = list(filter)
        else:
            raise ValueError("MLPBlock(filter=Tags) needs a schema; pass a Schema or a list of names")
    return MLP(layers, filter_names=names, block_name=block_name, dropout=dropout)


class FMPairwiseInteraction(Block):
    """blocks/interaction.py:205-253: inputs (bs, n_features, embedding_dim) -> 0.5 * ((sum over axis 1)^2 - sum over axis 1
    of the squares), shape (bs, embedding_dim)."""

    def __init__(self, name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("fm_pairwise_interaction"))

    def call(self, inputs: torch.Tensor, **kwargs) -> torch.Tensor:
        assert inputs.dim() == 3, "inputs should be a 3-D tensor"
        return ops.fm_pairwise(inputs.contiguous())


class FM(Block):
    """What FMBlock() returns (blocks/interaction.py:256-332): (B, 1) = wide + pairwise.

    wide     `Dense(1, linear)` over concat(one-hot of every categorical feature, continuous features) in sorted-name order
             (CategoryEncoding(multi_hot) + ToSparse + "concat", :307-316).  The Keras kernel has one row per category
             of every feature (int_domain.max + 1 rows each) and one per continuous feature; the product with a one-hot
             vector is a row lookup.
    pairwise the embeddings (dim = factors_dim) are stacked on the LAST axis (StackFeatures(axis=-1)) before
             FMPairwiseInteraction, which reduces axis 1: per feature 0.5 ((sum_d e)^2 - sum_d e^2), then summed over the
             features (:323-328).  Restated as the reference computes it.
    One-hot categorical features only (list columns would need the multi-hot wide encoding)."""

    def __init__(self, schema: Schema, embeddings: EmbeddingsBlock, name: Optional[str] = None):
        super().__init__(name or unique_name("fm_block"))
        cat = schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)
        cont = schema.select_by_tag(Tags.CONTINUOUS).excluding_by_tag(Tags.TARGET)
        if not len(cat):
            raise ValueError("FMBlock requires categorical features")
        lists = [c.name for c in cat if c.is_list]
        if lists:
            raise NotImplementedError(f"FMBlock: list (multi-hot) categorical features {lists} are not implemented")
        self.embeddings = embeddings
        self.cat_names = [c.name for c in cat]
        self.cont_names = [c.name for c in cont]
        dims = {embeddings.feature_to_table[f].dim for f in self.cat_names}
        if len(dims) != 1:
            raise ValueError(f"FMBlock needs all embedding tables to share one dimension, got {sorted(dims)}")
        self.dim = dims.pop()
        # rows of the wide kernel: sorted over ALL feature names (ConcatFeatures, core/aggregation.py:54-66)
        self.wide_offsets: Dict[str, int] = {}
        off = 0
        for n in sorted(self.cat_names + self.cont_names):
            self.wide_offsets[n] = off
            off += (int(schema.get(n).int_domain.max) + 1) if n in self.cat_names else 1
        self.wide_width = off
        self.wide = _Dense(1, activation="linear", use_bias=True, name=f"{self.name}/wide_logit")

    def build(self, device=None):
        self.embeddings.build(device)
        self.wide.build(self.wide_width, device)
        self.built = True
        return self

    def weights(self):
        return {f"wide/{k}": v for k, v in self.wide.weights().items()}

    def head(self, inputs: TabularData, addend: Optional[torch.Tensor] = None, out_layer: Optional["_Dense"] = None) -> torch.Tensor:
        """(B, 1) = [out_layer](wide + pairwise [+ addend]) in one kernel (ops.deepfm_head)."""
        from .core import get_feature
        from .inputs import _as_index

        dev = next(iter(inputs.values())).device
        self.build(dev)
        B = batch_size_of(inputs)
        emb = self.embeddings
        raw = [get_feature(inputs, f) for f in self.cat_names]
        idx = [i if i.dtype in (torch.uint8, torch.uint16) else _as_index(i).reshape(-1) for i in raw]
        tabs = [emb.feature_to_table[f].table for f in self.cat_names]
        cont = []
        for n in self.cont_names:
            if n not in inputs:
                raise ValueError(f"missing continuous feature {n!r}")
            cont.append(inputs[n])
        out = torch.empty((B, 1), dtype=torch.float32, device=dev)
        oob = emb.counter(dev)
        ow = ob = act = None
        if out_layer is not None:
            out_layer.build(1, dev)
            ow, ob, act = out_layer.kernel.reshape(-1), out_layer.bias, out_layer.activation
        ops.deepfm_head(tabs, idx, [self.wide_offsets[f] for f in self.cat_names], cont, [self.wide_offsets[n] for n in self.cont_names],
                        self.wide.kernel.reshape(-1), self.wide.bias, None if addend is None else addend.reshape(-1), ow, ob, act,
                        out.reshape(-1), oob)
        emb.finish_check(oob)
        return out

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        return self.head(inputs)


def FMBlock(schema: Schema, fm_input_block=None, wide_input_block=None, wide_logit_block=None, factors_dim: Optional[int] = None,
            **kwargs) -> FM:
    """blocks/interaction.py:256-332 with the default wide blocks (custom wide_input_block / wide_logit_block are not
    implemented).  fm_input_block: an InputBlockV2 / EmbeddingsBlock whose tables are used for the pairwise term;
    default: Embeddings(categorical schema, dim=factors_dim)."""
    if wide_input_block is not None or wide_logit_block is not None:
        raise NotImplementedError("FMBlock: custom wide_input_block / wide_logit_block are not implemented")
    cat = schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)
    if fm_input_block is None:
        if factors_dim is None:
            raise ValueError("FMBlock needs `factors_dim` when no fm_input_block is given")
        emb = Embeddings(cat, dim=factors_dim)
    else:
        emb = fm_input_block if isinstance(fm_input_block, EmbeddingsBlock) else getattr(fm_input_block, "embeddings", None)
        if emb is None:
            raise ValueError("fm_input_block must be an InputBlockV2 with embeddings or an Embeddings block")
    return FM(schema, emb)


_INTERACTION_TYPES = (None, "field_all", "field_each", "field_interaction")


class DotProductInteraction(Block):
    """blocks/interaction.py:35-130 with interaction_type=None: (B,F,D) -> (B, F(F-1)/2) strict
    upper triangle of X X^T, row-major ((B, F(F+1)/2) with self_interaction)."""

    def __init__(self, interaction_type=None, self_interaction: bool = False, name: Optional[str] = None, **kwargs):
        if interaction_type not in _INTERACTION_TYPES:
            raise ValueError("Unknown interaction type {}".format(interaction_type))
        if interaction_type is not None:
            raise NotImplementedError("FiBiNet bilinear interaction types are outside the DLRM hot path")
        super().__init__(name or unique_name("dot_product_interaction"))
        self.interaction_type = interaction_type
        self.self_interaction = self_interaction

    def compute_output_shape(self, input_shape):
        F = input_shape[1]
        return input_shape[0], (F * (F + 1) // 2 if self.self_interaction else F * (F - 1) // 2)

    def call(self, inputs: torch.Tensor, prefix: Optional[torch.Tensor] = None, **kwargs) -> torch.Tensor:
        if inputs.dim() != 3:
            raise ValueError(f"DotProductInteraction expects (batch, features, dim), got {tuple(inputs.shape)}")
        B, n = self.compute_output_shape(inputs.shape)
        P = 0 if prefix is None else prefix.shape[1]
        out = torch.empty((B, P + n), dtype=torch.float32, device=inputs.device)
        return ops.dot_interaction(inputs.contiguous(), out, prefix=prefix, self_interaction=self.self_interaction)


class Cross(Block):
    """blocks/cross.py:113-221: x_{l+1} = x0 * (x_l W + b) + x_l (full rank) or W = U V."""

    def __init__(self, low_rank_dim: Optional[int] = None, use_bias: bool = True,
                 kernel_initializer: InitializerType = "truncated_normal", bias_initializer: InitializerType = "zeros",
                 output_x0: bool = False, name: Optional[str] = None, **kwargs):
        super().__init__(name or unique_name("cross"))
        self.low_rank_dim = low_rank_dim
        self.use_bias = use_bias
        self.kernel_initializer = kernel_initializer
        self.bias_initializer = bias_initializer
        self.output_x0 = output_x0
        self.dense: Optional[_Dense] = None
        self.dense_u: Optional[_Dense] = None

    def build(self, d: Optional[int] = None, device=None):
        if self.dense is None:
            if d is None:
                raise ValueError("Cross: cannot build without the input width")
            self.dense = _Dense(d, activation="linear", use_bias=self.use_bias,
                                kernel_initializer=self.kernel_initializer, bias_initializer=self.bias_initializer,
                                name=f"{self.name}/dense")
            if self.low_rank_dim is not None:
                self.dense_u = _Dense(self.low_rank_dim, activation="linear", use_bias=False,
                                      kernel_initializer=self.kernel_initializer, name=f"{self.name}/dense_u")
                self.dense_u.build(d, device)
                self.dense.build(self.low_rank_dim, device)
            else:
                self.dense.build(d, device)
        self.built = True
        return self

    def weights(self):
        out = {f"dense/{k}": v for k, v in self.dense.weights().items()}
        if self.dense_u is not None:
            out["dense_u/kernel"] = self.dense_u.kernel
        return out

    def call(self, inputs, **kwargs):
        x0, x = inputs if isinstance(inputs, tuple) else (inputs, inputs)
        if tuple(x0.shape) != tuple(x.shape):
            raise ValueError("`x0` ({}) and `x` ({}) shapes mismatch!".format(tuple(x0.shape), tuple(x.shape)))
        self.build(x.shape[1], x.device)
        if self.dense_u is None:
            out = self.dense(x, x0=x0)  # fused epilogue x0 * (xW + b) + x
        else:
            out = _cross_lowrank(self.dense_u, self.dense, x0, x)
        return (x0, out) if self.output_x0 else out


def _cross_lowrank(dense_u: _Dense, dense: _Dense, x0, x):
    """DenseMaybeLowRank (blocks/mlp.py:389-396): projection = dense(dense_u(x)) with dense_u (d -> r, no bias) and
    dense (r -> d, bias); then the cross x0 * projection + x (blocks/cross.py:196-198).  Two GEMMs: U emits the
    split-bf16 operand of V directly, V runs with the cross epilogue (K = r, N = d)."""
    B, d = x.shape
    out = torch.empty((B, d), dtype=torch.float32, device=x.device)
    if not _use_tc():
        u = ops.dense_fp32(x, dense_u.kernel, None, dense_u.activation, torch.empty((B, dense_u.units), dtype=torch.float32, device=x.device))
        proj = ops.dense_fp32(u, dense.kernel, dense.bias, dense.activation, torch.empty_like(x))
        return ops.cross_combine(x0, proj, x, out)
    r = dense_u.units
    ubuf = dense_u.split_buffer(B, x.device)
    ops.dense_tc(ops.split_rows(x), d, dense_u.split_kernel(), r, None, dense_u.activation, out_split=ubuf)
    if dense.activation == "linear":
        ops.dense_tc(ubuf, r, dense.split_kernel(), d, dense.bias, "linear", out_f32=out, x0=x0, xres=x)
        return out
    proj = torch.empty_like(x)
    ops.dense_tc(ubuf, r, dense.split_kernel(), d, dense.bias, dense.activation, out_f32=proj)
    return ops.cross_combine(x0, proj, x, out)


class CrossBlockSeq(SequentialBlock):
    def __init__(self, layers, inputs: Optional[Block] = None):
        super().__init__(layers, block_name="CrossBlock")
        self.inputs = inputs

    @property
    def cross_layers(self) -> List[Cross]:
        return [l for l in self.layers if isinstance(l, Cross)]

    def call(self, x, **kwargs):
        if self.inputs is not None:
            x = self.inputs(x)
        if isinstance(x, dict):
            x = concat_sorted(x)
        layers = self.cross_layers
        if _use_tc() and all(l.low_rank_dim is None for l in layers):
            return self._call_tc(x, layers)
        for l in layers:
            x = l(x)
        return x

    def _call_tc(self, x0: torch.Tensor, layers) -> torch.Tensor:
        """x_{l+1} = x0 * (x_l W_l + b_l) + x_l with every layer one wgmma launch: the epilogue reads
        x0 and x_l (fp32) and writes x_{l+1} both as fp32 (next residual) and split-bf16 (next operand)."""
        B, d = x0.shape
        for l in layers:
            l.build(d, x0.device)
        a = ops.split_rows(x0)
        x = x0
        for i, l in enumerate(layers):
            last = i == len(layers) - 1
            out = torch.empty((B, d), dtype=torch.float32, device=x0.device)
            nxt = None if last else l.dense.split_buffer(B, x0.device)
            ops.dense_tc(a, d, l.dense.split_kernel(), d, l.dense.bias, "linear", out_f32=out, out_split=nxt, x0=x0, xres=x)
            a, x = nxt, out
        return x

    def oracle_layers(self):
        return [{"kernel": l.dense.kernel.cpu().numpy(),
                 "bias": None if l.dense.bias is None else l.dense.bias.cpu().numpy()} for l in self.cross_layers]


def CrossBlock(depth: int = 1, filter=None, low_rank_dim: Optional[int] = None, use_bias: bool = True,
               kernel_initializer: InitializerType = "truncated_normal", bias_initializer: InitializerType = "zeros",
               kernel_regularizer=None, bias_regularizer=None, inputs: Optional[Block] = None, **kwargs) -> CrossBlockSeq:
    """blocks/cross.py:29-109."""
    if depth <= 0:
        raise ValueError(f"Number of cross layers (depth) should be positive but is {depth}.")
    layers = [Cross(low_rank_dim=low_rank_dim, use_bias=use_bias, kernel_initializer=kernel_initializer,
                    bias_initializer=bias_initializer, output_x0=i < depth - 1) for i in range(depth)]
    return CrossBlockSeq(layers, inputs=inputs)


class DLRM(Block):
    """What DLRMBlock() returns (blocks/dlrm.py:32-133).

    forward:  embeddings (T x (B,D))  +  bottom MLP(continuous) (B,D)
              -> stack in sorted(name) order, "bottom_block" last for C*/I* style names
              -> pairwise dots (B, F(F-1)/2) -> [bottom | interactions] -> top MLP
    `fused=True` runs gather + stack + interaction + concat as ONE kernel (the (B,F,D) stack never
    reaches HBM); `fused=False` keeps the reference's staging ((B,F,D) materialised once) for
    block-level parity tests.
    """

    def __init__(self, embeddings: EmbeddingsBlock, continuous: Optional[ContinuousFeatures], bottom_block: Optional[MLP],
                 top_block: Optional[MLP], embedding_dim: int, fused: bool = True):
        super().__init__(unique_name("dlrm_block"))
        self.embeddings = embeddings
        self.continuous = continuous
        self.bottom_block = bottom_block
        self.top_block = top_block
        self.embedding_dim = embedding_dim
        self.fused = fused
        self.sharded = None  # models_b200.sharded.ShardedEmbeddings when the tables are row-sharded

    # stack order = sorted over {feature names} U {"bottom_block"} (core/aggregation.py:104-108)
    def slots(self) -> Dict[str, int]:
        keys = list(self.embeddings.feature_names)
        if self.bottom_block is not None:
            keys.append("bottom_block")
        return {k: i for i, k in enumerate(sorted(keys))}

    def build(self, device=None):
        if self.sharded is not None:
            self.sharded.build(device)  # local shards only: full tables are never materialised
        else:
            self.embeddings.build(device)
        if self.bottom_block is not None:
            self.bottom_block.build_from_width(len(self.continuous.features), device)
        if self.top_block is not None:
            self.top_block.build_from_width(self.output_width_before_top(), device)
        self.built = True
        return self

    def output_width_before_top(self) -> int:
        F = len(self.embeddings.feature_names) + (1 if self.bottom_block is not None else 0)
        return F * (F - 1) // 2 + (self.embedding_dim if (self.bottom_block is not None and self.top_block is not None) else 0)

    def weights(self):
        out = {f"embeddings/{k}": v for k, v in self.embeddings.weights().items()}
        if self.bottom_block is not None:
            out.update({f"bottom_block/{k}": v for k, v in self.bottom_block.weights().items()})
        if self.top_block is not None:
            out.update({f"top_block/{k}": v for k, v in self.top_block.weights().items()})
        return out

    def can_emit_split(self) -> bool:
        """True when the tensor-core interaction kernel applies (F <= 32, D % 16 == 0)."""
        F = len(self.embeddings.feature_names) + (1 if self.bottom_block is not None else 0)
        return 2 <= F <= 32 and self.embedding_dim in (16, 32, 64, 128)

    def bottom_forward(self, inputs: TabularData, operand_out: bool = False) -> Optional[torch.Tensor]:
        """Bottom MLP over the continuous columns: (B, D) fp32, or — operand_out — the same rows in the interaction
        kernel's operand format (written by the tower kernel's last epilogue, no fp32 round trip)."""
        if self.bottom_block is None:
            return None
        return self.bottom_block(self.continuous(inputs), operand_out=operand_out)

    def use_operand_rows(self, as_split: bool = True) -> bool:
        """Operand-format table mirrors + operand-format bottom vector for the fused kernel: only on the production
        path (split-bf16 output feeding the top MLP), when mirrors are enabled (blocks.set_table_mirror)."""
        ok = bool(as_split and self.fused and table_mirror() and self.can_emit_split() and self.bottom_block is not None
                  and self.top_block is not None and self.embedding_dim == 64)
        if ok and self.sharded is not None:
            ok = bool(self.sharded.mirrors)  # built collectively in ShardedEmbeddings.build (never lazily inside a step)
        return ok

    def interaction_forward(self, inputs: TabularData, bottom: Optional[torch.Tensor], as_split: bool = False,
                            operand_rows: bool = False) -> torch.Tensor:
        """[bottom |] interactions, (B, P + F(F-1)/2) fp32 — or, with as_split, the split-bf16 operand
        (B, 2*Kp) of the top MLP's first tensor-core layer, written directly by the kernel.  operand_rows: `bottom` is in
        operand format and the tables' operand-format mirrors are used (see use_operand_rows)."""
        self.build(next(iter(inputs.values())).device)
        D = self.embedding_dim
        slots = self.slots()
        F = len(slots)
        B = batch_size_of(inputs)
        dev = next(iter(inputs.values())).device
        with_prefix = bottom is not None and self.top_block is not None
        P = D if with_prefix else 0
        width = P + F * (F - 1) // 2
        if as_split:
            out = torch.empty((B, 2 * ops.tc_padded_k(width)), dtype=torch.bfloat16, device=dev)
        else:
            out = torch.empty((B, width), dtype=torch.float32, device=dev)
        emb = self.embeddings
        feats = emb.feature_names
        from .core import get_feature
        from .inputs import _as_index, _raise_on_oob

        if self.sharded is not None:
            oob = emb.counter(dev)
            if with_prefix == (bottom is not None) and self.can_emit_split():
                # row-sharded tables, product path: the lookup is part of the interaction kernel — rows owned
                # by other ranks are read over NVLink straight into shared memory (no exchange, no barrier)
                self.sharded.lookup_interact(inputs, slots, bottom, out, oob, operand_rows=operand_rows)
                emb.finish_check(oob)
                return out
            # staged protocol (index all-gather + owner-computes NVLink push + barrier) rebuilds the (B,F,D)
            # stack of the local samples; the interaction then reads it like the staged path
            stack = self.sharded.lookup_stack(inputs, slots, F, oob)
            emb.finish_check(oob)
            if bottom is not None:
                ops.concat_columns([bottom], stack, [slots["bottom_block"] * D])
            return ops.dot_interaction(stack.view(B, F, D), out, prefix=bottom if with_prefix else None)
        all_onehot = all(emb.feature_to_table[f].lookup_kind(get_feature(inputs, f)) == "onehot" for f in feats)
        if self.fused and all_onehot and with_prefix == (bottom is not None):
            oob = emb.counter(dev)
            raw = [get_feature(inputs, f) for f in feats]
            if self.can_emit_split():
                # ids travel at their own width (packed uint8 / uint16 / 24-bit host batches, int32, int64)
                idx = [i if i.dtype in (torch.uint8, torch.uint16) else _as_index(i).reshape(-1) for i in raw]
                tabs = [emb.feature_to_table[f].operand_mirror() if operand_rows else emb.feature_to_table[f].table for f in feats]
                ops.dlrm_lookup_interact(tabs, idx, [slots[f] for f in feats], [t.shape[0] for t in tabs], D, bottom,
                                         slots.get("bottom_block", -1), out, oob, operand_rows=operand_rows)
            else:
                idx = [_as_index(i).reshape(-1) for i in raw]
                if len({i.dtype for i in idx}) > 1:
                    idx = [i.to(torch.int64) for i in idx]
                ops.dlrm_gather_interact([emb.feature_to_table[f].table for f in feats], idx, [slots[f] for f in feats], D,
                                         bottom, slots.get("bottom_block", -1), out, oob)
            emb.finish_check(oob)
            return out
        # staged path: one fused gather into the (B,F,D) stack, then the interaction kernel
        stack = torch.empty((B, F * D), dtype=torch.float32, device=dev)
        emb.lookup_all_into(inputs, stack, {f: slots[f] * D for f in feats})
        if bottom is not None:
            ops.concat_columns([bottom], stack, [slots["bottom_block"] * D])
        return ops.dot_interaction(stack.view(B, F, D), out, prefix=bottom if with_prefix else None)

    def call(self, inputs: TabularData, **kwargs) -> torch.Tensor:
        bottom = self.bottom_forward(inputs)
        x = self.interaction_forward(inputs, bottom)
        if self.top_block is not None:
            x = self.top_block(x)
        return x


def DLRMBlock(schema: Schema, *, embedding_dim: int = None, embedding_options: EmbeddingOptions = None,
              embeddings: Optional[EmbeddingsBlock] = None, bottom_block: Optional[MLP] = None,
              top_block: Optional[MLP] = None) -> DLRM:
    """blocks/dlrm.py:32-133 (same checks, same messages)."""
    if schema is None:
        raise ValueError("The schema is required by DLRM")
    con_schema = schema.select_by_tag(Tags.CONTINUOUS).excluding_by_tag(Tags.TARGET)
    cat_schema = schema.select_by_tag(Tags.CATEGORICAL).excluding_by_tag(Tags.TARGET)
    if not len(cat_schema) > 0:
        raise ValueError("DLRM requires categorical features")
    if embeddings is not None and embedding_options is not None:
        raise ValueError("Only one-of `embeddings` or `embedding_options` may be provided.")
    if embeddings is None:
        embeddings = _get_embeddings(embedding_dim, embedding_options, bottom_block, cat_schema)
    dims = set(embeddings.output_dims().values())
    if len(dims) != 1:
        raise ValueError(f"DLRM needs all embedding tables to share one dimension, got {sorted(dims)}")
    dim = dims.pop()
    continuous = None
    if len(con_schema) > 0:
        if bottom_block is None:
            raise ValueError(
                "The bottom_block is required by DLRM when "
                "continuous features are available in the schema"
            )
        continuous = ContinuousFeatures.from_schema(con_schema)
        last_units = bottom_block.dense_layers[-1].units
        if last_units != dim:
            raise ValueError(
                f"The embedding_dim ({dim}) needs to match the "
                f"last layer of bottom MLP ({last_units}) "
            )
    else:
        bottom_block = None
    return DLRM(embeddings, continuous, bottom_block, top_block, dim)


def _get_embeddings(embedding_dim, embedding_options, bottom_block, cat_schema) -> EmbeddingsBlock:
    """blocks/dlrm.py:136-166."""
    if embedding_dim is None:
        raise ValueError("The embedding_dim is required")
    if embedding_options is not None:
        embedding_options.embedding_dim_default = embedding_dim
    else:
        embedding_options = EmbeddingOptions(embedding_dim_default=embedding_dim)
    if embedding_dim is not None and bottom_block is not None:
        last = bottom_block.dense_layers[-1]
        if embedding_dim != last.units:
            raise ValueError(
                f"The embedding_dim ({embedding_dim}) needs to match the "
                f"last layer of bottom MLP ({last.units}) "
            )
    return Embeddings(cat_schema, sequence_combiner=embedding_options.combiner,
                      embeddings_initializer=embedding_options.embeddings_initializers,
                      dim=embedding_options.embedding_dim_default)
