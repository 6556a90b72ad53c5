"""Multi-gate mixture of experts (merlin/models/tf/blocks/experts.py:37-208): MMOEBlock.

`MMOEBlock(outputs, expert_block, num_experts)` makes num_experts independent copies of expert_block, `expert_0 ..
expert_{E-1}`, that all read the block's input x, and one gate per output: softmax(gate_final(x) / T) with gate_final a
bias-free Dense(E), glorot-uniform.  Gate t returns m_t = sum_e p_t,e expert_e(x).  The reference stacks the experts'
outputs in sorted-name order (StackFeatures over a dict keyed by name), so gate column e pairs with the e-th name in that
order: expert_0, expert_1, expert_10, expert_11, expert_2, ... from 11 experts on.

The block owns the experts' layer as ONE stacked Dense (d -> E U) whose column block e is the expert with the e-th sorted
name.  Without a gate_block the gates are one stacked bias-free Dense (d -> H E) whose column block t is the gate of
output t (output order of the model's output block); with one, gate t is its own copy of gate_block followed by its
gate_final.  Each expert's (and stacked gate's) own variables are views of the stacked layers.  Without task towers the
mixture and the heads after it are one kernel (ops.mmoe_heads_fwd_bwd); with them ops.mmoe_mix_fwd / mmoe_mix_bwd.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .blocks import MLP, _Dense
from .core import Block, unique_name


def _output_names(outputs) -> List[str]:
    from .models import BinaryOutput, ParallelOutputs

    if isinstance(outputs, ParallelOutputs):
        return list(outputs.names)
    if isinstance(outputs, BinaryOutput):
        return [outputs.name]
    if isinstance(outputs, (list, tuple)) and outputs and all(isinstance(n, str) for n in outputs):
        return list(outputs)
    raise ValueError("MMOEBlock: outputs must be a list of output names or the output block (OutputBlock(schema))")


class MMOEBlock(Block):
    """blocks/experts.py:37-140.  Implemented for an expert_block that is one Dense layer (MLPBlock([units])).  Without a
    gate_block the gates are one stacked bias-free Dense; with one, gate t is its own copy of gate_block followed by its
    gate_final."""

    def __init__(self, outputs, expert_block: MLP, num_experts: int, gate_block: Optional[Block] = None,
                 gate_softmax_temperature: float = 1.0, enable_gate_weights_metrics: bool = False, name: Optional[str] = None,
                 **kwargs):
        super().__init__(name or "mmoe")
        if enable_gate_weights_metrics:
            raise NotImplementedError("MMOEBlock(enable_gate_weights_metrics=True): gate-weight metrics are not implemented")
        if gate_block is not None and (not isinstance(gate_block, MLP) or gate_block.has_normalization):
            raise NotImplementedError(f"MMOEBlock: gate_block must be an MLPBlock without normalization, got {gate_block!r}")
        if not isinstance(expert_block, MLP) or len(expert_block.dense_layers) != 1 or expert_block.has_normalization:
            raise NotImplementedError("MMOEBlock: the expert_block must be one Dense layer without normalization "
                                      "(MLPBlock([units])); deeper experts are not implemented")
        from .ops import MMOE_MAX_EXPERTS, MMOE_MAX_TASKS, MMOE_MAX_UNITS

        E = int(num_experts)
        if not 1 <= E <= MMOE_MAX_EXPERTS:
            raise NotImplementedError(f"MMOEBlock: 1..{MMOE_MAX_EXPERTS} experts are supported, got {num_experts}")
        proto = expert_block.dense_layers[0]
        if proto.units > MMOE_MAX_UNITS:
            raise NotImplementedError(f"MMOEBlock: experts of at most {MMOE_MAX_UNITS} units are supported, got {proto.units}")
        if not float(gate_softmax_temperature) > 0:
            raise ValueError(f"gate_softmax_temperature must be > 0, got {gate_softmax_temperature}")
        self.output_names = _output_names(outputs)
        if len(set(self.output_names)) != len(self.output_names) or len(self.output_names) > MMOE_MAX_TASKS:
            raise NotImplementedError(f"MMOEBlock: 1..{MMOE_MAX_TASKS} distinct outputs are supported, got {self.output_names}")
        self.num_experts = E
        self.temperature = float(gate_softmax_temperature)
        self.dropout = expert_block.dropout
        # expert_block.copy() per expert: fresh names, independently initialised variables
        self.expert_names = sorted(f"expert_{i}" for i in range(E))
        self.expert_blocks: Dict[str, MLP] = {n: expert_block.copy() for n in (f"expert_{i}" for i in range(E))}
        self.gate_finals: Dict[str, _Dense] = {n: _Dense(E, use_bias=False, name=unique_name("gate_final"))
                                               for n in self.output_names}
        # gate_block.copy() per output: each gate's layers are its own
        self.gate_blocks: Optional[Dict[str, MLP]] = (None if gate_block is None else
                                                      {n: gate_block.copy() for n in self.output_names})
        self.units = proto.units
        self.experts = _Dense(E * proto.units, activation=proto.activation, use_bias=proto.use_bias, name=f"{self.name}/experts")
        self.gates = (_Dense(len(self.output_names) * E, use_bias=False, name=f"{self.name}/gates")
                      if gate_block is None else None)

    def bind(self, names: Sequence[str]) -> None:
        """Put the gates in the order of the output block's outputs (the order the heads kernel reads them)."""
        if sorted(names) != sorted(self.output_names):
            raise ValueError(f"MMOEBlock outputs {sorted(self.output_names)} differ from the output block's {sorted(names)}")
        if self.experts.kernel is not None and list(names) != self.output_names:
            raise ValueError("MMOEBlock: the gates were built for another output order")
        self.output_names = list(names)

    @property
    def num_gates(self) -> int:
        return len(self.output_names)

    def build(self, width: Optional[int] = None, device=None):
        """The stacked layers from each expert's and gate's own initialiser, then those become views of them."""
        if self.experts.kernel is None:
            if width is None:
                raise ValueError(f"{self.name}: cannot build without the input width")
            layers = [self.expert_blocks[n].dense_layers[0] for n in self.expert_names]
            for l in layers:
                l.build(width, device)
            self.experts.build(width, device)
            self.experts.kernel.copy_(torch.cat([l.kernel for l in layers], dim=1))
            if self.experts.bias is not None:
                self.experts.bias.copy_(torch.cat([l.bias for l in layers]))
            for l in layers:  # the stacked kernel is the variable
                l.kernel = l.bias = None
            self.experts._weights_changed()
            gates = [self.gate_finals[n] for n in self.output_names]
            if self.gate_blocks is None:
                for g in gates:
                    g.build(width, device)
                self.gates.build(width, device)
                self.gates.kernel.copy_(torch.cat([g.kernel for g in gates], dim=1))
                for g in gates:
                    g.kernel = None
                self.gates._weights_changed()
            else:
                for n, g in zip(self.output_names, gates):
                    self.gate_blocks[n].build_from_width(width, device)
                    g.build(self.gate_blocks[n].dense_layers[-1].units, device)
        self.built = True
        return self

    def weights(self):
        """`expert_{i}/<layer>/{kernel,bias}` and `gate_<output>/gate_final/kernel`, views of the stacked layers."""
        out = {}
        if self.experts.kernel is None:
            return out
        U, E = self.units, self.num_experts
        for e, n in enumerate(self.expert_names):
            lname = self.expert_blocks[n].dense_layers[0].name
            out[f"{n}/{lname}/kernel"] = self.experts.kernel[:, e * U:(e + 1) * U]
            if self.experts.bias is not None:
                out[f"{n}/{lname}/bias"] = self.experts.bias[e * U:(e + 1) * U]
        for t, n in enumerate(self.output_names):
            if self.gate_blocks is None:
                out[f"gate_{n}/gate_final/kernel"] = self.gates.kernel[:, t * E:(t + 1) * E]
            else:
                out.update({f"gate_{n}/gate_block/{k}": v for k, v in self.gate_blocks[n].weights().items()})
                out[f"gate_{n}/gate_final/kernel"] = self.gate_finals[n].kernel
        return out

    def gate_chain(self, t: int) -> List[_Dense]:
        """The layers of gate t with a gate_block: its copy's Dense layers, then its gate_final."""
        n = self.output_names[t]
        return self.gate_blocks[n].dense_layers + [self.gate_finals[n]]

    def gate_logits(self, L: torch.Tensor) -> List[torch.Tensor]:
        """The (B, E) column block of each gate in stacked (B, H E) gate logits, in output order."""
        E = self.num_experts
        return [L[:, t * E:(t + 1) * E] for t in range(self.num_gates)]

    def call(self, inputs, **kwargs):
        raise NotImplementedError("MMOEBlock runs inside its Model (the mixture is fused with the output heads)")


def CGCBlock(*args, **kwargs):
    raise NotImplementedError("CGCBlock (progressive layered extraction) is not implemented")


def PLEBlock(*args, **kwargs):
    raise NotImplementedError("PLEBlock (progressive layered extraction) is not implemented")
