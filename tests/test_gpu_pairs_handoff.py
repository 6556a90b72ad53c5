"""The pairs-only hand-off between the fused DLRM lookup + interaction kernel and the top tower.

With operand-format rows the interaction kernel can write the pairs alone (MM_ROWS_OPERAND_PAIRS, rows of
2 * pairs_cols(F(F-1)/2) bf16), and the whole-tower kernel reads layer 1's k-block 0 from the bottom tower's own operand
rows (mm_mlp_tc_pairs).  The k-blocks, the MMAs and their order are those of the concatenated [bottom | pairs] row, so
every output must be byte-identical to the concatenated layout's: predictions, fp32 tower rows and multi-head outputs, at
batch sizes that end on, just before and just after a 64-row tile, and at the benchmark's 65 536.

The pairs buffer's last column and the rows of the bottom buffer past the batch hold NaN when the tower runs: the padding
of the last k-block must come from the TMA's zero fill, not from memory."""
import pytest
import torch

import models_b200 as mm
from models_b200 import blocks, datasets, ops
from models_b200.core import get_feature
from models_b200.graph import HostBatch
from tests import helpers as H
from tests.test_gpu_multitask import _batch, _mt_schema

pytestmark = pytest.mark.gpu
SIZES = [1, 127, 128, 129, 1001, 65536]


def _schema(targets=None):
    if targets:
        return _mt_schema(20000, targets)
    return datasets.criteo_schema({k: min(v, 20000) for k, v in datasets.CRITEO_MAX.items()})


def _model(schema, heads=False, seed=11):
    mm.set_seed(seed)
    kw = dict(prediction_tasks=mm.OutputBlock(schema)) if heads else {}
    return mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]),
                        top_block=mm.MLPBlock([128, 64, 32]), **kw)


def _inputs(schema, B, seed, device):
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=seed, index_law="uniform"))
    return H.device_batch(feats, device)


def _lookup(model, inputs, bottom, out, pairs_only):
    body = model.body
    emb, slots = body.embeddings, body.slots()
    feats = emb.feature_names
    tabs = [emb.feature_to_table[f].operand_mirror() for f in feats]
    ops.dlrm_lookup_interact(tabs, [ops.fused_ids(get_feature(inputs, f)) for f in feats], [slots[f] for f in feats],
                             [t.shape[0] for t in tabs], 64, bottom, slots["bottom_block"], out, operand_rows=True,
                             pairs_only=pairs_only)
    return out


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape)
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), f"{what}: not byte-identical"


def _rows_and_guarded_bottom(model, inputs, B, device):
    """(bottom rows inside a NaN-guarded buffer, the concatenated [bottom | pairs] rows, the NaN-padded pairs rows)."""
    body = model.body
    K = body.output_width_before_top()
    bottom = body.bottom_forward(inputs, operand_out=True)
    assert tuple(bottom.shape) == (B, 128)
    full = _lookup(model, inputs, bottom, torch.empty((B, 2 * ops.tc_padded_k(K)), dtype=torch.bfloat16, device=device), False)
    Kq = ops.pairs_cols(K - 64)
    pairs = _lookup(model, inputs, bottom, torch.full((B, 2 * Kq), float("nan"), dtype=torch.bfloat16, device=device), True)
    Kp, npairs = full.shape[1] // 2, K - 64
    # the pairs rows are the concatenated rows without the bottom columns and the padding
    assert torch.equal(_bits(pairs[:, :npairs]), _bits(full[:, 64:K]))
    assert torch.equal(_bits(pairs[:, Kq:Kq + npairs]), _bits(full[:, Kp + 64:Kp + K]))
    assert torch.equal(_bits(full[:, :64]), _bits(bottom[:, :64])) and torch.equal(_bits(full[:, Kp:Kp + 64]), _bits(bottom[:, 64:]))
    # columns past the pairs are never read by the tower: make them NaN, and the bottom rows past the batch too
    pairs[:, npairs:Kq] = float("nan")
    pairs[:, Kq + npairs:] = float("nan")
    guard = torch.full((B + 64, 128), float("nan"), dtype=torch.bfloat16, device=device)
    guard[:B] = bottom
    return guard[:B], full, pairs


def _tower_args(model):
    layers = model.body.top_block.dense_layers
    return ([l.split_kernel() for l in layers], [l.units for l in layers], [l.bias for l in layers],
            [l.activation for l in layers])


@pytest.mark.parametrize("B", SIZES)
def test_pairs_handoff_is_byte_identical(device, B):
    schema = _schema()
    model = _model(schema)
    inputs = _inputs(schema, B, 100 + B, device)
    model.build(device)
    K = model.body.output_width_before_top()
    bottom, full, pairs = _rows_and_guarded_bottom(model, inputs, B, device)
    ws, widths, bs, acts = _tower_args(model)
    head = model.prediction.to_call

    def run(**kw):  # the tower over the concatenated rows, then over bottom + pairs rows
        got = []
        for a, extra in ((full, {}), (pairs, dict(a_bottom=bottom))):
            o = {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in kw.items()}
            ops.mlp_tc(a, K, ws, widths, bs, acts, **o, **extra)
            got.append(o)
        return got

    old, new = run(head_w=head.kernel.reshape(-1), head_b=head.bias_value(), head_act="sigmoid",
                   head_out=torch.full((B, 1), float("nan"), device=device))
    _same(new["head_out"], old["head_out"], "predictions")
    old, new = run(out=torch.full((B, 32), float("nan"), device=device))
    _same(new["out"], old["out"], "fp32 top-tower rows")

    g = torch.Generator().manual_seed(B)
    hw = (torch.randn((32, 3), generator=g) * 0.3).to(device)
    hb = (torch.randn(3, generator=g) * 0.1).to(device)
    heads = []
    for a, kw in ((full, {}), (pairs, dict(a_bottom=bottom))):
        out = torch.full((3, B), float("nan"), device=device)
        ops.mlp_tc_heads(a, K, ws, widths, bs, acts, hw, hb, ["sigmoid", "linear", "sigmoid"], out, **kw)
        heads.append(out)
    _same(heads[1], heads[0], "multi-head outputs")

    # the model's forward takes the pairs hand-off and gives what the concatenated layout gives
    layers, _ = model.body.top_block.chain([head])
    want = blocks.run_dense_chain(None, layers, a_split=full, K=K)
    got = model(inputs)
    assert blocks.last_dense_path() == "mlp_tc"
    _same(got, want, "model predictions")


@pytest.mark.parametrize("B", [129, 65536])
def test_pairs_handoff_multi_head_model(device, B):
    schema = _schema(("click", "conversion", "rating"))
    model = _model(schema, heads=True)
    feats, _ = _batch(schema, B, 7 + B)
    inputs = H.device_batch(feats, device)
    model.build(device)
    model(inputs)  # builds the heads
    K = model.body.output_width_before_top()
    body, heads = model.body, model.prediction
    bottom = body.bottom_forward(inputs, operand_out=True)
    full = body.interaction_forward(inputs, bottom, as_split=True, operand_rows=True)
    want = heads.split(blocks.run_dense_chain(None, body.top_block.dense_layers, a_split=full, K=K, heads=heads))
    got = model(inputs)
    got = got.outputs if isinstance(got, mm.Prediction) else got
    assert blocks.last_dense_path() == "mlp_tc"
    assert list(got) == list(want)
    for k in want:
        _same(got[k], want[k], f"output {k}")


def test_pairs_handoff_in_captured_graphs(device):
    """The compiled forward and the pipelined forward replay the pairs hand-off: same predictions as the eager call."""
    B = 1001
    schema = _schema()
    model = _model(schema)
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, B, seed=5, index_law="uniform"))
    hb = HostBatch.like(feats, model.input_columns(), id_bytes=model.id_bytes())
    want = model(H.device_batch(feats, device))
    cf = model.compile(hb)
    _same(cf(hb).to(device), want, "compiled forward")
    pf = model.pipeline(hb, depth=2)
    t = pf.submit(hb)
    _same(pf.result(t).to(device), want, "pipelined forward")


def test_pairs_handoff_empty_batch(device):
    schema = _schema()
    model = _model(schema)
    model.build(device)
    K = model.body.output_width_before_top()
    ws, widths, bs, acts = _tower_args(model)
    head = model.prediction.to_call
    bottom = torch.empty((0, 128), dtype=torch.bfloat16, device=device)
    pairs = torch.empty((0, 2 * ops.pairs_cols(K - 64)), dtype=torch.bfloat16, device=device)
    out = torch.empty((0, 1), device=device)
    ops.mlp_tc(pairs, K, ws, widths, bs, acts, head_w=head.kernel.reshape(-1), head_b=0.0, head_act="sigmoid", head_out=out,
               a_bottom=bottom)
    torch.cuda.synchronize()
