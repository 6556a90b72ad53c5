"""CPU checks of the DCN-v2 training restatement (tests/dcn_train_oracle.py) against the reference's torch DCNModel step
(tests/golden/dcn_train/ref_torch_dcn_train.npz, written by tests/golden/make_golden_dcn_train.py)."""
from pathlib import Path

import numpy as np
import pytest

from models_b200.inputs import infer_embedding_dim
from models_b200.schema import ColumnSchema
from tests.dcn_train_oracle import dcn_loss_and_grads, golden_inputs

FIXTURE = Path(__file__).parent / "golden" / "dcn_train" / "ref_torch_dcn_train.npz"


def _close(a, b, tol=2e-4):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    scale = max(1.0, float(np.abs(b).max()) if b.size else 1.0)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.abs(a - b).max() <= tol * scale, float(np.abs(a - b).max())


@pytest.mark.parametrize("tag", ["stacked", "parallel"])
def test_restatement_matches_reference_step(tag):
    z = np.load(FIXTURE)
    batch, tables, conts, cross, deep, heads, ys, order, _ = golden_inputs(z, tag)
    loss, _, logits, grads = dcn_loss_and_grads(batch, tables, conts, cross, deep, heads, ys, stacked=tag == "stacked", order=order)
    assert abs(loss - float(z[f"{tag}_loss"])) <= 2e-4 * max(1.0, abs(loss))
    p = 1.0 / (1.0 + np.exp(-logits[0]))
    _close(p, z[f"{tag}_out"].reshape(-1))
    for f in tables:
        _close(grads[f"table/{f}"], z[f"{tag}_grad_table_{f}_rows"])
    for grp, ls in (("cross", cross), ("deep", deep)):
        for i in range(len(ls)):
            _close(grads[f"{grp}/kernel_{i}"], z[f"{tag}_grad_{grp}_kernel_{i}"])
            _close(grads[f"{grp}/bias_{i}"], z[f"{tag}_grad_{grp}_bias_{i}"])
    _close(grads["head/click/binary_output/kernel"], z[f"{tag}_grad_head_kernel_0"])
    _close(grads["head/click/binary_output/bias"], z[f"{tag}_grad_head_bias_0"])


def test_fixture_widths_and_unaligned_offsets():
    """The fixture exercises widths the sparse update formerly rejected, at column offsets that are not multiples of 4."""
    z = np.load(FIXTURE)
    cat = [str(n) for n in z["cat_names"]]
    widths = {f: z[f"stacked_table_{f}_rows"].shape[1] for f in cat}
    for f, mx in zip(cat, z["cat_max"]):
        col = ColumnSchema(f, tags=("categorical",), dtype="int64", properties={"domain": {"min": 0, "max": int(mx), "name": f}})
        assert infer_embedding_dim(col) == widths[f]
    assert {24, 48} <= set(widths.values())
    names = sorted(cat + [str(n) for n in z["cont_names"]])
    off, offsets = 0, {}
    for n in names:
        offsets[n] = off
        off += widths.get(n, 1)
    assert any(offsets[f] % 4 for f in cat)
