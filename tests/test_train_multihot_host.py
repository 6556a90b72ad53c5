"""Host-side checks of the multi-hot training restatement (tests/multihot_oracle.py) on hand-made bags."""
from pathlib import Path

import numpy as np
import torch

from oracle import oracle_train
from tests import multihot_oracle as MO

TABLE = np.arange(24, dtype=np.float64).reshape(6, 4) + 1.0  # row r = [4r+1 .. 4r+4]


def _pool(batch, comb):
    return MO.pool(batch, "f", torch.tensor(TABLE), comb).numpy()


def test_ragged_bags_prune_negative_ids_and_empty_bags_give_zeros():
    batch = {"f__values": np.array([1, -1, 3, -5, 2, 2, 2, 9]), "f__offsets": np.array([0, 3, 3, 4, 8])}
    # bag 0: ids 1, 3 (the -1 is pruned); bag 1: empty; bag 2: only a pruned id; bag 3: 2, 2, 2 and 9 (>= rows: no row)
    s = _pool(batch, "sum")
    np.testing.assert_array_equal(s[0], TABLE[1] + TABLE[3])
    np.testing.assert_array_equal(s[1], 0.0)
    np.testing.assert_array_equal(s[2], 0.0)
    np.testing.assert_array_equal(s[3], 3 * TABLE[2])
    m = _pool(batch, "mean")
    np.testing.assert_allclose(m[0], (TABLE[1] + TABLE[3]) / 2)
    np.testing.assert_allclose(m[3], TABLE[2])
    np.testing.assert_array_equal(m[1], 0.0)
    q = _pool(batch, "sqrtn")
    np.testing.assert_allclose(q[0], (TABLE[1] + TABLE[3]) / np.sqrt(2))
    np.testing.assert_allclose(q[3], 3 * TABLE[2] / np.sqrt(3))


def test_fixed_length_bags_do_not_mask_padding():
    batch = {"f": np.array([[1, 0, 0], [5, 4, 3]])}  # id 0 is an ordinary row: padding is not masked
    np.testing.assert_allclose(_pool(batch, "mean")[0], (TABLE[1] + 2 * TABLE[0]) / 3)
    np.testing.assert_allclose(_pool(batch, "sum")[1], TABLE[5] + TABLE[4] + TABLE[3])
    batch = {"f": np.array([[1, 7], [2, 2]])}  # an id outside [0, rows) reads a zero row and still counts in L
    np.testing.assert_allclose(_pool(batch, "mean")[0], TABLE[1] / 2)


def _dlrm(batch, combiners, rng):
    tables = {"a": rng.standard_normal((7, 4)), "b": rng.standard_normal((5, 4))}
    bottom = [{"kernel": rng.standard_normal((2, 4)), "bias": rng.standard_normal(4), "activation": "relu"}]
    top = [{"kernel": rng.standard_normal((4 + 3, 3)), "bias": rng.standard_normal(3), "activation": "relu"}]
    head = {"kernel": rng.standard_normal((3, 1)), "bias": rng.standard_normal(1)}
    return tables, bottom, top, head


def test_one_hot_features_reproduce_the_one_hot_oracle():
    rng = np.random.default_rng(0)
    B = 9
    batch = {"a": rng.integers(0, 7, B), "b": rng.integers(0, 5, B), "I1": rng.random(B), "I2": rng.random(B)}
    tables, bottom, top, head = _dlrm(batch, {}, rng)
    y = (rng.random(B) < 0.5).astype(np.float64)
    f2t = {"a": "a", "b": "b"}
    want = oracle_train.dlrm_loss_and_grads(batch, tables, f2t, ["I1", "I2"], bottom, top, head, y)
    got = MO.dlrm_loss_and_grads(batch, tables, f2t, {}, ["I1", "I2"], bottom, top, head, y)
    assert got[0] == want[0]
    np.testing.assert_array_equal(got[1], want[1])
    for k in want[2]:
        np.testing.assert_array_equal(got[2][k], want[2][k])


def test_bag_gradient_is_the_scaled_pooled_gradient():
    """d loss / d table row r = sum over the bag positions holding r of scale(bag) * d loss / d pooled[bag]."""
    rng = np.random.default_rng(1)
    B = 4
    batch = {"a__values": np.array([0, 2, 2, -1, 6, 1]), "a__offsets": np.array([0, 3, 3, 5, 6]), "b": np.array([[0, 1], [1, 1], [4, 0], [2, 3]]),
             "I1": rng.random(B), "I2": rng.random(B)}
    tables, bottom, top, head = _dlrm(batch, {}, rng)
    y = np.array([1.0, 0.0, 1.0, 0.0])
    f2t = {"a": "a", "b": "b"}
    for comb in ("mean", "sum", "sqrtn"):
        _, _, g = MO.dlrm_loss_and_grads(batch, tables, f2t, {"a": comb, "b": "mean"}, ["I1", "I2"], bottom, top, head, y)
        # bag 2 = ids (-1 pruned, 6): one id kept, so every combiner gives it scale 1; bag 0 = ids 0, 2, 2
        eps = 1e-6
        t2 = {k: v.copy() for k, v in tables.items()}
        t2["a"][6, 1] += eps
        lp = MO.dlrm_loss_and_grads(batch, t2, f2t, {"a": comb, "b": "mean"}, ["I1", "I2"], bottom, top, head, y)[0]
        l0 = MO.dlrm_loss_and_grads(batch, tables, f2t, {"a": comb, "b": "mean"}, ["I1", "I2"], bottom, top, head, y)[0]
        np.testing.assert_allclose((lp - l0) / eps, g["table/a"][6, 1], rtol=1e-4, atol=1e-9)
        assert np.all(g["table/a"][[3, 4, 5]] == 0.0)  # rows no bag holds


GOLDEN = Path(__file__).parent / "golden" / "multihot" / "ref_torch_dlrm_train_multihot.npz"


def test_restatement_matches_the_reference_torch_backend():
    """Loss, outputs and every gradient of one BCE step of the reference's torch DLRMModel on one-hot columns plus a
    ragged column (its default bag combiner, empty bags included; tests/golden/make_golden_multihot.py) against the
    restatement, at 2e-4."""
    from tests.golden import replay

    z = replay.load(GOLDEN)
    cat = [str(n) for n in z["cat_names"]]
    batch = {k[len("batch_"):]: z[k] for k in z if k.startswith("batch_")}
    tables = {n: z[f"table_{n}"] for n in cat}
    comb = {str(n): str(z["combiner"]) for n in z["list_names"]}
    loss, logits, grads = MO.dlrm_loss_and_grads(batch, tables, {n: n for n in cat}, comb, [str(n) for n in z["cont_names"]],
                                                 replay.unpack_layers(z, "bottom"), replay.unpack_layers(z, "top"),
                                                 replay.unpack_layers(z, "head")[0], z["targets"])
    np.testing.assert_allclose(1.0 / (1.0 + np.exp(-logits)), z["out"].reshape(-1), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(loss, float(z["loss"]), rtol=1e-5)
    for name, want in replay.train_grad_items(z):
        np.testing.assert_allclose(grads[name], want, rtol=2e-4, atol=1e-7, err_msg=name)
    assert np.any(z["batch_genres__offsets"][1:] == z["batch_genres__offsets"][:-1])  # the fixture has empty bags
    assert np.abs(z["grad_table_genres"]).max() > 0
