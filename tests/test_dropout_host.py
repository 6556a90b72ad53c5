"""Training-mode dropout of the weight-tied next-item step without a GPU: the numpy Philox4x32-10 port against the
generator's published known-answer vectors, the mask's threshold, the placement of dropout in an MLPBlock with
no_activation_last_layer on and off, and the refusals that stay: MLP.__call__(training=True) and every other trainer."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets
from tests.dropout_mask import keep_mask, philox4x32_10, threshold


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10(*ctr, *key)
    assert tuple(int(w) for w in got) == want


def test_mask_threshold_and_keep_fraction():
    assert threshold(0.0) == 0 and threshold(0.5) == 2**31 and threshold(0.999999999999) == 2**32 - 1
    assert keep_mask(16, 8, 0.0, 7, 0, 0).all()
    m = keep_mask(1000, 200, 0.2, 7, 3, 1)
    assert abs(m.mean() - 0.8) < 5 * np.sqrt(0.16 / m.size)
    # every coordinate of the counter and the key changes the mask
    for other in (keep_mask(1000, 200, 0.2, 7, 4, 1), keep_mask(1000, 200, 0.2, 7, 3, 2), keep_mask(1000, 200, 0.2, 8, 3, 1),
                  keep_mask(1000, 200, 0.2, 7 + (1 << 32), 3, 1)):
        assert 0.25 < (other != m).mean() < 0.4  # independent masks differ in 2 p (1 - p) = 32 % of the elements


def test_dropout_placement():
    """blocks/mlp.py:97-131: a Dropout after every Dense, except the last one when no_activation_last_layer."""
    assert mm.MLPBlock([128, 64], dropout=0.2).dropout_rates() == [0.2, 0.2]
    assert mm.MLPBlock([128, 64], no_activation_last_layer=True, dropout=0.2).dropout_rates() == [0.2, 0.0]
    assert mm.MLPBlock([128, 64, 32], no_activation_last_layer=True, dropout=0.1).dropout_rates() == [0.1, 0.1, 0.0]
    assert mm.MLPBlock([128, 64], no_activation_last_layer=True).dropout_rates() == [0.0, 0.0]


def test_mlp_call_in_training_mode_still_refuses_dropout():
    mlp = mm.MLPBlock([8], dropout=0.2)
    with pytest.raises(NotImplementedError, match="dropout in training mode is outside the forward hot path"):
        mlp(torch.zeros(2, 4), training=True)


def test_other_trainers_still_refuse_dropout():
    schema = datasets.criteo_schema({k: min(v, 1000) for k, v in datasets.CRITEO_MAX.items()})
    model = mm.DLRMModel(schema, embedding_dim=16, bottom_block=mm.MLPBlock([32, 16], dropout=0.2),
                         top_block=mm.MLPBlock([32, 16]))
    model.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="supports MLPBlocks without normalization / dropout"):
        mm.train.DLRMTrainer(model, model.optimizer, 8, device="cpu")
