"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol the
header declares, constructors mirror the reference's argument checks and messages, and nothing
computes without a GPU (no CPU fallback)."""
import ctypes
import re

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, datasets


def test_library_exports_every_declared_symbol():
    lib = _cabi.load()
    declared = _cabi.declared_symbols()
    assert len(declared) >= 14
    assert set(declared) == set(_cabi.SIGNATURES), "binding table and include/mm_b200.h disagree"
    for name in declared:
        assert hasattr(lib, name), f"libmm_b200.so does not export {name}"
    assert lib.mm_version() >= 100
    assert lib.mm_launch_count() == 0 or lib.mm_launch_count() > 0


def test_struct_layouts_match_header():
    assert ctypes.sizeof(_cabi.GatherTable) == 32
    assert ctypes.sizeof(_cabi.ConcatPiece) == 32
    assert ctypes.sizeof(_cabi.LookupTable) == 40
    assert ctypes.sizeof(_cabi.SparseTable) == 80


def test_argument_errors_are_reported_without_a_gpu():
    lib = _cabi.load()
    rc = lib.mm_gather_multi(None, 0, 0, 10, None, 64, None, None)
    assert rc == -1 and b"n_tables" in lib.mm_last_error()
    rc = lib.mm_dense_fp32(None, 1, 1, 1, None, None, 1, 0, None, 0, None, 1, None)
    assert rc == -1
    with pytest.raises(ValueError, match="mm_dense_fp32"):
        _cabi.check(rc, "mm_dense_fp32")


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_calling_a_model_without_cuda_fails_loudly():
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([16]))
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        model({k: torch.from_numpy(v) for k, v in feats.items()})


def test_product_does_not_import_the_oracle():
    import pathlib

    for p in pathlib.Path(mm.__file__).parent.rglob("*.py"):
        text = p.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle", text, flags=re.M), f"{p} imports the oracle"


# --- constructor errors: tests/unit/tf/blocks/test_dlrm.py:63-112 ---------------------------------
def test_dlrm_constructor_errors():
    schema = datasets.criteo_schema()
    with pytest.raises(ValueError, match="The schema is required by DLRM"):
        mm.DLRMBlock(None, embedding_dim=8)
    with pytest.raises(ValueError, match="DLRM requires categorical features"):
        mm.DLRMBlock(schema.select_by_tag(mm.Tags.CONTINUOUS), embedding_dim=8, bottom_block=mm.MLPBlock([8]))
    with pytest.raises(ValueError, match="The bottom_block is required by DLRM"):
        mm.DLRMBlock(schema, embedding_dim=8)
    with pytest.raises(ValueError, match="needs to match the last layer of bottom MLP"):
        mm.DLRMBlock(schema, embedding_dim=8, bottom_block=mm.MLPBlock([16, 4]))
    with pytest.raises(ValueError, match="Only one-of `embeddings` or `embedding_options` may be provided"):
        mm.DLRMBlock(schema, embeddings=mm.Embeddings(schema.select_by_tag(mm.Tags.CATEGORICAL), dim=8),
                     embedding_options=mm.EmbeddingOptions(), bottom_block=mm.MLPBlock([8]))
    with pytest.raises(ValueError, match="The embedding_dim is required"):
        mm.DLRMBlock(schema, bottom_block=mm.MLPBlock([8]))


def test_two_tower_constructor_errors():
    """tests/unit/tf/blocks/retrieval/test_two_tower.py:184-207."""
    schema = datasets.movielens_1m_schema()
    with pytest.raises(ValueError, match="The schema is required by TwoTower"):
        mm.TwoTowerBlock(None, query_tower=mm.MLPBlock([8]))
    with pytest.raises(ValueError, match="The query_tower is required by TwoTower"):
        mm.TwoTowerBlock(schema, query_tower=None)
    no_items = schema.excluding_by_tag(mm.Tags.ITEM)
    with pytest.raises(ValueError, match="required by item-tower"):
        mm.TwoTowerBlock(no_items, query_tower=mm.MLPBlock([8]))


def test_mlp_and_cross_constructor_errors():
    with pytest.raises(ValueError, match="Activation and Dimensions length mismatch"):
        mm.MLPBlock([8, 4], activation=["relu"])
    with pytest.raises(ValueError, match="Number of cross layers"):
        mm.CrossBlock(0)
    with pytest.raises(ValueError, match="Unknown interaction type"):
        mm.DotProductInteraction(interaction_type="nope")
    mlp = mm.MLPBlock([32, 16], activation=["relu", "tanh"], no_activation_last_layer=True)
    assert [l.activation for l in mlp.dense_layers] == ["relu", "linear"]
    assert [l.units for l in mlp.dense_layers] == [32, 16]


def test_model_plans_follow_the_reference_ordering_rules():
    schema = datasets.criteo_schema()
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]),
                         top_block=mm.MLPBlock([128, 64, 32]))
    slots = model.body.slots()
    order = sorted(slots, key=slots.get)
    # StackFeatures iterates sorted(names): 'C1','C10',...,'C9', then 'bottom_block' ('C' < 'b')
    assert order[:4] == ["C1", "C10", "C11", "C12"] and order[-2:] == ["C9", "bottom_block"]
    assert model.body.output_width_before_top() == 64 + 351
    # embedding tables: rows = int_domain.max + 1
    assert model.body.embeddings.tables["C1"].input_dim == 10_000_000
    assert sum(t.input_dim for t in model.body.embeddings.tables.values()) == 45_621_194
    # inferred dims (utils/schema_utils.py:169-207)
    assert mm.infer_embedding_dim(schema["C1"]) == 120 and mm.infer_embedding_dim(schema["C6"]) == 8
    assert model.input_columns()[0] == "C21" and len(model.input_columns()) == 39


def test_integration_doc_lists_every_exported_symbol():
    """INTEGRATION.md is the maintainer-facing table of the C ABI: it must mention every symbol of include/mm_b200.h."""
    from pathlib import Path

    from models_b200 import _cabi

    doc = (Path(__file__).resolve().parent.parent / "INTEGRATION.md").read_text()
    missing = [s for s in sorted(_cabi.declared_symbols()) if s not in doc]
    assert not missing, f"INTEGRATION.md does not mention: {missing}"


def test_model_file_unpickler_refuses_everything_but_package_classes(tmp_path):
    """ADVICE r1: model.pkl may only name classes defined in models_b200 (plus a few inert value types); builtins.eval,
    functools.partial, torch.load or a module re-exported by one of the package's modules must be refused."""
    import io as _io
    import pickle

    import torch

    from models_b200 import io as mmio

    def payload(mod, name):
        return pickle.PROTO + bytes([4]) + b"\x8c" + bytes([len(mod)]) + mod.encode() + b"\x8c" + bytes([len(name)]) + name.encode() + b"\x93."

    def load(mod, name):
        return mmio._TensorUnpickler(_io.BytesIO(payload(mod, name)), tmp_path, {"variables": []}, torch.device("cpu")).load()

    for mod, name in (("builtins", "eval"), ("builtins", "getattr"), ("builtins", "__import__"), ("functools", "partial"),
                      ("torch", "load"), ("numpy", "load"), ("os", "system"), ("models_b200.csrc.build", "subprocess"),
                      ("models_b200.csrc.build", "subprocess.run"), ("models_b200.io", "pickle")):
        with pytest.raises(pickle.UnpicklingError, match="refusing to load"):
            load(mod, name)
    import models_b200 as mm

    assert load("models_b200.schema", "Schema") is mm.Schema
    assert load("collections", "OrderedDict").__name__ == "OrderedDict"
