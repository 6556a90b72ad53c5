"""Weights and metadata at the reference's checkpoint boundary.

The reference saves a Keras SavedModel plus `.merlin/{input,output}_schema.json`
(merlin/models/tf/models/base.py:1687-1728, merlin/models/io.py:26-55) and moves embedding tables in and
out as (rows, dim) matrices (`EmbeddingTable.from_pretrained` / `to_df`, inputs/embedding.py:283-379).
TensorFlow is not a dependency here, so the on-disk form is:

    export_path/
      .merlin/input_schema.json, .merlin/output_schema.json   tensorflow-metadata JSON, as the reference
      variables/manifest.json     ordered [{name, file, shape, dtype}], Keras layouts:
                                  embeddings (int_domain.max + 1, dim) fp32, Dense kernel (in, out), bias (out,)
      variables/NNNN.npy          one array per variable (np.load(..., mmap_mode="r") friendly)
      model.pkl                   the block structure (Python objects of THIS package, tensors replaced by
                                  references into variables/) — the analogue of SavedModel's custom objects

`Model.load_weights` also accepts a plain {name: array} mapping, which is how a Keras checkpoint exported
with `{v.name: v.numpy() for v in keras_model.variables}` (plus a name map) is served by the H100 path.
"""
from __future__ import annotations

import io as _io
import json
import os
import pathlib
import pickle
from typing import Callable, Dict, Mapping, Optional, Union

import numpy as np
import torch

from .core import Block, default_device
from .schema import Schema

_MERLIN_METADATA_DIR_NAME = ".merlin"
_VARIABLES_DIR_NAME = "variables"
FORMAT_VERSION = 1


def save_merlin_metadata(export_path, input_schema: Optional[Schema], output_schema: Optional[Schema]) -> None:
    """merlin/models/io.py:26-55: schemas as tensorflow-metadata JSON under `<export_path>/.merlin/`."""
    d = pathlib.Path(export_path) / _MERLIN_METADATA_DIR_NAME
    d.mkdir(parents=True, exist_ok=True)
    if input_schema is not None:
        input_schema.to_json(d / "input_schema.json")
    if output_schema is not None:
        output_schema.to_json(d / "output_schema.json")


def load_merlin_metadata(export_path):
    d = pathlib.Path(export_path) / _MERLIN_METADATA_DIR_NAME
    inp = Schema.load(str(d / "input_schema.json")) if (d / "input_schema.json").exists() else None
    out = Schema.load(str(d / "output_schema.json")) if (d / "output_schema.json").exists() else None
    return inp, out


# ------------------------------------------------------------------------------------------------
# name -> array views of a model
# ------------------------------------------------------------------------------------------------
def state_dict(model: Block) -> Dict[str, np.ndarray]:
    """Keras-style variable names -> host fp32 arrays (copies)."""
    return {k: v.detach().cpu().numpy() for k, v in model.weights().items()}


def _notify_weights_changed(obj, seen=None, depth=0) -> None:
    seen = seen if seen is not None else set()
    if id(obj) in seen or depth > 8:
        return
    seen.add(id(obj))
    if isinstance(obj, Block):
        hook = getattr(obj, "_weights_changed", None)
        if hook is not None:
            hook()
        for v in vars(obj).values():
            _notify_weights_changed(v, seen, depth + 1)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _notify_weights_changed(v, seen, depth + 1)
    elif isinstance(obj, dict):
        for v in obj.values():
            _notify_weights_changed(v, seen, depth + 1)


def load_weights(model: Block, source: Union[str, os.PathLike, Mapping[str, np.ndarray]],
                 name_map: Optional[Union[Mapping[str, str], Callable[[str], str]]] = None, strict: bool = True) -> Dict[str, str]:
    """Copy arrays into the model's (already built) variables.

    source: an export directory written by `save_model`, or a {name: array} mapping (e.g. exported from a
    Keras checkpoint).  name_map translates THIS model's variable names to the source's names (dict or
    callable).  strict: every model variable must be found and every shape must match; otherwise missing
    ones are skipped.  Returns {model variable: source name} for what was loaded."""
    if not isinstance(source, Mapping):
        source = _LazyVariables(pathlib.Path(source))
    targets = model.weights()
    if not targets:
        raise ValueError("the model has no variables yet: call model.build(device) (or run one batch) before load_weights")
    loaded = {}
    for name, t in targets.items():
        src_name = name_map(name) if callable(name_map) else (name_map or {}).get(name, name)
        if src_name not in source:
            if strict:
                raise KeyError(f"variable {name!r} (looked up as {src_name!r}) not found in the checkpoint")
            continue
        arr = np.asarray(source[src_name])
        if tuple(arr.shape) != tuple(t.shape):
            raise ValueError(f"variable {name!r}: checkpoint shape {tuple(arr.shape)} != model shape {tuple(t.shape)}")
        t.copy_(torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float32)).to(t.device, non_blocking=False))
        loaded[name] = src_name
    _notify_weights_changed(model)
    from .core import bump_weights_version

    bump_weights_version()  # captured graphs (graph.CompiledForward) re-capture before their next replay
    return loaded


class _LazyVariables(Mapping):
    """{name: array} over an export directory; arrays are memory-mapped, one at a time."""

    def __init__(self, path: pathlib.Path):
        self.dir = path / _VARIABLES_DIR_NAME
        with open(self.dir / "manifest.json") as f:
            self.manifest = json.load(f)
        self.by_name = {e["name"]: e for e in self.manifest["variables"] if e.get("name")}

    def __getitem__(self, name):
        return np.load(self.dir / self.by_name[name]["file"], mmap_mode="r")

    def __iter__(self):
        return iter(self.by_name)

    def __len__(self):
        return len(self.by_name)


# ------------------------------------------------------------------------------------------------
# whole-model save / load
# ------------------------------------------------------------------------------------------------
class _TensorPickler(pickle.Pickler):
    """Pickles the block structure; every torch.Tensor becomes a reference to variables/NNNN.npy."""

    def __init__(self, file, var_dir: pathlib.Path, names: Dict[int, str]):
        super().__init__(file, protocol=pickle.HIGHEST_PROTOCOL)
        self.var_dir, self.names = var_dir, names
        self.entries, self.index_of = [], {}

    def persistent_id(self, obj):
        if not isinstance(obj, torch.Tensor):
            return None
        key = (obj.data_ptr(), tuple(obj.shape), tuple(obj.stride()), str(obj.dtype))
        if key not in self.index_of:
            idx = len(self.entries)
            fname = f"{idx:04d}.npy"
            host = obj.detach().cpu()
            arr = host.view(torch.int16).numpy() if host.dtype == torch.bfloat16 else host.numpy()
            np.save(self.var_dir / fname, arr)
            self.entries.append({"name": self.names.get(obj.data_ptr()), "file": fname, "shape": list(obj.shape),
                                 "dtype": str(obj.dtype).replace("torch.", ""), "device": obj.device.type})
            self.index_of[key] = idx
        return ("mm_b200_tensor", self.index_of[key])


class _TensorUnpickler(pickle.Unpickler):
    def __init__(self, file, var_dir: pathlib.Path, manifest, device):
        super().__init__(file)
        self.var_dir, self.manifest, self.device = var_dir, manifest, device
        self.cache = {}

    def persistent_load(self, pid):
        tag, idx = pid
        if tag != "mm_b200_tensor":
            raise pickle.UnpicklingError(f"unknown persistent id {tag!r}")
        if idx not in self.cache:
            e = self.manifest["variables"][idx]
            arr = np.load(self.var_dir / e["file"])
            t = torch.from_numpy(arr)
            if e["dtype"] == "bfloat16":
                t = t.view(torch.bfloat16)
            self.cache[idx] = t.to(self.device) if e.get("device") == "cuda" else t
        return self.cache[idx]

    # value types a structure file may legitimately name besides this package's own classes
    _ALLOWED = {("collections", "OrderedDict"), ("builtins", "set"), ("builtins", "frozenset"), ("builtins", "slice"),
                ("builtins", "range"), ("builtins", "complex"), ("builtins", "bytearray")}

    def find_class(self, module, name):
        """Exact allowlist: classes DEFINED in this package (types whose __module__ is models_b200.*, looked up by a
        plain, undotted name) plus a few inert value types.  Anything else — builtins.eval / getattr / __import__,
        functools.partial, torch.load, numpy.load, or a module object re-exported by one of this package's modules
        (`models_b200.csrc.build.subprocess`) — is refused, so loading an untrusted export cannot run code."""
        if (module, name) in self._ALLOWED:
            return super().find_class(module, name)
        if (module == "models_b200" or module.startswith("models_b200.")) and "." not in name:
            obj = super().find_class(module, name)
            if isinstance(obj, type) and (obj.__module__ == "models_b200" or obj.__module__.startswith("models_b200.")):
                return obj
        raise pickle.UnpicklingError(f"refusing to load {module}.{name} from a model file")


def save_model(model: Block, export_path) -> None:
    """`model.save(export_path)` of the reference (models/base.py:1687-1716): variables + structure + `.merlin` metadata."""
    path = pathlib.Path(export_path)
    var_dir = path / _VARIABLES_DIR_NAME
    var_dir.mkdir(parents=True, exist_ok=True)
    weights = model.weights()
    if not weights:
        raise ValueError("the model has no variables yet: call model.build(device) (or run one batch) before save")
    names = {t.data_ptr(): n for n, t in weights.items()}
    buf = _io.BytesIO()
    pk = _TensorPickler(buf, var_dir, names)
    pk.dump(model)
    with open(path / "model.pkl", "wb") as f:
        f.write(buf.getvalue())
    with open(var_dir / "manifest.json", "w") as f:
        json.dump({"format_version": FORMAT_VERSION, "variables": pk.entries}, f, indent=1)
    schema = getattr(model, "schema", None)
    out_schema = model.output_schema() if hasattr(model, "output_schema") else None
    save_merlin_metadata(path, schema, out_schema)


def load_model(export_path, device=None) -> Block:
    """`Model.load(export_path)` (models/base.py:1718-1728)."""
    path = pathlib.Path(export_path)
    var_dir = path / _VARIABLES_DIR_NAME
    with open(var_dir / "manifest.json") as f:
        manifest = json.load(f)
    if manifest.get("format_version") != FORMAT_VERSION:
        raise ValueError(f"unsupported model format version {manifest.get('format_version')!r}")
    device = device or default_device()
    with open(path / "model.pkl", "rb") as f:
        return _TensorUnpickler(f, var_dir, manifest, device).load()
