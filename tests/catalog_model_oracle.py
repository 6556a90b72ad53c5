"""Float64 restatement of one training step of Model(InputBlockV2, MLPBlock, CategoricalOutput(to_call=EmbeddingTable)):
the sorted-name concat of the embedding rows (one-hot rows, or the mean / sum of a fixed-length list's rows) and the
continuous columns, the MLP, z = (x E^T + b) / T and Keras CategoricalCrossentropy(from_logits=True) with per-row weights
c = sample_weight / B.  Torch autograd (CPU, float64) gives every gradient; the tied table's is the sum of its input-side
lookups and its output-side product, as TensorFlow sums both paths of one variable.  Also the schema and model builders the
host and GPU tests share, and the Keras dense update rules."""
from pathlib import Path

import numpy as np
import torch

import models_b200 as mm
from models_b200.schema import ColumnSchema, Schema, Tags

N_USERS = 50


def schema(n_items: int, tied: str, L: int = 4, n_users: int = N_USERS) -> Schema:
    """user_id (one-hot), the item feature (tied = "onehot": last_item; "list": a fixed-length (B, L) item_history;
    "none": no item feature), two continuous columns and the next_item target."""
    cols = [ColumnSchema("user_id", tags=(Tags.CATEGORICAL, Tags.USER_ID), dtype="int64",
                         properties={"domain": {"min": 0, "max": n_users - 1, "name": "user_id"}})]
    item_dom = {"domain": {"min": 0, "max": n_items - 1, "name": "item_id"}}
    if tied == "onehot":
        cols.append(ColumnSchema("last_item", tags=(Tags.CATEGORICAL, Tags.ITEM_ID), dtype="int64", properties=item_dom))
    elif tied == "list":
        cols.append(ColumnSchema("item_history", tags=(Tags.CATEGORICAL,), dtype="int64", is_list=True, is_ragged=False,
                                 properties={**item_dom, "value_count": {"min": L, "max": L}}))
    cols += [ColumnSchema(n, tags=(Tags.CONTINUOUS,), dtype="float32") for n in ("c1", "c2")]
    cols.append(ColumnSchema("next_item", tags=(Tags.TARGET,), dtype="int64"))
    return Schema(cols)


def build(n_items: int, D: int, tied: str, widths=(32,), T: float = 1.0, use_bias: bool = True, combiner: str = "mean",
          seed: int = 7, L: int = 4, n_users: int = N_USERS):
    """(model, schema, item table) of the tied case `tied`."""
    mm.set_seed(seed)
    s = schema(n_items, tied, L, n_users)
    emb = mm.Embeddings(s.select_by_tag(Tags.CATEGORICAL), dim=D, sequence_combiner=combiner)
    ib = mm.InputBlockV2(s, categorical=emb)
    if tied == "none":
        table = mm.EmbeddingTable(D, ColumnSchema("item", tags=(Tags.CATEGORICAL,), dtype="int64",
                                                  properties={"domain": {"min": 0, "max": n_items - 1, "name": "item_id"}}))
    else:
        table = emb.tables["item_id"]
    out = mm.CategoricalOutput(to_call=table, logits_temperature=T, use_bias=use_bias, target_name="next_item")
    model = mm.Model(ib, mm.MLPBlock(list(widths) + [D]), out)
    return model, s, table


def batch(s: Schema, n_items: int, B: int, seed: int = 0, L: int = 4, hot: int = 0):
    """Host features and labels; ids repeat within the batch (hot > 0: the first `hot` items take half the draws)."""
    rng = np.random.default_rng(seed)

    def items(shape):
        v = rng.integers(0, n_items, shape)
        if hot:
            m = rng.random(shape) < 0.5
            v[m] = rng.integers(0, hot, int(m.sum()))
        return v.astype(np.int64)

    f = {"user_id": rng.integers(0, s.get("user_id").int_domain.max + 1, B).astype(np.int64),
         "c1": rng.standard_normal(B).astype(np.float32), "c2": rng.standard_normal(B).astype(np.float32)}
    if "last_item" in s.column_names:
        f["last_item"] = items(B)
    if "item_history" in s.column_names:
        f["item_history"] = items((B, L))
    return f, items(B)


def restated_query(model, feats) -> np.ndarray:
    """The MLP's output x (B, D) in float64."""
    with torch.no_grad():
        return _forward(model, feats, {})[0].numpy()


def _forward(model, feats, leaves):
    """x (B, D) and the input block's width, with every variable a float64 leaf in `leaves` (by restated_step's names)."""
    ib = model.body.input_block
    cols, widths, d = ib.layout()

    def leaf(name, t):
        if name not in leaves:
            leaves[name] = torch.tensor(t.detach().cpu().numpy().astype(np.float64), requires_grad=torch.is_grad_enabled())
        return leaves[name]

    B = len(next(iter(feats.values())))
    pieces = {}
    for f, tb in ib.embeddings.feature_to_table.items():
        E = leaf(f"tables/{tb.table_name}", tb.table)
        ids = torch.from_numpy(np.asarray(feats[f]).astype(np.int64))
        if ids.dim() == 1:
            pieces[f] = E[ids]
        else:
            rows = E[ids.reshape(-1)].reshape(ids.shape[0], ids.shape[1], -1)
            pieces[f] = rows.mean(1) if (tb.sequence_combiner or "mean") == "mean" else rows.sum(1)
    for n in ib.continuous.features:
        pieces[n] = torch.from_numpy(np.asarray(feats[n]).astype(np.float64)).reshape(B, 1)
    h = torch.cat([pieces[n] for n in sorted(pieces)], dim=1)
    assert h.shape[1] == d
    for i, l in enumerate(model.mlp.dense_layers):
        h = h @ leaf(f"mlp/{i}/kernel", l.kernel)
        if l.bias is not None:
            h = h + leaf(f"mlp/{i}/bias", l.bias)
        if l.activation == "relu":
            h = torch.relu(h)
    return h, leaf


def restated_step(model, feats, labels, sample_weight=None):
    """(loss, grads) in float64: grads by variable name, "tables/<table>" (dense, the tied table's both paths),
    "mlp/<i>/kernel" / "mlp/<i>/bias" and "bias"."""
    out = model.prediction
    T = out.logits_temperature
    leaves = {}
    B = len(labels)
    h, leaf = _forward(model, feats, leaves)
    E = leaf(f"tables/{out.table.table_name}", out.table.table)
    z = h @ E.T
    if out.bias is not None:
        z = z + leaf("bias", out.bias)
    z = z / T
    y = torch.from_numpy(np.asarray(labels).astype(np.int64))
    per = torch.nn.functional.cross_entropy(z, y, reduction="none")
    w = torch.ones(B, dtype=torch.float64) if sample_weight is None else torch.from_numpy(np.asarray(sample_weight, np.float64))
    loss = (per * w).sum() / B
    loss.backward()
    return float(loss.item()), {k: v.grad.numpy() for k, v in leaves.items()}


def restated_terms(model, feats, labels, sample_weight=None):
    """The magnitudes the kernels' rounding scales with, per element, in float64: x (B, D), |G| (B, N) with
    G = c (softmax(z) - onehot), and the output side's |G|^T |x| / T (N, D) and sum_b |G| / T (N,)."""
    out = model.prediction
    T = out.logits_temperature
    x = restated_query(model, feats)
    E = out.table.table.detach().cpu().double().numpy()
    z = x @ E.T
    if out.bias is not None:
        z = z + out.bias.detach().cpu().double().numpy()[None, :]
    z /= T
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    B = len(labels)
    c = (np.ones(B) if sample_weight is None else np.asarray(sample_weight, np.float64)) / B
    onehot = np.zeros_like(p)
    onehot[np.arange(B), np.asarray(labels)] = 1.0
    aG = np.abs(c[:, None] * (p - onehot))
    return x, aG, aG.T @ np.abs(x) / T, aG.sum(0) / T


def dense_update(kind: str, w, g, s1, s2, lr, t: int, beta_1=0.9, beta_2=0.999, eps=1e-7):
    """One Keras update of every element (SGD, Adagrad, Adam; LazyAdam on a dense gradient is Adam): (w, s1, s2) after
    step t (1-based), float64."""
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    if kind == "sgd":
        return w - lr * g, s1, s2
    if kind == "adagrad":
        s1 = s1 + g * g
        return w - lr * g / (np.sqrt(s1) + eps), s1, s2
    s1 = beta_1 * s1 + (1 - beta_1) * g
    s2 = beta_2 * s2 + (1 - beta_2) * g * g
    lr_t = lr * np.sqrt(1 - beta_2 ** t) / (1 - beta_1 ** t)
    return w - lr_t * s1 / (np.sqrt(s2) + eps), s1, s2


GOLDEN = Path(__file__).resolve().parent / "golden" / "catalog_train" / "ref_torch_catalog_train.npz"


def golden_model(device=None):
    """(model, feats, labels, sample_weight, golden) of tests/golden/make_golden_catalog_train.py: the same model built
    here (an item history tied to the output, T = 0.05, a bias) with the golden's weights; device None keeps the variables
    on the CPU (for the restatement)."""
    z = np.load(GOLDEN)
    model, s, table = build(int(z["n_items"]), int(z["dim"]), "list", widths=(24,), T=float(z["temperature"]),
                            L=int(z["hist_len"]))
    emb = model.body.input_block.embeddings
    vals = {"item_id": z["table_item_id"], "user_id": z["table_user_id"]}
    if device is None:
        for n, tb in emb.tables.items():
            tb.table = torch.from_numpy(vals[n].copy())
        for i, l in enumerate(model.mlp.dense_layers):
            l.kernel, l.bias = torch.from_numpy(z[f"mlp_kernel_{i}"].copy()), torch.from_numpy(z[f"mlp_bias_{i}"].copy())
        model.prediction.bias = torch.from_numpy(z["bias"].copy())
    else:
        model.build(device)
        for n, tb in emb.tables.items():
            tb.table.copy_(torch.from_numpy(vals[n]))
        for i, l in enumerate(model.mlp.dense_layers):
            l.kernel.copy_(torch.from_numpy(z[f"mlp_kernel_{i}"]))
            l.bias.copy_(torch.from_numpy(z[f"mlp_bias_{i}"]))
            l._weights_changed()
        model.prediction.bias.copy_(torch.from_numpy(z["bias"]))
        model.prediction.refresh()
    feats = {k[len("batch_"):]: z[k] for k in z.files if k.startswith("batch_")}
    return model, feats, z["labels"], z["sample_weight"], z


def golden_grads(z) -> dict:
    """The golden's gradients under restated_step's names."""
    out = {"tables/item_id": z["grad_table_item_id"], "tables/user_id": z["grad_table_user_id"], "bias": z["grad_bias"]}
    for i in range(2):
        out[f"mlp/{i}/kernel"], out[f"mlp/{i}/bias"] = z[f"grad_mlp_kernel_{i}"], z[f"grad_mlp_bias_{i}"]
    return out
