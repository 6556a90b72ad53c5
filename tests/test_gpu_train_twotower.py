"""The two-tower training step on the GPU: mm_inbatch_softmax_ce_backward and mm_l2_normalize_backward against float64
autograd, then TwoTowerTrainer (mm.TwoTowerModel compile / train_step / fit) against tests/twotower_train_oracle.py with
the Keras update rules, graph replay, memory, and what training leaves in the model."""
import ctypes as C

import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import _cabi, datasets, ops
from tests import helpers as H
from tests import twotower_train_oracle as O

pytestmark = pytest.mark.gpu


def close(got, ref, tol, what=""):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    ref = np.asarray(ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got - ref))) / scale if ref.size else 0.0
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


def allclose(got, ref, rtol=1e-3, atol_rel=1e-4, what="", floor=0.0):
    """|got - ref| <= atol + rtol |ref| with atol = atol_rel max|ref|, at least `floor`: a gradient is a sum of terms of
    opposite sign, so when they cancel its fp32 error is set by the terms, not by the result."""
    got = got.detach().cpu().double().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    ref = ref.detach().cpu().double().numpy() if isinstance(ref, torch.Tensor) else np.asarray(ref, np.float64)
    atol = max(atol_rel * float(np.abs(ref).max()), floor, 1e-30)
    bad = np.abs(got - ref) > atol + rtol * np.abs(ref)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} off, worst {float(np.abs(got - ref).max()):.3e} (atol {atol:.3e})"


# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
def _ce_case(device, B, N, D, downscore, logq, T, seed):
    g = np.random.default_rng(seed)
    s = 1.0 / np.sqrt(np.sqrt(D))  # dot products of order 1, as for normalised embeddings
    q = torch.from_numpy((g.standard_normal((B, D)) * s).astype(np.float32)).to(device)
    pos = torch.from_numpy((g.standard_normal((B, D)) * s).astype(np.float32)).to(device)
    neg = pos if N == B and seed % 2 == 0 else torch.from_numpy((g.standard_normal((N, D)) * s).astype(np.float32)).to(device)
    n_ids = max(2, min(B, N) // 4)  # many duplicates
    pid = torch.from_numpy(g.integers(0, n_ids, B).astype(np.int64)).to(device)
    nid = pid if neg is pos else torch.from_numpy(g.integers(0, n_ids, N).astype(np.int64)).to(device)
    prob = torch.from_numpy(g.uniform(1e-4, 0.5, N).astype(np.float32)).to(device) if logq else None
    return q, pos, neg, pid, nid, prob


def _ce_ref(q, pos, neg, pid, nid, prob, downscore, T, c):
    """float64 autograd: loss = sum_b c (lse_b - s_b0) with the logits of mm_inbatch_softmax_ce."""
    qd, pd, nd = (t.detach().cpu().double().requires_grad_(True) for t in (q, pos, neg))
    s0 = (qd * pd).sum(-1, keepdim=True) / T
    sn = qd @ nd.T
    if prob is not None:
        sn = sn - torch.log(prob.cpu().double() + 1e-16).view(1, -1)
    if downscore:
        m = pid.cpu().view(-1, 1) == nid.cpu().view(1, -1)
        sn = torch.where(m, torch.full_like(sn, float(np.float32(O.MIN_FLOAT))), sn)
    s = torch.cat([s0, sn / T], dim=1)
    loss = (c * (torch.logsumexp(s, 1) - s[:, 0])).sum()
    loss.backward()
    return float(loss.item()), qd.grad, pd.grad, nd.grad


def _ce_run(q, pos, neg, pid, nid, prob, downscore, T, c_dev, alias=False):
    B, D = q.shape
    N = neg.shape[0]
    stats = ops.inbatch_softmax_ce(q, pos, neg, pos_ids=pid, neg_ids=nid, downscore=downscore, false_neg_score=O.MIN_FLOAT,
                                   neg_prob=prob, temperature=T)
    qs = ops.split_rows(q)
    ns = ops.split_rows(neg)
    dq = torch.full((B, D), float("nan"), device=q.device)
    dneg = torch.full((N, D), float("nan"), device=q.device)
    dpos = dneg if alias else torch.full((B, D), float("nan"), device=q.device)
    loss = torch.zeros(1, device=q.device)
    ops.inbatch_softmax_ce_backward(qs, ns, D, stats, q, pos, c_dev, dq, dpos, dneg, loss=loss, pos_ids=pid, neg_ids=nid,
                                    downscore=downscore, false_neg_score=O.MIN_FLOAT, neg_prob=prob, temperature=T)
    torch.cuda.synchronize()
    return dq, dpos, dneg, loss


@pytest.mark.parametrize("T", [1.0, 0.05])
@pytest.mark.parametrize("logq", [False, True])
@pytest.mark.parametrize("downscore", [True, False])
@pytest.mark.parametrize("D", [16, 64, 128])
@pytest.mark.parametrize("BN", [(1, 1), (37, 37), (129, 256), (300, 1000), (1024, 1024)])
def test_ce_backward_matches_float64(device, BN, D, downscore, logq, T):
    B, N = BN
    q, pos, neg, pid, nid, prob = _ce_case(device, B, N, D, downscore, logq, T, seed=B * 1000 + N + D)
    c = torch.full((1,), 1.0 / B, device=device)
    dq, dpos, dneg, loss = _ce_run(q, pos, neg, pid, nid, prob, downscore, T, c)
    want_loss, gq, gp, gn = _ce_ref(q, pos, neg, pid, nid, prob, downscore, T, 1.0 / B)
    assert abs(float(loss.item()) - want_loss) <= 1e-4 * max(1.0, abs(want_loss)), (float(loss.item()), want_loss)
    # fp32 rounding of one term c p x / T (p <= 1) at a few ulps
    floor = 1e-6 / B / T * max(float(t.abs().max()) for t in (q, pos, neg))
    allclose(dq, gq, what="dq", floor=floor)
    allclose(dpos, gp, what="dpos", floor=floor)
    allclose(dneg, gn, what="dneg", floor=floor)
    if neg is pos:  # in-batch: the item tower's gradient is the sum
        allclose(dpos + dneg, gp + gn, what="dpos + dneg", floor=floor)


@pytest.mark.parametrize("D", [64, 128])
def test_ce_backward_alias_deterministic_and_row_scale(device, D):
    """dpos aliasing dneg writes the sum; two calls are bit-identical; a per-row scale vector equals its scalar."""
    B = 700
    q, pos, neg, pid, nid, prob = _ce_case(device, B, B, D, True, False, 0.5, seed=2)
    assert neg is pos
    c = torch.full((1,), 1.0 / B, device=device)
    dq, dpos, dneg, loss = _ce_run(q, pos, neg, pid, nid, None, True, 0.5, c)
    dq2, dsum, _, loss2 = _ce_run(q, pos, neg, pid, nid, None, True, 0.5, c, alias=True)
    assert torch.equal(dq, dq2) and torch.equal(loss, loss2)
    close(dsum, dpos.double() + dneg.double(), 1e-6, "aliased dpos + dneg")
    dq3, dsum3, _, loss3 = _ce_run(q, pos, neg, pid, nid, None, True, 0.5, c, alias=True)
    assert torch.equal(dq2, dq3) and torch.equal(dsum, dsum3) and torch.equal(loss2, loss3), "two calls differ"
    cv = torch.full((B,), 1.0 / B, device=device)
    dq4, dsum4, _, loss4 = _ce_run(q, pos, neg, pid, nid, None, True, 0.5, cv, alias=True)
    assert torch.equal(dq4, dq2) and torch.equal(dsum4, dsum)


def test_ce_backward_rejects_bad_arguments(device):
    lib = _cabi.load()
    B, D = 64, 64
    qs = torch.zeros((B, 256), dtype=torch.bfloat16, device=device)
    f = torch.zeros((B, 160), device=device)
    st = torch.zeros((B, 3), device=device)
    one = torch.ones(1, device=device)
    p = f.data_ptr()

    def call(D=D, q_split=qs.data_ptr(), T=1.0, stats=st.data_ptr(), dpos=p + 4096 * 4, dneg=p + 8192 * 4, N=B):
        return lib.mm_inbatch_softmax_ce_backward(q_split, qs.data_ptr(), B, N, D, None, None, _cabi.MM_I64, 0, -1.0, None, T, stats,
                                                  p, p, one.data_ptr(), 1, p + 2048 * 4, dpos, dneg, None, None)

    assert call(D=129) == -2  # MM_ERR_UNSUPPORTED: Kp > 128
    assert call(q_split=qs.data_ptr() + 2) == -3  # MM_ERR_ALIGN
    assert call(T=0.0) == -1 and call(T=-1.0) == -1
    assert call(stats=None) == -1
    assert call(dpos=p + 4096 * 4, dneg=p + 4096 * 4, N=B - 1) == -1  # aliasing needs N == B
    assert lib.mm_inbatch_softmax_ce_backward(qs.data_ptr(), qs.data_ptr(), B, B, D, None, None, _cabi.MM_I64, 1, -1.0, None, 1.0,
                                              st.data_ptr(), p, p, one.data_ptr(), 1, p, p + 16, p + 32, None, None) == -1  # ids
    torch.cuda.synchronize()


def test_l2_normalize_backward_matches_float64(device):
    g = np.random.default_rng(5)
    x = g.standard_normal((257, 48)).astype(np.float32)
    x[3] = 0.0  # an all-zero row: the gradient passes the constant 1e-6 denominator
    x[4] = 1e-8  # sum of squares below 1e-12
    dy = g.standard_normal(x.shape).astype(np.float32)
    xd = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    y = xd / torch.sqrt(torch.clamp((xd * xd).sum(-1, keepdim=True), min=1e-12))
    (y * torch.tensor(dy, dtype=torch.float64)).sum().backward()
    X, DY = torch.from_numpy(x).to(device), torch.from_numpy(dy).to(device)
    got = ops.l2_normalize_backward(X, DY)
    close(got, xd.grad, 1e-5, "dx")
    np.testing.assert_allclose(got[3].cpu().numpy(), dy[3] / 1e-6, rtol=1e-6)
    ops.l2_normalize_backward(X, DY, DY)  # in place
    assert torch.equal(DY, got)


# ---------------------------------------------------------------------------------------------------------------
# the training step
# ---------------------------------------------------------------------------------------------------------------
def _ml1m_model(post=None, T=1.0, dims=(64, 32), seed=7):
    mm.set_seed(seed)
    schema = datasets.movielens_1m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock(list(dims)), post=post, logits_temperature=T)
    return schema, model


def _batch(schema, n, seed):
    batch = datasets.generate_batch(schema, n, seed=seed)
    feats, _ = datasets.split_targets(schema, batch)
    return feats


def _oracle_towers(model):
    out = {}
    for tag, tb in (("query", model.body.query), ("item", model.body.item)):
        emb = tb.inputs.embeddings
        out[tag] = {"tables": {f: H.to_numpy(t.table) for f, t in emb.feature_to_table.items()},
                    "combiner": {f: t.sequence_combiner or "mean" for f, t in emb.feature_to_table.items()},
                    "continuous": list(tb.inputs.continuous.features) if tb.inputs.continuous is not None else [],
                    "layers": H.mlp_layers(tb.mlp)}
    return out


def _oracle_batch(feats, towers):
    b = dict(feats)
    for t in towers.values():
        for f in t["tables"]:
            if f + "__values" in feats:
                b[f] = (feats[f + "__values"], feats[f + "__offsets"])
    return b


def _hyper(opt):
    return dict(beta_1=float(np.float32(0.9)), beta_2=float(np.float32(0.999)), epsilon=float(np.float32(1e-7))) if opt == "adam" else {}


@pytest.mark.parametrize("post", [None, "l2-norm"])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_three_steps_match_restatement(device, opt, post):
    """Three steps on ML-1M (one-hot ids, the ragged genres bag, continuous columns), the last batch smaller than the
    compiled one: losses and every trained variable against the float64 restatement with the Keras update rules."""
    schema, model = _ml1m_model(post=post, T=0.5)
    feats = [_batch(schema, n, 100 + i) for i, n in enumerate((256, 256, 200))]
    model.build(device)
    towers0 = _oracle_towers(model)
    lr = {"sgd": 0.05, "adagrad": 0.05, "adam": 0.002}[opt]
    model.compile(optimizer={"sgd": mm.SGD, "adagrad": mm.Adagrad, "adam": mm.Adam}[opt](learning_rate=lr))
    model.trainer(256)
    got = []
    for f in feats:
        got.append(float(model.train_step((H.device_batch(f, device),))["loss"].item()))
    want, towers = O.train_steps([_oracle_batch(f, towers0) for f in feats], towers0, "movieId", opt, lr, temperature=0.5,
                                 l2=post is not None, **_hyper(opt))
    np.testing.assert_allclose(got, want, rtol=2e-4)
    tol = 2e-3 if opt == "adam" else 5e-4
    now = _oracle_towers(model)
    for tag in ("query", "item"):
        for i, (l, l0) in enumerate(zip(now[tag]["layers"], towers0[tag]["layers"])):
            close(l["kernel"] - l0["kernel"], towers[tag]["layers"][i]["kernel"] - l0["kernel"], tol, f"{tag} kernel {i} update")
        for f in now[tag]["tables"]:
            close(now[tag]["tables"][f] - towers0[tag]["tables"][f], towers[tag]["tables"][f] - towers0[tag]["tables"][f], tol,
                  f"{tag} table {f} update")


GOLDEN = __import__("pathlib").Path(__file__).parent / "golden" / "twotower_train" / "ref_torch_twotower_train.npz"


@pytest.mark.parametrize("variant", [0, 1])
def test_one_step_matches_reference(device, variant):
    """One step of mm.TwoTowerModel on the weights and batch of the reference's torch two-tower step
    (tests/golden/twotower_train/ref_torch_twotower_train.npz: TabularInputBlock + EmbeddingTables(mean) -> MLPBlock per
    tower, in-batch ContrastiveOutput with false-negative rescoring, F.cross_entropy against class 0, autograd): the loss
    at rtol 1e-5, every tower variable's gradient and the summed IndexedSlices of every table at 3e-4 of each tensor's
    scale, at T = 1 and T = 0.5."""
    from models_b200.schema import ColumnSchema, Schema

    z = np.load(GOLDEN)
    vt, T = O.golden_variants(z)[variant]
    dim = int(z["dim"])

    def col(name, tower):
        tags = ("user",) if tower == "query" else ("item",)
        key = f"{tower}_table_{name}_rows_total"
        if key in z.files:
            is_list = name == "genres"
            props = {"domain": {"min": 0, "max": int(z[key]) - 1, "name": name}}
            if is_list:
                props["value_count"] = {"min": 1, "max": 4}
            extra = ("user_id",) if name == "userId" else ("item_id",) if name == "movieId" else ()
            return ColumnSchema(name, tags=("categorical",) + tags + extra, dtype="int64", is_list=is_list, is_ragged=is_list,
                                properties=props)
        return ColumnSchema(name, tags=("continuous",) + tags, dtype="float32")

    cols = [col(str(n), "query") for n in z["query_cols"]] + [col(str(n), "item") for n in z["item_cols"]]
    tower = [int(u) for u in z["tower"]]
    model = mm.TwoTowerModel(Schema(cols), query_tower=mm.MLPBlock(tower), item_tower=mm.MLPBlock(tower),
                             embedding_options=mm.EmbeddingOptions(embedding_dim_default=dim), logits_temperature=T)
    for tag, tw in (("query", model.body.query), ("item", model.body.item)):
        for name, table in tw.inputs.embeddings.tables.items():
            full = torch.zeros((int(z[f"{tag}_table_{name}_rows_total"]), dim), dtype=torch.float32)
            full[torch.from_numpy(z[f"{tag}_table_{name}_ids"])] = torch.from_numpy(z[f"{tag}_table_{name}_rows"])
            table.table = full.to(device).contiguous()
            table.built = True
        for l, i in zip(tw.mlp.dense_layers, range(len(tower))):
            l.set_weights(z[f"{tag}_kernel_{i}"], z[f"{tag}_bias_{i}"])
    model.build(device)
    batch = {k[len("batch_"):]: torch.from_numpy(z[k]).to(device) for k in z.files if k.startswith("batch_")}
    B = int(z["batch_movieId"].shape[0])
    model.compile(optimizer="sgd")
    tr = model.trainer(B)
    tr.forward_backward(batch)
    torch.cuda.synchronize()
    want = float(z[f"{vt}_loss"])
    got = float(tr.loss[0].item())
    assert abs(got - want) <= 1e-5 * abs(want), (got, want)
    grads = tr.gradients()
    for tag, tw in (("query", model.body.query), ("item", model.body.item)):
        for i, l in enumerate(tw.mlp.dense_layers):
            close(grads[f"{tw.name}/{l.name}/kernel"], z[f"{vt}_grad_{tag}_kernel_{i}"], 3e-4, f"{tag} kernel {i}")
            close(grads[f"{tw.name}/{l.name}/bias"], z[f"{vt}_grad_{tag}_bias_{i}"], 3e-4, f"{tag} bias {i}")
    slices = tr.table_gradients()
    for tag in ("query", "item"):
        for name in [str(n) for n in z[f"{tag}_cols"]]:
            if f"{tag}_table_{name}_ids" not in z.files:
                continue
            ids, rows = (t.cpu().numpy() for t in slices[name])
            ref_ids = z[f"{tag}_table_{name}_ids"]
            summed = np.zeros((len(ref_ids), dim))
            ok = ids >= 0
            np.add.at(summed, np.searchsorted(ref_ids, ids[ok]), rows[ok].astype(np.float64))
            assert np.isin(ids[ok], ref_ids).all()
            close(summed, z[f"{vt}_grad_{tag}_table_{name}_rows"], 3e-4, f"table {name}")


def _retrieval_model(B, seed=3):
    mm.set_seed(seed)
    schema = datasets.retrieval_10m_schema(n_items=50_000, n_users=5_000)
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([128, 64]))
    return schema, model


def test_graph_replay_equals_eager(device):
    B = 512
    feats = None
    results = []
    for mode in ("eager", "graph"):
        schema, model = _retrieval_model(B)
        feats = feats or [_batch(schema, B, 40 + i) for i in range(3)]
        model.compile(optimizer=mm.Adagrad(0.05))
        tr = model.trainer(B)
        losses = []
        if mode == "eager":
            for f in feats:
                losses.append(float(tr.step(H.device_batch(f, device), None)[0].item()))
        else:
            tr.capture(H.device_batch(feats[0], device))
            for f in feats:
                losses.append(float(tr.replay(H.device_batch(f, device))[0].item()))
        torch.cuda.synchronize()
        results.append((losses, {k: np.array(v) for k, v in model.state_dict().items()}))
    (le, we), (lg, wg) = results
    np.testing.assert_allclose(lg, le, rtol=1e-6)
    for k in we:
        np.testing.assert_allclose(wg[k], we[k], rtol=1e-6, atol=1e-7, err_msg=k)


def test_no_logits_materialised(device):
    """At B = 8192 the (B, 1+B) logits would take 268 MB; one more step after a warm one allocates well under 64 MB."""
    B = 8192
    schema, model = _retrieval_model(B)
    model.compile(optimizer=mm.Adagrad(0.05))
    model.trainer(B)
    x = H.device_batch(_batch(schema, B, 9), device)
    model.train_step((x,))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(device)
    base = torch.cuda.memory_allocated(device)
    model.train_step((x,))
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(device) - base < 64 * 2**20


def test_training_reaches_the_model(device, tmp_path):
    """After fit, model(batch, training=True) gives the logits the restatement computes from state_dict(); save / load
    round-trips the trained weights."""
    schema, model = _ml1m_model(post="l2-norm", T=0.2)
    feats = [_batch(schema, 128, 60 + i) for i in range(3)]
    model.compile(optimizer="adam")
    hist = model.fit([H.device_batch(f, device) for f in feats], batch_size=128, epochs=2)
    assert len(hist.history["loss"]) == 2 and all(np.isfinite(hist.history["loss"]))
    f = feats[0]
    pred = model(H.device_batch(f, device), training=True)
    towers = _oracle_towers(model)
    P = {}
    for tag, t in towers.items():
        for k, w in t["tables"].items():
            P[f"{tag}/table/{k}"] = torch.tensor(w, dtype=torch.float64)
        for i, l in enumerate(t["layers"]):
            P[f"{tag}/kernel_{i}"] = torch.tensor(l["kernel"], dtype=torch.float64)
            P[f"{tag}/bias_{i}"] = torch.tensor(l["bias"], dtype=torch.float64)
    ob = _oracle_batch(f, towers)
    q = O.l2_normalize(O.tower_forward(P, "query", towers["query"], ob, torch.float64))
    it = O.l2_normalize(O.tower_forward(P, "item", towers["item"], ob, torch.float64))
    s = torch.cat([(q * it).sum(-1, keepdim=True), q @ it.T], 1) / 0.2
    ids = torch.as_tensor(f["movieId"].astype(np.int64))
    mask = torch.cat([torch.zeros(len(ids), 1, dtype=torch.bool), ids.view(-1, 1) == ids.view(1, -1)], 1)
    got = pred.outputs.cpu().double()
    close(got[~mask], s[~mask], 1e-4, "training logits after fit")
    model.save(str(tmp_path / "m"))
    back = mm.Model.load(str(tmp_path / "m"), device=device)
    sd, sd2 = model.state_dict(), back.state_dict()
    assert sd.keys() == sd2.keys()
    for k in sd:
        assert np.array_equal(sd[k], sd2[k]), k


def test_fit_learns_a_planted_rule(device):
    """Item id = f(user id): in-batch recall@10 rises well above its value before training."""
    schema, model = _retrieval_model(256, seed=11)
    g = np.random.default_rng(0)
    n_users = 2000
    rule = g.integers(0, 50_000, n_users)

    def batch(seed):
        r = np.random.default_rng(seed)
        f = _batch(schema, 256, seed)
        f["user_id"] = r.integers(0, n_users, 256).astype(f["user_id"].dtype)
        f["item_id"] = rule[f["user_id"]].astype(f["item_id"].dtype)
        return H.device_batch(f, device)

    train = [batch(1000 + i) for i in range(40)]
    held = [batch(5000 + i) for i in range(4)]
    before = model.evaluate(held)["recall_at_10"]
    model.compile(optimizer=mm.Adam(0.01))
    hist = model.fit(train, batch_size=256, epochs=5)
    after = model.evaluate(held)["recall_at_10"]
    assert hist.history["loss"][-1] < hist.history["loss"][0], hist.history["loss"]
    assert after > before + 0.3, (before, after, hist.history["loss"])


def test_unsupported_configurations(device):
    from models_b200.retrieval import PopularityBasedSamplerV2

    schema = datasets.movielens_1m_schema()
    x = H.device_batch(_batch(schema, 64, 1), device)

    def fails(model, match, loss=None):
        model.compile(optimizer="sgd", **({"loss": loss} if loss else {}))
        with pytest.raises(NotImplementedError, match=match):
            model.train_step((x,))

    with pytest.raises(NotImplementedError, match="loss"):
        mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32])).compile(optimizer="sgd", loss="mse")
    fails(mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32]), samplers=[PopularityBasedSamplerV2(max_id=3000)]), "in-batch")
    fails(mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32], normalization="batch_norm")), "normalization")
    fails(mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32], dropout=0.1)), "dropout")
    fails(mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32], activation="tanh")), "activation")
    m = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32]))
    m.prediction.scorer.sampled_softmax_mode = True
    fails(m, "sampled_softmax_mode")
    m = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32]))
    m.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="process group"):
        m.trainer(64, group=object())
    mm.set_dense_engine("fp32")
    try:
        fails(mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32])), "fp32")
    finally:
        mm.set_dense_engine("auto")
    m = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32]))
    m.body.query.inputs.embeddings.tables["userId"].trainable = False
    fails(m, "frozen")
    from models_b200.schema import Schema

    shared = Schema(list(schema) + [datasets._cat("userId_alt", 6040, tags=(mm.Tags.USER,), domain_name="userId")])
    xs = H.device_batch(_batch(shared, 64, 2), device)
    m = mm.TwoTowerModel(shared, query_tower=mm.MLPBlock([32]))
    m.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="shared"):
        m.train_step((xs,))
    m = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([32]))
    m.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="sample_weight"):
        m.train_step((x, None, torch.ones(64, device=device)))
    q = mm.Encoder(schema.select_by_tag(mm.Tags.USER), mm.MLPBlock([32]))
    c = mm.Encoder(schema.select_by_tag(mm.Tags.ITEM), mm.MLPBlock([32]))
    v2 = mm.TwoTowerModelV2(q, c)
    v2.compile(optimizer="sgd")
    with pytest.raises(NotImplementedError, match="TwoTowerModelV2"):
        v2.trainer(64)
