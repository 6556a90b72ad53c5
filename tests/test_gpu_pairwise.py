"""The in-batch pairwise ranking losses on the GPU: mm_inbatch_pairwise_fwd / _bwd against the float64 restatement
(tests/pairwise_oracle.py) for every loss kind, then TwoTowerModel and MatrixFactorizationModel compiled with them
(TwoTowerTrainer): one step, three steps under each optimizer, graph replay, memory, learning, and one step at the
benchmark's shape."""
import numpy as np
import pytest
import torch

import models_b200 as mm
from models_b200 import datasets, ops
from tests import helpers as H
from tests import pairwise_oracle as O

pytestmark = pytest.mark.gpu

KINDS = O.KINDS
# (B, N, D, downscore, T, in_batch): every (padded width 64 / 128) x kind kernel instantiation is reached
# (tests/test_pairwise_host.py).  in_batch: the negatives are the positives with their ids (N == B), the trainer's case:
# the row's own column is the one down-scored and dpos may alias dneg; the other cases draw separate negatives.
KERNEL_CASES = [(B, N, D, ds, T, ib) for B, N in ((1, 1), (37, 37), (129, 256), (300, 1000), (1024, 1024)) for D in (16, 64, 128)
                for ds in (True, False) for T in (1.0, 0.05) for ib in ((False, True) if B == N else (False,))]


def allclose(got, ref, rtol=2e-3, atol_rel=2e-4, what="", floor=0.0, terms=None):
    """|got - ref| <= atol + rtol |ref| + 5e-5 terms with atol = atol_rel max|ref|, at least `floor`.  terms (same shape,
    optional): the sum of the magnitudes of the terms each value sums (a gradient that cancels carries the fp32 error of
    its terms, not of its result)."""
    got = got.detach().cpu().double().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    ref = ref.detach().cpu().double().numpy() if isinstance(ref, torch.Tensor) else np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    atol = max(atol_rel * float(np.abs(ref).max()) if ref.size else 0.0, floor, 1e-30)
    if terms is not None:
        atol = atol + 5e-5 * (terms.detach().cpu().double().numpy() if isinstance(terms, torch.Tensor) else np.asarray(terms))
    bad = np.abs(got - ref) > atol + rtol * np.abs(ref)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} off, worst {float(np.abs(got - ref).max()):.3e} (atol {atol:.3e})"


# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
def _case(device, B, N, D, seed, in_batch=None):
    g = np.random.default_rng(seed)
    in_batch = (N == B and seed % 2 == 0) if in_batch is None else in_batch
    s = 1.0 / np.sqrt(np.sqrt(D))  # dot products of order 1, as for normalised embeddings
    q = torch.from_numpy((g.standard_normal((B, D)) * s).astype(np.float32)).to(device)
    pos = torch.from_numpy((g.standard_normal((B, D)) * s).astype(np.float32)).to(device)
    neg = pos if in_batch else torch.from_numpy((g.standard_normal((N, D)) * s).astype(np.float32)).to(device)
    n_ids = max(2, min(B, N) // 4)  # many duplicates
    pid = torch.from_numpy(g.integers(0, n_ids, B).astype(np.int64)).to(device)
    nid = pid if neg is pos else torch.from_numpy(g.integers(0, n_ids, N).astype(np.int64)).to(device)
    return q, pos, neg, pid, nid


def _run(q, pos, neg, pid, nid, kind, downscore, T, alias=False, lam=1.0):
    B, D = q.shape
    N = neg.shape[0]
    sp = torch.empty(B, device=q.device)
    ops.positive_scores(q, pos, sp, temperature=T)
    qs, ns = ops.split_rows(q), ops.split_rows(neg)
    stats = torch.full((B, 4), float("nan"), device=q.device)
    loss = torch.zeros(1, device=q.device)
    kw = dict(pos_ids=pid, neg_ids=nid, downscore=downscore, false_neg_score=O.MIN_FLOAT, temperature=T, reg_lambda=lam)
    ops.inbatch_pairwise(qs, ns, D, sp, stats, kind, loss=loss, **kw)
    dq = torch.full((B, D), float("nan"), device=q.device)
    dneg = torch.full((N, D), float("nan"), device=q.device)
    dpos = dneg if alias else torch.full((B, D), float("nan"), device=q.device)
    ops.inbatch_pairwise_backward(qs, ns, D, sp, stats, q, pos, dq, dpos, dneg, kind, **kw)
    torch.cuda.synchronize()
    return loss, stats, dq, dpos, dneg


def _ref(q, pos, neg, pid, nid, kind, downscore, T, lam=1.0):
    qd, pd, nd = (t.detach().cpu().double().requires_grad_(True) for t in (q, pos, neg))
    loss = O.pairwise_loss(qd, pd, nd, kind, pid.cpu().numpy(), nid.cpu().numpy(), T, downscore, lam)
    loss.backward()
    return float(loss.item()), qd.grad, pd.grad, nd.grad


def _terms(q, pos, neg, pid, nid, kind, downscore, T, lam=1.0):
    """(dq, dpos, dneg) of the magnitudes: |dL/dsp| |pos| + |dL/dsn| |neg|, |dL/dsp| |q|, |dL/dsn|^T |q| (each / T, the
    down-scored constants excluded): the scale of the terms each gradient value sums."""
    qd, pd, nd = (t.detach().cpu().double() for t in (q, pos, neg))
    sp, sn = O.inbatch_scores(qd, pd, nd, pid.cpu().numpy(), nid.cpu().numpy(), T, downscore)
    sp.requires_grad_(True), sn.requires_grad_(True)
    (O.element_losses(sp, sn, kind, lam).mean()).backward()
    gp, gn = sp.grad.abs() / T, sn.grad.abs() / T
    with torch.no_grad():  # the -max kinds' dloss/ds is itself a sum over the row's soft-max Jacobian: its terms' scale
        c = 1.0 / sn.numel()
        w = torch.softmax(sn, dim=1)
        if kind == "top1-max":
            e = torch.sigmoid(sn - sp) + torch.sigmoid(sn * sn)
            gn = gn + c * w * (e + (e * w).sum(1, keepdim=True)) / T
        elif kind == "bpr-max":
            gn = gn + c * (torch.sigmoid(sp - sn) + w * (sn.shape[1] + lam * (sn * sn * w).sum(1, keepdim=True)
                                                         + lam * (2 * sn + sn * sn).abs())) / T
    if downscore:
        gn = gn * (pid.cpu().view(-1, 1) != nid.cpu().view(1, -1))
    return gp * pd.abs() + gn @ nd.abs(), gp * qd.abs(), gn.T @ qd.abs()


def _floor(q, pos, neg, T, kind=None):
    """One element of the (B, N) gradient tile, c / T |x| (c = 1 / (B N)): what an element on the other side of a kink
    (its score within fp32 rounding of it) moves a gradient row by.  Only kinds with a kink the scores can reach get it:
    hinge (1 + u = 0), logistic (TF's gradient 0 at exactly u = 0, the own column without down-scoring) and, at T = 0.05
    where d can pass -104, the eps0 branch of BPR / BPR-max; every other comparison is relative to max |ref|."""
    if kind is not None and not (kind in ("hinge", "logistic") or (kind in ("bpr", "bpr-max") and T < 1.0)):
        return 0.0
    B, N = q.shape[0], neg.shape[0]
    return 4.0 / (B * N) / T * max(float(t.abs().max()) for t in (q, pos, neg))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B,N,D,downscore,T,in_batch", KERNEL_CASES)
def test_kernels_match_float64(device, B, N, D, downscore, T, in_batch, kind):
    q, pos, neg, pid, nid = _case(device, B, N, D, seed=B * 1000 + N + D, in_batch=in_batch)
    assert (neg is pos) == in_batch
    loss, stats, dq, dpos, dneg = _run(q, pos, neg, pid, nid, kind, downscore, T)
    want, gq, gp, gn = _ref(q, pos, neg, pid, nid, kind, downscore, T)
    got = float(loss.item())
    assert np.isfinite(got) and abs(got - want) <= 1e-4 * max(1.0, abs(want)), (got, want)
    floor = _floor(q, pos, neg, T, kind)
    tq, tp, tn = _terms(q, pos, neg, pid, nid, kind, downscore, T)
    allclose(dq, gq, what="dq", floor=floor, terms=tq)
    allclose(dpos, gp, what="dpos", floor=floor, terms=tp)
    allclose(dneg, gn, what="dneg", floor=floor, terms=tn)
    if neg is pos:  # in-batch: the item tower's gradient is the sum, written in one buffer when dpos aliases dneg
        _, _, dq2, dsum, _ = _run(q, pos, neg, pid, nid, kind, downscore, T, alias=True)
        assert torch.equal(dq2, dq)
        allclose(dsum, gp + gn, what="dpos + dneg", floor=2 * floor, terms=tp + tn)


@pytest.mark.parametrize("kind", KINDS)
def test_reruns_are_bit_identical(device, kind):
    """Two calls give the same bits (every output row is written by one CTA, sums in a fixed order); reg_lambda reaches
    BPR-max only."""
    q, pos, neg, pid, nid = _case(device, 700, 700, 64, seed=2)
    a = _run(q, pos, neg, pid, nid, kind, True, 0.5, alias=True)
    b = _run(q, pos, neg, pid, nid, kind, True, 0.5, alias=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    c = _run(q, pos, neg, pid, nid, kind, True, 0.5, alias=True, lam=0.25)
    assert torch.equal(a[2], c[2]) == (kind != "bpr-max")
    if kind == "bpr-max":
        want = _ref(q, pos, neg, pid, nid, kind, True, 0.5, lam=0.25)
        assert abs(float(c[0].item()) - want[0]) <= 1e-4 * abs(want[0])


def test_eps0_constants_on_the_device(device):
    """T = 1, down-scoring: every row's own column adds sigmoid(655^2) = 1 to TOP1 and -log(1e-24) = 55.26 to BPR-max
    (its float32 soft-max weight is 0) — the row sums of the kernel carry them."""
    B, D = 64, 32
    q, pos, _, _, _ = _case(device, B, B, D, seed=4)
    ids = torch.arange(B, device=device)
    for kind, const in (("top1", 1.0), ("bpr-max", O.EPS0_LOSS)):
        _, stats, *_ = _run(q, pos, pos, ids, ids, kind, True, 1.0)
        sp, sn = O.inbatch_scores(q.cpu().double(), pos.cpu().double(), pos.cpu().double(), ids.cpu().numpy(), ids.cpu().numpy())
        per_row = O.element_losses(sp, sn, kind).sum(1)
        np.testing.assert_allclose(stats[:, 0].cpu().double().numpy(), per_row.numpy(), rtol=1e-5)
        assert float(per_row.min()) > const - 1e-3


# ---------------------------------------------------------------------------------------------------------------
# the training step
# ---------------------------------------------------------------------------------------------------------------
def _batch(schema, n, seed):
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, n, seed=seed))
    return feats


def _oracle_towers(model):
    out = {}
    for tag, tb in (("query", model.body.query), ("item", model.body.item)):
        emb = tb.inputs.embeddings
        out[tag] = {"tables": {f: H.to_numpy(t.table) for f, t in emb.feature_to_table.items()},
                    "combiner": {f: t.sequence_combiner or "mean" for f, t in emb.feature_to_table.items()},
                    "continuous": list(tb.inputs.continuous.features) if tb.inputs.continuous is not None else [],
                    "layers": H.mlp_layers(tb.mlp) if tb.mlp is not None else []}
    return out


def _oracle_batch(feats, towers):
    b = dict(feats)
    for t in towers.values():
        for f in t["tables"]:
            if f + "__values" in feats:
                b[f] = (feats[f + "__values"], feats[f + "__offsets"])
    return b


def _model(variant, T=0.5, seed=7, activation="relu"):
    """(schema, model, l2 (post), l2_reg) on ML-1M."""
    mm.set_seed(seed)
    schema = datasets.movielens_1m_schema()
    if variant in ("two-tower", "two-tower l2-norm"):
        post = "l2-norm" if variant.endswith("l2-norm") else None
        model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([64, 32], activation=activation), post=post, logits_temperature=T)
        return schema, model, post is not None, None
    lam = 1e-3 if variant == "mf l2_reg" else 0.0
    model = mm.MatrixFactorizationModel(schema, 32, embeddings_l2_reg=lam, logits_temperature=T)
    return schema, model, False, {"query": lam, "item": lam}


def _close(got, ref, tol, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30)
    err = float(np.abs(got - ref).max()) / scale
    assert err < tol, f"{what}: max |diff| / max |ref| = {err:.3e} (tol {tol})"


@pytest.mark.parametrize("variant", ["two-tower", "two-tower l2-norm", "mf", "mf l2_reg"])
@pytest.mark.parametrize("kind", KINDS)
def test_one_step_matches_restatement(device, kind, variant):
    """One step of TwoTowerModel (post None / l2-norm) or MatrixFactorizationModel (with / without embeddings_l2_reg)
    compiled with `kind`: the loss, the regularization and every dense and table gradient."""
    schema, model, l2, l2_reg = _model(variant)
    feats = _batch(schema, 256, 31)
    model.build(device)
    towers = _oracle_towers(model)
    lam = 0.5 if kind == "bpr-max" else 1.0
    loss = mm.losses.BPRmaxLoss(reg_lambda=lam) if kind == "bpr-max" else kind
    want, want_reg, grads = O.loss_and_grads(_oracle_batch(feats, towers), towers, "movieId", kind, lam, 0.5, l2, l2_reg)
    model.compile(optimizer="sgd", loss=loss)
    tr = model.trainer(256)
    tr.forward_backward(H.device_batch(feats, device))
    torch.cuda.synchronize()
    got = float(tr.loss[0].item())
    assert abs(got - want) <= 5e-5 * max(1.0, abs(want)), (got, want)
    assert abs(float(tr.loss[1].item()) - want_reg) <= 1e-5 * max(want_reg, 1e-12)
    g = tr.gradients()
    for tag, tw in (("query", model.body.query), ("item", model.body.item)):
        for i, l in enumerate(tw.mlp.dense_layers if tw.mlp is not None else []):
            _close(H.to_numpy(g[f"{tw.name}/{l.name}/kernel"]), grads[f"{tag}/kernel_{i}"], 5e-4, f"{tag} kernel {i}")
            _close(H.to_numpy(g[f"{tw.name}/{l.name}/bias"]), grads[f"{tag}/bias_{i}"], 5e-4, f"{tag} bias {i}")
    for f, (ids, rows) in tr.table_gradients().items():
        tag = "query" if f in towers["query"]["tables"] else "item"
        ref = grads[f"{tag}/table/{f}"]
        dense = np.zeros_like(ref)
        ids, rows = ids.cpu().numpy().astype(np.int64), rows.cpu().numpy().astype(np.float64)
        ok = ids >= 0
        np.add.at(dense, ids[ok], rows[ok])
        _close(dense, ref, 5e-4, f"table {f}")


def _hyper(opt):
    return dict(beta_1=float(np.float32(0.9)), beta_2=float(np.float32(0.999)), epsilon=float(np.float32(1e-7))) if opt == "adam" else {}


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("kind", KINDS)
def test_three_steps_match_restatement(device, kind, opt):
    """Three steps, the last batch smaller than the compiled one (its leading rows): the losses and every trained
    variable against the restatement with the Keras update rules.  The towers are linear: a trajectory through relu
    towers can bring a pre-activation within the fp32 error of the forward of zero, and then the step's relu mask, not the
    loss, decides the comparison (the one-step tests train relu towers)."""
    schema, model, l2, _ = _model("two-tower l2-norm", T=0.5, activation="linear")
    feats = [_batch(schema, n, 100 + i) for i, n in enumerate((256, 256, 200))]
    model.build(device)
    towers0 = _oracle_towers(model)
    lr = {"sgd": 0.05, "adagrad": 0.05, "adam": 0.002}[opt]
    model.compile(optimizer={"sgd": mm.SGD, "adagrad": mm.Adagrad, "adam": mm.Adam}[opt](learning_rate=lr), loss=kind)
    model.trainer(256)
    got = [float(model.train_step((H.device_batch(f, device),))["loss"].item()) for f in feats]
    want, towers = O.train_steps([_oracle_batch(f, towers0) for f in feats], towers0, "movieId", kind, opt, lr, temperature=0.5,
                                 l2=True, **_hyper(opt))
    np.testing.assert_allclose(got, want, rtol=2e-4)
    # Adam divides by |g| + eps: an fp32 error dg of a small gradient moves its update by lr dg / (|g| + eps), so its
    # bound is looser than SGD's and Adagrad's, whose updates are linear in the gradient to fp32 precision here
    tol = 5e-3 if opt == "adam" else 1e-3
    now = _oracle_towers(model)

    def update_close(w, w0, ref, what):
        # c = 1 / (B N) makes these gradients ~B times smaller than the soft-max's: an fp32 weight then moves by few of its
        # ulps per step, so each step may round the update by half an ulp of the weight
        ulps = 3 * float(np.abs(w0).max()) * 2.0 ** -23
        d, r = np.asarray(w - w0, np.float64), np.asarray(ref - w0, np.float64)
        err = float(np.abs(d - r).max())
        assert err <= tol * float(np.abs(r).max()) + ulps, f"{what}: max |diff| {err:.3e}, max |ref| {float(np.abs(r).max()):.3e}"

    for tag in ("query", "item"):
        for i, (l, l0) in enumerate(zip(now[tag]["layers"], towers0[tag]["layers"])):
            update_close(l["kernel"], l0["kernel"], towers[tag]["layers"][i]["kernel"], f"{tag} kernel {i} update")
        for f in now[tag]["tables"]:
            update_close(now[tag]["tables"][f], towers0[tag]["tables"][f], towers[tag]["tables"][f], f"{tag} table {f} update")


def _retrieval_model(seed=3):
    mm.set_seed(seed)
    schema = datasets.retrieval_10m_schema(n_items=50_000, n_users=5_000)
    return schema, mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([128, 64]))


@pytest.mark.parametrize("kind", ["bpr-max", "top1_v2"])
def test_graph_replay_equals_eager(device, kind):
    B = 512
    feats = None
    results = []
    for mode in ("eager", "graph"):
        schema, model = _retrieval_model()
        feats = feats or [_batch(schema, B, 40 + i) for i in range(3)]
        model.compile(optimizer=mm.Adagrad(0.05), loss=kind)
        tr = model.trainer(B)
        if mode == "eager":
            losses = [float(tr.step(H.device_batch(f, device), None)[0].item()) for f in feats]
        else:
            tr.capture(H.device_batch(feats[0], device))
            losses = [float(tr.replay(H.device_batch(f, device))[0].item()) for f in feats]
        torch.cuda.synchronize()
        results.append((losses, {k: np.array(v) for k, v in model.state_dict().items()}))
    (le, we), (lg, wg) = results
    np.testing.assert_allclose(lg, le, rtol=1e-6)
    for k in we:
        np.testing.assert_allclose(wg[k], we[k], rtol=1e-6, atol=1e-7, err_msg=k)


def test_no_scores_materialised(device):
    """At B = 8192 the (B, B) scores would take 268 MB; one more step after a warm one allocates well under 64 MB."""
    B = 8192
    schema, model = _retrieval_model()
    model.compile(optimizer=mm.Adagrad(0.05), loss="bpr-max")
    model.trainer(B)
    x = H.device_batch(_batch(schema, B, 9), device)
    model.train_step((x,))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(device)
    base = torch.cuda.memory_allocated(device)
    model.train_step((x,))
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(device) - base < 64 * 2**20


@pytest.mark.parametrize("kind", ["bpr", "bpr-max"])
def test_fit_learns_a_planted_rule(device, kind):
    """Item id = f(user id): in-batch recall@10 rises well above its value before training."""
    schema, model = _retrieval_model(seed=11)
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
    model.compile(optimizer=mm.Adam(0.01), loss=kind)
    hist = model.fit(train, batch_size=256, epochs=5)
    after = model.evaluate(held)["recall_at_10"]
    assert hist.history["loss"][-1] < hist.history["loss"][0], hist.history["loss"]
    assert after > before + 0.3, (before, after, hist.history["loss"])


def test_benchmark_shape_step(device):
    """tools/train_pairwise_bench.py's shape (retrieval_10m_schema, towers [256, 128], B = 16 384): one step per kind is
    finite, and the kernels' row losses and query gradients on sampled rows match the float64 restatement of those
    rows (each row's losses and dq depend on that row's scores alone)."""
    B = 16384
    mm.set_seed(5)
    schema = datasets.retrieval_10m_schema()
    model = mm.TwoTowerModel(schema, query_tower=mm.MLPBlock([256, 128]))
    x = H.device_batch(_batch(schema, B, 3), device)
    rows = torch.from_numpy(np.random.default_rng(0).choice(B, 48, replace=False)).to(device)
    for kind in KINDS:
        model.compile(optimizer=mm.Adagrad(0.05), loss=kind)
        tr = model.trainer(B)
        tr.forward_backward(x)
        torch.cuda.synchronize()
        assert np.isfinite(float(tr.loss[0].item())), kind
        q, it = tr.towers[0]["h"][-1][:B], tr.towers[1]["h"][-1][:B]
        ids = x["item_id"].reshape(-1).long()
        loss, stats, dq, _, _ = _run(q.contiguous(), it.contiguous(), it.contiguous(), ids, ids, kind, True, 1.0, alias=True)
        assert torch.isfinite(stats).all() and torch.isfinite(dq).all(), kind
        qd = q[rows].double().requires_grad_(True)
        itd = it.double()
        sp = (qd * itd[rows]).sum(-1, keepdim=True)
        sn = qd @ itd.T
        sn = torch.where(ids[rows].view(-1, 1) == ids.view(1, -1), torch.full_like(sn, float(np.float32(O.MIN_FLOAT))), sn)
        el = O.element_losses(sp, sn, kind)
        per_row = el.sum(1) if kind != "top1_v2" else el.sum(1) * B
        (el.sum() / (B * (B if kind != "top1_v2" else 1))).backward()
        np.testing.assert_allclose(stats[rows, 0].cpu().double().numpy(), per_row.detach().cpu().numpy(), rtol=2e-4, atol=1e-3)
        allclose(dq[rows], qd.grad, what=f"{kind} dq rows", floor=_floor(q, it, it, 1.0, kind))
        assert abs(float(loss.item()) - float(tr.loss[0].item())) <= 1e-6 * max(1.0, abs(float(loss.item())))
