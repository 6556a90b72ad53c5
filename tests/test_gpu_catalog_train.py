"""Full-catalog soft-max cross-entropy backward (mm_catalog_softmax_ce_backward, inbatch_flash_kernel<CatalogCE, DQ / DN>)
against float64: dx, dE, db and the loss over batch sizes around the 128-row tile, catalogs from one row to 100 003 and
10 M, every padded width, temperatures, bias on and off, per-row weights, both label dtypes, the split dq path and
bit-identical repeats."""
import numpy as np
import pytest
import torch

from models_b200 import ops
from oracle import oracle
from tests.catalog_train_oracle import catalog_ce

pytestmark = pytest.mark.gpu

EPS_SPLIT = 2.0 ** -15  # 3-pass split-bf16 products: a few units of 2^-16 of the sum of |terms|


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def run(device, x, E, b, y, T, sw, label_dtype=torch.int64, oob=None):
    """The kernels through the public operands: stats from mm_catalog_score on (x / T, b / T), then the backward."""
    B, D = x.shape
    N = E.shape[0]
    xt = dev((x / np.float32(T)).astype(np.float32) if T != 1.0 else x, device)
    bt = None if b is None else dev((b / np.float32(T)).astype(np.float32) if T != 1.0 else b, device)
    labels = dev(y, device).to(label_dtype)
    e_split = ops.split_rows(dev(E, device))
    stats, _, _ = ops.catalog_score(xt, e_split, N, bias=bt, targets=labels, k=0)
    c = dev((np.ones(B, np.float32) if sw is None else sw.astype(np.float32)) / np.float32(B), device)
    dx = torch.full((B, D), float("nan"), device=device)
    de = torch.full((N, D), float("nan"), device=device)
    db = torch.full((N,), float("nan"), device=device) if b is not None else None
    loss = torch.zeros(1, device=device)
    ops.catalog_softmax_ce_backward(ops.split_rows(xt), e_split, D, stats, labels, c, dx, de, db=db, bias=bt, loss=loss,
                                    temperature=T, oob=oob)
    return stats, loss, dx, de, db


def bounds(x, E, b, y, T, sw, lse):
    """Per-element bounds from the error model of the kernels: each score carries the split-bf16 product's error
    (EPS_SPLIT of sum_d |x_d e_d| / T), which moves G = c (p - onehot) by about c p (ds_bj + ds of the row's lse); the second
    product adds EPS_SPLIT of the sum of |G| |operand|; fp32 sums add their own rounding (folded into the factor 4)."""
    x, E = x.astype(np.float64), E.astype(np.float64)
    B, N = x.shape[0], E.shape[0]
    z = x @ E.T + (0 if b is None else b.astype(np.float64)[None, :])
    z /= T
    p = np.exp(z - lse[:, None])
    ds = EPS_SPLIT * (np.abs(x) @ np.abs(E).T) / T + 2.0 ** -22 * np.abs(z)
    c = (np.ones(B) if sw is None else sw.astype(np.float64)) / B
    dG = c[:, None] * p * (ds + (p * ds).sum(axis=1, keepdims=True))
    ok = (y >= 0) & (y < N)
    onehot = np.zeros((B, N))
    onehot[np.nonzero(ok)[0], y[ok]] = 1.0
    aG = c[:, None] * (p + onehot)
    ex = (dG @ np.abs(E) + EPS_SPLIT * aG @ np.abs(E)) / T
    ee = (dG.T @ np.abs(x) + EPS_SPLIT * aG.T @ np.abs(x)) / T
    eb = (dG.sum(axis=0) + 2.0 ** -22 * aG.sum(axis=0) * np.sqrt(B)) / T
    return 4 * ex + 1e-12, 4 * ee + 1e-12, 4 * eb + 1e-12


CASES = [  # B, N, D, T, bias, weights, label dtype
    (1, 1, 4, 1.0, True, False, torch.int64),
    (127, 127, 60, 0.05, False, True, torch.int32),
    (128, 128, 64, 1.0, True, True, torch.int64),
    (129, 3000, 100, 0.05, True, False, torch.int32),
    (4096 + 37, 128, 128, 1.0, True, True, torch.int64),
    (4096 + 37, 3000, 64, 0.05, False, False, torch.int64),
    (1, 100_003, 128, 1.0, True, True, torch.int32),  # one query tile: the catalog is split over many CTAs
    (129, 100_003, 4, 0.05, True, False, torch.int64),  # two query tiles, split
    (127, 3000, 128, 1.0, False, True, torch.int64),
    (128, 1, 60, 0.05, True, True, torch.int32),
]


@pytest.mark.parametrize("B,N,D,T,use_bias,weights,label_dtype", CASES)
def test_catalog_ce_backward_against_float64(device, B, N, D, T, use_bias, weights, label_dtype):
    rng = np.random.default_rng(B * 7 + N + D)
    x = (rng.standard_normal((B, D)) * (0.3 if T < 1 else 1.0)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.5 / np.sqrt(D / 16)).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32) if use_bias else None
    y = rng.integers(0, N, B).astype(np.int64)
    y[: min(B, 2)] = [0, N - 1][: min(B, 2)]  # labels on the first and last catalog rows
    sw = rng.uniform(0.2, 2.0, B).astype(np.float32) if weights else None
    stats, loss, dx, de, db = run(device, x, E, b, y, T, sw, label_dtype)
    lse = stats[:, 1].double().cpu().numpy()
    rl, rdx, rde, rdb = catalog_ce(x, E, b, y, T, sw)
    ex, ee, eb = bounds(x, E, b, y, T, sw, lse)
    for name, got, ref, bound in (("dx", dx, rdx, ex), ("dE", de, rde, ee)):
        err = np.abs(got.double().cpu().numpy() - ref)
        worst = np.unravel_index(np.argmax(err / bound), err.shape)
        assert np.all(err <= bound), f"{name}: |err| {err[worst]:.3e} > bound {bound[worst]:.3e} at {worst}"
    if use_bias:
        err = np.abs(db.double().cpu().numpy() - rdb)
        assert np.all(err <= eb), f"db: max |err| / bound {np.max(err / eb):.3f}"
    assert abs(loss.item() - rl) <= 1e-5 * max(1.0, abs(rl)) + 3e-4 * max(1.0, 1 / T) * np.sqrt(D / 64)


def test_catalog_ce_backward_repeats_bit_identical(device):
    """Split dq path (one query tile over a 100 003-row catalog) and the dn kernel: no atomics, fixed summation order."""
    rng = np.random.default_rng(11)
    B, N, D = 200, 100_003, 64
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.25).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32)
    y = rng.integers(0, N, B)
    assert ops.catalog_softmax_ce_workspace_bytes(B, N, D) > 0  # the split path
    first = run(device, x, E, b, y, 0.5, None)
    for _ in range(2):
        again = run(device, x, E, b, y, 0.5, None)
        for a, c in zip(first, again):
            assert torch.equal(a, c)


def test_out_of_range_labels_are_never_read_as_addresses(device):
    """A label outside [0, N) matches no column: its row keeps the soft-max term only (the oracle's rule), and each such
    label adds one to the out-of-range counter, once per row whatever the number of catalog splits."""
    rng = np.random.default_rng(12)
    B, N, D = 130, 500, 64
    x = rng.standard_normal((B, D)).astype(np.float32)
    E = (rng.standard_normal((N, D)) * 0.3).astype(np.float32)
    y = rng.integers(0, N, B)
    y[[0, 5, 129]] = [N, -1, 1 << 40]
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    stats, loss, dx, de, db = run(device, x, E, None, y, 1.0, None, oob=oob)
    assert oob.item() == 3
    run(device, x[:1], E, None, y[:1], 1.0, None, oob=oob)  # one query tile, the catalog split over several CTAs
    assert ops.catalog_softmax_ce_workspace_bytes(1, N, D) > 0 and oob.item() == 4
    _, rdx, rde, _ = catalog_ce(x, E, None, y, 1.0)
    ex, ee, _ = bounds(x, E, None, y, 1.0, None, stats[:, 1].double().cpu().numpy())
    assert np.all(np.abs(dx.double().cpu().numpy() - rdx) <= ex)
    assert np.all(np.abs(de.double().cpu().numpy() - rde) <= ee)


def test_catalog_10m_sampled_rows(device):
    """10 M x 64 catalog (BASELINE configs[2]) with B = 4096, the split dq shape: dE and db of sampled catalog rows and dx
    of sampled queries recomputed on the host in float64 over the hash-initialised table, with the kernels' own log-sum-exp
    (mm_catalog_score's statistics, checked at this size by test_gpu_catalog.py).  Each of the 4 splits streams 19 532
    tiles: without the kernels' periodic flush of the wgmma accumulator, dx came out 0.2 % small here."""
    I, D, B = 10_000_000, 64, 4096
    rng = np.random.default_rng(21)
    E = torch.empty((I, D), dtype=torch.float32, device=device)
    ops.init_uniform_hash(E, 77, -0.5, 0.5)
    bias = torch.empty((I, 1), dtype=torch.float32, device=device)
    ops.init_uniform_hash(bias, 78, -0.2, 0.2)
    bias = bias.reshape(-1)
    x = (rng.standard_normal((B, D)) * 0.5).astype(np.float32)
    y = rng.integers(0, I, B).astype(np.int64)
    rows = np.array([0, 1, 127, 128, 5_000_000, I - 1] + list(y[:4]), dtype=np.int64)
    y[4:6] = [0, I - 1]
    assert ops.catalog_softmax_ce_workspace_bytes(B, I, D) > 0
    e_split = ops.split_rows(E)
    labels = dev(y, device)
    stats, _, _ = ops.catalog_score(dev(x, device), e_split, I, bias=bias, targets=labels, k=0)
    c = torch.full((1,), 1.0 / B, device=device)
    dx = torch.empty((B, D), device=device)
    de = torch.empty((I, D), device=device)
    db = torch.empty(I, device=device)
    ops.catalog_softmax_ce_backward(ops.split_rows(dev(x, device)), e_split, D, stats, labels, c, dx, de, db=db, bias=bias)
    lse = stats[:, 1].double().cpu().numpy()
    xd = x.astype(np.float64)
    Er = oracle.hash_table_rows(rows, D, 77, -0.5, 0.5).astype(np.float64)
    br = bias[torch.from_numpy(rows).to(device)].double().cpu().numpy()
    G = (np.exp(xd @ Er.T + br[None, :] - lse[:, None]) - (y[:, None] == rows[None, :])) / B  # (B, rows)
    # bounds: 1e-3 of the sum of |terms| (the split products' and the exp's relative error is ~1e-4 at these magnitudes)
    ridx = torch.from_numpy(rows).to(device)
    err = np.abs(de[ridx].double().cpu().numpy() - G.T @ xd)
    assert np.all(err <= 1e-3 * (np.abs(G).T @ np.abs(xd)) + 1e-12)
    err = np.abs(db[ridx].double().cpu().numpy() - G.sum(axis=0))
    assert np.all(err <= 1e-3 * np.abs(G).sum(axis=0) + 1e-12)
    qs = [0, 1, 4, 5, 2047, 4095]
    acc = np.zeros((len(qs), D))
    bias_h = bias.double().cpu().numpy()
    step = 1_000_000
    for r0 in range(0, I, step):
        r = np.arange(r0, min(I, r0 + step))
        blk = oracle.hash_table_rows(r, D, 77, -0.5, 0.5).astype(np.float64)
        p = np.exp(xd[qs] @ blk.T + bias_h[r][None, :] - lse[qs][:, None])
        acc += p @ blk
    acc -= oracle.hash_table_rows(y[qs], D, 77, -0.5, 0.5).astype(np.float64)
    np.testing.assert_allclose(dx[qs].double().cpu().numpy(), acc / B, rtol=0, atol=2e-7)
