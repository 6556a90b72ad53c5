"""mm_dlrm_lookup_interact (csrc/interaction_v2.cu) against the oracle: per-table id widths (1/2/3/4/8 bytes),
every supported (F, D), fp32 and split-bf16 outputs, out-of-range ids, and the row-sharded placement
(owner = id % world, local row = id // world) — exercised on ONE GPU by handing the kernel the `world`
shards as "peer" pointers that happen to live in the same HBM (the address arithmetic is what is tested;
tests/dist_sharded_check.py runs the same launch over real NVLink peers)."""
import numpy as np
import pytest
import torch

from models_b200 import ops
from oracle import oracle

pytestmark = pytest.mark.gpu


def dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def pack_ids(idx: np.ndarray, width: int) -> np.ndarray:
    if width == 1:
        return idx.astype(np.uint8)
    if width == 2:
        return idx.astype(np.uint16)
    if width == 3:
        return idx.astype("<u4").view(np.uint8).reshape(-1, 4)[:, :3].copy()
    return idx.astype(np.int32 if width == 4 else np.int64)


def reference(tables, idx, rows, slots, bottom, bslot, F, D):
    B = len(idx[0])
    stack = np.zeros((B, F, D), dtype=np.float32)
    for t in range(len(tables)):
        ok = (idx[t] >= 0) & (idx[t] < rows[t])
        stack[ok, slots[t]] = tables[t][idx[t][ok]]
    if bottom is not None:
        stack[:, bslot] = bottom
    inter = oracle.dot_interaction(stack)
    return inter if bottom is None else np.concatenate([bottom, inter], axis=1)


def unsplit(out, W):
    Kp = out.shape[1] // 2
    o = out.float().cpu().numpy()
    assert not o[:, W:Kp].any() and not o[:, Kp + W:].any(), "padding columns must be zero"
    return o[:, :W] + o[:, Kp:Kp + W]


@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("T,with_bottom", [(26, True), (1, True), (31, True), (32, False), (7, False), (12, True)])
def test_lookup_interact_shapes(device, D, T, with_bottom):
    rng = np.random.default_rng(100 + D + T)
    B = 777
    F = T + (1 if with_bottom else 0)
    rows = rng.integers(3, 4000, T)
    tables = [rng.standard_normal((int(r), D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, int(r), B).astype(np.int64) for r in rows]
    perm = rng.permutation(F).tolist()
    slots, bslot = perm[:T], (perm[T] if with_bottom else -1)
    bottom = rng.standard_normal((B, D)).astype(np.float32) if with_bottom else None
    W = (D if with_bottom else 0) + F * (F - 1) // 2
    out = torch.empty((B, W), dtype=torch.float32, device=device)
    ops.dlrm_lookup_interact([dev(t, device) for t in tables], [dev(i.astype(np.int32), device) for i in idx], slots,
                             [int(r) for r in rows], D, None if bottom is None else dev(bottom, device), bslot, out)
    ref = reference(tables, idx, rows, slots, bottom, bslot, F, D)
    got = out.cpu().numpy()
    if with_bottom:
        assert np.array_equal(got[:, :D], bottom)  # the prefix is a pure copy
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-4 * np.sqrt(D / 16))


@pytest.mark.parametrize("as_split", [False, True])
def test_lookup_interact_packed_id_widths_are_bit_identical_to_int32(device, as_split):
    rng = np.random.default_rng(7)
    B, D = 4099, 64
    # the bundled Criteo shape: 8 tables <= 2^8 rows, 10 <= 2^16, 8 <= 2^24 (capped here to keep the test small)
    rows = [4, 62, 11, 72, 5, 15, 96, 256] + [29428, 15128, 7296, 19902, 6466, 1311, 2210, 9780, 964, 65536] + [300000] * 4 + [70000] * 4
    widths = [1] * 8 + [2] * 10 + [3] * 4 + [4, 8, 3, 4]
    T = len(rows)
    F = T + 1
    tables = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(np.int64) for r in rows]
    idx[7][5] = 255
    idx[17][9] = 65535  # extreme values of the narrow widths
    bottom = rng.standard_normal((B, D)).astype(np.float32)
    slots = list(range(T))
    W = D + F * (F - 1) // 2
    tw = [dev(t, device) for t in tables]

    def run(id_arrays):
        if as_split:
            out = torch.empty((B, 2 * ops.tc_padded_k(W)), dtype=torch.bfloat16, device=device)
        else:
            out = torch.empty((B, W), dtype=torch.float32, device=device)
        oob = torch.zeros(1, dtype=torch.int32, device=device)
        ops.dlrm_lookup_interact(tw, id_arrays, slots, rows, D, dev(bottom, device), T, out, oob)
        assert int(oob.item()) == 0
        return out

    # packed arrays sit at odd byte offsets inside one buffer (as in a packed host batch they need no alignment)
    blob = torch.zeros(sum(B * w for w in widths) + 64, dtype=torch.uint8, device=device)
    packed, off = [], 1
    for i, w in zip(idx, widths):
        a = pack_ids(i, w)
        if w in (4, 8):
            packed.append(dev(a, device))
            continue
        raw = torch.from_numpy(a.view(np.uint8).reshape(-1)).to(device)
        if w == 2:
            off += off & 1  # torch views of uint16 need 2-byte alignment
        blob[off: off + raw.numel()] = raw
        v = blob[off: off + raw.numel()]
        packed.append(v.view(torch.uint16) if w == 2 else v.view(B, 3) if w == 3 else v)
        off += raw.numel() + 1
    a = run(packed)
    b = run([dev(i.astype(np.int32), device) for i in idx])
    assert torch.equal(a, b)
    ref = reference(tables, idx, rows, slots, bottom, T, F, D)
    got = unsplit(a, W) if as_split else a.cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=2e-4, atol=4e-4)


def test_lookup_interact_out_of_range_narrow_ids(device):
    rng = np.random.default_rng(8)
    B, D, T = 300, 64, 5
    rows = [200, 3000, 100000, 17, 50]
    widths = [1, 2, 3, 4, 8]
    tables = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(np.int64) for r in rows]
    idx[0][3] = 250      # fits a byte, not the table
    idx[1][4] = 65535
    idx[2][5] = (1 << 24) - 1
    idx[3][6] = -1
    idx[4][7] = 1 << 40
    out = torch.empty((B, T * (T - 1) // 2), dtype=torch.float32, device=device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    ops.dlrm_lookup_interact([dev(t, device) for t in tables], [dev(pack_ids(i, w), device) for i, w in zip(idx, widths)],
                             list(range(T)), rows, D, None, -1, out, oob)
    assert int(oob.item()) == 5
    ref = reference(tables, idx, rows, list(range(T)), None, -1, T, D)
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-4, atol=4e-4)


@pytest.mark.parametrize("idx_dtype", [np.int32, np.int64])
def test_lookup_interact_wide_ids_match_oracle(device, idx_dtype):
    """4- and 8-byte ids, permuted slots and a bottom vector: the prefix is a pure copy and the interactions
    match the oracle."""
    rng = np.random.default_rng(9)
    B, T, D = 515, 26, 64
    rows = [int(r) for r in rng.integers(3, 5000, T)]
    tables = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(idx_dtype) for r in rows]
    bottom = rng.standard_normal((B, D)).astype(np.float32)
    slots = rng.permutation(T + 1).tolist()
    bslot, tslots = slots[-1], slots[:-1]
    F = T + 1
    out = torch.empty((B, D + F * (F - 1) // 2), dtype=torch.float32, device=device)
    ops.dlrm_lookup_interact([dev(t, device) for t in tables], [dev(i, device) for i in idx], tslots, rows, D,
                             dev(bottom, device), bslot, out)
    got = out.cpu().numpy()
    assert np.array_equal(got[:, :D], bottom)
    ref = reference(tables, idx, rows, tslots, bottom, bslot, F, D)
    np.testing.assert_allclose(got[:, D:], ref[:, D:], rtol=1e-4, atol=2e-4)


def test_lookup_interact_split_output_and_out_of_range_wide_ids(device):
    """4-byte ids below 0 and at or above `rows` read zero rows and are counted; split-bf16 output."""
    rng = np.random.default_rng(21)
    B, T, D = 3000, 26, 64
    rows = [int(r) for r in rng.integers(3, 5000, T)]
    tables = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(np.int32) for r in rows]
    idx[3][7] = rows[3] + 5
    idx[9][11] = -2
    bottom = rng.standard_normal((B, D)).astype(np.float32)
    F = T + 1
    W = D + F * (F - 1) // 2
    out = torch.empty((B, 2 * ops.tc_padded_k(W)), dtype=torch.bfloat16, device=device)
    oob = torch.zeros(1, dtype=torch.int32, device=device)
    ops.dlrm_lookup_interact([dev(t, device) for t in tables], [dev(i, device) for i in idx], list(range(T)), rows, D,
                             dev(bottom, device), T, out, oob)
    assert int(oob.item()) == 2
    ref = reference(tables, idx, rows, list(range(T)), bottom, T, F, D)
    np.testing.assert_allclose(unsplit(out, W), ref, rtol=2e-4, atol=2e-4)


def test_lookup_interact_rejects_bad_descriptors(device):
    t = torch.zeros((300, 64), device=device)
    out = torch.empty((4, 1), dtype=torch.float32, device=device)
    with pytest.raises(ValueError, match="do not fit"):
        ops.dlrm_lookup_interact([t, t], [torch.zeros(4, dtype=torch.uint8, device=device)] * 2, [0, 1], [300, 300], 64, None, -1, out)
    with pytest.raises(ValueError, match="slot 0 used twice"):
        ops.dlrm_lookup_interact([t, t], [torch.zeros(4, dtype=torch.int32, device=device)] * 2, [0, 0], [300, 300], 64, None, -1, out)
    with pytest.raises(TypeError):
        ops.dlrm_lookup_interact([t, t], [torch.zeros(4, dtype=torch.float32, device=device)] * 2, [0, 1], [300, 300], 64, None, -1, out)


@pytest.mark.parametrize("world", [2, 4, 8, 3])
def test_lookup_interact_sharded_address_arithmetic(device, world):
    """Row r of a sharded table lives on rank r % world at local row r // world.  All `world` shards live on
    this GPU and are handed over as the peer pointers; small tables stay replicated (mixed placement)."""
    rng = np.random.default_rng(50 + world)
    B, D, T = 2053, 64, 26
    rows = [int(r) for r in rng.integers(1, 6000, T)]
    rows[0], rows[1] = 1, world  # degenerate shards: some ranks own no row / exactly one row
    tables = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    idx = [rng.integers(0, r, B).astype(np.int64) for r in rows]
    idx[5][:] = idx[5][0]  # skew: one owner serves every sample
    bottom = rng.standard_normal((B, D)).astype(np.float32)
    F = T + 1
    W = D + F * (F - 1) // 2
    full = [dev(t, device) for t in tables]
    ids = [dev(i.astype(np.int32), device) for i in idx]
    want = torch.empty((B, W), dtype=torch.float32, device=device)
    ops.dlrm_lookup_interact(full, ids, list(range(T)), rows, D, dev(bottom, device), T, want)
    for rank in (0, world - 1):
        weights, peers = [], []
        for t in range(T):
            if t % 5 == 4:  # replicated
                weights.append(full[t])
                peers.append(None)
                continue
            shards = [torch.cat([full[t][k::world], torch.zeros((1, D), device=device)]).contiguous() for k in range(world)]
            weights.append(shards[rank])
            peers.append([s.data_ptr() for s in shards])
            weights[-1]._keep = shards
        got = torch.empty((B, W), dtype=torch.float32, device=device)
        oob = torch.zeros(1, dtype=torch.int32, device=device)
        ops.dlrm_lookup_interact(weights, ids, list(range(T)), rows, D, dev(bottom, device), T, got, oob, peers=peers,
                                 rank=rank, world=world)
        assert int(oob.item()) == 0
        assert torch.equal(got, want)


def test_dlrm_model_accepts_packed_host_batch(device):
    """Model.id_bytes() + HostBatch packing: the compiled forward on a packed batch equals the int32 one."""
    import models_b200 as mm
    from models_b200 import datasets

    mm.set_seed(5)
    schema = datasets.criteo_schema({k: min(v, 70000) for k, v in datasets.CRITEO_MAX.items()})
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]))
    model.build(device)
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 1024, seed=3, index_law="uniform", index_dtype=np.int32))
    widths = model.id_bytes()
    assert sorted(set(widths.values())) == [1, 2, 3] and len(widths) == 26
    plain = mm.HostBatch.like(feats, model.input_columns())
    packed = mm.HostBatch.like(feats, model.input_columns(), id_bytes=widths)
    assert packed.payload_bytes() < plain.payload_bytes() - 1024 * 40
    a = model.compile(plain)(plain).clone()
    b = model.compile(packed)(packed).clone()
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="cannot travel"):
        bad = dict(feats)
        bad["C6"] = feats["C6"].copy()
        bad["C6"][0] = 300
        packed.fill(bad)


@pytest.mark.parametrize("T,with_perm", [(26, False), (26, True), (31, True), (1, False), (12, True)])
def test_operand_format_rows_match_fp32_rows(device, T, with_perm):
    """MM_ROWS_OPERAND: tables and bottom as bf16 split rows [hi | lo] (ops.split_rows), fragments by ldmatrix.  Same
    products as the fp32-row kernel; the k order inside an MMA differs, so equality holds to fp32 rounding."""
    D = 64
    rng = np.random.default_rng(D + T)
    B = 1531
    F = T + 1
    rows = [int(r) for r in rng.integers(3, 3000, T)]
    tn = [rng.standard_normal((r, D)).astype(np.float32) for r in rows]
    tables = [dev(t, device) for t in tn]
    idn = [rng.integers(0, r, B).astype(np.int64) for r in rows]
    idn[0][7] = rows[0] + 3  # out of range -> zero row in both formats
    idx = [dev(i.astype(np.int32), device) for i in idn]
    bn = rng.standard_normal((B, D)).astype(np.float32)
    bottom = dev(bn, device)
    perm = rng.permutation(F).tolist() if with_perm else list(range(F))
    W = D + F * (F - 1) // 2
    a = torch.empty((B, 2 * ops.tc_padded_k(W)), dtype=torch.bfloat16, device=device)
    b = torch.empty_like(a)
    oa, ob = torch.zeros(1, dtype=torch.int32, device=device), torch.zeros(1, dtype=torch.int32, device=device)
    ops.dlrm_lookup_interact(tables, idx, perm[:T], rows, D, bottom, perm[T], a, oa)
    ops.dlrm_lookup_interact([ops.split_rows(t) for t in tables], idx, perm[:T], rows, D, ops.split_rows(bottom), perm[T], b, ob,
                             operand_rows=True)
    assert int(oa.item()) == int(ob.item()) == 1
    ua, ub = unsplit(a, W), unsplit(b, W)
    assert np.array_equal(ua[:, :D], ub[:, :D])  # the prefix is the same hi/lo pair either way
    np.testing.assert_allclose(ub, ua, rtol=1e-5, atol=1e-5)
    ref = reference(tn, idn, rows, perm[:T], bn, perm[T], F, D)
    np.testing.assert_allclose(ub, ref, rtol=2e-4, atol=4e-4)
    with pytest.raises(ValueError, match="operand-format rows need the split-bf16 output"):
        ops.dlrm_lookup_interact([ops.split_rows(t) for t in tables], idx, perm[:T], rows, D, ops.split_rows(bottom), perm[T],
                                 torch.empty((B, W), device=device), operand_rows=True)


def test_tower_kernel_operand_output_equals_split_of_fp32_output(device):
    rng = np.random.default_rng(3)
    M, K, widths = 1000, 13, [128, 64]
    x = dev(rng.standard_normal((M, K)).astype(np.float32), device)
    Ws = [dev((rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32), device) for k, n in zip([K] + widths[:-1], widths)]
    bs = [dev(rng.standard_normal(n).astype(np.float32) * 0.1, device) for n in widths]
    a = ops.split_rows(x)
    ws = [ops.split_weights(w) for w in Ws]
    out = torch.empty((M, 64), device=device)
    op = torch.empty((M, 128), dtype=torch.bfloat16, device=device)
    ops.mlp_tc(a, K, ws, widths, bs, ["relu", "relu"], out=out)
    ops.mlp_tc(a, K, ws, widths, bs, ["relu", "relu"], out_operand=op)
    assert torch.equal(ops.split_rows(out).view(torch.int16), op.view(torch.int16))
    both_f, both_o = torch.empty_like(out), torch.empty_like(op)
    ops.mlp_tc(a, K, ws, widths, bs, ["relu", "relu"], out=both_f, out_operand=both_o)
    assert torch.equal(both_f, out) and torch.equal(both_o.view(torch.int16), op.view(torch.int16))


def test_dlrm_model_table_mirror_on_off_agree(device):
    import models_b200 as mm
    from models_b200 import blocks, datasets

    mm.set_seed(12)
    schema = datasets.criteo_schema({k: min(v, 9000) for k, v in datasets.CRITEO_MAX.items()})
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]), top_block=mm.MLPBlock([128, 64, 32]))
    model.build(device)
    feats, _ = datasets.split_targets(schema, datasets.generate_batch(schema, 2048, seed=5, index_law="uniform", index_dtype=np.int32))
    batch = {k: dev(v, device) for k, v in feats.items()}
    try:
        blocks.set_table_mirror(False)
        assert not model.body.use_operand_rows()
        ref = model(batch).clone()
        blocks.set_table_mirror(True)
        assert model.body.use_operand_rows()
        got = model(batch)
        close = lambda x, y: torch.allclose(x, y, rtol=1e-5, atol=1e-6)  # same products, different k order inside the MMAs
        assert close(ref, got)
        hb = mm.HostBatch.like(feats, model.input_columns(), id_bytes=model.id_bytes())
        cf = model.compile(hb)
        assert torch.equal(cf(hb).to(device), got)
        # a table reassigned after the capture: the mirror is refreshed in place and the graph re-captured
        t = model.body.embeddings.tables["C2"]
        t.table.mul_(0.5)
        t._weights_changed()
        blocks.set_table_mirror(False)
        ref2 = model(batch).clone()
        blocks.set_table_mirror(True)
        assert not close(ref2, ref) and close(cf(hb).to(device), ref2)
    finally:
        blocks.set_table_mirror(None)
