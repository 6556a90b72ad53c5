"""mm_mlp_tc at the tile-count edges of its ping-pong schedule: the two consumer warpgroups of a CTA take alternate
64-row tiles, so batches of fewer than 64 rows, a ragged last tile, and CTAs with an odd or an even number of tiles
(the last tile has no partner) must all give the same rows as the layer-by-layer mm_dense_tc chain, leave the rows
past M untouched, and give every fused head exactly what a single-head launch gives."""
import pytest
import torch

from models_b200 import ops

pytestmark = pytest.mark.gpu

TILE = 64
SIZES = [1, 63, 64, 65, 127, 128 * 132 - 64, 128 * 132 + 64, 65536, 65573]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles_per_cta(M):
    tiles = -(-M // TILE)
    grid = min(tiles, _sms())
    return {tiles // grid + (1 if c < tiles % grid else 0) for c in range(grid)}


def test_sizes_cover_odd_and_even_tile_counts(device):
    counts = set().union(*(_tiles_per_cta(M) for M in SIZES))
    assert any(c % 2 for c in counts) and any(c % 2 == 0 for c in counts) and any(c % 2 and c > 1 for c in counts)


def _tower(device, M, K=415, widths=(128, 64, 32)):
    g = torch.Generator(device="cpu").manual_seed(M)
    x = (torch.randn((M, K), generator=g) * 0.5).to(device)
    ws, bs, k = [], [], K
    for n in widths:
        W = (torch.randn((k, n), generator=g) / k ** 0.5).to(device)
        ws.append(ops.split_weights(W))
        bs.append((torch.randn(n, generator=g) * 0.1).to(device))
        k = n
    return ops.split_rows(x), K, list(widths), ws, bs


def _layer_by_layer(a, K, widths, ws, bs):
    M = a.shape[0]
    cur, k = a, K
    for i, n in enumerate(widths):
        last = i == len(widths) - 1
        nxt = None if last else torch.zeros((M, 2 * ops.tc_padded_k(n)), dtype=torch.bfloat16, device=a.device)
        o = torch.empty((M, n), dtype=torch.float32, device=a.device) if last else None
        ops.dense_tc(cur, k, ws[i], n, bs[i], "relu", passes=3, out_f32=o, out_split=nxt)
        cur, k = nxt, n
    return o


@pytest.mark.parametrize("M", SIZES)
def test_mlp_tc_tile_edges_match_layer_by_layer(device, M):
    a, K, widths, ws, bs = _tower(device, M)
    acts = ["relu"] * 3
    g = torch.Generator(device="cpu").manual_seed(M + 1)
    hw = (torch.randn((widths[-1], 3), generator=g) * 0.2).to(device)
    hb = (torch.randn(3, generator=g) * 0.1).to(device)
    body_buf = torch.full((M + TILE, widths[-1]), 7.0, dtype=torch.float32, device=device)
    head_buf = torch.full((M + TILE, 1), 7.0, dtype=torch.float32, device=device)
    body, head = body_buf[:M], head_buf[:M]
    ops.mlp_tc(a, K, ws, widths, bs, acts, out=body, head_w=hw[:, 0].contiguous(), head_b=float(hb[0]), head_act="sigmoid",
               head_out=head)
    ref = _layer_by_layer(a, K, widths, ws, bs)
    # same operands, different accumulation order of the three passes: a few fp32 ulps per layer
    diff = float((body - ref).abs().max())
    assert diff < 2e-5, diff
    assert float(body_buf[M:].min()) == 7.0 and float(body_buf[M:].max()) == 7.0
    assert float(head_buf[M:].min()) == 7.0 and float(head_buf[M:].max()) == 7.0
    want = torch.sigmoid(ref.double() @ hw[:, 0].double() + float(hb[0])).float()
    assert float((head[:, 0] - want).abs().max()) < 1e-4
    again = torch.empty_like(head)
    ops.mlp_tc(a, K, ws, widths, bs, acts, head_w=hw[:, 0].contiguous(), head_b=float(hb[0]), head_act="sigmoid", head_out=again)
    assert torch.equal(again, head)  # deterministic, and the same with or without the fp32 rows

    # multi-head instantiation: head h is bit for bit the single-head launch with that head's weights and bias
    heads_act = ["sigmoid", "linear", "relu"]
    multi = torch.empty((3, M), dtype=torch.float32, device=device)
    ops.mlp_tc_heads(a, K, ws, widths, bs, acts, hw, hb, heads_act, multi)
    for h, act in enumerate(heads_act):
        one = torch.empty((M, 1), dtype=torch.float32, device=device)
        ops.mlp_tc(a, K, ws, widths, bs, acts, head_w=hw[:, h].contiguous(), head_b=float(hb[h]), head_act=act, head_out=one)
        assert torch.equal(multi[h], one[:, 0]), h
