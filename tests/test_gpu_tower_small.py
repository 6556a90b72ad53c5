"""mm_tower2_small, the narrow-input two-layer tower kernel (the DLRM bottom tower): the all-fp32 and the mixed-dtype
instantiations agree bit for bit, the split output is the split of the fp32 output, no row at or past B is written, and
every (N1, N2) shape matches a float64 restatement of the 3-pass split arithmetic."""
import numpy as np
import pytest
import torch

from models_b200 import ops

pytestmark = pytest.mark.gpu

SHAPES = [(128, 64), (128, 32), (128, 16), (64, 64), (64, 32), (64, 16), (32, 64), (32, 32), (32, 16)]
ACTS = {"relu": lambda v: np.maximum(v, 0.0), "linear": lambda v: v, "tanh": np.tanh,
        "sigmoid": lambda v: 1.0 / (1.0 + np.exp(-v))}


def _bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(torch.bfloat16).to(torch.float64).numpy()


def _split_dot(x, W):
    """x (M, K) . W (K, N) as the kernels compute it: hi*lo + lo*hi + hi*hi of the bf16 splits, summed in float64."""
    xh = _bf16(x)
    xl = _bf16(x.astype(np.float64) - xh)
    wh = _bf16(W)
    wl = _bf16(W.astype(np.float64) - wh)
    return xh @ wl + xl @ wh + xh @ wh


def _restated(x, W1, b1, act1, W2, b2, act2):
    h = ACTS[act1](_split_dot(x, W1) + b1).astype(np.float32)
    return ACTS[act2](_split_dot(h, W2) + b2)


def _tower(rng, K, N1, N2, device):
    # glorot-scaled, as the Dense layers initialise them
    W1 = (rng.standard_normal((K, N1)) * np.sqrt(2.0 / (K + N1))).astype(np.float32)
    b1 = (rng.standard_normal(N1) * 0.1).astype(np.float32)
    W2 = (rng.standard_normal((N1, N2)) * np.sqrt(2.0 / (N1 + N2))).astype(np.float32)
    b2 = (rng.standard_normal(N2) * 0.1).astype(np.float32)
    d = {n: torch.from_numpy(v).to(device) for n, v in dict(W1=W1, b1=b1, W2=W2, b2=b2).items()}
    return (W1, b1, W2, b2), (ops.split_weights(d["W1"]), d["b1"], ops.split_weights(d["W2"]), d["b2"])


def _columns(rng, B, K, mixed):
    """K input columns as (B,) / (B, 1) / (B, 2) pieces; mixed: int32, int64, fp64 pieces besides fp32 ones."""
    pieces, k = [], 0
    while k < K:
        if k == 2 and K - k >= 2:
            pieces.append(rng.standard_normal((B, 2)).astype(np.float32))
            k += 2
            continue
        kind = k % 4 if mixed else 0
        if kind == 1:
            pieces.append(rng.integers(-3, 4, B).astype(np.int64))
        elif kind == 2:
            pieces.append(rng.integers(-3, 4, (B, 1)).astype(np.int32))
        elif kind == 3:
            pieces.append(rng.standard_normal((B, 1)).astype(np.float64))
        else:
            pieces.append(rng.standard_normal(B).astype(np.float32))
        k += 1
    x = np.concatenate([p.reshape(B, -1).astype(np.float32) for p in pieces], axis=1)
    return pieces, x


def _run(pieces, dev_w, N1, N2, acts, out=None, out_split=None):
    w1, b1, w2, b2 = dev_w
    ops.tower2_small(pieces, w1, N1, b1, acts[0], w2, N2, b2, acts[1], out=out, out_split=out_split)
    torch.cuda.synchronize()


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


@pytest.mark.parametrize("acts", [("relu", "relu"), ("tanh", "sigmoid")])
def test_fp32_path_and_general_path_are_bit_identical(device, acts):
    rng = np.random.default_rng(5)
    B, K, N1, N2 = 4099, 13, 128, 64
    _, dev_w = _tower(rng, K, N1, N2, device)
    x = rng.standard_normal((B, K)).astype(np.float32)
    as_f32 = [torch.from_numpy(np.ascontiguousarray(x[:, k])).to(device) for k in range(K)]
    as_f64 = [t.double() for t in as_f32]  # the same values through the per-column dtype conversion
    mixed = [as_f32[k] if k % 2 else as_f64[k] for k in range(K)]
    res = []
    for pieces in (as_f32, as_f64, mixed):
        out = torch.empty((B, N2), dtype=torch.float32, device=device)
        spl = torch.empty((B, 2 * N2), dtype=torch.bfloat16, device=device)
        _run(pieces, dev_w, N1, N2, acts, out=out, out_split=spl)
        res.append((out, spl))
    for out, spl in res[1:]:
        assert torch.equal(_bits(out), _bits(res[0][0]))
        assert torch.equal(_bits(spl), _bits(res[0][1]))


@pytest.mark.parametrize("N1,N2", [(128, 64), (64, 32), (32, 16)])
def test_split_output_is_the_split_of_the_fp32_output(device, N1, N2):
    rng = np.random.default_rng(N1 + N2)
    B, K = 1037, 13
    _, dev_w = _tower(rng, K, N1, N2, device)
    pieces, _ = _columns(rng, B, K, mixed=False)
    pieces = [torch.from_numpy(p).to(device) for p in pieces]
    out = torch.empty((B, N2), dtype=torch.float32, device=device)
    spl = torch.empty((B, 2 * N2), dtype=torch.bfloat16, device=device)
    _run(pieces, dev_w, N1, N2, ("relu", "relu"), out=out, out_split=spl)
    ref = ops.split_rows(out)
    Kp = ref.shape[1] // 2
    assert torch.equal(_bits(spl[:, :N2]), _bits(ref[:, :N2]))
    assert torch.equal(_bits(spl[:, N2:]), _bits(ref[:, Kp:Kp + N2]))
    # the split output alone is the same as with both outputs requested
    alone = torch.empty_like(spl)
    _run(pieces, dev_w, N1, N2, ("relu", "relu"), out_split=alone)
    assert torch.equal(_bits(alone), _bits(spl))


@pytest.mark.parametrize("B", [1, 15, 16, 17, 4095, 65539])
@pytest.mark.parametrize("aligned", [True, False])
def test_batch_sizes_write_no_row_past_B(device, B, aligned):
    """Rows at or past B stay untouched; aligned=False takes the narrow-store paths (an out_split that is only 4-byte
    aligned, an fp32 row stride that is not a multiple of 4)."""
    rng = np.random.default_rng(B)
    K, N1, N2 = 13, 128, 64
    host_w, dev_w = _tower(rng, K, N1, N2, device)
    pieces, x = _columns(rng, B, K, mixed=False)
    pieces = [torch.from_numpy(p).to(device) for p in pieces]
    guard = 24
    pitch = N2 + 4 if aligned else N2 + 2
    fbuf = torch.full((B + guard, pitch), 7.0, dtype=torch.float32, device=device)
    out = fbuf[:B, :N2]
    off = 0 if aligned else 2
    sflat = torch.full(((B + guard) * 2 * N2 + off,), -3.0, dtype=torch.bfloat16, device=device)
    spl = sflat[off: off + B * 2 * N2].view(B, 2 * N2)
    _run(pieces, dev_w, N1, N2, ("relu", "relu"), out=out, out_split=spl)
    assert bool((fbuf[B:] == 7.0).all()) and bool((fbuf[:B, N2:] == 7.0).all())
    assert bool((sflat[:off] == -3.0).all()) and bool((sflat[off + B * 2 * N2:] == -3.0).all())
    ref = _restated(x, *host_w[:2], "relu", *host_w[2:], "relu")
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-4, atol=2e-5)
    ref_split = ops.split_rows(out.contiguous())
    Kp = ref_split.shape[1] // 2
    assert torch.equal(_bits(spl[:, :N2]), _bits(ref_split[:, :N2]))
    assert torch.equal(_bits(spl[:, N2:]), _bits(ref_split[:, Kp:Kp + N2]))


@pytest.mark.parametrize("N1,N2", SHAPES)
@pytest.mark.parametrize("acts,mixed", [(("relu", "relu"), False), (("relu", "relu"), True), (("tanh", "sigmoid"), False),
                                        (("linear", "tanh"), True)])
def test_every_shape_matches_the_split_arithmetic(device, N1, N2, acts, mixed):
    rng = np.random.default_rng(N1 * 7 + N2)
    B, K = 1001, 11 if mixed else 13
    host_w, dev_w = _tower(rng, K, N1, N2, device)
    pieces, x = _columns(rng, B, K, mixed)
    pieces = [torch.from_numpy(p).to(device) for p in pieces]
    out = torch.empty((B, N2), dtype=torch.float32, device=device)
    spl = torch.empty((B, 2 * N2), dtype=torch.bfloat16, device=device)
    _run(pieces, dev_w, N1, N2, acts, out=out, out_split=spl)
    ref = _restated(x, host_w[0], host_w[1], acts[0], host_w[2], host_w[3], acts[1])
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-4, atol=2e-5)
    rec = spl.float().cpu().numpy()
    np.testing.assert_allclose(rec[:, :N2] + rec[:, N2:], out.cpu().numpy(), rtol=2e-5, atol=1e-6)
