"""Numpy port of the training-mode dropout mask (models_b200/csrc/dropout.cuh): Philox4x32-10 of the counter
(col, row, layer, step) under the key (seed & 0xffffffff, seed >> 32); an element is kept when word 0 of the output is
at least round(rate * 2^32)."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """The four output words (uint32 arrays, broadcast over the inputs)."""
    c = [np.asarray(x, dtype=np.uint64) & _LO for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _LO]
        k0, k1 = (k0 + np.uint64(W0)) & _LO, (k1 + np.uint64(W1)) & _LO
    return [x.astype(np.uint32) for x in c]


def threshold(rate: float) -> int:
    t = int(np.floor(float(rate) * 4294967296.0 + 0.5))
    return min(t, 0xFFFFFFFF)


def keep_mask(rows: int, cols: int, rate: float, seed: int, step: int, layer: int) -> np.ndarray:
    """(rows, cols) bool: the elements the layer keeps at this step."""
    r, c = np.meshgrid(np.arange(rows, dtype=np.uint64), np.arange(cols, dtype=np.uint64), indexing="ij")
    seed = int(seed) & (2**64 - 1)
    w0 = philox4x32_10(c, r, layer, step, seed & 0xFFFFFFFF, seed >> 32)[0]
    return w0 >= np.uint32(threshold(rate))
