"""TEST INFRASTRUCTURE - numpy restatement of Philox4x32-10 (Salmon et al., SC'11; the Random123 library) and of
the dropout-mask convention of youku-mplug_b200/csrc/philox.cuh, so that the CPU oracle can run the decoder WITH
dropout and be compared against the H100 kernels element for element.

Pinned by the published known-answer vectors of Random123 (kat_vectors: philox4x32-10), checked in
tests/test_oracle_golden.py.  Only tests / oracle code may import this module."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised over numpy uint32 arrays (broadcast); returns 4 uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & MASK for c in (c0, c1, c2, c3))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK
        n0 = hi1 ^ c1 ^ np.uint64(k0)
        n2 = hi0 ^ c3 ^ np.uint64(k1)
        c0, c1, c2, c3 = n0, lo1, n2, lo0
        k0 = (k0 + W0) & 0xFFFFFFFF
        k1 = (k1 + W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def threshold(p):
    """The keep threshold of drop_state (philox.cuh): the kernels receive p as an fp32, so floor(fl32(p) * 2^32)
    (exact in double), saturating at 0xFFFFFFFF.  At p = 0.1 this is 429496736, not the 429496729 of the double p."""
    t = float(np.float32(p)) * 4294967296.0
    return 0xFFFFFFFF if t >= 4294967295.0 else int(t)


def scale(p):
    """The kept-value multiplier of drop_state: 1.0f / (1.0f - fl32(p)), every step in fp32."""
    one = np.float32(1.0)
    return float(one / (one - np.float32(p)))


def words(seed, offset, site, rows, cols):
    """uint32 [len(rows), cols]: the Philox word of every (row, column), counter = (col >> 2, row, site, offset),
    key = seed, word col & 3 of the four."""
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1, 1)
    c4 = (np.arange((cols + 3) // 4, dtype=np.uint64)).reshape(1, -1)
    w = philox4x32_10(np.broadcast_to(c4, (rows.shape[0], c4.shape[1])), np.broadcast_to(rows, (rows.shape[0], c4.shape[1])),
                      np.uint64(site), np.uint64(int(offset) & 0xFFFFFFFF), int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF)
    return np.stack(w, axis=-1).reshape(rows.shape[0], -1)[:, :cols]


def keep_mask(seed, offset, site, rows, cols, p):
    """Boolean keep-mask [len(rows), cols] for logical rows `rows` (1-D integer array) and columns 0..cols-1:
    keep iff word(row, col) >= threshold(p)."""
    return words(seed, offset, site, rows, cols) >= np.uint32(threshold(p))


def dropout(x, seed, offset, site, p, rows=None):
    """torch tensor [R, C] -> dropout(x) with the kernels' mask and scale; rows default to 0..R-1."""
    import torch
    if p <= 0.0:
        return x
    R, C = x.shape
    m = keep_mask(seed, offset, site, np.arange(R) if rows is None else rows, C, p)
    return x * torch.from_numpy(m).to(x.dtype) * scale(p)
