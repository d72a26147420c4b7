"""Random seq2sdbg sort items and a NumPy reference of their sort order (shared by the CPU and GPU sort tests)."""
import numpy as np

from megahit_b200 import lib


def make_items(rng, n: int, k: int, buckets=None, pool: int = 0) -> np.ndarray:
    """n valid seq2sdbg items ((n, W) uint32): 2k random key bits from the top of word 0, zero fill, flags (bit 19
    non-dollar, bits 16-18 prev in 0..4) and a random 65535 - multiplicity.  buckets: the 16-bit bucket of every item is
    drawn from this list.  pool > 0: the key bits and flags are drawn from `pool` distinct values (equal keys)."""
    W = lib.s2s_record_words(k)
    m = max(1, pool) if pool else n
    bits = rng.integers(0, 1 << 32, size=(m, W), dtype=np.uint64).astype(np.uint32)
    total, key = 32 * W, 2 * k
    for j in range(W):  # keep the top 2k bits
        keep = min(32, max(0, key - 32 * j))
        mask = 0 if keep == 0 else ((0xFFFFFFFF << (32 - keep)) & 0xFFFFFFFF)
        bits[:, j] &= np.uint32(mask)
    flags = (rng.integers(0, 2, size=m).astype(np.uint32) << 19) | (rng.integers(0, 5, size=m).astype(np.uint32) << 16)
    bits[:, W - 1] |= flags
    assert total - key >= 20
    rec = bits[rng.integers(0, m, size=n)] if pool else bits
    rec = rec.copy()
    if buckets is not None:
        b = np.asarray(buckets, dtype=np.uint32)[rng.integers(0, len(buckets), size=n)]
        rec[:, 0] = (rec[:, 0] & np.uint32(0xFFFF)) | (b << 16)
    rec[:, W - 1] |= rng.integers(0, 1 << 16, size=n).astype(np.uint32)
    return rec


def sort_byte_matrix(rec: np.ndarray, k: int) -> np.ndarray:
    """(n, len(sort bytes)) uint8, most significant sort byte first"""
    W = rec.shape[1]
    cols = []
    for b in reversed(lib.s2s_sort_bytes(k)):
        cols.append((rec[:, W - 1 - (b >> 2)] >> np.uint32(8 * (b & 3))) & np.uint32(255))
    return np.stack(cols, axis=1).astype(np.uint8) if cols else np.zeros((len(rec), 0), np.uint8)


def dense_rank(mat: np.ndarray) -> np.ndarray:
    """rank of every row among the distinct rows (lexicographic, first column most significant)"""
    if len(mat) == 0:
        return np.zeros(0, np.int64)
    _, inv = np.unique(mat, axis=0, return_inverse=True)
    return inv.reshape(-1)


def check_sorted(inp: np.ndarray, out: np.ndarray, k: int):
    """out is ascending on the sort bytes and the same multiset of whole records as inp"""
    assert out.shape == inp.shape
    if len(out) > 1:
        r = dense_rank(sort_byte_matrix(out, k))
        bad = np.flatnonzero(np.diff(r) < 0)
        assert len(bad) == 0, f"{len(bad)} descents, first at {bad[:5]}"
    a = inp[np.lexsort(inp.T[::-1])]
    b = out[np.lexsort(out.T[::-1])]
    assert np.array_equal(a, b), "output is not a permutation of the input"
