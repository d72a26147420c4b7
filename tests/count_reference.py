"""Exact NumPy restatement of the solid-edge count (A5): KmerCounter::Lv2Postprocess + PackEdge
(kmer_counter.cpp:254-305, :32-52) applied to count records as the device stores them.

A count record is mhb_count_record_words(k) uint32 words: the canonical (k+1)-mer left-aligned, zero fill, and
prev << 3 | next in the low 6 bits of the last word (0..3 = a base, 4 = none).  Counts and tallies are int64 here, so
nothing wraps or saturates except where the reference itself clamps (the 16-bit multiplicity, kMaxMul = 65535).
Used by the GPU tests as the yardstick for both count paths (hashed and sort + run-length)."""
import numpy as np

MAX_MUL = 65535


def words_per_edge(k: int) -> int:
    return (2 * (k + 1) + 16 + 31) // 32  # kmer_counter.cpp:79-80


def count_record_words(k: int) -> int:
    return (2 * (k + 1) + 6 + 31) // 32


def make_records(keys, prev, nxt, k: int) -> np.ndarray:
    """Count records for k <= 31 (whose (k+1)-mer fits 64 bits): keys = uint64 (k+1)-mers left-aligned, masked here to
    their 2(k+1) leading bits so that the records are valid for this k; prev / next 0..4 per record."""
    assert k <= 31
    keys = np.asarray(keys, np.uint64)
    keys = keys & ~np.uint64((1 << (64 - 2 * (k + 1))) - 1) if k < 31 else keys
    pn = (np.asarray(prev, np.uint64) << np.uint64(3)) | np.asarray(nxt, np.uint64)
    hi, lo = (keys >> np.uint64(32)).astype(np.uint32), (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    if count_record_words(k) == 2:
        return np.stack([hi, lo | pn.astype(np.uint32)], axis=1)
    return np.stack([hi, lo, pn.astype(np.uint32)], axis=1)


def records_from_tallies(keys, pt, nt, k: int) -> np.ndarray:
    """Records with exactly the given per-key prev / next tallies: pt, nt (n_keys, 5) counts of prev / next = 0..4,
    equal row sums (= the key's occurrences).  Records come out grouped by key; callers permute them."""
    pt, nt = np.asarray(pt, np.int64), np.asarray(nt, np.int64)
    cnt = pt.sum(axis=1)
    assert (cnt == nt.sum(axis=1)).all()
    sym = np.tile(np.arange(5, dtype=np.uint64), len(cnt))
    kidx = np.repeat(np.arange(len(cnt)), cnt)
    return make_records(np.asarray(keys, np.uint64)[kidx], np.repeat(sym, pt.reshape(-1)), np.repeat(sym, nt.reshape(-1)), k)


def _key_columns(recs: np.ndarray) -> list:
    """the key (record without its low 6 bits) as big-endian uint64 columns, most significant first"""
    w = [recs[:, j].astype(np.uint64) for j in range(recs.shape[1])]
    w[-1] = w[-1] & np.uint64(~63 & 0xFFFFFFFF)
    cols = []
    for j in range(0, len(w), 2):
        cols.append((w[j] << np.uint64(32)) | w[j + 1] if j + 1 < len(w) else w[j] << np.uint64(32))
    return cols


def count_records_reference(recs: np.ndarray, k: int, m: int):
    """recs: (n, WR) uint32 count records in any order.  Returns (edges, aux, mul_hist, n_solid):
    edges (n_solid, words_per_edge(k)) uint32, the solid (k+1)-mers ascending with min(count, 65535) in the low 16 bits
    of the last word; aux (n_solid,) uint8, bit 0 = no incoming, bit 1 = no outgoing; mul_hist (65536,) int64 over all
    distinct (k+1)-mers; n_solid = number of keys with count >= m."""
    recs = np.ascontiguousarray(recs, dtype=np.uint32)
    n, wr = recs.shape
    assert wr == count_record_words(k), (wr, k)
    assert m >= 1
    we = words_per_edge(k)
    pn = recs[:, -1] & np.uint32(63)
    prev, nxt = (pn >> np.uint32(3)).astype(np.int64), (pn & np.uint32(7)).astype(np.int64)
    assert (prev <= 4).all() and (nxt <= 4).all(), "prev / next must be 0..4"
    # valid records: the zero fill between the (k+1)-mer and prev / next is record bits [6, 6 + pad), counted from the
    # least significant bit of the last word
    pad = 32 * wr - 2 * (k + 1) - 6
    for j in range(wr):
        base = 32 * (wr - 1 - j)
        a, b = max(6, base), min(6 + pad, base + 32)
        if a < b:
            mask = ((1 << (b - a)) - 1) << (a - base)
            assert not (recs[:, j] & np.uint32(mask)).any(), "bits between the (k+1)-mer and prev / next must be zero"
    mul_hist = np.zeros(MAX_MUL + 1, np.int64)
    if n == 0:
        return np.zeros((0, we), np.uint32), np.zeros(0, np.uint8), mul_hist, 0

    cols = _key_columns(recs)
    order = np.lexsort(cols[::-1])  # last key = primary
    sc = [c[order] for c in cols]
    head = np.ones(n, bool)
    diff = np.zeros(n - 1, bool)
    for c in sc:
        diff |= c[1:] != c[:-1]
    head[1:] = diff
    gid_sorted = np.cumsum(head) - 1
    n_keys = int(gid_sorted[-1]) + 1
    inverse = np.empty(n, np.int64)
    inverse[order] = gid_sorted

    count = np.bincount(inverse, minlength=n_keys).astype(np.int64)
    pt = np.bincount(inverse * 5 + prev, minlength=5 * n_keys).reshape(n_keys, 5)
    nt = np.bincount(inverse * 5 + nxt, minlength=5 * n_keys).reshape(n_keys, 5)
    has_in = (pt[:, :4] >= m).any(axis=1)
    has_out = (nt[:, :4] >= m).any(axis=1)
    c16 = np.minimum(count, MAX_MUL)
    mul_hist += np.bincount(c16, minlength=MAX_MUL + 1)

    solid = count >= m
    n_solid = int(solid.sum())
    first_rec = recs[order[head]]  # one record per key, keys ascending
    key_words = first_rec[solid].copy()
    key_words[:, -1] &= np.uint32(~63 & 0xFFFFFFFF)
    edges = np.zeros((n_solid, we), np.uint32)
    edges[:, :wr] = key_words
    edges[:, -1] |= c16[solid].astype(np.uint32)
    aux = ((~has_in[solid]).astype(np.uint8) | ((~has_out[solid]).astype(np.uint8) << 1)).astype(np.uint8)
    return edges, aux, mul_hist, n_solid
