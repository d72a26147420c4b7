"""Exact NumPy restatement of the solid-edge count (A5): KmerCounter::Lv2Postprocess + PackEdge
(kmer_counter.cpp:254-305, :32-52) applied to count records as the device stores them.

A count record is mhb_count_record_words(k) uint32 words: the canonical (k+1)-mer left-aligned, zero fill, and
prev << 3 | next in the low 6 bits of the last word (0..3 = a base, 4 = none).  Counts and tallies are int64 here, so
nothing wraps or saturates except where the reference itself clamps (the 16-bit multiplicity, kMaxMul = 65535).
Used by the GPU tests as the yardstick for both count paths (hashed and sort + run-length).  extract_records and
reference_marks restate the extraction and the mercy marks for any k, so that every record width has a yardstick."""
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


def count_key_words(k: int) -> int:
    return (2 * (k + 1) + 31) // 32


def key_mask(k: int) -> np.ndarray:
    """(count_key_words(k),) uint32: the 2(k+1) leading bits of a left-aligned (k+1)-mer"""
    bits = np.clip(2 * (k + 1) - 32 * np.arange(count_key_words(k)), 0, 32)
    return np.array([(0xFFFFFFFF << (32 - int(b))) & 0xFFFFFFFF for b in bits], np.uint32)


def make_records_wide(key_words, prev, nxt, k: int) -> np.ndarray:
    """Count records for any k: key_words = (n, >= count_key_words(k)) uint32, the (k+1)-mer left-aligned from word 0,
    masked here to its 2(k+1) leading bits (the rest is zero fill); prev / next 0..4 in the low 6 bits of the last word."""
    w, wr = count_key_words(k), count_record_words(k)
    key_words = np.asarray(key_words, np.uint32).reshape(len(key_words), -1)
    recs = np.zeros((len(key_words), wr), np.uint32)
    recs[:, :w] = key_words[:, :w] & key_mask(k)
    recs[:, -1] |= (np.asarray(prev, np.uint32) << np.uint32(3)) | np.asarray(nxt, np.uint32)
    return recs


def read_layout(bin_words, n_reads: int):
    """length and first word of every read of a `.bin` word stream"""
    lens, starts, pos = np.empty(n_reads, np.int64), np.empty(n_reads, np.int64), 0
    for r in range(n_reads):
        lens[r], starts[r] = int(bin_words[pos]), pos
        pos += 1 + (lens[r] + 15) // 16
    return lens, starts


def _pack_bases(b: np.ndarray, n_words: int) -> np.ndarray:
    """(n, nb) bases 0..3 -> (n, n_words) uint32, first base in the top bits of word 0, zero fill"""
    pad = np.zeros((len(b), 16 * n_words), np.uint32)
    pad[:, : b.shape[1]] = b
    sh = (30 - 2 * np.arange(16, dtype=np.uint32)).astype(np.uint32)
    return np.bitwise_or.reduce(pad.reshape(len(b), n_words, 16) << sh, axis=2).astype(np.uint32)


def _less_rows(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """row-wise x < y, words compared most significant first"""
    less, decided = np.zeros(len(x), bool), np.zeros(len(x), bool)
    for j in range(x.shape[1]):
        less |= ~decided & (x[:, j] < y[:, j])
        decided |= x[:, j] != y[:, j]
    return less


def extract_records(bin_words, n_reads: int, k: int, max_bases: int = 1 << 22):
    """KmerCounter's edge extraction (kmer_counter.cpp:158-252) restated per base for any k, on a `.bin` word stream
    (file orientation).  The reference works on the reversed read: with S = read[q, q + k + 1) the package-orientation
    edge is reverse(S) and its reverse complement is complement(S); the canonical edge is the smaller of the two as a
    base string (ties: strand 0, reverse(S)), and prev / next are the package neighbours, swapped and complemented on
    strand 1.  Returns (records (n_edges, count_record_words(k)) uint32, strand (n_edges,) uint8) in read order, record
    edge_off[r] + q for position q of read r, as mhb_count_extract stores them.  Reads are taken in groups of equal
    length, windows in blocks of about max_bases bases."""
    bin_words = np.asarray(bin_words, np.uint32)
    K1, W, WR = k + 1, count_key_words(k), count_record_words(k)
    lens, starts = read_layout(bin_words, n_reads)
    n_e = np.maximum(lens - k, 0)
    edge_off = np.concatenate([[0], np.cumsum(n_e)])
    recs = np.zeros((int(edge_off[-1]), WR), np.uint32)
    strand = np.zeros(int(edge_off[-1]), np.uint8)
    sh = np.arange(30, -1, -2, dtype=np.uint32)
    for L in np.unique(lens[lens >= K1]):
        ids = np.flatnonzero(lens == L)
        ne = int(L) - k
        nw = (int(L) + 15) // 16
        q_step = max(1, min(ne, max_bases // K1))
        r_step = max(1, max_bases // (q_step * K1))
        for r0 in range(0, len(ids), r_step):
            rid = ids[r0:r0 + r_step]
            w = bin_words[starts[rid][:, None] + 1 + np.arange(nw)[None, :]]
            b = ((w[:, :, None] >> sh[None, None, :]) & np.uint32(3)).reshape(len(rid), -1)[:, :L].astype(np.uint8)
            win = np.lib.stride_tricks.sliding_window_view(b, K1, axis=1)  # (g, ne, K1)
            for q0 in range(0, ne, q_step):
                q1 = min(ne, q0 + q_step)
                S = win[:, q0:q1].reshape(-1, K1)
                A = _pack_bases(S[:, ::-1], W)       # reverse(S): the package-orientation edge
                B = _pack_bases(3 - S, W)            # complement(S): its reverse complement
                st = _less_rows(B, A)
                q = np.tile(np.arange(q0, q1), len(rid))
                row = np.repeat(np.arange(len(rid)), q1 - q0)
                prev = np.where(q + K1 < L, b[row, np.minimum(q + K1, L - 1)], 4).astype(np.uint32)
                nxt = np.where(q > 0, b[row, np.maximum(q - 1, 0)], 4).astype(np.uint32)
                p = np.where(st, np.where(nxt == 4, 4, 3 - nxt), prev)
                n = np.where(st, np.where(prev == 4, 4, 3 - prev), nxt)
                at = edge_off[rid][row] + q
                recs[at] = make_records_wide(np.where(st[:, None], B, A), p, n, k)
                strand[at] = st
    return recs, strand


def record_byte_hist(recs: np.ndarray, byte: int) -> np.ndarray:
    """256-bin histogram of record byte `byte` (0 = least significant byte of the last word)"""
    col = recs[:, recs.shape[1] - 1 - byte // 4] if len(recs) else np.zeros(0, np.uint32)
    return np.bincount((col >> np.uint32(8 * (byte % 4))) & np.uint32(255), minlength=256).astype(np.int64)


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


SENTINEL = 0xFFFFFFFF


def reference_marks(bin_words, n_reads: int, k: int, m: int):
    """The per-read mercy marks of KmerCounter (first_0_out / last_0_in, kmer_counter.cpp:307-367) for any k, from the
    solid edges and in / out flags of count_records_reference over extract_records.  -> first, last (uint32 per read,
    SENTINEL when unset), edges, aux, n_tip (solid edges with a flag)."""
    recs, strand = extract_records(bin_words, n_reads, k)
    edges, aux, _, n_solid = count_records_reference(recs, k, m)
    first = np.full(n_reads, SENTINEL, np.int64)
    last = np.full(n_reads, -1, np.int64)
    if n_solid:
        w, mask = count_key_words(k), key_mask(k)
        as_void = lambda x: np.ascontiguousarray(x[:, :w] & mask).astype(">u4").view(f"V{4 * w}").ravel()
        ekey, rkey = as_void(edges), as_void(recs)  # edges are ascending: big-endian bytes sort as the keys do
        i = np.minimum(np.searchsorted(ekey, rkey), n_solid - 1)
        flags = np.where(ekey[i] == rkey, aux[i], 0)
        lens, _ = read_layout(bin_words, n_reads)
        n_e = np.maximum(lens - k, 0)
        rid = np.repeat(np.arange(n_reads), n_e)
        q = np.arange(len(recs)) - np.repeat(np.concatenate([[0], np.cumsum(n_e)[:-1]]), n_e)
        off = lens[rid] - (k + 1) - q  # package offset of the edge
        st = strand.astype(bool)
        no_in, no_out = (flags & 1) != 0, (flags & 2) != 0
        to_last = (no_in & ~st) | (no_out & st)
        to_first = (no_in & st) | (no_out & ~st)
        np.maximum.at(last, rid[to_last], off[to_last])
        np.minimum.at(first, rid[to_first], off[to_first] + 1)
    last = np.where(last >= 0, last, SENTINEL)
    return first.astype(np.uint32), last.astype(np.uint32), edges, aux, int((aux != 0).sum())
