"""The NumPy count reference (tests/count_reference.py) against a deliberately naive restatement of
KmerCounter::Lv2Postprocess + PackEdge (kmer_counter.cpp:254-305, :32-52): a dict of per-key tallies and a loop per
record.  The any-k extraction and mercy-mark restatements against the C oracle at every record width.  No GPU: a bug in
the yardstick must not be mistaken for a kernel bug."""
import numpy as np
import pytest

from count_reference import (count_key_words, count_records_reference, count_record_words, extract_records, make_records,
                             make_records_wide, record_byte_hist, records_from_tallies, reference_marks, words_per_edge)
from count_wide_cases import library, pack, palindrome, width_classes


def naive_count(recs, k, m):
    wr = recs.shape[1]
    we = words_per_edge(k)
    tally = {}
    for r in recs.tolist():
        key = tuple(r[:-1]) + (r[-1] & ~63 & 0xFFFFFFFF,)
        pn = r[-1] & 63
        t = tally.setdefault(key, [0, [0] * 5, [0] * 5])
        t[0] += 1
        t[1][pn >> 3] += 1
        t[2][pn & 7] += 1
    hist = np.zeros(65536, np.int64)
    edges, aux = [], []
    for key in sorted(tally):
        count, cp, cn = tally[key]
        hist[min(count, 65535)] += 1
        if count < m:
            continue
        has_in = any(cp[j] >= m for j in range(4))
        has_out = any(cn[j] >= m for j in range(4))
        dest = [key[i] if i < wr else 0 for i in range(we)]
        chars_in_last_word, which = (k + 1) % 16, (k + 1) // 16
        if chars_in_last_word:
            s = (16 - chars_in_last_word) * 2
            dest[which] = (dest[which] >> s) << s
        else:
            dest[which] = 0
        for i in range(which + 1, we):
            dest[i] = 0
        dest[we - 1] |= min(65535, count)
        edges.append(dest)
        aux.append((0 if has_in else 1) | (0 if has_out else 2))
    return np.array(edges, np.uint32).reshape(-1, we), np.array(aux, np.uint8), hist, len(edges)


def _tally_row(rng, c, m, kind):
    """prev (or next) tallies over 0..4 summing to c"""
    t = np.zeros(5, np.int64)
    b = int(rng.integers(0, 4))
    if kind == "random":
        t = np.bincount(rng.integers(0, 5, c), minlength=5)
    elif kind == "exact_m":
        t[b] = min(m, c)
    elif kind == "below_m":
        for j in range(4):
            t[j] = min(m - 1, c - t.sum())
    elif kind == "wrap":  # a byte tally would wrap to 0 (or to m - 1)
        t[b] = min(c, 256 + (m - 1 if rng.integers(0, 2) else 0))
    t[4] = c - t[:4].sum()  # kind "none" keeps everything at 4
    return t


def random_set(rng, k, m):
    n_keys = int(rng.integers(1, 12))
    kb = 2 * (k + 1)
    # few distinct high bits so that keys share words / prefixes, random low bits
    keys = (rng.integers(0, 4, n_keys, dtype=np.uint64) << np.uint64(62)) | rng.integers(0, 1 << 62, n_keys, dtype=np.uint64)
    if rng.integers(0, 3) == 0:  # keys that differ only in their last base
        keys[:] = keys[0]
        keys ^= rng.integers(0, 4, n_keys, dtype=np.uint64) << np.uint64(64 - kb)
    choices = [1, max(1, m - 1), m, m + 1, int(rng.integers(1, 3 * m + 3)), 255, 256, 257, int(rng.integers(256, 700))]
    counts = [choices[int(rng.integers(0, len(choices)))] for _ in range(n_keys)]
    kinds = ["random", "none", "exact_m", "below_m", "wrap"]
    pt = np.array([_tally_row(rng, c, m, kinds[int(rng.integers(0, 5))]) for c in counts])
    nt = np.array([_tally_row(rng, c, m, kinds[int(rng.integers(0, 5))]) for c in counts])
    recs = records_from_tallies(keys, pt, nt, k)
    return recs[rng.permutation(len(recs))]


@pytest.mark.parametrize("m,n_sets", [(1, 500), (2, 600), (3, 500), (256, 250), (1024, 120)])
def test_reference_matches_naive_on_random_sets(m, n_sets):
    rng = np.random.default_rng(1000 + m)
    seen = {"hot": 0, "all_prev_none": 0, "tally_m": 0, "tally_m_minus_1": 0, "solid": 0}
    for i in range(n_sets):
        k = (13, 20, 21, 27, 28, 29, 31)[i % 7]
        recs = random_set(rng, k, m)
        assert recs.shape[1] == count_record_words(k)
        e0, a0, h0, n0 = naive_count(recs, k, m)
        e1, a1, h1, n1 = count_records_reference(recs, k, m)
        assert n0 == n1 and (e0 == e1).all() and (a0 == a1).all() and (h0 == h1).all(), (m, i, k)
        # what this set covered
        key = recs.copy()
        key[:, -1] &= np.uint32(~63 & 0xFFFFFFFF)
        _, inv, cnt = np.unique(key, axis=0, return_inverse=True, return_counts=True)
        inv = inv.reshape(-1)
        prev = (recs[:, -1] >> 3) & 7
        pt = np.zeros((len(cnt), 5), np.int64)
        np.add.at(pt, (inv, prev), 1)
        seen["hot"] += int((cnt >= 256).sum())
        seen["all_prev_none"] += int((pt[:, 4] == cnt).sum())
        seen["tally_m"] += int((pt[:, :4] == m).any(axis=1).sum())
        seen["tally_m_minus_1"] += int((pt[:, :4] == m - 1).any(axis=1).sum()) if m > 1 else 1
        seen["solid"] += n0
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("m", [1, 2, 1024])
def test_reference_matches_naive_across_the_multiplicity_clamp(m):
    rng = np.random.default_rng(7 + m)
    k = 27
    counts = np.array([65534, 65535, 65536, 65537, 3, 1024])
    keys = rng.integers(0, 1 << 63, len(counts), dtype=np.uint64)
    pt = np.array([_tally_row(rng, int(c), m, kind) for c, kind in zip(counts, ["wrap", "none", "exact_m", "random", "random", "below_m"])])
    nt = np.array([_tally_row(rng, int(c), m, "random") for c in counts])
    recs = records_from_tallies(keys, pt, nt, k)
    recs = recs[rng.permutation(len(recs))]
    e0, a0, h0, n0 = naive_count(recs, k, m)
    e1, a1, h1, n1 = count_records_reference(recs, k, m)
    assert n0 == n1 and (e0 == e1).all() and (a0 == a1).all() and (h0 == h1).all()
    assert h1[65535] == 3 and h1[65534] == 1
    assert sorted((e1[:, -1] & 0xFFFF).tolist())[-4:] == [65534, 65535, 65535, 65535]


def test_reference_edge_layout_and_empty_input():
    # k = 28: the key reaches record bit 6 (2 words), the edge needs a third word for the multiplicity
    recs = make_records(np.array([~np.uint64(0), ~np.uint64(0), 0], np.uint64), [4, 0, 4], [1, 4, 4], 28)
    assert (recs[:, 1] & 63).tolist() == [33, 4, 36] and recs[0, 1] >> 6 == (1 << 26) - 1
    edges, aux, hist, n = count_records_reference(recs, 28, 1)
    assert n == 2 and edges.shape == (2, 3)
    assert edges.tolist() == [[0, 0, 1], [0xFFFFFFFF, 0xFFFFFFC0, 2]]
    assert aux.tolist() == [3, 0] and hist[1] == 1 and hist[2] == 1
    # k = 21 (2-word edge, the multiplicity shares the last key word) and k = 31 (3-word records)
    e21 = count_records_reference(make_records(np.array([1 << 63], np.uint64), [2], [3], 21), 21, 1)[0]
    assert e21.tolist() == [[1 << 31, 1]]
    e31 = count_records_reference(make_records(np.array([(1 << 64) - 1] * 2, np.uint64), [0, 0], [3, 3], 31), 31, 2)
    assert e31[0].tolist() == [[0xFFFFFFFF, 0xFFFFFFFF, 2]] and e31[1].tolist() == [0]
    e, a, h, n = count_records_reference(np.zeros((0, 2), np.uint32), 27, 2)
    assert n == 0 and e.shape == (0, 3) and len(a) == 0 and not h.any()
    with pytest.raises(AssertionError):  # a set bit between the (k+1)-mer and prev / next
        count_records_reference(np.array([[0, 1 << 6]], np.uint32), 27, 1)


# ------------------------------------------------------------------------------------------------
# every record width: the extraction restatement and the count reference against the C oracle
# ------------------------------------------------------------------------------------------------
WIDE_K = width_classes(9, 255)


def test_width_classes_cover_every_record_geometry():
    classes = {(count_key_words(k), count_record_words(k), words_per_edge(k)) for k in range(9, 256)}
    assert len(WIDE_K) == len(classes) == 47 and WIDE_K[0] == 12 and WIDE_K[-1] == 255
    assert {(count_key_words(k), count_record_words(k), words_per_edge(k)) for k in WIDE_K} == classes


@pytest.mark.parametrize("k", WIDE_K)
def test_extract_count_and_marks_match_the_oracle_at_every_width(k):
    """extract_records -> count_records_reference == oracle.count (edges, .counting) and reference_marks == its
    first_0_out / last_0_in, on variable-length reads with zero-length ones and (odd k) palindromic (k+1)-mers"""
    from oracle import oracle as O
    m = 2
    binw, n_reads, lens = library(k, 70 + k)
    assert (lens == 0).sum() >= 2 and (lens == k).any() and (lens == k + 1).any()
    assert {0, 1, 15} <= set((lens[lens > k] % 16).tolist())
    recs, strand = extract_records(binw, n_reads, k)
    assert recs.shape == (np.maximum(lens - k, 0).sum(), count_record_words(k))
    edges, aux, hist, n = count_records_reference(recs, k, m)
    oc = O.count(O.unpack_bin(binw.tobytes(), reverse=True), k, m)
    assert n == oc["n_solid"] > 0 and (edges == oc["edges"]).all()
    assert (hist[1:] == oc["counting"][1:]).all()
    first, last, _, _, n_tip = reference_marks(binw, n_reads, k, m)
    assert n_tip > 0 and (first != 0xFFFFFFFF).any()
    assert (first == oc["first_0_out"]).all() and (last == oc["last_0_in"]).all()
    assert (strand == 0).any() and (strand == 1).any()


@pytest.mark.parametrize("k", [31, 47, 63, 127, 255])
def test_palindromes_take_strand_zero(k):
    """a (k+1)-mer equal to its reverse complement keeps the package orientation (rc < fwd is false on a tie):
    prev / next are the package neighbours, not their complements"""
    rng = np.random.default_rng(k)
    pal = palindrome(rng, k)
    x, y = np.array([0, 1, 2], np.uint8), np.array([3, 0], np.uint8)  # file neighbours 2 (before) and 3 (after)
    recs, strand = extract_records(pack([pal, np.concatenate([x, pal, y])]), 2, k)
    assert len(recs) == 1 + (len(x) + len(y) + 1) and strand[0] == 0 and strand[1 + len(x)] == 0
    assert recs[0, -1] & 63 == (4 << 3) | 4 and recs[1 + len(x), -1] & 63 == (3 << 3) | 2
    assert ((recs[0] ^ recs[1 + len(x)]) & ~np.uint32(63) == 0).all()


def _wide_set(rng, k, m):
    """keys that share their leading words and differ in one word, tallies as random_set"""
    w = count_key_words(k)
    n_keys = int(rng.integers(1, 10))
    keys = np.repeat(rng.integers(0, 1 << 32, (1, w), dtype=np.uint64).astype(np.uint32), n_keys, axis=0)
    col = int(rng.integers(0, w))
    keys[:, col] = rng.integers(0, 1 << 32, n_keys, dtype=np.uint64).astype(np.uint32)
    choices = [1, max(1, m - 1), m, m + 1, 256, 257, int(rng.integers(1, 3 * m + 3))]
    counts = [choices[int(rng.integers(0, len(choices)))] for _ in range(n_keys)]
    kinds = ["random", "none", "exact_m", "below_m", "wrap"]
    pt = np.array([_tally_row(rng, c, m, kinds[int(rng.integers(0, 5))]) for c in counts])
    nt = np.array([_tally_row(rng, c, m, kinds[int(rng.integers(0, 5))]) for c in counts])
    sym = np.tile(np.arange(5), n_keys)
    kidx = np.repeat(np.arange(n_keys), pt.sum(axis=1))
    recs = make_records_wide(keys[kidx], np.repeat(sym, pt.reshape(-1)), np.repeat(sym, nt.reshape(-1)), k)
    return recs[rng.permutation(len(recs))]


@pytest.mark.parametrize("m", [1, 2, 3])
def test_reference_matches_naive_at_wide_records(m):
    rng = np.random.default_rng(2000 + m)
    for i in range(150):
        k = (32, 39, 44, 47, 63, 127, 141, 199, 253, 255)[i % 10]
        recs = _wide_set(rng, k, m)
        assert recs.shape[1] == count_record_words(k) >= 3
        e0, a0, h0, n0 = naive_count(recs, k, m)
        e1, a1, h1, n1 = count_records_reference(recs, k, m)
        assert n0 == n1 and (e0 == e1).all() and (a0 == a1).all() and (h0 == h1).all(), (m, i, k)


def test_wide_record_layout_and_empty_input():
    ones = np.full((2, 16), 0xFFFFFFFF, np.uint32)
    # k = 47 (W = 3, WR = 4): the last record word holds prev / next only
    r47 = make_records_wide(ones, [4, 0], [1, 4], 47)
    assert r47.shape == (2, 4) and (r47[:, :3] == 0xFFFFFFFF).all() and r47[:, 3].tolist() == [33, 4]
    e47, a47, h47, n47 = count_records_reference(r47, 47, 1)
    assert n47 == 1 and e47.tolist() == [[0xFFFFFFFF] * 3 + [2]] and a47.tolist() == [0] and h47[2] == 1
    # k = 39 (W = WR = WE = 3): 80 key bits, the multiplicity shares the last key word
    e39 = count_records_reference(make_records_wide(ones[:1], [2], [3], 39), 39, 1)[0]
    assert e39.tolist() == [[0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF0001]]
    # k = 44 (W = WR = 3, WE = 4): the key reaches record bit 6, the multiplicity takes a word of its own
    r44 = make_records_wide(ones[:1], [1], [1], 44)
    assert r44[0, 2] == 0xFFFFFFC0 | 9
    assert count_records_reference(r44, 44, 1)[0].tolist() == [[0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFC0, 1]]
    # k = 255: 17-word records and edges
    r255 = make_records_wide(np.zeros((3, 16), np.uint32), [0, 1, 2], [4, 4, 4], 255)
    e255, a255, _, n255 = count_records_reference(r255, 255, 3)
    assert n255 == 1 and e255.shape == (1, 17) and e255[0, -1] == 3 and a255.tolist() == [3]
    e, a, h, n = count_records_reference(np.zeros((0, 17), np.uint32), 255, 2)
    assert n == 0 and e.shape == (0, 17) and len(a) == 0 and not h.any()
    recs, strand = extract_records(pack([np.zeros(0, np.uint8), np.zeros(255, np.uint8)]), 2, 255)
    assert recs.shape == (0, 17) and len(strand) == 0 and not record_byte_hist(recs, 3).any()
    with pytest.raises(AssertionError):  # a set bit between the (k+1)-mer and prev / next
        count_records_reference(np.array([[0, 0, 0, 1 << 6]], np.uint32), 47, 1)
