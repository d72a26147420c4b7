"""read2sdbg on a streamed library, host code only (no GPU needed): the offsets a chunk derives from its own records
(r2s_read_geom + exclusive scans, as k_r2s_chunk_geom and scan32 do on the device) against slices of index_pkg, and the
residency rule of mhb_read2sdbg_host on crafted library sizes."""
import numpy as np
import pytest

from megahit_b200 import lib


def make_bin(lengths, seed=0):
    """a `.bin` image of reads with the given lengths (random bases)"""
    rng = np.random.default_rng(seed)
    out = []
    for L in lengths:
        out.append(np.array([L], np.uint32))
        out.append(rng.integers(0, 2 ** 32, size=(L + 15) // 16, dtype=np.uint64).astype(np.uint32))
    return np.concatenate(out) if out else np.zeros(0, np.uint32)


def chunks_of(n, cuts):
    first = [0] + sorted(set(c for c in cuts if 0 < c < n)) + [n]
    return list(zip(first[:-1], first[1:]))


def check_chunks(lengths, k, cuts):
    b = make_bin(lengths)
    n = len(lengths)
    whole = lib.selftest_r2s_chunk_index(b, n, k, 0, n, derive=False)
    for f, e in chunks_of(n, cuts):
        want = lib.selftest_r2s_chunk_index(b, n, k, f, e - f, derive=False)
        got = lib.selftest_r2s_chunk_index(b, n, k, f, e - f, derive=True)
        for key in ("len", "word_off", "base_off", "s1_off", "edge_off"):
            assert (got[key] == want[key]).all(), (key, f, e)
        assert got["base0"] == want["base0"] == int(whole["base_off"][f])


@pytest.mark.parametrize("k", [9, 21, 27, 99])
def test_chunk_index_with_zero_length_reads(k):
    """zero-length reads first, last and alone in a chunk: each counts as one base and one package word"""
    lengths = [0, 150, 0, 0, 30, k, k + 1, 0, 17, 16, 0, 300, 5, 0]
    n = len(lengths)
    check_chunks(lengths, k, [])                           # the whole library as one chunk
    check_chunks(lengths, k, range(n))                     # one read per chunk
    check_chunks(lengths, k, [1, 2, 4, 7, 8, 11, 13])      # zero-length reads first and last in chunks
    got = lib.selftest_r2s_chunk_index(make_bin(lengths), n, k, 2, 2, derive=True)
    assert list(got["len"]) == [1, 1] and list(got["word_off"]) == [0, 1, 2] and got["base0"] == 1 + 150


def test_chunk_index_random_library():
    rng = np.random.default_rng(3)
    lengths = rng.integers(0, 260, size=3000)
    lengths[rng.integers(0, 3000, size=300)] = 0
    cuts = rng.integers(1, 3000, size=40).tolist()
    for k in (21, 59, 141):
        check_chunks(lengths.tolist(), k, cuts)


def test_chunk_index_of_short_reads():
    """reads shorter than k + 1 have no stage-1 records and no edges"""
    lengths = [5, 26, 27, 28, 0, 100]
    got = lib.selftest_r2s_chunk_index(make_bin(lengths), 6, 27, 0, 6, derive=True)
    assert list(np.diff(got["s1_off"])) == [0, 0, 0, 5, 0, 77]
    assert list(np.diff(got["edge_off"])) == [0, 0, 0, 1, 0, 73]


def test_fixed_length_chunk_base():
    """a fixed-length chunk keeps no per-read arrays: its global base is first * L"""
    b = make_bin([150] * 40)
    for f, c in ((0, 40), (7, 1), (13, 20), (39, 1)):
        got = lib.selftest_r2s_chunk_index(b, 40, 27, f, c, derive=True)
        assert got["base0"] == 150 * f
        assert (got["base_off"] == 150 * np.arange(c + 1)).all()
        assert (got["word_off"] == 10 * np.arange(c + 1)).all()
        assert (got["s1_off"] == 127 * np.arange(c + 1)).all() and (got["edge_off"] == 123 * np.arange(c + 1)).all()
    with pytest.raises(lib.MhbError, match="fixed-length"):
        lib.selftest_r2s_chunk_index(b, 40, 27, 0, 40, derive=False)


def sizes(n_reads, L, k):
    """the index sizes of n_reads fixed-length reads of L bases"""
    w = (L + 15) // 16
    return dict(n_reads=n_reads, bin_words=n_reads * (1 + w), fixed_len=L, n_words=n_reads * w, n_bases=n_reads * L,
                n_s1=n_reads * (L - k + 4) if L > k else 0, n_edges=n_reads * (L - k) if L > k else 0)


def decide(sz, k=27, m=2, mercy=True, free=0, cap=0):
    return lib.r2s_stream_decide(**sz, k=k, m=m, need_mercy=mercy, free_bytes=free, chunk_limit=cap)


def threshold(sz, **kw):
    """the least free device memory at which the library stays resident (the rule is monotone in it)"""
    lo, hi = 0, 1 << 44
    assert not decide(sz, free=hi, **kw)["stream"]
    while lo + 1 < hi:
        mid = (lo + hi) // 2
        if decide(sz, free=mid, **kw)["stream"]:
            lo = mid
        else:
            hi = mid
    return hi


def test_residency_rule_on_crafted_sizes():
    gb = 1 << 30
    sz = sizes(10_000_000, 150, 27)
    d = decide(sz, free=80 * gb)
    assert not d["stream"]
    # ~178 bytes per 150 bp read with mercy, before any round buffer (package 40, planes 4 bits per base, upload 44)
    assert 170 * 10 ** 7 < d["resident"] + d["upload"] < 185 * 10 ** 7
    # a chunk cap streams whatever the memory
    assert decide(sz, free=80 * gb, cap=64 << 20)["stream"]
    # the resident form and its upload do not fit
    assert decide(sz, free=d["resident"] + d["upload"] - 1)["stream"]
    # they fit, but leave no room for a stage-1 round: still streamed
    t = threshold(sz)
    assert t > d["resident"] + d["upload"]
    assert decide(sz, free=t)["stream"] is False and decide(sz, free=t - 1)["stream"] is True
    # with 80 GB free, 460 M reads of 150 bp are streamed (the resident form and its upload alone need ~178 bytes a
    # read), 400 M stay resident
    assert decide(sizes(460_000_000, 150, 27), free=80 * 10 ** 9)["stream"]
    assert not decide(sizes(400_000_000, 150, 27), free=80 * 10 ** 9)["stream"]


def test_residency_rule_parts():
    sz = sizes(1_000_000, 150, 27)
    with_mercy = decide(sz, free=1 << 40)["resident"]
    no_mercy = decide(sz, mercy=False, free=1 << 40)["resident"]
    m1 = decide(sz, m=1, mercy=False, free=1 << 40)["resident"]
    bases = 150 * 1_000_000
    assert abs((with_mercy - no_mercy) - bases // 2) < 4096      # 4 bits per base: three candidate planes + mercy
    assert abs((no_mercy - m1) - bases // 8) < 4096              # m == 1 keeps no solid plane
    # reads shorter than k + 1: nothing to sort, so no round to fit: resident exactly when the library and upload fit
    short = sizes(1_000_000, 20, 27)
    d = decide(short, free=1 << 40)
    assert threshold(short) == d["resident"] + d["upload"] + 1
