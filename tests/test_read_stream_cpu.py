"""The chunk plan and the residency rule of the streamed read library (mhb_plan_read_chunks, mhb_read_stream_decide):
host logic only, no GPU needed."""
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


def record_bytes(lengths):
    return [4 * (1 + (L + 15) // 16) for L in lengths]


def check_plan(lengths, cap):
    b = make_bin(lengths)
    first = lib.plan_read_chunks(b, len(lengths), cap)
    n = len(lengths)
    if n == 0:
        assert first == [0]
        return first
    # the chunks tile the reads in order
    assert first[0] == 0 and first[-1] == n
    assert all(first[i] < first[i + 1] for i in range(len(first) - 1))
    rb = record_bytes(lengths)
    for i in range(len(first) - 1):
        size = sum(rb[first[i]:first[i + 1]])
        # at most the cap, unless a single read alone exceeds it
        assert size <= cap or first[i + 1] - first[i] == 1, (i, size, cap)
        # greedy: the next read would not have fit
        if i + 2 < len(first):
            assert size + rb[first[i + 1]] > cap
    return first


def test_fixed_length():
    first = check_plan([150] * 1000, 44 * 10)
    assert len(first) - 1 == 100 and all(first[i] == 10 * i for i in range(101))
    first = check_plan([150] * 1001, 44 * 10 + 43)  # a cap between multiples of the record keeps whole reads
    assert first[1] == 10 and len(first) - 1 == 101


def test_variable_length():
    rng = np.random.default_rng(7)
    lengths = rng.integers(0, 400, size=2000).tolist()
    for cap in (64, 500, 4096, 1 << 20):
        check_plan(lengths, cap)
    assert lib.plan_read_chunks(make_bin(lengths), len(lengths), 1 << 30) == [0, len(lengths)]


def test_zero_length_reads():
    lengths = [0, 0, 5, 0, 16, 17, 0, 0, 0, 33]
    first = check_plan(lengths, 8)  # a zero-length read is one word, so two fit in 8 bytes
    assert first[:2] == [0, 2]
    check_plan([0] * 100, 4)
    assert len(check_plan([0] * 100, 4)) - 1 == 100


def test_empty_library():
    assert lib.plan_read_chunks(np.zeros(0, np.uint32), 0, 1024) == [0]


def test_read_larger_than_cap_gets_its_own_chunk():
    lengths = [20, 20, 5000, 20, 20, 20, 4000]
    first = check_plan(lengths, 64)
    assert [2, 3] == [r for r in first if r in (2, 3)]
    assert 6 in first and first[-1] == 7
    # a cap below every read: one read per chunk
    assert check_plan([150] * 50, 16) == list(range(51))


def test_bad_arguments():
    with pytest.raises(lib.MhbError, match="truncated"):
        lib.plan_read_chunks(np.array([40, 0], np.uint32), 1, 1024)
    with pytest.raises(lib.MhbError, match="bad chunk plan"):
        lib.plan_read_chunks(make_bin([10]), 1, 0)


def test_residency_rule():
    gb = 1 << 30
    # resident whenever the resident part fits the available memory and its plan works, with no cap set
    assert not lib.read_stream_decide(10 * gb, 70 * gb)
    # streamed when the resident part alone does not fit ...
    assert lib.read_stream_decide(70 * gb, 70 * gb)
    assert lib.read_stream_decide(90 * gb, 70 * gb)
    # ... when the plan next to it fails (one bucket larger than the room left) ...
    assert lib.read_stream_decide(10 * gb, 70 * gb, plan_failed=True)
    # ... or when a chunk cap is set
    assert lib.read_stream_decide(1, 70 * gb, chunk_limit=1 << 20)
