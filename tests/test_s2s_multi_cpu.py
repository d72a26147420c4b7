"""The share planner of the multi-GPU seq2sdbg (mhb_plan_seq_shares, host logic only): contiguous shares that cover
every sequence once, balanced on their sort items to within one sequence, also with more ranks than sequences."""
import numpy as np
import pytest

from megahit_b200 import lib


def items(length, k):
    length = np.asarray(length, np.int64)
    return np.where(length >= k + 1, 2 * (length - k + 2), 0)


def check(length, k, n):
    first = lib.plan_seq_shares(np.asarray(length, np.uint32), k, n)
    assert len(first) == n + 1 and first[0] == 0 and first[-1] == len(length)
    assert all(a <= b for a, b in zip(first, first[1:])), first  # contiguous, every sequence in exactly one share
    it = items(length, k)
    cum = np.concatenate([[0], np.cumsum(it)])
    total = int(cum[-1])
    biggest = int(it.max()) if len(it) else 0
    for r in range(1, n):
        # every cut is the boundary closest to r / n of the items, so it is off by at most half a sequence
        target = total * r // n
        assert 2 * abs(int(cum[first[r]]) - target) <= biggest, (r, first)
    for r in range(n):
        assert abs(int(cum[first[r + 1]] - cum[first[r]]) - total / n) <= biggest + 1, (r, first)
    return first


@pytest.mark.parametrize("k", [21, 59, 141, 227])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_random_lengths(k, n):
    rng = np.random.default_rng(k * 10 + n)
    length = rng.integers(1, 3 * k + 400, size=5000)
    check(length, k, n)


def test_sequences_without_items_anywhere():
    """sequences shorter than k + 1 carry no items: they ride along with their neighbours"""
    k = 31
    length = np.array([5, 40, 10, 10, 100, 3, 3, 60, 2], np.uint32)
    check(length, k, 3)
    check(np.full(50, 10, np.uint32), k, 4)


def test_more_ranks_than_sequences():
    first = check(np.array([100, 200, 150], np.uint32), 21, 8)
    sizes = np.diff(first)
    assert sizes.sum() == 3 and (sizes == 0).sum() >= 5


def test_no_sequences():
    assert lib.plan_seq_shares(np.zeros(0, np.uint32), 21, 4) == [0, 0, 0, 0, 0]


def test_one_huge_sequence_among_small_ones():
    length = np.array([30] * 20 + [100000] + [30] * 20, np.uint32)
    first = check(length, 21, 4)
    assert first[0] == 0 and first[-1] == len(length)
