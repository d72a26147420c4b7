"""The round budget of a multi-GPU SdBG stage (mhb_sdbg_round_budget, host only): the most sort items one owner takes in
one round of `seq2sdbg --gpus N` or of the k_min graph of `count --gpus N`.  It never exceeds the
mhb_set_s2s_round_limit cap or the items there are, is 0 when not even a one-item round fits, and does not decrease as
the free memory grows."""
import pytest

from megahit_b200 import lib

FIXED = 64 << 20
KS = [21, 59, 141, 227]


@pytest.fixture(autouse=True)
def _no_cap():
    lib.set_s2s_round_limit(0)
    yield
    lib.set_s2s_round_limit(0)


def _one_item_bytes(k):
    """the smallest avail that admits a one-item round"""
    lo, hi = FIXED, FIXED + (1 << 30)
    while lo < hi:
        mid = (lo + hi) // 2
        if lib.sdbg_round_budget(mid, FIXED, k, 10 ** 9):
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("k", KS)
def test_zero_when_not_one_item_fits(k):
    first = _one_item_bytes(k)
    assert lib.sdbg_round_budget(first, FIXED, k, 10 ** 9) >= 1
    assert lib.sdbg_round_budget(first - 1, FIXED, k, 10 ** 9) == 0
    assert lib.sdbg_round_budget(0, FIXED, k, 10 ** 9) == 0
    assert lib.sdbg_round_budget(FIXED, FIXED, k, 10 ** 9) == 0


@pytest.mark.parametrize("k", KS)
def test_grows_with_free_memory(k):
    prev = 0
    for gib in [0.1, 0.25, 0.5, 1, 2, 4, 8, 16, 40, 80]:
        avail = int(gib * (1 << 30))
        b = lib.sdbg_round_budget(avail, FIXED, k, 10 ** 12)
        assert b >= prev
        prev = b
        assert lib.sdbg_round_budget(avail - 1, FIXED, k, 10 ** 12) <= b
    assert prev > 10 ** 8  # 80 GiB hold rounds of more than 100 M items at every k


@pytest.mark.parametrize("k", KS)
def test_never_more_than_the_items(k):
    for n in [0, 1, 7, 1000, 123456]:
        assert lib.sdbg_round_budget(80 << 30, FIXED, k, n) == max(n, 1)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("cap", [1, 1000, 5_000_000])
def test_never_exceeds_the_cap(k, cap):
    free = lib.sdbg_round_budget(80 << 30, FIXED, k, 10 ** 12)
    lib.set_s2s_round_limit(cap)
    assert lib.sdbg_round_budget(80 << 30, FIXED, k, 10 ** 12) == min(cap, free)
    assert lib.sdbg_round_budget(80 << 30, FIXED, k, 10) == min(cap, 10)
    # the cap never makes a round fit that does not
    assert lib.sdbg_round_budget(_one_item_bytes(k) - 1, FIXED, k, 10 ** 12) == 0


def test_bad_k_has_no_budget():
    assert lib.sdbg_round_budget(80 << 30, FIXED, 8, 100) == 0
    assert lib.sdbg_round_budget(80 << 30, FIXED, 256, 100) == 0
