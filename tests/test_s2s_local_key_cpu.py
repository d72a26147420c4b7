"""The in-bucket key of the seq2sdbg sort (s2s_local_key, run on the host through mhb_selftest_s2s_local_key): for every
k the bucket sort takes, ordering records by (16-bit bucket, key) is ordering them by mhb_s2s_sort_bytes."""
import numpy as np
import pytest

from megahit_b200 import lib
from s2s_sort_cases import dense_rank, make_items, sort_byte_matrix


@pytest.mark.parametrize("k", list(range(9, 39)))
def test_local_key_orders_like_the_sort_bytes(k):
    rng = np.random.default_rng(k)
    # few buckets so that most records share theirs; half of the records from a small pool so that keys repeat
    buckets = rng.integers(0, 1 << 16, size=4)
    rec = np.concatenate([make_items(rng, 3000, k, buckets), make_items(rng, 3000, k, buckets, pool=200)])
    # records that differ only in the flag bits or only in the last key bit
    base = np.repeat(rec[:1], 16, axis=0)
    W = rec.shape[1]
    base[:, W - 1] &= np.uint32(~(0xF << 16) & 0xFFFFFFFF)
    base[:, W - 1] |= (np.arange(16, dtype=np.uint32) << 16)
    last = np.repeat(rec[:1], 2, axis=0)
    kb = 2 * k - 1  # bit index (from the top of word 0) of the last key bit
    last[1, kb // 32] ^= np.uint32(1 << (31 - kb % 32))
    rec = np.concatenate([rec, base, last])
    keys = lib.selftest_s2s_local_key(rec, k)
    mine = np.stack([rec[:, 0] >> np.uint32(16), (keys >> np.uint64(32)).astype(np.uint32),
                     (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)], axis=1)
    assert np.array_equal(dense_rank(mine), dense_rank(sort_byte_matrix(rec, k)))


def test_hist_byte_and_workspace():
    """the bucket path (first pass on byte 4W-2) up to 3/4 of 65 536 buckets x 8192 items; above that, and for wider
    items, the full relaxed sort (first pass on byte 2)"""
    limit = 65536 * 8192 * 3 // 4
    for k in (9, 21, 22, 23, 27, 38):
        assert lib.s2s_sort_hist_byte(118_000_000, k) == 4 * lib.s2s_record_words(k) - 2
        assert lib.s2s_sort_hist_byte(limit, k) == 4 * lib.s2s_record_words(k) - 2
        assert lib.s2s_sort_hist_byte(limit + 1, k) == lib.s2s_sort_bytes(k)[0] == 2
    for k in (39, 63):
        assert lib.s2s_sort_hist_byte(1000, k) == lib.s2s_sort_bytes(k)[0]
    L = lib.load()
    assert L.mhb_s2s_sort_workspace_bytes(1 << 20, 27) > L.mhb_sort_workspace_bytes(1 << 20, 3)
