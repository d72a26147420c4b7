"""read2sdbg on several GPUs in rounds over bucket ranges, without a GPU: stage 1 of mhb_read2sdbg_run_multi emulated
round by round with the device code's host-callable pieces, against the oracle.

The owner ranges and their rounds come from the planner the workers use (mhb_plan_count_owner_rounds with a cap).  In
round t every rank's block of its share's records in owner o's sub-range lands at the plan's offset of o's receive
buffer, ranks in rank order; the owner runs stage 1 (stable bucket partition, kmsort, Lv2Postprocess) on that round's
records into the same planes and multiplicity histogram as its earlier rounds.  Then every rank ORs the planes of all
owners over its share's words and runs the mercy step over its share, as in tests/test_r2s_multi_cpu.py."""
import ctypes as C

import numpy as np
import pytest

from megahit_b200 import lib
from test_r2s_multi_cpu import LR, K, M, N, balanced, deep  # noqa: F401  (deep: the tie-heavy library, a fixture)


def owner_hists(recs, per, first):
    """(ranks, 65536) bucket histograms of the ranks' shares"""
    b = (recs[:, 0] >> 16).astype(np.int64)
    return np.stack([np.bincount(b[first[s] * per:first[s + 1] * per], minlength=65536)
                     for s in range(len(first) - 1)]).astype(np.uint64)


def rounds_stage1(recs, per, first, cap, rank_order):
    """(solid bits of every base, multiplicity histogram, mercy count, rounds) of the emulated stage 1 in rounds"""
    L_ = lib.load()
    nw = recs.shape[1] - 2
    W = len(first) - 1
    bw = N * LR // 32 + 2
    plan = lib.plan_count_owner_rounds(owner_hists(recs, per, first), cap)
    planes = np.zeros((W, 4, bw), np.uint32)  # every owner's is_solid, no_in, no_out, any
    counting = np.zeros(65536, np.int64)
    seen = 0
    for t in range(plan["rounds"]):
        for o in range(W):
            lo, hi = int(plan["lo"][t, o]), int(plan["hi"][t, o])
            own_lo, own_hi = plan["owners"][o]
            assert lo > hi or own_lo <= lo <= hi <= own_hi
            if t:  # the rounds of an owner ascend and leave no gap
                plo, phi = int(plan["lo"][t - 1, o]), int(plan["hi"][t - 1, o])
                assert lo > hi or (plo <= phi and lo == phi + 1)
            # the receive buffer of the round: every rank's block at the plan's offset
            buf = np.zeros((int(plan["n"][t, o].sum()), nw + 2), np.uint32)
            at = 0
            for s in rank_order:
                mine = recs[first[s] * per:first[s + 1] * per]
                b = mine[:, 0] >> 16
                blk = mine[(b >= lo) & (b <= hi)]
                assert len(blk) == plan["n"][t, o, s]
                buf[at:at + len(blk)] = blk
                at += len(blk)
            assert at == len(buf)
            seen += len(buf)
            got = buf[np.argsort(buf[:, 0] >> 16, kind="stable")]
            bounds = np.searchsorted(got[:, 0] >> 16, np.arange(65537))
            for b in np.nonzero(np.diff(bounds))[0]:
                seg = lib.selftest_kmsort(got[bounds[b]:bounds[b + 1]], nw)
                lib._check(L_.mhb_selftest_r2s_s1_group(seg.ctypes.data, len(seg), K, M, LR, N, 1, planes[o, 0].ctypes.data,
                                                        planes[o, 1].ctypes.data, planes[o, 2].ctypes.data,
                                                        planes[o, 3].ctypes.data, counting.ctypes.data))
    assert seen == len(recs)
    # the plane merge and the mercy step over every share
    solid = np.zeros(N * LR, np.uint8)
    n_mercy = 0
    added = C.c_uint32()
    for s in range(W):
        if first[s] == first[s + 1]:
            continue
        w0, w_end = first[s] * LR // 32, first[s + 1] * LR // 32 + 2
        mine = planes[s].copy()
        for o in range(W):
            if o != s:
                mine[:, w0:w_end] |= planes[o][:, w0:w_end]
        mercy = np.zeros(bw, np.uint32)
        for r in range(first[s], first[s + 1]):
            lib._check(L_.mhb_selftest_r2s_mercy_read(LR, N, r, K, mine[0].ctypes.data, mine[1].ctypes.data,
                                                      mine[2].ctypes.data, mine[3].ctypes.data, mercy.ctypes.data,
                                                      C.byref(added)))
            n_mercy += added.value
        bits = np.unpackbits((mine[0] | mercy).view(np.uint8), bitorder="little")
        solid[first[s] * LR:first[s + 1] * LR] = bits[first[s] * LR:first[s + 1] * LR]
    return solid, counting, n_mercy, plan["rounds"]


def loads(recs, per, first):
    """(records of the largest owner, of the largest leading byte, of the largest bucket)"""
    h = owner_hists(recs, per, first)
    tot = h.sum(axis=0)
    plan = lib.plan_count_owner_rounds(h)
    most = max(int(tot[a:c + 1].sum()) for a, c in plan["owners"])
    return most, int(tot.reshape(256, 256).sum(axis=1).max()), int(tot.max())


@pytest.mark.parametrize("n_ranks", [2, 3])
@pytest.mark.parametrize("div", [3, 7, "byte"])
def test_rounds_match_oracle(deep, n_ranks, div):
    recs, per, want = deep
    first = balanced(n_ranks)
    most, top_byte, top_bucket = loads(recs, per, first)
    if div == "byte":  # below the largest leading byte: that byte is cut on bucket ids
        assert top_bucket < top_byte
        cap = (top_bucket + top_byte) // 2
    else:
        cap = max(most // div, top_bucket)
    solid, counting, n_mercy, R = rounds_stage1(recs, per, first, cap, range(n_ranks))
    assert R > 1
    assert n_mercy == want["n_mercy"]
    assert (counting == want["counting"]).all()
    assert (solid == np.unpackbits(want["is_solid"], bitorder="little")[:N * LR]).all()


def test_rounds_out_of_read_order_differ(deep):
    """the same rounds with the ranks' blocks of every round in reverse order: the owners' kmsort sees another tie order"""
    recs, per, want = deep
    first = balanced(2)
    most, _, top_bucket = loads(recs, per, first)
    solid, counting, n_mercy, R = rounds_stage1(recs, per, first, max(most // 3, top_bucket), [1, 0])
    assert R > 1
    assert not (solid == np.unpackbits(want["is_solid"], bitorder="little")[:N * LR]).all() or n_mercy != want["n_mercy"]


def test_a_bucket_above_the_cap_is_refused(deep):
    recs, per, _ = deep
    first = balanced(2)
    _, _, top_bucket = loads(recs, per, first)
    with pytest.raises(lib.MhbError, match=r"libmhb error 4: bucket 0x[0-9a-f]{4} alone holds \d+ records, more than one "
                                           r"round of rank \d can take"):
        lib.plan_count_owner_rounds(owner_hists(recs, per, first), top_bucket - 1)
