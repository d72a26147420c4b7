"""count on several GPUs (mhb_count_run_multi) without a GPU: the owner and round plan every rank computes from the
all-gathered bucket histograms (mhb_plan_count_owner_rounds), and the read shares on variable-length images.

Each owner's bucket range is cut greedily into ascending sub-ranges that fit one round; a leading byte that alone
exceeds a round is cut on bucket ids; a single bucket above the cap is an error.  The rounds are as many as the owner
with the most sub-ranges needs, the others get empty ranges at the end, and every rank knows where its block of every
(round, owner) pair starts in the owner's receive buffer."""
import numpy as np
import pytest

from megahit_b200 import lib
from megahit_b200.lib import MhbError


def skewed_hists(n_ranks, seed, total=200000):
    """n_ranks bucket histograms with the skew of canonical (k+1)-mers: heavy towards A-prefixes, many empty buckets"""
    rng = np.random.default_rng(seed)
    w = np.exp(-np.arange(65536) / 9000.0) * (rng.random(65536) < 0.6)
    w[0] *= 40  # a poly-A bucket
    h = np.zeros((n_ranks, 65536), np.uint64)
    for r in range(n_ranks):
        h[r] = rng.multinomial(total // n_ranks + r * 17, w / w.sum()).astype(np.uint64)
    return h


def owner_sub_ranges(plan, o):
    return [(int(plan["lo"][t, o]), int(plan["hi"][t, o])) for t in range(plan["rounds"])
            if plan["lo"][t, o] <= plan["hi"][t, o]]


def greedy(tot, lo, hi, cap):
    """the cut of one owner's buckets [lo, hi], restated: whole leading bytes, bucket ids inside an oversized byte"""
    out, start, acc = [], lo, 0
    atoms = []
    for B in range(lo >> 8, (hi >> 8) + 1):
        bt = int(tot[B << 8:(B + 1) << 8].sum())
        atoms += [(B << 8, bt)] if bt <= cap else [((B << 8) | c, int(tot[(B << 8) | c])) for c in range(256)]
    for a, cnt in atoms:
        assert cnt <= cap
        if acc + cnt > cap:
            out.append((start, a - 1))
            start, acc = a, 0
        acc += cnt
    out.append((start, hi))
    return out


@pytest.mark.parametrize("n_ranks", [2, 3, 5])
@pytest.mark.parametrize("frac", [1.0, 1 / 3, 1 / 7, 1 / 40])
def test_sub_ranges_tile_each_owner_and_fit_the_cap(n_ranks, frac):
    h = skewed_hists(n_ranks, seed=n_ranks)
    tot = h.sum(axis=0).astype(np.int64)
    free = lib.plan_count_owner_rounds(h)
    biggest = max(int(tot[a:b + 1].sum()) for a, b in free["owners"])
    cap = max(int(biggest * frac), int(tot.max()))
    plan = lib.plan_count_owner_rounds(h, cap)
    assert plan["owners"] == free["owners"]
    R = plan["rounds"]
    assert R == max(len(owner_sub_ranges(plan, o)) for o in range(n_ranks))
    if frac < 1:
        assert R > 1
    for o, (olo, ohi) in enumerate(plan["owners"]):
        sub = owner_sub_ranges(plan, o)
        # ascending, exactly tiling the owner's bucket range
        assert sub[0][0] == olo and sub[-1][1] == ohi
        assert all(b[0] == a[1] + 1 for a, b in zip(sub, sub[1:]))
        assert all(a <= b for a, b in sub)
        # within the cap, and the greedy cut restated
        for a, b in sub:
            assert int(tot[a:b + 1].sum()) <= cap or a == b
        assert sub == greedy(tot, olo, ohi, cap)
        # the rounds beyond the owner's sub-ranges are empty
        for t in range(len(sub), R):
            assert plan["lo"][t, o] > plan["hi"][t, o]
            assert (plan["n"][t, o] == 0).all()


def test_oversized_leading_byte_is_cut_on_bucket_ids():
    h = np.zeros((2, 65536), np.uint64)
    h[0, 0x0000:0x0100] = 30  # leading byte 0x00: 7680 + 7680 records
    h[1, 0x0000:0x0100] = 30
    h[0, 0x4000:0x4100] = 1
    h[1, 0xc000] = 50
    cap = 1000
    plan = lib.plan_count_owner_rounds(h, cap)
    sub = owner_sub_ranges(plan, 0)
    cuts = [a for a, _ in sub[1:]]
    assert cuts and any(a & 255 for a in cuts)  # cuts inside byte 0x00
    assert all(a < 0x100 for a in cuts)          # and only there: the other bytes fit whole
    for a, b in sub:
        assert int(h[:, a:b + 1].sum()) <= cap


def test_a_single_bucket_above_the_cap_is_an_error_naming_it():
    h = np.zeros((3, 65536), np.uint64)
    h[:, 0x0000] = 400  # every record in bucket 0x0000 (poly-A)
    h[1, 0x8123] = 5
    with pytest.raises(MhbError) as e:
        lib.plan_count_owner_rounds(h, 1199)
    msg = str(e.value)
    assert "bucket 0x0000" in msg and "rank 0" in msg and "1200" in msg
    assert lib.plan_count_owner_rounds(h, 1200)["rounds"] == 1


@pytest.mark.parametrize("n_ranks,cap", [(2, 5000), (3, 3000), (4, 20000), (5, 900)])
def test_block_offsets_equal_a_recount(n_ranks, cap):
    h = skewed_hists(n_ranks, seed=10 + n_ranks)
    cap = max(cap, int(h.sum(axis=0).max()))
    plan = lib.plan_count_owner_rounds(h, cap)
    for t in range(plan["rounds"]):
        for o in range(n_ranks):
            lo, hi = int(plan["lo"][t, o]), int(plan["hi"][t, o])
            at = 0
            for s in range(n_ranks):
                want = int(h[s, lo:hi + 1].sum()) if lo <= hi else 0
                assert int(plan["n"][t, o, s]) == want
                assert int(plan["off"][t, o, s]) == at
                at += want
    # every record of every rank is sent exactly once
    assert (plan["n"].sum(axis=(0, 1)) == h.sum(axis=1)).all()


@pytest.mark.parametrize("n_ranks", [2, 3, 8])
def test_no_cap_is_one_round_of_the_owner_ranges(n_ranks):
    h = skewed_hists(n_ranks, seed=30 + n_ranks)
    plan = lib.plan_count_owner_rounds(h)
    assert plan["rounds"] == 1
    # the owner ranges of the other multi-GPU stages, from the histogram of all ranks
    assert plan["owners"] == lib.plan_r2s_owners(h.sum(axis=0), n_ranks)
    assert [(int(a), int(b)) for a, b in zip(plan["lo"][0], plan["hi"][0])] == plan["owners"]
    assert plan["owners"][0][0] == 0 and plan["owners"][-1][1] == 65535


def test_empty_histograms():
    h = np.zeros((3, 65536), np.uint64)
    plan = lib.plan_count_owner_rounds(h, 10)
    assert plan["rounds"] == 1 and (plan["n"] == 0).all()


def var_image(lengths, seed):
    rng = np.random.default_rng(seed)
    out = []
    for L in lengths:
        out.append(L)
        out += list(rng.integers(0, 1 << 32, size=(L + 15) // 16, dtype=np.uint64).astype(np.uint32))
    return np.array(out, np.uint32)


@pytest.mark.parametrize("n_ranks", [2, 3, 7])
def test_read_shares_on_variable_length_images(n_ranks):
    rng = np.random.default_rng(n_ranks)
    lengths = rng.integers(0, 301, size=500)
    lengths[::7] = 0  # reads TrimN cut to nothing
    lengths[:n_ranks] = 0
    b = var_image(lengths, seed=n_ranks)
    first = lib.plan_read_shares(b, len(lengths), n_ranks)
    assert first[0] == 0 and first[-1] == len(lengths) and all(a <= c for a, c in zip(first, first[1:]))
    cum = np.concatenate([[0], np.cumsum(lengths)])
    total = int(cum[-1])
    for r in range(1, n_ranks):  # every cut lies within one read's bases of its ideal position
        assert abs(int(cum[first[r]]) - total * r // n_ranks) <= max(int(lengths.max()), 1)


def test_read_shares_of_exactly_n_reads():
    b = var_image([40, 0, 35], seed=1)
    first = lib.plan_read_shares(b, 3, 3)
    assert first[0] == 0 and first[-1] == 3 and first == sorted(first)
