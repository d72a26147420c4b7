"""Every planning entry point of libmhb (mhb_plan.cpp, host logic only) against a restatement of its two rules.

Greedy cut: atoms in order; a run closes before an atom when it holds weight and the atom would take it past the
target; an atom above the limit is an error.  Owner rule: bound r is the leading byte whose cumulative count is closest
to r / world of the total, leaving at least one byte for every later rank.  Rounds cut whole leading bytes, and the
buckets of a byte that alone exceeds the cap; chunks cut reads or sequences with no limit; mercy segments cut leading
bytes of edges with a target at or below the limit."""
import numpy as np
import pytest

from megahit_b200 import lib
from megahit_b200.lib import MhbError

INF = 2**64


def greedy_cut(weights, target, limit=INF):
    """the first atom of every run after the first, or ("bad", i) for the first atom above limit"""
    cuts, acc = [], 0
    for i, w in enumerate(weights):
        if w > limit:
            return ("bad", i)
        if acc and acc + w > target:
            cuts.append(i)
            acc = 0
        acc += w
    return cuts


def owner_bounds(total256, world):
    cum = np.concatenate([[0], np.cumsum(np.asarray(total256, dtype=object))])
    bounds = [0]
    for r in range(1, world):
        target = int(cum[256]) * r // world
        cands = range(bounds[-1] + 1, 256 - (world - r) + 1)
        bounds.append(min(cands, key=lambda c: (abs(int(cum[c]) - target), c)))
    return bounds + [256]


def bucket_rounds(h256, h16, byte_lo, byte_hi, cap):
    """ranges of bucket ids over [byte_lo, byte_hi), or ("bad", bucket)"""
    atoms = []
    for b in range(byte_lo, byte_hi):
        split = h16 is not None and h256[b] > cap
        atoms += [((b << 8) | c, int(h16[(b << 8) | c])) for c in range(256)] if split else [(b << 8, int(h256[b]))]
    cuts = greedy_cut([w for _, w in atoms], cap, cap)
    if cuts and cuts[0] == "bad":
        return ("bad", atoms[cuts[1]][0])
    starts = [byte_lo << 8] + [atoms[i][0] for i in cuts]
    return list(zip(starts, [s - 1 for s in starts[1:]] + [(byte_hi << 8) - 1]))


def hist(rng, n, scale):
    """counts with empty stretches between full ones, sometimes one spike or nothing at all"""
    kind = rng.integers(0, 5)
    h = np.zeros(n, np.uint64)
    if kind == 0:
        return h
    if kind == 1:  # a single bucket holding everything
        h[rng.integers(0, n)] = rng.integers(1, 50 * scale)
        return h
    h[:] = rng.integers(0, scale + 1, n)
    h[rng.random(n) < rng.random()] = 0
    return h


def cap_near(rng, h):
    """a cap at exactly one atom's count, one below it, or at random"""
    v = [int(x) for x in h if x] or [1]
    c = max(v) if rng.random() < 0.5 else v[rng.integers(0, len(v))]
    return max(1, [c, c - 1, int(rng.integers(1, 2 * c + 2)), sum(v)][rng.integers(0, 4)])


@pytest.mark.parametrize("seed", range(4))
def test_rounds_and_rounds16(seed):
    rng = np.random.default_rng(seed)
    for _ in range(150):
        h = hist(rng, 256, int(rng.choice([3, 100])))
        cap = cap_near(rng, h)
        want = bucket_rounds(h, None, 0, 256, cap)
        if want[0] == "bad":
            with pytest.raises(MhbError, match=f"leading byte 0x{want[1] >> 8:02x} .*more than one round can take"):
                lib.plan_rounds(h, cap)
            with pytest.raises(MhbError, match=f"leading byte 0x{want[1] >> 8:02x} .*more than one round can take"):
                lib.plan_rounds16(h, None, cap)
        else:
            assert lib.plan_rounds(h, cap) == [(lo >> 8, hi >> 8) for lo, hi in want]
            assert lib.plan_rounds16(h, None, cap) == want
        sub = np.zeros((256, 256), np.uint64)
        for b in np.nonzero(h > cap)[0]:
            sub[b] = rng.multinomial(int(h[b]), rng.dirichlet(np.full(256, rng.choice([0.05, 1.0]))))
        want = bucket_rounds(h, sub.reshape(-1), 0, 256, cap)
        if want[0] == "bad":
            with pytest.raises(MhbError, match=f"bucket 0x{want[1]:04x} .*more than one round can take"):
                lib.plan_rounds16(h, sub, cap)
            continue
        assert lib.plan_rounds16(h, sub, cap) == want
        assert lib.plan_rounds16(h, sub, cap, cap=len(want)) == want
        if len(want) > 1:  # cap_out overflow
            with pytest.raises(MhbError, match=f"round plan needs more than {len(want) - 1} ranges"):
                lib.plan_rounds16(h, sub, cap, cap=len(want) - 1)


def test_round_errors_name_the_byte_and_the_bucket():
    h = np.zeros(256, np.uint64)
    h[3] = 1000
    with pytest.raises(MhbError, match="leading byte 0x03 .*more than one round can take"):
        lib.plan_rounds(h, 999)
    sub = np.zeros((256, 256), np.uint64)
    sub[3, 9] = 1000
    with pytest.raises(MhbError, match="bucket 0x0309 .*more than one round can take"):
        lib.plan_rounds16(h, sub, 999)
    assert lib.plan_rounds16(h, sub, 1000) == [(0, 65535)]
    assert lib.plan_rounds(np.zeros(256, np.uint64), 1) == [(0, 255)]


@pytest.mark.parametrize("seed", range(3))
def test_owners_and_count_owner_rounds(seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(25):
        W = int(rng.integers(1, 17))
        hs = np.zeros((W, 65536), np.uint64)
        for s in range(W):
            if rng.random() < 0.8:  # otherwise a rank with no records
                hs[s] = hist(rng, 65536, int(rng.choice([2, 40])))
        tot = hs.sum(0)
        bounds = owner_bounds(tot.reshape(256, 256).sum(1), W)
        owners = [(bounds[o] << 8, (bounds[o + 1] << 8) - 1) for o in range(W)]
        assert lib.plan_r2s_owners(tot, W) == owners
        cap = 0 if rng.random() < 0.3 else cap_near(rng, np.concatenate([tot[tot > 0], tot.reshape(256, 256).sum(1)]))
        subs = [bucket_rounds(tot.reshape(256, 256).sum(1), tot, bounds[o], bounds[o + 1], cap or INF) for o in range(W)]
        bad = [(o, s[1]) for o, s in enumerate(subs) if s[0] == "bad"]
        if bad:
            o, b = bad[0]
            with pytest.raises(MhbError, match=f"bucket 0x{b:04x} .*round of rank {o} can take \\({cap}\\)"):
                lib.plan_count_owner_rounds(hs, cap)
            continue
        plan = lib.plan_count_owner_rounds(hs, cap)
        assert plan["owners"] == owners
        assert plan["rounds"] == max(len(s) for s in subs)
        pre = np.concatenate([np.zeros((W, 1), np.uint64), np.cumsum(hs, axis=1, dtype=np.uint64)], axis=1)
        for t in range(plan["rounds"]):
            for o in range(W):
                if t >= len(subs[o]):
                    assert plan["lo"][t, o] > plan["hi"][t, o] and not plan["n"][t, o].any()
                    continue
                a, b = subs[o][t]
                assert (plan["lo"][t, o], plan["hi"][t, o]) == (a, b)
                n = pre[:, b + 1] - pre[:, a]
                assert list(plan["n"][t, o]) == list(n)
                assert list(plan["off"][t, o]) == list(np.concatenate([[0], np.cumsum(n)[:-1]]))


def test_owners_of_empty_and_single_bucket_histograms():
    for W in range(1, 17):
        h = np.zeros(65536, np.uint64)
        assert lib.plan_r2s_owners(h, W) == [(o << 8, ((o + 1) << 8) - 1) for o in range(W - 1)] + [((W - 1) << 8, 65535)]
        h[0x4000] = 7
        assert lib.plan_r2s_owners(h, W)[-1][1] == 65535


def shares(weights, n_ranks):
    """cut r at the item boundary whose weight before it is closest to r / n_ranks of the total (ties: the earlier)"""
    total, first, b, cum = sum(weights), [0], 0, 0
    for r in range(1, n_ranks):
        target = total * r // n_ranks
        while b < len(weights) and cum + weights[b] <= target:
            cum, b = cum + weights[b], b + 1
        if b < len(weights) and cum < target and cum + weights[b] - target < target - cum:
            cum, b = cum + weights[b], b + 1
        first.append(b)
    return first + [len(weights)]


def read_image(lengths):
    words = []
    for L in lengths:
        words += [int(L)] + [0x1B1B1B1B] * ((int(L) + 15) // 16)
    return np.array(words, np.uint32)


@pytest.mark.parametrize("seed", range(3))
def test_shares_and_chunks(seed):
    rng = np.random.default_rng(200 + seed)
    for _ in range(60):
        n = int(rng.choice([0, 1, 7, 200]))
        lengths = np.full(n, int(rng.integers(1, 200))) if rng.random() < 0.3 else rng.integers(0, 300, n)
        b = read_image(lengths)  # zero-length reads included
        W = int(rng.integers(1, 17))
        assert lib.plan_read_shares(b, n, W) == shares([int(x) for x in lengths], W)
        cap = int(rng.choice([1, 8, 40, 500, 10**6]))
        per = [4 * (1 + (int(x) + 15) // 16) for x in lengths]
        if n and (lengths == lengths[0]).all() and lengths[0]:  # fixed length: cut in closed form
            step = max(1, cap // per[0])
            want = list(range(0, n, step)) + [n]
        else:
            want = [0] + greedy_cut(per, cap) + ([n] if n else [])
        assert lib.plan_read_chunks(b, n, cap) == want
        k = int(rng.integers(9, 120))
        lens = rng.integers(0, 300, n).astype(np.uint32)
        assert lib.plan_seq_shares(lens, k, W) == shares([2 * (int(x) - k + 2) if x >= k + 1 else 0 for x in lens], W)
        word_off = np.concatenate([[0], np.cumsum((lens.astype(np.uint64) + 15) // 16)]).astype(np.uint64)
        per = [4 * int(word_off[i + 1] - word_off[i]) + 22 for i in range(n)]
        assert lib.plan_seq_chunks(word_off, lens, k, cap) == [0] + greedy_cut(per, cap) + ([n] if n else [])


@pytest.mark.parametrize("seed", range(3))
def test_mercy_segments(seed):
    rng = np.random.default_rng(300 + seed)
    for _ in range(80):
        k = int(rng.integers(12, 256))
        WE = (2 * (k + 1) + 16 + 31) // 32
        per_byte = hist(rng, 256, int(rng.choice([1, 6])))
        e = np.zeros((int(per_byte.sum()), WE), np.uint32)
        e[:, 0] = np.repeat(np.arange(256, dtype=np.uint32), per_byte.astype(np.int64)) << 24
        size = [int(x) * WE * 4 for x in per_byte]
        cap = cap_near(rng, size)
        want = greedy_cut(size, cap, cap)
        if want and want[0] == "bad":
            b = want[1]
            with pytest.raises(MhbError, match=f"leading byte 0x{b:02x} .*more than one mercy segment can take \\({cap} bytes"):
                lib.plan_mercy_segments(e, k, cap)
        else:
            assert lib.plan_mercy_segments(e, k, cap) == [0] + want + [256]


def test_mercy_byte_above_target_within_limit():
    """without a cap, segments are packed to 1 GiB, and a larger byte that fits a device slot is a segment of its own"""
    k, WE, gib = 27, 2, 1 << 30
    per_byte = np.zeros(256, np.uint64)
    per_byte[[1, 2, 5]] = [gib // 32, gib // 8 + 1, gib // 32]  # 1/4 GiB, 1 GiB + 8 bytes, 1/4 GiB of edges
    plan = lib.mercy_auto_plan(per_byte, k, 10, 1000, 150, 80 * gib)
    # the empty byte 3 after the oversized one still closes it (its run holds more than the target)
    assert plan["first"] == [0] + greedy_cut([int(x) * WE * 4 for x in per_byte], gib) + [256] == [0, 2, 3, 256]
    assert plan["slot_bytes"] >= (gib // 8 + 1) * WE * 4
    with pytest.raises(MhbError, match="leading byte 0x02 .*more than one mercy segment can take"):
        lib.mercy_auto_plan(per_byte, k, 10, 1000, 150, 2 * gib)
