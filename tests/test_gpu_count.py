"""Both count paths - mhb_count_solid_hashed (partition + per-slice hash aggregation) and mhb_sort_records +
mhb_count_solid (full sort + run-length count) - against the exact NumPy reference of A5 (tests/count_reference.py):
edges, aux flags, the whole multiplicity histogram and the solid count, record by record.

The adversarial cases are built around the constants of k_hash_count (megahit_b200/csrc/mhb_hashcount.cu); each case
asserts, on its own input, the property it exists for, so that it cannot silently stop testing it when a constant moves.
Adversarial keys of a case share one 24-bit prefix group: slices are key-closed at that prefix, so the keys land in one
slice whatever the slice length."""
import ctypes as C

import numpy as np
import pytest

from count_reference import count_records_reference, make_records, records_from_tallies
from megahit_b200 import lib, synth

pytestmark = pytest.mark.gpu

# ---- k_hash_count constants (mhb_hashcount.cu: HcGeomB = HcGeom<512, 12, 2>) ----
SLOTS = 4096          # table slots (1 << LOG_SLOTS)
MAX_SOLID = 1024      # solid keys per sub-range (SLOTS / 4); more -> the sub-range is split
HOT = 256             # kHcHotCount: keys this frequent get exact 32-bit tallies
HOT_ROUND = 32        # kHcHotRound: hot keys per extra sweep
SLICE = 7495          # records per slice (SLOTS * 1.83)
MAX_PROBES = 48       # kHcMaxProbes: a longer probe sequence = table overflow
REM_BITS = 42         # record bits 47..6 key the table
MAX_M = 1024          # kHcHist: hashed path supports 1 <= m <= 1024


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


# ------------------------------------------------------------------------------------------------
# running the two paths
# ------------------------------------------------------------------------------------------------
def _dev_recs(recs):
    torch = _torch()
    flat = np.concatenate([np.ascontiguousarray(recs, np.uint32).reshape(-1), np.zeros(4, np.uint32)])
    a = torch.from_numpy(flat.view(np.int32)).cuda()
    return a, torch.empty_like(a)


def run_count(recs, k, m, hashed, cap=None, room=None, sentinel=False, hist_byte5=None, ws=None):
    """One call of a count path on `recs` (numpy, any order) with capacity_edges = cap.  The output buffers hold `room`
    (default cap) entries, filled with 0xA5 bytes when sentinel is set.  Returns (edges (room, we), aux (room,),
    mul_hist, n_solid) with the whole output buffers, so that callers can check what lies past the solid edges."""
    torch = _torch()
    from megahit_b200 import dev
    L = lib.load()
    n, wr = recs.shape
    we = lib.words_per_edge(k)
    cap = n // m + 1 if cap is None else cap
    room = cap if room is None else room
    a, b = _dev_recs(recs)
    edges = torch.full((room * we + 4,), -0x5A5A5A5B if sentinel else 0, dtype=torch.int32, device="cuda")
    aux = torch.full((room + 4,), 0xA5 if sentinel else 0, dtype=torch.uint8, device="cuda")
    hist = torch.zeros(65536, dtype=torch.int64, device="cuda")
    ns = torch.zeros(8, dtype=torch.int64, device="cuda")
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    if hashed:
        if ws is None:
            ws = torch.empty(L.mhb_count_hashed_workspace_bytes(n, k, m), dtype=torch.uint8, device="cuda")
        h5 = None if hist_byte5 is None else torch.from_numpy(hist_byte5.astype(np.int64)).cuda()
        lib._check(L.mhb_count_solid_hashed(None, ptr(a), ptr(b), n, k, m, ptr(h5), ptr(edges), ptr(aux), cap, ptr(hist),
                                            ptr(ns), ptr(ws), ws.numel()))
    else:
        srt = dev.sort_records(a, b, n, wr, lib.count_sort_bytes(k))
        sc = torch.empty(max(1, L.mhb_count_solid_scratch_bytes(n)), dtype=torch.uint8, device="cuda")
        lib._check(L.mhb_count_solid(None, ptr(srt), n, k, m, ptr(edges), ptr(aux), cap, ptr(hist), ptr(ns), ptr(sc),
                                     sc.numel()))
    torch.cuda.synchronize()
    e = edges[: room * we].cpu().numpy().view(np.uint32).reshape(room, we)
    return e, aux[:room].cpu().numpy(), hist.cpu().numpy(), int(ns[0].item())


def check_against_reference(recs, k, m, paths=("hashed", "sort")):
    """Both paths == the reference on recs (given to the device in a fresh random order)"""
    rng = np.random.default_rng(len(recs) * 31 + k * 7 + m)
    recs = recs[rng.permutation(len(recs))]
    ref_e, ref_a, ref_h, ref_n = count_records_reference(recs, k, m)
    for path in paths:
        e, a, h, n = run_count(recs, k, m, hashed=path == "hashed")
        assert n == ref_n, (path, n, ref_n)
        assert (e[:n] == ref_e).all(), (path, "edges", int((e[:n] != ref_e).any(axis=1).sum()))
        bad = np.nonzero(a[:n] != ref_a)[0]
        assert len(bad) == 0, (path, "aux", len(bad), [(ref_e[i].tolist(), int(a[i]), int(ref_a[i])) for i in bad[:5]])
        assert (h == ref_h).all(), (path, "mul_hist", [(int(i), int(h[i]), int(ref_h[i])) for i in np.nonzero(h != ref_h)[0][:8]])
    return ref_e, ref_a, ref_h, ref_n


# ------------------------------------------------------------------------------------------------
# building adversarial key sets
# ------------------------------------------------------------------------------------------------
def rem42(keys):
    """the 42 record bits (47..6) that key the hash table"""
    return (np.asarray(keys, np.uint64) >> np.uint64(6)) & np.uint64((1 << REM_BITS) - 1)


def distinct(rng, n, bits):
    out = np.zeros(0, np.uint64)
    while len(out) < n:
        out = np.unique(np.concatenate([out, rng.integers(0, 1 << bits, 2 * n, dtype=np.uint64)]))
    return out[rng.permutation(len(out))[:n]]


def group_keys(rng, prefix24, n, k):
    """n distinct (k+1)-mers (uint64, left-aligned, valid for k) in the 24-bit prefix group `prefix24`"""
    free = 2 * (k + 1) - 24
    return (np.uint64(prefix24) << np.uint64(40)) | (distinct(rng, n, free) << np.uint64(64 - 2 * (k + 1)))


def fits_table(keys) -> bool:
    """True when these distinct keys are certain to fit k_hash_count's table without overflow: linear probing leaves
    the same occupied slots in any insertion order, and no probe sequence is longer than the longest cluster + 1."""
    r = rem42(keys)
    if len(r) >= SLOTS:
        return False
    homes = ((r * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(64 - 12)).astype(np.int64).tolist()
    occ = bytearray(SLOTS)
    for h in homes:
        while occ[h]:
            h = (h + 1) & (SLOTS - 1)
        occ[h] = 1
    start = occ.index(0)  # walk the ring from an empty slot
    run = longest = 0
    for i in range(SLOTS):
        if occ[(start + i) & (SLOTS - 1)]:
            run += 1
            longest = max(longest, run)
        else:
            run = 0
    return longest + 1 <= MAX_PROBES


def tally_row(rng, c, m, kind):
    """prev (or next) tallies over 0..3 and 4 (none) summing to c; a kind that needs more than c occurrences falls
    back to "random\""""
    need = {"wrap256": 256, "wrap512": 256, "wrap_below_m": 256 + m - 1, "exact_m": m, "below_m": 4 * (m - 1)}
    if c < need.get(kind, 0):
        kind = "random"
    if kind == "random":
        return np.bincount(rng.choice(5, c, p=rng.dirichlet(np.ones(5))), minlength=5)
    t = np.zeros(5, np.int64)
    b = int(rng.integers(0, 4))
    if kind == "wrap256":    # a byte tally wraps to 0
        t[b] = 256
    elif kind == "wrap512":
        t[b] = 512 if c >= 512 else 256
    elif kind == "wrap_below_m":  # wraps to m - 1 < m
        t[b] = 256 + m - 1
    elif kind == "exact_m":  # exactly m on a single base
        t[b] = m
    elif kind == "below_m":
        t[:4] = m - 1
    t[4] = c - t[:4].sum()  # kind "none": every neighbour is 4
    assert t.sum() == c and (t >= 0).all(), (kind, c, t)
    return t


HOT_KINDS = ["wrap256", "wrap512", "wrap_below_m", "none", "exact_m", "below_m", "random"]


def hot_tallies(rng, counts, m, kinds=HOT_KINDS):
    pt = np.array([tally_row(rng, int(c), m, kinds[int(rng.integers(0, len(kinds)))]) for c in counts])
    nt = np.array([tally_row(rng, int(c), m, kinds[int(rng.integers(0, len(kinds)))]) for c in counts])
    return pt, nt


def flags(t, m):
    return (t[:, :4] >= m).any(axis=1)


def byte_flags(t, m):
    return ((t[:, :4] & 255) >= m).any(axis=1)


def random_records(rng, keys, counts, k):
    """records of keys repeated counts times, prev / next uniform over 0..4"""
    kk = np.repeat(np.asarray(keys, np.uint64), counts)
    return make_records(kk, rng.integers(0, 5, len(kk)), rng.integers(0, 5, len(kk)), k)


def key_of(recs):
    return ((recs[:, 0].astype(np.uint64) << np.uint64(32)) | recs[:, 1].astype(np.uint64)) & ~np.uint64(63)


def key_counts(recs):
    return np.unique(key_of(recs), return_counts=True)


# ------------------------------------------------------------------------------------------------
# adversarial cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 3])
def test_hot_flags(m):
    """~100 hot keys in one group whose exact prev / next answer differs from the byte-wrapped one: tallies of 256 /
    512 (wrap to 0), 256 + m - 1 (wraps below m), no prev at all, exactly m on one base; more than one hot round"""
    rng = np.random.default_rng(100 + m)
    k = 27
    keys = group_keys(rng, 0x3A51C7, 400, k)
    hot_keys, cold_keys = keys[:100], keys[100:]
    counts = rng.integers(HOT + 8, 1500, len(hot_keys))
    pt, nt = hot_tallies(rng, counts, m)
    recs = np.concatenate([records_from_tallies(hot_keys, pt, nt, k),
                           random_records(rng, cold_keys, rng.integers(1, 2 * m + 2, len(cold_keys)), k)])
    # the properties this case exists for
    assert (counts >= HOT).sum() >= 40 and len(hot_keys) > 3 * HOT_ROUND
    for t in (pt, nt):
        wrapped = flags(t, m) & ~byte_flags(t, m)
        assert wrapped.sum() >= 5, "exact tallies >= m that a byte would wrap below m"
        assert ((t[:, :4] == m).any(axis=1) & ((t[:, :4] <= m).all(axis=1))).sum() >= 3, "exactly m on a single base"
    assert (pt[:, 4] == counts).sum() >= 3, "hot keys without any prev"
    assert ((~flags(pt, m)) | (~flags(nt, m))).sum() > HOT_ROUND + 8, "flagged hot keys beyond the first hot round"
    assert fits_table(keys), "the group must not overflow: the hot sweeps run on the slice itself"
    check_against_reference(recs, k, m)


@pytest.mark.parametrize("m", [2, 256])
def test_hot_boundary(m):
    """counts 255, 256, 257 (the hot threshold) with a single-base tally equal to the count, all else 4"""
    rng = np.random.default_rng(200 + m)
    k = 27
    counts = np.repeat([HOT - 1, HOT, HOT + 1], 12)
    keys = group_keys(rng, 0x00C0DE, len(counts), k)
    pt = np.zeros((len(counts), 5), np.int64)
    nt = np.zeros((len(counts), 5), np.int64)
    for i, c in enumerate(counts):
        side = (pt, nt) if i % 2 == 0 else (nt, pt)
        side[0][i, i % 4] = c  # one base carries every occurrence ...
        side[1][i, 4] = c      # ... the other side has no neighbour at all
    recs = records_from_tallies(keys, pt, nt, k)
    assert sorted(set(key_counts(recs)[1].tolist())) == [HOT - 1, HOT, HOT + 1]
    _, aux, _, n = check_against_reference(recs, k, m)
    assert n == (len(counts) if m <= HOT - 1 else 24) and set(aux.tolist()) == {1, 2}


def test_hot_in_split():
    """~1100 hot keys in one group: MAX_SOLID splits it, and the hot sweeps run in children with a key prefix"""
    rng = np.random.default_rng(300)
    k, m = 27, 2
    keys = group_keys(rng, 0x7F0123, 1100, k)
    counts = rng.integers(HOT, HOT + 60, len(keys))
    pt, nt = hot_tallies(rng, counts, m)
    recs = records_from_tallies(keys, pt, nt, k)
    assert len(keys) > MAX_SOLID and fits_table(keys), "split on MAX_SOLID, not on overflow"
    child = rem42(keys) >> np.uint64(REM_BITS - 10)  # first split level whose children partition the group
    per_child = np.bincount(np.unique(child, return_inverse=True)[1])
    assert per_child.max() <= MAX_SOLID and per_child.min() > HOT_ROUND, per_child
    check_against_reference(recs, k, m)


def test_max_solid_edge():
    """one group with exactly MAX_SOLID solid keys (no split) and one with MAX_SOLID + 1 (split after the judge has
    histogrammed the keys: the children must not count them again), each with non-solid keys of multiplicity 1..m-1"""
    rng = np.random.default_rng(400)
    k, m = 27, 3
    parts = []
    for prefix, n_solid in ((0x4100AA, MAX_SOLID), (0x4200AA, MAX_SOLID + 1)):  # different 16-bit buckets
        keys = group_keys(rng, prefix, n_solid + 400, k)
        counts = np.concatenate([rng.integers(m, m + 4, n_solid), rng.integers(1, m, 400)])
        assert (counts >= m).sum() == n_solid and fits_table(keys)
        parts.append(random_records(rng, keys, counts, k))
    check_against_reference(np.concatenate(parts), k, m)


@pytest.mark.parametrize("n_hot", [0, 40])
def test_deep_split(n_hot):
    """4096 solid keys whose remainders differ only in the low 12 bits (k = 28: every remainder bit is a key bit):
    overflow splits while other keys of the group still share the prefix, then a chain of splits ~16 levels deep down
    to four sub-ranges of exactly MAX_SOLID keys.  n_hot of them are hot"""
    rng = np.random.default_rng(500 + n_hot)
    k, m = 28, 2
    base = (np.uint64(0x5C3D1E) << np.uint64(40)) | (rng.integers(0, 1 << 22, dtype=np.uint64) << np.uint64(18))
    solid = base | (np.arange(4096, dtype=np.uint64) << np.uint64(6))
    # 2500 singletons sharing the top 20 remainder bits with them: the table overflows for the first ten levels
    noise = (base & ~np.uint64((1 << 28) - 1)) | (distinct(rng, 2500, 22) << np.uint64(6))
    noise = noise[(rem42(noise) >> np.uint64(12)) != (rem42(base) >> np.uint64(12))]
    counts = rng.integers(m, m + 3, len(solid))
    hot = rng.choice(len(solid), n_hot, replace=False)
    counts[hot] = rng.integers(HOT, HOT + 200, n_hot)
    pt, nt = hot_tallies(rng, counts, m, kinds=HOT_KINDS if n_hot else ["random"])
    recs = np.concatenate([records_from_tallies(solid, pt, nt, k), random_records(rng, noise, np.ones(len(noise), int), k)])
    r = rem42(solid)
    assert len(np.unique(r >> np.uint64(12))) == 1 and len(np.unique(r)) == 4096
    assert len(np.unique(np.concatenate([r, rem42(noise)]) >> np.uint64(22))) == 1 and len(solid) + len(noise) > SLOTS
    check_against_reference(recs, k, m)


def test_overflow_then_maxsolid():
    """~20 000 solid keys in one group: the table overflows, the sub-ranges split until they fit, then each still holds
    more than MAX_SOLID solid keys and splits again - the not-histogrammed-yet flag must survive both kinds of split"""
    rng = np.random.default_rng(600)
    k, m = 27, 2
    keys = group_keys(rng, 0x2B2B2B, 25_000, k)
    counts = np.concatenate([rng.integers(m, m + 2, 20_000), np.ones(5_000, int)])
    recs = random_records(rng, keys, counts, k)
    r = rem42(keys)
    at10 = np.bincount((r >> np.uint64(REM_BITS - 10)).astype(np.int64) & 3, minlength=4)
    assert at10.min() > SLOTS, "every 10-bit sub-range overflows"
    solid_keys = keys[counts >= m]
    sub12 = (r >> np.uint64(REM_BITS - 12)).astype(np.int64) & 15
    solid12 = np.bincount(sub12[counts >= m], minlength=16)
    assert solid12.min() > MAX_SOLID, "every 12-bit sub-range splits on MAX_SOLID"
    assert all(fits_table(keys[sub12 == s]) for s in range(16)), "... and not on overflow"
    assert len(solid_keys) == 20_000
    check_against_reference(recs, k, m)


@pytest.mark.parametrize("m", [2, MAX_M])
def test_clamp(m):
    """multiplicities 65534, 65535, 65536, 65537: the 16-bit clamp of the edge multiplicity and the histogram, while
    solidity uses the unclamped count"""
    rng = np.random.default_rng(700 + m)
    k = 27
    counts = np.array([65534, 65535, 65536, 65537, 1500, m, max(1, m - 1)])
    keys = group_keys(rng, 0x0FFFF0, len(counts), k)
    pt, nt = hot_tallies(rng, counts, m, kinds=["random", "wrap256", "exact_m", "none"])
    recs = records_from_tallies(keys, pt, nt, k)
    e, _, h, _ = check_against_reference(recs, k, m)
    assert h[65535] == 3 and h[65534] == 1 and (e[:, -1] & 0xFFFF).max() == 65535


@pytest.fixture(scope="module")
def reads_records_k27():
    """extracted k = 27 records of three read sets: 30x background, and two small genomes at ~270x and ~1000x"""
    torch = _torch()
    parts = []
    for n_reads, genome, seed in ((20_000, 100_000, 5), (2_900, 1_000, 6), (5_500, 500, 7)):
        b = synth.synth_reads_torch(n_reads, 150, genome, 0.01, seed, "cuda").reshape(-1)
        parts.append(extract(torch.cat([b, torch.zeros(8, dtype=torch.int32, device="cuda")]), n_reads, 150, 27))
    return np.concatenate(parts)


def extract(bin_dev, n_reads, read_len, k):
    """mhb_count_extract of a fixed-length library on the device -> (n, WR) uint32 records"""
    torch = _torch()
    wr = lib.count_record_words(k)
    n = n_reads * (read_len - k)
    a = torch.empty(n * wr + 4, dtype=torch.int32, device="cuda")
    rd = lib.DevReads(bin_dev.data_ptr(), bin_dev.numel(), n_reads, read_len, None, None)
    lib._check(lib.load().mhb_count_extract(None, C.byref(rd), k, C.c_void_p(a.data_ptr()), n, None, 0))
    torch.cuda.synchronize()
    return a[: n * wr].cpu().numpy().view(np.uint32).reshape(n, wr)


@pytest.mark.parametrize("m", [1, 2, 3, 255, 256, 257, 1023, MAX_M])
def test_m_sweep(reads_records_k27, m):
    """real extractions at thresholds around the hot count and the shared-memory histogram (multiplicities above 1023
    go to the global histogram)"""
    recs = reads_records_k27
    cnt = key_counts(recs)[1]
    if m > 3:
        assert ((cnt >= m - 16) & (cnt < m)).sum() > 0 and ((cnt >= m) & (cnt < m + 16)).sum() > 0, "keys on both sides of m"
    assert (cnt >= 1024).sum() > 0
    check_against_reference(recs, 27, m)


@pytest.mark.parametrize("k", [27, 28])
def test_bucket_extremes(k):
    """keys in bucket 0x0000 and 0xFFFF with remainders of all zeros and all ones (and their neighbours)"""
    rng = np.random.default_rng(800 + k)
    unit = np.uint64(1 << (64 - 2 * (k + 1)))
    ones = ~np.uint64(0)
    keys = np.array([0, unit, 2 * unit, 0x0000FFFFFFFFFFFF, 0xFFFF000000000000, ones, ones - unit, ones - 2 * unit,
                     0x00FFFFFFFFFFFFFF & ~np.uint64(0xFFFFFFFFFF), 0xFF00000000000000], np.uint64)
    keys = np.unique(keys & ~(unit - np.uint64(1)))
    counts = np.array([1, 2, 3, 300, 5, 600, 2, 1, 4, 7][: len(keys)])
    pt, nt = hot_tallies(rng, counts, 2, kinds=["random", "none", "exact_m"])
    recs = records_from_tallies(keys, pt, nt, k)
    top = recs[:, 0] >> 16
    assert (top == 0).any() and (top == 0xFFFF).any()
    assert ((recs[:, 1] & ~np.uint32(63)) == 0).any() and (key_of(recs) == (ones & ~(unit - np.uint64(1)))).any()
    check_against_reference(recs, k, 2)


def test_gauntlet():
    """~3 M records over ~3000 buckets, each with one pattern - ordinary keys, a table overflow, hot keys, a MAX_SOLID
    split, one key repeated past a slice (swallowed slices) - all permuted: a CTA meets overflowing, hot, empty and
    ordinary slices back to back (ticket pipeline, parity-indexed control words)"""
    rng = np.random.default_rng(900)
    k, m = 27, 2
    buckets = rng.permutation(65536)[:3000]
    plan = ["ordinary"] * 2790 + ["overflow"] * 60 + ["hot"] * 50 + ["maxsolid"] * 50 + ["swallow"] * 50
    parts, seen = [], set()
    for bkt, kind in zip(buckets, plan):
        prefix = (int(bkt) << 8) | int(rng.integers(0, 256))
        if kind == "ordinary":
            keys = np.concatenate([group_keys(rng, (int(bkt) << 8) | int(g), 25, k) for g in rng.choice(256, 6, replace=False)])
            parts.append(random_records(rng, keys, rng.integers(1, 7, len(keys)), k))
        elif kind == "overflow":
            keys = group_keys(rng, prefix, 6000, k)
            parts.append(random_records(rng, keys, rng.integers(1, 3, len(keys)), k))
        elif kind == "hot":
            keys = group_keys(rng, prefix, 40, k)
            counts = rng.integers(HOT, 420, len(keys))
            pt, nt = hot_tallies(rng, counts, m)
            parts.append(records_from_tallies(keys, pt, nt, k))
        elif kind == "maxsolid":
            keys = group_keys(rng, prefix, MAX_SOLID + 80, k)
            parts.append(random_records(rng, keys, rng.integers(m, m + 2, len(keys)), k))
        else:
            keys = group_keys(rng, prefix, 1, k)
            counts = rng.integers(SLICE + 1, 3 * SLICE, 1)
            pt, nt = hot_tallies(rng, counts, m, kinds=["random"])
            parts.append(records_from_tallies(keys, pt, nt, k))
        seen.add(kind)
    recs = np.concatenate(parts)
    assert 2_000_000 <= len(recs) <= 4_000_000 and len(seen) == 5
    _, cnt = np.unique(recs[:, 0] >> 8, return_counts=True)  # 24-bit groups
    assert (cnt > SLICE).sum() >= 50, "groups longer than a slice"
    check_against_reference(recs, k, m)


def _polya_reads(n_reads, seed):
    b = synth.synth_reads(n_reads, 150, 20_000, 0.01, seed=seed).copy()
    b[::2, 1:7] = 0            # every other read starts with 96 A's
    b[1::3, 4:10] = 0xFFFFFFFF  # and some carry long poly-T stretches
    return b


@pytest.mark.parametrize("k,polya", [(13, False), (14, False), (15, False), (17, False), (19, False), (20, False),
                                     (23, False), (25, False), (28, False), (13, True), (28, True)])
def test_k_sweep(k, polya):
    """every record geometry of the hashed path (k = 13: 28-bit keys, at most 16 keys per 24-bit group; k = 28: the
    key reaches record bit 6); poly-A reads make giant groups that swallow whole slices"""
    torch = _torch()
    n_reads = 10_000
    if polya:
        b = torch.from_numpy(_polya_reads(n_reads, 40 + k).reshape(-1).view(np.int32)).cuda()
    else:
        b = synth.synth_reads_torch(n_reads, 150, 50_000, 0.01, 30 + k, "cuda").reshape(-1)
    recs = extract(torch.cat([b, torch.zeros(8, dtype=torch.int32, device="cuda")]), n_reads, 150, k)
    assert lib.load().mhb_count_hashed_supported(k, 2) == 1
    if polya:
        _, cnt = np.unique(recs[:, 0] >> 8, return_counts=True)
        assert cnt.max() > 2 * SLICE, "a 24-bit group swallows slices"
    check_against_reference(recs, k, 2)


def test_sort_path_k31():
    """the same reference on 12-byte records (k = 31, sort path only: the hashed path needs 8-byte records)"""
    torch = _torch()
    n_reads = 8_000
    b = synth.synth_reads_torch(n_reads, 150, 40_000, 0.01, 31, "cuda").reshape(-1)
    recs = extract(torch.cat([b, torch.zeros(8, dtype=torch.int32, device="cuda")]), n_reads, 150, 31)
    assert recs.shape[1] == 3 and lib.load().mhb_count_hashed_supported(31, 2) == 0
    check_against_reference(recs, 31, 2, paths=("sort",))


# ------------------------------------------------------------------------------------------------
# end to end at every hashed k: count_host (extraction, hashed count, mercy marks) == the C oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [13, 15, 17, 19, 23, 25, 28])
def test_count_host_matches_oracle_across_k(k):
    import oracle_pipeline as OP
    from oracle import oracle as O
    n_reads, m = 3000, 2
    b = synth.synth_reads(n_reads, 150, 15_000, 0.01, seed=60 + k)
    reads = O.unpack_bin(b.tobytes(), reverse=True)
    oc = OP.oracle_count(reads, k, m)
    g = lib.count_host(b.reshape(-1), n_reads, k, m, want_mercy=True)
    assert g["n_solid"] == oc["n_solid"] > 0
    assert (g["edges"] == oc["edges"]).all()
    assert (g["counting"] == oc["counting"]).all()
    assert (g["cand_ids"] == oc["cand_ids"]).all() and len(oc["cand_ids"]) > 0


# ------------------------------------------------------------------------------------------------
# API contract
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed_records():
    rng = np.random.default_rng(1000)
    keys = rng.integers(0, 1 << 63, 40_000, dtype=np.uint64) << np.uint64(1)
    return random_records(rng, keys, rng.integers(1, 5, len(keys)), 27)


@pytest.mark.parametrize("path", ["hashed", "sort"])
def test_capacity_below_solid_count(mixed_records, path):
    """capacity_edges < n_solid: the first `capacity` edges and aux bytes are right, nothing past them is written, and
    *n_solid_out is the true count"""
    k, m = 27, 2
    ref_e, ref_a, ref_h, ref_n = count_records_reference(mixed_records, k, m)
    assert ref_n > 1000
    for cap in (0, ref_n - 7):
        e, a, h, n = run_count(mixed_records, k, m, path == "hashed", cap=cap, room=ref_n + 16, sentinel=True)
        assert n == ref_n and (h == ref_h).all()
        assert (e[:cap] == ref_e[:cap]).all() and (a[:cap] == ref_a[:cap]).all()
        assert (e[cap:] == np.uint32(0xA5A5A5A5)).all() and (a[cap:] == 0xA5).all()


@pytest.mark.parametrize("path", ["hashed", "sort"])
def test_empty_input_leaves_outputs_untouched(path):
    torch = _torch()
    L = lib.load()
    k, m = 27, 2
    hist = torch.full((65536,), 7, dtype=torch.int64, device="cuda")
    ns = torch.full((8,), 12345, dtype=torch.int64, device="cuda")
    buf = torch.zeros(64, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.mhb_count_hashed_workspace_bytes(1, k, m), dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    if path == "hashed":
        rc = L.mhb_count_solid_hashed(None, p(buf), p(buf), 0, k, m, None, p(buf), p(buf), 0, p(hist), p(ns), p(ws), ws.numel())
    else:
        rc = L.mhb_count_solid(None, p(buf), 0, k, m, p(buf), p(buf), 0, p(hist), p(ns), p(ws), ws.numel())
    torch.cuda.synchronize()
    assert rc == 0
    assert (hist.cpu().numpy() == 7).all() and (ns.cpu().numpy() == 12345).all()


def test_hist_byte5_gives_the_same_result(mixed_records):
    k, m = 27, 2
    h5 = np.bincount((mixed_records[:, 0] >> 8) & 255, minlength=256)
    without = run_count(mixed_records, k, m, True)
    with_h = run_count(mixed_records, k, m, True, hist_byte5=h5)
    ref_e, ref_a, ref_h, ref_n = count_records_reference(mixed_records, k, m)
    for e, a, h, n in (without, with_h):
        assert n == ref_n and (e[:n] == ref_e).all() and (a[:n] == ref_a).all() and (h == ref_h).all()


def test_workspace_reused_across_calls():
    """one workspace sized for 2 M records serves a 2 M call and then a 50 k call on other data"""
    torch = _torch()
    L = lib.load()
    rng = np.random.default_rng(1100)
    k, m = 25, 2
    big = random_records(rng, rng.integers(0, 1 << 63, 900_000, dtype=np.uint64), rng.integers(1, 5, 900_000), k)
    small = random_records(rng, rng.integers(0, 1 << 63, 25_000, dtype=np.uint64), rng.integers(1, 4, 25_000), k)
    big, small = big[rng.permutation(len(big))[:2_000_000]], small[rng.permutation(len(small))[:50_000]]
    assert len(big) == 2_000_000 and len(small) == 50_000
    ws = torch.empty(L.mhb_count_hashed_workspace_bytes(len(big), k, m), dtype=torch.uint8, device="cuda")
    assert ws.numel() >= L.mhb_count_hashed_workspace_bytes(len(small), k, m)
    for recs in (big, small):
        e, a, h, n = run_count(recs, k, m, True, ws=ws)
        ref_e, ref_a, ref_h, ref_n = count_records_reference(recs, k, m)
        assert n == ref_n and (e[:n] == ref_e).all() and (a[:n] == ref_a).all() and (h == ref_h).all()


def test_hashed_argument_errors(mixed_records):
    """a workspace one byte short and missing output pointers are MHB_ERR_ARG, before anything runs"""
    torch = _torch()
    L = lib.load()
    k, m = 27, 2
    n = len(mixed_records)
    a, b = _dev_recs(mixed_records)
    out = torch.zeros(n * 3 + 8, dtype=torch.int32, device="cuda")
    aux = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
    hist = torch.zeros(65536, dtype=torch.int64, device="cuda")
    ns = torch.zeros(8, dtype=torch.int64, device="cuda")
    need = L.mhb_count_hashed_workspace_bytes(n, k, m)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    call = lambda kk, mm, h, s, wsb: L.mhb_count_solid_hashed(None, p(a), p(b), n, kk, mm, None, p(out), p(aux), n, p(h), p(s),
                                                                p(ws), wsb)
    assert call(k, m, hist, ns, need - 1) == 1 and b"workspace too small" in L.mhb_last_error()
    assert call(k, m, None, ns, need) == 1 and call(k, m, hist, None, need) == 1
    for kk, mm in ((12, 2), (29, 2), (27, 0), (27, MAX_M + 1)):
        assert call(kk, mm, hist, ns, need) == 1
    torch.cuda.synchronize()
    assert not hist.cpu().numpy().any() and not ns.cpu().numpy().any()
    assert call(k, m, hist, ns, need) == 0  # the same buffers are fine
