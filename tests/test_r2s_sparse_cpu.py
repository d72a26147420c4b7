"""read2sdbg's mercy candidates in the list form, without a GPU: the host-callable pieces of the device code make each
stage-1 round's candidates as position entries (position << 2 | code) from the group walk's candidate bytes, and the
mercy step scatters every chunk's slice of every round's list into chunk-sized planes before the unchanged per-read
mercy walk.  Against the oracle on the r2s fixtures, and against the plane form on crafted libraries: chunk
boundaries inside a 32-base word, zero-length reads, one read per chunk, positions at and above 2^32.  Also the
choice between the two forms on crafted sizes."""
import numpy as np
import pytest

from megahit_b200 import lib, synth
from oracle import oracle as O
from test_oracle_r2s import r2s_reads


def pad256(x):
    return (x + 255) // 256 * 256


def fixture(case):
    if case == "syn150":
        b, n, Lr, k, m = np.frombuffer(r2s_reads("golden/syn150_k27"), np.uint32), 3000, 150, 27, 2
        b, n = b.reshape(n, -1)[:700].reshape(-1), 700
    elif case == "lowcov":
        b, n, Lr, k, m = np.frombuffer(r2s_reads("golden/lowcov_k21"), np.uint32), 400, 150, 21, 2
    else:  # tie classes far above the insertion-sort threshold
        n, Lr, k, m = 4000, 100, 27, 2
        b = synth.synth_reads(n, Lr, 1500, 0.01, seed=5).reshape(-1)
    return np.ascontiguousarray(b), n, Lr, k, m


def stage1_lists(b, n, Lr, k, m, n_rounds):
    """stage 1 in n_rounds rounds over contiguous bucket ranges, each round's candidates as one sorted list; returns
    (is_solid, counting, lists) and the same stage in the plane form (is_solid, counting, planes)"""
    reads = O.unpack_bin(b.tobytes(), reverse=True)
    nw = lib.r2s_s1_key_words(k)
    per = Lr - k + 4
    recs = np.zeros((n * per, nw + 2), np.uint32)
    for r in range(n):
        w = reads.words[int(reads.word_off[r]):int(reads.word_off[r + 1])]
        for e in range(per):
            recs[r * per + e] = lib.selftest_r2s_s1_record(w, Lr, k, e, r * Lr)
    recs = recs[np.argsort(recs[:, 0] >> 16, kind="stable")]
    bounds = np.searchsorted(recs[:, 0] >> 16, np.arange(65537))
    buckets = np.nonzero(np.diff(bounds))[0]
    # round t takes the buckets whose first record lies in the t-th n_rounds-th of the records
    round_of = np.minimum(bounds[buckets] * n_rounds // len(recs), n_rounds - 1)
    bw = n * Lr // 32 + 2
    solid_l, count_l = np.zeros(bw, np.uint32), np.zeros(65536, np.int64)
    planes = np.zeros((4, bw), np.uint32)
    count_p = np.zeros(65536, np.int64)
    lists = [[] for _ in range(n_rounds)]
    L_ = lib.load()
    for b_, t in zip(buckets, round_of):
        seg = lib.selftest_kmsort(recs[bounds[b_]:bounds[b_ + 1]], nw)
        lists[t].append(lib.selftest_r2s_s1_cand(seg, k, m, Lr, n, solid_l, count_l))
        lib._check(L_.mhb_selftest_r2s_s1_group(seg.ctypes.data, len(seg), k, m, Lr, n, 1, planes[0].ctypes.data,
                                                planes[1].ctypes.data, planes[2].ctypes.data, planes[3].ctypes.data,
                                                count_p.ctypes.data))
    lists = [np.sort(np.concatenate(x)) if x else np.zeros(0, np.uint64) for x in lists]
    return (solid_l, count_l, lists), (planes[0], count_p, planes[1:])


def planes_of(entries, n_words, base0=0):
    """no_in, no_out, any of the entries on the word grid from base0 // 32"""
    p = np.zeros((3, n_words * 32), np.uint8)
    pos = (entries >> np.uint64(2)).astype(np.int64) - (base0 // 32) * 32
    code = (entries & np.uint64(3)).astype(np.int64)
    p[2, pos] = 1
    p[0, pos[code == 1]] = 1
    p[1, pos[code == 2]] = 1
    return np.packbits(p, axis=1, bitorder="little").view(np.uint32)


@pytest.mark.parametrize("case,n_rounds", [("syn150", 1), ("syn150", 9), ("lowcov", 5), ("deep", 2), ("deep", 40)])
def test_lists_match_planes_and_oracle(case, n_rounds):
    b, n, Lr, k, m = fixture(case)
    (solid, counting, lists), (solid_p, counting_p, planes) = stage1_lists(b, n, Lr, k, m, n_rounds)
    assert (solid == solid_p).all() and (counting == counting_p).all()
    assert sum(len(x) for x in lists) > 0 and sum(len(x) > 0 for x in lists) == min(n_rounds, len(lists))
    # the lists hold the positions of exactly the planes' marks (duplicates allowed)
    assert (planes_of(np.concatenate(lists), planes.shape[1]) == planes).all()
    reads = O.unpack_bin(b.tobytes(), reverse=True)
    want = O.read2sdbg(reads, k, m, True, want_solid=True)
    ref_bits = np.unpackbits(want["is_solid"], bitorder="little")[:n * Lr]
    mer_p, added_p = lib.selftest_r2s_mercy_lists(k, solid, n, fixed_len=Lr, planes=planes)
    rng = np.random.default_rng(n_rounds)
    for first in ([0, n], list(range(n + 1)), [0] + sorted(rng.choice(np.arange(1, n), 13, replace=False)) + [n]):
        mer, added = lib.selftest_r2s_mercy_lists(k, solid, n, fixed_len=Lr, rounds=lists, chunk_first=first)
        assert added == added_p == want["n_mercy"]
        assert (mer == mer_p).all()
        got = np.unpackbits((solid | mer).view(np.uint8), bitorder="little")[:n * Lr]
        assert (got == ref_bits).all()


def crafted(seed, n, k, base0, zero_every=7):
    """variable lengths (zero-length reads among them, counted as one base), random solid bits and candidates"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(k - 3, 3 * k, n).astype(np.uint32)
    lens[::zero_every] = 0
    eff = np.maximum(lens, 1).astype(np.int64)
    base = base0 + np.concatenate([[0], np.cumsum(eff)])
    n_bases = int(eff.sum())
    words = (base0 + n_bases) // 32 + 2 - base0 // 32
    bits = np.zeros(words * 32, np.uint8)
    off = base0 // 32 * 32
    pos = []
    for r in range(n):
        L = int(eff[r])
        bits[base[r] - off + np.nonzero(rng.random(L) < 0.04)[0]] = 1
        pos.append(base[r] + np.nonzero(rng.random(L) < 0.15)[0])
    pos = np.concatenate(pos).astype(np.uint64)
    entries = pos << np.uint64(2) | rng.integers(0, 3, len(pos)).astype(np.uint64)
    solid = np.packbits(bits, bitorder="little").view(np.uint32)
    return lens, base, solid, entries, words


@pytest.mark.parametrize("base0", [0, 37, (1 << 32) - 45, (1 << 32) + 13, (1 << 36) + 5])
def test_lists_match_planes_on_crafted_libraries(base0):
    n, k = 300, 21
    lens, base, solid, entries, words = crafted(base0 % 1000, n, k, base0)
    if base0 >= 1 << 32:
        assert (entries >> np.uint64(2)).min() >= 1 << 32
    planes = planes_of(entries, words, base0)
    mer_p, added_p = lib.selftest_r2s_mercy_lists(k, solid, n, lens=lens, base0=base0, planes=planes)
    assert added_p > 0
    rng = np.random.default_rng(1)
    # rounds: the entries dealt at random to 6 lists, each sorted, with duplicates in two of them
    deal = rng.integers(0, 6, len(entries))
    rounds = [np.sort(entries[deal == t]) for t in range(6)]
    rounds[2] = np.sort(np.concatenate([rounds[2], entries[::5]]))
    rounds[4] = np.sort(np.concatenate([rounds[4], rounds[4][::3]]))
    inside = [r for r in range(1, n) if base[r] % 32 not in (0, 31)]  # boundaries inside a 32-base word
    chunkings = [[0, n], list(range(n + 1)), [0] + inside[::17] + [n], [0, 1, 2, n - 1, n], [0, 7, 7, 8, 14, 15, n]]
    for first in chunkings:
        mer, added = lib.selftest_r2s_mercy_lists(k, solid, n, lens=lens, base0=base0, rounds=rounds, chunk_first=first)
        assert added == added_p
        assert (mer == mer_p).all()
    # one list per round with every entry in it, and no entries at all
    mer, added = lib.selftest_r2s_mercy_lists(k, solid, n, lens=lens, base0=base0, rounds=[np.sort(entries)],
                                              chunk_first=[0, n // 2, n])
    assert added == added_p and (mer == mer_p).all()
    mer, added = lib.selftest_r2s_mercy_lists(k, solid, n, lens=lens, base0=base0, rounds=[np.zeros(0, np.uint64)],
                                              chunk_first=[0, n])
    assert added == 0 and not mer.any()


def test_form_choice_on_crafted_sizes():
    gb = 1 << 30
    n_bases, pw, streamed = 150 * 10 ** 9, 40 << 20, 3 * gb
    bit_words = n_bases // 32 + 2
    rest = pad256(bit_words * 4) + pad256(pw * 4) + streamed + pad256(65536 * 8) + pad256(64) + pad256(65536 * 32) + pad256(128)
    planes = rest + 3 * pad256(bit_words * 4)  # the streamed form's bytes before the list form existed
    f = lib.r2s_mercy_form(n_bases, pw, streamed, 2, True, planes)
    assert f["planes"] == planes and not f["sparse"]  # the plane-form threshold has not moved
    assert lib.r2s_mercy_form(n_bases, pw, streamed, 2, True, planes - 1)["sparse"]
    assert f["lists"] == rest + pad256(3 * pw * 4) + pad256((1 << 20) * 8) and f["lists"] < planes
    assert lib.r2s_mercy_form(n_bases, pw, streamed, 2, True, 1 << 50, force=1)["sparse"]
    for m, mercy in ((1, True), (2, False)):  # no candidates: never the list form
        assert not lib.r2s_mercy_form(n_bases, pw, streamed, m, mercy, 1, force=1)["sparse"]
    assert lib.r2s_mercy_form(n_bases, pw, streamed, 2, False, 0)["planes"] == rest - pad256(pw * 4)  # no mercy plane


def test_form_choice_leaves_the_residency_rule_alone():
    """the resident form still counts four whole-library planes with need_mercy: the list form is streamed only"""
    gb = 1 << 30
    n, L = 10 ** 9, 150
    sz = dict(n_reads=n, bin_words=n * 11, fixed_len=L, n_words=n * 10, n_bases=n * L, n_s1=n * (L - 27 + 4),
              n_edges=n * (L - 27))
    with_m = lib.r2s_stream_decide(**sz, k=27, m=2, need_mercy=True, free_bytes=80 * gb)
    without = lib.r2s_stream_decide(**sz, k=27, m=2, need_mercy=False, free_bytes=80 * gb)
    assert with_m["resident"] - without["resident"] == 4 * pad256((n * L // 32 + 2) * 4)
