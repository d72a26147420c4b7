"""seq2sdbg and its mercy search on inputs larger than device memory, host logic only (no GPU): the sequence chunk
plan, the mercy segment plan, and the residency rules with the device bytes they are decided on."""
import numpy as np
import pytest

from megahit_b200 import lib


def fixed_layout(n, L):
    w = (L + 15) // 16
    return np.arange(n + 1, dtype=np.uint64) * w, np.full(n, L, np.uint32)


def var_layout(lengths):
    ln = np.asarray(lengths, np.uint32)
    wo = np.concatenate([[0], np.cumsum((ln.astype(np.uint64) + 15) // 16)]).astype(np.uint64)
    return wo, ln


def greedy(wo, ln, cap, extra):
    """reference cut: a chunk ends before the sequence that would take it past cap, unless the chunk is empty"""
    first, acc = [0], 0
    for s in range(len(ln)):
        b = 4 * int(wo[s + 1] - wo[s]) + extra
        if s > first[-1] and acc + b > cap:
            first.append(s)
            acc = 0
        acc += b
    return first + [len(ln)] if len(ln) else [0]


@pytest.mark.parametrize("cap", [1, 50, 100, 777, 4096, 1 << 20])
def test_seq_chunk_plan_variable_length(cap):
    rng = np.random.default_rng(cap)
    lengths = rng.integers(1, 400, 500)
    lengths[7] = 5000  # a sequence larger than most caps
    wo, ln = var_layout(lengths)
    plan = lib.plan_seq_chunks(wo, ln, 29, cap)
    assert plan == greedy(wo, ln, cap, 22)
    assert plan[0] == 0 and plan[-1] == len(ln) and all(a < b for a, b in zip(plan, plan[1:]))
    for a, b in zip(plan, plan[1:]):  # every chunk fits, or is one sequence
        assert b - a == 1 or 4 * int(wo[b] - wo[a]) + 22 * (b - a) <= cap


@pytest.mark.parametrize("k,cap", [(27, 1), (27, 10), (27, 11), (27, 9999), (31, 64 << 20), (59, 4096)])
def test_seq_chunk_plan_fixed_length_closed_form(k, cap):
    n = 1234
    wo, ln = fixed_layout(n, k + 1)
    per = max(1, cap // (4 * ((k + 1 + 15) // 16) + 2))  # words + multiplicity
    exp = list(range(0, n, per)) + [n]
    assert lib.plan_seq_chunks(wo, ln, k, cap) == exp
    assert exp == greedy(wo, ln, cap, 2)


def test_seq_chunk_plan_edges():
    assert lib.plan_seq_chunks(np.zeros(1, np.uint64), np.zeros(0, np.uint32), 27, 100) == [0]
    wo, ln = var_layout([20, 3000, 20])
    assert lib.plan_seq_chunks(wo, ln, 27, 64) == [0, 1, 2, 3]
    # equal lengths below k + 1 are not the fixed edge layout: offsets and lengths travel too
    wo, ln = fixed_layout(10, 20)
    assert lib.plan_seq_chunks(wo, ln, 27, 2 * (8 + 22)) == [0, 2, 4, 6, 8, 10]
    with pytest.raises(lib.MhbError, match="bad chunk plan"):
        lib.plan_seq_chunks(wo, ln, 27, 0)


def sorted_edges(k, top_counts, seed=0):
    """sorted `.edges`-like records whose leading bytes have the given counts"""
    we = lib.words_per_edge(k)
    rng = np.random.default_rng(seed)
    tops = np.repeat(np.arange(256, dtype=np.uint32), top_counts)
    e = np.zeros((len(tops), we), np.uint32)
    e[:, 0] = (tops << 24) | rng.integers(0, 1 << 24, len(tops), dtype=np.uint32)
    e[:, 1:] = rng.integers(0, 1 << 32, (len(tops), we - 1), dtype=np.uint64).astype(np.uint32)
    return e[np.lexsort(e.T[::-1])]


def test_mercy_segment_plan_contiguous_and_covering():
    rng = np.random.default_rng(5)
    counts = rng.integers(0, 60, 256)
    counts[:17] = 0
    counts[200:] = 0
    k = 27
    e = sorted_edges(k, counts)
    per = 4 * lib.words_per_edge(k)
    for cap in (int(counts.max()) * per, 1000 * per, int(counts.sum()) * per):
        segs = lib.plan_mercy_segments(e, k, cap)
        assert segs[0] == 0 and segs[-1] == 256 and all(a < b for a, b in zip(segs, segs[1:]))
        sizes = [int(counts[a:b].sum()) * per for a, b in zip(segs, segs[1:])]
        assert all(0 < s <= cap for s in sizes)
        for i in range(len(segs) - 2):  # greedy: the next non-empty byte would not have fitted
            nxt = counts[segs[i + 1]:][counts[segs[i + 1]:] > 0][0]
            assert sizes[i] + int(nxt) * per > cap
    assert lib.plan_mercy_segments(e, k, int(counts.sum()) * per) == [0, 256]
    assert lib.plan_mercy_segments(e[:0], k, 100) == [0, 256]


def test_mercy_segment_plan_oversized_byte():
    counts = np.zeros(256, np.int64)
    counts[0x41] = 10
    counts[0x42] = 3
    k = 21
    e = sorted_edges(k, counts)
    per = 4 * lib.words_per_edge(k)
    assert lib.plan_mercy_segments(e, k, 10 * per) == [0, 0x42, 256]
    with pytest.raises(lib.MhbError, match="leading byte 0x41 alone holds 10 edges"):
        lib.plan_mercy_segments(e, k, 10 * per - 1)


def test_s2s_residency_rule():
    gb = 1 << 30
    # k = 27: 2 words of sequence + word_off 8 + item_off 8 + len 4 + mult 2 = 30 bytes per edge, before any round
    n = 10 ** 9
    d = lib.s2s_stream_decide(n, 2 * n, 27, free_bytes=80 * gb)
    assert 30 * n < d["resident"] < 30 * n + (16 << 20)
    assert not d["stream"]
    assert lib.s2s_stream_decide(n, 2 * n, 27, free_bytes=80 * gb, chunk_limit=64 << 20)["stream"]
    # 92 % of free memory: the largest edge set that stays resident on 80 GB is ~2.4 G edges
    free = 80 * 10 ** 9
    assert not lib.s2s_stream_decide(2_400_000_000, 4_800_000_000, 27, free)["stream"]
    assert lib.s2s_stream_decide(2_500_000_000, 5_000_000_000, 27, free)["stream"]
    # the rule flips exactly where the resident form meets 92 % of free memory
    r = d["resident"]
    f = int(np.ceil(r / 0.92)) + 2
    assert not lib.s2s_stream_decide(n, 2 * n, 27, f)["stream"]
    assert lib.s2s_stream_decide(n, 2 * n, 27, int(r / 0.92) - 2)["stream"]


def test_mercy_residency_rule():
    gb = 1 << 30
    # k = 27: 12 bytes per sorted edge, next to the candidate reads and the scratch
    n_edges = 2 * 10 ** 9
    small = lib.mercy_stream_decide(0, 27, 20_000, 20_000 * 11, 150, free_bytes=80 * gb)
    big = lib.mercy_stream_decide(n_edges, 27, 20_000, 20_000 * 11, 150, free_bytes=80 * gb)
    assert abs((big["resident"] - small["resident"]) - 12 * n_edges) < 512
    assert not small["stream"] and big["stream"] is False
    assert lib.mercy_stream_decide(n_edges, 27, 20_000, 20_000 * 11, 150, free_bytes=80 * gb, chunk_limit=1 << 30)["stream"]
    assert lib.mercy_stream_decide(7 * 10 ** 9, 27, 20_000, 20_000 * 11, 150, free_bytes=80 * gb)["stream"]
    r = big["resident"]
    assert lib.mercy_stream_decide(n_edges, 27, 20_000, 20_000 * 11, 150, free_bytes=int(r / 0.92) - 2)["stream"]
    assert not lib.mercy_stream_decide(n_edges, 27, 20_000, 20_000 * 11, 150, free_bytes=int(np.ceil(r / 0.92)) + 2)["stream"]


def test_mercy_automatic_plan_takes_a_leading_byte_above_the_packing_target():
    """without a cap the segments are packed to about 1 GiB, but a skewed leading byte of several GiB still plans (a
    segment of its own, with slots sized to it); only a byte above half the room left beside the reads is refused"""
    gb = 1 << 30
    k = 27
    per = 4 * lib.words_per_edge(k)
    h = np.full(256, 20_000_000, np.uint64)  # 240 MB of edges per byte
    h[0] = 5 * gb // per                      # A-skew: 5 GiB in byte 0x00
    h[0xFF] = 3 * gb // per + 7
    cand = dict(n_cand_reads=20_000, cand_words=20_000 * 11, max_read_len=150)
    p = lib.mercy_auto_plan(h, k, free_bytes=80 * 10 ** 9, **cand)
    first = p["first"]
    assert first[0] == 0 and first[-1] == 256 and all(a < b for a, b in zip(first, first[1:]))
    assert first[:2] == [0, 1] and first[-2] == 0xFF  # the two large bytes are segments of their own
    sizes = [int(h[a:b].sum()) * per for a, b in zip(first, first[1:])]
    assert all(s <= gb for s, (a, b) in zip(sizes, zip(first, first[1:])) if b - a > 1)  # packed ones stay <= 1 GiB
    assert len(first) - 1 >= int(h.sum()) * per // gb
    assert p["slot_bytes"] >= 5 * gb - per and p["slot_bytes"] < 5 * gb + 4096
    # the same histogram on a device whose room cannot take two 5 GiB slots
    with pytest.raises(lib.MhbError, match="leading byte 0x00 alone holds"):
        lib.mercy_auto_plan(h, k, free_bytes=10 * 10 ** 9, **cand)
    # nothing above the packing target: slots of at most 1 GiB
    small = np.full(256, 1_000_000, np.uint64)
    q = lib.mercy_auto_plan(small, k, free_bytes=80 * 10 ** 9, **cand)
    assert q["slot_bytes"] <= gb + 4096
    assert all(int(small[a:b].sum()) * per <= gb for a, b in zip(q["first"], q["first"][1:]))
