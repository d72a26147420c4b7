"""The count stage at every record width (k = 9 .. 255; MEGAHIT's default k list runs seven of its eight k on these
kernels): the extraction kernels (k_count_extract<W, WR>, k_count_extract_range) against the per-base restatement
count_reference.extract_records, the sort-path counter (k_count_lanes -> scan -> k_count_write, mhb_count.cuh) on
records laid out so that every run sits exactly where a case puts it relative to lanes and chunks, and count_host end
to end against the C oracle.  Each case asserts, on its own input, the property it exists for."""
import ctypes as C

import numpy as np
import pytest

from count_reference import (count_key_words, count_record_words, count_records_reference, extract_records, key_mask,
                             make_records_wide, record_byte_hist, words_per_edge)
from count_wide_cases import STAGE_WORDS, batch_words, library, width_classes
from megahit_b200 import lib

pytestmark = pytest.mark.gpu

WIDTH_K = width_classes(9, 255)   # one k per (W, WR, WE) class
WIDE_K = width_classes(29, 255)   # the classes only the sort path counts


# ---- k_count_lanes geometry (mhb_count.cuh:713-714: count3_ipl; :737: CH = 32 * IPL) ----
def ipl(wr: int) -> int:
    return 16 if wr <= 4 else (8 if wr <= 8 else 4)


def chunk(wr: int) -> int:
    return 32 * ipl(wr)


MUL_HIST_SMEM = 1024  # mhb_count.cuh:264 kMulHistSmem: multiplicities below it go to the shared-memory histogram
MAX_MUL = 65535


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _dev(words):
    torch = _torch()
    flat = np.concatenate([np.ascontiguousarray(words, np.uint32).reshape(-1), np.zeros(8, np.uint32)])
    return torch.from_numpy(flat.view(np.int32)).cuda()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class Reads:
    """a `.bin` word stream on the device as mhb_dev_reads: fixed-length (fixed > 0) or indexed"""

    def __init__(self, binw, n_reads, k, fixed=0):
        torch = _torch()
        from count_reference import read_layout
        lens, starts = read_layout(binw, n_reads)
        self.d_bin = _dev(binw)
        self.d_ro = torch.from_numpy(np.append(starts, len(binw)).astype(np.int64)).cuda()
        self.d_eo = torch.from_numpy(np.concatenate([[0], np.cumsum(np.maximum(lens - k, 0))]).astype(np.int64)).cuda()
        self.n_edges = int(np.maximum(lens - k, 0).sum())
        self.rd = lib.DevReads(self.d_bin.data_ptr(), len(binw), n_reads, fixed, None if fixed else self.d_ro.data_ptr(),
                               None if fixed else self.d_eo.data_ptr())


def device_extract(reads, k, hist_byte):
    torch = _torch()
    wr = count_record_words(k)
    out = torch.full((reads.n_edges * wr + 8,), -1, dtype=torch.int32, device="cuda")
    hist = torch.zeros(256, dtype=torch.int64, device="cuda")
    lib._check(lib.load().mhb_count_extract(None, C.byref(reads.rd), k, _p(out), reads.n_edges, _p(hist), hist_byte))
    torch.cuda.synchronize()
    return out[: reads.n_edges * wr].cpu().numpy().view(np.uint32).reshape(-1, wr), hist.cpu().numpy()


def device_extract_range(reads, n_reads, k, lo, hi, hist_byte):
    """count call, then write call -> per_read offsets, records, histogram of the write call"""
    torch = _torch()
    L = lib.load()
    wr = count_record_words(k)
    per_read = torch.full((n_reads + 1,), -1, dtype=torch.int64, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    args = lambda write, recs, hist: (None, C.byref(reads.rd), C.c_uint32(k), C.c_uint32(lo), C.c_uint32(hi), C.c_int(write),
                                      _p(per_read), _p(recs), _p(hist), C.c_int(hist_byte), _p(total))
    lib._check(L.mhb_count_extract_range(*args(0, None, None)))
    torch.cuda.synchronize()
    n = int(total.item())
    recs = torch.full((n * wr + 8,), -1, dtype=torch.int32, device="cuda")
    hist = torch.zeros(256, dtype=torch.int64, device="cuda")
    lib._check(L.mhb_count_extract_range(*args(1, recs, hist)))
    torch.cuda.synchronize()
    return (per_read.cpu().numpy(), recs[: n * wr].cpu().numpy().view(np.uint32).reshape(-1, wr), hist.cpu().numpy())


def device_count(recs, k, m, device_sort=False, cap=None, room=None, sentinel=False):
    """mhb_count_solid on recs as given (already sorted), or after mhb_sort_records on the count sort bytes.
    -> (edges (room, WE), aux (room,), mul_hist, n_solid) over the whole output buffers"""
    torch = _torch()
    from megahit_b200 import dev
    L = lib.load()
    n, wr = recs.shape
    we = words_per_edge(k)
    cap = n // m + 1 if cap is None else cap
    room = cap if room is None else room
    a = _dev(recs)
    if device_sort:
        a = dev.sort_records(a, torch.empty_like(a), n, wr, lib.count_sort_bytes(k))
    edges = torch.full((room * we + 4,), -0x5A5A5A5B if sentinel else 0, dtype=torch.int32, device="cuda")
    aux = torch.full((room + 4,), 0xA5 if sentinel else 0, dtype=torch.uint8, device="cuda")
    hist = torch.zeros(65536, dtype=torch.int64, device="cuda")
    ns = torch.zeros(8, dtype=torch.int64, device="cuda")
    sc = torch.empty(max(1, L.mhb_count_solid_scratch_bytes(n)), dtype=torch.uint8, device="cuda")
    lib._check(L.mhb_count_solid(None, _p(a), n, k, m, _p(edges), _p(aux), cap, _p(hist), _p(ns), _p(sc), sc.numel()))
    torch.cuda.synchronize()
    e = edges[: room * we].cpu().numpy().view(np.uint32).reshape(room, we)
    return e, aux[:room].cpu().numpy(), hist.cpu().numpy(), int(ns[0].item())


def check_count(recs, k, m, device_sort=False, what=""):
    ref_e, ref_a, ref_h, ref_n = count_records_reference(recs, k, m)
    e, a, h, n = device_count(recs, k, m, device_sort=device_sort)
    assert n == ref_n, (what, n, ref_n)
    bad = np.flatnonzero((e[:n] != ref_e).any(axis=1))
    assert not len(bad), (what, "edges", len(bad), [(e[i].tolist(), ref_e[i].tolist()) for i in bad[:3]])
    bad = np.flatnonzero(a[:n] != ref_a)
    assert not len(bad), (what, "aux", len(bad), [(int(a[i]), int(ref_a[i])) for i in bad[:5]])
    bad = np.flatnonzero(h != ref_h)
    assert not len(bad), (what, "mul_hist", [(int(i), int(h[i]), int(ref_h[i])) for i in bad[:8]])
    return ref_e, ref_a, ref_h, ref_n


# ------------------------------------------------------------------------------------------------
# a. extraction, record for record in read order
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", WIDTH_K)
def test_extract_matches_reference(k):
    binw, n_reads, lens = library(k, 300 + k, n_reads=600, long_reads=True)
    bw = batch_words(binw, n_reads)
    assert (bw > STAGE_WORDS).sum() >= 2 and (bw <= STAGE_WORDS).sum() >= 2, "staged and unstaged batches"
    assert lens.max() == 70_000 and (lens == 0).any() and (lens == k).any() and (lens == k + 1).any()
    ref, strand = extract_records(binw, n_reads, k)
    if k % 2:
        assert (strand == 0).any() and (strand == 1).any()
    sort_byte = lib.count_sort_bytes(k)[0]
    reads = Reads(binw, n_reads, k)
    for hb in (sort_byte, min(5, 4 * count_record_words(k) - 1)):  # byte 5, or the top byte of a 4-byte record
        recs, hist = device_extract(reads, k, hb)
        bad = np.flatnonzero((recs != ref).any(axis=1))
        assert not len(bad), (k, hb, len(bad), bad[:5])
        assert (hist == record_byte_hist(ref, hb)).all(), (k, hb)
    # fixed-length libraries: the 70 000 bp read alone, then 256 copies of an ordinary read
    starts = np.concatenate([[0], np.cumsum(1 + (lens + 15) // 16)])
    for L in (70_000, int(lens[(lens > k) & (lens < 1000)].max())):
        i = int(np.flatnonzero(lens == L)[0])
        one = binw[starts[i]:starts[i + 1]]
        fixed = np.tile(one, 1 if L > 1000 else 256)
        nf = len(fixed) // len(one)
        ref_f, _ = extract_records(fixed, nf, k)
        recs, hist = device_extract(Reads(fixed, nf, k, fixed=L), k, sort_byte)
        assert (recs == ref_f).all() and (hist == record_byte_hist(ref_f, sort_byte)).all(), (k, L)


def _lengths_with(k):
    return [0, k, k + 1, 16 * ((k + 16) // 16), 16 * ((k + 16) // 16) + 1, 16 * ((k + 16) // 16) + 15]


@pytest.mark.parametrize("k", [31, 47, 127, 255])
def test_extract_range_matches_reference(k):
    """count, then write, over bucket ranges: the in-range records of the reference in read order"""
    binw, n_reads, lens = library(k, 400 + k, n_reads=600, long_reads=True)
    ref, _ = extract_records(binw, n_reads, k)
    bucket = ref[:, 0] >> 16
    reads = Reads(binw, n_reads, k)
    n_e = np.maximum(lens - k, 0)
    rid = np.repeat(np.arange(n_reads), n_e)
    med = int(np.median(bucket))
    ranges = [(0, 65535), (0, med - 1), (med, med), (med + 1, 65535), (0x8000, 0xBFFF)]
    for lo, hi in ranges:
        inr = (bucket >= lo) & (bucket <= hi)
        assert inr.any() or (lo, hi) == (0x8000, 0xBFFF)
        per_read, recs, hist = device_extract_range(reads, n_reads, k, lo, hi, 5)
        expect_off = np.concatenate([[0], np.cumsum(np.bincount(rid[inr], minlength=n_reads))])
        assert (per_read == expect_off).all(), (k, lo, hi)
        assert recs.shape == (inr.sum(), count_record_words(k)) and (recs == ref[inr]).all(), (k, lo, hi)
        assert (hist == record_byte_hist(ref[inr], 5)).all()


# ------------------------------------------------------------------------------------------------
# b. the sort-path count on laid-out records
# ------------------------------------------------------------------------------------------------
def k_of_wr(wr: int) -> int:
    """one k per record width 1..17: the smallest k of the width (W = WR - 1: the last word holds prev / next only)
    at even WR, the largest (the key reaches record bit 6) at odd WR"""
    ks = [k for k in range(1, 256) if count_record_words(k) == wr]
    return ks[0] if wr % 2 == 0 and ks[0] >= 9 else ks[-1]


class Layout:
    """runs in key order, each placed at a chosen position: lengths, prev / next per record"""

    def __init__(self, rng, wr):
        self.rng, self.wr, self.IPL, self.CH = rng, wr, ipl(wr), chunk(wr)
        self.runs = []   # (start, prev array, next array)
        self.n = 0
        self.named = {}

    def run(self, length, prev=None, nxt=None, name=None):
        prev = self.rng.integers(0, 5, length) if prev is None else np.asarray(prev)
        nxt = self.rng.integers(0, 5, length) if nxt is None else np.asarray(nxt)
        assert len(prev) == len(nxt) == length
        if name:
            self.named[name] = (self.n, length, len(self.runs))
        self.runs.append((self.n, prev, nxt))
        self.n += length

    def fill_to(self, pos):
        assert pos >= self.n
        while self.n < pos:
            self.run(1)

    def next_boundary(self, kind, at_least):
        """first lane boundary inside a chunk (kind "lane") or chunk boundary >= at_least"""
        step = self.IPL if kind == "lane" else self.CH
        b = -(-at_least // step) * step
        while kind == "lane" and b % self.CH == 0:
            b += step
        return b

    def lane(self, pos):
        return (pos % self.CH) // self.IPL

    def records(self, k):
        """(n, WR) records: ascending distinct keys, one per run, with special neighbours at the named runs"""
        w = count_key_words(k)
        n_runs = len(self.runs)
        keys = self.rng.integers(0, 1 << 32, (2 * n_runs, w), dtype=np.uint64).astype(np.uint32) & key_mask(k)
        keys[:, 0] |= np.uint32(1 << 31)  # every key has the top bit, except the one named "top0" below
        keys = np.unique(keys, axis=0)    # distinct, ascending
        assert len(keys) >= n_runs
        keys = keys[np.sort(self.rng.choice(len(keys), n_runs, replace=False))]
        low = np.zeros(w, np.uint32)  # the lowest key bit
        nb = 2 * (k + 1) - 32 * (w - 1)
        low[-1] = np.uint32(1 << (32 - nb))
        for name, (_, _, i) in self.named.items():
            if name == "top0":       # the run before it has the same key without the top bit of word 0
                keys[i - 1] = keys[i]
                keys[i - 1, 0] &= np.uint32(0x7FFFFFFF)
            elif name == "lowbit":   # the same key but the lowest key bit
                keys[i] = keys[i - 1] & ~low | low
                keys[i - 1] &= ~low
            elif name == "midbit" and w >= 3:
                keys[i] = keys[i - 1]
                keys[i - 1, w // 2] &= ~np.uint32(1)
                keys[i, w // 2] |= np.uint32(1)
        assert (keys[1:] != keys[:-1]).any(axis=1).all()
        order = np.lexsort(keys.T[::-1])
        assert (order == np.arange(n_runs)).all(), "keys ascend in layout order"
        lens = np.array([len(p) for _, p, _ in self.runs])
        return make_records_wide(np.repeat(keys, lens, axis=0), np.concatenate([p for _, p, _ in self.runs]),
                                 np.concatenate([x for _, _, x in self.runs]), k)


def build_layout(wr, m, seed):
    """the placed runs of one record width (m = 3); see the test's docstring"""
    rng = np.random.default_rng(seed)
    lay = Layout(rng, wr)
    IPL, CH = lay.IPL, lay.CH
    lay.run(2)
    lay.run(2, name="top0")  # keys differing only in the top bit of word 0 (the first run has the top bit clear)
    # run lengths around a lane and a chunk, starting at -1, 0, +1 from a lane boundary and from a chunk boundary
    for length in (1, IPL - 1, IPL, IPL + 1, CH - 1, CH, CH + 1):
        for kind in ("lane", "chunk"):
            for d in (-1, 0, 1):
                lay.fill_to(lay.next_boundary(kind, lay.n + 2) + d)
                lay.run(length, name=f"len{length}_{kind}{d:+d}")
    # a run whose head is in the last lane of a chunk and that covers >= 3 whole chunks
    start = lay.next_boundary("chunk", lay.n + 1) + 31 * IPL + IPL // 2
    lay.fill_to(start)
    lay.run(CH - (start % CH) + 3 * CH + 7, name="last_lane_3_chunks")
    # a run that ends exactly at a chunk end, followed by a head
    end = lay.next_boundary("chunk", lay.n + CH + 10)
    lay.fill_to(end - CH - 5)
    lay.run(CH + 5, name="ends_at_chunk_end")
    lay.run(3, name="head_after_chunk_end")
    # tallies reaching m = 3 only with the head lane, a later lane and the records past the chunk end, and twins one
    # short (m - 1), whose in / out flag must flip
    for twin in ("", "drop_head", "drop_later", "drop_past"):
        start = lay.next_boundary("chunk", lay.n + 1) + 20 * IPL + 1
        lay.fill_to(start)
        length = CH - (start % CH) + 2 * IPL
        head, later, past = 0, CH - (start % CH) - 1, CH - (start % CH) + 1  # offsets inside the run
        prev, nxt = np.full(length, 4), np.full(length, 4)
        for o, which in ((head, "drop_head"), (later, "drop_later"), (past, "drop_past")):
            if twin != which:
                prev[o] = 2
                nxt[o + 1] = 1
        lay.run(length, prev, nxt, name=f"tally{('_' + twin) if twin else ''}")
    # neighbouring keys differing in the lowest key bit / one bit of a middle word; one key with all 25 prev / next pairs
    lay.run(3)
    lay.run(4, name="lowbit")
    lay.run(2)
    lay.run(3, name="midbit")
    p, x = np.meshgrid(np.arange(5), np.arange(5))
    lay.run(25, p.reshape(-1), x.reshape(-1), name="all_pairs")
    # multiplicities around the histogram split and the 16-bit clamp
    for c in (1, MUL_HIST_SMEM - 1, MUL_HIST_SMEM, MAX_MUL - 1, MAX_MUL, MAX_MUL + 1, MAX_MUL + 2):
        lay.run(c, name=f"mul{c}")
    # random runs up to a few thousand chunks, then a run that reaches n inside a partial last chunk
    for i in range(10**9):
        if lay.n >= 2000 * CH and i >= 5000:
            break
        lay.run(int(rng.integers(1, 3 * IPL)))
    lay.fill_to(lay.next_boundary("chunk", lay.n + 1) + CH // 2)
    lay.run(CH + CH // 3, name="reaches_n")
    return lay


@pytest.mark.parametrize("wr", range(1, 18))
def test_sort_path_on_laid_out_records(wr):
    """Sorted records handed straight to mhb_count_solid, so that every run sits where the case puts it: run lengths
    1, IPL - 1, IPL, IPL + 1, CH - 1, CH, CH + 1 at -1 / 0 / +1 from a lane and from a chunk boundary; a head in lane 31
    covering >= 3 chunks; a run ending at a chunk end; tallies that reach m only across the head lane, later lanes and
    the records past the chunk end, with m - 1 twins; keys one bit apart; all 25 prev / next pairs in one run;
    multiplicities 1, 1023, 1024 and 65534 - 65537; a run that reaches n; n = 1, CH - 1, CH, CH + 1 and thousands of
    chunks.  Then the same records permuted and sorted on the device."""
    k, m = k_of_wr(wr), 3
    assert count_record_words(k) == wr
    lay = build_layout(wr, m, 5000 + wr)
    IPL, CH = lay.IPL, lay.CH
    nm = lay.named
    # the properties the cases exist for
    for length in (1, IPL - 1, IPL, IPL + 1, CH - 1, CH, CH + 1):
        for kind, step in (("lane", IPL), ("chunk", CH)):
            for d in (-1, 0, 1):
                s, ln, _ = nm[f"len{length}_{kind}{d:+d}"]
                assert ln == length and (s - d) % step == 0 and (kind == "chunk" or (s - d) % CH != 0)
    s, ln, _ = nm["last_lane_3_chunks"]
    assert lay.lane(s) == 31 and (s + ln) // CH - (s // CH + 1) >= 3
    s, ln, _ = nm["ends_at_chunk_end"]
    assert (s + ln) % CH == 0 and nm["head_after_chunk_end"][0] == s + ln
    for name in ("tally", "tally_drop_head", "tally_drop_later", "tally_drop_past"):
        s, ln, _ = nm[name]
        assert lay.lane(s) == 20 and s // CH < (s + ln - 1) // CH
    s, ln, _ = nm["reaches_n"]
    assert s + ln == lay.n and lay.n % CH != 0 and lay.n // CH >= 2000
    recs = lay.records(k)
    assert len(recs) == lay.n
    e, a, h, n = check_count(recs, k, m, what="laid out")
    # tallies: the full run has an incoming and an outgoing base at m; each twin is one short on both
    key_of = lambda name: recs[nm[name][0]]
    keys = e[:, : count_key_words(k)] & key_mask(k)
    flag = {}
    for name in ("tally", "tally_drop_head", "tally_drop_later", "tally_drop_past"):
        i = np.flatnonzero((keys == (key_of(name)[: count_key_words(k)] & key_mask(k))).all(axis=1))
        assert len(i) == 1
        flag[name] = int(a[i[0]])
    assert flag == {"tally": 0, "tally_drop_head": 3, "tally_drop_later": 3, "tally_drop_past": 3}, flag
    assert h[MUL_HIST_SMEM - 1] >= 1 and h[MUL_HIST_SMEM] >= 1 and h[MAX_MUL] >= 3 and h[MAX_MUL - 1] >= 1
    if count_key_words(k) >= 3:
        assert "midbit" in nm
    # prefixes: n = 1, CH - 1, CH, CH + 1
    for nn in (1, CH - 1, CH, CH + 1):
        check_count(recs[:nn], k, m, what=f"n={nn}")
    # the full path: permuted, sorted on the device
    rng = np.random.default_rng(wr)
    check_count(recs[rng.permutation(len(recs))], k, m, device_sort=True, what="device sort")


@pytest.mark.parametrize("wr", [2, 3, 4, 9, 17])
def test_sort_path_clamp_at_a_huge_threshold(wr):
    """a run of 70 001 at m = 70 000: solid by its unclamped count, multiplicity 65 535; 65 535 .. 65 537 beside it
    are not solid"""
    k = k_of_wr(wr)
    lay = Layout(np.random.default_rng(wr), wr)
    for c in (3, MAX_MUL, 70_001, MAX_MUL + 2, 1):
        lay.run(c)
    recs = lay.records(k)
    e, a, h, n = check_count(recs, k, 70_000)
    assert n == 1 and e[0, -1] & 0xFFFF == MAX_MUL and h[MAX_MUL] == 3
    check_count(recs[np.random.default_rng(0).permutation(len(recs))], k, 70_000, device_sort=True)


@pytest.mark.parametrize("wr", [5, 9, 13, 16, 17])
def test_sort_path_capacity_below_solid_count(wr):
    """capacity_edges < n_solid at wide edges: the first `capacity` edges and aux bytes are right, nothing past them
    is written, and *n_solid_out is the true count"""
    k, m = k_of_wr(wr), 2
    rng = np.random.default_rng(6000 + wr)
    lay = Layout(rng, wr)
    while lay.n < 40 * lay.CH:
        lay.run(int(rng.integers(1, 6)))
    recs = lay.records(k)
    ref_e, ref_a, ref_h, ref_n = count_records_reference(recs, k, m)
    assert ref_n > 100 and words_per_edge(k) >= 5
    for cap in (0, ref_n - 7):
        e, a, h, n = device_count(recs, k, m, cap=cap, room=ref_n + 16, sentinel=True)
        assert n == ref_n and (h == ref_h).all()
        assert (e[:cap] == ref_e[:cap]).all() and (a[:cap] == ref_a[:cap]).all()
        assert (e[cap:] == np.uint32(0xA5A5A5A5)).all() and (a[cap:] == 0xA5).all()


# ------------------------------------------------------------------------------------------------
# d. count_host end to end against the C oracle
# ------------------------------------------------------------------------------------------------
def _oracle_check(binw, n_reads, k, m):
    import oracle_pipeline as OP
    from oracle import oracle as O
    oc = OP.oracle_count(O.unpack_bin(binw.tobytes(), reverse=True), k, m)
    g = lib.count_host(binw, n_reads, k, m, want_mercy=True)
    assert g["n_solid"] == oc["n_solid"] > 0
    assert (g["edges"] == oc["edges"]).all()
    assert (g["counting"] == oc["counting"]).all()
    assert (g["cand_ids"] == oc["cand_ids"]).all()
    return g, oc


@pytest.mark.parametrize("k", WIDE_K)
def test_count_host_matches_oracle_at_wide_k(k):
    binw, n_reads, _ = library(k, 500 + k, n_reads=600, long_reads=True)
    g, oc = _oracle_check(binw, n_reads, k, 2)
    assert len(oc["cand_ids"]) > 0
    if k in (47, 127, 255):
        try:
            lib.set_round_limit(g["n_edge_records"] // 5)
            r = lib.count_host(binw, n_reads, k, 2, want_mercy=True)
        finally:
            lib.set_round_limit(0)
        assert r["n_rounds"] > 1
        for key in ("edges", "counting", "cand_ids"):
            assert (r[key] == g[key]).all(), key


@pytest.mark.parametrize("k", [29, 63, 127, 255])
def test_count_host_matches_oracle_on_poly_a_and_tandem_repeats(k):
    """1 000 poly-A and 300 poly-T reads of 400 bp, tandem repeats and ordinary reads: the all-A (k+1)-mer occurs
    > 65 535 times (runs over hundreds of chunks, the multiplicity clamp)"""
    from count_wide_cases import pack
    rng = np.random.default_rng(700 + k)
    genome = rng.integers(0, 4, 6000, dtype=np.uint8)
    reads = [np.zeros(400, np.uint8)] * 1000 + [np.full(400, 3, np.uint8)] * 300
    unit = rng.integers(0, 4, 7, dtype=np.uint8)
    reads += [np.tile(unit, 60)[int(rng.integers(0, 7)):][:400] for _ in range(200)]
    for _ in range(1500):
        L = int(rng.integers(k + 1, k + 300))
        p = int(rng.integers(0, len(genome) - L))
        reads.append(genome[p:p + L])
    order = rng.permutation(len(reads))
    binw = pack([reads[i] for i in order])
    assert 1300 * (400 - k) > MAX_MUL
    g, _ = _oracle_check(binw, len(reads), k, 2)
    assert g["counting"][MAX_MUL] >= 1
