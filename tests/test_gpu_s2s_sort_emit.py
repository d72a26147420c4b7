"""mhb_s2s_sort_emit (the bucket kernel emits every bucket it sorts) against mhb_s2s_sort followed by mhb_s2s_emit on the
same items: the same item bytes, the same 65 536 x 4 bucket table, the same 16 totals and the same sort statistics, on
every path of the bucket sort (small and large geometry, buckets passed to the large one, buckets left to the radix
engine one by one or all at once)."""
import ctypes as C

import numpy as np
import pytest

from megahit_b200 import lib
from s2s_sort_cases import make_items

pytestmark = pytest.mark.gpu

CAP = 3072       # items the small geometry of the bucket kernel sorts (kLsCapS)
CAP_L = 8192     # items the large geometry sorts (kLsCapL)
LIST_CAP = 16    # buckets left to the radix engine sorted one by one (kLsListCap); more = one whole-array sort
KS = [21, 22, 23, 27, 38]


def _hist(rec, n, k, W):
    import torch
    hb = lib.s2s_sort_hist_byte(n, k)
    col = (rec[:, W - 1 - (hb >> 2)] >> np.uint32(8 * (hb & 3))) & np.uint32(255)
    return torch.from_numpy(np.bincount(col, minlength=256).astype(np.int64)).cuda()


def _pair(a_dev, n, W):
    """two copies of the first n items of a_dev, each with its other buffer"""
    import torch
    bufs = []
    for _ in range(2):
        a = torch.zeros(n * W + 8, dtype=torch.int32, device=a_dev.device)
        a[: n * W] = a_dev[: n * W]
        bufs.append((a, torch.zeros_like(a)))
    return bufs


def separate(a, b, n, k, hist, cap_bytes):
    """mhb_s2s_sort, then mhb_s2s_emit: (bytes, table, totals, sort stats)"""
    import torch

    from megahit_b200 import dev
    L = lib.load()
    srt = dev.s2s_sort(a, b, n, k, hist)
    stats = lib.s2s_sort_stats()
    out = torch.zeros(cap_bytes + 64, dtype=torch.uint8, device=a.device)
    table = torch.full((65536 * 4,), -1, dtype=torch.int64, device=a.device)
    totals = torch.full((16,), -1, dtype=torch.int64, device=a.device)
    scr = torch.empty(L.mhb_s2s_emit_scratch_bytes(n, k), dtype=torch.uint8, device=a.device)
    lib._check(L.mhb_s2s_emit(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(srt.data_ptr()), n, k,
                              C.c_void_p(out.data_ptr()), cap_bytes, C.c_void_p(table.data_ptr()),
                              C.c_void_p(totals.data_ptr()), C.c_void_p(scr.data_ptr()), scr.numel()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), table.cpu().numpy(), totals.cpu().numpy(), stats


def fused(a, b, n, k, hist, cap_bytes):
    """mhb_s2s_sort_emit: (bytes, table, totals, sort stats); bytes carries 64 guard bytes behind cap_bytes"""
    import torch

    from megahit_b200 import dev
    out = torch.full((cap_bytes + 64,), 0xAB, dtype=torch.uint8, device=a.device)
    table = torch.full((65536 * 4,), -1, dtype=torch.int64, device=a.device)
    totals = torch.full((16,), -1, dtype=torch.int64, device=a.device)
    dev.s2s_sort_emit(a, b, n, k, hist, out, table, totals, cap_bytes=cap_bytes)
    torch.cuda.synchronize()
    return out.cpu().numpy(), table.cpu().numpy(), totals.cpu().numpy(), lib.s2s_sort_stats()


def compare_dev(a_dev, n, k, hist, cap_bytes=None):
    """fused against separate on the n items of a_dev; returns the sort stats (the same for both)"""
    W = lib.s2s_record_words(k)
    full = n * (4 + 4 * ((k + 15) // 16)) + 16
    (a1, b1), (a2, b2) = _pair(a_dev, n, W)
    rb, rt, rtot, rst = separate(a1, b1, n, k, hist, full)
    cap = full if cap_bytes is None else cap_bytes
    fb, ft, ftot, fst = fused(a2, b2, n, k, hist, cap)
    assert fst == rst, "sort statistics differ"
    assert np.array_equal(ftot, rtot), f"totals differ: {ftot} vs {rtot}"
    assert np.array_equal(ft, rt), f"bucket table differs at {np.flatnonzero(ft != rt)[:8]}"
    nbytes = int(rtot[0])
    if nbytes <= cap:
        assert np.array_equal(fb[:nbytes], rb[:nbytes]), f"item bytes differ at {np.flatnonzero(fb[:nbytes] != rb[:nbytes])[:8]}"
    assert (fb[cap:] == 0xAB).all(), "bytes written past the capacity"
    return fst


def compare(rec, k, cap_bytes=None, hist=True):
    import torch
    W = lib.s2s_record_words(k)
    n = len(rec)
    a = torch.zeros(n * W + 8, dtype=torch.int32, device="cuda")
    if n:
        a[: n * W] = torch.from_numpy(rec.reshape(-1).view(np.int32)).cuda()
    return compare_dev(a, n, k, _hist(rec, n, k, W) if hist and n else None, cap_bytes)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n", [0, 1, 2, 5000, 1 << 20])
def test_random(k, n):
    rng = np.random.default_rng(n * 31 + k)
    st = compare(make_items(rng, n, k), k)
    if n == 1 << 20:
        assert st == (0, 0, 0)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("size", [CAP, CAP + 1, CAP_L, CAP_L + 1])
def test_bucket_at_capacity(k, size):
    rng = np.random.default_rng(size * 3 + k)
    rec = make_items(rng, 100000, k)
    rec[:, 0] = np.where((rec[:, 0] >> np.uint32(16)) == 0x1234, rec[:, 0] ^ np.uint32(1 << 16), rec[:, 0])
    rec = np.concatenate([rec, make_items(rng, size, k, buckets=[0x1234])])
    n_over, _, n_large = compare(rec[rng.permutation(len(rec))], k)
    assert n_over == (1 if size > CAP_L else 0)
    assert n_large == (1 if CAP < size <= CAP_L else 0)


@pytest.mark.parametrize("k", KS)
def test_buckets_for_the_large_geometry(k):
    rng = np.random.default_rng(k + 60)
    assert compare(make_items(rng, 60000, k, buckets=list(range(0x100, 0x108))), k) == (0, 0, 8)


@pytest.mark.parametrize("k", KS)
def test_one_bucket_holds_everything(k):
    rng = np.random.default_rng(k + 61)
    assert compare(make_items(rng, 300000, k, buckets=[0xABCD]), k)[:2] == (1, 300000)


@pytest.mark.parametrize("k", [21, 27, 38])
@pytest.mark.parametrize("n_big", [LIST_CAP, LIST_CAP + 1])
def test_oversized_buckets_around_the_list_capacity(k, n_big):
    """16 buckets: each sorted as a segment and emitted on its own; 17: the whole-array sort and emitter"""
    rng = np.random.default_rng(n_big * 11 + k)
    big = list(range(0x4000, 0x4000 + n_big))
    parts = [make_items(rng, 1 << 20, k, buckets=list(range(0x8000, 0x10000)))]
    parts += [make_items(rng, CAP_L + 1 + 37 * i, k, buckets=[b]) for i, b in enumerate(big)]
    rec = np.concatenate(parts)
    assert compare(rec[rng.permutation(len(rec))], k)[0] == n_big


@pytest.mark.parametrize("k", KS)
def test_equal_key_runs(k):
    """a run of 2000 equal keys (its bucket left to the engine) and one of 200 (ranked inside the bucket kernel)"""
    rng = np.random.default_rng(k + 62)
    rec = make_items(rng, 1 << 20, k)
    rec[:, 0] = np.where(np.isin(rec[:, 0] >> np.uint32(16), [0x7777, 0x7779]), rec[:, 0] ^ np.uint32(4 << 16), rec[:, 0])
    rec = np.concatenate([rec, make_items(rng, 2000, k, buckets=[0x7777], pool=1), make_items(rng, 200, k, buckets=[0x7779], pool=1)])
    assert compare(rec[rng.permutation(len(rec))], k)[:2] == (1, 2000)


@pytest.mark.parametrize("k", KS)
def test_first_and_last_bucket(k):
    rng = np.random.default_rng(k + 63)
    rec = np.concatenate([make_items(rng, 3000, k, buckets=[0x0000]), make_items(rng, 3000, k, buckets=[0xFFFF]),
                          make_items(rng, 20001, k)])
    compare(rec[rng.permutation(len(rec))], k)


@pytest.mark.parametrize("k", [21, 27])
def test_capacity_smaller_than_the_stream(k):
    """nothing is written past the capacity; the table and totals still describe the whole stream"""
    rng = np.random.default_rng(k + 64)
    rec = make_items(rng, 200000, k)
    compare(rec, k, cap_bytes=100000)


@pytest.mark.parametrize("k", [21, 27])
@pytest.mark.parametrize("pruned", [True, False])
def test_real_items_with_mercy_edges(k, pruned):
    """the items of a synthetic library's solid + mercy edges, pruned by the count stage's flags or all six per edge"""
    import torch

    from megahit_b200 import dev, synth
    dv = torch.device("cuda")
    m, n_reads, L = 2, 20000, 150
    bin2d = synth.synth_reads_torch(n_reads, L, 100000, 0.01, seed=k, device=dv)
    bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=dv)])
    plan = dev.CountPlan(n_reads, L, k, m, dv, want_mercy=True)
    ns = plan.run(bin_dev)
    nm = plan.mercy_edges(bin_dev, ns)
    assert nm > 0
    ne = ns + nm
    W = lib.s2s_record_words(k)
    cap = ne * 6
    items = torch.zeros(cap * W + 8, dtype=torch.int32, device=dv)
    hist = torch.zeros(256, dtype=torch.int64, device=dv)
    Lb = lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if pruned:
        cursor = torch.zeros(1, dtype=torch.int64, device=dv)
        lib._check(Lb.mhb_s2s_extract_edges_pruned(st, C.c_void_p(plan.edges.data_ptr()), C.c_void_p(plan.aux.data_ptr()), ne,
                                                   ns, k, C.c_void_p(items.data_ptr()), cap, C.c_void_p(cursor.data_ptr()),
                                                   C.c_void_p(hist.data_ptr()), lib.s2s_sort_hist_byte(cap, k)))
        n = int(cursor.item())
        if lib.s2s_sort_hist_byte(n, k) != lib.s2s_sort_hist_byte(cap, k):
            hist = None
    else:
        seqs = lib.DevSeqs(plan.edges.data_ptr(), plan.edges.numel(), ne, k + 1, None, None, None, None, plan.WE)
        lib._check(Lb.mhb_s2s_extract(st, C.byref(seqs), k, C.c_void_p(items.data_ptr()), cap, C.c_void_p(hist.data_ptr()),
                                      lib.s2s_sort_hist_byte(cap, k)))
        n = cap
    assert compare_dev(items, n, k, hist)[:2] == (0, 0)
