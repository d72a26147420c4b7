"""mhb_s2s_sort (two radix passes to the 16-bit bucket, then every bucket in shared memory) against a NumPy reference of
mhb_s2s_sort_bytes: ascending on those bytes and the same multiset of whole records, multiplicity bits included."""
import numpy as np
import pytest

from megahit_b200 import lib
from s2s_sort_cases import check_sorted, make_items

pytestmark = pytest.mark.gpu

CAP = 3072       # items the small geometry of the bucket kernel sorts (kLsCapS)
CAP_L = 8192     # items the large geometry sorts (kLsCapL)
LIST_CAP = 16    # buckets left to the radix engine sorted one by one (kLsListCap); more = one whole-array sort


def run_sort(rec: np.ndarray, k: int, hist: bool = True):
    import torch

    from megahit_b200 import dev
    W = lib.s2s_record_words(k)
    n = len(rec)
    dv = torch.device("cuda")
    a = torch.zeros(n * W + 8, dtype=torch.int32, device=dv)
    b = torch.zeros(n * W + 8, dtype=torch.int32, device=dv)
    if n:
        a[: n * W] = torch.from_numpy(rec.reshape(-1).view(np.int32)).to(dv)
    h = None
    if hist:
        hb = lib.s2s_sort_hist_byte(n, k)
        col = (rec[:, W - 1 - (hb >> 2)] >> np.uint32(8 * (hb & 3))) & np.uint32(255)
        h = torch.from_numpy(np.bincount(col, minlength=256).astype(np.int64)).to(dv)
    out = dev.s2s_sort(a, b, n, k, h)
    torch.cuda.synchronize()
    return out[: n * W].cpu().numpy().view(np.uint32).reshape(n, W)


KS = [21, 22, 23, 27, 38]


@pytest.mark.parametrize("k", KS + [45])
@pytest.mark.parametrize("n", [0, 1, 2, 7, 100, 5000])
def test_small(k, n):
    rng = np.random.default_rng(n * 100 + k)
    rec = make_items(rng, n, k)
    check_sorted(rec, run_sort(rec, k), k)


@pytest.mark.parametrize("k", KS + [45])
def test_random_1m(k):
    rng = np.random.default_rng(k)
    rec = make_items(rng, 1 << 20, k)
    check_sorted(rec, run_sort(rec, k), k)
    if k <= 38:
        assert lib.s2s_sort_stats() == (0, 0, 0)


@pytest.mark.parametrize("k", KS)
def test_no_first_histogram(k):
    rng = np.random.default_rng(k + 1)
    rec = make_items(rng, 200000, k)
    check_sorted(rec, run_sort(rec, k, hist=False), k)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("size", [CAP, CAP + 1, CAP_L, CAP_L + 1])
def test_bucket_at_capacity(k, size):
    rng = np.random.default_rng(size + k)
    rec = make_items(rng, 100000, k)
    rec[:, 0] = np.where((rec[:, 0] >> np.uint32(16)) == 0x1234, rec[:, 0] ^ np.uint32(1 << 16), rec[:, 0])  # free the bucket
    rec = np.concatenate([rec, make_items(rng, size, k, buckets=[0x1234])])
    rec = rec[rng.permutation(len(rec))]
    check_sorted(rec, run_sort(rec, k), k)
    n_over, _, n_large = lib.s2s_sort_stats()
    assert n_over == (1 if size > CAP_L else 0)
    assert n_large == (1 if CAP < size <= CAP_L else 0)


@pytest.mark.parametrize("k", KS)
def test_one_bucket_holds_everything(k):
    rng = np.random.default_rng(k + 2)
    rec = make_items(rng, 300000, k, buckets=[0xABCD])
    check_sorted(rec, run_sort(rec, k), k)
    assert lib.s2s_sort_stats()[:2] == (1, 300000)


@pytest.mark.parametrize("k", [21, 27, 38])
@pytest.mark.parametrize("n_big", [LIST_CAP, LIST_CAP + 1])
def test_oversized_buckets_around_the_threshold(k, n_big):
    rng = np.random.default_rng(n_big * 7 + k)
    big = list(range(0x4000, 0x4000 + n_big))
    parts = [make_items(rng, 200000, k, buckets=list(range(0x8000, 0x10000)))]
    parts += [make_items(rng, CAP_L + 1 + 37 * i, k, buckets=[b]) for i, b in enumerate(big)]
    rec = np.concatenate(parts)
    rec = rec[rng.permutation(len(rec))]
    check_sorted(rec, run_sort(rec, k), k)
    assert lib.s2s_sort_stats()[0] == n_big


@pytest.mark.parametrize("k", KS)
def test_keys_differing_only_in_flags_or_last_key_bit(k):
    rng = np.random.default_rng(k + 3)
    W = lib.s2s_record_words(k)
    base = make_items(rng, 64, k, buckets=[0x0101, 0x0102])
    rec = np.repeat(base, 40, axis=0)
    rec[:, W - 1] &= np.uint32(~(0xFFFFF) & 0xFFFFFFFF)
    nd = rng.integers(0, 2, size=len(rec)).astype(np.uint32)
    prev = rng.integers(0, 5, size=len(rec)).astype(np.uint32)
    rec[:, W - 1] |= (nd << 19) | (prev << 16) | rng.integers(0, 1 << 16, size=len(rec)).astype(np.uint32)
    kb = 2 * k - 1
    flip = rng.integers(0, 2, size=len(rec)).astype(bool)
    rec[flip, kb // 32] ^= np.uint32(1 << (31 - kb % 32))
    rec = rec[rng.permutation(len(rec))]
    check_sorted(rec, run_sort(rec, k), k)


@pytest.mark.parametrize("k", KS)
def test_equal_keys_with_different_multiplicities(k):
    rng = np.random.default_rng(k + 4)
    rec = make_items(rng, 50000, k)
    rec[:, 0] = np.where(np.isin(rec[:, 0] >> np.uint32(16), [0x7777, 0x7778, 0x7779]), rec[:, 0] ^ np.uint32(4 << 16), rec[:, 0])
    # one run of 2000 equal keys and three of ~667 (groups far above 256: left to the engine), and a bucket whose
    # 200 equal keys stay in one 12-bit group of the bucket kernel (ranked by counting)
    rec = np.concatenate([rec, make_items(rng, 2000, k, buckets=[0x7777], pool=1),
                          make_items(rng, 2000, k, buckets=[0x7778], pool=3), make_items(rng, 200, k, buckets=[0x7779], pool=1)])
    rec = rec[rng.permutation(len(rec))]
    check_sorted(rec, run_sort(rec, k), k)
    assert lib.s2s_sort_stats()[:2] == (2, 4000)


@pytest.mark.parametrize("k", KS)
def test_buckets_between_the_two_capacities(k):
    """buckets of 3073..8192 items: the small geometry passes them on, the large one sorts them in a second launch"""
    rng = np.random.default_rng(k + 6)
    rec = make_items(rng, 60000, k, buckets=list(range(0x100, 0x108)))  # ~7500 items per bucket
    check_sorted(rec, run_sort(rec, k), k)
    assert lib.s2s_sort_stats() == (0, 0, 8)


@pytest.mark.parametrize("k", KS)
def test_first_and_last_bucket(k):
    rng = np.random.default_rng(k + 5)
    rec = np.concatenate([make_items(rng, 3000, k, buckets=[0x0000]), make_items(rng, 3000, k, buckets=[0xFFFF]),
                          make_items(rng, 20001, k)])
    rec = rec[rng.permutation(len(rec))]
    check_sorted(rec, run_sort(rec, k), k)


def test_trace_has_one_entry_per_sort():
    """after a device seq2sdbg step, the latest entry of the sort trace is the two bucket passes over the items and the
    one before it is the count stage's sort"""
    import torch

    from megahit_b200 import dev, synth
    dv = torch.device("cuda")
    k, m, n_reads, L = 27, 2, 20000, 150
    bin2d = synth.synth_reads_torch(n_reads, L, 100000, 0.005, seed=3, device=dv)
    bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=dv)])
    plan = dev.CountPlan(n_reads, L, k, m, dv, want_mercy=True)
    ns = plan.run(bin_dev)
    s2s = dev.S2sPlan(ns + 1024, k + 1, k, dv)
    s2s.run(plan.edges, None, ns, plan.WE, aux=plan.aux, n_aux=ns)
    torch.cuda.synchronize()
    passes, n_rec, words = lib.sort_pass_ms(0)
    assert len(passes) == 2 and n_rec == s2s.n_items and words == s2s.W
    _, n_rec1, words1 = lib.sort_pass_ms(1)
    assert n_rec1 == plan.n and words1 == plan.WR
