"""GPU tests of read2sdbg in rounds: libraries whose stage-1 records or stage-2 items do not fit the device at once are
sorted in passes over contiguous ranges of 16-bit bucket ids (as the reference's Lv1 passes, base_engine.cpp:54-141,
:254-281).  The rounds are forced here with lib.set_r2s_round_limit, and every test checks that they happened.  The
result must not depend on the plan: the reference's digests (tests/golden_r2s/r2s.json, tests/golden_cli/cli.json) and
the one-pass result are the yardsticks.
"""
import json
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from oracle import oracle as O
from test_gpu_r2s import gpu_cases, n_reads_of
from test_oracle_r2s import R2S, r2s_reads

pytestmark = pytest.mark.gpu


def read_lengths(data: bytes) -> np.ndarray:
    """lengths of the reads of a `.bin` image (u32 length + ceil(L / 16) words per read); a zero-length read counts as one
    base (sequence_package.h:276-281)"""
    w = np.frombuffer(data, np.uint32)
    out, pos = [], 0
    while pos < len(w):
        L = int(w[pos])
        out.append(max(L, 1))
        pos += 1 + (L + 15) // 16
    return np.array(out, np.int64)


def n_s1_records(data: bytes, k: int) -> int:
    L = read_lengths(data)
    L = L[L >= k + 1]
    return int((L - k + 4).sum())


def run(data, n_reads, k, m, mercy, s1=0, s2=0, env=None):
    env = env or {}
    lib.set_r2s_round_limit(s1, s2)
    os.environ.update(env)
    try:
        return lib.read2sdbg_host(np.frombuffer(data, np.uint32), n_reads, k, m, mercy)
    finally:
        lib.set_r2s_round_limit(0, 0)
        for k_ in env:
            del os.environ[k_]


def fit_cap(attempt, cap):
    """attempt(cap) with cap raised to the size of a bucket the planner reports as larger than a round, until it fits
    (skewed libraries such as poly-A: a bucket is the unit of a round)"""
    for _ in range(64):
        try:
            return attempt(cap), cap
        except lib.MhbError as e:
            hit = re.search(r"alone holds (\d+) records, more than one round can take", str(e))
            if not hit:
                raise
            cap = int(hit.group(1))
    raise AssertionError("round cap did not converge")


def ceil_div(a, b):
    return -(-a // b)


def assert_reference(g, gold):
    assert g["n_mercy"] == gold["n_mercy"]
    if gold["m"] > 1:
        assert F.sha256(O.counting_text(g["counting"])) == gold["counting_sha256"]
    assert g["n_items"] == gold["sdbg_items"] and g["n_tips"] == gold["sdbg_tips"]
    assert g["n_large_mul"] == gold["sdbg_large_mul"] and g["words_per_tip_label"] == gold["sdbg_words_per_tip_label"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


def assert_same(a, b):
    """two plans of one library: everything the call returns, byte offsets of the bucket table included"""
    assert (a["bucket_table"] == b["bucket_table"]).all()
    assert (a["w_count"] == b["w_count"]).all() and a["ones_in_last"] == b["ones_in_last"]
    assert (a["counting"] == b["counting"]).all()
    for key in ("n_sort_items", "n_distinct_items", "n_items", "n_tips", "n_large_mul", "n_mercy", "n_bytes"):
        assert a[key] == b[key], key
    assert a["bytes"] == b["bytes"]


def gold_run(lib_name, k=27, m=2, mercy=1):
    return [r for r in R2S["runs"] if r["lib"] == lib_name and r["k"] == k and r["m"] == m and r["mercy"] == mercy][0]


@pytest.mark.parametrize("gold", gpu_cases())
def test_rounds_match_reference(gold):
    """every GPU case of the reference fixtures with each stage that runs cut into >= 4 rounds (fewer only where a
    single bucket holds more than a quarter of the records: a bucket never spans two rounds)"""
    data = r2s_reads(gold["lib"])
    n_reads, k, m, mercy = n_reads_of(gold["lib"], data), gold["k"], gold["m"], bool(gold["mercy"])
    one = run(data, n_reads, k, m, mercy)
    assert one["n_rounds_s1"] == (1 if m > 1 and n_s1_records(data, k) else 0)
    assert one["n_rounds_s2"] == (1 if one["n_sort_items"] else 0)
    n1 = n_s1_records(data, k) if m > 1 else 0
    n2 = one["n_sort_items"]
    c1 = ceil_div(n1, 6) if n1 else 0
    if c1:
        _, c1 = fit_cap(lambda c: run(data, n_reads, k, m, mercy, s1=c), c1)
    c2 = ceil_div(n2, 6) if n2 else 0
    if c2:
        g, c2 = fit_cap(lambda c: run(data, n_reads, k, m, mercy, s1=c1, s2=c), c2)
    else:
        g = run(data, n_reads, k, m, mercy, s1=c1)
    if n1:
        assert g["n_rounds_s1"] >= min(4, ceil_div(n1, c1))
    if n2:
        assert g["n_rounds_s2"] >= min(4, ceil_div(n2, c2))
    assert_reference(g, gold)
    assert_same(g, one)


@pytest.mark.parametrize("stage", [1, 2])
def test_one_stage_in_rounds(stage):
    """synth:deep: only stage 1 in rounds, then only stage 2; the other stage takes one pass"""
    lib_name = "synth:deep"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    one = run(data, n_reads, 27, 2, True)
    if stage == 1:
        g = run(data, n_reads, 27, 2, True, s1=ceil_div(n_s1_records(data, 27), 5))
        assert g["n_rounds_s1"] >= 5 and g["n_rounds_s2"] == 1
    else:
        g = run(data, n_reads, 27, 2, True, s2=ceil_div(one["n_sort_items"], 5))
        assert g["n_rounds_s1"] == 1 and g["n_rounds_s2"] >= 5
    assert_reference(g, gold)
    assert_same(g, one)


def test_round_count_does_not_matter():
    """synth:wide at 2, about 8 and about 64 rounds per stage against one pass"""
    lib_name = "synth:wide"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    one = run(data, n_reads, 27, 2, True)
    assert one["n_rounds_s1"] == 1 and one["n_rounds_s2"] == 1
    assert_reference(one, gold)
    n1, n2 = n_s1_records(data, 27), one["n_sort_items"]
    for div, lo_rounds, hi_rounds in ((1.6, 2, 2), (8, 8, 10), (64, 64, 80)):
        g = run(data, n_reads, 27, 2, True, s1=int(n1 / div) + 1, s2=int(n2 / div) + 1)
        assert lo_rounds <= g["n_rounds_s1"] <= hi_rounds and lo_rounds <= g["n_rounds_s2"] <= hi_rounds, (
            div, g["n_rounds_s1"], g["n_rounds_s2"])
        assert_same(g, one)


@pytest.mark.parametrize("env", [{"MHB_R2S_KMSORT_GLOBAL": "1"}, {"MHB_R2S_KM_CAP": "1024"}])
@pytest.mark.parametrize("lib_name", ["synth:deep", "golden/polya_k27"])
def test_kmsort_fallbacks_in_rounds(lib_name, env):
    """the in-place kmsort walk (whole sort, and the per-bucket fall-back) on the records of one round"""
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    n1 = n_s1_records(data, 27)
    g, c1 = fit_cap(lambda c: run(data, n_reads, 27, 2, True, s1=c, env=env), ceil_div(n1, 5))
    assert g["n_rounds_s1"] >= 2 and g["n_rounds_s1"] >= min(4, ceil_div(n1, c1))  # polya: one bucket holds 98 %
    assert_reference(g, gold)


def s1_bucket_hist(data: bytes, k: int) -> np.ndarray:
    """histogram of the 16-bit bucket ids of the stage-1 records of a fixed-length library, restated in NumPy: the first
    eight bases of the (k-1)-mer at p = 0 and p = L-k+1 on both strands, and of the smaller strand in between
    (read_to_sdbg_s1.cpp:254-279; a palindrome has the same bucket on both)"""
    s = O.unpack_bin(data, reverse=True)
    L, kk = int(s.len[0]), k - 1
    assert (s.len == L).all() and kk <= 32
    nw = (L + 15) // 16
    shifts = (30 - 2 * np.arange(16)).astype(np.uint32)
    b = ((s.words.reshape(-1, nw)[:, :, None] >> shifts) & 3).reshape(s.n, -1)[:, :L].astype(np.uint64)
    P = L - k + 2  # (k-1)-mer positions 0 .. L-k+1
    F = np.zeros((s.n, P), np.uint64)
    R = np.zeros((s.n, P), np.uint64)
    for j in range(kk):
        F = (F << np.uint64(2)) | b[:, j:j + P]
        R = (R << np.uint64(2)) | (np.uint64(3) - b[:, kk - 1 - j:kk - 1 - j + P])
    top = lambda v: (v >> np.uint64(2 * kk - 16)).astype(np.int64)  # noqa: E731
    ids = np.concatenate([top(F[:, 0]), top(R[:, 0]), top(np.minimum(F, R)[:, 1:P - 1]).ravel(), top(F[:, P - 1]),
                          top(R[:, P - 1])])
    return np.bincount(ids, minlength=65536)


def test_plan_cuts_a_leading_byte_on_its_second_byte():
    """synth:deep with a stage-1 cap below its largest leading byte but not below any bucket: that byte is split over
    rounds at bucket boundaries, and the reference's digests hold"""
    lib_name = "synth:deep"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    h = s1_bucket_hist(data, 27)
    assert h.sum() == n_s1_records(data, 27)
    lead = h.reshape(256, 256).sum(axis=1)
    cap = int(lead.max()) - 1
    assert cap >= h.max()
    g = run(data, n_reads, 27, 2, True, s1=cap)
    assert g["n_rounds_s1"] >= ceil_div(int(h.sum()), cap)
    assert_reference(g, gold)


def test_bucket_larger_than_a_round_fails_cleanly():
    """golden/polya_k27 (one bucket holds most stage-1 records): a cap of that bucket works, one record less fails with
    the planner's error, and an uncapped call afterwards gives the reference's digests (the failed call left nothing)"""
    lib_name = "golden/polya_k27"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    h = s1_bucket_hist(data, 27)
    assert h.sum() == n_s1_records(data, 27)
    biggest = int(h.max())
    g = run(data, n_reads, 27, 2, True, s1=biggest)
    assert g["n_rounds_s1"] >= 2
    assert_reference(g, gold)
    with pytest.raises(lib.MhbError, match="more than one round can take"):
        run(data, n_reads, 27, 2, True, s1=biggest - 1)
    assert_reference(run(data, n_reads, 27, 2, True), gold)


@pytest.mark.parametrize("m,mercy", [(2, True), (1, False)])
def test_cli_read2sdbg_in_rounds_at_300k_reads(tmp_path, m, mercy):
    """`megahit_core read2sdbg`'s in-process entry point with >= 5 rounds per stage that runs, against the digests of
    what the reference binary writes for the same library (37 M stage-1 records, 70+ M stage-2 items)"""
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"][f"m{m}"]
    libp = GC.r2s_lib(tmp_path)
    data = open(libp + ".bin", "rb").read()
    n_reads = F.read_lib_info(libp)[1]
    one = run(data, n_reads, 27, m, mercy)
    c1 = ceil_div(n_s1_records(data, 27), 5) if m > 1 else 0
    c2 = ceil_div(one["n_sort_items"], 5)
    g = run(data, n_reads, 27, m, mercy, s1=c1, s2=c2)
    assert g["n_rounds_s2"] >= 5 and (m == 1 or g["n_rounds_s1"] >= 5)
    assert_same(g, one)
    p = str(tmp_path / "ours")
    lib.set_r2s_round_limit(c1, c2)
    try:
        lib.read2sdbg_run(libp, p, k=27, m=m, need_mercy=mercy, host_mem=3e10, num_cpu_threads=min(32, os.cpu_count() or 8))
    finally:
        lib.set_r2s_round_limit(0, 0)
    assert GC.r2s_digest(p, m) == ref
