"""The multi-GPU iterate without a GPU: the read-share planner (mhb_plan_read_shares), which must give contiguous shares
balanced on bases to within one read, on variable-length libraries and with more ranks than reads; the share planner
of seq2sdbg, which now shares its cut loop, unchanged; and `iterate --gpus N` forwarded to the reference without
--gpus where the device path does not run (k < 9, reads from stdin)."""
import os
import stat
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import lib
from test_s2s_multi_cpu import check as check_seq_shares

CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def make_bin(length, seed=0):
    """a `.bin` image of reads of the given lengths: per read its length word, then ceil(L / 16) words of bases"""
    rng = np.random.default_rng(seed)
    parts = []
    for L in length:
        parts.append(np.array([L], np.uint32))
        parts.append(rng.integers(0, 1 << 32, size=(int(L) + 15) // 16, dtype=np.uint64).astype(np.uint32))
    return np.concatenate(parts) if parts else np.zeros(0, np.uint32)


def check(length, n):
    length = np.asarray(length, np.int64)
    first = lib.plan_read_shares(make_bin(length), len(length), n)
    assert len(first) == n + 1 and first[0] == 0 and first[-1] == len(length)
    assert all(a <= b for a, b in zip(first, first[1:])), first  # contiguous, every read in exactly one share
    cum = np.concatenate([[0], np.cumsum(length)])
    total = int(cum[-1])
    longest = int(length.max()) if len(length) else 0
    for r in range(1, n):
        target = total * r // n  # every cut is the read boundary closest to r / n of the bases
        assert abs(int(cum[first[r]]) - target) <= longest, (r, first)
        assert 2 * abs(int(cum[first[r]]) - target) <= longest, (r, first)
    return first


@pytest.mark.parametrize("n", list(range(1, 17)))
def test_random_variable_length_libraries(n):
    rng = np.random.default_rng(100 + n)
    check(rng.integers(1, 400, size=3000), n)
    check(rng.choice([100, 150, 250], size=2000), n)


@pytest.mark.parametrize("n", [2, 3, 7, 16])
def test_fixed_length_library(n):
    first = check(np.full(1000, 150), n)
    sizes = np.diff(first)
    assert sizes.max() - sizes.min() <= 1


@pytest.mark.parametrize("n_reads,n", [(1, 2), (1, 16), (3, 8), (15, 16)])
def test_fewer_reads_than_ranks(n_reads, n):
    first = check(np.full(n_reads, 150), n)
    sizes = np.diff(first)
    assert sizes.sum() == n_reads and (sizes == 0).sum() >= n - n_reads


def test_no_reads():
    for n in (1, 2, 5, 16):
        assert lib.plan_read_shares(np.zeros(0, np.uint32), 0, n) == [0] * (n + 1)


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_one_long_read_among_short_ones(n):
    """a 2 000 bp read outweighs a whole share of the 150 bp ones"""
    length = np.array([150] * 20 + [2000] + [150] * 20)
    first = check(length, n)
    owner = np.searchsorted(first, 20, side="right") - 1
    assert first[owner] <= 20 < first[owner + 1]


def test_truncated_image_is_refused():
    b = make_bin([150, 150])[:-1]
    with pytest.raises(lib.MhbError):
        lib.plan_read_shares(b, 2, 2)


@pytest.mark.parametrize("k", [21, 227])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_seq_shares_unchanged(k, n):
    """the cases of the seq2sdbg share planner, now one caller of the shared cut loop"""
    rng = np.random.default_rng(k * 10 + n)
    check_seq_shares(rng.integers(1, 3 * k + 400, size=5000), k, n)
    check_seq_shares(np.array([5, 40, 10, 10, 100, 3, 3, 60, 2], np.uint32), 31, 3)
    check_seq_shares(np.array([30] * 20 + [100000] + [30] * 20, np.uint32), 21, 4)
    assert lib.plan_seq_shares(np.zeros(0, np.uint32), 21, 4) == [0, 0, 0, 0, 0]


def _seq_shares_before(length, k, n_ranks):
    """the cut loop of the seq2sdbg planner as it was written before the read planner shared it"""
    items = [2 * (int(L) - k + 2) if L >= k + 1 else 0 for L in length]
    total, n = sum(items), len(items)
    first, b, cum = [0], 0, 0
    for r in range(1, n_ranks):
        target = total * r // n_ranks
        while b < n and cum + items[b] <= target:
            cum += items[b]
            b += 1
        if b < n and cum < target and cum + items[b] - target < target - cum:
            cum += items[b]
            b += 1
        first.append(b)
    return first + [n]


@pytest.mark.parametrize("seed", range(6))
def test_seq_shares_exactly_as_before(seed):
    rng = np.random.default_rng(seed)
    k = int(rng.choice([21, 59, 141, 227]))
    for size in (0, 1, 3, 50, 2000):
        length = rng.integers(1, 3 * k + 400, size=size).astype(np.uint32)
        for n in (1, 2, 3, 5, 8, 16):
            assert lib.plan_seq_shares(length, k, n) == _seq_shares_before(length, k, n), (size, n)


# ---- forwarding to the reference ----
def _stub(tmp_path):
    stub = tmp_path / "ref_stub.sh"
    stub.write_text("#!/bin/sh\necho forwarded \"$@\" > \"$(dirname \"$0\")/forwarded.txt\"\nexit 0\n")
    stub.chmod(stub.stat().st_mode | stat.S_IXUSR)
    return stub


@pytest.mark.skipif(not os.access(CLI, os.X_OK), reason="CLI not built")
@pytest.mark.parametrize("gpus", [["--gpus", "2"], ["--gpus=2"]])
@pytest.mark.parametrize("case", ["k7", "stdin"])
def test_forwarded_iterate_drops_gpus(tmp_path, gpus, case):
    stub = _stub(tmp_path)
    env = dict(os.environ, MHB_REFERENCE_CORE=str(stub), MHB_GPUS="2")
    reads = "-" if case == "stdin" else str(tmp_path / "r.bin")
    k = "7" if case == "k7" else "21"
    before = ["-c", str(tmp_path / "c.fa"), "-b", str(tmp_path / "b.fa"), "-t", "4"]
    after = ["-k", k, "-s", "2", "-r", reads, "--output_prefix", str(tmp_path / "o")]
    r = subprocess.run([CLI, "iterate"] + before + gpus + after, capture_output=True, text=True, env=env, timeout=60)
    assert r.returncode == 0, r.stderr
    assert "forwarded to the reference" in r.stderr
    got = (tmp_path / "forwarded.txt").read_text().split()
    assert got == ["forwarded", "iterate"] + before + after
