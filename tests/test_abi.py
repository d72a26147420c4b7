"""C-ABI checks that need no GPU: libmhb.so loads, exports every symbol include/mhb.h declares, the
geometry helpers agree with the reference's formulas, and compute entry points refuse to run without CUDA."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import lib


def header_symbols():
    src = open(os.path.join(ROOT, "include", "mhb.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mhb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = lib.load()
    declared = header_symbols()
    assert declared, "no declarations parsed"
    for s in declared:
        assert hasattr(L, s), f"{s} declared in include/mhb.h but not exported by libmhb.so"
    assert sorted(lib.SYMBOLS) == declared


def test_version_and_error_strings():
    L = lib.load()
    assert b"sm_90a" in L.mhb_version()
    assert isinstance(L.mhb_last_error(), bytes)


@pytest.mark.parametrize("k", [9, 15, 16, 21, 27, 28, 29, 31, 32, 39, 59, 79, 99, 119, 141, 254, 255])
def test_geometry(k):
    K1 = k + 1
    assert lib.words_per_edge(k) == (2 * K1 + 16 + 31) // 32  # kmer_counter.cpp:79-80
    assert lib.s2s_record_words(k) == (2 * k + 20 + 31) // 32  # seq_to_sdbg.cpp:510-512
    wr = lib.count_record_words(k)
    assert wr == (2 * K1 + 6 + 31) // 32
    cb = lib.count_sort_bytes(k)
    # every key bit is covered, no byte twice, ascending
    assert cb == sorted(set(cb)) and cb[-1] == 4 * wr - 1 and cb[0] * 8 <= 32 * wr - 2 * K1 < cb[0] * 8 + 8
    sb = lib.s2s_sort_bytes(k)
    w = lib.s2s_record_words(k)
    # bytes 0-1 (65535 - multiplicity) are not sorted: the emit kernel takes each run's minimum instead
    assert sb == sorted(set(sb)) and sb[0] == 2 and 0 not in sb and 1 not in sb and sb[-1] == 4 * w - 1
    lo = (32 * w - 2 * k) // 8
    assert all(b in sb for b in range(lo, 4 * w))


def test_k27_matches_survey_sizes():
    assert lib.count_record_words(27) == 2 and len(lib.count_sort_bytes(27)) == 7
    assert lib.words_per_edge(27) == 3 and lib.s2s_record_words(27) == 3


@pytest.mark.skipif(lib.load().mhb_device_count() > 0, reason="GPU present")
def test_no_cpu_fallback():
    with pytest.raises(lib.MhbError, match="no CUDA device"):
        lib.count_host(np.array([4, 0], np.uint32), 1, 21, 2)
    with pytest.raises(lib.MhbError, match="no CUDA device"):
        lib.s2s_host(np.zeros(2, np.uint32), np.array([0, 2], np.uint64), np.array([30], np.uint32),
                     np.array([1], np.uint16), 21)


def test_hashed_count_supported_range():
    """the hashed count needs 8-byte records (13 <= k <= 28) and 1 <= m <= 1024; outside that range a call is refused
    with MHB_ERR_ARG before it touches any pointer"""
    L = lib.load()
    for k, m in ((13, 2), (28, 2), (21, 1), (27, 1024)):
        assert L.mhb_count_hashed_supported(k, m) == 1, (k, m)
    for k, m in ((12, 2), (29, 2), (11, 2), (31, 2), (27, 0), (27, 1025), (27, -1)):
        assert L.mhb_count_hashed_supported(k, m) == 0, (k, m)
        rc = L.mhb_count_solid_hashed(None, None, None, 100, k, m, None, None, None, 0, None, None, None, 0)
        assert rc == 1 and b"13 <= k <= 28" in L.mhb_last_error(), (k, m)
    assert all(lib.count_record_words(k) == 2 for k in range(13, 29))
    assert lib.count_record_words(12) == 1 and lib.count_record_words(29) == 3
