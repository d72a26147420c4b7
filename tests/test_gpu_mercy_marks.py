"""The per-read mercy marks (first_0_out / last_0_in, kmer_counter.cpp:307-367) of mhb_count_mark_mercy, word for word,
for every tip-set filter plan ($MHB_TIPSET_FILTER: the default, the global-memory filter, a filter of 1024 words and a
saturated one of 4 words, where every position probes the table) against a NumPy restatement built on
count_reference.py's solid edges and in/out flags (count_reference.reference_marks, any k).  The device tip set is built
from those same edges."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from count_reference import SENTINEL, read_layout as _layout, reference_marks
from count_wide_cases import library

pytestmark = pytest.mark.gpu

ARMS = ("default", "global", "1024", "1")


def device_marks(binw, n_reads, k, edges, aux, spec):
    """mhb_tipset_build + mhb_count_mark_mercy over the given solid edges with MHB_TIPSET_FILTER = spec
    -> first, last, tip-set header (uint32 words)"""
    import torch
    from megahit_b200 import lib
    L = lib.load()
    old = os.environ.pop("MHB_TIPSET_FILTER", None)
    if spec != "default":
        os.environ["MHB_TIPSET_FILTER"] = spec
    try:
        lens, starts = _layout(binw, n_reads)
        rec_off = np.append(starts, len(binw))
        edge_off = np.concatenate([[0], np.cumsum(np.maximum(lens - k, 0))])
        fixed = int(lens[0]) if n_reads and (lens == lens[0]).all() else 0
        d_bin = torch.from_numpy(np.concatenate([binw, np.zeros(8, np.uint32)]).view(np.int32)).cuda()
        d_ro = torch.from_numpy(rec_off.astype(np.int64)).cuda()
        d_eo = torch.from_numpy(edge_off.astype(np.int64)).cuda()
        rd = lib.DevReads(d_bin.data_ptr(), len(binw), n_reads, fixed, None if fixed else d_ro.data_ptr(),
                          None if fixed else d_eo.data_ptr())
        n_solid = len(edges)
        d_edges = torch.from_numpy(np.concatenate([edges.reshape(-1), np.zeros(4, np.uint32)]).view(np.int32)).cuda()
        d_aux = torch.from_numpy(np.concatenate([aux, np.zeros(8, np.uint8)])).cuda()
        n_tip = C.c_uint64(0)
        lib._check(L.mhb_count_tip_edges(None, C.c_void_p(d_aux.data_ptr()), n_solid, C.byref(n_tip)))
        need = L.mhb_tipset_bytes(n_tip.value, k)
        tips = torch.empty(need, dtype=torch.uint8, device="cuda")
        lib._check(L.mhb_tipset_build(None, C.c_void_p(d_edges.data_ptr()), C.c_void_p(d_aux.data_ptr()), n_solid, k,
                                      C.c_void_p(tips.data_ptr()), need, n_tip.value))
        first = torch.full((n_reads + 1,), -7, dtype=torch.int32, device="cuda")
        last = torch.full((n_reads + 1,), -7, dtype=torch.int32, device="cuda")
        lib._check(L.mhb_count_mark_mercy(None, C.byref(rd), k, C.c_void_p(tips.data_ptr()), need, n_tip.value,
                                          C.c_void_p(first.data_ptr()), C.c_void_p(last.data_ptr())))
        torch.cuda.synchronize()
        hdr = tips[:32].cpu().numpy().view(np.uint32).copy()
        return (first[:n_reads].cpu().numpy().view(np.uint32), last[:n_reads].cpu().numpy().view(np.uint32), hdr)
    finally:
        os.environ.pop("MHB_TIPSET_FILTER", None)
        if old is not None:
            os.environ["MHB_TIPSET_FILTER"] = old


def _check_all_arms(binw, n_reads, k, m):
    first, last, edges, aux, n_tip = reference_marks(binw, n_reads, k, m)
    headers = {}
    for spec in ARMS:
        f, l, hdr = device_marks(binw, n_reads, k, edges, aux, spec)
        bad_f, bad_l = np.flatnonzero(f != first), np.flatnonzero(l != last)
        assert not len(bad_f) and not len(bad_l), (spec, n_tip, bad_f[:5], bad_l[:5])
        headers[spec] = hdr
    return headers, n_tip, (first != SENTINEL).sum() + (last != SENTINEL).sum()


def _lib(name):
    from megahit_b200 import formats as F
    case = os.path.join(GOLDEN, name)
    binw = np.fromfile(os.path.join(case, "reads.lib.bin"), np.uint32)
    _, n_reads = F.read_lib_info(os.path.join(case, "reads.lib"))
    return binw, n_reads


@pytest.mark.parametrize("name,k,m", [("syn150_k27", 27, 2), ("lowcov_k21", 21, 2), ("polya_k27", 27, 2),
                                      ("tandem_k27", 27, 2), ("synvar_k21_m3", 21, 3)])
def test_marks_match_reference_on_fixtures(name, k, m):
    headers, _, _ = _check_all_arms(*_lib(name), k, m)
    assert headers["default"][6] == 1 and headers["global"][6] == 0  # resident flag
    assert headers["1"][2] == 4 and headers["1"][4] == 1  # 4 words, no fold: saturated, every probe reaches the table


@pytest.mark.parametrize("k", [13, 16, 28, 29, 31, 32, 39, 44, 47, 48, 63, 95, 127, 141, 199, 255])
def test_marks_match_reference_across_widths(k):
    """k = 13: generic kernel, one-word keys; 16 and 28: the two ends of the rolling kernel; 29 and 31: generic
    kernel, 3-word records.  Wider keys on a low-coverage variable-length library: 32, 39 (W = WR, the multiplicity
    shares the last edge word), 44 (an edge word of its own), 47 (W = WR - 1), 48 (the first 256-thread kernel), 63, 95,
    127, 141, 199, 255 (multi-word tip hashing and keys)"""
    if k <= 31:
        binw, n_reads = _lib("syn150_k27")
    else:
        binw, n_reads, _ = library(k, 900 + k, n_reads=800, genome_len=12_000)
    headers, n_tip, n_marked = _check_all_arms(binw, n_reads, k, 2)
    assert n_tip > 0 and n_marked > 0


def test_marks_match_reference_when_the_tip_set_outgrows_shared_memory():
    """unrelated random reads at m = 1: every read contributes its first and last edge as tips (~800 k tip edges),
    more than the shared-memory filter can hold at 3 bits per tip, so the default plan probes the global filter"""
    from megahit_b200 import formats as F
    rng = np.random.default_rng(20261015)
    n_reads, L, k = 400_000, 36, 27
    binw = F.pack_reads_fixed(rng.integers(0, 4, size=(n_reads, L), dtype=np.uint8)).reshape(-1)
    headers, n_tip, n_marked = _check_all_arms(binw, n_reads, k, 1)
    assert n_tip > 32 * (224 * 1024 // 4) // 3
    assert headers["default"][6] == 0 and headers["default"][4] > 1  # not resident; global filter of >= 32 bits per tip
