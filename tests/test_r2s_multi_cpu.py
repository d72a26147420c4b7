"""read2sdbg on several GPUs (mhb_read2sdbg_run_multi) without a GPU: the split of stage 1 and the mercy step over ranks,
emulated with the device code's host-callable pieces, against the oracle; the owner-range plan; the CLI's --gpus.

The emulation follows the worker: the reads are dealt in contiguous shares, every owner receives the records of its
leading-byte range from the ranks in rank order, runs stage 1 (stable bucket partition, kmsort, Lv2Postprocess) into
planes on the whole library's word grid, every rank ORs the planes of all owners over its share's words and runs the
mercy step over its share.  The records of one owner must come in global read order: concatenated in another rank order
the tie-heavy case gives other solid edges."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib, synth
from oracle import oracle as O

CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
N, LR, K, M = 4000, 100, 27, 2  # the `deep` case of test_r2s_cpu: tie classes far above the insertion-sort threshold


@pytest.fixture(scope="module")
def deep():
    b = np.ascontiguousarray(synth.synth_reads(N, LR, 1500, 0.01, seed=5).reshape(-1))
    reads = O.unpack_bin(b.tobytes(), reverse=True)
    nw = lib.r2s_s1_key_words(K)
    per = LR - K + 4
    recs = np.zeros((N * per, nw + 2), np.uint32)
    for r in range(N):  # every read's records in emission order: the global stage-1 input order
        w = reads.words[int(reads.word_off[r]):int(reads.word_off[r + 1])]
        for e in range(per):
            recs[r * per + e] = lib.selftest_r2s_s1_record(w, LR, K, e, r * LR)
    want = O.read2sdbg(reads, K, M, True, want_solid=True)
    return recs, per, want


def split_stage1(recs, per, first, rank_order):
    """solid bits of every base, multiplicity histogram and mercy count of the emulated multi-rank stage 1"""
    L_ = lib.load()
    nw = recs.shape[1] - 2
    n_ranks = len(first) - 1
    n_bits = N * LR
    bw = n_bits // 32 + 2
    bucket = recs[:, 0] >> 16
    owners = lib.plan_r2s_owners(np.bincount(bucket, minlength=65536).astype(np.uint64), n_ranks)
    planes = np.zeros((n_ranks, 4, bw), np.uint32)  # every owner's is_solid, no_in, no_out, any
    counting = np.zeros(65536, np.int64)
    for o, (lo, hi) in enumerate(owners):
        # the receive buffer: each rank's block of its share's records in this owner's range, in rank_order
        parts = []
        for s in rank_order:
            mine = recs[first[s] * per:first[s + 1] * per]
            b = mine[:, 0] >> 16
            parts.append(mine[(b >= lo) & (b <= hi)])
        got = np.concatenate(parts)
        got = got[np.argsort(got[:, 0] >> 16, kind="stable")]
        bounds = np.searchsorted(got[:, 0] >> 16, np.arange(65537))
        for b in np.nonzero(np.diff(bounds))[0]:
            seg = lib.selftest_kmsort(got[bounds[b]:bounds[b + 1]], nw)
            lib._check(L_.mhb_selftest_r2s_s1_group(seg.ctypes.data, len(seg), K, M, LR, N, 1, planes[o, 0].ctypes.data,
                                                    planes[o, 1].ctypes.data, planes[o, 2].ctypes.data,
                                                    planes[o, 3].ctypes.data, counting.ctypes.data))
    solid = np.zeros(n_bits, np.uint8)
    n_mercy = 0
    added = C.c_uint32()
    for s in range(n_ranks):
        if first[s] == first[s + 1]:
            continue
        w0, w_end = first[s] * LR // 32, first[s + 1] * LR // 32 + 2  # the share's words (PkgChunk::w0 / w_end)
        mine = planes[s].copy()
        for o in range(n_ranks):  # the plane merge
            if o != s:
                mine[:, w0:w_end] |= planes[o][:, w0:w_end]
        mercy = np.zeros(bw, np.uint32)
        for r in range(first[s], first[s + 1]):
            lib._check(L_.mhb_selftest_r2s_mercy_read(LR, N, r, K, mine[0].ctypes.data, mine[1].ctypes.data,
                                                      mine[2].ctypes.data, mine[3].ctypes.data, mercy.ctypes.data,
                                                      C.byref(added)))
            n_mercy += added.value
        bits = np.unpackbits((mine[0] | mercy).view(np.uint8), bitorder="little")
        solid[first[s] * LR:first[s + 1] * LR] = bits[first[s] * LR:first[s + 1] * LR]
    return solid, counting, n_mercy


def balanced(n_ranks):
    b = synth.synth_reads(N, LR, 1500, 0.01, seed=5).reshape(-1)
    return lib.plan_read_shares(b, N, n_ranks)


@pytest.mark.parametrize("first", [pytest.param(balanced(n), id=f"balanced{n}") for n in (1, 2, 3, 4)] +
                         [pytest.param([0, 1, 1377, 4000], id="uneven3-inside-a-word"), pytest.param([0, 3999, 4000], id="last-read"),
                          pytest.param([0, 0, 2001, 4000], id="empty-share")])
def test_split_stage1_matches_oracle(deep, first):
    recs, per, want = deep
    solid, counting, n_mercy = split_stage1(recs, per, first, range(len(first) - 1))
    assert n_mercy == want["n_mercy"]
    assert (counting == want["counting"]).all()
    assert (solid == np.unpackbits(want["is_solid"], bitorder="little")[:N * LR]).all()


def test_records_out_of_read_order_differ(deep):
    """the same split with the ranks' blocks in reverse order: the owners' kmsort sees another tie order"""
    recs, per, want = deep
    first = balanced(2)
    solid, counting, n_mercy = split_stage1(recs, per, first, [1, 0])
    assert not (solid == np.unpackbits(want["is_solid"], bitorder="little")[:N * LR]).all() or n_mercy != want["n_mercy"]


# ---- the owner plan ----
def test_owner_ranges_fold_and_cover():
    rng = np.random.default_rng(3)
    h = np.zeros(65536, np.uint64)
    h[rng.integers(0, 65536, 5000)] += rng.integers(1, 1000, 5000).astype(np.uint64)
    h256 = h.reshape(256, 256).sum(axis=1)
    for n in range(1, 17):
        rg = lib.plan_r2s_owners(h, n)
        assert rg[0][0] == 0 and rg[-1][1] == 65535
        for (lo, hi), (lo2, _) in zip(rg, rg[1:]):
            assert lo2 == hi + 1
        for lo, hi in rg:  # whole leading bytes, at least one per rank
            assert lo % 256 == 0 and hi % 256 == 255 and hi >= lo
        # rank 1's cut: the leading byte whose cumulative count is closest to 1 / n of the total
        if n > 1:
            cum = np.concatenate([[0], np.cumsum(h256)])
            c = rg[1][0] // 256
            t = int(h256.sum()) // n
            assert all(abs(int(cum[c]) - t) <= abs(int(cum[x]) - t) for x in range(1, 256 - (n - 1) + 1))


def test_owner_ranges_bad_args():
    with pytest.raises(Exception):
        lib.plan_r2s_owners(np.zeros(65536, np.uint64), 17)


# ---- the CLI ----
def _lib(tmp_path, n_reads):
    b = synth.synth_reads(max(n_reads, 1), 100, 1000, 0.0, seed=1)[:n_reads]
    p = str(tmp_path / "reads.lib")
    F.write_lib(p, b.reshape(-1), n_reads, n_reads * 100, 100)
    return p


def _read2sdbg(tmp_path, libp, extra, env=None):
    cmd = [CLI, "read2sdbg", "-k", "21", "-m", "2", "--host_mem", "1e9", "--read_lib_file", libp,
           "--output_prefix", str(tmp_path / "o")] + extra
    return subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=120)


@pytest.mark.skipif(not os.access(CLI, os.X_OK), reason="CLI not built")
@pytest.mark.parametrize("how", ["--gpus", "--gpus=", "MHB_GPUS"])
def test_cli_takes_gpus(tmp_path, how):
    libp = _lib(tmp_path, 1)
    if how == "MHB_GPUS":
        r = _read2sdbg(tmp_path, libp, [], env=dict(os.environ, MHB_GPUS="17"))
    else:
        r = _read2sdbg(tmp_path, libp, ["--gpus", "17"] if how == "--gpus" else ["--gpus=17"])
    assert r.returncode == 1 and "at most 16 GPUs" in r.stderr, r.stderr
    # fewer reads than ranks: one GPU (which this machine may not have), after the library is loaded
    r = _read2sdbg(tmp_path, libp, ["--gpus", "3"])
    assert "1 reads for 3 GPUs: running on one GPU" in r.stderr, r.stderr
    assert os.path.exists(str(tmp_path / "o") + ".mercy_cand.0")
