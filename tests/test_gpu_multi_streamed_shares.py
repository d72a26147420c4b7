"""`count --gpus N` and `seq2sdbg --gpus N` with every rank's share streamed from host memory: a chunk cap
(lib.set_read_chunk_limit for the count, lib.set_s2s_chunk_limit for seq2sdbg), set in a fresh process whose forked
workers inherit it, sends each share through its device in chunks, and every pass over the share - the bucket
histogram, each round's extraction into the owners, the count's mercy marks - goes over the chunks.

* count on the reference's fixtures (fixed and variable length, more mercy than solid edges, k >= 29) at N = 2 and 3
  with a cap of about a quarter of a share, alone and with forced count and SdBG rounds: every file byte for byte as
  without a cap, the reference's digests, and more than one chunk on every rank;
* a rank that owns no records, a share without mercy candidates or records, a cap below one read;
* seq2sdbg on the multi-k chain fixtures at N = 2 and 3, with and without SdBG rounds: the single-GPU stream and bytes
  (the owners' sort and emitter see their items in another order than with the share resident) and the reference's
  digests;
* the seeded 1 M-read library on 2 ranks: the files of the resident run.
Ranks share a device when N exceeds the device count, so all of it runs on one GPU."""
import glob
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN
from megahit_b200 import formats as F
from megahit_b200 import lib, synth
from test_gpu_count_multi import _MODE, _count_cmd, _digest, _gold, _mercy_cmd, _owner_loads, _run, check_gold
from test_gpu_count_multi import big_lib, big_single  # noqa: F401
from test_gpu_s2s_multi import CHAIN, _chain_cmd, check_chain
from test_gpu_sdbg_multi_rounds import (_caps, _chain_args, _check_against_one_gpu, _in_fresh_process, _loads, _rounds,
                                        _seq2sdbg_call, _single_gpu)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")]

STREAM_CASES = ["syn150_k27", "synvar_k21_m3", "lowcov_k21", "synvar_k31_m1"]


def _line(p, call, read_cap=0, s2s_cap=0, count_rounds=0, sdbg_rounds=0):
    """one run of the fresh process, its log behind '@@run <prefix>': the caps first (0 = none), then the call"""
    return (f"print('@@run {p}', file=sys.stderr, flush=True)\nlib.set_read_chunk_limit({read_cap})\n"
            f"lib.set_s2s_chunk_limit({s2s_cap})\nlib.set_round_limit({count_rounds})\n"
            f"lib.set_s2s_round_limit({sdbg_rounds})\n{call}\n")


def _count_call(libp, p, k, m, n):
    return f"lib.count_run({libp!r}, {p!r}, k={k}, m={m}, gpus={n})"


def _chunks(log, n, what):
    """every rank's chunks as its log line reports them ('<what> resident' = 0, '<what> in <c> chunks' = c)"""
    got = {int(r): int(c or 0) for r, c in re.findall(rf"rank (\d+): .*; {what} (?:resident|in (\d+) chunks)", log)}
    assert sorted(got) == list(range(n)), log[-3000:]
    return [got[r] for r in range(n)]


def _count_rounds(log):
    m = re.search(r"count plan: (\d+) rounds? over bucket ranges", log)
    assert m, log[-2000:]
    return int(m.group(1))


def _files(p):
    """every file of a run by its suffix"""
    return {f[len(p):]: open(f, "rb").read() for f in sorted(glob.glob(p + ".*"))}


def _read_starts(b):
    """the first word of every read of a `.bin` image, then its end"""
    starts, pos = [0], 0
    while pos < len(b):
        pos += 1 + (int(b[pos]) + 15) // 16
        starts.append(pos)
    return starts


def _read_chunks(b, n, cap):
    """the chunks of every rank's share of a `.bin` image under a cap of cap bytes, as the chunk planner cuts them"""
    starts = _read_starts(b)
    first = lib.plan_read_shares(b, len(starts) - 1, n)
    return [len(lib.plan_read_chunks(b[starts[first[r]]:starts[first[r + 1]]], first[r + 1] - first[r], cap)) - 1
            for r in range(n)]


def _quarter_share(path, n):
    """about a quarter of one of n shares of the input at path"""
    return max(16, os.path.getsize(path) // (4 * n))


# ------------------------------------------------------------------------------------------------
# 1. count --gpus N on the reference's fixtures: streamed, alone and in forced rounds
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", STREAM_CASES)
@pytest.mark.parametrize("n", [2, 3])
def test_count_streamed_shares(name, n, tmp_path):
    m, by_k = _gold(name)
    k, gold = next(iter(by_k.items()))
    libp = os.path.join(GOLDEN, name, "reads.lib")
    plain = str(tmp_path / "plain")
    r = _run(_count_cmd(libp, plain, k, m, gpus=n))
    assert _chunks(r.stderr, n, "reads") == [0] * n
    check_gold(plain, gold, n)
    most, _, top_bucket = _owner_loads(libp, k, n)
    count_cap, sdbg_cap = max(most // 3, top_bucket), _caps(_loads(r.stderr))[0]
    cap = _quarter_share(libp + ".bin", n)
    streamed, rounds = str(tmp_path / "streamed"), str(tmp_path / "rounds")
    _, _, _, logs = _in_fresh_process([
        _line(streamed, _count_call(libp, streamed, k, m, n), read_cap=cap),
        _line(rounds, _count_call(libp, rounds, k, m, n), read_cap=cap, count_rounds=count_cap, sdbg_rounds=sdbg_cap)])
    want = _read_chunks(np.fromfile(libp + ".bin", np.uint32), n, cap)
    assert min(want) > 1
    for p in (streamed, rounds):
        assert _chunks(logs[p], n, "reads") == want
        assert _files(p) == _files(plain)
        check_gold(p, gold, n)
    assert _count_rounds(logs[streamed]) == 1 and _rounds(logs[streamed]) == 1
    assert _count_rounds(logs[rounds]) > 1 or count_cap >= most
    assert _rounds(logs[rounds]) > 1


# ------------------------------------------------------------------------------------------------
# 2. edge cases, against the single-GPU count
# ------------------------------------------------------------------------------------------------
def _write_lib(b, tmp_path, tag):
    lens, pos = [], 0
    while pos < len(b):
        lens.append(int(b[pos]))
        pos += 1 + (lens[-1] + 15) // 16
    libp = str(tmp_path / f"{tag}.lib")
    F.write_lib(libp, b, len(lens), sum(lens), max(lens))
    return libp, len(lens)


def _streamed_against_one_gpu(b, k, m, n, cap, tmp_path, tag, count_rounds=0):
    """the streamed count on n ranks against the single-GPU count + seq2sdbg --need_mercy; its log"""
    libp, _ = _write_lib(b, tmp_path, tag)
    one = str(tmp_path / f"{tag}_one")
    _run(_count_cmd(libp, one, k, m))
    _run(_mercy_cmd(one, k))
    p = str(tmp_path / f"{tag}_n")
    _, _, _, logs = _in_fresh_process([_line(p, _count_call(libp, p, k, m, n), read_cap=cap, count_rounds=count_rounds)])
    assert _digest(p) == _digest(one)
    assert F.parse_edges_info(p).num_files == n and F.parse_sdbg_info(p).num_files == n
    return logs[p]


def _poly_a(n_reads, length):
    return np.tile(np.array([length] + [0] * ((length + 15) // 16), np.uint32), n_reads)


def test_streamed_ranks_that_own_no_records(tmp_path):
    # every record is the all-A edge, whose leading byte rank 0 owns: ranks 1 and 2 send records and own none
    b = _poly_a(60, 100)
    log = _streamed_against_one_gpu(b, 21, 1, 3, 64, tmp_path, "polya")
    assert _chunks(log, 3, "reads") == _read_chunks(b, 3, 64) == [10, 10, 10]
    for rank in (1, 2):
        assert re.search(rf"rank {rank}: \d+ reads, [1-9]\d* records sent, 0 owned", log), log[-3000:]


def test_streamed_share_without_candidates_or_records_and_a_cap_below_one_read(tmp_path):
    # one 2000-base read, then 100 reads of 20 bases (< k + 1): rank 1 gets only reads without a (k+1)-mer - no record,
    # no mark, no candidate - in 12-byte reads, five to a 64-byte chunk; rank 0's read of 504 bytes exceeds the cap and
    # is a chunk of its own
    long_read = synth.synth_reads_varlen(1, 2000, 2000, genome_len=4000, seed=3)
    short = synth.synth_reads_varlen(100, 20, 20, genome_len=4000, seed=4)
    b = np.concatenate([long_read, short])
    assert lib.plan_read_shares(b, 101, 2)[1] == 1
    log = _streamed_against_one_gpu(b, 21, 1, 2, 64, tmp_path, "empty")
    assert _chunks(log, 2, "reads") == _read_chunks(b, 2, 64) == [1, 20]
    assert re.search(r"rank 1: \d+ reads, 0 records sent", log), log[-3000:]


@pytest.mark.parametrize("n", [2, 3])
def test_streamed_read_by_read_in_rounds(n, tmp_path):
    # a cap below one read: every read is a chunk of its own, through count rounds and the mercy marks
    m, by_k = _gold("synvar_k21_m3")
    k = next(iter(by_k))
    libp = os.path.join(GOLDEN, "synvar_k21_m3", "reads.lib")
    b = np.fromfile(libp + ".bin", np.uint32)
    most, _, top_bucket = _owner_loads(libp, k, n)
    log = _streamed_against_one_gpu(b, k, m, n, 4, tmp_path, "perread", count_rounds=max(most // 3, top_bucket))
    first = lib.plan_read_shares(b, len(_read_starts(b)) - 1, n)
    assert _chunks(log, n, "reads") == [first[r + 1] - first[r] for r in range(n)] == _read_chunks(b, n, 4)
    assert _count_rounds(log) > 1


# ------------------------------------------------------------------------------------------------
# 3. seq2sdbg --gpus N on the chain fixtures
# ------------------------------------------------------------------------------------------------
def _chain_bytes(a):
    """about the bytes of a chain's sequence set: its edges, and its FASTA bases at four to a byte"""
    return os.path.getsize(a["input_prefix"] + ".edges.0") + sum(os.path.getsize(a[f]) // 4
                                                                 for f in ("contig", "bubble", "addi", "local"))


@pytest.mark.parametrize("name", CHAIN)
@pytest.mark.parametrize("n", [2, 3])
def test_seq2sdbg_streamed_shares(name, n, tmp_path):
    g, a = _chain_args(name)
    one = _single_gpu(_chain_cmd(name, str(tmp_path / "one"), None)[1])
    plain = str(tmp_path / "plain")
    r = _run(_chain_cmd(name, plain, n)[1])
    assert _chunks(r.stderr, n, "sequences") == [0] * n
    sdbg_cap = _caps(_loads(r.stderr))[0]
    cap = max(64, _chain_bytes(a) // (4 * n))
    streamed, rounds, tiny = (str(tmp_path / t) for t in ("streamed", "rounds", "tiny"))
    _, _, _, logs = _in_fresh_process([
        _line(streamed, _seq2sdbg_call(streamed, n, **a), s2s_cap=cap),
        _line(rounds, _seq2sdbg_call(rounds, n, **a), s2s_cap=cap, sdbg_rounds=sdbg_cap),
        _line(tiny, _seq2sdbg_call(tiny, n, **a), s2s_cap=4)])  # below one sequence: a chunk per sequence
    for p in (streamed, rounds, tiny):
        assert min(_chunks(logs[p], n, "sequences")) > 1, logs[p][-3000:]
        check_chain(p, g)
        _check_against_one_gpu(p, n, one)
    assert _rounds(logs[streamed]) == 1 and _rounds(logs[rounds]) > 1
    seqs = {int(r): int(c) for r, c in re.findall(r"rank (\d+): (\d+) sequences", logs[tiny])}
    assert _chunks(logs[tiny], n, "sequences") == [seqs[r] for r in range(n)]


# ------------------------------------------------------------------------------------------------
# 4. the seeded 1 M-read library
# ------------------------------------------------------------------------------------------------
def test_one_million_reads_streamed(big_lib, big_single, tmp_path):
    libp, _ = big_lib
    resident, streamed = str(tmp_path / "resident"), str(tmp_path / "streamed")
    _, _, _, logs = _in_fresh_process([
        _line(resident, _count_call(libp, resident, 27, 2, 2)),
        _line(streamed, _count_call(libp, streamed, 27, 2, 2), read_cap=_quarter_share(libp + ".bin", 2))])
    assert _chunks(logs[resident], 2, "reads") == [0, 0]
    assert min(_chunks(logs[streamed], 2, "reads")) > 1
    assert _files(streamed) == _files(resident)
    assert _digest(streamed) == big_single
