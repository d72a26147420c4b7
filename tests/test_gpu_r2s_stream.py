"""GPU tests of read2sdbg on a streamed read library: the `.bin` image stays in host memory and goes through the device
in chunks (mhb_set_read_chunk_limit forces it), each chunk reversed into a chunk-sized package and, for variable-length
libraries, indexed on the device.  The reference's digests (tests/golden_r2s/r2s.json, tests/golden_cli/cli.json) and
the resident result are the yardsticks; the stream statistics show that the library really was streamed, in as many
passes as the plan implies.
"""
import json
import os

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from test_gpu_r2s import gpu_cases, n_reads_of
from test_gpu_r2s_rounds import (assert_reference, assert_same, ceil_div, gold_run, n_s1_records, read_lengths,
                                 s1_bucket_hist)
from test_oracle_r2s import r2s_reads

pytestmark = pytest.mark.gpu


def run(data, n_reads, k, m, mercy, cap=0, s1=0, s2=0, env=None):
    """read2sdbg_host with a chunk cap (0 = resident) and round caps; returns the result and the stream statistics"""
    env = env or {}
    lib.set_read_chunk_limit(cap)
    lib.set_r2s_round_limit(s1, s2)
    os.environ.update(env)
    try:
        g = lib.read2sdbg_host(np.frombuffer(data, np.uint32), n_reads, k, m, mercy)
        return g, lib.read_stream_stats()
    finally:
        lib.set_read_chunk_limit(0)
        lib.set_r2s_round_limit(0, 0)
        for k_ in env:
            del os.environ[k_]


def n_edge_positions(data, k):
    L = read_lengths(data)
    L = L[L >= k + 1]
    return int((L - k).sum())


def expected_passes(g, data, k, m, mercy):
    """passes over the reads of a streamed call: stage 1 (one, or a histogram pass + one per round), the mercy step
    with the stage-2 item count, stage 2 (one, or a histogram pass + one per round)"""
    has_edges = n_edge_positions(data, k) > 0
    p = 0
    if m > 1 and has_edges:
        p += 1 if g["n_rounds_s1"] == 1 else 1 + g["n_rounds_s1"]
    if has_edges:
        p += 1
    if g["n_sort_items"]:
        p += 1 if g["n_rounds_s2"] == 1 else 1 + g["n_rounds_s2"]
    return p


def check_streamed(g, st, one, data, n_reads, k, m, mercy, min_chunks=2):
    assert_same(g, one)
    if n_reads == 0:
        assert st["n_chunks"] == 0
        return
    assert st["n_chunks"] >= min_chunks
    assert st["n_passes"] == expected_passes(g, data, k, m, mercy), (st, g["n_rounds_s1"], g["n_rounds_s2"])
    L = read_lengths(data)
    fixed = L.size > 0 and (np.frombuffer(data, np.uint32)[0] > 0) and (L == L[0]).all()
    per_pass = len(data) + (0 if fixed else 8 * (n_reads + st["n_chunks"]))  # image + rebased record offsets
    assert st["h2d_bytes"] == st["n_passes"] * per_pass


@pytest.mark.parametrize("cap", ["fifth", "one_read"])
@pytest.mark.parametrize("gold", gpu_cases())
def test_streamed_matches_reference(gold, cap):
    """every GPU case of the reference fixtures streamed in ~5 chunks and one read per chunk"""
    data = r2s_reads(gold["lib"])
    n_reads, k, m, mercy = n_reads_of(gold["lib"], data), gold["k"], gold["m"], bool(gold["mercy"])
    one, st0 = run(data, n_reads, k, m, mercy)
    assert st0["n_chunks"] == 0 and st0["n_passes"] == 0
    assert_reference(one, gold)
    c = max(len(data) // 5, 1) if cap == "fifth" else 4
    g, st = run(data, n_reads, k, m, mercy, cap=c)
    assert_reference(g, gold)
    check_streamed(g, st, one, data, n_reads, k, m, mercy, min_chunks=5 if cap == "fifth" else n_reads)
    if cap == "one_read":
        assert st["n_chunks"] == n_reads


@pytest.mark.parametrize("lib_name", ["synth:deep", "synth:mid", "synth:wide"])
def test_streamed_rounds_on_kmsort_tie_libraries(lib_name):
    """kmsort's tie order decides the bytes on these libraries: streamed in ~7 chunks with 2 and ~8 rounds per stage,
    the rounds' records must reach the sort in global read order"""
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    one, _ = run(data, n_reads, 27, 2, True)
    n1, n2 = n_s1_records(data, 27), one["n_sort_items"]
    for div, lo_rounds in ((1.6, 2), (8, 8)):
        g, st = run(data, n_reads, 27, 2, True, cap=len(data) // 7, s1=int(n1 / div) + 1, s2=int(n2 / div) + 1)
        assert min(g["n_rounds_s1"], g["n_rounds_s2"]) >= lo_rounds, (div, g["n_rounds_s1"], g["n_rounds_s2"])
        assert_reference(g, gold)
        check_streamed(g, st, one, data, n_reads, 27, 2, True, min_chunks=7)


def test_streamed_plan_cuts_a_leading_byte_on_its_second_byte():
    """synth:deep streamed, with a stage-1 cap below its largest leading byte but not below any bucket"""
    lib_name = "synth:deep"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    h = s1_bucket_hist(data, 27)
    cap = int(h.reshape(256, 256).sum(axis=1).max()) - 1
    assert cap >= h.max()
    one, _ = run(data, n_reads, 27, 2, True)
    g, st = run(data, n_reads, 27, 2, True, cap=len(data) // 5, s1=cap)
    assert g["n_rounds_s1"] >= ceil_div(int(h.sum()), cap)
    assert_reference(g, gold)
    check_streamed(g, st, one, data, n_reads, 27, 2, True, min_chunks=5)


def test_streamed_rounds_with_global_kmsort():
    """the in-place kmsort walk on the records of a streamed round"""
    lib_name = "synth:deep"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    env = {"MHB_R2S_KMSORT_GLOBAL": "1"}
    one, _ = run(data, n_reads, 27, 2, True, env=env)
    g, st = run(data, n_reads, 27, 2, True, cap=len(data) // 6, s1=ceil_div(n_s1_records(data, 27), 5),
                s2=ceil_div(one["n_sort_items"], 3), env=env)
    assert g["n_rounds_s1"] >= 5 and g["n_rounds_s2"] >= 3
    assert_reference(g, gold)
    check_streamed(g, st, one, data, n_reads, 27, 2, True, min_chunks=6)


def edge_library(seed=11):
    """a variable-length library with chunk edges the plans below hit: blocks of [zero-length read, reads, zero-length
    read] of 96 image bytes each, some with reads shorter than k + 1, and one 5 000 bp read.  With a 96-byte cap every
    block is one chunk (zero-length reads first and last), the long read a chunk of its own."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, size=12000).astype(np.uint8)

    def read(L):
        p = int(rng.integers(0, len(genome) - L))
        b = genome[p:p + L].copy()
        err = rng.random(L) < 0.003
        b[err] = (b[err] + rng.integers(1, 4, size=int(err.sum()))) % 4
        return F.pack_read(3 - b[::-1] if rng.random() < 0.5 else b)

    empty = F.pack_read(np.zeros(0, np.uint8))
    recs = []
    for i in range(700):
        if i % 5 == 0:
            mid = [read(20), read(26), read(64), read(150)]  # 12 + 12 + 20 + 44 bytes
        elif i % 5 == 1:
            mid = [read(300), read(10)]                      # 80 + 8 bytes
        else:
            mid = [read(150), read(150)]                     # 44 + 44 bytes
        block = [empty] + mid + [empty]
        assert sum(len(r) for r in block) == 24
        recs += block
        if i == 350:
            recs.append(read(5000))
    data = np.concatenate(recs).astype(np.uint32).tobytes()
    return data, len(read_lengths(data))


@pytest.mark.parametrize("k,m,mercy", [(27, 2, True), (27, 2, False), (21, 3, True), (29, 1, False), (255, 1, False),
                                       (237, 2, True)])
def test_streamed_chunk_edges(k, m, mercy):
    """zero-length reads first and last in a chunk, reads shorter than k + 1, a read larger than the cap, one read per
    chunk, and a cap just below the image: the streamed result is the resident one"""
    data, n_reads = edge_library()
    one, _ = run(data, n_reads, k, m, mercy)
    assert one["n_items"] > 0 and (k > 27 or m == 1 or not mercy or one["n_mercy"] > 0)
    for cap in (96, 4, len(data) - 4):
        g, st = run(data, n_reads, k, m, mercy, cap=cap)
        check_streamed(g, st, one, data, n_reads, k, m, mercy)
        if cap == 96:
            assert st["n_chunks"] == 701  # 700 blocks and the long read
    # and with rounds on top
    if m > 1:
        g, st = run(data, n_reads, k, m, mercy, cap=96 * 37, s1=ceil_div(n_s1_records(data, k), 4),
                    s2=ceil_div(one["n_sort_items"], 4))
        assert g["n_rounds_s1"] >= 4 and g["n_rounds_s2"] >= 4
        check_streamed(g, st, one, data, n_reads, k, m, mercy)


def test_streamed_empty_library_and_reset():
    """no reads: nothing to stream; a call after the cap is reset to 0 is resident again"""
    g, st = run(b"", 0, 21, 2, True, cap=1 << 20)
    assert st["n_chunks"] == 0 and g["n_items"] == 0 and g["n_bytes"] == 0
    data = r2s_reads("golden/toy_k21")
    n_reads = n_reads_of("golden/toy_k21", data)
    g, st = run(data, n_reads, 21, 2, True, cap=1024)
    assert st["n_chunks"] > 1
    g2, st2 = run(data, n_reads, 21, 2, True)
    assert st2["n_chunks"] == 0 and st2["n_passes"] == 0
    assert_same(g, g2)


@pytest.mark.parametrize("m,mercy", [(2, True), (1, False)])
def test_cli_read2sdbg_streamed_at_300k_reads(tmp_path, m, mercy):
    """`megahit_core read2sdbg`'s in-process entry point on a streamed library, against the digests of what the
    reference binary writes for the same library"""
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"][f"m{m}"]
    libp = GC.r2s_lib(tmp_path)
    p = str(tmp_path / "ours")
    lib.set_read_chunk_limit(2 << 20)
    try:
        lib.read2sdbg_run(libp, p, k=27, m=m, need_mercy=mercy, host_mem=3e10,
                          num_cpu_threads=min(32, os.cpu_count() or 8))
        st = lib.read_stream_stats()
    finally:
        lib.set_read_chunk_limit(0)
    assert st["n_chunks"] >= 6
    assert GC.r2s_digest(p, m) == ref
