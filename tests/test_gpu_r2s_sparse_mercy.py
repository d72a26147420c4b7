"""GPU tests of read2sdbg with the mercy candidates in the list form (mhb_set_r2s_sparse_mercy(1)): on one GPU the
library is streamed (mhb_set_read_chunk_limit) and every stage-1 round's candidates become a sorted list in host
memory, scattered chunk by chunk into chunk-sized planes for the mercy step; on several GPUs every owner publishes its
lists and every rank fetches the entries of its share.  The reference's digests (tests/golden_r2s/r2s.json,
tests/golden_cli/cli.json) and the plane-form result are the yardsticks; the statistics and the rank logs show which
form ran."""
import json
import os
import re
import subprocess
import sys
import uuid

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from test_gpu_r2s import gpu_cases, n_reads_of
from test_gpu_r2s_multi import _MODE, _cmd, _lib_prefix, _n_reads, _run
from test_gpu_r2s_multi_rounds import _loads, _rounds, cap_of, check_output
from test_gpu_r2s_rounds import assert_reference, assert_same, ceil_div, fit_cap, gold_run, n_s1_records
from test_oracle_r2s import R2S, r2s_reads

pytestmark = pytest.mark.gpu


def run(data, n_reads, k, m, mercy, cap=0, s1=0, s2=0, sparse=1, env=None):
    """read2sdbg_host with the list form forced (sparse = 1), a chunk cap and round caps; returns the result and the
    mercy statistics"""
    env = env or {}
    lib.set_r2s_sparse_mercy(sparse)
    lib.set_read_chunk_limit(cap)
    lib.set_r2s_round_limit(s1, s2)
    os.environ.update(env)
    try:
        g = lib.read2sdbg_host(np.frombuffer(data, np.uint32), n_reads, k, m, mercy)
        return g, lib.r2s_mercy_stats()
    finally:
        lib.set_r2s_sparse_mercy(0)
        lib.set_read_chunk_limit(0)
        lib.set_r2s_round_limit(0, 0)
        for k_ in env:
            del os.environ[k_]


def check_lists(g, ms, plane, n_reads, k, m, mercy):
    """the list form ran exactly when it should, and found the plane form's mercy edges"""
    assert_same(g, plane)
    assert g["n_mercy"] == plane["n_mercy"]
    lists = mercy and m > 1
    assert ms["sparse"] == lists
    if lists and g["n_mercy"]:
        assert ms["n_entries"] > 0 and ms["host_bytes"] == 8 * ms["n_entries"]


def mercy_cases():
    return [p for p in gpu_cases() if p.values[0]["mercy"]]


@pytest.mark.parametrize("div", [0, 1.6, 8])
@pytest.mark.parametrize("gold", mercy_cases())
def test_lists_match_reference(gold, div):
    """every need_mercy GPU case streamed in ~5 chunks with the list form, in one pass and with ~2 and ~8 rounds"""
    data = r2s_reads(gold["lib"])
    n_reads, k, m = n_reads_of(gold["lib"], data), gold["k"], gold["m"]
    plane, ms0 = run(data, n_reads, k, m, True, sparse=0)
    assert not ms0["sparse"]  # resident: the plane form, whatever the setting
    assert not run(data, n_reads, k, m, True)[1]["sparse"]
    n1 = n_s1_records(data, k) if m > 1 else 0
    s1 = int(n1 / div) + 1 if div and n1 else 0
    s2 = int(plane["n_sort_items"] / div) + 1 if div and plane["n_sort_items"] else 0
    if s1:  # raised to the largest bucket where one holds more (a bucket never spans two rounds)
        _, s1 = fit_cap(lambda c: run(data, n_reads, k, m, True, s1=c, sparse=0), s1)
    if s2:
        _, s2 = fit_cap(lambda c: run(data, n_reads, k, m, True, s1=s1, s2=c, sparse=0), s2)
    g, ms = run(data, n_reads, k, m, True, cap=max(len(data) // 5, 4), s1=s1, s2=s2)
    assert_reference(g, gold)
    check_lists(g, ms, plane, n_reads, k, m, True)
    if s1:
        assert g["n_rounds_s1"] >= min(int(div), ceil_div(n1, s1))


@pytest.mark.parametrize("lib_name", ["synth:deep", "synth:mid", "synth:wide"])
def test_lists_on_kmsort_tie_libraries(lib_name):
    """kmsort's tie order decides the bytes: one read per 64-byte chunk ... ~7 chunks, 2 and ~8 rounds per stage"""
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    plane, _ = run(data, n_reads, 27, 2, True, sparse=0)
    n1, n2 = n_s1_records(data, 27), plane["n_sort_items"]
    for div, cap in ((1.6, len(data) // 7), (8, len(data) // 7), (1, 4096)):
        g, ms = run(data, n_reads, 27, 2, True, cap=cap, s1=int(n1 / div) + 1, s2=int(n2 / div) + 1)
        assert_reference(g, gold)
        check_lists(g, ms, plane, n_reads, 27, 2, True)


def test_lists_with_global_kmsort():
    lib_name = "synth:deep"
    gold = gold_run(lib_name)
    data = r2s_reads(lib_name)
    n_reads = n_reads_of(lib_name, data)
    env = {"MHB_R2S_KMSORT_GLOBAL": "1"}
    plane, _ = run(data, n_reads, 27, 2, True, sparse=0, env=env)
    for s1 in (0, ceil_div(n_s1_records(data, 27), 5)):
        g, ms = run(data, n_reads, 27, 2, True, cap=len(data) // 6, s1=s1, env=env)
        assert_reference(g, gold)
        check_lists(g, ms, plane, n_reads, 27, 2, True)


def test_lists_at_300k_reads_against_the_cli_reference(tmp_path):
    """the 300 k-read library streamed with the list form and rounds, and `megahit_core read2sdbg`'s in-process entry
    point with the same settings, against the digests of what the reference binary writes"""
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"]["m2"]
    libp = GC.r2s_lib(tmp_path)
    data = open(libp + ".bin", "rb").read()
    n_reads = F.read_lib_info(libp)[1]
    plane, _ = run(data, n_reads, 27, 2, True, sparse=0)
    c1, c2 = ceil_div(n_s1_records(data, 27), 5), ceil_div(plane["n_sort_items"], 3)
    g, ms = run(data, n_reads, 27, 2, True, cap=len(data) // 9, s1=c1, s2=c2)
    assert g["n_rounds_s1"] >= 5
    check_lists(g, ms, plane, n_reads, 27, 2, True)
    p = str(tmp_path / "ours")
    lib.set_r2s_sparse_mercy(1)
    lib.set_read_chunk_limit(len(data) // 9)
    lib.set_r2s_round_limit(c1, c2)
    try:
        lib.read2sdbg_run(libp, p, k=27, m=2, need_mercy=True, host_mem=3e10, num_cpu_threads=min(32, os.cpu_count() or 8))
    finally:
        lib.set_r2s_sparse_mercy(0)
        lib.set_read_chunk_limit(0)
        lib.set_r2s_round_limit(0, 0)
    assert lib.r2s_mercy_stats()["sparse"]
    assert GC.r2s_digest(p, 2) == ref


def test_bad_mode():
    with pytest.raises(lib.MhbError):
        lib.set_r2s_sparse_mercy(2)


# ---- several GPUs: ranks share one device when N exceeds the device count ----
def _multi(libp, k, m, mercy, n, runs):
    """lib.read2sdbg_run(gpus=n) with the list form forced, once per (prefix, s1 cap, s2 cap), in one fresh process
    (the forked workers inherit the settings); returns each run's log"""
    tag = uuid.uuid4().hex
    code = (f"# {tag}\nimport sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\n"
            f"lib.set_r2s_sparse_mercy(1)\n"
            f"for p, s1, s2 in {runs!r}:\n"
            f"    print('@@run ' + p, file=sys.stderr, flush=True)\n"
            f"    lib.set_r2s_round_limit(s1, s2)\n"
            f"    lib.read2sdbg_run({libp!r}, p, k={k}, m={m}, need_mercy={bool(mercy)}, gpus={n})\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(re.findall(r"@@run (\S+)\n(.*?)(?=@@run |\Z)", r.stderr, re.S))


def _id(r):
    return f"{r['lib'].split('/')[-1]}-k{r['k']}-m{r['m']}"


@pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("gold", [pytest.param(r, id=_id(r)) for r in R2S["runs"] if r["mercy"] and r["m"] > 1])
def test_multi_gpu_lists(gold, n, tmp_path):
    """read2sdbg --gpus n with the list form on every rank, in one round per stage and in forced rounds: the
    reference's digests, the single-GPU stream, and no rank holds candidate planes of the whole library"""
    if _n_reads(gold["lib"]) < n:
        pytest.skip("fewer reads than ranks: one GPU")
    libp = _lib_prefix(gold["lib"], tmp_path)
    k, m = gold["k"], gold["m"]
    p0 = str(tmp_path / "plain")
    loads = _loads(_run(_cmd(libp, p0, k, m, True, n)).stderr)
    runs = [(str(tmp_path / "one"), 0, 0), (str(tmp_path / "rounds"), cap_of(loads, 1, 7), cap_of(loads, 2, 3))]
    logs = _multi(libp, k, m, True, n, runs)
    for (p, s1, _), log in zip(runs, (logs[p] for p, _, _ in runs)):
        check_output(gold, p, n, log)
        assert os.path.exists(p + ".mercy_cand.0")
        r1, _ = _rounds(log)
        assert (r1 > 1) == (s1 > 0 and s1 < loads[1][0])
        for r in range(n):
            assert f"rank {r}: mercy candidates as sorted lists: the solid plane of the whole library, the candidate " \
                   f"planes of my share only" in log
            assert re.search(rf"rank {r}: mercy candidates: \d+ list entries made, \d+ inside the share", log)
        made = sum(int(x) for x in re.findall(r"mercy candidates: (\d+) list entries made", log))
        got = sum(int(x) for x in re.findall(r"list entries made, (\d+) inside the share", log))
        assert made == got and made > 0
