"""GPU tests of read2sdbg (m > 1) and iterate at the k where their sort records take the narrow layout (k > 237 / k + 1 >
240; DESIGN.md §4.10), against the digests the unmodified reference wrote (tests/golden_widek/widek.json): through the
C ABI and the CLI, with stage-1 rounds and with the read library streamed, and the narrow layout against the wide one
at the k where both fit."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_r2s as GR
from oracle import oracle as O
from oracle.gen_golden_iter import edge_set_digest
from test_gpu_r2s_rounds import assert_same, fit_cap, n_s1_records
from test_gpu_read_stream import chunk_limit
from test_widek_cpu import WIDEK, iter_contigs, iter_params, r2s_params, repeat_library, widek_reads

pytestmark = pytest.mark.gpu

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def host(gold, **kw):
    data, n = widek_reads(gold["lib"])
    return lib.read2sdbg_host(np.frombuffer(data, np.uint32), n, gold["k"], gold["m"], bool(gold["mercy"]), **kw)


def assert_r2s_reference(g, gold):
    assert g["n_mercy"] == gold["n_mercy"]
    assert F.sha256(O.counting_text(g["counting"])) == gold["counting_sha256"]
    assert g["n_items"] == gold["sdbg_items"] and g["n_tips"] == gold["sdbg_tips"]
    assert g["n_large_mul"] == gold["sdbg_large_mul"] and g["words_per_tip_label"] == gold["sdbg_words_per_tip_label"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


def assert_iter_reference(g, gold):
    assert g["n_edges"] == gold["n_edges"] and g["edges"].shape[1] == gold["words_per_edge"]
    assert F.sha256(g["edges"].tobytes()) == gold["edges_sha256"]
    assert g["n_flanks"] == gold["n_flanks"] and g["n_aligned_reads"] == gold["n_aligned"]


# ---- read2sdbg ----
@pytest.mark.parametrize("gold", r2s_params())
def test_read2sdbg_host_widek_matches_reference(gold):
    g = host(gold)
    assert_r2s_reference(g, gold)
    assert g["n_rounds_s1"] == 1


@pytest.mark.parametrize("gold", [p for p in r2s_params() if p.values[0]["m"] == 2 and p.values[0]["k"] in (239, 255)])
def test_read2sdbg_widek_in_rounds_and_streamed(gold):
    """stage 1 in about five rounds, then the library streamed in about four chunks: the same result"""
    data, n = widek_reads(gold["lib"])
    one = host(gold)
    lib.set_r2s_round_limit(0, 0)
    try:
        g, _ = fit_cap(lambda cap: (lib.set_r2s_round_limit(cap, 0), host(gold))[1], n_s1_records(data, gold["k"]) // 5)
    finally:
        lib.set_r2s_round_limit(0, 0)
    assert g["n_rounds_s1"] > 1
    assert_same(g, one)
    with chunk_limit(max(4, len(data) // 4)):
        s = host(gold)
    assert lib.read_stream_stats()["n_chunks"] > 1
    assert_same(s, one)
    assert_r2s_reference(s, gold)


@pytest.mark.parametrize("k,lib_name", [(237, "synth:deep300"), (237, "golden_kmax/syn300_k255"), (199, "synth:deep300")])
@pytest.mark.parametrize("m,mercy", [(2, 1), (3, 0)])
def test_read2sdbg_narrow_equals_wide_where_both_fit(k, lib_name, m, mercy):
    gold = {"lib": lib_name, "k": k, "m": m, "mercy": mercy}
    assert_same(host(gold, narrow=True), host(gold))


@pytest.mark.parametrize("gold", [p for p in r2s_params() if p.values[0]["k"] == 255 and p.values[0]["m"] == 2])
def test_cli_read2sdbg_widek(gold, tmp_path):
    if gold["lib"].startswith("synth:"):
        data, n = widek_reads(gold["lib"])
        a = WIDEK["synth"][gold["lib"][6:]]
        libp = str(tmp_path / "reads.lib")
        F.write_lib(libp, np.frombuffer(data, np.uint32), n, n * a["read_len"], a["read_len"])
    else:
        libp = os.path.join(ROOT, "tests", gold["lib"], "reads.lib")
    p = str(tmp_path / "ours")
    r = subprocess.run([OURS, "read2sdbg", "-k", "255", "-m", "2", "--host_mem", "4e9", "--output_prefix", p,
                        "--read_lib_file", libp] + (["--need_mercy"] if gold["mercy"] else []), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "forwarded" not in r.stderr
    d = GR.digest(p, 2)
    for key in ("sdbg_sha256", "sdbg_items", "sdbg_tips", "sdbg_large_mul", "counting_sha256"):
        assert d[key] == gold[key], key


# ---- iterate ----
@pytest.mark.parametrize("gold", iter_params())
def test_iterate_host_widek_matches_reference(gold, tmp_path):
    _, b, n = repeat_library(tmp_path)
    cs, _ = iter_contigs(gold)
    g = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, gold["k"], gold["step"])
    assert_iter_reference(g, gold)
    with chunk_limit(max(4, len(b) // 5)):
        s = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, gold["k"], gold["step"])
    assert lib.read_stream_stats()["n_chunks"] > 1
    assert_iter_reference(s, gold)


@pytest.mark.parametrize("gold", iter_params())
def test_cli_iterate_widek(gold, tmp_path):
    p, _, _ = repeat_library(tmp_path)
    _, paths = iter_contigs(gold)
    o = str(tmp_path / "ours")
    r = subprocess.run([OURS, "iterate", "-c", paths[0], "-b", paths[1], "-r", p + ".bin", "-k", str(gold["k"]), "-s",
                        str(gold["step"]), "-o", o], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "forwarded" not in r.stderr
    d = edge_set_digest(o)
    assert d["edges_sha256"] == gold["edges_sha256"] and d["n_edges"] == gold["n_edges"] and d["all_mult_zero"]


@pytest.mark.parametrize("gold", [p for p in iter_params() if p.values[0]["k"] in (239, 227)])
def test_iterate_narrow_equals_wide_where_both_fit(gold, tmp_path):
    """k + 1 = 240 and 228: the narrow flank index (key + row index, best value per key picked afterwards) gives the
    wide one's flank table, hence the same edges"""
    _, b, n = repeat_library(tmp_path)
    cs, _ = iter_contigs(gold)
    w = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, gold["k"], gold["step"])
    g = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, gold["k"], gold["step"], narrow=True)
    assert (g["edges"] == w["edges"]).all() and g["n_flanks"] == w["n_flanks"]
    assert g["n_candidates"] == w["n_candidates"] and g["n_aligned_reads"] == w["n_aligned_reads"]
    assert_iter_reference(g, gold)


def test_iterate_narrow_equals_wide_on_planted_flank_ties(tmp_path):
    """k + 1 = 240 on the seeded wide-k case whose contigs give one key two extension lengths and two extensions of one
    length: the narrow index must keep the same surviving value per key"""
    from test_oracle_iter_wide import load_case, wide_cases
    c = [p.values[0] for p in wide_cases() if p.values[0]["k"] == 239][0]
    cs, b, n, _ = load_case(c, tmp_path)
    w = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, c["k"], c["step"])
    g = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, c["k"], c["step"], narrow=True)
    assert (g["edges"] == w["edges"]).all() and g["n_flanks"] == w["n_flanks"] == c["n_flanks"]
    assert g["n_candidates"] == w["n_candidates"] and g["n_aligned_reads"] == w["n_aligned_reads"]
