"""GPU tests of the streamed read library: count, the staged fused build and iterate with the `.bin` image kept in host
memory and streamed through the device in chunks (mhb_set_read_chunk_limit forces it) give the same bytes as the
resident path and as the reference, and the stream statistics show that the library really was streamed."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, golden_cases
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from oracle import oracle as O
from test_oracle_iter import contig_seqs, iter_cases, iter_inputs

pytestmark = pytest.mark.gpu

CLI = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))


def _load(name):
    case = os.path.join(GOLDEN, name)
    bin_words = np.fromfile(os.path.join(case, "reads.lib.bin"), np.uint32)
    _, n_reads = F.read_lib_info(os.path.join(case, "reads.lib"))
    return case, bin_words, n_reads


def _lengths(bin_words, n_reads):
    out, pos = [], 0
    for _ in range(n_reads):
        L = int(bin_words[pos])
        out.append(L)
        pos += 1 + (L + 15) // 16
    return out


def _bytes_per_pass(bin_words, n_reads, n_chunks):
    """image bytes + the rebased offsets (two uint64 arrays of n + 1 per chunk) of a variable-length library"""
    lengths = _lengths(bin_words, n_reads)
    fixed = n_reads > 0 and lengths[0] > 0 and all(L == lengths[0] for L in lengths)
    return 4 * len(bin_words) + (0 if fixed else 16 * (n_reads + n_chunks))


class chunk_limit:
    def __init__(self, n_bytes, round_limit=0):
        self.n, self.r = n_bytes, round_limit

    def __enter__(self):
        lib.set_read_chunk_limit(self.n)
        if self.r:
            lib.set_round_limit(self.r)

    def __exit__(self, *a):
        lib.set_read_chunk_limit(0)
        lib.set_round_limit(0)


def _check_streamed_count(g, one, gold, bin_words, n_reads, oversized_ok=False):
    st = lib.read_stream_stats()
    assert g["n_solid"] == one["n_solid"] and (g["edges"] == one["edges"]).all()
    if gold["n_solid"]:
        assert F.sha256(g["edges"].tobytes()) == gold["edges_sha256"]
    assert (g["counting"] == one["counting"]).all()
    assert (g["cand_ids"] == one["cand_ids"]).all() and g["n_has_tips"] == one["n_has_tips"]
    if n_reads == 0:
        assert st["n_chunks"] == 0
        return st
    extra = st["n_passes"] - (g["n_rounds"] + 2)
    assert extra == 0 or (oversized_ok and extra == 1), (st, g["n_rounds"])
    assert st["h2d_bytes"] == st["n_passes"] * _bytes_per_pass(bin_words, n_reads, st["n_chunks"])
    return st


@pytest.mark.parametrize("name,k,m,gold", golden_cases())
def test_count_streamed_matches_golden(name, k, m, gold):
    import oracle_pipeline as OP
    case, bin_words, n_reads = _load(name)
    one = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
    assert lib.read_stream_stats()["n_chunks"] == 0  # resident
    with chunk_limit(max(4, 4 * len(bin_words) // 5)):
        g = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
    st = _check_streamed_count(g, one, gold, bin_words, n_reads)
    if n_reads > 1:
        assert st["n_chunks"] > 1
    assert F.sha256(OP.load_reads(case).bin_bytes(g["cand_ids"])) == gold["cand_sha256"]
    assert F.sha256(O.counting_text(g["counting"])) == gold["counting_sha256"]


@pytest.mark.parametrize("name,k,m,gold", [c for c in golden_cases() if c.values[0] in ("toy_k21", "syn150_k27", "synvar_k21_m3")])
def test_count_one_read_per_chunk(name, k, m, gold):
    """a cap below one read: every read is a chunk of its own"""
    _, bin_words, n_reads = _load(name)
    one = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
    with chunk_limit(4):
        g = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
    st = _check_streamed_count(g, one, gold, bin_words, n_reads)
    assert st["n_chunks"] == n_reads


@pytest.mark.parametrize("name,k,m,gold", [c for c in golden_cases() if c.values[0] in ("toy_k21", "syn150_k27", "synvar_k21_m3", "synvar_k31_m1", "polya_k27")])
@pytest.mark.parametrize("div", [3, 17])
def test_count_streamed_in_rounds(name, k, m, gold, div):
    """the round caps of the resident rounds test, with the library streamed: one pass per round"""
    _, bin_words, n_reads = _load(name)
    one = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
    n = int(one["n_edge_records"])
    if n == 0:
        pytest.skip("no edges")
    with chunk_limit(max(4, 4 * len(bin_words) // 5), max(1, n // div)):
        try:
            g = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
        except lib.MhbError as e:
            assert "more than one round can take" in str(e)  # a single bucket above the cap is reported
            return
    assert g["n_rounds"] > 1
    st = _check_streamed_count(g, one, gold, bin_words, n_reads, oversized_ok=True)
    assert st["n_chunks"] > 1


@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("toy_k21", 21), ("lowcov_k21", 21), ("synvar_k21_m3", 21), ("syn150_klist", 59)])
def test_fused_build_streamed_matches_reference(name, k):
    """mhb_build_host with a chunk cap takes the staged route (count streamed -> mercy edges from the `.cand` reads ->
    seq2sdbg): same edges / SdBG bytes"""
    gold_case = [c for c in golden_cases() if c.id == f"{name}-k{k}"][0]
    m, gold = gold_case.values[2], gold_case.values[3]
    _, bin_words, n_reads = _load(name)
    one = lib.build_host(bin_words, n_reads, k, m, need_mercy=True)
    with chunk_limit(max(4, 4 * len(bin_words) // 5)):
        g = lib.build_host(bin_words, n_reads, k, m, need_mercy=True, want_edges=True)
    assert lib.read_stream_stats()["n_chunks"] > 1
    assert g["n_solid"] == gold["n_solid"] and g["n_mercy"] == one["n_mercy"]
    if gold["n_solid"]:
        assert F.sha256(g["edges"].tobytes()) == gold["edges_sha256"]
    assert g["n_items"] == gold["sdbg_items"] and g["n_tips"] == gold["sdbg_tips"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


def test_bench_scale_count_streamed_in_rounds_matches_reference_binary(tmp_path):
    """1 M x 150 bp reads through `count` with 8 MiB chunks and rounds of n/6 records, then seq2sdbg: the reference
    binary's digests"""
    libp, _, n_reads = GC.count_lib(tmp_path)
    p = str(tmp_path / "streamed")
    with chunk_limit(8 << 20, n_reads * (150 - 27) // 6):
        lib.count_run(libp, p, k=27, m=2, host_mem=3e10, num_cpu_threads=8)
        st = lib.read_stream_stats()
    assert st["n_chunks"] > 1 and st["n_passes"] >= 8
    assert st["h2d_bytes"] == st["n_passes"] * n_reads * 44
    lib.seq2sdbg_run(p, k=27, input_prefix=p, need_mercy=True, host_mem=3e10, num_cpu_threads=8)
    assert GC.count_digest(p) == CLI["count_1m"]


@pytest.mark.parametrize("step", iter_cases())
def test_iterate_streamed_matches_reference(step):
    files, data = iter_inputs(step)
    cs = contig_seqs(files)
    reads = O.unpack_bin(data, reverse=False)
    b = np.frombuffer(data, np.uint32)
    one = lib.iterate_host(cs.words, cs.word_off, cs.len, b, reads.n, step["k"], step["step"])
    with chunk_limit(max(4, len(data) // 5)):
        g = lib.iterate_host(cs.words, cs.word_off, cs.len, b, reads.n, step["k"], step["step"])
    st = lib.read_stream_stats()
    assert st["n_chunks"] > 1 and st["n_passes"] == 1
    assert st["h2d_bytes"] == _bytes_per_pass(b, reads.n, st["n_chunks"])
    assert g["n_edges"] == step["n_edges"] and F.sha256(g["edges"].tobytes()) == step["edges_sha256"]
    assert (g["edges"] == one["edges"]).all()
    assert g["n_candidates"] == one["n_candidates"] and g["n_aligned_reads"] == one["n_aligned_reads"]


def test_iterate_streamed_at_300k_reads_matches_reference_binary(tmp_path):
    ref = CLI["iterate_300k"]
    contigs, bubble, binp = GC.iterate_inputs(tmp_path)
    cap = max(4, os.path.getsize(binp) // 7)
    for step in GC.ITER_STEPS:
        p = str(tmp_path / f"streamed_{step}")
        with chunk_limit(cap):
            lib.iterate_run(contigs, bubble, binp, p, 21, step, num_cpu_threads=8)
            st = lib.read_stream_stats()
        assert st["n_chunks"] > 1
        assert GC.edge_set_digest(p) == ref[str(step)]
