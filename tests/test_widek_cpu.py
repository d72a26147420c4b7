"""read2sdbg (m > 1) and iterate at the k where their sort records take the narrow layout (k > 237 / k + 1 > 240): the
oracle pinned against the reference-minted fixtures of tests/golden_widek/ (oracle/gen_golden_widek.py), the narrow
stage-1 layout's kmsort permutation on the host mirror, the stage-1 round bound, and the CLI no longer forwarding these
k to the reference.  CPU only."""
import ctypes as C
import json
import os
import stat
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib, synth
from oracle import gen_golden_widek as GW
from oracle import oracle as O
from test_oracle_iter import contig_seqs
from test_oracle_r2s import check_against_gold

GOLD = os.path.join(ROOT, "tests", "golden_widek")
WIDEK = json.load(open(os.path.join(GOLD, "widek.json")))
CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
_cache = {}


def widek_reads(lib_name):
    """(`.bin` bytes, n_reads) of a read2sdbg fixture library: committed, or seeded (digest-only)"""
    if lib_name not in _cache:
        if lib_name.startswith("synth:"):
            a = WIDEK["synth"][lib_name[6:]]
            b = synth.synth_reads(a["n_reads"], a["read_len"], a["genome_len"], a["err"], seed=a["seed"])
            _cache[lib_name] = (b.tobytes(), a["n_reads"])
        else:
            p = os.path.join(ROOT, "tests", lib_name, "reads.lib")
            _cache[lib_name] = (open(p + ".bin", "rb").read(), F.read_lib_info(p)[1])
    return _cache[lib_name]


def repeat_library(d):
    """the iterate fixtures' read library, regenerated from its seed: (path prefix, `.bin` words, n_reads)"""
    p = GW.repeat_lib(os.path.join(str(d), "rep300"))
    return p, np.fromfile(p + ".bin", np.uint32), WIDEK["repeats"]["n_reads"]


def iter_contigs(run):
    paths = [os.path.join(GOLD, run["contigs"]), os.path.join(GOLD, run["bubbles"])]
    return contig_seqs(paths), paths


def r2s_params():
    return [pytest.param(r, id=f"{r['lib'].split('/')[-1]}-k{r['k']}-m{r['m']}-mercy{r['mercy']}") for r in WIDEK["read2sdbg"]]


def iter_params():
    return [pytest.param(r, id=f"k{r['k']}-s{r['step']}") for r in WIDEK["iterate"]]


def test_fixture_covers_the_wide_k_range():
    assert {r["k"] for r in WIDEK["read2sdbg"]} == {239, 247, 255}
    assert {(r["m"], r["mercy"]) for r in WIDEK["read2sdbg"]} == {(2, 0), (2, 1), (3, 0), (3, 1)}
    assert [(r["k"], r["step"]) for r in WIDEK["iterate"]] == [(239, 2), (241, 14), (227, 28)]
    assert max(r["k"] + r["step"] + 1 for r in WIDEK["iterate"]) == 256
    assert all(r["n_edges"] > 0 and r["n_aligned"] > 0 for r in WIDEK["iterate"])


@pytest.mark.parametrize("gold", r2s_params())
def test_oracle_read2sdbg_matches_widek_reference(gold):
    data, _ = widek_reads(gold["lib"])
    s = O.read2sdbg(O.unpack_bin(data, reverse=True), gold["k"], gold["m"], bool(gold["mercy"]))
    assert s["n_mercy"] == gold["n_mercy"]
    assert F.sha256(O.counting_text(s["counting"])) == gold["counting_sha256"]
    check_against_gold(s, gold)


@pytest.mark.parametrize("gold", iter_params())
def test_oracle_iterate_matches_widek_reference(gold, tmp_path):
    _, b, _ = repeat_library(tmp_path)
    cs, _ = iter_contigs(gold)
    want, aligned = O.iterate(cs, O.unpack_bin(b.tobytes(), reverse=False), gold["k"], gold["step"])
    assert len(want) == gold["n_edges"] and want.shape[1] == gold["words_per_edge"]
    assert F.sha256(want.tobytes()) == gold["edges_sha256"] and aligned == gold["n_aligned"]


@pytest.mark.parametrize("gold", iter_params())
def test_iterate_host_mirror_matches_widek_reference(gold, tmp_path):
    """the host mirror of the device building blocks at k + 1 up to 242 (flank records wider than 17 words)"""
    _, b, n = repeat_library(tmp_path)
    cs, _ = iter_contigs(gold)
    m = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, gold["k"], gold["step"], selftest=True)
    assert F.sha256(m["edges"].tobytes()) == gold["edges_sha256"]
    assert m["n_flanks"] == gold["n_flanks"] and m["n_aligned_reads"] == gold["n_aligned"]


# ---- the narrow stage-1 layout on the host mirror ----
def s1_records(data, n_reads, k, read_len):
    """every stage-1 record of a fixed-length library in bucket input order (key words + 2 read_info words)"""
    reads = O.unpack_bin(data, reverse=True)
    per = read_len - k + 4
    nw = lib.r2s_s1_key_words(k)
    recs = np.zeros((n_reads * per, nw + 2), np.uint32)
    for r in range(n_reads):
        w = reads.words[int(reads.word_off[r]):int(reads.word_off[r + 1])]
        for e in range(per):
            recs[r * per + e] = lib.selftest_r2s_s1_record(w, read_len, k, e, r * read_len)
    return recs


def largest_buckets(recs, count):
    order = np.argsort(recs[:, 0] >> 16, kind="stable")  # the stable bucket partition
    recs = recs[order]
    bounds = np.searchsorted(recs[:, 0] >> 16, np.arange(65537))
    sizes = np.diff(bounds)
    return [recs[bounds[b]:bounds[b + 1]] for b in np.argsort(sizes)[::-1][:count]]


def narrow_of(wide, nw):
    """key words + row index (the bucket's input position); read_info of row i = the wide record's payload"""
    out = np.zeros((len(wide), nw + 1), np.uint32)
    out[:, :nw] = wide[:, :nw]
    out[:, nw] = np.arange(len(wide), dtype=np.uint32)
    return out


def oracle_kmsort(recs, nw):
    recs = np.ascontiguousarray(recs, np.uint32).copy()
    O.lib().mhbo_kmsort(C.c_void_p(recs.ctypes.data), C.c_int64(len(recs)), C.c_uint(nw), C.c_uint(recs.shape[1]))
    return recs


@pytest.fixture(scope="module")
def deep_buckets():
    data, n = widek_reads("synth:deep300")
    n = 4000  # buckets of 100 - 130 records
    L = WIDEK["synth"]["deep300"]["read_len"]
    data = data[: n * (1 + (L + 15) // 16) * 4]
    return {k: largest_buckets(s1_records(data, n, k, L), 4) for k in (237, 255)}


def test_kmsort_narrow_equals_wide_at_k237(deep_buckets):
    """k = 237: both layouts fit; the narrow one must leave every record where the wide one does"""
    nw = lib.r2s_s1_key_words(237)
    for bucket in deep_buckets[237]:
        assert len(bucket) > 4 * 64  # far above the insertion-sort threshold
        want = lib.selftest_kmsort(bucket, nw)
        for smem, cap, wcap in ((False, 65535, 0), (True, 65535, 0), (True, 65535, 70), (True, 100, 0)):
            got = lib.selftest_kmsort_narrow(narrow_of(bucket, nw), nw, smem=smem, cap=cap, wcap=wcap)
            assert (got[:, :nw] == want[:, :nw]).all()
            assert (bucket[got[:, nw], nw:] == want[:, nw:]).all(), (smem, cap, wcap)


def test_kmsort_narrow_matches_oracle_at_k255(deep_buckets):
    """k = 255: 17 key words; the narrow layout against the oracle's kmsort of the wide records"""
    nw = lib.r2s_s1_key_words(255)
    assert nw == 17
    for bucket in deep_buckets[255]:
        want = oracle_kmsort(bucket, nw)
        for smem, cap, wcap in ((False, 65535, 0), (True, 65535, 0), (True, 100, 0)):
            got = lib.selftest_kmsort_narrow(narrow_of(bucket, nw), nw, smem=smem, cap=cap, wcap=wcap)
            assert (got[:, :nw] == want[:, :nw]).all()
            assert (bucket[got[:, nw], nw:] == want[:, nw:]).all(), (smem, cap, wcap)
        assert (oracle_kmsort(narrow_of(bucket, nw), nw)[:, :nw] == want[:, :nw]).all()


@pytest.mark.parametrize("k", [239, 247, 253, 255])
def test_stage1_records_wide_k_match_oracle(k):
    """the stage-1 record builder at 16 and 17 key words against the oracle"""
    from test_r2s_cpu import oracle_s1_records
    rng = np.random.default_rng(k)
    for Ln in (k + 1, k + 2, 300):
        reads = O.unpack_bin(F.pack_read(rng.integers(0, 4, Ln, dtype=np.uint8)).tobytes(), reverse=True)
        want = oracle_s1_records(reads, 0, k, 777)
        w = reads.words[: int(reads.word_off[1])]
        for e in range(len(want)):
            assert (lib.selftest_r2s_s1_record(w, Ln, k, e, 777) == want[e]).all(), (k, Ln, e)


# ---- the stage-1 round plan ----
def test_stage1_layout_by_k():
    assert lib.r2s_s1_plan(237, 1000, 10, 1 << 40)["rec_words"] == 17   # wide: 15 key words + 2
    assert lib.r2s_s1_plan(239, 1000, 10, 1 << 40)["rec_words"] == 17   # narrow: 16 key words + row index
    assert lib.r2s_s1_plan(255, 1000, 10, 1 << 40)["rec_words"] == 18   # narrow: 17 key words + row index


@pytest.mark.parametrize("k", [239, 255])
def test_stage1_round_holds_fewer_than_2_32_records(k):
    big = 10_000_000_000
    p = lib.r2s_s1_plan(k, big, 1_000_000, 1 << 50)  # memory for all of them at once
    assert 0 < p["max_n"] < 2 ** 32
    assert lib.r2s_s1_plan(k, big, 1_000_000, 1 << 50, limit=2 ** 33)["max_n"] < 2 ** 32
    assert lib.r2s_s1_plan(k, 2 ** 32 - 1, 1_000_000, 1 << 50)["max_n"] == 0  # one pass still fits the row index
    assert lib.r2s_s1_plan(k, 2 ** 32, 1_000_000, 1 << 50)["max_n"] == 2 ** 32 - 1
    small = lib.r2s_s1_plan(k, big, 1_000_000, 40 << 30)  # 40 GB: memory bounds the round first
    assert 0 < small["max_n"] < 2 ** 32
    assert lib.r2s_s1_plan(k, big, 1_000_000, 1 << 50, limit=1000)["max_n"] == 1000


def test_stage1_round_bound_leaves_the_wide_layout_alone():
    assert lib.r2s_s1_plan(237, 10_000_000_000, 1_000_000, 1 << 50)["max_n"] == 0  # one pass, as before


# ---- the CLI ----
def _stub(tmp_path):
    stub = tmp_path / "ref_stub.sh"
    stub.write_text("#!/bin/sh\necho forwarded \"$@\" > \"$(dirname \"$0\")/forwarded.txt\"\nexit 0\n")
    stub.chmod(stub.stat().st_mode | stat.S_IXUSR)
    return stub


@pytest.mark.skipif(not os.access(CLI, os.X_OK), reason="CLI not built")
@pytest.mark.parametrize("cmd", ["iterate", "read2sdbg"])
def test_cli_keeps_wide_k_on_the_gpu_path(tmp_path, cmd):
    """without a GPU the device path fails; the stub reference is never reached"""
    if lib.device_count() > 0:
        pytest.skip("needs a machine without a GPU")
    stub = _stub(tmp_path)
    env = dict(os.environ, MHB_REFERENCE_CORE=str(stub))
    libp = os.path.join(ROOT, "tests", "golden_kmax", "syn300_k255", "reads.lib")
    if cmd == "iterate":
        c = tmp_path / "c.fa"
        c.write_text(">c0 flag=0 multi=1.0 len=4\nACGT\n")
        argv = [CLI, "iterate", "-c", str(c), "-b", str(c), "-r", libp + ".bin", "-k", "241", "-s", "14", "-o",
                str(tmp_path / "o")]
    else:
        argv = [CLI, "read2sdbg", "-k", "255", "-m", "2", "--need_mercy", "--host_mem", "1e9", "--read_lib_file", libp,
                "--output_prefix", str(tmp_path / "o")]
    r = subprocess.run(argv, capture_output=True, text=True, env=env, timeout=120)
    assert not (tmp_path / "forwarded.txt").exists()
    assert "forwarded" not in r.stderr
    assert r.returncode != 0 and "no CUDA device" in r.stderr
