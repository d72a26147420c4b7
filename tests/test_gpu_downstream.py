"""GPU tests at the scale of the benchmark and across several GPUs, against what the UNMODIFIED reference binary wrote
for the same inputs (digests minted by oracle/gen_golden_cli.py -> tests/golden_cli/cli.json, tests/golden/):

* bench-scale parity: 1 M synthetic 150 bp reads (123 M edge records; thousands of radix tiles per pass, every CTA of
  the persistent kernels busy) through the file-level commands, byte-compared with what the reference binary writes
  for the same library (canonical streams, SURVEY.md 8c) - also with the count stage forced into >= 5 rounds and
  through the fused build;
* the multi-GPU `count --gpus N` of the CLI (needs >= 2 devices).
"""
import json
import os
import subprocess

import pytest

from conftest import GOLDEN, ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
CLI = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))


def _run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r


def _ref_build(core, lib_prefix, p, k, m, threads=8, mercy=True):
    _run([core, "count", "-k", str(k), "-m", str(m), "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", p,
          "--num_cpu_threads", str(threads), "--read_lib_file", lib_prefix])
    _run([core, "seq2sdbg", "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", p, "--num_cpu_threads",
          str(threads), "-k", str(k), "--kmer_from", "0", "--input_prefix", p] + (["--need_mercy"] if mercy else []))


_digests = GC.count_digest


@pytest.fixture(scope="module")
def big_case(tmp_path_factory):
    """1 M x 150 bp, 30x, 1 % substitutions; the reference binary's output for it (k=27, m=2, mercy on)"""
    d = tmp_path_factory.mktemp("big")
    libp, b, n_reads = GC.count_lib(d)
    return {"lib": libp, "bin": b, "n_reads": n_reads, "ref": CLI["count_1m"], "dir": d}


def test_bench_scale_file_level_matches_reference_binary(big_case):
    p = str(big_case["dir"] / "ours")
    lib.count_run(big_case["lib"], p, k=27, m=2, host_mem=3e10, num_cpu_threads=8)
    lib.seq2sdbg_run(p, k=27, input_prefix=p, need_mercy=True, host_mem=3e10, num_cpu_threads=8)
    assert _digests(p) == big_case["ref"]


def test_bench_scale_count_in_rounds_matches_reference_binary(big_case):
    """A13: the count stage forced into >= 5 rounds at this size"""
    n_rec = big_case["n_reads"] * (150 - 27)
    p = str(big_case["dir"] / "rounds")
    lib.set_round_limit(n_rec // 6)
    try:
        lib.count_run(big_case["lib"], p, k=27, m=2, host_mem=3e10, num_cpu_threads=8)
    finally:
        lib.set_round_limit(0)
    lib.seq2sdbg_run(p, k=27, input_prefix=p, need_mercy=True, host_mem=3e10, num_cpu_threads=8)
    assert _digests(p) == big_case["ref"]


def test_bench_scale_fused_build_matches_reference_binary(big_case):
    g = lib.build_host(big_case["bin"].reshape(-1), big_case["n_reads"], 27, 2, need_mercy=True, want_edges=True)
    ref = big_case["ref"]
    assert F.sha256(g["edges"].tobytes()) == ref["edges"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == ref["sdbg"]
    assert (int(g["n_items"]), int(g["n_tips"]), int(g["n_large_mul"])) == (ref["items"], ref["tips"], ref["large"])


ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95",
       "--cleaning_rounds", "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2",
       "--bubble_level", "2", "--max_tip_len", "-1", "--careful_bubble"]  # src/megahit:866-899 with its defaults


# ------------------------------------------------------------------------------------------------
# several GPUs behind the CLI (C++ driver, one forked worker per GPU; needs >= 2 devices)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("syn150_klist", 59), ("lowcov_k21", 21), ("polya_k27", 27)])
def test_cli_multi_gpu_count_matches_reference(name, k, tmp_path):
    """`megahit_core count --gpus N` (mhb_count_run_multi): per-rank `.edges.<r>` / `.sdbg.<r>` + merged tables whose
    canonical streams equal the reference's digests; the following `seq2sdbg --need_mercy` finds the graph already
    built; the reference's `assemble` reads the N-file SdBG and gives the contigs of the reference-built graph"""
    n_dev = lib.device_count()
    if n_dev < 2:
        pytest.skip("needs at least 2 GPUs")
    n = min(n_dev, 4)
    gold_all = json.load(open(os.path.join(GOLDEN, name, "golden.json")))
    m, gold = gold_all["m"], gold_all["by_k"][str(k)]
    libp = os.path.join(GOLDEN, name, "reads.lib")
    p = str(tmp_path / "multi")
    r = subprocess.run([OURS, "count", "-k", str(k), "-m", str(m), "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p,
                        "--num_cpu_threads", "4", "--read_lib_file", libp, "--gpus", str(n)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    assert f"{n} GPUs" in r.stderr
    r2 = subprocess.run([OURS, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p, "--num_cpu_threads", "4",
                         "-k", str(k), "--kmer_from", "0", "--input_prefix", p, "--need_mercy"], capture_output=True, text=True)
    assert r2.returncode == 0, r2.stderr[-3000:]
    assert "nothing to do" in r2.stderr
    d = _digests(p)
    assert F.parse_edges_info(p).num_files == n and F.parse_sdbg_info(p).num_files == n
    if gold["n_solid"]:
        assert d["edges"] == gold["edges_sha256"]
    assert d["cand"] == gold["cand_sha256"] and d["counting"] == gold["counting_sha256"]
    assert d["sdbg"] == gold["sdbg_sha256"] and d["items"] == gold["sdbg_items"] and d["tips"] == gold["sdbg_tips"]
    # without --need_mercy the marker does not apply: the ordinary single-GPU seq2sdbg reads the N edge files
    q = str(tmp_path / "nomercy")
    r3 = subprocess.run([OURS, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", q, "--num_cpu_threads", "4",
                         "-k", str(k), "--kmer_from", "0", "--input_prefix", p], capture_output=True, text=True)
    assert r3.returncode == 0 and "nothing to do" not in r3.stderr, r3.stderr[-2000:]
    if os.path.exists(REF) and gold["sdbg_items"]:
        rp = str(tmp_path / "ref")
        _ref_build(REF, libp, rp, k, m, threads=4)
        outs = []
        for tag, pre in (("ref", rp), ("ours", p)):
            cp = str(tmp_path / ("contigs_" + tag))
            _run([REF, "assemble", "-s", pre, "-o", cp, "-t", "1"] + ASM)
            outs.append(open(cp + ".contigs.fa", "rb").read())
        assert outs[0] == outs[1]
