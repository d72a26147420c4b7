"""GPU tests of read2sdbg (SURVEY.md 8a A12, the 1-pass route: `megahit --kmin-1pass`, and what the driver runs for
--min-count 1): the CUDA path through the C ABI against

* the fixtures minted by the unmodified reference binary (tests/golden_r2s/r2s.json) - 28 runs: toy set, synthetic
  150 bp reads at k = 21 ... 141 and the reference's k = 255 / min-count 1 case, variable-length reads, poly-A,
  tandem repeats, end-overlapping reads (13 x more mercy than solid edges), and three seeded libraries whose buckets lie
  far above kmsort's insertion-sort threshold, where the reference's result depends on kmsort's order among tied
  records (a stable sort gives other bytes - checked on the oracle, tests/test_oracle_r2s.py);
* the oracle on the intermediate state (solid-edge bits are not visible through the ABI; the SdBG is);
* what the reference binary writes at 300 k reads (oracle/gen_golden_cli.py -> tests/golden_cli/cli.json), through the
  CLI (`megahit_core read2sdbg`).
"""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from oracle import oracle as O
from test_oracle_r2s import R2S, r2s_reads

pytestmark = pytest.mark.gpu

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def gpu_cases():
    out = []
    for r in R2S["runs"]:
        if r["m"] > 1 and r["k"] > 237:
            continue  # stage-1 records wider than 17 words: the CLI forwards these to the reference binary
        out.append(pytest.param(r, id=f"{r['lib'].split('/')[-1]}-k{r['k']}-m{r['m']}-mercy{r['mercy']}"))
    return out


def n_reads_of(lib_name, data):
    if lib_name.startswith("synth:"):
        return R2S["synth"][lib_name[6:]]["n_reads"]
    return F.read_lib_info(os.path.join(ROOT, "tests", lib_name, "reads.lib"))[1]


@pytest.mark.parametrize("gold", gpu_cases())
def test_read2sdbg_host_matches_reference(gold):
    data = r2s_reads(gold["lib"])
    g = lib.read2sdbg_host(np.frombuffer(data, np.uint32), n_reads_of(gold["lib"], data), gold["k"], gold["m"],
                           bool(gold["mercy"]))
    assert g["n_mercy"] == gold["n_mercy"]
    if gold["m"] > 1:
        assert F.sha256(O.counting_text(g["counting"])) == gold["counting_sha256"]
    assert g["n_items"] == gold["sdbg_items"] and g["n_tips"] == gold["sdbg_tips"]
    assert g["n_large_mul"] == gold["sdbg_large_mul"] and g["words_per_tip_label"] == gold["sdbg_words_per_tip_label"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


@pytest.mark.parametrize("env", [{"MHB_R2S_KMSORT_GLOBAL": "1"}, {"MHB_R2S_KM_CAP": "1024"}])
@pytest.mark.parametrize("lib_name", ["synth:deep", "synth:mid", "golden/polya_k27"])
def test_read2sdbg_kmsort_fallback_paths(lib_name, env):
    """the in-place walk on global memory - as the whole sort (MHB_R2S_KMSORT_GLOBAL) and as the per-bucket fall-back of
    the shared-memory form for buckets that exceed the tag capacity of a CTA (forced by a tiny capacity)"""
    gold = [r for r in R2S["runs"] if r["lib"] == lib_name and r["k"] == 27 and r["m"] == 2 and r["mercy"] == 1][0]
    data = r2s_reads(lib_name)
    os.environ.update(env)
    try:
        g = lib.read2sdbg_host(np.frombuffer(data, np.uint32), n_reads_of(lib_name, data), 27, 2, True)
    finally:
        for k_ in env:
            del os.environ[k_]
    assert g["n_mercy"] == gold["n_mercy"] and F.sha256(O.counting_text(g["counting"])) == gold["counting_sha256"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


def test_read2sdbg_matches_oracle_tables():
    """bucket table / w counts / ones, which the digests do not cover"""
    data = r2s_reads("golden/syn150_k27")
    reads = O.unpack_bin(data, reverse=True)
    o = O.read2sdbg(reads, 27, 2, True)
    g = lib.read2sdbg_host(np.frombuffer(data, np.uint32), 3000, 27, 2, True)
    assert g["bytes"] == o["bytes"]
    assert (g["bucket_table"][:, 1] == o["bucket_items"]).all() and (g["bucket_table"][:, 2] == o["bucket_tips"]).all()
    nz = o["bucket_items"] > 0
    assert (g["bucket_table"][nz, 0] == o["bucket_byte_off"][:-1][nz]).all()
    assert (g["w_count"] == o["w_count"]).all() and g["ones_in_last"] == o["ones_in_last"]
    assert (g["counting"] == o["counting"]).all()


def _run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r


@pytest.mark.parametrize("m,mercy", [(2, True), (1, False)])
def test_cli_read2sdbg_matches_reference_binary_at_300k_reads(tmp_path, m, mercy):
    """the sub-command itself, against the digests of what the reference binary writes for the same library; buckets of
    ~600 stage-1 records (kmsort's radix levels decide the tie order), 37 M stage-1 records, 70+ M stage-2 items"""
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"][f"m{m}"]
    libp = GC.r2s_lib(tmp_path)
    p = str(tmp_path / "ours")
    _run([OURS, "read2sdbg", "-k", "27", "-m", str(m), "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", p,
          "--num_cpu_threads", str(min(32, os.cpu_count() or 8)), "--read_lib_file", libp] + (["--need_mercy"] if mercy else []))
    assert os.path.exists(p + ".mercy_cand.0")
    assert GC.r2s_digest(p, m) == ref
