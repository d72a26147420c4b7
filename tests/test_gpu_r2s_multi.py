"""read2sdbg on several GPUs (`megahit_core read2sdbg --gpus N`, mhb_read2sdbg_run_multi): every case runs the N-rank
build through the CLI and checks the reference's digests (canonical SdBG stream, item / tip / large-multiplicity
counts, P.counting) and that the canonical stream equals the single-GPU build's.  Ranks share a device when N exceeds the
device count, so all of it runs on one GPU."""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC
from test_oracle_r2s import R2S, r2s_reads

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def _one_process_only():
    """the compute mode of a device that admits one process only (ranks sharing it could not run), else None"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
    except (OSError, subprocess.TimeoutExpired):
        return None
    modes = [m.strip() for m in r.stdout.splitlines() if m.strip()]
    bad = [m for m in modes if m in ("Exclusive_Process", "Prohibited")]
    return bad[0] if bad and len(modes) < 3 else None  # up to 3 ranks: fewer devices are shared


_MODE = _one_process_only()
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")]


def _run(cmd, env=None, ok=True):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if ok:
        assert r.returncode == 0, (cmd, r.stderr[-3000:])
    return r


def _lib_prefix(name, tmp_path):
    """a `.lib_info` + `.bin` prefix of a fixture library (synthetic ones are written to tmp_path)"""
    if not name.startswith("synth:"):
        return os.path.join(ROOT, "tests", name, "reads.lib")
    a = R2S["synth"][name[6:]]
    p = str(tmp_path / "reads.lib")
    F.write_lib(p, np.frombuffer(r2s_reads(name), np.uint32), a["n_reads"], a["n_reads"] * a["read_len"], a["read_len"])
    return p


def _cmd(libp, p, k, m, mercy, gpus=None):
    cmd = [OURS, "read2sdbg", "-k", str(k), "-m", str(m), "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p,
           "--num_cpu_threads", "4", "--read_lib_file", libp] + (["--need_mercy"] if mercy else [])
    return cmd + (["--gpus", str(gpus)] if gpus else [])


def _single_stream(name, k, m, mercy):
    """the canonical stream of the single-GPU build of the same library (mhb_read2sdbg_host in this process)"""
    g = lib.read2sdbg_host(np.frombuffer(r2s_reads(name), np.uint32), _n_reads(name), k, m, bool(mercy))
    return lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])


def _n_reads(name):
    if name.startswith("synth:"):
        return R2S["synth"][name[6:]]["n_reads"]
    return F.read_lib_info(os.path.join(ROOT, "tests", name, "reads.lib"))[1]


def check_ranks(gold, tmp_path, ranks, env=None):
    libp = _lib_prefix(gold["lib"], tmp_path)
    k, m, mercy = gold["k"], gold["m"], gold["mercy"]
    want = _single_stream(gold["lib"], k, m, mercy)
    logs = {}
    for n in ranks:
        p = str(tmp_path / f"n{n}")
        r = _run(_cmd(libp, p, k, m, mercy, None if env else n), env=env)
        info, stream, table = F.canonical_sdbg(p)
        if _n_reads(gold["lib"]) >= n:
            assert info.num_files == n and all(os.path.exists(f"{p}.sdbg.{i}") for i in range(n))
            assert f"read2sdbg on {n} GPUs done" in r.stderr
        else:  # fewer reads than ranks: the single-GPU files
            assert "running on one GPU" in r.stderr
        assert os.path.exists(p + ".mercy_cand.0")
        assert stream == want, f"{n} ranks: not the single-GPU stream"
        assert F.sha256(stream) == gold["sdbg_sha256"]
        assert int(table[:, 0].sum()) == gold["sdbg_items"] and int(table[:, 1].sum()) == gold["sdbg_tips"]
        assert int(table[:, 2].sum()) == gold["sdbg_large_mul"] and info.words_per_tip_label == gold["sdbg_words_per_tip_label"]
        if m > 1:
            assert F.file_sha256(p + ".counting") == gold["counting_sha256"]
            if mercy:
                assert f"Number mercy: {gold['n_mercy']}" in r.stderr
        logs[n] = r.stderr
    return logs


@pytest.mark.parametrize("gold", [pytest.param(r, id=f"{r['lib'].split('/')[-1]}-k{r['k']}-m{r['m']}-mercy{r['mercy']}")
                                  for r in R2S["runs"]])
def test_golden_runs(gold, tmp_path):
    check_ranks(gold, tmp_path, (2, 3))


def test_gpus_from_the_environment(tmp_path):
    gold = [r for r in R2S["runs"] if r["lib"] == "golden/syn150_k27" and r["k"] == 27 and r["mercy"] == 1 and r["m"] == 2][0]
    assert "read2sdbg on 2 GPUs done" in check_ranks(gold, tmp_path, (2,), env=dict(os.environ, MHB_GPUS="2"))[2]


@pytest.mark.parametrize("env", [{"MHB_R2S_KMSORT_GLOBAL": "1"}, {"MHB_R2S_KM_CAP": "1024"}])
def test_kmsort_fallback_paths(env, tmp_path):
    gold = [r for r in R2S["runs"] if r["lib"] == "synth:deep" and r["k"] == 27][0]
    libp = _lib_prefix(gold["lib"], tmp_path)
    p = str(tmp_path / "n2")
    _run(_cmd(libp, p, 27, 2, True, 2), env=dict(os.environ, **env))
    assert F.sha256(F.canonical_sdbg(p)[1]) == gold["sdbg_sha256"]
    assert F.file_sha256(p + ".counting") == gold["counting_sha256"]


@pytest.mark.parametrize("m,mercy", [(2, True), (1, False)])
def test_300k_reads_against_the_reference_binary(tmp_path, m, mercy):
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"][f"m{m}"]
    libp = GC.r2s_lib(tmp_path)
    p = str(tmp_path / "n2")
    _run(_cmd(libp, p, 27, m, mercy, 2))
    assert GC.r2s_digest(p, m) == ref


def test_too_many_gpus(tmp_path):
    r = _run(_cmd(os.path.join(ROOT, "tests", "golden", "toy_k21", "reads.lib"), str(tmp_path / "o"), 21, 2, True, 17),
             ok=False)
    assert r.returncode == 1 and "at most 16 GPUs" in r.stderr


@pytest.mark.parametrize("n_reads", [1, 2])
def test_fewer_reads_than_ranks(n_reads, tmp_path):
    data = np.frombuffer(r2s_reads("golden/syn150_k27"), np.uint32).reshape(3000, -1)[:n_reads]
    libp = str(tmp_path / "reads.lib")
    F.write_lib(libp, data.reshape(-1), n_reads, n_reads * 150, 150)
    p, p1 = str(tmp_path / "n3"), str(tmp_path / "n1")
    r = _run(_cmd(libp, p, 27, 2, True, 3))
    assert f"{n_reads} reads for 3 GPUs: running on one GPU" in r.stderr
    _run(_cmd(libp, p1, 27, 2, True))
    for suffix in (".sdbg_info", ".counting"):  # the single-GPU files
        assert open(p + suffix, "rb").read() == open(p1 + suffix, "rb").read()


ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95",
       "--cleaning_rounds", "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2",
       "--bubble_level", "2", "--max_tip_len", "-1", "--careful_bubble"]  # src/megahit:866-899 with its defaults


@pytest.mark.skipif(not os.path.exists(REF), reason="the reference binary is not built")
def test_reference_assembles_the_n_file_graph(tmp_path):
    libp = os.path.join(ROOT, "tests", "golden", "syn150_k27", "reads.lib")
    outs = []
    for who in ("ref", "ours"):
        p = str(tmp_path / who)
        cmd = _cmd(libp, p, 27, 2, True, 3)
        _run([REF] + cmd[1:-2] if who == "ref" else cmd)
        if who == "ours":
            assert F.parse_sdbg_info(p).num_files == 3
        cp = str(tmp_path / f"contigs_{who}")
        _run([REF, "assemble", "-s", p, "-o", cp, "-t", "1"] + ASM)
        outs.append(open(cp + ".contigs.fa", "rb").read())
    assert outs[0] == outs[1] and len(outs[0]) > 0
