"""read2sdbg on several GPUs in rounds over bucket ranges (`megahit_core read2sdbg --gpus N`, mhb_read2sdbg_run_multi):
every owner takes its bucket range of a sort stage in rounds when the range does not fit its device at once.  The
rounds are forced here with lib.set_r2s_round_limit in a fresh process that then calls lib.read2sdbg_run(gpus=N) (the
forked workers inherit the caps).  The caps come from the loads rank 0 logs on an uncapped run of the same library -
the largest owner's records / items divided by 3 or 7, never below the largest bucket - and every capped run must
write the reference's digests, the single-GPU stream (canonical, and byte for byte once the ranks' files are joined in
rank order), and log more than one round.  Ranks share a device when N exceeds the device count, so all of it runs on
one GPU."""
import functools
import glob
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
from test_gpu_r2s_multi import _MODE, _cmd, _lib_prefix, _n_reads, _run
from test_oracle_r2s import R2S, r2s_reads

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")]


@functools.lru_cache(maxsize=None)
def _single(name, k, m, mercy):
    """(canonical stream, raw SdBG bytes) of the single-GPU build of the same library (mhb_read2sdbg_host)"""
    g = lib.read2sdbg_host(np.frombuffer(r2s_reads(name), np.uint32), _n_reads(name), k, m, bool(mercy))
    return lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"]), g["bytes"]


def _loads(stderr):
    """{stage: (largest owner, largest leading byte, largest bucket)} as rank 0 logs them"""
    return {int(s): tuple(int(x) for x in v) for s, *v in re.findall(
        r"read2sdbg stage (\d): largest owner (\d+), largest leading byte (\d+), largest bucket (\d+)", stderr)}


def _rounds(stderr):
    m = re.search(r"read2sdbg plan: stage 1 in (\d+) rounds?, stage 2 in (\d+) rounds?", stderr)
    assert m, stderr[-2000:]
    return int(m.group(1)), int(m.group(2))


def _with_caps(libp, k, m, mercy, n, runs, env=None, ok=True):
    """lib.read2sdbg_run(gpus=n) once per (prefix, s1 cap, s2 cap) in runs, in one fresh process that sets the caps
    first (no CUDA in it: the workers are forked).  Returns the process, its tag and pid, and each run's log."""
    tag = uuid.uuid4().hex
    code = (f"# {tag}\nimport sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\n"
            f"for p, s1, s2 in {runs!r}:\n"
            f"    print('@@run ' + p, file=sys.stderr, flush=True)\n"
            f"    lib.set_r2s_round_limit(s1, s2)\n"
            f"    lib.read2sdbg_run({libp!r}, p, k={k}, m={m}, need_mercy={bool(mercy)}, gpus={n})\n")
    pr = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                          env=dict(os.environ, **(env or {})))
    out, err = pr.communicate()
    r = subprocess.CompletedProcess(pr.args, pr.returncode, out, err)
    if ok:
        assert r.returncode == 0, r.stderr[-3000:]
    logs = dict(re.findall(r"@@run (\S+)\n(.*?)(?=@@run |\Z)", err, re.S))
    return r, tag, pr.pid, logs


def check_output(gold, p, n, stderr):
    """the reference's digests, the single-GPU stream and one file per rank"""
    k, m, mercy = gold["k"], gold["m"], gold["mercy"]
    want, want_bytes = _single(gold["lib"], k, m, mercy)
    info, stream, table = F.canonical_sdbg(p)
    assert info.num_files == n
    assert stream == want, "not the single-GPU stream"
    # the owners' rounds follow each other in bucket order: the ranks' files joined are the single-GPU byte stream
    assert b"".join(open(f"{p}.sdbg.{i}", "rb").read() for i in range(n)) == want_bytes
    assert F.sha256(stream) == gold["sdbg_sha256"]
    assert int(table[:, 0].sum()) == gold["sdbg_items"] and int(table[:, 1].sum()) == gold["sdbg_tips"]
    assert int(table[:, 2].sum()) == gold["sdbg_large_mul"] and info.words_per_tip_label == gold["sdbg_words_per_tip_label"]
    if m > 1:
        assert F.file_sha256(p + ".counting") == gold["counting_sha256"]
        if mercy:
            assert f"Number mercy: {gold['n_mercy']}" in stderr


def cap_of(loads, stage, div):
    most, _, top_bucket = loads[stage]
    return max(most // div, top_bucket)


def check_rounds(stderr, loads, s1, s2):
    """more than one round in every stage whose cap is below its largest owner's load"""
    r1, r2 = _rounds(stderr)
    if s1:
        assert r1 > 1 or s1 >= loads[1][0], (r1, s1, loads)
    else:
        assert r1 == (1 if 1 in loads else 0)
    if s2:
        assert r2 > 1 or s2 >= loads[2][0], (r2, s2, loads)
    else:
        assert r2 == 1
    return r1, r2


def _gold_id(r):
    return f"{r['lib'].split('/')[-1]}-k{r['k']}-m{r['m']}-mercy{r['mercy']}"


@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("gold", [pytest.param(r, id=_gold_id(r)) for r in R2S["runs"]])
def test_golden_runs_in_rounds(gold, n, tmp_path):
    libp = _lib_prefix(gold["lib"], tmp_path)
    k, m, mercy = gold["k"], gold["m"], gold["mercy"]
    p0 = str(tmp_path / "plain")
    r = _run(_cmd(libp, p0, k, m, mercy, n))
    if _n_reads(gold["lib"]) < n:
        assert "running on one GPU" in r.stderr
        return
    assert _rounds(r.stderr) == ((1 if m > 1 else 0), 1)  # everything fits: one round per stage
    check_output(gold, p0, n, r.stderr)
    loads = _loads(r.stderr)
    assert (1 in loads) == (m > 1) and 2 in loads
    # stage 1 alone (÷ 3), stage 2 alone (÷ 7), both (÷ 7, ÷ 3); m = 1 has no stage 1
    caps = [(0, cap_of(loads, 2, 7)), (0, cap_of(loads, 2, 3))]
    if m > 1:
        caps = [(cap_of(loads, 1, 3), 0), caps[0], (cap_of(loads, 1, 7), cap_of(loads, 2, 3))]
    if gold["lib"] in ("golden/polya_k27", "synth:deep"):
        # a cap below the largest leading byte cuts that byte on bucket ids (poly-A: in the stage where a byte holds
        # more than one bucket)
        cut = [s for s in loads if loads[s][2] < loads[s][1]]
        assert cut or gold["lib"] == "golden/polya_k27"
        for s in cut:
            c = (loads[s][2] + loads[s][1]) // 2
            caps.append((c, 0) if s == 1 else (0, c))
    runs = [(str(tmp_path / f"c{i}"), s1, s2) for i, (s1, s2) in enumerate(caps)]
    _, _, _, logs = _with_caps(libp, k, m, mercy, n, runs)
    for p, s1, s2 in runs:
        check_rounds(logs[p], loads, s1, s2)
        check_output(gold, p, n, logs[p])


@pytest.mark.parametrize("env", [{"MHB_R2S_KMSORT_GLOBAL": "1"}, {"MHB_R2S_KM_CAP": "1024"}])
def test_kmsort_fallback_paths_in_rounds(env, tmp_path):
    gold = [r for r in R2S["runs"] if r["lib"] == "synth:deep" and r["k"] == 27][0]
    libp = _lib_prefix(gold["lib"], tmp_path)
    r = _run(_cmd(libp, str(tmp_path / "plain"), 27, 2, True, 2))
    loads = _loads(r.stderr)
    runs = [(str(tmp_path / "c"), cap_of(loads, 1, 7), cap_of(loads, 2, 3))]
    _, _, _, logs = _with_caps(libp, 27, 2, True, 2, runs, env=env)
    p = runs[0][0]
    r1, r2 = check_rounds(logs[p], loads, runs[0][1], runs[0][2])
    assert r1 > 1 and r2 > 1
    check_output(gold, p, 2, logs[p])


def test_a_bucket_above_the_cap_is_refused(tmp_path):
    libp = os.path.join(ROOT, "tests", "golden", "polya_k27", "reads.lib")
    r = _run(_cmd(libp, str(tmp_path / "plain"), 27, 2, True, 2))
    top_bucket = _loads(r.stderr)[1][2]
    r, tag, pid, _ = _with_caps(libp, 27, 2, True, 2, [(str(tmp_path / "p"), top_bucket - 1, 0)], ok=False)
    assert r.returncode != 0
    assert "libmhb error 4" in r.stderr and re.search(r"bucket 0x[0-9a-f]{4} alone holds", r.stderr), r.stderr[-2000:]
    assert re.search(r"rank \d", r.stderr), r.stderr[-2000:]
    left = []
    for c in glob.glob("/proc/[0-9]*/cmdline"):
        try:
            if tag.encode() in open(c, "rb").read():
                left.append(c)
        except OSError:
            pass
    assert not left
    assert not glob.glob(f"/dev/shm/mhb_{pid}.*")


@pytest.mark.parametrize("m,mercy", [(2, True), (1, False)])
def test_300k_reads_in_rounds_against_the_reference_binary(tmp_path, m, mercy):
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["read2sdbg_300k"][f"m{m}"]
    libp = GC.r2s_lib(tmp_path)
    r = _run(_cmd(libp, str(tmp_path / "plain"), 27, m, mercy, 2))
    loads = _loads(r.stderr)
    runs = [(str(tmp_path / "c"), cap_of(loads, 1, 3) if m > 1 else 0, cap_of(loads, 2, 3))]
    _, _, _, logs = _with_caps(libp, 27, m, mercy, 2, runs)
    p = runs[0][0]
    r1, r2 = check_rounds(logs[p], loads, runs[0][1], runs[0][2])
    assert r2 > 1 and (r1 > 1 or m == 1)
    assert GC.r2s_digest(p, m) == ref
