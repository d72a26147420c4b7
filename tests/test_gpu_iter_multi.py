"""iterate on several GPUs (`megahit_core iterate --gpus N`, mhb_iterate_run_multi): every case runs the single-GPU
iterate and the N-rank one on the same inputs and asserts that P.edges.0 and P.edges.info are byte-identical, and
checks the reference's digest where one exists.  Ranks share a device when N exceeds the device count, so all of it
runs on one GPU.  lib.iterate_run(gpus=) runs only in a fresh process that has not touched CUDA."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from megahit_b200 import formats as F
from oracle import gen_golden_cli as GC
from oracle.gen_golden_iter import edge_set_digest
from test_oracle_iter import ITER, iter_inputs
from test_widek_cpu import iter_contigs, iter_params, repeat_library

pytestmark = pytest.mark.gpu

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def _run(cmd, env=None):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, (cmd, r.stderr[-3000:])
    return r


def _iter_cmd(contigs, bubbles, reads, k, step, p, gpus=None):
    cmd = [OURS, "iterate", "-c", contigs, "-b", bubbles, "-r", reads, "-t", "4", "-k", str(k), "-s", str(step), "-o", p]
    return cmd + (["--gpus", str(gpus)] if gpus else [])


def _files(p):
    return open(p + ".edges.0", "rb").read(), open(p + ".edges.info", "rb").read()


def same_as_one_gpu(tmp_path, contigs, bubbles, reads, k, step, ranks, env=None):
    """runs 1 GPU and every N in ranks on the same inputs; returns the single-GPU prefix and the N-rank stderr"""
    one = str(tmp_path / "one")
    _run(_iter_cmd(contigs, bubbles, reads, k, step, one))
    want = _files(one)
    logs = {}
    for n in ranks:
        p = str(tmp_path / f"n{n}")
        r = _run(_iter_cmd(contigs, bubbles, reads, k, step, p, None if env else n), env=env)
        assert f"{n} GPUs" in r.stderr
        assert _files(p) == want, f"{n} ranks"
        logs[n] = r.stderr
    return one, logs


def _write_fasta(path, seqs):
    with open(path, "w") as f:
        for i, s in enumerate(seqs):
            f.write(f">c{i} flag=0 multi=5.0000 len={len(s)}\n" + "".join("ACGT"[b] for b in s) + "\n")
    return path


def _write_reads(path, reads):
    parts = [F.pack_reads_fixed(np.asarray(r, np.uint8)[None, :])[0] for r in reads]
    (np.concatenate(parts) if parts else np.zeros(0, np.uint32)).astype(np.uint32).tofile(path)
    return path


# ------------------------------------------------------------------------------------------------
# the reference's sets of iterative edges
# ------------------------------------------------------------------------------------------------
def _golden_step(step, tmp_path):
    files, data = iter_inputs(step)
    reads = str(tmp_path / "reads.bin")
    open(reads, "wb").write(data)
    return files, reads


@pytest.mark.parametrize("step", [pytest.param(s, id=f"{s.get('chain', 'repeats')}-k{s['k']}+{s['step']}")
                                  for s in ITER["steps"]])
def test_golden_iter_steps(step, tmp_path):
    files, reads = _golden_step(step, tmp_path)
    one, _ = same_as_one_gpu(tmp_path, files[0], files[1], reads, step["k"], step["step"], (2, 3))
    d = edge_set_digest(one)
    assert d["edges_sha256"] == step["edges_sha256"] and d["n_edges"] == step["n_edges"]


def test_gpus_from_the_environment(tmp_path):
    step = [s for s in ITER["steps"] if "chain" not in s and s["k"] == 29][0]
    files, reads = _golden_step(step, tmp_path)
    one, _ = same_as_one_gpu(tmp_path, files[0], files[1], reads, 29, 20, (2,), env=dict(os.environ, MHB_GPUS="2"))
    assert edge_set_digest(one)["edges_sha256"] == step["edges_sha256"]


@pytest.fixture(scope="module")
def inputs_300k(tmp_path_factory):
    return GC.iterate_inputs(tmp_path_factory.mktemp("iter300k"))


@pytest.mark.parametrize("step", GC.ITER_STEPS)
def test_300k_reads_against_the_reference_binary(step, inputs_300k, tmp_path):
    want = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["iterate_300k"][str(step)]
    one, _ = same_as_one_gpu(tmp_path, *inputs_300k, 21, step, (2, 3))
    assert GC.edge_set_digest(one) == want


@pytest.mark.parametrize("gold", iter_params())
def test_wide_k(gold, tmp_path):
    """k + 1 > 240 builds the narrow flank table on every rank"""
    p, _, _ = repeat_library(tmp_path)
    _, paths = iter_contigs(gold)
    one, _ = same_as_one_gpu(tmp_path, paths[0], paths[1], p + ".bin", gold["k"], gold["step"], (2,))
    d = edge_set_digest(one)
    assert d["edges_sha256"] == gold["edges_sha256"] and d["n_edges"] == gold["n_edges"] and d["all_mult_zero"]


# ------------------------------------------------------------------------------------------------
# shapes
# ------------------------------------------------------------------------------------------------
K, STEP = 21, 8
KN = K + STEP + 1


def _genome_case(seed=5):
    """a genome with repeats, cut into 30 - 200 bp contigs, and variable-length reads (40 - 250 bp) from both strands"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, 100_000)
    for rl, copies in ((30, 60), (45, 40), (70, 30)):
        rep = rng.integers(0, 4, rl)
        for q in rng.choice(len(g) - rl, copies, replace=False):
            g[q:q + rl] = rep
    cuts = np.cumsum(rng.integers(30, 201, size=len(g) // 30))
    cuts = [0] + [int(c) for c in cuts if c < len(g)] + [len(g)]
    contigs = [g[a:z] for a, z in zip(cuts[:-1], cuts[1:])]
    reads = []
    for _ in range(20_000):
        L = int(rng.integers(40, 251))
        s = int(rng.integers(0, len(g) - L))
        reads.append(3 - g[s:s + L][::-1] if rng.random() < 0.5 else g[s:s + L])
    return contigs, reads


def _case(tmp_path, contigs, reads, ranks=(2, 3), k=K, step=STEP):
    c = _write_fasta(str(tmp_path / "c.fa"), contigs)
    b = _write_fasta(str(tmp_path / "b.fa"), [])
    r = _write_reads(str(tmp_path / "r.bin"), reads)
    one, logs = same_as_one_gpu(tmp_path, c, b, r, k, step, ranks)
    info = F.parse_edges_info(one)
    return np.fromfile(one + ".edges.0", np.uint32).reshape(-1, info.words_per_edge), logs


@pytest.mark.parametrize("k,step", [(21, 8), (29, 20)])
def test_variable_length_library(k, step, tmp_path):
    contigs, reads = _genome_case()
    e, _ = _case(tmp_path, contigs, reads, k=k, step=step)
    assert len(e) > 100


@pytest.mark.parametrize("n_reads", [0, 1, 2])
def test_fewer_reads_than_ranks(n_reads, tmp_path):
    contigs, reads = _genome_case()
    _case(tmp_path, contigs, reads[:n_reads], ranks=(3,))


def _one_lead_contigs(n, seed):
    """contigs of exactly k + step + 1 bases that are their own canonical form and end in CGTA: read back as reads, each
    gives one edge, and every edge starts with the same byte (the record holds the canonical (k+step+1)-mer reversed)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        x = rng.integers(0, 4, KN)
        x[0] = 0
        x[-4:] = [1, 2, 3, 0]
        out.append(x)
    return out


@pytest.mark.parametrize("what", ["none", "short", "palindromic"])
def test_no_flanks(what, tmp_path):
    reads = _one_lead_contigs(40, seed=1)
    rng = np.random.default_rng(2)
    half = rng.integers(0, 4, (K + 1) // 2)
    contigs = {"none": [], "short": [rng.integers(0, 4, K) for _ in range(30)],
               "palindromic": [np.concatenate([half, 3 - half[::-1]])]}[what]
    e, logs = _case(tmp_path, contigs, reads)
    assert len(e) == 0 and "Number of flank kmers: 0" in logs[2]


def test_reads_shorter_than_the_edges(tmp_path):
    contigs, reads = _genome_case()
    e, _ = _case(tmp_path, contigs, [r[:KN - 1] for r in reads[:3000]])
    assert len(e) == 0


def test_a_share_without_candidates(tmp_path):
    """the first half of the bases are random reads, which match no flank: rank 0 of 2 finds no candidate"""
    contigs, reads = _genome_case()
    rng = np.random.default_rng(9)
    junk = [rng.integers(0, 4, len(r)) for r in reads[:5000]]
    e, logs = _case(tmp_path, contigs, junk + reads[:5000], ranks=(2,))
    assert len(e) > 0 and "rank 0: 5000 reads (resident), 0 candidates" in logs[2]


def test_an_owner_that_receives_nothing(tmp_path):
    cs = _one_lead_contigs(50, seed=3)
    e, logs = _case(tmp_path, cs, cs + cs[:10], ranks=(2, 3))
    assert len(e) == 50 and len(np.unique(e[:, 0] >> 24)) == 1
    for n, log in logs.items():
        assert sum(", 0 received, 0 owned" in ln for ln in log.splitlines()) == n - 1, log


# ------------------------------------------------------------------------------------------------
# streamed shares, through lib.iterate_run in a fresh process
# ------------------------------------------------------------------------------------------------
def test_streamed_shares(tmp_path):
    step = [s for s in ITER["steps"] if "chain" not in s and s["k"] == 21][0]
    files, reads = _golden_step(step, tmp_path)
    one = str(tmp_path / "one")
    _run(_iter_cmd(files[0], files[1], reads, step["k"], step["step"], one))
    p = str(tmp_path / "streamed")
    cap = max(4, os.path.getsize(reads) // 9)  # about four chunks per rank of 2
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from megahit_b200 import lib; "
            "lib.set_read_chunk_limit(int(sys.argv[2])); "
            "lib.iterate_run(sys.argv[3], sys.argv[4], sys.argv[5], sys.argv[6], int(sys.argv[7]), int(sys.argv[8]), gpus=2)")
    r = _run([sys.executable, "-c", code, ROOT, str(cap), files[0], files[1], reads, p, str(step["k"]), str(step["step"])])
    assert _files(p) == _files(one)
    for rank in (0, 1):
        line = [ln for ln in r.stderr.splitlines() if f"rank {rank}: " in ln][0]
        assert int(line.split("(")[1].split(" chunks")[0]) > 1, line
    assert edge_set_digest(p)["edges_sha256"] == step["edges_sha256"]


# ------------------------------------------------------------------------------------------------
# a chain: iterate --gpus 2, then seq2sdbg --gpus 2 on its edges, assembled by the reference
# ------------------------------------------------------------------------------------------------
ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95",
       "--cleaning_rounds", "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2",
       "--bubble_level", "2", "--max_tip_len", "-1", "--careful_bubble"]  # src/megahit:866-899 with its defaults


@pytest.mark.skipif(not os.path.exists(REF), reason="the reference binary is not built")
def test_chain_through_seq2sdbg_and_assemble(tmp_path):
    step = [s for s in ITER["steps"] if s.get("chain") == "chain_syn150"][0]
    case = os.path.join(GOLDEN, "chain_syn150")
    g = json.load(open(os.path.join(case, "chain.json")))
    k, kf = g["k"], g["k_from"]
    assert (step["k"], step["k"] + step["step"]) == (kf, k)
    files, reads = _golden_step(step, tmp_path)
    outs = []
    for n in (1, 2):
        e = str(tmp_path / f"edges{n}")
        _run(_iter_cmd(files[0], files[1], reads, kf, step["step"], e, n if n > 1 else None))
        s = str(tmp_path / f"graph{n}")
        cmd = [OURS, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", s, "--num_cpu_threads", "4",
               "-k", str(k), "--kmer_from", str(kf), "--input_prefix", e,
               "--contig", os.path.join(case, f"k{kf}.contigs.fa"), "--bubble", os.path.join(case, f"k{kf}.bubble_seq.fa"),
               "--addi_contig", os.path.join(case, f"k{kf}.addi.fa"), "--local_contig", os.path.join(case, f"k{kf}.local.fa")]
        _run(cmd + (["--gpus", str(n)] if n > 1 else []))
        info, stream, _ = F.canonical_sdbg(s)
        assert F.sha256(stream) == g["sdbg_sha256"]
        cp = str(tmp_path / f"contigs{n}")
        _run([REF, "assemble", "-s", s, "-o", cp, "-t", "1"] + ASM)
        outs.append(open(cp + ".contigs.fa", "rb").read())
    assert outs[0] == outs[1] and len(outs[0]) > 0
