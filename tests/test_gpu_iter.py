"""GPU tests of `iterate` (SURVEY.md 8f N2): the CUDA path through the C ABI against the sets of iterative edges the
unmodified reference wrote (tests/golden_iter/, chain fixtures), against the oracle, through the CLI, and against the
digests of what the reference binary writes at 300 k reads (oracle/gen_golden_cli.py -> tests/golden_cli/cli.json)."""
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
from test_oracle_iter import contig_seqs, iter_cases, iter_inputs

pytestmark = pytest.mark.gpu

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


@pytest.mark.parametrize("step", iter_cases())
def test_iterate_host_matches_reference(step):
    files, data = iter_inputs(step)
    cs = contig_seqs(files)
    reads = O.unpack_bin(data, reverse=False)
    g = lib.iterate_host(cs.words, cs.word_off, cs.len, np.frombuffer(data, np.uint32), reads.n, step["k"], step["step"])
    assert g["n_edges"] == step["n_edges"] and g["edges"].shape[1] == step["words_per_edge"]
    assert F.sha256(g["edges"].tobytes()) == step["edges_sha256"]
    want, aligned = O.iterate(cs, reads, step["k"], step["step"])
    assert (g["edges"] == want).all() and g["n_aligned_reads"] == aligned
    mirror = lib.iterate_host(cs.words, cs.word_off, cs.len, np.frombuffer(data, np.uint32), reads.n, step["k"], step["step"],
                              selftest=True)
    assert g["n_flanks"] == mirror["n_flanks"] and g["n_candidates"] == mirror["n_candidates"]


def _run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r


_edge_set = GC.edge_set


def test_cli_iterate_on_fixture(tmp_path):
    step = [s for s in __import__("test_oracle_iter").ITER["steps"] if "chain" not in s and s["k"] == 29][0]
    files, _ = iter_inputs(step)
    p = str(tmp_path / "o")
    _run([OURS, "iterate", "-c", files[0], "-b", files[1], "-t", "4", "-k", "29", "-s", "20", "-o", p, "-r",
          os.path.join(ROOT, "tests", "golden_iter", "reads.lib.bin")])
    ks, u = _edge_set(p)
    assert ks == 49 and F.sha256(u.tobytes()) == step["edges_sha256"]


def test_cli_iterate_matches_reference_binary_at_300k_reads(tmp_path):
    """a 1.5 Mb repeat-rich synthetic genome cut into 30 - 200 bp pieces as the k = 21 contigs, then `iterate` 21 -> 29
    and 21 -> 41 over 300 k reads: the same set of edges as the reference binary writes"""
    ref = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))["iterate_300k"]
    contigs, bubble, binp = GC.iterate_inputs(tmp_path)
    t = str(min(32, os.cpu_count() or 8))
    for step in GC.ITER_STEPS:
        p = str(tmp_path / f"ours_{step}")
        r = _run([OURS, "iterate", "-c", contigs, "-b", bubble, "-t", t, "-k", "21", "-s", str(step), "-o", p, "-r", binp])
        gpu = [l for l in r.stderr.splitlines() if "iterate done" in l]
        print(f"iterate 21+{step}: {gpu[-1].split('- ')[-1] if gpu else ''}")
        want = ref[str(step)]
        assert want["k"] == 21 + step and want["n_edges"] > 100
        assert GC.edge_set_digest(p) == want
