"""Pins the oracle's `iterate` (oracle/mhb_oracle_iter.c) and the host mirror of the device code (mhb_selftest_iterate)
against what the UNMODIFIED reference wrote for the wide-k matrix of tests/iter_wide_cases.py (every register class up to
k + step + 1 = 256, variable-length reads, a non-empty bubble file; oracle/gen_golden_iter_wide.py ->
tests/golden_iter_wide/iter_wide.json).  CPU only."""
import json
import os

import numpy as np
import pytest

import iter_wide_cases as IW
from conftest import ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import oracle as O
from test_oracle_iter import contig_seqs

WIDE = json.load(open(os.path.join(ROOT, "tests", "golden_iter_wide", "iter_wide.json")))


def wide_cases(kind="matrix"):
    return [pytest.param(c, id=f"k{c['k']}+{c['step']}") for c in WIDE[kind]]


def load_case(c, d, scale=False):
    """(contigs as O.Seqs, `.bin` words, n_reads, the written files) of a fixture case, regenerated from its seed"""
    case = (IW.make_scale_case if scale else IW.make_case)(c["k"], c["step"], c["seed"])
    paths = IW.write_case(case, str(d))
    assert case["n_reads"] == c["n_reads"]
    return contig_seqs(paths[:2]), case["bin"], case["n_reads"], paths


def test_matrix_covers_every_register_class():
    kn = {c["k"] + c["step"] + 1 for c in WIDE["matrix"]}
    assert [(c["k"], c["step"]) for c in WIDE["matrix"]] == IW.MATRIX and [(c["k"], c["step"]) for c in WIDE["scale"]] == IW.SCALE
    assert {12, 32, 34, 60, 64, 66, 128, 130, 142, 170, 240, 256} <= kn
    assert max(c["k"] + 1 for c in WIDE["matrix"]) == 240


@pytest.mark.parametrize("c", wide_cases())
def test_oracle_matches_reference_wide(c, tmp_path):
    cs, b, n, _ = load_case(c, tmp_path)
    edges, aligned = O.iterate(cs, O.unpack_bin(b.tobytes(), reverse=False), c["k"], c["step"])
    assert len(edges) == c["n_edges"] and edges.shape[1] == c["words_per_edge"]
    assert F.sha256(edges.tobytes()) == c["edges_sha256"]
    assert aligned == c["n_aligned"]


@pytest.mark.parametrize("c", wide_cases())
def test_host_mirror_matches_reference_wide(c, tmp_path):
    cs, b, n, _ = load_case(c, tmp_path)
    g = lib.iterate_host(cs.words, cs.word_off, cs.len, b, n, c["k"], c["step"], selftest=True)
    assert g["n_edges"] == c["n_edges"] and g["edges"].shape[1] == c["words_per_edge"]
    assert F.sha256(g["edges"].tobytes()) == c["edges_sha256"]
    assert g["n_flanks"] == c["n_flanks"] and g["n_aligned_reads"] == c["n_aligned"]
    assert c["all_mult_zero"] and ((g["edges"][:, -1] & 0xFFFF) == 0).all()
