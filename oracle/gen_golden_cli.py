#!/usr/bin/env python
"""Mint the digests that the CLI-scale GPU tests compare against, by running the UNMODIFIED reference binary
(oracle/_ref/megahit_core_ref) on seeded synthetic libraries that the tests regenerate identically (only the digests are
committed):

* count + seq2sdbg --need_mercy on 1 M x 150 bp reads (tests/test_gpu_downstream.py, bench-scale parity);
* read2sdbg on 300 k reads, min count 2 with mercy and min count 1 without (tests/test_gpu_r2s.py);
* iterate 21 -> 29 and 21 -> 41 on 300 k reads from a repeat-rich genome, with that genome cut into pieces as the k = 21
  contigs (tests/test_gpu_iter.py).

    python oracle/gen_golden_cli.py

Output: tests/golden_cli/cli.json.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from megahit_b200 import formats as F  # noqa: E402
from megahit_b200 import synth  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
OUT = os.path.join(ROOT, "tests", "golden_cli", "cli.json")

COUNT_K, COUNT_M = 27, 2
R2S_RUNS = ((2, True), (1, False))  # (min count, need_mercy)
ITER_STEPS = (8, 20)


def _run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r


# ---- inputs, shared with the tests ----
def count_lib(d):
    """1 M x 150 bp, 30x, 1 % substitutions; returns (library prefix, `.bin` image, n_reads)"""
    n_reads, L = 1_000_000, 150
    b = synth.synth_reads(n_reads, L, 5 * n_reads, 0.01, seed=4242)
    libp = os.path.join(str(d), "reads.lib")
    F.write_lib(libp, b, n_reads, n_reads * L, L)
    return libp, b, n_reads


def r2s_lib(d):
    """300 k x 150 bp reads: buckets of ~600 stage-1 records, 37 M stage-1 records, 70+ M stage-2 items"""
    n_reads, L = 300_000, 150
    b = synth.synth_reads(n_reads, L, 5 * n_reads, 0.01, seed=777)
    libp = os.path.join(str(d), "reads.lib")
    F.write_lib(libp, b, n_reads, n_reads * L, L)
    return libp


def iterate_inputs(d):
    """300 k x 150 bp reads of a 1.5 Mb genome with three repeat families planted in it; the k = 21 contigs are that
    genome cut into pieces of 30 - 200 bp (flag 0) and the bubble file is empty.  Returns (contigs, bubbles, `.bin`)."""
    rng = np.random.default_rng(11)
    n_reads, L, G = 300_000, 150, 1_500_000
    g = rng.integers(0, 4, G, dtype=np.uint8)
    for rl, copies in ((30, 400), (45, 300), (70, 200)):
        rep = rng.integers(0, 4, rl, dtype=np.uint8)
        for p in rng.choice(G - rl, copies, replace=False):
            g[p:p + rl] = rep
    pos = rng.integers(0, G - L + 1, size=n_reads)
    b = g[pos[:, None] + np.arange(L)[None, :]]
    rc = rng.integers(0, 2, size=n_reads).astype(bool)
    b[rc] = 3 - b[rc][:, ::-1]
    e = rng.random(b.shape) < 0.01
    b[e] = (b[e] + rng.integers(1, 4, size=int(e.sum()), dtype=np.uint8)) & 3
    libp = os.path.join(str(d), "reads.lib")
    F.write_lib(libp, F.pack_reads_fixed(b), n_reads, n_reads * L, L)
    cuts = np.cumsum(rng.integers(30, 201, size=G // 30))
    cuts = [0] + [int(c) for c in cuts if c < G] + [G]
    contigs, bubbles = os.path.join(str(d), "k21.contigs.fa"), os.path.join(str(d), "k21.bubble_seq.fa")
    with open(contigs, "w") as f:
        for i, (a, z) in enumerate(zip(cuts[:-1], cuts[1:])):
            f.write(f">k21_{i} flag=0 multi=30.0000 len={z - a}\n" + "".join("ACGT"[c] for c in g[a:z]) + "\n")
    open(bubbles, "w").close()
    return contigs, bubbles, libp + ".bin"


# ---- digests, shared with the tests ----
def sdbg_digest(p):
    info, stream, table = F.canonical_sdbg(p)
    return {"sdbg": F.sha256(stream), "k": info.k, "wpt": info.words_per_tip_label, "items": int(table[:, 0].sum()),
            "tips": int(table[:, 1].sum()), "large": int(table[:, 2].sum())}


def count_digest(p):
    return {"edges": F.sha256(F.canonical_edges(p).tobytes()), "cand": F.file_sha256(p + ".cand"),
            "counting": F.file_sha256(p + ".counting"), **sdbg_digest(p)}


def r2s_digest(p, m):
    d = sdbg_digest(p)
    if m > 1:
        d["counting"] = F.file_sha256(p + ".counting")
    return d


def edge_set(prefix):
    """(k + 1 of the edges, sorted unique (k+1)-mer records) of an unsorted `iterate` output"""
    info = open(prefix + ".edges.info").read().split()
    assert info[0] == "kmer_size" and info[10] == "is_sorted" and info[11] == "0" and info[7] == "0"
    W, n = int(info[3]), int(info[9])
    e = np.fromfile(prefix + ".edges.0", np.uint32).reshape(-1, W)
    assert len(e) == n
    u = np.unique(e, axis=0)
    assert len(u) == n
    return int(info[1]), u


def edge_set_digest(prefix):
    k, u = edge_set(prefix)
    return {"k": k, "n_edges": len(u), "edges_sha256": F.sha256(u.tobytes())}


def main():
    t = str(min(32, os.cpu_count() or 8))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        d = os.path.join(tmp, "count")
        os.makedirs(d)
        libp, _, _ = count_lib(d)
        p = os.path.join(d, "ref")
        _run([REF, "count", "-k", str(COUNT_K), "-m", str(COUNT_M), "--host_mem", "3e10", "--mem_flag", "1",
              "--output_prefix", p, "--num_cpu_threads", t, "--read_lib_file", libp])
        _run([REF, "seq2sdbg", "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", p, "--num_cpu_threads", t,
              "-k", str(COUNT_K), "--kmer_from", "0", "--input_prefix", p, "--need_mercy"])
        out["count_1m"] = count_digest(p)

        d = os.path.join(tmp, "r2s")
        os.makedirs(d)
        libp = r2s_lib(d)
        out["read2sdbg_300k"] = {}
        for m, mercy in R2S_RUNS:
            p = os.path.join(d, f"ref_m{m}")
            _run([REF, "read2sdbg", "-k", "27", "-m", str(m), "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", p,
                  "--num_cpu_threads", t, "--read_lib_file", libp] + (["--need_mercy"] if mercy else []))
            out["read2sdbg_300k"][f"m{m}"] = r2s_digest(p, m)

        d = os.path.join(tmp, "iter")
        os.makedirs(d)
        contigs, bubbles, binp = iterate_inputs(d)
        out["iterate_300k"] = {}
        for step in ITER_STEPS:
            p = os.path.join(d, f"ref_{step}")
            _run([REF, "iterate", "-c", contigs, "-b", bubbles, "-t", t, "-k", "21", "-s", str(step), "-o", p, "-r", binp])
            out["iterate_300k"][str(step)] = edge_set_digest(p)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    json.dump(out, open(OUT, "w"), indent=1, sort_keys=True)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    if not os.path.exists(REF):
        raise SystemExit("build oracle/_ref first: make -C oracle ref")
    main()
