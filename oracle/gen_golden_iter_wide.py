#!/usr/bin/env python
"""Mint the digests of the wide-k `iterate` tests with the UNMODIFIED reference binary (oracle/_ref/megahit_core_ref):
for every (k, step) of tests/iter_wide_cases.py (MATRIX, 500-odd reads, and SCALE, 200 k reads of 200 - 400 bp) the
seeded contig / bubble FASTA files and `.bin` image are written, `megahit_core iterate` is run on them with 1 and 4
threads (the set must not depend on it), and the digest of the edge set is stored with the reference's logged number of
flank k-mers and of aligned reads.  Only digests are committed; the tests regenerate the inputs from the seed.

    python oracle/gen_golden_iter_wide.py      ->  tests/golden_iter_wide/iter_wide.json
"""
from __future__ import annotations

import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import iter_wide_cases as IW  # noqa: E402
from oracle.gen_golden_iter import edge_set_digest  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
OUT = os.path.join(ROOT, "tests", "golden_iter_wide", "iter_wide.json")
SEED = 1


def run_reference(paths, k, step, prefix, threads):
    """edge-set digest + the last logged `Number of flank kmers` and `Total: T, aligned: A`"""
    c, b, r = paths
    p = subprocess.run([REF, "iterate", "-c", c, "-b", b, "-t", str(threads), "-k", str(k), "-s", str(step), "-o", prefix,
                        "-r", r], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    flanks = [int(x) for x in re.findall(r"Number of flank kmers: (\d+)", p.stderr)]
    total = re.findall(r"Total: (\d+), aligned: (\d+)", p.stderr)
    assert flanks and len(total) == 1, p.stderr[-2000:]
    return {**edge_set_digest(prefix), "n_flanks": flanks[-1], "n_reads": int(total[0][0]), "n_aligned": int(total[0][1])}


def mint(case, k, step, tmp, tag):
    paths = IW.write_case(case, os.path.join(tmp, tag))
    d = run_reference(paths, k, step, os.path.join(tmp, tag, "t1"), 1)
    assert run_reference(paths, k, step, os.path.join(tmp, tag, "t4"), 4) == d, "iterate depends on the thread count"
    assert d["n_reads"] == case["n_reads"] and d["kmer_size"] == k + step and d["all_mult_zero"]
    assert d["n_edges"] > 0 and d["n_aligned"] > 0, "vacuous case"
    d.update({"k": k, "step": step, "seed": SEED})
    print(tag, d["n_flanks"], d["n_aligned"], d["n_edges"], flush=True)
    return d


def main():
    res = {"matrix": [], "scale": []}
    with tempfile.TemporaryDirectory() as tmp:
        for k, step in IW.MATRIX:
            res["matrix"].append(mint(IW.make_case(k, step, SEED), k, step, tmp, f"k{k}_{step}"))
        for k, step in IW.SCALE:
            res["scale"].append(mint(IW.make_scale_case(k, step, SEED), k, step, tmp, f"scale_k{k}_{step}"))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if not os.path.exists(REF):
        raise SystemExit("build oracle/_ref first: make -C oracle ref")
    main()
