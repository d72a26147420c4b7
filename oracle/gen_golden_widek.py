#!/usr/bin/env python
"""Mint the wide-k fixtures of `read2sdbg` (m > 1, k > 237) and `iterate` (k + 1 > 240) with the UNMODIFIED reference
binary (oracle/_ref/megahit_core_ref): the k range where both use their narrow sort records (DESIGN.md §4.10).

* read2sdbg at k = 239, 247, 255, m = 2, 3, with and without --need_mercy, on 300 bp reads: the committed
  golden_kmax/syn300_k255 library and a seeded deep library (regenerated at test time, only digests committed) whose
  buckets lie far above kmsort's insertion-sort threshold, where the tie order decides the output.  Every run is
  repeated with 1 thread and --mem_flag 0 and must give the same digests.
* iterate at (k, step) = (239, 2), (241, 14), (227, 28) - k + step + 1 up to 256 - on a seeded 300 bp library with
  repeats longer than k + 1 (so that the contigs end there), with the contigs and bubbles of the reference's own
  `read2sdbg` + `assemble` at k (committed), run with 1 and 4 threads.

    python oracle/gen_golden_widek.py      ->  tests/golden_widek/
"""
from __future__ import annotations

import json
import os

import numpy as np
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from megahit_b200 import formats as F  # noqa: E402
from megahit_b200 import synth  # noqa: E402
from oracle.gen_golden_iter import edge_set_digest  # noqa: E402
from oracle.gen_golden_r2s import digest as r2s_digest  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
OUT = os.path.join(ROOT, "tests", "golden_widek")
SYN300 = os.path.join(ROOT, "tests", "golden_kmax", "syn300_k255", "reads.lib")
# 900x on a 2 kb genome: (k-1)-mer groups and buckets of 100 - 200 stage-1 records at k = 239 ... 255
SYNTH = {"deep300": dict(n_reads=6000, read_len=300, genome_len=2000, err=0.004, seed=301)}
R2S_K = [239, 247, 255]
# the iterate library: 120x of 300 bp reads over a 30 kb genome with four copies each of a 250 and a 275 bp repeat
REPEATS = dict(n_reads=12000, read_len=300, genome_len=30000, repeats=(250, 275), copies=4, err=0.001, seed=302)
ITER_KS = [(239, 2), (241, 14), (227, 28)]


def run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    if r.returncode != 0:
        sys.stderr.write(r.stderr.decode()[-3000:])
        raise SystemExit("reference failed: " + " ".join(cmd))
    return r.stderr.decode()


def write_synth(name, prefix):
    a = SYNTH[name]
    b = synth.synth_reads(a["n_reads"], a["read_len"], a["genome_len"], a["err"], seed=a["seed"])
    F.write_lib(prefix, b, a["n_reads"], a["n_reads"] * a["read_len"], a["read_len"])


def repeat_lib(prefix):
    a = REPEATS
    rng = np.random.default_rng(a["seed"])
    g = rng.integers(0, 4, a["genome_len"], dtype=np.uint8)
    for rl in a["repeats"]:
        unit = rng.integers(0, 4, rl, dtype=np.uint8)
        for p in np.sort(rng.choice(np.arange(0, a["genome_len"] - rl, 1000), a["copies"], replace=False)):
            g[p:p + rl] = unit
    n, L = a["n_reads"], a["read_len"]
    pos = rng.integers(0, len(g) - L + 1, size=n)
    b = g[pos[:, None] + np.arange(L)[None, :]]
    flip = rng.integers(0, 2, size=n).astype(bool)
    b[flip] = 3 - b[flip][:, ::-1]
    e = rng.random(b.shape) < a["err"]
    b[e] = (b[e] + rng.integers(1, 4, size=int(e.sum()), dtype=np.uint8)) & 3
    F.write_lib(prefix, F.pack_reads_fixed(b), n, n * L, L)
    return prefix


def ref_r2s(lib, prefix, k, m, mercy, threads, mem_flag):
    cmd = [REF, "read2sdbg", "-k", str(k), "-m", str(m), "--host_mem", "4e9", "--mem_flag", str(mem_flag),
           "--output_prefix", prefix, "--num_cpu_threads", str(threads), "--read_lib_file", lib]
    return run(cmd + (["--need_mercy"] if mercy else []))


def mint_r2s(tmp):
    libs = {"golden_kmax/syn300_k255": SYN300}
    for name in SYNTH:
        libs["synth:" + name] = os.path.join(tmp, name)
        write_synth(name, libs["synth:" + name])
    runs = []
    for lib, path in libs.items():
        for k in R2S_K:
            for m in (2, 3):
                for mercy in (0, 1):
                    p = os.path.join(tmp, "r")
                    log = ref_r2s(path, p, k, m, mercy, 4, 1)
                    d = r2s_digest(p, m)
                    ref_r2s(path, p + "x", k, m, mercy, 1, 0)
                    assert r2s_digest(p + "x", m) == d, f"{lib} k={k} m={m}: depends on threads / pass boundaries"
                    n_mercy = [line.split()[-1] for line in log.splitlines() if "Number mercy" in line]
                    d.update({"lib": lib, "k": k, "m": m, "mercy": mercy, "n_mercy": int(n_mercy[0]) if n_mercy else 0})
                    runs.append(d)
                    print("read2sdbg", lib, k, m, mercy, d["sdbg_items"], d["sdbg_tips"], d["n_mercy"], flush=True)
    return runs


def mint_iter(tmp):
    lib = repeat_lib(os.path.join(tmp, "rep300"))
    runs = []
    for k, step in ITER_KS:
        p = os.path.join(tmp, f"s{k}")
        ref_r2s(lib, p, k, 2, 1, 4, 1)
        a = os.path.join(tmp, f"a{k}")
        run([REF, "assemble", "-s", p, "-o", a, "-t", "4"])
        names = {}
        for suf in ("contigs.fa", "bubble_seq.fa"):
            names[suf] = f"k{k}.{suf}"
            shutil.copy(f"{a}.{suf}", os.path.join(OUT, names[suf]))
        res = []
        for threads in (1, 4):
            o = os.path.join(tmp, f"i{k}_{threads}")
            log = run([REF, "iterate", "-c", f"{a}.contigs.fa", "-b", f"{a}.bubble_seq.fa", "-t", str(threads), "-k", str(k),
                       "-s", str(step), "-o", o, "-r", lib + ".bin"])
            flanks = [int(x) for x in re.findall(r"Number of flank kmers: (\d+)", log)]
            total = re.findall(r"Total: (\d+), aligned: (\d+)", log)
            res.append({**edge_set_digest(o), "n_flanks": flanks[-1], "n_aligned": int(total[0][1])})
        assert res[0] == res[1], "iterate depends on the thread count"
        d = res[0]
        assert d["n_edges"] > 0 and d["kmer_size"] == k + step and d["all_mult_zero"]
        d.update({"k": k, "step": step, "contigs": names["contigs.fa"], "bubbles": names["bubble_seq.fa"]})
        runs.append(d)
        print("iterate", k, step, d["n_flanks"], d["n_aligned"], d["n_edges"], flush=True)
    return runs


def main():
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        res = {"synth": SYNTH, "repeats": REPEATS, "read2sdbg": mint_r2s(tmp), "iterate": mint_iter(tmp)}
    with open(os.path.join(OUT, "widek.json"), "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if not os.path.exists(REF):
        raise SystemExit("build oracle/_ref first: make -C oracle ref")
    main()
