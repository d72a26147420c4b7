#!/usr/bin/env python
"""Times the file-level `iterate` on 1 rank and on N ranks (`megahit_core iterate --gpus N`, mhb_iterate_run_multi) on
a seeded case of the size a user runs: `synth.synth_reads` reads (default 20 M x 150 bp) and contigs of 60 - 300 bp
cut from the same genome, at a mid-chain step (default 59 -> 79).  Every run is its own CLI process; the arms alternate
within each repetition after one warm-up call each.  Records: the card name and power limit of every device and their
count, wall time per run, each rank's share as it logs it, and whether both arms write byte-identical P.edges.0 and
P.edges.info.

When the ranks outnumber the devices they share a device, and the N-rank times then say how much the shared-device
path costs, not how it scales: the speed-up is reported as "not measured" until the script runs on N devices.

  iter_multi_time.py [--gpus 2] [--reads 20e6] [--k 59] [--step 20] [--repeat 3] [--out DIR]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CORE = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
SEED = 2024


def devices():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [dict(zip(("name", "power_limit"), ln.split(", "))) for ln in r.stdout.strip().splitlines() if ln.strip()]


def make_case(d, n_reads, read_len):
    """the read library and the contigs of its genome (cut into 60 - 300 bp pieces, flag 0: at k = 59
    the iterative edges come from reads across the ends of contigs this short); empty bubble file"""
    from megahit_b200 import synth
    genome_len = max(read_len + 1, 5 * n_reads)
    b = synth.synth_reads(n_reads, read_len, genome_len=genome_len, seed=SEED)
    reads = os.path.join(d, "reads.bin")
    b.tofile(reads)
    del b
    genome = np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(SEED).integers(0, 4, size=genome_len, dtype=np.uint8)]
    rng = np.random.default_rng(SEED + 1)
    cuts = np.cumsum(rng.integers(60, 301, size=genome_len // 60))
    cuts = [0] + [int(c) for c in cuts if c < genome_len] + [genome_len]
    contigs, bubbles = os.path.join(d, "contigs.fa"), os.path.join(d, "bubbles.fa")
    with open(contigs, "wb") as f:
        for i, (a, z) in enumerate(zip(cuts[:-1], cuts[1:])):
            f.write(b">c%d flag=0 multi=30.0000 len=%d\n" % (i, z - a) + genome[a:z].tobytes() + b"\n")
    open(bubbles, "w").close()
    return contigs, bubbles, reads, len(cuts) - 1


def run_arm(case, k, step, out, gpus):
    contigs, bubbles, reads = case
    cmd = [CORE, "iterate", "-c", contigs, "-b", bubbles, "-r", reads, "-t", "16", "-k", str(k), "-s", str(step), "-o", out]
    if gpus > 1:
        cmd += ["--gpus", str(gpus)]
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    wall = time.time() - t0
    if r.returncode:
        sys.exit(r.stderr[-3000:])
    ranks = [ln.split(" - ", 1)[1] for ln in r.stderr.splitlines() if " - rank " in ln]
    edges = [ln.split(" - ", 1)[1] for ln in r.stderr.splitlines() if "Iterative edges" in ln]
    return wall, ranks, edges[-1] if edges else ""


def digest(p):
    h = hashlib.sha256()
    for suffix in (".edges.0", ".edges.info"):
        with open(p + suffix, "rb") as f:
            for block in iter(lambda: f.read(1 << 24), b""):
                h.update(block)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--reads", type=float, default=20e6)
    ap.add_argument("--read-len", type=int, default=150)
    ap.add_argument("--k", type=int, default=59)
    ap.add_argument("--step", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    a = ap.parse_args()

    devs = devices()
    shared = a.gpus > len(devs)
    head = {"devices": devs, "device_count": len(devs), "ranks": a.gpus, "ranks_share_devices": shared}
    print(json.dumps(head), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.time()
        contigs, bubbles, reads, n_contigs = make_case(d, int(a.reads), a.read_len)
        case = (contigs, bubbles, reads)
        print(json.dumps({"case_s": round(time.time() - t0, 1), "reads": int(a.reads), "contigs": n_contigs}), flush=True)
        arms = {"1_rank": 1, f"{a.gpus}_ranks": a.gpus}
        times, lines, shas = {arm: [] for arm in arms}, [], {}
        for arm, g in arms.items():
            run_arm(case, a.k, a.step, os.path.join(d, "warm"), g)
        for rep in range(a.repeat):
            for arm, g in arms.items():
                p = os.path.join(d, arm)
                wall, ranks, edges = run_arm(case, a.k, a.step, p, g)
                shas[arm] = digest(p)
                line = {"arm": arm, "rep": rep, "wall_s": round(wall, 3), "result": edges, "ranks": ranks}
                print(json.dumps(line), flush=True)
                lines.append(line)
                times[arm].append(wall)
        med = {arm: statistics.median(t) for arm, t in times.items()}
        summary = {"k": a.k, "step": a.step, "reads": int(a.reads), "read_len": a.read_len, "median_s": med,
                   "outputs_identical": len(set(shas.values())) == 1,
                   "speedup": ("not measured: the ranks share %d device(s)" % len(devs)) if shared
                   else round(med["1_rank"] / med[f"{a.gpus}_ranks"], 3), **head}
        print(json.dumps(summary), flush=True)
        with open(os.path.join(a.out, "iter_multi_time.json"), "w") as f:
            json.dump({"summary": summary, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
