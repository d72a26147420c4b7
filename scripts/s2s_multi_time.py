#!/usr/bin/env python
"""Times the file-level `seq2sdbg` for k > k_min on 1 rank and on N ranks (`megahit_core seq2sdbg --gpus N`,
mhb_seq2sdbg_run_multi) on a seeded synthetic contig set of realistic size (default about 300 M sort items at k = 79).
Every run is its own CLI process; the arms alternate within each repetition after one warm-up call each.  Records in
the same call: the devices (index, name, power limit) and their count; wall time per run; the peak device memory of
every process nvidia-smi lists during the run (polled; inside a container it may list only some of them) and, for the
N-rank runs, the peak each rank allocated as the rank itself logs it; and whether every arm gives the same canonical
SdBG.  --cap N adds an N-rank arm whose owners take at most N items per round (mhb_set_s2s_round_limit, set in a fresh
process that then runs lib.seq2sdbg_run), so that the SdBG stage runs in rounds over bucket ranges.

When the ranks outnumber the devices they share a device, and the N-rank times then say how much the shared-device
path costs, not how it scales: the speed-up is reported as "not measured" until the script runs on N devices.

  s2s_multi_time.py [--gpus 2] [--k 79] [--items 300e6] [--cap N] [--repeat 2] [--out DIR]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CORE = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def smi(query, *extra):
    r = subprocess.run(["nvidia-smi", f"--query-{query}", "--format=csv,noheader,nounits", *extra], capture_output=True,
                       text=True)
    return [ln.split(", ") for ln in r.stdout.strip().splitlines() if ln.strip()]


def write_contigs(path, k, n_items, seed):
    """contigs of 1000 - 3000 bp cut from a random genome, multiplicities 1 - 400, until n_items sort items"""
    rng = np.random.default_rng(seed)
    genome = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=50_000_000)]
    got, i = 0, 0
    with open(path, "wb") as f:
        while got < n_items:
            L = int(rng.integers(1000, 3000))
            s = int(rng.integers(0, len(genome) - L))
            f.write(b">k%d_%d flag=0 multi=%.4f len=%d\n" % (k, i, rng.uniform(1, 400), L))
            f.write(genome[s:s + L].tobytes() + b"\n")
            got += 2 * (L - k + 2)
            i += 1
    return got, i


def run_arm(contigs, k, out, gpus, cap=0):
    cmd = [CORE, "seq2sdbg", "--host_mem", "3e10", "--mem_flag", "1", "--output_prefix", out, "--num_cpu_threads", "16",
           "-k", str(k), "--contig", contigs]
    if gpus > 1:
        cmd += ["--gpus", str(gpus)]
    if cap:  # no CUDA in the process that sets the cap: its workers are forked
        cmd = [sys.executable, "-c", f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\n"
               f"lib.set_s2s_round_limit({cap})\nlib.seq2sdbg_run({out!r}, {k}, contig={contigs!r}, host_mem=3e10, "
               f"num_cpu_threads=16, gpus={gpus})\n"]
    peak, stop = {}, threading.Event()

    def poll():
        while not stop.is_set():
            for row in smi("compute-apps=pid,used_memory"):
                if len(row) == 2 and row[1].strip().isdigit():
                    peak[row[0]] = max(peak.get(row[0], 0), int(row[1]))
            time.sleep(0.1)

    th = threading.Thread(target=poll)
    th.start()
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    wall = time.time() - t0
    stop.set()
    th.join()
    if r.returncode:
        sys.exit(r.stderr[-3000:])
    # each rank of a multi-GPU run logs the most device memory it allocated (its CUDA context not included)
    ranks = {int(m.group(1)): float(m.group(2)) for m in re.finditer(r"rank (\d+): .*peak device memory ([\d.]+) MiB", r.stderr)}
    rounds = re.search(r"SdBG plan: (\d+) round", r.stderr)
    return wall, sorted(peak.values(), reverse=True), [ranks[i] for i in sorted(ranks)], int(rounds.group(1)) if rounds else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--k", type=int, default=79)
    ap.add_argument("--items", type=float, default=300e6)
    ap.add_argument("--cap", type=int, default=0, help="items per owner round of an extra N-rank arm (0 = no such arm)")
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    a = ap.parse_args()
    from megahit_b200 import formats as F

    devices = [{"index": int(d[0]), "name": d[1], "power_limit_w": d[2]} for d in smi("gpu=index,name,power.limit")]
    shared = a.gpus > len(devices)
    head = {"devices": devices, "device_count": len(devices), "ranks": a.gpus, "ranks_share_devices": shared}
    print(json.dumps(head), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        contigs = os.path.join(d, "contigs.fa")
        n_items, n_contigs = write_contigs(contigs, a.k, int(a.items), seed=4321)
        arms = {"1_rank": (1, 0), f"{a.gpus}_ranks": (a.gpus, 0)}
        if a.cap:
            arms[f"{a.gpus}_ranks_cap"] = (a.gpus, a.cap)
        times, lines, shas = {arm: [] for arm in arms}, [], {}
        for arm, (g, c) in arms.items():
            run_arm(contigs, a.k, os.path.join(d, "warm"), g, c)
        for rep in range(a.repeat):
            for arm, (g, c) in arms.items():
                p = os.path.join(d, arm)
                wall, peak, rank_peak, rounds = run_arm(contigs, a.k, p, g, c)
                shas[arm] = F.sha256(F.canonical_sdbg(p)[1])
                line = {"arm": arm, "rep": rep, "wall_s": round(wall, 3), "sdbg_rounds": rounds, "peak_device_mib_per_process": peak,
                        "peak_allocated_mib_per_rank": rank_peak}
                print(json.dumps(line), flush=True)
                lines.append(line)
                times[arm].append(wall)
        med = {arm: statistics.median(t) for arm, t in times.items()}
        summary = {"k": a.k, "sort_items": n_items, "contigs": n_contigs, "median_s": med,
                   "same_sdbg_in_every_arm": len(set(shas.values())) == 1,
                   "speedup": ("not measured: the ranks share %d device(s)" % len(devices)) if shared
                   else round(med["1_rank"] / med[f"{a.gpus}_ranks"], 3), **head}
        print(json.dumps(summary), flush=True)
        with open(os.path.join(a.out, "s2s_multi_time.json"), "w") as f:
            json.dump({"summary": summary, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
