#!/usr/bin/env python
"""Times the file-level `count` on 1 rank and on N ranks (`count --gpus N`, mhb_count_run_multi) on a seeded
variable-length library (synth.synth_reads_trimmed: 0 - 300 bp reads, tails cut as TrimN would, 1 % errors; default
10 M reads, k = 27, m = 2), with the owners' records resident and with a round cap (mhb_set_round_limit) that forces
several rounds (optionally with an SdBG cap, mhb_set_s2s_round_limit, that also runs the k_min SdBG stage in rounds).
Every run is its own process (lib.count_run after lib.set_round_limit, no CUDA in the parent); the arms
alternate within each repetition after one warm-up call each.  The N-rank count also builds the k_min SdBG, so the
1-rank arm is timed both alone and followed by `seq2sdbg --need_mercy`.  Records: the card name and power limit of
every device and their count, wall time per run, rounds, each rank's log line (peak device memory included), and
whether every arm writes the same canonical edges, P.cand, P.counting and SdBG stream.

When the ranks outnumber the devices they share a device, and the N-rank times then say how much the shared-device
path costs, not how it scales: the speed-up is reported as "not measured" until the script runs on N devices.

  count_multi_time.py [--gpus 2] [--reads 1e7] [--k 27] [--m 2] [--rounds 4] [--sdbg-cap N] [--repeat 2] [--out DIR]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CORE = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
SEED = 2026


def devices():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [dict(zip(("name", "power_limit"), ln.split(", "))) for ln in r.stdout.strip().splitlines() if ln.strip()]


def make_lib(d, n_reads, k):
    from megahit_b200 import formats as F
    from megahit_b200 import synth
    b, bases = synth.synth_reads_trimmed(n_reads, 300, err=0.01, seed=SEED)
    p = os.path.join(d, "reads.lib")
    F.write_lib(p, b, n_reads, bases, 300)
    # records = sum over the reads of max(0, L - k), from the length words
    w, n_rec = 0, 0
    while w < len(b):
        ln = int(b[w])
        n_rec += max(0, ln - k)
        w += 1 + (ln + 15) // 16
    return p, n_rec


def run_arm(libp, a, out, gpus, cap, sdbg_cap=0):
    code = (f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\nlib.set_round_limit({cap})\n"
            f"lib.set_s2s_round_limit({sdbg_cap})\n"
            f"lib.count_run({libp!r}, {out!r}, k={a.k}, m={a.m}, host_mem=6e10, num_cpu_threads=16, gpus={gpus})\n")
    t0 = time.time()
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    wall = time.time() - t0
    if r.returncode:
        sys.exit(r.stderr[-3000:])
    mercy = None
    if gpus == 1:
        t1 = time.time()
        r2 = subprocess.run([CORE, "seq2sdbg", "--host_mem", "6e10", "--mem_flag", "1", "--output_prefix", out,
                             "--num_cpu_threads", "16", "-k", str(a.k), "--kmer_from", "0", "--input_prefix", out,
                             "--need_mercy"], capture_output=True, text=True)
        if r2.returncode:
            sys.exit(r2.stderr[-3000:])
        mercy = time.time() - t1
    ranks = [ln.split(" - ", 1)[1] for ln in r.stderr.splitlines() if " - rank " in ln]
    m = re.search(r"count plan: (\d+) round", r.stderr)
    s = re.search(r"SdBG plan: (\d+) round", r.stderr)
    return wall, mercy, int(m.group(1)) if m else None, int(s.group(1)) if s else None, ranks


def digest(p):
    from oracle import gen_golden_cli as GC
    return GC.count_digest(p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--reads", type=float, default=1e7)
    ap.add_argument("--k", type=int, default=27)
    ap.add_argument("--m", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=4, help="round cap = records / (gpus * rounds)")
    ap.add_argument("--sdbg-cap", type=int, default=0, help="SdBG items per owner round of the rounds arm (0 = none)")
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    a = ap.parse_args()

    devs = devices()
    if not devs:
        sys.exit("no CUDA device: the timing needs the GPU")
    shared = a.gpus > len(devs)
    head = {"devices": devs, "device_count": len(devs), "ranks": a.gpus, "ranks_share_devices": shared}
    print(json.dumps(head), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.time()
        libp, n_rec = make_lib(d, int(a.reads), a.k)
        cap = max(1, n_rec // (a.gpus * a.rounds))
        print(json.dumps({"case_s": round(time.time() - t0, 1), "reads": int(a.reads), "records": n_rec,
                          "round_cap": cap}), flush=True)
        arms = {"1_rank": (1, 0, 0), f"{a.gpus}_ranks": (a.gpus, 0, 0), f"{a.gpus}_ranks_rounds": (a.gpus, cap, a.sdbg_cap)}
        times, lines, digests = {arm: [] for arm in arms}, [], {}
        for arm, (g, c, sc) in arms.items():
            run_arm(libp, a, os.path.join(d, "warm"), g, c, sc)
        for rep in range(a.repeat):
            for arm, (g, c, sc) in arms.items():
                p = os.path.join(d, arm)
                wall, mercy, rounds, sdbg_rounds, ranks = run_arm(libp, a, p, g, c, sc)
                digests[arm] = digest(p)
                line = {"arm": arm, "rep": rep, "count_wall_s": round(wall, 3), "rounds": rounds, "sdbg_rounds": sdbg_rounds,
                        "then_seq2sdbg_need_mercy_s": None if mercy is None else round(mercy, 3), **digests[arm],
                        "ranks": ranks}
                print(json.dumps(line), flush=True)
                lines.append(line)
                times[arm].append(wall + (mercy or 0.0))
        med = {arm: round(statistics.median(t), 3) for arm, t in times.items()}
        summary = {"k": a.k, "m": a.m, "reads": int(a.reads), "records": n_rec, "round_cap": cap, "sdbg_cap": a.sdbg_cap,
                   "median_s_count_to_kmin_sdbg": med,
                   "outputs_identical": len({json.dumps(x, sort_keys=True) for x in digests.values()}) == 1,
                   "speedup": ("not measured: the ranks share %d device(s)" % len(devs)) if shared
                   else round(med["1_rank"] / med[f"{a.gpus}_ranks"], 3), **head}
        print(json.dumps(summary), flush=True)
        with open(os.path.join(a.out, "count_multi_time.json"), "w") as f:
            json.dump({"summary": summary, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
