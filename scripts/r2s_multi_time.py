#!/usr/bin/env python
"""Times the file-level `read2sdbg` on 1 rank and on N ranks (`megahit_core read2sdbg --gpus N`,
mhb_read2sdbg_run_multi) on a seeded `synth.synth_reads` library of the size a user runs (default 5 M x 150 bp, 30x,
k = 27, m = 2, --need_mercy).  Every run is its own CLI process; the arms alternate within each repetition after one
warm-up call each.  Records: the card name and power limit of every device and their count, wall time per run, each
rank's log line, and whether both arms write the same canonical SdBG stream (sha256 read through P.sdbg_info) and the
same P.counting.

When the ranks outnumber the devices they share a device, and the N-rank times then say how much the shared-device
path costs, not how it scales: the speed-up is reported as "not measured" until the script runs on N devices.

--core-b PATH adds an N-rank arm run by another build's megahit_core (an A/B of two builds on the same library, the
arms alternating); --no-single drops the 1-rank arm and --no-warmup the warm-up calls (a library that takes minutes
per run).  Rank 0's round plan line is recorded with the rank lines.

  r2s_multi_time.py [--gpus 2] [--reads 5e6] [--k 27] [--m 2] [--no-mercy] [--repeat 3] [--core-b PATH] [--no-single]
                    [--no-warmup] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CORE = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
SEED = 2025


def devices():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [dict(zip(("name", "power_limit"), ln.split(", "))) for ln in r.stdout.strip().splitlines() if ln.strip()]


def make_lib(d, n_reads, read_len):
    from megahit_b200 import formats as F
    from megahit_b200 import synth
    b = synth.synth_reads(n_reads, read_len, genome_len=max(read_len + 1, 5 * n_reads), err=0.01, seed=SEED)
    p = os.path.join(d, "reads.lib")
    F.write_lib(p, b.reshape(-1), n_reads, n_reads * read_len, read_len)
    return p


def run_arm(libp, a, out, gpus, core=CORE):
    cmd = [core, "read2sdbg", "-k", str(a.k), "-m", str(a.m), "--host_mem", "6e10", "--mem_flag", "1",
           "--num_cpu_threads", "16", "--read_lib_file", libp, "--output_prefix", out]
    cmd += [] if a.no_mercy else ["--need_mercy"]
    cmd += ["--gpus", str(gpus)] if gpus > 1 else []
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    wall = time.time() - t0
    if r.returncode:
        sys.exit(r.stderr[-3000:])
    ranks = [ln.split(" - ", 1)[1] for ln in r.stderr.splitlines() if " - rank " in ln or "read2sdbg plan:" in ln]
    return wall, ranks


def digest(p, m):
    from megahit_b200 import formats as F
    d = {"sdbg_sha256": F.sha256(F.canonical_sdbg(p)[1])}
    if m > 1:
        d["counting_sha256"] = F.file_sha256(p + ".counting")
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--reads", type=float, default=5e6)
    ap.add_argument("--read-len", type=int, default=150)
    ap.add_argument("--k", type=int, default=27)
    ap.add_argument("--m", type=int, default=2)
    ap.add_argument("--no-mercy", action="store_true")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--core-b", default=None)
    ap.add_argument("--no-single", action="store_true")
    ap.add_argument("--no-warmup", action="store_true")
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
        libp = make_lib(d, int(a.reads), a.read_len)
        print(json.dumps({"case_s": round(time.time() - t0, 1), "reads": int(a.reads)}), flush=True)
        arms = {} if a.no_single else {"1_rank": (1, CORE)}
        arms[f"{a.gpus}_ranks"] = (a.gpus, CORE)
        if a.core_b:
            arms[f"b_{a.gpus}_ranks"] = (a.gpus, os.path.abspath(a.core_b))
        times, lines, digests = {arm: [] for arm in arms}, [], {}
        for arm, (g, core) in arms.items():
            if not a.no_warmup:
                run_arm(libp, a, os.path.join(d, "warm"), g, core)
        for rep in range(a.repeat):
            for arm, (g, core) in arms.items():
                p = os.path.join(d, arm)
                wall, ranks = run_arm(libp, a, p, g, core)
                digests[arm] = digest(p, a.m)
                line = {"arm": arm, "rep": rep, "wall_s": round(wall, 3), **digests[arm], "ranks": ranks}
                print(json.dumps(line), flush=True)
                lines.append(line)
                times[arm].append(wall)
        med = {arm: statistics.median(t) for arm, t in times.items()}
        summary = {"k": a.k, "m": a.m, "need_mercy": not a.no_mercy, "reads": int(a.reads), "read_len": a.read_len,
                   "median_s": med, "outputs_identical": len({json.dumps(x, sort_keys=True) for x in digests.values()}) == 1,
                   "speedup": ("not measured: the ranks share %d device(s)" % len(devs)) if shared
                   else round(med["1_rank"] / med[f"{a.gpus}_ranks"], 3) if "1_rank" in med else "not measured", **head}
        print(json.dumps(summary), flush=True)
        with open(os.path.join(a.out, "r2s_multi_time.json"), "w") as f:
            json.dump({"summary": summary, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
