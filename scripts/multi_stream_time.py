#!/usr/bin/env python
"""Times `count --gpus N` and `seq2sdbg --gpus N` (k > k_min) with every rank's share resident on its device against
streamed from host memory in chunks (lib.set_read_chunk_limit / lib.set_s2s_chunk_limit, set in a fresh process whose
forked workers inherit them), on the workloads of count_multi_time.py (seeded 0 - 300 bp library, default 10 M reads,
k = 27, m = 2) and s2s_multi_time.py (seeded contigs, default 300 M sort items at k = 79).  The cap is about a
--chunks'th of a share.  A process per run after a warm-up of every arm, arms alternated within each repetition.
Records: the card names, power limits and SM clocks and their count; wall time per run; each rank's log line, which
gives its chunks, its passes over the share and their wall time; the streamed cost per pass (the difference of the
median wall times over the passes of a rank); and whether both arms of a stage write byte-identical files.

When the ranks outnumber the devices they share a device, as the other *_multi_time.py scripts run them.

  multi_stream_time.py [--gpus 2] [--reads 1e7] [--items 300e6] [--chunks 4] [--repeat 2] [--out DIR]
"""
import argparse
import glob
import hashlib
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from count_multi_time import make_lib  # noqa: E402
from s2s_multi_time import write_contigs  # noqa: E402

RANK = re.compile(r"rank (\d+): .*; (?:reads|sequences) (?:resident|in (\d+) chunks, (\d+) passes in ([\d.]+) ms)")


def devices():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    keys = ("name", "power_limit", "sm_clock", "max_sm_clock")
    return [dict(zip(keys, ln.split(", "))) for ln in r.stdout.strip().splitlines() if ln.strip()]


def run(call, cap_fn, cap):
    code = (f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\nlib.{cap_fn}({cap})\n{call}\n")
    t0 = time.time()
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    wall = time.time() - t0
    if r.returncode:
        sys.exit(r.stderr[-3000:])
    ranks = [ln.split(" - ", 1)[1] for ln in r.stderr.splitlines() if RANK.search(ln)]
    passes = [(int(m.group(3)), float(m.group(4))) for m in map(RANK.search, ranks) if m.group(2)]
    return wall, ranks, passes


def files_sha(p):
    return {f[len(p):]: hashlib.sha256(open(f, "rb").read()).hexdigest() for f in sorted(glob.glob(p + ".*"))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--reads", type=float, default=1e7)
    ap.add_argument("--items", type=float, default=300e6)
    ap.add_argument("--chunks", type=int, default=4, help="the chunk cap is about a share / chunks")
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(HERE, "out"))
    a = ap.parse_args()

    devs = devices()
    if not devs:
        sys.exit("no CUDA device: the timing needs the GPU")
    head = {"devices": devs, "device_count": len(devs), "ranks": a.gpus, "ranks_share_devices": a.gpus > len(devs)}
    print(json.dumps(head), flush=True)
    os.makedirs(a.out, exist_ok=True)
    g = a.gpus
    with tempfile.TemporaryDirectory() as d:
        libp, n_rec = make_lib(d, int(a.reads), 27)
        contigs = os.path.join(d, "contigs.fa")
        n_items, _ = write_contigs(contigs, 79, int(a.items), seed=4321)
        read_cap = max(1, os.path.getsize(libp + ".bin") // (g * a.chunks))
        seq_cap = max(1, os.path.getsize(contigs) // 4 // (g * a.chunks))  # about the packed bases of a share
        stages = {
            "count": (f"lib.count_run({libp!r}, OUT, k=27, m=2, host_mem=6e10, num_cpu_threads=16, gpus={g})",
                      "set_read_chunk_limit", read_cap),
            "seq2sdbg": (f"lib.seq2sdbg_run(OUT, 79, contig={contigs!r}, host_mem=3e10, num_cpu_threads=16, gpus={g})",
                         "set_s2s_chunk_limit", seq_cap)}
        print(json.dumps({"reads": int(a.reads), "records": n_rec, "sort_items": n_items, "read_cap": read_cap,
                          "seq_cap": seq_cap}), flush=True)
        arms = [(st, form) for st in stages for form in ("resident", "streamed")]
        times = {arm: [] for arm in arms}
        passes, shas, lines = {}, {}, []

        def one(arm, out):
            st, form = arm
            call, fn, cap = stages[st]
            return run(call.replace("OUT", repr(out)), fn, cap if form == "streamed" else 0)

        for arm in arms:
            one(arm, os.path.join(d, "warm"))
        for rep in range(a.repeat):
            for arm in arms:
                out = os.path.join(d, "_".join(arm))
                wall, ranks, ps = one(arm, out)
                times[arm].append(wall)
                shas[arm] = files_sha(out)
                if ps:
                    passes[arm] = ps
                line = {"stage": arm[0], "form": arm[1], "rep": rep, "wall_s": round(wall, 3), "ranks": ranks}
                print(json.dumps(line), flush=True)
                lines.append(line)
        summary = {"median_s": {"_".join(arm): round(statistics.median(t), 3) for arm, t in times.items()}}
        for st in stages:
            ps = passes.get((st, "streamed"), [])
            n_pass = max((p for p, _ in ps), default=0)
            extra = statistics.median(times[(st, "streamed")]) - statistics.median(times[(st, "resident")])
            summary[st] = {"identical_files": shas[(st, "streamed")] == shas[(st, "resident")],
                           "passes_per_rank": n_pass,
                           "streamed_minus_resident_ms_per_pass": round(1e3 * extra / n_pass, 1) if n_pass else None,
                           "logged_pass_ms_per_rank": [round(ms / p, 1) for p, ms in ps]}
        summary.update(head)
        print(json.dumps(summary), flush=True)
        with open(os.path.join(a.out, "multi_stream_time.json"), "w") as f:
            json.dump({"summary": summary, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
