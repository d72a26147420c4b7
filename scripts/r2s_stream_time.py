#!/usr/bin/env python
"""Times the 1-pass build (mhb_read2sdbg_host) with the read library resident and streamed from host memory in chunks
(lib.set_read_chunk_limit), each with and without forced rounds, on a synthetic library (150 bp reads at 30x, k = 27,
m = 2, need_mercy).  Every arm runs in a process of its own (a warm-up call, then one timed call), and the arms
alternate within each repetition, so that a drift of the machine hits all of them alike.  --parent-lib adds a resident
arm on another build of libmhb (MHB_LIB) to compare against.  Prints one JSON line per timed call: the library's total
time, the passes over the reads and the stream statistics, the round plan and a sha256 of the canonical SdBG stream;
then one summary line per arm with the median.

  r2s_stream_time.py [--n-reads N] [--chunk-mib 64] [--repeat 5] [--parent-lib PATH] [--out DIR]
  r2s_stream_time.py --big N_COPIES [--n-reads N]    # one streamed call on N_COPIES copies of the library, with the
                                                     # peak device memory nvidia-smi sees during the call
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
import numpy as np  # noqa: E402

K, M, L = 27, 2, 150


def worker(a):
    from megahit_b200 import formats as F
    from megahit_b200 import lib
    b = np.fromfile(a.lib, np.uint32)
    n_reads = a.n_reads * a.copies
    if a.copies > 1:
        b = np.tile(b, a.copies)
    lib.set_read_chunk_limit(a.chunk)
    lib.set_r2s_round_limit(a.s1, a.s2)
    smi = None
    try:
        if a.copies == 1:
            lib.read2sdbg_host(b, n_reads, K, M, True)  # warm-up: module load, allocations
        else:  # peak device memory of the call, sampled by nvidia-smi every 100 ms
            smi = subprocess.Popen(["nvidia-smi", "--query-gpu=memory.used", "--format=csv,noheader,nounits", "-i", "0",
                                    "-lms", "100"], stdout=subprocess.PIPE, text=True)
        t0 = time.time()
        g = lib.read2sdbg_host(b, n_reads, K, M, True)
        wall = time.time() - t0
        st = lib.read_stream_stats() if a.arm != "parent" else {}
    finally:
        lib.set_read_chunk_limit(0)
        lib.set_r2s_round_limit(0, 0)
        if smi:
            smi.terminate()
            out, _ = smi.communicate(timeout=30)
    line = {"arm": a.arm, "n_reads": n_reads, "k": K, "m": M, "mercy": True, "chunk_bytes": a.chunk, "caps": [a.s1, a.s2],
            "total_ms": round(g["ms"]["total"], 1), "wall_s": round(wall, 3), "n_rounds_s1": g["n_rounds_s1"],
            "n_rounds_s2": g["n_rounds_s2"], "sort_items": g["n_sort_items"], "n_mercy": g["n_mercy"],
            "sdbg_items": g["n_items"], "sdbg_sha256": F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"]))}
    line.update({k: (round(v, 1) if isinstance(v, float) else v) for k, v in st.items()})
    if smi:
        used = [int(x) for x in out.split() if x.strip().isdigit()]
        line["peak_device_mib"] = max(used) if used else None
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-reads", type=int, default=5_000_000)
    ap.add_argument("--chunk-mib", type=int, default=64)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--parent-lib", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    ap.add_argument("--big", type=int, default=0)
    # worker mode
    ap.add_argument("--arm", default="")
    ap.add_argument("--lib", default="")
    ap.add_argument("--chunk", type=int, default=0)
    ap.add_argument("--s1", type=int, default=0)
    ap.add_argument("--s2", type=int, default=0)
    ap.add_argument("--copies", type=int, default=1)
    a = ap.parse_args()
    if a.arm:
        return worker(a)
    from megahit_b200 import synth
    os.makedirs(a.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "reads.bin")
        synth.synth_reads(a.n_reads, L, 5 * a.n_reads, 0.01, seed=99).tofile(path)
        chunk = a.chunk_mib << 20

        def run(arm, chunk=0, s1=0, s2=0, copies=1):
            env = dict(os.environ)
            if arm == "parent":
                env["MHB_LIB"] = a.parent_lib
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--lib", path, "--n-reads", str(a.n_reads),
                   "--chunk", str(chunk), "--s1", str(s1), "--s2", str(s2), "--copies", str(copies)]
            out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
            line = json.loads(out.strip().splitlines()[-1])
            print(json.dumps(line), flush=True)
            with open(os.path.join(a.out, "r2s_stream_time.jsonl"), "a") as f:
                f.write(json.dumps(line) + "\n")
            return line

        if a.big:
            run("big", chunk=chunk, copies=a.big)
            return
        first = run("resident")
        n_s1 = a.n_reads * (L - K + 4)
        s1, s2 = n_s1 // 4 + 1, first["sort_items"] // 4 + 1  # about 4 rounds per stage
        arms = [("resident", {}), ("resident+rounds", {"s1": s1, "s2": s2}), ("streamed", {"chunk": chunk}),
                ("streamed+rounds", {"chunk": chunk, "s1": s1, "s2": s2})]
        if a.parent_lib:
            arms.insert(1, ("parent", {}))
        res = {name: [] for name, _ in arms}
        for _ in range(a.repeat):
            for name, kw in arms:
                res[name].append(run(name, **kw))
        shas = {line["sdbg_sha256"] for lines in res.values() for line in lines} | {first["sdbg_sha256"]}
        for name, lines in res.items():
            t = [x["total_ms"] for x in lines]
            summ = {"summary": name, "median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t),
                    "n_passes": lines[0].get("n_passes"), "n_chunks": lines[0].get("n_chunks"),
                    "n_rounds": [lines[0]["n_rounds_s1"], lines[0]["n_rounds_s2"]],
                    "median_pass_ms": statistics.median([x.get("pass_ms", 0) for x in lines]),
                    "median_h2d_ms": statistics.median([x.get("h2d_ms", 0) for x in lines]),
                    "median_fill_ms": statistics.median([x.get("fill_ms", 0) for x in lines]),
                    "median_kernel_ms": statistics.median([x.get("kernel_ms", 0) for x in lines]),
                    "sha_equal_in_all_arms": len(shas) == 1}
            print(json.dumps(summ), flush=True)
            with open(os.path.join(a.out, "r2s_stream_time.jsonl"), "a") as f:
                f.write(json.dumps(summ) + "\n")


if __name__ == "__main__":
    main()
