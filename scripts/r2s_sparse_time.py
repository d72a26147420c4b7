#!/usr/bin/env python
"""Times the 1-pass build (mhb_read2sdbg_host, need_mercy) on a streamed read library with the mercy candidates as
planes of the whole library against the list form (lib.set_r2s_sparse_mercy(1)), on synthetic libraries of 150 bp
reads at k = 27, m = 2, at two coverages (30x and 5x by default).  Every call runs in a process of its own (a warm-up
call, then one timed call) and the two forms alternate within each repetition.  Per timed call it prints one JSON line:
wall time, the library's total time, the peak device memory of the call (the device's used memory as nvidia-smi
reports it every 100 ms, less what was used before the call), the list entries (all rounds) per base and their host bytes, the device bytes of the candidates in either
form, and a sha256 of the canonical SdBG stream; then one summary line per coverage and form with the medians, the
GPU name, SM clock and power limit.

  r2s_sparse_time.py [--n-reads 5000000] [--cov 30 5] [--chunk-mib 64] [--repeat 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

K, M, L = 27, 2, 150


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def used_mib():
    out = subprocess.run(["nvidia-smi", "--query-gpu=memory.used", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return int(out) if out.isdigit() else 0


class PeakMemory:
    """the peak of the device's used memory (MiB, nvidia-smi) during the call, less what was used before it: the
    call's own peak when nothing else on the device allocates meanwhile"""

    def __init__(self):
        self.peak, self.stop_ = 0, threading.Event()
        self.t = threading.Thread(target=self.loop, daemon=True)

    def loop(self):
        while not self.stop_.is_set():
            self.peak = max(self.peak, used_mib() - self.before)
            time.sleep(0.1)

    def __enter__(self):
        self.before = used_mib()
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.stop_.set()
        self.t.join()


def worker(a):
    from megahit_b200 import formats as F
    from megahit_b200 import lib
    b = np.fromfile(a.lib, np.uint32)
    lib.set_read_chunk_limit(a.chunk)
    lib.set_r2s_sparse_mercy(1 if a.arm == "lists" else 0)
    try:
        lib.read2sdbg_host(b, a.n_reads, K, M, True)  # warm-up: module load, allocations
        with PeakMemory() as pm:
            t0 = time.time()
            g = lib.read2sdbg_host(b, a.n_reads, K, M, True)
            wall = time.time() - t0
        ms = lib.r2s_mercy_stats()
        st = lib.read_stream_stats()
    finally:
        lib.set_read_chunk_limit(0)
        lib.set_r2s_sparse_mercy(0)
    n_bases = a.n_reads * L
    plane_words = a.chunk // (4 + (L + 15) // 16 * 4) * L // 32 + 2  # the most reads of one chunk
    line = {"arm": a.arm, "cov": a.cov[0], "n_reads": a.n_reads, "k": K, "m": M, "chunk_bytes": a.chunk,
            "n_chunks": st["n_chunks"], "wall_s": round(wall, 3), "total_ms": round(g["ms"]["total"], 1),
            "peak_device_mib": pm.peak, "sparse": ms["sparse"], "list_entries": ms["n_entries"],
            "entries_per_base": round(ms["n_entries"] / n_bases, 5), "list_host_bytes": ms["host_bytes"],
            "list_bits_per_base": round(8 * ms["host_bytes"] / n_bases, 3),
            "device_candidate_bytes": (3 * 4 * (n_bases // 32 + 2) if not ms["sparse"]
                                       else 3 * 4 * plane_words + 8 * (1 << 20)),
            "n_rounds_s1": g["n_rounds_s1"], "n_mercy": g["n_mercy"], "sdbg_items": g["n_items"],
            "sdbg_sha256": F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"]))}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-reads", type=int, default=5_000_000)
    ap.add_argument("--cov", type=int, nargs="+", default=[30, 5])
    ap.add_argument("--chunk-mib", type=int, default=64)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    # worker mode
    ap.add_argument("--arm", default="")
    ap.add_argument("--lib", default="")
    ap.add_argument("--chunk", type=int, default=0)
    a = ap.parse_args()
    if a.arm:
        return worker(a)
    from megahit_b200 import synth
    os.makedirs(a.out, exist_ok=True)
    gpu = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        for cov in a.cov:
            path = os.path.join(tmp, f"reads_{cov}x.bin")
            synth.synth_reads(a.n_reads, L, a.n_reads * L // cov, 0.01, seed=7).tofile(path)
            res = {"planes": [], "lists": []}
            for _ in range(a.repeat):
                for arm in res:
                    cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--lib", path, "--n-reads",
                           str(a.n_reads), "--chunk", str(a.chunk_mib << 20), "--cov", str(cov)]
                    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
                    line = json.loads(out.strip().splitlines()[-1])
                    print(json.dumps(line), flush=True)
                    with open(os.path.join(a.out, "r2s_sparse_time.jsonl"), "a") as f:
                        f.write(json.dumps(line) + "\n")
                    res[arm].append(line)
            shas = {x["sdbg_sha256"] for v in res.values() for x in v}
            for arm, lines in res.items():
                s = {"summary": arm, "cov": cov, "n_reads": a.n_reads, "same_sdbg": len(shas) == 1,
                     "median_wall_s": statistics.median(x["wall_s"] for x in lines),
                     "median_total_ms": statistics.median(x["total_ms"] for x in lines),
                     "peak_device_mib": max(x["peak_device_mib"] for x in lines),
                     "entries_per_base": lines[-1]["entries_per_base"],
                     "list_bits_per_base": lines[-1]["list_bits_per_base"],
                     "list_host_bytes": lines[-1]["list_host_bytes"],
                     "device_candidate_bytes": lines[-1]["device_candidate_bytes"], "gpu": gpu}
                print(json.dumps(s), flush=True)
                with open(os.path.join(a.out, "r2s_sparse_time.jsonl"), "a") as f:
                    f.write(json.dumps(s) + "\n")


if __name__ == "__main__":
    main()
