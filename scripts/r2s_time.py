#!/usr/bin/env python
"""Times the 1-pass build (mhb_read2sdbg_host) on a synthetic library (150 bp reads at 30x) and, optionally, the
reference binary's `read2sdbg` on the same library (host cores).  Prints one JSON line per configuration, with the
round plan each stage took, the free device memory before the call and a sha256 of the canonical SdBG stream, so that
two plans of one library can be compared.

  r2s_time.py N_READS [ref] [--s1 RECORDS] [--s2 ITEMS] [--m2-only] [--no-warmup] [--repeat R]

--s1 / --s2 cap the stage-1 records / stage-2 items of one round (lib.set_r2s_round_limit; 0 = derive from memory).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from megahit_b200 import formats as F  # noqa: E402
from megahit_b200 import lib, synth  # noqa: E402


def free_device_mib():
    """free memory of device 0 as nvidia-smi reports it (None when it cannot be asked)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=memory.free", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return int(out.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


ap = argparse.ArgumentParser()
ap.add_argument("n_reads", type=int, nargs="?", default=2_000_000)
ap.add_argument("ref", nargs="?", default="")
ap.add_argument("--s1", type=int, default=0)
ap.add_argument("--s2", type=int, default=0)
ap.add_argument("--m2-only", action="store_true")
ap.add_argument("--no-warmup", action="store_true")
ap.add_argument("--repeat", type=int, default=1)
args = ap.parse_args()
n_reads, with_ref = args.n_reads, args.ref == "ref"
L, k = 150, 27
t0 = time.time()
b = synth.synth_reads(n_reads, L, 5 * n_reads, 0.01, seed=99)
synth_s = time.time() - t0
runs = ((2, True),) if args.m2_only else ((2, True), (1, False))
for m, mercy in runs:
    if not args.no_warmup:
        lib.read2sdbg_host(b.reshape(-1), n_reads, k, m, mercy)  # warm-up (allocations, module load)
    for _ in range(args.repeat):
        free_mib = free_device_mib()
        capped = bool(args.s1 or args.s2)  # (MHB_LIB may select a build without the caps)
        if capped:
            lib.set_r2s_round_limit(args.s1, args.s2)
        os.environ["MHB_R2S_TRACE"] = "1"  # per-phase times on stderr
        t0 = time.time()
        try:
            g = lib.read2sdbg_host(b.reshape(-1), n_reads, k, m, mercy)
        finally:
            del os.environ["MHB_R2S_TRACE"]
            if capped:
                lib.set_r2s_round_limit(0, 0)
        wall = time.time() - t0
        n_s1 = n_reads * (L - k + 4) if m > 1 else 0
        rw = ((2 * (k - 1) + 6 + 31) // 32) + 2
        line = {"what": "read2sdbg", "n_reads": n_reads, "k": k, "m": m, "mercy": mercy, "edge_positions": g["n_edge_records"],
                "s1_records": n_s1, "s1_record_bytes_x2": 2 * n_s1 * rw * 4,
                "sort_items": g["n_sort_items"], "distinct_items": g["n_distinct_items"], "sdbg_items": g["n_items"],
                "n_mercy": g["n_mercy"], "caps": [args.s1, args.s2], "n_rounds_s1": g["n_rounds_s1"],
                "n_rounds_s2": g["n_rounds_s2"], "free_device_mib_before": free_mib,
                "sdbg_sha256": F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])),
                "ms": g["ms"], "wall_s": round(wall, 3), "synth_s": round(synth_s, 1),
                "edges_per_s": g["n_edge_records"] / (g["ms"]["total"] / 1e3)}
        del g
        if with_ref:
            ref = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
            with tempfile.TemporaryDirectory() as tmp:
                F.write_lib(f"{tmp}/r", b, n_reads, n_reads * L, L)
                t0 = time.time()
                subprocess.run([ref, "read2sdbg", "-k", str(k), "-m", str(m), "--host_mem", "6e10", "--mem_flag", "1",
                                "--output_prefix", f"{tmp}/o", "--num_cpu_threads", str(os.cpu_count()), "--read_lib_file",
                                f"{tmp}/r"] + (["--need_mercy"] if mercy else []), check=True, capture_output=True)
                line["reference_s"] = round(time.time() - t0, 3)
                line["reference_cores"] = os.cpu_count()
        print(json.dumps(line), flush=True)
