#!/usr/bin/env python
"""Times count_host and iterate_host with the read library resident against the same calls with the library streamed
from host memory in chunks (mhb_set_read_chunk_limit), on bench.py's synthetic library (10 M x 150 bp reads, 30x,
1 % substitutions, seed 1, k = 27, m = 2), at round caps giving about 1 / 4 / 16 rounds.

Per arm: wall time of the call (median of --reps), passes over the reads, chunks, bytes host to device, the achieved
H2D rate (bytes / copy-engine busy time), the wall time per pass, how much of the copy time the compute stream hides
(copy + kernel busy time - wall time of the passes, as a share of the copy time), whether the host fill or the PCIe
copy is the longer per pass, and whether the outputs equal the resident call's.  iterate runs once per chunk size
(one pass; contigs = the genome cut into 200 bp pieces).

  read_stream_time.py [--reads N] [--chunks 64,256,1024] [--rounds 1,4,16] [--reps R]

Prints one JSON document and writes it to scripts/out/read_stream_time.json.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from megahit_b200 import lib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reads", type=int, default=10_000_000)
ap.add_argument("--k", type=int, default=27)
ap.add_argument("--m", type=int, default=2)
ap.add_argument("--chunks", default="64,256,1024", help="chunk caps in MiB")
ap.add_argument("--rounds", default="1,4,16")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--iter-step", type=int, default=8)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("read_stream_time.py needs a CUDA device")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "nvidia-smi": f"unavailable ({type(e).__name__})"}


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


n_reads, RL, k, m = args.reads, 150, args.k, args.m
device = torch.device("cuda", 0)
G = 5 * n_reads
bin_np = synth.synth_reads_torch(n_reads, RL, G, 0.01, seed=1, device=device).cpu().numpy().view(np.uint32).reshape(-1)
torch.cuda.empty_cache()
bin_np = np.ascontiguousarray(bin_np)
image_bytes = 4 * len(bin_np)
n_edges = n_reads * (RL - k)
chunks = [int(c) << 20 for c in args.chunks.split(",")]
rounds = [int(r) for r in args.rounds.split(",")]
out = {"gpu": gpu_info(), "reads": n_reads, "read_len": RL, "k": k, "m": m, "image_bytes": image_bytes, "count": [],
       "iterate": []}


def timed(fn):
    ts, r = [], None
    for _ in range(args.reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), r


def arm_stats(st, wall_ms):
    d = dict(st)
    if st["n_chunks"]:
        d["ms_per_pass"] = st["pass_ms"] / max(1, st["n_passes"])
        d["h2d_gb_s"] = st["h2d_bytes"] / (st["h2d_ms"] * 1e6) if st["h2d_ms"] else None
        # copy time that ran under the kernels: copy + kernel busy time minus the passes' wall time
        d["copy_hidden_share"] = max(0.0, min(1.0, (st["h2d_ms"] + st["kernel_ms"] - st["pass_ms"]) / st["h2d_ms"])) if st["h2d_ms"] else None
        d["pass_bound_by"] = "host fill" if st["fill_ms"] > st["h2d_ms"] else "pcie"
    return d


for r in rounds:
    limit = 0 if r == 1 else n_edges // r + 1
    lib.set_round_limit(limit)
    try:
        lib.set_read_chunk_limit(0)
        lib.count_host(bin_np, n_reads, k, m)  # warm-up
        ms, g = timed(lambda: lib.count_host(bin_np, n_reads, k, m))
        ref = sha(g["edges"], g["cand_ids"], g["counting"])
        out["count"].append({"rounds_cap": r, "n_rounds": g["n_rounds"], "chunk_mib": 0, "ms": ms, "sha": ref,
                             **arm_stats(lib.read_stream_stats(), ms)})
        print(json.dumps(out["count"][-1]), flush=True)
        for c in chunks:
            lib.set_read_chunk_limit(c)
            ms, g = timed(lambda: lib.count_host(bin_np, n_reads, k, m))
            s = sha(g["edges"], g["cand_ids"], g["counting"])
            out["count"].append({"rounds_cap": r, "n_rounds": g["n_rounds"], "chunk_mib": c >> 20, "ms": ms, "sha": s,
                                 "equal": s == ref, **arm_stats(lib.read_stream_stats(), ms)})
            print(json.dumps(out["count"][-1]), flush=True)
    finally:
        lib.set_round_limit(0)
        lib.set_read_chunk_limit(0)

# iterate: the contigs are the first 500 k reads themselves (150 bp each, file orientation like the `.bin`), so that the
# reads drawn from the same regions of the genome align to them
contig_words = bin_np.reshape(n_reads, -1)[:, 1:]
n_ctg = min(n_reads, 500_000)
cw = np.ascontiguousarray(contig_words[:n_ctg]).reshape(-1)
W = contig_words.shape[1]
co = (np.arange(n_ctg + 1, dtype=np.uint64) * W)
cl = np.full(n_ctg, RL, np.uint32)
lib.set_read_chunk_limit(0)
lib.iterate_host(cw, co, cl, bin_np, n_reads, k, args.iter_step)  # warm-up
ms, g = timed(lambda: lib.iterate_host(cw, co, cl, bin_np, n_reads, k, args.iter_step))
ref = sha(g["edges"])
out["iterate"].append({"chunk_mib": 0, "ms": ms, "n_edges": g["n_edges"], "n_candidates": g["n_candidates"], "sha": ref,
                       **arm_stats(lib.read_stream_stats(), ms)})
print(json.dumps(out["iterate"][-1]), flush=True)
try:
    for c in chunks:
        lib.set_read_chunk_limit(c)
        ms, g = timed(lambda: lib.iterate_host(cw, co, cl, bin_np, n_reads, k, args.iter_step))
        s = sha(g["edges"])
        out["iterate"].append({"chunk_mib": c >> 20, "ms": ms, "n_edges": g["n_edges"], "sha": s, "equal": s == ref,
                               **arm_stats(lib.read_stream_stats(), ms)})
        print(json.dumps(out["iterate"][-1]), flush=True)
finally:
    lib.set_read_chunk_limit(0)
out["gpu_after"] = gpu_info()

os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
with open(os.path.join(ROOT, "scripts", "out", "read_stream_time.json"), "w") as f:
    json.dump(out, f, indent=1)
if os.environ.get("READ_STREAM_OUT"):
    with open(os.environ["READ_STREAM_OUT"], "w") as f:
        json.dump(out, f, indent=1)
print(json.dumps(out))
