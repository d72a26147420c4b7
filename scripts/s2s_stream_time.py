#!/usr/bin/env python
"""Times the file-level `seq2sdbg --need_mercy` (mhb_seq2sdbg_run: mercy search + seq2sdbg) with its input resident and
streamed from host memory (lib.set_s2s_chunk_limit), on the edges `count` writes for a synthetic library (150 bp reads at
30x, k = 27, m = 2).  Arms: resident; 64 MiB chunks / segments; 64 MiB chunks plus forced rounds (about 6).  Every arm
runs in a process of its own (a warm-up call, then one timed call), and the arms alternate within each repetition, so
that a drift of the machine hits all of them alike.  Prints the card's name and power limit, one JSON line per timed
call (wall time, passes, rounds, bytes host to device, copy / kernel / fill times of seq2sdbg and of the mercy search, and
a sha256 of the canonical SdBG stream), then one summary line per arm with the median.

  s2s_stream_time.py [--n-reads N] [--chunk-mib 64] [--repeat 3] [--out DIR]
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

K, M, L = 27, 2, 150


def worker(a):
    from megahit_b200 import formats as F
    from megahit_b200 import lib

    def run(out):
        lib.seq2sdbg_run(out, k=K, input_prefix=a.prefix, need_mercy=True, host_mem=3e10, num_cpu_threads=16)

    lib.set_s2s_chunk_limit(a.chunk)
    lib.set_s2s_round_limit(a.rounds)
    try:
        run(a.prefix + f".warm_{a.arm}")  # warm-up: module load, allocations
        t0 = time.time()
        run(a.prefix + f".{a.arm}")
        wall = time.time() - t0
        st, ms = lib.s2s_stream_stats(), lib.s2s_stream_stats(mercy=True)
    finally:
        lib.set_s2s_chunk_limit(0)
        lib.set_s2s_round_limit(0)
    line = {"arm": a.arm, "chunk_bytes": a.chunk, "round_cap": a.rounds, "wall_s": round(wall, 3),
            "sdbg_sha256": F.sha256(F.canonical_sdbg(a.prefix + f".{a.arm}")[1])}
    line.update({f"s2s_{k}": (round(v, 1) if isinstance(v, float) else v) for k, v in st.items()})
    line.update({f"mercy_{k}": (round(v, 1) if isinstance(v, float) else v) for k, v in ms.items() if k != "n_rounds"})
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-reads", type=int, default=10_000_000)
    ap.add_argument("--chunk-mib", type=int, default=64)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "scripts", "out"))
    # worker mode
    ap.add_argument("--arm", default="")
    ap.add_argument("--prefix", default="")
    ap.add_argument("--chunk", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=0)
    a = ap.parse_args()
    if a.arm:
        return worker(a)

    from megahit_b200 import formats as F
    from megahit_b200 import lib, synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        b = synth.synth_reads(a.n_reads, L, 5 * a.n_reads, 0.01, seed=1234)
        libp = os.path.join(d, "reads.lib")
        F.write_lib(libp, b, a.n_reads, a.n_reads * L, L)
        del b
        p = os.path.join(d, "k27")
        lib.count_run(libp, p, k=K, m=M, host_mem=3e10, num_cpu_threads=16)
        n_edges = len(F.canonical_edges(p))
        chunk = a.chunk_mib << 20
        # ~6 rounds: 6 sort items per solid edge, the mercy edges on top
        arms = {"resident": (0, 0), f"chunks_{a.chunk_mib}mib": (chunk, 0),
                f"chunks_{a.chunk_mib}mib_rounds": (chunk, 6 * n_edges // 5 + 1)}
        times = {arm: [] for arm in arms}
        lines = []
        for _ in range(a.repeat):
            for arm, (c, r) in arms.items():
                out = subprocess.run([sys.executable, __file__, "--arm", arm, "--prefix", p, "--chunk", str(c), "--rounds", str(r)],
                                     capture_output=True, text=True)
                if out.returncode:
                    sys.exit(out.stderr[-3000:])
                line = json.loads(out.stdout.strip().splitlines()[-1])
                print(json.dumps(line), flush=True)
                lines.append(line)
                times[arm].append(line["wall_s"])
        shas = {ln["sdbg_sha256"] for ln in lines}
        for arm in arms:
            last = [ln for ln in lines if ln["arm"] == arm][-1]
            print(json.dumps({"arm": arm, "median_s": statistics.median(times[arm]), "runs": times[arm], "n_solid": n_edges,
                              "s2s_passes": last["s2s_n_passes"], "s2s_rounds": last["s2s_n_rounds"],
                              "s2s_h2d_bytes": last["s2s_h2d_bytes"], "mercy_segments": last["mercy_n_chunks"],
                              "same_sdbg_in_every_arm": len(shas) == 1, "gpu": gpu}), flush=True)
        with open(os.path.join(a.out, "s2s_stream_time.json"), "w") as f:
            json.dump({"gpu": gpu, "lines": lines}, f, indent=1)


if __name__ == "__main__":
    main()
