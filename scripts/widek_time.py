#!/usr/bin/env python
"""Times `read2sdbg` (m = 2, with mercy) at k = 239 and 255 and `iterate` at (k, step) = (239, 16) and (241, 14) - the k
where the stage-1 records / the flank index take the narrow layout (k = 255, 241) and just below it - on the device
(mhb_read2sdbg_host / mhb_iterate_host, after one warm-up call) and, when oracle/_ref/megahit_core_ref exists, the
reference binary on the same files with every host core.  Reads: the synthetic 300 bp generator (megahit_b200.synth) at
30x for read2sdbg; the seeded iterate cases of tests/iter_wide_cases.py for iterate.  Prints the card's name and power
limit, then one JSON line per configuration.

  widek_time.py [--r2s-reads N] [--iter-reads N] [--repeat R]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import iter_wide_cases as IW  # noqa: E402
from megahit_b200 import formats as F  # noqa: E402
from megahit_b200 import lib, synth  # noqa: E402
from test_oracle_iter import contig_seqs  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=60)
    return out.stdout.strip()


def timed(fn, repeat):
    fn()  # warm-up: module load, allocations
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        out = fn()  # the host calls end in a device synchronise
        ts.append(1000 * (time.perf_counter() - t0))
    return out, ts


def ref_time(cmd):
    if not os.path.exists(REF):
        return None
    t0 = time.perf_counter()
    subprocess.run([REF] + cmd, check=True, capture_output=True)
    return 1000 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--r2s-reads", type=int, default=1_000_000)
    ap.add_argument("--iter-reads", type=int, default=1_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    threads = str(os.cpu_count() or 8)
    with tempfile.TemporaryDirectory() as tmp:
        n, L = a.r2s_reads, 300
        b = synth.synth_reads(n, L, n * L // 30, 0.004, seed=255)
        libp = os.path.join(tmp, "r")
        F.write_lib(libp, b, n, n * L, L)
        for k in (239, 255):
            g, ts = timed(lambda: lib.read2sdbg_host(b.reshape(-1), n, k, 2, True), a.repeat)
            ref = ref_time(["read2sdbg", "-k", str(k), "-m", "2", "--need_mercy", "--host_mem", "6e10", "--mem_flag", "1",
                            "--num_cpu_threads", threads, "--output_prefix", os.path.join(tmp, "o"), "--read_lib_file", libp])
            print(json.dumps({"cmd": "read2sdbg", "k": k, "m": 2, "mercy": True, "n_reads": n, "read_len": L,
                              "device_ms": [round(t, 1) for t in ts], "phases_ms": {x: round(y, 1) for x, y in g["ms"].items()},
                              "n_items": g["n_items"], "n_rounds_s1": g["n_rounds_s1"],
                              "ref_ms": None if ref is None else round(ref, 1), "ref_threads": int(threads),
                              "sha256": F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"]))[:16]}), flush=True)
        del b
        for k, step in ((239, 16), (241, 14)):
            case = IW.make_case(k, step, 1, n_reads=a.iter_reads, read_len=(300, 301), G=1_000_000)
            paths = IW.write_case(case, os.path.join(tmp, f"i{k}"))
            cs = contig_seqs(paths[:2])
            g, ts = timed(lambda: lib.iterate_host(cs.words, cs.word_off, cs.len, case["bin"], case["n_reads"], k, step),
                          a.repeat)
            ref = ref_time(["iterate", "-c", paths[0], "-b", paths[1], "-r", paths[2], "-k", str(k), "-s", str(step), "-t",
                            threads, "-o", os.path.join(tmp, "io")])
            print(json.dumps({"cmd": "iterate", "k": k, "step": step, "n_reads": case["n_reads"],
                              "device_ms": [round(t, 1) for t in ts], "n_flanks": g["n_flanks"], "n_edges": g["n_edges"],
                              "ref_ms": None if ref is None else round(ref, 1), "ref_threads": int(threads),
                              "sha256": F.sha256(np.ascontiguousarray(g["edges"]).tobytes())[:16]}), flush=True)


if __name__ == "__main__":
    main()
