"""Times `megahit_core buildlib` on the GPU against the reference binary (oracle/_ref/megahit_core_ref) on a seeded
FASTQ of N x L bp reads (4-line records, ~1 % N), read from the page cache and, for ours, also through a FIFO fed by
`cat`, as the driver feeds `gzip -cd` output.  Prints one JSON line: seconds, GB/s of text, reads/s and the sha256 of
P.bin and the peak RSS per run, with the GPU's name, power limit and SM clock.

    python scripts/buildlib_time.py [--reads 10000000] [--len 150] [--out DIR]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def write_fastq(path, n, length, seed, block=1 << 20):
    rng = np.random.default_rng(seed)
    hdr_w = 12  # "@r%09d\n"
    rec = hdr_w + (length + 1) + 2 + (length + 1)
    with open(path, "wb") as f:
        for b0 in range(0, n, block):
            m = min(block, n - b0)
            a = np.empty((m, rec), np.uint8)
            ids = np.char.encode(np.char.mod("@r%09d\n", np.arange(b0, b0 + m)), "ascii")
            a[:, :hdr_w] = np.frombuffer(b"".join(ids), np.uint8).reshape(m, hdr_w)
            s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=(m, length))]
            s[rng.random((m, length)) < 0.01] = ord("N")
            o = hdr_w
            a[:, o:o + length] = s
            a[:, o + length] = ord("\n")
            o += length + 1
            a[:, o:o + 2] = np.frombuffer(b"+\n", np.uint8)
            o += 2
            a[:, o:o + length] = ord("I")
            a[:, o + length] = ord("\n")
            f.write(a.tobytes())


def sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def timed(cmd):
    """wall seconds and peak RSS (MB) of one run of cmd"""
    log("running " + " ".join(os.path.basename(c) for c in cmd[:2]))
    with tempfile.TemporaryFile() as err:
        t0 = time.perf_counter()
        p = subprocess.Popen(cmd, stdout=subprocess.DEVNULL, stderr=err)
        _, status, ru = os.wait4(p.pid, 0)
        dt = time.perf_counter() - t0
        p.returncode = os.waitstatus_to_exitcode(status)
        if p.returncode != 0:
            err.seek(0)
            sys.exit(f"{cmd} failed: {err.read().decode()[-2000:]}")
    return dt, ru.ru_maxrss / 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--len", type=int, default=150)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: print only)")
    ap.add_argument("--write-fastq", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.write_fastq:
        write_fastq(a.write_fastq, a.reads, a.len, seed=1)
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as d:
        fq = os.path.join(d, "reads.fq")
        log(f"writing {a.reads} reads")
        # in a process of its own: a child's peak RSS (ru_maxrss) starts from what its parent held when it forked
        subprocess.run([sys.executable, os.path.abspath(__file__), "--reads", str(a.reads), "--len", str(a.len),
                        "--write-fastq", fq], check=True)
        size = os.path.getsize(fq)
        subprocess.run(["cat", fq], stdout=subprocess.DEVNULL, check=True)  # into the page cache
        lib = os.path.join(d, "reads.lib")
        with open(lib, "w") as f:
            f.write(f"{fq}\nse {fq}\n")
        res = {"reads": a.reads, "len": a.len, "text_bytes": size, "gpu": gpu, "runs": {}}

        def record(name, t, prefix):
            dt, rss = t
            res["runs"][name] = {"s": round(dt, 3), "max_rss_MB": round(rss), "GB_per_s": round(size / dt / 1e9, 3),
                                 "reads_per_s": round(a.reads / dt), "bin_sha256": sha(prefix + ".bin")}
            log(f"{name}: {res['runs'][name]}")

        timed([CLI, "buildlib", lib, os.path.join(d, "warm")])  # CUDA context, module load
        for rep in range(2):
            p = os.path.join(d, f"ours{rep}")
            record(f"ours_page_cache_{rep}", timed([CLI, "buildlib", lib, p]), p)
        fifo = os.path.join(d, "reads.fifo")
        os.mkfifo(fifo)
        libf = os.path.join(d, "fifo.lib")
        with open(libf, "w") as f:
            f.write(f"{fq}\nse {fifo}\n")
        feeder = threading.Thread(target=lambda: subprocess.run(f"cat {fq} > {fifo}", shell=True))
        feeder.start()
        p = os.path.join(d, "ours_fifo")
        record("ours_fifo", timed([CLI, "buildlib", libf, p]), p)
        feeder.join()
        if os.access(REF, os.X_OK):
            p = os.path.join(d, "ref")
            record("reference_page_cache", timed([REF, "buildlib", lib, p]), p)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "buildlib_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
