#!/usr/bin/env python
"""bench.py -- SdBG-construction hot path (count -> seq2sdbg) on synthetic 150 bp reads, k=27.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

One "step" = one pass of the hot path over one batch of reads: canonical (k+1)-mer edge extraction, LSD
radix sort, solid-edge counting + mercy bookkeeping, then seq2sdbg item extraction, radix sort and SdBG
emission from the device-resident solid edges.  `value` is whole-job edges/s with the read library already
in HBM; `e2e` is the same metric through the host-buffer C ABI (mhb_build_host: count -> device mercy edges -> seq2sdbg), H2D/D2H
inside the timed region.  `--impl reference` times the unmodified reference's OpenMP path
(oracle/_ref/megahit_core_ref count + seq2sdbg) on the host cores on a bounded sample.  `--dump-outputs DIR` writes what
the last timed step computed as DIR/<name>.npy (see dump_outputs), so that two builds can be compared on the same inputs.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "sorted (k+1)-mer edges/sec at k=27 on 150bp reads"
READ_LEN = 150
GENOME_PER_READ = 5  # 5 Mb of genome per 1 M reads ~ 30x coverage (SURVEY.md 8d)
ERR = 0.01


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        j = json.load(open(p))
        return float(j["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx, self.proc, self.lines = gpu_index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.idx)], stdout=subprocess.PIPE, text=True)
            self.th = threading.Thread(target=lambda: [self.lines.append(l) for l in self.proc.stdout], daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        self.th.join(timeout=2)
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for l in self.lines:
            f = [x.strip() for x in l.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
            except ValueError:
                continue
            for nm, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ------------------------------------------------------------------------------------------------
# reference arm / cpu baseline: the unmodified reference binary on the host cores, bounded sample
# ------------------------------------------------------------------------------------------------
def reference_run(n_reads: int, k: int, m: int, threads: int, seed: int = 1234):
    from megahit_b200 import formats as F
    from megahit_b200 import synth
    ref = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
    if not os.path.exists(ref):
        return None
    tmp = tempfile.mkdtemp(prefix="mhb_ref_")
    try:
        b = synth.synth_reads(n_reads, READ_LEN, GENOME_PER_READ * n_reads, ERR, seed=seed)
        F.write_lib(os.path.join(tmp, "r"), b, n_reads, n_reads * READ_LEN, READ_LEN)
        p = os.path.join(tmp, "k")
        t0 = time.perf_counter()
        subprocess.run([ref, "count", "-k", str(k), "-m", str(m), "--host_mem", "6e10", "--mem_flag", "1",
                        "--output_prefix", p, "--num_cpu_threads", str(threads), "--read_lib_file",
                        os.path.join(tmp, "r")], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        t1 = time.perf_counter()
        subprocess.run([ref, "seq2sdbg", "--host_mem", "6e10", "--mem_flag", "1", "--output_prefix", p,
                        "--num_cpu_threads", str(threads), "-k", str(k), "--kmer_from", "0", "--input_prefix", p,
                        "--need_mercy"], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        t2 = time.perf_counter()
        return {"n_edges": n_reads * (READ_LEN - k), "t_count": t1 - t0, "t_s2s": t2 - t1}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def cpu_info():
    """CPU model / sockets / NUMA nodes of the box the CPU arm runs on (the arm varied 3x between boxes in round 1)"""
    info = {"logical_cpus": os.cpu_count()}
    try:
        txt = open("/proc/cpuinfo").read()
        models = [l.split(":", 1)[1].strip() for l in txt.splitlines() if l.startswith("model name")]
        info["model"] = models[0] if models else None
        info["sockets"] = len({l.split(":", 1)[1].strip() for l in txt.splitlines() if l.startswith("physical id")}) or None
        info["numa_nodes"] = len([d for d in os.listdir("/sys/devices/system/node") if d.startswith("node")])
        info["loadavg_1m"] = float(open("/proc/loadavg").read().split()[0])
    except Exception:
        pass
    return info


def reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = os.cpu_count() or 1
    sample = args.sample_reads
    times = []
    for i in range(args.warmup + args.steps):
        r = reference_run(sample, args.k, args.m, threads, seed=1234)  # the same library every step
        if r is None:
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/megahit_core_ref was not built"}))
            return
        if i >= args.warmup:
            times.append(r["t_count"] + r["t_s2s"])
    n_edges = sample * (READ_LEN - args.k)
    t = float(np.mean(times))
    v = n_edges / t
    desc = f"{sample} synthetic 150 bp reads/step (seed 1234), count+seq2sdbg --need_mercy, mem_flag 1"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "edges/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": t * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u32", "data": "synthetic",
        "config": {"workload": f"reference megahit_core count+seq2sdbg k={args.k} m={args.m} on host cores", "sample": desc},
        "cpu_baseline": {"value": v, "unit": "edges/s", "cores": threads, "kind": "reference", "sample": desc,
                         "step_times_s": [round(x, 3) for x in times], "cpu": cpu_info()},
        "e2e": {"value": v, "unit": "edges/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }))


def bind_to_gpu_numa(local: int):
    """Run this process (and the pinned host buffers it allocates from here on) on the CPUs of the NUMA node the GPU
    hangs off - what `numactl --cpunodebind` would do.  Round 1 measured 21.8 GB/s host-to-device next to 55 GB/s
    device-to-host on the same link: the pinned pages lived on the other socket.  Returns a description for the JSON."""
    try:
        import torch
        pr = torch.cuda.get_device_properties(local)
        dev = f"{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        base = f"/sys/bus/pci/devices/{dev}"
        cpus = set()
        for part in open(f"{base}/local_cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        node = open(f"{base}/numa_node").read().strip()
        if cpus:
            os.sched_setaffinity(0, cpus)
            return f"GPU {dev}: NUMA node {node}, {len(cpus)} local CPUs"
    except Exception as e:  # pragma: no cover - informational
        return f"unbound ({type(e).__name__})"
    return "unbound"


DUMP_SAMPLE = 1 << 20  # SdBG stream bytes and about this many edge words sampled by --dump-outputs


def dump_outputs(d, plan, s2s, n_edges_out):
    """Writes what the timed path handed back in its last step as float64 / float32 .npy files under d (every value is
    an integer the float holds exactly; about 23 MB in all at k = 27): the SdBG bucket table {byte offset, items, tips, large
    multiplicities} and totals, the multiplicity histogram of the count stage (`.counting`), a seeded sample of the SdBG
    item stream with its byte positions, and the solid + mercy edges whose content hashes into a fixed range, sorted
    (the device writes the edges in no fixed order, so a sample by position would not be comparable)."""
    import torch
    os.makedirs(d, exist_ok=True)
    totals = s2s.totals.cpu().numpy()
    n_bytes = int(totals[0])
    pos = np.unique(np.random.default_rng(0).integers(0, max(1, n_bytes), size=DUMP_SAMPLE if n_bytes else 0))
    vals = s2s.bytes[torch.from_numpy(pos).to(s2s.bytes.device)].cpu().numpy()
    WE = plan.WE
    e = plan.edges[: n_edges_out * WE].view(-1, WE).to(torch.int64) & 0xFFFFFFFF
    h = torch.zeros(len(e), dtype=torch.int64, device=e.device)
    for j in range(WE):
        h = (h * 0x9E3779B1 + e[:, j]) & 0xFFFFFFFF
    keep = h < int((1 << 32) * min(1.0, DUMP_SAMPLE / max(1, n_edges_out * WE)))
    edges = e[keep].cpu().numpy()
    edges = edges[np.lexsort(edges.T[::-1])] if len(edges) else edges.reshape(0, WE)
    out = {"sdbg_bucket_table": s2s.table.view(-1, 4).cpu().numpy(), "sdbg_totals": totals,
           "counting_hist": plan.mul_hist.cpu().numpy(), "sdbg_bytes_sample_pos": pos,
           "sdbg_bytes_sample": vals.astype(np.float32), "edges_sample": edges}
    for name, a in out.items():
        np.save(os.path.join(d, name + ".npy"), a if a.dtype == np.float32 else a.astype(np.float64))


# ------------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------------
def ours(args):
    import torch
    import torch.distributed as dist

    from megahit_b200 import dev, lib, synth

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: libmhb has no CPU path")
    torch.cuda.set_device(local)
    lib.load().mhb_set_device(local)
    device = torch.device("cuda", local)
    args.all_cpus = os.sched_getaffinity(0)
    args.affinity = bind_to_gpu_numa(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)

    k, m, n_reads, L = args.k, args.m, args.reads, READ_LEN
    n_edges = n_reads * (L - k)
    bin2d = synth.synth_reads_torch(n_reads, L, GENOME_PER_READ * n_reads, ERR, seed=1 + rank, device=device)
    bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=device)])
    bin_words = n_reads * bin2d.shape[1]
    del bin2d

    if world > 1:
        from megahit_b200 import multigpu
        return multigpu.bench(args, bin_dev, bin_words, rank, world, device, METRIC, clocks=ClockSampler(local))

    plan = dev.CountPlan(n_reads, L, k, m, device, want_mercy=True, mode=args.count_mode)
    n_solid = plan.run(bin_dev)  # sizes the SdBG stage (also the first warm-up)
    n_mercy0 = plan.mercy_edges(bin_dev, n_solid)  # wide k: far more than a few per cent of the solid edges
    s2s = dev.S2sPlan(int((n_solid + n_mercy0) * 1.05) + 1024, k + 1, k, device)

    mercy_ev = []
    last = {}

    def step(timed=False):
        # count (extract, partition/sort, solid edges, mercy marks) -> mercy edges -> seq2sdbg over solid + mercy edges:
        # what `megahit_core count` + `seq2sdbg --need_mercy` compute, nothing skipped
        ns = plan.run(bin_dev, timed=timed)
        nm = plan.mercy_edges(bin_dev, ns)
        if timed:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            mercy_ev.append(e)
        s2s.run(plan.edges, None, ns + nm, plan.WE, timed=timed, aux=plan.aux, n_aux=ns)
        last["n_edges_out"] = ns + nm
        return ns

    for _ in range(max(0, args.warmup - 1)):
        step()
    torch.cuda.synchronize()
    clocks = ClockSampler(local)
    clocks.start()
    plan.events.clear()
    s2s.events.clear()
    mercy_ev.clear()
    sort_ms = {"count": [], "s2s": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    launches0 = lib.launch_count()
    for _ in range(args.steps):
        step(timed=True)
        # per-pass device times of this step's two sorts (events recorded inside the timed region)
        sort_ms["s2s"].append(lib.sort_pass_ms(0)[0])
        sort_ms["count"].append(lib.sort_pass_ms(1)[0])
    e1.record()
    launches = (lib.launch_count() - launches0) // max(1, args.steps)  # counted by libmhb at every launch site
    torch.cuda.synchronize()
    clk = clocks.stop()
    ms_per_step = e0.elapsed_time(e1) / args.steps
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, plan, s2s, last["n_edges_out"])
    value = n_edges / (ms_per_step * 1e-3)

    # stage split of the count stage
    ev = plan.events
    stage = {}
    for a, b in (("t0", "extract"), ("extract", "sort"), ("sort", "count"), ("count", "mercy")):
        stage[b] = float(np.mean([x.elapsed_time(y) for x, y in zip(ev[a], ev[b])]))
    if plan.hashed:
        # the two partition passes run inside the count call: split the stage with their own event times
        p_ms = float(np.mean([sum(x) for x in sort_ms["count"]]))
        stage["sort"], stage["count"] = p_ms, stage["count"] - p_ms

    stage["mercy_edges"] = float(np.mean([x.elapsed_time(y) for x, y in zip(ev["mercy"], mercy_ev)]))
    for i, nm in enumerate(("s2s_extract", "s2s_sort", "s2s_emit")):
        stage[nm] = float(np.mean([e[i].elapsed_time(e[i + 1]) for e in s2s.events]))

    # roofline of the dominant kernel: the radix pass over the count records (2*N*S algorithmic bytes per launch)
    peak, peak_src = peaks()
    S = plan.WR * 4
    cpass = np.array(sort_ms["count"])  # steps x passes
    avg_pass_ms = float(cpass.mean())
    achieved = 2.0 * n_edges * S / (avg_pass_ms * 1e-3) / 1e9
    spass = np.array(sort_ms["s2s"])
    n_items = s2s.n_items
    s2s_achieved = 2.0 * n_items * s2s.W * 4 / (float(spass.mean()) * 1e-3) / 1e9
    roofline = {
        "bound": "hbm", "kernel": f"radix passes over the count records ({S} B): k_radix_pass3<{plan.WR}> (stable, look-back); "
                                   "the first pass of a sort is k_part_unstable (no look-back) for 8/12-byte records",
        "achieved": achieved, "peak": peak,
        "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
        "algorithmic_bytes_per_launch": 2 * n_edges * S, "avg_launch_ms": avg_pass_ms,
        "per_pass_ms": [float(x) for x in cpass.mean(axis=0)],
        "per_pass_frac": [float(2.0 * n_edges * S / (x * 1e-3) / 1e9 / peak) for x in cpass.mean(axis=0)],
        "s2s_pass": {"kernel": f"k_radix_pass<{s2s.W}>", "records": int(n_items), "avg_launch_ms": float(spass.mean()),
                     "achieved": s2s_achieved, "frac": s2s_achieved / peak},
    }

    # achieved HBM GB/s of the other stages against their algorithmic bytes (SURVEY.md 8d); informational, never fatal
    stage_roofline = {}
    try:
        E, WE = int(n_solid), plan.WE
        M_items, W2 = int(n_items), s2s.W
        alg = {
            "extract": n_edges * S + bin_words * 4,                      # records written + packed reads read
            "sort": int(cpass.shape[1]) * 2 * n_edges * S,                     # the passes this step really ran
            "count": n_edges * S + E * (WE * 4 + 1),                     # sorted records read + edges and flags written
            "mercy": bin_words * 4,                                      # reads re-scanned against the tip set
            "s2s_extract": E * WE * 4 + M_items * W2 * 4,
            "s2s_sort": len(s2s.sort_bytes) * 2 * M_items * W2 * 4,
            "s2s_emit": 2 * M_items * W2 * 4,
        }
        for nm, b in alg.items():
            if stage.get(nm):
                gbs = b / (stage[nm] * 1e-3) / 1e9
                stage_roofline[nm] = {"algorithmic_bytes": int(b), "gbs": gbs, "frac": gbs / peak}
    except Exception as e:  # pragma: no cover
        stage_roofline = {"error": str(e)}

    count_mode = (f"hashed: {int(cpass.shape[1])} radix passes on the leading key bytes (first one unstable) + per-slice hash "
                  "aggregation in shared memory" if plan.hashed else "sort: LSD radix sort on all key bytes + run-length count")
    # ---- e2e: host buffers through the C ABI (fused build), H2D/D2H copies inside the timed region ----
    host_bin = torch.empty(bin_words, dtype=torch.int32).pin_memory()
    host_bin.copy_(bin_dev[:bin_words])
    hb = host_bin.numpy().view(np.uint32)
    n_items_dev = int(n_items)
    del plan, s2s
    torch.cuda.empty_cache()
    out_buf = torch.empty(max(1 << 20, 3 * n_items_dev), dtype=torch.uint8).pin_memory().numpy()
    e2e_t, h2d, d2h, e2e_ms = [], 0, 0, {}
    for i in range((1 + args.e2e_steps) if args.e2e_steps > 0 else 0):
        t0 = time.perf_counter()
        g = lib.build_host(hb, n_reads, k, m, need_mercy=True, want_edges=False, sdbg_out=out_buf, copy_bytes=False)
        t1 = time.perf_counter()
        if i > 0:
            e2e_t.append(t1 - t0)
        h2d = hb.nbytes
        d2h = int(g["n_bytes"]) + 65536 * 32 + 16 * 8
        e2e_ms = {**g["ms"], "n_mercy": int(g["n_mercy"]), "n_cand": int(g["n_cand"]), "sdbg_items": int(g["n_items"])}
    lib.load().mhb_release()
    e2e_v = n_edges / float(np.mean(e2e_t)) if e2e_t else None

    cpu = None
    if rank == 0 and not args.no_cpu_baseline:
        os.sched_setaffinity(0, args.all_cpus)  # the CPU arm gets every core of the box again
        threads = os.cpu_count() or 1
        runs = [reference_run(args.sample_reads, k, m, threads) for _ in range(3)]  # same library, three times: median
        if all(runs):
            runs.sort(key=lambda r: r["t_count"] + r["t_s2s"])
            r = runs[1]
            cpu = {"value": r["n_edges"] / (r["t_count"] + r["t_s2s"]), "unit": "edges/s", "cores": threads,
                   "kind": "reference",
                   "sample": f"{args.sample_reads} synthetic 150 bp reads (seed 1234), megahit_core count+seq2sdbg --need_mercy, "
                             f"median of 3 runs (count {r['t_count']:.2f} s, seq2sdbg {r['t_s2s']:.2f} s)",
                   "run_times_s": [round(x["t_count"] + x["t_s2s"], 3) for x in runs], "cpu": cpu_info()}

    print(json.dumps({
        "metric": METRIC, "value": value, "unit": "edges/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u32",
        "data": "synthetic",
        "config": {"workload": f"synthetic {n_reads}x{L}bp reads (30x, 1% subst.), k={k}, m={m}, 1xH100 single-GPU "
                               "sdbg_build: count (extract + partition/sort + solid count + mercy marks) + mercy-edge "
                               "generation + seq2sdbg (extract+radix+emit) over solid + mercy edges; the seq2sdbg extract skips the $-items the count stage's in/out flags prove the emitter would discard (same bytes out)",
                   "count_mode": count_mode, "host_affinity": args.affinity,
                   "n_edge_records": n_edges, "n_solid_edges": int(n_solid), "n_sdbg_sort_items": int(n_items),
                   "l2_note": "inputs (>= 4.9 GB per kernel) exceed the 50 MB L2, no explicit flush needed"},
        "stage_ms": stage, "stage_roofline": stage_roofline,
        "roofline": roofline, "cpu_baseline": cpu, "clocks": clk,
        "e2e": {"value": e2e_v, "unit": "edges/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
                "ms_per_step": float(np.mean(e2e_t)) * 1e3 if e2e_t else None, "api": "mhb_build_host (pinned host buffers; count -> device mercy edges -> seq2sdbg, SdBG stream D2H)",
                "stages": e2e_ms},
        "gpu_launches": launches,
    }))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--reads", type=int, default=10_000_000, help="reads per GPU")
    ap.add_argument("--k", type=int, default=27)
    ap.add_argument("--m", type=int, default=2)
    ap.add_argument("--sample-reads", type=int, default=1_000_000, help="bounded CPU sample (reference arm / cpu_baseline)")
    ap.add_argument("--e2e-steps", type=int, default=2)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed to DIR/<name>.npy")
    ap.add_argument("--count-mode", default=None, choices=["sort", "hashed", "auto"],
                    help="count stage algorithm (default: $MHB_COUNT_MODE, else hashed where supported)")
    args = ap.parse_args()
    if args.impl == "reference":
        # exactly K timed + W warm-up steps; the per-step sample is sized so the whole run stays within minutes
        # (~8 s per 1 M reads on 8 host cores)
        budget_s = 160.0
        per_step = budget_s / max(1, args.steps + args.warmup)
        args.sample_reads = int(max(100_000, min(args.sample_reads, 1_000_000 * per_step / 8.0)))
        reference_arm(args)
    else:
        ours(args)


if __name__ == "__main__":
    main()
