#!/usr/bin/env python
"""Times the seq2sdbg sort + emit at the bench workload (bench.py's synthetic library: 10 M x 150 bp reads, 30x, 1 %
substitutions, seed 1, k = 27, m = 2): the items of the bench step (pruned extract over solid + mercy edges; with
--all-six every edge's six items, as file-level seq2sdbg makes them) are made once, then sorted and emitted --reps
times by

  old    mhb_s2s_sort followed by mhb_s2s_emit (the bucket kernel writes the sorted items back, the emitter reads them
         again: k_s2s_judge, the chunk-total scans, k_s2s_gather, k_bucket_starts, k_bucket_finalize);
  new    mhb_s2s_sort_emit (the bucket kernel emits every bucket it sorts; k_s2s_row_sums, k_s2s_bucket_table and
         k_s2s_bucket_gather finish the stream).

Reports the whole call (CUDA events, includes the host read-backs of the bucket kernel's leftovers), the per-kernel
split from torch.profiler and the kernel launches per call, as medians of --reps, and checks that both give the same
item bytes, bucket table and totals.  Prints one JSON document and writes it to scripts/out/s2s_emit_time[_six].json.

  s2s_emit_time.py [--reads N] [--k K] [--reps R] [--all-six]
"""
import argparse
import ctypes as C
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from megahit_b200 import dev, lib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reads", type=int, default=10_000_000)
ap.add_argument("--k", type=int, default=27)
ap.add_argument("--m", type=int, default=2)
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--all-six", action="store_true", help="every edge's six items (no pruning), as file-level seq2sdbg")
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("s2s_emit_time.py needs a CUDA device")

L = lib.load()
device = torch.device("cuda", 0)
n_reads, RL, k, m = args.reads, 150, args.k, args.m
bin2d = synth.synth_reads_torch(n_reads, RL, 5 * n_reads, 0.01, seed=1, device=device)  # bench.py's library
bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=device)])
del bin2d
plan = dev.CountPlan(n_reads, RL, k, m, device, want_mercy=True)
ns = plan.run(bin_dev)
nm = plan.mercy_edges(bin_dev, ns)
ne = ns + nm
W = lib.s2s_record_words(k)
cap = 6 * ne
items = torch.zeros(cap * W + 8, dtype=torch.int32, device=device)
hist = torch.zeros(256, dtype=torch.int64, device=device)
if args.all_six:
    seqs = lib.DevSeqs(plan.edges.data_ptr(), plan.edges.numel(), ne, k + 1, None, None, None, None, plan.WE)
    lib._check(L.mhb_s2s_extract(dev._stream(), C.byref(seqs), k, dev._ptr(items), cap, dev._ptr(hist),
                                 lib.s2s_sort_hist_byte(cap, k)))
    n = cap
else:
    cursor = torch.zeros(1, dtype=torch.int64, device=device)
    lib._check(L.mhb_s2s_extract_edges_pruned(dev._stream(), dev._ptr(plan.edges), dev._ptr(plan.aux), ne, ns, k,
                                              dev._ptr(items), cap, dev._ptr(cursor), dev._ptr(hist),
                                              lib.s2s_sort_hist_byte(cap, k)))
    n = int(cursor.item())
    assert lib.s2s_sort_hist_byte(n, k) == lib.s2s_sort_hist_byte(cap, k)
del plan, bin_dev
items = items[: n * W + 8].clone()
torch.cuda.synchronize()

i32 = dict(dtype=torch.int32, device=device)
a, b = torch.empty(n * W + 8, **i32), torch.empty(n * W + 8, **i32)
cap_bytes = n * (4 + 4 * ((k + 15) // 16)) + 16
out = torch.empty(cap_bytes, dtype=torch.uint8, device=device)
table = torch.zeros(65536 * 4, dtype=torch.int64, device=device)
totals = torch.zeros(16, dtype=torch.int64, device=device)
ws_new = torch.empty(L.mhb_s2s_sort_emit_workspace_bytes(n, k), dtype=torch.uint8, device=device)
ws_old = torch.empty(L.mhb_s2s_sort_workspace_bytes(n, k), dtype=torch.uint8, device=device)
scr_old = torch.empty(L.mhb_s2s_emit_scratch_bytes(n, k), dtype=torch.uint8, device=device)


def run_old():
    srt = dev.s2s_sort(a, b, n, k, hist, ws_old)
    lib._check(L.mhb_s2s_emit(dev._stream(), dev._ptr(srt), n, k, dev._ptr(out), cap_bytes, dev._ptr(table),
                              dev._ptr(totals), dev._ptr(scr_old), scr_old.numel()))


def run_new():
    dev.s2s_sort_emit(a, b, n, k, hist, out, table, totals, ws_new, cap_bytes)


def timed(fn):
    """(whole call ms, {kernel group: ms}, launches) of one run from fresh items"""
    a[: n * W + 8].copy_(items)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = lib.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
    launches = lib.launch_count() - l0
    kern = defaultdict(float)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        if "k_part_unstable" in name or "k_radix_pass" in name or "k_hist_scan256" in name:
            key = "bucket passes"
        elif "k_s2s_local_sort" in name:
            key = "k_s2s_local_sort (sort+emit)" if "true" in name or "Lb1E" in name else "k_s2s_local_sort"
        else:
            for nm_ in ("k_bucket_bounds", "k_s2s_judge", "k_s2s_gather", "k_bucket_starts", "k_bucket_finalize",
                        "k_s2s_bucket_table", "k_s2s_row_sums", "k_s2s_bucket_gather", "k_s2s_fold_bucket", "scan"):
                if nm_ in name:
                    key = nm_ if nm_ != "scan" else "scan32 (chunk totals)"
                    break
            else:
                key = "other: " + name[:60]
        kern[key] += us / 1e3
    return e0.elapsed_time(e1), dict(kern), launches


def result():
    torch.cuda.synchronize()
    tot = totals.cpu().numpy().copy()
    return tot, table.cpu().numpy().copy(), out[: int(tot[0])].cpu().numpy().copy()


timed(run_old)
timed(run_new)
res = {}
for name, fn in (("old", run_old), ("new", run_new)):
    res[name] = {"ms": [], "kern": defaultdict(list), "launches": 0}
for _ in range(args.reps):  # alternating
    for name, fn in (("old", run_old), ("new", run_new)):
        ms, kern, launches = timed(fn)
        res[name]["ms"].append(ms)
        res[name]["launches"] = launches
        for key, v in kern.items():
            res[name]["kern"][key].append(v)
timed(run_old)
ref = result()
st_old = lib.s2s_sort_stats()
timed(run_new)
got = result()
st_new = lib.s2s_sort_stats()
same = all(np.array_equal(x, y) for x, y in zip(ref, got))
gpu = torch.cuda.get_device_properties(0)
doc = {
    "gpu": gpu.name, "n_items": int(n), "k": k, "all_six": bool(args.all_six), "reps": args.reps,
    "sdbg_items": int(ref[0][1]), "sdbg_bytes": int(ref[0][0]),
    "sort_stats_old": list(st_old), "sort_stats_new": list(st_new),
    "same_bytes_table_totals": bool(same),
}
for name in ("old", "new"):
    r = res[name]
    doc[name] = {"total_ms": float(np.median(r["ms"])), "all_ms": [round(float(x), 3) for x in r["ms"]],
                 "launches": int(r["launches"]),
                 "kernels_ms": {key: round(float(np.median(v)), 3) for key, v in sorted(r["kern"].items())}}
doc["saved_ms"] = doc["old"]["total_ms"] - doc["new"]["total_ms"]
print(json.dumps(doc, indent=1))
os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
with open(os.path.join(ROOT, "scripts", "out", "s2s_emit_time%s.json" % ("_six" if args.all_six else "")), "w") as f:
    json.dump(doc, f, indent=1)
if not same:
    raise SystemExit("the fused call's output differs from sort + emit")
