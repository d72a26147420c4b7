#!/usr/bin/env python
"""Times the seq2sdbg item sort alone at the bench workload (bench.py's synthetic library: 10 M x 150 bp reads, 30x,
1 % substitutions, seed 1, k = 27, m = 2): the items of the bench step (pruned extract over solid + mercy edges) are
made once, then sorted --reps times by

  new    mhb_s2s_sort: the two bucket passes, k_bucket_bounds and k_s2s_local_sort, each from torch.profiler's kernel
         times, plus the whole call with CUDA events (includes the host read-back of the oversized-bucket count);
  old    mhb_sort_records_relaxed on every byte of mhb_s2s_sort_bytes (the sort before the bucket kernel).

Reports medians, the largest bucket, the number of buckets the bucket kernel left to the radix engine, and checks that
both sorts give the same key sequence.  Prints one JSON document and writes it to scripts/out/s2s_sort_time.json.

  s2s_sort_time.py [--reads N] [--k K] [--reps R]
"""
import argparse
import json
import os
import sys

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
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("s2s_sort_time.py needs a CUDA device")

L = lib.load()
device = torch.device("cuda", 0)
n_reads, RL, k, m = args.reads, 150, args.k, args.m
bin2d = synth.synth_reads_torch(n_reads, RL, 5 * n_reads, 0.01, seed=1, device=device)  # bench.py's library
bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=device)])
del bin2d
plan = dev.CountPlan(n_reads, RL, k, m, device, want_mercy=True)
ns = plan.run(bin_dev)
nm = plan.mercy_edges(bin_dev, ns)
s2s = dev.S2sPlan(int((ns + nm) * 1.05) + 1024, k + 1, k, device)
s2s.run(plan.edges, None, ns + nm, plan.WE, aux=plan.aux, n_aux=ns)
n, W = s2s.n_items, s2s.W
s2s.hist0.zero_()  # the sort has run in place: extract again for an unsorted copy
s2s.cursor.zero_()
lib._check(L.mhb_s2s_extract_edges_pruned(dev._stream(), dev._ptr(plan.edges), dev._ptr(plan.aux), ns + nm, ns, k,
                                          dev._ptr(s2s.a), s2s.a.numel() // W, dev._ptr(s2s.cursor), dev._ptr(s2s.hist0),
                                          lib.s2s_sort_hist_byte(n, k)))
items = s2s.a[: n * W].clone()
hist_new = s2s.hist0.clone()
hist_old = torch.zeros(256, dtype=torch.int64, device=device)
s2s.cursor.zero_()
lib._check(L.mhb_s2s_extract_edges_pruned(dev._stream(), dev._ptr(plan.edges), dev._ptr(plan.aux), ns + nm, ns, k,
                                          dev._ptr(s2s.b), s2s.b.numel() // W, dev._ptr(s2s.cursor), dev._ptr(hist_old),
                                          s2s.sort_bytes[0]))
del plan
torch.cuda.synchronize()
a, b = s2s.a, s2s.b
ws_old = torch.empty(L.mhb_sort_workspace_bytes(n, W), dtype=torch.uint8, device=device)


def run_new():
    a[: n * W].copy_(items)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = dev.s2s_sort(a, b, n, k, hist_new, s2s.ws)
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def run_old():
    a[: n * W].copy_(items)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = dev.sort_records(a, b, n, W, s2s.sort_bytes, hist_old, ws_old, relaxed=True)
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def key_words(t):
    r = t[: n * W].view(-1, W).clone()
    r[:, W - 1] &= ~0xFFFF  # the multiplicity bits are not sorted
    return r


run_new()
run_old()
new_ms, old_ms, kern = [], [], {"passes": [], "bounds": [], "bucket": []}
for _ in range(args.reps):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out, ms = run_new()
    new_ms.append(ms)
    t = {"passes": 0.0, "bounds": 0.0, "bucket": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        if "k_part_unstable" in name or "k_radix_pass" in name or "k_hist_scan256" in name:
            t["passes"] += us / 1e3
        elif "k_bucket_bounds" in name:
            t["bounds"] += us / 1e3
        elif "k_s2s_local_sort" in name:
            t["bucket"] += us / 1e3
    for key in kern:
        kern[key].append(t[key])
    old_out, ms = run_old()
    old_ms.append(ms)

new_out, _ = run_new()
new_keys = key_words(new_out)
bucket = (new_keys[:, 0] >> 16) & 0xFFFF
sizes = torch.bincount(bucket.to(torch.int64), minlength=65536)
old_out, _ = run_old()
same = bool(torch.equal(new_keys, key_words(old_out)))
n_over, items_over, n_large = lib.s2s_sort_stats()
gpu = torch.cuda.get_device_properties(0)
res = {
    "gpu": gpu.name, "n_items": int(n), "record_bytes": 4 * W, "k": k, "reps": args.reps,
    "new_ms": {"total": float(np.median(new_ms)), **{key: float(np.median(v)) for key, v in kern.items()}},
    "old_ms": float(np.median(old_ms)), "old_passes": len(s2s.sort_bytes),
    "new_total_all": [float(x) for x in new_ms], "old_all": [float(x) for x in old_ms],
    "largest_bucket": int(sizes.max().item()), "mean_bucket": float(n / 65536),
    "oversized_buckets": int(n_over), "oversized_items": int(items_over), "large_geometry_buckets": int(n_large),
    "same_key_sequence_as_old": same,
}
print(json.dumps(res, indent=1))
os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
with open(os.path.join(ROOT, "scripts", "out", "s2s_sort_time.json"), "w") as f:
    json.dump(res, f, indent=1)
