#!/usr/bin/env python
"""Times each piece of the count stage's mercy path at the bench workload (bench.py's synthetic library: 10 M x 150 bp
reads, 30x, 1 % substitutions, seed 1, k = 27, m = 2) with CUDA events, after a warm-up:

  tip_edges     mhb_count_tip_edges            tipset_build   mhb_tipset_build
  mark          mhb_count_mark_mercy           mark_empty     the same kernel against an empty tip set (the scan's floor)
  candidates    mhb_mercy_candidates           lut            the 12-mer look-up table (mhb_edge_lut_build)
  edges_count   mhb_mercy_edges_count          edges_write    mhb_mercy_edges_write
  stage_mercy / stage_mercy_edges: the two bench stages (dev.CountPlan.mercy / .mercy_edges) timed whole; the gap between
  a stage and the sum of its pieces is host synchronisation.

  mercy_time.py [--reads N] [--reps R] [--filter SPEC ...]

Every --filter SPEC is one arm: the value of MHB_TIPSET_FILTER for that arm ("default" = unset, "global", or a word
count); arms alternate within each repetition, so two filter plans are compared in one process.  Prints one JSON
document and writes it to scripts/out/mercy_time.json.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
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
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--filter", action="append", default=None, help="MHB_TIPSET_FILTER of one arm (default: unset)")
args = ap.parse_args()
arms = args.filter or ["default"]
if not torch.cuda.is_available():
    raise SystemExit("mercy_time.py needs a CUDA device")

L = lib.load()
device = torch.device("cuda", 0)
n_reads, RL, k, m = args.reads, 150, args.k, args.m
bin2d = synth.synth_reads_torch(n_reads, RL, 5 * n_reads, 0.01, seed=1, device=device)  # bench.py's library
bin_dev = torch.cat([bin2d.reshape(-1), torch.zeros(8, dtype=torch.int32, device=device)])
del bin2d
plan = dev.CountPlan(n_reads, RL, k, m, device, want_mercy=True)
n_solid = plan.run(bin_dev)
plan.mercy_edges(bin_dev, n_solid)
reads = plan._reads(bin_dev)
S = dev._stream
P = dev._ptr
first_e, last_e = torch.empty_like(plan.first), torch.empty_like(plan.last)


def set_arm(spec):
    if spec == "default":
        os.environ.pop("MHB_TIPSET_FILTER", None)
    else:
        os.environ["MHB_TIPSET_FILTER"] = spec


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def one_rep():
    t = {}
    t["stage_mercy"], _ = timed(lambda: plan.mercy(bin_dev))
    t["stage_mercy_edges"], n_mercy = timed(lambda: plan.mercy_edges(bin_dev, n_solid))
    n_tip = C.c_uint64(0)
    t["tip_edges"], _ = timed(lambda: lib._check(L.mhb_count_tip_edges(S(), P(plan.aux), n_solid, C.byref(n_tip))))
    nt = n_tip.value
    need = L.mhb_tipset_bytes(nt, k)
    t["tipset_build"], _ = timed(lambda: lib._check(L.mhb_tipset_build(S(), P(plan.edges), P(plan.aux), n_solid, k,
                                                                        P(plan.tipset), need, nt)))
    t["mark"], _ = timed(lambda: lib._check(L.mhb_count_mark_mercy(S(), C.byref(reads), k, P(plan.tipset), need, nt,
                                                                    P(plan.first), P(plan.last))))
    nc = C.c_uint64(0)
    t["candidates"], _ = timed(lambda: lib._check(L.mhb_mercy_candidates(S(), P(plan.first), P(plan.last), n_reads, P(plan.cand),
                                                                          C.byref(nc), P(plan.cand_scratch),
                                                                          plan.cand_scratch.numel())))
    ms_need = L.mhb_mercy_edges_scratch_bytes(nc.value, RL)
    core = ms_need - 512 - L.mhb_edge_lut_bytes()
    lut = C.c_void_p(plan.mercy_scratch.data_ptr() + core)
    t["lut"], _ = timed(lambda: lib._check(L.mhb_edge_lut_build(S(), P(plan.edges), n_solid, k, lut)))
    seg_e = (C.c_void_p * 1)(plan.edges.data_ptr())
    seg_n = (C.c_uint64 * 1)(n_solid)
    seg_l = (C.c_void_p * 1)(lut)
    nm = C.c_uint64(0)
    t["edges_count"], _ = timed(lambda: lib._check(L.mhb_mercy_edges_count(S(), C.byref(reads), P(plan.cand), nc.value, RL, k, 1,
                                                                            seg_e, seg_n, seg_l, None, C.byref(nm),
                                                                            P(plan.mercy_scratch), core)))
    out = C.c_void_p(plan.edges.data_ptr() + n_solid * plan.WE * 4)
    t["edges_write"], _ = timed(lambda: lib._check(L.mhb_mercy_edges_write(S(), C.byref(reads), P(plan.cand), nc.value, RL, k, out,
                                                                            plan.cap_edges - n_solid, nm.value,
                                                                            P(plan.mercy_scratch), core)))
    # the scan against an empty tip set: every filter probe misses, no table probe
    empty = torch.zeros(L.mhb_tipset_bytes(0, k), dtype=torch.uint8, device=device)
    lib._check(L.mhb_tipset_build(S(), P(plan.edges), P(plan.aux), 0, k, P(empty), empty.numel(), 0))
    t["mark_empty"], _ = timed(lambda: lib._check(L.mhb_count_mark_mercy(S(), C.byref(reads), k, P(empty), empty.numel(), 0,
                                                                          P(first_e), P(last_e))))
    t["gap_mercy"] = t["stage_mercy"] - (t["tip_edges"] + t["tipset_build"] + t["mark"])
    t["gap_mercy_edges"] = t["stage_mercy_edges"] - (t["candidates"] + t["lut"] + t["edges_count"] + t["edges_write"])
    hdr = plan.tipset[:32].cpu().numpy().view(np.uint32)
    counts = {"n_solid": int(n_solid), "n_tip": int(nt), "n_cand": int(nc.value), "n_mercy": int(nm.value),
              "n_mercy_stage": int(n_mercy), "tipset_bytes": int(need), "tipset_header_u32": [int(x) for x in hdr]}
    marks = (int(plan.first[:n_reads].sum().item()), int(plan.last[:n_reads].sum().item()))
    return t, counts, marks


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "nvidia-smi": f"unavailable ({type(e).__name__})"}


res = {a: {"t": [], "counts": None, "marks": set()} for a in arms}
for i in range(args.warmup + args.reps):
    for a in arms:
        set_arm(a)
        t, counts, marks = one_rep()
        if i >= args.warmup:
            res[a]["t"].append(t)
        res[a]["counts"] = counts
        res[a]["marks"].add(marks)
set_arm("default")
info = gpu_info()
doc = {"workload": f"{n_reads} x {RL} bp synthetic reads (seed 1), k={k}, m={m}", "reps": args.reps, "gpu": info, "arms": {}}
for a in arms:
    keys = res[a]["t"][0].keys()
    doc["arms"][a] = {
        "counts": res[a]["counts"],
        "marks_checksum": sorted(res[a]["marks"]),
        "ms_median": {kk: round(float(np.median([t[kk] for t in res[a]["t"]])), 3) for kk in keys},
        "ms_min": {kk: round(float(np.min([t[kk] for t in res[a]["t"]])), 3) for kk in keys},
        "ms_max": {kk: round(float(np.max([t[kk] for t in res[a]["t"]])), 3) for kk in keys},
    }
os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
with open(os.path.join(ROOT, "scripts", "out", "mercy_time.json"), "w") as f:
    json.dump(doc, f, indent=1)
print(json.dumps(doc, indent=1))
