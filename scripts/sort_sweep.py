"""Radix-pass variant sweep (run on the GPU box): for every MHB_SORT_CFG value, in its own process (a hang or a
crash only loses that variant), check the sort against torch's stable sort and time the passes on a count-sized
(WR=2) and a seq2sdbg-sized (WR=3) array.  Writes scripts/out/sort_sweep.json and scripts/out/best_cfg."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHILD = r'''
import json, sys, os
import numpy as np, torch
sys.path.insert(0, %r)
from megahit_b200 import dev, lib
cfg = int(sys.argv[1]); n2 = int(sys.argv[2]); n3 = int(sys.argv[3])
lib._check(lib.load().mhb_set_sort_cfg(cfg))
res = {"cfg": cfg}
g = torch.Generator(device="cuda"); g.manual_seed(7)

def check(words, n, sort_bytes):
    a = torch.randint(-2**31, 2**31 - 1, (n * words + 4,), generator=g, device="cuda", dtype=torch.int32)
    if words == 2:
        a[0:2 * n:2] &= 0x0F0F0F0F   # long ties in the high word: stability matters
    recs = a[: n * words].clone().view(n, words)
    out = dev.sort_records(a, torch.empty_like(a), n, words, sort_bytes)
    got = out[: n * words].view(n, words)
    order = torch.arange(n, device="cuda")
    for b in sort_bytes:
        digit = (recs[order, words - 1 - (b >> 2)].to(torch.int64) >> (8 * (b & 3))) & 255
        order = order[torch.sort(digit, stable=True).indices]
    return bool((got == recs[order]).all().item())

ok = True
for words, n, sb in ((2, 1, [1, 2, 3, 4, 5, 6, 7]), (2, 4607, [1, 2, 3, 4, 5, 6, 7]), (2, 6145, [1, 2, 3, 4, 5, 6, 7]),
                     (2, 6912 * 5 + 17, [1, 2, 3, 4, 5, 6, 7]), (2, 3_000_001, [1, 2, 3, 4, 5, 6, 7]),
                     (3, 1_500_007, [0, 1, 2, 4, 5, 6, 7, 8, 9, 10]), (3, 3071, [2, 5, 11])):
    c = check(words, n, sb)
    ok = ok and c
    if not c:
        res.setdefault("failed", []).append([words, n])
res["ok"] = ok

def timeit(words, n, sort_bytes, reps=2):
    a = torch.randint(-2**31, 2**31 - 1, (n * words + 4,), generator=g, device="cuda", dtype=torch.int32)
    b = torch.empty_like(a)
    ws = torch.empty(lib.load().mhb_sort_workspace_bytes(n, words), dtype=torch.uint8, device="cuda")
    best = None
    for _ in range(reps):
        dev.sort_records(a, b, n, words, sort_bytes, None, ws)
        torch.cuda.synchronize()
        ms = lib.sort_pass_ms(0)[0]
        if best is None or sum(ms) < sum(best):
            best = ms
    return [float(x) for x in best]

if ok:
    ms2 = timeit(2, n2, [1, 2, 3, 4, 5, 6, 7])
    res["wr2_pass_ms"] = ms2
    res["wr2_gbs"] = 2 * n2 * 8 / (sum(ms2) / len(ms2) * 1e-3) / 1e9
    # the same passes when every record carries the same digit (byte 0 cleared): the scatter degenerates to a copy,
    # so the difference to the random-digit time is what the 256-stream write pattern costs
    a = torch.randint(-2**31, 2**31 - 1, (n2 * 2 + 4,), generator=g, device="cuda", dtype=torch.int32)
    a[1:2 * n2:2] &= 0x7FFFFF00
    b = torch.empty_like(a)
    dev.sort_records(a, b, n2, 2, [0, 0, 0])
    torch.cuda.synchronize()
    res["wr2_const_digit_pass_ms"] = [float(x) for x in lib.sort_pass_ms(0)[0]]
    del a, b
    ms3 = timeit(3, n3, [0, 1, 2, 4, 5, 6, 7, 8, 9, 10])
    res["wr3_pass_ms"] = ms3
    res["wr3_gbs"] = 2 * n3 * 12 / (sum(ms3) / len(ms3) * 1e-3) / 1e9
print("RESULT " + json.dumps(res))
''' % ROOT


def main():
    cfgs = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else [256 + b for b in (0x080, 0x180, 0x1080, 0x8080, 0x10080, 0x18080, 0x9080, 0x8082, 0x10082, 0x082)]
    n2 = int(float(sys.argv[2])) if len(sys.argv) > 2 else 1_230_000_000
    n3 = int(float(sys.argv[3])) if len(sys.argv) > 3 else 347_000_000
    os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
    out = []
    for c in cfgs:
        try:
            p = subprocess.run([sys.executable, "-c", CHILD, str(c), str(n2), str(n3)], capture_output=True, text=True,
                               timeout=int(os.environ.get("MHB_SWEEP_TIMEOUT", "75")))
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            r = json.loads(line[-1][7:]) if line else {"cfg": c, "ok": False, "error": (p.stderr or "")[-600:]}
        except subprocess.TimeoutExpired:
            r = {"cfg": c, "ok": False, "error": "timeout (hang?)"}
        out.append(r)
        print(json.dumps(r), flush=True)
    json.dump(out, open(os.path.join(ROOT, "scripts", "out", "sort_sweep.json"), "w"), indent=1)
    good = [r for r in out if r.get("ok") and "wr2_gbs" in r]
    if good:
        best = max(good, key=lambda r: r["wr2_gbs"])
        open(os.path.join(ROOT, "scripts", "out", "best_cfg"), "w").write(str(best["cfg"]))
        print("best:", best["cfg"], "%.0f GB/s (WR=2), %.0f GB/s (WR=3)" % (best["wr2_gbs"], best["wr3_gbs"]))


if __name__ == "__main__":
    main()
