"""count on several GPUs for any read library (`megahit_core count --gpus N`, mhb_count_run_multi, lib.count_run(gpus=N)):

* the extraction into the owners (mhb_count_extract_owners) against mhb_count_extract, at every record width class,
  on variable-length reads, with and without a round filter, and its bucket histogram;
* the reference's fixtures at N = 2 and 3 (variable-length ones included): digests, one file per rank, and nothing left
  for `seq2sdbg --need_mercy`;
* forced rounds (mhb_set_round_limit in the calling process, which the forked workers inherit): the same digests, and a
  single bucket above the cap refused before any round buffer exists;
* a seeded 1 M-read variable-length library against the single-GPU count (and the reference binary when it is built);
* a library of exactly N reads, a rank whose share holds no record, a rank without mercy candidates.
Ranks share a device when N exceeds the device count, so all of it runs on one GPU."""
import ctypes as C
import glob
import json
import os
import re
import subprocess
import sys
import uuid

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib, synth
from oracle import gen_golden_cli as GC

OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def _one_process_only():
    """the compute mode of a device that admits one process only (ranks sharing it could not run), else None"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
    except (OSError, subprocess.TimeoutExpired):
        return None
    modes = [m.strip() for m in r.stdout.splitlines() if m.strip()]
    bad = [m for m in modes if m in ("Exclusive_Process", "Prohibited")]
    return bad[0] if bad and len(modes) < 3 else None  # up to 3 ranks: fewer devices are shared


_MODE = _one_process_only()
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")]


def _run(cmd, env=None, ok=True):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if ok:
        assert r.returncode == 0, (cmd, r.stderr[-3000:])
    return r


def _count_cmd(libp, p, k, m, gpus=None, core=OURS):
    cmd = [core, "count", "-k", str(k), "-m", str(m), "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p,
           "--num_cpu_threads", "4", "--read_lib_file", libp]
    return cmd + (["--gpus", str(gpus)] if gpus else [])


def _mercy_cmd(p, k, core=OURS):
    return [core, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p, "--num_cpu_threads", "4",
            "-k", str(k), "--kmer_from", "0", "--input_prefix", p, "--need_mercy"]


def _index(b, n_reads, k):
    """rec_off / edge_off of a `.bin` word stream"""
    rec, edge = np.zeros(n_reads + 1, np.uint64), np.zeros(n_reads + 1, np.uint64)
    pos = 0
    for r in range(n_reads):
        L = int(b[pos])
        rec[r], rec[r + 1] = pos, pos + 1 + (L + 15) // 16
        edge[r + 1] = edge[r] + max(0, L - k)
        pos = int(rec[r + 1])
    return rec, edge


def _dev_reads(b, n_reads, k, keep):
    import torch
    dv = torch.device("cuda")
    rec, edge = _index(b, n_reads, k)
    buf = torch.from_numpy(np.concatenate([b, np.zeros(16, np.uint32)]).view(np.int32)).to(dv)
    d_rec = torch.from_numpy(rec.view(np.int64)).to(dv)
    d_edge = torch.from_numpy(edge.view(np.int64)).to(dv)
    keep += [buf, d_rec, d_edge]
    return lib.DevReads(buf.data_ptr(), len(b), n_reads, 0, d_rec.data_ptr(), d_edge.data_ptr()), int(edge[-1])


def _records(b, n_reads, k):
    """every count record of a `.bin` stream (mhb_count_extract), (n, WR) uint32"""
    import torch
    keep = []
    rd, n = _dev_reads(b, n_reads, k, keep)
    WR = lib.count_record_words(k)
    a = torch.zeros(n * WR + 8, dtype=torch.int32, device="cuda")
    lib._check(lib.load().mhb_count_extract(None, C.byref(rd), k, C.c_void_p(a.data_ptr()), n, None, 0))
    torch.cuda.synchronize()
    return a.cpu().numpy().view(np.uint32)[: n * WR].reshape(-1, WR)


def _sorted_rows(a):
    return a[np.lexsort(a.T[::-1])] if len(a) else a


# ------------------------------------------------------------------------------------------------
# 1. the extraction into the owners
# ------------------------------------------------------------------------------------------------
def _width_classes():
    """one k per (key words, record words) pair the count dispatch instantiates"""
    seen = {}
    for k in range(12, 256):
        c = ((k + 1 + 15) // 16, lib.count_record_words(k))
        seen.setdefault(c, k)
    return sorted(seen.values())


def _var_lib(k, seed):
    """variable-length reads: zero-length ones, ones shorter than k + 1, and one of 2000 bases"""
    b = synth.synth_reads_varlen(300, 0, k + 200, genome_len=5000, seed=seed)
    long_read = synth.synth_reads_varlen(1, 2000, 2000, genome_len=5000, seed=seed + 1)
    return np.concatenate([b, np.array([0], np.uint32), long_read, np.array([5, 0x1B000000], np.uint32)])


def _n_reads(b):
    n, pos = 0, 0
    while pos < len(b):
        pos += 1 + (int(b[pos]) + 15) // 16
        n += 1
    assert pos == len(b)
    return n


def owner_check(b, k, n_owners, filt, seed):
    import torch
    dv = torch.device("cuda")
    L = lib.load()
    n_reads = _n_reads(b)
    ref = _records(b, n_reads, k)
    WR = ref.shape[1] if len(ref) else lib.count_record_words(k)
    bucket = (ref[:, 0] >> np.uint32(16)).astype(np.int64)
    keep = []
    rd, n = _dev_reads(b, n_reads, k, keep)
    assert n == len(ref)
    # histogram mode
    h = torch.zeros(65536, dtype=torch.int64, device=dv)
    lib._check(L.mhb_count_extract_owners(None, C.byref(rd), k, C.c_void_p(h.data_ptr()), None, None, None, None, None, None))
    torch.cuda.synchronize()
    assert np.array_equal(h.cpu().numpy(), np.bincount(bucket, minlength=65536))
    # write mode: random owners, every owner's range [lo, hi] (empty for the last owner when filtering)
    rng = np.random.default_rng(seed)
    lut = rng.integers(0, n_owners, size=256).astype(np.uint8)
    lo = np.zeros(n_owners, np.uint32)
    hi = np.full(n_owners, 65535, np.uint32)
    if filt:
        for o in range(n_owners):
            a, c = sorted(rng.integers(0, 65536, size=2))
            lo[o], hi[o] = a, c
        lo[-1], hi[-1] = 7, 6
    own = lut[bucket >> 8] if len(ref) else np.zeros(0, np.uint8)
    sel = [(own == o) & (bucket >= lo[o]) & (bucket <= hi[o]) for o in range(n_owners)]
    counts = np.array([int(s.sum()) for s in sel], np.int64)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    gap = 3  # guard records between the segments, which must stay untouched
    buf = torch.full((int(off[-1] + gap * n_owners) * WR + 8,), -7, dtype=torch.int32, device=dv)
    base = np.array([buf.data_ptr() + 4 * WR * int(off[o] + gap * o) for o in range(n_owners)], np.uint64)
    d_lut = torch.from_numpy(lut.view(np.int8)).to(dv)
    d_base = torch.from_numpy(base.view(np.int64)).to(dv)
    d_cursor = torch.zeros(n_owners, dtype=torch.int64, device=dv)
    d_cap = torch.from_numpy(counts).to(dv)
    d_lo = torch.from_numpy(lo.view(np.int32)).to(dv)
    d_hi = torch.from_numpy(hi.view(np.int32)).to(dv)
    lib._check(L.mhb_count_extract_owners(None, C.byref(rd), k, None, C.c_void_p(d_lut.data_ptr()),
                                          C.c_void_p(d_base.data_ptr()), C.c_void_p(d_cursor.data_ptr()),
                                          C.c_void_p(d_cap.data_ptr()), C.c_void_p(d_lo.data_ptr()),
                                          C.c_void_p(d_hi.data_ptr())))
    torch.cuda.synchronize()
    assert (d_cursor.cpu().numpy() == counts).all()
    out = buf.cpu().numpy().view(np.uint32)
    for o in range(n_owners):
        s = (int(off[o]) + gap * o) * WR
        got = out[s: s + int(counts[o]) * WR].reshape(-1, WR)
        assert np.array_equal(_sorted_rows(got), _sorted_rows(ref[sel[o]])), f"owner {o}"
        assert (out[s + int(counts[o]) * WR: s + (int(counts[o]) + gap) * WR] == np.uint32(0xFFFFFFF9)).all(), f"guard {o}"
    return len(ref), counts


@pytest.mark.parametrize("k", _width_classes())
@pytest.mark.parametrize("filt", [False, True])
def test_extract_owners_at_every_width(k, filt):
    b = _var_lib(k, seed=k)
    n, counts = owner_check(b, k, 3, filt, seed=k)
    assert n > 0 and counts.sum() > 0
    if not filt:
        assert counts.sum() == n


def test_extract_owners_on_a_skewed_library():
    b = np.fromfile(os.path.join(GOLDEN, "polya_k27", "reads.lib.bin"), np.uint32)
    n, counts = owner_check(b, 27, 2, False, seed=1)
    assert n > 0 and counts.sum() == n


# ------------------------------------------------------------------------------------------------
# 2. the reference's fixtures
# ------------------------------------------------------------------------------------------------
FIXTURES = ["synvar_k21_m3", "synvar_k31_m1", "toy_k21", "syn150_k27", "lowcov_k21", "tandem_k27"]


def _gold(name):
    g = json.load(open(os.path.join(GOLDEN, name, "golden.json")))
    return g["m"], {int(k): v for k, v in g["by_k"].items()}


def check_gold(p, gold, n):
    d = GC.count_digest(p)
    if gold["n_solid"]:
        assert d["edges"] == gold["edges_sha256"]
    assert d["cand"] == gold["cand_sha256"] and d["counting"] == gold["counting_sha256"]
    assert d["sdbg"] == gold["sdbg_sha256"] and d["items"] == gold["sdbg_items"] and d["tips"] == gold["sdbg_tips"]
    assert F.parse_edges_info(p).num_files == n and F.parse_sdbg_info(p).num_files == n


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("n", [2, 3])
def test_fixtures(name, n, tmp_path):
    m, by_k = _gold(name)
    for k, gold in by_k.items():
        p = str(tmp_path / f"k{k}")
        r = _run(_count_cmd(os.path.join(GOLDEN, name, "reads.lib"), p, k, m, gpus=n))
        assert f"{n} GPUs" in r.stderr and "running on one GPU" not in r.stderr
        assert "Total number of solid edges" in r.stderr
        check_gold(p, gold, n)
        assert "nothing to do" in _run(_mercy_cmd(p, k)).stderr


# ------------------------------------------------------------------------------------------------
# 3. forced rounds
# ------------------------------------------------------------------------------------------------
def _with_cap(libp, p, k, m, n, cap, ok=True):
    """lib.count_run(gpus=n) in a fresh process that set the round cap first (no CUDA in it: the workers are forked)"""
    tag = uuid.uuid4().hex
    code = (f"# {tag}\nimport sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\n"
            f"lib.set_round_limit({cap})\nlib.count_run({libp!r}, {p!r}, k={k}, m={m}, gpus={n})\n")
    pr = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    out, err = pr.communicate()
    r = subprocess.CompletedProcess(pr.args, pr.returncode, out, err)
    if ok:
        assert r.returncode == 0, r.stderr[-3000:]
    return r, tag, pr.pid


def _rounds(stderr):
    m = re.search(r"count plan: (\d+) round", stderr)
    assert m, stderr[-2000:]
    return int(m.group(1))


def _owner_loads(libp, k, n):
    """(records of the largest owner, largest leading byte, largest bucket) of a library split over n owners"""
    b = np.fromfile(libp + ".bin", np.uint32)
    rec = _records(b, _n_reads(b), k)
    h = np.bincount((rec[:, 0] >> np.uint32(16)).astype(np.int64), minlength=65536).astype(np.uint64)
    plan = lib.plan_count_owner_rounds(np.vstack([h[None, :], np.zeros((n - 1, 65536), np.uint64)]))
    most = max(int(h[a:c + 1].sum()) for a, c in plan["owners"])
    return most, int(h.reshape(256, 256).sum(axis=1).max()), int(h.max())


@pytest.mark.parametrize("name", ["syn150_k27", "synvar_k21_m3", "lowcov_k21"])
@pytest.mark.parametrize("n", [2, 3])
def test_forced_rounds(name, n, tmp_path):
    m, by_k = _gold(name)
    k, gold = next(iter(by_k.items()))
    libp = os.path.join(GOLDEN, name, "reads.lib")
    most, top_byte, top_bucket = _owner_loads(libp, k, n)
    caps = [max(most // 3, top_bucket), max(most // 7, top_bucket)]
    if name == "syn150_k27":
        assert top_bucket < top_byte
        caps.append((top_bucket + top_byte) // 2)  # below the largest leading byte: cut on bucket ids
    for cap in caps:
        p = str(tmp_path / f"c{cap}")
        r, _, _ = _with_cap(libp, p, k, m, n, cap)
        assert _rounds(r.stderr) > 1 or cap >= most
        check_gold(p, gold, n)


def test_a_bucket_above_the_cap_is_refused(tmp_path):
    m, by_k = _gold("polya_k27")
    libp = os.path.join(GOLDEN, "polya_k27", "reads.lib")
    _, _, top_bucket = _owner_loads(libp, 27, 2)
    r, tag, pid = _with_cap(libp, str(tmp_path / "p"), 27, m, 2, top_bucket - 1, ok=False)
    assert r.returncode != 0
    assert "libmhb error 4" in r.stderr and "bucket 0x0000" in r.stderr and re.search(r"rank \d", r.stderr), r.stderr
    left = []
    for c in glob.glob("/proc/[0-9]*/cmdline"):
        try:
            if tag.encode() in open(c, "rb").read():
                left.append(c)
        except OSError:
            pass
    assert not left
    assert not glob.glob(f"/dev/shm/mhb_{pid}.*")


# ------------------------------------------------------------------------------------------------
# 4. a seeded 1 M-read variable-length library
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("big")
    n = 1_000_000
    b, bases = synth.synth_reads_trimmed(n, 300, genome_len=3_000_000, err=0.01, seed=11)
    p = str(d / "reads.lib")
    F.write_lib(p, b, n, bases, 300)
    return p, n


def _digest(p):
    return GC.count_digest(p)


@pytest.fixture(scope="module")
def big_single(big_lib, tmp_path_factory):
    libp, _ = big_lib
    p = str(tmp_path_factory.mktemp("one") / "one")
    _run(_count_cmd(libp, p, 27, 2))
    _run(_mercy_cmd(p, 27))
    return _digest(p)


@pytest.mark.parametrize("n", [2, 3])
def test_one_million_reads(big_lib, big_single, n, tmp_path):
    libp, _ = big_lib
    p = str(tmp_path / "res")
    r = _run(_count_cmd(libp, p, 27, 2, gpus=n))
    assert f"{n} GPUs" in r.stderr and _rounds(r.stderr) == 1
    assert _digest(p) == big_single
    most, _, top_bucket = _owner_loads(libp, 27, n)
    p = str(tmp_path / "rounds")
    r, _, _ = _with_cap(libp, p, 27, 2, n, max(most // 4, top_bucket))
    assert _rounds(r.stderr) > 1
    assert _digest(p) == big_single
    assert F.parse_edges_info(p).num_files == n and F.parse_sdbg_info(p).num_files == n


ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95",
       "--cleaning_rounds", "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2",
       "--bubble_level", "2", "--max_tip_len", "-1", "--careful_bubble"]  # src/megahit:866-899 with its defaults


@pytest.mark.skipif(not os.path.exists(REF), reason="the reference binary is not built")
def test_one_million_reads_against_the_reference(big_lib, big_single, tmp_path):
    libp, _ = big_lib
    pr = str(tmp_path / "ref")
    _run(_count_cmd(libp, pr, 27, 2, core=REF))
    _run(_mercy_cmd(pr, 27, core=REF))
    assert _digest(pr) == big_single
    p = str(tmp_path / "multi")
    _run(_count_cmd(libp, p, 27, 2, gpus=2))
    contigs = []
    for g in (pr, p):
        cp = g + "_asm"
        _run([REF, "assemble", "-s", g, "-o", cp, "-t", "1"] + ASM)  # one thread: contig ids in a fixed order
        contigs.append(open(cp + ".contigs.fa", "rb").read())
    assert contigs[0] == contigs[1] and len(contigs[0]) > 0


# ------------------------------------------------------------------------------------------------
# 5. edge cases
# ------------------------------------------------------------------------------------------------
def _against_one_gpu(b, n_reads, k, m, n, tmp_path, tag):
    libp = str(tmp_path / f"{tag}.lib")
    lens, pos = [], 0
    while pos < len(b):
        lens.append(int(b[pos]))
        pos += 1 + (lens[-1] + 15) // 16
    F.write_lib(libp, b, n_reads, sum(lens), max(lens))
    one = str(tmp_path / f"{tag}_one")
    _run(_count_cmd(libp, one, k, m))
    _run(_mercy_cmd(one, k))
    p = str(tmp_path / f"{tag}_n")
    r = _run(_count_cmd(libp, p, k, m, gpus=n))
    assert f"{n} GPUs" in r.stderr and "running on one GPU" not in r.stderr
    assert _digest(p) == _digest(one)
    assert F.parse_edges_info(p).num_files == n
    return r


@pytest.mark.parametrize("n", [2, 3])
def test_exactly_n_reads(n, tmp_path):
    b = synth.synth_reads_varlen(n, 60, 400, genome_len=2000, seed=n)
    _against_one_gpu(b, n, 21, 1, n, tmp_path, "exact")


def test_a_share_without_records_or_candidates(tmp_path):
    # one 2000-base read, then 100 reads of 20 bases (< k + 1): the shares balance on bases, so the second rank gets
    # only reads without a (k+1)-mer - no record, no mark, no candidate
    long_read = synth.synth_reads_varlen(1, 2000, 2000, genome_len=4000, seed=3)
    short = synth.synth_reads_varlen(100, 20, 20, genome_len=4000, seed=4)
    b = np.concatenate([long_read, short])
    first = lib.plan_read_shares(b, 101, 2)
    assert first[1] >= 1
    r = _against_one_gpu(b, 101, 21, 1, 2, tmp_path, "empty")
    assert re.search(r"rank 1: \d+ reads, 0 records sent", r.stderr), r.stderr[-2000:]


def test_fewer_reads_than_gpus(tmp_path):
    b = synth.synth_reads_varlen(2, 100, 200, genome_len=2000, seed=5)
    libp = str(tmp_path / "two.lib")
    F.write_lib(libp, b, 2, 400, 200)
    r = _run(_count_cmd(libp, str(tmp_path / "o"), 21, 1, gpus=3))
    assert "2 reads for 3 GPUs: running on one GPU" in r.stderr
