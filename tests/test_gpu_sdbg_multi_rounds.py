"""The SdBG stage on several GPUs in rounds over bucket ranges (`megahit_core seq2sdbg --gpus N` and the k_min graph of
`count --gpus N`): every owner takes its bucket range of the sort items in rounds when the range does not fit its
device at once, or exceeds the mhb_set_s2s_round_limit cap.

* the kernels: the 65536-bin bucket histograms of the items of sequences (mhb_s2s_bucket_hist) and of pruned edges
  (mhb_s2s_edges_owners with a histogram) against the extraction they plan, and the range-restricted owner stores
  (mhb_s2s_extract_owners_round, mhb_s2s_edges_owners) against the reference rows filtered by owner and range;
* `seq2sdbg --gpus N` with caps: the reference's digests of the chain inputs and the single-GPU stream and bytes;
* `count --gpus N` with an SdBG cap, alone and with a count cap: the reference's digests;
* a cap below the largest bucket is refused before any receive buffer exists, and nothing is left behind.

The rounds are forced with lib.set_s2s_round_limit in a fresh process that then runs the stage on N GPUs (the forked
workers inherit the cap).  The caps come from the loads rank 0 logs on an uncapped run.  Ranks share a device when N
exceeds the device count, so all of it runs on one GPU."""
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
from megahit_b200 import lib
from test_gpu_count_multi import _MODE, _count_cmd, _gold, _owner_loads, big_lib, big_single, check_gold  # noqa: F401
from test_gpu_count_multi import _digest as count_digest
from test_gpu_s2s_multi import CHAIN, _chain_cmd, _s2s_cmd, _write_contigs, check_chain, check_ranks

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_MODE is not None, reason=f"the device's compute mode ({_MODE}) admits one process only")]

KS = [21, 59, 141, 227]


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, (cmd, r.stderr[-3000:])
    return r


# ------------------------------------------------------------------------------------------------
# 1. the kernels
# ------------------------------------------------------------------------------------------------
def _random_seqs(k, n, seed, polya=False):
    """n sequences, some shorter than k + 1; polya: most of them poly-A with a few other bases"""
    rng = np.random.default_rng(seed)
    length = rng.integers(max(1, k - 10), k + 300, size=n).astype(np.uint32)
    bases = [rng.integers(0, 4, size=int(L)).astype(np.uint8) for L in length]
    if polya:
        for b in bases[: n * 3 // 4]:
            b[rng.random(len(b)) < 0.97] = 0
    nw = (length.astype(np.int64) + 15) // 16
    word_off = np.concatenate([[0], np.cumsum(nw)]).astype(np.uint64)
    words = np.zeros(max(int(word_off[-1]), 1), np.uint32)
    for i, b in enumerate(bases):
        pad = np.zeros(int(nw[i]) * 16, np.uint8)
        pad[: len(b)] = b
        w = pad.reshape(-1, 16).astype(np.uint32) << (30 - 2 * np.arange(16, dtype=np.uint32))
        words[int(word_off[i]): int(word_off[i + 1])] = np.bitwise_or.reduce(w, axis=1)
    mult = rng.integers(1, 300, size=n).astype(np.uint16)
    return words, word_off, length, mult


def _random_edges(k, n, seed, polya=False):
    """n `.edges` records of k: (k+1)-mers left-aligned in words_per_edge(k) words, multiplicity in the low 16 bits"""
    rng = np.random.default_rng(seed)
    WE = lib.words_per_edge(k)
    b = rng.integers(0, 4, size=(n, WE * 16)).astype(np.uint32)
    if polya:
        b[: n * 3 // 4][rng.random((n * 3 // 4, WE * 16)) < 0.97] = 0
    b[:, k + 1:] = 0
    rec = np.bitwise_or.reduce(b.reshape(n, WE, 16) << (30 - 2 * np.arange(16, dtype=np.uint32)), axis=2)
    rec = rec.astype(np.uint32).reshape(n, WE)
    rec[:, -1] |= rng.integers(1, 300, size=n).astype(np.uint32)
    return rec


class Dev:
    """device copies of numpy arrays, kept alive with the object"""

    def __init__(self):
        import torch
        self.torch = torch
        self.keep = []

    def __call__(self, a, pad=16):
        t = self.torch.from_numpy(np.concatenate([np.ascontiguousarray(a).ravel().view(np.uint8),
                                                  np.zeros(pad * 4, np.uint8)]).view(np.int8)).cuda()
        self.keep.append(t)
        return t.data_ptr()

    def zeros(self, nbytes, fill=0):
        t = self.torch.full((nbytes,), fill, dtype=self.torch.int8, device="cuda")
        self.keep.append(t)
        return t

    def stream(self):
        return C.c_void_p(self.torch.cuda.current_stream().cuda_stream)


def _seqs_view(d, words, word_off, length, mult, k):
    items = np.where(length >= k + 1, 2 * (length.astype(np.int64) - k + 2), 0)
    item_off = np.concatenate([[0], np.cumsum(items)]).astype(np.uint64)
    seqs = lib.DevSeqs(d(words), len(words), len(length), 0, d(word_off), d(length), d(item_off), d(mult), 0)
    return seqs, int(item_off[-1])


def _extract_ref(d, seqs, k, n_items):
    """the rows of mhb_s2s_extract"""
    W = lib.s2s_record_words(k)
    out = d.zeros(max(n_items, 1) * W * 4 + 64)
    lib._check(lib.load().mhb_s2s_extract(d.stream(), C.byref(seqs), k, C.c_void_p(out.data_ptr()), n_items, None, 0))
    d.torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32)[: n_items * W].reshape(-1, W)


def _pruned_ref(d, edges, aux, n_aux, k):
    """the rows of mhb_s2s_extract_edges_pruned"""
    W, n = lib.s2s_record_words(k), len(edges)
    out, cur = d.zeros(max(6 * n, 1) * W * 4 + 64), d.zeros(64)
    lib._check(lib.load().mhb_s2s_extract_edges_pruned(d.stream(), C.c_void_p(d(edges)), C.c_void_p(d(aux)), n, n_aux, k,
                                                       C.c_void_p(out.data_ptr()), 6 * n, C.c_void_p(cur.data_ptr()),
                                                       None, 0))
    d.torch.cuda.synchronize()
    kept = int(cur.cpu().numpy().view(np.uint64)[0])
    return out.cpu().numpy().view(np.uint32)[: kept * W].reshape(-1, W)


def _hist(ref):
    return np.bincount((ref[:, 0] >> np.uint32(16)).astype(np.int64), minlength=65536)


def _edge_input(k, n, seed, polya):
    rng = np.random.default_rng(seed + 1)
    edges = _random_edges(k, n, seed, polya) if n else np.zeros((0, lib.words_per_edge(k)), np.uint32)
    aux = rng.integers(0, 4, size=max(n, 1)).astype(np.uint8)
    return edges, aux, n * 2 // 3  # the last third without flags, as the mercy edges behind the solid ones


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("case", ["random", "polya", "empty"])
def test_bucket_histograms(k, case):
    n = 0 if case == "empty" else 2000
    polya = case == "polya"
    d = Dev()
    L = lib.load()
    words, word_off, length, mult = _random_seqs(k, n, seed=k, polya=polya)
    seqs, n_items = _seqs_view(d, words, word_off, length, mult, k)
    h = d.zeros(65536 * 8)
    lib._check(L.mhb_s2s_bucket_hist(d.stream(), C.byref(seqs), k, n_items, C.c_void_p(h.data_ptr())))
    d.torch.cuda.synchronize()
    got = h.cpu().numpy().view(np.uint64)
    want = _hist(_extract_ref(d, seqs, k, n_items))
    assert (got == want).all() and int(got.sum()) == n_items
    if polya:
        assert want.max() > n_items // 10  # skewed: one bucket holds a tenth of the items

    edges, aux, n_aux = _edge_input(k, n, seed=k, polya=polya)
    h = d.zeros(65536 * 8)
    lib._check(L.mhb_s2s_edges_owners(d.stream(), C.c_void_p(d(edges)), C.c_void_p(d(aux)), n, n_aux, k,
                                      C.c_void_p(h.data_ptr()), None, None, None, None, None, None))
    d.torch.cuda.synchronize()
    ref = _pruned_ref(d, edges, aux, n_aux, k)
    assert (h.cpu().numpy().view(np.uint64) == _hist(ref)).all()
    assert n == 0 or 2 * n < len(ref) < 6 * n  # some items pruned, some kept


def _owner_round_check(d, ref, store, k, n_owners, seed):
    """store(lut, base, cursor, cap, lo, hi) against the rows of ref filtered by owner and range; guard rows between the
    owners' segments stay untouched"""
    W = lib.s2s_record_words(k)
    rng = np.random.default_rng(seed)
    lut = np.sort(rng.integers(0, n_owners, size=256)).astype(np.uint8)  # contiguous leading-byte ranges
    b = (ref[:, 0] >> np.uint32(16)).astype(np.int64)
    lo = np.zeros(n_owners, np.uint32)
    hi = np.zeros(n_owners, np.uint32)
    for o in range(n_owners):
        mine = np.nonzero(lut == o)[0]
        if o == n_owners - 1 or not len(mine):  # an empty range: nothing goes to this owner
            lo[o], hi[o] = 1, 0
            continue
        a, c = int(mine[0]) << 8, (int(mine[-1]) << 8) | 255
        x = sorted(int(v) for v in rng.integers(a, c + 1, size=2))
        lo[o], hi[o] = x[0], x[1]
    owner = lut[b >> 8]
    take = (b >= lo[owner]) & (b <= hi[owner])
    counts = np.bincount(owner[take], minlength=n_owners).astype(np.int64)
    gap = 3
    off = np.concatenate([[0], np.cumsum(counts + gap)]).astype(np.int64)
    buf = d.zeros(int(off[-1]) * W * 4 + 64, fill=-7)
    base = np.array([buf.data_ptr() + 4 * W * int(off[o]) for o in range(n_owners)], np.uint64)
    cursor = d.zeros(8 * n_owners)
    store(d(lut), d(base), cursor.data_ptr(), d(counts), d(lo), d(hi))
    d.torch.cuda.synchronize()
    assert (cursor.cpu().numpy().view(np.int64) == counts).all()
    out = buf.cpu().numpy().view(np.uint32)
    for o in range(n_owners):
        s = int(off[o]) * W
        got = out[s: s + int(counts[o]) * W].reshape(-1, W)
        want = ref[take & (owner == o)]
        srt = lambda a: a[np.lexsort(a.T[::-1])] if len(a) else a  # noqa: E731
        assert np.array_equal(srt(got), srt(want)), f"owner {o}"
        assert (out[s + int(counts[o]) * W: s + int(counts[o] + gap) * W] == np.uint32(0xF9F9F9F9)).all(), f"guard {o}"
    return int(counts.sum())


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n_owners", [1, 3, 5])
@pytest.mark.parametrize("case", ["random", "polya", "empty"])
def test_owner_stores_in_a_round(k, n_owners, case):
    n = 0 if case == "empty" else 1500
    d = Dev()
    L = lib.load()
    st = d.stream()
    words, word_off, length, mult = _random_seqs(k, n, seed=k + n_owners, polya=case == "polya")
    seqs, n_items = _seqs_view(d, words, word_off, length, mult, k)

    def seq_store(lut, base, cursor, cap, lo, hi):
        lib._check(L.mhb_s2s_extract_owners_round(st, C.byref(seqs), k, n_items, *(C.c_void_p(p) for p in
                                                                                    (lut, base, cursor, cap, lo, hi))))

    sent = _owner_round_check(d, _extract_ref(d, seqs, k, n_items), seq_store, k, n_owners, seed=k)
    assert sent > 0 or n == 0 or n_owners == 1 or case == "polya"

    edges, aux, n_aux = _edge_input(k, n, seed=k + n_owners, polya=case == "polya")
    d_edges, d_aux = d(edges), d(aux)

    def edge_store(lut, base, cursor, cap, lo, hi):
        lib._check(L.mhb_s2s_edges_owners(st, C.c_void_p(d_edges), C.c_void_p(d_aux), n, n_aux, k, None,
                                          *(C.c_void_p(p) for p in (lut, base, cursor, cap, lo, hi))))

    sent = _owner_round_check(d, _pruned_ref(d, edges, aux, n_aux, k), edge_store, k, n_owners, seed=k + 1)
    assert sent > 0 or n == 0 or n_owners == 1 or case == "polya"


# ------------------------------------------------------------------------------------------------
# 2. rounds forced by a cap, in a fresh process
# ------------------------------------------------------------------------------------------------
def _loads(stderr):
    """(largest owner, largest leading byte, largest bucket) of the SdBG items, as rank 0 logs them"""
    m = re.search(r"SdBG items: largest owner (\d+), largest leading byte (\d+), largest bucket (\d+)", stderr)
    assert m, stderr[-2000:]
    return tuple(int(x) for x in m.groups())


def _rounds(stderr):
    m = re.search(r"SdBG plan: (\d+) rounds? over bucket ranges", stderr)
    assert m, stderr[-2000:]
    return int(m.group(1))


def _caps(loads):
    """the largest owner's load / 3 and / 7, floored at the largest bucket, and one cap below the largest leading byte
    when that byte holds more than one bucket's items"""
    most, top_byte, top_bucket = loads
    caps = [max(most // 3, top_bucket), max(most // 7, top_bucket)]
    if top_bucket < top_byte:
        caps.append((top_bucket + top_byte) // 2)
    return caps


def _in_fresh_process(calls, ok=True):
    """the lib calls (source lines) in one fresh process (no CUDA in it: the workers are forked); each run's log follows
    its '@@run <prefix>' line"""
    tag = uuid.uuid4().hex
    code = f"# {tag}\nimport sys\nsys.path.insert(0, {ROOT!r})\nfrom megahit_b200 import lib\n" + "".join(calls)
    pr = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    out, err = pr.communicate()
    r = subprocess.CompletedProcess(pr.args, pr.returncode, out, err)
    if ok:
        assert r.returncode == 0, r.stderr[-3000:]
    logs = dict(re.findall(r"@@run (\S+)\n(.*?)(?=@@run |\Z)", err, re.S))
    return r, tag, pr.pid, logs


def _run_line(p, cap, call, count_cap=0):
    return (f"print('@@run {p}', file=sys.stderr, flush=True)\nlib.set_s2s_round_limit({cap})\n"
            f"lib.set_round_limit({count_cap})\n{call}\n")


def _seq2sdbg_call(p, n, k, k_from=0, input_prefix="", contig="", bubble="", addi="", local=""):
    return (f"lib.seq2sdbg_run({p!r}, {k}, {k_from}, input_prefix={input_prefix!r}, contig={contig!r}, bubble={bubble!r}, "
            f"addi_contig={addi!r}, local_contig={local!r}, gpus={n})")


def _single_gpu(cmd_one):
    """(canonical stream, raw bytes) of the single-GPU seq2sdbg"""
    p = cmd_one[cmd_one.index("--output_prefix") + 1]
    _run(cmd_one)
    assert F.parse_sdbg_info(p).num_files == 1
    return F.canonical_sdbg(p)[1], open(p + ".sdbg.0", "rb").read()


def _check_against_one_gpu(p, n, one):
    stream, raw = one
    assert F.canonical_sdbg(p)[1] == stream, "not the single-GPU stream"
    # an owner's rounds follow each other in bucket order: the ranks' files joined are the single-GPU bytes
    assert b"".join(open(f"{p}.sdbg.{i}", "rb").read() for i in range(n)) == raw
    check_ranks(p, n)


def _chain_args(name):
    case = os.path.join(GOLDEN, name)
    g = json.load(open(os.path.join(case, "chain.json")))
    k, kf = g["k"], g["k_from"]
    return g, dict(k=k, k_from=kf, input_prefix=os.path.join(case, str(k)), contig=os.path.join(case, f"k{kf}.contigs.fa"),
                   bubble=os.path.join(case, f"k{kf}.bubble_seq.fa"), addi=os.path.join(case, f"k{kf}.addi.fa"),
                   local=os.path.join(case, f"k{kf}.local.fa"))


@pytest.mark.parametrize("name", CHAIN)
@pytest.mark.parametrize("n", [2, 3])
def test_seq2sdbg_chain_in_rounds(name, n, tmp_path):
    g, a = _chain_args(name)
    one = _single_gpu(_chain_cmd(name, str(tmp_path / "one"), None)[1])
    p0 = str(tmp_path / "plain")
    r = _run(_chain_cmd(name, p0, n)[1])
    assert _rounds(r.stderr) == 1  # everything fits: one round
    check_chain(p0, g)
    _check_against_one_gpu(p0, n, one)
    loads = _loads(r.stderr)
    caps = _caps(loads)
    runs = [(str(tmp_path / f"c{i}"), c) for i, c in enumerate(caps)]
    _, _, _, logs = _in_fresh_process([_run_line(p, c, _seq2sdbg_call(p, n, **a)) for p, c in runs])
    for p, c in runs:
        assert _rounds(logs[p]) > 1, (c, loads)
        check_chain(p, g)
        _check_against_one_gpu(p, n, one)


@pytest.mark.parametrize("k", [141, 227])
def test_seq2sdbg_wide_k_in_rounds(k, tmp_path):
    contigs = str(tmp_path / "c.fa")
    _write_contigs(contigs, k, 400, seed=k)
    one = _single_gpu(_s2s_cmd(str(tmp_path / "one"), k, contig=contigs))
    for n in (2, 3):
        r = _run(_s2s_cmd(str(tmp_path / f"plain{n}"), k, contig=contigs, gpus=n))
        assert _rounds(r.stderr) == 1
        runs = [(str(tmp_path / f"n{n}c{i}"), c) for i, c in enumerate(_caps(_loads(r.stderr)))]
        _, _, _, logs = _in_fresh_process([_run_line(p, c, _seq2sdbg_call(p, n, k, contig=contigs)) for p, c in runs])
        for p, c in runs:
            assert _rounds(logs[p]) > 1
            _check_against_one_gpu(p, n, one)


COUNT_CASES = ["syn150_k27", "lowcov_k21", "polya_k27", "synvar_k21_m3"]


@pytest.mark.parametrize("name", COUNT_CASES)
@pytest.mark.parametrize("n", [2, 3])
def test_count_sdbg_in_rounds(name, n, tmp_path):
    m, by_k = _gold(name)
    k, gold = next(iter(by_k.items()))
    libp = os.path.join(GOLDEN, name, "reads.lib")
    r = _run(_count_cmd(libp, str(tmp_path / "plain"), k, m, gpus=n))
    assert _rounds(r.stderr) == 1
    loads = _loads(r.stderr)
    cap3, cap7 = _caps(loads)[:2]
    most, _, top_bucket = _owner_loads(libp, k, n)
    count_cap = max(most // 3, top_bucket)  # the count records in rounds too
    runs = [(str(tmp_path / "s3"), cap3, 0), (str(tmp_path / "s7"), cap7, 0), (str(tmp_path / "both"), cap7, count_cap)]
    call = "lib.count_run({libp!r}, {p!r}, k={k}, m={m}, gpus={n})"
    _, _, _, logs = _in_fresh_process([_run_line(p, c, call.format(libp=libp, p=p, k=k, m=m, n=n), cc)
                                       for p, c, cc in runs])
    for p, c, cc in runs:
        assert _rounds(logs[p]) > 1 or c >= loads[0], (c, loads)
        if cc:
            assert int(re.search(r"count plan: (\d+) round", logs[p]).group(1)) > 1 or count_cap >= most
        check_gold(p, gold, n)


@pytest.mark.parametrize("n", [2, 3])
def test_one_million_reads_in_sdbg_rounds(big_lib, big_single, n, tmp_path):
    libp, _ = big_lib
    r = _run(_count_cmd(libp, str(tmp_path / "plain"), 27, 2, gpus=n))
    loads = _loads(r.stderr)
    p = str(tmp_path / "rounds")
    _, _, _, logs = _in_fresh_process([_run_line(p, max(loads[0] // 4, loads[2]),
                                                 f"lib.count_run({libp!r}, {p!r}, k=27, m=2, gpus={n})")])
    assert _rounds(logs[p]) > 1
    assert count_digest(p) == big_single
    assert F.parse_sdbg_info(p).num_files == n


# ------------------------------------------------------------------------------------------------
# 3. a cap below the largest bucket
# ------------------------------------------------------------------------------------------------
def _left_behind(tag, pid):
    left = []
    for c in glob.glob("/proc/[0-9]*/cmdline"):
        try:
            if tag.encode() in open(c, "rb").read():
                left.append(c)
        except OSError:
            pass
    return left, glob.glob(f"/dev/shm/mhb_{pid}.*")


def _refused(r):
    assert r.returncode != 0
    assert "libmhb error 4" in r.stderr and re.search(r"bucket 0x[0-9a-f]{4} alone holds \d+ records", r.stderr), \
        r.stderr[-2000:]
    assert re.search(r"rank \d", r.stderr), r.stderr[-2000:]


def test_seq2sdbg_cap_below_a_bucket_is_refused(tmp_path):
    _, a = _chain_args("chain_syn150")
    r = _run(_chain_cmd("chain_syn150", str(tmp_path / "plain"), 2)[1])
    p = str(tmp_path / "p")
    r, tag, pid, _ = _in_fresh_process([_run_line(p, _loads(r.stderr)[2] - 1, _seq2sdbg_call(p, 2, **a))], ok=False)
    _refused(r)
    assert _left_behind(tag, pid) == ([], [])


def test_count_sdbg_cap_below_a_bucket_is_refused(tmp_path):
    m, _ = _gold("syn150_k27")
    libp = os.path.join(GOLDEN, "syn150_k27", "reads.lib")
    r = _run(_count_cmd(libp, str(tmp_path / "plain"), 27, m, gpus=2))
    top_bucket = _loads(r.stderr)[2]
    assert top_bucket > 1
    p = str(tmp_path / "p")
    r, tag, pid, _ = _in_fresh_process([_run_line(p, top_bucket - 1,
                                                  f"lib.count_run({libp!r}, {p!r}, k=27, m={m}, gpus=2)")], ok=False)
    _refused(r)
    assert _left_behind(tag, pid) == ([], [])
