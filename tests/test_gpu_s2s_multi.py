"""seq2sdbg on several GPUs (`megahit_core seq2sdbg --gpus N`, mhb_seq2sdbg_run_multi) and the multi-GPU CLI on
however many devices there are (ranks share a device when N exceeds the device count):

* the owner sink of the item extraction (mhb_s2s_extract_owners) against mhb_s2s_extract, at every record width class;
* k > k_min parity with the reference's multi-k run (tests/golden/chain_*), and with the single-GPU seq2sdbg at wide k;
* routing: --need_mercy runs on one GPU unless the multi-GPU count left its graph;
* `count --gpus 2` against the reference's digests, and the reference's `assemble` on an N-file SdBG.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
OURS = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")
CHAIN = ["chain_syn150", "chain_toy"]


def _run(cmd, env=None):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, (cmd, r.stderr[-3000:])
    return r


# ------------------------------------------------------------------------------------------------
# 1. the owner sink
# ------------------------------------------------------------------------------------------------
def _items(length, k):
    length = np.asarray(length, np.int64)
    return np.where(length >= k + 1, 2 * (length - k + 2), 0)


def _synthetic(k, n, seed):
    """n random sequences, some of them shorter than k + 1 (no items)"""
    rng = np.random.default_rng(seed)
    length = rng.integers(max(1, k - 10), k + 400, size=n).astype(np.uint32)
    nw = (length.astype(np.int64) + 15) // 16
    word_off = np.concatenate([[0], np.cumsum(nw)]).astype(np.uint64)
    words = rng.integers(0, 1 << 32, size=max(int(word_off[-1]), 1), dtype=np.uint64).astype(np.uint32)
    for i, L in enumerate(length):  # clean tails, as the loader leaves them
        if L % 16:
            w = int(word_off[i]) + int(nw[i]) - 1
            words[w] &= np.uint32((0xFFFFFFFF << (32 - 2 * int(L % 16))) & 0xFFFFFFFF)
    mult = rng.integers(1, 300, size=n).astype(np.uint16)
    return words, word_off, length, mult


def _chain(name):
    import oracle_pipeline as OP
    case = os.path.join(GOLDEN, name)
    g = json.load(open(os.path.join(case, "chain.json")))
    seqs, mult = OP.load_chain_seqs(case, g["k"], g["k_from"])
    return g["k"], seqs.words, seqs.word_off, seqs.len, mult


def _sorted_rows(a, W):
    a = np.ascontiguousarray(a.reshape(-1, W))
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def owner_sink_check(words, word_off, length, mult, k, n_owners, seed):
    import torch
    dv = torch.device("cuda")
    L = lib.load()
    W = lib.s2s_record_words(k)
    n = len(length)
    item_off = np.concatenate([[0], np.cumsum(_items(length, k))]).astype(np.uint64)
    n_items = int(item_off[-1])

    def dev(a, dtype):
        a = np.ascontiguousarray(a) if len(a) else np.zeros(8, a.dtype)
        return torch.from_numpy(a.view(dtype)).to(dv)

    keep = [dev(np.concatenate([words, np.zeros(16, np.uint32)]), np.int32), dev(word_off, np.int64), dev(item_off, np.int64),
            dev(length, np.int32), dev(mult, np.int16)]
    seqs = lib.DevSeqs(keep[0].data_ptr(), len(words), n, 0, keep[1].data_ptr(), keep[3].data_ptr(), keep[2].data_ptr(),
                       keep[4].data_ptr(), 0)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ref = torch.zeros(n_items * W + 8, dtype=torch.int32, device=dv)
    lib._check(L.mhb_s2s_extract(st, C.byref(seqs), k, C.c_void_p(ref.data_ptr()), n_items, None, 0))
    torch.cuda.synchronize()
    ref_h = ref.cpu().numpy().view(np.uint32)[: n_items * W].reshape(-1, W)

    # the owner of every leading byte; the last owner receives nothing
    rng = np.random.default_rng(seed)
    lut = rng.integers(0, max(n_owners - 1, 1), size=256).astype(np.uint8)
    lead = ref_h[:, 0] >> np.uint32(24)
    counts = np.bincount(lut[lead], minlength=n_owners)[:n_owners] if n_items else np.zeros(n_owners, np.int64)
    assert n_owners < 2 or counts[-1] == 0
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    gap = 3  # guard records between the slices, which must stay untouched
    buf = torch.full((int(off[-1] + gap * n_owners) * W + 8,), -7, dtype=torch.int32, device=dv)
    base = np.array([buf.data_ptr() + 4 * W * int(off[o] + gap * o) for o in range(n_owners)], np.uint64)
    d_lut = torch.from_numpy(lut.view(np.int8)).to(dv)
    d_base = torch.from_numpy(base.view(np.int64)).to(dv)
    d_cursor = torch.zeros(n_owners, dtype=torch.int64, device=dv)
    d_cap = torch.from_numpy(counts.astype(np.int64)).to(dv)
    lib._check(L.mhb_s2s_extract_owners(st, C.byref(seqs), k, n_items, C.c_void_p(d_lut.data_ptr()),
                                        C.c_void_p(d_base.data_ptr()), C.c_void_p(d_cursor.data_ptr()),
                                        C.c_void_p(d_cap.data_ptr())))
    torch.cuda.synchronize()
    assert (d_cursor.cpu().numpy() == counts).all()
    out = buf.cpu().numpy().view(np.uint32)
    for o in range(n_owners):
        s = (int(off[o]) + gap * o) * W
        got = out[s: s + int(counts[o]) * W]
        want = ref_h[lut[lead] == o] if n_items else ref_h[:0]
        assert np.array_equal(_sorted_rows(got, W), _sorted_rows(want, W)), f"owner {o}"
        assert (out[s + int(counts[o]) * W: s + (int(counts[o]) + gap) * W] == np.uint32(0xFFFFFFF9)).all(), f"guard {o}"
    return n_items


@pytest.mark.parametrize("name", CHAIN)
@pytest.mark.parametrize("n_owners", [2, 4])
def test_owner_sink_on_chain_inputs(name, n_owners):
    k, words, word_off, length, mult = _chain(name)
    assert owner_sink_check(words, word_off, length, mult, k, n_owners, seed=n_owners) > 0


@pytest.mark.parametrize("k", [21, 59, 141, 227])
@pytest.mark.parametrize("n_owners", [1, 3, 5])
def test_owner_sink_synthetic(k, n_owners):
    words, word_off, length, mult = _synthetic(k, 3000, seed=k + n_owners)
    assert (length < k + 1).any()
    assert owner_sink_check(words, word_off, length, mult, k, n_owners, seed=k) > 0


def test_owner_sink_empty_set():
    k = 27
    e = np.zeros(0, np.uint32)
    assert owner_sink_check(e, np.zeros(1, np.uint64), e, np.zeros(0, np.uint16), k, 3, seed=1) == 0


# ------------------------------------------------------------------------------------------------
# 2. k > k_min: the reference's multi-k run
# ------------------------------------------------------------------------------------------------
def _s2s_cmd(p, k, kf=0, input_prefix=None, contig=None, bubble=None, addi=None, local=None, mercy=False, gpus=None):
    cmd = [OURS, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p, "--num_cpu_threads", "4",
           "-k", str(k), "--kmer_from", str(kf)]
    for opt, v in (("--input_prefix", input_prefix), ("--contig", contig), ("--bubble", bubble), ("--addi_contig", addi),
                   ("--local_contig", local)):
        if v:
            cmd += [opt, v]
    if mercy:
        cmd.append("--need_mercy")
    if gpus:
        cmd += ["--gpus", str(gpus)]
    return cmd


def _chain_cmd(name, p, gpus):
    case = os.path.join(GOLDEN, name)
    g = json.load(open(os.path.join(case, "chain.json")))
    k, kf = g["k"], g["k_from"]
    return g, _s2s_cmd(p, k, kf, os.path.join(case, str(k)), os.path.join(case, f"k{kf}.contigs.fa"),
                       os.path.join(case, f"k{kf}.bubble_seq.fa"), os.path.join(case, f"k{kf}.addi.fa"),
                       os.path.join(case, f"k{kf}.local.fa"), gpus=gpus)


def check_ranks(p, n):
    """num_files == n; every `.sdbg.<r>` holds an ascending run of buckets, the runs of the ranks follow each other and
    no bucket is on two ranks; the files hold exactly the bytes the records describe"""
    info = F.parse_sdbg_info(p)
    assert info.num_files == n
    recs = info.records[info.records[:, 0] != np.uint64(F.NULL_ID)].astype(np.int64)
    assert len(np.unique(recs[:, 0])) == len(recs)
    prev_hi = -1
    for r in range(n):
        mine = recs[recs[:, 1] == r]
        size = os.path.getsize(f"{p}.sdbg.{r}")
        if not len(mine):
            assert size == 0
            continue
        assert (np.diff(mine[:, 0]) > 0).all() and (np.diff(mine[:, 2]) > 0).all()
        assert mine[0, 0] > prev_hi
        prev_hi = mine[-1, 0]
        nbytes = 2 * mine[:, 3] + 2 * mine[:, 5] + 4 * info.words_per_tip_label * mine[:, 4]
        assert mine[0, 2] == 0 and (mine[1:, 2] == np.cumsum(nbytes)[:-1]).all() and size == nbytes.sum()


def check_chain(p, g):
    info, stream, table = F.canonical_sdbg(p)
    assert info.k == g["sdbg_k"] and info.words_per_tip_label == g["sdbg_words_per_tip_label"]
    assert int(table[:, 0].sum()) == g["sdbg_items"] and int(table[:, 1].sum()) == g["sdbg_tips"]
    assert int(table[:, 2].sum()) == g["sdbg_large_mul"]
    assert F.sha256(stream) == g["sdbg_sha256"]


@pytest.mark.parametrize("name", CHAIN)
@pytest.mark.parametrize("n", [2, 3])
def test_seq2sdbg_gpus_on_chain_inputs(name, n, tmp_path):
    p = str(tmp_path / "multi")
    g, cmd = _chain_cmd(name, p, n)
    r = _run(cmd)
    assert f"{n} GPUs" in r.stderr
    check_chain(p, g)
    check_ranks(p, n)


def test_seq2sdbg_gpus_from_the_environment(tmp_path):
    p = str(tmp_path / "env")
    g, cmd = _chain_cmd("chain_syn150", p, None)
    r = _run(cmd, env=dict(os.environ, MHB_GPUS="2"))
    assert "2 GPUs" in r.stderr
    check_chain(p, g)
    check_ranks(p, 2)


# ------------------------------------------------------------------------------------------------
# 3. wide k: the single-GPU seq2sdbg on the same files
# ------------------------------------------------------------------------------------------------
def _write_contigs(path, k, n, seed):
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, size=60000)
    with open(path, "w") as f:
        for i in range(n):
            L = int(rng.integers(k + 1, k + 600))
            s = int(rng.integers(0, len(genome) - L))
            seq = "".join("ACGT"[b] for b in genome[s:s + L])
            f.write(f">k{k}_{i} flag=0 multi={rng.uniform(1, 400):.4f} len={L}\n{seq}\n")


@pytest.mark.parametrize("k", [141, 227])
def test_wide_k_matches_one_gpu(k, tmp_path):
    contigs = str(tmp_path / "c.fa")
    _write_contigs(contigs, k, 400, seed=k)
    one = str(tmp_path / "one")
    _run(_s2s_cmd(one, k, contig=contigs))
    _, s1, t1 = F.canonical_sdbg(one)
    assert len(s1) > 0
    for n in (2, 3):
        p = str(tmp_path / f"n{n}")
        _run(_s2s_cmd(p, k, contig=contigs, gpus=n))
        _, sn, tn = F.canonical_sdbg(p)
        assert sn == s1 and np.array_equal(tn, t1)
        check_ranks(p, n)


# ------------------------------------------------------------------------------------------------
# 4. routing of --need_mercy
# ------------------------------------------------------------------------------------------------
def _count_cmd(libp, p, k, m, gpus=None):
    cmd = [OURS, "count", "-k", str(k), "-m", str(m), "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", p,
           "--num_cpu_threads", "4", "--read_lib_file", libp]
    return cmd + (["--gpus", str(gpus)] if gpus else [])


def test_need_mercy_runs_on_one_gpu(tmp_path):
    gold_all = json.load(open(os.path.join(GOLDEN, "syn150_k27", "golden.json")))
    k = 27
    m, gold = gold_all["m"], gold_all["by_k"][str(k)]
    p = str(tmp_path / "one")
    _run(_count_cmd(os.path.join(GOLDEN, "syn150_k27", "reads.lib"), p, k, m))
    r = _run(_s2s_cmd(p, k, input_prefix=p, mercy=True, gpus=2))
    assert "runs on one GPU" in r.stderr and "nothing to do" not in r.stderr
    d = GC.count_digest(p)
    assert d["sdbg"] == gold["sdbg_sha256"] and d["items"] == gold["sdbg_items"] and d["tips"] == gold["sdbg_tips"]
    assert F.parse_sdbg_info(p).num_files == 1


def test_need_mercy_after_multi_gpu_count_has_nothing_to_do(tmp_path):
    k, m = 27, json.load(open(os.path.join(GOLDEN, "syn150_k27", "golden.json")))["m"]
    p = str(tmp_path / "multi")
    _run(_count_cmd(os.path.join(GOLDEN, "syn150_k27", "reads.lib"), p, k, m, gpus=2))
    r = _run(_s2s_cmd(p, k, input_prefix=p, mercy=True, gpus=2))
    assert "nothing to do" in r.stderr


# ------------------------------------------------------------------------------------------------
# 5. + 6. `count --gpus 2` on the available devices; the reference's assemble on N-file graphs
# ------------------------------------------------------------------------------------------------
ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95",
       "--cleaning_rounds", "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2",
       "--bubble_level", "2", "--max_tip_len", "-1", "--careful_bubble"]  # src/megahit:866-899 with its defaults


@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("syn150_klist", 59), ("lowcov_k21", 21), ("polya_k27", 27)])
def test_count_gpus_2_on_available_devices(name, k, tmp_path):
    gold_all = json.load(open(os.path.join(GOLDEN, name, "golden.json")))
    m, gold = gold_all["m"], gold_all["by_k"][str(k)]
    p = str(tmp_path / "multi")
    r = _run(_count_cmd(os.path.join(GOLDEN, name, "reads.lib"), p, k, m, gpus=2))
    assert "2 GPUs" in r.stderr
    r2 = _run(_s2s_cmd(p, k, input_prefix=p, mercy=True))
    assert "nothing to do" in r2.stderr
    d = GC.count_digest(p)
    assert F.parse_edges_info(p).num_files == 2 and F.parse_sdbg_info(p).num_files == 2
    if gold["n_solid"]:
        assert d["edges"] == gold["edges_sha256"]
    assert d["cand"] == gold["cand_sha256"] and d["counting"] == gold["counting_sha256"]
    assert d["sdbg"] == gold["sdbg_sha256"] and d["items"] == gold["sdbg_items"] and d["tips"] == gold["sdbg_tips"]


@pytest.mark.skipif(not os.path.exists(REF), reason="the reference binary is not built")
@pytest.mark.parametrize("name", CHAIN)
def test_reference_assembles_the_two_file_graph(name, tmp_path):
    outs = []
    for n in (1, 2):
        p = str(tmp_path / f"g{n}")
        _run(_chain_cmd(name, p, n if n > 1 else None)[1])
        assert F.parse_sdbg_info(p).num_files == n
        cp = str(tmp_path / f"contigs{n}")
        _run([REF, "assemble", "-s", p, "-o", cp, "-t", "1"] + ASM)
        outs.append(open(cp + ".contigs.fa", "rb").read())
    assert outs[0] == outs[1] and len(outs[0]) > 0
