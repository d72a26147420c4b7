"""GPU tests of seq2sdbg and its mercy search on inputs kept in host memory: the sequences go through the device in
chunks that end on sequence boundaries, the sorted edges of the mercy search in leading-byte segments
(mhb_set_s2s_chunk_limit forces both).  The reference's digests (tests/golden/, tests/golden_cli/cli.json), the
oracle's GenMercyEdges and the resident call are the yardsticks; the stream statistics show that the input really was
streamed, in as many passes as the plan implies.
"""
import json
import os
from contextlib import contextmanager

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, golden_cases
from megahit_b200 import formats as F
from megahit_b200 import lib
from oracle import gen_golden_cli as GC

pytestmark = pytest.mark.gpu

CLI = json.load(open(os.path.join(ROOT, "tests", "golden_cli", "cli.json")))


@contextmanager
def caps(chunk=0, rounds=0):
    lib.set_s2s_chunk_limit(chunk)
    lib.set_s2s_round_limit(rounds)
    try:
        yield
    finally:
        lib.set_s2s_chunk_limit(0)
        lib.set_s2s_round_limit(0)


def _oracle():
    import oracle_pipeline as OP
    from oracle import oracle as O
    return OP, O


_inputs = {}


def case_inputs(name, k, m):
    """solid edges (GPU count, checked against the reference elsewhere), the `.cand` image and the resident mercy edges"""
    if (name, k) not in _inputs:
        OP, _ = _oracle()
        case = os.path.join(GOLDEN, name)
        reads = OP.load_reads(case)
        bin_words = np.fromfile(os.path.join(case, "reads.lib.bin"), np.uint32)
        _, n_reads = F.read_lib_info(os.path.join(case, "reads.lib"))
        c = lib.count_host(bin_words, n_reads, k, m, want_mercy=True)
        cand = np.frombuffer(reads.bin_bytes(c["cand_ids"]), np.uint32)
        mercy = lib.mercy_host(k, c["edges"], cand) if k >= 12 else np.zeros((0, c["words_per_edge"]), np.uint32)
        _inputs[(name, k)] = (c["edges"], cand, mercy)
    return _inputs[(name, k)]


def seqs_of(edges, mercy, k):
    _, O = _oracle()
    seqs, mult = O.edges_as_seqs(np.concatenate([edges, mercy]).reshape(-1, edges.shape[1]), k)
    return seqs, mult


def s2s(seqs, mult, k, chunk=0, rounds=0):
    with caps(chunk, rounds):
        g = lib.s2s_host(seqs.words, seqs.word_off, seqs.len, mult, k)
        return g, lib.s2s_stream_stats()


def assert_same_sdbg(g, one):
    assert g["bytes"] == one["bytes"] and g["n_items"] == one["n_items"]
    assert (g["bucket_table"] == one["bucket_table"]).all()
    assert (g["w_count"] == one["w_count"]).all() and g["ones_in_last"] == one["ones_in_last"]
    assert g["n_tips"] == one["n_tips"] and g["n_large_mul"] == one["n_large_mul"]


def assert_gold(g, gold):
    assert g["n_items"] == gold["sdbg_items"] and g["n_tips"] == gold["sdbg_tips"]
    assert g["n_large_mul"] == gold["sdbg_large_mul"]
    assert F.sha256(lib.sdbg_stream_from_table(g["bucket_table"], g["bytes"])) == gold["sdbg_sha256"]


def bytes_per_pass(seqs, n_chunks, fixed):
    n, nw = len(seqs.len), int(seqs.word_off[-1]) if len(seqs.len) else 0
    return 4 * nw + (2 * n if fixed else 16 * (n + n_chunks) + 6 * n)


def is_fixed(seqs, k):
    L = np.asarray(seqs.len)
    return len(L) > 0 and (L == L[0]).all() and L[0] >= k + 1 and \
        (np.asarray(seqs.word_off[:-1]) == np.arange(len(L)) * ((int(L[0]) + 15) // 16)).all()


def check_stats(st, seqs, k, cap, extra_pass=(0,)):
    n = len(seqs.len)
    plan = lib.plan_seq_chunks(seqs.word_off, seqs.len, k, cap)
    assert st["n_chunks"] == len(plan) - 1
    if n == 0:
        assert st["n_passes"] == 0 and st["h2d_bytes"] == 0
        return
    assert st["n_passes"] - 1 - st["n_rounds"] in extra_pass, st
    assert st["h2d_bytes"] == st["n_passes"] * bytes_per_pass(seqs, st["n_chunks"], is_fixed(seqs, k))


# ------------------------------------------------------------------------------------------------
# seq2sdbg over streamed sequences
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", ["fifth", "one_seq"])
@pytest.mark.parametrize("name,k,m,gold", golden_cases())
def test_streamed_s2s_matches_reference(name, k, m, gold, cap):
    """every golden case's edges + mercy edges through mhb_s2s_host in ~5 chunks and one sequence per chunk"""
    edges, _, mercy = case_inputs(name, k, m)
    seqs, mult = seqs_of(edges, mercy, k)
    one, st0 = s2s(seqs, mult, k)
    assert st0["n_chunks"] == 0 and st0["n_passes"] == 0 and st0["n_rounds"] == 1
    assert_gold(one, gold)
    image = bytes_per_pass(seqs, 0, True)
    n = len(seqs.len)
    c = max(image // 5, 1) if cap == "fifth" else (1 if n <= 20000 else image // 20000)
    g, st = s2s(seqs, mult, k, chunk=c)
    assert_gold(g, gold)
    assert_same_sdbg(g, one)
    check_stats(st, seqs, k, c)
    if n:
        assert st["n_rounds"] == 1 and st["n_passes"] == 2
        assert st["n_chunks"] >= min(n, 5 if cap == "fifth" else 20000)
    if cap == "one_seq" and n <= 20000:
        assert st["n_chunks"] == n


@pytest.mark.parametrize("name", ["chain_toy", "chain_syn150"])
@pytest.mark.parametrize("cap", [1, 4096])
def test_streamed_variable_length_chain(name, cap, tmp_path):
    """k = 29 from contigs, bubbles, addi and local contigs plus iterate edges: variable-length chunks, through the
    sub-command and through mhb_s2s_host against the resident call"""
    OP, _ = _oracle()
    case = os.path.join(GOLDEN, name)
    g = json.load(open(os.path.join(case, "chain.json")))
    k, kf = g["k"], g["k_from"]
    seqs, mult = OP.load_chain_seqs(case, k, kf)
    assert not is_fixed(seqs, k)
    one, _ = s2s(seqs, mult, k)
    got, st = s2s(seqs, mult, k, chunk=cap)
    assert_same_sdbg(got, one)
    check_stats(st, seqs, k, cap)
    assert st["n_chunks"] > 1
    if cap == 1:
        assert st["n_chunks"] == len(seqs.len)
    p = str(tmp_path / str(k))
    with caps(cap):
        lib.seq2sdbg_run(p, k=k, k_from=kf, input_prefix=os.path.join(case, str(k)),
                         contig=os.path.join(case, f"k{kf}.contigs.fa"), bubble=os.path.join(case, f"k{kf}.bubble_seq.fa"),
                         addi_contig=os.path.join(case, f"k{kf}.addi.fa"), local_contig=os.path.join(case, f"k{kf}.local.fa"),
                         need_mercy=False, host_mem=1e9, num_cpu_threads=2)
        assert lib.s2s_stream_stats()["n_chunks"] > 1
    info, stream, table = F.canonical_sdbg(p)
    assert int(table[:, 0].sum()) == g["sdbg_items"] and int(table[:, 1].sum()) == g["sdbg_tips"]
    assert F.sha256(stream) == g["sdbg_sha256"]


@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("polya_k27", 27), ("toy_k21", 21), ("synvar_k21_m3", 21)])
def test_streamed_s2s_in_rounds(name, k):
    """streaming combined with round caps of about 2 and about 8 rounds; a leading byte above the cap is cut on its
    second byte (one more pass), a single bucket above the cap is reported, never mis-sorted"""
    gold_case = [c for c in golden_cases() if c.id == f"{name}-k{k}"][0]
    m, gold = gold_case.values[2], gold_case.values[3]
    edges, _, mercy = case_inputs(name, k, m)
    seqs, mult = seqs_of(edges, mercy, k)
    one, _ = s2s(seqs, mult, k)
    n_items = int(one["n_records"])
    cap = max(bytes_per_pass(seqs, 0, True) // 7, 1)
    ran = 0
    for div, lo_rounds in ((1.6, 2), (8, 8)):
        try:
            g, st = s2s(seqs, mult, k, chunk=cap, rounds=int(n_items / div) + 1)
        except lib.MhbError as e:  # poly-A: one bucket may hold more than a round
            assert "alone holds" in str(e) and name == "polya_k27"
            continue
        ran += 1
        assert st["n_rounds"] >= lo_rounds
        assert_gold(g, gold)
        assert_same_sdbg(g, one)
        check_stats(st, seqs, k, cap, extra_pass=(0, 1))
    # a cap of ~1/300 of the items lies below the larger leading bytes but above every bucket of random data: those
    # bytes are cut on their second byte, which takes one more pass
    try:
        g, st = s2s(seqs, mult, k, chunk=cap, rounds=max(1, n_items // 300))
    except lib.MhbError as e:
        assert "alone holds" in str(e) and name != "syn150_k27"
    else:
        assert st["n_passes"] == 2 + st["n_rounds"]
        assert_same_sdbg(g, one)
    with pytest.raises(lib.MhbError, match="alone holds"):
        s2s(seqs, mult, k, chunk=cap, rounds=1)
    assert ran == 2 or name == "polya_k27"


def test_resident_s2s_leaves_read_stream_stats_alone():
    edges, cand, mercy = case_inputs("toy_k21", 21, 2)
    seqs, mult = seqs_of(edges, mercy, 21)
    lib.set_read_chunk_limit(4096)
    try:
        bin_words = np.fromfile(os.path.join(GOLDEN, "toy_k21", "reads.lib.bin"), np.uint32)
        _, n_reads = F.read_lib_info(os.path.join(GOLDEN, "toy_k21", "reads.lib"))
        lib.count_host(bin_words, n_reads, 21, 2)
    finally:
        lib.set_read_chunk_limit(0)
    before = lib.read_stream_stats()
    assert before["n_chunks"] > 1
    _, st = s2s(seqs, mult, 21)
    assert st["n_chunks"] == 0
    s2s(seqs, mult, 21, chunk=4096)
    with caps(4096):
        lib.mercy_host(21, edges, cand)
    after = lib.read_stream_stats()
    assert {k: before[k] for k in ("n_chunks", "n_passes", "h2d_bytes")} == {k: after[k] for k in ("n_chunks", "n_passes", "h2d_bytes")}


# ------------------------------------------------------------------------------------------------
# the mercy search over streamed edge segments
# ------------------------------------------------------------------------------------------------
def _bare_kmers(a, k, bare=False):
    a = np.ascontiguousarray(a, np.uint32).reshape(len(a), -1).copy()
    wm = (k + 1 + 15) // 16
    if not bare:
        assert ((a[:, -1] & 0xFFFF) == 1).all()
        a[:, -1] &= np.uint32(0xFFFF0000)
        assert (a[:, wm:] == 0).all()
    return sorted(map(bytes, np.ascontiguousarray(a[:, :wm])))


def byte_bytes(edges):
    return np.bincount(edges[:, 0] >> 24, minlength=256) * edges.shape[1] * 4


def equal_bytes(edges):
    """the first n edges of every leading byte that has at least n (n = the lower quartile of the non-empty bytes): a
    sorted edge array whose non-empty bytes all take the same bytes, so that a cap of one byte's size plans one
    segment per non-empty byte"""
    top = edges[:, 0] >> 24
    cnt = np.bincount(top, minlength=256)
    n = max(1, int(np.percentile(cnt[cnt > 0], 25)))
    rank = np.arange(len(edges)) - np.searchsorted(top, top)
    return edges[(cnt[top] >= n) & (rank < n)], n


@pytest.mark.parametrize("plan", ["one", "three", "per_byte"])
@pytest.mark.parametrize("name,k,m", [("syn150_k27", 27, 2), ("toy_k21", 21, 2), ("lowcov_k21", 21, 2)])
def test_streamed_mercy_matches_resident_and_oracle(name, k, m, plan):
    OP, O = _oracle()
    edges, cand, resident = case_inputs(name, k, m)
    if plan == "per_byte":
        edges, n = equal_bytes(edges)
        resident = lib.mercy_host(k, edges, cand)
    bb = byte_bytes(edges)
    cap = {"one": int(bb.sum()), "three": max(int(bb.sum()) // 3, int(bb.max())), "per_byte": int(bb.max())}[plan]
    segs = lib.plan_mercy_segments(edges, k, cap)
    if plan == "per_byte":  # one segment per non-empty byte
        nz = np.nonzero(bb)[0]
        assert segs == [0] + nz[1:].tolist() + [256]
    assert segs[0] == 0 and segs[-1] == 256 and all(a < b for a, b in zip(segs, segs[1:]))
    with caps(cap):
        got = lib.mercy_host(k, edges, cand)
        st = lib.s2s_stream_stats(mercy=True)
    n_cand = len(cand) > 0
    if n_cand:
        assert st["n_chunks"] == len(segs) - 1 and st["n_passes"] == 1
        assert st["h2d_bytes"] == edges.nbytes
        if plan == "one":
            assert st["n_chunks"] == 1
        elif plan == "three":
            assert st["n_chunks"] >= 3
        else:
            assert st["n_chunks"] == int((bb > 0).sum()) > 8
    exp = O.gen_mercy(edges, O.unpack_bin(cand.tobytes(), reverse=False), k)
    assert len(got) == len(resident) == len(exp)
    if len(exp):
        assert _bare_kmers(got, k) == _bare_kmers(resident, k) == _bare_kmers(np.asarray(exp, np.uint32), k, bare=True)
    lib.mercy_host(k, edges, cand)
    assert lib.s2s_stream_stats(mercy=True)["n_chunks"] == 0


def test_streamed_mercy_oversized_byte_is_reported():
    edges, cand, _ = case_inputs("syn150_k27", 27, 2)
    bb = byte_bytes(edges)
    big = int(np.argmax(bb))
    with pytest.raises(lib.MhbError, match="leading byte 0x%02x alone holds" % big):
        lib.plan_mercy_segments(edges, 27, int(bb.max()) - 1)
    with caps(int(bb.max()) - 1), pytest.raises(lib.MhbError, match="leading byte 0x%02x alone holds" % big):
        lib.mercy_host(27, edges, cand)


# ------------------------------------------------------------------------------------------------
# the staged build and the sub-commands
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("toy_k21", 21), ("lowcov_k21", 21), ("syn150_klist", 59)])
def test_staged_build_with_every_cap(name, k):
    gold_case = [c for c in golden_cases() if c.id == f"{name}-k{k}"][0]
    m, gold = gold_case.values[2], gold_case.values[3]
    bin_words = np.fromfile(os.path.join(GOLDEN, name, "reads.lib.bin"), np.uint32)
    _, n_reads = F.read_lib_info(os.path.join(GOLDEN, name, "reads.lib"))
    one = lib.build_host(bin_words, n_reads, k, m, need_mercy=True)
    lib.set_read_chunk_limit(max(4, len(bin_words) // 2))
    lib.set_round_limit(max(1, int(one["n_edge_records"]) // 3))
    try:
        with caps(max(1, 12 * int(one["n_solid"]) // 3), max(1, int(one["n_solid"] + one["n_mercy"]) * 6 // 3)):
            try:
                g = lib.build_host(bin_words, n_reads, k, m, need_mercy=True, want_edges=True)
            except lib.MhbError as e:  # a single bucket or leading byte above a cap is reported, never mis-sorted
                # on a uniform random genome no byte or bucket comes near a third of the edges
                assert "alone holds" in str(e) and name not in ("syn150_k27", "syn150_klist")
                return
            st, ms = lib.s2s_stream_stats(), lib.s2s_stream_stats(mercy=True)
    finally:
        lib.set_read_chunk_limit(0)
        lib.set_round_limit(0)
    assert st["n_chunks"] > 1 and st["n_rounds"] > 1
    assert ms["n_chunks"] >= 1 or one["n_cand"] == 0
    assert g["n_solid"] == gold["n_solid"] and g["n_mercy"] == one["n_mercy"]
    assert F.sha256(g["edges"].tobytes()) == gold["edges_sha256"]
    assert_gold(g, gold)


def test_cli_seq2sdbg_streamed_at_1m_reads(tmp_path):
    """1 M x 150 bp reads: `count`, then `seq2sdbg --need_mercy` with sequences and mercy edges streamed in 8 MiB
    chunks / segments: the reference binary's digests"""
    libp, _, _ = GC.count_lib(tmp_path)
    p = str(tmp_path / "streamed")
    lib.count_run(libp, p, k=27, m=2, host_mem=3e10, num_cpu_threads=8)
    with caps(8 << 20):
        lib.seq2sdbg_run(p, k=27, input_prefix=p, need_mercy=True, host_mem=3e10, num_cpu_threads=8)
        st, ms = lib.s2s_stream_stats(), lib.s2s_stream_stats(mercy=True)
    assert st["n_chunks"] > 1 and st["n_passes"] == 1 + st["n_rounds"]
    assert ms["n_chunks"] > 1 and ms["n_passes"] == 1
    assert GC.count_digest(p) == CLI["count_1m"]
