"""mhb_build_host is one chain: count -> mercy edges -> seq2sdbg.  A stage that runs in one pass over resident data
hands its result to the next on the device, any other stage through host memory.  Every combination of hand-offs must
give the one-pass build's outputs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, golden_cases
from megahit_b200 import formats as F
from megahit_b200 import lib, synth

pytestmark = pytest.mark.gpu

_SAME = ("n_edge_records", "n_solid", "n_cand", "n_mercy", "n_items", "n_tips", "n_large_mul", "n_bytes",
         "words_per_tip_label", "ones_in_last")


def _load(name):
    bin_words = np.fromfile(os.path.join(GOLDEN, name, "reads.lib.bin"), np.uint32)
    _, n_reads = F.read_lib_info(os.path.join(GOLDEN, name, "reads.lib"))
    return bin_words, n_reads


def _gold(name, k):
    return [c for c in golden_cases() if c.id == f"{name}-k{k}"][0].values[2:]


def _assert_same(g, one):
    """every output of g equals the one-pass build's; g's seq2sdbg ran from host memory or in rounds, so it sorted all
    six items per edge where the one-pass build skips the ones the count's flags rule out"""
    for f in _SAME:
        assert g[f] == one[f], f
    assert g["bytes"] == one["bytes"]
    assert (g["bucket_table"] == one["bucket_table"]).all() and (g["w_count"] == one["w_count"]).all()
    assert (g["edges"] == one["edges"]).all() and (g["cand_ids"] == one["cand_ids"]).all()
    assert (g["counting"] == one["counting"]).all()
    assert g["n_sort_items"] == 6 * (int(g["n_solid"]) + int(g["n_mercy"]))


def _build(bin_words, n_reads, k, m, need_mercy=True, round_limit=0, s2s_round_limit=0, chunk_limit=0):
    lib.set_round_limit(round_limit)
    lib.set_s2s_round_limit(s2s_round_limit)
    lib.set_read_chunk_limit(chunk_limit)
    try:
        return lib.build_host(bin_words, n_reads, k, m, need_mercy=need_mercy, want_edges=True)
    finally:
        lib.set_round_limit(0)
        lib.set_s2s_round_limit(0)
        lib.set_read_chunk_limit(0)


@pytest.mark.parametrize("name,k", [("syn150_k27", 27), ("synvar_k21_m3", 21), ("lowcov_k21", 21), ("empty_k21", 21)])
def test_hand_offs_match_the_one_pass_build(name, k):
    """count in one pass + seq2sdbg in rounds; count in rounds + seq2sdbg in one pass from host memory; a streamed
    library; on a fixed-length, a variable-length, a low-coverage (mercy edges beyond the solid-edge capacity) and an
    empty library"""
    m, gold = _gold(name, k)
    bin_words, n_reads = _load(name)
    one = _build(bin_words, n_reads, k, m)
    assert F.sha256(lib.sdbg_stream_from_table(one["bucket_table"], one["bytes"])) == gold["sdbg_sha256"]
    if gold["n_solid"]:
        assert F.sha256(one["edges"].tobytes()) == gold["edges_sha256"]
    n_seqs = int(one["n_solid"] + one["n_mercy"])
    assert one["n_sort_items"] <= 6 * n_seqs
    # seq2sdbg in rounds over the edges the count left on the device (downloaded once)
    _assert_same(_build(bin_words, n_reads, k, m, s2s_round_limit=max(1, 6 * n_seqs // 4)), one)
    # the count in rounds, mercy edges and seq2sdbg from host memory
    _assert_same(_build(bin_words, n_reads, k, m, round_limit=max(1, int(one["n_edge_records"]) // 4)), one)
    # the library streamed through the device in chunks
    _assert_same(_build(bin_words, n_reads, k, m, chunk_limit=max(4, len(bin_words))), one)
    if name == "lowcov_k21":  # more mercy edges than the count's edge buffer holds behind the solid ones
        assert one["n_mercy"] > int(one["n_edge_records"]) // m + 1 - int(one["n_solid"])


def test_library_without_candidates():
    """reads tiling a circular genome without errors: no tip edges, so no candidate reads and no mercy edges"""
    rng = np.random.default_rng(11)
    L, G = 150, 1500
    genome = rng.integers(0, 4, size=G, dtype=np.uint8)
    ring = np.concatenate([genome, genome[: L - 1]])
    b = F.pack_reads_fixed(np.stack([ring[s: s + L] for s in range(G)] * 2))
    one = _build(b.reshape(-1), len(b), 27, 2)
    assert one["n_cand"] == 0 and one["n_mercy"] == 0 and one["n_solid"] > 0
    _assert_same(_build(b.reshape(-1), len(b), 27, 2, round_limit=max(1, int(one["n_edge_records"]) // 3)), one)


@pytest.mark.parametrize("k", [9, 10, 11, 127])
def test_small_and_wide_k(k):
    """k = 9 .. 11 (no mercy edges below 12) and a wide k: the device chain against the host hand-offs.  At k = 9 and 11
    the one-pass build's SdBG differs from the full extraction's (test_pruned_sdbg_differs_at_k_9_and_11); there the
    count's outputs are compared with the one-pass build, and the SdBG between the two host hand-offs."""
    b = synth.synth_reads(2000, 150, 10000, 0.01, seed=5)
    need_mercy = k >= 12
    one = _build(b.reshape(-1), len(b), k, 2, need_mercy=need_mercy)
    assert one["n_solid"] > 0
    rounds = _build(b.reshape(-1), len(b), k, 2, need_mercy=need_mercy, round_limit=max(1, int(one["n_edge_records"]) // 3))
    s2s_rounds = _build(b.reshape(-1), len(b), k, 2, need_mercy=need_mercy,
                        s2s_round_limit=max(1, 6 * int(one["n_solid"] + one["n_mercy"]) // 3))
    _assert_same(s2s_rounds, rounds)
    if k in (9, 11):
        assert (rounds["edges"] == one["edges"]).all() and (rounds["counting"] == one["counting"]).all()
        assert rounds["n_edge_records"] == one["n_edge_records"] and rounds["n_mercy"] == one["n_mercy"] == 0
    else:
        _assert_same(rounds, one)


_CHILD = r"""
import json, os, sys
import numpy as np
sys.path.insert(0, %r)
from megahit_b200 import formats as F, lib
name, k, m, need_mercy = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4] == "1"
bin_words = np.fromfile(os.path.join(name, "reads.lib.bin"), np.uint32)
_, n_reads = F.read_lib_info(os.path.join(name, "reads.lib"))
g = lib.build_host(bin_words, n_reads, k, m, need_mercy=need_mercy, want_edges=True)
print("RESULT " + json.dumps(%s))
""" % (ROOT, "{f: (F.sha256(np.ascontiguousarray(v).tobytes()) if isinstance(v, (np.ndarray, bytes)) else int(v)) "
              "for f, v in g.items() if f != 'ms'}")


def _digest(g):
    """the child's digest of a build_host result"""
    return {f: (F.sha256(np.ascontiguousarray(v).tobytes()) if isinstance(v, (np.ndarray, bytes)) else int(v))
            for f, v in g.items() if f != "ms"}


def _child(env_name, value, name="syn150_k27", k=27, m=2, need_mercy=True):
    env = dict(os.environ)
    env.pop("MHB_S2S_NO_PRUNE", None)
    env.pop("MHB_H2D_CHUNKS", None)
    if value is not None:
        env[env_name] = value
    p = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(GOLDEN, name), str(k), str(m), str(int(need_mercy))], env=env,
                       capture_output=True, text=True, timeout=300)
    line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
    assert line, p.stderr[-800:]
    return json.loads(line[-1][7:])


def test_no_prune_and_single_upload_match_the_default():
    """MHB_S2S_NO_PRUNE=1 (all six items per edge) and MHB_H2D_CHUNKS=1 (the library in one copy) against the
    default build: same outputs; only the pruned build sorts fewer items"""
    base = _child("MHB_H2D_CHUNKS", None)
    no_prune = _child("MHB_S2S_NO_PRUNE", "1")
    one_copy = _child("MHB_H2D_CHUNKS", "1")
    assert one_copy == base
    assert no_prune["n_sort_items"] == 6 * (no_prune["n_solid"] + no_prune["n_mercy"]) > base["n_sort_items"]
    assert {f: v for f, v in no_prune.items() if f != "n_sort_items"} == {f: v for f, v in base.items() if f != "n_sort_items"}


@pytest.mark.parametrize("k", [9, 11])
def test_pruned_sdbg_differs_at_k_9_and_11(k, tmp_path):
    """A known difference, not made by the chain (DESIGN.md section 4.7): at k = 9 and 11 the one-pass build's pruned
    extraction gives a different SdBG from the full extraction of the host hand-offs, on a library where k = 10 and
    the wider k give the same.  MHB_S2S_NO_PRUNE=1 gives the full extraction's outputs on the one-pass path."""
    b = synth.synth_reads(2000, 150, 10000, 0.01, seed=5)
    F.write_lib(str(tmp_path / "reads.lib"), b, len(b), len(b) * 150, 150)
    full = _build(b.reshape(-1), len(b), k, 2, need_mercy=False, round_limit=len(b) * (150 - k) // 3)
    pruned = _child("MHB_S2S_NO_PRUNE", None, str(tmp_path), k, 2, need_mercy=False)
    no_prune = _child("MHB_S2S_NO_PRUNE", "1", str(tmp_path), k, 2, need_mercy=False)
    assert no_prune == _digest(full)
    assert pruned["edges"] == no_prune["edges"] and pruned["counting"] == no_prune["counting"]
    assert pruned["n_items"] != no_prune["n_items"] and pruned["bytes"] != no_prune["bytes"]
