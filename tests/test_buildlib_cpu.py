"""buildlib without a GPU: the plain restatement (tests/buildlib_reference.py) against the reference's digests and, when
oracle/_ref holds the reference binary, against the binary itself; the device code's line walk, TrimN and packing (run
serially through the self-test hook) against the restatement; the CLI's decision to forward stdin / gzip input."""
import hashlib
import json
import os
import random
import stat
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import buildlib_cases as BC  # noqa: E402
import buildlib_reference as R  # noqa: E402

GOLDEN = json.load(open(os.path.join(HERE, "golden_buildlib", "buildlib.json")))
CASES = BC.all_cases()
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def oracle(libs):
    try:
        b, info = R.buildlib([(f"lib{i} {t}", t, d) for i, (t, d) in enumerate(libs)])
    except R.LibError:
        return {"rc": 1}
    return {"rc": 0, "bin": hashlib.sha256(b).hexdigest(), "lib_info": hashlib.sha256(info.encode()).hexdigest()}


def same(got, want):
    return (got["rc"] != 0) == (want["rc"] != 0) and (want["rc"] != 0 or (got["bin"], got["lib_info"]) == (want["bin"], want["lib_info"]))


def test_fixture_set_matches_cases():
    assert sorted(GOLDEN) == sorted(CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_digests(name):
    assert same(oracle(CASES[name]), GOLDEN[name])


@pytest.mark.skipif(not os.access(REF, os.X_OK), reason="reference binary not built")
def test_oracle_matches_live_reference_fuzz(tmp_path):
    rng = random.Random(2024)
    alpha = b"ACGTNn\n\r>@+ xacgt"
    for t in range(150):
        data = bytes(rng.choice(alpha) for _ in range(rng.randint(0, 160)))
        d = tmp_path / str(t)
        d.mkdir()
        lib = BC.write_lib(str(d), [("se", [data])])
        r = subprocess.run([REF, "buildlib", lib, str(d / "out")], capture_output=True)
        want = {"rc": r.returncode, **(BC.digests(str(d / "out")) if r.returncode == 0 else {})}
        assert same(oracle([("se", [data])]), want), data


def test_lib_file_istream_quirks():
    # whitespace splits a path; a trailing blank line re-reads the last library (the failed `>> type` keeps the old value)
    assert R.parse_lib_file("m\nse a b\n") == [("m", "se", ["a"])]
    assert R.parse_lib_file("m\npe x y\n\n") == [("m", "pe", ["x", "y"]), ("", "pe", ["x", "y"])]
    with pytest.raises(R.LibError):
        R.parse_lib_file("m\nfoo x\n")


def _selftest_matches(data):
    from megahit_b200 import lib
    recs = R.kseq_records(data)
    st = lib.selftest_fastx(data)
    want_len = [0xFFFFFFFF if r is None else len(R.trim_n(r)) for r in recs]
    want_bin = b"".join(R.pack_read(R.trim_n(r)) for r in recs if r is not None)
    return list(st["len"]) == want_len and st["bin"] == want_bin


@pytest.mark.parametrize("name", sorted(BC.edge_cases()))
def test_selftest_walk_trim_pack_edge(name):
    assert _selftest_matches(BC.edge_cases()[name])


def test_selftest_walk_trim_pack_fuzz():
    rng = random.Random(7)
    alpha = b"ACGTNn\n\r>@+ xacgtRY"
    for _ in range(3000):
        data = bytes(rng.choice(alpha) for _ in range(rng.randint(0, 200)))
        assert _selftest_matches(data), data


def test_selftest_generated():
    assert _selftest_matches(BC.wrapped_fasta(200, seed=3))
    assert _selftest_matches(BC.misguided(50))
    assert _selftest_matches(BC.fastq(200, 150, seed=4))


def _stub(tmp_path):
    stub = tmp_path / "ref_stub.sh"
    stub.write_text("#!/bin/sh\necho forwarded \"$@\" > \"$(dirname \"$0\")/forwarded.txt\"\nexit 0\n")
    stub.chmod(stub.stat().st_mode | stat.S_IXUSR)
    return stub


@pytest.mark.skipif(not os.access(CLI, os.X_OK), reason="CLI not built")
@pytest.mark.parametrize("kind", ["stdin", "gzip", "gzip_pe"])
def test_cli_forwards_stdin_and_gzip(tmp_path, kind):
    import gzip
    stub = _stub(tmp_path)
    plain = tmp_path / "a.fa"
    plain.write_bytes(b">a\nACGT\n")
    gz = tmp_path / "b.fa.gz"
    gz.write_bytes(gzip.compress(b">a\nACGT\n"))
    lib = tmp_path / "reads.lib"
    lib.write_text({"stdin": "m\nse -\n", "gzip": f"m\nse {gz}\n", "gzip_pe": f"m\npe {plain} {gz}\n"}[kind])
    env = dict(os.environ, MHB_REFERENCE_CORE=str(stub))
    r = subprocess.run([CLI, "buildlib", str(lib), str(tmp_path / "out")], capture_output=True, env=env, stdin=subprocess.DEVNULL)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "forwarded.txt").read_text().split()[:2] == ["forwarded", "buildlib"]


@pytest.mark.skipif(not os.access(CLI, os.X_OK), reason="CLI not built")
def test_cli_keeps_plain_text_and_fifo(tmp_path):
    # plain files (and a FIFO, which is not a regular file and is not opened for the check) stay on the GPU path:
    # without a GPU that path fails instead of reaching the stub
    stub = _stub(tmp_path)
    plain = tmp_path / "a.fa"
    plain.write_bytes(b"\x1f>a\nACGT\n")
    fifo = tmp_path / "p.fifo"
    os.mkfifo(fifo)
    lib = tmp_path / "reads.lib"
    lib.write_text(f"m\npe {plain} {fifo}\n")
    from megahit_b200 import lib as L
    if L.device_count() > 0:
        pytest.skip("needs a machine without a GPU (the GPU path would block on the FIFO)")
    env = dict(os.environ, MHB_REFERENCE_CORE=str(stub))
    r = subprocess.run([CLI, "buildlib", str(lib), str(tmp_path / "out")], capture_output=True, env=env, timeout=60)
    assert not (tmp_path / "forwarded.txt").exists()
    assert r.returncode == 1
