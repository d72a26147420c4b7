"""buildlib on the GPU: mhb_buildlib_host, mhb_buildlib_run and the CLI against the reference's digests
(tests/golden_buildlib/buildlib.json), at the default chunk size and at chunk caps of a few hundred bytes; the
speculative record walk on input where every guess is wrong; pe inputs through FIFOs; a round trip of every committed
`.bin` library through FASTA; a 2 M-read FASTQ against the reference binary when oracle/_ref holds it."""
import glob
import hashlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import buildlib_cases as BC  # noqa: E402
import buildlib_reference as R  # noqa: E402
from megahit_b200 import lib  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(HERE, "golden_buildlib", "buildlib.json")))
CASES = BC.all_cases()
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
CLI = os.path.join(ROOT, "megahit_b200", "bin", "megahit_core")


def lib_info_text(libs, res):
    s = f"{res['n_bases']} {res['n_reads']}\n"
    for i, (t, _) in enumerate(libs):
        s += f"lib{i} {t}\n{res['lib_begin'][i]} {res['lib_end'][i]} {res['lib_max_len'][i]} {0 if t == 'se' else 1}\n"
    return s


def host_digests(libs):
    try:
        res = lib.buildlib_host(libs)
    except lib.MhbError:
        return {"rc": 1}
    return {"rc": 0, "bin": hashlib.sha256(res["bin"].tobytes()).hexdigest(),
            "lib_info": hashlib.sha256(lib_info_text(libs, res).encode()).hexdigest(), "res": res}


def same(got, want):
    return (got["rc"] != 0) == (want["rc"] != 0) and (want["rc"] != 0 or (got["bin"], got["lib_info"]) == (want["bin"], want["lib_info"]))


@pytest.fixture
def chunk_cap():
    yield lib.set_buildlib_chunk
    lib.set_buildlib_chunk(0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_matches_reference(name):
    assert same(host_digests(CASES[name]), GOLDEN[name])


SMALL = [c for c in sorted(CASES) if c != "gen_megabase"]


@pytest.mark.parametrize("cap", [64, 193, 500])
@pytest.mark.parametrize("name", SMALL)
def test_host_small_chunks(name, cap, chunk_cap):
    chunk_cap(cap)
    got = host_digests(CASES[name])
    assert same(got, GOLDEN[name])


def test_record_larger_than_chunk(chunk_cap):
    chunk_cap(300)
    got = host_digests(CASES["gen_megabase"])
    assert same(got, GOLDEN["gen_megabase"])


def test_every_guess_wrong_same_bytes():
    data = BC.misguided(20000)
    got = host_digests([("se", [data])])
    b, info = R.buildlib([("lib0 se", "se", [data])])
    assert got["bin"] == hashlib.sha256(b).hexdigest()
    # one chunk: the first walk plus at least one fix-up pass (a walk started from a wrong state re-synchronises
    # within its segment, so one re-walk from the predecessors' exits is usually enough)
    assert got["res"]["n_chunks"] == 1 and got["res"]["n_walk_passes"] >= 2, got["res"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_run_and_cli_match_reference(name, tmp_path):
    libs = CASES[name]
    lf = BC.write_lib(str(tmp_path), libs)
    try:
        lib.buildlib_run(lf, str(tmp_path / "api"))
        got = {"rc": 0, **BC.digests(str(tmp_path / "api"))}
    except lib.MhbError:
        got = {"rc": 1}
    assert same(got, GOLDEN[name])
    r = subprocess.run([CLI, "buildlib", lf, str(tmp_path / "cli")], capture_output=True)
    got = {"rc": r.returncode, **(BC.digests(str(tmp_path / "cli")) if r.returncode == 0 else {})}
    assert same(got, GOLDEN[name]), r.stderr.decode()[-2000:]
    if GOLDEN[name]["rc"] != 0:
        assert r.returncode == 1


def test_cli_unopenable_input(tmp_path):
    lf = tmp_path / "reads.lib"
    lf.write_text(f"m\nse {tmp_path / 'missing.fa'}\n")
    r = subprocess.run([CLI, "buildlib", str(lf), str(tmp_path / "out")], capture_output=True)
    assert r.returncode != 0 and b"FATAL" in r.stderr


@pytest.mark.parametrize("cap", [0, 4096])
def test_pe_through_fifos(tmp_path, cap, chunk_cap):
    chunk_cap(cap)
    a, b = BC.fastq(3000, 150, seed=1), BC.fastq(2000, 100, seed=3)
    fa, fb = tmp_path / "a.fifo", tmp_path / "b.fifo"
    os.mkfifo(fa)
    os.mkfifo(fb)

    def feed(path, data):
        try:
            with open(path, "wb") as f:
                for i in range(0, len(data), 65536):
                    f.write(data[i:i + 65536])
        except BrokenPipeError:  # the reader stops at the end of the shorter file
            pass

    ts = [threading.Thread(target=feed, args=(fa, a)), threading.Thread(target=feed, args=(fb, b))]
    for t in ts:
        t.start()
    lf = tmp_path / "reads.lib"
    lf.write_text(f"lib0 pe\npe {fa} {fb}\n")
    try:
        lib.buildlib_run(str(lf), str(tmp_path / "out"))
    finally:
        for p in (fa, fb):  # unblock a writer the reader stopped early on
            try:
                fd = os.open(p, os.O_RDONLY | os.O_NONBLOCK)
                while os.read(fd, 1 << 20):
                    pass
                os.close(fd)
            except OSError:
                pass
        for t in ts:
            t.join(timeout=60)
    assert not any(t.is_alive() for t in ts)
    want = GOLDEN["gen_fastq_pe_unequal"]
    assert BC.digests(str(tmp_path / "out")) == {"bin": want["bin"], "lib_info": want["lib_info"]}


def _bin_to_fasta(path):
    """FASTA of a `.bin` library, and the `.bin` buildlib writes for it: the library itself, except that a zero-length read
    (some synthetic test libraries hold them; buildlib never writes one) comes back as the one-base read "A"."""
    w = np.fromfile(path, np.uint32)
    out, want, p, i = [], [], 0, 0
    while p < len(w):
        L = int(w[p])
        nw = (L + 15) // 16
        words = w[p + 1:p + 1 + nw]
        s = bytearray()
        for q in range(L):
            s.append(b"ACGT"[(int(words[q // 16]) >> (30 - 2 * (q % 16))) & 3])
        out.append(b">r%d\n" % i + bytes(s) + b"\n")
        want.append(w[p:p + 1 + nw].tobytes() if L else R.pack_read(b""))
        p += 1 + nw
        i += 1
    return b"".join(out), b"".join(want)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(HERE, "golden*", "**", "reads.lib.bin"), recursive=True)))
def test_round_trip_committed_libraries(path):
    fasta, raw = _bin_to_fasta(path)
    res = lib.buildlib_host([("se", [fasta])])
    assert res["bin"].tobytes() == raw


@pytest.mark.skipif(not os.access(REF, os.X_OK), reason="reference binary not built")
def test_2m_reads_against_reference_binary(tmp_path):
    data = BC.fastq(2_000_000, 150, seed=99)
    lf = BC.write_lib(str(tmp_path), [("se", [data])])
    r = subprocess.run([REF, "buildlib", lf, str(tmp_path / "ref")], capture_output=True)
    assert r.returncode == 0
    lib.buildlib_run(lf, str(tmp_path / "ours"))
    assert BC.digests(str(tmp_path / "ours")) == BC.digests(str(tmp_path / "ref"))


def test_chunk_of_short_lines_many_segments():
    # 2 lines per record, 33.6 M lines in one chunk: more than 2^17 walk segments of 256 lines, so the segment scan needs
    # more block sums than the chunk's tile scan
    n = 16_800_000
    res = lib.buildlib_host([("se", [b">\nC\n" * n])])
    assert res["n_chunks"] == 1 and res["n_reads"] == n and res["n_bases"] == n and res["lib_max_len"] == [1]
    want = np.empty(2 * n, np.uint32)
    want[0::2] = 1
    want[1::2] = 1 << 30  # C = 1 in the top two bits
    assert np.array_equal(res["bin"], want)


@pytest.mark.parametrize("name", ["gen_fastq_se", "gen_fastq_pe_unequal", "gen_multi_lib", "edge_fq_short_qual_twice"])
def test_run_writes_chunk_by_chunk(name, tmp_path, chunk_cap):
    # P.bin is written as each chunk completes: many small chunks must give the same file
    chunk_cap(700)
    lf = BC.write_lib(str(tmp_path), CASES[name])
    lib.buildlib_run(lf, str(tmp_path / "out"))
    want = GOLDEN[name]
    assert BC.digests(str(tmp_path / "out")) == {"bin": want["bin"], "lib_info": want["lib_info"]}
