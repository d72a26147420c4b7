"""Inputs of the buildlib tests: hand-written edge cases and seeded generated files.  tests/golden_buildlib/buildlib.json
holds, per case, the sha256 of the `.bin` / `.lib_info` that the reference `megahit_core buildlib` wrote for them
(scripts/gen_golden_buildlib.py)."""
import hashlib
import os
import random

EDGE = {
    "fa_single": b">r1 x\nACGTACGT\n>r2\nGGCCAATT\n",
    "fa_wrap60": None,  # generated below
    "fa_wrap80": None,
    "fa_blank_lines": b">a\n\nACGT\n\n\nTTGG\n>b\n\n",
    "fa_header_only": b">a\n>b\nAC\n>c\n>d",
    "fa_gt_in_header": b">a>b>c\nACGT\n>x@y\nGG\n",
    "fa_junk_first": b"junk line\nmore>hdr\nACGT\n>h2\nCC\n",
    "fa_no_final_nl": b">a\nACG\n>b\nTTTA",
    "empty": b"",
    "fq_4line": b"@r1\nACGT\n+\nIIII\n@r2\nGGCC\n+r2\nHHHH\n",
    "fq_multiline": b"@r1\nACGT\nTTAA\n+\nIIII\nIIII\n@r2\nGG\nCC\n+\nI\nIII\n",
    "fq_qual_markers": b"@r1\nACGT\n+\n@III\n@r2\nACGT\n+\n+III\n@r3\nACGT\n+\n>III\n@r4\nAC\n+\nII\n",
    "fq_plus_name": b"@r1\nACGT\n+r1 comment\nIIII\n",
    "fq_short_qual": b"@r1\nACGT\n+\nIIII\n@r2\nACGT\n+\nII\n@r3\nGGGG\n+\nIIII\n",
    "fq_short_qual_twice": b"@r1\nACGT\n+\nIIII\n@r2\nACGT\n+\nII\n@r3\nGGGG\n+\nI\n@r4\nTT\n+\nII\n",
    "fq_bad_first": b"@r1\nACGT\n+\nII\n@r2\nGGGG\n+\nIIII\n",
    "fq_truncated": b"@r1\nACGT\n+\nIIII\n@r2\nACGT\n+",
    "fq_truncated_qual": b"@r1\nACGT\n+\nIIII\n@r2\nACGT\n+\nII",
    "fq_empty_seq_last": b"@r1\nAC\n+\nII\n>r2\n+",
    "mixed": b">a\nACGT\n@b\nGG\n+\nII\n>c\nTTT\nAAA\n@d\nC\n+\nI\n",
    "crlf": b">a\r\nAC\r\n\r\nGT\r\n>b\r\n\r\nAC\r\n@q\r\nACG\r\n+\r\nIII\r\n",
    "crlf_bare_cr_line": b">a\r\n\r\nACGT\r\n>b\r\nA\r\n\r\n>c\nG\n\r",
    "n_handling": b">lead\nNNACGT\n>trail\nACGTNN\n>inner\nACNNGTNA\n>alln\nNNNN\n>lower\nacgtnacgt\n>iupac\nRYKMSWacgtBDHV\n",
    "lengths": None,
}


def _wrap(seq: bytes, w: int) -> bytes:
    return b"\n".join(seq[i:i + w] for i in range(0, len(seq), w))


def _rand_seq(rng, n, alphabet=b"ACGT"):
    return bytes(rng.choice(alphabet) for _ in range(n))


def edge_cases():
    rng = random.Random(11)
    out = dict(EDGE)
    out["fa_wrap60"] = b"".join(b">s%d\n" % i + _wrap(_rand_seq(rng, 50 + 37 * i), 60) + b"\n" for i in range(8))
    out["fa_wrap80"] = b"".join(b">s%d\n" % i + _wrap(_rand_seq(rng, 70 + 53 * i), 80) + b"\n" for i in range(8))
    out["lengths"] = b"".join(b">l%d\n" % n + _rand_seq(rng, n) + b"\n" for n in (0, 1, 15, 16, 17, 31, 32, 33))
    return out


def fastq(n_reads: int, length: int, seed: int, n_rate: float = 0.01) -> bytes:
    """Seeded FASTQ of n_reads reads of `length` bases (a few N), 4 lines per record."""
    import numpy as np
    rng = np.random.default_rng(seed)
    codes = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=(n_reads, length))]
    codes[rng.random((n_reads, length)) < n_rate] = ord("N")
    lines = np.full((n_reads, length + 1), ord("\n"), np.uint8)
    lines[:, :length] = codes
    qual = np.full((n_reads, length + 1), ord("I"), np.uint8)
    qual[:, length] = ord("\n")
    hdr = [b"@r%d\n" % i for i in range(n_reads)]
    plus = b"+\n"
    seqb = lines.tobytes()
    qb = qual.tobytes()
    w = length + 1
    return b"".join(hdr[i] + seqb[i * w:(i + 1) * w] + plus + qb[i * w:(i + 1) * w] for i in range(n_reads))


def wrapped_fasta(n_reads: int, seed: int, width: int = 60, max_len: int = 400) -> bytes:
    rng = random.Random(seed)
    return b"".join(b">c%d\n" % i + _wrap(_rand_seq(rng, rng.randint(0, max_len), b"ACGTNacgtn"), width) + b"\n"
                    for i in range(n_reads))


def megabase_record(seed: int) -> bytes:
    import numpy as np
    rng = np.random.default_rng(seed)
    s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=2_100_000)].tobytes()
    return b">big\n" + _wrap(s, 70) + b"\n>after\nACGT\n"


def misguided(n: int) -> bytes:
    """FASTQ whose quality lines start with '>' and whose records have the 4-line '@' shape shifted by one line, so
    that the walk's guess at every line a segment could start on is wrong."""
    rec = b"@h\nACGTACGT\nACGTACGT\n+\n>IIIIIII\n>IIIIIII\n"
    return rec * n


def generated():
    """name -> list of (type, [bytes]) libraries"""
    fq1 = fastq(3000, 150, seed=1)
    fq2 = fastq(3000, 150, seed=2)
    return {
        "gen_fastq_se": [("se", [fq1])],
        "gen_fastq_pe": [("pe", [fq1, fq2])],
        "gen_fastq_pe_unequal": [("pe", [fq1, fastq(2000, 100, seed=3)])],
        "gen_fasta_wrapped": [("se", [wrapped_fasta(2000, seed=4)])],
        "gen_interleaved": [("interleaved", [fastq(1000, 120, seed=5)])],
        "gen_interleaved_odd": [("interleaved", [fastq(999, 120, seed=6)])],
        "gen_megabase": [("se", [megabase_record(7)])],
        "gen_misguided": [("se", [misguided(3000)])],
        "gen_multi_lib": [("pe", [fastq(500, 100, seed=8), fastq(500, 100, seed=9)]), ("se", [wrapped_fasta(300, seed=10)]),
                          ("interleaved", [fastq(200, 90, seed=12)])],
    }


def all_cases():
    """name -> list of (type, [bytes]) libraries: every edge case as one se library, plus the generated ones"""
    out = {f"edge_{k}": [("se", [v])] for k, v in edge_cases().items()}
    out.update(generated())
    return out


def write_lib(d, libs):
    """input files + lib file for `libs` under d; returns the lib file path"""
    lines = []
    for i, (typ, datas) in enumerate(libs):
        paths = []
        for j, b in enumerate(datas):
            p = os.path.join(d, f"l{i}_{j}.fx")
            with open(p, "wb") as f:
                f.write(b)
            paths.append(p)
        lines.append(f"lib{i} {typ}\n{typ} {' '.join(paths)}\n")
    lib = os.path.join(d, "reads.lib")
    with open(lib, "w") as f:
        f.write("".join(lines))
    return lib


def digests(prefix):
    out = {}
    for ext in ("bin", "lib_info"):
        with open(f"{prefix}.{ext}", "rb") as f:
            out[ext] = hashlib.sha256(f.read()).hexdigest()
    return out
