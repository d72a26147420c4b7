"""Seeded inputs of the wide-k `iterate` tests: from (k, step, seed) the contig and bubble FASTA text and a variable-length
`.bin` read image, regenerated identically by the CPU and GPU tests.  tests/golden_iter_wide/iter_wide.json holds what
the unmodified reference wrote for them (oracle/gen_golden_iter_wide.py).

The (k, step) matrix covers every register class of the kernels (2 / 4 / 8 / 17 words) at its bottom and top, the
reference's own k-mer type boundaries (k + 1 = 32, 64, 128, and k + step + 1 = 32 ... 256) and w2 = wn + 1, where the
last edge word lies beyond the (k+step+1)-mer's words."""
import os

import numpy as np

from megahit_b200 import formats as F

MATRIX = [(9, 2), (21, 10), (31, 2), (49, 10), (41, 22), (63, 2), (99, 28), (119, 22), (127, 2), (141, 28), (211, 28),
          (227, 28), (239, 16)]
SCALE = [(119, 22), (227, 28)]
SCALE_READS = 200_000
SCALE_LEN = (200, 401)


def rc(s):
    return (3 - np.asarray(s, np.uint8)[::-1]).astype(np.uint8)


def pack_padded(b: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """(n, maxL) uint8 bases (anything past a read's length ignored) + lengths -> the `.bin` image (uint32 words)"""
    n = len(lens)
    if n == 0:
        return np.zeros(0, np.uint32)
    lens = np.asarray(lens, np.int64)
    W = max(1, (int(lens.max()) + 15) // 16)
    pad = np.zeros((n, 16 * W), np.uint8)
    m = min(b.shape[1], 16 * W)
    pad[:, :m] = b[:, :m]
    pad[np.arange(16 * W)[None, :] >= lens[:, None]] = 0
    pad = pad.reshape(n, W, 16)
    words = np.zeros((n, W), np.uint32)
    for j in range(16):
        words |= pad[:, :, j].astype(np.uint32) << np.uint32(30 - 2 * j)
    full = np.concatenate([lens.astype(np.uint32)[:, None], words], axis=1)
    keep = np.arange(W + 1)[None, :] < 1 + (lens[:, None] + 15) // 16
    return full[keep]


def pack_list(reads) -> np.ndarray:
    lens = np.array([len(r) for r in reads], np.int64)
    b = np.zeros((len(reads), max(1, int(lens.max()) if len(reads) else 1)), np.uint8)
    for i, r in enumerate(reads):
        b[i, :len(r)] = r
    return pack_padded(b, lens)


def sample_reads(rng, g, n, lo, hi, err=0.004):
    """n reads of lengths in [lo, hi) from g, either strand, with substitutions: (padded bases, lengths)"""
    G = len(g)
    lens = rng.integers(lo, hi, size=n)
    pos = rng.integers(0, G - lens + 1)
    ar = np.arange(hi)[None, :]
    b = g[np.minimum(pos[:, None] + ar, G - 1)]
    flip = rng.integers(0, 2, size=n).astype(bool)
    ridx = np.clip(lens[flip, None] - 1 - ar, 0, hi - 1)
    b[flip] = 3 - np.take_along_axis(b[flip], ridx, axis=1)
    e = (rng.random(b.shape) < err) & (ar < lens[:, None])
    b[e] = (b[e] + rng.integers(1, 4, size=int(e.sum()), dtype=np.uint8)) & 3
    return b, lens


def _fasta(records, rng):
    """(bases, flag) -> FASTA text: some records lowercase in runs, a few N, some wrapped over several lines"""
    out = []
    for i, (s, flag) in enumerate(records):
        t = np.array(list("ACGT"))[s].astype(object)
        if i % 3 == 1 and len(s) > 20:
            a = int(rng.integers(0, len(s) - 10))
            z = a + int(rng.integers(5, 60))
            t[a:z] = [c.lower() for c in t[a:z]]
        if i % 7 == 3 and len(s) > 4:
            for p in rng.choice(len(s), 2, replace=False):
                t[p] = "N" if rng.integers(0, 2) else "n"
        seq = "".join(t)
        wrap = (0, 60, 0, 77)[i % 4]
        body = "\n".join(seq[j:j + wrap] for j in range(0, len(seq), wrap)) if wrap and seq else seq
        out.append(f">c{i} flag={flag} multi=1.0000 len={len(s)}\n{body}\n")
    return "".join(out)


def make_case(k, step, seed, n_reads=500, read_len=None, G=None):
    """dict(contigs=FASTA text, bubbles=FASTA text, bin=`.bin` words, n_reads, genome=the bases the reads come from)"""
    rng = np.random.default_rng([k, step, seed])
    K1, KN = k + 1, k + step + 1
    G = G or 6000 + 20 * k
    g = rng.integers(0, 4, G, dtype=np.uint8)
    copies = 3 if G < 100_000 else 60
    for rl in (k + 3, k + step // 2, 2 * k):  # repeats: contigs break there, reads across them give iterative edges
        rep = rng.integers(0, 4, rl, dtype=np.uint8)
        for p in rng.choice(G - rl, copies, replace=False):
            g[p:p + rl] = rep
    n_cuts = 14 if G < 100_000 else G // 1500
    cuts = np.sort(rng.choice(np.arange(k + 2, G - k - 2), n_cuts, replace=False))
    bounds = [0] + [int(c) for c in cuts] + [G]
    pieces = [g[max(0, a - k):b] for a, b in zip(bounds[:-1], bounds[1:])]  # k-base overlaps, as unitigs
    contigs = [(rc(c) if i % 3 == 2 else c, 0) for i, c in enumerate(pieces)]
    contigs += [(rc(c), 0) for c in pieces[::4]]                       # a few on both strands
    contigs += [(g[100:100 + K1], 0), (g[300:300 + k], 0), (g[400:405], 0)]  # exactly k + 1 bases; too short
    h = rng.integers(0, 4, K1 // 2, dtype=np.uint8)
    pal = np.concatenate([h, rc(h)])                                   # a palindromic (k+1)-mer (k + 1 is even)
    contigs += [(np.concatenate([pal, g[500:500 + step + 10]]), 0), (pal, 0)]
    contigs += [(g[700:700 + K1 + step + 20], 0), (g[700:700 + K1 + (step - 1) // 2], 0)]  # a prefix: one key, two ext lengths
    variants = []
    for p in (900, 1100, 1300):  # one key, two extensions of the same length: the larger one survives
        v = np.concatenate([g[p:p + K1], rng.integers(0, 4, step + 10, dtype=np.uint8)])
        variants.append(np.concatenate([g[p - 40:p], v]))
        contigs += [(g[p:p + K1 + step + 10], 0), (v, 0)]
    contigs += [(g[1500:1500 + 2 * k], 1), (g[1800:1800 + 2 * k + 7], 2), (g[2100:2100 + k + 30], 3)]  # discarded
    rng.shuffle(contigs)
    bubbles = []
    for p in (2500, 2900, 3300, 3700):
        s = g[p:p + 2 * k + 4].copy()
        s[k + 2] = (s[k + 2] + 1) & 3
        bubbles.append((s, 0))
    bubbles.append((g[4100:4100 + 2 * k], 1))

    lo, hi = read_len or (k, 3 * k + 2 * step + 40)
    b, lens = sample_reads(rng, g, n_reads, lo, hi)
    extra = [g[q:q + KN] for q in rng.integers(0, G - KN, 5)] + [g[q:q + KN - 1] for q in rng.integers(0, G - KN, 5)]
    extra += [rc(v) if i % 2 else v for i, v in enumerate(variants * 4)] + [np.zeros(0, np.uint8)] * 3
    eb = np.zeros((len(extra), b.shape[1] if len(extra) == 0 else max(b.shape[1], max(len(x) for x in extra))), np.uint8)
    for i, x in enumerate(extra):
        eb[i, :len(x)] = x
    allb = np.zeros((len(lens) + len(extra), eb.shape[1]), np.uint8)
    allb[:len(lens), :b.shape[1]] = b
    allb[len(lens):] = eb
    alll = np.concatenate([lens, [len(x) for x in extra]]).astype(np.int64)
    order = rng.permutation(len(alll))
    return {"contigs": _fasta(contigs, rng), "bubbles": _fasta(bubbles, rng), "bin": pack_padded(allb[order], alll[order]),
            "n_reads": len(alll), "genome": g}


def make_scale_case(k, step, seed=1):
    return make_case(k, step, seed, n_reads=SCALE_READS, read_len=SCALE_LEN, G=1_000_000)


def write_case(case, d):
    """the case's files under d: (contigs, bubbles, `.bin`)"""
    os.makedirs(d, exist_ok=True)
    paths = tuple(os.path.join(d, f) for f in ("contigs.fa", "bubble_seq.fa", "reads.lib.bin"))
    for p, key in zip(paths[:2], ("contigs", "bubbles")):
        with open(p, "w") as f:
            f.write(case[key])
    case["bin"].tofile(paths[2])
    return paths


def read_lengths(bin_words, n_reads):
    out, pos = [], 0
    for _ in range(n_reads):
        L = int(bin_words[pos])
        out.append(L)
        pos += 1 + (L + 15) // 16
    return out


def split_bin(bin_words, n_reads):
    """the `.bin` image as a list of per-read records (uint32 arrays)"""
    out, pos = [], 0
    for _ in range(n_reads):
        w = 1 + (int(bin_words[pos]) + 15) // 16
        out.append(bin_words[pos:pos + w])
        pos += w
    return out
