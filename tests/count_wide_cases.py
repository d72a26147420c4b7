"""Read libraries and k lists for the tests of the count stage at every record width (tests/test_count_reference_cpu.py,
tests/test_gpu_count_wide.py)."""
import numpy as np

from count_reference import count_key_words, count_record_words, words_per_edge
from megahit_b200 import formats as F

READS_PER_BATCH = 64   # mhb_count.cuh kReadsPerBatch: for_each_read walks the reads in batches of 64
STAGE_WORDS = 4096     # mhb_count.cuh kStageWords: a batch whose words do not fit a 16 KiB stage is read from global memory


def width_classes(k_lo: int = 9, k_hi: int = 255) -> list:
    """one k per (W, WR, WE) = (key words, record words, edge words) class in [k_lo, k_hi]: the largest, where the key
    reaches furthest into the record (W = WR - 1 at k = 16w - 17: the last record word holds prev / next only)"""
    out = {}
    for k in range(k_lo, k_hi + 1):
        out[(count_key_words(k), count_record_words(k), words_per_edge(k))] = k
    return sorted(out.values())


def palindrome(rng, k: int) -> np.ndarray:
    """a (k+1)-mer equal to its reverse complement (k odd): reverse(S) == complement(S), the strand tie"""
    assert k % 2 == 1
    half = rng.integers(0, 4, (k + 1) // 2, dtype=np.uint8)
    return np.concatenate([half, 3 - half[::-1]]).astype(np.uint8)


def pack(reads) -> np.ndarray:
    return np.concatenate([F.pack_read(r) for r in reads]) if reads else np.zeros(0, np.uint32)


def batch_words(bin_words: np.ndarray, n_reads: int) -> np.ndarray:
    """the 16-byte aligned words every batch of for_each_read spans (a1 - a0 in the kernel)"""
    from count_reference import read_layout
    _, starts = read_layout(bin_words, n_reads)
    w0 = starts[::READS_PER_BATCH]
    w1 = np.append(w0[1:], len(bin_words))
    return ((w1 + 3) & ~3) - (w0 & ~3)


def library(k: int, seed: int, n_reads: int = 1500, max_len: int = 0, genome_len: int = 8000, err: float = 0.01,
            long_reads: bool = False):
    """Variable-length reads of 0 .. max_len (default k + 200) bases of a random genome with the lengths where extraction goes wrong:
    0, k, k + 1, k + 2 and L = 0, 1, 15 (mod 16); at odd k reads holding palindromic (k+1)-mers, three copies each so
    that they are solid at m <= 3.  long_reads: 64 reads of 1 100 - 1 400 bp filling one batch of for_each_read (more
    words than a stage holds) and one read of 70 000 bp covering the genome several times.
    -> (.bin word stream, n_reads, lengths)"""
    rng = np.random.default_rng(seed)
    max_len = max_len or k + 200
    genome = rng.integers(0, 4, genome_len, dtype=np.uint8)

    def sample(L):
        L = int(L)
        p = int(rng.integers(0, genome_len - L + 1))
        b = genome[p:p + L].copy()
        if rng.integers(0, 2):
            b = 3 - b[::-1]
        e = rng.random(L) < err
        b[e] = (b[e] + rng.integers(1, 4, int(e.sum()), dtype=np.uint8)) & 3
        return b.astype(np.uint8)

    reads = [sample(L) for L in rng.integers(0, max_len + 1, n_reads)]
    w = (k + 16) // 16
    for L in [0, 0, k, k + 1, k + 2, 16 * w, 16 * w + 1, 16 * w + 15, 16 * (w + 3), 16 * (w + 3) + 1, 16 * (w + 3) + 15]:
        reads.insert(int(rng.integers(0, len(reads) + 1)), sample(L))
    if k % 2 == 1:
        for _ in range(4):
            pal = palindrome(rng, k)
            flank = sample(int(rng.integers(0, 40)))
            for r in (pal, np.concatenate([flank, pal, sample(7)]), np.concatenate([sample(3), pal])):
                reads.insert(int(rng.integers(0, len(reads) + 1)), r)
    if long_reads:
        long = np.tile(genome, 70_000 // genome_len + 1)[:70_000].copy()
        e = rng.random(len(long)) < err
        long[e] = (long[e] + 1) & 3
        reads.insert(int(rng.integers(0, len(reads) + 1)), long)
        at = READS_PER_BATCH * int(rng.integers(1, len(reads) // READS_PER_BATCH))  # a batch of its own
        reads[at:at] = [sample(L) for L in rng.integers(1100, 1401, READS_PER_BATCH)]
    return pack(reads), len(reads), np.array([len(r) for r in reads], np.int64)
