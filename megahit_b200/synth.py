"""Seeded synthetic read sets (SURVEY.md 8d): random genome, fixed-length reads at uniform positions,
random strand, substitution errors, no N.  numpy on the host; `synth_reads_torch` builds the same
distribution on the GPU for the large bench configs (data generation is plumbing, not the product)."""
from __future__ import annotations

import numpy as np

from .formats import pack_reads_fixed


def synth_reads(n_reads: int, read_len: int = 150, genome_len: int | None = None, err: float = 0.01,
                seed: int = 1, chunk: int = 1 << 18) -> np.ndarray:
    """Returns the `.bin` image as an (n_reads, 1 + ceil(read_len/16)) uint32 array."""
    rng = np.random.default_rng(seed)
    if genome_len is None:
        genome_len = max(read_len + 1, 5 * n_reads)  # ~30x coverage for 150 bp reads
    genome = rng.integers(0, 4, size=genome_len, dtype=np.uint8)
    out = []
    ar = np.arange(read_len, dtype=np.int64)
    for s in range(0, n_reads, chunk):
        n = min(chunk, n_reads - s)
        pos = rng.integers(0, genome_len - read_len + 1, size=n, dtype=np.int64)
        b = genome[pos[:, None] + ar[None, :]]
        rc = rng.integers(0, 2, size=n, dtype=np.uint8).astype(bool)
        b[rc] = 3 - b[rc][:, ::-1]
        if err > 0:
            e = rng.random(size=b.shape) < err
            b[e] = (b[e] + rng.integers(1, 4, size=int(e.sum()), dtype=np.uint8)) & 3
        out.append(pack_reads_fixed(b))
    return np.concatenate(out) if out else np.zeros((0, 1 + (read_len + 15) // 16), np.uint32)


def synth_reads_varlen(n_reads: int, min_len: int, max_len: int, genome_len: int, err: float = 0.01,
                       seed: int = 2) -> np.ndarray:
    """Variable-length reads (including ones shorter than k+1).  Returns the flat `.bin` word stream."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, size=genome_len, dtype=np.uint8)
    parts = []
    for _ in range(n_reads):
        L = int(rng.integers(min_len, max_len + 1))
        if L == 0:
            parts.append(np.array([0], np.uint32))
            continue
        p = int(rng.integers(0, genome_len - L + 1))
        b = genome[p:p + L].copy()
        if rng.integers(0, 2):
            b = 3 - b[::-1]
        e = rng.random(L) < err
        b[e] = (b[e] + rng.integers(1, 4, size=int(e.sum()), dtype=np.uint8)) & 3
        parts.append(pack_reads_fixed(b[None, :])[0])
    return np.concatenate(parts)


def synth_reads_trimmed(n_reads: int, max_len: int = 300, genome_len: int | None = None, err: float = 0.01,
                        seed: int = 3) -> tuple[np.ndarray, int]:
    """Reads of max_len bases (synth_reads) with their tails cut at a uniform position in [0, max_len], as buildlib's
    TrimN leaves reads at their first N; zero-length reads included.  Vectorised: millions of reads in seconds.
    Returns the flat `.bin` word stream and the number of bases."""
    b = synth_reads(n_reads, max_len, genome_len, err, seed)
    rng = np.random.default_rng(seed + 1)
    L = rng.integers(0, max_len + 1, size=n_reads).astype(np.int64)
    b[:, 0] = L.astype(np.uint32)
    nw = (L + 15) // 16
    w = np.arange(b.shape[1] - 1)
    tail = L % 16  # bases in the last kept word; clear the bits after them
    last = np.where(tail > 0, (0xFFFFFFFF << (32 - 2 * tail)) & 0xFFFFFFFF, 0xFFFFFFFF).astype(np.uint32)
    pay = b[:, 1:]
    at_last = w[None, :] == (nw - 1)[:, None]
    pay[at_last] &= np.broadcast_to(last[:, None], pay.shape)[at_last]
    keep = np.concatenate([np.ones((n_reads, 1), bool), w[None, :] < nw[:, None]], axis=1)
    return np.ascontiguousarray(b[keep]), int(L.sum())


def synth_reads_torch(n_reads: int, read_len: int, genome_len: int, err: float, seed: int, device):
    """Same distribution generated with torch on `device`; returns an (n_reads, 1+W) int32 tensor holding
    the `.bin` records (bit pattern of uint32)."""
    import torch

    g = torch.Generator(device=device)
    g.manual_seed(seed)
    genome = torch.randint(0, 4, (genome_len,), generator=g, device=device, dtype=torch.uint8)
    W = (read_len + 15) // 16
    out = torch.empty((n_reads, 1 + W), dtype=torch.int32, device=device)
    ar = torch.arange(read_len, device=device)
    shifts = (30 - 2 * torch.arange(16, device=device)).to(torch.int64)
    chunk = 1 << 20
    for s in range(0, n_reads, chunk):
        n = min(chunk, n_reads - s)
        pos = torch.randint(0, genome_len - read_len + 1, (n,), generator=g, device=device)
        b = genome[pos[:, None] + ar[None, :]].to(torch.int64)
        rc = torch.randint(0, 2, (n,), generator=g, device=device).bool()
        b = torch.where(rc[:, None], 3 - b.flip(1), b)
        e = torch.rand((n, read_len), generator=g, device=device) < err
        sub = torch.randint(1, 4, (n, read_len), generator=g, device=device)
        b = torch.where(e, (b + sub) & 3, b)
        pad = torch.zeros((n, W * 16), dtype=torch.int64, device=device)
        pad[:, :read_len] = b
        words = (pad.view(n, W, 16) << shifts).sum(dim=2)  # < 2^32
        words = torch.where(words >= (1 << 31), words - (1 << 32), words).to(torch.int32)
        out[s:s + n, 0] = read_len
        out[s:s + n, 1:] = words
    return out
