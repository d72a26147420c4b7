"""Device-level stages on torch tensors (PyTorch = device memory + streams; the kernels are libmhb's).

`CountPlan` / `S2sPlan` pre-allocate every buffer a stage needs so that a timed step launches kernels
only; all launches go to torch's current stream, so `torch.cuda.Event` timing sees them.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def sort_records(a: torch.Tensor, b: torch.Tensor, n: int, words: int, sort_bytes, first_hist=None, ws=None, relaxed=False):
    """LSD radix sort of n records (int32 tensors a, b of >= n*words elements).  Returns the tensor
    holding the result.  relaxed: the order among records with all sorted bytes equal may be arbitrary (what the count
    and seq2sdbg stages need: mhb_sort_records_relaxed)."""
    L = lib.load()
    need = L.mhb_sort_workspace_bytes(n, words)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=a.device)
    bytes_arr = (C.c_uint8 * len(sort_bytes))(*sort_bytes)
    in_b = C.c_int(0)
    fn = L.mhb_sort_records_relaxed if relaxed else L.mhb_sort_records
    lib._check(fn(_stream(), _ptr(a), _ptr(b), n, words, bytes_arr, len(sort_bytes), _ptr(first_hist), _ptr(ws), ws.numel(),
                  C.byref(in_b)))
    return b if in_b.value else a


def s2s_sort(a: torch.Tensor, b: torch.Tensor, n: int, k: int, first_hist=None, ws=None):
    """The seq2sdbg item sort (mhb_s2s_sort) of n items in a; b is the other buffer (same size, 16-byte aligned).
    first_hist: histogram of record byte lib.s2s_sort_hist_byte(n, k), or None.  Returns the tensor holding the result."""
    L = lib.load()
    need = L.mhb_s2s_sort_workspace_bytes(n, k)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=a.device)
    in_b = C.c_int(0)
    lib._check(L.mhb_s2s_sort(_stream(), _ptr(a), _ptr(b), n, k, _ptr(first_hist), _ptr(ws), ws.numel(), C.byref(in_b)))
    return b if in_b.value else a


def s2s_sort_emit(a: torch.Tensor, b: torch.Tensor, n: int, k: int, first_hist, bytes_out: torch.Tensor, table: torch.Tensor,
                  totals: torch.Tensor, ws=None, cap_bytes: int | None = None):
    """The seq2sdbg item sort and the SdBG emitter in one call (mhb_s2s_sort_emit) over the n items in a (b: the other
    buffer; both are overwritten): the item stream goes to bytes_out (cap_bytes, default its size), the bucket table to
    table (int64[65536 * 4]) and the totals to totals (int64[16])."""
    L = lib.load()
    need = L.mhb_s2s_sort_emit_workspace_bytes(n, k)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=a.device)
    cap = bytes_out.numel() if cap_bytes is None else cap_bytes
    lib._check(L.mhb_s2s_sort_emit(_stream(), _ptr(a), _ptr(b), n, k, _ptr(first_hist), _ptr(bytes_out), cap, _ptr(table),
                                   _ptr(totals), _ptr(ws), ws.numel()))
    return totals


class CountPlan:
    """`count` (extract -> sort -> solid edges [-> mercy bookkeeping]) for a fixed-length read library
    resident on the device."""

    def __init__(self, n_reads: int, read_len: int, k: int, m: int, device, want_mercy: bool = True, mode: str | None = None):
        """mode: "sort" = LSD sort on every key byte + run-length count; "hashed" = two partition passes + per-bucket hash
        aggregation (8-byte records, mhb_count_solid_hashed); None = $MHB_COUNT_MODE, else hashed where supported."""
        import os
        L = lib.load()
        self.L, self.k, self.m, self.n_reads, self.read_len, self.device = L, k, m, n_reads, read_len, device
        self.want_mercy = want_mercy
        mode = mode or os.environ.get("MHB_COUNT_MODE") or "auto"
        ok = bool(L.mhb_count_hashed_supported(k, m))
        if mode == "hashed" and not ok:
            raise lib.MhbError(f"hashed count is not available for k={k}, m={m}")
        self.hashed = ok and mode in ("hashed", "auto")
        self.n = n_reads * (read_len - k) if read_len >= k + 1 else 0
        self.WR, self.WE = lib.count_record_words(k), lib.words_per_edge(k)
        self.sort_bytes = lib.count_sort_bytes(k)
        n = self.n
        i32 = dict(dtype=torch.int32, device=device)
        self.a = torch.empty(n * self.WR + 4, **i32)
        self.b = torch.empty(n * self.WR + 4, **i32)
        if self.hashed:
            self.ws = torch.empty(L.mhb_count_hashed_workspace_bytes(n, k, m), dtype=torch.uint8, device=device)
            self.scratch = None
        else:
            self.ws = torch.empty(L.mhb_sort_workspace_bytes(n, self.WR), dtype=torch.uint8, device=device)
            self.scratch = torch.empty(L.mhb_count_solid_scratch_bytes(n), dtype=torch.uint8, device=device)
        self.cap_edges = n // max(1, m) + 1
        self.edges = torch.empty(self.cap_edges * self.WE, **i32)
        self.aux = torch.empty(self.cap_edges, dtype=torch.uint8, device=device)
        self.mul_hist = torch.zeros(65536, dtype=torch.int64, device=device)
        self.hist0 = torch.zeros(256, dtype=torch.int64, device=device)
        self.n_solid_dev = torch.zeros(8, dtype=torch.int64, device=device)
        self.first = torch.empty(n_reads + 1, **i32) if want_mercy else None
        self.last = torch.empty(n_reads + 1, **i32) if want_mercy else None
        self.tipset = None
        self.events = {}

    def _reads(self, bin_dev: torch.Tensor) -> lib.DevReads:
        return lib.DevReads(bin_dev.data_ptr(), bin_dev.numel(), self.n_reads, self.read_len, None, None)

    def _mark(self, name):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self.events.setdefault(name, []).append(ev)

    def extract(self, bin_dev):
        self.hist0.zero_()
        lib._check(self.L.mhb_count_extract(_stream(), C.byref(self._reads(bin_dev)), self.k, _ptr(self.a), self.n,
                                            _ptr(self.hist0), 5 if self.hashed else self.sort_bytes[0]))

    def sort(self):
        if self.hashed:
            return None  # the two partition passes run inside count()
        self.sorted = sort_records(self.a, self.b, self.n, self.WR, self.sort_bytes, self.hist0, self.ws, relaxed=True)
        return self.sorted

    def count(self):
        self.mul_hist.zero_()
        self.n_solid_dev.zero_()
        if self.hashed:
            lib._check(self.L.mhb_count_solid_hashed(_stream(), _ptr(self.a), _ptr(self.b), self.n, self.k, self.m,
                                                     _ptr(self.hist0), _ptr(self.edges), _ptr(self.aux), self.cap_edges,
                                                     _ptr(self.mul_hist), _ptr(self.n_solid_dev), _ptr(self.ws), self.ws.numel()))
            return
        lib._check(self.L.mhb_count_solid(_stream(), _ptr(self.sorted), self.n, self.k, self.m, _ptr(self.edges),
                                          _ptr(self.aux), self.cap_edges, _ptr(self.mul_hist), _ptr(self.n_solid_dev),
                                          _ptr(self.scratch), self.scratch.numel()))

    def mercy(self, bin_dev):
        n_solid = int(self.n_solid_dev[0].item())
        n_tip = C.c_uint64(0)
        lib._check(self.L.mhb_count_tip_edges(_stream(), _ptr(self.aux), n_solid, C.byref(n_tip)))
        need = self.L.mhb_tipset_bytes(n_tip.value, self.k)
        if self.tipset is None or self.tipset.numel() < need:
            self.tipset = torch.empty(need, dtype=torch.uint8, device=self.device)
        lib._check(self.L.mhb_tipset_build(_stream(), _ptr(self.edges), _ptr(self.aux), n_solid, self.k,
                                           _ptr(self.tipset), need, n_tip.value))
        lib._check(self.L.mhb_count_mark_mercy(_stream(), C.byref(self._reads(bin_dev)), self.k, _ptr(self.tipset),
                                               need, n_tip.value, _ptr(self.first), _ptr(self.last)))
        return n_solid, n_tip.value

    def mercy_edges(self, bin_dev: torch.Tensor, n_solid: int) -> int:
        """A11 on the device (SeqToSdbg::GenMercyEdges): the candidate reads of the marks just computed, their mercy
        (k+1)-mers appended behind the n_solid solid edges in self.edges.  Returns the number of mercy edges."""
        L = self.L
        if not hasattr(self, "cand"):
            self.cand = torch.empty(self.n_reads + 1, dtype=torch.int64, device=self.device)
            self.cand_scratch = torch.empty(L.mhb_mercy_candidates_scratch_bytes(self.n_reads), dtype=torch.uint8, device=self.device)
            self.mercy_scratch = None
        nc = C.c_uint64(0)
        lib._check(L.mhb_mercy_candidates(_stream(), _ptr(self.first), _ptr(self.last), self.n_reads, _ptr(self.cand), C.byref(nc),
                                          _ptr(self.cand_scratch), self.cand_scratch.numel()))
        self.n_cand = nc.value
        if not self.n_cand:
            return 0
        need = L.mhb_mercy_edges_scratch_bytes(self.n_cand, self.read_len)
        if self.mercy_scratch is None or self.mercy_scratch.numel() < need:
            self.mercy_scratch = torch.empty(int(need * 1.2), dtype=torch.uint8, device=self.device)
        nm = C.c_uint64(0)
        lib._check(L.mhb_mercy_edges(_stream(), C.byref(self._reads(bin_dev)), _ptr(self.cand), self.n_cand, self.read_len, self.k,
                                     _ptr(self.edges), n_solid, C.c_void_p(self.edges.data_ptr() + n_solid * self.WE * 4),
                                     self.cap_edges - n_solid, C.byref(nm), _ptr(self.mercy_scratch), self.mercy_scratch.numel()))
        return nm.value

    def run(self, bin_dev: torch.Tensor, timed: bool = False):
        """One pass of the count stage over the resident library.  Returns n_solid (host int)."""
        if timed:
            self._mark("t0")
        self.extract(bin_dev)
        if timed:
            self._mark("extract")
        self.sort()
        if timed:
            self._mark("sort")
        self.count()
        if timed:
            self._mark("count")
        if self.want_mercy:
            n_solid, _ = self.mercy(bin_dev)
        else:
            n_solid = int(self.n_solid_dev[0].item())
        if timed:
            self._mark("mercy")
        return n_solid

    def edges_host(self, n_solid: int) -> np.ndarray:
        return self.edges[: n_solid * self.WE].cpu().numpy().view(np.uint32).reshape(-1, self.WE)


class S2sPlan:
    """`seq2sdbg` for fixed-length sequences ((k+1)-mer edges) resident on the device."""

    def __init__(self, n_seqs: int, seq_len: int, k: int, device):
        L = lib.load()
        self.L, self.k, self.n_seqs, self.seq_len, self.device = L, k, n_seqs, seq_len, device
        self.W = lib.s2s_record_words(k)
        self.sort_bytes = lib.s2s_sort_bytes(k)
        self.n_items = n_seqs * 2 * (seq_len - k + 2)
        n = self.n_items
        i32 = dict(dtype=torch.int32, device=device)
        self.a = torch.empty(n * self.W + 4, **i32)
        self.b = torch.empty(n * self.W + 4, **i32)
        # sort + emit workspace (mhb_s2s_sort_emit)
        self.ws = torch.empty(L.mhb_s2s_sort_emit_workspace_bytes(n, k), dtype=torch.uint8, device=device)
        wpt = (k + 15) // 16
        self.cap_bytes = n * (4 + 4 * wpt) + 16
        self.bytes = torch.empty(self.cap_bytes, dtype=torch.uint8, device=device)
        self.table = torch.zeros(65536 * 4, dtype=torch.int64, device=device)
        self.totals = torch.zeros(16, dtype=torch.int64, device=device)
        self.hist0 = torch.zeros(256, dtype=torch.int64, device=device)
        self.cursor = torch.zeros(1, dtype=torch.int64, device=device)
        self.events = []

    def run(self, words: torch.Tensor, mult: torch.Tensor | None = None, n_seqs: int | None = None, stride: int = 0,
            timed: bool = False, aux: torch.Tensor | None = None, n_aux: int = 0):
        """words: packed sequences; with mult=None they are `.edges` records of `stride` words each.  aux (with
        mult=None): the count stage's in/out flags of the first n_aux edges - the $-items the emitter is certain to
        discard are then not generated (mhb_s2s_extract_edges_pruned)."""
        n_seqs = self.n_seqs if n_seqs is None else n_seqs
        assert n_seqs <= self.n_seqs
        self.n_items = n_seqs * 2 * (self.seq_len - self.k + 2)
        if aux is not None and mult is None and not os.environ.get("MHB_S2S_NO_PRUNE"):
            return self._run_pruned(words, n_seqs, aux, n_aux, timed)
        seqs = lib.DevSeqs(words.data_ptr(), words.numel(), n_seqs, self.seq_len, None, None, None,
                           mult.data_ptr() if mult is not None else None, stride)
        self.hist0.zero_()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timed else None
        if timed:
            ev[0].record()
        lib._check(self.L.mhb_s2s_extract(_stream(), C.byref(seqs), self.k, _ptr(self.a), self.n_items, _ptr(self.hist0),
                                          lib.s2s_sort_hist_byte(self.n_items, self.k)))
        if timed:
            ev[1].record()
        self._sort_emit(self.hist0)
        if timed:  # sort and emit are one call: ev[1] -> ev[2] is both, ev[2] -> ev[3] is empty
            ev[2].record()
            ev[3].record()
            self.events.append(ev)
        return self.totals

    def _sort_emit(self, hist):
        s2s_sort_emit(self.a, self.b, self.n_items, self.k, hist, self.bytes, self.table, self.totals, self.ws, self.cap_bytes)

    def _run_pruned(self, edges: torch.Tensor, n_edges: int, aux: torch.Tensor, n_aux: int, timed: bool):
        cap = self.n_items
        self.hist0.zero_()
        self.cursor.zero_()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if timed else None
        if timed:
            ev[0].record()
        lib._check(self.L.mhb_s2s_extract_edges_pruned(_stream(), _ptr(edges), _ptr(aux), n_edges, n_aux, self.k, _ptr(self.a),
                                                       cap, _ptr(self.cursor), _ptr(self.hist0),
                                                       lib.s2s_sort_hist_byte(cap, self.k)))
        self.n_items = int(self.cursor.item())  # host read-back of the item count (launch geometry of the sort)
        assert self.n_items <= cap
        if timed:
            ev[1].record()
        # the histogram is of the byte a sort of `cap` items starts with; pass it only if this sort starts there too
        same = lib.s2s_sort_hist_byte(self.n_items, self.k) == lib.s2s_sort_hist_byte(cap, self.k)
        self._sort_emit(self.hist0 if same else None)
        if timed:  # sort and emit are one call: ev[1] -> ev[2] is both, ev[2] -> ev[3] is empty
            ev[2].record()
            ev[3].record()
            self.events.append(ev)
        return self.totals
