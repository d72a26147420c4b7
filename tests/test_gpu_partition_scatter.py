"""The fused partition + exchange pass of the multi-GPU build (mhb_partition_scatter / _hist) on one GPU: every owner's
destination is its own region of one local buffer, with guard words between the regions.  Each region must receive
exactly its owner's records (as a multiset: the pass leaves no order within an owner), nothing outside the regions may
change, and the per-owner histogram of the next sort byte must equal NumPy's."""
import ctypes as C

import numpy as np
import pytest

from megahit_b200 import lib

pytestmark = pytest.mark.gpu

GUARD = 0x5EC7A11D
PART_THREADS = 384


def _tile(words):  # records per tile of the partition pass (mhb_part.cuh: 384 threads x the stable pass's IPT)
    ipt = 18 if words <= 2 else 12 if words <= 3 else 10 if words <= 4 else 6 if words <= 6 else 4 if words <= 9 else 2
    return PART_THREADS * ipt


def _multiset(x, words):
    return np.sort(np.ascontiguousarray(x).view([("", np.uint32)] * words).reshape(-1))


def _scatter(L, torch, recs, words, lut, next_byte):
    """runs the pass (with the owner histogram when next_byte is not None) into guarded regions of one buffer; returns
    (buffer on the host, region offsets in words, owner of every record, histogram or None)"""
    n = len(recs)
    n_owner = int(lut.max()) + 1
    owner = lut[recs[:, 0] >> 24]
    cnt = np.bincount(owner, minlength=n_owner)
    # every region starts 16-byte aligned (the pass stores 16- or 8-byte pieces) and is followed by at least 4 guard words
    off, pos = [], 4
    for o in range(n_owner):
        off.append(pos)
        pos += (int(cnt[o]) * words + 4 + 3) // 4 * 4
    buf = torch.full((pos + 4,), GUARD, dtype=torch.int32, device="cuda")
    addr = np.zeros(256, np.int64)
    addr[:n_owner] = [buf.data_ptr() + 4 * x for x in off]
    d_addr = torch.from_numpy(addr).cuda()
    d_lut = torch.from_numpy(lut.astype(np.uint8)).cuda()
    d_recs = torch.from_numpy(np.concatenate([recs.reshape(-1), np.zeros(4, np.uint32)]).view(np.int32)).cuda()
    ws = torch.empty(L.mhb_sort_workspace_bytes(max(n, 1), words), dtype=torch.uint8, device="cuda")
    ptr = lambda t: C.c_void_p(t.data_ptr())
    byte = 4 * words - 1  # the leading byte
    hist = None
    if next_byte is None:
        lib._check(L.mhb_partition_scatter(None, ptr(d_recs), n, words, byte, ptr(d_lut), ptr(d_addr), ptr(ws), ws.numel()))
    else:
        d_hist = torch.zeros(16 * 256, dtype=torch.int64, device="cuda")
        lib._check(L.mhb_partition_scatter_hist(None, ptr(d_recs), n, words, byte, ptr(d_lut), ptr(d_addr), ptr(ws),
                                                ws.numel(), next_byte, ptr(d_hist)))
        hist = d_hist.cpu().numpy().reshape(16, 256)
    torch.cuda.synchronize()
    return buf.cpu().numpy().view(np.uint32), off, owner, cnt, hist


@pytest.mark.parametrize("n_owner", [1, 2, 5, 16])
@pytest.mark.parametrize("words", range(1, 18))
def test_partition_scatter_fills_each_owner_region(words, n_owner):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    L = lib.load()
    rng = np.random.default_rng(words * 100 + n_owner)
    lut = rng.permutation(np.arange(256) % n_owner)  # every owner holds some leading bytes, scattered over the range
    t = _tile(words)
    for n in (0, 1, t - 1, t, t + 1, 3 * t + 17):
        recs = rng.integers(0, 2 ** 32, size=(n, words), dtype=np.uint64).astype(np.uint32)
        if n > 10:
            recs[: n // 4, 0] &= np.uint32(0x0FFFFFFF)  # skew: a quarter of the records on 16 leading bytes
        next_byte = int(rng.integers(0, 4 * words))
        for with_hist in (False, True):
            got, off, owner, cnt, hist = _scatter(L, torch, recs, words, lut, next_byte if with_hist else None)
            mask = np.ones(len(got), bool)
            for o in range(n_owner):
                reg = got[off[o]: off[o] + int(cnt[o]) * words].reshape(-1, words)
                mask[off[o]: off[o] + int(cnt[o]) * words] = False
                assert (_multiset(reg, words) == _multiset(recs[owner == o], words)).all(), (n, o, with_hist)
            assert (got[mask] == GUARD).all(), (n, with_hist, "guard words overwritten")
            if with_hist:
                w, s = words - 1 - (next_byte >> 2), 8 * (next_byte & 3)
                v = (recs[:, w] >> np.uint32(s)) & 255
                exp = np.zeros((16, 256), np.int64)
                np.add.at(exp, (owner, v.astype(np.int64)), 1)
                assert (hist == exp).all(), (n, "owner histogram")
    # the owner table is required (the destinations are valid, so that nothing could be stored out of bounds anyway)
    d_recs = torch.zeros(16 * words + 4, dtype=torch.int32, device="cuda")
    d_out = torch.zeros(16 * words + 4, dtype=torch.int32, device="cuda")
    d_addr = torch.full((256,), d_out.data_ptr(), dtype=torch.int64, device="cuda")
    ws = torch.empty(L.mhb_sort_workspace_bytes(16, words), dtype=torch.uint8, device="cuda")
    with pytest.raises(lib.MhbError):
        lib._check(L.mhb_partition_scatter(None, C.c_void_p(d_recs.data_ptr()), 16, words, 4 * words - 1, None,
                                           C.c_void_p(d_addr.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel()))
