// mhb_s2s_sort.cu -- the seq2sdbg item sort (include/mhb.h: mhb_s2s_sort).
//
// The emitter only needs the items ordered inside their 16-bit bucket (the first eight bases, the top half of word 0):
// every (k-1)-mer group it walks lies inside one bucket because k - 1 >= 8, and the bucket table is cut on the same
// buckets.  Order among items with equal sort bytes does not matter (the emitter takes the minimum multiplicity of a
// run).  So for 8- and 12-byte items (9 <= k <= 38) the sort is
//   1. two global radix passes of the relaxed engine (mhb_sortdisp.cu) on the bucket bytes 4W-2 (unstable, fed by the
//      extract kernel's histogram) and 4W-1 (stable): every item lands in its bucket;
//   2. k_bucket_bounds: the 65 537 bucket boundaries by binary search on word 0;
//   3. k_s2s_local_sort: a persistent CTA takes buckets by ticket, stages a bucket's records in shared memory and orders
//      them there on the rest of the key (s2s_local_key: 2k - 12 bits), then writes them to the other buffer with
//      coalesced stores.  The local sort is one counting pass on the top 12 key bits (4096 groups of about 0.45 items
//      at the bench's 1 800 items per bucket) followed by ranking every item inside its group by counting the smaller
//      keys.  Two geometries: 3072 items (2 CTAs/SM) and 8192 items (1 CTA/SM).  The small one runs first when the
//      buckets average at most 3/4 of it and passes the buckets of 3073..8192 items on to a second launch of the large
//      one; otherwise the large one takes every bucket.  A bucket of more than 8192 items, or one with a 12-bit group
//      of more than kLsGroupMax items (long runs of equal keys: tandem repeats, poly-A), is not sorted here; its range
//      goes to a small device list;
//   4. the listed buckets are sorted as segments by the relaxed engine on the remaining sort bytes; with more than
//      kLsListCap of them the whole array is sorted again by the full relaxed sort instead (the data is a permutation,
//      so that is correct from wherever it stands).  Deciding this costs one stream synchronisation per sort (two when
//      the large geometry has a second launch).
// Sorts of more than 3/4 of 65 536 x 8192 = 403 M items (their buckets could not be held) do not try the bucket path:
// they are the full relaxed sort from the start, and mhb_s2s_sort_hist_byte(n, k) then names byte 2 for the extract
// kernel's histogram, so they cost what the relaxed sort costs.
// HBM traffic: 2 x 2 passes + bucket kernel = 6 x N x 4W bytes, against 2 x N x 4W per byte for the 8-pass LSD sort.
// Only the two global passes take a slot of the per-pass timing ring (mhb_sort_pass_ms).  Wider items (k >= 39) and
// k < 9 keep the full relaxed sort.
#include <cuda_runtime.h>

#include <algorithm>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "mhb.h"
#include "mhb_common.cuh"
#include "mhb_kernels.cuh"

using namespace mhb;

namespace {

// Two geometries of the bucket kernel: the small one (3072 items, 512 threads, 2 CTAs/SM) for libraries whose buckets
// average up to 3/4 of it (the bench: 1 800, largest 2 002), the large one (8192 items, 1024 threads, 1 CTA/SM) for
// libraries up to 3/4 of 65 536 x 8192 = 403 M items, and for the buckets of 3073..8192 items the small one met.
constexpr u32 kLsCapS = 3072, kLsCapL = 8192;
constexpr int kLsThreadsS = 512, kLsThreadsL = 1024;
constexpr int kLsDigitBits = 12;
constexpr u32 kLsDigits = 1u << kLsDigitBits;
constexpr u32 kLsGroupMax = 256;              // largest 12-bit group ranked by counting (O(group) per item)
constexpr u32 kLsListCap = 16;                // buckets left to the engine sorted one by one; more = one whole-array sort
// above this many items the bucket path is not tried: the buckets would not fit even the large geometry
constexpr uint64_t kLsMaxItems = (uint64_t)MHB_NUM_BUCKETS * kLsCapL * 3 / 4;
constexpr uint64_t kLsSmallMaxItems = (uint64_t)MHB_NUM_BUCKETS * kLsCapS * 3 / 4;

struct LsCtl {
  unsigned int ticket, ticket2;     // next bucket of the first and of the second launch
  unsigned int n_mid;               // buckets of kLsCapS < size <= kLsCapL the small geometry passed on (ids in `mid`)
  unsigned int n_over;              // buckets left to the engine
  unsigned long long items_over;    // their items
  unsigned long long range[2 * kLsListCap];  // [lo, hi) of the first kLsListCap of them
};

template <int W, u32 CAP>
constexpr size_t ls_smem() {
  return (size_t)CAP * 8 /*keys*/ + ((size_t)CAP * W + 4) * 4 /*records*/ + (kLsDigits + 4) * 4 /*groups*/ +
         (size_t)CAP * 2 * 2 /*source index, permutation*/;
}

// ids == nullptr: buckets 0 .. 65535; else the n_ids buckets listed there.  mid != nullptr: buckets of more than CAP
// but at most kLsCapL items are appended to `mid` (for the large geometry) instead of being left to the engine.
template <int W, u32 CAP, int THREADS>
__global__ void __launch_bounds__(THREADS, CAP == kLsCapS ? 2 : 1)
    k_s2s_local_sort(const u32 *__restrict__ in, u32 *__restrict__ out, const u64 *__restrict__ bounds, u32 k, LsCtl *ctl,
                     unsigned int *ticket, const u32 *__restrict__ ids, u32 n_ids, u32 *mid) {
  constexpr u32 kLsCap = CAP;
  constexpr int kLsThreads = THREADS;
  constexpr int kLsIpt = CAP / THREADS;  // items per thread
  extern __shared__ __align__(16) unsigned char smem_ls[];
  u64 *s_key = reinterpret_cast<u64 *>(smem_ls);                  // keys in group order
  u32 *s_rec = reinterpret_cast<u32 *>(s_key + kLsCap);           // the bucket's records (from a 16-byte boundary)
  u32 *s_grp = s_rec + kLsCap * W + 4;                            // group counts, then group starts (+ end)
  uint16_t *s_src = reinterpret_cast<uint16_t *>(s_grp + kLsDigits + 4);  // record of each key in s_key
  uint16_t *s_perm = s_src + kLsCap;                                      // record at each output position
  __shared__ u32 s_ticket;
  __shared__ u32 s_scan[kLsThreads / 32 + 1];
  const u32 tid = threadIdx.x;
  const u32 n_units = ids ? n_ids : (u32)MHB_NUM_BUCKETS;
  if (tid == 0) s_ticket = atomicAdd(ticket, 1u);
  __syncthreads();
  u32 t = s_ticket;
  while (t < n_units) {
    u32 next = 0;
    if (tid == 0) next = atomicAdd(ticket, 1u);  // its latency hides behind this bucket
    const u32 b = ids ? ids[t] : t;
    const u64 lo = bounds[b], hi = bounds[b + 1];
    bool local = hi - lo <= kLsCap;
    if (!local && mid && hi - lo <= kLsCapL) {  // the large geometry takes it
      if (tid == 0) mid[atomicAdd(&ctl->n_mid, 1u)] = b;
      local = true;
    } else if (local && hi > lo) {
      const u32 n = (u32)(hi - lo);
      // ---- stage the records: 16-byte pieces from the 16-byte boundary at or below the bucket, then the tail ----
      const u64 w_begin = lo * W, w_end = hi * W, a0 = w_begin & ~3ull;
      const u32 off = (u32)(w_begin - a0);
      const u32 nvec = (u32)((w_end - a0) >> 2);
      const uint4 *src4 = reinterpret_cast<const uint4 *>(in + a0);
      uint4 *dst4 = reinterpret_cast<uint4 *>(s_rec);
      for (u32 j0 = 0; j0 < nvec; j0 += 4 * kLsThreads) {
        uint4 v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const u32 j = j0 + q * kLsThreads + tid;
          if (j < nvec) v[q] = __ldg(src4 + j);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const u32 j = j0 + q * kLsThreads + tid;
          if (j < nvec) dst4[j] = v[q];
        }
      }
      for (u64 x = a0 + 4ull * nvec + tid; x < w_end; x += kLsThreads) s_rec[x - a0] = __ldg(in + x);
      for (u32 i = tid; i <= kLsDigits; i += kLsThreads) s_grp[i] = 0;
      __syncthreads();
      // ---- keys; counting pass on their top 12 bits (rank inside the group from a shared-memory atomic) ----
      u64 key[kLsIpt];
      u32 dr[kLsIpt];  // group << 16 | rank inside the group
#pragma unroll
      for (int q = 0; q < kLsIpt; ++q) {
        const u32 i = tid + q * kLsThreads;
        if (i < n) {
          u32 r[W];
#pragma unroll
          for (int j = 0; j < W; ++j) r[j] = s_rec[off + i * W + j];
          key[q] = s2s_local_key<W>(r, k);
          const u32 d = (u32)(key[q] >> (64 - kLsDigitBits));
          dr[q] = (d << 16) | atomicAdd(&s_grp[d], 1u);
        }
      }
      __syncthreads();
      // ---- group starts (exclusive scan, kLsDigits / kLsThreads groups per thread) ----
      constexpr int GPT = kLsDigits / kLsThreads;
      u32 c[GPT], sum = 0, cmax = 0;
#pragma unroll
      for (int j = 0; j < GPT; ++j) {
        c[j] = s_grp[tid * GPT + j];
        sum += c[j];
        cmax = max(cmax, c[j]);
      }
      u32 total;
      u32 run = block_excl_scan<kLsThreads>(sum, s_scan, total);
#pragma unroll
      for (int j = 0; j < GPT; ++j) {
        s_grp[tid * GPT + j] = run;
        run += c[j];
      }
      if (tid == 0) s_grp[kLsDigits] = n;
      local = !__syncthreads_or(cmax > kLsGroupMax);
      if (local) {
#pragma unroll
        for (int q = 0; q < kLsIpt; ++q) {
          const u32 i = tid + q * kLsThreads;
          if (i < n) {
            const u32 p = s_grp[dr[q] >> 16] + (dr[q] & 0xFFFFu);
            s_key[p] = key[q];
            s_src[p] = (uint16_t)i;
          }
        }
        __syncthreads();
        // ---- rank inside the group: smaller keys, and equal keys at smaller positions ----
        for (u32 p = tid; p < n; p += kLsThreads) {
          const u64 x = s_key[p];
          const u32 d = (u32)(x >> (64 - kLsDigitBits));
          const u32 g0 = s_grp[d], g1 = s_grp[d + 1];
          u32 rank = g0;
          for (u32 u = g0; u < g1; ++u) {
            const u64 y = s_key[u];
            rank += (y < x || (y == x && u < p)) ? 1u : 0u;
          }
          s_perm[rank] = s_src[p];
        }
        __syncthreads();
        // ---- write the bucket in order: coalesced word stores ----
        for (u32 x = tid; x < n * W; x += kLsThreads) {
          const u32 i = x / W, j = x - i * W;
          out[w_begin + x] = s_rec[off + (u32)s_perm[i] * W + j];
        }
      }
    }
    if (!local && tid == 0) {
      const u32 slot = atomicAdd(&ctl->n_over, 1u);
      atomicAdd(&ctl->items_over, (unsigned long long)(hi - lo));
      if (slot < kLsListCap) {
        ctl->range[2 * slot] = lo;
        ctl->range[2 * slot + 1] = hi;
      }
    }
    __syncthreads();
    if (tid == 0) s_ticket = next;
    __syncthreads();
    t = s_ticket;
  }
}

bool s2s_local_path(uint32_t k) {
  const u32 w = s2s_record_words(k);
  return k >= 9 && (w == 2 || w == 3);
}
size_t pad256(size_t x) { return (x + 255) & ~(size_t)255; }

// ids / n_ids / mid: as k_s2s_local_sort
template <int W, u32 CAP, int THREADS>
int launch_local_sort(cudaStream_t st, const u32 *in, u32 *out, const u64 *bounds, u32 k, LsCtl *ctl, unsigned int *ticket,
                      const u32 *ids, u32 n_ids, u32 *mid) {
  constexpr size_t smem = ls_smem<W, CAP>();
  static int bps = 0;
  if (!bps) {
    CK(cudaFuncSetAttribute(k_s2s_local_sort<W, CAP, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_s2s_local_sort<W, CAP, THREADS>, THREADS, smem));
    if (bps < 1) return mhb_set_error(MHB_ERR_CUDA, "bucket sort kernel (W=%d, capacity %u) does not fit an SM", W, CAP);
    if (getenv("MHB_VERBOSE")) fprintf(stderr, "[mhb] s2s bucket sort W=%d: %d threads, capacity %u, %zu B smem, %d CTA/SM\n", W, THREADS, CAP, smem, bps);
  }
  const u32 units = ids ? n_ids : (u32)MHB_NUM_BUCKETS;
  const int grid = (int)std::min<u64>((u64)bps * sm_count(), units);
  k_s2s_local_sort<W, CAP, THREADS><<<grid, THREADS, smem, st>>>(in, out, bounds, k, ctl, ticket, ids, n_ids, mid);
  CK_LAUNCH();
  return MHB_OK;
}

template <int W>
int launch_local(cudaStream_t st, bool large, const u32 *in, u32 *out, const u64 *bounds, u32 k, LsCtl *ctl, unsigned int *ticket,
                 const u32 *ids, u32 n_ids, u32 *mid) {
  if (large) return launch_local_sort<W, kLsCapL, kLsThreadsL>(st, in, out, bounds, k, ctl, ticket, ids, n_ids, nullptr);
  return launch_local_sort<W, kLsCapS, kLsThreadsS>(st, in, out, bounds, k, ctl, ticket, ids, n_ids, mid);
}

bool s2s_bucket_path(uint64_t n, uint32_t k) { return s2s_local_path(k) && n <= kLsMaxItems; }

// what the bucket kernel of the last mhb_s2s_sort left to the engine (mhb_s2s_sort_stats)
LsCtl g_last_ctl;

}  // namespace

extern "C" int mhb_s2s_sort_hist_byte(uint64_t n, uint32_t k) {
  // the byte the first pass of a sort of n items sorts on: the extract kernels histogram it so that the sort needs no
  // histogram pass (byte 2 for the full relaxed sort)
  return s2s_bucket_path(n, k) ? (int)(4 * s2s_record_words(k) - 2) : 2;
}

extern "C" size_t mhb_s2s_sort_workspace_bytes(uint64_t n, uint32_t k) {
  const uint32_t W = s2s_record_words(k);
  const size_t base = pad256(mhb_sort_workspace_bytes(n, W));
  if (!s2s_local_path(k)) return base;
  return base + pad256((size_t)(MHB_NUM_BUCKETS + 1) * 8) + pad256(sizeof(LsCtl)) + pad256((size_t)MHB_NUM_BUCKETS * 4);
}

extern "C" int mhb_s2s_sort(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t k, const uint64_t *first_hist,
                            void *ws, size_t ws_bytes, int *result_in_b) {
  if (k < 1 || k > MHB_MAX_K || !result_in_b) return mhb_set_error(MHB_ERR_ARG, "bad seq2sdbg sort arguments (k=%u)", k);
  const uint32_t W = s2s_record_words(k);
  uint8_t bytes[80];
  const uint32_t nb = mhb_s2s_sort_bytes(k, bytes);
  const size_t sort_ws = mhb_sort_workspace_bytes(n, W);
  g_last_ctl = LsCtl{};
  if (!s2s_bucket_path(n, k)) return mhb_sort_records_relaxed(stream, a, b, n, W, bytes, nb, first_hist, ws, ws_bytes, result_in_b);
  *result_in_b = 0;
  if (n == 0) return MHB_OK;
  if (ws_bytes < mhb_s2s_sort_workspace_bytes(n, k)) return mhb_set_error(MHB_ERR_ARG, "seq2sdbg sort workspace too small");
  if ((((uintptr_t)a | (uintptr_t)b) & 15) != 0) return mhb_set_error(MHB_ERR_ARG, "seq2sdbg sort buffers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  // 1. the two bucket bytes (the only entry of this sort in the timing ring)
  const uint8_t top[2] = {(uint8_t)(4 * W - 2), (uint8_t)(4 * W - 1)};
  int in_b = 0;
  if (int rc = mhb_sort_records_ex(stream, a, b, n, W, top, 2, first_hist, ws, sort_ws, &in_b, nullptr, 1)) return rc;
  u32 *x = in_b ? b : a, *y = in_b ? a : b;
  // 2. bucket bounds, 3. buckets in shared memory: x -> y (small geometry first unless the buckets average more than
  // 3/4 of it; the buckets it cannot hold but the large one can go to a second launch of the large one)
  u64 *bounds = reinterpret_cast<u64 *>((char *)ws + pad256(sort_ws));
  LsCtl *ctl = reinterpret_cast<LsCtl *>((char *)bounds + pad256((size_t)(MHB_NUM_BUCKETS + 1) * 8));
  u32 *mid = reinterpret_cast<u32 *>((char *)ctl + pad256(sizeof(LsCtl)));
  CK(cudaMemsetAsync(ctl, 0, sizeof(LsCtl), st));
  if (W == 2) k_bucket_bounds<2><<<(65537 + 255) / 256, 256, 0, st>>>(x, n, bounds);
  else k_bucket_bounds<3><<<(65537 + 255) / 256, 256, 0, st>>>(x, n, bounds);
  CK_LAUNCH();
  const bool large = n > kLsSmallMaxItems;
  if (int rc = W == 2 ? launch_local<2>(st, large, x, y, bounds, k, ctl, &ctl->ticket, nullptr, 0, mid)
                      : launch_local<3>(st, large, x, y, bounds, k, ctl, &ctl->ticket, nullptr, 0, mid)) return rc;
  // 4. what the bucket kernel left over
  LsCtl h;
  CK(cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (h.n_mid) {
    if (int rc = W == 2 ? launch_local<2>(st, true, x, y, bounds, k, ctl, &ctl->ticket2, mid, h.n_mid, nullptr)
                        : launch_local<3>(st, true, x, y, bounds, k, ctl, &ctl->ticket2, mid, h.n_mid, nullptr)) return rc;
    CK(cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  g_last_ctl = h;
  *result_in_b = y == b ? 1 : 0;
  if (h.n_over == 0) return MHB_OK;
  if (h.n_over > kLsListCap) {
    int r_in_b = 0;
    if (int rc = mhb_sort_records_untraced(stream, x, y, n, W, bytes, nb, nullptr, ws, sort_ws, &r_in_b)) return rc;
    *result_in_b = (r_in_b ? y : x) == b ? 1 : 0;
    return MHB_OK;
  }
  for (u32 s = 0; s < h.n_over; ++s) {
    const u64 lo = h.range[2 * s], hi = h.range[2 * s + 1];
    int r_in_b = 0;
    if (int rc = mhb_sort_records_untraced(stream, x + lo * W, y + lo * W, hi - lo, W, bytes, nb - 2, nullptr, ws, sort_ws, &r_in_b)) return rc;
    if (!r_in_b) CK(cudaMemcpyAsync(y + lo * W, x + lo * W, (hi - lo) * W * 4, cudaMemcpyDeviceToDevice, st));
  }
  return MHB_OK;
}

extern "C" void mhb_s2s_sort_stats(uint64_t *n_oversized, uint64_t *oversized_items, uint64_t *n_large) {
  if (n_oversized) *n_oversized = g_last_ctl.n_over;
  if (oversized_items) *oversized_items = g_last_ctl.items_over;
  if (n_large) *n_large = g_last_ctl.n_mid;
}

extern "C" int mhb_selftest_s2s_local_key(const uint32_t *recs, uint64_t n, uint32_t k, uint64_t *keys) {
  if (!s2s_local_path(k) || !recs || !keys) return mhb_set_error(MHB_ERR_ARG, "bad local-key arguments (k=%u)", k);
  const uint32_t W = s2s_record_words(k);
  for (uint64_t i = 0; i < n; ++i) {
    if (W == 2) {
      const u32 r[2] = {recs[2 * i], recs[2 * i + 1]};
      keys[i] = s2s_local_key<2>(r, k);
    } else {
      const u32 r[3] = {recs[3 * i], recs[3 * i + 1], recs[3 * i + 2]};
      keys[i] = s2s_local_key<3>(r, k);
    }
  }
  return MHB_OK;
}
