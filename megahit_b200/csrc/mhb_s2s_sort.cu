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
//
// mhb_s2s_sort_emit is this sort followed by the emitter (mhb_s2s_emit) without writing the sorted items back: the
// same bucket kernel with EMIT = true walks every sorted bucket's (k-1)-mer groups straight out of shared memory
// (s2s_group2, the emitter's group logic) once, into per-thread slots of the dead key array, and copies the bucket's item
// bytes to a staging slot at bounds[b] x maxb bytes - known before the kernel runs - and writes its row {bytes, items,
// tips, large}.  Two small launches scan the 65 536
// rows into the bucket table and one gather copies every bucket's bytes to its offset.  A listed bucket is sorted as a
// segment and emitted on its own by mhb_s2s_emit, with its side table and totals in the other buffer; more than
// kLsListCap of them (or one too large for the other buffer) -> the whole array is sorted again and emitted by
// mhb_s2s_emit, which works because the emitting kernel leaves its input a permutation of the items.
#include <cuda_runtime.h>

#include <algorithm>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "mhb.h"
#include "mhb_common.cuh"
#include "mhb_kernels.cuh"
#include "mhb_s2s.cuh"

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

// Where the emitting bucket kernel (EMIT = true) puts a bucket's SdBG items (mhb_s2s_sort_emit).
struct LsEmit {
  uint8_t *stage;  // bucket b's item bytes at stage + bounds[b] * maxb (known before the kernel runs)
  u64 *rows;       // 65536 x {bytes, items, tips, large}, one row per bucket
  u64 *totals;     // the emitter's totals: [4..12] w counts and [13] ones are added here
  u32 maxb;        // emit2_max_item_bytes(k)
};

// Record t (in sorted order) of the bucket staged in shared memory: s_rec read through s_perm.  A (k-1)-mer group
// never leaves its bucket (k - 1 >= 8), so the emitter's group walk needs nothing outside it.
template <int W>
struct BucketRecs {
  const u32 *rec;
  const uint16_t *perm;
  __device__ __forceinline__ void get(u32 t, u32 (&r)[W]) const {
    const u32 *p = rec + (u32)perm[t] * W;
#pragma unroll
    for (int j = 0; j < W; ++j) r[j] = p[j];
  }
};

// EMIT part of k_s2s_local_sort for one sorted bucket of n items (staged at rec, in sorted order through perm):
// thread tid owns sorted positions tid * IPT .. +IPT and walks the groups that start there to their end, as k_s2s_judge
// does, and the bucket's row is written.  One walk: every thread writes its items to its own SLOT bytes of s_out (the
// dead key array) while it counts them; a block scan of the sizes places them, and each thread copies its bytes to the
// bucket's staging slot.  (Two walks - sizes, scan, then writes straight to the staging slot - would cost twice the
// walk.)  Only when some thread's items do not fit its SLOT bytes does the block walk a second time, writing straight
// to the staging slot.
template <int W, int THREADS, int IPT, u32 SLOT>
__device__ __forceinline__ void ls_emit_bucket(const u32 *rec, const uint16_t *perm, u32 n, const u64 *bounds, u32 k, u32 *s_scan,
                                               u32 *s_w, uint8_t *s_out, const LsEmit &eo) {
  const u32 tid = threadIdx.x;
  const BucketRecs<W> br{rec, perm};
  const u32 p0 = tid * IPT, p1 = min(p0 + IPT, n);
  u32 first = p1;
  if (p0 < p1) {
    u32 p[W], c[W];
    if (p0 > 0) br.get(p0 - 1, p);
    for (u32 t = p0; t < p1; ++t) {
      br.get(t, c);
      if (t == 0 || diff_km1<W>(p, c, k)) {
        first = t;
        break;
      }
#pragma unroll
      for (int q = 0; q < W; ++q) p[q] = c[q];
    }
  }
  // the walk: items into this thread's slot (w and `last` counted here, once)
  EmitAcc acc = {0, 0, 0, 0};
  u32 ones = 0;
  uint8_t *mine = s_out + tid * SLOT;
  for (u32 t = first; t < p1;) t = s2s_group2<W, true>(br, n, t, k, acc, mine, s_w, ones, 0u, SLOT);
  for (int d = 16; d; d >>= 1) ones += __shfl_xor_sync(0xffffffffu, ones, d);
  if (lane_id() == 0 && ones) atomicAdd(&s_w[9], ones);
  const bool overflow = __syncthreads_or(acc.bytes > SLOT);
  // block prefixes of {bytes, items} and totals of {tips, large}
  u32 tot_bi, tot_tl;
  const u32 pre_bi = block_excl_scan<THREADS>((acc.bytes << 14) | acc.items, s_scan, tot_bi);
  block_excl_scan<THREADS>((acc.tips << 16) | acc.large, s_scan, tot_tl);
  const u32 b = rec[0] >> 16;  // re-derived here, not held through the sort (its registers are at their limit there)
  uint8_t *dst = eo.stage + bounds[b] * eo.maxb + (pre_bi >> 14);
  if (!overflow) {
    const uint16_t *src = reinterpret_cast<const uint16_t *>(mine);
    uint16_t *d = reinterpret_cast<uint16_t *>(dst);
    for (u32 x = 0; x < acc.bytes / 2; ++x) d[x] = src[x];
  } else {  // walk again, straight to the staging slot; w and `last` go to throw-away counters (counted above)
    EmitAcc wacc = {0, 0, 0, 0};
    u32 unused = 0;
    for (u32 t = first; t < p1;) t = s2s_group2<W, true>(br, n, t, k, wacc, dst, s_w + 10, unused, 0u);
  }
  if (tid == 0) {
    u64 *row = eo.rows + 4ull * b;
    row[0] = tot_bi >> 14;
    row[1] = tot_bi & 0x3FFFu;
    row[2] = tot_tl >> 16;
    row[3] = tot_tl & 0xFFFFu;
  }
}

// ids == nullptr: buckets 0 .. 65535; else the n_ids buckets listed there.  mid != nullptr: buckets of more than CAP
// but at most kLsCapL items are appended to `mid` (for the large geometry) instead of being left to the engine.
// EMIT = false writes every sorted bucket to `out`.  EMIT = true writes no records (`in` stays a permutation of the
// items): it walks the sorted bucket's (k-1)-mer groups out of shared memory as k_s2s_judge does, writes their item
// bytes to the bucket's staging slot and the bucket's row (a zero row for an empty bucket), and adds the w counts and
// ones to eo.totals.  Buckets it passes on (mid) or leaves to the engine get their row from whoever finishes them.
template <int W, u32 CAP, int THREADS, bool EMIT>
__global__ void __launch_bounds__(THREADS, CAP == kLsCapS ? 2 : 1)
    k_s2s_local_sort(const u32 *__restrict__ in, u32 *__restrict__ out, const u64 *__restrict__ bounds, u32 k, LsCtl *ctl,
                     unsigned int *ticket, const u32 *__restrict__ ids, u32 n_ids, u32 *mid, LsEmit eo) {
  constexpr u32 kLsCap = CAP;
  constexpr int kLsThreads = THREADS;
  constexpr int kLsIpt = CAP / THREADS;  // items per thread
  // EMIT packs {bytes, items} of a bucket into one 32-bit scan: items <= 8192 < 2^14, bytes <= 8192 x 16 = 2^17
  static_assert(kLsCapL <= (1u << 13), "bucket item count must fit the packed emit scan");
  extern __shared__ __align__(16) unsigned char smem_ls[];
  u64 *s_key = reinterpret_cast<u64 *>(smem_ls);                  // keys in group order
  u32 *s_rec = reinterpret_cast<u32 *>(s_key + kLsCap);           // the bucket's records (from a 16-byte boundary)
  u32 *s_grp = s_rec + kLsCap * W + 4;                            // group counts, then group starts (+ end)
  uint16_t *s_src = reinterpret_cast<uint16_t *>(s_grp + kLsDigits + 4);  // record of each key in s_key
  uint16_t *s_perm = s_src + kLsCap;                                      // record at each output position
  __shared__ u32 s_ticket;
  __shared__ u32 s_scan[kLsThreads / 32 + 1];
  __shared__ u32 s_w[19];  // EMIT: w counts of this CTA, its items with `last` set, throw-away w counts
  const u32 tid = threadIdx.x;
  const u32 n_units = ids ? n_ids : (u32)MHB_NUM_BUCKETS;
  if (EMIT && tid < 10) s_w[tid] = 0;
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
        if constexpr (!EMIT) {
          // ---- write the bucket in order: coalesced word stores ----
          for (u32 x = tid; x < n * W; x += kLsThreads) {
            const u32 i = x / W, j = x - i * W;
            out[w_begin + x] = s_rec[off + (u32)s_perm[i] * W + j];
          }
        } else {
          ls_emit_bucket<W, kLsThreads, kLsIpt, kLsCap * 8 / kLsThreads>(s_rec + off, s_perm, n, bounds, k, s_scan, s_w,
                                                                    reinterpret_cast<uint8_t *>(s_key), eo);
        }
      }
    } else if (EMIT && local && tid == 0) {  // an empty bucket
      u64 *row = eo.rows + 4ull * b;
      row[0] = row[1] = row[2] = row[3] = 0;
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
  if constexpr (EMIT) {  // (the loop ended on a barrier)
    if (tid < 10 && s_w[tid]) atomicAdd((unsigned long long *)&eo.totals[4 + tid], (unsigned long long)s_w[tid]);
  }
}

// One bucket left to the engine, sorted as a segment and emitted by mhb_s2s_emit on its own (side table and totals):
// its totals become the bucket's row, its w counts and ones are added to the totals.  seg: the sorted segment (every
// record in the bucket).
__global__ void k_s2s_fold_bucket(const u64 *__restrict__ side_totals, const u32 *__restrict__ seg, u64 *rows, u64 *totals) {
  const u32 t = threadIdx.x, b = seg[0] >> 16;
  if (t < 4) rows[4ull * b + t] = side_totals[t];
  else if (t < 14 && side_totals[t]) atomicAdd((unsigned long long *)&totals[t], (unsigned long long)side_totals[t]);
}

// block-wide sum of one u64 per thread (THREADS = 256)
__device__ __forceinline__ u64 block_sum_u64(u64 v, u64 *s_warp /*8*/) {
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();
  if (lane_id() == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  u64 t = 0;
  for (int w = 0; w < 8; ++w) t += s_warp[w];
  return t;
}

// The 65 536 rows {bytes, items, tips, large} -> bucket_table {byte offset, items, tips, large} and totals[0..3], as
// k_bucket_finalize leaves them: a row for every bucket with items (every bucket with sort items has some: each
// (k-1)-mer group emits at least one), zeros for the others.  Two launches of 256 blocks x 256 buckets: the block sums
// of the four columns, then every block scans its buckets behind the sum of the blocks before it.
constexpr int kRowBlocks = MHB_NUM_BUCKETS / 256;
__global__ void __launch_bounds__(256) k_s2s_row_sums(const u64 *__restrict__ rows, u64 *__restrict__ bsum /*4 x 256*/) {
  __shared__ u64 s_warp[8];
  const u64 *r = rows + 4ull * (blockIdx.x * 256 + threadIdx.x);
  for (int q = 0; q < 4; ++q) {
    const u64 t = block_sum_u64(r[q], s_warp);
    if (threadIdx.x == 0) bsum[q * kRowBlocks + blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256)
    k_s2s_bucket_table(const u64 *__restrict__ rows, const u64 *__restrict__ bsum, u64 *__restrict__ bucket_table, u64 *totals) {
  __shared__ u64 s_warp[8];
  __shared__ u64 s_scan[257];
  const u32 t = threadIdx.x, b = blockIdx.x * 256 + t;
  // bytes before this block; block 0 also reports the four totals
  u64 base = block_sum_u64(t < blockIdx.x ? bsum[t] : 0ull, s_warp);
  if (blockIdx.x == 0)
    for (int q = 0; q < 4; ++q) {
      const u64 tot = block_sum_u64(bsum[q * kRowBlocks + t], s_warp);
      if (t == 0) totals[q] = tot;
    }
  const u64 *r = rows + 4ull * b;
  const u64 nb = r[0], items = r[1];
  // exclusive scan of the bytes inside the block (Hillis-Steele in shared memory; 256 values)
  s_scan[t + 1] = nb;
  if (t == 0) s_scan[0] = 0;
  __syncthreads();
  for (u32 d = 1; d < 256; d <<= 1) {
    const u64 v = t + 1 > d ? s_scan[t + 1 - d] : 0ull;
    __syncthreads();
    s_scan[t + 1] += v;
    __syncthreads();
  }
  u64 *o = bucket_table + 4ull * b;
  o[0] = items ? base + s_scan[t] : 0;
  o[1] = items;
  o[2] = items ? r[2] : 0;
  o[3] = items ? r[3] : 0;
}

// Copy every bucket's item bytes from its staging slot to its offset in the stream, one warp per bucket; a bucket that
// would end past `capacity` is not copied (the totals still report the whole stream).  All sizes and offsets are even.
__global__ void __launch_bounds__(256)
    k_s2s_bucket_gather(const uint8_t *__restrict__ stage, const u64 *__restrict__ bounds, u32 maxb, const u64 *__restrict__ rows,
                        const u64 *__restrict__ bucket_table, uint8_t *__restrict__ out, u64 capacity) {
  const u32 b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = lane_id();
  const u64 nb = rows[4ull * b], off = bucket_table[4ull * b];
  if (nb == 0 || off + nb > capacity) return;
  const uint16_t *src = reinterpret_cast<const uint16_t *>(stage + bounds[b] * maxb);
  uint16_t *dst = reinterpret_cast<uint16_t *>(out + off);
  for (u64 x = lane; x < nb / 2; x += 32) dst[x] = src[x];
}

bool s2s_local_path(uint32_t k) {
  const u32 w = s2s_record_words(k);
  return k >= 9 && (w == 2 || w == 3);
}

// ids / n_ids / mid / eo: as k_s2s_local_sort
template <int W, u32 CAP, int THREADS, bool EMIT>
int launch_local_sort(cudaStream_t st, const u32 *in, u32 *out, const u64 *bounds, u32 k, LsCtl *ctl, unsigned int *ticket,
                      const u32 *ids, u32 n_ids, u32 *mid, const LsEmit &eo) {
  constexpr size_t smem = ls_smem<W, CAP>();
  static int bps = 0;
  if (!bps) {
    CK(cudaFuncSetAttribute(k_s2s_local_sort<W, CAP, THREADS, EMIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_s2s_local_sort<W, CAP, THREADS, EMIT>, THREADS, smem));
    if (bps < 1) return mhb_set_error(MHB_ERR_CUDA, "bucket sort kernel (W=%d, capacity %u) does not fit an SM", W, CAP);
    if (getenv("MHB_VERBOSE"))
      fprintf(stderr, "[mhb] s2s bucket %s W=%d: %d threads, capacity %u, %zu B smem, %d CTA/SM\n", EMIT ? "sort+emit" : "sort", W,
              THREADS, CAP, smem, bps);
  }
  const u32 units = ids ? n_ids : (u32)MHB_NUM_BUCKETS;
  const int grid = (int)std::min<u64>((u64)bps * sm_count(), units);
  k_s2s_local_sort<W, CAP, THREADS, EMIT><<<grid, THREADS, smem, st>>>(in, out, bounds, k, ctl, ticket, ids, n_ids, mid, eo);
  CK_LAUNCH();
  return MHB_OK;
}

template <int W, bool EMIT>
int launch_local(cudaStream_t st, bool large, const u32 *in, u32 *out, const u64 *bounds, u32 k, LsCtl *ctl, unsigned int *ticket,
                 const u32 *ids, u32 n_ids, u32 *mid, const LsEmit &eo) {
  if (large) return launch_local_sort<W, kLsCapL, kLsThreadsL, EMIT>(st, in, out, bounds, k, ctl, ticket, ids, n_ids, nullptr, eo);
  return launch_local_sort<W, kLsCapS, kLsThreadsS, EMIT>(st, in, out, bounds, k, ctl, ticket, ids, n_ids, mid, eo);
}

template <bool EMIT>
int launch_local_w(cudaStream_t st, u32 W, bool large, const u32 *in, u32 *out, const u64 *bounds, u32 k, LsCtl *ctl,
                   unsigned int *ticket, const u32 *ids, u32 n_ids, u32 *mid, const LsEmit &eo) {
  return W == 2 ? launch_local<2, EMIT>(st, large, in, out, bounds, k, ctl, ticket, ids, n_ids, mid, eo)
                : launch_local<3, EMIT>(st, large, in, out, bounds, k, ctl, ticket, ids, n_ids, mid, eo);
}

bool s2s_bucket_path(uint64_t n, uint32_t k) { return s2s_local_path(k) && n <= kLsMaxItems; }

// what the bucket kernel of the last mhb_s2s_sort left to the engine (mhb_s2s_sort_stats)
LsCtl g_last_ctl;

// Steps 1-3 of the bucket path, shared by mhb_s2s_sort and mhb_s2s_sort_emit (n >= 1, workspace and alignment
// checked): the two bucket passes, the bucket bounds and the bucket kernel(s) over x.  eo == nullptr: the sorted buckets
// go to y; else they are emitted (LsEmit) and y is not written.  *h: what the bucket kernel(s) left over.
struct BucketStage {
  u32 *x, *y;    // the items after the two passes, the other buffer
  u64 *bounds;   // 65 537 bucket boundaries in x
  LsCtl h;
};
int bucket_stage(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t k, const uint64_t *first_hist, void *ws,
                 const LsEmit *eo, BucketStage *bs) {
  const uint32_t W = s2s_record_words(k);
  const size_t sort_ws = mhb_sort_workspace_bytes(n, W);
  cudaStream_t st = (cudaStream_t)stream;
  // 1. the two bucket bytes (the only entry of this sort in the timing ring)
  const uint8_t top[2] = {(uint8_t)(4 * W - 2), (uint8_t)(4 * W - 1)};
  int in_b = 0;
  if (int rc = mhb_sort_records_ex(stream, a, b, n, W, top, 2, first_hist, ws, sort_ws, &in_b, nullptr, 1)) return rc;
  u32 *x = in_b ? b : a, *y = in_b ? a : b;
  // 2. bucket bounds, 3. buckets in shared memory (small geometry first unless the buckets average more than 3/4 of
  // it; the buckets it cannot hold but the large one can go to a second launch of the large one)
  u64 *bounds = reinterpret_cast<u64 *>((char *)ws + pad256(sort_ws));
  LsCtl *ctl = reinterpret_cast<LsCtl *>((char *)bounds + pad256((size_t)(MHB_NUM_BUCKETS + 1) * 8));
  u32 *mid = reinterpret_cast<u32 *>((char *)ctl + pad256(sizeof(LsCtl)));
  CK(cudaMemsetAsync(ctl, 0, sizeof(LsCtl), st));
  if (W == 2) k_bucket_bounds<2><<<(65537 + 255) / 256, 256, 0, st>>>(x, n, bounds);
  else k_bucket_bounds<3><<<(65537 + 255) / 256, 256, 0, st>>>(x, n, bounds);
  CK_LAUNCH();
  const bool large = n > kLsSmallMaxItems;
  const LsEmit none{};
  auto launch = [&](bool lg, unsigned int *ticket, const u32 *ids, u32 n_ids, u32 *m) {
    return eo ? launch_local_w<true>(st, W, lg, x, nullptr, bounds, k, ctl, ticket, ids, n_ids, m, *eo)
              : launch_local_w<false>(st, W, lg, x, y, bounds, k, ctl, ticket, ids, n_ids, m, none);
  };
  if (int rc = launch(large, &ctl->ticket, nullptr, 0, mid)) return rc;
  // 4. what the bucket kernel left over
  LsCtl &h = bs->h;
  CK(cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (h.n_mid) {
    if (int rc = launch(true, &ctl->ticket2, mid, h.n_mid, nullptr)) return rc;
    CK(cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  g_last_ctl = h;
  bs->x = x;
  bs->y = y;
  bs->bounds = bounds;
  return MHB_OK;
}

// mhb_s2s_sort_emit: the bucket rows and the staging area behind the sort workspace
size_t fused_rows_bytes() { return pad256((size_t)MHB_NUM_BUCKETS * 4 * 8); }
constexpr size_t kBlockSumBytes = 4 * kRowBlocks * 8;  // k_s2s_row_sums
size_t fused_stage_bytes(uint64_t n, uint32_t k) { return pad256((size_t)n * emit2_max_item_bytes(k)); }
// an oversized bucket of s items is emitted in the other buffer: side table, side totals, emit scratch
size_t side_bytes(uint64_t s, uint32_t k) { return fused_rows_bytes() + 256 + mhb_s2s_emit_scratch_bytes(s, k); }

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
  BucketStage bs;
  if (int rc = bucket_stage(stream, a, b, n, k, first_hist, ws, nullptr, &bs)) return rc;
  u32 *x = bs.x, *y = bs.y;
  const LsCtl &h = bs.h;
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

extern "C" size_t mhb_s2s_sort_emit_workspace_bytes(uint64_t n, uint32_t k) {
  const size_t sort_ws = pad256(mhb_s2s_sort_workspace_bytes(n, k)), emit = mhb_s2s_emit_scratch_bytes(n, k);
  if (!s2s_bucket_path(n, k)) return sort_ws + emit;
  // the bucket path's rows and staging area, or (oversized buckets beyond the list) the whole-array emitter's scratch
  return sort_ws + std::max(emit, fused_rows_bytes() + fused_stage_bytes(n, k) + kBlockSumBytes);
}

extern "C" int mhb_s2s_sort_emit(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t k, const uint64_t *first_hist,
                                 uint8_t *bytes_out, uint64_t capacity_bytes, uint64_t *bucket_table, uint64_t *totals, void *ws,
                                 size_t ws_bytes) {
  if (k < 1 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "bad seq2sdbg sort arguments (k=%u)", k);
  if (ws_bytes < mhb_s2s_sort_emit_workspace_bytes(n, k)) return mhb_set_error(MHB_ERR_ARG, "seq2sdbg sort+emit workspace too small");
  const size_t sws = pad256(mhb_s2s_sort_workspace_bytes(n, k));
  char *scratch = (char *)ws + sws;
  const size_t scratch_bytes = ws_bytes - sws;
  if (!s2s_bucket_path(n, k) || n == 0) {  // the sort, then the emitter
    int in_b = 0;
    if (int rc = mhb_s2s_sort(stream, a, b, n, k, first_hist, ws, sws, &in_b)) return rc;
    return mhb_s2s_emit(stream, in_b ? b : a, n, k, bytes_out, capacity_bytes, bucket_table, totals, scratch, scratch_bytes);
  }
  if (!bucket_table || !totals) return mhb_set_error(MHB_ERR_ARG, "bad args");
  if ((((uintptr_t)a | (uintptr_t)b) & 15) != 0) return mhb_set_error(MHB_ERR_ARG, "seq2sdbg sort buffers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const uint32_t W = s2s_record_words(k);
  uint8_t bytes[80];
  const uint32_t nb = mhb_s2s_sort_bytes(k, bytes);
  const size_t sort_ws = mhb_sort_workspace_bytes(n, W);
  const LsEmit eo{(uint8_t *)scratch + fused_rows_bytes(), (u64 *)scratch, totals, emit2_max_item_bytes(k)};
  CK(cudaMemsetAsync(totals, 0, 16 * 8, st));
  BucketStage bs;
  if (int rc = bucket_stage(stream, a, b, n, k, first_hist, ws, &eo, &bs)) return rc;
  u32 *x = bs.x, *y = bs.y;
  const LsCtl &h = bs.h;
  if (h.n_over) {
    u64 s_max = 0;
    for (u32 s = 0; s < std::min(h.n_over, kLsListCap); ++s) s_max = std::max<u64>(s_max, h.range[2 * s + 1] - h.range[2 * s]);
    if (h.n_over > kLsListCap || side_bytes(s_max, k) > (size_t)n * W * 4) {
      // more buckets than the list holds, or too large to emit in the other buffer: the whole array is sorted again
      // (the bucket kernel left x a permutation of the items) and emitted by the whole-array emitter
      int r_in_b = 0;
      if (int rc = mhb_sort_records_untraced(stream, x, y, n, W, bytes, nb, nullptr, ws, sort_ws, &r_in_b)) return rc;
      return mhb_s2s_emit(stream, r_in_b ? y : x, n, k, bytes_out, capacity_bytes, bucket_table, totals, scratch, scratch_bytes);
    }
    // every listed bucket: sorted as a segment (back in x), emitted into its staging slot with side table and totals
    // in y, folded into its row and the totals
    u64 *side_table = reinterpret_cast<u64 *>(y);
    u64 *side_totals = reinterpret_cast<u64 *>((char *)y + fused_rows_bytes());
    char *side_scratch = (char *)side_totals + 256;
    for (u32 s = 0; s < h.n_over; ++s) {
      const u64 lo = h.range[2 * s], hi = h.range[2 * s + 1];
      int r_in_b = 0;
      if (int rc = mhb_sort_records_untraced(stream, x + lo * W, y + lo * W, hi - lo, W, bytes, nb - 2, nullptr, ws, sort_ws, &r_in_b)) return rc;
      if (r_in_b) CK(cudaMemcpyAsync(x + lo * W, y + lo * W, (hi - lo) * W * 4, cudaMemcpyDeviceToDevice, st));
      if (int rc = mhb_s2s_emit(stream, x + lo * W, hi - lo, k, eo.stage + lo * eo.maxb, (hi - lo) * eo.maxb, side_table,
                                side_totals, side_scratch, mhb_s2s_emit_scratch_bytes(hi - lo, k))) return rc;
      k_s2s_fold_bucket<<<1, 32, 0, st>>>(side_totals, x + lo * W, eo.rows, totals);
      CK_LAUNCH();
    }
  }
  // the bucket table, the totals, and every bucket's bytes at their offset (block sums behind the staging area)
  u64 *bsum = reinterpret_cast<u64 *>(eo.stage + fused_stage_bytes(n, k));
  k_s2s_row_sums<<<kRowBlocks, 256, 0, st>>>(eo.rows, bsum);
  CK_LAUNCH();
  k_s2s_bucket_table<<<kRowBlocks, 256, 0, st>>>(eo.rows, bsum, bucket_table, totals);
  CK_LAUNCH();
  k_s2s_bucket_gather<<<MHB_NUM_BUCKETS / 8, 256, 0, st>>>(eo.stage, bs.bounds, eo.maxb, eo.rows, bucket_table, bytes_out, capacity_bytes);
  CK_LAUNCH();
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
