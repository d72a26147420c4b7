// mhb_kernels.cuh -- device-side building blocks (sm_90a) shared by the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mhb_bits.cuh"

namespace mhb {

static constexpr u32 kSentinel = 4;  // kmer_counter.h:48 kSentinelValue

// ------------------------------------------------------------------------------------------------
// record builders (host+device so they can be unit-tested on the CPU against the oracle)
// ------------------------------------------------------------------------------------------------

// `count` sort record for the (k+1)-mer starting at FILE-orientation position q of a read of L bases
// whose packed words start at s (nwords words).  KmerCounter works on the REVERSED read
// (kmer_counter.cpp:61,72): with S = read[q, q+k+1), the package-orientation forward edge is
// reverse(S) and its reverse complement is complement(S); package offset = L-(k+1)-q.
// Record = canonical edge (kmer_counter.cpp:182: rc < fwd ? rc : fwd) left-aligned in WR words with
// prev<<3|next in the low 6 bits of the last word (prev/next as kmer_counter.cpp:223-248).
template <int W, int WR>
MHB_HD void make_count_record(const u32 *s, u32 nwords, u32 L, u32 k, u32 q, u32 (&rec)[WR], u32 &strand) {
  const u32 K1 = k + 1;
  u32 prev_pkg, next_pkg;
  bool st;
  if constexpr (W == 2) {
    // 17 <= k+1 <= 32: the whole edge fits one 64-bit word -- same arithmetic as the generic path below
    const u32 w0 = q >> 4, sh = (q & 15) * 2;
    const u32 x0 = s[w0];
    const u32 x1 = (w0 + 1 < nwords) ? s[w0 + 1] : 0u;
    const u32 x2 = (w0 + 2 < nwords) ? s[w0 + 2] : 0u;
    // neighbours from the words already in registers: base q+K1 lives in word w0+1 or w0+2, base q-1 in w0 or w0-1
    const u32 pi = q + K1;
    const u32 pw = ((pi >> 4) == w0 + 1) ? x1 : x2;
    prev_pkg = (pi < L) ? ((pw >> (30 - 2 * (pi & 15))) & 3u) : kSentinel;
    const u32 nwd = (q & 15) ? x0 : (q ? s[w0 - 1] : 0u);
    next_pkg = (q > 0) ? ((nwd >> (30 - 2 * ((q - 1) & 15))) & 3u) : kSentinel;
    const u32 T = 64u - 2u * K1;  // zero bits below the edge, 0..30
    const u64 S = ((((u64)fshl(x0, x1, sh) << 32) | fshl(x1, x2, sh)) >> T) << T;
    const u64 B = ((~S) >> T) << T;                                      // complement(S)
    const u64 A = (((u64)rev2((u32)S) << 32) | rev2((u32)(S >> 32))) << T;  // reverse(S)
    st = B < A;
    const u64 key = st ? B : A;
    rec[0] = (u32)(key >> 32);
    rec[1] = (u32)key;
    if constexpr (WR == 3) rec[2] = 0u;
  } else {
    prev_pkg = (q + K1 < L) ? base_at(s, q + K1) : kSentinel;
    next_pkg = (q > 0) ? base_at(s, q - 1) : kSentinel;
    u32 S[W], A[W], B[W];
    load_sub<W>(s, nwords, q, K1, S);
    reverse_sub<W>(S, K1, A);
    complement_sub<W>(S, K1, B);
    st = less_words<W>(B, A);
#pragma unroll
    for (int j = 0; j < WR; ++j) rec[j] = j < W ? (st ? B[j] : A[j]) : 0u;
  }
  u32 p = prev_pkg, n = next_pkg;
  if (st) {
    p = next_pkg == kSentinel ? kSentinel : 3u - next_pkg;
    n = prev_pkg == kSentinel ? kSentinel : 3u - prev_pkg;
  }
  rec[WR - 1] |= (p << 3) | n;
  strand = st ? 1u : 0u;
}

// The same records for R consecutive positions q, q+1, .., q+R-1 of one read, 17 <= k+1 <= 32 (8-byte records): the
// first one is built from the packed words, every further one by ROLLING the three 64-bit strings one base on
// (S = read[q, q+k+1) left-aligned, A = reverse(S), B = complement(S)):  S' = S<<2 | b<<T,  B' = B<<2 | (3-b)<<T,
// A' = (A>>2 with the dropped base cleared) | b<<62,  b = read[q+k+1], T = 64 - 2(k+1); prev of position q is that
// same b, next of position q+1 is the top base of S.  ~35 instructions per extra record instead of ~120 from scratch.
// rec[j] = record word 0 << 32 | word 1 exactly as make_count_record<2, 2> builds them; only the first `cnt` entries
// (positions that exist, q + j + k + 1 <= L) are meaningful.
template <int R>
MHB_HD void make_count_records_roll(const u32 *s, u32 nwords, u32 L, u32 k, u32 q, u64 (&rec)[R], u32 (&strand)[R]) {
  const u32 K1 = k + 1;
  const u32 T = 64u - 2u * K1;  // zero bits below the edge, 0..30
  const u32 w0 = q >> 4, sh = (q & 15) * 2;
  const u32 x0 = s[w0];
  const u32 x1 = (w0 + 1 < nwords) ? s[w0 + 1] : 0u;
  const u32 x2 = (w0 + 2 < nwords) ? s[w0 + 2] : 0u;
  const u32 x3 = (w0 + 3 < nwords) ? s[w0 + 3] : 0u;
  u64 S = ((((u64)fshl(x0, x1, sh) << 32) | fshl(x1, x2, sh)) >> T) << T;
  u64 B = ((~S) >> T) << T;                                            // complement(S)
  u64 A = (((u64)rev2((u32)S) << 32) | rev2((u32)(S >> 32))) << T;     // reverse(S)
  // look-ahead: the bases from position q + K1 on, left-aligned in 32 bits (R <= 8 of them are used)
  const u32 pi = q + K1;
  const u32 wa = (pi >> 4) - w0;  // 1 or 2, because 17 <= (q & 15) + K1 <= 47
  u32 LA = fshl(wa == 1 ? x1 : x2, wa == 1 ? x2 : x3, (pi & 15) * 2);
  u32 next_pkg = (q > 0) ? (((q & 15) ? (x0 >> (32 - sh)) : s[w0 - 1]) & 3u) : kSentinel;  // base q - 1
  const u64 lowmask = ~((1ull << T) - 1ull);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const u32 b = LA >> 30;                                  // read[q + j + K1] if it exists
    const u32 prev_pkg = (pi + j < L) ? b : kSentinel;
    const bool st = B < A;
    const u64 key = st ? B : A;
    u32 p = prev_pkg, n = next_pkg;
    if (st) {
      p = next_pkg == kSentinel ? kSentinel : 3u - next_pkg;
      n = prev_pkg == kSentinel ? kSentinel : 3u - prev_pkg;
    }
    rec[j] = key | (u64)((p << 3) | n);
    strand[j] = st ? 1u : 0u;
    // roll on to position q + j + 1
    next_pkg = (u32)(S >> 62);
    S = (S << 2) | ((u64)b << T);
    B = (B << 2) | ((u64)(3u - b) << T);
    A = ((A >> 2) & lowmask) | ((u64)b << 62);
    LA <<= 2;
  }
}

// seq2sdbg sort record (seq_to_sdbg.cpp:630-700) for item `offset` of strand `strand` of a
// package-orientation sequence.  W = s2s_record_words(k).
template <int W>
MHB_HD void make_s2s_record(const u32 *s, u32 nwords, u32 L, u32 k, u32 strand, u32 offset, u32 mult,
                            u32 (&rec)[W]) {
  const u32 nc = k - ((offset + k > L) ? 1u : 0u);
  const u32 counting = (offset > 0 && offset + k <= L) ? mult : 0u;  // :641-643
  u32 prev;
  if (strand == 0) {
    prev = offset == 0 ? kSentinel : base_at(s, offset - 1);
    load_sub<W>(s, nwords, offset, nc, rec);
  } else {
    prev = offset == 0 ? kSentinel : 3u - base_at(s, L - offset);  // :678
    int off2 = (int)L - (int)k - (int)offset;                       // :681
    if (off2 < 0) off2 = 0;                                         // :683-686
    u32 S[W], T[W];
    load_sub<W>(s, nwords, (u32)off2, nc, S);
    reverse_sub<W>(S, nc, T);
    complement_sub<W>(T, nc, rec);
  }
  rec[W - 1] |= ((nc == k) ? 1u : 0u) << 19;  // :664-670
  rec[W - 1] |= prev << 16;
  rec[W - 1] |= 65535u - counting;
}

// Key of a seq2sdbg sort record INSIDE its 16-bit bucket (the first eight bases): the 2k - 16 key bits below the
// bucket followed by the four flag bits (non-dollar, prev), left-aligned in 64 bits.  Comparing these keys orders two
// records of one bucket exactly as mhb_s2s_sort_bytes does: the zero fill between the k-mer and the flags is constant
// and the multiplicity bits are not sorted.  9 <= k <= 38 (W = 2 or 3): 2k - 12 <= 64 bits.
template <int W>
MHB_HD u64 s2s_local_key(const u32 (&r)[W], u32 k) {
  u32 w2 = 0;
  if constexpr (W >= 3) w2 = r[2];
  const u64 top = ((u64)r[0] << 48) | ((u64)r[1] << 16) | (w2 >> 16);  // the record from bit 16 on
  const u32 kb = 2 * k - 16;
  const u64 flags = (r[W - 1] >> 16) & 15u;
  return (top & ~(~0ull >> kb)) | (flags << (60 - kb));
}

#if defined(__CUDACC__)
// ------------------------------------------------------------------------------------------------
// record load/store (AoS, WR words; 8- and 16-byte records use vector accesses)
// ------------------------------------------------------------------------------------------------
template <int WR>
__device__ __forceinline__ void ld_rec(const u32 *base, u64 idx, u32 (&r)[WR]) {
  // records start at multiples of their own size in buffers that are at least 16-byte aligned: widths that are a
  // multiple of 4 (2) words move as 128-bit (64-bit) pieces - one access per 16 (8) bytes instead of per word
  if constexpr (WR % 4 == 0) {
    const uint4 *p = reinterpret_cast<const uint4 *>(base + idx * WR);
#pragma unroll
    for (int j = 0; j < WR / 4; ++j) {
      const uint4 v = p[j];
      r[4 * j] = v.x;
      r[4 * j + 1] = v.y;
      r[4 * j + 2] = v.z;
      r[4 * j + 3] = v.w;
    }
  } else if constexpr (WR % 2 == 0) {
    const uint2 *p = reinterpret_cast<const uint2 *>(base + idx * WR);
#pragma unroll
    for (int j = 0; j < WR / 2; ++j) {
      const uint2 v = p[j];
      r[2 * j] = v.x;
      r[2 * j + 1] = v.y;
    }
  } else {
    const u32 *p = base + idx * WR;
#pragma unroll
    for (int j = 0; j < WR; ++j) r[j] = p[j];
  }
}
template <int WR>
__device__ __forceinline__ void st_rec(u32 *base, u64 idx, const u32 (&r)[WR]) {
  if constexpr (WR % 4 == 0) {
    uint4 *p = reinterpret_cast<uint4 *>(base + idx * WR);
#pragma unroll
    for (int j = 0; j < WR / 4; ++j) p[j] = make_uint4(r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
  } else if constexpr (WR % 2 == 0) {
    uint2 *p = reinterpret_cast<uint2 *>(base + idx * WR);
#pragma unroll
    for (int j = 0; j < WR / 2; ++j) p[j] = make_uint2(r[2 * j], r[2 * j + 1]);
  } else {
    u32 *p = base + idx * WR;
#pragma unroll
    for (int j = 0; j < WR; ++j) p[j] = r[j];
  }
}

// byte b (0 = least significant byte of the last word) of a record, b warp-uniform
template <int WR>
__device__ __forceinline__ u32 rec_byte(const u32 (&r)[WR], int b) {
  return (pick<WR>(r, (u32)(WR - 1 - (b >> 2))) >> (8 * (b & 3))) & 255u;
}

// bounds[b] = first record whose 16-bit prefix (top half of word 0) is >= b, b = 0..65536; the W-word records are
// sorted on that prefix
template <int W>
__global__ void k_bucket_bounds(const u32 *__restrict__ recs, u64 n, u64 *__restrict__ bounds) {
  const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > 65536u) return;
  u64 lo = 0, hi = n;
  while (lo < hi) {
    const u64 mid = (lo + hi) >> 1;
    if ((recs[mid * W] >> 16) < b) lo = mid + 1;
    else hi = mid;
  }
  bounds[b] = lo;
}

__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ u32 lanemask_lt() {
  u32 m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// Where the extraction kernels of the multi-GPU stages put a warp's records (in = this lane holds one, mask = the ballot
// of `in`, lt = lanemask_lt; every lane of the warp calls put).  OwnerSink: record -> rank owner[leading record byte],
// stored at base[owner] + cursor[owner] (base[o] = this rank's segment of owner o's receive buffer, which may be another
// process's memory opened through CUDA IPC; the cursors are this rank's).  The lanes of a warp are grouped by owner;
// one atomic per group, each lane stores at the group's base plus its rank in the group.  Records beyond
// capacity[owner] are counted but not stored.
struct OwnerSink {
  const uint8_t *owner;  // 256 entries
  const u64 *base;       // device addresses, one per owner
  unsigned long long *cursor;
  const u64 *capacity;
  template <int W>
  __device__ __forceinline__ void put(bool in, const u32 (&rec)[W], u32, u32 lane, u32 lt) const {
    const u32 o = in ? (u32)__ldg(owner + (rec[0] >> 24)) : 0xFFFFFFFFu;
    const u32 peers = __match_any_sync(0xffffffffu, o);
    if (!in) return;
    const u32 leader = (u32)__ffs(peers) - 1;
    unsigned long long at = 0;
    if (lane == leader) at = atomicAdd(cursor + o, (unsigned long long)__popc(peers));
    at = __shfl_sync(peers, at, leader);
    const u64 pos = at + __popc(peers & lt);
    if (pos < capacity[o]) st_rec<W>(reinterpret_cast<u32 *>(base[o]), pos, rec);
  }
};

// ------------------------------------------------------------------------------------------------
// mbarrier + bulk async copy (TMA 1-D: cp.async.bulk, SASS UBLKCP)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, u32 bytes, u64 *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(u64 *bar, u32 parity) {
  u32 ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// relaxed gpu-scope 64-bit load/store for the decoupled look-back descriptors
__device__ __forceinline__ u64 ld_relaxed(const u64 *p) {
  u64 v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed(u64 *p, u64 v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// look-back descriptor: [63:62] status (0 invalid, 1 partial, 2 inclusive) [61:54] epoch [53:0] value
static constexpr u64 kLbPartial = 1ull << 62, kLbInclusive = 2ull << 62, kLbStatusMask = 3ull << 62;
static constexpr u64 kLbValueMask = (1ull << 54) - 1;
__host__ __device__ inline u64 lb_epoch(u32 e) { return (u64)(e & 255u) << 54; }

// block-wide exclusive scan of one u32 per thread (all THREADS threads must call)
template <int THREADS>
__device__ __forceinline__ u32 block_excl_scan(u32 v, u32 *s_warp /*THREADS/32 + 1*/, u32 &total) {
  const u32 lane = lane_id(), warp = threadIdx.x >> 5;
  u32 inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    u32 t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= (u32)d) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    u32 w = lane < THREADS / 32 ? s_warp[lane] : 0u;
    u32 winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      u32 t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= (u32)d) winc += t;
    }
    if (lane < THREADS / 32) s_warp[lane] = winc - w;
    if (lane == 31) s_warp[THREADS / 32] = winc;
  }
  __syncthreads();
  u32 res = s_warp[warp] + inc - v;
  total = s_warp[THREADS / 32];
  __syncthreads();
  return res;
}
#endif  // __CUDACC__

}  // namespace mhb
