// mhb_multi.cu -- device-level entry points used only by the multi-GPU build (one process per GPU; see
// megahit_b200/multigpu.py and include/mhb.h):
//
//   mhb_plan_partition        the bucket-range plan of a stage as ONE small kernel over the all-gathered top-byte
//                             histograms: owner ranges, owner look-up table, the byte address inside every owner's
//                             receive buffer where this rank's block starts, and the record counts each rank will own -
//                             no host round trip between the histogram all-gather and the fused partition+exchange pass
//   mhb_mercy_probe_owned     the mercy searches (seq_to_sdbg.cpp:171-357) of candidate reads of ALL ranks restricted to
//                             the edges THIS rank owns: every binary search of GenMercyEdges targets exactly one owner
//                             (edges sharing a 12-base prefix share their leading byte), and the has_in / has_out logic
//                             is an OR over search outcomes, so each rank answers the searches that land in its own
//                             bucket range from local HBM and the per-position answer bits are exchanged instead of
//                             the edges (instead of bisecting the peers' edge arrays over NVLink)
//   mhb_mercy_count_planes    OR the answer planes of all ranks into (A, O, N) and count the mercy edges
// The single-GPU mercy search of an edge array larger than device memory (mhb_mercy_host) runs the same probe once per
// leading-byte segment, OR-ing each segment's answers into one set of planes (mercy_probe_owned, accumulate = true).
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "mhb.h"
#include "mhb_common.cuh"
#include "mhb_count.cuh"
#include "mhb_mercy.cuh"

using namespace mhb;

// ------------------------------------------------------------------------------------------------
// partition plan
// ------------------------------------------------------------------------------------------------
namespace {

struct PlanArgs {
  u64 peer_base[16];  // byte address of every owner's receive buffer as seen from this rank
};

// hist_all[world][256]: top-byte histograms of every rank.  One thread: 256 x world additions are nothing.
// Cuts (same rule as multigpu.plan_ranges): bound r = the byte value whose cumulative count is closest to r/world of
// the total, leaving at least one value for every later rank.
__global__ void k_plan_partition(const u64 *__restrict__ hist_all, u32 world, u32 rank, u32 rec_bytes, PlanArgs pa,
                                 uint8_t *owner_lut, u64 *bin_addr, u64 *plan_out) {
  __shared__ u64 cum[257];
  __shared__ u32 bounds[17];
  if (threadIdx.x == 0) {
    u64 acc = 0;
    cum[0] = 0;
    for (u32 b = 0; b < 256; ++b) {
      for (u32 r = 0; r < world; ++r) acc += hist_all[(u64)r * 256 + b];
      cum[b + 1] = acc;
    }
    const u64 total = acc;
    bounds[0] = 0;
    for (u32 r = 1; r < world; ++r) {
      const u32 lo = bounds[r - 1] + 1, hi = 256 - (world - r);
      const u64 target = total * r / world;
      u32 best = lo;
      u64 bestd = ~0ull;
      for (u32 c = lo; c <= hi; ++c) {
        const u64 d = cum[c] > target ? cum[c] - target : target - cum[c];
        if (d < bestd) {
          bestd = d;
          best = c;
        }
      }
      bounds[r] = best;
    }
    bounds[world] = 256;
  }
  __syncthreads();
  const u32 t = threadIdx.x;
  if (t < 256) {
    u32 o = 0;
    while (t >= bounds[o + 1]) ++o;
    owner_lut[t] = (uint8_t)o;
  }
  __syncthreads();
  if (t < world) {
    // owner t: what every rank sends to it
    u64 before_me = 0, tot = 0, mine = 0;
    for (u32 r = 0; r < world; ++r) {
      u64 s = 0;
      for (u32 b = bounds[t]; b < bounds[t + 1]; ++b) s += hist_all[(u64)r * 256 + b];
      if (r < rank) before_me += s;
      if (r == rank) mine = s;
      tot += s;
    }
    bin_addr[t] = pa.peer_base[t] + before_me * rec_bytes;
    plan_out[t] = tot;          // records owner t receives in total
    plan_out[16 + t] = mine;    // records this rank sends to owner t
    plan_out[32 + t] = bounds[t];
  }
  if (t == 0) plan_out[32 + world] = 256;
}

}  // namespace

extern "C" int mhb_plan_partition(void *stream, const uint64_t *hist_all_dev, uint32_t world, uint32_t rank,
                                  uint32_t record_bytes, const uint64_t *peer_base_host, uint8_t *owner_lut_dev,
                                  uint64_t *bin_addr_dev, uint64_t *plan_dev) {
  if (!hist_all_dev || !peer_base_host || !owner_lut_dev || !bin_addr_dev || !plan_dev || world < 1 || world > 16 || rank >= world)
    return mhb_set_error(MHB_ERR_ARG, "bad partition plan arguments (world %u, rank %u)", world, rank);
  PlanArgs pa;
  memset(&pa, 0, sizeof(pa));
  for (u32 i = 0; i < world; ++i) pa.peer_base[i] = peer_base_host[i];
  k_plan_partition<<<1, 256, 0, (cudaStream_t)stream>>>(hist_all_dev, world, rank, record_bytes, pa, owner_lut_dev, bin_addr_dev,
                                                        plan_dev);
  CK_LAUNCH();
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// tip edges (aux != 0) of a rank, compacted for the exchange (order is irrelevant: they go into a hash set)
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void k_compact_tips(const u32 *__restrict__ edges, const uint8_t *__restrict__ aux, u64 n, u32 we,
                               u32 *__restrict__ tips, uint8_t *__restrict__ tip_aux, u64 capacity, unsigned long long *cursor) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const uint8_t a = aux[i];
    if (!a) continue;
    const u64 at = atomicAdd(cursor, 1ull);
    if (at >= capacity) continue;
    for (u32 w = 0; w < we; ++w) tips[at * we + w] = edges[i * we + w];
    tip_aux[at] = a;
  }
}
}  // namespace

extern "C" int mhb_compact_tip_edges(void *stream, const uint32_t *edges, const uint8_t *aux, uint64_t n_solid, uint32_t k,
                                     uint32_t *tips_out, uint8_t *tip_aux_out, uint64_t capacity, uint64_t *cursor_dev) {
  if (n_solid == 0) return MHB_OK;
  if (!edges || !aux || !tips_out || !tip_aux_out || !cursor_dev) return mhb_set_error(MHB_ERR_ARG, "null buffer");
  k_compact_tips<<<grid_cap(n_solid, 256, 16), 256, 0, (cudaStream_t)stream>>>(edges, aux, n_solid, words_per_edge(k), tips_out, tip_aux_out,
                                                              capacity, (unsigned long long *)cursor_dev);
  CK_LAUNCH();
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// mercy searches restricted to the owned bucket range
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kOwnedPlanes = 5;  // A' = any in-search hit, O' = any out-search hit, G1 = km hit, G1n = km hit and next base matches, G2

template <int WM>
struct OwnedOps {
  using Ops = MercyOps<WM>;
  // BinarySearchKmer inside this rank's edges when the query's leading byte is owned here, else "not mine"
  __device__ static const u32 *search(const u32 *edges, long long n, const uint2 *lut, const uint8_t *owner, u32 me, u32 we,
                                      const u32 (&km)[WM], u32 ksz) {
    if (owner[km[0] >> 24] != me || n == 0) return nullptr;
    const uint2 lr = lut[km[0] >> 8];
    if (lr.x == 0xFFFFFFFFu) return nullptr;
    long long l = lr.x, r = lr.y;
    while (l <= r) {
      const long long mid = (l + r) / 2;
      const int c = Ops::cmp(km, edges + mid * we, ksz);
      if (c > 0) l = mid + 1;
      else if (c < 0) r = mid - 1;
      else return edges + mid * we;
    }
    return nullptr;
  }
};

struct OwnerTab {
  uint8_t owner[256];
};

// Every search GenMercyEdges could issue for position i, evaluated unconditionally (seq_to_sdbg.cpp:225-298):
//   in :  F1 = S(rvk, k);  F2 = OR_ch S(ch + km, k+1) for ch = 0.. while (ch + km) <= rvk + 'T'
//   out:  G1 = S(km, k) (+ G1n: base k of the hit == next read base);  G2 = S(next' + rvk, k+1) if <= km + 'T';
//         G3 = OR_{ch != next'} S(ch + rvk, k+1) while <= km + 'T'
// With hits OR-ed over the owners:  A = F1|F2,  O = G1|G2|G3,  N = G1 ? G1n : G2  - identical to the reference's
// nested ifs because the else-branches only matter when the earlier search missed everywhere.
// Accumulate: OR the answers into planes already holding those of other segments (one edge array streamed through the
// device in leading-byte segments), instead of storing them.
template <int WM, bool Accumulate>
__global__ void __launch_bounds__(256)
    k_mercy_probe_owned(ReadsView rv, const u64 *__restrict__ cand_ids, u64 n_cand, u32 k, const u32 *__restrict__ edges,
                        long long n_edges, const uint2 *__restrict__ lut, OwnerTab ot, u32 me, u32 we, u32 *__restrict__ planes,
                        u32 words_per_read) {
  using Ops = MercyOps<WM>;
  using Own = OwnedOps<WM>;
  __shared__ uint8_t s_owner[256];
  s_owner[threadIdx.x] = ot.owner[threadIdx.x];
  __syncthreads();
  const u32 lane = lane_id();
  for (u64 c = (u64)blockIdx.x * 8 + (threadIdx.x >> 5); c < n_cand; c += (u64)gridDim.x * 8) {
    const u64 r = cand_ids ? cand_ids[c] : c;
    const u32 *rec0 = rv.bin + rv.rec_start(r);
    const u32 L = rec0[0];
    const u32 *s = rec0 + 1;
    const u32 nwords = div_ceil(L, 16);
    u32 *pl = planes + c * (u64)kOwnedPlanes * words_per_read;
    const u32 npos = L >= k + 2 ? L - k + 1 : 0;
    for (u32 i0 = 0; i0 < words_per_read * 32; i0 += 32) {
      const u32 i = i0 + lane;
      bool A = false, O = false, G1 = false, G1n = false, G2 = false;
      if (i < npos) {
        u32 S[WM], km[WM], rvk[WM];
        load_sub<WM>(s, nwords, L - i - k, k, S);
        reverse_sub<WM>(S, k, km);
        complement_sub<WM>(S, k, rvk);
        // ---- in-searches ----
        if (Own::search(edges, n_edges, lut, s_owner, me, we, rvk, k) != nullptr) A = true;
        {
          u32 rv1[WM], km1[WM];
#pragma unroll
          for (int j = 0; j < WM; ++j) rv1[j] = rvk[j];
          Ops::set_base(rv1, k, 3);
          Ops::preappend(km, 0, k, km1);
          for (u32 ch = 0; ch < 4; ++ch) {
            Ops::set_base(km1, 0, ch);
            if (Ops::cmp(km1, rv1, k + 1) > 0) break;
            if (Own::search(edges, n_edges, lut, s_owner, me, we, km1, k + 1) != nullptr) A = true;
          }
        }
        // ---- out-searches ----
        const u32 *e = Own::search(edges, n_edges, lut, s_owner, me, we, km, k);
        if (e != nullptr) {
          O = true;
          G1 = true;
          if (i + k < L && base_at(e, k) == pkg_base(s, L, i + k)) G1n = true;
        }
        {
          u32 km1[WM], rv1[WM];
#pragma unroll
          for (int j = 0; j < WM; ++j) km1[j] = km[j];
          Ops::set_base(km1, k, 3);
          const u32 next_char = i + k < L ? 3u - pkg_base(s, L, i + k) : 0u;
          Ops::preappend(rvk, next_char, k, rv1);
          if (Ops::cmp(rv1, km1, k + 1) <= 0 && Own::search(edges, n_edges, lut, s_owner, me, we, rv1, k + 1) != nullptr) {
            O = true;
            G2 = true;
          }
          for (u32 ch = 0; ch < 4; ++ch) {
            if (ch == next_char) continue;
            Ops::set_base(rv1, 0, ch);
            if (Ops::cmp(rv1, km1, k + 1) > 0) break;
            if (Own::search(edges, n_edges, lut, s_owner, me, we, rv1, k + 1) != nullptr) O = true;
          }
        }
      }
      const u32 m0 = __ballot_sync(0xffffffffu, A), m1 = __ballot_sync(0xffffffffu, O), m2 = __ballot_sync(0xffffffffu, G1),
                m3 = __ballot_sync(0xffffffffu, G1n), m4 = __ballot_sync(0xffffffffu, G2);
      if (lane == 0) {
        const u32 w = i0 >> 5;
        if (Accumulate) {
          pl[w] |= m0;
          pl[words_per_read + w] |= m1;
          pl[2 * words_per_read + w] |= m2;
          pl[3 * words_per_read + w] |= m3;
          pl[4 * words_per_read + w] |= m4;
        } else {
          pl[w] = m0;
          pl[words_per_read + w] = m1;
          pl[2 * words_per_read + w] = m2;
          pl[3 * words_per_read + w] = m3;
          pl[4 * words_per_read + w] = m4;
        }
      }
    }
  }
}

// planes[src][cand][5][wpr] of n_src ranks -> bits[cand][3][wpr] = (A, O, N) as k_mercy_emit expects them
__global__ void k_mercy_combine(const u32 *__restrict__ planes, u32 n_src, u64 src_stride_words, u64 n_cand, u32 wpr,
                                u32 *__restrict__ bits) {
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_cand * wpr) return;
  const u64 c = t / wpr;
  const u32 w = (u32)(t - c * wpr);
  u32 A = 0, O = 0, G1 = 0, G1n = 0, G2 = 0;
  for (u32 s = 0; s < n_src; ++s) {
    const u32 *pl = planes + s * src_stride_words + c * (u64)kOwnedPlanes * wpr;
    A |= pl[w];
    O |= pl[wpr + w];
    G1 |= pl[2 * wpr + w];
    G1n |= pl[3 * wpr + w];
    G2 |= pl[4 * wpr + w];
  }
  u32 *b = bits + c * 3ull * wpr;
  b[w] = A;
  b[wpr + w] = O;
  b[2 * wpr + w] = (G1 & G1n) | (~G1 & G2);
}

}  // namespace

extern "C" size_t mhb_mercy_planes_words(uint64_t n_cand, uint32_t max_read_len) {
  return (size_t)n_cand * kOwnedPlanes * ((max_read_len + 31) / 32 + 1);
}

int mercy_probe_owned(void *stream, const mhb_dev_reads *reads, const uint64_t *cand_ids, uint64_t n_cand,
                      uint32_t max_read_len, uint32_t k, const uint32_t *edges, uint64_t n_edges, const void *lut,
                      const uint8_t *owner_of_byte, uint32_t me, uint32_t *planes_out, bool accumulate) {
  if (int rc = check_reads(reads, k)) return rc;
  if (n_cand == 0) return MHB_OK;
  if (k < 12) return mhb_set_error(MHB_ERR_ARG, "mercy edges need k >= 12 (12-mer look-up prefix)");
  if (!lut || !owner_of_byte || !planes_out) return mhb_set_error(MHB_ERR_ARG, "null lut / owner table / planes");
  const ReadsView rv = make_reads_view(reads);
  OwnerTab ot;
  memcpy(ot.owner, owner_of_byte, 256);
  const u32 wpr = (max_read_len + 31) / 32 + 1, WE = words_per_edge(k), WM = div_ceil(k + 1, 16);
  const unsigned g64 = grid_cap(n_cand, 8, 16);
  cudaStream_t st = (cudaStream_t)stream;
#define M(WW)                                                                                                               \
  if (WM == WW) {                                                                                                           \
    if (accumulate)                                                                                                         \
      k_mercy_probe_owned<WW, true><<<g64, 256, 0, st>>>(rv, cand_ids, n_cand, k, edges, (long long)n_edges,                 \
                                                                   (const uint2 *)lut, ot, me, WE, planes_out, wpr);         \
    else                                                                                                                    \
      k_mercy_probe_owned<WW, false><<<g64, 256, 0, st>>>(rv, cand_ids, n_cand, k, edges, (long long)n_edges,                \
                                                                    (const uint2 *)lut, ot, me, WE, planes_out, wpr);        \
  }
  MHB_FOR_W(M)
#undef M
  CK_LAUNCH();
  return MHB_OK;
}

extern "C" int mhb_mercy_probe_owned(void *stream, const mhb_dev_reads *reads, const uint64_t *cand_ids, uint64_t n_cand,
                                     uint32_t max_read_len, uint32_t k, const uint32_t *edges, uint64_t n_edges, const void *lut,
                                     const uint8_t *owner_of_byte, uint32_t me, uint32_t *planes_out) {
  return mercy_probe_owned(stream, reads, cand_ids, n_cand, max_read_len, k, edges, n_edges, lut, owner_of_byte, me,
                           planes_out, false);
}

extern "C" int mhb_mercy_count_planes(void *stream, const mhb_dev_reads *reads, const uint64_t *cand_ids, uint64_t n_cand,
                                      uint32_t max_read_len, uint32_t k, const uint32_t *planes, uint32_t n_src,
                                      uint64_t src_stride_words, uint64_t *n_mercy_host, void *scratch, size_t scratch_bytes) {
  *n_mercy_host = 0;
  if (int rc = check_reads(reads, k)) return rc;
  if (n_cand == 0) return MHB_OK;
  if (!planes || n_src < 1) return mhb_set_error(MHB_ERR_ARG, "no answer planes");
  if (scratch_bytes < mercy_core_scratch(n_cand, max_read_len)) return mhb_set_error(MHB_ERR_ARG, "scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  const ReadsView rv = make_reads_view(reads);
  const MercyScratch ms = mercy_scratch_layout(scratch, n_cand, max_read_len);
  const u64 nt = n_cand * ms.wpr;
  k_mercy_combine<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(planes, n_src, src_stride_words, n_cand, ms.wpr, ms.bits);
  CK_LAUNCH();
  const unsigned g = (unsigned)((n_cand + 127) / 128);
  k_mercy_emit<false><<<g, 128, 0, st>>>(rv, cand_ids, n_cand, k, ms.bits, ms.wpr, ms.count, nullptr, nullptr, words_per_edge(k));
  CK_LAUNCH();
  if (int rc = scan32(st, ms.count, n_cand, ms.off, ms.total, ms.bsum)) return rc;
  CK(cudaMemcpyAsync(n_mercy_host, ms.total, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MHB_OK;
}
