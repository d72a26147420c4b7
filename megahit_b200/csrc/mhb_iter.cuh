// mhb_iter.cuh -- `iterate` (SURVEY.md 8f N2): the (k+step+1)-mers of the reads spanned by contig flanks, i.e. the
// iterative edges the next k starts from.  Reference: voutcn/megahit src/main_iterate.cpp:117-221,
// src/iterate/contig_flank_index.h:16-221, src/iterate/kmer_collector.h:37-79.
//
// The reference keeps the flanks in a hash set and the edges in a concurrent hash set; here the flank index is a sorted,
// de-duplicated array (radix sort of {(k+1)-mer, ~(ext_len, ext_seq)} records: the entry with the largest extension
// sorts first within its key and survives, contig_flank_index.h:67-75) searched by bisection behind a 16-bit prefix
// table, every read is scanned by one thread exactly as FindNextKmersFromReads does (the scan is sequential: a hit
// skips the positions its extension covers), and the emitted edges are sorted + made unique by the library's radix sort.
// All multiplicities are 0, as in the reference (FlankInfo::mul is never filled in, :66).
#pragma once
#include "mhb.h"
#include "mhb_kernels.cuh"

namespace mhb {

struct IterReads {  // `.bin` image, FILE orientation (iterate loads reads with reverse = false)
  const u32 *bin;
  u64 n_reads;
  u32 fixed_len;       // > 0: record r starts at word r * (1 + ceil(fixed_len/16)), base offset r * fixed_len
  const u64 *rec_off;  // variable-length: n_reads + 1
  const u64 *base_off; // n_reads + 1
  MHB_HD const u32 *rec(u64 r) const { return bin + (fixed_len ? r * (u64)(1 + div_ceil(fixed_len, 16)) : rec_off[r]); }
  MHB_HD u64 base(u64 r) const { return fixed_len ? r * (u64)fixed_len : base_off[r]; }
};

struct FlankTable {
  const u32 *recs;     // n records of wk + 2 words: key, then ~val (hi, lo); ascending, unique keys
  u64 n;
  u32 wk;              // words per (k+1)-mer key
  const u32 *lut;      // 65537 entries: first record whose leading 16 key bits are >= p
};

// val = ext_len << 58 | ext_seq (contig_flank_index.h:19-23)
MHB_HD u64 flank_val(const u32 *rec, u32 wk) { return ~(((u64)rec[wk] << 32) | rec[wk + 1]); }

// index of the flank with this key, or -1
template <int WC>
MHB_HD long long flank_find(const FlankTable &t, const u32 (&key)[WC]) {
  if (t.n == 0) return -1;
  const u32 p = key[0] >> 16;
  long long lo = t.lut[p], hi = (long long)t.lut[p + 1] - 1;
  const u32 rw = t.wk + 2;
  while (lo <= hi) {
    const long long mid = (lo + hi) >> 1;
    const u32 *e = t.recs + (u64)mid * rw;
    int c = 0;
    for (u32 j = 0; j < t.wk && c == 0; ++j) {
      const u32 kj = pick<WC>(key, j);
      if (e[j] != kj) c = e[j] < kj ? -1 : 1;
    }
    if (c == 0) return mid;
    if (c < 0) lo = mid + 1; else hi = mid - 1;
  }
  return -1;
}

#if defined(__CUDA_ARCH__)
#define MHB_IT_OR32(p, v) atomicOr((p), (v))
#else
#define MHB_IT_OR32(p, v) (*(p) |= (v))
#endif
MHB_HD void it_bit_set(u32 *bits, u64 i) { MHB_IT_OR32(&bits[i >> 5], 1u << (i & 31)); }
MHB_HD bool it_bit_get(const u32 *bits, u64 i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// FindNextKmersFromReads, first half (contig_flank_index.h:88-170): marks in exist[base + j] every (k+1)-mer position j
// of the read that a contig flank (or its matched extension) covers.  WC: register words, >= ceil((k+1)/16).
template <int WC>
MHB_HD void iter_mark_read(const IterReads &rd, u64 r, u32 k, u32 step, const FlankTable &t, u32 *exist) {
  const u32 *rec = rd.rec(r);
  const u32 L = rec[0];
  if (L < k + step + 1) return;
  const u32 *s = rec + 1;
  const u32 nwords = div_ceil(L, 16), K1 = k + 1;
  const u64 b = rd.base(r);
  u32 cur = 0;
  while (cur + K1 <= L) {
    u32 next = cur + 1;
    if (!it_bit_get(exist, b + cur)) {
      u32 F[WC], T[WC], R[WC];
      load_sub<WC>(s, nwords, cur, K1, F);
      long long f = flank_find<WC>(t, F);
      if (f >= 0) {
        it_bit_set(exist, b + cur);
        const u64 v = flank_val(t.recs + (u64)f * (t.wk + 2), t.wk);
        const u32 ext_len = (u32)(v >> 58);
        for (u32 j = 0; j < ext_len && cur + K1 + j < L; ++j, ++next) {
          if (base_at(s, cur + K1 + j) == (u32)((v >> (2 * j)) & 3u)) it_bit_set(exist, b + cur + j + 1);
          else break;
        }
      }
      reverse_sub<WC>(F, K1, T);
      complement_sub<WC>(T, K1, R);
      f = flank_find<WC>(t, R);
      if (f >= 0) {
        it_bit_set(exist, b + cur);
        const u64 v = flank_val(t.recs + (u64)f * (t.wk + 2), t.wk);
        const u32 ext_len = (u32)(v >> 58);
        for (u32 j = 0; j < ext_len && cur >= j + 1; ++j) {
          if ((3u ^ base_at(s, cur - 1 - j)) == (u32)((v >> (2 * j)) & 3u)) it_bit_set(exist, b + cur - 1 - j);
          else break;
        }
      }
    }
    if (next + K1 <= L) cur = next; else break;
  }
}

// second half (:172-212): every position that ends a run of >= step+1 marked positions yields the canonical
// (k+step+1)-mer ending there, written as KmerCollector::WriteToFile does (kmer_collector.h:50-69: the k-mer REVERSED,
// left-aligned, multiplicity 0).  out == nullptr: count only.  Returns the number of edges of this read.
template <int WC>
MHB_HD u32 iter_emit_read(const IterReads &rd, u64 r, u32 k, u32 step, const u32 *exist, u32 w2, u32 *out) {
  const u32 *rec = rd.rec(r);
  const u32 L = rec[0];
  const u32 KN = k + step + 1;
  if (L < KN) return 0;
  const u32 *s = rec + 1;
  const u32 nwords = div_ceil(L, 16);
  const u64 b = rd.base(r);
  u32 acc = 0, n = 0;
  for (u32 j = 0; j + k < L; ++j) {
    acc = it_bit_get(exist, b + j) ? acc + 1 : 0;
    if (acc >= step + 1) {
      if (out) {
        u32 S[WC], T[WC], R[WC];
        load_sub<WC>(s, nwords, j + k + 1 - KN, KN, S);
        reverse_sub<WC>(S, KN, T);      // T = reverse(S)
        complement_sub<WC>(T, KN, R);   // R = reverse complement
        // canonical = S < R ? S : R, stored reversed: reverse(S) = T, reverse(R) = complement(S)
        u32 C[WC];
        if (less_words<WC>(S, R)) {
#pragma unroll
          for (int q = 0; q < WC; ++q) C[q] = T[q];
        } else {
          complement_sub<WC>(S, KN, C);
        }
        u32 *o = out + (u64)n * w2;
        for (u32 q = 0; q < w2; ++q) o[q] = pick<WC>(C, q);
      }
      ++n;
    }
  }
  return n;
}

// flank record of (contig c, strand): key + ~val; returns false when the contig yields none (short, palindrome)
template <int WC>
MHB_HD bool iter_flank_record(const u32 *s, u32 L, u32 k, u32 step, u32 strand, u32 wk, u32 *rec_out) {
  const u32 K1 = k + 1, nwords = div_ceil(L, 16);
  if (L < K1) return false;
  if (strand == 1 && L == K1) return false;  // contig_flank_index.h:82-84
  u32 F[WC], T[WC], R[WC];
  load_sub<WC>(s, nwords, strand == 0 ? 0 : L - K1, K1, F);
  reverse_sub<WC>(F, K1, T);
  complement_sub<WC>(T, K1, R);
  bool pal = true;
#pragma unroll
  for (int q = 0; q < WC; ++q) pal = pal && F[q] == R[q];
  if (pal) return false;  // :46-48 (the reverse complement of a palindrome is one too)
  const u32 ext_len = step - 1 < L - K1 ? step - 1 : L - K1;
  u64 ext = 0;
  for (u32 j = 0; j < ext_len; ++j) {
    const u32 c = strand == 0 ? base_at(s, K1 + j) : 3u ^ base_at(s, L - 1 - (K1 + j));
    ext |= (u64)c << (2 * j);
  }
  const u64 nv = ~(((u64)ext_len << 58) | ext);
  for (u32 q = 0; q < wk; ++q) rec_out[q] = strand == 0 ? pick<WC>(F, q) : pick<WC>(R, q);
  rec_out[wk] = (u32)(nv >> 32);
  rec_out[wk + 1] = (u32)nv;
  return true;
}

#if defined(__CUDACC__)
struct IterContigs {
  const u32 *words;
  const u64 *word_off;
  const u32 *len;
  u64 n;
};

// vals == nullptr: records of wk + 2 words (key, ~val).  Otherwise the narrow layout for keys too wide for a
// (wk + 2)-word sort record: wk key words + the 32-bit row index, and ~val of row i in vals[i].
template <int WC>
__global__ void __launch_bounds__(256) k_iter_flanks(IterContigs cs, u32 k, u32 step, u32 wk, u32 *__restrict__ recs,
                                                    u64 *__restrict__ vals, unsigned long long *__restrict__ cursor) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < 2 * cs.n; t += (u64)gridDim.x * 256) {
    const u64 c = t >> 1;
    u32 rec[20];
    if (iter_flank_record<WC>(cs.words + cs.word_off[c], cs.len[c], k, step, (u32)(t & 1), wk, rec)) {
      const unsigned long long at = atomicAdd(cursor, 1ull);
      if (vals) {
        for (u32 q = 0; q < wk; ++q) recs[at * (wk + 1) + q] = rec[q];
        recs[at * (wk + 1) + wk] = (u32)at;
        vals[at] = ((u64)rec[wk] << 32) | rec[wk + 1];
      } else {
        for (u32 q = 0; q < wk + 2; ++q) recs[at * (wk + 2) + q] = rec[q];
      }
    }
  }
}

// Narrow flank records (wk key words + row index) sorted on the key, run heads flagged: per run of equal keys the
// smallest ~val - the largest (ext_len, ext_seq), which the wide layout's sort on {key, ~val} puts first - goes with
// the key into the (wk + 2)-word flank table at off[head].
__global__ void __launch_bounds__(256) k_iter_best(const u32 *__restrict__ recs, u64 n, u32 wk, const u64 *__restrict__ vals,
                                                  const u32 *__restrict__ flag, const u64 *__restrict__ off,
                                                  u32 *__restrict__ out) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    if (!flag[i]) continue;
    u64 best = ~0ull;
    for (u64 j = i; j < n && (j == i || !flag[j]); ++j) {
      const u64 v = vals[recs[j * (wk + 1) + wk]];
      best = v < best ? v : best;
    }
    u32 *o = out + off[i] * (wk + 2);
    for (u32 q = 0; q < wk; ++q) o[q] = recs[i * (wk + 1) + q];
    o[wk] = (u32)(best >> 32);
    o[wk + 1] = (u32)best;
  }
}

// heads of runs of equal keys (first `wcmp` words) in sorted records of `rw` words
__global__ void __launch_bounds__(256) k_iter_heads(const u32 *__restrict__ recs, u64 n, u32 rw, u32 wcmp, u32 *__restrict__ flag) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    bool head = i == 0;
    if (!head)
      for (u32 q = 0; q < wcmp; ++q) head = head || recs[i * rw + q] != recs[(i - 1) * rw + q];
    flag[i] = head ? 1u : 0u;
  }
}
__global__ void __launch_bounds__(256) k_iter_compact(const u32 *__restrict__ recs, u64 n, u32 rw, const u32 *__restrict__ flag,
                                                     const u64 *__restrict__ off, u32 *__restrict__ out) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256)
    if (flag[i])
      for (u32 q = 0; q < rw; ++q) out[off[i] * rw + q] = recs[i * rw + q];
}
__global__ void k_iter_lut(const u32 *__restrict__ recs, u64 n, u32 rw, u32 *__restrict__ lut) {
  const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > 65536) return;
  u64 lo = 0, hi = n;
  while (lo < hi) {
    const u64 mid = (lo + hi) >> 1;
    if ((recs[mid * rw] >> 16) < p) lo = mid + 1; else hi = mid;
  }
  lut[p] = (u32)lo;
}

template <int WC>
__global__ void __launch_bounds__(128) k_iter_mark(IterReads rd, u32 k, u32 step, FlankTable t, u32 *__restrict__ exist) {
  for (u64 r = (u64)blockIdx.x * 128 + threadIdx.x; r < rd.n_reads; r += (u64)gridDim.x * 128)
    iter_mark_read<WC>(rd, r, k, step, t, exist);
}

// WRITE = false: per-read edge counts summed into *cursor and the number of aligned reads into cursor[1];
// WRITE = true: the read's edges appended at out[*cursor ...) (one atomic per aligned read)
template <int WC, bool WRITE>
__global__ void __launch_bounds__(128) k_iter_emit(IterReads rd, u32 k, u32 step, const u32 *__restrict__ exist, u32 w2,
                                                  u32 *__restrict__ out, unsigned long long *__restrict__ cursor, u64 capacity) {
  unsigned long long tot = 0, aligned = 0;
  for (u64 r = (u64)blockIdx.x * 128 + threadIdx.x; r < rd.n_reads; r += (u64)gridDim.x * 128) {
    const u32 n = iter_emit_read<WC>(rd, r, k, step, exist, w2, nullptr);
    if (!n) continue;
    if (WRITE) {
      const unsigned long long at = atomicAdd(cursor, (unsigned long long)n);
      if (at + n <= capacity) iter_emit_read<WC>(rd, r, k, step, exist, w2, out + at * w2);
    } else {
      tot += n;
      ++aligned;
    }
  }
  if (!WRITE) {
    for (int d = 16; d; d >>= 1) {
      tot += __shfl_xor_sync(0xffffffffu, tot, d);
      aligned += __shfl_xor_sync(0xffffffffu, aligned, d);
    }
    if (lane_id() == 0 && tot) {
      atomicAdd(cursor, tot);
      atomicAdd(cursor + 1, aligned);
    }
  }
}
#endif  // __CUDACC__

}  // namespace mhb
