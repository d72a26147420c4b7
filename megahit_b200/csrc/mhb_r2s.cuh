// mhb_r2s.cuh -- `read2sdbg` (the 1-pass SdBG build, SURVEY.md 8a A12): building blocks and kernels.
// Reference: voutcn/megahit src/sorting/read_to_sdbg_s1.cpp, read_to_sdbg_s2.cpp, kmlib/kmsort.h.
//
// Stage 1 (min-count > 1) marks the solid (k+1)-mer occurrences of every read and collects mercy candidates; the
// reference's output depends on the order kmlib::kmsort leaves among records with equal keys
// (read_to_sdbg_s1.cpp:393-401 reads prev/next of the FIRST record of a (k-1)-mer group for the whole group), so the
// in-bucket sort here is not one of the library's LSD sorts but a literal emulation of kmsort's American-flag
// permutation: records are brought into the reference's per-bucket input order (global read order) by two STABLE
// radix passes on the 16-bit bucket id, then every bucket - later every sub-range above the insertion-sort
// threshold - is permuted by one thread exactly as radix_sort_core does it (kmsort.h:43-101).  The walk is serial
// by nature (each step pops the head of the bin the previous record belongs to); the parallelism is across the
// 65 536 buckets and their sub-ranges.
// Stage 2 builds one sort item per (solid edge occurrence, strand, $-variant), sorts whole items (ties are identical,
// so any sort will do), collapses equal items into one with its run length as multiplicity and hands them to the
// seq2sdbg emitter (the group logic of read_to_sdbg_s2.cpp:521-614 equals seq_to_sdbg.cpp:702-789).
#pragma once
#include "mhb.h"
#include "mhb_kernels.cuh"
#if defined(__CUDACC__)
#include "mhb_s2s.cuh"
#endif

namespace mhb {

// ---- geometry ----
MHB_HD u32 r2s_s1_key_words(u32 k) { return div_ceil(2 * (k - 1) + 6, 32); }  // read_to_sdbg_s1.cpp:103-104
MHB_HD u32 r2s_s2_words(u32 k) { return div_ceil(2 * k + 4, 32); }            // read_to_sdbg_s2.cpp:97-98
static constexpr int kKmInsertThreshold = 64;                                 // kmsort.h:16

// Reads in PACKAGE orientation (reversed, not complemented: read_to_sdbg_s1.cpp:89,100), one word-aligned run per read.
// A view covers the whole library or one streamed chunk of it: read indices, words and the offset arrays are relative
// to the view, base(r) - every bit-plane index and stage-1 payload - is global.
struct PkgView {
  const u32 *words;
  u64 n_reads;
  u32 fixed_len;        // > 0: every read has this length; read r starts at word r * fixed_words, base r * fixed_len
  u32 fixed_words;
  const u64 *word_off;  // variable-length libraries: n_reads + 1
  const u32 *len;       // n_reads (a zero-length read counts as one base, sequence_package.h:276-281)
  const u64 *base_off;  // n_reads + 1: bases before read r in the view
  const u64 *s1_off;    // n_reads + 1: stage-1 records before read r in the view
  const u64 *edge_off;  // n_reads + 1: (k+1)-mer positions before read r in the view
  u64 base0;            // full_offset_in_pkg of the view's read 0 (0 for the whole library)
  MHB_HD u32 L(u64 r) const { return fixed_len ? fixed_len : len[r]; }
  MHB_HD const u32 *ptr(u64 r) const { return words + (fixed_len ? r * (u64)fixed_words : word_off[r]); }
  MHB_HD u64 base(u64 r) const { return base0 + (fixed_len ? r * (u64)fixed_len : base_off[r]); }
  // last r with off_array[r] <= x
  static MHB_HD u64 find(const u64 *off, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (hi - lo > 1) {
      const u64 mid = (lo + hi) >> 1;
      if (off[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
  }
  MHB_HD u64 read_of_base(u64 off) const {
    return fixed_len ? (off - base0) / fixed_len : find(base_off, n_reads, off - base0);
  }
};

// Package geometry of one read of file length L_file (the `.bin` length word), as index_pkg counts it: bases (a
// zero-length read counts as one, sequence_package.h:276-281), package words, stage-1 records, (k+1)-mer positions.
// Exclusive scans of these over a chunk give the chunk's base_off / word_off / s1_off / edge_off.
MHB_HD void r2s_read_geom(u32 L_file, u32 k, u32 &len, u32 &words, u32 &s1, u32 &edges) {
  len = L_file == 0 ? 1u : L_file;
  words = div_ceil(len, 16);
  s1 = len >= k + 1 ? len - k + 4 : 0u;
  edges = len >= k + 1 ? len - k : 0u;
}

MHB_HD u32 comp_or_sentinel(u32 c) { return c == kSentinel ? kSentinel : 3u - c; }

// ------------------------------------------------------------------------------------------------
// Stage-1 record (Lv1FillOffsets read_to_sdbg_s1.cpp:207-293 + Lv2ExtractSubString :295-366) of the (k-1)-mer at
// position p of a package-orientation read: NW key words ((k-1)-mer of the chosen strand left-aligned, head<<3|tail
// in the low 6 bits of the last key word) + 2 payload words (full_offset<<6 | prev<<3 | next, high word first).
// want = 0/1: that strand (first and last position are emitted on both); want = 2: the canonical one (:254-279).
// ------------------------------------------------------------------------------------------------
template <int NW>
MHB_HD void make_s1_record(const u32 *s, u32 nwords, u32 L, u32 k, u32 p, u32 want, u64 base_off, u32 (&rec)[NW + 2]) {
  const u32 kk = k - 1;
  u32 F[NW], T[NW], R[NW];
  load_sub<NW>(s, nwords, p, kk, F);
  reverse_sub<NW>(F, kk, T);
  complement_sub<NW>(T, kk, R);
  u32 strand = want;
  if (want == 2) {
    if (less_words<NW>(R, F)) {
      strand = 1;
    } else if (less_words<NW>(F, R)) {
      strand = 0;
    } else {  // palindrome: "not-that-math-correct", :263-279
      const u32 pv = base_at(s, p - 1), nx = base_at(s, p + kk);
      strand = pv <= 3u - nx ? 0u : 1u;
    }
  }
  u32 head, prev, tail, next;  // (k+1)-mer = head S tail, prev / next one further out (:303-330)
  if (p > 1) {
    head = base_at(s, p - 1);
    prev = base_at(s, p - 2);
  } else {
    prev = kSentinel;
    head = p > 0 ? base_at(s, p - 1) : kSentinel;
  }
  if (p + k < L) {
    tail = base_at(s, p + k - 1);
    next = base_at(s, p + k);
  } else {
    next = kSentinel;
    tail = p + k - 1 < L ? base_at(s, p + k - 1) : kSentinel;
  }
  const u64 full = ((base_off + p) << 1) | strand;
  u64 info;
  if (strand == 0) {
#pragma unroll
    for (int j = 0; j < NW; ++j) rec[j] = F[j];
    rec[NW - 1] |= (head << 3) | tail;
    info = (full << 6) | (prev << 3) | next;
  } else {
#pragma unroll
    for (int j = 0; j < NW; ++j) rec[j] = R[j];
    rec[NW - 1] |= (comp_or_sentinel(tail) << 3) | comp_or_sentinel(head);
    info = (full << 6) | (comp_or_sentinel(next) << 3) | comp_or_sentinel(prev);
  }
  rec[NW] = (u32)(info >> 32);
  rec[NW + 1] = (u32)info;
}

// stage-1 record e (0-based emission index, the reference's bucket input order) of a read with L >= k+1:
// (p=0,s0) (p=0,s1) (p=1..L-k, canonical) (p=L-k+1,s0) (p=L-k+1,s1)
MHB_HD void s1_emission(u32 L, u32 k, u32 e, u32 &p, u32 &want) {
  const u32 last = L - k + 1;
  if (e < 2) {
    p = 0;
    want = e;
  } else if (e < last + 1) {
    p = e - 1;
    want = 2;
  } else {
    p = last;
    want = e - (last + 1);
  }
}

// ------------------------------------------------------------------------------------------------
// Stage-2 sort item (Lv1FillOffsets read_to_sdbg_s2.cpp:347-436 + Lv2ExtractSubString :438-519) of the edge at
// position i, in the SEQ2SDBG record layout (W = s2s_record_words(k) words: chars, then nondollar<<19 | prev<<16 |
// stored multiplicity in the low 20 bits of the last word) so that the library's seq2sdbg sort and emitter take it;
// the reference's own layout keeps nondollar<<3 | prev in the low 4 bits of word r2s_s2_words(k)-1, which only shows in
// the raw words of a tip label (the emitter rebuilds them, label_fmt = 1).  type 0 = left $, 1 = solid, 2 = right $.
// ------------------------------------------------------------------------------------------------
template <int W>
MHB_HD void make_r2s_item(const u32 *s, u32 nwords, u32 k, u32 i, u32 strand, u32 type, u32 (&rec)[W]) {
  u32 nc = k, prev = kSentinel;
  if (strand == 0) {
    u32 off = i;
    if (type == 1) {
      prev = base_at(s, i);
      off = i + 1;
    } else if (type == 2) {
      prev = base_at(s, i + 1);
      off = i + 2;
      nc = k - 1;
    }
    load_sub<W>(s, nwords, off, nc, rec);
  } else {
    u32 off = i;
    if (type == 0) {
      nc = k - 1;
      prev = 3u - base_at(s, i + k - 1);
    } else if (type == 1) {
      prev = 3u - base_at(s, i + k);
    } else {
      off = i + 1;
    }
    u32 S[W], T[W];
    load_sub<W>(s, nwords, off, nc, S);
    reverse_sub<W>(S, nc, T);
    complement_sub<W>(T, nc, rec);
  }
  rec[W - 1] |= ((nc == k) ? 1u : 0u) << 19;
  rec[W - 1] |= prev << 16;
  rec[W - 1] |= 0xFFFFu;  // replaced by 65535 - run length once equal items are collapsed
}

// is the (k+1)-mer at position i its own reverse complement?  (read_to_sdbg_s2.cpp:386)
template <int W>
MHB_HD bool edge_is_palindrome(const u32 *s, u32 nwords, u32 k, u32 i) {
  u32 E[W], T[W], R[W];
  load_sub<W>(s, nwords, i, k + 1, E);
  reverse_sub<W>(E, k + 1, T);
  complement_sub<W>(T, k + 1, R);
  bool eq = true;
#pragma unroll
  for (int j = 0; j < W; ++j) eq = eq && (E[j] == R[j]);
  return eq;
}

// ------------------------------------------------------------------------------------------------
// kmlib::kmsort, emulated.  Records of RW words, the first nw of them the key; radix byte kb (0 = least significant
// byte of the last KEY word, kmsort_selector.cpp:29-33), n_bytes = 4 nw - 2 (:17).
// ------------------------------------------------------------------------------------------------
template <int RW>
MHB_HD void km_ld(const u32 *a, u64 i, u32 (&r)[RW]) {
#pragma unroll
  for (int j = 0; j < RW; ++j) r[j] = a[i * RW + j];
}
template <int RW>
MHB_HD void km_st(u32 *a, u64 i, const u32 (&r)[RW]) {
#pragma unroll
  for (int j = 0; j < RW; ++j) a[i * RW + j] = r[j];
}
template <int RW>
MHB_HD u32 km_byte(const u32 (&r)[RW], u32 nw, int kb) {
  return (pick<RW>(r, nw - 1 - ((u32)kb >> 2)) >> (8 * (kb & 3))) & 255u;
}
MHB_HD u32 km_byte_mem(const u32 *rec, u32 nw, int kb) { return (rec[nw - 1 - ((u32)kb >> 2)] >> (8 * (kb & 3))) & 255u; }
template <int RW>
MHB_HD bool km_less(const u32 (&x)[RW], const u32 (&y)[RW], u32 nw) {
  bool lt = false, decided = false;
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    if ((u32)j < nw && !decided && x[j] != y[j]) {
      lt = x[j] < y[j];
      decided = true;
    }
  }
  return lt;
}

// insert_sort_core (kmsort.h:22-35): stable
template <int RW>
MHB_HD void km_insertion(u32 *a, u32 n, u32 nw) {
  u32 cur[RW], prv[RW], tmp[RW];
  for (u32 i = 1; i < n; ++i) {
    km_ld<RW>(a, i, cur);
    km_ld<RW>(a, i - 1, prv);
    if (km_less<RW>(cur, prv, nw)) {
      km_st<RW>(a, i, prv);
      u32 j = i - 1;
      while (j > 0) {
        km_ld<RW>(a, j - 1, tmp);
        if (!km_less<RW>(cur, tmp, nw)) break;
        km_st<RW>(a, j, tmp);
        --j;
      }
      km_st<RW>(a, j, cur);
    }
  }
}

// radix_sort_core (kmsort.h:43-101) on one range, WITHOUT the recursion: permutes the range in place on byte kb and
// leaves the bin sizes in count[0..255] (bin i starts at the sum of the earlier counts); the caller sorts children of
// 2..64 records with km_insertion and queues larger ones for byte kb-1 (only when kb > 0).  last: 256-entry scratch.
template <int RW>
MHB_HD void km_radix_range(u32 *a, u32 n, u32 nw, int kb, u32 *count, u32 *last) {
  for (int i = 0; i < 256; ++i) count[i] = 0;
  for (u32 i = 0; i < n; ++i) ++count[km_byte_mem(a + (u64)i * RW, nw, kb)];
  {
    u32 acc = 0;
    for (int i = 0; i < 256; ++i) {
      last[i] = acc;
      acc += count[i];
    }
  }
  u32 begin = 0;
  for (int i = 0; i < 256; ++i) {
    const u32 end = begin + count[i];
    if (end == n) break;  // :66-69: the last populated bin is in place once all the others are
    while (last[i] != end) {
      u32 swapper[RW], other[RW];
      km_ld<RW>(a, last[i], swapper);
      u32 tag = km_byte<RW>(swapper, nw, kb);
      if (tag != (u32)i) {
        do {  // :75-79
          const u32 q = last[tag]++;
          km_ld<RW>(a, q, other);
          km_st<RW>(a, q, swapper);
#pragma unroll
          for (int j = 0; j < RW; ++j) swapper[j] = other[j];
          tag = km_byte<RW>(swapper, nw, kb);
        } while (tag != (u32)i);
        km_st<RW>(a, last[i], swapper);
      }
      ++last[i];
    }
    begin = end;
  }
}

// The same permutation from the TAGS alone.  Positions at or behind a bin's cursor still hold their original record
// (the walk only ever writes at a cursor and then advances it), so "the record displaced from slot q" is the record
// that started at q: the walk needs nothing but tags[] and the 256 cursors, and yields src[q] = original index of the
// record that ends in slot q.  cnt = bin sizes, last = bin starts on entry (cursors, clobbered).  With the tags in
// shared memory a step costs two shared-memory round trips instead of a dependent global load + store.
template <class IT>
MHB_HD void km_walk_src(const uint8_t *tags, u32 n, const u32 *cnt, u32 *last, IT *src) {
  u32 begin = 0;
  int i = 0;
  for (; i < 256; ++i) {
    const u32 end = begin + cnt[i];
    if (end == n) break;  // kmsort.h:66-69
    while (last[i] != end) {
      u32 p = last[i];
      u32 t = tags[p];
      while (t != (u32)i) {  // :75-79
        const u32 q = last[t]++;
        src[q] = (IT)p;
        p = q;
        t = tags[p];
      }
      src[last[i]] = (IT)p;
      ++last[i];
    }
    begin = end;
  }
  if (i < 256)
    for (u32 q = last[i]; q < n; ++q) src[q] = (IT)q;  // the last populated bin: what is left stays where it is
}

MHB_HD bool km_less_mem(const u32 *x, const u32 *y, u32 nw) {
  for (u32 j = 0; j < nw; ++j)
    if (x[j] != y[j]) return x[j] < y[j];
  return false;
}

// insert_sort_core (kmsort.h:22-35) on an index array: slot j holds record staged[idx[j]]
template <class IT>
MHB_HD void km_insertion_idx(const u32 *staged, u32 rw, IT *idx, u32 c, u32 nw) {
  for (u32 i = 1; i < c; ++i) {
    const IT cur = idx[i];
    if (km_less_mem(staged + (u32)cur * rw, staged + (u32)idx[i - 1] * rw, nw)) {
      idx[i] = idx[i - 1];
      u32 j = i - 1;
      while (j > 0 && km_less_mem(staged + (u32)cur * rw, staged + (u32)idx[j - 1] * rw, nw)) {
        idx[j] = idx[j - 1];
        --j;
      }
      idx[j] = cur;
    }
  }
}

// records a warp stages in shared memory for one range (8 KB of records)
__host__ __device__ constexpr u32 km_wcap(int rw) { return 2048u / (u32)rw; }

// ------------------------------------------------------------------------------------------------
// Stage 1, Lv2Postprocess (read_to_sdbg_s1.cpp:368-555) for the (k-1)-mer group starting at record g0.
// ------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define MHB_OR32(p, v) atomicOr((p), (v))
#else
#define MHB_OR32(p, v) (*(p) |= (v))
#endif
MHB_HD void bit_or(u32 *bits, u64 i) { MHB_OR32(&bits[i >> 5], 1u << (i & 31)); }
MHB_HD bool bit_at(const u32 *bits, u64 i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// IsDiffKMinusOneMer (read_to_sdbg_s1.cpp:40-63) on records in memory
MHB_HD bool s1_diff_km1(const u32 *x, const u32 *y, u32 k) {
  const u32 bits = 2 * (k - 1);
  const u32 full = bits >> 5, rem = bits & 31;
  for (u32 j = 0; j < full; ++j)
    if (x[j] != y[j]) return true;
  if (rem && ((x[full] ^ y[full]) >> (32 - rem))) return true;
  return false;
}

struct S1Out {
  u32 *is_solid;   // bit per base of the package: the (k+1)-mer starting there is solid
  u32 *no_in;      // mercy candidate planes, bit per base: k-mer position with code 1 / code 2 / any code
  u32 *no_out;     // (read_to_sdbg_s2.cpp:183-195 consumes the candidates as these three sets)
  u32 *any;
};

// read_info (full_offset<<6 | prev<<3 | next) of a stage-1 record: its two payload words, or - narrow layout, info !=
// nullptr - the side-array entry its row index (the word after the nw key words) points at
MHB_HD u64 s1_info(const u32 *r, u32 nw, const u64 *info) {
  return info ? info[r[nw]] : ((u64)r[nw] << 32) | r[nw + 1];
}

// ---- the list form of the mercy candidates (DESIGN.md §4.9): one u64 entry per marked position, position << 2 | code
// (code 0 = any, 1 = no in, 2 = no out; 1 and 2 imply any), as Read2SdbgS1 writes P.mercy_cand.* ----
// Per stage-1 record the group walk leaves one candidate byte: (left code + 1) | (right code + 1) << 2, 0 = none.
MHB_HD u32 cand_count(u32 c) { return ((c & 3u) ? 1u : 0u) + ((c >> 2) ? 1u : 0u); }
// the entries of a record with candidate byte c and read_info `info` (full_offset << 6 | prev << 3 | next), left first
MHB_HD u32 cand_entries(u32 c, u64 info, u64 *out) {
  const u64 full = info >> 6, pos = full >> 1;
  const bool fwd = (full & 1) == 0;
  u32 n = 0;
  if (c & 3u) out[n++] = (fwd ? pos - 1 : pos) << 2 | ((c & 3u) - 1);
  if (c >> 2) out[n++] = (fwd ? pos : pos - 1) << 2 | ((c >> 2) - 1);
  return n;
}
// one entry into the three candidate planes (indexed by global base; the caller shifts them to its word grid)
MHB_HD void cand_mark(const S1Out &o, u64 e) {
  const u64 pos = e >> 2;
  const u32 code = (u32)(e & 3);
  bit_or(o.any, pos);
  if (code == 1) bit_or(o.no_in, pos);
  if (code == 2) bit_or(o.no_out, pos);
}

// walks the group [g0, end) twice: tallies, then per-record outputs.  Returns the group's end.  hist_vals[0..n_hist)
// (room for 16) receives the occurrence count of every distinct (k+1)-mer of the group (edge_counter_.Add, :430-432).
// With need_mercy the candidates go to the planes of o, or - cand != nullptr, the list form - to cand[record].
MHB_HD u64 s1_group(const u32 *recs, const u64 *info, u64 n, u64 g0, u32 rw, u32 nw, u32 k, int m, const PkgView &pv,
                    const S1Out &o, bool need_mercy, u32 *hist_vals, u32 &n_hist, uint8_t *cand = nullptr) {
  n_hist = 0;
  const u32 *first = recs + g0 * rw;
  u32 cht[40];  // count_head_tail, index head<<3|tail <= 36
  for (int i = 0; i < 40; ++i) cht[i] = 0;
  u64 end = g0;
  while (end < n && (end == g0 || !s1_diff_km1(first, recs + end * rw, k))) {
    ++cht[recs[end * rw + nw - 1] & 63u];
    ++end;
  }
  // :393-401: prev/next of the FIRST record stand in for every member, so has_in / has_out exist only when the first
  // record has a prev / next at all, and then count heads / tails over the whole group
  const u32 pn_first = (u32)s1_info(first, nw, info) & 63u;
  u32 has_in = 0, has_out = 0, l_has_out = 0, r_has_in = 0;
  for (u32 j = 0; j < 4; ++j) {
    u32 heads = 0, tails = 0;
    for (u32 x = 0; x < 5; ++x) {
      heads += cht[(j << 3) | x];
      tails += cht[(x << 3) | j];
    }
    if ((pn_first >> 3) < 4 && heads >= (u32)m) has_in |= 1u << j;
    if ((pn_first & 7) < 4 && tails >= (u32)m) has_out |= 1u << j;
    for (u32 x = 0; x < 4; ++x) {
      if (cht[(j << 3) | x] >= (u32)m) {
        l_has_out |= 1u << j;
        r_has_in |= 1u << x;
      }
    }
  }
  u32 seen = 0xFFu;  // head<<3|tail of the class being walked
  for (u64 q = g0; q < end; ++q) {
    const u32 *r = recs + q * rw;
    const u32 ht = r[nw - 1] & 63u, head = ht >> 3, tail = ht & 7;
    const bool both = head != kSentinel && tail != kSentinel;
    if (ht != seen) {  // records of one class are contiguous (the key includes head<<3|tail)
      seen = ht;
      if (both) hist_vals[n_hist++] = cht[ht];
    }
    if (!both && !need_mercy) continue;
    const u64 full = s1_info(r, nw, info) >> 6;
    const u32 strand = (u32)(full & 1);
    const u64 pos = full >> 1;  // full offset of the (k-1)-mer; the (k+1)-mer head S tail starts one base earlier
    const bool solid = both && cht[ht] >= (u32)m;
    if (solid) bit_or(o.is_solid, pos - 1);  // :441
    if (!need_mercy) continue;
    const u64 l_off = strand == 0 ? pos - 1 : pos, r_off = strand == 0 ? pos : pos - 1;
    // codes: 1 = no in, 2 = no out, 0 = has both (:443-551); code 1+strand / 2-strand = 1 or 2
    int lc = -1, rc = -1;
    if (solid) {
      if (!((has_in >> head) & 1u)) lc = 1 + (int)strand;
      if (!((has_out >> tail) & 1u)) rc = 2 - (int)strand;
    } else {
      if (head != kSentinel) {
        if ((l_has_out >> head) & 1u)
          lc = ((has_in >> head) & 1u) ? 0 : 1 + (int)strand;
        else if ((has_in >> head) & 1u)
          lc = 2 - (int)strand;
      }
      if (tail != kSentinel) {
        if ((r_has_in >> tail) & 1u)
          rc = ((has_out >> tail) & 1u) ? 0 : 2 - (int)strand;
        else if ((has_out >> tail) & 1u)
          rc = 1 + (int)strand;
      }
    }
    if (cand) {
      cand[q] = (uint8_t)((lc + 1) | (rc + 1) << 2);
      continue;
    }
    if (lc >= 0) {
      bit_or(o.any, l_off);
      if (lc == 1) bit_or(o.no_in, l_off);
      if (lc == 2) bit_or(o.no_out, l_off);
    }
    if (rc >= 0) {
      bit_or(o.any, r_off);
      if (rc == 1) bit_or(o.no_in, r_off);
      if (rc == 2) bit_or(o.no_out, r_off);
    }
  }
  return end;
}

// Read2SdbgS2::Initialize, the mercy step (read_to_sdbg_s2.cpp:172-254) for one read: every (k+1)-mer between a
// "no out" k-mer and the next "no in" k-mer with no solid k-mer in between becomes solid.  Reads the stage-1 bits,
// writes `mercy` (OR-ed into is_solid afterwards: has_solid_kmer must see the stage-1 state only).  Returns the number added.
// any bit set in [lo, hi)?
MHB_HD bool bits_any(const u32 *bits, u64 lo, u64 hi) {
  if (lo >= hi) return false;
  const u64 w0 = lo >> 5, w1 = (hi - 1) >> 5;
  for (u64 w = w0; w <= w1; ++w) {
    u32 v = bits[w];
    if (w == w0) v &= 0xFFFFFFFFu << (lo & 31);
    if (w == w1 && ((hi & 31) != 0)) v &= 0xFFFFFFFFu >> (32 - (hi & 31));
    if (v) return true;
  }
  return false;
}

MHB_HD u32 r2s_mercy_read(const PkgView &pv, u64 r, u32 k, const S1Out &o, u32 *mercy) {
  const u32 L = pv.L(r);
  if (L < k + 1) return 0;
  const u64 b = pv.base(r);
  // most reads have no tip at all: two word-level looks instead of a walk over every position
  if (!bits_any(o.no_out, b, b + L) || !bits_any(o.no_in, b, b + L)) return 0;
  int first_0_out = -1, last_0_in = -1;
  bool any = false;
  for (u32 i = 0; i + k <= L; ++i) {
    if (bit_at(o.no_out, b + i) && first_0_out < 0) first_0_out = (int)i;
    if (bit_at(o.no_in, b + i)) last_0_in = (int)i;
    any = any || bit_at(o.any, b + i);
  }
  if (!any) return 0;                                                // the read has no candidate at all (:172)
  if (first_0_out < 0 || last_0_in < first_0_out) return 0;          // :197-199
  int last_no_out = -1;
  u32 added = 0;
  for (u32 i = 0; i + k <= L; ++i) {
    if (bit_at(o.no_in, b + i) && last_no_out != -1) {
      for (u32 j = (u32)last_no_out; j < i; ++j) bit_or(mercy, b + j);
      added += i - (u32)last_no_out;
    }
    // has_solid_kmer[i] (:193, :204-208): a candidate of any code at i, or a solid edge starting at i or at i-1
    bool hs = bit_at(o.any, b + i);
    if (i + k < L && bit_at(o.is_solid, b + i)) hs = true;
    if (i > 0 && bit_at(o.is_solid, b + i - 1)) hs = true;
    if (hs) last_no_out = -1;
    if (bit_at(o.no_out, b + i)) last_no_out = (int)i;
  }
  return added;
}

#if defined(__CUDACC__)
// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------

// `.bin` image (file orientation, u32 length + words per read) -> package-orientation words (reversed reads)
__global__ void __launch_bounds__(256) k_r2s_reverse(const u32 *__restrict__ bin, u64 n_reads, u32 fixed_len,
                                                     const u64 *__restrict__ rec_off, PkgView pv, u32 *__restrict__ out,
                                                     u64 n_out_words) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < n_out_words; t += (u64)gridDim.x * 256) {
    u64 r;
    u32 j;
    if (fixed_len) {
      r = t / pv.fixed_words;
      j = (u32)(t - r * pv.fixed_words);
    } else {
      r = PkgView::find(pv.word_off, n_reads, t);
      j = (u32)(t - pv.word_off[r]);
    }
    const u32 *src = bin + (fixed_len ? r * (u64)(1 + pv.fixed_words) : rec_off[r]);
    const u32 L = src[0];  // file length; 0 -> one fake 'A'
    u32 w = 0;
    for (u32 c = 0; c < 16; ++c) {
      const u32 i = 16 * j + c;
      if (i < L) w |= base_at(src + 1, L - 1 - i) << (30 - 2 * c);
    }
    out[t] = w;
  }
}

// per-read geometry (r2s_read_geom) of a variable-length `.bin` chunk, rec_off rebased to the chunk
__global__ void __launch_bounds__(256) k_r2s_chunk_geom(const u32 *__restrict__ bin, const u64 *__restrict__ rec_off, u64 n_reads,
                                                       u32 k, u32 *__restrict__ len, u32 *__restrict__ words,
                                                       u32 *__restrict__ s1, u32 *__restrict__ edges) {
  for (u64 r = (u64)blockIdx.x * 256 + threadIdx.x; r < n_reads; r += (u64)gridDim.x * 256) {
    u32 l, w, s, e;
    r2s_read_geom(bin[rec_off[r]], k, l, w, s, e);
    len[r] = l;
    words[r] = w;
    s1[r] = s;
    edges[r] = e;
  }
}

// row i of a stage-1 buffer: the whole record (info == nullptr), or the narrow layout - the NW key words and the row
// index i, read_info in info[i]
template <int NW>
__device__ __forceinline__ void s1_store(u32 *recs, u64 *info, u64 i, const u32 (&rec)[NW + 2]) {
  if (!info) {
    st_rec<NW + 2>(recs, i, rec);
    return;
  }
  u32 *o = recs + i * (NW + 1);
#pragma unroll
  for (int j = 0; j < NW; ++j) o[j] = rec[j];
  o[NW] = (u32)i;
  info[i] = ((u64)rec[NW] << 32) | rec[NW + 1];
}

// stage-1 records in the reference's bucket input order: record s1_off[r] + e at row at0 + s1_off[r] + e
template <int NW>
__global__ void __launch_bounds__(256) k_r2s_s1_extract(PkgView pv, u32 k, u32 *__restrict__ recs, u64 *__restrict__ info,
                                                       u64 at0, u64 n_recs) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < n_recs; t += (u64)gridDim.x * 256) {
    u64 r;
    u32 e;
    if (pv.fixed_len) {
      const u32 per = pv.fixed_len - k + 4;
      r = t / per;
      e = (u32)(t - r * per);
    } else {
      r = PkgView::find(pv.s1_off, pv.n_reads, t);
      e = (u32)(t - pv.s1_off[r]);
    }
    const u32 L = pv.L(r);
    u32 p, want;
    s1_emission(L, k, e, p, want);
    u32 rec[NW + 2];
    make_s1_record<NW>(pv.ptr(r), div_ceil(L, 16), L, k, p, want, pv.base(r), rec);
    s1_store<NW>(recs, info, at0 + t, rec);
  }
}

// Stage 1 in rounds (libraries whose records do not fit the device at once; base_engine.cpp:54-141, :254-281 plan Lv1
// passes over bucket ranges the same way).  One warp per read, lane = emission index; the record's 16-bit bucket id is
// the top of key word 0.  No atomics on the records and no reordering: a round's records come out in the same order
// k_r2s_s1_extract gives them, so the stable bucket partition and kmsort see the reference's bucket input order.
//   kS1Hist : hist[bucket id] += 1 over the whole library (the round planner's input)
//   kS1Count: per_read[r] = number of records of read r with bucket id in [lo, hi]
//   kS1Write: those records, stored at rows at0 + off[r] on (off = exclusive scan of the counts)
enum { kS1Hist = 0, kS1Count = 1, kS1Write = 2 };
template <int NW, int MODE>
__global__ void __launch_bounds__(256) k_r2s_s1_range(PkgView pv, u32 k, u32 lo, u32 hi, unsigned long long *__restrict__ hist,
                                                     u32 *__restrict__ per_read, const u64 *__restrict__ off, u32 *__restrict__ recs,
                                                     u64 *__restrict__ info = nullptr, u64 at0 = 0) {
  const u32 lane = lane_id(), lt = lanemask_lt();
  const u64 n_warps = (u64)gridDim.x * 8;
  for (u64 r = ((u64)blockIdx.x * 256 + threadIdx.x) >> 5; r < pv.n_reads; r += n_warps) {
    const u32 L = pv.L(r);
    u64 run = MODE == kS1Write ? at0 + off[r] : 0;
    if (L >= k + 1) {
      const u32 n_e = L - k + 4, nwords = div_ceil(L, 16);
      const u32 *s = pv.ptr(r);
      const u64 base = pv.base(r);
      for (u32 e0 = 0; e0 < n_e; e0 += 32) {
        const u32 e = e0 + lane;
        u32 rec[NW + 2];
        bool in = false;
        if (e < n_e) {
          u32 p, want;
          s1_emission(L, k, e, p, want);
          make_s1_record<NW>(s, nwords, L, k, p, want, base, rec);
          const u32 b = rec[0] >> 16;
          if (MODE == kS1Hist) atomicAdd(&hist[b], 1ull);
          in = b >= lo && b <= hi;
        }
        if (MODE == kS1Hist) continue;
        const u32 mask = __ballot_sync(0xffffffffu, in);
        if (MODE == kS1Write && in) s1_store<NW>(recs, info, run + __popc(mask & lt), rec);
        run += __popc(mask);
      }
    }
    if (MODE == kS1Count && lane == 0) per_read[r] = (u32)run;
  }
}

// Stage 1 on several GPUs: every record of a rank's share straight into the receive buffer of the rank that owns its
// leading byte, in global read order, one round over bucket ranges at a time.  A record of bucket id b goes to owner
// o = owner[b >> 8] only when round_lo[o] <= b <= round_hi[o] (an empty range, lo > hi, sends nothing to o); both modes
// apply the same test, so the counts and the stores agree.  One warp per read, lane = emission index, as
// k_r2s_s1_range; the lanes of a batch are grouped by owner (__match_any_sync) and s_run holds, per owner, the read's
// records placed so far.
//   kS1OwnerCount: per_read[o * n_reads + r] = records of read r for owner o in the round
//   kS1OwnerWrite: the record goes to row my_off[o] + off[o * (n_reads + 1) + r] + its rank among read r's records for
//                  o, of owner o's buffer rec_base[o] (narrow layout: read_info at that row of info_base[o]; the row
//                  index the record carries is that owner-local row of the round)
// The shares ascend with the rank and my_off[o] puts this rank's block after those of the lower ranks, so every owner
// holds the records of its round in global read order - the reference's bucket input order - without an atomic.
static constexpr int kS1MaxOwners = 16;
enum { kS1OwnerCount = 0, kS1OwnerWrite = 1 };
template <int NW, int MODE>
__global__ void __launch_bounds__(256) k_r2s_s1_owners(PkgView pv, u32 k, const uint8_t *__restrict__ owner, u32 n_owners,
                                                      const u32 *__restrict__ round_lo, const u32 *__restrict__ round_hi,
                                                      u32 *__restrict__ per_read, const u64 *__restrict__ off,
                                                      const u64 *__restrict__ rec_base, const u64 *__restrict__ info_base,
                                                      const u64 *__restrict__ my_off) {
  __shared__ u32 s_run[8][kS1MaxOwners];
  const u32 lane = lane_id(), lt = lanemask_lt(), warp = threadIdx.x >> 5;
  const u64 n_warps = (u64)gridDim.x * 8;
  for (u64 r = ((u64)blockIdx.x * 256 + threadIdx.x) >> 5; r < pv.n_reads; r += n_warps) {  // warp-uniform
    if (lane < (u32)kS1MaxOwners) s_run[warp][lane] = 0;
    __syncwarp();
    const u32 L = pv.L(r);
    if (L >= k + 1) {
      const u32 n_e = L - k + 4, nwords = div_ceil(L, 16);
      const u32 *s = pv.ptr(r);
      const u64 base = pv.base(r);
      for (u32 e0 = 0; e0 < n_e; e0 += 32) {
        const u32 e = e0 + lane;
        u32 rec[NW + 2];
        u32 o = 0xFFFFFFFFu;
        if (e < n_e) {
          u32 p, want;
          s1_emission(L, k, e, p, want);
          make_s1_record<NW>(s, nwords, L, k, p, want, base, rec);
          const u32 b = rec[0] >> 16;
          o = __ldg(owner + (b >> 8));
          if (b < __ldg(round_lo + o) || b > __ldg(round_hi + o)) o = 0xFFFFFFFFu;  // not in o's range this round
        }
        const bool in = o != 0xFFFFFFFFu;
        const u32 peers = __match_any_sync(0xffffffffu, o);
        if (MODE == kS1OwnerWrite && in) {
          const u64 row = my_off[o] + off[(u64)o * (pv.n_reads + 1) + r] + s_run[warp][o] + __popc(peers & lt);
          s1_store<NW>(reinterpret_cast<u32 *>(rec_base[o]), info_base ? reinterpret_cast<u64 *>(info_base[o]) : nullptr,
                       row, rec);
        }
        __syncwarp();
        if (in && lane == (u32)__ffs(peers) - 1) s_run[warp][o] += __popc(peers);
        __syncwarp();
      }
    }
    if (MODE == kS1OwnerCount && lane < n_owners) per_read[(u64)lane * pv.n_reads + r] = s_run[warp][lane];
    __syncwarp();
  }
}

// The bucket partition of the narrow layout, whose records may be wider than mhb_sort_records takes: (word 0, row)
// pairs are sorted stably on the bucket id, then the records gathered in that order.  Row r sits at position r and its
// index word says r, so the gathered records keep their side-array rows.
__global__ void __launch_bounds__(256) k_r2s_s1_pairs(const u32 *__restrict__ recs, u64 n, u32 rw, u32 *__restrict__ pairs) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    pairs[2 * i] = recs[i * rw];
    pairs[2 * i + 1] = (u32)i;
  }
}
__global__ void __launch_bounds__(256) k_r2s_s1_gather(const u32 *__restrict__ recs, const u32 *__restrict__ pairs, u64 n,
                                                      u32 rw, u32 *__restrict__ out) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < n * rw; t += (u64)gridDim.x * 256) {
    const u64 i = t / rw;
    out[t] = recs[(u64)pairs[2 * i + 1] * rw + (t - i * rw)];
  }
}

// first record of every 16-bit bucket in records sorted by their two leading bytes: bstart[b], b = 0..65536
__global__ void k_r2s_bucket_bounds(const u32 *__restrict__ recs, u64 n, u32 rw, u64 *__restrict__ bstart) {
  const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > MHB_NUM_BUCKETS) return;
  u64 lo = 0, hi = n;  // first record with (word0 >> 16) >= b
  while (lo < hi) {
    const u64 mid = (lo + hi) >> 1;
    if ((recs[mid * rw] >> 16) < b) lo = mid + 1; else hi = mid;
  }
  bstart[b] = lo;
}

struct KmSeg {
  u64 start;  // first record
  u64 len;
};

// one kmsort level: thread t permutes range segs[t] on byte kb (level 0: the 65 536 buckets, radix_sort_entry
// kmsort.h:103-117) and queues the children above the insertion-sort threshold for byte kb - 1.  Children of 2..64
// records (and buckets that small) are NOT sorted here - 256 serial insertion sorts per thread were 80 % of the first
// version's time -: every range start is marked in the bit array `bnd`, and k_r2s_kmsort_finish sorts all small ranges
// of all levels afterwards, one thread per range (their order does not depend on anything outside the range).
template <int RW>
__global__ void __launch_bounds__(128) k_r2s_kmsort_level(u32 *__restrict__ recs, u32 nw, int kb, const KmSeg *__restrict__ segs,
                                                         const u64 *__restrict__ bstart, u64 n_segs, KmSeg *__restrict__ next,
                                                         unsigned long long *__restrict__ n_next, u64 next_cap,
                                                         u32 *__restrict__ bnd) {
  const u64 t = (u64)blockIdx.x * 128 + threadIdx.x;
  if (t >= n_segs) return;
  u64 start, len;
  if (bstart) {  // level 0
    start = bstart[t];
    len = bstart[t + 1] - start;
    if (len == 0) return;
    bit_or(bnd, start);
    if (len <= (u64)kKmInsertThreshold) return;
  } else {
    start = segs[t].start;
    len = segs[t].len;
  }
  u32 count[256], last[256];
  u32 *a = recs + start * RW;
  km_radix_range<RW>(a, (u32)len, nw, kb, count, last);
  u32 b0 = 0;
  for (int i = 0; i < 256; ++i) {
    const u32 c = count[i];
    if (c) bit_or(bnd, start + b0);
    if (c > (u32)kKmInsertThreshold && kb > 0) {  // :84 / :93: no level below byte 0
      const unsigned long long slot = atomicAdd(n_next, 1ull);
      if (slot < next_cap) next[slot] = KmSeg{start + b0, c};
    }
    b0 += c;
  }
}

// length of the marked range starting at i if it has at most `lim` records, else 0 (bit n counts as a boundary)
MHB_HD u32 km_small_range(const u32 *bnd, u64 n, u64 i, u32 lim) {
  for (u32 d = 1; d <= lim; ++d) {
    if (i + d >= n || bit_at(bnd, i + d)) return d;
  }
  return 0;
}

// the insertion sorts of every level (kmsort.h:88-99, :106-108): one thread per marked range of 2..64 records.  A
// marked range of more than 64 records with no mark inside went through every radix level as a single bin: all its
// keys are equal.
template <int RW>
__global__ void __launch_bounds__(256) k_r2s_kmsort_finish(u32 *__restrict__ recs, u64 n, u32 nw, const u32 *__restrict__ bnd,
                                                          const u32 *__restrict__ todo) {
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    if (!bit_at(todo ? todo : bnd, i)) continue;  // todo: only the small ranges nobody has sorted yet
    const u32 len = km_small_range(bnd, n, i, (u32)kKmInsertThreshold);
    if (len >= 2) km_insertion<RW>(recs + i * RW, len, nw);
  }
}

// ------------------------------------------------------------------------------------------------
// kmsort on shared memory (the default path; k_r2s_kmsort_level above remains the in-place form used for ranges that do
// not fit).  Level 0: one CTA per bucket - tags + histogram by all threads (the bucket is contiguous), the walk by
// thread 0 on shared-memory tags (km_walk_src), the records gathered into the second buffer by all threads.  Levels
// >= 1: one WARP per range of at most km_wcap(RW) records staged in shared memory: tags, walk, the insertion sorts of
// the children of 2..64 records (one lane per child, on the index array), write-back in place.
// `todo` marks the small ranges nobody has sorted yet (k_r2s_kmsort_finish), `bnd` every range start.
// ------------------------------------------------------------------------------------------------
template <int RW>
__global__ void __launch_bounds__(128) k_r2s_km_bucket(const u32 *__restrict__ in, u32 *__restrict__ out, const u64 *__restrict__ bstart,
                                                      u32 nw, int kb, u32 cap, uint16_t *__restrict__ src_g, u32 *__restrict__ bnd,
                                                      u32 *__restrict__ todo, KmSeg *__restrict__ next,
                                                      unsigned long long *__restrict__ n_next, u64 next_cap) {
  extern __shared__ uint8_t s_tags[];
  __shared__ u32 s_cnt[256], s_last[256], s_beg[256];
  const u32 tid = threadIdx.x;
  const u64 start = bstart[blockIdx.x];
  const u64 len64 = bstart[blockIdx.x + 1] - start;
  if (len64 == 0) return;
  const u32 *a = in + start * RW;
  u32 *o = out + start * RW;
  if (tid == 0) bit_or(bnd, start);
  if (len64 <= (u64)kKmInsertThreshold) {
    for (u32 w = tid; w < (u32)len64 * RW; w += 128) o[w] = a[w];
    if (tid == 0 && len64 >= 2) bit_or(todo, start);
    return;
  }
  if (len64 > (u64)cap || len64 > 65535ull) {  // does not fit: the in-place walk on global memory, then the copy
    if (tid == 0) km_radix_range<RW>(const_cast<u32 *>(a), (u32)len64, nw, kb, s_cnt, s_last);
    __syncthreads();
    for (u64 w = tid; w < len64 * RW; w += 128) o[w] = a[w];
  } else {
    const u32 len = (u32)len64;
    for (u32 i = tid; i < 256; i += 128) s_cnt[i] = 0;
    __syncthreads();
    for (u32 i = tid; i < len; i += 128) {
      const u32 t = km_byte_mem(a + (u64)i * RW, nw, kb);
      s_tags[i] = (uint8_t)t;
      atomicAdd(&s_cnt[t], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      u32 acc = 0;
      for (int i = 0; i < 256; ++i) {
        s_last[i] = acc;
        acc += s_cnt[i];
      }
      km_walk_src<uint16_t>(s_tags, len, s_cnt, s_last, src_g + start);
    }
    __syncthreads();
    const uint16_t *src = src_g + start;
    for (u32 q = tid; q < len; q += 128) {
      u32 r[RW];
      ld_rec<RW>(a, src[q], r);
      st_rec<RW>(o, q, r);
    }
  }
  if (tid == 0) {
    u32 acc = 0;
    for (int i = 0; i < 256; ++i) {
      s_beg[i] = acc;
      acc += s_cnt[i];
    }
  }
  __syncthreads();
  for (u32 b = tid; b < 256; b += 128) {
    const u32 c = s_cnt[b];
    if (!c) continue;
    bit_or(bnd, start + s_beg[b]);
    if (kb == 0) continue;  // kmsort.h:84 / :93: no level below byte 0
    if (c > (u32)kKmInsertThreshold) {
      const unsigned long long slot = atomicAdd(n_next, 1ull);
      if (slot < next_cap) next[slot] = KmSeg{start + s_beg[b], c};
    } else if (c >= 2) {
      bit_or(todo, start + s_beg[b]);
    }
  }
}

static constexpr int kKmWarps = 8;
template <int RW>
__host__ __device__ constexpr size_t km_warp_smem() {  // per warp: staged records, index array, tags, 3 x 256 counters
  // rounded up to 16 bytes: the next warp's staged records and counters start there (an odd km_wcap would leave them
  // 2 bytes off a word boundary)
  return ((size_t)km_wcap(RW) * RW * 4 + (size_t)km_wcap(RW) * 2 + (size_t)((km_wcap(RW) + 3) & ~3u) + 3 * 256 * 4 + 15) &
         ~(size_t)15;
}

template <int RW>
__global__ void __launch_bounds__(kKmWarps * 32) k_r2s_km_warp(u32 *__restrict__ recs, u32 nw, int kb, const KmSeg *__restrict__ segs,
                                                              u64 n_segs, KmSeg *__restrict__ next,
                                                              unsigned long long *__restrict__ n_next, u64 next_cap,
                                                              u32 *__restrict__ bnd, u32 *__restrict__ todo) {
  constexpr u32 WCAP = km_wcap(RW);
  extern __shared__ __align__(16) uint8_t s_raw[];
  const u32 lane = lane_id(), warp = threadIdx.x >> 5;
  uint8_t *base = s_raw + (size_t)warp * km_warp_smem<RW>();
  u32 *staged = reinterpret_cast<u32 *>(base);
  u32 *cnt = staged + (size_t)WCAP * RW;
  u32 *last = cnt + 256;
  u32 *beg = last + 256;
  uint16_t *src = reinterpret_cast<uint16_t *>(beg + 256);
  uint8_t *tags = reinterpret_cast<uint8_t *>(src + WCAP);
  for (u64 sg = (u64)blockIdx.x * kKmWarps + warp; sg < n_segs; sg += (u64)gridDim.x * kKmWarps) {
    const u64 start = segs[sg].start;
    const u32 len = (u32)segs[sg].len;
    u32 *a = recs + start * RW;
    __syncwarp();
    const bool fits = len <= WCAP;
    if (!fits) {
      if (lane == 0) km_radix_range<RW>(a, len, nw, kb, cnt, last);  // in place on global memory, counters in shared
      __syncwarp();
    } else {
      for (u32 w = lane; w < len * RW; w += 32) staged[w] = a[w];
      for (u32 i = lane; i < 256; i += 32) cnt[i] = 0;
      __syncwarp();
      for (u32 i = lane; i < len; i += 32) {
        const u32 t = km_byte_mem(staged + i * RW, nw, kb);
        tags[i] = (uint8_t)t;
        atomicAdd(&cnt[t], 1u);
      }
      __syncwarp();
    }
    {  // bin starts: 8 bins per lane + warp scan
      u32 c8[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c8[j] = cnt[lane * 8 + j];
        sum += c8[j];
      }
      u32 inc = sum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const u32 v = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= (u32)d) inc += v;
      }
      u32 acc = inc - sum;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        beg[lane * 8 + j] = acc;
        if (fits) last[lane * 8 + j] = acc;
        acc += c8[j];
      }
    }
    __syncwarp();
    if (fits) {
      if (lane == 0) km_walk_src<uint16_t>(tags, len, cnt, last, src);
      __syncwarp();
      if (kb > 0) {  // the children of 2..64 records: insertion sort on their slice of the index array
        for (u32 b = lane; b < 256; b += 32) {
          const u32 c = cnt[b];
          if (c >= 2 && c <= (u32)kKmInsertThreshold) km_insertion_idx<uint16_t>(staged, RW, src + beg[b], c, nw);
        }
      }
      __syncwarp();
      for (u32 w = lane; w < len * RW; w += 32) {
        const u32 q = w / RW, j = w - q * RW;
        a[w] = staged[(u32)src[q] * RW + j];
      }
    }
    for (u32 b = lane; b < 256; b += 32) {
      const u32 c = cnt[b];
      if (!c) continue;
      bit_or(bnd, start + beg[b]);
      if (kb == 0) continue;
      if (c > (u32)kKmInsertThreshold) {
        const unsigned long long slot = atomicAdd(n_next, 1ull);
        if (slot < next_cap) next[slot] = KmSeg{start + beg[b], c};
      } else if (c >= 2 && !fits) {
        bit_or(todo, start + beg[b]);
      }
    }
  }
}

static constexpr int kS1HistSmem = 2048;

// Lv2Postprocess of stage 1: the thread whose record opens a (k-1)-mer group walks it (info: the narrow layout's
// read_info side array, nullptr for the wide layout)
template <int RW>
__global__ void __launch_bounds__(256) k_r2s_s1_post(const u32 *__restrict__ recs, const u64 *__restrict__ info, u64 n, u32 nw,
                                                    u32 k, int m, PkgView pv, S1Out o, int need_mercy,
                                                    unsigned long long *__restrict__ mul_hist, uint8_t *__restrict__ cand) {
  __shared__ u32 s_hist[kS1HistSmem];
  for (int i = threadIdx.x; i < kS1HistSmem; i += 256) s_hist[i] = 0;
  __syncthreads();
  for (u64 i = (u64)blockIdx.x * 256 + threadIdx.x; i < n; i += (u64)gridDim.x * 256) {
    const bool head = i == 0 || s1_diff_km1(recs + (i - 1) * RW, recs + i * RW, k);
    if (head) {
      u32 hv[16], nh;
      s1_group(recs, info, n, i, RW, nw, k, m, pv, o, need_mercy != 0, hv, nh, cand);
      for (u32 q = 0; q < nh; ++q) {
        const u32 c = hv[q];
        if (c < (u32)kS1HistSmem) atomicAdd(&s_hist[c], 1u);
        else atomicAdd(&mul_hist[c > MHB_MAX_MUL ? MHB_MAX_MUL : c], 1ull);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kS1HistSmem; i += 256)
    if (s_hist[i]) atomicAdd(&mul_hist[i], (unsigned long long)s_hist[i]);
}

__global__ void __launch_bounds__(256) k_r2s_mercy(PkgView pv, u32 k, S1Out o, u32 *__restrict__ mercy,
                                                  unsigned long long *__restrict__ n_mercy) {
  u32 added = 0;
  for (u64 r = (u64)blockIdx.x * 256 + threadIdx.x; r < pv.n_reads; r += (u64)gridDim.x * 256)
    added += r2s_mercy_read(pv, r, k, o, mercy);
  for (int d = 16; d; d >>= 1) added += __shfl_xor_sync(0xffffffffu, added, d);
  if (lane_id() == 0 && added) atomicAdd(n_mercy, (unsigned long long)added);
}

__global__ void __launch_bounds__(256) k_r2s_or_words(u32 *__restrict__ dst, const u32 *__restrict__ src, u64 n_words) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < n_words; t += (u64)gridDim.x * 256) dst[t] |= src[t];
}

// ---- the list form of the candidates: count -> scan32 -> write over the candidate bytes of a stage-1 round, tiles of
// kCandTile records (kCandPer consecutive records per thread), entries in record order ----
static constexpr int kCandPer = 4, kCandTile = 256 * kCandPer;
__global__ void __launch_bounds__(256) k_r2s_cand_count(const uint8_t *__restrict__ cand, u64 n, u32 *__restrict__ tile_n) {
  __shared__ u32 s_w[8];
  const u64 i0 = (u64)blockIdx.x * kCandTile + (u64)threadIdx.x * kCandPer;
  u32 c = 0;
  for (int j = 0; j < kCandPer; ++j)
    if (i0 + j < n) c += cand_count(cand[i0 + j]);
  for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if (lane_id() == 0) s_w[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 t = 0;
    for (int w = 0; w < 8; ++w) t += s_w[w];
    tile_n[blockIdx.x] = t;
  }
}

// recs: the round's records (rw words, read_info as s1_info reads it); tile_off: the scan of k_r2s_cand_count's tiles
__global__ void __launch_bounds__(256) k_r2s_cand_write(const uint8_t *__restrict__ cand, u64 n, const u32 *__restrict__ recs,
                                                        const u64 *__restrict__ info, u32 rw, u32 nw,
                                                        const u64 *__restrict__ tile_off, u64 *__restrict__ out) {
  __shared__ u32 s_w[8];
  const u64 i0 = (u64)blockIdx.x * kCandTile + (u64)threadIdx.x * kCandPer;
  u32 c = 0;
  for (int j = 0; j < kCandPer; ++j)
    if (i0 + j < n) c += cand_count(cand[i0 + j]);
  // exclusive prefix of c over the block: inclusive warp scan, then the sums of the warps before
  const u32 lane = lane_id(), warp = threadIdx.x >> 5;
  u32 inc = c;
  for (int d = 1; d < 32; d <<= 1) {
    const u32 v = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= (u32)d) inc += v;
  }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  u64 at = tile_off[blockIdx.x] + inc - c;
  for (u32 w = 0; w < warp; ++w) at += s_w[w];
  for (int j = 0; j < kCandPer; ++j) {
    const u64 i = i0 + j;
    if (i >= n || !cand[i]) continue;
    u64 e[2];
    const u32 ne = cand_entries(cand[i], s1_info(recs + i * rw, nw, info), e);
    for (u32 q = 0; q < ne; ++q) out[at++] = e[q];
  }
}

// the n entries e[] into the candidate planes of o (each on the caller's word grid, indexed by global base)
__global__ void __launch_bounds__(256) k_r2s_cand_scatter(const u64 *__restrict__ e, u64 n, S1Out o) {
  for (u64 t = (u64)blockIdx.x * 256 + threadIdx.x; t < n; t += (u64)gridDim.x * 256) cand_mark(o, e[t]);
}

// stage-2 items of edge position t (global index over all reads): which $-variants exist (read_to_sdbg_s2.cpp:389-431)
MHB_HD u32 r2s_edge_types(const u32 *is_solid, bool sure, u64 b, u32 i, u32 L, u32 k) {
  if (!(sure || bit_at(is_solid, b + i))) return 0;
  u32 types = 2u;  // bit t = type t present
  if (i == 0 || !(sure || bit_at(is_solid, b + i - 1))) types |= 1u;
  if (i + k == L - 1 || !(sure || bit_at(is_solid, b + i + 1))) types |= 4u;
  return types;
}

// MODE kS2Count: total number of items -> *cursor.  kS2Write: items appended at recs[*cursor ...] in no particular
// order (whole-record sort keys).  For stage 2 in rounds: kS2Hist adds every item's 16-bit bucket id (top of word 0)
// to hist[65536]; kS2Range appends only the items whose bucket id lies in [lo, hi].  On several GPUs, kS2Owner hands
// an item of bucket id b to `sink`, which stores it in the receive buffer of the rank o = sink.owner[b >> 8], when
// round_lo[o] <= b <= round_hi[o] (the round's range of o; lo > hi: nothing); each block first folds the ranges into a
// shared table of second-byte ranges per leading byte (blocks of 256 threads).  One thread per (k+1)-mer position.
enum { kS2Count = 0, kS2Write = 1, kS2Hist = 2, kS2Range = 3, kS2Owner = 4 };
template <int W, int MODE>
__global__ void __launch_bounds__(256) k_r2s_s2_extract(PkgView pv, u32 k, const u32 *__restrict__ is_solid, int sure, u64 n_edges,
                                                       u32 *__restrict__ recs, unsigned long long *__restrict__ cursor, u64 capacity,
                                                       u32 lo = 0, u32 hi = 0, unsigned long long *__restrict__ hist = nullptr,
                                                       OwnerSink sink = {}, const u32 *__restrict__ round_lo = nullptr,
                                                       const u32 *__restrict__ round_hi = nullptr) {
  // kS2Owner: the round's second-byte range of every leading byte B's owner, (first | last << 8) (first > last: none)
  __shared__ u32 s_rng[MODE == kS2Owner ? 256 : 1];
  if (MODE == kS2Owner) {
    const u32 B = threadIdx.x, o = sink.owner[B], a = max(round_lo[o], B << 8), z = min(round_hi[o], B << 8 | 255u);
    s_rng[B] = a <= z ? ((a & 255u) | (z & 255u) << 8) : 255u;
    __syncthreads();
  }
  const u32 lane = lane_id();
  u64 t0 = (u64)blockIdx.x * 256 + threadIdx.x;
  const u64 step = (u64)gridDim.x * 256;
  unsigned long long local_total = 0;
  for (u64 base_t = t0 - lane; base_t < n_edges; base_t += step) {  // warp-uniform loop
    const u64 t = base_t + lane;
    u32 types = 0, pal = 0, L = 0, i = 0;
    u64 r = 0;
    if (t < n_edges) {
      if (pv.fixed_len) {
        const u32 per = pv.fixed_len - k;
        r = t / per;
        i = (u32)(t - r * per);
      } else {
        r = PkgView::find(pv.edge_off, pv.n_reads, t);
        i = (u32)(t - pv.edge_off[r]);
      }
      L = pv.L(r);
      types = r2s_edge_types(is_solid, sure != 0, pv.base(r), i, L, k);
      if (types) pal = edge_is_palindrome<W>(pv.ptr(r), div_ceil(L, 16), k, i) ? 1u : 0u;
    }
    const u32 cnt = (u32)__popc(types) * (pal ? 1u : 2u);
    if (MODE == kS2Count) {
      local_total += cnt;
      continue;
    }
    if (MODE == kS2Hist || MODE == kS2Range || MODE == kS2Owner) {
      // one (type, strand) slot at a time: a warp-aggregated append per slot for the items in range
      const u32 *s = pv.ptr(r);
      const u32 nwords = div_ceil(L, 16);
      for (u32 slot = 0; slot < 6; ++slot) {
        const u32 type = slot >> 1, strand = slot & 1u;
        u32 rec[W];
        bool in = false;
        if (((types >> type) & 1u) && (strand == 0 || !pal)) {
          make_r2s_item<W>(s, nwords, k, i, strand, type, rec);
          const u32 b = rec[0] >> 16;
          if (MODE == kS2Hist) atomicAdd(&hist[b], 1ull);
          if (MODE == kS2Owner) {
            const u32 x = s_rng[b >> 8], c = b & 255u;
            in = c >= (x & 255u) && c <= (x >> 8);
          } else {
            in = b >= lo && b <= hi;
          }
        }
        if (MODE == kS2Hist) continue;
        const u32 mask = __ballot_sync(0xffffffffu, in);
        if (!mask) continue;
        if (MODE == kS2Owner) {
          sink.template put<W>(in, rec, mask, lane, lanemask_lt());
          continue;
        }
        unsigned long long wbase = 0;
        if (lane == 0) wbase = atomicAdd(cursor, (unsigned long long)__popc(mask));
        wbase = __shfl_sync(0xffffffffu, wbase, 0);
        const u64 dst = wbase + __popc(mask & lanemask_lt());
        if (in && dst < capacity) st_rec<W>(recs, dst, rec);
      }
      continue;
    }
    u32 inc = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 v = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= (u32)d) inc += v;
    }
    const u32 warp_total = __shfl_sync(0xffffffffu, inc, 31);
    unsigned long long wbase = 0;
    if (lane == 31 && warp_total) wbase = atomicAdd(cursor, (unsigned long long)warp_total);
    wbase = __shfl_sync(0xffffffffu, wbase, 31);
    u64 dst = wbase + inc - cnt;
    if (cnt) {
      const u32 *s = pv.ptr(r);
      const u32 nwords = div_ceil(L, 16);
      for (u32 type = 0; type < 3; ++type) {
        if (!((types >> type) & 1u)) continue;
        for (u32 strand = 0; strand < (pal ? 1u : 2u); ++strand) {
          u32 rec[W];
          make_r2s_item<W>(s, nwords, k, i, strand, type, rec);
          if (dst < capacity) st_rec<W>(recs, dst, rec);
          ++dst;
        }
      }
    }
  }
  if (MODE == kS2Count) {
    for (int d = 16; d; d >>= 1) local_total += __shfl_xor_sync(0xffffffffu, local_total, d);
    if (lane == 0 && local_total) atomicAdd(cursor, local_total);
  }
}

// ---- collapse runs of equal items (all bits but the 16 multiplicity bits) ----
template <int W>
__device__ __forceinline__ bool r2s_item_head(const u32 *recs, u64 i) {
  if (i == 0) return true;
  u32 a[W], b[W];
  ld_rec<W>(recs, i - 1, a);
  ld_rec<W>(recs, i, b);
  bool diff = ((a[W - 1] ^ b[W - 1]) & 0xFFFF0000u) != 0;
#pragma unroll
  for (int j = 0; j < W - 1; ++j) diff = diff || a[j] != b[j];
  return diff;
}

static constexpr int kDdThreads = 256, kDdItems = 4, kDdTile = kDdThreads * kDdItems;

// phase 1: heads per tile of 1024 items
template <int W>
__global__ void __launch_bounds__(kDdThreads) k_r2s_dd_count(const u32 *__restrict__ recs, u64 n, u32 *__restrict__ tile_heads) {
  __shared__ u32 s_scan[kDdThreads / 32 + 1];
  const u64 base = (u64)blockIdx.x * kDdTile + (u64)threadIdx.x * kDdItems;
  u32 c = 0;
#pragma unroll
  for (int j = 0; j < kDdItems; ++j)
    if (base + j < n && r2s_item_head<W>(recs, base + j)) ++c;
  u32 total;
  block_excl_scan<kDdThreads>(c, s_scan, total);
  if (threadIdx.x == 0) tile_heads[blockIdx.x] = total;
}

// phase 2: index of every head, in order
template <int W>
__global__ void __launch_bounds__(kDdThreads) k_r2s_dd_heads(const u32 *__restrict__ recs, u64 n, const u64 *__restrict__ tile_off,
                                                            u64 *__restrict__ heads) {
  __shared__ u32 s_scan[kDdThreads / 32 + 1];
  const u64 base = (u64)blockIdx.x * kDdTile + (u64)threadIdx.x * kDdItems;
  u32 flag = 0, c = 0;
#pragma unroll
  for (int j = 0; j < kDdItems; ++j)
    if (base + j < n && r2s_item_head<W>(recs, base + j)) {
      flag |= 1u << j;
      ++c;
    }
  u32 total;
  u64 off = tile_off[blockIdx.x] + block_excl_scan<kDdThreads>(c, s_scan, total);
#pragma unroll
  for (int j = 0; j < kDdItems; ++j)
    if ((flag >> j) & 1u) heads[off++] = base + j;
}

// phase 3: one item per run, stored multiplicity = 65535 - min(run length, kMaxMul) (read_to_sdbg_s2.cpp:572)
template <int W>
__global__ void __launch_bounds__(256) k_r2s_dd_build(const u32 *__restrict__ recs, u64 n, const u64 *__restrict__ heads, u64 n_heads,
                                                     u32 *__restrict__ out) {
  for (u64 j = (u64)blockIdx.x * 256 + threadIdx.x; j < n_heads; j += (u64)gridDim.x * 256) {
    const u64 i = heads[j];
    const u64 e = j + 1 < n_heads ? heads[j + 1] : n;
    const u64 cnt = e - i > MHB_MAX_MUL ? MHB_MAX_MUL : e - i;
    u32 r[W];
    ld_rec<W>(recs, i, r);
    r[W - 1] = (r[W - 1] & 0xFFFF0000u) | (u32)(65535u - cnt);
    st_rec<W>(out, j, r);
  }
}
#endif  // __CUDACC__

}  // namespace mhb
