// mhb_plan.cpp -- every host-side plan of libmhb: rounds over bucket ranges, owner ranges, read and sequence shares,
// streamed chunks and mercy segments, and the C ABI entry points that expose them.  Host logic only: nothing here
// touches CUDA, so every plan can be checked without a GPU.
#include <string.h>

#include <algorithm>
#include <vector>

#include "mhb.h"
#include "mhb_internal.h"

namespace {

// The greedy cut every plan uses: atoms 0..n-1 of weight w(i), taken in order into contiguous runs.  A run closes
// before atom i when it holds weight (acc > 0) and acc + w(i) > target, so an atom above target is a run of its own.
// Appends the first atom of every run after the first to *cuts.  Returns n, or the first atom with w(i) > limit (the
// runs closed before it are in *cuts); the caller words that error.
template <class Weight, class Cuts>
uint64_t greedy_cut(uint64_t n, Weight w, uint64_t target, uint64_t limit, Cuts *cuts) {
  uint64_t acc = 0;
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t x = w(i);
    if (x > limit) return i;
    if (acc && acc + x > target) {
      cuts->push_back(i);
      acc = 0;
    }
    acc += x;
  }
  return n;
}

// n_ranks contiguous shares of n items, cut r at the item boundary whose weight before it is closest to r / n_ranks of
// the total (so a share is off its ideal weight by at most one item's); first gets n_ranks + 1 entries
template <class Weight>
void plan_shares(uint64_t n, uint32_t n_ranks, Weight weight, uint64_t *first) {
  uint64_t total = 0;
  for (uint64_t i = 0; i < n; ++i) total += weight(i);
  first[0] = 0;
  uint64_t b = 0, cum = 0;  // cum = weight of the items before b
  for (uint32_t r = 1; r < n_ranks; ++r) {
    const uint64_t target = (uint64_t)((unsigned __int128)total * r / n_ranks);
    while (b < n && cum + weight(b) <= target) cum += weight(b++);
    // the previous cut may already lie beyond this target (cum > target): then the cut stays where it is
    if (b < n && cum < target && cum + weight(b) - target < target - cum) cum += weight(b++);
    first[r] = b;
  }
  first[n_ranks] = n;
}

// prefix sums of a 65536-bin bucket histogram: the records in the buckets [lo, hi] are pre[hi + 1] - pre[lo]
std::vector<uint64_t> bucket_prefix(const uint64_t *h16) {
  std::vector<uint64_t> pre(65537, 0);
  for (uint32_t b = 0; b < 65536; ++b) pre[b + 1] = pre[b] + h16[b];
  return pre;
}

}  // namespace

void owner_bounds(const uint64_t *total256, int world, uint32_t *bounds, uint8_t *owner) {
  uint64_t cum[257];
  cum[0] = 0;
  for (int b = 0; b < 256; ++b) cum[b + 1] = cum[b] + total256[b];
  const uint64_t total = cum[256];
  bounds[0] = 0;
  for (int r = 1; r < world; ++r) {
    const uint32_t lo = bounds[r - 1] + 1, hi = 256 - (world - r);
    const uint64_t target = total * r / world;
    uint32_t best = lo;
    uint64_t bestd = ~0ull;
    for (uint32_t c = lo; c <= hi; ++c) {
      const uint64_t d = cum[c] > target ? cum[c] - target : target - cum[c];
      if (d < bestd) {
        bestd = d;
        best = c;
      }
    }
    bounds[r] = best;
  }
  bounds[world] = 256;
  for (int o = 0; o < world; ++o)
    for (uint32_t b = bounds[o]; b < bounds[o + 1]; ++b) owner[b] = (uint8_t)o;
}

int plan_bucket_rounds(const uint64_t *h256, const uint64_t *h16, uint32_t byte_lo, uint32_t byte_hi, uint64_t cap,
                       uint32_t cap_out, int rank, BucketRanges *ranges) {
  const auto split = [&](uint32_t b) { return h16 && h256[b] > cap; };
  std::vector<uint32_t> atom;  // the first bucket of every atom
  for (uint32_t b = byte_lo; b < byte_hi; ++b)
    for (uint32_t c = 0; c < (split(b) ? 256u : 1u); ++c) atom.push_back((b << 8) | c);
  std::vector<uint32_t> cuts;
  const uint64_t stop = greedy_cut(
      atom.size(), [&](uint64_t i) { return split(atom[i] >> 8) ? h16[atom[i]] : h256[atom[i] >> 8]; }, cap, cap, &cuts);
  ranges->clear();
  uint32_t lo = byte_lo << 8;
  for (uint32_t i : cuts) {
    ranges->push_back({lo, atom[i] - 1});
    lo = atom[i];
  }
  if (cuts.size() + (stop < atom.size() ? 0 : 1) > cap_out)
    return mhb_set_error(MHB_ERR_NOMEM, "round plan needs more than %u ranges", cap_out);
  if (stop < atom.size()) {
    const uint32_t a = atom[stop];
    if (!h16)
      return mhb_set_error(MHB_ERR_NOMEM, "leading byte 0x%02x alone holds %llu records, more than one round can take (%llu)",
                           a >> 8, (unsigned long long)h256[a >> 8], (unsigned long long)cap);
    char of[32] = "";
    if (rank >= 0) snprintf(of, sizeof(of), " of rank %d", rank);
    return mhb_set_error(MHB_ERR_NOMEM, "bucket 0x%04x alone holds %llu records, more than one round%s can take (%llu)", a,
                         (unsigned long long)h16[a], of, (unsigned long long)cap);
  }
  ranges->push_back({lo, (byte_hi << 8) - 1});
  return MHB_OK;
}

int plan_stage_rounds(const uint64_t *h16, uint64_t cap, BucketRanges *ranges) {
  uint64_t h256[256];
  fold_bucket_hist(h16, h256);
  return plan_bucket_rounds(h256, h16, 0, 256, cap, 65536, -1, ranges);
}

int plan_bucket_passes(uint64_t cap, const std::function<int(uint64_t *)> &top,
                       const std::function<int(const std::vector<uint32_t> &, uint64_t *)> &sub, BucketRanges *ranges,
                       std::vector<uint64_t> *pre) {
  uint64_t h256[256];
  CKR(top(h256));
  std::vector<uint32_t> over;  // leading bytes that alone exceed a round
  for (uint32_t b = 0; b < 256; ++b)
    if (h256[b] > cap) over.push_back(b);
  std::vector<uint64_t> h16(65536, 0);
  if (!over.empty()) CKR(sub(over, h16.data()));
  for (uint32_t b = 0; b < 256; ++b)
    if (h256[b] <= cap) h16[b << 8] = h256[b];
  if (plan_stage_rounds(h16.data(), cap, ranges)) return -1;
  *pre = bucket_prefix(h16.data());
  return MHB_OK;
}

int plan_owner_rounds(const uint64_t *const *h16, int world, const uint64_t *cap, OwnerPlan *cp) {
  cp->world = world;
  std::vector<uint64_t> tot(65536, 0);
  for (int s = 0; s < world; ++s)
    for (uint32_t b = 0; b < 65536; ++b) tot[b] += h16[s][b];
  uint64_t h256[256];
  fold_bucket_hist(tot.data(), h256);
  owner_bounds(h256, world, cp->bounds, cp->owner);
  std::vector<BucketRanges> sub(world);
  for (int o = 0; o < world; ++o)
    CKR(plan_bucket_rounds(h256, tot.data(), cp->bounds[o], cp->bounds[o + 1], cap[o], 65536, o, &sub[o]));
  cp->R = 1;
  for (int o = 0; o < world; ++o) cp->R = std::max(cp->R, (int)sub[o].size());
  std::vector<std::vector<uint64_t>> pre(world);
  for (int s = 0; s < world; ++s) pre[s] = bucket_prefix(h16[s]);
  const size_t RW = (size_t)cp->R * world;
  cp->lo.assign(RW, 1);
  cp->hi.assign(RW, 0);
  cp->n.assign(RW * world, 0);
  cp->off.assign(RW * world, 0);
  for (int t = 0; t < cp->R; ++t)
    for (int o = 0; o < world; ++o) {
      if (t >= (int)sub[o].size()) continue;  // empty range: nothing for o in this round
      const uint32_t a = sub[o][t].first, b = sub[o][t].second;
      cp->lo[(size_t)t * world + o] = a;
      cp->hi[(size_t)t * world + o] = b;
      uint64_t at = 0;
      for (int s = 0; s < world; ++s) {
        const size_t i = cp->at(t, o, s);
        cp->n[i] = pre[s][b + 1] - pre[s][a];
        cp->off[i] = at;
        at += cp->n[i];
      }
    }
  return MHB_OK;
}

void plan_chunks(const uint64_t *word_off, uint64_t stride_words, uint64_t extra_bytes, uint64_t n, uint64_t max_bytes,
                 std::vector<uint64_t> *first) {
  first->assign(1, 0);
  if (!word_off) {
    const uint64_t per = std::max<uint64_t>(1, max_bytes / (4 * stride_words + extra_bytes));
    for (uint64_t r = per; r < n; r += per) first->push_back(r);
  } else {
    greedy_cut(n, [&](uint64_t r) { return 4 * (word_off[r + 1] - word_off[r]) + extra_bytes; }, max_bytes, ~0ull, first);
  }
  if (n) first->push_back(n);
}

void edge_byte_starts(const uint32_t *edges, uint64_t n_edges, uint32_t WE, uint64_t start[257]) {
  uint64_t lo = 0;
  for (uint32_t b = 0; b < 256; ++b) {
    uint64_t l = lo, r = n_edges;  // first edge with leading byte >= b
    while (l < r) {
      const uint64_t mid = l + (r - l) / 2;
      if ((edges[mid * WE] >> 24) < b) l = mid + 1;
      else r = mid;
    }
    start[b] = lo = l;
  }
  start[256] = n_edges;
}

int plan_mercy_segments(const uint64_t start[257], uint32_t WE, uint64_t target, uint64_t limit, std::vector<uint32_t> *first) {
  first->assign(1, 0);
  const auto bytes = [&](uint64_t b) { return (start[b + 1] - start[b]) * WE * 4ull; };
  const uint64_t b = greedy_cut(256, bytes, target, limit, first);
  if (b < 256)
    return mhb_set_error(MHB_ERR_NOMEM, "leading byte 0x%02x alone holds %llu edges (%llu bytes), more than one mercy segment can take (%llu bytes)",
                         (uint32_t)b, (unsigned long long)(start[b + 1] - start[b]), (unsigned long long)bytes(b),
                         (unsigned long long)limit);
  first->push_back(256);
  return MHB_OK;
}

void plan_seq_shares(const uint32_t *len, uint64_t n, uint32_t k, uint32_t n_ranks, uint64_t *first) {
  plan_shares(n, n_ranks, [&](uint64_t i) { return seq_items(len[i], k); }, first);
}

void plan_read_shares(const uint32_t *bin, const ReadLibIndex &ix, uint64_t n_reads, uint32_t n_ranks, uint64_t *first) {
  plan_shares(n_reads, n_ranks, [&](uint64_t i) { return (uint64_t)bin[ix.word_of(i)]; }, first);
}

// ================================================================================================
// C ABI: argument checks around the plans above
// ================================================================================================
namespace {
// mhb_plan_rounds (shift 8: leading bytes) and mhb_plan_rounds16 (shift 0: bucket ids): the ranges closed before a
// failure are written too, at most cap_out of them
int plan_rounds_out(const uint64_t *hist256, const uint64_t *sub_hist, uint64_t max_records, uint32_t *lo_out,
                    uint32_t *hi_out, uint32_t cap_out, int shift) {
  if (!hist256 || !lo_out || !hi_out || max_records == 0 || cap_out == 0) {
    mhb_set_error(MHB_ERR_ARG, "bad round plan arguments");
    return -1;
  }
  BucketRanges r;
  const int rc = plan_bucket_rounds(hist256, sub_hist, 0, 256, max_records, cap_out, -1, &r);
  for (size_t i = 0; i < std::min<size_t>(r.size(), cap_out); ++i) {
    lo_out[i] = r[i].first >> shift;
    hi_out[i] = r[i].second >> shift;
  }
  return rc ? -1 : (int)r.size();
}
}  // namespace

extern "C" int mhb_plan_rounds(const uint64_t *hist256, uint64_t max_records, uint32_t *lo_out, uint32_t *hi_out) {
  return plan_rounds_out(hist256, nullptr, max_records, lo_out, hi_out, 256, 8);
}

extern "C" int mhb_plan_rounds16(const uint64_t *hist256, const uint64_t *sub_hist, uint64_t max_records, uint32_t *lo_out,
                                 uint32_t *hi_out, uint32_t cap_out) {
  return plan_rounds_out(hist256, sub_hist, max_records, lo_out, hi_out, cap_out, 0);
}

extern "C" int mhb_plan_r2s_owners(const uint64_t *hist16, uint32_t n_ranks, uint32_t *bucket_lo, uint32_t *bucket_hi) {
  if (!hist16 || !bucket_lo || !bucket_hi || n_ranks < 1 || n_ranks > (uint32_t)kMaxRanks)
    return mhb_set_error(MHB_ERR_ARG, "bad args");
  uint64_t h256[256];
  fold_bucket_hist(hist16, h256);
  uint32_t bounds[kMaxRanks + 1];
  uint8_t owner[256];
  owner_bounds(h256, (int)n_ranks, bounds, owner);
  for (uint32_t o = 0; o < n_ranks; ++o) {
    bucket_lo[o] = bounds[o] << 8;
    bucket_hi[o] = (bounds[o + 1] << 8) - 1;
  }
  return MHB_OK;
}

extern "C" int mhb_plan_count_owner_rounds(const uint64_t *hist16, uint32_t n_ranks, uint64_t max_records, uint32_t max_rounds,
                                           uint32_t *owner_lo, uint32_t *owner_hi, uint32_t *round_lo, uint32_t *round_hi,
                                           uint64_t *block_n, uint64_t *block_off, uint32_t *n_rounds_out) {
  if (!hist16 || !owner_lo || !owner_hi || !round_lo || !round_hi || !block_n || !block_off || !n_rounds_out || n_ranks < 1 ||
      n_ranks > (uint32_t)kMaxRanks || max_rounds < 1)
    return mhb_set_error(MHB_ERR_ARG, "bad args");
  const int W = (int)n_ranks;
  std::vector<const uint64_t *> h(W);
  for (int s = 0; s < W; ++s) h[s] = hist16 + (size_t)s * 65536;
  uint64_t cap[kMaxRanks];
  for (int o = 0; o < W; ++o) cap[o] = max_records ? max_records : ~0ull;
  OwnerPlan cp;
  CKR(plan_owner_rounds(h.data(), W, cap, &cp));
  if ((uint32_t)cp.R > max_rounds)
    return mhb_set_error(MHB_ERR_NOMEM, "the plan needs %d rounds, more than %u", cp.R, max_rounds);
  for (int o = 0; o < W; ++o) {
    owner_lo[o] = cp.bounds[o] << 8;
    owner_hi[o] = (cp.bounds[o + 1] << 8) - 1;
  }
  std::copy(cp.lo.begin(), cp.lo.end(), round_lo);
  std::copy(cp.hi.begin(), cp.hi.end(), round_hi);
  std::copy(cp.n.begin(), cp.n.end(), block_n);
  std::copy(cp.off.begin(), cp.off.end(), block_off);
  *n_rounds_out = (uint32_t)cp.R;
  return MHB_OK;
}

extern "C" int mhb_plan_read_shares(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t n_ranks,
                                    uint64_t *first_out) {
  if ((!bin && bin_words) || !first_out || n_ranks < 1) return mhb_set_error(MHB_ERR_ARG, "bad args");
  ReadLibIndex ix;  // serially, as mhb_iterate_run_multi before its fork
  CKR(index_read_lib(bin, bin_words, n_reads, 0, &ix, FixedCheck::kSerial));
  plan_read_shares(bin, ix, n_reads, n_ranks, first_out);
  return MHB_OK;
}

extern "C" int mhb_plan_seq_shares(const uint32_t *len, uint64_t n_seqs, uint32_t k, uint32_t n_ranks, uint64_t *first_out) {
  if ((!len && n_seqs) || !first_out || n_ranks < 1) return mhb_set_error(MHB_ERR_ARG, "bad args");
  plan_seq_shares(len, n_seqs, k, n_ranks, first_out);
  return MHB_OK;
}

extern "C" int mhb_plan_mercy_segments(const uint32_t *edges, uint64_t n_edges, uint32_t k, uint64_t max_segment_bytes,
                                       uint32_t *first_byte_out, uint32_t cap_out) {
  if ((n_edges && !edges) || max_segment_bytes == 0 || k < 12 || k > MHB_MAX_K) {
    mhb_set_error(MHB_ERR_ARG, "bad segment plan arguments");
    return -1;
  }
  uint64_t start[257];
  edge_byte_starts(edges, n_edges, mhb_words_per_edge(k), start);
  std::vector<uint32_t> first;
  if (plan_mercy_segments(start, mhb_words_per_edge(k), max_segment_bytes, max_segment_bytes, &first)) return -1;
  if (first_byte_out) {
    if (first.size() > cap_out) {
      mhb_set_error(MHB_ERR_ARG, "segment plan needs %llu entries, room for %u", (unsigned long long)first.size(), cap_out);
      return -1;
    }
    memcpy(first_byte_out, first.data(), first.size() * 4);
  }
  return (int)(first.size() - 1);
}
