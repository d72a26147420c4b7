// mhb_r2s.cu -- `read2sdbg` on the device (SURVEY.md 8a A12): host-level entry point mhb_read2sdbg_host and the
// self-test hooks of its building blocks.  Kernels: mhb_r2s.cuh.  Reference: main_sdbg_build.cpp:88-156,
// sorting/read_to_sdbg_s1.cpp, sorting/read_to_sdbg_s2.cpp.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <vector>

#include "mhb_common.cuh"
#include "mhb_r2s.cuh"

using namespace mhb;

// three-phase scan of mhb_device.cu
int scan32(cudaStream_t st, const uint32_t *in, uint64_t n, uint64_t *out, uint64_t *total_dev, uint64_t *bsum);
#define MHB_FOR_RW(M) M(3) M(4) M(5) M(6) M(7) M(8) M(9) M(10) M(11) M(12) M(13) M(14) M(15) M(16) M(17) M(18)

namespace {

// the record / item ping-pong buffers and the sort workspace, shared by stage 1 and stage 2 (cudaMalloc + cudaFree of
// 20-GB buffers between the stages cost ~0.2 s at 10 M reads)
struct BigBufs {
  DevBuf a, b, ws;
};

// phase marks on the stream: deltas include host-side gaps (allocations, synchronisations) between the marks
struct PhaseTrace {
  std::vector<std::pair<const char *, cudaEvent_t>> ev;
  cudaStream_t st = 0;
  void mark(const char *name) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, st);
    ev.emplace_back(name, e);
  }
  // ms spent in the phases whose name starts with `prefix` (all when empty); call after a stream synchronise
  double sum(const char *prefix) const {
    double t = 0;
    for (size_t i = 1; i < ev.size(); ++i)
      if (strncmp(ev[i].first, prefix, strlen(prefix)) == 0) {
        float ms = 0;
        cudaEventElapsedTime(&ms, ev[i - 1].second, ev[i].second);
        t += ms;
      }
    return t;
  }
  void report() const {
    if (!getenv("MHB_R2S_TRACE")) return;
    for (size_t i = 1; i < ev.size(); ++i) {
      float ms = 0;
      cudaEventElapsedTime(&ms, ev[i - 1].second, ev[i].second);
      fprintf(stderr, "[r2s] %-28s %9.3f ms\n", ev[i].first, ms);
    }
  }
  ~PhaseTrace() {
    for (auto &e : ev) cudaEventDestroy(e.second);
  }
};

// host index of the `.bin` image: package geometry of every read, derived from the record offsets of index_read_lib
struct PkgIndex {
  ReadLibIndex li;  // fixed-length check and record offsets (no unit offsets: streamed chunks derive theirs on the device)
  uint32_t fixed_len = 0, fixed_words = 0, max_len = 0;
  uint64_t n_reads = 0, n_words = 0, n_bases = 0, n_s1 = 0, n_edges = 0;
  std::vector<uint64_t> word_off, base_off, s1_off, edge_off;
  std::vector<uint32_t> len;
};

// the package geometry of every read, from the record offsets in ix->li and ix->n_reads
void pkg_geometry(const uint32_t *bin, uint32_t k, PkgIndex *ix) {
  const uint64_t n_reads = ix->n_reads;
  if (n_reads == 0) return;
  const uint32_t L0 = ix->li.fixed_len;
  if (L0) {
    ix->fixed_len = ix->max_len = L0;
    ix->fixed_words = div_ceil(L0, 16);
    ix->n_words = n_reads * ix->fixed_words;
    ix->n_bases = n_reads * (uint64_t)L0;
    if (L0 >= k + 1) {
      ix->n_s1 = n_reads * (uint64_t)(L0 - k + 4);
      ix->n_edges = n_reads * (uint64_t)(L0 - k);
    }
    return;
  }
  ix->word_off.resize(n_reads + 1);
  ix->base_off.resize(n_reads + 1);
  ix->s1_off.resize(n_reads + 1);
  ix->edge_off.resize(n_reads + 1);
  ix->len.resize(n_reads);
  uint64_t w = 0, b = 0, s1 = 0, e = 0;
  for (uint64_t r = 0; r < n_reads; ++r) {
    const uint32_t L = bin[ix->li.rec_off[r]];
    const uint32_t eff = L == 0 ? 1 : L;  // sequence_package.h:276-281
    ix->word_off[r] = w;
    ix->base_off[r] = b;
    ix->s1_off[r] = s1;
    ix->edge_off[r] = e;
    ix->len[r] = eff;
    ix->max_len = std::max(ix->max_len, eff);
    w += div_ceil(eff, 16);
    b += eff;
    if (eff >= k + 1) {
      s1 += eff - k + 4;
      e += eff - k;
    }
  }
  ix->word_off[n_reads] = w;
  ix->base_off[n_reads] = b;
  ix->s1_off[n_reads] = s1;
  ix->edge_off[n_reads] = e;
  ix->n_words = w;
  ix->n_bases = b;
  ix->n_s1 = s1;
  ix->n_edges = e;
}

int index_pkg(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t k, PkgIndex *ix) {
  ix->n_reads = n_reads;
  CKR(index_read_lib(bin, bin_words, n_reads, 0, &ix->li));
  std::vector<uint64_t>().swap(ix->li.unit_off);
  pkg_geometry(bin, k, ix);
  return MHB_OK;
}

template <class T>
int upload(DevBuf &d, const std::vector<T> &v, const char *what) {
  CKR(d.alloc(v.size() * sizeof(T), what));
  if (!v.empty()) CK(cudaMemcpy(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return MHB_OK;
}

// ---- device memory plan ----
// Caps on the records / items of one round (mhb_set_r2s_round_limit); 0 = derive from free device memory
uint64_t g_r2s_s1_limit = 0, g_r2s_s2_limit = 0;

// The stage-1 record layout of k (DESIGN.md §4.10).  Wide: NW key words + the 2 read_info words, sorted as whole
// records.  Narrow, where that exceeds the 17-word records of mhb_sort_records (k > 237): NW key words + a 32-bit row
// index into a side array of read_info; the bucket partition sorts (word 0, row) pairs and gathers the records.  Both
// order records by the key bytes and the input order alone, so both give kmsort's permutation.
bool g_r2s_force_narrow = false;  // mhb_selftest_read2sdbg_narrow: the narrow layout where the wide one fits
struct S1Layout {
  uint32_t NW, RW;
  bool narrow;
};
S1Layout s1_layout(uint32_t k) {
  const uint32_t NW = r2s_s1_key_words(k);
  const bool narrow = NW + 2 > 17 || g_r2s_force_narrow;
  return {NW, narrow ? NW + 1 : NW + 2, narrow};
}
// most records of one stage-1 round: the narrow layout's row index is 32 bits
uint64_t s1_round_cap(const S1Layout &l) { return l.narrow ? 0xFFFFFFFFull : (1ull << 40) - 1; }
// workspace of the bucket partition: the records themselves, or the (word 0, row) pairs
size_t s1_ws_bytes(uint64_t n, const S1Layout &l) { return mhb_sort_workspace_bytes(n, l.narrow ? 2 : l.RW); }

// device bytes of one stage-1 pass over n records: records, sort buffer and workspace, kmsort scratch; narrow: the
// read_info side array and the two pair buffers
size_t s1_pass_bytes(uint64_t n, const S1Layout &l) {
  const uint64_t seg_cap = n / (kKmInsertThreshold + 1) + 2;
  return 2 * pad256((size_t)n * l.RW * 4 + 16) + pad256(s1_ws_bytes(n, l)) + pad256((MHB_NUM_BUCKETS + 1) * 8) +
         2 * pad256(seg_cap * sizeof(KmSeg)) + 2 * pad256((n / 32 + 2) * 4) + pad256((size_t)n * 2 + 64) + 256 +
         (l.narrow ? 3 * pad256((size_t)n * 8 + 16) : 0);
}

// The stage-1 round plan: *max_n = 0 for one pass over all n_s1 records, else the most records of one round - the
// cap `limit` (mhb_set_r2s_round_limit) or what fits `avail` next to the per-chunk scratch of max_reads reads - and
// never more than s1_round_cap.  Returns non-zero when not even a one-record round fits.
int s1_plan_round(const S1Layout &l, uint64_t n_s1, uint64_t max_reads, size_t avail, uint64_t limit, uint64_t *max_n) {
  *max_n = 0;
  const uint64_t cap = s1_round_cap(l);
  if (!((limit && n_s1 > limit) || s1_pass_bytes(n_s1, l) > avail || n_s1 > cap)) return 0;
  uint64_t mx = limit;
  if (!mx) {
    const size_t fixed = pad256(max_reads * 4) + pad256((max_reads + 1) * 8) + pad256((max_reads / 4096 + 4) * 8) +
                         pad256(MHB_NUM_BUCKETS * 8) + 256;
    mx = largest_round(n_s1, fixed, avail, [&](uint64_t n) { return s1_pass_bytes(n, l); });
    if (!mx) return 1;
  }
  *max_n = std::min({mx, n_s1, cap});
  return 0;
}

// device bytes of one stage-2 pass over n items: items, sort buffer and workspace, run collapse, emitter scratch + stream
size_t s2_pass_bytes(uint64_t n, uint32_t W, uint32_t k) {
  const uint64_t n_tiles = (n + kDdTile - 1) / kDdTile;
  return 2 * pad256((size_t)n * W * 4 + 16) + pad256(mhb_s2s_sort_workspace_bytes(n, k)) + pad256(n_tiles * 4) + pad256(n_tiles * 8) +
         pad256((n_tiles / 4096 + 4) * 8) + pad256((size_t)n * 8) + pad256(mhb_s2s_emit_scratch_bytes(n, k)) +
         pad256((size_t)n * (4ull + 4ull * words_per_tip_label(k)) + 16);
}

// ---- the package, resident or streamed (DESIGN.md §4.9) ----
// One chunk of the package on the device, handed to the stage code in read order: pv covers the chunk's reads (read
// indices, words and offset arrays relative to the chunk, pv.base0 = global base of its first read, so every bit-plane
// index and stage-1 payload stays global).  The rest comes from the host index.
struct PkgChunk {
  PkgView pv;
  uint64_t n_words = 0;            // package words of the chunk
  uint64_t s1_0 = 0, n_s1 = 0;     // stage-1 records before the chunk / in it
  uint64_t n_edges = 0;            // (k+1)-mer positions in the chunk
  uint64_t w0 = 0, w_end = 0;      // the chunk's words of the bit planes: [base0 / 32, base_end / 32 + 2)
  uint64_t base_end = 0;           // global base after the chunk's last read
};
using ChunkFn = std::function<int(const PkgChunk &)>;
using EachChunk = std::function<int(const ChunkFn &)>;  // one pass over the package: fn once per chunk, in read order

PkgChunk chunk_of(const PkgIndex &ix, uint64_t f, uint64_t e, uint32_t k) {
  PkgChunk c;
  memset(&c.pv, 0, sizeof(c.pv));
  c.pv.n_reads = e - f;
  c.pv.fixed_len = ix.fixed_len;
  c.pv.fixed_words = ix.fixed_words;
  uint64_t bases;
  if (ix.fixed_len) {
    const uint32_t L = ix.fixed_len;
    const uint64_t per_s1 = L >= k + 1 ? L - k + 4 : 0, per_e = L >= k + 1 ? L - k : 0;
    c.pv.base0 = f * L;
    bases = (e - f) * L;
    c.n_words = (e - f) * ix.fixed_words;
    c.s1_0 = f * per_s1;
    c.n_s1 = (e - f) * per_s1;
    c.n_edges = (e - f) * per_e;
  } else {
    c.pv.base0 = ix.base_off[f];
    bases = ix.base_off[e] - ix.base_off[f];
    c.n_words = ix.word_off[e] - ix.word_off[f];
    c.s1_0 = ix.s1_off[f];
    c.n_s1 = ix.s1_off[e] - ix.s1_off[f];
    c.n_edges = ix.edge_off[e] - ix.edge_off[f];
  }
  c.w0 = c.pv.base0 / 32;
  c.w_end = (c.pv.base0 + bases) / 32 + 2;  // the whole library: bit_words
  c.base_end = c.pv.base0 + bases;
  return c;
}

// ---- the list form of the mercy candidates (DESIGN.md §4.9) ----
int g_r2s_sparse_mercy = 0;  // mhb_set_r2s_sparse_mercy: 1 = lists whenever the library is streamed
struct MercyStats {
  int sparse = 0;
  uint64_t n_entries = 0, host_bytes = 0;
} g_mercy_stats;  // mhb_r2s_mercy_stats: the last mhb_read2sdbg_host call

// The candidates of every stage-1 round as a list of entries (cand_entries: position << 2 | code), each sorted by
// position, in host memory.  Duplicates are allowed: the planes they stand for are sets.
struct CandLists {
  std::vector<std::vector<uint64_t>> rounds;
  uint32_t sort_bytes = 8;  // the low bytes of an entry that can be non-zero
  void init(uint64_t n_bases) {
    rounds.clear();
    const uint64_t top = n_bases << 2 | 3;
    for (sort_bytes = 1; sort_bytes < 8 && (top >> (8 * sort_bytes)); ++sort_bytes) {}
  }
  uint64_t n_entries() const {
    uint64_t n = 0;
    for (const auto &v : rounds) n += v.size();
    return n;
  }
  // fn(entries, count) for the slice of every round with positions in [b0, b1) (binary search)
  template <class F>
  int each_slice(uint64_t b0, uint64_t b1, F fn) const {
    for (const auto &v : rounds) {
      const auto lo = std::lower_bound(v.begin(), v.end(), b0 << 2), hi = std::lower_bound(lo, v.end(), b1 << 2);
      if (hi > lo) CKR(fn(&*lo, (uint64_t)(hi - lo)));
    }
    return MHB_OK;
  }
};

// The chunk's candidates into three planes of plane_words words each at `planes` (no in, no out, any), on the global
// word grid from word w0; returns o with its candidate planes pointing there.  Slices go through `stage` (device,
// stage_cap entries) one piece at a time.
int cand_scatter(cudaStream_t st, const CandLists &lists, uint64_t b0, uint64_t b1, uint64_t w0, u32 *planes,
                 uint64_t plane_words, u64 *stage, uint64_t stage_cap, S1Out *o) {
  CK(cudaMemsetAsync(planes, 0, 3 * plane_words * 4, st));
  o->no_in = planes - w0;
  o->no_out = planes + plane_words - w0;
  o->any = planes + 2 * plane_words - w0;
  const S1Out so = *o;
  return lists.each_slice(b0, b1, [&](const uint64_t *e, uint64_t n) -> int {
    for (uint64_t at = 0; at < n; at += stage_cap) {
      const uint64_t piece = std::min(stage_cap, n - at);
      CK(cudaMemcpyAsync(stage, e + at, piece * 8, cudaMemcpyHostToDevice, st));
      k_r2s_cand_scatter<<<grid_cap(piece, 256, 16), 256, 0, st>>>(stage, piece, so);
      CK_LAUNCH();
    }
    return MHB_OK;
  });
}
constexpr uint64_t kCandStage = (uint64_t)1 << 20;  // entries of the staging slot of the scatter (8 MiB)

// Every pass over the package.  Resident: the package of the whole library, uploaded and reversed once, is the only
// chunk.  Streamed: the `.bin` image stays in host memory (init_read_stream); per chunk the reads are reversed into a
// chunk-sized package slot and, for variable-length libraries, the chunk's offsets are derived on the device from its
// length words (k_r2s_chunk_geom + scan32).
class PkgSource {
 public:
  std::vector<PkgChunk> chunks;  // host geometry of every chunk (none for an empty library)
  uint64_t max_reads = 0, max_words = 0, max_plane_words = 0;

  int plan(const mhb_build_args *a, const PkgIndex &ix, uint32_t k, bool stream, uint64_t chunk_bytes) {
    args_ = a;
    k_ = k;
    streamed_ = stream;
    fixed_ = ix.fixed_len != 0;
    std::vector<uint64_t> first = {0, ix.n_reads};
    if (stream) {
      CKR(init_read_stream(&rs_, a->bin, a->bin_words, ix.n_reads, ix.li, chunk_bytes));
      first = rs_.bounds();
    }
    for (size_t i = 0; i + 1 < first.size() && ix.n_reads; ++i) {
      chunks.push_back(chunk_of(ix, first[i], first[i + 1], k));
      const PkgChunk &c = chunks.back();
      max_reads = std::max(max_reads, c.pv.n_reads);
      max_words = std::max(max_words, c.n_words);
      max_plane_words = std::max(max_plane_words, c.w_end - c.w0);
    }
    return MHB_OK;
  }
  // device bytes of the streamed form: both `.bin` chunk slots, the package slot, the chunk's offsets and their scratch
  size_t streamed_bytes() const {
    return pad256(rs_.device_bytes()) + pad256((size_t)max_words * 4 + 64) +
           (fixed_ ? 0 : 4 * pad256((max_reads + 1) * 8) + 4 * pad256(max_reads * 4) + pad256((max_reads / 4096 + 4) * 8));
  }
  // resident: upload + reverse now; streamed: the chunk buffers
  int bind(cudaStream_t st, const PkgIndex &ix) {
    CKR(pkg_.alloc((size_t)max_words * 4 + 64, streamed_ ? "read2sdbg: package chunk" : "read2sdbg: package"));
    if (streamed_) {
      CKR(lib_.alloc(rs_.device_bytes(), "read2sdbg: .bin chunk slots"));
      CKR(rs_.bind(lib_.p, st));
      if (!fixed_) {
        CKR(word_off_.alloc((max_reads + 1) * 8, "read2sdbg: chunk word offsets"));
        CKR(len_.alloc(max_reads * 4, "read2sdbg: chunk lengths"));
        CKR(base_off_.alloc((max_reads + 1) * 8, "read2sdbg: chunk base offsets"));
        CKR(s1_off_.alloc((max_reads + 1) * 8, "read2sdbg: chunk stage-1 offsets"));
        CKR(edge_off_.alloc((max_reads + 1) * 8, "read2sdbg: chunk edge offsets"));
        CKR(geom_.alloc(3 * pad256(max_reads * 4), "read2sdbg: chunk read geometry"));
        CKR(bsum_.alloc((max_reads / 4096 + 4) * 8, "read2sdbg: scan sums"));
      }
      return MHB_OK;
    }
    if (chunks.empty()) return MHB_OK;
    PkgChunk &c = chunks[0];
    DevBuf d_bin, d_rec_off;
    CKR(d_bin.alloc((size_t)args_->bin_words * 4 + 64, "read2sdbg: .bin image"));
    CK(cudaMemcpyAsync(d_bin.p, args_->bin, (size_t)args_->bin_words * 4, cudaMemcpyHostToDevice, st));
    if (!fixed_) {
      CKR(upload(d_rec_off, ix.li.rec_off, "read2sdbg: record offsets"));
      CKR(upload(word_off_, ix.word_off, "read2sdbg: word offsets"));
      CKR(upload(len_, ix.len, "read2sdbg: lengths"));
      CKR(upload(base_off_, ix.base_off, "read2sdbg: base offsets"));
      CKR(upload(s1_off_, ix.s1_off, "read2sdbg: stage-1 offsets"));
      CKR(upload(edge_off_, ix.edge_off, "read2sdbg: edge offsets"));
      set_offsets(c.pv);
    }
    if (c.n_words) {
      k_r2s_reverse<<<grid_cap(c.n_words, 256, 16), 256, 0, st>>>(d_bin.as<u32>(), c.pv.n_reads, c.pv.fixed_len,
                                                             d_rec_off.as<u64>(), c.pv, pkg_.as<u32>(), c.n_words);
      CK_LAUNCH();
    }
    c.pv.words = pkg_.as<u32>();
    CK(cudaStreamSynchronize(st));  // d_bin / d_rec_off go out of scope
    return MHB_OK;
  }
  int each(cudaStream_t st, const ChunkFn &fn) {
    if (!streamed_) return chunks.empty() ? MHB_OK : fn(chunks[0]);
    return rs_.pass(st, [&](const ChunkView &v) -> int {
      PkgChunk c = chunks[v.index];
      const uint64_t n = c.pv.n_reads;
      if (!fixed_) {
        u32 *words = geom_.as<u32>(), *s1 = words + pad256(max_reads * 4) / 4, *edges = s1 + pad256(max_reads * 4) / 4;
        k_r2s_chunk_geom<<<grid_cap(n, 256, 16), 256, 0, st>>>(v.words, v.at<uint64_t>(0), n, k_, len_.as<u32>(), words,
                                                               s1, edges);
        CK_LAUNCH();
        u64 *bs = bsum_.as<u64>();
        CKR(scan32(st, words, n, word_off_.as<u64>(), word_off_.as<u64>() + n, bs));
        CKR(scan32(st, len_.as<u32>(), n, base_off_.as<u64>(), base_off_.as<u64>() + n, bs));
        CKR(scan32(st, s1, n, s1_off_.as<u64>(), s1_off_.as<u64>() + n, bs));
        CKR(scan32(st, edges, n, edge_off_.as<u64>(), edge_off_.as<u64>() + n, bs));
        set_offsets(c.pv);
      }
      if (c.n_words) {
        k_r2s_reverse<<<grid_cap(c.n_words, 256, 16), 256, 0, st>>>(v.words, n, c.pv.fixed_len, v.at<uint64_t>(0), c.pv,
                                                               pkg_.as<u32>(), c.n_words);
        CK_LAUNCH();
      }
      c.pv.words = pkg_.as<u32>();
      return fn(c);
    });
  }

 private:
  void set_offsets(PkgView &pv) const {
    pv.word_off = word_off_.as<u64>();
    pv.len = len_.as<u32>();
    pv.base_off = base_off_.as<u64>();
    pv.s1_off = s1_off_.as<u64>();
    pv.edge_off = edge_off_.as<u64>();
  }
  const mhb_build_args *args_ = nullptr;
  uint32_t k_ = 0;
  bool streamed_ = false, fixed_ = false;
  ChunkStream rs_;
  DevBuf lib_, pkg_, word_off_, len_, base_off_, s1_off_, edge_off_, geom_, bsum_;
};

// ---- residency (DESIGN.md §4.9) ----
// What the resident form holds for the whole call: the package and, for variable-length libraries, its offsets, the
// solid plane (m > 1), the mercy planes (need_mercy), the histogram, counters and bucket table; and, while the package
// is built, the `.bin` image and its record offsets.
struct ResidentPlan {
  size_t resident = 0, upload = 0;
};
ResidentPlan resident_plan(const PkgIndex &ix, uint64_t bin_words, int32_t m, bool mercy) {
  const uint64_t bit_words = ix.n_bases / 32 + 2;
  const size_t planes = (m > 1 ? pad256(bit_words * 4) : 0) + (mercy ? 4 * pad256(bit_words * 4) : 0);
  ResidentPlan p;
  p.resident = pad256((size_t)ix.n_words * 4 + 64) + (ix.fixed_len ? 0 : 5 * pad256((ix.n_reads + 1) * 8) + pad256(ix.n_reads * 4)) +
               planes + pad256(65536 * 8) + pad256(64) + pad256((size_t)MHB_NUM_BUCKETS * 32) + pad256(128);
  p.upload = pad256((size_t)bin_words * 4 + 64) + (ix.fixed_len ? 0 : pad256((ix.n_reads + 1) * 8));
  return p;
}

// One residency rule (mhb_read_stream_decide, as count and iterate): stream when the resident form and its upload do
// not fit free_b, when next to it not even a one-record stage-1 round or a one-item stage-2 round fits, or when a
// chunk cap is set.
bool stream_decide(const ResidentPlan &p, const PkgIndex &ix, uint32_t k, int32_t m, size_t free_b, uint64_t chunk_limit) {
  const double room = free_b > p.resident ? 0.92 * (double)(free_b - p.resident) : 0.0;
  const uint32_t W = s2s_record_words(k);
  const size_t s1_fixed = pad256(ix.n_reads * 4) + pad256((ix.n_reads + 1) * 8) + pad256((ix.n_reads / 4096 + 4) * 8) +
                          pad256(MHB_NUM_BUCKETS * 8) + 256;
  const bool no_round = (m > 1 && ix.n_s1 && (double)(s1_fixed + s1_pass_bytes(1, s1_layout(k))) > room) ||
                        (ix.n_edges && (double)s2_pass_bytes(1, W, k) > room);
  return mhb_read_stream_decide(p.resident + p.upload, free_b, no_round ? 1 : 0, chunk_limit) != 0;
}

// ---- the form of the mercy candidates (DESIGN.md §4.9) ----
// Device bytes the streamed form holds for the whole call in either form: the solid plane (m > 1), the candidates -
// three planes of the whole library, or (list form) three chunk-sized planes and the staging slot of the scatter -,
// the mercy plane of a chunk, the read chunk buffers, the histogram, counters and bucket table.  The list form is taken
// when the planes do not fit free_b, or always with force (mhb_set_r2s_sparse_mercy), and only with need_mercy.
struct MercyForm {
  size_t planes = 0, lists = 0;
  bool sparse = false;
};
MercyForm mercy_form(uint64_t bit_words, uint64_t max_plane_words, size_t streamed_bytes, int32_t m, bool mercy,
                     size_t free_b, int force) {
  const size_t rest = (m > 1 ? pad256(bit_words * 4) : 0) + (mercy ? pad256(max_plane_words * 4) : 0) + streamed_bytes +
                      pad256(65536 * 8) + pad256(64) + pad256((size_t)MHB_NUM_BUCKETS * 32) + pad256(128);
  MercyForm f;
  f.planes = rest + (mercy ? 3 * pad256(bit_words * 4) : 0);
  f.lists = rest + (mercy ? pad256(3 * max_plane_words * 4) + pad256(kCandStage * 8) : 0);
  f.sparse = mercy && (force || f.planes > free_b);
  return f;
}

// ---- stage 1 on the device: is_solid bits, mercy planes, multiplicity histogram ----
struct S1Side {  // the narrow layout's read_info side array and the pair buffers of its bucket partition
  DevBuf info, pa, pb;
};
// the buffers of one stage-1 pass over n records: the records (a, overwritten), a sort buffer of as many records (b),
// the workspace s1_ws_bytes(n); narrow layout: the read_info side array and the two pair buffers, n entries each
struct S1Bufs {
  u32 *a, *b;
  void *ws;
  u64 *info;
  u32 *pa, *pb;
};
int s1_sort_post(cudaStream_t st, const PkgView &pv, uint32_t k, int32_t m, bool need_mercy, const S1Out &out,
                 unsigned long long *d_mul_hist, PhaseTrace &tr, const S1Bufs &bufs, uint64_t n, CandLists *lists);

// Stage 1 in rounds over contiguous ranges of bucket ids, each of at most max_n records; *n_rounds counts the
// non-empty ones.  max_n == 0: one pass, the one range over all bucket ids, known without a pass: each chunk's records
// go to its global stage-1 offset, so chunks taken in read order give the reference's bucket input order (read order),
// as one k_r2s_s1_extract over the whole library does, and the shared buffers get at least min_rec_bytes /
// min_ws_bytes (stage 2's share).  Otherwise one histogram pass over the library plans the ranges, then per range one
// pass extracts the in-range records of every chunk in read order (count, scan, write at the round's cursor).  Each
// round is sorted and post-processed alike.  A (k-1)-mer group lies in one bucket, so in one round; is_solid, the mercy
// planes and the multiplicity histogram accumulate across rounds (lists != nullptr: each round adds its candidate list).
int run_stage1(cudaStream_t st, const EachChunk &each, const PkgView &shape, const PkgIndex &ix, uint64_t chunk_reads,
               uint32_t k, int32_t m, bool need_mercy, const S1Out &out, unsigned long long *d_mul_hist, PhaseTrace &tr,
               BigBufs &big, uint64_t max_n, size_t min_rec_bytes, size_t min_ws_bytes, uint32_t *n_rounds,
               CandLists *lists) {
  const S1Layout l = s1_layout(k);
  const uint32_t NW = l.NW, RW = l.RW;
  const bool one_pass = max_n == 0;
  if (one_pass) max_n = ix.n_s1;
  if (max_n > s1_round_cap(l)) return mhb_set_error(MHB_ERR_ARG, "read2sdbg: too many stage-1 records for one round");
  CKR(big.a.ensure(std::max((size_t)max_n * RW * 4 + 16, min_rec_bytes), "read2sdbg: records"));
  CKR(big.b.ensure(std::max((size_t)max_n * RW * 4 + 16, min_rec_bytes), "read2sdbg: records (sort buffer)"));
  CKR(big.ws.ensure(std::max(s1_ws_bytes(max_n, l), min_ws_bytes), "read2sdbg: sort workspace"));
  S1Side side;
  if (l.narrow) {
    CKR(side.info.alloc((size_t)max_n * 8 + 16, "read2sdbg: stage-1 read_info"));
    CKR(side.pa.alloc((size_t)max_n * 8 + 16, "read2sdbg: bucket partition pairs"));
    CKR(side.pb.alloc((size_t)max_n * 8 + 16, "read2sdbg: bucket partition pairs (sort buffer)"));
  }
  u64 *d_info = l.narrow ? side.info.as<u64>() : nullptr;
  BucketRanges ranges = {{0u, 65535u}};
  DevBuf per_read, off, bsum, total;
  if (!one_pass) {
    DevBuf h16;
    CKR(per_read.alloc(chunk_reads * 4, "read2sdbg: per-read record counts"));
    CKR(off.alloc((chunk_reads + 1) * 8, "read2sdbg: per-read record offsets"));
    CKR(bsum.alloc((chunk_reads / 4096 + 4) * 8, "read2sdbg: scan sums"));
    CKR(h16.alloc(MHB_NUM_BUCKETS * 8, "read2sdbg: bucket histogram"));
    CKR(total.alloc(8, "read2sdbg: round size"));
    CK(cudaMemsetAsync(h16.p, 0, MHB_NUM_BUCKETS * 8, st));
    if (int rc_ = each([&](const PkgChunk &c) -> int {
      const unsigned grid = grid_cap(c.pv.n_reads * 32, 256, 16);  // one warp per read
#define M(WW)   \
  if (NW == WW) \
    k_r2s_s1_range<WW, kS1Hist><<<grid, 256, 0, st>>>(c.pv, k, 0, 65535, h16.as<unsigned long long>(), nullptr, nullptr, nullptr);
      MHB_FOR_WR(M)
#undef M
      CK_LAUNCH();
      return MHB_OK;
    }))
      return rc_;
    std::vector<uint64_t> h_h16(MHB_NUM_BUCKETS);
    CK(cudaMemcpyAsync(h_h16.data(), h16.p, MHB_NUM_BUCKETS * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    tr.mark("s1.extract.plan");
    CKR(plan_stage_rounds(h_h16.data(), max_n, &ranges));
  }
  uint64_t seen = 0;
  for (const auto &rg : ranges) {
    uint64_t n = 0;  // the round's cursor
    if (int rc_ = each([&](const PkgChunk &c) -> int {
      if (one_pass) {
        if (c.n_s1) {
#define M(WW)                                                                                                      \
  if (NW == WW)                                                                                                    \
    k_r2s_s1_extract<WW><<<grid_cap(c.n_s1, 256, 16), 256, 0, st>>>(c.pv, k, big.a.as<u32>(), d_info, c.s1_0, c.n_s1);
          MHB_FOR_WR(M)
#undef M
          CK_LAUNCH();
        }
        n += c.n_s1;
        return MHB_OK;
      }
      const unsigned grid = grid_cap(c.pv.n_reads * 32, 256, 16);
#define M(WW)                                                                                                          \
  if (NW == WW)                                                                                                        \
    k_r2s_s1_range<WW, kS1Count><<<grid, 256, 0, st>>>(c.pv, k, rg.first, rg.second, nullptr, per_read.as<u32>(), nullptr, \
                                                       nullptr);
      MHB_FOR_WR(M)
#undef M
      CK_LAUNCH();
      CKR(scan32(st, per_read.as<u32>(), c.pv.n_reads, off.as<u64>(), total.as<u64>(), bsum.as<u64>()));
      uint64_t t = 0;
      CK(cudaMemcpyAsync(&t, total.p, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (n + t > max_n)
        return mhb_set_error(MHB_ERR_CUDA, "read2sdbg: internal: round of %llu stage-1 records exceeds its plan (%llu)",
                             (unsigned long long)(n + t), (unsigned long long)max_n);
      if (t) {  // rows n on: after the records of the chunks before, read order
#define M(WW)                                                                                                          \
  if (NW == WW)                                                                                                        \
    k_r2s_s1_range<WW, kS1Write><<<grid, 256, 0, st>>>(c.pv, k, rg.first, rg.second, nullptr, nullptr, off.as<u64>(), \
                                                       big.a.as<u32>(), d_info, n);
        MHB_FOR_WR(M)
#undef M
        CK_LAUNCH();
      }
      n += t;
      return MHB_OK;
    }))
      return rc_;
    seen += n;
    if (n == 0) continue;
    tr.mark("s1.extract");
    const S1Bufs bufs{big.a.as<u32>(), big.b.as<u32>(), big.ws.p, d_info, side.pa.as<u32>(), side.pb.as<u32>()};
    CKR(s1_sort_post(st, shape, k, m, need_mercy, out, d_mul_hist, tr, bufs, n, lists));
    ++*n_rounds;
  }
  if (seen != ix.n_s1)
    return mhb_set_error(MHB_ERR_CUDA, "read2sdbg: internal: the rounds saw %llu of %llu stage-1 records",
                         (unsigned long long)seen, (unsigned long long)ix.n_s1);
  return MHB_OK;
}

// The candidate bytes of a post-processed round of n records (recs) -> the round's entries, sorted by position, appended
// to lists.  Count -> scan32 -> write in record order; entries in `spare` (the other record buffer) when they fit, and
// the stable radix sort on the position bytes into recs, which the write leaves unused.
int cand_round(cudaStream_t st, const uint8_t *cand, uint64_t n, u32 *recs, u32 *spare, const S1Layout &l,
               const S1Bufs &bufs, CandLists *lists) {
  const uint64_t n_tiles = (n + kCandTile - 1) / kCandTile;
  const size_t rec_bytes = (size_t)n * l.RW * 4;  // the least either record buffer holds
  DevBuf tile_n, tile_off, bsum, ent, srt, ws;
  CKR(tile_n.alloc(n_tiles * 4, "read2sdbg: candidate counts"));
  CKR(tile_off.alloc((n_tiles + 1) * 8, "read2sdbg: candidate offsets"));
  CKR(bsum.alloc((n_tiles / 4096 + 4) * 8, "read2sdbg: scan sums"));
  k_r2s_cand_count<<<(unsigned)n_tiles, 256, 0, st>>>(cand, n, tile_n.as<u32>());
  CK_LAUNCH();
  CKR(scan32(st, tile_n.as<u32>(), n_tiles, tile_off.as<u64>(), tile_off.as<u64>() + n_tiles, bsum.as<u64>()));
  uint64_t cnt = 0;
  CK(cudaMemcpyAsync(&cnt, tile_off.as<u64>() + n_tiles, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  lists->rounds.emplace_back(cnt);
  if (!cnt) return MHB_OK;
  u64 *e = (u64 *)spare;
  if (cnt * 8 > rec_bytes) {
    CKR(ent.alloc(cnt * 8, "read2sdbg: candidate entries"));
    e = ent.as<u64>();
  }
  k_r2s_cand_write<<<(unsigned)n_tiles, 256, 0, st>>>(cand, n, recs, l.narrow ? bufs.info : nullptr, l.RW, l.NW,
                                                      tile_off.as<u64>(), e);
  CK_LAUNCH();
  u32 *sb = recs;
  if (cnt * 8 > rec_bytes) {
    CKR(srt.alloc(cnt * 8, "read2sdbg: candidate entries (sort buffer)"));
    sb = srt.as<u32>();
  }
  const size_t ws_need = mhb_sort_workspace_bytes(cnt, 2);
  void *w = bufs.ws;
  if (ws_need > s1_ws_bytes(n, l)) {
    CKR(ws.alloc(ws_need, "read2sdbg: candidate sort workspace"));
    w = ws.p;
  }
  static const uint8_t pos_bytes[8] = {4, 5, 6, 7, 0, 1, 2, 3};  // low word first: the entry's bytes, least significant first
  int in_b = 0;
  CKR(mhb_sort_records(st, (u32 *)e, sb, cnt, 2, pos_bytes, lists->sort_bytes, nullptr, w, ws_need, &in_b));
  CK(cudaMemcpyAsync(lists->rounds.back().data(), in_b ? (const void *)sb : (const void *)e, cnt * 8,
                     cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MHB_OK;
}

// stable bucket partition, kmsort emulation and Lv2Postprocess of the n records in bufs.a; lists != nullptr: the
// candidates go to a new round of lists instead of the planes of out
int s1_sort_post(cudaStream_t st, const PkgView &pv, uint32_t k, int32_t m, bool need_mercy, const S1Out &out,
                 unsigned long long *d_mul_hist, PhaseTrace &tr, const S1Bufs &bufs, uint64_t n, CandLists *lists) {
  const S1Layout l = s1_layout(k);
  const uint32_t NW = l.NW, RW = l.RW;
  DevBuf bstart, segs0, segs1, counter, bnd;
  u32 *const a = bufs.a, *const b = bufs.b;
  const size_t ws_bytes = s1_ws_bytes(n, l);
  CKR(bstart.alloc((MHB_NUM_BUCKETS + 1) * 8, "read2sdbg: bucket bounds"));
  const uint64_t seg_cap = n / (kKmInsertThreshold + 1) + 2;
  CKR(segs0.alloc(seg_cap * sizeof(KmSeg), "read2sdbg: kmsort ranges"));
  CKR(segs1.alloc(seg_cap * sizeof(KmSeg), "read2sdbg: kmsort ranges"));
  CKR(counter.alloc(8, "read2sdbg: counter"));
  CKR(bnd.alloc((n / 32 + 2) * 4, "read2sdbg: range marks"));
  CK(cudaMemsetAsync(bnd.p, 0, (n / 32 + 2) * 4, st));
  // the reference's bucket input order: records of one 16-bit bucket in global read order = a STABLE sort on the two
  // leading key bytes (base_engine.cpp:323-348 fills every bucket thread by thread, i.e. in read order)
  int in_b = 0;
  if (l.narrow) {
    const uint8_t bytes[2] = {6, 7};  // the two leading bytes of a (word 0, row) pair
    k_r2s_s1_pairs<<<grid_cap(n, 256, 16), 256, 0, st>>>(a, n, RW, bufs.pa);
    CK_LAUNCH();
    int in_pb = 0;
    CKR(mhb_sort_records(st, bufs.pa, bufs.pb, n, 2, bytes, 2, nullptr, bufs.ws, ws_bytes, &in_pb));
    k_r2s_s1_gather<<<grid_cap(n * RW, 256, 16), 256, 0, st>>>(a, in_pb ? bufs.pb : bufs.pa, n, RW, b);
    CK_LAUNCH();
    in_b = 1;
  } else {
    const uint8_t bytes[2] = {(uint8_t)(4 * RW - 2), (uint8_t)(4 * RW - 1)};
    CKR(mhb_sort_records(st, a, b, n, RW, bytes, 2, nullptr, bufs.ws, ws_bytes, &in_b));
  }
  u32 *recs = in_b ? b : a;
  tr.mark("s1.partition");
  k_r2s_bucket_bounds<<<(MHB_NUM_BUCKETS + 1 + 255) / 256, 256, 0, st>>>(recs, n, RW, bstart.as<u64>());
  CK_LAUNCH();
  // kmsort (kmsort.h:103-117 entry, :43-101 per range), level by level
  int kb = 4 * (int)NW - 2 - 1;
  KmSeg *cur = segs0.as<KmSeg>(), *nxt = segs1.as<KmSeg>();
  unsigned long long *d_cnt = counter.as<unsigned long long>();
  CK(cudaMemsetAsync(d_cnt, 0, 8, st));
  const bool km_global = getenv("MHB_R2S_KMSORT_GLOBAL") != nullptr;  // the in-place form of every level (A/B, tests)
  static char level_names[72][24];
  int level = 0;
  DevBuf todo, src16;
  u32 *d_todo = nullptr;
  if (lists) CKR(src16.alloc((size_t)n * 2 + 64, "read2sdbg: kmsort source indices"));  // then the candidate bytes
  if (!km_global) {
    // level 0 on shared-memory tags: bucket sizes decide the tag capacity of a CTA
    std::vector<uint64_t> h_b(MHB_NUM_BUCKETS + 1);
    CK(cudaMemcpyAsync(h_b.data(), bstart.p, h_b.size() * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint64_t max_bucket = 0;
    for (int i = 0; i < MHB_NUM_BUCKETS; ++i) max_bucket = std::max(max_bucket, h_b[i + 1] - h_b[i]);
    uint32_t cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(max_bucket, 1024), 65535);
    cap = (cap + 1023) & ~1023u;
    if (const char *e = getenv("MHB_R2S_KM_CAP")) cap = std::max(1024u, (uint32_t)atoi(e) & ~1023u);  // tests: force the fall-back
    CKR(todo.alloc((n / 32 + 2) * 4, "read2sdbg: unsorted-range marks"));
    CK(cudaMemsetAsync(todo.p, 0, (n / 32 + 2) * 4, st));
    CKR(src16.ensure((size_t)n * 2 + 64, "read2sdbg: kmsort source indices"));
    d_todo = todo.as<u32>();
    u32 *other = in_b ? a : b;
#define M(WW)                                                                                                           \
  if (RW == WW) {                                                                                                       \
    CK(cudaFuncSetAttribute(k_r2s_km_bucket<WW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));               \
    k_r2s_km_bucket<WW><<<MHB_NUM_BUCKETS, 128, cap, st>>>(recs, other, bstart.as<u64>(), NW, kb, cap,                   \
                                                           src16.as<uint16_t>(), bnd.as<u32>(), d_todo, nxt, d_cnt, seg_cap); \
  }
    MHB_FOR_RW(M)
#undef M
    CK_LAUNCH();
    recs = other;
  } else {
#define M(WW)                                                                                                      \
  if (RW == WW)                                                                                                    \
    k_r2s_kmsort_level<WW><<<MHB_NUM_BUCKETS / 128, 128, 0, st>>>(recs, NW, kb, nullptr, bstart.as<u64>(),          \
                                                                  MHB_NUM_BUCKETS, nxt, d_cnt, seg_cap, bnd.as<u32>());
    MHB_FOR_RW(M)
#undef M
    CK_LAUNCH();
  }
  for (;;) {
    snprintf(level_names[level], sizeof(level_names[level]), "s1.kmsort.L%d", level);
    tr.mark(level_names[level]);
    if (level < 71) ++level;
    unsigned long long n_next = 0;
    CK(cudaMemcpyAsync(&n_next, d_cnt, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (n_next == 0 || kb == 0) break;
    if (n_next > seg_cap) return mhb_set_error(MHB_ERR_CUDA, "read2sdbg: internal: kmsort range list overflow");
    std::swap(cur, nxt);
    --kb;
    CK(cudaMemsetAsync(d_cnt, 0, 8, st));
    if (!km_global) {
#define M(WW)                                                                                                            \
  if (RW == WW) {                                                                                                        \
    const size_t smem = (size_t)kKmWarps * km_warp_smem<WW>();                                                           \
    static bool attr = false;                                                                                            \
    if (!attr) {                                                                                                         \
      CK(cudaFuncSetAttribute(k_r2s_km_warp<WW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));               \
      attr = true;                                                                                                       \
    }                                                                                                                    \
    k_r2s_km_warp<WW><<<grid_cap(n_next, kKmWarps, 8), kKmWarps * 32, smem, st>>>(recs, NW, kb, cur, n_next, nxt, d_cnt, seg_cap, \
                                                              bnd.as<u32>(), d_todo);                                    \
  }
      MHB_FOR_RW(M)
#undef M
    } else {
#define M(WW)                                                                                                         \
  if (RW == WW)                                                                                                       \
    k_r2s_kmsort_level<WW><<<(unsigned)((n_next + 127) / 128), 128, 0, st>>>(recs, NW, kb, cur, nullptr, n_next, nxt, \
                                                                            d_cnt, seg_cap, bnd.as<u32>());
      MHB_FOR_RW(M)
#undef M
    }
    CK_LAUNCH();
  }
#define M(WW) \
  if (RW == WW) k_r2s_kmsort_finish<WW><<<grid_cap(n, 256, 32), 256, 0, st>>>(recs, n, NW, bnd.as<u32>(), d_todo);
  MHB_FOR_RW(M)
#undef M
  CK_LAUNCH();
  tr.mark("s1.kmsort.finish");
  uint8_t *const cand = lists ? src16.as<uint8_t>() : nullptr;  // the kmsort source indices are dead by now
#define M(WW)                                                                                                          \
  if (RW == WW)                                                                                                        \
    k_r2s_s1_post<WW><<<grid_cap(n, 256, 32), 256, 0, st>>>(recs, l.narrow ? bufs.info : nullptr, n, NW, k, m, \
                                                            pv, out, need_mercy ? 1 : 0, d_mul_hist, cand);
  MHB_FOR_RW(M)
#undef M
  CK_LAUNCH();
  if (lists) CKR(cand_round(st, cand, n, recs, recs == a ? b : a, l, bufs, lists));
  tr.mark("s1.post");
  CK(cudaStreamSynchronize(st));
  return MHB_OK;
}

// ---- stage 2 ----
struct S2Bufs {  // collapse and emitter buffers, kept across rounds
  DevBuf tile_heads, tile_off, bsum, heads, scr, bytes;
};

// relaxed sort -> collapse of equal items -> emitter, on the n items in a (b: a buffer of as many items, ws: the sort
// workspace); leaves the SdBG stream in sb.bytes (capacity *cap_bytes) and the bucket table / totals in d_table /
// d_totals; *n_u = distinct items
int s2_sort_emit(cudaStream_t st, uint32_t k, u32 *a, u32 *b, void *ws, S2Bufs &sb, uint64_t n, u64 *d_table, u64 *d_totals,
                 unsigned long long *d_counter, PhaseTrace &tr, uint64_t *n_u_out, uint64_t *cap_bytes) {
  const uint32_t W = s2s_record_words(k), WPT = words_per_tip_label(k);
  const size_t ws_bytes = mhb_s2s_sort_workspace_bytes(n, k);
  int in_b = 0;
  CKR(mhb_s2s_sort(st, a, b, n, k, nullptr, ws, ws_bytes, &in_b));
  tr.mark("s2.sort");
  const u32 *sorted = in_b ? b : a;
  u32 *uniq = in_b ? a : b;
  // equal items -> one item carrying the run length (read_to_sdbg_s2.cpp:560-572)
  const uint64_t n_tiles = (n + kDdTile - 1) / kDdTile;
  CKR(sb.tile_heads.ensure(n_tiles * 4, "read2sdbg: tile counts"));
  CKR(sb.tile_off.ensure(n_tiles * 8, "read2sdbg: tile offsets"));
  CKR(sb.bsum.ensure((n_tiles / 4096 + 4) * 8, "read2sdbg: scan sums"));
#define M(WW) \
  if (W == WW) k_r2s_dd_count<WW><<<(unsigned)n_tiles, kDdThreads, 0, st>>>(sorted, n, sb.tile_heads.as<u32>());
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  CKR(scan32(st, sb.tile_heads.as<u32>(), n_tiles, sb.tile_off.as<u64>(), (uint64_t *)(d_counter + 2), sb.bsum.as<u64>()));
  unsigned long long n_u = 0;
  CK(cudaMemcpyAsync(&n_u, d_counter + 2, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CKR(sb.heads.ensure((size_t)n_u * 8, "read2sdbg: run heads"));
#define M(WW)                                                                                                             \
  if (W == WW)                                                                                                            \
    k_r2s_dd_heads<WW><<<(unsigned)n_tiles, kDdThreads, 0, st>>>(sorted, n, sb.tile_off.as<u64>(), sb.heads.as<u64>());
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
#define M(WW) \
  if (W == WW) k_r2s_dd_build<WW><<<grid_cap(n_u, 256, 16), 256, 0, st>>>(sorted, n, sb.heads.as<u64>(), n_u, uniq);
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  tr.mark("s2.collapse");
  const size_t scr_bytes = mhb_s2s_emit_scratch_bytes(n_u, k);
  *cap_bytes = (uint64_t)n_u * (4ull + 4ull * WPT) + 16;
  CKR(sb.scr.ensure(scr_bytes, "read2sdbg: emit scratch"));
  CKR(sb.bytes.ensure(*cap_bytes, "read2sdbg: SdBG stream"));
  CKR(mhb_s2s_emit_fmt(st, uniq, n_u, k, sb.bytes.as<uint8_t>(), *cap_bytes, d_table, d_totals, sb.scr.p, scr_bytes, 1));
  *n_u_out = n_u;
  return MHB_OK;
}

// res->bytes for res->n_bytes bytes: the caller's sdbg_out when it is large enough, else a host allocation
int result_bytes(const mhb_build_args *args, mhb_build_result *res) {
  if (args->sdbg_out && args->sdbg_out_capacity >= res->n_bytes) res->bytes = args->sdbg_out;
  else res->bytes = (uint8_t *)malloc(std::max<size_t>(1, res->n_bytes));
  return res->bytes ? MHB_OK : mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
}

// ---- one pass: the mercy step (Read2SdbgS2::Initialize, read_to_sdbg_s2.cpp:117-263) and the stage-2 item count ----
// A read reads the stage-1 planes and writes mercy bits at its own positions only, so each chunk's mercy bits go to a
// chunk-sized plane on the global word grid (d_mplane - w0) and are OR-ed into the solid plane over the chunk's words
// right away: no read of another chunk looks at them, and a boundary word shared with the next chunk gets nothing
// but this chunk's bits.  The chunk's solid bits are then final, so its stage-2 items are counted in the same pass.
// List form (cl): the chunk's slice of every round's candidate list is scattered into the chunk-sized candidate planes
// first (the same word grid), and the unchanged mercy kernel reads those.
struct CandPlanes {  // the list form's chunk-sized candidate planes and staging slot
  const CandLists *lists = nullptr;
  u32 *planes = nullptr;  // 3 x plane_words
  uint64_t plane_words = 0;
  u64 *stage = nullptr;
  uint64_t stage_cap = 0;
};
int mercy_count_pass(cudaStream_t st, const EachChunk &each, uint32_t k, int32_t m, bool mercy, const S1Out &so,
                     u32 *d_mplane, unsigned long long *d_counter, PhaseTrace &tr, uint64_t *n_items, uint64_t *n_mercy,
                     const CandPlanes &cl) {
  const uint32_t W = s2s_record_words(k);
  CK(cudaMemsetAsync(d_counter, 0, 8, st));
  if (int rc_ = each([&](const PkgChunk &c) -> int {
    if (mercy) {
      const uint64_t nw = c.w_end - c.w0;
      S1Out o = so;
      if (cl.lists)
        CKR(cand_scatter(st, *cl.lists, c.pv.base0, c.base_end, c.w0, cl.planes, cl.plane_words, cl.stage, cl.stage_cap, &o));
      CK(cudaMemsetAsync(d_mplane, 0, nw * 4, st));
      k_r2s_mercy<<<grid_cap(c.pv.n_reads, 256, 16), 256, 0, st>>>(c.pv, k, o, d_mplane - c.w0, d_counter + 1);
      CK_LAUNCH();
      k_r2s_or_words<<<grid_cap(nw, 256, 16), 256, 0, st>>>(so.is_solid + c.w0, d_mplane, nw);
      CK_LAUNCH();
      tr.mark("s1.mercy");
    }
    if (c.n_edges) {
#define M(WW)                                                                                                 \
  if (W == WW)                                                                                                \
    k_r2s_s2_extract<WW, kS2Count><<<grid_cap(c.n_edges, 256, 16), 256, 0, st>>>(c.pv, k, so.is_solid, m == 1, \
                                                                            c.n_edges, nullptr, d_counter, 0);
      MHB_FOR_WR(M)
#undef M
      CK_LAUNCH();
      tr.mark("s2.count");
    }
    return MHB_OK;
  }))
    return rc_;
  unsigned long long c[2] = {0, 0};
  CK(cudaMemcpyAsync(c, d_counter, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  *n_items = c[0];
  *n_mercy = c[1];
  return MHB_OK;
}

// Stage 2 over contiguous ranges of bucket ids, as s2s_host_rounds does for seq2sdbg.  one_pass: the one range over all
// bucket ids, known without a pass, its items written by one pass into the buffers stage 1 left.  Otherwise the stage-1
// buffers are released, a histogram pass plans the ranges from the exact item count, and per range the in-range items
// of every chunk are appended.  Each non-empty range is sorted, collapsed and emitted.  Equal items share a bucket, so a
// run never spans rounds; the whole item is the sort key, so the order the chunks append in does not matter.  A single
// round's bytes and bucket table go straight into the result; several rounds are stitched onto it.
int run_stage2(const mhb_build_args *args, mhb_build_result *res, cudaStream_t st, const EachChunk &each,
               const u32 *d_solid, unsigned long long *d_counter, u64 *d_table, u64 *d_totals, PhaseTrace &tr, BigBufs &big,
               uint64_t n_items, bool one_pass, const char *held) {
  const uint32_t k = args->k, W = s2s_record_words(k);
  const bool all = args->m == 1;  // stage 2 takes every edge
  uint64_t max_items = n_items;
  BucketRanges ranges = {{0u, 65535u}};
  if (!one_pass) {
    big.a.release();  // sized for stage 1
    big.b.release();
    big.ws.release();
    DevBuf h16;
    CKR(h16.alloc(MHB_NUM_BUCKETS * 8, "read2sdbg: bucket histogram"));
    max_items = g_r2s_s2_limit;
    if (!max_items) {
      const size_t avail = (size_t)(0.92 * (double)free_device_bytes());
      max_items = largest_round(n_items, 0, avail, [&](uint64_t n) { return s2_pass_bytes(n, W, k); });
      if (!max_items)
        return mhb_set_error(MHB_ERR_NOMEM, "read2sdbg: %s no room for a stage-2 round (%zu bytes free)", held, avail);
    }
    max_items = std::min(max_items, n_items);
    CK(cudaMemsetAsync(h16.p, 0, MHB_NUM_BUCKETS * 8, st));
    if (int rc_ = each([&](const PkgChunk &c) -> int {
      if (!c.n_edges) return MHB_OK;
#define M(WW)                                                                                                          \
  if (W == WW)                                                                                                         \
    k_r2s_s2_extract<WW, kS2Hist><<<grid_cap(c.n_edges, 256, 16), 256, 0, st>>>(c.pv, k, d_solid, all, c.n_edges, nullptr, \
                                                                           nullptr, 0, 0, 65535,                      \
                                                                           h16.as<unsigned long long>());
      MHB_FOR_WR(M)
#undef M
      CK_LAUNCH();
      return MHB_OK;
    }))
      return rc_;
    std::vector<uint64_t> h_h16(MHB_NUM_BUCKETS);
    CK(cudaMemcpyAsync(h_h16.data(), h16.p, MHB_NUM_BUCKETS * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    tr.mark("s2.extract.plan");
    CKR(plan_stage_rounds(h_h16.data(), max_items, &ranges));
  }
  CKR(big.a.ensure((size_t)max_items * W * 4 + 16, "read2sdbg: stage-2 items"));
  CKR(big.b.ensure((size_t)max_items * W * 4 + 16, "read2sdbg: stage-2 items (sort buffer)"));
  CKR(big.ws.ensure(mhb_s2s_sort_workspace_bytes(max_items, k), "read2sdbg: sort workspace"));
  S2Bufs sb;
  SdbgStitch out;
  uint64_t seen = 0;
  for (const auto &rg : ranges) {
    CK(cudaMemsetAsync(d_counter, 0, 8, st));
    if (int rc_ = each([&](const PkgChunk &c) -> int {
      if (!c.n_edges) return MHB_OK;
      u32 *dst = big.a.as<u32>();
      if (one_pass) {
#define M(WW)                                                                                                       \
  if (W == WW)                                                                                                      \
    k_r2s_s2_extract<WW, kS2Write><<<grid_cap(c.n_edges, 256, 16), 256, 0, st>>>(c.pv, k, d_solid, all, c.n_edges, dst, \
                                                                            d_counter, n_items);
        MHB_FOR_WR(M)
#undef M
      } else {
#define M(WW)                                                                                                       \
  if (W == WW)                                                                                                      \
    k_r2s_s2_extract<WW, kS2Range><<<grid_cap(c.n_edges, 256, 16), 256, 0, st>>>(c.pv, k, d_solid, all, c.n_edges, dst, \
                                                                            d_counter, max_items, rg.first,        \
                                                                            rg.second, nullptr);
        MHB_FOR_WR(M)
#undef M
      }
      CK_LAUNCH();
      return MHB_OK;
    }))
      return rc_;
    unsigned long long n = n_items;  // one pass: every item, no read-back
    if (!one_pass) {
      CK(cudaMemcpyAsync(&n, d_counter, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
    tr.mark("s2.extract");
    if (n > max_items)
      return mhb_set_error(MHB_ERR_CUDA, "read2sdbg: internal: round of %llu stage-2 items exceeds its plan (%llu)",
                           (unsigned long long)n, (unsigned long long)max_items);
    seen += n;
    if (n == 0) continue;
    uint64_t n_u = 0, cap_bytes = 0;
    CKR(s2_sort_emit(st, k, big.a.as<u32>(), big.b.as<u32>(), big.ws.p, sb, n, d_table, d_totals, d_counter, tr, &n_u,
                     &cap_bytes));
    tr.mark("s2.emit");
    if (ranges.size() > 1) {
      CKR(out.append(st, sb.bytes.as<uint8_t>(), cap_bytes, d_table, d_totals));
    } else {
      uint64_t tot[16];
      CK(cudaMemcpyAsync(tot, d_totals, sizeof(tot), cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      set_sdbg_totals(res, tot);
      if (res->n_bytes > cap_bytes) return mhb_set_error(MHB_ERR_NOMEM, "internal: SdBG byte stream exceeds capacity");
      CKR(result_bytes(args, res));
      CK(cudaMemcpyAsync(res->bucket_table, d_table, (size_t)MHB_NUM_BUCKETS * 32, cudaMemcpyDeviceToHost, st));
      if (res->n_bytes) CK(cudaMemcpyAsync(res->bytes, sb.bytes.p, res->n_bytes, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
    tr.mark("d2h");
    res->n_solid += n_u;  // distinct stage-2 items
    ++res->n_rounds_s2;
  }
  if (seen != n_items)
    return mhb_set_error(MHB_ERR_CUDA, "read2sdbg: internal: the rounds saw %llu of %llu stage-2 items",
                         (unsigned long long)seen, (unsigned long long)n_items);
  if (ranges.size() == 1) return MHB_OK;
  set_sdbg_totals(res, out.tot);
  memcpy(res->bucket_table, out.table.data(), (size_t)MHB_NUM_BUCKETS * 32);
  CKR(result_bytes(args, res));
  if (res->n_bytes) memcpy(res->bytes, out.bytes.data(), res->n_bytes);
  return MHB_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// One rank's share of a build on several GPUs (R2sShare, mhb_internal.h; the steps of mhb_read2sdbg_run_multi)
// ------------------------------------------------------------------------------------------------
struct R2sShare::Impl {
  mhb_build_args a;
  uint32_t k = 0;
  int32_t m = 0;
  bool mercy = false;  // need_mercy with a stage 1
  bool sparse = false; // the candidates as lists (bind_planes)
  PkgIndex ix;         // the whole library
  PkgChunk c;          // the share, package words in pkg
  PkgView shape;       // the library's shape for the post-processing of stage 1
  uint64_t bit_words = 0;
  int n_planes = 0;
  DevBuf pkg, word_off, len, base_off, s1_off, edge_off, planes, mplane, hist, cnt, table, totals;
  DevBuf s1_per_read, s1_rows, s1_bsum;  // from s1_count to s1_store: records per read and owner, their scan
  DevBuf sort_b, sort_ws, pa, pb;        // the owner's sort buffer, workspace and narrow pairs, for the largest round
  S2Bufs s2b;
  SdbgStitch out;                        // the owner's stage-2 rounds
  CandLists made, got;                   // list form: my stage-1 rounds' candidates, and those of my share
  DevBuf cplanes, stage;                 // list form: the share's candidate planes and the staging slot of their scatter
  S1Out so;
  PhaseTrace tr;
  cudaStream_t st = 0;
};

R2sShare::R2sShare() : d_(new Impl) {}
R2sShare::~R2sShare() { delete d_; }
uint32_t R2sShare::s1_record_words() const { return s1_layout(d_->k).RW; }
bool R2sShare::s1_narrow() const { return s1_layout(d_->k).narrow; }
void *R2sShare::planes() const { return d_->planes.p; }

// fixed: the exchange's route and small tables, counters, and the buffers an allocation rounds up to
static constexpr size_t kOwnerFixed = (size_t)64 << 20;

uint64_t R2sShare::s1_round_budget(size_t avail, int n_owners, uint64_t n_total) const {
  const S1Layout l = s1_layout(d_->k);
  const uint64_t n = d_->c.pv.n_reads;
  const size_t fixed = kOwnerFixed + (size_t)n_owners * (pad256(n * 4) + pad256((n + 1) * 8)) + pad256((n / 4096 + 4) * 8);
  // s1_pass_bytes holds the receive buffer (the records) and, narrow, its read_info rows
  uint64_t cap = largest_round(std::max<uint64_t>(n_total, 1), fixed, avail, [&](uint64_t r) { return s1_pass_bytes(r, l); });
  if (cap && g_r2s_s1_limit) cap = std::min(cap, g_r2s_s1_limit);
  return std::min(cap, ::s1_round_cap(l));
}

uint64_t R2sShare::s2_round_budget(size_t avail, uint64_t n_total) const {
  const uint32_t k = d_->k;
  uint64_t cap = largest_round(std::max<uint64_t>(n_total, 1), kOwnerFixed, avail,
                               [&](uint64_t r) { return s2_pass_bytes(r, s2s_record_words(k), k); });
  if (cap && g_r2s_s2_limit) cap = std::min(cap, g_r2s_s2_limit);
  return cap;
}
uint64_t R2sShare::n_reads() const { return d_->c.pv.n_reads; }

namespace {
// the slice [f, e] of a whole-library offset array, rebased to its first entry, on the device
int upload_slice(DevBuf &d, const std::vector<uint64_t> &v, uint64_t f, uint64_t e, const char *what) {
  std::vector<uint64_t> s(v.begin() + f, v.begin() + e + 1);
  for (uint64_t &x : s) x -= v[f];
  return upload(d, s, what);
}
}  // namespace

int R2sShare::load(const mhb_build_args *a, const ReadLibIndex &li, uint64_t first, uint64_t end) {
  Impl &d = *d_;
  d.a = *a;
  d.k = a->k;
  d.m = a->m;
  if (d.k < 9 || d.k > MHB_MAX_K || d.m < 1) return mhb_set_error(MHB_ERR_ARG, "read2sdbg: need 9 <= k <= 255 and m >= 1");
  PkgIndex &ix = d.ix;
  ix.n_reads = a->n_reads;
  ix.li = li;
  pkg_geometry(a->bin, d.k, &ix);
  d.mercy = a->need_mercy && d.m > 1 && ix.n_s1 > 0;
  memset(&d.shape, 0, sizeof(d.shape));
  d.shape.n_reads = ix.n_reads;
  d.shape.fixed_len = ix.fixed_len;
  d.shape.fixed_words = ix.fixed_words;
  PkgChunk &c = d.c;
  c = chunk_of(ix, first, end, d.k);
  const uint64_t n = c.pv.n_reads;
  const cudaStream_t st = d.st;
  CKR(d.pkg.alloc((size_t)c.n_words * 4 + 64, "read2sdbg: package of the share"));
  if (n) {
    const uint64_t w0 = li.word_of(first), nw = li.word_of(end) - w0;
    DevBuf d_bin, d_rec_off;
    CKR(d_bin.alloc((size_t)nw * 4 + 64, "read2sdbg: .bin image of the share"));
    CK(cudaMemcpyAsync(d_bin.p, a->bin + w0, (size_t)nw * 4, cudaMemcpyHostToDevice, st));
    if (!ix.fixed_len) {
      CKR(upload_slice(d_rec_off, li.rec_off, first, end, "read2sdbg: record offsets of the share"));
      CKR(upload_slice(d.word_off, ix.word_off, first, end, "read2sdbg: word offsets of the share"));
      CKR(upload_slice(d.base_off, ix.base_off, first, end, "read2sdbg: base offsets of the share"));
      CKR(upload_slice(d.s1_off, ix.s1_off, first, end, "read2sdbg: stage-1 offsets of the share"));
      CKR(upload_slice(d.edge_off, ix.edge_off, first, end, "read2sdbg: edge offsets of the share"));
      CKR(upload(d.len, std::vector<uint32_t>(ix.len.begin() + first, ix.len.begin() + end), "read2sdbg: lengths of the share"));
      c.pv.word_off = d.word_off.as<u64>();
      c.pv.len = d.len.as<u32>();
      c.pv.base_off = d.base_off.as<u64>();
      c.pv.s1_off = d.s1_off.as<u64>();
      c.pv.edge_off = d.edge_off.as<u64>();
    }
    if (c.n_words) {
      k_r2s_reverse<<<grid_cap(c.n_words, 256, 16), 256, 0, st>>>(d_bin.as<u32>(), n, c.pv.fixed_len, d_rec_off.as<u64>(),
                                                                   c.pv, d.pkg.as<u32>(), c.n_words);
      CK_LAUNCH();
    }
    CK(cudaStreamSynchronize(st));  // d_bin / d_rec_off go out of scope
  }
  c.pv.words = d.pkg.as<u32>();
  d.bit_words = ix.n_bases / 32 + 2;
  memset(&d.so, 0, sizeof(d.so));
  CKR(d.hist.alloc(65536 * 8, "read2sdbg: multiplicity histogram"));
  CK(cudaMemsetAsync(d.hist.p, 0, 65536 * 8, st));
  CKR(d.cnt.alloc(64, "read2sdbg: counters"));
  CK(cudaMemsetAsync(d.cnt.p, 0, 64, st));
  CKR(d.table.alloc((size_t)MHB_NUM_BUCKETS * 32, "read2sdbg: bucket table"));
  CKR(d.totals.alloc(16 * 8, "read2sdbg: totals"));
  CK(cudaStreamSynchronize(st));
  return MHB_OK;
}

bool R2sShare::want_cand_lists(size_t avail) const {
  const Impl &d = *d_;
  return d.mercy && (g_r2s_sparse_mercy || 4 * pad256(d.bit_words * 4) > avail);
}

int R2sShare::bind_planes(bool lists) {
  Impl &d = *d_;
  const PkgChunk &c = d.c;
  const cudaStream_t st = d.st;
  d.sparse = lists && d.mercy;
  if (d.m > 1) {  // m == 1: stage 2 takes every edge and never reads the solid plane
    d.n_planes = d.mercy && !d.sparse ? 4 : 1;
    const size_t pb = (size_t)d.n_planes * d.bit_words * 4;
    CKR(d.planes.alloc(pb, d.sparse ? "read2sdbg: solid plane of the whole library" : "read2sdbg: bit planes of the whole library"));
    CK(cudaMemsetAsync(d.planes.p, 0, pb, st));
    d.so.is_solid = d.planes.as<u32>();
    if (d.mercy && !d.sparse) {
      d.so.no_in = d.so.is_solid + d.bit_words;
      d.so.no_out = d.so.no_in + d.bit_words;
      d.so.any = d.so.no_out + d.bit_words;
    }
    if (d.mercy) CKR(d.mplane.alloc((c.w_end - c.w0) * 4, "read2sdbg: mercy plane of the share"));
    if (d.sparse) {
      CKR(d.cplanes.alloc(3 * (c.w_end - c.w0) * 4, "read2sdbg: mercy candidate planes of the share"));
      CKR(d.stage.alloc(kCandStage * 8, "read2sdbg: mercy candidate staging slot"));
      d.made.init(d.ix.n_bases);
    }
  }
  CK(cudaStreamSynchronize(st));
  return MHB_OK;
}

bool R2sShare::cand_lists() const { return d_->sparse; }
uint64_t R2sShare::base_of(uint64_t read) const {
  const PkgIndex &ix = d_->ix;
  return ix.fixed_len ? read * ix.fixed_len : ix.base_off[read];
}
const std::vector<std::vector<uint64_t>> &R2sShare::cand_made() const { return d_->made.rounds; }
void R2sShare::cand_take(std::vector<std::vector<uint64_t>> *lists) {
  Impl &d = *d_;
  std::vector<std::vector<uint64_t>>().swap(d.made.rounds);
  d.got.rounds.swap(*lists);
}

int R2sShare::s1_hist(uint64_t *hist) {
  Impl &d = *d_;
  memset(hist, 0, 65536 * 8);
  const PkgChunk &c = d.c;
  if (d.m < 2 || !c.n_s1) return MHB_OK;
  const uint32_t NW = s1_layout(d.k).NW;
  DevBuf h16;
  CKR(h16.alloc(MHB_NUM_BUCKETS * 8, "read2sdbg: bucket histogram"));
  CK(cudaMemsetAsync(h16.p, 0, MHB_NUM_BUCKETS * 8, d.st));
  const unsigned grid = grid_cap(c.pv.n_reads * 32, 256, 16);  // one warp per read
#define M(WW) \
  if (NW == WW) k_r2s_s1_range<WW, kS1Hist><<<grid, 256, 0, d.st>>>(c.pv, d.k, 0, 65535, h16.as<unsigned long long>(), nullptr, nullptr, nullptr);
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  CK(cudaMemcpyAsync(hist, h16.p, MHB_NUM_BUCKETS * 8, cudaMemcpyDeviceToHost, d.st));
  CK(cudaStreamSynchronize(d.st));
  return MHB_OK;
}

int R2sShare::s1_count(const OwnerRoute &rt) {
  Impl &d = *d_;
  const PkgChunk &c = d.c;
  const uint64_t n = c.pv.n_reads;
  const int n_owners = rt.n_owners;
  if (n_owners < 1 || n_owners > kS1MaxOwners) return mhb_set_error(MHB_ERR_ARG, "read2sdbg: 1 .. %d owners", kS1MaxOwners);
  if (d.m < 2 || !c.n_s1) return MHB_OK;
  const uint32_t NW = s1_layout(d.k).NW;
  const cudaStream_t st = d.st;
  CKR(d.s1_per_read.ensure((size_t)n_owners * n * 4, "read2sdbg: per-read record counts per owner"));
  CKR(d.s1_rows.ensure((size_t)n_owners * (n + 1) * 8, "read2sdbg: per-read record offsets per owner"));
  CKR(d.s1_bsum.ensure((n / 4096 + 4) * 8, "read2sdbg: scan sums"));
  const unsigned grid = grid_cap(n * 32, 256, 16);  // one warp per read
#define M(WW)                                                                                                        \
  if (NW == WW)                                                                                                      \
    k_r2s_s1_owners<WW, kS1OwnerCount><<<grid, 256, 0, st>>>(c.pv, d.k, rt.owner, (u32)n_owners, rt.lo, rt.hi,       \
                                                             d.s1_per_read.as<u32>(), nullptr, nullptr, nullptr, nullptr);
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  for (int o = 0; o < n_owners; ++o) {
    u64 *oo = d.s1_rows.as<u64>() + (size_t)o * (n + 1);
    CKR(scan32(st, d.s1_per_read.as<u32>() + (size_t)o * n, n, oo, rt.cursor + o, d.s1_bsum.as<u64>()));
  }
  return MHB_OK;
}

int R2sShare::s1_store(const OwnerRoute &rt) {
  Impl &d = *d_;
  const PkgChunk &c = d.c;
  if (d.m < 2 || !c.n_s1) return MHB_OK;
  const uint32_t NW = s1_layout(d.k).NW;
  const unsigned grid = grid_cap(c.pv.n_reads * 32, 256, 16);
#define M(WW)                                                                                                          \
  if (NW == WW)                                                                                                        \
    k_r2s_s1_owners<WW, kS1OwnerWrite><<<grid, 256, 0, d.st>>>(c.pv, d.k, rt.owner, (u32)rt.n_owners, rt.lo, rt.hi,   \
                                                               nullptr, d.s1_rows.as<u64>(), rt.row0, rt.info0, rt.off);
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  return MHB_OK;
}

int R2sShare::s1_own(uint32_t *recs, uint64_t *info, uint64_t n, uint64_t n_max) {
  Impl &d = *d_;
  if (!n) return MHB_OK;
  const S1Layout l = s1_layout(d.k);
  CKR(d.sort_b.ensure((size_t)n_max * l.RW * 4 + 16, "read2sdbg: records (sort buffer)"));
  CKR(d.sort_ws.ensure(s1_ws_bytes(n_max, l), "read2sdbg: sort workspace"));
  if (l.narrow) {
    CKR(d.pa.ensure((size_t)n_max * 8 + 16, "read2sdbg: bucket partition pairs"));
    CKR(d.pb.ensure((size_t)n_max * 8 + 16, "read2sdbg: bucket partition pairs (sort buffer)"));
  }
  const S1Bufs bufs{recs, d.sort_b.as<u32>(), d.sort_ws.p, l.narrow ? info : nullptr, d.pa.as<u32>(), d.pb.as<u32>()};
  return s1_sort_post(d.st, d.shape, d.k, d.m, d.mercy, d.so, d.hist.as<unsigned long long>(), d.tr, bufs, n,
                      d.sparse ? &d.made : nullptr);
}

void R2sShare::s1_end() {
  Impl &d = *d_;
  for (DevBuf *b : {&d.s1_per_read, &d.s1_rows, &d.s1_bsum, &d.sort_b, &d.sort_ws, &d.pa, &d.pb}) b->release();
}

int R2sShare::or_planes(const void *peer_planes) {
  Impl &d = *d_;
  const PkgChunk &c = d.c;
  if (!d.n_planes || !c.pv.n_reads) return MHB_OK;
  const uint64_t nw = c.w_end - c.w0;
  for (int p = 0; p < d.n_planes; ++p) {
    const uint64_t at = (uint64_t)p * d.bit_words + c.w0;
    k_r2s_or_words<<<grid_cap(nw, 256, 16), 256, 0, d.st>>>(d.planes.as<u32>() + at, (const u32 *)peer_planes + at, nw);
    CK_LAUNCH();
  }
  CK(cudaStreamSynchronize(d.st));
  return MHB_OK;
}

int R2sShare::mercy_count(uint64_t *n_items, uint64_t *n_mercy) {
  Impl &d = *d_;
  *n_items = *n_mercy = 0;
  if (!d.c.pv.n_reads) return MHB_OK;
  const EachChunk each = [&](const ChunkFn &fn) { return fn(d.c); };
  CandPlanes cp;
  if (d.sparse) {
    cp.lists = &d.got;
    cp.planes = d.cplanes.as<u32>();
    cp.plane_words = d.c.w_end - d.c.w0;
    cp.stage = d.stage.as<u64>();
    cp.stage_cap = kCandStage;
  }
  CKR(mercy_count_pass(d.st, each, d.k, d.m, d.mercy, d.so, d.mplane.as<u32>(), d.cnt.as<unsigned long long>(), d.tr,
                       n_items, n_mercy, cp));
  if (d.sparse) {
    for (DevBuf *b : {&d.cplanes, &d.stage}) b->release();
    std::vector<std::vector<uint64_t>>().swap(d.got.rounds);
  }
  return MHB_OK;
}

int R2sShare::s2_hist(uint64_t *hist) {
  Impl &d = *d_;
  memset(hist, 0, 65536 * 8);
  const PkgChunk &c = d.c;
  if (!c.n_edges) return MHB_OK;
  const uint32_t W = s2s_record_words(d.k);
  DevBuf h16;
  CKR(h16.alloc(MHB_NUM_BUCKETS * 8, "read2sdbg: bucket histogram"));
  CK(cudaMemsetAsync(h16.p, 0, MHB_NUM_BUCKETS * 8, d.st));
#define M(WW)                                                                                                          \
  if (W == WW)                                                                                                         \
    k_r2s_s2_extract<WW, kS2Hist><<<grid_cap(c.n_edges, 256, 16), 256, 0, d.st>>>(c.pv, d.k, d.so.is_solid, d.m == 1,     \
                                                                                c.n_edges, nullptr, nullptr, 0, 0, 65535, \
                                                                                h16.as<unsigned long long>());
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  CK(cudaMemcpyAsync(hist, h16.p, MHB_NUM_BUCKETS * 8, cudaMemcpyDeviceToHost, d.st));
  CK(cudaStreamSynchronize(d.st));
  return MHB_OK;
}

int R2sShare::s2_send(const OwnerRoute &rt) {
  Impl &d = *d_;
  const PkgChunk &c = d.c;
  if (!c.n_edges) return MHB_OK;
  const uint32_t W = s2s_record_words(d.k);
  const OwnerSink sink{rt.owner, rt.base, (unsigned long long *)rt.cursor, rt.cap};
#define M(WW)                                                                                                         \
  if (W == WW)                                                                                                        \
    k_r2s_s2_extract<WW, kS2Owner><<<grid_cap(c.n_edges, 256, 16), 256, 0, d.st>>>(c.pv, d.k, d.so.is_solid, d.m == 1, \
                                                                                 c.n_edges, nullptr, nullptr, 0, 0, 0, \
                                                                                 nullptr, sink, rt.lo, rt.hi);
  MHB_FOR_WR(M)
#undef M
  CK_LAUNCH();
  return MHB_OK;
}

int R2sShare::s2_own(uint32_t *items, uint64_t n, uint64_t n_max) {
  Impl &d = *d_;
  if (!n) return MHB_OK;
  const uint32_t W = s2s_record_words(d.k);
  CKR(d.sort_b.ensure((size_t)n_max * W * 4 + 16, "read2sdbg: stage-2 items (sort buffer)"));
  CKR(d.sort_ws.ensure(mhb_s2s_sort_workspace_bytes(n_max, d.k), "read2sdbg: sort workspace"));
  uint64_t n_u = 0, cap_bytes = 0;
  CKR(s2_sort_emit(d.st, d.k, items, d.sort_b.as<u32>(), d.sort_ws.p, d.s2b, n, d.table.as<u64>(), d.totals.as<u64>(),
                   d.cnt.as<unsigned long long>(), d.tr, &n_u, &cap_bytes));
  return d.out.append(d.st, d.s2b.bytes.as<uint8_t>(), cap_bytes, d.table.as<u64>(), d.totals.as<u64>());
}

void R2sShare::s2_result(std::vector<uint8_t> *bytes, std::vector<uint64_t> *table, uint64_t *totals) {
  Impl &d = *d_;
  bytes->swap(d.out.bytes);
  table->swap(d.out.table);
  memcpy(totals, d.out.tot, 16 * 8);
  d.out = SdbgStitch();
  for (DevBuf *b : {&d.sort_b, &d.sort_ws, &d.s2b.tile_heads, &d.s2b.tile_off, &d.s2b.bsum, &d.s2b.heads, &d.s2b.scr,
                    &d.s2b.bytes})
    b->release();
}

int R2sShare::counting(uint64_t *hist) {
  CK(cudaMemcpy(hist, d_->hist.p, 65536 * 8, cudaMemcpyDeviceToHost));
  return MHB_OK;
}

extern "C" int mhb_set_r2s_round_limit(uint64_t max_s1_records, uint64_t max_s2_items) {
  g_r2s_s1_limit = max_s1_records;
  g_r2s_s2_limit = max_s2_items;
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// main_read2sdbg (main_sdbg_build.cpp:88-156) from a host `.bin` image: SdBG item stream + bucket table out.
// ------------------------------------------------------------------------------------------------
extern "C" int mhb_read2sdbg_host(const mhb_build_args *args, mhb_build_result *res) {
  if (!args || !res) return mhb_set_error(MHB_ERR_ARG, "null argument");
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k;
  const int32_t m = args->m;
  if (k < 9 || k > MHB_MAX_K || m < 1) return mhb_set_error(MHB_ERR_ARG, "read2sdbg: need 9 <= k <= 255 and m >= 1");
  if (mhb_device_count() <= 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  read_stream_stats_reset();
  cudaStream_t st = 0;
  PhaseTrace tr;
  tr.mark("start");
  PkgIndex ix;
  CKR(index_pkg(args->bin, args->bin_words, args->n_reads, k, &ix));
  const uint32_t W = s2s_record_words(k), WPT = words_per_tip_label(k);
  res->words_per_tip_label = WPT;
  res->n_edge_records = ix.n_edges;
  res->bucket_table = (uint64_t *)calloc((size_t)MHB_NUM_BUCKETS * 4, 8);
  res->counting = (int64_t *)calloc(65536, 8);
  struct ResGuard {  // a failing call hands nothing back
    mhb_build_result *r;
    const uint8_t *caller_buf;
    bool ok = false;
    ~ResGuard() {
      if (ok) return;
      free(r->bucket_table);
      free(r->counting);
      if (r->bytes != caller_buf) free(r->bytes);
      r->bucket_table = nullptr;
      r->counting = nullptr;
      r->bytes = nullptr;
    }
  } guard{res, args->sdbg_out};
  if (!res->bucket_table || !res->counting) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");

  // ---- device memory: the package resident, or streamed from host memory in chunks (DESIGN.md §4.9) ----
  const S1Layout l1 = s1_layout(k);
  const bool s1_runs = m > 1 && ix.n_s1 > 0;
  const bool mercy = args->need_mercy && m > 1;
  const uint64_t bit_words = ix.n_bases / 32 + 2;
  const ResidentPlan rp = resident_plan(ix, args->bin_words, m, mercy);
  const uint64_t est_items = (uint64_t)(2.2 * (double)ix.n_edges) + 1024;
  const size_t s1_one = s1_runs ? s1_pass_bytes(ix.n_s1, l1) : 0;
  const size_t s2_est = ix.n_edges ? s2_pass_bytes(est_items, W, k) : 0;
  // the arena earlier host-level calls keep is reclaimable: free it when it stands in the way of this call
  if (mhb_arena_bytes() &&
      (double)(rp.resident + std::max({rp.upload, s1_one, s2_est})) > 0.92 * (double)free_device_bytes())
    mhb_release();
  const bool stream = stream_decide(rp, ix, k, m, free_device_bytes(), read_chunk_limit());
  PkgSource src;
  CKR(src.plan(args, ix, k, stream, read_chunk_limit() ? read_chunk_limit() : read_chunk_auto_bytes()));
  const char *held = stream ? "the bit planes and read chunk buffers leave" : "the resident read library leaves";
  MercyForm form;
  if (stream) {  // resident: the solid plane, the mercy candidates (planes or lists), a chunk's mercy plane, the chunk buffers
    form = mercy_form(bit_words, src.max_plane_words, src.streamed_bytes(), m, mercy, free_device_bytes(), g_r2s_sparse_mercy);
    const size_t need = form.sparse ? form.lists : form.planes;
    if (need > free_device_bytes())
      return mhb_set_error(MHB_ERR_NOMEM,
                           "read2sdbg: the streamed read library needs %zu bytes of device memory (mercy candidates as "
                           "%s, read chunk buffers %zu), %zu are free",
                           need, form.sparse ? "lists" : "planes", src.streamed_bytes(), free_device_bytes());
  }
  g_mercy_stats = MercyStats();
  g_mercy_stats.sparse = form.sparse ? 1 : 0;
  CandLists lists;
  lists.init(ix.n_bases);
  CKR(src.bind(st, ix));
  tr.mark("h2d.upload+reverse");
  const EachChunk each = [&](const ChunkFn &fn) { return src.each(st, fn); };
  PkgView shape;  // the library's shape for the post-processing of stage 1, which reads no reads
  memset(&shape, 0, sizeof(shape));
  shape.n_reads = ix.n_reads;
  shape.fixed_len = ix.fixed_len;
  shape.fixed_words = ix.fixed_words;

  // ---- stage 1 (only when the threshold can reject anything, main_sdbg_build.cpp:141-147) ----
  DevBuf d_solid, d_planes, d_mplane, d_hist, d_cnt;
  if (m > 1) {  // m == 1: stage 2 takes every edge and never reads the solid plane
    CKR(d_solid.alloc(bit_words * 4, "read2sdbg: solid plane"));
    CK(cudaMemsetAsync(d_solid.p, 0, bit_words * 4, st));
  }
  CKR(d_hist.alloc(65536 * 8, "read2sdbg: multiplicity histogram"));
  CK(cudaMemsetAsync(d_hist.p, 0, 65536 * 8, st));
  CKR(d_cnt.alloc(64, "read2sdbg: counters"));
  CK(cudaMemsetAsync(d_cnt.p, 0, 64, st));
  unsigned long long *d_counter = d_cnt.as<unsigned long long>();
  DevBuf d_table, d_totals;
  CKR(d_table.alloc((size_t)MHB_NUM_BUCKETS * 32, "read2sdbg: bucket table"));
  CKR(d_totals.alloc(16 * 8, "read2sdbg: totals"));
  BigBufs big;
  S1Out so;
  memset(&so, 0, sizeof(so));
  CandPlanes cp;
  DevBuf d_cplanes, d_stage;
  so.is_solid = d_solid.as<u32>();
  if (s1_runs) {
    if (mercy && !form.sparse) {
      CKR(d_planes.alloc(bit_words * 4 * 3, "read2sdbg: mercy candidate planes"));
      CK(cudaMemsetAsync(d_planes.p, 0, bit_words * 4 * 3, st));
      so.no_in = d_planes.as<u32>();
      so.no_out = so.no_in + bit_words;
      so.any = so.no_out + bit_words;
    }
    if (mercy) CKR(d_mplane.alloc(src.max_plane_words * 4, "read2sdbg: mercy plane of a chunk"));
    if (mercy && form.sparse) {  // the list form: chunk-sized candidate planes and the staging slot of their scatter
      cp.lists = &lists;
      cp.plane_words = src.max_plane_words;
      cp.stage_cap = kCandStage;
      CKR(d_cplanes.alloc(3 * cp.plane_words * 4, "read2sdbg: mercy candidate planes of a chunk"));
      CKR(d_stage.alloc(cp.stage_cap * 8, "read2sdbg: mercy candidate staging slot"));
      cp.planes = d_cplanes.as<u32>();
      cp.stage = d_stage.as<u64>();
    }
    // one pass when the records fit (and no cap is set), else rounds over bucket ranges
    const size_t avail = (size_t)(0.92 * (double)free_device_bytes());
    uint64_t max_n = 0;  // one pass
    size_t min_rec = 0, min_ws = 0;
    if (s1_plan_round(l1, ix.n_s1, src.max_reads, avail, g_r2s_s1_limit, &max_n))
      return mhb_set_error(MHB_ERR_NOMEM, "read2sdbg: %s no room for a stage-1 round (%zu bytes free)", held, avail);
    if (max_n == 0) {
      // size the shared buffers for stage 2 as well when that fits: ~1.6 items per edge position on a 30x library, 2.2
      // to be safe (stage 2 reallocates when its count launch says more)
      const size_t rec1 = pad256((size_t)ix.n_s1 * l1.RW * 4 + 16), ws1 = pad256(s1_ws_bytes(ix.n_s1, l1));
      const size_t rec2 = pad256((size_t)est_items * W * 4 + 16), ws2 = pad256(mhb_s2s_sort_workspace_bytes(est_items, k));
      if (s1_one - 2 * rec1 - ws1 + 2 * std::max(rec1, rec2) + std::max(ws1, ws2) <= avail) {
        min_rec = (size_t)est_items * W * 4 + 16;
        min_ws = mhb_s2s_sort_workspace_bytes(est_items, k);
      }
    }
    CKR(run_stage1(st, each, shape, ix, src.max_reads, k, m, mercy, so, d_hist.as<unsigned long long>(), tr, big, max_n,
                   min_rec, min_ws, &res->n_rounds_s1, form.sparse ? &lists : nullptr));
  }

  // ---- the mercy step and the stage-2 item count, then stage 2 ----
  const bool mercy_runs = s1_runs && mercy;
  uint64_t n_items = 0;
  if (cp.lists) {
    g_mercy_stats.n_entries = lists.n_entries();
    g_mercy_stats.host_bytes = g_mercy_stats.n_entries * 8;
  }
  if (mercy_runs || ix.n_edges)
    CKR(mercy_count_pass(st, each, k, m, mercy_runs, so, d_mplane.as<u32>(), d_counter, tr, &n_items, &res->n_mercy, cp));
  if (s1_runs) {
    CK(cudaMemcpyAsync(res->counting, d_hist.p, 65536 * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    d_planes.release();
    d_mplane.release();
    d_cplanes.release();
    d_stage.release();
    std::vector<std::vector<uint64_t>>().swap(lists.rounds);
  }
  res->n_sort_items = n_items;
  if (n_items) {
    // one pass when the items fit next to what stage 1 left allocated (its buffers count as free), else rounds
    const size_t held_b = big.a.bytes + big.b.bytes + big.ws.bytes;
    const bool rounds = (g_r2s_s2_limit && n_items > g_r2s_s2_limit) ||
                        (double)s2_pass_bytes(n_items, W, k) > 0.92 * (double)(free_device_bytes() + held_b);
    CKR(run_stage2(args, res, st, each, d_solid.as<u32>(), d_counter, d_table.as<u64>(), d_totals.as<u64>(), tr, big,
                   n_items, !rounds, held));
  } else {
    CKR(result_bytes(args, res));
  }
  tr.mark("release");
  CK(cudaStreamSynchronize(st));
  res->t_h2d_ms = tr.sum("h2d");
  res->t_count_ms = tr.sum("s1.extract") + tr.sum("s1.partition");  // records + stable bucket partition
  res->t_mercy_ms = tr.sum("s1.kmsort");                            // kmsort emulation (levels + finish)
  res->t_s2s_ms = tr.sum("s2");
  res->t_d2h_ms = tr.sum("d2h");
  res->t_total_ms = tr.sum("");
  tr.report();
  guard.ok = true;
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// Self-test hooks (host): the same __host__ __device__ code the kernels run, for the CPU-only tests (tests/test_r2s_cpu.py).
// ------------------------------------------------------------------------------------------------
extern "C" int mhb_selftest_r2s_s1_record(const uint32_t *pkg_words, uint32_t nwords, uint32_t L, uint32_t k, uint32_t e,
                                          uint64_t base_off, uint32_t *rec_out) {
  if (k < 9 || k > MHB_MAX_K || L < k + 1 || e >= L - k + 4) return mhb_set_error(MHB_ERR_ARG, "bad args");
  const uint32_t NW = r2s_s1_key_words(k);
  u32 p, want;
  s1_emission(L, k, e, p, want);
#define M(WW)                                                       \
  if (NW == WW) {                                                   \
    u32 rec[WW + 2];                                                \
    make_s1_record<WW>(pkg_words, nwords, L, k, p, want, base_off, rec); \
    memcpy(rec_out, rec, sizeof(rec));                              \
  }
  MHB_FOR_WR(M)
#undef M
  return MHB_OK;
}

extern "C" int mhb_selftest_r2s_item(const uint32_t *pkg_words, uint32_t nwords, uint32_t L, uint32_t k, uint32_t i,
                                     uint32_t strand, uint32_t type, uint32_t *rec_out, uint32_t *palindrome_out) {
  if (k < 9 || k > MHB_MAX_K || i + k >= L || strand > 1 || type > 2) return mhb_set_error(MHB_ERR_ARG, "bad args");
  const uint32_t W = s2s_record_words(k);
#define M(WW)                                                              \
  if (W == WW) {                                                           \
    u32 rec[WW];                                                           \
    make_r2s_item<WW>(pkg_words, nwords, k, i, strand, type, rec);         \
    memcpy(rec_out, rec, sizeof(rec));                                     \
    *palindrome_out = edge_is_palindrome<WW>(pkg_words, nwords, k, i) ? 1u : 0u; \
  }
  MHB_FOR_WR(M)
#undef M
  return MHB_OK;
}

// kmsort emulation of ONE bucket on the host, exactly as the kernels do it (records of nw + 2 words): radix levels that
// mark the range starts, then the insertion sorts of all marked small ranges
namespace {
int kmsort_host(uint32_t *recs, uint64_t n, uint32_t nw, uint32_t RW) {
  if (n <= 1) return MHB_OK;
  std::vector<KmSeg> cur, nxt;
  std::vector<u32> count(256), last(256), bnd(n / 32 + 2, 0u);
  int kb = 4 * (int)nw - 2 - 1;
  bit_or(bnd.data(), 0);
#define M(WW)                                                                                           \
  if (RW == WW) {                                                                                       \
    if (n > (uint64_t)kKmInsertThreshold) cur.push_back(KmSeg{0, n});                                   \
    while (!cur.empty()) {                                                                              \
      nxt.clear();                                                                                      \
      for (const KmSeg &s : cur) {                                                                      \
        km_radix_range<WW>(recs + s.start * WW, (u32)s.len, nw, kb, count.data(), last.data());         \
        u32 b0 = 0;                                                                                     \
        for (int i = 0; i < 256; ++i) {                                                                 \
          const u32 c = count[i];                                                                       \
          if (c) bit_or(bnd.data(), s.start + b0);                                                      \
          if (c > (u32)kKmInsertThreshold && kb > 0) nxt.push_back(KmSeg{s.start + b0, c});             \
          b0 += c;                                                                                      \
        }                                                                                               \
      }                                                                                                 \
      cur.swap(nxt);                                                                                    \
      --kb;                                                                                             \
    }                                                                                                   \
    for (u64 i = 0; i < n; ++i) {                                                                       \
      if (!bit_at(bnd.data(), i)) continue;                                                             \
      const u32 len = km_small_range(bnd.data(), n, i, (u32)kKmInsertThreshold);                        \
      if (len >= 2) km_insertion<WW>(recs + i * WW, len, nw);                                           \
    }                                                                                                   \
  }
  MHB_FOR_RW(M)
#undef M
  return MHB_OK;
}

// The shared-memory form of the same sort, mirrored on the host with the same building blocks (km_walk_src on the tags,
// km_insertion_idx on the index array of a staged range): level 0 gathers the bucket into a second buffer, later levels
// stage ranges of at most `wcap` records (0 = km_wcap of the record width, as on the device), larger ones and buckets
// above `cap` tags take the in-place walk; what is left unsorted is marked and finished by insertion.
int kmsort_smem_host(uint32_t *recs, uint64_t n, uint32_t nw, uint32_t RW, uint32_t cap, uint32_t wcap) {
  if (n <= 1) return MHB_OK;
  std::vector<KmSeg> cur, nxt;
  std::vector<u32> cnt(256), last(256), beg(256), bnd(n / 32 + 2, 0u), todo(n / 32 + 2, 0u);
  std::vector<uint8_t> tags(n);
  std::vector<uint16_t> src(n);
  std::vector<u32> other((size_t)n * RW), staged;
  int kb = 4 * (int)nw - 2 - 1;
#define M(WW)                                                                                                         \
  if (RW == WW) {                                                                                                     \
    if (!wcap) wcap = km_wcap(WW);                                                                                    \
    bit_or(bnd.data(), 0);                                                                                            \
    auto children = [&](u64 start, bool sorted_small) {                                                               \
      u32 acc = 0;                                                                                                    \
      for (int i = 0; i < 256; ++i) {                                                                                 \
        const u32 c = cnt[i];                                                                                         \
        if (c) {                                                                                                      \
          bit_or(bnd.data(), start + acc);                                                                            \
          if (kb > 0) {                                                                                               \
            if (c > (u32)kKmInsertThreshold) nxt.push_back(KmSeg{start + acc, c});                                    \
            else if (c >= 2 && !sorted_small) bit_or(todo.data(), start + acc);                                       \
          }                                                                                                           \
        }                                                                                                             \
        acc += c;                                                                                                     \
      }                                                                                                               \
    };                                                                                                                \
    /* level 0 (k_r2s_km_bucket) */                                                                                   \
    if (n <= (uint64_t)kKmInsertThreshold) {                                                                          \
      bit_or(todo.data(), 0);                                                                                         \
    } else if (n > cap || n > 65535) {                                                                                \
      km_radix_range<WW>(recs, (u32)n, nw, kb, cnt.data(), last.data());                                              \
      children(0, false);                                                                                             \
    } else {                                                                                                          \
      std::fill(cnt.begin(), cnt.end(), 0u);                                                                          \
      for (u32 i = 0; i < n; ++i) ++cnt[tags[i] = (uint8_t)km_byte_mem(recs + (size_t)i * WW, nw, kb)];               \
      for (u32 i = 0, acc = 0; i < 256; ++i) {                                                                        \
        last[i] = acc;                                                                                                \
        acc += cnt[i];                                                                                                \
      }                                                                                                               \
      km_walk_src<uint16_t>(tags.data(), (u32)n, cnt.data(), last.data(), src.data());                                \
      for (u32 q = 0; q < n; ++q) memcpy(&other[(size_t)q * WW], recs + (size_t)src[q] * WW, 4 * WW);                 \
      memcpy(recs, other.data(), (size_t)n * WW * 4);                                                                 \
      children(0, false);                                                                                             \
    }                                                                                                                 \
    /* levels >= 1 (k_r2s_km_warp) */                                                                                 \
    while (!nxt.empty() && kb > 0) {                                                                                  \
      cur.swap(nxt);                                                                                                  \
      nxt.clear();                                                                                                    \
      --kb;                                                                                                           \
      for (const KmSeg &sg : cur) {                                                                                   \
        u32 *a = recs + sg.start * WW;                                                                                \
        const u32 len = (u32)sg.len;                                                                                  \
        if (len > wcap) {                                                                                             \
          km_radix_range<WW>(a, len, nw, kb, cnt.data(), last.data());                                                \
          children(sg.start, false);                                                                                  \
          continue;                                                                                                   \
        }                                                                                                             \
        staged.assign(a, a + (size_t)len * WW);                                                                       \
        std::fill(cnt.begin(), cnt.end(), 0u);                                                                        \
        for (u32 i = 0; i < len; ++i) ++cnt[tags[i] = (uint8_t)km_byte_mem(&staged[(size_t)i * WW], nw, kb)];         \
        for (u32 i = 0, acc = 0; i < 256; ++i) {                                                                      \
          beg[i] = last[i] = acc;                                                                                     \
          acc += cnt[i];                                                                                              \
        }                                                                                                             \
        km_walk_src<uint16_t>(tags.data(), len, cnt.data(), last.data(), src.data());                                 \
        if (kb > 0)                                                                                                   \
          for (int b = 0; b < 256; ++b)                                                                               \
            if (cnt[b] >= 2 && cnt[b] <= (u32)kKmInsertThreshold)                                                     \
              km_insertion_idx<uint16_t>(staged.data(), WW, src.data() + beg[b], cnt[b], nw);                         \
        for (u32 q = 0; q < len; ++q) memcpy(a + (size_t)q * WW, &staged[(size_t)src[q] * WW], 4 * WW);               \
        children(sg.start, true);                                                                                     \
      }                                                                                                               \
    }                                                                                                                 \
    /* k_r2s_kmsort_finish */                                                                                         \
    for (u64 i = 0; i < n; ++i) {                                                                                     \
      if (!bit_at(todo.data(), i)) continue;                                                                          \
      const u32 len = km_small_range(bnd.data(), n, i, (u32)kKmInsertThreshold);                                      \
      if (len >= 2) km_insertion<WW>(recs + i * WW, len, nw);                                                         \
    }                                                                                                                 \
  }
  MHB_FOR_RW(M)
#undef M
  return MHB_OK;
}
}  // namespace

extern "C" int mhb_selftest_kmsort(uint32_t *recs, uint64_t n, uint32_t nw) {
  if (nw < 1 || nw + 2 > 17 || n >= (1ull << 32)) return mhb_set_error(MHB_ERR_ARG, "bad args");
  return kmsort_host(recs, n, nw, nw + 2);
}

extern "C" int mhb_selftest_kmsort_smem(uint32_t *recs, uint64_t n, uint32_t nw, uint32_t cap, uint32_t wcap) {
  if (nw < 1 || nw + 2 > 17 || n >= (1ull << 32)) return mhb_set_error(MHB_ERR_ARG, "bad args");
  return kmsort_smem_host(recs, n, nw, nw + 2, cap, wcap);
}

// The same two forms on the narrow stage-1 layout: records of nw key words + one row-index word (nw <= 17)
extern "C" int mhb_selftest_kmsort_narrow(uint32_t *recs, uint64_t n, uint32_t nw, int smem, uint32_t cap, uint32_t wcap) {
  if (nw < 2 || nw > 17 || n >= (1ull << 32)) return mhb_set_error(MHB_ERR_ARG, "bad args");
  return smem ? kmsort_smem_host(recs, n, nw, nw + 1, cap, wcap) : kmsort_host(recs, n, nw, nw + 1);
}

// stage-1 Lv2Postprocess + the mercy step on host arrays (one sorted bucket / one read), same code as the kernels
extern "C" int mhb_selftest_r2s_s1_group(const uint32_t *recs, uint64_t n, uint32_t k, int32_t m, uint32_t fixed_len,
                                         uint64_t n_reads, int need_mercy, uint32_t *is_solid, uint32_t *no_in,
                                         uint32_t *no_out, uint32_t *any, int64_t *counting) {
  const uint32_t nw = r2s_s1_key_words(k), rw = nw + 2;
  PkgView pv;
  memset(&pv, 0, sizeof(pv));
  pv.fixed_len = fixed_len;
  pv.n_reads = n_reads;
  S1Out o{is_solid, no_in, no_out, any};
  for (u64 g = 0; g < n;) {
    u32 hv[16], nh;
    g = s1_group(recs, nullptr, n, g, rw, nw, k, m, pv, o, need_mercy != 0, hv, nh);
    for (u32 q = 0; q < nh; ++q) counting[hv[q] > MHB_MAX_MUL ? MHB_MAX_MUL : hv[q]]++;
  }
  return MHB_OK;
}

extern "C" int mhb_selftest_r2s_mercy_read(uint32_t fixed_len, uint64_t n_reads, uint64_t r, uint32_t k,
                                           const uint32_t *is_solid, const uint32_t *no_in, const uint32_t *no_out,
                                           const uint32_t *any, uint32_t *mercy, uint32_t *added_out) {
  PkgView pv;
  memset(&pv, 0, sizeof(pv));
  pv.fixed_len = fixed_len;
  pv.n_reads = n_reads;
  S1Out o{const_cast<u32 *>(is_solid), const_cast<u32 *>(no_in), const_cast<u32 *>(no_out), const_cast<u32 *>(any)};
  *added_out = r2s_mercy_read(pv, r, k, o, mercy);
  return MHB_OK;
}

// The offsets of one chunk [first, first + count) of a `.bin` library.  derive = 1: as the streamed path derives them on
// the device, from the chunk's records alone (r2s_read_geom per read, exclusive scans; record offsets rebased to the
// chunk as the read stream hands them over), and *base0_out = the chunk's global base (PkgView::base0).  derive = 0:
// index_pkg's arrays of the whole library sliced to the chunk and rebased (variable-length libraries only).  len_out
// gets count entries, the offset arrays count + 1.
extern "C" int mhb_selftest_r2s_chunk_index(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t k,
                                            uint64_t first, uint64_t count, int derive, uint32_t *len_out,
                                            uint64_t *word_off_out, uint64_t *base_off_out, uint64_t *s1_off_out,
                                            uint64_t *edge_off_out, uint64_t *base0_out) {
  if (first + count > n_reads) return mhb_set_error(MHB_ERR_ARG, "chunk beyond the library");
  PkgIndex ix;
  CKR(index_pkg(bin, bin_words, n_reads, k, &ix));
  if (!derive) {
    if (ix.fixed_len) return mhb_set_error(MHB_ERR_ARG, "fixed-length library: index_pkg keeps no per-read arrays");
    for (uint64_t r = 0; r <= count; ++r) {
      if (r < count) len_out[r] = ix.len[first + r];
      word_off_out[r] = ix.word_off[first + r] - ix.word_off[first];
      base_off_out[r] = ix.base_off[first + r] - ix.base_off[first];
      s1_off_out[r] = ix.s1_off[first + r] - ix.s1_off[first];
      edge_off_out[r] = ix.edge_off[first + r] - ix.edge_off[first];
    }
    *base0_out = ix.base_off[first];
    return MHB_OK;
  }
  const ReadLibIndex &li = ix.li;
  const uint32_t *chunk = bin + li.word_of(first);
  uint64_t w = 0, b = 0, s = 0, e = 0;
  for (uint64_t r = 0; r <= count; ++r) {
    word_off_out[r] = w;
    base_off_out[r] = b;
    s1_off_out[r] = s;
    edge_off_out[r] = e;
    if (r == count) break;
    u32 l, lw, ls, le;
    r2s_read_geom(chunk[li.word_of(first + r) - li.word_of(first)], k, l, lw, ls, le);
    len_out[r] = l;
    w += lw;
    b += l;
    s += ls;
    e += le;
  }
  *base0_out = chunk_of(ix, first, first + count, k).pv.base0;
  return MHB_OK;
}

// The residency rule of mhb_read2sdbg_host on given library sizes and free device bytes: *stream_out = 1 when the
// library would be streamed; *resident_out / *upload_out = the bytes of its resident form and of the upload.
extern "C" int mhb_selftest_r2s_stream_decide(uint64_t n_reads, uint64_t bin_words, uint32_t fixed_len, uint64_t n_words,
                                              uint64_t n_bases, uint64_t n_s1, uint64_t n_edges, uint32_t k, int32_t m,
                                              int need_mercy, uint64_t free_bytes, uint64_t chunk_limit,
                                              uint64_t *resident_out, uint64_t *upload_out, int *stream_out) {
  if (k < 9 || k > MHB_MAX_K || m < 1) return mhb_set_error(MHB_ERR_ARG, "bad args");
  PkgIndex ix;
  ix.n_reads = n_reads;
  ix.fixed_len = fixed_len;
  ix.fixed_words = div_ceil(fixed_len, 16);
  ix.n_words = n_words;
  ix.n_bases = n_bases;
  ix.n_s1 = n_s1;
  ix.n_edges = n_edges;
  const ResidentPlan p = resident_plan(ix, bin_words, m, need_mercy && m > 1);
  *resident_out = p.resident;
  *upload_out = p.upload;
  *stream_out = stream_decide(p, ix, k, m, free_bytes, chunk_limit) ? 1 : 0;
  return MHB_OK;
}

// mhb_read2sdbg_host with the narrow stage-1 layout (key + row index records, read_info in a side array) at any k: the
// layout mhb_read2sdbg_host takes only for k > 237, run where both fit so that the tests can compare the two
extern "C" int mhb_selftest_read2sdbg_narrow(const mhb_build_args *args, mhb_build_result *res) {
  g_r2s_force_narrow = true;
  const int rc = mhb_read2sdbg_host(args, res);
  g_r2s_force_narrow = false;
  return rc;
}

// The stage-1 round plan of mhb_read2sdbg_host for n_s1 records of k, chunks of at most max_reads reads, avail free
// device bytes and the round cap `limit` (0 = none): *max_n_out = 0 for one pass, else the most records of a round;
// *rec_words_out = words per stage-1 sort record.
extern "C" int mhb_selftest_r2s_s1_plan(uint32_t k, uint64_t n_s1, uint64_t max_reads, uint64_t avail, uint64_t limit,
                                        uint64_t *max_n_out, uint32_t *rec_words_out) {
  if (k < 9 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "bad args");
  const S1Layout l = s1_layout(k);
  *rec_words_out = l.RW;
  if (s1_plan_round(l, n_s1, max_reads, (size_t)avail, limit, max_n_out))
    return mhb_set_error(MHB_ERR_NOMEM, "read2sdbg: no room for a stage-1 round");
  return MHB_OK;
}

extern "C" int mhb_set_r2s_sparse_mercy(int mode) {
  if (mode < 0 || mode > 1) return mhb_set_error(MHB_ERR_ARG, "mhb_set_r2s_sparse_mercy: 0 = automatic, 1 = lists");
  g_r2s_sparse_mercy = mode;
  return MHB_OK;
}

extern "C" int mhb_r2s_mercy_stats(int *sparse, uint64_t *n_entries, uint64_t *host_bytes) {
  if (sparse) *sparse = g_mercy_stats.sparse;
  if (n_entries) *n_entries = g_mercy_stats.n_entries;
  if (host_bytes) *host_bytes = g_mercy_stats.host_bytes;
  return MHB_OK;
}

// The form of the mercy candidates mhb_read2sdbg_host takes for a streamed library (mercy_form)
extern "C" int mhb_selftest_r2s_mercy_form(uint64_t n_bases, uint64_t max_plane_words, uint64_t streamed_bytes, int32_t m,
                                           int need_mercy, uint64_t free_bytes, int force, uint64_t *planes_out,
                                           uint64_t *lists_out, int *sparse_out) {
  const MercyForm f = mercy_form(n_bases / 32 + 2, max_plane_words, (size_t)streamed_bytes, m, need_mercy && m > 1,
                                 (size_t)free_bytes, force);
  *planes_out = f.planes;
  *lists_out = f.lists;
  *sparse_out = f.sparse ? 1 : 0;
  return MHB_OK;
}

// Stage-1 Lv2Postprocess of one sorted bucket (wide layout) in the list form: the candidate bytes of the group walk,
// then every record's entries in record order (k_r2s_cand_write); *n_out = entries written (room for 2 n)
extern "C" int mhb_selftest_r2s_s1_cand(const uint32_t *recs, uint64_t n, uint32_t k, int32_t m, uint32_t fixed_len,
                                        uint64_t n_reads, uint32_t *is_solid, int64_t *counting, uint64_t *entries_out,
                                        uint64_t *n_out) {
  const uint32_t nw = r2s_s1_key_words(k), rw = nw + 2;
  PkgView pv;
  memset(&pv, 0, sizeof(pv));
  pv.fixed_len = fixed_len;
  pv.n_reads = n_reads;
  S1Out o{is_solid, nullptr, nullptr, nullptr};
  std::vector<uint8_t> cand(n, 0xFF);
  for (u64 g = 0; g < n;) {
    u32 hv[16], nh;
    g = s1_group(recs, nullptr, n, g, rw, nw, k, m, pv, o, true, hv, nh, cand.data());
    for (u32 q = 0; q < nh; ++q) counting[hv[q] > MHB_MAX_MUL ? MHB_MAX_MUL : hv[q]]++;
  }
  uint64_t at = 0;
  for (u64 i = 0; i < n; ++i) {
    if (cand[i] == 0xFF) return mhb_set_error(MHB_ERR_CUDA, "record %llu got no candidate byte", (unsigned long long)i);
    at += cand_entries(cand[i], s1_info(recs + i * rw, nw, nullptr), entries_out + at);
  }
  *n_out = at;
  return MHB_OK;
}

// The mercy step over a library in chunks, as mercy_count_pass runs it.  Library: fixed_len, or the n_reads lengths
// len[] (a zero-length read as one base), its first base at global base0.  is_solid and mercy: bit planes on the word
// grid from word base0 / 32.  List form (entries != nullptr): n_rounds lists back to back, round t ends at
// round_end[t], each sorted; per chunk [chunk_first[i], chunk_first[i + 1]) the slice of every list in its base range is
// scattered into chunk-sized candidate planes, and the reads of the chunk run r2s_mercy_read on them.  Plane form
// (entries == nullptr): planes holds no_in, no_out, any, each n_plane_words words on the same grid as is_solid.
extern "C" int mhb_selftest_r2s_mercy_lists(uint32_t fixed_len, uint64_t n_reads, const uint32_t *len, uint64_t base0,
                                            uint32_t k, const uint32_t *is_solid, const uint64_t *entries,
                                            const uint64_t *round_end, uint32_t n_rounds, const uint64_t *chunk_first,
                                            uint32_t n_chunks, const uint32_t *planes, uint64_t n_plane_words,
                                            uint32_t *mercy, uint64_t *added_out) {
  PkgView pv;
  memset(&pv, 0, sizeof(pv));
  pv.fixed_len = fixed_len;
  pv.n_reads = n_reads;
  pv.base0 = base0;
  std::vector<uint64_t> base_off(n_reads + 1, 0);
  if (!fixed_len) {
    for (uint64_t r = 0; r < n_reads; ++r) base_off[r + 1] = base_off[r] + std::max<uint32_t>(len[r], 1);
    pv.len = len;
    pv.base_off = base_off.data();
  }
  const uint64_t g0 = base0 / 32;  // the callers' planes start at this word
  S1Out o{const_cast<u32 *>(is_solid) - g0, nullptr, nullptr, nullptr};
  u32 *const mer = mercy - g0;
  *added_out = 0;
  if (!entries) {
    o.no_in = const_cast<u32 *>(planes) - g0;
    o.no_out = o.no_in + n_plane_words;
    o.any = o.no_out + n_plane_words;
    for (uint64_t r = 0; r < n_reads; ++r) *added_out += r2s_mercy_read(pv, r, k, o, mer);
    return MHB_OK;
  }
  CandLists lists;
  for (uint32_t t = 0; t < n_rounds; ++t)
    lists.rounds.emplace_back(entries + (t ? round_end[t - 1] : 0), entries + round_end[t]);
  for (uint32_t i = 0; i < n_chunks; ++i) {
    const uint64_t f = chunk_first[i], e = chunk_first[i + 1];
    if (f > e || e > n_reads) return mhb_set_error(MHB_ERR_ARG, "bad chunk bounds");
    if (f == e) continue;
    const uint64_t b0 = pv.base(f), b1 = pv.base(e);  // base_off has n_reads + 1 entries
    const uint64_t w0 = b0 / 32, nw = b1 / 32 + 2 - w0;
    std::vector<u32> cp(3 * nw, 0);
    S1Out c = o;
    c.no_in = cp.data() - w0;
    c.no_out = cp.data() + nw - w0;
    c.any = cp.data() + 2 * nw - w0;
    CKR(lists.each_slice(b0, b1, [&](const uint64_t *s, uint64_t n) -> int {
      for (uint64_t q = 0; q < n; ++q) cand_mark(c, s[q]);
      return MHB_OK;
    }));
    for (uint64_t r = f; r < e; ++r) *added_out += r2s_mercy_read(pv, r, k, c, mer);
  }
  return MHB_OK;
}
