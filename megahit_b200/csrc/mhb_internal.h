// mhb_internal.h -- declarations shared by the translation units of libmhb (not part of the C ABI).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <sys/time.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "mhb.h"

int mhb_set_error(int code, const char *fmt, ...);

// an INFO line on stderr, in the reference's log format
#define XINFO(...)                                                    \
  do {                                                                \
    fprintf(stderr, "INFO  %-30s: %4d - ", "megahit_b200", __LINE__); \
    fprintf(stderr, __VA_ARGS__);                                     \
  } while (0)

// wall-clock seconds, for the "Time elapsed" lines
inline double now_s() {
  timeval tv;
  gettimeofday(&tv, nullptr);
  return tv.tv_sec + tv.tv_usec * 1e-6;
}

// ---- host helpers of every stage (device-side ones, which need CUDA types: mhb_common.cuh) ----
// return a non-zero status code at once
#define CKR(call)        \
  do {                   \
    int rc_ = (call);    \
    if (rc_) return rc_; \
  } while (0)

// the 256-byte alignment of every device sub-allocation
inline size_t pad256(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// free memory of the current device; 0 when cudaMemGetInfo fails (the error is cleared) (mhb_stream.cu)
size_t free_device_bytes();

// One device allocation, released with the object (mhb_stream.cu).  alloc rounds max(bytes, 1) up to 256 and
// reallocates; ensure only grows, and contents do not survive growth.  A failed cudaMalloc clears the CUDA error and is
// MHB_ERR_NOMEM, its message "<what>: cudaMalloc of <bytes> bytes failed" (what starts with the stage).  The process
// counts the bytes all its DevBufs hold: peak_bytes() is the most they have held since the last reset_peak().
struct DevBuf {
  void *p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { release(); }
  int alloc(size_t b, const char *what);
  int ensure(size_t b, const char *what) { return p && bytes >= b ? MHB_OK : alloc(b, what); }
  void release();
  void swap(DevBuf &o) {
    std::swap(p, o.p);
    std::swap(bytes, o.bytes);
  }
  template <class T>
  T *as() const { return reinterpret_cast<T *>(p); }
  static void reset_peak();
  static size_t peak_bytes();
};

// largest n <= n_max with fixed + bytes(n) <= avail (bytes(n) grows with n); 0 when not even one fits
template <class F>
uint64_t largest_round(uint64_t n_max, size_t fixed, size_t avail, F bytes) {
  if (fixed + bytes(1) > avail) return 0;
  uint64_t lo = 1, hi = std::max<uint64_t>(n_max, 1);
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo + 1) / 2;
    if (fixed + bytes(mid) <= avail) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// ---- the count stage (mhb_host.cu), shared by the single-GPU rounds and the owners of a multi-GPU count ----
// Its work area for n records: either the LSD sort on every key byte followed by the run-length count, or - 8-byte
// records, the default where available - two partition passes + per-bucket hash aggregation (mhb_count_solid_hashed).
// MHB_COUNT_MODE=sort forces the former.
struct CountWork {
  bool hashed;
  size_t bytes;      // one work area: sort workspace + count scratch, or the hashed path's workspace
  size_t ws_bytes;   // sort path: size of the leading sort workspace
  int hist_byte;     // record byte whose histogram the extraction must deliver
};
CountWork count_work_plan(uint64_t n, uint32_t k, int32_t m);
// The count stage on the n records in d_a (d_b: a buffer of the same size; both clobbered): solid edges and flags into
// d_edges / d_aux (cap_edges), the multiplicity histogram added to d_mul_hist, the number of solid edges to *d_nsolid.
// d_hist0: the histogram of record byte cw.hist_byte, or NULL.  pass_ms / n_passes (may be NULL): per-pass timings.
int run_count_stage(void *stream, const CountWork &cw, uint32_t *d_a, uint32_t *d_b, uint64_t n, uint32_t k, int32_t m,
                    const uint64_t *d_hist0, uint32_t *d_edges, uint8_t *d_aux, uint64_t cap_edges, uint64_t *d_mul_hist,
                    uint64_t *d_nsolid, char *work, double *pass_ms, uint32_t *n_passes);
// bytes of device memory one count round of n records needs: two record buffers, the work area, edges and flags
size_t round_bytes(uint64_t n, uint32_t WR, uint32_t WE, int32_t m, uint32_t k);
// the cap on the records of one count round (mhb_set_round_limit), 0 = none
uint64_t count_round_limit();

// mhb_sort_records + optional per-pass timings (host array of n_bytes doubles, ms; forces a stream sync)
int mhb_sort_records_impl(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                          uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                          double *pass_ms_host);
// relaxed: as mhb_sort_records_relaxed (1) or mhb_sort_records (0), + per-pass timings as above
int mhb_sort_records_ex(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                        uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                        double *pass_ms_host, int relaxed);
// mhb_sort_records_relaxed without an entry in the per-pass timing ring (a sort inside another sort)
int mhb_sort_records_untraced(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                              uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b);

// bytes held by the arena the host-level calls keep between calls (mhb_release frees it)
size_t mhb_arena_bytes(void);

// The host-side index of a `.bin` image (sequence_package.h:224-240), mhb_stream.cu.  A fixed-length library needs no
// side arrays; otherwise rec_off[r] = first word of read r and unit_off[r] = sum over the reads before r of
// max(0, L - k): edge offsets for the count stage's k, base offsets for k = 0.  Both have n_reads + 1 entries.
struct ReadLibIndex {
  uint32_t fixed_len = 0;
  std::vector<uint64_t> rec_off, unit_off;
  uint64_t n_units = 0;  // sum of max(0, L - k) over all reads
  // the first word of read r (its length word); r = n_reads: the end of the image (0 for an empty library, which
  // index_read_lib leaves without offsets)
  uint64_t word_of(uint64_t r) const {
    return fixed_len ? r * (1 + (fixed_len + 15) / 16) : rec_off.empty() ? 0 : rec_off[r];
  }
};
// How index_read_lib checks a library whose size matches n_reads x (1 + ceil(L0/16)) for fixed-length reads:
// - kFull: every length word, on all host threads;
// - kSerial: every length word on the calling thread, for a process that forks workers afterwards (GNU OpenMP's
//   thread pool does not survive fork(): the first parallel region of a child would wait for the parent's threads);
// - kSampled: ~2048 of its length words only; the caller must then verify ALL of them on the device
//   (mhb_check_fixed_len) and come back with kFull when that fails.  (The full host scan touches every cache line of
//   the image: ~10 ms for 10 M reads, all of it inside the end-to-end time of the fused build.)
enum class FixedCheck { kFull, kSerial, kSampled };
int index_read_lib(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t k, ReadLibIndex *ix,
                   FixedCheck check = FixedCheck::kFull);
// A read library from disk (mhb_files.cpp): the counts of `prefix.lib_info` and the image of `prefix.bin`
int load_read_lib(const std::string &prefix, std::vector<uint32_t> *bin, long long *n_reads, long long *total_bases);

// ---- the reference's output formats (mhb_files.cpp), each written in one place for the single- and multi-GPU paths;
// a file that cannot be written is MHB_ERR_IO ----
// n raw bytes: `.sdbg.<i>`, `.edges.<i>`, `.cand`
int write_bytes(const std::string &path, const void *data, size_t n);
// P.sdbg_info (sdbg_meta.cpp:44-61).  tables: one 65536 x {byte offset, items, tips, large_mul} bucket table per
// `.sdbg.<i>` file, in file order.  Rows of the used buckets, files in order and buckets ascending, then unused rows.
int write_sdbg_info(const std::string &prefix, uint32_t k, uint32_t words_per_tip_label, int num_files,
                    const std::vector<const uint64_t *> &tables);
// P.edges.info of sorted edges (edge_io_meta.h:25-44).  counts: one 65536-bin bucket histogram per `.edges.<i>` file,
// whose edges are in bucket order; offsets run per file, and a bucket with edges in two files is MHB_ERR_ARG.
int write_edges_info(const std::string &prefix, uint32_t k, uint32_t words_per_edge,
                     const std::vector<std::vector<int64_t>> &counts);
// P.counting (edge_counter.h:44-52): multiplicities 1 .. MHB_MAX_MUL of hist
int write_counting(const std::string &prefix, const int64_t *hist);
// one read of a `.bin` image, given at its length word, appended to a `.cand` image in the reversed orientation
// KmerCounter holds candidate reads in (kmer_counter.cpp:387-401; sequence_package.h:284-295: reverse, no complement)
void append_cand_reversed(const uint32_t *read, std::vector<uint32_t> *out);
// the closing lines of the reference's seq2sdbg / read2sdbg, from the emitter's totals (SdbgStitch::tot layout)
void log_sdbg_summary(const uint64_t tot[16]);

// Streaming statistics of one host-level call: chunks (0 = resident), passes, bytes host to device, and the copy-engine
// and compute-stream busy time, host fill time and wall time of the passes (ms).
struct StreamStats {
  uint64_t chunks = 0, passes = 0, h2d_bytes = 0;
  double copy_ms = 0, kernel_ms = 0, fill_ms = 0, pass_ms = 0;
};

// ---- the plans (mhb_plan.cpp): host logic only; every greedy cut is the one rule of greedy_cut there ----
constexpr int kMaxRanks = 16;  // GPUs of one multi-GPU run
// the sort items of a sequence of len bases at k
inline uint64_t seq_items(uint32_t len, uint32_t k) { return len >= k + 1 ? 2ull * (len - k + 2) : 0; }
// the 256 leading-byte bins of a 65536-bin bucket histogram
inline void fold_bucket_hist(const uint64_t *h16, uint64_t *h256) {
  for (int b = 0; b < 256; ++b) h256[b] = 0;
  for (int b = 0; b < 65536; ++b) h256[b >> 8] += h16[b];
}
// Owner o takes the leading bytes [bounds[o], bounds[o+1]) (owner[b] = o): bound r is the byte whose cumulative count
// in total256 is closest to r/world of the total, leaving at least one byte for every later rank (k_plan_partition).
void owner_bounds(const uint64_t *total256, int world, uint32_t *bounds, uint8_t *owner);
using BucketRanges = std::vector<std::pair<uint32_t, uint32_t>>;  // [lo, hi] of 16-bit bucket ids, ascending
// Ranges tiling the leading bytes [byte_lo, byte_hi), of at most cap records each (cf. Lv1FindEndBuckets,
// base_engine.cpp:254-281): a byte is one atom of h256[b] records when that fits cap, else its buckets are atoms of
// h16[b << 8 | c] (h16 NULL: the byte stays one atom).  MHB_ERR_NOMEM naming the byte or bucket that alone exceeds cap
// (and rank >= 0, the owner), or when more than cap_out ranges are needed; *ranges then holds those closed before.
int plan_bucket_rounds(const uint64_t *h256, const uint64_t *h16, uint32_t byte_lo, uint32_t byte_hi, uint64_t cap,
                       uint32_t cap_out, int rank, BucketRanges *ranges);
// the rounds of a stage over all bucket ids from its 65536-bin histogram
int plan_stage_rounds(const uint64_t *h16, uint64_t cap, BucketRanges *ranges);
// The same from two histogram passes: top(h256) stores the leading-byte histogram; sub(bytes, h16), called when some
// bytes alone exceed cap, the second-byte histogram of each listed byte b in h16[b << 8 | c].  *pre: prefix sums of
// that histogram with every other byte's count in its first bucket, so the records of a range [lo, hi] are
// pre[hi + 1] - pre[lo].  MHB_OK, a pass's error, or -1 (MHB_ERR_NOMEM message set) when the plan fails.
int plan_bucket_passes(uint64_t cap, const std::function<int(uint64_t *)> &top,
                       const std::function<int(const std::vector<uint32_t> &, uint64_t *)> &sub, BucketRanges *ranges,
                       std::vector<uint64_t> *pre);
// The plan of every multi-GPU owner exchange (mhb_plan_count_owner_rounds), from every rank's 65536-bin histogram
// h16[s] and the most records owner o takes in one round, cap[o] (UINT64_MAX: no cap, one round).  A stage that
// histograms 256 leading bytes places byte b at bucket b << 8.
struct OwnerPlan {
  int world = 0;
  uint32_t bounds[kMaxRanks + 1];
  uint8_t owner[256];
  int R = 1;                       // rounds
  std::vector<uint32_t> lo, hi;    // [R][world]: owner o's bucket range in round t (lo > hi: empty)
  std::vector<uint64_t> n, off;    // [R][world owner][world rank]: records rank s sends to o in round t, and where
                                   // they start in o's receive buffer
  size_t at(int t, int o, int s) const { return ((size_t)t * world + o) * world + s; }
};
int plan_owner_rounds(const uint64_t *const *h16, int world, const uint64_t *cap, OwnerPlan *p);
// Greedy cut of n items into contiguous chunks [first[i], first[i+1]) of at most max_bytes each; a larger item gets a
// chunk of its own.  Item r takes 4 * (word_off[r+1] - word_off[r]) + extra_bytes, or with word_off == NULL
// 4 * stride_words + extra_bytes, cut in closed form.  first gets n_chunks + 1 entries ({0} when n == 0).
void plan_chunks(const uint64_t *word_off, uint64_t stride_words, uint64_t extra_bytes, uint64_t n, uint64_t max_bytes,
                 std::vector<uint64_t> *first);
// first edge of every leading byte in a sorted edge array (start[256] = n_edges)
void edge_byte_starts(const uint32_t *edges, uint64_t n_edges, uint32_t WE, uint64_t start[257]);
// Leading-byte segments [first[i], first[i+1]) of a streamed mercy search, packed to target bytes of edges; a byte above
// target is a segment of its own, one above limit (a device slot) MHB_ERR_NOMEM.
int plan_mercy_segments(const uint64_t start[257], uint32_t WE, uint64_t target, uint64_t limit, std::vector<uint32_t> *first);
// n_ranks contiguous shares (n_ranks + 1 entries) of the sequences balanced on their items, of the reads on their bases
void plan_seq_shares(const uint32_t *len, uint64_t n, uint32_t k, uint32_t n_ranks, uint64_t *first);
void plan_read_shares(const uint32_t *bin, const ReadLibIndex &ix, uint64_t n_reads, uint32_t n_ranks, uint64_t *first);

// The uploads of data kept in host memory, chunk by chunk, through two device slots (mhb_stream.cu): two pinned staging
// buffers, a non-blocking copy stream and four events per chunk.  While host threads fill the staging buffer of chunk
// i+1, chunk i uploads on the copy stream and the compute stream works on chunk i-1.  Each chunk's bytes land at the
// same offsets of its device slot as fill put them in the staging buffer.
class ChunkStager {
 public:
  struct Copies {  // the ranges of the staging buffer fill wrote, uploaded in this order
    size_t off[6], bytes[6];
    int n = 0;
    void add(size_t o, size_t b) {
      if (b) {
        off[n] = o;
        bytes[n++] = b;
      }
    }
  };
  using Fill = std::function<int(uint64_t chunk, char *host, Copies *up)>;  // host threads, off the compute stream
  using Run = std::function<int(uint64_t chunk, const char *slot)>;       // on the compute stream
  ChunkStager() = default;
  ChunkStager(const ChunkStager &) = delete;
  ChunkStager &operator=(const ChunkStager &) = delete;
  ~ChunkStager();
  // n_chunks chunks of at most slot_bytes; the passes are counted into *stats.  slot_bytes = 0: no staging (upload)
  int init(size_t slot_bytes, uint64_t n_chunks, StreamStats *stats);
  size_t device_bytes() const { return 2 * slot_bytes_; }
  void bind(char *device) { dev_ = device; }  // device_bytes() bytes, 256-byte aligned
  // one pass: every chunk filled, uploaded and handed to run, in order
  int pass(void *stream, const Fill &fill, const Run &run);
  // One pass over n_chunks pieces of host memory that need no staging: piece i, bytes [off[i], off[i+1]) of host, is
  // copied to the same offsets of the bound device memory on the copy stream, behind the work already queued on
  // `stream`, and run(i, its device address) is queued on `stream` behind that copy.  Counts nothing in the stats.
  int upload(void *stream, const char *host, const std::vector<size_t> &off, const Run &run);

 private:
  int stage(uint64_t i, const Fill &fill);
  size_t slot_bytes_ = 0;
  uint64_t n_chunks_ = 0;
  StreamStats *st_ = nullptr;
  char *dev_ = nullptr;
  char *host_[2] = {nullptr, nullptr};
  void *copy_ = nullptr;    // cudaStream_t
  std::vector<void *> ev_;  // cudaEvent_t: 4 per chunk (copy begin/end, compute begin/end)
};

// A chunk of a ChunkStream on the device: units [first, first + n) of the input, its image at offset 0 of the slot
// and each side array (offset arrays rebased to the chunk's first unit) after it; NULL where the input has none.
struct ChunkView {
  uint64_t index, first, n;
  const uint32_t *words;
  uint64_t n_words;
  const void *side[4];
  template <class T>
  const T *at(int j) const { return static_cast<const T *>(side[j]); }
};
// Every pass over an input held in host memory - a read library, a sequence set, sorted edges (mhb_stream.cu).  The
// input is an image of n units, unit i at words [word_of(i), word_of(i+1)), and up to four side arrays.  It is on the
// device in one of three forms:
// - resident: uploaded once by bind, and a pass hands it over whole as chunk 0;
// - resident in pieces: a fixed-stride image without side arrays goes up during the first pass in pieces, each
//   handed over as a chunk while the next one is still being copied;
// - streamed: it stays in host memory and goes through the two device slots of a ChunkStager in chunks that end on
//   unit boundaries.
// A slot holds the image, 16-byte aligned + 16 bytes for the read extraction's bulk copies, then each side array,
// 256-byte aligned.
class ChunkStream {
 public:
  struct Side {
    const void *host = nullptr;  // NULL: no such array
    uint32_t elem = 0;           // 0: n + 1 uint64 offsets, rebased to each chunk; else n elements of elem bytes
  };
  struct Input {
    const uint32_t *image = nullptr;
    uint64_t words = 0;                  // the whole image: what the resident form uploads and views
    uint64_t n = 0;                      // units
    const uint64_t *word_off = nullptr;  // n + 1 word offsets of the units, or NULL: unit i at i * stride
    uint64_t stride = 0;
    Side side[4];
    uint64_t word_of(uint64_t i) const { return !n ? 0 : word_off ? word_off[i] : i * stride; }
  };
  ChunkStream() = default;
  ChunkStream(const ChunkStream &) = delete;
  ChunkStream &operator=(const ChunkStream &) = delete;
  // first: the unit bounds of the streamed form's chunks, from the chunk planners; empty: resident.  in's arrays are
  // read by every pass and must outlive them.  pieces > 1: a resident fixed-stride image goes up in that many pieces of
  // a multiple of 4 units (16-byte aligned).  The chunks and passes are counted into *stats.
  int init(const Input &in, std::vector<uint64_t> first, StreamStats *stats, uint32_t pieces = 1);
  // the slot parts of an image of `words` words and of one side array of `units` units with elem-byte elements
  static size_t image_bytes(uint64_t words) { return pad256(((words * 4 + 15) & ~(uint64_t)15) + 16); }
  static size_t side_bytes(uint64_t units, uint32_t elem) { return pad256((units + 1) * (elem ? elem : 8)); }
  size_t device_bytes() const { return (resident_ ? 1 : 2) * slot_bytes_; }  // the input, or both chunk slots
  // device_bytes() bytes, 256-byte aligned; the resident form uploads the input there on `stream`
  int bind(void *device, void *stream);
  uint64_t n_chunks() const { return resident_ ? 0 : first_.size() - 1; }  // chunks of the stream, 0 when resident
  uint64_t max_chunk_units() const { return max_units_; }
  const std::vector<uint64_t> &bounds() const { return first_; }  // unit bounds of the views, {0, n} resident
  // one pass: fn runs once per chunk, in order, on the compute stream `stream`, while the chunk is on the device; the
  // resident form calls it once, with the whole input as chunk 0, and counts nothing in the stream statistics
  int pass(void *stream, const std::function<int(const ChunkView &)> &fn);

 private:
  int fill(uint64_t i, char *h, ChunkStager::Copies *up) const;
  ChunkView view(uint64_t i, const char *slot) const;
  Input in_;
  bool resident_ = true;
  std::vector<uint64_t> first_, pieces_;  // pieces_: unit bounds of the pieces still to upload
  uint64_t max_units_ = 0;
  size_t side_at_[4] = {0, 0, 0, 0}, slot_bytes_ = 0;
  char *dev_ = nullptr;
  ChunkStager stager_;
};
// A read library's stream: the `.bin` image and, for a variable-length library, side 0 = rec_off and side 1 = unit_off
// (when the index has it).  max_chunk_bytes = 0: resident, otherwise streamed in chunks that end on read boundaries;
// pieces as ChunkStream::init, for a fixed-length library.  The index must outlive the passes.
int init_read_stream(ChunkStream *rs, const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, const ReadLibIndex &ix,
                     uint64_t max_chunk_bytes, uint32_t pieces = 1);
// streaming statistics of the current host-level call (mhb_read_stream_stats)
void read_stream_stats_reset();
// the chunk cap: mhb_set_read_chunk_limit, or 0
uint64_t read_chunk_limit();
// the chunk size of a library that is streamed because it does not fit (no cap set)
uint64_t read_chunk_auto_bytes();
// the sequence chunk cap of seq2sdbg: mhb_set_s2s_chunk_limit, or 0 (mhb_host.cu)
uint64_t s2s_chunk_limit();

// host container mirroring what SeqPackage holds for seq2sdbg: word-aligned package-orientation sequences (mhb_files.cpp)
struct HostSeqs {
  std::vector<uint32_t> words;
  std::vector<uint64_t> word_off{0};
  std::vector<uint32_t> len;
  std::vector<uint16_t> mult;
  size_t size() const { return len.size(); }
  void append_packed(const uint32_t *w, uint32_t L, uint16_t m);  // already left-aligned, tail bits may be dirty
  void append_ascii(const char *s, uint32_t L, bool reverse, uint16_t m);  // sequence_package.h:245-273
};

// The parts of mhb_seq2sdbg_run that mhb_seq2sdbg_run_multi shares (mhb_files.cpp): the argument checks; whether a
// multi-GPU count has already built this graph (logs so, with the time since t0); and the loader of every input
// (edges, mercy edges with --need_mercy, contig / bubble / addi / local FASTA) into one sequence set.
int seq2sdbg_check_opts(const mhb_seq2sdbg_opts *o);
bool seq2sdbg_prebuilt(const mhb_seq2sdbg_opts *o, double t0);
int seq2sdbg_load(const mhb_seq2sdbg_opts *o, HostSeqs *seqs);

// The parts of mhb_iterate_run that mhb_iterate_run_multi shares (mhb_files.cpp): the option checks; the loader, checks
// included, of the contigs and bubbles (file orientation, standalone and loop contigs discarded) and of the `.bin`
// image (n_reads counted from its length words); and P.edges.info of n unordered edges of k_out = k + step.
int iterate_check_opts(const mhb_iterate_opts *o);
int iterate_load(const mhb_iterate_opts *o, HostSeqs *contigs, std::vector<uint32_t> *bin, uint64_t *n_reads);
int iterate_write_info(const std::string &prefix, uint32_t k_out, uint32_t words_per_edge, uint64_t n);

// ---- iterate's device pieces (mhb_iter.cu), shared by mhb_iterate_host and the multi-GPU worker ----
// the checks of mhb_iterate_host on k and step (main_iterate.cpp:73-93, and the 17-word records of the device sort)
int iterate_check_args(uint32_t k, uint32_t step);
// The flank index (FeedBatchContigs) of a's contigs on the current device: n unique records of ceil((k+1)/16) + 2
// words in tab, and its 65537-entry prefix table in lut.  Every caller gets the same table from the same contigs.
struct IterFlanks {
  DevBuf tab, lut;
  uint64_t n = 0;
};
int iter_build_flanks(const mhb_iterate_args *a, IterFlanks *f);
// The read pass (FindNextKmersFromReads) over a's reads against the flank index: resident, or streamed in chunks when a
// chunk cap is set or when the resident buffers do not fit.  *set = the n_set unique candidate edges, ascending, on the
// device (nothing allocated when there are none); n_cand = candidates before the dedup; n_aligned = reads with one.
int iter_collect(const mhb_iterate_args *a, const IterFlanks &f, DevBuf *set, uint64_t *n_set, uint64_t *n_cand,
                 uint64_t *n_aligned);
// KmerCollector's set semantics on n edge records of k + step in a (b: a buffer of the same size): sort, then the first
// record of every run of equal ones; *out = where the n_out unique records are (a or b)
int iter_sort_unique(uint32_t *a, uint32_t *b, uint64_t n, uint32_t k, uint32_t step, uint32_t **out, uint64_t *n_out);
// hist[v] += records among the n of `words` words whose byte `byte` (the sort's numbering) is v (mhb_sortdisp.cu)
int hist_byte(void *stream, const uint32_t *recs, uint64_t n, uint32_t words, int byte, uint64_t *hist);

// The two halves of mhb_read2sdbg_run, which mhb_read2sdbg_run_multi shares (mhb_files.cpp): the option checks, the
// library and the (empty) P.mercy_cand.<i> files; then the single-GPU build and its files and summary lines.
int read2sdbg_load(const mhb_read2sdbg_opts *o, std::vector<uint32_t> *bin, long long *n_reads);
int read2sdbg_build(const mhb_read2sdbg_opts *o, std::vector<uint32_t> &bin, long long n_reads, double t0);

// One round of a multi-GPU owner exchange on the device (OwnerExchange, mhb_mgpu.cpp); every pointer is device memory.
// owner[b]: the rank owning leading byte b.  Per owner o: base[o] = where this rank's block of o's receive buffer
// starts (256 entries, the rest 0: mhb_partition_scatter reads as many); row0[o] / info0[o] = row 0 of that buffer
// and of its read_info buffer (info0 nullptr unless read2sdbg's narrow stage 1); off[o] = the rows of the lower
// ranks' blocks; cap[o] = the rows of my block; cursor[o] = zeroed, the records the store counted; lo[o] .. hi[o] =
// o's bucket range in the round.  Device addresses are uint64_t.
struct OwnerRoute {
  int n_owners;
  const uint8_t *owner;
  const uint64_t *base, *row0, *info0, *off, *cap;
  uint64_t *cursor;
  const uint32_t *lo, *hi;
};

// ---- read2sdbg's device pieces (mhb_r2s.cu), driven step by step by the multi-GPU worker ----
// One rank's share [first, end) of the reads of a build, resident on the current device as one package chunk: read
// indices are local, bases - stage-1 payload positions and bit-plane indices - global, and the bit planes (solid; with
// need_mercy in the plane form the three candidate planes after it, in one allocation) cover the whole library's word
// grid.  Records
// reach their owners (ranks of contiguous leading-byte ranges) through an OwnerRoute, one round over ascending bucket
// sub-ranges at a time (rt.lo / rt.hi).
class R2sShare {
 public:
  R2sShare();
  ~R2sShare();
  R2sShare(const R2sShare &) = delete;
  R2sShare &operator=(const R2sShare &) = delete;
  // a: the whole library and the build's k, m, need_mercy; li: its index_read_lib (made before the fork)
  int load(const mhb_build_args *a, const ReadLibIndex &li, uint64_t first, uint64_t end);
  // The mercy candidates of a need_mercy build: planes of the whole library, or (list form, DESIGN.md §4.9) sorted
  // lists made by the owners of stage 1 and planes of the share only.  want_cand_lists: this rank's wish - the list
  // form is forced (mhb_set_r2s_sparse_mercy) or the four planes of the whole library exceed avail; every rank must
  // then bind the same form.  bind_planes allocates the planes of the form (after load, before stage 1).
  bool want_cand_lists(size_t avail) const;
  int bind_planes(bool lists);
  bool cand_lists() const;
  uint64_t base_of(uint64_t read) const;  // global base of a read of the library
  // list form: every stage-1 round's candidates this rank owned (sorted by position), after the last s1_own; then
  // cand_take hands over every owner's entries inside my share (any number of lists, each sorted), for mercy_count
  const std::vector<std::vector<uint64_t>> &cand_made() const;
  void cand_take(std::vector<std::vector<uint64_t>> *lists);
  uint32_t s1_record_words() const;  // words of a stage-1 record row
  bool s1_narrow() const;            // read_info in a side array of 8 bytes per row
  // The most stage-1 records / stage-2 items one owner takes in one round (at most n_total): the largest round whose
  // receive buffer and sort pass fit `avail` device bytes next to the stage's fixed arrays (stage 1: the per-read
  // arrays of n_owners owners), capped by mhb_set_r2s_round_limit and, stage 1, by the narrow layout's 2^32 rows.
  // 0 when not even one fits.
  uint64_t s1_round_budget(size_t avail, int n_owners, uint64_t n_total) const;
  uint64_t s2_round_budget(size_t avail, uint64_t n_total) const;
  // hist[65536] = the 16-bit bucket ids of the share's stage-1 records / stage-2 items (s2 after mercy_count)
  int s1_hist(uint64_t *hist);
  int s2_hist(uint64_t *hist);
  // the share's stage-1 records of one round to their owners in global read order, in two passes: s1_count puts the
  // records of every owner into rt.cursor, s1_store stores them at rt.row0 / rt.info0 from row rt.off (it has no
  // capacity: the caller checks the counts in between).  The per-read arrays between them are kept for the stage.
  int s1_count(const OwnerRoute &rt);
  int s1_store(const OwnerRoute &rt);
  // owner, once per round: stable bucket partition, kmsort and Lv2Postprocess of the n records received (overwritten),
  // into the local planes and multiplicity histogram.  Its buffers are sized for n_max, the largest round, and kept.
  int s1_own(uint32_t *recs, uint64_t *info, uint64_t n, uint64_t n_max);
  void s1_end();  // after the last round: the stage-1 round buffers go
  void *planes() const;  // the allocation of the planes, for CUDA IPC (nullptr when m == 1)
  // OR another rank's planes (same layout) into mine over my share's words
  int or_planes(const void *peer_planes);
  // the mercy step and the stage-2 item count over the share
  int mercy_count(uint64_t *n_items, uint64_t *n_mercy);
  // the share's stage-2 items of one round to their owners through rt (OwnerSink)
  int s2_send(const OwnerRoute &rt);
  // owner, once per round in ascending bucket order: relaxed sort, collapse and emitter (label_fmt 1) of the n items
  // received (overwritten), appended to the owner's output (SdbgStitch); buffers sized for n_max and kept
  int s2_own(uint32_t *items, uint64_t n, uint64_t n_max);
  // after the last round: SdBG bytes, bucket table (65536 x {offset, items, tips, large_mul}) and the emitter's 16
  // totals of every round; the round buffers go
  void s2_result(std::vector<uint8_t> *bytes, std::vector<uint64_t> *table, uint64_t *totals);
  int counting(uint64_t *hist);  // the multiplicity histogram (65536) of the records this rank owned
  uint64_t n_reads() const;

 private:
  struct Impl;
  Impl *d_;
};
// mhb_mercy_probe_owned, with accumulate = true OR-ing the answers into planes_out instead of storing them (mhb_multi.cu)
int mercy_probe_owned(void *stream, const mhb_dev_reads *reads, const uint64_t *cand_ids, uint64_t n_cand,
                      uint32_t max_read_len, uint32_t k, const uint32_t *edges, uint64_t n_edges, const void *lut,
                      const uint8_t *owner_of_byte, uint32_t me, uint32_t *planes_out, bool accumulate);

// The SdBG output of a build that runs its stage-2 sort in rounds over ascending bucket ranges: every round's emitter
// output (mhb_s2s_emit / mhb_s2s_emit_fmt) is appended to one byte stream, its non-empty rows of the bucket table are
// taken over with their byte offsets moved by the bytes before them, and the totals are summed.
struct SdbgStitch {
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> table = std::vector<uint64_t>((size_t)65536 * 4);  // {byte offset, items, tips, large_mul}
  uint64_t tot[16] = {0};  // the emitter's totals layout: [0] bytes [1] items [2] tips [3] large_mul [4..12] w [13] ones
  int append(void *stream, const uint8_t *d_bytes, uint64_t cap_bytes, const uint64_t *d_table, const uint64_t *d_totals);

 private:
  std::vector<uint64_t> round_table = std::vector<uint64_t>((size_t)65536 * 4);
};

// the emitter's totals (SdbgStitch::tot layout) into the counts of a result (mhb_build_result, mhb_s2s_result)
template <class R>
void set_sdbg_totals(R *res, const uint64_t tot[16]) {
  res->n_bytes = tot[0];
  res->n_items = tot[1];
  res->n_tips = tot[2];
  res->n_large_mul = tot[3];
  for (int i = 0; i < 9; ++i) res->w_count[i] = tot[4 + i];
  res->ones_in_last = tot[13];
}
// ... and back
template <class R>
void get_sdbg_totals(const R &res, uint64_t tot[16]) {
  std::fill(tot, tot + 16, 0);
  tot[0] = res.n_bytes;
  tot[1] = res.n_items;
  tot[2] = res.n_tips;
  tot[3] = res.n_large_mul;
  for (int i = 0; i < 9; ++i) tot[4 + i] = res.w_count[i];
  tot[13] = res.ones_in_last;
}
