// mhb_mgpu.cpp -- `count`, `seq2sdbg`, `iterate` and `read2sdbg` on several GPUs of one node behind the file-level
// C ABI (mhb_*_run_multi, include/mhb.h).
//
// One worker PROCESS per GPU (forked before CUDA is touched; libmhb keeps per-process state: arena, kernel attributes),
// with no Python, torch or NCCL underneath.  The parent loads the input and deals it in contiguous shares (reads
// balanced on bases, sequences on items); rank order is input order.  The count and seq2sdbg workers read their shares
// through a chunk stream: on the device when a share fits, otherwise streamed from the host copy they inherit.
//
// Every stage moves its records to their owners with one exchange (OwnerExchange):
//   1. every rank all-gathers its 65536-bin bucket histogram (a stage that histograms leading bytes puts byte b in
//      bucket b << 8);
//   2. every rank computes the same plan from them (plan_owner_rounds, mhb_plan.cpp): owner o takes the leading bytes
//      [bounds[o], bounds[o+1]), in rounds over ascending bucket sub-ranges when o has a per-round cap, and the plan's
//      blocks say how many records rank s sends to o in round t and where they start in o's receive buffer;
//   3. every rank allocates its receive buffer (its largest round) and opens every other rank's through CUDA IPC;
//   4. per round the route (OwnerRoute: owner of each byte, base address, rows and capacity per owner, cursors) goes to
//      the device, one launch stores every record straight into its owner's buffer, the cursors come back and are
//      checked against the plan's blocks, and a barrier hands the complete buffers to their owners.
// The small collectives (histograms, counters, IPC handles) are all-gathers of uint64 rows through one MAP_SHARED
// control block with a process-shared barrier; the medium ones (tip edges, candidate reads, answer planes of the mercy
// searches, per-bucket tables) go through files in /dev/shm written by one rank and read by the others.
//
// `count` (mhb_count_run_multi): the count records go to their owners in rounds, each owner counts what it received;
// the mercy searches are answered by the owners of the searched prefixes (mhb_mercy_probe_owned); the k_min SdBG is
// built in the same run because the solid and mercy edges are already on the devices.  Reference behaviour reproduced:
// KmerCounter::Run (sorting/kmer_counter.cpp) + SeqToSdbg::Run with need_mercy (sorting/seq_to_sdbg.cpp) at k_min;
// files as edge_io_meta.h:25-44 / sdbg_meta.cpp:44-61 with num_files = n_gpus.
// `seq2sdbg` for k > k_min (mhb_seq2sdbg_run_multi): the items go to their owners, which sort and emit as the count's
// SdBG stage does (sdbg_stage, sdbg_merge_info), in rounds over ascending bucket ranges when an owner's items do not
// fit its device at once (or exceed mhb_set_s2s_round_limit).
// `iterate` (mhb_iterate_run_multi): each rank builds the whole flank index, runs the single-GPU read pass over its share
// and sends its unique candidates to their owners, which sort and dedup them; the owners' ascending runs, written in
// rank order, are the single-GPU P.edges.0.
// `read2sdbg` (mhb_read2sdbg_run_multi): the stage-1 records reach their owners in global read order, the owners run
// stage 1 into planes of the whole library, every rank ORs all planes over its share's words, runs the mercy step over
// its share and sends its stage-2 items to their owners, which sort, collapse and emit as the single-GPU read2sdbg does.
// Where the candidate planes of the whole library do not fit, the owners make sorted candidate lists instead and every
// rank fetches the entries of its share into candidate planes of the share (cand_exchange).
// Both sort stages run in rounds over ascending bucket ranges when an owner's records do not fit its device at once
// (or exceed mhb_set_r2s_round_limit), as the count's records do.
#include <cuda_runtime.h>
#include <dirent.h>
#include <fcntl.h>
#include <pthread.h>
#include <signal.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <numeric>
#include <optional>
#include <string>
#include <vector>

#include "mhb.h"
#include "mhb_bits.cuh"
#include "mhb_internal.h"

using namespace mhb;

namespace {

// control block shared by the workers (anonymous MAP_SHARED mapping created before the fork, zero-filled)
struct Control {
  pthread_barrier_t bar;
  char err[kMaxRanks][512];
  int err_code[kMaxRanks];                // MHB_ERR_* of a failed rank
  uint64_t rows[2][kMaxRanks][65536];     // Exchange::gather, alternately
};

struct Fail {
  std::string msg;
  int code;
};
[[noreturn]] void vfail(int code, const char *fmt, va_list ap) {
  char buf[480];
  vsnprintf(buf, sizeof(buf), fmt, ap);
  throw Fail{buf, code};
}
[[noreturn]] void fail(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfail(MHB_ERR_CUDA, fmt, ap);
}
[[noreturn]] void fail_nomem(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfail(MHB_ERR_NOMEM, fmt, ap);
}
#define CKC(call)                                                                            \
  do {                                                                                       \
    cudaError_t e_ = (call);                                                                 \
    if (e_ != cudaSuccess) fail("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); \
  } while (0)
// a libmhb call, or a helper in its convention (a DevBuf allocation, a file writer): its failure with its own code
#define CKL(call)                                              \
  do {                                                         \
    if (int rc_ = (call)) throw Fail{mhb_last_error(), rc_};   \
  } while (0)

// rank r runs on device r % device_count.  With more ranks than devices, ranks share a device: CUDA IPC between two
// processes on one device is legal, and the exchange's stores to a peer on the same device stay in local HBM.
void bind_device(int rank, int world) {
  int n_dev = 0;
  CKC(cudaGetDeviceCount(&n_dev));
  if (n_dev < 1) fail("no CUDA device");
  const int dev = rank % n_dev;
  if (world > n_dev) {
    int mode = cudaComputeModeDefault;
    CKC(cudaDeviceGetAttribute(&mode, cudaDevAttrComputeMode, dev));
    if (mode == cudaComputeModeExclusiveProcess || mode == cudaComputeModeProhibited)
      fail("%d ranks on %d device(s) share device %d, but its compute mode (%s) admits only one process: use at most %d GPUs",
           world, n_dev, dev, mode == cudaComputeModeProhibited ? "prohibited" : "exclusive process", n_dev);
    if (rank == 0) XINFO("%d ranks on %d device(s): rank r runs on device r %% %d\n", world, n_dev, n_dev);
  }
  CKC(cudaSetDevice(dev));
  CKL(mhb_set_device(dev));
}

// ---- what the ranks share on the host: a barrier, all-gathers of uint64 rows, and files in /dev/shm (rank r writes
// <base>.<tag>.<r>, the others read it; run_workers removes them) ----
struct Exchange {
  std::string base;
  int rank, world;
  Control *C;
  int n_gathers = 0;
  void barrier() { pthread_barrier_wait(&C->bar); }
  // every rank's n values (n <= 65536), rank after rank.  The two row sets alternate: a rank writes one only after
  // every rank has entered the gather that used the other, so every rank has copied what it read there.
  std::vector<uint64_t> gather(const uint64_t *mine, size_t n) {
    uint64_t(*rows)[65536] = C->rows[n_gathers++ & 1];
    memcpy(rows[rank], mine, n * 8);
    barrier();
    std::vector<uint64_t> all((size_t)world * n);
    for (int o = 0; o < world; ++o) memcpy(&all[(size_t)o * n], rows[o], n * 8);
    return all;
  }
  std::string path(const char *tag, int r) const { return base + "." + tag + "." + std::to_string(r); }
  void publish(const char *tag, const void *data, size_t bytes) { CKL(write_bytes(path(tag, rank), data, bytes)); }
  // whole file of rank r, or the byte range [off, off + bytes)
  std::vector<char> fetch(const char *tag, int r, size_t off = 0, size_t bytes = (size_t)-1) {
    FILE *f = fopen(path(tag, r).c_str(), "rb");
    if (!f) fail("cannot open %s", path(tag, r).c_str());
    if (bytes == (size_t)-1) {
      fseek(f, 0, SEEK_END);
      bytes = (size_t)ftell(f) - off;
    }
    fseek(f, (long)off, SEEK_SET);
    std::vector<char> v(bytes);
    if (bytes && fread(v.data(), 1, bytes, f) != bytes) {
      fclose(f);
      fail("short read on %s", path(tag, r).c_str());
    }
    fclose(f);
    return v;
  }
};

// ---- the owner exchange of a stage (the steps of the header comment) ----
struct OwnerExchange {
  // the route of one round as uploaded; OwnerRoute points into its device copy
  struct Route {
    uint64_t base[256], row0[kMaxRanks], info0[kMaxRanks], off[kMaxRanks], cap[kMaxRanks], cursor[kMaxRanks];
    uint32_t lo[kMaxRanks], hi[kMaxRanks];
    uint8_t owner[256];
  };
  std::vector<uint64_t> hist;  // [world][65536]: every rank's bucket histogram
  OwnerPlan plan;
  std::vector<uint64_t> own;         // the records I receive in each round
  uint64_t n_own = 0, n_sent = 0;    // ... and over all rounds, and the records I send
  uint32_t row_bytes = 0;
  DevBuf mine, info;                 // my receive buffer, and its read_info rows (read2sdbg's narrow stage 1)
  void *peer[2][kMaxRanks] = {};     // every rank's receive buffer [0] and read_info buffer [1]
  DevBuf dev;                        // the Route on the device
  OwnerRoute rt;

  // 1: my histogram of 65536 buckets, or of 256 leading bytes (byte b -> bucket b << 8)
  void gather(Exchange &X, const uint64_t *h, int bins) {
    std::vector<uint64_t> h16(65536, 0);
    for (int b = 0; b < bins; ++b) h16[bins == 256 ? b << 8 : b] = h[b];
    hist = X.gather(h16.data(), 65536);
  }

  // 2 + 3: the plan (cap[o]: the most records owner o takes in one round; nullptr: one round), a receive buffer of
  // rows of row_bytes (+ read_info rows of 8 bytes when info_what names them) opened by every rank, and the device route
  void open(Exchange &X, const uint64_t *cap, uint32_t row_bytes_, const char *what, const char *info_what = nullptr) {
    const int W = X.world, r = X.rank;
    std::vector<const uint64_t *> h(W);
    uint64_t no_cap[kMaxRanks];
    for (int s = 0; s < W; ++s) {
      h[s] = &hist[(size_t)s * 65536];
      no_cap[s] = ~0ull;
    }
    CKL(plan_owner_rounds(h.data(), W, cap ? cap : no_cap, &plan));
    own.assign(plan.R, 0);
    for (int t = 0; t < plan.R; ++t)
      for (int s = 0; s < W; ++s) {
        own[t] += plan.n[plan.at(t, r, s)];
        n_sent += plan.n[plan.at(t, s, r)];
      }
    for (uint64_t n : own) n_own += n;
    const uint64_t rows = *std::max_element(own.begin(), own.end());
    row_bytes = row_bytes_;
    CKL(mine.alloc(rows * row_bytes + 256, what));
    if (info_what) CKL(info.alloc(rows * 8 + 256, info_what));
    uint64_t handles[2][8];
    CKL(mhb_ipc_export(mine.p, (uint8_t *)handles[0]));
    if (info_what) CKL(mhb_ipc_export(info.p, (uint8_t *)handles[1]));
    const int nb = info_what ? 2 : 1;
    const std::vector<uint64_t> all = X.gather(&handles[0][0], 8 * nb);
    for (int o = 0; o < W; ++o)
      for (int i = 0; i < nb; ++i) {
        if (o == r) peer[i][o] = i ? info.p : mine.p;
        else CKL(mhb_ipc_open((const uint8_t *)&all[(size_t)o * 8 * nb + 8 * i], &peer[i][o]));
      }
    CKL(dev.alloc(sizeof(Route), "exchange: route"));
    const Route *d = dev.as<Route>();
    rt = {W, d->owner, d->base, d->row0, info_what ? d->info0 : nullptr, d->off, d->cap, (uint64_t *)d->cursor, d->lo, d->hi};
  }

  // 4: round t.  store(rt) launches the stores; what names the records in the check, nullptr for a store that counts
  // nothing (mhb_partition_scatter places the records from the histogram).
  template <class Store>
  void send(Exchange &X, int t, const char *what, Store store) {
    Route h;
    memset(&h, 0, sizeof(h));
    for (int o = 0; o < X.world; ++o) {
      const size_t i = plan.at(t, o, X.rank);
      h.row0[o] = (uint64_t)(uintptr_t)peer[0][o];
      h.info0[o] = (uint64_t)(uintptr_t)peer[1][o];
      h.off[o] = plan.off[i];
      h.cap[o] = plan.n[i];
      h.base[o] = h.row0[o] + plan.off[i] * row_bytes;
      h.lo[o] = plan.lo[(size_t)t * X.world + o];
      h.hi[o] = plan.hi[(size_t)t * X.world + o];
    }
    memcpy(h.owner, plan.owner, 256);
    CKC(cudaMemcpy(dev.p, &h, sizeof(h), cudaMemcpyHostToDevice));
    store(rt);
    check(X, t, what);
    if (t + 1 == plan.R) dev.release();  // no stores after the last round
    X.barrier();  // every rank's stores of the round have completed: my receive buffer is complete
  }

  // every owner got exactly the records of my block in round t (what == nullptr: only wait for the stores)
  void check(const Exchange &X, int t, const char *what) {
    uint64_t sent[kMaxRanks];
    CKC(cudaMemcpy(sent, rt.cursor, X.world * 8, cudaMemcpyDeviceToHost));
    for (int o = 0; what && o < X.world; ++o) {
      const uint64_t want = plan.n[plan.at(t, o, X.rank)];
      if (sent[o] != want)
        fail("internal: %llu %s for rank %d, the histogram said %llu", (unsigned long long)sent[o], what, o,
             (unsigned long long)want);
    }
  }

  void close(Exchange &X) {
    X.barrier();  // nobody reads or writes the buffers any more
    for (int i = 0; i < 2; ++i)
      for (int o = 0; o < X.world; ++o)
        if (o != X.rank && peer[i][o]) mhb_ipc_close(peer[i][o]);
    X.barrier();
    mine.release();
    info.release();
  }
};

// ---- the owner side of the SdBG stage, the same in the count and seq2sdbg workers ----
// My P.sdbg.<r>, and for rank 0 my bucket table and totals ("stab": 65536 x 4 + 16 words)
void sdbg_publish(Exchange &X, const uint64_t *totals, const std::vector<uint8_t> &sdbg_bytes,
                  std::vector<uint64_t> table, const std::string &prefix) {
  CKL(write_bytes(prefix + ".sdbg." + std::to_string(X.rank), sdbg_bytes.data(), sdbg_bytes.size()));
  table.insert(table.end(), totals, totals + 16);
  X.publish("stab", table.data(), table.size() * 8);
}

// This rank's part of its device's free memory for the rounds of a stage: 92 % of it, split evenly among the ranks
// bound to the device.  Called by every rank between two barriers, when nobody allocates.
size_t rank_round_bytes(int rank, int world) {
  int n_dev = 1, sharers = 0;
  CKC(cudaGetDeviceCount(&n_dev));
  for (int q = 0; q < world; ++q) sharers += q % n_dev == rank % n_dev;
  return (size_t)(0.92 * (double)free_device_bytes()) / (size_t)std::max(1, sharers);
}

// An XINFO line in one write: the lines of ranks that log at the same time stay whole
#define RANK_INFO(...) rank_info(__LINE__, __VA_ARGS__)
void rank_info(int line, const char *fmt, ...) {
  char buf[1024];
  int n = snprintf(buf, sizeof(buf), "INFO  %-30s: %4d - ", "megahit_b200", line);
  va_list ap;
  va_start(ap, fmt);
  n += vsnprintf(buf + n, sizeof(buf) - n, fmt, ap);
  va_end(ap);
  fflush(stderr);
  if (write(2, buf, std::min<size_t>((size_t)n, sizeof(buf) - 1)) < 0) return;
}

// How a rank's share went through its device, for its log line: "resident", or "in <c> chunks, <p> passes in <t> ms"
std::string share_form(const StreamStats &st) {
  if (!st.chunks) return "resident";
  char buf[96];
  snprintf(buf, sizeof(buf), "in %llu chunks, %llu passes in %.1f ms", (unsigned long long)st.chunks,
           (unsigned long long)st.passes, st.pass_ms);
  return buf;
}

// Rank 0: the loads of a stage's plan - the records of the largest owner, leading byte and bucket - from which a
// round cap can be chosen, as "<label>: largest owner ..., largest leading byte ..., largest bucket ..."
void log_loads(const Exchange &X, const OwnerExchange &ex, const char *label) {
  if (X.rank) return;
  std::vector<uint64_t> tot(65536, 0);
  for (int s = 0; s < X.world; ++s)
    for (int b = 0; b < 65536; ++b) tot[b] += ex.hist[(size_t)s * 65536 + b];
  uint64_t owner = 0, byte = 0, bucket = 0;
  for (int o = 0; o < X.world; ++o) {
    uint64_t n = 0;
    for (uint32_t b = ex.plan.bounds[o] << 8; b < ex.plan.bounds[o + 1] << 8; ++b) n += tot[b];
    owner = std::max(owner, n);
  }
  for (int b = 0; b < 256; ++b) {
    uint64_t n = 0;
    for (int c = 0; c < 256; ++c) n += tot[b << 8 | c];
    byte = std::max(byte, n);
  }
  for (uint64_t n : tot) bucket = std::max(bucket, n);
  XINFO("%s: largest owner %llu, largest leading byte %llu, largest bucket %llu\n", label, (unsigned long long)owner,
        (unsigned long long)byte, (unsigned long long)bucket);
}

// The SdBG stage of the count and seq2sdbg workers, from this rank's 65536-bin bucket histogram of its items (h16).
// The plan caps every owner at its round budget (mhb_sdbg_round_budget, taken while nobody allocates); per round,
// store(rt) puts my items of the round's bucket ranges straight into their owners' buffers, and every owner sorts and
// emits what it received (mhb_s2s_sort_emit) and appends it to its output.  An owner's rounds ascend, so its
// P.sdbg.<r> is in bucket order.  Then the exchange closes and the result is published.  Returns the rounds.
template <class Store>
int sdbg_stage(Exchange &X, const uint64_t *h16, uint32_t k, const std::string &prefix, uint64_t *n_own, Store store) {
  const uint32_t W2 = mhb_s2s_record_words(k), wpt = div_ceil(k, 16);
  OwnerExchange ex;
  ex.gather(X, h16, 65536);  // ... behind which nobody allocates until the budgets are gathered
  uint64_t n_total = 0;
  for (uint64_t c : ex.hist) n_total += c;
  const size_t avail = rank_round_bytes(X.rank, X.world);
  const size_t fixed = (size_t)64 << 20;  // bucket table, totals, the exchange's small tables
  const uint64_t budget = mhb_sdbg_round_budget(avail, fixed, k, n_total);
  if (!budget) fail_nomem("%zu free bytes for this rank: not even a one-item SdBG round fits", avail);
  ex.open(X, X.gather(&budget, 1).data(), W2 * 4, "SdBG owner: items received");
  const int R = ex.plan.R;
  if (X.rank == 0) XINFO("SdBG plan: %d round%s over bucket ranges\n", R, R > 1 ? "s" : "");
  log_loads(X, ex, "SdBG items");
  *n_own = ex.n_own;

  SdbgStitch out;  // my rounds, in bucket order
  {
    const uint64_t n_max = *std::max_element(ex.own.begin(), ex.own.end());
    const uint64_t cap_b = n_max * (4ull + 4ull * wpt) + 16;
    const size_t ws_bytes = mhb_s2s_sort_emit_workspace_bytes(std::max<uint64_t>(n_max, 1), k);
    DevBuf tmp, ws, bytes, d_table, d_tot;
    CKL(tmp.alloc((n_max * W2 + 16) * 4, "SdBG owner: sort buffer"));
    CKL(ws.alloc(ws_bytes, "SdBG owner: sort and emit workspace"));
    CKL(bytes.alloc(cap_b, "SdBG owner: SdBG bytes"));
    CKL(d_table.alloc(65536 * 32, "SdBG owner: bucket table"));
    CKL(d_tot.alloc(128, "SdBG owner: totals"));
    for (int t = 0; t < R; ++t) {
      ex.send(X, t, "SdBG items", store);
      if (const uint64_t n_t = ex.own[t]) {
        CKL(mhb_s2s_sort_emit(nullptr, ex.mine.as<uint32_t>(), tmp.as<uint32_t>(), n_t, k, nullptr, bytes.as<uint8_t>(),
                              cap_b, d_table.as<uint64_t>(), d_tot.as<uint64_t>(), ws.p, ws_bytes));
        CKL(out.append(nullptr, bytes.as<uint8_t>(), cap_b, d_table.as<uint64_t>(), d_tot.as<uint64_t>()));
      }
      if (t + 1 < R) X.barrier();  // nobody stores into my receive buffer before I have sorted it
    }
  }
  ex.close(X);
  sdbg_publish(X, out.tot, out.bytes, std::move(out.table), prefix);
  return R;
}

// Rank 0, once every rank's sdbg_publish is behind a barrier: the merged P.sdbg_info, one file per rank, and the
// reference's closing lines of seq2sdbg.
void sdbg_merge_info(Exchange &X, uint32_t k, const std::string &prefix) {
  std::vector<std::vector<char>> stab(X.world);
  std::vector<const uint64_t *> tables(X.world);
  uint64_t tot[16] = {0};
  for (int o = 0; o < X.world; ++o) {
    stab[o] = X.fetch("stab", o);
    tables[o] = (const uint64_t *)stab[o].data();
    for (int i = 0; i < 16; ++i) tot[i] += tables[o][65536 * 4 + i];
  }
  CKL(write_sdbg_info(prefix, k, div_ceil(k, 16), X.world, tables));
  log_sdbg_summary(tot);
}

// Rank 0: the sum of every rank's 65536-bin multiplicity histogram ("mul"), for P.counting
std::vector<int64_t> sum_mul(Exchange &X) {
  std::vector<int64_t> mul(65536, 0);
  for (int o = 0; o < X.world; ++o) {
    const std::vector<char> v = X.fetch("mul", o);
    const int64_t *h = (const int64_t *)v.data();
    for (int i = 0; i < 65536; ++i) mul[i] += h[i];
  }
  return mul;
}

// ================================================================================================
// count on several GPUs: one rank = one GPU, its stages in order
// ================================================================================================
struct Job {
  uint32_t k;
  int32_t m;
  const uint32_t *bin;          // whole library (host, inherited by the workers)
  const ReadLibIndex *ix;       // its index for k, made before the fork
  std::vector<uint64_t> first;  // read shares
  std::string prefix;
};

// The most count records this rank may take in one round: the largest round (round_bytes, as the single-GPU count
// plans it) that fits rank_round_bytes, capped by mhb_set_round_limit.  Called when every share is on its device.
uint64_t count_round_budget(int rank, int world, uint64_t n_total, uint32_t k, int32_t m) {
  const size_t avail = rank_round_bytes(rank, world);
  const size_t fixed = (size_t)64 << 20;  // round arrays, counters, the exchange's small tables
  const uint32_t WR = mhb_count_record_words(k), WE = mhb_words_per_edge(k);
  uint64_t cap = largest_round(std::max<uint64_t>(n_total, 1), fixed, avail,
                               [&](uint64_t n) { return round_bytes(n, WR, WE, m, k); });
  if (!cap) fail_nomem("%zu free bytes for this rank: not even one count record fits", avail);
  if (count_round_limit()) cap = std::min(cap, count_round_limit());
  return cap;
}

// A small read library in host memory (an image of n reads and its index) to the device, for the mercy kernels: bufs[0]
// the image, bufs[1] / bufs[2] the read and edge offsets of variable-length reads
mhb_dev_reads upload_reads(const std::vector<uint32_t> &img, uint64_t n, const ReadLibIndex &ix, DevBuf *bufs,
                           const char *what) {
  mhb_dev_reads v;
  memset(&v, 0, sizeof(v));
  CKL(bufs[0].alloc((img.size() + 16) * 4, what));
  if (!img.empty()) CKC(cudaMemcpy(bufs[0].p, img.data(), img.size() * 4, cudaMemcpyHostToDevice));
  v.bin = bufs[0].as<uint32_t>();
  v.bin_words = img.size();
  v.n_reads = n;
  v.fixed_len = ix.fixed_len;
  if (!ix.fixed_len) {
    for (int j = 1; j < 3; ++j) {
      CKL(bufs[j].alloc((n + 1) * 8, what));
      CKC(cudaMemcpy(bufs[j].p, (j == 1 ? ix.rec_off : ix.unit_off).data(), (n + 1) * 8, cudaMemcpyHostToDevice));
    }
    v.rec_off = bufs[1].as<uint64_t>();
    v.edge_off = bufs[2].as<uint64_t>();
  }
  return v;
}

struct CountRank {
  const Job &J;
  Exchange &X;
  const int W, r;
  const uint32_t k, WR, WE;
  const int32_t m;
  const uint64_t r0, nr, w0;  // my share of the reads, and its first image word
  ReadLibIndex six;           // its index, rebased to the share
  std::optional<ChunkStream> rs;  // ... resident on the device or streamed from the inherited host image
  DevBuf lib, mul, ns;        // lib: the stream's device memory
  uint8_t owner[256];         // the count's owner of every leading byte, which also answers the mercy searches
  int R = 1;
  uint64_t n_sent = 0, n_own = 0;
  DevBuf edges, aux;          // my solid edges and flags (then the mercy edges behind them, when they fit: cap_all)
  uint64_t n_solid = 0, cap_all = 0;
  std::vector<uint32_t> edges_h;  // my solid edges on the host: appended round by round, or copied once by files()
  std::vector<uint64_t> cand_ids;
  uint64_t n_cand = 0, has_tips = 0, n_mercy = 0;
  DevBuf big;                 // solid + mercy edges, when they do not fit in edges
  uint32_t *all_edges = nullptr;

  CountRank(const Job &J_, Exchange &X_)
      : J(J_), X(X_), W(X_.world), r(X_.rank), k(J_.k), WR(mhb_count_record_words(J_.k)), WE(mhb_words_per_edge(J_.k)),
        m(J_.m), r0(J_.first[X_.rank]), nr(J_.first[X_.rank + 1] - r0), w0(J_.ix->word_of(r0)) {}
  const uint32_t *read_at(uint64_t i) const { return J.bin + J.ix->word_of(r0 + i); }  // my read i, at its length word

  // My share as a chunk stream over the inherited host image (J.bin + w0, for variable-length reads with offsets
  // rebased to the share): resident when it fits, next to the mercy marks and the smallest count round, in what this
  // rank may use (mhb_read_stream_decide, the rule of the single-GPU count); otherwise, or when mhb_set_read_chunk_limit
  // is set, streamed through the device in chunks that end on read boundaries.  Every pass over my reads goes through it.
  void load() {
    const ReadLibIndex &ix = *J.ix;
    const uint64_t nw = ix.word_of(r0 + nr) - w0;
    six.fixed_len = ix.fixed_len;
    six.n_units = ix.fixed_len > k ? nr * (ix.fixed_len - k) : 0;
    if (!ix.fixed_len) {
      six.rec_off.resize(nr + 1);
      six.unit_off.resize(nr + 1);
      for (uint64_t i = 0; i <= nr; ++i) {
        six.rec_off[i] = ix.rec_off[r0 + i] - w0;
        six.unit_off[i] = ix.unit_off[r0 + i] - ix.unit_off[r0];
      }
      six.n_units = six.unit_off[nr];
    }
    X.barrier();  // every rank has its context: nobody allocates until the free memory is read
    const size_t avail = rank_round_bytes(r, W);
    X.barrier();
    const size_t share = ChunkStream::image_bytes(nw) + (ix.fixed_len ? 0 : 2 * ChunkStream::side_bytes(nr, 0));
    const size_t marks = 2 * pad256((nr + 1) * 4) + pad256((nr + 1) * 8);  // first, last, candidates: either form
    const size_t smallest = ((size_t)64 << 20) + round_bytes(1, WR, WE, m, k);  // as count_round_budget plans it
    const bool stream = mhb_read_stream_decide(share + marks + smallest, avail, 0, read_chunk_limit()) != 0;
    read_stream_stats_reset();
    rs.emplace();
    CKL(init_read_stream(&*rs, J.bin + w0, nw, nr, six,
                         stream ? (read_chunk_limit() ? read_chunk_limit() : read_chunk_auto_bytes()) : 0));
    CKL(lib.alloc(rs->device_bytes(), stream ? "count: read chunk buffers" : "count: reads"));
    CKL(rs->bind(lib.p, nullptr));
    CKL(mul.alloc(65536 * 8, "count: multiplicity histogram"));
    CKL(ns.alloc(8 * 8, "count: counters"));
    CKC(cudaMemset(mul.p, 0, 65536 * 8));
    CKC(cudaMemset(ns.p, 0, 64));
  }

  // one pass over my share: fn(a chunk as a read library, the share's index of its first read), once per chunk
  void each_chunk(const std::function<int(const mhb_dev_reads &, uint64_t)> &fn) {
    CKL(rs->pass(nullptr, [&](const ChunkView &c) {
      mhb_dev_reads v;
      v.bin = c.words;
      v.bin_words = c.n_words;
      v.n_reads = c.n;
      v.fixed_len = six.fixed_len;
      v.rec_off = c.at<uint64_t>(0);
      v.edge_off = c.at<uint64_t>(1);
      return fn(v, c.first);
    }));
  }

  // The count rounds: my records of the round straight into their owners, then every owner counts what it received.
  // The plan caps every owner at its round budget.  The histogram and every round are one pass over my share: the
  // route's cursors keep counting across the launches of a round, and the owner counts the same multiset of records
  // whatever the chunks.
  void count_rounds() {
    OwnerExchange ex;
    {
      std::vector<uint64_t> h(65536);
      DevBuf h16;
      CKL(h16.alloc(65536 * 8, "count: bucket histogram"));
      CKC(cudaMemset(h16.p, 0, 65536 * 8));
      each_chunk([&](const mhb_dev_reads &v, uint64_t) {
        return mhb_count_extract_owners(nullptr, &v, k, h16.as<uint64_t>(), nullptr, nullptr, nullptr, nullptr, nullptr,
                                        nullptr);
      });
      CKC(cudaMemcpy(h.data(), h16.p, 65536 * 8, cudaMemcpyDeviceToHost));
      h16.release();
      ex.gather(X, h.data(), 65536);  // ... behind which every share is on its device: what is left the rounds may take
    }
    const uint64_t budget = count_round_budget(r, W, J.ix->n_units, k, m);
    ex.open(X, X.gather(&budget, 1).data(), WR * 4, "count: edge records received");
    R = ex.plan.R;
    n_sent = ex.n_sent;
    n_own = ex.n_own;
    memcpy(owner, ex.plan.owner, 256);
    if (r == 0) XINFO("count plan: %d round%s over bucket ranges\n", R, R > 1 ? "s" : "");

    const uint64_t n_round_max = *std::max_element(ex.own.begin(), ex.own.end());
    const uint64_t cap = n_round_max / (uint64_t)std::max(1, m) + 1;
    CKL(edges.alloc((cap * WE + 16) * 4, "count: solid edges"));
    CKL(aux.alloc(cap + 16, "count: edge flags"));
    std::vector<uint8_t> aux_h;  // the flags of every round, on the host, when there are several rounds
    {
      DevBuf tmp, work;
      CKL(tmp.alloc((n_round_max * WR + 16) * 4, "count: sort buffer"));
      const CountWork cw = count_work_plan(std::max<uint64_t>(n_round_max, 1), k, m);
      CKL(work.alloc(cw.bytes, "count: count work area"));
      uint64_t *d_ns = ns.as<uint64_t>();
      for (int t = 0; t < R; ++t) {
        ex.send(X, t, "count records", [&](const OwnerRoute &rt) {
          each_chunk([&](const mhb_dev_reads &v, uint64_t) {
            return mhb_count_extract_owners(nullptr, &v, k, nullptr, rt.owner, rt.base, rt.cursor, rt.cap, rt.lo, rt.hi);
          });
        });
        const uint64_t n_t = ex.own[t];
        uint64_t s_t = 0;
        if (n_t) {
          CKC(cudaMemset(d_ns, 0, 8));
          CKL(run_count_stage(nullptr, cw, ex.mine.as<uint32_t>(), tmp.as<uint32_t>(), n_t, k, m, nullptr,
                              edges.as<uint32_t>(), aux.as<uint8_t>(), cap, mul.as<uint64_t>(), d_ns, work.as<char>(),
                              nullptr, nullptr));
          CKC(cudaMemcpy(&s_t, d_ns, 8, cudaMemcpyDeviceToHost));
          if (s_t > cap) fail("internal: solid edges exceed capacity");
        }
        if (R > 1 && s_t) {  // the round's edges follow those of the lower bucket ranges (count_host_rounds)
          edges_h.resize((n_solid + s_t) * WE);
          aux_h.resize(n_solid + s_t);
          CKC(cudaMemcpy(edges_h.data() + n_solid * WE, edges.p, s_t * WE * 4, cudaMemcpyDeviceToHost));
          CKC(cudaMemcpy(aux_h.data() + n_solid, aux.p, s_t, cudaMemcpyDeviceToHost));
        }
        n_solid += s_t;
        X.barrier();  // nobody stores into my receive buffer before I have counted it
      }
    }
    ex.close(X);  // the count records are gone: give the memory back before the mercy and SdBG stages
    cap_all = cap;
    if (R > 1) {  // exactly my n_solid edges and flags back to the device
      edges.release();
      aux.release();
      cap_all = n_solid;
      CKL(edges.alloc((n_solid * WE + 16) * 4, "count: solid edges"));
      CKL(aux.alloc(n_solid + 16, "count: edge flags"));
      if (n_solid) {
        CKC(cudaMemcpy(edges.p, edges_h.data(), n_solid * WE * 4, cudaMemcpyHostToDevice));
        CKC(cudaMemcpy(aux.p, aux_h.data(), n_solid, cudaMemcpyHostToDevice));
      }
    }
    std::vector<uint64_t> h(65536);
    CKC(cudaMemcpy(h.data(), mul.p, 65536 * 8, cudaMemcpyDeviceToHost));
    X.publish("mul", h.data(), 65536 * 8);
  }

  // Mercy edges answered by the owners: the tip edges of every rank mark my reads, my candidate reads go to every rank,
  // and every rank answers, for the candidates of ALL ranks, the searches that land in its bucket range.
  void mercy() {
    const uint32_t *d_edges = edges.as<uint32_t>();
    all_edges = edges.as<uint32_t>();
    uint64_t *d_ns = ns.as<uint64_t>();
    uint64_t n_tip = 0;
    CKL(mhb_count_tip_edges(nullptr, aux.as<uint8_t>(), n_solid, &n_tip));
    {
      DevBuf tips, taux;
      CKL(tips.alloc((n_tip * WE + 16) * 4, "count: tip edges"));
      CKL(taux.alloc(n_tip + 16, "count: tip edge flags"));
      CKC(cudaMemset(d_ns, 0, 8));
      CKL(mhb_compact_tip_edges(nullptr, d_edges, aux.as<uint8_t>(), n_solid, k, tips.as<uint32_t>(), taux.as<uint8_t>(),
                                n_tip, d_ns));
      std::vector<char> buf(n_tip * (WE * 4 + 1));
      if (n_tip) {
        CKC(cudaMemcpy(buf.data(), tips.p, n_tip * WE * 4, cudaMemcpyDeviceToHost));
        CKC(cudaMemcpy(buf.data() + n_tip * WE * 4, taux.p, n_tip, cudaMemcpyDeviceToHost));
      }
      X.publish("tips", buf.data(), buf.size());
    }
    const std::vector<uint64_t> n_tips = X.gather(&n_tip, 1);
    uint64_t n_tip_all = 0;
    for (uint64_t c : n_tips) n_tip_all += c;
    DevBuf first, last, cand;
    CKL(first.alloc((nr + 1) * 4, "count: first tip marks"));
    CKL(last.alloc((nr + 1) * 4, "count: last tip marks"));
    CKL(cand.alloc((nr + 1) * 8, "count: candidate reads"));
    uint64_t *d_cand = cand.as<uint64_t>();
    {
      std::vector<uint32_t> te(n_tip_all * WE + 4);
      std::vector<uint8_t> ta(n_tip_all + 4);
      uint64_t at = 0;
      for (int o = 0; o < W; ++o) {
        const uint64_t c = n_tips[o];
        if (!c) continue;
        const std::vector<char> v = X.fetch("tips", o);
        memcpy(te.data() + at * WE, v.data(), c * WE * 4);
        memcpy(ta.data() + at, v.data() + c * WE * 4, c);
        at += c;
      }
      DevBuf d_te, d_ta, tipset, cs;
      CKL(d_te.alloc((n_tip_all * WE + 16) * 4, "count: tip edges of every rank"));
      CKL(d_ta.alloc(n_tip_all + 16, "count: tip edge flags of every rank"));
      if (n_tip_all) {
        CKC(cudaMemcpy(d_te.p, te.data(), n_tip_all * WE * 4, cudaMemcpyHostToDevice));
        CKC(cudaMemcpy(d_ta.p, ta.data(), n_tip_all, cudaMemcpyHostToDevice));
      }
      const size_t tb = mhb_tipset_bytes(n_tip_all, k);
      CKL(tipset.alloc(tb, "count: tip set"));
      CKL(mhb_tipset_build(nullptr, d_te.as<uint32_t>(), d_ta.as<uint8_t>(), n_tip_all, k, tipset.p, tb, n_tip_all));
      each_chunk([&](const mhb_dev_reads &v, uint64_t c0) {  // every chunk marks its reads at its first read
        return mhb_count_mark_mercy(nullptr, &v, k, tipset.p, tb, n_tip_all, first.as<uint32_t>() + c0,
                                    last.as<uint32_t>() + c0);
      });
      const size_t csb = mhb_mercy_candidates_scratch_bytes(nr);
      CKL(cs.alloc(csb, "count: candidate scratch"));
      CKL(mhb_mercy_candidates(nullptr, first.as<uint32_t>(), last.as<uint32_t>(), nr, d_cand, &n_cand, cs.p, csb));
    }
    cand_ids.resize(n_cand);
    if (n_cand) CKC(cudaMemcpy(cand_ids.data(), d_cand, n_cand * 8, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> cr;  // my candidate reads as their image words (length word + payload), in read order
    {  // number of reads with both marks set (the "(%d)" of the reference's log line) + my candidate reads
      std::vector<uint32_t> f(nr), l(nr);
      if (nr) {
        CKC(cudaMemcpy(f.data(), first.p, nr * 4, cudaMemcpyDeviceToHost));
        CKC(cudaMemcpy(l.data(), last.p, nr * 4, cudaMemcpyDeviceToHost));
      }
      for (uint64_t i = 0; i < nr; ++i) has_tips += f[i] != MHB_SENTINEL_OFFSET && l[i] != MHB_SENTINEL_OFFSET;
      for (uint64_t c = 0; c < n_cand; ++c) {
        const uint32_t *rd = read_at(cand_ids[c]);
        cr.insert(cr.end(), rd, rd + 1 + div_ceil(rd[0], 16));
      }
      X.publish("cand", cr.data(), cr.size() * 4);
    }
    const std::vector<uint64_t> n_cands = X.gather(&n_cand, 1);
    uint64_t n_cand_all = 0, cand_off[kMaxRanks + 1];
    for (int o = 0; o < W; ++o) {
      cand_off[o] = n_cand_all;
      n_cand_all += n_cands[o];
    }
    cand_off[W] = n_cand_all;
    if (!n_cand_all) return;
    // the candidates of every rank, in rank order, indexed as a library of their own; the longest of them sizes the
    // answer planes on every rank alike
    std::vector<uint32_t> all;
    for (int o = 0; o < W; ++o)
      if (n_cands[o]) {
        const std::vector<char> v = X.fetch("cand", o);
        all.insert(all.end(), (const uint32_t *)v.data(), (const uint32_t *)(v.data() + v.size()));
      }
    ReadLibIndex cix;
    CKL(index_read_lib(all.data(), all.size(), n_cand_all, k, &cix, FixedCheck::kSerial));
    uint32_t L = 0;
    for (uint64_t c = 0; c < n_cand_all; ++c) L = std::max(L, all[cix.word_of(c)]);
    {
      DevBuf call[3], lut, planes;
      const mhb_dev_reads greads = upload_reads(all, n_cand_all, cix, call, "count: candidate reads of every rank");
      CKL(lut.alloc(mhb_edge_lut_bytes(), "count: edge lookup table"));
      CKL(mhb_edge_lut_build(nullptr, d_edges, n_solid, k, lut.p));
      const size_t pw_all = mhb_mercy_planes_words(n_cand_all, L);
      CKL(planes.alloc(pw_all * 4, "count: mercy answer planes"));
      CKL(mhb_mercy_probe_owned(nullptr, &greads, nullptr, n_cand_all, L, k, d_edges, n_solid, lut.p, owner, (uint32_t)r,
                                planes.as<uint32_t>()));
      std::vector<uint32_t> hp(pw_all);
      CKC(cudaMemcpy(hp.data(), planes.p, pw_all * 4, cudaMemcpyDeviceToHost));
      X.publish("planes", hp.data(), pw_all * 4);
    }
    X.barrier();
    if (!n_cand) return;
    // the answers of every rank about MY candidates: rank s's file holds them at [cand_off[r], cand_off[r] + n_cand)
    const size_t pw1 = mhb_mercy_planes_words(1, L), pw_mine = pw1 * n_cand;
    std::vector<uint32_t> mine((size_t)W * pw_mine);
    for (int s = 0; s < W; ++s) {
      const std::vector<char> v = X.fetch("planes", s, cand_off[r] * pw1 * 4, pw_mine * 4);
      memcpy(mine.data() + (size_t)s * pw_mine, v.data(), pw_mine * 4);
    }
    // my candidates as a library of their own, the image published as "cand": candidate c is its read c, so the
    // last steps read no more than the candidates, whether my share is resident or streamed
    ReadLibIndex mix;
    CKL(index_read_lib(cr.data(), cr.size(), n_cand, k, &mix, FixedCheck::kSerial));
    DevBuf mbuf[3], d_mine, ms;
    const mhb_dev_reads creads = upload_reads(cr, n_cand, mix, mbuf, "count: my candidate reads");
    {
      std::vector<uint64_t> ids(n_cand);
      std::iota(ids.begin(), ids.end(), 0ull);
      CKC(cudaMemcpy(d_cand, ids.data(), n_cand * 8, cudaMemcpyHostToDevice));
    }
    CKL(d_mine.alloc(mine.size() * 4, "count: mercy answers about my candidates"));
    CKC(cudaMemcpy(d_mine.p, mine.data(), mine.size() * 4, cudaMemcpyHostToDevice));
    const size_t msb = mhb_mercy_edges_scratch_bytes(n_cand, L) - mhb_edge_lut_bytes();
    CKL(ms.alloc(msb, "count: mercy edge scratch"));
    CKL(mhb_mercy_count_planes(nullptr, &creads, d_cand, n_cand, L, k, d_mine.as<uint32_t>(), (uint32_t)W, pw_mine, &n_mercy,
                               ms.p, msb));
    if (!n_mercy) return;
    if (n_solid + n_mercy > cap_all) {  // reads overlapping only at their ends: more mercy than solid edges
      CKL(big.alloc(((n_solid + n_mercy) * WE + 16) * 4, "count: solid and mercy edges"));
      CKC(cudaMemcpy(big.p, d_edges, n_solid * WE * 4, cudaMemcpyDeviceToDevice));
      all_edges = big.as<uint32_t>();
    }
    CKL(mhb_mercy_edges_write(nullptr, &creads, d_cand, n_cand, L, k, all_edges + n_solid * WE, n_mercy, n_mercy, ms.p, msb));
    CKC(cudaDeviceSynchronize());
  }

  // the marks were the last pass over my share: its stream goes; files() reads the host image
  void release_share() {
    rs.reset();
    lib.release();
  }

  // The SdBG stage over solid + mercy edges, in rounds over bucket ranges when an owner's items do not fit its device
  // at once: in every round my items go straight from the edges into their owners' buffers, and each owner sorts and
  // emits what it received.  The owned solid edges still carry the count stage's in/out flags: the $-items the emitter
  // is certain to discard are neither generated nor exchanged (mhb_s2s_edges_owners, DESIGN.md 4.7); under
  // MHB_S2S_NO_PRUNE all six items of every edge go, through the sequence view of the edge records.
  void sdbg() {
    const bool prune = !getenv("MHB_S2S_NO_PRUNE");
    const uint64_t n_seqs = n_solid + n_mercy;
    mhb_dev_seqs seqs;
    memset(&seqs, 0, sizeof(seqs));
    seqs.words = all_edges;
    seqs.n_words = n_seqs * WE;
    seqs.n_seqs = n_seqs;
    seqs.fixed_len = k + 1;
    seqs.fixed_stride = WE;
    const uint8_t *flags = aux.as<uint8_t>();
    std::vector<uint64_t> h(65536);
    {
      DevBuf h16;
      CKL(h16.alloc(65536 * 8, "count: SdBG bucket histogram"));
      CKC(cudaMemset(h16.p, 0, 65536 * 8));
      if (prune)
        CKL(mhb_s2s_edges_owners(nullptr, all_edges, flags, n_seqs, n_solid, k, h16.as<uint64_t>(), nullptr, nullptr,
                                 nullptr, nullptr, nullptr, nullptr));
      else
        CKL(mhb_s2s_bucket_hist(nullptr, &seqs, k, n_seqs * 6, h16.as<uint64_t>()));
      CKC(cudaMemcpy(h.data(), h16.p, 65536 * 8, cudaMemcpyDeviceToHost));
    }
    uint64_t n_sdbg_own = 0;
    const int R_sdbg = sdbg_stage(X, h.data(), k, J.prefix, &n_sdbg_own, [&](const OwnerRoute &rt) {
      if (prune)
        CKL(mhb_s2s_edges_owners(nullptr, all_edges, flags, n_seqs, n_solid, k, nullptr, rt.owner, rt.base, rt.cursor,
                                 rt.cap, rt.lo, rt.hi));
      else
        CKL(mhb_s2s_extract_owners_round(nullptr, &seqs, k, n_seqs * 6, rt.owner, rt.base, rt.cursor, rt.cap, rt.lo,
                                         rt.hi));
    });
    StreamStats st;
    mhb_read_stream_stats(&st.chunks, &st.passes, &st.h2d_bytes);
    mhb_read_stream_times(nullptr, nullptr, nullptr, &st.pass_ms);
    RANK_INFO("rank %d: %llu reads, %llu records sent, %llu owned in %d round%s, %llu solid edges, %llu SdBG items owned "
              "in %d round%s; reads %s; peak device memory %.1f MiB\n",
              r, (unsigned long long)nr, (unsigned long long)n_sent, (unsigned long long)n_own, R, R > 1 ? "s" : "",
              (unsigned long long)n_solid, (unsigned long long)n_sdbg_own, R_sdbg, R_sdbg > 1 ? "s" : "",
              share_form(st).c_str(), DevBuf::peak_bytes() / 1048576.0);
  }

  // The files: my bucket range of the edges; rank 0 merges the tables and writes the library-wide files
  void files() {
    if (R == 1) {
      edges_h.resize(n_solid * WE);
      if (n_solid) CKC(cudaMemcpy(edges_h.data(), edges.p, n_solid * WE * 4, cudaMemcpyDeviceToHost));
    }
    CKL(write_bytes(J.prefix + ".edges." + std::to_string(r), edges_h.data(), n_solid * WE * 4));
    {
      std::vector<int64_t> cnt(65536, 0);
      for (uint64_t i = 0; i < n_solid; ++i) cnt[edges_h[i * WE] >> 16]++;
      X.publish("ecnt", cnt.data(), 65536 * 8);
      std::vector<uint32_t> rec;
      for (uint64_t c = 0; c < n_cand; ++c) append_cand_reversed(read_at(cand_ids[c]), &rec);
      X.publish("candrev", rec.data(), rec.size() * 4);
    }
    const uint64_t mine[4] = {n_solid, n_cand, has_tips, n_mercy};
    const std::vector<uint64_t> all = X.gather(mine, 4);
    if (r == 0) {
      // merged P.edges.info: bucket -> (file = owner rank, offset inside that file, count)
      std::vector<std::vector<int64_t>> ec(W);
      for (int o = 0; o < W; ++o) {
        const std::vector<char> v = X.fetch("ecnt", o);
        ec[o].assign((const int64_t *)v.data(), (const int64_t *)v.data() + 65536);
      }
      CKL(write_edges_info(J.prefix, k, WE, ec));
      // P.cand (rank order = read order: the reads were dealt in contiguous blocks) and P.counting (global histogram)
      std::vector<char> cand_file;
      uint64_t tot[4] = {0};
      for (int o = 0; o < W; ++o) {
        const std::vector<char> v = X.fetch("candrev", o);
        cand_file.insert(cand_file.end(), v.begin(), v.end());
        for (int i = 0; i < 4; ++i) tot[i] += all[o * 4 + i];
      }
      CKL(write_bytes(J.prefix + ".cand", cand_file.data(), cand_file.size()));
      CKL(write_counting(J.prefix, sum_mul(X).data()));
      FILE *f = fopen((J.prefix + ".sdbg_fused").c_str(), "w");
      if (f) {
        fprintf(f, "%u 1 %d\n", k, W);
        fclose(f);
      }
      XINFO("Total number of candidate reads: %llu (%llu)\n", (unsigned long long)tot[1], (unsigned long long)tot[2]);
      XINFO("Total number of solid edges: %llu\n", (unsigned long long)tot[0]);
      XINFO("Number of mercy edges: %llu\n", (unsigned long long)tot[3]);
      sdbg_merge_info(X, k, J.prefix);  // merged P.sdbg_info
    }
    X.barrier();
  }
};

void worker(const Job &J, Exchange &X) {
  bind_device(X.rank, X.world);
  CountRank c(J, X);
  c.load();
  c.count_rounds();
  c.mercy();
  c.release_share();
  c.sdbg();
  c.files();
}

// ================================================================================================
// seq2sdbg on several GPUs: the sequences are dealt in contiguous shares, the items meet on their owners
// ================================================================================================
struct SeqJob {
  uint32_t k;
  const HostSeqs *seqs;                // every sequence (host, inherited by the workers)
  std::vector<uint64_t> first;         // shares
  std::string prefix;
};

void s2s_worker(const SeqJob &J, Exchange &X) {
  const int W = X.world, r = X.rank;
  const uint32_t k = J.k;
  bind_device(r, W);

  // ---- my share as a chunk stream over the inherited sequences: their words and, rebased to the share (and by the
  // stream to each chunk), word offsets, item offsets, lengths and multiplicities.  Resident when it fits, next to the
  // smallest SdBG round, in what this rank may use (mhb_read_stream_decide); otherwise, or when mhb_set_s2s_chunk_limit
  // is set, streamed through the device in chunks that end on sequence boundaries ----
  const HostSeqs &S = *J.seqs;
  const uint64_t s0 = J.first[r], n = J.first[r + 1] - s0, w0 = S.word_off[s0], nw = S.word_off[s0 + n] - w0;
  std::vector<uint64_t> wo(n + 1), io(n + 1, 0);
  for (uint64_t i = 0; i <= n; ++i) wo[i] = S.word_off[s0 + i] - w0;
  for (uint64_t i = 0; i < n; ++i) io[i + 1] = io[i] + seq_items(S.len[s0 + i], k);
  const uint64_t n_items = io[n];
  ChunkStream::Input in;
  in.image = S.words.data() + w0;
  in.words = nw;
  in.n = n;
  in.word_off = wo.data();
  in.side[0] = {wo.data(), 0};
  in.side[1] = {io.data(), 0};
  in.side[2] = {S.len.data() + s0, 4};
  in.side[3] = {S.mult.data() + s0, 2};
  X.barrier();  // every rank has its context: nobody allocates until the free memory is read
  const size_t avail = rank_round_bytes(r, W);
  X.barrier();
  const size_t share = ChunkStream::image_bytes(nw) + 2 * ChunkStream::side_bytes(n, 0) + ChunkStream::side_bytes(n, 4) +
                       ChunkStream::side_bytes(n, 2);
  const size_t fixed = (size_t)64 << 20;  // as sdbg_stage plans its rounds
  const int no_round = mhb_sdbg_round_budget(avail, share + fixed, k, 1) == 0;
  const bool stream = mhb_read_stream_decide(share, avail, no_round, s2s_chunk_limit()) != 0;
  std::vector<uint64_t> first;  // a sequence costs its words, two offsets, its length and its multiplicity
  if (stream)
    plan_chunks(wo.data(), 0, 8 + 8 + 4 + 2, n, s2s_chunk_limit() ? s2s_chunk_limit() : read_chunk_auto_bytes(), &first);
  StreamStats st;
  DevBuf dev;
  {
    ChunkStream cs;
    CKL(cs.init(in, std::move(first), &st));
    CKL(dev.alloc(cs.device_bytes(), stream ? "seq2sdbg: sequence chunk buffers" : "seq2sdbg: sequences"));
    CKL(cs.bind(dev.p, nullptr));
    // one pass over my share: fn(a chunk as a sequence set, its items), once per chunk
    auto each_chunk = [&](const std::function<int(const mhb_dev_seqs &, uint64_t)> &fn) {
      CKL(cs.pass(nullptr, [&](const ChunkView &c) {
        mhb_dev_seqs v;
        memset(&v, 0, sizeof(v));
        v.words = c.words;
        v.n_words = c.n_words;
        v.n_seqs = c.n;
        v.word_off = c.at<uint64_t>(0);
        v.item_off = c.at<uint64_t>(1);
        v.len = c.at<uint32_t>(2);
        v.mult = c.at<uint16_t>(3);
        return fn(v, io[c.first + c.n] - io[c.first]);
      }));
    };

    // ---- bucket histogram of my items -> the plan; per round, every item of the round's bucket ranges straight into
    // its owner's buffer, one pass over my share (it stays on the device, or in host memory, until the last round:
    // every round extracts from it again) ----
    std::vector<uint64_t> h(65536);
    {
      DevBuf h16;
      CKL(h16.alloc(65536 * 8, "seq2sdbg: bucket histogram"));
      CKC(cudaMemset(h16.p, 0, 65536 * 8));
      each_chunk([&](const mhb_dev_seqs &v, uint64_t n_v) {
        return mhb_s2s_bucket_hist(nullptr, &v, k, n_v, h16.as<uint64_t>());
      });
      CKC(cudaMemcpy(h.data(), h16.p, 65536 * 8, cudaMemcpyDeviceToHost));
    }
    uint64_t n_own = 0;
    const int R = sdbg_stage(X, h.data(), k, J.prefix, &n_own, [&](const OwnerRoute &rt) {
      each_chunk([&](const mhb_dev_seqs &v, uint64_t n_v) {
        return mhb_s2s_extract_owners_round(nullptr, &v, k, n_v, rt.owner, rt.base, rt.cursor, rt.cap, rt.lo, rt.hi);
      });
    });
    RANK_INFO("rank %d: %llu sequences, %llu items sent, %llu owned in %d round%s; sequences %s; peak device memory "
              "%.1f MiB\n", r, (unsigned long long)n, (unsigned long long)n_items, (unsigned long long)n_own, R,
              R > 1 ? "s" : "", share_form(st).c_str(), DevBuf::peak_bytes() / 1048576.0);
  }
  dev.release();
  X.barrier();
  if (r == 0) sdbg_merge_info(X, k, J.prefix);
  X.barrier();
}

// ================================================================================================
// iterate on several GPUs: the reads are dealt in contiguous shares, the candidate sets meet on their owners
// ================================================================================================
struct IterJob {
  mhb_iterate_args a;          // every contig and the whole `.bin` image (host, inherited by the workers)
  std::vector<uint64_t> first;  // read shares
  std::vector<uint64_t> word;   // first word of every share, n_ranks + 1 entries
  int fd;                       // P.edges.0, created empty by the parent
  std::string prefix;
};

void iter_worker(const IterJob &J, Exchange &X) {
  const int W = X.world, r = X.rank;
  const uint32_t k = J.a.k, step = J.a.step, w2 = mhb_words_per_edge(k + step);
  const int top = (int)(4 * w2 - 1);
  bind_device(r, W);

  // ---- the flank index of every contig, then the read pass over my share: my unique candidates, on the device ----
  mhb_iterate_args a = J.a;
  a.bin = J.a.bin + J.word[r];
  a.bin_words = J.word[r + 1] - J.word[r];
  a.n_reads = J.first[r + 1] - J.first[r];
  DevBuf set;
  uint64_t n_flanks = 0, n_set = 0, n_cand = 0, n_aligned = 0, n_chunks = 0;
  read_stream_stats_reset();
  {
    IterFlanks flanks;
    CKL(iter_build_flanks(&a, &flanks));
    n_flanks = flanks.n;
    CKL(iter_collect(&a, flanks, &set, &n_set, &n_cand, &n_aligned));
    CKL(mhb_read_stream_stats(&n_chunks, nullptr, nullptr));
  }  // the flank table and the buffers of the read pass are freed: only the set stays

  // ---- every edge to the rank owning its leading byte ----
  OwnerExchange ex;
  {
    DevBuf hist, ws;
    CKL(hist.alloc(256 * 8, "iterate: leading-byte histogram"));
    CKC(cudaMemset(hist.p, 0, 256 * 8));
    CKL(hist_byte(nullptr, set.as<uint32_t>(), n_set, w2, top, hist.as<uint64_t>()));
    const size_t ws_bytes = mhb_sort_workspace_bytes(std::max<uint64_t>(n_set, 1), w2);
    CKL(ws.alloc(ws_bytes, "iterate: partition workspace"));
    uint64_t h[256];
    CKC(cudaMemcpy(h, hist.p, sizeof(h), cudaMemcpyDeviceToHost));
    ex.gather(X, h, 256);
    ex.open(X, nullptr, w2 * 4, "iterate: edges received");
    ex.send(X, 0, nullptr, [&](const OwnerRoute &rt) {
      CKL(mhb_partition_scatter(nullptr, set.as<uint32_t>(), n_set, w2, top, rt.owner, rt.base, ws.p, ws_bytes));
    });
  }
  set.release();

  // ---- the owner's sort + unique over what it received: an ascending run of the whole set ----
  const uint64_t n_own = ex.n_own;
  uint64_t n_uniq = 0;
  std::vector<uint32_t> edges;
  {
    DevBuf tmp;
    CKL(tmp.alloc((n_own * w2 + 16) * 4, "iterate: sort buffer"));
    uint32_t *uniq = nullptr;
    CKL(iter_sort_unique(ex.mine.as<uint32_t>(), tmp.as<uint32_t>(), n_own, k, step, &uniq, &n_uniq));
    edges.resize(n_uniq * w2);
    if (n_uniq) CKC(cudaMemcpy(edges.data(), uniq, n_uniq * w2 * 4, cudaMemcpyDeviceToHost));
  }
  ex.close(X);
  XINFO("rank %d: %llu reads (%s), %llu candidates, %llu unique sent, %llu received, %llu owned; peak device memory "
        "%.1f MiB\n", r, (unsigned long long)a.n_reads, n_chunks ? (std::to_string(n_chunks) + " chunks").c_str() : "resident",
        (unsigned long long)n_cand, (unsigned long long)n_set, (unsigned long long)n_own, (unsigned long long)n_uniq,
        DevBuf::peak_bytes() / 1048576.0);
  const uint64_t mine[2] = {n_uniq, n_aligned};
  const std::vector<uint64_t> all = X.gather(mine, 2);

  // ---- the owners' runs follow each other in rank order: one P.edges.0, as the single-GPU iterate writes it ----
  uint64_t before = 0;
  for (int o = 0; o < r; ++o) before += all[2 * o];
  const char *p = (const char *)edges.data();
  size_t left = edges.size() * 4;
  off_t at = (off_t)(before * w2 * 4);
  while (left) {
    const ssize_t got = pwrite(J.fd, p, left, at);
    if (got <= 0) throw Fail{"write to " + J.prefix + ".edges.0 failed", MHB_ERR_IO};
    p += got;
    left -= (size_t)got;
    at += got;
  }
  X.barrier();
  if (r == 0) {
    uint64_t n_edges = 0, aligned = 0;
    for (int o = 0; o < W; ++o) {
      n_edges += all[2 * o];
      aligned += all[2 * o + 1];
    }
    CKL(iterate_write_info(J.prefix, k + step, w2, n_edges));
    XINFO("Number of flank kmers: %llu\n", (unsigned long long)n_flanks);
    XINFO("Total: %llu, aligned: %llu. Iterative edges: %llu\n", (unsigned long long)J.first[W],
          (unsigned long long)aligned, (unsigned long long)n_edges);
  }
}

// ================================================================================================
// read2sdbg on several GPUs: the reads are dealt in contiguous shares; the stage-1 records meet on their owners in
// global read order, the bit planes are merged per share, the stage-2 items meet on their owners
// ================================================================================================
struct R2sJob {
  mhb_build_args a;             // the whole `.bin` image (host, inherited by the workers), k, m, need_mercy
  const ReadLibIndex *li;       // its index, made before the fork
  std::vector<uint64_t> first;  // read shares
  std::string prefix;
};

// The list form's candidates to the shares they lie in: I publish my stage-1 rounds' lists back to back ("cand") and,
// per round, the entry offsets at every share's first base ("candix": rounds x (world + 1)); every rank fetches from
// every owner the slice of each round inside its share.  Each slice is sorted, as its round is.
void cand_exchange(const R2sJob &J, Exchange &X, R2sShare &sh) {
  const int W = X.world, r = X.rank;
  const std::vector<std::vector<uint64_t>> &made = sh.cand_made();
  std::vector<uint64_t> all, ix;
  uint64_t n_made = 0;
  for (const auto &v : made) {
    for (int s = 0; s <= W; ++s) {
      const uint64_t key = s == W ? ~0ull : sh.base_of(J.first[s]) << 2;
      ix.push_back(all.size() + (uint64_t)(std::lower_bound(v.begin(), v.end(), key) - v.begin()));
    }
    all.insert(all.end(), v.begin(), v.end());
    n_made += v.size();
  }
  X.publish("cand", all.data(), all.size() * 8);
  X.publish("candix", ix.data(), ix.size() * 8);
  std::vector<uint64_t>().swap(all);
  X.barrier();  // every list is published
  std::vector<std::vector<uint64_t>> mine;
  uint64_t n_got = 0;
  for (int o = 0; o < W; ++o) {
    const std::vector<char> oix = X.fetch("candix", o);
    const uint64_t *p = (const uint64_t *)oix.data();
    const size_t rounds = oix.size() / 8 / (W + 1);
    for (size_t t = 0; t < rounds; ++t) {
      const uint64_t lo = p[t * (W + 1) + r], hi = p[t * (W + 1) + r + 1];
      if (hi <= lo) continue;
      const std::vector<char> b = X.fetch("cand", o, lo * 8, (hi - lo) * 8);
      mine.emplace_back((const uint64_t *)b.data(), (const uint64_t *)b.data() + (hi - lo));
      n_got += hi - lo;
    }
  }
  sh.cand_take(&mine);
  XINFO("rank %d: mercy candidates: %llu list entries made, %llu inside the share\n", r, (unsigned long long)n_made,
        (unsigned long long)n_got);
}

void r2s_worker(const R2sJob &J, Exchange &X) {
  const int W = X.world, r = X.rank;
  const uint32_t k = J.a.k, W2 = mhb_s2s_record_words(k);
  const int32_t m = J.a.m;
  bind_device(r, W);
  R2sShare sh;
  CKL(sh.load(&J.a, *J.li, J.first[r], J.first[r + 1]));
  // the form of the mercy candidates, the same on every rank: lists when one rank wants them (DESIGN.md §4.9)
  const int want = sh.want_cand_lists(rank_round_bytes(r, W)) ? 1 : 0;
  const uint64_t want64 = (uint64_t)want;
  bool lists = false;
  for (uint64_t w : X.gather(&want64, 1)) lists = lists || w;
  CKL(sh.bind_planes(lists));
  lists = sh.cand_lists();
  if (lists)
    XINFO("rank %d: mercy candidates as sorted lists: the solid plane of the whole library, the candidate planes of my "
          "share only\n", r);
  std::vector<uint64_t> h16(65536);
  uint64_t n_s1_own = 0;
  int R1 = 0;

  // ---- stage 1: my records straight into their owners' buffers, in global read order, in rounds over ascending
  // bucket ranges; each owner's planes ----
  if (m > 1) {
    CKL(sh.s1_hist(h16.data()));
    OwnerExchange ex;
    ex.gather(X, h16.data(), 65536);  // ... behind which every share and its planes are on the device
    uint64_t n_s1 = 0;
    for (uint64_t c : ex.hist) n_s1 += c;
    const uint64_t budget = sh.s1_round_budget(rank_round_bytes(r, W), W, n_s1);
    if (!budget) fail_nomem("%zu free bytes for this rank: not even a one-record stage-1 round fits", rank_round_bytes(r, W));
    ex.open(X, X.gather(&budget, 1).data(), sh.s1_record_words() * 4, "read2sdbg: stage-1 records received",
            sh.s1_narrow() ? "read2sdbg: stage-1 read_info received" : nullptr);
    log_loads(X, ex, "read2sdbg stage 1");
    R1 = ex.plan.R;
    n_s1_own = ex.n_own;
    const uint64_t n_max = *std::max_element(ex.own.begin(), ex.own.end());
    for (int t = 0; t < R1; ++t) {
      ex.send(X, t, "stage-1 records", [&](const OwnerRoute &rt) {
        CKL(sh.s1_count(rt));
        ex.check(X, t, "stage-1 records");  // the stores have no capacity: they run once the counts match the plan
        CKL(sh.s1_store(rt));
      });
      CKL(sh.s1_own(ex.mine.as<uint32_t>(), ex.info.as<uint64_t>(), ex.own[t], n_max));
      if (t + 1 < R1) X.barrier();  // nobody stores into my receive buffer before I have sorted it
    }
    sh.s1_end();
    ex.close(X);
    if (lists) cand_exchange(J, X, sh);

    // ---- plane merge: the words of my share's reads, OR-ed over every rank's planes (read through CUDA IPC) ----
    uint64_t handle[8];
    CKL(mhb_ipc_export(sh.planes(), (uint8_t *)handle));
    const std::vector<uint64_t> handles = X.gather(handle, 8);
    for (int o = 0; o < W; ++o) {
      if (o == r) continue;
      void *peer = nullptr;
      CKL(mhb_ipc_open((const uint8_t *)&handles[(size_t)o * 8], &peer));
      CKL(sh.or_planes(peer));
      CKL(mhb_ipc_close(peer));
    }
    X.barrier();  // nobody reads my planes any more: the mercy step may add to them
  }

  // ---- the mercy step and the stage-2 item count over my share ----
  uint64_t n_items = 0, n_mercy = 0;
  CKL(sh.mercy_count(&n_items, &n_mercy));

  // ---- stage 2: every item straight into its owner's buffer, in rounds over ascending bucket ranges; the owner sorts,
  // collapses and emits each round, and its rounds follow each other in bucket order ----
  CKL(sh.s2_hist(h16.data()));
  OwnerExchange ex;
  ex.gather(X, h16.data(), 65536);  // ... behind which the stage-1 buffers are gone on every rank
  uint64_t n_s2 = 0;
  for (uint64_t c : ex.hist) n_s2 += c;
  const uint64_t budget = sh.s2_round_budget(rank_round_bytes(r, W), n_s2);
  if (!budget) fail_nomem("%zu free bytes for this rank: not even a one-item stage-2 round fits", rank_round_bytes(r, W));
  ex.open(X, X.gather(&budget, 1).data(), W2 * 4, "read2sdbg: stage-2 items received");
  log_loads(X, ex, "read2sdbg stage 2");
  const int R2 = ex.plan.R;
  if (r == 0)
    XINFO("read2sdbg plan: stage 1 in %d round%s, stage 2 in %d round%s\n", R1, R1 == 1 ? "" : "s", R2, R2 == 1 ? "" : "s");
  const uint64_t n_max = *std::max_element(ex.own.begin(), ex.own.end());
  for (int t = 0; t < R2; ++t) {
    ex.send(X, t, "stage-2 items", [&](const OwnerRoute &rt) { CKL(sh.s2_send(rt)); });
    CKL(sh.s2_own(ex.mine.as<uint32_t>(), ex.own[t], n_max));
    if (t + 1 < R2) X.barrier();  // nobody stores into my receive buffer before I have sorted it
  }
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> table;
  uint64_t totals[16];
  sh.s2_result(&bytes, &table, totals);
  ex.close(X);
  sdbg_publish(X, totals, bytes, std::move(table), J.prefix);
  if (m > 1) {
    CKL(sh.counting(h16.data()));
    X.publish("mul", h16.data(), 65536 * 8);
  }
  XINFO("rank %d: %llu reads, %llu stage-1 records owned, %llu mercy edges, %llu items sent, %llu owned; peak device "
        "memory %.1f MiB\n", r, (unsigned long long)sh.n_reads(), (unsigned long long)n_s1_own, (unsigned long long)n_mercy,
        (unsigned long long)n_items, (unsigned long long)ex.n_own, DevBuf::peak_bytes() / 1048576.0);
  const std::vector<uint64_t> n_mercies = X.gather(&n_mercy, 1);
  if (r == 0) {
    if (m > 1) {  // Read2SdbgS1::Lv0Postprocess, read_to_sdbg_s1.cpp:557-566: the histogram over every owner's groups
      CKL(write_counting(J.prefix, sum_mul(X).data()));
      if (J.a.need_mercy) {
        uint64_t n_mercy_tot = 0;
        for (uint64_t c : n_mercies) n_mercy_tot += c;
        XINFO("Number mercy: %llu\n", (unsigned long long)n_mercy_tot);
      }
    }
    sdbg_merge_info(X, k, J.prefix);
  }
  X.barrier();
}

// Forks one worker per rank around a fresh control block and waits for all of them.  A worker that dies would leave
// the others at a barrier: the first abnormal exit takes the rest down.  A failure is reported with the error code of
// the first failed rank that set one (MHB_ERR_CUDA otherwise) and every rank's message.  Whatever the outcome, the
// exchange files of the run are removed once the workers are gone.
template <class Body>
int run_workers(int n, const char *what, Body body) {
  Control *C = (Control *)mmap(nullptr, sizeof(Control), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  if (C == MAP_FAILED) return mhb_set_error(MHB_ERR_NOMEM, "mmap of the control block failed");
  pthread_barrierattr_t ba;
  pthread_barrierattr_init(&ba);
  pthread_barrierattr_setpshared(&ba, PTHREAD_PROCESS_SHARED);
  pthread_barrier_init(&C->bar, &ba, (unsigned)n);
  const std::string xname = "mhb_" + std::to_string((long long)getpid());
  std::vector<pid_t> pids;
  fflush(nullptr);
  for (int r = 0; r < n; ++r) {
    const pid_t p = fork();
    if (p < 0) {
      for (pid_t q : pids) kill(q, SIGKILL);
      munmap(C, sizeof(Control));
      return mhb_set_error(MHB_ERR_NOMEM, "fork failed");
    }
    if (p == 0) {
      Exchange X{"/dev/shm/" + xname, r, n, C};
      DevBuf::reset_peak();  // the peak device memory a rank logs is its own
      int rc = 0;
      try {
        body(X);
      } catch (const Fail &e) {
        snprintf(C->err[r], sizeof(C->err[r]), "rank %d: %s", r, e.msg.c_str());
        C->err_code[r] = e.code;
        rc = 1;
      }
      fflush(nullptr);
      _exit(rc);
    }
    pids.push_back(p);
  }
  int failed = 0;
  for (size_t done = 0; done < pids.size(); ++done) {
    int st = 0;
    const pid_t p = wait(&st);
    if (p < 0) break;
    if (!(WIFEXITED(st) && WEXITSTATUS(st) == 0) && !failed) {
      failed = 1;
      for (pid_t q : pids)
        if (q != p) kill(q, SIGKILL);
    }
  }
  int rc = MHB_OK;
  if (failed) {
    std::string msg;
    int code = 0;
    for (int r = 0; r < n; ++r)
      if (C->err[r][0]) {
        msg += std::string(msg.empty() ? "" : "; ") + C->err[r];
        if (!code) code = C->err_code[r];
      }
    rc = mhb_set_error(code ? code : MHB_ERR_CUDA, "multi-GPU %s failed: %s", what, msg.empty() ? "a worker process died" : msg.c_str());
  }
  if (DIR *d = opendir("/dev/shm")) {  // <xname>.<tag>.<rank>
    while (const dirent *e = readdir(d))
      if (!strncmp(e->d_name, (xname + ".").c_str(), xname.size() + 1)) unlinkat(dirfd(d), e->d_name, 0);
    closedir(d);
  }
  pthread_barrier_destroy(&C->bar);
  munmap(C, sizeof(Control));
  return rc;
}

}  // namespace

extern "C" int mhb_count_run_multi(const mhb_count_opts *o, int n_gpus) {
  if (!o || !o->read_lib_file || !o->read_lib_file[0]) return mhb_set_error(MHB_ERR_ARG, "No read library configuration file!");
  if (o->host_mem == 0) return mhb_set_error(MHB_ERR_ARG, "Please specify the host memory!");
  if (n_gpus <= 1) return mhb_count_run(o);
  if (n_gpus > kMaxRanks) return mhb_set_error(MHB_ERR_ARG, "at most %d GPUs of one node are supported", kMaxRanks);
  const std::string lib = o->read_lib_file, prefix = o->output_prefix ? o->output_prefix : "out";
  const double t0 = now_s();
  long long total_bases = 0, n_reads = 0;
  std::vector<uint32_t> bin;
  if (int rc = load_read_lib(lib, &bin, &n_reads, &total_bases)) return rc;
  if (n_reads < n_gpus) {
    XINFO("%lld reads for %d GPUs: running on one GPU\n", n_reads, n_gpus);
    return mhb_count_run(o);
  }
  if (o->k < 12) {
    XINFO("k = %u is below 12, the mercy search's 12-base look-up prefix: running on one GPU\n", o->k);
    return mhb_count_run(o);
  }
  ReadLibIndex ix;  // indexed serially: the workers are forked next
  if (index_read_lib(bin.data(), bin.size(), (uint64_t)n_reads, o->k, &ix, FixedCheck::kSerial)) {
    XINFO("%s.bin ends inside a read: running on one GPU\n", lib.c_str());
    return mhb_count_run(o);
  }
  XINFO("%lld reads, %lld bases; k = %u, m = %d; %d GPUs\n", n_reads, total_bases, o->k, o->m, n_gpus);
  Job J;
  J.k = o->k;
  J.m = o->m;
  J.bin = bin.data();
  J.ix = &ix;
  J.first.resize(n_gpus + 1);
  plan_read_shares(bin.data(), ix, (uint64_t)n_reads, (uint32_t)n_gpus, J.first.data());
  J.prefix = prefix;
  const int rc = run_workers(n_gpus, "count", [&](Exchange &X) { worker(J, X); });
  if (!rc) XINFO("count (+ k_min SdBG) on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
}

extern "C" int mhb_seq2sdbg_run_multi(const mhb_seq2sdbg_opts *o, int n_gpus) {
  if (n_gpus <= 1) return mhb_seq2sdbg_run(o);
  if (int rc = seq2sdbg_check_opts(o)) return rc;
  const double t0 = now_s();
  if (seq2sdbg_prebuilt(o, t0)) return MHB_OK;
  if (o->need_mercy) {
    XINFO("--need_mercy without a graph built by the multi-GPU count: the mercy search runs on one GPU\n");
    return mhb_seq2sdbg_run(o);
  }
  if (n_gpus > kMaxRanks) return mhb_set_error(MHB_ERR_ARG, "at most %d GPUs of one node are supported", kMaxRanks);
  SeqJob J;
  J.k = o->k;
  J.prefix = o->output_prefix ? o->output_prefix : "";
  HostSeqs seqs;  // loaded before the fork: no CUDA in this process
  if (int rc = seq2sdbg_load(o, &seqs)) return rc;
  J.seqs = &seqs;
  J.first.resize(n_gpus + 1);
  plan_seq_shares(seqs.len.data(), seqs.size(), J.k, (uint32_t)n_gpus, J.first.data());
  uint64_t n_items = 0;
  for (uint32_t l : seqs.len) n_items += seq_items(l, J.k);
  XINFO("%zu sequences, %llu sort items; k = %u; %d GPUs\n", seqs.size(), (unsigned long long)n_items, J.k, n_gpus);
  const int rc = run_workers(n_gpus, "seq2sdbg", [&](Exchange &X) { s2s_worker(J, X); });
  if (!rc) XINFO("seq2sdbg on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
}

extern "C" int mhb_iterate_run_multi(const mhb_iterate_opts *o, int n_gpus) {
  if (n_gpus <= 1) return mhb_iterate_run(o);
  if (int rc = iterate_check_opts(o)) return rc;
  if (n_gpus > kMaxRanks) return mhb_set_error(MHB_ERR_ARG, "at most %d GPUs of one node are supported", kMaxRanks);
  if (int rc = iterate_check_args(o->k, o->step)) return rc;
  const double t0 = now_s();
  HostSeqs seqs;  // loaded before the fork: no CUDA in this process
  std::vector<uint32_t> bin;
  uint64_t n_reads = 0;
  if (int rc = iterate_load(o, &seqs, &bin, &n_reads)) return rc;
  ReadLibIndex ix;  // indexed serially: the workers are forked next
  if (index_read_lib(bin.data(), bin.size(), n_reads, 0, &ix, FixedCheck::kSerial))
    return mhb_set_error(MHB_ERR_IO, "%s ends inside a read", o->read_file);
  IterJob J;
  memset(&J.a, 0, sizeof(J.a));
  J.a.k = o->k;
  J.a.step = o->step;
  if (seqs.words.empty()) seqs.words.push_back(0);
  J.a.contig_words = seqs.words.data();
  J.a.contig_word_off = seqs.word_off.data();
  J.a.contig_len = seqs.len.data();
  J.a.n_contigs = seqs.size();
  J.a.bin = bin.data();
  J.a.bin_words = bin.size();
  J.a.n_reads = n_reads;
  J.first.resize(n_gpus + 1);
  plan_read_shares(bin.data(), ix, n_reads, (uint32_t)n_gpus, J.first.data());
  for (uint64_t f : J.first) J.word.push_back(ix.word_of(f));
  J.prefix = o->output_prefix;
  J.fd = open((J.prefix + ".edges.0").c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0666);
  if (J.fd < 0) return mhb_set_error(MHB_ERR_IO, "cannot open %s.edges.0 for writing", J.prefix.c_str());
  XINFO("%llu reads, %zu contigs; k = %u, step = %u; %d GPUs\n", (unsigned long long)n_reads, seqs.size(), o->k, o->step,
        n_gpus);
  const int rc = run_workers(n_gpus, "iterate", [&](Exchange &X) { iter_worker(J, X); });
  close(J.fd);
  if (!rc) XINFO("iterate on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
}

extern "C" int mhb_read2sdbg_run_multi(const mhb_read2sdbg_opts *o, int n_gpus) {
  if (n_gpus <= 1) return mhb_read2sdbg_run(o);
  if (n_gpus > kMaxRanks) return mhb_set_error(MHB_ERR_ARG, "at most %d GPUs of one node are supported", kMaxRanks);
  const double t0 = now_s();
  std::vector<uint32_t> bin;
  long long n_reads = 0;
  if (int rc = read2sdbg_load(o, &bin, &n_reads)) return rc;  // no CUDA in this process
  if (n_reads < n_gpus) {
    XINFO("%lld reads for %d GPUs: running on one GPU\n", n_reads, n_gpus);
    return read2sdbg_build(o, bin, n_reads, t0);
  }
  ReadLibIndex ix;  // indexed serially: the workers are forked next
  if (index_read_lib(bin.data(), bin.size(), (uint64_t)n_reads, 0, &ix, FixedCheck::kSerial))
    return mhb_set_error(MHB_ERR_IO, "%s.bin ends inside a read", o->read_lib_file);
  R2sJob J;
  memset(&J.a, 0, sizeof(J.a));
  J.a.k = o->k;
  J.a.m = o->m;
  J.a.bin = bin.data();
  J.a.bin_words = bin.size();
  J.a.n_reads = (uint64_t)n_reads;
  J.a.need_mercy = o->need_mercy;
  J.li = &ix;
  J.first.resize(n_gpus + 1);
  plan_read_shares(bin.data(), ix, (uint64_t)n_reads, (uint32_t)n_gpus, J.first.data());
  J.prefix = o->output_prefix ? o->output_prefix : "out";
  XINFO("read2sdbg: %lld reads; k = %u, m = %d; %d GPUs\n", n_reads, o->k, o->m, n_gpus);
  const int rc = run_workers(n_gpus, "read2sdbg", [&](Exchange &X) { r2s_worker(J, X); });
  if (!rc) XINFO("read2sdbg on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
}
