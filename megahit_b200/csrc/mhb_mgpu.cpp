// mhb_mgpu.cpp -- `count` on several GPUs of one node behind the file-level C ABI (mhb_count_run_multi, include/mhb.h).
//
// One worker PROCESS per GPU (forked before CUDA is touched; libmhb keeps per-process state: arena, kernel attributes),
// the same pipeline as megahit_b200/multigpu.py but with no Python, torch or NCCL underneath:
//   * records travel GPU -> GPU inside the fused partition + exchange kernel (mhb_partition_scatter storing into the
//     owners' receive buffers, opened through CUDA IPC);
//   * the small collectives (256-bin histograms, counters, IPC handles) go through one MAP_SHARED control block with a
//     process-shared barrier; the medium ones (tip edges, candidate reads, answer planes of the mercy searches, the
//     per-bucket tables) through files in /dev/shm written by one rank and read by the others;
//   * the plan of a stage (owner ranges from the all-gathered histograms) is computed by every rank from the same data
//     (plan_partition_host = the rule of k_plan_partition / multigpu.plan_ranges).
// The mercy searches are answered by the owners of the searched prefixes (mhb_mercy_probe_owned); the k_min SdBG is
// built in the same run because the solid edges are already on the devices.
//
// Reference behaviour reproduced: KmerCounter::Run (sorting/kmer_counter.cpp) + SeqToSdbg::Run with need_mercy
// (sorting/seq_to_sdbg.cpp) at k_min; files as edge_io_meta.h:25-44 / sdbg_meta.cpp:44-61 with num_files = n_gpus.
//
// `seq2sdbg` for k > k_min (mhb_seq2sdbg_run_multi) uses the same machinery: the parent loads every sequence and deals
// contiguous shares, balanced on their item count; each rank histograms its items' leading bytes, and after the plan
// extracts every item straight into its owner's receive buffer (mhb_s2s_extract_owners); the owners sort and emit as
// the count worker's SdBG stage does (sdbg_owner_stage, sdbg_merge_info).
//
// `iterate` (mhb_iterate_run_multi) deals contiguous read shares, balanced on bases; each rank builds the whole flank
// index, runs the single-GPU read pass over its share and sends its unique candidates to their owners, which sort and
// dedup them; the owners' ascending runs, written in rank order, are the single-GPU P.edges.0.
//
// `read2sdbg` (mhb_read2sdbg_run_multi) deals contiguous read shares too; each rank sends its stage-1 records to their
// owners in global read order (R2sShare::s1_send), the owners run stage 1 into planes of the whole library, every rank
// ORs all planes over its share's words, runs the mercy step over its share and sends its stage-2 items to their
// owners, which sort, collapse and emit as the single-GPU read2sdbg does.
#include <cuda_runtime.h>
#include <fcntl.h>
#include <pthread.h>
#include <signal.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <vector>

#include "mhb.h"
#include "mhb_bits.cuh"
#include "mhb_internal.h"

using namespace mhb;

namespace {

constexpr int kMaxRanks = 16;

#define XINFO(...)                                                         \
  do {                                                                     \
    fprintf(stderr, "INFO  %-30s: %4d - ", "megahit_b200", __LINE__);      \
    fprintf(stderr, __VA_ARGS__);                                          \
  } while (0)

double now_s() {
  timeval tv;
  gettimeofday(&tv, nullptr);
  return tv.tv_sec + tv.tv_usec * 1e-6;
}

// control block shared by the workers (anonymous MAP_SHARED mapping created before the fork)
struct Control {
  pthread_barrier_t bar;
  int world;
  char err[kMaxRanks][512];
  uint64_t hist[2][kMaxRanks][256];
  uint8_t ipc[4][kMaxRanks][64];
  uint64_t n_solid[kMaxRanks], n_tip[kMaxRanks], n_cand[kMaxRanks], n_mercy[kMaxRanks], n_records[kMaxRanks];
  uint64_t sdbg_totals[kMaxRanks][16];
  uint64_t has_tips[kMaxRanks];
  uint64_t n_edges[kMaxRanks], n_aligned[kMaxRanks];  // iterate
  int err_code[kMaxRanks];  // MHB_ERR_* of a failed rank
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
#define CKM(call)                                     \
  do {                                                \
    if ((call) != MHB_OK) fail("%s", mhb_last_error()); \
  } while (0)

// the device memory this worker holds through dev_alloc, and the most it has held
struct DevBytes {
  size_t live = 0, peak = 0;
  std::vector<std::pair<void *, size_t>> blocks;
} g_dev;

// the paths are resident only: a device allocation that fails is reported as MHB_ERR_NOMEM with its size
void *dev_alloc(size_t bytes) {
  void *p = nullptr;
  const cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    fail_nomem("cannot allocate %zu bytes of device memory", bytes);
  }
  CKC(e);
  g_dev.blocks.push_back({p, bytes});
  g_dev.live += bytes;
  g_dev.peak = std::max(g_dev.peak, g_dev.live);
  return p;
}
void dev_free(void *p) {
  for (auto &b : g_dev.blocks)
    if (b.first == p) {
      g_dev.live -= b.second;
      b = {nullptr, 0};
    }
  cudaFree(p);
}

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
  CKM(mhb_set_device(dev));
}

// device memory owned by a worker, released at its end
struct DevPool {
  std::vector<void *> ptrs;
  template <class T>
  T *get(size_t count) {
    void *p = dev_alloc(std::max<size_t>(count * sizeof(T), 256));
    ptrs.push_back(p);
    return (T *)p;
  }
  void drop(void *p) {
    for (auto &q : ptrs)
      if (q == p) {
        dev_free(q);
        q = nullptr;
      }
  }
  ~DevPool() {
    for (void *p : ptrs)
      if (p) dev_free(p);
  }
};

// ---- exchange of medium-sized host data through /dev/shm files: rank r writes <base>.<tag>.<r>, the others read it ----
struct Exchange {
  std::string base;
  int rank, world;
  Control *C;
  void barrier() { pthread_barrier_wait(&C->bar); }
  std::string path(const char *tag, int r) const { return base + "." + tag + "." + std::to_string(r); }
  void publish(const char *tag, const void *data, size_t bytes) {
    FILE *f = fopen(path(tag, rank).c_str(), "wb");
    if (!f) fail("cannot create %s", path(tag, rank).c_str());
    if (bytes && fwrite(data, 1, bytes, f) != bytes) {
      fclose(f);
      fail("short write on %s", path(tag, rank).c_str());
    }
    fclose(f);
  }
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
  void cleanup(const char *tag) { unlink(path(tag, rank).c_str()); }
};

// owner ranges from the all-gathered top-byte histograms: bound r = the byte value whose cumulative count is closest
// to r/world of the total, leaving at least one value for every later rank (k_plan_partition, multigpu.plan_ranges)
struct Plan {
  uint32_t bounds[kMaxRanks + 1];
  uint8_t owner[256];
  uint64_t recv_tot[kMaxRanks], send[kMaxRanks], my_off[kMaxRanks];
};
Plan plan_partition_host(const uint64_t (*hist)[256], int world, int rank) {
  Plan p;
  uint64_t cum[257];
  cum[0] = 0;
  for (int b = 0; b < 256; ++b) {
    uint64_t a = 0;
    for (int r = 0; r < world; ++r) a += hist[r][b];
    cum[b + 1] = cum[b] + a;
  }
  const uint64_t total = cum[256];
  p.bounds[0] = 0;
  for (int r = 1; r < world; ++r) {
    const uint32_t lo = p.bounds[r - 1] + 1, hi = 256 - (world - r);
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
    p.bounds[r] = best;
  }
  p.bounds[world] = 256;
  for (int o = 0; o < world; ++o) {
    for (uint32_t b = p.bounds[o]; b < p.bounds[o + 1]; ++b) p.owner[b] = (uint8_t)o;
    uint64_t before = 0, tot = 0, mine = 0;
    for (int r = 0; r < world; ++r) {
      uint64_t s = 0;
      for (uint32_t b = p.bounds[o]; b < p.bounds[o + 1]; ++b) s += hist[r][b];
      if (r < rank) before += s;
      if (r == rank) mine = s;
      tot += s;
    }
    p.recv_tot[o] = tot;
    p.send[o] = mine;
    p.my_off[o] = before;
  }
  return p;
}

struct PeerBuf {
  void *mine = nullptr;
  void *peer[kMaxRanks] = {nullptr};
  size_t bytes = 0;
};

// A receive buffer of `bytes` on every rank (the same size everywhere), exported through IPC slot `slot` and opened by
// every other rank.
void open_peers(Exchange &X, int slot, size_t bytes, PeerBuf *pb) {
  Control *C = X.C;
  const int W = X.world, r = X.rank;
  pb->bytes = bytes;
  pb->mine = dev_alloc(pb->bytes);
  CKM(mhb_ipc_export(pb->mine, C->ipc[slot][r]));
  X.barrier();
  for (int o = 0; o < W; ++o) {
    if (o == r) pb->peer[o] = pb->mine;
    else CKM(mhb_ipc_open(C->ipc[slot][o], &pb->peer[o]));
  }
}

// The exchange of one stage, up to the stores: all-gather the leading-byte histograms (d_hist on the device, or hist
// on the host), plan the owner ranges, allocate, export and open the receive buffers.  Returns the plan; *d_addr (256,
// in pool) = where this rank's records for owner o begin, *d_lut = the owner of every leading byte.
Plan open_receive(Exchange &X, int stage, const uint64_t *d_hist, uint32_t words, DevPool &pool, PeerBuf *pb,
                  uint64_t **d_addr, uint8_t **d_lut, const uint64_t *hist = nullptr) {
  Control *C = X.C;
  const int W = X.world, r = X.rank;
  if (hist) memcpy(C->hist[stage][r], hist, 256 * 8);
  else CKC(cudaMemcpy(C->hist[stage][r], d_hist, 256 * 8, cudaMemcpyDeviceToHost));
  X.barrier();
  const Plan P = plan_partition_host(C->hist[stage], W, r);
  uint64_t mx = 0;
  for (int o = 0; o < W; ++o) mx = std::max(mx, P.recv_tot[o]);
  open_peers(X, stage, (size_t)mx * words * 4 + 256, pb);
  uint64_t addr[256] = {0};
  for (int o = 0; o < W; ++o) addr[o] = (uint64_t)(uintptr_t)pb->peer[o] + P.my_off[o] * (uint64_t)words * 4;
  *d_addr = pool.get<uint64_t>(256);
  *d_lut = pool.get<uint8_t>(256);
  CKC(cudaMemcpy(*d_addr, addr, sizeof(addr), cudaMemcpyHostToDevice));
  CKC(cudaMemcpy(*d_lut, P.owner, 256, cudaMemcpyHostToDevice));
  return P;
}

// extract-side records -> the rank owning their leading byte; returns the local receive buffer and the plan
Plan partition_and_exchange(Exchange &X, int stage, uint32_t *recs, uint64_t n, uint32_t words, int top_byte, uint64_t *d_hist,
                            void *d_ws, size_t ws_bytes, DevPool &pool, PeerBuf *pb) {
  uint64_t *d_addr = nullptr;
  uint8_t *d_lut = nullptr;
  const Plan P = open_receive(X, stage, d_hist, words, pool, pb, &d_addr, &d_lut);
  CKM(mhb_partition_scatter(nullptr, recs, n, words, top_byte, d_lut, d_addr, d_ws, ws_bytes));
  CKC(cudaDeviceSynchronize());
  X.barrier();  // every rank's scatter has completed: my receive buffer is complete
  return P;
}

void close_peers(Exchange &X, PeerBuf *pb) {
  X.barrier();  // nobody reads or writes the buffers any more
  for (int o = 0; o < X.world; ++o)
    if (o != X.rank && pb->peer[o]) mhb_ipc_close(pb->peer[o]);
  X.barrier();
  if (pb->mine) dev_free(pb->mine);
  pb->mine = nullptr;
}

struct Job {
  uint32_t k;
  int32_t m;
  const uint32_t *bin;  // whole library (host, inherited by the workers)
  uint64_t n_reads;
  uint32_t read_len;
  std::string prefix;
};

void write_file(const std::string &path, const void *data, size_t bytes) {
  FILE *f = fopen(path.c_str(), "wb");
  if (!f) fail("cannot open %s for writing", path.c_str());
  if (bytes && fwrite(data, 1, bytes, f) != bytes) {
    fclose(f);
    fail("write to %s failed", path.c_str());
  }
  fclose(f);
}

// My P.sdbg.<r> and, for rank 0, my totals (C->sdbg_totals) and bucket table ("stab")
void sdbg_publish(Exchange &X, const uint64_t *totals, const std::vector<uint8_t> &sdbg_bytes,
                  const std::vector<uint64_t> &table, const std::string &prefix) {
  memcpy(X.C->sdbg_totals[X.rank], totals, 16 * 8);
  write_file(prefix + ".sdbg." + std::to_string(X.rank), sdbg_bytes.data(), sdbg_bytes.size());
  X.publish("stab", table.data(), 65536 * 32);
}

// ---- the owner side of the SdBG stage, the same in the count and seq2sdbg workers ----
// Sort and emit the n_own SdBG items of my receive buffer (my bucket range), close the exchange, write P.sdbg.<r> and
// publish my totals (C->sdbg_totals) and bucket table ("stab") for rank 0.
void sdbg_owner_stage(Exchange &X, PeerBuf *ps, uint64_t n_own, uint32_t k, const std::string &prefix, DevPool &pool) {
  const int r = X.rank;
  const uint32_t W2 = mhb_s2s_record_words(k), wpt = div_ceil(k, 16);
  uint8_t sbytes[72];
  const uint32_t n_ssort = mhb_s2s_sort_bytes(k, sbytes);
  std::vector<uint8_t> sdbg_bytes;
  std::vector<uint64_t> table(65536 * 4, 0);
  uint64_t totals[16] = {0};
  {
    uint32_t *d_tmp = pool.get<uint32_t>(n_own * W2 + 16);
    const size_t sb = mhb_sort_workspace_bytes(std::max<uint64_t>(n_own, 1), W2), eb = mhb_s2s_emit_scratch_bytes(n_own, k);
    void *d_s = pool.get<char>(sb);
    int in_b = 0;
    CKM(mhb_sort_records_relaxed(nullptr, (uint32_t *)ps->mine, d_tmp, n_own, W2, sbytes, n_ssort, nullptr, d_s, sb, &in_b));
    pool.drop(d_s);

    void *d_e = pool.get<char>(eb);
    const uint64_t cap_b = n_own * (4ull + 4ull * wpt) + 16;
    uint8_t *d_out = pool.get<uint8_t>(cap_b);
    uint64_t *d_table = pool.get<uint64_t>(65536 * 4), *d_tot = pool.get<uint64_t>(16);
    CKC(cudaMemset(d_table, 0, 65536 * 32));
    CKC(cudaMemset(d_tot, 0, 128));
    CKM(mhb_s2s_emit(nullptr, in_b ? d_tmp : (uint32_t *)ps->mine, n_own, k, d_out, cap_b, d_table, d_tot, d_e, eb));
    CKC(cudaMemcpy(totals, d_tot, sizeof(totals), cudaMemcpyDeviceToHost));
    if (totals[0] > cap_b) fail("internal: SdBG byte stream exceeds capacity");
    sdbg_bytes.resize(totals[0]);
    if (totals[0]) CKC(cudaMemcpy(sdbg_bytes.data(), d_out, totals[0], cudaMemcpyDeviceToHost));
    CKC(cudaMemcpy(table.data(), d_table, 65536 * 32, cudaMemcpyDeviceToHost));
    for (void *p : {(void *)d_tmp, d_e, (void *)d_out, (void *)d_table, (void *)d_tot}) pool.drop(p);
  }
  close_peers(X, ps);
  sdbg_publish(X, totals, sdbg_bytes, table, prefix);
}

// Rank 0, once every rank's sdbg_owner_stage is behind a barrier: the merged P.sdbg_info (sdbg_meta.cpp:44-61: records
// ordered by (file, starting offset), unused ones last) and the reference's closing lines of seq2sdbg.
void sdbg_merge_info(Exchange &X, uint32_t k, const std::string &prefix) {
  Control *C = X.C;
  const int W = X.world;
  FILE *g = fopen((prefix + ".sdbg_info").c_str(), "w");
  if (!g) fail("cannot open %s.sdbg_info", prefix.c_str());
  fprintf(g, "k %u\nwords_per_tip_label %u\nnum_buckets %d\nnum_files %d\n", k, div_ceil(k, 16), MHB_NUM_BUCKETS, W);
  int used = 0;
  uint64_t w_count[9] = {0}, items = 0, tips = 0, ones = 0;
  for (int o = 0; o < W; ++o) {
    const std::vector<char> v = X.fetch("stab", o);
    const uint64_t *t = (const uint64_t *)v.data();
    for (int b = 0; b < MHB_NUM_BUCKETS; ++b)
      if (t[4 * b + 1]) {
        fprintf(g, "%d %d %llu %llu %llu %llu\n", b, o, (unsigned long long)t[4 * b], (unsigned long long)t[4 * b + 1],
                (unsigned long long)t[4 * b + 2], (unsigned long long)t[4 * b + 3]);
        ++used;
      }
    items += C->sdbg_totals[o][1];
    tips += C->sdbg_totals[o][2];
    for (int i = 0; i < 9; ++i) w_count[i] += C->sdbg_totals[o][4 + i];
    ones += C->sdbg_totals[o][13];
  }
  for (int i = used; i < MHB_NUM_BUCKETS; ++i) fprintf(g, "18446744073709551615 18446744073709551615 0 0 0 0\n");
  fclose(g);
  XINFO("Number of $ A C G T A- C- G- T-:\n");
  XINFO("%llu %llu %llu %llu %llu %llu %llu %llu %llu\n", (unsigned long long)w_count[0], (unsigned long long)w_count[1],
        (unsigned long long)w_count[2], (unsigned long long)w_count[3], (unsigned long long)w_count[4],
        (unsigned long long)w_count[5], (unsigned long long)w_count[6], (unsigned long long)w_count[7],
        (unsigned long long)w_count[8]);
  XINFO("Total number of edges: %llu\n", (unsigned long long)items);
  XINFO("Total number of ONEs: %llu\n", (unsigned long long)ones);
  XINFO("Total number of $v edges: %llu\n", (unsigned long long)tips);
}

// ================================================================================================
// one worker = one GPU
// ================================================================================================
void worker(const Job &J, Exchange &X) {
  Control *C = X.C;
  const int W = X.world, r = X.rank;
  const uint32_t k = J.k, L = J.read_len;
  const int32_t m = J.m;
  bind_device(r, W);
  DevPool pool;
  const uint32_t WR = mhb_count_record_words(k), WE = mhb_words_per_edge(k), W2 = mhb_s2s_record_words(k);
  const uint32_t stride = 1 + div_ceil(L, 16);
  const uint64_t per = (J.n_reads + W - 1) / W;
  const uint64_t r0 = std::min<uint64_t>(J.n_reads, (uint64_t)r * per), r1 = std::min<uint64_t>(J.n_reads, r0 + per);
  const uint64_t nr = r1 - r0;                                    // my block of reads
  const uint64_t n = L >= k + 1 ? nr * (uint64_t)(L - k) : 0;     // my edge records
  const uint32_t *my_bin = J.bin + r0 * stride;
  uint8_t cbytes[72];
  const uint32_t n_csort = mhb_count_sort_bytes(k, cbytes);
  const int top = (int)(4 * WR - 1), top2 = (int)(4 * W2 - 1);

  // ---- reads to the device, extraction ----
  uint32_t *d_bin = pool.get<uint32_t>(nr * stride + 16);
  if (nr) CKC(cudaMemcpy(d_bin, my_bin, nr * stride * 4, cudaMemcpyHostToDevice));
  mhb_dev_reads reads;
  reads.bin = d_bin;
  reads.bin_words = nr * stride;
  reads.n_reads = nr;
  reads.fixed_len = L;
  reads.rec_off = nullptr;
  reads.edge_off = nullptr;
  uint32_t *d_a = pool.get<uint32_t>(n * WR + 16);
  uint64_t *d_hist = pool.get<uint64_t>(256);
  CKC(cudaMemset(d_hist, 0, 256 * 8));
  CKM(mhb_count_extract(nullptr, &reads, k, d_a, n, d_hist, top));
  size_t ws_bytes = mhb_sort_workspace_bytes(std::max<uint64_t>(n, 1), WR);
  void *d_ws = pool.get<char>(ws_bytes);
  PeerBuf pc;
  const Plan P = partition_and_exchange(X, 0, d_a, n, WR, top, d_hist, d_ws, ws_bytes, pool, &pc);
  pool.drop(d_a);
  pool.drop(d_ws);
  const uint64_t n_own = P.recv_tot[r];
  C->n_records[r] = n_own;

  // ---- count stage on the owned records ----
  const uint64_t cap = n_own / (uint64_t)std::max(1, m) + 1;
  uint32_t *d_edges = pool.get<uint32_t>(cap * WE + 16);
  uint8_t *d_aux = pool.get<uint8_t>(cap + 16);
  uint64_t *d_mul = pool.get<uint64_t>(65536);
  uint64_t *d_ns = pool.get<uint64_t>(8);
  CKC(cudaMemset(d_mul, 0, 65536 * 8));
  CKC(cudaMemset(d_ns, 0, 64));
  {
    uint32_t *d_tmp = pool.get<uint32_t>(n_own * WR + 16);
    if (mhb_count_hashed_supported(k, m) && !(getenv("MHB_COUNT_MODE") && !strcmp(getenv("MHB_COUNT_MODE"), "sort"))) {
      const size_t hb = mhb_count_hashed_workspace_bytes(std::max<uint64_t>(n_own, 1), k, m);
      void *d_h = pool.get<char>(hb);
      CKM(mhb_count_solid_hashed(nullptr, (uint32_t *)pc.mine, d_tmp, n_own, k, m, nullptr, d_edges, d_aux, cap, d_mul, d_ns, d_h, hb));
      CKC(cudaDeviceSynchronize());
      pool.drop(d_h);
    } else {
      const size_t sb = mhb_sort_workspace_bytes(std::max<uint64_t>(n_own, 1), WR), cb = mhb_count_solid_scratch_bytes(n_own);
      void *d_s = pool.get<char>(sb), *d_c = pool.get<char>(cb);
      int in_b = 0;
      CKM(mhb_sort_records_relaxed(nullptr, (uint32_t *)pc.mine, d_tmp, n_own, WR, cbytes, n_csort, nullptr, d_s, sb, &in_b));
      CKM(mhb_count_solid(nullptr, in_b ? d_tmp : (uint32_t *)pc.mine, n_own, k, m, d_edges, d_aux, cap, d_mul, d_ns, d_c, cb));
      CKC(cudaDeviceSynchronize());
      pool.drop(d_s);
      pool.drop(d_c);
    }
    pool.drop(d_tmp);
  }
  uint64_t n_solid = 0;
  CKC(cudaMemcpy(&n_solid, d_ns, 8, cudaMemcpyDeviceToHost));
  if (n_solid > cap) fail("internal: solid edges exceed capacity");
  C->n_solid[r] = n_solid;
  close_peers(X, &pc);  // the count records are gone: give the memory back before the SdBG stage
  {
    std::vector<uint64_t> h(65536);
    CKC(cudaMemcpy(h.data(), d_mul, 65536 * 8, cudaMemcpyDeviceToHost));
    X.publish("mul", h.data(), 65536 * 8);
  }

  // ---- mercy bookkeeping: tip edges of every rank -> per-read marks -> candidate reads ----
  uint64_t n_tip = 0;
  CKM(mhb_count_tip_edges(nullptr, d_aux, n_solid, &n_tip));
  {
    uint32_t *d_tips = pool.get<uint32_t>(n_tip * WE + 16);
    uint8_t *d_taux = pool.get<uint8_t>(n_tip + 16);
    CKC(cudaMemset(d_ns, 0, 8));
    CKM(mhb_compact_tip_edges(nullptr, d_edges, d_aux, n_solid, k, d_tips, d_taux, n_tip, d_ns));
    std::vector<char> buf(n_tip * (WE * 4 + 1));
    if (n_tip) {
      CKC(cudaMemcpy(buf.data(), d_tips, n_tip * WE * 4, cudaMemcpyDeviceToHost));
      CKC(cudaMemcpy(buf.data() + n_tip * WE * 4, d_taux, n_tip, cudaMemcpyDeviceToHost));
    }
    C->n_tip[r] = n_tip;
    X.publish("tips", buf.data(), buf.size());
    pool.drop(d_tips);
    pool.drop(d_taux);
  }
  X.barrier();
  uint64_t n_tip_all = 0;
  for (int o = 0; o < W; ++o) n_tip_all += C->n_tip[o];
  uint32_t *d_first = pool.get<uint32_t>(nr + 1), *d_last = pool.get<uint32_t>(nr + 1);
  uint64_t *d_cand = pool.get<uint64_t>(nr + 1);
  uint64_t n_cand = 0;
  {
    std::vector<uint32_t> te(n_tip_all * WE + 4);
    std::vector<uint8_t> ta(n_tip_all + 4);
    uint64_t at = 0;
    for (int o = 0; o < W; ++o) {
      const uint64_t c = C->n_tip[o];
      if (!c) continue;
      const std::vector<char> v = X.fetch("tips", o);
      memcpy(te.data() + at * WE, v.data(), c * WE * 4);
      memcpy(ta.data() + at, v.data() + c * WE * 4, c);
      at += c;
    }
    uint32_t *d_te = pool.get<uint32_t>(n_tip_all * WE + 16);
    uint8_t *d_ta = pool.get<uint8_t>(n_tip_all + 16);
    if (n_tip_all) {
      CKC(cudaMemcpy(d_te, te.data(), n_tip_all * WE * 4, cudaMemcpyHostToDevice));
      CKC(cudaMemcpy(d_ta, ta.data(), n_tip_all, cudaMemcpyHostToDevice));
    }
    const size_t tb = mhb_tipset_bytes(n_tip_all, k);
    void *d_tipset = pool.get<char>(tb);
    CKM(mhb_tipset_build(nullptr, d_te, d_ta, n_tip_all, k, d_tipset, tb, n_tip_all));
    CKM(mhb_count_mark_mercy(nullptr, &reads, k, d_tipset, tb, n_tip_all, d_first, d_last));
    const size_t cs = mhb_mercy_candidates_scratch_bytes(nr);
    void *d_cs = pool.get<char>(cs);
    CKM(mhb_mercy_candidates(nullptr, d_first, d_last, nr, d_cand, &n_cand, d_cs, cs));
    pool.drop(d_cs);
    pool.drop(d_tipset);
    pool.drop(d_te);
    pool.drop(d_ta);
  }
  C->n_cand[r] = n_cand;
  std::vector<uint64_t> cand_ids(n_cand);
  if (n_cand) CKC(cudaMemcpy(cand_ids.data(), d_cand, n_cand * 8, cudaMemcpyDeviceToHost));
  {  // number of reads with both marks set (the "(%d)" of the reference's log line) + my candidate reads, file orientation
    std::vector<uint32_t> f(nr), l(nr);
    if (nr) {
      CKC(cudaMemcpy(f.data(), d_first, nr * 4, cudaMemcpyDeviceToHost));
      CKC(cudaMemcpy(l.data(), d_last, nr * 4, cudaMemcpyDeviceToHost));
    }
    uint64_t ht = 0;
    for (uint64_t i = 0; i < nr; ++i) ht += f[i] != MHB_SENTINEL_OFFSET && l[i] != MHB_SENTINEL_OFFSET;
    C->has_tips[r] = ht;
    std::vector<uint32_t> cr(n_cand * stride);
    for (uint64_t c = 0; c < n_cand; ++c) memcpy(cr.data() + c * stride, my_bin + cand_ids[c] * stride, stride * 4);
    X.publish("cand", cr.data(), cr.size() * 4);
  }
  X.barrier();
  // ---- mercy edges: every rank answers, for the candidates of ALL ranks, the searches that land in its bucket range ----
  uint64_t n_cand_all = 0, cand_off[kMaxRanks + 1];
  for (int o = 0; o < W; ++o) {
    cand_off[o] = n_cand_all;
    n_cand_all += C->n_cand[o];
  }
  cand_off[W] = n_cand_all;
  uint64_t n_mercy = 0;
  uint32_t *d_all_edges = d_edges;  // solid + mercy edges, the sequences of the SdBG stage
  if (n_cand_all) {
    std::vector<uint32_t> all(n_cand_all * stride + 4);
    for (int o = 0; o < W; ++o)
      if (C->n_cand[o]) {
        const std::vector<char> v = X.fetch("cand", o);
        memcpy(all.data() + cand_off[o] * stride, v.data(), v.size());
      }
    uint32_t *d_call = pool.get<uint32_t>(n_cand_all * stride + 16);
    CKC(cudaMemcpy(d_call, all.data(), n_cand_all * stride * 4, cudaMemcpyHostToDevice));
    mhb_dev_reads greads = reads;
    greads.bin = d_call;
    greads.bin_words = n_cand_all * stride;
    greads.n_reads = n_cand_all;
    void *d_lut = pool.get<char>(mhb_edge_lut_bytes());
    CKM(mhb_edge_lut_build(nullptr, d_edges, n_solid, k, d_lut));
    const size_t pw_all = mhb_mercy_planes_words(n_cand_all, L);
    uint32_t *d_planes = pool.get<uint32_t>(pw_all);
    CKM(mhb_mercy_probe_owned(nullptr, &greads, nullptr, n_cand_all, L, k, d_edges, n_solid, d_lut, P.owner, (uint32_t)r, d_planes));
    std::vector<uint32_t> hp(pw_all);
    CKC(cudaMemcpy(hp.data(), d_planes, pw_all * 4, cudaMemcpyDeviceToHost));
    X.publish("planes", hp.data(), pw_all * 4);
    pool.drop(d_planes);
    pool.drop(d_lut);
    pool.drop(d_call);
    X.barrier();
    if (n_cand) {
      // the answers of every rank about MY candidates: rank s's file holds them at [cand_off[r], cand_off[r] + n_cand)
      const size_t pw1 = mhb_mercy_planes_words(1, L), pw_mine = pw1 * n_cand;
      std::vector<uint32_t> mine((size_t)W * pw_mine);
      for (int s = 0; s < W; ++s) {
        const std::vector<char> v = X.fetch("planes", s, cand_off[r] * pw1 * 4, pw_mine * 4);
        memcpy(mine.data() + (size_t)s * pw_mine, v.data(), pw_mine * 4);
      }
      uint32_t *d_mine = pool.get<uint32_t>(mine.size());
      CKC(cudaMemcpy(d_mine, mine.data(), mine.size() * 4, cudaMemcpyHostToDevice));
      const size_t ms = mhb_mercy_edges_scratch_bytes(n_cand, L) - mhb_edge_lut_bytes();
      void *d_ms = pool.get<char>(ms);
      CKM(mhb_mercy_count_planes(nullptr, &reads, d_cand, n_cand, L, k, d_mine, (uint32_t)W, pw_mine, &n_mercy, d_ms, ms));
      if (n_mercy) {
        if (n_solid + n_mercy > cap) {  // reads overlapping only at their ends: more mercy than solid edges
          uint32_t *big = pool.get<uint32_t>((n_solid + n_mercy) * WE + 16);
          CKC(cudaMemcpy(big, d_edges, n_solid * WE * 4, cudaMemcpyDeviceToDevice));
          d_all_edges = big;
        }
        CKM(mhb_mercy_edges_write(nullptr, &reads, d_cand, n_cand, L, k, d_all_edges + n_solid * WE, n_mercy, n_mercy, d_ms, ms));
        CKC(cudaDeviceSynchronize());
      }
      pool.drop(d_ms);
      pool.drop(d_mine);
    }
  }
  C->n_mercy[r] = n_mercy;
  X.barrier();

  // ---- SdBG stage over solid + mercy edges ----
  const uint64_t n_seqs = n_solid + n_mercy;
  uint64_t n_items = n_seqs * 6;
  mhb_dev_seqs seqs;
  memset(&seqs, 0, sizeof(seqs));
  seqs.words = d_all_edges;
  seqs.n_words = n_seqs * WE;
  seqs.n_seqs = n_seqs;
  seqs.fixed_len = k + 1;
  seqs.fixed_stride = WE;
  uint32_t *d_sa = pool.get<uint32_t>(n_items * W2 + 16);
  CKC(cudaMemset(d_hist, 0, 256 * 8));
  if (getenv("MHB_S2S_NO_PRUNE")) {
    CKM(mhb_s2s_extract(nullptr, &seqs, k, d_sa, n_items, d_hist, top2));
  } else {
    // the owned solid edges still carry the count stage's in/out flags: the $-items the emitter is certain to discard are
    // neither generated nor exchanged (mhb_s2s_extract_edges_pruned, DESIGN.md 4.7)
    CKC(cudaMemset(d_ns + 4, 0, 8));
    CKM(mhb_s2s_extract_edges_pruned(nullptr, d_all_edges, d_aux, n_seqs, n_solid, k, d_sa, n_items, d_ns + 4, d_hist, top2));
    uint64_t kept = 0;
    CKC(cudaMemcpy(&kept, d_ns + 4, 8, cudaMemcpyDeviceToHost));
    if (kept > n_items) fail("internal: pruned item count exceeds 6 per edge");
    n_items = kept;
  }
  ws_bytes = mhb_sort_workspace_bytes(std::max<uint64_t>(n_items, 1), W2);
  d_ws = pool.get<char>(ws_bytes);
  PeerBuf ps;
  const Plan P2 = partition_and_exchange(X, 1, d_sa, n_items, W2, top2, d_hist, d_ws, ws_bytes, pool, &ps);
  pool.drop(d_sa);
  pool.drop(d_ws);
  sdbg_owner_stage(X, &ps, P2.recv_tot[r], k, J.prefix, pool);

  // ---- files: my bucket range of the edges; the tables go to rank 0 ----
  std::vector<uint32_t> edges(n_solid * WE);
  if (n_solid) CKC(cudaMemcpy(edges.data(), d_edges, n_solid * WE * 4, cudaMemcpyDeviceToHost));
  write_file(J.prefix + ".edges." + std::to_string(r), edges.data(), edges.size() * 4);
  {
    std::vector<int64_t> cnt(65536, 0);
    for (uint64_t i = 0; i < n_solid; ++i) cnt[edges[i * WE] >> 16]++;
    X.publish("ecnt", cnt.data(), 65536 * 8);
    // `.cand`: my candidate reads in the REVERSED orientation KmerCounter holds them in (kmer_counter.cpp:387-401)
    std::vector<uint32_t> rec((size_t)n_cand * stride, 0);
    for (uint64_t c = 0; c < n_cand; ++c) {
      const uint32_t *src = my_bin + cand_ids[c] * stride;
      uint32_t *dst = rec.data() + c * stride;
      dst[0] = L;
      for (uint32_t i = 0; i < L; ++i) dst[1 + (i >> 4)] |= base_at(src + 1, L - 1 - i) << (30 - 2 * (i & 15));
    }
    X.publish("candrev", rec.data(), rec.size() * 4);
  }
  X.barrier();
  if (r == 0) {
    // merged P.edges.info (edge_io_meta.h:25-44): bucket -> (file = owner rank, offset inside that file, count)
    std::vector<std::vector<int64_t>> ec(W);
    uint64_t n_edges = 0;
    for (int o = 0; o < W; ++o) {
      const std::vector<char> v = X.fetch("ecnt", o);
      ec[o].assign((const int64_t *)v.data(), (const int64_t *)v.data() + 65536);
      n_edges += C->n_solid[o];
    }
    FILE *g = fopen((J.prefix + ".edges.info").c_str(), "w");
    if (!g) fail("cannot open %s.edges.info", J.prefix.c_str());
    fprintf(g, "kmer_size %u\nwords_per_edge %u\nnum_files %d\nnum_buckets %d\nnum_edges %llu\nis_sorted 1\n", k, WE, W,
            MHB_NUM_BUCKETS, (unsigned long long)n_edges);
    std::vector<int64_t> off(W, 0);
    for (int b = 0; b < MHB_NUM_BUCKETS; ++b) {
      int who = -1;
      for (int o = 0; o < W; ++o)
        if (ec[o][b]) {
          if (who >= 0) fail("bucket %d landed on two ranks", b);
          who = o;
        }
      if (who < 0) fprintf(g, "%d -1 0 0\n", b);
      else {
        fprintf(g, "%d %d %lld %lld\n", b, who, (long long)off[who], (long long)ec[who][b]);
        off[who] += ec[who][b];
      }
    }
    fclose(g);
    // P.cand (rank order = read order: the reads were dealt in contiguous blocks) and P.counting (global histogram)
    FILE *f = fopen((J.prefix + ".cand").c_str(), "wb");
    if (!f) fail("cannot open %s.cand", J.prefix.c_str());
    uint64_t n_cand_tot = 0, has_tips = 0, n_mercy_tot = 0;
    for (int o = 0; o < W; ++o) {
      const std::vector<char> v = X.fetch("candrev", o);
      if (!v.empty()) fwrite(v.data(), 1, v.size(), f);
      n_cand_tot += C->n_cand[o];
      has_tips += C->has_tips[o];
      n_mercy_tot += C->n_mercy[o];
    }
    fclose(f);
    std::vector<uint64_t> mul(65536, 0);
    for (int o = 0; o < W; ++o) {
      const std::vector<char> v = X.fetch("mul", o);
      const uint64_t *h = (const uint64_t *)v.data();
      for (int i = 0; i < 65536; ++i) mul[i] += h[i];
    }
    f = fopen((J.prefix + ".counting").c_str(), "w");
    if (!f) fail("cannot open %s.counting", J.prefix.c_str());
    for (int i = 1; i <= MHB_MAX_MUL; ++i) fprintf(f, "%d %lld\n", i, (long long)mul[i]);
    fclose(f);
    f = fopen((J.prefix + ".sdbg_fused").c_str(), "w");
    if (f) {
      fprintf(f, "%u 1 %d\n", k, W);
      fclose(f);
    }
    XINFO("Total number of candidate reads: %llu (%llu)\n", (unsigned long long)n_cand_tot, (unsigned long long)has_tips);
    XINFO("Total number of solid edges: %llu\n", (unsigned long long)n_edges);
    XINFO("Number of mercy edges: %llu\n", (unsigned long long)n_mercy_tot);
    sdbg_merge_info(X, k, J.prefix);  // merged P.sdbg_info
  }
  X.barrier();
  for (const char *t : {"mul", "tips", "cand", "planes", "ecnt", "stab", "candrev"}) X.cleanup(t);
}


// ================================================================================================
// seq2sdbg on several GPUs: the sequences are dealt in contiguous shares, the items meet on their owners
// ================================================================================================
uint64_t seq_items(uint32_t len, uint32_t k) { return len >= k + 1 ? 2ull * (len - k + 2) : 0; }

// n_ranks contiguous shares of the sequences, balanced on their items (plan_shares)
void plan_seq_shares(const uint32_t *len, uint64_t n, uint32_t k, uint32_t n_ranks, uint64_t *first) {
  plan_shares(n, n_ranks, [&](uint64_t i) { return seq_items(len[i], k); }, first);
}

struct SeqJob {
  uint32_t k;
  const HostSeqs *seqs;                // every sequence (host, inherited by the workers)
  std::vector<uint64_t> first;         // shares
  std::string prefix;
};

void s2s_worker(const SeqJob &J, Exchange &X) {
  const int W = X.world, r = X.rank;
  const uint32_t k = J.k, W2 = mhb_s2s_record_words(k);
  const int top2 = (int)(4 * W2 - 1);
  bind_device(r, W);
  DevPool pool;

  // ---- my share to the device ----
  const HostSeqs &S = *J.seqs;
  const uint64_t s0 = J.first[r], n = J.first[r + 1] - s0, w0 = S.word_off[s0], nw = S.word_off[s0 + n] - w0;
  std::vector<uint64_t> wo(n + 1), io(n + 1, 0);
  for (uint64_t i = 0; i <= n; ++i) wo[i] = S.word_off[s0 + i] - w0;
  for (uint64_t i = 0; i < n; ++i) io[i + 1] = io[i] + seq_items(S.len[s0 + i], k);
  const uint64_t n_items = io[n];
  uint32_t *d_words = pool.get<uint32_t>(nw + 16);
  uint64_t *d_wo = pool.get<uint64_t>(n + 1), *d_io = pool.get<uint64_t>(n + 1);
  uint32_t *d_len = pool.get<uint32_t>(n + 1);
  uint16_t *d_mult = pool.get<uint16_t>(n + 1);
  if (nw) CKC(cudaMemcpy(d_words, S.words.data() + w0, nw * 4, cudaMemcpyHostToDevice));
  CKC(cudaMemcpy(d_wo, wo.data(), (n + 1) * 8, cudaMemcpyHostToDevice));
  CKC(cudaMemcpy(d_io, io.data(), (n + 1) * 8, cudaMemcpyHostToDevice));
  if (n) {
    CKC(cudaMemcpy(d_len, S.len.data() + s0, n * 4, cudaMemcpyHostToDevice));
    CKC(cudaMemcpy(d_mult, S.mult.data() + s0, n * 2, cudaMemcpyHostToDevice));
  }
  mhb_dev_seqs seqs;
  memset(&seqs, 0, sizeof(seqs));
  seqs.words = d_words;
  seqs.n_words = nw;
  seqs.n_seqs = n;
  seqs.word_off = d_wo;
  seqs.len = d_len;
  seqs.item_off = d_io;
  seqs.mult = d_mult;

  // ---- leading-byte histogram of my items -> owner ranges, receive buffers ----
  uint64_t *d_hist = pool.get<uint64_t>(256);
  CKC(cudaMemset(d_hist, 0, 256 * 8));
  CKM(mhb_s2s_extract_range(nullptr, &seqs, k, nullptr, n_items, 0, 65535, nullptr, 0, d_hist, top2));
  PeerBuf ps;
  uint64_t *d_addr = nullptr;
  uint8_t *d_lut = nullptr;
  const Plan P = open_receive(X, 1, d_hist, W2, pool, &ps, &d_addr, &d_lut);

  // ---- every item straight into its owner's buffer ----
  uint64_t *d_cursor = pool.get<uint64_t>(kMaxRanks), *d_cap = pool.get<uint64_t>(kMaxRanks);
  CKC(cudaMemset(d_cursor, 0, kMaxRanks * 8));
  CKC(cudaMemcpy(d_cap, P.send, W * 8, cudaMemcpyHostToDevice));
  CKM(mhb_s2s_extract_owners(nullptr, &seqs, k, n_items, d_lut, d_addr, d_cursor, d_cap));
  uint64_t sent[kMaxRanks];
  CKC(cudaMemcpy(sent, d_cursor, W * 8, cudaMemcpyDeviceToHost));
  for (int o = 0; o < W; ++o)
    if (sent[o] != P.send[o])
      fail("internal: %llu items for rank %d, the histogram said %llu", (unsigned long long)sent[o], o,
           (unsigned long long)P.send[o]);
  for (void *p : {(void *)d_words, (void *)d_wo, (void *)d_io, (void *)d_len, (void *)d_mult}) pool.drop(p);
  X.barrier();  // every rank's stores have completed: my receive buffer is complete

  sdbg_owner_stage(X, &ps, P.recv_tot[r], k, J.prefix, pool);
  XINFO("rank %d: %llu sequences, %llu items sent, %llu owned; peak device memory %.1f MiB\n", r, (unsigned long long)n,
        (unsigned long long)n_items, (unsigned long long)P.recv_tot[r], g_dev.peak / 1048576.0);
  X.barrier();
  if (r == 0) sdbg_merge_info(X, k, J.prefix);
  X.barrier();
  X.cleanup("stab");
}

// ================================================================================================
// iterate on several GPUs: the reads are dealt in contiguous shares, the candidate sets meet on their owners
// ================================================================================================
// n_ranks contiguous shares of the n_reads reads, balanced on their bases: the mark pass scans every base of every read
void plan_read_shares(const uint32_t *bin, const ReadLibIndex &ix, uint64_t n_reads, uint32_t n_ranks, uint64_t *first) {
  plan_shares(n_reads, n_ranks, [&](uint64_t i) { return (uint64_t)bin[ix.word_of(i)]; }, first);
}

struct IterJob {
  mhb_iterate_args a;          // every contig and the whole `.bin` image (host, inherited by the workers)
  std::vector<uint64_t> first;  // read shares
  std::vector<uint64_t> word;   // first word of every share, n_ranks + 1 entries
  int fd;                       // P.edges.0, created empty by the parent
  std::string prefix;
};

#define CKI(call)                                      \
  do {                                                 \
    if (int rc_ = (call)) throw Fail{mhb_last_error(), rc_}; \
  } while (0)

void iter_worker(const IterJob &J, Exchange &X) {
  Control *C = X.C;
  const int W = X.world, r = X.rank;
  const uint32_t k = J.a.k, step = J.a.step, w2 = mhb_words_per_edge(k + step);
  const int top = (int)(4 * w2 - 1);
  bind_device(r, W);
  DevPool pool;

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
    CKI(iter_build_flanks(&a, &flanks));
    n_flanks = flanks.n;
    CKI(iter_collect(&a, flanks, &set, &n_set, &n_cand, &n_aligned));
    CKM(mhb_read_stream_stats(&n_chunks, nullptr, nullptr));
  }  // the flank table and the buffers of the read pass are freed: only the set stays

  // ---- every edge to the rank owning its leading byte ----
  uint64_t *d_hist = pool.get<uint64_t>(256);
  CKC(cudaMemset(d_hist, 0, 256 * 8));
  CKI(hist_byte(nullptr, set.as<uint32_t>(), n_set, w2, top, d_hist));
  const size_t ws_bytes = mhb_sort_workspace_bytes(std::max<uint64_t>(n_set, 1), w2);
  void *d_ws = pool.get<char>(ws_bytes);
  PeerBuf pb;
  const Plan P = partition_and_exchange(X, 0, set.as<uint32_t>(), n_set, w2, top, d_hist, d_ws, ws_bytes, pool, &pb);
  set.release();
  pool.drop(d_ws);

  // ---- the owner's sort + unique over what it received: an ascending run of the whole set ----
  const uint64_t n_own = P.recv_tot[r];
  uint64_t n_uniq = 0;
  std::vector<uint32_t> edges;
  {
    uint32_t *d_tmp = pool.get<uint32_t>(n_own * w2 + 16), *uniq = nullptr;
    CKI(iter_sort_unique((uint32_t *)pb.mine, d_tmp, n_own, k, step, &uniq, &n_uniq));
    edges.resize(n_uniq * w2);
    if (n_uniq) CKC(cudaMemcpy(edges.data(), uniq, n_uniq * w2 * 4, cudaMemcpyDeviceToHost));
    pool.drop(d_tmp);
  }
  close_peers(X, &pb);
  C->n_edges[r] = n_uniq;
  C->n_cand[r] = n_cand;
  C->n_aligned[r] = n_aligned;
  XINFO("rank %d: %llu reads (%s), %llu candidates, %llu unique sent, %llu received, %llu owned\n", r,
        (unsigned long long)a.n_reads, n_chunks ? (std::to_string(n_chunks) + " chunks").c_str() : "resident",
        (unsigned long long)n_cand, (unsigned long long)n_set, (unsigned long long)n_own, (unsigned long long)n_uniq);
  X.barrier();

  // ---- the owners' runs follow each other in rank order: one P.edges.0, as the single-GPU iterate writes it ----
  uint64_t before = 0;
  for (int o = 0; o < r; ++o) before += C->n_edges[o];
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
      n_edges += C->n_edges[o];
      aligned += C->n_aligned[o];
    }
    CKI(iterate_write_info(J.prefix, k + step, w2, n_edges));
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

// the owner plan of a stage from my 65536-bin bucket histogram (stages 0 and 1 use Control::hist[0] / [1])
Plan r2s_plan(Exchange &X, int stage, const uint64_t *h16, uint32_t words, DevPool &pool, PeerBuf *pb, uint64_t **d_addr,
              uint8_t **d_lut) {
  uint64_t h256[256];
  fold_bucket_hist(h16, h256);
  return open_receive(X, stage, nullptr, words, pool, pb, d_addr, d_lut, h256);
}

void r2s_worker(const R2sJob &J, Exchange &X) {
  Control *C = X.C;
  const int W = X.world, r = X.rank;
  const uint32_t k = J.a.k, W2 = mhb_s2s_record_words(k);
  const int32_t m = J.a.m;
  bind_device(r, W);
  DevPool pool;
  R2sShare sh;
  CKI(sh.load(&J.a, *J.li, J.first[r], J.first[r + 1]));
  std::vector<uint64_t> h16(65536);
  uint64_t n_s1_own = 0;

  // ---- stage 1: my records straight into their owners' buffers, in global read order; each owner's planes ----
  if (m > 1) {
    CKI(sh.s1_hist(h16.data()));
    const uint32_t RW = sh.s1_record_words();
    PeerBuf pr, pi;
    uint64_t *d_addr = nullptr;
    uint8_t *d_lut = nullptr;
    const Plan P = r2s_plan(X, 0, h16.data(), RW, pool, &pr, &d_addr, &d_lut);
    n_s1_own = P.recv_tot[r];
    if (n_s1_own > sh.s1_round_cap())
      fail_nomem("%llu stage-1 records in my bucket range, more than the %llu one pass sorts (%llu bytes)",
                 (unsigned long long)n_s1_own, (unsigned long long)sh.s1_round_cap(),
                 (unsigned long long)(n_s1_own * RW * 4));
    uint64_t mx = 0;
    for (int o = 0; o < W; ++o) mx = std::max(mx, P.recv_tot[o]);
    if (sh.s1_narrow()) open_peers(X, 2, (size_t)mx * 8 + 256, &pi);
    uint64_t rec_base[kMaxRanks], info_base[kMaxRanks];
    for (int o = 0; o < W; ++o) {
      rec_base[o] = (uint64_t)(uintptr_t)pr.peer[o];
      info_base[o] = (uint64_t)(uintptr_t)pi.peer[o];
    }
    CKI(sh.s1_send(P.owner, W, rec_base, sh.s1_narrow() ? info_base : nullptr, P.my_off, P.send));
    X.barrier();  // every rank's stores have completed: my receive buffer is complete
    CKI(sh.s1_own((uint32_t *)pr.mine, (uint64_t *)pi.mine, n_s1_own));
    close_peers(X, &pr);
    if (sh.s1_narrow()) close_peers(X, &pi);

    // ---- plane merge: the words of my share's reads, OR-ed over every rank's planes (read through CUDA IPC) ----
    CKM(mhb_ipc_export(sh.planes(), C->ipc[3][r]));
    X.barrier();
    for (int o = 0; o < W; ++o) {
      if (o == r) continue;
      void *peer = nullptr;
      CKM(mhb_ipc_open(C->ipc[3][o], &peer));
      CKI(sh.or_planes(peer));
      CKM(mhb_ipc_close(peer));
    }
    X.barrier();  // nobody reads my planes any more: the mercy step may add to them
  }

  // ---- the mercy step and the stage-2 item count over my share ----
  uint64_t n_items = 0, n_mercy = 0;
  CKI(sh.mercy_count(&n_items, &n_mercy));
  C->n_mercy[r] = n_mercy;

  // ---- stage 2: every item straight into its owner's buffer; the owner sorts, collapses and emits ----
  CKI(sh.s2_hist(h16.data()));
  PeerBuf ps;
  uint64_t *d_addr = nullptr;
  uint8_t *d_lut = nullptr;
  const Plan P2 = r2s_plan(X, 1, h16.data(), W2, pool, &ps, &d_addr, &d_lut);
  uint64_t base[kMaxRanks], sent[kMaxRanks];
  for (int o = 0; o < W; ++o) base[o] = (uint64_t)(uintptr_t)ps.peer[o] + P2.my_off[o] * (uint64_t)W2 * 4;
  CKI(sh.s2_send(P2.owner, W, base, P2.send, sent));
  for (int o = 0; o < W; ++o)
    if (sent[o] != P2.send[o])
      fail("internal: %llu stage-2 items for rank %d, the histogram said %llu", (unsigned long long)sent[o], o,
           (unsigned long long)P2.send[o]);
  X.barrier();  // every rank's stores have completed: my receive buffer is complete
  const uint64_t n_own = P2.recv_tot[r];
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> table;
  uint64_t totals[16];
  CKI(sh.s2_own((uint32_t *)ps.mine, n_own, &bytes, &table, totals));
  close_peers(X, &ps);
  sdbg_publish(X, totals, bytes, table, J.prefix);
  if (m > 1) {
    CKI(sh.counting(h16.data()));
    X.publish("mul", h16.data(), 65536 * 8);
  }
  XINFO("rank %d: %llu reads, %llu stage-1 records owned, %llu mercy edges, %llu items sent, %llu owned; peak device "
        "memory %.1f MiB\n", r, (unsigned long long)sh.n_reads(), (unsigned long long)n_s1_own, (unsigned long long)n_mercy,
        (unsigned long long)n_items, (unsigned long long)n_own, g_dev.peak / 1048576.0);
  X.barrier();
  if (r == 0) {
    if (m > 1) {  // Read2SdbgS1::Lv0Postprocess, read_to_sdbg_s1.cpp:557-566: the histogram over every owner's groups
      std::vector<uint64_t> mul(65536, 0);
      for (int o = 0; o < W; ++o) {
        const std::vector<char> v = X.fetch("mul", o);
        const uint64_t *h = (const uint64_t *)v.data();
        for (int i = 0; i < 65536; ++i) mul[i] += h[i];
      }
      FILE *f = fopen((J.prefix + ".counting").c_str(), "w");
      if (!f) throw Fail{"cannot open " + J.prefix + ".counting", MHB_ERR_IO};
      for (int i = 1; i <= MHB_MAX_MUL; ++i) fprintf(f, "%d %lld\n", i, (long long)mul[i]);
      fclose(f);
      if (J.a.need_mercy) {
        uint64_t n_mercy_tot = 0;
        for (int o = 0; o < W; ++o) n_mercy_tot += C->n_mercy[o];
        XINFO("Number mercy: %llu\n", (unsigned long long)n_mercy_tot);
      }
    }
    sdbg_merge_info(X, k, J.prefix);
  }
  X.barrier();
  for (const char *t : {"stab", "mul"}) X.cleanup(t);
}

// Forks one worker per rank around a fresh control block and waits for all of them.  A worker that dies would leave
// the others at a barrier: the first abnormal exit takes the rest down.  A failure is reported with the error code of
// the first failed rank that set one (MHB_ERR_CUDA otherwise) and every rank's message; the exchange files of `tags`
// are removed.
template <class Body>
int run_workers(int n, const char *what, std::initializer_list<const char *> tags, Body body) {
  Control *C = (Control *)mmap(nullptr, sizeof(Control), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  if (C == MAP_FAILED) return mhb_set_error(MHB_ERR_NOMEM, "mmap of the control block failed");
  memset(C, 0, sizeof(Control));
  C->world = n;
  pthread_barrierattr_t ba;
  pthread_barrierattr_init(&ba);
  pthread_barrierattr_setpshared(&ba, PTHREAD_PROCESS_SHARED);
  pthread_barrier_init(&C->bar, &ba, (unsigned)n);
  const std::string xbase = "/dev/shm/mhb_" + std::to_string((long long)getpid());
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
      Exchange X{xbase, r, n, C};
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
    for (int r = 0; r < n; ++r)
      for (const char *t : tags) unlink((xbase + "." + t + "." + std::to_string(r)).c_str());
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
  // the partitioned build deals contiguous blocks of a FIXED-length library to the GPUs; anything else (a truncated
  // image included, which the single-GPU count reports): one GPU.  Indexed serially: the workers are forked next.
  ReadLibIndex ix;
  const bool fixed = o->k >= 12 && n_reads >= n_gpus &&
                     !index_read_lib(bin.data(), bin.size(), n_reads, 0, &ix, FixedCheck::kSerial) && ix.fixed_len;
  const uint32_t L = ix.fixed_len;
  if (!fixed) {
    XINFO("variable-length or tiny library: running on one GPU\n");
    return mhb_count_run(o);
  }
  XINFO("%lld reads, %lld bases; k = %u, m = %d; %d GPUs\n", n_reads, total_bases, o->k, o->m, n_gpus);
  const Job J{o->k, o->m, bin.data(), (uint64_t)n_reads, L, prefix};
  const int rc = run_workers(n_gpus, "count", {"mul", "tips", "cand", "planes", "ecnt", "stab", "candrev"},
                             [&](Exchange &X) { worker(J, X); });
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
  const int rc = run_workers(n_gpus, "seq2sdbg", {"stab"}, [&](Exchange &X) { s2s_worker(J, X); });
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
  const int rc = run_workers(n_gpus, "iterate", {}, [&](Exchange &X) { iter_worker(J, X); });
  close(J.fd);
  if (!rc) XINFO("iterate on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
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
  const int rc = run_workers(n_gpus, "read2sdbg", {"stab", "mul"}, [&](Exchange &X) { r2s_worker(J, X); });
  if (!rc) XINFO("read2sdbg on %d GPUs done. Time elapsed: %.4f\n", n_gpus, now_s() - t0);
  return rc;
}

extern "C" int mhb_plan_r2s_owners(const uint64_t *hist16, uint32_t n_ranks, uint32_t *bucket_lo, uint32_t *bucket_hi) {
  if (!hist16 || !bucket_lo || !bucket_hi || n_ranks < 1 || n_ranks > (uint32_t)kMaxRanks)
    return mhb_set_error(MHB_ERR_ARG, "bad args");
  static uint64_t h[kMaxRanks][256];  // rank 0's histogram holds everything
  memset(h, 0, sizeof(h));
  fold_bucket_hist(hist16, h[0]);
  const Plan P = plan_partition_host(h, (int)n_ranks, 0);
  for (uint32_t o = 0; o < n_ranks; ++o) {
    bucket_lo[o] = P.bounds[o] << 8;
    bucket_hi[o] = (P.bounds[o + 1] << 8) - 1;
  }
  return MHB_OK;
}
