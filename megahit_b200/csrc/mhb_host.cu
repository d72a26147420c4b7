// mhb_host.cu -- host-level C ABI (include/mhb.h, layer 2): host buffers in, host buffers out.
// Orchestrates the device-level entry points on one GPU with a grow-only device arena that is kept
// between calls (so repeated steps do not pay cudaMalloc).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <optional>
#include <vector>

#include "mhb.h"
#include "mhb_bits.cuh"
#include "mhb_common.cuh"

using namespace mhb;

namespace {

struct Arena {
  char *base = nullptr;
  size_t cap = 0, used = 0;
  int reserve(size_t bytes) {
    used = 0;
    if (bytes <= cap) return MHB_OK;
    if (base) cudaFree(base);
    base = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc((void **)&base, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return mhb_set_error(MHB_ERR_NOMEM, "cudaMalloc of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
    }
    cap = bytes;
    return MHB_OK;
  }
  template <class T>
  T *take(size_t count) {
    char *p = base + used;
    used += pad256(count * sizeof(T));
    return reinterpret_cast<T *>(p);
  }
  // `bytes` from what is left of the arena, else a separate allocation in *own
  int take_or_alloc(size_t bytes, DevBuf *own, const char *what, char **p) {
    if (used + pad256(bytes) <= cap) {
      *p = take<char>(bytes);
      return MHB_OK;
    }
    CKR(own->alloc(bytes, what));
    *p = own->as<char>();
    return MHB_OK;
  }
};
Arena g_arena;

// what a plan may take: 92 % of the free device memory and of the arena, which the call may reallocate
double arena_avail_bytes() { return 0.92 * (double)(free_device_bytes() + g_arena.cap); }

}  // namespace

extern "C" int mhb_release(void) {
  if (g_arena.base) cudaFree(g_arena.base);
  g_arena = Arena();
  return MHB_OK;
}

size_t mhb_arena_bytes(void) { return g_arena.cap; }

int SdbgStitch::append(void *stream, const uint8_t *d_bytes, uint64_t cap_bytes, const uint64_t *d_table,
                       const uint64_t *d_totals) {
  cudaStream_t st = (cudaStream_t)stream;
  uint64_t rt[16];
  CK(cudaMemcpyAsync(rt, d_totals, sizeof(rt), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(round_table.data(), d_table, round_table.size() * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (rt[0] > cap_bytes) return mhb_set_error(MHB_ERR_NOMEM, "internal: SdBG byte stream exceeds capacity");
  const size_t base = bytes.size();
  bytes.resize(base + rt[0]);
  if (rt[0]) CK(cudaMemcpy(bytes.data() + base, d_bytes, rt[0], cudaMemcpyDeviceToHost));
  for (size_t b = 0; b < (size_t)MHB_NUM_BUCKETS; ++b)
    if (round_table[4 * b + 1]) {
      table[4 * b + 0] = round_table[4 * b + 0] + base;
      table[4 * b + 1] = round_table[4 * b + 1];
      table[4 * b + 2] = round_table[4 * b + 2];
      table[4 * b + 3] = round_table[4 * b + 3];
    }
  for (int i = 0; i < 16; ++i) tot[i] += rt[i];
  return MHB_OK;
}


// ------------------------------------------------------------------------------------------------
// The count stage on extracted records resident in d_a: either the LSD sort on every key byte followed by the
// run-length count, or - 8-byte records, the default where available - two partition passes + per-bucket hash
// aggregation (mhb_count_solid_hashed).  MHB_COUNT_MODE=sort forces the former.  Both leave the same edges / aux /
// histogram; both clobber d_a and d_b.
// ------------------------------------------------------------------------------------------------
CountWork count_work_plan(uint64_t n, uint32_t k, int32_t m) {
  static const bool force_sort = getenv("MHB_COUNT_MODE") && !strcmp(getenv("MHB_COUNT_MODE"), "sort");
  CountWork cw;
  cw.hashed = !force_sort && mhb_count_hashed_supported(k, m);
  if (cw.hashed) {
    cw.bytes = mhb_count_hashed_workspace_bytes(n, k, m);
    cw.ws_bytes = 0;
    cw.hist_byte = 5;
  } else {
    uint8_t sb[72];
    mhb_count_sort_bytes(k, sb);
    cw.ws_bytes = pad256(mhb_sort_workspace_bytes(n, count_record_words(k)));
    cw.bytes = cw.ws_bytes + pad256(mhb_count_solid_scratch_bytes(n));
    cw.hist_byte = sb[0];
  }
  return cw;
}
int run_count_stage(void *stream, const CountWork &cw, uint32_t *d_a, uint32_t *d_b, uint64_t n, uint32_t k, int32_t m,
                    const uint64_t *d_hist0, uint32_t *d_edges, uint8_t *d_aux, uint64_t cap_edges, uint64_t *d_mul_hist,
                    uint64_t *d_nsolid, char *work, double *pass_ms, uint32_t *n_passes) {
  cudaStream_t st = (cudaStream_t)stream;
  const uint32_t WR = count_record_words(k);
  if (cw.hashed) {
    if (n_passes) *n_passes = n ? 2 : 0;
    CKR(mhb_count_solid_hashed(st, d_a, d_b, n, k, m, d_hist0, d_edges, d_aux, cap_edges, d_mul_hist, d_nsolid, work, cw.bytes));
    if (pass_ms && n) {
      uint32_t np = 0, w = 0;
      uint64_t nr = 0;
      CKR(mhb_sort_pass_ms(0, pass_ms, 64, &np, &nr, &w));
    }
    return MHB_OK;
  }
  uint8_t sort_bytes[72];
  const uint32_t n_sort = mhb_count_sort_bytes(k, sort_bytes);
  if (n_passes) *n_passes = n ? n_sort : 0;
  int in_b = 0;
  CKR(mhb_sort_records_impl(st, d_a, d_b, n, WR, sort_bytes, n_sort, d_hist0, work, cw.ws_bytes, &in_b, pass_ms));
  return mhb_count_solid(st, in_b ? d_b : d_a, n, k, m, d_edges, d_aux, cap_edges, d_mul_hist, d_nsolid, work + cw.ws_bytes,
                         cw.bytes - cw.ws_bytes);
}

// bytes of device memory one round of `n` records needs besides the read library
size_t round_bytes(uint64_t n, uint32_t WR, uint32_t WE, int32_t m, uint32_t k) {
  const uint64_t cap_edges = n / (uint64_t)std::max(1, m) + 1;
  return 2 * pad256((size_t)n * WR * 4 + 16) + pad256(count_work_plan(n, k, m).bytes) +
         pad256((size_t)cap_edges * WE * 4) + pad256(cap_edges);
}

// ================================================================================================
// count (A13): one round over all records, or rounds over ranges of bucket ids
// ================================================================================================
namespace {
uint64_t g_round_limit = 0;      // count records per round; 0 = derive from free device memory
uint64_t g_s2s_round_limit = 0;  // seq2sdbg sort items per round; 0 = derive from free device memory
}  // namespace

uint64_t count_round_limit() { return g_round_limit; }

extern "C" int mhb_set_round_limit(uint64_t max_records_per_round) {
  g_round_limit = max_records_per_round;
  return MHB_OK;
}
extern "C" int mhb_set_s2s_round_limit(uint64_t max_items_per_round) {
  g_s2s_round_limit = max_items_per_round;
  return MHB_OK;
}

namespace {
// What a count that ran in one round over a resident library leaves on the device for the build's next stages
// (count_host_rounds with keep), all in the arena: the library, the solid edges and their flags, the multiplicity
// histogram and the candidate ids.  The arena from work_mark on, the round buffers, is free again.
struct CountOnDevice {
  bool valid = false;
  mhb_dev_reads reads;   // the whole library (set when need_mercy found reads)
  uint32_t max_len = 0;  // its longest read
  uint32_t *edges = nullptr;
  uint8_t *aux = nullptr;
  uint64_t cap_edges = 0;
  uint64_t *mul_hist = nullptr, *cand = nullptr;
  size_t work_mark = 0;
};
}  // namespace

// The reference plans Lv1 passes over bucket ranges so that every pass fits the memory it was given
// (base_engine.cpp:54-141 AdjustMemory, :254-281 Lv1FindEndBuckets); the output does not depend on where the pass
// boundaries fall.  Here a round = a contiguous range of bucket ids whose records fit in HBM next to the read library:
// extract that range -> sort -> solid edges -> append to the host result.  Rounds ascend, so the concatenated edges are
// sorted.  The mercy bookkeeping runs once at the end over the whole library, with a tip set built from the edges still
// on the device after a single round, or from the tip edges (aux != 0) of all rounds collected on the host.
//
// The plan is known without a pass when the library is resident and all records fit next to it (no round cap below
// them): one range over all bucket ids, extracted by mhb_count_extract.  Otherwise a histogram pass over the leading
// record byte (+ a pass for the second byte of the leading bytes that alone exceed a round) plans the ranges.
//
// stream: the `.bin` image stays in host memory and every pass over the reads (leading-byte histogram, second-byte
// histograms of oversized bytes, one pass per round, mercy marks) streams it through the device in chunks
// (init_read_stream); the round buffers get the memory the resident image would have taken.  A resident call switches
// to streaming when the library alone does not fit or when one bucket exceeds the round that fits next to it.
//
// check: how the index checks a library whose size matches fixed-length reads.  kSampled is verified on the device
// during the one pass only (mhb_check_fixed_len): a call known to take another plan (streamed, or a round cap below
// the records) indexes in full at once, and the call starts again with kFull when the check fails or when the one pass
// does not fit.  keep (may be NULL): a count that runs in one pass leaves its result on the device (keep->valid, the
// candidates found there too, MHB_H2D_CHUNKS pieces of the upload overlapping the extraction); the host result then
// holds the counts and times only.
static int count_host_rounds(const mhb_count_args *args, mhb_count_result *res, bool stream, FixedCheck check,
                             CountOnDevice *keep) {
  const uint32_t k = args->k;
  const int32_t m = args->m;
  const uint64_t n_reads = args->n_reads;
  const uint32_t WR = count_record_words(k), WE = words_per_edge(k);
  const int top_byte = (int)(4 * WR - 1);
  ReadLibIndex ix;
  if (stream) check = FixedCheck::kFull;
  CKR(index_read_lib(args->bin, args->bin_words, n_reads, k, &ix, check));
  if (check == FixedCheck::kSampled && ix.fixed_len && g_round_limit && ix.n_units > g_round_limit) {
    check = FixedCheck::kFull;
    CKR(index_read_lib(args->bin, args->bin_words, n_reads, k, &ix, check));
  }
  const uint64_t n = ix.n_units;
  res->words_per_edge = WE;
  res->n_edge_records = n;
  cudaStream_t st = 0;
  EventTimer t_all(st), t(st);
  t_all.start();
  auto restart = [&](bool streamed) {
    memset(res, 0, sizeof(*res));
    return count_host_rounds(args, res, streamed, FixedCheck::kFull, keep);
  };

  // fixed-length reads: C pieces (MHB_H2D_CHUNKS, default 4; 1 = one copy), the edges of piece i extracted while piece
  // i+1 is still crossing PCIe
  static const int h2d_pieces = getenv("MHB_H2D_CHUNKS") ? atoi(getenv("MHB_H2D_CHUNKS")) : 4;
  const bool pieces = keep && h2d_pieces > 1 && ix.fixed_len >= k + 1 && n_reads >= (uint64_t)h2d_pieces * 64;
  ChunkStream rs;
  const uint64_t chunk_cap = read_chunk_limit() ? read_chunk_limit() : read_chunk_auto_bytes();
  CKR(init_read_stream(&rs, args->bin, args->bin_words, n_reads, ix, stream ? chunk_cap : 0, pieces ? h2d_pieces : 1));
  const uint64_t chunk_reads = rs.max_chunk_units();  // reads the per-read arrays hold
  // besides the round buffers: the library (or its chunk slots), the mercy marks, the histograms and scalars
  size_t fixed = pad256(rs.device_bytes()) + pad256(65536 * 8) + pad256(256 * 8) + 4096;
  if (args->want_mercy) fixed += 2 * pad256((size_t)(chunk_reads + 1) * 4);
  const size_t cand_bytes = keep && args->want_mercy ? pad256((n_reads + 1) * 8) : 0;  // kept: the candidate ids
  bool one_pass = false;
  if (!stream && !(g_round_limit && n > g_round_limit)) {
    const size_t need = fixed + cand_bytes + round_bytes(n, WR, WE, m, k);
    one_pass = need <= g_arena.cap || (double)need <= arena_avail_bytes();
  }
  if (!one_pass && check == FixedCheck::kSampled && ix.fixed_len) return restart(stream);
  uint64_t max_records = n;
  if (!one_pass) {  // + the per-read counts of the extraction and the second-byte histograms
    fixed += pad256((chunk_reads + 2) * 8) + pad256(256 * 256 * 8) + pad256(256 * 8) + pad256(64) + 4096;
    max_records = g_round_limit;
    if (!max_records) {
      const size_t avail = (size_t)arena_avail_bytes();
      if (!stream && mhb_read_stream_decide(fixed, avail, 0, read_chunk_limit())) return restart(true);
      max_records = largest_round(n, fixed, avail, [&](uint64_t r) { return round_bytes(r, WR, WE, m, k); });
      if (!max_records)
        return mhb_set_error(MHB_ERR_NOMEM, "the read library's %s (%zu bytes) does not fit the device",
                             stream ? "chunk buffers" : "image", fixed);
    }
    max_records = std::min<uint64_t>(std::max<uint64_t>(max_records, 1), std::max<uint64_t>(n, 1));
  } else {
    fixed += cand_bytes;
  }
  const bool on_device = keep && one_pass;
  const uint64_t cap_edges = max_records / (uint64_t)std::max(1, m) + 1;
  CKR(g_arena.reserve(fixed + round_bytes(max_records, WR, WE, m, k)));

  char *d_lib = g_arena.take<char>(rs.device_bytes());
  uint64_t *d_per_read = nullptr, *d_sub = nullptr;  // second-byte histograms of the oversized leading bytes
  if (!one_pass) {
    d_per_read = g_arena.take<uint64_t>(chunk_reads + 2);
    d_sub = g_arena.take<uint64_t>(256 * 256);
  }
  uint64_t *d_mul_hist = g_arena.take<uint64_t>(65536);
  uint64_t *d_hist0 = g_arena.take<uint64_t>(256);
  uint64_t *d_hist_top = g_arena.take<uint64_t>(256);
  uint64_t *d_scalars = g_arena.take<uint64_t>(8);  // [0] n_solid, [1] round total, [2] a read of another length
  uint32_t *d_first = nullptr, *d_last = nullptr;
  if (args->want_mercy) {
    d_first = g_arena.take<uint32_t>(chunk_reads + 1);
    d_last = g_arena.take<uint32_t>(chunk_reads + 1);
  }
  uint64_t *d_cand = on_device && cand_bytes ? g_arena.take<uint64_t>(n_reads + 1) : nullptr;
  uint32_t *d_edges = g_arena.take<uint32_t>((size_t)cap_edges * WE);
  uint8_t *d_aux = g_arena.take<uint8_t>(cap_edges);
  const size_t work_mark = g_arena.used;  // the round buffers come last: the build's later stages reuse them
  uint32_t *d_a = g_arena.take<uint32_t>((size_t)max_records * WR + 4);
  uint32_t *d_b = g_arena.take<uint32_t>((size_t)max_records * WR + 4);
  const CountWork cw = count_work_plan(max_records, k, m);
  char *d_work = g_arena.take<char>(cw.bytes);
  const size_t work_bytes = g_arena.used - work_mark;

  t.start();
  CKR(rs.bind(d_lib, st));
  CK(cudaMemsetAsync(d_mul_hist, 0, 65536 * 8, st));
  CK(cudaMemsetAsync(d_hist_top, 0, 256 * 8, st));
  res->t_h2d_ms = t.stop();

  // one pass over the reads: fn(view of a chunk, its first read), once per chunk
  auto each_chunk = [&](const std::function<int(const mhb_dev_reads &, uint64_t)> &fn) -> int {
    return rs.pass(st, [&](const ChunkView &c) {
      mhb_dev_reads v;
      v.bin = c.words;
      v.bin_words = c.n_words;
      v.n_reads = c.n;
      v.fixed_len = ix.fixed_len;
      v.rec_off = c.at<uint64_t>(0);
      v.edge_off = c.at<uint64_t>(1);
      return fn(v, c.first);
    });
  };

  // ---- plan: one range over all bucket ids, or histogram of the leading byte over the whole library (+ of the second
  // byte inside every leading byte that alone exceeds a round), then greedy contiguous ranges of bucket ids ----
  BucketRanges ranges = {{0u, 65535u}};
  std::vector<uint64_t> pre;  // prefix sums of the bucket histogram the plan read
  if (!one_pass) {
    t.start();
    const int rc = plan_bucket_passes(
        max_records,
        [&](uint64_t *h256) {
          CKR(each_chunk([&](const mhb_dev_reads &v, uint64_t) {
            return mhb_count_extract_range(st, &v, k, 0, 65535, 0, d_per_read, nullptr, d_hist_top, top_byte, d_scalars + 1);
          }));
          CK(cudaMemcpyAsync(h256, d_hist_top, 256 * 8, cudaMemcpyDeviceToHost, st));
          CK(cudaStreamSynchronize(st));
          return MHB_OK;
        },
        [&](const std::vector<uint32_t> &over, uint64_t *h16) {  // every oversized byte in the same pass
          if (WR * 4 < 2)
            return mhb_set_error(MHB_ERR_NOMEM, "leading byte 0x%02x exceeds a round and the record has no second byte", over[0]);
          CK(cudaMemsetAsync(d_sub, 0, over.size() * 256 * 8, st));
          CKR(each_chunk([&](const mhb_dev_reads &v, uint64_t) {
            for (size_t j = 0; j < over.size(); ++j)
              CKR(mhb_count_extract_range(st, &v, k, over[j] << 8, (over[j] << 8) | 255u, 0, d_per_read, nullptr,
                                          d_sub + j * 256, top_byte - 1, d_scalars + 1));
            return MHB_OK;
          }));
          for (size_t j = 0; j < over.size(); ++j)
            CK(cudaMemcpyAsync(h16 + (size_t)over[j] * 256, d_sub + j * 256, 256 * 8, cudaMemcpyDeviceToHost, st));
          CK(cudaStreamSynchronize(st));
          return MHB_OK;
        },
        &ranges, &pre);
    if (rc == -1) {
      // one bucket exceeds the round that fits next to the resident library: stream it, which leaves more room
      if (!stream && !g_round_limit) return restart(true);
      return MHB_ERR_NOMEM;
    }
    CKR(rc);
    res->t_extract_ms = t.stop();
  }

  const bool tips_on_device = ranges.size() == 1;  // the only round's edges are still on the device for the mercy step
  const bool verify = check == FixedCheck::kSampled && ix.fixed_len;  // one pass only (restarted above otherwise)
  const uint64_t piece_units = pieces ? ix.fixed_len - k : 0;         // edges per read of the uploaded pieces
  std::vector<uint32_t> h_tip_edges;                                  // otherwise the tip edges (aux != 0) of every round
  std::vector<uint8_t> h_tip_aux, h_aux;
  uint64_t n_solid_total = 0;
  for (const auto &rg : ranges) {
    // ---- extract the range: all records at once, or per view, count its in-range records, then write them at the
    // round's cursor ----
    t.start();
    CK(cudaMemsetAsync(d_hist0, 0, 256 * 8, st));
    CK(cudaMemsetAsync(d_scalars, 0, 24, st));
    uint64_t n_round = n;
    if (one_pass) {
      CKR(each_chunk([&](const mhb_dev_reads &v, uint64_t r0) {
        return mhb_count_extract(st, &v, k, d_a + r0 * piece_units * WR, pieces ? v.n_reads * piece_units : n, d_hist0, cw.hist_byte);
      }));
      if (verify) CKR(mhb_check_fixed_len(st, (const uint32_t *)d_lib, n_reads, ix.fixed_len, d_scalars + 2));
    } else {
      if (pre[rg.second + 1] == pre[rg.first]) continue;  // known empty from the histograms: no pass
      n_round = 0;
      CKR(each_chunk([&](const mhb_dev_reads &v, uint64_t) {
        uint64_t n_view = 0;
        CKR(mhb_count_extract_range(st, &v, k, rg.first, rg.second, 0, d_per_read, nullptr, nullptr, 0, d_scalars + 1));
        CK(cudaMemcpyAsync(&n_view, d_scalars + 1, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (n_round + n_view > max_records)
          return mhb_set_error(MHB_ERR_NOMEM, "internal: round of %llu records exceeds its plan", (unsigned long long)(n_round + n_view));
        if (n_view)
          CKR(mhb_count_extract_range(st, &v, k, rg.first, rg.second, 1, d_per_read, d_a + n_round * WR, d_hist0, cw.hist_byte, nullptr));
        n_round += n_view;
        return MHB_OK;
      }));
      if (n_round == 0) continue;
    }
    if (!on_device) {  // kept on the device: extraction and count are timed as one, with no synchronisation between
      res->t_extract_ms += t.stop();
      t.start();
    }
    // ---- sort / partition + solid edges ----
    CKR(run_count_stage(st, cw, d_a, d_b, n_round, k, m, d_hist0, d_edges, d_aux, cap_edges, d_mul_hist, d_scalars, d_work,
                        one_pass && !keep ? res->sort_pass_ms : nullptr, one_pass && !keep ? &res->n_sort_passes : nullptr));
    uint64_t sc[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(sc, d_scalars, sizeof(sc), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (verify && sc[2]) return restart(false);  // not fixed-length after all: the indexed path
    const uint64_t n_solid = sc[0];
    res->t_count_ms += t.stop();
    if (n_solid > cap_edges) return mhb_set_error(MHB_ERR_NOMEM, "internal: solid edges exceed capacity");
    n_solid_total += n_solid;
    ++res->n_rounds;
    if (on_device) continue;
    // ---- append to the host result ----
    t.start();
    const size_t e0 = (size_t)(n_solid_total - n_solid) * WE;
    uint32_t *edges = (uint32_t *)realloc(res->edges, std::max<size_t>(1, (e0 + (size_t)n_solid * WE) * 4));
    if (!edges) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
    res->edges = edges;
    if (n_solid) {
      CK(cudaMemcpyAsync(res->edges + e0, d_edges, (size_t)n_solid * WE * 4, cudaMemcpyDeviceToHost, st));
      if (args->want_mercy && !tips_on_device) {
        h_aux.resize(n_solid);
        CK(cudaMemcpyAsync(h_aux.data(), d_aux, n_solid, cudaMemcpyDeviceToHost, st));
      }
      CK(cudaStreamSynchronize(st));
    }
    if (args->want_mercy && !tips_on_device)
      for (uint64_t i = 0; i < n_solid; ++i)
        if (h_aux[i]) {
          h_tip_edges.insert(h_tip_edges.end(), res->edges + e0 + i * WE, res->edges + e0 + (i + 1) * WE);
          h_tip_aux.push_back(h_aux[i]);
        }
    res->t_d2h_ms += t.stop();
  }
  res->n_solid = n_solid_total;
  for (uint32_t p = 0; p < res->n_sort_passes; ++p) res->t_sort_ms += res->sort_pass_ms[p];

  // ---- mercy bookkeeping over the whole library: the marks, and on the device the candidates too ----
  std::vector<uint32_t> h_first, h_last;
  if (args->want_mercy && n_reads) {
    t.start();
    uint64_t n_tip = h_tip_aux.size();
    if (tips_on_device) CKR(mhb_count_tip_edges(st, d_aux, n_solid_total, &n_tip));
    const size_t ts_bytes = mhb_tipset_bytes(n_tip, k);
    const size_t list_bytes = pad256(h_tip_edges.size() * 4 + 16) + pad256(h_tip_aux.size() + 16);
    const size_t cs_bytes = on_device ? mhb_mercy_candidates_scratch_bytes(n_reads) : 0;
    // the round buffers are free now
    DevBuf own;
    char *d_tmp = (char *)d_a;
    if (list_bytes + pad256(ts_bytes) + pad256(cs_bytes) + 256 > work_bytes) {
      CKR(own.alloc(list_bytes + pad256(ts_bytes) + pad256(cs_bytes) + 256, "count: mercy tip set"));
      d_tmp = own.as<char>();
    }
    const uint32_t *d_tip_edges = tips_on_device ? d_edges : (uint32_t *)d_tmp;
    const uint8_t *d_tip_aux = tips_on_device ? d_aux : (uint8_t *)(d_tmp + pad256(h_tip_edges.size() * 4 + 16));
    char *d_tips = d_tmp + list_bytes, *d_cs = d_tips + pad256(ts_bytes);
    int rc = MHB_OK;
    if (!h_tip_aux.empty()) {
      if (cudaMemcpyAsync((void *)d_tip_edges, h_tip_edges.data(), h_tip_edges.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
          cudaMemcpyAsync((void *)d_tip_aux, h_tip_aux.data(), n_tip, cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = mhb_set_error(MHB_ERR_CUDA, "tip edge upload failed");
    }
    if (!rc)
      rc = mhb_tipset_build(st, d_tip_edges, d_tip_aux, tips_on_device ? n_solid_total : n_tip, k, d_tips, ts_bytes, n_tip);
    if (!rc && on_device) {
      rc = each_chunk([&](const mhb_dev_reads &v, uint64_t) {
        keep->reads = v;
        return mhb_count_mark_mercy(st, &v, k, d_tips, ts_bytes, n_tip, d_first, d_last);
      });
      if (!rc) rc = mhb_mercy_candidates(st, d_first, d_last, n_reads, d_cand, &res->n_cand, d_cs, cs_bytes);
    } else if (!rc) {
      // per view: marks into the view-sized first/last arrays, copied to the host arrays at the view's first read; the
      // host arrays are zeroed while the first marks run
      rc = each_chunk([&](const mhb_dev_reads &v, uint64_t r0) {
        CKR(mhb_count_mark_mercy(st, &v, k, d_tips, ts_bytes, n_tip, d_first, d_last));
        h_first.resize(n_reads);
        h_last.resize(n_reads);
        cudaMemcpyAsync(h_first.data() + r0, d_first, v.n_reads * 4, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(h_last.data() + r0, d_last, v.n_reads * 4, cudaMemcpyDeviceToHost, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) return mhb_set_error(MHB_ERR_CUDA, "mercy marking failed: %s", cudaGetErrorString(cudaGetLastError()));
        return MHB_OK;
      });
    }
    own.release();
    if (rc) return rc;
    res->t_mercy_ms = t.stop();
  }
  if (stream) {
    double h2d_ms = 0;
    mhb_read_stream_times(&h2d_ms, nullptr, nullptr, nullptr);
    res->t_h2d_ms = h2d_ms;
  }
  if (on_device) {
    keep->valid = true;
    keep->max_len = ix.fixed_len;
    for (uint64_t r = 0; !ix.fixed_len && r < n_reads; ++r) keep->max_len = std::max(keep->max_len, args->bin[ix.rec_off[r]]);
    keep->edges = d_edges;
    keep->aux = d_aux;
    keep->cap_edges = cap_edges;
    keep->mul_hist = d_mul_hist;
    keep->cand = d_cand;
    keep->work_mark = g_arena.used = work_mark;
    res->t_total_ms = t_all.stop();
    return MHB_OK;
  }

  if (!res->edges) res->edges = (uint32_t *)malloc(1);
  if (!res->edges) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  std::vector<uint64_t> h_hist(65536);
  CK(cudaMemcpy(h_hist.data(), d_mul_hist, 65536 * 8, cudaMemcpyDeviceToHost));
  for (int i = 0; i <= MHB_MAX_MUL; ++i) res->counting[i] = (int64_t)h_hist[i];
  if (args->want_mercy) {  // kmer_counter.cpp:390-401
    std::vector<uint64_t> ids;
    for (uint64_t r = 0; r < n_reads; ++r) {
      const uint32_t f = h_first[r], l = h_last[r];
      if (f != MHB_SENTINEL_OFFSET && l != MHB_SENTINEL_OFFSET) {
        ++res->n_has_tips;
        if (l > f) ids.push_back(r);
      }
    }
    res->n_cand = ids.size();
    res->cand_ids = (uint64_t *)malloc(std::max<size_t>(1, ids.size() * 8));
    if (!ids.empty()) memcpy(res->cand_ids, ids.data(), ids.size() * 8);
  }
  res->t_total_ms = t_all.stop();
  return MHB_OK;
}

// ================================================================================================
// count
// ================================================================================================
extern "C" int mhb_count_host(const mhb_count_args *args, mhb_count_result *res) {
  if (!args || !res) return mhb_set_error(MHB_ERR_ARG, "null args");
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k;
  if (k < 1 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "kmer size %u out of range", k);
  if (mhb_device_count() == 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  read_stream_stats_reset();
  // A13: when one pass over all records does not fit the device (or the caller capped the round size), the stage runs
  // in rounds over ranges of bucket ids; a chunk cap streams the library through those rounds
  return count_host_rounds(args, res, read_chunk_limit() != 0, FixedCheck::kFull, nullptr);
}

// ================================================================================================
// seq2sdbg, out of core (A13): rounds over ranges of the leading record byte, sequences resident or streamed
// ================================================================================================
namespace {
uint64_t g_s2s_chunk_limit = 0;  // sequence chunk / mercy segment cap in bytes; 0 = stream only what does not fit
StreamStats g_s2s_st, g_mercy_st;
uint64_t g_s2s_rounds = 0;

size_t s2s_round_bytes(uint64_t n, uint32_t W, uint32_t k) {
  return 2 * pad256((size_t)n * W * 4 + 16) + pad256(mhb_s2s_sort_workspace_bytes(n, k)) +
         pad256(mhb_s2s_emit_scratch_bytes(n, k)) + pad256((size_t)n * (4ull + 4ull * words_per_tip_label(k)) + 16);
}
// what the rounds keep next to the sequences: bucket table, the histogram of the sort's first byte, totals and, to plan
// rounds, the top-byte histogram, the second-byte rows of oversized bytes and the cursor
size_t s2s_table_bytes(bool plan) {
  return pad256((size_t)MHB_NUM_BUCKETS * 4 * 8) + pad256(256 * 8) + pad256(16 * 8) +
         (plan ? pad256(256 * 8) + pad256(256 * 256 * 8) + pad256(64) + 8192 : 4096);
}

// The layout of mhb_s2s_args: item offsets (exclusive prefix of 2 * (len - k + 2) over sequences of len >= k + 1) and
// whether it is the fixed-length, gap-free layout of edges (every sequence L0 >= k + 1 bases at stride ceil(L0 / 16)).
struct SeqLayout {
  std::vector<uint64_t> item_off;
  uint64_t n_items = 0, n_words = 0;
  bool fixed = false;
  uint32_t L0 = 0;
};
void seq_layout(const uint64_t *word_off, const uint32_t *len, uint64_t ns, uint32_t k, SeqLayout *ly) {
  ly->item_off.resize(ns + 1);
  ly->n_items = 0;
  ly->fixed = ns > 0;
  ly->L0 = ns ? len[0] : 0;
  for (uint64_t s = 0; s < ns; ++s) {
    ly->item_off[s] = ly->n_items;
    const uint32_t L = len[s];
    if (L >= k + 1) ly->n_items += 2ull * (L - k + 2);
    if (L != ly->L0 || word_off[s] != s * (uint64_t)div_ceil(ly->L0, 16)) ly->fixed = false;
  }
  ly->item_off[ns] = ly->n_items;
  if (ly->L0 < k + 1) ly->fixed = false;
  ly->n_words = ns ? word_off[ns] : 0;
}
// upload bytes of one sequence in a chunk: its words, its multiplicity and, unless fixed-length, word_off + item_off +
// len
uint64_t seq_extra_bytes(bool fixed) { return fixed ? 2 : 8 + 8 + 4 + 2; }
void plan_seq_chunks(const uint64_t *word_off, const SeqLayout &ly, uint64_t ns, uint64_t max_bytes, std::vector<uint64_t> *first) {
  plan_chunks(ly.fixed ? nullptr : word_off, div_ceil(ly.L0, 16), seq_extra_bytes(ly.fixed), ns, max_bytes, first);
}

// The sequences of one seq2sdbg driver call as its round loop sees them, one pass at a time.  Either mhb_s2s_args
// sequences, or `.edges`-layout records (stride words_per_edge(k), the multiplicity in the low 16 bits of the last
// word) in host memory or already on the device, the latter possibly with the count's flags of its first records.
// Host data goes through a ChunkStream, resident or streamed in chunks that end on sequence boundaries.  A chunk of
// fixed-length sequences carries their words and multiplicities and is viewed with fixed_len set; a variable-length
// one also carries word_off and item_off rebased to the chunk, and len; one of edge records carries the records.
class SeqSource {
 public:
  SeqSource(const mhb_s2s_args *a, const SeqLayout &ly) : a_(a), ly_(&ly), ns_(a->n_seqs) {}
  // n edge records of k in host memory, or on the device with the flags of the first n_aux of them (aux may be NULL)
  SeqSource(const uint32_t *edges, uint64_t n, uint32_t k, bool on_device, const uint8_t *aux = nullptr, uint64_t n_aux = 0)
      : edges_(edges), ns_(n), stride_(words_per_edge(k)), k1_(k + 1), on_device_(on_device), aux_(aux), n_aux_(n_aux) {}
  // max_chunk_bytes = 0: resident
  int init(uint64_t max_chunk_bytes) {
    if (on_device_) {
      g_s2s_st.chunks = 0;
      return MHB_OK;
    }
    ChunkStream::Input in;
    in.n = ns_;
    std::vector<uint64_t> first;
    if (edges()) {
      in.image = edges_;
      in.stride = stride_;
      if (max_chunk_bytes) plan_chunks(nullptr, stride_, 0, ns_, max_chunk_bytes, &first);
    } else {
      in.image = a_->words;
      in.word_off = a_->word_off;
      if (max_chunk_bytes) plan_seq_chunks(a_->word_off, *ly_, ns_, max_chunk_bytes, &first);
      if (!max_chunk_bytes || !ly_->fixed) {  // the resident form keeps all four
        in.side[0] = {a_->word_off, 0};
        in.side[1] = {ly_->item_off.data(), 0};
        in.side[2] = {a_->len, 4};
      }
      in.side[3] = {a_->mult, 2};
    }
    in.words = in.word_of(ns_);
    return cs_.init(in, std::move(first), &g_s2s_st);
  }
  static size_t resident_bytes(uint64_t ns, uint64_t n_words) {
    return ChunkStream::image_bytes(n_words) + 2 * ChunkStream::side_bytes(ns, 0) + ChunkStream::side_bytes(ns, 4) +
           ChunkStream::side_bytes(ns, 2);
  }
  size_t resident_size() const {
    return edges() ? ChunkStream::image_bytes(ns_ * stride_) : resident_bytes(ns_, ly_->n_words);
  }
  size_t device_bytes() const { return on_device_ ? 0 : cs_.device_bytes(); }
  uint64_t n_chunks() const { return cs_.n_chunks(); }
  bool on_device() const { return on_device_; }
  bool pruned() const { return aux_ != nullptr; }  // the extraction may skip the $-items the flags rule out
  // device_bytes() bytes; the resident form uploads the sequences there on st
  int bind(char *dev, cudaStream_t st) { return on_device_ ? MHB_OK : cs_.bind(dev, st); }
  // fn(view, items of the chunk) once per chunk, in order, on st
  int pass(cudaStream_t st, const std::function<int(const mhb_dev_seqs &, uint64_t)> &fn) {
    if (on_device_) return fn(view({0, 0, ns_, edges_, ns_ * stride_, {}}), 6 * ns_);
    return cs_.pass(st, [&](const ChunkView &c) { return fn(view(c), items(c.first, c.first + c.n)); });
  }
  // pruned(): the items of the device records that the flags do not rule out (mhb_s2s_extract_edges_pruned)
  int extract_pruned(cudaStream_t st, uint32_t *records, uint64_t capacity, uint64_t *cursor, uint64_t *hist, int hist_byte) const {
    return mhb_s2s_extract_edges_pruned(st, edges_, aux_, ns_, n_aux_, k1_ - 1, records, capacity, cursor, hist, hist_byte);
  }

 private:
  bool edges() const { return stride_ != 0; }  // the records form
  uint64_t items(uint64_t b, uint64_t e) const { return edges() ? 6 * (e - b) : ly_->item_off[e] - ly_->item_off[b]; }
  mhb_dev_seqs view(const ChunkView &c) const {
    mhb_dev_seqs v;
    v.words = c.words;
    v.n_words = c.n_words;
    v.n_seqs = c.n;
    v.fixed_len = edges() ? k1_ : ly_->fixed ? ly_->L0 : 0;
    v.word_off = c.at<uint64_t>(0);
    v.item_off = c.at<uint64_t>(1);
    v.len = c.at<uint32_t>(2);
    v.mult = c.at<uint16_t>(3);
    v.fixed_stride = stride_;
    return v;
  }
  const mhb_s2s_args *a_ = nullptr;
  const SeqLayout *ly_ = nullptr;
  const uint32_t *edges_ = nullptr;
  uint64_t ns_ = 0;
  uint32_t stride_ = 0, k1_ = 0;
  bool on_device_ = false;
  const uint8_t *aux_ = nullptr;
  uint64_t n_aux_ = 0;
  ChunkStream cs_;
};

// the smallest device footprint of the rounds over resident sequences: the sequences, the tables and a one-item round
size_t s2s_resident_round_bytes(size_t resident, uint32_t k) {
  return resident + s2s_table_bytes(true) + s2s_round_bytes(1, s2s_record_words(k), k);
}
// what one pass over n items of device records takes: the tables, the item buffers, the workspace and the stream
size_t s2s_device_bytes(uint64_t n, uint32_t k) {
  return s2s_table_bytes(false) + 2 * pad256((size_t)n * s2s_record_words(k) * 4 + 16) +
         pad256(mhb_s2s_sort_emit_workspace_bytes(n, k)) + pad256(n * (4ull + 4ull * words_per_tip_label(k)) + 16);
}

// Where a seq2sdbg driver leaves the SdBG: the item stream in `user` when that holds user_cap bytes, else malloc'ed;
// the bucket table in table (host, 65536 x 4); the emitter's totals; the items it sorted (fewer than the layout's
// when pruned) and its times
struct S2sOut {
  uint64_t *table = nullptr;
  uint8_t *user = nullptr;
  uint64_t user_cap = 0;
  uint8_t *bytes = nullptr;
  uint64_t tot[16] = {0};
  uint64_t n_sorted = 0;
  double t_extract_ms = 0, t_sort_ms = 0, t_emit_ms = 0, t_d2h_ms = 0, t_total_ms = 0;
};
}  // namespace

// Same idea as count_host_rounds: the stage runs once per contiguous range of leading record bytes (a (k-1)-mer group,
// and a bucket, never spans two ranges): extract the range -> sort -> emit -> append the item bytes and that range's
// rows of the bucket table to the result.  Ranges ascend, so the concatenated stream is in bucket order.  Every
// extraction is one pass over the sequences (SeqSource).  one_pass (resident sequences whose items all fit next to
// them): the one range over all bucket ids, known without a pass, extracted by mhb_s2s_extract (edge records with flags:
// mhb_s2s_extract_edges_pruned), its output straight into the result.  Otherwise the top-byte histogram and the
// second-byte histograms of the leading bytes that alone exceed a round plan the ranges, and each non-empty round's
// chunks append their in-range items at its cursor.  Records on the device run in one pass next to what the arena
// already holds, in its free part or in an allocation of their own.
static int s2s_host_rounds(uint32_t k, SeqSource &src, uint64_t n_items, uint64_t max_items, bool one_pass, S2sOut *out) {
  const uint32_t W = s2s_record_words(k), WPT = words_per_tip_label(k);
  const int top_byte = (int)(4 * W - 1);
  cudaStream_t st = 0;
  EventTimer t_all(st), t(st);
  t_all.start();

  const size_t fixed_b = src.device_bytes() + s2s_table_bytes(!one_pass);
  if (one_pass) {
    max_items = n_items;
  } else {
    if (!max_items) {
      const size_t avail = (size_t)arena_avail_bytes();
      max_items = largest_round(n_items, fixed_b, avail, [&](uint64_t n) { return s2s_round_bytes(n, W, k); });
      if (!max_items)
        return mhb_set_error(MHB_ERR_NOMEM, "the sequences%s alone (%zu bytes) do not fit the device",
                             src.n_chunks() ? "' chunk buffers" : "", fixed_b);
    }
    max_items = std::min<uint64_t>(max_items, std::max<uint64_t>(n_items, 1));
  }
  Arena area, *ar = &g_arena;
  DevBuf own;
  if (src.on_device()) {
    area.cap = s2s_device_bytes(max_items, k);
    CKR(g_arena.take_or_alloc(area.cap, &own, "build: SdBG stage", &area.base));
    ar = &area;
  } else {
    CKR(g_arena.reserve(fixed_b + s2s_round_bytes(max_items, W, k)));
  }
  char *d_seqs = ar->take<char>(src.device_bytes());
  uint64_t *d_table = ar->take<uint64_t>((size_t)MHB_NUM_BUCKETS * 4);
  uint64_t *d_hist0 = ar->take<uint64_t>(256);
  uint64_t *d_totals = ar->take<uint64_t>(16);
  uint64_t *d_hist_top = nullptr, *d_sub = nullptr, *d_cursor = nullptr;  // to plan rounds
  if (!one_pass) {
    d_hist_top = ar->take<uint64_t>(256);
    d_sub = ar->take<uint64_t>(256 * 256);
  }
  if (!one_pass || src.pruned()) d_cursor = ar->take<uint64_t>(8);
  uint32_t *d_a = ar->take<uint32_t>((size_t)max_items * W + 4);
  uint32_t *d_b = ar->take<uint32_t>((size_t)max_items * W + 4);
  // sort + emit workspace (at most the sort workspace plus the emit scratch s2s_round_bytes reserves)
  const size_t ws_bytes = mhb_s2s_sort_emit_workspace_bytes(max_items, k);
  // worst case bytes per sort item: 2 + 2 + 4*WPT (every item a large-multiplicity tip)
  const uint64_t cap_bytes = max_items * (4ull + 4ull * WPT) + 16;
  char *d_ws = ar->take<char>(ws_bytes);
  uint8_t *d_bytes = ar->take<uint8_t>(cap_bytes);
  CKR(src.bind(d_seqs, st));

  // ---- plan: one range over all bucket ids, or from the two histogram passes, as in count_host_rounds ----
  BucketRanges ranges = {{0u, 65535u}};
  std::vector<uint64_t> pre;  // prefix sums of the bucket histogram the plan read
  if (!one_pass) {
    t.start();
    const int rc = plan_bucket_passes(
        max_items,
        [&](uint64_t *h256) {
          CK(cudaMemsetAsync(d_hist_top, 0, 256 * 8, st));
          CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
            return mhb_s2s_extract_range(st, &s, k, nullptr, n, 0, 65535, nullptr, 0, d_hist_top, top_byte);
          }));
          CK(cudaMemcpyAsync(h256, d_hist_top, 256 * 8, cudaMemcpyDeviceToHost, st));
          CK(cudaStreamSynchronize(st));
          return MHB_OK;
        },
        [&](const std::vector<uint32_t> &over, uint64_t *h16) {
          CK(cudaMemsetAsync(d_sub, 0, 256 * 256 * 8, st));
          CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
            for (uint32_t b : over)
              CKR(mhb_s2s_extract_range(st, &s, k, nullptr, n, b << 8, (b << 8) | 255u, nullptr, 0, d_sub + (size_t)b * 256,
                                        top_byte - 1));
            return MHB_OK;
          }));
          CK(cudaMemcpyAsync(h16, d_sub, 256 * 256 * 8, cudaMemcpyDeviceToHost, st));
          CK(cudaStreamSynchronize(st));
          return MHB_OK;
        },
        &ranges, &pre);
    CKR(rc == -1 ? MHB_ERR_NOMEM : rc);
    out->t_extract_ms = t.stop();
  }

  std::optional<SdbgStitch> stitch;  // rounds: their output stitched together (4 MB of tables, not made for one pass)
  if (!one_pass) stitch.emplace();
  uint64_t tot[16] = {0};  // one pass: the emitter's totals
  // the time since the last lap into *ms; device records are timed as one, with no synchronisation before the totals
  auto lap = [&](double *ms) {
    if (src.on_device()) return;
    *ms += t.stop();
    t.start();
  };
  for (const auto &rg : ranges) {
    const uint64_t planned = one_pass ? n_items : pre[rg.second + 1] - pre[rg.first];  // the range's items
    if (!one_pass && planned == 0) continue;
    ++g_s2s_rounds;
    t.start();
    CK(cudaMemsetAsync(d_hist0, 0, 256 * 8, st));
    uint64_t n_round = n_items;
    if (one_pass && !src.pruned()) {
      CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
        return mhb_s2s_extract(st, &s, k, d_a, n, d_hist0, mhb_s2s_sort_hist_byte(max_items, k));
      }));
    } else {
      CK(cudaMemsetAsync(d_cursor, 0, 64, st));
      if (one_pass)
        CKR(src.extract_pruned(st, d_a, max_items, d_cursor, d_hist0, mhb_s2s_sort_hist_byte(max_items, k)));
      else
        CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
          return mhb_s2s_extract_range(st, &s, k, d_a, n, rg.first, rg.second, d_cursor, max_items, d_hist0,
                                       mhb_s2s_sort_hist_byte(max_items, k));
        }));
      CK(cudaMemcpyAsync(&n_round, d_cursor, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
    lap(&out->t_extract_ms);
    if (src.pruned() ? n_round > planned : n_round != planned)
      return mhb_set_error(MHB_ERR_NOMEM, "internal: round of %llu items, %llu planned", (unsigned long long)n_round,
                           (unsigned long long)planned);
    out->n_sorted += n_round;
    // the histogram is of the byte a sort of max_items items starts with: pass it only if this round's sort does too
    const bool hist_ok = mhb_s2s_sort_hist_byte(n_round, k) == mhb_s2s_sort_hist_byte(max_items, k);
    // sort and emit in one call (the bucket kernel emits every bucket it sorts): t_sort_ms carries both
    CKR(mhb_s2s_sort_emit(st, d_a, d_b, n_round, k, hist_ok ? d_hist0 : nullptr, d_bytes, cap_bytes, d_table, d_totals, d_ws,
                          ws_bytes));
    lap(&out->t_sort_ms);
    if (one_pass) {
      CK(cudaMemcpyAsync(tot, d_totals, sizeof(tot), cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(out->table, d_table, (size_t)MHB_NUM_BUCKETS * 32, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (tot[0] > cap_bytes) return mhb_set_error(MHB_ERR_NOMEM, "internal: SdBG byte stream exceeds capacity");
    } else {
      CKR(stitch->append(st, d_bytes, cap_bytes, d_table, d_totals));
    }
    out->t_emit_ms += t.stop();
  }
  memcpy(out->tot, one_pass ? tot : stitch->tot, sizeof(out->tot));
  if (!one_pass) memcpy(out->table, stitch->table.data(), (size_t)MHB_NUM_BUCKETS * 32);
  const uint64_t n_bytes = out->tot[0];
  out->bytes = out->user && out->user_cap >= n_bytes ? out->user : (uint8_t *)malloc(std::max<size_t>(1, n_bytes));
  if (!out->bytes) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  t.start();
  if (n_bytes && one_pass) CK(cudaMemcpy(out->bytes, d_bytes, n_bytes, cudaMemcpyDeviceToHost));
  else if (n_bytes) memcpy(out->bytes, stitch->bytes.data(), n_bytes);
  out->t_d2h_ms = t.stop();
  out->t_total_ms = t_all.stop();
  return MHB_OK;
}

// A13 for sequences in host memory: items that do not fit the device at once (or a caller-imposed cap) -> rounds over
// leading-byte ranges; the sequences are streamed when a chunk cap is set or when they leave no room for even a
// one-item round
static int s2s_run(uint32_t k, SeqSource &src, uint64_t n_items, S2sOut *out) {
  g_s2s_st = StreamStats();
  g_s2s_rounds = 0;
  const size_t need = src.resident_size() + s2s_table_bytes(false) + s2s_round_bytes(n_items, s2s_record_words(k), k);
  bool rounds = g_s2s_round_limit && n_items > g_s2s_round_limit;
  if (!rounds && need > g_arena.cap) {
    rounds = (double)need > arena_avail_bytes();
  }
  const bool stream = g_s2s_chunk_limit != 0 ||
                      (rounds && mhb_read_stream_decide(s2s_resident_round_bytes(src.resident_size(), k), (uint64_t)arena_avail_bytes(), 0, 0));
  CKR(src.init(stream ? (g_s2s_chunk_limit ? g_s2s_chunk_limit : read_chunk_auto_bytes()) : 0));
  return s2s_host_rounds(k, src, n_items, g_s2s_round_limit, !rounds && !stream, out);
}

// a round of a multi-GPU SdBG owner holds what one of s2s_host_rounds does: its receive buffer and the sort buffer,
// the sort + emit workspace (at most the sort workspace plus the emit scratch) and the SdBG bytes
extern "C" uint64_t mhb_sdbg_round_budget(uint64_t avail_bytes, uint64_t fixed_bytes, uint32_t k, uint64_t n_total) {
  if (k < 9 || k > MHB_MAX_K) return 0;
  const uint32_t W = s2s_record_words(k);
  uint64_t cap = largest_round(std::max<uint64_t>(n_total, 1), fixed_bytes, avail_bytes,
                               [&](uint64_t n) { return s2s_round_bytes(n, W, k); });
  if (cap && g_s2s_round_limit) cap = std::min(cap, g_s2s_round_limit);
  return cap;
}

extern "C" int mhb_set_s2s_chunk_limit(uint64_t bytes) {
  g_s2s_chunk_limit = bytes;
  return MHB_OK;
}
uint64_t s2s_chunk_limit() { return g_s2s_chunk_limit; }

extern "C" int mhb_s2s_stream_stats(int mercy, uint64_t *n_chunks, uint64_t *n_passes, uint64_t *n_rounds, uint64_t *h2d_bytes) {
  const StreamStats &s = mercy ? g_mercy_st : g_s2s_st;
  if (n_chunks) *n_chunks = s.chunks;
  if (n_passes) *n_passes = s.passes;
  if (n_rounds) *n_rounds = mercy ? 0 : g_s2s_rounds;
  if (h2d_bytes) *h2d_bytes = s.h2d_bytes;
  return MHB_OK;
}

extern "C" int mhb_s2s_stream_times(int mercy, double *h2d_ms, double *kernel_ms, double *fill_ms, double *pass_ms) {
  const StreamStats &s = mercy ? g_mercy_st : g_s2s_st;
  if (h2d_ms) *h2d_ms = s.copy_ms;
  if (kernel_ms) *kernel_ms = s.kernel_ms;
  if (fill_ms) *fill_ms = s.fill_ms;
  if (pass_ms) *pass_ms = s.pass_ms;
  return MHB_OK;
}

extern "C" int mhb_plan_seq_chunks(const uint64_t *word_off, const uint32_t *len, uint64_t n_seqs, uint32_t k,
                                   uint64_t max_chunk_bytes, uint64_t *first_seq_out, uint32_t cap_out) {
  if ((n_seqs && (!word_off || !len)) || max_chunk_bytes == 0) {
    mhb_set_error(MHB_ERR_ARG, "bad chunk plan arguments");
    return -1;
  }
  SeqLayout ly;
  seq_layout(word_off, len, n_seqs, k, &ly);
  std::vector<uint64_t> first;
  plan_seq_chunks(word_off, ly, n_seqs, max_chunk_bytes, &first);
  if (first_seq_out) {
    if (first.size() > cap_out) {
      mhb_set_error(MHB_ERR_ARG, "chunk plan needs %llu entries, room for %u", (unsigned long long)first.size(), cap_out);
      return -1;
    }
    memcpy(first_seq_out, first.data(), first.size() * 8);
  }
  return (int)(first.size() - 1);
}

extern "C" int mhb_selftest_s2s_stream_decide(uint64_t n_seqs, uint64_t n_words, uint32_t k, uint64_t free_bytes,
                                              uint64_t chunk_limit, uint64_t *resident_bytes, int *stream) {
  *resident_bytes = s2s_resident_round_bytes(SeqSource::resident_bytes(n_seqs, n_words), k);
  *stream = mhb_read_stream_decide(*resident_bytes, (uint64_t)(0.92 * (double)free_bytes), 0, chunk_limit);
  return MHB_OK;
}

// ================================================================================================
// seq2sdbg
// ================================================================================================
extern "C" int mhb_s2s_host(const mhb_s2s_args *args, mhb_s2s_result *res) {
  if (!args || !res) return mhb_set_error(MHB_ERR_ARG, "null args");
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k;
  if (k < 9 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "kmer size must be >= 9!");
  if (mhb_device_count() == 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  res->words_per_tip_label = words_per_tip_label(k);
  SeqLayout ly;
  seq_layout(args->word_off, args->len, args->n_seqs, k, &ly);
  res->n_records = ly.n_items;
  SeqSource src(args, ly);
  S2sOut out;
  out.table = res->bucket_table;
  CKR(s2s_run(k, src, ly.n_items, &out));
  res->bytes = out.bytes;
  set_sdbg_totals(res, out.tot);
  res->t_extract_ms = out.t_extract_ms;
  res->t_sort_ms = out.t_sort_ms;
  res->t_emit_ms = out.t_emit_ms;
  res->t_total_ms = out.t_total_ms;
  return MHB_OK;
}

// ================================================================================================
// mercy edges from host buffers, the sorted edges resident or streamed in leading-byte segments
// ================================================================================================
namespace {
// device bytes of a streamed search besides its two segment slots: candidate reads, scratch and the answer planes
size_t mercy_stream_fixed_bytes(uint64_t n_reads, uint64_t cand_words, uint32_t max_len) {
  const size_t bin_bytes = (cand_words * 4 + 15) & ~(size_t)15;
  return pad256(bin_bytes + 16) + 3 * pad256((n_reads + 1) * 8) + pad256(mhb_mercy_edges_scratch_bytes(n_reads, max_len)) +
         4096 + pad256(mhb_mercy_planes_words(n_reads, max_len) * 4);
}
// Segment sizes of a search streamed because its edges do not fit (no cap set): segments are packed to 1 GiB, which
// keeps the pinned staging small and the uploads overlapping, but a leading byte may take a slot of up to half the room
// the reads, scratch and planes leave.
constexpr uint64_t kMercySegmentTarget = 1ull << 30;
void mercy_auto_segment_bytes(double avail, size_t fixed, uint64_t *target, uint64_t *limit) {
  const double room = avail - (double)fixed;
  *limit = room > 2.0 * 4096 ? (uint64_t)(room / 2) - 4096 : 0;
  *target = std::min(*limit, kMercySegmentTarget);
}
// the resident search: candidate reads (image, record and edge offsets, ids), the sorted edges and the scratch
size_t mercy_resident_bytes(uint64_t n_edges, uint32_t k, uint64_t n_reads, uint64_t cand_words, uint32_t max_len) {
  const size_t bin_bytes = (cand_words * 4 + 15) & ~(size_t)15;
  return pad256(bin_bytes + 16) + 3 * pad256((n_reads + 1) * 8) + pad256((size_t)n_edges * words_per_edge(k) * 4 + 16) +
         pad256(mhb_mercy_edges_scratch_bytes(n_reads, max_len)) + 4096;
}
// The candidate reads of a mercy search in host memory, in file orientation as the device kernels take a library, with
// the offsets of an mhb_dev_reads
struct CandReads {
  std::vector<uint32_t> bin;
  std::vector<uint64_t> rec_off{0}, edge_off{0};
  uint32_t max_len = 0;
  uint64_t n() const { return rec_off.size() - 1; }
  // one read, given at its length word; reversed: its bases are stored last to first, as `.cand` holds them
  void add(const uint32_t *read, bool reversed, uint32_t k) {
    const uint32_t L = read[0], nw = div_ceil(L, 16);
    const size_t at = bin.size();
    if (reversed) {
      bin.resize(at + 1 + nw, 0);
      bin[at] = L;
      for (uint32_t i = 0; i < L; ++i) bin[at + 1 + (i >> 4)] |= base_at(read + 1, L - 1 - i) << (30 - 2 * (i & 15));
    } else {
      bin.insert(bin.end(), read, read + 1 + nw);
    }
    rec_off.push_back(bin.size());
    edge_off.push_back(edge_off.back() + (L >= k + 1 ? L - k : 0));
    max_len = std::max(max_len, L);
  }
};

// The resident search (GenMercyEdges, seq_to_sdbg.cpp:171-357) of the n_cand reads `ids` of `reads` in the n_edges
// sorted edges, in mhb_mercy_edges_scratch_bytes(n_cand, max_len) bytes of scratch: the look-up table, the count, then
// dest(n_mercy, &where) sizes the destination before the edges are written there.  Reads that overlap only at their
// ends can put more mercy edges between two tips than any bound known in advance (the reference reserves +25 % and
// grows, seq_to_sdbg.cpp:371-379); here the exact number is known before anything is written.
using MercyDest = std::function<int(uint64_t, uint32_t **)>;
int mercy_edges_resident(cudaStream_t st, const mhb_dev_reads &reads, const uint64_t *ids, uint64_t n_cand, uint32_t max_len,
                         uint32_t k, const uint32_t *edges, uint64_t n_edges, char *scratch, const MercyDest &dest,
                         uint64_t *n_mercy) {
  const size_t core = mhb_mercy_edges_scratch_bytes(n_cand, max_len) - mhb_edge_lut_bytes();
  void *lut = scratch + core;
  CKR(mhb_edge_lut_build(st, edges, n_edges, k, lut));
  const uint32_t *seg_e[1] = {edges};
  const uint64_t seg_n[1] = {n_edges};
  const void *seg_l[1] = {lut};
  CKR(mhb_mercy_edges_count(st, &reads, ids, n_cand, max_len, k, 1, seg_e, seg_n, seg_l, nullptr, n_mercy, scratch, core));
  if (!*n_mercy) return MHB_OK;
  uint32_t *out = nullptr;
  CKR(dest(*n_mercy, &out));
  return mhb_mercy_edges_write(st, &reads, ids, n_cand, max_len, k, out, *n_mercy, *n_mercy, scratch, core);
}

// mhb_mercy_host on candidate reads in file orientation: the edges resident, or streamed in leading-byte segments when
// they do not fit next to the candidate reads and the scratch, or when a chunk cap is set (every search stays inside
// one 12-base prefix, so inside one leading byte and one segment)
int mercy_from_host(uint32_t k, const uint32_t *edges, uint64_t n_edges, const CandReads &c, uint32_t **mercy_out,
                    uint64_t *n_mercy_out) {
  const uint32_t WE = words_per_edge(k), max_len = c.max_len;
  const uint64_t n_reads = c.n();
  g_mercy_st = StreamStats();
  if (n_reads == 0 || n_edges == 0) {
    *mercy_out = (uint32_t *)malloc(4);
    return MHB_OK;
  }
  const size_t bin_bytes = (c.bin.size() * 4 + 15) & ~(size_t)15;
  const size_t ms_bytes = mhb_mercy_edges_scratch_bytes(n_reads, max_len);
  const size_t need = mercy_resident_bytes(n_edges, k, n_reads, c.bin.size(), max_len);
  const bool stream = g_s2s_chunk_limit != 0 ||
                      (need > g_arena.cap && mhb_read_stream_decide(need, (uint64_t)arena_avail_bytes(), 0, 0));
  const size_t pw = stream ? mhb_mercy_planes_words(n_reads, max_len) : 0;
  const size_t fixed_b = mercy_stream_fixed_bytes(n_reads, c.bin.size(), max_len);
  // streamed: the edges cut at the first edge of every segment
  std::vector<uint32_t> seg_first;
  ChunkStream segs;
  if (stream) {
    uint64_t target = g_s2s_chunk_limit, limit = g_s2s_chunk_limit, start[257];
    if (!target) mercy_auto_segment_bytes(arena_avail_bytes(), fixed_b, &target, &limit);
    edge_byte_starts(edges, n_edges, WE, start);
    CKR(plan_mercy_segments(start, WE, target, limit, &seg_first));
    std::vector<uint64_t> first;
    for (uint32_t b : seg_first) first.push_back(start[b]);
    ChunkStream::Input in;
    in.image = edges;
    in.words = n_edges * WE;
    in.n = n_edges;
    in.stride = WE;
    CKR(segs.init(in, std::move(first), &g_mercy_st));
  }
  CKR(g_arena.reserve(stream ? fixed_b + segs.device_bytes() : need));
  cudaStream_t st = 0;
  uint32_t *d_bin = g_arena.take<uint32_t>(bin_bytes / 4 + 4);
  uint64_t *d_rec_off = g_arena.take<uint64_t>(n_reads + 1);
  uint64_t *d_edge_off = g_arena.take<uint64_t>(n_reads + 1);
  uint64_t *d_ids = g_arena.take<uint64_t>(n_reads + 1);
  uint32_t *d_edges = stream ? nullptr : g_arena.take<uint32_t>((size_t)n_edges * WE + 4);
  char *d_ms = g_arena.take<char>(ms_bytes);
  std::vector<uint64_t> ids(n_reads);
  for (uint64_t r = 0; r < n_reads; ++r) ids[r] = r;
  CK(cudaMemcpyAsync(d_bin, c.bin.data(), c.bin.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_rec_off, c.rec_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_edge_off, c.edge_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_ids, ids.data(), n_reads * 8, cudaMemcpyHostToDevice, st));
  if (!stream) CK(cudaMemcpyAsync(d_edges, edges, (size_t)n_edges * WE * 4, cudaMemcpyHostToDevice, st));
  mhb_dev_reads reads;
  reads.bin = d_bin;
  reads.bin_words = c.bin.size();
  reads.n_reads = n_reads;
  reads.fixed_len = 0;
  reads.rec_off = d_rec_off;
  reads.edge_off = d_edge_off;
  DevBuf out;
  const MercyDest dest = [&](uint64_t n, uint32_t **d) {
    CKR(out.alloc((size_t)n * WE * 4, "mercy: edges"));
    *d = out.as<uint32_t>();
    return MHB_OK;
  };
  uint64_t n_mercy = 0;
  if (!stream) {
    CKR(mercy_edges_resident(st, reads, d_ids, n_reads, max_len, k, d_edges, n_edges, d_ms, dest, &n_mercy));
  } else {
    // segment i answers the searches whose leading byte it holds; the answers of all segments are OR-ed into one set
    // of planes, which then stands for the single-segment search
    const size_t core = ms_bytes - mhb_edge_lut_bytes();
    void *lut = d_ms + core;
    uint32_t *d_planes = g_arena.take<uint32_t>(pw);
    char *d_slots = g_arena.take<char>(segs.device_bytes());
    uint8_t owner[256];
    for (uint64_t i = 0; i < segs.n_chunks(); ++i)
      for (uint32_t b = seg_first[i]; b < seg_first[i + 1]; ++b) owner[b] = (uint8_t)i;
    CK(cudaMemsetAsync(d_planes, 0, pw * 4, st));
    CKR(segs.bind(d_slots, st));
    CKR(segs.pass(st, [&](const ChunkView &c) {
      CKR(mhb_edge_lut_build(st, c.words, c.n, k, lut));
      return mercy_probe_owned(st, &reads, d_ids, n_reads, max_len, k, c.words, c.n, lut, owner, (uint32_t)c.index,
                               d_planes, true);
    }));
    CKR(mhb_mercy_count_planes(st, &reads, d_ids, n_reads, max_len, k, d_planes, 1, pw, &n_mercy, d_ms, core));
    uint32_t *d_out = nullptr;
    if (n_mercy) CKR(dest(n_mercy, &d_out));
    if (n_mercy) CKR(mhb_mercy_edges_write(st, &reads, d_ids, n_reads, max_len, k, d_out, n_mercy, n_mercy, d_ms, core));
  }
  *mercy_out = (uint32_t *)malloc(std::max<size_t>(4, (size_t)n_mercy * WE * 4));
  if (!*mercy_out) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  if (n_mercy) {
    int rc = MHB_OK;
    if (cudaMemcpyAsync(*mercy_out, out.p, (size_t)n_mercy * WE * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = mhb_set_error(MHB_ERR_CUDA, "mercy edge download failed");
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess)
      rc = mhb_set_error(MHB_ERR_CUDA, "mercy edge kernels failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (rc) {
      free(*mercy_out);
      *mercy_out = nullptr;
      return rc;
    }
  }
  *n_mercy_out = n_mercy;
  return MHB_OK;
}
}  // namespace

extern "C" int mhb_selftest_mercy_stream_decide(uint64_t n_edges, uint32_t k, uint64_t n_cand_reads, uint64_t cand_words,
                                                uint32_t max_read_len, uint64_t free_bytes, uint64_t chunk_limit,
                                                uint64_t *resident_bytes, int *stream) {
  *resident_bytes = mercy_resident_bytes(n_edges, k, n_cand_reads, cand_words, max_read_len);
  *stream = mhb_read_stream_decide(*resident_bytes, (uint64_t)(0.92 * (double)free_bytes), 0, chunk_limit);
  return MHB_OK;
}

extern "C" int mhb_selftest_mercy_auto_plan(const uint64_t *byte_edges, uint32_t k, uint64_t n_cand_reads, uint64_t cand_words,
                                            uint32_t max_read_len, uint64_t free_bytes, uint32_t *first_byte_out,
                                            uint64_t *slot_bytes) {
  uint64_t start[257] = {0};
  for (int b = 0; b < 256; ++b) start[b + 1] = start[b] + byte_edges[b];
  uint64_t target = 0, limit = 0;
  mercy_auto_segment_bytes(0.92 * (double)free_bytes, mercy_stream_fixed_bytes(n_cand_reads, cand_words, max_read_len), &target,
                           &limit);
  std::vector<uint32_t> first;
  if (plan_mercy_segments(start, words_per_edge(k), target, limit, &first)) return -1;
  memcpy(first_byte_out, first.data(), first.size() * 4);
  uint64_t max_seg = 0;
  for (size_t i = 0; i + 1 < first.size(); ++i) max_seg = std::max(max_seg, start[first[i + 1]] - start[first[i]]);
  *slot_bytes = ChunkStream::image_bytes(max_seg * words_per_edge(k));
  return (int)(first.size() - 1);
}

extern "C" int mhb_mercy_host(uint32_t k, const uint32_t *edges, uint64_t n_edges, const uint32_t *cand_bin,
                              uint64_t cand_words, uint32_t **mercy_out, uint64_t *n_mercy_out, uint64_t *n_cand_reads_out) {
  if (!mercy_out || !n_mercy_out) return mhb_set_error(MHB_ERR_ARG, "null output");
  *mercy_out = nullptr;
  *n_mercy_out = 0;
  if (n_cand_reads_out) *n_cand_reads_out = 0;
  if (k < 12 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "mercy edges need 12 <= k <= 255");
  if (mhb_device_count() == 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  // `.cand` holds the reads as KmerCounter held them: REVERSED (kmer_counter.cpp:387-401; read back with reverse=false,
  // seq_to_sdbg.cpp:175-176).  The device kernels take a library in file orientation and apply the reversal themselves,
  // so every candidate read is turned around once here (they are ~0.2 % of a library).
  CandReads c;
  for (uint64_t pos = 0; pos < cand_words; pos += 1 + div_ceil(cand_bin[pos], 16)) {
    if (pos + 1 + div_ceil(cand_bin[pos], 16) > cand_words) return mhb_set_error(MHB_ERR_IO, "candidate read image is truncated");
    c.add(cand_bin + pos, true, k);
  }
  if (n_cand_reads_out) *n_cand_reads_out = c.n();
  return mercy_from_host(k, edges, n_edges, c, mercy_out, n_mercy_out);
}

// ================================================================================================
// fused k_min build: count -> mercy edges -> seq2sdbg
// ================================================================================================
// One chain of the stage drivers.  A stage that ran in one pass over resident data hands its result to the next one on
// the device: the count leaves its edges, flags, library and candidate ids in the arena, the mercy edges are written
// behind the solid edges, and seq2sdbg sorts them where they are, its buffers in the count's round buffers whenever
// those are large enough.  Otherwise the result passes through host memory once, as between the reference's `count`
// and `seq2sdbg` (base_engine.cpp:54-141 plans its passes the same way: the output does not depend on where the
// boundaries fall).
extern "C" int mhb_build_host(const mhb_build_args *args, mhb_build_result *res) {
  if (!args || !res) return mhb_set_error(MHB_ERR_ARG, "null args");
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k;
  if (k < 9 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "kmer size must be >= 9 and <= 255");
  if (args->need_mercy && k < 12) return mhb_set_error(MHB_ERR_ARG, "mercy edges need k >= 12");
  if (mhb_device_count() == 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  const uint32_t WE = words_per_edge(k);
  res->words_per_edge = WE;
  res->words_per_tip_label = words_per_tip_label(k);
  cudaStream_t st = 0;
  EventTimer t_all(st), t(st);
  t_all.start();

  // ---- count ----
  mhb_count_args ca;
  memset(&ca, 0, sizeof(ca));
  ca.k = k;
  ca.m = args->m;
  ca.bin = args->bin;
  ca.bin_words = args->bin_words;
  ca.n_reads = args->n_reads;
  ca.want_mercy = args->need_mercy;
  std::vector<char> cbuf(sizeof(mhb_count_result));
  mhb_count_result *cr = reinterpret_cast<mhb_count_result *>(cbuf.data());
  struct Owned {  // the host result's buffers, unless handed on to the caller
    mhb_count_result *r;
    uint32_t *mercy = nullptr;
    ~Owned() {
      free(r->edges);
      free(r->cand_ids);
      free(mercy);
    }
  } owned{cr};
  CountOnDevice dev;
  read_stream_stats_reset();
  CKR(count_host_rounds(&ca, cr, read_chunk_limit() != 0, FixedCheck::kSampled, &dev));
  const uint64_t n_solid = cr->n_solid, n_cand = cr->n_cand;
  res->n_edge_records = cr->n_edge_records;
  res->n_solid = n_solid;
  res->n_cand = n_cand;
  res->t_h2d_ms = cr->t_h2d_ms;
  res->t_count_ms = cr->t_extract_ms + cr->t_count_ms;
  res->t_mercy_ms = cr->t_mercy_ms;

  // ---- mercy edges: on the device behind the solid edges, or from the candidate reads in file orientation ----
  t.start();
  uint64_t n_mercy = 0;
  uint32_t *d_edges = dev.edges;
  DevBuf big_edges;  // solid + mercy edges when the mercy edges do not fit behind the solid ones in the count's buffer
  if (args->need_mercy && n_cand && dev.valid) {
    DevBuf own;
    char *d_ms;
    CKR(g_arena.take_or_alloc(mhb_mercy_edges_scratch_bytes(n_cand, dev.max_len), &own, "build: mercy edge scratch", &d_ms));
    const MercyDest dest = [&](uint64_t n, uint32_t **d) {
      if (n > dev.cap_edges - n_solid) {
        CKR(big_edges.alloc((size_t)(n_solid + n) * WE * 4 + 16, "build: solid + mercy edges"));
        CK(cudaMemcpyAsync(big_edges.p, dev.edges, (size_t)n_solid * WE * 4, cudaMemcpyDeviceToDevice, st));
        d_edges = big_edges.as<uint32_t>();
      }
      *d = d_edges + (size_t)n_solid * WE;
      return MHB_OK;
    };
    CKR(mercy_edges_resident(st, dev.reads, dev.cand, n_cand, dev.max_len, k, dev.edges, n_solid, d_ms, dest, &n_mercy));
    g_arena.used = dev.work_mark;
  } else if (args->need_mercy && n_cand) {
    CandReads c;
    uint64_t r = 0, pos = 0;
    for (uint64_t i = 0; i < n_cand; ++i) {
      for (; r < cr->cand_ids[i]; ++r) pos += 1 + div_ceil(args->bin[pos], 16);
      c.add(args->bin + pos, false, k);
    }
    CKR(mercy_from_host(k, cr->edges, n_solid, c, &owned.mercy, &n_mercy));
  }
  res->n_mercy = n_mercy;
  res->t_mercy_ms += t.stop();

  // ---- what `count` writes to disk: the downloads are queued ahead of seq2sdbg on the same stream, so they read the
  // count's buffers before anything reuses them, and seq2sdbg's own synchronisation completes them ----
  t.start();
  if (args->want_edges) {
    res->counting = (int64_t *)malloc(65536 * 8);
    if (!res->counting) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
    if (dev.valid) {
      res->edges = (uint32_t *)malloc(std::max<size_t>(1, (size_t)n_solid * WE * 4));
      res->cand_ids = (uint64_t *)malloc(std::max<size_t>(1, n_cand * 8));
      if (!res->edges || !res->cand_ids) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
      if (n_solid) CK(cudaMemcpyAsync(res->edges, dev.edges, (size_t)n_solid * WE * 4, cudaMemcpyDeviceToHost, st));
      if (n_cand) CK(cudaMemcpyAsync(res->cand_ids, dev.cand, n_cand * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(res->counting, dev.mul_hist, 65536 * 8, cudaMemcpyDeviceToHost, st));
    } else {
      memcpy(res->counting, cr->counting, 65536 * 8);
      std::swap(res->edges, cr->edges);
      std::swap(res->cand_ids, cr->cand_ids);
      if (!res->cand_ids) res->cand_ids = (uint64_t *)malloc(8);  // no mercy bookkeeping: an empty list, as above
      if (!res->cand_ids) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
    }
  }
  CK(cudaEventRecord(t.b, st));  // read once seq2sdbg has synchronised

  // ---- seq2sdbg over solid + mercy edges: in one pass where they are, or through host memory ----
  const uint64_t n_seqs = n_solid + n_mercy, n_items = 6 * n_seqs;  // 2 strands x (k+1 - k + 2)
  const size_t s2s_bytes = s2s_device_bytes(n_items, k);
  const bool s2s_on_device = dev.valid && !(g_s2s_round_limit && n_items > g_s2s_round_limit) &&
                             (g_arena.used + s2s_bytes <= g_arena.cap || (double)s2s_bytes <= 0.92 * (double)free_device_bytes());
  std::vector<uint32_t> h_edges;
  if (!s2s_on_device) {
    h_edges.resize((size_t)n_seqs * WE);
    if (dev.valid && n_seqs) CK(cudaMemcpy(h_edges.data(), d_edges, (size_t)n_seqs * WE * 4, cudaMemcpyDeviceToHost));
    if (!dev.valid && n_solid) memcpy(h_edges.data(), res->edges ? res->edges : cr->edges, (size_t)n_solid * WE * 4);
    if (!dev.valid && n_mercy) memcpy(h_edges.data() + (size_t)n_solid * WE, owned.mercy, (size_t)n_mercy * WE * 4);
    big_edges.release();
  }
  res->bucket_table = (uint64_t *)malloc((size_t)MHB_NUM_BUCKETS * 32);
  if (!res->bucket_table) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  S2sOut out;
  out.table = res->bucket_table;
  out.user = args->sdbg_out;
  out.user_cap = args->sdbg_out_capacity;
  if (s2s_on_device) {
    // the solid edges still have the count stage's in/out flags: the $-items the emitter would discard for certain are
    // not generated (2.02 instead of 6 items per edge on a 30x genome), same bytes out
    static const bool no_prune = getenv("MHB_S2S_NO_PRUNE") != nullptr;
    SeqSource src(d_edges, n_seqs, k, true, no_prune ? nullptr : dev.aux, n_solid);
    CKR(src.init(0));
    CKR(s2s_host_rounds(k, src, n_items, 0, true, &out));
  } else {
    SeqSource src(h_edges.data(), n_seqs, k, false);
    CKR(s2s_run(k, src, n_items, &out));
  }
  res->bytes = out.bytes;
  set_sdbg_totals(res, out.tot);
  res->n_sort_items = out.n_sorted;
  res->t_s2s_ms = out.t_extract_ms + out.t_sort_ms + out.t_emit_ms;
  float edges_ms = 0;
  CK(cudaEventElapsedTime(&edges_ms, t.a, t.b));
  res->t_d2h_ms = cr->t_d2h_ms + edges_ms + out.t_d2h_ms;
  res->t_total_ms = t_all.stop();
  return MHB_OK;
}

// ================================================================================================
// Self-test hooks: run the SAME record builders the kernels use (mhb_kernels.cuh, __host__ __device__)
// on the host, so that `pytest -m "not gpu"` can check the bit arithmetic against the oracle without a
// GPU.  They build one record at a time and are not a compute path.
// ================================================================================================
#include "mhb_kernels.cuh"

extern "C" int mhb_selftest_count_record(const uint32_t *read_words, uint32_t nwords, uint32_t L, uint32_t k, uint32_t q,
                                         uint32_t *rec_out, uint32_t *strand_out) {
  const uint32_t W = count_key_words(k), WR = count_record_words(k);
  if (k < 1 || k > MHB_MAX_K || L < k + 1 || q + k + 1 > L) return mhb_set_error(MHB_ERR_ARG, "bad selftest args");
#define M(WW)                                                                       \
  if (W == WW && WR == WW) {                                                        \
    uint32_t r[WW];                                                                 \
    make_count_record<WW, WW>(read_words, nwords, L, k, q, r, *strand_out);         \
    memcpy(rec_out, r, sizeof(r));                                                  \
    return MHB_OK;                                                                  \
  }                                                                                 \
  if (W == WW && WR == WW + 1) {                                                    \
    uint32_t r[WW + 1];                                                             \
    make_count_record<WW, WW + 1>(read_words, nwords, L, k, q, r, *strand_out);     \
    memcpy(rec_out, r, sizeof(r));                                                  \
    return MHB_OK;                                                                  \
  }
  M(1) M(2) M(3) M(4) M(5) M(6) M(7) M(8) M(9) M(10) M(11) M(12) M(13) M(14) M(15) M(16)
#undef M
  return mhb_set_error(MHB_ERR_ARG, "unsupported k");
}

// the rolling builder (mhb_kernels.cuh make_count_records_roll) run on the host: 4 records from position q on
extern "C" int mhb_selftest_count_records_roll(const uint32_t *read_words, uint32_t nwords, uint32_t L, uint32_t k, uint32_t q,
                                               uint64_t *rec4_out, uint32_t *strand4_out) {
  if (k + 1 < 17 || k + 1 > 32 || L < k + 1 || q + k + 1 > L) return mhb_set_error(MHB_ERR_ARG, "bad selftest args");
  u64 r[4];
  u32 st[4];
  make_count_records_roll<4>(read_words, nwords, L, k, q, r, st);
  for (int j = 0; j < 4; ++j) {
    rec4_out[j] = r[j];
    strand4_out[j] = st[j];
  }
  return MHB_OK;
}

extern "C" int mhb_selftest_s2s_record(const uint32_t *seq_words, uint32_t nwords, uint32_t L, uint32_t k, uint32_t strand,
                                       uint32_t offset, uint32_t mult, uint32_t *rec_out) {
  const uint32_t W = s2s_record_words(k);
  if (k < 9 || k > MHB_MAX_K || L < k + 1 || offset > L - k + 1) return mhb_set_error(MHB_ERR_ARG, "bad selftest args");
#define M(WW)                                                                \
  if (W == WW) {                                                             \
    uint32_t r[WW];                                                          \
    make_s2s_record<WW>(seq_words, nwords, L, k, strand, offset, mult, r);   \
    memcpy(rec_out, r, sizeof(r));                                           \
    return MHB_OK;                                                           \
  }
  M(1) M(2) M(3) M(4) M(5) M(6) M(7) M(8) M(9) M(10) M(11) M(12) M(13) M(14) M(15) M(16) M(17)
#undef M
  return mhb_set_error(MHB_ERR_ARG, "unsupported k");
}
