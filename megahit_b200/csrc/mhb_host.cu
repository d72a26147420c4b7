// mhb_host.cu -- host-level C ABI (include/mhb.h, layer 2): host buffers in, host buffers out.
// Orchestrates the device-level entry points on one GPU with a grow-only device arena that is kept
// between calls (so repeated steps do not pay cudaMalloc).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
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
// (ReadStream); the round buffers get the memory the resident image would have taken.  A resident call switches to
// streaming when the library alone does not fit or when one bucket exceeds the round that fits next to it.
static int count_host_rounds(const mhb_count_args *args, mhb_count_result *res, const ReadLibIndex &ix, bool stream) {
  const uint32_t k = args->k;
  const int32_t m = args->m;
  const uint64_t n = ix.n_units, n_reads = args->n_reads;
  const uint32_t WR = count_record_words(k), WE = words_per_edge(k);
  const int top_byte = (int)(4 * WR - 1);
  cudaStream_t st = 0;
  EventTimer t_all(st), t(st);
  t_all.start();
  auto restart_streamed = [&]() {
    const uint32_t we = res->words_per_edge;
    const uint64_t ne = res->n_edge_records;
    memset(res, 0, sizeof(*res));
    res->words_per_edge = we;
    res->n_edge_records = ne;
    return count_host_rounds(args, res, ix, true);
  };

  ReadStream rs;
  const uint64_t chunk_cap = read_chunk_limit() ? read_chunk_limit() : read_chunk_auto_bytes();
  CKR(rs.init(args->bin, args->bin_words, n_reads, ix, stream ? chunk_cap : 0));
  const uint64_t chunk_reads = rs.max_chunk_reads();  // reads the per-read arrays hold
  // besides the round buffers: the library (or its chunk slots), the mercy marks, the histograms and scalars
  size_t fixed = pad256(rs.device_bytes()) + pad256(65536 * 8) + pad256(256 * 8) + 4096;
  if (args->want_mercy) fixed += 2 * pad256((size_t)(chunk_reads + 1) * 4);
  bool one_pass = false;
  if (!stream && !(g_round_limit && n > g_round_limit)) {
    const size_t need = fixed + round_bytes(n, WR, WE, m, k);
    one_pass = need <= g_arena.cap;
    if (!one_pass) {
      one_pass = (double)need <= arena_avail_bytes();
    }
  }
  uint64_t max_records = n;
  if (!one_pass) {  // + the per-read counts of the extraction and the second-byte histograms
    fixed += pad256((chunk_reads + 2) * 8) + pad256(256 * 256 * 8) + pad256(256 * 8) + pad256(64) + 4096;
    max_records = g_round_limit;
    if (!max_records) {
      const size_t avail = (size_t)arena_avail_bytes();
      if (!stream && mhb_read_stream_decide(fixed, avail, 0, read_chunk_limit())) return restart_streamed();
      max_records = largest_round(n, fixed, avail, [&](uint64_t r) { return round_bytes(r, WR, WE, m, k); });
      if (!max_records)
        return mhb_set_error(MHB_ERR_NOMEM, "the read library's %s (%zu bytes) does not fit the device",
                             stream ? "chunk buffers" : "image", fixed);
    }
    max_records = std::min<uint64_t>(std::max<uint64_t>(max_records, 1), std::max<uint64_t>(n, 1));
  }
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
  uint64_t *d_scalars = g_arena.take<uint64_t>(8);  // [0] n_solid, [1] round total
  uint32_t *d_first = nullptr, *d_last = nullptr;
  if (args->want_mercy) {
    d_first = g_arena.take<uint32_t>(chunk_reads + 1);
    d_last = g_arena.take<uint32_t>(chunk_reads + 1);
  }
  uint32_t *d_a = g_arena.take<uint32_t>((size_t)max_records * WR + 4);
  uint32_t *d_b = g_arena.take<uint32_t>((size_t)max_records * WR + 4);
  const CountWork cw = count_work_plan(max_records, k, m);
  char *d_work = g_arena.take<char>(cw.bytes);
  uint32_t *d_edges = g_arena.take<uint32_t>((size_t)cap_edges * WE);
  uint8_t *d_aux = g_arena.take<uint8_t>(cap_edges);

  t.start();
  CKR(rs.bind(d_lib, st));
  CK(cudaMemsetAsync(d_mul_hist, 0, 65536 * 8, st));
  CK(cudaMemsetAsync(d_hist_top, 0, 256 * 8, st));
  res->t_h2d_ms = t.stop();

  // one pass over the reads: fn(view of a chunk, its first read), once per chunk
  auto each_chunk = [&](const std::function<int(const mhb_dev_reads &, uint64_t)> &fn) -> int {
    return rs.pass(st, [&](const ReadChunkView &c) {
      mhb_dev_reads v;
      v.bin = c.bin;
      v.bin_words = c.bin_words;
      v.n_reads = c.n_reads;
      v.fixed_len = ix.fixed_len;
      v.rec_off = c.rec_off;
      v.edge_off = c.aux_off;
      return fn(v, c.first_read);
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
      if (!stream && !g_round_limit) return restart_streamed();
      return MHB_ERR_NOMEM;
    }
    CKR(rc);
    res->t_extract_ms = t.stop();
  }

  const bool tips_on_device = ranges.size() == 1;  // the only round's edges are still on the device for the mercy step
  std::vector<uint32_t> h_tip_edges;               // otherwise the tip edges (aux != 0) of every round
  std::vector<uint8_t> h_tip_aux, h_aux;
  uint64_t n_solid_total = 0;
  for (const auto &rg : ranges) {
    // ---- extract the range: all records at once, or per view, count its in-range records, then write them at the
    // round's cursor ----
    t.start();
    CK(cudaMemsetAsync(d_hist0, 0, 256 * 8, st));
    CK(cudaMemsetAsync(d_scalars, 0, 8, st));
    uint64_t n_round = n;
    if (one_pass) {
      CKR(each_chunk([&](const mhb_dev_reads &v, uint64_t) { return mhb_count_extract(st, &v, k, d_a, n, d_hist0, cw.hist_byte); }));
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
    res->t_extract_ms += t.stop();
    // ---- sort / partition + solid edges ----
    t.start();
    CKR(run_count_stage(st, cw, d_a, d_b, n_round, k, m, d_hist0, d_edges, d_aux, cap_edges, d_mul_hist, d_scalars, d_work,
                        one_pass ? res->sort_pass_ms : nullptr, one_pass ? &res->n_sort_passes : nullptr));
    uint64_t n_solid = 0;
    CK(cudaMemcpyAsync(&n_solid, d_scalars, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    res->t_count_ms += t.stop();
    if (n_solid > cap_edges) return mhb_set_error(MHB_ERR_NOMEM, "internal: solid edges exceed capacity");
    // ---- append to the host result ----
    t.start();
    const size_t e0 = (size_t)n_solid_total * WE;
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
    n_solid_total += n_solid;
    res->t_d2h_ms += t.stop();
    ++res->n_rounds;
  }
  res->n_solid = n_solid_total;
  for (uint32_t p = 0; p < res->n_sort_passes; ++p) res->t_sort_ms += res->sort_pass_ms[p];

  // ---- mercy bookkeeping over the whole library ----
  std::vector<uint32_t> h_first, h_last;
  if (args->want_mercy && n_reads) {
    t.start();
    uint64_t n_tip = h_tip_aux.size();
    if (tips_on_device) CKR(mhb_count_tip_edges(st, d_aux, n_solid_total, &n_tip));
    const size_t ts_bytes = mhb_tipset_bytes(n_tip, k);
    const size_t list_bytes = pad256(h_tip_edges.size() * 4 + 16) + pad256(h_tip_aux.size() + 16);
    // the per-round buffers are free now
    DevBuf own;
    char *d_tmp = (char *)d_a;
    if (ts_bytes + list_bytes + 512 > (size_t)max_records * WR * 4 * 2) {
      CKR(own.alloc(ts_bytes + list_bytes + 512, "count: mercy tip set"));
      d_tmp = own.as<char>();
    }
    const uint32_t *d_tip_edges = tips_on_device ? d_edges : (uint32_t *)d_tmp;
    const uint8_t *d_tip_aux = tips_on_device ? d_aux : (uint8_t *)(d_tmp + pad256(h_tip_edges.size() * 4 + 16));
    char *d_tips = d_tmp + list_bytes;
    int rc = MHB_OK;
    if (!h_tip_aux.empty()) {
      if (cudaMemcpyAsync((void *)d_tip_edges, h_tip_edges.data(), h_tip_edges.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
          cudaMemcpyAsync((void *)d_tip_aux, h_tip_aux.data(), n_tip, cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = mhb_set_error(MHB_ERR_CUDA, "tip edge upload failed");
    }
    if (!rc)
      rc = mhb_tipset_build(st, d_tip_edges, d_tip_aux, tips_on_device ? n_solid_total : n_tip, k, d_tips, ts_bytes, n_tip);
    // per view: marks into the view-sized first/last arrays, copied to the host arrays at the view's first read; the
    // host arrays are zeroed while the first marks run
    if (!rc) rc = each_chunk([&](const mhb_dev_reads &v, uint64_t r0) {
      CKR(mhb_count_mark_mercy(st, &v, k, d_tips, ts_bytes, n_tip, d_first, d_last));
      h_first.resize(n_reads);
      h_last.resize(n_reads);
      cudaMemcpyAsync(h_first.data() + r0, d_first, v.n_reads * 4, cudaMemcpyDeviceToHost, st);
      cudaMemcpyAsync(h_last.data() + r0, d_last, v.n_reads * 4, cudaMemcpyDeviceToHost, st);
      if (cudaStreamSynchronize(st) != cudaSuccess) return mhb_set_error(MHB_ERR_CUDA, "mercy marking failed: %s", cudaGetErrorString(cudaGetLastError()));
      return MHB_OK;
    });
    own.release();
    if (rc) return rc;
    res->t_mercy_ms = t.stop();
  }
  if (stream) {
    double h2d_ms = 0;
    mhb_read_stream_times(&h2d_ms, nullptr, nullptr, nullptr);
    res->t_h2d_ms = h2d_ms;
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
  res->words_per_edge = words_per_edge(k);
  read_stream_stats_reset();

  ReadLibIndex ix;
  CKR(index_read_lib(args->bin, args->bin_words, args->n_reads, k, &ix));
  res->n_edge_records = ix.n_units;
  // A13: when one pass over all records does not fit the device (or the caller capped the round size), the stage runs
  // in rounds over ranges of bucket ids; a chunk cap streams the library through those rounds
  return count_host_rounds(args, res, ix, read_chunk_limit() != 0);
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

// The sequences of one mhb_s2s_host call as its round loop sees them, one pass at a time: resident (uploaded once and
// handed over whole as one chunk, the arrays every call had), or kept in host memory and streamed through two device
// slots in chunks that end on sequence boundaries.  A fixed-length chunk carries its words and multiplicities and is
// viewed with fixed_len set; a variable-length one also carries word_off and item_off rebased to the chunk, and len.
class SeqSource {
 public:
  SeqSource(const mhb_s2s_args *a, const SeqLayout &ly) : a_(a), ly_(ly) {}
  // max_chunk_bytes = 0: resident
  int init(uint64_t max_chunk_bytes) {
    const uint64_t ns = a_->n_seqs;
    resident_ = max_chunk_bytes == 0;
    uint64_t max_words = ly_.n_words, max_n = ns;
    if (resident_) {
      first_ = {0, ns};
    } else {
      plan_seq_chunks(a_->word_off, ly_, ns, max_chunk_bytes, &first_);
      max_words = max_n = 0;
      for (uint64_t i = 0; i < n_chunks(); ++i) {
        max_n = std::max(max_n, first_[i + 1] - first_[i]);
        max_words = std::max(max_words, a_->word_off[first_[i + 1]] - a_->word_off[first_[i]]);
      }
    }
    const bool arrays = resident_ || !ly_.fixed;  // the resident form keeps all four arrays, as it always did
    o_wo_ = pad256(max_words * 4 + 64);
    o_io_ = o_wo_ + (arrays ? pad256((max_n + 1) * 8) : 0);
    o_len_ = o_io_ + (arrays ? pad256((max_n + 1) * 8) : 0);
    o_mult_ = o_len_ + (arrays ? pad256((max_n + 1) * 4) : 0);
    slot_bytes_ = o_mult_ + pad256((max_n + 1) * 2);
    g_s2s_st.chunks = n_chunks();
    return resident_ ? MHB_OK : stager_.init(slot_bytes_, n_chunks(), &g_s2s_st);
  }
  static size_t resident_bytes(uint64_t ns, uint64_t n_words) {
    return pad256(n_words * 4 + 64) + 2 * pad256((ns + 1) * 8) + pad256((ns + 1) * 4) + pad256((ns + 1) * 2);
  }
  size_t device_bytes() const { return (resident_ ? 1 : 2) * slot_bytes_; }
  uint64_t n_chunks() const { return resident_ ? 0 : first_.size() - 1; }
  // device_bytes() bytes; the resident form uploads the sequences there on st
  int bind(char *dev, cudaStream_t st) {
    dev_ = dev;
    stager_.bind(dev);
    const uint64_t ns = a_->n_seqs;
    if (!resident_ || !ns) return MHB_OK;
    CK(cudaMemcpyAsync(dev_, a_->words, ly_.n_words * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dev_ + o_wo_, a_->word_off, (ns + 1) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dev_ + o_io_, ly_.item_off.data(), (ns + 1) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dev_ + o_len_, a_->len, ns * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dev_ + o_mult_, a_->mult, ns * 2, cudaMemcpyHostToDevice, st));
    return MHB_OK;
  }
  // fn(view, items of the chunk) once per chunk, in order, on st
  int pass(cudaStream_t st, const std::function<int(const mhb_dev_seqs &, uint64_t)> &fn) {
    if (resident_) return fn(view(0, dev_), ly_.n_items);
    return stager_.pass(
        st, [this](uint64_t i, char *h, ChunkStager::Copies *up) { return fill(i, h, up); },
        [&](uint64_t i, const char *slot) { return fn(view(i, slot), ly_.item_off[first_[i + 1]] - ly_.item_off[first_[i]]); });
  }

 private:
  mhb_dev_seqs view(uint64_t i, const char *slot) const {
    const uint64_t b = first_[i], e = first_[i + 1];
    const bool arrays = resident_ || !ly_.fixed;
    mhb_dev_seqs v;
    v.words = (const uint32_t *)slot;
    v.n_words = e > b ? a_->word_off[e] - a_->word_off[b] : 0;  // no word_off read for an empty set
    v.n_seqs = e - b;
    v.fixed_len = ly_.fixed ? ly_.L0 : 0;
    v.word_off = arrays ? (const uint64_t *)(slot + o_wo_) : nullptr;
    v.item_off = arrays ? (const uint64_t *)(slot + o_io_) : nullptr;
    v.len = arrays ? (const uint32_t *)(slot + o_len_) : nullptr;
    v.mult = (const uint16_t *)(slot + o_mult_);
    v.fixed_stride = 0;
    return v;
  }
  int fill(uint64_t i, char *h, ChunkStager::Copies *up) const {
    const uint64_t b = first_[i], e = first_[i + 1], n = e - b, w0 = a_->word_off[b], nw = a_->word_off[e] - w0;
    {
      const uint64_t bytes = nw * 4, blk = 4ull << 20, nblk = (bytes + blk - 1) / blk;
#pragma omp parallel for schedule(static)
      for (long long j = 0; j < (long long)nblk; ++j) {
        const uint64_t o = (uint64_t)j * blk;
        memcpy(h + o, (const char *)(a_->words + w0) + o, std::min(blk, bytes - o));
      }
    }
    up->add(0, nw * 4);
    if (!ly_.fixed) {
      uint64_t *wo = (uint64_t *)(h + o_wo_), *io = (uint64_t *)(h + o_io_);
      const uint64_t i0 = ly_.item_off[b];
#pragma omp parallel for schedule(static)
      for (long long s = 0; s <= (long long)n; ++s) {
        wo[s] = a_->word_off[b + s] - w0;
        io[s] = ly_.item_off[b + s] - i0;
      }
      memcpy(h + o_len_, a_->len + b, n * 4);
      up->add(o_wo_, (n + 1) * 8);
      up->add(o_io_, (n + 1) * 8);
      up->add(o_len_, n * 4);
    }
    memcpy(h + o_mult_, a_->mult + b, n * 2);
    up->add(o_mult_, n * 2);
    return MHB_OK;
  }
  const mhb_s2s_args *a_;
  const SeqLayout &ly_;
  bool resident_ = true;
  std::vector<uint64_t> first_;
  size_t o_wo_ = 0, o_io_ = 0, o_len_ = 0, o_mult_ = 0, slot_bytes_ = 0;
  char *dev_ = nullptr;
  ChunkStager stager_;
};

// the smallest device footprint of the rounds over resident sequences: the sequences, the tables and a one-item round
size_t s2s_resident_round_bytes(uint64_t ns, uint64_t n_words, uint32_t k) {
  return SeqSource::resident_bytes(ns, n_words) + s2s_table_bytes(true) + s2s_round_bytes(1, s2s_record_words(k), k);
}
}  // namespace

// Same idea as count_host_rounds: the stage runs once per contiguous range of leading record bytes (a (k-1)-mer group,
// and a bucket, never spans two ranges): extract the range -> sort -> emit -> append the item bytes and that range's
// rows of the bucket table to the host result.  Ranges ascend, so the concatenated stream is in bucket order.  Every
// extraction is one pass over the sequences (SeqSource).  one_pass (resident sequences whose items all fit next to
// them): the one range over all bucket ids, known without a pass, extracted by mhb_s2s_extract, its output straight
// into the result.  Otherwise the top-byte histogram and the second-byte histograms of the leading bytes that alone
// exceed a round plan the ranges, and each non-empty round's chunks append their in-range items at its cursor.
static int s2s_host_rounds(const mhb_s2s_args *args, mhb_s2s_result *res, SeqSource &src, uint64_t n_items, uint64_t max_items,
                           bool one_pass) {
  const uint32_t k = args->k;
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
  CKR(g_arena.reserve(fixed_b + s2s_round_bytes(max_items, W, k)));
  char *d_seqs = g_arena.take<char>(src.device_bytes());
  uint64_t *d_table = g_arena.take<uint64_t>((size_t)MHB_NUM_BUCKETS * 4);
  uint64_t *d_hist0 = g_arena.take<uint64_t>(256);
  uint64_t *d_totals = g_arena.take<uint64_t>(16);
  uint64_t *d_hist_top = nullptr, *d_sub = nullptr, *d_cursor = nullptr;  // to plan rounds
  if (!one_pass) {
    d_hist_top = g_arena.take<uint64_t>(256);
    d_sub = g_arena.take<uint64_t>(256 * 256);
    d_cursor = g_arena.take<uint64_t>(8);
  }
  uint32_t *d_a = g_arena.take<uint32_t>((size_t)max_items * W + 4);
  uint32_t *d_b = g_arena.take<uint32_t>((size_t)max_items * W + 4);
  // sort + emit workspace (at most the sort workspace plus the emit scratch s2s_round_bytes reserves)
  const size_t ws_bytes = mhb_s2s_sort_emit_workspace_bytes(max_items, k);
  // worst case bytes per sort item: 2 + 2 + 4*WPT (every item a large-multiplicity tip)
  const uint64_t cap_bytes = max_items * (4ull + 4ull * WPT) + 16;
  char *d_ws = g_arena.take<char>(ws_bytes);
  uint8_t *d_bytes = g_arena.take<uint8_t>(cap_bytes);
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
    res->t_extract_ms = t.stop();
  }

  SdbgStitch out;
  uint64_t tot[16] = {0};  // one pass: the emitter's totals
  for (const auto &rg : ranges) {
    const uint64_t planned = one_pass ? n_items : pre[rg.second + 1] - pre[rg.first];  // the range's items
    if (!one_pass && planned == 0) continue;
    ++g_s2s_rounds;
    t.start();
    CK(cudaMemsetAsync(d_hist0, 0, 256 * 8, st));
    uint64_t n_round = n_items;
    if (one_pass) {
      CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
        return mhb_s2s_extract(st, &s, k, d_a, n, d_hist0, mhb_s2s_sort_hist_byte(max_items, k));
      }));
    } else {
      CK(cudaMemsetAsync(d_cursor, 0, 64, st));
      CKR(src.pass(st, [&](const mhb_dev_seqs &s, uint64_t n) {
        return mhb_s2s_extract_range(st, &s, k, d_a, n, rg.first, rg.second, d_cursor, max_items, d_hist0,
                                     mhb_s2s_sort_hist_byte(max_items, k));
      }));
      CK(cudaMemcpyAsync(&n_round, d_cursor, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
    res->t_extract_ms += t.stop();
    if (n_round != planned)
      return mhb_set_error(MHB_ERR_NOMEM, "internal: round of %llu items, %llu planned", (unsigned long long)n_round,
                           (unsigned long long)planned);
    t.start();
    // the histogram is of the byte a sort of max_items items starts with: pass it only if this round's sort does too
    const bool hist_ok = mhb_s2s_sort_hist_byte(n_round, k) == mhb_s2s_sort_hist_byte(max_items, k);
    // sort and emit in one call (the bucket kernel emits every bucket it sorts): t_sort_ms carries both
    CKR(mhb_s2s_sort_emit(st, d_a, d_b, n_round, k, hist_ok ? d_hist0 : nullptr, d_bytes, cap_bytes, d_table, d_totals, d_ws,
                          ws_bytes));
    res->t_sort_ms += t.stop();
    t.start();
    if (one_pass) {
      CK(cudaMemcpyAsync(tot, d_totals, sizeof(tot), cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(res->bucket_table, d_table, sizeof(res->bucket_table), cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (tot[0] > cap_bytes) return mhb_set_error(MHB_ERR_NOMEM, "internal: SdBG byte stream exceeds capacity");
    } else {
      CKR(out.append(st, d_bytes, cap_bytes, d_table, d_totals));
    }
    res->t_emit_ms += t.stop();
  }
  set_sdbg_totals(res, one_pass ? tot : out.tot);
  if (!one_pass) memcpy(res->bucket_table, out.table.data(), sizeof(res->bucket_table));
  res->bytes = (uint8_t *)malloc(std::max<size_t>(1, res->n_bytes));
  if (!res->bytes) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  if (res->n_bytes && one_pass) CK(cudaMemcpy(res->bytes, d_bytes, res->n_bytes, cudaMemcpyDeviceToHost));
  else if (res->n_bytes) memcpy(res->bytes, out.bytes.data(), res->n_bytes);
  res->t_total_ms = t_all.stop();
  return MHB_OK;
}

extern "C" int mhb_set_s2s_chunk_limit(uint64_t bytes) {
  g_s2s_chunk_limit = bytes;
  return MHB_OK;
}

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
  *resident_bytes = s2s_resident_round_bytes(n_seqs, n_words, k);
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
  const uint64_t ns = args->n_seqs;
  g_s2s_st = StreamStats();
  g_s2s_rounds = 0;

  SeqLayout ly;
  seq_layout(args->word_off, args->len, ns, k, &ly);
  const uint64_t n_items = ly.n_items, n_words = ly.n_words;
  res->n_records = n_items;

  // A13: items that do not fit the device at once (or a caller-imposed cap) -> rounds over leading-byte ranges; the
  // sequences are streamed when a chunk cap is set or when they leave no room for even a one-item round
  const size_t need = SeqSource::resident_bytes(ns, n_words) + s2s_table_bytes(false) +
                      s2s_round_bytes(n_items, s2s_record_words(k), k);
  bool rounds = g_s2s_round_limit && n_items > g_s2s_round_limit;
  if (!rounds && need > g_arena.cap) {
    rounds = (double)need > arena_avail_bytes();
  }
  const bool stream = g_s2s_chunk_limit != 0 ||
                      (rounds && mhb_read_stream_decide(s2s_resident_round_bytes(ns, n_words, k), (uint64_t)arena_avail_bytes(), 0, 0));
  SeqSource src(args, ly);
  CKR(src.init(stream ? (g_s2s_chunk_limit ? g_s2s_chunk_limit : read_chunk_auto_bytes()) : 0));
  return s2s_host_rounds(args, res, src, n_items, g_s2s_round_limit, !rounds && !stream);
}

// ================================================================================================
// fused k_min build: count -> mercy edges -> seq2sdbg, device resident
// ================================================================================================
static int build_host_impl(const mhb_build_args *args, mhb_build_result *res, bool full_index);

// A13 for the fused build: when the records of the whole library do not fit next to it in HBM (or a round cap is set),
// the same graph is built stage by stage through the host-level calls that already work in rounds - count (rounds over
// bucket ranges) -> mercy edges -> seq2sdbg (rounds over bucket ranges) - with the solid edges passing through host
// memory once, as they do between the reference's two sub-commands (base_engine.cpp:54-141 plans its passes the same
// way: the output does not depend on where the boundaries fall).
static int build_host_rounds(const mhb_build_args *args, mhb_build_result *res) {
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k, WE = words_per_edge(k), NWE = div_ceil(k + 1, 16);
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
  CKR(mhb_count_host(&ca, cr));
  struct Owned {  // the count result's buffers, unless handed on to the caller
    mhb_count_result *r;
    ~Owned() {
      free(r->edges);
      free(r->cand_ids);
    }
  } owned{cr};
  res->n_edge_records = cr->n_edge_records;
  res->n_solid = cr->n_solid;
  res->n_cand = cr->n_cand;
  res->words_per_edge = WE;
  res->words_per_tip_label = words_per_tip_label(k);
  res->t_count_ms = cr->t_total_ms;
  uint32_t *mercy = nullptr;
  uint64_t n_mercy = 0;
  if (args->need_mercy && cr->n_cand) {  // the `.cand` image: candidate reads reversed (kmer_counter.cpp:387-401)
    std::vector<uint32_t> cand;
    uint64_t r = 0;
    size_t pos = 0;
    for (uint64_t c = 0; c < cr->n_cand; ++c) {
      while (r < cr->cand_ids[c]) {
        pos += 1 + div_ceil(args->bin[pos], 16);
        ++r;
      }
      const uint32_t L = args->bin[pos], nw = div_ceil(L, 16);
      const size_t at = cand.size();
      cand.resize(at + 1 + nw, 0u);
      cand[at] = L;
      for (uint32_t i = 0; i < L; ++i) cand[at + 1 + (i >> 4)] |= base_at(&args->bin[pos + 1], L - 1 - i) << (30 - 2 * (i & 15));
    }
    uint64_t n_cr = 0;
    CKR(mhb_mercy_host(k, cr->edges, cr->n_solid, cand.data(), cand.size(), &mercy, &n_mercy, &n_cr));
  }
  struct FreeMercy {
    uint32_t *&p;
    ~FreeMercy() { free(p); }
  } fm{mercy};
  res->n_mercy = n_mercy;
  // the edge (k+1)-mers as seq2sdbg loads them (seq_to_sdbg.cpp:424-450)
  const uint64_t n_seqs = cr->n_solid + n_mercy;
  std::vector<uint32_t> words((size_t)n_seqs * NWE + 1, 0u), len(n_seqs, k + 1);
  std::vector<uint64_t> word_off(n_seqs + 1);
  std::vector<uint16_t> mult(n_seqs);
  const uint32_t tail = (k + 1) % 16;
  for (uint64_t i = 0; i < n_seqs; ++i) {
    const uint32_t *e = i < cr->n_solid ? cr->edges + i * WE : mercy + (i - cr->n_solid) * WE;
    for (uint32_t j = 0; j < NWE; ++j) words[i * NWE + j] = e[j];
    if (tail) words[i * NWE + NWE - 1] &= top_mask(2 * tail);
    word_off[i] = i * NWE;
    mult[i] = (uint16_t)(e[WE - 1] & 0xFFFFu);
  }
  word_off[n_seqs] = n_seqs * NWE;
  mhb_s2s_args sa;
  memset(&sa, 0, sizeof(sa));
  sa.k = k;
  sa.words = words.data();
  sa.word_off = word_off.data();
  sa.len = len.data();
  sa.mult = mult.data();
  sa.n_seqs = n_seqs;
  std::vector<char> sbuf(sizeof(mhb_s2s_result));
  mhb_s2s_result *sr = reinterpret_cast<mhb_s2s_result *>(sbuf.data());
  CKR(mhb_s2s_host(&sa, sr));
  res->n_sort_items = sr->n_records;
  res->n_items = sr->n_items;
  res->n_tips = sr->n_tips;
  res->n_large_mul = sr->n_large_mul;
  res->n_bytes = sr->n_bytes;
  for (int i = 0; i < 9; ++i) res->w_count[i] = sr->w_count[i];
  res->ones_in_last = sr->ones_in_last;
  res->t_s2s_ms = sr->t_total_ms;
  res->bucket_table = (uint64_t *)malloc((size_t)MHB_NUM_BUCKETS * 32);
  if (!res->bucket_table) {
    free(sr->bytes);
    return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  }
  memcpy(res->bucket_table, sr->bucket_table, (size_t)MHB_NUM_BUCKETS * 32);
  if (args->sdbg_out && args->sdbg_out_capacity >= sr->n_bytes) {
    if (sr->n_bytes) memcpy(args->sdbg_out, sr->bytes, sr->n_bytes);
    free(sr->bytes);
    res->bytes = args->sdbg_out;
  } else {
    res->bytes = sr->bytes;
  }
  if (args->want_edges) {
    res->counting = (int64_t *)malloc(65536 * 8);
    if (!res->counting) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
    memcpy(res->counting, cr->counting, 65536 * 8);
    res->edges = cr->edges;
    res->cand_ids = cr->cand_ids;
    cr->edges = nullptr;
    cr->cand_ids = nullptr;
  }
  res->t_total_ms = res->t_count_ms + res->t_s2s_ms;
  return MHB_OK;
}

extern "C" int mhb_build_host(const mhb_build_args *args, mhb_build_result *res) {
  if (!args || !res) return mhb_set_error(MHB_ERR_ARG, "null args");
  // explicit caps (tests, small devices); the staged route uploads the whole library nowhere (count streams it, the
  // mercy edges use the `.cand` reads only)
  if (g_round_limit || g_s2s_round_limit || read_chunk_limit()) return build_host_rounds(args, res);
  const int rc = build_host_impl(args, res, false);
  if (rc == MHB_ERR_NOMEM) {  // everything resident does not fit: the staged build, whose stages plan their own rounds
    mhb_free(res->bytes == args->sdbg_out ? nullptr : res->bytes);
    mhb_free(res->bucket_table);
    mhb_free(res->edges);
    mhb_free(res->cand_ids);
    mhb_free(res->counting);
    mhb_release();
    return build_host_rounds(args, res);
  }
  return rc;
}
static int build_host_impl(const mhb_build_args *args, mhb_build_result *res, bool full_index) {
  memset(res, 0, sizeof(*res));
  const uint32_t k = args->k;
  if (k < 9 || k > MHB_MAX_K) return mhb_set_error(MHB_ERR_ARG, "kmer size must be >= 9 and <= 255");
  if (args->need_mercy && k < 12) return mhb_set_error(MHB_ERR_ARG, "mercy edges need k >= 12");
  if (mhb_device_count() == 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  const uint32_t WR = count_record_words(k), WE = words_per_edge(k), W2 = s2s_record_words(k), WPT = words_per_tip_label(k);
  res->words_per_edge = WE;
  res->words_per_tip_label = WPT;

  ReadLibIndex ix;
  CKR(index_read_lib(args->bin, args->bin_words, args->n_reads, k, &ix, full_index ? FixedCheck::kFull : FixedCheck::kSampled));
  const bool verify_fixed = !full_index && ix.fixed_len != 0;  // the device checks every length word (below)
  const uint64_t n = ix.n_units, n_reads = args->n_reads;
  res->n_edge_records = n;
  uint32_t max_len = ix.fixed_len;
  if (!ix.fixed_len)
    for (uint64_t r = 0; r < n_reads; ++r) max_len = std::max(max_len, args->bin[ix.rec_off[r]]);

  cudaStream_t st = 0;
  EventTimer t_all(st), t(st);
  t_all.start();

  uint8_t cbytes[72];
  const uint32_t n_csort = mhb_count_sort_bytes(k, cbytes);
  const int32_t m = args->m;
  const uint64_t cap_edges = n / (uint64_t)std::max(1, m) + 1;
  const size_t bin_bytes = (args->bin_words * 4 + 15) & ~(size_t)15;
  const CountWork cw = count_work_plan(n, k, m);
  const size_t count_work = 2 * pad256((size_t)n * WR * 4 + 16) + pad256(cw.bytes);
  // fixed part
  size_t fixed = pad256(bin_bytes + 16) + pad256((size_t)cap_edges * WE * 4) + pad256(cap_edges) +
                 pad256(65536 * 8) + 2 * pad256(256 * 8) + pad256(64) + pad256((size_t)MHB_NUM_BUCKETS * 32) +
                 pad256(128) + 8192;
  if (!ix.fixed_len) fixed += 2 * pad256((n_reads + 1) * 8);
  if (args->need_mercy) fixed += 2 * pad256((n_reads + 1) * 4) + pad256((n_reads + 1) * 8);
  CKR(g_arena.reserve(fixed + count_work));

  uint32_t *d_bin = g_arena.take<uint32_t>(bin_bytes / 4 + 4);
  uint32_t *d_edges = g_arena.take<uint32_t>((size_t)cap_edges * WE);
  uint8_t *d_aux = g_arena.take<uint8_t>(cap_edges);
  uint64_t *d_mul_hist = g_arena.take<uint64_t>(65536);
  uint64_t *d_hist0 = g_arena.take<uint64_t>(256);
  uint64_t *d_hist1 = g_arena.take<uint64_t>(256);
  uint64_t *d_nsolid = g_arena.take<uint64_t>(8);
  uint64_t *d_table = g_arena.take<uint64_t>((size_t)MHB_NUM_BUCKETS * 4);
  uint64_t *d_totals = g_arena.take<uint64_t>(16);
  uint64_t *d_rec_off = nullptr, *d_edge_off = nullptr, *d_cand = nullptr;
  uint32_t *d_first = nullptr, *d_last = nullptr;
  if (!ix.fixed_len) {
    d_rec_off = g_arena.take<uint64_t>(n_reads + 1);
    d_edge_off = g_arena.take<uint64_t>(n_reads + 1);
  }
  if (args->need_mercy) {
    d_first = g_arena.take<uint32_t>(n_reads + 1);
    d_last = g_arena.take<uint32_t>(n_reads + 1);
    d_cand = g_arena.take<uint64_t>(n_reads + 1);
  }
  char *work = g_arena.take<char>(count_work);
  size_t work_bytes = count_work;
  DevBuf extra;      // separately allocated work area when a later stage outgrows the count stage's
  DevBuf big_edges;  // solid + mercy edges when the mercy edges do not fit behind the solid ones in d_edges
  uint32_t *d_all_edges = d_edges;

  // ---- H2D ----
  // Fixed-length libraries are uploaded in C pieces on a copy stream and the edges of piece i are extracted while piece
  // i+1 is still crossing PCIe, instead of upload-then-extract (C = 4; MHB_H2D_CHUNKS=1 restores the single copy).
  static const int h2d_chunks_env = getenv("MHB_H2D_CHUNKS") ? atoi(getenv("MHB_H2D_CHUNKS")) : 4;
  const bool chunked = h2d_chunks_env > 1 && ix.fixed_len >= k + 1 && n_reads >= (uint64_t)h2d_chunks_env * 64;
  t.start();
  CK(cudaMemsetAsync(d_mul_hist, 0, 65536 * 8, st));
  CK(cudaMemsetAsync(d_hist0, 0, 256 * 8, st));
  CK(cudaMemsetAsync(d_hist1, 0, 256 * 8, st));
  CK(cudaMemsetAsync(d_nsolid, 0, 64, st));
  if (!chunked) {
    if (args->bin_words) CK(cudaMemcpyAsync(d_bin, args->bin, args->bin_words * 4, cudaMemcpyHostToDevice, st));
    if (!ix.fixed_len && n_reads) {
      CK(cudaMemcpyAsync(d_rec_off, ix.rec_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(d_edge_off, ix.unit_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
    }
  }
  res->t_h2d_ms = t.stop();

  mhb_dev_reads reads;
  reads.bin = d_bin;
  reads.bin_words = args->bin_words;
  reads.n_reads = n_reads;
  reads.fixed_len = ix.fixed_len;
  reads.rec_off = d_rec_off;
  reads.edge_off = d_edge_off;

  // ---- count stage ----
  t.start();
  uint32_t *c_a = (uint32_t *)work;
  uint32_t *c_b = (uint32_t *)(work + pad256((size_t)n * WR * 4 + 16));
  char *c_wsp = work + 2 * pad256((size_t)n * WR * 4 + 16);
  if (!chunked) {
    CKR(mhb_count_extract(st, &reads, k, c_a, n, d_hist0, cw.hist_byte));
  } else {
    static cudaStream_t copy_st = nullptr;
    static cudaEvent_t ev[64];
    static bool ev_ready = false;
    if (!ev_ready) {
      CK(cudaStreamCreateWithFlags(&copy_st, cudaStreamNonBlocking));
      for (int i = 0; i < 64; ++i) CK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
      ev_ready = true;
    }
    const int C = std::min(h2d_chunks_env, 60);  // ev[63] is the start marker
    const uint64_t stride = 1 + div_ceil(ix.fixed_len, 16);          // words per read
    const uint64_t per = ((n_reads + C - 1) / C + 3) & ~(uint64_t)3;  // reads per piece, multiple of 4 -> 16-byte aligned
    const uint64_t e_per_read = ix.fixed_len - k;
    cudaEvent_t start_ev = ev[63];
    CK(cudaEventRecord(start_ev, st));  // the copy stream must not run ahead of this call's place in `st`
    CK(cudaStreamWaitEvent(copy_st, start_ev, 0));
    int c = 0;
    for (uint64_t r0 = 0; r0 < n_reads; r0 += per, ++c) {
      const uint64_t r1 = std::min(n_reads, r0 + per);
      const uint64_t w0 = r0 * stride, w1 = r1 * stride;
      CK(cudaMemcpyAsync(d_bin + w0, args->bin + w0, (w1 - w0) * 4, cudaMemcpyHostToDevice, copy_st));
      CK(cudaEventRecord(ev[c], copy_st));
      CK(cudaStreamWaitEvent(st, ev[c], 0));
      mhb_dev_reads piece = reads;
      piece.bin = d_bin + w0;
      piece.bin_words = w1 - w0;
      piece.n_reads = r1 - r0;
      CKR(mhb_count_extract(st, &piece, k, c_a + (size_t)r0 * e_per_read * WR, (r1 - r0) * e_per_read, d_hist0, cw.hist_byte));
    }
  }
  if (verify_fixed) CKR(mhb_check_fixed_len(st, d_bin, n_reads, ix.fixed_len, d_nsolid + 1));
  CKR(run_count_stage(st, cw, c_a, c_b, n, k, m, d_hist0, d_edges, d_aux, cap_edges, d_mul_hist, d_nsolid, c_wsp, nullptr, nullptr));
  uint64_t h_scal[2] = {0, 0};
  CK(cudaMemcpyAsync(h_scal, d_nsolid, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (verify_fixed && h_scal[1]) return build_host_impl(args, res, true);  // not fixed-length after all: indexed path
  const uint64_t n_solid = h_scal[0];
  if (n_solid > cap_edges) return mhb_set_error(MHB_ERR_NOMEM, "internal: solid edges exceed capacity");
  res->n_solid = n_solid;
  res->t_count_ms = t.stop();

  // ---- mercy: per-read marks -> candidates -> mercy edges appended to the solid edges ----
  uint64_t n_cand = 0, n_mercy = 0;
  if (args->need_mercy && n_reads) {
    t.start();
    uint64_t n_tip = 0;
    CKR(mhb_count_tip_edges(st, d_aux, n_solid, &n_tip));
    const size_t ts_bytes = mhb_tipset_bytes(n_tip, k);
    const size_t cs_bytes = mhb_mercy_candidates_scratch_bytes(n_reads);
    // the count stage's work area is free now; small inputs may need more than it offers (12-mer look-up table)
    char *d_tips = work;
    if (pad256(ts_bytes) + pad256(cs_bytes) > work_bytes) {
      CKR(extra.alloc(pad256(ts_bytes) + pad256(cs_bytes), "build: mercy tip set"));
      d_tips = extra.as<char>();
    }
    char *d_cs = d_tips + pad256(ts_bytes);
    CKR(mhb_tipset_build(st, d_edges, d_aux, n_solid, k, d_tips, ts_bytes, n_tip));
    CKR(mhb_count_mark_mercy(st, &reads, k, d_tips, ts_bytes, n_tip, d_first, d_last));
    CKR(mhb_mercy_candidates(st, d_first, d_last, n_reads, d_cand, &n_cand, d_cs, cs_bytes));
    if (n_cand) {
      const size_t ms_bytes = mhb_mercy_edges_scratch_bytes(n_cand, max_len);
      CK(cudaStreamSynchronize(st));  // the tip set / candidate scratch may be released below
      char *d_ms = work;
      if (ms_bytes > work_bytes) {
        CKR(extra.alloc(ms_bytes, "build: mercy edge scratch"));
        d_ms = extra.as<char>();
      }
      // count first (probe + per-read counts + scan), then size the destination: reads that overlap only at their ends
      // can put more mercy edges between two tips than n/m + 1 - n_solid (the reference reserves +25 % and grows,
      // seq_to_sdbg.cpp:371-379; here the exact number is known before anything is written)
      const size_t core = ms_bytes - mhb_edge_lut_bytes();
      void *lut = d_ms + core;
      CKR(mhb_edge_lut_build(st, d_edges, n_solid, k, lut));
      const uint32_t *seg_e[1] = {d_edges};
      const uint64_t seg_n[1] = {n_solid};
      const void *seg_l[1] = {lut};
      CKR(mhb_mercy_edges_count(st, &reads, d_cand, n_cand, max_len, k, 1, seg_e, seg_n, seg_l, nullptr, &n_mercy, d_ms, core));
      if (n_mercy > cap_edges - n_solid) {
        CKR(big_edges.alloc((size_t)(n_solid + n_mercy) * WE * 4 + 16, "build: solid + mercy edges"));
        CK(cudaMemcpyAsync(big_edges.p, d_edges, (size_t)n_solid * WE * 4, cudaMemcpyDeviceToDevice, st));
        d_all_edges = big_edges.as<uint32_t>();
      }
      CKR(mhb_mercy_edges_write(st, &reads, d_cand, n_cand, max_len, k, d_all_edges + (size_t)n_solid * WE, n_mercy, n_mercy,
                                d_ms, core));
    }
    res->t_mercy_ms = t.stop();
  }
  res->n_cand = n_cand;
  res->n_mercy = n_mercy;

  // ---- SdBG stage over solid + mercy edges, straight from the device-resident edge records ----
  t.start();
  const uint64_t n_seqs = n_solid + n_mercy;
  const uint64_t n_items = n_seqs * 6;  // 2 strands x (k+1 - k + 2)
  res->n_sort_items = n_items;
  const size_t s_ws = mhb_s2s_sort_emit_workspace_bytes(n_items, k);
  const uint64_t cap_bytes = n_items * (4ull + 4ull * WPT) + 16;
  const size_t s2s_work = 2 * pad256((size_t)n_items * W2 * 4 + 16) + pad256(s_ws) + pad256(cap_bytes);
  char *sw = work;
  if (s2s_work > work_bytes) {
    CK(cudaStreamSynchronize(st));
    CKR(extra.alloc(s2s_work, "build: SdBG stage"));
    sw = extra.as<char>();
  }
  uint32_t *s_a = (uint32_t *)sw;
  uint32_t *s_b = (uint32_t *)(sw + pad256((size_t)n_items * W2 * 4 + 16));
  char *s_wsp = sw + 2 * pad256((size_t)n_items * W2 * 4 + 16);
  uint8_t *d_bytes = (uint8_t *)(s_wsp + pad256(s_ws));
  mhb_dev_seqs seqs;
  memset(&seqs, 0, sizeof(seqs));
  seqs.words = d_all_edges;
  seqs.n_words = n_seqs * WE;
  seqs.n_seqs = n_seqs;
  seqs.fixed_len = k + 1;
  seqs.fixed_stride = WE;
  // the solid edges still have the count stage's in/out flags: the $-items the emitter would discard for certain are
  // not generated (mhb_s2s_extract_edges_pruned; 2.02 instead of 6 items per edge on a 30x genome), same bytes out
  static const bool no_prune = getenv("MHB_S2S_NO_PRUNE") != nullptr;
  uint64_t n_sorted = n_items;
  if (!no_prune) {
    CK(cudaMemsetAsync(d_nsolid + 4, 0, 8, st));
    CKR(mhb_s2s_extract_edges_pruned(st, d_all_edges, d_aux, n_seqs, n_solid, k, s_a, n_items, d_nsolid + 4, d_hist1, mhb_s2s_sort_hist_byte(n_items, k)));
    CK(cudaMemcpyAsync(&n_sorted, d_nsolid + 4, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (n_sorted > n_items) return mhb_set_error(MHB_ERR_CUDA, "internal: pruned item count exceeds 6 per edge");
    res->n_sort_items = n_sorted;
  } else {
    CKR(mhb_s2s_extract(st, &seqs, k, s_a, n_items, d_hist1, mhb_s2s_sort_hist_byte(n_items, k)));
  }
  // the extraction histogrammed the byte a sort of n_items (the bound) starts with; the pruned count may start with another
  const bool hist_ok = mhb_s2s_sort_hist_byte(n_sorted, k) == mhb_s2s_sort_hist_byte(n_items, k);
  CKR(mhb_s2s_sort_emit(st, s_a, s_b, n_sorted, k, hist_ok ? d_hist1 : nullptr, d_bytes, cap_bytes, d_table, d_totals, s_wsp, s_ws));
  uint64_t totals[16];
  CK(cudaMemcpyAsync(totals, d_totals, sizeof(totals), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  res->t_s2s_ms = t.stop();
  set_sdbg_totals(res, totals);
  if (res->n_bytes > cap_bytes) return mhb_set_error(MHB_ERR_NOMEM, "internal: SdBG byte stream exceeds capacity");

  // ---- D2H ----
  t.start();
  res->bucket_table = (uint64_t *)malloc((size_t)MHB_NUM_BUCKETS * 32);
  if (args->sdbg_out && args->sdbg_out_capacity >= res->n_bytes) res->bytes = args->sdbg_out;
  else res->bytes = (uint8_t *)malloc(std::max<size_t>(1, res->n_bytes));
  if (!res->bucket_table || !res->bytes) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  CK(cudaMemcpyAsync(res->bucket_table, d_table, (size_t)MHB_NUM_BUCKETS * 32, cudaMemcpyDeviceToHost, st));
  if (res->n_bytes) CK(cudaMemcpyAsync(res->bytes, d_bytes, res->n_bytes, cudaMemcpyDeviceToHost, st));
  if (args->want_edges) {
    res->edges = (uint32_t *)malloc(std::max<size_t>(1, (size_t)n_solid * WE * 4));
    res->cand_ids = (uint64_t *)malloc(std::max<size_t>(1, n_cand * 8));
    res->counting = (int64_t *)malloc(65536 * 8);
    if (!res->edges || !res->cand_ids || !res->counting) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
    if (n_solid) CK(cudaMemcpyAsync(res->edges, d_edges, (size_t)n_solid * WE * 4, cudaMemcpyDeviceToHost, st));
    if (n_cand) CK(cudaMemcpyAsync(res->cand_ids, d_cand, n_cand * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(res->counting, d_mul_hist, 65536 * 8, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  res->t_d2h_ms = t.stop();
  res->t_total_ms = t_all.stop();
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
  *slot_bytes = pad256(max_seg * words_per_edge(k) * 4 + 16);
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
  const uint32_t WE = words_per_edge(k);
  g_mercy_st = StreamStats();
  // `.cand` holds the reads as KmerCounter held them: REVERSED (kmer_counter.cpp:387-401; read back with reverse=false,
  // seq_to_sdbg.cpp:175-176).  The device kernels take a library in file orientation and apply the reversal themselves,
  // so every candidate read is turned around once here (they are ~0.2 % of a library).
  std::vector<uint32_t> bin;
  std::vector<uint64_t> rec_off, edge_off;
  bin.reserve(cand_words + 8);
  uint32_t max_len = 0;
  uint64_t pos = 0, e = 0;
  while (pos < cand_words) {
    const uint32_t L = cand_bin[pos], nw = div_ceil(L, 16);
    if (pos + 1 + nw > cand_words) return mhb_set_error(MHB_ERR_IO, "candidate read image is truncated");
    rec_off.push_back(bin.size());
    edge_off.push_back(e);
    if (L >= k + 1) e += L - k;
    const size_t at = bin.size();
    bin.resize(at + 1 + nw, 0);
    bin[at] = L;
    for (uint32_t i = 0; i < L; ++i)
      bin[at + 1 + (i >> 4)] |= base_at(cand_bin + pos + 1, L - 1 - i) << (30 - 2 * (i & 15));
    max_len = std::max(max_len, L);
    pos += 1 + nw;
  }
  const uint64_t n_reads = rec_off.size();
  rec_off.push_back(bin.size());
  edge_off.push_back(e);
  if (n_cand_reads_out) *n_cand_reads_out = n_reads;
  if (n_reads == 0 || n_edges == 0) {
    *mercy_out = (uint32_t *)malloc(4);
    return MHB_OK;
  }
  const size_t bin_bytes = (bin.size() * 4 + 15) & ~(size_t)15;
  const size_t ms_bytes = mhb_mercy_edges_scratch_bytes(n_reads, max_len);
  const size_t need = mercy_resident_bytes(n_edges, k, n_reads, bin.size(), max_len);
  // The edges are streamed in leading-byte segments when they do not fit next to the candidate reads and the scratch,
  // or when a chunk cap is set: every search stays inside one 12-base prefix, so inside one leading byte and one segment
  const bool stream = g_s2s_chunk_limit != 0 ||
                      (need > g_arena.cap && mhb_read_stream_decide(need, (uint64_t)arena_avail_bytes(), 0, 0));
  const size_t pw = stream ? mhb_mercy_planes_words(n_reads, max_len) : 0;
  const size_t fixed_b = mercy_stream_fixed_bytes(n_reads, bin.size(), max_len);
  uint64_t start[257];
  std::vector<uint32_t> seg_first;
  size_t slot_bytes = 0;
  if (stream) {
    uint64_t target = g_s2s_chunk_limit, limit = g_s2s_chunk_limit;
    if (!target) mercy_auto_segment_bytes(arena_avail_bytes(), fixed_b, &target, &limit);
    edge_byte_starts(edges, n_edges, WE, start);
    CKR(plan_mercy_segments(start, WE, target, limit, &seg_first));
    uint64_t max_seg = 0;
    for (size_t i = 0; i + 1 < seg_first.size(); ++i) max_seg = std::max(max_seg, start[seg_first[i + 1]] - start[seg_first[i]]);
    slot_bytes = pad256(max_seg * WE * 4 + 16);
  }
  CKR(g_arena.reserve(stream ? fixed_b + 2 * slot_bytes : need));
  cudaStream_t st = 0;
  uint32_t *d_bin = g_arena.take<uint32_t>(bin_bytes / 4 + 4);
  uint64_t *d_rec_off = g_arena.take<uint64_t>(n_reads + 1);
  uint64_t *d_edge_off = g_arena.take<uint64_t>(n_reads + 1);
  uint64_t *d_ids = g_arena.take<uint64_t>(n_reads + 1);
  uint32_t *d_edges = stream ? nullptr : g_arena.take<uint32_t>((size_t)n_edges * WE + 4);
  char *d_ms = g_arena.take<char>(ms_bytes);
  std::vector<uint64_t> ids(n_reads);
  for (uint64_t r = 0; r < n_reads; ++r) ids[r] = r;
  CK(cudaMemcpyAsync(d_bin, bin.data(), bin.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_rec_off, rec_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_edge_off, edge_off.data(), (n_reads + 1) * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_ids, ids.data(), n_reads * 8, cudaMemcpyHostToDevice, st));
  if (!stream) CK(cudaMemcpyAsync(d_edges, edges, (size_t)n_edges * WE * 4, cudaMemcpyHostToDevice, st));
  mhb_dev_reads reads;
  reads.bin = d_bin;
  reads.bin_words = bin.size();
  reads.n_reads = n_reads;
  reads.fixed_len = 0;
  reads.rec_off = d_rec_off;
  reads.edge_off = d_edge_off;
  const size_t core = ms_bytes - mhb_edge_lut_bytes();
  void *lut = d_ms + core;
  uint64_t n_mercy = 0;
  if (!stream) {
    CKR(mhb_edge_lut_build(st, d_edges, n_edges, k, lut));
    const uint32_t *seg_e[1] = {d_edges};
    const uint64_t seg_n[1] = {n_edges};
    const void *seg_l[1] = {lut};
    CKR(mhb_mercy_edges_count(st, &reads, d_ids, n_reads, max_len, k, 1, seg_e, seg_n, seg_l, nullptr, &n_mercy, d_ms, core));
  } else {
    // segment i answers the searches whose leading byte it holds; the answers of all segments are OR-ed into one set
    // of planes, which then stands for the single-segment search
    uint32_t *d_planes = g_arena.take<uint32_t>(pw);
    char *d_slots = g_arena.take<char>(2 * slot_bytes);
    const uint64_t n_seg = seg_first.size() - 1;
    uint8_t owner[256];
    for (uint64_t i = 0; i < n_seg; ++i)
      for (uint32_t b = seg_first[i]; b < seg_first[i + 1]; ++b) owner[b] = (uint8_t)i;
    CK(cudaMemsetAsync(d_planes, 0, pw * 4, st));
    ChunkStager stager;
    g_mercy_st.chunks = n_seg;
    CKR(stager.init(slot_bytes, n_seg, &g_mercy_st));
    stager.bind(d_slots);
    auto seg_edges = [&](uint64_t i) { return start[seg_first[i + 1]] - start[seg_first[i]]; };
    const ChunkStager::Fill fill = [&](uint64_t i, char *h, ChunkStager::Copies *up) {
      const uint64_t bytes = seg_edges(i) * WE * 4, blk = 4ull << 20, nblk = (bytes + blk - 1) / blk;
      const char *src = (const char *)(edges + start[seg_first[i]] * WE);
#pragma omp parallel for schedule(static)
      for (long long j = 0; j < (long long)nblk; ++j) {
        const uint64_t o = (uint64_t)j * blk;
        memcpy(h + o, src + o, std::min(blk, bytes - o));
      }
      up->add(0, bytes);
      return MHB_OK;
    };
    const ChunkStager::Run run = [&](uint64_t i, const char *slot) {
      const uint32_t *d_seg = (const uint32_t *)slot;
      CKR(mhb_edge_lut_build(st, d_seg, seg_edges(i), k, lut));
      return mercy_probe_owned(st, &reads, d_ids, n_reads, max_len, k, d_seg, seg_edges(i), lut, owner, (uint32_t)i, d_planes,
                               true);
    };
    CKR(stager.pass(st, fill, run));
    CKR(mhb_mercy_count_planes(st, &reads, d_ids, n_reads, max_len, k, d_planes, 1, pw, &n_mercy, d_ms, core));
  }
  *mercy_out = (uint32_t *)malloc(std::max<size_t>(4, (size_t)n_mercy * WE * 4));
  if (!*mercy_out) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  if (n_mercy) {
    DevBuf out;
    int rc = out.alloc((size_t)n_mercy * WE * 4, "mercy: edges");
    if (!rc) rc = mhb_mercy_edges_write(st, &reads, d_ids, n_reads, max_len, k, out.as<uint32_t>(), n_mercy, n_mercy, d_ms, core);
    if (!rc && cudaMemcpyAsync(*mercy_out, out.p, (size_t)n_mercy * WE * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = mhb_set_error(MHB_ERR_CUDA, "mercy edge download failed");
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess)
      rc = mhb_set_error(MHB_ERR_CUDA, "mercy edge kernels failed: %s", cudaGetErrorString(cudaGetLastError()));
    out.release();
    if (rc) {
      free(*mercy_out);
      *mercy_out = nullptr;
      return rc;
    }
  }
  *n_mercy_out = n_mercy;
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
