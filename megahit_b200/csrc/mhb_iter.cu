// mhb_iter.cu -- `iterate` on the device (SURVEY.md 8f N2): host-level entry point mhb_iterate_host and the host mirror
// used by the CPU tests.  Kernels and building blocks: mhb_iter.cuh.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "mhb_common.cuh"
#include "mhb_iter.cuh"

using namespace mhb;

int scan32(cudaStream_t st, const uint32_t *in, uint64_t n, uint64_t *out, uint64_t *total_dev, uint64_t *bsum);

namespace {

// ascending byte positions of a record of `words` words that hold the first `bits` bits (from the top)
uint32_t top_bytes(uint32_t words, uint32_t bits, uint8_t *out) {
  const uint32_t lo = (32 * words - bits) / 8;
  uint32_t n = 0;
  for (uint32_t b = lo; b < 4 * words; ++b) out[n++] = (uint8_t)b;
  return n;
}

// register words for the kernels: capacity classes instead of one instantiation per width
int cap_class(uint32_t words) { return words <= 2 ? 2 : words <= 4 ? 4 : words <= 8 ? 8 : 17; }
#define IT_FOR_WC(M) M(2) M(4) M(8) M(17)

// the kernels' capacity class of (k, step): the wider of the (k+1)-mer keys and the (k+step+1)-mers
int iter_class(uint32_t k, uint32_t step) { return cap_class(std::max(div_ceil(k + step + 1, 16), div_ceil(k + 1, 16))); }

int iter_reads(const mhb_iterate_args *a, const ReadLibIndex &ix, const FlankTable &tab, bool stream, DevBuf *set,
               uint64_t *n_set_out, uint64_t *n_cand_out, uint64_t *n_aligned_out);

// mhb_selftest_iterate_narrow: the narrow flank index at a k whose wide records fit, to compare the two layouts
bool g_iter_force_narrow = false;

}  // namespace

int iterate_check_args(uint32_t k, uint32_t step) {
  // main_iterate.cpp:73-93: step even, 0 < step <= 28
  if (k < 9 || step == 0 || step > 28 || (step & 1)) return mhb_set_error(MHB_ERR_ARG, "iterate: invalid k / step");
  if (words_per_edge(k + step) > 17)
    return mhb_set_error(MHB_ERR_ARG, "iterate: k + step + 1 = %u is beyond the 17-word edge records of the device sort",
                         k + step + 1);
  return MHB_OK;
}

int iter_build_flanks(const mhb_iterate_args *a, IterFlanks *f) {
  const uint32_t k = a->k, step = a->step, K1 = k + 1, wk = div_ceil(K1, 16), frw = wk + 2;
  const int WCc = iter_class(k, step);
  cudaStream_t st = 0;
  DevBuf d_cw, d_co, d_cl, d_fl, d_fl2, d_val, d_ws, d_flag, d_off, d_bsum, d_cnt;
  CKR(d_cnt.alloc(64, "iterate: counters"));
  CK(cudaMemsetAsync(d_cnt.p, 0, 64, st));
  unsigned long long *cnt = d_cnt.as<unsigned long long>();
  f->n = 0;
  f->tab.release();
  if (a->n_contigs) {
    const uint64_t cw = a->contig_word_off[a->n_contigs];
    CKR(d_cw.alloc(cw * 4 + 64, "iterate: contigs"));
    CKR(d_co.alloc((a->n_contigs + 1) * 8, "iterate: contig offsets"));
    CKR(d_cl.alloc(a->n_contigs * 4, "iterate: contig lengths"));
    CK(cudaMemcpyAsync(d_cw.p, a->contig_words, cw * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_co.p, a->contig_word_off, (a->n_contigs + 1) * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_cl.p, a->contig_len, a->n_contigs * 4, cudaMemcpyHostToDevice, st));
    const uint64_t cap = 2 * a->n_contigs;
    // wide: {key, ~val} records of frw words.  Narrow (frw beyond the 17-word records of the device sort): key + row
    // index records of wk + 1 words, ~val in a side array.
    const bool narrow = frw > 17 || g_iter_force_narrow;
    const uint32_t srw = narrow ? wk + 1 : frw;
    if (cap >= (1ull << 32) && narrow) return mhb_set_error(MHB_ERR_ARG, "iterate: too many contigs for 32-bit flank rows");
    CKR(d_fl.alloc(cap * srw * 4 + 16, "iterate: flank records"));
    CKR(d_fl2.alloc(cap * srw * 4 + 16, "iterate: flank records (sort buffer)"));
    if (narrow) CKR(d_val.alloc(cap * 8 + 16, "iterate: flank values"));
    IterContigs cs{d_cw.as<u32>(), d_co.as<u64>(), d_cl.as<u32>(), a->n_contigs};
#define M(WW)                                                                                                    \
  if (WCc == WW)                                                                                                 \
    k_iter_flanks<WW><<<grid_cap(cap, 256, 16), 256, 0, st>>>(cs, k, step, wk, d_fl.as<u32>(), narrow ? d_val.as<u64>() : nullptr, \
                                                       cnt);
    IT_FOR_WC(M)
#undef M
    CK_LAUNCH();
    unsigned long long nf = 0;
    CK(cudaMemcpyAsync(&nf, cnt, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (nf) {
      uint8_t bytes[72];
      uint32_t nb = 0;
      uint8_t kb[72];
      const uint32_t nkb = top_bytes(wk, 2 * K1, kb);  // key bytes inside the key words
      if (narrow) {  // the key alone: the best value of each key is picked from its run afterwards
        for (uint32_t i = 0; i < nkb; ++i) bytes[nb++] = (uint8_t)(kb[i] + 4);  // above the row-index word
      } else {
        // ascending on key, then on ~val: within a key the largest (ext_len, ext_seq) comes first and survives
        for (uint32_t b = 0; b < 8; ++b) bytes[nb++] = (uint8_t)b;               // the two ~val words
        for (uint32_t i = 0; i < nkb; ++i) bytes[nb++] = (uint8_t)(kb[i] + 8);  // the key bytes above them
      }
      const size_t wsb = mhb_sort_workspace_bytes(nf, srw);
      CKR(d_ws.alloc(wsb, "iterate: sort workspace"));
      int in_b = 0;
      if (narrow)
        CKR(mhb_sort_records_relaxed(st, d_fl.as<u32>(), d_fl2.as<u32>(), nf, srw, bytes, nb, nullptr, d_ws.p, wsb, &in_b));
      else
        CKR(mhb_sort_records(st, d_fl.as<u32>(), d_fl2.as<u32>(), nf, srw, bytes, nb, nullptr, d_ws.p, wsb, &in_b));
      const u32 *sorted = in_b ? d_fl2.as<u32>() : d_fl.as<u32>();
      CKR(d_flag.alloc(nf * 4 + 16, "iterate: flags"));
      CKR(d_off.alloc(nf * 8 + 16, "iterate: offsets"));
      CKR(d_bsum.alloc((nf / 4096 + 4) * 8, "iterate: scan sums"));
      k_iter_heads<<<grid_cap(nf, 256, 16), 256, 0, st>>>(sorted, nf, srw, wk, d_flag.as<u32>());
      CK_LAUNCH();
      CKR(scan32(st, d_flag.as<u32>(), nf, d_off.as<u64>(), (uint64_t *)(cnt + 2), d_bsum.as<u64>()));
      unsigned long long nu = 0;
      CK(cudaMemcpyAsync(&nu, cnt + 2, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      CKR(f->tab.alloc((size_t)nu * frw * 4 + 16, "iterate: flank table"));
      if (narrow)
        k_iter_best<<<grid_cap(nf, 256, 16), 256, 0, st>>>(sorted, nf, wk, d_val.as<u64>(), d_flag.as<u32>(), d_off.as<u64>(),
                                                    f->tab.as<u32>());
      else
        k_iter_compact<<<grid_cap(nf, 256, 16), 256, 0, st>>>(sorted, nf, frw, d_flag.as<u32>(), d_off.as<u64>(), f->tab.as<u32>());
      CK_LAUNCH();
      f->n = nu;
    }
  }
  CKR(f->lut.alloc(65537 * 4, "iterate: flank prefix table"));
  CK(cudaMemsetAsync(f->lut.p, 0, 65537 * 4, st));
  if (f->n) {
    k_iter_lut<<<(65537 + 255) / 256, 256, 0, st>>>(f->tab.as<u32>(), f->n, frw, f->lut.as<u32>());
    CK_LAUNCH();
  }
  CK(cudaStreamSynchronize(st));  // the scratch buffers above are freed on return
  return MHB_OK;
}

int iter_collect(const mhb_iterate_args *a, const IterFlanks &f, DevBuf *set, uint64_t *n_set, uint64_t *n_cand,
                 uint64_t *n_aligned) {
  *n_set = *n_cand = *n_aligned = 0;
  set->release();
  ReadLibIndex ix;
  CKR(index_read_lib(a->bin, a->bin_words, a->n_reads, 0, &ix));
  if (!a->n_reads || !f.n) return MHB_OK;
  const FlankTable tab{f.tab.as<u32>(), f.n, div_ceil(a->k + 1, 16), f.lut.as<u32>()};
  // resident; streamed in chunks when a chunk cap is set or when the resident buffers do not fit
  int rc = iter_reads(a, ix, tab, read_chunk_limit() != 0, set, n_set, n_cand, n_aligned);
  if (rc == MHB_ERR_NOMEM && !read_chunk_limit()) rc = iter_reads(a, ix, tab, true, set, n_set, n_cand, n_aligned);
  return rc;
}

extern "C" int mhb_iterate_host(const mhb_iterate_args *a, mhb_iterate_result *res) {
  if (!a || !res) return mhb_set_error(MHB_ERR_ARG, "null argument");
  memset(res, 0, sizeof(*res));
  CKR(iterate_check_args(a->k, a->step));
  if (mhb_device_count() <= 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  const uint32_t w2 = words_per_edge(a->k + a->step);
  res->words_per_edge = w2;
  read_stream_stats_reset();
  cudaStream_t st = 0;
  EventTimer t(st);
  t.start();
  IterFlanks flanks;
  CKR(iter_build_flanks(a, &flanks));
  res->n_flanks = flanks.n;
  DevBuf set;
  uint64_t n_set = 0, n_cand = 0, n_aligned = 0;
  CKR(iter_collect(a, flanks, &set, &n_set, &n_cand, &n_aligned));
  res->edges = (uint32_t *)malloc(std::max<size_t>(4, (size_t)n_set * w2 * 4));
  if (!res->edges) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  if (n_set) CK(cudaMemcpyAsync(res->edges, set.p, (size_t)n_set * w2 * 4, cudaMemcpyDeviceToHost, st));
  res->n_aligned_reads = n_aligned;
  res->n_candidates = n_cand;
  res->n_edges = n_set;
  res->t_total_ms = t.stop();
  return MHB_OK;
}

namespace {
// KmerCollector's set semantics on n records in a (b: same-sized buffer): relaxed sort on the key bytes, then the first
// record of every run of equal records; *out points at the n_out unique records (in a or b)
int sort_unique(cudaStream_t st, u32 *a, u32 *b, uint64_t n, uint32_t w2, uint32_t KN, DevBuf &ws, DevBuf &flag, DevBuf &off,
                DevBuf &bsum, unsigned long long *cnt_slot, u32 **out, uint64_t *n_out) {
  uint8_t bytes[72];
  const uint32_t nb = top_bytes(w2, 2 * KN, bytes);
  const size_t wsb = mhb_sort_workspace_bytes(n, w2);
  CKR(ws.ensure(wsb, "iterate: sort workspace"));
  int in_b = 0;
  CKR(mhb_sort_records_relaxed(st, a, b, n, w2, bytes, nb, nullptr, ws.p, wsb, &in_b));
  const u32 *sorted = in_b ? b : a;
  u32 *uniq = in_b ? a : b;
  CKR(flag.ensure(n * 4 + 16, "iterate: flags"));
  CKR(off.ensure(n * 8 + 16, "iterate: offsets"));
  CKR(bsum.ensure((n / 4096 + 4) * 8, "iterate: scan sums"));
  k_iter_heads<<<grid_cap(n, 256, 16), 256, 0, st>>>(sorted, n, w2, w2, flag.as<u32>());
  CK_LAUNCH();
  CKR(scan32(st, flag.as<u32>(), n, off.as<u64>(), (uint64_t *)cnt_slot, bsum.as<u64>()));
  unsigned long long nu = 0;
  CK(cudaMemcpyAsync(&nu, cnt_slot, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  k_iter_compact<<<grid_cap(n, 256, 16), 256, 0, st>>>(sorted, n, w2, flag.as<u32>(), off.as<u64>(), uniq);
  CK_LAUNCH();
  *out = uniq;
  *n_out = nu;
  return MHB_OK;
}

// The reads (init_read_stream: resident, or streamed from host memory in chunks), the flank index resident: per
// chunk mark + emit into a mark array of the chunk's bases, make the chunk's candidates unique and merge them into the
// running set by the same sort + unique over the union.  KmerCollector is a set, so the result does not depend on the
// chunks.
int iter_reads(const mhb_iterate_args *a, const ReadLibIndex &ix, const FlankTable &tab, bool stream, DevBuf *set,
               uint64_t *n_set_out, uint64_t *n_cand_out, uint64_t *n_aligned_out) {
  const uint32_t k = a->k, step = a->step, KN = k + step + 1, w2 = words_per_edge(k + step);
  const int WCc = iter_class(k, step);
  cudaStream_t st = 0;
  ChunkStream rs;
  const uint64_t cap = read_chunk_limit() ? read_chunk_limit() : read_chunk_auto_bytes();
  CKR(init_read_stream(&rs, a->bin, a->bin_words, a->n_reads, ix, stream ? cap : 0));
  const std::vector<uint64_t> &first = rs.bounds();
  auto bases_of = [&](uint64_t b, uint64_t e) { return ix.fixed_len ? (e - b) * ix.fixed_len : ix.unit_off[e] - ix.unit_off[b]; };
  uint64_t max_bases = 0;
  for (uint64_t i = 0; i + 1 < first.size(); ++i) max_bases = std::max(max_bases, bases_of(first[i], first[i + 1]));
  DevBuf d_lib, d_exist, d_cnt;
  CKR(d_cnt.alloc(64, "iterate: counters"));
  unsigned long long *cnt = d_cnt.as<unsigned long long>();
  CKR(d_lib.alloc(rs.device_bytes(), stream ? "iterate: read chunk buffers" : "iterate: .bin image"));
  CKR(rs.bind(d_lib.p, st));
  CKR(d_exist.alloc((max_bases / 32 + 2) * 4, "iterate: position marks"));
  DevBuf c, c2, u, u2, ws, flag, off, bsum;
  uint64_t n_cand = 0, n_set = 0, n_aligned = 0;
  auto chunk = [&](const ChunkView &v) -> int {
    IterReads rd{v.words, v.n, ix.fixed_len, v.at<uint64_t>(0), v.at<uint64_t>(1)};
    const uint64_t bw = bases_of(v.first, v.first + v.n) / 32 + 2;
    CK(cudaMemsetAsync(d_exist.p, 0, bw * 4, st));
    CK(cudaMemsetAsync(cnt + 4, 0, 16, st));
#define M(WW)                                                                                                    \
  if (WCc == WW) {                                                                                               \
    k_iter_mark<WW><<<grid_cap(v.n, 128, 32), 128, 0, st>>>(rd, k, step, tab, d_exist.as<u32>());               \
    k_iter_emit<WW, false><<<grid_cap(v.n, 128, 32), 128, 0, st>>>(rd, k, step, d_exist.as<u32>(), w2, nullptr, \
                                                                  cnt + 4, 0);                                   \
  }
    IT_FOR_WC(M)
#undef M
    CK_LAUNCH();
    unsigned long long hc[2] = {0, 0};
    CK(cudaMemcpyAsync(hc, cnt + 4, 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    n_cand += hc[0];
    n_aligned += hc[1];
    if (!hc[0]) return MHB_OK;
    const uint64_t nc = hc[0];
    CKR(c.ensure((size_t)nc * w2 * 4 + 16, "iterate: edges"));
    CKR(c2.ensure((size_t)nc * w2 * 4 + 16, "iterate: edges (sort buffer)"));
    CK(cudaMemsetAsync(cnt + 6, 0, 8, st));
#define M(WW)                                                                                                   \
  if (WCc == WW)                                                                                                \
    k_iter_emit<WW, true><<<grid_cap(v.n, 128, 32), 128, 0, st>>>(rd, k, step, d_exist.as<u32>(), w2, c.as<u32>(), \
                                                                cnt + 6, nc);
    IT_FOR_WC(M)
#undef M
    CK_LAUNCH();
    u32 *cu = nullptr;
    uint64_t ncu = 0;
    CKR(sort_unique(st, c.as<u32>(), c2.as<u32>(), nc, w2, KN, ws, flag, off, bsum, cnt + 7, &cu, &ncu));
    if (n_set == 0) {  // the first candidates are the set: take over their buffers
      const bool in_c = cu == c.as<u32>();
      u.swap(in_c ? c : c2);
      u2.swap(in_c ? c2 : c);
      n_set = ncu;
      return MHB_OK;
    }
    // union = running set followed by this chunk's unique candidates
    const size_t need = (size_t)(n_set + ncu) * w2 * 4 + 16;
    if (need > u.bytes) {
      DevBuf g;
      CKR(g.alloc(std::max(need, 2 * u.bytes), "iterate: edge set"));
      if (n_set) CK(cudaMemcpyAsync(g.p, u.p, (size_t)n_set * w2 * 4, cudaMemcpyDeviceToDevice, st));
      CK(cudaStreamSynchronize(st));
      u.swap(g);
      CKR(u2.ensure(u.bytes, "iterate: edge set (sort buffer)"));
    }
    CK(cudaMemcpyAsync(u.as<u32>() + (size_t)n_set * w2, cu, (size_t)ncu * w2 * 4, cudaMemcpyDeviceToDevice, st));
    u32 *su = nullptr;
    CKR(sort_unique(st, u.as<u32>(), u2.as<u32>(), n_set + ncu, w2, KN, ws, flag, off, bsum, cnt + 7, &su, &n_set));
    if (su != u.as<u32>()) u.swap(u2);
    return MHB_OK;
  };
  CKR(rs.pass(st, chunk));
  CK(cudaStreamSynchronize(st));
  set->swap(u);  // the set leaves with the caller; every other buffer is freed here
  *n_set_out = n_set;
  *n_cand_out = n_cand;
  *n_aligned_out = n_aligned;
  return MHB_OK;
}
}  // namespace

int iter_sort_unique(uint32_t *a, uint32_t *b, uint64_t n, uint32_t k, uint32_t step, uint32_t **out, uint64_t *n_out) {
  *out = a;
  *n_out = 0;
  if (!n) return MHB_OK;
  DevBuf cnt;
  CKR(cnt.alloc(64, "iterate: counters"));
  DevBuf ws, flag, off, bsum;
  CKR(sort_unique(0, a, b, n, words_per_edge(k + step), k + step + 1, ws, flag, off, bsum, cnt.as<unsigned long long>(), out,
                  n_out));
  CK(cudaStreamSynchronize(0));
  return MHB_OK;
}

// mhb_iterate_host with the narrow flank index (key + row index records, values in a side array) at any k: the layout
// mhb_iterate_host takes only when k + 1 > 240, run where both fit so that the tests can compare the two
extern "C" int mhb_selftest_iterate_narrow(const mhb_iterate_args *a, mhb_iterate_result *res) {
  g_iter_force_narrow = true;
  const int rc = mhb_iterate_host(a, res);
  g_iter_force_narrow = false;
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Host mirror for the CPU tests: the same __host__ __device__ building blocks (flank records, flank search, read
// marking, edge emission) driven serially; std::sort stands in for the device radix sort.  Not a compute path of the
// library (nothing calls it but tests/test_iter_cpu.py).
// ------------------------------------------------------------------------------------------------
extern "C" int mhb_selftest_iterate(const mhb_iterate_args *a, mhb_iterate_result *res) {
  if (!a || !res) return mhb_set_error(MHB_ERR_ARG, "null argument");
  memset(res, 0, sizeof(*res));
  const uint32_t k = a->k, step = a->step, K1 = k + 1, KN = k + step + 1;
  if (k < 9 || step == 0 || step > 28 || (step & 1)) return mhb_set_error(MHB_ERR_ARG, "iterate: invalid k / step");
  const uint32_t wk = div_ceil(K1, 16), w2 = words_per_edge(k + step), wn = div_ceil(KN, 16), frw = wk + 2;
  if (w2 > 17) return mhb_set_error(MHB_ERR_ARG, "iterate: record too wide");
  res->words_per_edge = w2;
  const int WCc = cap_class(std::max(wn, wk));
  std::vector<std::vector<u32>> fl;
  for (uint64_t c = 0; c < a->n_contigs; ++c)
    for (u32 strand = 0; strand < 2; ++strand) {
      u32 rec[20];
      bool ok = false;
#define M(WW) \
  if (WCc == WW) ok = iter_flank_record<WW>(a->contig_words + a->contig_word_off[c], a->contig_len[c], k, step, strand, wk, rec);
      IT_FOR_WC(M)
#undef M
      if (ok) fl.emplace_back(rec, rec + frw);
    }
  std::sort(fl.begin(), fl.end());  // key words, then ~val: the largest extension first within a key
  std::vector<u32> tab;
  uint64_t nt = 0;
  for (size_t i = 0; i < fl.size(); ++i)
    if (i == 0 || !std::equal(fl[i].begin(), fl[i].begin() + wk, fl[i - 1].begin())) {
      tab.insert(tab.end(), fl[i].begin(), fl[i].end());
      ++nt;
    }
  std::vector<u32> lut(65537);
  for (u32 p = 0; p <= 65536; ++p) {
    uint64_t lo = 0, hi = nt;
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if ((tab[mid * frw] >> 16) < p) lo = mid + 1; else hi = mid;
    }
    lut[p] = (u32)lo;
  }
  res->n_flanks = nt;
  FlankTable t{tab.data(), nt, wk, lut.data()};
  ReadLibIndex ix;
  CKR(index_read_lib(a->bin, a->bin_words, a->n_reads, 0, &ix));
  IterReads rd{a->bin, a->n_reads, ix.fixed_len, ix.rec_off.data(), ix.unit_off.data()};
  std::vector<u32> exist(ix.n_units / 32 + 2, 0u);
  std::vector<std::vector<u32>> out;
  std::vector<u32> tmp;
  for (uint64_t r = 0; r < a->n_reads && nt; ++r) {
#define M(WW)                                                                          \
  if (WCc == WW) {                                                                     \
    iter_mark_read<WW>(rd, r, k, step, t, exist.data());                               \
    const u32 n = iter_emit_read<WW>(rd, r, k, step, exist.data(), w2, nullptr);       \
    if (n) {                                                                           \
      tmp.assign((size_t)n * w2, 0u);                                                  \
      iter_emit_read<WW>(rd, r, k, step, exist.data(), w2, tmp.data());                \
      for (u32 i = 0; i < n; ++i) out.emplace_back(tmp.begin() + (size_t)i * w2, tmp.begin() + (size_t)(i + 1) * w2); \
      ++res->n_aligned_reads;                                                          \
    }                                                                                  \
  }
    IT_FOR_WC(M)
#undef M
  }
  res->n_candidates = out.size();
  std::sort(out.begin(), out.end());
  out.erase(std::unique(out.begin(), out.end()), out.end());
  res->n_edges = out.size();
  res->edges = (uint32_t *)malloc(std::max<size_t>(4, out.size() * w2 * 4));
  for (size_t i = 0; i < out.size(); ++i) memcpy(res->edges + i * w2, out[i].data(), w2 * 4);
  return MHB_OK;
}
