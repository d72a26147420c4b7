// mhb_files.cpp -- file-level C ABI (include/mhb.h, layer 3): the `count` and `seq2sdbg` sub-commands on
// the reference's on-disk formats.  Host-side IO only; all sorting/counting/mercy-edge search/emission runs on the
// GPU through mhb_count_host / mhb_mercy_host / mhb_s2s_host.
//
// Formats follow voutcn/megahit v1.2.9 (paths relative to src/):
//   read library   sequence/io/sequence_lib.cpp:93-118, sequence/sequence_package.h:224-240
//   edges          sequence/io/edge/edge_io_meta.h:25-70, edge_writer.h:68-111, edge_reader.h:40-138
//   candidates     sorting/kmer_counter.cpp:383-401 ; counting: sorting/edge_counter.h:44-52
//   contigs        sequence/io/contig/contig_reader.h:52-119
//   SdBG           sdbg/sdbg_writer.cpp:25-79, sdbg/sdbg_meta.cpp:12-61
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <fstream>
#include <string>
#include <vector>

#include "mhb.h"
#include "mhb_bits.cuh"
#include "mhb_internal.h"

using namespace mhb;

void HostSeqs::append_packed(const uint32_t *w, uint32_t L, uint16_t m) {
  const uint32_t nw = div_ceil(L, 16);
  const size_t at = words.size();
  words.insert(words.end(), w, w + nw);
  if (L % 16) words[at + nw - 1] &= top_mask(2 * (L % 16));
  word_off.push_back(words.size());
  len.push_back(L);
  mult.push_back(m);
}

void HostSeqs::append_ascii(const char *s, uint32_t L, bool reverse, uint16_t m) {
  static const struct Map {
    uint8_t v[256];
    Map() {
      memset(v, 0, sizeof(v));
      const char *a = "ACGTNacgtn", *b = "0123201232";
      for (int i = 0; i < 10; ++i) v[(int)a[i]] = b[i] - '0';
    }
  } map;
  const uint32_t nw = div_ceil(L, 16);
  const size_t at = words.size();
  words.resize(at + nw, 0);
  for (uint32_t i = 0; i < L; ++i) {
    const uint8_t c = map.v[(uint8_t)s[reverse ? L - 1 - i : i]];
    words[at + (i >> 4)] |= (uint32_t)c << (30 - 2 * (i & 15));
  }
  word_off.push_back(words.size());
  len.push_back(L);
  mult.push_back(m);
}

namespace {

bool read_file(const std::string &path, std::vector<uint32_t> *out, bool must_exist = true) {
  FILE *f = fopen(path.c_str(), "rb");
  if (!f) {
    if (must_exist) mhb_set_error(MHB_ERR_IO, "cannot open %s", path.c_str());
    return false;
  }
  fseek(f, 0, SEEK_END);
  const long sz = ftell(f);
  fseek(f, 0, SEEK_SET);
  out->resize(((size_t)sz + 3) / 4 + 4, 0);  // padded so the image can be handed to the device as is
  const size_t got = sz ? fread(out->data(), 1, (size_t)sz, f) : 0;
  fclose(f);
  if (got != (size_t)sz) {
    mhb_set_error(MHB_ERR_IO, "short read on %s", path.c_str());
    return false;
  }
  out->resize(((size_t)sz + 3) / 4);
  return true;
}

// ------------------------------------------------------------------------------------------------
// edges
// ------------------------------------------------------------------------------------------------
struct EdgeMeta {
  uint32_t kmer_size = 0, words_per_edge = 0, num_files = 0, num_buckets = 0;
  int64_t num_edges = 0;
  int is_sorted = 1;
  struct B {
    int file_id;
    int64_t off, cnt;
  };
  std::vector<B> buckets;
};

bool scan_field(std::istream &is, const char *name, long long *v) {  // utils.h ScanField
  std::string s;
  if (!(is >> s) || s != name || !(is >> *v)) {
    mhb_set_error(MHB_ERR_IO, "Invalid format. Expect field %s", name);
    return false;
  }
  return true;
}

int read_edge_meta(const std::string &prefix, EdgeMeta *m) {
  std::ifstream is(prefix + ".edges.info");
  if (!is) return mhb_set_error(MHB_ERR_IO, "cannot open %s.edges.info", prefix.c_str());
  long long v[6];
  const char *names[6] = {"kmer_size", "words_per_edge", "num_files", "num_buckets", "num_edges", "is_sorted"};
  for (int i = 0; i < 6; ++i)
    if (!scan_field(is, names[i], &v[i])) return MHB_ERR_IO;
  m->kmer_size = (uint32_t)v[0];
  m->words_per_edge = (uint32_t)v[1];
  m->num_files = (uint32_t)v[2];
  m->num_buckets = (uint32_t)v[3];
  m->num_edges = v[4];
  m->is_sorted = (int)v[5];
  m->buckets.resize(m->num_buckets);
  for (uint32_t i = 0; i < m->num_buckets; ++i) {
    long long id;
    is >> id >> m->buckets[i].file_id >> m->buckets[i].off >> m->buckets[i].cnt;
    if (!is || id != (long long)i) return mhb_set_error(MHB_ERR_IO, "Invalid format: bucket id not matched!");
    if (m->buckets[i].file_id >= (int)m->num_files)
      return mhb_set_error(MHB_ERR_IO, "Record ID %d is greater than number of files %u", m->buckets[i].file_id, m->num_files);
  }
  return MHB_OK;
}

// All edges in reader order (edge_reader.h:40-138): bucket order when sorted, file order otherwise.
int read_all_edges(const std::string &prefix, EdgeMeta *meta, std::vector<uint32_t> *edges) {
  if (int rc = read_edge_meta(prefix, meta)) return rc;
  const uint32_t W = meta->words_per_edge;
  std::vector<std::vector<uint32_t>> files(meta->num_files);
  for (uint32_t i = 0; i < meta->num_files; ++i)
    if (!read_file(prefix + ".edges." + std::to_string(i), &files[i])) return MHB_ERR_IO;
  edges->clear();
  if (!meta->is_sorted) {
    if (files.empty() || files[0].size() < (size_t)meta->num_edges * W) return mhb_set_error(MHB_ERR_IO, "%s.edges.0 is truncated", prefix.c_str());
    edges->assign(files[0].begin(), files[0].begin() + (size_t)meta->num_edges * W);
    return MHB_OK;
  }
  edges->reserve((size_t)meta->num_edges * W);
  for (const auto &b : meta->buckets) {
    if (b.file_id < 0 || b.cnt == 0) continue;
    const auto &f = files[b.file_id];
    if ((size_t)(b.off + b.cnt) * W > f.size()) return mhb_set_error(MHB_ERR_IO, "%s.edges.%d is truncated", prefix.c_str(), b.file_id);
    edges->insert(edges->end(), f.begin() + (size_t)b.off * W, f.begin() + (size_t)(b.off + b.cnt) * W);
  }
  return MHB_OK;
}

int write_edges(const std::string &prefix, uint32_t k, const uint32_t *edges, uint64_t n) {
  const uint32_t W = words_per_edge(k);
  CKR(write_bytes(prefix + ".edges.0", edges, n * W * 4));
  std::vector<std::vector<int64_t>> cnt(1, std::vector<int64_t>(MHB_NUM_BUCKETS, 0));
  for (uint64_t i = 0; i < n; ++i) cnt[0][edges[i * W] >> 16]++;
  return write_edges_info(prefix, k, W, cnt);
}

// ------------------------------------------------------------------------------------------------
// contigs (contig_reader.h:52-119): FASTA with "flag=F multi=M len=N" comments
// ------------------------------------------------------------------------------------------------
int read_contigs(const std::string &path, uint32_t min_len, uint32_t k_from, uint32_t k_to, bool reverse,
                 HostSeqs *out, int64_t *n_read, unsigned discard_flag = 0) {
  *n_read = 0;
  FILE *f = fopen(path.c_str(), "rb");
  if (!f) return MHB_OK;  // the reference opens a missing file as an empty stream
  {
    const int c0 = fgetc(f), c1 = fgetc(f);
    if (c0 == 0x1f && c1 == 0x8b) {
      fclose(f);
      return mhb_set_error(MHB_ERR_IO, "%s is gzip-compressed: the GPU seq2sdbg reads plain FASTA contigs only", path.c_str());
    }
    rewind(f);
  }
  const bool extend_loop = k_from < k_to;
  std::string header, seq, line;
  char *buf = nullptr;
  size_t cap = 0;
  ssize_t got;
  bool have = false;
  auto flush = [&]() {
    if (!have) return;
    have = false;
    if (seq.size() < min_len) return;
    const size_t sp = header.find_first_of(" \t");
    const std::string comment = sp == std::string::npos ? "" : header.substr(header.find_first_not_of(" \t", sp));
    const unsigned flag = comment.size() > 5 ? (unsigned)(comment[5] - '0') : 0u;
    if (discard_flag & flag) return;  // contig_reader.h:66-69
    const double m = comment.size() > 13 ? atof(comment.c_str() + 13) : 0.0;
    const uint16_t mult = (uint16_t)(int32_t)(m + .5);
    if (extend_loop && (flag & 2u)) {  // contig_flag::kLoop, contig_reader.h:73-86
      if (seq.size() < k_to + 1u) return;
      std::string ss(seq);
      for (uint32_t i = k_from; i < k_to; ++i) ss.push_back(ss[i]);
      out->append_ascii(ss.data(), (uint32_t)ss.size(), reverse, mult);
    } else {
      out->append_ascii(seq.data(), (uint32_t)seq.size(), reverse, mult);
    }
    ++*n_read;
  };
  while ((got = getline(&buf, &cap, f)) >= 0) {
    while (got > 0 && (buf[got - 1] == '\n' || buf[got - 1] == '\r')) --got;
    if (got > 0 && buf[0] == '>') {
      flush();
      header.assign(buf + 1, got - 1);
      seq.clear();
      have = true;
    } else if (have) {
      seq.append(buf, got);
    }
  }
  flush();
  free(buf);
  fclose(f);
  return MHB_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// output formats shared with the multi-GPU workers (mhb_mgpu.cpp)
// ------------------------------------------------------------------------------------------------
int write_bytes(const std::string &path, const void *data, size_t n) {
  FILE *f = fopen(path.c_str(), "wb");
  if (!f) return mhb_set_error(MHB_ERR_IO, "cannot open %s for writing", path.c_str());
  const bool ok = !n || fwrite(data, 1, n, f) == n;
  fclose(f);
  return ok ? MHB_OK : mhb_set_error(MHB_ERR_IO, "write to %s failed", path.c_str());
}

int write_sdbg_info(const std::string &prefix, uint32_t k, uint32_t words_per_tip_label, int num_files,
                    const std::vector<const uint64_t *> &tables) {
  FILE *g = fopen((prefix + ".sdbg_info").c_str(), "w");
  if (!g) return mhb_set_error(MHB_ERR_IO, "cannot open %s.sdbg_info", prefix.c_str());
  fprintf(g, "k %u\nwords_per_tip_label %u\nnum_buckets %d\nnum_files %d\n", k, words_per_tip_label, MHB_NUM_BUCKETS,
          num_files);
  int used = 0;
  for (size_t f = 0; f < tables.size(); ++f)
    for (int b = 0; b < MHB_NUM_BUCKETS; ++b) {
      const uint64_t *t = tables[f] + 4 * (size_t)b;
      if (!t[1]) continue;
      fprintf(g, "%d %d %llu %llu %llu %llu\n", b, (int)f, (unsigned long long)t[0], (unsigned long long)t[1],
              (unsigned long long)t[2], (unsigned long long)t[3]);
      ++used;
    }
  for (int i = used; i < MHB_NUM_BUCKETS; ++i) fprintf(g, "18446744073709551615 18446744073709551615 0 0 0 0\n");
  fclose(g);
  return MHB_OK;
}

int write_edges_info(const std::string &prefix, uint32_t k, uint32_t words_per_edge,
                     const std::vector<std::vector<int64_t>> &counts) {
  const int n_files = (int)counts.size();
  std::vector<int> file_of(MHB_NUM_BUCKETS, -1);
  int64_t n_edges = 0;
  for (int f = 0; f < n_files; ++f)
    for (int b = 0; b < MHB_NUM_BUCKETS; ++b)
      if (counts[f][b]) {
        if (file_of[b] >= 0) return mhb_set_error(MHB_ERR_ARG, "bucket %d landed on two ranks", b);
        file_of[b] = f;
        n_edges += counts[f][b];
      }
  FILE *g = fopen((prefix + ".edges.info").c_str(), "w");
  if (!g) return mhb_set_error(MHB_ERR_IO, "cannot open %s.edges.info for writing", prefix.c_str());
  fprintf(g, "kmer_size %u\nwords_per_edge %u\nnum_files %d\nnum_buckets %d\nnum_edges %lld\nis_sorted 1\n", k,
          words_per_edge, n_files, MHB_NUM_BUCKETS, (long long)n_edges);
  std::vector<int64_t> off(n_files, 0);
  for (int b = 0; b < MHB_NUM_BUCKETS; ++b) {
    const int f = file_of[b];
    if (f < 0) {
      fprintf(g, "%d -1 0 0\n", b);
    } else {
      fprintf(g, "%d %d %lld %lld\n", b, f, (long long)off[f], (long long)counts[f][b]);
      off[f] += counts[f][b];
    }
  }
  fclose(g);
  return MHB_OK;
}

int write_counting(const std::string &prefix, const int64_t *hist) {
  FILE *f = fopen((prefix + ".counting").c_str(), "w");
  if (!f) return mhb_set_error(MHB_ERR_IO, "cannot open %s.counting", prefix.c_str());
  for (int i = 1; i <= MHB_MAX_MUL; ++i) fprintf(f, "%d %lld\n", i, (long long)hist[i]);
  fclose(f);
  return MHB_OK;
}

void append_cand_reversed(const uint32_t *read, std::vector<uint32_t> *out) {
  const uint32_t L = read[0];
  const size_t at = out->size();
  out->resize(at + 1 + div_ceil(L, 16), 0);
  uint32_t *rec = out->data() + at;
  rec[0] = L;
  for (uint32_t i = 0; i < L; ++i) rec[1 + (i >> 4)] |= base_at(read + 1, L - 1 - i) << (30 - 2 * (i & 15));
}

void log_sdbg_summary(const uint64_t tot[16]) {  // seq_to_sdbg.cpp:793-802, read_to_sdbg_s2.cpp:618-626
  char w[9 * 21 + 1];
  int at = 0;
  for (int i = 0; i < 9; ++i) at += snprintf(w + at, sizeof(w) - at, "%llu ", (unsigned long long)tot[4 + i]);
  XINFO("Number of $ A C G T A- C- G- T-:\n");
  XINFO("%s\n", w);
  XINFO("Total number of edges: %llu\n", (unsigned long long)tot[1]);
  XINFO("Total number of ONEs: %llu\n", (unsigned long long)tot[13]);
  XINFO("Total number of $v edges: %llu\n", (unsigned long long)tot[2]);
}

int load_read_lib(const std::string &prefix, std::vector<uint32_t> *bin, long long *n_reads, long long *total_bases) {
  {
    std::ifstream is(prefix + ".lib_info");
    if (!(is >> *total_bases >> *n_reads)) return mhb_set_error(MHB_ERR_IO, "cannot read %s.lib_info", prefix.c_str());
  }
  return read_file(prefix + ".bin", bin) ? MHB_OK : MHB_ERR_IO;
}

// ================================================================================================
// count
// ================================================================================================
extern "C" int mhb_count_run(const mhb_count_opts *o) {
  if (!o || !o->read_lib_file || !o->read_lib_file[0]) return mhb_set_error(MHB_ERR_ARG, "No read library configuration file!");
  if (o->host_mem == 0) return mhb_set_error(MHB_ERR_ARG, "Please specify the host memory!");
  const std::string lib = o->read_lib_file, prefix = o->output_prefix ? o->output_prefix : "out";
  const double t0 = now_s();
  long long total_bases = 0, n_reads = 0;
  std::vector<uint32_t> bin;
  if (int rc = load_read_lib(lib, &bin, &n_reads, &total_bases)) return rc;
  XINFO("%lld reads, %lld bases; k = %u, m = %d\n", n_reads, total_bases, o->k, o->m);

  mhb_count_args a;
  memset(&a, 0, sizeof(a));
  a.k = o->k;
  a.m = o->m;
  a.bin = bin.data();
  a.bin_words = bin.size();
  a.n_reads = (uint64_t)n_reads;
  a.want_mercy = 1;
  std::vector<char> resbuf(sizeof(mhb_count_result));
  mhb_count_result *res = reinterpret_cast<mhb_count_result *>(resbuf.data());
  if (int rc = mhb_count_host(&a, res)) return rc;
  XINFO("GPU count: %llu edge records, h2d %.2f ms, extract %.2f ms, sort %.2f ms (%u passes), count %.2f ms, mercy %.2f ms, d2h %.2f ms\n",
        (unsigned long long)res->n_edge_records, res->t_h2d_ms, res->t_extract_ms, res->t_sort_ms, res->n_sort_passes,
        res->t_count_ms, res->t_mercy_ms, res->t_d2h_ms);

  int rc = write_edges(prefix, o->k, res->edges, res->n_solid);
  if (!rc) {  // kmer_counter.cpp:383-401: the candidate reads
    std::vector<uint32_t> cand;
    uint64_t r = 0;
    size_t pos = 0;
    for (uint64_t c = 0; c < res->n_cand; ++c) {
      for (; r < res->cand_ids[c]; ++r) pos += 1 + div_ceil(bin[pos], 16);
      append_cand_reversed(&bin[pos], &cand);
    }
    rc = write_bytes(prefix + ".cand", cand.data(), cand.size() * 4);
  }
  if (!rc) rc = write_counting(prefix, res->counting);
  XINFO("Total number of candidate reads: %llu (%llu)\n", (unsigned long long)res->n_cand, (unsigned long long)res->n_has_tips);
  XINFO("Total number of solid edges: %llu\n", (unsigned long long)res->n_solid);
  XINFO("count done. Time elapsed: %.4f\n", now_s() - t0);
  mhb_free(res->edges);
  mhb_free(res->cand_ids);
  return rc;
}

// ================================================================================================
// seq2sdbg
// ================================================================================================
static std::string opt_str(const char *s) { return std::string(s ? s : ""); }

int seq2sdbg_check_opts(const mhb_seq2sdbg_opts *o) {
  if (!o) return mhb_set_error(MHB_ERR_ARG, "null options");
  if (opt_str(o->input_prefix).empty() && opt_str(o->contig).empty() && opt_str(o->addi_contig).empty())
    return mhb_set_error(MHB_ERR_ARG, "No input files!");
  if (o->k < 9) return mhb_set_error(MHB_ERR_ARG, "kmer size must be >= 9!");
  if (o->host_mem == 0) return mhb_set_error(MHB_ERR_ARG, "Please specify the host memory!");
  return MHB_OK;
}

// A multi-GPU `count` (mhb_count_run_multi) has already built this very graph - same prefix, same k, mercy edges
// included - while the solid edges were on the devices, and left a marker: nothing to do.
bool seq2sdbg_prebuilt(const mhb_seq2sdbg_opts *o, double t0) {
  const std::string input = opt_str(o->input_prefix), prefix = opt_str(o->output_prefix);
  const uint32_t k = o->k;
  if (!input.empty() && input == prefix && opt_str(o->contig).empty() && opt_str(o->addi_contig).empty() &&
      opt_str(o->local_contig).empty() && o->need_mercy) {
    std::ifstream mk(prefix + ".sdbg_fused");
    unsigned mk_k = 0, mk_mercy = 0, mk_files = 0;
    if (mk && (mk >> mk_k >> mk_mercy >> mk_files) && mk_k == k && mk_mercy == 1) {
      bool all = std::ifstream(prefix + ".sdbg_info").good();
      for (unsigned i = 0; i < mk_files; ++i) all = all && std::ifstream(prefix + ".sdbg." + std::to_string(i)).good();
      if (all) {
        XINFO("SdBG for k = %u was built by the %u-GPU count stage; nothing to do\n", k, mk_files);
        XINFO("seq2sdbg done. Time elapsed: %.4f\n", now_s() - t0);
        return true;
      }
    }
  }
  return false;
}

int seq2sdbg_load(const mhb_seq2sdbg_opts *o, HostSeqs *out) {
  const std::string input = opt_str(o->input_prefix), contig = opt_str(o->contig), bubble = opt_str(o->bubble),
                    addi = opt_str(o->addi_contig), local = opt_str(o->local_contig);
  const uint32_t k = o->k;
  HostSeqs &seqs = *out;
  if (!input.empty()) {  // seq_to_sdbg.cpp:424-434
    EdgeMeta meta;
    std::vector<uint32_t> edges;
    if (int rc = read_all_edges(input, &meta, &edges)) return rc;
    if (meta.kmer_size != k) return mhb_set_error(MHB_ERR_ARG, "edges were built for k=%u, not %u", meta.kmer_size, k);
    const uint32_t W = meta.words_per_edge;
    const size_t n = edges.size() / W;
    seqs.words.reserve(n * div_ceil(k + 1, 16) * 5 / 4);
    for (size_t i = 0; i < n; ++i) seqs.append_packed(&edges[i * W], k + 1, (uint16_t)(edges[i * W + W - 1] & 0xFFFF));
    XINFO("Read %zu edges.\n", n);
    if (o->need_mercy) {  // :436-450
      const double t1 = now_s();
      std::vector<uint32_t> cand;
      if (!meta.is_sorted) return mhb_set_error(MHB_ERR_ARG, "--need_mercy needs sorted edges");
      read_file(input + ".cand", &cand, false);
      // GenMercyEdges (seq_to_sdbg.cpp:171-357) on the device: k_mercy_probe / k_mercy_emit through the host-level ABI
      uint32_t *mercy = nullptr;
      uint64_t nm = 0, nr = 0;
      if (int rc = mhb_mercy_host(k, edges.data(), n, cand.data(), cand.size(), &mercy, &nm, &nr)) return rc;
      uint64_t n_seg = 0;
      mhb_s2s_stream_stats(1, &n_seg, nullptr, nullptr, nullptr);
      if (n_seg) XINFO("Mercy search: edges streamed in %llu leading-byte segments\n", (unsigned long long)n_seg);
      for (uint64_t i = 0; i < nm; ++i) seqs.append_packed(mercy + i * W, k + 1, 1);
      mhb_free(mercy);
      XINFO("Number of reads: %lld, Number of mercy edges: %lld\n", (long long)nr, (long long)nm);
      XINFO("Adding mercy Done. Time elapsed: %.4f\n", now_s() - t1);
    }
  }
  int64_t nr = 0;
  if (!contig.empty()) {  // :452-476
    if (int rc = read_contigs(contig, k + 1, o->k_from, k, true, &seqs, &nr)) return rc;
    XINFO("Read %lld contigs from %s.\n", (long long)nr, contig.c_str());
    if (int rc = read_contigs(bubble, k + 1, 0, 0, true, &seqs, &nr)) return rc;
    XINFO("Read %lld contigs from %s.\n", (long long)nr, bubble.c_str());
  }
  if (!addi.empty()) {
    if (int rc = read_contigs(addi, k + 1, 0, 0, true, &seqs, &nr)) return rc;
    XINFO("Read %lld contigs from %s.\n", (long long)nr, addi.c_str());
  }
  if (!local.empty()) {
    if (int rc = read_contigs(local, k + 1, 0, 0, true, &seqs, &nr)) return rc;
    XINFO("Read %lld contigs from %s.\n", (long long)nr, local.c_str());
  }
  return MHB_OK;
}

extern "C" int mhb_seq2sdbg_run(const mhb_seq2sdbg_opts *o) {
  if (int rc = seq2sdbg_check_opts(o)) return rc;
  const std::string prefix = opt_str(o->output_prefix);
  const uint32_t k = o->k;
  const double t0 = now_s();
  if (seq2sdbg_prebuilt(o, t0)) return MHB_OK;
  HostSeqs seqs;
  if (int rc = seq2sdbg_load(o, &seqs)) return rc;

  mhb_s2s_args a;
  memset(&a, 0, sizeof(a));
  a.k = k;
  if (seqs.words.empty()) seqs.words.push_back(0);
  a.words = seqs.words.data();
  a.word_off = seqs.word_off.data();
  a.len = seqs.len.data();
  a.mult = seqs.mult.data();
  a.n_seqs = seqs.size();
  std::vector<char> resbuf(sizeof(mhb_s2s_result));
  mhb_s2s_result *res = reinterpret_cast<mhb_s2s_result *>(resbuf.data());
  if (int rc = mhb_s2s_host(&a, res)) return rc;
  XINFO("GPU seq2sdbg: %llu sort items, extract %.2f ms, sort %.2f ms, emit %.2f ms\n", (unsigned long long)res->n_records,
        res->t_extract_ms, res->t_sort_ms, res->t_emit_ms);
  {
    uint64_t nc = 0, np = 0, nrd = 0, nb = 0;
    mhb_s2s_stream_stats(0, &nc, &np, &nrd, &nb);
    if (nc) XINFO("GPU seq2sdbg: sequences streamed in %llu chunks, %llu passes, %llu rounds, %.1f MB host to device\n",
                  (unsigned long long)nc, (unsigned long long)np, (unsigned long long)nrd, nb / 1e6);
    else XINFO("GPU seq2sdbg: sequences resident, %llu round(s)\n", (unsigned long long)nrd);
  }

  int rc = write_bytes(prefix + ".sdbg.0", res->bytes, res->n_bytes);  // sdbg_writer.cpp:25-79: one file
  if (!rc) rc = write_sdbg_info(prefix, k, res->words_per_tip_label, res->n_items ? 1 : 0, {res->bucket_table});
  uint64_t tot[16];
  get_sdbg_totals(*res, tot);
  log_sdbg_summary(tot);
  XINFO("seq2sdbg done. Time elapsed: %.4f\n", now_s() - t0);
  mhb_free(res->bytes);
  return rc;
}

// ================================================================================================
// read2sdbg (main_read2sdbg, main_sdbg_build.cpp:88-156)
// ================================================================================================
int read2sdbg_load(const mhb_read2sdbg_opts *o, std::vector<uint32_t> *bin, long long *n_reads_out) {
  if (!o || !o->read_lib_file || !o->read_lib_file[0]) return mhb_set_error(MHB_ERR_ARG, "No input file!");
  if (o->host_mem == 0) return mhb_set_error(MHB_ERR_ARG, "Please specify the host memory!");
  const std::string lib = o->read_lib_file, prefix = o->output_prefix ? o->output_prefix : "out";
  long long total_bases = 0, n_reads = 0;
  if (int rc = load_read_lib(lib, bin, &n_reads, &total_bases)) return rc;
  *n_reads_out = n_reads;
  XINFO("%lld reads, %lld total bases; k = %u, m = %d, need_mercy = %d\n", n_reads, total_bases, o->k, o->m, o->need_mercy);
  // the candidate files stage 1 hands to stage 2 inside the reference process (read_to_sdbg_s1.cpp:111-126: 1, 2, 4 .. 64
  // files by read count); here the candidates never leave the device (three bit planes), the files are created empty so
  // that whatever cleans up after the reference finds them
  int n_mercy_files = 1;
  while (n_mercy_files * 10485760LL < n_reads && n_mercy_files < 64) n_mercy_files <<= 1;
  for (int i = 0; i < n_mercy_files; ++i) {
    FILE *f = fopen((prefix + ".mercy_cand." + std::to_string(i)).c_str(), "wb");
    if (!f) return mhb_set_error(MHB_ERR_IO, "cannot open %s.mercy_cand.%d", prefix.c_str(), i);
    fclose(f);
  }
  return MHB_OK;
}

int read2sdbg_build(const mhb_read2sdbg_opts *o, std::vector<uint32_t> &bin, long long n_reads, double t0) {
  const std::string prefix = o->output_prefix ? o->output_prefix : "out";
  mhb_build_args a;
  memset(&a, 0, sizeof(a));
  a.k = o->k;
  a.m = o->m;
  a.bin = bin.data();
  a.bin_words = bin.size();
  a.n_reads = (uint64_t)n_reads;
  a.need_mercy = o->need_mercy;
  mhb_build_result res;
  if (int rc = mhb_read2sdbg_host(&a, &res)) return rc;
  XINFO("GPU read2sdbg: %llu (k+1)-mer positions, bucket partition %.2f ms, kmsort %.2f ms, %llu mercy edges, %llu sort items, total %.2f ms\n",
        (unsigned long long)res.n_edge_records, res.t_count_ms, res.t_mercy_ms, (unsigned long long)res.n_mercy,
        (unsigned long long)res.n_sort_items, res.t_total_ms);
  int rc = MHB_OK;
  if (o->m > 1) {  // Read2SdbgS1::Lv0Postprocess, read_to_sdbg_s1.cpp:557-566
    rc = write_counting(prefix, res.counting);
    if (o->need_mercy) XINFO("Number mercy: %llu\n", (unsigned long long)res.n_mercy);
  }
  if (!rc) rc = write_bytes(prefix + ".sdbg.0", res.bytes, res.n_bytes);
  if (!rc) rc = write_sdbg_info(prefix, o->k, res.words_per_tip_label, res.n_items ? 1 : 0, {res.bucket_table});
  uint64_t tot[16];
  get_sdbg_totals(res, tot);
  log_sdbg_summary(tot);
  XINFO("read2sdbg done. Time elapsed: %.4f\n", now_s() - t0);
  mhb_free(res.bytes);
  mhb_free(res.bucket_table);
  mhb_free(res.counting);
  return rc;
}

extern "C" int mhb_read2sdbg_run(const mhb_read2sdbg_opts *o) {
  const double t0 = now_s();
  std::vector<uint32_t> bin;
  long long n_reads = 0;
  if (int rc = read2sdbg_load(o, &bin, &n_reads)) return rc;
  return read2sdbg_build(o, bin, n_reads, t0);
}

// ================================================================================================
// iterate (main_iterate, main_iterate.cpp:196-221)
// ================================================================================================
int iterate_check_opts(const mhb_iterate_opts *o) {
  if (!o) return mhb_set_error(MHB_ERR_ARG, "null options");
  if (opt_str(o->contig_file).empty()) return mhb_set_error(MHB_ERR_ARG, "No contig file!");
  if (opt_str(o->bubble_file).empty()) return mhb_set_error(MHB_ERR_ARG, "No bubble file!");
  if (opt_str(o->read_file).empty()) return mhb_set_error(MHB_ERR_ARG, "No reads file!");
  if (o->k == 0) return mhb_set_error(MHB_ERR_ARG, "Invalid kmer size!");
  if (o->step == 0 || o->step > 28 || (o->step & 1)) return mhb_set_error(MHB_ERR_ARG, "Invalid step size!");
  if (opt_str(o->output_prefix).empty()) return mhb_set_error(MHB_ERR_ARG, "No output prefix!");
  return MHB_OK;
}

int iterate_load(const mhb_iterate_opts *o, HostSeqs *seqs, std::vector<uint32_t> *bin, uint64_t *n_reads) {
  if (int rc = iterate_check_opts(o)) return rc;
  const std::string contig = opt_str(o->contig_file), bubble = opt_str(o->bubble_file), reads = opt_str(o->read_file);
  // the flank index reads contigs and bubbles in file orientation, without the standalone and loop ones
  // (async_sequence_reader.h:82-101: SetDiscardFlag(kLoop | kStandalone), reverse = false)
  int64_t nr = 0;
  if (int rc = read_contigs(contig, 0, 0, 0, false, seqs, &nr, 3u)) return rc;
  XINFO("Read %lld contigs\n", (long long)nr);
  if (int rc = read_contigs(bubble, 0, 0, 0, false, seqs, &nr, 3u)) return rc;
  XINFO("Read %lld contigs\n", (long long)nr);
  if (!read_file(reads, bin)) return MHB_ERR_IO;
  *n_reads = 0;
  for (size_t pos = 0; pos < bin->size(); ++*n_reads) pos += 1 + div_ceil((*bin)[pos], 16);  // binary_reader.h:23-53
  return MHB_OK;
}

// edge_writer.h:94-99 / edge_io_meta.h:25-44, unordered
int iterate_write_info(const std::string &prefix, uint32_t k_out, uint32_t words_per_edge, uint64_t n) {
  FILE *g = fopen((prefix + ".edges.info").c_str(), "w");
  if (!g) return mhb_set_error(MHB_ERR_IO, "cannot open %s.edges.info for writing", prefix.c_str());
  fprintf(g, "kmer_size %u\nwords_per_edge %u\nnum_files 1\nnum_buckets 0\nnum_edges %llu\nis_sorted 0\n", k_out,
          words_per_edge, (unsigned long long)n);
  fclose(g);
  return MHB_OK;
}

extern "C" int mhb_iterate_run(const mhb_iterate_opts *o) {
  const double t0 = now_s();
  HostSeqs seqs;
  std::vector<uint32_t> bin;
  uint64_t n_reads = 0;
  if (int rc = iterate_load(o, &seqs, &bin, &n_reads)) return rc;
  const std::string prefix = opt_str(o->output_prefix);
  mhb_iterate_args a;
  memset(&a, 0, sizeof(a));
  a.k = o->k;
  a.step = o->step;
  if (seqs.words.empty()) seqs.words.push_back(0);
  a.contig_words = seqs.words.data();
  a.contig_word_off = seqs.word_off.data();
  a.contig_len = seqs.len.data();
  a.n_contigs = seqs.size();
  a.bin = bin.data();
  a.bin_words = bin.size();
  a.n_reads = n_reads;
  mhb_iterate_result res;
  if (int rc = mhb_iterate_host(&a, &res)) return rc;
  XINFO("Number of flank kmers: %llu\n", (unsigned long long)res.n_flanks);
  XINFO("Total: %llu, aligned: %llu. Iterative edges: %llu\n", (unsigned long long)n_reads,
        (unsigned long long)res.n_aligned_reads, (unsigned long long)res.n_edges);
  int rc = write_bytes(prefix + ".edges.0", res.edges, res.n_edges * res.words_per_edge * 4);
  if (!rc) rc = iterate_write_info(prefix, o->k + o->step, res.words_per_edge, res.n_edges);
  XINFO("iterate done. Time elapsed: %.4f (GPU %.2f ms)\n", now_s() - t0, res.t_total_ms);
  mhb_free(res.edges);
  return rc;
}
