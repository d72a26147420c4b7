// mhb_stream.cu -- read libraries larger than device memory: the `.bin` image stays in host memory and every pass over
// the reads streams it through the device in chunks that end on read boundaries (ReadStream, mhb_internal.h).  The
// count and iterate stages hand each chunk to the same extraction / marking / emission kernels as a resident library.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>

#include "mhb.h"
#include "mhb_bits.cuh"
#include "mhb_common.cuh"

using namespace mhb;

#define CKR(call)        \
  do {                   \
    int rc_ = (call);    \
    if (rc_) return rc_; \
  } while (0)

namespace {
uint64_t g_chunk_limit = 0;
struct {
  uint64_t chunks, passes, h2d_bytes;
  double copy_ms, kernel_ms, fill_ms, pass_ms;
} g_st = {0, 0, 0, 0, 0, 0, 0};

inline size_t pad256(size_t b) { return (b + 255) & ~(size_t)255; }

// Greedy cut into chunks of at most max_bytes of image; a read larger than the cap gets a chunk of its own.
// words_of(r) = image words of read r.  first gets n_chunks + 1 entries.
template <class F>
void plan_chunks(uint64_t n_reads, uint64_t max_bytes, F words_of, std::vector<uint64_t> *first) {
  first->clear();
  first->push_back(0);
  uint64_t acc = 0, in = 0;
  for (uint64_t r = 0; r < n_reads; ++r) {
    const uint64_t b = 4 * words_of(r);
    if (in && acc + b > max_bytes) {
      first->push_back(r);
      acc = 0;
      in = 0;
    }
    acc += b;
    ++in;
  }
  if (n_reads) first->push_back(n_reads);
}
}  // namespace

void read_stream_stats_reset() { memset(&g_st, 0, sizeof(g_st)); }
uint64_t read_chunk_limit() { return g_chunk_limit; }
// 64 MiB: the shortest passes of scripts/read_stream_time.py (DESIGN.md A13); larger chunks overlap less
uint64_t read_chunk_auto_bytes() { return 64ull << 20; }

extern "C" int mhb_set_read_chunk_limit(uint64_t bytes) {
  g_chunk_limit = bytes;
  return MHB_OK;
}

extern "C" int mhb_read_stream_stats(uint64_t *n_chunks, uint64_t *n_passes, uint64_t *h2d_bytes) {
  if (n_chunks) *n_chunks = g_st.chunks;
  if (n_passes) *n_passes = g_st.passes;
  if (h2d_bytes) *h2d_bytes = g_st.h2d_bytes;
  return MHB_OK;
}

extern "C" int mhb_read_stream_times(double *h2d_ms, double *kernel_ms, double *fill_ms, double *pass_ms) {
  if (pass_ms) *pass_ms = g_st.pass_ms;
  if (h2d_ms) *h2d_ms = g_st.copy_ms;
  if (kernel_ms) *kernel_ms = g_st.kernel_ms;
  if (fill_ms) *fill_ms = g_st.fill_ms;
  return MHB_OK;
}

extern "C" int mhb_read_stream_decide(uint64_t resident_bytes, uint64_t avail_bytes, int plan_failed, uint64_t chunk_limit) {
  return chunk_limit != 0 || plan_failed != 0 || resident_bytes >= avail_bytes;
}

extern "C" int mhb_plan_read_chunks(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint64_t max_chunk_bytes,
                                    uint64_t *first_read_out, uint32_t cap_out) {
  if ((n_reads && !bin) || max_chunk_bytes == 0) {
    mhb_set_error(MHB_ERR_ARG, "bad chunk plan arguments");
    return -1;
  }
  std::vector<uint64_t> words(n_reads);
  uint64_t pos = 0;
  for (uint64_t r = 0; r < n_reads; ++r) {
    if (pos >= bin_words) {
      mhb_set_error(MHB_ERR_ARG, ".bin image truncated at read %llu", (unsigned long long)r);
      return -1;
    }
    words[r] = 1 + div_ceil(bin[pos], 16);
    pos += words[r];
  }
  if (pos > bin_words) {
    mhb_set_error(MHB_ERR_ARG, ".bin image truncated");
    return -1;
  }
  std::vector<uint64_t> first;
  plan_chunks(n_reads, max_chunk_bytes, [&](uint64_t r) { return words[r]; }, &first);
  const uint64_t n = first.size() - 1;
  if (first_read_out) {
    if (first.size() > cap_out) {
      mhb_set_error(MHB_ERR_ARG, "chunk plan needs %llu entries, room for %u", (unsigned long long)first.size(), cap_out);
      return -1;
    }
    memcpy(first_read_out, first.data(), first.size() * 8);
  }
  return (int)n;
}

// ------------------------------------------------------------------------------------------------
// ReadStream
// ------------------------------------------------------------------------------------------------
ReadStream::~ReadStream() {
  if (copy_) cudaStreamSynchronize((cudaStream_t)copy_);
  for (void *e : ev_) cudaEventDestroy((cudaEvent_t)e);
  for (char *h : host_)
    if (h) cudaFreeHost(h);
  if (copy_) cudaStreamDestroy((cudaStream_t)copy_);
}

int ReadStream::init(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t fixed_len, const uint64_t *rec_off,
                     const uint64_t *aux_off, uint64_t max_chunk_bytes) {
  bin_ = bin;
  n_reads_ = n_reads;
  fixed_len_ = fixed_len;
  stride_ = fixed_len ? 1 + div_ceil(fixed_len, 16) : 0;
  rec_off_ = rec_off;
  aux_off_ = aux_off;
  if (n_reads && !fixed_len && (!rec_off || !aux_off)) return mhb_set_error(MHB_ERR_ARG, "internal: stream of a variable-length library without offsets");
  (void)bin_words;
  if (fixed_len) {  // the greedy plan in closed form: floor(cap / record) reads per chunk
    const uint64_t per = std::max<uint64_t>(1, max_chunk_bytes / (4 * stride_));
    first_.clear();
    for (uint64_t r = 0; r < n_reads; r += per) first_.push_back(r);
    if (n_reads) first_.push_back(n_reads);
    else first_.push_back(0);
  } else {
    plan_chunks(n_reads, max_chunk_bytes, [&](uint64_t r) { return rec_off[r + 1] - rec_off[r]; }, &first_);
  }
  uint64_t max_words = 0;
  max_reads_ = 0;
  for (uint64_t i = 0; i < n_chunks(); ++i) {
    max_reads_ = std::max(max_reads_, first_[i + 1] - first_[i]);
    max_words = std::max(max_words, word_of(first_[i + 1]) - word_of(first_[i]));
  }
  off_at_ = pad256(max_words * 4 + 64);
  slot_bytes_ = off_at_ + (fixed_len ? 0 : 2 * pad256((max_reads_ + 1) * 8));
  g_st.chunks = n_chunks();
  if (!n_chunks()) return MHB_OK;
  for (int s = 0; s < 2; ++s) CK(cudaHostAlloc((void **)&host_[s], slot_bytes_, cudaHostAllocDefault));
  cudaStream_t cs;
  CK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  copy_ = cs;
  ev_.assign(4 * n_chunks(), nullptr);
  for (auto &e : ev_) CK(cudaEventCreate((cudaEvent_t *)&e));
  return MHB_OK;
}

void ReadStream::bind(void *device_slots) { dev_ = (char *)device_slots; }

// fill the staging buffer of chunk i (host threads) and queue its upload on the copy stream
int ReadStream::stage(uint64_t i) {
  const int s = (int)(i & 1);
  cudaStream_t cs = (cudaStream_t)copy_;
  if (i >= 2) CK(cudaEventSynchronize((cudaEvent_t)ev_[4 * (i - 2) + 1]));  // upload of chunk i-2 has left staging s
  const auto t0 = std::chrono::steady_clock::now();
  const uint64_t b = first_[i], e = first_[i + 1], w0 = word_of(b), nw = word_of(e) - w0;
  char *h = host_[s];
  {
    const uint64_t bytes = nw * 4, blk = 4ull << 20, nblk = (bytes + blk - 1) / blk;
#pragma omp parallel for schedule(static)
    for (long long j = 0; j < (long long)nblk; ++j) {
      const uint64_t o = (uint64_t)j * blk;
      memcpy(h + o, (const char *)(bin_ + w0) + o, std::min(blk, bytes - o));
    }
  }
  const uint64_t nr = e - b;
  uint64_t *ro = (uint64_t *)(h + off_at_), *ao = (uint64_t *)(h + off_at_ + pad256((max_reads_ + 1) * 8));
  if (!fixed_len_) {
    const uint64_t r0 = rec_off_[b], a0 = aux_off_[b];
#pragma omp parallel for schedule(static)
    for (long long r = 0; r <= (long long)nr; ++r) {
      ro[r] = rec_off_[b + r] - r0;
      ao[r] = aux_off_[b + r] - a0;
    }
  }
  g_st.fill_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  char *d = dev_ + s * slot_bytes_;
  if (i >= 2) CK(cudaStreamWaitEvent(cs, (cudaEvent_t)ev_[4 * (i - 2) + 3], 0));  // kernels of chunk i-2 are done with slot s
  CK(cudaEventRecord((cudaEvent_t)ev_[4 * i], cs));
  if (nw) CK(cudaMemcpyAsync(d, h, nw * 4, cudaMemcpyHostToDevice, cs));
  g_st.h2d_bytes += nw * 4;
  if (!fixed_len_) {
    CK(cudaMemcpyAsync(d + off_at_, ro, (nr + 1) * 8, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(d + off_at_ + pad256((max_reads_ + 1) * 8), ao, (nr + 1) * 8, cudaMemcpyHostToDevice, cs));
    g_st.h2d_bytes += 2 * (nr + 1) * 8;
  }
  CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 1], cs));
  return MHB_OK;
}

int ReadStream::pass(void *stream, const std::function<int(const ReadChunkView &)> &fn) {
  const uint64_t nc = n_chunks();
  if (!nc) return MHB_OK;
  if (!dev_) return mhb_set_error(MHB_ERR_ARG, "internal: read stream without device slots");
  cudaStream_t st = (cudaStream_t)stream;
  ++g_st.passes;
  const auto t0 = std::chrono::steady_clock::now();
  CKR(stage(0));
  for (uint64_t i = 0; i < nc; ++i) {
    // the next upload is queued before the kernels of this chunk, so a host read inside fn does not stall the copy
    if (i + 1 < nc) CKR(stage(i + 1));
    CK(cudaStreamWaitEvent(st, (cudaEvent_t)ev_[4 * i + 1], 0));
    CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 2], st));
    const char *d = dev_ + (i & 1) * slot_bytes_;
    ReadChunkView v;
    v.index = i;
    v.first_read = first_[i];
    v.n_reads = first_[i + 1] - first_[i];
    v.bin = (const uint32_t *)d;
    v.bin_words = word_of(first_[i + 1]) - word_of(first_[i]);
    v.rec_off = fixed_len_ ? nullptr : (const uint64_t *)(d + off_at_);
    v.aux_off = fixed_len_ ? nullptr : (const uint64_t *)(d + off_at_ + pad256((max_reads_ + 1) * 8));
    CKR(fn(v));
    CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 3], st));
  }
  CK(cudaEventSynchronize((cudaEvent_t)ev_[4 * (nc - 1) + 3]));
  CK(cudaStreamSynchronize((cudaStream_t)copy_));
  g_st.pass_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  for (uint64_t i = 0; i < nc; ++i) {
    float a = 0, b = 0;
    CK(cudaEventElapsedTime(&a, (cudaEvent_t)ev_[4 * i], (cudaEvent_t)ev_[4 * i + 1]));
    CK(cudaEventElapsedTime(&b, (cudaEvent_t)ev_[4 * i + 2], (cudaEvent_t)ev_[4 * i + 3]));
    g_st.copy_ms += a;
    g_st.kernel_ms += b;
  }
  return MHB_OK;
}
