// mhb_stream.cu -- the host-side `.bin` index and every pass over an input in host memory (ChunkStream,
// mhb_internal.h): read libraries, sequence sets and sorted edges, resident in device memory or, when larger than
// device memory, kept in host memory and streamed through the device in chunks that end on unit boundaries.  The stages
// hand each chunk to the same kernels whichever form the input takes.
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

namespace {
uint64_t g_chunk_limit = 0;
StreamStats g_st;
size_t g_dev_live = 0, g_dev_peak = 0;  // bytes the process's DevBufs hold, and the most since DevBuf::reset_peak
}  // namespace

size_t free_device_bytes() {
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return free_b;
}

void DevBuf::release() {
  if (p) {
    cudaFree(p);
    g_dev_live -= bytes;
  }
  p = nullptr;
  bytes = 0;
}

int DevBuf::alloc(size_t b, const char *what) {
  release();
  b = pad256(std::max<size_t>(b, 1));
  const cudaError_t e = cudaMalloc(&p, b);
  if (e != cudaSuccess) {
    cudaGetLastError();
    p = nullptr;
    return mhb_set_error(MHB_ERR_NOMEM, "%s: cudaMalloc of %zu bytes failed: %s", what, b, cudaGetErrorString(e));
  }
  bytes = b;
  g_dev_live += b;
  g_dev_peak = std::max(g_dev_peak, g_dev_live);
  return MHB_OK;
}

void DevBuf::reset_peak() { g_dev_peak = g_dev_live; }
size_t DevBuf::peak_bytes() { return g_dev_peak; }

// a library's read chunks: the image only, a fixed-length library cut in closed form
static void plan_read_chunks(const ReadLibIndex &ix, uint64_t n_reads, uint64_t max_bytes, std::vector<uint64_t> *first) {
  plan_chunks(ix.fixed_len ? nullptr : ix.rec_off.data(), 1 + div_ceil(ix.fixed_len, 16), 0, n_reads, max_bytes, first);
}

int index_read_lib(const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, uint32_t k, ReadLibIndex *ix,
                   FixedCheck check) {
  *ix = ReadLibIndex();
  if (n_reads == 0) return MHB_OK;
  if (bin_words == 0) return mhb_set_error(MHB_ERR_ARG, "empty .bin image for %llu reads", (unsigned long long)n_reads);
  const uint32_t L0 = bin[0];
  const uint64_t stride = 1 + div_ceil(L0, 16);
  bool fixed = L0 > 0 && bin_words == n_reads * stride;
  if (fixed && check == FixedCheck::kSampled) {
    const uint64_t step = std::max<uint64_t>(1, n_reads / 1024);
    for (uint64_t r = 0; r < n_reads && fixed; r += step) fixed = bin[r * stride] == L0;
    for (uint64_t r = 0; r < std::min<uint64_t>(n_reads, 1024) && fixed; ++r) fixed = bin[r * stride] == L0;
    fixed = fixed && bin[(n_reads - 1) * stride] == L0;
  } else if (fixed && check == FixedCheck::kSerial) {
    for (uint64_t r = 0; r < n_reads && fixed; ++r) fixed = bin[r * stride] == L0;
  } else if (fixed) {
    int bad = 0;
#pragma omp parallel for reduction(| : bad) schedule(static)
    for (long long r = 0; r < (long long)n_reads; ++r) bad |= bin[(uint64_t)r * stride] != L0;
    fixed = !bad;
  }
  if (fixed) {
    ix->fixed_len = L0;
    ix->n_units = L0 > k ? n_reads * (uint64_t)(L0 - k) : 0;
    return MHB_OK;
  }
  ix->rec_off.resize(n_reads + 1);
  ix->unit_off.resize(n_reads + 1);
  uint64_t pos = 0, u = 0;
  for (uint64_t r = 0; r < n_reads; ++r) {
    if (pos >= bin_words) return mhb_set_error(MHB_ERR_ARG, ".bin image truncated at read %llu", (unsigned long long)r);
    const uint32_t L = bin[pos];
    ix->rec_off[r] = pos;
    ix->unit_off[r] = u;
    if (L > k) u += L - k;
    pos += 1 + div_ceil(L, 16);
  }
  if (pos > bin_words) return mhb_set_error(MHB_ERR_ARG, ".bin image truncated");
  ix->rec_off[n_reads] = pos;
  ix->unit_off[n_reads] = u;
  ix->n_units = u;
  return MHB_OK;
}

void read_stream_stats_reset() { g_st = StreamStats(); }
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
  ReadLibIndex ix;
  if (index_read_lib(bin, bin_words, n_reads, 0, &ix)) return -1;
  std::vector<uint64_t> first;
  plan_read_chunks(ix, n_reads, max_chunk_bytes, &first);
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
// ChunkStager
// ------------------------------------------------------------------------------------------------
ChunkStager::~ChunkStager() {
  if (copy_) cudaStreamSynchronize((cudaStream_t)copy_);
  for (void *e : ev_) cudaEventDestroy((cudaEvent_t)e);
  for (char *h : host_)
    if (h) cudaFreeHost(h);
  if (copy_) cudaStreamDestroy((cudaStream_t)copy_);
}

int ChunkStager::init(size_t slot_bytes, uint64_t n_chunks, StreamStats *stats) {
  slot_bytes_ = slot_bytes;
  n_chunks_ = n_chunks;
  st_ = stats;
  if (!n_chunks) return MHB_OK;
  for (int s = 0; s < 2 && slot_bytes_; ++s) CK(cudaHostAlloc((void **)&host_[s], slot_bytes_, cudaHostAllocDefault));
  cudaStream_t cs;
  CK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  copy_ = cs;
  ev_.assign(4 * n_chunks, nullptr);
  for (auto &e : ev_) CK(cudaEventCreate((cudaEvent_t *)&e));
  return MHB_OK;
}

// fill the staging buffer of chunk i (host threads) and queue its upload on the copy stream
int ChunkStager::stage(uint64_t i, const Fill &fill) {
  const int s = (int)(i & 1);
  cudaStream_t cs = (cudaStream_t)copy_;
  if (i >= 2) CK(cudaEventSynchronize((cudaEvent_t)ev_[4 * (i - 2) + 1]));  // upload of chunk i-2 has left staging s
  const auto t0 = std::chrono::steady_clock::now();
  Copies up;
  CKR(fill(i, host_[s], &up));
  st_->fill_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  char *d = dev_ + s * slot_bytes_;
  if (i >= 2) CK(cudaStreamWaitEvent(cs, (cudaEvent_t)ev_[4 * (i - 2) + 3], 0));  // kernels of chunk i-2 are done with slot s
  CK(cudaEventRecord((cudaEvent_t)ev_[4 * i], cs));
  for (int j = 0; j < up.n; ++j) {
    CK(cudaMemcpyAsync(d + up.off[j], host_[s] + up.off[j], up.bytes[j], cudaMemcpyHostToDevice, cs));
    st_->h2d_bytes += up.bytes[j];
  }
  CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 1], cs));
  return MHB_OK;
}

int ChunkStager::pass(void *stream, const Fill &fill, const Run &run) {
  const uint64_t nc = n_chunks_;
  if (!nc) return MHB_OK;
  if (!dev_) return mhb_set_error(MHB_ERR_ARG, "internal: chunk stager without device memory");
  cudaStream_t st = (cudaStream_t)stream;
  ++st_->passes;
  const auto t0 = std::chrono::steady_clock::now();
  CKR(stage(0, fill));
  for (uint64_t i = 0; i < nc; ++i) {
    // the next upload is queued before the kernels of this chunk, so a host read inside run does not stall the copy
    if (i + 1 < nc) CKR(stage(i + 1, fill));
    CK(cudaStreamWaitEvent(st, (cudaEvent_t)ev_[4 * i + 1], 0));
    CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 2], st));
    CKR(run(i, dev_ + (i & 1) * slot_bytes_));
    CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 3], st));
  }
  CK(cudaEventSynchronize((cudaEvent_t)ev_[4 * (nc - 1) + 3]));
  CK(cudaStreamSynchronize((cudaStream_t)copy_));
  st_->pass_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  for (uint64_t i = 0; i < nc; ++i) {
    float a = 0, b = 0;
    CK(cudaEventElapsedTime(&a, (cudaEvent_t)ev_[4 * i], (cudaEvent_t)ev_[4 * i + 1]));
    CK(cudaEventElapsedTime(&b, (cudaEvent_t)ev_[4 * i + 2], (cudaEvent_t)ev_[4 * i + 3]));
    st_->copy_ms += a;
    st_->kernel_ms += b;
  }
  return MHB_OK;
}

int ChunkStager::upload(void *stream, const char *host, const std::vector<size_t> &off, const Run &run) {
  cudaStream_t st = (cudaStream_t)stream, cs = (cudaStream_t)copy_;
  CK(cudaEventRecord((cudaEvent_t)ev_[0], st));
  CK(cudaStreamWaitEvent(cs, (cudaEvent_t)ev_[0], 0));
  for (uint64_t i = 0; i < n_chunks_; ++i) {
    CK(cudaMemcpyAsync(dev_ + off[i], host + off[i], off[i + 1] - off[i], cudaMemcpyHostToDevice, cs));
    CK(cudaEventRecord((cudaEvent_t)ev_[4 * i + 1], cs));
    CK(cudaStreamWaitEvent(st, (cudaEvent_t)ev_[4 * i + 1], 0));
    CKR(run(i, dev_ + off[i]));
  }
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// ChunkStream
// ------------------------------------------------------------------------------------------------
int ChunkStream::init(const Input &in, std::vector<uint64_t> first, StreamStats *stats, uint32_t pieces) {
  in_ = in;
  resident_ = first.empty();
  first_ = resident_ ? std::vector<uint64_t>{0, in.n} : std::move(first);
  uint64_t max_words = in.words;
  max_units_ = in.n;
  if (!resident_) {
    max_words = max_units_ = 0;
    for (uint64_t i = 0; i < n_chunks(); ++i) {
      max_units_ = std::max(max_units_, first_[i + 1] - first_[i]);
      max_words = std::max(max_words, in.word_of(first_[i + 1]) - in.word_of(first_[i]));
    }
  }
  slot_bytes_ = image_bytes(max_words);
  for (int j = 0; j < 4; ++j) {
    side_at_[j] = slot_bytes_;
    if (in.side[j].host) slot_bytes_ += side_bytes(max_units_, in.side[j].elem);
  }
  stats->chunks = n_chunks();
  pieces_.clear();
  if (resident_ && pieces > 1) {
    const uint64_t per = ((in.n + pieces - 1) / pieces + 3) & ~(uint64_t)3;
    for (uint64_t u = 0; u < in.n; u += per) pieces_.push_back(u);
    pieces_.push_back(in.n);
    return stager_.init(0, pieces_.size() - 1, stats);
  }
  return stager_.init(slot_bytes_, n_chunks(), stats);
}

int ChunkStream::bind(void *device, void *stream) {
  dev_ = (char *)device;
  stager_.bind(dev_);
  if (!resident_ || !pieces_.empty()) return MHB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (in_.words) CK(cudaMemcpyAsync(dev_, in_.image, in_.words * 4, cudaMemcpyHostToDevice, st));
  for (int j = 0; j < 4 && in_.n; ++j) {
    const Side &s = in_.side[j];
    const size_t bytes = s.elem ? in_.n * s.elem : (in_.n + 1) * 8;
    if (s.host) CK(cudaMemcpyAsync(dev_ + side_at_[j], s.host, bytes, cudaMemcpyHostToDevice, st));
  }
  return MHB_OK;
}

ChunkView ChunkStream::view(uint64_t i, const char *slot) const {
  ChunkView v;
  v.index = i;
  v.first = first_[i];
  v.n = first_[i + 1] - first_[i];
  v.words = (const uint32_t *)slot;
  v.n_words = resident_ ? in_.words : in_.word_of(first_[i + 1]) - in_.word_of(first_[i]);
  for (int j = 0; j < 4; ++j) v.side[j] = in_.side[j].host ? slot + side_at_[j] : nullptr;
  return v;
}

// chunk i into a staging buffer: its image, then its slice of every side array, offsets rebased to the chunk
int ChunkStream::fill(uint64_t i, char *h, ChunkStager::Copies *up) const {
  const uint64_t b = first_[i], n = first_[i + 1] - b, w0 = in_.word_of(b);
  const uint64_t bytes = (in_.word_of(b + n) - w0) * 4, blk = 4ull << 20, nblk = (bytes + blk - 1) / blk;
#pragma omp parallel for schedule(static)
  for (long long j = 0; j < (long long)nblk; ++j) {
    const uint64_t o = (uint64_t)j * blk;
    memcpy(h + o, (const char *)(in_.image + w0) + o, std::min(blk, bytes - o));
  }
  up->add(0, bytes);
  for (int j = 0; j < 4; ++j) {
    const Side &s = in_.side[j];
    if (!s.host) continue;
    char *d = h + side_at_[j];
    if (s.elem) {
      memcpy(d, (const char *)s.host + b * s.elem, n * s.elem);
      up->add(side_at_[j], n * s.elem);
      continue;
    }
    const uint64_t *src = (const uint64_t *)s.host + b;
    uint64_t *dst = (uint64_t *)d;
#pragma omp parallel for schedule(static)
    for (long long u = 0; u <= (long long)n; ++u) dst[u] = src[u] - src[0];
    up->add(side_at_[j], (n + 1) * 8);
  }
  return MHB_OK;
}

int ChunkStream::pass(void *stream, const std::function<int(const ChunkView &)> &fn) {
  if (!dev_) return mhb_set_error(MHB_ERR_ARG, "internal: chunk stream without device memory");
  if (resident_ && !pieces_.empty()) {
    std::vector<uint64_t> p;
    p.swap(pieces_);
    std::vector<size_t> off;
    for (uint64_t u : p) off.push_back(in_.word_of(u) * 4);
    return stager_.upload(stream, (const char *)in_.image, off, [&](uint64_t i, const char *piece) {
      ChunkView v = view(0, piece);
      v.index = i;
      v.first = p[i];
      v.n = p[i + 1] - p[i];
      v.n_words = in_.word_of(p[i + 1]) - in_.word_of(p[i]);
      return fn(v);
    });
  }
  if (resident_) return fn(view(0, dev_));
  return stager_.pass(
      stream, [this](uint64_t i, char *h, ChunkStager::Copies *up) { return fill(i, h, up); },
      [&](uint64_t i, const char *slot) { return fn(view(i, slot)); });
}

int init_read_stream(ChunkStream *rs, const uint32_t *bin, uint64_t bin_words, uint64_t n_reads, const ReadLibIndex &ix,
                     uint64_t max_chunk_bytes, uint32_t pieces) {
  ChunkStream::Input in;
  in.image = bin;
  in.words = bin_words;
  in.n = n_reads;
  in.word_off = ix.fixed_len ? nullptr : ix.rec_off.data();
  in.stride = 1 + div_ceil(ix.fixed_len, 16);
  if (!ix.fixed_len) in.side[0].host = ix.rec_off.data();
  if (!ix.fixed_len && !ix.unit_off.empty()) in.side[1].host = ix.unit_off.data();
  std::vector<uint64_t> first;
  if (max_chunk_bytes) plan_read_chunks(ix, n_reads, max_chunk_bytes, &first);
  return rs->init(in, std::move(first), &g_st, ix.fixed_len ? pieces : 1);
}
