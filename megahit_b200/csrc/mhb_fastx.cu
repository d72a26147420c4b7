// mhb_fastx.cu -- `buildlib` on the device: FASTA/FASTQ text -> the `.bin` read library (SURVEY.md 8f N3).
// Kernels per chunk of one stream: '\n' index -> speculative segment walk + fix-up -> record descriptors -> TrimN ->
// scan -> 2-bit pack; for `pe` a zip kernel interleaves the two streams.  Host level: chunked streams with carried
// tails, the reference's batch rules (an error ends a batch; at a batch start it ends the library), mhb_buildlib_host
// and mhb_buildlib_run.  Building blocks: mhb_fastx.cuh.
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <fstream>
#include <string>
#include <vector>

#include "mhb_common.cuh"
#include "mhb_fastx.cuh"

using namespace mhb::fx;
typedef uint32_t u32;
typedef uint64_t u64;

int scan32(cudaStream_t st, const uint32_t *in, uint64_t n, uint64_t *out, uint64_t *total_dev, uint64_t *bsum);

namespace {

constexpr u32 kTile = 4096;      // bytes per block of the '\n' index
constexpr u32 kSegLines = 256;   // nominal lines per walk segment
constexpr u64 kBatchReads = 1ull << 22, kBatchBases = 1ull << 28;  // async_sequence_reader.h:46-47
u64 g_chunk_cap = 0;             // mhb_set_buildlib_chunk; 0 = kDefaultChunk
constexpr u64 kDefaultChunk = 256ull << 20;

// ---------------------------------------------------------------------------------------------- line index
__global__ void k_nl_count(const uint8_t *t, u64 n, u32 *cnt) {
  const u64 base = (u64)blockIdx.x * kTile;
  u32 c = 0;
  for (u32 i = threadIdx.x; i < kTile; i += blockDim.x) {
    const u64 p = base + i;
    c += p < n && t[p] == '\n';
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  __shared__ u32 s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 tot = 0;
    for (u32 w = 0; w < blockDim.x / 32; ++w) tot += s[w];
    cnt[blockIdx.x] = tot;
  }
}

// positions of the '\n' bytes of tile b, in order, at nl[off[b] ...)
__global__ void k_nl_write(const uint8_t *t, u64 n, const u64 *off, u64 *nl) {
  const u64 base = (u64)blockIdx.x * kTile;
  __shared__ u32 wsum[32];
  __shared__ u64 run;
  if (threadIdx.x == 0) run = off[blockIdx.x];
  const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (u32 r = 0; r < kTile; r += blockDim.x) {
    const u64 p = base + r + threadIdx.x;
    const bool hit = p < n && t[p] == '\n';
    const u32 m = __ballot_sync(0xffffffffu, hit);
    __syncthreads();
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    u32 before = 0;
    for (u32 w = 0; w < warp; ++w) before += wsum[w];
    if (hit) nl[run + before + __popc(m & ((1u << lane) - 1))] = p;
    __syncthreads();
    if (threadIdx.x == 0) {
      u32 tot = 0;
      for (u32 w = 0; w < nw; ++w) tot += wsum[w];
      run += tot;
    }
  }
}

// ---------------------------------------------------------------------------------------------- segment walk
__global__ void k_fx_seg_start(FxLines L, u32 n_seg, u32 *seg) {
  const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n_seg) return;
  if (s == 0 || s == n_seg) {
    seg[s] = s == 0 ? 0 : L.n_lines;
    return;
  }
  const u32 lo = s * kSegLines, hi = min(lo + kSegLines, L.n_lines);
  u32 p = lo;
  while (p < hi && !fx_sync_line(L, p)) ++p;
  seg[s] = p < hi ? p : lo;
}

struct CountEmit {
  u32 n = 0;
  __device__ void operator()(const FxRec &) { ++n; }
};
struct ArrayEmit {
  FxRec *out;
  u64 i;
  __host__ __device__ void operator()(const FxRec &r) { out[i++] = r; }
};

// emit = 0: count the records of every segment (only_dirty: the segments the check pass flagged) and store its exit state;
// emit = 1: write them at rec[off[s] ...)
__global__ void k_fx_walk(FxLines L, u32 n_seg, const u32 *seg, const FxState *entry, FxState *exit_st, u32 *count,
                          const u32 *dirty, int emit, const u64 *off, FxRec *rec) {
  const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg || (dirty && !dirty[s])) return;
  FxState st = entry[s];
  const u32 a = seg[s], b = seg[s + 1];
  auto run = [&](auto &em) {
    for (u32 j = a; j < b && st.mode != END; ++j) fx_step(L, j, st, em);
    if (s + 1 < n_seg) fx_normalise(L, b, st, em);
    else if (L.final_chunk) fx_finish(L, st, em);
  };
  if (emit) {
    ArrayEmit em{rec, off[s]};
    run(em);
  } else {
    CountEmit em;
    run(em);
    count[s] = em.n;
    exit_st[s] = st;
  }
}

__global__ void k_fx_check(u32 n_seg, FxState *entry, const FxState *exit_st, u32 *dirty, u32 *n_dirty) {
  const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  u32 d = 0;
  if (s > 0 && !fx_same(entry[s], exit_st[s - 1])) {
    entry[s] = exit_st[s - 1];
    d = 1;
    atomicAdd(n_dirty, 1u);
  }
  dirty[s] = d;
}

// ---------------------------------------------------------------------------------------------- trim + pack
// one warp per record: first N-free run (bpos, len in sequence coordinates; len = kErrLen for error records) and the
// words it takes in `.bin` (1 + ceil(max(len, 1) / 16); 0 for errors)
__global__ void k_fx_trim(FxLines L, const FxRec *rec, u64 n, u32 *bpos, u32 *len, u32 *words) {
  const u32 lane = threadIdx.x & 31;
  for (u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((u64)gridDim.x * blockDim.x) >> 5) {
    const FxRec R = rec[r];
    if (!R.ok) {
      if (lane == 0) bpos[r] = 0, len[r] = kErrLen, words[r] = 0;
      continue;
    }
    u32 acc = 0, first = kErrLen, e = kErrLen;
    for (u32 j = R.hdr + 1; j < R.seq_end && e == kErrLen; ++j) {
      const u64 s = L.start(j);
      if (L.end(j) == s) continue;
      const u32 m = fx_seq_add(L, j, acc);
      for (u32 o = 0; o < m && e == kErrLen; o += 32) {
        const bool valid = o + lane < m;
        const bool isn = valid && fx_is_n(L.text[s + o + lane]);
        const u32 nonn = __ballot_sync(0xffffffffu, valid && !isn), nm = __ballot_sync(0xffffffffu, isn);
        u32 from = 0;
        if (first == kErrLen) {
          if (!nonn) continue;
          const u32 f = __ffs(nonn) - 1;
          first = acc + o + f;
          from = f + 1;
        }
        const u32 after = from >= 32 ? 0 : nm & (0xffffffffu << from);
        if (after) e = acc + o + __ffs(after) - 1;
      }
      acc += m;
    }
    if (first == kErrLen) first = acc;
    if (e == kErrLen) e = acc;
    if (lane == 0) {
      const u32 l = e - first;
      bpos[r] = first;
      len[r] = l;
      words[r] = 1 + ((l ? l : 1) + 15) / 16;
    }
  }
}

constexpr u32 kStage = 1024;  // staged bases per warp
__global__ void k_fx_pack(FxLines L, const FxRec *rec, u64 n, const u32 *bpos, const u32 *len, const u64 *woff, u32 *out) {
  __shared__ uint8_t stage_all[8][kStage];
  const u32 lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  uint8_t *stage = stage_all[wib];
  for (u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((u64)gridDim.x * blockDim.x) >> 5) {
    const u32 l = len[r];
    if (l == kErrLen) continue;
    u32 *o = out + woff[r];
    if (l == 0) {  // sequence_package.h: an empty read is stored as "A"
      if (lane == 0) o[0] = 1, o[1] = 0;
      continue;
    }
    if (lane == 0) o[0] = l;
    const FxRec R = rec[r];
    const u32 b = bpos[r];
    u32 base = 0;  // q of stage[0]
    auto flush = [&](u32 upto) {  // words [base/16, (base+upto+15)/16)
      __syncwarp();
      const u32 nwds = (upto + 15) / 16;
      for (u32 w = lane; w < nwds; w += 32) {
        u32 v = 0;
        for (u32 t = 0; t < 16; ++t) {
          const u32 q = w * 16 + t;
          if (q < upto) v |= (u32)stage[q] << (30 - 2 * t);
        }
        o[1 + base / 16 + w] = v;
      }
      __syncwarp();
    };
    u32 acc = 0;
    for (u32 j = R.hdr + 1; j < R.seq_end && acc < b + l; ++j) {
      const u64 s = L.start(j);
      if (L.end(j) == s) continue;
      const u32 m = fx_seq_add(L, j, acc);
      for (u32 off = 0; off < m; off += 32) {
        const u32 pos = acc + off + lane;
        const bool in = off + lane < m && pos >= b && pos < b + l;
        const u32 q = pos - b;
        const uint8_t c = in ? (uint8_t)fx_code(L.text[s + off + lane]) : 0;
        if (in && q < base + kStage) stage[q - base] = c;
        // this strip's last byte lies beyond the staged window (and the read goes on): everything before it is staged
        if (acc + min(off + 32, m) > b + base + kStage && base + kStage < l) {
          flush(kStage);
          base += kStage;
          if (in && q >= base) stage[q - base] = c;
        }
      }
      acc += m;
    }
    flush(l - base);
  }
}

// pe: pair j (j < n_pairs) = read j of stream A then read j of stream B, kept when both are reads and j < stop
__global__ void k_fx_zip_words(const u32 *la, const u32 *lb, const u32 *wa, const u32 *wb, u64 n_pairs, u64 stop, u32 *w) {
  for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n_pairs; j += (u64)gridDim.x * blockDim.x)
    w[j] = (j < stop && la[j] != kErrLen && lb[j] != kErrLen) ? wa[j] + wb[j] : 0;
}
__global__ void k_fx_zip(const u32 *pa, const u32 *pb, const u64 *oa, const u64 *ob, const u32 *wa, const u32 *w,
                         const u64 *off, u64 n_pairs, u32 *out) {
  const u32 lane = threadIdx.x & 31;
  for (u64 j = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_pairs; j += ((u64)gridDim.x * blockDim.x) >> 5) {
    const u32 tw = w[j];
    if (!tw) continue;
    const u32 na = wa[j];
    for (u32 i = lane; i < tw; i += 32) out[off[j] + i] = i < na ? pa[oa[j] + i] : pb[ob[j] + i - na];
  }
}

// scan32 with its per-4096-input block sums in `bsum`, grown to fit n first (every scan of a chunk has its own n: tiles,
// segments, records, pairs)
int scan_n(cudaStream_t st, const u32 *in, u64 n, u64 *out, u64 *total_dev, DevBuf &bsum) {
  CKR(bsum.ensure((n / 4096 + 4) * 8, "buildlib"));
  return scan32(st, in, n, out, total_dev, bsum.as<u64>());
}

// One chunk of one stream parsed on the device.  The packed reads stay on the device (pack, at woff[r]); the host gets
// per record its trimmed length (kErrLen = error) and where the stream resumes after it.
struct FxChunk {
  DevBuf text, tcnt, toff, bsum, tot, nl, seg, entry, exit_st, count, dirty, ndirty, roff, rec, bpos, len, words, woff, pack;
  std::vector<FxRec> h_rec;
  std::vector<u32> h_len;
  u64 n_rec = 0, n_words = 0, n_lines = 0;
  FxState exit_last{SEEK, 0, 0, 0, 0};
  u64 walk_passes = 0;

  // text[0, n): complete lines (plus an unterminated last line when final); the carried state is SEEK or HDR
  int parse(cudaStream_t st, const uint8_t *h_text, u64 n, int final_chunk, u32 carry_mode) {
    CKR(text.ensure(n + 16, "buildlib"));
    if (n) CK(cudaMemcpyAsync(text.p, h_text, n, cudaMemcpyHostToDevice, st));
    const u64 tiles = std::max<u64>(1, (n + kTile - 1) / kTile);
    CKR(tcnt.ensure(tiles * 4, "buildlib"));
    CKR(toff.ensure(tiles * 8, "buildlib"));
    CKR(tot.ensure(64, "buildlib"));
    CK(cudaMemsetAsync(tcnt.p, 0, tiles * 4, st));
    if (n) {
      k_nl_count<<<(unsigned)tiles, 256, 0, st>>>(text.as<uint8_t>(), n, tcnt.as<u32>());
      CK_LAUNCH();
    }
    CKR(scan_n(st, tcnt.as<u32>(), tiles, toff.as<u64>(), tot.as<u64>(), bsum));
    u64 n_nl = 0;
    CK(cudaMemcpyAsync(&n_nl, tot.p, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CKR(nl.ensure((n_nl + 1) * 8, "buildlib"));
    if (n) {
      k_nl_write<<<(unsigned)tiles, 256, 0, st>>>(text.as<uint8_t>(), n, toff.as<u64>(), nl.as<u64>());
      CK_LAUNCH();
    }
    const bool unterminated_last = final_chunk && n > 0 && h_text[n - 1] != '\n';
    n_lines = n_nl + (unterminated_last ? 1 : 0);
    if (n_lines >= 0xFFFFFFF0ull) return mhb_set_error(MHB_ERR_ARG, "buildlib: a chunk of more than 2^32 lines");
    FxLines L{text.as<uint8_t>(), nl.as<u64>(), (u32)n_lines, n, final_chunk};
    const u32 n_seg = (u32)std::max<u64>(1, (n_lines + kSegLines - 1) / kSegLines);
    CKR(seg.ensure((n_seg + 1) * 4, "buildlib"));
    CKR(entry.ensure(n_seg * sizeof(FxState), "buildlib"));
    CKR(exit_st.ensure(n_seg * sizeof(FxState), "buildlib"));
    CKR(count.ensure(n_seg * 4, "buildlib"));
    CKR(dirty.ensure(n_seg * 4, "buildlib"));
    CKR(ndirty.ensure(8, "buildlib"));
    CKR(roff.ensure(n_seg * 8, "buildlib"));
    const unsigned gs = (n_seg + 1 + 255) / 256, gw = (n_seg + 127) / 128;
    k_fx_seg_start<<<gs, 256, 0, st>>>(L, n_seg, seg.as<u32>());
    CK_LAUNCH();
    // every segment but the first guesses "a header line starts here"
    std::vector<FxState> h_entry(n_seg, FxState{HDR, 0, 0, 0, 0});
    h_entry[0] = FxState{carry_mode, 0, 0, 0, 0};
    CK(cudaMemcpyAsync(entry.p, h_entry.data(), n_seg * sizeof(FxState), cudaMemcpyHostToDevice, st));
    k_fx_walk<<<gw, 128, 0, st>>>(L, n_seg, seg.as<u32>(), entry.as<FxState>(), exit_st.as<FxState>(), count.as<u32>(),
                                  nullptr, 0, nullptr, nullptr);
    CK_LAUNCH();
    walk_passes = 1;
    for (;;) {  // fix-up: re-walk every segment whose guess differs from its predecessor's exit until all edges agree
      u32 nd = 0;
      CK(cudaMemsetAsync(ndirty.p, 0, 4, st));
      k_fx_check<<<gs, 256, 0, st>>>(n_seg, entry.as<FxState>(), exit_st.as<FxState>(), dirty.as<u32>(), ndirty.as<u32>());
      CK_LAUNCH();
      CK(cudaMemcpyAsync(&nd, ndirty.p, 4, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (!nd) break;
      k_fx_walk<<<gw, 128, 0, st>>>(L, n_seg, seg.as<u32>(), entry.as<FxState>(), exit_st.as<FxState>(), count.as<u32>(),
                                    dirty.as<u32>(), 0, nullptr, nullptr);
      CK_LAUNCH();
      ++walk_passes;
    }
    CKR(scan_n(st, count.as<u32>(), n_seg, roff.as<u64>(), tot.as<u64>(), bsum));
    CK(cudaMemcpyAsync(&n_rec, tot.p, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&exit_last, exit_st.as<FxState>() + (n_seg - 1), sizeof(FxState), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CKR(rec.ensure((n_rec + 1) * sizeof(FxRec), "buildlib"));
    CKR(bpos.ensure((n_rec + 1) * 4, "buildlib"));
    CKR(len.ensure((n_rec + 1) * 4, "buildlib"));
    CKR(words.ensure((n_rec + 1) * 4, "buildlib"));
    CKR(woff.ensure((n_rec + 1) * 8, "buildlib"));
    n_words = 0;
    if (n_rec) {
      k_fx_walk<<<gw, 128, 0, st>>>(L, n_seg, seg.as<u32>(), entry.as<FxState>(), exit_st.as<FxState>(), count.as<u32>(),
                                    nullptr, 1, roff.as<u64>(), rec.as<FxRec>());
      CK_LAUNCH();
      k_fx_trim<<<grid_cap(n_rec * 32, 256, 32), 256, 0, st>>>(L, rec.as<FxRec>(), n_rec, bpos.as<u32>(), len.as<u32>(),
                                                             words.as<u32>());
      CK_LAUNCH();
      CKR(scan_n(st, words.as<u32>(), n_rec, woff.as<u64>(), tot.as<u64>(), bsum));
      CK(cudaMemcpyAsync(&n_words, tot.p, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      CKR(pack.ensure(n_words * 4 + 16, "buildlib"));
      k_fx_pack<<<grid_cap(n_rec * 32, 256, 32), 256, 0, st>>>(L, rec.as<FxRec>(), n_rec, bpos.as<u32>(), len.as<u32>(),
                                                             woff.as<u64>(), pack.as<u32>());
      CK_LAUNCH();
    }
    h_rec.resize(n_rec);
    h_len.resize(n_rec);
    if (n_rec) {
      CK(cudaMemcpyAsync(h_rec.data(), rec.p, n_rec * sizeof(FxRec), cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(h_len.data(), len.p, n_rec * 4, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    return MHB_OK;
  }
  // byte offset of line j (j <= number of complete lines): one entry of the device '\n' index
  int line_start(cudaStream_t st, u64 j, u64 *out) const {
    u64 v = 0;
    if (j > 0) {
      CK(cudaMemcpyAsync(&v, nl.as<u64>() + (j - 1), 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      ++v;
    }
    *out = v;
    return MHB_OK;
  }
};

// One input stream: an in-memory buffer or a file descriptor read sequentially (FIFOs welcome: no seeks, no sizes).
struct FxInput {
  const uint8_t *mem = nullptr;
  u64 mem_n = 0, mem_pos = 0;
  int fd = -1;
  bool eof = false;
  std::vector<uint8_t> buf;
  u64 head = 0;  // buf[head, size) is pending text
  u32 mode = SEEK;
  bool ended = false;  // no more records
  int fill(u64 want) {  // pending text >= want bytes, or eof
    if (head > 0 && head * 2 > buf.size()) {
      buf.erase(buf.begin(), buf.begin() + head);
      head = 0;
    }
    while (!eof && buf.size() - head < want) {
      const u64 need = want - (buf.size() - head);
      if (mem) {
        const u64 take = std::min(need, mem_n - mem_pos);
        buf.insert(buf.end(), mem + mem_pos, mem + mem_pos + take);
        mem_pos += take;
        if (mem_pos == mem_n) eof = true;
      } else {  // a pipe returns at most its buffer per read(): grow once, then fill
        const u64 old = buf.size();
        buf.resize(old + need);
        u64 got = 0;
        while (got < need) {
          const ssize_t r = read(fd, buf.data() + old + got, need - got);
          if (r < 0) {
            if (errno == EINTR) continue;
            buf.resize(old + got);
            return mhb_set_error(MHB_ERR_IO, "buildlib: read failed: %s", strerror(errno));
          }
          if (r == 0) {
            eof = true;
            break;
          }
          got += (u64)r;
        }
        buf.resize(old + got);
      }
    }
    return MHB_OK;
  }
  u64 pending() const { return buf.size() - head; }
};

// Where a library's packed reads go, chunk by chunk: appended to `bin` (mhb_buildlib_host), or written to `file` as soon as
// they are back on the host (mhb_buildlib_run: host memory stays at one chunk's output, as the reference writes P.bin
// batch by batch).
struct LibOut {
  std::vector<u32> bin;
  FILE *file = nullptr;
  const char *file_name = "";
  std::vector<u32> stage;  // file mode: one chunk's words
  u64 reads = 0, bases = 0;
  u32 max_len = 0;
  u64 chunks = 0, walk_passes = 0;

  int put(cudaStream_t st, const void *dev, u64 words) {
    if (!words) return MHB_OK;
    u32 *dst;
    if (file) {
      if (stage.size() < words) stage.resize(words);
      dst = stage.data();
    } else {
      bin.resize(bin.size() + words);
      dst = bin.data() + bin.size() - words;
    }
    CK(cudaMemcpyAsync(dst, dev, words * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (file && fwrite(dst, 4, words, file) != words) return mhb_set_error(MHB_ERR_IO, "write to %s failed", file_name);
    return MHB_OK;
  }
};

struct BatchState {  // FastxReader::Read / PairedFastxReader::Read batch bookkeeping
  u64 i = 0, bases = 0;
  bool stopped = false;
};

// the resume point (byte offset into the parsed text, carried mode) after record r of a chunk
int resume_after(cudaStream_t st, const FxChunk &c, u64 r, u64 *bytes, u32 *mode) {
  const FxRec &R = c.h_rec[r];
  *mode = R.resume_mode == END ? SEEK : R.resume_mode;
  return c.line_start(st, R.resume_line, bytes);
}

// parses the next chunk of `in`; *got = false when nothing could be consumed and the chunk has to grow
int parse_next(cudaStream_t st, FxInput &in, FxChunk &c, u64 chunk, u64 *text_n, bool *final_chunk) {
  CKR(in.fill(chunk));
  const uint8_t *t = in.buf.data() + in.head;
  u64 n = std::min<u64>(in.pending(), chunk);
  bool fin = in.eof && n == in.pending();
  if (!fin) {  // complete lines only
    u64 k = n;
    while (k > 0 && t[k - 1] != '\n') --k;
    n = k;
  }
  *text_n = n;
  *final_chunk = fin;
  return c.parse(st, t, n, fin ? 1 : 0, in.mode);
}

int do_se(cudaStream_t st, FxInput &in, u64 chunk0, LibOut &out) {
  FxChunk c;
  BatchState bs;
  u64 chunk = chunk0;
  while (!bs.stopped) {
    u64 n;
    bool fin;
    CKR(parse_next(st, in, c, chunk, &n, &fin));
    ++out.chunks;
    out.walk_passes += c.walk_passes;
    if (!fin && c.n_rec == 0 && (c.exit_last.mode != SEEK || n == 0)) {  // a record (or line) larger than the chunk
      chunk *= 2;
      continue;
    }
    chunk = chunk0;
    u64 stop = c.n_rec;
    for (u64 r = 0; r < c.n_rec; ++r) {
      const u32 l = c.h_len[r];
      if (l == kErrLen) {
        if (bs.i == 0) {
          stop = r;
          bs.stopped = true;
          break;
        }
        bs.i = bs.bases = 0;
        continue;
      }
      ++out.reads;
      out.bases += std::max(l, 1u);
      out.max_len = std::max(out.max_len, std::max(l, 1u));
      bs.bases += l;
      const u64 i = bs.i++;
      if ((bs.bases >= kBatchBases && i % 2 == 1) || bs.i == kBatchReads) bs.i = bs.bases = 0;
    }
    u64 words = c.n_words;
    if (stop < c.n_rec) {
      std::vector<u64> wo(1);
      CK(cudaMemcpyAsync(wo.data(), c.woff.as<u64>() + stop, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      words = wo[0];
    }
    CKR(out.put(st, c.pack.p, words));
    if (fin) break;
    u64 used;
    u32 mode;
    if (c.exit_last.mode == SEEK) used = n, mode = SEEK;
    else CKR(resume_after(st, c, c.n_rec - 1, &used, &mode));
    in.head += used;
    in.mode = mode;
  }
  return MHB_OK;
}

int do_pe(cudaStream_t st, FxInput &ia, FxInput &ib, u64 chunk0, LibOut &out) {
  FxChunk ca, cb;
  BatchState bs;
  DevBuf w, off, tot, bsum, zip;
  u64 chunk_a = chunk0, chunk_b = chunk0;
  for (;;) {
    u64 na, nb;
    bool fa, fb;
    CKR(parse_next(st, ia, ca, chunk_a, &na, &fa));
    CKR(parse_next(st, ib, cb, chunk_b, &nb, &fb));
    out.chunks += 2;
    out.walk_passes += ca.walk_passes + cb.walk_passes;
    const u64 m = std::min(ca.n_rec, cb.n_rec);
    const bool a_ends = fa && ca.n_rec == m, b_ends = fb && cb.n_rec == m;
    if (m == 0 && !a_ends && !b_ends) {  // one stream has no complete record in its chunk
      if (ca.n_rec == 0) {
        if (ca.exit_last.mode == SEEK && na) ia.head += na; else chunk_a *= 2;
      }
      if (cb.n_rec == 0) {
        if (cb.exit_last.mode == SEEK && nb) ib.head += nb; else chunk_b *= 2;
      }
      continue;
    }
    chunk_a = chunk_b = chunk0;
    u64 stop = m;
    for (u64 j = 0; j < m; ++j) {
      const u32 la = ca.h_len[j], lb = cb.h_len[j];
      if (la == kErrLen || lb == kErrLen) {
        if (bs.i == 0) {
          stop = j;
          bs.stopped = true;
          break;
        }
        bs.i = bs.bases = 0;
        continue;
      }
      out.reads += 2;
      out.bases += std::max(la, 1u) + std::max(lb, 1u);
      out.max_len = std::max(out.max_len, std::max(std::max(la, 1u), std::max(lb, 1u)));
      bs.bases += (u64)la + lb;
      bs.i += 2;
      if (bs.bases >= kBatchBases || bs.i >= kBatchReads) bs.i = bs.bases = 0;
    }
    if (m) {
      CKR(w.ensure(m * 4, "buildlib"));
      CKR(off.ensure(m * 8, "buildlib"));
      CKR(tot.ensure(64, "buildlib"));
      k_fx_zip_words<<<grid_cap(m, 256, 32), 256, 0, st>>>(ca.len.as<u32>(), cb.len.as<u32>(), ca.words.as<u32>(),
                                                       cb.words.as<u32>(), m, stop, w.as<u32>());
      CK_LAUNCH();
      CKR(scan_n(st, w.as<u32>(), m, off.as<u64>(), tot.as<u64>(), bsum));
      u64 words = 0;
      CK(cudaMemcpyAsync(&words, tot.p, 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      CKR(zip.ensure(words * 4 + 16, "buildlib"));
      k_fx_zip<<<grid_cap(m * 32, 256, 32), 256, 0, st>>>(ca.pack.as<u32>(), cb.pack.as<u32>(), ca.woff.as<u64>(),
                                                      cb.woff.as<u64>(), ca.words.as<u32>(), w.as<u32>(), off.as<u64>(), m,
                                                      zip.as<u32>());
      CK_LAUNCH();
      CKR(out.put(st, zip.p, words));
    }
    if (bs.stopped || a_ends || b_ends) break;
    u64 used;
    u32 mode;
    CKR(resume_after(st, ca, m - 1, &used, &mode));
    ia.head += used, ia.mode = mode;
    CKR(resume_after(st, cb, m - 1, &used, &mode));
    ib.head += used, ib.mode = mode;
  }
  return MHB_OK;
}

int run_lib(cudaStream_t st, const char *type, FxInput *in, LibOut &out) {
  const u64 chunk = g_chunk_cap ? g_chunk_cap : kDefaultChunk;
  if (!strcmp(type, "pe")) return do_pe(st, in[0], in[1], chunk, out);
  return do_se(st, in[0], chunk, out);
}

int valid_type(const char *t) { return !strcmp(t, "pe") || !strcmp(t, "se") || !strcmp(t, "interleaved"); }

}  // namespace

extern "C" int mhb_set_buildlib_chunk(uint64_t bytes) {
  g_chunk_cap = bytes;
  return MHB_OK;
}

extern "C" int mhb_buildlib_host(const mhb_buildlib_args *a, mhb_buildlib_result *res) {
  if (!a || !res || (a->n_libs && !a->libs)) return mhb_set_error(MHB_ERR_ARG, "null argument");
  memset(res, 0, sizeof(*res));
  if (mhb_device_count() <= 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  const auto t0 = std::chrono::steady_clock::now();
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  std::vector<u32> bin;
  std::vector<u64> begin(a->n_libs), end(a->n_libs);
  std::vector<u32> maxl(a->n_libs);
  int rc = MHB_OK;
  for (u32 i = 0; i < a->n_libs && !rc; ++i) {
    const mhb_buildlib_lib &lib = a->libs[i];
    if (!lib.type || !valid_type(lib.type)) {
      rc = mhb_set_error(MHB_ERR_ARG, "Valid types: pe, se, interleaved");
      break;
    }
    FxInput in[2];
    const int ns = !strcmp(lib.type, "pe") ? 2 : 1;
    for (int s = 0; s < ns; ++s) {
      in[s].mem = lib.data[s] ? lib.data[s] : (const uint8_t *)"";
      in[s].mem_n = lib.size[s];
      in[s].eof = lib.size[s] == 0;
    }
    LibOut o;
    if ((rc = run_lib(st, lib.type, in, o))) break;
    if (strcmp(lib.type, "se") && o.reads % 2) {
      rc = mhb_set_error(MHB_ERR_ARG, "PE library number of reads is odd: %llu!", (unsigned long long)o.reads);
      break;
    }
    begin[i] = res->n_reads;
    res->n_reads += o.reads;
    end[i] = res->n_reads;
    res->n_bases += o.bases;
    maxl[i] = o.max_len;
    res->n_chunks += o.chunks;
    res->n_walk_passes += o.walk_passes;
    bin.insert(bin.end(), o.bin.begin(), o.bin.end());
  }
  cudaStreamDestroy(st);
  if (rc) return rc;
  res->n_libs = a->n_libs;
  res->bin_words = bin.size();
  res->bin = (u32 *)malloc(std::max<size_t>(bin.size(), 1) * 4);
  res->lib_begin = (u64 *)malloc(std::max<size_t>(a->n_libs, 1) * 8);
  res->lib_end = (u64 *)malloc(std::max<size_t>(a->n_libs, 1) * 8);
  res->lib_max_len = (u32 *)malloc(std::max<size_t>(a->n_libs, 1) * 4);
  if (!res->bin || !res->lib_begin || !res->lib_end || !res->lib_max_len) return mhb_set_error(MHB_ERR_NOMEM, "host malloc failed");
  memcpy(res->bin, bin.data(), bin.size() * 4);
  for (u32 i = 0; i < a->n_libs; ++i) res->lib_begin[i] = begin[i], res->lib_end[i] = end[i], res->lib_max_len[i] = maxl[i];
  res->t_total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return MHB_OK;
}

// `megahit_core buildlib lib_file out_prefix` (sequence_lib.cpp:8-91): the lib file is read with the same istream
// operations (getline, >> type, >> files, getline), so its quirks carry over; P.bin is written chunk by chunk.
extern "C" int mhb_buildlib_run(const char *lib_file, const char *out_prefix) {
  if (!lib_file || !out_prefix) return mhb_set_error(MHB_ERR_ARG, "null argument");
  std::ifstream cfg(lib_file);
  if (!cfg.is_open()) return mhb_set_error(MHB_ERR_IO, "File to open read_lib file: %s", lib_file);
  if (mhb_device_count() <= 0) return mhb_set_error(MHB_ERR_CUDA, "no CUDA device: libmhb has no CPU path");
  const std::string prefix = out_prefix;
  FILE *bin = fopen((prefix + ".bin").c_str(), "wb");
  if (!bin) return mhb_set_error(MHB_ERR_IO, "cannot write %s.bin", out_prefix);
  cudaStream_t st;
  if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) {
    fclose(bin);
    return mhb_set_error(MHB_ERR_CUDA, "cudaStreamCreate failed");
  }
  std::string metadata, type, f1, f2, info;
  u64 total_reads = 0, total_bases = 0;
  int rc = MHB_OK, lib_no = 0;
  while (!rc && std::getline(cfg, metadata)) {
    cfg >> type;
    std::vector<std::string> files;
    if (type == "pe") {
      cfg >> f1 >> f2;
      files = {f1, f2};
    } else if (type == "se" || type == "interleaved") {
      cfg >> f1;
      files = {f1};
    } else {
      fprintf(stderr, "ERROR %-30s: %4d - Cannot identify read library type %s\n", "megahit_b200", __LINE__, type.c_str());
      rc = mhb_set_error(MHB_ERR_ARG, "Valid types: pe, se, interleaved");
      break;
    }
    FxInput in[2];
    for (size_t s = 0; s < files.size() && !rc; ++s) {
      in[s].fd = open(files[s].c_str(), O_RDONLY);
      if (in[s].fd < 0) rc = mhb_set_error(MHB_ERR_IO, "Cannot open file %s", files[s].c_str());
    }
    const std::string bin_name = prefix + ".bin";
    LibOut o;
    o.file = bin;
    o.file_name = bin_name.c_str();
    if (!rc) rc = run_lib(st, type.c_str(), in, o);
    for (auto &x : in)
      if (x.fd >= 0) close(x.fd);
    if (rc) break;
    if (type != "se" && o.reads % 2) {
      fprintf(stderr, "ERROR %-30s: %4d - PE library number of reads is odd: %llu!\n", "megahit_b200", __LINE__,
              (unsigned long long)o.reads);
      rc = mhb_set_error(MHB_ERR_ARG, "File(s): %s", metadata.c_str());
      break;
    }
    fprintf(stderr, "INFO  %-30s: %4d - Lib %d (%s): %s, %llu reads, %u max length\n", "megahit_b200", __LINE__, lib_no++,
            metadata.c_str(), type.c_str(), (unsigned long long)o.reads, o.max_len);
    char line[128];
    snprintf(line, sizeof(line), "%llu %llu %u %d\n", (unsigned long long)total_reads,
             (unsigned long long)(total_reads + o.reads), o.max_len, type != "se" ? 1 : 0);
    info += metadata + "\n" + line;
    total_reads += o.reads;
    total_bases += o.bases;
    std::getline(cfg, metadata);  // the rest of the line
  }
  cudaStreamDestroy(st);
  if (fclose(bin) != 0 && !rc) rc = mhb_set_error(MHB_ERR_IO, "write to %s.bin failed", out_prefix);
  if (rc) return rc;
  FILE *li = fopen((prefix + ".lib_info").c_str(), "w");
  if (!li) return mhb_set_error(MHB_ERR_IO, "cannot write %s.lib_info", out_prefix);
  fprintf(li, "%llu %llu\n%s", (unsigned long long)total_bases, (unsigned long long)total_reads, info.c_str());
  if (fclose(li) != 0) return mhb_set_error(MHB_ERR_IO, "write to %s.lib_info failed", out_prefix);
  return MHB_OK;
}

extern "C" void mhb_buildlib_free(mhb_buildlib_result *res) {
  if (!res) return;
  free(res->bin);
  free(res->lib_begin);
  free(res->lib_end);
  free(res->lib_max_len);
  memset(res, 0, sizeof(*res));
}

// Self-test hook: the line walk, TrimN and packing of mhb_fastx.cuh driven serially over one whole stream (no batches).
// Per record: trimmed length (kErrLen = error) and first kept position; bin_out = the packed reads of the ok records.
extern "C" int mhb_selftest_fastx(const uint8_t *text, uint64_t n, uint32_t *len_out, uint32_t *bpos_out, uint64_t cap,
                                  uint64_t *n_rec_out, uint32_t *bin_out, uint64_t bin_cap, uint64_t *bin_words_out) {
  std::vector<u64> nl;
  for (u64 i = 0; i < n; ++i)
    if (text[i] == '\n') nl.push_back(i);
  const u64 n_lines = nl.size() + (n > 0 && text[n - 1] != '\n' ? 1 : 0);
  nl.push_back(0);
  FxLines L{text, nl.data(), (u32)n_lines, n, 1};
  std::vector<FxRec> recs(n_lines + 2);  // at most one record ends per line, plus the end of the stream
  ArrayEmit em{recs.data(), 0};
  FxState st{SEEK, 0, 0, 0, 0};
  for (u32 j = 0; j < n_lines && st.mode != END; ++j) fx_step(L, j, st, em);
  fx_finish(L, st, em);
  recs.resize(em.i);
  *n_rec_out = recs.size();
  u64 w = 0;
  for (u64 r = 0; r < recs.size(); ++r) {
    u32 b = 0, l = kErrLen;
    if (recs[r].ok) fx_trim_serial(L, recs[r].hdr + 1, recs[r].seq_end, &b, &l);
    if (r < cap) len_out[r] = l, bpos_out[r] = b;
    if (l == kErrLen) continue;
    const u32 ol = l ? l : 1, nw = (ol + 15) / 16;
    if (w + 1 + nw > bin_cap) return mhb_set_error(MHB_ERR_ARG, "selftest: bin_cap too small");
    bin_out[w] = ol;
    std::vector<u32> words(nw, 0);
    u32 acc = 0;
    for (u32 j = recs[r].hdr + 1; j < recs[r].seq_end; ++j) {
      const u64 s = L.start(j);
      if (L.end(j) == s) continue;
      const u32 m = fx_seq_add(L, j, acc);
      for (u32 i = 0; i < m; ++i) {
        const u32 q = acc + i - b;
        if (acc + i >= b && q < l) words[q / 16] |= fx_code(text[s + i]) << (30 - 2 * (q % 16));
      }
      acc += m;
    }
    for (u32 i = 0; i < nw; ++i) bin_out[w + 1 + i] = words[i];
    w += 1 + nw;
  }
  *bin_words_out = w;
  return MHB_OK;
}
