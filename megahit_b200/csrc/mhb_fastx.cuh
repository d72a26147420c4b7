// mhb_fastx.cuh -- building blocks of `buildlib` on the device (FASTA/FASTQ text -> `.bin` records).
//
// The text of one stream is cut into lines (byte-parallel '\n' index); the kseq record grammar (kseq.h:193-246) is then
// walked at line level by one thread per segment of lines.  A walk state at a line boundary is small (FxState), so
// segments start from a guessed state and a check pass re-walks every segment whose guess differs from its
// predecessor's exit state, until all edges agree (the first segment starts from the true state): the result never
// depends on the guesses, only the number of passes does.  Everything here is __host__ __device__ so that the CPU
// self-test hook runs the same code.
#pragma once
#include <stdint.h>

namespace mhb {
namespace fx {

enum : uint32_t {
  SEEK = 0,  // looking for the next '>' / '@' anywhere (file start, after a FASTQ record)
  HDR = 1,   // the next line is a header whose marker is its first byte (it ended the previous FASTA record)
  SEQ = 2,   // sequence lines of record `hdr`
  QUAL = 3,  // quality lines of record `hdr` (the '+' line was `plus`)
  END = 4,   // end of the stream (a bare marker as the unterminated last line)
};
constexpr uint32_t kErrLen = 0xFFFFFFFFu;

struct FxState {
  uint32_t mode, hdr, plus, seq, qual;
};
__host__ __device__ inline bool fx_same(const FxState &a, const FxState &b) {
  return a.mode == b.mode && a.hdr == b.hdr && a.plus == b.plus && a.seq == b.seq && a.qual == b.qual;
}

// one record as the walk emits it: header line, sequence lines [hdr+1, seq_end), ok/error, where the stream resumes
struct FxRec {
  uint32_t hdr, seq_end, ok, resume_line, resume_mode, pad;
};

// line j of a chunk: [start, end) without its '\n'; only the last line of the final chunk may be unterminated
struct FxLines {
  const uint8_t *text;
  const uint64_t *nl;  // positions of the '\n' bytes
  uint32_t n_lines;
  uint64_t n_bytes;
  int final_chunk;     // the last line may lack its '\n' (n_lines then counts it)
  __host__ __device__ uint64_t start(uint32_t j) const { return j == 0 ? 0 : nl[j - 1] + 1; }
  __host__ __device__ uint64_t end(uint32_t j) const { return term(j) ? nl[j] : n_bytes; }
  __host__ __device__ bool term(uint32_t j) const { return !(final_chunk && j + 1 == n_lines && (n_bytes == 0 || text[n_bytes - 1] != '\n')); }
};

__host__ __device__ inline bool is_marker(uint8_t c) { return c == '>' || c == '@'; }

// the seq / qual length a line adds (kseq drops a trailing '\r' from the accumulated string when it is longer than one
// byte; a one-byte sequence line without '\n' is appended by ks_getc alone and never stripped)
__host__ __device__ inline uint32_t fx_seq_add(const FxLines &L, uint32_t j, uint32_t acc) {
  const uint64_t s = L.start(j), e = L.end(j);
  const uint32_t len = (uint32_t)(e - s);
  const bool strip = len > 0 && L.text[e - 1] == '\r' && acc + len > 1 && (L.term(j) || len >= 2);
  return len - (strip ? 1 : 0);
}
__host__ __device__ inline uint32_t fx_qual_add(const FxLines &L, uint32_t j, uint32_t acc) {
  const uint64_t s = L.start(j), e = L.end(j);
  const uint32_t len = (uint32_t)(e - s);
  const bool strip = len > 0 && L.text[e - 1] == '\r' && acc + len > 1;
  return len - (strip ? 1 : 0);
}

// The header line j (marker at byte p): a bare marker as the unterminated last line is the end of the stream.
__host__ __device__ inline void fx_header(const FxLines &L, uint32_t j, uint64_t p, FxState &st) {
  if (p + 1 == L.end(j) && !L.term(j)) {
    st = FxState{END, 0, 0, 0, 0};
    return;
  }
  st = FxState{SEQ, j, 0, 0, 0};
}

// Walks line j from state st; calls emit(rec) for a record that ends here.
template <class Emit>
__host__ __device__ inline void fx_step(const FxLines &L, uint32_t j, FxState &st, Emit &&emit) {
  const uint64_t s = L.start(j), e = L.end(j);
  switch (st.mode) {
    case SEEK: {
      uint64_t p = s;
      while (p < e && !is_marker(L.text[p])) ++p;
      if (p < e) fx_header(L, j, p, st);
      return;
    }
    case HDR:
      fx_header(L, j, s, st);
      return;
    case SEQ: {
      if (e == s) return;  // empty line
      const uint8_t c = L.text[s];
      if (is_marker(c)) {
        emit(FxRec{st.hdr, j, 1, j, HDR, 0});
        fx_header(L, j, s, st);
        return;
      }
      if (c == '+') {
        if (!L.term(j)) {  // the '+' line ends the stream
          emit(FxRec{st.hdr, j, 0, j + 1, END, 0});
          st = FxState{END, 0, 0, 0, 0};
          return;
        }
        st.mode = QUAL;
        st.plus = j;
        st.qual = 0;
        return;
      }
      st.seq += fx_seq_add(L, j, st.seq);
      return;
    }
    case QUAL:
      st.qual += fx_qual_add(L, j, st.qual);
      if (st.qual >= st.seq) {
        emit(FxRec{st.hdr, st.plus, st.qual == st.seq ? 1u : 0u, j + 1, SEEK, 0});
        st = FxState{SEEK, 0, 0, 0, 0};
      }
      return;
    default:
      return;
  }
}

// the end of the stream after the last line (final chunk only)
template <class Emit>
__host__ __device__ inline void fx_finish(const FxLines &L, FxState &st, Emit &&emit) {
  if (st.mode == SEQ) emit(FxRec{st.hdr, L.n_lines, 1, L.n_lines, END, 0});
  // the quality block ran out of lines: well formed only for an empty sequence whose '+' line is the last line
  if (st.mode == QUAL) emit(FxRec{st.hdr, st.plus, st.qual == st.seq ? 1u : 0u, L.n_lines, END, 0});
  st = FxState{END, 0, 0, 0, 0};
}

// After the lines of a segment: a SEQ / SEEK state followed by a line that starts with a marker is the same as HDR at
// that line (a SEQ record ends there) - the canonical form the next segment's guess is compared with.
template <class Emit>
__host__ __device__ inline void fx_normalise(const FxLines &L, uint32_t next, FxState &st, Emit &&emit) {
  if (next >= L.n_lines || (st.mode != SEQ && st.mode != SEEK)) return;
  const uint64_t s = L.start(next);
  if (L.end(next) == s || !is_marker(L.text[s])) return;
  if (st.mode == SEQ) emit(FxRec{st.hdr, next, 1, next, HDR, 0});
  st = FxState{HDR, 0, 0, 0, 0};
}

// a line where a segment may start: a '>' line, or the 4-line FASTQ shape @ / seq / + / qual of equal length
__host__ __device__ inline bool fx_sync_line(const FxLines &L, uint32_t j) {
  const uint64_t s = L.start(j);
  if (L.end(j) == s) return false;
  const uint8_t c = L.text[s];
  if (c == '>') return true;
  if (c != '@' || j + 3 >= L.n_lines) return false;
  const uint64_t s1 = L.start(j + 1), s2 = L.start(j + 2);
  if (L.end(j + 1) == s1 || L.end(j + 2) == s2 || L.text[s2] != '+') return false;
  const uint8_t c1 = L.text[s1];
  if (c1 == '>' || c1 == '+' || c1 == '@') return false;
  return L.end(j + 1) - s1 == L.end(j + 3) - L.start(j + 3);
}

__host__ __device__ inline uint32_t fx_code(uint8_t c) {
  switch (c) {
    case 'C': case 'c': return 1;
    case 'G': case 'g': return 2;
    case 'T': case 't': return 3;
    default: return 0;  // A/a, N and every other byte (IUPAC codes, a kept '\r', spaces)
  }
}
__host__ __device__ inline bool fx_is_n(uint8_t c) { return c == 'N' || c == 'n'; }

// TrimN over the sequence lines [a, b) of a record (the host mirror of the warp loop in k_fx_trim): first non-N
// position and the length of the N-free run from there, in sequence coordinates
__host__ __device__ inline void fx_trim_serial(const FxLines &L, uint32_t a, uint32_t b, uint32_t *bpos, uint32_t *len) {
  uint32_t acc = 0, first = kErrLen, e = 0;
  bool done = false;
  for (uint32_t j = a; j < b && !done; ++j) {
    const uint64_t s = L.start(j);
    if (L.end(j) == s) continue;
    const uint32_t n = fx_seq_add(L, j, acc);
    for (uint32_t i = 0; i < n; ++i) {
      const bool isn = fx_is_n(L.text[s + i]);
      if (first == kErrLen) {
        if (!isn) first = acc + i;
      } else if (isn) {
        e = acc + i;
        done = true;
        break;
      }
    }
    acc += n;
  }
  if (first == kErrLen) first = acc;
  if (!done) e = acc;
  *bpos = first;
  *len = e - first;
}

}  // namespace fx
}  // namespace mhb
