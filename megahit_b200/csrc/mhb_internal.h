// mhb_internal.h -- declarations shared by the translation units of libmhb (not part of the C ABI).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

int mhb_set_error(int code, const char *fmt, ...);

// mhb_sort_records + optional per-pass timings (host array of n_bytes doubles, ms; forces a stream sync)
int mhb_sort_records_impl(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                          uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                          double *pass_ms_host);
// relaxed: as mhb_sort_records_relaxed (1) or mhb_sort_records (0), + per-pass timings as above
int mhb_sort_records_ex(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                        uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                        double *pass_ms_host, int relaxed);
// mhb_sort_records_relaxed without an entry in the per-pass timing ring (a sort inside another sort)
int mhb_sort_records_untraced(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                              uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b);

// bytes held by the arena the host-level calls keep between calls (mhb_release frees it)
size_t mhb_arena_bytes(void);

// The SdBG output of a build that runs its stage-2 sort in rounds over ascending bucket ranges: every round's emitter
// output (mhb_s2s_emit / mhb_s2s_emit_fmt) is appended to one byte stream, its non-empty rows of the bucket table are
// taken over with their byte offsets moved by the bytes before them, and the totals are summed.
struct SdbgStitch {
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> table = std::vector<uint64_t>((size_t)65536 * 4);  // {byte offset, items, tips, large_mul}
  uint64_t tot[16] = {0};  // the emitter's totals layout: [0] bytes [1] items [2] tips [3] large_mul [4..12] w [13] ones
  int append(void *stream, const uint8_t *d_bytes, uint64_t cap_bytes, const uint64_t *d_table, const uint64_t *d_totals);

 private:
  std::vector<uint64_t> round_table = std::vector<uint64_t>((size_t)65536 * 4);
};
