// mhb_sortdisp.cu -- the radix-sort part of the device-level C ABI (include/mhb.h, layer 1): variant selection,
// per-width dispatch of the radix pass kernels (mhb_sort.cuh v2 = partition pass, mhb_sort3.cuh v3 = sort passes),
// the fused partition + exchange pass, CUDA-IPC buffer helpers and the per-pass timing trace.  Its own translation
// unit because the kernel instantiations (17 record widths x variants) dominate the build time of the library.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "mhb.h"
#include "mhb_common.cuh"
#include "mhb_kernels.cuh"
#include "mhb_sort.cuh"
#include "mhb_sort3.cuh"
#include "mhb_part.cuh"

using namespace mhb;

// ------------------------------------------------------------------------------------------------
// sort
// ------------------------------------------------------------------------------------------------
// Radix-pass variants.  0..3 = v2 geometries (mhb_sort.cuh); 256 + bits = v3 (mhb_sort3.cuh, see SortCfg3 for the
// bit field).  Only the listed v3 combinations are instantiated (all for 8- and 12-byte records, the first one for
// every record width).
#define MHB_V3_DEFAULT 0x180
#define MHB_V3_LIST(X) X(0x180) X(0x080) X(0x000) X(0x1080) X(0x082)
static bool v3_listed(int bits) {
#define X(B) \
  if (bits == B) return true;
  MHB_V3_LIST(X)
#undef X
  return false;
}
static int g_sort_cfg = -1;
extern "C" int mhb_set_sort_cfg(int cfg) {
  if (!((cfg >= 0 && cfg <= 3) || (cfg >= 256 && v3_listed(cfg - 256))))
    return mhb_set_error(MHB_ERR_ARG, "unknown sort configuration %d", cfg);
  g_sort_cfg = cfg;
  return MHB_OK;
}
static int sort_cfg() {
  int &cfg = g_sort_cfg;
  if (cfg < 0) {
    const char *e = getenv("MHB_SORT_CFG");
    cfg = e ? atoi(e) : 256 + MHB_V3_DEFAULT;
    if (!((cfg >= 0 && cfg <= 3) || (cfg >= 256 && v3_listed(cfg - 256)))) cfg = 256 + MHB_V3_DEFAULT;
  }
  return cfg;
}
template <int WR, int CFG>
static u64 sort_tiles_cfg(u64 n) {
  return (n + SortCfg<WR, CFG>::TILE - 1) / SortCfg<WR, CFG>::TILE;
}
template <int WR, int CFG>
static u64 sort_tiles_cfg3(u64 n) {
  return (n + SortCfg3<WR, CFG>::TILE - 1) / SortCfg3<WR, CFG>::TILE;
}
template <int WR>
static u64 sort_tiles(u64 n) {
  const int cfg = sort_cfg();
  if (cfg >= 256) {
    if constexpr (WR == 2 || WR == 3) {
#define X(B) \
  if (cfg - 256 == B) return sort_tiles_cfg3<WR, B>(n);
      MHB_V3_LIST(X)
#undef X
    }
    return sort_tiles_cfg3<WR, MHB_V3_DEFAULT>(n);
  }
  if constexpr (WR <= 3) {
    switch (cfg) {
      case 1: return sort_tiles_cfg<WR, 1>(n);
      case 2: return sort_tiles_cfg<WR, 2>(n);
      case 3: return sort_tiles_cfg<WR, 3>(n);
      default: break;
    }
  }
  return sort_tiles_cfg<WR, 0>(n);
}
static u64 sort_num_tiles(u64 n, u32 words) {
#define M(WW) \
  if (words == WW) return sort_tiles<WW>(n);
  MHB_FOR_WR(M)
#undef M
  return 0;
}
static constexpr size_t kSortHeadBytes = (size_t)(72 + 1) * 256 * 8 /*hist*/ + 256 * 8 /*bin_base*/ + 128 * 4 + 256 * 8 /*gcursor*/;
// look-back storage for `tiles` tiles: 256 64-bit descriptors per tile + (compact-descriptor variants) one 16-byte
// word per digit and group of four tiles behind them
static size_t lb_bytes(u64 tiles) { return (size_t)tiles * 256 * 8 + (size_t)((tiles + 3) / 4) * 256 * 16; }

extern "C" size_t mhb_sort_workspace_bytes(uint64_t n, uint32_t words) {
  // sized for the smallest tile of any configuration so that a workspace stays valid across MHB_SORT_CFG values
  u64 tiles = sort_num_tiles(n, words);
  if (words <= 3) tiles = (n + 256 * 8 - 1) / (256 * 8) > tiles ? (n + 256 * 8 - 1) / (256 * 8) : tiles;
#define M(WW) \
  if (words == WW && sort_tiles_cfg<WW, 0>(n) > tiles) tiles = sort_tiles_cfg<WW, 0>(n);  // partition pass geometry
  MHB_FOR_WR(M)
#undef M
  return kSortHeadBytes + lb_bytes(tiles) + 256;
}

template <int WR, int CFG>
static int launch_radix_pass_cfg(cudaStream_t st, const u32 *in, u64 n, int byte_idx, const u64 *bin_base,
                                 u64 *lookback, u32 *tile_counter, u64 *next_hist, int next_byte, u32 epoch) {
  using C = SortCfg<WR, CFG>;
  static int blocks_per_sm = 0;
  if (!blocks_per_sm) {
    CK(cudaFuncSetAttribute(k_radix_pass<WR, CFG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k_radix_pass<WR, CFG>, C::THREADS, C::SMEM));
    if (blocks_per_sm < 1) return mhb_set_error(MHB_ERR_CUDA, "radix pass kernel (WR=%d) does not fit an SM", WR);
    if (getenv("MHB_VERBOSE")) fprintf(stderr, "[mhb] radix pass WR=%d cfg=%d: %d threads x %d rec, %zu B smem, %d CTA/SM\n", WR, CFG, C::THREADS, C::IPT, C::SMEM, blocks_per_sm);
  }
  const u64 tiles = sort_tiles_cfg<WR, CFG>(n);
  u64 grid = (u64)blocks_per_sm * sm_count();
  if (grid > tiles) grid = tiles;
  k_radix_pass<WR, CFG><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, lookback,
                                                                 tile_counter, next_hist, next_byte, epoch);
  CK_LAUNCH();
  return MHB_OK;
}

template <int WR, int CFG>
static int launch_radix_pass_cfg3(cudaStream_t st, const u32 *in, u64 n, int byte_idx, const u64 *bin_base,
                                  u64 *lookback, u32 *tile_counter, u64 *next_hist, int next_byte, u32 epoch) {
  using C = SortCfg3<WR, CFG>;
  static int blocks_per_sm = 0;
  if (!blocks_per_sm) {
    CK(cudaFuncSetAttribute(k_radix_pass3<WR, CFG, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaFuncSetAttribute(k_radix_pass3<WR, CFG, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k_radix_pass3<WR, CFG, false, true>, C::THREADS, C::SMEM));
    if (blocks_per_sm < 1) return mhb_set_error(MHB_ERR_CUDA, "radix pass v3 kernel (WR=%d) does not fit an SM", WR);
    if (getenv("MHB_VERBOSE")) fprintf(stderr, "[mhb] radix pass v3 WR=%d bits=0x%03x: %d threads x %d rec, rank %d, prefetch %d, look-back %d/%d, batch %d, early %d, %zu B smem, %d CTA/SM\n", WR, CFG, C::THREADS, C::IPT, C::RANK, (int)C::PREFETCH, C::LB1, C::LBW, (int)C::BATCH, (int)C::EARLY, C::SMEM, blocks_per_sm);
  }
  const u64 tiles = sort_tiles_cfg3<WR, CFG>(n);
  u64 grid = (u64)blocks_per_sm * sm_count();
  if (grid > tiles) grid = tiles;
  if (next_hist)
    k_radix_pass3<WR, CFG, false, true><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, lookback,
                                                                                 tile_counter, next_hist, next_byte, epoch);
  else
    k_radix_pass3<WR, CFG, false, false><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, lookback,
                                                                                  tile_counter, nullptr, 0, epoch);
  CK_LAUNCH();
  return MHB_OK;
}

// first pass of a sort whose caller does not need a deterministic order among fully equal keys (mhb_part.cuh)
template <int WR>
static int launch_part_unstable(cudaStream_t st, const u32 *in, u64 n, int byte_idx, const u64 *bin_base,
                                unsigned long long *gcursor, u32 *tile_counter, u64 *next_hist, int next_byte,
                                const uint8_t *lut) {
  using C = PartCfg<WR>;
  static int bps = 0;
  if (!bps) {
    CK(cudaFuncSetAttribute(k_part_unstable<WR, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaFuncSetAttribute(k_part_unstable<WR, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaFuncSetAttribute(k_part_unstable<WR, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaFuncSetAttribute(k_part_unstable<WR, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_OWNER_HIST));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_part_unstable<WR, false, true>, C::THREADS, C::SMEM));
    if (bps < 1) return mhb_set_error(MHB_ERR_CUDA, "partition pass (WR=%d) does not fit an SM", WR);
    if (getenv("MHB_VERBOSE")) fprintf(stderr, "[mhb] unstable partition pass WR=%d: %d threads x %d rec, %zu B smem, %d CTA/SM\n", WR, C::THREADS, C::IPT, C::SMEM, bps);
  }
  const u64 tiles = (n + C::TILE - 1) / C::TILE;
  u64 grid = (u64)bps * sm_count();
  if (grid > tiles) grid = tiles;
  if (lut && next_hist)
    k_part_unstable<WR, true, true><<<(int)grid, C::THREADS, C::SMEM_OWNER_HIST, st>>>(in, n, (u32)tiles, byte_idx, bin_base, gcursor,
                                                                                       tile_counter, next_hist, next_byte, lut);
  else if (lut)
    k_part_unstable<WR, true, false><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, gcursor,
                                                                             tile_counter, nullptr, 0, lut);
  else if (next_hist)
    k_part_unstable<WR, false, true><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, gcursor,
                                                                             tile_counter, next_hist, next_byte, nullptr);
  else
    k_part_unstable<WR, false, false><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_base, gcursor,
                                                                              tile_counter, nullptr, 0, nullptr);
  CK_LAUNCH();
  return MHB_OK;
}

template <int WR>
static int launch_radix_pass(cudaStream_t st, const u32 *in, u64 n, int byte_idx, const u64 *bin_base,
                             u64 *lookback, u32 *tile_counter, u64 *next_hist, int next_byte, u32 epoch) {
  const int cfg = sort_cfg();
  if (cfg >= 256) {
    if constexpr (WR == 2 || WR == 3) {
#define X(B) \
  if (cfg - 256 == B) return launch_radix_pass_cfg3<WR, B>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
      MHB_V3_LIST(X)
#undef X
    }
    return launch_radix_pass_cfg3<WR, MHB_V3_DEFAULT>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
  }
  if constexpr (WR <= 3) {
    switch (cfg) {
      case 1: return launch_radix_pass_cfg<WR, 1>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
      case 2: return launch_radix_pass_cfg<WR, 2>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
      case 3: return launch_radix_pass_cfg<WR, 3>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
      default: break;
    }
  }
  return launch_radix_pass_cfg<WR, 0>(st, in, n, byte_idx, bin_base, lookback, tile_counter, next_hist, next_byte, epoch);
}

#ifdef MHB_SORT_TIMELINE
// diagnostic build only: point the v3 radix pass at a device buffer of rows x 16 uint64 (see mhb_sort3.cuh)
extern "C" int mhb_debug_set_sort_timeline(unsigned long long *dev_buf, unsigned long long rows) {
  CK(cudaMemcpyToSymbol(g_sort_timeline, &dev_buf, sizeof(dev_buf)));
  CK(cudaMemcpyToSymbol(g_sort_timeline_rows, &rows, sizeof(rows)));
  return MHB_OK;
}
#endif

// Per-pass timing: every sort records one event before and after each pass into a small ring, so a
// caller can ask afterwards (mhb_sort_pass_ms) how long each pass of a recent sort took without putting a
// synchronisation inside its timed region.
namespace {
struct SortTrace {
  cudaEvent_t ev[74];
  bool created = false;
  uint32_t n_passes = 0, words = 0;
  uint64_t n = 0;
};
SortTrace g_trace[4];
uint64_t g_trace_seq = 0;
}  // namespace

// relaxed != 0: the first pass may be the unstable partition pass (mhb_part.cuh) - the order among records whose sorted
// bytes are ALL equal is then unspecified; MHB_SORT_STABLE_FIRST=1 keeps the stable pass everywhere (A/B hook).
// trace: the sort takes a slot of the per-pass timing ring (mhb_sort_pass_ms); the sorts a larger sort runs inside
// itself (mhb_s2s_sort's oversized buckets) do not, so that the ring keeps one entry per sort a caller issued.
static int sort_records_core(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                             uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                             double *pass_ms_host, int relaxed, bool trace);
int mhb_sort_records_impl(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                          uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                          double *pass_ms_host) {
  // the library's own stages tally or minimise over records with equal sort keys: their order is irrelevant
  return sort_records_core(stream, a, b, n, words, bytes, n_bytes, first_hist, ws, ws_bytes, result_in_b, pass_ms_host, 1, true);
}
int mhb_sort_records_ex(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                        uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                        double *pass_ms_host, int relaxed) {
  return sort_records_core(stream, a, b, n, words, bytes, n_bytes, first_hist, ws, ws_bytes, result_in_b, pass_ms_host, relaxed, true);
}
int mhb_sort_records_untraced(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                              uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b) {
  return sort_records_core(stream, a, b, n, words, bytes, n_bytes, first_hist, ws, ws_bytes, result_in_b, nullptr, 1, false);
}
static int sort_records_core(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words, const uint8_t *bytes,
                             uint32_t n_bytes, const uint64_t *first_hist, void *ws, size_t ws_bytes, int *result_in_b,
                             double *pass_ms_host, int relaxed, bool trace) {
  if (pass_ms_host && !trace) return mhb_set_error(MHB_ERR_ARG, "per-pass times need a traced sort");
  static const bool stable_first = getenv("MHB_SORT_STABLE_FIRST") != nullptr;
  if (stable_first) relaxed = 0;
  if (words < 1 || words > 17 || n_bytes > 72 || !result_in_b)
    return mhb_set_error(MHB_ERR_ARG, "bad sort geometry (words=%u n_bytes=%u)", words, n_bytes);
  *result_in_b = 0;
  if (n == 0 || n_bytes == 0) return MHB_OK;
  if (ws_bytes < mhb_sort_workspace_bytes(n, words)) return mhb_set_error(MHB_ERR_ARG, "sort workspace too small");
  if (n >= (1ull << 53)) return mhb_set_error(MHB_ERR_ARG, "too many records");
  cudaStream_t st = (cudaStream_t)stream;
  u64 *hist = (u64 *)ws;                        // [n_bytes+1][256]
  u64 *bin_base = hist + (72 + 1) * 256;        // [256]
  u32 *tile_counter = (u32 *)(bin_base + 256);  // [128]
  unsigned long long *gcursor = (unsigned long long *)(tile_counter + 128);  // [256]: unstable first pass
  u64 *lookback = (u64 *)((char *)ws + kSortHeadBytes);
  // only what this sort's tile geometry touches (the workspace itself is sized for the smallest tile of any variant)
  CK(cudaMemsetAsync(ws, 0, kSortHeadBytes + lb_bytes(sort_num_tiles(n, words)) + 256, st));
  if (first_hist) {
    CK(cudaMemcpyAsync(hist, first_hist, 256 * 8, cudaMemcpyDeviceToDevice, st));
  } else {
#define M(WW) \
  if (words == WW) k_hist_byte<WW><<<sm_count() * 4, 256, 0, st>>>(a, n, bytes[0], hist);
    MHB_FOR_WR(M)
#undef M
    CK_LAUNCH();
  }
  SortTrace *tr = nullptr;
  if (trace) {
    tr = &g_trace[g_trace_seq++ & 3];
    if (!tr->created) {
      for (int i = 0; i < 74; ++i) CK(cudaEventCreate(&tr->ev[i]));
      tr->created = true;
    }
    tr->n_passes = n_bytes;
    tr->words = words;
    tr->n = n;
    CK(cudaEventRecord(tr->ev[0], st));
  }
  u32 *in = a, *out = b;
  for (u32 p = 0; p < n_bytes; ++p) {
    k_hist_scan256<<<1, 256, 0, st>>>(hist + (u64)p * 256, bin_base, (u64)(uintptr_t)out, words * 4);
    CK_LAUNCH();
    u64 *next_hist = p + 1 < n_bytes ? hist + (u64)(p + 1) * 256 : nullptr;
    const int next_byte = p + 1 < n_bytes ? bytes[p + 1] : 0;
    int rc = MHB_ERR_ARG;
    if (p == 0 && relaxed && words == 2) rc = launch_part_unstable<2>(st, in, n, bytes[p], bin_base, gcursor, tile_counter + p, next_hist, next_byte, nullptr);
    else if (p == 0 && relaxed && words == 3) rc = launch_part_unstable<3>(st, in, n, bytes[p], bin_base, gcursor, tile_counter + p, next_hist, next_byte, nullptr);
    else {
#define M(WW) \
  if (words == WW) rc = launch_radix_pass<WW>(st, in, n, bytes[p], bin_base, lookback, tile_counter + p, next_hist, next_byte, p + 1);
      MHB_FOR_WR(M)
#undef M
    }
    if (rc) return rc;
    if (tr) CK(cudaEventRecord(tr->ev[p + 1], st));
    u32 *t = in;
    in = out;
    out = t;
  }
  *result_in_b = (in == b) ? 1 : 0;
  if (pass_ms_host) {
    CK(cudaEventSynchronize(tr->ev[n_bytes]));
    for (u32 p = 0; p < n_bytes; ++p) {
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, tr->ev[p], tr->ev[p + 1]));
      pass_ms_host[p] = ms;
    }
  }
  return MHB_OK;
}

// ------------------------------------------------------------------------------------------------
// fused partition + exchange: one radix pass whose per-digit destinations are arbitrary device addresses, e.g.
// slots inside OTHER GPUs' receive buffers opened through CUDA IPC.  The scatter stores travel over NVLink while
// the rest of the tile is still being ranked - no separate all-to-all.
// ------------------------------------------------------------------------------------------------
template <int WR>
static int launch_partition_pass(cudaStream_t st, const u32 *in, u64 n, int byte_idx, const u64 *bin_addr, u64 *lookback,
                                 u32 *tile_counter, const uint8_t *lut) {
  using C = SortCfg<WR, 0>;
  static int blocks_per_sm = 0;
  if (!blocks_per_sm) {
    CK(cudaFuncSetAttribute(k_radix_pass<WR, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k_radix_pass<WR, 0, true>, C::THREADS, C::SMEM));
    if (blocks_per_sm < 1) return mhb_set_error(MHB_ERR_CUDA, "partition pass kernel (WR=%d) does not fit an SM", WR);
  }
  const u64 tiles = sort_tiles_cfg<WR, 0>(n);
  u64 grid = (u64)blocks_per_sm * sm_count();
  if (grid > tiles) grid = tiles;
  k_radix_pass<WR, 0, true><<<(int)grid, C::THREADS, C::SMEM, st>>>(in, n, (u32)tiles, byte_idx, bin_addr, lookback,
                                                                     tile_counter, nullptr, 0, 1, lut);
  CK_LAUNCH();
  return MHB_OK;
}

static int partition_scatter_impl(void *stream, const uint32_t *recs, uint64_t n, uint32_t words, int byte,
                                  const uint8_t *owner_of_byte_dev, const uint64_t *bin_addr_dev, void *ws, size_t ws_bytes,
                                  int next_byte, uint64_t *owner_next_hist, int *hist_done);
extern "C" int mhb_partition_scatter(void *stream, const uint32_t *recs, uint64_t n, uint32_t words, int byte,
                                     const uint8_t *owner_of_byte_dev, const uint64_t *bin_addr_dev, void *ws,
                                     size_t ws_bytes) {
  return partition_scatter_impl(stream, recs, n, words, byte, owner_of_byte_dev, bin_addr_dev, ws, ws_bytes, 0, nullptr, nullptr);
}
extern "C" int mhb_partition_scatter_hist(void *stream, const uint32_t *recs, uint64_t n, uint32_t words, int byte,
                                          const uint8_t *owner_of_byte_dev, const uint64_t *bin_addr_dev, void *ws,
                                          size_t ws_bytes, int next_byte, uint64_t *owner_next_hist, int *hist_done) {
  if (!owner_of_byte_dev || !owner_next_hist || !hist_done || next_byte < 0 || next_byte >= (int)(4 * words))
    return mhb_set_error(MHB_ERR_ARG, "bad owner-histogram arguments");
  return partition_scatter_impl(stream, recs, n, words, byte, owner_of_byte_dev, bin_addr_dev, ws, ws_bytes, next_byte,
                                owner_next_hist, hist_done);
}
static int partition_scatter_impl(void *stream, const uint32_t *recs, uint64_t n, uint32_t words, int byte,
                                  const uint8_t *owner_of_byte_dev, const uint64_t *bin_addr_dev, void *ws, size_t ws_bytes,
                                  int next_byte, uint64_t *owner_next_hist, int *hist_done) {
  if (hist_done) *hist_done = 0;
  if (words < 1 || words > 17 || byte < 0 || byte >= (int)(4 * words)) return mhb_set_error(MHB_ERR_ARG, "bad geometry");
  if (n == 0) return MHB_OK;
  // the partition pass always runs the v2 kernel in geometry 0, whatever variant the sorts use
  u64 tiles = 0;
#define M(WW) \
  if (words == WW) tiles = sort_tiles_cfg<WW, 0>(n);
  MHB_FOR_WR(M)
#undef M
  const size_t need = kSortHeadBytes + (size_t)tiles * 256 * 8 + 256;
  if (ws_bytes < need) return mhb_set_error(MHB_ERR_ARG, "sort workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  u64 *hist = (u64 *)ws;
  u32 *tile_counter = (u32 *)(hist + (72 + 1) * 256 + 256);
  u64 *lookback = (u64 *)((char *)ws + kSortHeadBytes);
  CK(cudaMemsetAsync(ws, 0, need, st));
  int rc = MHB_ERR_ARG;
  static const bool stable_first = getenv("MHB_SORT_STABLE_FIRST") != nullptr;
  if (owner_of_byte_dev && !stable_first && (words == 2 || words == 3)) {
    // the exchange has no earlier order to preserve: unstable pass (no look-back chain), 8- and 12-byte records
    unsigned long long *gcursor = (unsigned long long *)(tile_counter + 128);
    rc = words == 2 ? launch_part_unstable<2>(st, recs, n, byte, bin_addr_dev, gcursor, tile_counter, owner_next_hist, next_byte, owner_of_byte_dev)
                    : launch_part_unstable<3>(st, recs, n, byte, bin_addr_dev, gcursor, tile_counter, owner_next_hist, next_byte, owner_of_byte_dev);
    if (!rc && owner_next_hist && hist_done) *hist_done = 1;
  } else if (owner_of_byte_dev) {
#define M(WW) \
  if (words == WW) rc = launch_partition_pass<WW>(st, recs, n, byte, bin_addr_dev, lookback, tile_counter, owner_of_byte_dev);
    MHB_FOR_WR(M)
#undef M
  } else {
#define M(WW) \
  if (words == WW) rc = launch_radix_pass_cfg<WW, 0>(st, recs, n, byte, bin_addr_dev, lookback, tile_counter, nullptr, 0, 1);
    MHB_FOR_WR(M)
#undef M
  }
  return rc;
}

extern "C" int mhb_dev_malloc(void **ptr, size_t bytes) {
  CK(cudaMalloc(ptr, bytes));
  return MHB_OK;
}
extern "C" int mhb_dev_free(void *ptr) {
  CK(cudaFree(ptr));
  return MHB_OK;
}
extern "C" int mhb_ipc_export(const void *dev_ptr, uint8_t *handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
  memcpy(handle64, &h, 64);
  return MHB_OK;
}
extern "C" int mhb_ipc_open(const uint8_t *handle64, void **peer_ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  CK(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return MHB_OK;
}
extern "C" int mhb_ipc_close(void *peer_ptr) {
  CK(cudaIpcCloseMemHandle(peer_ptr));
  return MHB_OK;
}

extern "C" int mhb_sort_pass_ms(int back, double *pass_ms, uint32_t max_passes, uint32_t *n_passes, uint64_t *n_records,
                                uint32_t *words) {
  if (back < 0 || back > 3 || (uint64_t)back >= g_trace_seq) return mhb_set_error(MHB_ERR_ARG, "no such sort in the trace ring");
  SortTrace &tr = g_trace[(g_trace_seq - 1 - back) & 3];
  CK(cudaEventSynchronize(tr.ev[tr.n_passes]));
  for (u32 p = 0; p < tr.n_passes && p < max_passes; ++p) {
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, tr.ev[p], tr.ev[p + 1]));
    pass_ms[p] = ms;
  }
  if (n_passes) *n_passes = tr.n_passes;
  if (n_records) *n_records = tr.n;
  if (words) *words = tr.words;
  return MHB_OK;
}

extern "C" int mhb_sort_records(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words,
                                const uint8_t *bytes, uint32_t n_bytes, const uint64_t *first_hist, void *ws,
                                size_t ws_bytes, int *result_in_b) {
  return mhb_sort_records_ex(stream, a, b, n, words, bytes, n_bytes, first_hist, ws, ws_bytes, result_in_b, nullptr, 0);
}

extern "C" int mhb_sort_records_relaxed(void *stream, uint32_t *a, uint32_t *b, uint64_t n, uint32_t words,
                                        const uint8_t *bytes, uint32_t n_bytes, const uint64_t *first_hist, void *ws,
                                        size_t ws_bytes, int *result_in_b) {
  return mhb_sort_records_ex(stream, a, b, n, words, bytes, n_bytes, first_hist, ws, ws_bytes, result_in_b, nullptr, 1);
}

