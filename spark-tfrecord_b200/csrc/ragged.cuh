// ragged.cuh -- ragged fields (include/tfrgpu.h, RAGGED): a depth-2 column x stored as the plain features x_values (its
// elements, flattened) and x_row_lengths (an Int64List of its inner lengths).
//
//   decode: ragged_assemble_kernel builds x from the two decoded parts.  x's level-0 offsets are the lengths part's, its
//     level-1 offsets one new array (the values part's level-0 offset of the row plus a running sum of the row's lengths), its
//     deeper offsets, leaf values and validity the values part's, reused as they are.  It checks the two parts agree and
//     raises TF_FALLBACK when they do not; the general path has already reported such a record (ragged_lengths_sum,
//     decode.cuh).
//   encode: ragged_split_kernel turns each depth-2 column into the two parts before the encoder's size pass, for column input
//     and after rows.cuh has built the depth-2 column from UnsafeRows, synchronous and pipelined alike.
// The row-splits partition (TFR_S_RAGGED_ROW_SPLITS) stores x_row_splits (k + 1 entries 0, l0, l0+l1, .. for a row of k inner
// lists) in place of x_row_lengths.  A row's splits entries are one more than its inner lists, so x's level-0 offsets are the
// splits part's minus one per earlier row with entries: a prefix count over rows, in scan.cuh's three steps (tile sums ->
// scan_tile_bases_kernel -> a tile-local scan), which the *_splits_* kernels below do.
#pragma once
#include "common.cuh"
#include "encode.cuh"
#include "scan.cuh"
#include "tile.cuh"

// one ragged field of a decoded batch: the parts' device buffers and x's new level-1 offsets
struct RaggedCol {
  const int32_t* len_off;       // lengths part: level-0 offsets [n + 1]
  const int64_t* len;           // its values
  const uint8_t* len_valid;     // its validity bitmap
  const int32_t* val_off;       // values part: level-0 offsets [n + 1]
  const uint8_t* val_valid;
  int32_t* off1;                // out: x's level-1 offsets, room for cap + 1 entries
  uint32_t cap;
};

// one thread per row of n rows (n_dev: a pipelined batch's row count, on the device, bounded by n).  TF_FALLBACK is ORed into
// *flag when a row's parts disagree or x does not fit: the tile and large-record kernels do not check the parts, and the batch
// goes to the general path.  flag = nullptr on the general path, whose pass 1 has failed every such record.
__global__ void __launch_bounds__(256) ragged_assemble_kernel(RaggedCol C, uint32_t n, const uint32_t* n_dev, uint32_t* flag) {
  if (n_dev) n = min(*n_dev, n);
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (n == 0 && r == 0) C.off1[0] = 0;
  if (r >= n) return;
  const uint32_t lo = (uint32_t)C.len_off[r], hi = (uint32_t)C.len_off[r + 1];
  const int64_t end = C.val_off[r + 1];
  int64_t acc = C.val_off[r];
  bool bad = (((C.len_valid[r >> 3] ^ C.val_valid[r >> 3]) >> (r & 7)) & 1u) != 0 || hi < lo || hi > C.cap;
  for (uint32_t i = lo; i < min(hi, C.cap); ++i) {
    C.off1[i] = (int32_t)acc;
    const int64_t l = C.len[i];
    if (l < 0 || l > end - acc) bad = true;
    else acc += l;
  }
  if (acc != end) bad = true;
  if (r == n - 1 && hi <= C.cap) C.off1[hi] = (int32_t)end;
  if (bad && flag) atomicOr(flag, (uint32_t)TF_FALLBACK);
}

// encode: the caller's columns `in` (a ragged x as its depth-2 column) become the lowered columns `out`: x's values part in x's
// place (level-0 offsets off1[off0[r]]; deeper offsets, values and validity reused) and its lengths part (off1 differences over
// level-0 offsets off0, x's validity).  The other entries of `out` are copied from `in` before the launch.  A row whose offsets
// are not a depth-2 column (off0 decreasing, negative or past the `cap` inner lists x has, off1 decreasing) is atomicMin'd into
// *bad.  Kernel arguments only: the pipelined row encode enqueues it with no upload.
#define RAGGED_PER_LAUNCH 8
struct RaggedPart {
  int32_t x, L;                 // x's column, its lengths part's
  uint32_t cap;                 // inner lists x's level-1 offsets hold (entries - 1), and the room of `len`
  int32_t* val_off;             // out: [n_rows + 1]
  int64_t* len;                 // out: [cap]
};
struct RaggedLower {
  const EncCol* in;
  EncCol* out;
  uint32_t n_rows, n_parts;
  RaggedPart p[RAGGED_PER_LAUNCH];
  uint32_t* bad;
};
// blockIdx.y: the part; threads stride over rows [0, n_rows]
__global__ void __launch_bounds__(256) ragged_split_kernel(RaggedLower A) {
  const RaggedPart P = A.p[blockIdx.y];
  const EncCol c = A.in[P.x];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    EncCol v{}, l{};
    v.validity = c.validity; v.off[0] = P.val_off; v.off[1] = c.off[2]; v.values = c.values;
    l.validity = c.validity; l.off[0] = c.off[0]; l.values = P.len;
    A.out[P.x] = v; A.out[P.L] = l;
  }
  const int32_t* off0 = c.off[0];
  const int32_t* off1 = c.off[1];
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= A.n_rows; r += gridDim.x * blockDim.x) {
    const int32_t a = off0[r];
    bool bad = a < 0 || (uint32_t)a > P.cap;
    if (!bad) P.val_off[r] = off1[a];
    if (r == A.n_rows) { if (bad) atomicMin(A.bad, r - 1); continue; }
    const int32_t b = off0[r + 1];
    bad = bad || b < a || (uint32_t)b > P.cap;
    for (int32_t i = a; i < b && !bad; ++i) {
      const int64_t d = (int64_t)off1[i + 1] - (int64_t)off1[i];
      if (d < 0) bad = true;
      P.len[i] = d;
    }
    if (bad) atomicMin(A.bad, r);
  }
}

// ---- the row-splits partition ----
// the exclusive prefix of each thread's sum `s` over a scan tile (SCAN_THREADS threads in thread order), plus the tile's `base`
__device__ __forceinline__ uint64_t ragged_tile_prefix(uint64_t s, uint64_t base) {
  __shared__ uint64_t wsum[SCAN_THREADS / 32];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint64_t w = lane < SCAN_THREADS / 32 ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULLMASK, w, o); if (lane >= (uint32_t)o) w += y; }
    if (lane < SCAN_THREADS / 32) wsum[lane] = w;
  }
  __syncthreads();
  return x - s + (wid ? wsum[wid - 1] : 0) + base;
}

// decode: one ragged field of a decoded batch stored with row splits
struct RaggedSplitsCol {
  const int32_t* spl_off;       // splits part: level-0 offsets [n + 1]
  const int64_t* spl;           // its values
  const uint8_t* spl_valid;     // its validity bitmap
  const int32_t* val_off;       // values part: level-0 offsets [n + 1]
  const uint8_t* val_valid;
  int32_t* off0;                // out: x's level-0 offsets [n + 1]
  int32_t* off1;                // out: x's level-1 offsets, room for cap + 1 entries
  uint32_t cap;
  uint64_t* tsum;               // [n_tiles] tile sums, made their exclusive prefix by scan_tile_bases_kernel; then total, overflow
};
// the inner lists row r holds: its splits entries less one (0 for none, and for offsets that decrease)
__device__ __forceinline__ uint32_t ragged_splits_lists(const RaggedSplitsCol& C, uint32_t r) {
  const int32_t lo = C.spl_off[r], hi = C.spl_off[r + 1];
  return hi > lo ? (uint32_t)(hi - lo - 1) : 0u;
}
// step 1: the inner lists of each scan tile of rows [0, n) (n_dev as in ragged_assemble_kernel)
__global__ void __launch_bounds__(SCAN_THREADS) ragged_splits_sums_kernel(RaggedSplitsCol C, uint32_t n, const uint32_t* n_dev) {
  __shared__ uint64_t sh[32];
  if (n_dev) n = min(*n_dev, n);
  uint64_t s = 0;
  const uint32_t base = blockIdx.x * SCAN_TILE;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { const uint32_t r = base + i * SCAN_THREADS + threadIdx.x; if (r < n) s += ragged_splits_lists(C, r); }
  s = block_reduce_u64(s, sh);
  if (threadIdx.x == 0) C.tsum[blockIdx.x] = s;
}
// step 3 (after scan_tile_bases_kernel): x's level-0 offsets (each thread SCAN_ITEMS consecutive rows of its tile) and, from
// them, its level-1 offsets (the values part's level-0 offset of the row plus each splits entry but the last).  TF_FALLBACK is
// ORed into *flag when a row's parts disagree (presence, an empty splits list, a first entry other than 0, a decrease, a last
// entry other than the row's values) or x does not fit, as ragged_assemble_kernel does; the general path's pass 1 has failed
// every such record (ragged_splits_ok, decode.cuh) and passes flag = nullptr.
__global__ void __launch_bounds__(SCAN_THREADS) ragged_assemble_splits_kernel(RaggedSplitsCol C, uint32_t n, const uint32_t* n_dev, uint32_t* flag) {
  if (n_dev) n = min(*n_dev, n);
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t k[SCAN_ITEMS];
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { k[i] = base + i < n ? ragged_splits_lists(C, base + i) : 0u; s += k[i]; }
  uint64_t o = ragged_tile_prefix(s, C.tsum[blockIdx.x]);
  if (n == 0 && blockIdx.x == 0 && threadIdx.x == 0) { C.off0[0] = 0; C.off1[0] = 0; }
  bool bad = false;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    const uint32_t r = base + i;
    if (r >= n) break;
    const int32_t lo = C.spl_off[r], hi = C.spl_off[r + 1];
    const int64_t v0 = C.val_off[r], v1 = C.val_off[r + 1];
    const bool present = ((C.spl_valid[r >> 3] >> (r & 7)) & 1u) != 0;
    bool b = (((C.spl_valid[r >> 3] ^ C.val_valid[r >> 3]) >> (r & 7)) & 1u) != 0 || hi < lo || (uint32_t)hi > C.cap ||
             (present ? hi == lo || o + k[i] > C.cap : hi != lo);
    if (!b && present) {
      int64_t prev = C.spl[lo];
      b = prev != 0;
      for (int32_t j = lo + 1; j < hi; ++j) {
        C.off1[o + (uint32_t)(j - lo - 1)] = (int32_t)(v0 + prev);
        const int64_t e = C.spl[j];
        if (e < prev) b = true;
        prev = e;
      }
      if (prev != v1 - v0) b = true;
    }
    C.off0[r] = (int32_t)o;
    o += k[i];
    if (r == n - 1) { C.off0[n] = (int32_t)o; if (o <= C.cap) C.off1[o] = (int32_t)v1; }
    bad = bad || b;
  }
  if (bad && flag) atomicOr(flag, (uint32_t)TF_FALLBACK);
}

// encode: the splits variant of ragged_split_kernel.  x's values part as there; its splits part has level-0 offsets
// off0[r] + (non-null rows before r), a prefix count (ragged_split_counts_kernel -> scan_tile_bases_kernel -> the split), and a
// non-null row's values off1[i] - off1[off0[r]] for i in [off0[r], off0[r + 1]].  A null row writes no values (the emit kernels
// skip it).  The same rows are atomicMin'd into *bad as there.  Kernel arguments only.
struct RaggedSplitsPart {
  int32_t x, L;                 // x's column, its splits part's
  uint32_t cap;                 // inner lists x's level-1 offsets hold
  int32_t* val_off;             // out: [n_rows + 1]
  int32_t* spl_off;             // out: [n_rows + 1]
  int64_t* spl;                 // out: [cap + n_rows]
  uint64_t* tsum;               // [n_tiles] non-null rows per tile -> their exclusive prefix; then total, overflow
};
struct RaggedSplitsLower {
  const EncCol* in;
  EncCol* out;
  uint32_t n_rows, n_parts;     // the grid's x covers rows [0, n_rows]: n_rows / SCAN_TILE + 1 tiles
  RaggedSplitsPart p[RAGGED_PER_LAUNCH];
  uint32_t* bad;
};
// blockIdx.y: the part; blockIdx.x: a scan tile
__global__ void __launch_bounds__(SCAN_THREADS) ragged_split_counts_kernel(RaggedSplitsLower A) {
  __shared__ uint64_t sh[32];
  const RaggedSplitsPart& P = A.p[blockIdx.y];
  const EncCol c = A.in[P.x];
  uint64_t s = 0;
  const uint32_t base = blockIdx.x * SCAN_TILE;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { const uint32_t r = base + i * SCAN_THREADS + threadIdx.x; if (r < A.n_rows && enc_valid(c, r)) ++s; }
  s = block_reduce_u64(s, sh);
  if (threadIdx.x == 0) P.tsum[blockIdx.x] = s;
}
__global__ void __launch_bounds__(SCAN_THREADS) ragged_split_splits_kernel(RaggedSplitsLower A) {
  const RaggedSplitsPart P = A.p[blockIdx.y];
  const EncCol c = A.in[P.x];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    EncCol v{}, l{};
    v.validity = c.validity; v.off[0] = P.val_off; v.off[1] = c.off[2]; v.values = c.values;
    l.validity = c.validity; l.off[0] = P.spl_off; l.values = P.spl;
    A.out[P.x] = v; A.out[P.L] = l;
  }
  const int32_t* off0 = c.off[0];
  const int32_t* off1 = c.off[1];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  bool nn[SCAN_ITEMS];
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { nn[i] = base + i < A.n_rows && enc_valid(c, base + i); s += nn[i] ? 1u : 0u; }
  uint64_t nb = ragged_tile_prefix(s, P.tsum[blockIdx.x]);
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    const uint32_t r = base + i;
    if (r > A.n_rows) break;
    const int32_t a = off0[r];
    bool bad = a < 0 || (uint32_t)a > P.cap;
    if (!bad) { P.val_off[r] = off1[a]; P.spl_off[r] = (int32_t)(a + nb); }
    if (r == A.n_rows) { if (bad) atomicMin(A.bad, r - 1); break; }
    const int32_t b = off0[r + 1];
    bad = bad || b < a || (uint32_t)b > P.cap;
    int64_t* out = P.spl + (size_t)a + nb;
    if (!bad && nn[i]) out[0] = 0;
    for (int32_t j = a; j < b && !bad; ++j) {
      if (off1[j + 1] < off1[j]) bad = true;
      else if (nn[i]) out[j - a + 1] = (int64_t)off1[j + 1] - (int64_t)off1[a];
    }
    if (bad) atomicMin(A.bad, r);
    nb += nn[i] ? 1u : 0u;
  }
}
