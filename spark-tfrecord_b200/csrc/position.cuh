// position.cuh -- the generated fields TFR_T_ROW_INDEX and TFR_T_RECORD_OFFSET (include/tfrgpu.h, POSITIONS): every delivered
// row's entry index and the file offset of its entry, written after a batch's final row set exists.  The parse kernels never
// see these fields (they are out of the key hash table, so every kernel writes them as an absent nullable field); this kernel
// then overwrites their values, sets every validity bit and zeroes their null counters.
//
// Row r -> (kept index s, entries k in front of it that gave no row of their own), from the batch's list of dropped / corrupt
// entries `bad` (block order, each with its entry index `row`, DroppedFrame):
//   rows are the kept frames (FAILFAST, DROPMALFORMED): k = the entries j with bad[j].row - j <= r (bad[j].row - j is the
//       number of kept rows in front of entry j, non-decreasing); s = r; entry = r + k.  FAILFAST has no list: entry = r.
//   rows are entries (PERMISSIVE): entry = r; k = the entries of the list below r; r is itself in the list when bad[k].row
//       == r (its offset is bad[k].off); otherwise s = r - k.
// A kept row's offset: rec_off[s] of the final decode round (which decoded the kept frames back to back) moved to the block:
// kept rows between two listed entries are contiguous in both, and the first kept row after bad[k-1] -- kept index
// bad[k-1].row - (k-1) -- starts where that entry ends.
#pragma once
#include "common.cuh"
#include "drop.cuh"

struct PositionArgs {
  int64_t* index; int64_t* offset;              // the columns' values (null: the field is not in the schema)
  uint32_t* index_bits; uint32_t* offset_bits;  // their validity bitmaps
  unsigned long long* index_nulls; unsigned long long* offset_nulls;   // their null counters
  const uint32_t* rec_off;                      // the final decode round's frame offsets
  const uint32_t* n_dev; uint32_t n;            // rows: min(*n_dev, n) when n_dev is set (pipelined: n is the capacity), else n
  const DroppedFrame* bad; uint32_t n_bad;      // the batch's dropped or corrupt entries, in block order
  uint32_t rows_are_entries;                    // PERMISSIVE
  int64_t first_entry, first_offset;            // the block's position in its file
};

#define POSITION_THREADS 256

// One thread per row, grid-stride by whole warps; validity words are written whole from the warp's ballot.
__global__ void __launch_bounds__(POSITION_THREADS) position_kernel(const PositionArgs A) {
  const uint32_t n = A.n_dev ? min(*A.n_dev, A.n) : A.n;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (A.index_nulls) *A.index_nulls = 0ull;
    if (A.offset_nulls) *A.offset_nulls = 0ull;
  }
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t r0 = (blockIdx.x * POSITION_THREADS + threadIdx.x) & ~31u; r0 < n; r0 += gridDim.x * POSITION_THREADS) {
    const uint32_t r = r0 + lane;
    const bool row = r < n;
    if (row) {
      uint32_t lo = 0, hi = A.n_bad;
      if (A.rows_are_entries) while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (A.bad[mid].row < r) lo = mid + 1; else hi = mid; }
      else while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (A.bad[mid].row - mid <= r) lo = mid + 1; else hi = mid; }
      const uint32_t k = lo;
      uint32_t off;
      if (A.rows_are_entries && k < A.n_bad && A.bad[k].row == r) off = A.bad[k].off;
      else {
        const uint32_t s = A.rows_are_entries ? r - k : r;
        off = k ? A.bad[k - 1].end + (A.rec_off[s] - A.rec_off[A.bad[k - 1].row - (k - 1)]) : A.rec_off[s];
      }
      const uint32_t entry = A.rows_are_entries ? r : r + k;
      if (A.index) A.index[r] = A.first_entry + (int64_t)entry;
      if (A.offset) A.offset[r] = A.first_offset + (int64_t)off;
    }
    const unsigned m = __ballot_sync(FULLMASK, row);
    if (lane == 0) {
      if (A.index_bits) A.index_bits[r0 >> 5] = m;
      if (A.offset_bits) A.offset_bits[r0 >> 5] = m;
    }
  }
}
