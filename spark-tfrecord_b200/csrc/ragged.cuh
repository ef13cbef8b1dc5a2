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
#pragma once
#include "common.cuh"
#include "encode.cuh"
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
