// permissive.cuh -- PERMISSIVE (TFR_F_PERMISSIVE): the rows of a batch's kept records (drop.cuh's second decode round)
// spread back over every frame of the batch, with a row of nulls at each failing frame.
//
// Output row r of n_total = n_kept + n_bad rows: bad_before(r) is the number of failing frames below r (a binary search of
// drop_list_kernel's list, which is in record order), and src = r - bad_before(r) is the kept row it takes.  A failing row
// is null in every data field with zero values, and zero-length in every list or string column (its level-0 offset
// repeats); the corrupt-record column is valid exactly there, its offsets the running sum of the failing payloads.  Deeper
// offsets levels and leaf values do not move: the host keeps the kept round's variable-width block as it is.
#pragma once
#include "common.cuh"
#include "drop.cuh"

enum ExpandKind : uint32_t { EXP_NONE = 0, EXP_FIX = 1, EXP_VAR = 2, EXP_CORRUPT = 3 };

// one schema field: what the expansion writes for it and where, as byte offsets into the kept round's fixed block (`src`)
// and the new one (`dst`): the fixed-width values (EXP_FIX), the level-0 offsets (EXP_VAR, EXP_CORRUPT), nothing beyond
// the validity bitmap (EXP_NONE: NullType)
struct ExpandField { uint32_t kind, width; uint64_t src, dst; };
static_assert(sizeof(ExpandField) == 24, "ExpandField layout");

struct ExpandArgs {
  const uint8_t* src_fx; uint8_t* dst_fx;       // the two fixed blocks (validity bitmaps at offset 0 of each)
  uint32_t src_stride, dst_stride;              // their bitmaps' stride
  uint64_t src_nullc, dst_nullc;                // their null counters
  const ExpandField* fields; uint32_t nf;
  const DroppedFrame* bad; uint32_t n_bad;      // the failing frames, in record order
  const uint32_t* cum;                          // [n_bad + 1]: payload bytes of the failing frames before each
  uint32_t n_total;
};

#define EXPAND_THREADS 256

// One warp per 32 output rows (and the end entry of the offsets, row n_total): one binary search per row, then every field.
// Validity words are written whole, from the warp's ballot, so no two threads write the same word.
__global__ void permissive_expand_kernel(const ExpandArgs A) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t r0 = ((blockIdx.x * EXPAND_THREADS + threadIdx.x) >> 5) * 32u;
  if (blockIdx.x == 0)
    for (uint32_t f = threadIdx.x; f < A.nf; f += EXPAND_THREADS) {
      const unsigned long long kept = reinterpret_cast<const unsigned long long*>(A.src_fx + A.src_nullc)[f];
      reinterpret_cast<unsigned long long*>(A.dst_fx + A.dst_nullc)[f] = A.fields[f].kind == EXP_CORRUPT ? (unsigned long long)(A.n_total - A.n_bad)
                                                                                                          : kept + A.n_bad;
    }
  if (r0 > A.n_total) return;                                    // (whole warps)
  const uint32_t r = r0 + lane;
  uint32_t lo = 0, hi = A.n_bad;                                 // bad_before(r): failing frames with an index below r
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (A.bad[mid].row < r) lo = mid + 1; else hi = mid; }
  const uint32_t bb = lo, src = r - bb;
  const bool row = r < A.n_total;
  const bool is_bad = row && bb < A.n_bad && A.bad[bb].row == r;
  for (uint32_t f = 0; f < A.nf; ++f) {
    const ExpandField F = A.fields[f];
    bool bit;
    if (F.kind == EXP_CORRUPT) bit = is_bad;
    else bit = row && !is_bad && ((A.src_fx[(size_t)f * A.src_stride + (src >> 3)] >> (src & 7u)) & 1u);
    const unsigned m = __ballot_sync(FULLMASK, bit);
    if (lane == 0 && r0 < A.n_total) reinterpret_cast<uint32_t*>(A.dst_fx + (size_t)f * A.dst_stride)[r0 >> 5] = m;
    if (F.kind == EXP_FIX) {
      if (!row) continue;
      if (F.width == 8) {
        const uint64_t v = is_bad ? 0ull : reinterpret_cast<const uint64_t*>(A.src_fx + F.src)[src];
        reinterpret_cast<uint64_t*>(A.dst_fx + F.dst)[r] = v;
      } else {
        const uint32_t v = is_bad ? 0u : reinterpret_cast<const uint32_t*>(A.src_fx + F.src)[src];
        reinterpret_cast<uint32_t*>(A.dst_fx + F.dst)[r] = v;
      }
    } else if (r <= A.n_total) {
      if (F.kind == EXP_VAR) reinterpret_cast<int32_t*>(A.dst_fx + F.dst)[r] = reinterpret_cast<const int32_t*>(A.src_fx + F.src)[src];
      else if (F.kind == EXP_CORRUPT) reinterpret_cast<int32_t*>(A.dst_fx + F.dst)[r] = (int32_t)A.cum[bb];
    }
  }
}
