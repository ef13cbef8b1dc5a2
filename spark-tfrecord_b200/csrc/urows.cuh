// urows.cuh -- a decoded batch's rows as Spark UnsafeRows, on the device (tfr_batch_rows).
//
// A separate pass over the batch's device columns (the Arrow outputs of any decode path: tile, general, ByteArray, redo);
// nothing of it runs unless a caller asks for rows.  include/tfrgpu.h restates the layout.  Three steps:
//   urows_size_kernel : lane = row.  Reads the validity words and the offsets of every column (coalesced at [r]) and sums the
//                       row's bytes in 64 bits: 8 * (null words + fields), plus each variable value padded to 8 bytes (and the
//                       partition row's variable region).  It
//                       also stores where each variable value starts inside its row (`pos`, [n_var][n_rows]), so that the
//                       emit kernel can hand fields to its warps independently: recomputing a field's position there would
//                       cost every warp a walk over all the variable fields in front of it (for string arrays, over their
//                       inner offsets too).  A row beyond INT32_MAX bytes (UnsafeRow.sizeInBytes is an int) is flagged.
//   (scan.cuh)        : row sizes -> int64 row offsets (the three scan launches, scan_apply64_kernel writing int64).
//   urows_emit_kernel : CTA = 32 consecutive rows, UROWS_WARPS warps.  The tile's output is one contiguous span
//                       [off[r0], off[r0 + 32]); it is assembled in shared memory -- zeroed first, so padding and null slots
//                       are defined -- and goes out with 16-byte stores (8-byte head / tail by single threads).  Warp w takes
//                       fields w, w + UROWS_WARPS, ...; lane = row writes the null bit and the slot (fixed-width values read at
//                       [r]), then the value: a short one by its lane, a long one (UROWS_BIG bytes or more) by the whole warp.
//                       A tile larger than the shared-memory budget is written to global memory by the same code with another
//                       base pointer.  Partition values (tfr_batch_rows_with_partition) are the same in every row: the warps
//                       then share each row's partition null bits, slots and variable region, lane = row, read from a
//                       small table in global memory that every CTA reads (L1 / L2 hits after the first).
// Only the batch's column buffers and this pass's own scratch are read.
//
// tfr_batch_rows_async enqueues the same pass before the batch's row count is known on the host (api_decode.inc): the size
// kernel's CAP instantiation runs over the batch's row CAPACITY and reads the true count from the control words (UrCtl) in
// device memory, the scans run over the capacity unchanged (so every offset from the count on equals the total),
// urows_verdict_kernel checks what the host could not (the decode's verdict, the rows block's capacity, a too-large row), and
// the emit kernel's GUARD instantiation does nothing once the verdict is raised.  The host then rebuilds the rows through the
// synchronous path.  CAP = false and GUARD = false are the kernels tfr_batch_rows launches; they never read the control words.
//
// Reference semantics: what Spark's UnsafeProjection makes of the SpecificInternalRow TFRecordDeserializer fills
// (M/TFRecordDeserializer.scala:21-61): the published UnsafeRow / UnsafeArrayData layout.
#pragma once
#include "common.cuh"
#include "scan.cuh"

#define UROWS_TILE 32
#define UROWS_WARPS 4
#define UROWS_SIZE_THREADS 256
#define UROWS_BIG 256u

// UR_VEC: a VectorUDT field (include/tfrgpu.h, VECTORS), a float64 list column written as the nested row of a dense vector.
// UR_SVEC: a sparse-vector field (SPARSE VECTORS), its values column written with its indices and size columns (cols[part],
// cols[part + 1], which are not row fields of their own) as the nested row of a sparse vector.
// UR_FIX1, UR_FIX2: a BooleanType / ByteType or ShortType scalar (include/tfrgpu.h, INT64 TYPES), whose arrays have 1- and 2-byte
// elements.  Only the emit kernel's NW instantiation writes them; NW = false is the kernel of every other schema.
enum { UR_NULL = 0, UR_FIX4 = 1, UR_FIX8 = 2, UR_BYTES = 3, UR_ARR = 4, UR_ARR2 = 5, UR_VEC = 6, UR_SVEC = 7, UR_FIX1 = 8, UR_FIX2 = 9 };
#define UR_VEC_HEAD 40u         // the nested row's fixed part: one null word and four slots

struct UrCol {                  // one decoded column (tfr_column), device pointers
  const uint32_t* valid;        // Arrow validity as 32-bit words
  const int32_t* off[3];        // offsets levels
  const uint8_t* values;
  int32_t kind;                 // UR_*
  int32_t width;                // leaf bytes of a numeric leaf (1 / 2 / 4 / 8); 0 for string / binary leaves
  int32_t var;                  // index among the variable-width fields (UR_BYTES, UR_ARR, UR_ARR2, UR_VEC, UR_SVEC), -1 otherwise
  int32_t part;                 // UR_SVEC: the column of its indices (its size's follows), 0 otherwise
};

struct UrArgs {
  const UrCol* cols;            // [nf], then the columns of the sparse vectors' parts
  uint32_t nf, nw, n_rows;      // nw: null words of the full row, (nf + np + 63) / 64
  // the partition values (tfr_batch_rows_with_partition), the same in every row: np slots after the nf data slots, null bit
  // nf + j, and the partition row's variable region (pvw words) at the end of the row.  np = pvw = 0 without them.
  uint32_t np, pt0, ptn, pvw;   // null words [pt0, pt0 + ptn) hold partition bits
  const unsigned long long* ptmpl;   // [nw] the partition null bits at their full-row indexes, every other bit zero
  const unsigned long long* pslot;   // [np] the partition slots; relocated ones hold (offset - Fp) << 32 | size
  const uint8_t* prel;               // [np] 1: add the row's start of the partition variable region to the offset
  const unsigned long long* pvar;    // [pvw] the partition row's variable region
  uint32_t* size;               // [n_rows] row bytes (0 for a row that is too large)
  uint32_t* pos;                // [n_var][n_rows] where each variable value starts in its row
  const int64_t* offs;          // [n_rows + 1] row offsets (scan output)
  uint8_t* out;                 // the rows (8-byte aligned)
  uint32_t* too_large;          // first row beyond INT32_MAX bytes, 0xffffffff none
  uint32_t smem_cap;            // tile bytes the shared-memory staging holds
};

// control words of the rows pass (uint32, in its scratch): the too-large row and the scan overflow are those of tfr_batch_rows;
// the asynchronous pass adds the row count and the decode flags it was given (copied from the decode's result block, or
// written by the host), the verdict, and the total bytes
enum { URC_TOO_LARGE = 0, URC_OVERFLOW = 1, URC_N = 2, URC_DFLAGS = 3, URC_VERDICT = 4, URC_TOTAL = 6, URC_WORDS = 8 };

__device__ __forceinline__ uint64_t ur_pad8(uint64_t v) { return (v + 7) & ~7ull; }
__device__ __forceinline__ uint64_t ur_hdr(uint64_t n) { return 8 + (n + 63) / 64 * 8; }     // numElements + element null bitset

// bytes of the 1-D array whose elements are [e0, e1) of offsets level `lvl` + 1 (numeric leaves: of the values)
__device__ __forceinline__ uint64_t ur_arr1_bytes(const UrCol& c, int lvl, int64_t e0, int64_t e1) {
  const uint64_t m = (uint64_t)(e1 - e0);
  if (c.width) return ur_hdr(m) + ur_pad8(m * (uint64_t)c.width);
  const int32_t* o = c.off[lvl + 1];
  uint64_t s = ur_hdr(m) + 8 * m;
  for (int64_t j = e0; j < e1; ++j) s += ur_pad8((uint64_t)(o[j + 1] - o[j]));
  return s;
}
__device__ __forceinline__ bool ur_present(const UrCol& c, uint32_t r) {
  return c.kind != UR_NULL && ((c.valid[r >> 5] >> (r & 31)) & 1u);
}
// the raw size of field c's value in row r (what its slot holds): string / binary length, array or nested row bytes
__device__ __forceinline__ uint64_t ur_value_bytes(const UrCol& c, const UrCol* cols, uint32_t r) {
  const int32_t* o0 = c.off[0];
  const int64_t a = o0[r], b = o0[r + 1];
  if (c.kind == UR_BYTES) return (uint64_t)(b - a);
  if (c.kind == UR_ARR) return ur_arr1_bytes(c, 0, a, b);
  if (c.kind == UR_VEC) return UR_VEC_HEAD + ur_arr1_bytes(c, 0, a, b);
  if (c.kind == UR_SVEC) {                                  // the indices array (when not null), then the values array
    const UrCol& ci = cols[c.part];
    return UR_VEC_HEAD + ur_arr1_bytes(c, 0, a, b) + (ur_present(ci, r) ? ur_arr1_bytes(ci, 0, ci.off[0][r], ci.off[0][r + 1]) : 0);
  }
  uint64_t s = ur_hdr((uint64_t)(b - a)) + 8 * (uint64_t)(b - a);          // UR_ARR2: steps are inner arrays
  const int32_t* o1 = c.off[1];
  for (int64_t k = a; k < b; ++k) s += ur_arr1_bytes(c, 1, o1[k], o1[k + 1]);
  return s;
}

// CAP: launched over the row capacity A.n_rows (the stride of `pos`); rows at or beyond ctl[URC_N] get size 0 and read no column
// memory (a speculative batch's offsets past its count are garbage), and so does every row when the decode raised a flag or
// counted more rows than the capacity.  CAP = false never reads `ctl`.
template <bool CAP>
__global__ void __launch_bounds__(UROWS_SIZE_THREADS) urows_size_kernel(UrArgs A, const uint32_t* ctl) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= A.n_rows) return;
  if (CAP) {
    const uint32_t n = ctl[URC_N];
    if (ctl[URC_DFLAGS] || n > A.n_rows || r >= n) { A.size[r] = 0u; return; }
  }
  uint64_t s = 8ull * (A.nw + A.nf + A.np);
  for (uint32_t f = 0; f < A.nf; ++f) {
    const UrCol& c = A.cols[f];
    if (c.var < 0) continue;
    A.pos[(size_t)c.var * A.n_rows + r] = (uint32_t)s;
    if (ur_present(c, r)) s += ur_pad8(ur_value_bytes(c, A.cols, r));
  }
  s += 8ull * A.pvw;
  const bool big = s > 0x7fffffffull;
  A.size[r] = big ? 0u : (uint32_t)s;
  if (big) atomicMin(A.too_large, r);
}

// 8 little-endian bytes of src[0 .. min(n, 8)), zero above
__device__ __forceinline__ uint64_t ur_gather8(const uint8_t* src, uint64_t n) {
  uint64_t w = 0;
  const uint32_t k = n < 8 ? (uint32_t)n : 8u;
  for (uint32_t j = 0; j < k; ++j) w |= (uint64_t)src[j] << (8 * j);
  return w;
}
// n bytes to an 8-byte aligned, zeroed destination whose padding up to 8 bytes belongs to the value: word k by k0, k0 + step, ...
__device__ __forceinline__ void ur_copy_bytes(uint8_t* dst, const uint8_t* src, uint64_t n, uint32_t k0, uint32_t step) {
  for (uint64_t k = 8ull * k0; k < n; k += 8ull * step)
    *reinterpret_cast<unsigned long long*>(dst + k) = ur_gather8(src + k, n - k);
}
// m numeric leaves of width w (4 / 8, and with NW 1 / 2; w-aligned source) to an 8-byte aligned destination
template <bool NW>
__device__ __forceinline__ void ur_copy_elems(uint8_t* dst, const uint8_t* src, uint64_t m, int w, uint32_t k0, uint32_t step) {
  if (NW && w == 1) {
    for (uint64_t i = k0; i < m; i += step) dst[i] = src[i];
  } else if (NW && w == 2) {
    for (uint64_t i = k0; i < m; i += step) reinterpret_cast<uint16_t*>(dst)[i] = reinterpret_cast<const uint16_t*>(src)[i];
  } else if (w == 4) {
    for (uint64_t i = k0; i < m; i += step) reinterpret_cast<uint32_t*>(dst)[i] = reinterpret_cast<const uint32_t*>(src)[i];
  } else {
    for (uint64_t i = k0; i < m; i += step) reinterpret_cast<unsigned long long*>(dst)[i] = reinterpret_cast<const unsigned long long*>(src)[i];
  }
}
__device__ __forceinline__ void ur_st64(uint8_t* p, uint64_t v) { *reinterpret_cast<unsigned long long*>(p) = v; }

// the fixed part of a dense vector's nested row at dst (zeroed) whose values array has `arr` bytes: null bits 1 (size) and 2
// (indices), type = 1, size and indices zero slots, values = (40 << 32) | arr
__device__ __forceinline__ void ur_vec_head(uint8_t* dst, uint64_t arr) {
  ur_st64(dst, 0x6ull);
  ur_st64(dst + 8, 1ull);
  ur_st64(dst + 32, ((uint64_t)UR_VEC_HEAD << 32) | arr);
}

// row r's sparse vector of field c at dst (zeroed): the nested row of VectorUDT.serialize(SparseVector(size, indices, values)),
// its fixed part (null bit 1: size null, bit 2: indices null; type 0; the size; the two array slots) and the arrays' headers by
// k0 == 0, the elements by k0, k0 + step, ...  (a lane: 0, 1; the whole warp: lane, 32)
__device__ void ur_emit_svec(const UrCol& c, const UrCol* cols, uint32_t r, uint8_t* dst, uint32_t k0, uint32_t step) {
  const UrCol& ci = cols[c.part];
  const UrCol& cs = cols[c.part + 1];
  const bool ip = ur_present(ci, r), sp = ur_present(cs, r);
  const int64_t a = c.off[0][r], b = c.off[0][r + 1], ia = ip ? ci.off[0][r] : 0, ib = ip ? ci.off[0][r + 1] : 0;
  const uint64_t m = (uint64_t)(b - a), mi = (uint64_t)(ib - ia);
  const uint64_t ibytes = ip ? ur_arr1_bytes(ci, 0, ia, ib) : 0, vo = UR_VEC_HEAD + ibytes;
  if (k0 == 0) {
    ur_st64(dst, (sp ? 0ull : 2ull) | (ip ? 0ull : 4ull));
    if (sp) ur_st64(dst + 16, (uint64_t)reinterpret_cast<const uint32_t*>(cs.values)[r]);
    if (ip) { ur_st64(dst + 24, ((uint64_t)UR_VEC_HEAD << 32) | ibytes); ur_st64(dst + UR_VEC_HEAD, mi); }
    ur_st64(dst + 32, (vo << 32) | ur_arr1_bytes(c, 0, a, b));
    ur_st64(dst + vo, m);
  }
  if (ip) ur_copy_elems<false>(dst + UR_VEC_HEAD + ur_hdr(mi), ci.values + (uint64_t)ia * 4, mi, 4, k0, step);
  ur_copy_elems<false>(dst + vo + ur_hdr(m), c.values + (uint64_t)a * 8, m, 8, k0, step);
}

// one lane writes the 1-D array of elements [e0, e1) of level lvl + 1 at dst (zeroed); returns its bytes
template <bool NW>
__device__ uint64_t ur_emit_arr1_lane(const UrCol& c, int lvl, int64_t e0, int64_t e1, uint8_t* dst) {
  const uint64_t m = (uint64_t)(e1 - e0), h = ur_hdr(m);
  ur_st64(dst, m);                                                           // the element null bitset stays zero
  if (c.width) {
    ur_copy_elems<NW>(dst + h, c.values + (uint64_t)e0 * c.width, m, c.width, 0, 1);
    return h + ur_pad8(m * (uint64_t)c.width);
  }
  const int32_t* o = c.off[lvl + 1];
  uint64_t p = h + 8 * m;
  for (int64_t j = e0; j < e1; ++j) {
    const uint64_t len = (uint64_t)(o[j + 1] - o[j]);
    ur_st64(dst + h + 8 * (uint64_t)(j - e0), (p << 32) | len);
    ur_copy_bytes(dst + p, c.values + o[j], len, 0, 1);
    p += ur_pad8(len);
  }
  return p;
}

// inclusive warp scan
__device__ __forceinline__ uint64_t ur_warp_scan(uint64_t x) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
  return x;
}

// the whole warp writes row r's value of field c at dst (zeroed); warp-uniform call
template <bool NW>
__device__ void ur_emit_warp(const UrCol& c, uint32_t r, uint8_t* dst) {
  const uint32_t lane = threadIdx.x & 31;
  const int64_t a = c.off[0][r], b = c.off[0][r + 1];
  if (c.kind == UR_BYTES) { ur_copy_bytes(dst, c.values + a, (uint64_t)(b - a), lane, 32); return; }
  const uint64_t m = (uint64_t)(b - a), h = ur_hdr(m);
  if (c.kind == UR_VEC) {                                  // the nested row's fixed part, then its values array as UR_ARR's
    if (lane == 0) ur_vec_head(dst, ur_arr1_bytes(c, 0, a, b));
    dst += UR_VEC_HEAD;
  }
  if (lane == 0) ur_st64(dst, m);
  if ((c.kind == UR_ARR || c.kind == UR_VEC) && c.width) { ur_copy_elems<NW>(dst + h, c.values + (uint64_t)a * c.width, m, c.width, lane, 32); return; }
  // elements with an (offset << 32 | size) slot each: strings / binaries (UR_ARR) or inner arrays (UR_ARR2).  32 at a time,
  // each lane sizes its element, a scan places them, each lane writes its element
  uint64_t base = h + 8 * m;
  for (int64_t k0 = a; k0 < b; k0 += 32) {
    const int64_t k = k0 + lane;
    const bool on = k < b;
    uint64_t len = 0;
    if (on) len = c.kind == UR_ARR ? (uint64_t)(c.off[1][k + 1] - c.off[1][k]) : ur_arr1_bytes(c, 1, c.off[1][k], c.off[1][k + 1]);
    const uint64_t incl = ur_warp_scan(ur_pad8(len)), p = base + incl - ur_pad8(len);
    if (on) {
      ur_st64(dst + h + 8 * (uint64_t)(k - a), (p << 32) | len);
      if (c.kind == UR_ARR) ur_copy_bytes(dst + p, c.values + c.off[1][k], len, 0, 1);
      else ur_emit_arr1_lane<NW>(c, 1, c.off[1][k], c.off[1][k + 1], dst + p);
    }
    base += __shfl_sync(FULLMASK, incl, 31);
  }
}

// one lane writes row r's value of field c at dst (zeroed)
template <bool NW>
__device__ void ur_emit_lane(const UrCol& c, uint32_t r, uint8_t* dst) {
  const int64_t a = c.off[0][r], b = c.off[0][r + 1];
  if (c.kind == UR_BYTES) { ur_copy_bytes(dst, c.values + a, (uint64_t)(b - a), 0, 1); return; }
  if (c.kind == UR_ARR) { ur_emit_arr1_lane<NW>(c, 0, a, b, dst); return; }
  if (c.kind == UR_VEC) { ur_vec_head(dst, ur_emit_arr1_lane<NW>(c, 0, a, b, dst + UR_VEC_HEAD)); return; }
  const uint64_t m = (uint64_t)(b - a), h = ur_hdr(m);
  ur_st64(dst, m);
  uint64_t p = h + 8 * m;
  for (int64_t k = a; k < b; ++k) {
    const uint64_t len = ur_emit_arr1_lane<NW>(c, 1, c.off[1][k], c.off[1][k + 1], dst + p);
    ur_st64(dst + h + 8 * (uint64_t)(k - a), (p << 32) | len);
    p += len;
  }
}

// After the scan, one thread: raises ctl[URC_VERDICT] when the rows the asynchronous pass built cannot be handed out -- the
// decode raised a flag or counted more rows than its capacity `n_alloc` (the batch is redone), the rows need more than the
// `rows_cap` bytes of their block, or a row is larger than INT32_MAX bytes -- and stores the total at ctl[URC_TOTAL].
__global__ void urows_verdict_kernel(uint32_t* ctl, const uint64_t* total, uint32_t n_alloc, unsigned long long rows_cap) {
  const uint64_t t = *total;
  const bool bad = ctl[URC_DFLAGS] != 0u || ctl[URC_N] > n_alloc || t > rows_cap || ctl[URC_TOO_LARGE] != 0xffffffffu;
  ctl[URC_VERDICT] = bad ? 1u : 0u;
  *reinterpret_cast<unsigned long long*>(ctl + URC_TOTAL) = t;
}

// GUARD: the asynchronous pass's instantiation.  It returns at once when urows_verdict_kernel has raised the verdict, takes the
// row count from ctl[URC_N] (A.n_rows is the capacity, the stride of `pos`), and CTAs past the count exit.  GUARD = false never
// reads `ctl`.  NW: the schema has a field of a 1- or 2-byte type (UR_FIX1, UR_FIX2).
template <bool GUARD, bool NW>
__global__ void __launch_bounds__(UROWS_WARPS * 32) urows_emit_kernel(UrArgs A, const uint32_t* ctl) {
  extern __shared__ __align__(16) uint8_t ur_smem[];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t n_rows = GUARD ? ctl[URC_N] : A.n_rows;
  if (GUARD && (ctl[URC_VERDICT] || blockIdx.x * UROWS_TILE >= n_rows)) return;
  const uint32_t r0 = blockIdx.x * UROWS_TILE, rows = min((uint32_t)UROWS_TILE, n_rows - r0);
  const int64_t t_lo = A.offs[r0], t_hi = A.offs[r0 + rows];
  const uint64_t span = (uint64_t)(t_hi - t_lo);
  const uint32_t phase = (uint32_t)(t_lo & 15);                   // smem keeps the output's 16-byte phase: 16-byte stores out
  const bool staged = span + phase <= A.smem_cap;
  uint8_t* gtile = A.out + t_lo;
  uint8_t* base = staged ? ur_smem + phase : gtile;
  // ---- zero the span: padding, null slots and element null bitsets stay so ----
  if (staged) {
    const uint32_t n16 = (uint32_t)((phase + span + 15) / 16);
    for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) reinterpret_cast<uint4*>(ur_smem)[i] = make_uint4(0, 0, 0, 0);
  } else {
    for (uint64_t i = threadIdx.x; i < span / 8; i += blockDim.x) ur_st64(gtile + 8 * i, 0);
  }
  __syncthreads();
  // ---- fields: warp w takes w, w + UROWS_WARPS, ...; lane = row ----
  const bool act = lane < rows;
  const uint32_t r = r0 + lane;
  uint8_t* row = base + (act ? (uint64_t)(A.offs[r] - t_lo) : 0);
  for (uint32_t f = warp; f < A.nf; f += UROWS_WARPS) {
    const UrCol& c = A.cols[f];
    const uint32_t vw = c.kind == UR_NULL ? 0u : c.valid[blockIdx.x];     // validity of rows r0 .. r0 + 31
    const bool present = act && ((vw >> lane) & 1u);
    if (act && !present) atomicOr(reinterpret_cast<unsigned long long*>(row + 8ull * (f >> 6)), 1ull << (f & 63));
    uint8_t* slot = row + 8ull * (A.nw + f);
    if (NW && (c.kind == UR_FIX1 || c.kind == UR_FIX2)) {            // the slot zeroed, then 1 or 2 bytes
      if (present) ur_st64(slot, c.kind == UR_FIX1 ? (uint64_t)c.values[r] : (uint64_t)reinterpret_cast<const uint16_t*>(c.values)[r]);
      continue;
    }
    if (c.kind == UR_FIX4 || c.kind == UR_FIX8) {
      if (present) ur_st64(slot, c.kind == UR_FIX4 ? (uint64_t)reinterpret_cast<const uint32_t*>(c.values)[r]
                                                   : (uint64_t)reinterpret_cast<const unsigned long long*>(c.values)[r]);
      continue;
    }
    if (c.var < 0) continue;
    uint64_t len = 0, p = 0;
    if (present) {
      len = ur_value_bytes(c, A.cols, r);
      p = A.pos[(size_t)c.var * A.n_rows + r];
      ur_st64(slot, (p << 32) | len);
    }
    const bool big = present && ur_pad8(len) >= UROWS_BIG;
    if (present && !big) { if (c.kind == UR_SVEC) ur_emit_svec(c, A.cols, r, row + p, 0, 1); else ur_emit_lane<NW>(c, r, row + p); }
    uint32_t mb = __ballot_sync(FULLMASK, big);
    while (mb) {
      const int l = __ffs(mb) - 1;
      mb &= mb - 1;
      uint8_t* d = (uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)(row + p), l);
      if (c.kind == UR_SVEC) ur_emit_svec(c, A.cols, r0 + (uint32_t)l, d, lane, 32);
      else ur_emit_warp<NW>(c, r0 + (uint32_t)l, d);
    }
  }
  // ---- the partition values: lane = row, warp w takes units w, w + UROWS_WARPS, ... of [the null words holding partition
  //      bits | the np slots | the variable region's words], so every thread of the CTA shares the constant part ----
  const uint32_t pn = A.ptn + A.np + A.pvw;
  if (act && pn) {
    const uint64_t pv0 = (uint64_t)(A.offs[r + 1] - A.offs[r]) - 8ull * A.pvw;     // where the region starts in this row
    for (uint32_t k = warp; k < pn; k += UROWS_WARPS) {
      if (k < A.ptn) {
        const unsigned long long m = A.ptmpl[A.pt0 + k];
        if (m) atomicOr(reinterpret_cast<unsigned long long*>(row + 8ull * (A.pt0 + k)), m);   // shares a word with data bits
      } else if (k < A.ptn + A.np) {
        const uint32_t j = k - A.ptn;
        ur_st64(row + 8ull * (A.nw + A.nf + j), A.pslot[j] + (A.prel[j] ? pv0 << 32 : 0ull));
      } else {
        const uint32_t i = k - A.ptn - A.np;
        ur_st64(row + pv0 + 8ull * i, A.pvar[i]);
      }
    }
  }
  if (!staged) return;
  // ---- the span out: 16-byte stores; an 8-byte head / tail by single threads ----
  __syncthreads();
  const uintptr_t g_lo = reinterpret_cast<uintptr_t>(gtile), g_hi = g_lo + span;
  const uintptr_t b_lo = (g_lo + 15) & ~uintptr_t(15), b_hi = max(g_hi & ~uintptr_t(15), b_lo);
  const uint8_t* s16 = ur_smem + (b_lo - (g_lo - phase));
  for (uintptr_t i = threadIdx.x; i < (b_hi - b_lo) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(b_lo)[i] = reinterpret_cast<const uint4*>(s16)[i];
  if (threadIdx.x == 0 && g_lo < min(b_lo, g_hi)) ur_st64(gtile, *reinterpret_cast<const unsigned long long*>(base));
  if (threadIdx.x == 32 && b_hi < g_hi) ur_st64(reinterpret_cast<uint8_t*>(b_hi), *reinterpret_cast<const unsigned long long*>(base + (b_hi - g_lo)));
}
