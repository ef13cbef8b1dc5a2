// rows.cuh -- Spark UnsafeRow batches -> the encoder's Arrow-layout columns (EncCol), on the device.
//
// Row r is rows[offs[r] .. offs[r+1]) in Spark's UnsafeRow layout (include/tfrgpu.h restates it).  Three kernels and the
// multi-array scan (scan.cuh) turn the rows into the columns tfr_encode would have been given for them; the encode kernels
// (encode.cuh, encode_tile.cuh, bytes_tile.cuh) then run unchanged:
//   rows_pass_a_kernel : CTA = 32 consecutive rows, lane = row.  Rows are contiguous, so the tile's bytes arrive in shared
//                        memory with one bulk copy (cp.async.bulk of the 16-byte groups inside [first, last); the 8-byte
//                        ends are copied by two lanes).  A tile larger than the staging area reads global memory instead.
//                        Each lane validates its row, the warp sets the validity words by ballot, fixed-width scalars are
//                        stored straight out and every variable-width column gets its per-level counts.
//   (scan.cuh)         : counts -> level-0 Arrow offsets (in place) and per-row bases of the inner levels.
//   rows_layout_kernel : places every variable column's inner offsets and values in two arenas sized from the input.
//   rows_pass_b_kernel : lane = row: inner offsets, string/binary bytes and array elements to their column positions.
//
// A malformed row (TFR_E_INVALID_ARG) or a row with a null string/binary/decimal element or a null inner array
// (TFR_E_NULL_IN_NONNULL) becomes an all-null row: the encode kernels then read nothing of it, and the host reports the
// first failing row.  No byte outside rows[first .. last) is ever read, whatever the input holds.
//
// Reference semantics: M/TFRecordSerializer.scala:20-60,68-207 (what the encode kernels implement); the row layout is
// Spark's published UnsafeRow / UnsafeArrayData format.
#pragma once
#include "common.cuh"
#include "encode.cuh"
#include "tile.cuh"
#include "narrow.cuh"

#define ROWS_TILE 32
#define ROWS_B_WARPS 4

struct RowsArgs {
  DevSchema sch;
  const uint8_t* rows;          // byte k of the batch is rows[k] (device address, 8-byte aligned)
  const int32_t* offs;          // [n_rows + 1]
  uint32_t n_rows;
  int64_t first, last;          // offs[0], offs[n_rows]
  uint32_t vwords;              // validity words per field, (n_rows + 31) / 32
  uint32_t* valid;              // [n_fields][vwords] Arrow bitmaps
  void* const* fixv;            // [n_fields] values of depth-0 fixed-width columns, nullptr for the others
  uint32_t* cnt;                // [n_cnt][n_rows] per-row counts of every offsets level
  int32_t* const* lev;          // [n_cnt] scan outputs: level 0 = the column's Arrow offsets, levels 1, 2 = per-row bases
  EncCol* cols;                 // [n_fields] the encoder's columns; the layout kernel fills the inner offsets and values
  uint32_t smem_cap;            // tile bytes the shared-memory staging holds
  EncStatus* st;                // rows_first_bad, rows_first_null, rows_overflow, rows_vec_lo / hi
  const uint8_t* vec;           // [n_fields] VK_*: VK_DENSE, VK_SPARSE a VectorUDT field (a float64 list column filled from the struct)
  const int32_t* part;          // [n_fields] VK_SPARSE: the field of its indices (its size's follows)
  uint32_t nu;                  // the rows' fields: the schema's but a sparse vector's parts, which are filled with it
};
// The NW instantiations of pass A and B take, beside RowsArgs, `nar`: [n_fields] a BooleanType .. TimestampType field's TFR_T_*
// (include/tfrgpu.h, INT64 TYPES), else 0.

enum { RW_OK = 0, RW_NULL = 1, RW_BAD = 2 };

__device__ __forceinline__ uint64_t rows_ld64(const uint8_t* p) { return *reinterpret_cast<const unsigned long long*>(p); }

// UnsafeArrayData at byte a of the row, sz bytes: numElements, then where the element slots start
__device__ __forceinline__ bool rows_array(const uint8_t* row, uint64_t a, uint64_t sz, uint32_t esz, uint32_t& n, uint64_t& data) {
  if (sz < 8) return false;
  const int64_t m = (int64_t)rows_ld64(row + a);
  if (m < 0 || (uint64_t)m > sz) return false;              // (also keeps the products below in range)
  const uint64_t nb = ((uint64_t)m + 63) / 64 * 8, eb = ((uint64_t)m * esz + 7) & ~7ull;
  if (8 + nb + eb > sz) return false;
  n = (uint32_t)m;
  data = a + 8 + nb;
  return true;
}
__device__ __forceinline__ bool rows_elem_null(const uint8_t* row, uint64_t a, uint32_t i) {
  return (rows_ld64(row + a + 8 + (uint64_t)(i >> 6) * 8) >> (i & 63)) & 1;
}
// (offset << 32 | size) slot of element i of the array at a (sz bytes): the element's bytes, row-relative
__device__ __forceinline__ bool rows_var_elem(const uint8_t* row, uint64_t a, uint64_t sz, uint64_t data, uint32_t i, uint64_t& eo, uint64_t& es) {
  const uint64_t s = rows_ld64(row + data + 8ull * i);
  eo = s >> 32;
  es = s & 0xffffffffu;
  if ((eo & 7) || eo + es > sz) return false;
  eo += a;
  return true;
}
__device__ __forceinline__ bool rows_is_var(const DevField& fd) { return fd.elem_type == TFR_T_STRING || fd.elem_type == TFR_T_BINARY; }

// INT64 TYPES: the int64 a row's value of type nt writes, from its slot or element bits (UnsafeRow.getBoolean is a byte != 0;
// getByte, getShort and getInt sign-extend; a timestamp is its long)
__device__ __forceinline__ long long rows_widen(int nt, uint64_t bits) {
  switch (nt) {
    case TFR_T_BOOL: return (bits & 0xffu) != 0 ? 1 : 0;
    case TFR_T_INT8: return (long long)(int8_t)bits;
    case TFR_T_INT16: return (long long)(int16_t)bits;
    case TFR_T_DATE: return (long long)(int32_t)bits;
    default: return (long long)bits;
  }
}
// element i of an UnsafeArrayData of type nt whose element slots start at row byte d (1, 1, 2, 4 or 8 bytes wide)
__device__ __forceinline__ uint64_t rows_narrow_elem(const uint8_t* row, uint64_t d, int nt, uint32_t i) {
  switch (nar_width(nt)) {
    case 1: return row[d + i];
    case 2: return reinterpret_cast<const uint16_t*>(row + d)[i];
    case 4: return reinterpret_cast<const uint32_t*>(row + d)[i];
    default: return rows_ld64(row + d + 8ull * i);
  }
}

// Counts of one non-null variable-width field: c[l] = the entries this row adds to offsets level l (level 0: bytes,
// elements or steps; deeper levels: their children).  `room` grows by the value bytes plus 8 per inner-level entry: a
// well-formed row spends at least that much of its own bytes on them, which bounds the column buffers by the input.
// NW: nt is an INT64 TYPES field's TFR_T_* (0 none), whose array elements are nar_width(nt) bytes wide in the row.
template <bool NW>
__device__ int rows_field_counts(const uint8_t* row, uint64_t len, const DevField& fd, uint64_t slot, uint32_t c[3], uint64_t& room, int nt) {
  const uint64_t o = slot >> 32, sz = slot & 0xffffffffu;
  if ((o & 7) || o + sz > len) return RW_BAD;
  const bool var = rows_is_var(fd);
  if (fd.depth == 0) { c[0] = (uint32_t)sz; room += sz; return RW_OK; }
  const uint32_t esz = var ? 8u : NW && nt ? (uint32_t)nar_width(nt) : (uint32_t)fd.width;      // int/float 4, long/double/decimal 8
  const bool null_elem_is_error = var || fd.elem_type == TFR_T_DECIMAL;   // getUTF8String / getBinary / getDecimal of a null (:118-135)
  uint32_t n;
  uint64_t d;
  if (!rows_array(row, o, sz, fd.depth == 2 ? 8u : esz, n, d)) return RW_BAD;
  c[0] = n;
  int st = RW_OK;
  if (fd.depth == 1) {
    if (!var) {
      if (null_elem_is_error)
        for (uint32_t i = 0; i < n; ++i) if (rows_elem_null(row, o, i)) { st = RW_NULL; break; }
      room += (uint64_t)n * esz;
      return st;
    }
    uint64_t bytes = 0, eo, es;
    for (uint32_t i = 0; i < n; ++i) {
      if (rows_elem_null(row, o, i)) { st = RW_NULL; continue; }
      if (!rows_var_elem(row, o, sz, d, i, eo, es)) return RW_BAD;
      bytes += es;
    }
    c[1] = (uint32_t)bytes;
    room += bytes + 8ull * n;
    return st;
  }
  // depth 2: the steps are arrays (a null step: the inner array's toArray of null, :141-142)
  uint64_t e1 = 0, e2 = 0, eo, es;
  for (uint32_t s = 0; s < n; ++s) {
    if (rows_elem_null(row, o, s)) { st = RW_NULL; continue; }
    if (!rows_var_elem(row, o, sz, d, s, eo, es)) return RW_BAD;
    uint32_t m;
    uint64_t d2;
    if (!rows_array(row, eo, es, esz, m, d2)) return RW_BAD;
    e1 += m;
    if (var) {
      uint64_t fo, fs;
      for (uint32_t j = 0; j < m; ++j) {
        if (rows_elem_null(row, eo, j)) { st = RW_NULL; continue; }
        if (!rows_var_elem(row, eo, es, d2, j, fo, fs)) return RW_BAD;
        e2 += fs;
      }
    } else if (null_elem_is_error) {
      for (uint32_t j = 0; j < m; ++j) if (rows_elem_null(row, eo, j)) { st = RW_NULL; break; }
    }
  }
  c[1] = (uint32_t)e1;
  c[2] = (uint32_t)e2;
  room += 8ull * n + (var ? 8ull * e1 + e2 : e1 * esz);
  return st;
}

// A VectorUDT value (include/tfrgpu.h, VECTORS): the nested UnsafeRow struct<type: tinyint, size: int, indices: array<int>,
// values: array<double>> of `slot`.  Its dense length (`size` when sparse) and where its arrays' elements start, row-relative.
struct RowsVec {
  bool sparse;
  uint32_t n, size;             // values (and indices) elements; the dense length
  uint64_t vals, idx;
};
// RW_OK or RW_BAD (VectorUDT.deserialize and SparseVector's constructor would throw).  `check`: the indices are checked too
// (pass A); pass B reads only rows pass A found well-formed.
__device__ int rows_vector(const uint8_t* row, uint64_t len, uint64_t slot, bool check, RowsVec& v) {
  const uint64_t o = slot >> 32, sz = slot & 0xffffffffu;
  if ((o & 7) || o + sz > len || sz < 40) return RW_BAD;
  const uint64_t nulls = rows_ld64(row + o);
  const int8_t type = (int8_t)row[o + 8];                   // getByte(0), whatever its null bit
  if (type != 0 && type != 1) return RW_BAD;                // MatchError
  v.sparse = type == 0;
  uint64_t eo, es;
  if ((nulls >> 3) & 1 || !rows_var_elem(row, o, sz, o + 8, 3, eo, es) || !rows_array(row, eo, es, 8, v.n, v.vals)) return RW_BAD;
  if (!v.sparse) { v.size = v.n; return RW_OK; }
  const int32_t size = (int32_t)(uint32_t)rows_ld64(row + o + 16);      // getInt(1)
  uint32_t m;
  if (size < 0 || (nulls >> 2) & 1 || !rows_var_elem(row, o, sz, o + 8, 2, eo, es) || !rows_array(row, eo, es, 4, m, v.idx) || m != v.n)
    return RW_BAD;
  v.size = (uint32_t)size;
  if (check) {
    int64_t prev = -1;
    for (uint32_t i = 0; i < m; ++i) {
      const int32_t k = reinterpret_cast<const int32_t*>(row + v.idx)[i];
      if (k <= prev || k >= size) return RW_BAD;            // strictly increasing, inside [0, size)
      prev = k;
    }
  }
  return RW_OK;
}

// The counts of a field: a dense-format vector's level 0 is its dense length.  Its values go to an arena of their own, sized
// from the scanned counts, so they add nothing to `room`.  A sparse-format vector's toSparse entries are counted by pass A
// itself (rows_sparse_count); they number no more than its stored values, which `room` takes at 8 bytes each, so its values
// are bounded by the input like a double array's and its int32 indices by half of that (rows_layout sizes the arena so).
template <bool NW>
__device__ __forceinline__ int rows_counts(const RowsArgs& A, uint32_t f, const uint8_t* row, uint64_t len, const DevField& fd, uint64_t slot,
                                           uint32_t c[3], uint64_t& room, const int8_t* nar) {
  if (A.vec[f] == VK_NONE) return rows_field_counts<NW>(row, len, fd, slot, c, room, NW ? nar[f] : 0);
  RowsVec v;
  if (rows_vector(row, len, slot, true, v) != RW_OK) return RW_BAD;
  c[0] = v.size;
  if (A.vec[f] == VK_SPARSE) room += 8ull * v.n;
  return RW_OK;
}

// toSparse keeps the entries whose double is != 0.0: not +0.0 or -0.0 (a NaN is kept)
__device__ __forceinline__ bool rows_nz(uint64_t bits) { return (bits << 1) != 0; }
#define ROWS_VEC_WARP 64u
// The toSparse entries of a (well-formed) vector at `slot`, and the vector in v; warp-uniform call, `act`: this lane has one.
// A vector of ROWS_VEC_WARP stored values or more is counted by the whole warp (a dense 2^18-value one is not one lane's scan).
__device__ __forceinline__ uint32_t rows_sparse_count(const uint8_t* row, uint64_t slot, bool act, RowsVec& v) {
  const uint32_t lane = threadIdx.x & 31;
  v = RowsVec{};
  if (act) rows_vector(row, ~0ull, slot, false, v);
  const bool big = act && v.n >= ROWS_VEC_WARP;
  uint32_t k = 0;
  if (act && !big) for (uint32_t i = 0; i < v.n; ++i) k += rows_nz(rows_ld64(row + v.vals + 8ull * i)) ? 1u : 0u;
  uint32_t m = __ballot_sync(FULLMASK, big);
  while (m) {
    const int l = __ffs(m) - 1;
    m &= m - 1;
    const uint8_t* rw = (const uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)row, l);
    const uint32_t n = __shfl_sync(FULLMASK, v.n, l);
    const uint64_t vals = __shfl_sync(FULLMASK, v.vals, l);
    uint32_t t = 0;
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
      const uint32_t i = i0 + lane;
      t += __popc(__ballot_sync(FULLMASK, i < n && rows_nz(rows_ld64(rw + vals + 8ull * i))));
    }
    if (lane == (uint32_t)l) k = t;
  }
  return k;
}

__device__ __forceinline__ bool rows_field_null(const uint8_t* row, uint32_t f) { return (rows_ld64(row + 8ull * (f >> 6)) >> (f & 63)) & 1; }

// NW: the schema has a BooleanType .. DateType field (nar); NW = false is the kernel of every other schema and never reads nar.
template <bool NW>
__global__ void __launch_bounds__(ROWS_TILE) rows_pass_a_kernel(RowsArgs A, const int8_t* nar) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  uint8_t* tile_b = smem_raw + 16;
  const uint32_t lane = threadIdx.x;
  const uint32_t row0 = blockIdx.x * ROWS_TILE, rows = min((uint32_t)ROWS_TILE, A.n_rows - row0);
  const bool active = lane < rows;
  const uint32_t r = row0 + lane;
  int64_t lo = A.first, hi = A.first;
  if (active) { lo = A.offs[r]; hi = A.offs[r + 1]; }
  // ---- the tile's bytes -> shared memory ----
  const int64_t t_lo = A.offs[row0], t_hi = A.offs[row0 + rows];
  const bool staged = t_lo >= A.first && t_hi <= A.last && t_lo <= t_hi && ((t_lo | t_hi) & 7) == 0 && t_hi - t_lo + 32 <= (int64_t)A.smem_cap;
  const uintptr_t a_lo = reinterpret_cast<uintptr_t>(A.rows + (staged ? t_lo : 0)), a_hi = reinterpret_cast<uintptr_t>(A.rows + (staged ? t_hi : 0));
  const uintptr_t g_lo = a_lo & ~uintptr_t(15), b_lo = (a_lo + 15) & ~uintptr_t(15), b_hi = max(a_hi & ~uintptr_t(15), b_lo);
  if (staged) {
    if (lane == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      mbar_expect_tx(bar, (uint32_t)(b_hi - b_lo));
      if (b_hi > b_lo) bulk_g2s(tile_b + (b_lo - g_lo), reinterpret_cast<const void*>(b_lo), (uint32_t)(b_hi - b_lo), bar);
    } else if (lane == 1 && a_lo < min(b_lo, a_hi)) {      // an 8-byte head before the first whole 16-byte group
      *reinterpret_cast<unsigned long long*>(tile_b + (a_lo - g_lo)) = *reinterpret_cast<const unsigned long long*>(a_lo);
    } else if (lane == 2 && b_hi < a_hi) {                 // an 8-byte tail after the last one
      *reinterpret_cast<unsigned long long*>(tile_b + (b_hi - g_lo)) = *reinterpret_cast<const unsigned long long*>(b_hi);
    }
    __syncwarp();
    mbar_wait(bar, 0);
  }
  __syncwarp();
  const bool in_tile = staged && lo >= t_lo && hi <= t_hi;
  const uint8_t* row = in_tile ? tile_b + (reinterpret_cast<uintptr_t>(A.rows + lo) - g_lo) : A.rows + lo;

  // ---- validate ----
  const uint32_t nf = A.nu, nw = (nf + 63) / 64;
  bool bad = active && (lo < A.first || hi > A.last || lo > hi || ((lo | hi) & 7) || hi - lo < 8ll * (nw + nf));
  bool nul = false;
  const uint64_t len = (active && !bad) ? (uint64_t)(hi - lo) : 0;
  if (active && !bad) {
    uint64_t room = 0;
    for (uint32_t f = 0; f < nf; ++f) {
      const DevField& fd = A.sch.fields[f];
      if (fd.n_levels == 0 || rows_field_null(row, f)) continue;
      uint32_t c[3];
      const int st = rows_counts<NW>(A, f, row, len, fd, rows_ld64(row + 8ull * (nw + f)), c, room, nar);
      if (st == RW_BAD) { bad = true; break; }
      if (st == RW_NULL) nul = true;
    }
    if (room > len) bad = true;
  }
  const uint32_t mb = __ballot_sync(FULLMASK, bad), mn = __ballot_sync(FULLMASK, nul && !bad);
  if (mb && lane == (uint32_t)__ffs(mb) - 1) atomicMin(&A.st->rows_first_bad, r);
  if (mn && lane == (uint32_t)__ffs(mn) - 1) atomicMin(&A.st->rows_first_null, r);
  const bool ok = active && !bad && !nul;

  // ---- columns ----
  for (uint32_t f = 0; f < nf; ++f) {
    const DevField& fd = A.sch.fields[f];
    const bool present = ok && fd.elem_type != TFR_T_NULL && !rows_field_null(row, f);
    const uint32_t vb = __ballot_sync(FULLMASK, present);
    if (lane == 0) A.valid[(size_t)f * A.vwords + blockIdx.x] = vb;
    if (A.vec[f] == VK_SPARSE) {                            // its values, and its parts: the indices (as many) and the size
      RowsVec v;
      const uint32_t k = rows_sparse_count(row, present ? rows_ld64(row + 8ull * (nw + f)) : 0, present, v);
      const int32_t pi = A.part[f];
      if (lane == 0) A.valid[(size_t)pi * A.vwords + blockIdx.x] = A.valid[(size_t)(pi + 1) * A.vwords + blockIdx.x] = vb;
      if (!active) continue;
      A.cnt[(size_t)fd.cnt_slot * A.n_rows + r] = k;
      A.cnt[(size_t)A.sch.fields[pi].cnt_slot * A.n_rows + r] = k;
      reinterpret_cast<uint32_t*>(A.fixv[pi + 1])[r] = present ? v.size : 0u;
      continue;
    }
    if (!active || fd.elem_type == TFR_T_NULL) continue;
    if (fd.n_levels == 0) {
      const uint64_t s = present ? rows_ld64(row + 8ull * (nw + f)) : 0;
      void* v = A.fixv[f];
      if (NW && nar[f]) { reinterpret_cast<long long*>(v)[r] = rows_widen(nar[f], s); continue; }   // a null's 0 widens to 0
      if (fd.width == 4) reinterpret_cast<uint32_t*>(v)[r] = (uint32_t)s;                      // IntegerType / FloatType: the low 4 bytes
      else if (fd.elem_type == TFR_T_DECIMAL)                                                    // BigDecimal(v, 0).floatValue, carried as float64
        reinterpret_cast<double*>(v)[r] = present ? (double)__ll2float_rn((long long)s) : 0.0;
      else reinterpret_cast<unsigned long long*>(v)[r] = s;
      continue;
    }
    uint32_t c[3] = {0, 0, 0};
    uint64_t room = 0;
    if (present) rows_counts<NW>(A, f, row, len, fd, rows_ld64(row + 8ull * (nw + f)), c, room, nar);
    for (int l = 0; l < fd.n_levels; ++l) A.cnt[(size_t)(fd.cnt_slot + l) * A.n_rows + r] = c[l];
  }
}

// Places the inner offsets levels and the values of every variable-width column in the two arenas, in schema order, and
// writes the last entry of each inner level.  The arenas are sized from the input (values <= its bytes, inner entries <=
// its bytes / 8, per-row `room` check of pass A), which holds when the offsets are non-decreasing.  Offsets that go down
// and back up can make well-formed rows overlap and the totals exceed the arenas (or int32): then the overflow flag is
// raised and every variable column becomes all-null AND empty -- validity and level-0 offsets all zero -- so that no
// kernel, including the ByteArray one that reads only the offsets, touches the unplaced buffers; the host reports the
// malformed row.  Every block recomputes the totals; block 0 writes.
// Vector fields (dense lengths, which the input does not bound) go to their own arena `xarena` (xcap bytes), sized by the host
// from the scanned counts (rows_vec_bytes).  Block 0 stores their values' total in rows_vec_lo / hi.  A pipelined batch sizes
// that arena from what the encoder learned: a batch it is too small for raises the overflow flag, which the encode's verdict
// turns into a redo (EVF_ROWS), and the synchronous path then sizes it from the counts.
__host__ __device__ __forceinline__ unsigned long long rows_vec_place(unsigned long long xpos, unsigned long long values) {
  return ((xpos + 15) & ~15ull) + values * 8ull;
}
__global__ void rows_layout_kernel(RowsArgs A, const unsigned long long* __restrict__ totals, uint8_t* varena, unsigned long long vcap,
                                   int32_t* iarena, unsigned long long icap, uint8_t* xarena, unsigned long long xcap) {
  __shared__ uint32_t over;
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  if (threadIdx.x == 0) {
    unsigned long long vpos = 0, ipos = 0, xpos = 0, xn = 0;
    for (uint32_t f = 0; f < nf; ++f) {
      const DevField& fd = A.sch.fields[f];
      if (fd.n_levels == 0) continue;
      if (A.vec[f] == VK_DENSE) { xpos = rows_vec_place(xpos, totals[fd.cnt_slot]); xn += totals[fd.cnt_slot]; continue; }
      for (int l = 1; l < fd.n_levels; ++l) ipos += totals[fd.cnt_slot + l - 1] + 1;
      vpos = ((vpos + 15) & ~15ull) + totals[fd.cnt_slot + fd.n_levels - 1] * (unsigned long long)fd.width;
    }
    over = (A.st->rows_overflow != 0 || vpos > vcap || ipos > icap || xpos > xcap) ? 1u : 0u;
    if (blockIdx.x == 0) { A.st->rows_vec_lo = (uint32_t)xn; A.st->rows_vec_hi = (uint32_t)(xn >> 32); }
    if (!over && blockIdx.x == 0) {
      vpos = ipos = xpos = 0;
      for (uint32_t f = 0; f < nf; ++f) {
        const DevField& fd = A.sch.fields[f];
        if (fd.n_levels == 0) continue;
        if (A.vec[f] == VK_DENSE) {
          xpos = (xpos + 15) & ~15ull;
          A.cols[f].values = xarena + xpos;
          xpos = rows_vec_place(xpos, totals[fd.cnt_slot]);
          continue;
        }
        for (int l = 1; l < fd.n_levels; ++l) {
          int32_t* o = iarena + ipos;
          const unsigned long long parents = totals[fd.cnt_slot + l - 1];
          o[parents] = (int32_t)totals[fd.cnt_slot + l];
          A.cols[f].off[l] = o;
          ipos += parents + 1;
        }
        vpos = (vpos + 15) & ~15ull;
        A.cols[f].values = varena + vpos;
        vpos += totals[fd.cnt_slot + fd.n_levels - 1] * (unsigned long long)fd.width;
      }
    }
    if (over && blockIdx.x == 0) A.st->rows_overflow = 1;
  }
  __syncthreads();
  if (!over) return;
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = t0; i < (size_t)nf * A.vwords; i += stride)
    if (A.sch.fields[i / A.vwords].n_levels) A.valid[i] = 0;
  for (uint32_t f = 0; f < nf; ++f) {
    const DevField& fd = A.sch.fields[f];
    if (fd.n_levels == 0) continue;
    int32_t* o0 = A.lev[fd.cnt_slot];
    for (size_t i = t0; i <= A.n_rows; i += stride) o0[i] = 0;
  }
}

// n bytes from an 8-byte aligned source (whose 8-byte words all lie in the row) to any destination
__device__ __forceinline__ void rows_copy_lane(uint8_t* dst, const uint8_t* src, uint32_t n) {
  const bool al = (reinterpret_cast<uintptr_t>(dst) & 7) == 0;
  for (uint32_t k = 0; k < n; k += 8) {
    uint64_t w = rows_ld64(src + k);
    if (al && k + 8 <= n) { *reinterpret_cast<unsigned long long*>(dst + k) = w; continue; }
    for (uint32_t j = 0; j < 8 && k + j < n; ++j, w >>= 8) dst[k + j] = (uint8_t)w;
  }
}
// warp-uniform call: short runs are copied by their lane, long ones by the whole warp in turn
__device__ __forceinline__ void rows_copy(uint8_t* dst, const uint8_t* src, uint32_t n, bool act) {
  const uint32_t lane = threadIdx.x & 31;
  const bool big = act && n >= 256;
  if (act && !big) rows_copy_lane(dst, src, n);
  uint32_t m = __ballot_sync(FULLMASK, big);
  while (m) {
    const int l = __ffs(m) - 1;
    m &= m - 1;
    uint8_t* d = (uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)dst, l);
    const uint8_t* s = (const uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)src, l);
    const uint32_t k = __shfl_sync(FULLMASK, n, l);
    for (uint32_t o = lane * 64; o < k; o += 32 * 64) rows_copy_lane(d + o, s + o, min(64u, k - o));
  }
}
// numeric elements [i0, i0 + m) of the array whose slots start at row byte d -> column values from index `at`.  NW: nt is an INT64
// TYPES field's TFR_T_* (0 none), whose elements widen into the int64 column (a null element: its slot's bits, as LongType's).
template <bool NW>
__device__ __forceinline__ void rows_copy_elems(const DevField& fd, void* values, uint64_t at, const uint8_t* row, uint64_t d, uint32_t m, int nt) {
  if (NW && nt) {
    long long* v = reinterpret_cast<long long*>(values) + at;
    for (uint32_t i = 0; i < m; ++i) v[i] = rows_widen(nt, rows_narrow_elem(row, d, nt, i));
  } else if (fd.width == 4) {
    uint32_t* v = reinterpret_cast<uint32_t*>(values) + at;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(row + d);
    for (uint32_t i = 0; i < m; ++i) v[i] = s[i];                    // a null element keeps its slot's bits (toIntArray / toFloatArray)
  } else if (fd.elem_type == TFR_T_DECIMAL) {
    double* v = reinterpret_cast<double*>(values) + at;
    for (uint32_t i = 0; i < m; ++i) v[i] = (double)__ll2float_rn((long long)rows_ld64(row + d + 8ull * i));
  } else {
    unsigned long long* v = reinterpret_cast<unsigned long long*>(values) + at;
    for (uint32_t i = 0; i < m; ++i) v[i] = rows_ld64(row + d + 8ull * i);
  }
}

// A vector's dense values (toArray) from index 0 of `out`; warp-uniform call, `act`: this lane has a (well-formed) vector.
// Dense: its lane copies the values, like a double array.  Sparse: a zero-fill of the dense range, then the scatter of the
// non-zeros; a range of ROWS_VEC_WARP values or more is filled and scattered by the whole warp (HashingTF's are 2^18 long).
__device__ __forceinline__ void rows_vector_fill(const uint8_t* row, uint64_t slot, unsigned long long* out, bool act) {
  const uint32_t lane = threadIdx.x & 31;
  RowsVec v{};
  if (act) rows_vector(row, ~0ull, slot, false, v);
  const bool big = act && v.sparse && v.size >= ROWS_VEC_WARP;
  if (act && !big) {
    if (v.sparse) for (uint32_t i = 0; i < v.size; ++i) out[i] = 0;
    for (uint32_t i = 0; i < v.n; ++i) {
      const uint32_t k = v.sparse ? (uint32_t)reinterpret_cast<const int32_t*>(row + v.idx)[i] : i;
      out[k] = rows_ld64(row + v.vals + 8ull * i);        // a null element keeps its slot's bits (toDoubleArray)
    }
  }
  uint32_t m = __ballot_sync(FULLMASK, big);
  while (m) {
    const int l = __ffs(m) - 1;
    m &= m - 1;
    unsigned long long* o = (unsigned long long*)__shfl_sync(FULLMASK, (unsigned long long)out, l);
    const uint8_t* rw = (const uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)row, l);
    const uint32_t size = __shfl_sync(FULLMASK, v.size, l), n = __shfl_sync(FULLMASK, v.n, l);
    const uint64_t vals = __shfl_sync(FULLMASK, v.vals, l), idx = __shfl_sync(FULLMASK, v.idx, l);
    for (uint32_t k = lane; k < size; k += 32) o[k] = 0;
    __syncwarp();                                           // (orders the zeros before the scatter)
    for (uint32_t i = lane; i < n; i += 32) o[reinterpret_cast<const int32_t*>(rw + idx)[i]] = rows_ld64(rw + vals + 8ull * i);
    __syncwarp();
  }
}

// A vector's toSparse (rows_sparse_count's entries): its values to `ov` and their indices to `oi`, from index 0, in index
// order; warp-uniform call, `act`: this lane has a (well-formed) vector.  ROWS_VEC_WARP stored values or more: the whole warp
// compacts 32 at a time, each entry placed by the ballot's population below its lane.
__device__ __forceinline__ void rows_sparse_fill(const uint8_t* row, uint64_t slot, unsigned long long* ov, int32_t* oi, bool act) {
  const uint32_t lane = threadIdx.x & 31;
  RowsVec v{};
  if (act) rows_vector(row, ~0ull, slot, false, v);
  const bool big = act && v.n >= ROWS_VEC_WARP;
  if (act && !big) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < v.n; ++i) {
      const uint64_t x = rows_ld64(row + v.vals + 8ull * i);
      if (!rows_nz(x)) continue;
      ov[k] = x;
      oi[k++] = v.sparse ? reinterpret_cast<const int32_t*>(row + v.idx)[i] : (int32_t)i;
    }
  }
  uint32_t m = __ballot_sync(FULLMASK, big);
  while (m) {
    const int l = __ffs(m) - 1;
    m &= m - 1;
    unsigned long long* o = (unsigned long long*)__shfl_sync(FULLMASK, (unsigned long long)ov, l);
    int32_t* q = (int32_t*)__shfl_sync(FULLMASK, (unsigned long long)oi, l);
    const uint8_t* rw = (const uint8_t*)__shfl_sync(FULLMASK, (unsigned long long)row, l);
    const uint32_t n = __shfl_sync(FULLMASK, v.n, l);
    const bool sp = __shfl_sync(FULLMASK, v.sparse ? 1 : 0, l) != 0;
    const uint64_t vals = __shfl_sync(FULLMASK, v.vals, l), idx = __shfl_sync(FULLMASK, v.idx, l);
    uint32_t base = 0;
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
      const uint32_t i = i0 + lane;
      const uint64_t x = i < n ? rows_ld64(rw + vals + 8ull * i) : 0;
      const uint32_t b = __ballot_sync(FULLMASK, rows_nz(x));
      if (rows_nz(x)) {
        const uint32_t p = base + __popc(b & ((1u << lane) - 1));
        o[p] = x;
        q[p] = sp ? reinterpret_cast<const int32_t*>(rw + idx)[i] : (int32_t)i;
      }
      base += __popc(b);
    }
  }
}

template <bool NW>
__global__ void __launch_bounds__(ROWS_B_WARPS * 32) rows_pass_b_kernel(RowsArgs A, const int8_t* nar) {
  if (A.st->rows_overflow) return;                                   // the columns were not placed: nothing to fill
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t w = blockIdx.x * ROWS_B_WARPS + (threadIdx.x >> 5);
  const uint32_t r = w * 32 + lane;
  if (w * 32 >= A.n_rows) return;                            // warp-uniform
  const bool active = r < A.n_rows;
  const uint32_t nf = A.nu, nw = (nf + 63) / 64;
  const uint8_t* row = A.rows + (active ? A.offs[r] : A.first);
  for (uint32_t f = 0; f < nf; ++f) {
    const DevField& fd = A.sch.fields[f];
    if (fd.n_levels == 0) continue;
    // validity is set only for well-formed rows without null elements: only those are read
    const bool v = active && ((A.valid[(size_t)f * A.vwords + w] >> lane) & 1);
    const EncCol& c = A.cols[f];
    uint8_t* values = (uint8_t*)c.values;
    const uint64_t slot = v ? rows_ld64(row + 8ull * (nw + f)) : 0;
    const uint64_t o = slot >> 32, sz = slot & 0xffffffffu;
    const int32_t e0 = v ? A.lev[fd.cnt_slot][r] : 0;
    if (A.vec[f] == VK_DENSE) { rows_vector_fill(row, slot, reinterpret_cast<unsigned long long*>(values) + e0, v); continue; }
    if (A.vec[f] == VK_SPARSE) {
      rows_sparse_fill(row, slot, reinterpret_cast<unsigned long long*>(values) + e0, (int32_t*)A.cols[A.part[f]].values + e0, v);
      continue;
    }
    if (fd.depth == 0) { rows_copy(values + e0, row + o, (uint32_t)sz, v); continue; }
    if (!v) continue;
    const bool var = rows_is_var(fd);
    const int nt = NW ? nar[f] : 0;
    const uint32_t esz = var ? 8u : NW && nt ? (uint32_t)nar_width(nt) : (uint32_t)fd.width;
    uint32_t n;
    uint64_t d, eo, es;
    rows_array(row, o, sz, fd.depth == 2 ? 8u : esz, n, d);
    if (fd.depth == 1) {
      if (!var) { rows_copy_elems<NW>(fd, values, (uint64_t)e0, row, d, n, nt); continue; }
      int32_t* o1 = const_cast<int32_t*>(c.off[1]);
      int32_t b = A.lev[fd.cnt_slot + 1][r];
      for (uint32_t i = 0; i < n; ++i) {
        rows_var_elem(row, o, sz, d, i, eo, es);
        o1[e0 + i] = b;
        rows_copy_lane(values + b, row + eo, (uint32_t)es);
        b += (int32_t)es;
      }
      continue;
    }
    int32_t* o1 = const_cast<int32_t*>(c.off[1]);
    int32_t* o2 = var ? const_cast<int32_t*>(c.off[2]) : nullptr;
    int32_t b1 = A.lev[fd.cnt_slot + 1][r];
    int32_t b2 = var ? A.lev[fd.cnt_slot + 2][r] : 0;
    for (uint32_t s = 0; s < n; ++s) {
      o1[e0 + s] = b1;
      rows_var_elem(row, o, sz, d, s, eo, es);
      uint32_t m;
      uint64_t d2, fo, fs;
      rows_array(row, eo, es, esz, m, d2);
      if (!var) { rows_copy_elems<NW>(fd, values, (uint64_t)b1, row, d2, m, nt); b1 += (int32_t)m; continue; }
      for (uint32_t j = 0; j < m; ++j) {
        rows_var_elem(row, eo, es, d2, j, fo, fs);
        o2[b1 + j] = b2;
        rows_copy_lane(values + b2, row + fo, (uint32_t)fs);
        b2 += (int32_t)fs;
      }
      b1 += (int32_t)m;
    }
  }
}
