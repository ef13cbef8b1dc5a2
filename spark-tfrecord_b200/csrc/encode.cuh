// encode.cuh -- K5: Arrow-layout columns -> protobuf wire bytes -> CRC-32C framing, the mirror of decode.
//
// Replaces, per row, serializeExample / serializeSequenceExample (M/TFRecordSerializer.scala:20-60, feature
// construction :68-207), Example.toByteArray (M/TFRecordOutputWriter.scala:31,33) and TFRecordWriter.write
// (:37).  Output bytes are identical to the reference writer's: map entries in schema order (protobuf-java
// keeps insertion order), nulls omitted, key then value inside each entry, packed lists, the `features` /
// `context` / `feature_lists` wrappers always present.
//
//   encode_size_kernel : one warp per row, one lane per field: nested protobuf sizes bottom-up
//                        (values -> list -> Feature -> entry), entry offsets inside the record by a
//                        warp prefix sum, record size = 16 + payload.
//   (scan.cuh)         : record sizes -> byte offset of every record in the output.
//   encode_emit_kernel : same mapping, each lane writes its entry; then the warp computes the masked
//                        CRC-32C of the payload it just wrote and lane 0 writes header and footer.
#pragma once
#include "common.cuh"

struct EncCol {                 // one input column (device pointers)
  const uint8_t* validity;      // Arrow bitmap or nullptr (all valid)
  const int32_t* off[3];
  const void* values;
};

// The encoder's status block: one per set of encode buffers on the device, mirrored in pinned host memory.  The size
// kernels, the row kernels (rows.cuh), encode_bytes_kernel and encode_verdict_kernel report through it, and the host
// reads a batch's errors, total and launch figures from the mirror.  0xffffffff in a "first row" word: no such row.
struct EncStatus {
  uint32_t first_null_row;      // atomicMin: first row with a null in a non-nullable column
  uint32_t overflow;            // the record-size scan passed 32 bits, or encode_bytes_kernel met a payload or offsets it cannot place
  uint32_t total_lo, total_hi;  // encode_bytes_kernel: the batch's framed bytes
  uint32_t max_word;            // atomicMax: largest framed record (Example, SequenceExample) or longest payload (ByteArray)
  uint32_t pad0[3];
  uint32_t rows_first_bad;      // row kernels, atomicMin: first malformed row
  uint32_t rows_first_null;     // row kernels, atomicMin: first row with a null element
  uint32_t rows_overflow;       // row kernels: a scan of counts overflowed or an arena is too small
  uint32_t rows_vec_lo, rows_vec_hi;   // rows_layout_kernel: the dense values of the batch's vector fields
  uint32_t pad1[3];
  uint32_t verdict_flag;        // encode_verdict_kernel: EVF_* (0: the batch can be emitted as launched)
  uint32_t verdict_total_lo, verdict_total_hi;   // and the batch's framed bytes
  uint32_t pad2[13];
  uint64_t total() const { return total_lo | (uint64_t)total_hi << 32; }
  uint64_t verdict_total() const { return verdict_total_lo | (uint64_t)verdict_total_hi << 32; }
  uint64_t rows_vec() const { return rows_vec_lo | (uint64_t)rows_vec_hi << 32; }
};
static_assert(sizeof(EncStatus) == 128, "the status block is copied whole");
static_assert(offsetof(EncStatus, total_lo) % 8 == 0, "the host copies a 64-bit scan total onto total_lo / total_hi");
static_assert(offsetof(EncStatus, rows_overflow) == offsetof(EncStatus, rows_first_bad) + 8, "the row kernels' words are set and copied as a group");

struct EncodeArgs {
  DevSchema sch;
  const EncCol* cols;           // [n_fields]
  uint32_t n_rows;
  const CrcTables* tabs;
  uint32_t* rec_size;           // [n_rows] framed size of each record
  uint32_t* cell_size;          // [n_fields][n_rows] size of the map-entry VALUE (Feature / FeatureList bytes)
  EncStatus* st;                // (sizes) first_null_row, max_word
  const int32_t* rec_off;       // [n_rows+1] (emit)
  uint8_t* out;                 // (emit)
};

__device__ __forceinline__ uint32_t vsize32(uint32_t v) { return v < 0x80 ? 1 : v < 0x4000 ? 2 : v < 0x200000 ? 3 : v < 0x10000000 ? 4 : 5; }
__device__ __forceinline__ uint32_t vsize64(uint64_t v) { return v == 0 ? 1u : (uint32_t)((63 - __clzll((long long)v)) / 7 + 1); }
__device__ __forceinline__ uint8_t* put_varint(uint8_t* p, uint64_t v) {
  while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; }
  *p++ = (uint8_t)v;
  return p;
}
__device__ __forceinline__ bool enc_valid(const EncCol& c, uint32_t row) { return !c.validity || ((c.validity[row >> 3] >> (row & 7)) & 1); }

// Double.toFloat: IEEE round-to-nearest-even narrowing; NaN keeps sign + the top payload bits and is quieted
// (what the JVM's d2f / x86 cvtsd2ss produce)
__device__ __forceinline__ uint32_t double_to_float_bits(double d) {
  if (d != d) {
    uint64_t b = (uint64_t)__double_as_longlong(d);
    return (uint32_t)((b >> 32) & 0x80000000u) | 0x7fc00000u | (uint32_t)((b >> 29) & 0x3fffffu);
  }
  return __float_as_uint(__double2float_rn(d));
}

// size of the list message body built from leaf elements [lo, hi) of column c
__device__ __forceinline__ uint32_t list_body_size(const DevField& fd, const EncCol& c, int32_t lo, int32_t hi) {
  uint32_t n = (uint32_t)(hi - lo);
  if (n == 0) return 0;
  if (fd.kind == K_INT64) {
    uint32_t pb = 0;
    if (fd.elem_type == TFR_T_INT32) { const int32_t* v = (const int32_t*)c.values; for (int32_t i = lo; i < hi; ++i) pb += vsize64((uint64_t)(int64_t)v[i]); }
    else { const int64_t* v = (const int64_t*)c.values; for (int32_t i = lo; i < hi; ++i) pb += vsize64((uint64_t)v[i]); }
    return 1 + vsize32(pb) + pb;
  }
  if (fd.kind == K_FLOAT) return 1 + vsize32(4 * n) + 4 * n;
  const int32_t* so = c.off[fd.n_levels - 1];
  uint32_t s = 0;
  for (int32_t i = lo; i < hi; ++i) { uint32_t l = (uint32_t)(so[i + 1] - so[i]); s += 1 + vsize32(l) + l; }
  return s;
}
// Feature message = oneof member tag + len + list body
__device__ __forceinline__ uint32_t feature_size(const DevField& fd, const EncCol& c, int32_t lo, int32_t hi) {
  uint32_t L = list_body_size(fd, c, lo, hi);
  return 1 + vsize32(L) + L;
}
__device__ __forceinline__ uint8_t* emit_list_body(uint8_t* p, const DevField& fd, const EncCol& c, int32_t lo, int32_t hi) {
  uint32_t n = (uint32_t)(hi - lo);
  if (n == 0) return p;
  if (fd.kind == K_INT64) {
    uint32_t pb = 0;
    if (fd.elem_type == TFR_T_INT32) { const int32_t* v = (const int32_t*)c.values; for (int32_t i = lo; i < hi; ++i) pb += vsize64((uint64_t)(int64_t)v[i]); }
    else { const int64_t* v = (const int64_t*)c.values; for (int32_t i = lo; i < hi; ++i) pb += vsize64((uint64_t)v[i]); }
    *p++ = 0x0A; p = put_varint(p, pb);
    if (fd.elem_type == TFR_T_INT32) { const int32_t* v = (const int32_t*)c.values; for (int32_t i = lo; i < hi; ++i) p = put_varint(p, (uint64_t)(int64_t)v[i]); }   // .toLong sign-extends (:74,104)
    else { const int64_t* v = (const int64_t*)c.values; for (int32_t i = lo; i < hi; ++i) p = put_varint(p, (uint64_t)v[i]); }
    return p;
  }
  if (fd.kind == K_FLOAT) {
    *p++ = 0x0A; p = put_varint(p, 4ull * n);
    const bool aligned = (reinterpret_cast<uintptr_t>(p) & 3u) == 0;            // whole-word stores when the packed floats happen to start on a word
    for (int32_t i = lo; i < hi; ++i) {
      uint32_t b = fd.elem_type == TFR_T_FLOAT32 ? ((const uint32_t*)c.values)[i] : double_to_float_bits(((const double*)c.values)[i]);   // toFloat (:86,113)
      if (aligned) *reinterpret_cast<uint32_t*>(p) = b;
      else { p[0] = (uint8_t)b; p[1] = (uint8_t)(b >> 8); p[2] = (uint8_t)(b >> 16); p[3] = (uint8_t)(b >> 24); }
      p += 4;
    }
    return p;
  }
  const int32_t* so = c.off[fd.n_levels - 1];
  const uint8_t* data = (const uint8_t*)c.values;
  for (int32_t i = lo; i < hi; ++i) {
    uint32_t l = (uint32_t)(so[i + 1] - so[i]);
    *p++ = 0x0A; p = put_varint(p, l);
    const uint8_t* s = data + so[i];
    uint32_t k = 0;
    if ((reinterpret_cast<uintptr_t>(s) & 3u) == 0) {                           // word loads from the column, bytes (or words) into the record
      const bool pal = (reinterpret_cast<uintptr_t>(p) & 3u) == 0;
      for (; k + 4 <= l; k += 4) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(s + k);
        if (pal) *reinterpret_cast<uint32_t*>(p + k) = w;
        else { p[k] = (uint8_t)w; p[k + 1] = (uint8_t)(w >> 8); p[k + 2] = (uint8_t)(w >> 16); p[k + 3] = (uint8_t)(w >> 24); }
      }
    }
    for (; k < l; ++k) p[k] = s[k];
    p += l;
  }
  return p;
}
__device__ __forceinline__ uint8_t* emit_feature(uint8_t* p, const DevField& fd, const EncCol& c, int32_t lo, int32_t hi) {
  uint32_t L = list_body_size(fd, c, lo, hi);
  *p++ = fd.kind == K_BYTES ? 0x0A : fd.kind == K_FLOAT ? 0x12 : 0x1A;
  p = put_varint(p, L);
  return emit_list_body(p, fd, c, lo, hi);
}

// value size of field f at `row` (Feature, or FeatureList for depth 2); 0xffffffff = null
__device__ __forceinline__ uint32_t cell_value_size(const DevField& fd, const EncCol& c, uint32_t row) {
  if (fd.elem_type == TFR_T_NULL || !enc_valid(c, row)) return 0xffffffffu;
  if (fd.depth == 0) return feature_size(fd, c, (int32_t)row, (int32_t)row + 1);
  const int32_t* o0 = c.off[0];
  if (fd.depth == 1) return feature_size(fd, c, o0[row], o0[row + 1]);
  const int32_t* o1 = c.off[1];
  uint32_t v = 0;
  for (int32_t s = o0[row]; s < o0[row + 1]; ++s) { uint32_t F = feature_size(fd, c, o1[s], o1[s + 1]); v += 1 + vsize32(F) + F; }
  return v;
}
__device__ __forceinline__ uint32_t entry_total(const DevField& fd, uint32_t V) {
  uint32_t E = 1 + vsize32(fd.name_len) + fd.name_len + 1 + vsize32(V) + V;
  return 1 + vsize32(E) + E;
}

// warp-wide exclusive prefix over lanes
__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
  total = __shfl_sync(FULLMASK, x, 31);
  return x - v;
}

// mode 0: sizes; mode 1: emit
// GUARD (MODE 1 only): the pipelined encoder's emit (api_encode.inc), which returns at once when encode_verdict_kernel (below)
// has raised *flag.  GUARD = false never reads `flag`.
template <int MODE, bool GUARD>
__global__ void __launch_bounds__(256) encode_kernel(EncodeArgs A, const uint32_t* __restrict__ flag) {
  if (GUARD && *flag) return;
  extern __shared__ uint32_t smem[];
  uint32_t* stab = smem;
  if (MODE == 1) { crc_stage_tables(stab, A.tabs); __syncthreads(); }
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  const bool seq = A.sch.record_type == TFR_RT_SEQUENCE_EXAMPLE;
  for (uint32_t row = blockIdx.x * warps + wid; row < A.n_rows; row += gridDim.x * warps) {
    if (A.sch.record_type == TFR_RT_BYTE_ARRAY) {               // serializeByteArray (:16-18)
      const EncCol& c = A.cols[0];
      uint32_t lo = (uint32_t)c.off[0][row], len = (uint32_t)c.off[0][row + 1] - lo;
      if (MODE == 0) { if (lane == 0) A.rec_size[row] = 16 + len; continue; }
      uint8_t* rec = A.out + A.rec_off[row];
      const uint8_t* s = (const uint8_t*)c.values + lo;
      for (uint32_t i = lane; i < len; i += 32) rec[12 + i] = s[i];
      __syncwarp();
      __threadfence_block();
      uint32_t crc = crc_mask(crc_warp(stab, rec + 12, len));
      if (lane == 0) {
        for (int i = 0; i < 4; ++i) { rec[i] = (uint8_t)(len >> (8 * i)); rec[4 + i] = 0; }
        uint32_t hc = crc_mask(crc_u64(CRC_T0(stab), len, 0));
        for (int i = 0; i < 4; ++i) { rec[8 + i] = (uint8_t)(hc >> (8 * i)); rec[12 + len + i] = (uint8_t)(crc >> (8 * i)); }
      }
      continue;
    }
    // pass over the fields in schema order, 32 at a time; group 0 = context/features, group 1 = feature_lists
    uint32_t gsize[2] = {0, 0};
    bool null_err = false;
    for (int pass = 0; pass < 2; ++pass) {
      // pass 0 computes the two group sizes; pass 1 (emit only) writes at the now known offsets
      uint32_t gpos[2] = {0, 0};
      uint8_t* payload = nullptr;
      uint32_t ctx_hdr = 0, fl_hdr = 0;
      if (pass == 1) {
        if (MODE == 0) break;
        payload = A.out + A.rec_off[row] + 12;
        ctx_hdr = 1 + vsize32(gsize[0]);
        fl_hdr = 1 + vsize32(gsize[1]);
      }
      for (uint32_t f0 = 0; f0 < nf; f0 += 32) {
        uint32_t f = f0 + lane;
        uint32_t V = 0xffffffffu, tot = 0;
        int grp = 0;
        if (f < nf) {
          const DevField& fd = A.sch.fields[f];
          grp = (seq && fd.depth == 2) ? 1 : 0;
          if (MODE == 0) {
            V = cell_value_size(fd, A.cols[f], row);
            A.cell_size[(size_t)f * A.n_rows + row] = V;
            if (V == 0xffffffffu && !fd.nullable) null_err = true;      // NullPointerException (:29-31,53-55)
          } else V = A.cell_size[(size_t)f * A.n_rows + row];
          if (V != 0xffffffffu) tot = entry_total(fd, V);
        }
        uint32_t t0, t1;
        uint32_t e0 = warp_excl_scan(grp == 0 ? tot : 0, t0);
        uint32_t e1 = warp_excl_scan(grp == 1 ? tot : 0, t1);
        if (pass == 1 && tot) {
          const DevField& fd = A.sch.fields[f];
          const EncCol& c = A.cols[f];
          uint8_t* p = payload + (grp == 0 ? ctx_hdr + gpos[0] + e0 : ctx_hdr + gsize[0] + fl_hdr + gpos[1] + e1);
          uint32_t E = 1 + vsize32(fd.name_len) + fd.name_len + 1 + vsize32(V) + V;
          *p++ = 0x0A; p = put_varint(p, E);
          *p++ = 0x0A; p = put_varint(p, fd.name_len);
          const uint8_t* nm = A.sch.names + fd.name_off;
          for (uint32_t k = 0; k < fd.name_len; ++k) p[k] = nm[k];
          p += fd.name_len;
          *p++ = 0x12; p = put_varint(p, V);
          if (fd.depth == 0) p = emit_feature(p, fd, c, (int32_t)row, (int32_t)row + 1);
          else if (fd.depth == 1) p = emit_feature(p, fd, c, c.off[0][row], c.off[0][row + 1]);
          else {
            const int32_t* o0 = c.off[0]; const int32_t* o1 = c.off[1];
            for (int32_t s = o0[row]; s < o0[row + 1]; ++s) {
              uint32_t F = feature_size(fd, c, o1[s], o1[s + 1]);
              *p++ = 0x0A; p = put_varint(p, F);
              p = emit_feature(p, fd, c, o1[s], o1[s + 1]);
            }
          }
        }
        gpos[0] += t0; gpos[1] += t1;
      }
      if (pass == 0) { gsize[0] = gpos[0]; gsize[1] = gpos[1]; }
    }
    uint32_t plen = 1 + vsize32(gsize[0]) + gsize[0] + (seq ? 1 + vsize32(gsize[1]) + gsize[1] : 0);
    if (MODE == 0) {
      if (__any_sync(FULLMASK, null_err) && lane == 0) atomicMin(&A.st->first_null_row, row);
      if (lane == 0) { A.rec_size[row] = 16 + plen; atomicMax(&A.st->max_word, 16 + plen); }
      continue;
    }
    uint8_t* rec = A.out + A.rec_off[row];
    if (lane == 0) {        // wrappers: setFeatures / setContext + setFeatureLists are always called (:33,57-58)
      uint8_t* p = rec + 12;
      *p++ = 0x0A; p = put_varint(p, gsize[0]);
      if (seq) { p += gsize[0]; *p++ = 0x12; put_varint(p, gsize[1]); }
    }
    __syncwarp();
    __threadfence_block();
    uint32_t crc = crc_mask(crc_warp(stab, rec + 12, plen));
    if (lane == 0) {
      for (int i = 0; i < 4; ++i) { rec[i] = (uint8_t)(plen >> (8 * i)); rec[4 + i] = 0; }
      uint32_t hc = crc_mask(crc_u64(CRC_T0(stab), plen, 0));
      for (int i = 0; i < 4; ++i) { rec[8 + i] = (uint8_t)(hc >> (8 * i)); rec[12 + plen + i] = (uint8_t)(crc >> (8 * i)); }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Verdict of a pipelined encode (api_encode.inc, tfr_encode_rows_submit).  Its outputs were sized from what the encoder
// learned on earlier batches, not from this batch's sizes; one thread checks them after the record-size scan and raises
// EncStatus::verdict_flag when the batch cannot be emitted as launched.  The guarded emit kernels read that word first, so
// a flagged batch writes nothing; the host redoes it through the synchronous path.  The total goes to the verdict too.
// ---------------------------------------------------------------------------------------------
enum { EVF_CAPACITY = 1, EVF_SLOT = 2, EVF_STRIDE = 4, EVF_ROWS = 8, EVF_NULL = 16 };
struct EncVerdictArgs {
  EncStatus* st;
  const unsigned long long* total;       // Example / SequenceExample: the scan's grand total
  const int32_t* bytes_offs;             // ByteArray: the column's offsets (total = offs[n] - offs[0] + 16 n); null otherwise
  uint32_t n_rows;
  unsigned long long cap;                // bytes of the output block
  uint32_t max_rec;                      // largest framed record the tile slot holds (0: the general emit kernel, no limit)
  uint32_t max_len;                      // ByteArray: largest payload the launched stride holds
};
__global__ void encode_verdict_kernel(EncVerdictArgs A) {
  if (threadIdx.x | blockIdx.x) return;
  EncStatus* s = A.st;
  uint32_t flag = 0;
  unsigned long long total;
  if (A.bytes_offs) {
    const int32_t o0 = A.bytes_offs[0], on = A.bytes_offs[A.n_rows];
    total = on >= o0 && o0 >= 0 ? (unsigned long long)(on - o0) + 16ull * A.n_rows : ~0ull;
    if (s->max_word > A.max_len) flag |= EVF_STRIDE;
  } else {
    total = *A.total;
    if (s->overflow) flag |= EVF_CAPACITY;
    if (A.max_rec && s->max_word > A.max_rec) flag |= EVF_SLOT;
  }
  if (total > A.cap || total > 0x7fffffffull) flag |= EVF_CAPACITY;
  if (s->rows_first_bad != 0xffffffffu || s->rows_first_null != 0xffffffffu || s->rows_overflow) flag |= EVF_ROWS;
  if (s->first_null_row != 0xffffffffu) flag |= EVF_NULL;
  s->verdict_flag = flag;
  s->verdict_total_lo = (uint32_t)total; s->verdict_total_hi = (uint32_t)(total >> 32);
}
