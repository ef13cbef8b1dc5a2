// large.cuh -- single-pass decode of records too large for a shared-memory tile (image and embedding Examples, large
// ByteArray payloads).
//
// The tile kernels (tile.cuh, bytes_tile.cuh) stage 32 whole records per CTA; once 32 x the largest record no longer fits the
// 227 KB opt-in (records of roughly 7 KB and more), a batch used to leave the pipelined path for the general kernels and a host
// synchronisation.  These kernels take such batches on the same path, with the same verdict contract: anything outside the
// canonical shapes raises TF_FALLBACK (TF_SHAPE for a shape miss, TF_OVERFLOW for a short buffer) and the host redoes the
// batch through decode_sync, so they never change a result.
//
// Mapping: one CTA of LARGE_WARPS warps per record; the record is read from global memory (L2), never staged whole.
//   CRC     every warp folds one contiguous range of the payload (crc_warp, common.cuh); the ranges are joined with one GF(2)
//           shift each, by x^(8 * bytes after the range), built from CrcTables::x8pow (x^(8 * 2^k)) with a five-step warp product.
//   parse   warp 0 runs the general path's map walk and per-entry parse (walk_map_body / parse_entry, decode.cuh: the full wire
//           rules, written once) for the record, 32 entries at a time; a cell it could not call canonical, an error, a
//           missing non-nullable field or malformed UTF-8 raises TF_FALLBACK.
//   output  the same three modes as the tile kernel, per column (TileArgs::uniform_len):
//             >= 0         uniform: values at row * L, the shape only verified;
//             TILE_RAGGED  ragged: decoupled look-back over records (tickets in start order, per-record totals and inclusive
//                          prefixes published with release / acquire at GPU scope), checked against the capacities;
//             -1           count mode (decode_sync): counts, sources and cell flags for the scans and pass 2.
//           Bulk values (bytes, packed floats) are copied global -> global by the whole CTA with 16-byte stores and 16-byte
//           source loads joined by funnel shifts; packed varints are decoded by the whole CTA (terminators counted per thread
//           range, then a block scan gives every thread the index of its first value).
//   ByteArray: the same kernel without the parse: CRC and copy, positions from the frame index.
// Not covered (these batches keep their paths): SequenceExample, schemas of more than 128 fields, malformed UTF-8 in a
// string column (the general path re-encodes it), and splitting one batch between the tile and the large-record kernel.
#pragma once
#include "common.cuh"
#include "decode.cuh"
#include "tile.cuh"

#define LARGE_WARPS 8
#define LARGE_THREADS (LARGE_WARPS * 32)
#define LARGE_MAX_FIELDS 128

struct LargeArgs {
  TileArgs t;            // input, record offsets, rows (n_dev), verification, bitmaps, null counters, outputs, look-back table
                         // (one entry per record), capacities, totals, flags -- as for the tile kernels
  DecodeArgs d;          // the general parse's view: data, sch, tabs, fix_values, cnt / src / cflag with stride d.n
};

// CRC-32C of payload[0, len), all threads of the CTA; the result is valid in thread 0.  s_part: [LARGE_WARPS] shared words.
__device__ __forceinline__ uint32_t large_crc(const uint32_t* stab, const uint32_t* x8pow, const uint8_t* payload, uint32_t len, uint32_t* s_part) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t lo = (uint32_t)((uint64_t)len * wid / LARGE_WARPS), hi = (uint32_t)((uint64_t)len * (wid + 1) / LARGE_WARPS);
  const uint32_t c = crc_warp(stab, payload + lo, hi - lo);
  // CRC(A || B) = shift_|B|(CRC(A)) ^ CRC(B): the shift by the bytes behind this range, as a product over its set bits
  const uint32_t after = len - hi;
  uint32_t f = ((after >> lane) & 1u) ? x8pow[lane] : 0x80000000u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) f = gf2_mulmod(f, __shfl_xor_sync(FULLMASK, f, o));
  if (lane == 0) s_part[wid] = after ? gf2_mulmod(f, c) : c;
  __syncthreads();
  uint32_t x = 0;
  if (threadIdx.x == 0) for (int w = 0; w < LARGE_WARPS; ++w) x ^= s_part[w];
  return x;
}

// n bytes src -> dst by `nt` threads (thread index t), any alignment of either side.  16-byte stores; a 16-byte group of the
// source is loaded whole only when it lies inside [lo, hi) (the input buffer: a caller's buffer needs no padding), the other
// bytes one by one.
__device__ __forceinline__ void large_copy(uint8_t* dst, const uint8_t* src, uint32_t n, uint32_t t, uint32_t nt, const uint8_t* lo, const uint8_t* hi) {
  const uint32_t h = min(n, (uint32_t)((0u - (uint32_t)reinterpret_cast<uintptr_t>(dst)) & 15u));
  if (t < h) dst[t] = src[t];
  const uint32_t chunks = (n - h) >> 4;
  const uint8_t* s = src + h;
  const uint32_t r = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 15u), q = r >> 2, sh = (r & 3u) * 8u;
  const uint8_t* a0 = s - r;
  for (uint32_t j = t; j < chunks; j += nt) {
    const uint8_t* g = a0 + 16ull * j;
    uint4 o;
    if (g >= lo && g + (r ? 32 : 16) <= hi) {
      const uint4 v = *reinterpret_cast<const uint4*>(g);
      if (r == 0) o = v;
      else {
        const uint4 u = *reinterpret_cast<const uint4*>(g + 16);
        uint32_t w0, w1, w2, w3, w4;                          // the five words that hold the chunk, from word q of v on
        if (q == 0) { w0 = v.x; w1 = v.y; w2 = v.z; w3 = v.w; w4 = u.x; }
        else if (q == 1) { w0 = v.y; w1 = v.z; w2 = v.w; w3 = u.x; w4 = u.y; }
        else if (q == 2) { w0 = v.z; w1 = v.w; w2 = u.x; w3 = u.y; w4 = u.z; }
        else { w0 = v.w; w1 = u.x; w2 = u.y; w3 = u.z; w4 = u.w; }
        o.x = __funnelshift_r(w0, w1, sh); o.y = __funnelshift_r(w1, w2, sh); o.z = __funnelshift_r(w2, w3, sh); o.w = __funnelshift_r(w3, w4, sh);
      }
    } else {
      uint8_t b[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) b[k] = s[16ull * j + k];
      o.x = b[0] | (b[1] << 8) | (b[2] << 16) | ((uint32_t)b[3] << 24); o.y = b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24);
      o.z = b[8] | (b[9] << 8) | (b[10] << 16) | ((uint32_t)b[11] << 24); o.w = b[12] | (b[13] << 8) | (b[14] << 16) | ((uint32_t)b[15] << 24);
    }
    *reinterpret_cast<uint4*>(dst + h + 16ull * j) = o;
  }
  const uint32_t done = h + 16 * chunks;
  if (t < n - done) dst[done + t] = src[done + t];
}

// A length varint as the canonical wire form writes it: minimal, at most 5 bytes, inside [p, end).  The general parse also
// accepts overlong varints; the cells this kernel emits itself are read back with this rule, and anything else is flagged.
__device__ __forceinline__ bool large_len(Cur& c, uint32_t& v) {
  const uint8_t* q = c.p;
  if (!rd_len(c, v)) return false;
  const uint32_t k = (uint32_t)(c.p - q);
  return k <= 5 && (k == 1 || q[k - 1] != 0);
}

// StringType cells: well-formed UTF-8 only (java_utf8_transcode can replace a malformed unit by U+FFFD without changing the
// length, so a length compare does not find it).  The `nt` threads of a warp (cta = false) or of the CTA (cta = true) look
// for a non-ASCII byte; one thread then runs utf8_valid.  s_flag: a shared word (CTA only).
__device__ __forceinline__ bool large_utf8_ok(const uint8_t* p, uint32_t n, uint32_t t, uint32_t nt, bool cta, uint32_t* s_flag) {
  uint32_t hi = 0;
  for (uint32_t i = t; i < n; i += nt) hi |= p[i];
  if (!cta) {
    if (!__any_sync(FULLMASK, hi >= 0x80u)) return true;
    return __shfl_sync(FULLMASK, t == 0 ? (uint32_t)utf8_valid(p, n) : 0u, 0) != 0;
  }
  if (!__syncthreads_or(hi >= 0x80u)) return true;
  if (t == 0) *s_flag = utf8_valid(p, n) ? 1u : 0u;
  __syncthreads();
  const bool ok = *s_flag != 0;
  __syncthreads();
  return ok;
}

// block-wide exclusive scan of one value per thread (LARGE_THREADS); s_w: [LARGE_WARPS] shared words
__device__ __forceinline__ uint32_t large_block_scan(uint32_t v, uint32_t* s_w, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t tot;
  const uint32_t ex = warp_excl_scan_u32(v, tot);
  __syncthreads();
  if (lane == 0) s_w[wid] = tot;
  __syncthreads();
  uint32_t base = 0;
  total = 0;
  for (uint32_t w = 0; w < LARGE_WARPS; ++w) { if (w < wid) base += s_w[w]; total += s_w[w]; }
  return base + ex;
}

// the n packed varints at p -> dst[0, n) as int64 / int32, by the whole CTA.  false (nothing trustworthy written) unless the
// packed field is canonical: a one-byte `0A` tag, a minimal length varint of at most 5 bytes, exactly n values, the last
// byte a terminator.
__device__ __forceinline__ bool large_varints(const uint8_t* p, uint32_t n, bool i64, void* dst, uint32_t* s_w) {
  // the packed length: the varint that ends right in front of the data.  Its bytes are the run of continuation bytes in front of
  // its last byte; the byte in front of that run must be the tag.
  uint32_t k = 1;
  while (k < 6 && (p[-1 - (int)k] & 0x80u)) ++k;
  if (k > 5 || p[-1 - (int)k] != 0x0Au || (k > 1 && p[-1] == 0)) return false;     // (the same for every thread)
  uint32_t plen = 0;
  for (uint32_t i = 0; i < k; ++i) plen |= (uint32_t)(p[(int)i - (int)k] & 0x7f) << (7 * i);
  const uint32_t t = threadIdx.x, seg = (plen + LARGE_THREADS - 1) / LARGE_THREADS;
  const uint32_t b0 = min(plen, t * seg), b1 = min(plen, b0 + seg);
  uint32_t c = 0;
  for (uint32_t i = b0; i < b1; ++i) c += p[i] < 0x80u;
  uint32_t total;
  uint32_t idx = large_block_scan(c, s_w, total);            // values that end in front of this thread's range
  for (uint32_t i = b0; i < b1; ++i) {                       // idx: the values that end in front of byte i
    if ((i == 0 || p[i - 1] < 0x80u) && idx < n) {           // the first byte of a varint: value idx
      uint64_t v = 0; uint32_t s = 0, j = i;
      for (;;) { const uint32_t b = p[j++]; v |= (uint64_t)(b & 0x7f) << s; s += 7; if (b < 0x80u || s >= 70) break; }
      if (i64) reinterpret_cast<int64_t*>(dst)[idx] = (int64_t)v; else reinterpret_cast<int32_t*>(dst)[idx] = (int32_t)(uint32_t)v;
    }
    idx += p[i] < 0x80u;
  }
  return total == n && plen > 0 && p[plen - 1] < 0x80u;
}

__device__ __forceinline__ void large_set_bit(uint8_t* bitmaps, uint32_t stride, uint32_t f, uint32_t row, bool valid, bool last) {
  uint32_t* w = reinterpret_cast<uint32_t*>(bitmaps + (size_t)f * stride) + (row >> 5);
  const uint32_t bit = 1u << (row & 31);
  if (valid) atomicOr(w, bit); else atomicAnd(w, ~bit);
  if (last && bit != 0x80000000u) atomicAnd(w, (bit << 1) - 1u);       // the bits behind the last row stay clear
}

// ByteArray rows: CRCs, then the payload to its place (the payload bytes of rows [0, i) are rec_off[i] - 16 i) -- one CTA per record
__global__ void __launch_bounds__(LARGE_THREADS) decode_large_bytes_kernel(LargeArgs L) {
  extern __shared__ uint32_t stab[];
  __shared__ uint32_t s_part[LARGE_WARPS];
  const TileArgs& A = L.t;
  const uint32_t row = blockIdx.x;
  uint32_t n_rows = A.n;
  if (A.n_dev) {
    n_rows = *A.n_dev;
    if (n_rows > A.n) { if (row == 0 && threadIdx.x == 0) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK); return; }
    if (row >= n_rows) return;
  }
  const uint32_t off = A.rec_off[row], len = A.rec_off[row + 1] - off - 16;
  const uint8_t* payload = A.data + off + 12;
  if (A.verify) {
    crc_stage_tables(stab, L.d.tabs);
    __syncthreads();
    const uint32_t c = large_crc(stab, L.d.tabs->x8pow, payload, len, s_part);
    if (threadIdx.x == 0) {
      const uint8_t* h = A.data + off;
      const bool bad = crc_mask(crc_u64(stab, load_u32_unaligned(h), load_u32_unaligned(h + 4))) != load_u32_unaligned(h + 8) ||
                       crc_mask(c) != load_u32_unaligned(payload + len);
      if (bad) atomicOr(A.flags, TF_FALLBACK);                   // the general path reports the error at the right record
    }
  }
  const uint32_t pre = off - 16u * row;
  large_copy(reinterpret_cast<uint8_t*>(A.var_values[0]) + pre, payload, len, threadIdx.x, LARGE_THREADS, A.data, A.data + A.nbytes);
  if (threadIdx.x == 0) {
    A.offs[0][row] = (int32_t)pre;
    const bool last = row + 1 == n_rows;
    large_set_bit(A.bitmaps, A.nb_stride, 0, row, true, last);
    if (last) {
      const uint32_t total = A.rec_off[n_rows] - 16u * n_rows;
      A.offs[0][n_rows] = (int32_t)total;
      if (A.totals) A.totals[0] = total;
      if (A.cap && total > A.cap[0]) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK);
    }
  }
}

// Example rows, one CTA per record (see the header)
__global__ void __launch_bounds__(LARGE_THREADS) decode_large_kernel(LargeArgs L) {
  extern __shared__ uint32_t stab[];
  __shared__ uint32_t s_part[LARGE_WARPS];
  __shared__ uint8_t fstate[LARGE_MAX_FIELDS];
  __shared__ unsigned long long s_base[LARGE_MAX_FIELDS];     // ragged mode: this record's exclusive base per count array
  __shared__ uint32_t s_row, s_bad, s_shape, s_utf8;
  const TileArgs& A = L.t;
  const DecodeArgs& D = L.d;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_row = A.ragged ? atomicAdd(A.ticket, 1u) : blockIdx.x; s_bad = 0; s_shape = 0; }
  __syncthreads();
  const uint32_t row = s_row;                                   // ragged: records in start order (a record only waits for running ones)
  uint32_t n_rows = A.n;
  if (A.n_dev) {
    n_rows = *A.n_dev;
    if (n_rows > A.n) { if (row == 0 && threadIdx.x == 0) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK); return; }   // (no record runs)
    if (row >= n_rows) return;
  }
  const bool last = row + 1 == n_rows;
  const uint32_t off = A.rec_off[row], len = A.rec_off[row + 1] - off - 16;
  const uint8_t* payload = A.data + off + 12;
  crc_stage_tables(stab, D.tabs);
  __syncthreads();
  if (A.verify) {
    const uint32_t c = large_crc(stab, L.d.tabs->x8pow, payload, len, s_part);
    if (threadIdx.x == 0) {
      const uint8_t* h = A.data + off;
      if (crc_mask(crc_u64(stab, load_u32_unaligned(h), load_u32_unaligned(h + 4))) != load_u32_unaligned(h + 8) ||
          crc_mask(c) != load_u32_unaligned(payload + len)) s_bad = 1;
    }
  }
  const uint32_t nf = (uint32_t)D.sch.n_fields, nv = (uint32_t)D.sch.n_var, nc = (uint32_t)D.sch.n_cnt;
  const size_t S = D.n;                                         // stride of the count / source / flag arrays
  // ---- warp 0: the record's map entries, parsed and checked by the general path's rules ----
  if (wid == 0) {
    for (uint32_t i = lane; i < nf; i += 32) fstate[i] = 0;
    __syncwarp();
    bool ok = true;
    uint32_t nent = 0, my_len = 0, my_pos = 0;
    const uint8_t* my_ptr = nullptr;
    Cur top{payload, payload + len};
    for (;;) {
      uint32_t tag;
      if (!rd_tag(top, tag)) { ok = false; break; }
      if (tag == 0) break;
      if (tag == 0x0A) {
        uint32_t l;
        if (!rd_len(top, l)) { ok = false; break; }
        if (!walk_map_body(D, row, Cur{top.p, top.p + l}, false, fstate, nent, my_ptr, my_len, my_pos)) { ok = false; break; }
        top.p += l;
      } else if (!skip_field(top, tag)) { ok = false; break; }
    }
    if (ok && nent) ok = process_round(D, row, nent, my_ptr, my_len, my_pos, false, fstate);
    __syncwarp();
    bool bad = !ok, shape = false;
    // absent fields: null (zero value, zero counts) or an error; validity and null counters
    for (uint32_t f = lane; f < nf && ok; f += 32) {
      const uint32_t st = fstate[f] & 0x3f;
      const DevField& fd = D.sch.fields[f];
      const bool valid = st == 1;
      if (st == 0 || st == 3) {
        if (st == 0 && !fd.nullable) bad = true;
        if (fd.fix_slot >= 0) {
          void* vp = D.fix_values[fd.fix_slot];
          if (fd.width == 8) reinterpret_cast<uint64_t*>(vp)[row] = 0; else reinterpret_cast<uint32_t*>(vp)[row] = 0;
        } else if (fd.var_slot >= 0) {
          for (int l = 0; l < fd.n_levels; ++l) D.cnt[(size_t)(fd.cnt_slot + l) * S + row] = 0;
        }
      } else if (!valid) bad = true;                           // a semantic error: the general path reports it
      large_set_bit(A.bitmaps, A.nb_stride, f, row, valid, last);
      if (!valid) atomicAdd(&A.null_counts[f], 1ull);
    }
    __syncwarp();
    // cells: canonical only; uniform columns must have their shape
    for (uint32_t v = lane; v < nv && ok; v += 32) {
      const DevField& fd = D.sch.fields[D.var_field ? D.var_field[v] : 0];
      const bool valid = (fstate[D.var_field[v]] & 0x3f) == 1;
      const int32_t ul = A.uniform_len[v];
      if (valid && D.cflag[(size_t)v * S + row] != CF_CANON) bad = true;
      if (ul >= 0 && D.cnt[(size_t)fd.cnt_slot * S + row] != (uint32_t)ul) shape = true;
    }
    bad = __any_sync(FULLMASK, bad);
    shape = __any_sync(FULLMASK, shape);
    if (lane == 0) { if (bad) s_bad = 1; if (shape) s_shape = 1; }
    // ---- ragged columns: this record's bases, by decoupled look-back over the records in front of it ----
    if (A.ragged) {
      const uint32_t nc4 = (nc + 3u) & ~3u;
      uint32_t c[4];
      unsigned long long base[4] = {0ull, 0ull, 0ull, 0ull};
#pragma unroll
      for (int k = 0; k < 4; ++k) { const uint32_t a = lane + 32u * k; c[k] = a < nc ? D.cnt[(size_t)a * S + row] : 0u; if (a < nc) A.lb_agg[(size_t)row * nc4 + a] = c[k]; }
      __threadfence();
      __syncwarp();
      if (lane == 0) st_release_u32(&A.lb_flag[row], 1u);
      for (int32_t p = (int32_t)row - 1; p >= 0;) {
        uint32_t fl = ld_acquire_u32(&A.lb_flag[p]);
        fl = __shfl_sync(FULLMASK, fl, 0);
        if (fl == 0u) { __nanosleep(64); continue; }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t a = lane + 32u * k;
          if (a < nc) base[k] += fl == 2u ? ld_cg_u64(A.lb_pre + (size_t)p * nc4 + a) : (unsigned long long)ld_cg_u32(A.lb_agg + (size_t)p * nc4 + a);
        }
        if (fl == 2u) break;
        --p;
      }
      bool over = false;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t a = lane + 32u * k;
        if (a >= nc) continue;
        const unsigned long long incl = base[k] + c[k];
        A.lb_pre[(size_t)row * nc4 + a] = incl;
        s_base[a] = base[k];
        if (incl > A.cap[a] || incl > 0x7fffffffull) over = true;      // target buffer (or int32 offsets) too small: the host redoes the batch
        if (last) A.totals[a] = incl;
      }
      __threadfence();
      __syncwarp();
      if (lane == 0) st_release_u32(&A.lb_flag[row], 2u);
      if (__any_sync(FULLMASK, over) && lane == 0) { s_bad = 1; atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK); }
    }
  }
  __syncthreads();
  if (s_bad || s_shape) {
    if (threadIdx.x == 0) atomicOr(A.flags, s_bad ? TF_FALLBACK : (TF_SHAPE | TF_FALLBACK));
    return;
  }
  // ---- values of the uniform and ragged columns, by the whole CTA ----
  const uint8_t* blo = A.data; const uint8_t* bhi = A.data + A.nbytes;
  for (uint32_t v = 0; v < nv; ++v) {
    const int32_t ul = A.uniform_len[v];
    if (ul == -1) continue;                                    // count mode: pass 2 emits it
    const int f = D.var_field[v];
    const DevField& fd = D.sch.fields[f];
    const bool valid = (fstate[f] & 0x3f) == 1;
    const uint32_t c0 = D.cnt[(size_t)fd.cnt_slot * S + row];
    const uint8_t* src = D.data + D.src[(size_t)v * S + row];
    uint8_t* vals = reinterpret_cast<uint8_t*>(A.var_values[v]);
    unsigned long long e0 = (unsigned long long)row * (uint32_t)max(ul, 0);    // first element (or byte) of the cell
    if (ul == TILE_RAGGED) {
      e0 = s_base[fd.cnt_slot];
      if (threadIdx.x == 0) {
        int32_t* o0 = A.offs[v * 3];
        o0[row] = (int32_t)e0;
        if (last) o0[n_rows] = (int32_t)(e0 + c0);
        if (c0 == 0 && last && fd.n_levels == 2) A.offs[v * 3 + 1][e0] = (int32_t)(s_base[fd.cnt_slot + 1] + D.cnt[(size_t)(fd.cnt_slot + 1) * S + row]);
      }
    }
    if (!valid || c0 == 0) continue;
    const bool is_str = fd.elem_type == TFR_T_STRING;
    if (fd.depth == 0) {                                       // scalar string / binary: the first element, c0 bytes
      Cur c{src, bhi};
      uint32_t raw = 0;
      // (c0 is the general parse's output length: a malformed string's Java re-encoding, which the general path writes)
      if (!large_len(c, raw) || raw != c0 || (is_str && !large_utf8_ok(c.p, raw, threadIdx.x, LARGE_THREADS, true, &s_utf8))) {
        if (threadIdx.x == 0) atomicOr(A.flags, TF_FALLBACK);
        continue;
      }
      large_copy(vals + e0, c.p, c0, threadIdx.x, LARGE_THREADS, blo, bhi);
    } else if (fd.kind == K_FLOAT) {
      if (fd.elem_type == TFR_T_FLOAT32) large_copy(vals + 4 * e0, src, 4 * c0, threadIdx.x, LARGE_THREADS, blo, bhi);
      else for (uint32_t i = threadIdx.x; i < c0; i += LARGE_THREADS) reinterpret_cast<double*>(vals)[e0 + i] = (double)__uint_as_float(load_u32_unaligned(src + 4 * i));
    } else if (fd.kind == K_INT64) {
      const bool i64 = fd.elem_type == TFR_T_INT64;
      if (!large_varints(src, c0, i64, vals + (i64 ? 8 : 4) * e0, s_part) && threadIdx.x == 0) atomicOr(A.flags, TF_FALLBACK);
    } else if (wid == 0) {                                     // list of strings / binaries (ragged): inner offsets + bytes, a warp per element
      int32_t* o1 = A.offs[v * 3 + 1];
      unsigned long long vpos = s_base[fd.cnt_slot + 1];
      const uint32_t want = D.cnt[(size_t)(fd.cnt_slot + 1) * S + row];
      Cur c{src, bhi};
      uint32_t got = 0;
      bool ok = true;
      // every element `0A blen bytes` in the canonical form, its bytes inside what the cell was given (want: its share of the
      // values buffer, checked against the capacity); anything else stops the copy and flags the batch
      for (uint32_t i = 0; i < c0 && ok; ++i) {
        uint32_t bl = 0;
        ok = c.p < bhi && *c.p == 0x0Au;
        if (!ok) break;
        ++c.p;
        ok = large_len(c, bl) && bl <= want - got && (size_t)(bhi - c.p) >= bl && (!is_str || large_utf8_ok(c.p, bl, lane, 32, false, nullptr));
        if (!ok) break;
        if (lane == 0) o1[e0 + i] = (int32_t)vpos;
        large_copy(vals + vpos, c.p, bl, lane, 32, blo, bhi);
        vpos += bl; got += bl; c.p += bl;
      }
      if (lane == 0 && last && ok) o1[e0 + c0] = (int32_t)vpos;
      if ((!ok || got != want) && lane == 0) atomicOr(A.flags, TF_FALLBACK);
    }
    __syncthreads();                                           // (s_part is reused by the next column's varint scan)
  }
}
