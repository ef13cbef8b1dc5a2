// recordType = ByteArray on the fast path: a row IS the record's payload (deserializeByteArray,
// M/TFRecordDeserializer.scala:17-19; framing and the two masked CRCs as in tensorflow-hadoop's TFRecordReader.read).
// Nothing is parsed, so the decode is: verify both CRCs, strip the 16 framing bytes, write Arrow offsets.  The output
// position of every payload follows from the frame index alone -- the payloads of rows [0, i) take rec_off[i] - 16 i
// bytes -- so tiles need no look-back and no count pass: one kernel, every byte read once and written once.
//
// Same tile machinery as decode_tile_kernel (tile.cuh): CTA = 32 consecutive records, lane = record, each record bulk-copied
// (cp.async.bulk + mbarrier) into its own shared-memory slot at an odd multiple of 16 bytes, so the 32 lanes' 16-byte CRC
// loads spread over all bank groups.  CW warps share the CRC of the 32 payloads (each folds a range of every record's
// 16-byte chunks, ranges are joined with one GF(2) multiply -- 190 instructions, so ranges are kept long: CW is 2 when many
// tiles fit an SM and grows only when large records leave room for few); XW warps meanwhile copy the payloads out, one
// record per warp at a time, 4 bytes per lane (conflict-free in shared memory, 128-byte coalesced in global memory).
#pragma once
#include "encode.cuh"
#include "tile.cuh"

// Register bound: 48 resident warps per SM (four 8 + 4 warp tiles, eight 4 + 2 warp tiles), i.e. 40 registers, 16-20 B of
// spills on sm_90a.  Unbounded, ptxas takes 56 registers and only three 12-warp tiles fit the register file.  On one H100
// SXM (1 KiB payloads, 0.5 GiB batches, two alternated runs): decode 1,133 / 1,140 GB/s with this bound, 1,113 / 1,134
// unbounded, 984 / 990 with five tiles (32 registers, 72 B of spills); encode 1,067 / 1,083, 1,070 / 1,074, 873 / 864.
#define BYTES_BOUNDS(CW, XW) __launch_bounds__((CW + XW) * 32, 48 / (CW + XW))

__host__ __device__ inline uint32_t bytes_const_bytes() { return TILE_CRC_BYTES + TILE_SEEN_BYTES; }    // the head of the schema's consts blob: g5 | xp16 | zeroed accumulators
__host__ __device__ inline uint32_t bytes_smem_bytes(uint32_t tile_cap) { return 16u + bytes_const_bytes() + tile_cap + 64u; }

// TileArgs fields used: data, nbytes, misalign, rec_off, n, n_dev, tile_cap, slot (never 0), tile_max, verify, consts,
// bitmaps (validity of the one column), offs[0] (Arrow offsets), var_values[0] (the bytes), totals (nullable), cap (nullable), flags
template <int CW, int XW>
__global__ void BYTES_BOUNDS(CW, XW) decode_bytes_kernel(TileArgs A) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* s8 = reinterpret_cast<uint32_t*>(smem_raw + 16);
  uint32_t* scrc = reinterpret_cast<uint32_t*>(smem_raw + 16 + TILE_CRC_BYTES) + 128;          // [32] per-record accumulators, zero in the blob
  const uint32_t* xp16 = s8 + 512;
  uint8_t* tile_b = smem_raw + 16 + bytes_const_bytes();
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t tile = blockIdx.x;
  const uint32_t row0 = tile * TILE_ROWS;
  uint32_t n_rows = A.n;
  if (A.n_dev) {
    n_rows = *A.n_dev;
    if (n_rows > A.n) {                                                    // more records than the host provisioned for: the host redoes the batch
      if (tile == 0 && threadIdx.x == 0) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK);
      return;
    }
    if (row0 >= n_rows) return;
  }
  const uint32_t rows = min((uint32_t)TILE_ROWS, n_rows - row0);
  const bool active = lane < rows;
  const uint32_t row = row0 + lane;
  uint32_t off = 0, flen = 16;
  if (active) { off = A.rec_off[row]; flen = A.rec_off[row + 1] - off; }
  // the record's 16-byte groups, clipped to the buffer (see decode_tile_kernel: any alignment, no padding)
  const uint32_t mis = A.misalign, lim = mis + A.nbytes;
  const uint8_t* base = A.data - mis;
  const uint32_t head = (off + mis) & 15u;
  const uint32_t g_lo = off + mis - head;
  const uint32_t cbytes = active ? (head + flen + 15u) & ~15u : 0u;
  uint32_t b_lo = g_lo, b_hi = g_lo + cbytes;
  if (active && b_lo < mis) b_lo += 16u;
  if (active && b_hi > lim) b_hi = lim & ~15u;
  const uint32_t bulk_bytes = (active && b_hi > b_lo) ? b_hi - b_lo : 0u;
  uint32_t stride = active ? (cbytes + 32u + 15u) & ~15u : 0u;
  if (active && ((stride >> 4) & 1u) == 0u) stride += 16u;
  const uint32_t rbase = lane * A.slot;
  if (A.tile_max) {                                                        // what the next batch's slots are sized from
    const uint32_t m = __reduce_max_sync(FULLMASK, stride);
    if (threadIdx.x == 0) atomicMax(A.tile_max, m * TILE_ROWS);
  }
  if (__any_sync(FULLMASK, stride > A.slot)) {                             // a record larger than the slot: the host redoes the batch
    if (threadIdx.x == 0) atomicOr(A.flags, TF_FALLBACK);
    return;
  }
  if (wid == 0) {
    if (lane == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const uint32_t total = __reduce_add_sync(FULLMASK, bulk_bytes);
    if (lane == 0) {
      mbar_expect_tx(bar, total + bytes_const_bytes());
      bulk_g2s(smem_raw + 16, A.consts, bytes_const_bytes(), bar);
    }
    __syncwarp();
    if (bulk_bytes) bulk_g2s(tile_b + rbase + (b_lo - g_lo), base + b_lo, bulk_bytes, bar);
    if (active) {
      uint8_t* sl = tile_b + rbase;
      const uint32_t e1 = min(b_lo, lim);
      if (b_lo > g_lo) for (uint32_t i = mis; i < e1; ++i) sl[i - g_lo] = base[i];                                  // clipped first group
      if (b_hi < g_lo + cbytes) for (uint32_t i = max(b_hi, e1); i < lim; ++i) sl[i - g_lo] = base[i];             // clipped last group
    }
  }
  __syncthreads();
  mbar_wait(bar, 0);

  const uint32_t len = flen - 16;
  const uint32_t pay = rbase + head + 12;
  const uint32_t end = pay + len;
  Tile T;
  T.b = tile_b;
  asm volatile("mov.u32 %0, %1;" : "=r"(T.s) : "r"(smem_u32(tile_b)) : "memory");   // ordered after mbar_wait

  if (wid < CW) {
    // ---- CRC of the 32 payloads, shared by the CRC warps (see crc_chunks in tile.cuh) ----
    const bool on = active && A.verify;
    const uint32_t hn = min(len, (0u - pay) & 15u);
    const uint32_t b0 = pay + hn;
    const uint32_t K = (end - b0) >> 4;
    if (on) {
      uint32_t c = 0;
      if (wid == 0) {
        c = 0xFFFFFFFFu;
        for (uint32_t i = 0; i < hn; ++i) c = crc_byte(s8, c, T.u8(pay + i));
      }
      if (wid == CW - 1) {       // the frame index chained the headers without checking them: the length CRC
        if (crc_mask(~crc_fold8(s8, 0xFFFFFFFFu, t_u32(T, pay - 12), t_u32(T, pay - 8))) != t_u32(T, pay - 4)) atomicOr(A.flags, TF_FALLBACK);
      }
      const uint32_t k0 = K * wid / CW, k1 = K * (wid + 1) / CW;
      c = crc_chunks(s8, T, b0 + 16 * k0, k1 - k0, c);
      if (CW == 1) scrc[lane] = c;
      else if (c) atomicXor(&scrc[lane], K - k1 ? gf2_mulmod(xp16[K - k1], c) : c);
    }
    if (CW > 1) asm volatile("bar.sync 1, %0;" ::"r"(CW * 32) : "memory");
    if (wid == 0 && on) {
      uint32_t c = scrc[lane];
      for (uint32_t o = b0 + 16 * K; o < end; ++o) c = crc_byte(s8, c, T.u8(o));
      if (crc_mask(~c) != t_u32(T, end)) atomicOr(A.flags, TF_FALLBACK);          // the general path reports the error at the right record
    }
    return;
  }

  // ---- rows out: bytes [pre, pre + len) of the values buffer, offsets[row] = pre ----
  const uint32_t pre = off - 16u * row;                                          // payload bytes of the rows before this one (rec_off[0] == 0)
  uint8_t* values = reinterpret_cast<uint8_t*>(A.var_values[0]);
  int32_t* offs = A.offs[0];
  if (wid == CW) {
    if (active) offs[row] = (int32_t)pre;
    if (lane == 0) reinterpret_cast<uint32_t*>(A.bitmaps)[tile] = rows == TILE_ROWS ? 0xFFFFFFFFu : (1u << rows) - 1u;      // every row is valid
    if (row0 + rows == n_rows && lane == 0) {
      const uint32_t total = A.rec_off[n_rows] - 16u * n_rows;
      offs[n_rows] = (int32_t)total;
      if (A.totals) A.totals[0] = total;
      if (A.cap && total > A.cap[0]) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK);   // (cannot happen: the host sizes the buffer from the input's size)
    }
  }
  if (wid == CW + XW - 1 && A.pf_dist) {
    // the tile that takes this CTA's place when it retires: ask L2 for its records now (see decode_tile_kernel)
    const uint32_t row2 = (tile + A.pf_dist) * TILE_ROWS + lane;
    if (row2 < n_rows) {
      const uint32_t o2 = A.rec_off[row2] + mis, e2 = min(A.rec_off[row2 + 1] + mis, lim & ~15u);
      const uint32_t a2 = (o2 + 15u) & ~15u;
      if (e2 > a2 + 16u) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + a2), "r"((e2 - a2) & ~15u) : "memory");
    }
  }
  for (uint32_t r = wid - CW; r < rows; r += XW) {
    const uint32_t spay = __shfl_sync(FULLMASK, pay, r), slen = __shfl_sync(FULLMASK, len, r), spre = __shfl_sync(FULLMASK, pre, r);
    uint8_t* dst = values + spre;
    const uint32_t hm = min(slen, (0u - (uint32_t)reinterpret_cast<uintptr_t>(dst)) & 3u);
    if (lane < hm) dst[lane] = (uint8_t)T.u8(spay + lane);
    const uint32_t words = (slen - hm) >> 2;
    const uint32_t so = spay + hm, sh = (so & 3u) * 8u, sa = so & ~3u;
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst + hm);
    if (sh == 0) for (uint32_t i = lane; i < words; i += 32) dw[i] = T.w32(sa + 4 * i);
    else for (uint32_t i = lane; i < words; i += 32) dw[i] = __funnelshift_r(T.w32(sa + 4 * i), T.w32(sa + 4 * i + 4), sh);
    const uint32_t tl = (slen - hm) & 3u;
    if (lane < tl) dst[hm + 4 * words + lane] = (uint8_t)T.u8(so + 4 * words + lane);
  }
}

// ---------------------------------------------------------------------------------------------
// The mirror: ByteArray rows -> framed records (serializeByteArray M/TFRecordSerializer.scala:16-18 + TFRecordWriter.write:
// u64 length | masked CRC32C of the length | payload | masked CRC32C of the payload).  Record r goes to byte
// (offs[r] - offs[0]) + 16 r of the output: positions follow from the column's offsets, so there is no size pass and no scan.
// Same tile shape as decode_bytes_kernel: the payloads of 32 consecutive rows are bulk-copied into shared-memory slots, CW
// warps share their CRCs (and write the 12-byte headers and 4-byte footers), XW warps copy the payloads into the frames.
// ---------------------------------------------------------------------------------------------
struct EncBytesArgs {
  const int32_t* offs;          // [n_rows + 1] Arrow offsets of the binary column
  const uint8_t* values;        // the payload bytes
  uint32_t n_values;            // offs[n_rows]: end of the bytes the rows use in `values` (what the bulk copies are clipped to)
  uint32_t misalign;            // values & 15
  uint32_t n_rows;
  uint32_t slot;                // odd multiple of 16, >= the largest payload + 78
  const uint8_t* consts;        // g5 | xp16 | zeroed accumulators (bytes_const_bytes())
  uint8_t* out;
  unsigned long long out_cap;
  EncStatus* st;                // overflow (a payload larger than the slot, inconsistent offsets), total_lo / total_hi
};

__global__ void bytes_max_len_kernel(const int32_t* __restrict__ offs, uint32_t n_rows, uint32_t* __restrict__ out) {
  uint32_t m = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows; i += gridDim.x * blockDim.x) m = max(m, (uint32_t)(offs[i + 1] - offs[i]));
  m = __reduce_max_sync(FULLMASK, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// GUARD: the pipelined encoder's instantiation (api_encode.inc): it returns at once when encode_verdict_kernel (encode.cuh) has
// raised *flag -- the stride was launched for a learned payload length the batch exceeds, the output block is too small, or the
// batch holds a data error.  GUARD = false (the synchronous path) never reads `flag`.
template <int CW, int XW, bool GUARD>
__global__ void BYTES_BOUNDS(CW, XW) encode_bytes_kernel(EncBytesArgs A, const uint32_t* __restrict__ flag) {
  if (GUARD && *flag) return;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* s8 = reinterpret_cast<uint32_t*>(smem_raw + 16);
  uint32_t* scrc = reinterpret_cast<uint32_t*>(smem_raw + 16 + TILE_CRC_BYTES) + 128;
  const uint32_t* xp16 = s8 + 512;
  uint8_t* tile_b = smem_raw + 16 + bytes_const_bytes();
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t row0 = blockIdx.x * TILE_ROWS;
  const uint32_t rows = min((uint32_t)TILE_ROWS, A.n_rows - row0);
  const bool active = lane < rows;
  const uint32_t row = row0 + lane;
  const uint32_t off0 = (uint32_t)A.offs[0];
  uint32_t lo = off0, len = 0;
  if (active) { lo = (uint32_t)A.offs[row]; len = (uint32_t)A.offs[row + 1] - lo; }
  // the payload's 16-byte groups inside `values`, clipped to [values, values + n_values) like the decoder's records
  const uint32_t mis = A.misalign, lim = mis + A.n_values;
  const uint8_t* base = A.values - mis;
  const uint32_t head = (lo + mis) & 15u;
  const uint32_t g_lo = lo + mis - head;
  const uint32_t cbytes = (active && len) ? (head + len + 15u) & ~15u : 0u;
  uint32_t b_lo = g_lo, b_hi = g_lo + cbytes;
  if (cbytes && b_lo < mis) b_lo += 16u;
  if (cbytes && b_hi > lim) b_hi = lim & ~15u;
  const uint32_t bulk_bytes = (cbytes && b_hi > b_lo) ? b_hi - b_lo : 0u;
  const uint32_t rbase = lane * A.slot;
  const unsigned long long o = (unsigned long long)(lo - off0) + 16ull * row;      // where the framed record starts
  const bool bad = active && (cbytes + 48u > A.slot || lo + len > A.n_values || lo < off0 || o + 16ull + len > A.out_cap);
  if (__any_sync(FULLMASK, bad)) {                          // a payload larger than the slot or inconsistent offsets: the host falls back (every warp sees the same rows: uniform exit)
    if (threadIdx.x == 0) atomicOr(&A.st->overflow, 1u);
    return;
  }
  if (wid == 0) {
    if (lane == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const uint32_t total = __reduce_add_sync(FULLMASK, bulk_bytes);
    if (lane == 0) {
      mbar_expect_tx(bar, total + bytes_const_bytes());
      bulk_g2s(smem_raw + 16, A.consts, bytes_const_bytes(), bar);
    }
    __syncwarp();
    if (bulk_bytes) bulk_g2s(tile_b + rbase + (b_lo - g_lo), base + b_lo, bulk_bytes, bar);
    if (cbytes) {
      uint8_t* sl = tile_b + rbase;
      const uint32_t e1 = min(b_lo, lim);
      if (b_lo > g_lo) for (uint32_t i = max(mis, g_lo); i < e1; ++i) sl[i - g_lo] = base[i];                      // clipped first group
      if (b_hi < g_lo + cbytes) for (uint32_t i = max(b_hi, e1); i < lim; ++i) sl[i - g_lo] = base[i];             // clipped last group
    }
  }
  __syncthreads();
  mbar_wait(bar, 0);

  const uint32_t pay = rbase + head;
  const uint32_t end = pay + len;
  Tile T;
  T.b = tile_b;
  asm volatile("mov.u32 %0, %1;" : "=r"(T.s) : "r"(smem_u32(tile_b)) : "memory");   // ordered after mbar_wait
  if (row0 + rows == A.n_rows && threadIdx.x == rows - 1) {
    const unsigned long long total = o + 16ull + len;
    A.st->total_lo = (uint32_t)total; A.st->total_hi = (uint32_t)(total >> 32);
  }

  if (wid < CW) {
    const uint32_t hn = min(len, (0u - pay) & 15u);
    const uint32_t b0 = pay + hn;
    const uint32_t K = (end - b0) >> 4;
    if (active) {
      uint32_t c = 0;
      if (wid == 0) {
        c = 0xFFFFFFFFu;
        for (uint32_t i = 0; i < hn; ++i) c = crc_byte(s8, c, T.u8(pay + i));
      }
      const uint32_t k0 = K * wid / CW, k1 = K * (wid + 1) / CW;
      c = crc_chunks(s8, T, b0 + 16 * k0, k1 - k0, c);
      if (CW == 1) scrc[lane] = c;
      else if (c) atomicXor(&scrc[lane], K - k1 ? gf2_mulmod(xp16[K - k1], c) : c);
    }
    if (CW > 1) asm volatile("bar.sync 1, %0;" ::"r"(CW * 32) : "memory");
    if (wid == 0 && active) {
      uint32_t c = scrc[lane];
      for (uint32_t q = b0 + 16 * K; q < end; ++q) c = crc_byte(s8, c, T.u8(q));
      const uint32_t fc = crc_mask(~c);
      const uint32_t hc = crc_mask(~crc_fold8(s8, 0xFFFFFFFFu, len, 0u));
      uint8_t* h = A.out + o;                                              // any alignment: bytes
      for (int i = 0; i < 4; ++i) { h[i] = (uint8_t)(len >> (8 * i)); h[4 + i] = 0; h[8 + i] = (uint8_t)(hc >> (8 * i)); }
      uint8_t* ft = h + 12 + len;
      for (int i = 0; i < 4; ++i) ft[i] = (uint8_t)(fc >> (8 * i));
    }
    return;
  }
  // ---- payloads into their frames ----
  const uint32_t olo = (uint32_t)o, ohi = (uint32_t)(o >> 32);
  for (uint32_t r = wid - CW; r < rows; r += XW) {
    const uint32_t spay = __shfl_sync(FULLMASK, pay, r), slen = __shfl_sync(FULLMASK, len, r);
    const unsigned long long so64 = ((unsigned long long)__shfl_sync(FULLMASK, ohi, r) << 32) | __shfl_sync(FULLMASK, olo, r);
    uint8_t* dst = A.out + so64 + 12;
    const uint32_t hm = min(slen, (0u - (uint32_t)reinterpret_cast<uintptr_t>(dst)) & 3u);
    if (lane < hm) dst[lane] = (uint8_t)T.u8(spay + lane);
    const uint32_t words = (slen - hm) >> 2;
    const uint32_t so = spay + hm, sh = (so & 3u) * 8u, sa = so & ~3u;
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst + hm);
    if (sh == 0) for (uint32_t i = lane; i < words; i += 32) dw[i] = T.w32(sa + 4 * i);
    else for (uint32_t i = lane; i < words; i += 32) dw[i] = __funnelshift_r(T.w32(sa + 4 * i), T.w32(sa + 4 * i + 4), sh);
    const uint32_t tl = (slen - hm) & 3u;
    if (lane < tl) dst[hm + 4 * words + lane] = (uint8_t)T.u8(so + 4 * words + lane);
  }
}
