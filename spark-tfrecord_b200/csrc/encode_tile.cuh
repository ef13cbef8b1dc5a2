// encode_tile.cuh -- emit pass of the encoder for Example records through shared-memory tiles: the mirror of tile.cuh.
//
// Same reference functions as encode.cuh (serializeExample M/TFRecordSerializer.scala:20-35, feature construction
// :68-207, Example.toByteArray M/TFRecordOutputWriter.scala:31, TFRecordWriter.write :37) and the same bytes.  The
// general emit kernel (encode.cuh: warp per row, lane per field) writes every entry byte by byte into HBM and reads
// the payload back for the CRC.  Here one CTA builds 32 consecutive records (lane = row, as in the decoder) in
// shared memory:
//   1. the Feature sizes of the tile (cell_size[f][row], written by the size pass) are loaded into shared memory
//      (lane = row: coalesced); warp 0 turns them into entry offsets inside each record (prefix over the fields);
//   2. warp w writes the map entries of fields f = w, w+W, ... of record `lane` into that record's slot: the column
//      reads of a warp cover 32 consecutive rows (coalesced), the byte stores go to shared memory.  The slot stride
//      is 4 (mod 128) bytes, so the lanes' records start in 32 different banks: stores, CRC loads and the copy-out are
//      free of bank conflicts when the lanes move in step;
//   3. every warp folds a share of the 16-byte chunks of record `lane`'s payload (aligned word loads, the 13 conflict-
//      free 5-bit tables of tile.cuh), shifts its state over the chunks after its range with one GF(2) multiply and
//      XORs it into the record's accumulator; warp 0 folds the < 16-byte tail and writes header and footer;
//   4. the records of the tile are contiguous in the output: each warp copies whole records, 32 consecutive bytes per
//      instruction (full sectors).
// Rows that do not fit a slot, SequenceExample / ByteArray schemas and more than 255 fields use encode.cuh.
#pragma once
#include "common.cuh"
#include "encode.cuh"
#include "tile.cuh"

#define ENC_TILE_ROWS 32
#ifndef ENC_TILE_WARPS
#define ENC_TILE_WARPS 8
#endif
#define ENC_TILE_THREADS (ENC_TILE_WARPS * 32)
#define ENC_SIZE_WARPS 8          // the size pass: little shared memory, six CTAs per SM
#define ENC_SIZE_THREADS (ENC_SIZE_WARPS * 32)

struct EncTileArgs {
  DevSchema sch;
  const EncCol* cols;           // [n_fields]
  uint32_t n_rows;
  const CrcTables* tabs;
  const uint32_t* cell_size;    // [n_fields][n_rows] Feature bytes of every cell (0xffffffff: null), from the size pass
  const int32_t* rec_off;       // [n_rows+1]
  uint8_t* out;
  uint32_t slot;                // bytes per record slot, 4 (mod 128)
  uint32_t names_bytes;         // bytes of sch.names (staged in shared memory by encode_tile_kernel)
};

// shared memory: g5 + xp16 (4 KiB) | CRC accumulators [32] | group size [32] | vsz u16 [nf][32] | eoff u16 [nf][32] | slots
__host__ __device__ inline uint32_t enc_tile_smem_bytes(uint32_t nf, uint32_t slot) {
  return 4096 + 128 + 128 + ((nf * 32 * 2 * 2 + 15u) & ~15u) + ENC_TILE_ROWS * slot + 16;
}
// encode_tile_kernel also keeps the schema's fields, the column pointers and the names in shared memory (in front of the slots):
// per (field, row) only the value loads go to global memory, not a chain fields[f] -> cols[f] -> values
__host__ __device__ inline uint32_t enc_tile_meta_bytes(uint32_t nf, uint32_t names_bytes) {
  return ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u) + ((nf * (uint32_t)sizeof(EncCol) + 15u) & ~15u) + ((names_bytes + 15u) & ~15u);
}

// size pass with the same mapping (lane = row, warp w takes fields w, w+W, ...): coalesced column reads, Feature sizes
// written [field][row], record sizes accumulated per row in shared memory.  Replaces encode_kernel<0> for Example schemas.
struct EncSizeArgs {
  DevSchema sch;
  const EncCol* cols;
  uint32_t n_rows;
  uint32_t* rec_size;           // [n_rows]
  uint32_t* cell_size;          // [n_fields][n_rows]
  EncStatus* st;                // first_null_row, max_word
};
__global__ void __launch_bounds__(ENC_SIZE_THREADS, 6) encode_tile_size_kernel(EncSizeArgs A) {
  __shared__ uint32_t sacc[ENC_TILE_ROWS];
  extern __shared__ __align__(16) uint8_t ssm[];              // fields | column pointers (enc_tile_meta_bytes(nf, 0)): no fields[f] -> cols[f] -> values chains
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  DevField* sfd = reinterpret_cast<DevField*>(ssm);
  EncCol* scol = reinterpret_cast<EncCol*>(ssm + ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u));
  {
    const uint32_t* gf = reinterpret_cast<const uint32_t*>(A.sch.fields);
    uint32_t* df = reinterpret_cast<uint32_t*>(sfd);
    for (uint32_t i = threadIdx.x; i < nf * (uint32_t)(sizeof(DevField) / 4); i += ENC_SIZE_THREADS) df[i] = gf[i];
    const uint32_t* gc = reinterpret_cast<const uint32_t*>(A.cols);
    uint32_t* dc = reinterpret_cast<uint32_t*>(scol);
    for (uint32_t i = threadIdx.x; i < nf * (uint32_t)(sizeof(EncCol) / 4); i += ENC_SIZE_THREADS) dc[i] = gc[i];
  }
  const uint32_t row = blockIdx.x * ENC_TILE_ROWS + lane;
  const bool active = row < A.n_rows;
  if (threadIdx.x < ENC_TILE_ROWS) sacc[threadIdx.x] = 0;
  __syncthreads();
  uint32_t sum = 0;
  bool null_err = false;
  if (active)
    for (uint32_t f = wid; f < nf; f += ENC_SIZE_WARPS) {
      const DevField& fd = sfd[f];
      const uint32_t V = cell_value_size(fd, scol[f], row);
      A.cell_size[(size_t)f * A.n_rows + row] = V;
      if (V == 0xffffffffu) { if (!fd.nullable) null_err = true; }      // NullPointerException (:29-31)
      else sum += entry_total(fd, V);
    }
  if (sum) atomicAdd(&sacc[lane], sum);
  if (null_err) atomicMin(&A.st->first_null_row, row);
  __syncthreads();
  if (wid == 0 && active) {
    const uint32_t G = sacc[lane], sz = 16 + 1 + vsize32(G) + G;
    A.rec_size[row] = sz;
    const uint32_t mx = __reduce_max_sync(__activemask(), sz);
    if (lane == 0) atomicMax(&A.st->max_word, mx);
  }
}

// GUARD: the instantiation of the pipelined encoder (api_encode.inc).  Its launch figures were learned on earlier batches, so it
// returns at once when encode_verdict_kernel (encode.cuh) has raised *flag: the output block or the slot would be too small, or
// the batch holds a data error.  GUARD = false (the synchronous path) never reads `flag`.
template <bool GUARD>
__global__ void __launch_bounds__(ENC_TILE_THREADS, 3) encode_tile_kernel(EncTileArgs A, const uint32_t* __restrict__ flag) {
  if (GUARD && *flag) return;
  extern __shared__ __align__(128) uint8_t esm[];
  uint32_t* g5 = reinterpret_cast<uint32_t*>(esm);
  const uint32_t* xp16 = g5 + 512;
  uint32_t* scrc = g5 + 1024;
  uint32_t* sgrp = scrc + 32;
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  uint16_t* vsz = reinterpret_cast<uint16_t*>(sgrp + 32);
  uint16_t* eoff = vsz + nf * 32;
  uint8_t* meta = esm + 4096 + 128 + 128 + ((nf * 32 * 2 * 2 + 15u) & ~15u);
  DevField* sfd = reinterpret_cast<DevField*>(meta);
  EncCol* scol = reinterpret_cast<EncCol*>(meta + ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u));
  uint8_t* snames = meta + ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u) + ((nf * (uint32_t)sizeof(EncCol) + 15u) & ~15u);
  uint8_t* slots = meta + enc_tile_meta_bytes(nf, A.names_bytes);
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t row0 = blockIdx.x * ENC_TILE_ROWS;
  const uint32_t rows = min((uint32_t)ENC_TILE_ROWS, A.n_rows - row0);
  const bool active = lane < rows;
  const uint32_t row = row0 + lane;

  {   // CRC tables (g5 and xp16 are contiguous in CrcTables), accumulators, Feature sizes of the tile
    const uint32_t* g = A.tabs->g5;
    for (uint32_t i = threadIdx.x; i < 1024; i += ENC_TILE_THREADS) g5[i] = g[i];
    if (threadIdx.x < 32) scrc[threadIdx.x] = 0;
    {
      const uint32_t* gf = reinterpret_cast<const uint32_t*>(A.sch.fields);          // DevField and EncCol are whole words
      uint32_t* df = reinterpret_cast<uint32_t*>(sfd);
      for (uint32_t i = threadIdx.x; i < nf * (uint32_t)(sizeof(DevField) / 4); i += ENC_TILE_THREADS) df[i] = gf[i];
      const uint32_t* gc = reinterpret_cast<const uint32_t*>(A.cols);
      uint32_t* dc = reinterpret_cast<uint32_t*>(scol);
      for (uint32_t i = threadIdx.x; i < nf * (uint32_t)(sizeof(EncCol) / 4); i += ENC_TILE_THREADS) dc[i] = gc[i];
      for (uint32_t i = threadIdx.x; i < A.names_bytes; i += ENC_TILE_THREADS) snames[i] = A.sch.names[i];
    }
    for (uint32_t f = wid; f < nf; f += ENC_TILE_WARPS) {
      const uint32_t V = active ? A.cell_size[(size_t)f * A.n_rows + row] : 0xffffffffu;
      vsz[f * 32 + lane] = V == 0xffffffffu ? (uint16_t)0xffff : (uint16_t)V;
    }
  }
  __syncthreads();
  if (wid == 0) {     // entry offsets inside the Features message, per row
    uint32_t acc = 0;
    for (uint32_t f = 0; f < nf; ++f) {
      const uint32_t V = vsz[f * 32 + lane];
      eoff[f * 32 + lane] = (uint16_t)acc;
      if (V != 0xffffu) acc += entry_total(sfd[f], V);
    }
    sgrp[lane] = acc;
  }
  __syncthreads();
  const uint32_t G = sgrp[lane];
  const uint32_t ghdr = 1 + vsize32(G);
  const uint32_t plen = ghdr + G;                                  // payload = 0A varint(G) Features
  uint8_t* rec = slots + lane * A.slot;                            // framed record: 12-byte header, payload, 4-byte footer
  // ---- entries ----
  if (active) {
    for (uint32_t f = wid; f < nf; f += ENC_TILE_WARPS) {
      const uint32_t V = vsz[f * 32 + lane];
      if (V == 0xffffu) continue;                                  // null: the feature is omitted (:29)
      const DevField& fd = sfd[f];
      const EncCol& c = scol[f];
      uint8_t* p = rec + 12 + ghdr + eoff[f * 32 + lane];
      const uint32_t E = 1 + vsize32(fd.name_len) + fd.name_len + 1 + vsize32(V) + V;
      *p++ = 0x0A; p = put_varint(p, E);
      *p++ = 0x0A; p = put_varint(p, fd.name_len);
      const uint8_t* nm = snames + fd.name_off;
      for (uint32_t k = 0; k < fd.name_len; ++k) p[k] = nm[k];
      p += fd.name_len;
      *p++ = 0x12; p = put_varint(p, V);
      if (fd.depth == 0) emit_feature(p, fd, c, (int32_t)row, (int32_t)row + 1);
      else emit_feature(p, fd, c, c.off[0][row], c.off[0][row + 1]);
    }
    if (wid == 0) {                                                // wrapper: setFeatures is always called (:33)
      uint8_t* p = rec + 12;
      *p++ = 0x0A; put_varint(p, G);
    }
  }
  __syncthreads();
  // ---- CRC-32C of the payload: every warp folds a share of the 16-byte chunks of record `lane` ----
  Tile T;
  T.b = slots;
  T.s = smem_u32(slots);
  const uint32_t pay = lane * A.slot + 12;                         // 4-byte aligned
  const uint32_t K = plen >> 4;
  if (active) {
    const uint32_t k0 = K * wid / ENC_TILE_WARPS, k1 = K * (wid + 1) / ENC_TILE_WARPS;
    uint32_t c = wid == 0 ? 0xFFFFFFFFu : 0u;
    for (uint32_t k = k0; k < k1; ++k) {
      const uint32_t o = pay + 16 * k;
      const uint32_t w0 = T.w32(o), w1 = T.w32(o + 4), w2 = T.w32(o + 8), w3 = T.w32(o + 12);
      c = crc_fold8(g5, c, w0, w1);
      c = crc_fold8(g5, c, w2, w3);
    }
    if (c) atomicXor(&scrc[lane], K - k1 ? gf2_mulmod(xp16[K - k1], c) : c);
  }
  __syncthreads();
  if (wid == 0 && active) {
    uint32_t c = scrc[lane];
    for (uint32_t o = pay + 16 * K; o < pay + plen; ++o) c = crc_byte(g5, c, T.u8(o));
    const uint32_t fc = crc_mask(~c);
    const uint32_t hc = crc_mask(~crc_fold8(g5, 0xFFFFFFFFu, plen, 0u));
    uint32_t* h = reinterpret_cast<uint32_t*>(rec);                // the slot is 4-byte aligned
    h[0] = plen; h[1] = 0; h[2] = hc;
    uint8_t* ft = rec + 12 + plen;
    for (int i = 0; i < 4; ++i) ft[i] = (uint8_t)(fc >> (8 * i));
  }
  __syncthreads();
  // ---- copy-out: whole records, 128 consecutive bytes per instruction (the output position decides the word alignment) ----
  for (uint32_t r = wid; r < rows; r += ENC_TILE_WARPS) {
    const uint32_t g0 = (uint32_t)A.rec_off[row0 + r], flen = (uint32_t)A.rec_off[row0 + r + 1] - g0;
    const uint32_t s0 = r * A.slot;                                // 4-byte aligned
    uint8_t* d = A.out + g0;
    const uint32_t hm = min(flen, (0u - (uint32_t)reinterpret_cast<uintptr_t>(d)) & 3u);
    if (lane < hm) d[lane] = (uint8_t)T.u8(s0 + lane);
    const uint32_t words = (flen - hm) >> 2;
    const uint32_t so = s0 + hm, sh = (so & 3u) * 8u, sa = so & ~3u;
    uint32_t* dw = reinterpret_cast<uint32_t*>(d + hm);
    if (sh == 0) for (uint32_t i = lane; i < words; i += 32) dw[i] = T.w32(sa + 4 * i);
    else for (uint32_t i = lane; i < words; i += 32) dw[i] = __funnelshift_r(T.w32(sa + 4 * i), T.w32(sa + 4 * i + 4), sh);   // (reads at most 3 bytes past the record: inside its slot)
    const uint32_t tl = (flen - hm) & 3u;
    if (lane < tl) d[hm + 4 * words + lane] = (uint8_t)T.u8(so + 4 * words + lane);
  }
}
