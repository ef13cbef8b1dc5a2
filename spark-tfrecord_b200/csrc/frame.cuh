// frame.cuh -- K1: TFRecord record-boundary index, built on the GPU.
//
// Replaces the sequential framing scan of tensorflow-hadoop's TFRecordReader.read (called from
// M/TFRecordFileReader.scala:51): off[i+1] = off[i] + 16 + len[i] is a serial pointer chase, which
// is why the reference declares files unsplittable (M/DefaultSource.scala:26-29).  Here the chase
// is parallelised by SPECULATION + EXACT VERIFICATION:
//   1. frame_scan   : the buffer is cut into chunks; one warp per chunk looks for the first byte
//                     offset whose 12-byte header is self-consistent (masked CRC-32C of the 8
//                     length bytes == the stored CRC; 32 candidates per step, __ballot_sync picks
//                     the first hit) and chains headers from there until it leaves the chunk.
//   2. frame_check  : chunk k's guess is right iff chunk k-1's chain ended exactly on it
//                     (induction from offset 0, which is a record start by contract).
//   3. frame_repair : only when a link is broken (a record larger than a chunk, payloads that
//                     themselves contain TFRecord streams, corruption): one warp re-chains the
//                     affected chunks sequentially from the true position -- always exact.
//   4. chunk counts are prefix-summed and frame_emit re-walks each chunk writing rec_off[].
// Four launches per batch: frame_search (candidates, also resets the result block), frame_scan (chains),
// frame_link (one block: link check + repair + stop + count prefix + result; steps 2-4 above) and frame_emit.
// The result is identical to the sequential scan for every input, including the error cases
// (bad length CRC, truncated tail, oversize length) which are reported at the first bad record.
#pragma once
#include "common.cuh"

#define FRAME_STAGE 256u      // record offsets staged per chunk by the chain walk (frame_emit copies them; longer chains are re-walked)

// how a chunk's chain (or the whole stream) stopped
enum {
  FS_LEFT = 0,        // walked past the end of the chunk: `end` is the next record start
  FS_EOF = 1,         // ended exactly at nbytes
  FS_STRAY = 2,       // 1..7 bytes left: TFRecordReader.read catches the EOFException -> clean EOF
  FS_PART_HDR = 3,    // 8..11 bytes left: EOF while reading the length CRC -> TRUNCATED
  FS_PART_REC = 4,    // header ok, payload/footer runs past nbytes -> TRUNCATED
  FS_BAD_CRC = 5,     // length CRC mismatch
  FS_TOO_LARGE = 6,   // length > Integer.MAX_VALUE
  FS_NONE = 7         // no candidate header in this chunk
};

struct ChunkInfo {
  uint32_t first;   // offset of the first record that starts in this chunk (0xffffffff none)
  uint32_t end;     // where the chain stopped (next record start, or the stop position)
  uint32_t count;   // complete, header-valid records that start in this chunk
  uint32_t stop;    // FS_*
};

struct FrameResult {       // written by the device, read back by the host (one small D2H)
  uint32_t n_records;      // complete records before the stop
  uint32_t stop;           // FS_EOF / FS_STRAY / FS_PART_HDR / FS_PART_REC / FS_BAD_CRC / FS_TOO_LARGE
  uint32_t stop_pos;       // byte offset of the record (or fragment) that stopped the scan
  uint32_t repairs;        // chunks re-chained by frame_repair
  uint32_t first_bad;      // first chunk whose link check failed, 0xffffffff if none
  uint32_t max_len;        // upper bound of the payload length of any record (sizes the shared-memory tiles)
  uint32_t pad[2];
};

// walk headers starting at q until the chain leaves [.., ce) or stops; returns stop code
__device__ __forceinline__ uint32_t frame_chain(const uint32_t* t0, const uint8_t* data, uint32_t nbytes, uint32_t ce,
                                                bool verify, uint32_t& q, uint32_t& count, uint32_t& max_len, uint32_t* stage = nullptr) {
  while (q < ce) {
    uint32_t left = nbytes - q;
    if (left < 8) return FS_STRAY;
    if (left < 12) return FS_PART_HDR;
    uint32_t lo = load_u32_unaligned(data + q), hi = load_u32_unaligned(data + q + 4);
    if (verify) {
      uint32_t crc = load_u32_unaligned(data + q + 8);
      if (crc_mask(crc_u64(t0, lo, hi)) != crc) return FS_BAD_CRC;
    }
    if (hi != 0 || lo > 0x7fffffffu) return FS_TOO_LARGE;
    if ((uint64_t)left < 16ull + lo) return FS_PART_REC;
    if (stage && count < FRAME_STAGE) stage[count] = q;
    q += 16 + lo;
#ifndef FRAME_NO_PREFETCH
    // the chain is a DRAM-latency-bound pointer chase; records of a file tend to have similar sizes, so the headers two
    // and three records ahead are probably near q + k*(16 + lo): ask L2 for those lines now
    {
      const uint32_t step = 16 + lo;
      if (step < 0x100000u) {
        const uint32_t a1 = q + step, a2 = a1 + step;
        if (a2 + 64 < nbytes) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(data + a1));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(data + a2));
        }
      }
    }
#endif
    max_len = max(max_len, lo);
    ++count;
  }
  return q == nbytes ? FS_EOF : FS_LEFT;
}

// a plausible header at p (its 12 bytes inside the buffer): the upper half of the length is zero (the cheapest test, first),
// the length fits an int32 and the stored CRC matches the masked CRC-32C of the 8 length bytes.  The candidate search below
// and resync_scan_kernel (resync.cuh) look for record starts with it.
__device__ __forceinline__ bool frame_header_ok(const uint32_t* t0, const uint8_t* data, uint32_t p) {
  if (load_u32_unaligned(data + p + 4) != 0) return false;
  const uint32_t lo = load_u32_unaligned(data + p);
  return lo <= 0x7fffffffu && crc_mask(crc_u64(t0, lo, 0)) == load_u32_unaligned(data + p + 8);
}

// K1a -- candidate search, one WARP per chunk: 32 consecutive candidate offsets per step (coalesced: the warp's
// loads fall into one or two sectors), cheapest condition first (the upper half of a plausible length is zero),
// __ballot_sync picks the first hit.  The first 2 KiB of the chunk are prefetched by 16 lanes up front so the
// steps hit L1 instead of paying one dependent DRAM miss per 128-byte line.
__global__ void __launch_bounds__(256) frame_search_kernel(const uint8_t* __restrict__ data, uint32_t nbytes, uint32_t chunk_bytes,
                                                           uint32_t n_chunks, const CrcTables* __restrict__ tabs, uint32_t* __restrict__ first_out,
                                                           uint32_t* __restrict__ reset_words, uint32_t n_reset) {
  __shared__ uint32_t t0[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) t0[i] = tabs->t0[i];
  // block 0 also resets the per-batch result block (FrameResult, tile flags, null counters ...) that the later kernels of
  // this batch accumulate into: one launch less than a memset, and stream order puts it in front of all of them
  if (blockIdx.x == 0) for (uint32_t i = threadIdx.x; i < n_reset; i += blockDim.x) reset_words[i] = 0u;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps_per_block = blockDim.x >> 5;
  for (uint32_t k = blockIdx.x * warps_per_block + (threadIdx.x >> 5); k < n_chunks; k += gridDim.x * warps_per_block) {
    const uint32_t cs = k * chunk_bytes;
    const uint32_t ce = (nbytes - cs > chunk_bytes) ? cs + chunk_bytes : nbytes;
    uint32_t first = 0xffffffffu;
    if (k == 0) first = 0;
    else if (nbytes - cs >= 12) {
      // a candidate p is plausible iff its 12-byte header is inside the buffer, the stored CRC matches the masked
      // CRC-32C of the 8 length bytes and the length fits an int32 (false positive 2^-32 per byte on random data;
      // adversarial data is caught by frame_check and fixed by frame_repair)
      const uint32_t last = min(ce - 1, nbytes - 12);
      for (uint32_t p0 = cs; p0 <= last && first == 0xffffffffu; p0 += 32) {
        if (((p0 - cs) & 2047u) == 0 && lane < 17 && p0 + 128u * lane < nbytes)
          asm volatile("prefetch.global.L1 [%0];" ::"l"(data + p0 + 128u * lane));
        const uint32_t p = p0 + lane;
        const bool hit = p <= last && frame_header_ok(t0, data, p);
        const uint32_t m = __ballot_sync(FULLMASK, hit);
        if (m) first = p0 + (uint32_t)(__ffs(m) - 1);
      }
    }
    if (lane == 0) first_out[k] = first;
  }
}

// K1b -- chain walk, one THREAD per chunk: a DRAM-latency-bound pointer chase, so the win is chains in flight.
__global__ void __launch_bounds__(128) frame_scan_kernel(const uint8_t* __restrict__ data, uint32_t nbytes, uint32_t chunk_bytes,
                                                         uint32_t n_chunks, uint32_t verify, const CrcTables* __restrict__ tabs,
                                                         const uint32_t* __restrict__ first_in, ChunkInfo* __restrict__ chunks,
                                                         uint32_t* __restrict__ stage, FrameResult* __restrict__ res) {
  __shared__ uint32_t t0[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) t0[i] = tabs->t0[i];
  __syncthreads();
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_chunks) return;
  const uint32_t cs = k * chunk_bytes;
  const uint32_t ce = (nbytes - cs > chunk_bytes) ? cs + chunk_bytes : nbytes;
  const uint32_t first = first_in[k];
  ChunkInfo ci;
  ci.first = first; ci.end = first; ci.count = 0; ci.stop = FS_NONE;
  if (first != 0xffffffffu) {
    uint32_t q = first, cnt = 0, mx = 0;
    ci.stop = frame_chain(t0, data, nbytes, ce, verify != 0, q, cnt, mx, stage + (size_t)k * FRAME_STAGE);
    ci.end = q; ci.count = cnt;
    if (mx) atomicMax(&res->max_len, mx);                                  // a false candidate can only enlarge the bound
  }
  chunks[k] = ci;
}

// K1c -- link check + repair + stop + count prefix + result, ONE block (the chunk table is a few hundred KB at most).
//   link check : chunk k (k >= 1) is consistent iff the previous chunk's chain left exactly onto its guess; a previous
//                chunk that already stopped the stream makes every later chunk irrelevant (they are cleared by the repair)
//   repair     : sequential, exact (thread 0): starts at the first broken link and re-chains until the speculation
//                re-synchronises
//   stop       : the first (and, after the repair, only) chunk whose chain did not leave the chunk
//   prefix     : chunk_base[k] = records that start before chunk k (n_chunks + 1 entries)
//   result     : FrameResult.  With `verify_stop` (the chains ran without header verification because the tile kernel
//                checks every length CRC of the records it is given) the header the stream stopped on is checked here: a
//                corrupt length must be a length-CRC error (the reference checks the CRC first), never a "partial tail"
//                or an oversize length.
__device__ __forceinline__ void frame_repair(const uint32_t* t0, const uint8_t* __restrict__ data, uint32_t nbytes, uint32_t chunk_bytes, uint32_t n_chunks,
                                             bool verify, ChunkInfo* __restrict__ chunks, uint32_t* __restrict__ stage, uint32_t first_bad,
                                             FrameResult* __restrict__ res) {
  uint32_t k = first_bad;               // >= 1
  uint32_t repairs = 0;
  ChunkInfo prev = chunks[k - 1];
  uint32_t F = prev.end;                // true position where the stream continues
  bool stopped = prev.stop != FS_LEFT;  // the stream already ended/failed in chunk k-1
  for (; k < n_chunks; ++k) {
    const uint32_t cs = k * chunk_bytes;
    const uint32_t ce = (nbytes - cs > chunk_bytes) ? cs + chunk_bytes : nbytes;
    ChunkInfo ci = chunks[k];
    if (stopped || F >= ce) {           // no record starts in this chunk
      if (ci.first != 0xffffffffu || ci.count) { ci.first = 0xffffffffu; ci.count = 0; ci.stop = FS_NONE; ci.end = F; chunks[k] = ci; ++repairs; }
      continue;
    }
    if (ci.first == F) {                // speculation is right from here on: re-synchronised
      if (ci.stop != FS_LEFT) { stopped = true; continue; }
      F = ci.end;                       // a later broken link keeps the loop going; consistent chunks are fast-forwarded
      continue;
    }
    uint32_t q = F, cnt = 0, mx = 0;
    ci.first = F;
    ci.stop = frame_chain(t0, data, nbytes, ce, verify, q, cnt, mx, stage + (size_t)k * FRAME_STAGE);
    if (mx > res->max_len) res->max_len = mx;
    ci.end = q; ci.count = cnt;
    chunks[k] = ci; ++repairs;
    if (ci.stop != FS_LEFT) stopped = true; else F = q;
  }
  res->repairs = repairs;
}

#define FRAME_LINK_THREADS 1024
__global__ void __launch_bounds__(FRAME_LINK_THREADS) frame_link_kernel(const uint8_t* __restrict__ data, uint32_t nbytes, uint32_t chunk_bytes,
                                                                        uint32_t n_chunks, uint32_t verify, uint32_t verify_stop,
                                                                        const CrcTables* __restrict__ tabs, ChunkInfo* __restrict__ chunks,
                                                                        uint32_t* __restrict__ stage, uint32_t* __restrict__ chunk_base,
                                                                        FrameResult* __restrict__ res) {
  __shared__ uint32_t t0[256];
  __shared__ uint32_t s_first_bad, s_stop_chunk, s_carry;
  __shared__ uint32_t wsum[FRAME_LINK_THREADS / 32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (uint32_t i = tid; i < 256; i += blockDim.x) t0[i] = tabs->t0[i];
  if (tid == 0) { s_first_bad = 0xffffffffu; s_stop_chunk = 0xffffffffu; s_carry = 0; }
  __syncthreads();
  if (n_chunks == 0) {
    if (tid == 0) { res->n_records = 0; res->stop = FS_EOF; res->stop_pos = 0; res->first_bad = 0xffffffffu; chunk_base[0] = 0; }
    return;
  }
  for (uint32_t k = tid + 1; k < n_chunks; k += blockDim.x) {
    const ChunkInfo prev = chunks[k - 1], cur = chunks[k];
    if (!(prev.stop == FS_LEFT && cur.first != 0xffffffffu && prev.end == cur.first)) atomicMin(&s_first_bad, k);
  }
  __syncthreads();
  if (tid == 0) {
    res->first_bad = s_first_bad;
    if (s_first_bad != 0xffffffffu) frame_repair(t0, data, nbytes, chunk_bytes, n_chunks, verify != 0, chunks, stage, s_first_bad, res);
    __threadfence_block();
  }
  __syncthreads();
  // exclusive prefix of the chunk counts + the stop chunk
  for (uint32_t base = 0; base < n_chunks; base += blockDim.x) {
    const uint32_t k = base + tid;
    uint32_t c = 0;
    if (k < n_chunks) {
      const ChunkInfo ci = chunks[k];
      c = ci.count;
      if (ci.first != 0xffffffffu && ci.stop != FS_LEFT) atomicMin(&s_stop_chunk, k);
    }
    uint32_t x = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      uint32_t w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, w, o); if (lane >= (uint32_t)o) w += y; }
      wsum[lane] = w;
    }
    __syncthreads();
    const uint32_t excl = x - c + (wid ? wsum[wid - 1] : 0u) + s_carry;
    if (k < n_chunks) chunk_base[k] = excl;
    __syncthreads();
    if (tid == blockDim.x - 1) s_carry = excl + c;
    __syncthreads();
  }
  if (tid != 0) return;
  chunk_base[n_chunks] = s_carry;
  // records that start after the stop chunk do not exist (the repair cleared them); the stop chunk is the first (and only)
  // chunk with a non-LEFT stop
  const uint32_t sc = s_stop_chunk;
  if (sc == 0xffffffffu) { res->n_records = s_carry; res->stop = FS_EOF; res->stop_pos = nbytes; return; }   // cannot happen for nbytes > 0
  const ChunkInfo ci = chunks[sc];
  uint32_t stop = ci.stop;
  if (verify_stop && (stop == FS_PART_REC || stop == FS_TOO_LARGE)) {
    const uint32_t q = ci.end;                      // >= 12 bytes are left at q for both stops
    const uint32_t lo = load_u32_unaligned(data + q), hi = load_u32_unaligned(data + q + 4);
    if (crc_mask(crc_u64(t0, lo, hi)) != load_u32_unaligned(data + q + 8)) stop = FS_BAD_CRC;
  }
  res->n_records = chunk_base[sc] + ci.count;
  res->stop = stop; res->stop_pos = ci.end;
}

// rec_off[] from the staged offsets: FRAME_EMIT_LANES threads per chunk copy (coalesced), chains longer than the
// staging capacity are re-walked from the last staged record; rec_off[n] = stop_pos
#define FRAME_EMIT_LANES 8u
__global__ void __launch_bounds__(256) frame_emit_kernel(const uint8_t* __restrict__ data, const ChunkInfo* __restrict__ chunks,
                                                         const uint32_t* __restrict__ chunk_base, uint32_t n_chunks, const uint32_t* __restrict__ stage,
                                                         const FrameResult* __restrict__ res, uint32_t* __restrict__ rec_off, uint32_t cap) {
  const uint32_t n = res->n_records;
  if (n > cap) return;                       // more records than rec_off was sized for (speculative submit): the host redoes the batch
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) rec_off[n] = res->stop_pos;
  const uint32_t k = t / FRAME_EMIT_LANES, sub = t % FRAME_EMIT_LANES;
  if (k >= n_chunks) return;
  ChunkInfo ci = chunks[k];
  if (ci.first == 0xffffffffu || ci.count == 0) return;
  const uint32_t base = chunk_base[k];
  const uint32_t* st = stage + (size_t)k * FRAME_STAGE;
  const uint32_t staged = min(ci.count, FRAME_STAGE);
  for (uint32_t i = sub; i < staged && base + i < n; i += FRAME_EMIT_LANES) rec_off[base + i] = st[i];
  if (sub == 0 && ci.count > FRAME_STAGE) {
    uint32_t q = st[FRAME_STAGE - 1];
    q += 16 + load_u32_unaligned(data + q);
    for (uint32_t i = FRAME_STAGE; i < ci.count && base + i < n; ++i) {
      rec_off[base + i] = q;
      q += 16 + load_u32_unaligned(data + q);
    }
  }
}
