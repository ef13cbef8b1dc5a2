// drop.cuh -- DROPMALFORMED (TFR_F_DROP_MALFORMED): the failing records of a batch, listed in record order, and the kept
// frames gathered back to back for a second decode.
//
// Pass 1 of the general path (decode.cuh) writes a status for every record of the batch.  In drop mode the host lists the
// failing ones (drop_count_kernel + drop_list_kernel: an order-preserving compaction of the status array), cuts their
// frames out and copies the frames around them, run by run, into one buffer (frame_gather_kernel).  That buffer holds only
// records that decode cleanly, so the ordinary decode of it -- the tile kernel as a rule -- gives the batch's rows.
#pragma once
#include "common.cuh"

// one dropped record: its frame index in the batch, its frame [off, end) in the batch's bytes, its pass-1 status (the status
// word of common.cuh: make_status, status_code, status_field, DF_REGION)
struct DroppedFrame { uint32_t row, off, end, status; };
static_assert(sizeof(DroppedFrame) == 16, "DroppedFrame layout");

#define DROP_THREADS 256

// the failing records of each CTA's segment [blockIdx.x * seg, + seg) of the batch's n records
__global__ void __launch_bounds__(DROP_THREADS) drop_count_kernel(const uint32_t* __restrict__ status, uint32_t n, uint32_t seg,
                                                                 uint32_t* __restrict__ seg_count) {
  __shared__ uint32_t s_w[DROP_THREADS / 32];
  const uint32_t lo = blockIdx.x * seg, hi = min(n, lo + seg);
  uint32_t c = 0;
  for (uint32_t i = lo + threadIdx.x; i < hi; i += DROP_THREADS) c += status[i] != 0u;
  c = __reduce_add_sync(FULLMASK, c);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < DROP_THREADS / 32; ++w) t += s_w[w];
    seg_count[blockIdx.x] = t;
  }
}

// Each CTA writes its segment's failing records at the place the segments before it leave free, in record order: *n_out
// (written by the last CTA) is the total, entries past `cap` are counted but not written.
__global__ void __launch_bounds__(DROP_THREADS) drop_list_kernel(const uint32_t* __restrict__ status, const uint32_t* __restrict__ rec_off,
                                                                uint32_t n, uint32_t seg, const uint32_t* __restrict__ seg_count, uint32_t cap,
                                                                DroppedFrame* __restrict__ out, uint32_t* __restrict__ n_out) {
  __shared__ uint32_t s_w[DROP_THREADS / 32];
  __shared__ uint32_t s_base;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t b = 0;
  for (uint32_t g = threadIdx.x; g < blockIdx.x; g += DROP_THREADS) b += seg_count[g];
  b = __reduce_add_sync(FULLMASK, b);
  if (lane == 0) s_w[wid] = b;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < DROP_THREADS / 32; ++w) t += s_w[w];
    s_base = t;
    if (blockIdx.x == gridDim.x - 1) *n_out = t + seg_count[blockIdx.x];
  }
  __syncthreads();
  uint32_t base = s_base;
  const uint32_t lo = blockIdx.x * seg, hi = min(n, lo + seg);
  for (uint32_t i0 = lo; i0 < hi; i0 += DROP_THREADS) {            // (the same trip count in every thread)
    const uint32_t i = i0 + threadIdx.x;
    const uint32_t st = i < hi ? status[i] : 0u;
    const unsigned m = __ballot_sync(FULLMASK, st != 0u);
    __syncthreads();                                                 // s_w of the previous step has been read
    if (lane == 0) s_w[wid] = __popc(m);
    __syncthreads();
    uint32_t before = 0, total = 0;
    for (uint32_t w = 0; w < DROP_THREADS / 32; ++w) { const uint32_t c = s_w[w]; before += w < wid ? c : 0u; total += c; }
    if (st) {
      const uint32_t k = base + before + __popc(m & ((1u << lane) - 1u));
      if (k < cap) out[k] = DroppedFrame{i, rec_off[i], rec_off[i + 1], st};
    }
    base += total;
  }
}

// a piece of a run of kept frames: `len` bytes from src + `src` to dst + `dst` (the host cuts runs into pieces of at most
// GATHER_PIECE bytes, so that one long run -- a block with a single bad record -- still spreads over every SM)
struct GatherPiece { uint32_t src, dst, len; };
#define GATHER_PIECE (64u << 10)

// One CTA per piece.  The destination is written in aligned 16-byte stores; the source is read as uint4 when it has the
// same alignment, as aligned 4-byte words otherwise (funnel-shifted when it is not 4-byte aligned either).  Every word read
// holds at least one byte of the piece, so no byte outside the batch's frames is touched.
__global__ void __launch_bounds__(256) frame_gather_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                          const GatherPiece* __restrict__ pieces, uint32_t n_pieces) {
  for (uint32_t p = blockIdx.x; p < n_pieces; p += gridDim.x) {
    const GatherPiece g = pieces[p];
    const uint8_t* s = src + g.src;
    uint8_t* d = dst + g.dst;
    const uint32_t head = min(g.len, (uint32_t)((16u - (reinterpret_cast<uintptr_t>(d) & 15u)) & 15u));
    if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
    const uint32_t n16 = (g.len - head) >> 4;
    const uint8_t* s2 = s + head;
    uint4* d2 = reinterpret_cast<uint4*>(d + head);
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(s2) & 15u);
    if (mis == 0) {
      const uint4* q = reinterpret_cast<const uint4*>(s2);
      for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) d2[i] = q[i];
    } else if ((mis & 3u) == 0) {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(s2);
      for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) d2[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
    } else {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(s2) & ~(uintptr_t)3);
      const uint32_t sh = (mis & 3u) * 8u;
      for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) {
        const uint32_t w0 = w[4 * i], w1 = w[4 * i + 1], w2 = w[4 * i + 2], w3 = w[4 * i + 3], w4 = w[4 * i + 4];
        d2[i] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
      }
    }
    for (uint32_t i = head + n16 * 16u + threadIdx.x; i < g.len; i += blockDim.x) d[i] = s[i];
  }
}
