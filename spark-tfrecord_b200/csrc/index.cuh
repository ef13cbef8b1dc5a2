// index.cuh -- the record index (include/tfrgpu.h, RECORD INDEX): checkpoints from a block's frame index (frame.cuh).
//
// A checkpoint k is (offset, entry) of the first frame whose header offset is >= k * stride.  Frame i is that frame for exactly
// the slots k with o[i-1] < k * stride <= o[i], so one thread per frame writes its own slots: the slot index is k, and no scan
// over the frames is needed.
#pragma once
#include "common.cuh"
#include "frame.cuh"

struct IndexCheckpoint {
  unsigned long long offset, entry;
};

// The checkpoints of one block.  Frame i (i < n = fr->n_records) has file offset base + rec_off[i] and entry e_base + i;
// the frame in front of frame 0 is at file offset `prev` (the last frame of the blocks before, -1 when there is none).  With
// `sentinel`, thread n stands for the end of the file (offset `end`, entry e_base + n) and fills the slots behind the last
// frame.  Slot k is written to out[k - k0] when k - k0 < k_cap; the host sizes k_cap to the slots the block can own.
__global__ void __launch_bounds__(256) index_checkpoint_kernel(const uint32_t* __restrict__ rec_off, const FrameResult* __restrict__ fr,
                                                               unsigned long long base, unsigned long long e_base, long long prev,
                                                               uint32_t log2_stride, unsigned long long end, uint32_t sentinel,
                                                               unsigned long long k0, unsigned long long k_cap, IndexCheckpoint* __restrict__ out) {
  const uint32_t n = fr->n_records;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n || (i == n && !sentinel)) return;
  const unsigned long long o = i < n ? base + rec_off[i] : end;
  const long long before = i == 0 ? prev : (long long)(base + rec_off[i - 1]);
  const unsigned long long k_lo = before < 0 ? 0ull : ((unsigned long long)before >> log2_stride) + 1ull;
  const unsigned long long k_hi = o >> log2_stride;                  // k * stride <= o
  const IndexCheckpoint c{o, e_base + i};
  for (unsigned long long k = k_lo; k <= k_hi && k - k0 < k_cap; ++k) out[k - k0] = c;
}

// tfr_index_seek on the device: out[0] = the frames of the block whose offset is below `target` (a lower bound over the sorted
// rec_off), out[1] = the offset of the first frame at or after it (the stop position when every frame is below it), out[2] =
// the length field of the header the chain stopped on when that header verified and its frame runs past the block.
__global__ void index_seek_kernel(const uint8_t* __restrict__ data, const uint32_t* __restrict__ rec_off, const FrameResult* __restrict__ fr,
                                  uint32_t target, unsigned long long* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const uint32_t n = fr->n_records;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (rec_off[mid] < target) lo = mid + 1; else hi = mid;
  }
  out[0] = lo;
  out[1] = lo < n ? rec_off[lo] : fr->stop_pos;
  out[2] = fr->stop == FS_PART_REC ? load_u32_unaligned(data + fr->stop_pos) : 0u;
}
