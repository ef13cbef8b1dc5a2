// resync.cuh -- TFR_F_RESYNC: after a framing error at offset o, the first position p > o where the frame chain can go on.
//
// TFRecord has no sync marker, but every frame carries two CRC-32Cs, so a frame whose length CRC and payload CRC both verify
// can be found again.  A RESYNC POINT is a position p > o with its 12-byte header inside the block, the header predicate of the
// frame index true (frame_header_ok), its whole frame [p, p + 16 + L) inside the block, its payload CRC verified, and
// p + 16 + L - o <= H (RESYNC_HORIZON, the largest block a decoder takes).  On a block that is not the file's last, a position
// is UNDECIDED when more bytes could still make it a resync point: its header is incomplete (p + 12 > end), or its header
// verifies and its frame runs past the block's end but stays within the horizon.  The scan returns the smallest DECISIVE
// position (a resync point or an undecided one): the rule of include/tfrgpu.h (TFR_F_RESYNC) and DESIGN.md section 2.
#pragma once
#include "common.cuh"
#include "frame.cuh"

#define RESYNC_HORIZON 0x7fffffffu      // H: tfr_decode takes blocks below 2 GiB
#define RESYNC_CHUNK 4096u              // candidate offsets per warp and chunk
#define RESYNC_NONE 0xffffffffu         // the result word when no position is decisive
enum { RS_POINT = 0, RS_UNDECIDED = 1 };  // the kind in the result word's low bit: (p << 1) | kind

// One warp per chunk of RESYNC_CHUNK candidate offsets in [o + 1, last] (the host bounds `last`: the last position whose
// header fits the block on a final block, the first one whose header does not on any other), chunks in ascending order over
// the grid.  32 candidates per step through the frame index's header predicate; each hit is judged in lane order, its payload
// CRC computed by the whole warp (crc_warp), and the first decisive position of the chunk goes into *result by atomicMin.  A warp
// leaves its chunk, and skips the later ones, once the result lies below where it is.
__global__ void __launch_bounds__(256) resync_scan_kernel(const uint8_t* __restrict__ data, uint32_t end, uint32_t o, uint32_t last,
                                                          uint32_t is_final, const CrcTables* __restrict__ tabs, uint32_t* result) {
  __shared__ uint32_t stab[CRC_SMEM_WORDS];
  crc_stage_tables(stab, tabs);
  __syncthreads();
  const uint32_t* t0 = CRC_T0(stab);
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  const uint32_t first = o + 1;
  if (last < first) return;
  const uint32_t n_chunks = (last - first) / RESYNC_CHUNK + 1;
  volatile uint32_t* vres = result;
  for (uint32_t k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < n_chunks; k += n_warps) {
    const uint32_t cs = first + k * RESYNC_CHUNK;
    const uint32_t ce = last - cs >= RESYNC_CHUNK ? cs + RESYNC_CHUNK - 1 : last;
    for (uint32_t p0 = cs; p0 <= ce; p0 += 32) {
      if ((p0 << 1) >= __shfl_sync(FULLMASK, *vres, 0)) return;     // a smaller decisive position is known
      const uint32_t p = p0 + lane;
      uint32_t cand = 0;                                             // 1: header hit, 2: incomplete header (not final)
      if (p <= ce) {
        if ((uint64_t)p + 12 > end) cand = 2;
        else if (frame_header_ok(t0, data, p)) cand = 1;
      }
      unsigned m = __ballot_sync(FULLMASK, cand != 0);
      while (m) {
        const uint32_t l = (uint32_t)(__ffs(m) - 1);
        m &= m - 1;
        const uint32_t q = p0 + l;
        uint32_t kind = RESYNC_NONE;
        if (__shfl_sync(FULLMASK, cand, l) == 2) {
          kind = RS_UNDECIDED;
        } else {
          const uint32_t len = load_u32_unaligned(data + q);
          const uint64_t fe = (uint64_t)q + 16 + len;              // the frame's end
          if (fe > end) {
            if (!is_final && fe - o <= RESYNC_HORIZON) kind = RS_UNDECIDED;
          } else if (fe - o <= RESYNC_HORIZON) {
            if (crc_mask(crc_warp(stab, data + q + 12, len)) == load_u32_unaligned(data + q + 12 + len)) kind = RS_POINT;
          }
        }
        if (kind != RESYNC_NONE) {                                   // (warp-uniform: every input of `kind` is)
          if (lane == 0) atomicMin(result, (q << 1) | kind);
          return;
        }
      }
    }
  }
}
