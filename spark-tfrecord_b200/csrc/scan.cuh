// scan.cuh -- K4: exclusive prefix sums of many per-row count arrays in three launches
// (tile sums -> tile bases -> local scan), turning element/byte counts into Arrow int32 offsets.
#pragma once
#include "common.cuh"

#define SCAN_THREADS 256
#define SCAN_ITEMS 8
#define SCAN_TILE (SCAN_THREADS * SCAN_ITEMS)

__device__ __forceinline__ uint64_t block_reduce_u64(uint64_t v, uint64_t* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULLMASK, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  uint64_t t = 0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(FULLMASK, t, o);
    if (threadIdx.x == 0) sh[0] = t;
  }
  __syncthreads();
  t = sh[0];
  __syncthreads();
  return t;
}

// cnt: [n_arr][n]; tsum: [n_arr][n_tiles]
__global__ void __launch_bounds__(SCAN_THREADS) scan_tile_sums_kernel(const uint32_t* __restrict__ cnt, uint32_t n, uint32_t n_tiles,
                                                                      uint64_t* __restrict__ tsum) {
  __shared__ uint64_t sh[32];
  const uint32_t a = blockIdx.y, t = blockIdx.x;
  const uint32_t* src = cnt + (size_t)a * n;
  uint64_t s = 0;
  uint32_t base = t * SCAN_TILE;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    uint32_t idx = base + i * SCAN_THREADS + threadIdx.x;
    if (idx < n) s += src[idx];
  }
  s = block_reduce_u64(s, sh);
  if (threadIdx.x == 0) tsum[(size_t)a * n_tiles + t] = s;
}

// one block per array: exclusive scan of its tile sums (in place), total -> totals_raw[a]; overflow flag
__global__ void __launch_bounds__(1024) scan_tile_bases_kernel(uint64_t* __restrict__ tsum, uint32_t n_tiles, uint64_t* __restrict__ totals_raw,
                                                               uint32_t* __restrict__ overflow) {
  __shared__ uint64_t wsum[32];
  __shared__ uint64_t carry;
  const uint32_t a = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t* ts = tsum + (size_t)a * n_tiles;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_tiles; base += blockDim.x) {
    uint32_t k = base + threadIdx.x;
    uint64_t c = k < n_tiles ? ts[k] : 0, x = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      uint64_t s = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(FULLMASK, s, o); if (lane >= (uint32_t)o) s += y; }
      wsum[lane] = s;
    }
    __syncthreads();
    uint64_t excl = x - c + (wid ? wsum[wid - 1] : 0) + carry;
    if (k < n_tiles) ts[k] = excl;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + c;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    totals_raw[a] = carry;
    if (carry > 0x7fffffffull) atomicOr(overflow, 1u);
  }
}

// Local scan of tile t of array a into dst (n+1 entries of Out), summing in Acc: uint32_t for int32 Arrow offsets (the
// totals were checked against int32 by scan_tile_bases_kernel), uint64_t for int64 offsets of totals beyond 4 GiB.
template <typename Out, typename Acc>
__device__ __forceinline__ void scan_apply_tile(const uint32_t* __restrict__ cnt, uint32_t n, uint32_t n_tiles, const uint64_t* __restrict__ tbase,
                                                const uint64_t* __restrict__ totals_raw, Out* dst) {
  __shared__ Acc wsum[SCAN_THREADS / 32];
  const uint32_t a = blockIdx.y, t = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t* src = cnt + (size_t)a * n;
  // thread owns SCAN_ITEMS consecutive elements
  uint32_t base = t * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS];
  Acc s = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { v[i] = base + i < n ? src[base + i] : 0; s += v[i]; }
  Acc x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { Acc y = __shfl_up_sync(FULLMASK, x, o); if (lane >= (uint32_t)o) x += y; }
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    Acc w = lane < SCAN_THREADS / 32 ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) { Acc y = __shfl_up_sync(FULLMASK, w, o); if (lane >= (uint32_t)o) w += y; }
    if (lane < SCAN_THREADS / 32) wsum[lane] = w;
  }
  __syncthreads();
  Acc run = x - s + (wid ? wsum[wid - 1] : 0) + (Acc)tbase[(size_t)a * n_tiles + t];
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) {
    if (base + i < n) dst[base + i] = (Out)run;
    run += v[i];
  }
  if (t == n_tiles - 1 && threadIdx.x == 0) dst[n] = (Out)(Acc)totals_raw[a];
}

// out[a]: n+1 int32 entries
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(const uint32_t* __restrict__ cnt, uint32_t n, uint32_t n_tiles,
                                                                  const uint64_t* __restrict__ tbase, const uint64_t* __restrict__ totals_raw,
                                                                  int32_t* const* __restrict__ out) {
  scan_apply_tile<int32_t, uint32_t>(cnt, n, n_tiles, tbase, totals_raw, out[blockIdx.y]);
}
// out: n+1 int64 entries (one array)
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply64_kernel(const uint32_t* __restrict__ cnt, uint32_t n, uint32_t n_tiles,
                                                                    const uint64_t* __restrict__ tbase, const uint64_t* __restrict__ totals_raw,
                                                                    int64_t* __restrict__ out) {
  scan_apply_tile<int64_t, uint64_t>(cnt, n, n_tiles, tbase, totals_raw, out);
}
