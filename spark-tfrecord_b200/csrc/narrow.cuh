// narrow.cuh -- BooleanType, ByteType, ShortType, DateType and TimestampType fields (include/tfrgpu.h, INT64 TYPES).
//
// Such a field is a LongType field to every parse and encode kernel.  These two kernels convert its leaf values at the edges:
//   narrow_kernel : after a decoded batch's columns are final, every narrowed column's int64 leaf values into the narrow type
//                   (and a boolean's bit-packed values, which the Arrow exports hand out), in the batch's output block.  One
//                   launch covers up to NARROW_MAX columns (blockIdx.y); the value count is read on the device from the column's
//                   offsets, so a pipelined batch needs no host synchronisation.  A timestamp's int64 values are its own.
//   widen_kernel  : tfr_encode's columns of these types, narrow leaf values into int64 in the encoder's scratch.
#pragma once
#include "common.cuh"

#define NARROW_MAX 64
#define NARROW_THREADS 256

// bytes per leaf value of a TFR_T_BOOL .. TFR_T_TIMESTAMP column; 0 for every other type
__host__ __device__ __forceinline__ int nar_width(int t) {
  switch (t) {
    case TFR_T_BOOL: case TFR_T_INT8: return 1;
    case TFR_T_INT16: return 2;
    case TFR_T_DATE: return 4;
    case TFR_T_TIMESTAMP: return 8;
    default: return 0;
  }
}
// where a boolean column's bit-packed values start behind its bytes, for `cap` values
__host__ __device__ __forceinline__ size_t nar_bits_at(uint64_t cap) { return (size_t)((cap + 15) & ~15ull); }

struct NarrowCol {
  const long long* src;         // the LongType column's leaf values
  uint8_t* dst;                 // the narrow values (a boolean: bytes, then its bits at nar_bits_at(cap))
  const int32_t* off0;          // null: a scalar (one value per row); else the column's offsets levels
  const int32_t* off1;          // depth 2: the inner level, else null
  uint32_t cap;                 // values dst holds
  uint32_t cap1;                // depth 2: inner lists off1 indexes (entries - 1)
  int32_t type;                 // TFR_T_BOOL .. TFR_T_DATE
  int32_t pad;
};
struct NarrowArgs {
  NarrowCol c[NARROW_MAX];
  uint32_t n_cols, n;           // n: the rows (a pipelined batch: its capacity, the count read from n_dev)
  const uint32_t* n_dev;
};

__device__ __forceinline__ long long nar_clamp(long long v, long long hi) { return v < 0 ? 0 : v > hi ? hi : v; }

__global__ void __launch_bounds__(NARROW_THREADS) narrow_kernel(NarrowArgs A) {
  const NarrowCol& C = A.c[blockIdx.y];
  const uint32_t n = A.n_dev ? min(A.n, *A.n_dev) : A.n;
  long long m = n;
  if (C.off0) {
    m = C.off0[n];
    if (C.off1) m = C.off1[nar_clamp(m, C.cap1)];
  }
  m = nar_clamp(m, C.cap);
  const uint32_t lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * NARROW_THREADS; base < m; base += (long long)gridDim.x * NARROW_THREADS) {
    const long long i = base + threadIdx.x;
    const bool on = i < m;
    const long long v = on ? C.src[i] : 0;
    if (C.type == TFR_T_BOOL) {
      const bool b = v != 0;
      if (on) C.dst[i] = b ? 1 : 0;
      const uint32_t w = __ballot_sync(FULLMASK, b);
      if (lane == 0 && i < m) reinterpret_cast<uint32_t*>(C.dst + nar_bits_at(C.cap))[i >> 5] = w;
    } else if (on) {
      if (C.type == TFR_T_INT8) C.dst[i] = (uint8_t)v;
      else if (C.type == TFR_T_INT16) reinterpret_cast<uint16_t*>(C.dst)[i] = (uint16_t)v;
      else reinterpret_cast<uint32_t*>(C.dst)[i] = (uint32_t)v;
    }
  }
}

struct WidenCol {
  const uint8_t* src;           // the caller's narrow leaf values
  long long* dst;
  unsigned long long n;         // leaf values
  int32_t type;
  int32_t pad;
};
struct WidenArgs { WidenCol c[NARROW_MAX]; uint32_t n_cols; };

__global__ void __launch_bounds__(NARROW_THREADS) widen_kernel(WidenArgs A) {
  const WidenCol& C = A.c[blockIdx.y];
  for (unsigned long long i = (unsigned long long)blockIdx.x * NARROW_THREADS + threadIdx.x; i < C.n; i += (unsigned long long)gridDim.x * NARROW_THREADS) {
    long long v;
    if (C.type == TFR_T_BOOL) v = C.src[i] != 0;
    else if (C.type == TFR_T_INT8) v = (int8_t)C.src[i];
    else if (C.type == TFR_T_INT16) v = reinterpret_cast<const int16_t*>(C.src)[i];
    else v = reinterpret_cast<const int32_t*>(C.src)[i];
    C.dst[i] = v;
  }
}
