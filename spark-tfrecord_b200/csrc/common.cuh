// common.cuh -- device-side primitives shared by the frame index, decode and encode kernels.
//
// sm_90a (H100) only.  Everything here is integer/byte work bounded by HBM bandwidth and issue
// slots; there is deliberately no tensor-core code (nothing on this path is a contraction).
//
// Reference shorthand: M/ = src/main/scala/com/linkedin/spark/datasources/tfrecord/
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tfrgpu.h"

#define TFR_WARP 32
#define FULLMASK 0xffffffffu

// ---------------------------------------------------------------------------------------------
// CRC-32C (Castagnoli, reflected 0x82F63B78) tables, built once on the host (api.cu) and copied
// to device global memory; kernels stage them into shared memory.
//   t0[256]      : byte-at-a-time table
//   k128[4][256] : "advance the register over 128 zero bytes" as 4 byte-sliced tables, used by the
//                  lane-strided Horner step (each lane owns every 32nd 4-byte word = 128 B apart)
//   xw[33]       : x^(32k) mod P, k = 0..32, to shift a lane's partial to the end of the buffer
// ---------------------------------------------------------------------------------------------
struct CrcTables {
  uint32_t t0[256];
  uint32_t k128[4][256];
  uint32_t xw[40];
  uint32_t s8[8][256];   // slicing-by-8 tables (source of the 5-bit tables below; the tile kernels use g5)
  // tile.cuh: the 8-byte fold through 5-BIT tables.  A 32-entry table is one word per shared-memory bank, so a lookup
  // is conflict-free whatever the 32 lanes index (a 256-entry table costs ~3 wavefronts per lookup with random bytes).
  //   g5[k*32 + v], k = 0..12: contribution of bits 5k..5k+4 (= v) of the 64-bit block to the state 8 bytes later
  //   g5[416 + v], g5[448 + w]: the byte-wise table split the same way, t0[x] = g5[416 + (x & 31)] ^ g5[448 + (x >> 5)]
  uint32_t g5[512];
  uint32_t xp16[512];    // x^(8*16*m) mod P: shifts a CRC state over m later 16-byte chunks (contiguous with g5)
  uint32_t x8pow[32];    // x^(8 * 2^k) mod P: shifts over any number of bytes as a product over its set bits (large.cuh)
};
#define CRC_SMEM_WORDS (256 + 1024 + 40)

__device__ __forceinline__ void crc_stage_tables(uint32_t* s, const CrcTables* __restrict__ g) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
  for (int i = threadIdx.x; i < CRC_SMEM_WORDS; i += blockDim.x) s[i] = src[i];
}
#define CRC_T0(s) (s)
#define CRC_K128(s) ((s) + 256)
#define CRC_XW(s) ((s) + 256 + 1024)

__device__ __forceinline__ uint32_t crc_mask(uint32_t c) { return ((c >> 15) | (c << 17)) + 0xa282ead8u; }

// GF(2) polynomial multiply mod P, reflected bit order (bit 31 = x^0)
__device__ __forceinline__ uint32_t gf2_mulmod(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll
  for (int i = 31; i >= 0; --i) {
    p ^= b & (0u - ((a >> i) & 1u));
    b = (b >> 1) ^ (0x82F63B78u & (0u - (b & 1u)));
  }
  return p;
}

// one thread, n bytes, generic pointer (used for the 8-byte length header and short payloads)
__device__ __forceinline__ uint32_t crc_bytes_serial(const uint32_t* t0, const uint8_t* p, uint32_t n, uint32_t state) {
  for (uint32_t i = 0; i < n; ++i) state = (state >> 8) ^ t0[(state ^ p[i]) & 0xff];
  return state;
}
// CRC of the 8 length bytes given as two LE words
__device__ __forceinline__ uint32_t crc_u64(const uint32_t* t0, uint32_t lo, uint32_t hi) {
  uint32_t c = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < 4; ++i) { c = (c >> 8) ^ t0[(c ^ lo) & 0xff]; lo >>= 8; }
#pragma unroll
  for (int i = 0; i < 4; ++i) { c = (c >> 8) ^ t0[(c ^ hi) & 0xff]; hi >>= 8; }
  return ~c;
}

// 4 bytes at an arbitrary byte address through aligned 32-bit loads (global or shared)
__device__ __forceinline__ uint32_t load_u32_unaligned(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  uint32_t sh = (uint32_t)(a & 3) * 8;
  uint32_t lo = w[0];
  if (sh == 0) return lo;
  return __funnelshift_r(lo, w[1], sh);
}

// Whole-warp CRC-32C of data[0..n).  All 32 lanes must call with identical arguments.
// Lane l folds words l, l+32, l+64, ... (coalesced 128-byte rows) with
//     r = Adv128(r) ^ w
// then shifts its partial by the number of words that follow its last word and the lanes are
// XOR-reduced; the 0..3 tail bytes are folded serially.  Unaligned starts are handled with
// aligned loads + funnel shifts (the word one past the end is never dereferenced beyond the
// 4-byte aligned word that contains the last payload byte).
__device__ __forceinline__ uint32_t crc_warp(const uint32_t* stab, const uint8_t* data, uint32_t n) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t* t0 = CRC_T0(stab);
  if (n < 4) return ~crc_bytes_serial(t0, data, n, 0xFFFFFFFFu);
  const uint32_t* k0 = CRC_K128(stab);
  const uint32_t W = n >> 2;
  uintptr_t a = reinterpret_cast<uintptr_t>(data);
  const uint32_t* base = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  // aligned words available: the last payload byte lives in aligned word index `last_aw`
  const uint32_t last_aw = (uint32_t)(((a & 3) + n - 1) >> 2);
  uint32_t r = 0;
  int32_t jl = -1;
  uint32_t cur = (lane <= last_aw) ? base[lane] : 0u;
  for (uint32_t j0 = 0; j0 < W; j0 += 32) {
    uint32_t nidx = j0 + 32 + lane;
    uint32_t nxt = (nidx <= last_aw) ? base[nidx] : 0u;
    uint32_t up = __shfl_down_sync(FULLMASK, cur, 1);
    uint32_t n0 = __shfl_sync(FULLMASK, nxt, 0);
    if (lane == 31) up = n0;
    uint32_t w = sh ? __funnelshift_r(cur, up, sh) : cur;
    uint32_t j = j0 + lane;
    if (j < W) {
      if (j == 0) w ^= 0xFFFFFFFFu;
      r = k0[r & 0xff] ^ k0[256 + ((r >> 8) & 0xff)] ^ k0[512 + ((r >> 16) & 0xff)] ^ k0[768 + (r >> 24)] ^ w;
      jl = (int32_t)j;
    }
    cur = nxt;
  }
  uint32_t part = 0;
  if (jl >= 0) part = gf2_mulmod(CRC_XW(stab)[W - (uint32_t)jl], r);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part ^= __shfl_xor_sync(FULLMASK, part, o);
  uint32_t c = crc_bytes_serial(t0, data + (size_t)W * 4, n & 3, part);
  return ~c;
}

// ---------------------------------------------------------------------------------------------
// warp-wide exclusive prefix sum over the lanes (+ the total)
__device__ __forceinline__ uint32_t warp_excl_scan_u32(uint32_t v, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
  total = __shfl_sync(0xffffffffu, x, 31);
  return x - v;
}

// protobuf wire primitives (protobuf-java CodedInputStream semantics, see oracle/tfr_oracle.c)
// ---------------------------------------------------------------------------------------------
struct Cur {
  const uint8_t* p;
  const uint8_t* end;
};

// readRawVarint64: <= 10 bytes, low 64 bits kept; false = truncated or malformed
__device__ __forceinline__ bool rd_varint64(Cur& c, uint64_t& out) {
  uint64_t v = 0;
#pragma unroll 1
  for (int i = 0; i < 10; ++i) {
    if (c.p >= c.end) return false;
    uint32_t b = *c.p++;
    v |= (uint64_t)(b & 0x7f) << (7 * i);   // i == 9: only bit 63 survives the shift
    if (!(b & 0x80)) { out = v; return true; }
  }
  return false;
}
// fast path for the very common 1- and 2-byte varints (tags, short lengths)
__device__ __forceinline__ bool rd_varint32(Cur& c, uint32_t& out) {
  if (c.p < c.end) {
    uint32_t b = *c.p;
    if (b < 0x80) { ++c.p; out = b; return true; }
  }
  uint64_t v;
  if (!rd_varint64(c, v)) return false;
  out = (uint32_t)v;
  return true;
}
// readTag: tag = 0 at the end of the current limit; field number 0 is invalid
__device__ __forceinline__ bool rd_tag(Cur& c, uint32_t& tag) {
  if (c.p >= c.end) { tag = 0; return true; }
  if (!rd_varint32(c, tag)) return false;
  return (tag >> 3) != 0;
}
// length prefix checked against the current limit (negativeSize / truncatedMessage)
__device__ __forceinline__ bool rd_len(Cur& c, uint32_t& len) {
  if (!rd_varint32(c, len)) return false;
  if ((int32_t)len < 0) return false;
  return (size_t)(c.end - c.p) >= len;
}
// UnknownFieldSet.mergeFieldFrom.  Groups are matched with an explicit stack; the reference's
// recursion limit is 100 messages, ours is TFR_MAX_GROUP_DEPTH nested groups (documented
// deviation: deeper nesting is reported as malformed; TensorFlow never emits groups).
#define TFR_MAX_GROUP_DEPTH 24
__device__ __noinline__ bool skip_group(Cur& c, uint32_t field) {
  uint32_t stack[TFR_MAX_GROUP_DEPTH];
  int depth = 0;
  stack[depth++] = field;
  while (depth > 0) {
    uint32_t t;
    if (!rd_tag(c, t) || t == 0) return false;
    switch (t & 7) {
      case 0: { uint64_t v; if (!rd_varint64(c, v)) return false; break; }
      case 1: if (c.end - c.p < 8) return false; c.p += 8; break;
      case 2: { uint32_t l; if (!rd_len(c, l)) return false; c.p += l; break; }
      case 3: if (depth >= TFR_MAX_GROUP_DEPTH) return false; stack[depth++] = t >> 3; break;
      case 4: if (stack[--depth] != (t >> 3)) return false; break;
      case 5: if (c.end - c.p < 4) return false; c.p += 4; break;
      default: return false;
    }
  }
  return true;
}
// returns false on malformed input; a stray END_GROUP is malformed at every call site
// (checkLastTagWas(0) fails after the enclosing message returns)
__device__ __forceinline__ bool skip_field(Cur& c, uint32_t tag) {
  switch (tag & 7) {
    case 0: { uint64_t v; return rd_varint64(c, v); }
    case 1: if (c.end - c.p < 8) return false; c.p += 8; return true;
    case 2: { uint32_t l; if (!rd_len(c, l)) return false; c.p += l; return true; }
    case 3: return skip_group(c, tag >> 3);
    case 5: if (c.end - c.p < 4) return false; c.p += 4; return true;
    default: return false;
  }
}

// protobuf Utf8.isValidUtf8 (readStringRequireUtf8 for proto3 map keys)
__device__ __forceinline__ bool utf8_valid(const uint8_t* p, uint32_t n) {
  uint32_t i = 0;
  while (i < n) {
    uint32_t b = p[i];
    if (b < 0x80) { ++i; continue; }
    if (b < 0xC2) return false;
    if (b < 0xE0) { if (i + 1 >= n || (p[i + 1] & 0xC0) != 0x80) return false; i += 2; continue; }
    if (b < 0xF0) {
      if (i + 2 >= n) return false;
      uint32_t b2 = p[i + 1], b3 = p[i + 2];
      if ((b2 & 0xC0) != 0x80 || (b3 & 0xC0) != 0x80) return false;
      if (b == 0xE0 && b2 < 0xA0) return false;
      if (b == 0xED && b2 >= 0xA0) return false;
      i += 3; continue;
    }
    if (b > 0xF4 || i + 3 >= n) return false;
    uint32_t b2 = p[i + 1], b3 = p[i + 2], b4 = p[i + 3];
    if ((b2 & 0xC0) != 0x80 || (b3 & 0xC0) != 0x80 || (b4 & 0xC0) != 0x80) return false;
    if (b == 0xF0 && b2 < 0x90) return false;
    if (b == 0xF4 && b2 >= 0x90) return false;
    i += 4;
  }
  return true;
}

// Java round trip ByteString.toStringUtf8 -> UTF8String.fromString (M/TFRecordDeserializer.scala:91,215):
// well-formed input is copied, every malformed unit becomes EF BF BD, grouped as the JDK decoder
// groups them (restated in oracle/tfr_oracle.c java_utf8_roundtrip).  dst == nullptr: length only.
__device__ __forceinline__ bool u8_not_cont(uint32_t b) { return (b & 0xc0) != 0x80; }
__device__ __noinline__ uint32_t java_utf8_transcode(const uint8_t* src, uint32_t sl, uint8_t* dst) {
  uint32_t sp = 0, dp = 0;
#define PUT_REPL() do { if (dst) { dst[dp] = 0xEF; dst[dp + 1] = 0xBF; dst[dp + 2] = 0xBD; } dp += 3; } while (0)
#define PUT_COPY(k) do { if (dst) for (uint32_t q = 0; q < (k); ++q) dst[dp + q] = src[sp + q]; dp += (k); sp += (k); } while (0)
  while (sp < sl) {
    uint32_t b1 = src[sp];
    if (b1 < 0x80) { if (dst) dst[dp] = (uint8_t)b1; ++dp; ++sp; continue; }
    if ((b1 >> 5) == 0x6 && (b1 & 0x1e) != 0) {
      if (sp + 1 < sl) {
        if (u8_not_cont(src[sp + 1])) { PUT_REPL(); sp += 1; } else PUT_COPY(2);
        continue;
      }
      PUT_REPL(); break;
    }
    if ((b1 >> 4) == 0xE) {
      if (sp + 2 < sl) {
        uint32_t b2 = src[sp + 1], b3 = src[sp + 2];
        bool e0 = (b1 == 0xe0 && (b2 & 0xe0) == 0x80);
        if (e0 || u8_not_cont(b2) || u8_not_cont(b3)) {
          PUT_REPL(); sp += (e0 || u8_not_cont(b2)) ? 1 : 2;
        } else {
          uint32_t cpt = ((b1 & 0x0f) << 12) | ((b2 & 0x3f) << 6) | (b3 & 0x3f);
          if (cpt >= 0xD800 && cpt <= 0xDFFF) { PUT_REPL(); sp += 3; } else PUT_COPY(3);
        }
        continue;
      }
      if (sp + 1 < sl && ((b1 == 0xe0 && (src[sp + 1] & 0xe0) == 0x80) || u8_not_cont(src[sp + 1]))) { PUT_REPL(); sp += 1; continue; }
      PUT_REPL(); break;
    }
    if ((b1 >> 3) == 0x1E) {
      if (sp + 3 < sl) {
        uint32_t b2 = src[sp + 1], b3 = src[sp + 2], b4 = src[sp + 3];
        uint32_t uc = ((b1 & 0x07) << 18) | ((b2 & 0x3f) << 12) | ((b3 & 0x3f) << 6) | (b4 & 0x3f);
        if (u8_not_cont(b2) || u8_not_cont(b3) || u8_not_cont(b4) || !(uc >= 0x10000 && uc <= 0x10FFFF)) {
          PUT_REPL();
          if (b1 > 0xf4 || (b1 == 0xf0 && (b2 < 0x90 || b2 > 0xbf)) || (b1 == 0xf4 && (b2 & 0xf0) != 0x80) || u8_not_cont(b2)) sp += 1;
          else if (u8_not_cont(b3)) sp += 2;
          else sp += 3;
        } else PUT_COPY(4);
        continue;
      }
      uint32_t b2 = sp + 1 < sl ? src[sp + 1] : 0;
      if (b1 > 0xf4 || (sp + 1 < sl && ((b1 == 0xf0 && (b2 < 0x90 || b2 > 0xbf)) || (b1 == 0xf4 && (b2 & 0xf0) != 0x80) || u8_not_cont(b2)))) { PUT_REPL(); sp += 1; continue; }
      if (sp + 2 < sl && u8_not_cont(src[sp + 2])) { PUT_REPL(); sp += 2; continue; }
      PUT_REPL(); break;
    }
    PUT_REPL(); sp += 1;
  }
#undef PUT_REPL
#undef PUT_COPY
  return dp;
}
// true when every byte is < 0x80 (the transcode is then the identity)
__device__ __forceinline__ bool all_ascii(const uint8_t* p, uint32_t n) {
  uint32_t acc = 0;
  for (uint32_t i = 0; i < n; ++i) acc |= p[i];
  return acc < 0x80;
}

// ---------------------------------------------------------------------------------------------
// schema as the kernels see it
// ---------------------------------------------------------------------------------------------
enum { K_NONE = 0, K_BYTES = 1, K_FLOAT = 2, K_INT64 = 3 };   // Feature.KindCase numbers

struct DevField {
  uint32_t name_off, name_len, hash;
  int8_t elem_type, depth, nullable, kind;   // kind = Feature kind this type requires
  int16_t n_levels;                          // offset levels (depth + varlen leaf)
  int16_t dup_next;                          // next schema field with the same name, -1 none
  int32_t fix_slot;                          // index among depth-0 fixed-width columns, -1
  int32_t var_slot;                          // index among columns with n_levels >= 1, -1
  int32_t cnt_slot;                          // first count array of this column (n_levels of them)
  int32_t width;                             // leaf width in bytes
};

struct DevSchema {
  int32_t n_fields, record_type, ht_mask, n_fix, n_var, n_cnt;
  const DevField* fields;
  const uint8_t* names;
  const int32_t* ht;   // open addressing: slot -> field index, -1 empty
};

__device__ __forceinline__ uint32_t name_hash(const uint8_t* p, uint32_t n) {   // FNV-1a
  uint32_t h = 2166136261u;
  for (uint32_t i = 0; i < n; ++i) h = (h ^ p[i]) * 16777619u;
  return h;
}
__host__ __device__ __forceinline__ int required_kind(int t) {
  switch (t) {
    case TFR_T_INT32: case TFR_T_INT64: return K_INT64;
    case TFR_T_FLOAT32: case TFR_T_FLOAT64: case TFR_T_DECIMAL: return K_FLOAT;
    case TFR_T_STRING: case TFR_T_BINARY: return K_BYTES;
    default: return K_NONE;
  }
}
__host__ __device__ __forceinline__ int type_width(int t) {
  switch (t) {
    case TFR_T_INT32: case TFR_T_FLOAT32: return 4;
    case TFR_T_INT64: case TFR_T_FLOAT64: case TFR_T_DECIMAL: return 8;
    case TFR_T_STRING: case TFR_T_BINARY: return 1;
    default: return 0;
  }
}

// per-record status word: code in the low 8 bits (negated TFR_E_*), field index + 1 above; the top bit is DF_REGION
__device__ __forceinline__ uint32_t make_status(int code, int field) { return (uint32_t)(-code) | ((uint32_t)(field + 1) << 8); }
// the status of a lost region (TFR_F_RESYNC) in a failing-record list: its code is the framing error, its field -1
#define DF_REGION 0x80000000u
__host__ __device__ __forceinline__ int32_t status_code(uint32_t s) { return -(int32_t)(s & 0xff); }
__host__ __device__ __forceinline__ int32_t status_field(uint32_t s) { return (int32_t)((s & ~DF_REGION) >> 8) - 1; }
