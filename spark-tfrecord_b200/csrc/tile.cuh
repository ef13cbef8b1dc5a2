// tile.cuh -- fast path of the decode: shared-memory record tiles, one record per thread.
//
// Same reference functions as decode.cuh (TFRecordReader payload CRC, Example.parseFrom,
// deserializeExample: M/TFRecordFileReader.scala:49-81, M/TFRecordDeserializer.scala:21-35,68-124), for
// the shape of data the reference writer itself produces ("canonical"):
//   payload  = 0A len Features                       (exactly one field)
//   Features = { 0A elen  0A klen key  12 vlen Feature }*
//   Feature  = kindtag llen List ;  Int64List/FloatList = [0A plen packed] ; BytesList = { 0A blen bytes }*
// Everything else that protobuf allows (unknown fields, merges, unpacked encodings, duplicate keys,
// overlong tags ...), every semantic error and every CRC mismatch is DETECTED here and makes the kernel
// raise a flag; the host then re-runs the batch through the general kernels of decode.cuh, which
// implement the full semantics.  So the fast path never changes a result, it only skips work.
//
// Mapping: one CTA = one tile = 32 consecutive records (rows 32t .. 32t+31, contiguous in memory),
// TILE_PARSE_WARPS parse warps + TILE_CRC_WARPS CRC warps, all working on the same staged bytes.
//   1. warp 0 arms an mbarrier; every lane issues cp.async.bulk (TMA bulk copy, SASS UBLKCP) of ITS record into its
//      place in the tile (records packed one behind the other at strides that are odd multiples of 16 bytes: they spread over all eight
//      16-byte bank groups), and one more bulk copy brings the per-schema constants (5-bit CRC tables, zeroed merge
//      words, field table, entry templates, names), which api.cu keeps in HBM in exactly the shared-memory layout.
//   2. role split over the same staged bytes: the C CRC warps each fold a third of the 16-byte chunks of record
//      `lane` (aligned 128-bit loads, 13 conflict-free 5-bit table lookups per 8 bytes) and combine through one GF(2)
//      shift each.  Parse warp w owns the map entries with index = w mod W of record `lane` and fully parses them.  In
//      the 12 + 3 warp kernels the last parse warp first walks the map-entry chain of record `lane` once (`0A elen` ->
//      p += elen) and writes where every entry starts into a shared-memory ENTRY TABLE (16-bit offsets from the payload,
//      one row per entry index, lane = record: conflict-free rows); the parse warps wait for it at a named barrier and
//      then go straight to each of their entries.  (Entries past the table's rows -- features the reader's schema
//      prunes -- or past 64 KiB of payload are reached by hopping on from the last entry the table holds.)  In the 4 + 1
//      warp kernel (small records: a tile's life is a latency chain that a walk in front of a barrier lengthens) each
//      warp hops from one of its entries to the next (`0A elen` -> p += elen, W - 1 hops).  An owned entry is first
//      matched against a per-field TEMPLATE of its constant bytes (0A ? 0A klen key 12 ? kind ?: masked word
//      compares), which also fixes the Feature kind and list length; only when that fails is it parsed byte by byte
//      (hash lookup of the key, full checks).  Shared-memory capacity limits how many records an SM can stage, so more
//      dependent chains per staged record = more warps to hide latency, and no single warp's chain is the tile's
//      critical path.
//   3. lane = row, rows are 32-aligned: every column store of the warp covers 32 consecutive rows
//      (coalesced by construction, no transpose) and validity bitmaps are one __ballot_sync per field.
//   4. variable-width columns either write element counts + source offsets (scan + decode_pass2_kernel
//      finish them), or -- once the decoder has learned that every such column has a uniform shape
//      (FloatList[8], 16-byte BytesList ...) -- write the values at row * L in the same pass and only
//      verify the shape ("uniform-shape speculation": input read once, output written once).
//   5. the row count can be read from the device (TileArgs::n_dev = the frame index's result): the host enqueues the
//      kernel without knowing it, with a grid sized from a capacity; surplus CTAs exit at once.
#pragma once
#include "common.cuh"
#include "decode.cuh"

#define TILE_ROWS 32
#ifndef TILE_PARSE_WARPS
#define TILE_PARSE_WARPS 12
#endif
#ifndef TILE_CRC_WARPS
#define TILE_CRC_WARPS 3       // warps W .. W+C-1: each takes 1/C of every record's payload CRC
#endif
#define TILE_THREADS ((TILE_PARSE_WARPS + TILE_CRC_WARPS) * 32)
#ifndef TILE_MIN_CTAS
#define TILE_MIN_CTAS 3       // registers are capped so that shared memory, not the register file, limits residency
#endif
#define TILE_TPL_WORDS 5          // template covers up to 20 bytes: key names up to 12 bytes

// constant bytes of a canonical map entry of one schema field, for masked word compares
struct FieldTemplate {
  uint32_t words[TILE_TPL_WORDS];
  uint32_t mask[TILE_TPL_WORDS];
  uint16_t n_words;             // 0: no template (long name): generic parse
  uint16_t klen;                // key length
  uint32_t kind;                // K_*
};

struct TileArgs {
  const uint8_t* data;          // framed bytes, any alignment
  uint32_t nbytes;
  uint32_t misalign;            // data & 15
  uint32_t pf_dist;             // L2 prefetch distance in tiles (CTAs resident on the whole GPU), 0: off
  const uint32_t* rec_off;      // [n+1]
  uint32_t n;                   // rows in the batch = stride of the scratch arrays; with n_dev: the CAPACITY the host sized everything for
  const uint32_t* n_dev;        // non-null: the number of rows is read here (FrameResult::n_records of this batch, still on the device when the
                                // kernel is enqueued); more rows than `n` raise TF_OVERFLOW and nothing is decoded
  uint32_t tile_cap;            // bytes of shared memory reserved for the record bytes of one tile (32 records, packed)
  uint32_t slot;                // != 0: fixed slots of this size (an ODD multiple of 16) per record; 0: records packed
  uint32_t* tile_max;           // device word: max over the tiles of the packed bytes they would need (atomicMax), or null
  uint32_t verify;
  uint32_t names_bytes;
  DevSchema sch;
  const uint8_t* consts;        // per-schema constants in the shared-memory layout (CRC tables | seen zeros | fields | templates | names)
  uint32_t const_bytes;         // multiple of 16
  uint8_t* bitmaps;             // [nf][nb_stride] Arrow validity bitmaps, written directly
  uint32_t nb_stride;
  unsigned long long* null_counts;   // [nf]
  void* const* fix_values;      // [n_fix]
  uint32_t* cnt;                // [n_cnt][n]   (count mode)
  uint32_t* src;                // [n_var][n]
  uint8_t* cflag;               // [n_var][n]
  const int32_t* uniform_len;   // [n_var] >= 0: speculated per-row count (elements, or bytes for scalar string/binary); -1: count mode;
                                // -2 (TILE_RAGGED): ragged column finished in THIS kernel (tile-local prefix + look-back across tiles)
  // ---- one-pass ragged mode (any uniform_len == TILE_RAGGED) ----
  uint32_t ragged;              // 1: tiles take ordered ids from `ticket`, publish per-array totals and look back for their bases
  uint32_t n_cnt;               // count arrays (offset levels) of the schema
  uint32_t* ticket;             // [1] zeroed per batch
  uint32_t* lb_flag;            // [tiles] 0 nothing, 1 aggregates published, 2 inclusive prefixes published; zeroed per batch
  uint32_t* lb_agg;             // [tiles][n_cnt] per-tile totals
  unsigned long long* lb_pre;   // [tiles][n_cnt] inclusive prefixes
  const unsigned long long* cap;     // [n_cnt] what each array's target buffer was sized for (elements of the next level / leaf values)
  unsigned long long* totals;   // [n_cnt] grand totals, written by the last tile
  int32_t* const* offs;         // [n_var*3] Arrow offsets arrays per level
  const int32_t* var_field;     // [n_var] schema field of each var slot
  void* const* var_values;      // [n_var] leaf buffers (uniform mode)
  uint32_t* flags;              // [0] bit0: fall back to the general path, bit1: a uniform-shape speculation failed
};

enum { TF_FALLBACK = 1u, TF_SHAPE = 2u, TF_OVERFLOW = 4u, TF_XCODE = 8u };
#define TILE_RAGGED (-2)

// ---- mbarrier + bulk async copy (PTX; sm_90+) ---------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
  } while (!ok);
}

// ---- look-back flags: release/acquire at GPU scope ----
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_cg_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_cg_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// ---- shared-memory byte helpers (offsets into the tile, not pointers: 32-bit address arithmetic) --
// The loads are explicit ld.shared on a 32-bit shared-window address held in a register: through a generic pointer the
// compiler re-derives the window base (S2R SR_CgaCtaId + LEA) at most access sites, extra instructions on every access.
// The tile is read-only after the mbarrier wait; `s` is produced by a volatile asm placed after that wait so that no
// load can be scheduled above it.
struct Tile {
  const uint8_t* b;   // tile base in shared memory (16-byte aligned), generic pointer for the rare helper calls
  uint32_t s;         // the same address in the shared window
  __device__ __forceinline__ uint32_t u8(uint32_t o) const {
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(s + o));
    return v;
  }
  __device__ __forceinline__ int32_t i8(uint32_t o) const {
    int32_t v;
    asm("ld.shared.s8 %0, [%1];" : "=r"(v) : "r"(s + o));
    return v;
  }
  __device__ __forceinline__ uint4 w128(uint32_t o) const {     // 16-byte aligned
    uint4 v;
    asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(s + o));
    return v;
  }
  __device__ __forceinline__ uint32_t w32(uint32_t o) const {   // aligned word
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(s + o));
    return v;
  }
};
__device__ __forceinline__ uint32_t t_u32(const Tile& t, uint32_t o) {   // 4 bytes at any alignment
  const uint32_t a = o & ~3u;
  uint32_t sh = (o & 3u) * 8;
  uint32_t lo = t.w32(a);
  return sh ? __funnelshift_r(lo, t.w32(a + 4), sh) : lo;
}
// length varint: 1..5 bytes (minimal or not); false if it runs past `end` or is longer (-> general path)
__device__ __forceinline__ bool t_len(const Tile& t, uint32_t& p, uint32_t end, uint32_t& v) {
  if (p >= end) return false;
  uint32_t b = t.u8(p++);
  if (b < 0x80) { v = b; return true; }
  uint32_t r = b & 0x7f;
#pragma unroll 1
  for (int sh = 7; sh < 35; sh += 7) {
    if (p >= end) return false;
    b = t.u8(p++);
    r |= (b & 0x7f) << sh;
    if (b < 0x80) { v = r; return (int32_t)r >= 0; }
  }
  return false;
}
// map entry at p (`0A elen ...`, p < end) -> the next one: one byte load + add, the full length varint only for entries of
// 128+ bytes.  The tag and the contents are the owner's to check; false if the length varint runs past `end`.
__device__ __forceinline__ bool t_next_entry(const Tile& t, uint32_t& p, uint32_t end) {
  const int32_t b1 = t.i8(p + 1);
  if (b1 >= 0) { p += 2u + (uint32_t)b1; return true; }
  uint32_t q = p + 1, el;
  if (!t_len(t, q, end, el)) return false;
  p = q + el;
  return true;
}

// l bytes of the tile -> global memory at any alignment: bytes up to the first aligned word, whole words, tail bytes.  The
// 32 lanes of a warp copy the cells of 32 consecutive rows, which are adjacent in the output: the partial lines merge in L2.
__device__ __forceinline__ void t_copy_out(const Tile& t, uint32_t src, uint8_t* dst, uint32_t l) {
  uint32_t i = 0;
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 3u);
  if (mis) for (const uint32_t h = min(l, 4u - mis); i < h; ++i) dst[i] = (uint8_t)t.u8(src + i);
  for (; i + 4 <= l; i += 4) *reinterpret_cast<uint32_t*>(dst + i) = t_u32(t, src + i);
  for (; i < l; ++i) dst[i] = (uint8_t)t.u8(src + i);
}

// a string cell of a row that holds malformed UTF-8 somewhere (rare): kept out of line so that the copy-out stays small.
// Well-formed (or pure ASCII) bytes are copied, anything else is re-encoded the way Java does; returns the bytes written.
__device__ __noinline__ uint32_t t_xcode_cell(const uint8_t* src, uint32_t raw, uint8_t* dst) {      // dst == nullptr: length only
  if (all_ascii(src, raw) || utf8_valid(src, raw)) { if (dst) for (uint32_t i = 0; i < raw; ++i) dst[i] = src[i]; return raw; }
  return java_utf8_transcode(src, raw, dst);
}

// ---- per-thread CRC-32C over shared memory: 8 bytes per step through 13 conflict-free 5-bit tables (CrcTables::g5) ----
__device__ __forceinline__ uint32_t crc_fold8(const uint32_t* g, uint32_t c, uint32_t lo, uint32_t hi) {
  const uint32_t a = lo ^ c;
  return g[0 * 32 + (a & 31)] ^ g[1 * 32 + ((a >> 5) & 31)] ^ g[2 * 32 + ((a >> 10) & 31)] ^ g[3 * 32 + ((a >> 15) & 31)] ^
         g[4 * 32 + ((a >> 20) & 31)] ^ g[5 * 32 + ((a >> 25) & 31)] ^ g[6 * 32 + (__funnelshift_r(a, hi, 30) & 31)] ^
         g[7 * 32 + ((hi >> 3) & 31)] ^ g[8 * 32 + ((hi >> 8) & 31)] ^ g[9 * 32 + ((hi >> 13) & 31)] ^ g[10 * 32 + ((hi >> 18) & 31)] ^
         g[11 * 32 + ((hi >> 23) & 31)] ^ g[12 * 32 + (hi >> 28)];
}
__device__ __forceinline__ uint32_t crc_byte(const uint32_t* g, uint32_t c, uint32_t b) {
  const uint32_t x = (c ^ b) & 0xff;
  return (c >> 8) ^ g[416 + (x & 31)] ^ g[448 + (x >> 5)];
}
// CRC-32C of a record's payload, split over the C CRC warps (lane = record, as everywhere in this kernel):
//   head   bytes up to the first 16-byte boundary: byte-wise, by CRC warp 0, from the initial state
//   body   K whole 16-byte chunks read with aligned 128-bit loads (the slots' stride is an odd multiple of 16 bytes, so
//          the 32 lanes spread over all eight 16-byte bank groups and a load costs the minimum of 4 wavefronts);
//          CRC warp c folds chunks [K*c/C, K*(c+1)/C) from state 0 (warp 0: from the head state), multiplies its state by
//          x^(8*16*chunks after its range) (ONE GF(2) multiply by a table constant: CRC(A||B) = CRC_B(0) ^ shift_|B|(CRC_A))
//          and XORs it into the record's accumulator in shared memory
//   tail   < 16 bytes, folded byte-wise from the accumulated state by CRC warp 0 after the CRC warps' barrier.
// A serial CRC is one dependent chain (a table round trip per 8 bytes) that a single warp cannot issue faster than its
// latency allows; as one warp per tile it was the tile's critical path.
__device__ __forceinline__ uint32_t crc_chunks(const uint32_t* g, const Tile& t, uint32_t o, uint32_t k, uint32_t c) {
#pragma unroll 2
  for (uint32_t i = 0; i < k; ++i) {
    const uint4 v = t.w128(o + 16 * i);
    c = crc_fold8(g, c, v.x, v.y);
    c = crc_fold8(g, c, v.z, v.w);
  }
  return c;
}
// x^(8*16*m) mod P for m >= 512, past the xp16 table: a packed tile can hold one record of 8 KiB and more, whose leading CRC
// warps shift further.  x^(8*16*m) = xp16[511]^q * xp16[m - 511 q]: one more GF(2) multiply per 511 chunks (8 KiB).  Out of
// line, so that the common case (an xp16 lookup) keeps the CRC warps' code and registers as they are.
__device__ __noinline__ uint32_t chunk_shift_far(const uint32_t* xp16, uint32_t m) {
  uint32_t f = xp16[511];
  for (m -= 511u; m; ) {
    const uint32_t s = min(m, 511u);
    f = gf2_mulmod(f, xp16[s]);
    m -= s;
  }
  return f;
}

// shared memory layout (dynamic), all sections 16-byte aligned:
//   [0,16) mbarrier | CRC tables g5 2 KiB + xp16 2 KiB | seen words [32][4] u32 + CRC accumulators [32] | DevField[nf] | FieldTemplate[nf] | names | entry table | tile bytes
// Everything between the mbarrier and the entry table is constant per schema ("consts": built once per decoder in this
// layout, api.cu) and arrives with ONE bulk copy on the same mbarrier as the tile.
#define TILE_SEEN_BYTES (512u + 128u + 16u) // seen words [32][4], the CRC accumulators [32], then the mask of rows some warp gave up on; zero in the consts blob
#define TILE_CRC_BYTES (2048u + 2048u)     // g5, xp16
__host__ __device__ inline uint32_t tile_schema_smem(uint32_t nf, uint32_t names_bytes) {
  return ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u) + ((nf * (uint32_t)sizeof(FieldTemplate) + 15u) & ~15u) + ((names_bytes + 15u) & ~15u);
}
__host__ __device__ inline uint32_t tile_const_bytes(uint32_t nf, uint32_t names_bytes) { return TILE_CRC_BYTES + TILE_SEEN_BYTES + tile_schema_smem(nf, names_bytes); }
// entry table of the Example features / SequenceExample context: where map entry e of record `lane` starts, as a u16 offset
// from the record's payload, at [e][lane] (a warp reading one row touches 64 consecutive bytes: no bank conflict); then per
// lane the number of entries [32] and how many of them the table holds [32] u32.  One row per schema field: a record the
// fast path takes has at most one entry per field it reads, and entries beyond (fields the reader prunes) are hopped to.
// Only the 12 + 3 warp kernels build it; the sizing counts it for every tile (small schemas: a few hundred bytes).
__host__ __device__ inline uint32_t tile_entry_rows(uint32_t nf) { return nf; }
__host__ __device__ inline uint32_t tile_entry_bytes(uint32_t nf) { return tile_entry_rows(nf) * 32u * 2u + 256u; }
// ragged mode scratch behind the tile: cell source offsets [n_var][32] | per-array counts -> local offsets [n_cnt][32] | totals [n_cnt] | bases u64 [n_cnt] | tile id
__host__ __device__ inline uint32_t tile_ragged_bytes(uint32_t n_var, uint32_t n_cnt) { return (n_var + n_cnt) * 128u + n_cnt * 4u + n_cnt * 8u + 16u + 16u + 96u; }
#define TILE_SQ_STEPS 128u       // FeatureList steps per record the one-pass mode keeps per-step element counts for
// SequenceExample scratch: FeatureList count sums [n_var][32][2] u32, then (one-pass mode, at most 4 variable-width columns)
// the per-step element counts [n_var][TILE_SQ_STEPS][32] u8
__host__ __device__ inline uint32_t tile_seq_bytes(uint32_t n_var, bool with_steps = false) { return n_var * 256u + 16u + (with_steps ? n_var * TILE_SQ_STEPS * 32u : 0u); }
__host__ __device__ inline uint32_t tile_smem_bytes(uint32_t nf, uint32_t names_bytes, uint32_t tile_cap, uint32_t ragged_bytes = 0) {
  return 16 + tile_const_bytes(nf, names_bytes) + tile_entry_bytes(nf) + tile_cap + 64 + ragged_bytes;   // +64: template compares may look a few bytes past the tile
}

// PW parse warps + CW CRC warps per tile.  Large records: shared memory allows three tiles per SM, so a tile gets 12 + 3 warps
// (45 resident warps).  Small records: a tile is a few KB, eight fit an SM, and 4 + 1 warps per tile give the same number of
// resident warps with three times as many records in flight (a tile's life is a latency chain: offsets -> bulk copy -> parse
// -> entry walk -> parse -> barriers -> stores).
// XC: the kernel can re-encode malformed UTF-8 strings of ragged columns itself (calls into the out-of-line Java transcoder).
// Merely containing those calls slows the kernel down (registers and code size, even when they never execute), so the
// default instantiation has none: it raises TF_XCODE instead and the host re-runs the batch -- and the next ones -- with XC.
template <bool SEQ, bool RG, int PW, int CW, bool XC>
__global__ void __launch_bounds__((PW + CW) * 32, (PW >= 16 ? 2 : PW >= 12 ? TILE_MIN_CTAS : 8)) decode_tile_kernel(TileArgs A) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* s8 = reinterpret_cast<uint32_t*>(smem_raw + 16);                               // g5 tables, then xp16
  uint32_t* sseen = reinterpret_cast<uint32_t*>(smem_raw + 16 + TILE_CRC_BYTES);                 // [32 rows][4 words], zero in the consts blob
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  uint8_t* sbase = smem_raw + 16 + TILE_CRC_BYTES + TILE_SEEN_BYTES;
  DevField* sfields = reinterpret_cast<DevField*>(sbase);
  FieldTemplate* stpl = reinterpret_cast<FieldTemplate*>(sbase + ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u));
  uint8_t* snames = sbase + ((nf * (uint32_t)sizeof(DevField) + 15u) & ~15u) + ((nf * (uint32_t)sizeof(FieldTemplate) + 15u) & ~15u);
  uint16_t* eoff = reinterpret_cast<uint16_t*>(sbase + tile_schema_smem(nf, A.names_bytes));    // entry table [E][32] (see tile_entry_bytes)
  uint32_t* ecnt = reinterpret_cast<uint32_t*>(eoff + tile_entry_rows(nf) * 32u);              // [32] entries, [32] entries in the table
  uint8_t* tile_b = sbase + tile_schema_smem(nf, A.names_bytes) + tile_entry_bytes(nf);
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;                          // warps 0..W-1 parse, warp W = CRC

  // Record r of the tile is copied to its place in the tile: bytes [off_r & ~15, off_r + framed length) -> tile + rbase_r.
  // (cp.async.bulk wants 16-byte aligned source, destination and size; the record starts (off_r & 15) bytes into its slot.)
  // ragged scratch behind the tile bytes (see tile_ragged_bytes)
  uint32_t* rg_src = reinterpret_cast<uint32_t*>(tile_b + A.tile_cap + 64);           // [n_var][32] tile offset of each cell's bytes
  uint32_t* rg_cnt = rg_src + (uint32_t)A.sch.n_var * 32u;                            // [n_cnt][32] counts, then tile-local exclusive offsets
  uint32_t* rg_tot = rg_cnt + A.n_cnt * 32u;                                          // [n_cnt] tile totals
  unsigned long long* rg_base = reinterpret_cast<unsigned long long*>(rg_tot + ((A.n_cnt + 1u) & ~1u) + 24u);  // [n_cnt] exclusive bases of this tile
  uint32_t* rg_tile = rg_tot + ((A.n_cnt + 1u) & ~1u);                                // [0] tile id, [1] skip-copy flag, [2..2+PW] look-back summaries of the parse warps + the give-up word (PW <= 16)
  // SequenceExample: per (column, row) element / byte counts of the FeatureLists, summed over the parse warps [n_var][32][2]
  uint32_t* sq_cnt = reinterpret_cast<uint32_t*>(tile_b + A.tile_cap + 64 + (RG ? tile_ragged_bytes((uint32_t)A.sch.n_var, A.n_cnt) : 0u));
  uint8_t* sq_tab = reinterpret_cast<uint8_t*>(sq_cnt + (uint32_t)A.sch.n_var * 64u + 4u);      // [n_var][TILE_SQ_STEPS][32] elements per step (SEQ && RG)
  if (SEQ) for (uint32_t i = threadIdx.x; i < (uint32_t)A.sch.n_var * 64u; i += (PW + CW) * 32) sq_cnt[i] = 0u;
  // Tile id.  Ragged mode: tiles look back at their predecessors' totals, so ids are handed out in start order (a tile only
  // ever waits for tiles that are already running); otherwise the block index.
  uint32_t tile = blockIdx.x;
  if (RG) {
    if (threadIdx.x == 0) { rg_tile[0] = atomicAdd(A.ticket, 1u); rg_tile[1] = 0u; rg_tile[2 + PW] = 0u; }
    for (uint32_t i = threadIdx.x; i < A.n_cnt * 32u; i += ((PW + CW) * 32)) rg_cnt[i] = 0u;      // absent cells count as empty
    __syncthreads();
    tile = rg_tile[0];
  }
  const uint32_t row0 = tile * TILE_ROWS;
  uint32_t n_rows = A.n;
  if (A.n_dev) {
    n_rows = *A.n_dev;
    if (n_rows > A.n) {                                                    // more records than the host provisioned for: the host redoes the batch
      if (tile == 0 && threadIdx.x == 0) atomicOr(A.flags, TF_OVERFLOW | TF_FALLBACK);
      return;                                                              // (no tile runs: nobody waits for anybody)
    }
    if (row0 >= n_rows) return;                                            // the grid was sized from the capacity
  }
  const uint32_t rows = min((uint32_t)TILE_ROWS, n_rows - row0);
  const bool active = lane < rows;
  const uint32_t row = row0 + lane;
  uint32_t off = 0, flen = 16;
  if (active) { off = A.rec_off[row]; flen = A.rec_off[row + 1] - off; }
  // cp.async.bulk wants 16-byte aligned source, destination and size.  Coordinates below are bytes from the 16-byte aligned
  // address at or below A.data (`base`): the buffer is [mis, lim).  A record's 16-byte groups that are not entirely inside the
  // buffer -- the first group of a misaligned buffer, the last group of the batch's last record -- are clipped from the bulk
  // copy and their bytes inside the buffer are moved with ordinary loads: a caller's device buffer needs neither alignment
  // nor padding.
  const uint32_t mis = A.misalign, lim = mis + A.nbytes;
  const uint8_t* base = A.data - mis;
  const uint32_t head = (off + mis) & 15u;
  const uint32_t g_lo = off + mis - head;                                  // the record's first 16-byte group
  const uint32_t cbytes = active ? (head + flen + 15u) & ~15u : 0u;
  uint32_t b_lo = g_lo, b_hi = g_lo + cbytes;
  if (active && b_lo < mis) b_lo += 16u;
  if (active && b_hi > lim) b_hi = lim & ~15u;
  const uint32_t bulk_bytes = (active && b_hi > b_lo) ? b_hi - b_lo : 0u;
  // Where the records sit in the tile.  A record's stride = its 16-byte groups + 32 bytes of slack (word loads of the parse
  // look a little past a record), made an ODD number of 16-byte units.
  //   fixed slots (A.slot != 0): every record at lane * slot, slot = the largest record's stride.  The 32 lanes then start in
  //     all eight 16-byte bank groups, four lanes each: the minimum of shared-memory wavefronts for the 16-byte CRC loads and
  //     the parse's word loads (same-sized records at an even stride put every lane on the same banks).
  //   packed (A.slot == 0): one behind the other at their own strides.  Records of very different sizes do not each pay for the
  //     largest one -- the tile is sized for a typical SUM of 32 records.  The host picks this when it lets one more tile
  //     live on an SM.
  uint32_t stride = active ? (cbytes + 32u + 15u) & ~15u : 0u;
  if (active && ((stride >> 4) & 1u) == 0u) stride += 16u;
  // packed: every stride is padded to 16 bytes more than a multiple of 128, so that record r starts in bank group r % 8 like
  // with fixed odd slots (64 bytes of padding per record on average; a plain prefix sum gives the places)
  uint32_t tile_tot;
  uint32_t rbase = warp_excl_scan_u32(active ? ((stride + 111u) & ~127u) + 16u : 0u, tile_tot);
  uint32_t tile_need = tile_tot;                                           // bytes of the tile this layout takes
  if (A.slot) { rbase = lane * A.slot; tile_need = __any_sync(FULLMASK, stride > A.slot) ? 0xffffffffu : 0u; }
  if (threadIdx.x == 0 && A.tile_max) atomicMax(A.tile_max, tile_tot);     // (the packed size, whatever the layout: what the next batch's tiles are sized from)
  if (tile_need > A.tile_cap) {                                             // the tile's records do not fit: general path
    if (threadIdx.x == 0) {
      atomicOr(A.flags, TF_FALLBACK);
      if (RG) {                                                            // successors must not wait for this tile (the batch is redone anyway)
        for (uint32_t a = 0; a < A.n_cnt; ++a) A.lb_pre[(size_t)tile * ((A.n_cnt + 3u) & ~3u) + a] = 0ull;
        __threadfence();
        st_release_u32(&A.lb_flag[tile], 2u);
      }
    }
    return;
  }
  if (wid == 0) {
    if (lane == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const uint32_t total = __reduce_add_sync(FULLMASK, bulk_bytes);
    if (lane == 0) {
      mbar_expect_tx(bar, total + A.const_bytes);
      bulk_g2s(smem_raw + 16, A.consts, A.const_bytes, bar);      // CRC tables, zeroed seen words, schema, templates, names
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
  __syncthreads();                                                // the barrier is initialised before anyone waits on it
  mbar_wait(bar, 0);

  const uint32_t len = flen - 16;
  const uint32_t pay = rbase + head + 12;                         // payload offset inside the tile
  const uint32_t end = pay + len;
  const uint32_t g0 = (off - head) - rbase;                       // tile offset + g0 = offset in the batch (mod 2^32)
  Tile T;
  T.b = tile_b;
  asm volatile("mov.u32 %0, %1;" : "=r"(T.s) : "r"(smem_u32(tile_b)) : "memory");   // ordered after mbar_wait

  // =============================== warps W .. W+C-1: CRC ===============================
  if (wid >= PW) {
    const uint32_t cw = wid - PW;
    uint32_t* scrc = sseen + 128;
    const uint32_t* xp16 = s8 + 512;
    const bool on = active && A.verify;
    const uint32_t hn = min(len, (0u - pay) & 15u);
    const uint32_t b0 = pay + hn;                                  // 16-byte aligned, or the end of a tiny payload
    const uint32_t K = (end - b0) >> 4;
    if (on) {
      uint32_t c = 0;
      if (cw == 0) {
        c = 0xFFFFFFFFu;
        for (uint32_t i = 0; i < hn; ++i) c = crc_byte(s8, c, T.u8(pay + i));
      }
      if (cw == CW - 1) {
        // the frame index chained the headers without checking them on the fast path: check the length CRC here
        if (crc_mask(~crc_fold8(s8, 0xFFFFFFFFu, t_u32(T, pay - 12), t_u32(T, pay - 8))) != t_u32(T, pay - 4)) atomicOr(A.flags, TF_FALLBACK);
      }
      const uint32_t k0 = K * cw / CW, k1 = K * (cw + 1) / CW;
      c = crc_chunks(s8, T, b0 + 16 * k0, k1 - k0, c);
      if (c) atomicXor(&scrc[lane], K - k1 ? gf2_mulmod(K - k1 < 512u ? xp16[K - k1] : chunk_shift_far(xp16, K - k1), c) : c);
    }
    asm volatile("bar.sync 2, %0;" ::"r"(CW * 32) : "memory");
    if (cw == 0 && on) {
      uint32_t c = scrc[lane];
      for (uint32_t o = b0 + 16 * K; o < end; ++o) c = crc_byte(s8, c, T.u8(o));
      if (crc_mask(~c) != t_u32(T, end)) atomicOr(A.flags, TF_FALLBACK);        // the general path reports the error at the right record
    }
    if (cw == CW - 1 && A.pf_dist) {
      // The tile that will take this CTA's place when it retires (tiles start in index order, pf_dist = resident CTAs of the
      // whole GPU): ask L2 for its records now, so that its bulk copies find them there instead of in DRAM.  A tile spends
      // its first microseconds waiting for those copies with its shared memory allocated and idle.
      const uint32_t row2 = (tile + A.pf_dist) * TILE_ROWS + lane;
      if (row2 < n_rows) {
        const uint32_t o2 = A.rec_off[row2] + mis, e2 = min(A.rec_off[row2 + 1] + mis, lim & ~15u);
        const uint32_t a2 = (o2 + 15u) & ~15u;
        if (e2 > a2 + 16u) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + a2), "r"((e2 - a2) & ~15u) : "memory");
      }
    }
    return;
  }

  // =============================== warps 0..W-1: parse ===============================
  bool bad = false;
  uint32_t shape_bad = 0;
  unsigned long long seen_lo = 0, seen_hi = 0;
  uint32_t p = pay;
  uint32_t cend = end, fl_start = end, fl_end = end;        // context/features region = [p, cend), feature_lists = [fl_start, fl_end)
  if (active) {
    // Example { features = 1 } / SequenceExample { context = 1, feature_lists = 2 }: exactly these fields, in this order
    uint32_t L = 0;
    if (len < 2 || T.u8(p) != 0x0A) bad = true;
    else {
      ++p;
      if (!t_len(T, p, end, L) || end - p < L) bad = true;
      else if (!SEQ) { if (p + L != end) bad = true; }
      else {
        cend = p + L;
        uint32_t q = cend, L2 = 0;
        if (q >= end || T.u8(q) != 0x12) bad = true;
        else { ++q; if (!t_len(T, q, end, L2) || q + L2 != end) bad = true; else { fl_start = q; fl_end = end; } }
      }
    }
  }
  // 12 + 3 warps (TABLE): the last parse warp (it owns the fewest entries) builds the entry table, the parse warps wait for
  // it at the barrier and then take every entry from the table.  4 + 1 warps: small records, where a tile's life is a
  // latency chain and a walk in front of the barrier lengthens it (measured: the 220-byte string records lost 1.5 %, and
  // 3.5 % when the other warps parsed their first entry during the walk): each warp hops from its last entry to its next
  // one (PW - 1 hops) and checks that the chain ends exactly on cend.
  constexpr bool TABLE = PW >= 12;
  constexpr uint32_t walker = PW - 1;
  if (TABLE && wid == walker) {
    // ---- the entry table: ONE walk of the record's `0A elen` chain, which must end exactly on cend (the owners validate
    //      the entries themselves).  A broken chain is recorded as ~0 entries: every parse warp gives the row up. ----
    const uint32_t rows_e = tile_entry_rows(nf);
    uint32_t ne = 0, ni = 0;
    if (active && !bad) {
      uint32_t q = p;
      while (q < cend) {
        if (ne < rows_e && q - pay <= 0xffffu) { eoff[ne * 32u + lane] = (uint16_t)(q - pay); ni = ne + 1; }
        if (!t_next_entry(T, q, cend)) break;
        ++ne;
      }
      if (q != cend) ne = ~0u;
    }
    ecnt[lane] = ne;
    ecnt[32 + lane] = ni;
  }
  uint32_t skip = 0;                       // SequenceExample: feature_lists entries to pass before the next one this warp owns
  uint32_t i = wid;                        // the next entry this warp owns (entry index % W == wid)
  uint32_t next_f = wid;                   // in-order data: this warp's k-th owned entry is field wid + k*W
#pragma unroll 1
  for (uint32_t phase = TABLE ? 1u : 0u; phase < (TABLE ? 2u : 1u); ++phase) {     // 0: by hopping (4 + 1 warps); 1: from the table
    if (phase) {
      __syncwarp();                                  // (the lanes of a warp arrive together)
      asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
      if (active && ecnt[lane] == ~0u) bad = true;
    }
    if (!active) continue;
    while (!bad && i < (phase ? ecnt[lane] : ~0u)) {
      const uint32_t n_idx = phase ? ecnt[32 + lane] : 0u;   // entries in the table
      if (i < n_idx) p = pay + eoff[i * 32u + lane];
      else {
        // not in the table: hop on from the later of this warp's position (p: the start of the entry after its last one,
        // or of entry 0) and the table's last entry.  Without the table the chain is checked here: a hop that reaches cend
        // means there is no such entry, and the chain must end exactly there (below).
        uint32_t at = i >= PW ? i - (PW - 1) : 0u;
        if (at + 1 < n_idx) { at = n_idx - 1; p = pay + eoff[at * 32u + lane]; }
        for (; at < i && p < cend; ++at) if (!t_next_entry(T, p, cend)) { bad = true; break; }
        if (bad || p >= cend) break;
      }
      i += PW;
      // ---- owned entry: try the expected field's template first ----
      uint32_t eend, kind, llen;
      int f = -1;
      bool located = false;
      if (next_f < nf && stpl[next_f].n_words) {
        const FieldTemplate& tp = stpl[next_f];
        const uint32_t klen = tp.klen;
        // the entry's first 20 bytes as 5 words at any alignment: 6 aligned loads + funnel shifts (words past the template
        // have an all-zero mask)
        const uint32_t ab = p & ~3u, sh = (p & 3u) * 8;
        uint32_t aw[TILE_TPL_WORDS + 1];
#pragma unroll
        for (int w = 0; w <= TILE_TPL_WORDS; ++w) aw[w] = T.w32(ab + 4 * w);
        uint32_t diff = 0, u0 = 0;
#pragma unroll
        for (int w = 0; w < TILE_TPL_WORDS; ++w) {
          const uint32_t u = __funnelshift_r(aw[w], aw[w + 1], sh);
          if (w == 0) u0 = u;
          diff |= (u ^ tp.words[w]) & tp.mask[w];
        }
        const uint32_t elen = (u0 >> 8) & 0xff, vl = T.u8(p + 5 + klen), ll = T.u8(p + 7 + klen);
        // single-byte lengths that nest exactly: entry = key part (klen+2) + 2 + value; value = 2 + list.  The template
        // covers the kind tag, so the Feature's oneof member is already known to be the one the schema wants.
        if (diff == 0 && elen < 0x80 && elen == klen + 4 + vl && vl == ll + 2 && p + 2 + elen <= cend) {
          f = (int)next_f; eend = p + 2 + elen; located = true;
          kind = tp.kind; llen = ll;
          p += klen + 8;                                      // at the list body
        }
      }
      if (!located) {
        // ---- generic: 0A elen 0A klen key 12 vlen, key looked up by hash ----
        uint32_t elen, klen, vlen;
        if (T.u8(p) != 0x0A) { bad = true; break; }
        ++p;
        if (!t_len(T, p, cend, elen) || cend - p < elen) { bad = true; break; }
        eend = p + elen;
        if (p >= eend || T.u8(p) != 0x0A) { bad = true; break; }
        ++p;
        if (!t_len(T, p, eend, klen) || eend - p < klen) { bad = true; break; }
        const uint32_t key = p;
        p += klen;
        if (p >= eend || T.u8(p) != 0x12) { bad = true; break; }
        ++p;
        if (!t_len(T, p, eend, vlen) || p + vlen != eend) { bad = true; break; }
        uint32_t hi = 0;
        for (uint32_t i = 0; i < klen; ++i) hi |= T.u8(key + i);
        if (hi >= 0x80 && !utf8_valid(T.b + key, klen)) { bad = true; break; }   // malformed key: the general path reports it
        uint32_t h = name_hash(T.b + key, klen);
        uint32_t slot = h & (uint32_t)A.sch.ht_mask;
        for (;;) {
          int cand = A.sch.ht[slot];
          if (cand < 0) break;
          if (sfields[cand].hash == h && sfields[cand].name_len == klen) {
            const uint8_t* nm = snames + sfields[cand].name_off;
            uint32_t diff = 0;
            for (uint32_t i = 0; i < klen; ++i) diff |= T.u8(key + i) ^ nm[i];
            if (diff == 0) { f = cand; break; }
          }
          slot = (slot + 1) & (uint32_t)A.sch.ht_mask;
        }
        if (f >= 0 && sfields[f].elem_type == TFR_T_NULL) f = -1;               // NullType: always null, value only validated
        // ---- Feature: exactly one oneof member spanning the value ----
        if (vlen == 0) { if (f >= 0) bad = true; p = eend; continue; }            // kind not set: an error if the schema wants it
        const uint32_t kt = T.u8(p++);
        kind = kt == 0x0A ? K_BYTES : kt == 0x12 ? K_FLOAT : kt == 0x1A ? K_INT64 : K_NONE;
        if (kind == K_NONE || !t_len(T, p, eend, llen) || p + llen != eend) { bad = true; break; }
        if (f >= 0 && (uint32_t)sfields[f].kind != kind) { bad = true; break; }   // kind mismatch: error path
      }
      const DevField* fd = f >= 0 ? &sfields[f] : nullptr;
      if (fd) {
        const uint32_t bit = 1u << (f & 31);                                      // duplicate key (inside this warp's entries)
        if (f < 64) {
          const unsigned long long b64 = (unsigned long long)bit << (f & 32);
          if (seen_lo & b64) { bad = true; break; }
          seen_lo |= b64;
        } else {
          const unsigned long long b64 = (unsigned long long)bit << (f & 32);
          if (seen_hi & b64) { bad = true; break; }
          seen_hi |= b64;
        }
        next_f = (uint32_t)f + PW;
        if (fd->depth > 1) { bad = true; break; }                                 // nesting in a Feature: error path
      }
      if (kind == K_BYTES) {
        // BytesList: { 0A blen bytes }*
        uint32_t n = 0, first_off = 0, first_len = 0, first_data = 0, total = 0;
        bool xcode = false;                                                   // a string of this cell is malformed UTF-8 (ragged columns only)
        const uint32_t body = p;
        const bool is_str = fd && fd->elem_type == TFR_T_STRING;
        while (p < eend) {
          uint32_t bl;
          if (T.u8(p) != 0x0A) { bad = true; break; }
          ++p;
          const uint32_t lp = p;
          if (!t_len(T, p, eend, bl) || eend - p < bl) { bad = true; break; }
          if (is_str) {
            // StringType = Java UTF-8 decode/re-encode: identity for well-formed input.  Malformed input becomes U+FFFD per
            // malformed unit (java_utf8_transcode): a ragged column flags the cell, its length is corrected behind the parse
            // barrier and the copy-out re-encodes; a uniform or count-mode column leaves the row to the general path.
            uint32_t acc = 0;
            for (uint32_t i = 0; i < bl; ++i) acc |= T.u8(p + i);
            if (acc >= 0x80 && !utf8_valid(T.b + p, bl)) {
              if (RG && XC && A.uniform_len[fd->var_slot] == TILE_RAGGED) xcode = true;      // counted with its raw length here, fixed up behind the parse barrier
              else {
                if (RG && A.uniform_len[fd->var_slot] == TILE_RAGGED) atomicOr(A.flags, TF_XCODE);   // the XC instantiation can take this batch
                bad = true; break;
              }
            }
          }
          if (n == 0) { first_off = lp + g0; first_len = bl; first_data = p; }
          ++n; total += bl;
          p += bl;
        }
        if (bad) break;
        if (fd) {
          if (fd->depth == 0) {
            if (n == 0) { bad = true; break; }                                  // .head of an empty list: error path
            const int32_t ul = A.uniform_len[fd->var_slot];
            if (RG && ul == TILE_RAGGED) {
              // (a malformed string: the copy-out re-reads the raw length from the varint in front of the data)
              rg_src[fd->var_slot * 32 + lane] = first_data | (xcode ? 0x80000000u : 0u);
              rg_cnt[fd->cnt_slot * 32 + lane] = first_len;
              if (xcode) atomicOr(&sseen[161], 1u);
            } else if (ul >= 0) {
              if ((uint32_t)ul != first_len) shape_bad = 1;
              else {
                uint8_t* dst = reinterpret_cast<uint8_t*>(A.var_values[fd->var_slot]) + (size_t)row * (uint32_t)ul;
                if ((ul & 15) == 0) {
                  for (uint32_t i = 0; i < (uint32_t)ul; i += 16) {
                    uint4 v;
                    v.x = t_u32(T, first_data + i); v.y = t_u32(T, first_data + i + 4); v.z = t_u32(T, first_data + i + 8); v.w = t_u32(T, first_data + i + 12);
                    *reinterpret_cast<uint4*>(dst + i) = v;
                  }
                } else for (uint32_t i = 0; i < (uint32_t)ul; ++i) dst[i] = T.u8(first_data + i);
              }
            } else {
              A.cnt[(size_t)fd->cnt_slot * A.n + row] = first_len;
              A.src[(size_t)fd->var_slot * A.n + row] = first_off;
              A.cflag[(size_t)fd->var_slot * A.n + row] = CF_CANON;
            }
          } else {
            // ArrayType(String/Binary): two offset levels -> ragged or count mode (never uniform)
            if (RG && A.uniform_len[fd->var_slot] == TILE_RAGGED) {
              if (xcode) atomicOr(&sseen[161], 1u);
              rg_src[fd->var_slot * 32 + lane] = body | (xcode ? 0x80000000u : 0u);
              rg_cnt[fd->cnt_slot * 32 + lane] = n;
              rg_cnt[(fd->cnt_slot + 1) * 32 + lane] = total;
            } else {
            A.cnt[(size_t)fd->cnt_slot * A.n + row] = n;
            A.cnt[(size_t)(fd->cnt_slot + 1) * A.n + row] = total;
            A.src[(size_t)fd->var_slot * A.n + row] = body + g0;
            A.cflag[(size_t)fd->var_slot * A.n + row] = CF_CANON;
            }
          }
        }
      } else {
        // Int64List / FloatList: empty, or one packed field spanning the list
        uint32_t plen = 0, pk = p;
        if (llen != 0) {
          if (T.u8(p) != 0x0A) { bad = true; break; }
          ++p;
          if (!t_len(T, p, eend, plen) || p + plen != eend) { bad = true; break; }
          pk = p;
        }
        uint32_t n;
        uint64_t v0 = 0;
        if (kind == K_FLOAT) {
          if (plen & 3) { bad = true; break; }
          n = plen >> 2;
        } else {
          // varints: count terminators, every run <= 10 bytes, the last byte terminates; first value decoded on the way.
          // Up to 8 bytes are handled in registers: terminator bits by mask, the first varint's 7-bit groups compacted
          // with three shift-and-mask rounds.
          n = 0;
          if (plen >= 1 && plen <= 8) {
            const uint32_t w0 = t_u32(T, pk), w1 = plen > 4 ? t_u32(T, pk + 4) : 0u;
            unsigned long long x = ((unsigned long long)w1 << 32) | w0;
            const unsigned long long live = ~0ull >> (64 - 8 * plen);
            const unsigned long long term = ~x & 0x8080808080808080ull & live;          // MSB clear: a varint ends here
            if (!((term >> (8 * plen - 1)) & 1)) { bad = true; break; }                 // the last byte must terminate
            n = (uint32_t)__popcll(term);
            const uint32_t k0 = (uint32_t)__ffsll((long long)term);                     // 8 * length of the first varint
            x &= (~0ull >> (64 - k0)) & 0x7f7f7f7f7f7f7f7full;
            x = ((x & 0x7f007f007f007f00ull) >> 1) | (x & 0x007f007f007f007full);
            x = ((x & 0x3fff00003fff0000ull) >> 2) | (x & 0x00003fff00003fffull);
            x = ((x & 0x0fffffff00000000ull) >> 4) | (x & 0x000000000fffffffull);
            v0 = x;
          } else {
            uint32_t run = 0;
            for (uint32_t i = 0; i < plen; ++i) {
              uint32_t b = T.u8(pk + i);
              if (n == 0) v0 |= (uint64_t)(b & 0x7f) << (7 * run);
              if (b & 0x80) { if (++run >= 10) { bad = true; break; } } else { ++n; run = 0; }
            }
            if (bad || run) { bad = true; break; }
          }
        }
        if (fd) {
          if (fd->depth == 0) {
            if (n == 0) { bad = true; break; }
            void* vp = A.fix_values[fd->fix_slot];
            if (kind == K_FLOAT) {
              uint32_t bits = t_u32(T, pk);
              if (fd->elem_type == TFR_T_FLOAT32) reinterpret_cast<uint32_t*>(vp)[row] = bits;
              else reinterpret_cast<double*>(vp)[row] = (double)__uint_as_float(bits);
            } else {
              if (fd->elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(vp)[row] = (int64_t)v0;
              else reinterpret_cast<int32_t*>(vp)[row] = (int32_t)(uint32_t)v0;
            }
          } else {
            const int32_t ul = A.uniform_len[fd->var_slot];
            if (RG && ul == TILE_RAGGED) {
              rg_src[fd->var_slot * 32 + lane] = pk;
              rg_cnt[fd->cnt_slot * 32 + lane] = n;
            } else if (ul >= 0) {
              if ((uint32_t)ul != n) shape_bad = 1;
              else if (kind == K_FLOAT) {
                if (fd->elem_type == TFR_T_FLOAT32) {
                  uint32_t* dst = reinterpret_cast<uint32_t*>(A.var_values[fd->var_slot]) + (size_t)row * n;
                  if ((n & 3) == 0) {
                    for (uint32_t i = 0; i < n; i += 4) {
                      uint4 v;
                      v.x = t_u32(T, pk + 4 * i); v.y = t_u32(T, pk + 4 * i + 4); v.z = t_u32(T, pk + 4 * i + 8); v.w = t_u32(T, pk + 4 * i + 12);
                      *reinterpret_cast<uint4*>(dst + i) = v;
                    }
                  } else for (uint32_t i = 0; i < n; ++i) dst[i] = t_u32(T, pk + 4 * i);
                } else {
                  double* dst = reinterpret_cast<double*>(A.var_values[fd->var_slot]) + (size_t)row * n;
                  for (uint32_t i = 0; i < n; ++i) dst[i] = (double)__uint_as_float(t_u32(T, pk + 4 * i));
                }
              } else {
                uint32_t q = pk;
                for (uint32_t e = 0; e < n; ++e) {
                  uint64_t v = 0; uint32_t sh = 0;
                  for (;;) { uint32_t b = T.u8(q++); v |= (uint64_t)(b & 0x7f) << sh; sh += 7; if (b < 0x80) break; }
                  if (fd->elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(A.var_values[fd->var_slot])[(size_t)row * n + e] = (int64_t)v;
                  else reinterpret_cast<int32_t*>(A.var_values[fd->var_slot])[(size_t)row * n + e] = (int32_t)(uint32_t)v;
                }
              }
            } else {
              A.cnt[(size_t)fd->cnt_slot * A.n + row] = n;
              A.src[(size_t)fd->var_slot * A.n + row] = pk + g0;
              A.cflag[(size_t)fd->var_slot * A.n + row] = CF_CANON;
            }
          }
        }
      }
      p = eend;
    }
    if (!TABLE && p != cend) bad = true;
  }
  if (active) {
    if (TABLE) skip = i - ecnt[lane];
    // ---- SequenceExample.feature_lists: { 0A elen 0A klen key 12 vlen FeatureList }*, FeatureList = { 0A flen Feature }* ----
    // A SequenceExample typically has few FeatureLists with many steps each: handing whole entries to warps would leave most
    // of the tile's warps idle behind the one that walks a 64-step list.  Every parse warp therefore walks EVERY entry's
    // header and step chain (`0A flen` hops), but fully parses only the steps s with s % W == its index; element and byte
    // counts are summed per (row, column) in shared memory and written out after the parse barrier.  The entry's owner
    // (entry index % W, continuing the count of the context entries) does the per-entry bookkeeping.
    p = fl_start;
    while (SEQ && !bad && p < fl_end) {
      const bool owner = skip == 0;
      skip = owner ? PW - 1 : skip - 1;
      uint32_t elen, klen, vlen;
      if (T.u8(p) != 0x0A) { bad = true; break; }
      ++p;
      const uint32_t entry_pos = p;                           // the entry's length varint: what pass 2's FeatureList walker starts from
      if (!t_len(T, p, fl_end, elen) || fl_end - p < elen) { bad = true; break; }
      const uint32_t eend = p + elen;
      if (p >= eend || T.u8(p) != 0x0A) { bad = true; break; }
      ++p;
      if (!t_len(T, p, eend, klen) || eend - p < klen) { bad = true; break; }
      const uint32_t key = p;
      p += klen;
      if (p >= eend || T.u8(p) != 0x12) { bad = true; break; }
      ++p;
      if (!t_len(T, p, eend, vlen) || p + vlen != eend) { bad = true; break; }
      if (owner) {
        uint32_t hi = 0;
        for (uint32_t i = 0; i < klen; ++i) hi |= T.u8(key + i);
        if (hi >= 0x80 && !utf8_valid(T.b + key, klen)) { bad = true; break; }
      }
      int f = -1;
      {
        uint32_t h = name_hash(T.b + key, klen);
        uint32_t slot = h & (uint32_t)A.sch.ht_mask;
        for (;;) {
          int cand = A.sch.ht[slot];
          if (cand < 0) break;
          if (sfields[cand].hash == h && sfields[cand].name_len == klen) {
            const uint8_t* nm = snames + sfields[cand].name_off;
            uint32_t diff = 0;
            for (uint32_t i = 0; i < klen; ++i) diff |= T.u8(key + i) ^ nm[i];
            if (diff == 0) { f = cand; break; }
          }
          slot = (slot + 1) & (uint32_t)A.sch.ht_mask;
        }
      }
      if (f >= 0 && sfields[f].elem_type == TFR_T_NULL) f = -1;
      const DevField* fd = f >= 0 ? &sfields[f] : nullptr;
      if (fd) {
        if (fd->depth != 2) { bad = true; break; }            // array of heads / scalar from a FeatureList: general path
        if (owner) {
          unsigned long long bit = 1ull << (f & 63);
          // a name present in context AND feature_lists (context wins) or twice here: general path
          if (f < 64) { if (seen_lo & bit) { bad = true; break; } seen_lo |= bit; }
          else { if (seen_hi & bit) { bad = true; break; } seen_hi |= bit; }
        }
      }
      uint32_t steps = 0, tot_n = 0, tot_bytes = 0;
      const uint32_t steps_start = p;
      uint32_t my_step = wid;                                 // the next step this warp parses; the others it only hops over
      while (p < eend) {                                      // steps
        uint32_t flen;
        if (steps != my_step) {
          // not ours: `0A flen` -> one byte load + add (the step's owner checks the tag and the contents; an overshoot of the
          // chain is caught by p != eend behind the loop)
          const int32_t b1 = T.i8(p + 1);
          if (b1 >= 0) p += 2u + (uint32_t)b1;
          else { uint32_t q = p + 1; if (!t_len(T, q, eend, flen)) { bad = true; break; } p = q + flen; }
          ++steps;
          continue;
        }
        my_step += PW;
        if (T.u8(p) != 0x0A) { bad = true; break; }
        ++p;
        if (!t_len(T, p, eend, flen) || eend - p < flen) { bad = true; break; }
        const uint32_t fend = p + flen;
        const uint32_t step_idx = steps, n_before = tot_n;
        ++steps;
        if (flen == 0) { if (fd) bad = true; continue; }     // kind not set: an error if the schema wants the column
        uint32_t kt = T.u8(p++), llen;
        uint32_t kind = kt == 0x0A ? K_BYTES : kt == 0x12 ? K_FLOAT : kt == 0x1A ? K_INT64 : K_NONE;
        if (kind == K_NONE || !t_len(T, p, fend, llen) || p + llen != fend) { bad = true; break; }
        if (fd && (uint32_t)fd->kind != kind) { bad = true; break; }
        if (kind == K_BYTES) {
          const bool is_str = fd && fd->elem_type == TFR_T_STRING;
          while (p < fend) {
            uint32_t bl;
            if (T.u8(p) != 0x0A) { bad = true; break; }
            ++p;
            if (!t_len(T, p, fend, bl) || fend - p < bl) { bad = true; break; }
            if (is_str) {
              uint32_t acc = 0;
              for (uint32_t i = 0; i < bl; ++i) acc |= T.u8(p + i);
              if (acc >= 0x80 && !utf8_valid(T.b + p, bl)) { bad = true; break; }
            }
            ++tot_n; tot_bytes += bl;
            p += bl;
          }
          if (bad) break;
        } else if (llen != 0) {
          uint32_t plen;
          if (T.u8(p) != 0x0A) { bad = true; break; }
          ++p;
          if (!t_len(T, p, fend, plen) || p + plen != fend) { bad = true; break; }
          if (kind == K_FLOAT) {
            if (plen & 3) { bad = true; break; }
            tot_n += plen >> 2;
          } else {
            uint32_t run = 0;
            for (uint32_t i = 0; i < plen; ++i) {
              if (T.u8(p + i) & 0x80) { if (++run >= 10) { bad = true; break; } } else { ++tot_n; run = 0; }
            }
            if (bad || run) { bad = true; break; }
          }
        }
        if (RG && fd && A.uniform_len[fd->var_slot] == TILE_RAGGED) {
          // one-pass mode: the copy-out needs every step's element count (its place in the row = the sum of the steps before it)
          const uint32_t cstep = tot_n - n_before;
          if (step_idx >= TILE_SQ_STEPS || cstep > 255u) { bad = true; break; }
          sq_tab[((uint32_t)fd->var_slot * TILE_SQ_STEPS + step_idx) * 32u + lane] = (uint8_t)cstep;
        }
        p = fend;
      }
      if (bad || p != eend) { bad = true; break; }
      if (fd) {
        if (tot_n) atomicAdd(&sq_cnt[(fd->var_slot * 32 + lane) * 2], tot_n);
        if (tot_bytes) atomicAdd(&sq_cnt[(fd->var_slot * 32 + lane) * 2 + 1], tot_bytes);
        if (owner) {
          if (RG && A.uniform_len[fd->var_slot] == TILE_RAGGED) {
            if (steps > TILE_SQ_STEPS) { bad = true; break; }
            rg_src[fd->var_slot * 32 + lane] = steps_start;              // where the steps begin; their number is the level-0 count
            rg_cnt[fd->cnt_slot * 32 + lane] = steps;
          } else {
            A.cnt[(size_t)fd->cnt_slot * A.n + row] = steps;
            A.src[(size_t)fd->var_slot * A.n + row] = entry_pos + g0;
            A.cflag[(size_t)fd->var_slot * A.n + row] = CF_FLIST;
          }
        }
      }
      p = eend;
    }
    if (!bad && p != fl_end) bad = true;
  }
  // ---- merge the parse warps' seen masks (a key seen by two warps is a duplicate: last-wins -> general path) ----
  {
    const uint32_t w4[4] = {(uint32_t)seen_lo, (uint32_t)(seen_lo >> 32), (uint32_t)seen_hi, (uint32_t)(seen_hi >> 32)};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (w4[k] && (atomicOr(&sseen[lane * 4 + k], w4[k]) & w4[k])) bad = true;
    if (bad) atomicOr(&sseen[160], 1u << lane);            // this row goes to the general path whatever else happens to it
  }
  asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
  if (RG) {
    // ================= ragged columns, finished in this pass =================
    if (XC && sseen[161]) {
      // Some string cell of this tile holds malformed UTF-8 (rare): its bytes in the column are the Java re-encoding, whose
      // length replaces the raw one before the offsets are computed.  Kept out of the parse loop (calls there cost the hot
      // path registers).
      for (uint32_t v = wid; v < (uint32_t)A.sch.n_var; v += PW) {
        const DevField& fd = sfields[A.var_field[v]];
        // (the source word of an absent or empty cell was never written: the count decides first)
        if (A.uniform_len[v] != TILE_RAGGED || fd.elem_type != TFR_T_STRING || !active || rg_cnt[fd.cnt_slot * 32 + lane] == 0u || !(rg_src[v * 32 + lane] >> 31)) continue;
        const uint32_t src = rg_src[v * 32 + lane] & 0x7fffffffu;
        if (fd.depth == 0) {
          uint32_t k = 1;
          while (k < 5 && (T.u8(src - 1 - k) & 0x80u)) ++k;                       // the raw length: the varint in front of the data
          uint32_t q = src - k, raw = 0;
          t_len(T, q, src, raw);
          rg_cnt[fd.cnt_slot * 32 + lane] = t_xcode_cell(T.b + src, raw, nullptr);
        } else if (fd.depth == 1) {
          const uint32_t cnt = rg_cnt[fd.cnt_slot * 32 + lane];
          uint32_t q = src, tot = 0;
          for (uint32_t i = 0; i < cnt; ++i) { uint32_t bl = 0; ++q; t_len(T, q, q + 5, bl); tot += t_xcode_cell(T.b + q, bl, nullptr); q += bl; }
          rg_cnt[(fd.cnt_slot + 1) * 32 + lane] = tot;
        }
      }
      asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
    }
    if (SEQ) {                                                                    // FeatureList columns: the warps' summed element counts
      for (uint32_t v = wid; v < (uint32_t)A.sch.n_var; v += PW) {
        const DevField& fd = sfields[A.var_field[v]];
        if (fd.depth == 2 && A.uniform_len[v] == TILE_RAGGED) rg_cnt[(fd.cnt_slot + 1) * 32 + lane] = sq_cnt[(v * 32 + lane) * 2];
      }
      asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
    }
    // (T) tile-local exclusive prefix of every count array over the 32 rows (lane = row); array a by warp a % W.  The tile's
    //     totals go out to the look-back table right away.
    const uint32_t nc = A.n_cnt, nc4 = (nc + 3u) & ~3u;                            // table rows are padded to whole uint4
    const uint32_t ptid = threadIdx.x;                                              // 0 .. W*32-1 (parse warps come first)
    for (uint32_t a = wid; a < nc; a += PW) {
      const uint32_t c = rg_cnt[a * 32 + lane];
      uint32_t tot;
      const uint32_t ex = warp_excl_scan_u32(c, tot);
      rg_cnt[a * 32 + lane] = ex;
      if (lane == 0) { rg_tot[a] = tot; rg_base[a] = 0ull; A.lb_agg[(size_t)tile * nc4 + a] = tot; }
    }
    asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
    if (ptid == 0) { __threadfence(); st_release_u32(&A.lb_flag[tile], 1u); }
    // (L) bases across tiles (decoupled look-back).  All parse warps look at once: thread j reads the flag of tile p - j
    //     (W*32 predecessors per round), the warps agree through shared memory on the nearest predecessor whose inclusive
    //     prefix is known (G_pre) and on whether every tile in front of it has published its totals; then the W*32 threads
    //     share the (tile, four arrays) loads -- one L2 round trip whatever the number of arrays -- and add them into the
    //     tile's bases with shared-memory atomics.
    {
      uint32_t* lbs = rg_tile + 2;                                                  // [W] per-warp summary: first prefix | first empty << 8
      int32_t p = (int32_t)tile - 1;
      uint32_t spins = 0;
      bool give_up = false;
      while (p >= 0) {
        const int32_t q = p - (int32_t)ptid;
        const uint32_t fl = q >= 0 ? ld_acquire_u32(&A.lb_flag[q]) : 2u;            // in front of tile 0: prefix 0
        const uint32_t pre_mask = __ballot_sync(FULLMASK, fl == 2u), emp_mask = __ballot_sync(FULLMASK, fl == 0u);
        if (lane == 0) lbs[wid] = (pre_mask ? (uint32_t)__ffs((int)pre_mask) - 1u : 32u) | ((emp_mask ? (uint32_t)__ffs((int)emp_mask) - 1u : 32u) << 8);
        asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
        // nearest known prefix / nearest unpublished tile over all windows: lane w reads warp w's summary, two warp reductions
        const uint32_t sx = lane < PW ? lbs[lane] : 0x2020u;
        const uint32_t g_pre = __reduce_min_sync(FULLMASK, (sx & 0xffu) < 32u ? 32u * lane + (sx & 0xffu) : 0xffffu);
        const uint32_t g_emp = __reduce_min_sync(FULLMASK, (sx >> 8) < 32u ? 32u * lane + (sx >> 8) : 0xffffu);
        const uint32_t span = min(g_pre, (uint32_t)(PW * 32 - 1));    // predecessors p .. p - span are needed
        if (g_emp <= span) {                                                        // one of them has not published yet
          // never hang: the batch may have been abandoned (another tile raised the fallback flag)
          ++spins;
          if (ptid == 0 && (spins & 31u) == 0u && ((ld_cg_u32(A.flags) & TF_FALLBACK) || spins > (1u << 22))) lbs[PW] = 1u;
          asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");  // everybody has read lbs before it is rewritten
          if (lbs[PW]) { give_up = true; break; }                    // one thread decides, all follow: the barriers stay matched
          __nanosleep(100);
          continue;
        }
        // (the flags were read with acquire loads at GPU scope and the values are read from L2: no further fence)
        // unit = (four arrays, 32 predecessors): lane = predecessor, one 16-byte load each, one warp reduction (REDUX) per
        // array, one shared-memory atomic per array and unit; the predecessor whose inclusive prefix is known adds its own
        const uint32_t chunks = nc4 >> 2, groups = (span >> 5) + 1u;
        for (uint32_t u = wid; u < chunks * groups; u += PW) {
          const uint32_t c4 = (u % chunks) * 4u, g = (u / chunks) * 32u + lane;
          const int32_t t2 = p - (int32_t)g;
          uint4 v = make_uint4(0u, 0u, 0u, 0u);
          if (g < g_pre && g <= span && t2 >= 0)
            asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(A.lb_agg + (size_t)t2 * nc4 + c4) : "memory");
          else if (g == g_pre && t2 >= 0) {
            const unsigned long long* r = A.lb_pre + (size_t)t2 * nc4 + c4;
#pragma unroll
            for (uint32_t j = 0; j < 4; ++j) if (c4 + j < nc) { const unsigned long long x = ld_cg_u64(r + j); if (x) atomicAdd(&rg_base[c4 + j], x); }
          }
          const uint32_t s0 = __reduce_add_sync(FULLMASK, v.x), s1 = __reduce_add_sync(FULLMASK, v.y), s2 = __reduce_add_sync(FULLMASK, v.z), s3 = __reduce_add_sync(FULLMASK, v.w);
          if (lane == 0) {                                                          // (32 tiles x < 2^26 bytes each: no overflow)
            if (s0) atomicAdd(&rg_base[c4], (unsigned long long)s0);
            if (s1) atomicAdd(&rg_base[c4 + 1], (unsigned long long)s1);
            if (s2) atomicAdd(&rg_base[c4 + 2], (unsigned long long)s2);
            if (s3) atomicAdd(&rg_base[c4 + 3], (unsigned long long)s3);
          }
        }
        asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
        if (g_pre < (uint32_t)(PW * 32)) break;
        p -= PW * 32;
      }
      // this tile's inclusive prefixes: published by warp 0; capacity / int32 checks
      if (wid == 0) {
        bool over = false;
        for (uint32_t a = lane; a < nc; a += 32) {
          const unsigned long long incl = rg_base[a] + rg_tot[a];
          A.lb_pre[(size_t)tile * nc4 + a] = incl;
          if (incl > A.cap[a] || incl > 0x7fffffffull) over = true;                 // target buffer (or int32 offsets) too small: the host redoes the batch
          if (row0 + TILE_ROWS >= n_rows) A.totals[a] = incl;                        // the last tile knows the grand totals
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release_u32(&A.lb_flag[tile], 2u);
        over = __any_sync(FULLMASK, over);
        if ((give_up || over) && lane == 0) { rg_tile[1] = 1u; atomicOr(A.flags, over ? (TF_OVERFLOW | TF_FALLBACK) : TF_FALLBACK); }
      }
    }
    asm volatile("bar.sync 1, %0;" ::"r"(PW * 32) : "memory");
    // (C) offsets + values: column v by warp v % W, lane = row.  Cells of consecutive rows are adjacent in the output.
    if (!rg_tile[1]) {
      if (SEQ) {
        // FeatureList columns (list<list<T>>, fixed-width T): EVERY warp walks the row's step chain again (one byte load per
        // step) adding up the steps' element counts from the table the parse filled, and emits the steps s with s % W == its
        // index: inner offset + values.  (One warp per column would leave the tile's other warps idle behind a 64-step walk.)
        for (uint32_t v = 0; v < (uint32_t)A.sch.n_var; ++v) {
          const DevField& fd = sfields[A.var_field[v]];
          if (fd.depth != 2 || A.uniform_len[v] != TILE_RAGGED || !active) continue;
          const uint32_t a0 = (uint32_t)fd.cnt_slot;
          const uint32_t ex0 = rg_cnt[a0 * 32 + lane], ex1 = rg_cnt[(a0 + 1) * 32 + lane];
          const uint32_t c0 = (lane == 31 ? rg_tot[a0] : rg_cnt[a0 * 32 + lane + 1]) - ex0;     // steps of this row
          const uint32_t c1 = (lane == 31 ? rg_tot[a0 + 1] : rg_cnt[(a0 + 1) * 32 + lane + 1]) - ex1;   // elements of this row
          const unsigned long long b0 = rg_base[a0], b1 = rg_base[a0 + 1];
          int32_t* o1 = A.offs[v * 3 + 1];
          if (wid == v % PW) {
            int32_t* o0 = A.offs[v * 3];
            o0[row] = (int32_t)(b0 + ex0);
            if (row + 1 == n_rows) { o0[n_rows] = (int32_t)(b0 + ex0 + c0); o1[b0 + ex0 + c0] = (int32_t)(b1 + ex1 + c1); }
          }
          uint8_t* vals = reinterpret_cast<uint8_t*>(A.var_values[v]);
          const uint8_t* tab = sq_tab + (size_t)v * TILE_SQ_STEPS * 32u + lane;
          uint32_t q = rg_src[v * 32 + lane], run = 0, my_step = wid;
          for (uint32_t st = 0; st < c0; ++st) {
            uint32_t fl = T.u8(q + 1), hq = q + 2;                                   // `0A flen`
            if (fl >= 0x80u) { hq = q + 1; t_len(T, hq, q + 6, fl); }
            const uint32_t cn = tab[st * 32u];
            if (st == my_step) {
              my_step += PW;
              const unsigned long long e0 = b1 + ex1 + run;
              o1[b0 + ex0 + st] = (int32_t)e0;
              if (cn) {
                // Feature = kind llen 0A plen packed (validated canonical by the parse): skip the two headers
                uint32_t x = hq + 1, l2;
                t_len(T, x, hq + 6, l2);                                             // list length
                ++x;                                                                 // 0A
                t_len(T, x, x + 5, l2);                                              // packed length
                if (fd.kind == K_FLOAT) {
                  if (fd.elem_type == TFR_T_FLOAT32) { uint32_t* d = reinterpret_cast<uint32_t*>(vals) + e0; for (uint32_t i = 0; i < cn; ++i) d[i] = t_u32(T, x + 4 * i); }
                  else { double* d = reinterpret_cast<double*>(vals) + e0; for (uint32_t i = 0; i < cn; ++i) d[i] = (double)__uint_as_float(t_u32(T, x + 4 * i)); }
                } else {
                  for (uint32_t i = 0; i < cn; ++i) {
                    uint64_t y = 0; uint32_t sh = 0;
                    for (;;) { const uint32_t b = T.u8(x++); y |= (uint64_t)(b & 0x7f) << sh; sh += 7; if (b < 0x80) break; }
                    if (fd.elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(vals)[e0 + i] = (int64_t)y;
                    else reinterpret_cast<int32_t*>(vals)[e0 + i] = (int32_t)(uint32_t)y;
                  }
                }
              }
            }
            run += cn;
            q = hq + fl;
          }
        }
      }
      for (uint32_t v = wid; v < (uint32_t)A.sch.n_var; v += PW) {
        if (A.uniform_len[v] != TILE_RAGGED) continue;
        const DevField& fd = sfields[A.var_field[v]];
        if (fd.depth == 2) continue;                           // (done above)
        const uint32_t a0 = (uint32_t)fd.cnt_slot;
        const uint32_t ex0 = rg_cnt[a0 * 32 + lane];
        const uint32_t c0 = (lane == 31 ? rg_tot[a0] : rg_cnt[a0 * 32 + lane + 1]) - ex0;       // this row's count at level 0
        const unsigned long long b0 = rg_base[a0];
        const bool last_row = row + 1 == n_rows;
        if (!active) continue;
        int32_t* o0 = A.offs[v * 3];
        o0[row] = (int32_t)(b0 + ex0);
        if (last_row) o0[n_rows] = (int32_t)(b0 + ex0 + c0);
        if (c0 == 0) { if (last_row && fd.n_levels == 2) A.offs[v * 3 + 1][b0 + ex0] = (int32_t)(rg_base[a0 + 1] + rg_cnt[(a0 + 1) * 32 + lane]); continue; }
        const uint32_t src = rg_src[v * 32 + lane] & 0x7fffffffu;
        const bool xcode = rg_src[v * 32 + lane] >> 31;          // a malformed UTF-8 string in this cell: re-encode instead of copy
        uint8_t* vals = reinterpret_cast<uint8_t*>(A.var_values[v]);
        if (fd.depth == 0) {                                   // scalar string / binary: c0 bytes
          if (XC && xcode) {
            // raw length: the varint that ends right in front of the data (its last byte has the top bit clear, the ones before
            // it set; the tag 0A in front of it has it clear again)
            uint32_t k = 1;
            while (k < 5 && (T.u8(src - 1 - k) & 0x80u)) ++k;
            uint32_t q = src - k, raw = 0;
            t_len(T, q, src, raw);
            if (XC) t_xcode_cell(T.b + src, raw, vals + b0 + ex0);
          }
          else t_copy_out(T, src, vals + b0 + ex0, c0);
        } else if (fd.kind == K_FLOAT) {                       // packed floats
          if (fd.elem_type == TFR_T_FLOAT32) { uint32_t* d = reinterpret_cast<uint32_t*>(vals) + b0 + ex0; for (uint32_t i = 0; i < c0; ++i) d[i] = t_u32(T, src + 4 * i); }
          else { double* d = reinterpret_cast<double*>(vals) + b0 + ex0; for (uint32_t i = 0; i < c0; ++i) d[i] = (double)__uint_as_float(t_u32(T, src + 4 * i)); }
        } else if (fd.kind == K_INT64) {                       // packed varints (validated by the parse)
          uint32_t q = src;
          for (uint32_t i = 0; i < c0; ++i) {
            uint64_t x = 0; uint32_t sh = 0;
            for (;;) { const uint32_t b = T.u8(q++); x |= (uint64_t)(b & 0x7f) << sh; sh += 7; if (b < 0x80) break; }
            if (fd.elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(vals)[b0 + ex0 + i] = (int64_t)x;
            else reinterpret_cast<int32_t*>(vals)[b0 + ex0 + i] = (int32_t)(uint32_t)x;
          }
        } else {                                               // list of strings / binaries: { 0A blen bytes }*, inner offsets + bytes
          int32_t* o1 = A.offs[v * 3 + 1];
          unsigned long long vpos = rg_base[a0 + 1] + rg_cnt[(a0 + 1) * 32 + lane];
          uint32_t q = src;
          for (uint32_t i = 0; i < c0; ++i) {
            uint32_t bl = 0;
            ++q;                                               // 0A
            uint32_t qq = q;
            t_len(T, qq, q + 5, bl);
            q = qq;
            o1[b0 + ex0 + i] = (int32_t)vpos;
            if (XC && xcode) vpos += t_xcode_cell(T.b + q, bl, vals + vpos);
            else { t_copy_out(T, q, vals + vpos, bl); vpos += bl; }
            q += bl;
          }
          if (last_row) o1[b0 + ex0 + c0] = (int32_t)vpos;
        }
      }
    }
  }
  {
    // a row that some warp gave up on has fields that were never looked at: their absence says nothing about the shapes
    const bool row_bad = (sseen[160] >> lane) & 1u;
    // ---- validity bitmaps by ballot (rows are 32-aligned), absent fields -> null / error; field f is finished by warp f % W ----
    uint32_t all[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) all[k] = sseen[lane * 4 + k];
    const uint32_t act_mask = __ballot_sync(FULLMASK, active);
    for (uint32_t f = wid; f < nf; f += PW) {
      const uint32_t wsel = f < 32 ? all[0] : f < 64 ? all[1] : f < 96 ? all[2] : all[3];
      const bool present = (wsel >> (f & 31)) & 1;
      const uint32_t m = __ballot_sync(FULLMASK, present && active);
      if (SEQ && active && present && sfields[f].depth == 2 && A.cnt) {      // FeatureList column: the warps' partial counts
        const DevField& fd = sfields[f];
        A.cnt[(size_t)(fd.cnt_slot + 1) * A.n + row] = sq_cnt[(fd.var_slot * 32 + lane) * 2];
        if (fd.n_levels == 3) A.cnt[(size_t)(fd.cnt_slot + 2) * A.n + row] = sq_cnt[(fd.var_slot * 32 + lane) * 2 + 1];
      }
      if (active && !present && sfields[f].elem_type != TFR_T_NULL) {
        const DevField& fd = sfields[f];
        if (!fd.nullable) bad = true;                                         // NullPointerException: error path
        if (fd.fix_slot >= 0) {
          void* vp = A.fix_values[fd.fix_slot];
          if (fd.width == 8) reinterpret_cast<uint64_t*>(vp)[row] = 0; else reinterpret_cast<uint32_t*>(vp)[row] = 0;
        } else if (fd.var_slot >= 0) {
          const int32_t ul = A.uniform_len[fd.var_slot];
          if (ul > 0 && !row_bad) shape_bad = 1;                              // a null row has no values: not uniform
          else if (ul == -1) for (int l = 0; l < fd.n_levels; ++l) A.cnt[(size_t)(fd.cnt_slot + l) * A.n + row] = 0;
        }
      }
      if (lane == 0) {
        reinterpret_cast<uint32_t*>(A.bitmaps + (size_t)f * A.nb_stride)[tile] = m;
        const uint32_t nulls = __popc(act_mask & ~m);
        if (nulls) atomicAdd(&A.null_counts[f], (unsigned long long)nulls);
      }
    }
  }
  if (bad) atomicOr(A.flags, TF_FALLBACK);
  if (shape_bad) atomicOr(A.flags, TF_SHAPE | TF_FALLBACK);
}

// offsets of a uniform column: offs[i] = i * L  (i = 0..n); n is read from the device when n_dev is given (pipelined submit:
// the kernel runs on the frame-index stream, under the previous batch's tile kernel) and nothing is written when it exceeds
// the capacity the arrays were sized for
__global__ void uniform_offsets_kernel(int32_t* const* __restrict__ offs, uint32_t stride, const int32_t* __restrict__ uniform_len, uint32_t n_var,
                                       uint32_t n, const uint32_t* __restrict__ n_dev) {
  const uint32_t v = blockIdx.y;
  if (v >= n_var) return;
  if (n_dev) { const uint32_t m = *n_dev; if (m > n) return; n = m; }
  const int32_t L = uniform_len[v];
  if (L < 0) return;
  int32_t* o = offs[v * stride];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) o[i] = (int32_t)(i * (uint32_t)L);
}
