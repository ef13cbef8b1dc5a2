// api.cu -- the C ABI of libtfrgpu.so (include/tfrgpu.h) and the host-side runtime above the kernels:
// schema lowering, per-task decoder/encoder handles (device + stream + reusable buffers), batch
// ownership, host copies and Arrow C Data Interface export.  No torch types, no CPU fallback: every
// compute path below launches the sm_90a kernels of frame.cuh / decode.cuh / scan.cuh / encode.cuh.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>      // header-only NVTX 3: ranges show up in Nsight Systems / ncu --nvtx, cost nothing when no tool is attached
#include <algorithm>
#include <cmath>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "drop.cuh"
#include "encode.cuh"
#include "encode_tile.cuh"
#include "bytes_tile.cuh"
#include "frame.cuh"
#include "host_util.h"
#include "index.cuh"
#include "infer.cuh"
#include "large.cuh"
#include "narrow.cuh"
#include "permissive.cuh"
#include "position.cuh"
#include "ragged.cuh"
#include "resync.cuh"
#include "rows.cuh"
#include "scan.cuh"
#include "tile.cuh"
#include "urows.cuh"

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static int32_t fail(int32_t code, const std::string& msg) { g_last_error = msg; return code; }
#define CUDA_TRY(expr)                                                                             \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) return fail(TFR_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

static int32_t dev_alloc_status(cudaError_t e) {
  if (e != cudaSuccess) return fail(e == cudaErrorMemoryAllocation ? TFR_E_OOM : TFR_E_CUDA, std::string("device allocation failed: ") + cudaGetErrorString(e));
  return TFR_OK;
}
int32_t DevBuf::ensure(size_t bytes) { return dev_alloc_status(ensure_raw(bytes)); }
int32_t DevBuf::ensure_exact(size_t bytes) { return bytes <= cap ? TFR_OK : dev_alloc_status(alloc(bytes)); }
#define TRY(expr) do { int32_t _rc = (expr); if (_rc) return _rc; } while (0)

// NVTX range over one C-ABI call (SURVEY.md section 5: the tracing hook of this path)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

extern "C" int32_t tfr_abi_version(void) { return TFR_ABI_VERSION; }
extern "C" const char* tfr_last_error(void) { return g_last_error.c_str(); }
extern "C" const char* tfr_status_string(int32_t s) {
  switch (s) {
    case TFR_OK: return "ok";
    case TFR_E_INVALID_ARG: return "invalid argument";
    case TFR_E_UNSUPPORTED_TYPE: return "unsupported data type";
    case TFR_E_BAD_RECORD_TYPE: return "unsupported recordType: recordType can be ByteArray, Example or SequenceExample";
    case TFR_E_CUDA: return "CUDA error / no usable device";
    case TFR_E_OOM: return "out of memory";
    case TFR_E_BATCH_TOO_LARGE: return "batch too large (2 GiB of framed bytes / int32 Arrow offsets)";
    case TFR_E_CRC_LENGTH: return "Length header crc32 checking failed";
    case TFR_E_CRC_DATA: return "Data crc32 checking failed";
    case TFR_E_TRUNCATED: return "End of file reached before reading fully";
    case TFR_E_RECORD_TOO_LARGE: return "Record size exceeds max value of int32";
    case TFR_E_MALFORMED_PROTO: return "Protocol message was malformed";
    case TFR_E_KIND_MISMATCH: return "Feature must be of the list kind the column type requires";
    case TFR_E_EMPTY_SCALAR: return "head of empty list";
    case TFR_E_NULL_IN_NONNULL: return "field does not allow null values";
    case TFR_E_BAD_NESTING: return "Cannot convert Feature/FeatureList to this array nesting";
    case TFR_E_INDEX_MISMATCH: return "record index does not describe its file";
    default: return "unknown status";
  }
}

// ---------------------------------------------------------------------------------------------
// per-device context: CRC tables
// ---------------------------------------------------------------------------------------------
struct DeviceCtx {
  std::once_flag once;
  CrcTables* d_tabs = nullptr;
  cudaError_t err = cudaSuccess;
  int sm_count = 132;
  int max_smem_optin = 48 * 1024;
  size_t smem_per_sm = 233472;        // 228 KB on sm_90; tile geometry packs CTAs into this (1 KB reserved per resident CTA)
};
static DeviceCtx g_ctx[64];

static void build_crc_tables(CrcTables& t) {
  const uint32_t POLY = 0x82F63B78u;
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (POLY & (0u - (c & 1u)));
    t.t0[i] = c;
  }
  auto mulmod = [&](uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 31; i >= 0; --i) {
      if ((a >> i) & 1u) p ^= b;
      b = (b >> 1) ^ (POLY & (0u - (b & 1u)));
    }
    return p;
  };
  auto xpow_bytes = [&](uint32_t nbytes) {     // x^(8*nbytes) mod P
    uint32_t x8 = 0x80000000u;
    for (int i = 0; i < 8; ++i) x8 = (x8 >> 1) ^ (POLY & (0u - (x8 & 1u)));
    uint32_t r = 0x80000000u, base = x8;
    while (nbytes) { if (nbytes & 1) r = mulmod(r, base); base = mulmod(base, base); nbytes >>= 1; }
    return r;
  };
  uint32_t x128 = xpow_bytes(128);
  for (int s = 0; s < 4; ++s)
    for (uint32_t b = 0; b < 256; ++b) t.k128[s][b] = mulmod(x128, b << (8 * s));
  for (uint32_t k = 0; k < 40; ++k) t.xw[k] = xpow_bytes(4 * k);
  for (uint32_t i = 0; i < 256; ++i) {
    t.s8[0][i] = t.t0[i];
    for (int k = 1; k < 8; ++k) t.s8[k][i] = (t.s8[k - 1][i] >> 8) ^ t.t0[t.s8[k - 1][i] & 0xff];
  }
  for (uint32_t m = 0; m < 512; ++m) t.xp16[m] = xpow_bytes(16 * m);
  for (uint32_t k = 0; k < 32; ++k) t.x8pow[k] = xpow_bytes(1u << k);
  memset(t.g5, 0, sizeof t.g5);
  for (uint32_t k = 0; k < 13; ++k)
    for (uint32_t v = 0; v < 32; ++v) {
      uint32_t r = 0;
      for (uint32_t j = 0; j < 5; ++j) {
        const uint32_t bit = 5 * k + j;
        if (((v >> j) & 1u) && bit < 64) r ^= t.s8[7 - bit / 8][1u << (bit % 8)];
      }
      t.g5[k * 32 + v] = r;
    }
  for (uint32_t v = 0; v < 32; ++v) t.g5[416 + v] = t.t0[v];
  for (uint32_t w = 0; w < 8; ++w) t.g5[448 + w] = t.t0[w << 5];
}

static int32_t get_ctx(int device, DeviceCtx** out) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail(TFR_E_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e));
  if (device < 0 || device >= ndev || device >= 64) return fail(TFR_E_INVALID_ARG, "bad device index");
  DeviceCtx& c = g_ctx[device];
  std::call_once(c.once, [&] {
    c.err = cudaSetDevice(device);
    if (c.err != cudaSuccess) return;
    cudaDeviceProp prop;
    c.err = cudaGetDeviceProperties(&prop, device);
    if (c.err != cudaSuccess) return;
    c.sm_count = prop.multiProcessorCount;
    c.max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    c.smem_per_sm = prop.sharedMemPerMultiprocessor;
    {   // keep stream-ordered allocations cached in the pool instead of returning them to the OS at every sync
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        unsigned long long thr = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
      }
    }
    // every handle's kernels read the tables from non-blocking streams, which are not ordered after the legacy default
    // stream: the copy is complete before any handle of this device exists
    auto h = std::make_unique<CrcTables>();
    build_crc_tables(*h);
    Stream st;
    c.err = st.create();
    // a raw allocation on purpose: the tables live as long as the process.  g_ctx is static, and an owner's destructor would
    // free them at exit, after the CUDA runtime has shut down.
    if (c.err == cudaSuccess) c.err = cudaMalloc(&c.d_tabs, sizeof(CrcTables));
    if (c.err == cudaSuccess) c.err = cudaMemcpyAsync(c.d_tabs, h.get(), sizeof(CrcTables), cudaMemcpyHostToDevice, st);
    if (c.err == cudaSuccess) c.err = cudaStreamSynchronize(st);
  });
  if (c.err != cudaSuccess) return fail(TFR_E_CUDA, std::string("device init: ") + cudaGetErrorString(c.err));
  *out = &c;
  return TFR_OK;
}

// ---------------------------------------------------------------------------------------------
// schema
// ---------------------------------------------------------------------------------------------
struct tfr_schema {
  int32_t record_type = 0;
  std::vector<DevField> fields;      // device layout, filled on the host
  std::vector<uint8_t> names;
  std::vector<int32_t> ht;
  std::vector<int32_t> var_field;    // var slot -> field
  std::vector<int32_t> fix_field;    // fix slot -> field
  int32_t n_fix = 0, n_var = 0, n_cnt = 0;
  // the generated fields (TFR_T_ROW_INDEX, TFR_T_RECORD_OFFSET): their field, -1 none.  Lowered to nullable int64 columns that
  // are left out of the key hash table; position_kernel fills them.
  int32_t gen_field[2] = {-1, -1};
  bool generated(int32_t f) const { return f >= 0 && (f == gen_field[0] || f == gen_field[1]); }
  bool has_generated() const { return gen_field[0] >= 0 || gen_field[1] >= 0; }
  // VectorUDT fields (include/tfrgpu.h, VECTORS, SPARSE VECTORS): VK_* per lowered field.  Lowered to ordinary fields (a dense
  // vector: a float64 list; a sparse one: its values, and its indices and size appended after the caller's n_user fields), so
  // every parse and encode kernel treats them as those types; only the UnsafeRow kernels (urows.cuh, rows.cuh) read these.
  // `part`: a sparse vector's indices field (its size field follows); a part's owner; -1 otherwise.
  std::vector<uint8_t> vec;
  std::vector<int32_t> part;
  int32_t n_user = 0;
  bool vector(int32_t f) const { return f >= 0 && f < (int32_t)vec.size() && vec[f] == VK_DENSE; }
  bool sparse(int32_t f) const { return f >= 0 && f < (int32_t)vec.size() && vec[f] == VK_SPARSE; }
  bool has_vector() const { return std::find(vec.begin(), vec.end(), (uint8_t)VK_DENSE) != vec.end(); }
  // the caller's field of lowered field f: a sparse vector's part reports its vector
  int32_t owner(int32_t f) const { return f >= n_user && f < (int32_t)part.size() ? part[f] : f; }
  // Ragged fields (include/tfrgpu.h, RAGGED): a ragged x is its values part here (depth 1) and rag_len[x] is its lengths part,
  // one of the last n_rag fields (part[] maps it back to x).  The caller sees the first n_cols() fields as columns, x as the
  // depth-2 column ragged.cuh assembles; the lengths parts are internal.
  std::vector<int32_t> rag_len;
  int32_t n_rag = 0;
  bool ragged(int32_t f) const { return f >= 0 && f < (int32_t)rag_len.size() && rag_len[f] >= 0; }
  bool rag_splits = false;           // the parts rag_len[x] are row splits (TFR_S_RAGGED_ROW_SPLITS), not row lengths
  int32_t n_cols() const { return (int32_t)fields.size() - n_rag; }
  // the same fields without the ragged lowering (x at depth 2), which the UnsafeRow encoders take rows apart by
  std::shared_ptr<tfr_schema> plain;
  // INT64 TYPES (include/tfrgpu.h): the caller's TFR_T_BOOL .. TFR_T_TIMESTAMP of a field lowered to TFR_T_INT64, 0 otherwise.
  // Every parse and encode kernel sees the LongType field; narrow.cuh converts its leaf values at the edges.
  std::vector<int8_t> nar;
  int32_t nar_type(int32_t f) const { return f >= 0 && f < (int32_t)nar.size() ? nar[f] : 0; }
  // a column whose leaf values narrow.cuh converts (a timestamp's int64 values are its own)
  bool narrowed(int32_t f) const { const int32_t t = nar_type(f); return t != 0 && t != TFR_T_TIMESTAMP; }
  bool has_narrowed() const { for (int32_t f = 0; f < (int32_t)nar.size(); ++f) if (narrowed(f)) return true; return false; }
  // a field of a 1- or 2-byte type, whose UnsafeRow slots and array elements only urows_emit_kernel<*, true> writes
  bool has_narrow_row_field() const { for (int32_t f = 0; f < (int32_t)nar.size(); ++f) if (narrowed(f) && nar_width(nar[f]) < 4) return true; return false; }
};

static uint32_t fnv1a(const uint8_t* p, uint32_t n) { uint32_t h = 2166136261u; for (uint32_t i = 0; i < n; ++i) h = (h ^ p[i]) * 16777619u; return h; }

// A generated field of `f` (TFR_T_ROW_INDEX, TFR_T_RECORD_OFFSET) appended to `s` as a nullable int64 column; false when f is
// not one.  Anything but depth 0 and one field of each kind is TFR_E_UNSUPPORTED_TYPE in *rc.
static bool add_generated(tfr_schema& s, const tfr_field& f, const std::string& nm, int32_t* rc) {
  if (f.elem_type != TFR_T_ROW_INDEX && f.elem_type != TFR_T_RECORD_OFFSET) return false;
  const int kind = f.elem_type - TFR_T_ROW_INDEX;
  if (f.depth != 0) { *rc = fail(TFR_E_UNSUPPORTED_TYPE, "field '" + nm + "': a generated field is a scalar (depth 0)"); return true; }
  if (s.gen_field[kind] >= 0) { *rc = fail(TFR_E_UNSUPPORTED_TYPE, "field '" + nm + "': a schema has at most one generated field of each kind"); return true; }
  DevField d{};
  d.name_off = (uint32_t)s.names.size(); d.name_len = (uint32_t)f.name_len;
  s.names.insert(s.names.end(), (const uint8_t*)f.name, (const uint8_t*)f.name + f.name_len);
  d.hash = fnv1a((const uint8_t*)f.name, d.name_len);
  d.elem_type = TFR_T_INT64; d.depth = 0; d.nullable = 1; d.kind = (int8_t)required_kind(TFR_T_INT64); d.n_levels = 0; d.dup_next = -1;
  d.width = 8; d.var_slot = -1; d.cnt_slot = -1;
  d.fix_slot = s.n_fix++; s.fix_field.push_back((int32_t)s.fields.size());
  s.gen_field[kind] = (int32_t)s.fields.size();
  s.fields.push_back(d);
  *rc = TFR_OK;
  return true;
}

static void schema_rehash(tfr_schema& s, int32_t skip);

extern "C" int32_t tfr_schema_create(const tfr_field* fields, int32_t n_fields, int32_t record_type, tfr_schema** out) {
  return tfr_schema_create_ex(fields, n_fields, record_type, 0, out);
}
extern "C" int32_t tfr_schema_create_ex(const tfr_field* fields, int32_t n_fields, int32_t record_type, uint32_t schema_flags,
                                        tfr_schema** out) {
  if (!out || n_fields < 0 || (n_fields > 0 && !fields)) return fail(TFR_E_INVALID_ARG, "null argument");
  if (schema_flags & ~(TFR_S_RAGGED | TFR_S_INT64_TYPES | TFR_S_RAGGED_ROW_SPLITS)) return fail(TFR_E_INVALID_ARG, "unknown schema flags");
  if ((schema_flags & TFR_S_RAGGED_ROW_SPLITS) && !(schema_flags & TFR_S_RAGGED))
    return fail(TFR_E_INVALID_ARG, "raggedPartition=rowSplits needs nestedArrayFormat=ragged");
  if (record_type < TFR_RT_EXAMPLE || record_type > TFR_RT_BYTE_ARRAY)
    return fail(TFR_E_BAD_RECORD_TYPE, "Unsupported recordType: recordType can be ByteArray, Example or SequenceExample");
  if ((schema_flags & TFR_S_RAGGED) && record_type == TFR_RT_SEQUENCE_EXAMPLE)
    return fail(TFR_E_INVALID_ARG, "nestedArrayFormat=ragged is for Example records: SequenceExample stores nested arrays as FeatureLists");
  if (n_fields > 4096) return fail(TFR_E_INVALID_ARG, "more than 4096 fields");
  auto s = std::make_unique<tfr_schema>();
  s->record_type = record_type;
  if (record_type == TFR_RT_BYTE_ARRAY) {
    // the single binary column of TensorFlowInferSchema.getSchemaForByteArray (M/TensorFlowInferSchema.scala:60-64);
    // the caller's field list is ignored like deserializeByteArray ignores the schema (:17-19), but for generated fields
    DevField d{};
    d.name_off = 0; d.name_len = 9; s->names.assign((const uint8_t*)"byteArray", (const uint8_t*)"byteArray" + 9);
    d.hash = fnv1a(s->names.data(), 9);
    d.elem_type = TFR_T_BINARY; d.depth = 0; d.nullable = 1; d.kind = K_BYTES; d.n_levels = 1; d.dup_next = -1;
    d.fix_slot = -1; d.var_slot = 0; d.cnt_slot = 0; d.width = 1;
    s->fields.push_back(d);
    s->var_field.push_back(0);
    s->n_var = 1; s->n_cnt = 1;
    s->ht.assign(2, -1);
    s->ht[d.hash & 1] = 0;
    for (int32_t i = 0; i < n_fields; ++i) {
      const tfr_field& f = fields[i];
      if (f.elem_type != TFR_T_ROW_INDEX && f.elem_type != TFR_T_RECORD_OFFSET) continue;
      if (f.name_len < 0 || (f.name_len > 0 && !f.name)) return fail(TFR_E_INVALID_ARG, "bad field name");
      int32_t rc = TFR_OK;
      add_generated(*s, f, std::string(f.name ? f.name : "", (size_t)f.name_len), &rc);
      if (rc) return rc;
    }
    s->vec.assign(s->fields.size(), VK_NONE);
    s->part.assign(s->fields.size(), -1);
    s->rag_len.assign(s->fields.size(), -1);
    s->nar.assign(s->fields.size(), 0);
    s->n_user = (int32_t)s->fields.size();
    *out = s.release();
    return TFR_OK;
  }
  // one lowered field, appended
  auto add = [&](const std::string& key, int32_t et, int32_t depth, bool nullable, uint8_t vk, int32_t part) {
    DevField d{};
    const int32_t idx = (int32_t)s->fields.size();
    d.name_off = (uint32_t)s->names.size();
    d.name_len = (uint32_t)key.size();
    s->names.insert(s->names.end(), key.begin(), key.end());
    d.hash = fnv1a((const uint8_t*)key.data(), d.name_len);
    d.elem_type = (int8_t)et; d.depth = (int8_t)depth; d.nullable = nullable ? 1 : 0;
    d.kind = (int8_t)required_kind(et);
    bool varlen = et == TFR_T_STRING || et == TFR_T_BINARY;
    d.n_levels = (int16_t)(depth + (varlen ? 1 : 0));
    d.dup_next = -1;
    d.width = type_width(et);
    d.fix_slot = -1; d.var_slot = -1; d.cnt_slot = -1;
    if (et == TFR_T_NULL) { /* no storage beyond validity */ }
    else if (d.n_levels == 0) { d.fix_slot = s->n_fix++; s->fix_field.push_back(idx); }
    else { d.var_slot = s->n_var++; d.cnt_slot = s->n_cnt; s->n_cnt += d.n_levels; s->var_field.push_back(idx); }
    s->fields.push_back(d);
    s->vec.push_back(vk);
    s->part.push_back(part);
    s->rag_len.push_back(-1);
    s->nar.push_back(0);
  };
  std::vector<std::string> user(n_fields);              // the caller's names
  std::vector<int32_t> sparse, ragged;                  // the sparse vectors and the ragged fields, in field order
  for (int32_t i = 0; i < n_fields; ++i) {
    const tfr_field& f = fields[i];
    if (f.name_len < 0 || (f.name_len > 0 && !f.name)) return fail(TFR_E_INVALID_ARG, "bad field name");
    std::string nm(f.name ? f.name : "", (size_t)f.name_len);
    user[i] = nm;
    int32_t rc = TFR_OK;
    if (add_generated(*s, f, nm, &rc)) { if (rc) return rc; s->vec.push_back(VK_NONE); s->part.push_back(-1); s->rag_len.push_back(-1); s->nar.push_back(0); continue; }
    // a VectorUDT field is an ArrayType(DoubleType) field to every kernel but the UnsafeRow ones (VECTORS); a sparse one is
    // its values field here, and its indices and size fields are appended below (SPARSE VECTORS)
    const bool vector = f.elem_type == TFR_T_VECTOR, sp = f.elem_type == TFR_T_SPARSE_VECTOR;
    if ((vector || sp) && f.depth != 0) return fail(TFR_E_UNSUPPORTED_TYPE, "field '" + nm + "': ArrayType(VectorUDT) is not supported");
    // a BooleanType .. TimestampType field is a LongType field to every kernel but narrow.cuh's (INT64 TYPES)
    const bool i64t = nar_width(f.elem_type) > 0;
    if (i64t && !(schema_flags & TFR_S_INT64_TYPES))
      return fail(TFR_E_UNSUPPORTED_TYPE, "field '" + nm + "': data type is not supported (Boolean, Byte, Short, Date and Timestamp need extendedTypes=true)");
    const int32_t et = vector || sp ? TFR_T_FLOAT64 : i64t ? TFR_T_INT64 : f.elem_type, depth = vector || sp ? 1 : f.depth;
    // newFeatureWriter / newFeatureConverter: anything but these types throws (M/TFRecordDeserializer.scala:119-123,
    // M/TFRecordSerializer.scala:147,151); ArrayType(NullType) falls into the same default branch
    bool ok_type = et >= TFR_T_NULL && et <= TFR_T_BINARY && depth >= 0 && depth <= 2 && !(et == TFR_T_NULL && depth > 0);
    if (!ok_type) return fail(TFR_E_UNSUPPORTED_TYPE, "field '" + nm + "': data type is not supported");
    if (sp) sparse.push_back(i);
    // a ragged field is its values part here (depth 1), and its lengths part is appended below (RAGGED)
    const bool rg = (schema_flags & TFR_S_RAGGED) && record_type == TFR_RT_EXAMPLE && depth == 2;
    if (rg) ragged.push_back(i);
    add(sp ? nm + TFR_SPARSE_VALUES_SUFFIX : rg ? nm + TFR_RAGGED_VALUES_SUFFIX : nm, et, rg ? 1 : depth, f.nullable != 0,
        vector ? VK_DENSE : sp ? VK_SPARSE : VK_NONE, -1);
    if (i64t) s->nar.back() = (int8_t)f.elem_type;
  }
  s->n_user = n_fields;
  for (int32_t v : sparse) {
    s->part[v] = (int32_t)s->fields.size();
    add(user[v] + TFR_SPARSE_INDICES_SUFFIX, TFR_T_INT32, 1, true, VK_INDICES, v);
    add(user[v] + TFR_SPARSE_SIZE_SUFFIX, TFR_T_INT32, 0, true, VK_SIZE, v);
  }
  s->rag_splits = (schema_flags & TFR_S_RAGGED_ROW_SPLITS) != 0;
  for (int32_t x : ragged) {
    s->rag_len[x] = (int32_t)s->fields.size();
    add(user[x] + (s->rag_splits ? TFR_RAGGED_ROW_SPLITS_SUFFIX : TFR_RAGGED_ROW_LENGTHS_SUFFIX), TFR_T_INT64, 1, true, VK_NONE, x);
  }
  s->n_rag = (int32_t)ragged.size();
  if (s->n_rag) {
    tfr_schema* p = nullptr;
    TRY(tfr_schema_create_ex(fields, n_fields, record_type, schema_flags & TFR_S_INT64_TYPES, &p));
    s->plain.reset(p);
  }
  // Spark refuses duplicate column names for file sources before the reader is built
  // (SchemaUtils.checkColumnNameDuplication), so they never reach TFRecordDeserializer
  if (std::unordered_set<std::string>(user.begin(), user.end()).size() != user.size())
    return fail(TFR_E_INVALID_ARG, "Found duplicate column(s) in the data schema");
  // and two fields may not share a feature key, which only a sparse vector's or a ragged field's keys can do past the check above
  const int32_t nl = (int32_t)s->fields.size();
  auto key = [&](int32_t f) { const DevField& d = s->fields[f]; return std::string((const char*)&s->names[d.name_off], d.name_len); };
  size_t hsz = 2; while (hsz < 2 * (size_t)nl + 2) hsz <<= 1;
  s->ht.assign(hsz, -1);
  for (int32_t i = 0; i < nl; ++i) {
    const DevField& d = s->fields[i];
    size_t slot = d.hash & (hsz - 1);
    while (s->ht[slot] >= 0) {
      const int32_t j = s->ht[slot];
      const DevField& o = s->fields[j];
      if (o.hash == d.hash && o.name_len == d.name_len && memcmp(&s->names[o.name_off], &s->names[d.name_off], d.name_len) == 0)
        return fail(TFR_E_INVALID_ARG, "fields '" + user[s->owner(j)] + "' and '" + user[s->owner(i)] + "' have the same feature key '" + key(i) + "'");
      slot = (slot + 1) & (hsz - 1);
    }
    s->ht[slot] = i;
  }
  if (s->has_generated()) schema_rehash(*s, -1);         // (after the duplicate-name check, which covers them too)
  *out = s.release();
  return TFR_OK;
}
// the key hash table without field `skip` and the generated fields: no feature of the record maps to them, so every kernel
// writes them as absent fields (a PERMISSIVE decoder's corrupt-record column; position_kernel then fills the generated ones)
static void schema_rehash(tfr_schema& s, int32_t skip) {
  std::fill(s.ht.begin(), s.ht.end(), -1);
  const size_t mask = s.ht.size() - 1;
  for (int32_t i = 0; i < (int32_t)s.fields.size(); ++i) {
    if (i == skip || s.generated(i)) continue;
    size_t slot = s.fields[i].hash & mask;
    while (s.ht[slot] >= 0) slot = (slot + 1) & mask;
    s.ht[slot] = i;
  }
}
extern "C" void tfr_schema_destroy(tfr_schema* s) { delete s; }
extern "C" int32_t tfr_schema_num_fields(const tfr_schema* s) { return s ? s->n_cols() : 0; }

// device copy of a schema.  The copies run on the handle's stream `st` and are waited for before returning: the handle's
// kernels run on non-blocking streams, which nothing orders after the legacy default stream, and `tp` is a local.
struct DevSchemaBuf {
  DevBuf fields, names, ht, var_field, templates;
  DevBuf vec, part;                                       // tfr_schema::vec and ::part, for the UnsafeRow kernels of the encoder
  DevBuf nar;                                             // tfr_schema::nar, for the same kernels (INT64 TYPES)
  DevBuf rag; int32_t n_rag = 0;                          // pairs (ragged field, its lengths part), for decode_pass1_kernel<true>
  DevBuf tile_consts; uint32_t tile_consts_bytes = 0;     // tile.cuh: per-schema constants in the shared-memory layout
  DevSchema view{};
  const int32_t* d_var_field() const { return (const int32_t*)var_field.p; }
  const uint8_t* d_vec() const { return (const uint8_t*)vec.p; }
  const int32_t* d_part() const { return (const int32_t*)part.p; }
  const int8_t* d_nar() const { return (const int8_t*)nar.p; }
  const uint8_t* d_tile_consts() const { return (const uint8_t*)tile_consts.p; }
  // `unkeyed`: a field no feature maps to (schema_rehash), which gets no entry template either
  int32_t upload(const tfr_schema& s, cudaStream_t st, int32_t unkeyed = -1) {
    size_t nf = s.fields.size();
    CUDA_TRY(fields.alloc(std::max<size_t>(1, nf) * sizeof(DevField)));
    CUDA_TRY(names.alloc(std::max<size_t>(1, s.names.size())));
    CUDA_TRY(ht.alloc(s.ht.size() * sizeof(int32_t)));
    CUDA_TRY(var_field.alloc(std::max<size_t>(1, s.var_field.size()) * sizeof(int32_t)));
    CUDA_TRY(vec.alloc(std::max<size_t>(1, nf)));
    CUDA_TRY(part.alloc(std::max<size_t>(1, nf) * sizeof(int32_t)));
    CUDA_TRY(nar.alloc(std::max<size_t>(1, nf)));
    if (!s.nar.empty()) CUDA_TRY(cudaMemcpyAsync(nar.p, s.nar.data(), s.nar.size(), cudaMemcpyHostToDevice, st));
    if (nf) CUDA_TRY(cudaMemcpyAsync(fields.p, s.fields.data(), nf * sizeof(DevField), cudaMemcpyHostToDevice, st));
    if (!s.vec.empty()) CUDA_TRY(cudaMemcpyAsync(vec.p, s.vec.data(), s.vec.size(), cudaMemcpyHostToDevice, st));
    if (!s.part.empty()) CUDA_TRY(cudaMemcpyAsync(part.p, s.part.data(), s.part.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (!s.names.empty()) CUDA_TRY(cudaMemcpyAsync(names.p, s.names.data(), s.names.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ht.p, s.ht.data(), s.ht.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (!s.var_field.empty()) CUDA_TRY(cudaMemcpyAsync(var_field.p, s.var_field.data(), s.var_field.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    std::vector<int32_t> pairs;
    for (int32_t f = 0; f < s.n_cols(); ++f) if (s.ragged(f)) { pairs.push_back(f); pairs.push_back(s.rag_len[f]); }
    n_rag = (int32_t)pairs.size() / 2;
    CUDA_TRY(rag.alloc(std::max<size_t>(2, pairs.size()) * sizeof(int32_t)));
    if (!pairs.empty()) CUDA_TRY(cudaMemcpyAsync(rag.p, pairs.data(), pairs.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    {
      // canonical entry prefix of every field: 0A ? 0A klen key 12 ? kindtag ?   (? = length bytes, masked out)
      std::vector<FieldTemplate> tp(std::max<size_t>(1, nf));
      for (size_t f = 0; f < nf; ++f) {
        FieldTemplate& t = tp[f];
        memset(&t, 0, sizeof t);
        const DevField& fd = s.fields[f];
        t.kind = (uint32_t)fd.kind;
        const uint32_t klen = fd.name_len, total = klen + 8;
        if (fd.kind == K_NONE || klen >= 0x80 || total > TILE_TPL_WORDS * 4 || (int32_t)f == unkeyed || s.generated((int32_t)f)) continue;      // no template: generic parse
        uint8_t bytes[TILE_TPL_WORDS * 4] = {0}, mask[TILE_TPL_WORDS * 4] = {0};
        auto put = [&](uint32_t i, uint8_t b, bool fixed) { bytes[i] = b; mask[i] = fixed ? 0xFF : 0x00; };
        put(0, 0x0A, true); put(1, 0, false); put(2, 0x0A, true); put(3, (uint8_t)klen, true);
        for (uint32_t i = 0; i < klen; ++i) put(4 + i, s.names[fd.name_off + i], true);
        put(4 + klen, 0x12, true); put(5 + klen, 0, false);
        put(6 + klen, fd.kind == K_BYTES ? 0x0A : fd.kind == K_FLOAT ? 0x12 : 0x1A, true); put(7 + klen, 0, false);
        t.n_words = (uint16_t)((total + 3) / 4); t.klen = (uint16_t)klen;
        memcpy(t.words, bytes, sizeof bytes); memcpy(t.mask, mask, sizeof mask);
      }
      CUDA_TRY(templates.alloc(tp.size() * sizeof(FieldTemplate)));
      CUDA_TRY(cudaMemcpyAsync(templates.p, tp.data(), tp.size() * sizeof(FieldTemplate), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaStreamSynchronize(st));
    }
    view.n_fields = (int32_t)nf; view.record_type = s.record_type; view.ht_mask = (int32_t)s.ht.size() - 1;
    view.n_fix = s.n_fix; view.n_var = s.n_var; view.n_cnt = s.n_cnt;
    view.fields = (DevField*)fields.p; view.names = (uint8_t*)names.p; view.ht = (int32_t*)ht.p;
    return TFR_OK;
  }
  // CRC tables | zeroed seen words | DevField[nf] | FieldTemplate[nf] | names, each section 16-byte aligned (tile_const_bytes)
  int32_t build_tile_consts(const tfr_schema& s, const CrcTables* d_tabs, cudaStream_t st) {
    const uint32_t nf = (uint32_t)s.fields.size(), nb = (uint32_t)s.names.size();
    tile_consts_bytes = tile_const_bytes(nf, nb);
    CUDA_TRY(tile_consts.alloc(tile_consts_bytes));
    CUDA_TRY(cudaMemsetAsync(tile_consts.p, 0, tile_consts_bytes, st));
    uint8_t* q = (uint8_t*)tile_consts.p;
    CUDA_TRY(cudaMemcpyAsync(q, d_tabs->g5, TILE_CRC_BYTES, cudaMemcpyDeviceToDevice, st));   // g5 then xp16, contiguous in CrcTables
    q += TILE_CRC_BYTES + TILE_SEEN_BYTES;
    if (nf) CUDA_TRY(cudaMemcpyAsync(q, fields.p, nf * sizeof(DevField), cudaMemcpyDeviceToDevice, st));
    q += (nf * sizeof(DevField) + 15) & ~(size_t)15;
    if (nf) CUDA_TRY(cudaMemcpyAsync(q, templates.p, nf * sizeof(FieldTemplate), cudaMemcpyDeviceToDevice, st));
    q += (nf * sizeof(FieldTemplate) + 15) & ~(size_t)15;
    if (nb) CUDA_TRY(cudaMemcpyAsync(q, names.p, nb, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));             // the decoder's kernels read these from its other streams too
    return TFR_OK;
  }
};

// Raises Kernel's opt-in dynamic shared memory to at least `smem` bytes on the current device; never lowers it.
// cudaFuncSetAttribute sets the limit, it does not take a maximum, and every thread of the process launches the same kernels:
// the check and the set happen under one lock, so that a thread asking for less cannot overwrite a larger grant another thread
// has just made (which would leave `granted` above the attribute and fail every later launch between the two sizes).
// `granted` only changes after the attribute does, so a value read without the lock that is already large enough is safe.
static std::mutex g_dyn_smem_mu;
template <auto Kernel>
static cudaError_t raise_dyn_smem(size_t smem) {
  static std::atomic<size_t> granted[64];               // per device; zero-initialised (static storage)
  int dev = 0; cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || granted[dev].load(std::memory_order_acquire) >= smem) return cudaSuccess;
  std::lock_guard<std::mutex> lk(g_dyn_smem_mu);
  if (granted[dev].load(std::memory_order_relaxed) >= smem) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) granted[dev].store(smem, std::memory_order_release);
  return e;
}

#include "api_frames.inc"
#include "api_index.inc"
#include "api_infer.inc"
#include "api_outputs.inc"
#include "api_decode.inc"
#include "api_rows.inc"

// ---------------------------------------------------------------------------------------------
// Arrow C Data Interface export (arrow/c/abi.h structs restated in host_util.h)
// ---------------------------------------------------------------------------------------------
struct ExportPriv { tfr_batch* batch; std::vector<const void*> buffers; std::vector<ArrowArray*> children; ArrowArray* child_storage = nullptr; };

static void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* p = (ExportPriv*)a->private_data;
  for (int64_t i = 0; i < a->n_children; ++i) {
    if (a->children[i]->release) a->children[i]->release(a->children[i]);
    delete a->children[i];
  }
  if (p) { if (p->batch) tfr_batch_release(p->batch); delete p; }
  a->release = nullptr;
}
static void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  for (int64_t i = 0; i < s->n_children; ++i) {
    if (s->children[i]->release) s->children[i]->release(s->children[i]);
    delete s->children[i];
  }
  delete[] s->children;
  free((void*)s->name);
  s->release = nullptr;
}
static const char* leaf_format(int t) {
  switch (t) {
    case TFR_T_INT32: return "i"; case TFR_T_INT64: return "l"; case TFR_T_FLOAT32: return "f";
    case TFR_T_FLOAT64: case TFR_T_DECIMAL: return "g"; case TFR_T_STRING: return "u"; case TFR_T_BINARY: return "z";
    case TFR_T_BOOL: return "b"; case TFR_T_INT8: return "c"; case TFR_T_INT16: return "s"; case TFR_T_DATE: return "tdD";
    case TFR_T_TIMESTAMP: return "tsu:UTC";
    default: return "n";
  }
}
static void build_schema(ArrowSchema* s, const char* name, int elem_type, int depth) {
  memset(s, 0, sizeof *s);
  s->name = strdup(name); s->flags = 2 /*ARROW_FLAG_NULLABLE*/; s->release = release_schema;
  if (depth == 0) { s->format = leaf_format(elem_type); return; }
  s->format = "+l";
  s->n_children = 1; s->children = new ArrowSchema*[1];
  s->children[0] = new ArrowSchema;
  build_schema(s->children[0], "item", elem_type, depth - 1);
}
// level: which offsets level this list node uses; leaves use the last level for utf8/binary.  bits: a boolean column's bit-packed
// values (INT64 TYPES), which its leaf hands out in place of the bytes of c.values
static void build_array(ArrowArray* a, const tfr_column& c, int level, int64_t length, tfr_batch* owner, const void* bits = nullptr) {
  memset(a, 0, sizeof *a);
  auto* p = new ExportPriv;
  p->batch = owner;
  if (owner) owner->refs.fetch_add(1);
  a->private_data = p; a->release = release_array; a->length = length; a->offset = 0;
  const bool varlen = c.elem_type == TFR_T_STRING || c.elem_type == TFR_T_BINARY;
  const void* validity = level == 0 ? c.validity : nullptr;
  a->null_count = level == 0 ? c.null_count : 0;
  if (level < c.depth) {                 // list node
    p->buffers = {validity, c.offsets[level]};
    a->n_buffers = 2;
    a->n_children = 1;
    p->children.resize(1); p->children[0] = new ArrowArray;
    a->children = p->children.data();
    int64_t child_len = level + 1 < c.n_levels ? c.n_offsets[level + 1] - 1 : c.n_values;
    build_array(a->children[0], c, level + 1, child_len, nullptr, bits);
  } else if (c.elem_type == TFR_T_NULL) {
    a->n_buffers = 0; a->null_count = length;
  } else if (varlen) {
    p->buffers = {validity, c.offsets[c.n_levels - 1], c.values};
    a->n_buffers = 3;
  } else {
    p->buffers = {validity, c.elem_type == TFR_T_BOOL ? bits : c.values};
    a->n_buffers = 2;
  }
  a->buffers = p->buffers.data();
}

extern "C" int32_t tfr_batch_export_arrow_host(tfr_batch* b, int32_t column, void* arrow_array, void* arrow_schema) {
  if (!b || !arrow_array || !arrow_schema || column < 0 || column >= (int32_t)b->out.cols.size()) return fail(TFR_E_INVALID_ARG, "bad argument");
  int32_t rc = tfr_batch_to_host(b, nullptr, (int32_t)b->out.cols.size());
  if (rc) return rc;
  const tfr_column& c = b->host_copy.cols[column];
  const tfr_schema& S = b->dec->schema;
  std::string nm((const char*)&S.names[S.fields[column].name_off], S.fields[column].name_len);
  if (S.ragged(column)) nm.resize(nm.size() - strlen(TFR_RAGGED_VALUES_SUFFIX));     // x, not its values part's key
  build_schema((ArrowSchema*)arrow_schema, nm.c_str(), c.elem_type, c.depth);
  const void* bits = c.elem_type == TFR_T_BOOL ? b->out.host_ptr((uint8_t*)b->host_copy.block.get(), b->out.bool_bits((uint32_t)column)) : nullptr;
  build_array((ArrowArray*)arrow_array, c, 0, c.n_rows, b, bits);
  return TFR_OK;
}
extern "C" int32_t tfr_batch_export_arrow_device(tfr_batch* b, int32_t column, void* arrow_device_array, void* arrow_schema) {
  if (!b || !arrow_device_array || !arrow_schema || column < 0 || column >= (int32_t)b->out.cols.size()) return fail(TFR_E_INVALID_ARG, "bad argument");
  int32_t rc = tfr_batch_wait(b);
  if (rc) return rc;
  const tfr_column& c = b->out.cols[column];
  const tfr_schema& S = b->dec->schema;
  std::string nm((const char*)&S.names[S.fields[column].name_off], S.fields[column].name_len);
  if (S.ragged(column)) nm.resize(nm.size() - strlen(TFR_RAGGED_VALUES_SUFFIX));     // x, not its values part's key
  build_schema((ArrowSchema*)arrow_schema, nm.c_str(), c.elem_type, c.depth);
  auto* da = (ArrowDeviceArray*)arrow_device_array;
  memset(da, 0, sizeof *da);
  build_array(&da->array, c, 0, c.n_rows, b, c.elem_type == TFR_T_BOOL ? b->out.bool_bits((uint32_t)column) : nullptr);
  da->device_id = b->dec->device; da->device_type = 2 /*ARROW_DEVICE_CUDA*/; da->sync_event = nullptr;   // batch already waited
  return TFR_OK;
}

#include "api_encode.inc"
