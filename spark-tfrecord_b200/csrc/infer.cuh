// infer.cuh -- K6: schema inference (SURVEY.md 8f.1).
//
// Replaces TensorFlowInferSchema.apply (M/TensorFlowInferSchema.scala:35-58): rdd.aggregate(empty)(
// inferExampleRowType / inferSequenceExampleRowType, mergeFieldTypes).  Per record every feature of the parsed
// map gets a lattice code (inferField :132-145 + parse*List :147-188: empty list -> null(0), one element ->
// Long/Float/String (1..3), more -> array of it (4..6); FeatureLists: max over the steps, then wrapped into
// ArrayType(ArrayType(T)) (7..9) :98-118); codes of one name merge with findTightestCommonType = max with
// null as identity (:213-228).  Here: warp per record, one map entry per lane (the full-semantics parser of
// decode.cuh), duplicate keys inside a record resolved last-wins before anything is merged, then one
// atomicMax per (name, record) into a device hash table.  A 64-bit hash of the name picks the slot and filters,
// names are equal only when their bytes are.
// A record's verdict is the reference's: a CRC or parse failure anywhere in the record (parseFrom throws before
// inference sees a value), else the first value error of the surviving entries in map order (the position of a key's
// first occurrence), context before feature_lists.
// infer_kernel<false> is FAILFAST: a failing record fails the call, so each map's clean survivors are merged as soon as the
// map is de-duplicated.  infer_kernel<true> serves DROPMALFORMED and PERMISSIVE, which skip a failing record: the merge is
// record-atomic -- every map of the record stays in shared memory (a SequenceExample has a second window per warp for its
// feature_lists) until the verdict is known, and only a clean record's survivors reach the table.  In PERMISSIVE an entry
// named like the corrupt-record column (A.corrupt) is parsed but neither merged nor a value error.
#pragma once
#include "common.cuh"
#include "decode.cuh"

struct InferSlot {
  unsigned long long hash;   // 0 = empty, INFER_CLAIMED = name being written
  uint32_t name_off;         // offset of the key bytes inside the batch that first inserted the name
  uint32_t name_len;
  uint32_t code;             // max lattice code seen (0..9)
  uint32_t flags;            // bit0: ArrayType(ArrayType(null)) seen (a FeatureList whose steps are all empty)
};
#define INFER_TABLE_SLOTS 65536u
#define INFER_MAX_ENT 1024     // entries of one map buffered per record for last-wins de-duplication; more raise INF_OVF_ENTRIES
static_assert(INFER_MAX_ENT <= 32 * 32, "infer_kernel<true> keeps one bit per entry of a lane in a 32-bit mask");
#define INFER_CLAIMED (~0ull)  // a slot whose name is being written: its hash is published after the name
enum { INF_OVF_TABLE = 1u, INF_OVF_ENTRIES = 2u, INF_OVF_KEY = 4u };   // limits hit: reported as an explicit error, never as a silently wrong schema
// per-entry record in shared memory: ecode = lattice code (bits 0-3) | value error (bits 4-7, INF_ERR_*) | key length << 8.
// infer_kernel<true> only: INF_ERR_IGNORED marks an entry of the corrupt-record column's name.
enum { INF_ERR_KIND = 1u, INF_ERR_EMPTY = 2u, INF_ERR_IGNORED = 4u };

struct InferArgs {
  const uint8_t* data;
  const uint32_t* rec_off;
  uint32_t n;
  uint32_t verify;
  uint32_t record_type;
  const CrcTables* tabs;
  InferSlot* table;
  uint32_t* first_err;       // [0] min failing record index, [1] INF_OVF_* flags, [4] min record index over a per-record limit
  uint32_t* status;          // [n]
  // PERMISSIVE (infer_kernel<true>): the corrupt-record column's name, its hash64; corrupt_len = 0 otherwise
  const uint8_t* corrupt;
  unsigned long long corrupt_hash;
  uint32_t corrupt_len;
};

__host__ __device__ __forceinline__ unsigned long long hash64(const uint8_t* p, uint32_t n) {
  unsigned long long h = 1469598103934665603ull;
  for (uint32_t i = 0; i < n; ++i) h = (h ^ p[i]) * 1099511628211ull;
  return (h == 0ull || h == INFER_CLAIMED) ? 1ull : h;          // 0 and INFER_CLAIMED mark slots
}
__device__ __forceinline__ bool bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t n) {
  if (a == b) return true;
  for (uint32_t i = 0; i < n; ++i) if (a[i] != b[i]) return false;
  return true;
}
__device__ __forceinline__ int feat_code(const FeatAcc& a) {       // inferField + parse*List
  if (a.kind == K_NONE) return -1;                                  // RuntimeException("unsupported type ...")
  if (a.n == 0) return 0;
  int base = a.kind == K_INT64 ? 1 : a.kind == K_FLOAT ? 2 : 3;
  return a.n > 1 ? base + 3 : base;
}
// Names are substrings of the block being inferred (A.data): the table is cleared before and gathered after every block.
__device__ __forceinline__ void infer_merge(InferSlot* table, const uint8_t* data, unsigned long long h, uint32_t name_off, uint32_t name_len,
                                            int code, uint32_t* ovf) {
  uint32_t slot = (uint32_t)(h ^ (h >> 32)) & (INFER_TABLE_SLOTS - 1);
  for (uint32_t probe = 0; probe < INFER_TABLE_SLOTS; ++probe) {
    InferSlot* s = &table[slot];
    unsigned long long cur = atomicCAS(&s->hash, 0ull, INFER_CLAIMED);
    bool same = false;
    if (cur == 0ull) {
      // claimed: write the name, then publish the hash; a reader that sees the hash sees the name
      s->name_off = name_off; s->name_len = name_len;
      __threadfence();
      atomicExch(&s->hash, h);
      same = true;
    } else {
      // another thread (maybe a lane of this warp) is writing this slot's name: independent thread scheduling lets it finish
      while (cur == INFER_CLAIMED) { __nanosleep(20); cur = *(volatile unsigned long long*)&s->hash; }
      if (cur == h) {
        __threadfence();
        const uint32_t off = *(volatile uint32_t*)&s->name_off, len = *(volatile uint32_t*)&s->name_len;
        same = len == name_len && bytes_equal(data + off, data + name_off, len);
      }
    }
    if (same) {
      if (code == 10) atomicOr(&s->flags, 1u);
      else atomicMax(&s->code, (uint32_t)code);
      return;
    }
    slot = (slot + 1) & (INFER_TABLE_SLOTS - 1);            // empty-to-us, another hash, or the same hash and other bytes
  }
  atomicOr(ovf, INF_OVF_TABLE);            // more distinct names than slots
}

// one map (Features or FeatureLists) of one record: entries -> (hash, code | value error, key) in shared memory.  Returns
// false when the map does not parse; `over` is set when the map passes a per-record limit (entries, key length).
template <bool TOL>
__device__ __forceinline__ bool infer_map(const InferArgs& A, Cur body, bool is_flist, unsigned long long* eh, uint32_t* ecode, uint32_t* ekey,
                                          uint32_t& nent, bool& over) {
  const uint32_t lane = threadIdx.x & 31;
  // (1) uniform hop collecting entry ranges; 32 at a time parsed one per lane
  uint32_t pend = 0, my_len = 0;
  const uint8_t* my_ptr = nullptr;
  auto flush = [&]() -> bool {
    int code = 0; uint32_t verr = 0; unsigned long long h = 0; uint32_t koff = 0, klen = 0; bool ok = true;
    if (lane < pend) {
      // entry: last key wins, values merge (same walk as decode.cuh parse_entry, without a schema)
      const uint8_t* key = nullptr;
      Cur c{my_ptr, my_ptr + my_len};
      FeatAcc acc; acc_reset(acc, K_NONE);
      int fl_code = -2;          // -2: no step seen yet
      bool step_unset = false;   // a step whose kind is not set (the steps are typed in order: the first one throws)
      for (;;) {
        uint32_t tag;
        if (!rd_tag(c, tag)) { ok = false; break; }
        if (tag == 0) break;
        if (tag == 0x0A) {
          uint32_t l; if (!rd_len(c, l) || !utf8_valid(c.p, l)) { ok = false; break; }
          key = c.p; klen = l; c.p += l;
        } else if (tag == 0x12) {
          uint32_t l; if (!rd_len(c, l)) { ok = false; break; }
          Cur v{c.p, c.p + l}; c.p += l;
          if (!is_flist) { if (!feature_scan(v, acc, false, A.data)) { ok = false; break; } }
          else {
            for (;;) {
              uint32_t t2;
              if (!rd_tag(v, t2)) { ok = false; break; }
              if (t2 == 0) break;
              if (t2 != 0x0A) { if (!skip_field(v, t2)) { ok = false; break; } continue; }
              uint32_t sl; if (!rd_len(v, sl)) { ok = false; break; }
              FeatAcc st; acc_reset(st, K_NONE);
              if (!feature_scan(Cur{v.p, v.p + sl}, st, false, A.data)) { ok = false; break; }
              v.p += sl;
              int sc = feat_code(st);
              if (sc < 0) step_unset = true;
              if (fl_code == -2) fl_code = sc; else if (sc > fl_code) fl_code = sc;      // reduceLeft(findTightestCommonType)
            }
            if (!ok) break;
          }
        } else if (!skip_field(c, tag)) { ok = false; break; }
      }
      if (ok) {
        h = hash64(key, klen);
        koff = key ? (uint32_t)(key - A.data) : 0;
        if (!is_flist) { code = feat_code(acc); if (code < 0) { verr = INF_ERR_KIND; code = 0; } }
        else if (fl_code == -2) verr = INF_ERR_EMPTY;                                   // empty.reduceLeft
        else if (step_unset) verr = INF_ERR_KIND;
        else if (fl_code == 0) code = 10;                                               // ArrayType(ArrayType(null))
        else code = 7 + (fl_code - 1) % 3;                                              // T or [T] -> [[T]]
        if constexpr (TOL) {
          if (klen == A.corrupt_len && h == A.corrupt_hash && bytes_equal(key, A.corrupt, klen)) { code = 0; verr = INF_ERR_IGNORED; }
        }
      }
    }
    if (__any_sync(FULLMASK, !ok)) return false;
    if (lane < pend && klen >= (1u << 24)) { atomicOr(&A.first_err[1], INF_OVF_KEY); over = true; }
    if (lane < pend && nent + lane < INFER_MAX_ENT) {
      eh[nent + lane] = h; ecode[nent + lane] = (uint32_t)code | (verr << 4) | (klen << 8); ekey[nent + lane] = koff;
    } else if (lane < pend) {
      // beyond the de-duplication window: last-wins cannot be decided any more
      atomicOr(&A.first_err[1], INF_OVF_ENTRIES); over = true;
    }
    nent = min(nent + pend, (uint32_t)INFER_MAX_ENT);
    pend = 0;
    __syncwarp();
    return true;
  };
  for (;;) {
    uint32_t tag;
    if (!rd_tag(body, tag)) return false;
    if (tag == 0) break;
    if (tag != 0x0A) { if (!skip_field(body, tag)) return false; continue; }
    uint32_t l;
    if (!rd_len(body, l)) return false;
    if (lane == pend) { my_ptr = body.p; my_len = l; }
    body.p += l;
    if (++pend == 32 && !flush()) return false;
  }
  if (pend && !flush()) return false;
  return true;
}

// entries i and j of one map have the same key (the hash filters, the bytes decide)
__device__ __forceinline__ bool same_key(const uint8_t* data, const unsigned long long* eh, const uint32_t* ecode, const uint32_t* ekey,
                                         uint32_t i, uint32_t j) {
  return eh[i] == eh[j] && (ecode[i] >> 8) == (ecode[j] >> 8) && bytes_equal(data + ekey[i], data + ekey[j], ecode[i] >> 8);
}

// shared memory of one launch: the CRC tables, then per warp one window of INFER_MAX_ENT entries per map kept at once
__host__ __device__ constexpr uint32_t infer_windows(bool tol, uint32_t record_type) { return tol && record_type == TFR_RT_SEQUENCE_EXAMPLE ? 2u : 1u; }
#define INFER_WINDOW_BYTES (INFER_MAX_ENT * 16)

template <bool TOL>
__global__ void __launch_bounds__(128) infer_kernel(InferArgs A) {
  extern __shared__ uint32_t smem[];
  uint32_t* stab = smem;
  crc_stage_tables(stab, A.tabs);
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nwin = infer_windows(TOL, A.record_type);
  uint8_t* wbase = reinterpret_cast<uint8_t*>(smem + CRC_SMEM_WORDS) + (size_t)wid * nwin * INFER_WINDOW_BYTES;
  unsigned long long* eh = reinterpret_cast<unsigned long long*>(wbase);
  uint32_t* ecode = reinterpret_cast<uint32_t*>(wbase + INFER_MAX_ENT * 8);
  uint32_t* ekey = reinterpret_cast<uint32_t*>(wbase + INFER_MAX_ENT * 12);
  __syncthreads();
  for (uint32_t row = blockIdx.x * warps + wid; row < A.n; row += gridDim.x * warps) {
    const uint32_t off = A.rec_off[row];
    const uint32_t len = A.rec_off[row + 1] - off - 16;
    const uint8_t* payload = A.data + off + 12;
    int err = 0;
    if (A.verify && crc_mask(crc_warp(stab, payload, len)) != load_u32_unaligned(payload + len)) err = TFR_E_CRC_DATA;
    bool ok = true, over = false;
    uint32_t verr = 0;         // the record's first value error (INF_ERR_*): context's before feature_lists'
    // infer_kernel<true>: per map, bit k set when entry lane + 32 k is a clean survivor (registers, not shared memory)
    uint32_t keep0 = 0u, keep1 = 0u;
    // pass 0: features/context (field 1), pass 1: feature_lists (field 2).  Both are parsed before a value error counts.
    for (int pass = 0; pass < 2 && ok && !err; ++pass) {
      if (pass == 1 && A.record_type != TFR_RT_SEQUENCE_EXAMPLE) break;
      if constexpr (TOL) {       // each map in its own window: nothing is merged before the record's verdict
        eh = reinterpret_cast<unsigned long long*>(wbase + pass * INFER_WINDOW_BYTES);
        ecode = reinterpret_cast<uint32_t*>(wbase + pass * INFER_WINDOW_BYTES + INFER_MAX_ENT * 8);
        ekey = reinterpret_cast<uint32_t*>(wbase + pass * INFER_WINDOW_BYTES + INFER_MAX_ENT * 12);
      }
      uint32_t nent = 0;
      Cur top{payload, payload + len};
      for (;;) {
        uint32_t tag;
        if (!rd_tag(top, tag)) { ok = false; break; }
        if (tag == 0) break;
        if (tag == 0x0A || (tag == 0x12 && A.record_type == TFR_RT_SEQUENCE_EXAMPLE)) {
          uint32_t l;
          if (!rd_len(top, l)) { ok = false; break; }
          if ((tag == 0x0A) == (pass == 0) && !infer_map<TOL>(A, Cur{top.p, top.p + l}, pass == 1, eh, ecode, ekey, nent, over)) { ok = false; break; }
          top.p += l;
        } else if (!skip_field(top, tag)) { ok = false; break; }
      }
      if (!ok) break;
      __syncwarp();
      // Map.put semantics: an entry counts only if no later entry of this map has the same key; it sits at the position
      // of the key's first occurrence, which orders the value errors
      uint32_t first_err = 0xffffffffu;     // (first-occurrence position << 8) | INF_ERR_*
      for (uint32_t i = lane; i < nent; i += 32) {
        if constexpr (TOL) {
          if ((ecode[i] >> 4) & INF_ERR_IGNORED) continue;      // (so is every entry of its key)
        }
        bool last = true;
        for (uint32_t j = i + 1; j < nent; ++j) if (same_key(A.data, eh, ecode, ekey, i, j)) { last = false; break; }
        if (!last) continue;
        const uint32_t e = (ecode[i] >> 4) & 0xf;
        if (e) {
          uint32_t pos = i;
          for (uint32_t j = 0; j < i; ++j) if (same_key(A.data, eh, ecode, ekey, i, j)) { pos = j; break; }
          first_err = min(first_err, (pos << 8) | e);
        } else if constexpr (TOL) {
          (pass ? keep1 : keep0) |= 1u << (i >> 5);              // merged below if the record is kept
        } else {
          infer_merge(A.table, A.data, eh[i], ekey[i], ecode[i] >> 8, (int)(ecode[i] & 0xf), &A.first_err[1]);
        }
      }
      first_err = __reduce_min_sync(FULLMASK, first_err);
      if (!verr && first_err != 0xffffffffu) verr = first_err & 0xff;
      __syncwarp();
    }
    over = __any_sync(FULLMASK, over);
    // FAILFAST: a record that fails spoils the whole call, so what it merged into the table before failing is never read
    uint32_t st = 0;
    if (err) st = make_status(err, -1);
    else if (!ok) st = make_status(TFR_E_MALFORMED_PROTO, -1);
    else if (over) { if (lane == 0) atomicMin(&A.first_err[4], row); }   // its entries past the window decide: unknown here
    else if (verr) st = make_status(verr == INF_ERR_KIND ? TFR_E_KIND_MISMATCH : TFR_E_EMPTY_SCALAR, -1);
    if constexpr (TOL) {
      if (!st && !over) {        // the record is kept: its clean survivors, context then feature_lists
        for (uint32_t w = 0; w < nwin; ++w) {
          const uint8_t* wb = wbase + w * INFER_WINDOW_BYTES;
          const unsigned long long* wh = reinterpret_cast<const unsigned long long*>(wb);
          const uint32_t* wc = reinterpret_cast<const uint32_t*>(wb + INFER_MAX_ENT * 8);
          const uint32_t* wk = reinterpret_cast<const uint32_t*>(wb + INFER_MAX_ENT * 12);
          for (uint32_t m = w ? keep1 : keep0; m; m &= m - 1) {
            const uint32_t i = lane + 32u * (uint32_t)__ffs(m) - 32u;
            infer_merge(A.table, A.data, wh[i], wk[i], wc[i] >> 8, (int)(wc[i] & 0xf), &A.first_err[1]);
          }
        }
      }
      __syncwarp();              // the windows are rewritten by the warp's next record
    }
    if (lane == 0) { A.status[row] = st; if (st) atomicMin(&A.first_err[0], row); }
  }
}

// compact the table: names copied out of the batch, one thread per slot
__global__ void infer_gather_kernel(const InferSlot* __restrict__ table, const uint8_t* __restrict__ data, uint32_t* __restrict__ counters /*[0] entries, [1] bytes*/,
                                    InferSlot* __restrict__ out_entries, uint8_t* __restrict__ out_names, uint32_t names_cap) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= INFER_TABLE_SLOTS || table[s].hash == 0ull) return;
  InferSlot e = table[s];
  uint32_t idx = atomicAdd(&counters[0], 1u);
  uint32_t off = atomicAdd(&counters[1], e.name_len);
  if (off + e.name_len <= names_cap) for (uint32_t i = 0; i < e.name_len; ++i) out_names[off + i] = data[e.name_off + i];
  e.name_off = off;
  out_entries[idx] = e;
}
