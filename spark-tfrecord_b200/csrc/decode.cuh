// decode.cuh -- K2/K3: CRC-32C verify + protobuf wire parse of Example / SequenceExample +
// schema-driven scatter into Arrow-layout columns.
//
// Replaces, per record, tensorflow-hadoop's payload CRC check, Example.parseFrom /
// SequenceExample.parseFrom (M/TFRecordFileReader.scala:73,76) and deserializeExample /
// deserializeSequenceExample (M/TFRecordDeserializer.scala:21-61, coercions :68-232).
//
// One warp owns one record.
//   pass 1 (decode_pass1_kernel): warp-parallel CRC of the payload; the map entries of Features are
//     discovered by a uniform hop over `0A len` fields, then parsed one entry per lane (32 at a time):
//     full validation of the wire format (every feature, in the schema or not, exactly like a full
//     protobuf parse), key lookup through a hash of the schema names, protobuf merge semantics
//     (duplicate key -> last wins, oneof switch discards, same kind concatenates, packed and unpacked
//     mixed), the reference's coercion/null rules, fixed-width scalars written directly, element and
//     byte counts + the source offset of each variable-width cell written to scratch.
//   scan: the counts are prefix-summed into Arrow offsets (scan.cuh).
//   pass 2 (decode_pass2_kernel): one lane per variable-width cell copies/decodes its values to
//     their final place (canonical cells straight from the packed payload, everything else through a
//     general two-walk emitter that reproduces the merge semantics).
#pragma once
#include "common.cuh"

// cell flags (pass 1 -> pass 2)
enum { CF_CANON = 0, CF_GENERAL = 1, CF_FLIST = 2 };

struct DecodeArgs {
  const uint8_t* data;        // framed bytes (device)
  const uint32_t* rec_off;    // [n+1]
  uint32_t n;                 // records to process
  uint32_t nbytes;            // size of `data`
  uint32_t verify;
  DevSchema sch;
  const CrcTables* tabs;
  // pass-1 outputs / pass-2 inputs
  uint32_t* status;           // [n]
  uint8_t* valid8;            // [nf][n]
  void* const* fix_values;    // [n_fix] typed value arrays
  uint32_t* cnt;              // [n_cnt][n]
  uint32_t* src;              // [n_var][n]
  uint8_t* cflag;             // [n_var][n]
  // pass-2 only
  uint32_t n_eff;             // rows to emit
  const int32_t* const* scan; // [n_cnt] exclusive prefix arrays (n+1 entries); level 0 ones are the Arrow offsets[0]
  int32_t* const* offs;       // [n_var*3] Arrow offsets arrays per level (level 0 == scan)
  void* const* var_values;    // [n_var] leaf value buffers
  const int32_t* var_field;   // [n_var] schema field of each var slot
  uint32_t flist_warp;        // 1: canonical FeatureList cells with fixed-width elements are emitted by decode_pass2_flist_kernel
  uint32_t canon_lean;        // 1: scalar string/binary cells and canonical 1-D list cells are emitted by decode_pass2_canon_kernel
  // pass 1 of a schema with ragged fields (decode_pass1_kernel<true>): [n_rag] pairs (x, its lengths part)
  const int32_t* rag;
  uint32_t n_rag;
};

// ---------------------------------------------------------------------------------------------
// Feature accumulation state (one map-entry value, possibly merged from several occurrences)
// ---------------------------------------------------------------------------------------------
struct FeatAcc {
  uint32_t kind;        // K_*
  uint32_t n;           // elements in the final run
  uint32_t nbytes;      // BYTES: sum of output lengths (java-transcoded when want_java) of the final run
  uint32_t first_len;   // BYTES: output length of the first element of the final run
  uint64_t first;       // INT64: value; FLOAT: bits; BYTES: batch offset of the first element's length varint
  uint32_t src;         // batch offset of the canonical payload (packed data / BytesList body)
  uint32_t nseg;        // value-carrying fields in the final run (FLOAT/INT64)
  uint32_t run_occ;     // kind-field occurrences in the final run
  bool simple;          // no unpacked / unknown fields seen in the final run
};
__device__ __forceinline__ void acc_reset(FeatAcc& a, uint32_t kind) {
  a.kind = kind; a.n = 0; a.nbytes = 0; a.first_len = 0; a.first = 0; a.src = 0; a.nseg = 0; a.run_occ = 0; a.simple = true;
}
__device__ __forceinline__ bool acc_canonical(const FeatAcc& a) {
  if (a.n == 0) return true;
  if (a.kind == K_BYTES) return a.run_occ <= 1 && a.simple;
  return a.nseg <= 1 && a.simple;
}

__device__ __forceinline__ uint32_t out_len_bytes(const uint8_t* p, uint32_t l, bool want_java) {
  if (!want_java || all_ascii(p, l)) return l;
  return java_utf8_transcode(p, l, nullptr);
}

// One occurrence of a oneof member of Feature: validates the list message and folds it into `a`.
__device__ __forceinline__ bool list_scan(uint32_t kind, Cur c, FeatAcc& a, bool want_java, const uint8_t* base) {
  if (kind != a.kind) acc_reset(a, kind);
  a.run_occ++;
  if (kind == K_BYTES && a.run_occ == 1) a.src = (uint32_t)(c.p - base);
  for (;;) {
    uint32_t tag;
    if (!rd_tag(c, tag)) return false;
    if (tag == 0) return true;
    if (kind == K_BYTES && tag == 0x0A) {
      const uint8_t* lp = c.p;
      uint32_t l;
      if (!rd_len(c, l)) return false;
      uint32_t ol = out_len_bytes(c.p, l, want_java);
      if (a.n == 0) { a.first = (uint64_t)(lp - base); a.first_len = ol; }
      a.n++; a.nbytes += ol;
      c.p += l;
    } else if (kind == K_FLOAT && tag == 0x0A) {
      uint32_t l;
      if (!rd_len(c, l)) return false;
      if (l & 3) return false;                       // readFloat past the limit: truncatedMessage
      if (l) {
        if (a.n == 0) a.first = load_u32_unaligned(c.p);
        a.nseg++; a.src = (uint32_t)(c.p - base);
        a.n += l >> 2;
      }
      c.p += l;
    } else if (kind == K_FLOAT && tag == 0x0D) {
      if (c.end - c.p < 4) return false;
      if (a.n == 0) a.first = load_u32_unaligned(c.p);
      a.nseg++; a.simple = false; a.n++;
      c.p += 4;
    } else if (kind == K_INT64 && tag == 0x0A) {
      uint32_t l;
      if (!rd_len(c, l)) return false;
      if (l) {
        Cur pk{c.p, c.p + l};
        a.nseg++; a.src = (uint32_t)(c.p - base);
        while (pk.p < pk.end) {
          uint64_t v;
          if (!rd_varint64(pk, v)) return false;
          if (a.n == 0) a.first = v;
          a.n++;
        }
      }
      c.p += l;
    } else if (kind == K_INT64 && tag == 0x08) {
      uint64_t v;
      if (!rd_varint64(c, v)) return false;
      if (a.n == 0) a.first = v;
      a.nseg++; a.simple = false; a.n++;
    } else {
      if (!skip_field(c, tag)) return false;
      a.simple = false;
    }
  }
}
// Feature message body merged into `a` (Feature.Builder.mergeFrom)
__device__ __forceinline__ bool feature_scan(Cur c, FeatAcc& a, bool want_java, const uint8_t* base) {
  for (;;) {
    uint32_t tag;
    if (!rd_tag(c, tag)) return false;
    if (tag == 0) return true;
    uint32_t kind = tag == 0x0A ? K_BYTES : tag == 0x12 ? K_FLOAT : tag == 0x1A ? K_INT64 : K_NONE;
    if (kind != K_NONE) {
      uint32_t l;
      if (!rd_len(c, l)) return false;
      Cur body{c.p, c.p + l};
      c.p += l;
      if (!list_scan(kind, body, a, want_java, base)) return false;
    } else if (!skip_field(c, tag)) return false;
  }
}

// ---------------------------------------------------------------------------------------------
// schema lookup
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int schema_lookup(const DevSchema& s, const uint8_t* key, uint32_t klen) {
  if (s.n_fields == 0) return -1;
  uint32_t h = name_hash(key, klen);
  uint32_t slot = h & (uint32_t)s.ht_mask;
  for (;;) {
    int f = s.ht[slot];
    if (f < 0) return -1;
    const DevField& fd = s.fields[f];
    if (fd.hash == h && fd.name_len == klen) {
      const uint8_t* nm = s.names + fd.name_off;
      bool eq = true;
      for (uint32_t i = 0; i < klen; ++i) if (nm[i] != key[i]) { eq = false; break; }
      if (eq) return f;
    }
    slot = (slot + 1) & (uint32_t)s.ht_mask;
  }
}

// FeatureList value accumulation (SequenceExample.feature_lists entries)
struct FlistAcc {
  uint32_t steps, tot_n, tot_bytes;
  int err;   // first failing step's error (TFR_E_*), 0 none
};

// ---------------------------------------------------------------------------------------------
// pass 1
// ---------------------------------------------------------------------------------------------
// writes the outputs of field f (and of every later schema field with the same name) for one row
__device__ __forceinline__ void write_feature_cell(const DecodeArgs& A, uint32_t row, int f, const FeatAcc& a, uint32_t entry_pos,
                                                   uint8_t* fstate) {
  for (; f >= 0; f = A.sch.fields[f].dup_next) {
    const DevField& fd = A.sch.fields[f];
    int code = 0;
    if (fd.elem_type == TFR_T_NULL) { fstate[f] = 3; continue; }          // NullType: always null (:71-72)
    if (fd.depth >= 2) code = TFR_E_BAD_NESTING;                            // :119
    else if (a.kind != (uint32_t)fd.kind) code = TFR_E_KIND_MISMATCH;       // require(...) :178,189,201,212
    else if (fd.depth == 0 && a.n == 0) code = TFR_E_EMPTY_SCALAR;          // .head
    if (code) { fstate[f] = (uint8_t)(-code); continue; }
    fstate[f] = 1;
    if (fd.depth == 0) {
      if (fd.fix_slot >= 0) {
        void* vp = A.fix_values[fd.fix_slot];
        switch (fd.elem_type) {
          case TFR_T_INT64: reinterpret_cast<int64_t*>(vp)[row] = (int64_t)a.first; break;
          case TFR_T_INT32: reinterpret_cast<int32_t*>(vp)[row] = (int32_t)(uint32_t)a.first; break;   // .toInt
          case TFR_T_FLOAT32: reinterpret_cast<uint32_t*>(vp)[row] = (uint32_t)a.first; break;
          default: reinterpret_cast<double*>(vp)[row] = (double)__uint_as_float((uint32_t)a.first); break;   // .toDouble
        }
      } else {   // scalar string / binary: first element
        A.cnt[(size_t)fd.cnt_slot * A.n + row] = a.first_len;
        A.src[(size_t)fd.var_slot * A.n + row] = (uint32_t)a.first;
        A.cflag[(size_t)fd.var_slot * A.n + row] = CF_CANON;
      }
    } else {     // depth 1
      A.cnt[(size_t)fd.cnt_slot * A.n + row] = a.n;
      if (fd.n_levels == 2) A.cnt[(size_t)(fd.cnt_slot + 1) * A.n + row] = a.nbytes;
      bool canon = acc_canonical(a);
      A.src[(size_t)fd.var_slot * A.n + row] = canon ? a.src : entry_pos;
      A.cflag[(size_t)fd.var_slot * A.n + row] = canon ? CF_CANON : CF_GENERAL;
    }
  }
}
__device__ __forceinline__ void write_flist_cell(const DecodeArgs& A, uint32_t row, int f, const FlistAcc& a, uint32_t entry_pos,
                                                 uint8_t* fstate) {
  const DevField& fd = A.sch.fields[f];
  if (a.err) { fstate[f] = (uint8_t)(-a.err); return; }
  fstate[f] = 1;
  A.cnt[(size_t)fd.cnt_slot * A.n + row] = a.steps;
  if (fd.depth == 1) {
    if (fd.n_levels == 2) A.cnt[(size_t)(fd.cnt_slot + 1) * A.n + row] = a.tot_bytes;
  } else {
    A.cnt[(size_t)(fd.cnt_slot + 1) * A.n + row] = a.tot_n;
    if (fd.n_levels == 3) A.cnt[(size_t)(fd.cnt_slot + 2) * A.n + row] = a.tot_bytes;
  }
  A.src[(size_t)fd.var_slot * A.n + row] = entry_pos;
  A.cflag[(size_t)fd.var_slot * A.n + row] = CF_FLIST;
}

// Parse one map entry {1: key, 2: value} of Features (is_flist = false) or FeatureLists (true).
// Returns false when the entry is malformed.  On return f = matched schema field or -1.
__device__ __forceinline__ bool parse_entry(const DecodeArgs& A, const uint8_t* ep, uint32_t elen, bool is_flist, int& f, FeatAcc& acc,
                                            FlistAcc& facc) {
  // (a) top-level fields of the entry: the last key wins; values are revisited in (b)
  const uint8_t* key = nullptr;
  uint32_t klen = 0;
  {
    Cur c{ep, ep + elen};
    for (;;) {
      uint32_t tag;
      if (!rd_tag(c, tag)) return false;
      if (tag == 0) break;
      if (tag == 0x0A) {
        uint32_t l;
        if (!rd_len(c, l)) return false;
        if (!utf8_valid(c.p, l)) return false;      // proto3 string key: readStringRequireUtf8
        key = c.p; klen = l; c.p += l;
      } else if (!skip_field(c, tag)) return false;
    }
  }
  f = schema_lookup(A.sch, key, klen);
  bool want_java = false;
  for (int g = f; g >= 0; g = A.sch.fields[g].dup_next) want_java |= A.sch.fields[g].elem_type == TFR_T_STRING;
  // (b) values, deep
  acc_reset(acc, K_NONE);
  facc.steps = facc.tot_n = facc.tot_bytes = 0; facc.err = 0;
  Cur c{ep, ep + elen};
  for (;;) {
    uint32_t tag;
    if (!rd_tag(c, tag)) return false;
    if (tag == 0) break;
    if (tag != 0x12) { if (!skip_field(c, tag)) return false; continue; }
    uint32_t l;
    if (!rd_len(c, l)) return false;
    Cur body{c.p, c.p + l};
    c.p += l;
    if (!is_flist) {
      if (!feature_scan(body, acc, want_java, A.data)) return false;
    } else {
      // FeatureList: repeated Feature feature = 1 (steps append across value occurrences)
      for (;;) {
        uint32_t t2;
        if (!rd_tag(body, t2)) return false;
        if (t2 == 0) break;
        if (t2 != 0x0A) { if (!skip_field(body, t2)) return false; continue; }
        uint32_t sl;
        if (!rd_len(body, sl)) return false;
        FeatAcc st;
        acc_reset(st, K_NONE);
        if (!feature_scan(Cur{body.p, body.p + sl}, st, want_java, A.data)) return false;
        body.p += sl;
        facc.steps++;
        if (f >= 0 && !facc.err) {
          const DevField& fd = A.sch.fields[f];
          if (fd.depth == 0) facc.err = TFR_E_BAD_NESTING;                              // :142
          else if (st.kind != (uint32_t)fd.kind) facc.err = TFR_E_KIND_MISMATCH;
          else if (fd.depth == 1) {                                                     // element = head of the step
            if (st.n == 0) facc.err = TFR_E_EMPTY_SCALAR;
            else { facc.tot_n++; facc.tot_bytes += st.first_len; }
          } else { facc.tot_n += st.n; facc.tot_bytes += st.nbytes; }
        }
      }
    }
  }
  if (is_flist && f >= 0 && A.sch.fields[f].depth == 0 && !facc.err) facc.err = TFR_E_BAD_NESTING;   // empty FeatureList into a scalar
  return true;
}

// Parses up to 32 entries (one per lane) and publishes the winners.  ent_ptr/ent_len are per-lane.
__device__ __forceinline__ bool process_round(const DecodeArgs& A, uint32_t row, uint32_t nent, const uint8_t* ent_ptr, uint32_t ent_len,
                                              uint32_t ent_pos, bool is_flist, uint8_t* fstate) {
  const uint32_t lane = threadIdx.x & 31;
  int f = -1;
  FeatAcc acc;
  FlistAcc facc;
  bool ok = true;
  if (lane < nent) ok = parse_entry(A, ent_ptr, ent_len, is_flist, f, acc, facc);
  if (__any_sync(FULLMASK, !ok)) return false;
  // duplicate keys inside the round: the last entry in wire order wins (Map.put)
  uint32_t same = __match_any_sync(FULLMASK, f);
  bool winner = f >= 0 && (31 - __clz(same)) == (int)lane;
  if (winner) {
    if (!is_flist) write_feature_cell(A, row, f, acc, ent_pos, fstate);
    else {
      // context wins over feature_lists for the same name (M/TFRecordDeserializer.scala:45-55); context
      // rounds are all done before the first feature_lists round.  fstate 2 marks "seen in feature_lists".
      for (int g = f; g >= 0; g = A.sch.fields[g].dup_next) {
        uint8_t st = fstate[g];
        if (st == 0 || (st & 0x40)) {     // unseen, or seen only in a previous feature_lists entry
          FlistAcc fa = facc;
          const DevField& fd = A.sch.fields[g];
          if (fd.elem_type == TFR_T_NULL) { fstate[g] = 0x40 | 3; continue; }
          // per-field re-evaluation is needed only for duplicate names with different types; parse_entry used
          // the first field of the chain
          if (g != f) {
            // conservative: recompute is not possible without re-parsing; duplicate-named columns of different
            // shapes fed from feature_lists are rejected at schema creation (api.cu)
          }
          write_flist_cell(A, row, g, fa, ent_pos, fstate);
          fstate[g] |= 0x40;
        }
      }
    }
  }
  __syncwarp();
  return true;
}

// Walks `0A len` entries of one Features / FeatureLists message body, 32 at a time.
__device__ __forceinline__ bool walk_map_body(const DecodeArgs& A, uint32_t row, Cur body, bool is_flist, uint8_t* fstate,
                                              uint32_t& nent, const uint8_t*& my_ptr, uint32_t& my_len, uint32_t& my_pos) {
  const uint32_t lane = threadIdx.x & 31;
  for (;;) {
    uint32_t tag;
    if (!rd_tag(body, tag)) return false;
    if (tag == 0) return true;
    if (tag != 0x0A) { if (!skip_field(body, tag)) return false; continue; }
    const uint8_t* lp = body.p;
    uint32_t l;
    if (!rd_len(body, l)) return false;
    if (lane == nent) { my_ptr = body.p; my_len = l; my_pos = (uint32_t)(lp - A.data); }
    body.p += l;
    if (++nent == 32) {
      if (!process_round(A, row, nent, my_ptr, my_len, my_pos, is_flist, fstate)) return false;
      nent = 0;
    }
  }
}

// a ragged field's consistency check (ragged.cuh): the sum of the lengths part's values in row `row` (the final run of the winning
// entry, by Feature's merge rules: a list of another kind discards what came before), ~0 when one is negative or above INT32_MAX.
// `src`: the packed varints (cflag CF_CANON, `count` of them) or the map entry's length prefix (CF_GENERAL).
__device__ __forceinline__ uint64_t ragged_lengths_sum(const uint8_t* data, uint32_t nbytes, uint32_t src, bool canon, uint32_t count) {
  uint64_t sum = 0;
  bool bad = false;
  auto add = [&](uint64_t v) { if (v > 0x7fffffffull) bad = true; else sum += v; };
  if (canon) {
    Cur pk{data + src, data + nbytes};
    for (uint32_t i = 0; i < count; ++i) { uint64_t v; if (!rd_varint64(pk, v)) return ~0ull; add(v); }
    return bad ? ~0ull : sum;
  }
  Cur c{data + src, data + nbytes};
  uint32_t l;
  if (!rd_len(c, l)) return ~0ull;
  Cur e{c.p, c.p + l};
  for (;;) {                                                   // MapEntry: value = 2 (repeated occurrences merge)
    uint32_t tag;
    if (!rd_tag(e, tag)) return ~0ull;
    if (tag == 0) break;
    if (tag != 0x12) { if (!skip_field(e, tag)) return ~0ull; continue; }
    if (!rd_len(e, l)) return ~0ull;
    Cur f{e.p, e.p + l};
    e.p += l;
    for (;;) {                                                 // Feature: bytes_list = 1, float_list = 2, int64_list = 3
      if (!rd_tag(f, tag)) return ~0ull;
      if (tag == 0) break;
      if (tag != 0x0A && tag != 0x12 && tag != 0x1A) { if (!skip_field(f, tag)) return ~0ull; continue; }
      if (!rd_len(f, l)) return ~0ull;
      Cur b{f.p, f.p + l};
      f.p += l;
      if (tag != 0x1A) { sum = 0; bad = false; continue; }    // the oneof switches: the int64 values before it are discarded
      for (;;) {                                               // Int64List: value = 1, packed or not
        if (!rd_tag(b, tag)) return ~0ull;
        if (tag == 0) break;
        if (tag == 0x08) { uint64_t v; if (!rd_varint64(b, v)) return ~0ull; add(v); }
        else if (tag == 0x0A) {
          if (!rd_len(b, l)) return ~0ull;
          Cur pk{b.p, b.p + l};
          while (pk.p < pk.end) { uint64_t v; if (!rd_varint64(pk, v)) return ~0ull; add(v); }
          b.p += l;
        } else if (!skip_field(b, tag)) return ~0ull;
      }
    }
  }
  return bad ? ~0ull : sum;
}

// the row-splits partition's consistency check (TFR_S_RAGGED_ROW_SPLITS): true when the splits part's values in row `row` (the
// final run of the winning entry, by Feature's merge rules, as in ragged_lengths_sum) are at least one entry, the first 0, none
// decreasing and the last `n_values`.  `src`, `canon`, `count` as there.
__device__ __forceinline__ bool ragged_splits_ok(const uint8_t* data, uint32_t nbytes, uint32_t src, bool canon, uint32_t count,
                                                 uint32_t n_values) {
  uint32_t m = 0;
  int64_t first = 0, last = 0;
  bool dec = false;
  auto add = [&](uint64_t u) { const int64_t v = (int64_t)u; if (m == 0) first = v; else if (v < last) dec = true; last = v; ++m; };
  if (canon) {
    Cur pk{data + src, data + nbytes};
    for (uint32_t i = 0; i < count; ++i) { uint64_t v; if (!rd_varint64(pk, v)) return false; add(v); }
  } else {
    Cur c{data + src, data + nbytes};
    uint32_t l;
    if (!rd_len(c, l)) return false;
    Cur e{c.p, c.p + l};
    for (;;) {                                                 // MapEntry: value = 2 (repeated occurrences merge)
      uint32_t tag;
      if (!rd_tag(e, tag)) return false;
      if (tag == 0) break;
      if (tag != 0x12) { if (!skip_field(e, tag)) return false; continue; }
      if (!rd_len(e, l)) return false;
      Cur f{e.p, e.p + l};
      e.p += l;
      for (;;) {                                               // Feature: bytes_list = 1, float_list = 2, int64_list = 3
        if (!rd_tag(f, tag)) return false;
        if (tag == 0) break;
        if (tag != 0x0A && tag != 0x12 && tag != 0x1A) { if (!skip_field(f, tag)) return false; continue; }
        if (!rd_len(f, l)) return false;
        Cur b{f.p, f.p + l};
        f.p += l;
        if (tag != 0x1A) { m = 0; dec = false; continue; }    // the oneof switches: the int64 values before it are discarded
        for (;;) {                                             // Int64List: value = 1, packed or not
          if (!rd_tag(b, tag)) return false;
          if (tag == 0) break;
          if (tag == 0x08) { uint64_t v; if (!rd_varint64(b, v)) return false; add(v); }
          else if (tag == 0x0A) {
            if (!rd_len(b, l)) return false;
            Cur pk{b.p, b.p + l};
            while (pk.p < pk.end) { uint64_t v; if (!rd_varint64(pk, v)) return false; add(v); }
            b.p += l;
          } else if (!skip_field(b, tag)) return false;
        }
      }
    }
  }
  return m > 0 && first == 0 && !dec && last == (int64_t)n_values;
}

// a row that fails before the per-field epilogue (bad CRC, malformed proto): zero counts, null validity
__device__ __forceinline__ void null_fill_row(const DecodeArgs& A, uint32_t row) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t f = lane; f < (uint32_t)A.sch.n_fields; f += 32) A.valid8[(size_t)f * A.n + row] = 0;
  for (uint32_t c = lane; c < (uint32_t)A.sch.n_cnt; c += 32) A.cnt[(size_t)c * A.n + row] = 0;
}

// RG: the schema has ragged fields, whose parts must agree (RAGGED, include/tfrgpu.h); without them the kernel is unchanged.
// RS: they are stored with row splits (TFR_S_RAGGED_ROW_SPLITS), decode_pass1_splits_kernel.
template <bool RG, bool RS>
__device__ __forceinline__ void decode_pass1(const DecodeArgs& A) {
  extern __shared__ uint32_t smem[];
  uint32_t* stab = smem;
  crc_stage_tables(stab, A.tabs);
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nf = (uint32_t)A.sch.n_fields;
  const uint32_t fstride = (nf + 3) & ~3u;
  uint8_t* fstate = reinterpret_cast<uint8_t*>(smem + CRC_SMEM_WORDS) + (size_t)wid * fstride;
  __syncthreads();
  for (uint32_t row = blockIdx.x * warps + wid; row < A.n; row += gridDim.x * warps) {
    const uint32_t off = A.rec_off[row];
    const uint32_t len = A.rec_off[row + 1] - off - 16;
    const uint8_t* payload = A.data + off + 12;
    uint32_t status = 0;
    if (A.verify) {
      uint32_t crc = crc_warp(stab, payload, len);
      if (crc_mask(crc) != load_u32_unaligned(payload + len)) status = make_status(TFR_E_CRC_DATA, -1);
    }
    if (A.sch.record_type == TFR_RT_BYTE_ARRAY) {            // deserializeByteArray (:17-19)
      if (lane == 0) {
        A.status[row] = status;
        A.cnt[row] = len; A.src[row] = off + 12; A.cflag[row] = CF_CANON; A.valid8[row] = 1;
      }
      continue;
    }
    if (status) { null_fill_row(A, row); if (lane == 0) A.status[row] = status; continue; }
    for (uint32_t i = lane; i < nf; i += 32) fstate[i] = 0;
    __syncwarp();
    bool ok = true;
    uint32_t nent = 0, my_len = 0, my_pos = 0;
    const uint8_t* my_ptr = nullptr;
    // Example.features / SequenceExample.context: field 1 (repeated occurrences merge)
    {
      Cur top{payload, payload + len};
      for (;;) {
        uint32_t tag;
        if (!rd_tag(top, tag)) { ok = false; break; }
        if (tag == 0) break;
        if (tag == 0x0A || (tag == 0x12 && A.sch.record_type == TFR_RT_SEQUENCE_EXAMPLE)) {
          uint32_t l;
          if (!rd_len(top, l)) { ok = false; break; }
          if (tag == 0x0A && !walk_map_body(A, row, Cur{top.p, top.p + l}, false, fstate, nent, my_ptr, my_len, my_pos)) { ok = false; break; }
          top.p += l;
        } else if (!skip_field(top, tag)) { ok = false; break; }
      }
      if (ok && nent) { ok = process_round(A, row, nent, my_ptr, my_len, my_pos, false, fstate); nent = 0; }
    }
    // SequenceExample.feature_lists: field 2, after every context entry has been seen
    if (ok && A.sch.record_type == TFR_RT_SEQUENCE_EXAMPLE) {
      Cur top{payload, payload + len};
      for (;;) {
        uint32_t tag;
        if (!rd_tag(top, tag) || tag == 0) break;                 // malformed input was caught above
        if (tag == 0x0A || tag == 0x12) {
          uint32_t l;
          if (!rd_len(top, l)) break;
          if (tag == 0x12 && !walk_map_body(A, row, Cur{top.p, top.p + l}, true, fstate, nent, my_ptr, my_len, my_pos)) { ok = false; break; }
          top.p += l;
        } else if (!skip_field(top, tag)) break;
      }
      if (ok && nent) { ok = process_round(A, row, nent, my_ptr, my_len, my_pos, true, fstate); nent = 0; }
    }
    if (!ok) { null_fill_row(A, row); if (lane == 0) A.status[row] = make_status(TFR_E_MALFORMED_PROTO, -1); continue; }
    __syncwarp();
    // absent fields -> null or NullPointerException; first error in schema order wins
    uint32_t worst = 0xffffffffu;
    for (uint32_t f = lane; f < nf; f += 32) {
      uint8_t st = fstate[f] & 0x3f;
      const DevField& fd = A.sch.fields[f];
      uint8_t valid = 0;
      if (st == 1) valid = 1;
      else if (st == 0 || st == 3) {                              // absent, or NullType
        if (st == 0 && !fd.nullable) worst = min(worst, (f << 8) | (uint32_t)(-TFR_E_NULL_IN_NONNULL));
        if (fd.fix_slot >= 0) {
          void* vp = A.fix_values[fd.fix_slot];
          if (fd.width == 8) reinterpret_cast<uint64_t*>(vp)[row] = 0; else reinterpret_cast<uint32_t*>(vp)[row] = 0;
        } else if (fd.var_slot >= 0) {
          for (int l = 0; l < fd.n_levels; ++l) A.cnt[(size_t)(fd.cnt_slot + l) * A.n + row] = 0;
        }
      } else worst = min(worst, (f << 8) | st);
      A.valid8[(size_t)f * A.n + row] = valid;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) worst = min(worst, __shfl_xor_sync(FULLMASK, worst, o));
    if constexpr (RG) {
      // last in a record's precedence: a ragged field whose parts disagree (one absent, a negative length, a wrong sum) is
      // TFR_E_BAD_NESTING at x; the first such x in field order
      if (worst == 0xffffffffu) {
        uint32_t bad = 0xffffffffu;
        for (uint32_t j = lane; j < A.n_rag; j += 32) {
          const int x = A.rag[2 * j], L = A.rag[2 * j + 1];
          const bool px = (fstate[x] & 0x3f) == 1, pl = (fstate[L] & 0x3f) == 1;
          bool mis = px != pl;
          if (px && pl) {
            const DevField& fl = A.sch.fields[L];
            const size_t vs = (size_t)fl.var_slot * A.n + row;
            if constexpr (RS) {
              mis = !ragged_splits_ok(A.data, A.nbytes, A.src[vs], A.cflag[vs] == CF_CANON, A.cnt[(size_t)fl.cnt_slot * A.n + row],
                                      A.cnt[(size_t)A.sch.fields[x].cnt_slot * A.n + row]);
            } else {
              const uint64_t sum = ragged_lengths_sum(A.data, A.nbytes, A.src[vs], A.cflag[vs] == CF_CANON, A.cnt[(size_t)fl.cnt_slot * A.n + row]);
              mis = sum != (uint64_t)A.cnt[(size_t)A.sch.fields[x].cnt_slot * A.n + row];
            }
          }
          if (mis) bad = min(bad, (uint32_t)x);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bad = min(bad, __shfl_xor_sync(FULLMASK, bad, o));
        if (bad != 0xffffffffu) worst = (bad << 8) | (uint32_t)(-TFR_E_BAD_NESTING);
      }
    }
    if (lane == 0) A.status[row] = worst == 0xffffffffu ? 0u : ((worst & 0xff) | (((worst >> 8) + 1) << 8));
  }
}
template <bool RG>
__global__ void __launch_bounds__(256) decode_pass1_kernel(DecodeArgs A) { decode_pass1<RG, false>(A); }
__global__ void __launch_bounds__(256) decode_pass1_splits_kernel(DecodeArgs A) { decode_pass1<true, true>(A); }

// ---------------------------------------------------------------------------------------------
// pass 2: emit variable-width cells
// ---------------------------------------------------------------------------------------------
struct ElemSink {
  int elem_type;
  uint8_t* values;     // leaf buffer
  uint32_t vpos;       // next leaf index (fixed width) or next byte (STRING/BINARY)
  int32_t* leaf_off;   // STRING/BINARY inside a list: offsets of the leaf level, else nullptr
  uint32_t epos;       // next element slot in leaf_off
  uint32_t limit;      // max elements to accept (1 = head only)
  uint32_t taken;
};
__device__ __forceinline__ void sink_int(ElemSink& s, uint64_t v) {
  if (s.taken >= s.limit) return;
  if (s.elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(s.values)[s.vpos] = (int64_t)v;
  else reinterpret_cast<int32_t*>(s.values)[s.vpos] = (int32_t)(uint32_t)v;
  s.vpos++; s.taken++;
}
__device__ __forceinline__ void sink_float(ElemSink& s, uint32_t bits) {
  if (s.taken >= s.limit) return;
  if (s.elem_type == TFR_T_FLOAT32) reinterpret_cast<uint32_t*>(s.values)[s.vpos] = bits;
  else reinterpret_cast<double*>(s.values)[s.vpos] = (double)__uint_as_float(bits);
  s.vpos++; s.taken++;
}
// copy l bytes (any alignment on both sides), 16 at a time: the bytes are loaded as words before they are stored (a plain
// byte loop is one dependent global load -> store chain: the compiler cannot move a load above the previous store of the
// other pointer).  Only words that hold a needed byte (plus the one word after, which is still inside the record: every
// payload is followed by its 4-byte CRC) are read.  With ascii_only, the copy stops BEFORE the first 16-byte group that
// holds a byte >= 0x80 and returns false (nothing past the ASCII prefix has been written).
__device__ __forceinline__ bool copy_bytes16(uint8_t* d, const uint8_t* p, uint32_t l, bool ascii_only) {
  for (uint32_t i = 0; i < l; i += 16) {
    const uint32_t r = min(16u, l - i);
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = (uint32_t)(4 * k) < r ? load_u32_unaligned(p + i + 4 * k) : 0u;
    if (ascii_only) {
      uint32_t hi = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t live = r >= (uint32_t)(4 * k + 4) ? 0xffffffffu : r > (uint32_t)(4 * k) ? (1u << (8 * (r - 4 * k))) - 1u : 0u;   // bytes of word k below l
        hi |= w[k] & live;
      }
      if (hi & 0x80808080u) return false;
    }
#pragma unroll
    for (int k = 0; k < 16; ++k)
      if ((uint32_t)k < r) d[i + k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
  }
  return true;
}
__device__ __forceinline__ void sink_bytes(ElemSink& s, const uint8_t* p, uint32_t l) {
  if (s.taken >= s.limit) return;
  uint8_t* d = s.values + s.vpos;
  // StringType = Java UTF-8 decode + re-encode: the identity for ASCII; anything else goes through the transcoder, which
  // rewrites the cell from its start (the ASCII prefix already copied is what it writes there too)
  if (copy_bytes16(d, p, l, s.elem_type == TFR_T_STRING)) s.vpos += l;
  else s.vpos += java_utf8_transcode(p, l, d);
  if (s.leaf_off) { s.leaf_off[s.epos + 1] = (int32_t)s.vpos; s.epos++; }
  s.taken++;
}
// emit every element of one list message body (kind known, input already validated by pass 1)
__device__ __forceinline__ void list_emit(uint32_t kind, Cur c, ElemSink& s) {
  for (;;) {
    uint32_t tag;
    if (!rd_tag(c, tag) || tag == 0) return;
    if (kind == K_BYTES && tag == 0x0A) {
      uint32_t l; if (!rd_len(c, l)) return;
      sink_bytes(s, c.p, l); c.p += l;
    } else if (kind == K_FLOAT && tag == 0x0A) {
      uint32_t l; if (!rd_len(c, l)) return;
      for (uint32_t i = 0; i + 4 <= l; i += 4) sink_float(s, load_u32_unaligned(c.p + i));
      c.p += l;
    } else if (kind == K_FLOAT && tag == 0x0D) {
      if (c.end - c.p < 4) return;
      sink_float(s, load_u32_unaligned(c.p)); c.p += 4;
    } else if (kind == K_INT64 && tag == 0x0A) {
      uint32_t l; if (!rd_len(c, l)) return;
      Cur pk{c.p, c.p + l};
      while (pk.p < pk.end) { uint64_t v; if (!rd_varint64(pk, v)) return; sink_int(s, v); }
      c.p += l;
    } else if (kind == K_INT64 && tag == 0x08) {
      uint64_t v; if (!rd_varint64(c, v)) return;
      sink_int(s, v);
    } else if (!skip_field(c, tag)) return;
  }
}
// Walk the kind-field occurrences of Feature bodies.  mode 0: find where the final run starts
// (returns its occurrence index through run_first, final kind through kind); mode 1: emit the
// occurrences >= run_first.
struct OccState { uint32_t occ, run_first, kind; };
__device__ __forceinline__ void feature_occ_walk(Cur c, OccState& o, int mode, ElemSink* s) {
  for (;;) {
    uint32_t tag;
    if (!rd_tag(c, tag) || tag == 0) return;
    uint32_t kind = tag == 0x0A ? K_BYTES : tag == 0x12 ? K_FLOAT : tag == 0x1A ? K_INT64 : K_NONE;
    if (kind != K_NONE) {
      uint32_t l; if (!rd_len(c, l)) return;
      if (mode == 0) { if (kind != o.kind) { o.kind = kind; o.run_first = o.occ; } }
      else if (o.occ >= o.run_first) list_emit(kind, Cur{c.p, c.p + l}, *s);
      o.occ++;
      c.p += l;
    } else if (!skip_field(c, tag)) return;
  }
}
// general emit of the merged Feature carried by the value fields (tag 0x12) of a map entry
__device__ __forceinline__ void entry_feature_emit(Cur entry, ElemSink& s) {
  OccState o{0, 0, K_NONE};
  for (int mode = 0; mode < 2; ++mode) {
    Cur c = entry;
    o.occ = 0;
    for (;;) {
      uint32_t tag;
      if (!rd_tag(c, tag) || tag == 0) break;
      if (tag == 0x12) {
        uint32_t l; if (!rd_len(c, l)) break;
        feature_occ_walk(Cur{c.p, c.p + l}, o, mode, &s);
        c.p += l;
      } else if (!skip_field(c, tag)) break;
    }
  }
}
// general emit of one step Feature (single message body)
__device__ __forceinline__ void step_feature_emit(Cur body, ElemSink& s) {
  OccState o{0, 0, K_NONE};
  feature_occ_walk(body, o, 0, &s);
  o.occ = 0;
  feature_occ_walk(body, o, 1, &s);
}

// the rare string that is not ASCII: kept out of line so that the lean kernel below stays small
__device__ __noinline__ uint32_t transcode_cell(const uint8_t* p, uint32_t l, uint8_t* d) { return java_utf8_transcode(p, l, d); }

// pass 2 for the cells every ordinary file consists of: scalar string / binary columns (the first element of a BytesList)
// and canonical 1-D lists (one packed field, or a plain BytesList).  Same thread-per-(row, cell) mapping as
// decode_pass2_kernel, but without the general two-walk emitter inlined: 32 registers instead of 128 + stack, four times
// the resident threads, and every cell is a chain of dependent loads, so the time goes with the resident threads.
#define CANON_STAGE_BYTES 2048
__global__ void __launch_bounds__(256, 6) decode_pass2_canon_kernel(DecodeArgs A) {
  // One warp takes 32 consecutive rows of ONE variable-width column (lane = row): the cells of those rows are adjacent in
  // the output, so the warp assembles them in shared memory and writes the range with coalesced word stores; a thread
  // per cell writing its own bytes costs one 32-byte sector per byte stored.
  __shared__ __align__(16) uint8_t s_stage[8][CANON_STAGE_BYTES + 16];
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nvar = (uint32_t)A.sch.n_var;
  const uint32_t groups = (A.n_eff + 31) / 32;
  const unsigned long long total = (unsigned long long)groups * nvar;
  for (unsigned long long gidx = (unsigned long long)blockIdx.x * warps + wid; gidx < total; gidx += (unsigned long long)gridDim.x * warps) {
    const uint32_t v = (uint32_t)(gidx % nvar), row = (uint32_t)(gidx / nvar) * 32 + lane;
    const DevField& fd = A.sch.fields[A.var_field[v]];
    if (fd.depth > 1) continue;                                           // warp-uniform
    const bool in = row < A.n_eff;
    const int32_t* sc = A.scan[fd.cnt_slot];
    const int32_t off0 = in ? sc[row] : 0;
    uint32_t cnt0 = in ? (uint32_t)(sc[row + 1] - off0) : 0u;             // elements, or bytes of a scalar string
    bool foreign = false;                                                 // a non-empty cell that decode_pass2_kernel writes
    if (cnt0 && fd.depth == 1 && A.cflag[(size_t)v * A.n + row] != CF_CANON) { cnt0 = 0; foreign = true; }
    const uint8_t* p = A.data + (cnt0 ? A.src[(size_t)v * A.n + row] : 0u);
    uint8_t* values = reinterpret_cast<uint8_t*>(A.var_values[v]);
    const bool is_str = fd.elem_type == TFR_T_STRING;
    const bool bytes_leaf = fd.kind == K_BYTES;
    if (fd.depth == 1 && bytes_leaf) {                                    // list of strings: element loop per lane, direct stores
      if (cnt0) {
        int32_t* leaf = A.offs[v * 3 + 1];
        uint32_t vpos = (uint32_t)A.scan[fd.cnt_slot + 1][row];
        Cur c{p, A.data + A.nbytes};
        for (uint32_t i = 0; i < cnt0; ++i) {
          uint32_t tag, l;
          if (!rd_tag(c, tag) || !rd_len(c, l)) break;
          uint8_t* d = values + vpos;
          if (copy_bytes16(d, c.p, l, is_str)) vpos += l; else vpos += transcode_cell(c.p, l, d);
          leaf[(uint32_t)off0 + i + 1] = (int32_t)vpos;
          c.p += l;
        }
      }
      continue;
    }
    // output bytes of this lane's cell and of the whole group (adjacent rows -> adjacent output)
    const uint32_t w = bytes_leaf ? 1u : (uint32_t)fd.width;
    const uint32_t my_bytes = cnt0 * w;
    uint32_t grp_bytes;
    const uint32_t my_off = warp_excl_scan_u32(my_bytes, grp_bytes);
    if (grp_bytes == 0) continue;
    // first output byte of the group: the first lane that has a cell knows it
    const uint32_t has = __ballot_sync(0xffffffffu, cnt0 != 0);
    const uint32_t first_lane = (uint32_t)__ffs((int)has) - 1;
    const unsigned long long base = __shfl_sync(0xffffffffu, (unsigned long long)(uint32_t)off0 * w, first_lane);
    // staging needs the group's cells to be one contiguous output range: no cell of another kernel in between
    const bool staged = grp_bytes <= CANON_STAGE_BYTES && !__any_sync(0xffffffffu, foreign);
    uint8_t* d = staged ? s_stage[wid] + (uint32_t)(base & 3) + my_off : values + (size_t)(uint32_t)off0 * w;
    bool redo = false;                                                    // a non-ASCII string: the transcoder writes it
    if (cnt0) {
      if (fd.depth == 0) {                                                // src = the length varint of the first element
        Cur c{p, p + 16};
        uint32_t l = 0; uint64_t lv;
        if (rd_varint64(c, lv)) l = (uint32_t)lv;
        p = c.p;
        if (!copy_bytes16(d, p, l, is_str)) { redo = true; if (!staged) transcode_cell(p, l, d); }
        cnt0 = l;
      } else if (fd.kind == K_FLOAT) {                                    // src = the packed payload
        if (fd.elem_type == TFR_T_FLOAT32) { uint32_t* q = reinterpret_cast<uint32_t*>(d); for (uint32_t i = 0; i < cnt0; ++i) { const uint32_t x = load_u32_unaligned(p + 4 * i); if (staged) memcpy(d + 4 * i, &x, 4); else q[i] = x; } }
        else { for (uint32_t i = 0; i < cnt0; ++i) { const double x = (double)__uint_as_float(load_u32_unaligned(p + 4 * i)); if (staged) memcpy(d + 8 * i, &x, 8); else reinterpret_cast<double*>(d)[i] = x; } }
      } else {
        Cur pk{p, p + (size_t)cnt0 * 10};
        for (uint32_t i = 0; i < cnt0; ++i) {
          uint64_t x; if (!rd_varint64(pk, x)) break;
          if (fd.elem_type == TFR_T_INT64) { const int64_t y = (int64_t)x; if (staged) memcpy(d + 8 * i, &y, 8); else reinterpret_cast<int64_t*>(d)[i] = y; }
          else { const int32_t y = (int32_t)(uint32_t)x; if (staged) memcpy(d + 4 * i, &y, 4); else reinterpret_cast<int32_t*>(d)[i] = y; }
        }
      }
    }
    if (!staged) continue;
    // a transcoded string may be longer than its raw bytes but its output length is what the offsets say: write it
    // straight to its place after the group's staged bytes are out (rare)
    __syncwarp();
    {
      uint8_t* g = values + base;                                         // group's first output byte
      const uint8_t* sb = s_stage[wid] + (uint32_t)(base & 3);
      // head bytes up to 4-byte alignment, aligned words, tail bytes
      const uint32_t headb = min(grp_bytes, (uint32_t)((4 - (base & 3)) & 3));
      if (lane < headb) g[lane] = sb[lane];
      const uint32_t nw = (grp_bytes - headb) >> 2;
      const uint32_t* sw = reinterpret_cast<const uint32_t*>(sb + headb);  // 4-byte aligned: (base & 3) + headb = 0 mod 4
      uint32_t* gw = reinterpret_cast<uint32_t*>(g + headb);
      for (uint32_t i = lane; i < nw; i += 32) gw[i] = sw[i];
      const uint32_t tailb = grp_bytes - headb - 4 * nw;
      if (lane < tailb) g[headb + 4 * nw + lane] = sb[headb + 4 * nw + lane];
    }
    __syncwarp();
    if (redo) transcode_cell(p, cnt0, values + (size_t)(uint32_t)off0 * w);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(256) decode_pass2_kernel(DecodeArgs A) {
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nvar = (uint32_t)A.sch.n_var;
  if (A.sch.record_type == TFR_RT_BYTE_ARRAY) {
    for (uint32_t row = blockIdx.x * warps + wid; row < A.n_eff; row += gridDim.x * warps) {
      // whole-warp copy of the payload
      const uint8_t* s = A.data + A.src[row];
      uint8_t* d = reinterpret_cast<uint8_t*>(A.var_values[0]) + A.scan[0][row];
      uint32_t l = (uint32_t)(A.scan[0][row + 1] - A.scan[0][row]);
      for (uint32_t i = lane; i < l; i += 32) d[i] = s[i];
    }
    return;
  }
  // one thread per (row, variable-width cell), cells of a row adjacent: every lane has work whatever the
  // number of variable-width columns is
  const unsigned long long total = (unsigned long long)A.n_eff * nvar;
  for (unsigned long long cidx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; cidx < total; cidx += (unsigned long long)gridDim.x * blockDim.x) {
    const uint32_t row = (uint32_t)(cidx / nvar);
    {
      const uint32_t v = (uint32_t)(cidx % nvar);
      {
      const int f = A.var_field[v];
      const DevField& fd = A.sch.fields[f];
      const int32_t off0 = A.scan[fd.cnt_slot][row];
      const uint32_t cnt0 = (uint32_t)(A.scan[fd.cnt_slot][row + 1] - off0);
      if (cnt0 == 0) continue;             // null, empty list or empty string: nothing to emit (src/cflag are undefined for nulls)
      const uint32_t src = A.src[(size_t)v * A.n + row];
      const uint32_t flag = A.cflag[(size_t)v * A.n + row];
      ElemSink s;
      s.elem_type = fd.elem_type; s.values = reinterpret_cast<uint8_t*>(A.var_values[v]);
      s.leaf_off = nullptr; s.epos = 0; s.limit = 0xffffffffu; s.taken = 0;
      const bool varlen = fd.elem_type == TFR_T_STRING || fd.elem_type == TFR_T_BINARY;
      if (A.canon_lean && (fd.depth == 0 || (fd.depth == 1 && flag == CF_CANON))) continue;   // decode_pass2_canon_kernel
      if (fd.depth == 0) {                                   // scalar string / binary
        Cur c{A.data + src, A.data + src + 16};              // length varint of the first element (validated in pass 1)
        uint32_t l = 0; uint64_t lv;
        if (rd_varint64(c, lv)) l = (uint32_t)lv;
        s.vpos = (uint32_t)off0; s.limit = 1;
        sink_bytes(s, c.p, l);
        continue;
      }
      if (flag == CF_FLIST) {
        if (A.flist_warp && fd.depth == 2 && !varlen) continue;   // decode_pass2_flist_kernel
        // FeatureList: steps across the value occurrences of the entry
        Cur e{A.data + src, A.data + src + 16};
        uint64_t elen; if (!rd_varint64(e, elen)) continue;
        Cur entry{e.p, e.p + (uint32_t)elen};
        int32_t* off1 = A.offs[v * 3 + 1];
        uint32_t step = 0;
        if (fd.depth == 1) {                                 // array of heads
          if (varlen) { s.leaf_off = off1; s.epos = (uint32_t)off0; s.vpos = (uint32_t)A.scan[fd.cnt_slot + 1][row]; }
          else s.vpos = (uint32_t)off0;
        } else {
          if (varlen) { s.leaf_off = A.offs[v * 3 + 2]; s.epos = (uint32_t)A.scan[fd.cnt_slot + 1][row]; s.vpos = (uint32_t)A.scan[fd.cnt_slot + 2][row]; }
          else s.vpos = (uint32_t)A.scan[fd.cnt_slot + 1][row];
        }
        for (;;) {
          uint32_t tag;
          if (!rd_tag(entry, tag) || tag == 0) break;
          if (tag != 0x12) { if (!skip_field(entry, tag)) break; continue; }
          uint32_t l; if (!rd_len(entry, l)) break;
          Cur fl{entry.p, entry.p + l};
          entry.p += l;
          for (;;) {
            uint32_t t2;
            if (!rd_tag(fl, t2) || t2 == 0) break;
            if (t2 != 0x0A) { if (!skip_field(fl, t2)) break; continue; }
            uint32_t sl; if (!rd_len(fl, sl)) break;
            s.taken = 0; s.limit = fd.depth == 1 ? 1u : 0xffffffffu;
            step_feature_emit(Cur{fl.p, fl.p + sl}, s);
            fl.p += sl;
            if (fd.depth == 2) off1[(uint32_t)off0 + step + 1] = (int32_t)(varlen ? s.epos : s.vpos);
            step++;
          }
        }
        continue;
      }
      // depth 1 from a Feature
      if (varlen) { s.leaf_off = A.offs[v * 3 + 1]; s.epos = (uint32_t)off0; s.vpos = (uint32_t)A.scan[fd.cnt_slot + 1][row]; }
      else s.vpos = (uint32_t)off0;
      if (flag == CF_CANON) {
        if (cnt0 == 0) continue;
        const uint8_t* p = A.data + src;
        if (fd.kind == K_FLOAT) {
          for (uint32_t i = 0; i < cnt0; ++i) sink_float(s, load_u32_unaligned(p + 4 * i));
        } else if (fd.kind == K_INT64) {
          Cur pk{p, p + (size_t)cnt0 * 10};
          for (uint32_t i = 0; i < cnt0; ++i) { uint64_t x; if (!rd_varint64(pk, x)) break; sink_int(s, x); }
        } else {
          Cur c{p, A.data + A.nbytes};
          for (uint32_t i = 0; i < cnt0; ++i) {
            uint32_t tag, l;
            if (!rd_tag(c, tag) || !rd_len(c, l)) break;
            sink_bytes(s, c.p, l); c.p += l;
          }
        }
      } else {
        Cur e{A.data + src, A.data + src + 16};
        uint64_t elen; if (!rd_varint64(e, elen)) continue;
        entry_feature_emit(Cur{e.p, e.p + (uint32_t)elen}, s);
      }
      }
    }
  }
}

// pass 2 for FeatureList cells (ArrayType(ArrayType(fixed-width))) whose bytes the tile kernel has validated as canonical
// (`{0A flen Feature}*`, Feature = kind llen [0A plen packed]): one WARP per cell instead of one thread.  Lane 0 walks
// the step headers (a dependent chain, but over a few consecutive cache lines), 32 steps at a time; then every lane
// takes one step: counts its elements, a warp prefix sum gives its position in the leaf buffer and the inner offsets,
// and it copies / converts its elements.  (decode_pass2_kernel walks all steps of a cell in one thread through the
// general two-walk emitter, which dominated the SequenceExample decode time.)
#define FLIST_BUF_BYTES 4096
__global__ void __launch_bounds__(256) decode_pass2_flist_kernel(DecodeArgs A) {
  __shared__ uint32_t s_pos[8][32], s_len[8][32];
  __shared__ __align__(16) uint8_t s_buf[8][FLIST_BUF_BYTES];
  const uint32_t warps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t nvar = (uint32_t)A.sch.n_var;
  const unsigned long long total = (unsigned long long)A.n_eff * nvar;
  for (unsigned long long cidx = (unsigned long long)blockIdx.x * warps + wid; cidx < total; cidx += (unsigned long long)gridDim.x * warps) {
    const uint32_t row = (uint32_t)(cidx / nvar), v = (uint32_t)(cidx % nvar);
    const DevField& fd = A.sch.fields[A.var_field[v]];
    if (fd.depth != 2 || fd.elem_type == TFR_T_STRING || fd.elem_type == TFR_T_BINARY) continue;
    const int32_t off0 = A.scan[fd.cnt_slot][row];
    const uint32_t steps = (uint32_t)(A.scan[fd.cnt_slot][row + 1] - off0);
    if (steps == 0 || A.cflag[(size_t)v * A.n + row] != CF_FLIST) continue;
    int32_t* off1 = A.offs[v * 3 + 1];
    uint32_t epos = (uint32_t)A.scan[fd.cnt_slot + 1][row];
    const uint32_t src = A.src[(size_t)v * A.n + row];
    // entry = elen | 0A klen key | 12 vlen | FeatureList body.  The whole entry is first copied into shared memory with
    // coalesced word loads (one DRAM round trip instead of one per cache line of the dependent walk); entries larger
    // than the buffer are walked in global memory.
    uint32_t span = 0;
    if (lane == 0) {
      Cur e{A.data + src, A.data + A.nbytes};
      uint64_t x = 0;
      rd_varint64(e, x);
      span = (uint32_t)(e.p - (A.data + src)) + (uint32_t)x;
    }
    span = __shfl_sync(0xffffffffu, span, 0);
    const uint32_t a0 = src & ~3u;
    const uint8_t* base = A.data;                       // byte at batch offset q = base[q - delta]
    uint32_t delta = 0;
    __syncwarp();
    if ((src - a0) + span + 4 <= FLIST_BUF_BYTES) {
      const uint32_t nw = ((src - a0) + span + 3) >> 2;
      const uint32_t* g = reinterpret_cast<const uint32_t*>(A.data + a0);
      uint32_t* sb = reinterpret_cast<uint32_t*>(s_buf[wid]);
      for (uint32_t i = lane; i < nw; i += 32) sb[i] = g[i];
      base = s_buf[wid]; delta = a0;
      __syncwarp();
    }
    const uint8_t* lim = base + (src - delta) + span;
    uint32_t p = 0;
    if (lane == 0) {
      Cur e{base + (src - delta), lim};
      uint64_t x; uint32_t tag, l;
      rd_varint64(e, x);
      rd_tag(e, tag); rd_len(e, l); e.p += l;          // key
      rd_tag(e, tag); rd_len(e, l);                    // value = FeatureList
      p = (uint32_t)(e.p - base) + delta;
    }
    for (uint32_t s0 = 0; s0 < steps; s0 += 32) {
      const uint32_t nb = min(32u, steps - s0);
      if (lane == 0) {
        // the walk is one dependent chain in one lane: keep it to a byte load + add per step (`0A flen`, flen < 128);
        // longer steps take the general varint reader
        const uint8_t* q = base + (p - delta);
        for (uint32_t i = 0; i < nb; ++i) {
          uint32_t l = q[1];
          if (l < 0x80) q += 2;
          else { Cur c{q + 1, lim}; l = 0; rd_len(c, l); q = c.p; }
          s_pos[wid][i] = (uint32_t)(q - base) + delta; s_len[wid][i] = l;
          q += l;
        }
        p = (uint32_t)(q - base) + delta;
      }
      __syncwarp();
      uint32_t cnt = 0, pk = 0, plen = 0;
      if (lane < nb && s_len[wid][lane] != 0) {
        Cur f{base + (s_pos[wid][lane] - delta), base + (s_pos[wid][lane] - delta) + s_len[wid][lane]};
        uint32_t tag, llen = 0;
        rd_tag(f, tag); rd_len(f, llen);               // kind tag, list length
        if (llen != 0) {
          rd_tag(f, tag); rd_len(f, plen);             // 0A plen: the packed field
          pk = (uint32_t)(f.p - base) + delta;
          if (fd.kind == K_FLOAT) cnt = plen >> 2;
          else for (uint32_t i = 0; i < plen; ++i) cnt += (base[pk - delta + i] & 0x80) ? 0u : 1u;
        }
      }
      uint32_t tot;
      const uint32_t ex = warp_excl_scan_u32(cnt, tot);
      if (lane < nb) {
        off1[(uint32_t)off0 + s0 + lane + 1] = (int32_t)(epos + ex + cnt);
        const uint32_t o = epos + ex;
        const uint8_t* q = base + (pk - delta);
        if (fd.kind == K_FLOAT) {
          if (fd.elem_type == TFR_T_FLOAT32) { uint32_t* d = reinterpret_cast<uint32_t*>(A.var_values[v]) + o; for (uint32_t i = 0; i < cnt; ++i) d[i] = load_u32_unaligned(q + 4 * i); }
          else { double* d = reinterpret_cast<double*>(A.var_values[v]) + o; for (uint32_t i = 0; i < cnt; ++i) d[i] = (double)__uint_as_float(load_u32_unaligned(q + 4 * i)); }
        } else {
          Cur c{q, q + plen};
          for (uint32_t i = 0; i < cnt; ++i) {
            uint64_t x = 0; rd_varint64(c, x);
            if (fd.elem_type == TFR_T_INT64) reinterpret_cast<int64_t*>(A.var_values[v])[o + i] = (int64_t)x;
            else reinterpret_cast<int32_t*>(A.var_values[v])[o + i] = (int32_t)(uint32_t)x;
          }
        }
      }
      epos += tot;
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// validity bytes -> Arrow bitmaps (+ null counts), first-error reduction
// ---------------------------------------------------------------------------------------------
__global__ void pack_validity_kernel(const uint8_t* __restrict__ valid8, uint32_t n, uint32_t n_eff, uint32_t nf, uint32_t bitmap_stride,
                                     uint8_t* __restrict__ bitmaps, unsigned long long* __restrict__ null_counts) {
  const uint32_t nb = (n_eff + 7) >> 3;
  const uint32_t f = blockIdx.y;
  if (f >= nf) return;
  unsigned long long local = 0;
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    uint32_t bits = 0;
    const uint8_t* v = valid8 + (size_t)f * n + (size_t)b * 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint32_t r = b * 8 + i;
      if (r < n_eff) { if (v[i]) bits |= 1u << i; else local++; }
    }
    bitmaps[(size_t)f * bitmap_stride + b] = (uint8_t)bits;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(FULLMASK, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(&null_counts[f], local);
}

struct DecodeSummary {       // device -> host after pass 1 + scans
  uint32_t first_err_row;    // 0xffffffff none
  uint32_t first_err_status;
  uint32_t n_eff;
  uint32_t consumed;         // rec_off[n_eff]: bytes of the delivered rows
};
__global__ void first_error_kernel(const uint32_t* __restrict__ status, uint32_t n, DecodeSummary* __restrict__ out) {
  uint32_t best = 0xffffffffu;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (status[i] != 0) { best = i; break; }    // indices visited by one thread are increasing
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(FULLMASK, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0xffffffffu) atomicMin(&out->first_err_row, best);
}
// n_eff + totals at n_eff for every scanned array (so that rows after the first error vanish)
__global__ void summary_kernel(const uint32_t* __restrict__ status, const uint32_t* __restrict__ rec_off, uint32_t n,
                               DecodeSummary* __restrict__ out, const int32_t* const* __restrict__ scan, uint32_t n_cnt,
                               int64_t* __restrict__ totals, int64_t* __restrict__ first_counts) {
  uint32_t e = out->first_err_row;
  uint32_t n_eff = e == 0xffffffffu ? n : e;
  if (threadIdx.x == 0) {
    out->n_eff = n_eff;
    out->first_err_status = (e == 0xffffffffu || !status) ? 0 : status[e];
    out->consumed = rec_off ? rec_off[n_eff] : 0;
  }
  for (uint32_t a = threadIdx.x; a < n_cnt; a += blockDim.x) {
    totals[a] = scan[a][n_eff];
    first_counts[a] = n_eff ? scan[a][1] : 0;       // count of row 0 (shape learning for the tile fast path)
  }
}
