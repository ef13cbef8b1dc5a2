/*
 * position_emulator.c -- plays, in plain C against include/tfrgpu.h ONLY, the row-reading BlockIterator of INTEGRATION.md with
 * Spark's generated metadata columns: the required schema holds _tmp_metadata_row_index and _tmp_metadata_record_offset,
 * lowered to TFR_T_ROW_INDEX and TFR_T_RECORD_OFFSET.  Line for line: block k is read into pinned staging slot k % slots behind
 * the tail block k-1 left unconsumed and submitted at its place in the file (tfr_decode_submit_at: the entries and bytes in
 * front of it), and its rows and their copy are enqueued at once (tfr_batch_rows_async); the reader then takes where block k
 * ends and the entries in it (tfr_batch_extent), submits block k+1 there, and only then reads block k's rows
 * (tfr_batch_rows).  After the last row of a batch its error, if any, ends the iteration.
 *
 *   position_emulator abi                   -> device-free checks of the C ABI this loop uses
 *   position_emulator positions FILE BLOCK MODE
 *                                           -> read FILE in BLOCK-byte blocks, MODE 0 FAILFAST or 1 DROPMALFORMED; one line per
 *                                              row, "ROW_INDEX RECORD_OFFSET" read from the row's UnsafeRow slots, then
 *                                              "status CODE row ERROR_ROW rows N"
 * Exit code 0 = every check passed.  The data schema is that of rowwrite_emulator.c.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tfrgpu.h"

#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "emulator: %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)
#define OK(call) do { int32_t rc_ = (call); CHECK(rc_ == 0, "%s -> %d (%s: %s)", #call, rc_, tfr_status_string(rc_), tfr_last_error()); } while (0)

/* StructType(id: Long, w: Float, name: String, emb: Array[Float]) plus Spark's two temporary metadata columns */
enum { N_FIELDS = 6, F_ROW_INDEX = 4, F_RECORD_OFFSET = 5 };
static const tfr_field FIELDS[N_FIELDS] = {
  {"id", 2, TFR_T_INT64, 0, 0}, {"w", 1, TFR_T_FLOAT32, 0, 1}, {"name", 4, TFR_T_STRING, 0, 1}, {"emb", 3, TFR_T_FLOAT32, 1, 1},
  {"_tmp_metadata_row_index", 23, TFR_T_ROW_INDEX, 0, 0}, {"_tmp_metadata_record_offset", 27, TFR_T_RECORD_OFFSET, 0, 0},
};

/* ================================ row-reading BlockIterator with positions (INTEGRATION.md) ================================ */
typedef struct {
  FILE* in; tfr_decoder* dec;
  size_t block; int slots, slot, eof, closed;
  uint8_t* carry; size_t carry_n;
  tfr_batch* ahead; uint8_t* ahead_buf; size_t ahead_bytes; int ahead_final;
  int64_t first_entry, first_offset;             /* the next block's place in the file: entries and bytes in front of it */
  tfr_batch* cur; const uint8_t* rows; const int64_t* offs; int64_t n, i;
  int32_t status; int64_t error_row;
} BlockIterator;

static void submit_next(BlockIterator* it) {
  if (it->eof) return;
  void* p = NULL; size_t cap = 0;
  OK(tfr_decoder_staging_slot(it->dec, it->slot, it->carry_n + it->block, &p, &cap));
  it->slot = (it->slot + 1) % it->slots;
  uint8_t* buf = p;
  if (it->carry_n) memcpy(buf, it->carry, it->carry_n);
  const size_t got = fread(buf + it->carry_n, 1, it->block, it->in);
  it->eof = got < it->block;
  it->ahead_buf = buf; it->ahead_bytes = it->carry_n + got; it->ahead_final = it->eof;
  OK(tfr_decode_submit_at(it->dec, buf, it->ahead_bytes, 0, it->ahead_final, it->first_entry, it->first_offset, &it->ahead));
  OK(tfr_batch_rows_async(it->ahead, 1, NULL, 0, 0, NULL));
}
static int advance(BlockIterator* it) {
  if (it->cur) {
    tfr_batch_info info;
    OK(tfr_batch_status(it->cur, &info));
    tfr_batch_release(it->cur); it->cur = NULL;
    if (info.error_code) { it->status = info.error_code; it->error_row = info.error_row; return 0; }
  }
  if (!it->ahead) return 0;
  tfr_batch* b = it->ahead; it->ahead = NULL;
  if (!it->ahead_final) {
    size_t used = 0; int64_t entries = 0;
    OK(tfr_batch_extent(b, &used, &entries));                        /* known after the frame index, before the rows */
    CHECK(used <= it->ahead_bytes && entries >= 0, "consumed %zu of %zu, %lld entries", used, it->ahead_bytes, (long long)entries);
    it->first_entry += entries; it->first_offset += (int64_t)used;
    it->carry_n = it->ahead_bytes - used;
    it->carry = realloc(it->carry, it->carry_n + 1);
    memcpy(it->carry, it->ahead_buf + used, it->carry_n);
    submit_next(it);                                                 /* block k+1 is copied and indexed while block k decodes */
  }
  it->cur = b;
  size_t nb = 0;
  OK(tfr_batch_rows(b, 1, (const void**)&it->rows, &it->offs, &it->n, &nb));
  CHECK(it->offs[0] == 0 && (size_t)it->offs[it->n] == nb, "row offsets 0..%lld do not span %zu bytes", (long long)it->n, nb);
  it->i = 0;
  return 1;
}
static int has_next(BlockIterator* it) {
  while (!it->closed && it->i >= it->n) if (!advance(it)) return 0;
  return !it->closed;
}
static void close_it(BlockIterator* it) {
  if (it->closed) return;
  if (it->cur) tfr_batch_release(it->cur);
  if (it->ahead) tfr_batch_release(it->ahead);
  it->cur = it->ahead = NULL;
  fclose(it->in);
  free(it->carry); it->carry = NULL;
  it->closed = 1;
}

/* an UnsafeRow's LongType slot f: one null-bit word (6 fields), then 8 bytes per field */
static int64_t long_slot(const uint8_t* row, int f) {
  int64_t v;
  memcpy(&v, row + 8 + 8 * f, 8);
  return v;
}

static int cmd_positions(const char* path, size_t block, int mode) {
  CHECK(block > 0 && (mode == 0 || mode == 1), "BLOCK must be positive, MODE 0 or 1");
  tfr_schema* schema = NULL;
  OK(tfr_schema_create(FIELDS, N_FIELDS, TFR_RT_EXAMPLE, &schema));
  BlockIterator it;
  memset(&it, 0, sizeof it);
  it.in = fopen(path, "rb");
  CHECK(it.in, "cannot open %s", path);
  OK(tfr_decoder_create(schema, 0, TFR_F_DEFAULT | (mode ? TFR_F_DROP_MALFORMED : 0u), &it.dec));
  it.block = block; it.slots = tfr_decoder_num_staging_slots(); it.error_row = -1;
  submit_next(&it);
  int64_t rows = 0, last = -1;
  while (has_next(&it)) {
    const uint8_t* row = it.rows + it.offs[it.i];
    CHECK((row[0] & 0x30) == 0, "row %lld: a generated field is null", (long long)rows);
    const int64_t ri = long_slot(row, F_ROW_INDEX), ro = long_slot(row, F_RECORD_OFFSET);
    CHECK(ri > last, "row %lld: row index %lld after %lld", (long long)rows, (long long)ri, (long long)last);
    last = ri;
    printf("%lld %lld\n", (long long)ri, (long long)ro);
    ++it.i; ++rows;
  }
  close_it(&it);
  printf("status %d row %lld rows %lld\n", it.status, (long long)it.error_row, (long long)rows);
  tfr_decoder_destroy(it.dec);
  tfr_schema_destroy(schema);
  return 0;
}

/* what the loop relies on, checked without a device: the schema's lowering and refusals, the argument errors of the calls */
static int cmd_abi(void) {
  printf("abi %d\n", tfr_abi_version());
  tfr_schema* s = NULL;
  OK(tfr_schema_create(FIELDS, N_FIELDS, TFR_RT_EXAMPLE, &s));
  CHECK(tfr_schema_num_fields(s) == N_FIELDS, "fields %d", tfr_schema_num_fields(s));
  tfr_encoder* enc = NULL;
  CHECK(tfr_encoder_create(s, 0, 0, &enc) == TFR_E_UNSUPPORTED_TYPE && !enc, "an encoder takes no generated field");
  tfr_schema_destroy(s);
  tfr_field nested = FIELDS[F_ROW_INDEX];
  nested.depth = 1;
  s = NULL;
  CHECK(tfr_schema_create(&nested, 1, TFR_RT_EXAMPLE, &s) == TFR_E_UNSUPPORTED_TYPE && !s, "a generated field at depth 1");
  CHECK(strstr(tfr_last_error(), "_tmp_metadata_row_index") != NULL, "the error names the field: %s", tfr_last_error());
  tfr_batch* b = NULL; size_t used = 0; int64_t entries = 0;
  CHECK(tfr_decode_submit_at(NULL, NULL, 0, 0, 1, 0, 0, &b) == TFR_E_INVALID_ARG && !b, "submit_at of a null decoder");
  CHECK(tfr_decode_at(NULL, NULL, 0, 0, 1, 0, 0, &b, &used) == TFR_E_INVALID_ARG && !b, "decode_at of a null decoder");
  CHECK(tfr_batch_extent(NULL, &used, &entries) == TFR_E_INVALID_ARG, "extent of a null batch");
  printf("staging slots %d\n", tfr_decoder_num_staging_slots());
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "abi")) return cmd_abi();
  if (argc >= 5 && !strcmp(argv[1], "positions")) return cmd_positions(argv[2], (size_t)atoll(argv[3]), atoi(argv[4]));
  fprintf(stderr, "usage: %s abi | positions FILE BLOCK MODE\n", argv[0]);
  return 2;
}
