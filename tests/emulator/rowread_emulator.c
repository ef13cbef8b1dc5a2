/*
 * rowread_emulator.c -- plays, in plain C against include/tfrgpu.h ONLY, the row-reading BlockIterator of INTEGRATION.md: the
 * read side Spark drives through the reference's buildReader (M/DefaultSource.scala:118-136, M/TFRecordFileReader.scala:16-83),
 * with every row handed out as a Spark UnsafeRow the GPU laid out.  Line for line: block k is read into pinned staging slot
 * k % slots behind the tail block k-1 left unconsumed, submitted (tfr_decode_submit), and its rows and their copy are enqueued
 * at once (tfr_batch_rows_async); the reader then takes where block k ends (tfr_batch_consumed), submits block k+1, and only
 * then reads block k's rows (tfr_batch_rows).  After the last row of a batch its error, if any, ends the iteration, like the
 * reference's next() throwing after the rows before the bad record.
 *
 *   rowread_emulator abi              -> device-free checks of the C ABI this loop uses
 *   rowread_emulator rowread FILE BLOCK -> read FILE in BLOCK-byte blocks; one line per row (FNV-1a 64 of its UnsafeRow bytes,
 *                                        16 hex digits), then "status CODE row ERROR_ROW rows N" and the decoder's counters
 * Exit code 0 = every check passed.  The schema is that of rowwrite_emulator.c and fileformat_emulator.c.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tfrgpu.h"

#define CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "emulator: %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); exit(1); } } while (0)
#define OK(call) do { int32_t rc_ = (call); CHECK(rc_ == 0, "%s -> %d (%s: %s)", #call, rc_, tfr_status_string(rc_), tfr_last_error()); } while (0)

/* ---- the data schema of this emulation: StructType(id: Long, w: Float, name: String (nullable), emb: Array[Float]) ---- */
enum { N_FIELDS = 4 };
static const tfr_field FIELDS[N_FIELDS] = {
  {"id", 2, TFR_T_INT64, 0, 0}, {"w", 1, TFR_T_FLOAT32, 0, 1}, {"name", 4, TFR_T_STRING, 0, 1}, {"emb", 3, TFR_T_FLOAT32, 1, 1},
};

static uint64_t fnv1a64(const uint8_t* p, size_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001b3ull; }
  return h;
}

/* ================================ row-reading BlockIterator (INTEGRATION.md) ================================ */
typedef struct {
  FILE* in; tfr_decoder* dec;
  size_t block; int slots, slot, eof, closed;
  uint8_t* carry; size_t carry_n;
  tfr_batch* ahead; uint8_t* ahead_buf; size_t ahead_bytes; int ahead_final;
  tfr_batch* cur; const uint8_t* rows; const int64_t* offs; int64_t n, i;
  int32_t status; int64_t error_row;             /* what the iteration ended with (the exception the reference throws) */
} BlockIterator;

/* [carry | next file bytes] -> pinned slot -> GPU, and the rows pass and its copy queued behind the decode; returns at once */
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
  OK(tfr_decode_submit(it->dec, buf, it->ahead_bytes, 0, it->ahead_final, &it->ahead));
  OK(tfr_batch_rows_async(it->ahead, 1, NULL, 0, 0, NULL));
}
static int advance(BlockIterator* it) {
  if (it->cur) {                                                     /* the reference's next() throws here */
    tfr_batch_info info;
    OK(tfr_batch_status(it->cur, &info));
    tfr_batch_release(it->cur); it->cur = NULL;
    if (info.error_code) { it->status = info.error_code; it->error_row = info.error_row; return 0; }
  }
  if (!it->ahead) return 0;
  tfr_batch* b = it->ahead; it->ahead = NULL;
  if (!it->ahead_final) {                                            /* the partial record behind `used` opens the next block */
    size_t used = 0;
    OK(tfr_batch_consumed(b, &used));                                /* known after the frame index, before the rows */
    CHECK(used <= it->ahead_bytes, "consumed %zu of %zu", used, it->ahead_bytes);
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
static void close_it(BlockIterator* it) {                           /* idempotent (M/TFRecordFileReader.scala:36-40) */
  if (it->closed) return;
  if (it->cur) tfr_batch_release(it->cur);
  if (it->ahead) tfr_batch_release(it->ahead);
  it->cur = it->ahead = NULL;
  fclose(it->in);
  free(it->carry); it->carry = NULL;
  it->closed = 1;
}

static int cmd_rowread(const char* path, size_t block) {
  CHECK(block > 0, "BLOCK must be positive");
  tfr_schema* schema = NULL;
  OK(tfr_schema_create(FIELDS, N_FIELDS, TFR_RT_EXAMPLE, &schema));
  BlockIterator it;
  memset(&it, 0, sizeof it);
  it.in = fopen(path, "rb");
  CHECK(it.in, "cannot open %s", path);
  OK(tfr_decoder_create(schema, 0, TFR_F_DEFAULT, &it.dec));
  it.block = block; it.slots = tfr_decoder_num_staging_slots(); it.error_row = -1;
  CHECK(it.slots >= 2, "staging slots %d", it.slots);
  submit_next(&it);
  int64_t rows = 0;
  while (has_next(&it)) {
    const int64_t o = it.offs[it.i], len = it.offs[it.i + 1] - o;
    CHECK(len >= 8 + 8 * N_FIELDS && len % 8 == 0, "row %lld: %lld bytes", (long long)rows, (long long)len);
    printf("%016llx\n", (unsigned long long)fnv1a64(it.rows + o, (size_t)len));
    ++it.i; ++rows;
  }
  close_it(&it);
  close_it(&it);                                                     /* a second close does nothing */
  int64_t st[10] = {0};
  OK(tfr_decoder_get_stats(it.dec, st, 10));
  printf("status %d row %lld rows %lld\n", it.status, (long long)it.error_row, (long long)rows);
  printf("rowread stats: batches=%lld pipelined=%lld redone=%lld rows_async=%lld rows_rebuilt=%lld\n", (long long)st[0], (long long)st[1],
         (long long)st[2], (long long)st[7], (long long)st[8]);
  tfr_decoder_destroy(it.dec);
  tfr_schema_destroy(schema);
  return 0;
}

/* what the loop relies on, checked without a device: the ABI version, the argument errors of tfr_batch_rows_async (a partition
 * row is checked before the batch), the counters' bound, the pipeline depth */
static int cmd_abi(void) {
  printf("abi %d\n", tfr_abi_version());
  CHECK(tfr_batch_rows_async(NULL, 1, NULL, 0, 0, NULL) == TFR_E_INVALID_ARG, "null batch");
  CHECK(strstr(tfr_last_error(), "null batch") != NULL, "null batch: %s", tfr_last_error());
  const uint8_t part[8] = {0}, var[1] = {0};
  CHECK(tfr_batch_rows_async(NULL, 1, part, 8, 1, var) == TFR_E_INVALID_ARG, "short partition row");
  CHECK(strstr(tfr_last_error(), "fixed region") != NULL, "short partition row: %s", tfr_last_error());
  CHECK(tfr_batch_rows_async(NULL, 0, part, 8, 0, NULL) == TFR_E_INVALID_ARG, "bytes without fields");
  int64_t st[10];
  CHECK(tfr_decoder_get_stats(NULL, st, 10) == TFR_E_INVALID_ARG, "stats of a null decoder");
  printf("staging slots %d\n", tfr_decoder_num_staging_slots());
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "abi")) return cmd_abi();
  if (argc >= 4 && !strcmp(argv[1], "rowread")) return cmd_rowread(argv[2], (size_t)atoll(argv[3]));
  fprintf(stderr, "usage: %s abi | rowread FILE BLOCK\n", argv[0]);
  return 2;
}
