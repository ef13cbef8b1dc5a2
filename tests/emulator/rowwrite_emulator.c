/*
 * rowwrite_emulator.c -- plays, in plain C against include/tfrgpu.h ONLY, the pipelined RowWriter of INTEGRATION.md: the
 * write side Spark drives through the reference's OutputWriter (M/TFRecordOutputWriter.scala:12-24 ctor, :26-38 write(row),
 * :40-43 close()), with each row handed over as a Spark UnsafeRow and the flushes encoded by tfr_encode_rows_submit while
 * the next rows are appended.
 *
 *   rowwrite_emulator rowwrite DIR N FLUSH   -> write N rows to DIR/part-00000.tfrecord, FLUSH rows per flush
 * Exit code 0 = every check passed.  The schema and the rows are those of fileformat_emulator.c (row_value_* below, the same
 * deterministic functions of the row index), so the Python side of the test regenerates them and compares the file with
 * the CPU oracle's reading of it.
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
static int64_t row_value_id(int64_t i) { return i * i - 7 * i - 3; }
static float row_value_w(int64_t i) { return (float)i * 0.5f - 100.0f; }
static int row_name_is_null(int64_t i) { return i % 11 == 5; }
static int row_value_name(int64_t i, char* out) { return sprintf(out, "row-%lld-%s", (long long)i, (i % 3) ? "x" : "yy"); }
static int row_emb_len(int64_t i) { return (int)(i % 6); }
static float row_value_emb(int64_t i, int k) { return (float)(i + k) * 0.25f; }

/* ================================ pipelined RowWriter (INTEGRATION.md) ================================ */
/* OutputWriter.write(row) receives an UnsafeRow: the JVM appends its bytes (one Platform.copyMemory) and its offset to the
 * current slot.  A flush submits the slot and moves on to the next one; before a slot is refilled, the submission that read
 * it is waited on and its framed bytes are written to the file.  close() flushes and drains the slots in order. */
enum { RW_MAX_ROW = 256 };           /* the largest row of this schema: 40 fixed bytes, a name below 64 bytes, 5 floats */
typedef struct {
  tfr_schema* schema; tfr_encoder* enc; FILE* out; int closed;
  int slots, k;                      /* k: the slot rows are appended to */
  uint8_t* st[8]; int32_t* offs[8]; tfr_encoded* pending[8];
  int64_t n, flush_rows, rows_written, flushes;
} RowWriter;

static void rw_put64(uint8_t* p, uint64_t v) { memcpy(p, &v, 8); }
/* row i of the generator as an UnsafeRow (null bitset word, 4 slots, then the variable region); returns its size */
static int32_t unsafe_row_of(int64_t i, uint8_t* row) {
  memset(row, 0, RW_MAX_ROW);
  const int32_t fixed = 8 + 8 * N_FIELDS;
  int32_t pos = fixed;
  uint64_t nulls = 0;
  rw_put64(row + 8, (uint64_t)row_value_id(i));
  float w = row_value_w(i); memcpy(row + 16, &w, 4);
  if (row_name_is_null(i)) nulls |= 1u << 2;
  else {
    char tmp[64]; const int l = row_value_name(i, tmp);
    memcpy(row + pos, tmp, (size_t)l);
    rw_put64(row + 24, ((uint64_t)pos << 32) | (uint32_t)l);
    pos += (l + 7) / 8 * 8;
  }
  const int el = row_emb_len(i);                                    /* UnsafeArrayData: numElements, null bits, the floats */
  const int32_t bits = (el + 63) / 64 * 8, alen = 8 + bits + (4 * el + 7) / 8 * 8;
  rw_put64(row + pos, (uint64_t)el);
  for (int k = 0; k < el; ++k) { float v = row_value_emb(i, k); memcpy(row + pos + 8 + bits + 4 * k, &v, 4); }
  rw_put64(row + 32, ((uint64_t)pos << 32) | (uint32_t)alen);
  pos += alen;
  rw_put64(row, nulls);
  return pos;
}
static void rw_open(RowWriter* W, const char* path, int64_t flush_rows) {
  memset(W, 0, sizeof *W);
  OK(tfr_schema_create(FIELDS, N_FIELDS, TFR_RT_EXAMPLE, &W->schema));
  OK(tfr_encoder_create(W->schema, 0, 0, &W->enc));
  W->out = fopen(path, "wb");
  CHECK(W->out, "cannot create %s", path);
  W->slots = tfr_encoder_num_row_slots();
  CHECK(W->slots >= 2 && W->slots <= 8, "row slots %d", W->slots);
  W->flush_rows = flush_rows;
  for (int k = 0; k < W->slots; ++k) {                              /* sized once: growing a slot would drop its rows */
    void* p = NULL; size_t cap = 0;
    OK(tfr_encoder_row_staging_slot(W->enc, k, (size_t)flush_rows * RW_MAX_ROW, &p, &cap));
    W->st[k] = p;
    W->offs[k] = malloc(4 * ((size_t)flush_rows + 1));
    W->offs[k][0] = 0;
  }
}
/* the slot's previous flush: wait, then writeAll its framed bytes */
static void rw_drain(RowWriter* W, int k) {
  if (!W->pending[k]) return;
  int64_t err_row = -1;
  OK(tfr_encoded_wait(W->pending[k], &err_row));
  void* host = NULL; size_t nb = 0;
  OK(tfr_encoded_result(W->pending[k], 1, &host, &nb));
  CHECK(fwrite(host, 1, nb, W->out) == nb, "short write");
  tfr_encoded_release(W->pending[k]);
  W->pending[k] = NULL;
}
static void rw_flush(RowWriter* W) {
  if (!W->n) return;
  OK(tfr_encode_rows_submit(W->enc, W->st[W->k], W->offs[W->k], W->n, 0, &W->pending[W->k]));
  W->rows_written += W->n; W->flushes++; W->n = 0;
  W->k = (W->k + 1) % W->slots;
  rw_drain(W, W->k);                                                /* before slot k is refilled */
}
static void rw_write(RowWriter* W, int64_t i) {
  CHECK(!W->closed, "write after close");
  int32_t* o = W->offs[W->k];
  o[W->n + 1] = o[W->n] + unsafe_row_of(i, W->st[W->k] + o[W->n]);
  if (++W->n == W->flush_rows) rw_flush(W);
}
static void rw_close(RowWriter* W) {
  CHECK(!W->closed, "OutputWriter.close called twice");
  rw_flush(W);
  for (int j = 0; j < W->slots; ++j) rw_drain(W, (W->k + j) % W->slots);   /* the oldest first */
  fclose(W->out);
  int64_t st[5] = {0};
  OK(tfr_encoder_get_stats(W->enc, st, 5));
  printf("rowwrite stats: submits=%lld pipelined=%lld redone=%lld topups=%lld\n", (long long)st[0], (long long)st[1], (long long)st[2], (long long)st[3]);
  tfr_encoder_destroy(W->enc); tfr_schema_destroy(W->schema);
  for (int k = 0; k < W->slots; ++k) free(W->offs[k]);
  W->closed = 1;
}

static int cmd_rowwrite(const char* dir, int64_t n, int64_t flush_rows) {
  char path[1024];
  snprintf(path, sizeof path, "%s/part-00000.tfrecord", dir);
  CHECK(flush_rows > 0, "FLUSH must be positive");
  RowWriter W;
  rw_open(&W, path, flush_rows);
  for (int64_t i = 0; i < n; ++i) rw_write(&W, i);
  rw_close(&W);
  CHECK(W.rows_written == n, "rows written %lld != %lld", (long long)W.rows_written, (long long)n);
  printf("rowwrite ok: rows=%lld flushes=%lld\n", (long long)n, (long long)W.flushes);
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 5 && !strcmp(argv[1], "rowwrite")) return cmd_rowwrite(argv[2], atoll(argv[3]), atoll(argv[4]));
  fprintf(stderr, "usage: %s rowwrite DIR N_ROWS FLUSH_ROWS\n", argv[0]);
  return 2;
}
