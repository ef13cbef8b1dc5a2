/*
 * tfrgpu.h -- C ABI of libtfrgpu.so: the H100-native TFRecord decode/encode hot path
 * behind the spark-tfrecord DataSource API.
 *
 * Every entry point below is what a JNI (or ctypes) shim binds; there are no C++ or
 * torch types in any signature.  Each declaration cites the reference interface
 * (linkedin/spark-tfrecord @ 5bc46ee) it replaces.  Shorthand:
 *   M/ = src/main/scala/com/linkedin/spark/datasources/tfrecord/
 *
 * Conventions
 *   - every function returns int32_t: 0 (TFR_OK) or a negative TFR_E_* code;
 *     a human-readable message for the last failure on a handle is available through
 *     tfr_last_error().  No exception ever crosses this boundary.
 *   - handles are thread-confined, the library is re-entrant: one decoder/encoder per
 *     Spark task thread (M/TFRecordFileReader.scala:16-20 is called once per file per
 *     task; M/TFRecordOutputWriter.scala:12-24 is one instance per task).
 *   - the CUDA device is mandatory.  There is no CPU fallback anywhere behind this ABI:
 *     creating a decoder/encoder without a usable sm_90 device fails with TFR_E_CUDA.
 */
#ifndef TFRGPU_H_
#define TFRGPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFR_ABI_VERSION 2

/* ---- status codes (SURVEY.md section 8b "error conventions") ------------------------- */
enum {
  TFR_OK = 0,
  TFR_E_INVALID_ARG      = -1,  /* bad handle / null pointer / bad enum              */
  TFR_E_UNSUPPORTED_TYPE = -2,  /* M/TFRecordDeserializer.scala:119,123 ; M/TFRecordSerializer.scala:147,151 -> RuntimeException at construction */
  TFR_E_BAD_RECORD_TYPE  = -3,  /* M/TFRecordFileReader.scala:78-79 -> IllegalArgumentException */
  TFR_E_CUDA             = -4,  /* no device / CUDA runtime error                     */
  TFR_E_OOM              = -5,
  TFR_E_BATCH_TOO_LARGE  = -6,  /* a batch must stay below 2 GiB of framed bytes and int32 Arrow offsets */
  /* per-record data errors; the JNI shim maps them to the Java exception the
   * reference would have thrown for the same record (see INTEGRATION.md)            */
  TFR_E_CRC_LENGTH       = -10, /* tensorflow-hadoop TFRecordReader: length CRC mismatch -> IOException      */
  TFR_E_CRC_DATA         = -11, /* payload CRC mismatch -> IOException                                        */
  TFR_E_TRUNCATED        = -12, /* EOF inside a record -> IOException                                         */
  TFR_E_RECORD_TOO_LARGE = -13, /* length > Integer.MAX_VALUE -> IOException                                  */
  TFR_E_MALFORMED_PROTO  = -14, /* Example.parseFrom / SequenceExample.parseFrom (M/TFRecordFileReader.scala:73,76) -> InvalidProtocolBufferException */
  TFR_E_KIND_MISMATCH    = -15, /* require(...) M/TFRecordDeserializer.scala:178,189,201,212 -> IllegalArgumentException */
  TFR_E_EMPTY_SCALAR     = -16, /* .head on empty list M/TFRecordDeserializer.scala:75-94 -> NoSuchElementException */
  TFR_E_NULL_IN_NONNULL  = -17, /* M/TFRecordDeserializer.scala:31,56 ; M/TFRecordSerializer.scala:29-31,53-55 -> NullPointerException */
  TFR_E_BAD_NESTING      = -18, /* 2-D column fed from context / scalar column fed from feature_lists:
                                   M/TFRecordDeserializer.scala:119,142 -> RuntimeException */
  TFR_E_INDEX_MISMATCH   = -19  /* a record index that does not describe its file (RECORD INDEX below) -> IOException */
};

/* ---- schema -------------------------------------------------------------------------- */
/* element types: the Spark SQL types the reference accepts (M/TFRecordDeserializer.scala:70-124,
 * M/TFRecordSerializer.scala:68-152; README "supported data types")                       */
enum {
  TFR_T_NULL    = 0,  /* NullType: always null on read (:71-72), never written (:70)          */
  TFR_T_INT32   = 1,  /* IntegerType <- Int64List, low 32 bits (:74-75)                       */
  TFR_T_INT64   = 2,  /* LongType                                                             */
  TFR_T_FLOAT32 = 3,  /* FloatType                                                            */
  TFR_T_FLOAT64 = 4,  /* DoubleType <- FloatList widened (:83-84); written via toFloat        */
  TFR_T_DECIMAL = 5,  /* DecimalType: carried as float64 (f.toDouble, :86-87); the JVM shim wraps it in Decimal */
  TFR_T_STRING  = 6,  /* StringType <- BytesList, Java UTF-8 decode/re-encode semantics (:89-91) */
  TFR_T_BINARY  = 7,  /* BinaryType <- BytesList raw (:93-95)                                 */
  /* Generated fields: metadata of the row, never read from a record (POSITIONS below).  Decoder schemas only: at depth 0,
   * at most one of each kind, or tfr_schema_create returns TFR_E_UNSUPPORTED_TYPE naming the field; tfr_encoder_create
   * refuses a schema that has one (TFR_E_UNSUPPORTED_TYPE).  Their tfr_column reports TFR_T_INT64, depth 0, null_count 0
   * and every validity bit set, so every view of a batch (columns, host copy, Arrow, UnsafeRows) reads them as LongType. */
  TFR_T_ROW_INDEX     = 8,  /* the row's entry index in its file                                */
  TFR_T_RECORD_OFFSET = 9,  /* the file offset of the row's entry                               */
  TFR_T_VECTOR        = 10, /* Spark ML's VectorUDT, read and written as a FloatList (VECTORS below) */
  TFR_T_SPARSE_VECTOR = 11, /* Spark ML's VectorUDT, read and written as TF sparse features (SPARSE VECTORS below) */
  /* Stored as an Int64List (INT64 TYPES below); only with the schema flag TFR_S_INT64_TYPES */
  TFR_T_BOOL      = 12, /* BooleanType                                                        */
  TFR_T_INT8      = 13, /* ByteType                                                           */
  TFR_T_INT16     = 14, /* ShortType                                                          */
  TFR_T_DATE      = 15, /* DateType: days since 1970-01-01                                    */
  TFR_T_TIMESTAMP = 16  /* TimestampType: microseconds since the epoch, UTC                   */
};
/* VECTORS: TFR_T_VECTOR is org.apache.spark.ml.linalg.VectorUDT (and org.apache.spark.mllib.linalg.VectorUDT, which has the
 * same sqlType: struct<type: tinyint not null, size: int, indices: array<int not null>, values: array<double not null>>).
 *   - Schema : depth 0 only; at depth 1 or 2 (ArrayType(VectorUDT)) tfr_schema_create returns TFR_E_UNSUPPORTED_TYPE naming
 *              the field.  Decoders and encoders take it; a ByteArray schema ignores it like any data field; schema inference
 *              never produces it (a FloatList infers as ArrayType(FloatType)).
 *   - Read   : the field reads what an ArrayType(DoubleType) field of the same name and nullability reads, by every rule of
 *              the decoder (kinds, SequenceExample heads, FAILFAST / DROPMALFORMED / PERMISSIVE, TFR_F_RESYNC), as a dense
 *              vector of those values: null, the error, its row and its field exactly where that field's would be.  Its
 *              tfr_column is that field's: TFR_T_FLOAT64, depth 1, n_levels 1 (host copy and Arrow export: list<double>).
 *   - Rows   : tfr_batch_rows (and _with_partition, _async) write what UnsafeProjection makes of
 *              VectorUDT.serialize(DenseVector(values)): the slot is (offset << 32) | size of a nested UnsafeRow of 4 fields:
 *              one null word with bits 1 and 2 set, the slots type = 1 (the low byte; the other bytes zero), size = 0,
 *              indices = 0, values = (40 << 32) | bytes (offset from the nested row), then the values' UnsafeArrayData
 *              (numElements, a zero element null bitset, the doubles).  A null vector has its bit set and a zero slot.
 *   - Write, tfr_encode : the column is list<double> of the dense values (TFR_T_FLOAT64, depth 1); the output is byte-identical
 *              to the same column as ArrayType(DoubleType).
 *   - Write, tfr_encode_rows / tfr_encode_rows_submit : the struct above, encoded as ArrayType(DoubleType) encodes
 *              vector.toArray (each element through toFloat): type 1 (dense) gives `values`; type 0 (sparse) gives `size` zeros
 *              (+0.0f) with values(i) at indices(i).  A null vector is omitted, or TFR_E_NULL_IN_NONNULL in a non-nullable
 *              field.  TFR_E_INVALID_ARG (a malformed row, with the existing precedence over a null): a struct slot outside
 *              its row, misaligned or shorter than the 40-byte fixed part; a type other than 0 or 1 (MatchError in
 *              VectorUDT.deserialize); a null `values`, or a null `indices` when sparse (NullPointerException); a malformed
 *              inner array; a sparse vector with size < 0, indices and values of different lengths, or an index outside
 *              [0, size) or not strictly increasing (the requires of SparseVector's constructor).  The type and size slots
 *              are read whatever their null bits (getByte / getInt); the element null bits of indices and values are ignored
 *              and their slots' bits copied (toIntArray / toDoubleArray).  A batch whose densified values exceed the
 *              encoder's limits is TFR_E_BATCH_TOO_LARGE with no output.
 * These rules are restated from Spark's sources (VectorUDT.serialize / deserialize, SparseVector's constructor,
 * UnsafeRowWriter for a nested struct) and are NOT checked against a JVM, like the partition-row and float-bits rules.  */

/* SPARSE VECTORS: TFR_T_SPARSE_VECTOR is the same VectorUDT (the DataSource option vectorFormat=sparse; `dense`, the default,
 * is TFR_T_VECTOR), stored as the three features tf.io.SparseFeature(index_key = v_indices, value_key = v_values,
 * dtype = tf.float32, size = N) reads, plus v_size for FixedLenFeature([], tf.int64):
 *     <name>TFR_SPARSE_INDICES_SUFFIX  Int64List               ArrayType(IntegerType)  the indices of v.toSparse
 *     <name>TFR_SPARSE_VALUES_SUFFIX   FloatList               ArrayType(DoubleType)   the values of v.toSparse (toFloat)
 *     <name>TFR_SPARSE_SIZE_SUFFIX     Int64List of one value  IntegerType             v.size
 * The values feature is not named <name>: a dense-format reader of a sparse file finds <name> absent (null, or
 * TFR_E_NULL_IN_NONNULL for a non-nullable field) and never reads the non-zeros as a short dense vector; the reverse alike.
 *   - Lowering : a sparse-vector field IS those three ordinary fields; every semantic follows from theirs.  The values field
 *              takes the vector's place, name aside, and its nullability; the indices and size fields are nullable and are
 *              appended after all n_fields of the caller, in field order (indices, size of the first sparse vector, then the
 *              next's).  tfr_schema_num_fields, tfr_batch_num_columns and the columns tfr_encode takes are n_fields + 2k for k
 *              sparse vectors: columns [0, n_fields) are the caller's fields (a sparse vector's is its values, list<double>),
 *              then each sparse vector's indices (list<int32>) and size (int32).  Encoded entries follow the lowered order.
 *   - Schema : depth 0 only (ArrayType(VectorUDT) is TFR_E_UNSUPPORTED_TYPE naming the field).  Two fields whose feature keys
 *              collide (a sparse `v` next to a field `v_values`) are TFR_E_INVALID_ARG naming both.  A ByteArray schema ignores
 *              it like any data field; schema inference never produces it (a sparse file infers as its three plain fields).
 *   - Read   : the parts read by every rule of their lowered types (kinds, .head for the size, SequenceExample context and
 *              heads, FAILFAST / DROPMALFORMED / PERMISSIVE, TFR_F_RESYNC, generated fields, the large-record path).  The vector
 *              is null exactly when its values are.  An error in a part reports the vector's field index (tfr_batch_info
 *              .error_field, tfr_batch_dropped's `field`); within a record the parts come after every caller field in
 *              precedence.  The reader does not check sparse structure (sorted indices inside [0, size), equal lengths), as
 *              Spark's Parquet and ORC readers of a VectorUDT column do not: SparseVector's constructor does, in
 *              VectorUDT.deserialize.
 *   - Rows   : tfr_batch_rows (and _with_partition, _async) have the caller's n_fields fields.  A sparse vector's slot is
 *              (offset << 32) | size of the nested row UnsafeProjection makes of VectorUDT.serialize(SparseVector(size,
 *              indices, values)): one null word (bit 1: size null, bit 2: indices null), the slots type = 0 (all zero), size
 *              (the int in the low 4 bytes), indices = (40 << 32) | bytes, values = (o << 32) | bytes, then the indices'
 *              UnsafeArrayData (int32 elements) and the values' (doubles), each with a zero element null bitset.  A null size or
 *              indices has a zero slot, and the array behind it moves up.  A null vector has its bit set and a zero slot.
 *   - Write, tfr_encode_rows / tfr_encode_rows_submit : the row holds the VectorUDT struct, dense or sparse, checked by every
 *              malformed-struct clause of VECTORS (TFR_E_INVALID_ARG at the same row).  The parts are those of vector.toSparse:
 *              the entries whose double is != 0.0 (-0.0 and stored zeros dropped, NaN kept; a tiny double may still become 0.0f
 *              through toFloat), the index of each, and size.  A null vector omits all three, or is TFR_E_NULL_IN_NONNULL in a
 *              non-nullable field.  A zero vector writes an empty values and indices list and its size.  The output is
 *              bounded by the input, so no densify limit applies.
 * These rules are restated from Spark's sources (VectorUDT.serialize, Vector.toSparse, UnsafeRowWriter for a nested struct) and
 * TensorFlow's tf.io.SparseFeature, and are NOT checked against a JVM or TensorFlow.  */
#define TFR_SPARSE_INDICES_SUFFIX "_indices"
#define TFR_SPARSE_VALUES_SUFFIX  "_values"
#define TFR_SPARSE_SIZE_SUFFIX    "_size"

/* RAGGED: the DataSource option nestedArrayFormat=ragged (`featureList`, the default, is today's behaviour; any other value is
 * IllegalArgumentException before any work) is tfr_schema_create_ex with TFR_S_RAGGED.  In an Example schema a field
 * x: ArrayType(ArrayType(T)) (depth 2, T any element type valid at depth 2) is stored as the two plain features
 * tf.io.RaggedFeature(dtype, value_key = x_values, partitions = [RaggedFeature.RowLengths(x_row_lengths)]) reads:
 *     <name>TFR_RAGGED_VALUES_SUFFIX       depth-1 list of T   the inner lists' elements, flattened in order
 *     <name>TFR_RAGGED_ROW_LENGTHS_SUFFIX  Int64List           the inner lists' lengths
 *   - Lowering : the values part takes x's place and nullability; the lengths part is nullable and appended after every caller
 *              field and every sparse-vector part, in field order.  Encoded entries follow the lowered order.  To the caller x is
 *              ONE column, laid out like a SequenceExample FeatureList column of T (depth 2, n_levels 2, or 3 for String /
 *              Binary): tfr_schema_num_fields, tfr_batch_num_columns and the columns tfr_encode takes do not count the lengths
 *              parts.  Feature keys that collide (ragged `x` next to a field `x_values`) are TFR_E_INVALID_ARG naming both.  A
 *              record feature named `x` is not looked up; it is validated like any feature outside the schema.
 *   - Schema : TFR_S_RAGGED with TFR_RT_SEQUENCE_EXAMPLE is TFR_E_INVALID_ARG (its 2-D columns are FeatureLists); a ByteArray
 *              schema ignores the flag.  Schema inference never produces it (a ragged file infers as its two plain fields).
 *   - Read   : both parts read by every rule of their lowered types (kinds, FAILFAST / DROPMALFORMED / PERMISSIVE, TFR_F_RESYNC,
 *              generated fields).  Then per record: both absent -> x is null (TFR_E_NULL_IN_NONNULL when x is non-nullable,
 *              through the values part); exactly one present -> TFR_E_BAD_NESTING at x's field index; both present -> every
 *              length >= 0 and their sum equal to the number of values, else TFR_E_BAD_NESTING at x.  Within a record the
 *              caller fields' errors come first (x's values part included), then the sparse-vector parts', then the lengths
 *              parts' own errors (reported at x), and the consistency check last.
 *   - Write  : a null x omits both features (TFR_E_NULL_IN_NONNULL when non-nullable); otherwise the flattened elements, each
 *              through the element type's existing conversion and null-element rule, and the inner sizes.  [] writes two empty
 *              lists; [[]] an empty values list and the lengths [0].  A null inner array (UnsafeRow input) is
 *              TFR_E_NULL_IN_NONNULL at its row.  tfr_encode, tfr_encode_rows and tfr_encode_rows_submit alike; a tfr_encode
 *              column whose offsets are not a depth-2 column (decreasing, negative, or past its n_offsets[1] - 1 inner
 *              lists) is TFR_E_INVALID_ARG at the first such row.
 *   - Paths  : every decode path takes ragged fields (tile, large-record, general, pipelined submit).  The tile and large-record
 *              kernels do not check the parts; a batch whose parts disagree goes to the general path, which reports it.
 *   - Row splits : the DataSource option raggedPartition=rowSplits (`rowLengths`, the default, is the layout above; any other
 *              value, or rowSplits without nestedArrayFormat=ragged, is IllegalArgumentException before any work) is
 *              TFR_S_RAGGED | TFR_S_RAGGED_ROW_SPLITS (TFR_S_RAGGED_ROW_SPLITS alone is TFR_E_INVALID_ARG).  The partition is
 *              RaggedFeature.RowSplits(x_row_splits), the encoding tf.RaggedTensor holds (rt.row_splits):
 *     <name>TFR_RAGGED_ROW_SPLITS_SUFFIX   Int64List           k + 1 entries 0, l0, l0+l1, .., the sum, for k inner lists
 *              in place of the lengths part, with its place in the lowering, its nullability and its key-collision rule.
 *              Write: null x omits both features; [] writes an empty values list and the splits [0]; [[]] the splits [0, 0].
 *              Read, both parts present: the splits must have at least one entry (an empty list is an error here, unlike the
 *              lengths), a first entry 0, no decreasing entry and a last entry equal to the number of values, else
 *              TFR_E_BAD_NESTING at x.  Absence, precedence and every other rule are the lengths part's.  So a file written with
 *              the other partition reads as TFR_E_BAD_NESTING (x_values present, the expected partition absent): lengths are
 *              never read as splits, nor splits as lengths.
 * These rules restate TensorFlow's tf.io.RaggedFeature and RaggedTensor.from_row_splits documentation and are NOT checked against
 * TensorFlow or a JVM.                                                                                                         */
#define TFR_RAGGED_VALUES_SUFFIX      "_values"
#define TFR_RAGGED_ROW_LENGTHS_SUFFIX "_row_lengths"
#define TFR_RAGGED_ROW_SPLITS_SUFFIX  "_row_splits"
#define TFR_S_RAGGED 0x1u
#define TFR_S_RAGGED_ROW_SPLITS 0x8u

/* INT64 TYPES: the DataSource option extendedTypes=true (`false`, the default, refuses these types as before; any other value is
 * IllegalArgumentException before any work) is tfr_schema_create_ex with TFR_S_INT64_TYPES, which may be combined with
 * TFR_S_RAGGED.  Without the flag the five ids below are TFR_E_UNSUPPORTED_TYPE naming the field; a ByteArray schema ignores it.
 *     type               tfr_column value_width   written as the Int64           read from Int64 v          Arrow format
 *     TFR_T_BOOL         1 (one byte, 0 or 1)     0 or 1 (a nonzero byte is 1)   v != 0, over all 64 bits   b (bit-packed)
 *     TFR_T_INT8         1                        sign-extended                  the low 8 bits             c
 *     TFR_T_INT16        2                        sign-extended                  the low 16 bits            s
 *     TFR_T_DATE         4                        days, sign-extended            the low 32 bits            tdD
 *     TFR_T_TIMESTAMP    8                        microseconds, UTC              v                          tsu:UTC
 *   - Lowering : such a field IS a LongType field of the same name, depth (0, 1, 2) and nullability; every rule follows from that
 *              one (kinds: a FloatList or BytesList is TFR_E_KIND_MISMATCH; .head of an empty list is TFR_E_EMPTY_SCALAR; nulls,
 *              non-nullable fields, SequenceExample context and FeatureLists, ragged fields, FAILFAST / DROPMALFORMED /
 *              PERMISSIVE, TFR_F_RESYNC, generated fields, every decode path).  The file bytes are those of the LongType field
 *              holding the widened values, so a reader without the flag, or TensorFlow, reads the file as LongType.  Schema
 *              inference never produces these types: an Int64List infers as LongType.
 *   - Read   : the field is parsed as LongType; then one kernel launch per batch narrows every such column's leaf values (all
 *              but TFR_T_TIMESTAMP, whose int64 values are its own) into the batch's outputs, and writes a boolean column's
 *              bit-packed values too.  Offsets and validity are the LongType column's.  tfr_column reports the type above and
 *              its value_width; the leaf values are in the narrow type.  tfr_batch_export_arrow_host / _device hand out the
 *              format above (a boolean's values buffer is the bit-packed one, bits past the length zero).
 *   - Rows   : tfr_batch_rows (and _with_partition, _async) write what UnsafeRowWriter and UnsafeArrayData write: a scalar slot
 *              is zeroed, then holds 1 (boolean 0/1), 1, 2, 4 or 8 bytes; an array element is 1, 1, 2, 4 or 8 bytes wide, and
 *              the element region is rounded up to 8 bytes and zero-padded.
 *   - Write, tfr_encode : a column of these types has to carry its value_width (above), else TFR_E_INVALID_ARG.  One widening
 *              launch turns every such column into int64 leaf values; a nonzero boolean byte becomes 1.
 *   - Write, tfr_encode_rows / tfr_encode_rows_submit : the rows hold the layouts of Rows above; a slot or element is read
 *              at its width and widened as in the table (a boolean byte read from a row is != 0, a byte, short or date is
 *              sign-extended).  Every existing row check applies to each offset and size, with the element width of the type.
 *              A null element of an array follows LongType's rule: its slot's bits are written.
 * The UnsafeRow layouts are restated from Spark's UnsafeRowWriter and UnsafeArrayData and are NOT checked against a JVM.      */
#define TFR_S_INT64_TYPES 0x4u

/* record types: the `recordType` DataSource option (M/TFRecordFileReader.scala:22,69-80) */
enum { TFR_RT_EXAMPLE = 0, TFR_RT_SEQUENCE_EXAMPLE = 1, TFR_RT_BYTE_ARRAY = 2 };

/* One StructField of the (required) schema.  depth 0 = scalar, 1 = ArrayType(elem),
 * 2 = ArrayType(ArrayType(elem)) (SequenceExample feature_lists only).                    */
typedef struct tfr_field {
  const char* name;      /* UTF-8 bytes, not necessarily NUL terminated */
  int32_t     name_len;
  int32_t     elem_type; /* TFR_T_*  */
  int32_t     depth;     /* 0, 1, 2 (TFR_T_VECTOR, TFR_T_SPARSE_VECTOR: 0) */
  int32_t     nullable;  /* StructField.nullable */
} tfr_field;

typedef struct tfr_schema  tfr_schema;
typedef struct tfr_decoder tfr_decoder;
typedef struct tfr_encoder tfr_encoder;
typedef struct tfr_batch   tfr_batch;

int32_t tfr_abi_version(void);
/* message text for a status code (static storage) */
const char* tfr_status_string(int32_t status);
/* last error text recorded on this thread by a failing call (create-time errors) */
const char* tfr_last_error(void);

/* Replaces `new TFRecordDeserializer(schema)` (M/TFRecordFileReader.scala:44) and
 * `new TFRecordSerializer(dataSchema)` (M/TFRecordOutputWriter.scala:24): validates the types
 * up front the way TFRecordSerializer's constructor does (M/TFRecordSerializer.scala:14).
 * TFR_RT_BYTE_ARRAY: the one field `byteArray`, then the generated fields of `fields` in their order; the other fields of
 * `fields` are ignored.                                                                                              */
int32_t tfr_schema_create(const tfr_field* fields, int32_t n_fields, int32_t record_type,
                          tfr_schema** out);
/* tfr_schema_create with schema flags: TFR_S_RAGGED and TFR_S_RAGGED_ROW_SPLITS (RAGGED above), TFR_S_INT64_TYPES (INT64 TYPES above); any other bit is TFR_E_INVALID_ARG.  tfr_schema_create is
 * this call with flags 0.                                                                                              */
int32_t tfr_schema_create_ex(const tfr_field* fields, int32_t n_fields, int32_t record_type, uint32_t schema_flags,
                             tfr_schema** out);
void    tfr_schema_destroy(tfr_schema*);
int32_t tfr_schema_num_fields(const tfr_schema*);   /* lowered: n_fields + 2 per sparse vector (SPARSE VECTORS); ragged fields add none */

/* ---- decode: replaces the body of the buildReader closure ---------------------------- */
/* flags */
#define TFR_F_VERIFY_CRC   0x1u  /* tensorflow-hadoop's CRC check (on by default there)   */
/* Spark's mode=DROPMALFORMED: a record that fails is dropped and decoding goes on (the default, FAILFAST, stops the block
 * at it).  Record errors are TFR_E_CRC_DATA, TFR_E_MALFORMED_PROTO, TFR_E_KIND_MISMATCH, TFR_E_EMPTY_SCALAR,
 * TFR_E_NULL_IN_NONNULL and TFR_E_BAD_NESTING: a dropped record's length CRC verified, so the next frame is known.  The
 * batch's rows, columns, null counts and UnsafeRows are those of the block with the dropped frames cut out.  Framing errors
 * (TFR_E_CRC_LENGTH, TFR_E_TRUNCATED, TFR_E_RECORD_TOO_LARGE) still end the block, as without the flag: without
 * TFR_F_RESYNC the frame chain is lost there.  tfr_batch_info in drop mode: n_rows = the rows delivered; n_records = the frames in the consumed bytes,
 * dropped ones included; consumed_bytes = what tfr_batch_consumed returns; error_code / error_row / error_field are set
 * for a framing error only, and error_row is then the frame index at which framing stopped, which can exceed n_rows by the
 * records dropped before it.  tfr_batch_dropped lists the dropped records.  Without TFR_F_VERIFY_CRC no CRC is checked,
 * so nothing is dropped for one.                                                                                          */
#define TFR_F_DROP_MALFORMED 0x2u
/* Spark's mode=PERMISSIVE: a record that fails with one of the record errors above does not end the block and is not
 * dropped: it yields one row, at its own position in record order, whose data fields are all null -- non-nullable ones
 * included, as Spark reads file sources with a nullable data schema.  The row's fixed-width values are 0 and every list or
 * string column has a zero-length entry there.  With a corrupt-record column (tfr_decoder_create_permissive) that column
 * holds the record's payload (the bytes between the 12-byte header and the 4-byte data CRC, for a payload-CRC failure
 * too) on such a row and is null on every other row; a feature of that name in a record is never looked up (it is still
 * validated, like any feature outside the schema).  Framing errors still end the block.  tfr_batch_info in PERMISSIVE:
 * n_rows = every frame before the framing stop, failing ones included; n_records and consumed_bytes as without the flag;
 * error_code / error_row / error_field are set for a framing error only, and error_row then equals n_rows.
 * tfr_batch_dropped lists the records delivered as corrupt rows (the frame index is the row index).  Example and
 * SequenceExample only; with TFR_F_DROP_MALFORMED or for TFR_RT_BYTE_ARRAY the create call returns TFR_E_INVALID_ARG.  */
#define TFR_F_PERMISSIVE   0x4u
/* Resynchronise after a framing error (DROPMALFORMED and PERMISSIVE; without this flag the frame chain is lost at a framing
 * error and there is no resynchronisation).  Valid only together with TFR_F_VERIFY_CRC and one of TFR_F_DROP_MALFORMED or
 * TFR_F_PERMISSIVE; any other combination is TFR_E_INVALID_ARG, before any device work.  `end` is the size of the block and
 * H = 2^31 - 1, the largest block a decoder takes.
 *   1. Framing stops at offset o when the header at o fails its length CRC, or its length is above INT32_MAX, or -- on the
 *      final block only -- the frame at o is truncated (8..11 bytes left, or the frame runs past end).  1..7 stray bytes at
 *      EOF stay a clean end; on a non-final block a partial frame stays the ordinary carry.
 *   2. The RESYNC POINT is the smallest p > o with p + 12 <= end, the masked CRC-32C of data[p, p+8) equal to the u32 at p+8,
 *      L = u64 at p <= INT32_MAX, p + 16 + L <= end, the payload CRC verified, and p + 16 + L - o <= H.  Framing goes on at p
 *      as from a record boundary.
 *   3. The LOST REGION is [o, p); on the final block without a resync point it is [o, end) and the batch ends cleanly.
 *   4. The result does not depend on where blocks are cut.  On a non-final block a position p > o is UNDECIDED when
 *      p + 16 <= o + H and either p + 12 > end, or its header verifies and its frame ends past end but within H of o.  When
 *      an undecided position comes before any resync point the region is UNRESOLVED: the batch ends at o (consumed = o, the
 *      rows before o are delivered, nothing is reported about the region) and the caller's next block starts at o with more
 *      bytes, as in front of a large record.  A block of H bytes from o always decides; on such a block a region without a
 *      resync point within H (some 2 GiB of damage) stays unresolved, as a record larger than H would.
 *   5. A batch's ENTRIES are its frames and its lost regions, in byte order.  n_records counts entries; tfr_batch_dropped
 *      lists a region with record = its entry index, offset = o, the framing code (TFR_E_CRC_LENGTH, TFR_E_RECORD_TOO_LARGE or
 *      TFR_E_TRUNCATED) and field = -1.  DROPMALFORMED drops a region; PERMISSIVE reads it as one corrupt row at its place
 *      (entry index = row index), data fields null, its corrupt-record column holding data[o, p) as it is, header included.
 *      error_code is never a framing code under the flag.
 *   6. Record errors are unchanged: a frame whose header verifies but whose payload CRC fails is a record error and its
 *      length is trusted.  So a record cut off by a truncation and followed by a concatenated file swallows the records of
 *      that file that lie inside its claimed length; the rule resyncs after them.
 * Batches without a framing error take the ordinary paths (pipelined submits stay free of host synchronisation; the chains of
 * the frame index verify every header); a pipelined batch whose frame index stopped on a framing error is resolved through
 * the synchronous path, by tfr_batch_consumed too, since its consumed count depends on it.  tfr_decoder_get_stats counts the
 * lost regions ([11]) and their bytes ([12]); counters [9] and [10] count records only.                                  */
#define TFR_F_RESYNC       0x8u
#define TFR_F_DEFAULT      (TFR_F_VERIFY_CRC)
/* POSITIONS: the generated fields TFR_T_ROW_INDEX and TFR_T_RECORD_OFFSET (Spark's `_metadata.row_index`).  A batch's
 * ENTRIES are its frames and its lost regions (TFR_F_RESYNC) in byte order: what n_records counts and what
 * tfr_batch_dropped's `record` indexes.  Within one file:
 *   - row index     = the row's entry index in the file, counted from 0 at the file's first byte.  Every frame counts:
 *                     dropped ones, corrupt ones, and the frames of a FAILFAST block before its error.  A lost region
 *                     counts as one entry.
 *   - record offset = the file offset of the entry's first byte: the frame's 12-byte header, or `o` for a lost region.  For
 *                     a compressed file it is an offset in the decompressed stream.
 *   - Both are int64 and non-null on every delivered row, PERMISSIVE's corrupt rows included: they are metadata, not data
 *     fields, so PERMISSIVE's "every data field null" does not apply to them.
 *   - A record feature named like a generated field is never looked up (it is still validated, like any feature outside
 *     the schema), as for the corrupt-record column.
 * A block knows its position in the file from tfr_decode_at / tfr_decode_submit_at (first_entry, first_offset: the file
 * position of its first byte); a streaming reader carries them from block to block with tfr_batch_extent.  So:
 *   - FAILFAST without errors: row r of a block has row index first_entry + r;
 *   - DROPMALFORMED: row indexes rise strictly and skip exactly the dropped entries;
 *   - PERMISSIVE: a corrupt row has (row index, record offset) = (first_entry + its tfr_batch_dropped record,
 *     first_offset + its tfr_batch_dropped offset);
 *   - in every mode the values do not depend on where the blocks are cut.                                               */

/* Replaces TFRecordFileReader.readFile's setup (M/TFRecordFileReader.scala:16-44):
 * binds a device, a CUDA stream and reusable device/pinned buffers.                        */
int32_t tfr_decoder_create(const tfr_schema*, int32_t device, uint32_t flags, tfr_decoder** out);
/* A TFR_F_PERMISSIVE decoder (the flag is required) whose schema field `corrupt_field` is the corrupt-record column:
 * BinaryType, depth 0 and nullable, or TFR_E_INVALID_ARG naming the field.  corrupt_field = -1: no such column (corrupt
 * records are rows of nulls only), which is what tfr_decoder_create with TFR_F_PERMISSIVE does.  Argument errors are
 * returned before any device work.                                                                                     */
int32_t tfr_decoder_create_permissive(const tfr_schema*, int32_t device, uint32_t flags, int32_t corrupt_field,
                                      tfr_decoder** out);
void    tfr_decoder_destroy(tfr_decoder*);

/* Pinned host staging the caller fills with framed file bytes (the JVM sees it as a direct
 * ByteBuffer).  Grows on demand; the pointer stays valid until the next call that needs
 * more capacity or destroy.  A decoder has tfr_decoder_num_staging_slots() such buffers so
 * that block t+1 can be read from the file while block t is in flight (tfr_decode_submit);
 * a slot may be refilled once the batch decoded from it has been waited on.
 * tfr_decoder_staging is slot 0.                                                           */
int32_t tfr_decoder_staging(tfr_decoder*, size_t min_bytes, void** host_ptr, size_t* capacity);
int32_t tfr_decoder_staging_slot(tfr_decoder*, int32_t slot, size_t min_bytes, void** host_ptr, size_t* capacity);
int32_t tfr_decoder_num_staging_slots(void);

/* The hot path.  Replaces the per-record loop recordReader.nextKeyValue -> parseFrom ->
 * deserializeExample (M/TFRecordFileReader.scala:49-81, M/TFRecordDeserializer.scala:21-61).
 *   data/nbytes : framed TFRecord bytes (u64 len | u32 maskedcrc(len) | payload | u32 maskedcrc)
 *                 starting at a record boundary; in host memory (pageable or the pinned
 *                 staging above) or in device memory (data_on_device != 0).  Device input: any
 *                 alignment gets the single-pass tile kernels, and NO padding around the buffer is
 *                 required: 16-byte groups that cross data or data + nbytes are never bulk-copied,
 *                 and no 4-byte aligned word that holds no byte of the buffer is ever touched.
 *                 The buffer must stay valid and unchanged until the batch has been waited on.
 *   is_final    : nonzero -> a trailing partial record is TFR_E_TRUNCATED (EOF inside a
 *                 record); zero -> it is left unconsumed (see *consumed).
 * tfr_decode returns when the batch is complete and verified (*consumed is final).
 * A data error does not fail the call: rows before the first bad record are delivered and
 * the error is reported by tfr_batch_status, like the reference's iterator which yields
 * rows until the throwing record.
 *
 * tfr_decode_submit is the pipelined form: it enqueues the copy, the frame index and the decode
 * and returns without waiting.  Once a decoder has seen its first batches (record size and
 * column shapes learned) this involves no host/device synchronisation at all; the batch's
 * result, including consumed_bytes, is available after tfr_batch_wait / tfr_batch_status /
 * tfr_batch_columns / tfr_batch_to_host, which also redo -- transparently, with identical
 * results -- any batch the single-pass kernels could not vouch for.  At most
 * tfr_decoder_num_staging_slots() submitted batches are in flight per decoder; a further
 * submit first waits for the oldest one.                                                   */
int32_t tfr_decode(tfr_decoder*, const void* data, size_t nbytes, int32_t data_on_device,
                   int32_t is_final, tfr_batch** out, size_t* consumed);
int32_t tfr_decode_submit(tfr_decoder*, const void* data, size_t nbytes, int32_t data_on_device,
                          int32_t is_final, tfr_batch** out);
/* The same calls for a block whose first byte is entry `first_entry` at offset `first_offset` of its file (POSITIONS
 * above): the base of the generated fields.  tfr_decode and tfr_decode_submit are these with (0, 0).  A negative value is
 * TFR_E_INVALID_ARG, before any device work.  Every redo of the batch keeps its base.                                  */
int32_t tfr_decode_at(tfr_decoder*, const void* data, size_t nbytes, int32_t data_on_device, int32_t is_final,
                      int64_t first_entry, int64_t first_offset, tfr_batch** out, size_t* consumed);
int32_t tfr_decode_submit_at(tfr_decoder*, const void* data, size_t nbytes, int32_t data_on_device, int32_t is_final,
                             int64_t first_entry, int64_t first_offset, tfr_batch** out);

int32_t tfr_decoder_stream(tfr_decoder*, void** cuda_stream /* cudaStream_t */);

/* Measurement hooks (bench.py): with profiling enabled the decoder brackets every stage with CUDA
 * events on its own stream.  tfr_decoder_get_profile synchronises the stream and returns cumulative
 * device milliseconds per stage since profiling was enabled:
 *   ms[0] frame index (scan+check+repair+finish+emit)   ms[1] decode pass 1 (CRC + parse)
 *   ms[2] scans + summary                               ms[3] decode pass 2 (variable-width emit)
 *   ms[4] validity pack                                 ms[5] H2D of the input (host input only)
 *   ms[6] D2H of the Arrow buffers (tfr_batch_to_host[_async]) or of the rows (tfr_batch_rows)
 *   ms[7] the rows pass of tfr_batch_rows (size kernel, scan, emit kernel)
 * plus the number of kernel launches and of pass-1 launches.                                  */
#define TFR_PROFILE_STAGES 8
int32_t tfr_decoder_set_profiling(tfr_decoder*, int32_t enable);
int32_t tfr_decoder_get_profile(tfr_decoder*, double* ms /* [TFR_PROFILE_STAGES] */, int64_t* kernel_launches,
                                int64_t* pass1_launches);
/* counters since creation: [0] batches decoded, [1] submitted speculatively (no host sync), [2] of those redone after
 * the device raised a flag, [3] batches through count mode (ragged / learning), [4] through the general kernels,
 * [5] column shapes (re)learned, [6] batches re-run by the single-pass kernel's transcoding instantiation (malformed
 * UTF-8 in a string column), [7] rows passes enqueued by tfr_batch_rows_async without a host synchronisation, [8] of
 * those rebuilt through the synchronous rows path (the batch was redone, or the rows did not fit what they were
 * launched with), [9] records dropped (TFR_F_DROP_MALFORMED), [10] records delivered as corrupt rows
 * (TFR_F_PERMISSIVE), [11] lost regions and [12] the bytes in them (TFR_F_RESYNC).  A caller passing n = 8 gets the
 * first eight.  The counters before [11] keep their meaning: n <= 11 gets them all, counter [10] being PERMISSIVE's, and a
 * caller passing 10 or fewer is unaffected; n = 13 adds the two of TFR_F_RESYNC.  [13] batches decoded by the
 * large-record kernel (records too large for a shared-memory tile, csrc/large.cuh); n <= 13 is unaffected by it.       */
int32_t tfr_decoder_get_stats(tfr_decoder*, int64_t* out, int32_t n /* <= 10 */);

int32_t tfr_batch_wait(tfr_batch*);
typedef struct tfr_batch_info {
  int64_t n_rows;          /* rows delivered (records before the first error)              */
  int64_t n_records;       /* record frames found in the consumed bytes                    */
  int64_t consumed_bytes;
  int32_t error_code;      /* TFR_OK or the TFR_E_* of the first failing record            */
  int64_t error_row;       /* its 0-based record index, -1 if none                         */
  int32_t error_field;     /* schema field index for semantic errors, -1 otherwise         */
  int64_t out_bytes;       /* Arrow bytes produced (validity+offsets+values, all columns)  */
  int32_t frame_repairs;   /* chunks whose speculative boundary had to be re-chained       */
} tfr_batch_info;
int32_t tfr_batch_status(tfr_batch*, tfr_batch_info* out);
/* Bytes of the submitted block this batch consumes, available as soon as the batch's frame index has run -- before its
 * rows are decoded.  The block loop of a streaming reader (TFRecordFileReader.scala:49-61: records are read one after
 * the other, so block t+1 starts where block t's last complete record ended) calls this right after tfr_decode_submit,
 * cuts and submits the next block, and only then waits for this one's rows: the decode of block t runs under the frame
 * index of block t+1.  For a batch that later reports an error, tfr_batch_info.consumed_bytes (the bytes in front of the
 * failing record) is what counts; the reader stops there anyway.                                                     */
int32_t tfr_batch_consumed(tfr_batch*, size_t* consumed);
/* tfr_batch_consumed plus the entries in the consumed bytes (POSITIONS above), with the same wait: a streaming reader passes
 * first_entry += *entries and first_offset += *consumed to its next submit.  Under TFR_F_RESYNC a framing stop resolves the
 * batch here, as in tfr_batch_consumed.  Either output may be NULL.                                                     */
int32_t tfr_batch_extent(tfr_batch*, size_t* consumed, int64_t* entries);
/* The records a TFR_F_DROP_MALFORMED decoder dropped from this batch.  Waits for and resolves the batch like
 * tfr_batch_status, sets *n_dropped to their number and fills the first min(*n_dropped, cap) entries, in record order:
 * the frame index within the block, the frame's byte offset in the submitted buffer (a reader adds the block's file
 * offset to log where the record was), the TFR_E_* code and the schema field (-1 when none).  Any of the arrays may be
 * NULL, and all of them when cap = 0.  Without the flag *n_dropped is 0.  A TFR_F_PERMISSIVE decoder lists the records
 * it delivered as corrupt rows, in the same format; their frame index is also their row index.                        */
int32_t tfr_batch_dropped(tfr_batch*, int64_t* n_dropped, int64_t* record, int64_t* offset, int32_t* code, int32_t* field,
                          int64_t cap);
/* tfr_batch_dropped's list plus each entry's byte length in nbytes (may be NULL): 16 + L for a frame, p - o for a lost
 * region (TFR_F_RESYNC).                                                                                                  */
int32_t tfr_batch_dropped_spans(tfr_batch*, int64_t* n_dropped, int64_t* record, int64_t* offset, int64_t* nbytes, int32_t* code,
                                int32_t* field, int64_t cap);

/* One output column in Arrow layout.  n_levels offset arrays (int32, Arrow list/binary
 * offsets) from the outermost (one entry per row + 1) to the innermost, then the leaf
 * values.  Scalar fixed width: n_levels = 0.  Pointers are device pointers
 * (tfr_batch_columns) or host pointers (tfr_batch_to_host).                                */
typedef struct tfr_column {
  int32_t  elem_type;      /* TFR_T_*                                                      */
  int32_t  depth;
  int32_t  n_levels;       /* depth + (elem is STRING/BINARY ? 1 : 0)                      */
  int32_t  value_width;    /* bytes per leaf value (1 for STRING/BINARY data)              */
  int64_t  n_rows;
  int64_t  null_count;
  uint8_t* validity;       /* Arrow bitmap, LSB first, bit=1 -> valid; (n_rows+7)/8 bytes  */
  int32_t* offsets[3];
  int64_t  n_offsets[3];   /* entries in offsets[i] (= parent count + 1)                   */
  void*    values;
  int64_t  n_values;       /* leaf elements (bytes for STRING/BINARY)                      */
} tfr_column;

int32_t tfr_batch_num_columns(tfr_batch*);   /* tfr_schema_num_fields: a sparse vector adds its indices and size (SPARSE VECTORS) */
/* device-resident view (zero copy; valid until tfr_batch_release) */
int32_t tfr_batch_columns(tfr_batch*, tfr_column* out, int32_t n);
/* copies every buffer to pinned host memory owned by the batch (D2H on the decoder's
 * copy-out stream) -- the path a row-based InternalRow consumer uses.  tfr_batch_to_host_async
 * only enqueues the copy behind the batch's kernels (so that it overlaps the next batch's
 * H2D and decode); tfr_batch_to_host waits for it and returns the host view.               */
int32_t tfr_batch_to_host_async(tfr_batch*);
int32_t tfr_batch_to_host(tfr_batch*, tfr_column* out, int32_t n);
/* Arrow C Data Interface export of one column from the host copy (struct ArrowArray /
 * struct ArrowSchema from arrow/c/abi.h, passed as void* to keep this header standalone);
 * the consumer calls ->release.  Device variant fills struct ArrowDeviceArray.             */
int32_t tfr_batch_export_arrow_host(tfr_batch*, int32_t column, void* arrow_array, void* arrow_schema);
int32_t tfr_batch_export_arrow_device(tfr_batch*, int32_t column, void* arrow_device_array, void* arrow_schema);
void    tfr_batch_release(tfr_batch*);

/* ---- decode to Spark UnsafeRows ---------------------------------------------------------
 * What a row-based FileFormat reader returns is an Iterator[InternalRow] (M/DefaultSource.scala:129-135), which Spark
 * turns into UnsafeRows with an UnsafeProjection, field by field on the JVM.  tfr_batch_rows lays the batch's rows out in
 * that format on the GPU, so the JVM side only points one reused UnsafeRow at each row (INTEGRATION.md).
 *
 * The batch's rows (the n_rows rows before its first error, tfr_batch_info.n_rows) as Spark UnsafeRows, back to back:
 * row r is rows[row_offsets[r] .. row_offsets[r+1]).  to_host = 0: device memory; 1: pinned host memory.  row_offsets
 * has n_rows + 1 int64 entries, offsets[0] = 0, every entry a multiple of 8 (the rows of one batch can exceed 2 GiB even
 * though its framed bytes cannot: an empty string is 2 bytes of protobuf and 8 of row).  Owned by the batch and valid
 * until tfr_batch_release; a second call returns the same buffers (to_host = 1 after 0 adds only the copy).  Waits for
 * the batch like tfr_batch_to_host, and returns when the rows (and their copy) are complete.  An empty batch gives
 * n_rows = 0, offsets = {0}, nbytes = 0.
 *
 * Output layout (the one tfr_encode_rows reads above): what Spark's UnsafeProjection makes of the SpecificInternalRow
 * the reference's deserializer fills (M/TFRecordDeserializer.scala:21-61):
 *   - a null bitset of (nf + 63) / 64 words, one 8-byte slot per field, then the variable-length region: variable values
 *     in field order, each 8-byte aligned with zeroed padding; the row size is a multiple of 8;
 *   - a null field, and every NullType field, has its bit set and a zero slot;
 *   - IntegerType, FloatType: the low 4 bytes, the high 4 bytes zero.  LongType, DoubleType: all 8 bytes;
 *   - float and double bits are copied from the decoded columns unchanged (the decoder has already quieted sNaN when
 *     it widened a float to double): Spark 3.5's UnsafeWriter (Platform.putFloat / putDouble) normalises neither NaN
 *     nor -0.0.  This rule is restated, not checked against a JVM;
 *   - StringType, BinaryType: slot (offset << 32) | size from the row start; strings are the Java re-encoded bytes the
 *     decoder emits;
 *   - arrays: UnsafeArrayData -- numElements, an all-zero element null bitset (decode never produces a null element),
 *     the elements padded to 8 bytes (4 bytes each for int and float, 8 for long and double, 8-byte (offset << 32) | size
 *     slots from the array start for strings, binaries and the inner arrays of 2-D columns), then the array's variable
 *     region;
 *   - ByteArray records are one binary field.
 * Errors: TFR_E_INVALID_ARG (a null batch or output pointer); TFR_E_UNSUPPORTED_TYPE when the schema has a DecimalType
 * field (its UnsafeRow layout depends on the declared precision and scale, which tfr_field does not carry;
 * tfr_last_error names the field); TFR_E_BATCH_TOO_LARGE when one row would exceed INT32_MAX bytes
 * (UnsafeRow.sizeInBytes is an int); TFR_E_OOM / TFR_E_CUDA.                                                            */
int32_t tfr_batch_rows(tfr_batch*, int32_t to_host, const void** rows, const int64_t** row_offsets,
                       int64_t* n_rows, size_t* nbytes);

/* The same rows with a file's partition values appended: what Spark's FileFormat.buildReaderWithPartitionValues makes of
 * each row, UnsafeProjection (GenerateUnsafeProjection) over D ++ P of JoinedRow(dataRow, file.partitionValues), where D
 * is the decoder's schema (nd fields) and P the partition schema (np = n_part_fields fields).  tfr_batch_rows is this
 * call with np = 0, and its output is the layout above.  Row layout:
 *   - a null bitset of (nd + np + 63) / 64 words: data field i is bit i, partition field j is bit nd + j;
 *   - nd + np slots, the data fields' then the partition fields';
 *   - the data fields' variable region, laid out as above after this larger fixed region;
 *   - then the partition row's variable region, unchanged.
 * part_row is the partition values as an UnsafeRow of P alone (UnsafeProjection.create(partitionSchema) applied to
 * file.partitionValues, once per file): host memory of any alignment, part_row_bytes long, copied during the call.
 * part_var[j] = 1 when partition slot j is (offset << 32) | size: StringType, BinaryType and DecimalType with precision
 * > 18; 0 for every other type, whose slot is copied as 8 opaque bytes (Boolean, Byte, Short, Integer, Long, Float,
 * Double, Date, Timestamp, Decimal with precision <= 18).  The GPU does not interpret the partition row: it ORs its null
 * bit j into bit nd + j, copies its slots, and copies its variable region (part_row_bytes - 8 * ((np + 63) / 64 + np)
 * bytes) to the end of each row.  A flagged slot whose 8 bytes are nonzero gets its offset moved to the region's place
 * in that row; a zero slot stays zero.  That rule is exact for the rows Spark's UnsafeRowWriter writes, restated here
 * and NOT checked against a JVM (unpinned, like the float-bits rule above):
 *   - a null string or binary has its bit set and a zero slot (setNullAt);
 *   - a null decimal with precision > 18 has its bit set, slot (offset << 32) | 0 and 16 reserved zero bytes in the
 *     variable region (the generated projection calls write(i, (Decimal) null, precision, scale));
 *   - a non-null decimal with precision > 18 reserves 16 zero bytes and writes BigInteger.toByteArray() (big-endian,
 *     minimal two's complement) at their start, its slot holding that length;
 *   - a non-null value, even an empty one, has an offset of at least 8 (past the null bitset), so its slot is nonzero;
 *   - Boolean, Byte and Short zero the slot and write 1 or 2 bytes; Date is an int of days, Timestamp a long of
 *     microseconds; a decimal with precision <= 18 puts its unscaled long in the slot.
 * With nd = 0 (SELECT of partition columns only, count(*)) every row equals part_row.
 * A batch's rows are built once: a later call must pass the same partition row (the same bytes, np and flags, nonzero
 * flags counting as 1; tfr_batch_rows counts as np = 0), or it gets TFR_E_INVALID_ARG and the batch stays usable.
 * TFR_E_INVALID_ARG, checked before any work and naming the partition field where there is one: n_part_fields outside
 * 0..4096; part_row or part_var null while np > 0; part_row_bytes not a multiple of 8, smaller than the fixed region
 * 8 * ((np + 63) / 64 + np), or nonzero while np = 0; a null bit set at an index >= np; a nonzero flagged slot whose
 * offset is not 8-aligned, lies inside the fixed region, or whose offset + size exceeds part_row_bytes.  The other errors
 * are tfr_batch_rows' (a DecimalType data field; TFR_E_BATCH_TOO_LARGE counts the partition bytes).                   */
int32_t tfr_batch_rows_with_partition(tfr_batch*, int32_t to_host, const void* part_row, size_t part_row_bytes,
                                      int32_t n_part_fields, const uint8_t* part_var, const void** rows,
                                      const int64_t** row_offsets, int64_t* n_rows, size_t* nbytes);

/* ---- pipelined rows of a decoded batch ---------------------------------------------------
 * tfr_batch_rows_async enqueues, behind the batch's kernels, the rows pass tfr_batch_rows_with_partition would run with the
 * same arguments (np = 0, part_row = part_var = NULL: tfr_batch_rows), and with to_host = 1 also their copy into pinned host
 * memory owned by the batch, and returns without waiting.  It may be called right after tfr_decode_submit, before
 * tfr_batch_consumed: a streaming reader then has the rows and their copy of block k queued behind its decode while it
 * submits block k+1, and its rows call for block k finds them done.
 *   Reading      : the rows are read with tfr_batch_rows / tfr_batch_rows_with_partition, whose bytes, offsets, n_rows and
 *                  nbytes are byte-identical to what they return without the asynchronous call, for either to_host (0 after
 *                  an asynchronous call gives the device rows; 1 after an asynchronous to_host = 0 adds only the copy).
 *   Partition    : the asynchronous call counts as the build: a later call with another partition row gets
 *                  TFR_E_INVALID_ARG, and the rows already asked for stay valid.  A second asynchronous call with the same
 *                  arguments, or one after the rows were built, does nothing (except that to_host = 1 after an asynchronous
 *                  to_host = 0 enqueues the copy).
 *   Errors       : returned at once are only the argument errors tfr_batch_rows_with_partition checks before any work (a
 *                  null batch, every partition-row case listed above, a DecimalType data field as TFR_E_UNSUPPORTED_TYPE
 *                  naming the field, the batch staying usable for columns), and TFR_E_OOM / TFR_E_CUDA.  A row above
 *                  INT32_MAX bytes (TFR_E_BATCH_TOO_LARGE) is reported by the later rows call, exactly as without it.
 *   Synchronisation : a decoder learns its row sizes from the first clean batch of more than 64 rows whose rows it builds,
 *                  on either path.  Before that the asynchronous call only records the request, and the rows call builds
 *                  the rows as it would without it.  After it, every asynchronous call enqueues with no host
 *                  synchronisation, for pipelined batches and for batches decoded synchronously alike.  The rows block is
 *                  sized from the learned data-row bytes per framed byte plus head-room, plus the partition bytes of every
 *                  row the batch can hold.
 *   Redo         : rows enqueued for a batch that is later redone (its pipelined decode raised a flag), or whose device
 *                  verdict says they did not fit what they were launched with, are dropped, and the rows call rebuilds them
 *                  through the synchronous path.  The caller never sees a speculative row.
 *   Release      : tfr_batch_release of a batch with rows enqueued waits for them before its buffers go back to the
 *                  decoder, as it does for built rows.
 * tfr_decoder_get_stats counts the passes enqueued ([7]) and those rebuilt ([8]).                                        */
int32_t tfr_batch_rows_async(tfr_batch*, int32_t to_host, const void* part_row, size_t part_row_bytes,
                             int32_t n_part_fields, const uint8_t* part_var);

/* ---- encode: replaces TFRecordOutputWriter.write/close -------------------------------- */
/* Replaces the constructor M/TFRecordOutputWriter.scala:12-24.                             */
int32_t tfr_encoder_create(const tfr_schema*, int32_t device, uint32_t flags, tfr_encoder** out);
void    tfr_encoder_destroy(tfr_encoder*);

/* Replaces write(row) for a batch of rows (M/TFRecordOutputWriter.scala:26-38 ->
 * serializeExample M/TFRecordSerializer.scala:20-35 -> toByteArray -> TFRecordWriter.write):
 * columns in the tfr_column layout above (host or device pointers), n = number of schema
 * fields (tfr_schema_num_fields: a sparse vector adds its indices and size columns, SPARSE VECTORS).  Produces the framed bytes of all rows, in row order, byte-identical to what the
 * reference writer appends to its output stream.  *out_dev is device memory owned by the
 * encoder, valid until the next tfr_encode/destroy.  A null in a non-nullable column is
 * TFR_E_NULL_IN_NONNULL with *error_row set.                                               */
int32_t tfr_encode(tfr_encoder*, const tfr_column* columns, int32_t n, int32_t columns_on_device,
                   void** out_dev, size_t* out_bytes, int64_t* error_row);
/* ---- encode from Spark UnsafeRows ------------------------------------------------------
 * What OutputWriter.write(row: InternalRow) receives is an UnsafeRow (plan output and
 * FileFormatWriter's partition projection both are), so the JVM side only appends each row's
 * bytes (one Platform.copyMemory) and its offset; the GPU takes the rows apart.
 *
 * Input layout (Spark's published UnsafeRow / UnsafeArrayData format; all words little-endian):
 *   row    : null bitset of ((nf + 63) / 64) 64-bit words (bit i set = field i is null), then
 *            one 8-byte slot per field, then the variable-length region.
 *   slots  : IntegerType, FloatType: the low 4 bytes.  LongType, DoubleType: all 8 bytes.
 *            DecimalType: the 8 bytes as a signed unscaled long.  StringType, BinaryType and
 *            arrays: (offset << 32) | size, offset relative to the row start.
 *   array  : int64 numElements n; element null bitset of ((n + 63) / 64) words; the elements,
 *            padded to 8 bytes (4 bytes each for int and float, 8 for long, double and decimal;
 *            string, binary and inner-array elements are 8-byte (offset << 32) | size slots with
 *            offset relative to the array start); then the variable-length region.
 *   batch  : row r is rows[row_offsets[r] .. row_offsets[r+1]); row_offsets has n_rows + 1
 *            int32 entries, multiples of 8, non-decreasing.  rows and row_offsets are both host
 *            memory (pageable or the staging below) or both device memory (on_device != 0); any
 *            8-byte aligned rows pointer works.  A batch stays below 2 GiB.
 *
 * Semantics: the framed bytes tfr_encode produces for the same rows given as columns, plus
 *   - a null field is omitted; in a non-nullable field (NullType included): TFR_E_NULL_IN_NONNULL;
 *   - DecimalType v: FloatList value (float)v, round to nearest even (BigDecimal(v, 0).floatValue,
 *     M/TFRecordSerializer.scala:88-90,170-171);
 *   - a null element of an int, long, float or double array: the slot's bits (toXArray copies
 *     them, :103-113; Spark writes 0);
 *   - a null element of a string, binary or decimal array, or a null inner array of a 2-D
 *     column: TFR_E_NULL_IN_NONNULL (:118-135,141-142);
 *   - a malformed row (a slot or element offset/size outside its row or array, a row shorter
 *     than its fixed region, a negative or oversized numElements, a misaligned offset):
 *     TFR_E_INVALID_ARG.  No byte outside rows[row_offsets[0] .. row_offsets[n_rows]) is read.
 *   *error_row is the first failing row; a row that fails both ways is TFR_E_INVALID_ARG.
 * The result is read like tfr_encode's (*out_dev, tfr_encoder_result_host).                  */
int32_t tfr_encoder_row_staging(tfr_encoder*, size_t min_bytes, void** host_ptr, size_t* capacity);
int32_t tfr_encode_rows(tfr_encoder*, const void* rows, const int32_t* row_offsets, int64_t n_rows,
                        int32_t on_device, void** out_dev, size_t* out_bytes, int64_t* error_row);
/* copy the last encode result to host memory (pinned staging owned by the encoder) */
int32_t tfr_encoder_result_host(tfr_encoder*, void** host_ptr, size_t* nbytes);
int32_t tfr_encoder_stream(tfr_encoder*, void** cuda_stream);

/* ---- pipelined encode of UnsafeRow batches ---------------------------------------------
 * tfr_encode_rows_submit is the pipelined form of tfr_encode_rows: it enqueues the copy of the rows, the row kernels, the
 * encode and the copy of the framed bytes to pinned host memory, and returns without waiting, so that a writer task can
 * fill the next batch of rows while the GPU encodes this one.  The H2D of batch k+1, the kernels of batch k and the D2H of
 * batch k-1 run at the same time.  Each submission owns its result; a tfr_encoded handle is thread-confined like its encoder.
 *   Input        : the layout and the semantics of tfr_encode_rows, for Example, SequenceExample and ByteArray schemas.
 *                  Host input must stay unchanged until the submission has been waited on or released; device input
 *                  until it has been waited on (a batch the pipelined kernels could not vouch for is encoded again from it).
 *   Staging      : tfr_encoder_num_row_slots() pinned buffers; slot 0 is the buffer tfr_encoder_row_staging returns.
 *                  Rows staged in slot k go through pipeline lane k.  A slot may be refilled once the submission that read
 *                  it has been waited on or released.
 *   Synchronisation : once the encoder has learned its sizes, submitting rows that sit in slot staging does no host
 *                  synchronisation.  Device input keeps the one read-back of row_offsets[0] and row_offsets[n_rows] that
 *                  tfr_encode_rows does.
 *   Learning     : the first submission of an encoder runs the synchronous path before it returns.  Later ones are sized
 *                  from the last clean batch (framed bytes per input byte, largest record, longest ByteArray payload);
 *                  the device checks those figures, and tfr_encoded_wait redoes -- transparently, with identical results --
 *                  any batch they did not fit.  A redo teaches the encoder its sizes, so the submission after it is pipelined
 *                  again.  A data error (a null or a malformed row) leaves what was learned as it was.
 *   Depth        : at most tfr_encoder_num_row_slots() submissions are in flight; a further submit first waits for the
 *                  oldest one on its lane.
 *   Errors       : tfr_encode_rows_submit returns only argument errors (those of tfr_encode_rows: null pointers, misaligned
 *                  rows, n_rows >= 2^31 as TFR_E_BATCH_TOO_LARGE), TFR_E_OOM and TFR_E_CUDA.  tfr_encoded_wait returns
 *                  exactly the status, *error_row and tfr_last_error class tfr_encode_rows returns for the same rows (a
 *                  malformed row wins over a null at the same or a later row; TFR_E_BATCH_TOO_LARGE).  A failed
 *                  submission has no bytes.
 *   Results      : tfr_encoded_result: to_host = 0 the device bytes, 1 the pinned host bytes; byte-identical to
 *                  tfr_encode_rows followed by tfr_encoder_result_host.  Valid until tfr_encoded_release; the call waits
 *                  first if needed.
 *   Release      : without a wait is allowed; the submission's buffers go back to its lane when its work has run, with no
 *                  host wait.  tfr_encoded_release(NULL) does nothing.
 *   Mixing calls : tfr_encode, tfr_encode_rows, and a staging call that grows a slot, first wait for the submissions in
 *                  flight; their results stay valid.  tfr_encoder_result_host keeps returning the last synchronous call's
 *                  result.
 *   Destroy      : tfr_encoder_destroy waits for and frees everything, unreleased submissions included; using such a
 *                  handle afterwards is a caller error.
 * tfr_encoder_get_stats: counters since creation: [0] submissions, [1] enqueued without a host synchronisation, [2] of those
 * redone after the device raised a flag, [3] results whose host copy needed a top-up at wait (the batch was larger than
 * predicted, within the head-room), [4] submissions that ran the general (non-tile) emit kernel.                        */
typedef struct tfr_encoded tfr_encoded;
int32_t tfr_encoder_num_row_slots(void);
int32_t tfr_encoder_row_staging_slot(tfr_encoder*, int32_t slot, size_t min_bytes, void** host_ptr, size_t* capacity);
int32_t tfr_encode_rows_submit(tfr_encoder*, const void* rows, const int32_t* row_offsets, int64_t n_rows,
                               int32_t on_device, tfr_encoded** out);
int32_t tfr_encoded_wait(tfr_encoded*, int64_t* error_row);
int32_t tfr_encoded_result(tfr_encoded*, int32_t to_host, void** ptr, size_t* nbytes);
void    tfr_encoded_release(tfr_encoded*);
int32_t tfr_encoder_get_stats(tfr_encoder*, int64_t* out, int32_t n /* <= 8 */);

/* ---- schema inference (SURVEY.md 8f.1; M/TensorFlowInferSchema.scala:35-58) ------------ */
/* lattice codes of M/TensorFlowInferSchema.scala:194-207; merge = max, 0 = identity     */
enum { TFR_INF_NULL = 0, TFR_INF_LONG = 1, TFR_INF_FLOAT = 2, TFR_INF_STRING = 3,
       TFR_INF_ARR_LONG = 4, TFR_INF_ARR_FLOAT = 5, TFR_INF_ARR_STRING = 6,
       TFR_INF_ARR2_LONG = 7, TFR_INF_ARR2_FLOAT = 8, TFR_INF_ARR2_STRING = 9,
       TFR_INF_ARR2_NULL = 10 /* ArrayType(ArrayType(null)): a FeatureList whose steps are all empty (:102-107) */ };
typedef struct tfr_infer tfr_infer;
/* FAILFAST, the reference's inference: the first failing record fails the update call.  Same as
 * tfr_infer_create_mode(record_type, device, 0, NULL, 0, out).                                            */
int32_t tfr_infer_create(int32_t record_type, int32_t device, tfr_infer** out);
/* Inference in one of the decoder's parse modes.  flags: 0 or TFR_F_VERIFY_CRC (FAILFAST; inference always verifies
 * the data CRC), TFR_F_DROP_MALFORMED or TFR_F_PERMISSIVE (either with TFR_F_VERIFY_CRC).  In the two tolerant modes a
 * record error -- TFR_E_CRC_DATA, TFR_E_MALFORMED_PROTO, TFR_E_KIND_MISMATCH (kind not set), TFR_E_EMPTY_SCALAR (a
 * FeatureList without steps), judged as FAILFAST judges them -- skips the record, which contributes nothing: none of its
 * names, no code, no ArrayType(ArrayType(null)) flag.  A record that does not fail contributes what it does in FAILFAST.
 * Framing errors (TFR_E_CRC_LENGTH, TFR_E_TRUNCATED, TFR_E_RECORD_TOO_LARGE) still fail the call after the names of the
 * records before the stop are merged, unless TFR_F_RESYNC is set (with the rules of the decoder's flag): a lost region is
 * skipped, listed by tfr_infer_skipped with its entry index, offset and framing code, and *consumed follows the same rule.  Limits of the device tables (more than 1,024 entries in one map, more than 65,536
 * names, a name of 16 MiB or more) still fail the call with TFR_E_BATCH_TOO_LARGE, unless the record over a limit fails
 * its CRC or its parse: then it is skipped.  The ArrayType(ArrayType(null)) conflict of tfr_infer_result is judged over
 * the kept records.  PERMISSIVE takes the corrupt-record column's name (corrupt_name_len bytes, 1 .. 2^24 - 1): an
 * entry of that key, in features / context or in feature_lists, is parsed but never merged, and its value errors do not
 * fail the record, as the decoder never looks that name up; in DROPMALFORMED it is an ordinary name.  TFR_E_INVALID_ARG,
 * before any device work, for both mode flags, TFR_F_RESYNC without a tolerant mode or without TFR_F_VERIFY_CRC, unknown flag bits, a name without TFR_F_PERMISSIVE, or PERMISSIVE without
 * a name or with a length out of range; TFR_RT_BYTE_ARRAY is TFR_E_BAD_RECORD_TYPE as for tfr_infer_create.          */
int32_t tfr_infer_create_mode(int32_t record_type, int32_t device, uint32_t flags,
                              const char* corrupt_name, int32_t corrupt_name_len, tfr_infer** out);
/* accumulate one block of framed bytes (seqOp of rdd.aggregate, :40,43).  tfr_infer_update takes a whole
 * file (a trailing partial record is TFR_E_TRUNCATED); tfr_infer_update_block streams a file of any size in
 * blocks below 2 GiB with the tfr_decode contract (is_final / *consumed).                                  */
int32_t tfr_infer_update(tfr_infer*, const void* data, size_t nbytes, int32_t data_on_device);
int32_t tfr_infer_update_block(tfr_infer*, const void* data, size_t nbytes, int32_t data_on_device,
                               int32_t is_final, size_t* consumed);
/* The records the last update call skipped (tolerant modes), in the shape of tfr_batch_dropped: *n_skipped is their
 * number and the first min(*n_skipped, cap) entries are filled in record order with the frame index within the
 * submitted block, the frame's byte offset in the submitted buffer and the TFR_E_* code (the field is always -1, so
 * there is no field array).  The arrays may be NULL when cap = 0.  After a call that failed with a framing error the list
 * holds the records skipped before the stop; after any other failing call, and always in FAILFAST, it is empty.       */
int32_t tfr_infer_skipped(tfr_infer*, int64_t* n_skipped, int64_t* record, int64_t* offset,
                          int32_t* code, int64_t cap);
/* number of distinct feature names seen so far, then the (name, code) pairs; names are
 * returned sorted bytewise so that ranks can merge them deterministically               */
int32_t tfr_infer_result(tfr_infer*, int32_t* n_names);
int32_t tfr_infer_name(tfr_infer*, int32_t i, const char** name, int32_t* name_len, int32_t* code);
void    tfr_infer_destroy(tfr_infer*);

/* ---- record index: split large files across tasks ----------------------------------------
 * RECORD INDEX: a sidecar that lets a reader start at a record boundary anywhere in an uncompressed TFRecord file and know
 * the entry number there, so a file can be read in splits (the DataSource option recordIndex=true).  A scan for the next
 * boundary is not safe: a payload can hold a complete, CRC-valid frame.  For data file dir/name the index is
 * dir/_name.tfrindex (Spark's file listing skips names that start with `_`; restated from Spark's sources, not checked
 * against a JVM).  All fields are little-endian:
 *   - a 32-byte header: the magic TFR_INDEX_MAGIC (8 bytes), u64 data_bytes (the data file's size), u64 n_entries (its
 *     frames) and u64 stride (a power of two, at least 16);
 *   - then K = ceil(data_bytes / stride) checkpoints of 16 bytes (K = 0 for an empty file).  Checkpoint k is (u64 offset,
 *     u64 entry) of the first frame whose header offset is >= k * stride; when there is no such frame it is
 *     (data_bytes, n_entries).
 * Building.  tfr_index_update streams a file in blocks with the tfr_infer_update_block contract (is_final, *consumed, a
 * partial frame of a non-final block carried into the next one; blocks below 2 GiB).  Each block runs the frame index
 * (frame.cuh, every length CRC verified), then index_checkpoint_kernel (index.cuh): one thread per frame, frame i writing the
 * slots k with o[i-1] < k * stride <= o[i].  A framing error (TFR_E_CRC_LENGTH, TFR_E_TRUNCATED, TFR_E_RECORD_TOO_LARGE) fails
 * the call with its file offset in tfr_last_error, and every later update and result call returns it: a damaged file gets
 * no index.  Payload CRCs and protobuf validity are not checked: those are record errors, which a reader's mode handles.
 * tfr_index_result returns the index bytes (owned by the handle, valid until destroy) once the final block is in.
 * Seeking.  tfr_index_seek takes bytes that start at a frame boundary (a checkpoint: entry base_entry at file offset
 * base_offset) and returns the first frame whose header offset is >= target, and its entry number:
 *   - target <= base_offset: the base itself, with no device work;
 *   - otherwise the frames are walked with the frame index, their length CRCs verified.  The bytes must reach target + 12
 *     or the end of the file (TFR_E_INVALID_ARG when they end more than one header before target): at most stride bytes
 *     plus one header from the checkpoint of floor(target / stride);
 *   - when the frame in front of target runs past the bytes given, its end is computed from its verified header;
 *   - when the bytes end (0..7 bytes after the last frame, as at a clean end of file) before target, the result is the end
 *     of the bytes and the frames before it: the index's (data_bytes, n_entries) when the bytes reach the file's end;
 *   - a length CRC that fails, a length above 2^31 - 1, a cut-off header or a frame that ends before target although the
 *     bytes end inside it is TFR_E_INDEX_MISMATCH, with the file offset in tfr_last_error.
 * A reader of the split [s, e) delivers exactly the frames whose header offset o has s <= o < e: it seeks s and e (e >=
 * data_bytes is the end of the file) and reads [offset(s), offset(e)) with tfr_decode_submit_at(entry(s), offset(s)), its last
 * block final.  When the split is read to its end with a different number of entries than entry(e) - entry(s), it fails with
 * TFR_E_INDEX_MISMATCH before any row of it is handed out.  Compressed files and TFR_F_RESYNC reads are not split.        */
#define TFR_INDEX_MAGIC            "TFRIDX01"
#define TFR_INDEX_HEADER_BYTES     32
#define TFR_INDEX_CHECKPOINT_BYTES 16
#define TFR_INDEX_MIN_STRIDE       16ull
#define TFR_INDEX_MAX_STRIDE       (1ull << 30)
typedef struct tfr_indexer tfr_indexer;
/* stride: a power of two from TFR_INDEX_MIN_STRIDE to TFR_INDEX_MAX_STRIDE, or TFR_E_INVALID_ARG before any device work */
int32_t tfr_indexer_create(int32_t device, uint64_t stride, tfr_indexer** out);
int32_t tfr_index_update(tfr_indexer*, const void* data, size_t nbytes, int32_t on_device, int32_t is_final, size_t* consumed);
int32_t tfr_index_result(tfr_indexer*, const void** bytes, size_t* nbytes);
int32_t tfr_index_seek(tfr_indexer*, const void* data, size_t nbytes, int32_t on_device, int64_t base_entry, int64_t base_offset,
                       int64_t target, int64_t* entry, int64_t* offset);
void    tfr_indexer_destroy(tfr_indexer*);

#ifdef __cplusplus
}
#endif
#endif /* TFRGPU_H_ */
