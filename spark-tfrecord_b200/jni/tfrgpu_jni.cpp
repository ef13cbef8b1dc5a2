// tfrgpu_jni.cpp -- JNI shim a spark-tfrecord maintainer adds next to the Scala sources.
// SOURCE ONLY: this image has no JDK (no jni.h), so this file is not compiled by build(); it is kept
// compile-clean against the JNI specification and exercises exactly the C ABI of include/tfrgpu.h.
//
// Java side (package com.linkedin.spark.datasources.tfrecord):
//   final class TfrGpu {
//     static native long schemaCreate(String[] names, int[] elemTypes, int[] depths, boolean[] nullable, int recordType);
//     static native long schemaCreateFormat(String[] names, int[] elemTypes, int[] depths, boolean[] nullable, int recordType,
//                                           String nestedArrayFormat);   // "featureList" (schemaCreate) or "ragged": TFR_S_RAGGED
//     static native long schemaCreateOptions(String[] names, int[] elemTypes, int[] depths, boolean[] nullable, int recordType,
//                                            String nestedArrayFormat, String extendedTypes);   // + extendedTypes "true": TFR_S_INT64_TYPES
//     static native long schemaCreatePartition(String[] names, int[] elemTypes, int[] depths, boolean[] nullable, int recordType,
//                                              String nestedArrayFormat, String extendedTypes, String raggedPartition);
//                                                 // + raggedPartition "rowSplits" (with "ragged"): TFR_S_RAGGED_ROW_SPLITS
//     static native int extendedElemType(String typeName, String extendedTypes);   // DataType.typeName of boolean, byte, short,
//                                                 // date, timestamp -> TFR_T_BOOL .. TFR_T_TIMESTAMP under "true"; -1 under "false"
//                                                 // (unsupported, as in the reference); -2 another type; -3 another option value
//     static native int udtElemType(String udtClassName);   // a UserDefinedType's TFR_T_* by class name (VectorUDT: 10), -1 none
//     static native int udtElemTypeFormat(String udtClassName, String vectorFormat);   // the same under the vectorFormat option:
//                                                 // VectorUDT 10 (dense) or 11 (sparse), -1 another UDT, -2 another format
//     static native void schemaDestroy(long schema);
//     static native long decoderCreate(long schema, int device, int flags);
//     static native long decoderCreatePermissive(long schema, int device, int flags, int corruptField);   // mode=PERMISSIVE; -1: no corrupt column
//     static native void decoderDestroy(long decoder);    // TaskCompletionListener + the iterator's idempotent close (M/TFRecordFileReader.scala:36-40,52-57)
//     static native java.nio.ByteBuffer decoderStaging(long decoder, int slot, long minBytes);   // direct, pinned; slots 0..stagingSlots()-1
//     static native int stagingSlots();
//     static native long decode(long decoder, java.nio.ByteBuffer staged, long nbytes, boolean isFinal, long[] consumedOut);
//     static native long decodeSubmit(long decoder, java.nio.ByteBuffer staged, long nbytes, boolean isFinal);   // pipelined: no wait
//     static native long decodeAt(long decoder, java.nio.ByteBuffer staged, long nbytes, boolean isFinal, long firstEntry,
//                                 long firstOffset, long[] consumedOut);   // the block's place in its file: _metadata.row_index
//     static native long decodeSubmitAt(long decoder, java.nio.ByteBuffer staged, long nbytes, boolean isFinal, long firstEntry,
//                                       long firstOffset);
//     static native long[] batchExtent(long batch);   // {consumed, entries}: the next block's firstOffset / firstEntry advance
//     static native void batchToHostAsync(long batch);                                                            // D2H behind the kernels
//     static native long[] batchStatus(long batch);      // {nRows, nRecords, consumed, errorCode, errorRow, errorField}; waits for a submitted batch
//     static native java.nio.ByteBuffer[] batchColumnHost(long batch, int column, long[] meta);  // validity, offsets*, values
//     static native void batchExportArrowDevice(long batch, int column, long arrowDeviceArrayAddr, long arrowSchemaAddr);  // ColumnarBatch on the GPU (spark-rapids)
//     static native long[] batchDropped(long batch, int maxEntries);   // {nDropped, (record, offset, code, field)*}: DROPMALFORMED, PERMISSIVE
//     static native long[] batchDroppedSpans(long batch, int maxEntries);   // {nDropped, (record, offset, nbytes, code, field)*}: + lost regions (resyncFraming)
//     static native void batchThrowIfError(long batch);   // the exception the reference would throw for the first failing record
//     static native void batchRelease(long batch);
//     static native java.nio.ByteBuffer[] batchRows(long batch);   // {rows, int64 row offsets}: pinned UnsafeRows, valid until batchRelease
//     static native java.nio.ByteBuffer[] batchRowsWithPartition(long batch, java.nio.ByteBuffer partRow, int partRowBytes,
//                                                                int numPartFields, boolean[] partVar);   // + a file's partition values
//     static native void batchRowsAsync(long batch);   // enqueue batchRows' rows and their copy behind the batch's kernels, no wait
//     static native void batchRowsWithPartitionAsync(long batch, java.nio.ByteBuffer partRow, int partRowBytes, int numPartFields,
//                                                    boolean[] partVar);
//     static native long encoderCreate(long schema, int device);
//     static native void encoderDestroy(long encoder);    // OutputWriter.close (M/TFRecordOutputWriter.scala:40-43)
//     static native java.nio.ByteBuffer encode(long encoder, long[] columnStructAddrs, int n);   // framed bytes, pinned
//     static native java.nio.ByteBuffer encoderRowStaging(long encoder, long minBytes);          // direct, pinned: UnsafeRow bytes
//     static native java.nio.ByteBuffer encodeRows(long encoder, java.nio.ByteBuffer rows, java.nio.ByteBuffer offsets, int nRows);
//     static native int encoderRowSlots();                                                        // pipelined RowWriter (INTEGRATION.md)
//     static native java.nio.ByteBuffer encoderRowStagingSlot(long encoder, int slot, long minBytes);   // direct, pinned: slot k's rows
//     static native long encodeRowsSubmit(long encoder, java.nio.ByteBuffer rows, java.nio.ByteBuffer offsets, int nRows);   // -> handle
//     static native java.nio.ByteBuffer encodedWait(long encoded);   // framed bytes, pinned, valid until encodedRelease
//     static native void encodedRelease(long encoded);
//     static native long inferCreate(int recordType, int device);                                 // DefaultSource.inferSchema (M/DefaultSource.scala:31-39)
//     static native long inferUpdate(long infer, java.nio.ByteBuffer block, long nbytes, boolean isFinal);   // -> consumed bytes
//     static native Object[] inferResult(long infer);     // {String[] names (bytewise sorted), int[] lattice codes}
//     static native void inferDestroy(long infer);
//     static native long indexerCreate(int device, long stride);                                 // the record index (recordIndex=true)
//     static native long indexUpdate(long indexer, java.nio.ByteBuffer block, long deviceAddr, long nbytes, boolean isFinal);   // -> consumed
//     static native java.nio.ByteBuffer indexResult(long indexer);                                // the _name.tfrindex bytes
//     static native long[] indexSeek(long indexer, java.nio.ByteBuffer bytes, long nbytes, long baseEntry, long baseOffset, long target);
//     static native void indexerDestroy(long indexer);
//   }
#ifdef TFR_BUILD_JNI
#include <jni.h>
#include <string>
#include <vector>
#include "../../include/tfrgpu.h"

static void throw_for(JNIEnv* env, int32_t code, int64_t row) {
  const char* cls = "java/lang/RuntimeException";
  switch (code) {
    case TFR_E_CRC_LENGTH: case TFR_E_CRC_DATA: case TFR_E_TRUNCATED: case TFR_E_RECORD_TOO_LARGE: case TFR_E_INDEX_MISMATCH: cls = "java/io/IOException"; break;
    case TFR_E_MALFORMED_PROTO: cls = "com/google/protobuf/InvalidProtocolBufferException"; break;
    case TFR_E_KIND_MISMATCH: case TFR_E_BAD_RECORD_TYPE: cls = "java/lang/IllegalArgumentException"; break;
    case TFR_E_EMPTY_SCALAR: cls = "java/util/NoSuchElementException"; break;
    case TFR_E_NULL_IN_NONNULL: cls = "java/lang/NullPointerException"; break;
    case TFR_E_UNSUPPORTED_TYPE: case TFR_E_BAD_NESTING: cls = "java/lang/RuntimeException"; break;
    default: break;
  }
  std::string msg = std::string(tfr_status_string(code)) + (row >= 0 ? " (record " + std::to_string(row) + ")" : "") + ": " + tfr_last_error();
  env->ThrowNew(env->FindClass(cls), msg.c_str());
}

static jlong schema_create(JNIEnv* env, jobjectArray names, jintArray elemTypes, jintArray depths, jbooleanArray nullable,
                           jint recordType, uint32_t schema_flags) {
  jsize n = env->GetArrayLength(names);
  std::vector<std::string> keep(n);
  std::vector<tfr_field> f(n);
  jint* et = env->GetIntArrayElements(elemTypes, nullptr);
  jint* dp = env->GetIntArrayElements(depths, nullptr);
  jboolean* nl = env->GetBooleanArrayElements(nullable, nullptr);
  for (jsize i = 0; i < n; ++i) {
    jstring s = (jstring)env->GetObjectArrayElement(names, i);
    const char* u = env->GetStringUTFChars(s, nullptr);      // note: modified UTF-8; use String.getBytes(UTF_8) for non-BMP names
    keep[i] = u; env->ReleaseStringUTFChars(s, u);
    f[i] = tfr_field{keep[i].data(), (int32_t)keep[i].size(), et[i], dp[i], nl[i] ? 1 : 0};
  }
  tfr_schema* out = nullptr;
  int32_t rc = tfr_schema_create_ex(f.data(), n, recordType, schema_flags, &out);
  env->ReleaseIntArrayElements(elemTypes, et, JNI_ABORT); env->ReleaseIntArrayElements(depths, dp, JNI_ABORT);
  env->ReleaseBooleanArrayElements(nullable, nl, JNI_ABORT);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)out;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_schemaCreate(
    JNIEnv* env, jclass, jobjectArray names, jintArray elemTypes, jintArray depths, jbooleanArray nullable, jint recordType) {
  return schema_create(env, names, elemTypes, depths, nullable, recordType, 0);
}
// DefaultSource's nestedArrayFormat option (include/tfrgpu.h, RAGGED) as schema flags: "featureList" 0, "ragged" TFR_S_RAGGED;
// -1 (IllegalArgumentException) for any other value, and for ragged with recordType=SequenceExample
static int64_t nested_array_flags(const std::string& format, int32_t record_type) {
  if (format == "featureList") return 0;
  if (format == "ragged" && record_type != TFR_RT_SEQUENCE_EXAMPLE) return TFR_S_RAGGED;
  return -1;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_schemaCreateFormat(
    JNIEnv* env, jclass, jobjectArray names, jintArray elemTypes, jintArray depths, jbooleanArray nullable, jint recordType,
    jstring nestedArrayFormat) {
  const char* u = env->GetStringUTFChars(nestedArrayFormat, nullptr);
  const std::string fmt = u ? u : "";
  if (u) env->ReleaseStringUTFChars(nestedArrayFormat, u);
  const int64_t flags = nested_array_flags(fmt, recordType);
  if (flags < 0) {
    env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                  ("nestedArrayFormat " + fmt + ": featureList, or ragged for Example records").c_str());
    return 0;
  }
  return schema_create(env, names, elemTypes, depths, nullable, recordType, (uint32_t)flags);
}
// DefaultSource's extendedTypes option (include/tfrgpu.h, INT64 TYPES) as schema flags: "false" (the default) 0, "true"
// TFR_S_INT64_TYPES; -1 (IllegalArgumentException) for any other value
static int64_t extended_types_flags(const std::string& value) {
  if (value == "false") return 0;
  if (value == "true") return TFR_S_INT64_TYPES;
  return -1;
}
// The element type of a Spark field by its DataType.typeName under the extendedTypes option: boolean, byte, short, date and
// timestamp are TFR_T_BOOL .. TFR_T_TIMESTAMP with "true", -1 (unsupported, as in the reference) with "false"; -2 for any other
// type name (the glue's own mapping applies); -3 for an option value other than these, which the glue refuses before any work
static int32_t extended_elem_type(const std::string& type_name, const std::string& value) {
  const int64_t flags = extended_types_flags(value);
  if (flags < 0) return -3;
  static const struct { const char* name; int32_t t; } M[] = {
      {"boolean", TFR_T_BOOL}, {"byte", TFR_T_INT8}, {"short", TFR_T_INT16}, {"date", TFR_T_DATE}, {"timestamp", TFR_T_TIMESTAMP}};
  for (const auto& m : M)
    if (type_name == m.name) return flags ? m.t : -1;
  return -2;
}
static std::string jstring_or(JNIEnv* env, jstring js, const char* dflt) {
  const char* u = js ? env->GetStringUTFChars(js, nullptr) : nullptr;
  const std::string out = u ? u : dflt;
  if (u) env->ReleaseStringUTFChars(js, u);
  return out;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_schemaCreateOptions(
    JNIEnv* env, jclass, jobjectArray names, jintArray elemTypes, jintArray depths, jbooleanArray nullable, jint recordType,
    jstring nestedArrayFormat, jstring extendedTypes) {
  const std::string fmt = jstring_or(env, nestedArrayFormat, "featureList"), ext = jstring_or(env, extendedTypes, "false");
  const int64_t nested = nested_array_flags(fmt, recordType), wide = extended_types_flags(ext);
  if (nested < 0 || wide < 0) {
    env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                  (nested < 0 ? "nestedArrayFormat " + fmt + ": featureList, or ragged for Example records"
                              : "extendedTypes " + ext + ": the option takes true or false").c_str());
    return 0;
  }
  return schema_create(env, names, elemTypes, depths, nullable, recordType, (uint32_t)(nested | wide));
}
// DefaultSource's raggedPartition option (include/tfrgpu.h, RAGGED, Row splits) as schema flags, given nestedArrayFormat's
// (`nested`, nested_array_flags): "rowLengths" (the default) 0, "rowSplits" TFR_S_RAGGED_ROW_SPLITS when nested has TFR_S_RAGGED;
// -1 (IllegalArgumentException) for any other value, and for rowSplits without ragged
static int64_t ragged_partition_flags(const std::string& value, int64_t nested) {
  if (value == "rowLengths") return 0;
  if (value == "rowSplits" && nested >= 0 && (nested & TFR_S_RAGGED)) return TFR_S_RAGGED_ROW_SPLITS;
  return -1;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_schemaCreatePartition(
    JNIEnv* env, jclass, jobjectArray names, jintArray elemTypes, jintArray depths, jbooleanArray nullable, jint recordType,
    jstring nestedArrayFormat, jstring extendedTypes, jstring raggedPartition) {
  const std::string fmt = jstring_or(env, nestedArrayFormat, "featureList"), ext = jstring_or(env, extendedTypes, "false"),
                    part = jstring_or(env, raggedPartition, "rowLengths");
  const int64_t nested = nested_array_flags(fmt, recordType), wide = extended_types_flags(ext), split = ragged_partition_flags(part, nested);
  if (nested < 0 || wide < 0 || split < 0) {
    env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                  (nested < 0 ? "nestedArrayFormat " + fmt + ": featureList, or ragged for Example records"
                   : wide < 0 ? "extendedTypes " + ext + ": the option takes true or false"
                              : "raggedPartition " + part + ": rowLengths, or rowSplits with nestedArrayFormat=ragged").c_str());
    return 0;
  }
  return schema_create(env, names, elemTypes, depths, nullable, recordType, (uint32_t)(nested | wide | split));
}
extern "C" JNIEXPORT jint JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_extendedElemType(JNIEnv* env, jclass, jstring typeName,
                                                                                                      jstring extendedTypes) {
  return extended_elem_type(jstring_or(env, typeName, ""), jstring_or(env, extendedTypes, "false"));
}
// The element type of a UserDefinedType field, by the UDT's class name, so that the glue needs no compile-time dependency on
// spark-mllib: both VectorUDTs (same sqlType) are TFR_T_VECTOR; any other UDT is -1 (unsupported, as in the reference).
extern "C" JNIEXPORT jint JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_udtElemType(JNIEnv* env, jclass, jstring className) {
  const char* u = env->GetStringUTFChars(className, nullptr);
  const std::string name = u ? u : "";
  if (u) env->ReleaseStringUTFChars(className, u);
  return name == "org.apache.spark.ml.linalg.VectorUDT" || name == "org.apache.spark.mllib.linalg.VectorUDT" ? TFR_T_VECTOR : -1;
}
// The element type of a UserDefinedType field under the `vectorFormat` option: both VectorUDTs are TFR_T_VECTOR ("dense", the
// default) or TFR_T_SPARSE_VECTOR ("sparse", include/tfrgpu.h, SPARSE VECTORS); any other UDT is -1; a format other than these
// is -2, which the glue refuses before any work, naming the option.
static int32_t udt_elem_type(const std::string& cls, const std::string& format) {
  if (format != "dense" && format != "sparse") return -2;
  if (cls != "org.apache.spark.ml.linalg.VectorUDT" && cls != "org.apache.spark.mllib.linalg.VectorUDT") return -1;
  return format == "sparse" ? TFR_T_SPARSE_VECTOR : TFR_T_VECTOR;
}
extern "C" JNIEXPORT jint JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_udtElemTypeFormat(JNIEnv* env, jclass, jstring className,
                                                                                                       jstring vectorFormat) {
  std::string s[2];
  jstring js[2] = {className, vectorFormat};
  for (int i = 0; i < 2; ++i) {
    const char* u = js[i] ? env->GetStringUTFChars(js[i], nullptr) : nullptr;
    s[i] = u ? u : (i ? "dense" : "");
    if (u) env->ReleaseStringUTFChars(js[i], u);
  }
  return udt_elem_type(s[0], s[1]);
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decoderCreate(JNIEnv* env, jclass, jlong schema, jint device, jint flags) {
  tfr_decoder* d = nullptr;
  int32_t rc = tfr_decoder_create((const tfr_schema*)schema, device, (uint32_t)flags, &d);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)d;
}
// mode=PERMISSIVE (flags hold TFR_F_PERMISSIVE): corruptField is the corrupt-record column's index in the required schema,
// -1 when a projection pruned it (failing records are then rows of nulls only)
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decoderCreatePermissive(JNIEnv* env, jclass, jlong schema, jint device,
                                                                                                           jint flags, jint corruptField) {
  tfr_decoder* d = nullptr;
  int32_t rc = tfr_decoder_create_permissive((const tfr_schema*)schema, device, (uint32_t)flags, corruptField, &d);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)d;
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_schemaDestroy(JNIEnv*, jclass, jlong schema) { tfr_schema_destroy((tfr_schema*)schema); }
// Safe while batches are still alive (they hold a reference on the decoder) and safe to call from the task-completion
// listener after the iterator already closed: the Scala side nulls its handle, a 0 handle is a no-op here.
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decoderDestroy(JNIEnv*, jclass, jlong dec) { if (dec) tfr_decoder_destroy((tfr_decoder*)dec); }
extern "C" JNIEXPORT jint JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_stagingSlots(JNIEnv*, jclass) { return tfr_decoder_num_staging_slots(); }
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decoderStaging(JNIEnv* env, jclass, jlong dec, jint slot, jlong minBytes) {
  void* p = nullptr; size_t cap = 0;
  int32_t rc = tfr_decoder_staging_slot((tfr_decoder*)dec, slot, (size_t)minBytes, &p, &cap);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(p, (jlong)cap);           // the InputStream is read straight into pinned memory
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decode(
    JNIEnv* env, jclass, jlong dec, jobject staged, jlong nbytes, jboolean isFinal, jlongArray consumedOut) {
  void* p = env->GetDirectBufferAddress(staged);
  tfr_batch* b = nullptr; size_t used = 0;
  int32_t rc = tfr_decode((tfr_decoder*)dec, p, (size_t)nbytes, 0, isFinal ? 1 : 0, &b, &used);
  if (rc) { throw_for(env, rc, -1); return 0; }
  jlong u = (jlong)used; env->SetLongArrayRegion(consumedOut, 0, 1, &u);
  return (jlong)b;
}
// pipelined form: block t+1 is read from the InputStream into another staging slot while block t is in flight
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decodeSubmit(
    JNIEnv* env, jclass, jlong dec, jobject staged, jlong nbytes, jboolean isFinal) {
  void* p = env->GetDirectBufferAddress(staged);
  tfr_batch* b = nullptr;
  int32_t rc = tfr_decode_submit((tfr_decoder*)dec, p, (size_t)nbytes, 0, isFinal ? 1 : 0, &b);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)b;
}
// the same two calls for a block at (firstEntry, firstOffset) of its file: the base of the generated metadata columns
// (_tmp_metadata_row_index, _tmp_metadata_record_offset, lowered to TFR_T_ROW_INDEX / TFR_T_RECORD_OFFSET by schemaCreate)
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decodeAt(
    JNIEnv* env, jclass, jlong dec, jobject staged, jlong nbytes, jboolean isFinal, jlong firstEntry, jlong firstOffset, jlongArray consumedOut) {
  void* p = env->GetDirectBufferAddress(staged);
  tfr_batch* b = nullptr; size_t used = 0;
  int32_t rc = tfr_decode_at((tfr_decoder*)dec, p, (size_t)nbytes, 0, isFinal ? 1 : 0, (int64_t)firstEntry, (int64_t)firstOffset, &b, &used);
  if (rc) { throw_for(env, rc, -1); return 0; }
  jlong u = (jlong)used; env->SetLongArrayRegion(consumedOut, 0, 1, &u);
  return (jlong)b;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decodeSubmitAt(
    JNIEnv* env, jclass, jlong dec, jobject staged, jlong nbytes, jboolean isFinal, jlong firstEntry, jlong firstOffset) {
  void* p = env->GetDirectBufferAddress(staged);
  tfr_batch* b = nullptr;
  int32_t rc = tfr_decode_submit_at((tfr_decoder*)dec, p, (size_t)nbytes, 0, isFinal ? 1 : 0, (int64_t)firstEntry, (int64_t)firstOffset, &b);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)b;
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchToHostAsync(JNIEnv* env, jclass, jlong batch) {
  int32_t rc = tfr_batch_to_host_async((tfr_batch*)batch);
  if (rc) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc, -1); }
}
// where the block after this one starts: known after the batch's frame index, before its rows (the reader submits the next block first)
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchConsumed(JNIEnv* env, jclass, jlong batch) {
  size_t used = 0;
  int32_t rc = tfr_batch_consumed((tfr_batch*)batch, &used);
  if (rc) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc, -1); return 0; }
  return (jlong)used;
}
// batchConsumed plus the entries in the consumed bytes, with the same wait: {consumed, entries}
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchExtent(JNIEnv* env, jclass, jlong batch) {
  size_t used = 0; int64_t entries = 0;
  int32_t rc = tfr_batch_extent((tfr_batch*)batch, &used, &entries);
  if (rc) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc, -1); return nullptr; }
  jlong v[2] = {(jlong)used, (jlong)entries};
  jlongArray out = env->NewLongArray(2);
  env->SetLongArrayRegion(out, 0, 2, v);
  return out;
}
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchStatus(JNIEnv* env, jclass, jlong batch) {
  tfr_batch_info i{};
  int32_t rc0 = tfr_batch_status((tfr_batch*)batch, &i);
  if (rc0) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc0, -1); return nullptr; }   // a CUDA failure: the batch is gone, the task fails
  jlong v[6] = {i.n_rows, i.n_records, i.consumed_bytes, i.error_code, i.error_row, i.error_field};
  jlongArray a = env->NewLongArray(6); env->SetLongArrayRegion(a, 0, 6, v);
  return a;
}
// mode=DROPMALFORMED (decoder flag TFR_F_DROP_MALFORMED): {nDropped, then per dropped record up to maxEntries of them
// record, offset, code, field}.  The reader logs the count and the first record's file offset (block offset + offset) once
// per block; it waits for a submitted batch like batchStatus.
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchDropped(JNIEnv* env, jclass, jlong batch, jint maxEntries) {
  int64_t n = 0;
  int32_t rc = tfr_batch_dropped((tfr_batch*)batch, &n, nullptr, nullptr, nullptr, nullptr, 0);
  if (rc) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc, -1); return nullptr; }
  const int64_t k = maxEntries < 0 ? 0 : (n < maxEntries ? n : (int64_t)maxEntries);
  std::vector<int64_t> rec(k), off(k);
  std::vector<int32_t> code(k), field(k);
  if (k) tfr_batch_dropped((tfr_batch*)batch, &n, rec.data(), off.data(), code.data(), field.data(), k);
  std::vector<jlong> v(1 + 4 * k);
  v[0] = (jlong)n;
  for (int64_t i = 0; i < k; ++i) { v[1 + 4 * i] = rec[i]; v[2 + 4 * i] = off[i]; v[3 + 4 * i] = code[i]; v[4 + 4 * i] = field[i]; }
  jlongArray a = env->NewLongArray((jsize)v.size()); env->SetLongArrayRegion(a, 0, (jsize)v.size(), v.data());
  return a;
}
// batchDropped with each entry's byte length: 16 + L for a frame, the region's length for a lost region (decoder flag
// TFR_F_RESYNC, option resyncFraming).  The reader logs each lost region once, at block offset + offset, with its length.
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchDroppedSpans(JNIEnv* env, jclass, jlong batch, jint maxEntries) {
  int64_t n = 0;
  int32_t rc = tfr_batch_dropped_spans((tfr_batch*)batch, &n, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
  if (rc) { tfr_batch_release((tfr_batch*)batch); throw_for(env, rc, -1); return nullptr; }
  const int64_t k = maxEntries < 0 ? 0 : (n < maxEntries ? n : (int64_t)maxEntries);
  std::vector<int64_t> rec(k), off(k), nb(k);
  std::vector<int32_t> code(k), field(k);
  if (k) tfr_batch_dropped_spans((tfr_batch*)batch, &n, rec.data(), off.data(), nb.data(), code.data(), field.data(), k);
  std::vector<jlong> v(1 + 5 * k);
  v[0] = (jlong)n;
  for (int64_t i = 0; i < k; ++i) {
    v[1 + 5 * i] = rec[i]; v[2 + 5 * i] = off[i]; v[3 + 5 * i] = nb[i]; v[4 + 5 * i] = code[i]; v[5 + 5 * i] = field[i];
  }
  jlongArray a = env->NewLongArray((jsize)v.size()); env->SetLongArrayRegion(a, 0, (jsize)v.size(), v.data());
  return a;
}
// The Scala iterator calls this once per column, wraps the buffers in OnHeap/OffHeap column vectors (or an
// ArrowColumnVector over the exported ArrowArray) and, after the last delivered row, throws the exception for
// batchStatus().errorCode -- the same point in the row stream at which the reference's iterator would throw.
extern "C" JNIEXPORT jobjectArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchColumnHost(
    JNIEnv* env, jclass, jlong batch, jint column, jlongArray meta) {
  tfr_batch* b = (tfr_batch*)batch;
  int32_t n = tfr_batch_num_columns(b);
  std::vector<tfr_column> cols(n);
  int32_t rc = tfr_batch_to_host(b, cols.data(), n);
  if (rc) { tfr_batch_release(b); throw_for(env, rc, -1); return nullptr; }      // nothing of this batch is reachable any more
  const tfr_column& c = cols[column];
  jobjectArray out = env->NewObjectArray(5, env->FindClass("java/nio/ByteBuffer"), nullptr);
  env->SetObjectArrayElement(out, 0, env->NewDirectByteBuffer(c.validity, (c.n_rows + 7) / 8));
  for (int l = 0; l < c.n_levels; ++l) env->SetObjectArrayElement(out, 1 + l, env->NewDirectByteBuffer(c.offsets[l], c.n_offsets[l] * 4));
  env->SetObjectArrayElement(out, 4, env->NewDirectByteBuffer(c.values, c.n_values * (c.value_width ? c.value_width : 1)));
  jlong m[4] = {c.n_rows, c.null_count, c.n_levels, c.n_values};
  env->SetLongArrayRegion(meta, 0, 4, m);
  return out;
}
// Device-resident hand-over (supportBatch = true with GPU column vectors): fills the caller's struct ArrowDeviceArray /
// struct ArrowSchema (addresses of off-heap memory the JVM allocated); the array's release callback drops the batch reference.
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchExportArrowDevice(
    JNIEnv* env, jclass, jlong batch, jint column, jlong arrowDeviceArrayAddr, jlong arrowSchemaAddr) {
  int32_t rc = tfr_batch_export_arrow_device((tfr_batch*)batch, column, (void*)arrowDeviceArrayAddr, (void*)arrowSchemaAddr);
  if (rc) throw_for(env, rc, -1);
}
// After the last delivered row of a block the iterator calls this: it throws what the reference's next() would have thrown
// for the first failing record (and releases the batch first: the exception ends the task's use of it).
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchThrowIfError(JNIEnv* env, jclass, jlong batch) {
  tfr_batch_info i{};
  int32_t rc = tfr_batch_status((tfr_batch*)batch, &i);
  if (rc == 0 && i.error_code == 0) return;
  tfr_batch_release((tfr_batch*)batch);
  throw_for(env, rc ? rc : i.error_code, rc ? -1 : i.error_row);
}
// The rows of a batch as UnsafeRows in pinned memory: the iterator points one reused UnsafeRow at row i with
// pointTo(null, address(rows) + off(i), (int)(off(i + 1) - off(i))) -- no per-field work on the JVM.
extern "C" JNIEXPORT jobjectArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchRows(JNIEnv* env, jclass, jlong batch) {
  const void* rows = nullptr; const int64_t* offs = nullptr; int64_t n = 0; size_t nb = 0;
  int32_t rc = tfr_batch_rows((tfr_batch*)batch, 1, &rows, &offs, &n, &nb);
  if (rc) { throw_for(env, rc, -1); return nullptr; }         // a decimal schema keeps the column views; the batch stays usable
  jobjectArray out = env->NewObjectArray(2, env->FindClass("java/nio/ByteBuffer"), nullptr);
  env->SetObjectArrayElement(out, 0, env->NewDirectByteBuffer(const_cast<void*>(rows), (jlong)nb));
  env->SetObjectArrayElement(out, 1, env->NewDirectByteBuffer(const_cast<int64_t*>(offs), (jlong)((n + 1) * 8)));
  return out;
}
// The same rows with the partition values of the batch's file appended (tfr_batch_rows_with_partition): partRow is a direct
// buffer holding the UnsafeRow of the partition schema alone (UnsafeProjection.create(partitionSchema)(partitionValues),
// partRowBytes = its getSizeInBytes), partVar one flag per partition field (String, Binary, Decimal precision > 18).
extern "C" JNIEXPORT jobjectArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchRowsWithPartition(
    JNIEnv* env, jclass, jlong batch, jobject partRow, jint partRowBytes, jint numPartFields, jbooleanArray partVar) {
  const void* pr = partRow ? env->GetDirectBufferAddress(partRow) : nullptr;
  std::vector<uint8_t> var;
  if (partVar) {
    jboolean* v = env->GetBooleanArrayElements(partVar, nullptr);
    var.assign(v, v + env->GetArrayLength(partVar));
    env->ReleaseBooleanArrayElements(partVar, v, JNI_ABORT);
  }
  if ((partVar && (jint)var.size() != numPartFields) || partRowBytes < 0) { throw_for(env, TFR_E_INVALID_ARG, -1); return nullptr; }
  const void* rows = nullptr; const int64_t* offs = nullptr; int64_t n = 0; size_t nb = 0;
  int32_t rc = tfr_batch_rows_with_partition((tfr_batch*)batch, 1, pr, (size_t)partRowBytes, numPartFields, partVar ? var.data() : nullptr,
                                             &rows, &offs, &n, &nb);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  jobjectArray out = env->NewObjectArray(2, env->FindClass("java/nio/ByteBuffer"), nullptr);
  env->SetObjectArrayElement(out, 0, env->NewDirectByteBuffer(const_cast<void*>(rows), (jlong)nb));
  env->SetObjectArrayElement(out, 1, env->NewDirectByteBuffer(const_cast<int64_t*>(offs), (jlong)((n + 1) * 8)));
  return out;
}
// The pipelined reader (INTEGRATION.md, submitNext): the rows batchRows / batchRowsWithPartition will return, and their pinned
// copy, enqueued right after the submit.  The batch stays usable after a failure (batchRows throws the same error again).
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchRowsAsync(JNIEnv* env, jclass, jlong batch) {
  int32_t rc = tfr_batch_rows_async((tfr_batch*)batch, 1, nullptr, 0, 0, nullptr);
  if (rc) throw_for(env, rc, -1);
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchRowsWithPartitionAsync(
    JNIEnv* env, jclass, jlong batch, jobject partRow, jint partRowBytes, jint numPartFields, jbooleanArray partVar) {
  const void* pr = partRow ? env->GetDirectBufferAddress(partRow) : nullptr;
  std::vector<uint8_t> var;
  if (partVar) {
    jboolean* v = env->GetBooleanArrayElements(partVar, nullptr);
    var.assign(v, v + env->GetArrayLength(partVar));
    env->ReleaseBooleanArrayElements(partVar, v, JNI_ABORT);
  }
  if ((partVar && (jint)var.size() != numPartFields) || partRowBytes < 0) { throw_for(env, TFR_E_INVALID_ARG, -1); return; }
  int32_t rc = tfr_batch_rows_async((tfr_batch*)batch, 1, pr, (size_t)partRowBytes, numPartFields, partVar ? var.data() : nullptr);
  if (rc) throw_for(env, rc, -1);
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchRelease(JNIEnv*, jclass, jlong batch) { if (batch) tfr_batch_release((tfr_batch*)batch); }
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encoderDestroy(JNIEnv*, jclass, jlong enc) { if (enc) tfr_encoder_destroy((tfr_encoder*)enc); }
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encoderCreate(JNIEnv* env, jclass, jlong schema, jint device) {
  tfr_encoder* e = nullptr;
  int32_t rc = tfr_encoder_create((const tfr_schema*)schema, device, 0, &e);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)e;
}
// columnStructAddrs: addresses of tfr_column structs the Scala writer filled from its row buffer (off-heap)
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encode(JNIEnv* env, jclass, jlong enc, jlongArray columnStructAddrs, jint n) {
  std::vector<tfr_column> cols(n);
  jlong* a = env->GetLongArrayElements(columnStructAddrs, nullptr);
  for (jint i = 0; i < n; ++i) cols[i] = *(const tfr_column*)a[i];
  env->ReleaseLongArrayElements(columnStructAddrs, a, JNI_ABORT);
  void* dev = nullptr; size_t nb = 0; int64_t err_row = -1;
  int32_t rc = tfr_encode((tfr_encoder*)enc, cols.data(), n, 0, &dev, &nb, &err_row);
  if (rc) { throw_for(env, rc, err_row); return nullptr; }
  void* host = nullptr;
  rc = tfr_encoder_result_host((tfr_encoder*)enc, &host, &nb);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(host, (jlong)nb);          // outputStream.write(...) of these bytes == the reference file
}
// Row path (INTEGRATION.md): write(row) copies the UnsafeRow's bytes into this pinned buffer and appends its offset
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encoderRowStaging(JNIEnv* env, jclass, jlong enc, jlong minBytes) {
  void* p = nullptr; size_t cap = 0;
  int32_t rc = tfr_encoder_row_staging((tfr_encoder*)enc, (size_t)minBytes, &p, &cap);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(p, (jlong)cap);
}
// rows: the staging buffer; offsets: a direct buffer of nRows + 1 int32 row starts.  A malformed row throws
// IllegalArgumentException, a null the reference cannot write NullPointerException, both with the row.
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encodeRows(JNIEnv* env, jclass, jlong enc, jobject rows,
                                                                                                 jobject offsets, jint nRows) {
  void* dev = nullptr; size_t nb = 0; int64_t err_row = -1;
  int32_t rc = tfr_encode_rows((tfr_encoder*)enc, env->GetDirectBufferAddress(rows), (const int32_t*)env->GetDirectBufferAddress(offsets),
                               (int64_t)nRows, 0, &dev, &nb, &err_row);
  if (rc == TFR_E_INVALID_ARG) {
    std::string msg = "malformed UnsafeRow" + (err_row >= 0 ? " (row " + std::to_string(err_row) + ")" : std::string()) + ": " + tfr_last_error();
    env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), msg.c_str());
    return nullptr;
  }
  if (rc) { throw_for(env, rc, err_row); return nullptr; }
  void* host = nullptr;
  rc = tfr_encoder_result_host((tfr_encoder*)enc, &host, &nb);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(host, (jlong)nb);
}

// ---- pipelined row path (INTEGRATION.md, RowWriter): flush k is submitted from slot k and waited for before the slot is refilled ----
static void throw_for_rows(JNIEnv* env, int32_t rc, int64_t err_row) {
  if (rc == TFR_E_INVALID_ARG) {
    std::string msg = "malformed UnsafeRow" + (err_row >= 0 ? " (row " + std::to_string(err_row) + ")" : std::string()) + ": " + tfr_last_error();
    env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), msg.c_str());
    return;
  }
  throw_for(env, rc, err_row);
}
extern "C" JNIEXPORT jint JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encoderRowSlots(JNIEnv*, jclass) { return tfr_encoder_num_row_slots(); }
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encoderRowStagingSlot(JNIEnv* env, jclass, jlong enc, jint slot,
                                                                                                            jlong minBytes) {
  void* p = nullptr; size_t cap = 0;
  int32_t rc = tfr_encoder_row_staging_slot((tfr_encoder*)enc, (int32_t)slot, (size_t)minBytes, &p, &cap);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(p, (jlong)cap);
}
// returns at once; the rows and offsets buffers must stay unchanged until encodedWait (or encodedRelease)
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encodeRowsSubmit(JNIEnv* env, jclass, jlong enc, jobject rows,
                                                                                                     jobject offsets, jint nRows) {
  tfr_encoded* h = nullptr;
  int32_t rc = tfr_encode_rows_submit((tfr_encoder*)enc, env->GetDirectBufferAddress(rows), (const int32_t*)env->GetDirectBufferAddress(offsets),
                                      (int64_t)nRows, 0, &h);
  if (rc) { throw_for_rows(env, rc, -1); return 0; }
  return (jlong)h;
}
// the framed bytes of the flush (what encodeRows returns for the same rows), or the exception encodeRows throws, with its row;
// a failed flush is released before the exception is thrown
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encodedWait(JNIEnv* env, jclass, jlong encoded) {
  tfr_encoded* h = (tfr_encoded*)encoded;
  int64_t err_row = -1;
  int32_t rc = tfr_encoded_wait(h, &err_row);
  void* host = nullptr; size_t nb = 0;
  if (!rc) rc = tfr_encoded_result(h, 1, &host, &nb);
  if (rc) { tfr_encoded_release(h); throw_for_rows(env, rc, err_row); return nullptr; }
  return env->NewDirectByteBuffer(host, (jlong)nb);
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_encodedRelease(JNIEnv*, jclass, jlong encoded) {
  if (encoded) tfr_encoded_release((tfr_encoded*)encoded);
}

// ---- schema inference: DefaultSource.inferSchema -> TensorFlowInferSchema (M/DefaultSource.scala:31-39,48-70) ----
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferCreate(JNIEnv* env, jclass, jint recordType, jint device) {
  tfr_infer* h = nullptr;
  int32_t rc = tfr_infer_create(recordType, device, &h);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)h;
}
// mode=DROPMALFORMED / PERMISSIVE (flags TFR_F_DROP_MALFORMED / TFR_F_PERMISSIVE): failing records are skipped.  corruptName:
// PERMISSIVE's columnNameOfCorruptRecord, its UTF-8 bytes in a direct ByteBuffer of corruptNameLen bytes (standard UTF-8,
// which GetStringUTFChars does not give for every name), ignored in every record; null and 0 in the other modes.
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferCreateMode(JNIEnv* env, jclass, jint recordType, jint device,
                                                                                                     jint flags, jobject corruptName, jint corruptNameLen) {
  const char* name = corruptName ? (const char*)env->GetDirectBufferAddress(corruptName) : nullptr;
  tfr_infer* h = nullptr;
  int32_t rc = tfr_infer_create_mode(recordType, device, (uint32_t)flags, name, (int32_t)corruptNameLen, &h);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)h;
}
// The records the last inferUpdate skipped: {nSkipped, then per skipped record up to maxEntries of them record, offset, code,
// field (always -1)}, the shape of batchDropped.  inferSchema logs the count and the first record's file offset (block offset
// + offset) once per file.
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferSkipped(JNIEnv* env, jclass, jlong infer, jint maxEntries) {
  int64_t n = 0;
  int32_t rc = tfr_infer_skipped((tfr_infer*)infer, &n, nullptr, nullptr, nullptr, 0);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  const int64_t k = maxEntries < 0 ? 0 : (n < maxEntries ? n : (int64_t)maxEntries);
  std::vector<int64_t> rec(k), off(k);
  std::vector<int32_t> code(k);
  if (k) tfr_infer_skipped((tfr_infer*)infer, &n, rec.data(), off.data(), code.data(), k);
  std::vector<jlong> v(1 + 4 * k);
  v[0] = (jlong)n;
  for (int64_t i = 0; i < k; ++i) { v[1 + 4 * i] = rec[i]; v[2 + 4 * i] = off[i]; v[3 + 4 * i] = code[i]; v[4 + 4 * i] = -1; }
  jlongArray a = env->NewLongArray((jsize)v.size()); env->SetLongArrayRegion(a, 0, (jsize)v.size(), v.data());
  return a;
}
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferUpdate(JNIEnv* env, jclass, jlong infer, jobject block, jlong nbytes, jboolean isFinal) {
  size_t used = 0;
  int32_t rc = tfr_infer_update_block((tfr_infer*)infer, env->GetDirectBufferAddress(block), (size_t)nbytes, 0, isFinal ? 1 : 0, &used);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)used;
}
extern "C" JNIEXPORT jobjectArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferResult(JNIEnv* env, jclass, jlong infer) {
  int32_t n = 0;
  int32_t rc = tfr_infer_result((tfr_infer*)infer, &n);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  jobjectArray names = env->NewObjectArray(n, env->FindClass("java/lang/String"), nullptr);
  std::vector<jint> codes(n);
  for (int32_t i = 0; i < n; ++i) {
    const char* nm = nullptr; int32_t len = 0, code = 0;
    tfr_infer_name((tfr_infer*)infer, i, &nm, &len, &code);
    env->SetObjectArrayElement(names, i, env->NewStringUTF(std::string(nm, (size_t)len).c_str()));
    codes[i] = code;
  }
  jintArray jc = env->NewIntArray(n);
  env->SetIntArrayRegion(jc, 0, n, codes.data());
  jobjectArray out = env->NewObjectArray(2, env->FindClass("java/lang/Object"), nullptr);
  env->SetObjectArrayElement(out, 0, names);
  env->SetObjectArrayElement(out, 1, jc);
  return out;
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_inferDestroy(JNIEnv*, jclass, jlong infer) { if (infer) tfr_infer_destroy((tfr_infer*)infer); }
// the record index (recordIndex=true): the writer's close() and DefaultSource.buildIndex, and a split's seek (INTEGRATION.md)
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_indexerCreate(JNIEnv* env, jclass, jint device, jlong stride) {
  tfr_indexer* h = nullptr;
  int32_t rc = tfr_indexer_create(device, (uint64_t)stride, &h);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)h;
}
// block: a direct ByteBuffer (host bytes), or with onDevice the device address of a drained encode (tfr_encoded_result(to_host = 0))
extern "C" JNIEXPORT jlong JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_indexUpdate(JNIEnv* env, jclass, jlong idx, jobject block, jlong deviceAddr,
                                                                                                 jlong nbytes, jboolean isFinal) {
  size_t used = 0;
  const void* p = block ? env->GetDirectBufferAddress(block) : (const void*)deviceAddr;
  int32_t rc = tfr_index_update((tfr_indexer*)idx, p, (size_t)nbytes, block ? 0 : 1, isFinal ? 1 : 0, &used);
  if (rc) { throw_for(env, rc, -1); return 0; }
  return (jlong)used;
}
extern "C" JNIEXPORT jobject JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_indexResult(JNIEnv* env, jclass, jlong idx) {
  const void* p = nullptr; size_t n = 0;
  int32_t rc = tfr_index_result((tfr_indexer*)idx, &p, &n);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  return env->NewDirectByteBuffer(const_cast<void*>(p), (jlong)n);     // owned by the indexer until indexerDestroy
}
// -> {entry, offset} of the first frame at or after target; bytes: the file from the checkpoint (base_entry, base_offset) on
extern "C" JNIEXPORT jlongArray JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_indexSeek(JNIEnv* env, jclass, jlong idx, jobject bytes, jlong nbytes,
                                                                                                      jlong baseEntry, jlong baseOffset, jlong target) {
  int64_t e = 0, o = 0;
  int32_t rc = tfr_index_seek((tfr_indexer*)idx, nbytes ? env->GetDirectBufferAddress(bytes) : nullptr, (size_t)nbytes, 0, baseEntry, baseOffset, target, &e, &o);
  if (rc) { throw_for(env, rc, -1); return nullptr; }
  jlong v[2] = {(jlong)e, (jlong)o};
  jlongArray a = env->NewLongArray(2); env->SetLongArrayRegion(a, 0, 2, v);
  return a;
}
extern "C" JNIEXPORT void JNICALL Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_indexerDestroy(JNIEnv*, jclass, jlong idx) { if (idx) tfr_indexer_destroy((tfr_indexer*)idx); }
#endif  // TFR_BUILD_JNI
