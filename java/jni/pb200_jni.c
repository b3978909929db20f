/*
 * pb200_jni.c -- JNI glue between org.apache.pinot.b200.B200Native and include/pinot_b200.h.
 * NOT COMPILED IN THIS REPOSITORY'S IMAGE (no jni.h).  Build where a JDK exists:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../include pb200_jni.c \
 *       -L../../pinot_b200 -lpinot_b200 -o libpb200_jni.so
 * Only marshalling lives here: direct ByteBuffers -> (pointer, size), int[] -> temporary C arrays.
 */
#include <jni.h>
#include <stdlib.h>
#include <string.h>

#include "pinot_b200.h"

#define CLS(name) Java_org_apache_pinot_b200_B200Native_##name

JNIEXPORT jlong JNICALL CLS(init)(JNIEnv* env, jclass cls, jint device) {
  pb200_ctx* ctx = NULL;
  return pb200_init(device, &ctx) == PB200_OK ? (jlong)(intptr_t)ctx : 0;
}

JNIEXPORT jint JNICALL CLS(shutdown)(JNIEnv* env, jclass cls, jlong ctx) { return pb200_shutdown((pb200_ctx*)(intptr_t)ctx); }

JNIEXPORT jstring JNICALL CLS(lastError)(JNIEnv* env, jclass cls) { return (*env)->NewStringUTF(env, pb200_last_error()); }

static const void* buf_addr(JNIEnv* env, jobjectArray arr, jsize i, uint64_t* size) {
  jobject b = (*env)->GetObjectArrayElement(env, arr, i);
  if (!b) { *size = 0; return NULL; }
  *size = (uint64_t)(*env)->GetDirectBufferCapacity(env, b);
  return (*env)->GetDirectBufferAddress(env, b); /* zero copy: PinotDataBuffer.toDirectByteBuffer memory */
}

JNIEXPORT jlong JNICALL CLS(segmentRegister)(JNIEnv* env, jclass cls, jlong ctx, jstring name, jint numDocs,
                                             jintArray fwdKind, jintArray storedType, jintArray bits,
                                             jintArray cardinality, jobjectArray fwd, jobjectArray dict,
                                             jobjectArray inv) {
  jsize n = (*env)->GetArrayLength(env, fwdKind);
  pb200_col_desc* cols = (pb200_col_desc*)calloc((size_t)n, sizeof *cols);
  jint* k = (*env)->GetIntArrayElements(env, fwdKind, NULL);
  jint* t = (*env)->GetIntArrayElements(env, storedType, NULL);
  jint* b = (*env)->GetIntArrayElements(env, bits, NULL);
  jint* c = (*env)->GetIntArrayElements(env, cardinality, NULL);
  for (jsize i = 0; i < n; i++) {
    cols[i].fwd_kind = k[i]; cols[i].stored_type = t[i]; cols[i].bits_per_value = b[i]; cols[i].cardinality = c[i];
    cols[i].fwd = buf_addr(env, fwd, i, &cols[i].fwd_bytes);
    cols[i].dict = buf_addr(env, dict, i, &cols[i].dict_bytes);
    cols[i].inv = buf_addr(env, inv, i, &cols[i].inv_bytes);
  }
  const char* cname = (*env)->GetStringUTFChars(env, name, NULL);
  pb200_segment* seg = NULL;
  int rc = pb200_segment_register((pb200_ctx*)(intptr_t)ctx, cname, numDocs, n, cols, &seg);
  (*env)->ReleaseStringUTFChars(env, name, cname);
  (*env)->ReleaseIntArrayElements(env, fwdKind, k, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, storedType, t, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, bits, b, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, cardinality, c, JNI_ABORT);
  free(cols);
  return rc == PB200_OK ? (jlong)(intptr_t)seg : 0;
}

JNIEXPORT jint JNICALL CLS(segmentRelease)(JNIEnv* env, jclass cls, jlong ctx, jlong seg) {
  return pb200_segment_release((pb200_ctx*)(intptr_t)ctx, (pb200_segment*)(intptr_t)seg);
}

JNIEXPORT jint JNICALL CLS(segmentDeriveColumn)(JNIEnv* env, jclass cls, jlong ctx, jlong seg, jint source, jintArray op,
                                                jlongArray iv, jdoubleArray dv) {
  jsize n = (*env)->GetArrayLength(env, op);
  if (n <= 0 || n > 64 || (*env)->GetArrayLength(env, iv) != n || (*env)->GetArrayLength(env, dv) != n) return PB200_E_INVALID;
  pb200_transform_op prog[64];
  jint* o = (*env)->GetIntArrayElements(env, op, NULL);
  jlong* i = (*env)->GetLongArrayElements(env, iv, NULL);
  jdouble* d = (*env)->GetDoubleArrayElements(env, dv, NULL);
  for (jsize k = 0; k < n; k++) { prog[k].op = o[k]; prog[k].reserved = 0; prog[k].i = i[k]; prog[k].d = d[k]; }
  (*env)->ReleaseIntArrayElements(env, op, o, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, iv, i, JNI_ABORT);
  (*env)->ReleaseDoubleArrayElements(env, dv, d, JNI_ABORT);
  int32_t column = -1;
  int32_t rc = pb200_segment_derive_column((pb200_ctx*)(intptr_t)ctx, (pb200_segment*)(intptr_t)seg, source, n, prog, &column);
  return rc ? rc : column;
}

JNIEXPORT jint JNICALL CLS(segmentColumnInfo)(JNIEnv* env, jclass cls, jlong seg, jint column, jlongArray infoOut) {
  if ((*env)->GetArrayLength(env, infoOut) < 6) return PB200_E_INVALID;
  int64_t info[6];
  int32_t rc = pb200_segment_column_info((const pb200_segment*)(intptr_t)seg, column, info);
  jlong* o = (*env)->GetLongArrayElements(env, infoOut, NULL);
  for (int k = 0; k < 6 && rc == PB200_OK; k++) o[k] = info[k];
  (*env)->ReleaseLongArrayElements(env, infoOut, o, 0);
  return rc;
}

JNIEXPORT jbyteArray JNICALL CLS(segmentDictionary)(JNIEnv* env, jclass cls, jlong ctx, jlong seg, jint column) {
  pb200_ctx* c = (pb200_ctx*)(intptr_t)ctx;
  const pb200_segment* s = (const pb200_segment*)(intptr_t)seg;
  int64_t n = pb200_segment_read_index(c, s, column, 1, NULL, 0);
  if (n < 0) return NULL;
  jbyteArray out = (*env)->NewByteArray(env, (jsize)n);
  if (!out || n == 0) return out;
  jbyte* b = (*env)->GetByteArrayElements(env, out, NULL);
  int64_t r = pb200_segment_read_index(c, s, column, 1, b, (uint64_t)n);
  (*env)->ReleaseByteArrayElements(env, out, b, 0);
  return r < 0 ? NULL : out;
}

JNIEXPORT jint JNICALL CLS(execute)(JNIEnv* env, jclass cls, jlong ctx, jlongArray segments, jint numNodes, jintArray op,
                                    jintArray column, jintArray numChildren, jintArray lo, jintArray hi, jintArray ids,
                                    jintArray idsOffset, jintArray idsLength, jintArray groupBy, jintArray aggFn,
                                    jintArray aggCol, jint numGroupsLimit, jint maxInitCapacity, jboolean merge,
                                    jlongArray resultsOut) {
  jsize nseg = (*env)->GetArrayLength(env, segments);
  jsize total = (*env)->GetArrayLength(env, op); /* nseg * numNodes nodes (one tree per segment) */
  jint *o = (*env)->GetIntArrayElements(env, op, NULL), *col = (*env)->GetIntArrayElements(env, column, NULL),
       *ch = (*env)->GetIntArrayElements(env, numChildren, NULL), *l = (*env)->GetIntArrayElements(env, lo, NULL),
       *h = (*env)->GetIntArrayElements(env, hi, NULL), *id = (*env)->GetIntArrayElements(env, ids, NULL),
       *io = (*env)->GetIntArrayElements(env, idsOffset, NULL), *il = (*env)->GetIntArrayElements(env, idsLength, NULL),
       *gb = (*env)->GetIntArrayElements(env, groupBy, NULL), *af = (*env)->GetIntArrayElements(env, aggFn, NULL),
       *ac = (*env)->GetIntArrayElements(env, aggCol, NULL);
  jlong* segs = (*env)->GetLongArrayElements(env, segments, NULL);
  pb200_filter_node* nodes = (pb200_filter_node*)calloc((size_t)(total ? total : 1), sizeof *nodes);
  for (jsize i = 0; i < total; i++) {
    nodes[i].op = o[i]; nodes[i].column = col[i]; nodes[i].num_children = ch[i]; nodes[i].lo = l[i]; nodes[i].hi = h[i];
    nodes[i].ids = (const int32_t*)(id + io[i]); nodes[i].num_ids = il[i];
  }
  jsize nagg = (*env)->GetArrayLength(env, aggFn);
  pb200_agg* aggs = (pb200_agg*)calloc((size_t)nagg, sizeof *aggs);
  for (jsize a = 0; a < nagg; a++) { aggs[a].function = af[a]; aggs[a].column = ac[a]; }
  pb200_query q;
  memset(&q, 0, sizeof q);
  q.num_filter_nodes = numNodes;
  q.num_group_by = (*env)->GetArrayLength(env, groupBy);
  q.num_aggs = nagg;
  q.num_groups_limit = numGroupsLimit;
  q.max_initial_result_holder_capacity = maxInitCapacity;
  q.flags = PB200_Q_PER_SEGMENT_FILTER | (merge ? PB200_Q_MERGE_SEGMENTS : 0);
  q.filter = nodes; q.group_by_columns = (const int32_t*)gb; q.aggs = aggs;
  pb200_segment** ps = (pb200_segment**)calloc((size_t)nseg, sizeof *ps);
  for (jsize s = 0; s < nseg; s++) ps[s] = (pb200_segment*)(intptr_t)segs[s];
  jsize nres = merge ? 1 : nseg;
  pb200_result** res = (pb200_result**)calloc((size_t)nres, sizeof *res);
  int rc = pb200_execute((pb200_ctx*)(intptr_t)ctx, &q, ps, nseg, res);
  if (rc == PB200_OK) {
    jlong* out = (*env)->GetLongArrayElements(env, resultsOut, NULL);
    for (jsize r = 0; r < nres; r++) out[r] = (jlong)(intptr_t)res[r];
    (*env)->ReleaseLongArrayElements(env, resultsOut, out, 0);
  }
  free(res); free(ps); free(aggs); free(nodes);
  (*env)->ReleaseLongArrayElements(env, segments, segs, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, op, o, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, column, col, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, numChildren, ch, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, lo, l, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, hi, h, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, ids, id, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, idsOffset, io, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, idsLength, il, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, groupBy, gb, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, aggFn, af, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, aggCol, ac, JNI_ABORT);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultMeta)(JNIEnv* env, jclass cls, jlong result, jlongArray out) {
  pb200_result_meta m;
  int rc = pb200_result_meta_get((const pb200_result*)(intptr_t)result, &m);
  jlong v[7] = {m.num_groups, m.regime, m.groups_limit_reached, m.num_docs_scanned, m.num_entries_scanned_in_filter,
                m.num_entries_scanned_post_filter, m.num_total_docs};
  (*env)->SetLongArrayRegion(env, out, 0, 7, v);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultGroupKeys)(JNIEnv* env, jclass cls, jlong result, jintArray out) {
  jint* p = (*env)->GetIntArrayElements(env, out, NULL);
  int rc = pb200_result_group_keys((const pb200_result*)(intptr_t)result, (int32_t*)p);
  (*env)->ReleaseIntArrayElements(env, out, p, 0);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultAgg)(JNIEnv* env, jclass cls, jlong result, jint agg, jdoubleArray d, jlongArray l) {
  jdouble* pd = (*env)->GetDoubleArrayElements(env, d, NULL);
  jlong* pl = (*env)->GetLongArrayElements(env, l, NULL);
  int rc = pb200_result_agg((const pb200_result*)(intptr_t)result, agg, pd, (int64_t*)pl);
  (*env)->ReleaseDoubleArrayElements(env, d, pd, 0);
  (*env)->ReleaseLongArrayElements(env, l, pl, 0);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultAggDictIds)(JNIEnv* env, jclass cls, jlong result, jint agg, jintArray out) {
  jint* p = (*env)->GetIntArrayElements(env, out, NULL);
  int rc = pb200_result_agg_dict_ids((const pb200_result*)(intptr_t)result, agg, (int32_t*)p);
  (*env)->ReleaseIntArrayElements(env, out, p, 0);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultFetch)(JNIEnv* env, jclass cls, jlong result, jintArray keys, jdoubleArray dbl,
                                        jlongArray lng, jintArray ids) {
  jint* k = keys ? (*env)->GetIntArrayElements(env, keys, NULL) : NULL;
  jdouble* d = dbl ? (*env)->GetDoubleArrayElements(env, dbl, NULL) : NULL;
  jlong* l = lng ? (*env)->GetLongArrayElements(env, lng, NULL) : NULL;
  jint* i = ids ? (*env)->GetIntArrayElements(env, ids, NULL) : NULL;
  int rc = pb200_result_fetch((const pb200_result*)(intptr_t)result, (int32_t*)k, (double*)d, (int64_t*)l, (int32_t*)i);
  if (k) (*env)->ReleaseIntArrayElements(env, keys, k, 0);
  if (d) (*env)->ReleaseDoubleArrayElements(env, dbl, d, 0);
  if (l) (*env)->ReleaseLongArrayElements(env, lng, l, 0);
  if (i) (*env)->ReleaseIntArrayElements(env, ids, i, 0);
  return rc;
}

JNIEXPORT jintArray JNICALL CLS(resultDistinct)(JNIEnv* env, jclass cls, jlong result, jint agg, jint row) {
  int64_t n = pb200_result_distinct((const pb200_result*)(intptr_t)result, agg, row, NULL, 0);
  if (n < 0) return NULL;
  jintArray out = (*env)->NewIntArray(env, (jsize)n);
  jint* p = (*env)->GetIntArrayElements(env, out, NULL);
  pb200_result_distinct((const pb200_result*)(intptr_t)result, agg, row, (int32_t*)p, n);
  (*env)->ReleaseIntArrayElements(env, out, p, 0);
  return out;
}

JNIEXPORT jint JNICALL CLS(resultFree)(JNIEnv* env, jclass cls, jlong result) {
  return pb200_result_free((pb200_result*)(intptr_t)result);
}

/* pb200_result_columns: one direct ByteBuffer per column of the pinned block (no copy); the Java side sets ByteOrder.nativeOrder() */
JNIEXPORT jobjectArray JNICALL CLS(resultColumns)(JNIEnv* env, jclass cls, jlong result) {
  const pb200_result* R = (const pb200_result*)(intptr_t)result;
  pb200_result_meta m;
  if (pb200_result_meta_get(R, &m) != PB200_OK) return NULL;
  const int32_t* keys = NULL;
  const double* d[8] = {0};
  const int64_t* l[8] = {0};
  const int32_t* ids[8] = {0};
  if (pb200_result_columns(R, &keys, d, l, ids) != PB200_OK) return NULL;
  const jlong rows = m.num_groups < 0 ? 1 : m.num_groups;
  jclass bb = (*env)->FindClass(env, "java/nio/ByteBuffer");
  jobjectArray out = (*env)->NewObjectArray(env, 1 + 3 * m.num_aggs, bb, NULL);
  if (keys) (*env)->SetObjectArrayElement(env, out, 0, (*env)->NewDirectByteBuffer(env, (void*)keys, rows * m.num_group_by * 4));
  for (int a = 0; a < m.num_aggs; a++) {
    if (d[a]) (*env)->SetObjectArrayElement(env, out, 1 + a, (*env)->NewDirectByteBuffer(env, (void*)d[a], rows * 8));
    if (l[a]) (*env)->SetObjectArrayElement(env, out, 1 + m.num_aggs + a, (*env)->NewDirectByteBuffer(env, (void*)l[a], rows * 8));
    if (ids[a]) (*env)->SetObjectArrayElement(env, out, 1 + 2 * m.num_aggs + a, (*env)->NewDirectByteBuffer(env, (void*)ids[a], rows * 4));
  }
  return out;
}

JNIEXPORT jbyteArray JNICALL CLS(commUniqueId)(JNIEnv* env, jclass cls) {
  unsigned char id[PB200_COMM_ID_BYTES];
  if (pb200_comm_unique_id(id) != PB200_OK) return NULL;
  jbyteArray out = (*env)->NewByteArray(env, PB200_COMM_ID_BYTES);
  (*env)->SetByteArrayRegion(env, out, 0, PB200_COMM_ID_BYTES, (const jbyte*)id);
  return out;
}

JNIEXPORT jint JNICALL CLS(commInit)(JNIEnv* env, jclass cls, jlong ctx, jbyteArray id, jint rank, jint world) {
  jbyte* p = (*env)->GetByteArrayElements(env, id, NULL);
  int rc = pb200_comm_init((pb200_ctx*)(intptr_t)ctx, p, rank, world);
  (*env)->ReleaseByteArrayElements(env, id, p, JNI_ABORT);
  return rc;
}

JNIEXPORT jint JNICALL CLS(resultCombine)(JNIEnv* env, jclass cls, jlong ctx, jlong result, jint root) {
  int32_t retry = 0;
  int rc = pb200_result_combine((pb200_ctx*)(intptr_t)ctx, (pb200_result*)(intptr_t)result, root, &retry);
  return rc != PB200_OK ? rc : retry;
}

JNIEXPORT jlong JNICALL CLS(docMaskUpload)(JNIEnv* env, jclass cls, jlong ctx, jint numDocs, jintArray words) {
  jint* p = (*env)->GetIntArrayElements(env, words, NULL);
  uint32_t* dev = NULL;
  int rc = pb200_doc_mask_upload((pb200_ctx*)(intptr_t)ctx, numDocs, (const uint32_t*)p, (*env)->GetArrayLength(env, words), &dev);
  (*env)->ReleaseIntArrayElements(env, words, p, JNI_ABORT);
  return rc == PB200_OK ? (jlong)(intptr_t)dev : 0;
}

JNIEXPORT jint JNICALL CLS(docMaskFree)(JNIEnv* env, jclass cls, jlong ctx, jlong mask) {
  return pb200_doc_mask_free((pb200_ctx*)(intptr_t)ctx, (uint32_t*)(intptr_t)mask);
}

JNIEXPORT jint JNICALL CLS(tuningSet)(JNIEnv* env, jclass cls, jlong ctx, jstring name, jlong value) {
  const char* n = (*env)->GetStringUTFChars(env, name, NULL);
  int rc = pb200_tuning_set((pb200_ctx*)(intptr_t)ctx, n, value);
  (*env)->ReleaseStringUTFChars(env, name, n);
  return rc;
}

JNIEXPORT jlong JNICALL CLS(domainFromSegments)(JNIEnv* env, jclass cls, jlong ctx, jlongArray segments, jintArray columns) {
  const jsize n = (*env)->GetArrayLength(env, segments), k = (*env)->GetArrayLength(env, columns);
  jlong* s = (*env)->GetLongArrayElements(env, segments, NULL);
  jint* c = (*env)->GetIntArrayElements(env, columns, NULL);
  pb200_segment* segs[1024];
  pb200_domain* dom = NULL;
  int rc = PB200_E_INVALID;
  if (n <= 1024) {
    for (jsize i = 0; i < n; i++) segs[i] = (pb200_segment*)(intptr_t)s[i];
    rc = pb200_domain_from_segments((pb200_ctx*)(intptr_t)ctx, segs, n, k, (const int32_t*)c, &dom);
  }
  (*env)->ReleaseLongArrayElements(env, segments, s, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, columns, c, JNI_ABORT);
  return rc == PB200_OK ? (jlong)(intptr_t)dom : 0;
}

JNIEXPORT jint JNICALL CLS(segmentBindDomain)(JNIEnv* env, jclass cls, jlong ctx, jlong segment, jlong domain) {
  return pb200_segment_bind_domain((pb200_ctx*)(intptr_t)ctx, (pb200_segment*)(intptr_t)segment, (pb200_domain*)(intptr_t)domain);
}

JNIEXPORT jint JNICALL CLS(domainRelease)(JNIEnv* env, jclass cls, jlong ctx, jlong domain) {
  return pb200_domain_release((pb200_ctx*)(intptr_t)ctx, (pb200_domain*)(intptr_t)domain);
}
