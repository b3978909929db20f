/**
 * JNI surface of libpinot_b200.so -- one native method per function of include/pinot_b200.h.
 * Handles are opaque {@code long}s; every method returns the C status code (0 = OK) unless noted and the caller turns
 * a non-zero code into a RuntimeException (or a fallback, see B200PlanMaker).  NOT COMPILED IN THIS REPOSITORY'S IMAGE.
 */
package org.apache.pinot.b200;

import java.nio.ByteBuffer;

public final class B200Native {
  static {
    System.loadLibrary("pb200_jni"); // which links libpinot_b200.so
  }

  private B200Native() {
  }

  public static final int OK = 0;
  public static final int E_INVALID = -1;
  public static final int E_UNSUPPORTED = -2;
  public static final int E_CUDA = -3;
  public static final int E_NOMEM = -4;
  public static final int E_LIMIT = -5;

  // pb200_init / pb200_shutdown / pb200_last_error
  public static native long init(int device);
  public static native int shutdown(long ctx);
  public static native String lastError();

  /**
   * pb200_segment_register.  Per column i: fwdKind[i], storedType[i], bits[i], cardinality[i] and the direct buffers
   * fwd[i] / dict[i] (null for STRING) / inv[i] (null if absent), each exactly the bytes of the index as obtained from
   * SegmentDirectory.Reader.getIndexFor(column, StandardIndexes.forward() | dictionary() | inverted())
   * .toDirectByteBuffer(0, size).  Returns the segment handle or 0 (see lastError()).
   */
  public static native long segmentRegister(long ctx, String segmentName, int numDocs, int[] fwdKind, int[] storedType,
      int[] bits, int[] cardinality, ByteBuffer[] fwd, ByteBuffer[] dict, ByteBuffer[] inv);
  public static native int segmentRelease(long ctx, long segment);
  /**
   * pb200_segment_derive_column: the postfix program (op[k], i[k], d[k]) of a single-column expression over
   * sourceColumn.  Returns the new column id, or a negative PB200_E_* code (see lastError(); E_UNSUPPORTED: run the
   * stock operator).
   */
  public static native int segmentDeriveColumn(long ctx, long segment, int sourceColumn, int[] op, long[] i, double[] d);
  /** pb200_segment_column_info into infoOut[6]: {fwd_kind, stored_type, bits, cardinality, has_inverted, fwd_bytes}. */
  public static native int segmentColumnInfo(long segment, int column, long[] infoOut);
  /** pb200_segment_read_index(..., which = 1): the column's big-endian dictionary bytes, or null. */
  public static native byte[] segmentDictionary(long ctx, long segment, int column);

  /**
   * pb200_execute for ONE query over n segments.  The filter is flattened in postfix order, one tree per segment
   * (PB200_Q_PER_SEGMENT_FILTER): op/column/numChildren/lo/hi per node, `ids` concatenated with idsOffset/idsLength per
   * node.  Returns result handles (one per segment, or one when mergeSegments).
   */
  public static native int execute(long ctx, long[] segments, int numFilterNodes, int[] op, int[] column,
      int[] numChildren, int[] lo, int[] hi, int[] ids, int[] idsOffset, int[] idsLength, int[] groupByColumns,
      int[] aggFunctions, int[] aggColumns, int numGroupsLimit, int maxInitialResultHolderCapacity,
      boolean mergeSegments, long[] resultsOut);

  // pb200_result_*
  /** {numGroups, regime, groupsLimitReached, numDocsScanned, entriesInFilter, entriesPostFilter, totalDocs} */
  public static native int resultMeta(long result, long[] metaOut);
  public static native int resultGroupKeys(long result, int[] dictIdsOut);
  public static native int resultAgg(long result, int agg, double[] doublesOut, long[] longsOut);
  public static native int resultAggDictIds(long result, int agg, int[] dictIdsOut);
  public static native int[] resultDistinct(long result, int agg, int row);
  /** pb200_result_fetch: keys [rows x groupBy], doubles / longs / dictIds [aggs x rows] in ONE JNI call (any may be null). */
  public static native int resultFetch(long result, int[] keysOut, double[] doublesOut, long[] longsOut, int[] dictIdsOut);
  public static native int resultFree(long result);

  /**
   * pb200_result_columns: the result's columns IN PLACE.  Group extraction leaves them in their final layout inside a pinned
   * host block; each returned buffer is a NewDirectByteBuffer over one column (native byte order; null = neutral column:
   * 0.0 / 0 / -1 for every row).  Layout of the returned array: [keys, doubles[0..aggs), longs[0..aggs), dictIds[0..aggs)].
   * Valid until resultFree(result).
   */
  public static native java.nio.ByteBuffer[] resultColumns(long result);

  // ---- table-wide dictionaries (pb200_domain_*), see INTEGRATION.md section 6
  public static native long domainFromSegments(long ctx, long[] segments, int[] columns);
  public static native int segmentBindDomain(long ctx, long segment, long domain);
  public static native int domainRelease(long ctx, long domain);

  // ---- cross-GPU combine inside the library (pb200_comm_*): one process (or one context + thread) per GPU
  /** pb200_comm_unique_id: 128 bytes made by rank 0; ship them to the other ranks over the server's own RPC. */
  public static native byte[] commUniqueId();
  public static native int commInit(long ctx, byte[] uniqueId, int rank, int worldSize);
  /**
   * pb200_result_combine: every rank passes ITS deferred result (execute with mergeSegments, deferFinalize, reduceWorld =
   * worldSize).  Returns 0 = combined (read the result on `root`, free it elsewhere), 1 = every rank must run the query again
   * with noCountCarrier, negative = error.
   */
  public static native int resultCombine(long ctx, long result, int root);

  // ---- doc-id sets kept in HBM (pb200_doc_mask_upload): a cached StarTreeFilterOperator / BitmapBasedFilterOperator result
  public static native long docMaskUpload(long ctx, int numDocs, int[] words);
  public static native int docMaskFree(long ctx, long mask);

  /** pb200_tuning_set: launch knobs (pinot.server.query.executor.b200.* properties). */
  public static native int tuningSet(long ctx, String name, long value);
}
