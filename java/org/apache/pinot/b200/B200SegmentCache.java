/**
 * Segment residency in HBM: index buffers are uploaded ONCE per (segment name, CRC) and released when the segment is
 * destroyed.  Raw index bytes are not exposed by the operator-level SPI (reader objects keep their PinotDataBuffers
 * private), so the segment directory is opened independently -- the route BaseQueriesTest uses
 * (pinot-core/src/test/java/org/apache/pinot/queries/BaseQueriesTest.java:262-266).
 * NOT COMPILED IN THIS REPOSITORY'S IMAGE (no JDK).
 */
package org.apache.pinot.b200;

import java.nio.ByteBuffer;
import java.util.Map;
import java.util.Set;
import java.util.concurrent.ConcurrentHashMap;
import org.apache.pinot.segment.spi.ColumnMetadata;
import org.apache.pinot.segment.spi.IndexSegment;
import org.apache.pinot.segment.spi.SegmentMetadata;
import org.apache.pinot.segment.spi.index.StandardIndexes;
import org.apache.pinot.segment.spi.loader.SegmentDirectoryLoaderContext;
import org.apache.pinot.segment.spi.loader.SegmentDirectoryLoaderRegistry;
import org.apache.pinot.segment.spi.memory.PinotDataBuffer;
import org.apache.pinot.segment.spi.store.SegmentDirectory;
import org.apache.pinot.spi.data.FieldSpec.DataType;

public final class B200SegmentCache {
  /** Column order of a registered segment == column ids used in queries. */
  public static final class Resident {
    public final long _handle;
    public final String[] _columns;

    Resident(long handle, String[] columns) {
      _handle = handle;
      _columns = columns;
    }

    public int columnId(String name) {
      for (int i = 0; i < _columns.length; i++) {
        if (_columns[i].equals(name)) {
          return i;
        }
      }
      return -1;
    }

    // Derived columns by the expression's canonical text (ExpressionContext.toString()): derived once per resident
    // segment, on the first query that names the expression; a refusal is remembered so that later queries go to the
    // stock operator without asking the device again
    private final Map<String, B200Transform.Derived> _derived = new java.util.HashMap<>();
    private final Set<String> _refused = new java.util.HashSet<>();

    /** The derived column of `expression`, or null when the library refuses it (the caller runs the stock operator). */
    public synchronized B200Transform.Derived derive(long ctx, org.apache.pinot.common.request.context.ExpressionContext expression) {
      String key = expression.toString();
      B200Transform.Derived d = _derived.get(key);
      if (d != null || _refused.contains(key)) {
        return d;
      }
      B200Transform.Program p;
      try {
        p = B200Transform.compile(expression);
      } catch (IllegalArgumentException e) {
        _refused.add(key);
        return null;
      }
      int source = columnId(p._column);
      int n = p._op.size();
      int column = source < 0 ? -1 : B200Native.segmentDeriveColumn(ctx, _handle, source,
          p._op.stream().mapToInt(Integer::intValue).toArray(), p._i.stream().mapToLong(Long::longValue).toArray(),
          p._d.stream().mapToDouble(Double::doubleValue).toArray());
      long[] info = new long[6];
      if (column >= 0 && B200Native.segmentColumnInfo(_handle, column, info) != 0) {
        column = -1;
      }
      byte[] dictionary = column < 0 ? null : B200Native.segmentDictionary(ctx, _handle, column);
      if (column < 0 || dictionary == null || n == 0) {
        _refused.add(key);
        return null;
      }
      d = new B200Transform.Derived(column, (int) info[1], dictionary);
      _derived.put(key, d);
      return d;
    }
  }

  private final long _ctx;
  private final Map<String, Resident> _resident = new ConcurrentHashMap<>();

  B200SegmentCache(long ctx) {
    _ctx = ctx;
  }

  public Resident get(IndexSegment segment) {
    SegmentMetadata metadata = segment.getSegmentMetadata();
    String key = metadata.getName() + "#" + metadata.getCrc();
    return _resident.computeIfAbsent(key, k -> upload(segment));
  }

  /** Called from the table data manager's segment-removal hook (IndexSegment.destroy()). */
  public void evict(IndexSegment segment) {
    SegmentMetadata metadata = segment.getSegmentMetadata();
    Resident r = _resident.remove(metadata.getName() + "#" + metadata.getCrc());
    if (r != null) {
      B200Native.segmentRelease(_ctx, r._handle);
    }
  }

  private Resident upload(IndexSegment segment) {
    SegmentMetadata metadata = segment.getSegmentMetadata();
    Set<String> names = segment.getPhysicalColumnNames();
    // Only columns the library can hold are registered; every other column is simply ABSENT from the resident copy
    // (columnId == -1), which makes B200PlanMaker fall back to the stock operator for queries that touch it -- a
    // segment with a raw STRING / LONG / DOUBLE metric or an LZ4 chunk column must still serve its other queries here.
    String[] columns = names.stream().filter(c -> isUploadable(metadata.getColumnMetadataFor(c))).toArray(String[]::new);
    int n = columns.length;
    int[] fwdKind = new int[n];
    int[] storedType = new int[n];
    int[] bits = new int[n];
    int[] cardinality = new int[n];
    ByteBuffer[] fwd = new ByteBuffer[n];
    ByteBuffer[] dict = new ByteBuffer[n];
    ByteBuffer[] inv = new ByteBuffer[n];
    try (SegmentDirectory directory = SegmentDirectoryLoaderRegistry.getDefaultSegmentDirectoryLoader()
        .load(metadata.getIndexDir().toURI(), new SegmentDirectoryLoaderContext.Builder().build());
        SegmentDirectory.Reader reader = directory.createReader()) {
      for (int i = 0; i < n; i++) {
        ColumnMetadata cm = metadata.getColumnMetadataFor(columns[i]);
        DataType stored = cm.getDataType().getStoredType();
        storedType[i] = stored == DataType.INT ? 0 : stored == DataType.LONG ? 1 : stored == DataType.FLOAT ? 2
            : stored == DataType.DOUBLE ? 3 : 4;
        bits[i] = cm.getBitsPerElement();
        cardinality[i] = cm.getCardinality();
        // ForwardIndexReaderFactory dispatch (:74-91): sorted -> SortedIndexReaderImpl, dict -> FixedBitSV..V2, raw chunk
        fwdKind[i] = !cm.hasDictionary() ? 2 : cm.isSorted() ? 1 : 0;
        fwd[i] = whole(reader.getIndexFor(columns[i], StandardIndexes.forward()));
        if (cm.hasDictionary() && storedType[i] != 4) {
          dict[i] = whole(reader.getIndexFor(columns[i], StandardIndexes.dictionary()));
        }
        if (reader.hasIndexFor(columns[i], StandardIndexes.inverted())) {
          inv[i] = whole(reader.getIndexFor(columns[i], StandardIndexes.inverted()));
        }
      }
      long handle = B200Native.segmentRegister(_ctx, metadata.getName(), metadata.getTotalDocs(), fwdKind, storedType,
          bits, cardinality, fwd, dict, inv);  // copies to HBM during the call; buffers may be unmapped afterwards
      if (handle == 0) {
        throw new IllegalStateException("pb200_segment_register failed: " + B200Native.lastError());
      }
      return new Resident(handle, columns);
    } catch (Exception e) {
      throw new RuntimeException("Caught exception while uploading segment " + metadata.getName(), e);
    }
  }

  /**
   * What pb200_segment_register accepts (include/pinot_b200.h): single-value columns that are dictionary encoded
   * (fixed-bit or sorted forward index), or raw PASS_THROUGH fixed-byte INT / FLOAT columns.  Compressed raw chunks
   * (the default for raw metrics), raw LONG / DOUBLE / STRING / BYTES and multi-value columns stay with the JVM.
   */
  static boolean isUploadable(ColumnMetadata cm) {
    if (!cm.isSingleValue()) {
      return false;
    }
    if (cm.hasDictionary()) {
      return true;
    }
    DataType stored = cm.getDataType().getStoredType();
    // the chunk compression type is only known from the forward index header; pb200_segment_register refuses anything
    // but PASS_THROUGH, and upload() then retries without the column
    return stored == DataType.INT || stored == DataType.FLOAT;
  }

  private static ByteBuffer whole(PinotDataBuffer buffer) {
    // index files beyond 2 GB need slicing (view(start, end)); the native side accepts them as separate uploads
    return buffer.toDirectByteBuffer(0, (int) buffer.size());
  }
}
