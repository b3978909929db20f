/**
 * The operator B200PlanMaker returns for one segment: DocIdSet -> Projection -> Aggregation/GroupBy executed by
 * libpinot_b200.so.  Predicate resolution (value -> dictIds), leaf-operator choice and result-block construction reuse
 * Pinot's own classes, so semantics above and below the device call are the reference's.
 * NOT COMPILED IN THIS REPOSITORY'S IMAGE (no JDK).
 */
package org.apache.pinot.b200;

import java.util.ArrayList;
import java.util.Arrays;
import java.util.Collections;
import java.util.HashSet;
import java.util.Iterator;
import java.util.List;
import java.util.Set;
import java.util.function.Supplier;
import org.apache.pinot.common.request.context.ExpressionContext;
import org.apache.pinot.common.request.context.FilterContext;
import org.apache.pinot.common.request.context.predicate.Predicate;
import org.apache.pinot.common.utils.DataSchema;
import org.apache.pinot.core.common.Operator;
import org.apache.pinot.core.operator.BaseOperator;
import org.apache.pinot.core.operator.ExecutionStatistics;
import org.apache.pinot.core.operator.blocks.results.AggregationResultsBlock;
import org.apache.pinot.core.operator.blocks.results.BaseResultsBlock;
import org.apache.pinot.core.operator.blocks.results.GroupByResultsBlock;
import org.apache.pinot.core.operator.filter.predicate.PredicateEvaluator;
import org.apache.pinot.core.operator.filter.predicate.PredicateEvaluatorProvider;
import org.apache.pinot.core.operator.filter.predicate.RangePredicateEvaluatorFactory.SortedDictionaryBasedRangePredicateEvaluator;
import org.apache.pinot.core.query.aggregation.function.AggregationFunction;
import org.apache.pinot.core.query.aggregation.groupby.AggregationGroupByResult;
import org.apache.pinot.core.query.aggregation.groupby.DoubleGroupByResultHolder;
import org.apache.pinot.core.query.aggregation.groupby.GroupByResultHolder;
import org.apache.pinot.core.query.aggregation.groupby.GroupKeyGenerator;
import org.apache.pinot.core.query.aggregation.groupby.ObjectGroupByResultHolder;
import org.apache.pinot.core.query.request.context.QueryContext;
import org.apache.pinot.segment.local.customobject.AvgPair;
import org.apache.pinot.segment.spi.IndexSegment;
import org.apache.pinot.spi.data.FieldSpec;
import org.apache.pinot.segment.spi.SegmentContext;
import org.apache.pinot.segment.spi.datasource.DataSource;
import org.apache.pinot.segment.spi.index.reader.Dictionary;
import org.apache.pinot.spi.trace.Tracing;
import org.apache.pinot.spi.utils.Pairs.IntPair;

public class B200Operator extends BaseOperator<BaseResultsBlock> {
  private static final String EXPLAIN_NAME = "B200_SCAN_AGGREGATE";
  // include/pinot_b200.h filter ops
  private static final int F_AND = 0, F_OR = 1, F_NOT = 2, F_MATCH_ALL = 3, F_EMPTY = 4, F_SCAN_RANGE = 5, F_SCAN_IN = 6,
      F_SCAN_NOT_IN = 7, F_INV_IN = 8, F_INV_NOT_IN = 9, F_DOC_RANGES = 10;

  private final long _ctx;
  private final B200SegmentCache _cache;
  private final IndexSegment _segment;
  private final QueryContext _queryContext;
  private final Supplier<Operator<? extends BaseResultsBlock>> _fallback;
  private ExecutionStatistics _statistics = new ExecutionStatistics(0, 0, 0, 0);

  B200Operator(long ctx, B200SegmentCache cache, SegmentContext segmentContext, QueryContext queryContext,
      Supplier<Operator<? extends BaseResultsBlock>> fallback) {
    _ctx = ctx;
    _cache = cache;
    _segment = segmentContext.getIndexSegment();
    _queryContext = queryContext;
    _fallback = fallback;
  }

  /**
   * AND / OR / NOT of EQ / NOT_EQ / IN / NOT_IN / RANGE on dictionary-encoded single-value identifiers, or on
   * single-column transform expressions (B200Transform: answered over a derived dictionary column).
   */
  static boolean filterIsAccelerated(FilterContext filter, IndexSegment segment) {
    if (filter == null) {
      return true;
    }
    switch (filter.getType()) {
      case AND: case OR: case NOT:
        return filter.getChildren().stream().allMatch(c -> filterIsAccelerated(c, segment));
      case PREDICATE:
        Predicate p = filter.getPredicate();
        if (p.getLhs().getType() != ExpressionContext.Type.IDENTIFIER) {
          if (!B200Transform.accepted(p.getLhs(), segment)) {
            return false;
          }
        } else {
          DataSource ds = segment.getDataSource(p.getLhs().getIdentifier());
          if (ds.getDictionary() == null || !ds.getDataSourceMetadata().isSingleValue()) {
            return false;
          }
        }
        switch (p.getType()) {
          case EQ: case NOT_EQ: case IN: case NOT_IN: case RANGE:
            return true;
          case REGEXP_LIKE:
            // a pattern on a dictionary STRING column resolves to dictIds like an IN (flatten() asks Pinot's own
            // PredicateEvaluator for them, so Java's regex semantics hold exactly)
            return p.getLhs().getType() == ExpressionContext.Type.IDENTIFIER
                && segment.getDataSource(p.getLhs().getIdentifier()).getDataSourceMetadata().getDataType().getStoredType()
                == FieldSpec.DataType.STRING;
          default:
            return false;
        }
      default:
        return false;
    }
  }

  // ---- filter tree in postfix order, dictId space (what FilterPlanNode + FilterOperatorUtils would build) ----
  private static final class Nodes {
    final List<int[]> _rows = new ArrayList<>(); // {op, column, numChildren, lo, hi, idsOffset, idsLength}
    final List<Integer> _ids = new ArrayList<>();

    void add(int op, int column, int numChildren, int lo, int hi, int[] ids) {
      int off = _ids.size();
      if (ids != null) {
        for (int id : ids) {
          _ids.add(id);
        }
      }
      _rows.add(new int[]{op, column, numChildren, lo, hi, off, ids == null ? 0 : ids.length});
    }
  }

  private void flatten(FilterContext filter, B200SegmentCache.Resident resident, Nodes out) {
    switch (filter.getType()) {
      case AND: case OR: case NOT:
        for (FilterContext child : filter.getChildren()) {
          flatten(child, resident, out);
        }
        out.add(filter.getType() == FilterContext.Type.AND ? F_AND : filter.getType() == FilterContext.Type.OR ? F_OR
            : F_NOT, -1, filter.getChildren().size(), 0, 0, null);
        return;
      default:
        break;
    }
    Predicate predicate = filter.getPredicate();
    if (predicate.getLhs().getType() != ExpressionContext.Type.IDENTIFIER) {
      // a derived column: resolved on its (sorted) dictionary; it has no inverted or sorted index, so the leaf is a scan
      B200Transform.Derived d = derived(predicate.getLhs());
      int[] ids = d.matchingIds(predicate);
      if (ids == null) {
        throw new Refused();
      }
      if (ids.length == 0) {
        out.add(F_EMPTY, d._column, 0, 0, 0, null);
      } else if (ids.length == d.cardinality()) {
        out.add(F_MATCH_ALL, d._column, 0, 0, 0, null);
      } else if (predicate.getType() == Predicate.Type.RANGE) {
        out.add(F_SCAN_RANGE, d._column, 0, ids[0], ids[ids.length - 1] + 1, null);
      } else {
        out.add(F_SCAN_IN, d._column, 0, 0, 0, ids);
      }
      return;
    }
    String column = predicate.getLhs().getIdentifier();
    DataSource ds = _segment.getDataSource(column);
    Dictionary dictionary = ds.getDictionary();
    PredicateEvaluator evaluator = PredicateEvaluatorProvider.getPredicateEvaluator(predicate, dictionary,
        ds.getDataSourceMetadata().getDataType());
    int col = resident.columnId(column);
    // FilterOperatorUtils.getLeafFilterOperator :74-133
    if (evaluator.isAlwaysFalse()) {
      out.add(F_EMPTY, col, 0, 0, 0, null);
    } else if (evaluator.isAlwaysTrue()) {
      out.add(F_MATCH_ALL, col, 0, 0, 0, null);
    } else if (ds.getDataSourceMetadata().isSorted()) {
      out.add(F_DOC_RANGES, col, 0, 0, 0, sortedDocRanges(ds, evaluator)); // SortedIndexBasedFilterOperator :60-135
    } else if (evaluator instanceof SortedDictionaryBasedRangePredicateEvaluator) {
      SortedDictionaryBasedRangePredicateEvaluator range = (SortedDictionaryBasedRangePredicateEvaluator) evaluator;
      out.add(F_SCAN_RANGE, col, 0, range.getStartDictId(), range.getEndDictId(), null);
    } else {
      boolean exclusive = evaluator.isExclusive();
      int[] ids = exclusive ? evaluator.getNonMatchingDictIds() : evaluator.getMatchingDictIds();
      boolean inverted = ds.getInvertedIndex() != null;
      out.add(inverted ? (exclusive ? F_INV_NOT_IN : F_INV_IN) : (exclusive ? F_SCAN_NOT_IN : F_SCAN_IN), col, 0, 0, 0,
          ids);
    }
  }

  /** Inclusive (start, end) docId pairs -- the range arithmetic of SortedIndexBasedFilterOperator :60-135. */
  private int[] sortedDocRanges(DataSource ds, PredicateEvaluator evaluator) {
    org.apache.pinot.segment.spi.index.reader.SortedIndexReader<?> sorted =
        (org.apache.pinot.segment.spi.index.reader.SortedIndexReader<?>) ds.getInvertedIndex();
    int numDocs = _segment.getSegmentMetadata().getTotalDocs();
    List<IntPair> ranges = new ArrayList<>();
    if (evaluator instanceof SortedDictionaryBasedRangePredicateEvaluator) {
      SortedDictionaryBasedRangePredicateEvaluator range = (SortedDictionaryBasedRangePredicateEvaluator) evaluator;
      ranges.add(new IntPair(sorted.getDocIds(range.getStartDictId()).getLeft(),
          sorted.getDocIds(range.getEndDictId() - 1).getRight()));
    } else {
      boolean exclusive = evaluator.isExclusive();
      int[] ids = exclusive ? evaluator.getNonMatchingDictIds() : evaluator.getMatchingDictIds();
      IntPair last = sorted.getDocIds(ids[0]);
      last = new IntPair(last.getLeft(), last.getRight());
      for (int i = 1; i < ids.length; i++) {
        IntPair cur = sorted.getDocIds(ids[i]);
        if (cur.getLeft() == last.getRight() + 1) {
          last.setRight(cur.getRight());
        } else {
          ranges.add(last);
          last = new IntPair(cur.getLeft(), cur.getRight());
        }
      }
      ranges.add(last);
      if (exclusive) {
        List<IntPair> inverted = new ArrayList<>();
        if (ranges.get(0).getLeft() > 0) {
          inverted.add(new IntPair(0, ranges.get(0).getLeft() - 1));
        }
        for (int i = 0; i + 1 < ranges.size(); i++) {
          inverted.add(new IntPair(ranges.get(i).getRight() + 1, ranges.get(i + 1).getLeft() - 1));
        }
        if (ranges.get(ranges.size() - 1).getRight() < numDocs - 1) {
          inverted.add(new IntPair(ranges.get(ranges.size() - 1).getRight() + 1, numDocs - 1));
        }
        ranges = inverted;
      }
    }
    int[] flat = new int[2 * ranges.size()];
    for (int i = 0; i < ranges.size(); i++) {
      flat[2 * i] = ranges.get(i).getLeft();
      flat[2 * i + 1] = ranges.get(i).getRight();
    }
    return flat;
  }

  /** The library refused a derived column (or a predicate on one): the stock operator answers the query. */
  private static final class Refused extends RuntimeException {
    Refused() {
      super(null, null, false, false);
    }
  }

  private B200SegmentCache.Resident _resident;

  /** The derived column of a transform expression on this segment (derived by the first query that names it). */
  private B200Transform.Derived derived(ExpressionContext e) {
    B200Transform.Derived d = _resident.derive(_ctx, e);
    if (d == null) {
      throw new Refused();
    }
    return d;
  }

  private int columnOf(ExpressionContext e) {
    return e.getType() == ExpressionContext.Type.IDENTIFIER ? _resident.columnId(e.getIdentifier()) : derived(e)._column;
  }

  /** Dictionary.getInternal(dictId) of a column or of a derived column. */
  private java.util.function.IntFunction<Object> decoder(ExpressionContext e) {
    if (e.getType() != ExpressionContext.Type.IDENTIFIER) {
      return derived(e)::get;
    }
    Dictionary dictionary = _segment.getDataSource(e.getIdentifier()).getDictionary();
    return dictionary::getInternal;
  }

  private BaseResultsBlock stock() {
    Operator<? extends BaseResultsBlock> stock = _fallback.get();
    BaseResultsBlock block = stock.nextBlock();
    _statistics = stock.getExecutionStatistics();
    return block;
  }

  @Override
  protected BaseResultsBlock getNextBlock() {
    _resident = _cache.get(_segment);
    B200SegmentCache.Resident resident = _resident;
    Nodes nodes = new Nodes();
    AggregationFunction[] functions = _queryContext.getAggregationFunctions();
    int[] aggFunctions = new int[functions.length];
    int[] aggColumns = new int[functions.length];
    List<ExpressionContext> groupBy = _queryContext.getGroupByExpressions();
    int[] groupByColumns;
    try {
      if (_queryContext.getFilter() != null) {
        flatten(_queryContext.getFilter(), resident, nodes);
      }
      for (int i = 0; i < functions.length; i++) {
        aggFunctions[i] = nativeFunction(functions[i]);
        List<ExpressionContext> inputs = functions[i].getInputExpressions();
        aggColumns[i] = inputs.isEmpty() ? -1 : columnOf(inputs.get(0));
      }
      groupByColumns = groupBy == null ? new int[0] : groupBy.stream().mapToInt(this::columnOf).toArray();
    } catch (Refused refused) {
      return stock();
    }
    int n = nodes._rows.size();
    int[] op = new int[n], column = new int[n], children = new int[n], lo = new int[n], hi = new int[n],
        idsOffset = new int[n], idsLength = new int[n];
    for (int i = 0; i < n; i++) {
      int[] r = nodes._rows.get(i);
      op[i] = r[0]; column[i] = r[1]; children[i] = r[2]; lo[i] = r[3]; hi[i] = r[4]; idsOffset[i] = r[5]; idsLength[i] = r[6];
    }
    int[] ids = nodes._ids.stream().mapToInt(Integer::intValue).toArray();
    long[] result = new long[1];
    int rc = B200Native.execute(_ctx, new long[]{resident._handle}, n, op, column, children, lo, hi, ids, idsOffset,
        idsLength, groupByColumns, aggFunctions, aggColumns, _queryContext.getNumGroupsLimit(),
        _queryContext.getMaxInitialResultHolderCapacity(), false, result);
    if (rc == B200Native.E_UNSUPPORTED || rc == B200Native.E_LIMIT) {
      // outside the accelerated set (e.g. LONG_MAP / ARRAY_MAP key spaces, numGroupsLimit binding): run the stock
      // operator so results stay exactly the reference's
      return stock();
    }
    if (rc != B200Native.OK) {
      throw new RuntimeException("pb200_execute failed for segment " + _segment.getSegmentName() + ": "
          + B200Native.lastError()); // wrapped by BaseCombineOperator.wrapOperatorException
    }
    try {
      return toResultsBlock(result[0], functions, groupBy);
    } finally {
      B200Native.resultFree(result[0]);
    }
  }

  private BaseResultsBlock toResultsBlock(long result, AggregationFunction[] functions, List<ExpressionContext> groupBy) {
    long[] meta = new long[7];
    B200Native.resultMeta(result, meta);
    _statistics = new ExecutionStatistics(meta[3], meta[4], meta[5], meta[6]);
    int rows = groupBy == null ? 1 : (int) meta[0];
    double[][] doubles = new double[functions.length][rows];
    long[][] longs = new long[functions.length][rows];
    for (int a = 0; a < functions.length; a++) {
      B200Native.resultAgg(result, a, doubles[a], longs[a]);
    }
    if (groupBy == null) {
      List<Object> results = new ArrayList<>(functions.length);
      for (int a = 0; a < functions.length; a++) {
        results.add(intermediate(result, functions[a], a, 0, doubles[a][0], longs[a][0]));
      }
      return new AggregationResultsBlock(functions, results, _queryContext);
    }
    // group keys: dictIds -> values with Dictionary.getInternal, exactly like DictionaryBasedGroupKeyGenerator.getKeys
    int k = groupBy.size();
    int[] keyIds = new int[rows * k];
    B200Native.resultGroupKeys(result, keyIds);
    List<java.util.function.IntFunction<Object>> dictionaries = new ArrayList<>();
    for (ExpressionContext e : groupBy) {
      dictionaries.add(decoder(e));
    }
    GroupKeyGenerator generator = new GroupKeyGenerator() {
      @Override public int getGlobalGroupKeyUpperBound() { return rows; }
      @Override public void generateKeysForBlock(org.apache.pinot.core.operator.blocks.ValueBlock b, int[] out) { throw new UnsupportedOperationException(); }
      @Override public void generateKeysForBlock(org.apache.pinot.core.operator.blocks.ValueBlock b, int[][] out) { throw new UnsupportedOperationException(); }
      @Override public int getCurrentGroupKeyUpperBound() { return rows; }
      @Override public int getNumKeys() { return rows; }
      @Override public Iterator<GroupKey> getGroupKeys() {
        return new Iterator<GroupKey>() {
          private int _next;
          private final GroupKey _groupKey = new GroupKey();
          @Override public boolean hasNext() { return _next < rows; }
          @Override public GroupKey next() {
            Object[] keys = new Object[k];
            for (int j = 0; j < k; j++) {
              keys[j] = dictionaries.get(j).apply(keyIds[_next * k + j]);
            }
            _groupKey._groupId = _next++;
            _groupKey._keys = keys;
            return _groupKey;
          }
        };
      }
    };
    GroupByResultHolder[] holders = new GroupByResultHolder[functions.length];
    for (int a = 0; a < functions.length; a++) {
      switch (functions[a].getType()) {
        case AVG: {
          ObjectGroupByResultHolder h = new ObjectGroupByResultHolder(rows, rows);
          h.ensureCapacity(rows);
          for (int g = 0; g < rows; g++) {
            h.setValueForKey(g, new AvgPair(doubles[a][g], longs[a][g]));
          }
          holders[a] = h;
          break;
        }
        default: {
          DoubleGroupByResultHolder h = new DoubleGroupByResultHolder(rows, rows, 0.0);
          h.ensureCapacity(rows);
          for (int g = 0; g < rows; g++) {
            h.setValueForKey(g, doubles[a][g]); // COUNT is held as a double too (CountAggregationFunction :112-116)
          }
          holders[a] = h;
        }
      }
    }
    DataSchema schema = buildSchema(functions, groupBy);
    GroupByResultsBlock block =
        new GroupByResultsBlock(schema, new AggregationGroupByResult(generator, functions, holders), _queryContext);
    block.setNumGroupsLimitReached(meta[2] != 0);
    return block;
  }

  private Object intermediate(long result, AggregationFunction function, int a, int row, double d, long l) {
    switch (function.getType()) {
      case COUNT:
        return l;
      case AVG:
        return new AvgPair(d, l);
      case DISTINCTCOUNT: {
        // the reference returns the VALUE set (BaseDistinctAggregateAggregationFunction.extractAggregationResult
        // converts the dictId bitmap with convertToValueSet): do the same from the returned dictIds
        java.util.function.IntFunction<Object> dictionary = decoder((ExpressionContext) function.getInputExpressions().get(0));
        Set<Object> values = new HashSet<>();
        for (int id : B200Native.resultDistinct(result, a, row)) {
          values.add(dictionary.apply(id));
        }
        return values;
      }
      default:
        return d; // SUM / MIN / MAX: Double
    }
  }

  private DataSchema buildSchema(AggregationFunction[] functions, List<ExpressionContext> groupBy) {
    // group-by columns then aggregation columns, as GroupByOperator's constructor does (:74-97)
    int k = groupBy.size();
    String[] names = new String[k + functions.length];
    DataSchema.ColumnDataType[] types = new DataSchema.ColumnDataType[k + functions.length];
    for (int j = 0; j < k; j++) {
      names[j] = groupBy.get(j).toString();
      ExpressionContext e = groupBy.get(j);
      types[j] = DataSchema.ColumnDataType.fromDataTypeSV(e.getType() == ExpressionContext.Type.IDENTIFIER
          ? _segment.getDataSource(e.getIdentifier()).getDataSourceMetadata().getDataType() : derived(e)._type);
    }
    for (int a = 0; a < functions.length; a++) {
      names[k + a] = functions[a].getResultColumnName();
      types[k + a] = functions[a].getIntermediateResultColumnType();
    }
    return new DataSchema(names, types);
  }

  private static int nativeFunction(AggregationFunction<?, ?> function) {
    switch (function.getType()) {
      case COUNT: return 0;
      case SUM: return 1;
      case MIN: return 2;
      case MAX: return 3;
      case AVG: return 4;
      case DISTINCTCOUNT: return 5;
      default: throw new IllegalStateException("not accelerated: " + function.getType());
    }
  }

  @Override
  public List<Operator> getChildOperators() {
    return Collections.emptyList();
  }

  @Override
  public String toExplainString() {
    return EXPLAIN_NAME;
  }

  @Override
  public IndexSegment getIndexSegment() {
    return _segment;
  }

  @Override
  public ExecutionStatistics getExecutionStatistics() {
    return _statistics;
  }
}
