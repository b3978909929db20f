/**
 * Plan maker that routes the scan -> filter -> (group-by) aggregate path of immutable segments to the GPU library and
 * leaves everything else to the stock implementation.  NOT COMPILED IN THIS REPOSITORY'S IMAGE (no JDK).
 *
 * Enable with   pinot.server.query.executor.plan.maker.class=org.apache.pinot.b200.B200PlanMaker
 * (CommonConstants.Server.CONFIG_OF_QUERY_EXECUTOR_PLAN_MAKER_CLASS; instantiated by
 *  ServerQueryExecutorV1Impl.init via PluginManager.get().createInstance + init(PinotConfiguration)).
 */
package org.apache.pinot.b200;

import java.util.List;
import org.apache.pinot.segment.spi.AggregationFunctionType;
import org.apache.pinot.common.request.context.ExpressionContext;
import org.apache.pinot.core.plan.PlanNode;
import org.apache.pinot.core.plan.maker.InstancePlanMakerImplV2;
import org.apache.pinot.core.query.aggregation.function.AggregationFunction;
import org.apache.pinot.core.query.request.context.QueryContext;
import org.apache.pinot.core.query.request.context.utils.QueryContextUtils;
import org.apache.pinot.segment.spi.ImmutableSegment;
import org.apache.pinot.segment.spi.IndexSegment;
import org.apache.pinot.segment.spi.SegmentContext;
import org.apache.pinot.spi.env.PinotConfiguration;

public class B200PlanMaker extends InstancePlanMakerImplV2 {
  public static final String DEVICE_KEY = "b200.device";
  private long _ctx;
  private B200SegmentCache _cache;

  @Override
  public void init(PinotConfiguration queryExecutorConfig) {
    super.init(queryExecutorConfig);
    _ctx = B200Native.init(queryExecutorConfig.getProperty(DEVICE_KEY, 0));
    if (_ctx == 0) {
      throw new IllegalStateException("pb200_init failed: " + B200Native.lastError());
    }
    _cache = new B200SegmentCache(_ctx);
  }

  @Override
  public PlanNode makeSegmentPlanNode(SegmentContext segmentContext, QueryContext queryContext) {
    IndexSegment segment = segmentContext.getIndexSegment();
    if (!(segment instanceof ImmutableSegment) || !QueryContextUtils.isAggregationQuery(queryContext)
        || !isAccelerated(queryContext, segment)) {
      return super.makeSegmentPlanNode(segmentContext, queryContext);
    }
    // run() builds the operator; B200Operator itself falls back to the stock operator when the native call answers
    // PB200_E_UNSUPPORTED (e.g. key space too large) or PB200_E_LIMIT (numGroupsLimit would bind)
    return () -> new B200Operator(_ctx, _cache, segmentContext, queryContext,
        () -> B200PlanMaker.super.makeSegmentPlanNode(segmentContext, queryContext).run());
  }

  /**
   * The accelerated set: identifiers and single-column transform expressions (B200Transform), no null handling,
   * COUNT/SUM/MIN/MAX/AVG/DISTINCTCOUNT.
   */
  static boolean isAccelerated(QueryContext queryContext, IndexSegment segment) {
    if (queryContext.isNullHandlingEnabled() || queryContext.getFilteredAggregationsIndexMap() != null
        && !queryContext.getFilteredAggregationsIndexMap().isEmpty()) {
      return false;
    }
    for (AggregationFunction<?, ?> function : queryContext.getAggregationFunctions()) {
      switch (function.getType()) {
        case COUNT: case SUM: case MIN: case MAX: case AVG: case DISTINCTCOUNT:
          break;
        default:
          return false;
      }
      for (Object e : function.getInputExpressions()) {
        ExpressionContext expression = (ExpressionContext) e;
        if (expression.getType() != ExpressionContext.Type.IDENTIFIER) {
          // a single-column transform: a derived column of the resident segment (B200Transform), numeric by construction
          if (!B200Transform.accepted(expression, segment)) {
            return false;
          }
          continue;
        }
        if (!segment.getDataSource(expression.getIdentifier()).getDataSourceMetadata().isSingleValue()) {
          return false;
        }
        // MIN / MAX of a STRING column come back as dictIds, which DoubleAggregationResultHolder cannot carry: stock operator
        if ((function.getType() == AggregationFunctionType.MIN || function.getType() == AggregationFunctionType.MAX)
            && segment.getDataSource(expression.getIdentifier()).getDataSourceMetadata().getDataType().getStoredType()
            == org.apache.pinot.spi.data.FieldSpec.DataType.STRING) {
          return false;
        }
      }
      // DISTINCTCOUNT with GROUP BY: the combine step merges value SETS per group (BaseDistinctAggregateAggregationFunction
      // :109-121, :306-321); B200Operator.toResultsBlock only builds the per-group sets for the aggregation-only case, so
      // the grouped form stays with the stock operator until that holder (ObjectGroupByResultHolder of Sets) is written
      if (function.getType() == AggregationFunctionType.DISTINCTCOUNT && queryContext.getGroupByExpressions() != null
          && !queryContext.getGroupByExpressions().isEmpty()) {
        return false;
      }
    }
    List<ExpressionContext> groupBy = queryContext.getGroupByExpressions();
    if (groupBy != null) {
      for (ExpressionContext expression : groupBy) {
        if (expression.getType() != ExpressionContext.Type.IDENTIFIER) {
          if (!B200Transform.accepted(expression, segment)) {
            return false;
          }
        } else if (segment.getDataSource(expression.getIdentifier()).getDictionary() == null) {
          return false;
        }
      }
    }
    return B200Operator.filterIsAccelerated(queryContext.getFilter(), segment);
  }
}
