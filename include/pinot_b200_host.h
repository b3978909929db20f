/*
 * pinot_b200_host.h -- the host side ABOVE the device C-ABI, in VALUE space.
 *
 * In a real deployment this layer is Java: `B200PlanMaker extends InstancePlanMakerImplV2` (java/ in this repo) reuses
 * Pinot's own PredicateEvaluators, FilterOperatorUtils selection rules and result-block classes and only calls
 * include/pinot_b200.h through JNI.  This image has no JDK, so the same logic is provided natively here, mirroring the
 * reference's interfaces for this path (names, argument meaning, error behaviour):
 *
 *   SegmentContext / IndexSegment.getDataSource(column)   -> pb200h_segment (+ pb200h_column descriptors by NAME)
 *   QueryContext (filter / aggregations / group-by)       -> pb200h_query   (values, not dictIds)
 *   PlanMaker.makeSegmentPlanNode(seg, query).run()       -> pb200h_plan_segments(): per segment, the operator kind
 *       + Operator.nextBlock()                               chosen and the dictId-space filter tree, then ONE device
 *                                                            submission for all segments (pb200_execute)
 *   PredicateEvaluatorProvider.getPredicateEvaluator      -> value -> dictId resolution on the sorted dictionaries
 *       (core/operator/filter/predicate/{Range,Equals,NotEquals,In,NotIn}PredicateEvaluatorFactory.java)
 *   FilterOperatorUtils.getLeafFilterOperator :74-133     -> leaf kind: sorted index / inverted index / scan
 *   AggregationPlanNode shortcuts :90-121,159-190          -> NonScanBasedAggregationOperator answered from the
 *                                                            dictionary + metadata without touching the device
 */
#ifndef PINOT_B200_HOST_H_
#define PINOT_B200_HOST_H_

#include "pinot_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pb200h_segment pb200h_segment;

typedef struct {
  const char* name;
  int32_t data_type;        /* PB200_INT .. PB200_STRING (stored type) */
  int32_t has_dictionary;
  int32_t bits_per_value;
  int32_t cardinality;
  int32_t is_sorted;        /* forward index is a sorted index (SortedIndexReaderImpl) */
  int32_t dict_entry_bytes; /* 4 / 8, or the padded entry length of a STRING dictionary */
  const void* fwd;
  uint64_t fwd_bytes;
  const void* dict;         /* big-endian fixed-width dictionary, or padded string entries */
  uint64_t dict_bytes;
  const void* inv;          /* bitmap inverted index or NULL */
  uint64_t inv_bytes;
} pb200h_column;

/* ImmutableSegmentLoader.load analogue for in-memory index buffers: uploads to HBM (pb200_segment_register) and keeps
 * the dictionaries on the host for predicate resolution. */
int32_t pb200h_segment_create(pb200_ctx* ctx, const char* name, int32_t num_docs, int32_t num_columns,
                              const pb200h_column* columns, pb200h_segment** segment);
/* Adopts a device-resident segment produced by pb200_synth_segment (dictionaries are read back from it). */
int32_t pb200h_segment_adopt(pb200_ctx* ctx, pb200_segment* device_segment, int32_t num_docs, int32_t num_columns,
                             const char* const* column_names, pb200h_segment** segment);
/* Loads a Pinot segment directory (v1 file-per-index, or v3 columns.psf + index_map) from disk. */
int32_t pb200h_segment_load_dir(pb200_ctx* ctx, const char* path, pb200h_segment** segment);
int32_t pb200h_segment_destroy(pb200h_segment* segment); /* IndexSegment.destroy() */
pb200_segment* pb200h_segment_device(pb200h_segment* segment);
int32_t pb200h_segment_num_docs(const pb200h_segment* segment);
int32_t pb200h_segment_num_columns(const pb200h_segment* segment);
int32_t pb200h_segment_column_index(const pb200h_segment* segment, const char* name);
const char* pb200h_segment_column_name(const pb200h_segment* segment, int32_t column);
/* {data_type, has_dictionary, bits, cardinality, is_sorted, has_inverted} */
int32_t pb200h_segment_column_info(const pb200h_segment* segment, int32_t column, int32_t out[6]);
/* Dictionary.getInternal(dictId): numeric -> *num (as double) / *lng; STRING -> bytes copied to str (NUL terminated) */
int32_t pb200h_dictionary_get(const pb200h_segment* segment, int32_t column, int32_t dict_id, double* num, int64_t* lng,
                              char* str, int32_t str_capacity);

/* ---- HBM residency (what BaseTableDataManager + SegmentDataManager reference counting are to the JVM heap / page cache) ---- */
/* Segments resident on the device, keyed by (segment name, CRC) -- SegmentMetadata.getName() / getCrc(); a new CRC under a
 * known name is a refresh (BaseTableDataManager.replaceSegment).  A byte budget (0 = 80 % of the device) with least-recently-
 * used eviction of segments no query holds; acquire / release bracket a query exactly like
 * SegmentDataManager.increaseReferenceCount / decreaseReferenceCount (ServerQueryExecutorV1Impl.java:217). */
typedef struct pb200h_cache pb200h_cache;
int32_t pb200h_cache_create(pb200_ctx* ctx, int64_t max_device_bytes, pb200h_cache** cache);
/* Hit: pins and returns the resident segment.  Miss: frees LRU unpinned segments until `size_hint` bytes (0 = unknown)
 * fit, loads `index_dir` (pb200h_segment_load_dir), pins.  PB200_E_NOMEM when everything resident is in use. */
int32_t pb200h_cache_acquire(pb200h_cache* cache, const char* segment_name, uint64_t crc, const char* index_dir,
                             int64_t size_hint, pb200h_segment** segment);
int32_t pb200h_cache_release(pb200h_cache* cache, pb200h_segment* segment);
/* The table dropped the segment (IndexSegment.destroy()): freed now, or by the last release. */
int32_t pb200h_cache_evict(pb200h_cache* cache, const char* segment_name, uint64_t crc);
/* {resident segments, resident bytes, budget, hits, misses, evictions} */
int32_t pb200h_cache_stats(pb200h_cache* cache, int64_t out[6]);
int32_t pb200h_cache_destroy(pb200h_cache* cache);

/* ---- table-wide dictionaries (include/pinot_b200.h "domains") by column NAME ------------------------------------- */
/* Union of the given segments' dictionaries for the named columns (every segment must hold them at the same position). */
int32_t pb200h_domain_build(pb200_ctx* ctx, pb200h_segment* const* segments, int32_t num_segments, int32_t num_columns,
                            const char* const* column_names, pb200_domain** domain);
/* pb200_segment_bind_domain + host bookkeeping: predicates keep being resolved against the segment's OWN dictionary
 * (identical alwaysTrue / alwaysFalse / index-choice decisions), ids are translated on the way to the device, and
 * pb200h_dictionary_get / pb200h_segment_column_info describe the domain dictionary (the id space of the results). */
int32_t pb200h_segment_bind_domain(pb200_ctx* ctx, pb200h_segment* segment, pb200_domain* domain);

/* ---- star-tree (StarTreeV2: seglocal/startree/v2/store/StarTreeLoaderUtils.java:54-88) -------------------------- */
typedef struct {
  int32_t function;     /* PB200_AGG_COUNT / SUM / MIN / MAX: the function of the function-column pair */
  int32_t reserved;
  const char* column;   /* NULL for count__* */
  const void* fwd;      /* raw fixed-byte forward index of the pre-aggregated values (PASS_THROUGH chunks; COUNT -> LONG,
                           others -> DOUBLE: ValueAggregatorFactory.getAggregatedValueType) */
  uint64_t fwd_bytes;
} pb200h_star_metric;

/* Attaches one star-tree to a loaded segment: `tree` = the OffHeapStarTree buffer (star_tree_index, LITTLE-endian
 * nodes), per dimension (split order) the fixed-bit forward index of the star-tree docs, per function-column pair the
 * raw forward index.  The star-tree docs are uploaded to HBM as a segment of their own; dimensions share the base
 * columns' dictionaries.  Queries that fit (StarTreeUtils rules) are then answered from it by pb200h_execute. */
int32_t pb200h_startree_attach(pb200_ctx* ctx, pb200h_segment* segment, const void* tree, uint64_t tree_bytes,
                               int32_t num_star_docs, int32_t num_dimensions, const char* const* dimension_names,
                               const void* const* dimension_fwd, const uint64_t* dimension_fwd_bytes,
                               int32_t num_metrics, const pb200h_star_metric* metrics);

/* ---- QueryContext ---------------------------------------------------------------------------------------------- */
enum { PB200H_AND = 0, PB200H_OR = 1, PB200H_NOT = 2, PB200H_EQ = 3, PB200H_NEQ = 4, PB200H_IN = 5, PB200H_NOT_IN = 6,
       PB200H_RANGE = 7 };

typedef struct {
  /* `d`: every numeric literal rounded to double (FLOAT columns compare (float)d).  `i`: the literal when it is an
     int64, so that (double)i == d; INT / LONG columns compare by exact value: `i` then, else a fractional `d` (no
     integer equals it), else (an integral or infinite `d`) a literal beyond the int64 range on the side of d */
  int64_t i;
  double d;
  const char* s; /* STRING columns */
} pb200h_literal;

typedef struct {                /* postfix order, root last (FilterContext tree flattened) */
  int32_t type;                 /* PB200H_* */
  const char* column;           /* leaves */
  int32_t num_children;         /* AND / OR */
  int32_t lower_inclusive, upper_inclusive, lower_unbounded, upper_unbounded; /* RANGE */
  int32_t num_values;           /* EQ/NEQ 1, IN/NOT_IN n, RANGE 2 */
  int32_t values_offset;
} pb200h_filter_node;

typedef struct {
  int32_t function;   /* PB200_AGG_* */
  const char* column; /* NULL for COUNT(*) */
} pb200h_agg;

typedef struct {
  int32_t num_filter_nodes;
  const pb200h_filter_node* filter;
  const pb200h_literal* literals;
  int32_t num_group_by;
  const char* const* group_by;
  int32_t num_aggs;
  const pb200h_agg* aggs;
  int32_t num_groups_limit;
  int32_t max_initial_result_holder_capacity;
  int32_t merge_segments; /* 1: device-side combine (group-by / MIN / MAX / DISTINCTCOUNT columns must have identical
                             dictionaries in all segments -- bind them to a domain -- else PB200_E_UNSUPPORTED);
                             2: combine and defer the group extraction (PB200_Q_DEFER_FINALIZE) */
  int32_t skip_star_tree; /* query option useStarTree=false */
  int32_t reduce_world;   /* merge_segments == 2: pb200_query.reduce_world */
  int32_t no_count_carrier; /* PB200_Q_NO_COUNT_CARRIER */
  int64_t merged_docs_bound;
  /* FILTER (WHERE ...) clauses (QueryContext.getFilteredAggregationFunctions, AggregationFunctionUtils.java:312-403):
   * aggregation a is filtered iff agg_filter_count[a] > 0; its postfix tree is agg_filter_nodes[agg_filter_start[a] ..
   * + agg_filter_count[a]) (literals shared with `filter`); equal (start, count) = the same clause.  NULL arrays: none.
   * Every distinct clause runs as one device submission over (filter AND clause), the functions without a clause over
   * `filter`; results are aligned by group key like FilteredGroupByOperator's shared key generator does. */
  const pb200h_filter_node* agg_filter_nodes;
  const int32_t* agg_filter_start;
  const int32_t* agg_filter_count;
} pb200h_query;

/* Which operator the plan maker chose per segment (AggregationPlanNode / GroupByPlanNode decisions). */
enum {
  PB200H_OP_AGGREGATION = 0,          /* AggregationOperator on the device */
  PB200H_OP_GROUP_BY = 1,             /* GroupByOperator on the device */
  PB200H_OP_NON_SCAN_AGGREGATION = 2, /* NonScanBasedAggregationOperator: dictionary / metadata only (host) */
  PB200H_OP_EMPTY = 3,                /* filter is EmptyFilterOperator: empty results block without any scan */
  PB200H_OP_STAR_TREE = 4             /* StarTreeFilterOperator + aggregation over the pre-aggregated star-tree docs */
};

/* makeSegmentPlanNode(...).run().nextBlock() for every segment; results[] receives num_segments handles (one when
 * merge_segments).  operator_kinds (optional) receives PB200H_OP_* per segment.  Errors: PB200_E_UNSUPPORTED means
 * "outside the accelerated set -- run the reference's operator" exactly like B200PlanMaker falling back to
 * super.makeSegmentPlanNode(). */
int32_t pb200h_execute(pb200_ctx* ctx, const pb200h_query* query, pb200h_segment* const* segments,
                       int32_t num_segments, pb200_result** results, int32_t* operator_kinds);
/* pb200h_execute with the group-by results ordered and trimmed (pb200_order_by of include/pinot_b200.h; group-by indices
 * refer to query->group_by, aggregation indices to query->aggs).  Results built on the host (star-tree, FILTER clauses) are
 * ordered and trimmed on the host by the same rule.  order == NULL: exactly pb200h_execute. */
int32_t pb200h_execute_ordered(pb200_ctx* ctx, const pb200h_query* query, const pb200_order_by* order,
                               pb200h_segment* const* segments, int32_t num_segments, pb200_result** results,
                               int32_t* operator_kinds);
/* The result as the server -> broker wire format: DataTableImplV4 bytes (pinot-common/.../datatable/DataTableImplV4.java:49-81)
 * exactly as GroupByResultsBlock.getDataTable() / AggregationResultsBlock.getDataTable() build them for the same rows
 * (GroupByResultsBlock.java:186-236): typed group-key values (STRING keys through the DataTable's own string dictionary),
 * COUNT as LONG, SUM / MIN / MAX as DOUBLE, AVG as OBJECT AvgPair, DISTINCTCOUNT as OBJECT value set, + the execution
 * statistics as metadata.  `segment` supplies the dictionaries the result's ids refer to (any segment of a merged
 * result: they share dictionaries).  Returns the size (or the size needed when out == NULL), < 0 on error. */
int64_t pb200h_result_to_datatable(const pb200h_query* query, const pb200h_segment* segment, const pb200_result* result,
                                   void* out, uint64_t capacity);

/* toExplainString()-style description of the plan of one segment (for tests / EXPLAIN); returns chars written. */
int32_t pb200h_explain(pb200_ctx* ctx, const pb200h_query* query, pb200h_segment* segment, char* out,
                       int32_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* PINOT_B200_HOST_H_ */
