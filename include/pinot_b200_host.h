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

/* ---- derived columns: single-column expressions by their canonical text (pb200_segment_derive_column) ------------- */
/* An expression is named by the text of the reference's ExpressionContext.toString(): function names in lower case
 * without '_', arguments separated by ',' without spaces, literals in single quotes -- datetrunc('DAY',ts),
 * divide(ts,'1000').  Aliases (DATE_TRUNC is datetrunc, ADD is plus, DOW is dayofweek, ...), time-unit literals in any
 * case and numeric literals by value are normalised first, so two spellings share one derived column.  That text is then
 * the column's name wherever a column name is accepted: pb200h_execute*, selection / DISTINCT columns and order items,
 * filter leaves, FILTER (WHERE ...) clauses, pb200h_domain_build, pb200h_explain -- each of them derives an expression it
 * does not know yet on every segment of the call, once per segment, before planning.  A stored column whose name equals
 * the text wins.  pb200h_segment_column_index / _column_info / pb200h_dictionary_get describe derived columns (types
 * LONG, INT or DOUBLE); pb200h_segment_num_columns counts stored columns only.  A derived column is never answered from
 * its dictionary alone (NonScanBasedAggregationOperator), has no inverted or sorted index, is no star-tree dimension, and
 * is freed with its segment.  Expressions derived in different orders on different segments can land at different
 * column ids: a call over such segments is PB200_E_UNSUPPORTED.
 * Explicit derivation: `column` receives the derived column's id.  PB200_E_INVALID: malformed text or an unknown column;
 * PB200_E_UNSUPPORTED: see pb200_segment_derive_column, plus two or more columns, unknown functions, wrong argument types
 * or counts, time zones other than UTC. */
int32_t pb200h_segment_derive(pb200_ctx* ctx, pb200h_segment* segment, const char* expression, int32_t* column);

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
       PB200H_RANGE = 7, PB200H_REGEXP_LIKE = 8 };
/* PB200H_REGEXP_LIKE: one literal, `s` = the pattern (pb200_match_pattern), on a STRING dictionary column.  Every pattern
 * leaf of a call -- filter and FILTER (WHERE ...) clauses -- is resolved on the device before planning, one
 * pb200_match_pattern per distinct (pattern, column) over all segments of the call; the leaf is then planned as an IN
 * over the matching dictIds (EMPTY / MATCH_ALL when none / all match; sorted, inverted or scan leaf as for IN).
 * PB200_E_UNSUPPORTED: a column that is not a STRING dictionary column, a derived column, a pattern outside the subset;
 * PB200_E_INVALID: a pattern that is not valid UTF-8. */

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
  int32_t merge_segments; /* 1: device-side combine (group-by / MIN / MAX / DISTINCT* columns must have identical
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
/* pb200h_execute_ordered with one argument per aggregation (pb200_execute_args: the percentile of a PERCENTILE).
 * PERCENTILE in a query with any FILTER (WHERE ...) clause is PB200_E_UNSUPPORTED; agg_args == NULL refuses PERCENTILE
 * with PB200_E_INVALID. */
int32_t pb200h_execute_args(pb200_ctx* ctx, const pb200h_query* query, const pb200_order_by* order, const double* agg_args,
                            pb200h_segment* const* segments, int32_t num_segments, pb200_result** results,
                            int32_t* operator_kinds);
/* pb200h_execute_args with the group-by rows filtered by HAVING (pb200_execute_having of include/pinot_b200.h; leaves index
 * query->aggs) before the ORDER BY and its trim.  having == NULL: exactly pb200h_execute_args.  Device results are filtered
 * on the device; results built on the host (star-tree, FILTER clauses) are filtered on the host by the same predicate,
 * after the FILTER clauses' submissions are aligned.  The same errors as pb200_execute_having (more than one result:
 * merge_segments == 0 with several segments; merge_segments == 2 is PB200_E_UNSUPPORTED). */
int32_t pb200h_execute_having(pb200_ctx* ctx, const pb200h_query* query, const pb200_order_by* order, const double* agg_args,
                              const pb200_having* having, pb200h_segment* const* segments, int32_t num_segments,
                              pb200_result** results, int32_t* operator_kinds);
/* One argument per aggregation (pb200_agg_arg of include/pinot_b200.h, the time column by name): p is the percentile of a
 * PERCENTILE or the log2m of a DISTINCTCOUNTHLL (0: the default 8); time_column (a column or an expression such as "datetrunc('HOUR',ts)", derived like any other name) and
 * value_type (PB200_INT ... PB200_STRING) belong to a FIRSTWITHTIME / LASTWITHTIME over pb200h_agg.column. */
typedef struct {
  double p;
  const char* time_column;
  int32_t value_type;
} pb200h_agg_arg;
/* pb200h_execute_having with a pb200h_agg_arg per aggregation (pb200_execute_agg_args).  args == NULL is
 * pb200h_execute_having without percentiles; the other entry points refuse FIRST/LASTWITHTIME with PB200_E_INVALID.
 * FIRST/LASTWITHTIME in a query with any FILTER (WHERE ...) clause is PB200_E_UNSUPPORTED. */
int32_t pb200h_execute_agg_args(pb200_ctx* ctx, const pb200h_query* query, const pb200_order_by* order, const pb200h_agg_arg* args,
                                const pb200_having* having, pb200h_segment* const* segments, int32_t num_segments,
                                pb200_result** results, int32_t* operator_kinds);
/* pb200h_execute_agg_args whose ORDER BY may name post-aggregation programs (pb200_execute_post of include/pinot_b200.h;
 * operands index query->aggs).  post == NULL: exactly pb200h_execute_agg_args.  Device results are ordered on the device;
 * star-tree results and the aligned results of FILTER clauses on the host, by the same evaluator.  The same errors as
 * pb200_execute_post. */
int32_t pb200h_execute_post(pb200_ctx* ctx, const pb200h_query* query, const pb200_order_by* order, const pb200h_agg_arg* args,
                            const pb200_having* having, const pb200_post_aggs* post, pb200h_segment* const* segments,
                            int32_t num_segments, pb200_result** results, int32_t* operator_kinds);
/* DISTINCTCOUNTHLL (the DISTINCTCOUNTHLL section of include/pinot_b200.h) through every entry point above, with the same
 * refusals.  A segment whose filter matches every doc is answered without a scan (PB200H_OP_NON_SCAN_AGGREGATION, as the
 * reference's NonScanBasedAggregationOperator does): the estimate over the whole dictionary, computed by the device
 * finalize.  PB200_E_UNSUPPORTED as well: a query with FILTER (WHERE ...) clauses, an argument that is an expression of
 * two or more columns; pb200h_result_to_datatable of a result with a DISTINCTCOUNTHLL (the reference serializes its
 * registers, which this library does not restate).  A star-tree never answers it: the raw scan runs. */
/* ---- selection (SELECT columns WHERE ... LIMIT n; pb200_execute_selection of include/pinot_b200.h) --------------- */
typedef struct {
  const char* column;
  int32_t descending;
} pb200h_select_order;
typedef struct {
  int32_t num_columns;
  const char* const* columns;  /* by name, in output order (SELECT * is resolved by the caller) */
  int32_t num_order_items;     /* 0 .. PB200_MAX_ORDER_BY (order columns need not be selected) */
  pb200h_select_order order[PB200_MAX_ORDER_BY];
  int64_t limit;
} pb200h_selection;
/* The filter and merge_segments of `query` (its group-by and aggregation fields are ignored) with the rows of `selection`
 * (ORDER BY semantics: pb200_execute_selection; a merged ORDER BY merges the segments' tops by value).
 * Predicates are resolved per segment like pb200h_execute; a segment whose filter folds to EMPTY is never scanned (its
 * result has no rows; merged: it contributes none), star-trees are never used.  results[] receives num_segments
 * handles (one when merge_segments); read them with pb200_result_selection -- segment_index refers to `segments`. */
int32_t pb200h_execute_selection(pb200_ctx* ctx, const pb200h_query* query, const pb200h_selection* selection,
                                 pb200h_segment* const* segments, int32_t num_segments, pb200_result** results);
/* SELECT DISTINCT (pb200_execute_distinct of include/pinot_b200.h): `distinct` names the DISTINCT columns and order
 * items (an order item must be one of the columns: PB200_E_INVALID otherwise).  Filters, EMPTY segments and results as
 * for pb200h_execute_selection; merge_segments needs the DISTINCT columns bound to one domain. */
int32_t pb200h_execute_distinct(pb200_ctx* ctx, const pb200h_query* query, const pb200h_selection* distinct,
                                pb200h_segment* const* segments, int32_t num_segments, pb200_result** results);

/* The result as the server -> broker wire format: DataTableImplV4 bytes (pinot-common/.../datatable/DataTableImplV4.java:49-81)
 * exactly as GroupByResultsBlock.getDataTable() / AggregationResultsBlock.getDataTable() build them for the same rows
 * (GroupByResultsBlock.java:186-236): typed group-key values (STRING keys through the DataTable's own string dictionary),
 * COUNT as LONG, SUM / MIN / MAX as DOUBLE, AVG as OBJECT AvgPair, DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG as OBJECT value set, + the execution
 * statistics as metadata.  `segment` supplies the dictionaries the result's ids refer to (any segment of a merged
 * result: they share dictionaries).  Returns the size (or the size needed when out == NULL), < 0 on error.
 * A result filtered by HAVING is PB200_E_UNSUPPORTED: a server's DataTable never carries rows HAVING removed. */
int64_t pb200h_result_to_datatable(const pb200h_query* query, const pb200h_segment* segment, const pb200_result* result,
                                   void* out, uint64_t capacity);

/* toExplainString()-style description of the plan of one segment (for tests / EXPLAIN); returns chars written. */
int32_t pb200h_explain(pb200_ctx* ctx, const pb200h_query* query, pb200h_segment* segment, char* out,
                       int32_t capacity);

/* ---- star-tree built on the device (MultipleTreesBuilder at segment load) ------------------------------------- */
/* One tree of a table's StarTreeIndexConfig. */
typedef struct {
  int32_t num_dimensions;
  const char* const* dimensions;    /* dimensionsSplitOrder */
  int32_t num_skip_star;
  const char* const* skip_star;     /* skipStarNodeCreationForDimensions (NULL when none) */
  int32_t num_pairs;
  const pb200h_agg* pairs;          /* functionColumnPairs: COUNT (column NULL or "*"), SUM, MIN, MAX */
  int32_t max_leaf_records;         /* maxLeafRecords (Pinot's default: 10000) */
} pb200h_startree_config;

enum { PB200H_STAR_PHASE_BASE = 0,      /* rows sorted by the split order, identical tuples merged */
       PB200H_STAR_PHASE_CONSTRUCT = 1, /* nodes and STAR children, level by level */
       PB200H_STAR_PHASE_AGGREGATE = 2, /* aggregated docs, bottom up */
       PB200H_STAR_PHASE_ENCODE = 3 };  /* star docs -> device segment (metric dictionaries) */

typedef struct {
  int64_t num_star_docs;
  int64_t num_base_docs;             /* docs of distinct dimension tuples: star docs [0, num_base_docs) */
  int32_t num_nodes;
  int32_t reserved;
  double phase_ms[4];                /* host wall clock per PB200H_STAR_PHASE_* */
} pb200h_startree_build_info;

/* Builds one star-tree from the segment's resident columns on the device (MultipleTreesBuilder at segment load) and
 * attaches it as pb200h_startree_attach would: the same tree as the reference's BaseSingleTreeBuilder up to how star
 * docs are numbered, the star docs a device segment with the same columns (dimensions, then count__* / sum__m / ...).
 * MIN / MAX follow Double.compare order; SUM over INT accumulates exactly and is rounded once, other SUMs accumulate in
 * double.  A load-time step like attach: not to be run concurrently with queries on that segment.  info may be NULL.
 * PB200_E_INVALID: unknown columns, an empty or repeated split order, a skip dimension outside it, maxLeafRecords < 1,
 * no pairs.  PB200_E_UNSUPPORTED: a dimension without dictIds, a derived column, a STRING metric, a function other
 * than COUNT / SUM / MIN / MAX, a domain-bound segment, more than 30 dimensions, a segment without docs, 2^31 or more
 * star docs.  A failure attaches nothing. */
int32_t pb200h_startree_build(pb200_ctx* ctx, pb200h_segment* segment, const pb200h_startree_config* config,
                              pb200h_startree_build_info* info);

/* The index-th star-tree of the segment, built or attached: its OffHeapStarTree buffer and the segment of its star
 * docs (owned by the segment; read it with the column accessors).  PB200_E_INVALID when there is no such tree. */
int32_t pb200h_startree_get(const pb200h_segment* segment, int32_t index, const void** tree, uint64_t* tree_bytes,
                            pb200h_segment** star_docs);

#ifdef __cplusplus
}
#endif
#endif /* PINOT_B200_HOST_H_ */
