/*
 * pinot_b200.h -- C-ABI of libpinot_b200.so: the H100-native (sm_90a) implementation of Apache Pinot's per-segment
 * scan -> filter -> project -> (group-by) aggregate operator chain.
 *
 * This is the drop-in boundary.  In the reference the path is entered through the plan-maker plugin seam
 *   PlanMaker.makeSegmentPlanNode(SegmentContext, QueryContext)
 *     (pinot-core/src/main/java/org/apache/pinot/core/plan/maker/PlanMaker.java:37-67, selected with
 *      pinot.server.query.executor.plan.maker.class, pinot-spi/.../utils/CommonConstants.java:690-691)
 * and the operator it returns is driven by  Operator.nextBlock()
 *     (core/operator/BaseOperator.java:39-50; called once per segment from
 *      core/operator/combine/BaseSingleBlockCombineOperator.java:85-108).
 * A Java `B200PlanMaker` (java/ in this repo, binding shown in INTEGRATION.md) keeps doing everything that is
 * dictionary / SQL / object work on the JVM side -- value -> dictId resolution with Pinot's own PredicateEvaluators,
 * filter-operator selection, result-block construction -- and calls the functions below through a thin JNI layer.
 * Everything crossing this boundary is plain pointers, sizes and fixed-width integers: no JNI, torch or C++ types.
 *
 * Conventions
 *  - every function returns 0 (PB200_OK) or a negative PB200_E_* code; pb200_last_error() gives the message of the
 *    calling thread's last failure.  No exceptions or longjmp cross the boundary.
 *  - thread safety: a pb200_ctx may be shared by any number of threads (Pinot runs one operator per worker thread,
 *    concurrently for many queries); pb200_segment handles are immutable after registration; pb200_result handles
 *    belong to the caller that received them.
 *  - ownership: index buffers passed to pb200_segment_register stay owned by the caller and are only read during the
 *    call (they are copied into 256-byte aligned HBM allocations; PinotDataBuffer.toDirectByteBuffer memory may be
 *    unmapped afterwards -- pinot-segment-spi/.../memory/PinotDataBuffer.java:632-654).
 */
#ifndef PINOT_B200_H_
#define PINOT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_ABI_VERSION 3 /* 2: pb200_query.reduce_world / merged_docs_bound, domains, tuning, pb200_result_meta.reserved bits;
                              3: pb200_comm_*, pb200_result_columns, doc masks, pb200h_query.agg_filter_* (the host query struct grew);
                                 pb200_order_by / pb200_execute_ordered / pb200h_execute_ordered were added later without a
                                 version change: they are new symbols and structs, no existing one changed; so were
                                 pb200_having / pb200_execute_having / pb200h_execute_having, and pb200_agg_arg /
                                 pb200_execute_agg_args / pb200h_execute_agg_args */

enum {
  PB200_OK = 0,
  PB200_E_INVALID = -1,     /* bad argument / malformed index bytes */
  PB200_E_UNSUPPORTED = -2, /* query shape outside the accelerated set: caller falls back to the Java operator */
  PB200_E_CUDA = -3,        /* CUDA runtime failure (message has the cudaError string) */
  PB200_E_NOMEM = -4,
  PB200_E_LIMIT = -5        /* numGroupsLimit would bind (first-seen order semantics): fall back */
};

typedef struct pb200_ctx pb200_ctx;
typedef struct pb200_segment pb200_segment;
typedef struct pb200_result pb200_result;

/* ---- context ------------------------------------------------------------------------------------------------- */
/* One context per (process, GPU).  `device` is the CUDA ordinal. Replaces nothing in the reference (there is no device
 * in it); lifetime == the server's QueryExecutor (ServerQueryExecutorV1Impl.init/shutDown :104-139). */
int32_t pb200_init(int32_t device, pb200_ctx** ctx);
int32_t pb200_shutdown(pb200_ctx* ctx);
const char* pb200_last_error(void);
int32_t pb200_abi_version(void);
/* Device facts for the caller's bookkeeping: {sm_count, major, minor, total_mem_mb, free_mem_mb}. */
int32_t pb200_device_info(pb200_ctx* ctx, int64_t out[5]);

/* Launch-tuning knobs of the scan kernel ("warps", "ctas_per_sm", "stages", "grid", "sparse_max", "sparse_max_agg",
 * "smem_groups", "smem_groups_max", "smem_copies", "dense_max", "defer", "gb_defer", "skip", "always_count"; DESIGN.md
 * section 3.1).  Their defaults are read from the environment (PB200_W, PB200_CTAS, ...) once, in pb200_init;
 * pb200_execute never reads the environment.  Not meant to be changed while queries are in flight on the context. */
int32_t pb200_tuning_set(pb200_ctx* ctx, const char* name, int64_t value);

/* ---- segments ------------------------------------------------------------------------------------------------ */
/* Stored types (FieldSpec.DataType.getStoredType()). */
enum { PB200_INT = 0, PB200_LONG = 1, PB200_FLOAT = 2, PB200_DOUBLE = 3, PB200_STRING = 4 };

/* Forward-index kinds (ForwardIndexReaderFactory.createIndexReader dispatch,
 * pinot-segment-local/.../segment/index/forward/ForwardIndexReaderFactory.java:74-91). */
enum {
  PB200_FWD_DICT_FIXEDBIT = 0, /* FixedBitSVForwardIndexReaderV2: MSB-first big-endian bit stream of dictIds */
  PB200_FWD_DICT_SORTED = 1,   /* SortedIndexReaderImpl: (startDocId, endDocId) BE int pairs per dictId */
  PB200_FWD_RAW_FIXEDBYTE = 2  /* FixedByteChunkSVForwardIndexReader, PASS_THROUGH chunks (file incl. header) */
};

#define PB200_COL_DEVICE_BUFFERS 1 /* flags: fwd/dict/inv already are device pointers in the layout below (adopted,
                                      not copied, not freed) -- used by the synthetic segment generator */

typedef struct {
  int32_t fwd_kind;       /* PB200_FWD_* */
  int32_t stored_type;    /* PB200_INT ... ; STRING dictionaries stay on the host (keys are dictIds on device) */
  int32_t bits_per_value; /* column.<c>.bitsPerElement (V1Constants.MetadataKeys.Column.BITS_PER_ELEMENT) */
  int32_t cardinality;    /* column.<c>.cardinality == Dictionary.length() */
  int32_t flags;
  int32_t reserved;       /* STRING dictionaries: width of one padded entry (column.<c>.lengthOfEachEntry); else 0 */
  const void* fwd;        /* forward index bytes exactly as in columns.psf / <col>.sv.unsorted.fwd */
  uint64_t fwd_bytes;
  const void* dict;       /* fixed-width BIG-endian sorted dictionary (<col>.dict without its 8-byte-less header: the
                             raw value array, cardinality * width bytes); NULL = no dictionary.  STRING dictionaries
                             (padded entries) stay on the host: they are only hashed / unioned (pb200_domain_*) */
  uint64_t dict_bytes;
  const void* inv;        /* bitmap inverted index file (<col>.bitmap.inv) or NULL:
                             BitmapInvertedIndexWriter layout, seglocal/.../inv/BitmapInvertedIndexWriter.java:33-50 */
  uint64_t inv_bytes;
} pb200_col_desc;

/* Uploads the listed columns of one immutable segment into HBM (once, at segment load: the analogue of
 * ImmutableSegmentLoader.load + PhysicalColumnIndexContainer; evict with pb200_segment_release from
 * IndexSegment.destroy()).  Column order defines the column ids used in queries. */
int32_t pb200_segment_register(pb200_ctx* ctx, const char* segment_name, int32_t num_docs, int32_t num_columns,
                               const pb200_col_desc* columns, pb200_segment** segment);
int32_t pb200_segment_release(pb200_ctx* ctx, pb200_segment* segment);
/* Bytes of HBM held by the segment. */
int64_t pb200_segment_device_bytes(const pb200_segment* segment);

/* ---- REGEXP_LIKE on STRING dictionaries (RegexpLikePredicateEvaluatorFactory: a pattern -> matching dictIds) --------- */
/* Matches `pattern` (UTF-8, NUL terminated; Java's Pattern.compile(pattern).matcher(value).find() over the subset of
 * DESIGN.md section 3.12) against every entry of column columns[s] of segments[s], for all segments in one launch, and
 * sets bit j of match_bits[s] (bit j % 32 of word j / 32) iff entry j of the segment's OWN dictionary matches: for a
 * column bound to a domain, ids are the segment's local dictIds, not the domain's.  match_bits[s] holds
 * ceil(cardinality / 32) words of that dictionary; the bits after the last entry of its last word are 0.  A value is
 * its dictionary entry up to the first NUL.  The first call on a column uploads a compact copy of its dictionary (counted
 * in pb200_segment_device_bytes, freed with the segment).  PB200_E_INVALID: a pattern that is not valid UTF-8, bad
 * arguments.  PB200_E_UNSUPPORTED: a pattern outside the subset, a column that is not a STRING dictionary column of the
 * segment (raw, derived). */
int32_t pb200_match_pattern(pb200_ctx* ctx, const char* pattern, int32_t num_segments, pb200_segment* const* segments,
                            const int32_t* columns, uint32_t* const* match_bits);

/* ---- table-wide dictionaries ("domains") ------------------------------------------------------------------------- */
/* dictIds are segment local in Pinot; the reference merges per-segment results BY VALUE
 * (GroupByCombineOperator.java:130-146 -> IndexedTable.upsert, AggregationFunction.merge).  A device-side or cross-GPU
 * merge of dictId-indexed tables needs ONE id space per column instead: a domain = the sorted union of the per-segment
 * dictionaries.  Binding a segment re-encodes the listed columns' forward indexes into the domain's ids (one streaming
 * pass at load time, no per-row work at query time) and lets the column adopt the shared table-wide dictionary; from
 * then on every id the library takes or returns for that column (filter leaves, group keys, MIN / MAX ids, DISTINCTCOUNT
 * sets, pb200_segment_read_index bytes) is a DOMAIN id.  PB200_Q_MERGE_SEGMENTS requires, for every group-by, MIN / MAX
 * and DISTINCTCOUNT column, identical dictionaries in all segments -- which bound segments have by construction. */
typedef struct pb200_domain pb200_domain;
typedef struct {
  int32_t column;               /* column id (registration order) */
  int32_t stored_type;          /* PB200_INT ... PB200_STRING */
  int32_t num_parts;            /* sorted dictionaries to union (one per segment, or per rank, ...) */
  int32_t reserved;
  const void* const* parts;     /* each: BIG-endian sorted values (or padded strings), cardinalities[i] entries */
  const int32_t* cardinalities;
  const int32_t* entry_bytes;   /* STRING: padded width of each part's entries; NULL for numeric types */
} pb200_domain_col;
int32_t pb200_domain_create(pb200_ctx* ctx, int32_t num_columns, const pb200_domain_col* columns, pb200_domain** domain);
/* Union over the given (unbound) segments' own dictionaries. */
int32_t pb200_domain_from_segments(pb200_ctx* ctx, pb200_segment* const* segments, int32_t num_segments,
                                   int32_t num_columns, const int32_t* columns, pb200_domain** domain);
/* {stored_type, cardinality, bits, entry_bytes} of one domain column. */
int32_t pb200_domain_column_info(const pb200_domain* domain, int32_t column, int64_t out[4]);
/* The domain dictionary's bytes (big-endian sorted values / padded strings); returns the size, or the needed size if
 * out == NULL.  Used to decode ids of bound columns and to exchange rank-local unions between GPUs. */
int64_t pb200_domain_dictionary(const pb200_domain* domain, int32_t column, void* out, uint64_t capacity);
/* Drops the caller's reference; bound segments keep the domain alive. */
int32_t pb200_domain_release(pb200_ctx* ctx, pb200_domain* domain);
/* Fails with PB200_E_INVALID (segment untouched) if a dictionary value of the segment is missing from the domain. */
int32_t pb200_segment_bind_domain(pb200_ctx* ctx, pb200_segment* segment, pb200_domain* domain);
/* The ids of `column` that occur in this segment, ascending (unbound: 0 .. cardinality-1).  Returns their number. */
int64_t pb200_segment_local_ids(const pb200_segment* segment, int32_t column, int32_t* out, int64_t capacity);

/* ---- query (dictId space) ------------------------------------------------------------------------------------ */
/* Filter tree in POSTFIX order (children before parent, root last), per SEGMENT because dictIds are segment local.
 * Leaves are what the reference's leaf filter operators consume AFTER PredicateEvaluator construction
 * (core/operator/filter/FilterOperatorUtils.java:74-133):                                                          */
enum {
  PB200_F_AND = 0,         /* AndFilterOperator      -- num_children operands */
  PB200_F_OR = 1,          /* OrFilterOperator */
  PB200_F_NOT = 2,         /* NotFilterOperator      -- 1 operand */
  PB200_F_MATCH_ALL = 3,   /* MatchAllFilterOperator */
  PB200_F_EMPTY = 4,       /* EmptyFilterOperator */
  PB200_F_SCAN_RANGE = 5,  /* ScanBasedFilterOperator + SortedDictionaryBasedRangePredicateEvaluator:
                              dictId in [lo, hi)  (RangePredicateEvaluatorFactory.java:220-222) */
  PB200_F_SCAN_IN = 6,     /* ScanBasedFilterOperator + EQ/IN evaluator: dictId in ids[] */
  PB200_F_SCAN_NOT_IN = 7, /* ... NEQ/NOT_IN: dictId not in ids[] */
  PB200_F_INV_IN = 8,      /* InvertedIndexFilterOperator: OR of the bitmaps of ids[] (InvertedIndexFilterOperator.java
                              :60-96); column must have been registered with an inverted index */
  PB200_F_INV_NOT_IN = 9,  /* ... flipped over [0, numDocs) */
  PB200_F_DOC_RANGES = 10, /* SortedIndexBasedFilterOperator: ids[] holds num_ids/2 inclusive (start,end) docId pairs */
  PB200_F_RAW_RANGE = 11,  /* scan of a raw INT/LONG/FLOAT/DOUBLE column: raw_lo <= v <= raw_hi with the flags below */
  PB200_F_DOC_MASK = 12    /* BitmapBasedFilterOperator over a caller-computed doc-id set (e.g. the star-tree traversal
                              result, core/startree/operator/StarTreeFilterOperator.java:168-171): ids points to
                              num_ids 32-bit words, bit j of word w = doc 32*w + j */
};

typedef struct {
  int32_t op;           /* PB200_F_* */
  int32_t column;       /* leaf: column id (index into the columns given at registration) */
  int32_t num_children; /* AND / OR */
  int32_t lo, hi;       /* SCAN_RANGE: [lo, hi) in dictId space */
  int32_t num_ids;
  const int32_t* ids;   /* host pointer; sorted ascending */
  double raw_lo, raw_hi;
  int32_t raw_flags;    /* bit0 lower unbounded, bit1 upper unbounded, bit2 lower exclusive, bit3 upper exclusive */
  int32_t reserved;     /* PB200_NODE_* bits */
} pb200_filter_node;
/* DOC_MASK whose `ids` is a DEVICE mask made by pb200_doc_mask_upload (a doc-id set reused by many queries, e.g. a cached
 * star-tree traversal): nothing is copied at query time; the caller keeps it alive until the queries using it returned. */
#define PB200_NODE_IDS_ON_DEVICE 1

/* Aggregation functions accelerated on this path (core/query/aggregation/function/{Count,Sum,Min,Max,Avg,
 * DistinctCount,Percentile,Variance,FirstWithTime,LastWithTime,DistinctSum,DistinctAvg,DistinctCountHLL}AggregationFunction.java).
 * PERCENTILE takes its percentile through pb200_execute_args; the four VarianceAggregationFunction types and
 * DISTINCTSUM / DISTINCTAVG take no argument (see pb200_result_moments and the DISTINCTSUM section below);
 * FIRSTWITHTIME / LASTWITHTIME take their time column through pb200_execute_agg_args; DISTINCTCOUNTHLL takes an optional
 * log2m through the same per-aggregation argument (see the DISTINCTCOUNTHLL section below). */
enum { PB200_AGG_COUNT = 0, PB200_AGG_SUM = 1, PB200_AGG_MIN = 2, PB200_AGG_MAX = 3, PB200_AGG_AVG = 4,
       PB200_AGG_DISTINCTCOUNT = 5, PB200_AGG_PERCENTILE = 6, PB200_AGG_VARPOP = 7, PB200_AGG_VARSAMP = 8,
       PB200_AGG_STDDEVPOP = 9, PB200_AGG_STDDEVSAMP = 10, PB200_AGG_FIRSTWITHTIME = 11, PB200_AGG_LASTWITHTIME = 12,
       PB200_AGG_DISTINCTSUM = 13, PB200_AGG_DISTINCTAVG = 14, PB200_AGG_DISTINCTCOUNTHLL = 15 };

typedef struct {
  int32_t function; /* PB200_AGG_* */
  int32_t column;   /* -1 for COUNT(*) */
} pb200_agg;

typedef struct {
  int32_t num_filter_nodes; /* 0 = match all */
  int32_t num_group_by;
  int32_t num_aggs;
  int32_t num_groups_limit;                   /* QueryContext.getNumGroupsLimit(), default 100000 */
  int32_t max_initial_result_holder_capacity; /* default 10000; selects the ARRAY regime like
                                                 DictionaryBasedGroupKeyGenerator.java:150-185 */
  int32_t flags;
  const pb200_filter_node* filter;            /* per segment: num_segments * num_filter_nodes entries when
                                                 PB200_Q_PER_SEGMENT_FILTER is set, else shared by all segments */
  const int32_t* group_by_columns;
  const pb200_agg* aggs;
  /* PB200_Q_DEFER_FINALIZE only: how many such tables (one per GPU) will be summed into the final one, and an upper bound
   * of the docs of ALL of them (0: this call's docs x reduce_world).  They size the count field of a count-carrying sum
   * identically on every rank; 0 / 1 = no cross-GPU reduce follows. */
  int32_t reduce_world;
  int32_t reserved;
  int64_t merged_docs_bound;
} pb200_query;

#define PB200_Q_PER_SEGMENT_FILTER 1 /* filter[] holds one tree per segment (segment-local dictIds) */
#define PB200_Q_MERGE_SEGMENTS 2     /* accumulate into ONE result (device-side combine, the GroupByCombineOperator /
                                        AggregationCombineOperator analogue).  Every group-by, MIN / MAX and DISTINCTCOUNT
                                        column must have the SAME dictionary in all segments (bind them to a domain);
                                        otherwise PB200_E_UNSUPPORTED -- never a merge of unrelated dictIds */
#define PB200_Q_NO_COUNT_CARRIER 8   /* keep a separate COUNT table (the retry of a cross-GPU combine whose carrier overflowed) */
#define PB200_Q_DEFER_FINALIZE 4     /* group-by with PB200_Q_MERGE_SEGMENTS: leave the groups in the dense device tables
                                        (pb200_result_device_buffers) and extract them later with pb200_result_finalize --
                                        for a cross-GPU reduce of the tables in between; only the reduce root extracts */

/* Runs the operator chain DocIdSet -> Projection -> Aggregation/GroupBy for `num_segments` segments in one device
 * submission (one persistent kernel over all segments' tiles).  Writes num_segments result handles (or exactly one
 * with PB200_Q_MERGE_SEGMENTS).  == Operator.nextBlock() of GroupByOperator / AggregationOperator
 * (core/operator/query/GroupByOperator.java:101-140, AggregationOperator.java:64-80). */
int32_t pb200_execute(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments,
                      int32_t num_segments, pb200_result** results);

/* ---- ORDER BY ... LIMIT of group-by results (GroupByCombineOperator's IndexedTable / TableResizer trim) ---------------- */
/* An order item compares the FINAL value of an aggregation (COUNT, SUM, MIN / MAX with +-inf for a group without rows,
 * AVG = sum / count or -inf at count 0, DISTINCTCOUNT = set size; doubles like Double.compare) or the dictId of a group-by
 * column; rows equal on every item are ordered by their group-key values ascending, in GROUP BY column order.  The rows of
 * an ordered result come back in that order, and only the first trim_size of them (trim_size <= 0: all, sorted).  The
 * numGroupsLimit check applies to the untrimmed group count; num_groups is the number of rows kept. */
#define PB200_MAX_ORDER_BY 8
enum { PB200_ORDER_AGG = 0, PB200_ORDER_GROUP_BY = 1, PB200_ORDER_POST = 2 };
typedef struct {
  int32_t kind;       /* PB200_ORDER_AGG: index into pb200_query.aggs; PB200_ORDER_GROUP_BY: index into group_by_columns;
                         PB200_ORDER_POST: index into pb200_post_aggs.programs (pb200_execute_post only) */
  int32_t index;
  int32_t descending; /* 0: ASC, else DESC */
} pb200_order_item;
typedef struct {
  int32_t num_items;  /* 1 .. PB200_MAX_ORDER_BY */
  int32_t trim_size;  /* rows kept per result; <= 0: sort without trimming */
  pb200_order_item items[PB200_MAX_ORDER_BY];
} pb200_order_by;
/* pb200_execute with the group-by results ordered and trimmed on the device (order == NULL: exactly pb200_execute).  A
 * PB200_Q_DEFER_FINALIZE result keeps the spec: pb200_result_finalize and pb200_result_combine apply it when they extract.
 * Aggregation-only queries ignore it.  A bad item index or num_items outside 1..8: PB200_E_INVALID. */
int32_t pb200_execute_ordered(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order,
                              pb200_segment* const* segments, int32_t num_segments, pb200_result** results);

/* ---- PERCENTILE(col, p): exact percentiles from per-group dictId histograms ------------------------------------------ */
/* pb200_execute_ordered with one argument per aggregation: agg_args[a] is the percentile p (0 <= p <= 100, fractions
 * allowed) of a PB200_AGG_PERCENTILE aggregation and is ignored for the other functions.  agg_args == NULL is
 * pb200_execute_ordered, which refuses PERCENTILE with PB200_E_INVALID (as does a p outside [0, 100] or NaN).
 * Semantics (PercentileAggregationFunction.extractFinalResult): the n values of the column over the group's matched rows,
 * as doubles, sorted ascending; n == 0: -inf; p == 100: the largest; otherwise the value at index
 * (int64)((double)n * p / 100.0), clamped to n - 1.  The column must carry dictIds (INT / LONG / FLOAT / DOUBLE
 * dictionaries, raw columns whose dictionary was synthesised at load): a dictionary is sorted, so a histogram of counts
 * over dictIds is the sorted value list.  Several PERCENTILEs of one column share one histogram.
 * Results: pb200_result_agg gives the value (double column) and n (long column), pb200_result_agg_dict_ids the selected
 * dictId (-1 when n == 0), so that a LONG beyond 2^53 can be looked up exactly; ORDER BY compares the double value.
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): STRING columns, raw columns streamed as 32-bit values,
 * histograms above 2^28 entries over all results of the call (aggregation only: 2^bits per result; group-by: table
 * entries x cardinality), a result over 2^32 docs or more, PB200_Q_DEFER_FINALIZE; a PB200_Q_MERGE_SEGMENTS submission
 * needs the column's dictionary to be the same in every segment.  NaN and -0.0 are out of scope, as for MIN / MAX. */
int32_t pb200_execute_args(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const double* agg_args,
                           pb200_segment* const* segments, int32_t num_segments, pb200_result** results);

/* ---- HAVING of group-by results (the broker's GroupByDataTableReducer filter, applied to a FINAL result) ----------- */
/* A POSTFIX tree (children before parent, root last) of at most PB200_MAX_HAVING_NODES nodes.  A leaf compares the FINAL
 * value of aggregation `agg` (index into pb200_query.aggs) as a double: COUNT / DISTINCTCOUNT the count, AVG sum / count
 * (-inf at count 0), the other functions their double column.  Comparisons are Java's <, <=, ==: a NaN value matches only
 * NEQ, -0.0 equals 0.0, +-inf compare as usual (NOT the Double.compare order of ORDER BY).  The caller expands IN into an
 * OR of EQ leaves and NOT IN into an AND of NEQ leaves. */
#define PB200_MAX_HAVING_NODES 32
enum { PB200_HAVING_AND = 0, PB200_HAVING_OR = 1, PB200_HAVING_NOT = 2, PB200_HAVING_RANGE = 3, PB200_HAVING_EQ = 4,
       PB200_HAVING_NEQ = 5 };
typedef struct {
  int32_t op;           /* PB200_HAVING_* */
  int32_t num_children; /* AND / OR: operands (>= 1); NOT: 1 */
  int32_t agg;          /* leaves: index into pb200_query.aggs */
  int32_t flags;        /* RANGE: as pb200_filter_node.raw_flags (bit0 lower unbounded, bit1 upper unbounded, bit2 lower
                           exclusive, bit3 upper exclusive); at least one side bounded */
  double lo, hi;        /* RANGE: bounds; EQ / NEQ: the literal in lo.  Never NaN */
} pb200_having_node;
typedef struct {
  int32_t num_nodes;    /* 1 .. PB200_MAX_HAVING_NODES */
  int32_t reserved;
  pb200_having_node nodes[PB200_MAX_HAVING_NODES];
} pb200_having;
/* pb200_execute_args with the group-by rows filtered by `having` on the device, before the ORDER BY and its trim
 * (having == NULL: exactly pb200_execute_args).  The numGroupsLimit check applies to the group count before HAVING;
 * num_groups is the number of rows kept; the execution statistics do not change.  HAVING needs a final result: a group-by
 * query that writes ONE result (PB200_Q_MERGE_SEGMENTS, or one segment).
 * PB200_E_INVALID: a malformed tree, an aggregation index out of range, a NaN bound, no group-by, more than one result.
 * PB200_E_UNSUPPORTED: PB200_Q_DEFER_FINALIZE or reduce_world > 1 (HAVING across GPUs is not offered). */
int32_t pb200_execute_having(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const double* agg_args,
                             const pb200_having* having, pb200_segment* const* segments, int32_t num_segments,
                             pb200_result** results);

/* ---- FIRSTWITHTIME / LASTWITHTIME(v, t, 'T'): the value of v in the first / last matched row by time ---------------- */
/* One argument per aggregation that may name a second column.  p: the percentile of a PERCENTILE (as agg_args of
 * pb200_execute_args).  time_column, value_type: the time column t (column id) and the type literal 'T' (PB200_INT ...
 * PB200_STRING; BOOLEAN names PB200_INT) of a FIRSTWITHTIME / LASTWITHTIME, whose pb200_agg.column is the data column v.
 * The other functions ignore the fields. */
typedef struct {
  double p;
  int32_t time_column;
  int32_t value_type;
} pb200_agg_arg;
/* pb200_execute_having with a pb200_agg_arg per aggregation (args == NULL: PERCENTILE and the *WITHTIME functions are
 * PB200_E_INVALID; pb200_execute, pb200_execute_ordered, pb200_execute_args and pb200_execute_having refuse the
 * *WITHTIME functions the same way).
 * Semantics (DESIGN.md section 3.13): LASTWITHTIME is the value of v in the matched row of the group with the largest t,
 * FIRSTWITHTIME with the smallest t.  Ties on t: LAST takes the tied row that comes last in the call's row order, FIRST
 * the one that comes first; that order is segments in submission order, then doc id.  t must be an INT or LONG column
 * with dictIds (a stored dictionary, a raw column whose dictionary was synthesised at load, a derived column): a
 * dictionary is sorted, so dictId order is time order.  v must be an INT, LONG, FLOAT, DOUBLE or STRING column with
 * dictIds, and value_type its stored type (the library never casts).
 * Results: pb200_result_agg gives the value of v as a double (STRING: its dictId, as for MIN / MAX; -inf when the group
 * has no matched row) and the winning row's time value, exact, in the long column; pb200_result_agg_dict_ids the dictId
 * of v (-1 when empty), so that STRING values and LONG values beyond 2^53 are looked up exactly.  ORDER BY and HAVING
 * compare the double.
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): a time column that is not INT / LONG or has no dictIds, a
 * data column without dictIds (raw 32-bit values), a value_type that is not the data column's stored type, a call over
 * 2^32 docs or more, PB200_Q_DEFER_FINALIZE or reduce_world > 1, ORDER BY or HAVING on a STRING-typed *WITHTIME; a
 * PB200_Q_MERGE_SEGMENTS submission needs the same dictionary for v and for t in every segment. */
int32_t pb200_execute_agg_args(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                               const pb200_having* having, pb200_segment* const* segments, int32_t num_segments,
                               pb200_result** results);
/* ---- ORDER BY arithmetic over aggregations: SUM(a) / SUM(b), COUNT(*) * 100.0 / SUM(n) (DESIGN.md section 3.18) ----- */
/* A post-aggregation program is POSTFIX (root last) over the FINAL values of a row's aggregations: AGG pushes the final
 * value of aggregation `agg` (index into pb200_query.aggs) as a double -- COUNT / DISTINCTCOUNT the count, AVG sum / count
 * (-inf at count 0), the other functions their double column, as HAVING reads them; LITERAL pushes `value` (finite);
 * ADD, SUB, MUL, DIV pop two operands and push one IEEE-754 double operation rounded to nearest (never an FMA; x / 0 is
 * +-inf, 0 / 0 NaN); NEG flips the sign of the top operand.  A PB200_ORDER_POST item orders rows by its program's value in
 * Double.compare order (-0.0 before 0.0, every NaN one value after +inf); ties, trim and numGroupsLimit as for the other
 * items. */
#define PB200_MAX_POST_NODES 16
enum { PB200_POST_AGG = 0, PB200_POST_LITERAL = 1, PB200_POST_ADD = 2, PB200_POST_SUB = 3, PB200_POST_MUL = 4,
       PB200_POST_DIV = 5, PB200_POST_NEG = 6 };
typedef struct {
  int32_t op;           /* PB200_POST_* */
  int32_t agg;          /* AGG: index into pb200_query.aggs */
  double value;         /* LITERAL: the literal */
} pb200_post_node;
typedef struct {
  int32_t num_nodes;    /* 1 .. PB200_MAX_POST_NODES */
  int32_t reserved;
  pb200_post_node nodes[PB200_MAX_POST_NODES];
} pb200_post_program;
typedef struct {
  int32_t num_programs; /* 0 .. PB200_MAX_ORDER_BY */
  int32_t reserved;
  pb200_post_program programs[PB200_MAX_ORDER_BY];
} pb200_post_aggs;
/* pb200_execute_agg_args whose ORDER BY may name programs of `post` (post == NULL: exactly pb200_execute_agg_args).  A
 * PB200_Q_DEFER_FINALIZE result keeps the programs with its order spec for pb200_result_finalize / pb200_result_combine.
 * PB200_E_INVALID: a malformed program (unknown op, an aggregation index out of range, a stack that does not end with one
 * value, a non-finite literal, num_nodes outside 1..16), num_programs outside 0..8, a PB200_ORDER_POST index past
 * num_programs.  PB200_E_UNSUPPORTED: a DISTINCTCOUNT operand without per-group sets, a STRING-typed *WITHTIME operand. */
int32_t pb200_execute_post(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                           const pb200_having* having, const pb200_post_aggs* post, pb200_segment* const* segments,
                           int32_t num_segments, pb200_result** results);

/* The histogram behind PERCENTILE aggregation `agg` in row `row`: its non-zero bins ascending by dictId (counts > 0), the
 * intermediate for merging per-segment results by value (the analogue of pb200_result_distinct).  Returns the number of
 * bins (or < 0 on error) and writes at most `capacity` of them; either output may be NULL.  The histograms are copied from
 * the device on the first call for a result, so a caller that reads only the final values pays nothing for them. */
int64_t pb200_result_histogram(const pb200_result* result, int32_t agg, int32_t row, int32_t* dict_ids, int64_t* counts,
                               int64_t capacity);

/* ---- VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP: exact moments over limb dictionaries ------------------------------ */
/* PB200_AGG_VARPOP / VARSAMP / STDDEVPOP / STDDEVSAMP through pb200_execute, pb200_execute_ordered or pb200_execute_args
 * (no argument).  Semantics (VarianceAggregationFunction): over the n values of the column in the group's matched rows,
 * M2 = sum (v - mean)^2, VARPOP = M2 / n, VARSAMP = M2 / (n - 1), STDDEV* = sqrt of the matching variance (a correctly
 * rounded sqrt of that double); n == 0, and *SAMP with n == 1, give -inf.  The variance is computed EXACTLY and rounded
 * once (the reference accumulates in double): every route and knob gives the same bits.
 * A column qualifies when every value of its dictionary is c + k * 2^e with c the smallest value and k an integer in
 * [0, 2^32): INT always; LONG when max - min < 2^32 (e = 0); FLOAT / DOUBLE on a common dyadic grid of that size (e.g.
 * integral values or halves; 0.1-steps do not qualify).  Several of these functions over one column share one set of
 * sums.  Results: pb200_result_agg gives the value (double column) and n (long column); ORDER BY compares the double.
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): STRING columns, raw columns streamed as 32-bit values,
 * columns that do not qualify, a result over 2^32 docs or more, more than 6 aggregations after the expansion (each
 * column adds 3 internal sums), PB200_Q_DEFER_FINALIZE; a PB200_Q_MERGE_SEGMENTS submission needs the column's
 * dictionary to be the same in every segment.  NaN, +-inf and -0.0 are out of scope, as for MIN / MAX. */
/* The exact intermediate behind aggregation `agg` in row `row`, for merging per-segment results by value: n values
 * v_i = c + k_i * 2^e with c = c_mant * 2^c_exp exactly, s1 = sum k_i and s2 = s2_hi * 2^64 + s2_lo = sum k_i^2.
 * Any output may be NULL.  PB200_E_INVALID when the aggregation is not one of the four functions. */
int32_t pb200_result_moments(const pb200_result* result, int32_t agg, int32_t row, int64_t* n, int64_t* c_mant,
                             int32_t* c_exp, int32_t* e, uint64_t* s1, uint64_t* s2_lo, uint64_t* s2_hi);

/* ---- DISTINCTSUM / DISTINCTAVG: exact sums over DISTINCTCOUNT's value sets (DESIGN.md section 3.14) ------------------ */
/* PB200_AGG_DISTINCTSUM / DISTINCTAVG through any pb200_execute* entry point (no argument).  Over S, the set of distinct
 * values of the column in the group's matched rows (the set DISTINCTCOUNT counts; -0.0 and 0.0 are two members, all NaNs
 * one): DISTINCTSUM is the exact sum of S rounded once to the nearest double (0.0 for an empty S), DISTINCTAVG that sum
 * divided by |S| rounded once (-inf for an empty S).  NaN in S, or both infinities, give NaN; otherwise an infinity in S
 * gives that infinity.  A column qualifies when it carries dictIds and its dictionary is INT or LONG, or FLOAT / DOUBLE
 * with every finite value j * 2^e for one exponent e and an integer |j| < 2^63 (integral values, halves: yes; 0.01-steps:
 * no).  Several of these functions and DISTINCTCOUNT over one column share one bitset.
 * Results: pb200_result_agg gives the value (double column) and |S| (long column); pb200_result_distinct the dictId set,
 * as for DISTINCTCOUNT; ORDER BY and HAVING compare the double.
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): STRING columns, raw columns streamed as 32-bit values, FLOAT /
 * DOUBLE dictionaries off such a grid, the DISTINCTCOUNT bitset budget; a PB200_Q_MERGE_SEGMENTS submission needs the
 * column's dictionary to be the same in every segment.  Like DISTINCTCOUNT they are not reduced across GPUs on the device. */

/* ---- DISTINCTCOUNTHLL(col[, log2m]): HyperLogLog estimates over DISTINCTCOUNT's value sets (DESIGN.md section 3.17) --- */
/* PB200_AGG_DISTINCTCOUNTHLL through any pb200_execute* entry point.  log2m is agg_args[a] (pb200_execute_args,
 * pb200_execute_having) or pb200_agg_arg.p (pb200_execute_agg_args): an integral value; 0, and every entry point without
 * arguments, mean the reference's default 8.  Over S, the set of distinct values of the column in the group's matched rows
 * (the set DISTINCTCOUNT counts; -0.0 and 0.0 are two members, all NaNs one), the result is the estimate of a HyperLogLog
 * with 2^log2m registers offered every member of S (stream-lib's HyperLogLog.cardinality over MurmurHash.hash(value), as
 * DistinctCountHLLAggregationFunction computes it): the registers depend only on S, so every route, schedule and knob gives
 * the same estimate.  An empty S gives 0.  Several DISTINCTCOUNTHLLs, DISTINCTCOUNTs, DISTINCTSUMs and DISTINCTAVGs over one
 * column share one bitset; DISTINCTCOUNTHLLs with the same log2m share one estimate.
 * Results: pb200_result_agg gives the estimate in the long column and the same value as a double in the double column;
 * pb200_result_distinct the dictId set, decoded on the first call for the aggregation (a caller that reads only the
 * estimates never pays for the sets); ORDER BY and HAVING compare the double.
 * PB200_E_INVALID: a log2m that is not integral or is outside 0..30 (the reference's range).
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): log2m outside 4..12, raw columns streamed as 32-bit values, a
 * STRING dictionary with an entry that is not valid UTF-8, the DISTINCTCOUNT bitset budget; a PB200_Q_MERGE_SEGMENTS
 * submission needs the column's dictionary to be the same in every segment.  Not reduced across GPUs on the device. */

/* ---- selection: SELECT columns WHERE ... [ORDER BY columns] LIMIT n (SelectionOnlyOperator, SelectionOrderByOperator) -- */
/* Without order items: per segment, the first `limit` matching docs in doc-id order with the values of the selected
 * columns.  With PB200_Q_MERGE_SEGMENTS one result: the segments are taken in submission order and each contributes a
 * doc-order prefix of its matches (one of the outcomes the reference's selection-only combine can produce).
 * With order items: per segment, the top `limit` rows by the order columns' values, ties by doc id ascending (the
 * reference keeps the lower doc ids among equal keys); merged, the segments' tops are merged by value with ties broken by
 * (segment index in the submission, doc id).  Value order: dictionary order (dictId order inside a segment, value order
 * across segments; STRING: the dictionary's byte order), numeric order for raw INT / FLOAT columns; NaN and -0.0 are out
 * of scope.  Order columns need not be selected.
 * Columns may have different dictionaries in different segments.  A selected column comes back typed: INT / LONG / STRING
 * as int64 (STRING: the dictId, looked up in the dictionary of the row's segment), FLOAT / DOUBLE as double; raw INT /
 * FLOAT columns read their 32-bit values.  limit 0 returns no rows, only the statistics; limit above
 * PB200_MAX_SELECT_LIMIT, or more than 65 535 segments, is PB200_E_UNSUPPORTED; more than PB200_MAX_ORDER_BY order items
 * is PB200_E_INVALID.
 * Statistics (device semantics): num_docs_scanned = matched docs in the doc range that was scanned.  Without ORDER BY a
 * segment is first scanned over a prefix of whole tiles (at least 2^20 docs); only where that prefix holds fewer than
 * `limit` matches is the whole segment scanned, and then the whole segment is the scanned range.  With ORDER BY every doc
 * is scanned.  num_entries_scanned_in_filter = scanned docs x scan leaves; num_entries_scanned_post_filter = rows x
 * num_columns.  device_ms = the scan launches; pb200_last_phases gives the host time of the scan and select phases. */
#define PB200_MAX_SELECT_LIMIT 1000000
typedef struct {
  int32_t column;     /* column id */
  int32_t descending; /* 0: ASC, else DESC */
} pb200_select_order;
typedef struct {
  int32_t num_columns;
  const int32_t* columns;   /* column ids, in output order */
  int32_t num_order_items;  /* 0 .. PB200_MAX_ORDER_BY */
  pb200_select_order order[PB200_MAX_ORDER_BY];
  int64_t limit;            /* 0 .. PB200_MAX_SELECT_LIMIT */
} pb200_selection;
/* filter_only: the filter part of a pb200_query (num_filter_nodes, filter, PB200_Q_PER_SEGMENT_FILTER in its flags; its
 * group-by and aggregation fields are ignored).  flags: PB200_Q_MERGE_SEGMENTS or 0.  Writes num_segments results (one
 * when merged). */
int32_t pb200_execute_selection(pb200_ctx* ctx, const pb200_query* filter_only, const pb200_selection* selection,
                                pb200_segment* const* segments, int32_t num_segments, int32_t flags, pb200_result** results);
/* The rows of a selection result: doc ids and the index (in the submission) of each row's segment, and per selected
 * column a pointer to `rows` int64 or double values (see pb200_execute_selection).  Any output may be NULL; columns
 * receives num_columns pointers.  Valid until pb200_result_free(result).  PB200_E_INVALID for other results. */
int32_t pb200_result_selection(const pb200_result* result, int64_t* rows, const int32_t** doc_ids,
                               const int32_t** segment_index, const void** columns);

/* ---- DISTINCT: SELECT DISTINCT columns WHERE ... [ORDER BY columns] LIMIT n (DistinctOperator) -------------------- */
/* `distinct` is a pb200_selection: its columns are the DISTINCT columns (1..8), its order items name some of them (an
 * order item on any other column is PB200_E_INVALID).  A row is one distinct tuple of the columns' values over the
 * matching docs, and carries the tuple's FIRST OCCURRENCE: the doc id and segment index of the first matching doc holding
 * it, in (segment index in the submission, doc id) order.
 * Without order items: the first `limit` tuples in order of first occurrence.  With order items: the top `limit` tuples
 * by the items (value order as for pb200_execute_selection, DESC reversed), ties by first occurrence ascending.
 * Per segment (flags 0) each result uses that segment's docs only; PB200_Q_MERGE_SEGMENTS gives one result over all
 * segments and needs every DISTINCT column to have one dictionary across them (bind the segments to a domain), otherwise
 * PB200_E_UNSUPPORTED as for group-by merges.
 * Values come back as for a selection (read them with pb200_result_selection): INT / LONG / STRING (the dictId) as
 * int64, FLOAT / DOUBLE as double.  PB200_E_UNSUPPORTED (the caller runs the stock operator): a column without dictIds
 * (a raw column streamed as 32-bit values; a raw column whose dictionary was synthesised at load is accepted), a key
 * space (product of the columns' cardinalities) above 2^24 for one result, tables above 2^27 entries over all results of
 * the call, more than 8 columns, limit above PB200_MAX_SELECT_LIMIT, more than 65 535 segments.
 * Statistics (device semantics): num_docs_scanned = matched docs in the scanned range; num_entries_scanned_in_filter =
 * scanned docs x scan leaves; num_entries_scanned_post_filter = matched docs x num_columns (every matched doc's key is
 * read).  Without order items each segment is first scanned over selection's prefix (at least 2^20 docs, whole tiles);
 * a result is final when at least `limit` of its tuples first occur before the prefix end of its earliest truncated
 * segment, otherwise its truncated segments are scanned in full.  With order items every doc is scanned.
 * device_ms = the scan launches and the table builds; pb200_last_phases reports PLAN, DEVICE_WAIT, EXTRACT and TOTAL. */
int32_t pb200_execute_distinct(pb200_ctx* ctx, const pb200_query* filter_only, const pb200_selection* distinct,
                               pb200_segment* const* segments, int32_t num_segments, int32_t flags, pb200_result** results);

/* ---- derived columns: single-column transforms (DATETRUNC, date parts, time conversions, arithmetic with literals) ---- */
/* A function of one dictionary column is a function of its dictId: the program is evaluated once per entry of the
 * column's (device) dictionary, the distinct results sorted into a new dictionary, and the forward index re-encoded
 * through dictId -> rank once.  The result is an ordinary dictionary column: every query route takes it unchanged.
 * Programs are POSTFIX: leaves push a value (the column, or a literal), operations pop their operands and push one value.
 * Semantics (DESIGN.md section 3.8):
 *   PLUS, MINUS, TIMES, DIVIDE, MOD (x, y), FLOOR, CEIL, ABS (x)  operands as doubles, one round-to-nearest operation each,
 *                                       MOD = C fmod (Java %), x / 0 = +-inf or NaN; result DOUBLE
 *   DATETRUNC (x)    i = unit | inUnit << 8 | outUnit << 16 (PB200_DT_* unit, PB200_TU_* time units): ms = inUnit.toMillis(x)
 *                    floored to the start of the UTC unit (WEEK: ISO, Monday), then outUnit.convert(ms, MILLISECONDS); LONG
 *   YEAR .. MILLISECOND (x)  UTC calendar fields of epoch ms x (proleptic Gregorian; WEEK is the ISO week, DAYOFWEEK
 *                    1 = Monday); INT
 *   TIMECONVERT (x)  i = inUnit | outUnit << 8: outUnit.convert(x, inUnit) (toward 0 when coarser, saturated when finer); LONG
 *   TOEPOCH (x), TOEPOCH_BUCKET / _ROUNDED (x, n)  i = PB200_TU_SECONDS .. DAYS: x ms in that unit (toward 0), / n,
 *                    (/ n) * n; n a positive LONG literal; LONG
 * Time functions take INT / LONG operands only (the column or another time function).  DATETRUNC and the calendar fields
 * refuse a dictionary holding an instant beyond +-2^53 ms (after the input-unit conversion). */
enum { PB200_T_COLUMN = 0, PB200_T_LONG_LITERAL = 1, PB200_T_DOUBLE_LITERAL = 2,
       PB200_T_PLUS = 3, PB200_T_MINUS = 4, PB200_T_TIMES = 5, PB200_T_DIVIDE = 6, PB200_T_MOD = 7,
       PB200_T_FLOOR = 8, PB200_T_CEIL = 9, PB200_T_ABS = 10, PB200_T_DATETRUNC = 11,
       PB200_T_YEAR = 12, PB200_T_QUARTER = 13, PB200_T_MONTH = 14, PB200_T_WEEK = 15, PB200_T_DAY = 16,
       PB200_T_DAYOFWEEK = 17, PB200_T_DAYOFYEAR = 18, PB200_T_HOUR = 19, PB200_T_MINUTE = 20, PB200_T_SECOND = 21,
       PB200_T_MILLISECOND = 22, PB200_T_TIMECONVERT = 23, PB200_T_TOEPOCH = 24, PB200_T_TOEPOCH_BUCKET = 25,
       PB200_T_TOEPOCH_ROUNDED = 26 };
enum { PB200_TU_NANOSECONDS = 0, PB200_TU_MICROSECONDS = 1, PB200_TU_MILLISECONDS = 2, PB200_TU_SECONDS = 3,
       PB200_TU_MINUTES = 4, PB200_TU_HOURS = 5, PB200_TU_DAYS = 6 };
enum { PB200_DT_MILLISECOND = 0, PB200_DT_SECOND = 1, PB200_DT_MINUTE = 2, PB200_DT_HOUR = 3, PB200_DT_DAY = 4,
       PB200_DT_WEEK = 5, PB200_DT_MONTH = 6, PB200_DT_QUARTER = 7, PB200_DT_YEAR = 8 };
typedef struct {
  int32_t op;        /* PB200_T_* */
  int32_t reserved;  /* 0 */
  int64_t i;         /* LONG literal, or the operation's units */
  double d;          /* DOUBLE literal */
} pb200_transform_op;
#define PB200_MAX_DERIVED_COLUMNS 32 /* derived columns per segment */

/* ---- aggregations over expressions of two or more columns: SUM / AVG / MIN / MAX(a * b) (DESIGN.md section 3.15) ---- */
/* One program per aggregation.  num_ops == 0: the aggregation reads its pb200_agg.column as usual.  Otherwise `ops` is a
 * POSTFIX program of the arithmetic operations above (PLUS, MINUS, TIMES, DIVIDE, MOD, FLOOR, CEIL, ABS, LONG / DOUBLE
 * literals; at most 16 operations) with 2 .. 8 PB200_T_COLUMN leaves whose `i` is a column id (the same column may
 * appear twice), and pb200_agg.column is ignored. */
typedef struct {
  int32_t num_ops;
  int32_t reserved;                 /* 0 */
  const pb200_transform_op* ops;
} pb200_expr_program;
/* pb200_execute_agg_args with a pb200_expr_program per aggregation (exprs == NULL: exactly pb200_execute_agg_args).
 * Semantics per matched row: every leaf value becomes a double (INT / LONG converted, LONG beyond 2^53 rounded to
 * nearest), every operation is one IEEE-754 round-to-nearest step without FMA, MOD is fmod, x / 0 is +-inf or NaN.
 * SUM adds the row values in IEEE arithmetic in any order (NaN when a row is NaN or both infinities occur; an exact zero
 * is +0.0); AVG is that sum over the group's COUNT(*); MIN / MAX are the first / last row value in Double.compare order
 * (-0.0 before 0.0, NaN after +inf), +inf / -inf without rows.  COUNT over a program is COUNT(*).  Leaves are INT, LONG,
 * FLOAT or DOUBLE columns with a device dictionary or raw INT / FLOAT 32-bit values; each segment reads them through its
 * own dictionary, so PB200_Q_MERGE_SEGMENTS needs no shared dictionary for them.
 * Results: pb200_result_agg gives the value in the double column (SUM / AVG: the sum, with the count in the long column;
 * MIN / MAX dictId -1); ORDER BY and HAVING compare it like a DOUBLE column's.
 * PB200_E_INVALID: a malformed program or a column id out of range.  PB200_E_UNSUPPORTED (the caller runs the stock
 * operator): a STRING leaf or one without dictIds or raw 32-bit values, a time function in the program, fewer than two
 * or more than 8 column leaves, a function other than SUM / AVG / MIN / MAX / COUNT over a program, and with GROUP BY
 * PB200_Q_DEFER_FINALIZE or reduce_world > 1. */
int32_t pb200_execute_exprs(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                            const pb200_having* having, const pb200_expr_program* exprs, pb200_segment* const* segments,
                            int32_t num_segments, pb200_result** results);

/* ---- CASE WHEN inside expression programs: SUM(CASE WHEN s = 'x' THEN b ELSE 0 END) (DESIGN.md section 3.19) ------- */
/* Five more program operations, accepted by pb200_execute_exprs_cond only:
 *   COND        a leaf: condition `i` of the call's pb200_expr_conds holds for the row (1.0) or not (0.0)
 *   AND, OR (x, y), NOT (x)   over conditions (COND, AND, OR, NOT results) only
 *   CASE (c, v, e)            v when the condition c holds, else e; v and e are values (never conditions).  A k-WHEN
 *                             CASE is k nested CASE nodes: c1 v1 c2 v2 e CASE CASE.
 * Branches are evaluated before one is selected: they have no side effects in double arithmetic.  The program's result
 * is a value.  COND leaves count as column leaves (at most 8 with the PB200_T_COLUMN leaves; one suffices). */
enum { PB200_T_COND = 27, PB200_T_AND = 28, PB200_T_OR = 29, PB200_T_NOT = 30, PB200_T_CASE = 31 };
/* A condition is a set of dictIds of one column, resolved by the caller per segment: a dictId range or a bitset. */
enum { PB200_COND_RANGE = 0, PB200_COND_BITSET = 1 };
#define PB200_MAX_EXPR_CONDS 32 /* conditions of one call */
typedef struct {
  int32_t column;           /* a column with dictIds (a device dictionary, STRING included) in every segment */
  int32_t kind;             /* PB200_COND_* */
  /* two per segment, in submission order: RANGE: the dictIds [args[2s], args[2s+1]) (0 <= lo <= hi <= cardinality);
     BITSET: the first word of segment s's bitset in pb200_expr_conds.words and its length in words (at least
     ceil(cardinality / 32)); bit j of word w is dictId 32 * w + j.  A bound segment's ids are the domain's. */
  const int64_t* args;
} pb200_expr_cond;
typedef struct {
  int32_t num_conds;        /* 1 .. PB200_MAX_EXPR_CONDS */
  int32_t reserved;         /* 0 */
  const pb200_expr_cond* conds;
  int64_t num_words;        /* bitset words (0 when every condition is a RANGE) */
  const uint32_t* words;    /* host pointer */
} pb200_expr_conds;
/* pb200_execute_exprs whose programs may hold COND / AND / OR / NOT / CASE (conds == NULL: exactly pb200_execute_exprs).
 * A condition's dictIds are read through the same forward index as a value leaf, once per distinct condition column
 * and row; the device never compares values, so the caller decides what a condition means.
 * PB200_E_INVALID as well: a condition index out of range, an operand of the wrong kind (a condition where a value
 * belongs or the reverse), a malformed condition table (range or bitset outside its segment's cardinality or words).
 * PB200_E_UNSUPPORTED as well: a condition column without dictIds (raw 32-bit values). */
int32_t pb200_execute_exprs_cond(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                                 const pb200_having* having, const pb200_expr_program* exprs, const pb200_expr_conds* conds,
                                 pb200_segment* const* segments, int32_t num_segments, pb200_result** results);

/* ---- predicates on expressions of two or more columns: WHERE a > b, WHERE price * qty > 1000 (DESIGN.md section 3.16) -- */
/* One predicate on the value of a pb200_expr_program (the rules of pb200_execute_exprs: 2 .. 8 column leaves by column
 * id, every leaf a double, every operation one IEEE-754 step without FMA).  The value is compared as a DOUBLE with Java's
 * <, > and ==: NaN matches only NEQ and NOT_IN, 0.0 matches both zeros.  RANGE takes lo / hi with `flags` as
 * pb200_filter_node.raw_flags (bit0 lower unbounded, bit1 upper unbounded, bit2 lower exclusive, bit3 upper exclusive);
 * EQ / NEQ compare values[0], IN / NOT_IN values[0 .. num_values). */
enum { PB200_EXPR_EQ = 0, PB200_EXPR_NEQ = 1, PB200_EXPR_IN = 2, PB200_EXPR_NOT_IN = 3, PB200_EXPR_RANGE = 4 };
#define PB200_MAX_EXPR_VALUES 1024 /* values of one EQ / NEQ / IN / NOT_IN predicate */
typedef struct {
  pb200_expr_program program;
  int32_t op;                 /* PB200_EXPR_* */
  int32_t flags;              /* RANGE: raw_flags bits; 0 otherwise */
  double lo, hi;              /* RANGE bounds */
  int32_t num_values;         /* EQ / NEQ: 1; IN / NOT_IN: 1 .. PB200_MAX_EXPR_VALUES; RANGE: 0 */
  int32_t reserved;           /* 0 */
  const double* values;       /* host pointer */
} pb200_expr_predicate;
/* The doc set of each predicate on each segment, as device masks for PB200_F_DOC_MASK | PB200_NODE_IDS_ON_DEVICE leaves:
 * masks[p * num_segments + s] is predicate p on segment s, bit j of word w = doc 32 * w + j, words past the segment's
 * docs zero, in the padded layout pb200_doc_mask_upload makes.  Every doc of every segment is evaluated, in one launch;
 * the call synchronises once before it returns, so the masks can be read from any stream.  Each segment reads the leaves
 * through its own dictionary (a bound segment through the domain's, which holds the same values), so merged submissions
 * need no shared dictionary for them.  Release every mask with pb200_doc_mask_free.  On an error no mask is returned.
 * PB200_E_INVALID: a malformed program, an unknown op, a column id out of range, bad value counts or flags.
 * PB200_E_UNSUPPORTED (the caller runs the stock operator): a STRING leaf or one without dictIds or raw 32-bit values, a
 * time function in the program, fewer than two or more than 8 column leaves, more than PB200_MAX_EXPR_VALUES values. */
int32_t pb200_expr_doc_masks(pb200_ctx* ctx, int32_t num_predicates, const pb200_expr_predicate* predicates,
                             pb200_segment* const* segments, int32_t num_segments, uint32_t** masks);
/* Adds the derived column `program(source_column)` to the segment and returns its column id (the next free id, after
 * the registered and earlier derived columns).  The source must carry dictIds: INT / LONG / FLOAT / DOUBLE dictionaries,
 * raw columns whose dictionary was synthesised at load, or a column bound to a domain (the program then runs over the
 * domain's dictionary, so every bound segment derives the same dictionary, and pb200_segment_local_ids gives the derived
 * ids this segment holds).  The new column has no inverted index, is never sorted, and counts in
 * pb200_segment_device_bytes.  Queries already running on the segment are not disturbed: no existing column moves.
 * PB200_E_UNSUPPORTED: STRING or raw 32-bit sources, a program outside the supported set, an instant beyond +-2^53 ms,
 * more than PB200_MAX_DERIVED_COLUMNS derived columns.  PB200_E_INVALID: a malformed program. */
int32_t pb200_segment_derive_column(pb200_ctx* ctx, pb200_segment* segment, int32_t source_column, int32_t num_ops,
                                    const pb200_transform_op* ops, int32_t* new_column);

/* ---- results (the data a GroupByResultsBlock / AggregationResultsBlock is built from) ---------------------------- */
enum { PB200_REGIME_NONE = 0, PB200_REGIME_ARRAY = 1, PB200_REGIME_INT_MAP = 2, PB200_REGIME_LONG_MAP = 3,
       PB200_REGIME_ARRAY_MAP = 4 };

typedef struct {
  int32_t num_groups;          /* -1: aggregation only (one row) */
  int32_t num_group_by;
  int32_t num_aggs;
  int32_t regime;              /* which key-holder regime the reference would have used (informational) */
  int32_t groups_limit_reached;
  int32_t reserved;            /* bit 0: group-by row counts were carried inside an INT sum's reductions (informational);
                                  bit 1 (PB200_Q_DEFER_FINALIZE results): that sum's field is NOT provably safe for the
                                  cross-GPU reduce -- every rank must run the query again with PB200_Q_NO_COUNT_CARRIER;
                                  bit 2: the int64 block of pb200_result_device_buffers ends with one extra element holding
                                  that verdict (0 / 1): SUM-all-reduce the block and every rank reads the agreed verdict there */
  /* ExecutionStatistics (core/operator/ExecutionStatistics.java) */
  int64_t num_docs_scanned;
  int64_t num_entries_scanned_in_filter; /* see DESIGN.md: device semantics = docs x scan leaves evaluated */
  int64_t num_entries_scanned_post_filter;
  int64_t num_total_docs;
  double device_ms;            /* CUDA-event time of the scan kernel(s) of this pb200_execute call */
} pb200_result_meta;

int32_t pb200_result_meta_get(const pb200_result* result, pb200_result_meta* meta);
/* group keys as dictIds, group-major [num_groups x num_group_by] (dictId -> value via Dictionary.getInternal on the
 * caller's side, as DictionaryBasedGroupKeyGenerator.getKeys does :577-605) */
int32_t pb200_result_group_keys(const pb200_result* result, int32_t* out);
/* aggregation `agg`: per group (or 1 row) the double intermediate (SUM, MIN, MAX, AVG's sum, COUNT as double) and the
 * long intermediate (COUNT, AVG's count, DISTINCTCOUNT's set size).  MIN/MAX of an empty input are +inf/-inf. */
int32_t pb200_result_agg(const pb200_result* result, int32_t agg, double* out_double, int64_t* out_long);
/* MIN/MAX as dictIds (dict-encoded columns; -1 when empty), for exact value lookup on the caller's side */
int32_t pb200_result_agg_dict_ids(const pb200_result* result, int32_t agg, int32_t* out);
/* DISTINCTCOUNT, DISTINCTSUM, DISTINCTAVG, DISTINCTCOUNTHLL: the dictId set of row `row` (ascending); returns the count
 * (or < 0 on error), writes <= capacity */
int64_t pb200_result_distinct(const pb200_result* result, int32_t agg, int32_t row, int32_t* out, int64_t capacity);
/* Everything of a result in ONE call (a JNI / ctypes round trip per accessor adds up when many small per-segment results
 * are read): keys [rows x num_group_by] (may be NULL), doubles / longs / dict_ids [num_aggs x rows] each (row-major by
 * aggregation; any may be NULL).  rows = num_groups, or 1 for an aggregation-only result. */
int32_t pb200_result_fetch(const pb200_result* result, int32_t* keys, double* doubles, int64_t* longs, int32_t* dict_ids);
/* Zero-copy face of the same data: pointers to the result's columns (group extraction leaves them in their final layout in
 * a pinned host block -- a JVM wraps them with NewDirectByteBuffer, numpy with frombuffer).  keys -> [rows x num_group_by];
 * doubles / longs / dict_ids -> arrays of num_aggs column pointers [rows] each; a NULL column means the neutral value
 * (0.0 / 0 / -1) for every row.  Valid until pb200_result_free(result). */
int32_t pb200_result_columns(const pb200_result* result, const int32_t** keys, const double** doubles, const int64_t** longs,
                             const int32_t** dict_ids);
int32_t pb200_result_free(pb200_result* result);

/* ---- multi-GPU combine support (dense group tables with shared dictionaries) ----------------------------------- */
/* Results with DISTINCTCOUNT bitsets or PERCENTILE histograms are refused (PB200_E_UNSUPPORTED).
 * Device pointers + element counts of the dense accumulator arrays of a merged group-by result, so that the caller's
 * collective layer (torch.distributed / NCCL) can all-reduce them in place across ranks:
 *   kind 0: int64 sums/counts (reduce SUM)   kind 1: double sums (SUM)   kind 2: uint32 max-encoded (reduce MAX)
 * After the collective, pb200_result_finalize() re-extracts the groups on the root rank. */
int32_t pb200_result_device_buffers(pb200_result* result, int32_t kind, void** device_ptr, int64_t* num_elements);
int32_t pb200_result_finalize(pb200_ctx* ctx, pb200_result* result);

/* Structural validation of one serialized RoaringBitmap (portable format) as pb200_segment_register applies it to every
 * posting list of an inverted index: containers inside the buffer, keys ascending, largest doc id < num_docs.  Pure host. */
int32_t pb200_roaring_validate(const void* bytes, uint64_t length, int64_t num_docs);

/* ---- resident doc-id sets for PB200_F_DOC_MASK | PB200_NODE_IDS_ON_DEVICE ------------------------------------------- */
int32_t pb200_doc_mask_upload(pb200_ctx* ctx, int32_t num_docs, const uint32_t* words, int64_t num_words /* >= ceil(num_docs/32) */,
                              uint32_t** device_mask);
int32_t pb200_doc_mask_free(pb200_ctx* ctx, uint32_t* device_mask);

/* ---- where a query's host time goes (diagnostics; thread-local, the calling thread's last pb200_execute) ------------- */
enum { PB200_PHASE_PLAN = 0, PB200_PHASE_LAUNCH = 1, PB200_PHASE_DEVICE_WAIT = 2, PB200_PHASE_RESULTS = 3,
       PB200_PHASE_EXTRACT = 4, PB200_PHASE_TOTAL = 5, PB200_NUM_PHASES = 6 };
int32_t pb200_last_phases(double* out_ms /* PB200_NUM_PHASES */);

/* ---- cross-GPU combine inside the library (NCCL over NVLink / NVSwitch; one process per GPU) ---------------------- */
/* NCCL is bound at run time (dlopen libnccl.so.2): everything else works without it.  Rank 0 creates the id, ships the
 * bytes to the other ranks over any transport (the JVM's own RPC, torch.distributed, a file), every rank calls
 * pb200_comm_init with its rank.  The reference merges per-server partial results by value on the JVM
 * (GroupByCombineOperator.java:130-146); with table-wide dictionaries the per-GPU group tables are element-wise mergeable. */
#define PB200_COMM_ID_BYTES 128
int32_t pb200_comm_unique_id(void* id_out /* PB200_COMM_ID_BYTES */);
int32_t pb200_comm_init(pb200_ctx* ctx, const void* id, int32_t rank, int32_t world_size);
int32_t pb200_comm_shutdown(pb200_ctx* ctx);
/* Every rank calls this with ITS deferred result (PB200_Q_MERGE_SEGMENTS | PB200_Q_DEFER_FINALIZE, reduce_world = world size)
 * of the same query: all table blocks are reduced into rank `root` in ONE NCCL group on the context's stream and the root
 * extracts the groups (the result is then read with the accessors; on the other ranks it stays empty -- free it).
 * *retry = 1 on EVERY rank when a count-carrying sum was not provably safe for the reduce: all ranks free the result and
 * execute again with PB200_Q_NO_COUNT_CARRIER.  It is a COLLECTIVE: all ranks must call it for the same queries in the same
 * order (calls of one context are serialised internally; concurrent queries need an agreed order across ranks, e.g. the
 * broker's request id).  Aggregation-only results (num_groups < 0) are combined too (sums / counts add, MIN / MAX by value;
 * an INT SUM / AVG adds the ranks' exact int64 sums and rounds the total once, as the group-by tables do). */
int32_t pb200_result_combine(pb200_ctx* ctx, pb200_result* result, int32_t root, int32_t* retry);
/* Aggregation-only result, SUM / AVG over an INT column: *out = the exact int64 sum the double column holds rounded
 * (after pb200_result_combine on the root: the whole table's).  Returns 1 when written, 0 when aggregation `agg` has no
 * exact sum (another function, a sum accumulated in double, a star-tree answer, a group-by result), < 0 on error.  A
 * caller that adds results across processes adds these and rounds once: rounded sums beyond 2^53 do not add exactly. */
int32_t pb200_result_exact_sum(const pb200_result* result, int32_t agg, int64_t* out);

/* ---- synthetic segments (SegmentIndexCreationDriverImpl stand-in for benchmarks; bytes are Pinot's formats) ---- */
typedef struct {
  int32_t cardinality;   /* dictionary = { value_base + value_step * i } (sorted INT) */
  int32_t value_base;
  int32_t value_step;
  int32_t with_inverted; /* build the bitmap inverted index on the device too */
  uint64_t seed;         /* dictId(doc) = mix64(seed, doc) % cardinality */
} pb200_synth_col;

/* Generates `num_columns` dict-encoded INT columns of `num_docs` rows directly in HBM, byte-identical to what
 * FixedBitSVForwardIndexWriter / SegmentDictionaryCreator would have written for the same values, and registers them
 * as a segment. */
int32_t pb200_synth_segment(pb200_ctx* ctx, const char* segment_name, int32_t num_docs, int32_t num_columns,
                            const pb200_synth_col* columns, pb200_segment** segment);
/* Copies a column's index bytes back to the host (tests: compare against the oracle's writer; bench: host-resident
 * copy for the end-to-end arm).  which: 0 fwd, 1 dict, 2 inv.  Returns bytes (or needed size when out == NULL). */
int64_t pb200_segment_read_index(pb200_ctx* ctx, const pb200_segment* segment, int32_t column, int32_t which,
                                 void* out, uint64_t capacity);
/* Column facts of a registered segment: {fwd_kind, stored_type, bits, cardinality, has_inverted, fwd_bytes}. */
int32_t pb200_segment_column_info(const pb200_segment* segment, int32_t column, int64_t out[6]);

#ifdef __cplusplus
}
#endif
#endif /* PINOT_B200_H_ */
