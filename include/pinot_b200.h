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
                              3: pb200_comm_*, pb200_result_columns, doc masks, pb200h_query.agg_filter_* (the host query struct grew) */

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
 * DistinctCount}AggregationFunction.java). */
enum { PB200_AGG_COUNT = 0, PB200_AGG_SUM = 1, PB200_AGG_MIN = 2, PB200_AGG_MAX = 3, PB200_AGG_AVG = 4,
       PB200_AGG_DISTINCTCOUNT = 5 };

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
/* DISTINCTCOUNT: the dictId set of row `row` (ascending); returns the count (or < 0 on error), writes <= capacity */
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
/* Device pointers + element counts of the dense accumulator arrays of a merged group-by result, so that the caller's
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
 * broker's request id).  Aggregation-only results (num_groups < 0) are combined too (sums / counts add, MIN / MAX by value). */
int32_t pb200_result_combine(pb200_ctx* ctx, pb200_result* result, int32_t root, int32_t* retry);

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
