// pb200_aggfn.h -- what each aggregation function (PB200_AGG_*) is: one descriptor per code for the host code that
// plans, checks, names and lays out aggregations, and the family predicates device code calls.  The Python package keeps
// the same facts in pinot_b200/query.py (AGG_FUNCTIONS); tests/test_aggfn_cpu.py holds the two to each other.
// Plain C++ when not compiled by nvcc (CPU tests compile it with g++).
#pragma once
#include "../../include/pinot_b200.h"

#ifdef __CUDACC__
#define PB200_HD __host__ __device__ __forceinline__
#else
#define PB200_HD inline
#endif

namespace pb200 {

PB200_HD bool is_moments_fn(int fn) { return fn >= PB200_AGG_VARPOP && fn <= PB200_AGG_STDDEVSAMP; }
PB200_HD bool is_distinct_value_fn(int fn) { return fn == PB200_AGG_DISTINCTSUM || fn == PB200_AGG_DISTINCTAVG; }
PB200_HD bool is_hll_fn(int fn) { return fn == PB200_AGG_DISTINCTCOUNTHLL; }
// a function that reads a DISTINCTCOUNT bitset it may not own (ScanPlan::ds_rep): the scan builds the set, a finalize after
// the scan turns it into the function's value
PB200_HD bool reads_distinct_set(int fn) { return is_distinct_value_fn(fn) || is_hll_fn(fn); }
PB200_HD bool is_withtime_fn(int fn) { return fn == PB200_AGG_FIRSTWITHTIME || fn == PB200_AGG_LASTWITHTIME; }

// the argument an aggregation takes besides its column
enum AggArg { ARG_NONE = 0, ARG_PERCENTILE = 1, ARG_LOG2M = 2, ARG_TIME_COLUMN = 3 };

struct AggFn {
  int code;              // PB200_AGG_*
  const char* name;      // upper case, as messages name it
  const char* family;    // as a refusal shared by the family names it ("VAR/STDDEV", "MIN/MAX", ...)
  bool dict_ids;         // reads its column's dictIds: a merged submission needs one dictionary for that column
  int arg;               // AggArg
  bool filter_clause;    // runs in a query with FILTER (WHERE ...) clauses (they run as one submission per clause)
  const char* datatable;          // DataTable column type of its intermediate, or nullptr: not written, ...
  const char* datatable_refusal;  // ... for this reason
  bool long_col, ids_col;  // the extraction lays out a long / a dictId column beside the double
};

// the reference's intermediates without a DataTable type here: a DoubleArrayList of values, a VarianceTuple, a (value,
// time) pair object, stream-lib's serialized HyperLogLog registers
constexpr const char *kNoDtPercentile = "PERCENTILE intermediates are not written as DataTable objects",
                     *kNoDtMoments = "VAR/STDDEV intermediates are not written as DataTable objects",
                     *kNoDtWithTime = "FIRST/LASTWITHTIME intermediates are not written as DataTable objects",
                     *kNoDtHll = "DISTINCTCOUNTHLL is not written as a server DataTable (the reference's HyperLogLog bytes are not restated)",
                     *kNoDtCase = "an aggregation over CASE is not written as a server DataTable (the reference's spelling of CASE is not restated)";

// FIRST/LASTWITHTIME: the data column's dictionary is checked with the time column's (plan_scan), not through dict_ids
constexpr AggFn kAggFns[] = {
  {PB200_AGG_COUNT, "COUNT", "COUNT", false, ARG_NONE, true, "LONG", nullptr, true, false},
  {PB200_AGG_SUM, "SUM", "SUM/AVG", false, ARG_NONE, true, "DOUBLE", nullptr, true, false},
  {PB200_AGG_MIN, "MIN", "MIN/MAX", true, ARG_NONE, true, "DOUBLE", nullptr, false, true},
  {PB200_AGG_MAX, "MAX", "MIN/MAX", true, ARG_NONE, true, "DOUBLE", nullptr, false, true},
  {PB200_AGG_AVG, "AVG", "SUM/AVG", false, ARG_NONE, true, "OBJECT", nullptr, true, false},
  {PB200_AGG_DISTINCTCOUNT, "DISTINCTCOUNT", "DISTINCTCOUNT", true, ARG_NONE, true, "OBJECT", nullptr, true, false},
  {PB200_AGG_PERCENTILE, "PERCENTILE", "PERCENTILE", true, ARG_PERCENTILE, false, nullptr, kNoDtPercentile, true, true},
  {PB200_AGG_VARPOP, "VARPOP", "VAR/STDDEV", true, ARG_NONE, false, nullptr, kNoDtMoments, true, false},
  {PB200_AGG_VARSAMP, "VARSAMP", "VAR/STDDEV", true, ARG_NONE, false, nullptr, kNoDtMoments, true, false},
  {PB200_AGG_STDDEVPOP, "STDDEVPOP", "VAR/STDDEV", true, ARG_NONE, false, nullptr, kNoDtMoments, true, false},
  {PB200_AGG_STDDEVSAMP, "STDDEVSAMP", "VAR/STDDEV", true, ARG_NONE, false, nullptr, kNoDtMoments, true, false},
  {PB200_AGG_FIRSTWITHTIME, "FIRSTWITHTIME", "FIRST/LASTWITHTIME", false, ARG_TIME_COLUMN, false, nullptr, kNoDtWithTime, true, true},
  {PB200_AGG_LASTWITHTIME, "LASTWITHTIME", "FIRST/LASTWITHTIME", false, ARG_TIME_COLUMN, false, nullptr, kNoDtWithTime, true, true},
  {PB200_AGG_DISTINCTSUM, "DISTINCTSUM", "DISTINCTSUM/DISTINCTAVG", true, ARG_NONE, false, "OBJECT", nullptr, true, false},
  {PB200_AGG_DISTINCTAVG, "DISTINCTAVG", "DISTINCTSUM/DISTINCTAVG", true, ARG_NONE, false, "OBJECT", nullptr, true, false},
  {PB200_AGG_DISTINCTCOUNTHLL, "DISTINCTCOUNTHLL", "DISTINCTCOUNTHLL", true, ARG_LOG2M, false, nullptr, kNoDtHll, true, false},
};
constexpr int kNumAggFns = (int)(sizeof kAggFns / sizeof kAggFns[0]);

constexpr bool agg_fns_indexed_by_code(int i = 0) { return i == kNumAggFns || (kAggFns[i].code == i && agg_fns_indexed_by_code(i + 1)); }
static_assert(agg_fns_indexed_by_code(), "kAggFns[i] must describe PB200_AGG_* code i");
static_assert(kAggFns[kNumAggFns - 1].code == PB200_AGG_DISTINCTCOUNTHLL, "kAggFns must end at the last PB200_AGG_* code");

// the descriptor of code fn; nullptr for an unknown code
inline const AggFn* agg_fn(int fn) { return fn >= 0 && fn < kNumAggFns ? &kAggFns[fn] : nullptr; }

// The checks of an aggregation's argument (a its position in the query), the same for the device planner and the host
// layer; each returns PB200_OK or the PB200_E_* code with the message set.
// PERCENTILE: PercentileAggregationFunction takes 0 <= p <= 100.
int check_percentile(double p, int a);
// DISTINCTCOUNTHLL: log2m none or 0 (the default 8) or an integer the reference accepts (0..30), accelerated in
// kHllMinLog2m..kHllMaxLog2m (the registers fit the finalize's shared memory); sets *log2m.
int hll_log2m(double arg, int a, int* log2m);

}  // namespace pb200
