// datatable.cpp -- the server -> broker wire format of a group-by / aggregation result: DataTableImplV4 bytes.
//
// In the reference the combined results block of a server is serialised by GroupByResultsBlock.getDataTable()
// (core/operator/blocks/results/GroupByResultsBlock.java:186-236) / AggregationResultsBlock.getDataTable() through
// DataTableBuilderV4 (core/common/datatable/DataTableBuilderV4.java, BaseDataTableBuilder.java:66-131) into the layout of
// pinot-common/.../datatable/DataTableImplV4.java:49-81,422-518:
//
//   13 big-endian ints: VERSION(4) NUM_ROWS NUM_COLUMNS, then (start, length) of EXCEPTIONS, DICTIONARY_MAP, DATA_SCHEMA,
//   FIXED_SIZE_DATA, VARIABLE_SIZE_DATA;  the five sections;  METADATA length + METADATA section.
//     exceptions     int n (= 0 here)
//     dictionary map int n, then per string: int length, UTF-8 bytes                       (:375-391)
//     data schema    int n, n x (int length, name), n x (int length, ColumnDataType name)    (common/utils/DataSchema.java:118-143)
//     fixed size     row major, column offsets by stored type: INT / FLOAT / STRING(dictionary id) 4 bytes, LONG / DOUBLE 8,
//                    OBJECT 8 = (position in the variable section, length)                    (DataTableUtils.java:41-65)
//     variable size  per OBJECT value: int ObjectSerDeUtils.ObjectType, then its bytes -- AvgPair(4) = double sum + long
//                    count (segment-local/customobject/AvgPair.java:57-62); DISTINCTCOUNT value sets IntSet(9) /
//                    LongSet(15) / FloatSet(16) / DoubleSet(17) / StringSet(18) = int size + values
//                    (core/common/ObjectSerDeUtils.java:119-137,926-1075)
//     metadata       int n, per entry: int MetadataKey id, then long / int big-endian or (int length, UTF-8)  (:531-560;
//                    ids: DataTable.java:105-142)
//
// The rows come from a pb200_result (merged over the server's segments by the device-side combine): group keys are
// decoded through the (domain) dictionaries of the segment, intermediates are COUNT -> LONG, SUM / MIN / MAX -> DOUBLE,
// AVG -> OBJECT(AvgPair), DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG -> OBJECT(value set) --
// AggregationFunction.getIntermediateResultColumnType().
// A JVM wraps these bytes with DataTableFactory.getDataTable(ByteBuffer) instead of building Key / Record objects.
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "host_internal.h"

using pb200::set_error;
using namespace pb200h;

namespace {

struct Out {
  std::vector<unsigned char> b;
  void i32(int32_t v) { for (int s = 24; s >= 0; s -= 8) b.push_back((unsigned char)((uint32_t)v >> s)); }
  void i64(int64_t v) { for (int s = 56; s >= 0; s -= 8) b.push_back((unsigned char)((uint64_t)v >> s)); }
  void f32(float v) { uint32_t u; memcpy(&u, &v, 4); i32((int32_t)u); }
  void f64(double v) { uint64_t u; memcpy(&u, &v, 8); i64((int64_t)u); }
  void str(const std::string& s) { i32((int32_t)s.size()); b.insert(b.end(), s.begin(), s.end()); }
  void bytes(const Out& o) { b.insert(b.end(), o.b.begin(), o.b.end()); }
};

const char* type_name(int t) {
  switch (t) {
    case PB200_INT: return "INT";
    case PB200_LONG: return "LONG";
    case PB200_FLOAT: return "FLOAT";
    case PB200_DOUBLE: return "DOUBLE";
    default: return "STRING";
  }
}

}  // namespace

extern "C" int64_t pb200h_result_to_datatable(const pb200h_query* q, const pb200h_segment* seg, const pb200_result* R,
                                              void* out, uint64_t capacity) {
  if (!q || !seg || !R) { set_error("null argument"); return PB200_E_INVALID; }
  pb200_result_meta meta;
  if (pb200_result_meta_get(R, &meta)) return PB200_E_INVALID;
  const int ngb = q->num_group_by, nagg = q->num_aggs;
  if (meta.num_group_by != ngb || meta.num_aggs != nagg) { set_error("result does not belong to this query"); return PB200_E_INVALID; }
  if (R->having.num_nodes > 0) {   // HAVING is the broker's: a server never sends rows it removed
    set_error("a result filtered by HAVING is final: it is not written as a server DataTable");
    return PB200_E_UNSUPPORTED;
  }
  // the reference's intermediates of the functions without a DataTable type: stream-lib's serialized HyperLogLog registers,
  // PERCENTILE's DoubleArrayList of values, a (value, time) pair object, a VarianceTuple
  for (int a : aggs_by_family(*q, {PB200_AGG_DISTINCTCOUNTHLL, PB200_AGG_PERCENTILE, PB200_AGG_FIRSTWITHTIME, PB200_AGG_VARPOP})) {
    const pb200::AggFn* d = pb200::agg_fn(q->aggs[a].function);
    if (!d) { set_error("unknown aggregation function %d", q->aggs[a].function); return PB200_E_INVALID; }
    if (!d->datatable) { set_error("%s", d->datatable_refusal); return PB200_E_UNSUPPORTED; }
  }
  const size_t rows = meta.num_groups < 0 ? 1 : (size_t)meta.num_groups;
  // ---- intermediates through the C-ABI accessors ----
  std::vector<int32_t> keys(rows * (size_t)std::max(ngb, 1));
  std::vector<double> dbl(rows * (size_t)nagg);
  std::vector<int64_t> lng(rows * (size_t)nagg);
  if (rows && pb200_result_fetch(R, ngb ? keys.data() : nullptr, dbl.data(), lng.data(), nullptr)) return PB200_E_INVALID;
  // ---- schema ----
  std::vector<const HostColumn*> key_cols(ngb), agg_cols(nagg, nullptr);
  std::vector<std::string> names, types;
  std::vector<int> width;  // bytes in the fixed section
  for (int g = 0; g < ngb; g++) {
    const int ci = seg->column_index(q->group_by[g]);
    if (ci < 0) { set_error("unknown group-by column '%s'", q->group_by[g]); return PB200_E_INVALID; }
    key_cols[g] = &seg->cols[ci].decode_column();
    names.push_back(q->group_by[g]);
    types.push_back(type_name(key_cols[g]->data_type));
    width.push_back((key_cols[g]->data_type == PB200_LONG || key_cols[g]->data_type == PB200_DOUBLE) ? 8 : 4);
  }
  for (int a = 0; a < nagg; a++) {
    const int fn = q->aggs[a].function;
    std::string arg = q->aggs[a].column ? q->aggs[a].column : "*";
    if (q->aggs[a].column) {
      const int ci = seg->column_index(q->aggs[a].column);
      std::vector<pb200_transform_op> ops;
      std::vector<std::string> leaves;
      // an expression over several columns: written like the function over a DOUBLE column, named by its canonical text
      if (ci < 0 && expression_function(fn) && is_multi_column_expression(q->aggs[a].column)) {
        std::vector<CaseCond> conds;
        if (int rc = compile_multi_expression(q->aggs[a].column, &arg, &ops, &leaves, &conds)) return rc;
        if (!conds.empty()) { set_error("%s", pb200::kNoDtCase); return PB200_E_UNSUPPORTED; }
      } else {
        if (ci < 0) { set_error("unknown aggregation column '%s'", q->aggs[a].column); return PB200_E_INVALID; }
        agg_cols[a] = &seg->cols[ci].decode_column();
      }
    }
    names.push_back(lower_fn_name(fn) + "(" + arg + ")");
    types.push_back(pb200::agg_fn(fn)->datatable);
    width.push_back(8);
  }
  // ---- rows ----
  Out fixed, var;
  std::map<std::string, int32_t> sdict;       // string -> dictionary id, ids in first-use order (DataTableBuilderV4.java:42-46)
  std::vector<std::string> sdict_rev;
  for (size_t r = 0; r < rows; r++) {
    for (int g = 0; g < ngb; g++) {
      const HostColumn& c = *key_cols[g];
      const int id = keys[r * ngb + g];
      if (id < 0 || id >= c.cardinality) { set_error("group key dictId %d out of range", id); return PB200_E_INVALID; }
      switch (c.data_type) {
        case PB200_INT: fixed.i32(c.get_int(id)); break;
        case PB200_LONG: fixed.i64(c.get_long(id)); break;
        case PB200_FLOAT: fixed.f32(c.get_float(id)); break;
        case PB200_DOUBLE: fixed.f64(c.get_double(id)); break;
        default: {
          const std::string s = c.get_string(id);
          auto it = sdict.find(s);
          if (it == sdict.end()) { it = sdict.emplace(s, (int32_t)sdict_rev.size()).first; sdict_rev.push_back(s); }
          fixed.i32(it->second);
        }
      }
    }
    for (int a = 0; a < nagg; a++) {
      const int fn = q->aggs[a].function;
      const double d = dbl[(size_t)a * rows + r];
      const int64_t l = lng[(size_t)a * rows + r];
      if (fn == PB200_AGG_COUNT) { fixed.i64(l); continue; }
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) { fixed.f64(d); continue; }
      // OBJECT: (position, length) in the fixed section; type code + bytes in the variable section
      Out obj;
      int type_code;
      if (fn == PB200_AGG_AVG) {
        type_code = 4;  // ObjectType.AvgPair
        obj.f64(d); obj.i64(l);
      } else {
        const HostColumn& c = *agg_cols[a];
        std::vector<int32_t> ids((size_t)l);
        if (l && pb200_result_distinct(R, a, (int32_t)r, ids.data(), l) != l) { set_error("distinct set of row %zu changed size", r); return PB200_E_INVALID; }
        obj.i32((int32_t)l);
        switch (c.data_type) {
          case PB200_INT: type_code = 9; for (int id : ids) obj.i32(c.get_int(id)); break;
          case PB200_LONG: type_code = 15; for (int id : ids) obj.i64(c.get_long(id)); break;
          case PB200_FLOAT: type_code = 16; for (int id : ids) obj.f32(c.get_float(id)); break;
          case PB200_DOUBLE: type_code = 17; for (int id : ids) obj.f64(c.get_double(id)); break;
          default: type_code = 18; for (int id : ids) obj.str(c.get_string(id)); break;
        }
      }
      fixed.i32((int32_t)var.b.size());
      fixed.i32((int32_t)obj.b.size());
      var.i32(type_code);
      var.bytes(obj);
    }
  }
  // ---- sections ----
  Out exceptions, dict, schema, metadata;
  exceptions.i32(0);
  const bool has_dict = std::find(types.begin(), types.end(), std::string("STRING")) != types.end();
  if (has_dict) { dict.i32((int32_t)sdict_rev.size()); for (auto& s : sdict_rev) dict.str(s); }
  schema.i32((int32_t)names.size());
  for (auto& n : names) schema.str(n);
  for (auto& t : types) schema.str(t);
  // metadata: the ExecutionStatistics the broker aggregates (InstanceResponseBlock.toDataTable / DataTable.MetadataKey ids)
  metadata.i32(5);
  metadata.i32(2); metadata.i64(meta.num_docs_scanned);                    // numDocsScanned (LONG)
  metadata.i32(3); metadata.i64(meta.num_entries_scanned_in_filter);       // numEntriesScannedInFilter
  metadata.i32(4); metadata.i64(meta.num_entries_scanned_post_filter);     // numEntriesScannedPostFilter
  metadata.i32(10); metadata.i64(meta.num_total_docs);                     // totalDocs
  metadata.i32(11); metadata.str(meta.groups_limit_reached ? "true" : "false");  // numGroupsLimitReached (STRING)
  Out head;
  int32_t off = 13 * 4;
  head.i32(4); head.i32((int32_t)rows); head.i32((int32_t)names.size());
  head.i32(off); head.i32((int32_t)exceptions.b.size()); off += (int32_t)exceptions.b.size();
  head.i32(off); head.i32((int32_t)dict.b.size()); off += (int32_t)dict.b.size();
  head.i32(off); head.i32((int32_t)schema.b.size()); off += (int32_t)schema.b.size();
  head.i32(off); head.i32((int32_t)fixed.b.size()); off += (int32_t)fixed.b.size();
  head.i32(off); head.i32((int32_t)var.b.size());
  const uint64_t total = head.b.size() + exceptions.b.size() + dict.b.size() + schema.b.size() + fixed.b.size() + var.b.size() + 4 + metadata.b.size();
  if (total > 0x7FFFFFFFull) { set_error("DataTable larger than 2 GB"); return PB200_E_UNSUPPORTED; }
  if (!out) return (int64_t)total;
  if (capacity < total) { set_error("buffer too small: need %llu bytes", (unsigned long long)total); return PB200_E_INVALID; }
  unsigned char* p = static_cast<unsigned char*>(out);
  auto put = [&](const Out& o) { if (!o.b.empty()) memcpy(p, o.b.data(), o.b.size()); p += o.b.size(); };
  put(head); put(exceptions); put(dict); put(schema); put(fixed); put(var);
  Out mlen; mlen.i32((int32_t)metadata.b.size());
  put(mlen); put(metadata);
  return (int64_t)total;
}
