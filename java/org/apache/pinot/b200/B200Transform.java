/*
 * Single-column transform expressions (DATETRUNC, date parts, time conversions, arithmetic with literals) as derived
 * dictionary columns of the resident segment (pb200_segment_derive_column, include/pinot_b200.h; DESIGN.md section 3.8).
 * An expression is keyed by ExpressionContext.toString(), the canonical text the native host layer uses too.  The
 * program sent to the device is the postfix form of the expression tree; the derived dictionary comes back as its
 * big-endian bytes and serves group keys, DISTINCTCOUNT sets and predicate resolution on the JVM side.
 */
package org.apache.pinot.b200;

import java.nio.ByteBuffer;
import java.util.ArrayList;
import java.util.Arrays;
import java.util.HashMap;
import java.util.List;
import java.util.Locale;
import java.util.Map;
import java.util.Set;
import org.apache.pinot.common.request.context.ExpressionContext;
import org.apache.pinot.common.request.context.FunctionContext;
import org.apache.pinot.common.request.context.predicate.EqPredicate;
import org.apache.pinot.common.request.context.predicate.InPredicate;
import org.apache.pinot.common.request.context.predicate.NotEqPredicate;
import org.apache.pinot.common.request.context.predicate.NotInPredicate;
import org.apache.pinot.common.request.context.predicate.Predicate;
import org.apache.pinot.common.request.context.predicate.RangePredicate;
import org.apache.pinot.segment.spi.IndexSegment;
import org.apache.pinot.segment.spi.datasource.DataSource;
import org.apache.pinot.spi.data.FieldSpec.DataType;

final class B200Transform {
  private B200Transform() {
  }

  // PB200_T_* / PB200_TU_* / PB200_DT_* of include/pinot_b200.h
  private static final int T_COLUMN = 0, T_LONG_LITERAL = 1, T_DOUBLE_LITERAL = 2, T_DATETRUNC = 11, T_TIMECONVERT = 23,
      T_TOEPOCH = 24, T_TOEPOCH_BUCKET = 25, T_TOEPOCH_ROUNDED = 26;
  private static final List<String> TIME_UNITS =
      Arrays.asList("NANOSECONDS", "MICROSECONDS", "MILLISECONDS", "SECONDS", "MINUTES", "HOURS", "DAYS");
  private static final List<String> TRUNC_UNITS =
      Arrays.asList("MILLISECOND", "SECOND", "MINUTE", "HOUR", "DAY", "WEEK", "MONTH", "QUARTER", "YEAR");
  private static final Map<String, Integer> OPS = new HashMap<>();
  static {
    String[] arithmetic = {"plus", "minus", "times", "divide", "mod", "floor", "ceil", "abs"};
    for (int k = 0; k < arithmetic.length; k++) {
      OPS.put(arithmetic[k], 3 + k);
    }
    OPS.put("add", 3); OPS.put("sub", 4); OPS.put("mult", 5); OPS.put("div", 6);
    OPS.put("datetrunc", T_DATETRUNC);
    String[] calendar = {"year", "quarter", "month", "week", "day", "dayofweek", "dayofyear", "hour", "minute", "second",
        "millisecond"};
    for (int k = 0; k < calendar.length; k++) {
      OPS.put(calendar[k], 12 + k);
    }
    OPS.put("weekofyear", 15); OPS.put("dayofmonth", 16); OPS.put("dow", 17); OPS.put("doy", 18);
    OPS.put("timeconvert", T_TIMECONVERT);
    for (String u : new String[]{"seconds", "minutes", "hours", "days"}) {
      OPS.put("toepoch" + u, T_TOEPOCH);
      OPS.put("toepoch" + u + "bucket", T_TOEPOCH_BUCKET);
      OPS.put("toepoch" + u + "rounded", T_TOEPOCH_ROUNDED);
    }
  }

  /** The name a column or expression has on the device path: the identifier, or the expression's canonical text. */
  static String name(ExpressionContext e) {
    return e.getType() == ExpressionContext.Type.IDENTIFIER ? e.getIdentifier() : e.toString();
  }

  /**
   * A FUNCTION expression of the supported set over exactly one single-value, dictionary-encoded numeric column.  The
   * native side applies the type rules again and refuses (the stock operator runs) what this check lets through.
   */
  static boolean accepted(ExpressionContext e, IndexSegment segment) {
    if (e.getType() != ExpressionContext.Type.FUNCTION) {
      return false;
    }
    Set<String> columns = new java.util.HashSet<>();
    e.getColumns(columns);
    if (columns.size() != 1 || !supportedTree(e)) {
      return false;
    }
    DataSource ds = segment.getDataSource(columns.iterator().next());
    return ds != null && ds.getDictionary() != null && ds.getDataSourceMetadata().isSingleValue()
        && ds.getDataSourceMetadata().getDataType().getStoredType().isNumeric();
  }

  private static boolean supportedTree(ExpressionContext e) {
    if (e.getType() != ExpressionContext.Type.FUNCTION) {
      return true;
    }
    if (!OPS.containsKey(e.getFunction().getFunctionName())) {
      return false;
    }
    for (ExpressionContext a : e.getFunction().getArguments()) {
      if (!supportedTree(a)) {
        return false;
      }
    }
    return true;
  }

  /** The postfix program (op, i, d per step) of an accepted expression, and its source column. */
  static final class Program {
    final List<Integer> _op = new ArrayList<>();
    final List<Long> _i = new ArrayList<>();
    final List<Double> _d = new ArrayList<>();
    String _column;

    void add(int op, long i, double d) {
      _op.add(op);
      _i.add(i);
      _d.add(d);
    }
  }

  static Program compile(ExpressionContext e) {
    Program p = new Program();
    emit(e, p);
    return p;
  }

  private static String literal(ExpressionContext e) {
    return e.getLiteral().getStringValue();
  }

  private static void emitLiteral(String text, Program p) {
    // integral values are LONG literals however they are spelled (the native compiler does the same); -0.0 stays a double
    double d = Double.parseDouble(text);
    if (!Double.isInfinite(d) && d == Math.floor(d) && Math.abs(d) < 9.2e18 && !(d == 0 && 1 / d < 0)) {
      long i;
      try {
        i = Long.parseLong(text.trim());
      } catch (NumberFormatException ex) {
        i = (long) d;
      }
      p.add(T_LONG_LITERAL, i, 0.0);
    } else {
      p.add(T_DOUBLE_LITERAL, 0, d);
    }
  }

  private static void emit(ExpressionContext e, Program p) {
    switch (e.getType()) {
      case IDENTIFIER:
        p._column = e.getIdentifier();
        p.add(T_COLUMN, 0, 0.0);
        return;
      case LITERAL:
        emitLiteral(literal(e), p);
        return;
      default:
        break;
    }
    FunctionContext f = e.getFunction();
    String fn = f.getFunctionName();
    List<ExpressionContext> args = f.getArguments();
    int op = OPS.get(fn);
    if (op == T_DATETRUNC) {
      int unit = TRUNC_UNITS.indexOf(literal(args.get(0)).toUpperCase(Locale.ROOT));
      int in = args.size() > 2 ? TIME_UNITS.indexOf(literal(args.get(2)).toUpperCase(Locale.ROOT)) : 2;
      if (args.size() > 3 && !"UTC".equalsIgnoreCase(literal(args.get(3)))) {
        throw new IllegalArgumentException("time zone " + literal(args.get(3)));
      }
      int out = args.size() > 4 ? TIME_UNITS.indexOf(literal(args.get(4)).toUpperCase(Locale.ROOT)) : in;
      if (unit < 0 || in < 0 || out < 0) {
        throw new IllegalArgumentException("unit of " + e);
      }
      emit(args.get(1), p);
      p.add(op, unit | in << 8 | out << 16, 0.0);
    } else if (op == T_TIMECONVERT) {
      int in = TIME_UNITS.indexOf(literal(args.get(1)).toUpperCase(Locale.ROOT));
      int out = TIME_UNITS.indexOf(literal(args.get(2)).toUpperCase(Locale.ROOT));
      if (in < 0 || out < 0) {
        throw new IllegalArgumentException("unit of " + e);
      }
      emit(args.get(0), p);
      p.add(op, in | out << 8, 0.0);
    } else {
      for (ExpressionContext a : args) {
        emit(a, p);
      }
      long unit = 0;
      if (op >= T_TOEPOCH) {
        String u = fn.substring("toepoch".length());
        unit = u.startsWith("seconds") ? 3 : u.startsWith("minutes") ? 4 : u.startsWith("hours") ? 5 : 6;
      }
      p.add(op, unit, 0.0);
    }
  }

  /** A derived column of a resident segment: its column id and its dictionary (sorted values, Double.compare order). */
  static final class Derived {
    final int _column;
    final DataType _type;  // INT, LONG or DOUBLE
    final long[] _longs;   // INT / LONG values
    final double[] _doubles;

    Derived(int column, int storedType, byte[] dictionary) {
      _column = column;
      ByteBuffer b = ByteBuffer.wrap(dictionary);  // big-endian
      if (storedType == 0 || storedType == 1) {
        _type = storedType == 0 ? DataType.INT : DataType.LONG;
        int width = storedType == 0 ? 4 : 8;
        _longs = new long[dictionary.length / width];
        for (int k = 0; k < _longs.length; k++) {
          _longs[k] = width == 4 ? b.getInt(4 * k) : b.getLong(8 * k);
        }
        _doubles = null;
      } else {
        _type = DataType.DOUBLE;
        _doubles = new double[dictionary.length / 8];
        for (int k = 0; k < _doubles.length; k++) {
          _doubles[k] = b.getDouble(8 * k);
        }
        _longs = null;
      }
    }

    int cardinality() {
      return _longs != null ? _longs.length : _doubles.length;
    }

    /** Dictionary.getInternal(dictId). */
    Object get(int id) {
      if (_type == DataType.INT) {
        return (int) _longs[id];
      }
      return _type == DataType.LONG ? (Object) _longs[id] : (Object) _doubles[id];
    }

    private int compare(int id, String literal) {
      double v = Double.parseDouble(literal);
      if (_longs != null) {
        try {
          return Long.compare(_longs[id], Long.parseLong(literal.trim()));
        } catch (NumberFormatException ex) {
          return Double.compare((double) _longs[id], v);  // a fractional literal equals no integer
        }
      }
      return Double.compare(_doubles[id], v);
    }

    /** First id whose value is >= literal (or > literal when strict). */
    private int lowerBound(String literal, boolean strict) {
      int lo = 0, hi = cardinality();
      while (lo < hi) {
        int mid = (lo + hi) >>> 1;
        int c = compare(mid, literal);
        if (c < 0 || (strict && c == 0)) {
          lo = mid + 1;
        } else {
          hi = mid;
        }
      }
      return lo;
    }

    /**
     * The ids a predicate on the derived column matches, sorted (what a PredicateEvaluator's getMatchingDictIds gives
     * over a sorted dictionary), or null for a predicate type this path does not resolve.
     */
    int[] matchingIds(Predicate predicate) {
      int n = cardinality();
      if (_doubles != null) {
        return valueMatches(predicate);
      }
      switch (predicate.getType()) {
        case RANGE: {
          RangePredicate r = (RangePredicate) predicate;
          int start = r.getLowerBound().equals(RangePredicate.UNBOUNDED) ? 0 : lowerBound(r.getLowerBound(), !r.isLowerInclusive());
          int end = r.getUpperBound().equals(RangePredicate.UNBOUNDED) ? n : lowerBound(r.getUpperBound(), r.isUpperInclusive());
          return range(start, Math.max(start, end));
        }
        case EQ:
          return members(List.of(((EqPredicate) predicate).getValue()), false);
        case NOT_EQ:
          return members(List.of(((NotEqPredicate) predicate).getValue()), true);
        case IN:
          return members(((InPredicate) predicate).getValues(), false);
        case NOT_IN:
          return members(((NotInPredicate) predicate).getValues(), true);
        default:
          return null;
      }
    }

    /**
     * A DOUBLE expression has no dictionary in the reference: ExpressionFilterOperator evaluates it per row and compares
     * each value with Java's <, > and == (the raw-value predicate evaluators).  So NaN matches only NOT_EQ / NOT_IN, and
     * 0 matches both zeros.  In Double.compare order the entries a RANGE matches are contiguous (the zeros are
     * neighbours, NaN is last and matches no range), so a scan of [first, last] selects exactly them.
     */
    private int[] valueMatches(Predicate predicate) {
      List<String> values;
      boolean negate = false;
      switch (predicate.getType()) {
        case RANGE: {
          RangePredicate r = (RangePredicate) predicate;
          boolean lowerOpen = r.getLowerBound().equals(RangePredicate.UNBOUNDED);
          boolean upperOpen = r.getUpperBound().equals(RangePredicate.UNBOUNDED);
          double lower = lowerOpen ? 0.0 : Double.parseDouble(r.getLowerBound());
          double upper = upperOpen ? 0.0 : Double.parseDouble(r.getUpperBound());
          List<Integer> out = new ArrayList<>();
          for (int k = 0; k < _doubles.length; k++) {
            double x = _doubles[k];
            boolean above = lowerOpen || (r.isLowerInclusive() ? x >= lower : x > lower);
            boolean below = upperOpen || (r.isUpperInclusive() ? x <= upper : x < upper);
            if (above && below && x == x) {  // an unbounded range matches no NaN either
              out.add(k);
            }
          }
          return out.stream().mapToInt(Integer::intValue).toArray();
        }
        case EQ:
          values = List.of(((EqPredicate) predicate).getValue());
          break;
        case NOT_EQ:
          values = List.of(((NotEqPredicate) predicate).getValue());
          negate = true;
          break;
        case IN:
          values = ((InPredicate) predicate).getValues();
          break;
        case NOT_IN:
          values = ((NotInPredicate) predicate).getValues();
          negate = true;
          break;
        default:
          return null;
      }
      double[] literals = new double[values.size()];
      for (int k = 0; k < literals.length; k++) {
        literals[k] = Double.parseDouble(values.get(k));
      }
      List<Integer> out = new ArrayList<>();
      for (int k = 0; k < _doubles.length; k++) {
        boolean hit = false;
        for (double l : literals) {
          hit |= _doubles[k] == l;
        }
        if (hit != negate) {
          out.add(k);
        }
      }
      return out.stream().mapToInt(Integer::intValue).toArray();
    }

    private static int[] range(int start, int end) {
      int[] ids = new int[end - start];
      for (int k = 0; k < ids.length; k++) {
        ids[k] = start + k;
      }
      return ids;
    }

    private int[] members(List<String> values, boolean negate) {
      java.util.TreeSet<Integer> hit = new java.util.TreeSet<>();
      for (String v : values) {
        int id = lowerBound(v, false);
        if (id < cardinality() && compare(id, v) == 0) {
          hit.add(id);
        }
      }
      List<Integer> out = new ArrayList<>();
      for (int k = 0; k < cardinality(); k++) {
        if (hit.contains(k) != negate) {
          out.add(k);
        }
      }
      return out.stream().mapToInt(Integer::intValue).toArray();
    }
  }
}
