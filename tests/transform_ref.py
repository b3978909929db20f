"""Independent reference of the single-column transforms (DESIGN.md section 3.8), sharing no code with the product:
its own parser of the canonical text, Python ints for the unit conversions, numpy.datetime64 (proleptic Gregorian) for
the calendar, Python floats with math.fmod / floor / ceil for the arithmetic.

    evaluate(text, value, source_type) -> (kind, value)   kind in "INT", "LONG", "DOUBLE"; raises Refused
    column(text, values, source_type)  -> numpy array of the results, typed (int32 / int64 / float64)

Its own copy of the rules:
  * TIMECONVERT / TOEPOCH* / DATETRUNC's unit steps: java.util.concurrent.TimeUnit -- toward 0 when coarser, saturated
    to the int64 ends when finer; TOEPOCH<unit>BUCKET(x, n) = that / n, ROUNDED = (that / n) * n (toward 0);
  * DATETRUNC and the calendar fields: UTC, proleptic Gregorian, floored toward -inf; WEEK / DAYOFWEEK are ISO (Monday);
    an instant beyond +-2^53 ms after the input-unit conversion is refused;
  * arithmetic: operands as doubles, one IEEE-754 round-to-nearest operation each; x / 0 = +-inf or NaN; MOD = fmod."""
import math

import numpy as np

NANOS = {"NANOSECONDS": 1, "MICROSECONDS": 10 ** 3, "MILLISECONDS": 10 ** 6, "SECONDS": 10 ** 9, "MINUTES": 60 * 10 ** 9,
         "HOURS": 3600 * 10 ** 9, "DAYS": 86400 * 10 ** 9}
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
BOUND = 1 << 53
CALENDAR = ("year", "quarter", "month", "week", "day", "dayofweek", "dayofyear", "hour", "minute", "second", "millisecond")


class Refused(Exception):
    pass


def _tdiv(a: int, b: int) -> int:  # Java long division
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def convert(d: int, src: str, dst: str) -> int:
    s, t = NANOS[src], NANOS[dst]
    if s == t:
        return d
    if s < t:
        return _tdiv(d, t // s)
    r = s // t
    m = INT64_MAX // r
    if d > m:
        return INT64_MAX
    if d < -m:
        return INT64_MIN
    return d * r


def _ms(x: int) -> np.datetime64:
    if not -BOUND <= x <= BOUND:
        raise Refused(f"instant {x} beyond 2^53 ms")
    return np.datetime64(int(x), "ms")


def _as_ms(t: np.datetime64) -> int:
    return int(t.astype("datetime64[ms]").astype(np.int64))


def _iso_dow(day: np.datetime64) -> int:  # 1 = Monday; day 0 (1970-01-01) was a Thursday
    return (int(day.astype(np.int64)) + 3) % 7 + 1


def truncate(unit: str, ms: int) -> int:
    t = _ms(ms)
    if unit == "MILLISECOND":
        return ms
    if unit in ("SECOND", "MINUTE", "HOUR", "DAY"):
        return _as_ms(t.astype({"SECOND": "datetime64[s]", "MINUTE": "datetime64[m]", "HOUR": "datetime64[h]", "DAY": "datetime64[D]"}[unit]))
    day = t.astype("datetime64[D]")
    if unit == "WEEK":
        return _as_ms(day - np.timedelta64(_iso_dow(day) - 1, "D"))
    month = t.astype("datetime64[M]")
    if unit == "MONTH":
        return _as_ms(month)
    if unit == "QUARTER":
        m = int(month.astype(np.int64))
        return _as_ms(np.datetime64(m - m % 3, "M"))
    return _as_ms(t.astype("datetime64[Y]"))


def calendar(fn: str, ms: int) -> int:
    t = _ms(ms)
    day = t.astype("datetime64[D]")
    month = t.astype("datetime64[M]")
    year = t.astype("datetime64[Y]")
    in_day = ms - _as_ms(day)
    if fn == "year":
        return int(year.astype(np.int64)) + 1970
    if fn == "month":
        return int(month.astype(np.int64)) % 12 + 1
    if fn == "quarter":
        return (int(month.astype(np.int64)) % 12) // 3 + 1
    if fn == "day":
        return int((day - month.astype("datetime64[D]")).astype(np.int64)) + 1
    if fn == "dayofweek":
        return _iso_dow(day)
    if fn == "dayofyear":
        return int((day - year.astype("datetime64[D]")).astype(np.int64)) + 1
    if fn == "hour":
        return in_day // 3_600_000
    if fn == "minute":
        return in_day // 60_000 % 60
    if fn == "second":
        return in_day // 1000 % 60
    if fn == "millisecond":
        return in_day % 1000
    # ISO week: the week's Thursday decides the week-based year; weeks count from that year's first Thursday's week
    thursday = day + np.timedelta64(4 - _iso_dow(day), "D")
    jan1 = thursday.astype("datetime64[Y]").astype("datetime64[D]")
    return int((thursday - jan1).astype(np.int64)) // 7 + 1


def _div(x: float, y: float) -> float:
    if y != 0:
        return x / y
    if x != x or x == 0:
        return math.nan
    return math.copysign(math.inf, x) * math.copysign(1.0, y)


def _fmod(x: float, y: float) -> float:
    if y == 0 or math.isinf(x) or x != x or y != y:
        return math.nan
    return math.fmod(x, y)


def _floor(x: float) -> float:
    if not math.isfinite(x) or x == int(x):
        return x
    return float(math.floor(x))


def _ceil(x: float) -> float:
    if not math.isfinite(x) or x == int(x):
        return x
    r = float(math.ceil(x))
    return -0.0 if r == 0 else r


ARITH = {"plus": lambda x, y: x + y, "minus": lambda x, y: x - y, "times": lambda x, y: x * y, "divide": _div, "mod": _fmod}


def parse(text: str):
    """Canonical text -> nested tuples: ("fn", name, args) | ("lit", text) | ("col", name)."""
    pos = 0

    def node():
        nonlocal pos
        if text[pos] == "'":
            end = text.index("'", pos + 1)
            lit = text[pos + 1:end]
            pos = end + 1
            return ("lit", lit)
        start = pos
        while pos < len(text) and text[pos] not in "(),":
            pos += 1
        name = text[start:pos]
        if pos < len(text) and text[pos] == "(":
            pos += 1
            args = [node()]
            while text[pos] == ",":
                pos += 1
                args.append(node())
            assert text[pos] == ")", text
            pos += 1
            return ("fn", name, args)
        return ("col", name)

    tree = node()
    assert pos == len(text), text
    return tree


def _number(lit: str):
    try:
        return int(lit)
    except ValueError:
        return float(lit)


def _eval(n, value, source_type):
    """-> (kind, value); kinds "INT" / "LONG" (Python int), "DOUBLE" (float), "FLOAT" for a FLOAT column."""
    if n[0] == "col":
        return ("LONG" if source_type in ("INT", "LONG") else "DOUBLE"), value
    if n[0] == "lit":
        v = _number(n[1])
        return ("LONG" if isinstance(v, int) else "DOUBLE"), v
    _, fn, args = n

    def integral(a):
        if a[0] == "lit":
            raise Refused(f"{fn} of a literal")
        k, v = _eval(a, value, source_type)
        if k not in ("INT", "LONG"):
            raise Refused(f"{fn} of a {k}")
        return v

    if fn in ARITH or fn in ("floor", "ceil", "abs"):
        xs = [float(_eval(a, value, source_type)[1]) for a in args]
        if fn in ARITH:
            return "DOUBLE", ARITH[fn](xs[0], xs[1])
        return "DOUBLE", {"floor": _floor, "ceil": _ceil, "abs": abs}[fn](xs[0])
    if fn == "datetrunc":
        unit = args[0][1]
        in_unit = args[2][1] if len(args) > 2 else "MILLISECONDS"
        if len(args) > 3 and args[3][1] != "UTC":
            raise Refused("time zone")
        out_unit = args[4][1] if len(args) > 4 else in_unit
        ms = convert(integral(args[1]), in_unit, "MILLISECONDS")
        return "LONG", convert(truncate(unit, ms), "MILLISECONDS", out_unit)
    if fn in CALENDAR:
        return "INT", calendar(fn, integral(args[0]))
    if fn == "timeconvert":
        return "LONG", convert(integral(args[0]), args[1][1], args[2][1])
    if fn.startswith("toepoch"):
        rest = fn[len("toepoch"):]
        unit = next(u for u in ("SECONDS", "MINUTES", "HOURS", "DAYS") if rest.upper().startswith(u))
        v = convert(integral(args[0]), "MILLISECONDS", unit)
        if rest.endswith("bucket"):
            return "LONG", _tdiv(v, int(args[1][1]))
        if rest.endswith("rounded"):
            n = int(args[1][1])
            return "LONG", _tdiv(v, n) * n
        return "LONG", v
    raise Refused(f"unknown function {fn}")


def evaluate(text: str, value, source_type: str):
    kind, v = _eval(parse(text), int(value) if source_type in ("INT", "LONG") else float(value), source_type)
    return kind, v


def column(text: str, values: np.ndarray, source_type: str) -> np.ndarray:
    """The expression over every value (numpy array of the source's values), typed like the derived column."""
    out = [evaluate(text, v, source_type) for v in values.tolist()]
    kind = out[0][0] if out else "LONG"
    dtype = {"INT": np.int32, "LONG": np.int64, "DOUBLE": np.float64}[kind]
    return np.array([v for _, v in out], dtype=dtype)


def double_order_key(x: float) -> int:
    """Double.compare order as an unsigned int: -0.0 before 0.0, one NaN after +inf."""
    if x != x:
        x = math.nan
    u = int(np.array([x], dtype=np.float64).view(np.uint64)[0])
    if x != x:
        u = 0x7FF8000000000000
    return (~u & 0xFFFFFFFFFFFFFFFF) if u >> 63 else u | (1 << 63)
