"""Tiny SQL front end for the query shapes the reference's own tests use on this path.

The reference compiles SQL with Calcite in pinot-common (``CalciteSqlParser`` -> ``PinotQuery`` ->
``QueryContextConverterUtils.getQueryContext``), which is OUT OF SCOPE here (the broker/server path above the plan maker
stays Java).  This module exists so the parity tests read like the reference's
(``getOperator("SELECT COUNT(*), SUM(column1) FROM testTable WHERE ... GROUP BY column9")``,
``pinot-core/src/test/java/org/apache/pinot/queries/BaseQueriesTest.java:97-102``).  Grammar:

    SELECT item[, item...] FROM table [WHERE cond] [GROUP BY col[, col...] [HAVING hcond]] [ORDER BY expr [ASC|DESC], ...]
           [LIMIT n]
    item  := agg | col | post
    item  := COUNT(*) | FN(col) | PERCENTILE(col, p) | PERCENTILE<n>(col) | FIRSTWITHTIME(col, col, 'T')
             | LASTWITHTIME(col, col, 'T') | COUNT(DISTINCT col) | SUM(DISTINCT col) | AVG(DISTINCT col) | col
             (COUNT / SUM / AVG(DISTINCT col) are DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG(col), named
             distinctcount(col) ...; MIN / MAX(DISTINCT col), COUNT(DISTINCT *) and COUNT(DISTINCT a, b) are refused)
             (FN also VAR_POP / VARPOP, VAR_SAMP / VARSAMP, STDDEV_POP / STDDEVPOP, STDDEV_SAMP / STDDEVSAMP; T is the
             data column's type, INT | LONG | FLOAT | DOUBLE | STRING | BOOLEAN, any case; the canonical text is
             lastwithtime(v,t,'INT'))
             (plain columns are allowed only when they are group-by keys; 0 <= p <= 100, fractions allowed)
    selection (parse_selection): SELECT * | col[, col...] FROM table [WHERE cond] [ORDER BY col [ASC|DESC], ...] [LIMIT n]
    distinct (parse_distinct): SELECT DISTINCT col[, col...] FROM table [WHERE cond] [ORDER BY col [ASC|DESC], ...] [LIMIT n]
                  (every ORDER BY column must be a DISTINCT column)
    cond  := cond AND cond | cond OR cond | NOT cond | (cond) | col op literal | col BETWEEN a AND b
             | col [NOT] IN (literal, ...) | col [NOT] LIKE 'pattern' | REGEXP_LIKE(col, 'regex')
             | literal op col | col op col
             (the reference's PredicateComparisonRewriter: `literal op col` is `col op' literal` with the operator
             mirrored, `a op b` with a non-literal right side is `minus(a,b) op 0`, so `a > b` names the expression
             minus(a,b), evaluated per row when it has two or more columns -- DESIGN.md section 3.16.  BETWEEN bounds
             and IN values must be literals)
             (LIKE is rewritten into REGEXP_LIKE by like_to_regexp; both only on STRING dictionary columns, never in
             HAVING)
    op    := = | != | <> | < | <= | > | >=
    hcond := cond whose left-hand sides are aggregation calls (COUNT(*), FN(col), PERCENTILE(col, p), ...) and whose
             literals are numbers.  An aggregation named only in HAVING is computed as a hidden one (Aggregation.hidden):
             ORDER BY may name it, it is never an output column.  HAVING on a column belongs in WHERE and is refused.
    case  := CASE WHEN ccond THEN value [WHEN ccond THEN value ...] ELSE value END, only as the whole argument of SUM,
             AVG, MIN, MAX or COUNT (DESIGN.md section 3.19); named case(c1,v1,...,e).  value := the arithmetic of col below
             (and a leading unary minus, times('-1',x)); ccond := AND / OR / NOT / parentheses over `col op literal`,
             col BETWEEN a AND b, col [NOT] IN (...), col [NOT] LIKE 'p', REGEXP_LIKE(col, 'p'), spelled equals(a,'1'),
             not_equals, less_than, less_than_or_equal, greater_than, greater_than_or_equal, between, in, not_in, like,
             regexp_like, and, or, not.  Refused: no ELSE, a nested or simple CASE, column against column, expression
             operands, string values, CASE anywhere else.
    post  := arithmetic over aggregation calls, a post-aggregation expression (DESIGN.md section 3.18):
             post := term (+|- term)* ; term := unary (*|/ unary)* ; unary := -unary | factor ;
             factor := agg | number | (post), with at least one agg.  Numbers are finite decimals; a column, a string, %
             or a function that is not an aggregation (ABS(SUM(x))) is refused.  Named by its normalised text
             (QueryContext.post_aggregations): SUM(a) / SUM(b) -> divide(sum(a),sum(b)), -x -> negate(x).  An aggregation
             named only in such expressions is a hidden one, as for HAVING.  An ORDER BY expression must be a SELECT
             item, compared by that text.
    col   := a column, or a single-column expression wherever a column is accepted (select list, GROUP BY, aggregation
             arguments, the left-hand side of predicates, ORDER BY, selection and DISTINCT lists):
             expr := term (+|- term)* ; term := factor (*|/|% factor)* ; factor := col | number | (expr) | fn(args)
             fn in TRANSFORMS (DATETRUNC('DAY', ts), YEAR(ts), TIMECONVERT(ts, 'MILLISECONDS', 'HOURS'), FLOOR(x / 10), ...).
             An expression is named by its canonical text (the reference's ExpressionContext.toString()):
             ts / 1000 -> divide(ts,'1000'), DATE_TRUNC('day', ts) -> datetrunc('DAY',ts)
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field
from typing import List, Optional

from .query import (AGG_FUNCTIONS, HLL_DEFAULT_LOG2M, WITHTIME_FUNCTIONS, WITHTIME_TYPES, Aggregation, Filter, FilterNode, PostAggregation,
                    Predicate, QueryContext, flatten, optimize_filter)

_TOKEN = re.compile(r"\s*(?:(\d+\.\d+(?:[eE][-+]?\d+)?|-?\d+\.\d+|-?\d+)|'((?:[^']|'')*)'|(<=|>=|<>|!=|[=<>(),*+/%-])|"
                    r"([A-Za-z_$][A-Za-z0-9_$]*))")

# VarianceAggregationFunction: both spellings of each function, the underscore one canonicalised to the other
_ALIASES = {"VAR_POP": "VARPOP", "VAR_SAMP": "VARSAMP", "STDDEV_POP": "STDDEVPOP", "STDDEV_SAMP": "STDDEVSAMP"}
_FUNCTIONS = set(AGG_FUNCTIONS) | set(_ALIASES)
# FN(DISTINCT col): the function Pinot's query compiler rewrites it into
_DISTINCT_OF = {"COUNT": "DISTINCTCOUNT", "SUM": "DISTINCTSUM", "AVG": "DISTINCTAVG"}
_PERCENTILE_N = re.compile(r"PERCENTILE(\d+)")

# single-column transforms (DESIGN.md section 3.8): SQL name (lower case, no '_') -> canonical name
TRANSFORMS = {n: n for n in (
    "plus", "minus", "times", "divide", "mod", "floor", "ceil", "abs", "datetrunc", "year", "quarter", "month", "week",
    "day", "dayofweek", "dayofyear", "hour", "minute", "second", "millisecond", "timeconvert",
    *(f"toepoch{u}{k}" for u in ("seconds", "minutes", "hours", "days") for k in ("", "bucket", "rounded")))}
TRANSFORMS.update(add="plus", sub="minus", mult="times", div="divide", weekofyear="week", dayofmonth="day",
                  dow="dayofweek", doy="dayofyear")
_DECIMAL = re.compile(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?")
_INFIX = {"+": "plus", "-": "minus", "*": "times", "/": "divide", "%": "mod"}


def _transform_name(name: str) -> Optional[str]:
    return TRANSFORMS.get(name.lower().replace("_", ""))


def _literal_text(v) -> str:
    """A literal of canonical text: strings (time units, time zones) in upper case, numbers by value."""
    if isinstance(v, str):
        if not _DECIMAL.fullmatch(v):
            return "'" + v.upper().replace("'", "''") + "'"
        v = float(v) if any(ch in v for ch in ".eE") else int(v)   # a quoted number: by value, like an unquoted one
    if isinstance(v, float) and v.is_integer() and abs(v) < 9.2e18 and not (v == 0 and str(v)[0] == "-"):  # -0.0 stays
        v = int(v)
    return f"'{v!r}'"


def _is_function(name: str) -> bool:
    return name.upper() in _FUNCTIONS or _PERCENTILE_N.fullmatch(name.upper()) is not None


def _percentile_arg(value) -> float:
    """The percentile of PERCENTILE(col, p) / PERCENTILE<n>(col): a numeric literal in [0, 100]."""
    if isinstance(value, bool) or not isinstance(value, (int, float)):
        raise SqlError(f"PERCENTILE needs a numeric percentile, got {value!r}")
    p = float(value)
    if not 0.0 <= p <= 100.0:
        raise SqlError(f"PERCENTILE percentile {value!r} is outside [0, 100]")
    return p


class SqlError(ValueError):
    pass


def having_name(agg: Aggregation) -> str:
    """How a HAVING leaf names an aggregation (QueryContext.having)."""
    if agg.function == "PERCENTILE":
        return f"percentile({agg.column},{agg.arg!r})"
    if agg.function == "DISTINCTCOUNTHLL" and agg.arg != HLL_DEFAULT_LOG2M:
        return f"distinctcounthll({agg.column},{agg.arg})"
    if agg.function in WITHTIME_FUNCTIONS:
        return str(agg)
    return f"{agg.function.lower()}({agg.column or '*'})"


MAX_HAVING_NODES = 32
MAX_POST_NODES = 16   # nodes of one post-aggregation program (pb200_post_program)

_POST_NAMES = {"ADD": "plus", "SUB": "minus", "MUL": "times", "DIV": "divide", "NEG": "negate"}


def _filter_text(n) -> str:
    """Canonical text of a FILTER clause's tree (how a filtered operand of a post-aggregation expression is named)."""
    if isinstance(n, Filter):
        return f"{n.type.lower()}({','.join(_filter_text(c) for c in n.children)})"
    if n.type == "RANGE":
        return (f"range({n.column},{'[' if n.lower_inclusive else '('}{'*' if n.lower is None else _literal_text(n.lower)},"
                f"{'*' if n.upper is None else _literal_text(n.upper)}{']' if n.upper_inclusive else ')'})")
    return f"{n.type.lower()}({n.column},{','.join(_literal_text(v) for v in n.values)})"


def _post_text(t) -> str:
    """Normalised text of a post-aggregation expression tree (_Parser.post_item): spacing, case and parentheses gone."""
    if t[0] == "AGG":
        return having_name(t[1]) + ("" if t[1].filter is None else f" filter({_filter_text(t[1].filter)})")
    if t[0] == "LIT":
        return _literal_text(t[1])
    return f"{_POST_NAMES[t[0]]}({','.join(_post_text(c) for c in t[1:])})"


def _post_aggs(t) -> List[Aggregation]:
    """The aggregation calls of a post-aggregation expression tree, left to right."""
    if t[0] == "AGG":
        return [t[1]]
    if t[0] in ("LIT", "COL", "STR"):
        return []
    return [a for c in (t[2] if t[0] == "FUNC" else t[1:]) for a in _post_aggs(c)]


def _post_check(t):
    """Refuses what a post-aggregation expression cannot hold (SqlError)."""
    kind = t[0]
    if kind == "COL":
        raise SqlError(f"the column {t[1]} in an expression over aggregations: operands must be aggregation calls or numbers")
    if kind == "STR":
        raise SqlError(f"the string literal {t[1]!r} in an expression over aggregations: only numbers are supported")
    if kind == "FUNC":
        if _post_aggs(t):
            raise SqlError(f"{t[1]}(...) over an aggregation: only +, -, * and / apply to aggregations")
        raise SqlError(f"the column expression {t[1]}(...) in an expression over aggregations: operands must be aggregation calls or numbers")
    if kind == "MOD":
        raise SqlError("% in an expression over aggregations is not supported (only +, -, * and /)")
    if kind == "LIT":
        try:
            v = float(t[1])
        except OverflowError:
            v = math.inf
        if not math.isfinite(v):
            raise SqlError(f"the literal {t[1]!r} in an expression over aggregations is not a finite number")
        return
    if kind == "AGG":
        if t[1].value_type == "STRING":
            raise SqlError(f"{having_name(t[1])} in an expression: a STRING FIRST/LASTWITHTIME is not a number")
        return
    for c in t[1:]:
        _post_check(c)

_REGEX_META = set("\\.^$|?*+()[]{}")


def like_to_regexp(like: str) -> str:
    """The REGEXP_LIKE pattern of `col LIKE like` (Pinot's RegexpPatternConverterUtils.likeToRegexpLike): a leading run
    of % drops the ^ anchor and a trailing run the $ anchor, % becomes .* and _ becomes ., every regex metacharacter is
    escaped; a pattern of only % is '' (every value) and '' is ^$.  A backslash is refused: Pinot's LIKE escapes are not
    restated here."""
    if "\\" in like:
        raise SqlError(f"LIKE pattern {like!r} contains a backslash: LIKE escapes are not supported")
    if like == "":
        return "^$"
    if set(like) == {"%"}:
        return ""
    lead = len(like) - len(like.lstrip("%"))
    trail = len(like) - len(like.rstrip("%"))
    body = "".join(".*" if ch == "%" else "." if ch == "_" else "\\" + ch if ch in _REGEX_META else ch
                   for ch in like[lead:len(like) - trail])
    return ("" if lead else "^") + body + ("" if trail else "$")



class _Parser:
    def __init__(self, text: str):
        self.toks = []
        pos = 0
        text = text.strip().rstrip(";")
        while pos < len(text):
            m = _TOKEN.match(text, pos)
            if not m or m.end() == pos:
                raise SqlError(f"cannot tokenize at: {text[pos:pos + 20]!r}")
            num, s, op, ident = m.groups()
            if num is not None:
                self.toks.append(("num", float(num) if ("." in num or "e" in num.lower()) else int(num)))
            elif s is not None:
                self.toks.append(("str", s.replace("''", "'")))
            elif op is not None:
                self.toks.append(("op", op))
            else:
                self.toks.append(("id", ident))
            pos = m.end()
        self.i = 0
        self.having: Optional[List[Aggregation]] = None   # inside HAVING: the aggregations its leaves name
        self.in_case = False   # inside a CASE's branches

    def peek(self):
        return self.toks[self.i] if self.i < len(self.toks) else (None, None)

    def kw(self, word) -> bool:
        k, v = self.peek()
        return k == "id" and v.upper() == word

    def take_kw(self, word) -> bool:
        if self.kw(word):
            self.i += 1
            return True
        return False

    def expect_kw(self, word):
        if not self.take_kw(word):
            raise SqlError(f"expected {word}, got {self.peek()}")

    def take_op(self, op) -> bool:
        k, v = self.peek()
        if k == "op" and v == op:
            self.i += 1
            return True
        return False

    def expect_op(self, op):
        if not self.take_op(op):
            raise SqlError(f"expected {op!r}, got {self.peek()}")

    def percentile_call(self, name: str):
        """After `name(`: the column and percentile of PERCENTILE(col, p) or PERCENTILE<n>(col), up to the `)`."""
        col = self.column()
        m = _PERCENTILE_N.fullmatch(name.upper())
        if m:
            p = _percentile_arg(int(m.group(1)))
        else:
            self.expect_op(",")
            p = _percentile_arg(self.literal())
        return col, p

    def hll_call(self):
        """After `DISTINCTCOUNTHLL(`: the column and log2m, an integer literal in 0..30 (the reference's range; default 8),
        up to the `)`."""
        col = self.column()
        log2m = HLL_DEFAULT_LOG2M
        if self.take_op(","):
            v = self.literal()
            if isinstance(v, bool) or not isinstance(v, int) or not 0 <= v <= 30:
                raise SqlError(f"DISTINCTCOUNTHLL needs an integer log2m in 0..30, got {v!r}")
            log2m = v
        return col, log2m

    def withtime_call(self, fn: str) -> Aggregation:
        """After `FIRSTWITHTIME(` / `LASTWITHTIME(`: data column, time column and type literal, up to the `)`."""
        col = self.column()
        self.expect_op(",")
        time_col = self.column()
        self.expect_op(",")
        k, v = self.peek()
        if k != "str" or v.upper() not in WITHTIME_TYPES:
            raise SqlError(f"{fn} needs the data column's type as a string literal ({', '.join(WITHTIME_TYPES)}), got {self.peek()}")
        self.i += 1
        return Aggregation(fn, col, time_column=time_col, value_type=v.upper())

    def ident(self) -> str:
        k, v = self.peek()
        if k != "id":
            raise SqlError(f"expected identifier, got {self.peek()}")
        self.i += 1
        return v

    # ---- single-column expressions: canonical text (a plain column stays its name) ---------------------------------
    def column(self) -> str:
        text, is_literal = self._additive()
        if is_literal:
            raise SqlError(f"expected a column or an expression, got the literal {text}")
        return text

    def _additive(self):
        left = self._multiplicative()
        while True:
            k, v = self.peek()
            if k == "op" and v in ("+", "-"):
                self.i += 1
                right = self._multiplicative()
            elif k == "num" and v < 0 and not left[1]:   # `x -1` is tokenized as x, -1
                self.i += 1
                v, right = "-", (_literal_text(-v), True)
            else:
                return left
            left = (f"{_INFIX[v]}({left[0]},{right[0]})", False)

    def _multiplicative(self):
        left = self._factor()
        while True:
            k, v = self.peek()
            if k != "op" or v not in ("*", "/", "%"):
                return left
            self.i += 1
            right = self._factor()
            left = (f"{_INFIX[v]}({left[0]},{right[0]})", False)

    def _factor(self):
        k, v = self.peek()
        if k == "id" and v.upper() == "CASE":
            if self.in_case:
                raise SqlError("a nested CASE is not supported")
            raise SqlError("CASE is accepted only as the whole argument of SUM, AVG, MIN, MAX or COUNT")
        if self.in_case and self.take_op("-"):   # a negated CASE value (THEN -bytes): IEEE negation, -1 * x
            return f"times('-1',{self._factor()[0]})", False
        if k in ("num", "str"):
            self.i += 1
            return _literal_text(v), True
        if self.take_op("("):
            inner = self._additive()
            self.expect_op(")")
            return inner
        name = self.ident()
        if self.peek() != ("op", "("):
            return name, False
        canonical = _transform_name(name)
        if canonical is None:
            raise SqlError(f"{name}(...) is not a single-column transform of this path")
        self.i += 1
        args = [] if self.peek() == ("op", ")") else [self._additive()]
        while self.take_op(","):
            args.append(self._additive())
        self.expect_op(")")
        return f"{canonical}({','.join(a[0] for a in args)})", False

    def literal(self):
        k, v = self.peek()
        if k not in ("num", "str"):
            raise SqlError(f"expected literal, got {self.peek()}")
        if k == "str" and self.having is not None:
            raise SqlError(f"HAVING compares aggregations with numbers, got the string literal {v!r}")
        self.i += 1
        return v

    def distinct_call(self, fn: str) -> str:
        """After `FN(DISTINCT`: the column of COUNT / SUM / AVG(DISTINCT col), up to the `)`."""
        if fn not in _DISTINCT_OF:
            raise SqlError(f"{fn}(DISTINCT ...) is not supported (COUNT, SUM and AVG take DISTINCT)")
        if self.take_op("*"):
            raise SqlError(f"{fn}(DISTINCT *) is not valid")
        col = self.column()
        if self.take_op(","):
            raise SqlError(f"{fn}(DISTINCT ...) over more than one column is not supported")
        return col

    def aggregation_call(self) -> Aggregation:
        """An aggregation call after its name, e.g. `SUM(` + `m)`: the name token is at self.i - 2."""
        name = self.toks[self.i - 2][1]
        fn = _ALIASES.get(name.upper(), name.upper())
        if self.take_kw("DISTINCT"):
            agg = Aggregation(_DISTINCT_OF.get(fn, fn), self.distinct_call(fn))
        elif fn.startswith("PERCENTILE"):
            col, pct = self.percentile_call(name)
            agg = Aggregation("PERCENTILE", col, arg=pct)
        elif fn in WITHTIME_FUNCTIONS:
            agg = self.withtime_call(fn)
        elif fn == "DISTINCTCOUNTHLL" and self.peek() != ("op", "*"):
            col, log2m = self.hll_call()
            agg = Aggregation(fn, col, arg=log2m)
        elif self.take_op("*"):
            if fn != "COUNT":
                raise SqlError(f"{fn}(*) is not valid")
            agg = Aggregation("COUNT", None)
        else:
            col = self.case_expr() if self.kw("CASE") and fn in _CASE_FUNCTIONS else self.column()
            agg = Aggregation("COUNT", None) if fn == "COUNT" else Aggregation(fn, col)
        self.expect_op(")")
        return agg

    # ---- CASE WHEN as an aggregation argument (DESIGN.md section 3.19) ----------------------------------------------
    def case_expr(self) -> str:
        """CASE WHEN cond THEN value [WHEN ...] ELSE value END, named case(c1,v1,...,e)."""
        self.expect_kw("CASE")
        if not self.kw("WHEN"):
            raise SqlError("simple CASE (CASE x WHEN v THEN ...) is not supported: write CASE WHEN x = v THEN ...")
        parts = []
        self.in_case = True
        try:
            while self.take_kw("WHEN"):
                parts.append(self.case_cond())
                self.expect_kw("THEN")
                parts.append(self._case_value())
            if not self.take_kw("ELSE"):
                raise SqlError("CASE without ELSE is not supported (an implicit ELSE NULL has no value without null handling)")
            parts.append(self._case_value())
            self.expect_kw("END")
        finally:
            self.in_case = False
        return f"case({','.join(parts)})"

    def _case_value(self) -> str:
        start = self.i
        text, is_literal = self._additive()
        if is_literal and self.toks[start][0] == "str" and not _DECIMAL.fullmatch(self.toks[start][1]):
            raise SqlError(f"CASE values are numbers, columns or arithmetic, got the string {self.toks[start][1]!r}")
        return text

    def case_cond(self) -> str:
        kids = [self._case_and()]
        while self.take_kw("OR"):
            kids.append(self._case_and())
        return kids[0] if len(kids) == 1 else f"or({','.join(kids)})"

    def _case_and(self) -> str:
        kids = [self._case_not()]
        while self.take_kw("AND"):
            kids.append(self._case_not())
        return kids[0] if len(kids) == 1 else f"and({','.join(kids)})"

    def _case_not(self) -> str:
        if self.take_kw("NOT"):
            return f"not({self._case_not()})"
        if self.take_op("("):
            inner = self.case_cond()
            self.expect_op(")")
            return inner
        return self._case_leaf()

    def _case_column(self) -> str:
        k, v = self.peek()
        nxt = self.toks[self.i + 1] if self.i + 1 < len(self.toks) else (None, None)
        if k != "id" or nxt == ("op", "(") or (nxt[0] == "op" and nxt[1] in "+-*/%") or (nxt[0] == "num" and nxt[1] < 0):
            raise SqlError(f"a CASE condition compares one column with literals, got {self.peek()}")
        self.i += 1
        return v

    def _case_literal(self) -> str:
        k, v = self.peek()
        if k not in ("num", "str"):
            raise SqlError(f"a CASE condition compares one column with literals (no column against column), got {self.peek()}")
        self.i += 1
        return _case_literal_text(v)

    def _case_leaf(self) -> str:
        k, v = self.peek()
        if k == "id" and v.upper() == "REGEXP_LIKE" and self.toks[self.i + 1:self.i + 2] == [("op", "(")]:
            self.i += 2
            col = self._case_column()
            self.expect_op(",")
            pat = self.pattern()
            self.expect_op(")")
            return f"regexp_like({col},{_quote(pat)})"
        if k in ("num", "str"):   # `literal op col` is `col op' literal`
            lit = self._case_literal()
            k, op = self.peek()
            if k != "op" or op not in _FLIPPED:
                raise SqlError(f"expected a comparison operator after the literal {lit}")
            self.i += 1
            return f"{_CASE_OPS[_FLIPPED[op]]}({self._case_column()},{lit})"
        col = self._case_column()
        if self.take_kw("BETWEEN"):
            lo = self._case_literal()
            self.expect_kw("AND")
            return f"between({col},{lo},{self._case_literal()})"
        negate = self.take_kw("NOT")
        if self.take_kw("LIKE"):
            pat = self.pattern()
            like_to_regexp(pat)   # the same refusals as a WHERE leaf
            leaf = f"like({col},{_quote(pat)})"
            return f"not({leaf})" if negate else leaf
        if self.take_kw("IN"):
            self.expect_op("(")
            vals = [self._case_literal()]
            while self.take_op(","):
                vals.append(self._case_literal())
            self.expect_op(")")
            return f"{'not_in' if negate else 'in'}({col},{','.join(vals)})"
        if negate:
            raise SqlError("NOT must be followed by IN or LIKE here")
        k, op = self.peek()
        if k != "op" or op not in _CASE_OPS:
            raise SqlError(f"expected a comparison operator in a CASE condition, got {self.peek()}")
        self.i += 1
        return f"{_CASE_OPS[op]}({col},{self._case_literal()})"

    # ---- post-aggregation expressions: arithmetic over aggregation calls -------------------------------------------
    def post_item(self):
        """At a SELECT or ORDER BY item: its tree when the item is arithmetic over aggregation calls (a post-aggregation
        expression; checked by _post_check), else None with the position unchanged -- a single aggregation call, a column
        or a single-column expression is parsed as before.  Tree nodes: ("AGG", Aggregation), ("LIT", number),
        ("NEG", x), ("ADD" | "SUB" | "MUL" | "DIV" | "MOD", x, y) and, refused by _post_check, ("COL", name),
        ("STR", text), ("FUNC", name, args)."""
        start = self.i
        try:
            tree = self._post_additive()
        except SqlError:
            tree = None
        if tree is None or not _post_aggs(tree) or (tree[0] == "AGG" and self.toks[start][0] == "id"):
            self.i = start
            return None
        _post_check(tree)
        return tree

    def _post_additive(self):
        left = self._post_term()
        while True:
            k, v = self.peek()
            if k == "op" and v in ("+", "-"):
                self.i += 1
                left = ("ADD" if v == "+" else "SUB", left, self._post_term())
            elif k == "num" and v < 0:   # `x -1` is tokenized as x, -1
                self.i += 1
                left = ("SUB", left, ("LIT", -v))
            else:
                return left

    def _post_term(self):
        left = self._post_unary()
        while True:
            k, v = self.peek()
            if k != "op" or v not in ("*", "/", "%"):
                return left
            self.i += 1
            left = ({"*": "MUL", "/": "DIV", "%": "MOD"}[v], left, self._post_unary())

    def _post_unary(self):
        if self.take_op("-"):
            return ("NEG", self._post_unary())
        return self._post_factor()

    def _post_factor(self):
        k, v = self.peek()
        if k in ("num", "str"):
            self.i += 1
            return ("LIT" if k == "num" else "STR", v)
        if self.take_op("("):
            inner = self._post_additive()
            self.expect_op(")")
            return inner
        name = self.ident()
        if not self.take_op("("):
            return ("COL", name)
        if _is_function(name):
            agg = self.aggregation_call()
            if self.take_kw("FILTER"):   # SUM(x) FILTER (WHERE cond)
                self.expect_op("(")
                self.expect_kw("WHERE")
                agg.filter = optimize_filter(self.cond())
                self.expect_op(")")
            return ("AGG", agg)
        args = [] if self.peek() == ("op", ")") else [self._post_additive()]
        while self.take_op(","):
            args.append(self._post_additive())
        self.expect_op(")")
        return ("FUNC", name, args)

    def having_operand(self) -> str:
        """Left-hand side of a HAVING comparison: an aggregation call, named by having_name."""
        k, v = self.peek()
        if k in ("num", "str"):
            raise SqlError(f"HAVING: the literal {v!r} is on the left-hand side; write the aggregation first")
        if k == "id" and _is_function(v) and self.toks[self.i + 1:self.i + 2] == [("op", "(")]:
            self.i += 2
            agg = self.aggregation_call()
            self.having.append(agg)
            return having_name(agg)
        col = self.column()
        raise SqlError(f"HAVING on the column {col}: HAVING filters aggregations, move the condition to WHERE")

    # cond := or
    def cond(self) -> FilterNode:
        left = self.and_()
        kids = [left]
        while self.take_kw("OR"):
            kids.append(self.and_())
        return kids[0] if len(kids) == 1 else Filter("OR", kids)

    def and_(self) -> FilterNode:
        kids = [self.not_()]
        while self.kw("AND"):
            self.i += 1
            kids.append(self.not_())
        return kids[0] if len(kids) == 1 else Filter("AND", kids)

    def not_(self) -> FilterNode:
        if self.take_kw("NOT"):
            return Filter("NOT", [self.not_()])
        if self.peek() == ("op", "("):
            start = self.i
            try:   # (cond), unless the parenthesis opens the expression on a comparison's left: `(x + 1) * 2 > 3`
                self.i += 1
                c = self.cond()
                self.expect_op(")")
                if self.peek()[0] != "op" or self.peek()[1] == ")":
                    return c
            except SqlError:
                pass
            self.i = start
        return self.comparison()

    def pattern(self) -> str:
        k, v = self.peek()
        if k != "str":
            raise SqlError(f"expected a string pattern, got {self.peek()}")
        self.i += 1
        return v

    def comparison(self) -> FilterNode:
        k, v = self.peek()
        if k == "id" and v.upper() == "REGEXP_LIKE" and self.toks[self.i + 1:self.i + 2] == [("op", "(")]:
            if self.having is not None:
                raise SqlError("REGEXP_LIKE in HAVING: HAVING filters aggregations, move the condition to WHERE")
            self.i += 2
            col = self.column()
            self.expect_op(",")
            pat = self.pattern()
            if self.peek() == ("op", ","):
                raise SqlError("REGEXP_LIKE with match flags is not supported")
            self.expect_op(")")
            return Predicate("REGEXP_LIKE", col, [pat])
        if self.having is not None:
            col = self.having_operand()
        else:
            col, left_literal, left_value = self.operand()
            if left_literal:   # PredicateComparisonRewriter: `literal op x` is `x op' literal`
                k, op = self.peek()
                if k != "op" or op not in _FLIPPED:
                    raise SqlError(f"expected a comparison operator after the literal {col}")
                self.i += 1
                right, right_literal, _ = self.operand()
                if right_literal:
                    raise SqlError(f"a comparison of two literals ({col} {op} {right}) is not supported")
                return _comparison(right, _FLIPPED[op], left_value)
        if self.take_kw("BETWEEN"):
            lo = self.bound("BETWEEN")
            self.expect_kw("AND")
            hi = self.bound("BETWEEN")
            return Predicate("RANGE", col, [], lo, hi, True, True)
        negate = self.take_kw("NOT")
        if self.take_kw("LIKE"):
            if self.having is not None:
                raise SqlError("LIKE in HAVING: HAVING compares aggregations with numbers")
            leaf = Predicate("REGEXP_LIKE", col, [like_to_regexp(self.pattern())])
            return Filter("NOT", [leaf]) if negate else leaf
        if self.take_kw("IN"):
            self.expect_op("(")
            vals = [self.bound("IN")]
            while self.take_op(","):
                vals.append(self.bound("IN"))
            self.expect_op(")")
            return Predicate("NOT_IN" if negate else "IN", col, vals)
        if negate:
            raise SqlError("NOT must be followed by IN or LIKE here")
        k, op = self.peek()
        if k != "op":
            raise SqlError(f"expected comparison operator, got {self.peek()}")
        self.i += 1
        if self.having is not None:
            return _comparison(col, op, self.literal())
        right, right_literal, v = self.operand()
        if not right_literal:   # PredicateComparisonRewriter: `a op b` is `minus(a,b) op 0`
            return _comparison(f"minus({col},{right})", op, 0)
        return _comparison(col, op, v)

    def operand(self):
        """One side of a WHERE comparison: (canonical text, is it a literal, the literal's value or None)."""
        start = self.i
        text, is_literal = self._additive()
        if not is_literal:
            return text, False, None
        if self.i != start + 1:
            raise SqlError(f"the constant expression {text} in a comparison is not supported")
        return text, True, self.toks[start][1]

    def bound(self, what: str):
        """A BETWEEN bound or an IN value: a literal (a column there is refused, as the reference's compiler does)."""
        if self.peek()[0] not in ("num", "str"):
            raise SqlError(f"{what} with a column or an expression among its {'bounds' if what == 'BETWEEN' else 'values'} "
                           f"is not supported, got {self.peek()}")
        return self.literal()


# `literal op x` written as `x op' literal`
_FLIPPED = {"=": "=", "!=": "!=", "<>": "<>", "<": ">", "<=": ">=", ">": "<", ">=": "<="}

# CASE WHEN (DESIGN.md section 3.19): the functions that take it, and its comparisons by canonical name
_CASE_FUNCTIONS = ("SUM", "AVG", "MIN", "MAX", "COUNT")
_CASE_OPS = {"=": "equals", "!=": "not_equals", "<>": "not_equals", "<": "less_than", "<=": "less_than_or_equal",
             ">": "greater_than", ">=": "greater_than_or_equal"}


def _quote(s: str) -> str:
    return "'" + s.replace("'", "''") + "'"


def _case_literal_text(v) -> str:
    """A CASE condition literal: strings as written, numbers by value.  A decimal literal beyond 2^53 keeps a decimal
    form ('1e+16'): it is integral as a double, and a LONG column refuses it rather than compare with its rounding."""
    if isinstance(v, str):
        return _quote(v)
    if isinstance(v, float) and math.isfinite(v) and abs(v) >= 2.0 ** 53:
        return f"'{v!r}'"
    return _literal_text(v)


def _comparison(col: str, op: str, v) -> Predicate:
    if op == "=":
        return Predicate("EQ", col, [v])
    if op in ("!=", "<>"):
        return Predicate("NEQ", col, [v])
    if op == ">":
        return Predicate("RANGE", col, [], v, None, False, True)
    if op == ">=":
        return Predicate("RANGE", col, [], v, None, True, True)
    if op == "<":
        return Predicate("RANGE", col, [], None, v, True, False)
    if op == "<=":
        return Predicate("RANGE", col, [], None, v, True, True)
    raise SqlError(f"unsupported operator {op}")


def resolve_order_by(query: QueryContext) -> List[tuple]:
    """ORDER BY expressions -> [(kind, index, ascending)]: kind "GROUP_BY" indexes query.group_by, "AGG" indexes
    query.aggregations (the first one the expression names), "POST" indexes query.post_aggregations (an arithmetic
    expression over aggregations of the SELECT list, matched by its normalised text).  Anything else is refused: ORDER BY
    on column expressions or on functions that are not in the SELECT list is outside this path."""
    out = []
    for expr, asc in query.order_by:
        if expr in query.group_by:
            out.append(("GROUP_BY", query.group_by.index(expr), asc))
            continue
        post = next((i for i, pa in enumerate(query.post_aggregations) if pa.text == expr), None)
        if post is not None:
            out.append(("POST", post, asc))
            continue
        m = re.fullmatch(r"([A-Za-z_$][A-Za-z0-9_$]*)\((.+?)(?:,([-+0-9.eE]+))?\)", expr)
        found = None
        for a, agg in enumerate(query.aggregations):
            if agg.function in WITHTIME_FUNCTIONS and having_name(agg) == expr:
                found = a
                break
        if found is None and m and _is_function(m.group(1)):
            fn, col = _ALIASES.get(m.group(1).upper(), m.group(1).upper()), m.group(2)
            arg = None if m.group(3) is None else float(m.group(3))
            for a, agg in enumerate(query.aggregations):
                if agg.function == fn and (fn == "COUNT" or agg.column == col) and (fn not in ("PERCENTILE", "DISTINCTCOUNTHLL") or agg.arg == arg):
                    found = a
                    break
        if found is None:
            raise SqlError(f"ORDER BY {expr}: neither a GROUP BY column nor an aggregation of the SELECT list")
        if query.aggregations[found].value_type == "STRING":
            raise SqlError(f"ORDER BY {expr}: a STRING FIRST/LASTWITHTIME is not ordered on this path")
        out.append(("AGG", found, asc))
    return out


def _same_aggregation(a: Aggregation, b: Aggregation) -> bool:
    """a computes what the HAVING leaf b names (a FILTER clause makes it another aggregation)."""
    return a.filter is None and having_name(a) == having_name(b)


def resolve_having(query: QueryContext) -> List[tuple]:
    """HAVING -> the library's postfix form (pb200_having), root last: ("AND" | "OR", operands), ("NOT",),
    ("EQ" | "NEQ", agg, value), ("RANGE", agg, lo or None, hi or None, lo inclusive, hi inclusive), where agg indexes
    query.aggregations and values are floats.  IN becomes an OR of EQ leaves, NOT IN an AND of NEQ leaves.  [] without
    HAVING; more than MAX_HAVING_NODES nodes is refused."""
    if query.having is None:
        return []
    out: List[tuple] = []

    def index(name):
        for a, agg in enumerate(query.aggregations):
            if agg.filter is None and having_name(agg) == name:
                if agg.value_type == "STRING":
                    raise SqlError(f"HAVING {name}: a STRING FIRST/LASTWITHTIME is not compared on this path")
                return a
        raise SqlError(f"HAVING {name}: no aggregation of the query computes it")

    def walk(n):
        if isinstance(n, Filter):
            for c in n.children:
                walk(c)
            out.append(("NOT",) if n.type == "NOT" else (n.type, len(n.children)))
            return
        a = index(n.column)
        if n.type in ("EQ", "NEQ"):
            out.append((n.type, a, float(n.values[0])))
        elif n.type in ("IN", "NOT_IN"):
            leaf = "EQ" if n.type == "IN" else "NEQ"
            out.extend((leaf, a, float(v)) for v in n.values)
            if len(n.values) > 1:
                out.append(("OR" if n.type == "IN" else "AND", len(n.values)))
        else:
            out.append(("RANGE", a, None if n.lower is None else float(n.lower), None if n.upper is None else float(n.upper),
                        n.lower_inclusive, n.upper_inclusive))

    walk(query.having)
    if len(out) > MAX_HAVING_NODES:
        raise SqlError(f"HAVING needs {len(out)} nodes, at most {MAX_HAVING_NODES} are supported")
    return out


def parse(sql: str, **options) -> QueryContext:
    """SQL text -> QueryContext (filter already run through the broker-side filter optimizers)."""
    p = _Parser(sql)
    p.expect_kw("SELECT")
    aggs: List[Aggregation] = []
    plain: List[str] = []
    select: List[tuple] = []
    posts: List[tuple] = []   # post-aggregation expression trees of the SELECT list
    while True:
        k, name = p.peek()
        tree = p.post_item()
        if tree is not None:
            select.append(("POST", len(posts)))
            posts.append(tree)
        elif k == "id" and _is_function(name) and p.toks[p.i + 1:p.i + 2] == [("op", "(")]:
            p.i += 2
            aggs.append(p.aggregation_call())
            select.append(("AGG", len(aggs) - 1))
            if p.take_kw("FILTER"):   # SUM(x) FILTER (WHERE cond)
                p.expect_op("(")
                p.expect_kw("WHERE")
                aggs[-1].filter = optimize_filter(p.cond())
                p.expect_op(")")
        else:
            plain.append(p.column())
            select.append(("COLUMN", plain[-1]))
        if not p.take_op(","):
            break
    p.expect_kw("FROM")
    table = p.ident()
    flt: Optional[FilterNode] = None
    if p.take_kw("WHERE"):
        flt = p.cond()
    group_by: List[str] = []
    if p.take_kw("GROUP"):
        p.expect_kw("BY")
        group_by.append(p.column())
        while p.take_op(","):
            group_by.append(p.column())
    having: Optional[FilterNode] = None
    if p.take_kw("HAVING"):
        if not group_by:
            raise SqlError("HAVING needs a GROUP BY (HAVING on an aggregation-only query is not supported)")
        p.having = []
        having = flatten(p.cond())
        for agg in p.having:   # aggregations named only in HAVING: hidden extra aggregations
            if not any(_same_aggregation(a, agg) for a in aggs):
                agg.hidden = True
                aggs.append(agg)
        p.having = None
    order_by = []
    if p.take_kw("ORDER"):
        p.expect_kw("BY")
        while True:
            k, name = p.peek()
            tree = p.post_item()
            if tree is not None:
                expr = _post_text(tree)
                if expr not in (_post_text(t) for t in posts):
                    raise SqlError(f"ORDER BY {expr}: an expression over aggregations must also be a SELECT item")
            elif k == "id" and _is_function(name) and p.toks[p.i + 1:p.i + 2] == [("op", "(")]:
                p.i += 2
                if name.upper().startswith("PERCENTILE"):
                    inner, pct = p.percentile_call(name)
                    p.expect_op(")")
                    expr = f"percentile({inner},{pct!r})"
                elif name.upper() in WITHTIME_FUNCTIONS:
                    expr = having_name(p.withtime_call(name.upper()))
                    p.expect_op(")")
                elif name.upper() == "DISTINCTCOUNTHLL":
                    inner, log2m = p.hll_call()
                    p.expect_op(")")
                    expr = f"distinctcounthll({inner},{log2m})"
                elif p.take_kw("DISTINCT"):
                    inner = p.distinct_call(name.upper())
                    p.expect_op(")")
                    expr = f"{_DISTINCT_OF[name.upper()].lower()}({inner})"
                else:
                    if p.kw("CASE") and name.upper() in _CASE_FUNCTIONS:   # named as in the SELECT list
                        inner = p.case_expr()
                        if name.upper() == "COUNT":
                            inner = "*"
                    else:
                        inner = "*" if p.take_op("*") else p.column()
                    p.expect_op(")")
                    expr = f"{name.lower()}({inner})"
            else:
                expr = p.column()
            asc = True
            if p.take_kw("DESC"):
                asc = False
            else:
                p.take_kw("ASC")
            order_by.append((expr, asc))
            if not p.take_op(","):
                break
    limit = 10
    if p.take_kw("LIMIT"):
        limit = int(p.literal())
    if p.peek()[0] is not None:
        raise SqlError(f"trailing tokens: {p.toks[p.i:]}")
    for c in plain:
        if c not in group_by:
            raise SqlError(f"column {c} must appear in GROUP BY (selection queries are outside this path)")
    post_aggregations = [_post_program(tree, aggs) for tree in posts]
    if not aggs:
        raise SqlError("only aggregation / group-by queries are on this path")
    query = QueryContext(aggregations=aggs, filter=optimize_filter(flt), group_by=group_by, table=table, limit=limit,
                         order_by=order_by, having=having, post_aggregations=post_aggregations, select=select, **options)
    resolve_order_by(query)
    resolve_having(query)
    return query


def _post_program(tree, aggs: List[Aggregation]) -> PostAggregation:
    """A post-aggregation expression tree -> its PostAggregation over `aggs`: each operand is the first aggregation that
    computes it (same function, arguments and FILTER clause), or a hidden one appended to `aggs`."""
    program: List[tuple] = []

    def emit(t):
        if t[0] == "AGG":
            found = next((a for a, x in enumerate(aggs) if having_name(x) == having_name(t[1]) and x.filter == t[1].filter), None)
            if found is None:
                t[1].hidden = True
                aggs.append(t[1])
                found = len(aggs) - 1
            program.append(("AGG", found))
        elif t[0] == "LIT":
            program.append(("LIT", float(t[1])))
        else:
            for c in t[1:]:
                emit(c)
            program.append((t[0],))

    emit(tree)
    if len(program) > MAX_POST_NODES:
        raise SqlError(f"{_post_text(tree)} needs {len(program)} nodes, at most {MAX_POST_NODES} are supported")
    return PostAggregation(_post_text(tree), program)


@dataclass
class SelectionQuery:
    """SELECT columns FROM table WHERE ... [ORDER BY col [ASC|DESC], ...] LIMIT n (the reference's selection query shape).
    columns None: SELECT * (the segment's columns in name order)."""
    columns: Optional[List[str]]
    filter: Optional[FilterNode] = None
    order_by: List[tuple] = field(default_factory=list)  # (column, ascending)
    limit: int = 10
    table: str = "testTable"


def is_selection(sql: str) -> bool:
    """True when the select list holds no aggregation function (the statement is a selection query)."""
    p = _Parser(sql)
    if not p.take_kw("SELECT"):
        return False
    while p.peek()[0] is not None and not p.kw("FROM"):
        k, v = p.peek()
        p.i += 1
        if k == "id" and _is_function(v) and p.take_op("("):
            return False
    return True


def parse_selection(sql: str) -> SelectionQuery:
    """SQL text of a selection query -> SelectionQuery (filter run through the broker-side filter optimizers)."""
    p = _Parser(sql)
    p.expect_kw("SELECT")
    columns: Optional[List[str]] = []
    if p.take_op("*"):
        columns = None
    else:
        while True:
            k, name = p.peek()
            if k == "id" and _is_function(name) and p.toks[p.i + 1:p.i + 2] == [("op", "(")]:
                raise SqlError(f"{name}(...) in a selection query: aggregations go through parse()")
            columns.append(p.column())
            if not p.take_op(","):
                break
    p.expect_kw("FROM")
    table = p.ident()
    flt: Optional[FilterNode] = None
    if p.take_kw("WHERE"):
        flt = p.cond()
    if p.kw("GROUP"):
        raise SqlError("GROUP BY needs an aggregation in the select list")
    order_by = []
    if p.take_kw("ORDER"):
        p.expect_kw("BY")
        while True:
            name = p.column()
            asc = not p.take_kw("DESC")
            if asc:
                p.take_kw("ASC")
            order_by.append((name, asc))
            if not p.take_op(","):
                break
    limit = 10
    if p.take_kw("LIMIT"):
        limit = p.literal()
        if not isinstance(limit, int) or limit < 0:
            raise SqlError(f"LIMIT must be a non-negative integer, got {limit!r}")
    if p.peek()[0] is not None:
        raise SqlError(f"trailing tokens: {p.toks[p.i:]}")
    return SelectionQuery(columns=columns, filter=optimize_filter(flt), order_by=order_by, limit=limit, table=table)


@dataclass
class DistinctQuery:
    """SELECT DISTINCT columns FROM table WHERE ... [ORDER BY col [ASC|DESC], ...] LIMIT n (the reference's DISTINCT
    query shape).  Every order column is one of `columns`."""
    columns: List[str]
    filter: Optional[FilterNode] = None
    order_by: List[tuple] = field(default_factory=list)  # (column, ascending)
    limit: int = 10
    table: str = "testTable"


def is_distinct(sql: str) -> bool:
    """True when the statement starts with SELECT DISTINCT."""
    p = _Parser(sql)
    return p.take_kw("SELECT") and p.kw("DISTINCT")


def parse_distinct(sql: str) -> DistinctQuery:
    """SQL text of a SELECT DISTINCT query -> DistinctQuery (filter run through the broker-side filter optimizers)."""
    p = _Parser(sql)
    p.expect_kw("SELECT")
    p.expect_kw("DISTINCT")
    if p.peek() == ("op", "*"):
        raise SqlError("DISTINCT * is not supported: name the columns")
    columns: List[str] = []
    while True:
        k, name = p.peek()
        if k == "id" and _is_function(name) and p.toks[p.i + 1:p.i + 2] == [("op", "(")]:
            raise SqlError(f"{name}(...) in a DISTINCT select list: aggregations are not supported")
        columns.append(p.column())
        if not p.take_op(","):
            break
    p.expect_kw("FROM")
    table = p.ident()
    flt: Optional[FilterNode] = None
    if p.take_kw("WHERE"):
        flt = p.cond()
    if p.kw("GROUP"):
        raise SqlError("GROUP BY in a DISTINCT query")
    order_by = []
    if p.take_kw("ORDER"):
        p.expect_kw("BY")
        while True:
            name = p.column()
            if name not in columns:
                raise SqlError(f"ORDER BY {name}: a DISTINCT query can only order by its selected columns")
            asc = not p.take_kw("DESC")
            if asc:
                p.take_kw("ASC")
            order_by.append((name, asc))
            if not p.take_op(","):
                break
    limit = 10
    if p.take_kw("LIMIT"):
        limit = p.literal()
        if not isinstance(limit, int) or limit < 0:
            raise SqlError(f"LIMIT must be a non-negative integer, got {limit!r}")
    if p.peek()[0] is not None:
        raise SqlError(f"trailing tokens: {p.toks[p.i:]}")
    return DistinctQuery(columns=columns, filter=optimize_filter(flt), order_by=order_by, limit=limit, table=table)
