"""Independent reference of REGEXP_LIKE on dictionary entries (DESIGN.md section 3.12), built on Python's `re`.

A pattern of the accepted subset is translated to an `re` pattern with the same meaning as Java's: `re.ASCII` gives
\\d \\w \\s their ASCII meanings, `.` becomes the explicit class of everything but Java's line terminators, a final `$`
becomes a lookahead for Java's end-of-input rule (the end, or before one final line terminator, but not between \\r and
\\n), \\e becomes \\x1b.  Entries are decoded with Python's strict UTF-8 codec, one code point at a time, and every byte
that does not start a valid sequence becomes U+FFFD.  The caller passes only patterns the library accepts.
"""
from __future__ import annotations

import re

_LT = "\\n\\r\\x85\\u2028\\u2029"
_DOT = f"[^{_LT}]"
_DOLLAR = f"(?:\\Z|(?=\\r\\n\\Z)|(?<!\\r)(?=\\n\\Z)|(?=[\\r\\x85\\u2028\\u2029]\\Z))"


def decode(b: bytes) -> str:
    """UTF-8 bytes -> str; every byte that does not start a valid sequence is one U+FFFD."""
    out, i = [], 0
    while i < len(b):
        lead = b[i]
        n = 1 if lead < 0x80 else 2 if lead >> 5 == 6 else 3 if lead >> 4 == 14 else 4 if lead >> 3 == 30 else 0
        try:
            if n == 0:
                raise UnicodeDecodeError("utf-8", b, i, i + 1, "bad lead byte")
            out.append(b[i:i + n].decode("utf-8", errors="strict"))
            if len(out[-1]) != 1:
                raise UnicodeDecodeError("utf-8", b, i, i + n, "short")
            i += n
        except UnicodeDecodeError:
            out.append("�")
            i += 1
    return "".join(out)


def to_python(pattern: str) -> str:
    """The `re` pattern (with re.ASCII) of an accepted Java pattern."""
    out, i, in_class = [], 0, False
    n = len(pattern)
    while i < n:
        c = pattern[i]
        if c == "\\":
            e = pattern[i + 1]
            out.append("\\x1b" if e == "e" else "\\" + e)
            i += 2
            continue
        if in_class:
            if c == "]":
                in_class = False
            out.append(c)
        elif c == "[":
            in_class = True
            out.append(c)
            if pattern[i + 1:i + 2] == "^":
                out.append("^")
                i += 1
        elif c == ".":
            out.append(_DOT)
        elif c == "$" and i == n - 1:
            out.append(_DOLLAR)
        elif c == "^" and i == 0:
            out.append("\\A")
        else:
            out.append(c)
        i += 1
    return "".join(out)


def matches(pattern: str, entry: bytes) -> bool:
    """REGEXP_LIKE(entry, pattern): Java's find() of the pattern in the entry up to its first NUL."""
    value = entry.split(b"\0", 1)[0]
    return re.search(to_python(pattern), decode(value), re.ASCII) is not None


def like_matches(like: str, value: str) -> bool:
    """SQL LIKE through the rewrite's rules, by dynamic programming over code points and independent of any regex: a
    leading (trailing) run of % leaves the start (end) free, an inner % is any run and _ any one code point, neither of
    them a line terminator; without a trailing %, the value may end with one line terminator after the match (`$`)."""
    lt = set("\n\r\x85\u2028\u2029")
    if like and set(like) == {"%"}:
        return True
    lead = len(like) - len(like.lstrip("%"))
    trail = len(like) - len(like.rstrip("%"))
    body = like[lead:len(like) - trail] if like else ""

    def exact(v):
        m, n = len(body), len(v)
        ok = [[False] * (n + 1) for _ in range(m + 1)]
        ok[0][0] = True
        for i in range(1, m + 1):
            p = body[i - 1]
            for j in range(0, n + 1):
                if p == "%":
                    ok[i][j] = ok[i - 1][j] or (j > 0 and ok[i][j - 1] and v[j - 1] not in lt)
                elif j > 0:
                    ok[i][j] = ok[i - 1][j - 1] and (v[j - 1] == p if p != "_" else v[j - 1] not in lt)
        return ok[m][n]

    n = len(value)
    ends = [n]
    if n >= 1 and value[-1] in lt and not (value[-1] == "\n" and n >= 2 and value[-2] == "\r"):
        ends.append(n - 1)
    if value.endswith("\r\n"):
        ends.append(n - 2)
    for i in (range(n + 1) if lead else [0]):
        for j in (range(i, n + 1) if trail else ends):
            if j >= i and exact(value[i:j]):
                return True
    return False
