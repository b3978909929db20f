// pb200_pattern.h -- THE matcher of REGEXP_LIKE (and of LIKE, which the SQL face rewrites into REGEXP_LIKE).
//
// One definition for every place that matches a pattern against dictionary entries: the device kernel of
// pb200_pattern.cu, and the CPU tests (tests/pattern_probe compiles this header with g++).  Semantics (DESIGN.md section
// 3.12): Java's Pattern.compile(p).matcher(value).find() -- an unanchored search, case-sensitive, no flags -- over the
// accepted subset below; everything outside it is refused by the compiler, so that the stock operator answers.
//
//   literal code points (UTF-8), `\` before a non-alphanumeric ASCII character, \t \n \r \f \a \e \xhh \uhhhh,
//   \d \D \w \W \s \S (ASCII classes), `.` (any code point but \n \r U+0085 U+2028 U+2029), [...] and [^...] with
//   members, ranges and the escapes above, (...) (?:...) and |, the quantifiers * + ? {n} {n,} {n,m} (lazy forms
//   too: the boolean answer is the same), `^` as the first character and `$` as the last.
//
// The compiler (host only) builds a bit-parallel Glushkov automaton over code points: at most 64 positions, the sets
// `first` and `last`, `nullable`, and Follow(D) as eight 256-entry tables indexed by the bytes of D.  The class of a
// position is a bit in an ASCII table of 128 masks, or in the mask of one interval of a partition of the non-ASCII code
// points.  pattern_match steps D' = (Follow(D) | first, while a match may start) & B(c) once per code point: no
// backtracking, time linear in the entry's length.
//
// Bytes of an entry that are not valid UTF-8 count one code point each, U+FFFD (what decoding them as a Java String
// gives): neither ASCII nor a line terminator.  Plain C++ when not compiled by nvcc.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define PB200_PHD __host__ __device__ __forceinline__
#else
#define PB200_PHD inline
#endif

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

namespace pb200 {

constexpr int kPatternMaxPositions = 64;
constexpr int kPatternMaxIntervals = 64;   // non-ASCII intervals of the class partition
constexpr uint32_t kReplacementChar = 0xFFFD;

struct alignas(16) PatternAutomaton {   // a multiple of 16 bytes: kernels copy it to shared memory as uint4
  uint64_t follow[8][256];                        // Follow(D) = OR over k of follow[k][byte k of D]
  uint64_t ascii[128];                            // B(c) of the ASCII code points
  uint64_t interval_mask[kPatternMaxIntervals];   // B(c) of the code points of interval i
  uint32_t interval_lo[kPatternMaxIntervals];     // interval i = [lo[i], lo[i + 1]), the last one up to 0x110000
  uint64_t first, last;
  int32_t num_intervals;                          // >= 1: interval 0 starts at 0x80
  int32_t num_positions;
  int32_t nullable, anchor_start, anchor_end, reserved;
};

PB200_PHD bool pattern_is_line_terminator(uint32_t c) {
  return c == '\n' || c == '\r' || c == 0x85 || c == 0x2028 || c == 0x2029;
}

// One code point of s[i, len): its value, and i advanced past it.  Malformed or truncated sequences, overlong forms,
// surrogates and values above U+10FFFF: one byte, U+FFFD.
PB200_PHD uint32_t pattern_decode(const unsigned char* s, int len, int& i) {
  const uint32_t b0 = s[i];
  if (b0 < 0x80) { i++; return b0; }
  int n;
  uint32_t c, min;
  if ((b0 & 0xE0) == 0xC0) { n = 1; c = b0 & 0x1F; min = 0x80; }
  else if ((b0 & 0xF0) == 0xE0) { n = 2; c = b0 & 0x0F; min = 0x800; }
  else if ((b0 & 0xF8) == 0xF0) { n = 3; c = b0 & 0x07; min = 0x10000; }
  else { i++; return kReplacementChar; }
  if (i + n > len - 1) { i++; return kReplacementChar; }   // truncated
  for (int k = 1; k <= n; k++) {
    const uint32_t b = s[i + k];
    if ((b & 0xC0) != 0x80) { i++; return kReplacementChar; }
    c = (c << 6) | (b & 0x3F);
  }
  if (c < min || c > 0x10FFFF || (c >= 0xD800 && c <= 0xDFFF)) { i++; return kReplacementChar; }
  i += n + 1;
  return c;
}

PB200_PHD uint64_t pattern_class_mask(const PatternAutomaton& a, uint32_t c) {
  if (c < 128) return a.ascii[c];
  int lo = 0, hi = a.num_intervals - 1;   // the last interval whose start is <= c
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.interval_lo[mid] <= c) lo = mid; else hi = mid - 1;
  }
  return a.interval_mask[lo];
}

PB200_PHD uint64_t pattern_follow(const PatternAutomaton& a, uint64_t d) {
  uint64_t f = 0;
#ifdef __CUDACC__
#pragma unroll
#endif
  for (int k = 0; k < 8; k++) f |= a.follow[k][(d >> (8 * k)) & 0xFF];
  return f;
}

// find() of the automaton's pattern in the len bytes at s.  A match ending after j code points exists iff the state
// after them holds a `last` position, or the pattern matches the empty string where a match may start.  `$` accepts at
// the end, before one final line terminator, and before a final \r\n (Java's Dollar without MULTILINE).
PB200_PHD bool pattern_match(const PatternAutomaton& a, const unsigned char* s, int len) {
  if (a.nullable && !a.anchor_end) return true;   // the empty match at 0
  uint64_t d = 0;
  // with `$`: the states after n - 2, n - 1 and n code points, and the last two code points
  uint64_t d1 = 0, d2 = 0;
  uint32_t c1 = 0, c2 = 0;
  int j = 0;
  for (int i = 0; i < len; j++) {
    const uint32_t c = pattern_decode(s, len, i);
    const uint64_t start = (!a.anchor_start || j == 0) ? a.first : 0;
    d2 = d1; d1 = d;
    c2 = c1; c1 = c;
    d = (pattern_follow(a, d) | start) & pattern_class_mask(a, c);
    if (!a.anchor_end) {
      if (d & a.last) return true;
      if (d == 0 && a.anchor_start) return false;
    }
  }
  if (!a.anchor_end) return false;
  // `$` positions: n; n - 1 before a final line terminator (not the \n of a final \r\n); n - 2 before a final \r\n
  auto ok = [&](uint64_t state, int at) { return (state & a.last) != 0 || (a.nullable && (!a.anchor_start || at == 0)); };
  if (ok(d, j)) return true;
  if (j >= 1 && pattern_is_line_terminator(c1) && !(c1 == '\n' && j >= 2 && c2 == '\r') && ok(d1, j - 1)) return true;
  if (j >= 2 && c2 == '\r' && c1 == '\n' && ok(d2, j - 2)) return true;
  return false;
}

// ---- the compiler (host only) ------------------------------------------------------------------------------------
enum { PATTERN_OK = 0, PATTERN_UNSUPPORTED = 1, PATTERN_INVALID = 2 };

namespace pattern_detail {

using Ranges = std::vector<std::pair<uint32_t, uint32_t>>;   // inclusive code-point ranges

struct Node {
  enum Kind { EMPTY, CHARS, CAT, ALT, STAR, PLUS, OPT, REPEAT } kind = EMPTY;
  Ranges chars;                 // CHARS
  std::vector<int> kids;        // CAT / ALT: operands; STAR / PLUS / OPT / REPEAT: one
  int min = 0, max = -1;        // REPEAT: {min, max}, max -1 = unbounded
};

inline Ranges normalized(Ranges r) {
  std::sort(r.begin(), r.end());
  Ranges out;
  for (auto& x : r) {
    if (!out.empty() && x.first <= out.back().second + 1) out.back().second = std::max(out.back().second, x.second);
    else out.push_back(x);
  }
  return out;
}

inline Ranges complement(const Ranges& r0) {
  Ranges r = normalized(r0), out;
  uint32_t next = 0;
  for (auto& x : r) {
    if (x.first > next) out.push_back({next, x.first - 1});
    next = x.second + 1;
  }
  if (next <= 0x10FFFF) out.push_back({next, 0x10FFFF});
  return out;
}

struct Parser {
  std::vector<uint32_t> cp;   // the pattern's code points
  size_t i = 0;
  std::vector<Node> nodes;
  int status = PATTERN_OK;
  std::string why;

  int fail(const char* w) { if (status == PATTERN_OK) { status = PATTERN_UNSUPPORTED; why = w; } return -1; }
  int add(Node n) { nodes.push_back(std::move(n)); return (int)nodes.size() - 1; }
  bool at_end() const { return i >= cp.size(); }
  uint32_t peek() const { return cp[i]; }

  static int hex(uint32_t c) {
    if (c >= '0' && c <= '9') return (int)(c - '0');
    if (c >= 'a' && c <= 'f') return (int)(c - 'a' + 10);
    if (c >= 'A' && c <= 'F') return (int)(c - 'A' + 10);
    return -1;
  }
  static bool alnum(uint32_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }

  // After a `\`: the escape's code points (one for a literal, a class for \d ...).  *single = it is one code point.
  bool escape(Ranges& out, bool* single) {
    if (at_end()) { fail("a trailing \\"); return false; }
    const uint32_t c = cp[i++];
    *single = true;
    auto one = [&](uint32_t v) { out.push_back({v, v}); return true; };
    switch (c) {
      case 't': return one('\t');
      case 'n': return one('\n');
      case 'r': return one('\r');
      case 'f': return one('\f');
      case 'a': return one(7);
      case 'e': return one(27);
      case 'x': case 'u': {
        const int digits = c == 'x' ? 2 : 4;
        uint32_t v = 0;
        for (int k = 0; k < digits; k++) {
          if (at_end() || hex(peek()) < 0) { fail("\\x needs two hex digits, \\u four"); return false; }
          v = v * 16 + (uint32_t)hex(cp[i++]);
        }
        if (v >= 0xD800 && v <= 0xDFFF) { fail("a surrogate escape"); return false; }
        return one(v);
      }
      case 'd': case 'D': case 'w': case 'W': case 's': case 'S': {
        Ranges r;
        const uint32_t l = c | 0x20;
        if (l == 'd') r = {{'0', '9'}};
        else if (l == 'w') r = {{'0', '9'}, {'A', 'Z'}, {'_', '_'}, {'a', 'z'}};
        else r = {{'\t', '\r'}, {' ', ' '}};   // [ \t\n\x0B\f\r]
        if (c != l) r = complement(r);
        out.insert(out.end(), r.begin(), r.end());
        *single = false;
        return true;
      }
      default:
        if (c < 128 && !alnum(c)) return one(c);
        fail("an escape outside the accepted set");
        return false;
    }
  }

  int char_class() {   // after `[`
    bool negate = false;
    if (!at_end() && peek() == '^') { negate = true; i++; }
    if (!at_end() && peek() == ']') return fail("] right after [ or [^");
    Ranges set;
    bool have_prev = false;   // the previous member was a single code point that can open a range
    uint32_t prev = 0;
    bool dash_pending = false;
    while (true) {
      if (at_end()) return fail("an unterminated class");
      const uint32_t c = cp[i];
      if (c == ']') {
        if (dash_pending) return fail("an unescaped - not between two members");
        i++;
        break;
      }
      if (c == '[') return fail("a nested [ in a class");
      if (c == '&' && i + 1 < cp.size() && cp[i + 1] == '&') return fail("&& in a class");
      if (c == '-') {
        if (dash_pending || !have_prev) return fail("an unescaped - not between two members");
        dash_pending = true;
        i++;
        continue;
      }
      Ranges member;
      bool single = true;
      i++;
      if (c == '\\') { if (!escape(member, &single)) return -1; }
      else member.push_back({c, c});
      if (dash_pending) {
        if (!single) return fail("a class escape as a range bound");
        const uint32_t hi = member[0].first;
        if (hi < prev) return fail("a range with its bounds reversed");
        set.push_back({prev, hi});
        dash_pending = false;
        have_prev = false;
        continue;
      }
      set.insert(set.end(), member.begin(), member.end());
      have_prev = single;
      prev = single ? member[0].first : 0;
    }
    Node n;
    n.kind = Node::CHARS;
    n.chars = normalized(negate ? complement(set) : set);
    return add(std::move(n));
  }

  int atom() {
    const uint32_t c = cp[i++];
    Node n;
    n.kind = Node::CHARS;
    switch (c) {
      case '(': {
        if (!at_end() && peek() == '?') {
          if (i + 1 < cp.size() && cp[i + 1] == ':') i += 2;
          else return fail("(? other than (?:");
        }
        const int inner = alternation();
        if (inner < 0) return -1;
        if (at_end() || peek() != ')') return fail("an unclosed (");
        i++;
        return inner;
      }
      case '[': return char_class();
      case '.': n.chars = complement({{'\n', '\n'}, {'\r', '\r'}, {0x85, 0x85}, {0x2028, 0x2029}}); return add(std::move(n));
      case '\\': {
        bool single;
        if (!escape(n.chars, &single)) return -1;
        n.chars = normalized(n.chars);
        return add(std::move(n));
      }
      case ')': return fail("an unmatched )");
      case ']': case '{': case '}': return fail("an unescaped ], { or } outside a valid construct");
      case '*': case '+': case '?': return fail("a quantifier with nothing to repeat");
      case '^': case '$': return fail("^ or $ other than at the ends of the pattern");
      default: n.chars = {{c, c}}; return add(std::move(n));
    }
  }

  // {n}, {n,}, {n,m} after `{`; false (and failed) when it is not one
  bool counted(int* lo, int* hi) {
    auto number = [&](int* v) {
      if (at_end() || peek() < '0' || peek() > '9') return false;
      long long x = 0;
      while (!at_end() && peek() >= '0' && peek() <= '9') { x = std::min<long long>(x * 10 + (cp[i++] - '0'), 1 << 30); }
      *v = (int)x;
      return true;
    };
    if (!number(lo)) { fail("an unescaped { outside a valid construct"); return false; }
    *hi = *lo;
    if (!at_end() && peek() == ',') {
      i++;
      if (!at_end() && peek() == '}') *hi = -1;
      else if (!number(hi)) { fail("an unescaped { outside a valid construct"); return false; }
    }
    if (at_end() || peek() != '}') { fail("an unescaped { outside a valid construct"); return false; }
    i++;
    if (*hi >= 0 && *lo > *hi) { fail("{n,m} with n > m"); return false; }
    return true;
  }

  int quantified() {
    int a = atom();
    if (a < 0) return -1;
    if (at_end()) return a;
    const uint32_t q = peek();
    Node n;
    if (q == '*') { n.kind = Node::STAR; i++; }
    else if (q == '+') { n.kind = Node::PLUS; i++; }
    else if (q == '?') { n.kind = Node::OPT; i++; }
    else if (q == '{') { i++; n.kind = Node::REPEAT; if (!counted(&n.min, &n.max)) return -1; }
    else return a;
    if (!at_end() && peek() == '?') i++;                 // lazy: the same boolean answer
    else if (!at_end() && peek() == '+') return fail("a possessive quantifier");
    if (!at_end() && (peek() == '*' || peek() == '+' || peek() == '?' || peek() == '{'))
      return fail("a quantifier with nothing to repeat");
    n.kids = {a};
    return add(std::move(n));
  }

  int sequence() {
    Node n;
    n.kind = Node::CAT;
    while (!at_end() && peek() != '|' && peek() != ')') {
      const int k = quantified();
      if (k < 0) return -1;
      n.kids.push_back(k);
    }
    if (n.kids.empty()) n.kind = Node::EMPTY;
    return add(std::move(n));
  }

  int alternation() {
    Node n;
    n.kind = Node::ALT;
    while (true) {
      const int k = sequence();
      if (k < 0) return -1;
      n.kids.push_back(k);
      if (at_end() || peek() != '|') break;
      i++;
    }
    return n.kids.size() == 1 ? n.kids[0] : add(std::move(n));
  }
};

// Glushkov construction; positions numbered in order of appearance, counted repeats expanded into copies
struct Glushkov {
  const std::vector<Node>& nodes;
  std::vector<Ranges> pos_chars;
  uint64_t follow[kPatternMaxPositions] = {};
  bool overflow = false;
  struct Sets { uint64_t first = 0, last = 0; bool nullable = true; };

  explicit Glushkov(const std::vector<Node>& n) : nodes(n) {}

  void link(uint64_t from, uint64_t to) {
    for (int p = 0; p < kPatternMaxPositions; p++) if ((from >> p) & 1) follow[p] |= to;
  }
  Sets cat(Sets a, Sets b) {
    link(a.last, b.first);
    Sets r;
    r.first = a.first | (a.nullable ? b.first : 0);
    r.last = b.last | (b.nullable ? a.last : 0);
    r.nullable = a.nullable && b.nullable;
    return r;
  }
  Sets star(Sets a) { link(a.last, a.first); a.nullable = true; return a; }

  Sets build(int id) {
    Sets s;
    if (overflow) return s;
    const Node& n = nodes[id];
    switch (n.kind) {
      case Node::EMPTY: return s;
      case Node::CHARS: {
        if ((int)pos_chars.size() >= kPatternMaxPositions) { overflow = true; return s; }
        const int p = (int)pos_chars.size();
        pos_chars.push_back(n.chars);
        s.first = s.last = 1ull << p;
        s.nullable = false;
        return s;
      }
      case Node::CAT:
        for (int k : n.kids) s = cat(s, build(k));
        return s;
      case Node::ALT: {
        s.nullable = false;
        for (int k : n.kids) { Sets t = build(k); s.first |= t.first; s.last |= t.last; s.nullable |= t.nullable; }
        return s;
      }
      case Node::STAR: return star(build(n.kids[0]));
      case Node::PLUS: { Sets a = build(n.kids[0]); link(a.last, a.first); return a; }
      case Node::OPT: { Sets a = build(n.kids[0]); a.nullable = true; return a; }
      case Node::REPEAT: {
        // a{n,m} = a^n (a (a (...)?)?)? ; a{n,} = a^n a*
        if (n.min > kPatternMaxPositions || (n.max > kPatternMaxPositions)) { overflow = true; return s; }
        for (int k = 0; k < n.min && !overflow; k++) s = cat(s, build(n.kids[0]));
        if (n.max < 0) return cat(s, star(build(n.kids[0])));
        // the optional part (a (a (...)?)?)?, folded from the innermost copy outwards
        std::vector<Sets> copies;
        for (int k = n.min; k < n.max && !overflow; k++) copies.push_back(build(n.kids[0]));
        Sets tail;
        for (size_t k = copies.size(); k-- > 0;) { tail = cat(copies[k], tail); tail.nullable = true; }
        return cat(s, tail);
      }
    }
    return s;
  }
};

// UTF-8 text -> code points; false when it is not valid UTF-8
inline bool decode_pattern(const char* text, std::vector<uint32_t>& out) {
  const unsigned char* s = (const unsigned char*)text;
  const int len = (int)strlen(text);
  for (int i = 0; i < len;) {
    const int at = i;
    const uint32_t c = pattern_decode(s, len, i);
    if (c == kReplacementChar && !(i - at == 3 && s[at] == 0xEF && s[at + 1] == 0xBF && s[at + 2] == 0xBD)) return false;
    out.push_back(c);
  }
  return true;
}

}  // namespace pattern_detail

// Compiles `text` (UTF-8, NUL-terminated) into *a.  PATTERN_OK; PATTERN_INVALID when it is not valid UTF-8;
// PATTERN_UNSUPPORTED outside the accepted subset, with what was refused in *why.
inline int pattern_compile(const char* text, PatternAutomaton* a, std::string* why) {
  using namespace pattern_detail;
  Parser p;
  if (!decode_pattern(text, p.cp)) { if (why) *why = "the pattern is not valid UTF-8"; return PATTERN_INVALID; }
  PatternAutomaton r{};
  size_t end = p.cp.size();
  if (end > 0 && p.cp[0] == '^') { r.anchor_start = 1; p.i = 1; }
  if (end > p.i && p.cp[end - 1] == '$') {
    size_t backslashes = 0;   // `\$` is a literal $
    while (backslashes + 1 < end && p.cp[end - 2 - backslashes] == '\\') backslashes++;
    if (backslashes % 2 == 0) { r.anchor_end = 1; p.cp.pop_back(); }
  }
  const int root = p.alternation();
  if (root >= 0 && !p.at_end()) p.fail(p.peek() == ')' ? "an unmatched )" : "an unexpected character");
  if (p.status != PATTERN_OK) { if (why) *why = p.why; return p.status; }
  if ((r.anchor_start || r.anchor_end) && p.nodes[root].kind == Node::ALT) {
    if (why) *why = "^ or $ next to a top-level |";
    return PATTERN_UNSUPPORTED;
  }
  Glushkov g(p.nodes);
  const Glushkov::Sets s = g.build(root);
  if (g.overflow) { if (why) *why = "more than 64 automaton positions"; return PATTERN_UNSUPPORTED; }
  r.first = s.first; r.last = s.last; r.nullable = s.nullable;
  r.num_positions = (int)g.pos_chars.size();
  // the partition of the non-ASCII code points: cut at every range bound of every position's class
  std::vector<uint32_t> cuts = {0x80, 0x110000};
  for (const Ranges& rs : g.pos_chars)
    for (auto& x : rs) {
      if (x.second < 0x80) continue;
      cuts.push_back(std::max<uint32_t>(x.first, 0x80));
      cuts.push_back(x.second + 1);
    }
  std::sort(cuts.begin(), cuts.end());
  cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
  if ((int)cuts.size() - 1 > kPatternMaxIntervals) { if (why) *why = "more than 64 non-ASCII class intervals"; return PATTERN_UNSUPPORTED; }
  r.num_intervals = (int)cuts.size() - 1;
  for (int k = 0; k < r.num_intervals; k++) r.interval_lo[k] = cuts[k];
  for (int p2 = 0; p2 < r.num_positions; p2++) {
    const uint64_t bit = 1ull << p2;
    for (auto& x : g.pos_chars[p2]) {
      for (uint32_t c = x.first; c <= x.second && c < 128; c++) r.ascii[c] |= bit;
      for (int k = 0; k < r.num_intervals; k++)   // interval k lies wholly inside or outside the range
        if (cuts[k] >= x.first && cuts[k] <= x.second) r.interval_mask[k] |= bit;
    }
  }
  for (int k = 0; k < 8; k++)
    for (int b = 0; b < 256; b++) {
      uint64_t f = 0;
      for (int bit = 0; bit < 8; bit++)
        if ((b >> bit) & 1) f |= g.follow[8 * k + bit];
      r.follow[k][b] = f;
    }
  *a = r;
  return PATTERN_OK;
}

}  // namespace pb200
