// event_line.h -- the parse of ONE line of the `pio import` / `pio export` JSON-lines event format
// (tools/src/main/scala/org/apache/predictionio/tools/imprt/FileToEvents.scala:93-103) into the fields the event
// columns carry, shared by the device scanner (events_scan.cuh) and the CPU test driver (tests/test_event_line.py).
// Plain C++ marked __host__ __device__ under nvcc; it compiles under g++ alone.
//
// The rule that keeps it exact: for a line it either arrives at exactly what the host path
//     Event.from_json(json.loads(line.strip())) -> PEventStore.find's filter -> DataMap.get(property, float)
// arrives at, or it answers FALLBACK and the host parses that line.  It answers NOT_MATCHED / MATCHED only for lines
// inside the accepted grammar (DESIGN.md section 3.1):
//   - the whole line is strict JSON whose top level is an object, with no NaN / Infinity, no raw control character in a
//     string, only valid escapes (\uXXXX decoded to UTF-8, surrogate pairs combined, a lone surrogate falls back),
//     nesting depth <= MAX_DEPTH, integer literals of <= MAX_INT_DIGITS digits (Python refuses longer ones), and
//     length <= MAX_LINE bytes;
//   - outside strings only printable ASCII, space and tab; inside strings raw UTF-8 that passes a strict check (no
//     overlongs, no surrogates, nothing above U+10FFFF);
//   - no key the parse reads (event, entityType, entityId, targetEntityType, targetEntityId, properties, eventTime at the
//     top level, the requested property inside properties) twice at its level;
//   - event / entityType strings; entityId a string or an integer (str(int) is the token itself, except "-0");
//     targetEntityType a string or null; targetEntityId a string, an integer or null; properties an object or null;
//     eventTime present and of the form YYYY-MM-DDTHH:MM:SS[.f{1,6}][Z|+HH:MM|-HH:MM] with Python's range checks
//     (no offset = UTC);
//   - in a matched line, the property value absent or a JSON number that is exact in double: an integer of magnitude
//     <= 2^53, or a decimal whose significand is <= 2^53 and whose power of ten is within +-22 (one correctly rounded
//     multiply or divide: Clinger's fast path).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PIO_EV_HD __host__ __device__ __forceinline__
#else
#define PIO_EV_HD inline
#endif

namespace pio {
namespace ev {

constexpr int MAX_LINE = 65536;        // bytes of one line (terminator removed)
constexpr int MAX_DEPTH = 64;          // JSON nesting
constexpr int MAX_INT_DIGITS = 4300;   // CPython's default limit for int(str); json.loads raises past it
constexpr int MIN_MATCHED_BYTES = 64;  // no line shorter than this can be MATCHED (4 keys + a 19-byte time)

enum Outcome : int { FALLBACK = 0, NOT_MATCHED = 1, MATCHED = 2, BLANK = 3 /* empty after stripping spaces / tabs */ };
enum TargetMode : int { TARGET_ANY = 0, TARGET_ABSENT = 1, TARGET_EQUALS = 2 };

// UTF-8 bytes; a length < 0 means "no restriction" (entity_type) / "no property" (prop)
struct Filter {
  const uint8_t* entity_type;
  int entity_type_len;
  const uint8_t* names;         // name k = names[name_off[k] .. name_off[k + 1])
  const int* name_off;
  int n_names;                  // < 0: any event name (code -1); 0: no event matches
  int target_mode;              // TargetMode
  const uint8_t* target;
  int target_len;
  const uint8_t* prop;
  int prop_len;
  int has_start, has_until;     // eventTime >= start_us, eventTime < until_us
  int64_t start_us, until_us;
};

struct Result {
  int outcome;
  int code;          // index of the event name in Filter::names (-1 when n_names < 0)
  double value;      // the property, when has_value
  int has_value;
  int has_target;    // targetEntityId present (not absent / null)
  int64_t time_us;   // eventTime, microseconds since 1970-01-01T00:00:00Z
  int eid_len;       // decoded entityId at scratch[0 .. eid_len)
  int tid_len;       // decoded targetEntityId at scratch[eid_len .. eid_len + tid_len)
};

enum Kind : uint8_t { K_ABSENT = 0, K_STR, K_INT, K_NUM, K_NULL, K_BOOL, K_OBJ, K_ARR };
enum Slot : int { S_EVENT = 0, S_ETYPE, S_EID, S_TTYPE, S_TID, S_PROPS, S_TIME, S_PROP, N_SLOTS };

struct Span {
  int b, e;      // token bytes [b, e); strings include their quotes
  uint8_t kind;  // Kind
  uint8_t esc;   // string token contains a backslash
};

PIO_EV_HD bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
PIO_EV_HD bool is_ws(uint8_t c) { return c == ' ' || c == '\t'; }

PIO_EV_HD int hex4(const uint8_t* s, int n, int i) {
  if (i + 4 > n) return -1;
  int v = 0;
  for (int k = 0; k < 4; ++k) {
    const uint8_t c = s[i + k];
    int d;
    if (c >= '0' && c <= '9') d = c - '0';
    else if (c >= 'a' && c <= 'f') d = c - 'a' + 10;
    else if (c >= 'A' && c <= 'F') d = c - 'A' + 10;
    else return -1;
    v = v * 16 + d;
  }
  return v;
}

// length of the strict UTF-8 sequence starting at s[i] (a byte >= 0x80), or -1
PIO_EV_HD int utf8_len(const uint8_t* s, int n, int i) {
  const uint8_t c = s[i];
  int len;
  uint8_t lo = 0x80, hi = 0xBF;   // range of the second byte
  if (c >= 0xC2 && c <= 0xDF) len = 2;
  else if (c == 0xE0) { len = 3; lo = 0xA0; }
  else if ((c >= 0xE1 && c <= 0xEC) || c == 0xEE || c == 0xEF) len = 3;
  else if (c == 0xED) { len = 3; hi = 0x9F; }   // no UTF-16 surrogates
  else if (c == 0xF0) { len = 4; lo = 0x90; }
  else if (c >= 0xF1 && c <= 0xF3) len = 4;
  else if (c == 0xF4) { len = 4; hi = 0x8F; }   // nothing above U+10FFFF
  else return -1;
  if (i + len > n) return -1;
  if (s[i + 1] < lo || s[i + 1] > hi) return -1;
  for (int k = 2; k < len; ++k)
    if (s[i + k] < 0x80 || s[i + k] > 0xBF) return -1;
  return len;
}

// s[i] == '"': index past the closing quote, or -1 (FALLBACK); *esc = a backslash occurred
PIO_EV_HD int scan_string(const uint8_t* s, int n, int i, uint8_t* esc) {
  *esc = 0;
  ++i;
  while (i < n) {
    const uint8_t c = s[i];
    if (c == '"') return i + 1;
    if (c < 0x20) return -1;   // raw control character
    if (c == '\\') {
      *esc = 1;
      if (i + 1 >= n) return -1;
      const uint8_t d = s[i + 1];
      if (d == 'u') {
        const int u = hex4(s, n, i + 2);
        if (u < 0) return -1;
        i += 6;
        if (u >= 0xDC00 && u <= 0xDFFF) return -1;   // lone low surrogate
        if (u >= 0xD800 && u <= 0xDBFF) {             // high surrogate: must pair with an escaped low one
          if (i + 1 >= n || s[i] != '\\' || s[i + 1] != 'u') return -1;
          const int l = hex4(s, n, i + 2);
          if (l < 0xDC00 || l > 0xDFFF) return -1;
          i += 6;
        }
        continue;
      }
      if (d == '"' || d == '\\' || d == '/' || d == 'b' || d == 'f' || d == 'n' || d == 'r' || d == 't') {
        i += 2;
        continue;
      }
      return -1;
    }
    if (c < 0x80) {
      ++i;
      continue;
    }
    const int len = utf8_len(s, n, i);
    if (len < 0) return -1;
    i += len;
  }
  return -1;
}

// decoded UTF-8 bytes of a validated string token [b, e) into out; returns their count (<= e - b - 2)
PIO_EV_HD int decode_string(const uint8_t* s, int b, int e, uint8_t* out) {
  int i = b + 1, o = 0;
  const int end = e - 1;
  while (i < end) {
    const uint8_t c = s[i];
    if (c != '\\') {
      out[o++] = c;
      ++i;
      continue;
    }
    const uint8_t d = s[i + 1];
    if (d != 'u') {
      out[o++] = d == 'b' ? 8 : d == 'f' ? 12 : d == 'n' ? 10 : d == 'r' ? 13 : d == 't' ? 9 : d;
      i += 2;
      continue;
    }
    uint32_t u = (uint32_t)hex4(s, e, i + 2);
    i += 6;
    if (u >= 0xD800 && u <= 0xDBFF) {
      const uint32_t l = (uint32_t)hex4(s, e, i + 2);
      u = 0x10000u + ((u - 0xD800u) << 10) + (l - 0xDC00u);
      i += 6;
    }
    if (u < 0x80) {
      out[o++] = (uint8_t)u;
    } else if (u < 0x800) {
      out[o++] = (uint8_t)(0xC0 | (u >> 6));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    } else if (u < 0x10000) {
      out[o++] = (uint8_t)(0xE0 | (u >> 12));
      out[o++] = (uint8_t)(0x80 | ((u >> 6) & 0x3F));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    } else {
      out[o++] = (uint8_t)(0xF0 | (u >> 18));
      out[o++] = (uint8_t)(0x80 | ((u >> 12) & 0x3F));
      out[o++] = (uint8_t)(0x80 | ((u >> 6) & 0x3F));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    }
  }
  return o;
}

// decode_string for a string token in which a \u escape may name an unpaired surrogate (json.dumps writes one for a
// Python string that holds it): such an escape becomes '?', as Java's getBytes(UTF_8) writes an unpaired surrogate, and
// an escaped pair still becomes one 4-byte character.  A malformed escape also becomes '?'.  Never writes more than
// e - b - 2 bytes and never reads outside [b, e).
PIO_EV_HD int decode_string_lenient(const uint8_t* s, int b, int e, uint8_t* out) {
  int i = b + 1, o = 0;
  const int end = e - 1;
  while (i < end) {
    const uint8_t c = s[i];
    if (c != '\\') {
      out[o++] = c;
      ++i;
      continue;
    }
    const uint8_t d = s[i + 1];
    if (d != 'u') {
      out[o++] = d == 'b' ? 8 : d == 'f' ? 12 : d == 'n' ? 10 : d == 'r' ? 13 : d == 't' ? 9 : d;
      i += 2;
      continue;
    }
    const int h = hex4(s, end, i + 2);
    i += 6;
    uint32_t u = (uint32_t)h;
    if (h < 0 || (h >= 0xDC00 && h <= 0xDFFF)) {
      out[o++] = '?';
      continue;
    }
    if (h >= 0xD800 && h <= 0xDBFF) {
      const int l = i + 1 < end && s[i] == '\\' && s[i + 1] == 'u' ? hex4(s, end, i + 2) : -1;
      if (l < 0xDC00 || l > 0xDFFF) {
        out[o++] = '?';
        continue;
      }
      u = 0x10000u + ((u - 0xD800u) << 10) + ((uint32_t)l - 0xDC00u);
      i += 6;
    }
    if (u < 0x80) {
      out[o++] = (uint8_t)u;
    } else if (u < 0x800) {
      out[o++] = (uint8_t)(0xC0 | (u >> 6));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    } else if (u < 0x10000) {
      out[o++] = (uint8_t)(0xE0 | (u >> 12));
      out[o++] = (uint8_t)(0x80 | ((u >> 6) & 0x3F));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    } else {
      out[o++] = (uint8_t)(0xF0 | (u >> 18));
      out[o++] = (uint8_t)(0x80 | ((u >> 12) & 0x3F));
      out[o++] = (uint8_t)(0x80 | ((u >> 6) & 0x3F));
      out[o++] = (uint8_t)(0x80 | (u & 0x3F));
    }
  }
  return o;
}

PIO_EV_HD bool bytes_eq(const uint8_t* a, const uint8_t* b, int n) {
  for (int k = 0; k < n; ++k)
    if (a[k] != b[k]) return false;
  return true;
}

// decoded string token == t[0 .. tn); tmp holds the decoded bytes when the token has escapes
PIO_EV_HD bool str_eq(const uint8_t* s, const Span& sp, const uint8_t* t, int tn, uint8_t* tmp) {
  if (!sp.esc) return sp.e - sp.b - 2 == tn && bytes_eq(s + sp.b + 1, t, tn);
  if (sp.e - sp.b - 2 < tn) return false;
  return decode_string(s, sp.b, sp.e, tmp) == tn && bytes_eq(tmp, t, tn);
}

// JSON number at s[i]: index past it, or -1; *kind = K_INT (no fraction / exponent) or K_NUM
PIO_EV_HD int scan_number(const uint8_t* s, int n, int i, uint8_t* kind) {
  if (s[i] == '-') ++i;
  if (i >= n) return -1;
  const int d0 = i;
  if (s[i] == '0') ++i;
  else if (s[i] >= '1' && s[i] <= '9') while (i < n && is_digit(s[i])) ++i;
  else return -1;   // also "-Infinity"
  const int int_digits = i - d0;
  *kind = K_INT;
  if (i < n && s[i] == '.') {
    ++i;
    if (i >= n || !is_digit(s[i])) return -1;
    while (i < n && is_digit(s[i])) ++i;
    *kind = K_NUM;
  }
  if (i < n && (s[i] == 'e' || s[i] == 'E')) {
    ++i;
    if (i < n && (s[i] == '+' || s[i] == '-')) ++i;
    if (i >= n || !is_digit(s[i])) return -1;
    while (i < n && is_digit(s[i])) ++i;
    *kind = K_NUM;
  }
  if (*kind == K_INT && int_digits > MAX_INT_DIGITS) return -1;
  return i;
}

// float(json value) when it is exact in double; false = the host decides
PIO_EV_HD bool number_value(const uint8_t* s, const Span& sp, double* out) {
  const uint64_t LIM = 1ull << 53;
  int i = sp.b;
  const bool neg = s[i] == '-';
  if (neg) ++i;
  uint64_t m = 0;
  int frac = 0;
  bool in_frac = false;
  for (; i < sp.e && s[i] != 'e' && s[i] != 'E'; ++i) {
    if (s[i] == '.') {
      in_frac = true;
      continue;
    }
    const uint64_t d = (uint64_t)(s[i] - '0');
    if (m > (LIM - d) / 10) return false;   // significand above 2^53
    m = m * 10 + d;
    if (in_frac) ++frac;
  }
  if (sp.kind == K_INT) {   // Python int -> float: "-0" is the integer 0, so +0.0
    *out = neg && m ? -(double)m : (double)m;
    return true;
  }
  int ex = 0;
  bool eneg = false;
  if (i < sp.e) {
    ++i;
    if (s[i] == '+' || s[i] == '-') eneg = s[i++] == '-';
    for (; i < sp.e; ++i)
      if (ex < 100000) ex = ex * 10 + (s[i] - '0');
  }
  const int e10 = (eneg ? -ex : ex) - frac;
  double v;
  if (m == 0) {
    v = 0.0;
  } else {
    if (e10 < -22 || e10 > 22) return false;
    double p = 1.0;   // 10^|e10| <= 10^22 is exact in double, and so is every step
    for (int k = 0; k < (e10 < 0 ? -e10 : e10); ++k) p *= 10.0;
    v = e10 < 0 ? (double)m / p : (double)m * p;
  }
  *out = neg ? -v : v;
  return true;
}

PIO_EV_HD int64_t days_from_civil(int y, int m, int d) {
  y -= m <= 2;
  const int era = y / 400;   // y >= 0 here
  const int yoe = y - era * 400;
  const int doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return (int64_t)era * 146097 + doe - 719468;
}

PIO_EV_HD int two(const uint8_t* t, int i) {
  return is_digit(t[i]) && is_digit(t[i + 1]) ? (t[i] - '0') * 10 + (t[i + 1] - '0') : -1;
}

// YYYY-MM-DDTHH:MM:SS[.f{1,6}][Z|+HH:MM|-HH:MM] -> microseconds since the epoch (UTC when there is no offset), and with
// OFF the UTC offset in minutes
template <bool OFF>
PIO_EV_HD bool parse_time_t(const uint8_t* t, int n, int64_t* us, int* off) {
  if (n < 19 || t[4] != '-' || t[7] != '-' || t[10] != 'T' || t[13] != ':' || t[16] != ':') return false;
  const int y0 = two(t, 0), y1 = two(t, 2), mo = two(t, 5), d = two(t, 8), h = two(t, 11), mi = two(t, 14), sec = two(t, 17);
  if (y0 < 0 || y1 < 0 || mo < 0 || d < 0 || h < 0 || mi < 0 || sec < 0) return false;
  const int y = y0 * 100 + y1;
  if (y < 1 || mo < 1 || mo > 12 || d < 1 || h > 23 || mi > 59 || sec > 59) return false;
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  const int dim = mo == 2 ? (leap ? 29 : 28) : (mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30 : 31;
  if (d > dim) return false;
  int p = 19;
  int64_t frac = 0;
  if (p < n && t[p] == '.') {
    ++p;
    int nd = 0;
    while (p < n && is_digit(t[p]) && nd < 7) {
      frac = frac * 10 + (t[p] - '0');
      ++p;
      ++nd;
    }
    if (nd < 1 || nd > 6) return false;
    for (; nd < 6; ++nd) frac *= 10;   // ".5" is 500000 microseconds
  }
  int off_min = 0;
  if (p < n) {
    if (t[p] == 'Z' && p + 1 == n) {
      p += 1;
    } else if ((t[p] == '+' || t[p] == '-') && p + 6 == n && t[p + 3] == ':') {
      const int oh = two(t, p + 1), om = two(t, p + 4);
      if (oh < 0 || om < 0 || oh > 23 || om > 59) return false;
      off_min = (t[p] == '-' ? -1 : 1) * (oh * 60 + om);
      p += 6;
    } else {
      return false;
    }
  }
  if (p != n) return false;
  const int64_t secs = days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + sec - (int64_t)off_min * 60;
  *us = secs * 1000000 + frac;
  if constexpr (OFF) *off = off_min;
  return true;
}

PIO_EV_HD bool parse_time(const uint8_t* t, int n, int64_t* us) { return parse_time_t<false>(t, n, us, nullptr); }

PIO_EV_HD bool key_is(const uint8_t* s, const Span& k, const char* name, int len, uint8_t* tmp) {
  return str_eq(s, k, (const uint8_t*)name, len, tmp);
}

// which slot a key fills (-1: none the parse reads)
PIO_EV_HD int top_slot(const uint8_t* s, const Span& k, uint8_t* tmp) {
  const int n = k.e - k.b - 2;   // raw length; a key with escapes is at least as long as its decoded form
  if (n < 5) return -1;
  if (key_is(s, k, "event", 5, tmp)) return S_EVENT;
  if (key_is(s, k, "entityType", 10, tmp)) return S_ETYPE;
  if (key_is(s, k, "entityId", 8, tmp)) return S_EID;
  if (key_is(s, k, "targetEntityType", 16, tmp)) return S_TTYPE;
  if (key_is(s, k, "targetEntityId", 14, tmp)) return S_TID;
  if (key_is(s, k, "properties", 10, tmp)) return S_PROPS;
  if (key_is(s, k, "eventTime", 9, tmp)) return S_TIME;
  return -1;
}

PIO_EV_HD bool int_id_ok(const uint8_t* s, const Span& sp) {   // str(int(token)) == token unless the token is "-0"
  return !(sp.e - sp.b == 2 && s[sp.b] == '-' && s[sp.b + 1] == '0');
}

// Keyed parse (parse_line_keys): the top-level keys of `properties` it reports, compared after unescaping.  The list is
// an argument of its own rather than a Filter field, so that Filter keeps its layout.
constexpr int MAX_KEYS = 8;

struct KeyList {
  const uint8_t* names;   // key q = names[off[q] .. off[q + 1])
  const int* off;
  int n;                  // 1 .. MAX_KEYS
};

// per key q of a MATCHED line (all zero otherwise)
struct KeyValues {
  uint32_t present;       // bit q: the key is in `properties` (a null value counts)
  uint32_t number;        // bit q: the value is a JSON number exact in double, in num[q]
  double num[MAX_KEYS];
  int tok_b[MAX_KEYS];    // the value's raw JSON token at [tok_b, tok_e) of the line; empty for an absent key and for a
  int tok_e[MAX_KEYS];    // fractional / exponent number on the fast path (num[q] is the value); an integer keeps its
                          // token as well, so the host can tell 5 from 5.0
};

// Whole-map parse (parse_line_props): every top-level key of `properties`, for a MATCHED line (all zero otherwise).
// The keys themselves are read by a second walk over the validated object (next_prop).
struct PropsInfo {
  int n_keys;             // top-level keys of `properties`: 0 for absent, null or {}
  int b, e;               // the `properties` object at [b, e) of the line (empty when it has no keys)
  int utc_off;            // eventTime's UTC offset in minutes (0 for Z or none)
};

// One line, terminator removed.  scratch: at least n bytes (decoded ids land at its start).  KEYS == false is
// parse_line; KEYS == true also fills *kv for the keys of *kl (Filter::prop_len must be < 0 then).  A tracked key twice
// in one `properties` object makes the line FALLBACK; a number off the fast path does not (the host decodes its token).
// ALL == true (KEYS false) fills *pi instead; it takes every key, so no key makes a line FALLBACK, duplicates included.
template <bool KEYS, bool ALL = false>
PIO_EV_HD Result parse_line_t(const uint8_t* s, int n, const Filter& f, uint8_t* scratch, const KeyList* kl,
                              KeyValues* kv, PropsInfo* pi = nullptr) {
  static_assert(!(KEYS && ALL), "one mode at a time");
  Result r;
  r.outcome = FALLBACK;
  r.code = -1;
  r.value = 0.0;
  r.has_value = 0;
  r.has_target = 0;
  r.time_us = 0;
  r.eid_len = 0;
  r.tid_len = 0;
  int i = 0;
  while (i < n && is_ws(s[i])) ++i;
  if (i == n) {
    r.outcome = BLANK;
    return r;
  }
  if (n > MAX_LINE || s[i] != '{') return r;

  Span sp[N_SLOTS];
  for (int k = 0; k < N_SLOTS; ++k) sp[k].kind = K_ABSENT, sp[k].b = sp[k].e = 0, sp[k].esc = 0;
  Span ksp[KEYS ? MAX_KEYS : 1];   // the tracked keys' values; `pending` = N_SLOTS + q while key q's value is read
  if constexpr (KEYS) {
    for (int q = 0; q < MAX_KEYS; ++q) ksp[q].kind = K_ABSENT, ksp[q].b = ksp[q].e = 0, ksp[q].esc = 0;
  }
  (void)ksp;
  int kopen = -1;   // a tracked key whose value is a container (at depth 3) still open: its token ends where it closes
  (void)kopen;
  int pkeys = 0, pend = 0;   // ALL: keys of `properties` so far, and where it closes
  (void)pkeys, (void)pend;
  enum { ST_VALUE, ST_VALUE_OR_END, ST_AFTER, ST_KEY_OR_END, ST_KEY, ST_COLON };
  int st = ST_VALUE, depth = 0, pending = -1;
  uint64_t arr = 0;   // bit d - 1: the container at depth d is an array
  bool in_props = false;
  for (;;) {
    while (i < n && is_ws(s[i])) ++i;
    if (st == ST_AFTER && depth == 0) {
      if (i != n) return r;   // trailing garbage
      break;
    }
    if (i >= n) return r;
    const uint8_t c = s[i];
    if (st == ST_VALUE || st == ST_VALUE_OR_END) {
      if (st == ST_VALUE_OR_END && c == ']') {
        if constexpr (KEYS) {
          if (depth == 3 && kopen >= 0) ksp[kopen].e = i + 1, kopen = -1;
        }
        --depth;
        ++i;
        st = ST_AFTER;
        continue;
      }
      Span v;
      v.b = i;
      v.esc = 0;
      if (c == '{' || c == '[') {
        if (++depth > MAX_DEPTH) return r;
        ++i;
        const bool is_arr = c == '[';
        if (is_arr) arr |= 1ull << (depth - 1);
        else arr &= ~(1ull << (depth - 1));
        if (depth == 2) in_props = !is_arr && pending == S_PROPS;
        v.kind = is_arr ? K_ARR : K_OBJ;
        st = is_arr ? ST_VALUE_OR_END : ST_KEY_OR_END;
      } else if (depth == 0) {
        return r;   // the top level must be an object
      } else if (c == '"') {
        i = scan_string(s, n, i, &v.esc);
        if (i < 0) return r;
        v.kind = K_STR;
        st = ST_AFTER;
      } else if (c == '-' || is_digit(c)) {
        i = scan_number(s, n, i, &v.kind);
        if (i < 0) return r;
        st = ST_AFTER;
      } else if (c == 't' && i + 4 <= n && s[i + 1] == 'r' && s[i + 2] == 'u' && s[i + 3] == 'e') {
        i += 4, v.kind = K_BOOL, st = ST_AFTER;
      } else if (c == 'f' && i + 5 <= n && s[i + 1] == 'a' && s[i + 2] == 'l' && s[i + 3] == 's' && s[i + 4] == 'e') {
        i += 5, v.kind = K_BOOL, st = ST_AFTER;
      } else if (c == 'n' && i + 4 <= n && s[i + 1] == 'u' && s[i + 2] == 'l' && s[i + 3] == 'l') {
        i += 4, v.kind = K_NULL, st = ST_AFTER;
      } else {
        return r;   // NaN, Infinity, bare words, stray punctuation, bytes >= 0x80
      }
      v.e = i;
      if constexpr (KEYS) {
        if (pending >= N_SLOTS && (v.kind == K_OBJ || v.kind == K_ARR)) kopen = pending - N_SLOTS;
        if (pending >= N_SLOTS) ksp[pending - N_SLOTS] = v;
        else if (pending >= 0) sp[pending] = v;
      } else {
        if (pending >= 0) sp[pending] = v;
      }
      pending = -1;
      continue;
    }
    if (st == ST_AFTER) {
      const bool is_arr = (arr >> (depth - 1)) & 1;
      if (c == ',') {
        st = is_arr ? ST_VALUE : ST_KEY;
      } else if (c == (is_arr ? ']' : '}')) {
        if constexpr (KEYS) {
          if (depth == 3 && kopen >= 0) ksp[kopen].e = i + 1, kopen = -1;
        }
        if constexpr (ALL) {
          if (depth == 2 && in_props) pend = i + 1;
        }
        if (--depth < 2) in_props = false;
        st = ST_AFTER;
      } else {
        return r;
      }
      ++i;
      continue;
    }
    if (st == ST_KEY_OR_END && c == '}') {
      if constexpr (KEYS) {
        if (depth == 3 && kopen >= 0) ksp[kopen].e = i + 1, kopen = -1;
      }
      if constexpr (ALL) {
        if (depth == 2 && in_props) pend = i + 1;
      }
      if (--depth < 2) in_props = false;
      ++i;
      st = ST_AFTER;
      continue;
    }
    if (st == ST_KEY || st == ST_KEY_OR_END) {
      if (c != '"') return r;
      Span k;
      k.b = i;
      i = scan_string(s, n, i, &k.esc);
      if (i < 0) return r;
      k.e = i;
      k.kind = K_STR;
      int slot = -1;
      if (depth == 1) slot = top_slot(s, k, scratch);
      else if (depth == 2 && in_props && f.prop_len >= 0 && str_eq(s, k, f.prop, f.prop_len, scratch)) slot = S_PROP;
      if (slot >= 0) {
        if (sp[slot].kind != K_ABSENT) return r;   // a key the parse reads, twice at its level
        sp[slot].kind = K_NULL;                     // placeholder: seen
      }
      if constexpr (KEYS) {
        if (depth == 2 && in_props) {
          for (int q = 0; q < kl->n; ++q) {
            if (!str_eq(s, k, kl->names + kl->off[q], kl->off[q + 1] - kl->off[q], scratch)) continue;
            if (ksp[q].kind != K_ABSENT) return r;   // a tracked key twice in `properties`
            ksp[q].kind = K_NULL;
            slot = N_SLOTS + q;
            break;
          }
        }
      }
      if constexpr (ALL) {
        if (depth == 2 && in_props) ++pkeys;
      }
      pending = slot;
      st = ST_COLON;
      continue;
    }
    // ST_COLON
    if (c != ':') return r;
    ++i;
    st = ST_VALUE;
  }
  // control characters other than tab and bytes >= 0x80 outside strings were refused above: no structural position
  // accepts them

  // Event.from_json
  if (sp[S_EVENT].kind != K_STR || sp[S_ETYPE].kind != K_STR) return r;
  if (!(sp[S_EID].kind == K_STR || (sp[S_EID].kind == K_INT && int_id_ok(s, sp[S_EID])))) return r;
  const uint8_t tt = sp[S_TTYPE].kind;
  if (tt != K_ABSENT && tt != K_NULL && tt != K_STR) return r;
  const uint8_t tk = sp[S_TID].kind;
  if (!(tk == K_ABSENT || tk == K_NULL || tk == K_STR || (tk == K_INT && int_id_ok(s, sp[S_TID])))) return r;
  const uint8_t pk = sp[S_PROPS].kind;
  if (pk != K_ABSENT && pk != K_NULL && pk != K_OBJ) return r;
  if (sp[S_TIME].kind != K_STR) return r;   // absent = now() on the host
  int utc_off = 0;
  (void)utc_off;
  {
    const int tn = decode_string(s, sp[S_TIME].b, sp[S_TIME].e, scratch);
    if constexpr (ALL) {
      if (!parse_time_t<true>(scratch, tn, &r.time_us, &utc_off)) return r;
    } else {
      if (!parse_time(scratch, tn, &r.time_us)) return r;
    }
  }

  // PEventStore.find's filter
  r.outcome = NOT_MATCHED;
  if (f.has_start && r.time_us < f.start_us) return r;
  if (f.has_until && r.time_us >= f.until_us) return r;
  if (f.entity_type_len >= 0 && !str_eq(s, sp[S_ETYPE], f.entity_type, f.entity_type_len, scratch)) return r;
  if (f.n_names >= 0) {
    int code = -1;
    for (int k = 0; k < f.n_names && code < 0; ++k)
      if (str_eq(s, sp[S_EVENT], f.names + f.name_off[k], f.name_off[k + 1] - f.name_off[k], scratch)) code = k;
    if (code < 0) return r;
    r.code = code;
  }
  if (f.target_mode == TARGET_ABSENT && tt == K_STR) return r;
  if (f.target_mode == TARGET_EQUALS && (tt != K_STR || !str_eq(s, sp[S_TTYPE], f.target, f.target_len, scratch))) return r;

  // matched: the property (DataMap.get(name, float)), then the ids
  const uint8_t vk = sp[S_PROP].kind;
  if (vk == K_INT || vk == K_NUM) {
    r.has_value = number_value(s, sp[S_PROP], &r.value);
    if (!r.has_value) {
      r.outcome = FALLBACK;
      return r;
    }
  } else if (vk != K_ABSENT) {
    r.outcome = FALLBACK;   // a string, bool, null or container: float() semantics stay on the host
    return r;
  }
  const Span& ei = sp[S_EID];
  if (ei.kind == K_STR) {
    r.eid_len = decode_string(s, ei.b, ei.e, scratch);
  } else {
    r.eid_len = ei.e - ei.b;
    for (int k = 0; k < r.eid_len; ++k) scratch[k] = s[ei.b + k];
  }
  const Span& ti = sp[S_TID];
  if (tk == K_STR) {
    r.tid_len = decode_string(s, ti.b, ti.e, scratch + r.eid_len);
    r.has_target = 1;
  } else if (tk == K_INT) {
    r.tid_len = ti.e - ti.b;
    for (int k = 0; k < r.tid_len; ++k) scratch[r.eid_len + k] = s[ti.b + k];
    r.has_target = 1;
  }
  if constexpr (KEYS) {
    for (int q = 0; q < kl->n; ++q) {
      const Span& v = ksp[q];
      if (v.kind == K_ABSENT) continue;
      kv->present |= 1u << q;
      if ((v.kind == K_INT || v.kind == K_NUM) && number_value(s, v, &kv->num[q])) {
        kv->number |= 1u << q;
        if (v.kind == K_NUM) continue;
      } else {
        kv->num[q] = 0.0;
      }
      kv->tok_b[q] = v.b;
      kv->tok_e[q] = v.e;
    }
  }
  if constexpr (ALL) {
    pi->utc_off = utc_off;
    if (pk == K_OBJ && pkeys > 0) pi->n_keys = pkeys, pi->b = sp[S_PROPS].b, pi->e = pend;
  }
  r.outcome = MATCHED;
  return r;
}

PIO_EV_HD Result parse_line(const uint8_t* s, int n, const Filter& f, uint8_t* scratch) {
  return parse_line_t<false>(s, n, f, scratch, nullptr, nullptr);
}

// *kv is cleared first, so that a line that is not MATCHED reports no keys
PIO_EV_HD Result parse_line_keys(const uint8_t* s, int n, const Filter& f, const KeyList& kl, uint8_t* scratch,
                                 KeyValues* kv) {
  kv->present = kv->number = 0;
  for (int q = 0; q < MAX_KEYS; ++q) kv->num[q] = 0.0, kv->tok_b[q] = kv->tok_e[q] = 0;
  return parse_line_t<true>(s, n, f, scratch, &kl, kv);
}

// *pi is cleared first, so that a line that is not MATCHED reports no keys
PIO_EV_HD Result parse_line_props(const uint8_t* s, int n, const Filter& f, uint8_t* scratch, PropsInfo* pi) {
  pi->n_keys = pi->b = pi->e = pi->utc_off = 0;
  return parse_line_t<false, true>(s, n, f, scratch, nullptr, nullptr, pi);
}

// ---- the second walk: one record per key of a MATCHED line's `properties` object, in object order -------------------
struct PropRec {
  int kb, ke;       // the key's string token, quotes included
  int vb, ve;       // the value's raw JSON token
};

// the end of the validated JSON value at s[i]
PIO_EV_HD int skip_value(const uint8_t* s, int n, int i) {
  uint8_t esc;
  const uint8_t c = s[i];
  if (c == '"') return scan_string(s, n, i, &esc);
  if (c != '{' && c != '[') {   // number, true, false, null
    while (i < n && s[i] != ',' && s[i] != '}' && s[i] != ']' && !is_ws(s[i])) ++i;
    return i;
  }
  int d = 0;
  for (;;) {
    const uint8_t x = s[i];
    if (x == '"') {
      i = scan_string(s, n, i, &esc);
      continue;
    }
    if (x == '{' || x == '[') ++d;
    else if ((x == '}' || x == ']') && --d == 0) return i + 1;
    ++i;
  }
}

// *at: just after the object's "{" or after the previous value (PropsInfo::b + 1 to start); the object ends before e.
// Fills *r and advances *at; false at the closing "}".
PIO_EV_HD bool next_prop(const uint8_t* s, int e, int* at, PropRec* r) {
  int i = *at;
  while (is_ws(s[i]) || s[i] == ',') ++i;
  if (s[i] == '}') return false;
  uint8_t esc;
  r->kb = i;
  i = scan_string(s, e, i, &esc);
  r->ke = i;
  while (is_ws(s[i]) || s[i] == ':') ++i;
  r->vb = i;
  i = skip_value(s, e, i);
  r->ve = i;
  *at = i;
  return true;
}

// the number of bytes decode_string writes for the validated string token [b, e)
PIO_EV_HD int decoded_len(const uint8_t* s, int b, int e) {
  int i = b + 1, o = 0;
  const int end = e - 1;
  while (i < end) {
    if (s[i] != '\\') {
      ++o, ++i;
      continue;
    }
    if (s[i + 1] != 'u') {
      ++o, i += 2;
      continue;
    }
    const int u = hex4(s, e, i + 2);
    i += 6;
    if (u >= 0xD800 && u <= 0xDBFF) {
      o += 4, i += 6;
      continue;
    }
    o += u < 0x80 ? 1 : u < 0x800 ? 2 : 3;
  }
  return o;
}

}  // namespace ev
}  // namespace pio
