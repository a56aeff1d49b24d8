// orc_protojson.h - restatement of protobuf-go v1.36.6 encoding/protojson as the reference calls
// it with default options (TEST INFRASTRUCTURE, see ggr_oracle.h):
//   protojson.Unmarshal(inputJSON, dynamicpb msg)  /root/reference/pkg/grpc/reflection.go:354-357
//   protojson.Marshal(outputMsg)                   /root/reference/pkg/grpc/reflection.go:381
// [upstream encoding/protojson/{decode,encode,well_known_types}.go,
//           internal/encoding/json/{decode,decode_number,decode_string,decode_token,encode}.go]
#pragma once
#include "orc_dyn.h"

namespace orc {

// ---------------- token reader (internal/encoding/json Decoder) ----------------
enum TokKind {
  K_INVALID = 0, K_EOF = 1, K_NULL = 2, K_BOOL = 4, K_NUMBER = 8, K_STRING = 16, K_NAME = 32,
  K_OBJ_OPEN = 64, K_OBJ_CLOSE = 128, K_ARR_OPEN = 256, K_ARR_CLOSE = 512, K_COMMA = 1024
};
static const int K_SCALAR = K_NULL | K_BOOL | K_NUMBER | K_STRING;

struct Tok {
  int kind = K_INVALID;
  bool b = false;
  std::string raw;  // raw text of the token
  Bytes str;        // parsed string (String / Name)
};

inline bool is_not_delim(uint8_t c) {
  return c == '-' || c == '+' || c == '.' || c == '_' || (c >= 'a' && c <= 'z') ||
         (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9');
}

// parseNumber of internal/encoding/json/decode_number.go; returns length or 0
inline size_t pj_parse_number(const uint8_t* in, size_t len) {
  size_t n = 0;
  if (len == 0) return 0;
  if (in[n] == '-') {
    n++;
    if (n == len) return 0;
  }
  if (in[n] == '0') n++;
  else if (in[n] >= '1' && in[n] <= '9') {
    n++;
    while (n < len && in[n] >= '0' && in[n] <= '9') n++;
  } else return 0;
  if (len - n >= 2 && in[n] == '.' && in[n + 1] >= '0' && in[n + 1] <= '9') {
    n += 2;
    while (n < len && in[n] >= '0' && in[n] <= '9') n++;
  }
  if (len - n >= 2 && (in[n] == 'e' || in[n] == 'E')) {
    size_t save = n;
    n++;
    if (in[n] == '+' || in[n] == '-') {
      n++;
      if (n == len) return 0;
    }
    size_t d0 = n;
    while (n < len && in[n] >= '0' && in[n] <= '9') n++;
    // NOTE: upstream accepts an exponent marker with no digits when a delimiter follows
    // (e.g. "1e "); the number-part parser then fails.  We reject here - same outcome
    // (the value is invalid), possibly a different error category.  See oracle/README.md.
    if (n == d0) {
      (void)save;
      return 0;
    }
  }
  if (n < len && is_not_delim(in[n])) return 0;
  return n;
}

struct PJTokens {
  const uint8_t* base;
  const uint8_t* p;
  const uint8_t* e;
  Err& err;
  std::vector<int> open;
  int last = 0;
  bool have_peek = false;
  Tok peeked;
  bool peek_ok = true;

  PJTokens(const uint8_t* b, size_t n, Err& er) : base(b), p(b), e(b + n), err(er) {}

  void ws() {
    while (p < e && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) p++;
  }
  bool syntax(const std::string& m) { return err.fail(ORC_SYNTAX, "syntax error: " + m); }

  bool parse_string(Tok& t) {
    const uint8_t* s0 = p;
    p++;  // opening quote
    while (true) {
      if (p >= e) return syntax("unexpected EOF");
      uint8_t c = *p;
      if (c == '"') {
        p++;
        t.raw.assign((const char*)s0, (size_t)(p - s0));
        return true;
      }
      if (c < 0x20) return syntax("invalid character in string");
      if (c == '\\') {
        if (e - p < 2) return syntax("unexpected EOF");
        uint8_t d = p[1];
        switch (d) {
          case '"': case '\\': case '/': t.str.push_back((char)d); p += 2; break;
          case 'b': t.str.push_back('\b'); p += 2; break;
          case 'f': t.str.push_back('\f'); p += 2; break;
          case 'n': t.str.push_back('\n'); p += 2; break;
          case 'r': t.str.push_back('\r'); p += 2; break;
          case 't': t.str.push_back('\t'); p += 2; break;
          case 'u': {
            auto hex4 = [&](const uint8_t* q, int& v) -> bool {
              v = 0;
              for (int i = 0; i < 4; i++) {
                int h = GoJsonHex(q[i]);
                if (h < 0) return false;
                v = v * 16 + h;
              }
              return true;
            };
            if (e - p < 6) return syntax("unexpected EOF");
            int v;
            if (!hex4(p + 2, v)) return syntax("invalid escape code in string");
            p += 6;
            uint32_t r = (uint32_t)v;
            if (r >= 0xD800 && r < 0xE000) {
              if (e - p < 6) return syntax("unexpected EOF");
              int v2;
              bool ok = hex4(p + 2, v2) && p[0] == '\\' && p[1] == 'u' && r < 0xDC00 && v2 >= 0xDC00 && v2 < 0xE000;
              if (!ok) return syntax("invalid escape code in string");
              r = 0x10000 + ((r - 0xD800) << 10) + ((uint32_t)v2 - 0xDC00);
              p += 6;
            }
            utf8_append(t.str, r);
            break;
          }
          default: return syntax("invalid escape code in string");
        }
        continue;
      }
      if (c < 0x80) {
        t.str.push_back((char)c);
        p++;
        continue;
      }
      int n;
      uint32_t r = utf8_decode(p, (size_t)(e - p), n);
      if (r == 0xFFFD && n == 1) return err.fail(ORC_INVALID_UTF8, "syntax error: invalid UTF-8 in string");
      t.str.append((const char*)p, (size_t)n);
      p += n;
    }
  }
  static int GoJsonHex(uint8_t c) {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
  }

  bool match_delim(const char* w) {
    size_t n = strlen(w);
    if ((size_t)(e - p) < n || memcmp(p, w, n) != 0) return false;
    if ((size_t)(e - p) > n && is_not_delim(p[n])) return false;
    return true;
  }

  bool parse_next(Tok& t) {
    ws();
    if (p >= e) {
      t.kind = K_EOF;
      return true;
    }
    switch (*p) {
      case 'n':
        if (match_delim("null")) { t.kind = K_NULL; t.raw = "null"; p += 4; return true; }
        break;
      case 't':
        if (match_delim("true")) { t.kind = K_BOOL; t.b = true; t.raw = "true"; p += 4; return true; }
        break;
      case 'f':
        if (match_delim("false")) { t.kind = K_BOOL; t.b = false; t.raw = "false"; p += 5; return true; }
        break;
      case '-': case '0': case '1': case '2': case '3': case '4': case '5': case '6': case '7': case '8': case '9': {
        size_t n = pj_parse_number(p, (size_t)(e - p));
        if (n) {
          t.kind = K_NUMBER;
          t.raw.assign((const char*)p, n);
          p += n;
          return true;
        }
        break;
      }
      case '"': t.kind = K_STRING; return parse_string(t);
      case '{': t.kind = K_OBJ_OPEN; t.raw = "{"; p++; return true;
      case '}': t.kind = K_OBJ_CLOSE; t.raw = "}"; p++; return true;
      case '[': t.kind = K_ARR_OPEN; t.raw = "["; p++; return true;
      case ']': t.kind = K_ARR_CLOSE; t.raw = "]"; p++; return true;
      case ',': t.kind = K_COMMA; t.raw = ","; p++; return true;
    }
    return syntax("invalid value");
  }

  bool is_value_next() {
    if (open.empty()) return last == 0;
    if (open.back() == K_OBJ_OPEN) return (last & K_NAME) != 0;
    return (last & (K_ARR_OPEN | K_COMMA)) != 0;
  }

  bool read_raw(Tok& t) {
    t = Tok();
    if (!parse_next(t)) return false;
    auto unexpected = [&]() { return syntax("unexpected token " + t.raw); };
    switch (t.kind) {
      case K_EOF:
        if (!open.empty() || (last & (K_SCALAR | K_OBJ_CLOSE | K_ARR_CLOSE)) == 0) return syntax("unexpected EOF");
        break;
      case K_NULL: case K_BOOL: case K_NUMBER:
        if (!is_value_next()) return unexpected();
        break;
      case K_STRING:
        if (is_value_next()) break;
        if ((last & (K_OBJ_OPEN | K_COMMA)) == 0) return unexpected();
        ws();
        if (p >= e) return syntax("unexpected EOF");
        if (*p != ':') return unexpected();
        p++;
        t.kind = K_NAME;
        break;
      case K_OBJ_OPEN: case K_ARR_OPEN:
        if (!is_value_next()) return unexpected();
        open.push_back(t.kind);
        break;
      case K_OBJ_CLOSE:
        if (open.empty() || (last & (K_NAME | K_COMMA)) != 0 || open.back() != K_OBJ_OPEN) return unexpected();
        open.pop_back();
        break;
      case K_ARR_CLOSE:
        if (open.empty() || last == K_COMMA || open.back() != K_ARR_OPEN) return unexpected();
        open.pop_back();
        break;
      case K_COMMA:
        if (open.empty() || (last & (K_SCALAR | K_OBJ_CLOSE | K_ARR_CLOSE)) == 0) return unexpected();
        break;
    }
    last = t.kind;
    if (t.kind == K_COMMA) return read_raw(t);
    return true;
  }
  bool read(Tok& t) {
    if (have_peek) {
      have_peek = false;
      t = peeked;
      return peek_ok;
    }
    return read_raw(t);
  }
  bool peek(Tok& t) {
    if (!have_peek) {
      peek_ok = read_raw(peeked);
      have_peek = true;
    }
    t = peeked;
    return peek_ok;
  }
};

// unicode.IsSpace, what strings.TrimSpace removes: the ASCII set and U+0085, U+00A0, U+1680, U+2000-200A, U+2028/9,
// U+202F, U+205F, U+3000
inline bool go_space_rune(uint32_t r) {
  return r == ' ' || (r >= 9 && r <= 13) || r == 0x85 || r == 0xA0 || r == 0x1680 || (r >= 0x2000 && r <= 0x200A) || r == 0x2028 ||
         r == 0x2029 || r == 0x202F || r == 0x205F || r == 0x3000;
}

// ---- number token -> integer (Token.Int / Token.Uint via getIntStr/normalizeToIntString) ----
struct NumParts {
  bool neg = false;
  std::string intp, frac;
  long exp = 0;
};
inline bool pj_number_parts(const std::string& raw, NumParts& np) {
  size_t i = 0, n = raw.size();
  if (n == 0) return false;
  if (raw[i] == '-') {
    np.neg = true;
    i++;
    if (i == n) return false;
  }
  if (raw[i] == '0') i++;  // leading 0 is not part of intp
  else if (raw[i] >= '1' && raw[i] <= '9') {
    size_t s = i;
    while (i < n && raw[i] >= '0' && raw[i] <= '9') i++;
    np.intp = raw.substr(s, i - s);
  } else return false;
  if (n - i >= 2 && raw[i] == '.' && raw[i + 1] >= '0' && raw[i + 1] <= '9') {
    size_t s = i + 1;
    i += 2;
    while (i < n && raw[i] >= '0' && raw[i] <= '9') i++;
    np.frac = raw.substr(s, i - s);
    while (!np.frac.empty() && np.frac.back() == '0') np.frac.pop_back();  // right-trim zeros
  }
  if (n - i >= 2 && (raw[i] == 'e' || raw[i] == 'E')) {
    i++;
    std::string ex = raw.substr(i);
    // the exponent's text: optional sign, digits (read as a 32-bit integer in pj_normalize_int)
    size_t k = 0;
    bool eneg = false;
    if (ex[k] == '+' || ex[k] == '-') {
      eneg = ex[k] == '-';
      k++;
    }
    if (k == ex.size()) return false;
    long v = 0;
    for (; k < ex.size(); k++) {
      if (ex[k] < '0' || ex[k] > '9') return false;
      if (v <= (1L << 32)) v = v * 10 + (ex[k] - '0');  // clamped: beyond int32 either way
    }
    np.exp = eneg ? -v : v;
    i = n;
  }
  return i == n;
}
inline bool pj_normalize_int(const NumParts& np, std::string& out) {
  size_t is = np.intp.size(), fs = np.frac.size();
  if (is == 0 && fs == 0) {  // no nonzero digit: 0 whatever the exponent (upstream returns before it reads the exponent)
    out = "0";
    return true;
  }
  if (np.exp > INT32_MAX || np.exp < INT32_MIN) return false;  // strconv.ParseInt(exp, 10, 32) fails
  std::string num;
  if (np.exp >= 0) {
    if ((long)fs > np.exp) return false;
    if ((long)is + np.exp > 20) return false;
    num = np.intp + np.frac;
    num.append((size_t)(np.exp - (long)fs), '0');
  } else {
    if (fs > 0) return false;
    long index = (long)is + np.exp;
    if (index < 0) return false;
    for (size_t i = (size_t)index; i < is; i++)
      if (np.intp[i] != '0') return false;
    num = np.intp.substr(0, (size_t)index);
  }
  out = np.neg ? "-" + num : num;
  return true;
}
// strconv.ParseInt(s, 10, bits) / ParseUint on the normalized string
inline bool parse_int_str(const std::string& s, int bits, int64_t& out) {
  size_t i = 0;
  bool neg = false;
  if (s.empty()) return false;
  if (s[0] == '-' || s[0] == '+') {
    neg = s[0] == '-';
    i++;
  }
  if (i == s.size()) return false;
  unsigned __int128 v = 0;
  for (; i < s.size(); i++) {
    if (s[i] < '0' || s[i] > '9') return false;
    v = v * 10 + (unsigned)(s[i] - '0');
    if (v > ((unsigned __int128)1 << 64)) return false;
  }
  unsigned __int128 lim = (unsigned __int128)1 << (bits - 1);
  if (neg) {
    if (v > lim) return false;
    out = (int64_t)(0 - (uint64_t)v);
  } else {
    if (v >= lim) return false;
    out = (int64_t)(uint64_t)v;
  }
  return true;
}
inline bool parse_uint_str(const std::string& s, int bits, uint64_t& out) {
  if (s.empty()) return false;
  unsigned __int128 v = 0;
  for (size_t i = 0; i < s.size(); i++) {
    if (s[i] < '0' || s[i] > '9') return false;  // ParseUint rejects signs
    v = v * 10 + (unsigned)(s[i] - '0');
    if (v > ((unsigned __int128)1 << 64)) return false;
  }
  if (bits < 64 && v >= ((unsigned __int128)1 << bits)) return false;
  if (bits == 64 && v > (unsigned __int128)UINT64_MAX) return false;
  out = (uint64_t)v;
  return true;
}
inline bool tok_int(const std::string& raw, int bits, int64_t& out) {
  NumParts np;
  std::string s;
  if (!pj_number_parts(raw, np) || !pj_normalize_int(np, s)) return false;
  return parse_int_str(s, bits, out);
}
inline bool tok_uint(const std::string& raw, int bits, uint64_t& out) {
  NumParts np;
  std::string s;
  if (!pj_number_parts(raw, np) || !pj_normalize_int(np, s)) return false;
  return parse_uint_str(s, bits, out);
}
// strconv.ParseFloat(raw, bits) with err != nil on overflow
inline bool tok_float(const std::string& raw, int bits, double& out) {
  if (bits == 32) {
    float f = strtof(raw.c_str(), nullptr);
    if (std::isinf(f)) return false;
    out = f;
    return true;
  }
  double d = strtod(raw.c_str(), nullptr);
  if (std::isinf(d)) return false;
  out = d;
  return true;
}

// ---------------- time helpers ----------------
inline int64_t days_from_civil(int64_t y, unsigned m, unsigned d) {
  y -= m <= 2;
  const int64_t era = (y >= 0 ? y : y - 399) / 400;
  const unsigned yoe = (unsigned)(y - era * 400);
  const unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + (int64_t)doe - 719468;
}
inline void civil_from_days(int64_t z, int64_t& y, unsigned& m, unsigned& d) {
  z += 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const unsigned doe = (unsigned)(z - era * 146097);
  const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  y = (int64_t)yoe + era * 400;
  const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const unsigned mp = (5 * doy + 2) / 153;
  d = doy - (153 * mp + 2) / 5 + 1;
  m = mp < 10 ? mp + 3 : mp - 9;
  y += m <= 2;
}
static const int64_t kMinTs = -62135596800LL, kMaxTs = 253402300799LL;

// time.Parse(time.RFC3339Nano, s) followed by protojson's own checks
// [upstream encoding/protojson/well_known_types.go unmarshalTimestamp; time/format.go parse]
// Accepts: YYYY-MM-DDTHH:MM:SS[(.|,)d+](Z|(+|-)HH:MM).  *long_frac: a '.' fraction of more than 9 digits, which
// protojson refuses only after its range check
inline bool parse_rfc3339(const Bytes& s, int64_t& secs, int32_t& nanos, bool* long_frac) {
  size_t i = 0, n = s.size();
  auto dig = [&](size_t k) { return k < n && s[k] >= '0' && s[k] <= '9'; };
  auto fixed2 = [&](int& v) {  // getnum(value, true)
    if (!dig(i) || !dig(i + 1)) return false;
    v = (s[i] - '0') * 10 + (s[i + 1] - '0');
    i += 2;
    return true;
  };
  auto lit = [&](char c) {
    if (i < n && s[i] == c) {
      i++;
      return true;
    }
    return false;
  };
  if (!(dig(0) && dig(1) && dig(2) && dig(3))) return false;
  int year = (s[0] - '0') * 1000 + (s[1] - '0') * 100 + (s[2] - '0') * 10 + (s[3] - '0');
  i = 4;
  int mon, day, hh, mi, ss;
  if (!lit('-') || !fixed2(mon) || !lit('-') || !fixed2(day) || !lit('T')) return false;
  // stdHour "15": getnum(value, false) - one or two digits (general parser, after the strict
  // RFC 3339 fast path declined)
  if (!dig(i)) return false;
  hh = s[i] - '0';
  i++;
  if (dig(i)) {
    hh = hh * 10 + (s[i] - '0');
    i++;
  }
  if (!lit(':') || !fixed2(mi) || !lit(':') || !fixed2(ss)) return false;
  int64_t ns = 0;
  size_t frac_digits = 0;
  bool frac_period = false;
  if (i + 1 < n && (s[i] == '.' || s[i] == ',') && dig(i + 1)) {
    frac_period = s[i] == '.';
    i++;
    int scale = 0;
    while (dig(i)) {
      if (scale < 9) {
        ns = ns * 10 + (s[i] - '0');
        scale++;
      }
      frac_digits++;
      i++;
    }
    while (scale < 9) {
      ns *= 10;
      scale++;
    }
  }
  if (i >= n) return false;
  int64_t off = 0;
  if (s[i] == 'Z') {
    i++;
  } else {
    if (n - i < 6) return false;
    if (s[i + 3] != ':') return false;
    char sign = s[i];
    i++;
    int oh, om;
    if (!fixed2(oh)) return false;
    i++;  // ':'
    if (!fixed2(om)) return false;
    if (oh > 24 || om > 60) return false;  // "time zone offset hour/minute" range checks (> not >=)
    off = (oh * 60 + om) * 60;
    if (sign == '-') off = -off;
    else if (sign != '+') return false;
  }
  if (i != n) return false;
  if (mon < 1 || mon > 12) return false;
  if (hh >= 24 || mi >= 60 || ss >= 60) return false;
  static const int dim[] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  int maxd = dim[mon - 1];
  bool leap = (year % 4 == 0 && year % 100 != 0) || year % 400 == 0;
  if (mon == 2 && leap) maxd = 29;
  if (day < 1 || day > maxd) return false;
  secs = days_from_civil(year, (unsigned)mon, (unsigned)day) * 86400 + hh * 3600 + mi * 60 + ss - off;
  nanos = (int32_t)ns;
  // protojson: a '.'-introduced subsecond field longer than ".999999999" is rejected
  // (LastIndexByte(s,'.') / LastIndexAny(s,"Z-+")); ','-introduced ones are truncated by time.Parse
  *long_frac = frac_period && frac_digits > 9;
  return true;
}
// [upstream internal/strs JSONSnakeCase / JSONCamelCase, protoreflect FullName.IsValid]
inline std::string fm_snake(const std::string& s) {
  std::string b;
  for (unsigned char c : s) {
    if (c >= 'A' && c <= 'Z') {
      b.push_back('_');
      c = (unsigned char)(c + ('a' - 'A'));
    }
    b.push_back((char)c);
  }
  return b;
}
inline std::string fm_camel(const std::string& s) {
  std::string b;
  bool was = false;
  for (unsigned char c : s) {
    if (c != '_') {
      if (was && c >= 'a' && c <= 'z') c = (unsigned char)(c - ('a' - 'A'));
      b.push_back((char)c);
    }
    was = c == '_';
  }
  return b;
}
inline bool fm_full_name_valid(const std::string& s) {
  auto letter = [](unsigned char c) { return c == '_' || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); };
  auto ident = [&](size_t i) -> long {
    if (i >= s.size() || !letter((unsigned char)s[i])) return -1;
    size_t k = i + 1;
    while (k < s.size() && (letter((unsigned char)s[k]) || (s[k] >= '0' && s[k] <= '9'))) k++;
    return (long)(k - i);
  };
  long n = ident(0);
  if (n < 0) return false;
  size_t i = (size_t)n;
  while (s.size() > i) {
    if (s[i] != '.') return false;
    i++;
    n = ident(i);
    if (n < 0) return false;
    i += (size_t)n;
  }
  return true;
}
inline std::string format_timestamp(int64_t secs, int64_t nanos) {
  // time.Unix(secs, nanos).UTC() normalizes nanos into [0,1e9)
  secs += nanos / 1000000000;
  nanos %= 1000000000;
  if (nanos < 0) {
    nanos += 1000000000;
    secs--;
  }
  int64_t days = secs / 86400, rem = secs % 86400;
  if (rem < 0) {
    rem += 86400;
    days--;
  }
  int64_t y;
  unsigned m, d;
  civil_from_days(days, y, m, d);
  char buf[64];
  snprintf(buf, sizeof buf, "%04lld-%02u-%02uT%02d:%02d:%02d.%09lld", (long long)y, m, d, (int)(rem / 3600),
           (int)(rem % 3600 / 60), (int)(rem % 60), (long long)nanos);
  std::string x(buf);
  auto trim = [&](const char* suf) {
    size_t n = strlen(suf);
    if (x.size() >= n && x.compare(x.size() - n, n, suf) == 0) x.resize(x.size() - n);
  };
  trim("000");
  trim("000");
  trim(".000");
  return x + "Z";
}

// ---------------- protojson.Unmarshal ----------------
struct PJUnmarshal {
  const Schema& S;
  PJTokens tk;
  Err& err;
  int depth = 10000;  // UnmarshalOptions.RecursionLimit default
  PJUnmarshal(const Schema& s, const uint8_t* b, size_t n, Err& e) : S(s), tk(b, n, e), err(e) {}

  bool unexpected(const Tok& t) { return err.fail(ORC_SYNTAX, "unexpected token " + t.raw); }
  bool invalid(const FieldDesc& f, const Tok& t) {
    return err.fail(ORC_INVALID_VALUE, "invalid value for field " + f.json_name + ": " + t.raw);
  }

  bool run(DynMsg& m) {
    if (!message(m)) return false;
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_EOF) return unexpected(t);
    return true;
  }

  // number-or-quoted-number helper [upstream unmarshalInt/unmarshalUint/unmarshalFloat]
  bool inner_number(const Tok& t, std::string& raw) {
    if (t.kind == K_NUMBER) {
      raw = t.raw;
      return true;
    }
    if (t.kind != K_STRING) return false;
    const Bytes& s = t.str;
    // strings.TrimSpace must be a no-op: neither the first nor the last rune is Unicode White_Space (a number token may
    // end in front of a multi-byte space, so "1\u00a0" is refused here, not by the number parser)
    if (!s.empty()) {
      int w;
      if (go_space_rune(utf8_decode((const uint8_t*)s.data(), s.size(), w))) return false;
      size_t k = s.size() - 1;
      while (k > 0 && ((uint8_t)s[k] & 0xC0) == 0x80 && s.size() - k < 4) k--;
      uint32_t r = utf8_decode((const uint8_t*)s.data() + k, s.size() - k, w);
      if ((size_t)w == s.size() - k && go_space_rune(r)) return false;
    }
    // a fresh decoder reads ONE token from the string; it must be a Number
    Err e2;
    PJTokens sub((const uint8_t*)s.data(), s.size(), e2);
    Tok t2;
    if (!sub.read(t2) || t2.kind != K_NUMBER) return false;
    raw = t2.raw;
    return true;
  }

  bool scalar(const FieldDesc& f, int type, Val& out) {
    Tok t;
    if (!tk.read(t)) return false;
    std::string raw;
    switch (type) {
      case T_BOOL:
        if (t.kind != K_BOOL) return invalid(f, t);
        out.u = t.b;
        return true;
      case T_INT32: case T_SINT32: case T_SFIXED32: {
        int64_t v;
        if (!inner_number(t, raw) || !tok_int(raw, 32, v)) return invalid(f, t);
        out.u = (uint64_t)v;
        return true;
      }
      case T_INT64: case T_SINT64: case T_SFIXED64: {
        int64_t v;
        if (!inner_number(t, raw) || !tok_int(raw, 64, v)) return invalid(f, t);
        out.u = (uint64_t)v;
        return true;
      }
      case T_UINT32: case T_FIXED32: {
        uint64_t v;
        if (!inner_number(t, raw) || !tok_uint(raw, 32, v)) return invalid(f, t);
        out.u = v;
        return true;
      }
      case T_UINT64: case T_FIXED64: {
        uint64_t v;
        if (!inner_number(t, raw) || !tok_uint(raw, 64, v)) return invalid(f, t);
        out.u = v;
        return true;
      }
      case T_FLOAT: case T_DOUBLE: {
        int bits = type == T_FLOAT ? 32 : 64;
        double d;
        if (t.kind == K_STRING) {
          if (t.str == "NaN") d = std::nan("");
          else if (t.str == "Infinity") d = INFINITY;
          else if (t.str == "-Infinity") d = -INFINITY;
          else if (!inner_number(t, raw) || !tok_float(raw, bits, d)) return invalid(f, t);
        } else if (t.kind == K_NUMBER) {
          if (!tok_float(t.raw, bits, d)) return invalid(f, t);
        } else return invalid(f, t);
        if (bits == 32) {
          float fl = (float)d;
          if (std::isnan(d)) out.u = 0x7FC00000u;  // math.NaN() converted to float32
          else out.u = float_bits(fl);
        } else {
          if (std::isnan(d)) out.u = 0x7FF8000000000001ULL;  // math.NaN() bit pattern
          else out.u = double_bits(d);
        }
        return true;
      }
      case T_STRING:
        if (t.kind != K_STRING) return invalid(f, t);
        out.s = t.str;  // tokenizer already enforced valid UTF-8
        return true;
      case T_BYTES: {
        if (t.kind != K_STRING) return invalid(f, t);
        Bytes b;
        if (!b64_decode_go((const uint8_t*)t.str.data(), t.str.size(), b)) return invalid(f, t);
        out.s = b;
        return true;
      }
      case T_ENUM: {
        if (t.kind == K_STRING) {
          int32_t num;
          if (!S.enums[f.enm].number_of(t.str, num)) return invalid(f, t);
          out.u = (uint64_t)(int64_t)num;
          return true;
        }
        if (t.kind == K_NUMBER) {
          int64_t v;
          if (!tok_int(t.raw, 32, v)) return invalid(f, t);
          out.u = (uint64_t)v;
          return true;
        }
        return invalid(f, t);
      }
      default:
        return err.fail(ORC_UNSUPPORTED, "unsupported kind");
    }
  }

  bool timestamp(DynMsg& m) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_STRING) return unexpected(t);
    int64_t secs;
    int32_t nanos;
    bool long_frac;
    if (!parse_rfc3339(t.str, secs, nanos, &long_frac)) return err.fail(ORC_INVALID_VALUE, "invalid google.protobuf.Timestamp value " + t.raw);
    // [upstream unmarshalTimestamp] the seconds range first, then the length of the subsecond field
    if (secs < kMinTs || secs > kMaxTs) return err.fail(ORC_RANGE, "google.protobuf.Timestamp value out of range: " + t.raw);
    if (long_frac) return err.fail(ORC_INVALID_VALUE, "invalid google.protobuf.Timestamp value " + t.raw);
    Val a, b;
    a.u = (uint64_t)secs;
    b.u = (uint64_t)(int64_t)nanos;
    m.known[1].list = {a};
    m.known[2].list = {b};
    return true;
  }

  // [upstream well_known_types.go unmarshalDuration / parseDuration]
  static bool parse_duration(const Bytes& in, int64_t& secs, int32_t& nanos) {
    size_t size = in.size();
    if (size < 2 || in[size - 1] != 's') return false;
    size_t i = 0, n = size - 1;
    bool neg = false;
    if (in[0] == '-') { neg = true; i = 1; }
    else if (in[0] == '+') i = 1;
    if (i == n) return false;
    std::string intp;
    if (in[i] == '0') {
      i++;
    } else if (in[i] >= '1' && in[i] <= '9') {
      while (i < n && in[i] >= '0' && in[i] <= '9') intp.push_back(in[i++]);
    } else if (in[i] != '.') {
      return false;
    }
    bool has_frac = false;
    char frac[9];
    if (i < n) {
      if (in[i] != '.') return false;
      i++;
      int k = 0;
      while (i < n && k < 9 && in[i] >= '0' && in[i] <= '9') frac[k++] = in[i++];
      if (i < n) return false;
      for (; k < 9; k++) frac[k] = '0';
      has_frac = true;
    }
    secs = 0;
    if (!intp.empty()) {  // strconv.ParseInt(intp, 10, 64)
      if (intp.size() > 19) return false;
      unsigned long long v = 0;
      for (char c : intp) v = v * 10 + (unsigned)(c - '0');
      if (intp.size() == 19 && intp > "9223372036854775807") return false;
      secs = (int64_t)v;
    }
    int64_t ns = 0;
    if (has_frac)
      for (int k = 0; k < 9; k++) ns = ns * 10 + (frac[k] - '0');
    if (neg) {
      if (secs > 0) secs = -secs;
      if (ns > 0) ns = -ns;
    }
    nanos = (int32_t)ns;
    return true;
  }
  bool duration(DynMsg& m) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_STRING) return unexpected(t);
    int64_t secs;
    int32_t nanos;
    if (!parse_duration(t.str, secs, nanos)) return err.fail(ORC_INVALID_VALUE, "invalid google.protobuf.Duration value " + t.raw);
    // validate seconds; no need to validate nanos because parseDuration would have covered that already
    if (secs < -315576000000ll || secs > 315576000000ll)
      return err.fail(ORC_RANGE, "google.protobuf.Duration value out of range: " + t.raw);
    Val a, b;
    a.u = (uint64_t)secs;
    b.u = (uint64_t)(int64_t)nanos;
    m.known[1].list = {a};
    m.known[2].list = {b};
    return true;
  }
  // [upstream unmarshalWrapperType: the value field read as a singular field of its kind]
  bool wrapper(DynMsg& m) {
    const FieldDesc* vf = m.d->find_number(1);
    if (!vf) return err.fail(ORC_UNSUPPORTED, "wrapper without a value field");
    Val v;
    if (!scalar(*vf, vf->type, v)) return false;
    m.known[1].list = {v};
    return true;
  }
  // [upstream unmarshalFieldMask: TrimSpace, split at ',', every path camelCase -> snake_case]
  bool fieldmask(DynMsg& m) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_STRING) return unexpected(t);
    std::string str(t.str.begin(), t.str.end());
    // strings.TrimSpace: Unicode White_Space (ASCII set + U+0085, U+00A0, U+1680, U+2000-200A, U+2028/9, U+202F, U+205F, U+3000)
    auto space_at = [&](size_t i, size_t& w) -> bool {
      int ww;
      uint32_t r = utf8_decode((const uint8_t*)str.data() + i, str.size() - i, ww);
      w = (size_t)ww;
      return go_space_rune(r);
    };
    size_t b = 0, e = str.size(), w;
    while (b < e && space_at(b, w)) b += w;
    while (e > b) {  // last rune
      size_t k = e - 1;
      while (k > b && ((unsigned char)str[k] & 0xC0) == 0x80) k--;
      if (!space_at(k, w) || k + w != e) break;
      e = k;
    }
    str = str.substr(b, e - b);
    if (str.empty()) return true;
    FieldVal& fv = m.known[1];
    size_t p = 0;
    while (true) {
      size_t c = str.find(',', p);
      std::string s0 = str.substr(p, c == std::string::npos ? std::string::npos : c - p);
      std::string sn = fm_snake(s0);
      if (s0.find('_') != std::string::npos || !fm_full_name_valid(sn))
        return err.fail(ORC_INVALID_VALUE, "google.protobuf.FieldMask.paths contains invalid path: \"" + s0 + "\"");
      Val v;
      v.s = Bytes(sn.begin(), sn.end());
      fv.list.push_back(v);
      if (c == std::string::npos) break;
      p = c + 1;
    }
    return true;
  }
  // [upstream unmarshalEmpty: an object without members (DiscardUnknown is off on this path)]
  bool empty(DynMsg&) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_OBJ_OPEN) return unexpected(t);
    if (!tk.read(t)) return false;
    if (t.kind == K_OBJ_CLOSE) return true;
    if (t.kind == K_NAME) return err.fail(ORC_UNKNOWN_FIELD, "unknown field " + t.raw);
    return unexpected(t);
  }

  bool message(DynMsg& m) {
    if (--depth < 0) return err.fail(ORC_DEPTH, "exceeded max recursion depth");
    bool ok = message1(m);
    depth++;
    return ok;
  }
  bool message1(DynMsg& m) {
    if (m.d->wkt == WKT_TIMESTAMP) return timestamp(m);
    if (m.d->wkt == WKT_DURATION) return duration(m);
    if (m.d->wkt == WKT_WRAPPER) return wrapper(m);
    if (m.d->wkt == WKT_EMPTY) return empty(m);
    if (m.d->wkt == WKT_FIELDMASK) return fieldmask(m);
    if (m.d->wkt != WKT_NONE) return err.fail(ORC_UNSUPPORTED, "well-known type " + m.d->full_name + " not supported");
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_OBJ_OPEN) return unexpected(t);
    std::map<int32_t, bool> seen;
    std::map<int, bool> seen_oneof;
    while (true) {
      if (!tk.read(t)) return false;
      if (t.kind == K_OBJ_CLOSE) return true;
      if (t.kind != K_NAME) return unexpected(t);
      const FieldDesc* f = nullptr;
      if (!(t.str.size() >= 2 && t.str.front() == '[' && t.str.back() == ']')) f = m.d->find_json_key(t.str);
      if (!f) return err.fail(ORC_UNKNOWN_FIELD, "unknown field " + t.raw);
      if (seen.count(f->number)) return err.fail(ORC_DUPLICATE, "duplicate field " + t.raw);
      seen[f->number] = true;
      Tok pk;
      if (!tk.peek(pk)) return false;
      if (pk.kind == K_NULL) {  // not Value / NullValue: field skipped
        tk.read(pk);
        continue;
      }
      if (f->is_map) {
        if (!map(m, *f)) return false;
      } else if (f->repeated) {
        if (!list(m, *f)) return false;
      } else {
        if (f->oneof_index >= 0) {
          if (seen_oneof.count(f->oneof_index))
            return err.fail(ORC_ONEOF, "error parsing " + t.raw + ", oneof " + m.d->oneofs[f->oneof_index] + " is already set");
          seen_oneof[f->oneof_index] = true;
        }
        Val v;
        if (f->type == T_MESSAGE) {
          v.m = std::make_shared<DynMsg>();
          v.m->d = &S.msgs[f->msg];
          if (!message(*v.m)) return false;
        } else if (!scalar(*f, f->type, v)) return false;
        m.known[f->number].list = {v};
      }
    }
  }

  bool list(DynMsg& m, const FieldDesc& f) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_ARR_OPEN) return unexpected(t);
    FieldVal& fv = m.known[f.number];
    while (true) {
      if (!tk.peek(t)) return false;
      if (t.kind == K_ARR_CLOSE) {
        tk.read(t);
        return true;
      }
      Val v;
      if (f.type == T_MESSAGE) {
        v.m = std::make_shared<DynMsg>();
        v.m->d = &S.msgs[f.msg];
        if (!message(*v.m)) return false;
      } else if (!scalar(f, f.type, v)) return false;
      fv.list.push_back(v);
    }
  }

  bool map_key(const FieldDesc& kf, const Tok& t, Val& key) {
    const Bytes& name = t.str;
    auto bad = [&]() { return err.fail(ORC_INVALID_VALUE, "invalid value for map key: " + t.raw); };
    switch (kf.type) {
      case T_STRING: key.s = name; return true;
      case T_BOOL:
        if (name == "true") key.u = 1;
        else if (name == "false") key.u = 0;
        else return bad();
        return true;
      case T_INT32: case T_SINT32: case T_SFIXED32: {
        int64_t v;
        if (!parse_int_str(name, 32, v)) return bad();  // strconv.ParseInt on the name itself
        key.u = (uint64_t)v;
        return true;
      }
      case T_INT64: case T_SINT64: case T_SFIXED64: {
        int64_t v;
        if (!parse_int_str(name, 64, v)) return bad();
        key.u = (uint64_t)v;
        return true;
      }
      case T_UINT32: case T_FIXED32: {
        uint64_t v;
        if (!parse_uint_str(name, 32, v)) return bad();
        key.u = v;
        return true;
      }
      case T_UINT64: case T_FIXED64: {
        uint64_t v;
        if (!parse_uint_str(name, 64, v)) return bad();
        key.u = v;
        return true;
      }
      default: return bad();
    }
  }

  bool map(DynMsg& m, const FieldDesc& f) {
    Tok t;
    if (!tk.read(t)) return false;
    if (t.kind != K_OBJ_OPEN) return unexpected(t);
    const MsgDesc& ed = S.msgs[f.msg];
    const FieldDesc& kf = *ed.find_number(1);
    const FieldDesc& vf = *ed.find_number(2);
    FieldVal& fv = m.known[f.number];
    while (true) {
      if (!tk.read(t)) return false;
      if (t.kind == K_OBJ_CLOSE) return true;
      if (t.kind != K_NAME) return unexpected(t);
      Val key;
      if (!map_key(kf, t, key)) return false;
      for (auto& kv : fv.map) {
        bool same = kf.type == T_STRING ? kv.first.s == key.s : kv.first.u == key.u;
        if (same) return err.fail(ORC_DUPLICATE, "duplicate map key " + t.raw);
      }
      Val v;
      if (vf.type == T_MESSAGE) {
        v.m = std::make_shared<DynMsg>();
        v.m->d = &S.msgs[vf.msg];
        if (!message(*v.m)) return false;
      } else if (!scalar(vf, vf.type, v)) return false;
      fv.map.push_back({key, v});
    }
  }
};

// ---------------- protojson.Marshal ----------------
struct PJMarshal {
  const Schema& S;
  uint32_t flags;
  Err& err;
  Bytes out;
  int last = 0;  // encoder lastKind
  PJMarshal(const Schema& s, uint32_t f, Err& e) : S(s), flags(f), err(e) {}

  enum { E_NAME = 1, E_SCALAR = 2, E_OBJ_OPEN = 4, E_OBJ_CLOSE = 8, E_ARR_OPEN = 16, E_ARR_CLOSE = 32 };
  void prepare(int next) {
    if ((last & (E_SCALAR | E_OBJ_CLOSE | E_ARR_CLOSE)) && (next & (E_NAME | E_SCALAR | E_OBJ_OPEN | E_ARR_OPEN))) {
      out.push_back(',');
      if (flags & ORC_F_COMMA_SPACE) out.push_back(' ');
    }
    last = next;
  }
  // internal/encoding/json appendString (no HTML escaping; invalid UTF-8 is an error)
  bool append_string(const uint8_t* s, size_t n) {
    static const char hex[] = "0123456789abcdef";
    out.push_back('"');
    size_t i = 0;
    while (i < n) {
      uint8_t c = s[i];
      if (c < 0x80) {
        if (c >= 0x20 && c != '"' && c != '\\') {
          out.push_back((char)c);
          i++;
          continue;
        }
        out.push_back('\\');
        switch (c) {
          case '"': case '\\': out.push_back((char)c); break;
          case '\b': out.push_back('b'); break;
          case '\f': out.push_back('f'); break;
          case '\n': out.push_back('n'); break;
          case '\r': out.push_back('r'); break;
          case '\t': out.push_back('t'); break;
          default:
            out += "u00";
            out.push_back(hex[c >> 4]);
            out.push_back(hex[c & 15]);
        }
        i++;
        continue;
      }
      int w;
      uint32_t r = utf8_decode(s + i, n - i, w);
      if (r == 0xFFFD && w == 1) return false;
      out.append((const char*)s + i, (size_t)w);
      i += w;
    }
    out.push_back('"');
    return true;
  }
  bool write_name(const std::string& s) {
    prepare(E_NAME);
    if (!append_string((const uint8_t*)s.data(), s.size())) return err.fail(ORC_INVALID_UTF8, "invalid UTF-8 in name");
    out.push_back(':');
    return true;
  }
  void write_raw_scalar(const std::string& s) {
    prepare(E_SCALAR);
    out += s;
  }
  bool write_string(const Bytes& s, const FieldDesc* f) {
    prepare(E_SCALAR);
    if (!append_string((const uint8_t*)s.data(), s.size()))
      return err.fail(ORC_INVALID_UTF8, std::string("field ") + (f ? f->name : "") + " contains invalid UTF-8");
    return true;
  }

  bool singular(const FieldDesc& f, int type, const Val& v) {
    switch (type) {
      case T_BOOL: write_raw_scalar(v.u ? "true" : "false"); return true;
      case T_STRING: return write_string(v.s, &f);
      case T_INT32: case T_SINT32: case T_SFIXED32: write_raw_scalar(std::to_string((int64_t)(int32_t)v.u)); return true;
      case T_UINT32: case T_FIXED32: write_raw_scalar(std::to_string((uint32_t)v.u)); return true;
      case T_INT64: case T_SINT64: case T_SFIXED64: return write_string(std::to_string((int64_t)v.u), &f);
      case T_UINT64: case T_FIXED64: return write_string(std::to_string(v.u), &f);
      case T_FLOAT: case T_DOUBLE: {
        double d = type == T_FLOAT ? (double)bits_to_float((uint32_t)v.u) : bits_to_double(v.u);
        if (std::isnan(d)) write_raw_scalar("\"NaN\"");
        else if (std::isinf(d)) write_raw_scalar(d > 0 ? "\"Infinity\"" : "\"-Infinity\"");
        else write_raw_scalar(format_float_go(d, type == T_FLOAT ? 32 : 64));
        return true;
      }
      case T_BYTES: {
        Bytes b;
        b64_encode(b, (const uint8_t*)v.s.data(), v.s.size());
        return write_string(b, &f);
      }
      case T_ENUM: {
        const std::string* nm = S.enums[f.enm].name_of((int32_t)v.u);
        if (nm) return write_string(*nm, &f);
        write_raw_scalar(std::to_string((int64_t)(int32_t)v.u));
        return true;
      }
      case T_MESSAGE: return message(*v.m);
      default: return err.fail(ORC_UNSUPPORTED, "unsupported kind");
    }
  }

  bool timestamp(const DynMsg& m) {
    int64_t secs = 0, nanos = 0;
    auto a = m.known.find(1);
    auto b = m.known.find(2);
    if (a != m.known.end() && !a->second.list.empty()) secs = (int64_t)a->second.list[0].u;
    if (b != m.known.end() && !b->second.list.empty()) nanos = (int64_t)(int32_t)b->second.list[0].u;
    if (secs < kMinTs || secs > kMaxTs) return err.fail(ORC_RANGE, "google.protobuf.Timestamp: seconds out of range");
    if (nanos < 0 || nanos > 999999999) return err.fail(ORC_RANGE, "google.protobuf.Timestamp: nanos out of range");  // secondsInNanos = 999999999
    Bytes s = format_timestamp(secs, nanos);
    prepare(E_SCALAR);
    append_string((const uint8_t*)s.data(), s.size());
    return true;
  }

  // [upstream marshalDuration]
  bool duration(const DynMsg& m) {
    int64_t secs = 0, nanos = 0;
    auto a = m.known.find(1);
    auto b = m.known.find(2);
    if (a != m.known.end() && !a->second.list.empty()) secs = (int64_t)a->second.list[0].u;
    if (b != m.known.end() && !b->second.list.empty()) nanos = (int64_t)(int32_t)b->second.list[0].u;
    if (secs < -315576000000ll || secs > 315576000000ll) return err.fail(ORC_RANGE, "google.protobuf.Duration: seconds out of range");
    if (nanos < -999999999 || nanos > 999999999) return err.fail(ORC_RANGE, "google.protobuf.Duration: nanos out of range");
    if ((secs > 0 && nanos < 0) || (secs < 0 && nanos > 0))
      return err.fail(ORC_RANGE, "google.protobuf.Duration: signs of seconds and nanos do not match");
    std::string x;
    if (secs < 0 || nanos < 0) {
      x = "-";
      secs = -secs;
      nanos = -nanos;
    }
    char buf[48];
    snprintf(buf, sizeof buf, "%lld.%09lld", (long long)secs, (long long)nanos);
    x += buf;
    auto trim = [&](const char* suf) {
      size_t n = strlen(suf);
      if (x.size() >= n && x.compare(x.size() - n, n, suf) == 0) x.resize(x.size() - n);
    };
    trim("000");
    trim("000");
    trim(".000");
    x += "s";
    prepare(E_SCALAR);
    append_string((const uint8_t*)x.data(), x.size());
    return true;
  }
  // [upstream marshalWrapperType: the value field written as a singular value, its default when unset]
  bool wrapper(const DynMsg& m) {
    const FieldDesc* vf = m.d->find_number(1);
    if (!vf) return err.fail(ORC_UNSUPPORTED, "wrapper without a value field");
    Val v;
    auto a = m.known.find(1);
    if (a != m.known.end() && !a->second.list.empty()) v = a->second.list[0];
    return singular(*vf, vf->type, v);
  }

  // [upstream marshalFieldMask]
  bool fieldmask(const DynMsg& m) {
    std::string joined;
    auto a = m.known.find(1);
    if (a != m.known.end()) {
      bool first = true;
      for (const Val& v : a->second.list) {
        std::string s(v.s.begin(), v.s.end());
        if (!fm_full_name_valid(s)) return err.fail(ORC_INVALID_VALUE, "google.protobuf.FieldMask.paths contains invalid path: \"" + s + "\"");
        std::string cc = fm_camel(s);
        if (s != fm_snake(cc)) return err.fail(ORC_INVALID_VALUE, "google.protobuf.FieldMask.paths contains irreversible value \"" + s + "\"");
        if (!first) joined.push_back(',');
        first = false;
        joined += cc;
      }
    }
    prepare(E_SCALAR);
    append_string((const uint8_t*)joined.data(), joined.size());
    return true;
  }

  bool message(const DynMsg& m) {
    if (m.d->wkt == WKT_TIMESTAMP) return timestamp(m);
    if (m.d->wkt == WKT_FIELDMASK) return fieldmask(m);
    if (m.d->wkt == WKT_DURATION) return duration(m);
    if (m.d->wkt == WKT_WRAPPER) return wrapper(m);
    if (m.d->wkt == WKT_EMPTY) {  // [upstream marshalEmpty]
      prepare(E_OBJ_OPEN);
      out.push_back('{');
      prepare(E_OBJ_CLOSE);
      out.push_back('}');
      return true;
    }
    if (m.d->wkt != WKT_NONE) return err.fail(ORC_UNSUPPORTED, "well-known type " + m.d->full_name + " not supported");
    prepare(E_OBJ_OPEN);
    out.push_back('{');
    // order.IndexOrder: declaration index
    for (auto& f : m.d->fields) {
      auto it = m.known.find(f.number);
      if (it == m.known.end()) continue;
      const FieldVal& fv = it->second;
      if (f.is_map) {
        if (fv.map.empty()) continue;
        if (!write_name(f.json_name)) return false;
        const MsgDesc& ed = S.msgs[f.msg];
        const FieldDesc& kf = *ed.find_number(1);
        const FieldDesc& vf = *ed.find_number(2);
        std::vector<const std::pair<Val, Val>*> ents;
        for (auto& kv : fv.map) ents.push_back(&kv);
        std::stable_sort(ents.begin(), ents.end(), [&](const std::pair<Val, Val>* x, const std::pair<Val, Val>* y) {
          return WireMarshal::key_less(kf.type, x->first, y->first);
        });
        prepare(E_OBJ_OPEN);
        out.push_back('{');
        for (auto* kv : ents) {
          std::string ks;
          switch (kf.type) {
            case T_STRING: ks = kv->first.s; break;
            case T_BOOL: ks = kv->first.u ? "true" : "false"; break;
            case T_UINT32: case T_UINT64: case T_FIXED32: case T_FIXED64: ks = std::to_string(kv->first.u); break;
            default: ks = std::to_string((int64_t)kv->first.u); break;
          }
          if (!write_name(ks)) return false;
          if (!singular(vf, vf.type, kv->second)) return false;
        }
        prepare(E_OBJ_CLOSE);
        out.push_back('}');
      } else if (f.repeated) {
        if (fv.list.empty()) continue;
        if (!write_name(f.json_name)) return false;
        prepare(E_ARR_OPEN);
        out.push_back('[');
        for (auto& v : fv.list)
          if (!singular(f, f.type, v)) return false;
        prepare(E_ARR_CLOSE);
        out.push_back(']');
      } else {
        if (fv.list.empty() || !scalar_is_set(f, fv.list[0])) continue;
        if (!write_name(f.json_name)) return false;
        if (!singular(f, f.type, fv.list[0])) return false;
      }
    }
    prepare(E_OBJ_CLOSE);
    out.push_back('}');
    return true;
  }
};

}  // namespace orc
