// ggr_json_in.cuh - JSON token readers of the request-side kernels.
//
// Token rules follow protobuf-go's own JSON tokenizer, which is what protojson.Unmarshal sees
// at /root/reference/pkg/grpc/reflection.go:355 [upstream internal/encoding/json/
// {decode,decode_number,decode_string}.go]: strict RFC 8259 grammar, strings must be valid UTF-8
// without raw control characters, \uXXXX escapes with mandatory surrogate pairing, literals and
// numbers must be followed by a delimiter.
#pragma once
#include "ggr_prim.cuh"

GGR_DEV void skip_ws(Rd& r) {
  while (!r.eof() && ggr_is_ws(r.peek())) r.skip(1);
}

GGR_DEV int hex_val(u32 c) {
  if (c - '0' < 10u) return (int)(c - '0');
  u32 l = c | 0x20u;
  if (l - 'a' < 6u) return (int)(l - 'a' + 10);
  return -1;
}

// SWAR: nonzero iff any of the 4 bytes is '"', '\\', < 0x20 or >= 0x80.  The lowest flagged byte
// is exact (borrows only travel upwards).
GGR_DEV u32 json_special_mask(u32 x) {
  const u32 ones = 0x01010101u, hi = 0x80808080u;
  u32 q = (x ^ 0x22222222u) - ones;
  u32 b = (x ^ 0x5C5C5C5Cu) - ones;
  u32 c = x - 0x20202020u;
  return (q | b | c | x) & hi;
}

// Validates one multi-byte UTF-8 sequence at the reader (first byte >= 0x80), Go utf8 rules.
// Returns its length (2..4) or 0 when invalid.  Does not consume.
GGR_DEV int utf8_seq_len(const Rd& r) {
  u32 w = r.peek4();
  u32 left = r.left();
  u32 c0 = w & 0xFF, c1 = (w >> 8) & 0xFF, c2 = (w >> 16) & 0xFF, c3 = w >> 24;
  if (c0 < 0xC2 || c0 > 0xF4) return 0;
  if (c0 < 0xE0) {
    if (left < 2 || (c1 & 0xC0) != 0x80) return 0;
    return 2;
  }
  if (c0 < 0xF0) {
    u32 lo = c0 == 0xE0 ? 0xA0u : 0x80u, hi = c0 == 0xED ? 0x9Fu : 0xBFu;
    if (left < 3 || c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80) return 0;
    return 3;
  }
  u32 lo = c0 == 0xF0 ? 0x90u : 0x80u, hi = c0 == 0xF4 ? 0x8Fu : 0xBFu;
  if (left < 4 || c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80 || (c3 & 0xC0) != 0x80) return 0;
  return 4;
}

// Reads the 4 hex digits of a \uXXXX escape; reader positioned at the backslash.
// Returns the code unit or -1.  Consumes the 6 bytes on success.
GGR_DEV int read_u_escape(Rd& r) {
  if (r.left() < 6) return -1;
  r.skip(2);  // \u
  u32 w = r.peek4();
  int a = hex_val(w & 0xFF), b = hex_val((w >> 8) & 0xFF), c = hex_val((w >> 16) & 0xFF), d = hex_val(w >> 24);
  if ((a | b | c | d) < 0) return -1;
  r.skip(4);
  return (a << 12) | (b << 8) | (c << 4) | d;
}

// Decodes one escape sequence at the reader (positioned at '\\').  On success consumes it and
// returns the number of UTF-8 bytes (1..4) placed in *out (lowest byte first); 0 on error.
GGR_DEV int read_escape(Rd& r, u32* out) {
  if (r.left() < 2) return 0;
  u32 e = (r.peek4() >> 8) & 0xFF;
  u32 v;
  switch (e) {
    case '"': v = '"'; break;
    case '\\': v = '\\'; break;
    case '/': v = '/'; break;
    case 'b': v = 8; break;
    case 'f': v = 12; break;
    case 'n': v = 10; break;
    case 'r': v = 13; break;
    case 't': v = 9; break;
    case 'u': {
      int cu = read_u_escape(r);
      if (cu < 0) return 0;
      u32 cp = (u32)cu;
      if (cp >= 0xD800 && cp < 0xE000) {
        // must be a high surrogate followed by \uDC00..\uDFFF
        if (cp >= 0xDC00) return 0;
        if (r.left() < 6 || (r.peek4() & 0xFFFF) != (u32)('\\' | ('u' << 8))) return 0;
        int lo = read_u_escape(r);
        if (lo < 0xDC00 || lo >= 0xE000) return 0;
        cp = 0x10000u + ((cp - 0xD800u) << 10) + ((u32)lo - 0xDC00u);
      }
      if (cp < 0x80) { *out = cp; return 1; }
      if (cp < 0x800) { *out = (0xC0 | (cp >> 6)) | ((0x80 | (cp & 0x3F)) << 8); return 2; }
      if (cp < 0x10000) {
        *out = (0xE0 | (cp >> 12)) | ((0x80 | ((cp >> 6) & 0x3F)) << 8) | ((0x80 | (cp & 0x3F)) << 16);
        return 3;
      }
      *out = (0xF0 | (cp >> 18)) | ((0x80 | ((cp >> 12) & 0x3F)) << 8) | ((0x80 | ((cp >> 6) & 0x3F)) << 16) |
             ((0x80 | (cp & 0x3F)) << 24);
      return 4;
    }
    default: return 0;
  }
  r.skip(2);
  *out = v;
  return 1;
}

struct StrInfo {
  u32 dec_len;   // decoded byte length
  u32 flags;     // SF_*
};
#define SF_ESCAPES 1u   /* contains backslash escapes */
#define SF_URLSAFE 2u   /* contains '-' or '_' (base64 alphabet choice) */
#define SF_NEWLINE 4u   /* decoded text contains \r or \n (only possible through escapes) */

// Scans a JSON string token; reader at the opening quote, left after the closing quote.
// Returns GST_OK / GST_SYNTAX / GST_INVALID_UTF8.
template <bool WANT_B64_FLAGS>
GGR_DEV int scan_string(Rd& r, StrInfo* si) {
  r.skip(1);
  u32 n = 0, flags = 0;
  for (;;) {
    // fast path: 4 plain ASCII bytes at a time
    while (r.left() >= 4) {
      u32 w = r.peek4();
      if (json_special_mask(w)) break;
      if (WANT_B64_FLAGS) {
        // '-' 0x2D or '_' 0x5F present?
        u32 a = (w ^ 0x2D2D2D2Du) - 0x01010101u, b = (w ^ 0x5F5F5F5Fu) - 0x01010101u;
        if ((a | b) & ~w & 0x80808080u) flags |= SF_URLSAFE;
      }
      r.skip(4);
      n += 4;
    }
    if (r.eof()) return GST_SYNTAX;
    u32 c = r.peek();
    if (c == '"') {
      r.skip(1);
      si->dec_len = n;
      si->flags = flags;
      return GST_OK;
    }
    if (c == '\\') {
      u32 v;
      int k = read_escape(r, &v);
      if (k == 0) return GST_SYNTAX;
      flags |= SF_ESCAPES;
      if (WANT_B64_FLAGS && k == 1) {
        if (v == '-' || v == '_') flags |= SF_URLSAFE;
        if (v == '\r' || v == '\n') flags |= SF_NEWLINE;
      }
      n += (u32)k;
      continue;
    }
    if (c < 0x20) return GST_SYNTAX;
    if (c < 0x80) {
      if (WANT_B64_FLAGS && (c == '-' || c == '_')) flags |= SF_URLSAFE;
      r.skip(1);
      n += 1;
      continue;
    }
    int k = utf8_seq_len(r);
    if (k == 0) return GST_INVALID_UTF8;
    r.skip(k);
    n += (u32)k;
  }
}

// ------------------------------------------------------------------------------------------
// StrIter: decoded-byte iterator over a string token that scan_string already validated.
// ------------------------------------------------------------------------------------------
struct StrIter {
  Rd r;
  u32 buf;
  int nbuf;
  bool done;
  GGR_DEV void fetch() {
    if (r.eof()) { done = true; return; }
    u32 c = r.peek();
    if (c == '"') { done = true; return; }
    if (c == '\\') {
      nbuf = read_escape(r, &buf);
      if (nbuf == 0) done = true;
      return;
    }
    buf = c;
    nbuf = 1;
    r.skip(1);
  }
  GGR_DEV void init(const u8* base, u32 quote_pos, u32 end) {
    r.init(base, quote_pos + 1, end);
    done = false;
    nbuf = 0;
    buf = 0;
    fetch();
  }
  GGR_DEV bool eof() const { return done; }
  GGR_DEV u32 peek() const { return buf & 0xFF; }
  GGR_DEV u32 get() const { return done ? 0u : (buf & 0xFF); }
  GGR_DEV void adv() {
    buf >>= 8;
    if (--nbuf <= 0) fetch();
  }
};
// adapter so the number parser can run directly on the JSON stream
struct RawIter {
  Rd* r;
  GGR_DEV bool eof() const { return r->eof(); }
  GGR_DEV u32 get() const { return r->get(); }
  GGR_DEV void adv() { r->skip(1); }
};
// an independent iterator at the same position, for a second pass over a token (a RawIter shares its
// reader, so its copy reads from `store`)
GGR_DEV StrIter it_fork(const StrIter& it, Rd*) { return it; }
GGR_DEV RawIter it_fork(const RawIter& it, Rd* store) {
  *store = *it.r;
  RawIter c = {store};
  return c;
}

// ------------------------------------------------------------------------------------------
// Number tokens.  m * 10^k is the exact value when the token is an integer (see DESIGN.md):
//   m   = all digits (integer part then fraction) with trailing zeros dropped, saturating
//   k   = (dropped trailing zeros) + exp - (fraction digits)
// ------------------------------------------------------------------------------------------
struct NumTok {
  bool neg;
  bool ovf;       // m overflowed 64 bits
  bool is_plain;  // only digits (no fraction / exponent)
  u64 m;
  i32 k;
  u32 sig;        // significant digits accumulated into m
  u32 int_digits; // digits of the integer part ("0" counts as none, like upstream's intp)
  i32 exp;        // exponent as written (clamped)
};

GGR_DEV bool mul10_add(u64& m, u32 d) {  // false on overflow
  if (m > 1844674407370955161ull || (m == 1844674407370955161ull && d > 5)) return false;
  m = m * 10 + d;
  return true;
}

// Parses a number per protobuf-go parseNumber and checks the trailing delimiter.
// Returns false when the text is not a valid number token.
template <class It>
GGR_DEV bool parse_number(It& it, NumTok* t) {
  t->neg = false;
  t->ovf = false;
  t->is_plain = true;
  t->m = 0;
  t->sig = 0;
  t->int_digits = 0;
  t->exp = 0;
  u32 pend = 0;       // zeros seen since the last nonzero digit
  u32 frac_total = 0;
  i64 exp = 0;
  u32 c = it.get();
  if (c == '-') {
    t->neg = true;
    it.adv();
    c = it.get();
  }
  auto digit = [&](u32 d) {
    if (d == 0) {
      if (t->m != 0 || t->ovf) pend++;
      return;
    }
    for (; pend > 0; pend--) {
      if (!t->ovf && !mul10_add(t->m, 0)) t->ovf = true;
    }
    if (!t->ovf && !mul10_add(t->m, d)) t->ovf = true;
    t->sig++;
  };
  if (c == '0') {
    it.adv();
  } else if (c - '1' < 9u) {
    do {
      digit(c - '0');
      t->int_digits++;
      it.adv();
      c = it.get();
    } while (c - '0' < 10u);
  } else {
    return false;
  }
  c = it.get();
  if (c == '.') {
    it.adv();
    c = it.get();
    if (!(c - '0' < 10u)) return false;  // '.' must be followed by a digit ('.' is not a delimiter)
    t->is_plain = false;
    do {
      digit(c - '0');
      frac_total++;
      it.adv();
      c = it.get();
    } while (c - '0' < 10u);
  }
  if (c == 'e' || c == 'E') {
    it.adv();
    c = it.get();
    bool eneg = false;
    if (c == '+' || c == '-') {
      eneg = c == '-';
      it.adv();
      c = it.get();
    }
    if (!(c - '0' < 10u)) return false;
    t->is_plain = false;
    do {
      if (exp <= 100000000) exp = exp * 10 + (i64)(c - '0');
      it.adv();
      c = it.get();
    } while (c - '0' < 10u);
    // beyond 10^8 the exponent stays clamped: an integer kind with a nonzero digit fails on it (num_to_int),
    // strconv.ParseFloat goes on - 0.0e2964595747023549 is 0, 1e-99999999999 underflows to 0, 1e99999999999 is out of range
    if (eneg) exp = -exp;
  }
  if (!it.eof() && ggr_not_delim(it.get())) return false;
  // when m == 0 (all digits zero) pend was never counted; k is irrelevant then
  i64 k = (i64)pend + exp - (i64)frac_total;
  if (k > 1000000) k = 1000000;
  if (k < -1000000) k = -1000000;
  t->k = (i32)k;
  t->exp = (i32)exp;
  return true;
}

// Integer value of a number token for a signed/unsigned kind of `bits` width.
// Returns false when the token is not an integer in range [upstream normalizeToIntString +
// strconv.ParseInt/ParseUint].
GGR_DEV bool num_to_int(const NumTok& t, bool is_signed, int bits, u64* out) {
  if (t.m == 0 && !t.ovf) {  // no nonzero digit: 0 whatever the exponent (normalizeToIntString returns before reading it)
    *out = 0;
    return true;
  }
  // beyond 10^8 the exponent is clamped: strconv.ParseInt(exp, 10, 32) fails, or a nonzero value has more than 20 digits
  // or shifts nonzero digits out
  if (t.exp > 100000000 || t.exp < -100000000) return false;
  if (t.ovf || t.k < 0 || t.k > 19) return false;
  // upstream's digit-count guard: integer-part digits + exponent may not exceed 20
  if (t.exp >= 0 && (i64)t.int_digits + t.exp > 20) return false;
  u64 v = t.m;
  for (int i = 0; i < t.k; i++)
    if (!mul10_add(v, 0)) return false;
  if (is_signed) {
    u64 lim = 1ull << (bits - 1);
    if (t.neg) {
      if (v > lim) return false;
      *out = (u64)(0 - v);
    } else {
      if (v >= lim) return false;
      *out = v;
    }
  } else {
    if (t.neg) return false;
    if (bits < 64 && v >= (1ull << bits)) return false;
    *out = v;
  }
  return true;
}

// strconv.ParseInt / ParseUint(name, 10, bits) on a map key: optional sign (signed only),
// decimal digits only, leading zeros allowed.
GGR_DEV bool parse_key_int(StrIter& it, bool is_signed, int bits, u64* out) {
  bool neg = false;
  u32 c = it.get();
  if (is_signed && (c == '+' || c == '-')) {
    neg = c == '-';
    it.adv();
  }
  if (it.eof()) return false;
  u64 v = 0;
  while (!it.eof()) {
    c = it.peek();
    if (!(c - '0' < 10u)) return false;
    if (!mul10_add(v, c - '0')) return false;
    it.adv();
  }
  if (is_signed) {
    u64 lim = 1ull << (bits - 1);
    if (neg) {
      if (v > lim) return false;
      *out = (u64)(0 - v);
    } else {
      if (v >= lim) return false;
      *out = v;
    }
  } else {
    if (bits < 64 && v >= (1ull << bits)) return false;
    *out = v;
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// Key hashing.  Keys are hashed a little-endian 32-bit word at a time (the last word zero padded)
// so that the common key - plain ASCII, no escapes - is hashed straight from the reader's 4-byte
// window while it is being validated; the table entry carries the first 16 bytes of the name
// inline, so a hit needs no second pass over the key and no pool access.
// (ggr_schema.cc computes the same function on the host: ggr::key_hash.)
// ------------------------------------------------------------------------------------------
struct KeyInfo {
  u32 len;     // decoded length
  u32 hash;
  u32 w[4];    // first 16 decoded bytes, zero padded
};
GGR_DEV u32 khash_mix(u32 h, u32 word) {
  h = (h ^ word) * 0x9E3779B1u;
  return h ^ (h >> 15);
}
GGR_DEV u32 khash_finish(u32 h, u32 len) {
  h ^= len;
  h *= 0x85EBCA6Bu;
  return h ^ (h >> 13);
}
#define GGR_KHASH_SEED 0x811C9DC5u

// Scans a key token (reader at the opening quote; left after the closing quote), validating it
// exactly like scan_string and filling KeyInfo on the way.  Returns GST_OK / GST_SYNTAX /
// GST_INVALID_UTF8.
GGR_DEV int scan_key(Rd& r, KeyInfo* k) {
  r.skip(1);
  u32 n = 0, h = GGR_KHASH_SEED;
  u32 w0 = 0, w1 = 0, w2 = 0, w3 = 0;
  u32 part = 0;  // bytes of the word under construction (n & 3 of them)
  for (;;) {
    // whole plain words
    while ((n & 3u) == 0 && r.left() >= 4) {
      u32 x = r.peek4();
      if (json_special_mask(x)) break;
      h = khash_mix(h, x);
      u32 i = n >> 2;
      if (i == 0) w0 = x;
      else if (i == 1) w1 = x;
      else if (i == 2) w2 = x;
      else if (i == 3) w3 = x;
      r.skip(4);
      n += 4;
    }
    if (r.eof()) return GST_SYNTAX;
    u32 c = r.peek();
    u32 bytes, nb;
    if (c == '"') {
      r.skip(1);
      break;
    }
    if (c == '\\') {
      nb = (u32)read_escape(r, &bytes);
      if (nb == 0) return GST_SYNTAX;
    } else if (c < 0x20) {
      return GST_SYNTAX;
    } else if (c < 0x80) {
      bytes = c;
      nb = 1;
      r.skip(1);
    } else {
      int q = utf8_seq_len(r);
      if (q == 0) return GST_INVALID_UTF8;
      bytes = r.peek4() & (0xFFFFFFFFu >> (8 * (4 - q)));
      nb = (u32)q;
      r.skip(q);
    }
    // feed nb decoded bytes
    for (u32 j = 0; j < nb; j++) {
      part |= ((bytes >> (8 * j)) & 0xFFu) << (8 * (n & 3u));
      n++;
      if ((n & 3u) == 0) {
        h = khash_mix(h, part);
        u32 i = (n >> 2) - 1;
        if (i == 0) w0 = part;
        else if (i == 1) w1 = part;
        else if (i == 2) w2 = part;
        else if (i == 3) w3 = part;
        part = 0;
      }
    }
  }
  if (n & 3u) {
    h = khash_mix(h, part);
    u32 i = n >> 2;
    if (i == 0) w0 = part;
    else if (i == 1) w1 = part;
    else if (i == 2) w2 = part;
    else if (i == 3) w3 = part;
  }
  k->len = n;
  k->hash = khash_finish(h, n);
  k->w[0] = w0;
  k->w[1] = w1;
  k->w[2] = w2;
  k->w[3] = w3;
  return GST_OK;
}

// Compares the decoded bytes of the string token at `quote_pos` with pool[off, off+len).
GGR_DEV bool str_equals_pool(const u8* base, u32 quote_pos, u32 end, const u8* pool, u32 off, u32 len) {
  StrIter it;
  it.init(base, quote_pos, end);
  Rd p;
  p.init(pool, off, off + len);
  while (!p.eof()) {
    if (it.eof() || it.peek() != p.peek()) return false;
    it.adv();
    p.skip(1);
  }
  return it.eof();
}

// Does the decoded string token equal the short literal `lit`?
GGR_DEV bool str_token_is(const u8* base, u32 quote_pos, u32 end, const char* lit, int n) {
  StrIter it;
  it.init(base, quote_pos, end);
  for (int i = 0; i < n; i++) {
    if (it.eof() || it.peek() != (u32)(u8)lit[i]) return false;
    it.adv();
  }
  return it.eof();
}

// Looks a scanned key up in an open-addressing GgrHashEnt table (32-byte entries: hash, pool
// offset, length, value, first 16 name bytes).  Names longer than 16 bytes compare their tail
// against the pool.
GGR_DEV bool hash_lookup(const Tables& t, u32 first, u32 mask, const KeyInfo& k, const u8* base, u32 quote_pos, u32 end,
                         i32* value) {
  u32 slot = k.hash & mask;
  for (u32 probes = 0; probes <= mask; probes++) {
    const u8* ep = t.hash + (size_t)(first + slot) * 32;
    U4 e = ggr_ld16(ep);
    if (e.z == 0xFFFFFFFFu) return false;
    if (e.x == k.hash && e.z == k.len) {
      U4 nm = ggr_ld16(ep + 16);
      if (nm.x == k.w[0] && nm.y == k.w[1] && nm.z == k.w[2] && nm.w == k.w[3]) {
        if (k.len <= 16 || str_equals_pool(base, quote_pos, end, t.pool, e.y, k.len)) {
          *value = (i32)e.w;
          return true;
        }
      }
    }
    slot = (slot + 1) & mask;
  }
  return false;
}

// true/false/null literal with delimiter check; returns 1 on match (consumed), 0 otherwise
GGR_DEV int match_literal(Rd& r, u32 lit4, int len, u32 fifth) {
  if (r.left() < (u32)len) return 0;
  if (r.peek4() != lit4) return 0;
  if (len == 5) {
    Rd t = r;
    t.skip(4);
    if (t.peek() != fifth) return 0;
    t.skip(1);
    if (!t.eof() && ggr_not_delim(t.peek())) return 0;
    r = t;
    return 1;
  }
  Rd t = r;
  t.skip(4);
  if (!t.eof() && ggr_not_delim(t.peek())) return 0;
  r = t;
  return 1;
}
#define LIT4(a, b, c, d) ((u32)(a) | ((u32)(b) << 8) | ((u32)(c) << 16) | ((u32)(d) << 24))
