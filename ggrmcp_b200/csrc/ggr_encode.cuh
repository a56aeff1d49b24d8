// ggr_encode.cuh - request side: canonical JSON arguments -> protobuf wire bytes.
//
// Replaces, per item, protojson.Unmarshal into a dynamicpb message followed by proto.Marshal
// inside conn.Invoke (/root/reference/pkg/grpc/reflection.go:351-357,373) with two streaming
// passes and no DOM:
//   pass A (encode_parse): one scan of the JSON text.  Validates tokens, resolves keys through
//          the per-message hash table, parses scalars, and writes one 16-byte IR node per value
//          into scratch HBM.  Children of a message are linked in wire-emit order (ascending
//          field number), map entries in key order, and every length-delimited size is known
//          when its container closes - so the exact output size of the item falls out.
//   pass B (encode_emit): walks the IR in emit order and writes tags, varints and payloads
//          (string bytes are copied/unescaped straight from the JSON text) at the item's final
//          offset, which a prefix sum over the pass-A sizes provides.
// Semantics restated from [upstream encoding/protojson/decode.go, proto/encode.go,
// types/dynamicpb/dynamic.go]; see oracle/orc_protojson.h for the line-by-line restatement the
// tests compare against.
#pragma once
#include "ggr_json_in.cuh"
#include "ggr_float.cuh"

#define GGR_MAX_DEPTH 32
// leave the current step with a result (used inside the convergent step loops)
#define GGR_RET(x) do { rr = (x); goto step_end; } while (0)
#define GGR_NIL 0xFFFFFu
#define GGR_MAX_NODES 0xFFFFFu

enum { N_SKIP = 0, N_VARINT = 1, N_FIX32 = 2, N_FIX64 = 3, N_STR = 4, N_BYTES = 5, N_MSG = 6, N_LIST = 7, N_MAP = 8, N_ENTRY = 9,
       N_FMPATH = 10 /* one path of a FieldMask: a = position of its first byte, b = byte count; written snake_case */ };
#define NF_ESC 1u     /* string token has escapes: decode while copying */
#define NF_PACKED 2u  /* N_LIST: packed */
#define NF_URL 4u     /* N_BYTES: URL-safe alphabet */
#define NF_PADDED 1u  /* N_BYTES: text length % 4 == 0 -> padded decoding mode */
#define NF_RAWKEY 8u  /* map key kept as its raw value; wire transform applied at emit time */

// IR node: a, b payload; link = next(20) | emit(12); meta = type(4) | flags(4) | tag(24)
struct Node {
  u32 a, b, link, meta;
};
GGR_DEV u32 node_meta(u32 type, u32 flags, u32 tag) { return type | (flags << 4) | (tag << 8); }
GGR_DEV void node_store(u8* ir, u32 idx, u32 a, u32 b, u32 next, u32 emit, u32 meta) {
  U4 v = {a, b, (next & 0xFFFFFu) | (emit << 20), meta};
  ggr_st16(ir + (size_t)idx * 16, v);
}
GGR_DEV U4 node_load(const u8* ir, u32 idx) { return ggr_ld16_rw(ir + (size_t)idx * 16); }
GGR_DEV void node_set_next(u8* ir, u32 idx, u32 next) {
  u8* p = ir + (size_t)idx * 16 + 8;
  u32 l = ggr_ld4_rw(p);
  ggr_st4(p, (l & 0xFFF00000u) | (next & 0xFFFFFu));
}

enum { FR_ROOT = 0, FR_MSG = 1, FR_LIST = 2, FR_MAP = 3 };

struct Frame {
  u32 node;      // IR index of the container's node
  u32 size;      // payload bytes accumulated
  u32 head, tail;
  u32 tail_emit; // FR_MSG: emit index of tail
  u32 oneofs;    // FR_MSG: real oneofs already set (bit per oneof index)
  u32 ref;       // FR_MSG: message index; FR_LIST / FR_MAP: global index of the field
  u32 kind;      // FR_*
  u32 st;        // 0 fresh, 1 after a value
  u32 emit;      // emit index of this container in its parent message (FR_MSG child of LIST/MAP: unused)
  u32 tag;       // tag to write in front of this container (0 = none)
  // FR_MAP: entry under construction
  u32 ent_node, key_node, key_body;
  u64 tail_key;  // FR_MAP: numeric key of tail entry / source position of its string key
  // FR_MSG: this message's key table and first field (cached from GgrMsg)
  u32 kh_first, kh_mask, field_first;
};

struct EncCtx {
  Tables T;
  const u8* in;  // 16-byte aligned base of the batch JSON buffer
  u32 end;       // end offset of this item
  u8* ir;
  u32 ir_cap, n_nodes;
  u32* ioff;     // lock-step parser only: output offset of every IR node (relative to the item)
};

GGR_DEV u32 zigzag32(u32 v) { return (v << 1) ^ (u32)((i32)v >> 31); }
GGR_DEV u64 zigzag64(u64 v) { return (v << 1) ^ (u64)((i64)v >> 63); }

// bytewise comparison of two string tokens (decoded), Go string ordering
GGR_DEV int cmp_str_tokens(const u8* base, u32 a_pos, u32 b_pos, u32 end) {
  StrIter a, b;
  a.init(base, a_pos, end);
  b.init(base, b_pos, end);
  for (;;) {
    if (a.eof()) return b.eof() ? 0 : -1;
    if (b.eof()) return 1;
    u32 x = a.peek(), y = b.peek();
    if (x != y) return x < y ? -1 : 1;
    a.adv();
    b.adv();
  }
}

// ---- base64 (Go encoding/base64 DecodeString as protojson's unmarshalBytes drives it) ----
GGR_DEV int b64_val(u32 c, bool url) {
  if (c - 'A' < 26u) return (int)(c - 'A');
  if (c - 'a' < 26u) return (int)(c - 'a' + 26);
  if (c - '0' < 10u) return (int)(c - '0' + 52);
  if (url) {
    if (c == '-') return 62;
    if (c == '_') return 63;
  } else {
    if (c == '+') return 62;
    if (c == '/') return 63;
  }
  return -1;
}
// Walks the base64 text; EMIT=false validates and counts, EMIT=true writes the bytes.
// `total_len` is the decoded-string length (newlines included) that selects padded / raw mode.
template <bool EMIT, class W>
GGR_DEV bool b64_run(StrIter& it, bool url, u32 total_len, W* w, u32* out_len) {
  bool padded = (total_len & 3u) == 0;
  u32 n = 0;
  bool end = false;
  while (!end) {
    u32 d[4] = {0, 0, 0, 0};
    int dlen = 4, j = 0;
    for (; j < 4; j++) {
      if (it.eof()) {
        if (j == 0) { *out_len = n; return true; }
        if (j == 1 || padded) return false;
        dlen = j;
        end = true;
        break;
      }
      u32 c = it.peek();
      it.adv();
      int v = b64_val(c, url);
      if (v >= 0) { d[j] = (u32)v; continue; }
      if (c == '\n' || c == '\r') { j--; continue; }
      if (c != '=' || !padded) return false;
      if (j < 2) return false;
      if (j == 2) {
        while (!it.eof() && (it.peek() == '\n' || it.peek() == '\r')) it.adv();
        if (it.eof() || it.peek() != '=') return false;
        it.adv();
      }
      while (!it.eof() && (it.peek() == '\n' || it.peek() == '\r')) it.adv();
      if (!it.eof()) return false;
      dlen = j;
      end = true;
      break;
    }
    u32 v = (d[0] << 18) | (d[1] << 12) | (d[2] << 6) | d[3];
    int nb = dlen - 1;
    if (nb > 0) {
      if (EMIT) {
        u32 bytes = ((v >> 16) & 0xFF) | (((v >> 8) & 0xFF) << 8) | ((v & 0xFF) << 16);
        if (nb < 3) bytes &= (nb == 2) ? 0xFFFFu : 0xFFu;
        w->put(bytes, nb);
      }
      n += (u32)nb;
    }
  }
  *out_len = n;
  return true;
}

// ---- RFC 3339 timestamps as time.Parse(RFC3339Nano) + protojson accept them ----
GGR_DEV i64 days_from_civil(i64 y, u32 m, u32 d) {
  y -= m <= 2;
  i64 era = (y >= 0 ? y : y - 399) / 400;
  u32 yoe = (u32)(y - era * 400);
  u32 doy = (153 * (m + (m > 2 ? (u32)-3 : 9u)) + 2) / 5 + d - 1;
  u32 doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + (i64)doe - 719468;
}
GGR_DEV int parse_timestamp(StrIter& it, i64* secs, i32* nanos) {
  auto dig = [&](u32* v) -> bool {
    u32 c = it.get();
    if (!(c - '0' < 10u)) return false;
    *v = c - '0';
    it.adv();
    return true;
  };
  auto two = [&](u32* v) -> bool {
    u32 a, b;
    if (!dig(&a) || !dig(&b)) return false;
    *v = a * 10 + b;
    return true;
  };
  auto lit = [&](u32 ch) -> bool {
    if (it.eof() || it.peek() != ch) return false;
    it.adv();
    return true;
  };
  u32 y0, y1, mon, day, hh, mi, ss;
  if (!two(&y0) || !two(&y1)) return GST_INVALID_VALUE;
  u32 year = y0 * 100 + y1;
  if (!lit('-') || !two(&mon) || !lit('-') || !two(&day) || !lit('T')) return GST_INVALID_VALUE;
  if (!dig(&hh)) return GST_INVALID_VALUE;  // stdHour: one or two digits
  {
    u32 c = it.get();
    if (c - '0' < 10u) {
      hh = hh * 10 + (c - '0');
      it.adv();
    }
  }
  if (!lit(':') || !two(&mi) || !lit(':') || !two(&ss)) return GST_INVALID_VALUE;
  u32 ns = 0, frac_digits = 0;
  bool frac_period = false;
  {
    u32 c = it.get();
    if (c == '.' || c == ',') {
      StrIter save = it;
      it.adv();
      u32 d0 = it.get();
      if (d0 - '0' < 10u) {
        frac_period = c == '.';
        u32 scale = 0;
        while (!it.eof() && it.peek() - '0' < 10u) {
          if (scale < 9) {
            ns = ns * 10 + (it.peek() - '0');
            scale++;
          }
          frac_digits++;
          it.adv();
        }
        for (; scale < 9; scale++) ns *= 10;
      } else {
        it = save;  // fractional second omitted; the separator will fail the zone match
      }
    }
  }
  i64 off = 0;
  if (it.eof()) return GST_INVALID_VALUE;
  if (it.peek() == 'Z') {
    it.adv();
  } else {
    u32 sign = it.peek();
    it.adv();
    u32 oh, om;
    if (!two(&oh) || !lit(':') || !two(&om)) return GST_INVALID_VALUE;
    if (sign != '+' && sign != '-') return GST_INVALID_VALUE;
    if (oh > 24 || om > 60) return GST_INVALID_VALUE;
    off = (i64)((oh * 60 + om) * 60);
    if (sign == '-') off = -off;
  }
  if (!it.eof()) return GST_INVALID_VALUE;
  if (mon < 1 || mon > 12 || hh >= 24 || mi >= 60 || ss >= 60) return GST_INVALID_VALUE;
  u32 maxd = (mon == 2) ? 28u : ((mon == 4 || mon == 6 || mon == 9 || mon == 11) ? 30u : 31u);
  bool leap = (year % 4 == 0 && year % 100 != 0) || year % 400 == 0;
  if (mon == 2 && leap) maxd = 29;
  if (day < 1 || day > maxd) return GST_INVALID_VALUE;
  i64 s = days_from_civil((i64)year, mon, day) * 86400 + (i64)(hh * 3600 + mi * 60 + ss) - off;
  // protojson checks the seconds range before the length of a '.' fraction: out of range with a long fraction is RANGE
  if (s < -62135596800ll || s > 253402300799ll) return GST_RANGE;
  if (frac_period && frac_digits > 9) return GST_INVALID_VALUE;
  *secs = s;
  *nanos = (i32)ns;
  return GST_OK;
}

// google.protobuf.Duration: "[+-]digits[.digits]s" exactly as protojson's parseDuration reads it (well_known_types.go):
// one leading '0' or a run of digits starting with 1-9 or nothing, an optional '.' with up to nine digits, the 's' last
GGR_DEV int parse_duration(StrIter& it, i64* secs, i32* nanos) {
  bool neg = false;
  u32 c = it.get();
  if (c == '-' || c == '+') {
    neg = c == '-';
    it.adv();
  }
  if (it.eof()) return GST_INVALID_VALUE;
  c = it.peek();
  u64 sv = 0;
  u32 nd = 0;
  bool ovf = false;
  if (c == 's') return GST_INVALID_VALUE;  // nothing in front of the suffix
  if (c == '0') {
    it.adv();
  } else if (c - '1' < 9u) {
    while (!it.eof() && it.peek() - '0' < 10u) {
      const u32 d = it.peek() - '0';
      if (sv > 922337203685477580ull || (sv == 922337203685477580ull && d > 7u)) ovf = true;  // strconv.ParseInt range
      sv = sv * 10u + d;
      nd++;
      it.adv();
    }
  } else if (c != '.') {
    return GST_INVALID_VALUE;
  }
  u32 ns = 0;
  if (it.get() == '.') {
    it.adv();
    u32 k = 0;
    while (!it.eof() && k < 9u && it.peek() - '0' < 10u) {
      ns = ns * 10u + (it.peek() - '0');
      k++;
      it.adv();
    }
    for (; k < 9u; k++) ns *= 10u;
  }
  if (it.get() != 's') return GST_INVALID_VALUE;
  it.adv();
  if (!it.eof() || ovf) return GST_INVALID_VALUE;
  i64 s = (i64)sv;
  i32 n = (i32)ns;
  if (neg) {
    s = -s;
    n = -n;
  }
  if (s < -315576000000ll || s > 315576000000ll) return GST_RANGE;
  *secs = s;
  *nanos = n;
  return GST_OK;
}

// ---- scalar -> node payload ----
struct Leaf {
  u32 type, a, b, body, flags;
  bool zero;
};
GGR_DEV void leaf_from_int(u32 kind, u64 v, Leaf* l) {
  l->flags = 0;
  l->zero = v == 0;
  switch (kind) {
    case GK_SINT32: v = zigzag32((u32)v); goto varint;
    case GK_SINT64: v = zigzag64(v); goto varint;
    case GK_FIXED32: case GK_SFIXED32: case GK_FLOAT:
      l->type = N_FIX32; l->a = (u32)v; l->b = 0; l->body = 4; return;
    case GK_FIXED64: case GK_SFIXED64: case GK_DOUBLE:
      l->type = N_FIX64; l->a = (u32)v; l->b = (u32)(v >> 32); l->body = 8; return;
    default:
    varint:
      l->type = N_VARINT; l->a = (u32)v; l->b = (u32)(v >> 32); l->body = varint_size(v); return;
  }
}

GGR_DEV bool kind_is_signed(u32 k) { return k == GK_INT32 || k == GK_INT64 || k == GK_SINT32 || k == GK_SINT64 || k == GK_SFIXED32 || k == GK_SFIXED64; }
GGR_DEV int kind_bits(u32 k) {
  return (k == GK_INT32 || k == GK_UINT32 || k == GK_SINT32 || k == GK_FIXED32 || k == GK_SFIXED32) ? 32 : 64;
}

// Does the decoded text of the valid string token at q end in a character strings.TrimSpace removes?  The ASCII spaces
// and U+0085, U+00A0, U+1680, U+2000-200A, U+2028, U+2029, U+202F, U+205F, U+3000.  (A quoted number that starts with
// one fails the number parser.)
GGR_DEV bool str_ends_in_space(const u8* in, u32 q, u32 end) {
  StrIter it;
  it.init(in, q, end);
  u32 c2 = 0, c1 = 0, c0 = 0;  // the last three decoded bytes, c0 the last
  while (!it.eof()) {
    c2 = c1;
    c1 = c0;
    c0 = it.peek();
    it.adv();
  }
  if (c0 == ' ' || (c0 - 9u) < 5u) return true;
  if (c1 == 0xC2u) return c0 == 0x85u || c0 == 0xA0u;
  if (c2 == 0xE1u) return c1 == 0x9Au && c0 == 0x80u;
  if (c2 == 0xE2u) return (c1 == 0x80u && (c0 - 0x80u <= 0x0Au || c0 == 0xA8u || c0 == 0xA9u || c0 == 0xAFu)) || (c1 == 0x81u && c0 == 0x9Fu);
  return c2 == 0xE3u && c1 == 0x80u && c0 == 0x80u;
}

// Parses one scalar value of `kind` at the reader.  Returns a GST_* status.
GGR_DEV int parse_scalar(EncCtx& cx, Rd& r, u32 kind, i32 child, Leaf* l) {
  u32 c = r.get();
  switch (kind) {
    case GK_BOOL: {
      if (match_literal(r, LIT4('t', 'r', 'u', 'e'), 4, 0)) { leaf_from_int(GK_BOOL, 1, l); return GST_OK; }
      if (match_literal(r, LIT4('f', 'a', 'l', 's'), 5, 'e')) { leaf_from_int(GK_BOOL, 0, l); return GST_OK; }
      break;
    }
    case GK_INT32: case GK_INT64: case GK_UINT32: case GK_UINT64: case GK_SINT32: case GK_SINT64:
    case GK_FIXED32: case GK_FIXED64: case GK_SFIXED32: case GK_SFIXED64: {
      NumTok t;
      u64 v;
      if (c == '"') {
        u32 q = r.pos;
        StrInfo si;
        int st = scan_string<false>(r, &si);
        if (st != GST_OK) return st;
        if (si.dec_len == 0) return GST_INVALID_VALUE;
        StrIter it;
        it.init(cx.in, q, cx.end);
        if (!parse_number(it, &t)) return GST_INVALID_VALUE;
        if (str_ends_in_space(cx.in, q, cx.end)) return GST_INVALID_VALUE;  // strings.TrimSpace must be a no-op
      } else if (c == '-' || c - '0' < 10u) {
        RawIter it = {&r};
        if (!parse_number(it, &t)) return GST_SYNTAX;
      } else {
        break;
      }
      if (!num_to_int(t, kind_is_signed(kind), kind_bits(kind), &v)) return GST_INVALID_VALUE;
      if (kind_bits(kind) == 32 && !kind_is_signed(kind)) v &= 0xFFFFFFFFull;
      leaf_from_int(kind, v, l);
      return GST_OK;
    }
    case GK_ENUM: {
      if (c == '"') {
        u32 q = r.pos;
        KeyInfo ki;
        int st = scan_key(r, &ki);
        if (st != GST_OK) return st;
        U4 e = ggr_ld16(cx.T.enums + (size_t)child * 16);
        i32 num;
        if (!hash_lookup(cx.T, e.z, e.w, ki, cx.in, q, cx.end, &num)) return GST_INVALID_VALUE;
        leaf_from_int(GK_ENUM, (u64)(i64)num, l);
        return GST_OK;
      }
      if (c == '-' || c - '0' < 10u) {
        NumTok t;
        u64 v;
        RawIter it = {&r};
        if (!parse_number(it, &t)) return GST_SYNTAX;
        if (!num_to_int(t, true, 32, &v)) return GST_INVALID_VALUE;
        leaf_from_int(GK_ENUM, v, l);
        return GST_OK;
      }
      break;
    }
    case GK_STRING: {
      if (c != '"') break;
      u32 q = r.pos;
      StrInfo si;
      int st = scan_string<false>(r, &si);
      if (st != GST_OK) return st;
      l->type = N_STR;
      l->a = q;
      l->b = si.dec_len;
      l->flags = (si.flags & SF_ESCAPES) ? NF_ESC : 0;
      l->body = varint_size(si.dec_len) + si.dec_len;
      l->zero = si.dec_len == 0;
      return GST_OK;
    }
    case GK_BYTES: {
      if (c != '"') break;
      u32 q = r.pos;
      StrInfo si;
      int st = scan_string<true>(r, &si);
      if (st != GST_OK) return st;
      StrIter it;
      it.init(cx.in, q, cx.end);
      u32 n;
      bool url = (si.flags & SF_URLSAFE) != 0;
      if (!b64_run<false, Cnt>(it, url, si.dec_len, (Cnt*)0, &n)) return GST_INVALID_VALUE;
      l->type = N_BYTES;
      l->a = q;
      l->b = n;
      l->flags = (url ? NF_URL : 0) | ((si.dec_len & 3u) ? 0 : NF_PADDED);
      l->body = varint_size(n) + n;
      l->zero = n == 0;
      return GST_OK;
    }
    case GK_FLOAT: case GK_DOUBLE: {
      // [upstream protojson unmarshalFloat]: number token, or a string holding NaN / Infinity /
      // -Infinity / one number token; strconv.ParseFloat decides, a range error is an error.
      const bool is32 = kind == GK_FLOAT;
      NumTok t;
      u64 bits = 0;
      bool ok;
      if (c == '"') {
        u32 q = r.pos;
        StrInfo si;
        int st = scan_string<false>(r, &si);
        if (st != GST_OK) return st;
        if (str_token_is(cx.in, q, cx.end, "NaN", 3)) {
          bits = is32 ? 0x7FC00000ull : 0x7FF8000000000001ull;  // float32(math.NaN()) / math.NaN()
          ok = true;
        } else if (str_token_is(cx.in, q, cx.end, "Infinity", 8)) {
          bits = is32 ? 0x7F800000ull : 0x7FF0000000000000ull;
          ok = true;
        } else if (str_token_is(cx.in, q, cx.end, "-Infinity", 9)) {
          bits = is32 ? 0xFF800000ull : 0xFFF0000000000000ull;
          ok = true;
        } else {
          if (si.dec_len == 0) return GST_INVALID_VALUE;
          StrIter it;
          it.init(cx.in, q, cx.end);
          if (!parse_number(it, &t)) return GST_INVALID_VALUE;
          if (str_ends_in_space(cx.in, q, cx.end)) return GST_INVALID_VALUE;  // strings.TrimSpace must be a no-op
          StrIter again;
          again.init(cx.in, q, cx.end);
          ok = float_from_token(again, t, is32, &bits);
        }
      } else if (c == '-' || c - '0' < 10u) {
        Rd start = r;
        RawIter it = {&r};
        if (!parse_number(it, &t)) return GST_SYNTAX;
        RawIter again = {&start};
        ok = float_from_token(again, t, is32, &bits);
      } else {
        break;
      }
      if (!ok) return GST_INVALID_VALUE;
      l->flags = 0;
      l->zero = bits == 0;  // -0.0 is "set" (dynamicpb isSet: value != 0 || signbit)
      if (is32) { l->type = N_FIX32; l->a = (u32)bits; l->b = 0; l->body = 4; }
      else { l->type = N_FIX64; l->a = (u32)bits; l->b = (u32)(bits >> 32); l->body = 8; }
      return GST_OK;
    }
    default:
      return GST_UNSUPPORTED;
  }
  // wrong token type for this kind: a syntactically valid value is an INVALID_VALUE, garbage is
  // a SYNTAX error; telling them apart needs the token, so classify by first byte
  if (c == '"' || c == '{' || c == '[' || c == '-' || c - '0' < 10u || c == 't' || c == 'f' || c == 'n') {
    // make sure literals are well formed before calling it a type error
    if (c == 't' && !match_literal(r, LIT4('t', 'r', 'u', 'e'), 4, 0)) return GST_SYNTAX;
    if (c == 'f' && !match_literal(r, LIT4('f', 'a', 'l', 's'), 5, 'e')) return GST_SYNTAX;
    if (c == 'n' && !match_literal(r, LIT4('n', 'u', 'l', 'l'), 4, 0)) return GST_SYNTAX;
    if (c == '"') {
      StrInfo si;
      int st = scan_string<false>(r, &si);
      if (st != GST_OK) return st;
    }
    if (c == '-' || c - '0' < 10u) {
      NumTok t;
      RawIter it = {&r};
      if (!parse_number(it, &t)) return GST_SYNTAX;
    }
    return GST_INVALID_VALUE;
  }
  return GST_SYNTAX;
}

// --------------------------------------------------------------------------------------------
// pass A
// --------------------------------------------------------------------------------------------
GGR_DEV int enc_new_node(EncCtx& cx, u32* idx) {
  if (cx.n_nodes >= cx.ir_cap || cx.n_nodes >= GGR_MAX_NODES) return GST_TOO_LARGE;
  *idx = cx.n_nodes++;
  return GST_OK;
}

// Links a finished child into the current frame and accounts for its bytes.
//   body  : bytes after the tag (varint / fixed / length prefix + payload)
//   live  : false for elided values (null, implicit zero) - linked for duplicate detection only
GGR_DEV int frame_add(EncCtx& cx, Frame& fr, u32 idx, u32 emit, u32 tag_len, u32 body, bool live, u32* next_out) {
  *next_out = GGR_NIL;
  if (fr.kind == FR_MSG) {
    if (fr.head == GGR_NIL) {
      fr.head = fr.tail = idx;
      fr.tail_emit = emit;
    } else if (emit > fr.tail_emit) {
      node_set_next(cx.ir, fr.tail, idx);
      fr.tail = idx;
      fr.tail_emit = emit;
    } else if (emit == fr.tail_emit) {
      return GST_DUPLICATE;
    } else {
      u32 prev = GGR_NIL, cur = fr.head;
      for (;;) {
        u32 l = ggr_ld4_rw(cx.ir + (size_t)cur * 16 + 8);
        u32 e = l >> 20;
        if (e == emit) return GST_DUPLICATE;
        if (e > emit) break;
        prev = cur;
        cur = l & 0xFFFFFu;
      }
      *next_out = cur;
      if (prev == GGR_NIL) fr.head = idx;
      else node_set_next(cx.ir, prev, idx);
    }
    if (live) fr.size += tag_len + body;
    return GST_OK;
  }
  if (fr.kind == FR_LIST) {
    if (fr.head == GGR_NIL) fr.head = idx;
    else node_set_next(cx.ir, fr.tail, idx);
    fr.tail = idx;
    fr.size += tag_len + body;  // caller passes tag_len = 0 for packed lists
    return GST_OK;
  }
  return GST_OK;
}

// Completes a map entry whose value node is `val_idx` with `val_body` bytes after its 1-byte tag.
GGR_DEV int map_entry_done(EncCtx& cx, Frame& fr, const FieldD& mapf, u32 key_kind, u64 key_val, u32 key_pos, u32 val_body) {
  u32 payload = fr.key_body + 1 + val_body;
  u32 total = mapf.tag_len + varint_size(payload) + payload;
  // sorted insertion by key; duplicates are an error
  u32 ent = fr.ent_node;
  u32 next = GGR_NIL;
  bool is_str = key_kind == GK_STRING;
  bool is_unsigned = key_kind == GK_UINT32 || key_kind == GK_UINT64 || key_kind == GK_FIXED32 || key_kind == GK_FIXED64 || key_kind == GK_BOOL;
  auto cmp = [&](u64 other_val, u32 other_pos) -> int {  // compare new key with an existing one
    if (is_str) return cmp_str_tokens(cx.in, key_pos, other_pos, cx.end);
    if (is_unsigned) return key_val < other_val ? -1 : (key_val > other_val ? 1 : 0);
    return (i64)key_val < (i64)other_val ? -1 : ((i64)key_val > (i64)other_val ? 1 : 0);
  };
  if (fr.head == GGR_NIL) {
    fr.head = fr.tail = ent;
  } else {
    int c = cmp(fr.tail_key, (u32)fr.tail_key);
    if (c == 0) return GST_DUPLICATE;
    if (c > 0) {
      node_set_next(cx.ir, fr.tail, ent);
      fr.tail = ent;
    } else {
      u32 prev = GGR_NIL, cur = fr.head;
      for (;;) {
        U4 en = node_load(cx.ir, cur);
        U4 kn = node_load(cx.ir, en.y);  // entry.b = key node
        u64 ov = is_str ? (u64)kn.x : ((u64)kn.x | ((u64)kn.y << 32));
        // numeric keys are stored in wire form; compare on the decoded value kept in kn for
        // varint kinds only when not zigzag - so the key node keeps the raw value in (a,b) and
        // the zigzag transform is applied at emit time (see NF_* use below)
        int cc = cmp(ov, kn.x);
        if (cc == 0) return GST_DUPLICATE;
        if (cc < 0) break;
        prev = cur;
        cur = en.z & 0xFFFFFu;
      }
      next = cur;
      if (prev == GGR_NIL) fr.head = ent;
      else node_set_next(cx.ir, prev, ent);
    }
  }
  if (fr.tail == ent) fr.tail_key = is_str ? (u64)key_pos : key_val;
  node_store(cx.ir, ent, payload, fr.key_node, next, 0, node_meta(N_ENTRY, 0, mapf.tag));
  fr.size += total;
  return GST_OK;
}

struct EncResult {
  u32 size;   // wire bytes of the item
  u32 first;  // first top-level node (GGR_NIL when the message is empty)
  u32 n_nodes;  // lock-step parser: IR nodes written (with offsets, for the lock-step emitter); 0 otherwise
  // envelope mode (request bodies): method index, position and length of the id token in the body
  u32 method, id_pos, id_len;
  // items that fail in the per-thread parser: byte offset (from the item's start) of the key token for unknown / duplicate
  // fields and oneof conflicts found while the key is at hand, else of the reader when the error was raised
  u32 err_pos;
};

// Rare value forms of encode_parse as calls (inlined they add 35 thousand instructions to the kernel): the text of a
// Timestamp / Duration string, the value of a wrapper message.
// google.protobuf.FieldMask: "a,fooBar.baz" -> paths a, foo_bar.baz (protojson unmarshalFieldMask: TrimSpace, split
// at ',', JSONSnakeCase, no '_' in the JSON form, the result a valid dotted name).  One N_FMPATH node per path, chained
// behind *head; *payload = their wire bytes.  The token must be free of escapes: a mask written with escapes is left to
// the caller as unsupported, never answered differently.
GGR_DEVN int parse_field_mask(EncCtx& cx, u32 quote_pos, u32 close_pos, bool escapes, u32* head, u32* payload) {
  *head = GGR_NIL;
  *payload = 0;
  if (escapes) return GST_UNSUPPORTED;
  const u8* in = cx.in;
  u32 b = quote_pos + 1u, e = close_pos;  // [b, e): the text between the quotes
  // strings.TrimSpace: ' ' (the other ASCII spaces cannot stand unescaped in a JSON string) and the Unicode spaces
  // U+0085, U+00A0, U+1680, U+2000-200A, U+2028, U+2029, U+202F, U+205F, U+3000
  auto space_len = [&](u32 p, u32 lim) -> u32 {  // bytes of the space that starts at p (0: none)
    const u32 c0 = in[p];
    if (c0 == ' ') return 1u;
    if (c0 == 0xC2u && p + 1u < lim && (in[p + 1u] == 0x85u || in[p + 1u] == 0xA0u)) return 2u;
    if (p + 2u < lim) {
      const u32 c1 = in[p + 1u], c2 = in[p + 2u];
      if (c0 == 0xE1u && c1 == 0x9Au && c2 == 0x80u) return 3u;
      if (c0 == 0xE2u && c1 == 0x80u && (c2 - 0x80u <= 0x0Au || c2 == 0xA8u || c2 == 0xA9u || c2 == 0xAFu)) return 3u;
      if (c0 == 0xE2u && c1 == 0x81u && c2 == 0x9Fu) return 3u;
      if (c0 == 0xE3u && c1 == 0x80u && c2 == 0x80u) return 3u;
    }
    return 0u;
  };
  for (u32 k; b < e && (k = space_len(b, e)) != 0u;) b += k;
  while (e > b) {
    u32 k = e - 1u;  // start of the last character
    while (k > b && (in[k] & 0xC0u) == 0x80u) k--;
    const u32 n = space_len(k, e);
    if (n == 0u || k + n != e) break;
    e = k;
  }
  if (b == e) return GST_OK;
  u32 tail = GGR_NIL;
  u32 p = b;
  for (;;) {
    // one path [p, q)
    u32 q = p, extra = 0;
    bool seg_start = true, valid = true;
    while (q < e && in[q] != ',') {
      const u32 c = in[q];
      const bool upper = c - 'A' < 26u, lower = c - 'a' < 26u, digit = c - '0' < 10u;
      if (c == '.') {
        if (seg_start) valid = false;  // empty segment
        seg_start = true;
      } else {
        if (upper) extra++;
        // after JSONSnakeCase an upper-case letter is "_x": a letter either way; '_' itself is not allowed in the JSON form
        if (!(upper || lower || (digit && !seg_start))) valid = false;
        seg_start = false;
      }
      q++;
    }
    if (seg_start || !valid) return GST_INVALID_VALUE;  // empty path, trailing '.', foreign characters
    const u32 out_len = (q - p) + extra;
    u32 idx;
    int st = enc_new_node(cx, &idx);
    if (st != GST_OK) return st;
    node_store(cx.ir, idx, p, q - p, GGR_NIL, 0, node_meta(N_FMPATH, 0, 0x0Au));
    if (tail == GGR_NIL) *head = idx;
    else node_set_next(cx.ir, tail, idx);
    tail = idx;
    *payload += 1u + varint_size(out_len) + out_len;
    if (q >= e) break;
    p = q + 1u;
    if (p >= e) return GST_INVALID_VALUE;  // "a," : an empty last path
  }
  return GST_OK;
}
GGR_DEVN int parse_time_value(const u8* in, u32 quote_pos, u32 end, bool duration, i64* secs, i32* nanos) {
  StrIter it;
  it.init(in, quote_pos, end);
  return duration ? parse_duration(it, secs, nanos) : parse_timestamp(it, secs, nanos);
}
GGR_DEVN int parse_scalar_at(EncCtx& cx, u32 pos, u32 kind, i32 child, Leaf* l, u32* next) {
  Rd r;
  r.init(cx.in, pos, cx.end);
  const int st = parse_scalar(cx, r, kind, child, l);
  *next = r.pos;
  return st;
}

// null as a list element or map value is a value like any other: protojson reads it as an unexpected token where a
// message is due (Timestamp, Duration, FieldMask and Empty included) and as an invalid value where a scalar is, the bare
// value of a wrapper too (unmarshalWrapperType reads the value field as a scalar)
GGR_DEV int null_element_status(const Tables& T, const FieldD& f) {
  if (f.kind != GK_MESSAGE) return GST_INVALID_VALUE;
  return ggr_msg(T, (u32)f.child).wkt == GGR_WKT_WRAPPER ? GST_INVALID_VALUE : GST_SYNTAX;
}

// `active` is false for lanes that have no item (they only take part in the convergence votes);
// `mask` names the lanes that call this function together.
GGR_DEV int encode_parse(const Tables& T, u32 root_msg, const u8* in, u32 start, u32 end, u8* ir, u32 ir_cap, EncResult* res,
                         bool active = true, unsigned mask = GGR_FULL_MASK) {
  res->size = 0;
  res->first = GGR_NIL;
  res->n_nodes = 0;
  res->err_pos = 0;
  bool finished = !active;
  int result = GST_OK;
  // reflection.go:354: "" and "{}" skip protojson entirely
  if (end == start) finished = true;
  EncCtx cx;
  cx.T = T;
  cx.in = in;
  cx.end = end;
  cx.ir = ir;
  cx.ir_cap = ir_cap;
  cx.n_nodes = 0;
  cx.ioff = nullptr;
  Rd r;
  if (!finished) {
    r.init(in, start, end);
    if (end - start == 2 && (r.peek4() & 0xFFFFu) == (u32)('{' | ('}' << 8))) finished = true;
  } else {
    r.base = in; r.pos = r.end = r.fetch = 0; r.avail = 0; r.rw = 0; r.cur = 0; r.ch.x = r.ch.y = r.ch.z = r.ch.w = 0;
  }

  Frame stk[GGR_MAX_DEPTH];
  int depth = 0;
  Frame fr;
  fr.kind = FR_ROOT;
  fr.st = 0;
  fr.size = 0;
  fr.head = fr.tail = GGR_NIL;
  fr.node = GGR_NIL;
  fr.ref = root_msg;
  fr.tag = 0;
  fr.emit = 0;
  fr.oneofs = 0;
  fr.tail_emit = 0;
  fr.ent_node = fr.key_node = GGR_NIL;
  fr.key_body = 0;
  fr.tail_key = 0;
  fr.kh_first = fr.kh_mask = fr.field_first = 0;

  // One step = one member / element / container close.  All lanes of `mask` re-converge at the
  // vote after every step (see ggr_prim.cuh).
  while (ggr_any(mask, !finished)) {
   if (!finished) {
    int rr = GGR_STEP_CONT;
    u32 ekey = 0xFFFFFFFFu;  // position of the member key read in this step (error reporting)
  for (int once = 0;; once++) {
    if (once) break;  // `continue` in the body below ends the step
    skip_ws(r);
    // ---- what does the current container expect? ----
    FieldD f;          // field the upcoming value belongs to
    u32 emit = 0;      // its emit index (FR_MSG)
    u32 vmsg = 0;      // message type when the value is a message
    bool want_value = false;
    u32 map_key_kind = 0, map_key_pos = 0;
    u64 map_key_val = 0;
    FieldD mapf;       // FR_MAP: the map field itself
    mapf.tag = 0; mapf.tag_len = 0;

    if (fr.kind == FR_ROOT) {
      if (fr.st == 0) {
        fr.st = 1;
        // the root behaves like a singular message value
        f.kind = GK_MESSAGE; f.child = (i32)root_msg; f.flags = GF_PRESENCE; f.tag = 0; f.tag_len = 0; f.oneof = -1;
        f.number = 0; f.wt = 2; f.decl_index = 0; f.name_off = 0; f.name_len = 0;
        want_value = true;
      } else {
        if (!r.eof()) GGR_RET(GST_SYNTAX);
        res->size = fr.size;
        res->first = fr.head;
        GGR_RET(GST_OK);
      }
    } else if (fr.kind == FR_MSG || fr.kind == FR_MAP) {
      u32 c = r.get();
      if (c == '}') {
        r.skip(1);
        goto close_container;
      }
      if (fr.st == 1) {
        if (c != ',') GGR_RET(GST_SYNTAX);
        r.skip(1);
        skip_ws(r);
        c = r.get();
      }
      if (c != '"') GGR_RET(GST_SYNTAX);
      u32 key_pos = r.pos;
      ekey = key_pos;
      StrInfo ks;
      KeyInfo ki;
      ks.dec_len = 0; ks.flags = 0;
      int st = (fr.kind == FR_MSG) ? scan_key(r, &ki) : scan_string<false>(r, &ks);
      if (st != GST_OK) GGR_RET(st);
      skip_ws(r);
      if (r.get() != ':') GGR_RET(GST_SYNTAX);
      r.skip(1);
      skip_ws(r);
      fr.st = 1;
      if (fr.kind == FR_MSG) {
        i32 ei;
        if (!hash_lookup(T, fr.kh_first, fr.kh_mask, ki, in, key_pos, end, &ei)) GGR_RET(GST_UNKNOWN_FIELD);
        emit = (u32)ei;
        f = ggr_field(T, fr.field_first + emit);
        // JSON null: the field is skipped, but it still counts for duplicate detection
        if (r.get() == 'n') {
          if (!match_literal(r, LIT4('n', 'u', 'l', 'l'), 4, 0)) GGR_RET(GST_SYNTAX);
          u32 idx, nx;
          st = enc_new_node(cx, &idx);
          if (st != GST_OK) GGR_RET(st);
          st = frame_add(cx, fr, idx, emit, 0, 0, false, &nx);
          if (st != GST_OK) GGR_RET(st);
          node_store(ir, idx, 0, 0, nx, emit, node_meta(N_SKIP, 0, 0));
          continue;
        }
        if (f.flags & GF_MAP) {
          if (r.get() != '{') GGR_RET(GST_SYNTAX);
          r.skip(1);
          if (depth >= GGR_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
          u32 idx;
          st = enc_new_node(cx, &idx);
          if (st != GST_OK) GGR_RET(st);
          stk[depth++] = fr;
          Frame nf;
          nf.kind = FR_MAP; nf.st = 0; nf.size = 0; nf.head = nf.tail = GGR_NIL; nf.node = idx;
          nf.ref = fr.field_first + emit; nf.emit = emit; nf.tag = f.tag; nf.oneofs = 0; nf.tail_emit = 0;
          nf.kh_first = nf.kh_mask = nf.field_first = 0;
          nf.ent_node = nf.key_node = GGR_NIL; nf.key_body = 0; nf.tail_key = 0;
          fr = nf;
          continue;
        }
        if (f.flags & GF_REPEATED) {
          if (r.get() != '[') GGR_RET(GST_SYNTAX);
          r.skip(1);
          if (depth >= GGR_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
          u32 idx;
          st = enc_new_node(cx, &idx);
          if (st != GST_OK) GGR_RET(st);
          stk[depth++] = fr;
          Frame nf;
          nf.kind = FR_LIST; nf.st = 0; nf.size = 0; nf.head = nf.tail = GGR_NIL; nf.node = idx;
          nf.ref = fr.field_first + emit; nf.emit = emit; nf.tag = f.tag; nf.oneofs = 0; nf.tail_emit = 0;
          nf.kh_first = nf.kh_mask = nf.field_first = 0;
          nf.ent_node = nf.key_node = GGR_NIL; nf.key_body = 0; nf.tail_key = 0;
          fr = nf;
          continue;
        }
        if (f.oneof >= 0) {
          u32 bit = 1u << (f.oneof & 31);
          if (fr.oneofs & bit) GGR_RET(GST_ONEOF);
          fr.oneofs |= bit;
        }
        want_value = true;
      } else {
        // ---- map entry: key ----
        mapf = ggr_field(T, fr.ref);
        MsgD ed = ggr_msg(T, (u32)mapf.child);
        FieldD kf = ggr_field(T, ed.field_first);
        f = ggr_field(T, ed.field_first + 1);  // value field
        map_key_kind = kf.kind;
        map_key_pos = key_pos;
        u32 kidx, eidx;
        st = enc_new_node(cx, &eidx);
        if (st != GST_OK) GGR_RET(st);
        st = enc_new_node(cx, &kidx);
        if (st != GST_OK) GGR_RET(st);
        fr.ent_node = eidx;
        fr.key_node = kidx;
        Leaf kl;
        if (kf.kind == GK_STRING) {
          kl.type = N_STR; kl.a = key_pos; kl.b = ks.dec_len; kl.flags = (ks.flags & SF_ESCAPES) ? NF_ESC : 0;
          kl.body = varint_size(ks.dec_len) + ks.dec_len;
        } else if (kf.kind == GK_BOOL) {
          // "true" / "false" exactly
          if (str_token_is(in, key_pos, end, "true", 4)) map_key_val = 1;
          else if (str_token_is(in, key_pos, end, "false", 5)) map_key_val = 0;
          else GGR_RET(GST_INVALID_VALUE);
          leaf_from_int(GK_BOOL, map_key_val, &kl);
        } else {
          StrIter it;
          it.init(in, key_pos, end);
          if (!parse_key_int(it, kind_is_signed(kf.kind), kind_bits(kf.kind), &map_key_val)) GGR_RET(GST_INVALID_VALUE);
          leaf_from_int(kf.kind, map_key_val, &kl);
        }
        fr.key_body = 1 + kl.body;  // key tag is one byte (field 1)
        // key node: raw key value kept for ordering; wire form derived at emit time
        if (kf.kind == GK_STRING) node_store(ir, kidx, kl.a, kl.b, GGR_NIL, 0, node_meta(N_STR, kl.flags, kf.tag));
        else node_store(ir, kidx, (u32)map_key_val, (u32)(map_key_val >> 32), GGR_NIL, kf.kind, node_meta(kl.type, NF_RAWKEY, kf.tag));
        if (r.get() == 'n' ) {
          // a null map value fails for every value kind
          if (!match_literal(r, LIT4('n', 'u', 'l', 'l'), 4, 0)) GGR_RET(GST_SYNTAX);
          GGR_RET(null_element_status(T, f));
        }
        want_value = true;
      }
    } else {  // FR_LIST
      u32 c = r.get();
      if (c == ']') {
        r.skip(1);
        goto close_container;
      }
      if (fr.st == 1) {
        if (c != ',') GGR_RET(GST_SYNTAX);
        r.skip(1);
        skip_ws(r);
        if (r.get() == ']') GGR_RET(GST_SYNTAX);
      }
      fr.st = 1;
      f = ggr_field(T, fr.ref);
      if (r.get() == 'n') {
        if (!match_literal(r, LIT4('n', 'u', 'l', 'l'), 4, 0)) GGR_RET(GST_SYNTAX);
        GGR_RET(null_element_status(T, f));
      }
      want_value = true;
    }

    if (want_value) {
      if (f.kind == GK_MESSAGE) {
        vmsg = (u32)f.child;
        MsgD vd = ggr_msg(T, vmsg);
        if (vd.wkt != GGR_WKT_NONE) {
          // well-known types with a JSON form of their own: the value is finished here, as a message node with
          // its leaves, and handed to the container
          u32 midx, first = GGR_NIL, payload = 0;
          int st;
          if (vd.wkt == GGR_WKT_TIMESTAMP || vd.wkt == GGR_WKT_DURATION) {
            if (r.get() != '"') GGR_RET(GST_SYNTAX);
            u32 q = r.pos;
            StrInfo si;
            st = scan_string<false>(r, &si);
            if (st != GST_OK) GGR_RET(st);
            i64 secs;
            i32 nanos;
            st = parse_time_value(in, q, end, vd.wkt == GGR_WKT_DURATION, &secs, &nanos);
            if (st != GST_OK) GGR_RET(st);
            u32 sidx = GGR_NIL, nidx = GGR_NIL;
            st = enc_new_node(cx, &midx);
            if (st != GST_OK) GGR_RET(st);
            if (nanos != 0) {
              const u64 nv = (u64)(i64)nanos;  // int32 on the wire: sign-extended
              st = enc_new_node(cx, &nidx);
              if (st != GST_OK) GGR_RET(st);
              node_store(ir, nidx, (u32)nv, (u32)(nv >> 32), GGR_NIL, 1, node_meta(N_VARINT, 0, 16));
              payload += 1 + varint_size(nv);
            }
            if (secs != 0) {
              st = enc_new_node(cx, &sidx);
              if (st != GST_OK) GGR_RET(st);
              node_store(ir, sidx, (u32)(u64)secs, (u32)((u64)secs >> 32), nidx, 0, node_meta(N_VARINT, 0, 8));
              payload += 1 + varint_size((u64)secs);
            }
            first = sidx != GGR_NIL ? sidx : nidx;
          } else if (vd.wkt == GGR_WKT_WRAPPER) {
            // the bare value of field 1 (unmarshalWrapperType); the zero value leaves an empty message
            const FieldD vf = ggr_field(T, vd.field_first);
            Leaf l;
            u32 after;
            st = parse_scalar_at(cx, r.pos, vf.kind, vf.child, &l, &after);
            if (st != GST_OK) GGR_RET(st);
            r.init(in, after, end);
            st = enc_new_node(cx, &midx);
            if (st != GST_OK) GGR_RET(st);
            if (!l.zero) {
              u32 lidx;
              st = enc_new_node(cx, &lidx);
              if (st != GST_OK) GGR_RET(st);
              node_store(ir, lidx, l.a, l.b, GGR_NIL, 0, node_meta(l.type, l.flags, vf.tag));
              first = lidx;
              payload = vf.tag_len + l.body;
            }
          } else if (vd.wkt == GGR_WKT_FIELDMASK) {
            if (r.get() != '"') GGR_RET(GST_SYNTAX);
            u32 q = r.pos;
            StrInfo si;
            st = scan_string<false>(r, &si);
            if (st != GST_OK) GGR_RET(st);
            st = enc_new_node(cx, &midx);
            if (st != GST_OK) GGR_RET(st);
            st = parse_field_mask(cx, q, r.pos - 1u, (si.flags & SF_ESCAPES) != 0, &first, &payload);
            if (st != GST_OK) GGR_RET(st);
          } else if (vd.wkt == GGR_WKT_EMPTY) {
            // an object without members (unmarshalEmpty; DiscardUnknown is off on this path)
            if (r.get() != '{') GGR_RET(GST_SYNTAX);
            r.skip(1);
            skip_ws(r);
            if (r.get() == '"') {
              StrInfo si;
              st = scan_string<false>(r, &si);
              if (st != GST_OK) GGR_RET(st);
              skip_ws(r);
              if (r.get() != ':') GGR_RET(GST_SYNTAX);
              GGR_RET(GST_UNKNOWN_FIELD);
            }
            if (r.get() != '}') GGR_RET(GST_SYNTAX);
            r.skip(1);
            st = enc_new_node(cx, &midx);
            if (st != GST_OK) GGR_RET(st);
          } else {
            GGR_RET(GST_UNSUPPORTED);
          }
          u32 body = varint_size(payload) + payload;
          if (fr.kind == FR_MAP) {
            node_store(ir, midx, payload, first, GGR_NIL, 1, node_meta(N_MSG, 0, f.tag));
            node_set_next(ir, fr.key_node, midx);
            st = map_entry_done(cx, fr, mapf, map_key_kind, map_key_val, map_key_pos, body);
            if (st != GST_OK) GGR_RET(st);
          } else if (fr.kind == FR_ROOT) {
            fr.size = payload;
            fr.head = first;
          } else {
            u32 nx;
            st = frame_add(cx, fr, midx, emit, f.tag_len, body, true, &nx);
            if (st != GST_OK) GGR_RET(st);
            node_store(ir, midx, payload, first, nx, emit, node_meta(N_MSG, 0, f.tag));
          }
          continue;
        }
        if (r.get() != '{') GGR_RET(GST_SYNTAX);
        r.skip(1);
        if (depth >= GGR_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
        u32 idx;
        int st = enc_new_node(cx, &idx);
        if (st != GST_OK) GGR_RET(st);
        if (fr.kind == FR_MAP) {
          // remember the pending key for when this message closes (FR_MAP frames do not use
          // tail_emit / oneofs otherwise; the numeric key rides in the child's tail_key)
          fr.tail_emit = map_key_kind;
          fr.oneofs = map_key_pos;
        }
        stk[depth++] = fr;
        Frame nf;
        nf.kind = FR_MSG; nf.st = 0; nf.size = 0; nf.head = nf.tail = GGR_NIL; nf.node = idx;
        nf.ref = vmsg; nf.emit = emit; nf.tag = f.tag; nf.oneofs = 0; nf.tail_emit = 0;
        nf.ent_node = nf.key_node = GGR_NIL; nf.key_body = f.tag_len; nf.tail_key = map_key_val;
        nf.kh_first = vd.key_hash_first; nf.kh_mask = vd.key_hash_mask; nf.field_first = vd.field_first;
        fr = nf;
        continue;
      }
      // ---- scalar ----
      Leaf l;
      int st = parse_scalar(cx, r, f.kind, f.child, &l);
      if (st != GST_OK) GGR_RET(st);
      u32 idx;
      st = enc_new_node(cx, &idx);
      if (st != GST_OK) GGR_RET(st);
      if (fr.kind == FR_MSG) {
        bool live = (f.flags & GF_PRESENCE) || !l.zero;
        u32 nx;
        st = frame_add(cx, fr, idx, emit, f.tag_len, l.body, live, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, idx, l.a, l.b, nx, emit, live ? node_meta(l.type, l.flags, f.tag) : node_meta(N_SKIP, 0, 0));
      } else if (fr.kind == FR_LIST) {
        bool packed = (f.flags & GF_PACKED) != 0;
        u32 nx;
        st = frame_add(cx, fr, idx, 0, packed ? 0 : f.tag_len, l.body, true, &nx);
        if (st != GST_OK) GGR_RET(st);
        // element tag: the unpacked wire type (f.tag is the LEN tag when packed)
        node_store(ir, idx, l.a, l.b, GGR_NIL, 0, node_meta(l.type, l.flags, packed ? 0 : f.tag));
      } else if (fr.kind == FR_MAP) {
        node_store(ir, idx, l.a, l.b, GGR_NIL, 1, node_meta(l.type, l.flags, f.tag));
        node_set_next(ir, fr.key_node, idx);
        st = map_entry_done(cx, fr, mapf, map_key_kind, map_key_val, map_key_pos, l.body);
        if (st != GST_OK) GGR_RET(st);
      } else {
        GGR_RET(GST_SYNTAX);  // scalar at the root
      }
      continue;
    }
    continue;

  close_container : {
    // fr is a finished FR_MSG / FR_LIST / FR_MAP; fold it into its parent
    Frame done = fr;
    fr = stk[--depth];
    if (done.kind == FR_MSG) {
      u32 payload = done.size;
      u32 body = varint_size(payload) + payload;
      if (fr.kind == FR_ROOT) {
        fr.size = payload;
        fr.head = done.head;
        continue;
      }
      if (fr.kind == FR_MSG) {
        u32 nx;
        int st = frame_add(cx, fr, done.node, done.emit, done.key_body, body, true, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, done.node, payload, done.head, nx, done.emit, node_meta(N_MSG, 0, done.tag));
      } else if (fr.kind == FR_LIST) {
        u32 nx;
        int st = frame_add(cx, fr, done.node, 0, done.key_body, body, true, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, done.node, payload, done.head, GGR_NIL, 0, node_meta(N_MSG, 0, done.tag));
      } else {  // FR_MAP: message-valued entry
        FieldD mf = ggr_field(T, fr.ref);
        node_store(ir, done.node, payload, done.head, GGR_NIL, 1, node_meta(N_MSG, 0, done.tag));
        node_set_next(ir, fr.key_node, done.node);
        u32 kkind = fr.tail_emit, kpos = fr.oneofs;
        fr.tail_emit = 0;
        fr.oneofs = 0;
        int st = map_entry_done(cx, fr, mf, kkind, done.tail_key, kpos, body);
        if (st != GST_OK) GGR_RET(st);
      }
      continue;
    }
    // lists and maps always sit in a message
    FieldD pf = ggr_field(T, done.ref);
    if (done.kind == FR_LIST) {
      bool packed = (pf.flags & GF_PACKED) != 0;
      u32 nx;
      if (done.head == GGR_NIL) {  // empty list: field absent
        int st = frame_add(cx, fr, done.node, done.emit, 0, 0, false, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, done.node, 0, 0, nx, done.emit, node_meta(N_SKIP, 0, 0));
        continue;
      }
      if (packed) {
        u32 body = varint_size(done.size) + done.size;
        int st = frame_add(cx, fr, done.node, done.emit, pf.tag_len, body, true, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, done.node, done.size, done.head, nx, done.emit, node_meta(N_LIST, NF_PACKED, pf.tag));
      } else {
        int st = frame_add(cx, fr, done.node, done.emit, 0, done.size, true, &nx);
        if (st != GST_OK) GGR_RET(st);
        node_store(ir, done.node, done.size, done.head, nx, done.emit, node_meta(N_LIST, 0, 0));
      }
      continue;
    }
    // FR_MAP
    {
      u32 nx;
      bool live = done.head != GGR_NIL;
      int st = frame_add(cx, fr, done.node, done.emit, 0, done.size, live, &nx);
      if (st != GST_OK) GGR_RET(st);
      node_store(ir, done.node, done.size, done.head, nx, done.emit, live ? node_meta(N_MAP, 0, 0) : node_meta(N_SKIP, 0, 0));
    }
    continue;
  }
  }
  step_end:
    if (rr != GGR_STEP_CONT) {
      finished = true;
      result = rr;
      if (rr != GST_OK)
        res->err_pos = (((rr == GST_UNKNOWN_FIELD || rr == GST_DUPLICATE || rr == GST_ONEOF) && ekey != 0xFFFFFFFFu) ? ekey : r.pos) - start;
    }
   }
  }
  return result;
}

// --------------------------------------------------------------------------------------------
// pass B
// --------------------------------------------------------------------------------------------
template <class W>
GGR_DEV void copy_string(W& w, const u8* in, u32 quote_pos, u32 end, u32 dec_len, bool escapes) {
  if (!escapes) {
    Rd r;
    r.init(in, quote_pos + 1, end);
    u32 n = dec_len;
    while (n >= 4) {
      w.put(r.peek4(), 4);
      r.skip(4);
      n -= 4;
    }
    if (n) w.put(r.peek4() & (0xFFFFFFFFu >> (8 * (4 - n))), (int)n);
    return;
  }
  StrIter it;
  it.init(in, quote_pos, end);
  while (!it.eof()) {
    w.put1(it.peek());
    it.adv();
  }
}

template <class W>
GGR_DEV void encode_emit(const u8* in, u32 end, const u8* ir, u32 first, W& w, bool active = true,
                         unsigned mask = GGR_FULL_MASK) {
  u32 stk[GGR_MAX_DEPTH * 3];
  int sp = 0;
  u32 cur = first;
  bool finished = !active;
  // one step = one IR node; lanes re-converge at the vote after every step
  while (ggr_any(mask, !finished)) {
   if (!finished) {
    bool more = false;
  for (int once = 0;; once++) {
    if (once) { more = true; break; }
    if (cur == GGR_NIL) {
      if (sp == 0) break;
      cur = stk[--sp];
      continue;
    }
    U4 nd = node_load(ir, cur);
    u32 next = nd.z & 0xFFFFFu;
    u32 type = nd.w & 0xFu, flags = (nd.w >> 4) & 0xFu, tag = nd.w >> 8;
    switch (type) {
      case N_SKIP: break;
      case N_VARINT: {
        if (tag) put_varint(w, tag);
        u64 v = (u64)nd.x | ((u64)nd.y << 32);
        if (flags & NF_RAWKEY) {  // map key stored raw: apply the wire transform of its kind
          u32 kind = nd.z >> 20;
          if (kind == GK_SINT32) v = zigzag32((u32)v);
          else if (kind == GK_SINT64) v = zigzag64(v);
        }
        put_varint(w, v);
        break;
      }
      case N_FIX32:
        if (tag) put_varint(w, tag);
        w.put(nd.x, 4);
        break;
      case N_FIX64:
        if (tag) put_varint(w, tag);
        w.put(nd.x, 4);
        w.put(nd.y, 4);
        break;
      case N_STR:
        if (tag) put_varint(w, tag);
        put_varint(w, nd.y);
        copy_string(w, in, nd.x, end, nd.y, (flags & NF_ESC) != 0);
        break;
      case N_FMPATH: {  // tag 0x0A, the length after JSONSnakeCase, then the text with "_x" for every "X"
        u32 out_len = nd.y;
        for (u32 k = 0; k < nd.y; k++) out_len += (u32)in[nd.x + k] - 'A' < 26u ? 1u : 0u;
        w.put1(0x0Au);
        put_varint(w, out_len);
        for (u32 k = 0; k < nd.y; k++) {
          u32 c = in[nd.x + k];
          if (c - 'A' < 26u) {
            w.put1('_');
            c += 'a' - 'A';
          }
          w.put1(c);
        }
        break;
      }
      case N_BYTES: {
        if (tag) put_varint(w, tag);
        put_varint(w, nd.y);
        StrIter it;
        it.init(in, nd.x, end);
        u32 n;
        // b64_run only looks at total_len & 3 (padded vs raw mode)
        b64_run<true, W>(it, (flags & NF_URL) != 0, (flags & NF_PADDED) ? 0u : 1u, &w, &n);
        break;
      }
      case N_MSG:
      case N_ENTRY:
        if (tag) put_varint(w, tag);
        put_varint(w, nd.x);
        stk[sp++] = next;
        cur = nd.y;
        continue;
      case N_LIST:
        if (flags & NF_PACKED) {
          put_varint(w, tag);
          put_varint(w, nd.x);
        }
        stk[sp++] = next;
        cur = nd.y;
        continue;
      case N_MAP:
        stk[sp++] = next;
        cur = nd.y;
        continue;
    }
    cur = next;
  }
    if (!more) finished = true;
   }
  }
}
