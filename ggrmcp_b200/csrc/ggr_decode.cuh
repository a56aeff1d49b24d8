// ggr_decode.cuh - response side: protobuf wire bytes -> protojson text.
//
// Replaces, per item, proto.Unmarshal into a dynamicpb message (inside conn.Invoke) followed by
// protojson.Marshal (/root/reference/pkg/grpc/reflection.go:363,373,381).  JSON has no length
// prefixes, so the text streams out in one walk of the wire bytes; the walk runs twice with the
// same code - once over a counting writer to size the item, once over the real writer at the
// item's final offset.
//
//  fast walk : wire fields arrive in declaration order, singular fields once, repeated elements
//              contiguous (what every generated-code backend emits when declaration order ==
//              field-number order).  Map entries are put in key order on the fly.
//  slow walk : anything else (out-of-order fields, duplicates with last-wins, split repeated
//              fields): for each field in declaration order, scan the payload for its
//              occurrences.  The size pass detects the need and records it per item.
// Semantics restated from [upstream proto/decode.go unmarshalMessageSlow,
// encoding/protojson/encode.go, internal/encoding/json/encode.go, internal/order];
// oracle/orc_dyn.h + orc_protojson.h hold the line-by-line restatement the tests compare against.
#pragma once
#include "ggr_prim.cuh"
#include "ggr_json_in.cuh"
#include "ggr_float.cuh"

#define GGR_DEC_MAX_DEPTH 32
#ifndef GGR_RET
#define GGR_RET(x) do { rr = (x); goto step_end; } while (0)
#endif
#ifndef GGR_F_COMMA_SPACE
#define GGR_F_COMMA_SPACE 1u
#endif

#define GGR_MODE_FAST 0u
#define GGR_MODE_SLOW 1u
/* flag on FAST / SLOW: a large item the per-thread kernels take alone in a warp (list-mode launches, ggr_engine.cu) */
#define GGR_MODE_SPREAD 0x100u
#define GGR_NEED_SLOW 1000  /* internal: fast walk met an ordering it cannot stream */

struct DecResult {
  u32 size;
  u32 mode;
};

// ---- wire readers ----
GGR_DEV void rd_jump(Rd& r, u32 pos) {
  u32 e = r.end;
  r.init(r.base, pos, e, r.rw);
}
// protowire.ConsumeVarint bounded by `lim`
GGR_DEV bool rd_varint(Rd& r, u32 lim, u64* out) {
  u64 v = 0;
  for (int i = 0; i < 10; i++) {
    if (r.pos >= lim) return false;
    u32 c = r.peek();
    r.skip(1);
    if (i == 9 && c > 1) return false;
    v |= (u64)(c & 0x7F) << (7 * i);
    if (c < 0x80) {
      *out = v;
      return true;
    }
  }
  return false;
}
GGR_DEV bool rd_fixed32(Rd& r, u32 lim, u32* out) {
  if (lim - r.pos < 4 || r.pos > lim) return false;
  *out = r.peek4();
  r.skip(4);
  return true;
}
GGR_DEV bool rd_fixed64(Rd& r, u32 lim, u64* out) {
  u32 lo, hi;
  if (!rd_fixed32(r, lim, &lo) || !rd_fixed32(r, lim, &hi)) return false;
  *out = (u64)lo | ((u64)hi << 32);
  return true;
}
// skips the value of an unknown field (after its tag)
GGR_DEV bool rd_skip_value(Rd& r, u32 lim, u32 num, u32 wt) {
  u64 v;
  switch (wt) {
    case 0: return rd_varint(r, lim, &v);
    case 1: if (lim - r.pos < 8) return false; rd_jump(r, r.pos + 8); return true;
    case 5: if (lim - r.pos < 4) return false; r.skip(4); return true;
    case 2:
      if (!rd_varint(r, lim, &v) || v > (u64)(lim - r.pos)) return false;
      rd_jump(r, r.pos + (u32)v);
      return true;
    case 3: {
      u32 nums[8];
      int sp = 0;
      nums[sp++] = num;
      while (sp > 0) {
        u64 tag;
        if (!rd_varint(r, lim, &tag)) return false;
        u64 n2 = tag >> 3;
        u32 w2 = (u32)(tag & 7);
        if (n2 == 0 || n2 > 0x1FFFFFFFull) return false;
        if (w2 == 4) {
          if ((u32)n2 != nums[sp - 1]) return false;
          sp--;
        } else if (w2 == 3) {
          if (sp >= 8) return false;
          nums[sp++] = (u32)n2;
        } else if (!rd_skip_value(r, lim, (u32)n2, w2)) {
          return false;
        }
      }
      return true;
    }
    default: return false;
  }
}

GGR_DEV u32 ggr_ctz64(u64 x) {  // x != 0
  const u32 lo = (u32)x;
  return lo ? (u32)ggr_ctz32(lo) : 32u + (u32)ggr_ctz32((u32)(x >> 32));
}
// Eight bytes of the item at `pos` (two aligned 8-byte loads, the second one only inside the item's last 16-byte
// chunk): tag, length prefix and the first value bytes of a field decode from registers - one round trip to the
// memory system per field instead of one per varint (the tables in shared memory leave the L1 too small to hold
// the items, so every dependent byte load is an L2 access).
GGR_DEV u64 coop_window(const u8* in, u32 pos, u32 end_al) {
  const u32 a = pos & ~7u;
#if defined(__CUDA_ARCH__)
  const u64 lo = __ldg(reinterpret_cast<const unsigned long long*>(in + a));
  const u64 hi = a + 8u < end_al ? __ldg(reinterpret_cast<const unsigned long long*>(in + a + 8u)) : 0ull;
#else
  u64 lo, hi = 0;
  memcpy(&lo, in + a, 8);
  if (a + 8u < end_al) memcpy(&hi, in + a + 8u, 8);
#endif
  const u32 sh = (pos & 7u) * 8u;
  return sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
}
// A field header out of the window W at pos: tag (one or two bytes) and, by wire type, the extent of the value.
// Returns false when the bytes do not fit the window (long tags, lengths of three bytes and more, varints that run
// past it): the caller then decodes byte by byte.  On success: *tag, *body (payload start of a length-delimited
// value, else the value start), *vend, *zero (varint / fixed32 value is 0; length is 0) - bounds are the caller's.
GGR_DEV bool coop_header(u64 W, u32 pos, u32* tag, u32* tag_len, u32* body, u32* vend, bool* zero) {
  const u32 b0 = (u32)W & 0xFFu;
  u32 t = b0, tl = 1;
  if (b0 >= 0x80u) {
    const u32 b1 = (u32)(W >> 8) & 0xFFu;
    if (b1 >= 0x80u) return false;
    t = (b0 & 0x7Fu) | (b1 << 7);
    tl = 2;
  }
  *tag = t;
  *tag_len = tl;
  const u64 V = W >> (8u * tl);  // 6 or 7 value bytes
  const u32 wt = t & 7u;
  const u32 vpos = pos + tl;
  if (wt == 2u) {
    const u32 l0 = (u32)V & 0xFFu;
    u32 len = l0, ll = 1;
    if (l0 >= 0x80u) {
      const u32 l1 = (u32)(V >> 8) & 0xFFu;
      if (l1 >= 0x80u) return false;
      len = (l0 & 0x7Fu) | (l1 << 7);
      ll = 2;
    }
    *body = vpos + ll;
    *vend = vpos + ll + len;
    *zero = len == 0;
    return true;
  }
  *body = vpos;
  if (wt == 0u) {
    // first byte without the continuation bit among the bytes the window holds
    const u64 keep = tl == 1 ? 0x00FFFFFFFFFFFFFFull : 0x0000FFFFFFFFFFFFull;
    const u64 stop = ~V & 0x8080808080808080ull & keep;
    if (!stop) return false;
    const u32 k = (u32)(ggr_ctz64(stop) >> 3);  // index of the last byte of the varint
    *vend = vpos + k + 1u;
    const u64 bits = V & (0x7F7F7F7F7F7F7F7Full >> (8u * (7u - k)));
    *zero = bits == 0;
    return true;
  }
  if (wt == 5u) {
    *vend = vpos + 4u;
    *zero = (u32)V == 0u;
    return true;
  }
  return false;  // fixed64 (the value does not fit), groups, invalid wire types
}

// Slow walk: from `pos`, the position of the next top-level field header in [pos, end) that carries field `number`,
// or that the window decoder does not take (long tags and lengths, fixed64, groups, malformed bytes: the streaming
// reader decides those), or `end`.  The occurrences of the OTHER fields between them cost one 8-byte window each instead
// of a pass through the streaming reader (the slow walk scans the message once per declared field: a reply of 1 800
// occurrences and 12 fields is 21 600 such visits per pass).  Only for read-only input (not the merged scratch).
GGR_DEV u32 dec_skip_others(const u8* in, u32 pos, u32 end, u32 number) {
  const u32 end_al = (end + 15u) & ~15u;
  while (pos < end) {
    u32 tg = 0, tl = 0, body = 0, vend = 0;
    bool z = false;
    if (!coop_header(coop_window(in, pos, end_al), pos, &tg, &tl, &body, &vend, &z) || vend > end || body > end) break;
    const u32 num = tg >> 3;
    if (num == number || num == 0u) break;
    pos = vend;
  }
  return pos;
}

// ---- JSON writers ----
template <class W>
GGR_DEV void put_pool(W& w, const u8* pool, u32 off, u32 len) {
  Rd p;
  p.init(pool, off, off + len);
  while (len >= 4) {
    w.put(p.peek4(), 4);
    p.skip(4);
    len -= 4;
  }
  if (len) w.put(p.peek4() & (0xFFFFFFFFu >> (8 * (4 - len))), (int)len);
}
template <class W>
GGR_DEV void put_group8(W& w, u64 p, int k) {  // k digits, most significant in the lowest byte
  if (k > 4) {
    w.put((u32)p, 4);
    w.put((u32)(p >> 32) & (0xFFFFFFFFu >> (8 * (8 - k))), k - 4);
  } else if (k > 0) {
    w.put((u32)p & (0xFFFFFFFFu >> (8 * (4 - k))), k);
  }
}
template <class W>
GGR_DEV void put_dec_u64(W& w, u64 v) {
  u64 p0 = 0, p1 = 0, p2 = 0;
  int n = 0;
  if ((v >> 32) == 0) {
    u32 x = (u32)v;
    do {
      u32 q = x / 10u;
      u32 d = x - q * 10u;
      if (n < 8) p0 = (p0 << 8) | (u64)('0' + d);
      else p1 = (p1 << 8) | (u64)('0' + d);
      n++;
      x = q;
    } while (x);
  } else {
    do {
      u64 q = v / 10u;
      u32 d = (u32)(v - q * 10u);
      if (n < 8) p0 = (p0 << 8) | (u64)('0' + d);
      else if (n < 16) p1 = (p1 << 8) | (u64)('0' + d);
      else p2 = (p2 << 8) | (u64)('0' + d);
      n++;
      v = q;
    } while (v);
  }
  if (n > 16) put_group8(w, p2, n - 16);
  if (n > 8) put_group8(w, p1, n > 16 ? 8 : n - 8);
  put_group8(w, p0, n > 8 ? 8 : n);
}
template <class W>
GGR_DEV void put_dec_i64(W& w, i64 v) {
  if (v < 0) {
    w.put1('-');
    put_dec_u64(w, (u64)0 - (u64)v);
  } else {
    put_dec_u64(w, (u64)v);
  }
}
template <class W>
GGR_DEV void put_2d(W& w, u32 v) { w.put(('0' + v / 10) | (('0' + v % 10) << 8), 2); }

// protojson string: reader `r` positioned at the first payload byte, `len` bytes long.
// [upstream internal/encoding/json appendString]
template <class W>
GGR_DEV int put_json_string(W& w, Rd& r, u32 len) {
  u32 save_end = r.end;
  r.end = r.pos + len;
  w.put1('"');
  int st = GST_OK;
  for (;;) {
    while (r.left() >= 4) {
      u32 x = r.peek4();
      if (json_special_mask(x)) break;
      w.put(x, 4);
      r.skip(4);
    }
    if (r.eof()) break;
    u32 c = r.peek();
    if (c >= 0x80) {
      int k = utf8_seq_len(r);
      if (k == 0) {
        st = GST_INVALID_UTF8;
        break;
      }
      w.put(r.peek4() & (0xFFFFFFFFu >> (8 * (4 - k))), k);
      r.skip(k);
      continue;
    }
    if (c >= 0x20 && c != '"' && c != '\\') {
      w.put1(c);
      r.skip(1);
      continue;
    }
    u32 e;
    switch (c) {
      case '"': e = '"'; break;
      case '\\': e = '\\'; break;
      case 8: e = 'b'; break;
      case 12: e = 'f'; break;
      case 10: e = 'n'; break;
      case 13: e = 'r'; break;
      case 9: e = 't'; break;
      default: e = 0; break;
    }
    if (e) {
      w.put('\\' | (e << 8), 2);
    } else {
      u32 hi = c >> 4, lo = c & 15;
      w.put(LIT4('\\', 'u', '0', '0'), 4);
      w.put(('0' + hi) | ((lo < 10 ? '0' + lo : 'a' + lo - 10) << 8), 2);
    }
    r.skip(1);
  }
  w.put1('"');
  if (st != GST_OK) rd_jump(r, r.end);
  r.end = save_end;
  return st;
}

GGR_DEV u32 b64_char(u32 v) {
  return v + 65u + (v >= 26u ? 6u : 0u) - (v >= 52u ? 75u : 0u) - (v >= 62u ? 15u : 0u) + (v >= 63u ? 3u : 0u);
}
template <class W>
GGR_DEV void put_base64(W& w, Rd& r, u32 len) {
  w.put1('"');
  while (len >= 3) {
    u32 x = r.peek4();
    u32 v = ((x & 0xFF) << 16) | (x & 0xFF00) | ((x >> 16) & 0xFF);
    w.put(b64_char(v >> 18) | (b64_char((v >> 12) & 63) << 8) | (b64_char((v >> 6) & 63) << 16) | (b64_char(v & 63) << 24), 4);
    r.skip(3);
    len -= 3;
  }
  if (len == 1) {
    u32 v = (r.peek() & 0xFF) << 16;
    w.put(b64_char(v >> 18) | (b64_char((v >> 12) & 63) << 8) | ('=' << 16) | ('=' << 24), 4);
    r.skip(1);
  } else if (len == 2) {
    u32 x = r.peek4();
    u32 v = ((x & 0xFF) << 16) | (x & 0xFF00);
    w.put(b64_char(v >> 18) | (b64_char((v >> 12) & 63) << 8) | (b64_char((v >> 6) & 63) << 16) | ('=' << 24), 4);
    r.skip(2);
  }
  w.put1('"');
}

// google.protobuf.Timestamp -> "YYYY-MM-DDTHH:MM:SS[.fff[fff[fff]]]Z" [upstream marshalTimestamp]
template <class W>
GGR_DEV int put_timestamp(W& w, i64 secs, i64 nanos) {
  if (secs < -62135596800ll || secs > 253402300799ll) return GST_RANGE;
  if (nanos < 0 || nanos > 999999999ll) return GST_RANGE;  // upstream: nanos > secondsInNanos (999999999)
  i64 days = secs / 86400, rem = secs % 86400;
  if (rem < 0) {
    rem += 86400;
    days--;
  }
  // civil_from_days
  i64 z = days + 719468;
  i64 era = (z >= 0 ? z : z - 146096) / 146097;
  u32 doe = (u32)(z - era * 146097);
  u32 yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  i64 y = (i64)yoe + era * 400;
  u32 doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  u32 mp = (5 * doy + 2) / 153;
  u32 d = doy - (153 * mp + 2) / 5 + 1;
  u32 m = mp < 10 ? mp + 3 : mp - 9;
  y += m <= 2;
  u32 yy = (u32)y;  // 1..9999 (range-checked above); the year 10000 cannot occur
  w.put1('"');
  put_2d(w, yy / 100);
  put_2d(w, yy % 100);
  w.put1('-');
  put_2d(w, m);
  w.put1('-');
  put_2d(w, d);
  w.put1('T');
  u32 sod = (u32)rem;
  put_2d(w, sod / 3600);
  w.put1(':');
  put_2d(w, sod % 3600 / 60);
  w.put1(':');
  put_2d(w, sod % 60);
  u32 ns = (u32)nanos;
  if (ns != 0) {
    w.put1('.');
    u32 a = ns / 1000000, b = ns / 1000 % 1000, c = ns % 1000;
    w.put(('0' + a / 100) | (('0' + a / 10 % 10) << 8) | (('0' + a % 10) << 16), 3);
    if (b != 0 || c != 0) {
      w.put(('0' + b / 100) | (('0' + b / 10 % 10) << 8) | (('0' + b % 10) << 16), 3);
      if (c != 0) w.put(('0' + c / 100) | (('0' + c / 10 % 10) << 8) | (('0' + c % 10) << 16), 3);
    }
  }
  w.put('Z' | ('"' << 8), 2);
  return GST_OK;
}

// google.protobuf.Duration -> "[-]S[.fff[fff[fff]]]s" [upstream marshalDuration]
template <class W>
GGR_DEV int put_duration(W& w, i64 secs, i64 nanos) {
  if (secs < -315576000000ll || secs > 315576000000ll) return GST_RANGE;
  if (nanos < -999999999ll || nanos > 999999999ll) return GST_RANGE;
  if ((secs > 0 && nanos < 0) || (secs < 0 && nanos > 0)) return GST_RANGE;  // signs of seconds and nanos do not match
  w.put1('"');
  if (secs < 0 || nanos < 0) {
    w.put1('-');
    secs = -secs;
    nanos = -nanos;
  }
  put_dec_u64(w, (u64)secs);
  u32 ns = (u32)nanos;
  if (ns != 0) {
    w.put1('.');
    u32 a = ns / 1000000, b = ns / 1000 % 1000, c = ns % 1000;
    w.put(('0' + a / 100) | (('0' + a / 10 % 10) << 8) | (('0' + a % 10) << 16), 3);
    if (b != 0 || c != 0) {
      w.put(('0' + b / 100) | (('0' + b / 10 % 10) << 8) | (('0' + b % 10) << 16), 3);
      if (c != 0) w.put(('0' + c / 100) | (('0' + c / 10 % 10) << 8) | (('0' + c % 10) << 16), 3);
    }
  }
  w.put('s' | ('"' << 8), 2);
  return GST_OK;
}

struct DecCtx {
  Tables T;
  const u8* in;
  u32 flags;
  // scratch for maps whose entries arrive unsorted (what a Go backend sends: map iteration order): 16-byte
  // (key, position) records handed out by a bump counter; nullptr: selection by repeated scans (quadratic)
  U4* sort_pool = nullptr;
  u32* sort_ctr = nullptr;
  u32 sort_cap = 0;
  // 1: `in` is scratch this thread wrote (the merged payload of a split sub-message): plain loads
  u32 rw = 0;
  // errors protojson.Marshal raises (Timestamp / Duration out of range) are parked here while the walk goes on:
  // proto.Unmarshal has read the whole item by then, so any wire error anywhere in the item comes first
  int* late = nullptr;
};

template <class W>
GGR_DEV void put_sep(W& w, const DecCtx& cx, u32& first) {
  if (!first) {
    w.put1(',');
    if (cx.flags & GGR_F_COMMA_SPACE) w.put1(' ');
  }
  first = 0;
}

// field lookup by number; returns emit index or -1
GGR_DEV i32 find_field(const Tables& T, const MsgD& md, u32 num) {
  if (num < md.lut_n) return (i32)ggr_u16(T, md.lut_first + num) - 1;
  for (u32 i = 0; i < md.n_fields; i++) {
    U4 a = ggr_ld16(T.fields + (size_t)(md.field_first + i) * 32);
    if (a.x == num) return (i32)i;
  }
  return -1;
}

// Reads a google.protobuf.Timestamp payload [r.pos, lim): last value wins, unknown fields skipped.
GGR_DEV int read_timestamp_payload(Rd& r, u32 lim, i64* secs, i64* nanos) {
  *secs = 0;
  *nanos = 0;
  while (r.pos < lim) {
    u64 tag, v;
    if (!rd_varint(r, lim, &tag)) return GST_BAD_WIRE;
    u64 num = tag >> 3;
    u32 wt = (u32)(tag & 7);
    if (num == 0 || num > 0x1FFFFFFFull || wt == 4) return GST_BAD_WIRE;
    if (num == 1 && wt == 0) {
      if (!rd_varint(r, lim, &v)) return GST_BAD_WIRE;
      *secs = (i64)v;
    } else if (num == 2 && wt == 0) {
      if (!rd_varint(r, lim, &v)) return GST_BAD_WIRE;
      *nanos = (i64)(i32)(u32)v;
    } else if (!rd_skip_value(r, lim, (u32)num, wt)) {
      return GST_BAD_WIRE;
    }
  }
  return r.pos == lim ? GST_OK : GST_BAD_WIRE;
}

// One scalar (non-message) value of field f read at r and written as JSON.
// *zero is set when the value is the zero value of its kind (implicit-presence elision).
// With EMIT=false the value is only read (and validated).
template <class W, bool EMIT>
GGR_DEV int scalar_value(W& w, const DecCtx& cx, Rd& r, u32 lim, u32 kind, i32 child, bool quoted_key, bool* zero) {
  u64 v = 0;
  switch (kind) {
    case GK_INT32: case GK_INT64: case GK_UINT32: case GK_UINT64: case GK_SINT32: case GK_SINT64: case GK_BOOL: case GK_ENUM:
      if (!rd_varint(r, lim, &v)) return GST_BAD_WIRE;
      break;
    case GK_FIXED32: case GK_SFIXED32: case GK_FLOAT: {
      u32 x;
      if (!rd_fixed32(r, lim, &x)) return GST_BAD_WIRE;
      v = x;
      break;
    }
    case GK_FIXED64: case GK_SFIXED64: case GK_DOUBLE:
      if (!rd_fixed64(r, lim, &v)) return GST_BAD_WIRE;
      break;
    case GK_STRING: case GK_BYTES: {
      u64 len;
      if (!rd_varint(r, lim, &len) || len > (u64)(lim - r.pos)) return GST_BAD_WIRE;
      *zero = len == 0;
      if (kind == GK_STRING) {
        // validation happens even for elided/unwritten strings (proto.Unmarshal rejects bad UTF-8)
        if (EMIT) return put_json_string(w, r, (u32)len);
        Cnt c;
        c.pos = 0;
        return put_json_string(c, r, (u32)len);
      }
      if (EMIT) put_base64(w, r, (u32)len);
      else rd_jump(r, r.pos + (u32)len);
      return GST_OK;
    }
    default: return GST_UNSUPPORTED;
  }
  i64 sv = 0;
  bool is_signed = false, is64 = false;
  switch (kind) {
    case GK_INT32: case GK_ENUM: sv = (i64)(i32)(u32)v; is_signed = true; break;
    case GK_SINT32: { u32 x = (u32)v; sv = (i64)(i32)((x >> 1) ^ (0u - (x & 1))); is_signed = true; break; }
    case GK_SFIXED32: sv = (i64)(i32)(u32)v; is_signed = true; break;
    case GK_UINT32: case GK_FIXED32: v = (u32)v; break;
    case GK_INT64: case GK_SFIXED64: sv = (i64)v; is_signed = true; is64 = true; break;
    case GK_SINT64: sv = (i64)((v >> 1) ^ (0ull - (v & 1))); is_signed = true; is64 = true; break;
    case GK_UINT64: case GK_FIXED64: is64 = true; break;
    case GK_BOOL: v = v != 0; break;
    case GK_FLOAT: case GK_DOUBLE:
      *zero = v == 0;  // bit pattern: -0.0 is set (dynamicpb isSet)
      if (EMIT) put_float_go(w, v, kind == GK_FLOAT);
      return GST_OK;
    default: break;
  }
  *zero = is_signed ? sv == 0 : v == 0;
  if (!EMIT) return GST_OK;
  if (kind == GK_BOOL) {
    if (quoted_key) w.put1('"');
    if (v) w.put(LIT4('t', 'r', 'u', 'e'), 4);
    else {
      w.put(LIT4('f', 'a', 'l', 's'), 4);
      w.put1('e');
    }
    if (quoted_key) w.put1('"');
    return GST_OK;
  }
  if (kind == GK_ENUM) {
    // protoreflect EnumValueDescriptors.ByNumber: binary search over the distinct numbers
    U4 e = ggr_ld16(cx.T.enums + (size_t)child * 16);
    u32 lo = 0, hi = e.y;
    while (lo < hi) {
      u32 mid = (lo + hi) >> 1;
      U4 ev = ggr_ld16(cx.T.evals + (size_t)(e.x + mid) * 16);
      i32 num = (i32)ev.x;
      if (num == (i32)sv) {
        w.put1('"');
        put_pool(w, cx.T.pool, ev.y, ev.z);
        w.put1('"');
        return GST_OK;
      }
      if (num < (i32)sv) lo = mid + 1;
      else hi = mid;
    }
    put_dec_i64(w, sv);
    return GST_OK;
  }
  bool q = is64 || quoted_key;
  if (q) w.put1('"');
  if (is_signed) put_dec_i64(w, sv);
  else put_dec_u64(w, v);
  if (q) w.put1('"');
  return GST_OK;
}

// scalar_value as a call (the per-thread walkers have a dozen call sites; inlined, each one is 6-8 thousand
// instructions): reads at `pos` with a reader of its own and returns the position after the value in the low 31 bits
// of *next, the "zero value" flag in bit 31.  The caller jumps its reader there.
template <class W, bool EMIT>
GGR_DEVN int scalar_value_at(W& w, const DecCtx& cx, u32 pos, u32 lim, u32 kind, i32 child, u32* next) {
  Rd r;
  r.init(cx.in, pos, lim, cx.rw);
  bool z = false;
  const int st = scalar_value<W, EMIT>(w, cx, r, lim, kind, child, false, &z);
  *next = r.pos | (z ? 0x80000000u : 0u);
  return st;
}

// ---- split sub-messages (proto.Unmarshal merges, reflection.go:363) ----
// A singular message field that occurs more than once on the wire is parsed occurrence after occurrence into the
// same message: scalars last-wins, repeated fields append, sub-messages merge again.  That is what parsing the
// concatenation of the payloads gives, once every occurrence is well-formed on its own (checked here, because a
// truncated occurrence must not borrow bytes from the next one).  The concatenation lives in the scratch pool.
GGR_DEV u8* dec_scratch(const DecCtx& cx, u32 bytes) {
  if (!cx.sort_pool) return nullptr;
  const u32 units = (bytes + 15u) / 16u + 1u;  // the readers fetch whole 16-byte chunks
  const u32 base = ggr_atomic_add_u32(cx.sort_ctr, units);
  if (base > cx.sort_cap || units > cx.sort_cap - base) return nullptr;
  return reinterpret_cast<u8*>(cx.sort_pool + base);
}
// payloads of all length-delimited occurrences of field `num` among the top-level fields of cx.in[start, end)
GGR_DEVN int merge_occurrences(const DecCtx& cx, u32 start, u32 end, u32 num, const u8** out, u32* out_len) {
  u8* dst = nullptr;
  u32 total = 0;
  for (int pass = 0; pass < 2; pass++) {
    Rd t;
    t.init(cx.in, start, end, cx.rw);
    u32 at = 0;
    while (t.pos < end) {
      u64 tag;
      if (!rd_varint(t, end, &tag)) return GST_BAD_WIRE;
      const u64 n2 = tag >> 3;
      const u32 wt = (u32)(tag & 7);
      if (n2 == 0 || n2 > 0x1FFFFFFFull || wt == 4 || wt > 5) return GST_BAD_WIRE;
      if ((u32)n2 != num || wt != 2) {
        if (!rd_skip_value(t, end, (u32)n2, wt)) return GST_BAD_WIRE;
        continue;
      }
      u64 len;
      if (!rd_varint(t, end, &len) || len > (u64)(end - t.pos)) return GST_BAD_WIRE;
      const u32 lim = t.pos + (u32)len;
      if (pass == 0) {
        total += (u32)len;
        while (t.pos < lim) {  // the occurrence on its own
          u64 tg;
          if (!rd_varint(t, lim, &tg)) return GST_BAD_WIRE;
          const u64 n3 = tg >> 3;
          const u32 w3 = (u32)(tg & 7);
          if (n3 == 0 || n3 > 0x1FFFFFFFull || w3 == 4 || w3 > 5) return GST_BAD_WIRE;
          if (!rd_skip_value(t, lim, (u32)n3, w3)) return GST_BAD_WIRE;
        }
        if (t.pos != lim) return GST_BAD_WIRE;
      } else {
        for (u32 p = t.pos; p < lim; p++) dst[at++] = cx.in[p];
        rd_jump(t, lim);
      }
    }
    if (pass == 0) {
      dst = dec_scratch(cx, total);
      if (!dst) return GST_UNSUPPORTED;  // no pool (or exhausted): never a different answer
    }
  }
  *out = dst;
  *out_len = total;
  return GST_OK;
}

// ---- map entries ----
struct MapEnt {
  u64 key;      // numeric key / (pos | len << 32) of a string key's payload
  u32 val_pos;  // position of the value's payload-or-varint start (after its tag); 0 = absent
  u32 val_len;  // for LEN values: payload length
  u32 end;      // end of the entry payload
  u32 beg;      // start of the entry payload
  u32 multi;    // message value split over several occurrences inside the entry: merged when written
  u32 dup;      // a string key or a string value occurs more than once inside the entry: the earlier ones are never written
};
// Parses one map entry payload [r.pos, lim): key (field 1) and value (field 2), last wins.
GGR_DEV int parse_map_entry(Rd& r, u32 lim, const FieldD& kf, const FieldD& vf, MapEnt* me) {
  me->key = 0;
  me->val_pos = 0;
  me->val_len = 0;
  me->end = lim;
  me->beg = r.pos;
  me->multi = 0;
  me->dup = 0;
  bool str_key = kf.kind == GK_STRING;
  if (str_key) me->key = (u64)r.pos;  // empty string key: len 0 at any position
  u32 val_seen = 0, key_seen = 0;
  while (r.pos < lim) {
    u64 tag, v;
    if (!rd_varint(r, lim, &tag)) return GST_BAD_WIRE;
    u64 num = tag >> 3;
    u32 wt = (u32)(tag & 7);
    if (num == 0 || num > 0x1FFFFFFFull || wt == 4) return GST_BAD_WIRE;
    if (num == 1 && wt == kf.wt) {
      if (str_key) {
        if (!rd_varint(r, lim, &v) || v > (u64)(lim - r.pos)) return GST_BAD_WIRE;
        if (key_seen) me->dup = 1;
        key_seen = 1;
        me->key = (u64)r.pos | (v << 32);
        rd_jump(r, r.pos + (u32)v);
      } else if (wt == 0) {
        if (!rd_varint(r, lim, &v)) return GST_BAD_WIRE;
        switch (kf.kind) {
          case GK_INT32: v = (u64)(i64)(i32)(u32)v; break;
          case GK_SINT32: { u32 x = (u32)v; v = (u64)(i64)(i32)((x >> 1) ^ (0u - (x & 1))); break; }
          case GK_SINT64: v = (v >> 1) ^ (0ull - (v & 1)); break;
          case GK_UINT32: v = (u32)v; break;
          case GK_BOOL: v = v != 0; break;
          default: break;
        }
        me->key = v;
      } else if (wt == 5) {
        u32 x;
        if (!rd_fixed32(r, lim, &x)) return GST_BAD_WIRE;
        me->key = kf.kind == GK_SFIXED32 ? (u64)(i64)(i32)x : (u64)x;
      } else {
        if (!rd_fixed64(r, lim, &me->key)) return GST_BAD_WIRE;
      }
    } else if (num == 2 && wt == vf.wt) {
      if (vf.kind == GK_MESSAGE && val_seen) me->multi = 1;  // split value: put_map_value merges
      if (vf.kind == GK_STRING && val_seen) me->dup = 1;
      val_seen = 1;
      me->val_pos = r.pos;
      if (wt == 2) {
        if (!rd_varint(r, lim, &v) || v > (u64)(lim - r.pos)) return GST_BAD_WIRE;
        me->val_pos = r.pos;
        me->val_len = (u32)v;
        rd_jump(r, r.pos + (u32)v);
      } else if (!rd_skip_value(r, lim, 2, wt)) {
        return GST_BAD_WIRE;
      }
    } else if (!rd_skip_value(r, lim, (u32)num, wt)) {
      return GST_BAD_WIRE;
    }
  }
  return r.pos == lim ? GST_OK : GST_BAD_WIRE;
}
// order.GenericKeyOrder: bool false<true, signed/unsigned numeric, strings bytewise
GGR_DEV int cmp_map_keys(const DecCtx& cx, u32 kkind, u64 a, u64 b) {
  if (kkind == GK_STRING) {
    u32 la = (u32)(a >> 32), lb = (u32)(b >> 32);
    Rd ra, rb;
    ra.init(cx.in, (u32)a, (u32)a + la, cx.rw);
    rb.init(cx.in, (u32)b, (u32)b + lb, cx.rw);
    u32 n = la < lb ? la : lb;
    while (n >= 4) {
      u32 x = ra.peek4(), y = rb.peek4();
      if (x != y) {
        // first differing byte decides (little-endian: lowest differing byte)
        u32 d = x ^ y;
        int sh = ggr_ctz32(d) & ~7;
        u32 bx = (x >> sh) & 0xFF, by = (y >> sh) & 0xFF;
        return bx < by ? -1 : 1;
      }
      ra.skip(4);
      rb.skip(4);
      n -= 4;
    }
    while (n > 0) {
      u32 x = ra.peek(), y = rb.peek();
      if (x != y) return x < y ? -1 : 1;
      ra.skip(1);
      rb.skip(1);
      n--;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
  }
  bool uns = kkind == GK_UINT32 || kkind == GK_UINT64 || kkind == GK_FIXED32 || kkind == GK_FIXED64 || kkind == GK_BOOL;
  if (uns) return a < b ? -1 : (a > b ? 1 : 0);
  return (i64)a < (i64)b ? -1 : ((i64)a > (i64)b ? 1 : 0);
}

template <class W>
GGR_DEVN int put_map_key(W& w, const DecCtx& cx, u32 kkind, u64 key) {
  if (kkind == GK_STRING) {
    Rd r;
    r.init(cx.in, (u32)key, (u32)key + (u32)(key >> 32), cx.rw);
    return put_json_string(w, r, (u32)(key >> 32));
  }
  w.put1('"');
  if (kkind == GK_BOOL) {
    if (key) w.put(LIT4('t', 'r', 'u', 'e'), 4);
    else {
      w.put(LIT4('f', 'a', 'l', 's'), 4);
      w.put1('e');
    }
  } else {
    bool uns = kkind == GK_UINT32 || kkind == GK_UINT64 || kkind == GK_FIXED32 || kkind == GK_FIXED64;
    if (uns) put_dec_u64(w, key);
    else put_dec_i64(w, (i64)key);
  }
  w.put1('"');
  return GST_OK;
}

struct DFrame {
  u32 end;        // payload end
  u32 msg;        // message index
  i32 last_decl;  // declaration index of the last field seen (fast) / cursor (slow)
  u32 open;       // fast: emit index + 1 of the repeated field whose '[' is open
  u32 first;      // nothing written yet inside this object
  u32 elem_first; // nothing written yet inside the open array
  u32 oneofs;     // oneofs already written
  // slow walk state
  u32 start;      // payload start
  u32 scan;       // resume position of the current field's occurrence scan
  u32 cur_emit;   // emit index of the field being scanned
  u32 state;      // slow: 0 = advance to next field, 1 = inside repeated occurrences
  const u8* base; // slow: the buffer the positions refer to (the input, or the merged payload of a split sub-message)
};

// Emits all entries of map field `f` found as a contiguous run of tags starting at r.pos
// (fast walk) or anywhere in [scan_from, lim) (slow walk, contiguous=false).  Entries come out
// in key order with last-wins on duplicate keys.  Message-valued entries are handled by
// returning to the caller one at a time: see walk loops.
//
// To keep the walkers simple, message-valued map entries are written through a nested call of
// the walker entry point for the value payload (depth-bounded); scalars are written here.
#define GGR_DEC_MAX_REC 3 /* message-valued map entries nest by (bounded) recursion */
template <class W, bool SLOW>
GGR_DEVN int walk_message(W& w, const DecCtx& cx, u32 msg, u32 start, u32 end, int rec, bool active, unsigned mask);

// Value of a scalar field that may be absent (map values, wrapper values): its text, or the text of the kind's zero
// value when me.val_pos == 0.
template <class W>
GGR_DEV int put_scalar_or_default(W& w, const DecCtx& cx, const FieldD& vf, const MapEnt& me) {
  if (!me.val_pos) {
    // absent value: zero value of the kind
    switch (vf.kind) {
      case GK_STRING: case GK_BYTES: w.put('"' | ('"' << 8), 2); return GST_OK;
      case GK_BOOL: w.put(LIT4('f', 'a', 'l', 's'), 4); w.put1('e'); return GST_OK;
      case GK_INT64: case GK_UINT64: case GK_SINT64: case GK_FIXED64: case GK_SFIXED64: w.put('"' | ('0' << 8) | ('"' << 16), 3); return GST_OK;
      case GK_FLOAT: case GK_DOUBLE: w.put1('0'); return GST_OK;
      case GK_ENUM: break;  // name of number 0 or the number itself: fall through to the generic writer
      default: w.put1('0'); return GST_OK;
    }
    if (vf.kind == GK_ENUM) {
      // run the generic writer over a synthetic zero varint: simplest is the name lookup inline
      U4 e = ggr_ld16(cx.T.enums + (size_t)vf.child * 16);
      u32 lo = 0, hi = e.y;
      while (lo < hi) {
        u32 mid = (lo + hi) >> 1;
        U4 ev = ggr_ld16(cx.T.evals + (size_t)(e.x + mid) * 16);
        if ((i32)ev.x == 0) {
          w.put1('"');
          put_pool(w, cx.T.pool, ev.y, ev.z);
          w.put1('"');
          return GST_OK;
        }
        if ((i32)ev.x < 0) lo = mid + 1;
        else hi = mid;
      }
      w.put1('0');
      return GST_OK;
    }
  }
  Rd r;
  u32 lim = me.end;
  r.init(cx.in, me.val_pos, lim, cx.rw);
  if (vf.wt == 2) {
    // scalar_value re-reads the length prefix: step back is not possible, so emit directly
    if (vf.kind == GK_STRING) return put_json_string(w, r, me.val_len);
    put_base64(w, r, me.val_len);
    return GST_OK;
  }
  bool z;
  return scalar_value<W, true>(w, cx, r, lim, vf.kind, vf.child, false, &z);
}

// Payload [r.pos, lim) of a wrapper message (google.protobuf.*Value): the last occurrence of field 1 wins, every
// string occurrence is checked the way proto.Unmarshal checks it.
GGR_DEV int parse_wrapper(const DecCtx& cx, Rd& r, u32 lim, const FieldD& vf, MapEnt* me) {
  me->key = 0;
  me->val_pos = 0;
  me->val_len = 0;
  me->end = lim;
  me->beg = r.pos;
  me->multi = 0;
  while (r.pos < lim) {
    u64 tag, v;
    if (!rd_varint(r, lim, &tag)) return GST_BAD_WIRE;
    u64 num = tag >> 3;
    u32 wt = (u32)(tag & 7);
    if (num == 0 || num > 0x1FFFFFFFull || wt == 4) return GST_BAD_WIRE;
    if (num == 1 && wt == vf.wt) {
      me->val_pos = r.pos;
      if (wt == 2) {
        if (!rd_varint(r, lim, &v) || v > (u64)(lim - r.pos)) return GST_BAD_WIRE;
        me->val_pos = r.pos;
        me->val_len = (u32)v;
        if (vf.kind == GK_STRING) {
          Cnt c;
          c.pos = 0;
          int st = put_json_string(c, r, (u32)v);
          if (st != GST_OK) return st;
        } else {
          rd_jump(r, r.pos + (u32)v);
        }
      } else if (!rd_skip_value(r, lim, 1, wt)) {
        return GST_BAD_WIRE;
      }
    } else if (!rd_skip_value(r, lim, (u32)num, wt)) {
      return GST_BAD_WIRE;
    }
  }
  return r.pos == lim ? GST_OK : GST_BAD_WIRE;
}

// A well-known type with a JSON form of its own, payload [r.pos, lim) (protojson well_known_types.go): Timestamp,
// Duration, the nine wrappers (the bare value, its zero when unset), Empty.
// Called, not inlined (a dozen call sites in the walkers): it reads the payload with a reader of its own, the caller
// jumps to `lim` afterwards.
template <class W>
GGR_DEVN int put_wkt(W& w, const DecCtx& cx, u32 msg, u32 start, u32 lim) {
  const MsgD cd = ggr_msg(cx.T, msg);
  Rd r;
  r.init(cx.in, start, lim, cx.rw);
  if (cd.wkt == GGR_WKT_TIMESTAMP || cd.wkt == GGR_WKT_DURATION) {
    i64 s, n;
    int st = read_timestamp_payload(r, lim, &s, &n);
    if (st != GST_OK) return st;
    st = cd.wkt == GGR_WKT_TIMESTAMP ? put_timestamp(w, s, n) : put_duration(w, s, n);
    if (st == GST_RANGE && cx.late) {
      if (*cx.late == GST_OK) *cx.late = GST_RANGE;  // Marshal stops at its first error: the first one parked stays
      return GST_OK;
    }
    return st;
  }
  if (cd.wkt == GGR_WKT_WRAPPER) {
    const FieldD vf = ggr_field(cx.T, cd.field_first);
    MapEnt me;
    int st = parse_wrapper(cx, r, lim, vf, &me);
    if (st != GST_OK) return st;
    return put_scalar_or_default(w, cx, vf, me);
  }
  if (cd.wkt == GGR_WKT_FIELDMASK) {
    // [upstream marshalFieldMask] the paths camelCase, joined with ','.  A path that is not a dotted name, or that does
    // not survive camelCase -> snake_case (upper-case letters, '_' not followed by a lower-case letter), is an error
    // of Marshal: parked like the range errors.  proto.Unmarshal has checked every path's UTF-8 before.
    w.put1('"');
    u32 first = 1;
    bool bad = false;
    while (r.pos < lim) {
      u64 tag, len;
      if (!rd_varint(r, lim, &tag)) return GST_BAD_WIRE;
      u64 num = tag >> 3;
      u32 wt = (u32)(tag & 7);
      if (num == 0 || num > 0x1FFFFFFFull || wt == 4) return GST_BAD_WIRE;
      if (num != 1 || wt != 2) {
        if (!rd_skip_value(r, lim, (u32)num, wt)) return GST_BAD_WIRE;
        continue;
      }
      if (!rd_varint(r, lim, &len) || len > (u64)(lim - r.pos)) return GST_BAD_WIRE;
      if (!first) w.put1(',');
      first = 0;
      bool seg_start = true, under = false;
      for (u32 k = 0; k < (u32)len; k++) {
        u32 c = r.peek();
        r.skip(1);
        if (c >= 0x80u) {  // not a name character; is it at least UTF-8?  (proto.Unmarshal's check comes first)
          Rd v;
          v.init(cx.in, r.pos - 1u, lim, cx.rw);
          Cnt cn;
          cn.pos = 0;
          int st = put_json_string(cn, v, (u32)len - k);
          if (st != GST_OK) return st;
          bad = true;
          rd_jump(r, r.pos - 1u + ((u32)len - k));
          break;
        }
        const bool upper = c - 'A' < 26u, lower = c - 'a' < 26u, digit = c - '0' < 10u;
        if (c == '.') {
          if (seg_start || under) bad = true;
          seg_start = true;
          under = false;
          w.put1(c);
          continue;
        }
        if (upper || !(lower || c == '_' || (digit && !seg_start))) bad = true;
        if (under && !lower) bad = true;  // '_' must be followed by a lower-case letter to come back from camelCase
        seg_start = false;
        if (c == '_') {
          under = true;
          continue;
        }
        w.put1(under ? c - ('a' - 'A') : c);
        under = false;
      }
      if (seg_start || under) bad = true;  // empty path, trailing '.', trailing '_'
    }
    if (r.pos != lim) return GST_BAD_WIRE;
    w.put1('"');
    if (bad) {
      if (cx.late) {
        if (*cx.late == GST_OK) *cx.late = GST_INVALID_VALUE;
        return GST_OK;
      }
      return GST_INVALID_VALUE;
    }
    return GST_OK;
  }
  if (cd.wkt == GGR_WKT_EMPTY) {
    while (r.pos < lim) {
      u64 tag;
      if (!rd_varint(r, lim, &tag)) return GST_BAD_WIRE;
      u64 num = tag >> 3;
      u32 wt = (u32)(tag & 7);
      if (num == 0 || num > 0x1FFFFFFFull || wt == 4) return GST_BAD_WIRE;
      if (!rd_skip_value(r, lim, (u32)num, wt)) return GST_BAD_WIRE;
    }
    if (r.pos != lim) return GST_BAD_WIRE;
    w.put('{' | ('}' << 8), 2);
    return GST_OK;
  }
  return GST_UNSUPPORTED;
}

template <class W, bool SLOW>
GGR_DEVN int put_map_value(W& w, const DecCtx& cx, FieldD vf, MapEnt me, int rec) {
  if (vf.kind == GK_MESSAGE && me.multi) {
    if (!SLOW) return GGR_NEED_SLOW;
    MsgD vd = ggr_msg(cx.T, (u32)vf.child);
    if (vd.wkt == GGR_WKT_UNSUPPORTED) return GST_UNSUPPORTED;
    DecCtx mc = cx;
    const u8* mb;
    u32 ml;
    int st = merge_occurrences(cx, me.beg, me.end, 2, &mb, &ml);
    if (st != GST_OK) return st;
    mc.in = mb;
    mc.rw = 1;
    return walk_message<W, SLOW>(w, mc, (u32)vf.child, 0, ml, rec + 1, true, ggr_activemask());
  }
  if (vf.kind == GK_MESSAGE) {
    MsgD vd = ggr_msg(cx.T, (u32)vf.child);
    if (vd.wkt != GGR_WKT_NONE) {
      // an absent value is the empty message
      const u32 vs = me.val_pos ? me.val_pos : me.end, ve = me.val_pos ? me.val_pos + me.val_len : me.end;
      return put_wkt(w, cx, (u32)vf.child, vs, ve);
    }
    if (!me.val_pos) {
      w.put('{' | ('}' << 8), 2);
      return GST_OK;
    }
    // nested walk: only the lanes that arrive here together vote with each other
    return walk_message<W, SLOW>(w, cx, (u32)vf.child, me.val_pos, me.val_pos + me.val_len, rec + 1, true, ggr_activemask());
  }
  return put_scalar_or_default(w, cx, vf, me);
}

// proto.Unmarshal parses every occurrence, also the ones that never reach the text: a map entry whose key comes again
// later (last wins), an earlier key or string value inside one entry.  Invalid UTF-8 or a malformed message in such a
// place fails the item in Go; the writers only see what they write.  These two checks run in the SIZE pass (the pass that
// decides an item's status) exactly where an occurrence is dropped.
template <class W> struct IsCountingWriter { static const bool v = false; };
template <> struct IsCountingWriter<Cnt> { static const bool v = true; };
// the value of an entry that a later entry with the same key replaces: walked into a counter; what Marshal would have said
// about it (ranges, field masks) does not count - Marshal never sees it
template <bool SLOW>
GGR_DEVN int check_shadowed_value(const DecCtx& cx, FieldD vf, MapEnt me, int rec) {
  if (vf.kind != GK_STRING && vf.kind != GK_MESSAGE) return GST_OK;
  Cnt c;
  c.pos = 0;
  DecCtx vc = cx;
  int late = GST_OK;
  vc.late = &late;
  const int st = put_map_value<Cnt, SLOW>(c, vc, vf, me, rec);
  return (st == GST_RANGE || st == GST_INVALID_VALUE) ? GST_OK : st;
}
// every string key / string value occurrence of the entry payload [beg, end) (parse_map_entry found it well-formed)
GGR_DEVN int check_entry_strings(const DecCtx& cx, u32 beg, u32 end, bool str_key, bool str_val) {
  Rd r;
  r.init(cx.in, beg, end, cx.rw);
  while (r.pos < end) {
    u64 tag, v;
    if (!rd_varint(r, end, &tag)) return GST_BAD_WIRE;
    const u64 num = tag >> 3;
    const u32 wt = (u32)(tag & 7);
    if (wt == 2 && ((num == 1 && str_key) || (num == 2 && str_val))) {
      if (!rd_varint(r, end, &v) || v > (u64)(end - r.pos)) return GST_BAD_WIRE;
      Cnt c;
      c.pos = 0;
      const u32 next = r.pos + (u32)v;
      const int st = put_json_string(c, r, (u32)v);
      if (st != GST_OK) return st;
      rd_jump(r, next);
    } else if (!rd_skip_value(r, end, (u32)num, wt)) {
      return GST_BAD_WIRE;
    }
  }
  return GST_OK;
}

// Map field writer.  `r` is positioned right after the tag of the first entry (fast walk) and is
// left after the last entry of the run.  In the slow walk the entries are all occurrences of the
// field inside [pstart, pend).
template <class W, bool SLOW>
GGR_DEVN int put_map_field(W& w, const DecCtx& cx, u32 rpos, u32* rend, FieldD f, u32 pstart, u32 pend, int rec, bool count_only = false) {
  Rd r;
  r.init(cx.in, SLOW ? pstart : rpos, pend, cx.rw);
  *rend = rpos;
  MsgD ed = ggr_msg(cx.T, (u32)f.child);
  FieldD kf = ggr_field(cx.T, ed.field_first), vf = ggr_field(cx.T, ed.field_first + 1);
  // pass 1: find the run / all occurrences, validate, check ordering
  u32 run_start, run_end;
  bool sorted = true;
  u32 count = 0;
  {
    u64 prev = 0;
    if (!SLOW) {
      run_start = r.pos;  // after the first tag
      bool first = true;
      for (;;) {
        if (!first) {
          // peek the next tag: same field and LEN?
          Rd t = r;
          u64 tag;
          if (t.pos >= pend || !rd_varint(t, pend, &tag) || tag != (u64)f.tag) break;
          r = t;
        }
        first = false;
        u64 len;
        if (!rd_varint(r, pend, &len) || len > (u64)(pend - r.pos)) return GST_BAD_WIRE;
        MapEnt me;
        u32 lim = r.pos + (u32)len;
        int st = parse_map_entry(r, lim, kf, vf, &me);
        if (st != GST_OK) return st;
        if (me.dup && IsCountingWriter<W>::v && !count_only) {
          st = check_entry_strings(cx, me.beg, me.end, kf.kind == GK_STRING, vf.kind == GK_STRING);
          if (st != GST_OK) return st;
        }
        if (count > 0 && cmp_map_keys(cx, kf.kind, prev, me.key) >= 0) sorted = false;
        prev = me.key;
        count++;
      }
      run_end = r.pos;
      *rend = run_end;
    } else {
      run_start = pstart;
      run_end = pend;
      Rd t;
      t.init(cx.in, pstart, pend, cx.rw);
      while (t.pos < pend) {
        u64 tag;
        if (!rd_varint(t, pend, &tag)) return GST_BAD_WIRE;
        u32 wt = (u32)(tag & 7);
        // this scan may be the only one that reads the message's other tags (a message whose declared fields are all maps)
        if ((tag >> 3) == 0 || (tag >> 3) > 0x1FFFFFFFull || wt == 4 || wt > 5) return GST_BAD_WIRE;
        if (tag == (u64)f.tag) {
          u64 len;
          if (!rd_varint(t, pend, &len) || len > (u64)(pend - t.pos)) return GST_BAD_WIRE;
          MapEnt me;
          int st = parse_map_entry(t, t.pos + (u32)len, kf, vf, &me);
          if (st != GST_OK) return st;
          if (me.dup && IsCountingWriter<W>::v && !count_only) {
            st = check_entry_strings(cx, me.beg, me.end, kf.kind == GK_STRING, vf.kind == GK_STRING);
            if (st != GST_OK) return st;
          }
          if (count > 0 && cmp_map_keys(cx, kf.kind, prev, me.key) >= 0) sorted = false;
          prev = me.key;
          count++;
        } else if (!rd_skip_value(t, pend, (u32)(tag >> 3), wt)) {
          return GST_BAD_WIRE;
        }
      }
    }
  }
  if (count_only) {  // slow walk: is there anything to write?  (*rend = number of well-formed entries)
    *rend = count;
    return GST_OK;
  }
  if (count == 0) return GST_OK;
  // Unsorted entries (Go map iteration order; the usual case behind a Go backend): collect (key, position) of every
  // entry into scratch, heap-sort them by key then position, emit in that order - of equal keys the last occurrence
  // (map semantics: last wins).  O(k log k) key comparisons instead of k scans over the run.
  if (!sorted && count > 8u && cx.sort_pool) {
    const u32 base = ggr_atomic_add_u32(cx.sort_ctr, count);
    if (base <= cx.sort_cap && count <= cx.sort_cap - base) {
      U4* A = cx.sort_pool + base;
      const bool str_keys = kf.kind == GK_STRING;
      {
        Rd t;
        t.init(cx.in, run_start, run_end, cx.rw);
        bool first_in_run = !SLOW;
        u32 k = 0;
        while (t.pos < run_end && k < count) {
          if (!first_in_run) {
            u64 tag;
            if (!rd_varint(t, run_end, &tag)) return GST_BAD_WIRE;
            if (tag != (u64)f.tag) {
              if (!rd_skip_value(t, run_end, (u32)(tag >> 3), (u32)(tag & 7))) return GST_BAD_WIRE;
              continue;
            }
          }
          first_in_run = false;
          const u32 at = t.pos;
          u64 len;
          if (!rd_varint(t, run_end, &len)) return GST_BAD_WIRE;
          MapEnt me;
          int st = parse_map_entry(t, t.pos + (u32)len, kf, vf, &me);
          if (st != GST_OK) return st;
          U4 rec = {(u32)me.key, (u32)(me.key >> 32), at, 0u};
          if (str_keys) {
            // string keys: the first eight bytes (big-endian, zero-padded) and the length travel in the record, so that
            // a comparison of the sort is two register compares instead of a chain of loads from the wire (a 400-entry
            // map costs about 7 000 comparisons per sort)
            const u32 kp = (u32)me.key, kl = (u32)(me.key >> 32);
            u64 P = 0;
            for (u32 j = 0; j < 8u; j++) P = (P << 8) | (j < kl ? (u64)cx.in[kp + j] : 0ull);
            rec.x = (u32)P;
            rec.y = (u32)(P >> 32);
            rec.w = kl;
          }
          A[k++] = rec;
        }
        if (k != count) return GST_INTERNAL;
      }
      // keys longer than eight bytes whose first eight agree: compare the texts (the entries are parsed again)
      auto cmp_long = [&](const U4& a, const U4& b) -> int {
        MapEnt ma, mb;
        Rd t;
        u64 len;
        t.init(cx.in, a.z, run_end, cx.rw);
        if (!rd_varint(t, run_end, &len) || parse_map_entry(t, t.pos + (u32)len, kf, vf, &ma) != GST_OK) return 0;
        t.init(cx.in, b.z, run_end, cx.rw);
        if (!rd_varint(t, run_end, &len) || parse_map_entry(t, t.pos + (u32)len, kf, vf, &mb) != GST_OK) return 0;
        return cmp_map_keys(cx, kf.kind, ma.key, mb.key);
      };
      auto cmp_rec = [&](const U4& a, const U4& b) -> int {
        if (!str_keys) return cmp_map_keys(cx, kf.kind, (u64)a.x | ((u64)a.y << 32), (u64)b.x | ((u64)b.y << 32));
        const u64 pa = (u64)a.x | ((u64)a.y << 32), pb = (u64)b.x | ((u64)b.y << 32);
        if (pa != pb) return pa < pb ? -1 : 1;
        if (a.w <= 8u || b.w <= 8u) return a.w < b.w ? -1 : (a.w > b.w ? 1 : 0);  // equal padded prefixes: the shorter key is a prefix of the longer
        return cmp_long(a, b);
      };
      auto less = [&](const U4& a, const U4& b) -> bool {
        const int c = cmp_rec(a, b);
        return c < 0 || (c == 0 && a.z < b.z);
      };
      // heap sort (ascending): sift-down on a max-heap
      auto sift = [&](u32 root, u32 n) {
        U4 v = A[root];
        for (;;) {
          u32 child = 2u * root + 1u;
          if (child >= n) break;
          if (child + 1u < n && less(A[child], A[child + 1u])) child++;
          if (!less(v, A[child])) break;
          A[root] = A[child];
          root = child;
        }
        A[root] = v;
      };
      for (u32 i = count / 2u; i-- > 0u;) sift(i, count);
      for (u32 n = count; n > 1u; n--) {
        const U4 top = A[0];
        A[0] = A[n - 1u];
        A[n - 1u] = top;
        sift(0u, n - 1u);
      }
      w.put1('{');
      u32 efirst2 = 1;
      for (u32 i = 0; i < count; i++) {
        const U4 e = A[i];
        if (i + 1u < count) {  // an equal key follows: that later occurrence wins
          const U4 nx = A[i + 1u];
          if (cmp_rec(e, nx) == 0) {
            if (IsCountingWriter<W>::v) {  // Unmarshal has parsed the entry all the same
              Rd ts;
              ts.init(cx.in, e.z, run_end, cx.rw);
              u64 slen;
              MapEnt sme;
              if (!rd_varint(ts, run_end, &slen)) return GST_BAD_WIRE;
              int sst = parse_map_entry(ts, ts.pos + (u32)slen, kf, vf, &sme);
              if (sst == GST_OK) sst = check_shadowed_value<SLOW>(cx, vf, sme, rec);
              if (sst != GST_OK) return sst;
            }
            continue;
          }
        }
        Rd t;
        t.init(cx.in, e.z, run_end, cx.rw);
        u64 len;
        if (!rd_varint(t, run_end, &len)) return GST_BAD_WIRE;
        MapEnt me;
        int st = parse_map_entry(t, t.pos + (u32)len, kf, vf, &me);
        if (st != GST_OK) return st;
        put_sep(w, cx, efirst2);
        st = put_map_key(w, cx, kf.kind, me.key);
        if (st != GST_OK) return st;
        w.put1(':');
        st = put_map_value<W, SLOW>(w, cx, vf, me, rec);
        if (st != GST_OK) return st;
      }
      w.put1('}');
      return GST_OK;
    }
  }
  // pass 2: emit in key order.  Already sorted (the usual case for deterministic backends): one
  // sweep.  Otherwise selection by key: each round picks the smallest key above the last one
  // written, taking the LAST occurrence of that key (map semantics: last wins).
  w.put1('{');
  u32 efirst = 1;
  u64 last_key = 0;
  bool have_last = false;
  u32 rounds = sorted ? 1u : count;
  for (u32 round = 0; round < rounds; round++) {
    MapEnt best;
    bool have_best = false;
    Rd t;
    t.init(cx.in, run_start, run_end, cx.rw);
    bool first_in_run = !SLOW;
    while (t.pos < run_end) {
      if (!first_in_run) {
        u64 tag;
        if (!rd_varint(t, run_end, &tag)) return GST_BAD_WIRE;
        if (tag != (u64)f.tag) {
          if (!rd_skip_value(t, run_end, (u32)(tag >> 3), (u32)(tag & 7))) return GST_BAD_WIRE;
          continue;
        }
      }
      first_in_run = false;
      u64 len;
      if (!rd_varint(t, run_end, &len)) return GST_BAD_WIRE;
      MapEnt me;
      int st = parse_map_entry(t, t.pos + (u32)len, kf, vf, &me);
      if (st != GST_OK) return st;
      if (sorted) {
        put_sep(w, cx, efirst);
        st = put_map_key(w, cx, kf.kind, me.key);
        if (st != GST_OK) return st;
        w.put1(':');
        st = put_map_value<W, SLOW>(w, cx, vf, me, rec);
        if (st != GST_OK) return st;
        continue;
      }
      if (have_last && cmp_map_keys(cx, kf.kind, me.key, last_key) <= 0) continue;
      const int cb = have_best ? cmp_map_keys(cx, kf.kind, me.key, best.key) : -1;
      if (cb <= 0) {
        if (have_best && cb == 0 && IsCountingWriter<W>::v) {  // `best` is replaced by a later entry with its key
          const int sst = check_shadowed_value<SLOW>(cx, vf, best, rec);
          if (sst != GST_OK) return sst;
        }
        best = me;  // smaller key, or a later occurrence of the same key
        have_best = true;
      }
    }
    if (sorted) break;
    if (!have_best) break;
    put_sep(w, cx, efirst);
    int st = put_map_key(w, cx, kf.kind, best.key);
    if (st != GST_OK) return st;
    w.put1(':');
    st = put_map_value<W, SLOW>(w, cx, vf, best, rec);
    if (st != GST_OK) return st;
    last_key = best.key;
    have_last = true;
  }
  w.put1('}');
  return GST_OK;
}

template <class W, bool SLOW>
GGR_DEVN int walk_message(W& w, const DecCtx& cx, u32 root_msg, u32 start, u32 end, int rec, bool active, unsigned mask);

// Slow walk, size pass: the occurrences of singular field f inside the frame [start, end) that never reach the text - every
// occurrence but the last of a string field set several times (keep_pos = position behind the tag of the one that is
// written), every occurrence of a oneof member that a sibling set later replaces (keep_pos = 0xFFFFFFFF).  proto.Unmarshal
// has parsed them all the same: invalid UTF-8 or a malformed message inside one fails the item.
GGR_DEVN int check_dropped_occurrences(const DecCtx& lc, const FieldD& f, u32 start, u32 end, u32 keep_pos, int rec) {
  if (f.kind != GK_STRING && f.kind != GK_MESSAGE) return GST_OK;
  Rd t;
  t.init(lc.in, start, end, lc.rw);
  while (t.pos < end) {
    u64 tag;
    if (!rd_varint(t, end, &tag)) return GST_BAD_WIRE;
    const u64 n2 = tag >> 3;
    const u32 wt = (u32)(tag & 7);
    if (n2 == 0 || n2 > 0x1FFFFFFFull || wt == 4 || wt > 5) return GST_BAD_WIRE;
    if ((u32)n2 != f.number || wt != 2u || t.pos == keep_pos) {
      if (!rd_skip_value(t, end, (u32)n2, wt)) return GST_BAD_WIRE;
      continue;
    }
    u64 len;
    if (!rd_varint(t, end, &len) || len > (u64)(end - t.pos)) return GST_BAD_WIRE;
    const u32 lim = t.pos + (u32)len;
    Cnt c;
    c.pos = 0;
    if (f.kind == GK_STRING) {
      const int st = put_json_string(c, t, (u32)len);
      if (st != GST_OK) return st;
    } else {
      DecCtx vc = lc;
      int late = GST_OK;
      vc.late = &late;  // what Marshal would say about the value does not count: it never sees it
      const MsgD cd = ggr_msg(lc.T, (u32)f.child);
      int st;
      if (cd.wkt != GGR_WKT_NONE) {
        st = put_wkt(c, vc, (u32)f.child, t.pos, lim);
      } else {
        st = walk_message<Cnt, false>(c, vc, (u32)f.child, t.pos, lim, rec + 1, true, ggr_activemask());
        if (st == GGR_NEED_SLOW) st = walk_message<Cnt, true>(c, vc, (u32)f.child, t.pos, lim, rec + 1, true, ggr_activemask());
      }
      if (st != GST_OK && st != GST_RANGE && st != GST_INVALID_VALUE) return st;
    }
    rd_jump(t, lim);
  }
  return GST_OK;
}

// ---------------------------------------------------------------------------------------------
// The walker.  Recursion is only used for message values inside map entries and is bounded by
// `depth`; ordinary nesting uses the explicit frame stack.
// ---------------------------------------------------------------------------------------------
template <class W, bool SLOW>
GGR_DEVN int walk_message(W& w, const DecCtx& cx, u32 root_msg, u32 start, u32 end, int rec, bool active, unsigned mask) {
  const Tables& T = cx.T;
  DFrame stk[GGR_DEC_MAX_DEPTH];
  int depth = 0;
  bool finished = !active;
  int result = GST_OK;
  Rd r;
  DFrame fr;
  fr.end = end; fr.msg = root_msg; fr.last_decl = -1; fr.open = 0; fr.first = 1; fr.elem_first = 1; fr.oneofs = 0;
  fr.start = start; fr.scan = start; fr.cur_emit = 0; fr.state = 0;
  fr.base = cx.in;
  DecCtx lc;  // slow walk: the context of the current frame (lc.in = fr.base)
  if (SLOW && !finished) lc = cx;
  MsgD md;
  if (!finished && rec > GGR_DEC_MAX_REC) {
    result = GST_DEPTH;
    finished = true;
  }
  if (!finished) {
    r.init(cx.in, start, end, cx.rw);
    md = ggr_msg(T, root_msg);
    if (md.wkt != GGR_WKT_NONE) {
      result = put_wkt(w, cx, root_msg, start, end);
      finished = true;
    } else {
      w.put1('{');
    }
  } else {
    r.base = cx.in; r.pos = r.end = r.fetch = 0; r.avail = 0; r.cur = 0; r.ch.x = r.ch.y = r.ch.z = r.ch.w = 0;
    md.field_first = md.n_fields = md.wkt = md.flags = md.key_hash_first = md.key_hash_mask = md.decl_first = md.lut_first = md.lut_n = md.n_oneofs = 0;
  }

  // one step = one wire field (fast walk) / one declared field scan (slow walk); the lanes of
  // `mask` re-converge at the vote after every step
  while (ggr_any(mask, !finished)) {
   if (!finished) {
    int rr = GGR_STEP_CONT;
  for (int once = 0;; once++) {
    if (once) break;
    if (!SLOW) {
      // ================= fast walk =================
      if (r.pos >= fr.end) {
        if (r.pos != fr.end) GGR_RET(GST_BAD_WIRE);
        if (fr.open) w.put1(']');
        w.put1('}');
        if (depth == 0) GGR_RET(GST_OK);
        fr = stk[--depth];
        md = ggr_msg(T, fr.msg);
        continue;
      }
      u64 tag;
      if (!rd_varint(r, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
      u64 num64 = tag >> 3;
      u32 wt = (u32)(tag & 7);
      if (num64 == 0 || num64 > 0x1FFFFFFFull || wt == 4 || wt > 5) GGR_RET(GST_BAD_WIRE);
      u32 num = (u32)num64;
      i32 ei = find_field(T, md, num);
      if (ei < 0) {
        if (!rd_skip_value(r, fr.end, num, wt)) GGR_RET(GST_BAD_WIRE);
        continue;
      }
      FieldD f = ggr_field(T, md.field_first + (u32)ei);
      bool packed_in = (f.flags & GF_PACKABLE) && wt == 2;
      if (wt != f.wt && !packed_in) {  // wire type mismatch: treated as an unknown field
        if (!rd_skip_value(r, fr.end, num, wt)) GGR_RET(GST_BAD_WIRE);
        continue;
      }
      if (f.flags & GF_MAP) {
        if (fr.open) { w.put1(']'); fr.open = 0; }
        if ((i32)f.decl_index <= fr.last_decl) GGR_RET(GGR_NEED_SLOW);
        fr.last_decl = (i32)f.decl_index;
        // the key text is written only when the map has entries (always true here)
        put_sep(w, cx, fr.first);
        put_pool(w, T.pool, f.name_off, f.name_len);
        u32 run_end;
        int st = put_map_field<W, false>(w, cx, r.pos, &run_end, f, r.pos, fr.end, rec);
        if (st != GST_OK) GGR_RET(st);
        rd_jump(r, run_end);
        continue;
      }
      if (f.flags & GF_REPEATED) {
        if (fr.open != (u32)ei + 1) {
          if (fr.open) w.put1(']');
          fr.open = 0;
          if ((i32)f.decl_index <= fr.last_decl) GGR_RET(GGR_NEED_SLOW);
          // a packed field with an empty payload contributes no elements: dynamicpb then holds
          // an empty list, which protojson omits.  Look ahead before writing the key.
          if (packed_in) {
            Rd t = r;
            u64 len;
            if (!rd_varint(t, fr.end, &len) || len > (u64)(fr.end - t.pos)) GGR_RET(GST_BAD_WIRE);
            if (len == 0) {
              r = t;
              continue;
            }
          }
          fr.last_decl = (i32)f.decl_index;
          put_sep(w, cx, fr.first);
          put_pool(w, T.pool, f.name_off, f.name_len);
          w.put1('[');
          fr.open = (u32)ei + 1;
          fr.elem_first = 1;
        }
        if (packed_in) {
          u64 len;
          if (!rd_varint(r, fr.end, &len) || len > (u64)(fr.end - r.pos)) GGR_RET(GST_BAD_WIRE);
          u32 lim = r.pos + (u32)len;
          while (r.pos < lim) {
            put_sep(w, cx, fr.elem_first);
            bool z;
            int st = scalar_value<W, true>(w, cx, r, lim, f.kind, f.child, false, &z);
            if (st != GST_OK) GGR_RET(st);
          }
          if (r.pos != lim) GGR_RET(GST_BAD_WIRE);
          continue;
        }
        put_sep(w, cx, fr.elem_first);
        if (f.kind != GK_MESSAGE) {
          bool z;
          int st = scalar_value<W, true>(w, cx, r, fr.end, f.kind, f.child, false, &z);
          if (st != GST_OK) GGR_RET(st);
          continue;
        }
        // message element: falls through to the message push below
      } else {
        if (fr.open) { w.put1(']'); fr.open = 0; }
        if ((i32)f.decl_index <= fr.last_decl) GGR_RET(GGR_NEED_SLOW);
        if (f.oneof >= 0) {
          u32 bit = 1u << (f.oneof & 31);
          if (fr.oneofs & bit) GGR_RET(GGR_NEED_SLOW);  // last member wins: needs the slow walk
          fr.oneofs |= bit;
        }
        fr.last_decl = (i32)f.decl_index;
        if (f.kind != GK_MESSAGE) {
          if (!(f.flags & GF_PRESENCE)) {
            // implicit presence: a zero value is not "set" (dynamicpb isSet) - read ahead.
            // Strings and bytes only need their length prefix for that.
            Rd t = r;
            bool z;
            if (f.wt == 2) {
              u64 len;
              if (!rd_varint(t, fr.end, &len) || len > (u64)(fr.end - t.pos)) GGR_RET(GST_BAD_WIRE);
              z = len == 0;
            } else {
              Cnt c;
              c.pos = 0;
              int st = scalar_value<Cnt, false>(c, cx, t, fr.end, f.kind, f.child, false, &z);
              if (st != GST_OK) GGR_RET(st);
            }
            if (z) {
              r = t;
              continue;
            }
          }
          put_sep(w, cx, fr.first);
          put_pool(w, T.pool, f.name_off, f.name_len);
          bool z;
          int st = scalar_value<W, true>(w, cx, r, fr.end, f.kind, f.child, false, &z);
          if (st != GST_OK) GGR_RET(st);
          continue;
        }
        put_sep(w, cx, fr.first);
        put_pool(w, T.pool, f.name_off, f.name_len);
      }
      // ---- message value (singular or repeated element) ----
      {
        u64 len;
        if (!rd_varint(r, fr.end, &len) || len > (u64)(fr.end - r.pos)) GGR_RET(GST_BAD_WIRE);
        u32 lim = r.pos + (u32)len;
        MsgD cd = ggr_msg(T, (u32)f.child);
        if (cd.wkt != GGR_WKT_NONE) {
          int st = put_wkt(w, cx, (u32)f.child, r.pos, lim);
          if (st != GST_OK) GGR_RET(st);
          rd_jump(r, lim);
          continue;
        }
        if (depth >= GGR_DEC_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
        stk[depth++] = fr;
        fr.end = lim; fr.msg = (u32)f.child; fr.last_decl = -1; fr.open = 0; fr.first = 1; fr.elem_first = 1; fr.oneofs = 0;
        fr.start = r.pos; fr.scan = r.pos; fr.cur_emit = 0; fr.state = 0;
        md = cd;
        w.put1('{');
        continue;
      }
    } else {
      // ================= slow walk =================
      lc.in = fr.base;
      lc.rw = fr.base != cx.in ? 1u : cx.rw;
      // fr.last_decl + 1 is the next declaration index to handle; fr.state == 1 means we are in
      // the middle of a repeated message field (resume scanning at fr.scan)
      if (fr.state == 0) {
        fr.last_decl++;
        if ((u32)fr.last_decl >= md.n_fields) {
          // validate the whole payload once more for unknown-field well-formedness is done by
          // the per-field scans (each scan walks every tag); nothing left to do
          if (md.n_fields == 0) {
            // still need to validate the bytes
            Rd t;
            t.init(lc.in, fr.start, fr.end, lc.rw);
            while (t.pos < fr.end) {
              u64 tag;
              if (!rd_varint(t, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
              u64 n2 = tag >> 3;
              if (n2 == 0 || n2 > 0x1FFFFFFFull || (tag & 7) == 4 || (tag & 7) > 5) GGR_RET(GST_BAD_WIRE);
              if (!rd_skip_value(t, fr.end, (u32)n2, (u32)(tag & 7))) GGR_RET(GST_BAD_WIRE);
            }
          }
          w.put1('}');
          if (depth == 0) GGR_RET(GST_OK);
          fr = stk[--depth];
          md = ggr_msg(T, fr.msg);
          continue;
        }
        fr.cur_emit = ggr_u16(T, md.decl_first + (u32)fr.last_decl);
        fr.scan = fr.start;
        fr.elem_first = 1;
        fr.open = 0;
      }
      FieldD f = ggr_field(T, md.field_first + fr.cur_emit);
      if (f.flags & GF_MAP) {
        fr.state = 0;
        // does the map have any entry?  put_map_field writes nothing for an empty map, but the
        // key must not be written either: count first with a counting writer
        u32 unused_end = 0;
        int st = put_map_field<W, true>(w, lc, fr.start, &unused_end, f, fr.start, fr.end, rec, true);
        if (st != GST_OK) GGR_RET(st);
        if (unused_end == 0) continue;  // no entry: nothing is written, the key neither
        put_sep(w, lc, fr.first);
        put_pool(w, T.pool, f.name_off, f.name_len);
        st = put_map_field<W, true>(w, lc, fr.start, &unused_end, f, fr.start, fr.end, rec);
        if (st != GST_OK) GGR_RET(st);
        continue;
      }
      bool repeated = (f.flags & GF_REPEATED) != 0;
      // scan for occurrences from fr.scan
      Rd t;
      t.init(lc.in, fr.scan, fr.end, lc.rw);
      u32 last_pos = 0, last_wt = 0;  // singular: position after the tag of the last occurrence
      u32 n_occ = 0;
      bool pushed = false;
      while (t.pos < fr.end) {
        if (!lc.rw) {  // the occurrences of other fields: one 8-byte window each
          const u32 p = dec_skip_others(lc.in, t.pos, fr.end, f.number);
          if (p != t.pos) rd_jump(t, p);
          if (p >= fr.end) break;
        }
        u64 tag;
        if (!rd_varint(t, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
        u64 n2 = tag >> 3;
        u32 wt = (u32)(tag & 7);
        if (n2 == 0 || n2 > 0x1FFFFFFFull || wt == 4 || wt > 5) GGR_RET(GST_BAD_WIRE);
        bool packed_in = (f.flags & GF_PACKABLE) && wt == 2;
        if ((u32)n2 != f.number || (wt != f.wt && !packed_in)) {
          if (!rd_skip_value(t, fr.end, (u32)n2, wt)) GGR_RET(GST_BAD_WIRE);
          continue;
        }
        if (!repeated) {
          last_pos = t.pos;
          last_wt = wt;
          n_occ++;
          if (!rd_skip_value(t, fr.end, (u32)n2, wt)) GGR_RET(GST_BAD_WIRE);
          continue;
        }
        // repeated occurrence
        if (packed_in) {
          u64 len;
          if (!rd_varint(t, fr.end, &len) || len > (u64)(fr.end - t.pos)) GGR_RET(GST_BAD_WIRE);
          u32 lim = t.pos + (u32)len;
          while (t.pos < lim) {
            if (!fr.open) {
              put_sep(w, lc, fr.first);
              put_pool(w, T.pool, f.name_off, f.name_len);
              w.put1('[');
              fr.open = 1;
            }
            put_sep(w, lc, fr.elem_first);
            u32 nx_;
            int st = scalar_value_at<W, true>(w, lc, t.pos, lim, f.kind, f.child, &nx_);
            rd_jump(t, nx_ & 0x7FFFFFFFu);
            if (st != GST_OK) GGR_RET(st);
          }
          if (t.pos != lim) GGR_RET(GST_BAD_WIRE);
          continue;
        }
        if (!fr.open) {
          put_sep(w, lc, fr.first);
          put_pool(w, T.pool, f.name_off, f.name_len);
          w.put1('[');
          fr.open = 1;
        }
        put_sep(w, lc, fr.elem_first);
        if (f.kind != GK_MESSAGE) {
          u32 nx_;
          int st = scalar_value_at<W, true>(w, lc, t.pos, fr.end, f.kind, f.child, &nx_);
          rd_jump(t, nx_ & 0x7FFFFFFFu);
          if (st != GST_OK) GGR_RET(st);
          continue;
        }
        // message element: push a frame, resume this scan afterwards
        u64 len;
        if (!rd_varint(t, fr.end, &len) || len > (u64)(fr.end - t.pos)) GGR_RET(GST_BAD_WIRE);
        u32 lim = t.pos + (u32)len;
        MsgD cd = ggr_msg(T, (u32)f.child);
        if (cd.wkt != GGR_WKT_NONE) {
          int st = put_wkt(w, lc, (u32)f.child, t.pos, lim);
          if (st != GST_OK) GGR_RET(st);
          rd_jump(t, lim);
          continue;
        }
        if (depth >= GGR_DEC_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
        fr.state = 1;
        fr.scan = lim;
        stk[depth++] = fr;
        fr.end = lim; fr.msg = (u32)f.child; fr.last_decl = -1; fr.open = 0; fr.first = 1; fr.elem_first = 1; fr.oneofs = 0;
        fr.start = t.pos; fr.scan = t.pos; fr.cur_emit = 0; fr.state = 0;
        md = cd;
        w.put1('{');
        pushed = true;
        break;
      }
      if (pushed) continue;
      if (repeated) {
        if (fr.open) w.put1(']');
        fr.open = 0;
        fr.state = 0;
        continue;
      }
      fr.state = 0;
      if (n_occ == 0) continue;
      // oneof: only the member set last on the wire survives
      if (f.oneof >= 0) {
        bool later = false;
        Rd q;
        q.init(lc.in, last_pos, fr.end, lc.rw);
        if (!rd_skip_value(q, fr.end, f.number, last_wt)) GGR_RET(GST_BAD_WIRE);
        while (q.pos < fr.end && !later) {
          u64 tag;
          if (!rd_varint(q, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
          u32 n3 = (u32)(tag >> 3), w3 = (u32)(tag & 7);
          i32 e3 = find_field(T, md, n3);
          if (e3 >= 0 && (u32)e3 != fr.cur_emit) {
            FieldD g = ggr_field(T, md.field_first + (u32)e3);
            if (g.oneof == f.oneof && (w3 == g.wt)) later = true;
          }
          if (!rd_skip_value(q, fr.end, n3, w3)) GGR_RET(GST_BAD_WIRE);
        }
        if (later) {
          if (IsCountingWriter<W>::v) {  // the member is replaced: Unmarshal has parsed its occurrences all the same
            const int cs = check_dropped_occurrences(lc, f, fr.start, fr.end, 0xFFFFFFFFu, rec);
            if (cs != GST_OK) GGR_RET(cs);
          }
          continue;
        }
      }
      if (n_occ > 1 && f.kind == GK_STRING && IsCountingWriter<W>::v) {  // set several times: the last one is written
        const int cs = check_dropped_occurrences(lc, f, fr.start, fr.end, last_pos, rec);
        if (cs != GST_OK) GGR_RET(cs);
      }
      if (f.kind == GK_MESSAGE) {
        MsgD cd = ggr_msg(T, (u32)f.child);
        if (n_occ > 1) {
          // split over several occurrences: walk the merged payload (its own buffer) as the child frame
          if (cd.wkt == GGR_WKT_UNSUPPORTED) GGR_RET(GST_UNSUPPORTED);
          u32 mstart = fr.start;
          if (f.oneof >= 0) {  // a sibling set in between clears the member: only what follows it merges
            Rd q;
            q.init(lc.in, fr.start, fr.end, lc.rw);
            while (q.pos < last_pos) {
              u64 tag;
              if (!rd_varint(q, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
              u32 n3 = (u32)(tag >> 3), w3 = (u32)(tag & 7);
              i32 e3 = find_field(T, md, n3);
              bool sib = false;
              if (e3 >= 0 && (u32)e3 != fr.cur_emit) {
                FieldD g = ggr_field(T, md.field_first + (u32)e3);
                sib = g.oneof == f.oneof && w3 == g.wt;
              }
              if (!rd_skip_value(q, fr.end, n3, w3)) GGR_RET(GST_BAD_WIRE);
              if (sib) mstart = q.pos;
            }
            if (mstart != fr.start && IsCountingWriter<W>::v) {  // the pieces in front of the sibling: parsed by Unmarshal, dropped here
              const int cs = check_dropped_occurrences(lc, f, fr.start, mstart, 0xFFFFFFFFu, rec);
              if (cs != GST_OK) GGR_RET(cs);
            }
          }
          const u8* mb;
          u32 ml;
          int st = merge_occurrences(lc, mstart, fr.end, f.number, &mb, &ml);
          if (st != GST_OK) GGR_RET(st);
          put_sep(w, lc, fr.first);
          put_pool(w, T.pool, f.name_off, f.name_len);
          if (cd.wkt != GGR_WKT_NONE) {
            DecCtx mc = lc;
            mc.in = mb;
            mc.rw = 1;
            st = put_wkt(w, mc, (u32)f.child, 0, ml);
            if (st != GST_OK) GGR_RET(st);
            continue;
          }
          if (depth >= GGR_DEC_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
          stk[depth++] = fr;
          fr.end = ml; fr.msg = (u32)f.child; fr.last_decl = -1; fr.open = 0; fr.first = 1; fr.elem_first = 1; fr.oneofs = 0;
          fr.start = 0; fr.scan = 0; fr.cur_emit = 0; fr.state = 0;
          fr.base = mb;
          md = cd;
          w.put1('{');
          continue;
        }
        Rd q;
        q.init(lc.in, last_pos, fr.end, lc.rw);
        u64 len;
        if (!rd_varint(q, fr.end, &len) || len > (u64)(fr.end - q.pos)) GGR_RET(GST_BAD_WIRE);
        u32 lim = q.pos + (u32)len;
        put_sep(w, lc, fr.first);
        put_pool(w, T.pool, f.name_off, f.name_len);
        if (cd.wkt != GGR_WKT_NONE) {
          int st = put_wkt(w, lc, (u32)f.child, q.pos, lim);
          if (st != GST_OK) GGR_RET(st);
          continue;
        }
        if (depth >= GGR_DEC_MAX_DEPTH - 1) GGR_RET(GST_DEPTH);
        stk[depth++] = fr;
        fr.end = lim; fr.msg = (u32)f.child; fr.last_decl = -1; fr.open = 0; fr.first = 1; fr.elem_first = 1; fr.oneofs = 0;
        fr.start = q.pos; fr.scan = q.pos; fr.cur_emit = 0; fr.state = 0;
        md = cd;
        w.put1('{');
        continue;
      }
      // singular scalar: the last occurrence wins; every occurrence must still be valid
      {
        Rd q;
        q.init(lc.in, fr.start, fr.end, lc.rw);
        // validate all occurrences (strings: UTF-8) the way proto.Unmarshal would; the scan above has been over every
        // field header of the message already, so only string fields have anything left to check
        while (f.kind == GK_STRING && q.pos < fr.end) {
          if (!lc.rw) {
            const u32 p = dec_skip_others(lc.in, q.pos, fr.end, f.number);
            if (p != q.pos) rd_jump(q, p);
            if (p >= fr.end) break;
          }
          u64 tag;
          if (!rd_varint(q, fr.end, &tag)) GGR_RET(GST_BAD_WIRE);
          u32 n3 = (u32)(tag >> 3), w3 = (u32)(tag & 7);
          if (n3 == f.number && w3 == f.wt && f.kind == GK_STRING) {
            bool z;
            Cnt c;
            c.pos = 0;
            u32 nz_;
            int st = scalar_value_at<Cnt, false>(c, lc, q.pos, fr.end, f.kind, f.child, &nz_);
            rd_jump(q, nz_ & 0x7FFFFFFFu);
            z = (nz_ >> 31) != 0;
            if (st != GST_OK) GGR_RET(st);
          } else if (!rd_skip_value(q, fr.end, n3, w3)) {
            GGR_RET(GST_BAD_WIRE);
          }
        }
        q.init(lc.in, last_pos, fr.end, lc.rw);
        if (!(f.flags & GF_PRESENCE)) {
          Rd t2 = q;
          bool z;
          Cnt c;
          c.pos = 0;
          u32 nz_;
          int st = scalar_value_at<Cnt, false>(c, lc, t2.pos, fr.end, f.kind, f.child, &nz_);
          rd_jump(t2, nz_ & 0x7FFFFFFFu);
          z = (nz_ >> 31) != 0;
          if (st != GST_OK) GGR_RET(st);
          if (z) continue;
        }
        put_sep(w, lc, fr.first);
        put_pool(w, T.pool, f.name_off, f.name_len);
        u32 nx_;
        int st = scalar_value_at<W, true>(w, lc, q.pos, fr.end, f.kind, f.child, &nx_);
        rd_jump(q, nx_ & 0x7FFFFFFFu);
        if (st != GST_OK) GGR_RET(st);
      }
    }
  }
  step_end:
    if (rr != GGR_STEP_CONT) {
      finished = true;
      result = rr;
    }
   }
  }
  return result;
}

// Size pass: tries the fast walk, falls back to the slow walk for the whole item.
// All lanes of `mask` call this together; lanes without an item pass active = false.
GGR_DEV int decode_size(const Tables& T, u32 msg, const u8* in, u32 start, u32 end, u32 flags, DecResult* res,
                        bool active = true, unsigned mask = GGR_FULL_MASK, U4* sort_pool = nullptr, u32* sort_ctr = nullptr, u32 sort_cap = 0) {
  DecCtx cx;
  cx.T = T;
  cx.in = in;
  cx.flags = flags;
  cx.sort_pool = sort_pool;
  cx.sort_ctr = sort_ctr;
  cx.sort_cap = sort_cap;
  int late = GST_OK;
  cx.late = &late;
  Cnt c;
  c.pos = 0;
  int st = walk_message<Cnt, false>(c, cx, msg, start, end, 0, active, mask);
  res->mode = GGR_MODE_FAST;
  bool need_slow = active && st == GGR_NEED_SLOW;
  if (need_slow) {
    c.pos = 0;
    late = GST_OK;
  }
  int st2 = walk_message<Cnt, true>(c, cx, msg, start, end, 0, need_slow, mask);
  if (need_slow) {
    st = st2;
    res->mode = GGR_MODE_SLOW;
  }
  res->size = c.pos;
  if (st == GST_OK && late != GST_OK) st = late;
  return st;
}

GGR_DEV int decode_write(const Tables& T, u32 msg, const u8* in, u32 start, u32 end, u32 flags, u32 mode, u8* out,
                         u32 out_off, u32* end_pos, bool active = true, unsigned mask = GGR_FULL_MASK, U4* sort_pool = nullptr,
                         u32* sort_ctr = nullptr, u32 sort_cap = 0) {
  DecCtx cx;
  cx.T = T;
  cx.in = in;
  cx.flags = flags;
  cx.sort_pool = sort_pool;
  cx.sort_ctr = sort_ctr;
  cx.sort_cap = sort_cap;
  Wr w;
  w.init(out, out_off);
  bool slow = mode == GGR_MODE_SLOW;
  int st_f = walk_message<Wr, false>(w, cx, msg, start, end, 0, active && !slow, mask);
  int st_s = walk_message<Wr, true>(w, cx, msg, start, end, 0, active && slow, mask);
  if (active) w.finish();
  *end_pos = w.pos;
  return slow ? st_s : st_f;
}
