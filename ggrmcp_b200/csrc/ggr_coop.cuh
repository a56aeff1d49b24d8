// ggr_coop.cuh - lock-step reply side: one warp per item, protobuf wire -> protojson text.
//
// The per-thread walker (ggr_decode.cuh) runs 32 unrelated state machines per warp.  Here the 32
// lanes work on ONE item:
//   R1 discover : level by level (root, its sub-messages, theirs, ...) one lane scans one message's
//                 top-level tags - length-delimited payloads are skipped in O(1) - and appends one
//                 table entry per field occurrence, linked to its parent message
//   R2 classes  : the whole warp builds a "plain text" bit mask of the item (16 bytes per lane and
//                 step) so that a string needs no per-byte scan unless it holds a quote, a
//                 backslash, a control or a non-ASCII byte; entries are bucketed by kind
//   R3 sizes    : one lane per leaf computes the size of its JSON text; message entries add up
//                 bottom-up, one level of R1's queue at a time; offsets go top-down
//   -- the entry table is saved, the batch-wide scan of the item sizes runs --
//   R4 write    : one lane per entry writes its text at its offset; long plain strings are copied
//                 by the whole warp
// Only the regular case is handled (fields in declaration order, no maps, table fits): anything
// else - including every malformed item - is left to the per-thread kernels, which own the
// semantics.  All lanes call the *_item functions together (see ggr_warp.cuh; the CPU tests run
// them on 32 fibers).
#pragma once
#include "ggr_decode.cuh"
#include "ggr_warp.cuh"

// why the lock-step tier left an item: recorded by the host simulation only (tests/hostsim: hs_coop_why = source line)
#if !defined(__CUDA_ARCH__) && !defined(__CUDACC__)
extern int g_coop_why;
#define COOP_BAIL(S) ((S).bail = 1, g_coop_why = __LINE__)
#else
#define COOP_BAIL(S) ((S).bail = 1)
#endif

// Entry tables: every item owns GGR_COOP_TAB_ENTRIES slots of the saved table in HBM; the size pass works on a copy in
// shared memory - 224 entries in the first tier (bench replies: 133 on average; 8.9 KB per warp with the masks below =
// 24 warps per SM), the full 320 in the second tier, which takes the few items the first leaves because of the table
// (one such item on the per-thread kernels costs half a millisecond of one lane: the tail of the whole batch).
#define GGR_COOP_TAB_ENTRIES 320
#define GGR_COOP_ENTRIES 224
#define GGR_COOP_DEPTH 24
#define GGR_COOP_MAX_WIRE 4096u  /* larger items: no plain-text masks, strings are classified one by one */
#define GGR_MODE_COOP 2u
#define GGR_MODE_PENDING 0xFFu

#define CF_MSG 0x0001u         /* entry is a (non-WKT) sub-message: has children */
#define CF_ARR_FIRST 0x0002u   /* first element of a repeated field: writes name and '[' */
#define CF_ARR_LAST 0x0004u    /* last element: writes ']' */
#define CF_ARR_ELEM 0x0008u    /* element of a repeated field */
#define CF_PACKED 0x0010u      /* packed repeated scalars: the entry holds the whole run */
#define CF_FIRST 0x0020u       /* first field written inside its parent: no leading comma */
#define CF_TIMESTAMP 0x0040u   /* google.protobuf.Timestamp leaf */
#define CF_PLAIN 0x0080u       /* string without quote / backslash / control / non-ASCII bytes */
#define CF_CLASS_SHIFT 8
enum { DC_MSG = 0, DC_STR = 1, DC_BYTES = 2, DC_VARINT = 3, DC_FIXED = 4, DC_FLOAT = 5, DC_TS = 6, DC_PACKED = 7, DC_N = 8 };

struct CoopEnt {            // 32 bytes: saved between the passes as two 16-byte words
  u32 vpos;                 // position right after the tag (length prefix / scalar bytes start)
  u32 vend;                 // end of the value
  u32 body;                 // length-delimited values: position of the payload
  u32 size;                 // full text size: separator + name + brackets + value
  u32 off;                  // output offset of the full text (relative to the item)
  u16 parent, next;         // parent message entry; next sibling (0xFFFF = none)
  u16 fc_msg;               // CF_MSG: message type until the entry is scanned, then its first child
  u16 gfield;               // global field index (0xFFFF for the root)
  u16 flags, depth;
};
#define GGR_COOP_ROOT 0xFFFFu
#define CE_CLASS(e) (((e).flags >> CF_CLASS_SHIFT) & 0xFu)

#define GGR_COOP_LONG 96u /* plain strings of at least this many bytes are copied by the whole warp */
#define GGR_COOP_LONG_MAX 32u
#define GGR_COOP_DIRTY_MAX 64u
template <int NE>
struct CoopSharedT {
  static const u32 ENTRIES = NE;
  CoopEnt ent[NE];
  // message entries level by level in [0, q_end) (R1 appends them; R3 closes and places them by level), then the
  // leaves bucketed by class in [q_end, leaf_end)
  u16 queue[NE];
  u16 lvl[GGR_COOP_DEPTH + 1];            // queue index where each level starts (and where the last one ends)
  u16 dmask[GGR_COOP_MAX_WIRE / 16 + 2];  // per 16-byte chunk: bytes that are not plain text
  u16 dpre[GGR_COOP_MAX_WIRE / 16 + 2];   // number of chunks with a nonzero mask before this one
  u32 cls_cnt[DC_N], cls_cur[DC_N];
  u32 n_ent, bail, leaf_end, q_end, n_dirty;
  u16 dlist[GGR_COOP_DIRTY_MAX];          // strings that need escaping / validation: sized by the whole warp
};
typedef CoopSharedT<GGR_COOP_ENTRIES> CoopShared;      // first tier
// second tier: replies of thousands of field occurrences (a 39 KB reply of the mixed replay holds 1 800: one lane of the
// per-thread kernels walks them one after the other); 141 KB of shared memory = one warp per SM, the saved table goes to a pool
#define GGR_COOP_BIG_ENTRIES 4096
typedef CoopSharedT<GGR_COOP_BIG_ENTRIES> CoopSharedBig;

GGR_DEV u32 coop_class(const FieldD& f, bool ts, bool packed) {
  if (packed) return DC_PACKED;
  if (ts) return DC_TS;
  switch (f.kind) {
    case GK_STRING: return DC_STR;
    case GK_BYTES: return DC_BYTES;
    case GK_FLOAT: case GK_DOUBLE: return DC_FLOAT;
    case GK_FIXED32: case GK_FIXED64: case GK_SFIXED32: case GK_SFIXED64: return DC_FIXED;
    default: return DC_VARINT;
  }
}

// ---- plain byte access for the discovery pass: tags and lengths are one or two bytes, a
// streaming reader with a 16-byte chunk and a shift register costs more than it saves here ----
GGR_DEV bool br_varint(const u8* b, u32& pos, u32 lim, u64* out) {
  if (pos >= lim) return false;
  u32 c = b[pos++];
  if (c < 0x80u) {
    *out = c;
    return true;
  }
  u64 v = c & 0x7Fu;
  for (int i = 1; i < 10; i++) {
    if (pos >= lim) return false;
    c = b[pos++];
    if (i == 9 && c > 1) return false;
    v |= (u64)(c & 0x7Fu) << (7 * i);
    if (c < 0x80u) {
      *out = v;
      return true;
    }
  }
  return false;
}
// skips one value of wire type wt (groups: not handled here -> false, the caller bails)
GGR_DEV bool br_skip(const u8* b, u32& pos, u32 lim, u32 wt) {
  u64 v;
  switch (wt) {
    case 0: return br_varint(b, pos, lim, &v);
    case 1: if (lim - pos < 8) return false; pos += 8; return true;
    case 5: if (lim - pos < 4) return false; pos += 4; return true;
    case 2:
      if (!br_varint(b, pos, lim, &v) || v > (u64)(lim - pos)) return false;
      pos += (u32)v;
      return true;
    default: return false;
  }
}
// Is the scalar at pos (wire type wt) the zero value of its kind?  (implicit presence: not written)
GGR_DEV bool coop_wire_zero(const u8* b, u32 pos, u32 lim, u32 wt, bool* ok) {
  *ok = true;
  u64 v;
  if (wt == 0 || wt == 2) {  // varint: zigzag(0) = 0, false = 0, enum 0; length-delimited: empty
    if (!br_varint(b, pos, lim, &v)) { *ok = false; return false; }
    if (wt == 2 && v > (u64)(lim - pos)) { *ok = false; return false; }
    return v == 0;
  }
  const u32 k = wt == 5 ? 4u : 8u;  // float / double: the bit pattern decides (-0.0 is set)
  if (lim - pos < k) { *ok = false; return false; }
  u32 any = 0;
  for (u32 j = 0; j < k; j++) any |= b[pos + j];
  return any == 0;
}

// coop_window / coop_header (a field header out of one 8-byte window): ggr_decode.cuh, shared with the slow walk

// R1, one lane: scan the top-level fields of message entry `me` and append its children.
template <class SH>
GGR_DEV void coop_scan_message(SH& S, const DecCtx& cx, u32 me) {
  const Tables& T = cx.T;
  const u8* const in = cx.in;
  const CoopEnt m = S.ent[me];
  const MsgD md = ggr_msg(T, m.fc_msg);
  S.ent[me].fc_msg = 0xFFFFu;  // from here on: first child
  if (md.wkt != GGR_WKT_NONE || m.depth + 1u >= GGR_COOP_DEPTH) { COOP_BAIL(S); return; }
  const u32 lim = m.vend;
  u32 pos = m.vpos;
  if (m.gfield != GGR_COOP_ROOT) {  // a field entry starts at its length prefix
    u64 len;
    if (!br_varint(in, pos, lim, &len) || len != (u64)(lim - pos)) { COOP_BAIL(S); return; }
  }
  i32 last_decl = -1;
  u32 open = 0;        // emit index + 1 of the repeated field currently being collected
  u32 oneofs = 0;
  u32 prev = 0xFFFFu;  // previous child entry
  bool any = false;
  const u32 end_al = (lim + 15u) & ~15u;  // the item's bytes are readable up to the end of their last 16-byte chunk
  while (pos < lim) {
    // the field header out of one 8-byte window; what does not fit it is decoded byte by byte
    u32 wtag = 0, wtl = 0, wbody = 0, wvend = 0;
    bool wzero = false;
    const u64 win = coop_window(in, pos, end_al);
    const bool fast = coop_header(win, pos, &wtag, &wtl, &wbody, &wvend, &wzero) && wvend <= lim && wbody <= lim;
    u64 tag = wtag;
    if (fast) pos += wtl;
    else if (!br_varint(in, pos, lim, &tag)) { COOP_BAIL(S); return; }
    const u64 num64 = tag >> 3;
    const u32 wt = (u32)(tag & 7);
    if (num64 == 0 || num64 > 0x1FFFFFFFull || wt == 3 || wt == 4 || wt > 5) { COOP_BAIL(S); return; }
    const u32 num = (u32)num64;
    const i32 ei = find_field(T, md, num);
    if (ei < 0) {
      if (fast) pos = wvend;
      else if (!br_skip(in, pos, lim, wt)) { COOP_BAIL(S); return; }
      continue;
    }
    const u32 gf = md.field_first + (u32)ei;
    const FieldD f = ggr_field(T, gf);
    const bool packed_in = (f.flags & GF_PACKABLE) && wt == 2;
    if (wt != f.wt && !packed_in) {
      if (fast) pos = wvend;
      else if (!br_skip(in, pos, lim, wt)) { COOP_BAIL(S); return; }
      continue;
    }
    if ((f.flags & GF_MAP) || gf >= 0xFFFFu) { COOP_BAIL(S); return; }
    const u32 vpos = pos;
    // value extent: [vpos, vend), payload of length-delimited values at body
    u32 body = pos, vend = pos;
    if (fast) {
      body = wbody;
      vend = wvend;
    } else if (wt == 2) {
      u64 len;
      if (!br_varint(in, body, lim, &len) || len > (u64)(lim - body)) { COOP_BAIL(S); return; }
      vend = body + (u32)len;
    } else {
      if (!br_skip(in, vend, lim, wt)) { COOP_BAIL(S); return; }
    }
    pos = vend;
    u32 flags = 0;
    const bool repeated = (f.flags & GF_REPEATED) != 0;
    if (repeated) {
      flags |= CF_ARR_ELEM;
      if (packed_in && vend == body) {  // an empty packed run contributes nothing (and opens nothing)
        if (open != (u32)ei + 1 && (i32)f.decl_index <= last_decl) { COOP_BAIL(S); return; }
        continue;
      }
      if (open != (u32)ei + 1) {
        if ((i32)f.decl_index <= last_decl) { COOP_BAIL(S); return; }
        if (open && prev != 0xFFFFu) S.ent[prev].flags |= CF_ARR_LAST;
        last_decl = (i32)f.decl_index;
        open = (u32)ei + 1;
        flags |= CF_ARR_FIRST;
      }
      if (packed_in) flags |= CF_PACKED;
    } else {
      if (open && prev != 0xFFFFu) S.ent[prev].flags |= CF_ARR_LAST;
      open = 0;
      if ((i32)f.decl_index <= last_decl) { COOP_BAIL(S); return; }
      if (f.oneof >= 0) {
        u32 bit = 1u << (f.oneof & 31);
        if (oneofs & bit) { COOP_BAIL(S); return; }
        oneofs |= bit;
      }
      last_decl = (i32)f.decl_index;
      if (f.kind != GK_MESSAGE && !(f.flags & GF_PRESENCE)) {
        bool ok = true;
        bool z = fast ? wzero : coop_wire_zero(in, vpos, lim, wt, &ok);
        if (!ok) { COOP_BAIL(S); return; }
        // a 32-bit kind keeps the low 32 bits of its varint (proto.Unmarshal): bits above them alone still make the zero value
        if (!z && wt == 0 && vend - vpos >= 5u && (f.kind == GK_INT32 || f.kind == GK_UINT32 || f.kind == GK_SINT32 || f.kind == GK_ENUM)) {
          u32 p = vpos;
          u64 v = 0;
          if (!br_varint(in, p, lim, &v)) { COOP_BAIL(S); return; }
          z = (u32)v == 0u;
        }
        if (z) continue;  // implicit presence: the zero value is not written
      }
    }
    const u32 slot = wp_atomic_add(&S.n_ent, 1u);
    if (slot >= SH::ENTRIES) { COOP_BAIL(S); return; }
    CoopEnt e;
    e.vpos = vpos;
    e.vend = vend;
    e.gfield = (u16)gf;
    e.parent = (u16)me;
    e.next = 0xFFFFu;
    e.size = 0;
    e.off = 0;
    e.fc_msg = 0xFFFFu;
    e.depth = (u16)(m.depth + 1);
    e.body = body;
    if (!any) flags |= CF_FIRST;
    bool ts = false;
    if (f.kind == GK_MESSAGE) {
      const u32 w = ggr_msg(T, (u32)f.child).wkt;
      if (w == GGR_WKT_TIMESTAMP) {
        flags |= CF_TIMESTAMP;
        ts = true;
      } else if (w != GGR_WKT_NONE || (u32)f.child >= 0xFFFFu) {
        COOP_BAIL(S);
        return;
      } else {
        flags |= CF_MSG;
        e.fc_msg = (u16)f.child;
      }
    }
    const u32 cls = (flags & CF_MSG) ? DC_MSG : coop_class(f, ts, (flags & CF_PACKED) != 0);
    e.flags = (u16)(flags | (cls << CF_CLASS_SHIFT));
    S.ent[slot] = e;
    if (flags & CF_MSG) S.queue[wp_atomic_add(&S.q_end, 1u)] = (u16)slot;
    if (prev == 0xFFFFu) S.ent[me].fc_msg = (u16)slot;
    else S.ent[prev].next = (u16)slot;
    prev = slot;
    any = true;
  }
  if (open && prev != 0xFFFFu) S.ent[prev].flags |= CF_ARR_LAST;
}

// flags in bit 7 of every byte -> 4 contiguous bits
GGR_DEV u32 coop_pack4(u32 x) { return (((x >> 7) * 0x00204081u) >> 21) & 0xFu; }
// per byte of w (bit 7 flags): not plain JSON string text (< 0x20, >= 0x80, '"', '\\')
GGR_DEV u32 coop_dirty_flags(u32 w) {
  const u32 lo7 = w & 0x7F7F7F7Fu;
  u32 ge20 = lo7 + 0x60606060u;               // bit 7: (byte & 0x7F) >= 0x20
  u32 q = (lo7 ^ 0x22222222u) + 0x7F7F7F7Fu;  // bit 7: (byte & 0x7F) != '"'
  u32 b = (lo7 ^ 0x5C5C5C5Cu) + 0x7F7F7F7Fu;  // bit 7: (byte & 0x7F) != '\\'
  return (w | ~(ge20 & q & b)) & 0x80808080u;
}

// R2, all lanes: dmask / dpre over the item's bytes [start, end)
template <class SH>
GGR_DEV void coop_plain_masks(SH& S, const u8* in, u32 start, u32 end) {
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u;
  const u32 nchunks = (end + 15u) >> 4;
  u32 base = 0;
  U4 vn;  // the next round's chunk is requested one round ahead
  vn.x = vn.y = vn.z = vn.w = 0u;
  if (lane < nchunks) vn = ggr_ld16(in + (lane << 4));
  for (u32 cb = 0; cb < nchunks; cb += 32) {
    const u32 ci = cb + lane;
    u32 D = 0;
    const U4 v = vn;
    if (ci + 32u < nchunks) vn = ggr_ld16(in + ((ci + 32u) << 4));
    if (ci < nchunks) {
      D = coop_pack4(coop_dirty_flags(v.x)) | (coop_pack4(coop_dirty_flags(v.y)) << 4) | (coop_pack4(coop_dirty_flags(v.z)) << 8) |
          (coop_pack4(coop_dirty_flags(v.w)) << 12);
    }
    const u32 any = WP_BALLOT(D != 0);
    if (ci < nchunks) {
      S.dmask[ci] = (u16)D;
      S.dpre[ci] = (u16)(base + wp_popc(any & lt));
    }
    base += wp_popc(any);
  }
  if (lane == 0) S.dpre[nchunks] = (u16)base;
  WP_SYNC();
}
// no byte of [s, e) needs escaping or validation (s < e, within the masks' range)
template <class SH>
GGR_DEV bool coop_is_plain(const SH& S, u32 s, u32 e) {
  const u32 c0 = s >> 4, c1 = (e - 1u) >> 4;
  u32 first = (u32)S.dmask[c0] & (0xFFFFu << (s & 15u));
  const u32 lastmask = 0xFFFFu >> (15u - ((e - 1u) & 15u));
  if (c0 == c1) return (first & lastmask) == 0;
  if (first & 0xFFFFu) return false;
  if ((u32)S.dmask[c1] & lastmask) return false;
  return S.dpre[c1] == S.dpre[c0 + 1];
}

// Text that surrounds an entry's value: separator, key, brackets.
GGR_DEV u32 coop_prefix_len(const DecCtx& cx, const CoopEnt& e, u32 name_len) {
  u32 n = 0;
  // a comma precedes everything except the first entry written inside its parent message
  // (CF_FIRST is only ever set on a message's first child, which for an array is its first element)
  if (!(e.flags & CF_FIRST)) n += (cx.flags & GGR_F_COMMA_SPACE) ? 2u : 1u;
  if (!(e.flags & CF_ARR_ELEM) || (e.flags & CF_ARR_FIRST)) n += name_len;
  if (e.flags & CF_ARR_FIRST) n += 1;
  return n;
}
template <class W>
GGR_DEV void coop_put_prefix(W& w, const DecCtx& cx, const CoopEnt& e, const FieldD& f) {
  if (!(e.flags & CF_FIRST)) {
    w.put1(',');
    if (cx.flags & GGR_F_COMMA_SPACE) w.put1(' ');
  }
  if (!(e.flags & CF_ARR_ELEM) || (e.flags & CF_ARR_FIRST)) put_pool(w, cx.T.pool, f.name_off, f.name_len);
  if (e.flags & CF_ARR_FIRST) w.put1('[');
}

// Value text of a leaf entry (scalar, packed run, timestamp) into any writer.
template <class W>
GGR_DEV int coop_leaf_value(W& w, const DecCtx& cx, const CoopEnt& e, const FieldD& f) {
  Rd r;
  r.init(cx.in, e.vpos, e.vend);
  if (e.flags & CF_TIMESTAMP) {
    u64 len;
    if (!rd_varint(r, e.vend, &len) || len > (u64)(e.vend - r.pos)) return GST_BAD_WIRE;
    i64 s, n;
    int st = read_timestamp_payload(r, r.pos + (u32)len, &s, &n);
    if (st != GST_OK) return st;
    return put_timestamp(w, s, n);
  }
  if (e.flags & CF_PACKED) {
    u64 len;
    if (!rd_varint(r, e.vend, &len) || len > (u64)(e.vend - r.pos)) return GST_BAD_WIRE;
    u32 lim = r.pos + (u32)len;
    u32 first = 1;
    while (r.pos < lim) {
      put_sep(w, cx, first);
      bool z;
      int st = scalar_value<W, true>(w, cx, r, lim, f.kind, f.child, false, &z);
      if (st != GST_OK) return st;
    }
    return r.pos == lim ? GST_OK : GST_BAD_WIRE;
  }
  bool z;
  return scalar_value<W, true>(w, cx, r, e.vend, f.kind, f.child, false, &z);
}

// ---- strings that hold quotes, backslashes, control or non-ASCII bytes: one byte per lane ----
// JSON text length of one string byte (protojson): 1, 2 (\" \\ \b \f \n \r \t) or 6 (\u00XX)
GGR_DEV u32 coop_esc_len(u32 c) {
  if (c >= 0x20u) return (c == '"' || c == '\\') ? 2u : 1u;
  return (c == 8u || c == 9u || c == 10u || c == 12u || c == 13u) ? 2u : 6u;
}
// all lanes: JSON text length of in[s, e) without the quotes; *ok = false on malformed UTF-8
GGR_DEV u32 coop_dirty_size(const u8* in, u32 s, u32 e, bool* ok) {
  const u32 lane = wp_lane();
  u32 total = 0, carry = 0, bad = 0;
  u32 cn = s + lane < e ? in[s + lane] : 0u;  // the next round's bytes are requested one round ahead
  for (u32 p = s; p < e; p += 32) {
    const u32 pos = p + lane;
    const bool valid = pos < e;
    const u32 c = cn;
    cn = pos + 32u < e ? in[pos + 32u] : 0u;
    const u32 l = valid ? coop_esc_len(c) : 0u;
    total += wp_popc(WP_BALLOT(valid)) + wp_popc(WP_BALLOT(l == 2u)) + 5u * wp_popc(WP_BALLOT(l == 6u));
    const u32 HI = WP_BALLOT(c >= 0x80u);
    if (HI | carry) {  // UTF-8: the continuation bytes the lead bytes announce == the ones present
      // the byte behind this lane's: the neighbour's, lane 31 takes lane 0's byte of the next round (0 past the end)
      const u32 nb = WP_SHFL(c, (lane + 1u) & 31u), n0 = WP_SHFL(cn, 0);
      const u32 c1 = lane == 31u ? n0 : nb;
      const bool lead = c >= 0xC0u;
      const u32 LD = WP_BALLOT(lead);
      const u32 L2 = WP_BALLOT(lead && c < 0xE0u), L3 = WP_BALLOT(lead && c >= 0xE0u && c < 0xF0u), L4 = WP_BALLOT(lead && c >= 0xF0u);
      const bool b = lead && (c < 0xC2u || c > 0xF4u || (c == 0xE0u && c1 < 0xA0u) || (c == 0xEDu && c1 >= 0xA0u) ||
                              (c == 0xF0u && c1 < 0x90u) || (c == 0xF4u && c1 >= 0x90u));
      if (WP_BALLOT(b)) bad = 1;
      const u64 EC = ((u64)(L2 | L3 | L4) << 1) | ((u64)(L3 | L4) << 2) | ((u64)L4 << 3);
      if (((u32)EC | carry) != (HI & ~LD)) bad = 1;
      carry = (u32)(EC >> 32);
    }
  }
  *ok = !bad && !carry;
  return total;
}
// all lanes: the escaped text of in[s, e) to d[0..)
GGR_DEV void coop_dirty_write(const u8* in, u32 s, u32 e, u8* d) {
  const u32 lane = wp_lane();
  u32 base = 0;
  u32 cn = s + lane < e ? in[s + lane] : 0u;  // the next round's bytes are requested one round ahead
  for (u32 p = s; p < e; p += 32) {
    const u32 pos = p + lane;
    const bool valid = pos < e;
    const u32 c = cn;
    cn = pos + 32u < e ? in[pos + 32u] : 0u;
    const u32 l = valid ? coop_esc_len(c) : 0u;
    u32 tot;
    const u32 o = base + WP_EXCL_SCAN(l, &tot);
    if (l == 1u) {
      d[o] = (u8)c;
    } else if (l == 2u) {
      d[o] = '\\';
      d[o + 1] = (u8)(c == 8u ? 'b' : c == 12u ? 'f' : c == 10u ? 'n' : c == 13u ? 'r' : c == 9u ? 't' : c);
    } else if (l == 6u) {
      const u32 hi = c >> 4, lo = c & 15u;
      d[o] = '\\'; d[o + 1] = 'u'; d[o + 2] = '0'; d[o + 3] = '0';
      d[o + 4] = (u8)('0' + hi);
      d[o + 5] = (u8)(lo < 10u ? '0' + lo : 'a' + lo - 10u);
    }
    base += tot;
  }
}

// all lanes: standard base64 (padded) of in[src, src + len) -> d[0..): 3 bytes per lane and step
GGR_DEV void coop_base64(const u8* in, u32 src, u32 len, u8* d) {
  const u32 lane = wp_lane();
  const u32 groups = len / 3u;
  for (u32 g = lane; g < groups; g += 32) {
    const u8* p = in + src + 3u * g;
    const u32 v = ((u32)p[0] << 16) | ((u32)p[1] << 8) | (u32)p[2];
    u8* o = d + 4u * g;
    o[0] = (u8)b64_char(v >> 18);
    o[1] = (u8)b64_char((v >> 12) & 63u);
    o[2] = (u8)b64_char((v >> 6) & 63u);
    o[3] = (u8)b64_char(v & 63u);
  }
  const u32 rem = len - groups * 3u;
  if (rem && lane == 0) {
    const u8* p = in + src + 3u * groups;
    u8* o = d + 4u * groups;
    const u32 v = ((u32)p[0] << 16) | (rem == 2u ? (u32)p[1] << 8 : 0u);
    o[0] = (u8)b64_char(v >> 18);
    o[1] = (u8)b64_char((v >> 12) & 63u);
    o[2] = rem == 2u ? (u8)b64_char((v >> 6) & 63u) : (u8)'=';
    o[3] = '=';
  }
}
// all lanes: does in[s, e) hold only plain text bytes?  512 bytes per step
GGR_DEV bool coop_plain_check(const u8* in, u32 s, u32 e) {
  const u32 lane = wp_lane();
  u32 any = 0;
  for (u32 c0 = s & ~15u; c0 < e; c0 += 512u) {
    const u32 c = c0 + (lane << 4);
    u32 D = 0;
    if (c < e) {
      const U4 v = ggr_ld16(in + c);
      D = coop_pack4(coop_dirty_flags(v.x)) | (coop_pack4(coop_dirty_flags(v.y)) << 4) | (coop_pack4(coop_dirty_flags(v.z)) << 8) |
          (coop_pack4(coop_dirty_flags(v.w)) << 12);
      if (c < s) D &= 0xFFFFu << (s - c);
      if (c + 16u > e) D &= 0xFFFFu >> (c + 16u - e);
    }
    any |= D;
  }
  return !WP_ANY(any != 0);
}

// R3, one lane: size of leaf entry ei (full text) added to its parent
template <class SH>
GGR_DEV void coop_size_leaf(SH& S, const DecCtx& cx, u32 ei, bool have_masks) {
  const CoopEnt e = S.ent[ei];
  const FieldD f = ggr_field(cx.T, e.gfield);
  u32 n = coop_prefix_len(cx, e, f.name_len);
  if (e.flags & CF_ARR_LAST) n += 1;
  const u32 cls = CE_CLASS(e);
  if (cls == DC_STR && have_masks && (e.vend == e.body || coop_is_plain(S, e.body, e.vend))) {
    S.ent[ei].flags = (u16)(e.flags | CF_PLAIN);
    n += 2u + (e.vend - e.body);
  } else if (cls == DC_BYTES) {
    n += 2u + ((e.vend - e.body + 2u) / 3u) * 4u;
  } else if (cls == DC_STR && !(e.flags & (CF_PACKED | CF_TIMESTAMP))) {
    // needs escaping / validation: the whole warp sizes it after this loop (the entry keeps the
    // size of everything but the string's own text until then)
    const u32 k = wp_atomic_add(&S.n_dirty, 1u);
    if (k < GGR_COOP_DIRTY_MAX) {
      S.dlist[k] = (u16)ei;
      S.ent[ei].size = n + 2u;
      return;
    }
    Cnt c;
    c.pos = 0;
    if (coop_leaf_value(c, cx, e, f) != GST_OK) {
      COOP_BAIL(S);
      return;
    }
    n += c.pos;
  } else {
    Cnt c;
    c.pos = 0;
    if (coop_leaf_value(c, cx, e, f) != GST_OK) {
      COOP_BAIL(S);
      return;
    }
    n += c.pos;
  }
  S.ent[ei].size = n;
  wp_atomic_add(&S.ent[e.parent].size, n);
}

// R3, one lane: message entry `me` has the sizes of all its children; add its own text and
// pass the total up
template <class SH>
GGR_DEV void coop_close_message(SH& S, const DecCtx& cx, u32 me) {
  const CoopEnt m = S.ent[me];
  u32 n = 2;  // { }
  if (m.gfield != GGR_COOP_ROOT) {
    const FieldD f = ggr_field(cx.T, m.gfield);
    n += coop_prefix_len(cx, m, f.name_len);
    if (m.flags & CF_ARR_LAST) n += 1;
  }
  const u32 total = m.size + n;
  S.ent[me].size = total;
  if (m.gfield != GGR_COOP_ROOT) wp_atomic_add(&S.ent[m.parent].size, total);
}

// R3, one lane: message entry hands out offsets to its children
template <class SH>
GGR_DEV void coop_offsets_message(SH& S, const DecCtx& cx, u32 me) {
  const CoopEnt m = S.ent[me];
  u32 pos = m.off;
  if (m.gfield != GGR_COOP_ROOT) {
    FieldD f = ggr_field(cx.T, m.gfield);
    pos += coop_prefix_len(cx, m, f.name_len);
  }
  pos += 1;  // '{'
  for (u32 c = m.fc_msg; c != 0xFFFFu; c = S.ent[c].next) {
    S.ent[c].off = pos;
    pos += S.ent[c].size;
  }
}

// ---- R4: the item's text is assembled in shared memory, then copied out with aligned 16-byte
// stores.  Entries are small (a key and a few dozen bytes), so a streaming writer with aligned
// groups would spend its time on the unaligned edges of every entry; plain byte stores into
// shared memory have no edges.
/* the writer's staging buffer; larger texts, of any size, are written in place.  6144 (configs[2]: texts up to 6.0 KB) with the kernel
   compiled for 7 blocks per SM (72 registers); 8 blocks (64 registers) spilled when tuned before the H100 port */
#define GGR_COOP_STAGE_BUF 6144u
struct
#if defined(__CUDACC__)
    __align__(16)
#else
    alignas(16)
#endif
        CoopStage {
  u8 buf[GGR_COOP_STAGE_BUF + 48];  // [pad, pad + size): pad = destination address & 15
  u32 lsrc[GGR_COOP_LONG_MAX], ldst[GGR_COOP_LONG_MAX], llen[GGR_COOP_LONG_MAX];
  u32 n_long, bad;
};
// R4, one lane: text of entry e into the staging buffer at pad + e.off.  Its byte copies switch to words from 24 bytes
// on (faster than 12 when tuned before the H100 port).
GGR_DEV int coop_write_entry(CoopStage& E, const DecCtx& cx, const CoopEnt& e, u8* B) {
  Sw w;
  w.init(B, e.off);
  if (e.gfield == GGR_COOP_ROOT) {
    B[e.off] = '{';
    B[e.off + e.size - 1] = '}';
    return GST_OK;
  }
  const FieldD f = ggr_field(cx.T, e.gfield);
  if (!(e.flags & CF_FIRST)) {
    w.put1(',');
    if (cx.flags & GGR_F_COMMA_SPACE) w.put1(' ');
  }
  if (!(e.flags & CF_ARR_ELEM) || (e.flags & CF_ARR_FIRST)) {
    coop_copy_bytes<24u>(B + w.pos, cx.T.pool + f.name_off, f.name_len);
    w.pos += f.name_len;
  }
  if (e.flags & CF_ARR_FIRST) w.put1('[');
  const u32 endpos = e.off + e.size;
  if (e.flags & CF_MSG) {
    w.put1('{');
    if (e.flags & CF_ARR_LAST) {
      B[endpos - 2] = '}';
      B[endpos - 1] = ']';
    } else {
      B[endpos - 1] = '}';
    }
    return GST_OK;
  }
  int st = GST_OK;
  if (e.flags & CF_PLAIN) {
    const u32 len = e.vend - e.body;
    w.put1('"');
    bool handed = false;
    if (len >= GGR_COOP_LONG) {
      const u32 k = wp_atomic_add(&E.n_long, 1u);
      if (k < GGR_COOP_LONG_MAX) {  // payload left to the whole warp
        E.lsrc[k] = e.body;
        E.ldst[k] = w.pos;
        E.llen[k] = len;
        handed = true;
      }
    }
    if (!handed) {
      coop_copy_bytes<24u>(B + w.pos, cx.in + e.body, len);
    }
    w.pos += len;
    w.put1('"');
  } else if (CE_CLASS(e) == DC_BYTES && !(e.flags & CF_PACKED) && e.vend - e.body >= GGR_COOP_LONG) {
    // long bytes field: base64 by the whole warp when the list has room
    const u32 k = wp_atomic_add(&E.n_long, 1u);
    if (k < GGR_COOP_LONG_MAX) {
      w.put1('"');
      E.lsrc[k] = e.body;
      E.ldst[k] = w.pos;
      E.llen[k] = (e.vend - e.body) | 0x40000000u;
      const u32 tail = (e.flags & CF_ARR_LAST) ? 2u : 1u;
      B[endpos - tail] = '"';
      if (e.flags & CF_ARR_LAST) B[endpos - 1] = ']';
      return GST_OK;
    }
    st = coop_leaf_value(w, cx, e, f);
  } else if (CE_CLASS(e) == DC_STR && !(e.flags & (CF_PACKED | CF_TIMESTAMP))) {
    // string that needs escaping: text left to the whole warp when the list has room
    const u32 k = wp_atomic_add(&E.n_long, 1u);
    if (k < GGR_COOP_LONG_MAX) {
      w.put1('"');
      E.lsrc[k] = e.body;
      E.ldst[k] = w.pos;
      E.llen[k] = (e.vend - e.body) | 0x80000000u;
      const u32 tail = (e.flags & CF_ARR_LAST) ? 2u : 1u;
      B[endpos - tail] = '"';
      if (e.flags & CF_ARR_LAST) B[endpos - 1] = ']';
      return GST_OK;
    }
    st = coop_leaf_value(w, cx, e, f);
  } else {
    st = coop_leaf_value(w, cx, e, f);
  }
  if (e.flags & CF_ARR_LAST) w.put1(']');
  if (st == GST_OK && w.pos != endpos) st = GST_INTERNAL;
  return st;
}

// Size pass of one item, all lanes.  Returns true when the item was handled: *size is its text
// size and, when `save` != nullptr, the entry table (n entries, *n_out) has been stored there for
// the write pass.
// pool != nullptr (second tier): the table is saved at pool + 2 * (*tab_off), *tab_off entries handed out by the bump
// counter *pool_ctr (pool_cap entries in all; an exhausted pool leaves the item to the per-thread kernels).
template <class SH>
GGR_DEV bool coop_size_item(SH& S, const DecCtx& cx, u32 root_msg, u32 start, u32 end, U4* save, u32* n_out, u32* size,
                            U4* pool = nullptr, u32* pool_ctr = nullptr, u32 pool_cap = 0, u32* tab_off = nullptr) {
  const u32 lane = wp_lane();
  *size = 0;
  *n_out = 0;
  if (root_msg >= 0xFFFFu) return false;
  const bool have_masks = end <= GGR_COOP_MAX_WIRE;  // larger items: strings are classified one by one
  WP_SYNC();  // persistent warps: nobody still reads the previous item's state
  if (lane == 0) {
    S.n_ent = 1;
    S.bail = 0;
    S.n_dirty = 0;
    CoopEnt r0;
    r0.vpos = start; r0.vend = end; r0.gfield = GGR_COOP_ROOT; r0.parent = 0xFFFFu; r0.next = 0xFFFFu;
    r0.size = 0; r0.off = 0; r0.fc_msg = (u16)root_msg; r0.depth = 0;
    r0.flags = (u16)(CF_MSG | CF_FIRST | (DC_MSG << CF_CLASS_SHIFT));
    r0.body = start;
    S.ent[0] = r0;
    S.queue[0] = 0;
    S.q_end = 1;
  }
  WP_SYNC();
  // R2 first: the plain-text masks read the whole item with coalesced 16-byte loads, which also brings
  // its lines into L1 for the byte-wise discovery below
  if (have_masks) coop_plain_masks(S, cx.in, start, end);
  // R1: level by level (level d holds the messages of depth d)
  u32 qb = 0, nl = 0;
  for (;;) {
    const u32 qe = S.q_end;
    if (lane == 0) S.lvl[nl] = (u16)qb;
    if (qb == qe) break;
    nl++;
    WP_SYNC();
    for (u32 i = qb + lane; i < qe; i += 32) coop_scan_message(S, cx, S.queue[i]);
    WP_SYNC();
    if (S.bail) return false;
    qb = qe;
  }
  const u32 n = S.n_ent;
  // leaves bucketed by class
  if (lane < DC_N) S.cls_cnt[lane] = 0;
  WP_SYNC();
  for (u32 i = lane; i < n; i += 32) {
    const u32 c = CE_CLASS(S.ent[i]);
    if (c != DC_MSG) wp_atomic_add(&S.cls_cnt[c], 1u);
  }
  WP_SYNC();
  const u32 q_end = S.q_end;
  if (lane == 0) {
    u32 run = q_end;
    for (u32 c = 0; c < DC_N; c++) {
      S.cls_cur[c] = run;
      run += S.cls_cnt[c];
    }
    S.leaf_end = run;
  }
  WP_SYNC();
  for (u32 i = lane; i < n; i += 32) {
    const u32 c = CE_CLASS(S.ent[i]);
    if (c != DC_MSG) S.queue[wp_atomic_add(&S.cls_cur[c], 1u)] = (u16)i;
  }
  WP_SYNC();
  // R3: leaf sizes, then messages bottom-up, then offsets top-down - the messages one level at a time, straight from
  // the queue: no lane visits a leaf or an entry of another depth
  const u32 leaf_end = S.leaf_end;
  for (u32 k = q_end + lane; k < leaf_end; k += 32) coop_size_leaf(S, cx, S.queue[k], have_masks);
  WP_SYNC();
  if (S.bail) return false;
  {
    const u32 nd = S.n_dirty < GGR_COOP_DIRTY_MAX ? S.n_dirty : GGR_COOP_DIRTY_MAX;
    for (u32 k = 0; k < nd; k++) {
      const u32 ei = S.dlist[k];
      bool ok;
      const u32 sb = S.ent[ei].body, se = S.ent[ei].vend;
      u32 js;
      if (se - sb >= 256u && coop_plain_check(cx.in, sb, se)) {  // long and plain (no masks for large items)
        js = se - sb;
        ok = true;
        if (lane == 0) S.ent[ei].flags |= CF_PLAIN;
      } else {
        js = coop_dirty_size(cx.in, sb, se, &ok);
      }
      if (!ok) return false;  // malformed UTF-8: the per-thread kernels report it
      if (lane == 0) {
        const u32 total = S.ent[ei].size + js;
        S.ent[ei].size = total;
        wp_atomic_add(&S.ent[S.ent[ei].parent].size, total);
      }
    }
    WP_SYNC();
  }
  for (u32 l = nl; l-- > 0;) {
    const u32 le = S.lvl[l + 1];
    for (u32 i = S.lvl[l] + lane; i < le; i += 32) coop_close_message(S, cx, S.queue[i]);
    WP_SYNC();
  }
  *size = S.ent[0].size;
  if (pool) {
    u32 base = 0;
    if (lane == 0) base = ggr_atomic_add_u32(pool_ctr, n);
    base = WP_SHFL(base, 0);
    if (base > pool_cap || n > pool_cap - base) return false;
    save = pool + 2 * (size_t)base;
    *tab_off = base;
  }
  if (!save) return true;
  for (u32 l = 0; l < nl; l++) {
    const u32 le = S.lvl[l + 1];
    for (u32 i = S.lvl[l] + lane; i < le; i += 32) coop_offsets_message(S, cx, S.queue[i]);
    WP_SYNC();
  }
  // save the table: two 16-byte stores per entry
  const U4* src = reinterpret_cast<const U4*>(S.ent);
  for (u32 i = lane; i < 2 * n; i += 32) save[i] = src[i];
  *n_out = n;
  return true;
}

// Write pass of one item, all lanes: `tab` holds the n entries the size pass saved; the text goes
// to dst[0, size).  Items whose text fits the staging buffer are assembled there and copied out
// in aligned chunks; larger ones (a few entries around a huge leaf) are written in place.
GGR_DEV int coop_write_item(CoopStage& E, const DecCtx& cx, const U4* tab, u32 n, u8* dst, u32 size) {
  const u32 lane = wp_lane();
  const bool staged = size <= GGR_COOP_STAGE_BUF;
  const u32 pad = wp_align_pad(dst);
  if (n) wp_prefetch(cx.in, tab[0].y);  // entry 0 is the root: vend = end of the item
  wp_copy_wait();  // persistent warps: the previous item's bulk copy has read the staging buffer
  if (lane == 0) {
    E.n_long = 0;
    E.bad = 0;
  }
  WP_SYNC();
  for (u32 i = lane; i < n; i += 32) {
    const U4 a = tab[2 * i], b = tab[2 * i + 1];
    CoopEnt e;
    e.vpos = a.x; e.vend = a.y; e.body = a.z; e.size = a.w;
    e.off = b.x; e.parent = (u16)b.y; e.next = (u16)(b.y >> 16);
    e.fc_msg = (u16)b.z; e.gfield = (u16)(b.z >> 16);
    e.flags = (u16)b.w; e.depth = (u16)(b.w >> 16);
    // two call sites so that the staged one keeps plain shared-memory stores
    const int st = staged ? coop_write_entry(E, cx, e, E.buf + pad) : coop_write_entry(E, cx, e, dst);
    if (st != GST_OK) E.bad = 1;
  }
  WP_SYNC();
  const u32 nl = E.n_long < GGR_COOP_LONG_MAX ? E.n_long : GGR_COOP_LONG_MAX;
  if (staged) {
    for (u32 k = 0; k < nl; k++) {
      u8* d = E.buf + pad + E.ldst[k];
      const u32 len = E.llen[k] & 0x3FFFFFFFu;
      if (E.llen[k] & 0x80000000u) coop_dirty_write(cx.in, E.lsrc[k], E.lsrc[k] + len, d);
      else if (E.llen[k] & 0x40000000u) coop_base64(cx.in, E.lsrc[k], len, d);
      else coop_copy_words(cx.in, E.lsrc[k], d, len);
    }
    WP_SYNC();
    wp_copy_out(E.buf, dst - pad, pad, size);
  } else {
    for (u32 k = 0; k < nl; k++) {
      u8* d = dst + E.ldst[k];
      const u32 len = E.llen[k] & 0x3FFFFFFFu;
      if (E.llen[k] & 0x80000000u) coop_dirty_write(cx.in, E.lsrc[k], E.lsrc[k] + len, d);
      else if (E.llen[k] & 0x40000000u) coop_base64(cx.in, E.lsrc[k], len, d);
      else coop_copy_words(cx.in, E.lsrc[k], d, len);
    }
  }
  return E.bad ? GST_INTERNAL : GST_OK;
}

// ---- item edge of the reply lock-step kernels (the host simulation calls the same functions) ------------------------
// Saved entry tables: the first tier's in fixed slots, COOP_TAB_U4 16-byte words per item; the second tier's in the pool,
// after its header (32 bytes, the bump counter in the first word), at the entry tab_off[item] hands out; nent[item] then
// has COOP_POOLED set.
#define COOP_TAB_U4 (2 * GGR_COOP_TAB_ENTRIES)
#define COOP_POOLED 0x80000000u
template <class P>
GGR_DEV P* coop_pool_table(P* pool, u32 toff) {
  return pool + 2 + 2 * (size_t)toff;
}
GGR_DEV const U4* coop_saved_table(const U4* tab, const U4* pool, const u32* tab_off, u32 nent_word, long long item) {
  return (nent_word & COOP_POOLED) ? coop_pool_table(pool, tab_off[item]) : tab + (size_t)item * COOP_TAB_U4;
}

// k_decode_coop_size: true when the item was sized and its entry table saved (*ne entries; POOLED, the second tier: in
// the pool from entry *toff).  A framed item (GGR_DF_GRPC_FRAME) with a bad header is left to the per-thread kernel,
// which reports it.  Sets cx.in to the item's first 16-byte chunk.
template <class SH, bool POOLED>
GGR_DEV bool coop_size_step(SH& S, DecCtx& cx, u32 n_msgs, const i32* msg_id, const u8* in, const u64* in_off, long long item, U4* tab,
                            U4* pool, u32 pool_cap, u32* ne, u32* sz, u32* toff) {
  u64 a = in_off[item];
  const u64 b = in_off[item + 1];
  const i32 m = msg_id[item];
  bool framed_ok = true;
  if (cx.flags & GGR_DF_GRPC_FRAME) {
    framed_ok = b >= a && ggr_frame_check(in, a, b) == GST_OK;
    a += GGR_FRAME_BYTES;
  }
  bool ok = false;
  if (framed_ok && m >= 0 && (u32)m < n_msgs && b >= a && b - a <= (u64)GGR_REP_ITEM_MAX) {
    cx.in = in + (a & ~15ull);
    const u32 s0 = (u32)(a & 15ull);
    // one instance of the item code per kernel (both would double the hot instruction stream of the first tier)
    if (POOLED)
      ok = coop_size_item(S, cx, (u32)m, s0, s0 + (u32)(b - a), nullptr, ne, sz, coop_pool_table(pool, 0), reinterpret_cast<u32*>(pool),
                          pool_cap, toff);
    else
      ok = coop_size_item(S, cx, (u32)m, s0, s0 + (u32)(b - a), tab + (size_t)item * COOP_TAB_U4, ne, sz);
  }
  return ok;
}

// Lane 0: a sized item's size, mode, status and table; one not sized gets mode PENDING and goes to `left` (if any).
template <bool POOLED>
GGR_DEV void coop_size_publish(bool ok, long long item, u32 sz, u32 ne, u32 toff, u32* size, u32* mode, i32* status, u32* nent,
                               u32* tab_off, GgrWork left) {
  if (wp_lane() != 0) return;
  if (ok) {
    size[item] = sz;
    mode[item] = GGR_MODE_COOP;
    status[item] = GST_OK;
    nent[item] = POOLED ? (ne | COOP_POOLED) : ne;
    if (POOLED) tab_off[item] = toff;
  } else {
    mode[item] = GGR_MODE_PENDING;
    nent[item] = 0;
    if (left.item) left.item[ggr_atomic_add_u32(&left.h->n, 1u)] = (u32)item;
  }
}

// k_decode_coop_write: the text of an item the size pass took, from its saved table; GST_OK for the others.
GGR_DEV int coop_write_step(CoopStage& E, DecCtx& cx, const u8* in, const u64* in_off, const u32* size, const u32* mode, const i32* status,
                            const U4* tab, const u32* nent, const U4* pool, const u32* tab_off, u8* out, const u64* out_off, long long item) {
  if (mode[item] != GGR_MODE_COOP || status[item] != GST_OK) return GST_OK;
  const u64 a = in_off[item] + ((cx.flags & GGR_DF_GRPC_FRAME) ? GGR_FRAME_BYTES : 0u);
  cx.in = in + (a & ~15ull);
  const u32 nw = nent[item];
  return coop_write_item(E, cx, coop_saved_table(tab, pool, tab_off, nw, item), nw & ~COOP_POOLED, out + out_off[item], size[item]);
}

// Lane 0: an item the write pass could not write gets GST_INTERNAL.
GGR_DEV void coop_write_publish(int ws, long long item, i32* status) {
  if (ws != GST_OK && wp_lane() == 0) status[item] = GST_INTERNAL;
}
