// ggr_diag.cuh - error detail of a failing request item, one warp per item (ggr_encode_diagnose_batch[_dev]).
//
// The per-thread parser (k_encode_parse) reports the status of the item and the byte position where it stopped.  From
// those and the item's bytes this file derives what protojson would print, `proto: (line L:C): <what>`:
//   position : clamped to the item's length (0 for an item that parses)
//   key token: when a '"' sits at the position, the raw token up to the next quote that no backslash escapes (quotes
//              included; a byte after a backslash is skipped, and no closing quote means no token)
//   L, C     : line and column of the position, counted in bytes from 1
//   what     : `unknown field <tok>`, `duplicate field <tok>`, `error parsing <tok>, oneof is already set` when a key token
//              was found for those statuses, the status name (ggr_status.h) otherwise
// An item may be 2 MiB long and fail near its end, so the newlines before the position are counted 512 bytes per step:
// one 16-byte load per lane, the counts gathered by ballots.  The same code runs in the host simulation
// (tests/hostsim/diagsim.cc) on 32 fibers.
#pragma once
#include "ggr_status.h"
#include "ggr_warp.cuh"

struct DgItem {
  i32 st;          // status of the re-parse
  u32 pos;         // error position inside the item
  u32 tok;         // length of the key token at pos (0: none)
  u32 line, col;   // of pos, from 1
  u32 len;         // bytes of the text (0 when st == GST_OK)
};

// bit k set: byte k of the 16 is '\n'
GGR_DEV u32 dg_newlines16(U4 v) {
  const u32 w[4] = {v.x, v.y, v.z, v.w};
  u32 m = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u32 t = w[k] ^ 0x0A0A0A0Au;
    const u32 z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t | 0x7F7F7F7Fu);  // 0x80 in every byte of w that is '\n'
    m |= (((z >> 7) & 1u) | ((z >> 14) & 2u) | ((z >> 21) & 4u) | ((z >> 28) & 8u)) << (4 * k);
  }
  return m;
}

GGR_DEV u32 dg_digits(u32 v) {
  u32 d = 1;
  while (v >= 10u) {
    v /= 10u;
    d++;
  }
  return d;
}

GGR_DEV u32 dg_strlen(const char* s) {
  u32 n = 0;
  while (s[n]) n++;
  return n;
}

// what follows the position prefix: the words before the token (or the status name alone), and after it
struct DgWords {
  const char* head;
  const char* tail;
  u32 head_n, tail_n;
  bool tok;  // the key token is printed between head and tail
};
GGR_DEV DgWords dg_words(i32 st, u32 tok) {
  DgWords w;
  w.tail = "";
  w.tail_n = 0;
  w.tok = tok != 0 && (st == GST_UNKNOWN_FIELD || st == GST_DUPLICATE || st == GST_ONEOF);
  if (w.tok && st == GST_UNKNOWN_FIELD) {
    w.head = "unknown field ";
  } else if (w.tok && st == GST_DUPLICATE) {
    w.head = "duplicate field ";
  } else if (w.tok) {
    w.head = "error parsing ";
    w.tail = ", oneof is already set";
    w.tail_n = 22;
  } else {
    w.head = ggr_status_name(st);
  }
  w.head_n = dg_strlen(w.head);
  return w;
}
#define DG_PREFIX "proto: (line "
#define DG_PREFIX_N 13u

// all lanes: the item in[a, b) whose re-parse gave status st and position raw_pos
GGR_DEV DgItem dg_locate(const u8* in, u64 a, u64 b, i32 st, u32 raw_pos) {
  const u32 lane = wp_lane();
  DgItem d;
  d.st = st;
  d.pos = d.tok = d.len = 0;
  d.line = d.col = 1;
  if (st == GST_OK) return d;
  const u64 n = b - a;
  d.pos = (u64)raw_pos < n ? raw_pos : (u32)n;
  // newlines in [a, a + pos): how many, and where the last one is
  const u64 hi = a + d.pos;
  u32 count = 0;
  u64 last = a - 1;  // none yet: the column counts from the item's first byte
  for (u64 base = a & ~15ull; base < hi; base += 512u) {
    const u64 c = base + 16ull * lane;
    u32 m = 0;
    if (c < hi) {
      m = dg_newlines16(ggr_ld16(in + c));
      if (c < a) m &= ~0u << (u32)(a - c);
      if (hi - c < 16u) m &= (1u << (u32)(hi - c)) - 1u;
    }
    const u32 k = wp_popc(m);  // at most 16: five bit planes
    for (u32 bit = 0; bit < 5u; bit++) count += wp_popc(WP_BALLOT((k >> bit) & 1u)) << bit;
    const u32 has = WP_BALLOT(m != 0u);
    if (has) {
      const u32 src = 31u - wp_clz(has);
      const u32 top = WP_SHFL(m ? 31u - wp_clz(m) : 0u, src);
      last = base + 16ull * src + top;
    }
  }
  d.line = 1u + count;
  d.col = (u32)(hi - last);
  // key token: from the quote at pos to the first quote after it that an even run of backslashes precedes
  if (d.pos < n && in[hi] == '"') {
    u32 carry = 0;  // parity of the run of backslashes that ends the window before
    for (u64 q0 = hi + 1u; q0 < b; q0 += 32u) {
      const u64 q = q0 + lane;
      const u32 ch = q < b ? (u32)in[q] : 0u;
      const u32 bs = WP_BALLOT(ch == '\\');
      const u32 other = ~bs & ((1u << lane) - 1u);  // bytes of the window before this lane's that are no backslash
      const u32 odd = other ? (lane - 1u - (31u - wp_clz(other))) & 1u : (lane + carry) & 1u;
      const u32 qm = WP_BALLOT(ch == '"' && !odd);
      if (qm) {
        d.tok = (u32)(q0 + wp_ffs0(qm) + 1u - hi);
        break;
      }
      carry = bs == 0xFFFFFFFFu ? carry : (wp_clz(~bs)) & 1u;
    }
  }
  const DgWords w = dg_words(st, d.tok);
  d.len = DG_PREFIX_N + dg_digits(d.line) + 1u + dg_digits(d.col) + 3u + w.head_n + (w.tok ? d.tok : 0u) + w.tail_n;
  return d;
}

template <class W>
GGR_DEV void dg_put_dec(W& w, u32 v) {
  char s[10];
  int k = 0;
  do {
    s[k++] = (char)('0' + v % 10u);
    v /= 10u;
  } while (v);
  while (k) w.put1((u32)(u8)s[--k]);
}
template <class W>
GGR_DEV void dg_put_str(W& w, const char* s, u32 n) {
  for (u32 i = 0; i < n; i++) w.put1((u32)(u8)s[i]);
}

// all lanes: the d.len bytes of the text to dst (any alignment); lane 0 writes the words, the warp copies the token
GGR_DEV void dg_write(const u8* in, u64 a, const DgItem& d, u8* dst) {
  if (d.len == 0) return;
  const u32 lane = wp_lane();
  const DgWords w = dg_words(d.st, d.tok);
  const u32 at = DG_PREFIX_N + dg_digits(d.line) + 1u + dg_digits(d.col) + 3u + w.head_n;  // where the token goes
  if (lane == 0) {
    Sw o;
    o.init(dst, 0);
    dg_put_str(o, DG_PREFIX, DG_PREFIX_N);
    dg_put_dec(o, d.line);
    o.put1(':');
    dg_put_dec(o, d.col);
    dg_put_str(o, "): ", 3u);
    dg_put_str(o, w.head, w.head_n);
    if (w.tok) {
      o.pos += d.tok;
      dg_put_str(o, w.tail, w.tail_n);
    }
  }
  if (w.tok)
    for (u32 j = lane; j < d.tok; j += 32u) dst[at + j] = in[a + d.pos + j];
}
