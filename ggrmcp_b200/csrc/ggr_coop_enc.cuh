// ggr_coop_enc.cuh - lock-step request side, pass A: one warp per item, JSON arguments -> IR.
//
// The per-thread parser (ggr_encode.cuh) spends 32 unrelated state machines per warp; here the 32
// lanes of a warp work on ONE item and execute the same code on different data:
//   T1 tokenize : every lane classifies one 16-byte chunk per round with bit masks (quotes,
//                 backslashes, structural characters, white space), the in-string state is carried
//                 across lanes by ballots; the result is a structural index in shared memory
//                 (one entry per { } [ ] : , string and scalar literal) plus the list of quotes
//   T2 match    : bracket matching by level (prefix counts + match_any), 32 tokens per round
//   T3 walk     : level by level, one lane per JSON object: resolves member names against the
//                 descriptor tables, appends one node per value (children kept in wire-emit order,
//                 which is also how duplicates are caught), nested objects are queued for the
//                 next level and skipped in O(1) through the bracket index
//   T4 leaves   : leaf nodes bucketed by kind, then one lane per leaf runs the very same scalar
//                 parsers as the per-thread path (parse_scalar), so accepted values are identical
//   T5 sizes    : bottom-up by depth, containers add their finished size to their parent
// The output is the same IR (ggr_encode.cuh) the per-thread parser writes, so pass B
// (k_encode_emit) is shared.  Only regular input is handled: any anomaly - syntax or type error,
// unknown or duplicate field, non-string map key, table overflow - sets `bail` and the item is left,
// untouched, to the next tier (the same code with larger tables, then the per-thread parser, which
// owns the error semantics).
#pragma once
#include "ggr_encode.cuh"
#include "ggr_warp.cuh"

#define CE_MAX_DEPTH 24
#define CE_MAX_INPUT 65000u
static_assert(GGR_REQ_ITEM_MAX + 15u <= CE_MAX_INPUT, "a taken item ends by CE_MAX_INPUT at every offset within its chunk");
#define CE_NIL 0xFFFFu
#define NF_SIMPLE 2u /* N_STR with NF_ESC: only two-character escapes (the tokenizer's O(1) sizing) */

enum { TK_LBRACE = 1, TK_RBRACE = 2, TK_LBRACK = 3, TK_RBRACK = 4, TK_COLON = 5, TK_COMMA = 6, TK_STR = 7, TK_SCALAR = 8 };
#define TK_POS(t) ((t) & 0xFFFFu)
#define TK_KIND(t) (((t) >> 16) & 0xFu)
#define TK_AUX(t) ((t) >> 20)

// node classes: containers first; everything >= CC_NULL is finished in the leaf phase
enum { CC_MSG = 0, CC_LIST = 1, CC_MAP = 2, CC_ENTRY = 3, CC_NULL = 4, CC_STR = 5, CC_BYTES = 6, CC_INT = 7, CC_FLOAT = 8, CC_TS = 9, CC_N = 10 };

struct CNode {       // 20 bytes
  u16 tok;           // token index of the value
  u16 parent;
  u16 next;          // next sibling in emit order (lists: document order)
  u16 head;          // containers: first child
  u16 emit;          // emit index within the parent message
  u16 gfield;        // global field index
  u16 msg;           // CC_MSG: message type
  u8 cls, depth;
  u32 body;          // containers: payload bytes accumulated from the children (their header length
                     // goes to `tok` once they are closed); leaves: bytes in the parent's payload
};

// Per-warp working set (shared memory).  MT tokens / MQ quotes / MN nodes; aux is 12 bits, so
// MT, MQ <= 4096.
template <int MT, int MQ, int MN>
struct CoopEncT {
  static const u32 MAX_TOK = MT, MAX_Q = MQ, MAX_NODE = MN;
  u32 tok[MT];     // pos(16) | kind(4) | aux(12): aux = matching bracket / index into qpos
  u16 qpos[MQ];    // positions of all unescaped quotes, in order
  u16 qesc[MQ];    // number of simple escape sequences (\" \\ \/ \b \f \n \r \t) before each quote, mod 2^16
  u16 qslow[MQ];   // number of bytes that need the full scanner (< 0x20, \u, bad escape) before each quote
  CNode node[MN];
  u16 order[MN];
  u16 queue[MN];
  u16 last_open[32];
  u32 cls_cnt[CC_N], cls_cur[CC_N];
  u32 dep_beg[CE_MAX_DEPTH + 2], dep_cur[CE_MAX_DEPTH + 2];  // containers bucketed by depth (in `queue`)
  u32 n_tok, n_q, n_node, q_end, n_leaf, max_depth, bail, cap;
  // envelope mode: brackets nested deeper than the validators allow; what the envelope walk found
  u32 deep, env, env_method, env_msg, env_args_tok, env_id_pos, env_id_len;
  // sink interface of ce_tokenize
  static const bool STRUCT_KINDS = false;  // structural characters: kind filled in by ce_match
  GGR_DEV void set_bail() { bail = 1; }
  GGR_DEV void put_q(u32 qi, u32 pos, u32 esc, u32 slow) {
    if (qi < MAX_Q) {
      qpos[qi] = (u16)pos;
      qesc[qi] = (u16)esc;
      qslow[qi] = (u16)slow;
    }
  }
  GGR_DEV void put_tok(u32 ti, u32 v) {
    if (ti < MAX_TOK) tok[ti] = v;
  }
  GGR_DEV void finish(u32 nt, u32 nq, bool fail) {
    n_tok = nt;
    n_q = nq;
    if (fail || nt > MAX_TOK || nq > MAX_Q) bail = 1;
  }
};
typedef CoopEncT<1024, 512, 224> CoopEnc;        // tier 1: ~12 KB per warp
typedef CoopEncT<2048, 1024, 512> CoopEncBig;   // tier 2: ~26 KB per warp (two blocks of four warps per SM)

// Working set of the token-index kernel (k_encode_coop_tok): what ce_tokenize / ce_match touch.  Tier 1
// runs T1 + T2 in a kernel of their own (small code, half the registers and shared memory of the
// walker, so twice the warps per SM); the index travels through the item's IR region, which the
// walker only starts to fill after it has copied the index into its own shared memory.
template <int MT, int MQ>
struct CoopTokT {
  static const u32 MAX_TOK = MT, MAX_Q = MQ;
  u32 tok[MT];
  u16 qpos[MQ], qesc[MQ], qslow[MQ];
  u16 last_open[32];
  u32 n_tok, n_q, bail, deep;
  static const bool STRUCT_KINDS = false;
  GGR_DEV void set_bail() { bail = 1; }
  GGR_DEV void put_q(u32 qi, u32 pos, u32 esc, u32 slow) {
    if (qi < MAX_Q) {
      qpos[qi] = (u16)pos;
      qesc[qi] = (u16)esc;
      qslow[qi] = (u16)slow;
    }
  }
  GGR_DEV void put_tok(u32 ti, u32 v) {
    if (ti < MAX_TOK) tok[ti] = v;
  }
  GGR_DEV void finish(u32 nt, u32 nq, bool fail) {
    n_tok = nt;
    n_q = nq;
    if (fail || nt > MAX_TOK || nq > MAX_Q) bail = 1;
  }
};
typedef CoopTokT<1024, 512> CoopTok;  // same limits as CoopEnc
// header {n_tok, n_q, bail, deep}, tok[n_tok], then qpos / qesc / qslow as (n_q + 1) / 2 words each
GGR_DEV u32 ce_tok_bytes(u32 n_tok, u32 n_q) { return 16u + 4u * n_tok + 12u * ((n_q + 1u) >> 1); }

struct CeLut {
  u32 cls[256];  // CE_L* class bits
  u8 kind[256];  // TK_* of the structural characters; bit 7: valid character after a backslash (simple escapes)
};

// byte classes for the tokenizer, one byte lane per class so that eight bytes accumulate in one word
#define CE_LQ 0x00000001u
#define CE_LB 0x00000100u
#define CE_LS 0x00010000u
#define CE_LW 0x01000000u
GGR_DEV u32 ce_class(u32 b) {
  if (b == '"') return CE_LQ;
  if (b == '\\') return CE_LB;
  if (b == '{' || b == '}' || b == '[' || b == ']' || b == ':' || b == ',') return CE_LS;
  if (b == ' ' || b == '\t' || b == '\n' || b == '\r') return CE_LW;
  return 0;
}

// Escaped positions of a 16-byte chunk from its backslash mask (the branch-free run-parity
// computation simdjson uses, on 16 bits); cin: the first byte is escaped by the previous chunk.
GGR_DEV u32 ce_escaped(u32 B, u32 cin, u32* cout) {
  B &= ~cin;
  u32 follows = (B << 1) | cin;
  const u32 EVEN = 0x5555u;
  u32 odd_starts = B & ~EVEN & ~follows;
  u32 sum = odd_starts + B;
  *cout = (sum >> 16) & 1u;
  return (EVEN ^ (sum << 1)) & follows & 0xFFFFu;
}
GGR_DEV u32 ce_prefix_xor16(u32 x) {
  x ^= x << 1;
  x ^= x << 2;
  x ^= x << 4;
  x ^= x << 8;
  return x & 0xFFFFu;
}
GGR_DEV u32 ce_struct_kind(u32 c) {
  return c == '{' ? TK_LBRACE : c == '}' ? TK_RBRACE : c == '[' ? TK_LBRACK : c == ']' ? TK_RBRACK : c == ':' ? TK_COLON : c == ',' ? TK_COMMA : 0;
}
// the same for a byte known to be one of { } [ ] : , - from its bits: 0x04 closes, 0x20 braces, < 0x40 colon / comma
GGR_DEV u32 ce_struct_kind_bits(u32 c) {
  return c < 0x40u ? (c == ':' ? (u32)TK_COLON : (u32)TK_COMMA) : 1u + ((c >> 2) & 1u) + ((((c >> 5) & 1u) ^ 1u) << 1);
}
GGR_DEV void ce_lut_init(CeLut& L, u32 first, u32 step) {
  for (u32 b = first; b < 256; b += step) {
    L.cls[b] = ce_class(b);
    bool simple = b == '"' || b == '\\' || b == '/' || b == 'b' || b == 'f' || b == 'n' || b == 'r' || b == 't';
    L.kind[b] = (u8)(ce_struct_kind(b) | (simple ? 0x80u : 0u));
  }
}
// flags in bit 7 of every byte -> 4 contiguous bits
GGR_DEV u32 ce_pack4(u32 x) { return (((x >> 7) * 0x00204081u) >> 21) & 0xFu; }
// per byte of w (bit 7 flags): control character (< 0x20)
GGR_DEV u32 ce_ctrl_flags(u32 w) {
  u32 ge20 = ((w & 0x7F7F7F7Fu) + 0x60606060u) | w;  // bit 7 set: byte >= 0x20
  return ~ge20 & 0x80808080u;
}
GGR_DEV u32 ce_byte16(const U4& v, u32 j) {  // byte j of a 16-byte chunk
  u32 w = j < 4 ? v.x : j < 8 ? v.y : j < 12 ? v.z : v.w;
  return (w >> (8 * (j & 3u))) & 0xFFu;
}

// T1.  All lanes.  lut: 256-entry class table (shared memory on the device).
template <class SH>
GGR_DEV void ce_tokenize(SH& S, const CeLut& L, const u8* in, u32 start, u32 end) {
  const u32* lut = L.cls;
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u;
  const u32 nchunks = (end + 15u) >> 4;
  u32 c_carry = 0, in_carry = 0, n_carry = 0, u_carry = 0;  // warp-uniform carries between rounds
  u32 tbase = 0, qbase = 0, dbase = 0, ebase = 0;
  U4 vn;  // the next round's chunk is requested one round ahead
  vn.x = vn.y = vn.z = vn.w = 0;
  if (lane < nchunks) vn = ggr_ld16(in + (lane << 4));
  for (u32 cb = 0; cb < nchunks; cb += 32) {
    const u32 ci = cb + lane;
    const u32 off = ci << 4;
    u32 Q = 0, B = 0, X = 0, W = 0xFFFFu, D = 0, HI = 0;
    const U4 v = vn;
    vn.x = vn.y = vn.z = vn.w = 0;
    if (ci + 32u < nchunks) vn = ggr_ld16(in + off + 512u);
    if (ci < nchunks) {
      u32 lo = 0, hi = 0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        lo |= lut[(v.x >> (8 * j)) & 0xFFu] << j;
        lo |= lut[(v.y >> (8 * j)) & 0xFFu] << (j + 4);
        hi |= lut[(v.z >> (8 * j)) & 0xFFu] << j;
        hi |= lut[(v.w >> (8 * j)) & 0xFFu] << (j + 4);
      }
      Q = (lo & 0xFFu) | ((hi & 0xFFu) << 8);
      B = ((lo >> 8) & 0xFFu) | (((hi >> 8) & 0xFFu) << 8);
      X = ((lo >> 16) & 0xFFu) | (((hi >> 16) & 0xFFu) << 8);
      W = ((lo >> 24) & 0xFFu) | (((hi >> 24) & 0xFFu) << 8);
      // bytes outside [start, end) count as white space
      u32 valid = 0xFFFFu;
      if (off < start) valid &= 0xFFFFu << (start - off);
      if (off + 16u > end) valid &= 0xFFFFu >> (off + 16u - end);
      Q &= valid;
      B &= valid;
      X &= valid;
      W = (W | ~valid) & 0xFFFFu;
      D = (ce_pack4(ce_ctrl_flags(v.x)) | (ce_pack4(ce_ctrl_flags(v.y)) << 4) | (ce_pack4(ce_ctrl_flags(v.z)) << 8) |
           (ce_pack4(ce_ctrl_flags(v.w)) << 12)) & valid;
      HI = (ce_pack4(v.x & 0x80808080u) | (ce_pack4(v.y & 0x80808080u) << 4) | (ce_pack4(v.z & 0x80808080u) << 8) |
            (ce_pack4(v.w & 0x80808080u) << 12)) & valid;
    }
    // UTF-8 over the whole text (structure and quotes are ASCII, so a malformed sequence anywhere
    // makes the item an error: left to the per-thread parser).  Lead bytes say where continuation
    // bytes must be; that mask, carried over the chunk boundary, has to equal the actual one.
    if (WP_ANY(HI != 0) || u_carry) {
      u32 C6 = 0, EC = 0;
      if (HI) {
        C6 = (ce_pack4((v.x << 1) & 0x80808080u) | (ce_pack4((v.y << 1) & 0x80808080u) << 4) |
              (ce_pack4((v.z << 1) & 0x80808080u) << 8) | (ce_pack4((v.w << 1) & 0x80808080u) << 12));
        for (u32 m = HI & C6; m; m &= m - 1u) {  // lead bytes (11xxxxxx)
          const u32 j = wp_ffs0(m);
          const u32 b0 = ce_byte16(v, j);
          const u32 b1 = j < 15 ? ce_byte16(v, j + 1) : (ggr_ld4(in + off + 16) & 0xFFu);
          u32 len = b0 < 0xC2u ? 0u : b0 < 0xE0u ? 2u : b0 < 0xF0u ? 3u : b0 < 0xF5u ? 4u : 0u;
          if ((b0 == 0xE0u && b1 < 0xA0u) || (b0 == 0xEDu && b1 >= 0xA0u) || (b0 == 0xF0u && b1 < 0x90u) || (b0 == 0xF4u && b1 >= 0x90u)) len = 0;
          if (len == 0) S.set_bail();
          else EC |= ((1u << (len - 1u)) - 1u) << (j + 1u);
        }
      }
      u32 ci = WP_SHFL_UP(EC >> 16, 1);
      if (lane == 0) ci = u_carry;
      u_carry = WP_SHFL(EC >> 16, 31);
      if (((EC & 0xFFFFu) | ci) != (HI & ~C6)) S.set_bail();
    }
    // escaped bytes: the carry into a chunk only matters through an all-backslash chunk
    u32 E = 0;
    if (WP_ANY(B != 0) || c_carry) {  // most rounds hold no backslash at all
      u32 co0, co1;
      u32 E0 = ce_escaped(B, 0, &co0);
      u32 E1 = ce_escaped(B, 1, &co1);
      u32 Pm = WP_BALLOT(co0 != co1);
      u32 Gm = WP_BALLOT(co0 != 0);
      u32 np = ~Pm & lt;
      u32 cin = np ? ((Gm >> (31u - wp_clz(np))) & 1u) : c_carry;
      E = cin ? E1 : E0;
      u32 cout = cin ? co1 : co0;
      c_carry = WP_SHFL(cout, 31);
    }
    u32 RQ = Q & ~E;
    // escape sequences: introducers, and escaped characters outside the simple set (incl. \u)
    const u32 EI = B & ~E;
    for (u32 m = E; m; m &= m - 1u) {
      u32 j = wp_ffs0(m);
      if (!(L.kind[ce_byte16(v, j)] & 0x80u)) D |= 1u << j;
    }
    // in-string state at the start of the chunk
    u32 PB = WP_BALLOT((wp_popc(RQ) & 1u) != 0);
    u32 in0 = (wp_popc(PB & lt) + in_carry) & 1u;
    in_carry = (in_carry + wp_popc(PB)) & 1u;
    u32 IS = ce_prefix_xor16(RQ) ^ (in0 ? 0xFFFFu : 0u);  // opening quote and content; closing quote excluded
    u32 SO = RQ & IS, SC = RQ & ~IS;
    u32 ST = X & ~IS;
    u32 N = ~(W | X | IS | SC) & 0xFFFFu;  // bytes of scalar literals
    u32 pn = WP_SHFL_UP(N >> 15, 1);
    if (lane == 0) pn = n_carry;
    n_carry = WP_SHFL(N >> 15, 31);
    u32 NS = N & ~((N << 1) | pn);
    u32 T = ST | SO | NS;
    u32 tot;
    // counters carried by prefix scans: tokens, quotes / escape introducers, slow bytes (each at most 512 per round)
    u32 ex = WP_EXCL_SCAN(wp_popc(T) | (wp_popc(RQ) << 16), &tot);
    u32 ti = tbase + (ex & 0xFFFFu), qi = qbase + (ex >> 16);
    tbase += tot & 0xFFFFu;
    qbase += tot >> 16;
    u32 ei = ebase, di = dbase;
    if (WP_ANY((EI | D) != 0)) {  // most rounds hold neither escapes nor bytes for the full scanner
      u32 tot2;
      const u32 ex2 = WP_EXCL_SCAN(wp_popc(EI) | (wp_popc(D) << 16), &tot2);
      ei += ex2 & 0xFFFFu;
      di += ex2 >> 16;
      ebase += tot2 & 0xFFFFu;
      dbase += tot2 >> 16;
    }
    const u32 qi0 = qi;
    for (u32 m = RQ; m; m &= m - 1u) {
      u32 j = wp_ffs0(m);
      S.put_q(qi, off + j, ei + wp_popc(EI & ((1u << j) - 1u)), di + wp_popc(D & ((1u << j) - 1u)));
      qi++;
    }
    for (u32 m = T; m; m &= m - 1u) {
      u32 j = wp_ffs0(m), bit = 1u << j;
      u32 kind, aux = 0;
      if (SO & bit) {
        kind = TK_STR;
        aux = qi0 + wp_popc(RQ & (bit - 1u));
      } else if (NS & bit) {
        kind = TK_SCALAR;
      } else {
        // structural character: ce_match looks it up (one lane per token there) unless the sink wants it now
        kind = SH::STRUCT_KINDS ? ce_struct_kind_bits(ce_byte16(v, j)) : 0u;
      }
      S.put_tok(ti, (off + j) | (kind << 16) | (aux << 20));
      ti++;
    }
  }
  if (lane == 0) S.finish(tbase, qbase, in_carry || u_carry || tbase == 0);
  WP_SYNC();
}

// T2.  All lanes.  Fills the aux field of every bracket token with the index of its partner.
template <class SH>
GGR_DEV void ce_match(SH& S, const CeLut& L, const u8* in) {
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u, le = lt | (1u << lane);
  const u32 n = S.n_tok;
  i32 depth = 0;
  for (u32 base = 0; base < n; base += 32) {
    const u32 i = base + lane;
    u32 t = i < n ? S.tok[i] : (TK_SCALAR << 16);
    if (TK_KIND(t) == 0) {  // structural character left open by the tokenizer
      t |= (u32)(L.kind[in[TK_POS(t)]] & 0xFu) << 16;
      S.tok[i] = t;
    }
    WP_SYNC();  // closing brackets read their partner's kind below
    const u32 k = TK_KIND(t);
    const bool op = k == TK_LBRACE || k == TK_LBRACK, cl = k == TK_RBRACE || k == TK_RBRACK;
    const u32 OM = WP_BALLOT(op), CM = WP_BALLOT(cl);
    // level of an opening bracket: depth after it; of a closing bracket: depth before it
    const i32 lvl = depth + (i32)wp_popc(OM & le) - (i32)wp_popc(CM & lt);
    const bool bad = (op || cl) && (lvl < 1 || lvl >= 32);
    if (op && lvl > 10) S.deep = 1;  // envelope mode: validateDepth (pkg/mcp/validation.go:163-184) might refuse
    const u32 m = WP_MATCH_ANY((op || cl) ? (u32)lvl : 0x10000u + lane);
    if (bad) S.bail = 1;
    if (cl && !bad) {
      u32 cand = m & OM & lt;
      u32 mt = cand ? base + 31u - wp_clz(cand) : (u32)S.last_open[lvl];
      if (mt >= i || TK_KIND(S.tok[mt]) + 1u != k) {
        S.bail = 1;
      } else {
        S.tok[i] = t | (mt << 20);
        S.tok[mt] |= i << 20;
      }
    }
    WP_SYNC();
    if (op && !bad && (m & OM & ~le) == 0) S.last_open[lvl] = (u16)i;
    WP_SYNC();
    depth += (i32)wp_popc(OM) - (i32)wp_popc(CM);
    if (depth < 0) depth = 0;  // already flagged by the lane that underflowed
  }
  if (depth != 0 && lane == 0) S.bail = 1;
  WP_SYNC();
}

template <class SH>
GGR_DEV u32 ce_new_node(SH& S, u32 tok, u32 parent, u32 gfield, u32 emit, u32 cls, u32 depth) {
  u32 idx = wp_atomic_add(&S.n_node, 1u);
  if (idx >= S.cap || gfield >= 0xFFFFu || emit >= 0xFFFu) {
    S.bail = 1;
    return CE_NIL;
  }
  CNode nd;
  nd.tok = (u16)tok;
  nd.parent = (u16)parent;
  nd.next = CE_NIL;
  nd.head = CE_NIL;
  nd.emit = (u16)emit;
  nd.gfield = (u16)gfield;
  nd.msg = 0;
  nd.cls = (u8)cls;
  nd.depth = (u8)depth;
  nd.body = 0;
  S.node[idx] = nd;
  return idx;
}
GGR_DEV u32 ce_leaf_class(const FieldD& f, bool timestamp) {
  if (timestamp) return CC_TS;
  switch (f.kind) {
    case GK_STRING: return CC_STR;
    case GK_BYTES: return CC_BYTES;
    case GK_FLOAT: case GK_DOUBLE: return CC_FLOAT;
    default: return CC_INT;
  }
}
// `null`, exactly, followed by a delimiter
GGR_DEV bool ce_is_null(const EncCtx& cx, u32 pos) {
  const u8* p = cx.in + pos;
  if (p[0] != 'n') return false;
  if (cx.end - pos < 4u || p[1] != 'u' || p[2] != 'l' || p[3] != 'l') return false;
  if (pos + 4u >= cx.end) return true;
  const u32 c = p[4];
  return ggr_is_ws(c) || c == ',' || c == '}' || c == ']';
}

// KeyInfo of a string token known to hold no escapes and valid UTF-8 (tokenizer counts): plain
// bytes [pos + 1, close)
GGR_DEV void ce_key_info_plain(const u8* in, u32 pos, u32 close, KeyInfo* k) {
  const u8* p = in + pos + 1u;
  const u32 n = close - pos - 1u;
  u32 h = GGR_KHASH_SEED;
  u32 w0 = 0, w1 = 0, w2 = 0, w3 = 0;
  const u32 nw = (n + 3u) >> 2;
  for (u32 i = 0; i < nw; i++) {
    const u32 base = i << 2;
    u32 x = p[base];
    if (base + 1u < n) x |= (u32)p[base + 1u] << 8;
    if (base + 2u < n) x |= (u32)p[base + 2u] << 16;
    if (base + 3u < n) x |= (u32)p[base + 3u] << 24;
    h = khash_mix(h, x);
    if (i == 0) w0 = x;
    else if (i == 1) w1 = x;
    else if (i == 2) w2 = x;
    else if (i == 3) w3 = x;
  }
  k->len = n;
  k->hash = khash_finish(h, n);
  k->w[0] = w0;
  k->w[1] = w1;
  k->w[2] = w2;
  k->w[3] = w3;
}

// T3, one lane: members of the JSON object behind message node `ni`.
template <class SH>
GGR_DEV void ce_walk_object(SH& S, const EncCtx& cx, u32 ni) {
  const Tables& T = cx.T;
  const u32 open = S.node[ni].tok;
  const u32 depth = S.node[ni].depth;
  const MsgD md = ggr_msg(T, S.node[ni].msg);
  if (md.wkt != GGR_WKT_NONE || depth + 2u >= CE_MAX_DEPTH) { S.bail = 1; return; }
  const u32 close = TK_AUX(S.tok[open]);
  u32 head = CE_NIL, tail = CE_NIL, tail_emit = 0, oneofs = 0;
  u32 t = open + 1;
  bool first = true;
  while (t != close) {
    if (!first) {
      if (TK_KIND(S.tok[t]) != TK_COMMA) { S.bail = 1; return; }
      t++;
    }
    first = false;
    // "key" : value
    if (t + 2u >= close) { S.bail = 1; return; }
    const u32 kt = S.tok[t];
    if (TK_KIND(kt) != TK_STR || TK_KIND(S.tok[t + 1]) != TK_COLON) { S.bail = 1; return; }
    const u32 key_pos = TK_POS(kt);
    KeyInfo ki;
    {
      const u32 kq = TK_AUX(kt);
      if (S.qslow[kq] == S.qslow[kq + 1] && S.qesc[kq] == S.qesc[kq + 1]) {
        ce_key_info_plain(cx.in, key_pos, S.qpos[kq + 1], &ki);
      } else {
        Rd r;
        r.init(cx.in, key_pos, cx.end);
        if (scan_key(r, &ki) != GST_OK) { S.bail = 1; return; }
      }
    }
    i32 ei;
    if (!hash_lookup(T, md.key_hash_first, md.key_hash_mask, ki, cx.in, key_pos, cx.end, &ei)) { S.bail = 1; return; }
    const u32 emit = (u32)ei;
    const u32 gf = md.field_first + emit;
    const FieldD f = ggr_field(T, gf);
    t += 2;
    const u32 vt = S.tok[t];
    const u32 vk = TK_KIND(vt);
    u32 child;
    if (vk == TK_SCALAR && ce_is_null(cx, TK_POS(vt))) {
      child = ce_new_node(S, t, ni, gf, emit, CC_NULL, depth + 1);
      t++;
    } else if (f.flags & GF_MAP) {
      if (vk != TK_LBRACE) { S.bail = 1; return; }
      child = ce_new_node(S, t, ni, gf, emit, CC_MAP, depth + 1);
      if (child == CE_NIL) return;
      S.queue[wp_atomic_add(&S.q_end, 1u)] = (u16)child;
      t = TK_AUX(vt) + 1u;
    } else if (f.flags & GF_REPEATED) {
      if (vk != TK_LBRACK) { S.bail = 1; return; }
      const u32 aend = TK_AUX(vt);
      child = ce_new_node(S, t, ni, gf, emit, CC_LIST, depth + 1);
      if (child == CE_NIL) return;
      bool ts = false, msg = false;
      if (f.kind == GK_MESSAGE) {
        u32 w = ggr_msg(T, (u32)f.child).wkt;
        ts = w == GGR_WKT_TIMESTAMP;
        msg = w == GGR_WKT_NONE;
        if (!ts && !msg) { S.bail = 1; return; }
      }
      const u32 lcls = ce_leaf_class(f, ts);
      u32 u = t + 1, ltail = CE_NIL;
      bool lfirst = true;
      while (u != aend) {
        if (!lfirst) {
          if (TK_KIND(S.tok[u]) != TK_COMMA) { S.bail = 1; return; }
          u++;
          if (u == aend) { S.bail = 1; return; }
        }
        lfirst = false;
        const u32 et = S.tok[u];
        const u32 ek = TK_KIND(et);
        u32 el;
        if (msg) {
          if (ek != TK_LBRACE) { S.bail = 1; return; }
          el = ce_new_node(S, u, child, gf, 0, CC_MSG, depth + 2);
          if (el == CE_NIL) return;
          S.node[el].msg = (u16)f.child;
          S.queue[wp_atomic_add(&S.q_end, 1u)] = (u16)el;
          u = TK_AUX(et) + 1u;
        } else {
          if (ek != TK_STR && ek != TK_SCALAR) { S.bail = 1; return; }
          if (ek == TK_SCALAR && ce_is_null(cx, TK_POS(et))) { S.bail = 1; return; }
          el = ce_new_node(S, u, child, gf, 0, lcls, depth + 2);
          if (el == CE_NIL) return;
          u++;
        }
        if (ltail == CE_NIL) S.node[child].head = (u16)el;
        else S.node[ltail].next = (u16)el;
        ltail = el;
      }
      wp_atomic_max(&S.max_depth, depth + 2);
      t = aend + 1;
    } else {
      if (f.oneof >= 0) {
        u32 bit = 1u << (f.oneof & 31);
        if (oneofs & bit) { S.bail = 1; return; }
        oneofs |= bit;
      }
      if (f.kind == GK_MESSAGE) {
        u32 w = ggr_msg(T, (u32)f.child).wkt;
        if (w == GGR_WKT_TIMESTAMP) {
          if (vk != TK_STR) { S.bail = 1; return; }
          child = ce_new_node(S, t, ni, gf, emit, CC_TS, depth + 1);
          t++;
        } else if (w == GGR_WKT_NONE) {
          if (vk != TK_LBRACE || (u32)f.child >= 0xFFFFu) { S.bail = 1; return; }
          child = ce_new_node(S, t, ni, gf, emit, CC_MSG, depth + 1);
          if (child == CE_NIL) return;
          S.node[child].msg = (u16)f.child;
          S.queue[wp_atomic_add(&S.q_end, 1u)] = (u16)child;
          t = TK_AUX(vt) + 1u;
        } else {
          S.bail = 1;
          return;
        }
      } else {
        if (vk != TK_STR && vk != TK_SCALAR) { S.bail = 1; return; }
        child = ce_new_node(S, t, ni, gf, emit, ce_leaf_class(f, false), depth + 1);
        t++;
      }
    }
    if (child == CE_NIL) return;
    if (t > close) { S.bail = 1; return; }
    // children in emit order; equal emit = the same field twice
    if (head == CE_NIL) {
      head = tail = child;
      tail_emit = emit;
    } else if (emit > tail_emit) {
      S.node[tail].next = (u16)child;
      tail = child;
      tail_emit = emit;
    } else if (emit == tail_emit) {
      S.bail = 1;
      return;
    } else {
      u32 prev = CE_NIL, cur = head;
      for (;;) {
        u32 e = S.node[cur].emit;
        if (e == emit) { S.bail = 1; return; }
        if (e > emit) break;
        prev = cur;
        cur = S.node[cur].next;
      }
      S.node[child].next = (u16)cur;
      if (prev == CE_NIL) head = child;
      else S.node[prev].next = (u16)child;
    }
  }
  S.node[ni].head = (u16)head;
  wp_atomic_max(&S.max_depth, depth + 1);
}

// T3, one lane: entries of the JSON object behind map node `ni` (string keys only).  Every entry
// becomes ENTRY{key leaf, value}; entries are kept in key order (decoded bytes, as Go compares
// strings), equal keys are left to the per-thread path.
template <class SH>
GGR_DEV void ce_walk_map(SH& S, const EncCtx& cx, u32 ni) {
  const Tables& T = cx.T;
  const u32 open = S.node[ni].tok;
  const u32 depth = S.node[ni].depth;
  const u32 mgf = S.node[ni].gfield;
  const FieldD mapf = ggr_field(T, mgf);
  const MsgD ed = ggr_msg(T, (u32)mapf.child);
  const u32 kgf = ed.field_first, vgf = ed.field_first + 1u;
  const FieldD kf = ggr_field(T, kgf);
  const FieldD vf = ggr_field(T, vgf);
  if (kf.kind != GK_STRING || depth + 3u >= CE_MAX_DEPTH) { S.bail = 1; return; }
  bool ts = false, msg = false;
  if (vf.kind == GK_MESSAGE) {
    u32 w = ggr_msg(T, (u32)vf.child).wkt;
    ts = w == GGR_WKT_TIMESTAMP;
    msg = w == GGR_WKT_NONE;
    if ((!ts && !msg) || (u32)vf.child >= 0xFFFFu) { S.bail = 1; return; }
  }
  const u32 vcls = ce_leaf_class(vf, ts);
  const u32 close = TK_AUX(S.tok[open]);
  u32 head = CE_NIL, tail = CE_NIL, tail_key = 0;
  u32 t = open + 1;
  bool first = true;
  while (t != close) {
    if (!first) {
      if (TK_KIND(S.tok[t]) != TK_COMMA) { S.bail = 1; return; }
      t++;
    }
    first = false;
    if (t + 2u >= close) { S.bail = 1; return; }
    const u32 kt = S.tok[t];
    if (TK_KIND(kt) != TK_STR || TK_KIND(S.tok[t + 1]) != TK_COLON) { S.bail = 1; return; }
    const u32 key_pos = TK_POS(kt);
    const u32 vt = S.tok[t + 2];
    const u32 vk = TK_KIND(vt);
    const u32 ent = ce_new_node(S, t, ni, mgf, 0, CC_ENTRY, depth + 1);
    const u32 key = ce_new_node(S, t, ent, kgf, 0, CC_STR, depth + 2);
    if (ent == CE_NIL || key == CE_NIL) return;
    u32 val;
    if (msg) {
      if (vk != TK_LBRACE) { S.bail = 1; return; }
      val = ce_new_node(S, t + 2, ent, vgf, 1, CC_MSG, depth + 2);
      if (val == CE_NIL) return;
      S.node[val].msg = (u16)vf.child;
      S.queue[wp_atomic_add(&S.q_end, 1u)] = (u16)val;
      t = TK_AUX(vt) + 1u;
    } else {
      if (vk != TK_STR && vk != TK_SCALAR) { S.bail = 1; return; }
      if (vk == TK_SCALAR && ce_is_null(cx, TK_POS(vt))) { S.bail = 1; return; }
      val = ce_new_node(S, t + 2, ent, vgf, 1, vcls, depth + 2);
      if (val == CE_NIL) return;
      t += 3;
    }
    if (t > close) { S.bail = 1; return; }
    S.node[ent].head = (u16)key;
    S.node[key].next = (u16)val;
    if (head == CE_NIL) {
      head = tail = ent;
      tail_key = key_pos;
    } else {
      int c = cmp_str_tokens(cx.in, key_pos, tail_key, cx.end);
      if (c == 0) { S.bail = 1; return; }
      if (c > 0) {
        S.node[tail].next = (u16)ent;
        tail = ent;
        tail_key = key_pos;
      } else {
        u32 prev = CE_NIL, cur = head;
        for (;;) {
          int cc = cmp_str_tokens(cx.in, key_pos, TK_POS(S.tok[S.node[cur].tok]), cx.end);
          if (cc == 0) { S.bail = 1; return; }
          if (cc < 0) break;
          prev = cur;
          cur = S.node[cur].next;
        }
        S.node[ent].next = (u16)cur;
        if (prev == CE_NIL) head = ent;
        else S.node[prev].next = (u16)ent;
      }
    }
  }
  S.node[ni].head = (u16)head;
  wp_atomic_max(&S.max_depth, depth + 2);
}

// ---- request envelope (SURVEY rows A1-A4): {"jsonrpc":"2.0","id":..,"method":"tools/call",
// "params":{"name":"<tool>","arguments":{..}}} ----
// plain string token (no escapes, valid UTF-8) equal to a literal
template <class SH>
GGR_DEV bool ce_tok_is(const SH& S, const u8* in, u32 tk, const char* lit, u32 n) {
  const u32 k = TK_AUX(tk);
  if (S.qslow[k] != S.qslow[k + 1] || S.qesc[k] != S.qesc[k + 1]) return false;
  const u32 pos = TK_POS(tk);
  if ((u32)S.qpos[k + 1] - pos - 1u != n) return false;
  for (u32 j = 0; j < n; j++)
    if (in[pos + 1u + j] != (u8)lit[j]) return false;
  return true;
}
// One lane.  Handles exactly the bodies for which handler.go:83-95,215-231 + pkg/mcp/validation.go
// accept the request AND json.Marshal(arguments) cannot change what protojson sees (together with
// the checks in the walker and the leaf phase): every key once, exact-case names, id a plain ASCII
// string or an integer of at most 15 digits, nesting within validateDepth's limit.  Everything else
// sets bail: the caller reports the item as unsupported, never a different answer.
template <class SH>
GGR_DEV void ce_envelope(SH& S, const EncCtx& cx) {
  const u8* in = cx.in;
  const u32 n_tok = S.n_tok;
  S.env_args_tok = CE_NIL;
  if (S.deep || TK_KIND(S.tok[0]) != TK_LBRACE || TK_AUX(S.tok[0]) != n_tok - 1u) { S.bail = 1; return; }
  const u32 close = n_tok - 1u;
  u32 seen = 0, t = 1;
  bool first = true, have_name = false;
  while (t != close) {
    if (!first) {
      if (TK_KIND(S.tok[t]) != TK_COMMA) { S.bail = 1; return; }
      t++;
    }
    first = false;
    if (t + 2u >= close) { S.bail = 1; return; }
    const u32 kt = S.tok[t];
    if (TK_KIND(kt) != TK_STR || TK_KIND(S.tok[t + 1]) != TK_COLON) { S.bail = 1; return; }
    const u32 vt = S.tok[t + 2];
    const u32 vk = TK_KIND(vt);
    u32 which;
    if (ce_tok_is(S, in, kt, "jsonrpc", 7)) which = 0;
    else if (ce_tok_is(S, in, kt, "id", 2)) which = 1;
    else if (ce_tok_is(S, in, kt, "method", 6)) which = 2;
    else if (ce_tok_is(S, in, kt, "params", 6)) which = 3;
    else { S.bail = 1; return; }
    if (seen & (1u << which)) { S.bail = 1; return; }
    seen |= 1u << which;
    if (which == 0) {
      if (vk != TK_STR || !ce_tok_is(S, in, vt, "2.0", 3)) { S.bail = 1; return; }
      t += 3;
    } else if (which == 2) {
      if (vk != TK_STR || !ce_tok_is(S, in, vt, "tools/call", 10)) { S.bail = 1; return; }
      t += 3;
    } else if (which == 1) {
      const u32 pos = TK_POS(vt);
      if (vk == TK_STR) {  // RequestID re-marshals the string: plain ASCII without HTML characters stays as it is
        const u32 k = TK_AUX(vt);
        if (S.qslow[k] != S.qslow[k + 1] || S.qesc[k] != S.qesc[k + 1]) { S.bail = 1; return; }
        const u32 q1 = S.qpos[k + 1];
        for (u32 j = pos + 1u; j < q1; j++) {
          const u32 c = in[j];
          if (c >= 0x80u || c == '<' || c == '>' || c == '&') { S.bail = 1; return; }
        }
        S.env_id_pos = pos;
        S.env_id_len = q1 - pos + 1u;
      } else if (vk == TK_SCALAR) {  // a number goes through float64: integers of at most 15 digits survive
        u32 j = pos, digits = 0;
        if (in[j] == '-') j++;
        const u32 d0 = j;
        while (j < cx.end && (u32)(in[j] - '0') < 10u) { j++; digits++; }
        const u32 c = j < cx.end ? in[j] : 0u;
        if (digits == 0 || digits > 15u || (digits > 1u && in[d0] == '0') || !(ggr_is_ws(c) || c == ',' || c == '}')) { S.bail = 1; return; }
        S.env_id_pos = pos;
        S.env_id_len = j - pos;
      } else {
        S.bail = 1;
        return;
      }
      t += 3;
    } else {  // params
      if (vk != TK_LBRACE) { S.bail = 1; return; }
      const u32 pclose = TK_AUX(vt);
      u32 u = t + 3, pseen = 0;
      bool pfirst = true;
      while (u != pclose) {
        if (!pfirst) {
          if (TK_KIND(S.tok[u]) != TK_COMMA) { S.bail = 1; return; }
          u++;
        }
        pfirst = false;
        if (u + 2u >= pclose) { S.bail = 1; return; }
        const u32 pk = S.tok[u];
        if (TK_KIND(pk) != TK_STR || TK_KIND(S.tok[u + 1]) != TK_COLON) { S.bail = 1; return; }
        const u32 pv = S.tok[u + 2];
        if (ce_tok_is(S, in, pk, "name", 4)) {
          if (pseen & 1u) { S.bail = 1; return; }
          pseen |= 1u;
          const u32 k = TK_AUX(pv);
          if (TK_KIND(pv) != TK_STR || S.qslow[k] != S.qslow[k + 1] || S.qesc[k] != S.qesc[k + 1]) { S.bail = 1; return; }
          const u32 p0 = TK_POS(pv), q1 = S.qpos[k + 1], len = q1 - p0 - 1u;
          if (len == 0 || len > 128u) { S.bail = 1; return; }
          for (u32 j = p0 + 1u; j < q1; j++) {  // isValidToolName (validation.go:227-232)
            const u32 c = in[j];
            if (!((c - 'a') < 26u || (c - 'A') < 26u || (c - '0') < 10u || c == '_' || c == '.')) { S.bail = 1; return; }
          }
          KeyInfo ki;
          ce_key_info_plain(in, p0, q1, &ki);
          const U4 tt = ggr_ld16(cx.T.tools);
          i32 m;
          if (!hash_lookup(cx.T, tt.x, tt.y, ki, in, p0, cx.end, &m)) { S.bail = 1; return; }
          const u32 msg = ggr_u16(cx.T, tt.z + (u32)m);
          if (msg == 0xFFFFu) { S.bail = 1; return; }  // streaming method
          S.env_method = (u32)m;
          S.env_msg = msg;
          have_name = true;
          u += 3;
        } else if (ce_tok_is(S, in, pk, "arguments", 9)) {
          if (pseen & 2u) { S.bail = 1; return; }
          pseen |= 2u;
          if (TK_KIND(pv) != TK_LBRACE) { S.bail = 1; return; }
          S.env_args_tok = u + 2u;
          u = TK_AUX(pv) + 1u;
        } else {
          S.bail = 1;
          return;
        }
        if (u > pclose) { S.bail = 1; return; }
      }
      t = pclose + 1u;
    }
    if (t > close) { S.bail = 1; return; }
  }
  if (seen != 0xFu || !have_name) S.bail = 1;
}

GGR_DEV u32 ce_link(u32 x) { return x == CE_NIL ? GGR_NIL : x; }

// Envelope mode, one lane: a number literal that json.Marshal would re-print differently.  Returns false
// when the literal is no float64 (range) or the re-printed text does not parse for the field.
GGR_DEVN bool ce_leaf_number_via_float64(EncCtx& cx, u32 pos, const FieldD& f, Leaf* l) {
  Leaf ld;
  {
    Rd r;
    r.init(cx.in, pos, cx.end);
    if (parse_scalar(cx, r, GK_DOUBLE, -1, &ld) != GST_OK) return false;
    if (!r.eof()) {
      const u32 c = r.peek();
      if (!(ggr_is_ws(c) || c == ',' || c == '}' || c == ']')) return false;
    }
  }
  const u64 bits = (u64)ld.a | ((u64)ld.b << 32);
#if defined(__CUDA_ARCH__)
  __align__(16) u8 buf[64];
#else
  alignas(16) u8 buf[64];
#endif
  for (int k = 0; k < 64; k++) buf[k] = 0;
  Sw w;
  w.init(buf, 0);
  put_float_go(w, bits, false);  // encoding/json floatEncoder == protojson's number format
  if (w.pos == 0 || w.pos > 30) return false;
  Rd r2;
  r2.init(buf, 0, w.pos, 1);  // a local buffer: not through the read-only path
  if (parse_scalar(cx, r2, f.kind, f.child, l) != GST_OK) return false;
  return r2.eof();
}

// T4, one lane: finish leaf node `ni` (IR node + size into its parent).  ENV: request-envelope mode.
template <class SH, bool ENV>
GGR_DEV void ce_leaf(SH& S, EncCtx& cx, u32 ni) {
  const CNode nd = S.node[ni];
  const u32 next = ce_link(nd.next);
  if (nd.cls == CC_NULL) {
    node_store(cx.ir, ni, 0, 0, next, nd.emit, node_meta(N_SKIP, 0, 0));
    return;
  }
  const FieldD f = ggr_field(cx.T, nd.gfield);
  const u32 tk = S.tok[nd.tok];
  const u32 pcls = S.node[nd.parent].cls;
  const bool in_list = pcls == CC_LIST || pcls == CC_ENTRY;  // no zero elision in lists and map entries
  const bool packed = pcls == CC_LIST && (f.flags & GF_PACKED);
  const u32 tag = packed ? 0u : f.tag, tag_len = packed ? 0u : f.tag_len;
  Rd r;
  r.init(cx.in, TK_POS(tk), cx.end);
  if (nd.cls == CC_TS) {
    const u32 q = r.pos;
    StrInfo si;
    if (scan_string<false>(r, &si) != GST_OK) { S.bail = 1; return; }
    StrIter it;
    it.init(cx.in, q, cx.end);
    i64 secs;
    i32 nanos;
    if (parse_timestamp(it, &secs, &nanos) != GST_OK) { S.bail = 1; return; }
    u32 sidx = GGR_NIL, nidx = GGR_NIL, payload = 0;
    if (nanos != 0) {
      nidx = wp_atomic_add(&S.n_node, 1u);
      if (nidx >= S.cap) { S.bail = 1; return; }
      node_store(cx.ir, nidx, (u32)nanos, 0, GGR_NIL, 1, node_meta(N_VARINT, 0, 16));
      payload += 1 + varint_size((u64)(u32)nanos);
    }
    if (secs != 0) {
      sidx = wp_atomic_add(&S.n_node, 1u);
      if (sidx >= S.cap) { S.bail = 1; return; }
      node_store(cx.ir, sidx, (u32)(u64)secs, (u32)((u64)secs >> 32), nidx, 0, node_meta(N_VARINT, 0, 8));
      payload += 1 + varint_size((u64)secs);
    }
    node_store(cx.ir, ni, payload, sidx != GGR_NIL ? sidx : nidx, next, nd.emit, node_meta(N_MSG, 0, f.tag));
    const u32 tsfull = f.tag_len + varint_size(payload) + payload;
    S.node[ni].body = tsfull;
    wp_atomic_add(&S.node[nd.parent].body, tsfull);
    // the seconds / nanos nodes have no entry of their own in the node table: the emitter writes
    // them together with this node
    if (sidx != GGR_NIL) cx.ioff[sidx] = 0xFFFFFFFFu;
    if (nidx != GGR_NIL) cx.ioff[nidx] = 0xFFFFFFFFu;
    return;
  }
  Leaf l;
  bool done = false;
  if (ENV && TK_KIND(tk) == TK_SCALAR) {
    // json.Marshal(arguments) re-prints every number from float64 (handler.go:224-231): plain integers of at
    // most 15 digits come out as they went in; any other literal is taken through the same round trip here -
    // text -> float64 -> encoding/json's shortest text -> the field's own parser on that text
    u32 j = TK_POS(tk), digits = 0;
    const u32 c0 = cx.in[j];
    if (c0 == '-' || (c0 - '0') < 10u) {
      if (c0 == '-') j++;
      while (j < cx.end && (u32)(cx.in[j] - '0') < 10u) { j++; digits++; }
      const u32 c = j < cx.end ? cx.in[j] : 0u;
      if (digits == 0 || digits > 15u || c == '.' || c == 'e' || c == 'E') {
        if (!ce_leaf_number_via_float64(cx, TK_POS(tk), f, &l)) { S.bail = 1; return; }
        done = true;
      }
    }
  }
  if (nd.cls == CC_STR && TK_KIND(tk) == TK_STR) {
    // the tokenizer validated UTF-8 and counted simple escapes and the bytes that need the full
    // scanner (control characters, \u, bad escapes): without the latter the string is valid and its
    // decoded length known
    const u32 k = TK_AUX(tk);
    if (S.qslow[k] == S.qslow[k + 1]) {
      const u32 nesc = (u16)(S.qesc[k + 1] - S.qesc[k]);
      const u32 q = TK_POS(tk), len = (u32)S.qpos[k + 1] - q - 1u - nesc;  // a simple escape decodes 2 bytes to 1
      l.type = N_STR;
      l.a = q;
      l.b = len;
      l.flags = nesc ? (NF_ESC | NF_SIMPLE) : 0;
      l.body = varint_size(len) + len;
      l.zero = len == 0;
      done = true;
    }
  }
  if (!done) {
    if (parse_scalar(cx, r, f.kind, f.child, &l) != GST_OK) { S.bail = 1; return; }
    if (TK_KIND(tk) == TK_SCALAR && !r.eof()) {  // the literal must end where the parser stopped
      u32 c = r.peek();
      if (!(ggr_is_ws(c) || c == ',' || c == '}' || c == ']')) { S.bail = 1; return; }
    }
  }
  const bool live = in_list || (f.flags & GF_PRESENCE) || !l.zero;
  node_store(cx.ir, ni, l.a, l.b, next, nd.emit, live ? node_meta(l.type, l.flags, tag) : node_meta(N_SKIP, 0, 0));
  if (live) {
    S.node[ni].body = tag_len + l.body;
    wp_atomic_add(&S.node[nd.parent].body, tag_len + l.body);
  }
}

// T5, one lane: container `ni` is complete; write its IR node and add its size to the parent.
template <class SH>
GGR_DEV void ce_close_container(SH& S, EncCtx& cx, u32 ni) {
  const CNode nd = S.node[ni];
  const FieldD f = ggr_field(cx.T, nd.gfield);
  const u32 next = ce_link(nd.next), head = ce_link(nd.head);
  u32 full;
  if (nd.cls == CC_ENTRY) {
    node_store(cx.ir, ni, nd.body, head, next, 0, node_meta(N_ENTRY, 0, f.tag));
    full = f.tag_len + varint_size(nd.body) + nd.body;
  } else if (nd.cls == CC_MAP) {
    node_store(cx.ir, ni, nd.body, head, next, nd.emit, nd.head == CE_NIL ? node_meta(N_SKIP, 0, 0) : node_meta(N_MAP, 0, 0));
    full = nd.body;
  } else if (nd.cls == CC_MSG) {
    node_store(cx.ir, ni, nd.body, head, next, nd.emit, node_meta(N_MSG, 0, f.tag));
    full = f.tag_len + varint_size(nd.body) + nd.body;
  } else if (nd.head == CE_NIL) {
    node_store(cx.ir, ni, 0, 0, next, nd.emit, node_meta(N_SKIP, 0, 0));
    full = 0;
  } else if (f.flags & GF_PACKED) {
    node_store(cx.ir, ni, nd.body, head, next, nd.emit, node_meta(N_LIST, NF_PACKED, f.tag));
    full = f.tag_len + varint_size(nd.body) + nd.body;
  } else {
    node_store(cx.ir, ni, nd.body, head, next, nd.emit, node_meta(N_LIST, 0, 0));
    full = nd.body;
  }
  S.node[ni].tok = (u16)(full - nd.body);  // header: tag and length prefix, if any (the token is no longer needed)
  wp_atomic_add(&S.node[nd.parent].body, full);
}

// T6, one lane: container `ni` knows its offset; hand out offsets to its children.  The offsets
// live in the token array, which is dead by now.
template <class SH>
GGR_DEV void ce_place_children(SH& S, u32 ni) {
  const CNode nd = S.node[ni];
  u32 pos = S.tok[ni] + nd.tok;
  for (u32 c = nd.head; c != CE_NIL; c = S.node[c].next) {
    const CNode ch = S.node[c];
    S.tok[c] = pos;
    pos += ch.cls <= CC_ENTRY ? ch.body + ch.tok : ch.body;
  }
}

// T1 + T2 of one item, all 32 lanes: the token index into the item's IR region (ir_cap nodes of 16
// bytes).  An item whose index does not fit there, or that the tokenizer gives up on, is marked
// `bail` for the walker.
template <class TS>
GGR_DEV void ce_tok_item(TS& S, const CeLut& lut, const u8* in, u32 start, u32 end, u8* ir, u32 ir_cap) {
  const u32 lane = wp_lane();
  if (end > CE_MAX_INPUT || ir_cap == 0 || end == start) return;  // decided by the walker before it looks at the index
  u32* g = reinterpret_cast<u32*>(ir);
  WP_SYNC();  // persistent warps: nobody still reads the previous item's state
  if (lane == 0) {
    S.bail = 0;
    S.deep = 0;
  }
  WP_SYNC();
  ce_tokenize(S, lut, in, start, end);
  if (!S.bail) ce_match(S, lut, in);
  const u32 n_tok = S.n_tok, n_q = S.n_q;
  const bool bail = S.bail != 0 || ce_tok_bytes(n_tok, n_q) > ir_cap * 16u;
  if (lane == 0) {
    g[0] = n_tok;
    g[1] = n_q;
    g[2] = bail ? 1u : 0u;
    g[3] = S.deep;
  }
  if (bail) return;
  u32* gt = g + 4;
  for (u32 i = lane; i < n_tok; i += 32) gt[i] = S.tok[i];
  const u32 nw = (n_q + 1u) >> 1;
  u32* gq = gt + n_tok;
  const u32* qp = reinterpret_cast<const u32*>(S.qpos);
  const u32* qe = reinterpret_cast<const u32*>(S.qesc);
  const u32* qs = reinterpret_cast<const u32*>(S.qslow);
  for (u32 i = lane; i < nw; i += 32) {
    gq[i] = qp[i];
    gq[nw + i] = qe[i];
    gq[2u * nw + i] = qs[i];
  }
}

// One item, all 32 lanes.  Returns true when the item was handled (IR written, *res filled);
// false leaves it to the per-thread parser.
// PRE: the token index was left in the IR region by ce_tok_item.
template <class SH, bool ENV, bool PRE = false>
GGR_DEV bool ce_parse_item(SH& S, const CeLut& lut, const Tables& T, u32 root_msg, const u8* in, u32 start, u32 end, u8* ir,
                           u32* ioff, u32 ir_cap, EncResult* res) {
  const bool envelope = ENV;
  const u32 lane = wp_lane();
  res->size = 0;
  res->first = GGR_NIL;
  res->n_nodes = 0;
  res->method = 0;
  res->id_pos = res->id_len = 0;
  if (end > CE_MAX_INPUT || ir_cap == 0) return false;
  if (end == start) return !envelope;  // reflection.go:354: "" skips protojson (an empty body is no request)
  WP_SYNC();  // persistent warps: nobody still reads the previous item's state
  if (lane == 0) {
    S.bail = 0;
    S.n_node = 0;
    S.q_end = 0;
    S.max_depth = 0;
    S.deep = 0;
    S.env = envelope ? 1u : 0u;
    S.cap = ir_cap < SH::MAX_NODE ? ir_cap : SH::MAX_NODE;
  }
  WP_SYNC();
  if (PRE) {
    const u32* g = reinterpret_cast<const u32*>(ir);
    const u32 nt = g[0], nq = g[1];
    if (g[2] != 0 || nt > SH::MAX_TOK || nq > SH::MAX_Q) return false;
    const u32* gt = g + 4;
    for (u32 i = lane; i < nt; i += 32) S.tok[i] = gt[i];
    const u32 nw = (nq + 1u) >> 1;
    const u32* gq = gt + nt;
    u32* qp = reinterpret_cast<u32*>(S.qpos);
    u32* qe = reinterpret_cast<u32*>(S.qesc);
    u32* qs = reinterpret_cast<u32*>(S.qslow);
    for (u32 i = lane; i < nw; i += 32) {
      qp[i] = gq[i];
      qe[i] = gq[nw + i];
      qs[i] = gq[2u * nw + i];
    }
    if (lane == 0) {
      S.n_tok = nt;
      S.n_q = nq;
      S.deep = g[3];
    }
    WP_SYNC();  // the index is in shared memory: from here on the region takes IR nodes
  } else {
    ce_tokenize(S, lut, in, start, end);
    if (S.bail) return false;
    ce_match(S, lut, in);
    if (S.bail) return false;
  }
  const u32 n_tok = S.n_tok;
  // exactly one top-level value, an object
  if (TK_KIND(S.tok[0]) != TK_LBRACE || TK_AUX(S.tok[0]) != n_tok - 1u) return false;
  EncCtx cx;
  cx.T = T;
  cx.in = in;
  cx.end = end;
  cx.ir = ir;
  cx.ir_cap = ir_cap;
  cx.n_nodes = 0;
  cx.ioff = ioff;
  u32 root_tok = 0;
  if (envelope) {  // the message is the `arguments` object of the request, its type comes from the tool name
    WP_SYNC();  // every lane has read `bail` above before lane 0 may set it again
    if (lane == 0) ce_envelope(S, cx);
    WP_SYNC();
    if (S.bail) return false;
    res->method = S.env_method;
    res->id_pos = S.env_id_pos;
    res->id_len = S.env_id_len;
    root_msg = S.env_msg;
    root_tok = S.env_args_tok;
    if (root_tok == CE_NIL) return true;  // no arguments: the empty message
    WP_SYNC();
  }
  if (lane == 0) {
    u32 r0 = ce_new_node(S, root_tok, CE_NIL, 0, 0, CC_MSG, 0);
    S.node[r0].msg = (u16)root_msg;
    S.queue[0] = (u16)r0;
    S.q_end = 1;
  }
  WP_SYNC();
  if (root_msg >= 0xFFFFu) return false;
  // T3: level by level
  u32 qb = 0;
  for (;;) {
    const u32 qe = S.q_end;
    if (qb == qe) break;
    WP_SYNC();  // everyone has read q_end before the walkers append to the queue
    for (u32 i = qb + lane; i < qe; i += 32) {
      const u32 ni = S.queue[i];
      if (S.node[ni].cls == CC_MAP) ce_walk_map(S, cx, ni);
      else ce_walk_object(S, cx, ni);
    }
    WP_SYNC();
    if (S.bail) return false;
    qb = qe;
  }
  const u32 n = S.n_node;
  // T4: bucket the leaves by class and the containers by depth (into `queue`, free since T3)
  if (lane < CC_N) S.cls_cnt[lane] = 0;
  if (lane < CE_MAX_DEPTH + 2) S.dep_cur[lane] = 0;
  WP_SYNC();
  for (u32 i = lane; i < n; i += 32) {
    const u32 c = S.node[i].cls;
    if (c >= CC_NULL) wp_atomic_add(&S.cls_cnt[c], 1u);
    else wp_atomic_add(&S.dep_cur[S.node[i].depth], 1u);
  }
  WP_SYNC();
  if (lane == 0) {
    u32 run = 0;
    for (u32 c = 0; c < CC_N; c++) {
      S.cls_cur[c] = run;
      run += S.cls_cnt[c];
    }
    S.n_leaf = run;
  }
  if (lane == 1) {
    u32 run = 0;
    for (u32 d = 0; d < CE_MAX_DEPTH + 1; d++) {
      const u32 c = S.dep_cur[d];
      S.dep_beg[d] = run;
      S.dep_cur[d] = run;
      run += c;
    }
    S.dep_beg[CE_MAX_DEPTH + 1] = run;
  }
  WP_SYNC();
  for (u32 i = lane; i < n; i += 32) {
    const u32 c = S.node[i].cls;
    if (c >= CC_NULL) S.order[wp_atomic_add(&S.cls_cur[c], 1u)] = (u16)i;
    else S.queue[wp_atomic_add(&S.dep_cur[S.node[i].depth], 1u)] = (u16)i;
  }
  WP_SYNC();
  const u32 n_leaf = S.n_leaf;
  for (u32 k = lane; k < n_leaf; k += 32) ce_leaf<SH, ENV>(S, cx, S.order[k]);
  WP_SYNC();
  if (S.bail) return false;
  // T5: containers, deepest first (the root, depth 0, has no node of its own in the IR)
  const u32 maxd = S.max_depth;
  for (u32 d = maxd; d >= 1; d--) {
    const u32 b = S.dep_beg[d], e = S.dep_beg[d + 1];
    for (u32 k = b + lane; k < e; k += 32) ce_close_container(S, cx, S.queue[k]);
    WP_SYNC();
  }
  // T6: offsets, top-down (the root message has no header)
  if (lane == 0) {
    S.node[0].tok = 0;
    S.tok[0] = 0;
  }
  WP_SYNC();
  for (u32 d = 0; d < maxd; d++) {
    const u32 b = S.dep_beg[d], e = S.dep_beg[d + 1];
    for (u32 k = b + lane; k < e; k += 32) ce_place_children(S, S.queue[k]);
    WP_SYNC();
  }
  for (u32 i = lane; i < n; i += 32) ioff[i] = S.tok[i];
  res->size = S.node[0].body;
  res->first = ce_link(S.node[0].head);
  res->n_nodes = S.n_node;
  return true;
}


// ------------------------------------------------------------------------------------------------
// Pass B, lock-step: every IR node of an item parsed above knows its output offset, so the lanes
// write nodes independently (one lane per node); long plain strings are then copied by the whole
// warp, 128 bytes per step.
// ------------------------------------------------------------------------------------------------
#define CE_LONG_STR 128u /* plain strings of at least this many bytes are copied by the whole warp (faster than 96 when tuned before the H100 port) */
#define CE_LONG_MAX 32u
#define CE_STAGE 8192u /* items with more wire bytes than this: per-thread emitter */
/* the emitter's staging buffer; larger items (up to CE_STAGE and beyond) are written in place.  4864 + the lists = 5.3 KB per
   warp = 10 blocks per SM instead of 6 with 8192 (configs[2]: wire items up to 4.6 KB) */
#define CE_STAGE_BUF 4864u
struct
#if defined(__CUDACC__)
    __align__(16)
#else
    alignas(16)
#endif
        CoopEmit {
  u8 buf[CE_STAGE_BUF + 48];  // [pad, pad + size): pad = destination address & 15
  u32 src[CE_LONG_MAX], dst[CE_LONG_MAX], len[CE_LONG_MAX];
  u32 n;
};

// one lane: bytes of node `i` into the staging buffer (long plain strings: payload left to the warp)
// STAGED: byte position p of the item lands in the staging buffer (plain shared-memory stores); otherwise - items too
// large to stage - at G[p], the destination itself shifted so that the same positions apply (two instances: a pointer
// that may be either makes every store a generic one, much slower on configs[2] when tuned before the H100 port)
// nd, off: node i and its offset, loaded by the caller (one round ahead: CE_EMIT_LOOP)
template <bool STAGED>
GGR_DEV void ce_emit_node(CoopEmit& E, u8* G, const u8* in, u32 end, const u8* ir, const u32* ioff, u32 i, u32 pad, const U4 nd, const u32 off) {
  u8* const B = STAGED ? E.buf : G;
  const u32 type = nd.w & 0xFu, flags = (nd.w >> 4) & 0xFu, tag = nd.w >> 8;
  if (type == N_SKIP || type == N_MAP || (type == N_LIST && !(flags & NF_PACKED))) return;
  if (off == 0xFFFFFFFFu) return;  // written together with its parent (Timestamp fields)
  Sw w;
  w.init(B, pad + off);
  switch (type) {
    case N_VARINT: {
      if (tag) put_varint(w, tag);
      u64 v = (u64)nd.x | ((u64)nd.y << 32);
      if (flags & NF_RAWKEY) {
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
      if (flags & NF_ESC) {
        u32 k = CE_LONG_MAX;
        if (flags & NF_SIMPLE) k = wp_atomic_add(&E.n, 1u);
        if (k < CE_LONG_MAX) {  // decoded by the whole warp
          E.src[k] = nd.x + 1u;
          E.dst[k] = w.pos;
          E.len[k] = nd.y | 0x80000000u;
        } else {
          copy_string(w, in, nd.x, end, nd.y, true);
        }
      } else {
        bool handed = false;
        if (nd.y >= CE_LONG_STR) {
          const u32 k = wp_atomic_add(&E.n, 1u);
          if (k < CE_LONG_MAX) {
            E.src[k] = nd.x + 1u;
            E.dst[k] = w.pos;
            E.len[k] = nd.y;
            handed = true;
          }
        }
        if (!handed) {  // words from 8 bytes on: faster than 12 when tuned before the H100 port
          coop_copy_bytes<8u>(B + w.pos, in + nd.x + 1u, nd.y);
        }
      }
      break;
    case N_BYTES: {
      if (tag) put_varint(w, tag);
      put_varint(w, nd.y);
      StrIter it;
      it.init(in, nd.x, end);
      u32 n;
      b64_run<true, Sw>(it, (flags & NF_URL) != 0, (flags & NF_PADDED) ? 0u : 1u, &w, &n);
      break;
    }
    case N_MSG:
    case N_ENTRY: {
      if (tag) put_varint(w, tag);
      put_varint(w, nd.x);
      // Timestamp: its seconds / nanos children are written here
      u32 c = nd.y;
      if (c != GGR_NIL && ioff[c] == 0xFFFFFFFFu) {
        while (c != GGR_NIL) {
          U4 cn = node_load(ir, c);
          put_varint(w, cn.w >> 8);
          put_varint(w, (u64)cn.x | ((u64)cn.y << 32));
          c = cn.z & 0xFFFFFu;
        }
      }
      break;
    }
    case N_LIST:
      put_varint(w, tag);
      put_varint(w, nd.x);
      break;
    default: break;
  }
}

// escaped positions of 32 bytes from their backslash mask (run parity as in the tokenizer)
GGR_DEV u32 ce_escaped32(u32 B, u32 cin, u32* cout) {
  B &= ~cin;
  const u64 follows = ((u64)B << 1) | cin;
  const u32 EVEN = 0x55555555u;
  const u32 odd_starts = B & ~EVEN & ~(u32)follows;
  const u64 sum = (u64)odd_starts + B;
  *cout = (u32)(sum >> 32) & 1u;
  return (EVEN ^ (u32)(sum << 1)) & (u32)follows;
}
// all lanes: JSON string text at in[src..) with two-character escapes only -> dec_len raw bytes at d[0..)
GGR_DEV void ce_unescape_coop(const u8* in, u32 src, u8* d, u32 dec_len) {
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u;
  u32 carry = 0, produced = 0;
  while (produced < dec_len) {
    u32 c = in[src + lane];
    const u32 Bm = WP_BALLOT(c == '\\');
    u32 cout;
    const u32 E = ce_escaped32(Bm, carry, &cout);
    const u32 emitm = ~(Bm & ~E);  // escape introducers produce nothing
    if ((E >> lane) & 1u) c = c == 'b' ? 8u : c == 'f' ? 12u : c == 'n' ? 10u : c == 'r' ? 13u : c == 't' ? 9u : c;
    const u32 idx = produced + wp_popc(emitm & lt);
    if (((emitm >> lane) & 1u) && idx < dec_len) d[idx] = (u8)c;
    produced += wp_popc(emitm);
    carry = cout;
    src += 32;
  }
}

// One item, all 32 lanes: size bytes to dst.  Items that fit the staging buffer are assembled there and leave with one
// bulk copy; larger ones (second tier of the walker: tens of KB of wire) are written in place.
// one lane per node, nodes 1 .. n_nodes - 1: the next round's node and offset are requested while this round's node is written
#define CE_EMIT_LOOP(STG, GP)                                                             \
  do {                                                                                    \
    U4 ndn;                                                                               \
    ndn.x = ndn.y = ndn.z = ndn.w = 0u;                                                   \
    u32 offn = 0;                                                                         \
    if (1u + lane < n_nodes) {                                                            \
      ndn = node_load(ir, 1u + lane);                                                     \
      offn = ioff[1u + lane];                                                             \
    }                                                                                     \
    for (u32 i = 1 + lane; i < n_nodes; i += 32) {                                        \
      const U4 nd_ = ndn;                                                                 \
      const u32 off_ = offn;                                                              \
      if (i + 32u < n_nodes) {                                                            \
        ndn = node_load(ir, i + 32u);                                                     \
        offn = ioff[i + 32u];                                                             \
      }                                                                                   \
      ce_emit_node<STG>(E, GP, in, end, ir, ioff, i, pad, nd_, off_);                     \
    }                                                                                     \
  } while (0)

GGR_DEV void ce_emit_item(CoopEmit& E, const u8* in, u32 end, const u8* ir, const u32* ioff, u32 n_nodes, u8* dst, u32 size) {
  const u32 lane = wp_lane();
  const u32 pad = wp_align_pad(dst);
  const bool staged = size <= CE_STAGE_BUF;
  wp_prefetch(in, end < 16384u ? end : 16384u);
  wp_copy_wait();  // persistent warps: the previous item's bulk copy has read the staging buffer
  if (lane == 0) E.n = 0;
  WP_SYNC();
  if (staged) {
    CE_EMIT_LOOP(true, nullptr);
  } else {
    CE_EMIT_LOOP(false, dst - pad);
  }
  WP_SYNC();
  const u32 nl = E.n < CE_LONG_MAX ? E.n : CE_LONG_MAX;
  if (staged) {
    for (u32 k = 0; k < nl; k++) {
      u8* d = E.buf + E.dst[k];
      const u32 len = E.len[k];
      if (len & 0x80000000u) ce_unescape_coop(in, E.src[k], d, len & 0x7FFFFFFFu);
      else coop_copy_words(in, E.src[k], d, len);
    }
    WP_SYNC();
    wp_copy_out(E.buf, dst - pad, pad, size);
  } else {
    for (u32 k = 0; k < nl; k++) {
      u8* d = dst - pad + E.dst[k];
      const u32 len = E.len[k];
      if (len & 0x80000000u) ce_unescape_coop(in, E.src[k], d, len & 0x7FFFFFFFu);
      else coop_copy_words(in, E.src[k], d, len);
    }
  }
}

// ---- item edge of the request lock-step kernels (the host simulation calls the same functions) ----------------------
// Every request lock-step kernel takes items of at most GGR_REQ_ITEM_MAX bytes.
GGR_DEV bool ce_admit(u64 a, u64 b) { return b >= a && b - a <= (u64)GGR_REQ_ITEM_MAX; }

// Which tier of the lock-step parser runs over the token index k_encode_coop_tok left in the IR region: the first (small
// tables); the second tokenizes each item itself.
template <class SH>
struct CeTokFirst {
  static constexpr bool value = false;
};
template <>
struct CeTokFirst<CoopEnc> {
  static constexpr bool value = true;
};

// k_encode_coop_tok, item `item` of the batch whose input starts at a0: its token index into its IR region.
template <class TS>
GGR_DEV void ce_tok_step(TS& S, const CeLut& lut, const u8* in, const u64* in_off, u64 a0, u8* ir, long long item) {
  const u64 a = in_off[item], b = in_off[item + 1];
  if (!ce_admit(a, b)) return;
  const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
  const u32 s0 = (u32)(a & 15ull);
  ce_tok_item(S, lut, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, r.cap);
}

// k_encode_coop_parse: true when the item was parsed into its IR region, *res filled (id_pos from the item's first byte).
// ENV: the item is a whole request body, its message type comes from the tool name.
template <class SH, bool ENV, bool PRE>
GGR_DEV bool ce_parse_step(SH& S, const CeLut& lut, const Tables& T, u32 n_msgs, const i32* msg_id, const u8* in,
                           const u64* in_off, u64 a0, u8* ir, u32* ioff, long long item, EncResult* res) {
  const u64 a = in_off[item], b = in_off[item + 1];
  const i32 m = ENV ? 0 : msg_id[item];
  if (m < 0 || (u32)m >= n_msgs || !ce_admit(a, b)) return false;
  const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
  const u32 s0 = (u32)(a & 15ull);
  const bool ok = ce_parse_item<SH, ENV, PRE>(S, lut, T, (u32)m, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16,
                                              ioff + r.node_off, r.cap, res);
  if (ENV) res->id_pos -= s0;
  return ok;
}

// nnodes of an item the lock-step emitter writes: node count | index of the first node within the item's region << 16.
GGR_DEV u32 ce_nodes_word(u32 n_nodes, u32 first_node) { return n_nodes | (first_node << 16); }

// Lane 0: a parsed item's size, first node, status and node count (and the body's method and id span), where items of
// more than CE_STAGE wire bytes get none (the per-thread emitter writes them).  An item not parsed gets final_status
// when that is >= 0 (the last tier of request bodies: no per-thread path), or goes to `left`.
template <bool ENV>
GGR_DEV void ce_parse_publish(bool ok, const EncResult& res, long long item, u32* size, u32* first, i32* status, u32* nnodes,
                              i32* method, u32* id_span, i32 final_status, GgrWork left) {
  if (wp_lane() != 0) return;
  if (ok) {
    size[item] = res.size;
    first[item] = res.first;
    status[item] = GST_OK;
    nnodes[item] = res.size <= CE_STAGE ? ce_nodes_word(res.n_nodes, 0) : 0;
    if (ENV) {
      method[item] = (i32)res.method;
      id_span[2 * item] = res.id_pos;
      id_span[2 * item + 1] = res.id_len;
    }
  } else {
    size[item] = 0;
    nnodes[item] = 0;
    first[item] = GGR_NIL;
    if (final_status >= 0) status[item] = final_status;
    else left.item[ggr_atomic_add_u32(&left.h->n, 1u)] = (u32)item;
  }
}

// k_encode_coop_emit: pass B of an item the lock-step parser or the walker took with more than one node, behind the
// frame-byte message header k_encode_emit wrote.  True when it wrote the item.
GGR_DEV bool ce_emit_step(CoopEmit& E, const u8* in, const u64* in_off, u64 a0, const u8* ir, const u32* ioff, const u32* nnodes,
                          const u32* size, const i32* status, u8* out, const u64* out_off, u32 frame, long long item) {
  const u32 nw = nnodes[item];
  const u32 nn = nw & 0xFFFFu;
  const u32 sz = size[item];
  if (nn <= 1 || sz <= frame || status[item] != GST_OK) return false;
  const u64 a = in_off[item], b = in_off[item + 1];
  const u64 node_off = ggr_item_region(a0, a, b, (u64)item).node_off + (u64)(nw >> 16);
  ce_emit_item(E, in + (a & ~15ull), (u32)(a & 15ull) + (u32)(b - a), ir + node_off * 16, ioff + node_off, nn, out + out_off[item] + frame,
               sz - frame);
  return true;
}
