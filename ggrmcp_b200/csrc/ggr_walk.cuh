// ggr_walk.cuh - lock-step request side, pass A, token-parallel form (one warp per item).
//
// Replaces, for regular items, the one-lane-per-object walker of ggr_coop_enc.cuh: every phase
// below runs one lane per TOKEN or per VALUE, never one lane per object, and holds no token table in
// shared memory (the index stays in the item's IR region in HBM and is read through L1).  What the
// reference does here is protojson.Unmarshal into a dynamicpb message followed by proto.Marshal's size
// pass (/root/reference/pkg/grpc/reflection.go:351-357,373).
//
// Three small kernels (each one's hot loop fits the instruction caches, which the fused form's did not):
//   k_encode_tok3  : T1 - bit-mask tokenizer as in ggr_coop_enc.cuh, but colons and commas are consumed
//                    here: which token may follow which is checked on bit masks (carry-propagating adds
//                    find every token's predecessor), the surviving tokens - brackets, strings, scalars -
//                    carry "after a comma" / "after a colon" flags.  Tokens and the quote table go straight
//                    to the item's IR region: [header][tokens ... records ... IR nodes ...   ... quote entries]
//   k_encode_place : W2 - innermost open bracket of every token (level + match_any), the context rules of
//                    the JSON grammar on adjacent tokens, one record per value in document order
//                    (token, enclosing value, level)
//   k_encode_type  : W3 - records bucketed by level (children of one container are contiguous), then level
//                         by level, one lane per value: key -> field through the key tables, duplicate / oneof
//                         detection by atomic masks on the parent, leaf values parsed and sized, rank of the
//                         value among its siblings in emit order
//                    W4 - sizes bottom-up by level: sizes scattered into emit order, segmented scan = offset
//                         within the parent, segment total = the parent's payload
//                    W5 - offsets top-down: absolute output offset of every IR node
// Output: the same IR nodes + one output offset per node that k_encode_coop_emit consumes (nodes carry no
// sibling links: items larger than the emitter's staging buffer are left to the other tiers).
// Only regular input is handled; anything else - syntax or type error, unknown / duplicate field, escapes
// in field names, floats, bytes, timestamps, quoted numbers, unsorted map keys, table overflow - leaves the
// item, untouched, to the next tier (the fused large-table kernel, then the per-thread parser, which owns
// the error semantics).
#pragma once
#include "ggr_coop_enc.cuh"

#define CW_LEVELS 16
// host simulation only: why an item was left to the next tier (tests print a histogram)
#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define CW_WHY(code) ((void)0)
#else
extern int g_cw_why;
#define CW_WHY(code) (g_cw_why = (code))
#endif
#define CW_NONE 0xFFFFu

// tokens: pos(16) | kind(3) | after-comma(1) | after-colon(1) | string number(11)
enum { K3_LBRACE = 1, K3_RBRACE = 2, K3_LBRACK = 3, K3_RBRACK = 4, K3_STR = 5, K3_SCALAR = 6 };
#define K3_POS(t) ((t) & 0xFFFFu)
#define K3_KIND(t) (((t) >> 16) & 7u)
#define K3_C(t) (((t) >> 19) & 1u)
#define K3_V(t) (((t) >> 20) & 1u)
#define K3_Q(t) (((t) >> 21) << 1) /* quote entry of the opening quote; the closing one follows */
#define K3_MAX_STR 2047u

// ---- token index in the item's IR region (cap nodes of 16 bytes) -------------------------------
// [0,16) header {n_tok, n_q, bail, n_rec (k_encode_place; 0xFFFFFFFF: left to the next tier)}; tokens grow up
// from byte 16, quote entries (8 bytes: pos | esc << 16, slow) grow down from the end; each may use half of the
// region.  Behind the tokens: the value records of k_encode_place (8 bytes each), then the IR nodes.
struct CwIndex {
  const u32* tok;
  const u8* qend;  // entry k at qend - 8 * (k + 1)
  u32 n_tok, n_q;
};
GGR_DEV u32 cw_tok_cap(u32 cap) { return cap >= 4u ? (cap * 8u - 16u) / 4u : 0u; }
GGR_DEV u32 cw_q_cap(u32 cap) { return cap < 2u * K3_MAX_STR ? cap : 2u * K3_MAX_STR; }
GGR_DEV u32 cw_ldg(const u32* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}
struct CwQ {
  u32 pos, esc, slow;
};
GGR_DEV CwQ cw_q(const CwIndex& X, u32 k) {
  const u32* p = reinterpret_cast<const u32*>(X.qend - 8u * (k + 1u));
  const u32 a = cw_ldg(p), b = cw_ldg(p + 1);
  CwQ q = {a & 0xFFFFu, a >> 16, b};
  return q;
}
// Key of the member whose value is token i (the token in front of it is the key's string): position of the key's text
// | length << 16 | bit 31 = "a plain key" (no escapes, no bytes for the full scanner, shorter than 32 768 bytes)
GGR_DEV u32 cw_key_pack(const CwIndex& X, u32 i) {
  const u32 kt = cw_ldg(X.tok + i - 1u);
  const CwQ q0 = cw_q(X, K3_Q(kt)), q1 = cw_q(X, K3_Q(kt) + 1u);
  const u32 kp = K3_POS(kt), len = (q1.pos - kp - 1u) & 0xFFFFu;
  const bool plain = K3_KIND(kt) == K3_STR && q0.slow == q1.slow && q0.esc == q1.esc && len < 0x8000u;
  return plain ? (((kp + 1u) & 0xFFFFu) | (len << 16) | 0x80000000u) : 0u;
}
GGR_DEV u32 cw_rec_off(u32 n_tok) { return (16u + 4u * n_tok + 15u) & ~15u; }

// second class table of the tokenizer: which structural character
#define CW_LO 0x00000001u /* { [ */
#define CW_LC 0x00000100u /* } ] */
#define CW_LY 0x00010000u /* { } */
#define CW_LN 0x01000000u /* : */
struct CwLut {
  CeLut base;
  u32 cls2[256];
};
GGR_DEV void cw_lut_init(CwLut& L, u32 first, u32 step) {
  ce_lut_init(L.base, first, step);
  for (u32 b = first; b < 256; b += step) {
    u32 c = 0;
    if (b == '{' || b == '[') c |= CW_LO;
    if (b == '}' || b == ']') c |= CW_LC;
    if (b == '{' || b == '}') c |= CW_LY;
    if (b == ':') c |= CW_LN;
    L.cls2[b] = c;
  }
}

// Tokens that follow the tokens of A (17-bit masks, bit 0 = the token in front of the chunk): adding A << 1 to
// the complement of the token mask lets the carry run through the bytes that start no token and set the next
// token's bit.
GGR_DEV u32 cw_next(u32 T, u32 A) { return ((~T & 0x3FFFFu) + (A << 1)) & T; }

// ---- the item's text travels global -> shared memory by bulk asynchronous copies (cp.async.bulk, the TMA's 1-D form)
// that complete on an mbarrier: two tiles of CW_TILE bytes per warp, tile t + 2 is requested as soon as every lane has
// taken its 16 bytes of the last round of tile t, so that the copy of the next tiles runs under the mask arithmetic of
// the current one and the lanes read their chunks with one conflict-free LDS.128 instead of a global load each.  The host
// simulation has no bulk copies: there every lane loads its 16 bytes from the text itself.
#define CW_TILE 2048u                 /* 128 chunks of 16 bytes = 4 rounds of the warp */
#define CW_TILE_CHUNKS (CW_TILE / 16u)
struct
#if defined(__CUDACC__)
    __align__(128)
#else
    alignas(128)
#endif
        CwTile {
  u8 buf[2][CW_TILE];
  unsigned long long bar[2];  // one mbarrier per stage (arrival count 1: the lane that issues the copy)
};
#if defined(__CUDACC__)
// lane 0 of the warp, once per kernel (followed by a block-wide barrier)
GGR_DEV void cw_tile_init(CwTile* tl) {
#if defined(__CUDA_ARCH__)
  const unsigned b0 = (unsigned)__cvta_generic_to_shared(&tl->bar[0]), b1 = (unsigned)__cvta_generic_to_shared(&tl->bar[1]);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b0) : "memory");
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b1) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
// one lane: bytes (a multiple of 16, > 0) from src (16-byte aligned) into stage stg; completes on the stage's barrier
GGR_DEV void cw_tile_issue(CwTile* tl, u32 stg, const u8* src, u32 bytes) {
#if defined(__CUDA_ARCH__)
  const unsigned bar = (unsigned)__cvta_generic_to_shared(&tl->bar[stg]);
  const unsigned dst = (unsigned)__cvta_generic_to_shared(&tl->buf[stg][0]);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(bar)
               : "memory");
#endif
}
// all lanes: the copy into stage stg of the phase with this parity has landed
GGR_DEV void cw_tile_wait(CwTile* tl, u32 stg, u32 parity) {
#if defined(__CUDA_ARCH__)
  const unsigned bar = (unsigned)__cvta_generic_to_shared(&tl->bar[stg]);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "CW_TILE_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra CW_TILE_DONE;\n"
      "bra CW_TILE_WAIT;\n"
      "CW_TILE_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
#endif
}
#endif

// T1 of one item, all 32 lanes.  tl: this warp's tile ring (device; the host simulation reads the text in place),
// ph: the parities of the two stages' barriers, carried from item to item by the persistent warp.
GGR_DEV void cw_tok_item(CwTile* tl, u32& ph, const CwLut& LT, const u8* in, u32 start, u32 end, u8* region, u32 cap) {
  const u32 lane = wp_lane();
  if (end > CE_MAX_INPUT || cap < 8u || end == start) return;  // decided again by the later kernels before they look at the index
  const u32* lut = LT.base.cls;
  const u32* lut2 = LT.cls2;
  u32* const gt = reinterpret_cast<u32*>(region) + 4;
  u8* const gqend = region + (size_t)cap * 16u;
  const u32 tcap = cw_tok_cap(cap), qcap = cw_q_cap(cap);
  const u32 lt = (1u << lane) - 1u;
  const u32 nchunks = (end + 15u) >> 4;
  u32 c_carry = 0, in_carry = 0, n_carry = 0, u_carry = 0;  // warp-uniform carries between rounds
  u32 k_carry = 0;                                            // kind of the last token so far (0: none yet; 7 colon, 8 comma)
  u32 tbase = 0, qbase = 0, dbase = 0, ebase = 0;
  u32 bail = 0;
#if defined(__CUDA_ARCH__)
  const u32 ntiles = (nchunks + CW_TILE_CHUNKS - 1u) / CW_TILE_CHUNKS;
  if (lane == 0) {  // the first two tiles are on their way before the first round starts
    cw_tile_issue(tl, 0, in, (nchunks < CW_TILE_CHUNKS ? nchunks : CW_TILE_CHUNKS) << 4);
    if (ntiles > 1u) cw_tile_issue(tl, 1, in + CW_TILE, ((nchunks - CW_TILE_CHUNKS) < CW_TILE_CHUNKS ? (nchunks - CW_TILE_CHUNKS) : CW_TILE_CHUNKS) << 4);
  }
#else
  (void)tl;
  (void)ph;
  U4 vn;  // the next round's chunk is requested one round ahead
  vn.x = vn.y = vn.z = vn.w = 0;
  if (lane < nchunks) vn = ggr_ld16(in + (lane << 4));
#endif
  for (u32 cb = 0; cb < nchunks; cb += 32) {
    const u32 ci = cb + lane;
    const u32 off = ci << 4;
    u32 Q = 0, B = 0, X = 0, W = 0xFFFFu, D = 0, HI = 0, XO = 0, XC = 0, XY = 0, XN = 0;
#if defined(__CUDA_ARCH__)
    U4 v;
    v.x = v.y = v.z = v.w = 0;
    {
      const u32 tile = cb / CW_TILE_CHUNKS, stg = tile & 1u, in_tile = cb & (CW_TILE_CHUNKS - 1u);
      if (in_tile == 0) {  // first round of a tile: wait for its bytes
        cw_tile_wait(tl, stg, (ph >> stg) & 1u);
        ph ^= 1u << stg;
      }
      if (ci < nchunks) {
        const uint4 q = *reinterpret_cast<const uint4*>(&tl->buf[stg][(in_tile + lane) << 4]);
        v.x = q.x; v.y = q.y; v.z = q.z; v.w = q.w;
      }
      // last round of the tile: once every lane holds its chunk the stage is free for tile + 2
      if ((in_tile == CW_TILE_CHUNKS - 32u || cb + 32u >= nchunks) && tile + 2u < ntiles) {
        __syncwarp();
        if (lane == 0) {
          const u32 c0 = (tile + 2u) * CW_TILE_CHUNKS, left = nchunks - c0;
          cw_tile_issue(tl, stg, in + ((size_t)c0 << 4), (left < CW_TILE_CHUNKS ? left : CW_TILE_CHUNKS) << 4);
        }
      }
    }
#else
    const U4 v = vn;
    vn.x = vn.y = vn.z = vn.w = 0;
    if (ci + 32u < nchunks) vn = ggr_ld16(in + off + 512u);
#endif
    if (ci < nchunks) {
      u32 lo = 0, hi = 0, lo2 = 0, hi2 = 0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const u32 b0 = (v.x >> (8 * j)) & 0xFFu, b1 = (v.y >> (8 * j)) & 0xFFu, b2 = (v.z >> (8 * j)) & 0xFFu, b3 = (v.w >> (8 * j)) & 0xFFu;
        lo |= lut[b0] << j;
        lo |= lut[b1] << (j + 4);
        hi |= lut[b2] << j;
        hi |= lut[b3] << (j + 4);
        lo2 |= lut2[b0] << j;
        lo2 |= lut2[b1] << (j + 4);
        hi2 |= lut2[b2] << j;
        hi2 |= lut2[b3] << (j + 4);
      }
      Q = (lo & 0xFFu) | ((hi & 0xFFu) << 8);
      B = ((lo >> 8) & 0xFFu) | (((hi >> 8) & 0xFFu) << 8);
      X = ((lo >> 16) & 0xFFu) | (((hi >> 16) & 0xFFu) << 8);
      W = ((lo >> 24) & 0xFFu) | (((hi >> 24) & 0xFFu) << 8);
      XO = (lo2 & 0xFFu) | ((hi2 & 0xFFu) << 8);
      XC = ((lo2 >> 8) & 0xFFu) | (((hi2 >> 8) & 0xFFu) << 8);
      XY = ((lo2 >> 16) & 0xFFu) | (((hi2 >> 16) & 0xFFu) << 8);
      XN = ((lo2 >> 24) & 0xFFu) | (((hi2 >> 24) & 0xFFu) << 8);
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
    // UTF-8 over the whole text (see ce_tokenize)
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
          if (len == 0) bail = 1;
          else EC |= ((1u << (len - 1u)) - 1u) << (j + 1u);
        }
      }
      u32 cin = WP_SHFL_UP(EC >> 16, 1);
      if (lane == 0) cin = u_carry;
      u_carry = WP_SHFL(EC >> 16, 31);
      if (((EC & 0xFFFFu) | cin) != (HI & ~C6)) bail = 1;
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
    const u32 RQ = Q & ~E;
    const u32 EI = B & ~E;
    for (u32 m = E; m; m &= m - 1u) {
      u32 j = wp_ffs0(m);
      if (!(LT.base.kind[ce_byte16(v, j)] & 0x80u)) D |= 1u << j;
    }
    // in-string state at the start of the chunk
    const u32 PB = WP_BALLOT((wp_popc(RQ) & 1u) != 0);
    const u32 in0 = (wp_popc(PB & lt) + in_carry) & 1u;
    in_carry = (in_carry + wp_popc(PB)) & 1u;
    const u32 IS = ce_prefix_xor16(RQ) ^ (in0 ? 0xFFFFu : 0u);  // opening quote and content; closing quote excluded
    const u32 SO = RQ & IS, SC = RQ & ~IS;
    const u32 ST = X & ~IS;
    const u32 N = ~(W | X | IS | SC) & 0xFFFFu;  // bytes of scalar literals
    u32 pn = WP_SHFL_UP(N >> 15, 1);
    if (lane == 0) pn = n_carry;
    n_carry = WP_SHFL(N >> 15, 31);
    const u32 NS = N & ~((N << 1) | pn);
    const u32 TF = ST | SO | NS;  // every token, colons and commas included
    // kinds of the structural tokens
    const u32 K1 = ST & XO & XY, K2 = ST & XC & XY, K3 = ST & XO & ~XY, K4 = ST & XC & ~XY, KN = ST & XN;
    const u32 KM = ST & ~(XO | XC | XN);  // commas
    // the token in front of this chunk: the last token of the nearest chunk before it that holds one
    u32 lastk = 0;
    if (TF) {
      const u32 top = 1u << (31u - wp_clz(TF));
      lastk = (top & K1) ? 1u : (top & K2) ? 2u : (top & K3) ? 3u : (top & K4) ? 4u : (top & SO) ? 5u : (top & NS) ? 6u : (top & KN) ? 7u : 8u;
    }
    const u32 NZ = WP_BALLOT(TF != 0);
    const u32 below = NZ & lt;
    const u32 src_k = WP_SHFL(lastk, below ? 31u - wp_clz(below) : 0u);
    const u32 kin = below ? src_k : k_carry;
    {
      const u32 last_any = WP_SHFL(lastk, NZ ? 31u - wp_clz(NZ) : 0u);
      if (NZ) k_carry = last_any;
    }
    // which token may follow which ([upstream encoding/json scanner, protobuf-go internal/encoding/json]: the
    // context-free part of the grammar; key / value alternation needs the container and is checked by the walker)
    const u32 T17 = (TF << 1) | 1u;
    const u32 a1 = (K1 << 1) | (kin == 1u), a3 = (K3 << 1) | (kin == 3u), a5 = (SO << 1) | (kin == 5u);
    const u32 ae = ((K2 | K4 | NS) << 1) | (kin == 2u || kin == 4u || kin == 6u);
    const u32 an = (KN << 1) | (kin == 7u), am = (KM << 1) | (kin == 8u);
    const u32 vstart = (SO | NS | K1 | K3) << 1, vfollow = (KM | K2 | K4) << 1;
    const u32 nx_n = cw_next(T17, an), nx_m = cw_next(T17, am);
    u32 wrong = cw_next(T17, a1) & ~((SO | K2) << 1);
    wrong |= cw_next(T17, a3) & ~(vstart | (K4 << 1));
    wrong |= cw_next(T17, a5) & ~(vfollow | (KN << 1));
    wrong |= cw_next(T17, ae) & ~vfollow;
    wrong |= (nx_n | nx_m) & ~vstart;
    if (kin == 0u) wrong |= (T17 & ~1u) & (0u - (T17 & ~1u)) & ~(K1 << 1);  // the first token of the item: {
    if (wrong & 0x1FFFEu) bail = 1;
    const u32 CF = (nx_m >> 1) & 0xFFFFu, VF = (nx_n >> 1) & 0xFFFFu;
    const u32 TE = TF & ~(KN | KM);  // tokens that are written
    u32 tot;
    // counters carried by prefix scans: tokens, quotes / escape introducers, slow bytes (each at most 512 per round)
    const u32 ex = WP_EXCL_SCAN(wp_popc(TE) | (wp_popc(RQ) << 16), &tot);
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
      const u32 j = wp_ffs0(m), below_j = (1u << j) - 1u;
      if (qi < qcap) {
        u32* p = reinterpret_cast<u32*>(gqend - 8u * (qi + 1u));
        p[0] = ((off + j) & 0xFFFFu) | ((ei + wp_popc(EI & below_j)) << 16);
        p[1] = (di + wp_popc(D & below_j)) & 0xFFFFu;
      }
      qi++;
    }
    const u32 CL = K2 | K4, SQ = K3 | K4;
    for (u32 m = TE; m; m &= m - 1u) {
      const u32 j = wp_ffs0(m), bit = 1u << j;
      u32 kind = 1u + ((CL >> j) & 1u) + (((SQ >> j) & 1u) << 1);
      if (SO & bit) kind = K3_STR;
      if (NS & bit) kind = K3_SCALAR;
      const u32 sn = (qi0 + wp_popc(RQ & (bit - 1u))) >> 1;  // strings: number of the string
      if (ti < tcap) gt[ti] = (off + j) | (kind << 16) | (((CF >> j) & 1u) << 19) | (((VF >> j) & 1u) << 20) | (sn << 21);
      ti++;
    }
  }
  const bool fail = WP_ANY(bail != 0) || in_carry || u_carry || tbase == 0 || tbase > tcap || qbase > qcap || k_carry != 2u;
  if (lane == 0) {
    U4 h = {tbase, qbase, fail ? 1u : 0u, 0xFFFFFFFFu};
    ggr_st16(region, h);
  }
}

// ---- W2: value records ---------------------------------------------------------------------------
struct CwPlaceSh {
  u32 lo[CW_LEVELS + 2];  // last open bracket per content level: record | kind << 16
};

// The context rules of the grammar for token k (c / v: after a comma / colon), pk / pv: the token in front of
// it, bk: kind of the container the boundary between the two lies in, nv: the next token follows a colon.
GGR_DEV bool cw_context_ok(u32 k, u32 c, u32 v, u32 pk, u32 pv, u32 bk, u32 nv) {
  const bool pk_close = pk == K3_RBRACE || pk == K3_RBRACK;
  const bool pk_leaf = pk == K3_STR || pk == K3_SCALAR;
  const bool in_obj = bk == K3_LBRACE, in_arr = bk == K3_LBRACK;
  const bool val_end = pk_close || (pk_leaf && (in_arr || pv));  // an object's values all follow a colon
  const bool first = pk == bk && !c;                              // right behind the opening bracket
  const bool next = val_end && c;
  const bool closes = (k == K3_RBRACE && in_obj) || (k == K3_RBRACK && in_arr);
  const bool is_close = k == K3_RBRACE || k == K3_RBRACK;
  const bool r_close = closes && !c && !v && (pk == bk || val_end);
  const bool r_objval = in_obj && v && !c && pk == K3_STR && !pv;      // "key" : value
  const bool r_key = in_obj && !v && k == K3_STR && nv && (first || next);
  const bool r_elem = in_arr && !v && (first || next);
  return is_close ? r_close : (r_objval || r_key || r_elem);
}

// One item, all 32 lanes: one record per value, in document order, behind the tokens:
// token(16) | record of the enclosing value(16) | level(8) << 32.  Writes n_rec into the header.
GGR_DEV void cw_place_item(CwPlaceSh& S, u8* region, u32 cap, u32 max_rec) {
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u, le = lt | (1u << lane);
  if (cap < 8u) return;
  const U4 h = ggr_ld16(region);
  if (h.z != 0 || h.x < 2u || h.x > 0xFFF0u) return;  // n_rec stays 0xFFFFFFFF
  const u32 n = h.x;
  const u32* tok = reinterpret_cast<const u32*>(region) + 4;
  const u32 rec_off = cw_rec_off(n);
  const u32 q_bytes = 8u * h.y;
  if (rec_off + q_bytes + 64u >= cap * 16u) return;
  u32 rec_cap = (cap * 16u - q_bytes - rec_off - 32u) / 8u;
  if (rec_cap > max_rec) rec_cap = max_rec;
  u32* recs = reinterpret_cast<u32*>(region + rec_off);
  WP_SYNC();  // persistent warps: nobody still reads the previous item's state
  if (lane < CW_LEVELS + 2) S.lo[lane] = 0;
  WP_SYNC();
  i32 depth = 0;
  u32 cnt = 0, c_pk = 0, c_pv = 0, c_x = CW_NONE, c_xk = 0, bad = 0;
  for (u32 base = 0; base < n; base += 32) {
    const u32 i = base + lane;
    const bool act = i < n;
    const u32 t = act ? cw_ldg(tok + i) : 0u;
    const u32 k = K3_KIND(t), c = K3_C(t), v = K3_V(t);
    u32 nv = WP_SHFL(v, lane + 1u);
    if (lane == 31) nv = i + 1u < n ? K3_V(cw_ldg(tok + i + 1u)) : 0u;
    u32 pk = WP_SHFL_UP(k, 1), pv = WP_SHFL_UP(v, 1);
    if (lane == 0) { pk = c_pk; pv = c_pv; }
    const bool op = k == K3_LBRACE || k == K3_LBRACK, cl = k == K3_RBRACE || k == K3_RBRACK;
    const u32 OM = WP_BALLOT(op), CM = WP_BALLOT(cl);
    const i32 Ls = depth + (i32)wp_popc(OM & lt) - (i32)wp_popc(CM & lt);  // brackets open before token i
    if (act && (Ls < 0 || Ls >= CW_LEVELS - 1)) bad = 1;
    const u32 L = (u32)Ls & 31u;
    const bool isval = act && (k == K3_STR || k == K3_SCALAR || op) && !(k == K3_STR && nv);
    const u32 VM = WP_BALLOT(isval);
    const u32 r = isval ? cnt + wp_popc(VM & lt) : CW_NONE;
    // innermost open bracket before a token that is not an opening bracket itself
    const u32 mv = act ? (op ? L + 1u : L) : 0x100u + lane;
    const u32 m = WP_MATCH_ANY(mv);
    const u32 cand = m & OM & lt;
    const u32 pl = cand ? 31u - wp_clz(cand) : 0u;
    const u32 r_pl = WP_SHFL(r, pl), k_pl = WP_SHFL(k, pl);
    u32 e_rec = CW_NONE, e_k = 0;
    if (!op && act) {
      if (cand) {
        e_rec = r_pl;
        e_k = k_pl;
      } else if (L >= 1u && L < CW_LEVELS) {
        const u32 w = S.lo[L];
        e_rec = w & 0xFFFFu;
        e_k = w >> 16;
      }
    }
    // a closing bracket: the container around the pair it closes (what an opening bracket right behind it lives in)
    const u32 mw = (act && (op || cl)) ? (op ? L + 1u : L - 1u) : 0x100u + lane;
    const u32 m2 = WP_MATCH_ANY(mw);
    const u32 cand2 = m2 & OM & lt;
    const u32 pl2 = cand2 ? 31u - wp_clz(cand2) : 0u;
    const u32 r_pl2 = WP_SHFL(r, pl2), k_pl2 = WP_SHFL(k, pl2);
    u32 o_rec = CW_NONE, o_k = 0;
    if (cl) {
      if (cand2) {
        o_rec = r_pl2;
        o_k = k_pl2;
      } else if (L >= 2u && L <= CW_LEVELS) {
        const u32 w = S.lo[L - 1u];
        o_rec = w & 0xFFFFu;
        o_k = w >> 16;
      }
    }
    // what the next token sees in front of it when it is an opening bracket
    const u32 x = op ? r : (cl ? o_rec : e_rec), xk = op ? k : (cl ? o_k : e_k);
    u32 px = WP_SHFL_UP(x, 1), pxk = WP_SHFL_UP(xk, 1);
    if (lane == 0) { px = c_x; pxk = c_xk; }
    const u32 bk = op ? pxk : e_k;
    const u32 prec = op ? px : e_rec;
    if (act) {
      if (i == 0) {
        if (k != K3_LBRACE) bad = 1;
      } else if (!cw_context_ok(k, c, v, pk, pv, bk, nv)) {
        bad = 1;
      }
      if (op && !isval) bad = 1;
      if (i == n - 1u && !(k == K3_RBRACE && e_rec == 0u)) bad = 1;  // the root closes with the last token
      if (isval && i != 0 && prec == CW_NONE) bad = 1;
    }
    if (isval && r < rec_cap) {
      recs[2u * r] = i | (prec << 16);
      recs[2u * r + 1u] = L;
    }
    // last opening bracket per content level of this round
    if (op && act && L + 1u < CW_LEVELS && (m & OM & ~le) == 0u) S.lo[L + 1u] = (r & 0xFFFFu) | (k << 16);
    WP_SYNC();
    depth += (i32)wp_popc(OM) - (i32)wp_popc(CM);
    cnt += wp_popc(VM);
    c_pk = WP_SHFL(k, 31);
    c_pv = WP_SHFL(v, 31);
    c_x = WP_SHFL(x, 31);
    c_xk = WP_SHFL(xk, 31);
  }
  const bool fail = WP_ANY(bad != 0) || depth != 0 || cnt == 0 || cnt > rec_cap;
  if (lane == 0 && !fail) reinterpret_cast<u32*>(region)[3] = cnt;
}

// ---- W3 - W5 ---------------------------------------------------------------------------------------
// value classes
enum {
  CW_MSG = 0, CW_LIST = 1, CW_LISTP = 2, CW_MAP = 3, CW_EMSG = 4,  // containers (EMSG: map entry whose value is a message)
  CW_LEAF = 5, CW_ELEAF = 6, CW_SKIP = 7                            // ELEAF: map entry with a scalar value; SKIP: null
};

template <int MN>
struct CoopWalkT {
  static const u32 MAX_NODE = MN;
  u16 vtok[MN];    // token index of the value
  u16 par[MN];     // record of the enclosing container
  u16 first[MN];   // containers: record index of the first child (children are contiguous)
  u16 slot[MN];    // position of this value among its siblings in emit order (an index into the same level range)
  u16 gfield[MN];  // global field index (MAP / EMSG / ELEAF: the map field)
  u16 aux[MN];     // MSG / EMSG: message type of the value; ELEAF / EMSG after W4: first extra IR node
  u8 cls[MN];
  u8 hdr[MN];      // containers: bytes in front of the children's payload (leaves: tag length until closed)
  u32 body[MN];    // W3: containers: oneof mask, leaves: full size; W4: containers: payload; W5: absolute offset
  u32 ssz[MN];     // W3: containers: mask of fields seen; W4: sizes by slot, then offsets within the parent
  u32 lvl_beg[CW_LEVELS + 2], lvl_cur[CW_LEVELS + 2];
  u32 bail, n_extra, cap;
};
typedef CoopWalkT<256> CoopWalk;       // first tier: 8.9 KB per warp
typedef CoopWalkT<1024> CoopWalkBig;  // second tier: 30.6 KB per warp (large items, every leaf form)
// third tier: request items of thousands of values (a 60 KB list of numbers holds 8 000); 22 bytes per value = 180 KB = one
// warp per SM.  Such an item costs the per-thread parser tens of milliseconds of one lane (mixed replay: half of the
// bytes of the items above 1 KB failed the second tier on the value count alone)
typedef CoopWalkT<8192> CoopWalkHuge;

// ---- cold paths kept out of line: the hot loop of k_encode_type has to fit the instruction caches ----
GGR_DEVN bool cw_long_name_equals(const u8* in, u32 quote_pos, u32 end, const u8* pool, u32 off, u32 len) {
  return str_equals_pool(in, quote_pos, end, pool, off, len);
}
GGR_DEVN int cw_cmp_decoded(const u8* in, u32 a_pos, u32 b_pos, u32 end) { return cmp_str_tokens(in, a_pos, b_pos, end); }

GGR_DEV u32 cw_funnel(u32 lo, u32 hi, u32 sh) {  // bytes of the pair starting at bit sh of lo (sh = 0, 8, 16, 24)
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(lo, hi, sh);
#else
  return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
}
// KeyInfo of the plain bytes in[p, p + n): word loads and funnel shifts (the text is readable 64 bytes past its end)
GGR_DEV void cw_key_info(const u8* in, u32 p, u32 n, KeyInfo* k) {
  const u8* base = in + (p & ~3u);
  const u32 sh = (p & 3u) * 8u;
  u32 h = GGR_KHASH_SEED;
  u32 w[4] = {0, 0, 0, 0};
  const u32 nw = (n + 3u) >> 2;
  u32 lo = ggr_ld4(base);
  for (u32 i = 0; i < nw; i++) {
    const u32 hi = ggr_ld4(base + 4u * (i + 1u));
    u32 x = cw_funnel(lo, hi, sh);
    lo = hi;
    const u32 left = n - 4u * i;
    if (left < 4u) x &= 0xFFFFFFFFu >> (8u * (4u - left));
    h = khash_mix(h, x);
    if (i == 0) w[0] = x;
    else if (i == 1) w[1] = x;
    else if (i == 2) w[2] = x;
    else if (i == 3) w[3] = x;
  }
  k->len = n;
  k->hash = khash_finish(h, n);
  k->w[0] = w[0];
  k->w[1] = w[1];
  k->w[2] = w[2];
  k->w[3] = w[3];
}
// hash_lookup of ggr_json_in.cuh with the tail comparison of long names out of line
GGR_DEV bool cw_hash_lookup(const Tables& t, u32 first, u32 mask, const KeyInfo& k, const u8* in, u32 quote_pos, u32 end, i32* value) {
  u32 slot = k.hash & mask;
  for (u32 probes = 0; probes <= mask; probes++) {
    const u8* ep = t.hash + (size_t)(first + slot) * 32;
    const U4 e = ggr_ld16(ep);
    if (e.z == 0xFFFFFFFFu) return false;
    if (e.x == k.hash && e.z == k.len) {
      const U4 nm = ggr_ld16(ep + 16);
      if (nm.x == k.w[0] && nm.y == k.w[1] && nm.z == k.w[2] && nm.w == k.w[3]) {
        if (k.len <= 16 || cw_long_name_equals(in, quote_pos, end, t.pool, e.y, k.len)) {
          *value = (i32)e.w;
          return true;
        }
      }
    }
    slot = (slot + 1) & mask;
  }
  return false;
}
// enum value by name (plain string token at pos, closing quote at close)
GGR_DEVN bool cw_enum_by_name(const Tables& T, const u8* in, u32 end, i32 child, u32 pos, u32 close, i32* num) {
  KeyInfo ki;
  cw_key_info(in, pos + 1u, close - pos - 1u, &ki);
  const U4 e = ggr_ld16(T.enums + (size_t)child * 16);
  return cw_hash_lookup(T, e.z, e.w, ki, in, pos, end, num);
}

struct CwLeaf {
  u32 type, a, b, flags, body;
  bool zero;
};

// plain decimal integer literal: [-] digits (no leading zero), at most 19 digits, then a delimiter
GGR_DEV bool cw_int_literal(const u8* in, u32 pos, u32 end, bool* neg, u64* mag) {
  u32 j = pos;
  const bool n = in[j] == '-';
  if (n) j++;
  const u32 d0 = j;
  u64 v = 0;
  u32 nd = 0;
  while (j < end && nd < 20u) {
    const u32 c = (u32)in[j] - '0';
    if (c >= 10u) break;
    v = v * 10u + c;
    j++;
    nd++;
  }
  if (nd == 0 || nd > 19u || (nd > 1u && in[d0] == '0')) return false;
  if (j < end) {
    const u32 c = in[j];
    if (!(ggr_is_ws(c) || c == ',' || c == '}' || c == ']')) return false;
  }
  *neg = n;
  *mag = v;
  return true;
}
GGR_DEV bool cw_int_value(u32 kind, bool neg, u64 mag, u64* out) {
  const bool sg = kind_is_signed(kind) || kind == GK_ENUM;
  const int bits = kind == GK_ENUM ? 32 : kind_bits(kind);
  if (sg) {
    const u64 lim = bits == 32 ? 0x80000000ull : 0x8000000000000000ull;
    if (neg ? mag > lim : mag >= lim) return false;
    *out = neg ? (u64)(0 - mag) : mag;  // sign-extended to 64 bits
    return true;
  }
  if (neg) return false;  // "-0" for an unsigned kind: left to the full parser
  if (bits == 32 && mag > 0xFFFFFFFFull) return false;
  *out = mag;
  return true;
}
// scalar token equal to a literal of n bytes followed by a delimiter
GGR_DEV bool cw_scalar_is(const u8* in, u32 pos, u32 end, const char* lit, u32 n) {
  if (end - pos < n) return false;
  for (u32 j = 0; j < n; j++)
    if (in[pos + j] != (u8)lit[j]) return false;
  if (pos + n >= end) return true;
  const u32 c = in[pos + n];
  return ggr_is_ws(c) || c == ',' || c == '}' || c == ']';
}

// quoted plain integer: "[-]digits" filling the string exactly (protojson takes quoted numbers; no spaces, no escapes here)
GGR_DEV bool cw_int_quoted(const u8* in, u32 pos, u32 close, bool* neg, u64* mag) {
  u32 j = pos + 1u;
  const bool n = j < close && in[j] == '-';
  if (n) j++;
  const u32 d0 = j;
  u64 v = 0;
  u32 nd = 0;
  while (j < close && nd < 20u) {
    const u32 c = (u32)in[j] - '0';
    if (c >= 10u) return false;
    v = v * 10u + c;
    j++;
    nd++;
  }
  if (j != close || nd == 0 || nd > 19u || (nd > 1u && in[d0] == '0')) return false;
  *neg = n;
  *mag = v;
  return true;
}

// float / double from a plain decimal literal with at most 15 significant digits and a decimal exponent within
// +-22: mantissa and power of ten are exact doubles, so one multiplication or division rounds correctly
// (Clinger's fast path; everything else - and NaN / Infinity - goes to the full parser of the next tier).
// lim: where the literal has to end (closing quote), or 0 for a bare token that ends at a delimiter.
GGR_DEVN bool cw_float_literal(const u8* in, u32 pos, u32 end, u32 lim, bool is32, u64* bits) {
  static const double P10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
  const u32 stop = lim ? lim : end;
  u32 j = pos;
  bool neg = false;
  if (j < stop && in[j] == '-') { neg = true; j++; }
  u64 m = 0;
  u32 sig = 0, nint = 0;
  const u32 i0 = j;
  while (j < stop && (u32)(in[j] - '0') < 10u) {
    const u32 c = in[j] - '0';
    if (sig || c) { if (sig >= 15u) return false; m = m * 10u + c; sig++; }
    j++;
    nint++;
  }
  if (nint == 0 || (nint > 1u && in[i0] == '0')) return false;
  i32 e10 = 0;
  if (j < stop && in[j] == '.') {
    j++;
    u32 nfrac = 0;
    while (j < stop && (u32)(in[j] - '0') < 10u) {
      const u32 c = in[j] - '0';
      if (sig || c) { if (sig >= 15u) return false; m = m * 10u + c; sig++; }
      e10--;
      j++;
      nfrac++;
    }
    if (nfrac == 0) return false;
  }
  if (j < stop && (in[j] == 'e' || in[j] == 'E')) {
    j++;
    bool eneg = false;
    if (j < stop && (in[j] == '+' || in[j] == '-')) { eneg = in[j] == '-'; j++; }
    u32 ne = 0, ev = 0;
    while (j < stop && (u32)(in[j] - '0') < 10u && ne < 4u) { ev = ev * 10u + (in[j] - '0'); j++; ne++; }
    if (ne == 0 || (j < stop && (u32)(in[j] - '0') < 10u)) return false;
    e10 += eneg ? -(i32)ev : (i32)ev;
  }
  if (lim) {
    if (j != lim) return false;
  } else if (j < end) {
    const u32 c = in[j];
    if (!(ggr_is_ws(c) || c == ',' || c == '}' || c == ']')) return false;
  }
  double d;
  if (m == 0) d = 0.0;
  else if (e10 >= 0 && e10 <= 22) d = (double)m * P10[e10];
  else if (e10 < 0 && e10 >= -22) d = (double)m / P10[-e10];
  else return false;
  if (neg) d = -d;
  if (is32) {
    const float f = (float)d;
    if ((double)f != d) return false;  // would round twice: the full parser rounds the decimal straight to float32
    u32 b;
    memcpy(&b, &f, 4);
    *bits = b;
  } else {
    memcpy(bits, &d, 8);
  }
  return true;
}

// bytes field: the base64 text validated and counted exactly as the per-thread parser does (one lane walks the string)
GGR_DEVN bool cw_bytes_leaf(const u8* in, u32 pos, u32 end, u32* n_out, u32* flags) {
  Rd r;
  r.init(in, pos, end);
  StrInfo si;
  if (scan_string<true>(r, &si) != GST_OK) return false;
  StrIter it;
  it.init(in, pos, end);
  const bool url = (si.flags & SF_URLSAFE) != 0;
  u32 n;
  if (!b64_run<false, Cnt>(it, url, si.dec_len, (Cnt*)0, &n)) return false;
  *n_out = n;
  *flags = (url ? NF_URL : 0u) | ((si.dec_len & 3u) ? 0u : NF_PADDED);
  return true;
}

// google.protobuf.Timestamp from a plain string token (no escapes): RFC 3339 as time.Parse + protojson accept it
GGR_DEVN bool cw_timestamp(const u8* in, u32 pos, u32 end, i64* secs, i32* nanos) {
  StrIter it;
  it.init(in, pos, end);
  return parse_timestamp(it, secs, nanos) == GST_OK;
}

// A map key with \u escapes (what encoding/json writes for < > & in a key) or bytes the full scanner has to judge: decoded
// length and node flags, false when the token is no valid string.  Out of line, full tiers only.
GGR_DEVN bool cw_slow_key(const u8* in, u32 key_pos, u32 end, u32* dec_len, u32* flags) {
  Rd r;
  r.init(in, key_pos, end);
  StrInfo si;
  if (scan_string<false>(r, &si) != GST_OK) return false;
  *dec_len = si.dec_len;
  *flags = (si.flags & SF_ESCAPES) ? NF_ESC : 0u;
  return true;
}

// Leaf value of field f at token t, every form this tier takes.  false: left to the next tier.  Out of line: the hot
// loop of k_encode_type (strings, plain integers, bools) must not carry this code's registers.
GGR_DEVN bool cw_leaf_rare(const Tables& T, const CwIndex& X, const u8* in, u32 end, const FieldD& f, u32 t, CwLeaf* l) {
  const u32 k = K3_KIND(t), pos = K3_POS(t);
  switch (f.kind) {
    case GK_STRING: {
      if (k != K3_STR) return false;
      const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
      if (q0.slow != q1.slow) {
        // \u escapes (what encoding/json writes for < > & and control characters), or bytes that are errors: the full
        // scanner decides and gives the decoded length; the emitter decodes such a string with the per-thread iterator
        Rd r;
        r.init(in, pos, end);
        StrInfo si;
        if (scan_string<false>(r, &si) != GST_OK) return false;
        l->type = N_STR;
        l->a = pos;
        l->b = si.dec_len;
        l->flags = (si.flags & SF_ESCAPES) ? NF_ESC : 0u;
        l->body = varint_size(si.dec_len) + si.dec_len;
        l->zero = si.dec_len == 0;
        return true;
      }
      const u32 nesc = (q1.esc - q0.esc) & 0xFFFFu;
      const u32 len = q1.pos - pos - 1u - nesc;  // a simple escape decodes 2 bytes to 1
      l->type = N_STR;
      l->a = pos;
      l->b = len;
      l->flags = nesc ? (NF_ESC | NF_SIMPLE) : 0u;
      l->body = varint_size(len) + len;
      l->zero = len == 0;
      return true;
    }
    case GK_BOOL: {
      if (k != K3_SCALAR) return false;
      Leaf x;
      if (cw_scalar_is(in, pos, end, "true", 4)) leaf_from_int(GK_BOOL, 1, &x);
      else if (cw_scalar_is(in, pos, end, "false", 5)) leaf_from_int(GK_BOOL, 0, &x);
      else return false;
      l->type = x.type; l->a = x.a; l->b = x.b; l->flags = 0; l->body = x.body; l->zero = x.zero;
      return true;
    }
    case GK_INT32: case GK_INT64: case GK_UINT32: case GK_UINT64: case GK_SINT32: case GK_SINT64:
    case GK_FIXED32: case GK_FIXED64: case GK_SFIXED32: case GK_SFIXED64: case GK_ENUM: {
      u64 v;
      if (k == K3_SCALAR) {
        bool neg;
        u64 mag;
        if (!cw_int_literal(in, pos, end, &neg, &mag) || !cw_int_value(f.kind, neg, mag, &v)) return false;
      } else if (k == K3_STR && f.kind != GK_ENUM) {  // quoted number: how clients send 64-bit values
        const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
        bool neg;
        u64 mag;
        if (q0.slow != q1.slow || q0.esc != q1.esc || !cw_int_quoted(in, pos, q1.pos, &neg, &mag) || !cw_int_value(f.kind, neg, mag, &v)) return false;
      } else if (k == K3_STR && f.kind == GK_ENUM) {  // enum by name
        const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
        if (q0.slow != q1.slow || q0.esc != q1.esc) return false;
        i32 num;
        if (!cw_enum_by_name(T, in, end, f.child, pos, q1.pos, &num)) return false;
        v = (u64)(i64)num;
      } else {
        return false;
      }
      Leaf x;
      leaf_from_int(f.kind, v, &x);
      l->type = x.type; l->a = x.a; l->b = x.b; l->flags = 0; l->body = x.body; l->zero = x.zero;
      return true;
    }
    case GK_FLOAT: case GK_DOUBLE: {
      const bool is32 = f.kind == GK_FLOAT;
      u64 bits;
      if (k == K3_SCALAR) {
        if (!cw_float_literal(in, pos, end, 0u, is32, &bits)) return false;
      } else if (k == K3_STR) {
        const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
        if (q0.slow != q1.slow || q0.esc != q1.esc || q1.pos <= pos + 1u || !cw_float_literal(in, pos + 1u, end, q1.pos, is32, &bits)) return false;
      } else {
        return false;
      }
      l->flags = 0;
      l->zero = bits == 0;  // -0.0 is "set"
      l->a = (u32)bits;
      if (is32) { l->type = N_FIX32; l->b = 0; l->body = 4; }
      else { l->type = N_FIX64; l->b = (u32)(bits >> 32); l->body = 8; }
      return true;
    }
    case GK_BYTES: {
      if (k != K3_STR) return false;
      u32 n, fl;
      if (!cw_bytes_leaf(in, pos, end, &n, &fl)) return false;
      l->type = N_BYTES;
      l->a = pos;
      l->b = n;
      l->flags = fl;
      l->body = varint_size(n) + n;
      l->zero = n == 0;
      return true;
    }
    default:
      return false;
  }
}

// The common leaves inline: strings sized in O(1) from the quote table, plain integer literals, bools.
// FULL = false (the first tier of k_encode_type): nothing else - the kernel stays small and spill-free; FULL = true (second
// tier, run over what the first leaves): every other form through cw_leaf_rare.
// String token t by its two quote entries: raw length | simple escapes << 16 | bit 31 = "no bytes for the full scanner"
// (0 when the counts do not fit: such a string takes the full scanner's path)
GGR_DEV u32 cw_str_pack(const CwIndex& X, u32 t) {
  const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
  const u32 nesc = (q1.esc - q0.esc) & 0xFFFFu, raw = (q1.pos - K3_POS(t) - 1u) & 0xFFFFu;
  return (q0.slow == q1.slow && nesc < 0x8000u) ? (raw | (nesc << 16) | 0x80000000u) : 0u;
}
template <bool FULL>
GGR_DEV bool cw_leaf(const Tables& T, const CwIndex& X, const u8* in, u32 end, const FieldD& f, u32 t, CwLeaf* l) {
  const u32 k = K3_KIND(t), pos = K3_POS(t);
  if (f.kind == GK_STRING) {
    if (k != K3_STR) return false;
    const u32 vinf = cw_str_pack(X, t);
    if (!(vinf >> 31)) return FULL ? cw_leaf_rare(T, X, in, end, f, t, l) : false;  // \u escapes, control characters
    const u32 nesc = (vinf >> 16) & 0x7FFFu;
    const u32 len = (vinf & 0xFFFFu) - nesc;  // a simple escape decodes 2 bytes to 1
    l->type = N_STR;
    l->a = pos;
    l->b = len;
    l->flags = nesc ? (NF_ESC | NF_SIMPLE) : 0u;
    l->body = varint_size(len) + len;
    l->zero = len == 0;
    return true;
  }
  if (k == K3_SCALAR && f.kind != GK_FLOAT && f.kind != GK_DOUBLE && f.kind != GK_BOOL && f.kind != GK_BYTES) {
    bool neg;
    u64 mag, v;
    if (cw_int_literal(in, pos, end, &neg, &mag) && cw_int_value(f.kind, neg, mag, &v)) {
      Leaf x;
      leaf_from_int(f.kind, v, &x);
      l->type = x.type; l->a = x.a; l->b = x.b; l->flags = 0; l->body = x.body; l->zero = x.zero;
      return true;
    }
    return false;  // 1.0, 1e2, out of range: the full parser decides
  }
  if (!FULL) return false;
  return cw_leaf_rare(T, X, in, end, f, t, l);
}

// plain string tokens a < b (raw bytes, Go string order)?  Both known to hold no escapes.
GGR_DEV bool cw_plain_less(const u8* in, u32 a_pos, u32 a_end, u32 b_pos, u32 b_end) {
  const u32 na = a_end - a_pos - 1u, nb = b_end - b_pos - 1u;
  const u32 n = na < nb ? na : nb;
  const u8* a = in + a_pos + 1u;
  const u8* b = in + b_pos + 1u;
  for (u32 j = 0; j < n; j++) {
    const u32 x = a[j], y = b[j];
    if (x != y) return x < y;
  }
  return na < nb;
}

// google.protobuf.Timestamp value at token t: a string in JSON, {seconds = 1, nanos = 2} on the wire; the two varints ride
// in extra IR nodes behind the message node r and are written with it (offset marker 0xFFFFFFFF).  Out of line (rare).
GGR_DEVN bool cw_ts_leaf(const CwIndex& X, const u8* in, u32 end, u32 t, u32 tag, u32 tag_len, u8* ir, u32* io, u32 r, u32 n_rec,
                         u32* n_extra, u32 cap, u32* body) {
  const CwQ q0 = cw_q(X, K3_Q(t)), q1 = cw_q(X, K3_Q(t) + 1u);
  i64 secs = 0;
  i32 nanos = 0;
  if (K3_KIND(t) != K3_STR || q0.slow != q1.slow || q0.esc != q1.esc || !cw_timestamp(in, K3_POS(t), end, &secs, &nanos)) return false;
  const u32 x = wp_atomic_add(n_extra, 2u);
  if (n_rec + x + 2u > cap) return false;
  const u32 sidx = n_rec + x, nidx = n_rec + x + 1u;
  u32 payload = 0;
  if (nanos != 0) payload += 1u + varint_size((u64)(u32)nanos);
  if (secs != 0) payload += 1u + varint_size((u64)secs);
  node_store(ir, nidx, (u32)nanos, 0, GGR_NIL, 1, nanos != 0 ? node_meta(N_VARINT, 0, 16) : node_meta(N_SKIP, 0, 0));
  node_store(ir, sidx, (u32)(u64)secs, (u32)((u64)secs >> 32), nanos != 0 ? nidx : GGR_NIL, 0,
             secs != 0 ? node_meta(N_VARINT, 0, 8) : node_meta(N_SKIP, 0, 0));
  const u32 first_child = secs != 0 ? sidx : (nanos != 0 ? nidx : GGR_NIL);
  node_store(ir, r, payload, first_child, GGR_NIL, 0, node_meta(N_MSG, 0, tag));
  io[sidx] = 0xFFFFFFFFu;
  io[nidx] = 0xFFFFFFFFu;
  *body = tag_len + varint_size(payload) + payload;
  return true;
}

// bytes of the key field of a map entry (tag, length, text) from its IR node
GGR_DEV u32 cw_keypart_of(const u8* ir, u32 x) {
  const u32 klen = node_load(ir, x).y;
  return 1u + varint_size(klen) + klen;
}

// One item, all 32 lanes.  Returns true when the item was handled (IR nodes + offsets written, *res
// filled); false leaves it to the next tier.  region / cap: the item's IR region with the token index of
// cw_tok_item and the value records of cw_place_item in it; ioff: one u32 per IR node of the region.
template <class SH, bool FULL>
GGR_DEV bool cw_type_item(SH& S, const Tables& T, u32 root_msg, const u8* in, u32 start, u32 end, u8* region, u32* ioff, u32 cap,
                          EncResult* res) {
  const u32 lane = wp_lane();
  const u32 lt = (1u << lane) - 1u, le = lt | (1u << lane);
  res->size = 0;
  res->first = GGR_NIL;
  res->n_nodes = 0;
  res->method = 0;
  res->id_pos = res->id_len = 0;
  if (end > CE_MAX_INPUT || cap < 8u || root_msg >= 0xFFFFu) return (CW_WHY(1), false);
  if (end == start) return true;  // reflection.go:354: "" skips protojson
  CwIndex X;
  u32 n_rec;
  {
    const U4 h = ggr_ld16(region);
    if (h.z != 0 || h.w == 0xFFFFFFFFu || h.w == 0u || h.w > SH::MAX_NODE) return (CW_WHY(2), false);
    X.n_tok = h.x;
    X.n_q = h.y;
    X.tok = reinterpret_cast<const u32*>(region) + 4;
    X.qend = region + (size_t)cap * 16u;
    n_rec = h.w;
  }
  // IR nodes go behind the records; they must stay clear of the quote entries
  const u32 rec_off = cw_rec_off(X.n_tok);
  const u32 shift = (rec_off + 8u * n_rec + 15u) >> 4;
  const u32 q_nodes = (8u * X.n_q + 15u) >> 4;
  if (shift + q_nodes + 2u >= cap) return (CW_WHY(3), false);
  const u32 node_cap = cap - shift - q_nodes - 1u;
  if (n_rec > node_cap) return (CW_WHY(4), false);
  u8* ir = region + (size_t)shift * 16u;
  u32* io = ioff + shift;
  WP_SYNC();  // persistent warps: nobody still reads the previous item's state
  if (lane == 0) {
    S.bail = 0;
    S.n_extra = 0;
    S.cap = node_cap;
  }
  if (lane < CW_LEVELS + 2) S.lvl_cur[lane] = 0;
  WP_SYNC();
  // ---- records of k_encode_place, bucketed by level (stable: children of a container stay together) ----
  // until W3 starts: gfield = token, aux = enclosing record, cls = level (document order), slot = new position
  {
    const u32* recs = reinterpret_cast<const u32*>(region + rec_off);
    for (u32 r = lane; r < n_rec; r += 32) {
      const u32 a = cw_ldg(recs + 2u * r), l = cw_ldg(recs + 2u * r + 1u) & 15u;
      S.gfield[r] = (u16)a;
      S.aux[r] = (u16)(a >> 16);
      S.cls[r] = (u8)l;
      wp_atomic_add(&S.lvl_cur[l], 1u);
    }
  }
  WP_SYNC();
  u32 max_level;
  {
    const u32 c = lane < CW_LEVELS ? S.lvl_cur[lane] : 0u;
    u32 tot;
    const u32 ex = WP_EXCL_SCAN(c, &tot);
    max_level = 31u - wp_clz(WP_BALLOT(c != 0) | 1u);
    WP_SYNC();
    if (lane <= CW_LEVELS) {
      S.lvl_beg[lane] = ex;
      S.lvl_cur[lane] = ex;
    }
  }
  WP_SYNC();
  if (S.lvl_beg[1] != 1u) return (CW_WHY(5), false);  // exactly one value at level 0: the root
  for (u32 rb = 0; rb < n_rec; rb += 32) {
    const u32 r = rb + lane;
    const bool act = r < n_rec;
    const u32 l = act ? (u32)S.cls[r] : 0xFFu;
    u32 pos = 0;
    for (u32 rem = WP_BALLOT(act); rem;) {
      const u32 ld = wp_ffs0(rem);
      const u32 lv = WP_SHFL(l, ld);
      const u32 mk = WP_BALLOT(l == lv);
      const u32 b = S.lvl_cur[lv];
      if (l == lv) pos = b + wp_popc(mk & lt);
      WP_SYNC();
      if (lane == ld) S.lvl_cur[lv] = b + wp_popc(mk);
      rem &= ~mk;
    }
    WP_SYNC();
    if (act) {
      S.slot[r] = (u16)pos;
      S.vtok[pos] = S.gfield[r];
    }
  }
  WP_SYNC();
  for (u32 r = lane; r < n_rec; r += 32) {
    const u32 pos = S.slot[r];
    const u32 pd = S.aux[r];  // enclosing record, document order
    S.par[pos] = pd == CW_NONE ? (u16)CW_NONE : S.slot[pd];
    // the first child of a container is the next record of the document
    if (r + 1u < n_rec && (u32)S.aux[r + 1u] == r) S.first[pos] = S.slot[r + 1u];
  }
  WP_SYNC();
  // ---- W3: types, top-down ----
  if (lane == 0) {
    S.cls[0] = CW_MSG;
    S.aux[0] = (u16)root_msg;
    S.gfield[0] = 0;
    S.hdr[0] = 0;
    S.body[0] = 0;
    S.ssz[0] = 0;
    S.slot[0] = 0;
  }
  WP_SYNC();
  if (ggr_msg(T, root_msg).wkt != GGR_WKT_NONE) return (CW_WHY(7), false);
  for (u32 d = 1; d <= max_level; d++) {
    const u32 lb = S.lvl_beg[d], le_ = S.lvl_beg[d + 1];
    for (u32 rb = lb; rb < le_; rb += 32) {
      const u32 r = rb + lane;
      const bool act = r < le_;
      u32 emit = 0, p = 0, pc = CW_SKIP;
      if (act) {
        const u32 i = S.vtok[r];
        p = S.par[r];
        pc = S.cls[p];
        const u32 t = cw_ldg(X.tok + i);
        const u32 k = K3_KIND(t);
        bool ok = true;
        u32 gf = 0, cls = CW_SKIP, aux = 0, hdr = 0, body = 0;
        FieldD f;
        bool in_list = false;
        u32 key_pos = 0, key_end = 0, key_esc = 0, key_dec = 0, key_flags = 0;
        bool key_slow = false;
        bool is_ts = false;
        if (pc == CW_MSG || pc == CW_EMSG) {
          // member of a message: "key" : value
          const u32 kinf = cw_key_pack(X, i);
          if (!(kinf >> 31)) ok = (CW_WHY(101), false);  // escapes in a key: the other tiers
          const MsgD md = ggr_msg(T, S.aux[p]);
          i32 ei = 0;
          if (ok) {
            KeyInfo ki;
            const u32 kpos = kinf & 0xFFFFu;
            cw_key_info(in, kpos, (kinf >> 16) & 0x7FFFu, &ki);
            ok = cw_hash_lookup(T, md.key_hash_first, md.key_hash_mask, ki, in, kpos - 1u, end, &ei);
          }
          if (ok && (u32)ei >= 32u) ok = (CW_WHY(102), false);
          if (ok) {
            emit = (u32)ei;
            gf = md.field_first + emit;
            f = ggr_field(T, gf);
            const u32 bit = 1u << emit;
            if (wp_atomic_or(&S.ssz[p], bit) & bit) ok = (CW_WHY(103), false);  // the same field twice (by either name)
          }
          if (ok) {
            if (gf >= 0xFFFFu) {
              ok = (CW_WHY(104), false);
            } else if (k == K3_SCALAR && cw_scalar_is(in, K3_POS(t), end, "null", 4)) {
              cls = CW_SKIP;
            } else {
              if (f.oneof >= 0 && !(f.flags & (GF_MAP | GF_REPEATED))) {
                const u32 ob = 1u << (f.oneof & 31);
                if (wp_atomic_or(&S.body[p], ob) & ob) ok = (CW_WHY(105), false);
              }
              if (f.flags & GF_MAP) {
                const MsgD ed = ggr_msg(T, (u32)f.child);
                const FieldD kf = ggr_field(T, ed.field_first);
                if (k != K3_LBRACE || kf.kind != GK_STRING) ok = (CW_WHY(106), false);
                cls = CW_MAP;
              } else if (f.flags & GF_REPEATED) {
                if (k != K3_LBRACK) ok = (CW_WHY(107), false);
                if (f.kind == GK_MESSAGE) {
                  const u32 w = ggr_msg(T, (u32)f.child).wkt;
                  if (w != GGR_WKT_NONE && w != GGR_WKT_TIMESTAMP) ok = (CW_WHY(108), false);
                }
                cls = (f.flags & GF_PACKED) ? CW_LISTP : CW_LIST;
                hdr = f.tag_len;
              } else if (f.kind == GK_MESSAGE && ggr_msg(T, (u32)f.child).wkt == GGR_WKT_TIMESTAMP) {
                cls = CW_LEAF;
                is_ts = true;
              } else if (f.kind == GK_MESSAGE) {
                if (k != K3_LBRACE || (u32)f.child >= 0xFFFFu || ggr_msg(T, (u32)f.child).wkt != GGR_WKT_NONE) ok = (CW_WHY(109), false);
                cls = CW_MSG;
                aux = (u32)f.child;
                hdr = f.tag_len;
              } else {
                cls = CW_LEAF;
              }
            }
          }
        } else if (pc == CW_LIST || pc == CW_LISTP) {
          gf = S.gfield[p];
          f = ggr_field(T, gf);
          in_list = true;
          if (f.kind == GK_MESSAGE && ggr_msg(T, (u32)f.child).wkt == GGR_WKT_TIMESTAMP) {
            cls = CW_LEAF;
            is_ts = true;
          } else if (f.kind == GK_MESSAGE) {
            if (k != K3_LBRACE || (u32)f.child >= 0xFFFFu) ok = (CW_WHY(110), false);
            cls = CW_MSG;
            aux = (u32)f.child;
            hdr = f.tag_len;
          } else {
            if (k == K3_SCALAR && cw_scalar_is(in, K3_POS(t), end, "null", 4)) ok = (CW_WHY(111), false);
            cls = CW_LEAF;
          }
        } else if (pc == CW_MAP) {
          // entry of a map with string keys: "key" : value, entries in key order
          gf = S.gfield[p];
          const FieldD mapf = ggr_field(T, gf);
          const MsgD ed = ggr_msg(T, (u32)mapf.child);
          f = ggr_field(T, ed.field_first + 1u);  // the value field
          const u32 kt = cw_ldg(X.tok + i - 1u);
          const CwQ q0 = cw_q(X, K3_Q(kt)), q1 = cw_q(X, K3_Q(kt) + 1u);
          key_pos = K3_POS(kt);
          key_end = q1.pos;
          key_esc = (q1.esc - q0.esc) & 0xFFFFu;
          key_slow = q0.slow != q1.slow;  // \u, control characters: the full scanner (full tiers; the first tier leaves the item)
          if (key_slow && (!FULL || !cw_slow_key(in, key_pos, end, &key_dec, &key_flags))) ok = (CW_WHY(112), false);
          if (ok && r > (u32)S.first[p]) {  // Go emits map entries sorted by key; equal keys are an error
            const u32 pt = cw_ldg(X.tok + (u32)S.vtok[r - 1u] - 1u);
            const CwQ p0 = cw_q(X, K3_Q(pt)), p1 = cw_q(X, K3_Q(pt) + 1u);
            if (p0.slow != p1.slow && !FULL) ok = (CW_WHY(113), false);
            else if (p0.slow == p1.slow && !key_slow && p0.esc == p1.esc && key_esc == 0u) ok = cw_plain_less(in, K3_POS(pt), p1.pos, key_pos, key_end);
            else ok = cw_cmp_decoded(in, K3_POS(pt), key_pos, end) < 0;  // decoded bytes
          }
          in_list = true;
          if (f.kind == GK_MESSAGE) {
            if (k != K3_LBRACE || (u32)f.child >= 0xFFFFu || ggr_msg(T, (u32)f.child).wkt != GGR_WKT_NONE) ok = (CW_WHY(114), false);
            cls = CW_EMSG;
            aux = (u32)f.child;
          } else {
            if (k == K3_SCALAR && cw_scalar_is(in, K3_POS(t), end, "null", 4)) ok = (CW_WHY(115), false);
            cls = CW_ELEAF;
          }
        } else {
          ok = (CW_WHY(116), false);
        }
        if (ok && is_ts) {
          if (!FULL || !cw_ts_leaf(X, in, end, t, f.tag, f.tag_len, ir, io, r, n_rec, &S.n_extra, S.cap, &body)) ok = (CW_WHY(119), false);
        } else if (ok && (cls == CW_LEAF || cls == CW_ELEAF)) {
          CwLeaf l;
          if ((k != K3_STR && k != K3_SCALAR) || !cw_leaf<FULL>(T, X, in, end, f, t, &l)) {
            ok = (CW_WHY(117), false);
          } else if (cls == CW_LEAF) {
            const bool packed = pc == CW_LISTP;
            const u32 tag = packed ? 0u : f.tag, tag_len = packed ? 0u : f.tag_len;
            const bool live = in_list || (f.flags & GF_PRESENCE) || !l.zero;
            node_store(ir, r, l.a, l.b, GGR_NIL, 0, live ? node_meta(l.type, l.flags, tag) : node_meta(N_SKIP, 0, 0));
            body = live ? tag_len + l.body : 0u;
          } else {
            // ENTRY { key = 1, value = 2 }: three IR nodes
            const u32 x = wp_atomic_add(&S.n_extra, 2u);
            const u32 klen = key_slow ? key_dec : key_end - key_pos - 1u - key_esc;  // a simple escape decodes 2 bytes to 1
            const u32 keypart = 1u + varint_size(klen) + klen;
            const u32 payload = keypart + f.tag_len + l.body;
            const FieldD mapf = ggr_field(T, gf);
            if (n_rec + x + 2u > S.cap) {
              ok = (CW_WHY(118), false);
            } else {
              node_store(ir, r, payload, GGR_NIL, GGR_NIL, 0, node_meta(N_ENTRY, 0, mapf.tag));
              node_store(ir, n_rec + x, key_pos, klen, GGR_NIL, 0, node_meta(N_STR, key_slow ? key_flags : (key_esc ? (NF_ESC | NF_SIMPLE) : 0u), 0x0Au));
              node_store(ir, n_rec + x + 1u, l.a, l.b, GGR_NIL, 1, node_meta(l.type, l.flags, f.tag));
              aux = x;
              hdr = mapf.tag_len + varint_size(payload);  // offset of the key node within the entry
              body = mapf.tag_len + varint_size(payload) + payload;
            }
          }
        }
        // a null member: no bytes, but the emitter walks every record's node - it must not meet what an earlier
        // batch left in this slot of the IR
        if (ok && cls == CW_SKIP) node_store(ir, r, 0, 0, GGR_NIL, 0, node_meta(N_SKIP, 0, 0));
        if (!ok) S.bail = 1;
        S.gfield[r] = (u16)gf;
        S.cls[r] = (u8)cls;
        S.aux[r] = (u16)aux;
        S.hdr[r] = (u8)hdr;
        S.body[r] = body;
        S.ssz[r] = 0;
        S.slot[r] = (u16)emit;
      }
    }
    WP_SYNC();
    if (S.bail) return false;
    // position among the siblings in emit order: fields by the mask of fields seen, elements and entries as they come
    for (u32 r = lb + lane; r < le_; r += 32) {
      const u32 p = S.par[r];
      const u32 pc = S.cls[p];
      if (pc == CW_MSG || pc == CW_EMSG) S.slot[r] = (u16)((u32)S.first[p] + wp_popc(S.ssz[p] & ((1u << S.slot[r]) - 1u)));
      else S.slot[r] = (u16)r;
    }
    WP_SYNC();
  }
  // ---- W4: sizes, bottom-up ----
  // the oneof masks and field masks of the containers are no longer needed
  for (u32 r = lane; r < n_rec; r += 32) {
    const u32 c = S.cls[r];
    if (c <= CW_EMSG) S.body[r] = 0;
  }
  WP_SYNC();
  for (u32 d = max_level; d >= 1; d--) {
    const u32 lb = S.lvl_beg[d], le_ = S.lvl_beg[d + 1];
    // A: full size of every value of the level into its emit-order slot
    for (u32 r = lb + lane; r < le_; r += 32) {
      const u32 c = S.cls[r];
      u32 full;
      if (c >= CW_LEAF) {
        full = S.body[r];
      } else {
        const u32 payload = S.body[r];
        const u32 gf = S.gfield[r];
        const u32 tag = ggr_ld4(T.fields + (size_t)gf * 32 + 4);
        u32 h;
        if (c == CW_MSG) {
          h = (u32)S.hdr[r] + varint_size(payload);
          node_store(ir, r, payload, GGR_NIL, GGR_NIL, 0, node_meta(N_MSG, 0, tag));
          full = h + payload;
        } else if (c == CW_LIST || c == CW_MAP) {
          h = 0;
          // empty list / map: field absent (elements and entries are never empty, so payload == 0 means no children)
          node_store(ir, r, payload, GGR_NIL, GGR_NIL, 0, node_meta(payload ? (c == CW_LIST ? N_LIST : N_MAP) : N_SKIP, 0, 0));
          full = payload;
        } else if (c == CW_LISTP) {
          const bool empty = payload == 0;
          h = empty ? 0u : (u32)S.hdr[r] + varint_size(payload);
          node_store(ir, r, payload, GGR_NIL, GGR_NIL, 0, empty ? node_meta(N_SKIP, 0, 0) : node_meta(N_LIST, NF_PACKED, tag));
          full = h + payload;
        } else {  // CW_EMSG: ENTRY { key, message value }
          const u32 i = S.vtok[r];
          const u32 kt = cw_ldg(X.tok + i - 1u);
          const CwQ q0 = cw_q(X, K3_Q(kt)), q1 = cw_q(X, K3_Q(kt) + 1u);
          const u32 key_esc = (q1.esc - q0.esc) & 0xFFFFu;
          const u32 key_pos = K3_POS(kt);
          const bool kslow = q0.slow != q1.slow;  // judged in the type pass already: full tiers only
          u32 kdec = 0, kflags = 0;
          if (kslow && (!FULL || !cw_slow_key(in, key_pos, end, &kdec, &kflags))) S.bail = 1;
          const u32 klen = kslow ? kdec : q1.pos - key_pos - 1u - key_esc;
          const u32 keypart = 1u + varint_size(klen) + klen;
          const FieldD mapf = ggr_field(T, gf);
          const MsgD ed = ggr_msg(T, (u32)mapf.child);
          const FieldD vf = ggr_field(T, ed.field_first + 1u);
          const u32 vfull = vf.tag_len + varint_size(payload) + payload;
          const u32 ent = keypart + vfull;
          const u32 x = wp_atomic_add(&S.n_extra, 2u);
          if (n_rec + x + 2u > S.cap) {
            S.bail = 1;
            h = 0;
          } else {
            const u32 eh = mapf.tag_len + varint_size(ent);
            node_store(ir, r, ent, GGR_NIL, GGR_NIL, 0, node_meta(N_ENTRY, 0, mapf.tag));
            node_store(ir, n_rec + x, key_pos, klen, GGR_NIL, 0, node_meta(N_STR, kslow ? kflags : (key_esc ? (NF_ESC | NF_SIMPLE) : 0u), 0x0Au));
            node_store(ir, n_rec + x + 1u, payload, GGR_NIL, GGR_NIL, 1, node_meta(N_MSG, 0, vf.tag));
            S.aux[r] = (u16)x;
            h = eh + keypart + vf.tag_len + varint_size(payload);
            if (h > 255u) S.bail = 1;
            S.vtok[r] = (u16)eh;  // W5: entry header (the token is no longer needed)
          }
          full = h + payload;
        }
        S.hdr[r] = (u8)h;
      }
      S.ssz[S.slot[r]] = full;
    }
    WP_SYNC();
    if (S.bail) return false;
    // B: segmented exclusive scan over the slots (segments = children of one container)
    for (u32 sb = lb; sb < le_; sb += 32) {
      const u32 s = sb + lane;
      const bool act = s < le_;
      const u32 p = act ? (u32)S.par[s] : 0x10000u + lane;
      const u32 v = act ? S.ssz[s] : 0u;
      u32 tot;
      const u32 ex = WP_EXCL_SCAN(v, &tot);
      u32 pp = WP_SHFL_UP(p, 1);
      const bool head = lane == 0 || pp != p;
      const u32 HM = WP_BALLOT(head);
      const u32 s0 = 31u - wp_clz(HM & le);
      const u32 ex0 = WP_SHFL(ex, s0);
      const u32 before = act ? S.body[p] : 0u;
      const bool last = act && (lane == 31 || ((HM >> (lane + 1u)) & 1u) || s + 1u == le_);
      WP_SYNC();
      if (act) S.ssz[s] = before + ex - ex0;
      if (last) S.body[p] = before + ex - ex0 + v;
      WP_SYNC();
    }
  }
  const u32 total = S.body[0];
  // the lock-step emitter stages an item in shared memory; larger ones are written in place - second tier only
  if (total > (FULL ? 0x0FFFFFFFu : CE_STAGE)) return (CW_WHY(10), false);
  WP_SYNC();
  // ---- W5: offsets, top-down ----
  if (lane == 0) S.body[0] = 0;
  WP_SYNC();
  for (u32 d = 1; d <= max_level; d++) {
    const u32 lb = S.lvl_beg[d], le_ = S.lvl_beg[d + 1];
    for (u32 r = lb + lane; r < le_; r += 32) {
      const u32 p = S.par[r];
      const u32 a = S.body[p] + (u32)S.hdr[p] + S.ssz[S.slot[r]];
      const u32 c = S.cls[r];
      io[r] = a;
      if (c == CW_ELEAF) {
        const u32 x = n_rec + S.aux[r];
        io[x] = a + (u32)S.hdr[r];
        io[x + 1u] = a + (u32)S.hdr[r] + cw_keypart_of(ir, x);
      } else if (c == CW_EMSG) {
        const u32 x = n_rec + S.aux[r];
        const u32 eh = S.vtok[r];
        io[x] = a + eh;
        io[x + 1u] = a + eh + cw_keypart_of(ir, x);
      }
      if (c <= CW_EMSG) S.body[r] = a;
    }
    WP_SYNC();
  }
  res->size = total;
  res->first = GGR_NIL;
  res->n_nodes = n_rec + S.n_extra;
  res->method = shift;  // where the IR nodes of this item start within its region (in nodes): travels with n_nodes
  return true;
}

// ---- item edge of the walker's kernels (the host simulation calls the same functions) ----------------------------------
// Admission is ce_admit's.  An empty item has no token index and no value records: k_encode_tok3 and k_encode_place skip
// it (cw_indexed), k_encode_type takes it as an empty message (cw_type_item).
GGR_DEV bool cw_indexed(u64 a, u64 b) { return b != a && ce_admit(a, b); }

// k_encode_tok3, item `item` of the batch whose input starts at a0.  tl / ph: as cw_tok_item.
GGR_DEV void cw_tok_step(CwTile* tl, u32& ph, const CwLut& lut, const u8* in, const u64* in_off, u64 a0, u8* ir, long long item) {
  const u64 a = in_off[item], b = in_off[item + 1];
  if (!cw_indexed(a, b)) return;
  const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
  const u32 s0 = (u32)(a & 15ull);
  cw_tok_item(tl, ph, lut, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, r.cap);
}

// k_encode_place
GGR_DEV void cw_place_step(CwPlaceSh& S, const u64* in_off, u64 a0, u8* ir, long long item) {
  const u64 a = in_off[item], b = in_off[item + 1];
  if (!cw_indexed(a, b)) return;
  const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
  cw_place_item(S, ir + r.node_off * 16, r.cap, CoopWalkHuge::MAX_NODE);
}

// k_encode_type: true when the item was taken (IR nodes and their offsets written, *res filled).
template <class SH, bool FULL>
GGR_DEV bool cw_type_step(SH& S, const Tables& T, u32 n_msgs, const i32* msg_id, const u8* in, const u64* in_off, u64 a0, u8* ir,
                          u32* ioff, long long item, EncResult* res) {
  const u64 a = in_off[item], b = in_off[item + 1];
  const i32 m = msg_id[item];
  res->size = 0;
  res->n_nodes = 0;
  res->method = 0;
  if (m < 0 || (u32)m >= n_msgs || !ce_admit(a, b)) return (CW_WHY(1), false);
  const GgrRegion r = ggr_item_region(a0, a, b, (u64)item);
  const u32 s0 = (u32)(a & 15ull);
  return cw_type_item<SH, FULL>(S, T, (u32)m, in + (a & ~15ull), s0, s0 + (u32)(b - a), ir + r.node_off * 16, ioff + r.node_off, r.cap,
                                res);
}

// Lane 0: a taken item's size, status and nodes (for k_encode_coop_emit); one not taken goes to `left`.
GGR_DEV void cw_type_publish(bool ok, const EncResult& res, long long item, u32* size, u32* first, i32* status, u32* nnodes,
                             GgrWork left) {
  if (wp_lane() != 0) return;
  if (ok) {
    size[item] = res.size;
    first[item] = GGR_NIL;
    status[item] = GST_OK;
    nnodes[item] = ce_nodes_word(res.n_nodes, res.method);  // cw_type_item: method = where the nodes start
  } else {
    size[item] = 0;
    nnodes[item] = 0;
    first[item] = GGR_NIL;
    left.item[ggr_atomic_add_u32(&left.h->n, 1u)] = (u32)item;
  }
}
