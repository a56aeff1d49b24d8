// ggr_float.cuh - float/double <-> decimal text on the device, bit-exact with Go's strconv as the
// reference path uses it:
//   print: strconv.AppendFloat(x, 'e'|'f', -1, 32|64) under protojson's appendFloat rules
//          (/root/reference/pkg/grpc/reflection.go:381 -> [upstream internal/encoding/json/encode.go])
//          shortest round-trip digits, computed Ryu-style (Ulf Adams, PLDI 2018) from exact 125-bit
//          powers of five (ggr_float_tables.h, generated with big-integer arithmetic);
//   parse: strconv.ParseFloat(token, 32|64) (reflection.go:355 -> [upstream protojson unmarshalFloat])
//          exact: Clinger's fast path when the decimal and the power of ten are exactly
//          representable, otherwise a big-integer evaluation with round-half-even (slow but
//          correctly rounded; an Eisel-Lemire fast path is a round-2 optimisation).
#pragma once
#include "ggr_float_tables.h"
#include "ggr_prim.cuh"
#include "ggr_json_in.cuh"

// ------------------------------------------------------------------------------------------------
// shortest digits
// ------------------------------------------------------------------------------------------------
GGR_DEV u32 fl_pow5bits(i32 e) { return (u32)(((u32)e * 1217359u) >> 19) + 1u; }
GGR_DEV u32 fl_log10pow2(i32 e) { return ((u32)e * 78913u) >> 18; }
GGR_DEV u32 fl_log10pow5(i32 e) { return ((u32)e * 732923u) >> 20; }
GGR_DEV u32 fl_pow5factor(u64 v) {
  u32 c = 0;
  for (;;) {
    u64 q = v / 5;
    if (q * 5 != v) break;
    v = q;
    c++;
  }
  return c;
}
GGR_DEV bool fl_mult_pow5(u64 v, u32 p) { return fl_pow5factor(v) >= p; }
GGR_DEV bool fl_mult_pow2(u64 v, u32 p) { return (v & ((1ull << p) - 1ull)) == 0; }
GGR_DEV void fl_mul64(u64 a, u64 b, u64* lo, u64* hi) {
  *lo = a * b;
  *hi = ggr_mulhi64(a, b);
}
// (m * mul) >> j for a 128-bit mul (mul[0] low), 64 <= j < 128+64
GGR_DEV u64 fl_mulshift(u64 m, u64 mul0, u64 mul1, i32 j) {
  u64 lo0, hi0, lo2, hi2;
  fl_mul64(m, mul0, &lo0, &hi0);
  fl_mul64(m, mul1, &lo2, &hi2);
  u64 sum = hi0 + lo2;
  if (sum < hi0) hi2++;
  i32 d = j - 64;
  if (d == 0) return sum;
  if (d >= 64) return hi2 >> (d - 64);
  return (hi2 << (64 - d)) | (sum >> d);
}

struct FlDec {
  u64 digits;  // shortest decimal significand
  i32 exp;     // value = digits * 10^exp
};

// Shortest decimal that round-trips an IEEE value with `mbits` mantissa bits (52 / 23).
// Not for zero, NaN, Inf.
GGR_DEV FlDec fl_shortest(u64 ieee_m, u32 ieee_e, int mbits, int bias) {
  i32 e2;
  u64 m2;
  if (ieee_e == 0) {
    e2 = 1 - bias - mbits - 2;
    m2 = ieee_m;
  } else {
    e2 = (i32)ieee_e - bias - mbits - 2;
    m2 = (1ull << mbits) | ieee_m;
  }
  const bool accept = (m2 & 1ull) == 0;
  const u64 mv = 4 * m2;
  const u32 mm_shift = (ieee_m != 0 || ieee_e <= 1) ? 1u : 0u;
  u64 vr, vp, vm;
  i32 e10;
  bool vm_tz = false, vr_tz = false;
  if (e2 >= 0) {
    u32 q = fl_log10pow2(e2) - (e2 > 3 ? 1u : 0u);
    e10 = (i32)q;
    i32 k = 125 + (i32)fl_pow5bits((i32)q) - 1;
    i32 i = -e2 + (i32)q + k;
    u64 c0 = GGR_POW5_INV[q][0], c1 = GGR_POW5_INV[q][1];
    vr = fl_mulshift(4 * m2, c0, c1, i);
    vp = fl_mulshift(4 * m2 + 2, c0, c1, i);
    vm = fl_mulshift(4 * m2 - 1 - mm_shift, c0, c1, i);
    if (q <= 21) {
      u32 mod5 = (u32)(mv % 5);
      if (mod5 == 0) vr_tz = fl_mult_pow5(mv, q);
      else if (accept) vm_tz = fl_mult_pow5(mv - 1 - mm_shift, q);
      else vp -= fl_mult_pow5(mv + 2, q) ? 1u : 0u;
    }
  } else {
    u32 q = fl_log10pow5(-e2) - (-e2 > 1 ? 1u : 0u);
    e10 = (i32)q + e2;
    i32 i = -e2 - (i32)q;
    i32 k = (i32)fl_pow5bits(i) - 125;
    i32 j = (i32)q - k;
    u64 c0 = GGR_POW5[i][0], c1 = GGR_POW5[i][1];
    vr = fl_mulshift(4 * m2, c0, c1, j);
    vp = fl_mulshift(4 * m2 + 2, c0, c1, j);
    vm = fl_mulshift(4 * m2 - 1 - mm_shift, c0, c1, j);
    if (q <= 1) {
      vr_tz = true;
      if (accept) vm_tz = mm_shift == 1;
      else --vp;
    } else if (q < 63) {
      vr_tz = fl_mult_pow2(mv, q);
    }
  }
  i32 removed = 0;
  u32 last = 0;
  u64 out;
  if (vm_tz || vr_tz) {
    for (;;) {
      u64 vp10 = vp / 10, vm10 = vm / 10;
      if (vp10 <= vm10) break;
      u32 vm_mod = (u32)(vm - 10 * vm10);
      u64 vr10 = vr / 10;
      u32 vr_mod = (u32)(vr - 10 * vr10);
      vm_tz &= vm_mod == 0;
      vr_tz &= last == 0;
      last = vr_mod;
      vr = vr10;
      vp = vp10;
      vm = vm10;
      removed++;
    }
    if (vm_tz) {
      for (;;) {
        u64 vm10 = vm / 10;
        u32 vm_mod = (u32)(vm - 10 * vm10);
        if (vm_mod != 0) break;
        u64 vp10 = vp / 10, vr10 = vr / 10;
        u32 vr_mod = (u32)(vr - 10 * vr10);
        vr_tz &= last == 0;
        last = vr_mod;
        vr = vr10;
        vp = vp10;
        vm = vm10;
        removed++;
      }
    }
    if (vr_tz && last == 5 && (vr & 1ull) == 0) last = 4;  // round half even
    out = vr + (((vr == vm && (!accept || !vm_tz)) || last >= 5) ? 1u : 0u);
  } else {
    bool round_up = false;
    for (;;) {
      u64 vp10 = vp / 10, vm10 = vm / 10;
      if (vp10 <= vm10) break;
      u64 vr10 = vr / 10;
      u32 vr_mod = (u32)(vr - 10 * vr10);
      round_up = vr_mod >= 5;
      vr = vr10;
      vp = vp10;
      vm = vm10;
      removed++;
    }
    out = vr + ((vr == vm || round_up) ? 1u : 0u);
  }
  FlDec d;
  d.digits = out;
  d.exp = e10 + removed;
  return d;
}

// Writes a finite or non-finite float the way protojson does.  `bits` holds the IEEE bits
// (float32 in the low word when is32).
// noinline: floats are rare on the hot path; keep their frames and registers out of the walkers
template <class W>
GGR_DEVN void put_float_go(W& w, u64 bits, bool is32) {
  const int mbits = is32 ? 23 : 52, ebits = is32 ? 8 : 11, bias = is32 ? 127 : 1023;
  bool neg = (bits >> (mbits + ebits)) & 1;
  u32 e = (u32)((bits >> mbits) & ((1u << ebits) - 1u));
  u64 m = bits & ((1ull << mbits) - 1ull);
  if (e == (1u << ebits) - 1u) {
    if (m != 0) {
      w.put(LIT4('"', 'N', 'a', 'N'), 4);
      w.put1('"');
    } else {
      w.put1('"');
      if (neg) w.put1('-');
      w.put(LIT4('I', 'n', 'f', 'i'), 4);
      w.put(LIT4('n', 'i', 't', 'y'), 4);
      w.put1('"');
    }
    return;
  }
  if (neg) w.put1('-');
  if (e == 0 && m == 0) {
    w.put1('0');
    return;
  }
  FlDec d = fl_shortest(m, e, mbits, bias);
  // digits, most significant first
  u8 dg[20];
  int nd = 0;
  {
    u64 v = d.digits;
    u8 tmp[20];
    int k = 0;
    do {
      u64 q = v / 10;
      tmp[k++] = (u8)('0' + (u32)(v - q * 10));
      v = q;
    } while (v);
    // fl_shortest never leaves trailing zeros except through rounding (e.g. 9.99 -> 10.0)
    int lo = 0;
    while (lo < k - 1 && tmp[lo] == '0') {
      lo++;
      d.exp++;
    }
    for (int i = k - 1; i >= lo; i--) dg[nd++] = tmp[i];
  }
  int x = nd + d.exp;  // value = 0.DIGITS * 10^x
  if (x < -5 || x > 21) {
    // 'e' format: d.ddde[-+]XX with protojson's "e-0X" -> "e-X" clean-up
    w.put1(dg[0]);
    if (nd > 1) {
      w.put1('.');
      for (int i = 1; i < nd; i++) w.put1(dg[i]);
    }
    int ex = x - 1;
    w.put1('e');
    if (ex < 0) {
      w.put1('-');
      ex = -ex;
      if (ex >= 100) w.put1('0' + ex / 100);
      if (ex >= 10) w.put1('0' + ex / 10 % 10);
      w.put1('0' + ex % 10);
    } else {
      w.put1('+');
      if (ex >= 100) w.put1('0' + ex / 100);
      w.put1('0' + ex / 10 % 10);
      w.put1('0' + ex % 10);
    }
    return;
  }
  if (x <= 0) {
    w.put('0' | ('.' << 8), 2);
    for (int i = 0; i < -x; i++) w.put1('0');
    for (int i = 0; i < nd; i++) w.put1(dg[i]);
  } else if (nd <= x) {
    for (int i = 0; i < nd; i++) w.put1(dg[i]);
    for (int i = nd; i < x; i++) w.put1('0');
  } else {
    for (int i = 0; i < x; i++) w.put1(dg[i]);
    w.put1('.');
    for (int i = x; i < nd; i++) w.put1(dg[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// decimal -> binary, correctly rounded
// ------------------------------------------------------------------------------------------------
#define GGR_BIG_WORDS 40
// little-endian u32 words; NW words of capacity
template <int NW>
struct BigN {
  u32 w[NW];
  int n;  // words in use (no leading zero words), 0 for zero
};
using Big = BigN<GGR_BIG_WORDS>;
template <int NW>
GGR_DEV void big_set64(BigN<NW>& b, u64 v) {
  b.n = 0;
  if (v) {
    b.w[b.n++] = (u32)v;
    if (v >> 32) b.w[b.n++] = (u32)(v >> 32);
  }
}
template <int NW>
GGR_DEV bool big_mul_small(BigN<NW>& b, u32 f, u32 add) {  // b = b*f + add; false on capacity overflow
  u64 carry = add;
  for (int i = 0; i < b.n; i++) {
    u64 t = (u64)b.w[i] * f + carry;
    b.w[i] = (u32)t;
    carry = t >> 32;
  }
  if (carry) {
    if (b.n >= NW) return false;
    b.w[b.n++] = (u32)carry;
  }
  return true;
}
template <int NW>
GGR_DEV bool big_mul_pow5(BigN<NW>& b, u32 k) {
  while (k >= 13) {
    if (!big_mul_small(b, 1220703125u, 0)) return false;
    k -= 13;
  }
  u32 f = 1;
  for (u32 i = 0; i < k; i++) f *= 5;
  return f == 1 ? true : big_mul_small(b, f, 0);
}
template <int NW>
GGR_DEV int big_bitlen(const BigN<NW>& b) {
  if (b.n == 0) return 0;
  u32 top = b.w[b.n - 1];
  return 32 * (b.n - 1) + (32 - (ggr_clz64((u64)top) - 32));
}
template <int NW>
GGR_DEV u32 big_bit(const BigN<NW>& b, int i) { return (i < 0 || (i >> 5) >= b.n) ? 0u : (b.w[i >> 5] >> (i & 31)) & 1u; }
template <int NW>
GGR_DEV int big_cmp(const BigN<NW>& a, const BigN<NW>& b) {
  if (a.n != b.n) return a.n < b.n ? -1 : 1;
  for (int i = a.n - 1; i >= 0; i--)
    if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
  return 0;
}
template <int NW>
GGR_DEV void big_sub(BigN<NW>& a, const BigN<NW>& b) {  // a -= b, a >= b
  u64 borrow = 0;
  for (int i = 0; i < a.n; i++) {
    u64 t = (u64)a.w[i] - (i < b.n ? b.w[i] : 0u) - borrow;
    a.w[i] = (u32)t;
    borrow = (t >> 63) & 1u;
  }
  while (a.n > 0 && a.w[a.n - 1] == 0) a.n--;
}
template <int NW>
GGR_DEV bool big_shl1_add(BigN<NW>& a, u32 bit) {  // a = a*2 + bit
  u32 carry = bit;
  for (int i = 0; i < a.n; i++) {
    u32 t = a.w[i];
    a.w[i] = (t << 1) | carry;
    carry = t >> 31;
  }
  if (carry) {
    if (a.n >= NW) return false;
    a.w[a.n++] = carry;
  }
  return true;
}
template <int NW>
GGR_DEV bool big_shl(BigN<NW>& a, u32 s) {  // a <<= s; false on capacity overflow
  if (a.n == 0) return true;
  const int ws = (int)(s >> 5), bs = (int)(s & 31u);
  const int n = a.n + ws + (bs != 0 && (a.w[a.n - 1] >> (32 - bs)) != 0 ? 1 : 0);
  if (n > NW) return false;
  for (int i = n - 1; i >= 0; i--) {
    const int j = i - ws;  // source word
    const u32 hi = j >= 0 && j < a.n ? a.w[j] : 0u;
    const u32 lo = j - 1 >= 0 && j - 1 < a.n ? a.w[j - 1] : 0u;
    a.w[i] = bs ? (hi << bs) | (lo >> (32 - bs)) : hi;
  }
  a.n = n;
  return true;
}

// q64 * 2^E (+ something smaller than one unit of q64 when sticky) -> IEEE bits, round half even.
// q64 has its top bit set.  Returns false on overflow to infinity.
GGR_DEV bool fl_round_ieee(u64 q64, i32 E, bool sticky, bool is32, u64* out) {
  const int mbits = is32 ? 23 : 52, bias = is32 ? 127 : 1023, emax = is32 ? 255 : 2047;
  // value = q64 * 2^E, q64 in [2^63, 2^64)  ->  1.xxx * 2^(E+63)
  i32 be = E + 63 + bias;  // biased exponent if normal
  int drop = 63 - mbits;   // bits to drop for a normal number
  if (be <= 0) {
    drop += 1 - be;  // subnormal: shift further so the exponent field becomes 0
    be = 0;
  }
  u64 mant;
  bool up;
  if (drop >= 64) {
    // everything is below half an ulp unless drop == 64 and q64 > 2^63 (or == with sticky)
    mant = 0;
    up = drop == 64 && (q64 > (1ull << 63) || (q64 == (1ull << 63) && sticky));
    if (drop > 64) up = false;
  } else {
    mant = q64 >> drop;
    u64 rem = q64 & ((1ull << drop) - 1ull);
    u64 half = 1ull << (drop - 1);
    up = rem > half || (rem == half && (sticky || (mant & 1ull)));
  }
  mant += up ? 1u : 0u;
  if (be == 0) {
    if (mant >> mbits) be = 1;  // rounded up into the normal range (mant == 2^mbits)
    *out = ((u64)be << mbits) | (mant & ((1ull << mbits) - 1ull));
    if (be == 1) *out = ((u64)1 << mbits) | (mant & ((1ull << mbits) - 1ull));
    return true;
  }
  if (mant >> (mbits + 1)) {  // mantissa overflowed to 2^(mbits+1)
    mant >>= 1;
    be++;
  }
  if (be >= emax) return false;
  *out = ((u64)be << mbits) | (mant & ((1ull << mbits) - 1ull));
  return true;
}

// value = D * 10^k with D given as a Big (D != 0).  sticky_in: digits beyond the ones in D were
// nonzero.  Returns false on overflow.
GGR_DEVN bool fl_from_big(Big& D, i32 k, bool sticky_in, bool is32, u64* out) {
  // quick range cuts (D < 10^(10*n_words) loosely): decimal magnitude ~ 10^(digits + k)
  int bl = big_bitlen(D);
  // digits10 ~ bl * 0.30103
  i32 mag10 = (i32)((bl * 1233) >> 12) + k;  // floor(log10(value)) within +-1
  if (mag10 > 330) return false;
  if (mag10 < -400) {
    *out = 0;
    return true;
  }
  if (k >= 0) {
    if (!big_mul_pow5(D, (u32)k)) return false;  // cannot happen within the range cut
    int L = big_bitlen(D);
    // top 64 bits
    u64 q = 0;
    for (int i = 0; i < 64; i++) q = (q << 1) | big_bit(D, L - 1 - i);
    bool sticky = sticky_in;
    if (!sticky) {
      for (int i = 0; i < L - 64 && !sticky; i++) sticky = big_bit(D, i) != 0;
    }
    return fl_round_ieee(q, L - 64 + k, sticky, is32, out);
  }
  // k < 0: quotient of D by R = 5^-k, bit by bit
  Big R;
  big_set64(R, 1);
  if (!big_mul_pow5(R, (u32)(-k))) return false;
  int LD = big_bitlen(D), LR = big_bitlen(R);
  int s = LR - LD + 65;  // (D << s) / R has 65 or 66 bits
  if (s < 0) s = 0;
  Big rem;
  rem.n = 0;
  u64 q = 0;
  int qbits = 0;     // significant quotient bits produced so far
  bool sticky = sticky_in;
  i32 extra = 0;     // quotient bits produced after the 64 kept ones
  int total = LD + s;
  for (int i = total - 1; i >= 0; i--) {
    u32 bit = i >= s ? big_bit(D, i - s) : 0u;
    if (!big_shl1_add(rem, bit)) return false;
    u32 qb = 0;
    if (big_cmp(rem, R) >= 0) {
      big_sub(rem, R);
      qb = 1;
    }
    if (qbits == 0 && qb == 0) continue;  // leading zeros of the quotient
    if (qbits < 64) {
      q = (q << 1) | qb;
      qbits++;
    } else {
      extra++;
      if (qb) sticky = true;
    }
  }
  if (rem.n != 0) sticky = true;
  if (qbits == 0) {
    *out = 0;
    return true;
  }
  // quotient Q = q * 2^extra (+sticky); value = Q * 2^(k - s)
  i32 E = extra + k - s;
  if (qbits < 64) {
    q <<= (64 - qbits);
    E -= (64 - qbits);
  }
  return fl_round_ieee(q, E, sticky, is32, out);
}

// ------------------------------------------------------------------------------------------------
// number token -> IEEE bits (strconv.ParseFloat semantics).  `t` is the already validated token,
// `again` an iterator positioned at its first character (used only when the token has more
// significant digits than fit 64 bits).  Returns false on overflow (ParseFloat's range error).
// ------------------------------------------------------------------------------------------------
GGR_TABLE static const double GGR_P10_D[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                               1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
GGR_TABLE static const float GGR_P10_F[11] = {1e0f, 1e1f, 1e2f, 1e3f, 1e4f, 1e5f, 1e6f, 1e7f, 1e8f, 1e9f, 1e10f};

GGR_DEV u64 fl_double_bits(double d) {
  u64 u;
  memcpy(&u, &d, 8);
  return u;
}
GGR_DEV u32 fl_float_bits(float f) {
  u32 u;
  memcpy(&u, &f, 4);
  return u;
}

// Long literals: the exact decision when the first 40 significant digits leave the rounding open, i.e. the
// value lies within about 10^-39 (relative) of the halfway point H = (2m+1) * 2^(e-1) between lo = m * 2^e and
// the next float up.  Like Go's strconv it reads at most 800 significant digits N, value = N * 10^k, plus
// whether a nonzero digit follows.  That is exact: a halfway point has at most 767 significant digits, so it
// never lies strictly between N * 10^k and (N+1) * 10^k.  Both sides of N * 10^k <=> (2m+1) * 2^(e-1) are
// scaled to integers; near a halfway point neither exceeds 2^2670 (binary64: N < 10^800, or 2^55 * 5^1124 with
// k >= -1124), which GGR_XBIG_WORDS covers with room to spare.  Kept out of float_from_token's frame: only
// literals that reach it pay for the large integers.  `it` is at the token's first character.  Returns the
// correctly rounded bits without the sign; false on overflow (ParseFloat's range error).
#define GGR_XBIG_WORDS 88
template <class It>
GGR_DEVN bool fl_decide_long(It it, i32 exp10, u64 lo, bool is32, u64* out) {
  using XBig = BigN<GGR_XBIG_WORDS>;
  XBig A, B;
  A.n = 0;
  if (it.get() == '-') it.adv();
  u32 kept = 0, acc = 0, nacc = 0, pow = 1;
  i64 k = exp10;
  bool more = false, in_frac = false;
  for (;;) {
    const u32 c = it.get();
    if (it.eof()) break;
    if (c == '.') {
      in_frac = true;
      it.adv();
      continue;
    }
    if (!(c - '0' < 10u)) break;
    const u32 dgt = c - '0';
    if (in_frac) k--;
    if (kept == 0 && dgt == 0) {  // leading zeros
      it.adv();
      continue;
    }
    if (kept < 800) {
      acc = acc * 10 + dgt;
      pow *= 10;
      kept++;
      if (++nacc == 9) {
        if (!big_mul_small(A, pow, acc)) return false;
        acc = nacc = 0;
        pow = 1;
      }
    } else {
      k++;
      if (dgt != 0) more = true;
    }
    it.adv();
  }
  if (nacc && !big_mul_small(A, pow, acc)) return false;
  const int mbits = is32 ? 23 : 52, bias = is32 ? 127 : 1023;
  const u32 be = (u32)(lo >> mbits);
  u64 m = lo & ((1ull << mbits) - 1ull);
  i32 e = 1 - bias - mbits;
  if (be != 0) {
    m |= 1ull << mbits;
    e = (i32)be - bias - mbits;
  }
  big_set64(B, 2 * m + 1);
  const i64 p = (i64)e - 1;  // H = B * 2^p
  if (k >= 0 ? !big_mul_pow5(A, (u32)k) : !big_mul_pow5(B, (u32)-k)) return false;
  if (k - p >= 0 ? !big_shl(A, (u32)(k - p)) : !big_shl(B, (u32)(p - k))) return false;
  int c = big_cmp(A, B);
  if (c == 0 && more) c = 1;
  const u64 r = lo + ((c > 0 || (c == 0 && (m & 1ull))) ? 1u : 0u);  // the carry runs into the exponent field
  if ((r >> mbits) >= (is32 ? 255u : 2047u)) return false;
  *out = r;
  return true;
}

template <class It>
GGR_DEVN bool float_from_token(It again, const NumTok& t, bool is32, u64* bits) {
  const u64 sign = t.neg ? (is32 ? 0x80000000ull : 0x8000000000000000ull) : 0ull;
  Big D;
  i32 k;
  bool sticky = false;
  if (!t.ovf) {
    if (t.m == 0) {
      *bits = sign;
      return true;
    }
    k = t.k;
    // Clinger: decimal significand and power of ten both exact -> one correctly rounded operation
    if (!is32 && t.m < (1ull << 53) && k >= -22 && k <= 22) {
      double v = (double)t.m;
#if defined(__CUDA_ARCH__)
      v = k >= 0 ? __dmul_rn(v, GGR_P10_D[k]) : __ddiv_rn(v, GGR_P10_D[-k]);
#else
      v = k >= 0 ? v * GGR_P10_D[k] : v / GGR_P10_D[-k];
#endif
      *bits = fl_double_bits(v) | sign;
      return true;
    }
    if (is32 && t.m < (1ull << 24) && k >= -10 && k <= 10) {
      float v = (float)t.m;
#if defined(__CUDA_ARCH__)
      v = k >= 0 ? __fmul_rn(v, GGR_P10_F[k]) : __fdiv_rn(v, GGR_P10_F[-k]);
#else
      v = k >= 0 ? v * GGR_P10_F[k] : v / GGR_P10_F[-k];
#endif
      *bits = (u64)fl_float_bits(v) | sign;
      return true;
    }
    big_set64(D, t.m);
  } else {
    // more significant digits than fit 64 bits: re-read them into a big integer (the first 40
    // significant digits exactly, the rest as a sticky bit; fl_decide_long reads them again if needed)
    Rd from_rd;
    const It from = it_fork(again, &from_rd);
    D.n = 0;
    u32 c = again.get();
    if (c == '-') again.adv();
    u32 kept = 0, dropped = 0, frac_total = 0;
    bool in_frac = false, started = false;
    for (;;) {
      c = again.get();
      if (again.eof()) break;
      if (c == '.') {
        in_frac = true;
        again.adv();
        continue;
      }
      if (!(c - '0' < 10u)) break;
      u32 dgt = c - '0';
      if (in_frac) frac_total++;
      if (dgt != 0) started = true;
      if (started) {
        if (kept < 40) {
          if (D.n == 0) big_set64(D, dgt);
          else big_mul_small(D, 10, dgt);
          kept++;
        } else {
          dropped++;
          if (dgt != 0) sticky = true;
        }
      }
      again.adv();
    }
    if (D.n == 0) {
      *bits = sign;
      return true;
    }
    i64 kk = (i64)t.exp - (i64)frac_total + (i64)dropped;
    if (kk > 100000) kk = 100000;
    if (kk < -100000) kk = -100000;
    k = (i32)kk;
    if (sticky) {
      // nonzero digits were dropped: D * 10^k < value < (D+1) * 10^k.  Rounding is monotone, so when
      // both bounds round to the same float that is the answer; otherwise the digits decide.
      Big D1;
      D1.n = D.n;
      for (int i = 0; i < D.n; i++) D1.w[i] = D.w[i];
      big_mul_small(D1, 1, 1);  // D has at most 40 digits: no capacity overflow
      u64 lo, hi;
      if (!fl_from_big(D, k, true, is32, &lo)) return false;  // the lower bound overflows: so does the value
      if ((!fl_from_big(D1, k, false, is32, &hi) || hi != lo) && !fl_decide_long(from, t.exp, lo, is32, &lo)) return false;
      *bits = lo | sign;
      return true;
    }
  }
  u64 out;
  if (!fl_from_big(D, k, sticky, is32, &out)) return false;
  *bits = out | sign;
  return true;
}
