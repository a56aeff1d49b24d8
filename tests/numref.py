"""Exact reference for float and double text conversion, as protojson does it with Go's strconv.

parse(text, bits)  - a protojson number token -> IEEE bits, correctly rounded (round half to even) from the
                     exact decimal value; RANGE for ParseFloat's range error.
format(bits, width) - IEEE bits -> the text protojson prints (shortest round-trip digits in ES6 layout).
wire_fixed(...)    - the wire bytes of a double / float field from its bits.

Plain Python (integers and the shortest digits of repr / numpy): independent of the oracle and of the device code.
"""
import decimal
import re
import struct
import sys

import numpy as np

sys.set_int_max_str_digits(0)

RANGE = "range error"

# (mantissa bits without the hidden one, exponent bias, largest biased exponent of a finite value)
_FMT = {64: (52, 1023, 2046), 32: (23, 127, 254)}
_NUM = re.compile(r"(-?)(0|[1-9][0-9]*)(?:\.([0-9]+))?(?:[eE]([+-]?[0-9]+))?\Z")


def _round_to_bits(num, den, width):
    """positive num/den -> IEEE bits (no sign), round half to even; RANGE on overflow"""
    mb, bias, emax_b = _FMT[width]
    emin = 1 - bias  # exponent of the smallest normal
    # E = floor(log2(num/den))
    E = num.bit_length() - den.bit_length()
    if (num << max(0, -E)) < (den << max(0, E)):
        E -= 1
    q = max(E, emin) - mb  # value of one unit in the last place
    n, d = (num, den << q) if q >= 0 else (num << -q, den)
    M, r = divmod(n, d)
    if 2 * r > d or (2 * r == d and M & 1):
        M += 1
    if M == 1 << (mb + 1):
        M >>= 1
        q += 1
    if M == 0:
        return 0
    if M < 1 << mb:  # subnormal (q == emin - mb)
        return M
    be = q + mb + bias
    if be > emax_b:
        return RANGE
    return (be << mb) | (M - (1 << mb))


def parse(text, bits=64):
    """protojson number token (bare or quoted; "NaN", "Infinity", "-Infinity" when quoted) -> IEEE bits as an int,
    or RANGE.  NaN is the quiet NaN Go's math.NaN() converts to (float64 0x7FF8000000000001, float32 0x7FC00000)."""
    if isinstance(text, (bytes, bytearray)):
        text = text.decode()
    sign = 1 << (bits - 1)
    if len(text) >= 2 and text[0] == text[-1] == '"':
        text = text[1:-1]
        special = {"NaN": 0x7FF8000000000001 if bits == 64 else 0x7FC00000,
                   "Infinity": 0x7FF0000000000000 if bits == 64 else 0x7F800000}
        if text in special:
            return special[text]
        if text == "-Infinity":
            return special["Infinity"] | sign
    m = _NUM.match(text)
    if not m:
        raise ValueError("not a JSON number: %r" % text[:80])
    neg, ip, fp, ex = m.group(1) == "-", m.group(2), m.group(3) or "", int(m.group(4) or 0)
    digits = (ip + fp).lstrip("0")
    s = sign if neg else 0
    if not digits:
        return s
    stripped = digits.rstrip("0")
    e10 = ex - len(fp) + (len(digits) - len(stripped))
    digits = stripped
    # value = digits * 10^e10 lies in [10^(mag-1), 10^mag): cut absurd exponents before building integers
    mag = len(digits) + e10
    if mag > 400:
        return RANGE
    if mag < -400:
        return s
    N = int(digits)
    num, den = (N * 10 ** e10, 1) if e10 >= 0 else (N, 10 ** -e10)
    b = _round_to_bits(num, den, bits)
    return b if b == RANGE else b | s


def _value(bits, width):
    return struct.unpack("<d", struct.pack("<Q", bits))[0] if width == 64 else \
        np.frombuffer(struct.pack("<I", bits), np.float32)[0]


def shortest_digits(bits, width):
    """finite nonzero value -> (digit string without leading or trailing zeros, e) with |value| = 0.DIGITS * 10^e"""
    v = abs(_value(bits, width))
    if width == 64:
        _, dg, exp = decimal.Decimal(repr(float(v))).as_tuple()
        ds = "".join(map(str, dg))
    else:
        mant, exp = np.format_float_scientific(v, unique=True).split("e")
        ds = mant.replace(".", "")
        exp = int(exp) - (len(ds) - 1)
    stripped = ds.rstrip("0")
    exp += len(ds) - len(stripped)
    ds = stripped.lstrip("0")
    return ds, len(ds) + exp


def layout(neg, ds, x, exp_form):
    """Go's ES6 layout of 0.DS * 10^x: 'e' form (d.ddde-7, d.ddde+21: protojson trims "e-07" to "e-7") or plain"""
    sg = "-" if neg else ""
    if exp_form:
        e = x - 1
        return sg + ds[0] + ("." + ds[1:] if len(ds) > 1 else "") + ("e-%d" % -e if e < 0 else "e+%02d" % e)
    if x <= 0:
        return sg + "0." + "0" * -x + ds
    if len(ds) <= x:
        return sg + ds + "0" * (x - len(ds))
    return sg + ds[:x] + "." + ds[x:]


_F32_1EM6, _F32_1E21 = np.float32(1e-6), np.float32(1e21)


def format(bits, width=64):
    """IEEE bits -> protojson text (strconv.AppendFloat(f, 'e' or 'f', -1, width) under encoding/json's rule:
    'e' when |f| < 1e-6 or |f| >= 1e21, both thresholds taken in the value's own width)"""
    mb, _, _ = _FMT[width]
    neg = bool(bits >> (width - 1) & 1)
    e = bits >> mb & ((1 << (width - 1 - mb)) - 1)
    m = bits & ((1 << mb) - 1)
    if e == (1 << (width - 1 - mb)) - 1:
        return '"NaN"' if m else ('"-Infinity"' if neg else '"Infinity"')
    if e == 0 and m == 0:
        return "-0" if neg else "0"
    a = abs(_value(bits, width))
    exp_form = (a < 1e-6 or a >= 1e21) if width == 64 else (a < _F32_1EM6 or a >= _F32_1E21)
    ds, x = shortest_digits(bits, width)
    return layout(neg, ds, x, exp_form)


def format_float(v, width=64):
    """the same for a Python float (width 32: the float32 nearest to v)"""
    if width == 64:
        return format(struct.unpack("<Q", struct.pack("<d", v))[0], 64)
    return format(int(np.array([v], np.float32).view(np.uint32)[0]), 32)


def f64_bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


# ---- wire -------------------------------------------------------------------------------------------------
def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def fixed(bits, width):
    return struct.pack("<Q" if width == 64 else "<I", bits)


def wire_fixed(num, bits, width):
    """one unpacked occurrence: tag (wire type 1 for a double, 5 for a float), then the little-endian bits"""
    return varint(num << 3 | (1 if width == 64 else 5)) + fixed(bits, width)


def wire_packed(num, bits_list, width):
    payload = b"".join(fixed(b, width) for b in bits_list)
    return varint(num << 3 | 2) + varint(len(payload)) + payload
