"""Seeded corpus of float / double conversions for the number tests: request literals (halfway points written
exactly, just above and just below, with the deciding digit far behind the first 40 significant digits; literals
around the fast-path edges; float32 double-rounding traps) placed in every kind of float position, and reply bit
patterns (sweeps, per-exponent edges, powers of ten, layout switch points, special values).  Expected values come
from numref alone."""
import random
import struct

import numref as R

A = "bench.All"
WK = "wkt.Wkt"
_FMT = {64: (52, 1023), 32: (23, 127)}
# significant-digit positions of the digit that decides a literal near a halfway point
POSITIONS = (41, 42, 60, 113, 768, 800, 801, 1500)


# ---- halfway points -------------------------------------------------------------------------------------------
def halfway(bits, width):
    """the exact halfway point between the positive value `bits` and the next one up, as (I, s): I * 10^s"""
    mb, bias = _FMT[width]
    be, m = bits >> mb, bits & ((1 << mb) - 1)
    e = 1 - bias - mb
    if be:
        m |= 1 << mb
        e = be - bias - mb
    p = e - 1  # H = (2m+1) * 2^p
    if p >= 0:
        return (2 * m + 1) << p, 0
    return (2 * m + 1) * 5 ** -p, p


def halfway_sample(width, rng, n_normal, n_sub):
    mb, bias = _FMT[width]
    top = (2 * bias + 1) << mb  # bits of the largest finite value + 1
    pts = [0, 1, (1 << mb) - 1, 1 << mb, (1 << mb) + 1, top - 1, top - 2]  # smallest subnormal, both sides of the
    pts += [(bias + k) << mb for k in (-20, -1, 0, 1, 30)]                  # normal boundary, MAX; powers of two
    pts += [((bias + k) << mb) - 1 for k in (0, 1, 30)]                      # their lower neighbours
    pts += [rng.randrange(1 << mb, top - 1) for _ in range(n_normal)]
    pts += [rng.randrange(1, 1 << mb) for _ in range(n_sub)]
    return pts


def _digits(I, s):
    """(digit string without trailing zeros, s) with I * 10^s"""
    ds = str(I)
    st = ds.rstrip("0")
    return st, s + len(ds) - len(st)


def near_literals(I, s, positions=POSITIONS):
    """the halfway point I * 10^s written exactly, padded with a thousand zeros, and just above / just below with
    the first differing significant digit at each of `positions`: [(digits, s)] with value int(digits) * 10^s"""
    ds, s = _digits(I, s)
    n = len(ds)
    out = [(ds, s), (ds + "0" * 1000, s - 1000)]
    for P in positions:
        if P > n:
            pad = P - n
            out.append((ds + "0" * (pad - 1) + "1", s - pad))                      # H + one unit at position P
            out.append((str(int(ds) - 1) + "9" * pad, s - pad))                    # H - one unit at position P
        else:
            head = ds[:P]
            out.append((str(int(head) + 1), s + n - P))                              # H rounded up to P digits
            out.append((head, s + n - P))                                            # H truncated to P digits
    return out


def spell(ds, s, style, neg=False, quoted=False):
    """int(ds) * 10^s as a JSON number: plain, d.ddde±X, dddde±X, or 0.000…ddde±X; optionally negative / quoted"""
    n = len(ds)
    if style == "plain":
        if s >= 0:
            t = ds + "0" * s
        elif n > -s:
            t = ds[: n + s] + "." + ds[n + s:]
        else:
            t = "0." + "0" * (-s - n) + ds
    elif style == "exp":
        t = ds[0] + ("." + ds[1:] if n > 1 else "") + "e%d" % (s + n - 1)
    elif style == "intexp":
        t = ds + "e%d" % s
    else:  # long zero prefix
        z = 40 + (n % 300)
        t = "0." + "0" * z + ds + "e%+d" % (s + n + z)
    t = ("-" if neg else "") + t
    return '"%s"' % t if quoted else t


STYLES = ("plain", "exp", "intexp", "zeros")


def long_literals(width, seed=0, n_normal=24, n_sub=10, positions=POSITIONS):
    """[(text, width)] around halfway points, in every spelling"""
    rng = random.Random(seed * 2 + width)
    out = []
    for b in halfway_sample(width, rng, n_normal, n_sub):
        for j, (ds, s) in enumerate(near_literals(*halfway(b, width), positions)):
            style = STYLES[(j + b) % 4]
            if style == "plain" and abs(s) > 2000:
                style = "exp"
            out.append((spell(ds, s, style, neg=rng.random() < 0.3, quoted=rng.random() < 0.15), width))
    return out


def short_literals(width, seed=0, n=300):
    """literals of at most 40 significant digits: Clinger's fast-path edges, halfway points cut to 17..40 digits,
    and for float32 decimals whose nearest double is exactly a float32 halfway point (double rounding traps)"""
    rng = random.Random(seed * 2 + width + 100)
    out = []
    if width == 64:
        ms, ks = (2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 3), (21, 22, 23)
    else:
        ms, ks = (2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3), (9, 10, 11)
    for m in ms:
        for k in ks:
            for sg in (1, -1):
                out.append(("%de%d" % (m, sg * k), width))
                out.append(("%d.%de%d" % (m // 10, m % 10, sg * k + 1), width))
    mb, bias = _FMT[width]
    top = (2 * bias + 1) << mb
    for _ in range(n):
        b = rng.randrange(1, top - 1)
        I, s = halfway(b, width)
        ds, s = _digits(I, s)
        P = rng.randrange(17, 41)
        if len(ds) > P:
            cut = len(ds) - P
            for d in (str(int(ds[:P]) + 1), ds[:P]):
                out.append((spell(d, s + cut, STYLES[b % 4]), width))
    if width == 32:
        # a float32 halfway point is exactly a double; literals within a double's half ulp of it round to it as a double
        for _ in range(n):
            b = rng.randrange(1 << 23, (254 << 23))
            I, s = halfway(b, 32)
            ds, s = _digits(I, s)
            pad = min(40, len(ds) + 12) - len(ds)
            if pad < 1:
                continue
            for delta in (1, -1):
                out.append((spell(str(int(ds) * 10 ** pad + delta), s - pad, STYLES[b % 4]), 32))
    return out


def request_literals(seed=0, full=True):
    """[(text, width, expected bits or numref.RANGE)]"""
    lits = []
    for w in (64, 32):
        lits += long_literals(w, seed) if full else long_literals(w, seed, 6, 3, (41, 113, 801))
        lits += short_literals(w, seed, 300 if full else 60)
    return [(t, w, R.parse(t, w)) for t, w in lits]


# ---- positions ------------------------------------------------------------------------------------------------
F_FLOAT, F_DOUBLE, R_FLOAT, R_DOUBLE, M_BOOL_DOUBLE, M_SINT32_FLOAT = 11, 12, 31, 32, 44, 47
WKT_FV, WKT_DV = 10, 11


def _ld(num, payload):
    return R.varint(num << 3 | 2) + R.varint(len(payload)) + payload


def request_items(lits, seed=0):
    """(message, json, expected wire or RANGE) for the literals in singular fields, packed lists of 1 to 600 values,
    map values and wrappers"""
    rng = random.Random(seed + 7)
    items = []

    def add(name, js, wire, ranged):
        items.append((name, js.encode(), R.RANGE if ranged else wire))

    for i, (t, w, b) in enumerate(lits):
        rg = b == R.RANGE
        fname, num = ("f_double", F_DOUBLE) if w == 64 else ("f_float", F_FLOAT)
        add(A, '{"%s":%s}' % (fname, t), b"" if rg or b == 0 else R.wire_fixed(num, b, w), rg)
        k = i % 3
        if k == 0:
            if w == 64:
                add(A, '{"m_bool_double":{"true":%s}}' % t, b"" if rg else _ld(M_BOOL_DOUBLE, b"\x08\x01" + R.wire_fixed(2, b, 64)), rg)
            else:
                add(A, '{"m_sint32_float":{"-3":%s}}' % t, b"" if rg else _ld(M_SINT32_FLOAT, b"\x08\x05" + R.wire_fixed(2, b, 32)), rg)
        elif k == 1:
            num = WKT_DV if w == 64 else WKT_FV
            add(WK, '{"%s":%s}' % ("dv" if w == 64 else "fv", t), b"" if rg else _ld(num, b"" if b == 0 else R.wire_fixed(1, b, w)), rg)
    # packed lists: runs of literals of one width, 1 to 600 values, with short plain values mixed in
    for w, fname, num in ((64, "r_double", R_DOUBLE), (32, "r_float", R_FLOAT)):
        pool = [(t, b) for t, ww, b in lits if ww == w]
        j = 0
        while j < len(pool):
            n = rng.choice([1, 2, 7, 33, 100, 250, 600])
            run = pool[j:j + n]
            j += n
            vals = []
            for t, b in run:
                vals.append((t, b))
                if rng.random() < 0.2:
                    x = rng.choice(["1.5", "-0", "0.1", "3e-5", "1e22"])
                    vals.append((x, R.parse(x, w)))
            rg = any(b == R.RANGE for _, b in vals)
            add(A, '{"%s":[%s]}' % (fname, ",".join(t for t, _ in vals)), b"" if rg else R.wire_packed(num, [b for _, b in vals], w), rg)
    return items


def body_round_trip(t, w):
    """expected bits of a literal inside `arguments` of a tools/call body: json.Marshal re-prints every bare number
    from float64, the field then parses that text; a quoted literal reaches the field unchanged"""
    if t.startswith('"'):
        return R.parse(t, w)
    b = R.parse(t, 64)
    if b == R.RANGE:
        return R.RANGE
    return R.parse(R.format(b, 64), w)


def body_items(lits, seed=0):
    """(HTTP body, expected request wire or RANGE) for bench_benchservice_echoall tools/call bodies"""
    out = []
    for i, (t, w, _) in enumerate(lits):
        b = body_round_trip(t, w)
        fname, num = ("f_double", F_DOUBLE) if w == 64 else ("f_float", F_FLOAT)
        body = ('{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"bench_benchservice_echoall",'
                '"arguments":{"%s":%s}}}' % (i, fname, t)).encode()
        out.append((body, R.RANGE if b == R.RANGE else (b"" if b == 0 else R.wire_fixed(num, b, w))))
    return out


# ---- reply bit patterns ---------------------------------------------------------------------------------------
def reply_bits(width, seed=0, n_random=1 << 20, stride=4099):
    """bit patterns: a strided sweep (binary32) or seeded random patterns (binary64), the per-exponent edges
    (mantissa 0, 1, 2, max-1, max, both signs), and for binary64 the powers of ten from 1e-323 to 1e308 and the
    layout switch points 1e-6 and 1e21 with their neighbours"""
    mb, bias = _FMT[width]
    ebits = width - 1 - mb
    mmax = (1 << mb) - 1
    out = []
    if width == 32:
        out += range(0, 1 << 32, stride)
    else:
        rng = random.Random(seed + 64)
        out += [rng.getrandbits(64) for _ in range(n_random)]
    for e in range(1 << ebits):
        for m in (0, 1, 2, mmax - 1, mmax):
            for sg in (0, 1):
                out.append(sg << (width - 1) | e << mb | m)
    if width == 64:
        for k in range(-323, 309):
            b = R.parse("1e%d" % k, 64)
            out += [b - 1, b, b + 1]
        for v in (1e-6, 1e21):
            b = R.f64_bits(v)
            out += [b - 1, b, b + 1]
    else:
        for t in ("1e-6", "1e21"):
            b = R.parse(t, 32)
            out += [b - 1, b, b + 1]
    for b in (0x7FF8000000000001, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF, 0x7FF4000000000000) if width == 64 else \
            (0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x7FA00000):
        out.append(b)
    return out


def reply_items(bits64, bits32, seed=0):
    """(message, wire, expected protojson text): packed runs of about 1000 values with unpacked occurrences of the
    same field (wire types 1 / 5) mixed in, singular fields, map values and wrappers"""
    rng = random.Random(seed + 9)
    items = []
    for w, bl, fnum, fname, rnum, rname in ((64, bits64, F_DOUBLE, "fDouble", R_DOUBLE, "rDouble"),
                                            (32, bits32, F_FLOAT, "fFloat", R_FLOAT, "rFloat")):
        j = 0
        while j < len(bl):
            n = rng.choice([1, 3, 200, 1000, 1000])
            run = bl[j:j + n]
            j += n
            wire = b""
            k = 0
            while k < len(run):  # packed pieces and single unpacked occurrences, in order
                if rng.random() < 0.3:
                    wire += R.wire_fixed(rnum, run[k], w)
                    k += 1
                else:
                    m = rng.randrange(1, 300)
                    wire += R.wire_packed(rnum, run[k:k + m], w)
                    k += m
            items.append((A, wire, '{"%s":[%s]}' % (rname, ",".join(R.format(b, w) for b in run))))
        for i in range(0, len(bl), max(1, len(bl) // 3000)):
            b = bl[i]
            text = R.format(b, w)
            items.append((A, R.wire_fixed(fnum, b, w), "{}" if b == 0 else '{"%s":%s}' % (fname, text)))
            if w == 64:
                items.append((A, _ld(M_BOOL_DOUBLE, b"\x08\x01" + R.wire_fixed(2, b, 64)), '{"mBoolDouble":{"true":%s}}' % text))
            else:
                items.append((A, _ld(M_SINT32_FLOAT, b"\x08\x05" + R.wire_fixed(2, b, 32)), '{"mSint32Float":{"-3":%s}}' % text))
            items.append((WK, _ld(WKT_DV if w == 64 else WKT_FV, R.wire_fixed(1, b, w)), '{"%s":%s}' % ("dv" if w == 64 else "fv", text)))
    return [(n, wire, t.encode()) for n, wire, t in items]
