"""Seeded corpus of integer, bool and enum values for the integer tests, every kind of tests/intref.py in both
directions.  Expected values come from intref alone.

Request items are (message, start offset, json, expected wire or status category): every number form (range
boundaries and their neighbours at 2^7k, 2^31, 2^32, 2^63 and 2^64 in both signs, exponents and fractions that do or do
not give an integer, exponents near the 20-digit guard and the 32-bit exponent limit, literals of more than 20 digits
whose zeros cancel, leading zeros) bare and quoted (with escapes, spaces and a second token inside the quotes), as a
singular field, a list element, a map key, a map value, a oneof member, a proto3 optional field and inside a wrapper.
Some carry a filler string (size routing) or sit behind 300 / 1100 list elements (the walker's later tiers and the
lock-step parser's large table).

Reply items are (message, start offset, wire, expected text, expected text with comma-space): varints of every length
1..10 with the value bits at each width edge, overlong, overflowing and cut varints, fixed values, zero values with
bits set above 32, placed at start offsets 0..15 behind headers of 0..10 bytes (so header and value straddle the 8-byte
header window), and on both sides of the 32 / 64 / 96-byte rounds and the 4 KB plain-mask limit; long packed and
unpacked runs for the pooled second reply tier; integer-keyed maps out of order and with repeated keys.
"""
import random

import intref as I

A, WK = "bench.All", "wkt.Wkt"
CUSTOM, F_STRING = 90, 14
F_NUM = dict({k: 1 + i for i, k in enumerate(I.INT_KINDS)}, bool=13, enum=16)
R_NUM = dict({k: 21 + i for i, k in enumerate(I.INT_KINDS)}, bool=33, enum=36)
# map fields by key kind: (json name, number, value json, value wire of field 2)
KEY_FIELD = {
    "int32": ("m_int32_str", 42, b'"v"', I.ld(2, b"v")),
    "sint32": ("m_sint32_float", 47, b"0", b"\x15\x00\x00\x00\x00"),
    "int64": ("m_int64_msg", 43, b"{}", I.ld(2, b"")),
    "uint64": ("m_uint64_bytes", 45, b'""', I.ld(2, b"")),
    "fixed64": ("m_fixed64_sfixed32", 48, b"0", b"\x15\x00\x00\x00\x00"),
    "bool": ("m_bool_double", 44, b"0", b"\x11" + b"\x00" * 8),
}
# map fields by value kind: (json name, number, key json, key wire of field 1)
VALUE_FIELD = {
    "int32": ("m_str_int32", 41, b'"k"', I.ld(1, b"k")),
    "enum": ("m_str_enum", 46, b'"k"', I.ld(1, b"k")),
    "sfixed32": ("m_fixed64_sfixed32", 48, b'"7"', b"\x09" + (7).to_bytes(8, "little")),
}
PRESENCE_FIELD = {"int32": [("o_int32", 51), ("opt_int32", 61)], "bool": [("o_bool", 54), ("opt_bool", 63)],
                  "enum": [("o_enum", 55)]}
WRAPPER_FIELD = {"bool": ("bv", 5), "int32": ("i32", 6), "int64": ("i64", 7), "uint32": ("u32", 8), "uint64": ("u64", 9)}
PLAIN = {"bool": (b"true", b"false"), "enum": (b'"RED"', b"3")}  # list neighbours; integers: 1 and 2


# ---- request forms ------------------------------------------------------------------------------------------------
def number_forms():
    """bare number tokens"""
    vals = {0, 1, 2}
    for k in range(1, 10):
        vals |= {(1 << (7 * k)) - 1, 1 << (7 * k)}
    for b in (31, 32, 63, 64):
        vals |= {(1 << b) + d for d in (-2, -1, 0, 1, 2)}
    vals |= {9007199254740993, 12345678901234567, 99999999999999999999, 100000000000000000000}
    out = []
    for v in sorted(vals):
        out += [b"%d" % v, b"-%d" % v] if v else [b"0", b"-0"]
    out += [b"0.0e5", b"1e2", b"100e-2", b"1.50e1", b"1.5", b"-1.5", b"1E2", b"1e+2", b"-1e2", b"1e0", b"0.5e1", b"0.05e2",
            b"10e-1", b"-10e-1", b"1e-1", b"0.0", b"-0.0", b"0e0", b"-0e-0", b"1.0", b"2.50e1", b"1.25e1",
            # the 20-digit guard: len(intp) + exp <= 20
            b"1e19", b"1e20", b"12e18", b"12e19", b"18446744073709551615e0", b"1844674407370955161.5e1",
            b"18446744073709551615e1", b"1.8446744073709551615e19", b"9.223372036854775807e18", b"9.223372036854775808e18",
            b"-9.223372036854775808e18", b"0.00000000000000000001e20", b"0.0000000000000000000001e22", b"1e21",
            b"2147483647e0", b"2.147483648e9", b"-2.147483648e9", b"4.294967295e9", b"4294967296e-0",
            # the exponent is read as a 32-bit integer (zero mantissas never read it)
            b"1e2147483647", b"1e2147483648", b"1e-2147483648", b"1e-2147483649", b"0e2147483648", b"0e200000000",
            b"0.0e99999999999999999999", b"-0e-99999999999", b"1e100000001", b"1e-100000001", b"0.000e-2147483649",
            # more than 20 digits whose zeros cancel
            b"1000000000000000000000000e-5", b"100000000000000000000000000000e-10", b"92233720368547758070000e-4",
            b"18446744073709551615000000e-6", b"-21474836480000000000000e-13", b"1000000000000000000000e-1",
            b"10000000000000000000000000000000000000000e-40", b"123000000000000000000000e-22",
            # leading zeros: no JSON number
            b"01", b"-01", b"00", b"007", b"0x10", b"1e", b"+1", b"-", b".5", b"1.", b"1e2.0"]
    return out


def quoted_forms():
    """string tokens (with quotes) of integer text"""
    out = [b'"%s"' % f for f in number_forms() if b'"' not in f]
    out += [b'"\\u0031\\u0032"', b'"1\\u0030"', b'"\\u002d5"', b'"4294967\\u00295"', b'"\\u0030"',
            b'" 1"', b'"1 "', b'"1 2"', b'"1\\t"', b'"\\t1"', b'"1\\n2"', b'"1]"', b'"1,"', b'"1}"', b'"1x"', b'"1\\u00a0"',
            b'"\\u20281"', b'""', b'" "', b'"-"', b'"true"', b'"[1]"', b'"\\"1\\""', b'"1e2 x"', b'"0e99999999999 "']
    return out


def bool_forms():
    return [b"true", b"false", b'"true"', b'"false"', b"1", b"0", b"True", b"tru", b'""', b"-0", b"1.5"]


def enum_forms():
    out = [b'"%s"' % n.encode() for n, _ in I.COLOR]
    out += [b'"red"', b'"RED "', b'"1"', b'"R\\u0045D"', b'"\\u0042IG"', b'"UNKNOWN"', b'""',
            b"0", b"1", b"7", b"-5", b"-1", b"1073741824", b"2147483647", b"2147483648", b"-2147483648", b"-2147483649",
            b"1e2", b"-0", b"1.5", b"10e-1", b"4294967297", b"0e99999999999", b"true", b"01"]
    return out


def forms(kind):
    if kind == "bool":
        return bool_forms()
    if kind == "enum":
        return enum_forms()
    return number_forms() + quoted_forms()


# ---- request items ------------------------------------------------------------------------------------------------
def _key_json(form):
    return form if form[:1] == b'"' else b'"' + form + b'"'


def request_item(kind, cont, form, s, filler=0, elems=0):
    """(message, start offset, json, expected wire or status category)"""
    v = I.value(kind, form)
    ok = not isinstance(v, str)
    msg = A
    if cont == "f":
        js = b'{"f_%s":%s' % (kind.encode(), form)
        want = (b"" if v in (0, False) else I.tagged(F_NUM[kind], kind, v)) if ok else v
    elif cont == "r":
        a, b = PLAIN.get(kind, (b"1", b"2"))
        # eight digits each in long lists, so that the list is not too dense for the walker's IR region
        e = b"12345678" if elems > 1000 and kind in I.INT_KINDS else a
        js = b'{"r_%s":[%s%s,%s,%s]' % (kind.encode(), (e + b",") * elems, a, form, b)
        av, bv, ev = I.value(kind, a), I.value(kind, b), I.value(kind, e)
        want = I.packed(R_NUM[kind], kind, [ev] * elems + [av, v, bv]) if ok else v
    elif cont == "k":
        name, num, vjs, vwire = KEY_FIELD[kind]
        kj = _key_json(form)
        kd = I.strref.parse_string(kj[1:-1])
        js = b'{"%s":{%s:%s}' % (name.encode(), kj, vjs)
        if isinstance(kd, str):
            want = I.SYNTAX if kd == I.strref.SYNTAX else kd
        else:
            k = I.key_value(kind, kd)
            want = I.ld(num, I.tagged(1, kind, k) + vwire) if not isinstance(k, str) else k
    elif cont == "m":
        name, num, kjs, kwire = VALUE_FIELD[kind]
        js = b'{"%s":{%s:%s}' % (name.encode(), kjs, form)
        want = I.ld(num, kwire + I.tagged(2, kind, v)) if ok else v
    elif cont in ("o", "p"):
        name, num = PRESENCE_FIELD[kind][0 if cont == "o" else -1]
        js = b'{"%s":%s' % (name.encode(), form)
        want = I.tagged(num, kind, v) if ok else v
    elif cont == "w":
        msg = WK
        name, num = WRAPPER_FIELD[kind]
        js = b'{"%s":%s' % (name.encode(), form)
        want = I.ld(num, b"" if v in (0, False) else I.tagged(1, kind, v)) if ok else v
    elif cont == "rw":
        msg = WK
        js = b'{"r_i32":[1,%s]' % form
        want = I.ld(20, I.tagged(1, kind, 1)) + I.ld(20, b"" if v == 0 else I.tagged(1, kind, v)) if ok else v
    else:  # "mw": int32 key -> Int64Value
        msg = WK
        js = b'{"m_i64":{"-3":%s}' % form
        want = I.ld(15, I.tagged(1, "int32", -3) + I.ld(2, b"" if v == 0 else I.tagged(1, kind, v))) if ok else v
    if filler:
        js += b',"custom":"' + b"r" * filler + b'"'
        if not isinstance(want, str):
            want += I.ld(CUSTOM, b"r" * filler)
    return (msg, s, js + b"}", want)


def containers(kind):
    """the containers after "f" and "r" that the schema has for this kind"""
    out = []
    if kind in KEY_FIELD:
        out.append("k")
    if kind in VALUE_FIELD:
        out.append("m")
    if kind in PRESENCE_FIELD:
        out += ["o", "p"] if len(PRESENCE_FIELD[kind]) > 1 else ["o"]
    if kind in WRAPPER_FIELD:
        out.append("w")
    if kind == "int32":
        out.append("rw")
    if kind == "int64":
        out.append("mw")
    return out


def request_items():
    """every form of every kind as a singular field and a list element, and in turn in each other container of its
    kind; one in three with a filler of 1100 bytes, one list in eleven behind 300 or 1100 plain elements"""
    out = []
    k = 0
    for kind in I.KINDS:
        extra = containers(kind)
        for j, form in enumerate(forms(kind)):
            rot = (["r"] + extra)[j % (1 + len(extra))]
            conts = ["f", rot] + (["r"] if rot != "r" and form[:1] != b'"' else [])  # quoted forms: one list in turn
            for cont in conts:
                elems = 0
                if cont == "r" and k % 11 == 0 and I.wire_type(kind) == 0:
                    # varint kinds only: a long list of fixed values grows past the simulation's output buffers
                    elems = (300, 1100)[(k // 11) % 2]
                filler = 1100 if k % 3 == 0 and cont not in ("w", "rw", "mw") else 0
                out.append(request_item(kind, cont, form, (k * 7) % 16, filler, elems))
                k += 1
    return out


def body_items(every=1):
    """(start offset, tools/call body, expected wire or status category / intref.FAIL) for every form of every kind
    as a singular field of bench_benchservice_echoall's arguments"""
    out = []
    i = 0
    for kind in I.KINDS:
        for form in forms(kind):
            i += 1
            if i % every:
                continue
            try:
                v = I.body_value(kind, form)
            except ValueError:  # no JSON number: encoding/json refuses the body
                v = I.FAIL
            body = (b'{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"bench_benchservice_echoall",'
                    b'"arguments":{"f_%s":%s}}}' % (i, kind.encode(), form))
            want = v if isinstance(v, str) else (b"" if v in (0, False) else I.tagged(F_NUM[kind], kind, v))
            out.append((i % 16, body, want))
    return out


# ---- reply items --------------------------------------------------------------------------------------------------
def varint_payloads():
    """unsigned 64-bit payloads: each varint length 1..10 at its ends, the 32 / 64-bit edges, zero low 32 bits"""
    vals = {0, 1, 2}
    for k in range(1, 10):
        vals |= {(1 << (7 * k)) - 1, 1 << (7 * k), (1 << (7 * k)) + 1}
    M = (1 << 64) - 1
    vals |= {(1 << 31) - 1, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, 1 << 33, (1 << 63) - 1, 1 << 63, M, M - 1,
             0xFFFFFFFF00000000, 0xFFFFFFFF80000000, 0xFFFFFFFF7FFFFFFF, (-5) & M, 1 << 30, 3 << 32, 0x8000000100000000}
    return sorted(vals)


def fixed_payloads(bits):
    if bits == 32:
        return [0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0x100, 0x01000000, 0xFFFFFFFE]
    return [0, 1, 0x7FFFFFFF, 1 << 31, 1 << 32, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 1 << 56, 0xFFFFFFFF00000000]


def overlong(u, n):
    """u as a varint of exactly n bytes (n at least its minimal length): continuation bits over zero groups"""
    out = bytearray()
    for k in range(n):
        b = (u >> (7 * k)) & 0x7F
        out.append(b | (0x80 if k < n - 1 else 0))
    return bytes(out)


def bad_varints():
    """varints protowire.ConsumeVarint refuses: 10th byte 2..0x7F, 11 bytes"""
    return [b"\xff" * 9 + b"\x02", b"\x80" * 9 + b"\x7f", b"\x80" * 10 + b"\x00", b"\xff" * 10 + b"\x01", b"\x81" * 9 + b"\x03"]


def _value_bytes(kind):
    """(payload bytes, wire type) of every reply value of a kind"""
    wt = I.wire_type(kind)
    if wt:
        bits = 64 if wt == 1 else 32
        return [(u.to_bytes(bits // 8, "little"), wt) for u in fixed_payloads(bits)]
    out = []
    for u in varint_payloads():
        n0 = len(I.varint(u))
        out.append((I.varint(u), 0))
        if u < 1 << 63:
            for n in sorted({n0 + 1, 10}):
                if n > n0:
                    out.append((overlong(u, n), 0))
    out += [(b, 0) for b in bad_varints()]
    return out


def _reply(msg, s, w):
    return (msg, s, w, I.decode(msg, w, 0), I.decode(msg, w, 1))


def _head(num, wt):
    return I.varint(num << 3 | wt)


def reply_singular():
    """each value of each kind as its singular field, at start offsets 0..15 behind 0..10 bytes of an f_int32 field,
    and cut at its end"""
    out = []
    k = 0
    for kind in I.KINDS:
        for pb, wt in _value_bytes(kind):
            num = F_NUM[kind]
            for r in range(3):
                s = (k * 5 + r * 6) % 16
                pre = b""
                if kind != "int32" and r:
                    n = 1 + (k + r) % 10  # an f_int32 of n varint bytes in front (value 2^(7(n-1)))
                    pre = b"\x08" + overlong(1 << (7 * (n - 1)), n)
                out.append(_reply(A, s, pre + _head(num, wt) + pb))
                k += 1
            if len(pb) > 1:
                out.append(_reply(A, k % 16, _head(num, wt) + pb[:-1]))  # cut
            if kind in PRESENCE_FIELD:
                out.append(_reply(A, k % 16, _head(PRESENCE_FIELD[kind][0][1], wt) + pb))
            if kind in WRAPPER_FIELD:
                out.append(_reply(WK, k % 16, I.ld(WRAPPER_FIELD[kind][1], _head(1, wt) + pb)))
    return out


EDGES = (32, 64, 96, 4096)


def reply_edges():
    """a value of each kind whose header (unpacked) or bytes (packed) start at rebased bytes E - 11 .. E + 2 for each
    32-byte round edge and the 4 KB plain-mask limit, behind an f_string of the right length"""
    out = []
    k = 0
    for kind in I.KINDS:
        wt = I.wire_type(kind)
        vals = _value_bytes(kind)
        num = R_NUM[kind]
        for e in EDGES:
            for d in range(-11, 3):
                pb, _ = vals[k % len(vals)]
                if len(pb) == 10 and pb[9] > 1 or len(pb) > 10:
                    pb = vals[(k + 1) % len(vals)][0]
                s = k % 16
                tail = (b"\x01" if wt == 0 else b"\x01" + b"\x00" * (3 if wt == 5 else 7))
                if k % 2:  # unpacked: header at e + d
                    body = _head(num, wt) + pb + _head(num, wt) + tail
                    at = 0
                else:  # packed: the value bytes at e + d
                    payload = tail * 3 + pb + tail
                    body = I.ld(num, payload)
                    at = len(body) - len(payload) + len(tail) * 3
                room = e + d - s - at  # bytes of the f_string in front
                pad = next((I.ld(F_STRING, b"p" * n) for n in (room - 2, room - 3) if n > 0 and len(I.ld(F_STRING, b"p" * n)) == room), None)
                if pad is None:
                    k += 1
                    continue
                assert s + len(pad) + at == e + d, (s, len(pad), at, e, d)
                out.append(_reply(A, s, pad + body))
                k += 1
    return out


def reply_runs(seed=0):
    """packed runs of 400 / 1000 values (one ending inside a varint), unpacked runs of 400 occurrences, and runs that
    mix packed and unpacked pieces of one field"""
    rng = random.Random(seed + 11)
    out = []
    for i, kind in enumerate(I.KINDS):
        wt = I.wire_type(kind)
        pool = [pb for pb, w in _value_bytes(kind) if len(pb) <= 10 and not (len(pb) == 10 and pb[9] > 1)]
        num = R_NUM[kind]
        for n in (400, 1000):
            vals = [rng.choice(pool) for _ in range(n)]
            out.append(_reply(A, (i + n) % 16, I.ld(num, b"".join(vals))))
            out.append(_reply(A, (i + n + 3) % 16, b"".join(_head(num, wt) + v for v in vals[:400])))
        pieces = b""
        for j in range(30):
            vals = [rng.choice(pool) for _ in range(rng.randrange(1, 40))]
            pieces += I.ld(num, b"".join(vals)) if j % 3 else b"".join(_head(num, wt) + v for v in vals)
        out.append(_reply(A, i % 16, pieces))
        if wt == 0:
            cut = b"".join(rng.choice(pool) for _ in range(50)) + b"\x80\x80"
            out.append(_reply(A, (i + 5) % 16, I.ld(num, cut)))  # a packed payload that ends inside a varint
        else:
            cut = b"".join(rng.choice(pool) for _ in range(50)) + b"\x01"
            out.append(_reply(A, (i + 5) % 16, I.ld(num, cut)))  # a packed payload that ends inside a fixed value
    # r_unpacked and the wrapper list
    vals = [rng.choice(varint_payloads()) for _ in range(500)]
    out.append(_reply(A, 3, b"".join(b"\xb0\x02" + I.varint(u) for u in vals)))
    out.append(_reply(A, 4, I.ld(38, b"".join(I.varint(u) for u in vals))))
    out.append(_reply(WK, 5, b"".join(I.ld(20, b"\x08" + I.varint(u)) for u in vals[:300])))
    return out


def reply_maps(seed=0):
    """integer-keyed maps out of key order and with repeated keys (the last entry wins), entries without key or value"""
    rng = random.Random(seed + 12)
    out = []
    M = (1 << 64) - 1
    specs = [(42, "int32", lambda j: I.ld(2, b"v%d" % j)),
             (45, "uint64", lambda j: I.ld(2, bytes([j & 255]))),
             (48, "fixed64", lambda j: b"\x15" + (j * 7919 & 0xFFFFFFFF).to_bytes(4, "little")),
             (47, "sint32", lambda j: b"\x15" + (0x3FC00000 + j).to_bytes(4, "little")),
             (44, "bool", lambda j: b"\x11" + (0x3FF8000000000000 + j).to_bytes(8, "little"))]
    for num, kk, vw in specs:
        bits = I.KINDS[kk][0]
        keys = [0, 1, 2, 127, 128, (1 << 31) - 1, 1 << 31, (1 << 32) - 1, (1 << 63) - 1, 1 << 63, M, (-1) & M, (-128) & M]
        for n in (1, 2, 5, 17, 40, 300):
            ents = b""
            for j in range(n):
                u = rng.choice(keys) if kk != "bool" else rng.randrange(3)
                if kk == "sint32" or I.wire_type(kk) == 1:
                    key = I.wire(kk, I.from_wire(kk, u)) if I.wire_type(kk) == 1 else I.varint(u)
                    kb = _head(1, I.wire_type(kk)) + key
                else:
                    kb = _head(1, 0) + I.varint(u)
                if j % 13 == 7:
                    kb = b""  # no key: the zero key
                ents += I.ld(num, kb + vw(j) if j % 11 != 5 else vw(j) + kb)  # value in front of the key
            out.append(_reply(A, (n + num) % 16, ents))
    # integer and enum values keyed by string
    for n in (3, 40):
        ents = b""
        for j in range(n):
            u = rng.choice(varint_payloads())
            ents += I.ld(41, I.ld(1, b"k%d" % (j % 7)) + b"\x10" + I.varint(u))
            ents += I.ld(46, I.ld(1, b"e%d" % (j % 5)) + b"\x10" + I.varint(rng.choice([0, 1, 3, (-5) & M, 1 << 30, 9, u])))
        out.append(_reply(A, n % 16, ents))
    vals = [0, 1, (-1) & M, 1 << 63, 1 << 32]
    out.append(_reply(WK, 6, b"".join(I.ld(15, b"\x08" + I.varint(u) + I.ld(2, b"\x08" + I.varint(u))) for u in vals)))
    return out


def reply_items(seed=0):
    return reply_singular() + reply_edges() + reply_runs(seed) + reply_maps(seed)
