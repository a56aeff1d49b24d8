"""Exact reference for integer, bool and enum values, as protojson reads and writes them and proto.Unmarshal /
proto.Marshal carry them on the wire.

Request side
  number_parts(raw)         - protobuf-go internal/encoding/json parseNumberParts on a number token.
  normalize(parts)          - normalizeToIntString: the integer text of the token, or None.
  parse_int(s, bits)        - strconv.ParseInt(s, 10, bits); parse_uint(s, bits) - strconv.ParseUint.
  value(kind, raw)          - a JSON value token (bare, or a string token with its quotes) for a field of `kind` ->
                              the Go value (int, or bool), or SYNTAX / INVALID_VALUE.
  key_value(kind, name)     - the decoded text of a map key -> the key value, or INVALID_VALUE.
  body_value(kind, raw)     - the same token inside `arguments` of a tools/call body, after encoding/json's round trip.
  wire(kind, v), tagged(num, kind, v), packed(num, kind, vals) - proto.Marshal of the value.
Reply side
  consume_varint(b, i)      - protowire.ConsumeVarint: (value, next index), or None.
  from_wire(kind, v)        - the Go value proto.Unmarshal keeps from a varint / fixed payload.
  text(kind, v)             - protojson's text of the value; key_text(kind, v) - of a map key.
  decode(msg, wire, flags)  - protojson.Marshal(proto.Unmarshal(wire)) for the integer, bool and enum fields of
                              bench.All and the integer wrappers of wkt.Wkt -> text, or BAD_WIRE.

Plain Python (integer arithmetic and, for the float64 round trip of the request envelope, numref): independent of the
oracle and of the device code.  The schema facts (field numbers, kinds, JSON names, declaration order) restate
tests/golden/make_descriptors.py.

Rules that rest on memory of protobuf-go v1.36 and Go's standard library, not on a source that can be read here:
  * normalizeToIntString returns "0" for a token without nonzero digits (no integer digits, fraction all zeros) before
    it looks at the exponent, so `0e99999999999999999999` is 0 for every integer kind.  Otherwise the exponent text is
    read by strconv.ParseInt(exp, 10, 32) and any error fails the value; for a positive exponent the fraction must fit
    (len(frac) <= exp, trailing fraction zeros trimmed first) and len(intp) + exp <= 20; for a negative one there is no
    fraction and the digits shifted out are all zeros (so a literal of more than 20 digits can still be an integer).
    intp excludes a lone leading 0.
  * strconv.ParseInt takes one optional sign ('+' or '-') and decimal digits, leading zeros allowed; ParseUint takes
    no sign.  Map keys of integer kinds are these calls on the key text itself (so "+3", "007", "-0" are keys); bool
    keys are exactly "true" / "false".
  * A quoted number: the decoded string must equal strings.TrimSpace of itself (Unicode White_Space), then a fresh
    decoder reads ONE token of it and that token must be a number: "1 2", "1]" and "1," are 1; "1x", " 1", "01" fail.
  * Bool fields take only the bare literals; enum fields take a declared name (exactly, as a string) or a bare number
    by Token.Int(32), declared or not; a quoted number is no enum value.
  * proto.Unmarshal keeps int32(v) for int32 and enum, uint32(v) for uint32, DecodeZigZag(v & 0xFFFFFFFF) as int32
    for sint32, v != 0 for bool; ConsumeVarint fails on a cut varint and on a 10th byte above 1.  A packed run whose
    payload ends inside a varint fails the message.  The last occurrence of a singular field and the last entry of a
    map key win; a map entry's missing key or value is the zero value.
  * protojson.Marshal writes 64-bit integer kinds as quoted decimals, the others as numbers, an enum by the first
    declared name of its number or else as a number, and map keys in numeric (bool: false first) order.
  * proto.Marshal writes an int32 or enum as the varint of its sign extension to 64 bits (10 bytes when negative),
    a sint32 as the 32-bit zigzag, and both key and value of every map entry.
  * encoding/json decodes a number of `arguments` to float64 and json.Marshal prints it like protojson prints a
    double; a number that float64 cannot hold makes the whole body fail.
Where this reference and the oracle disagreed the decision is recorded in oracle/README.md.
"""
import base64

import numref
import strref

SYNTAX, INVALID_VALUE, BAD_WIRE = "syntax", "invalid_value", "bad_wire"
STATUS = {SYNTAX: 1, INVALID_VALUE: 3, BAD_WIRE: 10}  # GGR_ST_* of each category

# kind -> (bits, signed, wire form): wire form v = varint, z = zigzag varint, f = fixed
KINDS = {
    "int32": (32, True, "v"), "int64": (64, True, "v"), "uint32": (32, False, "v"), "uint64": (64, False, "v"),
    "sint32": (32, True, "z"), "sint64": (64, True, "z"), "fixed32": (32, False, "f"), "fixed64": (64, False, "f"),
    "sfixed32": (32, True, "f"), "sfixed64": (64, True, "f"), "bool": (1, False, "v"), "enum": (32, True, "v"),
}
INT_KINDS = [k for k in KINDS if k not in ("bool", "enum")]
COLOR = [("COLOR_UNSPECIFIED", 0), ("RED", 1), ("GREEN", 2), ("BLUE", 3), ("NEGATIVE", -5), ("BIG", 1 << 30)]

# ---- request text ------------------------------------------------------------------------------------------------
_DIGITS = frozenset(b"0123456789")
_NOT_DELIM = frozenset(b"-+._abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789")
_JSON_WS = b" \t\r\n"
# unicode.IsSpace: what strings.TrimSpace removes
_GO_SPACE = "\t\n\v\f\r \x85\xa0\u1680" + "".join(map(chr, range(0x2000, 0x200B))) + "\u2028\u2029\u202f\u205f\u3000"


def scan_number(b, i=0):
    """internal/encoding/json parseNumber: length of the number token at b[i], or 0.  An exponent marker may go
    without digits when a delimiter follows; the value then fails in number_parts"""
    n = len(b)
    j = i
    if j < n and b[j] == 0x2D:
        j += 1
        if j == n:
            return 0
    if j < n and b[j] == 0x30:
        j += 1
    elif j < n and 0x31 <= b[j] <= 0x39:
        while j < n and b[j] in _DIGITS:
            j += 1
    else:
        return 0
    if n - j >= 2 and b[j] == 0x2E and b[j + 1] in _DIGITS:
        j += 2
        while j < n and b[j] in _DIGITS:
            j += 1
    if n - j >= 2 and b[j] in b"eE":
        j += 1
        if b[j] in b"+-":
            j += 1
            if j == n:
                return 0
        while j < n and b[j] in _DIGITS:
            j += 1
    if j < n and b[j] in _NOT_DELIM:
        return 0
    return j - i


def number_parts(raw):
    """parseNumberParts on a whole number token -> (neg, intp, frac with trailing zeros trimmed, exp text) or None"""
    s = bytes(raw)
    neg = s[:1] == b"-"
    if neg:
        s = s[1:]
    if not s:
        return None
    if s[0] == 0x30:
        intp, s = b"", s[1:]
    elif 0x31 <= s[0] <= 0x39:
        k = 1
        while k < len(s) and s[k] in _DIGITS:
            k += 1
        intp, s = s[:k], s[k:]
    else:
        return None
    frac = b""
    if len(s) >= 2 and s[0] == 0x2E and s[1] in _DIGITS:
        k = 2
        while k < len(s) and s[k] in _DIGITS:
            k += 1
        frac, s = s[1:k], s[k:]
    exp = b""
    if len(s) >= 2 and s[0] in b"eE":
        k = 1
        if s[k] in b"+-":
            k += 1
        while k < len(s) and s[k] in _DIGITS:
            k += 1
        exp, s = s[1:k], s[k:]
    if s:
        return None
    return neg, intp, frac.rstrip(b"0"), exp


def parse_int(s, bits):
    """strconv.ParseInt(s, 10, bits) -> int or None"""
    s = bytes(s)
    neg = s[:1] == b"-"
    if s[:1] in (b"+", b"-"):
        s = s[1:]
    if not s or any(c not in _DIGITS for c in s):
        return None
    v = -int(s) if neg else int(s)
    return v if -(1 << (bits - 1)) <= v < 1 << (bits - 1) else None


def parse_uint(s, bits):
    """strconv.ParseUint(s, 10, bits) -> int or None"""
    s = bytes(s)
    if not s or any(c not in _DIGITS for c in s):
        return None
    v = int(s)
    return v if v < 1 << bits else None


def normalize(parts):
    """normalizeToIntString -> integer text or None"""
    neg, intp, frac, exp = parts
    if not intp and not frac:
        return b"0"
    e = 0
    if exp:
        e = parse_int(exp, 32)
        if e is None:
            return None
    if e >= 0:
        if len(frac) > e or len(intp) + e > 20:
            return None
        num = intp + frac + b"0" * (e - len(frac))
    else:
        if frac:
            return None
        index = len(intp) + e
        if index < 0 or intp[index:].strip(b"0"):
            return None
        num = intp[:index]
    return b"-" + num if neg else num


def token_int(raw, kind):
    """Token.Int / Token.Uint of a number token for an integer kind (enum: Int(32)) -> int or None"""
    bits, signed, _ = KINDS[kind]
    parts = number_parts(raw)
    s = normalize(parts) if parts else None
    if s is None:
        return None
    return parse_int(s, bits) if signed else parse_uint(s, bits)


def _first_token_number(s):
    """a fresh decoder's first token of s, if it is a number: its text, else None"""
    i = 0
    while i < len(s) and s[i] in _JSON_WS:
        i += 1
    if i == len(s) or not (s[i] == 0x2D or s[i] in _DIGITS):
        return None
    n = scan_number(s, i)
    return s[i:i + n] if n else None


def value(kind, raw):
    """a JSON value token for a field of `kind` -> int (bool: True / False), or SYNTAX / INVALID_VALUE.
    `raw` is one bare token (number or literal, delimited) or one string token with its quotes."""
    raw = bytes(raw)
    if raw[:1] == b'"':
        s = strref.parse_string(raw[1:-1])
        if isinstance(s, str):
            return SYNTAX if s == strref.SYNTAX else s
        if kind == "bool":
            return INVALID_VALUE
        if kind == "enum":
            names = dict(COLOR)
            try:
                return names.get(s.decode("utf-8"), INVALID_VALUE)
            except UnicodeDecodeError:
                return INVALID_VALUE
        try:
            t = s.decode("utf-8")
        except UnicodeDecodeError:
            return INVALID_VALUE
        if t.strip(_GO_SPACE) != t:
            return INVALID_VALUE
        tok = _first_token_number(s)
        v = token_int(tok, kind) if tok else None
        return INVALID_VALUE if v is None else v
    if raw in (b"true", b"false"):
        return (raw == b"true") if kind == "bool" else INVALID_VALUE
    if raw == b"null":
        raise ValueError("null is not a value of this corpus")
    if scan_number(raw) != len(raw):
        return SYNTAX
    if kind == "bool":
        return INVALID_VALUE
    v = token_int(raw, kind)
    return INVALID_VALUE if v is None else v


def key_value(kind, name):
    """unmarshalMapKey on the decoded key text -> key value or INVALID_VALUE"""
    name = bytes(name)
    if kind == "bool":
        return {b"true": True, b"false": False}.get(name, INVALID_VALUE)
    bits, signed, _ = KINDS[kind]
    v = parse_int(name, bits) if signed else parse_uint(name, bits)
    return INVALID_VALUE if v is None else v


FAIL = "fail"  # encoding/json refuses the body


def body_value(kind, raw):
    """the value a field receives from a token inside `arguments` of a tools/call body: a bare number goes through
    float64 and json.Marshal's text first; strings and literals arrive unchanged.  FAIL where encoding/json refuses
    the number (no float64)."""
    raw = bytes(raw)
    if raw[:1] != b'"' and raw not in (b"true", b"false"):
        b = numref.parse(raw.decode(), 64)
        if b == numref.RANGE:
            return FAIL
        raw = numref.format(b, 64).encode()
    return value(kind, raw)


# ---- wire ----------------------------------------------------------------------------------------------------------
def varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def zigzag(v, bits):
    return ((v << 1) ^ (v >> (bits - 1))) & ((1 << bits) - 1)


def unzigzag(u):
    return (u >> 1) ^ -(u & 1)


def wire_type(kind):
    f = KINDS[kind]
    return (1 if f[0] == 64 else 5) if f[2] == "f" else 0


def wire(kind, v):
    """the payload of one value (no tag)"""
    bits, _, form = KINDS[kind]
    v = int(v)
    if form == "f":
        return (v & ((1 << bits) - 1)).to_bytes(bits // 8, "little")
    if form == "z":
        return varint(zigzag(v, bits))
    return varint(v)  # int32 / enum: sign extended to 64 bits


def tagged(num, kind, v):
    return varint(num << 3 | wire_type(kind)) + wire(kind, v)


def ld(num, payload):
    return varint(num << 3 | 2) + varint(len(payload)) + payload


def packed(num, kind, vals):
    return ld(num, b"".join(wire(kind, v) for v in vals)) if vals else b""


# ---- reply side ----------------------------------------------------------------------------------------------------
def consume_varint(b, i):
    """protowire.ConsumeVarint at b[i] -> (value, next index) or None (cut, or a 10th byte above 1)"""
    v = 0
    for k in range(10):
        if i + k >= len(b):
            return None
        c = b[i + k]
        if k == 9 and c > 1:
            return None
        v |= (c & 0x7F) << (7 * k)
        if c < 0x80:
            return v, i + k + 1
    return None


def from_wire(kind, u):
    """the Go value proto.Unmarshal keeps from the unsigned payload u (varint, or fixed bits)"""
    bits, signed, form = KINDS[kind]
    if kind == "bool":
        return u != 0
    if form == "z":
        return unzigzag(u & 0xFFFFFFFF) if bits == 32 else unzigzag(u)
    u &= (1 << bits) - 1
    return u - (1 << bits) if signed and u >> (bits - 1) else u


def text(kind, v):
    if kind == "bool":
        return b"true" if v else b"false"
    if kind == "enum":
        name = next((n for n, x in COLOR if x == v), None)
        return b'"%s"' % name.encode() if name else b"%d" % v
    return b'"%d"' % v if KINDS[kind][0] == 64 else b"%d" % v


def key_text(kind, v):
    if kind == "string":
        return strref.format_string(v)
    if kind == "bool":
        return b'"true"' if v else b'"false"'
    return b'"%d"' % v


def _consume_fixed(b, i, n):
    if i + n > len(b):
        return None
    return int.from_bytes(b[i:i + n], "little"), i + n


def _consume_value(b, i, wt):
    """a value of wire type 0 / 1 / 5 -> (unsigned payload, next) or None"""
    if wt == 0:
        return consume_varint(b, i)
    return _consume_fixed(b, i, 8 if wt == 1 else 4)


def _fields(b):
    """(number, wire type, payload start, payload end or value, next) for each field of a message; None if malformed.
    Length-delimited: (num, 2, start, end); others: (num, wt, unsigned value, None)"""
    out = []
    i = 0
    while i < len(b):
        r = consume_varint(b, i)
        if r is None:
            return None
        tag, i = r
        num, wt = tag >> 3, tag & 7
        if num == 0 or num > (1 << 29) - 1 or wt not in (0, 1, 2, 5):
            return None
        if wt == 2:
            r = consume_varint(b, i)
            if r is None or r[0] > len(b) - r[1]:
                return None
            out.append((num, 2, r[1], r[1] + r[0]))
            i = r[1] + r[0]
        else:
            r = _consume_value(b, i, wt)
            if r is None:
                return None
            out.append((num, wt, r[0], None))
            i = r[1]
    return out


# bench.All: (number, JSON name, kind, shape) in declaration order; shape s = implicit presence, p = explicit presence
# (oneof member or proto3 optional), r = repeated, m = map (kind is (key kind, value kind)), x = a string field
ALL_FIELDS = (
    [(1 + i, "f" + k.capitalize(), k, "s") for i, k in enumerate(INT_KINDS)]
    + [(13, "fBool", "bool", "s"), (14, "fString", "string", "x"), (16, "fEnum", "enum", "s")]
    + [(21 + i, "r" + k.capitalize(), k, "r") for i, k in enumerate(INT_KINDS)]
    + [(33, "rBool", "bool", "r"), (36, "rEnum", "enum", "r"), (38, "rUnpacked", "int32", "r"),
       (41, "mStrInt32", ("string", "int32"), "m"), (42, "mInt32Str", ("int32", "string"), "m"),
       (44, "mBoolDouble", ("bool", "double"), "m"), (45, "mUint64Bytes", ("uint64", "bytes"), "m"),
       (46, "mStrEnum", ("string", "enum"), "m"), (47, "mSint32Float", ("sint32", "float"), "m"),
       (48, "mFixed64Sfixed32", ("fixed64", "sfixed32"), "m"),
       (51, "oInt32", "int32", "o"), (54, "oBool", "bool", "o"), (55, "oEnum", "enum", "o"),
       (61, "optInt32", "int32", "p"), (63, "optBool", "bool", "p"), (90, "CustomJSON", "string", "x")])
# wkt.Wkt: the integer and bool wrappers (a message holding the value as field 1), a list of Int32Value, a map of
# int32 to Int64Value
WKT_FIELDS = ((5, "bv", "bool", "w"), (6, "i32", "int32", "w"), (7, "i64", "int64", "w"), (8, "u32", "uint32", "w"),
              (9, "u64", "uint64", "w"), (15, "mI64", ("int32", "int64"), "mw"), (20, "rI32", "int32", "rw"))
FIELDS = {"bench.All": ALL_FIELDS, "wkt.Wkt": WKT_FIELDS}


def _scalar(kind, occ, b):
    """one non-message value occurrence (wt, value or (start, end)) of a field of `kind` -> Go value, None for a
    wire type that does not fit (an unknown field), BAD_WIRE"""
    wt, x, end = occ
    if kind in ("string", "bytes"):
        if wt != 2:
            return None
        s = bytes(b[x:end])
        if kind == "string":
            try:
                s.decode("utf-8")
            except UnicodeDecodeError:
                return BAD_WIRE
        return s
    if kind in ("double", "float"):
        return x if wt == (1 if kind == "double" else 5) else None
    return from_wire(kind, x) if wt == wire_type(kind) else None


def _packed_values(kind, b, s, e):
    out = []
    wt = wire_type(kind)
    while s < e:
        r = _consume_value(b[:e], s, wt)
        if r is None:
            return BAD_WIRE
        out.append(from_wire(kind, r[0]))
        s = r[1]
    return out


def _wrapper(kind, b, s, e):
    """a wrapper message's value: the last field 1 of its kind (zero when none); unknown fields skipped"""
    fs = _fields(b[s:e])
    if fs is None:
        return BAD_WIRE
    v = False if kind == "bool" else 0
    for num, wt, x, end in fs:
        if num == 1:
            got = _scalar(kind, (wt, x, end), b[s:e])
            if got is not None:
                v = got
    return v


def _entry(kinds, b, s, e, wrapped):
    fs = _fields(b[s:e])
    if fs is None:
        return BAD_WIRE
    kk, vk = kinds
    zero = lambda k: False if k == "bool" else b"" if k in ("string", "bytes") else 0
    key, val = zero(kk), zero(vk)
    sub = b[s:e]
    for num, wt, x, end in fs:
        if num == 1:
            got = _scalar(kk, (wt, x, end), sub)
        elif num == 2:
            got = _wrapper(vk, sub, x, end) if wrapped and wt == 2 else None if wrapped else _scalar(vk, (wt, x, end), sub)
        else:
            continue
        if got == BAD_WIRE:
            return BAD_WIRE
        if got is not None:
            if num == 1:
                key = got
            else:
                val = got
    return key, val


def _map_value_text(kind, v):
    if kind == "string":
        return strref.format_string(v)
    if kind == "bytes":
        return b'"' + base64.b64encode(v) + b'"'
    if kind in ("double", "float"):
        return numref.format(v, 64 if kind == "double" else 32).encode()
    return text(kind, v)


def decode(msg, b, flags=0):
    """protojson.Marshal(proto.Unmarshal(b)) for the fields of FIELDS[msg] (other fields must not occur) -> text or
    BAD_WIRE.  flags & 1: ", " between members, list elements and map entries."""
    table = FIELDS[msg]
    by_num = {f[0]: f for f in table}
    fs = _fields(b)
    if fs is None:
        return BAD_WIRE
    vals = {}
    oneof_last = None
    for num, wt, x, end in fs:
        f = by_num.get(num)
        if f is None:
            raise ValueError("field %d is not in this reference's table" % num)
        _, name, kind, shape = f
        if shape in ("s", "p", "o", "x"):
            got = _scalar(kind, (wt, x, end), b)
            if got == BAD_WIRE:
                return BAD_WIRE
            if got is not None:
                vals[num] = got
                if shape == "o":
                    if oneof_last is not None and oneof_last != num:
                        vals.pop(oneof_last, None)
                    oneof_last = num
        elif shape == "w":
            if wt != 2:
                continue
            got = _wrapper(kind, b, x, end)
            if got == BAD_WIRE:
                return BAD_WIRE
            vals[num] = got
        elif shape in ("r", "rw"):
            lst = vals.setdefault(num, [])
            if shape == "rw":
                if wt == 2:
                    got = _wrapper(kind, b, x, end)
                    if got == BAD_WIRE:
                        return BAD_WIRE
                    lst.append(got)
            elif wt == 2:
                got = _packed_values(kind, b, x, end)
                if got == BAD_WIRE:
                    return BAD_WIRE
                lst += got
            else:
                got = _scalar(kind, (wt, x, end), b)
                if got is not None:
                    lst.append(got)
        else:  # maps
            if wt != 2:
                continue
            got = _entry(kind, b, x, end, shape == "mw")
            if got == BAD_WIRE:
                return BAD_WIRE
            vals.setdefault(num, {})[got[0]] = got[1]
    sep = b", " if flags & 1 else b","
    parts = []
    for num, name, kind, shape in table:
        if num not in vals:
            continue
        v = vals[num]
        head = b'"' + name.encode() + b'":'
        if shape in ("s", "x"):
            if v in (0, False, b""):
                continue
            parts.append(head + (strref.format_string(v) if shape == "x" else text(kind, v)))
        elif shape in ("p", "o", "w"):
            parts.append(head + text(kind, v))
        elif shape in ("r", "rw"):
            if v:
                parts.append(head + b"[" + sep.join(text(kind, x) for x in v) + b"]")
        else:
            if v:
                kk, vk = kind
                keys = sorted(v)
                parts.append(head + b"{" + sep.join(key_text(kk, k) + b":" + _map_value_text(vk, v[k]) for k in keys) + b"}")
    return b"{" + sep.join(parts) + b"}"
