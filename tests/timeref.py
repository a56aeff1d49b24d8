"""Exact reference for the well-known types with a JSON form of their own - google.protobuf.Timestamp, Duration,
FieldMask, the nine wrappers and Empty - as protojson reads and writes them and proto.Unmarshal / proto.Marshal carry
them on the wire.

Request side
  days_from_civil(y, m, d)  - days from 1970-01-01, proleptic Gregorian, year 0000 included (own formula).
  timestamp(s)              - the decoded text of a Timestamp string -> (seconds, nanos), INVALID_VALUE or RANGE.
  duration(s)               - the same for a Duration; field_mask(s) -> [snake_case paths] or INVALID_VALUE.
  value(typ, raw)           - one JSON value token (a string token with its quotes, or a bare token) for a field of
                              type `typ` (TS, DUR, FM, EMPTY or a wrapper) -> the Go value, or a status category.
  payload(typ, v)           - proto.Marshal of that value as the body of its message (no tag, no length).
  root_value(typ, raw)      - value() for the whole request of a method whose input message is the type itself.
Reply side
  decode(msg, wire, flags)  - protojson.Marshal(proto.Unmarshal(wire)) for wkt.Times (TIMES) and the method roots
                              google.protobuf.Timestamp / Duration / FieldMask -> text, or a status category.

Status categories: INVALID_VALUE means the text is refused; RANGE means a value was read but lies outside protojson's
bounds (Timestamp seconds, Duration seconds, and on the reply side the nanos and sign checks).  Go reports both as one
kind of error; the split is this project's own.  A reply that proto.Unmarshal refuses is BAD_WIRE, or INVALID_UTF8 for
a proto3 string (a FieldMask path, a StringValue, a string map key or oneof member) that is not UTF-8.

Plain Python with integer arithmetic (intref, strref and numref for the wrapper values); independent of the oracle and
of the device code.  The schema facts restate tests/timecorpus.py's wkt.Times.

Rules that rest on memory of protobuf-go v1.36 and Go's standard library, not on a source that can be read here:
  * time.Parse(RFC3339Nano) tries a strict RFC 3339 reader first and falls back to the general layout parser, so the
    union of both is accepted; the general parser is the wider one: a 4-digit year (0000 included); 2-digit month
    (1..12) and day; 'T' exactly; an hour of one or two digits (< 24); 2-digit minute and second (< 60); '.' or ','
    followed by at least one digit starts a fraction of any length, cut to 9 digits (no rounding); then 'Z' exactly,
    or a sign, 2-digit hour, ':', 2-digit minute checked with '>' (so +24:60 passes); nothing after it.  The day is
    checked against daysIn(month, year) with the Gregorian leap rule after the whole text is read.
  * protojson.unmarshalTimestamp: the seconds range [-62135596800, 253402300799] is checked on t.Unix() (after the
    offset) BEFORE its own fraction check, which refuses a '.' fraction longer than 9 digits through
    LastIndexByte(s, '.') / LastIndexAny(s, "Z-+") (a ',' fraction is only cut).  So an out-of-range value with a long
    '.' fraction is a RANGE error.
  * protojson.parseDuration: an 's' last; an optional sign; then one '0', a run of digits starting with 1-9, or
    nothing before a '.'; after an optional '.' up to 9 digits (none is allowed: "1.s" and ".s" are 0 nanos, missing
    digits count as zeros); the integer part through strconv.ParseInt(_, 10, 64); a '-' negates seconds and nanos
    both.  Then |seconds| <= 315576000000.  (The corpus puts no sign inside a fraction.)
  * protojson.unmarshalFieldMask: strings.TrimSpace (unicode.IsSpace), "" is an empty mask, else strings.Split(",");
    every path s0 is refused when it holds '_' or JSONSnakeCase(s0) is no protoreflect.FullName.IsValid (ASCII letters
    and '_' first in each '.'-segment, then letters, digits, '_'); JSONSnakeCase puts '_' before an ASCII capital and
    lowers it.
  * A wrapper in JSON is its bare value (read as a singular field of its kind); its zero value leaves the wrapper
    message present but empty.  Empty is an object without members.  `null` for a singular or oneof field leaves it
    unset (the oneof is not marked), but is a value like any other as a list element or map value: a wrapper refuses
    it as an invalid value, the other types as an unexpected token (SYNTAX).
  * proto.Marshal writes fields in number order (the schema declares them so), map entries sorted by key, the key and
    the value of every entry, a present message even when empty, int64 / int32 as varints of their 64-bit sign
    extension.
  * proto.Unmarshal keeps int64(v) for seconds and int32(v) for nanos; the last value of a field wins; a field of the
    wrong wire type, an unknown field and a group are skipped (a group up to the end-group of its own number; an
    unmatched end-group, field number 0 or wire types 6 / 7 fail); a singular message field met several times is
    merged field by field (FieldMask paths append), unless a sibling oneof member was set in between (then the
    member starts afresh); several value fields inside one map entry merge the same way, a later entry with the same
    key replaces the whole value; an entry without value holds the empty message.
  * protojson.Marshal: Timestamp checks seconds against the range above and 0 <= nanos <= 999999999, then writes UTC
    text with 0, 3, 6 or 9 fraction digits and 'Z'; Duration checks |seconds| <= 315576000000, |nanos| <= 999999999
    and that their signs do not differ, then writes [-]seconds with 0, 3, 6 or 9 fraction digits and 's'; FieldMask
    checks FullName.IsValid and JSONSnakeCase(JSONCamelCase(s)) == s for each path and joins the camelCase forms with
    ','.  Fields go in declaration order, map keys sorted (strings by bytes, integers by value).  These errors come
    after proto.Unmarshal has read the whole item, so any wire error anywhere in it is reported instead; among them the
    first in output order wins.
"""
import base64
import datetime

import intref
import numref
import strref

SYNTAX, INVALID_VALUE, RANGE = "syntax", "invalid_value", "range"
INVALID_UTF8, BAD_WIRE, UNSUPPORTED = "invalid_utf8", "bad_wire", "unsupported"
# GGR_ST_* of each category
STATUS = {SYNTAX: 1, INVALID_VALUE: 3, RANGE: 4, INVALID_UTF8: 5, BAD_WIRE: 10, UNSUPPORTED: 11}

TS, DUR, FM, EMPTY = "ts", "dur", "fm", "empty"
WRAPPERS = {"bool": "BoolValue", "int32": "Int32Value", "int64": "Int64Value", "uint32": "UInt32Value",
            "uint64": "UInt64Value", "float": "FloatValue", "double": "DoubleValue", "string": "StringValue",
            "bytes": "BytesValue"}
MIN_TS, MAX_TS = -62135596800, 253402300799  # 0001-01-01T00:00:00Z, 9999-12-31T23:59:59Z
MAX_DUR = 315576000000  # 10 000 years of 365.25 days


def wrapper(kind):
    return ("w", kind)


def is_wrapper(typ):
    return isinstance(typ, tuple) and typ[0] == "w"


# ---- calendar ------------------------------------------------------------------------------------------------------
def is_leap(y):
    return y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)


_MONTH_DAYS = (31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31)
_DAYS_BEFORE = [sum(_MONTH_DAYS[:m]) for m in range(12)]


def days_in(m, y):
    return 29 if m == 2 and is_leap(y) else _MONTH_DAYS[m - 1]


def _days_from_year0(y, m, d):
    """days from 0000-01-01 to y-m-d (y >= 0): 365 a year plus one for each leap year in [0, y)"""
    leaps = (y + 3) // 4 - (y + 99) // 100 + (y + 399) // 400
    return 365 * y + leaps + _DAYS_BEFORE[m - 1] + (1 if m > 2 and is_leap(y) else 0) + d - 1


_EPOCH = _days_from_year0(1970, 1, 1)


def days_from_civil(y, m, d):
    return _days_from_year0(y, m, d) - _EPOCH


# ---- request text --------------------------------------------------------------------------------------------------
def _digit(s, i):
    return i < len(s) and 0x30 <= s[i] <= 0x39


def _getnum(s, i, fixed):
    """time.getnum: one or two digits (fixed: exactly two) -> (value, next) or None"""
    if not _digit(s, i):
        return None
    if not _digit(s, i + 1):
        return None if fixed else (s[i] - 0x30, i + 1)
    return (s[i] - 0x30) * 10 + s[i + 1] - 0x30, i + 2


def timestamp(s):
    """time.Parse(time.RFC3339Nano, s) and protojson's checks -> (seconds, nanos), INVALID_VALUE or RANGE"""
    s = bytes(s)
    n = len(s)
    if n < 4 or not all(_digit(s, k) for k in range(4)):
        return INVALID_VALUE
    year, i = int(s[:4]), 4
    fields = []
    for sep, fixed, top in ((b"-", True, 12), (b"-", True, 99), (b"T", False, 23), (b":", True, 59), (b":", True, 59)):
        if s[i:i + 1] != sep:
            return INVALID_VALUE
        r = _getnum(s, i + 1, fixed)
        if r is None or r[0] > top:
            return INVALID_VALUE
        fields.append(r[0])
        i = r[1]
    month, day, hour, minute, sec = fields
    if month < 1:
        return INVALID_VALUE
    nanos = 0
    if n - i >= 2 and s[i] in b".," and _digit(s, i + 1):
        j = i + 1
        while _digit(s, j):
            j += 1
        nanos = int(s[i + 1:j][:9].ljust(9, b"0"))
        i = j
    if s[i:i + 1] == b"Z":
        off, i = 0, i + 1
    else:
        if n - i < 6 or s[i + 3] != 0x3A:
            return INVALID_VALUE
        oh, om = _getnum(s[i + 1:i + 3], 0, True), _getnum(s[i + 4:i + 6], 0, True)
        if oh is None or om is None or oh[0] > 24 or om[0] > 60 or s[i] not in b"+-":
            return INVALID_VALUE
        off = (oh[0] * 60 + om[0]) * 60 * (-1 if s[i] == 0x2D else 1)
        i += 6
    if i != n or day < 1 or day > days_in(month, year):
        return INVALID_VALUE
    secs = days_from_civil(year, month, day) * 86400 + hour * 3600 + minute * 60 + sec - off
    if not MIN_TS <= secs <= MAX_TS:
        return RANGE
    p = s.rfind(b".")
    z = max(s.rfind(b"Z"), s.rfind(b"-"), s.rfind(b"+"))
    if p >= 0 and z >= p and z - p > len(".999999999"):
        return INVALID_VALUE
    return secs, nanos


def duration(s):
    """protojson parseDuration and the seconds range -> (seconds, nanos), INVALID_VALUE or RANGE"""
    s = bytes(s)
    if len(s) < 2 or s[-1:] != b"s":
        return INVALID_VALUE
    b = s[:-1]
    neg = b[:1] == b"-"
    if b[:1] in (b"-", b"+"):
        b = b[1:]
    if not b:
        return INVALID_VALUE
    intp = b""
    if b[0] == 0x30:
        b = b[1:]
    elif 0x31 <= b[0] <= 0x39:
        k = 1
        while _digit(b, k):
            k += 1
        intp, b = b[:k], b[k:]
    elif b[0] != 0x2E:
        return INVALID_VALUE
    nanos = 0
    if b:
        if b[0] != 0x2E or len(b) - 1 > 9 or not all(_digit(b, k) for k in range(1, len(b))):
            return INVALID_VALUE
        nanos = int(b[1:].ljust(9, b"0"))
    secs = intref.parse_int(intp, 64) if intp else 0
    if secs is None:
        return INVALID_VALUE
    if neg:
        secs, nanos = -secs, -nanos
    if not -MAX_DUR <= secs <= MAX_DUR:
        return RANGE
    return secs, nanos


GO_SPACE = intref._GO_SPACE  # unicode.IsSpace


def snake(s):
    """strs.JSONSnakeCase (bytes)"""
    out = bytearray()
    for c in s:
        if 0x41 <= c <= 0x5A:
            out += b"_" + bytes([c + 32])
        else:
            out.append(c)
    return bytes(out)


def camel(s):
    """strs.JSONCamelCase (bytes)"""
    out = bytearray()
    was = False
    for c in s:
        if c != 0x5F:
            out.append(c - 32 if was and 0x61 <= c <= 0x7A else c)
        was = c == 0x5F
    return bytes(out)


def _ident_char(c, first):
    return c == 0x5F or 0x41 <= c <= 0x5A or 0x61 <= c <= 0x7A or (not first and 0x30 <= c <= 0x39)


def full_name_valid(s):
    """protoreflect.FullName(s).IsValid"""
    return all(seg and _ident_char(seg[0], True) and all(_ident_char(c, False) for c in seg[1:]) for seg in bytes(s).split(b"."))


def field_mask(s):
    """protojson unmarshalFieldMask on the decoded text -> [paths] or INVALID_VALUE"""
    t = bytes(s).decode("utf-8").strip(GO_SPACE).encode()
    if not t:
        return []
    out = []
    for s0 in t.split(b","):
        p = snake(s0)
        if b"_" in s0 or not full_name_valid(p):
            return INVALID_VALUE
        out.append(p)
    return out


def _wrapper_value(kind, raw):
    if kind in ("float", "double"):
        if raw[:1] == b'"' or raw in (b"true", b"false", b"null"):
            raise ValueError("the corpus writes float wrappers as bare numbers")
        v = numref.parse(raw, 64 if kind == "double" else 32)
        return INVALID_VALUE if v == numref.RANGE else v
    if kind in ("string", "bytes"):
        if raw[:1] != b'"':
            return INVALID_VALUE
        t = strref.parse_string(raw[1:-1])
        if isinstance(t, str):
            return t
        return t if kind == "string" else strref.b64_parse(t)
    return intref.value(kind, raw)


def value(typ, raw, element=False):
    """one JSON value token for a field of `typ` -> Go value (TS / DUR: (seconds, nanos); FM: [paths]; EMPTY: True;
    wrapper: its value), None for a null that leaves the field unset, or a status category.  `element`: the token is
    a list element or map value, where null is a value."""
    raw = bytes(raw)
    if raw == b"null":
        if not element:
            return None
        return INVALID_VALUE if is_wrapper(typ) else SYNTAX
    if is_wrapper(typ):
        return _wrapper_value(typ[1], raw)
    if typ == EMPTY:
        return True if raw.replace(b" ", b"") == b"{}" else SYNTAX
    if raw[:1] != b'"':
        return SYNTAX
    t = strref.parse_string(raw[1:-1])
    if isinstance(t, str):
        return t
    return {TS: timestamp, DUR: duration, FM: field_mask}[typ](t)


def root_value(typ, raw):
    """the whole request text of a method whose input is `typ`: the tool handler of the reference gives "" and "{}" to
    no parser (an empty message); anything else is protojson.Unmarshal, where null is a token like any other"""
    return True if bytes(raw) in (b"", b"{}") else value(typ, raw, element=True)


def _varint_field(num, v):
    return intref.varint(num << 3) + intref.varint(v) if v else b""


def payload(typ, v):
    """proto.Marshal of a value as the body of its message"""
    if typ in (TS, DUR):
        return _varint_field(1, v[0]) + _varint_field(2, v[1])
    if typ == FM:
        return b"".join(intref.ld(1, p) for p in v)
    if typ == EMPTY:
        return b""
    kind = typ[1]
    if kind in ("float", "double"):
        return b"" if v == 0 else (b"\x0d" + v.to_bytes(4, "little") if kind == "float" else b"\x09" + v.to_bytes(8, "little"))
    if kind in ("string", "bytes"):
        return intref.ld(1, v) if v else b""
    return b"" if v in (0, False) else intref.tagged(1, kind, int(v))


# ---- wkt.Times -----------------------------------------------------------------------------------------------------
# (number, JSON name, type, shape): s = singular message, r = repeated, m = map (type = (key kind, value type)),
# o = oneof member; "times" is wkt.Times itself, "string" the oneof's string member
TIMES = (
    (1, "ts", TS, "s"), (2, "rTs", TS, "r"), (3, "mTs", ("string", TS), "m"), (4, "mI64Ts", ("int64", TS), "m"),
    (5, "mD", ("string", DUR), "m"), (6, "d", DUR, "s"), (7, "rD", DUR, "r"), (8, "fm", FM, "s"),
    (9, "oTs", TS, "o"), (10, "oD", DUR, "o"), (11, "oFm", FM, "o"), (12, "oS", "string", "o"),
    (13, "inner", "times", "s"), (14, "e", EMPTY, "s"), (15, "rE", EMPTY, "r"),
    (16, "bv", wrapper("bool"), "s"), (17, "i32v", wrapper("int32"), "s"), (18, "i64v", wrapper("int64"), "s"),
    (19, "u32v", wrapper("uint32"), "s"), (20, "u64v", wrapper("uint64"), "s"), (21, "fv", wrapper("float"), "s"),
    (22, "dv", wrapper("double"), "s"), (23, "sv", wrapper("string"), "s"), (24, "byv", wrapper("bytes"), "s"),
    (25, "rI64v", wrapper("int64"), "r"), (26, "mSv", ("string", wrapper("string")), "m"), (27, "rFm", FM, "r"),
)
ROOTS = {"google.protobuf.Timestamp": TS, "google.protobuf.Duration": DUR, "google.protobuf.FieldMask": FM}


class _Fail(Exception):
    def __init__(self, cat):
        super().__init__(cat)
        self.cat = cat


def _skip_group(b, i, num):
    while True:
        r = intref.consume_varint(b, i)
        if r is None:
            raise _Fail(BAD_WIRE)
        tag, i = r
        n, wt = tag >> 3, tag & 7
        if n == 0 or n > (1 << 29) - 1:
            raise _Fail(BAD_WIRE)
        if wt == 4:
            if n != num:
                raise _Fail(BAD_WIRE)
            return i
        i = _skip_value(b, i, n, wt)


def _skip_value(b, i, num, wt):
    if wt == 0:
        r = intref.consume_varint(b, i)
        if r is None:
            raise _Fail(BAD_WIRE)
        return r[1]
    if wt in (1, 5):
        k = 8 if wt == 1 else 4
        if i + k > len(b):
            raise _Fail(BAD_WIRE)
        return i + k
    if wt == 2:
        r = intref.consume_varint(b, i)
        if r is None or r[0] > len(b) - r[1]:
            raise _Fail(BAD_WIRE)
        return r[1] + r[0]
    if wt == 3:
        return _skip_group(b, i, num)
    raise _Fail(BAD_WIRE)  # an end-group without its start, wire types 6 and 7


def _fields(b):
    """[(number, wire type, value (wt 0 / 1 / 5) or payload bytes (wt 2))] of one message; groups are skipped"""
    out, i = [], 0
    while i < len(b):
        r = intref.consume_varint(b, i)
        if r is None:
            raise _Fail(BAD_WIRE)
        tag, i = r
        num, wt = tag >> 3, tag & 7
        if num == 0 or num > (1 << 29) - 1:
            raise _Fail(BAD_WIRE)
        j = _skip_value(b, i, num, wt)
        if wt == 0:
            out.append((num, 0, intref.consume_varint(b, i)[0]))
        elif wt in (1, 5):
            out.append((num, wt, int.from_bytes(b[i:j], "little")))
        elif wt == 2:
            start = intref.consume_varint(b, i)[1]
            out.append((num, 2, bytes(b[start:j])))
        i = j
    return out


def _utf8(s):
    try:
        s.decode("utf-8")
    except UnicodeDecodeError:
        raise _Fail(INVALID_UTF8)
    return s


def _new(typ):
    if typ in (TS, DUR):
        return [0, 0]
    if typ == FM:
        return []
    if typ == "times":
        return {}
    if typ == EMPTY:
        return True
    return {"bool": False, "float": 0, "double": 0, "string": b"", "bytes": b""}.get(typ[1], 0)


def _merge(typ, cur, b):
    """proto.Unmarshal of message bytes b into the value cur of type typ -> the merged value"""
    fs = _fields(b)
    if typ in (TS, DUR):
        for num, wt, x in fs:
            if num == 1 and wt == 0:
                cur[0] = intref.from_wire("int64", x)
            elif num == 2 and wt == 0:
                cur[1] = intref.from_wire("int32", x)
        return cur
    if typ == FM:
        for num, wt, x in fs:
            if num == 1 and wt == 2:
                cur.append(_utf8(x))
        return cur
    if typ == EMPTY:
        return cur
    if typ == "times":
        _merge_times(cur, fs)
        return cur
    kind = typ[1]
    for num, wt, x in fs:
        if num != 1:
            continue
        if kind in ("string", "bytes"):
            if wt == 2:
                cur = _utf8(x) if kind == "string" else x
        elif kind in ("float", "double"):
            if wt == (5 if kind == "float" else 1):
                cur = x
        elif wt == 0:
            cur = intref.from_wire(kind, x)
    return cur


def _map_key(kind, x, wt):
    if kind == "string":
        return _utf8(x) if wt == 2 else None
    return intref.from_wire("int64", x) if wt == 0 else None


def _merge_times(m, fs):
    by_num = {f[0]: f for f in TIMES}
    for num, wt, x in fs:
        f = by_num.get(num)
        if f is None:
            continue  # unknown field
        _, _, typ, shape = f
        if wt != 2:
            continue  # every field of wkt.Times is length-delimited: another wire type is an unknown field
        if shape == "o":
            if m.get("oneof") != num:
                m.pop(m.get("oneof"), None)
                m["oneof"] = num
            if typ == "string":
                m[num] = _utf8(x)
                continue
        if shape in ("s", "o"):
            m[num] = _merge(typ, m[num] if num in m else _new(typ), x)
        elif shape == "r":
            m.setdefault(num, []).append(_merge(typ, _new(typ), x))
        else:
            kk, vt = typ
            key, val = (b"" if kk == "string" else 0), _new(vt)
            for n2, wt2, x2 in _fields(x):
                if n2 == 1:
                    k = _map_key(kk, x2, wt2)
                    if k is not None:
                        key = k
                elif n2 == 2 and wt2 == 2:
                    val = _merge(vt, val, x2)
            m.setdefault(num, {})[key] = val


def _ts_text(v):
    secs, nanos = v
    if not MIN_TS <= secs <= MAX_TS or not 0 <= nanos <= 999999999:
        raise _Fail(RANGE)
    t = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=secs)
    x = b"%04d-%02d-%02dT%02d:%02d:%02d.%09d" % (t.year, t.month, t.day, t.hour, t.minute, t.second, nanos)
    return b'"' + _trim(x) + b'Z"'


def _trim(x):
    for suf in (b"000", b"000", b".000"):
        if x.endswith(suf):
            x = x[:-len(suf)]
    return x


def _dur_text(v):
    secs, nanos = v
    if not -MAX_DUR <= secs <= MAX_DUR or not -999999999 <= nanos <= 999999999 or (secs > 0 > nanos) or (secs < 0 < nanos):
        raise _Fail(RANGE)
    sign = b"-" if secs < 0 or nanos < 0 else b""
    return b'"' + _trim(sign + b"%d.%09d" % (abs(secs), abs(nanos))) + b's"'


def _fm_text(v):
    out = []
    for s in v:
        cc = camel(s)
        if not full_name_valid(s) or snake(cc) != s:
            raise _Fail(INVALID_VALUE)
        out.append(cc)
    return b'"' + b",".join(out) + b'"'


def _float_text(bits, width):
    inf = 0x7FF0000000000000 if width == 64 else 0x7F800000
    mag = bits & ~(1 << (width - 1))
    if mag > inf:
        return b'"NaN"'
    if mag == inf:
        return b'"-Infinity"' if bits >> (width - 1) else b'"Infinity"'
    return numref.format(bits, width).encode()


def text(typ, v, sep):
    if typ == TS:
        return _ts_text(v)
    if typ == DUR:
        return _dur_text(v)
    if typ == FM:
        return _fm_text(v)
    if typ == EMPTY:
        return b"{}"
    if typ == "times":
        return _times_text(v, sep)
    kind = typ[1]
    if kind == "string":
        return strref.format_string(v)
    if kind == "bytes":
        return b'"' + base64.b64encode(v) + b'"'
    if kind in ("float", "double"):
        return _float_text(v, 32 if kind == "float" else 64)
    return intref.text(kind, v)


def _times_text(m, sep):
    parts = []
    for num, name, typ, shape in TIMES:
        if num not in m:
            continue
        v = m[num]
        head = b'"' + name.encode() + b'":'
        if shape == "o" and typ == "string":
            parts.append(head + strref.format_string(v))
        elif shape in ("s", "o"):
            parts.append(head + text(typ, v, sep))
        elif shape == "r":
            parts.append(head + b"[" + sep.join(text(typ, x, sep) for x in v) + b"]")
        else:
            kk, vt = typ
            ents = [intref.key_text(kk, k) + b":" + text(vt, v[k], sep) for k in sorted(v)]
            parts.append(head + b"{" + sep.join(ents) + b"}")
    return b"{" + sep.join(parts) + b"}"


def decode(msg, wire, flags=0):
    """protojson.Marshal(proto.Unmarshal(wire)) -> text or a status category.  flags & 1: ", " between members, list
    elements and map entries."""
    typ = ROOTS.get(msg, "times" if msg == "wkt.Times" else None)
    if typ is None:
        raise ValueError("no table for " + msg)
    try:
        v = _merge(typ, _new(typ), bytes(wire))
    except _Fail as e:
        return e.cat
    try:
        return text(typ, v, b", " if flags & 1 else b",")
    except _Fail as e:
        return e.cat
