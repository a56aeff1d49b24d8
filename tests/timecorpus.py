"""Seeded corpus of Timestamp, Duration, FieldMask, wrapper and Empty values for the time tests, in both directions.
Expected values come from tests/timeref.py alone.

The schema fixture has no map of Timestamps and no Timestamp inside a oneof, so the corpus adds one message in memory:
wkt.Times (times.proto, service wkt.TimesService with method EchoTimes), appended to tests/golden/schemas.binpb by
extended_fds().  It holds a singular, a repeated and an int64- and string-keyed map of Timestamps, a Duration in the
same shapes, a FieldMask singular and repeated, a oneof of {Timestamp, Duration, FieldMask, string}, Empty singular and
repeated, the nine wrappers, a list of Int64Value, a map of StringValue and a field of its own type.

Request items are (message, start offset, json, expected wire or status category, escape gap): every text form of each
type (timeref's edges: month ends, leap days, both range ends reached directly and through offsets -24:60..+24:60,
hours of one and two digits, fractions of 0..12 digits after '.' and ',', Duration integer parts of 1..20 digits,
FieldMask case and space edges), each also with a \\u escape, in every position of wkt.Times (singular, list element,
map value under a string and an int64 key, oneof member, nested member) and as the method root.  `escape gap` is set
for a FieldMask written with escapes: the kernels refuse those as GGR_ST_UNSUPPORTED.  Long Timestamp lists sit at,
below and above the value limits of the walker's tiers, large Timestamp maps reach the lock-step parser's big tables.

Reply items are (message, start offset, wire, expected text, expected text with comma-space): seconds varints of every
length 1..10, nanos at and beyond their bounds and above 32 bits, fields repeated, unknown fields and groups inside a
payload, split occurrences with a oneof sibling in between, payloads placed across the 8-byte header window, the 32 /
64 / 96-byte rounds and the 4 KB plain-mask limit, Marshal-time errors behind a later wire error, Timestamp lists of
200..250 and 1000 entries for both lock-step reply tiers, and unsorted Timestamp maps with repeated keys.
"""
import datetime
import os
import random
import sys

import intref as I
import timeref as T

TM = "wkt.Times"
TOOL = "wkt_timesservice_echotimes"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = ".google.protobuf."


# ---- schema --------------------------------------------------------------------------------------------------------
def times_file():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_descriptors as MD
    from google.protobuf import descriptor_pb2 as dpb
    fd = dpb.FileDescriptorProto(name="times.proto", package="wkt", syntax="proto3")
    for dep in ("timestamp", "duration", "wrappers", "empty", "field_mask"):
        fd.dependency.append("google/protobuf/%s.proto" % dep)
    m = fd.message_type.add(name="Times")
    W = ".wkt.Times"
    wkt = {T.TS: G + "Timestamp", T.DUR: G + "Duration", T.FM: G + "FieldMask", T.EMPTY: G + "Empty", "times": W,
           "string": "string"}
    m.oneof_decl.add(name="choice")
    for num, json_name, typ, shape in T.TIMES:
        name = MD_NAMES[num]
        if shape == "m":
            kk, vt = typ
            MD.add_map(m, W, name, num, kk, wkt[vt] if vt in wkt else G + T.WRAPPERS[vt[1]])
            continue
        t = wkt[typ] if typ in wkt else G + T.WRAPPERS[typ[1]]
        f = MD.add_field(m, name, num, t, repeated=shape == "r", oneof=0 if shape == "o" else None)
        assert f.json_name == json_name, (f.json_name, json_name)
    s = fd.service.add(name="TimesService")
    MD.add_method(s, "EchoTimes", W, W)
    return fd


MD_NAMES = {1: "ts", 2: "r_ts", 3: "m_ts", 4: "m_i64_ts", 5: "m_d", 6: "d", 7: "r_d", 8: "fm", 9: "o_ts", 10: "o_d",
            11: "o_fm", 12: "o_s", 13: "inner", 14: "e", 15: "r_e", 16: "bv", 17: "i32v", 18: "i64v", 19: "u32v",
            20: "u64v", 21: "fv", 22: "dv", 23: "sv", 24: "byv", 25: "r_i64v", 26: "m_sv", 27: "r_fm"}
NUM = {v: k for k, v in MD_NAMES.items()}


def extended_fds():
    """tests/golden/schemas.binpb with times.proto appended (a FileDescriptorSet is a list of field 1)"""
    with open(os.path.join(ROOT, "tests", "golden", "schemas.binpb"), "rb") as fh:
        base = fh.read()
    return base + I.ld(1, times_file().SerializeToString(deterministic=True))


# ---- request forms ------------------------------------------------------------------------------------------------
def _q(s):
    return b'"' + (s.encode() if isinstance(s, str) else s) + b'"'


def _civil(secs):
    """UTC text (no zone) of secs; year 0000 for the days in front of 0001-01-01"""
    if secs >= T.MIN_TS:
        t = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=secs)
        return "%04d-%02d-%02dT%02d:%02d:%02d" % (t.year, t.month, t.day, t.hour, t.minute, t.second)
    back = T.MIN_TS - secs  # seconds in front of 0001-01-01T00:00:00
    d, r = divmod(back + 86399, 86400)
    r = 86400 * d - back
    return "0000-12-%02dT%02d:%02d:%02d" % (32 - d, r // 3600, r // 60 % 60, r % 60)


def _offsets():
    out = [(0, 0), (0, 1), (1, 0), (5, 30), (12, 0), (23, 59), (24, 0), (24, 59), (24, 60), (0, 60), (23, 60)]
    return [(sg, h, m) for h, m in out for sg in "+-"]


def timestamp_forms():
    """decoded texts of Timestamp strings"""
    out = []
    for y in (2023, 2024, 1):
        for m in range(1, 13):
            last = T.days_in(m, y)
            out += ["%04d-%02d-%02dT12:00:00Z" % (y, m, d) for d in (last, last + 1)]
    for y in (0, 4, 1900, 2000, 2024, 2100, 9996):
        out += ["%04d-02-29T00:00:00Z" % y, "%04d-02-28T23:59:59.5Z" % y, "%04d-03-01T00:00:00Z" % y]
    out += ["0000-01-01T00:00:00Z", "9999-12-31T23:59:59.999999999Z", "1969-12-31T23:59:59.999999999Z", "1970-01-01T00:00:00Z"]
    for target in (T.MIN_TS, T.MIN_TS - 1, T.MAX_TS, T.MAX_TS + 1, 0, -1):
        if target <= T.MAX_TS:
            out.append(_civil(target) + "Z")
        for sg, h, m in _offsets():
            off = (h * 60 + m) * 60 * (1 if sg == "+" else -1)
            local = target + off
            if local <= T.MAX_TS:  # else the local time would lie in year 10000
                out.append(_civil(local) + "%s%02d:%02d" % (sg, h, m))
    out += ["2024-05-06T%sZ" % t for t in ("7:08:09", "07:08:09", "24:00:00", "23:59:59", "1:2:3", "7:8:09", "07:08:9",
                                          "007:08:09", "23:60:00", "23:59:60", "-1:00:00")]
    for sep in ".,":
        for k in range(13):
            for zone in ("Z", "+01:00", "-00:30"):
                out.append("2024-05-06T07:08:09" + (sep + "123456789012"[:k] if k else "") + zone)
    out += ["9999-12-31T23:59:59.1234567890-00:01", "0000-12-31T23:59:59.1234567890Z",  # out of range, '.' too long
            "9999-12-31T23:59:59,1234567890-00:01", "2024-05-06T07:08:09.Z", "2024-05-06T07:08:09,Z", "2024-05-06T07:08:09.x1Z"]
    out += ["2024-05-06t07:08:09Z", "2024-05-06T07:08:09z", "2024-05-06T07:08Z", "2024-05-06", "2024-05-06T07:08:09",
            "2024-05-06T07:08:09Z ", " 2024-05-06T07:08:09Z", "2024-05-06T07:08:09ZZ", "2024-05-06T07:08:09+01:00:00",
            "2024-05-06T07:08:09+0100", "2024-05-06T07:08:09+1:00", "2024-05-06T07:08:09+01:0", "2024-5-06T07:08:09Z",
            "2024-05-6T07:08:09Z", "24-05-06T07:08:09Z", "20240-05-06T07:08:09Z", "2024-00-06T07:08:09Z",
            "2024-13-06T07:08:09Z", "2024-05-00T07:08:09Z", "2024-05-06 07:08:09Z", "2024/05/06T07:08:09Z", "",
            "2024-05-06T07:08:09*01:00", "2024-05-06T07:08:09+01-00", "2024-05-06T07:08:09+25:00", "2024-05-06T07:08:09-24:61"]
    return list(dict.fromkeys(out))


def duration_forms():
    out = []
    for k in range(1, 21):
        d = "12345678901234567890"[:k]
        out += [d + "s", "-" + d + "s", "+" + d + ".5s"]
    out += ["9223372036854775807s", "9223372036854775808s", "-9223372036854775808s", "-9223372036854775807s",
            "315576000000s", "315576000001s", "-315576000000s", "-315576000001s", "315576000000.999999999s",
            "-315576000000.999999999s", "315576000001.000000001s"]
    for k in range(11):
        out += ["1." + "1234567890"[:k] + "s", "-0." + "9876543210"[:k] + "s"]
    out += ["0", "00s", ".s", "1.s", "-.5s", "+", "+s", "-s", "s", "0s", "-0s", "+0s", "01s", "1", "1S", " 1s", "1s ",
            "1.5e3s", "0.s", "1..5s", "--1s", "+-1s", ".5s", "-.s", "1.5", "1.0000000000s", "0.000000001s", "-0.000000001s",
            "1.x5s", "1 s", "0x10s", "", "és"]
    return list(dict.fromkeys(out))


_SPACES = " \x85\xa0 " + "".join(map(chr, range(0x2000, 0x200B))) + "    　"


def field_mask_forms():
    out = ["", " ", "a", "fooBar", "FooBar", "fooBaR", "fOO", "foo.barBaz", "a,b", "a,,b", ",a", "a,", ",", "foo_bar",
           "1abc", "a.1b", "a1", "a.b1", "a..b", ".a", "a.", "é", "a b", "a-b", "A", "aB.cD,eF", "x​", "a,b.C1d"]
    for k, sp in enumerate(_SPACES):
        out += [sp + "fooBar" + sp, sp * 2 + "a,b" + sp]
    return list(dict.fromkeys(out))


def _escape(raw):
    """the same string token with its first ASCII letter or digit (else its first character) as a \\u escape"""
    body = raw[1:-1]
    for i, c in enumerate(body):
        if chr(c).isalnum() and c < 0x80:
            return b'"' + body[:i] + b"\\u%04x" % c + body[i + 1:] + b'"'
    if body and body[0] < 0x80:
        return b'"\\u%04x' % body[0] + body[1:] + b'"'
    return None


def forms(typ):
    """raw JSON tokens of a type, each string also with one \\u escape"""
    if typ == T.EMPTY:
        return [b"{}", b"{ }", b"[]", b"1", b'""', b"null"]
    if T.is_wrapper(typ):
        return WRAPPER_FORMS[typ[1]] + [b"null"]
    texts = {T.TS: timestamp_forms, T.DUR: duration_forms, T.FM: field_mask_forms}[typ]()
    out = []
    for t in texts:
        raw = _q(t)
        out.append(raw)
        e = _escape(raw)
        if e:
            out.append(e)
    out += [b"1", b"{}", b"[]", b"true", b"null"]
    return out


WRAPPER_FORMS = {
    "bool": [b"true", b"false", b'"true"', b"1"],
    "int32": [b"0", b"-1", b"2147483647", b"2147483648", b'"5"', b"-0", b"1e2"],
    "int64": [b"0", b'"-9223372036854775808"', b"1e2", b"9223372036854775808"],
    "uint32": [b"0", b"4294967295", b"-1"],
    "uint64": [b"0", b'"18446744073709551615"', b"1.5"],
    "float": [b"0", b"-0", b"1.5", b"3.4028235e38", b"1e39"],
    "double": [b"0", b"-0", b"1.5", b"1e308", b"-2.5e-308"],
    "string": [b'""', b'"a"', b'"\\u00e9"', b"1", b'"\\ud800"'],
    "bytes": [b'""', b'"YQ=="', b'"YQ"', b'"!"'],
}


# ---- request items ------------------------------------------------------------------------------------------------
def _gap(typ, raw):
    return typ == T.FM and b"\\" in raw


NEIGHBOURS = {T.TS: (b'"1970-01-01T00:00:00Z"', b'"2000-02-29T12:34:56.5+01:00"'), T.DUR: (b'"1s"', b'"-0.5s"'),
              T.FM: (b'"a"', b'"bC"'), T.EMPTY: (b"{}", b"{}"), T.wrapper("int64"): (b"1", b'"-2"')}
POSITIONS = {T.TS: ["f", "r", "ms", "mi", "o", "n", "root"], T.DUR: ["f", "r", "ms", "o", "n", "root"],
             T.FM: ["f", "r", "o", "n", "root"], T.EMPTY: ["f", "r", "n"]}
FIELD = {T.TS: ("ts", "r_ts", "m_ts", "m_i64_ts", "o_ts"), T.DUR: ("d", "r_d", "m_d", None, "o_d"),
         T.FM: ("fm", "r_fm", None, None, "o_fm"), T.EMPTY: ("e", "r_e", None, None, None)}
ROOT_MSG = {v: k for k, v in T.ROOTS.items()}
WRAPPER_FIELD = {"bool": "bv", "int32": "i32v", "int64": "i64v", "uint32": "u32v", "uint64": "u64v", "float": "fv",
                 "double": "dv", "string": "sv", "bytes": "byv"}


def _pl(typ, v):
    return T.payload(typ, v)


def request_item(typ, pos, raw, s):
    """(message, start offset, json, want, gap) for one value token in one position"""
    el = pos in ("r", "ms", "mi")
    v = T.value(typ, raw, element=el)
    bad = isinstance(v, str)
    if T.is_wrapper(typ):
        name = {"r": "r_i64v", "ms": "m_sv"}.get(pos, WRAPPER_FIELD[typ[1]])
    else:
        name = FIELD[typ][{"f": 0, "n": 0, "r": 1, "ms": 2, "mi": 3, "o": 4}.get(pos, 0)]
    num = NUM[name]
    if pos == "root":
        v = T.root_value(typ, raw)
        return (ROOT_MSG[typ], s, raw, v if isinstance(v, str) else b"" if v is True else _pl(typ, v), _gap(typ, raw))
    if pos == "f" or pos == "o":
        js = b'{"%s":%s}' % (name.encode(), raw)
        want = v if bad else (b"" if v is None else I.ld(num, _pl(typ, v)))
    elif pos == "n":
        js = b'{"inner":{"%s":%s}}' % (name.encode(), raw)
        want = v if bad else I.ld(NUM["inner"], b"" if v is None else I.ld(num, _pl(typ, v)))
    elif pos == "r":
        a, b = NEIGHBOURS[typ]
        js = b'{"%s":[%s,%s,%s]}' % (name.encode(), a, raw, b)
        want = v if bad else b"".join(I.ld(num, _pl(typ, x)) for x in (T.value(typ, a), v, T.value(typ, b)))
    else:
        key, kw = (b'"k"', I.ld(1, b"k")) if pos == "ms" else (b'"-7"', I.tagged(1, "int64", -7))
        js = b'{"%s":{%s:%s}}' % (name.encode(), key, raw)
        want = v if bad else I.ld(num, kw + I.ld(2, _pl(typ, v)))
    return (TM, s, js, want, _gap(typ, raw))


def request_items():
    out = []
    k = 0
    for typ in (T.TS, T.DUR, T.FM, T.EMPTY):
        pos = POSITIONS[typ]
        for j, raw in enumerate(forms(typ)):
            # each form as a singular field and in turn in the other positions
            for p in dict.fromkeys(["f", pos[1 + j % (len(pos) - 1)], pos[1 + (j + 3) % (len(pos) - 1)]]):
                out.append(request_item(typ, p, raw, (k * 7) % 16))
                k += 1
    for kind in T.WRAPPERS:
        typ = T.wrapper(kind)
        for raw in forms(typ):
            ps = ["f", "n"] + (["r"] if kind == "int64" else ["ms"] if kind == "string" else [])
            for p in ps:
                out.append(request_item(typ, p, raw, (k * 7) % 16))
                k += 1
    # null in a oneof leaves it unmarked; two members set is a oneof error, which this corpus does not need
    for raw, want in ((b'{"o_ts":null,"o_s":"x"}', I.ld(12, b"x")), (b'{"o_d":null,"o_fm":"aB"}', I.ld(11, I.ld(1, b"a_b"))),
                      (b'{"o_s":"","inner":{"o_ts":null}}', I.ld(12, b"") + I.ld(13, b""))):
        out.append((TM, (k * 7) % 16, raw, want, False))
        k += 1
    out += size_items()
    return out


# walker tiers: value records a list of n elements takes in bench.All-like items is n + 2 (root object, list); see
# tests/limits.py W1_LAST / W2_LAST / W3_LAST
W1_LAST, W2_LAST, W3_LAST = 254, 1022, 8190


def _ts_list(n, s, rng):
    vals = [rng.randrange(-62135596800, 253402300800) for _ in range(n)]
    texts = [_q(_civil(x) + ("Z" if i % 3 else ".%03dZ" % (i % 1000))) for i, x in enumerate(vals)]
    js = b'{"r_ts":[' + b",".join(texts) + b"]}"
    want = b"".join(I.ld(2, _pl(T.TS, T.value(T.TS, t))) for t in texts)
    return (TM, s, js, want, False)


def size_items(seed=0):
    """Timestamp lists around the walker tiers' value limits (and one small enough for tier 1), Timestamp maps for the
    lock-step parser's large tables.  A list at tier 3's limit is longer than the lock-step kernels' largest item (a
    Timestamp takes at least 23 bytes of text), so those go to the per-thread parser; the lists of 2 000 and 2 700 are
    the longest tier 3 can take."""
    rng = random.Random(seed + 21)
    out = []
    for i, n in enumerate((100, W1_LAST, W2_LAST - 1, W2_LAST, W2_LAST + 1, 2000, 2700, W3_LAST - 1, W3_LAST, W3_LAST + 1)):
        out.append(_ts_list(n, (i * 5) % 16, rng))
    for i, n in enumerate((40, 300, 1100)):
        for field, keyed in (("m_ts", "string"), ("m_i64_ts", "int64")):
            keys = rng.sample(range(-10 ** 12, 10 ** 12), n)
            ents = []
            for kv in keys:
                secs = rng.randrange(-62135596800, 253402300800)
                ents.append((kv, _q(_civil(secs) + "Z")))
            kj = (lambda kv: b'"k%d"' % kv) if keyed == "string" else (lambda kv: b'"%d"' % kv)
            js = b'{"%s":{' % field.encode() + b",".join(kj(kv) + b":" + t for kv, t in ents) + b"}}"
            num = NUM[field]
            if keyed == "string":
                srt = sorted(ents, key=lambda e: b"k%d" % e[0])
                want = b"".join(I.ld(num, I.ld(1, b"k%d" % kv) + I.ld(2, _pl(T.TS, T.value(T.TS, t)))) for kv, t in srt)
            else:
                srt = sorted(ents)
                want = b"".join(I.ld(num, I.tagged(1, "int64", kv) + I.ld(2, _pl(T.TS, T.value(T.TS, t)))) for kv, t in srt)
            out.append((TM, (i * 3 + len(field)) % 16, js, want, False))
    return out


def body_items(every=1):
    """(start offset, tools/call body, expected wire or status category) for the Timestamp and Duration forms as the
    singular fields of EchoTimes' arguments"""
    out = []
    i = 0
    for typ, name in ((T.TS, b"ts"), (T.DUR, b"d")):
        for raw in forms(typ):
            i += 1
            if i % every:
                continue
            v = T.value(typ, raw)
            body = (b'{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"%s","arguments":{"%s":%s}}}'
                    % (i, TOOL.encode(), name, raw))
            want = v if isinstance(v, str) else b"" if v is None else I.ld(NUM[name.decode()], _pl(typ, v))
            out.append((i % 16, body, want))
    return out


# ---- reply items --------------------------------------------------------------------------------------------------
def _reply(msg, s, w):
    return (msg, s, w, T.decode(msg, w, 0), T.decode(msg, w, 1))


def _vf(num, v):
    return I.varint(num << 3) + I.varint(v)


def seconds_values():
    """seconds (as unsigned 64-bit varint payloads) of every varint length 1..10, in and out of range"""
    M = (1 << 64) - 1
    vals = {0, 1, 127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 35) - 1, 1 << 35,
            T.MAX_TS, T.MAX_TS + 1, (1 << 42) - 1, 1 << 42, (1 << 49), (1 << 56), (1 << 63) - 1, T.MIN_TS & M,
            (T.MIN_TS - 1) & M, (-1) & M, (-86400 * 365) & M, 1 << 63, T.MAX_DUR, T.MAX_DUR + 1, (-T.MAX_DUR) & M,
            (-T.MAX_DUR - 1) & M, 1700000000}
    return sorted(vals)


NANOS = [0, 1, 999999999, 1000000000, (1 << 32) + 5, (-1) & ((1 << 64) - 1), 500000000, 123000, 120, (1 << 32) - 1,
         (-999999999) & ((1 << 64) - 1), (-1000000000) & ((1 << 64) - 1)]


def _ts_payload(sv, nv, k):
    """seconds and nanos fields in one of several shapes: plain, nanos first, a field repeated, unknown fields and a
    group in between, wrong wire types"""
    shape = k % 6
    if shape == 0:
        return _vf(1, sv) + _vf(2, nv)
    if shape == 1:
        return _vf(2, nv) + _vf(1, sv)
    if shape == 2:
        return _vf(1, 99) + _vf(2, 7) + _vf(1, sv) + _vf(2, nv)
    if shape == 3:
        return _vf(1, sv) + b"\x1b\x08\x01\x12\x00\x1c" + _vf(5, 3) + I.ld(6, b"xy") + _vf(2, nv) + b"\x3d\x01\x02\x03\x04"
    if shape == 4:
        return _vf(1, sv) + b"\x11" + b"\x00" * 8 + _vf(2, nv) + b"\x12\x00"  # seconds as fixed64, nanos as bytes: unknown
    return (_vf(1, sv) if sv else b"") + (_vf(2, nv) if nv else b"")


def reply_singular():
    out = []
    k = 0
    for sv in seconds_values():
        for nv in NANOS:
            p = _ts_payload(sv, nv, k)
            num = NUM[("ts", "o_ts", "d", "o_d", "inner", "r_ts", "m_ts", "m_i64_ts", "m_d", "r_d")[k % 10]]
            if num == NUM["inner"]:
                w = I.ld(num, I.ld(1, p))
            elif num in (NUM["m_ts"], NUM["m_d"]):
                w = I.ld(num, I.ld(1, b"k") + I.ld(2, p))
            elif num == NUM["m_i64_ts"]:
                w = I.ld(num, _vf(1, sv) + I.ld(2, p))
            else:
                w = I.ld(num, p)
            out.append(_reply(TM, k % 16, w))
            if k % 4 == 0:
                out.append(_reply("google.protobuf.Timestamp" if k % 8 else "google.protobuf.Duration", (k + 3) % 16, p))
            k += 1
    return out


def fm_paths():
    return [b"a", b"foo_bar", b"foo_bar.baz_qux", b"fooBar", b"foo__bar", b"_foo", b"foo_", b"1a", b"a..b", b"", b"a.b1",
            b"a_1", b"a_b_c", b"\xc3\xa9", b"\xff", b"foo_bAr", b"x.y.z"]


def reply_misc(seed=0):
    """FieldMask paths, wrappers, Empty, split and oneof-interleaved occurrences, Marshal errors behind wire errors"""
    rng = random.Random(seed + 31)
    out = []
    paths = fm_paths()
    for i, p in enumerate(paths):
        out.append(_reply(TM, i % 16, I.ld(NUM["fm"], I.ld(1, p))))
        out.append(_reply(TM, (i + 5) % 16, I.ld(NUM["r_fm"], I.ld(1, b"a") + I.ld(1, p)) + I.ld(NUM["o_fm"], I.ld(1, p))))
        out.append(_reply("google.protobuf.FieldMask", (i + 9) % 16, I.ld(1, p) + I.ld(1, b"b_c")))
    # wrappers and Empty: zero, nonzero, wrong wire type, unknown fields
    wvals = {"bool": [0, 1, 1 << 32], "int32": [0, 1, (1 << 32) + 3, (-1) & ((1 << 64) - 1)], "int64": [0, 1 << 63, 5],
             "uint32": [0, (1 << 32) - 1, 1 << 32], "uint64": [0, (1 << 64) - 1]}
    k = 0
    for kind, vals in wvals.items():
        for v in vals:
            num = NUM[WRAPPER_FIELD[kind]]
            out.append(_reply(TM, k % 16, I.ld(num, _vf(1, v))))
            out.append(_reply(TM, (k + 1) % 16, I.ld(num, _vf(1, v) + b"\x15\x01\x00\x00\x00" + _vf(7, 1))))
            k += 2
    for p in (b"\x0d\x00\x00\x00\x80", b"\x0d\x00\x00\xc0\x3f", b"\x09\x00\x00\x00\x00\x00\x00\xf8\x3f", b"\x08\x01", b""):
        out.append(_reply(TM, k % 16, I.ld(NUM["fv"], p) + I.ld(NUM["dv"], p)))
        k += 1
    for p in (b"", b"a", b"\xc3\xa9", b"\xff", b"\x00<&"):
        out.append(_reply(TM, k % 16, I.ld(NUM["sv"], I.ld(1, p)) + I.ld(NUM["byv"], I.ld(1, p))))
        out.append(_reply(TM, (k + 2) % 16, I.ld(NUM["m_sv"], I.ld(1, b"k") + I.ld(2, I.ld(1, p)))))
        k += 1
    out.append(_reply(TM, 3, I.ld(NUM["e"], b"") + I.ld(NUM["r_e"], b"") + I.ld(NUM["r_e"], _vf(1, 5) + b"\x0b\x0c")))
    out.append(_reply(TM, 4, I.ld(NUM["r_i64v"], b"") + I.ld(NUM["r_i64v"], _vf(1, (-2) & ((1 << 64) - 1)))))
    # split occurrences: merged field by field; a oneof sibling in between starts the member afresh
    a, b = _vf(1, 1700000000), _vf(2, 5)
    out += [_reply(TM, 5, I.ld(1, a) + I.ld(1, b)), _reply(TM, 6, I.ld(9, a) + I.ld(9, b)),
            _reply(TM, 7, I.ld(9, a) + I.ld(12, b"x") + I.ld(9, b)), _reply(TM, 8, I.ld(9, a) + I.ld(10, b) + I.ld(9, b)),
            _reply(TM, 9, I.ld(10, _vf(1, 3)) + I.ld(9, a) + I.ld(10, _vf(2, (-1) & ((1 << 64) - 1)))),
            _reply(TM, 10, I.ld(13, I.ld(1, a)) + I.ld(13, I.ld(1, b))), _reply(TM, 11, I.ld(8, I.ld(1, b"a")) + I.ld(8, I.ld(1, b"b"))),
            _reply(TM, 12, I.ld(3, I.ld(1, b"k") + I.ld(2, a) + I.ld(2, b))),  # two values inside one entry merge
            _reply(TM, 13, I.ld(3, I.ld(1, b"k") + I.ld(2, a)) + I.ld(3, I.ld(1, b"k") + I.ld(2, b))),  # replaced
            _reply(TM, 14, I.ld(3, I.ld(2, a))), _reply(TM, 15, I.ld(4, I.ld(2, b))), _reply(TM, 0, I.ld(3, I.ld(1, b"k"))),
            _reply(TM, 1, I.ld(11, I.ld(1, b"a")) + I.ld(9, a) + I.ld(11, I.ld(1, b"bC")))]
    # Marshal-time errors followed by a wire error later in the item, and alone
    errs = [I.ld(1, _vf(1, T.MAX_TS + 1)), I.ld(6, _vf(1, 1) + _vf(2, (-1) & ((1 << 64) - 1))), I.ld(8, I.ld(1, b"fooBar")),
            I.ld(1, _vf(2, 1000000000)), I.ld(5, I.ld(1, b"k") + I.ld(2, _vf(1, T.MAX_DUR + 1))), I.ld(13, I.ld(8, I.ld(1, b"1a")))]
    tails = [b"\x08", b"\x0f", I.ld(13, b"\x0b"), b"\xfa\x01\x05ab", I.ld(12, b"\xff")]
    for i, e in enumerate(errs):
        out.append(_reply(TM, i % 16, e))
        for j, t in enumerate(tails):
            out.append(_reply(TM, (i + j) % 16, e + I.ld(12, b"pad" * (i + j)) + t))
    # random payload damage around Timestamps
    for i in range(40):
        p = _ts_payload(rng.choice(seconds_values()), rng.choice(NANOS), i)
        cut = rng.randrange(len(p))
        out.append(_reply(TM, i % 16, I.ld(1, p[:cut]) + I.ld(2, p)))
        out.append(_reply(TM, (i + 7) % 16, I.ld(2, p) + bytes([0x0a, len(p) + 1]) + p))  # length past the end
    return out


EDGES = (8, 32, 64, 96, 4096)


def reply_edges():
    """a Timestamp payload whose field header starts at rebased bytes E - 11 .. E + 2 of each edge, behind an o_s
    string of the right length"""
    out = []
    k = 0
    svals = seconds_values()
    for e in EDGES:
        for d in range(-11, 3):
            sv, nv = svals[k % len(svals)], NANOS[k % len(NANOS)]
            body = I.ld((1, 2, 3)[k % 3], _ts_payload(sv, nv, k) if k % 3 != 2 else I.ld(1, b"k") + I.ld(2, _vf(1, sv) + _vf(2, nv)))
            s = k % 16
            room = e + d - s
            pad = next((I.ld(12, b"p" * n) for n in (room - 2, room - 3) if n >= 0 and len(I.ld(12, b"p" * n)) == room), None)
            k += 1
            if pad is None:
                if room == 0:
                    out.append(_reply(TM, s, body))
                continue
            out.append(_reply(TM, s, pad + body))
    return out


def reply_lists(seed=0):
    """Timestamp lists of 200..250 entries (the first lock-step reply tier holds 224) and of 1 000, a Timestamp map of
    300 entries out of key order with repeated keys"""
    rng = random.Random(seed + 41)
    out = []
    pool = [(sv, nv) for sv in seconds_values() for nv in NANOS[:4]]
    for i, n in enumerate(list(range(200, 251, 5)) + [221, 222, 223, 224, 225, 1000, 1500]):
        items = [rng.choice(pool) for _ in range(n)]
        ok = [(sv, nv) for sv, nv in items if sv <= T.MAX_TS and nv < 10 ** 9 or i % 3 == 0]
        out.append(_reply(TM, i % 16, b"".join(I.ld(2, _vf(1, sv) + _vf(2, nv)) for sv, nv in ok)))
    for n in (5, 40, 300):
        ents = b""
        for j in range(n):
            kv = rng.randrange(n // 2 + 1)
            sv = rng.randrange(0, T.MAX_TS)
            ents += I.ld(4, _vf(1, (kv * 7919 - 1000) & ((1 << 64) - 1)) + I.ld(2, _vf(1, sv) + _vf(2, j)))
            ents += I.ld(3, I.ld(1, b"k%d" % kv) + I.ld(2, _vf(1, sv)))
        out.append(_reply(TM, n % 16, ents))
    return out


def reply_items(seed=0):
    return reply_singular() + reply_misc(seed) + reply_edges() + reply_lists(seed)
