"""Seeded corpus of string and bytes text for the string tests: byte events (valid UTF-8 at the ends of each sequence
length, invalid sequences, escapes, backslash runs, control bytes) placed at every offset 0..33 of a string and on both
sides of the 16-byte chunk, 32-byte round, 512-byte tokenizer round and 2048 / 4096-byte tile edges, in every string
container (singular field, list element, map key, value behind an escaped name), in items sized for each tier; base64
text at every length mod 3 and mod 4, short, long and written in place.  Expected values come from strref alone.

Positions are rebased: the kernels rebase an item to the 16-byte aligned address at or below its start, so every item
carries the start offset s (mod 16) it is built for, and an event meant for rebased byte R sits at item byte R - s.
"""
import random

import strref as S

A = "bench.All"
F_STRING, F_BYTES, R_STRING, R_BYTES, M_STR_INT32, CUSTOM, Z_LAST = 14, 15, 34, 35, 41, 90, 100

# ---- events -----------------------------------------------------------------------------------------------------
VALID = [chr(c).encode() for c in (0x80, 0x7FF, 0x800, 0xD7FF, 0xE000, 0xFFFD, 0xFFFF, 0x10000, 0x10FFFF)] + [b"\x7f"]
INVALID = [b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf0\x80\x80\x80",
           b"\xf0\x8f\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf4\xbf\xbf\xbf", b"\xf5\x80\x80\x80", b"\xf8\x88\x80\x80", b"\xff",
           b"\x80", b"\xbf", b"\xc3\xc3\xa9", b"\xe2\xe2\x82\xac", b"\xf0\xf0\x9f\x98\x80"]
ESCAPES = [b'\\"', b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t", b"\\u0041", b"\\u007F", b"\\u0080", b"\\u07ff",
           b"\\u0800", b"\\uFFFF", b"\\u0000", b"\\u001f", b"\\ud800\\udc00", b"\\uDBFF\\uDFFF", b"\\ud83d\\ude00",
           b"\\" * 17 + b"/", b"\\" * 18, b"\\" * 33 + b'"', b"\\" * 34, b"\\" * 65 + b"n", b"\\" * 66]
BAD_ESCAPES = [b"\\ud800x", b"\\udc00", b"\\ud83d\\u0041", b"\\ud83d\\ud83d", b"\\udbff\\ue000", b"\\u00g0", b"\\x",
               b"\\U0041", b"\\'", b"\\" * 17 + b"q"]
CONTROL = [b"\x00", b"\x01", b"\x1f", b"\t", b"\n"]
# events that end a string: a sequence cut by the closing quote, a \u cut by it
AT_END = [b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"\\u12", b"\\ud83d"]
# sequences cut in front of a backslash
BEFORE_BS = [b"\xe2\x82\\n", b"\xf0\x9f\x98\\\\", b"\xc3\\u00e9"]
REQ_EVENTS = VALID + INVALID + ESCAPES + BAD_ESCAPES + CONTROL + BEFORE_BS
# reply side: the bytes of the wire string itself
REP_EVENTS = VALID + INVALID + [b'"', b"\\", b"\x00", b"\x01", b"\x1f", b"\t", b"\n", b"\x08", b"\x0c", b"\r", b"<>&",
                                "\u2028".encode(), "\u2029".encode(), b"\xe2\x80", b"\xf0\x9f\x98"]

# rebased edges: 16-byte chunks / 32-byte rounds are reached by the offset sweep, the rest here
REQ_EDGES = (512, 1024, 2048, 4096)
REP_EDGES = (64, 96, 128, 512)
# wire bytes in front of the string of each reply container (reply_item), for its short strings
REP_HEAD = {"f": 2, "r": 7, "m": 13, "z": 6}


# ---- wire ---------------------------------------------------------------------------------------------------------
def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def ld(num, payload):
    return varint(num << 3 | 2) + varint(len(payload)) + payload


def _entry(k, v):
    return ld(M_STR_INT32, ld(1, k) + varint(2 << 3) + varint(v))


# ---- request items ------------------------------------------------------------------------------------------------
# containers: (json before the string, json after it, function of the decoded string -> wire of the item)
REQ_CONTAINERS = {
    "f": (b'{"f_string":"', b'"', lambda v: ld(F_STRING, v) if v else b""),
    "r": (b'{"r_string":["a","', b'","b"]', lambda v: ld(R_STRING, b"a") + ld(R_STRING, v) + ld(R_STRING, b"b")),
    "m": (b'{"m_str_int32":{"m":2,"', b'":1}', lambda v: b"".join(_entry(k, x) for k, x in sorted([(b"m", 2), (v, 1)]))),
    "k": (b'{"f_str\\u0069ng":"', b'"', lambda v: ld(F_STRING, v) if v else b""),
}


def request_item(cont, s, content, filler=0, elems=0):
    """(message, start offset, json, expected wire or status category) for `content` (raw JSON string body) in
    container `cont`; `filler` bytes of a plain "custom" value after it (size routing), `elems` extra plain list
    elements in front of an "r" string (walker tiers by value count; eight letters each, so that the list is not too
    dense for the walker's IR region)"""
    head, tail, wire = REQ_CONTAINERS[cont]
    if cont == "r" and elems:
        head = b'{"r_string":[' + b'"eeeeeeee",' * elems + b'"a","'
        wire0 = wire
        wire = lambda v: ld(R_STRING, b"eeeeeeee") * elems + wire0(v)
    js = head + content + tail
    v = S.parse_string(content)
    if cont == "m" and v == b"m":
        v = S.SYNTAX  # never built: a duplicate key
    if filler:
        js += b',"custom":"' + b"r" * filler + b'"'
    js += b"}"
    if isinstance(v, str):
        return (A, s, js, v)
    want = wire(v) + (ld(CUSTOM, b"r" * filler) if filler else b"")
    return (A, s, js, want)


def _head_len(cont, elems=0):
    return len(REQ_CONTAINERS[cont][0]) + (11 * elems if cont == "r" and elems else 0)


def start_offset(k, off, head):
    """start offset of the k-th item of a sweep whose event sits at string offset `off` behind `head` bytes of the
    item: the event's rebased byte is (k // 40 + 9 * off) mod 16, so 16 consecutive offsets of an event reach every
    byte position of a 16-byte chunk, and the start offset still takes every value over the corpus"""
    return (k // 40 + 8 * off - head) % 16


def request_items(seed=0):
    """every request event at string offsets 0..33 and at each rebased edge (its first byte two bytes in front of the
    edge up to on it), in the four containers in turn, short and long strings, with and without a filler that
    sends the item to the lock-step tiers under size routing"""
    rng = random.Random(seed + 1)
    out = []
    conts = "frmk"
    k = 0
    for ev in REQ_EVENTS:
        for off in range(34):
            cont = conts[k % 4]
            s = start_offset(k, off, _head_len(cont))
            tail = (3, 40, 150, 600)[(k // 4) % 4]
            content = b"a" * off + ev + b"z" * tail
            out.append(request_item(cont, s, content, filler=1100 if k % 3 == 0 else 0))
            k += 1
        for edge in REQ_EDGES:
            for d in (-3, -2, -1, 0):
                cont = conts[k % 4]
                s = k % 16
                elems = 0
                if cont == "r":
                    elems = (0, 300, 1100)[(k // 4) % 3]
                off = edge + d - s - _head_len(cont, elems)
                content = b"a" * off + ev + b"z" * rng.randrange(2, 60)
                out.append(request_item(cont, s, content, elems=elems))
                k += 1
    for ev in AT_END:
        for off in list(range(34)) + [e + d for e in REQ_EDGES for d in (-4, -3, -2, -1, 0)]:
            cont = conts[k % 4]
            s = k % 16
            n = off - s - _head_len(cont) if off >= 100 else off
            out.append(request_item(cont, s, b"a" * n + ev))
            k += 1
    out += many_strings_items()
    return out


def many_strings_items():
    """request items of 40 to 80 strings in one list: more escaped strings and more long strings than one warp's
    hand-off lists take, with one bad event among them or none"""
    out = []
    for n, long_len, bad in ((70, 0, None), (40, 140, None), (80, 140, None), (70, 0, b"\xed\xa0\x80"), (40, 140, b"\\ud800x"),
                             (70, 130, b"\x01"), (66, 0, b"\\ud83d\\ude00"), (34, 200, b"\xf4\x90\x80\x80")):
        vals = []
        for i in range(n):
            body = (b"w%d\\n" % i) + b"q" * long_len
            if bad is not None and i == n // 2:
                body = b"x" * i + bad + body
            vals.append(body)
        js = b'{"r_string":["' + b'","'.join(vals) + b'"]}'
        dec = [S.parse_string(v) for v in vals]
        bad_st = next((d for d in dec if isinstance(d, str)), None)
        out.append((A, n % 16, js, bad_st if bad_st else b"".join(ld(R_STRING, d) for d in dec)))
    return out


# ---- request bytes ------------------------------------------------------------------------------------------------
def _b64_texts(rng):
    """decoded JSON strings of a bytes field: both alphabets, padded and not, with \\r / \\n, and damaged"""
    out = []
    lens = list(range(0, 41)) + [94, 95, 96, 97, 98, 126, 127, 128, 129, 130, 3000]
    for n in lens:
        data = bytes(rng.randrange(256) for _ in range(n))
        std = S.b64_format(data)
        url = std.replace(b"+", b"-").replace(b"/", b"_")
        out += [std, std.rstrip(b"="), url, url.rstrip(b"=")]
        if len(std) > 4:
            i = rng.randrange(1, len(std) - 1)
            out.append(std[:i] + b"\n" + std[i:])
            out.append(std.rstrip(b"=")[:i] + b"\r\n" + std.rstrip(b"=")[i:])
            out.append(std[:i] + b"=" + std[i + 1:])            # misplaced '='
            out.append(std[:i] + b" " + std[i:])                 # a space
            out.append(std[:i] + b"-" + std[i + 1:] + b"+")      # mixed alphabets
            out.append(std + b"\n")
            out.append(std[:-1] if std.endswith(b"=") else std + b"=")
    out += [b"QR==", b"QR=", b"QR", b"Q", b"Q===", b"QRS=", b"QRS", b"====", b"=", b"Q=\n=", b"QR=\n=", b"QR\n==", b"YQ==YQ==",
            b"\n", b"\r\n\r\n", b"a\nb\nc\nd", b"ab\ncd=", b"-_-_", b"+/+/", b"-/+_", b"YQ==\n", b"YQ=\n="]
    return out


def _json_escape(b):
    return b.replace(b"\\", b"\\\\").replace(b"\n", b"\\n").replace(b"\r", b"\\r")


def request_bytes_items(seed=0):
    rng = random.Random(seed + 2)
    out = []
    for i, t in enumerate(_b64_texts(rng)):
        v = S.b64_parse(t)
        js = b'{"f_bytes":"' + _json_escape(t) + b'"}'
        out.append((A, i % 16, js, v if isinstance(v, str) else (ld(F_BYTES, v) if v else b"")))
        if i % 3 == 0:
            js = b'{"r_bytes":["YQ==","' + _json_escape(t) + b'"]}'
            out.append((A, (i + 7) % 16, js, v if isinstance(v, str) else ld(R_BYTES, b"a") + ld(R_BYTES, v)))
    return out


# ---- tools/call bodies --------------------------------------------------------------------------------------------
def body_items(req_items, every=3):
    """(start offset, body, expected wire or SYNTAX, identity) for every `every`-th f_string request item, its
    arguments inside a bench_benchservice_echoall call"""
    out = []
    head = REQ_CONTAINERS["f"][0]
    for i, (name, s, js, want) in enumerate(req_items):
        if i % every or not js.startswith(head) or b'"custom"' in js:
            continue
        content = js[len(head):-2]
        v, ident = S.body_value(content)
        body = b'{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"bench_benchservice_echoall","arguments":%s}}' % (i, js)
        out.append((s, body, v if isinstance(v, str) else (ld(F_STRING, v) if v else b""), ident))
    return out


# ---- reply items --------------------------------------------------------------------------------------------------
def _jstr(b):
    return S.format_string(b)


def reply_item(cont, s, val, filler=0, flags=0):
    """(message, start offset, wire, expected text or INVALID_UTF8) for the string bytes `val` in container `cont`:
    f = fString, r = an rString element, m = an mStrInt32 key, z = zLast written in front of fString on the wire
    (fields out of order: the per-thread slow walk)"""
    sep = b", " if flags & 1 else b","
    t = _jstr(val)
    if t == S.INVALID_UTF8:
        t = None
    if cont == "f":
        wire = ld(F_STRING, val)
        parts = [b'"fString":' + t] if t and val else []
    elif cont == "r":
        wire = ld(R_STRING, b"a") + ld(R_STRING, val) + ld(R_STRING, b"b")
        parts = [b'"rString":[' + sep.join([b'"a"', t, b'"b"']) + b"]"] if t else []
    elif cont == "m":
        ent = sorted([(b"m", 2), (val, 1)]) if val != b"m" else [(b"m", 1)]
        wire = _entry(b"m", 2) + _entry(val, 1)
        parts = [b'"mStrInt32":{' + sep.join(_jstr(k) + b":" + b"%d" % x for k, x in ent) + b"}"] if t else []
    else:
        wire = ld(Z_LAST, b"q") + ld(F_STRING, val)
        parts = ([b'"fString":' + t] if val else []) + [b'"zLast":"q"'] if t else []
    if filler:
        wire += ld(CUSTOM, b"r" * filler)
        parts.insert(len(parts) - (cont == "z"), b'"CustomJSON":"' + b"r" * filler + b'"')
    if t is None:
        return (A, s, wire, S.INVALID_UTF8)
    return (A, s, wire, b"{" + sep.join(parts) + b"}")


def reply_specs(seed=0):
    """(container, start offset, string bytes, filler) for every reply event at string offsets 0..33 and around the
    32-byte round edges, in short (< 96 bytes), long and in-place (text past 6144 bytes) strings"""
    rng = random.Random(seed + 3)
    out = []
    conts = "frmz"
    k = 0
    for ev in REP_EVENTS:
        for off in list(range(34)) + [e + d for e in REP_EDGES for d in (-3, -2, -1, 0)]:
            cont = conts[k % 4]
            tail = (2, 30, 100, 300)[(k // 4) % 4]
            if k % 29 == 0:
                tail = 6300
            out.append((cont, start_offset(k, off, REP_HEAD[cont]), b"a" * off + ev + b"z" * tail, 700 if k % 3 == 0 else 0))
            k += 1
    # a string ending on a cut sequence, and strings of only events
    for ev in (b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"\xed\xa0"):
        for off in range(0, 70):
            out.append((conts[k % 4], k % 16, b"a" * off + ev, 0))
            k += 1
    for i in range(60):
        n = rng.choice([1, 31, 32, 33, 95, 96, 97, 200, 6200])
        pool = VALID + [b'"', b"\\", b"\x01", b"\n", b"<", "\u2028".encode()]
        val = b"".join(rng.choice(pool) for _ in range(n))
        out.append((conts[i % 4], i % 16, val, 0))
    return out


def reply_many_strings():
    """items of more dirty strings (escapes) than the warp sizes and more long strings than its hand-off list holds"""
    out = []
    for n, long_len, bad in ((70, 0, None), (40, 120, None), (80, 100, None), (70, 0, b"\xff"), (40, 120, b"\xed\xa0\x80"),
                             (66, 97, b"\xe2\x80\xa8"), (34, 300, b"\xf4\x90\x80\x80")):
        vals = [(b"w%d\n" % i) + b"q" * long_len for i in range(n)]
        if bad is not None:
            vals[n // 2] = b"x" * (n // 2) + bad + vals[n // 2]
        wire = b"".join(ld(R_STRING, v) for v in vals)
        ts = [_jstr(v) for v in vals]
        if S.INVALID_UTF8 in ts:
            out.append((A, n % 16, wire, S.INVALID_UTF8, S.INVALID_UTF8))
        else:
            out.append((A, n % 16, wire, b'{"rString":[' + b",".join(ts) + b"]}", b'{"rString":[' + b", ".join(ts) + b"]}"))
    return out


def reply_big_tables():
    """items of more entries than the first lock-step reply tier's table (GGR_COOP_TAB_ENTRIES = 320): 400 or 1000
    short list elements in front of the string with the event, at a few offsets each"""
    out = []
    k = 0
    for ev in REP_EVENTS:
        for off in (0, 15, 31, 40):
            n = 400 if k % 3 else 1000
            vals = [b"e"] * n + [b"a" * off + ev + b"z" * (k % 7)]
            wire = b"".join(ld(R_STRING, v) for v in vals)
            ts = [_jstr(v) for v in vals]
            if S.INVALID_UTF8 in ts:
                out.append((A, k % 16, wire, S.INVALID_UTF8, S.INVALID_UTF8))
            else:
                out.append((A, k % 16, wire, b'{"rString":[' + b",".join(ts) + b"]}", b'{"rString":[' + b", ".join(ts) + b"]}"))
            k += 1
    return out


def reply_bytes_items(seed=0):
    """(message, start offset, wire, text, text with comma-space) for bytes fields of every length 0..100, 3k +- 1
    around 96 and 128, and long enough to be written in place"""
    rng = random.Random(seed + 4)
    out = []
    lens = list(range(0, 101)) + [125, 126, 127, 128, 129, 130, 131, 8190, 9000, 20000]
    for i, n in enumerate(lens):
        data = bytes(rng.randrange(256) for _ in range(n))
        b64 = S.b64_format(data)
        w = ld(F_BYTES, data)
        t = b'{"fBytes":"' + b64 + b'"}' if n else b"{}"
        out.append((A, i % 16, w, t, t))
        w = ld(R_BYTES, data) + ld(R_BYTES, b"\x00") + ld(F_STRING, b"s")
        t = b'{"fString":"s","rBytes":["%s","AA=="]}' % b64, b'{"fString":"s", "rBytes":["%s", "AA=="]}' % b64
        out.append((A, (i + 5) % 16, w) + t)
        # the same in field order: the lock-step reply tiers take it (they leave fields out of order to the slow walk)
        out.append((A, (i + 9) % 16, ld(F_STRING, b"s") + ld(R_BYTES, data) + ld(R_BYTES, b"\x00")) + t)
    return out


def reply_items(seed=0):
    """(message, start offset, wire, expected text flags 0, expected text flags 1); INVALID_UTF8 for both when the
    item must fail"""
    out = []
    for cont, s, val, filler in reply_specs(seed):
        m, s, w, t0 = reply_item(cont, s, val, filler, 0)
        t1 = reply_item(cont, s, val, filler, 1)[3]
        out.append((m, s, w, t0, t1))
    return out + reply_many_strings() + reply_big_tables() + reply_bytes_items(seed)


def wrap_texts(seed=0):
    """protojson texts for the result wrapper: < > & and U+2028 / U+2029 (three bytes that can straddle lanes) at
    every offset 0..70, between plain and escaped text"""
    rng = random.Random(seed + 5)
    out = []
    for ev in ("\u2028", "\u2029", "<", ">", "&", "\u2028\u2029", "<\u2028&", "\u00e9", "\U0001F600", '\\"', "\\u0001"):
        for off in range(71):
            out.append(('{"fString":"' + "a" * off + ev + "z" * rng.randrange(0, 40) + '"}').encode())
    return out
