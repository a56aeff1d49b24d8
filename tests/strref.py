"""Exact reference for string and bytes text, as protojson and encoding/json write and read it.

parse_string(body)  - the bytes between the quotes of a JSON string token -> decoded bytes, or SYNTAX / INVALID_UTF8.
format_string(b)    - a string field's bytes -> its protojson text, or INVALID_UTF8.
html_string(t)      - a protojson text -> the JSON string encoding/json writes for it in a result body.
b64_format(b)       - a bytes field -> its protojson text (without the quotes).
b64_parse(s)        - the decoded JSON string of a bytes field -> the bytes, or INVALID_VALUE.
body_value(body)    - the bytes of a string inside `arguments` as the field receives it after encoding/json's round
                      trip, and whether the device may refuse the body instead.

Plain Python (the strict `utf-8` codec and integer arithmetic): independent of the oracle and of the device code.

Status categories are the project's (`GGR_ST_*`), not Go's error texts: protojson's tokenizer reports a raw byte that is
not UTF-8 as a syntax error ("invalid UTF-8 in string"); the project reports it as INVALID_UTF8, the status
proto.Unmarshal's check of the same bytes gives on the reply side, so that a client can tell bad text from bad JSON.
Escapes, raw control bytes and unterminated strings are SYNTAX; a bytes field whose text is not base64 is INVALID_VALUE.
"""
import base64

SYNTAX, INVALID_VALUE, INVALID_UTF8 = "syntax", "invalid_value", "invalid_utf8"
STATUS = {SYNTAX: 1, INVALID_VALUE: 3, INVALID_UTF8: 5}  # GGR_ST_* of each category

_SHORT = {ord('"'): b'"', ord("\\"): b"\\", ord("/"): b"/", ord("b"): b"\b", ord("f"): b"\f", ord("n"): b"\n",
          ord("r"): b"\r", ord("t"): b"\t"}
_HEX = frozenset(b"0123456789abcdefABCDEF")


def utf8_len(b, i):
    """length of the valid UTF-8 sequence at b[i], or 0 (utf8.DecodeRune's RuneError with size 1)"""
    c = b[i]
    n = 1 if c < 0x80 else 2 if 0xC2 <= c <= 0xDF else 3 if 0xE0 <= c <= 0xEF else 4 if 0xF0 <= c <= 0xF4 else 0
    if n == 0:
        return 0
    try:
        b[i:i + n].decode("utf-8")
    except UnicodeDecodeError:
        return 0
    return n if i + n <= len(b) else 0


def _hex4(b, i):
    s = b[i:i + 4]
    return int(s, 16) if len(s) == 4 and all(c in _HEX for c in s) else None


def parse_string(body):
    """protobuf-go internal/encoding/json decode_string.go parseString on '"' + body + '"': the first problem from
    the left decides.  Raw bytes: not UTF-8 -> INVALID_UTF8 (see the module docstring), below 0x20 -> SYNTAX.
    Escapes: the eight short ones, and \\uXXXX with four hex digits of either case (strconv.ParseUint(s, 16, 16));
    a \\u in D800-DFFF must be a high surrogate directly followed by \\u and a low one (utf16.DecodeRune gives U+FFFD
    for anything else, which parseString refuses); any other escape, or one cut by the end of the token, is SYNTAX.
    `body` must not hold an unescaped '"' (it would end the token)."""
    b = bytes(body)
    out = bytearray()
    i, n = 0, len(b)
    while i < n:
        c = b[i]
        if c == 0x5C:
            if i + 1 >= n:
                return SYNTAX
            e = b[i + 1]
            if e in _SHORT:
                out += _SHORT[e]
                i += 2
                continue
            if e != ord("u"):
                return SYNTAX
            r = _hex4(b, i + 2)
            if r is None:
                return SYNTAX
            i += 6
            if 0xD800 <= r <= 0xDFFF:
                r2 = _hex4(b, i + 2) if b[i:i + 2] == b"\\u" else None
                if r >= 0xDC00 or r2 is None or not 0xDC00 <= r2 <= 0xDFFF:
                    return SYNTAX
                r = 0x10000 + ((r - 0xD800) << 10) + (r2 - 0xDC00)
                i += 6
            out += chr(r).encode("utf-8")
            continue
        k = utf8_len(b, i)
        if k == 0:
            return INVALID_UTF8
        if c < 0x20:
            return SYNTAX
        out += b[i:i + k]
        i += k
    return bytes(out)


def format_string(b):
    """protobuf-go internal/encoding/json encode.go appendString: '"', '\\\\', \\b \\f \\n \\r \\t, other bytes below 0x20 as
    \\u00xx in lower-case hex; 0x7F, U+2028 / U+2029 and all other valid UTF-8 as they are.  INVALID_UTF8 if `b` is
    not UTF-8 (proto.Unmarshal refuses such a proto3 string before protojson sees it)."""
    try:
        t = bytes(b).decode("utf-8")
    except UnicodeDecodeError:
        return INVALID_UTF8
    out = bytearray(b'"')
    for ch in t:
        c = ord(ch)
        if ch in '"\\':
            out += b"\\" + ch.encode()
        elif c < 0x20:
            out += {8: b"\\b", 12: b"\\f", 10: b"\\n", 13: b"\\r", 9: b"\\t"}.get(c) or b"\\u%04x" % c
        else:
            out += ch.encode("utf-8")
    return bytes(out + b'"')


def html_string(t):
    """encoding/json encode.go appendString with escapeHTML = true, for valid UTF-8: '"', '\\\\', the five short
    escapes, other bytes below 0x20 and < > & as \\u00xx, U+2028 / U+2029 as \\u2028 / \\u2029, all else as it is"""
    out = bytearray(b'"')
    for ch in t.decode("utf-8"):
        c = ord(ch)
        if ch in '"\\':
            out += b"\\" + ch.encode()
        elif ch in "\n\r\t\b\f":
            out += {"\n": b"\\n", "\r": b"\\r", "\t": b"\\t", "\b": b"\\b", "\f": b"\\f"}[ch]
        elif c < 0x20 or ch in "<>&" or c in (0x2028, 0x2029):
            out += b"\\u%04x" % c
        else:
            out += ch.encode("utf-8")
    return bytes(out + b'"')


def b64_format(b):
    """protojson encoder.go marshalSingular for bytes: base64.StdEncoding.EncodeToString (padded)"""
    return base64.b64encode(bytes(b))


_STD = {c: i for i, c in enumerate(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/")}
_URL = {c: i for i, c in enumerate(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789-_")}


def b64_parse(s):
    """protojson decoder.go unmarshalBytes on the decoded string `s`: base64.URLEncoding if `s` holds '-' or '_', else
    StdEncoding; WithPadding(NoPadding) if len(s) % 4 != 0, that length counting the \\r and \\n the decoder then skips.
    Go's decodeQuantum restated: \\r and \\n are skipped anywhere; '=' is an error before the third symbol of a quantum,
    and (padded) must be followed by a second '=' after the third symbol and by nothing but \\r / \\n after the
    padding; with NoPadding '=' is just a byte outside the alphabet; a quantum of one symbol is an error, and a cut
    quantum is an error when padding is expected.  Nonzero trailing bits are accepted (the decoder is not Strict)."""
    s = bytes(s)
    dmap = _URL if (b"-" in s or b"_" in s) else _STD
    padded = len(s) % 4 == 0
    out = bytearray()
    si, n = 0, len(s)
    while True:
        dbuf, j, end = [0, 0, 0, 0], 0, False
        while j < 4:
            if si == n:
                if j == 0:
                    return bytes(out)
                if j == 1 or padded:
                    return INVALID_VALUE
                end = True
                break
            c = s[si]
            si += 1
            if c in dmap:
                dbuf[j] = dmap[c]
                j += 1
                continue
            if c in b"\r\n":
                continue
            if c != ord("=") or not padded or j < 2:
                return INVALID_VALUE
            if j == 2:
                while si < n and s[si] in b"\r\n":
                    si += 1
                if si == n or s[si] != ord("="):
                    return INVALID_VALUE
                si += 1
            while si < n and s[si] in b"\r\n":
                si += 1
            if si < n:
                return INVALID_VALUE
            end = True
            break
        v = dbuf[0] << 18 | dbuf[1] << 12 | dbuf[2] << 6 | dbuf[3]
        out += bytes([v >> 16 & 255, v >> 8 & 255, v & 255])[: j - 1]
        if end:
            return bytes(out)


def go_replace_invalid(b):
    """encoding/json decode.go unquote on raw bytes: each byte where utf8.DecodeRune fails becomes U+FFFD"""
    out = bytearray()
    i = 0
    while i < len(b):
        k = utf8_len(b, i)
        if k == 0:
            out += "�".encode()
            i += 1
        else:
            out += b[i:i + k]
            i += k
    return bytes(out)


def body_value(body):
    """a string inside `arguments` of a tools/call body: the reference decodes the body with encoding/json into
    interface{}, re-marshals `arguments` with json.Marshal and hands that text to protojson.  -> (value, identity):
    `value` is the field's bytes after that round trip, or SYNTAX if encoding/json refuses the body; `identity` is
    False when the round trip changes the value (a raw byte that is not UTF-8, or a surrogate escape that is not a
    well-formed pair, each becomes U+FFFD); the device may answer GGR_ST_UNSUPPORTED for those (DESIGN §9), never
    other bytes."""
    b = bytes(body)
    direct = parse_string(b)
    if direct == SYNTAX:
        # encoding/json refuses the same escapes and control bytes, but it accepts any \\uXXXX, surrogates included
        lenient = _parse_lenient(b)
        return (SYNTAX, True) if lenient is None else (lenient, False)
    if direct == INVALID_UTF8:
        lenient = _parse_lenient(b)
        return (SYNTAX, True) if lenient is None else (lenient, False)
    return direct, True


def _parse_lenient(b):
    """encoding/json unquote: like parse_string, but a byte that is not UTF-8 and a surrogate escape that does not
    pair become U+FFFD; None where encoding/json's scanner refuses the token (bad escape, control byte)"""
    out = bytearray()
    i, n = 0, len(b)
    while i < n:
        c = b[i]
        if c == 0x5C:
            if i + 1 >= n:
                return None
            e = b[i + 1]
            if e in _SHORT:
                out += _SHORT[e]
                i += 2
                continue
            if e != ord("u"):
                return None
            r = _hex4(b, i + 2)
            if r is None:
                return None
            i += 6
            if 0xD800 <= r <= 0xDFFF:
                r2 = _hex4(b, i + 2) if b[i:i + 2] == b"\\u" else None
                if r < 0xDC00 and r2 is not None and 0xDC00 <= r2 <= 0xDFFF:
                    r = 0x10000 + ((r - 0xD800) << 10) + (r2 - 0xDC00)
                    i += 6
                else:
                    r = 0xFFFD
            out += chr(r).encode("utf-8")
            continue
        if c < 0x20:
            return None
        k = utf8_len(b, i)
        if k == 0:
            out += "�".encode()
            i += 1
        else:
            out += b[i:i + k]
            i += k
    return bytes(out)
