"""Boundary corpus of the lock-step kernels: items built on both sides of every fixed capacity of the reply tiers
(ggr_coop.cuh) and the request walker / emitter (ggr_walk.cuh, ggr_coop_enc.cuh).

Every item is `Item(limit_id, side, message, data, damaged)`: `limit_id` names the capacity (R1..R9 reply side, W0..W10
request side), `side` is "below", "at" (the last item the capacity takes) or "above" (the first it leaves, and beyond).
Reply items are wire bytes (python-protobuf, deterministic serialisation), request items are JSON arguments written
directly where the shape needs control over bytes.  Damaged items (truncated at the boundary, or with one string's UTF-8
broken there) carry damaged=True.  The counts below were pinned on the host simulation, not worked out on paper: the
kernels count value records, table entries or bytes in ways that depend on the item (entry 0 is the root, packed runs are
one entry, the walker counts the root and every container).  Expected results come from the oracle.
"""
import random
from collections import namedtuple

import pbgen

Item = namedtuple("Item", "limit_id side message data damaged")
NODE = "com.example.complex.Node"
A = "bench.All"
PNR = "com.example.complex.ProcessNodeRequest"

# ---- reply side: capacities and the counts pinned at them ------------------------------------------------------
COOP_ENTRIES = 224          # GGR_COOP_ENTRIES: first tier's table
R1_LAST = 223               # empty children of a Node the first tier still takes (+ the root entry = 224)
COOP_BIG_ENTRIES = 4096     # GGR_COOP_BIG_ENTRIES: second tier's table
R2_LAST = 4095
COOP_MAX_WIRE = 4096        # GGR_COOP_MAX_WIRE, tested on the item's end (start offset mod 16 included)
DIRTY_MAX = 64              # GGR_COOP_DIRTY_MAX: strings sized by the whole warp
LONG_MAX = 32               # GGR_COOP_LONG_MAX: hand-off list of whole-warp copies
COOP_LONG = 96              # GGR_COOP_LONG: plain strings / bytes of at least this many bytes go to the list
STAGE_BUF = 6144            # GGR_COOP_STAGE_BUF: text bytes assembled in shared memory
R8_LAST = 22                # nesting depth (Node.children) the lock-step reply tiers still take
DEC_MAX_DEPTH = 32          # GGR_DEC_MAX_DEPTH frames of the per-thread kernels
R8_PT_LAST = 31             # nesting depth (Node.children) the per-thread kernels take; GGR_ST_DEPTH beyond
POOL_MAX = 4 << 20          # second tier's entry pool: in_bytes / 2 + 4096 entries per call, at most 4 M

# ---- request side ----------------------------------------------------------------------------------------------
W1_LAST = 254               # six-digit elements of one list the walker's first tier takes (256 value records)
W2_LAST = 1022              # ... the second tier (1024 records)
W3_LAST = 8190              # ... the third tier (8192 records)
W0_LEN = 400                # list length of the IR-space row
W0_LAST_WIDTH = 2           # digits per element: up to this width the list is too dense for the IR region
FIELDS_LAST = 31            # the first fields of bench.All in declaration order the walker takes: its 32-bit "fields seen"
                            # mask indexes fields in number order, where late_low (18) sits ahead of r_int32 (21)
W5_WALK_LAST = 6            # nesting through Node.children (a list and an object per level) the walker takes
W5_NODE_PT_LAST = 14        # ... the per-thread parser
W5_COOP_LAST = 21           # nesting through bench.All.recursive the lock-step parser takes (the walker: field index >= 32)
W5_PT_LAST = 30             # ... the per-thread parser (GGR_MAX_DEPTH frames, the root included)
MAX_DEPTH = 32              # GGR_MAX_DEPTH: the per-thread parser answers GGR_ST_DEPTH beyond it
CE_MAX_INPUT = 65000        # CE_MAX_INPUT: the walker takes items that end at or before this byte
CE_STAGE_BUF = 4864         # CE_STAGE_BUF: wire bytes assembled in shared memory
CE_STAGE = 8192             # CE_STAGE: the walker's first tier leaves items with more wire bytes
CE_LONG_MAX = 32            # CE_LONG_MAX: the emitter's hand-off list
CE_LONG_STR = 128           # CE_LONG_STR: plain strings of at least this many bytes go to the list
CW_TILE = 2048              # CW_TILE: the tokenizer stages request text in tiles of this many bytes
TOO_LARGE = (2 << 20) - 16  # request items above this many bytes: GGR_ST_TOO_LARGE


def _side(v, last):
    return "below" if v < last else ("at" if v == last else "above")


def _around(last, far=()):
    """the last one taken and the first one left, one more on each side, and a few far above"""
    return [last - 1, last, last + 1, last + 2] + list(far)


def _wire(m):
    return pbgen.wire(m)


def _fit(build, target, measure, lo=0):
    """smallest pad length L >= lo with measure(build(L)) == target (measure grows by one per pad byte, varint widths
    aside)"""
    L = lo
    for _ in range(8):
        got = measure(build(L))
        if got == target:
            return build(L)
        L = max(lo, L + target - got)
    for d in (-1, 1, -2, 2):
        if measure(build(L + d)) == target:
            return build(L + d)
    raise AssertionError(("no pad length fits", target))


def _node(children=(), id=None, value=None):
    m = pbgen.cls(NODE)()
    if id is not None:
        m.id = id
    if value is not None:
        m.value = value
    for c in children:
        m.children.add().CopyFrom(c)
    return m


def _empty_children(k):
    m = pbgen.cls(NODE)()
    for _ in range(k):
        m.children.add()
    return m


def _chain(depth):
    """Node nested `depth` levels below the root through children"""
    m = _node(id="leaf")
    for _ in range(depth):
        m = _node([m])
    return m


_DIRTY = ["a\"b", "tab\there", "café", "日本", "line\nnext", "\U0001F600!", "back\\slash", "x€y"]


def _text_len(oracle, name, wire, flags=0):
    st, js, _ = oracle.decode(name, wire, flags)
    assert st == 0, (name, st)
    return len(js)


def _wire_len(oracle, name, js):
    st, w, _ = oracle.encode(name, js)
    assert st == 0, (name, js[:100], st)
    return len(w)


def reply_items(oracle):
    rng = random.Random(0x5EED)
    out = []
    add = lambda lid, side, name, w, dmg=False: out.append(Item(lid, side, name, w, dmg))
    # R1 / R2: table entries (the root and one per empty child)
    for k in _around(R1_LAST, (300,)):
        add("R1", _side(k, R1_LAST), NODE, _wire(_empty_children(k)))
    for k in _around(R2_LAST, (5000,)):
        add("R2", _side(k, R2_LAST), NODE, _wire(_empty_children(k)))
    # damaged: a child's length byte cut off at the boundary
    add("R1", "above", NODE, _wire(_empty_children(R1_LAST + 1))[:-1], True)
    add("R2", "at", NODE, _wire(_empty_children(R2_LAST))[:-1], True)
    # R3: items that end at byte 4096 of their 16-byte aligned chunk run; plain and non-plain strings on both sides of it
    def r3(L):
        kids = []
        for j in range(24):
            v = ("plain %02d " % j) * 4 if j % 3 else _DIRTY[j % len(_DIRTY)] * 3
            kids.append(_node(id="c%d" % j, value=v))
        tail = [_node(id="t", value=_DIRTY[2] * 2), _node(id="u", value="plain tail"), _node(id="w", value="é")]
        return _wire(_node(kids + tail, id="p" * L, value="x" * 40))
    for n in (4080, 4081, 4082, 4095, 4096, 4097, 4098):
        w = _fit(r3, n, len)
        add("R3", _side(n, COOP_MAX_WIRE), NODE, w)
    w = bytearray(_fit(r3, 4096, len))
    w[-1] = 0xFF  # the last string's final byte (a non-plain one) is no longer UTF-8
    add("R3", "at", NODE, bytes(w), True)
    # R4: strings that need escaping or hold non-ASCII bytes, one per child
    for k in _around(DIRTY_MAX, (100,)):
        kids = [_node(value=_DIRTY[j % len(_DIRTY)] + "-%d" % j) for j in range(k)]
        add("R4", _side(k, DIRTY_MAX), NODE, _wire(_node(kids, id="root")))
    kids = [_node(value=_DIRTY[j % len(_DIRTY)]) for j in range(DIRTY_MAX + 1)]
    w = bytearray(_wire(_node(kids)))
    w[-1] = 0xC3  # the 65th string ends inside a two-byte sequence
    add("R4", "above", NODE, bytes(w), True)
    # R5: the hand-off list: long plain strings, escaped strings, long bytes (base64)
    for k in _around(LONG_MAX, (60,)):
        kids = [_node(value=chr(97 + j % 26) * COOP_LONG + "%03d" % j) for j in range(k)]
        add("R5", _side(k, LONG_MAX), NODE, _wire(_node(kids)))
    for ln in (COOP_LONG - 1, COOP_LONG, COOP_LONG + 1):
        for k in (LONG_MAX, LONG_MAX + 1):
            kids = [_node(value=(("%02d" % j) * ln)[:ln]) for j in range(k)]
            n_long = k if ln >= COOP_LONG else 0
            add("R5", _side(n_long, LONG_MAX), NODE, _wire(_node(kids)))
    for k in _around(LONG_MAX, (45,)):
        m = pbgen.cls(A)()
        for j in range(k):
            c = j % 3
            if c == 0:
                m.r_string.append(chr(65 + j % 26) * (COOP_LONG + j))
            elif c == 1:
                m.r_string.append(_DIRTY[j % len(_DIRTY)] * (1 + j % 5))
            else:
                m.r_bytes.append(bytes(rng.randrange(256) for _ in range(COOP_LONG + j % 7)))
        add("R5", _side(k, LONG_MAX), A, _wire(m))
    # R6: text assembled in shared memory up to 6144 bytes, written in place beyond (flags 0: no space after commas)
    def r6(L):
        return _wire(_node([_node(id="k%d" % j, value="v") for j in range(40)], id="i" * L, value="val"))
    for t in (STAGE_BUF - 2, STAGE_BUF - 1, STAGE_BUF, STAGE_BUF + 1, STAGE_BUF + 2):
        add("R6", _side(t, STAGE_BUF), NODE, _fit(r6, t, lambda w: _text_len(oracle, NODE, w)))
    # R7: many small entries next to one large leaf, texts of 8191..8193 bytes and far above, written in place
    def r7(L):
        return _wire(_node([_node(id="k%d" % j, value=_DIRTY[j % len(_DIRTY)] if j % 4 == 0 else "v%d" % j) for j in range(120)],
                           id="I" * L, value="tail"))
    for t in (8191, 8192, 8193, 20000, 70000):
        add("R7", _side(t, 8192), NODE, _fit(r7, t, lambda w: _text_len(oracle, NODE, w)))
    # R8: nesting through children
    for d in _around(R8_LAST) + [DEC_MAX_DEPTH - 1, DEC_MAX_DEPTH, DEC_MAX_DEPTH + 1, 40]:
        add("R8", _side(d, R8_LAST), NODE, _wire(_chain(d)))
    add("R8", "above", NODE, _wire(_chain(R8_LAST + 1))[:-2], True)
    return out


# ---- request side ------------------------------------------------------------------------------------------------
_LIT = {1: "2.5", 2: "1.5", 3: '"-3"', 4: '"4"', 5: "-5", 6: '"6"', 7: "7", 8: "true", 12: '"YWJj"', 13: "13",
        14: '"RED"', 15: "-15", 16: '"-16"', 17: "17", 18: '"-18"'}


def _literal(fd, rng):
    from google.protobuf.descriptor import FieldDescriptor as FD
    if fd.type == FD.TYPE_STRING:
        return '"s%d"' % fd.number
    if fd.type == FD.TYPE_MESSAGE:
        mt = fd.message_type
        if mt.GetOptions().map_entry:
            k, v = mt.fields_by_name["key"], mt.fields_by_name["value"]
            key = {FD.TYPE_STRING: '"k"', FD.TYPE_BOOL: '"true"'}.get(k.type, '"7"')
            return "{%s:%s}" % (key, _literal(v, rng))
        if mt.full_name == "google.protobuf.Timestamp":
            return '"2024-01-01T12:00:00Z"'
        if mt.full_name == "bench.All":
            return '{"f_int32":1}'
        return '{"x":%d}' % fd.number
    return _LIT[fd.type]


def _repeated(fd):
    from google.protobuf.descriptor import FieldDescriptor as FD
    return fd.is_repeated if hasattr(fd, "is_repeated") else fd.label == FD.LABEL_REPEATED


def _fields_object(k):
    """one object holding the first k fields of bench.All in declaration order (a oneof contributes one member)"""
    rng = random.Random(k)
    from google.protobuf.descriptor import FieldDescriptor as FD
    parts, seen_oneof = [], False
    for fd in pbgen.cls(A).DESCRIPTOR.fields[:k]:
        v = _literal(fd, rng)
        if _repeated(fd) and not (fd.message_type and fd.message_type.GetOptions().map_entry):
            v = "[%s]" % v
        if fd.containing_oneof is not None and not fd.containing_oneof.name.startswith("_"):
            if seen_oneof:
                continue
            seen_oneof = True
        parts.append('"%s":%s' % (fd.name, v))
    return ("{" + ",".join(parts) + "}").encode()


def _int_list(k, width=6, field="r_int32"):
    lo = 10 ** (width - 1) if width > 1 else 0
    return ('{"%s":[%s]}' % (field, ",".join(str(lo + j % (9 * max(lo, 1))) for j in range(k)))).encode()


def _node_nest(d):
    return b'{"root_node":' + b'{"id":"n","children":[' * d + b'{"id":"leaf","value":"v"}' + b"]}" * d + b"}"


def _nest(d):
    return b'{"recursive":' * d + b'{"f_int32":1}' + b"}" * d


def _str_item(L, extra=b""):
    return b'{"f_int32":7' + extra + b',"f_string":"' + b"s" * L + b'"}'


def request_items(oracle):
    rng = random.Random(0x1EAF)
    out = []
    add = lambda lid, side, js, dmg=False: out.append(Item(lid, side, A, js, dmg))
    # W0: IR region space, 8 bytes per input byte: a list of W0_LEN elements gets denser as its elements get shorter
    for wdt in range(1, 7):
        add("W0", "above" if wdt <= W0_LAST_WIDTH else ("at" if wdt == W0_LAST_WIDTH + 1 else "below"), _int_list(W0_LEN, wdt))
    for js in (b'{"r_msg":[' + b",".join([b"{}"] * W0_LEN) + b"]}", b'{"r_bool":[' + b",".join([b"true"] * W0_LEN) + b"]}",
               b'{"r_msg":[' + b",".join(b'{"x":%d}' % (j % 10) for j in range(W0_LEN)) + b"]}"):
        add("W0", "below" if b"true" in js else "above", js)
    # W1..W3: value records of the walker's three tiers (the root, the list and its six-digit elements)
    for lid, last, far in (("W1", W1_LAST, (400,)), ("W2", W2_LAST, (2000,)), ("W3", W3_LAST, (8500,))):
        for k in _around(last, far):
            add(lid, _side(k, last), _int_list(k))
        js = _int_list(last + 1)
        add(lid, "above", js[: len(js) // 2], True)
    # W4: the walker's 32 fields per message
    for k in _around(FIELDS_LAST, (57,)):
        add("W4", _side(k, FIELDS_LAST), _fields_object(k))
    add("W4", "above", _fields_object(FIELDS_LAST + 1)[:-2], True)
    # W5: nesting through Node.children (walker) and through `recursive` (lock-step parser, per-thread parser)
    for d in _around(W5_WALK_LAST, (W5_NODE_PT_LAST, W5_NODE_PT_LAST + 1, 20)):
        out.append(Item("W5", _side(d, W5_WALK_LAST), PNR, _node_nest(d), False))
    out.append(Item("W5", "above", PNR, _node_nest(W5_WALK_LAST + 1)[:-4], True))
    for d in _around(W5_COOP_LAST) + _around(W5_PT_LAST, (40,)):
        add("W5", _side(d, W5_COOP_LAST), _nest(d))
    add("W5", "above", _nest(W5_COOP_LAST + 1)[:-3], True)
    # W6: 16-bit positions: the walker takes items that end by byte 65000 (start offset included)
    for n in (64983, 64984, 64985, 64986, 64999, 65000, 65001, 65002, 70000):
        js = _fit(lambda L: _str_item(L, b',"r_int32":[1,2,3],"f_msg":{"x":1,"y":"yy"}'), n, len)
        add("W6", _side(n, CE_MAX_INPUT), js)
    js = bytearray(_fit(lambda L: _str_item(L), CE_MAX_INPUT, len))
    js[-4] = 0xFF
    add("W6", "at", bytes(js), True)
    # W7: wire bytes staged (<= 4864) or written in place; the first tier leaves items with more than 8192
    def w7(L):
        strs = ",".join('"%s"' % (chr(97 + j % 26) * (20 + j % 50)) for j in range(60))
        return ('{"f_int32":5,"r_string":[%s],"f_string":"%s","r_sint32":[1,-2,3]}' % (strs, "z" * L)).encode()
    for t in (CE_STAGE_BUF - 1, CE_STAGE_BUF, CE_STAGE_BUF + 1, CE_STAGE - 1, CE_STAGE, CE_STAGE + 1, CE_STAGE + 2, 20000):
        add("W7", _side(t, CE_STAGE), _fit(w7, t, lambda js: _wire_len(oracle, A, js)))
    # W8: the emitter's hand-off list: long plain strings and strings with two-character escapes
    for k in _around(CE_LONG_MAX, (50,)):
        add("W8", _side(k, CE_LONG_MAX), ('{"r_string":[%s]}' % ",".join('"%s"' % ((chr(97 + j % 26) + "%03d" % j) * 40)[:CE_LONG_STR + j % 9]
                                                                            for j in range(k))).encode())
    for ln in (CE_LONG_STR - 1, CE_LONG_STR, CE_LONG_STR + 1):
        for k in (CE_LONG_MAX, CE_LONG_MAX + 1):
            add("W8", _side(k if ln >= CE_LONG_STR else 0, CE_LONG_MAX),
                ('{"f_int32":1,"r_string":[%s]}' % ",".join('"%s"' % (("%03d" % j) * ln)[:ln] for j in range(k))).encode())
    # escaped strings (two-character escapes only: one list entry each, whatever their length), with backslash runs and
    # escapes straddling the 32-byte rounds of the whole-warp decoder
    esc = [b"\\\\", b"\\n", b"\\\"", b"\\\\\\\\", b"\\t\\\\", b"\\/\\b\\f\\r"]
    def esc_str(j):
        e = esc[j % len(esc)]
        pre = 26 + j % 12  # the escape starts at bytes 26..37 of the string's text
        return b"a" * pre + e + b"b" * (j % 40) + e
    for k in _around(CE_LONG_MAX, (40,)):
        add("W8", _side(k, CE_LONG_MAX), b'{"r_string":[' + b",".join(b'"' + esc_str(j) + b'"' for j in range(k)) + b"]}")
    for k in (CE_LONG_MAX - 1, CE_LONG_MAX, CE_LONG_MAX + 1):  # backslash runs around the end of a round, next to a long string
        strs = [b'"' + b"x" * (29 + j % 5) + b"\\\\" * (1 + j % 3) + b"\\n" + b"y" * (j % 7) + b'"' for j in range(k - 1)]
        add("W8", _side(k, CE_LONG_MAX), b'{"f_string":"' + b"p" * 200 + b'","r_string":[' + b",".join(strs) + b"]}")
    add("W8", "at", b'{"r_string":[' + b",".join(b'"' + esc_str(j) + b'"' for j in range(CE_LONG_MAX)) + b"]", True)
    # W10: request items of 2 MiB - 16 bytes and one byte either side
    for n in (TOO_LARGE - 1, TOO_LARGE, TOO_LARGE + 1):
        add("W10", _side(n, TOO_LARGE), _fit(lambda L: _str_item(L), n, len))
    return out


def corpus(oracle):
    """reply items, request items"""
    return reply_items(oracle), request_items(oracle)


# ---- device-only rows ----------------------------------------------------------------------------------------------
TILE_EVENTS = [b'"', b"\\\\", b"\\\\\\\\", b'\\"', "é".encode(), "日".encode(), "\U0001F600".encode(), b","]
TILE_EDGES = (CW_TILE - 1, CW_TILE, CW_TILE + 1, 2 * CW_TILE - 1, 2 * CW_TILE, 2 * CW_TILE + 1)


def tile_items(seed=9):
    """W9: request text staged in 2 KB tiles: a closing quote, an even or odd backslash run, a two-, three- or four-byte
    UTF-8 sequence or a token start (a comma) at rebased bytes 2047 / 2048 / 2049 and 4095 / 4096 / 4097, in items of 2, 3
    and 5 tiles, and items of 1 tile with the same events inside it.  The tokenizer rebases an item to the 16-byte aligned
    address at or below its start, so an event at byte k of an item that starts at offset s (mod 16) sits at rebased byte
    s + k; each item is built for its own start offset, 0..15 in turn.  Returns (start offset, rebased edge, event, json)."""
    rng = random.Random(seed)
    out = []
    for tiles in (1, 2, 3, 5):
        n_target = tiles * CW_TILE - rng.randrange(0, 300)
        edges = TILE_EDGES if tiles > 1 else (40, 1023, 1500)
        for pos in edges:
            if pos + 40 > n_target:
                continue
            for ev in TILE_EVENTS:
                for rep in range(4):
                    s = len(out) % 16
                    p = pos - s  # the event's first byte within the item
                    if ev == b",":  # the comma at p, the key after it starts a token at p + 1
                        body = b'{"f_string":"' + b"q" * (p - 14) + b'","r_int32":[1,2]'
                    elif ev == b'"':  # the closing quote of a string
                        body = b'{"f_string":"' + b"q" * (p - 13) + b'","opt_string":"qqqqq"'
                    else:
                        body = b'{"f_string":"' + b"q" * (p - 13) + ev + b"q" * 5 + b'"'
                    assert body[p:p + len(ev)] == ev
                    rest = n_target - len(body) - 2
                    if rest > 20:
                        body += b',"custom":"' + b"r" * (rest - 12) + b'"'
                    out.append((s, pos, ev, body + b"}"))
    return out


def pool_batch(n_items=2500, children=2000):
    """R9: Node replies of `children` empty children each (one table entry per child, 2 bytes of wire) and a one-byte id
    (one more entry; it makes the reply 4003 bytes long, so the replies start at every offset mod 16): past the first tier's
    table, within the second's; together more entries than one call's pool holds.  Returns (message, wire, entries)."""
    m = _empty_children(children)
    m.id = "x"
    return NODE, _wire(m), 2 + children, n_items


# ---- nesting past the per-thread frames (GGR_ST_DEPTH, a documented gap) ------------------------------------------
def nesting(it):
    """levels of Node.children / bench.All.recursive below the root of an R8 or W5 item (None: not a nesting item, or a
    damaged one that does not parse)"""
    if it.limit_id == "W5":
        return it.data.count(b'"children"' if it.message == PNR else b'"recursive"')
    if it.limit_id != "R8":
        return None
    m = pbgen.cls(NODE)()
    try:
        m.ParseFromString(it.data)
    except Exception:
        return None
    d = 0
    while len(m.children):
        m = m.children[0]
        d += 1
    return d


def pt_depth_last(it):
    """the deepest nesting of the item's kind the per-thread code takes"""
    if it.limit_id == "R8":
        return R8_PT_LAST
    return W5_NODE_PT_LAST if it.message == PNR else W5_PT_LAST


def past_frames(it):
    """nested deeper than the per-thread code's frames: GGR_ST_DEPTH where the oracle answers is a documented gap"""
    d = nesting(it)
    return d is not None and d > pt_depth_last(it)
