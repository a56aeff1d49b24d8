"""Long mixed runs of items for the persistent lock-step kernels.

A persistent warp draws item after item and keeps its shared memory, its registers and its async state from one to the
next.  The unique items below come from the generators the other tests use (edge cases, random and damaged items, merges,
well-known types, the capacity limits, the number corpus and a slice of the mixed workload).  A replication plan repeats
each one and shuffles the copies into one long batch, so that every warp of every lock-step list runs many items in a row,
after items of every other kind, and each copy starts at a different offset mod 16.

Item.gap is the status the engine documents for an item the oracle accepts (DESIGN.md section 6): GGR_ST_DEPTH for
nesting past the per-thread frames, GGR_ST_TOO_LARGE for request items above 2 MiB - 16 bytes, GGR_ST_UNSUPPORTED for
Struct fields and FieldMask strings with escapes.  Item.damaged marks request JSON with byte-level damage, where only
acceptance is compared with the oracle (the parser may meet a different error first)."""
import collections
import random

import cases
import limits as LM
import numcorpus as NC
import wiremut

Item = collections.namedtuple("Item", "message data gap damaged")

ST_DEPTH, ST_TOO_LARGE, ST_UNSUPPORTED = 8, 9, 11
SMALL = 16 << 10        # items up to this size: more copies the smaller they are
MID = 256 << 10         # items up to this size: at most MID_COPIES copies; larger ones: one copy
MID_COPIES = 4
MAX_COPIES = 64
MIN_ITEMS = 100000      # 132 SMs x 64 resident warps = 8448 warps: more than 10 items per warp of any list
MAX_BYTES = 64 << 20
MIN_RESIDUES = 4        # distinct start offsets mod 16 of every replicated item
SEEDS = (11, 12)        # the two orders of the device runs

_cache = {}


def _mixed(n, first):
    import benchgen
    names = {}

    def mi(name):
        return names.setdefault(name, len(names))

    wl = benchgen.mixed(n, mi, first=first)
    inv = {v: k for k, v in names.items()}
    req = [(inv[int(wl.req_msg[i])], wl.req_json[int(wl.req_off[i]):int(wl.req_off[i + 1])].tobytes()) for i in range(n)]
    rep = [(inv[int(wl.rep_msg[i])], wl.rep_wire[int(wl.rep_off[i]):int(wl.rep_off[i + 1])].tobytes()) for i in range(n)]
    return req, rep


def _wkt_gap(name, js):
    return ST_UNSUPPORTED if (name == "wkt.HasStruct" and b"s" in js) or cases.fieldmask_gap(js) else None


def _limit_gap(it):
    if LM.past_frames(it):
        return ST_DEPTH
    if it.limit_id == "W10" and len(it.data) > LM.TOO_LARGE:
        return ST_TOO_LARGE
    return None


def _unique(items):
    seen, out = set(), []
    for it in items:
        k = (it.message, it.data)
        if k not in seen:
            seen.add(k)
            out.append(it)
    return out


def requests(oracle):
    """request items: (message, canonical arguments JSON)"""
    if "req" not in _cache:
        rng = random.Random(5)
        out = [Item(n, js, None, False) for n, js, _ in cases.ENCODE_EDGE]
        out += [Item(n, js, None, False) for n, js in cases.random_encode_cases(150)]
        out += [Item(n, cases.mutate_json(js, rng), None, True) for n, js in cases.random_encode_cases(80, seed0=700) for _ in range(3)]
        out += [Item(n, js, _wkt_gap(n, js), False) for n, js in cases.WKT_ENCODE]
        out += [Item(it.message, it.data, _limit_gap(it), False) for it in LM.corpus(oracle)[1]]
        out += [Item(LM.A, js, None, False) for *_, js in LM.tile_items()]
        out += [Item(n, js, None, False) for n, js, _ in NC.request_items(_literals())]
        out += [Item(n, js, None, False) for n, js in _mixed(1500, 0)[0]]
        _cache["req"] = _unique(out)
    return _cache["req"]


def replies(oracle):
    """reply items: (message, wire)"""
    if "rep" not in _cache:
        rng = random.Random(6)
        out = [Item(n, bytes.fromhex(h), None, False) for n, h in cases.DECODE_EDGE_HEX]
        out += [Item(n, w, None, False) for n, w in cases.random_decode_cases(120)]
        out += [Item(n, w, None, False) for n, w in cases.merge_cases() + cases.wkt_decode_cases()]
        # valid replies cut short and with damaged bytes: the random messages and the mixed workload's replies
        mixed = _mixed(1500, 7)[1]
        for n, w in cases.random_decode_cases(40, seed0=5000, mutators=False) + mixed[:400]:
            out += [Item(n, wiremut.truncate(w, rng), None, False), Item(n, wiremut.corrupt(w, rng), None, False)]
        out += [Item(it.message, it.data, _limit_gap(it), False) for it in LM.corpus(oracle)[0]]
        out += [Item(n, w, None, False) for n, w, _ in NC.reply_items(NC.reply_bits(64, n_random=30000), NC.reply_bits(32, stride=65521))]
        out += [Item(n, w, None, False) for n, w in mixed]
        _cache["rep"] = _unique(out)
    return _cache["rep"]


def bodies(oracle):
    """JSON-RPC tools/call request bodies (Item.message is None): the bodies of the request-body tests, the number corpus's
    bodies, and every request item whose message is a method's input as the arguments of a call of that method"""
    if "body" not in _cache:
        out = [Item(None, b, None, False) for b in cases.request_bodies(oracle)]
        out += [Item(None, b, None, False) for b, _ in NC.body_items(_literals())]
        tool = {}
        for m in reversed(oracle.methods()):
            tool[m["input"]] = m["tool"].encode()
        ids = [b"1", b'"abc"', b"-7", b"123456789012345", b'"a<b"', b"null", b"0"]
        for k, it in enumerate(requests(oracle)):
            t = tool.get(oracle.msg(it.message))
            if t is not None and len(it.data) <= 4096:
                out.append(Item(None, b'{"jsonrpc":"2.0","id":%s,"method":"tools/call","params":{"name":"%s","arguments":%s}}'
                                % (ids[k % len(ids)], t, it.data), None, False))
        _cache["body"] = _unique(out)
    return _cache["body"]


def _literals():
    if "lits" not in _cache:
        _cache["lits"] = NC.request_literals()
    return _cache["lits"]


def copies(n_bytes, k):
    """copies of an item of n_bytes: about k / n_bytes, from MIN_RESIDUES up to MAX_COPIES, for items up to SMALL"""
    if n_bytes > MID:
        return 1
    if n_bytes > SMALL:
        return MID_COPIES
    return max(MIN_RESIDUES, min(MAX_COPIES, k // max(n_bytes, 1)))


def plan(items, seed, min_items=MIN_ITEMS, max_bytes=MAX_BYTES):
    """one long batch: a list of indices into `items`, every item repeated (copies(), with the smallest k that makes the
    batch min_items long) and the copies shuffled with a fixed seed; adjacent copies are then swapped until every
    replicated item starts at MIN_RESIDUES offsets mod 16 or more"""
    lo, hi = 0, MAX_COPIES * (SMALL + 1)
    while lo < hi:
        k = (lo + hi) // 2
        if sum(copies(len(it.data), k) for it in items) >= min_items:
            hi = k
        else:
            lo = k + 1
    order = [u for u, it in enumerate(items) for _ in range(copies(len(it.data), lo))]
    assert len(order) >= min_items and sum(len(items[u].data) for u in order) <= max_bytes, \
        (len(order), sum(len(items[u].data) for u in order))
    random.Random(seed).shuffle(order)
    _spread_offsets(items, order)
    short = [u for u, r in residues(items, order).items() if len(r) < min(MIN_RESIDUES, copies(len(items[u].data), lo))]
    assert not short, ("items at fewer than %d offsets mod 16" % MIN_RESIDUES, len(short), short[:5])
    return order


def offsets(items, order):
    out, pos = [], 0
    for u in order:
        out.append(pos)
        pos += len(items[u].data)
    return out


def residues(items, order):
    """item index -> Counter of its copies' start offsets mod 16"""
    res = collections.defaultdict(collections.Counter)
    for u, off in zip(order, offsets(items, order)):
        res[u][off % 16] += 1
    return res


def _spread_offsets(items, order):
    """swapping two copies whose lengths are equal mod 16 leaves every start offset mod 16 where it was (the items between
    them move by a multiple of 16): for every replicated item at fewer than MIN_RESIDUES offsets, trade a copy at an offset
    it already has for a copy of another item at one it lacks, while that item keeps enough offsets of its own"""
    r16 = [o % 16 for o in offsets(items, order)]
    res = residues(items, order)
    pos = collections.defaultdict(list)
    by_class = collections.defaultdict(list)
    for p, u in enumerate(order):
        pos[u].append(p)
        by_class[len(items[u].data) % 16].append(p)
    need = lambda u: min(MIN_RESIDUES, len(pos[u]))
    rng = random.Random(len(order))
    for u in sorted(u for u in res if len(res[u]) < need(u)):
        cand = by_class[len(items[u].data) % 16]
        while len(res[u]) < need(u):
            p = next(p for p in pos[u] if res[u][r16[p]] > 1)
            start = rng.randrange(len(cand))
            for j in range(len(cand)):
                q = cand[(start + j) % len(cand)]
                v = order[q]
                if v == u or r16[q] in res[u]:
                    continue
                kept = len(res[v]) - (res[v][r16[q]] == 1) + (r16[p] not in res[v])
                if kept < min(len(res[v]), need(v)):
                    continue
                for w, a, b in ((u, p, q), (v, q, p)):
                    res[w][r16[a]] -= 1
                    if not res[w][r16[a]]:
                        del res[w][r16[a]]
                    res[w][r16[b]] += 1
                    pos[w][pos[w].index(a)] = b
                order[p], order[q] = v, u
                break
            else:
                break  # no copy to trade for this item: plan() reports it
