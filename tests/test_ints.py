"""Integer, bool and enum values against the exact reference (intref): the oracle on the whole corpus of
tests/intcorpus.py in both directions and on tools/call bodies, then every entry point of the host simulation.  Each
item gives exactly intref's bytes and status category, or (lock-step entry points only) is left to the per-thread
kernels with rc 200; a lock-step tier never answers rc 0 for an item intref refuses."""
import collections

import pytest

import intcorpus as IC
import intref as I
from test_strings import LEFT, _stop_at

_cache = {}


def _corpus():
    if not _cache:
        _cache["req"] = IC.request_items()
        _cache["bodies"] = IC.body_items()
        _cache["rep"] = IC.reply_items()
    return _cache


def _matches(st, out, want):
    if isinstance(want, str):
        return st == I.STATUS[want]
    return st == 0 and out == want


def test_corpus_shape():
    """the corpus reaches what it exists for (pinned counts): every kind, start offsets 0..15, failing and passing
    items in each direction, varints of every length 1..10 as singular values"""
    c = _corpus()
    req, rep = c["req"], c["rep"]
    assert (len(req), len(c["bodies"]), len(rep)) == (7548, 3432, 5646)
    assert {s for _, s, _, _ in req} == set(range(16)) == {s for _, s, _, _, _ in rep}
    cats = collections.Counter(w if isinstance(w, str) else "ok" for *_, w in req)
    assert cats == {"ok": 3257, I.INVALID_VALUE: 4037, I.SYNTAX: 254}, cats
    cats = collections.Counter(w if isinstance(w, str) else "ok" for *_, w, _ in rep)
    assert cats == {"ok": 4504, I.BAD_WIRE: 1142}, cats
    lens = {len(pb) for pb, wt in IC._value_bytes("int64") if wt == 0}
    assert set(range(1, 12)) == lens, lens
    assert max(len(js) for _, _, js, _ in req) > 4096 and max(len(w) for _, _, w, _, _ in rep) > 4096


def test_intref_rules():
    """intref on hand-checked cases of each rule"""
    V = I.value
    assert V("int32", b"2147483647") == 2**31 - 1 and V("int32", b"2147483648") == I.INVALID_VALUE
    assert V("int32", b"-2147483648") == -2**31 and V("uint32", b"-0") == 0 and V("uint64", b"-1") == I.INVALID_VALUE
    assert V("int64", b"1e2") == 100 and V("int64", b"100e-2") == 1 and V("int64", b"1.50e1") == 15
    assert V("int64", b"1.5") == I.INVALID_VALUE and V("int64", b"0.0e5") == 0
    assert V("uint64", b"12e18") == 12 * 10**18 and V("uint64", b"123e18") == I.INVALID_VALUE  # 3 + 18 > 20
    assert V("uint64", b"0.00000000000000000001e20") == 1 and V("uint64", b"0.0000000000000000000001e22") == I.INVALID_VALUE
    assert V("int64", b"1000000000000000000000000e-5") == I.INVALID_VALUE  # 10^19 > int64
    assert V("uint64", b"1000000000000000000000000e-5") == 10**19
    assert V("int32", b"0e2147483648") == 0 and V("int32", b"0.0e99999999999999999999") == 0
    assert V("int32", b"1e2147483648") == I.INVALID_VALUE and V("int32", b"1e-2147483649") == I.INVALID_VALUE
    assert V("int32", b"01") == I.SYNTAX and V("int32", b'"01"') == I.INVALID_VALUE and V("int32", b'"007 "') == I.INVALID_VALUE
    assert V("int32", b'"1 2"') == 1 and V("int32", b'"1]"') == 1 and V("int32", b'" 1"') == I.INVALID_VALUE
    assert V("int32", b'"\\u0031\\u0032"') == 12 and V("int32", b'"1\\u00a0"') == I.INVALID_VALUE
    assert V("bool", b"true") is True and V("bool", b'"true"') == I.INVALID_VALUE and V("bool", b"1") == I.INVALID_VALUE
    assert V("enum", b'"NEGATIVE"') == -5 and V("enum", b"7") == 7 and V("enum", b'"1"') == I.INVALID_VALUE
    assert V("enum", b"1e2") == 100 and V("enum", b"2147483648") == I.INVALID_VALUE
    assert I.key_value("int32", b"+3") == 3 and I.key_value("int32", b"007") == 7 and I.key_value("int32", b"-0") == 0
    assert I.key_value("uint64", b"+3") == I.INVALID_VALUE and I.key_value("int32", b"1e2") == I.INVALID_VALUE
    assert I.key_value("bool", b"True") == I.INVALID_VALUE
    assert I.body_value("int64", b"9007199254740993") == 9007199254740992
    assert I.body_value("uint64", b"12345678901234567") == 12345678901234568
    assert I.body_value("uint64", b"1e21") == I.INVALID_VALUE  # json.Marshal prints 1e+21: 1 + 21 digits > 20
    assert I.wire("int32", -1) == b"\xff" * 9 + b"\x01" and I.wire("enum", -5)[-1] == 1 and len(I.wire("enum", -5)) == 10
    assert I.wire("sint32", -1) == b"\x01" and I.wire("sint32", -2**31) == b"\xff\xff\xff\xff\x0f"
    assert I.consume_varint(b"\xff" * 9 + b"\x01", 0) == (2**64 - 1, 10) and I.consume_varint(b"\xff" * 9 + b"\x02", 0) is None
    assert I.consume_varint(b"\x80" * 10 + b"\x00", 0) is None and I.consume_varint(b"\x80\x00", 0) == (0, 2)
    assert I.from_wire("int32", 1 << 32) == 0 and I.from_wire("sint32", (1 << 32) | 3) == -2 and I.from_wire("bool", 1 << 32) is True
    assert I.from_wire("enum", 2**64 - 5) == -5 and I.from_wire("uint32", 2**64 - 1) == 2**32 - 1
    assert I.decode("bench.All", b"\x08\x80\x80\x80\x80\x10") == b"{}"  # int32 of 2^32
    assert I.decode("bench.All", b"\x80\x01\x07") == b'{"fEnum":7}' and I.decode("bench.All", b"\x10\x01") == b'{"fInt64":"1"}'
    assert I.decode("bench.All", b"\xaa\x01\x02\x01\x80") == I.BAD_WIRE  # packed payload ending inside a varint
    assert I.decode("bench.All", b"\xd2\x02\x05\x08\x03\x12\x01a\xd2\x02\x05\x08\x01\x12\x01b\xd2\x02\x05\x08\x03\x12\x01c", 1) \
        == b'{"mInt32Str":{"1":"b", "3":"c"}}'


# ---- the oracle --------------------------------------------------------------------------------------------------
def test_oracle_requests(oracle):
    bad = []
    for name, _, js, want in _corpus()["req"]:
        st, wire, _ = oracle.encode(name, js)
        if not _matches(st, wire, want):
            bad.append((js[:150], st, want if isinstance(want, str) else want.hex()[:60], wire.hex()[:60]))
    assert not bad, (len(bad), bad[:8])


def test_oracle_replies(oracle):
    bad = []
    for name, _, w, t0, t1 in _corpus()["rep"]:
        for fl, want in ((0, t0), (1, t1)):
            st, js, _ = oracle.decode(name, w, fl)
            if not _matches(st, js, want):
                bad.append((fl, w[:40].hex(), st, js[:150], want[:150]))
    assert not bad, (len(bad), bad[:5])


def test_oracle_bodies(oracle):
    """tools/call bodies: the wire of intref's value after encoding/json's float64 round trip; never rc 0 for a value
    intref refuses or a body encoding/json refuses"""
    bad = []
    for _, body, want in _corpus()["bodies"]:
        r = oracle.request(body)
        ok = r["kind"] != 0 if isinstance(want, str) else (r["kind"] == 0 and r["wire"] == want)
        if not ok:
            bad.append((body[90:200], r["kind"], r["status"], r["wire"].hex()))
    assert not bad, (len(bad), bad[:5])


# ---- host simulation: every entry point --------------------------------------------------------------------------
def _offs(i, s):
    return s, (i * 5) % 16


def test_hostsim_encode(hsim):
    """the per-thread parser takes every item"""
    bad = []
    for i, (name, s, js, want) in enumerate(_corpus()["req"]):
        st, out = hsim.encode(name, js, *_offs(i, s))
        if not _matches(st, out, want):
            bad.append((js[:150], st, want if isinstance(want, str) else want.hex()[:80], out.hex()[:80]))
    assert not bad, (len(bad), bad[:5])


def _taken(run, items, idx, want_of):
    bad, taken = [], []
    for i in idx:
        st, out = run(i)
        if st == LEFT:
            continue
        if not _matches(st, out, want_of(i)):
            w = want_of(i)
            bad.append((items[i][2][:150], st, out[:150], w if isinstance(w, str) else w[:150]))
        if st == 0:
            taken.append(i)
    assert not bad, (len(bad), bad[:5])
    return taken


# valid items each lock-step request tier takes, pinned on this corpus: the lock-step parser's two tiers (separate
# entry points), and what each walker tier adds over the tiers before it
_REQ_FLOORS = {"coop0": 2748, "coop1": 2792, "walk1": 518, "walk2": 404, "walk3": 2}
# the lock-step reply tiers: the first, and what the pooled second one adds
_REP_FLOORS = (3872, 28)


@pytest.mark.parametrize("tier", [0, 1])
def test_hostsim_encode_coop(hsim, tier):
    """the lock-step parser: exact bytes and status, or left (200); never rc 0 for an item intref refuses"""
    req = _corpus()["req"]
    run = lambda i: hsim.encode_coop(req[i][0], req[i][2], *_offs(i, req[i][1]), tier=tier)
    taken = _taken(run, req, range(len(req)), lambda i: req[i][3])
    assert len(taken) >= _REQ_FLOORS["coop%d" % tier], len(taken)


def test_hostsim_encode_walk(hsim, monkeypatch):
    """the token-parallel walker, whole and stopped after its first and second tier"""
    req = _corpus()["req"]
    run = lambda i: hsim.encode_walk(req[i][0], req[i][2], *_offs(i, req[i][1]))
    _stop_at(monkeypatch)
    full = _taken(run, req, range(len(req)), lambda i: req[i][3])
    _stop_at(monkeypatch, "HS_WALK_TIER2_ONLY")
    upto2 = _taken(run, req, full, lambda i: req[i][3])
    _stop_at(monkeypatch, "HS_WALK_TIER1_ONLY")
    upto1 = _taken(run, req, upto2, lambda i: req[i][3])
    got = (len(upto1), len(upto2) - len(upto1), len(full) - len(upto2))
    assert all(g >= w for g, w in zip(got, (_REQ_FLOORS["walk1"], _REQ_FLOORS["walk2"], _REQ_FLOORS["walk3"]))), got


@pytest.mark.parametrize("tier", [0, 1])
def test_hostsim_request_envelope(hsim, tier):
    """tools/call bodies through the lock-step parser (the envelope's float64 round trip): intref's wire, or left"""
    bad = []
    handled = 0
    for i, (s, body, want) in enumerate(_corpus()["bodies"]):
        rc, wire, method, idt = hsim.request_coop(body, s, (i * 3) % 16, tier)
        if rc == LEFT:
            continue
        if isinstance(want, str) or rc != 0 or wire != want:
            bad.append((body[90:200], rc, wire.hex()[:80], want if isinstance(want, str) else want.hex()))
        handled += 1
    assert not bad, (len(bad), bad[:5])
    assert handled >= 1556, handled  # every body intref accepts


@pytest.mark.parametrize("flags", [0, 1])
def test_hostsim_decode(hsim, flags):
    """the per-thread reply kernels take every item"""
    bad = []
    for i, (name, s, w, t0, t1) in enumerate(_corpus()["rep"]):
        want = t1 if flags else t0
        st, out = hsim.decode(name, w, flags, *_offs(i, s))
        if not _matches(st, out, want):
            bad.append((w[:60].hex(), st, out[:150], want[:150]))
    assert not bad, (len(bad), bad[:5])


def test_hostsim_decode_lockstep(hsim, monkeypatch):
    """the lock-step reply tiers, whole and stopped after the first"""
    rep = _corpus()["rep"]
    run = lambda i: hsim.decode_coop(rep[i][0], rep[i][2], i & 1, *_offs(i, rep[i][1]))
    want_of = lambda i: rep[i][4] if i & 1 else rep[i][3]
    _stop_at(monkeypatch)
    full = _taken(run, rep, range(len(rep)), want_of)
    _stop_at(monkeypatch, "HS_COOP_TIER1_ONLY")
    upto1 = _taken(run, rep, full, want_of)
    got = (len(upto1), len(full) - len(upto1))
    assert got[0] >= _REP_FLOORS[0] and got[1] >= _REP_FLOORS[1], got
