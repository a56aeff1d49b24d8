"""Timestamp, Duration, FieldMask, wrapper and Empty values against the exact reference (timeref): the oracle on the
whole corpus of tests/timecorpus.py in both directions and on tools/call bodies, then every entry point of the host
simulation.  Each item gives exactly timeref's bytes and status category, or (lock-step entry points only) is left to
the per-thread kernels with rc 200; a lock-step tier never answers rc 0 for an item timeref refuses.  A FieldMask
written with escapes is the kernels' one documented gap: exactly GGR_ST_UNSUPPORTED.  The schema is the fixture with
wkt.Times appended (timecorpus.extended_fds), registered here on objects of this module's own."""
import collections
import datetime

import pytest

import timecorpus as TC
import timeref as T
from test_strings import LEFT, _stop_at

_cache = {}


def _corpus():
    if not _cache:
        _cache["req"] = TC.request_items()
        _cache["bodies"] = TC.body_items()
        _cache["rep"] = TC.reply_items()
    return _cache


@pytest.fixture(scope="module")
def times_fds():
    return TC.extended_fds()


@pytest.fixture(scope="module")
def oracle_t(times_fds):
    import orc
    return orc.Schema(times_fds)


@pytest.fixture(scope="module")
def hsim_t(times_fds):
    import hostsim
    return hostsim.Schema(times_fds)


def _matches(st, out, want, gap=False):
    if gap:
        return st == T.STATUS[T.UNSUPPORTED]
    if isinstance(want, str):
        return st == T.STATUS[want]
    return st == 0 and out == want


def test_corpus_shape():
    """the corpus reaches what it exists for (pinned counts): every category in both directions, start offsets 0..15,
    escaped FieldMasks, seconds varints of every length, items past 4 KB"""
    c = _corpus()
    req, rep = c["req"], c["rep"]
    assert (len(req), len(c["bodies"]), len(rep)) == (3305, 914, 739)
    assert {s for _, s, *_ in req} == set(range(16)) == {s for _, s, *_ in rep}
    cats = collections.Counter(w if isinstance(w, str) else "ok" for _, _, _, w, _ in req)
    assert cats == {"ok": 2084, T.INVALID_VALUE: 775, T.RANGE: 396, T.SYNTAX: 50}, cats
    assert sum(g for *_, g in req) == 198
    cats = collections.Counter(w if isinstance(w, str) else "ok" for *_, w, _ in rep)
    assert cats == {"ok": 291, T.RANGE: 310, T.BAD_WIRE: 97, T.INVALID_VALUE: 30, T.INVALID_UTF8: 11}, cats
    assert {len(T.intref.varint(v)) for v in TC.seconds_values()} == set(range(1, 11))
    assert {m for m, *_ in req} == {TC.TM, *T.ROOTS} == {m for m, *_ in rep}
    assert max(len(js) for _, _, js, _, _ in req) > 65000 and max(len(w) for _, _, w, _, _ in rep) > 4096


def test_timeref_rules():
    """timeref on hand-worked cases of each rule"""
    TS, D, F = T.timestamp, T.duration, T.field_mask
    assert TS(b"1970-01-01T00:00:00Z") == (0, 0) and TS(b"1969-12-31T23:59:59.5Z") == (-1, 500000000)
    assert TS(b"0001-01-01T00:00:00Z") == (T.MIN_TS, 0) and TS(b"0000-12-31T23:59:59Z") == T.RANGE
    assert TS(b"0000-12-31T23:00:00-01:00") == (T.MIN_TS, 0)  # year 0000 brought into range by its offset
    assert TS(b"9999-12-31T23:59:59Z") == (T.MAX_TS, 0) and TS(b"9999-12-31T23:59:59-00:01") == T.RANGE
    assert TS(b"2024-01-01T12:00:00+24:60") == (1704110400 - 90000, 0) and TS(b"2024-01-01T12:00:00+24:61") == T.INVALID_VALUE
    assert TS(b"2024-01-01T1:02:03Z") == (1704070923, 0) and TS(b"2024-01-01T24:00:00Z") == T.INVALID_VALUE
    assert TS(b"2024-01-01T00:00:00,1234567891Z") == (1704067200, 123456789)
    assert TS(b"2024-01-01T00:00:00.1234567891Z") == T.INVALID_VALUE  # protojson's own check of a '.' fraction
    assert TS(b"9999-12-31T23:59:59.1234567890-00:01") == T.RANGE  # the range check comes first
    assert TS(b"2024-02-29T00:00:00Z") != T.INVALID_VALUE and TS(b"2100-02-29T00:00:00Z") == T.INVALID_VALUE
    assert TS(b"2000-02-29T00:00:00Z") != T.INVALID_VALUE and TS(b"0000-02-29T00:00:00Z") == T.RANGE
    assert TS(b"2024-01-01t00:00:00Z") == TS(b"2024-01-01T00:00:00z") == TS(b"2024-01-01T00:00:00Z ") == T.INVALID_VALUE
    assert D(b"1.s") == (1, 0) and D(b".s") == (0, 0) and D(b"-.5s") == (0, -500000000) and D(b"-1.5s") == (-1, -500000000)
    assert D(b"00s") == D(b"0") == D(b"+") == D(b"1.0000000000s") == T.INVALID_VALUE and D(b"+1s") == (1, 0)
    assert D(b"9223372036854775807s") == T.RANGE and D(b"9223372036854775808s") == T.INVALID_VALUE
    assert D(b"-9223372036854775808s") == T.INVALID_VALUE  # ParseInt reads the digits without the sign
    assert D(b"315576000000.999999999s") == (315576000000, 999999999) and D(b"-315576000001s") == T.RANGE
    assert F(b"fooBar.bazQux,a") == [b"foo_bar.baz_qux", b"a"] and F("\u3000 \u2028".encode()) == []
    assert F(b"FooBar") == [b"_foo_bar"] and F(b"foo_bar") == F(b"a.1b") == F(b"a,") == F(b"a..b") == T.INVALID_VALUE
    assert F(b"a1.b2") == [b"a1.b2"] and F(" a ".encode()) == [b"a"]
    assert T.value(T.TS, b"null") is None and T.value(T.TS, b"null", element=True) == T.SYNTAX
    assert T.value(T.wrapper("int32"), b"null", element=True) == T.INVALID_VALUE and T.value(T.EMPTY, b"[]") == T.SYNTAX
    assert T.payload(T.wrapper("double"), T.value(T.wrapper("double"), b"-0")) == b"\x09" + b"\x00" * 7 + b"\x80"
    assert T.payload(T.DUR, (-1, -5)) == b"\x08" + b"\xff" * 9 + b"\x01\x10" + b"\xfb" + b"\xff" * 8 + b"\x01"
    W = lambda *fs: b"".join(fs)
    assert T.decode("google.protobuf.Timestamp", b"") == b'"1970-01-01T00:00:00Z"'
    assert T.decode("google.protobuf.Timestamp", W(b"\x08\x01", b"\x10\x85\x80\x80\x80\x10")) == b'"1970-01-01T00:00:01.000000005Z"'
    assert T.decode("google.protobuf.Timestamp", b"\x10\xff\xff\xff\xff\x0f") == T.RANGE  # nanos int32(v) = -1
    assert T.decode("google.protobuf.Timestamp", b"\x10\x80\x94\xeb\xdc\x03") == T.RANGE  # nanos 10^9
    assert T.decode("google.protobuf.Timestamp", b"\x10\x80\xc2\xd7\x2f") == b'"1970-01-01T00:00:00.100Z"'
    assert T.decode("google.protobuf.Duration", W(b"\x08\x01", b"\x10\xff\xff\xff\xff\x0f")) == T.RANGE  # signs differ
    assert T.decode("google.protobuf.Duration", W(b"\x08\xfe\xff\xff\xff\xff\xff\xff\xff\xff\x01", b"\x10\x80\x82\xb8\x20")) == T.RANGE
    assert T.decode("google.protobuf.Duration", b"\x10" + T.intref.varint(-10 ** 7)) == b'"-0.010s"'
    assert T.decode("google.protobuf.FieldMask", b"\x0a\x07foo_bar\x0a\x01a") == b'"fooBar,a"'
    assert T.decode("google.protobuf.FieldMask", b"\x0a\x06fooBar") == T.INVALID_VALUE  # irreversible
    assert T.decode("google.protobuf.FieldMask", b"\x0a\x01\xff") == T.INVALID_UTF8
    assert T.decode("google.protobuf.Timestamp", b"\x0b\x08\x01\x0c\x08\x02") == b'"1970-01-01T00:00:02Z"'  # group skipped
    assert T.decode("google.protobuf.Timestamp", b"\x0c") == T.BAD_WIRE
    # a oneof sibling between two pieces of o_ts: the member starts afresh
    assert T.decode("wkt.Times", b"\x4a\x02\x08\x05\x62\x00\x4a\x02\x10\x07") == b'{"oTs":"1970-01-01T00:00:00.000000007Z"}'
    assert T.decode("wkt.Times", b"\x0a\x02\x08\x05\x0a\x02\x10\x07", 1) == b'{"ts":"1970-01-01T00:00:05.000000007Z"}'
    # a Marshal-time range error is reported only when the whole item reads
    assert T.decode("wkt.Times", b"\x0a\x07\x08\x80\x80\x80\x80\x80\x08") == T.RANGE
    assert T.decode("wkt.Times", b"\x0a\x07\x08\x80\x80\x80\x80\x80\x08\x08") == T.BAD_WIRE


def test_days_against_datetime():
    """timeref's own day arithmetic against datetime.date.toordinal on every day of years 1..9999"""
    base = T.days_from_civil(1, 1, 1) - 1
    d = datetime.date(1, 1, 1)
    one = datetime.timedelta(days=1)
    bad = []
    while True:
        if T.days_from_civil(d.year, d.month, d.day) - base != d.toordinal():
            bad.append(d)
        if d == datetime.date.max:
            break
        d += one
    assert not bad, bad[:5]
    assert T.days_from_civil(1970, 1, 1) == 0 and T.days_from_civil(0, 12, 31) * 86400 + 86399 == T.MIN_TS - 1
    assert sum(T.days_in(m, 0) for m in range(1, 13)) == 366 and T.days_in(2, 1900) == 28


# ---- the oracle --------------------------------------------------------------------------------------------------
def test_oracle_requests(oracle_t):
    bad = []
    for name, _, js, want, _ in _corpus()["req"]:
        st, wire, _ = oracle_t.encode(name, js)
        if not _matches(st, wire, want):
            bad.append((js[:150], st, want if isinstance(want, str) else want.hex()[:60], wire.hex()[:60]))
    assert not bad, (len(bad), bad[:8])


def test_oracle_replies(oracle_t):
    bad = []
    for name, _, w, t0, t1 in _corpus()["rep"]:
        for fl, want in ((0, t0), (1, t1)):
            st, js, _ = oracle_t.decode(name, w, fl)
            if not _matches(st, js, want):
                bad.append((fl, w[:40].hex(), st, js[:150], want[:150]))
    assert not bad, (len(bad), bad[:5])


def test_oracle_bodies(oracle_t):
    """tools/call bodies of EchoTimes: timeref's wire; never rc 0 for a value timeref refuses"""
    bad = []
    for _, body, want in _corpus()["bodies"]:
        r = oracle_t.request(body)
        ok = r["kind"] != 0 if isinstance(want, str) else (r["kind"] == 0 and r["wire"] == want)
        if not ok:
            bad.append((body[90:200], r["kind"], r["status"], r["wire"].hex()))
    assert not bad, (len(bad), bad[:5])


# ---- host simulation: every entry point --------------------------------------------------------------------------
def _offs(i, s):
    return s, (i * 5) % 16


def test_hostsim_encode(hsim_t):
    """the per-thread parser takes every item"""
    bad = []
    for i, (name, s, js, want, gap) in enumerate(_corpus()["req"]):
        st, out = hsim_t.encode(name, js, *_offs(i, s))
        if not _matches(st, out, want, gap):
            bad.append((js[:150], st, want if isinstance(want, str) else want.hex()[:80], out.hex()[:80]))
    assert not bad, (len(bad), bad[:5])


def test_fieldmask_escape_gap(hsim_t):
    """a FieldMask written with escapes gives exactly GGR_ST_UNSUPPORTED, in every position; the same text without
    escapes is answered"""
    gaps = [it for it in _corpus()["req"] if it[4]]
    assert len(gaps) == 198
    assert all(hsim_t.encode(name, js)[0] == T.STATUS[T.UNSUPPORTED] for name, _, js, _, _ in gaps)
    plain = [it for it in _corpus()["req"] if not it[4] and b"fm" in it[2].lower() and not isinstance(it[3], str)]
    assert len(plain) >= 138 and all(hsim_t.encode(name, js)[0] == 0 for name, _, js, _, _ in plain)


def _taken(run, items, idx, want_of):
    bad, taken = [], []
    for i in idx:
        st, out = run(i)
        if st == LEFT:
            continue
        if not _matches(st, out, want_of(i), items[i][4] is True):  # request items: the escape gap
            w = want_of(i)
            bad.append((items[i][2][:150], st, out[:150], w if isinstance(w, str) else w[:150]))
        if st == 0:
            taken.append(i)
    assert not bad, (len(bad), bad[:5])
    return taken


def _is_ts(it):
    """a request item with a Timestamp value"""
    if it[0] == "google.protobuf.Timestamp":
        return it[2] not in (b"", b"{}")
    return any(b'"%s":' % k in it[2] for k in (b"ts", b"r_ts", b"m_ts", b"m_i64_ts", b"o_ts")) and b":null" not in it[2]


# valid items each lock-step request tier takes, pinned on this corpus (all, and those with a Timestamp): the lock-step
# parser's two tiers (separate entry points), and what each walker tier adds over the tiers before it
_REQ_FLOORS = {"coop0": (975, 947), "coop1": (976, 948), "walk1": (28, 0), "walk2": (407, 407), "walk3": (2, 2)}
_MAP_TS_FLOOR = 135  # items with a Timestamp map value the lock-step parser takes (its ce_walk_map Timestamp branch)
# the lock-step reply tiers: the first, and what the pooled second one adds (all, and those with a Timestamp)
_REP_FLOORS = ((60, 43), (2, 2))


def _count(req, idx):
    return len(idx), sum(1 for i in idx if _is_ts(req[i]))


@pytest.mark.parametrize("tier", [0, 1])
def test_hostsim_encode_coop(hsim_t, tier):
    """the lock-step parser: exact bytes and status, or left (200); never rc 0 for an item timeref refuses"""
    req = _corpus()["req"]
    run = lambda i: hsim_t.encode_coop(req[i][0], req[i][2], *_offs(i, req[i][1]), tier=tier)
    taken = _taken(run, req, range(len(req)), lambda i: req[i][3])
    got = _count(req, taken)
    maps = sum(1 for i in taken if b'"m_ts"' in req[i][2] or b'"m_i64_ts"' in req[i][2])
    assert all(g >= w for g, w in zip(got, _REQ_FLOORS["coop%d" % tier])) and maps >= _MAP_TS_FLOOR, (got, maps)


def test_hostsim_encode_walk(hsim_t, monkeypatch):
    """the token-parallel walker, whole and stopped after its first and second tier"""
    req = _corpus()["req"]
    run = lambda i: hsim_t.encode_walk(req[i][0], req[i][2], *_offs(i, req[i][1]))
    _stop_at(monkeypatch)
    full = _taken(run, req, range(len(req)), lambda i: req[i][3])
    _stop_at(monkeypatch, "HS_WALK_TIER2_ONLY")
    upto2 = _taken(run, req, full, lambda i: req[i][3])
    _stop_at(monkeypatch, "HS_WALK_TIER1_ONLY")
    upto1 = _taken(run, req, upto2, lambda i: req[i][3])
    s1, s2 = set(upto1), set(upto2)
    got = (_count(req, upto1), _count(req, [i for i in upto2 if i not in s1]), _count(req, [i for i in full if i not in s2]))
    assert got[0][1] == 0, "the walker's first tier leaves Timestamps"
    for g, w in zip(got, (_REQ_FLOORS["walk1"], _REQ_FLOORS["walk2"], _REQ_FLOORS["walk3"])):
        assert g[0] >= w[0] and g[1] >= w[1], got


@pytest.mark.parametrize("tier", [0, 1])
def test_hostsim_request_envelope(hsim_t, tier):
    """tools/call bodies of EchoTimes through the lock-step parser: timeref's wire, or left"""
    bad = []
    handled = 0
    for i, (s, body, want) in enumerate(_corpus()["bodies"]):
        rc, wire, method, idt = hsim_t.request_coop(body, s, (i * 3) % 16, tier)
        if rc == LEFT:
            continue
        if isinstance(want, str) or rc != 0 or wire != want:
            bad.append((body[90:200], rc, wire.hex()[:80], want if isinstance(want, str) else want.hex()))
        handled += 1
    assert not bad, (len(bad), bad[:5])
    assert handled >= 410, handled


@pytest.mark.parametrize("flags", [0, 1])
def test_hostsim_decode(hsim_t, flags):
    """the per-thread reply kernels take every item"""
    bad = []
    for i, (name, s, w, t0, t1) in enumerate(_corpus()["rep"]):
        want = t1 if flags else t0
        st, out = hsim_t.decode(name, w, flags, *_offs(i, s))
        if not _matches(st, out, want):
            bad.append((w[:60].hex(), st, out[:150], want[:150]))
    assert not bad, (len(bad), bad[:5])


def test_hostsim_decode_lockstep(hsim_t, monkeypatch):
    """the lock-step reply tiers, whole and stopped after the first"""
    rep = _corpus()["rep"]
    run = lambda i: hsim_t.decode_coop(rep[i][0], rep[i][2], i & 1, *_offs(i, rep[i][1]))
    want_of = lambda i: rep[i][4] if i & 1 else rep[i][3]
    _stop_at(monkeypatch)
    full = _taken(run, rep, range(len(rep)), want_of)
    _stop_at(monkeypatch, "HS_COOP_TIER1_ONLY")
    upto1 = _taken(run, rep, full, want_of)
    s1 = set(upto1)
    # items that start with a Timestamp field of wkt.Times, and Timestamp roots
    ts = lambda idx: sum(1 for i in idx if rep[i][0] == "google.protobuf.Timestamp"
                         or rep[i][0] == TC.TM and rep[i][2][:1] and rep[i][2][0] >> 3 in (1, 2, 3, 4, 9))
    got = ((len(upto1), ts(upto1)), (len(full) - len(upto1), ts([i for i in full if i not in s1])))
    assert all(g[0] >= w[0] and g[1] >= w[1] for g, w in zip(got, _REP_FLOORS)), got
