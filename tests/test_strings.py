"""String and bytes text against the exact reference (strref): the oracle on the whole corpus of tests/strcorpus.py in
both directions, tools/call bodies and result bodies, then every entry point of the host simulation.  Each item gives
exactly strref's bytes and status category, or (lock-step entry points only) is left to the per-thread kernels with
rc 200; a lock-step tier never answers rc 0 for an item strref refuses."""
import collections

import pytest

import strcorpus as SC
import strref as S

LEFT = 200  # a lock-step entry point leaves the item to the per-thread kernels
ID = b'"i<d>"'

_cache = {}


def _corpus():
    if not _cache:
        req = SC.request_items()
        _cache["req"] = req + SC.request_bytes_items()
        _cache["bodies"] = SC.body_items(req)
        _cache["rep"] = SC.reply_items()
        _cache["wrap"] = SC.wrap_texts()
    return _cache


def _matches(st, out, want):
    """status and bytes against a reference answer (bytes, or a status category)"""
    if isinstance(want, str):
        return st == S.STATUS[want]
    return st == 0 and out == want


def _result_body(text, idt):
    return b'{"jsonrpc":"2.0","result":{"content":[{"type":"text","text":' + S.html_string(text) + b'}]},"id":' + idt + b"}\n"


def test_corpus_shape():
    """the corpus reaches what it exists for: every event on both sides of every edge, start offsets 0..15, every
    length of base64 text mod 4, failing and passing items in each direction (pinned counts)"""
    c = _corpus()
    req, rep = c["req"], c["rep"]
    assert (len(req), len(c["bodies"]), len(rep), len(c["wrap"])) == (4583, 118, 3002, 781)
    assert {s for _, s, _, _ in req} == set(range(16)) == {s for _, s, _, _, _ in rep}
    cats = collections.Counter(w if isinstance(w, str) else "ok" for *_, w in req)
    assert cats == {"ok": 2143, S.SYNTAX: 860, S.INVALID_UTF8: 1214, S.INVALID_VALUE: 366}, cats
    cats = collections.Counter(w if isinstance(w, str) else "ok" for *_, w, _ in rep)
    assert cats == {"ok": 1639, S.INVALID_UTF8: 1363}, cats
    # the offset sweep puts each event on every byte position of a 16-byte chunk, in rebased bytes
    for j in range(len(SC.REQ_EVENTS)):
        k0 = j * (34 + 4 * len(SC.REQ_EDGES))
        heads = [SC._head_len("frmk"[(k0 + off) % 4]) for off in range(34)]
        assert {(SC.start_offset(k0 + off, off, h) + h + off) % 16 for off, h in enumerate(heads)} == set(range(16))
    assert max(len(js) for _, _, js, _ in req) > 8192 and max(len(w) for _, _, w, _, _ in rep) > 20000


def test_strref_rules():
    """strref on hand-checked cases of each rule"""
    P = S.parse_string
    assert P(b"a\\u00e9\\ud83d\\ude00\\/") == "a\u00e9\U0001F600/".encode()
    assert P(b"\\uD83D\\uDE00") == "\U0001F600".encode()
    for bad in (b"\\ud83d", b"\\ude00", b"\\ud83dx", b"\\ud83d\\u0041", b"\\ud83d\\ud83d", b"\\x", b"\\u12", b"\\", b"a\nb"):
        assert P(bad) == S.SYNTAX, bad
    for bad in (b"\xc0\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\x80", b"\xe2\x82", b"\xff"):
        assert P(bad) == S.INVALID_UTF8, bad
    assert P(b"\\x\xff") == S.SYNTAX and P(b"\xff\\x") == S.INVALID_UTF8  # the first problem from the left
    assert S.format_string(b'\x00\x1f"\\\x7f\n') == b'"\\u0000\\u001f\\"\\\\\x7f\\n"'
    assert S.format_string(b"\xed\xa0\x80") == S.INVALID_UTF8
    assert S.html_string("<\u2028&".encode()) == b'"\\u003c\\u2028\\u0026"'
    B = S.b64_parse
    assert B(b"QR==") == b"A" and B(b"QR") == b"A" and B(b"QR=") == S.INVALID_VALUE and B(b"Q") == S.INVALID_VALUE
    assert B(b"aGVs\nbG8=") == S.INVALID_VALUE  # length 9 before \n is skipped: no padding expected
    assert B(b"aGVs\r\nbG8") == b"hello" and B(b"aGVs\nbG8") == S.INVALID_VALUE  # 8 bytes: padding expected
    assert B(b"aGVsbG8=\n") == S.INVALID_VALUE and B(b"aGVs\nbG8=\n\n\n") == b"hello"
    assert B(b"-_-_") == b"\xfb\xff\xbf" and B(b"-/+_") == S.INVALID_VALUE and B(b"YQ==YQ==") == S.INVALID_VALUE
    assert S.body_value(b"a\xffb") == ("a\ufffdb".encode(), False)
    assert S.body_value(b"\xe2\x82A") == ("\ufffd\ufffdA".encode(), False)  # one U+FFFD per byte, as encoding/json
    assert S.body_value(b"\\ud800\\ud83d\\ude00") == ("\ufffd\U0001F600".encode(), False)
    assert S.body_value(b"\\x") == (S.SYNTAX, True) and S.body_value(b"ok") == (b"ok", True)


# ---- the oracle --------------------------------------------------------------------------------------------------
def test_oracle_requests(oracle):
    bad = []
    for name, _, js, want in _corpus()["req"]:
        st, wire, _ = oracle.encode(name, js)
        if not _matches(st, wire, want):
            bad.append((js[:150], st))
    assert not bad, (len(bad), bad[:5])


def test_oracle_replies(oracle):
    bad = []
    for name, _, w, t0, t1 in _corpus()["rep"]:
        for fl, want in ((0, t0), (1, t1)):
            st, js, _ = oracle.decode(name, w, fl)
            if not _matches(st, js, want):
                bad.append((fl, w[:100], st, js[:150]))
    assert not bad, (len(bad), bad[:5])


def test_oracle_bodies_and_results(oracle):
    """tools/call bodies: the wire of strref's value after encoding/json's round trip, an error where encoding/json
    refuses the body; result bodies around the reply texts and the wrapper texts"""
    bad = []
    for _, body, want, ident in _corpus()["bodies"]:
        r = oracle.request(body)
        ok = r["kind"] != 0 if want == S.SYNTAX else (r["kind"] == 0 and r["wire"] == want)
        if not ok:
            bad.append((body[:200], r["kind"], r["status"], r["wire"].hex()))
    assert not bad, (len(bad), bad[:5])
    for name, _, w, t0, _ in _corpus()["rep"][::5]:
        if isinstance(t0, bytes):
            st, body = oracle.response(name, w, ID)
            assert st == 0 and body == _result_body(t0, ID), (w[:80], body[:200])


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


_TIER_STOPS = ("HS_WALK_TIER1_ONLY", "HS_WALK_TIER2_ONLY", "HS_COOP_TIER1_ONLY")


def _stop_at(monkeypatch, name=None):
    """the host simulation's tier switches: with `name` set, the chain of lock-step tiers ends at that tier"""
    for k in _TIER_STOPS:
        monkeypatch.delenv(k, raising=False)
    if name:
        monkeypatch.setenv(name, "1")


def _taken(run, items, idx, want_of):
    """indices in `idx` that `run` answers with rc 0; every answer other than 200 must match strref's, want_of(i)"""
    bad, taken = [], []
    for i in idx:
        st, out = run(i)
        if st == LEFT:
            continue
        if not _matches(st, out, want_of(i)):
            bad.append((items[i][2][:150], st, out[:150]))
        if st == 0:
            taken.append(i)
    assert not bad, (len(bad), bad[:5])
    return taken


# valid items each lock-step request tier takes, pinned on this corpus: the lock-step parser's two tiers (separate entry
# points), and what each walker tier adds over the tiers before it
_REQ_FLOORS = {"coop0": 2050, "coop1": 2097, "walk1": 402, "walk2": 529, "walk3": 46}


@pytest.mark.parametrize("tier", [0, 1])
def test_hostsim_encode_coop(hsim, tier):
    """the lock-step parser: exact bytes and status, or left (200); never rc 0 for an item strref refuses"""
    req = _corpus()["req"]
    run = lambda i: hsim.encode_coop(req[i][0], req[i][2], *_offs(i, req[i][1]), tier=tier)
    taken = _taken(run, req, range(len(req)), lambda i: req[i][3])
    assert len(taken) >= _REQ_FLOORS["coop%d" % tier], len(taken)


def test_hostsim_encode_walk(hsim, monkeypatch):
    """the token-parallel walker, whole and stopped after its first and second tier: exact bytes and status, or left
    (200); every tier takes valid items the tiers before it leave (a stopped chain takes a subset of the whole one)"""
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
    """tools/call bodies through the lock-step parser: strref's wire after the round trip, or left (200); a body whose
    round trip is not the identity may be left, never answered with other bytes"""
    bad = []
    handled = 0
    for i, (s, body, want, ident) in enumerate(_corpus()["bodies"]):
        rc, wire, method, idt = hsim.request_coop(body, s, (i * 3) % 16, tier)
        if rc == LEFT:
            continue
        if want == S.SYNTAX or rc != 0 or wire != want:
            bad.append((body[:200], rc, wire.hex()[:80]))
        handled += 1
    assert not bad, (len(bad), bad[:5])
    assert handled >= 47, handled  # every body whose round trip is the identity


@pytest.mark.parametrize("flags", [0, 1])
def test_hostsim_decode(hsim, flags):
    """the per-thread reply kernels (fast walk, and the slow walk for zLast in front of fString) take every item"""
    bad = []
    for i, (name, s, w, t0, t1) in enumerate(_corpus()["rep"]):
        want = t1 if flags else t0
        st, out = hsim.decode(name, w, flags, *_offs(i, s))
        if not _matches(st, out, want):
            bad.append((w[:100], st, out[:150], want[:150]))
    assert not bad, (len(bad), bad[:5])


def test_hostsim_decode_lockstep(hsim, monkeypatch):
    """the lock-step reply tiers, whole and stopped after the first: exact text and status, or left (200); the pooled
    second tier takes valid items (more table entries than the first tier's table) the first one leaves"""
    rep = _corpus()["rep"]
    run = lambda i: hsim.decode_coop(rep[i][0], rep[i][2], i & 1, *_offs(i, rep[i][1]))
    want_of = lambda i: rep[i][4] if i & 1 else rep[i][3]
    _stop_at(monkeypatch)
    full = _taken(run, rep, range(len(rep)), want_of)
    _stop_at(monkeypatch, "HS_COOP_TIER1_ONLY")
    upto1 = _taken(run, rep, full, want_of)
    got = (len(upto1), len(full) - len(upto1))
    assert got[0] >= 832 and got[1] >= 92, got


def test_hostsim_wrap():
    """result bodies around the reply texts and the wrapper texts (U+2028 / U+2029 straddling lanes)"""
    import hostsim
    texts = [t0 for *_, t0, _ in _corpus()["rep"] if isinstance(t0, bytes)] + _corpus()["wrap"]
    bad = []
    for t in texts:
        rc, out = hostsim.wrap(t, ID)
        if rc != 0 or out != _result_body(t, ID):
            bad.append((t[:100], rc, out[:200]))
    assert not bad, (len(bad), bad[:3])
