"""The lock-step kernels at their fixed capacities (tests/limits.py), on the host simulation: every item against the oracle on
the per-thread code and on every lock-step tier, and, per capacity, proof that the items sit on both sides of it - which
tier takes or leaves each one (the tier switches of hostsim.cc and its reason codes), or, where a kernel switches to a
second path inside itself, the count or size that decides the path.  The GPU run of the same corpus is
tests/test_gpu_limits.py."""
import json

import pytest

import cases
import limits as LM

_corpus = {}

REPLY_ROWS = ["R1", "R2", "R3", "R4", "R5", "R6", "R7", "R8"]
REQUEST_ROWS = ["W0", "W1", "W2", "W3", "W4", "W5", "W6", "W7", "W8", "W10"]
_TIER_ENV = ("HS_COOP_TIER1_ONLY", "HS_WALK_TIER1_ONLY", "HS_WALK_TIER2_ONLY")


def _items(oracle, row):
    if not _corpus:
        _corpus["rep"], _corpus["req"] = LM.corpus(oracle)
    got = [it for it in _corpus["rep" if row[0] == "R" else "req"] if it.limit_id == row]
    assert {it.side for it in got if not it.damaged} == {"below", "at", "above"}, row
    return got


def _tier(monkeypatch, name=None):
    for k in _TIER_ENV:
        monkeypatch.delenv(k, raising=False)
    if name:
        monkeypatch.setenv(name, "1")


def _why(hsim):
    import hostsim
    return hostsim.lib().hs_cw_why()


def _depth_gap(it, ost, est):
    """nesting beyond the per-thread code's frames: GGR_ST_DEPTH where the oracle answers (DESIGN.md section 6), for items
    nested past that limit only"""
    return est == 8 and ost == 0 and LM.past_frames(it)


def _check_frames(oracle, items, per_thread):
    """the per-thread code answers at the deepest nesting it takes, with the oracle's bytes, and GGR_ST_DEPTH one level
    deeper; `per_thread(it)` -> (status, bytes)"""
    seen = set()
    for it in items:
        d = LM.nesting(it)
        if it.damaged or d is None:
            continue
        last = LM.pt_depth_last(it)
        ost, ob = oracle.decode(it.message, it.data)[:2] if it.limit_id[0] == "R" else oracle.encode(it.message, it.data)[:2]
        est, eb = per_thread(it)
        assert ost == 0, (it[:3], d)
        assert (est, eb) == ((0, ob) if d <= last else (8, b"")), (it[:3], d, last, est)
        seen.add((last, d - last))
    assert {(last, 0) for last, _ in seen} | {(last, 1) for last, _ in seen} <= seen, seen


# ---- reply side ------------------------------------------------------------------------------------------------
def _strings(name, wire):
    """(kind, text or bytes) of every string and bytes field of a reply, recursively"""
    import pbgen
    from google.protobuf.descriptor import FieldDescriptor as FD
    m = pbgen.cls(name)()
    m.ParseFromString(wire)
    out = []

    def walk(msg):
        for fd, v in msg.ListFields():
            vals = v if LM._repeated(fd) else [v]
            for x in vals:
                if fd.type == FD.TYPE_MESSAGE:
                    walk(x)
                elif fd.type in (FD.TYPE_STRING, FD.TYPE_BYTES):
                    out.append((fd.type, x))
    walk(m)
    return out


def _dirty(s):
    return any(c in '"\\' or ord(c) < 0x20 or ord(c) >= 0x80 for c in s)


def _n_dirty(name, wire):
    from google.protobuf.descriptor import FieldDescriptor as FD
    return sum(1 for t, x in _strings(name, wire) if t == FD.TYPE_STRING and _dirty(x))


def _n_long(name, wire):
    """entries of the writer's hand-off list: plain strings and bytes of at least GGR_COOP_LONG bytes, strings that need
    escaping"""
    from google.protobuf.descriptor import FieldDescriptor as FD
    n = 0
    for t, x in _strings(name, wire):
        if t == FD.TYPE_BYTES:
            n += len(x) >= LM.COOP_LONG
        else:
            n += _dirty(x) or len(x.encode()) >= LM.COOP_LONG
    return n


def _reply_parity(oracle, hsim, it, i, flags, io=None):
    """per-thread and lock-step reply code against the oracle; returns the lock-step rc (0 taken, 200 left)"""
    io = i % 16 if io is None else io
    oo = (i * 5 + flags) % 16
    ost, oj, _ = oracle.decode(it.message, it.data, flags)
    est, ej = hsim.decode(it.message, it.data, flags, io, oo)
    if not _depth_gap(it, ost, est):
        assert cases.status_compatible(ost, est), (it[:3], ost, est)
        if ost == 0:
            assert ej == oj, (it[:3], flags)
    rc, out = hsim.decode_coop(it.message, it.data, flags, io, oo)
    assert rc in (0, 200), (it[:3], rc)
    if rc == 0:
        assert ost == 0 and out == oj, (it[:3], flags, io, len(oj), len(out))
    return rc


@pytest.mark.parametrize("row", REPLY_ROWS)
def test_reply_limits(oracle, hsim, monkeypatch, row):
    items = _items(oracle, row)
    _tier(monkeypatch)
    for i, it in enumerate(items):
        for flags in (0, 1):
            if row == "R3":  # the limit is on the item's end: start offsets 0 and 15
                rcs = [_reply_parity(oracle, hsim, it, i, flags, io) for io in (0, 15)]
            else:
                rcs = [_reply_parity(oracle, hsim, it, i, flags)]
            if it.damaged:
                continue
            taken = all(rc == 0 for rc in rcs)
            if row in ("R2", "R8"):  # the second tier / the lock-step depth leaves the item to the per-thread kernels
                assert taken == (it.side != "above"), (row, it.side, len(it.data), rcs)
            else:  # R1 (the second tier takes what the first leaves), R3..R7: a second path inside the same kernel
                assert taken, (row, it.side, len(it.data), rcs)
    real = [it for it in items if not it.damaged]
    if row == "R1":
        _tier(monkeypatch, "HS_COOP_TIER1_ONLY")
        for i, it in enumerate(items):
            if not it.damaged:
                assert (_reply_parity(oracle, hsim, it, i, 0) == 0) == (it.side != "above"), (it.side, len(it.data))
    if row == "R2":
        _tier(monkeypatch, "HS_COOP_TIER1_ONLY")
        assert all(_reply_parity(oracle, hsim, it, i, 0) == 200 for i, it in enumerate(items) if not it.damaged)
    # the count or size that decides the path, on the side the corpus says
    for it in real:
        if row in ("R1", "R2"):
            n_ent = 1 + len(it.data) // 2  # the root and one entry per empty child
            cap = LM.COOP_ENTRIES if row == "R1" else LM.COOP_BIG_ENTRIES
            assert (n_ent <= cap) == (it.side != "above") and (it.side != "at" or n_ent == cap)
        elif row == "R3":
            assert (len(it.data) <= LM.COOP_MAX_WIRE) == (it.side != "above")
        elif row == "R4":
            n = _n_dirty(it.message, it.data)
            assert (n <= LM.DIRTY_MAX) == (it.side != "above") and (it.side != "at" or n == LM.DIRTY_MAX), (it.side, n)
        elif row == "R5":
            n = _n_long(it.message, it.data)
            assert (n <= LM.LONG_MAX) == (it.side != "above") and (it.side != "at" or n == LM.LONG_MAX), (it.side, n)
        elif row in ("R6", "R7"):
            lim = LM.STAGE_BUF if row == "R6" else 8192
            t0 = len(oracle.decode(it.message, it.data, 0)[1])
            assert (t0 <= lim) == (it.side != "above") and (it.side != "at" or t0 == lim), (it.side, t0)
    if row == "R6":  # the same wire on both sides of the staging buffer under the two flags
        t = [(len(oracle.decode(it.message, it.data, 0)[1]), len(oracle.decode(it.message, it.data, 1)[1])) for it in real]
        assert any(a <= LM.STAGE_BUF < b for a, b in t)
    if row == "R5":
        assert {LM.COOP_LONG - 1, LM.COOP_LONG, LM.COOP_LONG + 1} <= {len(x.encode()) if isinstance(x, str) else len(x)
                                                                     for it in real for _, x in _strings(it.message, it.data)}
    if row == "R8":
        _check_frames(oracle, items, lambda it: hsim.decode(it.message, it.data))
    assert any(it.damaged for it in items) or row in ("R5", "R6", "R7")


# ---- request side ----------------------------------------------------------------------------------------------
def _request_parity(oracle, hsim, it, i, io=None):
    """per-thread parser, walker and both lock-step parser tiers against the oracle; returns the walker's rc and why"""
    io = i % 16 if io is None else io
    oo = (i * 5) % 16
    ost, ow, _ = oracle.encode(it.message, it.data)
    est, ew = hsim.encode(it.message, it.data, io, oo)
    if not _depth_gap(it, ost, est):
        assert cases.status_compatible(ost, est) or (ost != 0 and est != 0 and {ost, est} <= {1, 3, 5}), (it[:3], ost, est)
        if ost == 0:
            assert ew == ow, it[:3]
    rc, out = hsim.encode_walk(it.message, it.data, io, oo)
    why = _why(hsim) if rc == 200 else 0
    assert rc in (0, 200), (it[:3], rc)
    if rc == 0:
        assert ost == 0 and out == ow, (it[:3], io)
    if len(it.data) <= 70000:
        for tier in (0, 1):
            crc, cout = hsim.encode_coop(it.message, it.data, io, oo, tier)
            assert crc in (0, 200), (it[:3], tier, crc)
            if crc == 0:
                assert ost == 0 and cout == ow, (it[:3], tier)
    return rc, why


def _n_handoff(js):
    """entries of the emitter's hand-off list: strings with two-character escapes, plain strings of at least CE_LONG_STR"""
    texts = []
    for v in json.loads(js).values():
        texts += v if isinstance(v, list) else [v]
    return sum(("\\" in json.dumps(t, ensure_ascii=False)) or len(t.encode()) >= LM.CE_LONG_STR for t in texts if isinstance(t, str))


@pytest.mark.parametrize("row", REQUEST_ROWS)
def test_request_limits(oracle, hsim, monkeypatch, row):
    items = _items(oracle, row)
    real = [it for it in items if not it.damaged]
    _tier(monkeypatch)
    res = {}
    for i, it in enumerate(items):
        if row == "W6":
            for io in (0, 15):
                rc, why = _request_parity(oracle, hsim, it, i, io)
                if not it.damaged:  # positions are 16 bits: the walker takes items of at most 64984 bytes at any offset
                    assert (rc == 0) == (len(it.data) <= LM.REQ_ITEM_MAX), (len(it.data), io, rc, why)
                    assert rc == 0 or why == 1
            continue
        res[i] = _request_parity(oracle, hsim, it, i)
    full = {i: res[i] for i, it in enumerate(items) if not it.damaged and i in res}
    side = {i: items[i].side for i in full}
    if row in ("W0", "W3", "W4"):  # every walker tier leaves the item
        code = {"W0": 4, "W3": 2, "W4": 102}[row]
        for i, (rc, why) in full.items():
            assert (rc == 0) == (side[i] != "above"), (row, side[i], len(items[i].data), rc, why)
            assert rc == 0 or why == code, (row, side[i], why)
    if row == "W5":  # Node.children through the walker, bench.All.recursive through the lock-step parser
        for i, it in enumerate(items):
            if it.damaged:
                continue
            if it.message == LM.PNR:
                assert (full[i][0] == 0) == (it.side != "above"), (it.side, it.data.count(b"["))
            else:
                for tier in (0, 1):
                    assert (hsim.encode_coop(it.message, it.data, 0, 0, tier)[0] == 0) == (it.side != "above"), (it.side, tier)
        _check_frames(oracle, items, lambda it: hsim.encode(it.message, it.data))
    if row in ("W1", "W2"):
        for i in full:
            assert full[i][0] == 0, (row, side[i])  # the next tier takes what this one leaves
        _tier(monkeypatch, "HS_WALK_TIER1_ONLY" if row == "W1" else "HS_WALK_TIER2_ONLY")
        for i in full:
            it = items[i]
            rc, why = _request_parity(oracle, hsim, it, i)
            assert (rc == 0) == (it.side != "above") and (rc == 0 or why == 2), (row, it.side, rc, why)
    if row == "W7":
        for i in full:
            assert full[i][0] == 0, side[i]
        _tier(monkeypatch, "HS_WALK_TIER1_ONLY")
        for i in full:
            it = items[i]
            rc, why = _request_parity(oracle, hsim, it, i)
            n = len(oracle.encode(it.message, it.data)[1])
            assert (rc == 0) == (n <= LM.CE_STAGE) == (it.side != "above"), (n, rc, why)
            assert rc == 0 or why == 10
        sizes = {len(oracle.encode(it.message, it.data)[1]) for it in real}
        assert {LM.CE_STAGE_BUF - 1, LM.CE_STAGE_BUF, LM.CE_STAGE_BUF + 1, LM.CE_STAGE, LM.CE_STAGE + 1} <= sizes
    if row == "W8":
        for i in full:
            assert full[i][0] == 0, side[i]
            n = _n_handoff(items[i].data)
            assert (n <= LM.CE_LONG_MAX) == (side[i] != "above") and (side[i] != "at" or n == LM.CE_LONG_MAX), (side[i], n)
    if row == "W10":
        for i in full:
            it = items[i]
            assert full[i][0] == 200 and full[i][1] == 1
            assert (len(it.data) <= LM.TOO_LARGE) == (it.side != "above")
    if row in ("W1", "W2", "W3", "W4", "W5", "W6", "W8"):
        assert any(it.damaged for it in items)
