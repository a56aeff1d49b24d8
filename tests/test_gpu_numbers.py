"""GPU tests of float and double text conversion against the exact reference (numref): request literals through
ggr_encode_batch, tools/call bodies through ggr_request_batch, reply bit patterns through ggr_decode_batch, on every
engine path.  Expected values come from numref only; the oracle's agreement with it is tested on the CPU."""
import numpy as np
import pytest

import numcorpus as NC
import numref

pytestmark = pytest.mark.gpu

_cache = {}


def _corpus():
    if not _cache:
        lits = NC.request_literals()
        _cache["req"] = NC.request_items(lits)
        _cache["bodies"] = NC.body_items(lits)
        _cache["rep"] = NC.reply_items(NC.reply_bits(64), NC.reply_bits(32))
    return _cache


def test_number_requests(engine, schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["req"]
    ids = np.array([schema.message(n) for n, _, _ in items], np.int32)
    data, off = pack([js for _, js, _ in items])
    out, ooff, st = engine.encode_batch(schema, ids, data, off)
    bad = []
    for i, (got, (n, js, want)) in enumerate(zip(unpack(out, ooff), items)):
        ok = int(st[i]) != 0 if want == numref.RANGE else (int(st[i]) == 0 and got == want)
        if not ok:
            bad.append((n, js[:120], int(st[i])))
    assert not bad, (len(bad), bad[:5])


def test_number_bodies(engine, schema):
    from ggrmcp_b200.engine import pack
    bodies = _corpus()["bodies"]
    data, off = pack([b for b, _ in bodies])
    out, ooff, method, id_span, st = engine.request_batch(schema, data, off)
    bad = []
    for i, (body, want) in enumerate(bodies):
        got = bytes(out[int(ooff[i]):int(ooff[i + 1])])
        ok = int(st[i]) != 0 if want == numref.RANGE else (int(st[i]) == 0 and got == want)
        if not ok:
            bad.append((body[:160], int(st[i]), got.hex()))
    assert not bad, (len(bad), bad[:5])


def test_number_replies(engine, schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["rep"]
    ids = np.array([schema.message(n) for n, _, _ in items], np.int32)
    data, off = pack([w for _, w, _ in items])
    out, ooff, st = engine.decode_batch(schema, ids, data, off)
    assert (st == 0).all(), np.nonzero(st)[0][:10]
    bad = [(i, want[:120], got[:120]) for i, (got, (_, _, want)) in enumerate(zip(unpack(out, ooff), items)) if got != want]
    assert not bad, (len(bad), bad[:3])
