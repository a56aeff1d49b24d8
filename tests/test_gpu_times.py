"""GPU tests of Timestamp, Duration, FieldMask, wrapper and Empty values against the exact reference (timeref), on every
engine path: the corpus of tests/timecorpus.py shuffled, each item once at the start offset (mod 16) it was built for
and twice more wherever it lands, through encode_batch, decode_batch (flags 0 and GGR_F_COMMA_SPACE), request_batch
on EchoTimes bodies and decode_wrap_batch, and once per direction through the device-resident entry point on a
caller's stream.  Expected answers come from timeref only (a FieldMask written with escapes: GGR_ST_UNSUPPORTED); the
oracle's agreement with it is tested on the CPU (tests/test_times.py).  The schema is the fixture with wkt.Times
appended, registered on each engine by this module."""
import random

import numpy as np
import pytest

import timecorpus as TC
import timeref as T
from test_gpu_strings import _fill
from test_strings import ID, _result_body

pytestmark = pytest.mark.gpu

_cache = {}


def _corpus():
    if not _cache:
        _cache["req"] = TC.request_items()
        _cache["bodies"] = TC.body_items()
        _cache["rep"] = TC.reply_items()
    return _cache


@pytest.fixture(scope="module")
def times_schema(engine):
    return engine.register(TC.extended_fds())


def _plan(items, request, seed):
    """[(index into items or -1 for a filler, data)]: shuffled, each item at its own start offset and twice more"""
    rng = random.Random(seed)
    order = [(i, c) for i in range(len(items)) for c in range(3)]
    rng.shuffle(order)
    plan, pos = [], 0
    for i, c in order:
        data = items[i][2]
        if c == 0:
            fill = 2 + (items[i][1] - (pos + 2)) % 16
            plan.append((-1, _fill(fill, request)))
            pos += fill
            assert pos % 16 == items[i][1]
        plan.append((i, data))
        pos += len(data)
    return plan


def _ids(schema, plan, items):
    # fillers are bench.All items (an empty object / zero-valued occurrences of f_int32 and custom)
    return np.array([schema.message(items[i][0] if i >= 0 else "bench.All") for i, _ in plan], np.int32)


def _want_req(it):
    return T.UNSUPPORTED if it[4] else it[3]


def _check(plan, items, st, outs, want_of, filler_want):
    bad = []
    for k, (i, _) in enumerate(plan):
        got = (int(st[k]), outs[k])
        if i < 0:
            if got != (0, filler_want):
                bad.append(("filler", got))
            continue
        want = want_of(items[i])
        ok = got[0] == T.STATUS[want] if isinstance(want, str) else got == (0, want)
        if not ok:
            bad.append((items[i][2][:150], got[0], got[1][:150], want if isinstance(want, str) else want[:150]))
    assert not bad, (len(bad), bad[:4])


def test_time_requests(engine, times_schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["req"]
    plan = _plan(items, True, 21)
    data, off = pack([d for _, d in plan])
    out, ooff, st = engine.encode_batch(times_schema, _ids(times_schema, plan, items), data, off)
    _check(plan, items, st, unpack(out, ooff), _want_req, b"")


@pytest.mark.parametrize("flags", [0, 1])
def test_time_replies(engine, times_schema, flags):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["rep"]
    plan = _plan(items, False, 22 + flags)
    data, off = pack([d for _, d in plan])
    out, ooff, st = engine.decode_batch(times_schema, _ids(times_schema, plan, items), data, off, flags=flags)
    _check(plan, items, st, unpack(out, ooff), lambda it: it[4] if flags else it[3], b"{}")


def test_time_bodies(engine, times_schema):
    """EchoTimes bodies: timeref's wire; never rc 0 for a value timeref refuses.  Request bodies have nothing behind the
    lock-step parser, which leaves Durations: a valid Duration body is GGR_ST_UNSUPPORTED, a Timestamp body is answered"""
    from ggrmcp_b200.engine import pack
    bodies = _corpus()["bodies"] * 3
    random.Random(24).shuffle(bodies)
    data, off = pack([b for _, b, _ in bodies])
    out, ooff, method, span, st = engine.request_batch(times_schema, data, off)
    bad = []
    for k, (_, body, want) in enumerate(bodies):
        got = bytes(out[int(ooff[k]):int(ooff[k + 1])])
        s = int(st[k])
        left = s == T.STATUS[T.UNSUPPORTED] and b'"arguments":{"d":' in body
        ok = s != 0 if isinstance(want, str) else (s == 0 and got == want) or left
        if not ok:
            bad.append((body[90:200], s, got.hex()[:80]))
    assert not bad, (len(bad), bad[:4])


def test_time_results(engine, times_schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["rep"]
    plan = _plan(items, False, 25)
    data, off = pack([d for _, d in plan])
    idt, ioff = pack([ID] * len(plan))
    out, ooff, st = engine.decode_wrap_batch(times_schema, _ids(times_schema, plan, items), data, off, idt, ioff)
    want_of = lambda it: it[3] if isinstance(it[3], str) else _result_body(it[3], ID)
    _check(plan, items, st, unpack(out, ooff), want_of, _result_body(b"{}", ID))


@pytest.mark.parametrize("direction", ["req", "rep"])
def test_time_dev_on_caller_stream(engine, times_schema, direction):
    """encode_batch_dev / decode_batch_dev on a caller's stream, input read from device memory"""
    import torch
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()[direction]
    plan = _plan(items, direction == "req", 26)
    dev = torch.device("cuda", 0)
    data, off = pack([d for _, d in plan])
    n = len(plan)
    d_in = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_in[: len(data)] = torch.from_numpy(data.copy())
    d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
    d_msg = torch.from_numpy(_ids(times_schema, plan, items)).to(dev)
    cap = len(data) * 8 + 64 * n + 64
    d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_ooff = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
    d_st = torch.full((n,), -99, dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    fn = engine.encode_batch_dev if direction == "req" else engine.decode_batch_dev
    with torch.cuda.stream(stream):
        fn(times_schema, n, d_msg.data_ptr(), d_in.data_ptr(), d_off.data_ptr(), len(data), d_out.data_ptr(), cap,
           d_ooff.data_ptr(), d_st.data_ptr(), 0, stream.cuda_stream)
    stream.synchronize()
    ooff = d_ooff.cpu().numpy()
    outs = unpack(d_out[: int(ooff[-1])].cpu().numpy(), ooff)
    want_of = _want_req if direction == "req" else (lambda it: it[3])
    _check(plan, items, d_st.cpu().numpy(), outs, want_of, b"" if direction == "req" else b"{}")
