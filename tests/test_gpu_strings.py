"""GPU tests of string and bytes text against the exact reference (strref), on every engine path: the corpus of
tests/strcorpus.py shuffled, each item once at the start offset (mod 16) it was built for and twice more wherever it
lands, through encode_batch, decode_batch (flags 0 and GGR_F_COMMA_SPACE), request_batch on echoall bodies and
decode_wrap_batch, and once per direction through the device-resident entry point on a caller's stream.  Expected
answers come from strref only; the oracle's agreement with it is tested on the CPU (tests/test_strings.py)."""
import random

import numpy as np
import pytest

import strcorpus as SC
import strref as S
from test_strings import ID, _result_body

pytestmark = pytest.mark.gpu

UNSUPPORTED = 11
_cache = {}


def _corpus():
    if not _cache:
        req = SC.request_items()
        _cache["req"] = req + SC.request_bytes_items()
        _cache["bodies"] = SC.body_items(req)
        _cache["rep"] = SC.reply_items()
    return _cache


def _fill(n, request):
    """a filler item of n >= 2 bytes with an empty answer: '{ .. }' or f_int32 = 0 / empty custom occurrences"""
    if request:
        return b"{" + b" " * (n - 2) + b"}"
    k3 = n % 2
    return b"\xd2\x05\x00" * k3 + b"\x08\x00" * ((n - 3 * k3) // 2)


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


def _check(plan, items, st, outs, want_of, filler_want):
    bad = []
    for k, (i, _) in enumerate(plan):
        got = (int(st[k]), outs[k])
        if i < 0:
            if got != (0, filler_want):
                bad.append(("filler", got))
            continue
        want = want_of(items[i])
        ok = got[0] == S.STATUS[want] if isinstance(want, str) else got == (0, want)
        if not ok:
            bad.append((items[i][2][:150], got[0], got[1][:150], want if isinstance(want, str) else want[:150]))
    assert not bad, (len(bad), bad[:4])


def test_string_requests(engine, schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["req"]
    plan = _plan(items, True, 1)
    ids = np.full(len(plan), schema.message(SC.A), np.int32)
    data, off = pack([d for _, d in plan])
    out, ooff, st = engine.encode_batch(schema, ids, data, off)
    _check(plan, items, st, unpack(out, ooff), lambda it: it[3], b"")


@pytest.mark.parametrize("flags", [0, 1])
def test_string_replies(engine, schema, flags):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["rep"]
    plan = _plan(items, False, 2 + flags)
    ids = np.full(len(plan), schema.message(SC.A), np.int32)
    data, off = pack([d for _, d in plan])
    out, ooff, st = engine.decode_batch(schema, ids, data, off, flags=flags)
    _check(plan, items, st, unpack(out, ooff), lambda it: it[4] if flags else it[3], b"{}")


def test_string_bodies(engine, schema):
    """a body whose encoding/json round trip is not the identity may be refused (unsupported), never answered with
    other bytes; a body encoding/json refuses is never answered"""
    from ggrmcp_b200.engine import pack
    bodies = _corpus()["bodies"] * 3
    random.Random(4).shuffle(bodies)
    data, off = pack([b for _, b, _, _ in bodies])
    out, ooff, method, span, st = engine.request_batch(schema, data, off)
    bad = []
    for k, (_, body, want, ident) in enumerate(bodies):
        got = bytes(out[int(ooff[k]):int(ooff[k + 1])])
        s = int(st[k])
        if want == S.SYNTAX:
            ok = s != 0
        else:
            ok = (s == 0 and got == want) or (not ident and s == UNSUPPORTED)
        if not ok:
            bad.append((body[:200], s, got.hex()[:80]))
    assert not bad, (len(bad), bad[:4])


def test_string_results(engine, schema):
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()["rep"]
    plan = _plan(items, False, 5)
    ids = np.full(len(plan), schema.message(SC.A), np.int32)
    data, off = pack([d for _, d in plan])
    idt, ioff = pack([ID] * len(plan))
    out, ooff, st = engine.decode_wrap_batch(schema, ids, data, off, idt, ioff)
    outs = unpack(out, ooff)
    want_of = lambda it: it[3] if isinstance(it[3], str) else _result_body(it[3], ID)
    _check(plan, items, st, outs, want_of, _result_body(b"{}", ID))


@pytest.mark.parametrize("direction", ["req", "rep"])
def test_string_dev_on_caller_stream(engine, schema, direction):
    """encode_batch_dev / decode_batch_dev on a caller's stream, input read from device memory"""
    import torch
    from ggrmcp_b200.engine import pack, unpack
    items = _corpus()[direction]
    plan = _plan(items, direction == "req", 6)
    dev = torch.device("cuda", 0)
    data, off = pack([d for _, d in plan])
    n = len(plan)
    d_in = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_in[: len(data)] = torch.from_numpy(data.copy())
    d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
    d_msg = torch.full((n,), schema.message(SC.A), dtype=torch.int32, device=dev)
    cap = len(data) * 8 + 64 * n + 64
    d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_ooff = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
    d_st = torch.full((n,), -99, dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    fn = engine.encode_batch_dev if direction == "req" else engine.decode_batch_dev
    with torch.cuda.stream(stream):
        fn(schema, n, d_msg.data_ptr(), d_in.data_ptr(), d_off.data_ptr(), len(data), d_out.data_ptr(), cap, d_ooff.data_ptr(),
           d_st.data_ptr(), 0, stream.cuda_stream)
    stream.synchronize()
    ooff = d_ooff.cpu().numpy()
    outs = unpack(d_out[: int(ooff[-1])].cpu().numpy(), ooff)
    _check(plan, items, d_st.cpu().numpy(), outs, lambda it: it[3], b"" if direction == "req" else b"{}")
