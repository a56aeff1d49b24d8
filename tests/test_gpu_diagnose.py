"""ggr_encode_diagnose_batch[_dev]: the error detail of every failing item of a request batch in one call, checked item by
item against ggr_encode_diagnose on that item alone, against the oracle's wording, and on the device-buffer form behind
other request-side calls."""
import ctypes as C
import functools
import random
import re

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu

NAME = "com.example.complex.GetUserProfileRequest"
PROBES = [b'{"invalid_field":1}', b'{"user_id":"a",\n  "nope": {"x":[1,2]}}', b'{"user_id":"a","user_id":"b"}', b'{"user_id":5}',
          b'{"user_id" "a"}', b'{"user_id":"a"', b'{"user_id":"ok"}', b'{ "userId":"a", "user_id":"b"}']
MAX_ITEM = 0x1FFFF0  # 2 MiB - 16: the largest item the per-thread parser takes


def late_item():
    """one item of about 2 MiB, one value per line, with an unknown field on its last line"""
    head, tail = b'{"r_int32":[', b'0],\n  "nope_late":1}'
    k = (MAX_ITEM - len(head) - len(tail)) // 3
    return head + b"".join(b"%d,\n" % (i % 10) for i in range(k)) + tail


def damaged(rng):
    out = []
    for k in range(40):
        out += [(cases.A, b'{"zz_%d":1}' % k), (cases.A, b'{"f_int32":%d,"f_int32":%d}' % (k, k + 1)),
                (cases.A, b'{"o_int32":%d,\n"o_string":"x"}' % k), (cases.A, b'{"f_int32":"x%d"}' % k),
                (cases.A, b'{"f_string":"a\xff%d"}' % k), (cases.A, b'{"f_msg":' * (k + 90) + b"{}" + b"}" * (k + 90)),
                (cases.A, b'{"f_str\\"ing":1}'), (cases.A, b'{"f_string":"\\' + b"\\" * k)]
    for n, j in cases.random_encode_cases(12, seed0=1900):
        i = rng.randrange(1, max(2, len(j)))
        out += [(n, j[:i]), (n, j[:i] + b"\n\xc3(" + j[i:]), (n, b'{\n"zz":' + j + b"}")]
    return out


@functools.lru_cache(maxsize=None)
def corpus():
    rng = random.Random(21)
    items = [(NAME, p) for p in PROBES]
    items += [(n, cases.mutate_json(j, rng)) for n, j in cases.random_encode_cases(60, seed0=1300) for _ in range(5)]
    items += [(n, js) for n, js, _ in cases.ENCODE_EDGE]
    items += damaged(rng)
    items += cases.random_encode_cases(10, seed0=1700)
    rng.shuffle(items)
    items.insert(len(items) // 2, (cases.A, late_item()))
    return items


def _pack(schema, items):
    from ggrmcp_b200.engine import pack
    ids = np.array([schema.message(n) for n, _ in items], np.int32)
    data, off = pack([b for _, b in items])  # back to back: every start offset mod 16 occurs
    return ids, data, off


def _single(engine, schema, msg_id, js):
    """ggr_encode_diagnose with room for any text: (status, err_pos, err_len, text)"""
    from ggrmcp_b200 import engine as E
    L = E._load()
    L.ggr_encode_diagnose.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
    st, pos, ln = C.c_int32(0), C.c_uint32(0), C.c_uint32(0)
    buf = C.create_string_buffer(len(js) + 256)
    rc = L.ggr_encode_diagnose(engine.h, schema.h, int(msg_id), bytes(js), len(js), 0, C.byref(st), C.byref(pos), C.byref(ln), buf, len(buf))
    assert rc == 0, rc
    return st.value, pos.value, ln.value, buf.value


@functools.lru_cache(maxsize=None)
def _batch_run(engine, schema):
    """the corpus through encode_batch and encode_diagnose_batch: (ids, data, off, status, err_pos, err_len, texts)"""
    items = corpus()
    ids, data, off = _pack(schema, items)
    _, _, st = engine.encode_batch(schema, ids, data, off)
    st = np.array(st, np.int32)
    pos, ln, texts = engine.encode_diagnose_batch(schema, ids, data, off, st)
    return ids, data, off, st, np.array(pos), np.array(ln), texts


def test_agrees_with_single_item_calls(engine, schema):
    items = corpus()
    ids, data, off, st, pos, ln, texts = _batch_run(engine, schema)
    failing = [i for i in range(len(items)) if st[i] != 0]
    assert len(items) >= 2000 and len(failing) >= 1000, (len(items), len(failing))
    assert len({int(off[i]) % 16 for i in failing}) == 16
    for i in failing:
        js = items[i][1]
        s1, p1, l1, t1 = _single(engine, schema, ids[i], js)
        assert s1 == st[i], (js[:200], s1, int(st[i]))
        assert (int(pos[i]), int(ln[i]), texts[i]) == (p1, l1, t1), (js[:200], int(st[i]), int(pos[i]), int(ln[i]), texts[i], p1, l1, t1)
        assert texts[i].startswith(b"proto: (line ")
    big = next(i for i, (_, js) in enumerate(items) if len(js) > 1 << 20)
    lines = items[big][1].count(b"\n")
    assert st[big] == 2 and texts[big] == b'proto: (line %d:3): unknown field "nope_late"' % (lines + 1), texts[big]


def test_agrees_with_oracle(engine, schema, oracle):
    """unknown and duplicate fields with a key token: the text less protojson's position is the oracle's message"""
    items = corpus()
    _, _, _, st, pos, ln, texts = _batch_run(engine, schema)
    named = 0
    for i, (n, js) in enumerate(items):
        if st[i] not in (2, 6) or not ln[i] or len(js) > 1 << 20:
            continue
        rc, _, err = oracle.encode(n, js)
        assert rc != 0
        assert js[pos[i]:pos[i] + ln[i]].startswith(b'"') and js[pos[i]:pos[i] + ln[i]].endswith(b'"')
        if "map key" in err:
            continue
        ours = re.sub(rb"\(line \d+:\d+\): ", b"", texts[i]).decode("utf-8", "replace")
        assert ours == err, (js[:200], ours, err)
        named += 1
    assert named >= 100, named


def test_skipped_items(engine, schema):
    """status 0 and 12 (no_space) are not looked at, whatever the item holds"""
    items = corpus()
    ids, data, off, st, _, _, _ = _batch_run(engine, schema)
    st2 = st.copy()
    failing = np.flatnonzero(st != 0)
    st2[failing[::3]] = 12
    pos, ln, texts = engine.encode_diagnose_batch(schema, ids, data, off, st2)
    for i in range(len(items)):
        if st2[i] in (0, 12):
            assert (int(pos[i]), int(ln[i]), texts[i]) == (0, 0, b""), i
    assert sum(1 for i in failing if st2[i] != 12 and texts[i]) == len(failing) - len(failing[::3])


class DevBatch:
    def __init__(self, torch, ids, data, off, text_cap):
        dev = torch.device("cuda", 0)
        n = len(ids)
        self.n, self.in_bytes, self.text_cap = n, len(data), int(text_cap)
        self.d_in = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
        self.d_in[: len(data)] = torch.from_numpy(np.array(data, np.uint8))
        self.d_off = torch.from_numpy(np.array(off, np.uint64).view(np.int64)).to(dev)
        self.d_msg = torch.from_numpy(np.array(ids, np.int32)).to(dev)
        self.d_st = torch.full((n,), -99, dtype=torch.int32, device=dev)
        self.d_wire = torch.empty(2 * len(data) + 4096, dtype=torch.uint8, device=dev)
        self.d_wire_off = torch.empty(n + 1, dtype=torch.int64, device=dev)

    def outputs(self, torch):
        dev = torch.device("cuda", 0)
        return (torch.full((self.n,), 7, dtype=torch.int32, device=dev), torch.full((self.n,), 7, dtype=torch.int32, device=dev),
                torch.full((self.text_cap + 1,), 0xEE, dtype=torch.uint8, device=dev), torch.full((self.n + 1,), -1, dtype=torch.int64, device=dev))

    def encode(self, engine, schema, stream):
        engine.encode_batch_dev(schema, self.n, self.d_msg.data_ptr(), self.d_in.data_ptr(), self.d_off.data_ptr(), self.in_bytes,
                                self.d_wire.data_ptr(), len(self.d_wire), self.d_wire_off.data_ptr(), self.d_st.data_ptr(), 0, stream)

    def diagnose(self, engine, schema, out, stream, text_cap=None):
        pos, ln, text, text_off = out
        engine.encode_diagnose_batch_dev(schema, self.n, self.d_msg.data_ptr(), self.d_in.data_ptr(), self.d_off.data_ptr(), self.in_bytes,
                                         self.d_st.data_ptr(), pos.data_ptr(), ln.data_ptr(), text.data_ptr(),
                                         self.text_cap if text_cap is None else text_cap, text_off.data_ptr(), stream)


def _fetch(out):
    pos, ln, text, text_off = (t.cpu().numpy() for t in out)
    text_off = text_off.astype(np.uint64)
    t = text.tobytes()
    return pos.astype(np.uint32), ln.astype(np.uint32), [t[int(text_off[i]): int(text_off[i + 1])] for i in range(len(text_off) - 1)], text_off


def test_dev_form_on_streams(engine, schema):
    """the device-buffer form behind ggr_encode_batch_dev of the same batch (engine stream, then a caller's stream), and
    behind another request-side call on another stream, ordered by an event: the results of the host form every time"""
    import torch
    ids, data, off, st, pos, ln, texts = _batch_run(engine, schema)
    need = sum(len(t) for t in texts)
    B = DevBatch(torch, ids, data, off, need + 4096)
    small = corpus()[:300]
    ids2, data2, off2 = _pack(schema, small)
    B2 = DevBatch(torch, ids2, data2, off2, 64)
    caller, other = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = [B.outputs(torch) for _ in range(3)]
    B.encode(engine, schema, None)
    B.diagnose(engine, schema, outs[0], None)
    engine.synchronize()
    B.d_st.fill_(-99)
    torch.cuda.synchronize()
    B.encode(engine, schema, caller.cuda_stream)
    B.diagnose(engine, schema, outs[1], caller.cuda_stream)
    caller.synchronize()
    # a request-side call of another batch on `other`, then this batch's diagnosis on `caller` once it is done
    B2.encode(engine, schema, other.cuda_stream)
    ev = torch.cuda.Event()
    ev.record(other)
    caller.wait_event(ev)
    B.diagnose(engine, schema, outs[2], caller.cuda_stream)
    caller.synchronize()
    assert (B.d_st.cpu().numpy() == st).all()
    for out in outs:
        p, l, t, t_off = _fetch(out)
        assert (p == pos).all() and (l == ln).all() and t == texts
        assert int(t_off[-1]) == need


def test_text_capacity(engine, schema):
    """a capacity of 0 or one byte short: GGR_ERR_NO_SPACE and the capacity that would do in text_off[n]; the retry
    succeeds.  On the device, the total comes back in text_off[n] and only the texts that fit are written"""
    import torch
    from ggrmcp_b200 import engine as E
    L = E._load()
    ids, data, off, st, pos, ln, texts = _batch_run(engine, schema)
    need = sum(len(t) for t in texts)
    n = len(ids)
    for cap in (0, need - 1, need):
        text = np.zeros(max(cap, 1), np.uint8)
        text_off = np.zeros(n + 1, np.uint64)
        p, l = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        rc = L.ggr_encode_diagnose_batch(engine.h, schema.h, n, ids.ctypes.data, data.ctypes.data, off.ctypes.data, st.ctypes.data,
                                         p.ctypes.data, l.ctypes.data, text.ctypes.data if cap else None, cap, text_off.ctypes.data)
        assert rc == (0 if cap == need else -5) and int(text_off[n]) == need, (cap, rc, int(text_off[n]))
        if rc == 0:
            assert (p == pos).all() and (l == ln).all()
            assert [text.tobytes()[int(text_off[i]): int(text_off[i + 1])] for i in range(n)] == texts
    B = DevBatch(torch, ids, data, off, need)
    B.d_st.copy_(torch.from_numpy(st))
    out = B.outputs(torch)
    B.diagnose(engine, schema, out, None, need - 1)
    engine.synchronize()
    p, l, t, t_off = _fetch(out)
    assert int(t_off[-1]) == need and (p == pos).all() and (l == ln).all()
    assert all(t[i] == texts[i] for i in range(n) if int(t_off[i + 1]) <= need - 1)


def test_launches_do_not_grow_with_failures(engine, schema):
    def launches(k):
        items = [(cases.A, b'{"zz_%d":%d}' % (i, i)) for i in range(k)] + [(cases.A, b'{"f_int32":1}')] * 50
        ids, data, off = _pack(schema, items)
        st = np.array([2] * k + [0] * 50, np.int32)
        before = engine.launch_count()
        pos, ln, texts = engine.encode_diagnose_batch(schema, ids, data, off, st)
        assert all(texts[i] == b'proto: (line 1:2): unknown field "zz_%d"' % i for i in range(k))
        return engine.launch_count() - before
    assert launches(1) == launches(5000)
