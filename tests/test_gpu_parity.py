"""GPU parity tests: the sm_90a kernels, driven through the C ABI (ggr_encode_batch /
ggr_decode_batch), against the CPU oracle on the same inputs.  Bit-exact for every item the
oracle accepts; equal status category for every item it rejects."""
import random

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu


def _run(engine, schema, encode, items, flags=0):
    from ggrmcp_b200.engine import pack, unpack
    ids = np.array([schema.message(n) for n, _ in items], np.int32)
    data, off = pack([b for _, b in items])
    # packed back to back: each item starts where the one before it ends, at whatever offset mod 16 that gives
    fn = engine.encode_batch if encode else engine.decode_batch
    out, ooff, st = fn(schema, ids, data, off, flags)
    return unpack(out, ooff), st


def _oracle(oracle, encode, items, flags=0):
    outs, sts = [], []
    for n, b in items:
        rc, o, _ = (oracle.encode(n, b, flags) if encode else oracle.decode(n, b, flags))
        outs.append(o)
        sts.append(rc)
    return outs, sts


def _compare(items, eo, es, oo, os_, allow_gap):
    gaps = 0
    for i, (name, b) in enumerate(items):
        if es[i] == 11 and os_[i] == 0:
            gaps += 1
            assert allow_gap(name, b), (name, b[:200], "unsupported")
            continue
        assert cases.status_compatible(os_[i], int(es[i])) or (os_[i] != 0 and es[i] != 0 and {os_[i], int(es[i])} <= {1, 3, 5}), \
            (name, b[:200], os_[i], int(es[i]))
        if os_[i] == 0:
            assert eo[i] == oo[i], (name, b[:200], oo[i][:200], eo[i][:200])
        else:
            assert eo[i] == b""
    return gaps


def test_reference_vectors(engine, schema, oracle):
    items = [(n, js) for n, js, _ in cases.K_REQUESTS]
    eo, es = _run(engine, schema, True, items)
    assert list(es) == [0] * len(items)
    assert [o.hex() for o in eo] == [w for _, _, w in cases.K_REQUESTS]
    items = [(n, bytes.fromhex(w)) for n, w, _ in cases.K_REPLIES]
    eo, es = _run(engine, schema, False, items)
    assert list(es) == [0] * len(items)
    assert eo == [j for _, _, j in cases.K_REPLIES]
    eo, es = _run(engine, schema, False, items, 1)
    assert eo == [j.replace(b',"', b', "') for _, _, j in cases.K_REPLIES]


def test_unknown_field_status(engine, schema):
    # tests/real_grpc_invocation_test.go:238-245
    eo, es = _run(engine, schema, True, [(cases.P + "ProcessNodeRequest", b'{"invalid_field":"value"}')])
    assert int(es[0]) == 2 and eo[0] == b""


def test_encode_edges(engine, schema, oracle):
    items = [(n, js) for n, js, _ in cases.ENCODE_EDGE]
    eo, es = _run(engine, schema, True, items)
    oo, os_ = _oracle(oracle, True, items)
    assert _compare(items, eo, es, oo, os_, lambda n, b: False) == 0


def test_encode_random(engine, schema, oracle):
    items = cases.random_encode_cases(150)
    eo, es = _run(engine, schema, True, items)
    oo, os_ = _oracle(oracle, True, items)
    assert _compare(items, eo, es, oo, os_, lambda n, b: False) == 0


def test_encode_damaged(engine, schema, oracle):
    rng = random.Random(5)
    items = [(n, cases.mutate_json(j, rng)) for n, j in cases.random_encode_cases(80, seed0=700) for _ in range(3)]
    eo, es = _run(engine, schema, True, items)
    oo, os_ = _oracle(oracle, True, items)
    for i in range(len(items)):
        assert (os_[i] == 0) == (int(es[i]) == 0), (items[i], os_[i], int(es[i]))
        if os_[i] == 0:
            assert eo[i] == oo[i]


def test_encode_diagnose(engine, schema, oracle):
    """ggr_encode_diagnose: the status of the batch call again, the position of the offending key and - for unknown and
    duplicate fields, the wording the reference's tests pin (tests/real_grpc_invocation_test.go:238-245) - the oracle's
    message once protojson's position prefix is taken off"""
    import re
    name = "com.example.complex.GetUserProfileRequest"
    mid = schema.message(name)
    probes = [b'{"invalid_field":1}', b'{"user_id":"a",\n  "nope": {"x":[1,2]}}', b'{"user_id":"a","user_id":"b"}', b'{"user_id":5}',
              b'{"user_id" "a"}', b'{"user_id":"a"', b'{"user_id":"ok"}', b'{ "userId":"a", "user_id":"b"}']
    rng = random.Random(9)
    items = [(name, p) for p in probes] + [(n, cases.mutate_json(j, rng)) for n, j in cases.random_encode_cases(40, seed0=900)]
    eo, es = _run(engine, schema, True, items)
    named = 0
    for (n, js), st_batch in zip(items, es):
        st, pos, ln, text = engine.encode_diagnose(schema, schema.message(n), js)
        assert st == int(st_batch), (js, st, int(st_batch))
        rc, _, err = oracle.encode(n, js)
        assert (rc == 0) == (st == 0)
        if st == 0:
            assert text == ""
            continue
        assert pos <= len(js) and text.startswith("proto: (line ")
        if st in (2, 6) and ln:  # unknown field / duplicate field: the raw key token
            assert js[pos:pos + ln].startswith(b'"') and js[pos:pos + ln].endswith(b'"')
            ours = re.sub(r"\(line \d+:\d+\): ", "", text)
            if "map key" not in err:
                assert ours == err, (js, ours, err)
                named += 1
    assert named >= 4
    st, pos, ln, text = engine.encode_diagnose(schema, mid, probes[1])
    assert (st, js_slice := probes[1][pos:pos + ln]) == (2, b'"nope"') and text == 'proto: (line 2:3): unknown field "nope"', (st, pos, ln, text)


def test_decode_edges(engine, schema, oracle):
    items = [(n, bytes.fromhex(h)) for n, h in cases.DECODE_EDGE_HEX]
    for flags in (0, 1):
        eo, es = _run(engine, schema, False, items, flags)
        oo, os_ = _oracle(oracle, False, items, flags)
        _compare(items, eo, es, oo, os_, lambda n, b: False)


def test_decode_random(engine, schema, oracle):
    items = cases.random_decode_cases(120)
    eo, es = _run(engine, schema, False, items)
    oo, os_ = _oracle(oracle, False, items)
    _compare(items, eo, es, oo, os_, lambda n, b: False)


def test_null_members_after_other_batches(engine, schema, oracle):
    """a null member has no bytes, but the lock-step emitter still visits its IR slot: it must not find what an earlier
    batch left there (found by the small_chunks path in round 2: 0x10 came out as 0xd0)"""
    first = [(cases.A, b'{"f_int32":%d,"f_int64":"%d","f_uint32":%d,"f_string":"abc","f_sint32":-%d}' % (k + 300, k * 77 + 1, k + 7, k + 1))
             for k in range(96)]
    eo, es = _run(engine, schema, True, first)
    oo, os_ = _oracle(oracle, True, first)
    _compare(first, eo, es, oo, os_, lambda n, b: False)
    for rep in range(3):
        second = [(cases.A, b'{"f_int32":null,"f_int64":"%d","f_uint32":null,"f_string":null,"f_sint32":%d}' % (k * 7 + rep, k + 1))
                  for k in range(96)] + [("wkt.HasStruct", b'{"s":null,"x":2}'), (cases.A, b'{"f_msg":null,"r_int32":null,"m_str_int32":null,"f_bool":true}')]
        eo, es = _run(engine, schema, True, second)
        oo, os_ = _oracle(oracle, True, second)
        _compare(second, eo, es, oo, os_, lambda n, b: False)
        assert all(x == 0 for x in os_)


def test_wkt_duration_wrappers_empty(engine, schema, oracle):
    """Duration, the nine wrappers and Empty (protojson well_known_types.go) in every position and as root messages,
    both directions, every kernel path; Struct stays refused"""
    items = cases.WKT_ENCODE
    eo, es = _run(engine, schema, True, items)
    oo, os_ = _oracle(oracle, True, items)
    _compare(items, eo, es, oo, os_, lambda n, b: (n == "wkt.HasStruct" and b"s" in b) or cases.fieldmask_gap(b))
    assert sum(1 for x in os_ if x == 0) >= 55
    items = cases.wkt_decode_cases()
    for flags in (0, 1):
        eo, es = _run(engine, schema, False, items, flags)
        oo, os_ = _oracle(oracle, False, items, flags)
        _compare(items, eo, es, oo, os_, lambda n, b: False)
    assert sum(1 for x in os_ if x == 0) >= 45


def test_decode_merges_split_submessages(engine, schema, oracle):
    """singular sub-messages that arrive in several occurrences are merged the way proto.Unmarshal does
    (reflection.go:363): plain fields, oneof members, map values, Timestamps, damaged pieces"""
    items = cases.merge_cases()
    for flags in (0, 1):
        eo, es = _run(engine, schema, False, items, flags)
        oo, os_ = _oracle(oracle, False, items, flags)
        _compare(items, eo, es, oo, os_, lambda n, b: False)
    assert sum(1 for x in os_ if x == 0) >= 20


def test_empty_and_ragged_batches(engine, schema, oracle):
    from ggrmcp_b200.engine import pack
    # empty batch
    out, off, st = engine.encode_batch(schema, np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert len(out) == 0 and list(off) == [0]
    # ragged: empty items between large ones, bad message ids
    big = b'{"f_string":"' + b"x" * 100000 + b'"}'
    items = [(cases.A, b""), (cases.A, big), (cases.A, b"{}"), (cases.A, b'{"f_int32":7}'), (cases.A, b"")]
    eo, es = _run(engine, schema, True, items)
    oo, os_ = _oracle(oracle, True, items)
    assert list(es) == os_ and eo == oo
    ids = np.array([-1, 99999, schema.message(cases.A)], np.int32)
    data, off = pack([b"{}", b"{}", b'{"f_int32":1}'])
    out, ooff, st = engine.encode_batch(schema, ids, data, off)
    assert list(st) == [11, 11, 0]


def test_full_size_properties(engine, schema, oracle):
    """BASELINE.json config sizes: round trip wire -> JSON -> wire and sampled oracle parity."""
    import benchgen
    n = 65536
    wl = benchgen.nested(n, schema.message)
    wire, woff, st = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    assert (st == 0).all()
    js, joff, st2 = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    assert (st2 == 0).all()
    # reply JSON fed back through the request side reproduces the reply wire (protojson output is
    # valid protojson input; Node / GetUserProfileResponse are symmetric)
    wire2, woff2, st3 = engine.encode_batch(schema, wl.rep_msg, js, joff)
    assert (st3 == 0).all()
    assert wire2.tobytes() == wl.rep_wire.tobytes()
    assert (woff2 == wl.rep_off).all()
    # bit-exact parity with the oracle on every item of the batch (the oracle runs on all host threads)
    import os
    thr = os.cpu_count() or 8
    omsg = np.array([oracle_index(oracle, schema, m) for m in wl.req_msg], np.int32)
    ow, owoff, ost = oracle.encode_batch(omsg, wl.req_json, wl.req_off, threads=thr)
    assert (ost == 0).all() and (owoff == woff).all() and ow.tobytes() == wire.tobytes()
    omsg = np.array([oracle_index(oracle, schema, m) for m in wl.rep_msg], np.int32)
    oj, ojoff, ost = oracle.decode_batch(omsg, wl.rep_wire, wl.rep_off, threads=thr)
    assert (ost == 0).all() and (ojoff == joff).all() and oj.tobytes() == js.tobytes()


_names = {}


def oracle_index(oracle, schema, engine_idx):
    """engine and oracle number messages independently: map through the full name"""
    if not _names:
        for nm in [cases.P + x for x in ("ProcessNodeRequest", "CreateDocumentRequest", "Node", "GetUserProfileResponse")] + \
                ["bench.Flat", "bench.Blob", cases.A]:
            _names[schema.message(nm)] = oracle.msg(nm)
    return _names[int(engine_idx)]


def test_flat_and_blob_configs(engine, schema, oracle):
    import benchgen
    wl = benchgen.flat(65536, schema.message)
    wire, woff, st = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    assert (st == 0).all()
    assert wire.tobytes() == wl.rep_wire.tobytes()  # EchoFlat: request wire == reply wire
    js, joff, st = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    assert (st == 0).all()
    for i in range(0, 65536, 257):
        b = wl.rep_wire[int(wl.rep_off[i]):int(wl.rep_off[i + 1])].tobytes()
        rc, oj, _ = oracle.decode("bench.Flat", b)
        assert rc == 0 and oj == js[int(joff[i]):int(joff[i + 1])].tobytes()
    # configs[3] at its full size: 4096 replies of 64 KiB, every one compared
    import os
    wb = benchgen.blob(4096, schema.message)
    js, joff, st = engine.decode_batch(schema, wb.rep_msg, wb.rep_wire, wb.rep_off)
    assert (st == 0).all()
    omsg = np.full(wb.n, oracle.msg("bench.Blob"), np.int32)
    oj, ojoff, ost = oracle.decode_batch(omsg, wb.rep_wire, wb.rep_off, threads=os.cpu_count() or 8)
    assert (ost == 0).all() and (ojoff == joff).all() and oj.tobytes() == js.tobytes()


@pytest.mark.gpu
def test_request_and_reply_batches_in_flight_together(engine, schema, oracle):
    """the host entry points take one batch per direction concurrently (bench.py's end-to-end run does
    exactly this from two threads): results must be those of the calls made one after the other"""
    import threading
    import benchgen
    n = 20000
    wl = benchgen.nested(n, schema.message)
    ref_req = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    ref_rep = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    for _ in range(3):
        got = {}

        def req():
            got["req"] = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)

        t = threading.Thread(target=req)
        t.start()
        got["rep"] = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
        t.join()
        for a, b in ((got["req"], ref_req), (got["rep"], ref_rep)):
            assert (a[2] == 0).all() and (a[1] == b[1]).all() and a[0].tobytes() == b[0].tobytes()


def test_result_bodies(engine, schema, oracle):
    """reply half + MCP result wrapping on the device (SURVEY row A10) against the oracle's orc_response"""
    from ggrmcp_b200.engine import pack
    rng = random.Random(12)
    items = cases.random_decode_cases(40) + [(n, bytes.fromhex(w)) for n, w, _ in cases.K_REPLIES]
    ids = [rng.choice([b"1", b'"req-42"', b"9007199254740993", b'"\\u00e9"']) for _ in items]
    msg = np.array([schema.message(n) for n, _ in items], np.int32)
    data, off = pack([w for _, w in items])
    idb, ioff = pack(ids)
    out, ooff, st = engine.decode_wrap_batch(schema, msg, data, off, idb, ioff)
    ok = 0
    for i, (n, w) in enumerate(items):
        ost, body = oracle.response(n, w, ids[i])
        got = bytes(out[int(ooff[i]):int(ooff[i + 1])])
        assert (ost == 0) == (st[i] == 0), (n, w.hex()[:80], ost, st[i])
        if ost == 0:
            assert got == body, (n, w.hex()[:80], got[:200], body[:200])
            ok += 1
        else:
            assert got == b""
    assert ok > len(items) // 2


def test_request_bodies(engine, schema, oracle):
    """request envelope on the device (SURVEY rows A1-A6) against orc_request: a body the device takes must
    give the oracle's wire bytes, method and id; every other body must come back as unsupported (11)"""
    from ggrmcp_b200.engine import pack
    bodies = cases.request_bodies(oracle)
    data, off = pack(bodies)
    out, ooff, method, id_span, st = engine.request_batch(schema, data, off)
    taken = 0
    for i, body in enumerate(bodies):
        r = oracle.request(body)
        got = bytes(out[int(ooff[i]):int(ooff[i + 1])])
        assert st[i] in (0, 11), (body[:120], st[i])
        if st[i] == 0:
            idt = body[int(id_span[i][0]): int(id_span[i][0]) + int(id_span[i][1])]
            assert r["kind"] == 0 and got == r["wire"] and int(method[i]) == r["method"] and idt == r["id"], (body[:200], r["kind"], r["status"])
            # the method index means the same thing on both sides
            assert schema.methods()[int(method[i])]["tool_name"] == oracle.methods()[r["method"]]["tool"]
            taken += 1
        else:
            assert got == b""
    assert taken >= 400  # every bench-shaped body at least


def test_go_legacy_field_order(schema, oracle, fds_bytes):
    """GGR_ORDER_GO_LEGACY (Go's order.LegacyFieldOrder: extensions, then fields by number with oneof members
    last) against the oracle's ORC_F_GO_LEGACY_ORDER, on the lock-step and the per-thread kernels"""
    import os
    import ggrmcp_b200
    from ggrmcp_b200.engine import pack, unpack, ORDER_GO_LEGACY
    items = cases.random_encode_cases(150, seed0=31000) + [(n, js) for n, js, _ in cases.ENCODE_EDGE]
    for env in ({"GGR_LOCKSTEP_MIN_BYTES": "0"}, {"GGR_COOP_ENC": "0"}):
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            eng = ggrmcp_b200.Engine(0, wire_order=ORDER_GO_LEGACY)
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        sch = eng.register(fds_bytes)
        ids = np.array([sch.message(n) for n, _ in items], np.int32)
        data, off = pack([b for _, b in items])
        out, ooff, st = eng.encode_batch(sch, ids, data, off)
        got = unpack(out, ooff)
        differs = 0
        for i, (n, b) in enumerate(items):
            rc, ow, _ = oracle.encode(n, b, 2)  # ORC_F_GO_LEGACY_ORDER
            assert (rc == 0) == (st[i] == 0), (n, b[:120], rc, st[i])
            if rc == 0:
                assert got[i] == ow, (n, b[:200])
                differs += ow != oracle.encode(n, b, 0)[1]
        assert differs > 0  # the two orders are not the same thing on this corpus (oneof members)
        sch.release()
        eng.close()


def test_small_output_capacity(engine, schema, oracle):
    """GGR_ERR_NO_SPACE: out_off[n] comes back as the capacity that would do, for one chunk and for many, in
    both directions and with result wrapping; the retry with that capacity gives the full result"""
    import ctypes as C
    import benchgen
    from ggrmcp_b200 import engine as E
    from ggrmcp_b200.engine import pack
    L = E._load()
    wl = benchgen.nested(3000, schema.message)
    idb, ioff = pack([b"%d" % i for i in range(wl.n)])

    def raw(fn, msg, data, off, cap, extra=()):
        n = len(msg)
        out = np.empty(max(cap, 1), np.uint8)
        out_off = np.zeros(n + 1, np.uint64)
        st = np.zeros(n, np.int32)
        msg = np.ascontiguousarray(msg, np.int32)
        args = [engine.h, schema.h, n, msg.ctypes.data, data.ctypes.data, off.ctypes.data] + [a.ctypes.data for a in extra] + \
               [out.ctypes.data, cap, out_off.ctypes.data, st.ctypes.data, 0]
        rc = fn(*args)
        return rc, out, out_off, st

    full_req = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    full_rep = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    full_wrap = engine.decode_wrap_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off, idb, ioff)
    # the chunked host path itself (chunk boundaries by items or bytes, short chunks at both ends) against the oracle
    names = {schema.message(nm): oracle.msg(nm) for nm in ("com.example.complex.ProcessNodeRequest", "com.example.complex.CreateDocumentRequest",
                                                           "com.example.complex.Node", "com.example.complex.GetUserProfileResponse")}
    ow, owoff, _ = oracle.encode_batch(np.array([names[int(i)] for i in wl.req_msg], np.int32), wl.req_json, wl.req_off)
    oj, ojoff, _ = oracle.decode_batch(np.array([names[int(i)] for i in wl.rep_msg], np.int32), wl.rep_wire, wl.rep_off)
    assert full_req[0].tobytes() == ow.tobytes() and (full_req[1] == owoff).all() and (full_req[2] == 0).all()
    assert full_rep[0].tobytes() == oj.tobytes() and (full_rep[1] == ojoff).all() and (full_rep[2] == 0).all()
    for fn, msg, data, off, extra, full in ((L.ggr_encode_batch, wl.req_msg, wl.req_json, wl.req_off, (), full_req),
                                            (L.ggr_decode_batch, wl.rep_msg, wl.rep_wire, wl.rep_off, (), full_rep),
                                            (L.ggr_decode_wrap_batch, wl.rep_msg, wl.rep_wire, wl.rep_off, (idb, ioff), full_wrap)):
        need = len(full[0])
        for cap in (0, 100, need // 3, need - 1):
            rc, out, out_off, st = raw(fn, msg, data, off, cap, extra)
            assert rc == -5, (fn.__name__, cap, rc)
            assert int(out_off[len(msg)]) == need, (fn.__name__, cap, int(out_off[len(msg)]), need)
        rc, out, out_off, st = raw(fn, msg, data, off, need, extra)
        assert rc == 0 and (st == 0).all() and out[:need].tobytes() == full[0].tobytes() and (out_off == full[1]).all()
    # the binding's own retry path
    a = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off, out_cap=10)
    assert a[0].tobytes() == full_req[0].tobytes()
    b = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off, out_cap=10)
    assert b[0].tobytes() == full_rep[0].tobytes()


def test_wrap_heterogeneous_chunks(engine, schema, oracle):
    """result wrapping: a chunk whose texts expand far more than the batch average (packed bools: 1 byte of wire,
    5-6 of text) next to chunks that do not must not lose items to the intermediate buffer"""
    from ggrmcp_b200.engine import pack
    import benchgen
    wl = benchgen.nested(600, schema.message)
    blob = wl.rep_wire.tobytes()
    items = [(int(wl.rep_msg[i]), blob[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]) for i in range(600)]
    # a repeated bool field of the all-kinds message
    import pbgen
    fld = [f for f in pbgen.cls(cases.A).DESCRIPTOR.fields if f.name == 'r_bool'][0]
    tag = (fld.number << 3) | 2
    tagb = bytes([tag & 0x7F | 0x80, tag >> 7]) if tag >= 128 else bytes([tag])
    payload = b"\x01\x00" * 1500
    ln = len(payload)
    heavy = (schema.message(cases.A), tagb + bytes([ln & 0x7F | 0x80, ln >> 7]) + payload)
    items = items[:300] + [heavy] * 300 + items[300:]
    msg = np.array([m for m, _ in items], np.int32)
    data, off = pack([w for _, w in items])
    idb, ioff = pack([b"7"] * len(items))
    out, ooff, st = engine.decode_wrap_batch(schema, msg, data, off, idb, ioff)
    assert (st == 0).all(), np.unique(st, return_counts=True)
    ost, body = oracle.response(cases.A, heavy[1], b"7")
    assert ost == 0 and bytes(out[int(ooff[300]):int(ooff[301])]) == body


_mixed_cache = {}


def test_mixed_replay(engine, schema, oracle):
    """configs[4]: 100 000 calls over 32 methods with Zipf-distributed sizes, every item against the oracle"""
    import os
    import benchgen
    if not _mixed_cache:
        wl = benchgen.mixed(100000, schema.message)
        thr = os.cpu_count() or 8
        # engine and oracle number messages independently: the oracle's ids through the method table
        fds = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "schemas.binpb"), "rb").read()
        plan, pairs = benchgen._mixed_plan(fds)
        oreq = np.array([oracle.msg(a) for a, _ in pairs], np.int32)[wl.method]
        orep = np.array([oracle.msg(b) for _, b in pairs], np.int32)[wl.method]
        _mixed_cache["wl"] = wl
        _mixed_cache["req"] = oracle.encode_batch(oreq, wl.req_json, wl.req_off, threads=thr)
        _mixed_cache["rep"] = oracle.decode_batch(orep, wl.rep_wire, wl.rep_off, threads=thr)
    wl = _mixed_cache["wl"]
    ow, owoff, ost = _mixed_cache["req"]
    oj, ojoff, ost2 = _mixed_cache["rep"]
    wire, woff, st = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    assert (ost == 0).all() and (st == 0).all()
    assert (woff == owoff).all() and wire.tobytes() == ow.tobytes()
    js, joff, st = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    assert (ost2 == 0).all() and (st == 0).all()
    assert (joff == ojoff).all() and js.tobytes() == oj.tobytes()



def test_single_process_device_set(oracle, fds_bytes):
    """SURVEY 8e from ONE process: one engine + batching thread + NUMA-local pinned arena per device, the batch cut
    by index, results gathered by index (threads, not torchrun).  On a one-GPU box two engines share the device."""
    import torch
    import benchgen
    from ggrmcp_b200.shard import DeviceSet
    ndev = torch.cuda.device_count()
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    ds = DeviceSet(fds_bytes, devices)
    try:
        names = {}

        def mi(n):
            names.setdefault(n, len(names))
            return names[n]

        wl = benchgen.nested(6001, mi)
        inv = {v: k for k, v in names.items()}
        req_names = [inv[int(m)] for m in wl.req_msg]
        rep_names = [inv[int(m)] for m in wl.rep_msg]
        wire, woff, st = ds.encode_batch(req_names, wl.req_json, wl.req_off)
        js, joff, st2 = ds.decode_batch(rep_names, wl.rep_wire, wl.rep_off)
        assert (st == 0).all() and (st2 == 0).all()
        om = np.array([oracle.msg(n) for n in req_names], np.int32)
        ow, owoff, _ = oracle.encode_batch(om, wl.req_json, wl.req_off, threads=8)
        assert (woff == owoff).all() and wire.tobytes() == ow.tobytes()
        om = np.array([oracle.msg(n) for n in rep_names], np.int32)
        oj, ojoff, _ = oracle.decode_batch(om, wl.rep_wire, wl.rep_off, threads=8)
        assert (joff == ojoff).all() and js.tobytes() == oj.tobytes()
        for e in ds.engines:
            assert e.numa_node() >= -1
    finally:
        ds.close()


def test_grpc_framing(engine, schema, oracle):
    """GGR_F_GRPC_FRAME against the oracle's ORC_F_GRPC_FRAME: the request half writes 0x00 | be32 length | wire, the reply
    half takes framed items; bad headers get the oracle's status (reflection.go:367-376)"""
    import struct
    import benchgen
    from ggrmcp_b200.engine import pack, unpack
    F = 2
    items = cases.random_encode_cases(60, seed0=41000) + [(n, js) for n, js, _ in cases.K_REQUESTS] + [(cases.A, b"{}"), (cases.A, b""), (cases.A, b"{")]
    eo, es = _run(engine, schema, True, items, F)
    for i, (n, b) in enumerate(items):
        rc, ow, _ = oracle.encode(n, b, 4)
        assert (rc == 0) == (es[i] == 0), (n, b[:100], rc, es[i])
        assert eo[i] == (ow if rc == 0 else b""), (n, b[:100], eo[i][:40].hex(), ow[:40].hex())
    wl = benchgen.nested(3000, schema.message)
    wire, woff, st = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off, F, out_cap=len(wl.req_json) + 5 * wl.n + 64)
    plain, poff, _ = engine.encode_batch(schema, wl.req_msg, wl.req_json, wl.req_off)
    assert (st == 0).all()
    fr, pl = unpack(wire, woff), unpack(plain, poff)
    assert all(f == b"\x00" + struct.pack(">I", len(p)) + p for f, p in zip(fr, pl))
    # reply side: framed replies in, the same texts out
    rep = unpack(wl.rep_wire, wl.rep_off)
    framed = [b"\x00" + struct.pack(">I", len(p)) + p for p in rep]
    data, off = pack(framed)
    js, joff, st = engine.decode_batch(schema, wl.rep_msg, data, off, F)
    js0, joff0, st0 = engine.decode_batch(schema, wl.rep_msg, wl.rep_wire, wl.rep_off)
    assert (st == 0).all() and (joff == joff0).all() and js.tobytes() == js0.tobytes()
    bad = [(cases.P + "Node", b"\x01\x00\x00\x00\x00"), (cases.P + "Node", b"\x00\x00\x00\x00\x09"), (cases.P + "Node", b"\x00\x00"),
           (cases.P + "Node", b"\x00\x00\x00\x00\x00"), (cases.P + "Node", b"\x02\x00\x00\x00\x00")]
    eo, es = _run(engine, schema, False, bad, F)
    for i, (n, b) in enumerate(bad):
        rc, oj, _ = oracle.decode(n, b, 4)
        assert int(es[i]) == rc and eo[i] == (oj if rc == 0 else b""), (b.hex(), rc, int(es[i]))


def test_descriptor_set_route_tool_names(fds_bytes):
    """GGR_NAMES_DESCRIPTOR_SET: tool names as the FileDescriptorSet route builds them (pkg/descriptors/loader.go:221-235),
    on the host (ggr_tool_lookup) and in the device's tool table (ggr_request_batch)"""
    import ggrmcp_b200
    import orc
    from ggrmcp_b200.engine import pack, NAMES_DESCRIPTOR_SET
    eng = ggrmcp_b200.Engine(0, tool_naming=NAMES_DESCRIPTOR_SET)
    sch = eng.register(fds_bytes)
    S = orc.Schema(fds_bytes, naming=1)
    assert sorted(m["tool_name"] for m in sch.methods()) == sorted(m["tool"] for m in S.methods())
    assert sch.tool("complex_userprofileservice_getuserprofile") >= 0 and sch.tool("com_example_complex_userprofileservice_getuserprofile") < 0
    bodies = [b'{"jsonrpc":"2.0","method":"tools/call","id":%d,"params":{"name":"%s","arguments":{"user_id":"u%d"}}}' % (i, t, i)
              for i, t in enumerate([b"complex_userprofileservice_getuserprofile", b"com_example_complex_userprofileservice_getuserprofile"])]
    data, off = pack(bodies)
    out, ooff, method, id_span, st = eng.request_batch(sch, data, off)
    assert st[0] == 0 and bytes(out[int(ooff[0]):int(ooff[1])]) == S.request(bodies[0])["wire"]
    assert sch.methods()[int(method[0])]["tool_name"] == "complex_userprofileservice_getuserprofile"
    assert st[1] == 11  # unknown under this naming: the shim answers "tool ... not found"
    sch.release()
    eng.close()
