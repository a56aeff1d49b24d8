"""CPU tests of the device code through the host simulation (tests/hostsim): the same per-thread
parser/emitter sources the kernels are built from, compiled with g++ and compared with the oracle.
These are the debugging ground for the kernels; the GPU run of the same cases is
tests/test_gpu_parity.py."""
import random

import pytest

import cases
from strref import html_string as _go_json_string


@pytest.mark.parametrize("name,js,wire", cases.K_REQUESTS)
def test_request_vectors(hsim, name, js, wire):
    for io, oo in ((0, 0), (3, 5), (15, 7)):
        rc, out = hsim.encode(name, js, io, oo)
        assert rc == 0 and out.hex() == wire


@pytest.mark.parametrize("name,wire,js", cases.K_REPLIES)
def test_reply_vectors(hsim, name, wire, js):
    for io, oo in ((0, 0), (3, 5), (15, 7)):
        rc, out = hsim.decode(name, bytes.fromhex(wire), 0, io, oo)
        assert rc == 0 and out == js
        rc, out = hsim.decode(name, bytes.fromhex(wire), 1, io, oo)
        assert rc == 0 and out == js.replace(b',"', b', "')


def _check_encode(oracle, hsim, name, js, i=0):
    ost, ow, _ = oracle.encode(name, js)
    est, ew = hsim.encode(name, js, i % 16, (i * 5) % 16)
    if est == 11 and ost == 0:
        return "gap"
    assert cases.status_compatible(ost, est) or (ost != 0 and est != 0 and {ost, est} <= {1, 3, 5}), (name, js, ost, est)
    if ost == 0:
        assert ew == ow, (name, js, ow.hex(), ew.hex())
    return "ok"


def test_encode_edge_cases(oracle, hsim):
    gaps = []
    for i, (name, js, want) in enumerate(cases.ENCODE_EDGE):
        if _check_encode(oracle, hsim, name, js, i) == "gap":
            gaps.append(js)
        if want is not None:
            est, _ = hsim.encode(name, js)
            assert ["ok", "syntax", "unknown_field"][est] == want
    assert not gaps, gaps


def test_encode_random(oracle, hsim):
    for i, (name, js) in enumerate(cases.random_encode_cases(120)):
        assert _check_encode(oracle, hsim, name, js, i) == "ok"


def test_encode_damaged_json(oracle, hsim):
    rng = random.Random(11)
    n_err = 0
    for i, (name, js) in enumerate(cases.random_encode_cases(60, seed0=500)):
        for _ in range(3):
            bad = cases.mutate_json(js, rng)
            ost, ow, _ = oracle.encode(name, bad)
            est, ew = hsim.encode(name, bad, i % 16, (i * 3) % 16)
            assert (ost == 0) == (est == 0), (name, bad, ost, est)
            if ost == 0:
                assert ow == ew, (name, bad)
            else:
                n_err += 1
    assert n_err > 100


def _check_decode(oracle, hsim, name, w, i=0, flags=0):
    ost, oj, _ = oracle.decode(name, w, flags)
    est, ej = hsim.decode(name, w, flags, i % 16, (i * 5) % 16)
    if est == 11 and ost == 0:
        return "gap"
    assert cases.status_compatible(ost, est), (name, w.hex(), ost, est)
    if ost == 0:
        assert ej == oj, (name, w.hex(), oj, ej)
    return "ok"


def test_decode_edge_cases(oracle, hsim):
    for i, (name, hx) in enumerate(cases.DECODE_EDGE_HEX):
        assert _check_decode(oracle, hsim, name, bytes.fromhex(hx), i) == "ok", hx


def test_decode_random(oracle, hsim):
    for i, (name, w) in enumerate(cases.random_decode_cases(100)):
        assert _check_decode(oracle, hsim, name, w, i, i & 1) == "ok", (name, w.hex())


def test_wkt_duration_wrappers_empty(oracle, hsim):
    """Duration, the nine wrappers and Empty in every position (singular, list element, map value, oneof member, root
    message) in both directions (protojson well_known_types.go); Struct is refused, never answered differently"""
    n_ok = n_err = 0
    for i, (name, js) in enumerate(cases.WKT_ENCODE):
        ost, ow, _ = oracle.encode(name, js)
        est, ew = hsim.encode(name, js, i % 16, (i * 5) % 16)
        if est == 11 and ost == 0 and cases.fieldmask_gap(js):
            continue  # a FieldMask written with escapes or non-ASCII spaces at its ends: refused, never answered differently
        assert ost == est or (ost != 0 and est != 0 and {ost, est} <= {1, 3, 5}), (name, js, ost, est)
        if ost == 0:
            assert ew == ow, (name, js, ow.hex(), ew.hex())
        n_ok += ost == 0
        n_err += ost != 0
    assert n_ok >= 55 and n_err >= 40
    n_ok = 0
    for i, (name, w) in enumerate(cases.wkt_decode_cases()):
        ost, oj, _ = oracle.decode(name, w, i & 1)
        est, ej = hsim.decode(name, w, i & 1, i % 16, (i * 5) % 16)
        assert cases.status_compatible(ost, est), (name, w.hex(), ost, est)
        if ost == 0:
            assert ej == oj, (name, w.hex(), oj, ej)
        n_ok += ost == 0
    assert n_ok >= 45


def test_decode_merges_split_submessages(oracle, hsim):
    """proto.Unmarshal merges the occurrences of a singular message field (reflection.go:363): plain fields, oneof
    members (a sibling in between clears), map values inside one entry, Timestamps; every piece is parsed on its own"""
    n_ok = 0
    for i, (name, w) in enumerate(cases.merge_cases()):
        assert _check_decode(oracle, hsim, name, w, i, i & 1) == "ok", (name, w.hex())
        n_ok += oracle.decode(name, w, 0)[0] == 0
    assert n_ok >= 20


# ---- lock-step request-side parser (ggr_coop_enc.cuh) on 32 fibers ---------------------------
def _check_coop_encode(hsim, name, js, i=0, tier=0):
    """the lock-step parser either leaves the item alone (200) or produces exactly the bytes of the
    per-thread path; 3xx = the fiber warp caught lanes at different collectives"""
    rc, out = hsim.encode_coop(name, js, i % 16, (i * 5) % 16, tier)
    assert rc in (0, 200), (name, js, rc)
    if rc == 200:
        return False
    est, ew = hsim.encode(name, js, i % 16, (i * 5) % 16)
    assert est == 0 and out == ew, (name, js, est, ew.hex(), out.hex())
    return True


def test_coop_encode_vectors_and_edges(hsim):
    handled = 0
    for name, js, wire in cases.K_REQUESTS:
        rc, out = hsim.encode_coop(name, js, 3, 5)
        assert rc in (0, 200) and (rc == 200 or out.hex() == wire)
        handled += rc == 0
    for i, (name, js, want) in enumerate(cases.ENCODE_EDGE):
        handled += _check_coop_encode(hsim, name, js, i)
    assert handled > 60


def test_coop_encode_random_and_damaged(hsim):
    rng = random.Random(23)
    handled = 0
    for i, (name, js) in enumerate(cases.random_encode_cases(150, seed0=4000)):
        handled += _check_coop_encode(hsim, name, js, i, i & 1)
        handled += _check_coop_encode(hsim, name, cases.mutate_json(js, rng), i + 1, i & 1)
    assert handled > 500


def test_coop_encode_bench_shapes(hsim):
    import benchgen
    names = {}

    def mi(name):
        names[hsim.msg(name)] = name
        return hsim.msg(name)

    # tier 0 = small per-warp tables (first kernel), tier 1 = large tables (second kernel): together
    # they must take every item of the benchmark shapes, or the per-thread parser becomes the tail
    for kind, n, tier, want in (("nested", 200, 0, 180), ("nested", 200, 1, 200), ("flat", 100, 0, 100)):
        wl = getattr(benchgen, kind)(n, mi)
        blob = wl.req_json.tobytes()
        handled = 0
        for i in range(n):
            js = blob[int(wl.req_off[i]):int(wl.req_off[i + 1])]
            handled += _check_coop_encode(hsim, names[int(wl.req_msg[i])], js, i, tier)
        assert handled >= want, (kind, tier, handled)


# ---- token-parallel walker (ggr_walk.cuh: tokenizer without colons / commas, place, type) on 32 fibers -------
def _check_walk(hsim, name, js, i=0):
    """either leaves the item alone (200) or produces exactly the bytes of the per-thread path"""
    rc, out = hsim.encode_walk(name, js, i % 16, (i * 5) % 16)
    assert rc in (0, 200), (name, js, rc)
    if rc == 200:
        return False
    est, ew = hsim.encode(name, js, i % 16, (i * 5) % 16)
    assert est == 0 and out == ew, (name, js, est, ew.hex(), out.hex())
    return True


def test_walk_vectors_and_edges(hsim):
    for name, js, wire in cases.K_REQUESTS:
        rc, out = hsim.encode_walk(name, js, 3, 5)
        assert rc == 0 and out.hex() == wire, (name, rc)
    handled = sum(_check_walk(hsim, name, js, i) for i, (name, js, want) in enumerate(cases.ENCODE_EDGE))
    assert handled > 20


def test_walk_random_and_damaged(hsim):
    rng = random.Random(29)
    handled = 0
    for i, (name, js) in enumerate(cases.random_encode_cases(150, seed0=5000)):
        handled += _check_walk(hsim, name, js, i)
        handled += _check_walk(hsim, name, cases.mutate_json(js, rng), i + 1)
        handled += _check_walk(hsim, name, cases.mutate_json(cases.mutate_json(js, rng), rng), i + 2)
    assert handled > 500


def test_walk_structure_mutations(hsim):
    """every single-character deletion / duplication / swap of a structural character of a small document:
    the grammar checks of the tokenizer and the place kernel must never let a broken document through"""
    name = "com.example.complex.ProcessNodeRequest"
    js = b'{"root_node":{"children":[{"id":"a","value":"b"},{"children":[{"id":"c"}],"id":"d"},{"children":[]}],"id":"r","value":"v"}}'
    n = 0
    for i in range(len(js)):
        if js[i:i + 1] in b'{}[]:,"':
            for mut in (js[:i] + js[i + 1:], js[:i] + js[i:i + 1] + js[i:], js[:i] + b"," + js[i:], js[:i] + b":" + js[i:],
                        js[:i] + b" " + js[i:], js[:i] + b"}" + js[i + 1:], js[:i] + b"]" + js[i + 1:]):
                _check_walk(hsim, name, mut, i)
                n += 1
    assert n > 400


def test_walk_bench_shapes(hsim):
    import benchgen
    names = {}

    def mi(name):
        names[hsim.msg(name)] = name
        return hsim.msg(name)

    for kind, n in (("nested", 250), ("flat", 100)):
        wl = getattr(benchgen, kind)(n, mi)
        blob = wl.req_json.tobytes()
        handled = 0
        for i in range(n):
            js = blob[int(wl.req_off[i]):int(wl.req_off[i + 1])]
            handled += _check_walk(hsim, names[int(wl.req_msg[i])], js, i)
        assert handled == n, (kind, handled)


# ---- lock-step reply side (ggr_coop.cuh) on 32 fibers -----------------------------------------
def _check_coop_decode(hsim, name, w, i=0, flags=0):
    rc, out = hsim.decode_coop(name, w, flags, i % 16, (i * 5) % 16)
    assert rc in (0, 200), (name, w.hex(), rc)
    if rc == 200:
        return False
    est, ej = hsim.decode(name, w, flags, i % 16, (i * 5) % 16)
    assert est == 0 and out == ej, (name, w.hex(), est, ej, out)
    return True


def test_coop_decode_vectors_and_edges(hsim):
    handled = 0
    for name, wire, js in cases.K_REPLIES:
        rc, out = hsim.decode_coop(name, bytes.fromhex(wire), 0, 3, 5)
        assert rc in (0, 200) and (rc == 200 or out == js)
        handled += rc == 0
    for i, (name, hexw) in enumerate(cases.DECODE_EDGE_HEX):
        handled += _check_coop_decode(hsim, name, bytes.fromhex(hexw), i, i & 1)
    assert handled > 30


def test_coop_decode_random(hsim):
    handled = 0
    for i, (name, w) in enumerate(cases.random_decode_cases(120, seed0=7000)):
        handled += _check_coop_decode(hsim, name, w, i, i & 1)
    assert handled > 1500


def test_coop_decode_bench_shapes(hsim):
    import benchgen
    names = {}

    def mi(name):
        names[hsim.msg(name)] = name
        return hsim.msg(name)

    for kind, n in (("nested", 200), ("flat", 100)):
        wl = getattr(benchgen, kind)(n, mi)
        blob = wl.rep_wire.tobytes()
        handled = 0
        for i in range(n):
            w = blob[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]
            handled += _check_coop_decode(hsim, names[int(wl.rep_msg[i])], w, i)
        assert handled == n, (kind, handled)


def test_coop_decode_large_leaves(hsim):
    """items larger than the staging buffer are written in place: long plain / escaped / non-ASCII strings
    and long bytes fields (base64) by the whole warp"""
    import benchgen
    names = {}

    def mi(name):
        names[hsim.msg(name)] = name
        return hsim.msg(name)

    wl = benchgen.blob(3, mi)
    blob = wl.rep_wire.tobytes()
    for i in range(3):
        w = blob[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]
        assert _check_coop_decode(hsim, names[int(wl.rep_msg[i])], w, i, i & 1)

    def varint(n):
        o = b""
        while n >= 0x80:
            o += bytes([n & 0x7F | 0x80])
            n >>= 7
        return o + bytes([n])

    rng = random.Random(3)
    for it in range(120):
        ln = rng.choice([0, 1, 2, 3, 95, 96, 97, 98, 255, 256, 257, 1000, 8190, 9000, 20000])
        data = bytes(rng.randrange(256) for _ in range(ln))
        sl = rng.choice([0, 5, 95, 96, 255, 256, 300, 2000, 8100, 8300, 15000])
        kind = rng.random()
        if kind < 0.5:
            name = bytes(rng.choice(b"abcdefghij KLMN") for _ in range(sl))
        elif kind < 0.75:
            name = bytearray(rng.choice(b"abcdefghij KLMN") for _ in range(sl))
            for _ in range(max(1, sl // 50)):
                if sl:
                    name[rng.randrange(sl)] = rng.choice(b'"\\\n\t\x01')
            name = bytes(name)
        else:
            name = "".join(rng.choice("abc \u00e9\u65e5\u20ac\U0001F600") for _ in range(sl // 2)).encode()
        w = b""
        if ln or rng.random() < 0.3:
            w += b"\x0a" + varint(len(data)) + data
        if name:
            w += b"\x12" + varint(len(name)) + name
        assert _check_coop_decode(hsim, "bench.Blob", w, it, it & 1), (ln, sl)


# ---- MCP result wrapping (ggr_wrap.cuh) on 32 fibers ---------------------------------------------
def test_wrap_result_bodies(oracle):
    import hostsim
    rng = random.Random(4)
    alpha = 'abc {}[]:,"\\<>&\n\t\x01\u00e9\u65e5\u20ac\U0001F600\u2028\u2029\u00a8\u0080 xyz0123456789'
    for it in range(1500):
        n = rng.choice([0, 1, 2, 7, 8, 9, 31, 32, 33, 255, 256, 257, 300, 1000])
        t = "".join(rng.choice(alpha) for _ in range(n)).encode("utf-8")
        idt = rng.choice([b"1", b'"abc"', b"123456789", b'"x-' + b"y" * 40 + b'"'])
        rc, out = hostsim.wrap(t, idt)
        assert rc == 0
        assert out == b'{"jsonrpc":"2.0","result":{"content":[{"type":"text","text":' + _go_json_string(t) + b'}]},"id":' + idt + b"}\n"
    # and the oracle's own body for a real reply (K-vector)
    name, wire, js = cases.K_REPLIES[0]
    st, body = oracle.response(name, bytes.fromhex(wire), b"7")
    rc, out = hostsim.wrap(js, b"7")
    assert st == 0 and rc == 0 and out == body


# ---- request envelope (SURVEY rows A1-A4) through the lock-step parser -----------------------------
def _tool_by_input(oracle):
    return {m["input"]: (i, m["tool"]) for i, m in reversed(list(enumerate(oracle.methods())))}


def _check_request(oracle, hsim, body, i=0):
    """handled (rc 0) => the oracle accepts the request and wire, method and id are identical;
    anything else must come back as 'unsupported' (200), never as a different answer"""
    r = oracle.request(body)
    rc, wire, method, idt = hsim.request_coop(body, i % 16, (i * 3) % 16, i & 1)
    assert rc in (0, 200), (body[:200], rc)
    if rc == 0:
        assert r["kind"] == 0 and wire == r["wire"] and method == r["method"] and idt == r["id"], (body[:300], r["kind"], r["status"])
    return rc == 0


def test_request_envelope_random(oracle, hsim):
    by_input = _tool_by_input(oracle)
    rng = random.Random(31)
    handled = total = 0
    for i, (name, js) in enumerate(cases.random_encode_cases(60, seed0=12000)):
        k = oracle.msg(name)
        if k not in by_input:
            continue
        tool = by_input[k][1].encode()
        idt = rng.choice([b"1", b"42", b'"abc"', b"-7", b"123456789012345", b"1.0", b"1e3", b'"a<b"', b'"\\u00e9"',
                          b"9007199254740993", b"null", b"0", b'"x y"'])
        parts = {"jsonrpc": b'"jsonrpc":"2.0"', "id": b'"id":' + idt, "method": b'"method":"tools/call"',
                 "params": b'"params":{"name":"' + tool + b'","arguments":' + js + b"}"}
        keys = list(parts)
        rng.shuffle(keys)
        body = b"{" + b",".join(parts[k2] for k2 in keys) + b"}"
        handled += _check_request(oracle, hsim, body, i)
        total += 1
        for variant in (body.replace(b'"jsonrpc":"2.0"', b'"jsonrpc":"1.0"'), body.replace(b'"method":"tools/call"', b'"method":"tools/list"'),
                        body.replace(b'"arguments":', b'"Arguments":'), body.replace(b",", b" ,\n"), body[:-1] + b',"extra":1}',
                        body.replace(b'"jsonrpc"', b'"JSONRPC"'), body.replace(b'"params":{', b'"params":{"name":"x",'),
                        b'{"jsonrpc":"2.0","id":1,"method":"tools/call","params":{"name":"' + tool + b'"}}')[i % 8:i % 8 + 1]:
            _check_request(oracle, hsim, variant, i)
    assert total > 100 and handled > total // 4


def test_request_envelope_vectors_and_bench_shapes(oracle, hsim):
    import benchgen
    from test_oracle import K_BODIES
    for k, (body, args, wire, rmsg, rwire, pj, http) in enumerate(K_BODIES):
        _check_request(oracle, hsim, body, k)
    by_input = _tool_by_input(oracle)
    wl = benchgen.nested(120, oracle.msg)
    blob = wl.req_json.tobytes()
    for i in range(120):
        js = blob[int(wl.req_off[i]):int(wl.req_off[i + 1])]
        tool = by_input[int(wl.req_msg[i])][1].encode()
        body = b'{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"%s","arguments":%s}}' % (i, tool, js)
        r = oracle.request(body)
        rc, w, method, idt = hsim.request_coop(body, i % 16, (i * 3) % 16, 1)
        assert rc == 0 and r["kind"] == 0 and w == r["wire"] and method == r["method"] and idt == r["id"]


def test_request_envelope_numbers(oracle, hsim):
    """json.Marshal(arguments) passes every number through float64: literals that are not plain short integers
    take the same round trip on the device (text -> float64 -> shortest text -> the field's parser)"""
    rng = random.Random(5)
    kinds = ["int32", "int64", "uint32", "uint64", "sint32", "sint64", "fixed32", "fixed64", "sfixed32", "sfixed64", "float", "double"]

    def lit():
        c = rng.random()
        if c < 0.15:
            return str(rng.randrange(-200, 200))
        if c < 0.3:
            return str(rng.choice([2**31 - 1, 2**31, -2**31, 2**32 - 1, 2**53, 2**53 + 1, 2**63 - 1, 2**63, -2**63, 2**64 - 1, 2**64,
                                   9007199254740993, 123456789012345678]))
        if c < 0.45:
            return "%d.%s" % (rng.randrange(-50, 50), rng.choice(["0", "5", "25", "000", "10"]))
        if c < 0.6:
            return "%de%d" % (rng.randrange(-99, 99), rng.randrange(0, 22))
        if c < 0.7:
            return "%d.%de%s%d" % (rng.randrange(0, 9), rng.randrange(0, 999), rng.choice(["", "+", "-"]), rng.randrange(0, 40))
        if c < 0.8:
            return repr(rng.uniform(-1e6, 1e6))
        if c < 0.9:
            return rng.choice(["-0", "-0.0", "0.0", "1e400", "1e-400", "0.1", "3.4028235e38", "3.4028236e38", "1.7976931348623157e308",
                               "4.9e-324", "16777217", "0.30000000000000004"])
        return rng.choice(["1.5", "2.5", "1e21", "1e20", "123456789012345678901234567890", "0.000001", "0.0000001", "1E3", "1e+3", "-1e-7"])

    handled = accepted_by_oracle = 0
    for it in range(1500):
        fs = rng.sample(kinds, rng.randrange(1, 5))
        args = "{" + ",".join('"f_%s":%s' % (k, lit()) for k in fs)
        if rng.random() < 0.3:
            args += ',"r_double":[%s]' % ",".join(lit() for _ in range(rng.randrange(0, 4)))
        args += "}"
        body = ('{"jsonrpc":"2.0","id":%d,"method":"tools/call","params":{"name":"bench_benchservice_echoall","arguments":%s}}' % (it, args)).encode()
        handled += _check_request(oracle, hsim, body, it)
        accepted_by_oracle += oracle.request(body)["kind"] == 0
    assert handled == accepted_by_oracle and handled > 200  # nothing the reference accepts is left to the host here


def test_mixed_replay_shapes(oracle, hsim):
    """configs[4] (32 methods, Zipf sizes): the per-thread device code against the oracle on a sample, and the
    token-parallel walker against the per-thread code"""
    import benchgen
    names = {}

    def mi(name):
        names[hsim.msg(name)] = name
        return hsim.msg(name)

    wl = benchgen.mixed(1500, mi)
    assert len(set(wl.method.tolist())) >= 24  # the popular methods dominate, most of the 32 still show up
    jb, wb = wl.req_json.tobytes(), wl.rep_wire.tobytes()
    walked = 0
    for i in range(wl.n):
        js = jb[int(wl.req_off[i]):int(wl.req_off[i + 1])]
        w = wb[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]
        if len(js) > 20000 or len(w) > 20000:
            continue  # the large ones: GPU test
        rn, pn = names[int(wl.req_msg[i])], names[int(wl.rep_msg[i])]
        rc, ow, _ = oracle.encode(rn, js)
        st, ew = hsim.encode(rn, js, i % 16, (i * 3) % 16)
        assert rc == 0 and st == 0 and ew == ow, (rn, js[:300])
        walked += _check_walk(hsim, rn, js, i)
        rc, oj, _ = oracle.decode(pn, w)
        st, ej = hsim.decode(pn, w, 0, i % 16, (i * 7) % 16)
        assert rc == 0 and st == 0 and ej == oj, (pn, w.hex()[:300])
    assert walked > 150  # floats, bytes, quoted numbers, timestamps: the fused kernel
    # request side, large items: the three walker tiers (the third: up to 8192 values) against the oracle
    huge = 0
    for i in range(wl.n):
        js = jb[int(wl.req_off[i]):int(wl.req_off[i + 1])]
        if len(js) <= 20000 or len(js) > 64000:
            continue
        rn = names[int(wl.req_msg[i])]
        rc, out = hsim.encode_walk(rn, js, i % 16, (i * 5) % 16)
        assert rc in (0, 200), (rn, rc)
        if rc == 0:
            rc2, ow, _ = oracle.encode(rn, js)
            assert rc2 == 0 and out == ow, (rn, len(js))
            huge += 1
    assert huge >= 5, huge
    # reply side, both lock-step tiers (the second one: tables of up to 4096 entries saved in a pool) on every reply of
    # the sample, the large ones included
    taken = big = 0
    for i in range(wl.n):
        w = wb[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]
        pn = names[int(wl.rep_msg[i])]
        rc, out = hsim.decode_coop(pn, w, 0, i % 16, (i * 5) % 16)
        assert rc in (0, 200), (pn, rc)
        if rc == 0:
            rc2, oj, _ = oracle.decode(pn, w)
            assert rc2 == 0 and out == oj, (pn, len(w))
            taken += 1
            big += len(w) > 6000
    assert taken > wl.n // 3 and big >= 5, (taken, big)


def test_decode_unsorted_maps(oracle, hsim):
    """maps as a Go backend sends them (iteration order, not key order), with duplicate keys: the sort-pool path of the
    per-thread walker against the oracle, for string, signed and unsigned keys, in the fast and in the slow walk"""
    rng = random.Random(44)

    def varint(v):
        out = bytearray()
        while v >= 0x80:
            out.append(v & 0x7F | 0x80)
            v >>= 7
        out.append(v)
        return bytes(out)

    def ld(num, payload):
        return varint(num << 3 | 2) + varint(len(payload)) + payload

    for trial in range(12):
        n = rng.choice([9, 40, 300])
        ent = []
        for i in range(n):
            # trials 4..: keys that agree in their first eight bytes and beyond (the sort records carry an 8-byte prefix)
            k = ("k%d_%s" if trial < 4 else ("shared__%d_%s" if trial < 8 else "%04d%s"))  % (rng.randrange(n), "x" * rng.randrange(3) + "\0" * rng.randrange(2))
            ent.append(ld(41, ld(1, k.encode()) + varint(2 << 3) + varint(rng.randrange(1 << 31))))              # m_str_int32
        for i in range(n):
            ent.append(ld(42, varint(1 << 3) + varint(rng.randrange(n) ^ ((1 << 64) - 1 if rng.random() < 0.3 else 0)) + ld(2, b"v%d" % i)))  # m_int32_str
        for i in range(n // 2):
            ent.append(ld(45, varint(1 << 3) + varint(rng.randrange(1 << 40)) + ld(2, bytes([i & 255]) * 3)))   # m_uint64_bytes
        wire = b"".join(ent)
        if trial & 1:
            wire = varint(100 << 3 | 2) + varint(1) + b"z" + wire  # z_last first: fields out of declaration order -> slow walk
        rc, oj, _ = oracle.decode(cases.A, wire)
        st, ej = hsim.decode(cases.A, wire, 0, trial % 16, (trial * 3) % 16)
        assert rc == 0 and st == 0 and ej == oj, (trial, n)


def test_byte_run_copies(hsim):
    """coop_copy_bytes (with the general word-copy threshold and the two the kernels use) / coop_copy_words (ggr_warp.cuh):
    every source and destination alignment, every length up to 300, against a byte-wise reference; nothing outside the
    destination run may change"""
    import ctypes as C
    import hostsim
    L = hostsim.lib()
    L.hs_copy_selftest.argtypes = [C.c_uint32]
    assert L.hs_copy_selftest(300) == 0


# ---- float and double text conversion against the exact reference (numref) ------------------------------------
_num_cache = {}


def _num_corpus():
    import numcorpus as NC
    if not _num_cache:
        lits = NC.request_literals()
        _num_cache["req"] = NC.request_items(lits)
        _num_cache["bodies"] = NC.body_items(lits)
        _num_cache["rep"] = NC.reply_items(NC.reply_bits(64, n_random=30000), NC.reply_bits(32, stride=65521))
    return _num_cache


def _wire_matches(st, out, want):
    import numref
    return st != 0 if want == numref.RANGE else (st == 0 and out == want)


def test_numbers_request_per_thread(hsim):
    """halfway points written exactly, just above and just below with the deciding digit up to 1500 significant
    digits in, fast-path edges, float32 double-rounding traps: the per-thread parser rounds like strconv.ParseFloat"""
    bad = [(n, js[:120]) for i, (n, js, want) in enumerate(_num_corpus()["req"]) if not _wire_matches(*hsim.encode(n, js, i % 16, (i * 5) % 16), want)]
    assert not bad, (len(bad), bad[:5])


@pytest.mark.parametrize("tier", [0, 1])
def test_numbers_request_lockstep(hsim, tier):
    """the lock-step parser either leaves an item to the per-thread parser (200) or gives the exact bytes"""
    handled = 0
    for i, (n, js, want) in enumerate(_num_corpus()["req"]):
        rc, out = hsim.encode_coop(n, js, i % 16, (i * 5) % 16, tier)
        if rc == 200:
            continue
        assert _wire_matches(rc, out, want), (n, js[:120], rc)
        handled += 1
    assert handled > len(_num_corpus()["req"]) // 2


def test_numbers_request_envelope(hsim):
    """tools/call bodies: a bare literal takes json.Marshal's float64 round trip, a quoted one reaches the field as
    written; every body is taken, a literal out of float64 range is refused"""
    import numref
    for i, (body, want) in enumerate(_num_corpus()["bodies"]):
        rc, wire, method, idt = hsim.request_coop(body, i % 16, (i * 3) % 16, i & 1)
        if want == numref.RANGE:
            assert rc != 0, body[:200]
        else:
            assert rc == 0 and wire == want, (body[:200], rc, wire.hex())


def test_numbers_reply(hsim):
    """shortest round-trip text of doubles and floats in packed runs, unpacked occurrences, singular fields, map
    values and wrappers; the lock-step reply side gives the same text or leaves the item (200)"""
    taken = 0
    for i, (n, w, want) in enumerate(_num_corpus()["rep"]):
        rc, out = hsim.decode(n, w, 0, i % 16, (i * 5) % 16)
        assert rc == 0 and out == want, (n, w.hex()[:80], out[:200], want[:200])
        rc, out = hsim.decode_coop(n, w, 0, i % 16, (i * 5) % 16)
        assert rc == 200 or (rc == 0 and out == want), (n, w.hex()[:80], rc, out[:200], want[:200])
        taken += rc == 0
    assert taken > 1000
