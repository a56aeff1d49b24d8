"""CPU tests that pin the oracle: the reference's own pinned vectors (SURVEY.md 8c, Appendix C),
Go float formatting against Python's shortest repr, and wire/JSON cross-checks against
python-protobuf (upb), the secondary oracle."""
import json
import math
import random
import struct

import pytest

import cases
import numref
import orc
import pbgen

K_BODIES = [
    # (HTTP body, canonical args, request wire hex, reply message, reply wire hex, protojson, HTTP response body)
    (b'{"jsonrpc":"2.0","method":"tools/call","id":2,"params":{"name":"hello_helloservice_sayhello","arguments":{"name":"World","email":"test@example.com"}}}',
     b'{"email":"test@example.com","name":"World"}', "0a05576f726c64121074657374406578616d706c652e636f6d", "hello.HelloReply",
     "0a2b48656c6c6f20576f726c642120596f757220656d61696c2069732074657374406578616d706c652e636f6d",
     b'{"message":"Hello World! Your email is test@example.com"}',
     b'{"jsonrpc":"2.0","result":{"content":[{"type":"text","text":"{\\"message\\":\\"Hello World! Your email is test@example.com\\"}"}]},"id":2}\n'),
    ('{"jsonrpc":"2.0","method":"tools/call","id":"abc","params":{"name":"com_example_complex_userprofileservice_getuserprofile","arguments":{"user_id":"premium"}}}'.encode(),
     b'{"user_id":"premium"}', "0a077072656d69756d", cases.P + "GetUserProfileResponse",
     "0a3b0a077072656d69756d1211546573742055736572207072656d69756d1a137072656d69756d406578616d706c652e636f6d20022a0608c0d2caac06",
     b'{"profile":{"userId":"premium","displayName":"Test User premium","email":"premium@example.com","userType":"PREMIUM","lastLogin":"2024-01-01T12:00:00Z"}}',
     b'{"jsonrpc":"2.0","result":{"content":[{"type":"text","text":"{\\"profile\\":{\\"userId\\":\\"premium\\",\\"displayName\\":\\"Test User premium\\",\\"email\\":\\"premium@example.com\\",\\"userType\\":\\"PREMIUM\\",\\"lastLogin\\":\\"2024-01-01T12:00:00Z\\"}}"}]},"id":"abc"}\n'),
    ('{"jsonrpc":"2.0","method":"tools/call","id":5,"params":{"name":"com_example_complex_nodeservice_processnode","arguments":{"root_node":{"id":"root","value":"Root Node","children":[{"id":"child1","value":"Child 1"},{"id":"child2","value":"Child 2","children":[{"id":"grandchild1","value":"Grandchild 1"}]}]}}}}'.encode(),
     cases.K_REQUESTS[5][1], cases.K_REQUESTS[5][2], cases.P + "ProcessNodeResponse",
     "0a2450726f6365737365642074726565207769746820726f6f742027526f6f74204e6f6465271004",
     b'{"processedSummary":"Processed tree with root \'Root Node\'","totalNodes":4}',
     b'{"jsonrpc":"2.0","result":{"content":[{"type":"text","text":"{\\"processedSummary\\":\\"Processed tree with root \'Root Node\'\\",\\"totalNodes\\":4}"}]},"id":5}\n'),
]


def test_tool_names(oracle):
    tools = [m["tool"] for m in oracle.methods()]
    # pkg/grpc/discovery_integration_test.go:140, tests/complex_service_translation_test.go:48-52
    assert "hello_helloservice_sayhello" in tools
    assert "com_example_complex_userprofileservice_getuserprofile" in tools
    assert "com_example_complex_documentservice_createdocument" in tools
    assert "com_example_complex_nodeservice_processnode" in tools
    paths = [m["path"] for m in oracle.methods()]
    assert "/com.example.complex.UserProfileService/GetUserProfile" in paths  # real_grpc_invocation_test.go:324-360


@pytest.mark.parametrize("k", range(len(K_BODIES)))
def test_end_to_end_vectors(oracle, k):
    body, args, wire, rmsg, rwire, pj, http = K_BODIES[k]
    r = oracle.request(body)
    assert r["kind"] == 0
    assert r["args"] == args
    assert r["wire"].hex() == wire
    rc, out, _ = oracle.decode(rmsg, bytes.fromhex(rwire))
    assert rc == 0 and out == pj
    rc, b = oracle.response(rmsg, bytes.fromhex(rwire), r["id"])
    assert rc == 0 and b == http


def test_pinned_boundary_string(oracle):
    # pkg/server/handler_header_test.go:128: arguments {"input":"test"} reach the boundary verbatim
    rc, out = orc.canon_json(b'{"input":"test"}')
    assert rc == 0 and out == b'{"input":"test"}'
    rc, out = orc.canon_json(b' { "b" : 1e2 , "a" : [ 1.0 , "<&>" , 9007199254740993 ] , "b" : 2 } ')
    assert out == b'{"a":[1,"\\u003c\\u0026\\u003e",9007199254740992],"b":2}'


@pytest.mark.parametrize("name,js,wire", cases.K_REQUESTS)
def test_request_vectors(oracle, name, js, wire):
    rc, out, err = oracle.encode(name, js)
    assert rc == 0, err
    assert out.hex() == wire


@pytest.mark.parametrize("name,wire,js", cases.K_REPLIES)
def test_reply_vectors(oracle, name, wire, js):
    rc, out, err = oracle.decode(name, bytes.fromhex(wire))
    assert rc == 0, err
    assert out == js
    rc, out2, _ = oracle.decode(name, bytes.fromhex(wire), orc.F_COMMA_SPACE)
    assert out2 == js.replace(b',"', b', "')


def test_error_envelopes(oracle):
    # tests/real_grpc_invocation_test.go:238-245: unknown field -> isError result containing "unknown field"
    r = oracle.request(b'{"jsonrpc":"2.0","method":"tools/call","id":7,"params":{"name":"com_example_complex_nodeservice_processnode","arguments":{"invalid_field":"value"}}}')
    assert r["kind"] == 2 and r["status"] == orc.UNKNOWN_FIELD
    assert b"unknown field" in r["resp"] and b'"isError":true' in r["resp"]
    # tests/integration_test.go:341-352: parse error -> -32700 "Parse error", id null
    r = oracle.request(b'{"jsonrpc":"2.0","method":')
    assert r["kind"] == 1 and r["resp"] == b'{"jsonrpc":"2.0","error":{"code":-32700,"message":"Parse error"},"id":null}\n'
    r = oracle.request(b'{"jsonrpc":"2.0","method":"nope","id":1}')
    assert b'"code":-32601' in r["resp"] and b"method not found: nope" in r["resp"]
    r = oracle.request(b'{"jsonrpc":"1.0","method":"tools/call","id":1}')
    assert b'"code":-32600' in r["resp"] and b"must be '2.0'" in r["resp"]
    r = oracle.request(b'{"jsonrpc":"2.0","method":"tools/call","id":1,"params":{"arguments":{}}}')
    assert b'"code":-32602' in r["resp"]
    # depth: params is depth 0, so an object nested 11 deep under it is rejected (validation.go:163-184)
    deep = b'{"a":' * 11 + b"1" + b"}" * 11
    r = oracle.request(b'{"jsonrpc":"2.0","method":"tools/call","id":1,"params":{"name":"x","arguments":' + deep + b"}}")
    assert b"nesting too deep" in r["resp"]
    # unknown tool -> tool-call error result, sanitized ("tool ... not found" has no secret words)
    r = oracle.request(b'{"jsonrpc":"2.0","method":"tools/call","id":1,"params":{"name":"nope_tool","arguments":{}}}')
    assert r["kind"] == 2 and b"tool nope_tool not found" in r["resp"]


def test_float_format_matches_shortest_repr():
    rng = random.Random(7)
    for i in range(20000):
        if i % 3 == 0:
            v = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
        elif i % 3 == 1:
            v = rng.uniform(-1, 1) * 10 ** rng.randint(-30, 30)
        else:
            v = float(rng.randint(-10 ** rng.randint(1, 18), 10 ** rng.randint(1, 18)))
        if v != v or math.isinf(v):
            continue
        assert orc.format_float(v) == numref.format_float(v), repr(v)
    for v, s in [(1.0, "1"), (1e21, "1e+21"), (1e-7, "1e-7"), (1e-6, "0.000001"), (123456789012345680000.0, "123456789012345680000"),
                 (5e-324, "5e-324"), (-0.0, "-0")]:
        assert orc.format_float(v) == s
    assert orc.format_float(3.4028234663852886e38, 32) == "3.4028235e+38"
    assert orc.format_float(0.10000000149011612, 32) == "0.1"


def test_float32_format_matches_numpy():
    """float32 printing: the oracle's shortest digits equal numpy's shortest float32 on a strided sweep of all bit
    patterns (with both layouts and their switch points), through numref's layout"""
    import numpy as np
    bits = np.arange(0, 1 << 32, 21011, dtype=np.uint64).astype(np.uint32)
    bits = np.concatenate([bits, np.array([numref.parse(t, 32) + d for t in ("1e-6", "1e21") for d in (-1, 0, 1)], np.uint32)])
    vals = bits.view(np.float32)
    n = 0
    for b, v in zip(bits.tolist(), vals.tolist()):
        if v != v or math.isinf(v):
            continue
        assert orc.format_float(v, 32) == numref.format(b, 32), hex(b)
        n += 1
    assert n > 200000


def test_number_corpus_matches_numref(oracle):
    """the oracle rounds like strconv.ParseFloat and prints like strconv.AppendFloat on the number corpus: request
    literals in every float position, tools/call bodies, and a reply sample"""
    import numcorpus as NC
    lits = NC.request_literals()
    for n, js, want in NC.request_items(lits):
        rc, out, _ = oracle.encode(n, js)
        assert (rc != 0) if want == numref.RANGE else (rc == 0 and out == want), (n, js[:120], rc)
    for body, want in NC.body_items(lits):
        r = oracle.request(body)
        assert (r["kind"] != 0) if want == numref.RANGE else (r["kind"] == 0 and r["wire"] == want), body[:200]
    for n, w, want in NC.reply_items(NC.reply_bits(64, n_random=20000), NC.reply_bits(32, stride=99991)):
        rc, out, _ = oracle.decode(n, w)
        assert rc == 0 and out == want, (n, w.hex()[:80], out[:200], want[:200])


def _json_equal(a, b):
    """structural equality of two protojson texts, floats compared as floats"""
    return json.loads(a, parse_int=float) == json.loads(b, parse_int=float)


def test_oracle_vs_upb():
    """wire bytes: identical to upb's deterministic serialization; JSON: equal after parsing."""
    O = orc.load_schema()
    names = [cases.A, cases.P + "CreateDocumentRequest", cases.P + "ProcessNodeRequest", cases.P + "GetUserProfileResponse",
             "bench.Flat", "bench.Blob", "wkt.Wkt"]
    for name in names:
        for seed in range(120):
            m = pbgen.random_message(name, seed, floats=True)
            W = pbgen.wire(m)
            for pn in (False, True):
                J = pbgen.to_json(m, pn).encode()
                rc, out, err = O.encode(name, J)
                assert rc == 0, (name, seed, err)
                if out != W:
                    # allowed differences: NaN payload bits (Go math.NaN() vs upb) and upb's own
                    # ordering of sint32/sint64 map keys (Go's GenericKeyOrder is numeric, which
                    # the oracle follows).  Anything else must re-serialize to upb's bytes.
                    if "NaN" in J.decode():
                        continue
                    m2 = pbgen.cls(name)()
                    m2.ParseFromString(out)
                    assert pbgen.wire(m2) == W, (name, seed)
            rc, out, err = O.decode(name, W)
            assert rc == 0, (name, seed, err)
            text = out.decode()
            # python's JSON reader loses the sign of -0 and rejects float32 values near FLT_MAX
            # printed in shortest form; NaN payloads differ - skip those for the round trip
            if "NaN" in text or "Infinity" in text or "e+38" in text or any(s in text for s in ("-0,", "-0]", "-0}")):
                continue
            from google.protobuf import json_format
            m3 = json_format.Parse(text, pbgen.cls(name)())
            assert pbgen.wire(m3) == W, (name, seed)


def test_descriptor_set_route_tool_names(fds_bytes):
    """the FileDescriptorSet route shortens the service name to its last package segment
    (/root/reference/pkg/descriptors/loader.go:221-235; names pinned by pkg/grpc/discovery_edge_cases_test.go:62-66)"""
    import orc
    S = orc.Schema(fds_bytes, naming=1)
    tools = {m["tool"] for m in S.methods()}
    assert "complex_userprofileservice_getuserprofile" in tools
    assert "hello_helloservice_sayhello" in tools        # one package segment: unchanged
    assert "com_example_complex_userprofileservice_getuserprofile" not in tools
    body = b'{"jsonrpc":"2.0","method":"tools/call","id":1,"params":{"name":"complex_userprofileservice_getuserprofile","arguments":{"user_id":"u"}}}'
    r = S.request(body)
    assert r["kind"] == 0 and r["wire"] == bytes.fromhex("0a0175")
