"""The error-text pass of ggr_encode_diagnose_batch (ggrmcp_b200/csrc/ggr_diag.cuh) in the host simulation, one warp of
32 fibers per item, against a plain restatement of the rule the header gives: position clamped to the item, key token up
to the next quote no backslash escapes, line and column in bytes from 1, protojson's wording or the status name."""
import ctypes as C
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATUS_NAMES = ["ok", "syntax", "unknown_field", "invalid_value", "range", "invalid_utf8", "duplicate",
                "oneof_conflict", "depth", "too_large", "bad_wire", "unsupported", "no_space", "internal"]


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("diagsim") / "libdiagsim.so")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-x", "c++", "-shared", "-o", lib,
                           os.path.join(ROOT, "tests", "hostsim", "diagsim.cc")])
    L = C.CDLL(lib)
    L.ds_diagnose.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_int32, C.c_uint32, C.POINTER(C.c_uint32), C.c_char_p, C.c_uint32,
                              C.POINTER(C.c_uint32)]
    return L


def run(sim, js, st, raw_pos, phase=0):
    res = (C.c_uint32 * 4)()
    cap = len(js) + 128
    text = C.create_string_buffer(cap)
    n = C.c_uint32()
    rc = sim.ds_diagnose(js, len(js), phase, st, raw_pos, res, text, cap, C.byref(n))
    assert rc == 0, (js[:80], st, raw_pos, phase, rc)
    return res[0], res[1], res[2], res[3], text.raw[: n.value]


def reference(js, st, raw_pos):
    """(pos, token length, line, column, text) as ggr_encode_diagnose composed them on the host"""
    if st == 0:
        return 0, 0, 1, 1, b""
    pos = min(raw_pos, len(js))
    ln = 0
    if pos < len(js) and js[pos] == ord('"'):
        q = pos + 1
        while q < len(js) and js[q] != ord('"'):
            q += 2 if js[q] == ord("\\") else 1
        if q < len(js):
            ln = q + 1 - pos
    line, col = 1, 1
    for c in js[:pos]:
        if c == ord("\n"):
            line, col = line + 1, 1
        else:
            col += 1
    tok = js[pos:pos + ln]
    text = b"proto: (line %d:%d): " % (line, col)
    if st == 2 and ln:
        text += b"unknown field " + tok
    elif st == 6 and ln:
        text += b"duplicate field " + tok
    elif st == 7 and ln:
        text += b"error parsing " + tok + b", oneof is already set"
    else:
        text += (STATUS_NAMES[st] if 0 <= st < len(STATUS_NAMES) else "?").encode()
    return pos, ln, line, col, text


def check(sim, js, st, raw_pos, phase=0):
    got = run(sim, js, st, raw_pos, phase)
    assert got == reference(js, st, raw_pos), (js[:120], st, raw_pos, phase, got)


KEYS = [b'"a"', b'"a\\"b"', b'"a\\\\"', b'"a\\\\\\"b"', b'"\\"', b'"abc', b'"abc\\', b'"\xc3\xa9t\xc3\xa9"', b'"x\\u0022y"',
        b'"' + b"\\" * 40 + b'"', b'"' + b"\\" * 41 + b'"q"', b'"' + b"k" * 70 + b'"'] + \
       [b'"' + b"a" * k + b"\\" * r + b'"x"' for k in (28, 29, 30, 31, 62, 63) for r in (1, 2, 3)]  # runs that end a 32-byte window


@pytest.mark.parametrize("phase", [0, 1, 7, 15])
def test_key_tokens(sim, phase):
    """escaped quotes, escaped backslashes, runs of backslashes across the 32-byte windows, a trailing backslash and a
    missing closing quote, for the three wordings that print the token and one that does not"""
    for key in KEYS:
        for lead in (b"", b"{", b'{"user_id":"a",\n  '):
            for tail in (b"", b":1}", b"\n}"):
                js = lead + key + tail
                for st in (2, 6, 7, 1):
                    check(sim, js, st, len(lead), phase)


def test_lines_and_columns(sim):
    """several lines and non-ASCII bytes (columns count bytes), newlines right before and right at the position, items
    longer than one 512-byte step of the warp, every start offset mod 16"""
    rng = random.Random(3)
    body = b'{\n "a": "\xc3\xa9\xe2\x82\xac\xff",\n\n  "b":\t[1,\n2]\n' + b"".join(b'  "k%d": "%s",\n' % (k, b"\xce\xbb" * k) for k in range(60)) + b"}"
    for phase in range(16):
        for pos in [0, 1, 2, 3, len(body) // 2, len(body) - 1, len(body), len(body) + 5] + [rng.randrange(len(body)) for _ in range(8)]:
            check(sim, body, 1, pos, phase)
    nl = [i for i, c in enumerate(body) if c == ord("\n")]
    for i in nl[:5] + nl[-5:]:
        check(sim, body, 3, i, 0)
        check(sim, body, 3, i + 1, 0)


def test_positions_at_the_ends(sim):
    for js in (b"", b"x", b"\n", b'"', b'{"a":1}', b"\n" * 600, b'"' + b"a" * 600):
        for st in range(15):
            for pos in (0, len(js), 0xFFFFFFFF):
                check(sim, js, st, pos, 5)


def test_random_items(sim):
    """random items over the bytes that matter (newline, quote, backslash) and a few others, random statuses and positions"""
    rng = random.Random(11)
    alphabet = b'\n"\\\\a{}:\xc3\xa9 '
    for _ in range(400):
        n = rng.choice([rng.randrange(40), rng.randrange(700), rng.randrange(3000)])
        js = bytes(rng.choice(alphabet) for _ in range(n))
        check(sim, js, rng.choice([1, 2, 2, 6, 6, 7, 7, 9, 11]), rng.randrange(n + 3), rng.randrange(16))
