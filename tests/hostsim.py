"""ctypes binding of tests/hostsim/libggr_hostsim.so - the host simulation of the device code."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIR = os.path.join(ROOT, "tests", "hostsim")
LIB = os.path.join(DIR, "libggr_hostsim.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", DIR])
        L = C.CDLL(LIB)
        L.hs_schema_new.restype = C.c_void_p
        L.hs_schema_new.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_char_p, C.c_size_t]
        L.hs_msg_index.argtypes = [C.c_void_p, C.c_char_p]
        L.hs_encode.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p,
                                C.c_uint32, C.POINTER(C.c_uint32)]
        L.hs_encode_coop.argtypes = L.hs_encode.argtypes + [C.c_int]
        L.hs_encode_walk.argtypes = L.hs_encode.argtypes
        if hasattr(L, "hs_decode_coop"):
            L.hs_decode_coop.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                         C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32)]
        if hasattr(L, "hs_decode"):
            L.hs_decode.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                    C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.hs_request_coop.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_uint32,
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_int]
        L.hs_wrap.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.hs_keep_state.argtypes = [C.c_int]
        _lib = L
    return _lib


def keep_state(on):
    """on: the lock-step entry points keep their per-warp structures from one item to the next, as persistent warps do;
    off (the default): every item starts on structures filled with 0xAB"""
    lib().hs_keep_state(1 if on else 0)


def wrap(text, id_tok):
    """MCP result body around a protojson text (host simulation of ggr_wrap.cuh)"""
    cap = len(text) * 6 + len(id_tok) + 128
    out = C.create_string_buffer(cap)
    n = C.c_uint32()
    rc = lib().hs_wrap(text, len(text), id_tok, len(id_tok), out, cap, C.byref(n))
    return rc, out.raw[: n.value]


class Schema:
    def __init__(self, fds, order=0):
        err = C.create_string_buffer(256)
        self.h = lib().hs_schema_new(fds, len(fds), order, err, 256)
        if not self.h:
            raise ValueError(err.value.decode())

    def msg(self, name):
        i = lib().hs_msg_index(self.h, name.encode())
        if i < 0:
            raise KeyError(name)
        return i

    def encode(self, name, data, in_off=0, out_off=0):
        cap = 2 * len(data) + 64  # a FieldMask can double: "A," -> tag, length, "_a"
        out = C.create_string_buffer(cap)
        n = C.c_uint32()
        rc = lib().hs_encode(self.h, self.msg(name), data, len(data), in_off, out_off, out, cap, C.byref(n))
        return rc, out.raw[: n.value]

    def decode(self, name, data, flags=0, in_off=0, out_off=0):
        cap = len(data) * 8 + 256
        out = C.create_string_buffer(cap)
        n = C.c_uint32()
        rc = lib().hs_decode(self.h, self.msg(name), data, len(data), in_off, out_off, flags, out, cap, C.byref(n))
        return rc, out.raw[: n.value]


def _decode_coop(self, name, data, flags=0, in_off=0, out_off=0):
    cap = len(data) * 8 + 256
    out = C.create_string_buffer(cap)
    n = C.c_uint32()
    rc = lib().hs_decode_coop(self.h, self.msg(name), data, len(data), in_off, out_off, flags, out, cap, C.byref(n))
    return rc, out.raw[: n.value]


Schema.decode_coop = _decode_coop


def _encode_coop(self, name, data, in_off=0, out_off=0, tier=0):
    cap = len(data) + 64
    out = C.create_string_buffer(cap)
    n = C.c_uint32()
    rc = lib().hs_encode_coop(self.h, self.msg(name), data, len(data), in_off, out_off, out, cap, C.byref(n), tier)
    return rc, out.raw[: n.value]


Schema.encode_coop = _encode_coop


def _encode_walk(self, name, data, in_off=0, out_off=0):
    """token-parallel walker (ggr_walk.cuh): token index, walker, lock-step emitter"""
    cap = len(data) + 64
    out = C.create_string_buffer(cap)
    n = C.c_uint32()
    rc = lib().hs_encode_walk(self.h, self.msg(name), data, len(data), in_off, out_off, out, cap, C.byref(n))
    return rc, out.raw[: n.value]


Schema.encode_walk = _encode_walk


def load_schema(order=0):
    with open(os.path.join(ROOT, "tests", "golden", "schemas.binpb"), "rb") as fh:
        return Schema(fh.read(), order)


def _request_coop(self, body, in_off=0, out_off=0, tier=0):
    """request envelope through the lock-step parser: (rc, wire, method index, id token)"""
    cap = len(body) + 64
    out = C.create_string_buffer(cap)
    n = C.c_uint32()
    env = (C.c_uint32 * 3)()
    rc = lib().hs_request_coop(self.h, body, len(body), in_off, out_off, out, cap, C.byref(n), env, tier)
    return rc, out.raw[: n.value], int(env[0]), body[env[1]: env[1] + env[2]]


Schema.request_coop = _request_coop
