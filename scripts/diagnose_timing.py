"""Error detail of a request batch: one ggr_encode_diagnose_batch call against a loop of ggr_encode_diagnose over the same
failing items, both called through ctypes on buffers prepared once.  The batch is the nested workload (benchgen.nested)
with a share of its items damaged by cases.mutate_json; both forms take host buffers and end in a device synchronise, so
the host clock around them is the call time.  Prints one JSON line with the GPU's name and power limit read in the same
run.

    python scripts/diagnose_timing.py [--items 100000] [--damaged 0.01] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import benchgen  # noqa: E402
import cases  # noqa: E402
import ggrmcp_b200  # noqa: E402
from ggrmcp_b200.engine import pack, unpack  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().split(",", 1))
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=100000)
    ap.add_argument("--damaged", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = gpu_info()
    fds = open(os.path.join(ROOT, "tests", "golden", "schemas.binpb"), "rb").read()
    eng = ggrmcp_b200.Engine(0)
    schema = eng.register(fds)
    wl = benchgen.nested(a.items, schema.message)
    items = unpack(wl.req_json, wl.req_off)
    rng = random.Random(7)
    for i in rng.sample(range(a.items), int(a.items * a.damaged)):
        items[i] = cases.mutate_json(items[i], rng)
    data, off = pack(items)
    ids = wl.req_msg
    _, _, st = eng.encode_batch(schema, ids, data, off)
    st = np.array(st, np.int32)
    failing = np.flatnonzero(st != 0)

    # the C calls themselves, on buffers prepared once
    L = ggrmcp_b200.engine._load()
    L.ggr_encode_diagnose.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_char_p, C.c_size_t]
    n = len(ids)
    cap = 128 * len(failing) + 64
    text, text_off = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint64)
    pos, ln = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    one = [(int(ids[i]), items[i]) for i in failing]
    s1, p1, l1, buf = C.c_int32(), C.c_uint32(), C.c_uint32(), C.create_string_buffer(1 << 16)

    def batch():
        rc = L.ggr_encode_diagnose_batch(eng.h, schema.h, n, ids.ctypes.data, data.ctypes.data, off.ctypes.data, st.ctypes.data,
                                         pos.ctypes.data, ln.ctypes.data, text.ctypes.data, cap, text_off.ctypes.data)
        assert rc == 0, rc

    def loop():
        out = []
        for m, js in one:
            rc = L.ggr_encode_diagnose(eng.h, schema.h, m, js, len(js), 0, C.byref(s1), C.byref(p1), C.byref(l1), buf, len(buf))
            assert rc == 0, rc
            out.append((s1.value, p1.value, l1.value, buf.value))
        return out

    batch()
    single = loop()
    for k, i in enumerate(failing):  # both give the same answers (the single-item text ends at its NUL)
        t = text[int(text_off[i]):int(text_off[i + 1])].tobytes().split(b"\0")[0]
        assert single[k] == (int(st[i]), int(pos[i]), int(ln[i]), t), i
    tb, tl = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        batch()
        tb.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        loop()
        tl.append((time.perf_counter() - t0) * 1e3)
    b, l = statistics.median(tb), statistics.median(tl)
    print(json.dumps({"gpu": name, "power_limit": power, "items": a.items, "input_bytes": int(off[-1]), "failing": int(len(failing)),
                      "diagnose_batch_ms": round(b, 3), "single_item_loop_ms": round(l, 3), "speedup": round(l / b, 1),
                      "batch_ms_all": [round(x, 3) for x in tb], "loop_ms_all": [round(x, 3) for x in tl]}))
    eng.close()


if __name__ == "__main__":
    main()
