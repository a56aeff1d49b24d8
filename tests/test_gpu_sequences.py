"""Persistent warps on the device: the long shuffled batches of tests/seqcorpus.py through the device-resident entry points
(ggr_encode_batch_dev, ggr_decode_batch_dev, ggr_request_batch_dev, ggr_decode_wrap_batch_dev), where one launch gives
every warp of every lock-step list a long run of items, and through the host entry points in one chunk.

The reference answer of each unique item comes from the same engine path, in calls of at most REF_CALL items, and is held
to the oracle by the rules of the other GPU tests.  (A warp holds two tickets at a time, so in such a call some warps still
process two items; what the reference answers rest on is the oracle, not a fresh warp.)  In the long batches every item
must then give exactly its reference status, bytes, method and id span, whatever the same warp processed before it; the
second call of each pair, on another stream and in another order, starts on the scratch area the first one left."""
import os
import time

import numpy as np
import pytest

import cases
import seqcorpus as SQ

pytestmark = pytest.mark.gpu

REF_CALL = 128
F_COMMA_SPACE = 1
IDS = [b"1", b'"req-42"', b"9007199254740993", b'"\\u00e9"', b"null", b'"a<b"']
SEEDS = SQ.SEEDS
_oracle_cache = {}
_ref_cache = {}


def _ids(order):
    return [IDS[u % len(IDS)] for u in order]


# ---- reference answers: unique items in short calls, against the oracle -------------------------------------------
def _oracle_answers(oracle, kind, flags=0):
    key = (kind, flags)
    if key not in _oracle_cache:
        if kind == "req":  # GGR_F_COMMA_SPACE spaces reply text only
            _oracle_cache[key] = [oracle.encode(it.message, it.data)[:2] for it in SQ.requests(oracle)]
        elif kind == "rep":
            _oracle_cache[key] = [oracle.decode(it.message, it.data, flags)[:2] for it in SQ.replies(oracle)]
        elif kind == "wrap":
            _oracle_cache[key] = [oracle.response(it.message, it.data, IDS[u % len(IDS)]) for u, it in enumerate(SQ.replies(oracle))]
        else:
            _oracle_cache[key] = [oracle.request(it.data) for it in SQ.bodies(oracle)]
    return _oracle_cache[key]


def _check_item(it, ost, oo, est, eo):
    """the rules of tests/test_gpu_parity.py and tests/test_gpu_limits.py for one item"""
    if it.gap is not None and ost == 0 and est == it.gap:
        assert eo == b""
        return
    if it.damaged:
        assert (ost == 0) == (est == 0), (it.message, it.data[:120], ost, est)
    else:
        assert est != SQ.ST_UNSUPPORTED or ost != 0, (it.message, it.data[:120], "unsupported")
        assert cases.status_compatible(ost, est) or (ost != 0 and est != 0 and {ost, est} <= {1, 3, 5}), \
            (it.message, it.data[:120], ost, est)
    assert eo == (oo if ost == 0 else b""), (it.message, it.data[:120], len(oo), len(eo))


def _chunks(n):
    return [(a, min(a + REF_CALL, n)) for a in range(0, n, REF_CALL)]


def _reference(path, engine, schema, oracle, kind, flags=0):
    """(status, bytes[, method, id span]) of every unique item on the engine of this path, from calls of at most REF_CALL
    items"""
    from ggrmcp_b200.engine import pack, unpack
    key = (path, kind, flags)
    if key in _ref_cache:
        return _ref_cache[key]
    items = {"req": SQ.requests, "rep": SQ.replies, "wrap": SQ.replies, "body": SQ.bodies}[kind](oracle)
    orc_ans = _oracle_answers(oracle, kind, flags)
    ref = []
    for a, b in _chunks(len(items)):
        part = items[a:b]
        data, off = pack([it.data for it in part])
        if kind == "body":
            out, ooff, method, span, st = engine.request_batch(schema, data, off)
            outs = unpack(out, ooff)
            for i, it in enumerate(part):
                s = int(st[i])
                r = orc_ans[a + i]
                assert s in (0, SQ.ST_UNSUPPORTED), (it.data[:120], s)
                if s == 0:
                    idt = it.data[int(span[i][0]):int(span[i][0]) + int(span[i][1])]
                    assert r["kind"] == 0 and outs[i] == r["wire"] and int(method[i]) == r["method"] and idt == r["id"], \
                        (it.data[:200], r["kind"], r["status"])
                    ref.append((0, outs[i], int(method[i]), int(span[i][0]), int(span[i][1])))
                else:
                    assert outs[i] == b""
                    ref.append((s, b"", None, None, None))
            continue
        ids = np.array([schema.message(it.message) for it in part], np.int32)
        if kind == "req":
            out, ooff, st = engine.encode_batch(schema, ids, data, off, flags)
        elif kind == "rep":
            out, ooff, st = engine.decode_batch(schema, ids, data, off, flags)
        else:
            idb, ioff = pack(_ids(range(a, b)))
            out, ooff, st = engine.decode_wrap_batch(schema, ids, data, off, idb, ioff, flags)
        outs = unpack(out, ooff)
        for i, it in enumerate(part):
            s = int(st[i])
            if kind == "wrap":
                ost, body = orc_ans[a + i]
                if not (it.gap is not None and ost == 0 and s == it.gap):
                    assert (ost == 0) == (s == 0), (it.message, it.data[:80].hex(), ost, s)
                    assert outs[i] == (body if ost == 0 else b""), (it.message, it.data[:80].hex())
            else:
                _check_item(it, *orc_ans[a + i], s, outs[i])
            ref.append((s, outs[i]))
    _ref_cache[key] = ref
    return ref


# ---- long batches on the device -------------------------------------------------------------------------------------
class Batch:
    """one shuffled plan of a direction in device memory: input 16-byte aligned and readable 64 bytes past its end"""

    def __init__(self, torch, schema, items, seed, with_ids=False):
        self.order = SQ.plan(items, seed)
        self.n = len(self.order)
        blob = b"".join(items[u].data for u in self.order)
        off = np.zeros(self.n + 1, np.uint64)
        off[1:] = np.cumsum([len(items[u].data) for u in self.order], dtype=np.uint64)
        self.in_bytes = len(blob)
        dev = torch.device("cuda", 0)
        self.d_in = self._to_dev(torch, np.frombuffer(blob, np.uint8), dev, 64)
        self.d_off = self._to_dev(torch, off, dev)
        if items[0].message is not None:
            msg = np.array([schema.message(items[u].message) for u in self.order], np.int32)
            self.d_msg = self._to_dev(torch, msg, dev)
        if with_ids:
            idt = _ids(self.order)
            ioff = np.zeros(self.n + 1, np.uint64)
            ioff[1:] = np.cumsum([len(t) for t in idt], dtype=np.uint64)
            self.ids_bytes = int(ioff[-1])
            self.d_ids = self._to_dev(torch, np.frombuffer(b"".join(idt), np.uint8), dev, 64)
            self.d_ids_off = self._to_dev(torch, ioff, dev)

    @staticmethod
    def _to_dev(torch, a, dev, pad=0):
        t = torch.zeros(a.nbytes + pad, dtype=torch.uint8, device=dev)
        t[: a.nbytes] = torch.from_numpy(a.view(np.uint8).reshape(-1).copy())
        return t


class Outputs:
    def __init__(self, torch, n, cap, body=False):
        dev = torch.device("cuda", 0)
        self.cap = int(cap)
        self.d_out = torch.empty(self.cap, dtype=torch.uint8, device=dev)
        self.d_off = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
        self.d_st = torch.full((n,), -99, dtype=torch.int32, device=dev)
        if body:
            self.d_method = torch.full((n,), -2, dtype=torch.int32, device=dev)
            self.d_span = torch.zeros(2 * n, dtype=torch.int32, device=dev)


def _launch(engine, schema, kind, B, O, flags, stream):
    from ggrmcp_b200 import engine as E
    L = E._load()
    if kind == "req":
        engine.encode_batch_dev(schema, B.n, B.d_msg.data_ptr(), B.d_in.data_ptr(), B.d_off.data_ptr(), B.in_bytes, O.d_out.data_ptr(),
                                O.cap, O.d_off.data_ptr(), O.d_st.data_ptr(), flags, stream)
    elif kind == "rep":
        engine.decode_batch_dev(schema, B.n, B.d_msg.data_ptr(), B.d_in.data_ptr(), B.d_off.data_ptr(), B.in_bytes, O.d_out.data_ptr(),
                                O.cap, O.d_off.data_ptr(), O.d_st.data_ptr(), flags, stream)
    elif kind == "body":
        rc = L.ggr_request_batch_dev(engine.h, schema.h, B.n, B.d_in.data_ptr(), B.d_off.data_ptr(), B.in_bytes, O.d_out.data_ptr(), O.cap,
                                     O.d_off.data_ptr(), O.d_method.data_ptr(), O.d_span.data_ptr(), O.d_st.data_ptr(), stream)
        assert rc == 0, (rc, L.ggr_last_error(engine.h))
    else:
        rc = L.ggr_decode_wrap_batch_dev(engine.h, schema.h, B.n, B.d_msg.data_ptr(), B.d_in.data_ptr(), B.d_off.data_ptr(), B.in_bytes,
                                         B.d_ids.data_ptr(), B.d_ids_off.data_ptr(), O.d_out.data_ptr(), O.cap, O.d_off.data_ptr(),
                                         O.d_st.data_ptr(), flags, stream)
        assert rc == 0, (rc, L.ggr_last_error(engine.h))


def _compare(label, items, order, ref, st, out, out_off, method=None, span=None):
    """the whole packed buffer against the concatenated reference answers; item by item only to name a mismatch"""
    want_st = np.array([ref[u][0] for u in order], np.int32)
    sizes = np.array([len(ref[u][1]) for u in order], np.uint64)
    want_off = np.zeros(len(order) + 1, np.uint64)
    want_off[1:] = np.cumsum(sizes, dtype=np.uint64)
    bad = np.nonzero(st != want_st)[0]
    assert not len(bad), [(label, int(p), order[p], items[order[p]].message, items[order[p]].data[:80], int(st[p]), int(want_st[p]),
                           "after", order[p - 1] if p else None) for p in bad[:5]]
    assert (out_off == want_off).all(), (label, int(np.nonzero(out_off != want_off)[0][0]))
    if out.tobytes() != b"".join(ref[u][1] for u in order):
        for p, u in enumerate(order):
            got = out[int(want_off[p]):int(want_off[p + 1])].tobytes()
            assert got == ref[u][1], (label, p, u, items[u].message, items[u].data[:80], got[:120], ref[u][1][:120],
                                      "after", order[p - 1] if p else None)
    if method is not None:
        ok = want_st == 0
        want_m = np.array([ref[u][2] if ref[u][0] == 0 else 0 for u in order], np.int64)
        want_s = np.array([(ref[u][3], ref[u][4]) if ref[u][0] == 0 else (0, 0) for u in order], np.int64)
        mism = np.nonzero(ok & ((method != want_m) | (span[:, 0] != want_s[:, 0]) | (span[:, 1] != want_s[:, 1])))[0]
        assert not len(mism), [(label, int(p), order[p], int(method[p]), list(span[p]), ref[order[p]][2:]) for p in mism[:5]]


def _lists(path, kind, items, order, ref):
    """items of the router's first lock-step list in one call (GGR_LOCKSTEP_MIN_BYTES and the switches of this path) and
    how many of them the reference answers accept.  The engine does not report which kernel took an item, so the later
    tiers' lists (what the tier before leaves) are not counted here; tests/test_sequences.py counts them on the host
    simulation"""
    from conftest import _ENGINE_PATHS
    env = _ENGINE_PATHS[path]
    if kind in ("req", "body"):
        if env.get("GGR_COOP_ENC") == "0":
            return 0, 0
        lo = int(env.get("GGR_LOCKSTEP_MIN_BYTES", 1024)) if kind == "req" else 0
        hi = 65000 - 16
    else:
        if env.get("GGR_COOP") == "0":
            return 0, 0
        lo, hi = int(env.get("GGR_LOCKSTEP_MIN_BYTES", 640)), 0x3FFFFF00
    on = [u for u in order if lo <= len(items[u].data) <= hi]
    return len(on), sum(1 for u in on if ref[u][0] == 0)


def _run_pair(engine, schema, oracle, request, kind, flags=0):
    import torch
    path = request.node.callspec.params["engine"]
    items = {"req": SQ.requests, "rep": SQ.replies, "wrap": SQ.replies, "body": SQ.bodies}[kind](oracle)
    t0 = time.perf_counter()
    ref = _reference(path, engine, schema, oracle, kind, flags)
    t1 = time.perf_counter()
    batches = [Batch(torch, schema, items, seed, with_ids=kind == "wrap") for seed in SEEDS]
    caps = []
    for B in batches:
        need = sum(len(ref[u][1]) for u in B.order)
        extra = B.in_bytes * 4 + 160 * B.n + (B.ids_bytes if kind == "wrap" else 0)  # room for intermediate texts
        caps.append(need + extra + 4096)
    outs = [Outputs(torch, B.n, cap, body=kind == "body") for B, cap in zip(batches, caps)]
    caller = torch.cuda.Stream()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    # the engine's own stream, then a caller stream: the second call starts on the scratch area the first one left
    _launch(engine, schema, kind, batches[0], outs[0], flags, None)
    engine.synchronize()
    _launch(engine, schema, kind, batches[1], outs[1], flags, caller.cuda_stream)
    caller.synchronize()
    t3 = time.perf_counter()
    for seed, B, O in zip(SEEDS, batches, outs):
        st = O.d_st.cpu().numpy()
        out_off = O.d_off.cpu().numpy().astype(np.uint64)
        out = O.d_out[: int(out_off[-1])].cpu().numpy()
        method = span = None
        if kind == "body":
            method = O.d_method.cpu().numpy().astype(np.int64)
            span = O.d_span.cpu().numpy().astype(np.int64).reshape(-1, 2)
        _compare("%s flags %d order %d" % (kind, flags, seed), items, B.order, ref, st, out, out_off, method, span)
        n_list, n_ok = _lists(path, kind, items, B.order, ref)
        print("%s %s flags %d order %d: %d items (%d unique, %.1f MB); first lock-step list %d items, %d accepted"
              % (path, kind, flags, seed, B.n, len(items), B.in_bytes / 1e6, n_list, n_ok))
    print("%s %s flags %d: reference %.2f s, two calls %.3f s, check %.2f s"
          % (path, kind, flags, t1 - t0, t3 - t2, time.perf_counter() - t3))


@pytest.mark.parametrize("flags", [0, F_COMMA_SPACE])
def test_encode_dev_sequences(engine, schema, oracle, request, flags):
    _run_pair(engine, schema, oracle, request, "req", flags)


@pytest.mark.parametrize("flags", [0, F_COMMA_SPACE])
def test_decode_dev_sequences(engine, schema, oracle, request, flags):
    _run_pair(engine, schema, oracle, request, "rep", flags)


def test_request_dev_sequences(engine, schema, oracle, request):
    _run_pair(engine, schema, oracle, request, "body")


def test_decode_wrap_dev_sequences(engine, schema, oracle, request):
    _run_pair(engine, schema, oracle, request, "wrap")


def test_host_one_chunk(oracle, fds_bytes):
    """ggr_encode_batch / ggr_decode_batch over the same long batches in one chunk and one slot, lock-step kernels first:
    the host pipeline around one long launch per kernel"""
    import ggrmcp_b200
    from ggrmcp_b200.engine import pack, unpack
    env = {"GGR_CHUNK_ITEMS": str(1 << 18), "GGR_CHUNK_BYTES": str(SQ.MAX_BYTES + (32 << 20)), "GGR_SLOTS": "1", "GGR_LOCKSTEP_MIN_BYTES": "0"}
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        eng = ggrmcp_b200.Engine(0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    sch = eng.register(fds_bytes)
    try:
        for kind, fn in (("req", eng.encode_batch), ("rep", eng.decode_batch)):
            items = SQ.requests(oracle) if kind == "req" else SQ.replies(oracle)
            ref = _reference("one_chunk", eng, sch, oracle, kind)
            order = SQ.plan(items, SEEDS[0])
            ids = np.array([sch.message(items[u].message) for u in order], np.int32)
            data, off = pack([items[u].data for u in order])
            out, ooff, st = fn(sch, ids, data, off)
            _compare("host %s" % kind, items, order, ref, np.asarray(st, np.int32), np.asarray(out), np.asarray(ooff, np.uint64))
    finally:
        sch.release()
        eng.close()
