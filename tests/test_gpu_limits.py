"""The boundary corpus of tests/limits.py on the device, through ggr_encode_batch / ggr_decode_batch on every engine path,
against the oracle: bit-exact where the oracle accepts, a compatible status where it refuses, never GGR_ST_UNSUPPORTED where
it answers.  Also the two capacities only the device has: the 2 KB tiles in which the request tokenizer stages its text
(W9) and the second reply tier's entry pool (R9)."""
import random
import time

import numpy as np
import pytest

import cases
import limits as LM

pytestmark = pytest.mark.gpu

_cache = {}


def _corpus(oracle):
    if not _cache:
        _cache["rep"], _cache["req"] = LM.corpus(oracle)
    return _cache["rep"], _cache["req"]


def _allowed_gap(it, ost, est):
    """documented gaps (DESIGN.md section 6): nesting past the per-thread kernels' frames, request items above 2 MiB - 16"""
    if ost != 0:
        return False
    if est == 8:
        return LM.past_frames(it)
    return est == 9 and it.limit_id == "W10" and len(it.data) > LM.TOO_LARGE


def _run(engine, schema, encode, items, flags=0):
    from ggrmcp_b200.engine import pack, unpack
    ids = np.array([schema.message(it.message) for it in items], np.int32)
    data, off = pack([it.data for it in items])
    fn = engine.encode_batch if encode else engine.decode_batch
    out, ooff, st = fn(schema, ids, data, off, flags)
    return unpack(out, ooff), [int(s) for s in st]


def _check(oracle, encode, items, eo, es, flags=0):
    gaps = 0
    for i, it in enumerate(items):
        ost, oo, _ = oracle.encode(it.message, it.data) if encode else oracle.decode(it.message, it.data, flags)
        if _allowed_gap(it, ost, es[i]):
            assert eo[i] == b""
            gaps += 1
            continue
        assert es[i] != 11 or ost != 0, (it[:3], len(it.data), "unsupported")
        assert cases.status_compatible(ost, es[i]) or (ost != 0 and es[i] != 0 and {ost, es[i]} <= {1, 3, 5}), \
            (it[:3], len(it.data), ost, es[i])
        if ost == 0:
            assert eo[i] == oo, (it[:3], len(it.data), flags, len(oo), len(eo[i]))
        else:
            assert eo[i] == b""
    return gaps


def _shuffled(items, seed):
    items = list(items)
    random.Random(seed).shuffle(items)
    return items


def test_reply_limits(engine, schema, oracle):
    rep, _ = _corpus(oracle)
    items = _shuffled(rep, 1)
    for flags in (0, 1):
        eo, es = _run(engine, schema, False, items, flags)
        _check(oracle, False, items, eo, es, flags)


def test_request_limits(engine, schema, oracle):
    _, req = _corpus(oracle)
    items = _shuffled(req, 2)
    eo, es = _run(engine, schema, True, items)
    gaps = _check(oracle, True, items, eo, es)
    # the item above 2 MiB - 16 bytes is refused whole; the one at the limit is not
    assert sum(1 for it, s in zip(items, es) if it.limit_id == "W10" and s == 9) == 1 and gaps >= 1


def test_tokenizer_tiles(engine, schema, oracle):
    """W9: quotes, backslash runs, multi-byte sequences and token starts at the 2 KB tile edges, items of 1 to 5 tiles
    shuffled together (persistent warps carry their barrier parities from item to item); each item is placed at the start
    offset it was built for, so its event sits exactly on its tile edge"""
    tiles = LM.tile_items()
    assert {(edge, ev) for _, edge, ev, _ in tiles if edge in LM.TILE_EDGES} == {(e, v) for e in LM.TILE_EDGES for v in LM.TILE_EVENTS}
    assert {len(js) // LM.CW_TILE for *_, js in tiles} >= {0, 1, 2, 4} and {s for s, *_ in tiles} == set(range(16))
    rng = random.Random(3)
    rng.shuffle(tiles)
    items, pos = [], 0
    for start, edge, ev, js in tiles:
        # a filler item in front places this one at its start offset
        fill = 2 + (start - (pos + 2)) % 16
        items.append(LM.Item("W9", "below", LM.A, b"{" + b" " * (fill - 2) + b"}", False))
        pos += fill
        assert pos % 16 == start and js[edge - start:edge - start + len(ev)] == ev
        items.append(LM.Item("W9", "at", LM.A, js, False))
        pos += len(js)
    eo, es = _run(engine, schema, True, items)
    _check(oracle, True, items, eo, es)
    assert sum(1 for s in es if s == 0) == len(items)


# host chunks each engine path forms (tests/conftest.py): items per chunk at most, and whether the lock-step reply kernels run
_CHUNK_ITEMS = {"small_chunks": 128, "ramped_chunks": 512}
_CHUNK_BYTES = {"ramped_chunks": 400000}
_NO_REPLY_POOL = ("per_thread", "lockstep_request_only")


def test_tabpool_overflow(engine, schema, oracle, request):
    """R9: more second-tier entries in one call than the pool holds.  Each reply is past the first tier and within the
    second; a chunk's pool holds in_bytes / 2 + 4096 entries, at most 4 M.  Where one chunk holds the whole batch the
    first replies to reach the pool are taken and the rest fall back to the per-thread kernels, with the same bytes; where
    the engine cuts the batch into small chunks every chunk's pool holds all of its items; two paths have no lock-step
    reply kernels at all.  The counts are worked out from those rules, for the chunks this path forms: the engine does not
    report which kernel wrote an item."""
    path = request.node.callspec.params["engine"]
    name, w, n_ent, n_items = LM.pool_batch()
    assert LM.COOP_ENTRIES < n_ent <= LM.COOP_BIG_ENTRIES and len(w) % 16 != 0
    per_chunk = min(n_items, _CHUNK_ITEMS.get(path, 8192), _CHUNK_BYTES.get(path, 32 << 20) // len(w))
    pool = min(per_chunk * len(w) // 2 + 4096, LM.POOL_MAX)
    taken = 0 if path in _NO_REPLY_POOL else min(per_chunk, pool // n_ent)
    past = 0 if path in _NO_REPLY_POOL else per_chunk - taken
    if per_chunk == n_items and path not in _NO_REPLY_POOL:
        assert taken > 0 and past > 0, (taken, past)  # both sides of the limit within one host chunk
    elif path not in _NO_REPLY_POOL:
        assert past == 0  # so is a shorter chunk at either end of a ramp
    items = [LM.Item("R9", "above", name, w, False)] * n_items
    ost, oj, _ = oracle.decode(name, w)
    assert ost == 0
    t0 = time.perf_counter()
    eo, es = _run(engine, schema, False, items)
    dt = time.perf_counter() - t0
    assert all(s == 0 for s in es)
    bad = [i for i, o in enumerate(eo) if o != oj]
    assert not bad, (len(bad), bad[:5])
    print("R9 %s: %d replies of %d entries (%d bytes each); chunks of at most %d: pool %d entries, %d taken, %d past it "
          "per chunk; decode_batch %.3f s" % (path, n_items, n_ent, len(w), per_chunk, pool, taken, past, dt))
