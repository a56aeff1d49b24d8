"""Persistent warps on the host simulation: the unique items of tests/seqcorpus.py in sequence through each lock-step entry
point, with the per-warp structures kept from one item to the next (hostsim.keep_state), in two shuffled orders.  Every
item must give exactly the return code and bytes it gives on a fresh warp, the answer the other host-simulation tests
compare with the oracle.  The device run of the same corpus is tests/test_gpu_sequences.py."""
import random

import pytest

import limits as LM
import seqcorpus as SQ

ORDERS = (101, 202)
MIN_UNIQUE = 5000
# the fiber warps of the host simulation are slow: a seeded sample of the unique items up to CPU_MAX_BYTES (all of the
# kinds the corpus holds), plus every larger item that a later tier takes (the walker's, the reply side's, the lock-step
# parser's large tables)
CPU_ITEMS = 5200
CPU_MAX_BYTES = 4096
WALK_STOPS = ("HS_WALK_TIER1_ONLY", "HS_WALK_TIER2_ONLY")
COOP_STOP = "HS_COOP_TIER1_ONLY"
COOP_MAX_BYTES = 70000  # the lock-step parser's largest items, as tests/test_limits.py runs them
IDS = [b"1", b'"req-42"', b"9007199254740993", b'"\\u00e9"', b"null"]


def _in_off(k):
    return (k * 7 + 3) % 16


def _out_off(k):
    return (k * 5) % 16


def _sample(items):
    sel = [it for it in items if len(it.data) <= CPU_MAX_BYTES]
    return random.Random(len(sel)).sample(sel, min(CPU_ITEMS, len(sel)))


def _check_sequences(run, n, label):
    """run(k) -> answer of unique item k; fresh warps first, then each order with the state kept"""
    import hostsim
    assert n >= MIN_UNIQUE, (label, n)
    hostsim.keep_state(False)
    fresh = [run(k) for k in range(n)]
    try:
        for seed in ORDERS:
            order = list(range(n))
            random.Random(seed).shuffle(order)
            hostsim.keep_state(True)
            for p, k in enumerate(order):
                got = run(k)
                if got != fresh[k]:
                    prev = order[p - 1] if p else None
                    pytest.fail("%s, order %d, position %d: item %d gives %r, on a fresh warp %r; the item before it was %r"
                                % (label, seed, p, k, _short(got), _short(fresh[k]), prev))
            hostsim.keep_state(False)
    finally:
        hostsim.keep_state(False)
    return fresh


def _short(ans):
    return tuple(x[:64] if isinstance(x, bytes) else x for x in ans)


def _tiers(monkeypatch, run, fresh, stops):
    """tier that takes each item on a fresh warp (0: none): stops[i] is the switch that ends the chain of tiers after tier
    i + 1, so an item taken with it set is taken by tier i + 1 or an earlier one"""
    out = []
    for k, ans in enumerate(fresh):
        t = 0
        if ans[0] == 0:
            t = len(stops) + 1
            for i, sw in enumerate(stops):
                monkeypatch.setenv(sw, "1")
                rc = run(k)[0]
                monkeypatch.delenv(sw)
                if rc == 0:
                    t = i + 1
                    break
        out.append(t)
    return out


def _with_later_tiers(monkeypatch, sample, items, run_item, stops, max_bytes):
    """the sample plus every larger item of the corpus (up to max_bytes) that a tier after the first takes: those tiers
    exist for large items, and a stale table entry past the first tier's capacity can only come from one"""
    large = [it for it in items if CPU_MAX_BYTES < len(it.data) <= max_bytes]
    run = lambda k: run_item(large[k], k)
    tiers = _tiers(monkeypatch, run, [run(k) for k in range(len(large))], stops)
    return sample + [it for it, t in zip(large, tiers) if t >= 2]


def _check_tiers(monkeypatch, run, fresh, stops, label):
    """every tier of the chain takes items of the sequence"""
    tiers = _tiers(monkeypatch, run, fresh, stops)
    counts = [tiers.count(t) for t in range(1, len(stops) + 2)]
    assert all(counts), (label, counts)
    return counts


@pytest.mark.parametrize("entry", ["coop0", "coop1", "walk"])
def test_request_sequences(oracle, hsim, monkeypatch, entry):
    """the lock-step parser's two tiers (k_encode_coop_tok / k_encode_coop_parse, then k_encode_coop_emit) and the walker
    (k_encode_tok3, k_encode_place, the three k_encode_type tiers, then the emitter)"""
    for k in WALK_STOPS:
        monkeypatch.delenv(k, raising=False)
    corpus = SQ.requests(oracle)
    items = _sample(corpus)
    if entry == "walk":
        walk = lambda it, k: hsim.encode_walk(it.message, it.data, _in_off(k), _out_off(k))
        items = _with_later_tiers(monkeypatch, items, corpus, walk, WALK_STOPS, LM.CE_MAX_INPUT)
        run = lambda k: walk(items[k], k)
    else:
        tier = int(entry[-1])
        coop = lambda it, k, t: hsim.encode_coop(it.message, it.data, _in_off(k), _out_off(k), t)
        if tier:  # the large tables: items past the small ones' capacities
            items += [it for k, it in enumerate(corpus) if CPU_MAX_BYTES < len(it.data) <= COOP_MAX_BYTES
                      and coop(it, k, 1)[0] == 0 and coop(it, k, 0)[0] != 0]
        run = lambda k: coop(items[k], k, tier)
    fresh = _check_sequences(run, len(items), entry)
    assert all(rc in (0, 200) for rc, _ in fresh)
    taken = sum(1 for rc, _ in fresh if rc == 0)
    assert taken
    counts = _check_tiers(monkeypatch, run, fresh, WALK_STOPS, entry) if entry == "walk" else [taken]
    print("%s: %d items, taken per tier %s" % (entry, len(items), counts))


@pytest.mark.parametrize("flags", [0, 1])
def test_reply_sequences(oracle, hsim, monkeypatch, flags):
    """both lock-step reply tiers (k_decode_coop_size, then k_decode_coop_write)"""
    monkeypatch.delenv(COOP_STOP, raising=False)
    corpus = SQ.replies(oracle)
    dec = lambda it, k: hsim.decode_coop(it.message, it.data, flags, _in_off(k), _out_off(k))
    items = _with_later_tiers(monkeypatch, _sample(corpus), corpus, dec, [COOP_STOP], SQ.MID)
    run = lambda k: dec(items[k], k)
    fresh = _check_sequences(run, len(items), "reply flags %d" % flags)
    assert all(rc in (0, 200) for rc, _ in fresh)
    counts = _check_tiers(monkeypatch, run, fresh, [COOP_STOP], "reply flags %d" % flags)
    print("reply flags %d: %d items, taken per tier %s" % (flags, len(items), counts))


@pytest.mark.parametrize("tier", [0, 1])
def test_envelope_sequences(oracle, hsim, tier):
    """request bodies through the lock-step parser in envelope mode"""
    items = _sample(SQ.bodies(oracle))
    fresh = _check_sequences(lambda k: hsim.request_coop(items[k].data, _in_off(k), _out_off(k), tier), len(items),
                             "envelope tier %d" % tier)
    assert all(a[0] in (0, 200) for a in fresh)
    print("envelope tier %d: %d bodies, %d taken" % (tier, len(items), sum(1 for a in fresh if a[0] == 0)))


def test_wrap_sequences(oracle, hsim):
    """result wrapping (k_wrap_size, k_wrap_write) around the texts of the replies the oracle accepts.  The wrapper keeps
    no per-warp state, so this shows only that its answers do not depend on the order of the items"""
    import hostsim
    texts = []
    for it in SQ.replies(oracle):
        st, text, _ = oracle.decode(it.message, it.data)
        if st == 0 and len(text) <= CPU_MAX_BYTES:
            texts.append(text)
    texts = random.Random(len(texts)).sample(texts, min(CPU_ITEMS, len(texts)))
    fresh = _check_sequences(lambda k: hostsim.wrap(texts[k], IDS[k % len(IDS)]), len(texts), "wrap")
    assert all(rc == 0 for rc, _ in fresh)


def test_plan_offsets(oracle):
    """the replication plans the device runs: at least MIN_ITEMS copies in at most MAX_BYTES, and every replicated item at
    MIN_RESIDUES start offsets mod 16 or more"""
    for items in (SQ.requests(oracle), SQ.replies(oracle), SQ.bodies(oracle)):
        for seed in SQ.SEEDS:
            order = SQ.plan(items, seed)
            assert len(order) >= SQ.MIN_ITEMS and sum(len(items[u].data) for u in order) <= SQ.MAX_BYTES
            res = SQ.residues(items, order)
            assert set(res) == set(range(len(items)))
            short = [(u, dict(r)) for u, r in res.items() if sum(r.values()) > 1 and len(r) < SQ.MIN_RESIDUES]
            assert not short, (len(short), short[:5])
