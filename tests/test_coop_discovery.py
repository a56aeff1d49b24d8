"""Discovery pass of the lock-step reply kernel (coop_size_item, ggr_coop.cuh) on 32 fibers.

Every item of the corpus below goes through the host simulation of both lock-step tiers.  Two checks per item:
  - an item a tier takes is written exactly as the oracle writes it, with status OK;
  - which tier takes it (first, second, or none: left to the per-thread kernels) is what it was when the fixture
    tests/golden/coop_decisions.bin was recorded.
Which items the lock-step tiers take is the OR of every rule the discovery pass checks over the item (declaration
order, repeated runs, oneofs, maps, well-known types, depth, malformed headers, table capacity): a rewrite of the pass
has to keep it exactly.  The fixture was recorded from the host simulation with
`python tests/test_coop_discovery.py --record`.  It starts with the SHA-256 of the corpus, so a change to the corpus
generator shows up as such and not as changed decisions.  Record it again only from a discovery pass whose decisions
are known to be right.
"""
import hashlib
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases  # noqa: E402
import pbgen  # noqa: E402
import wiremut  # noqa: E402
from cases import wire_field as F  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "coop_decisions.bin")
NODE = cases.P + "Node"
UP = cases.P + "GetUserProfileResponse"
A = cases.A
TAKE1, TAKE2, LEAVE = 0, 1, 2


def node(id_=None, value=None, children=()):
    w = b""
    if id_ is not None:
        w += F(1, 2, id_)
    if value is not None:
        w += F(2, 2, value)
    for c in children:
        w += F(3, 2, c)
    return w


def chain(depth):
    """a Node chain whose deepest message is at depth `depth` (the root is at 0)"""
    w = node(b"leaf")
    for _ in range(depth):
        w = node(b"n", None, [w])
    return w


def unk(rng):
    num = rng.choice([19, 200, 1000, 99999, 536870911])
    return rng.choice([F(num, 0, rng.getrandbits(40)), F(num, 1, bytes(8)), F(num, 2, b"xyz"), F(num, 5, b"\x01\x02\x03\x04")])


def targeted():
    """(message, wire) on both sides of each rule the discovery pass decides by"""
    rng = random.Random(41)
    out = []
    add = lambda name, w: out.append((name, w))  # noqa: E731
    # fields out of declaration order; a singular set twice
    add(NODE, node(b"a", b"b"))
    add(NODE, F(2, 2, b"b") + F(1, 2, b"a"))
    add(NODE, F(3, 2, node(b"c")) + F(1, 2, b"a"))
    add(NODE, F(1, 2, b"a") + F(1, 2, b"b"))
    add(A, F(1, 0, 5) + F(18, 0, 7))            # late_low (number 18) is declared last
    add(A, F(18, 0, 7) + F(1, 0, 5))
    add(A, F(100, 2, b"z") + F(18, 0, 7))
    add(A, F(18, 0, 7) + F(100, 2, b"z"))
    # repeated runs closed by another field, by an elided zero, and reopened
    for tail in (b"", F(100, 2, b""), F(18, 0, 0), F(18, 0, 3), F(100, 2, b"") + F(37, 2, F(1, 0, 1)),
                 F(18, 0, 0) + F(37, 2, b""), F(37, 2, F(1, 0, 2)), unk(rng) + F(37, 2, b"")):
        add(A, F(37, 2, F(1, 0, 1)) + F(37, 2, F(2, 2, b"q")) + tail)
    add(A, F(38, 0, 1) + F(38, 0, 0) + F(18, 0, 0) + F(38, 0, 4))
    add(A, F(38, 0, 1) + F(100, 2, b"") + F(38, 0, 4))
    add(A, F(38, 0, 1) + F(38, 2, cases._vi(2) + cases._vi(3)) + F(38, 0, 4))
    add(NODE, node(b"", b"", [node(b"x")]) + F(1, 2, b""))
    # empty packed runs: at the start, in the middle of a run, after a run, out of order, alone
    add(A, F(21, 2, b"") + F(21, 2, b"\x01\x02") + F(22, 2, b"\x03"))
    add(A, F(21, 2, b"\x01") + F(21, 2, b"") + F(21, 2, b"\x02"))
    add(A, F(21, 2, b"\x01") + F(22, 2, b"") + F(23, 2, b"\x05"))
    add(A, F(22, 2, b"\x01") + F(21, 2, b""))
    add(A, F(22, 2, b"") + F(21, 2, b""))
    add(A, F(21, 2, b""))
    add(A, F(21, 2, b"") + F(21, 2, b""))
    add(A, F(1, 0, 3) + F(21, 2, b"") + F(2, 0, 4))
    add(A, F(2, 0, 3) + F(21, 2, b""))
    add(A, F(38, 0, 1) + F(38, 2, b"") + F(38, 0, 2))
    add(A, F(38, 2, b"") + F(37, 2, b""))
    # oneof members twice, a zero member (explicit presence: written), proto3 optional
    add(A, F(51, 0, 1) + F(52, 2, b"s"))
    add(A, F(51, 0, 0) + F(54, 0, 0))
    add(A, F(51, 0, 0))
    add(A, F(53, 2, b"") + F(55, 0, 2))
    add(A, F(52, 2, b"") + F(61, 0, 0) + F(62, 2, b"") + F(63, 0, 0))
    add(A, F(61, 0, 0) + F(61, 0, 1))
    # unknown fields and wrong wire types among known ones
    for _ in range(12):
        fs = [F(1, 0, rng.randrange(3)), F(14, 2, b"s"), F(16, 0, 2), F(17, 2, F(1, 0, 9)), F(21, 2, b"\x01"), F(37, 2, b""),
              F(100, 2, b"z")]
        bad = [unk(rng), F(1, 2, b"ab"), F(14, 0, 3), F(17, 0, 1), F(21, 5, b"\x00\x00\x00\x01"), F(37, 1, bytes(8))]
        for _ in range(rng.randint(1, 4)):
            fs.insert(rng.randrange(len(fs) + 1), rng.choice(bad))
        add(A, b"".join(fs))
    # 32-bit kinds: varints with bits above the low word
    for num in (1, 3, 5, 16, 2, 4, 6):   # int32 uint32 sint32 enum | int64 uint64 sint64
        for v in (1 << 32, (1 << 35) | 1, 1 << 63, (1 << 64) - (1 << 32), 0xFFFFFFFF):
            add(A, F(num, 0, v))
    add(A, F(1, 0, 1 << 32) + F(1, 0, 1))
    # 223 / 224 / 225 kept entries (the root is one): first tier's table; 4095 / 4096 / 4097: second tier's
    for n in (221, 222, 223, 224, 4094, 4095, 4096):
        add(A, b"".join(F(38, 0, i + 1) for i in range(n)))
    for n in (222, 223, 224):
        add(A, b"".join(F(38, 0, i + 1) + (unk(rng) if i % 7 == 0 else b"") + (F(38, 2, b"") if i % 11 == 0 else b"")
                        for i in range(n)))
        add(A, F(1, 0, 0) + F(2, 0, 0) + b"".join(F(38, 0, i + 1) for i in range(n)) + F(18, 0, 0) + F(100, 2, b""))
        add(NODE, node(b"r", None, [node(b"%d" % i) for i in range((n - 2) // 2)]))
    # depth: the deepest message at 22, 23, 24
    for d in (21, 22, 23, 24):
        add(NODE, chain(d))
    # 1, 31, 32, 33, 100 field occurrences in one message, and levels of 1 and 40+ messages
    for k in (1, 31, 32, 33, 100):
        add(A, b"".join(F(28, 2, b"s%d" % i) for i in range(k)))
        add(NODE, node(b"r", b"v", [node(b"c") for _ in range(k - 2)]) if k > 2 else node(b"r"))
        add(A, b"".join(F(n, 0, 1) for n in list(range(1, 5))[: min(k, 4)]) + b"".join(F(38, 0, i) for i in range(k)))
    add(NODE, node(b"r", None, [node(b"a", b"b", [node(b"c", b"d") for _ in range(3)]) for _ in range(45)]))
    add(NODE, node(b"r", None, [node(None, None, [node(b"x") for _ in range(40)])]))
    add(UP, F(1, 2, F(1, 2, b"u") + F(4, 0, 2) + F(5, 2, F(1, 0, 1700000000) + F(2, 0, 5))))
    add(UP, F(1, 2, F(1, 2, b"u") + F(5, 2, b"") + F(4, 0, 0)))
    add(UP, F(1, 2, F(4, 0, 1) + F(1, 2, b"u")))
    return out


def deep_mutate(w, rng, depth=0):
    try:
        fields = wiremut.split_fields(w)
    except Exception:
        return rng.choice((wiremut.truncate, wiremut.corrupt))(w, rng) if w else w
    subs = [k for k, (num, wt, raw) in enumerate(fields) if wt == 2 and len(raw) > 3]
    if subs and depth < 3 and rng.random() < 0.7:
        k = rng.choice(subs)
        num, wt, raw = fields[k]
        _, i = wiremut.read_varint(raw, 0)
        ln, j = wiremut.read_varint(raw, i)
        newp = deep_mutate(raw[j:j + ln], rng, depth + 1)
        fields[k] = (num, wt, raw[:i] + wiremut.put_varint(len(newp)) + newp)
        out = b"".join(r for _, _, r in fields)
        return rng.choice((wiremut.shuffle, wiremut.duplicate_some, wiremut.inject_unknown))(out, rng) if rng.random() < 0.4 else out
    muts = (wiremut.shuffle, wiremut.duplicate_some, wiremut.inject_unknown, wiremut.truncate, wiremut.corrupt)
    return rng.choice(muts[:3] if rng.random() < 0.8 else muts)(w, rng)


def mutated(n_per_msg=80, seed0=91000):
    names = [A, cases.P + "CreateDocumentRequest", NODE, UP, cases.P + "ProcessNodeResponse"]
    out = []
    for name in names:
        for seed in range(seed0, seed0 + n_per_msg):
            rng = random.Random(seed)
            w = pbgen.wire(pbgen.random_message(name, seed))
            out.append((name, w))
            for _ in range(9):
                out.append((name, deep_mutate(w, rng)))
    return out


def bench_shapes(msg_index, names):
    import benchgen

    def mi(name):
        names[msg_index(name)] = name
        return msg_index(name)

    out = []
    for kind, n in (("nested", 40), ("mixed", 400)):
        wl = getattr(benchgen, kind)(n, mi)
        blob = wl.rep_wire.tobytes()
        for i in range(wl.n):
            w = blob[int(wl.rep_off[i]):int(wl.rep_off[i + 1])]
            if len(w) <= 40000:
                out.append((names[int(wl.rep_msg[i])], w))
    return out


def corpus(hsim):
    names = {}
    return targeted() + mutated() + bench_shapes(hsim.msg, names)


def corpus_digest(items):
    h = hashlib.sha256()
    for name, w in items:
        h.update(name.encode() + b"\0" + len(w).to_bytes(4, "little") + w)
    return h.digest()


def decide(hsim, name, w, i):
    """(decision, text of the taking tier or None)"""
    os.environ["HS_COOP_TIER1_ONLY"] = "1"
    try:
        rc1, out1 = hsim.decode_coop(name, w, i & 1, i % 16, (i * 5) % 16)
    finally:
        del os.environ["HS_COOP_TIER1_ONLY"]
    assert rc1 in (0, 200), (name, w.hex()[:200], rc1)
    if rc1 == 0:
        return TAKE1, out1
    rc2, out2 = hsim.decode_coop(name, w, i & 1, i % 16, (i * 5) % 16)
    assert rc2 in (0, 200), (name, w.hex()[:200], rc2)
    return (TAKE2, out2) if rc2 == 0 else (LEAVE, None)


def test_discovery_decisions_and_text(oracle, hsim):
    items = corpus(hsim)
    with open(FIXTURE, "rb") as fh:
        rec = fh.read()
    assert rec[:32] == corpus_digest(items), "the corpus is not the one the fixture was recorded for"
    want = rec[32:]
    assert len(want) == len(items)
    counts = [0, 0, 0]
    for i, (name, w) in enumerate(items):
        d, out = decide(hsim, name, w, i)
        counts[d] += 1
        assert d == want[i], (i, name, w.hex()[:300], "decision", d, "recorded", want[i])
        if d != LEAVE:
            rc, oj, _ = oracle.decode(name, w, i & 1)
            assert rc == 0 and out == oj, (i, name, w.hex()[:300], rc, oj[:200], out[:200])
    # every outcome is represented, the first tier's most of all
    assert counts[TAKE1] > 2000 and counts[TAKE2] >= 5 and counts[LEAVE] > 1000, counts


@pytest.mark.parametrize("d", [21, 22, 23, 24])
def test_depth_limit(hsim, d):
    """the deepest message a lock-step tier scans is at depth 22 (GGR_COOP_DEPTH - 2)"""
    rc, _ = hsim.decode_coop(NODE, chain(d))
    assert (rc == 0) == (d <= 22), (d, rc)


@pytest.mark.parametrize("n,tier1", [(222, True), (223, True), (224, False)])
def test_first_tier_capacity_ignores_skipped_fields(hsim, n, tier1):
    """unknown fields, empty packed runs and elided zeros take no slot of the first tier's 224"""
    rng = random.Random(n)
    w = F(1, 0, 0) + b"".join(
        F(38, 0, i + 1) + (unk(rng) if i % 5 == 0 else b"") + (F(38, 2, b"") if i % 3 == 0 else b"") for i in range(n)) + F(18, 0, 0)
    os.environ["HS_COOP_TIER1_ONLY"] = "1"
    try:
        rc, _ = hsim.decode_coop(A, w)
    finally:
        del os.environ["HS_COOP_TIER1_ONLY"]
    assert (rc == 0) == tier1, (n, rc)


if __name__ == "__main__" and "--record" in sys.argv:
    import hostsim
    with open(os.path.join(ROOT, "tests", "golden", "schemas.binpb"), "rb") as fh:
        hs = hostsim.Schema(fh.read())
    items = corpus(hs)
    dec = bytes(decide(hs, name, w, i)[0] for i, (name, w) in enumerate(items))
    with open(FIXTURE, "wb") as fh:
        fh.write(corpus_digest(items) + dec)
    print("%d items: %d first tier, %d second tier, %d left" % (len(items), dec.count(0), dec.count(1), dec.count(2)))
