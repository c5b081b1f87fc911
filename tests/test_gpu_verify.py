"""sw_verify_events, sw_set_member_keys and sw_ingest_verified on the GPU: every verdict equals libsodium's (PyNaCl) and
every id check equals hashlib's BLAKE2b, exactly; a verified ingest equals a plain ingest of the burst without the
events that fail; and a gossip run whose peers corrupt part of their replies checks each reply in one call."""
import pickle
import random

import numpy as np
import pytest

import host_sim
import node_sim
import sodium
import verify_cases as vc
from swirld_b200 import engine as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases():
    return vc.build()


def _expected(cs):
    return np.array([int(c.ok_sig) | (int(c.ok_id) << 1) for c in cs], np.uint8)


def _filler(rng, k):
    return [vc.nb.crypto_sign_seed_keypair(rng.randbytes(32))[0] for _ in range(k)]


def _verify_all(M, cs, rng):
    """Every case through engines of M members: the distinct keys go in groups of at most M; every member holds one
    key of its group (a key sits on several members when the group is smaller than M) and each event names one of
    them at random.  Returns (flags, expected) in case order."""
    e = E.Engine(M, 16)
    keys = list(dict.fromkeys(c.pk for c in cs))
    got = np.full(len(cs), 255, np.uint8)
    for g in range(0, len(keys), M):
        group = keys[g:g + M]
        members = {k: [] for k in group}
        table = []
        for m in range(M):
            k = group[m % len(group)]
            members[k].append(m)
            table.append(k)
        e.set_member_keys(table)
        sel = [i for i, c in enumerate(cs) if c.pk in members]
        rng.shuffle(sel)
        cr = [rng.choice(members[cs[i].pk]) for i in sel]
        f = e.verify_events(cr, np.frombuffer(b"".join(cs[i].sig for i in sel), np.uint8), [cs[i].msg for i in sel],
                            [cs[i].pre for i in sel], np.frombuffer(b"".join(cs[i].id for i in sel), np.uint8))
        got[sel] = f
    e.close()
    return got, _expected(cs)


@pytest.mark.parametrize("M", [1, 2, 64, 65, 1024])
def test_every_family_every_member_count(cases, M):
    got, want = _verify_all(M, cases, random.Random(M))
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(int(i), cases[i].family, int(got[i]), int(want[i])) for i in bad[:20]]


def _pool(rng, n_keys, n):
    """n distinct signed event-shaped messages under n_keys members, 1 in 8 tampered in one of four ways."""
    keys = [vc.nb.crypto_sign_seed_keypair(rng.randbytes(32)) for _ in range(n_keys)]
    out = []
    for j in range(n):
        c = j % n_keys
        pk, sk = keys[c]
        msg, sig, pre, id_ = vc.event_shapes(rng, pk, sk, 1)[0]
        kind = rng.randrange(8)
        if kind == 1:
            sig = vc.flip(sig, rng.randrange(512))
        elif kind == 2:
            msg = vc.flip(msg, rng.randrange(8 * len(msg)))
        elif kind == 3:
            pre = vc.flip(pre, rng.randrange(8 * len(pre)))
        elif kind == 4:
            id_ = vc.flip(id_, rng.randrange(256))
        out.append((c, sig, msg, pre, id_, int(vc.nacl_ok(sig, msg, pk)) | (int(vc.blake(pre) == id_) << 1)))
    return [k[0] for k in keys], out


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 1 << 17])
def test_batch_sizes(n):
    rng = random.Random(n)
    pks, pool = _pool(rng, 64, 4096)
    e = E.Engine(64, 16)
    e.set_member_keys(pks)
    pos = [rng.randrange(len(pool)) for _ in range(n)]
    sel = [pool[p] for p in pos]
    f = e.verify_events([s[0] for s in sel], np.frombuffer(b"".join(s[1] for s in sel), np.uint8),
                        [s[2] for s in sel], [s[3] for s in sel], np.frombuffer(b"".join(s[4] for s in sel), np.uint8))
    assert f.shape == (n,)
    assert np.array_equal(f, np.array([s[5] for s in sel], np.uint8))
    st = e.stats()
    assert st["kernel_launches"] == 2 + (2 if n else 0)        # the two table builds, then the call's two kernels
    assert st["d2h_bytes"] == n


def _raw_verify(e, n, creator, off_m, off_p):
    """sw_verify_events straight through ctypes with flags_out pre-filled, so a refusal can be seen to leave it."""
    sig = np.zeros(64 * max(n, 1), np.uint8)
    ids = np.zeros(32 * max(n, 1), np.uint8)
    buf = np.zeros(max(1, int(max(off_m[-1], off_p[-1]))), np.uint8)
    out = np.full(max(n, 1), 0xAB, np.uint8)
    cr = np.ascontiguousarray(creator, np.int32)
    om, op = np.ascontiguousarray(off_m, np.int64), np.ascontiguousarray(off_p, np.int64)
    rc = e._lib.sw_verify_events(e._h, n, E._ptr(cr), E._ptr(sig), E._ptr(buf), E._ptr(om), E._ptr(buf), E._ptr(op),
                                 E._ptr(ids), E._ptr(out))
    return rc, out


def test_key_handling(cases, tmp_path):
    rng = random.Random(7)
    good = [c for c in cases if c.family == "valid"][:40]
    pk_a = good[0].pk
    sel = [c for c in good if c.pk == pk_a]
    other = _filler(rng, 1)[0]
    e = E.Engine(2, 64)

    def run():
        return e.verify_events([0] * len(sel), np.frombuffer(b"".join(c.sig for c in sel), np.uint8),
                               [c.msg for c in sel], [c.pre for c in sel], np.frombuffer(b"".join(c.id for c in sel), np.uint8))

    # no keys: SW_E_ARG, flags unwritten
    rc, out = _raw_verify(e, 1, [0], [0, 0], [0, 0])
    assert rc == -1 and out[0] == 0xAB
    with pytest.raises(E.EngineError):
        run()
    e.set_member_keys([pk_a, other])
    assert (run() == 3).all()
    e.set_member_keys([other, pk_a])                 # replaced: member 0 is now someone else
    assert (run() == 2).all()
    e.set_member_keys(np.frombuffer(pk_a + other, np.uint8).reshape(2, 32))
    assert (run() == 3).all()
    for what in (e.reset, e.rewind):                 # the keys survive both
        what()
        assert (run() == 3).all()
    # refusals before anything runs, flags_out unwritten
    for creator, om, op in (([2], [0, 0], [0, 0]), ([-1], [0, 0], [0, 0]), ([0, 0], [0, 5, 3], [0, 0, 0]),
                            ([0], [1, 2], [0, 0]), ([0, 0], [0, 0, 0], [0, 4, 2])):
        rc, out = _raw_verify(e, len(creator), creator, om, op)
        assert rc == -1 and (out == 0xAB).all(), (creator, om, op)
    rc, _ = _raw_verify(e, 0, [], [0], [0])
    assert rc == 0
    # a checkpoint does not hold the keys
    p = str(tmp_path / "ck.bin")
    e.save(p)
    e2 = E.Engine.load(p)
    rc, out = _raw_verify(e2, 1, [0], [0, 0], [0, 0])
    assert rc == -1 and out[0] == 0xAB
    e2.set_member_keys([pk_a, other])
    assert (e2.verify_events([0], np.frombuffer(sel[0].sig, np.uint8), [sel[0].msg], [sel[0].pre],
                             np.frombuffer(sel[0].id, np.uint8)) == 3).all()


# ---------------------------------------------------------------- sw_ingest_verified
def _gossip(M, n_events, seed):
    """A fork-free graph of real events (the reference's shapes, swirld.py:88-95) in creation order, cut into bursts
    of consecutive events: a list of bursts, each a list of (id, Event, msg, preimage, member)."""
    rng = random.Random(seed)
    keys = [vc.nb.crypto_sign_seed_keypair(rng.randbytes(32)) for _ in range(M)]
    heads, evs = [None] * M, []
    t = 1.7e9

    def make(c, p):
        nonlocal t
        t += rng.random()
        d = None if rng.random() < 0.7 else [rng.randbytes(8)]
        pk, sk = keys[c]
        msg = pickle.dumps((d, p, t, pk))
        ev = vc.Event(d, p, t, pk, vc.sign(sk, msg))
        pre = pickle.dumps(ev)
        h = vc.blake(pre)
        heads[c] = h
        evs.append((h, ev, msg, pre, c))

    for c in range(M):
        make(c, ())
    while len(evs) < n_events:
        c = rng.randrange(M)
        o = rng.choice([x for x in range(M) if x != c])
        make(c, (heads[c], heads[o]))
    bursts, i = [], 0
    while i < len(evs):
        k = rng.randrange(20, 80)
        bursts.append(evs[i:i + k])
        i += k
    return [k[0] for k in keys], bursts


def _cols(items):
    zero = bytes(32)
    ids = np.frombuffer(b"".join(h for h, *_ in items), np.uint8)
    p0 = np.frombuffer(b"".join(ev.p[0] if ev.p else zero for _, ev, *_ in items), np.uint8)
    p1 = np.frombuffer(b"".join(ev.p[1] if ev.p else zero for _, ev, *_ in items), np.uint8)
    cr = np.array([c for *_, c in items], np.int32)
    t = np.array([ev.t for _, ev, *_ in items], np.float64)
    sig = np.frombuffer(b"".join(ev.s for _, ev, *_ in items), np.uint8)
    return ids, p0, p1, cr, t, sig


@pytest.mark.parametrize("M,wide", [(8, False), (8, True), (72, False)])
def test_ingest_verified_equals_ingest_without_the_failures(M, wide, monkeypatch):
    """Bursts of a gossip graph, shuffled, some events tampered with (signature, signed bytes or preimage).  Whatever
    a burst rejects comes again, intact, in the next one, as a peer would send it again."""
    if wide:
        monkeypatch.setenv("SW_FORCE_WIDE", "1")
    rng = random.Random(M * 3 + wide)
    pks, bursts = _gossip(M, 1500 if M <= 8 else 8000, seed=M + wide)
    a, b = E.Engine(M, 8192), E.Engine(M, 8192)
    a.set_member_keys(pks)
    known, known_ids, pending = [], set(), []
    n_bad = n_below = 0
    for burst in bursts + [[]]:
        items = pending + list(burst)
        inb = {h for h, *_ in items}
        bad = set()
        # tamper with events none of whose parents are in the burst: the burst's parents-first order of everything
        # else is then the same with or without them
        for j, (h, ev, msg, pre, c) in enumerate(items):
            if burst and (not ev.p or not (set(ev.p) & inb)) and rng.random() < 0.4:
                kind = rng.randrange(3)
                if kind == 0:
                    ev = ev._replace(s=vc.flip(ev.s, rng.randrange(512)))
                elif kind == 1:
                    msg = vc.flip(msg, rng.randrange(8 * len(msg)))
                else:
                    pre = vc.flip(pre, rng.randrange(8 * len(pre)))
                items[j] = (h, ev, msg, pre, c)
                bad.add(h)
        below = set(bad)                               # what hangs below a failure in this burst
        for h, ev, *_ in sorted(items, key=lambda x: x[1].t):
            if ev.p and set(ev.p) & below:
                below.add(h)
        # a known event sent again with a corrupted signature keeps its index
        resend = []
        if known:
            h, ev, msg, pre, c = rng.choice(known)
            resend = [(h, ev._replace(s=vc.flip(ev.s, 3)), msg, pre, c)]
        items += resend
        rng.shuffle(items)
        ia, ma = a.ingest(*_cols(items), msgs=[x[2] for x in items], preimages=[x[3] for x in items])
        keep = [x for x in items if x[0] not in bad]
        ib, mb = b.ingest(*_cols(keep)) if keep else (np.zeros(0, np.int32), 0)
        assert ma == mb
        got_a = {x[0]: int(i) for x, i in zip(items, ia)}
        assert {x[0]: int(i) for x, i in zip(keep, ib)} == {h: i for h, i in got_a.items() if h not in bad}
        assert all(got_a[h] == -1 for h in below)
        originals = {x[0]: x for x in burst}
        originals.update({x[0]: x for x in pending})
        pending = [originals[h] for h, i in got_a.items() if i < 0]
        for h, i in got_a.items():
            if i >= 0 and h not in known_ids:
                known_ids.add(h)
                known.append(originals[h])
        for r in resend:
            assert got_a[r[0]] >= 0
        n_bad += len(bad)
        n_below += len(below - bad)
    assert n_bad > 10 and n_below > 0
    assert not pending and a.n_events == b.n_events == sum(len(x) for x in bursts)
    assert np.array_equal(a.heights(), b.heights())
    assert np.array_equal(a.lookup(np.frombuffer(b"".join(x[0] for x in known), np.uint8)),
                          b.lookup(np.frombuffer(b"".join(x[0] for x in known), np.uint8)))
    n = a.n_events
    for x in (a, b):
        x.divide_rounds(0, n)
        x.find_order(x.decide_fame())
    assert np.array_equal(a.can_see(), b.can_see())
    ra, rb = a.results(), b.results()
    for k in ("round", "witness", "famous", "consensus", "transactions"):
        assert np.array_equal(ra[k], rb[k]), k
    assert a.max_round >= 3 and a.n_transactions > 0


# ---------------------------------------------------------------- a gossip run with faulty peers
class VerifyingHost(host_sim.HostNode):
    """The tests' gossip host, whose peers corrupt a seeded share of what they send; each reply is checked in one
    verify_events call, and every item's GPU verdict must equal the inherited libsodium check."""
    fault_rng = random.Random(11)
    checked = [0, 0]                                   # items checked, items that failed

    def _keys(self):
        if getattr(self, "_keyed", None) is not self._eng:
            self._eng.set_member_keys(self._m2pk)
            self._keyed = self._eng

    def sync(self, peer, payload):
        self._keys()
        request = sodium.crypto_sign(pickle.dumps(dict(self._heads)), self.sk)
        their_head, items = pickle.loads(sodium.crypto_sign_open(self.network[peer](self.pk, request), peer))
        rng = self.fault_rng
        out = []
        for h, ev in items:                            # a faulty peer, after the reply was opened
            if rng.random() < 0.1:
                kind = rng.randrange(3)
                if kind == 0:
                    ev = ev._replace(s=vc.flip(ev.s, rng.randrange(512)))
                elif kind == 1:
                    ev = ev._replace(t=ev.t + 1e-3)
                else:
                    h = vc.flip(h, rng.randrange(256))
            out.append((h, ev))
        if out:
            flags = self._eng.verify_events([self._pk2m[ev.c] for _, ev in out],
                                            np.frombuffer(b"".join(ev.s for _, ev in out), np.uint8),
                                            [pickle.dumps(tuple(ev[:4])) for _, ev in out],
                                            [pickle.dumps(ev) for _, ev in out],
                                            np.frombuffer(b"".join(h for h, _ in out), np.uint8))
            for (h, ev), f in zip(out, flags):
                try:
                    sodium.crypto_sign_verify_detached(ev.s, pickle.dumps(tuple(ev[:4])), ev.c)
                    sig_ok = True
                except ValueError:
                    sig_ok = False
                id_ok = host_sim._event_id(ev) == h
                assert int(f) == int(sig_ok) | (int(id_ok) << 1), (f, sig_ok, id_ok)
                self.checked[0] += 1
                self.checked[1] += f != 3
        fresh = []
        for h, ev in out:
            if h not in self.hg and self.is_valid_event(h, ev):
                self.add_event(h, ev)
                fresh.append(h)
        if their_head in self.hg:
            h, ev = self.new_event(payload, (self.head, their_head))
            self.add_event(h, ev)
            self.head = h
            fresh.append(h)
        return tuple(fresh)


def test_gossip_with_faulty_peers():
    random.seed(23)                                    # (the hosts pick their peers with the module's generator)
    VerifyingHost.fault_rng, VerifyingHost.checked = random.Random(11), [0, 0]
    nodes = node_sim.run_sim(4, 300, host_cls=VerifyingHost, capacity=1 << 12, seed=23)
    assert VerifyingHost.checked[0] > 500 and VerifyingHost.checked[1] > 20
    for nd in nodes:
        assert len(nd.transactions) > 10
    for x in nodes:
        for y in nodes:
            k = min(len(x.transactions), len(y.transactions))
            assert x.transactions[:k] == y.transactions[:k]
