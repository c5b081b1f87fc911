"""swirld_sign.cuh on the H100: the device harness against the host harness and libsodium, and sw_set_signing_key /
sw_new_events / sw_batch_new_events through the engine."""
import hashlib
import os
import pickle
import random
import tempfile

import numpy as np
import pytest

import sign_harness as SH
from host_sim import Event
from test_sign_host import L, arr, base_enc, le, signing_case, all_eights

nacl = pytest.importorskip("nacl.bindings")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    d = tmp_path_factory.mktemp("sign_dev")
    return SH.SignHarness(SH.compile_lib(d, True), True)


def test_device_arith(dev):
    rng = random.Random(11)
    tab = dev.table()
    for k in range(32):
        for j in range(8):
            assert bytes(tab[k, j]) == base_enc((j + 1) * 256 ** k)
    xs = [0, 1, L - 1] + all_eights() + [rng.randrange(L) for _ in range(300)]
    a = arr([le(x) for x in xs], 32)
    want = [base_enc(x) for x in xs]
    assert [bytes(r) for r in dev.base_mult(a)] == want
    ys = [0, L - 1, L, 2 * L - 1, 5 * L, 2 ** 512 - 1] + [rng.randrange(2 ** 512) for _ in range(300)]
    got = dev.reduce(arr([le(y, 64) for y in ys], 64))
    assert [int.from_bytes(bytes(g), "little") for g in got] == [y % L for y in ys]
    ks, As, rs = ([rng.randrange(L) for _ in range(200)], [rng.randrange(2 ** 254, 2 ** 255) & ~7 for _ in range(200)],
                  [rng.randrange(L) for _ in range(200)])
    got = dev.muladd(arr([le(x) for x in ks], 32), arr([le(x) for x in As], 32), arr([le(x) for x in rs], 32))
    assert [int.from_bytes(bytes(g), "little") for g in got] == [(r + k * x) % L for k, x, r in zip(ks, As, rs)]


def test_device_sign(dev):
    seeds, msgs, who = signing_case()
    sk = dev.signing_key(arr(seeds, 32))
    kp = [nacl.crypto_sign_seed_keypair(s) for s in seeds]
    assert [bytes(r[64:]) for r in sk] == [pk for pk, _ in kp]
    pres = [b"(" + m + bytes(64) + b")" for m in msgs]
    at = [1 + len(m) for m in msgs]
    for lanes in (1, 8):
        sig, ids = dev.sign_events(lanes, sk[who], msgs, pres, at)
        for i, m in enumerate(msgs):
            pk, s = kp[who[i]]
            want = nacl.crypto_sign(m, s)[:64]
            assert bytes(sig[i]) == want, (lanes, i, len(m))
            assert bytes(ids[i]) == hashlib.blake2b(b"(" + m + want + b")", digest_size=32).digest()


# ---------------------------------------------------------------- the engine
def engine_mod():
    from swirld_b200 import engine
    return engine


def keys(M, seed):
    rng = random.Random(seed)
    return [nacl.crypto_sign_seed_keypair(bytes(rng.randrange(256) for _ in range(32))) for _ in range(M)]


def view(M, kp, member, cap=4096):
    E = engine_mod()
    e = E.Engine(M, cap)
    e.set_member_keys([pk for pk, _ in kp])
    e.set_signing_key(member, kp[member][1])
    return e


def templates(kp, member, n, parents=None, t0=1.0):
    from swirld_b200.events import event_template
    out = []
    for i in range(n):
        p = parents[i] if parents else ()
        out.append(event_template(Event, b"payload %d" % i, p, t0 + i, kp[member][0]))
    return out


def check_events(tmpl, kp, member, sig, ids):
    for (msg, pre, at), s, h in zip(tmpl, sig, ids):
        want = nacl.crypto_sign(msg, kp[member][1])[:64]
        assert bytes(s) == want
        nacl.crypto_sign_open(want + msg, kp[member][0])
        full = pre[:at] + want + pre[at + 64:]
        assert full == pickle.dumps(Event(*pickle.loads(msg), want))
        assert bytes(h) == hashlib.blake2b(full, digest_size=32).digest()


def test_new_events_match_libsodium():
    kp = keys(8, 1)
    e = view(8, kp, 3)
    tm = templates(kp, 3, 40)
    sig, ids = e.new_events(tm, ingest=False)
    check_events(tm, kp, 3, sig, ids)
    flags = e.verify_events(np.full(40, 3, np.int32), sig, [m for m, _, _ in tm],
                            [p[:a] + bytes(s) + p[a + 64:] for (_, p, a), s in zip(tm, sig)], ids)
    assert (flags == 3).all()
    assert e.n_events == 0


@pytest.mark.parametrize("M", [4, 64, 1024])
def test_batch_equals_single(M):
    E = engine_mod()
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    kp = keys(M, 2)
    for B in sorted({1, 2, 17, n_sm + 3}):
        members = [(3 * v) % M for v in range(B)]
        A = [view(M, kp, m, 64) for m in members]
        S = [view(M, kp, m, 64) for m in members]
        tm = [templates(kp, m, 1, t0=10.0 + v) for v, m in enumerate(members)]
        zero = [np.zeros((1, 32), np.uint8)] * B
        before = A[0].stats()["kernel_launches"]
        got = E.batch_new_events(A, tm, ingest=False)
        assert A[0].stats()["kernel_launches"] - before == 1
        got_i = E.batch_new_events(A, tm, zero, zero, [[10.0 + v] for v in range(B)])
        for v in range(B):
            s1, i1, x1, m1 = S[v].new_events(tm[v], zero[v], zero[v], [10.0 + v])
            assert bytes(got[v][0]) == bytes(s1) and bytes(got[v][1]) == bytes(i1)
            s2, i2, x2, m2 = got_i[v]
            assert bytes(s2) == bytes(s1) and bytes(i2) == bytes(i1) and list(x2) == list(x1) and m2 == m1 == 1
            assert S[v].n_events == A[v].n_events == 1
            assert bytes(S[v].ids()) == bytes(A[v].ids())
            check_events(tm[v], kp, members[v], s1, i1)


def test_refusals_write_nothing():
    E = engine_mod()
    kp = keys(4, 3)
    e = view(4, kp, 0)
    bare = E.Engine(4, 64)
    bare.set_member_keys([pk for pk, _ in kp])
    tm = templates(kp, 0, 2)
    with pytest.raises(E.EngineError):
        bare.new_events(tm, ingest=False)
    L_ = e._lib
    msg, moff, pre, poff, at = E._templates(tm)
    sig, ids = np.zeros((2, 64), np.uint8), np.zeros((2, 32), np.uint8)
    for bad in ("moff", "at_neg", "at_high"):
        mo, a = moff.copy(), at.copy()
        if bad == "moff":
            mo[1] = mo[2] + 1
        elif bad == "at_neg":
            a[0] = -1
        else:
            a[1] = poff[2] - poff[1] - 63
        rc = L_.sw_new_events(e._h, 2, None, None, None, E._ptr(msg), E._ptr(mo), E._ptr(pre), E._ptr(poff), E._ptr(a),
                              E._ptr(sig), E._ptr(ids), None)
        assert rc == -1 and not sig.any() and not ids.any()
    with pytest.raises(E.EngineError):
        E.batch_new_events([e, bare], [tm[:1], tm[1:]], ingest=False)
    assert e.n_events == 0 and bare.n_events == 0


def test_key_lifecycle():
    E = engine_mod()
    kp = keys(4, 4)
    e = view(4, kp, 1)
    with pytest.raises(E.EngineError):
        e.set_signing_key(0, kp[1][1])                         # pk is member 1's, not member 0's
    other_seed = nacl.crypto_sign_seed_keypair(b"\x07" * 32)[1][:32]
    with pytest.raises(E.EngineError):
        e.set_signing_key(1, other_seed + kp[1][0])            # the right pk, another seed: the device refuses it
    tm = templates(kp, 1, 3)
    check_events(tm, kp, 1, *e.new_events(tm, ingest=False))   # the refused calls kept the key
    e.reset()
    check_events(tm, kp, 1, *e.new_events(tm, ingest=False))
    e.set_signing_key(2, kp[2][1])
    tm2 = templates(kp, 2, 3)
    check_events(tm2, kp, 2, *e.new_events(tm2, ingest=False))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ck.bin")
        e.save(path)
        with open(path, "rb") as f:
            blob = f.read()
        assert hashlib.sha512(kp[2][1][:32]).digest()[32:] not in blob
        f2 = E.Engine.load(path)
        f2.set_member_keys([pk for pk, _ in kp])
        with pytest.raises(E.EngineError):
            f2.new_events(tm2, ingest=False)


def test_own_events_entered():
    E = engine_mod()
    kp = keys(2, 5)
    a, b = view(2, kp, 0), view(2, kp, 1)
    z = np.zeros((1, 32), np.uint8)
    ta = templates(kp, 0, 1)
    _, ida, xa, ma = a.new_events(ta, z, z, [1.0])
    assert ma == 1 and list(xa) == [0] and list(a.lookup(ida)) == [0]
    tb = templates(kp, 1, 1)
    sb, idb, _, _ = b.new_events(tb, z, z, [1.0])
    # a learns b's root, then makes an event on (its head, b's root)
    a.ingest(idb, z, z, [1], [1.0], sb)
    from swirld_b200.events import event_template
    t2 = [event_template(Event, b"x", (bytes(ida[0]), bytes(idb[0])), 2.0, kp[0][0])]
    _, id2, x2, m2 = a.new_events(t2, ida, idb, [2.0])
    assert m2 == 1 and list(x2) == [2] and list(a.lookup(id2)) == [2]
    # a second event on the same self-parent is a fork: not entered
    t3 = [event_template(Event, b"y", (bytes(ida[0]), bytes(idb[0])), 3.0, kp[0][0])]
    _, id3, x3, m3 = a.new_events(t3, ida, idb, [3.0])
    assert m3 == 0 and list(x3) == [-1] and list(a.lookup(id3)) == [-1]
    a.divide_rounds(0, a.n_events)
    idx, cols = a.sync_reply(2, np.array([-1, -1], np.int32))
    assert list(idx) == [0, 1, 2]
    assert bytes(cols[0][0]) == bytes(ida[0]) and bytes(cols[0][2]) == bytes(id2[0])


def test_gossip_batched_turns():
    """16 views of a signed gossip through whole batched turns, one with batch_new_events, a twin whose new events come
    from libsodium through batch_ingest; both end with the same ids, heights and consensus results."""
    E = engine_mod()
    from swirld_b200.events import event_template
    M, B, turns = 16, 16, 40
    kp = keys(M, 6)
    runs = []
    for mode in ("gpu", "host"):
        V = [view(M, kp, v, 4096) for v in range(B)]
        rng = random.Random(9)
        zero = np.zeros(32, np.uint8)
        # every view's root
        roots = [[event_template(Event, b"", (), 0.5 + v, kp[v][0])] for v in range(B)]
        def make(tms, p0s, p1s, ts):
            if mode == "gpu":
                res = E.batch_new_events(V, tms, p0s, p1s, ts)
                return [r[1] for r in res]
            out = []
            batches = []
            for v in range(B):
                sig = np.array([list(nacl.crypto_sign(m, kp[v][1])[:64]) for m, _, _ in tms[v]], np.uint8).reshape(-1, 64)
                ids = np.array([list(hashlib.blake2b(p[:a] + bytes(s) + p[a + 64:], digest_size=32).digest())
                                for (m, p, a), s in zip(tms[v], sig)], np.uint8).reshape(-1, 32)
                pres = [p[:a] + bytes(s) + p[a + 64:] for (m, p, a), s in zip(tms[v], sig)]
                batches.append((ids, p0s[v], p1s[v], [v] * len(tms[v]), ts[v], sig, [m for m, _, _ in tms[v]], pres))
                out.append(ids)
            E.batch_ingest(V, batches)
            return out
        ids = make(roots, [zero[None]] * B, [zero[None]] * B, [[0.5 + v] for v in range(B)])
        heads = [bytes(i[0]) for i in ids]
        E.batch_divide_rounds(V, [0] * B, [1] * B)
        divided = [1] * B
        for turn in range(turns):
            peers = [(v + 1 + rng.randrange(B - 1)) % B for v in range(B)]
            summ = E.batch_sync_summary(V, [V[v].n_events - 1 for v in range(B)])
            # view v asks peer p: p answers from its head with v's summary
            P = [V[p] for p in peers]
            if len({id(x) for x in P}) < B:      # a batch takes each engine once: answer one by one
                replies = [V[p].sync_reply(V[p].n_events - 1, summ[v]) for v, p in enumerate(peers)]
            else:
                idx, cols = E.batch_sync_reply(P, [x.n_events - 1 for x in P], summ)
                replies = list(zip(idx, cols))
            for v, (ix, c) in enumerate(replies):
                V[v].ingest(*c)
            tms, p0s, p1s, ts = [], [], [], []
            for v in range(B):
                their = bytes(replies[v][1][0][-1])
                t = 1.0 + turn + v / 100
                tms.append([event_template(Event, b"t%d" % turn, (heads[v], their), t, kp[v][0])])
                p0s.append(np.frombuffer(heads[v], np.uint8)[None])
                p1s.append(np.frombuffer(their, np.uint8)[None])
                ts.append([t])
            new = make(tms, p0s, p1s, ts)
            heads = [bytes(i[0]) for i in new]
            n = [x.n_events for x in V]
            E.batch_divide_rounds(V, divided, [a - b for a, b in zip(n, divided)])
            divided = n
            ncs = E.batch_decide_fame(V)
            E.batch_find_order_out(V, ncs)
        runs.append([(bytes(x.ids()), x.heights().tolist(), x.rounds().tolist(), x.consensus().tolist(),
                      x.transactions().tolist()) for x in V])
    assert runs[0] == runs[1]
    assert any(len(r[4]) for r in runs[0])
