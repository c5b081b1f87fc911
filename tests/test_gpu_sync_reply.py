"""sw_sync_summary / sw_sync_reply and their batched forms: the sending end of Node.sync selected on the GPU.  Every
reply is compared with ask_sync's BFS restated in tests/sync_model.py, in arrival order, and its rows with the engine's
own columns and id map.  Views are node-views of generator traces, ingested under ids made from (creator, chain
position), which name an event the same way in every view of one fork-free gossip.  Covered: M = 4, 16, 33 and 64 on
both kernel families and M = 97 to 1024; roots, heads the requester has and every divided event of a short view; a
checkpoint round trip; a view built by append; the round trip into a requester's ingest; batches of 1 to n_sm + 3
views of mixed M beside a 262 144-event view, each equal to its single call; launches per call; SW_E_CAPACITY and
the refusals; a round-stream piece in flight and appends beyond the head; and 16 views of a signed gossip through
the whole batched turn."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

import sync_model as sm
from swirld_b200 import engine as E
from swirld_b200 import traces

pytestmark = pytest.mark.gpu


def chain_ids(tr):
    """(N, 32) ids of a view's events: BLAKE2b of (creator, position in its chain); zeros stand for no parent."""
    seq, cnt = np.zeros(tr.N, np.int64), {}
    for i, c in enumerate(tr.creator.tolist()):
        seq[i] = cnt.get(c, 0)
        cnt[c] = seq[i] + 1
    ids = np.frombuffer(b"".join(hashlib.blake2b(b"%d:%d" % (c, s), digest_size=32).digest()
                                 for c, s in zip(tr.creator.tolist(), seq.tolist())), np.uint8).reshape(-1, 32)
    return ids


def parent_ids(tr, ids):
    z = np.zeros((1, 32), np.uint8)
    pick = lambda p: np.where((p >= 0)[:, None], ids[np.maximum(p, 0)], z)
    return pick(tr.p0), pick(tr.p1)


def ingested(tr, cap=None, n=None, divide=True):
    """An engine that ingested the first n events of view tr (in its index order, so indices agree) and divided them."""
    n = tr.N if n is None else n
    ids = chain_ids(tr)
    p0, p1 = parent_ids(tr, ids)
    e = E.Engine(tr.M, cap or max(tr.N, 64))
    idx, m = e.ingest(ids[:n], p0[:n], p1[:n], tr.creator[:n], tr.t[:n], tr.sig[:n])
    assert m == n and np.array_equal(idx, np.arange(n))
    if divide and n:
        e.divide_rounds(0, n)
    return e, ids


def check_reply(e, tr, ids, view, head, S):
    idx, (rid, rp0, rp1, rc, rt, rs) = e.sync_reply(head, S)
    exp = sm.bfs_reply(view, head, S)
    assert np.array_equal(idx, exp), "head %d" % head
    p0, p1 = parent_ids(tr, ids)
    assert np.array_equal(rid, ids[idx]) and np.array_equal(rp0, p0[idx]) and np.array_equal(rp1, p1[idx])
    assert np.array_equal(rc, tr.creator[idx]) and np.array_equal(rt, tr.t[idx]) and np.array_equal(rs, tr.sig[idx])
    assert np.array_equal(e.lookup(rid), idx)
    assert np.array_equal(e.ids(0, e.n_events)[idx], rid)
    return idx


def requester_summaries(base, X, k, rng):
    """Summaries of k other members' views of base at random points, and the empty one."""
    out = [np.full(base.M, -1, np.int32)]
    for Y in rng.sample([y for y in range(base.M) if y != X], min(k, base.M - 1)):
        vt, _ = traces.node_view(base, Y)
        vy = sm.View(vt)
        out.append(sm.summary(vy, rng.randrange(vt.N)))
    return out


@pytest.mark.parametrize("M,wide", [(4, False), (4, True), (16, False), (16, True), (33, False), (33, True),
                                    (64, False), (64, True), (97, True), (129, True), (300, True), (1024, True)])
def test_single_reply_equals_bfs(M, wide, monkeypatch):
    if wide and M <= 64:
        monkeypatch.setenv("SW_FORCE_WIDE", "1")
    rng = random.Random(M)
    base = traces.gossip(M, max(600, 3 * M), seed=M)
    tr, _ = traces.node_view(base, 1)
    v = sm.View(tr)
    e, ids = ingested(tr)
    roots = [i for i in range(tr.N) if tr.p0[i] < 0]
    heads = roots[:4] + [rng.randrange(tr.N) for _ in range(6)] + [tr.N - 1]
    sums = requester_summaries(base, 1, 3, rng)
    for h in heads:
        assert np.array_equal(e.sync_summary(h), sm.summary(v, h))
        for S in sums + [sm.summary(v, h)]:                      # the last one: the requester has the head
            check_reply(e, tr, ids, v, h, S)


def test_every_divided_event_of_a_short_view():
    base = traces.gossip(8, 160, seed=5)
    tr, _ = traces.node_view(base, 2)
    v = sm.View(tr)
    e, ids = ingested(tr)
    S = requester_summaries(base, 2, 1, random.Random(5))[1]
    for h in range(tr.N):
        check_reply(e, tr, ids, v, h, S)
        check_reply(e, tr, ids, v, h, np.full(8, -1, np.int32))


def test_reply_after_load(tmp_path):
    base = traces.gossip(16, 900, seed=6)
    tr, _ = traces.node_view(base, 0)
    e, ids = ingested(tr)
    S = requester_summaries(base, 0, 1, random.Random(6))[1]
    before = [e.sync_reply(h, S) for h in (0, 300, tr.N - 1)]
    e.save(str(tmp_path / "ck"))
    f = E.Engine.load(str(tmp_path / "ck"))
    after = [f.sync_reply(h, S) for h in (0, 300, tr.N - 1)]
    for (a, ca), (b, cb) in zip(before, after):
        assert np.array_equal(a, b) and all(np.array_equal(x, y) for x, y in zip(ca, cb))
    assert np.array_equal(f.ids(), e.ids())


def test_appended_view_refuses_id_columns():
    tr = traces.gossip(8, 300, seed=7)
    e = E.Engine(8, 300)
    e.append_trace(tr)
    e.divide_rounds(0, tr.N)
    v = sm.View(tr)
    S = np.full(8, -1, np.int32)
    with pytest.raises(E.EngineError) as ex:
        e.sync_reply(250, S)
    assert ex.value.code == -1 and "no id" in str(ex.value)
    assert np.array_equal(e.sync_reply(250, S, rows=False), sm.bfs_reply(v, 250, S))
    assert not e.ids().any()


def test_round_trip_into_ingest():
    """v.ingest of u's reply to v's summary adds exactly the events the reference's sync adds (the reply's events v
    lacks), in the reply's order."""
    base = traces.gossip(16, 1200, seed=8)
    (tu, _), (tv, _) = traces.node_view(base, 3), traces.node_view(base, 9)
    u, uid = ingested(tu)
    nv = tv.N // 2
    v, vid = ingested(tv, cap=tv.N + tu.N, n=nv)
    for uh, vh in ((tu.N - 1, nv - 1), (tu.N // 3, nv // 2)):
        S = v.sync_summary(vh)
        idx, cols = u.sync_reply(uh, S)
        known = {bytes(x) for x in v.ids()}
        new = [i for i, x in zip(idx.tolist(), cols[0]) if bytes(x) not in known]
        assert np.array_equal(idx, sm.bfs_reply(sm.View(tu), uh, S))
        n0 = v.n_events
        got, m = v.ingest(*cols)
        assert m == len(new)
        added = [g for g, i in zip(got.tolist(), idx.tolist()) if i in new]
        assert added == list(range(n0, n0 + m))
        assert np.array_equal(v.ids(n0, m), uid[new])


def _views(spec, seed):
    """(engine, view trace, ids, model) per view: spec = [(M, members)]."""
    out = []
    for M, k in spec:
        base = traces.gossip(M, 600, seed=seed + M)
        for X in range(k):
            tr, _ = traces.node_view(base, X % M)
            e, ids = ingested(tr)
            out.append((e, tr, ids, sm.View(tr), base))
    return out


def _batch_case(views, rng):
    heads = [rng.randrange(tr.N) for _, tr, _, _, _ in views]
    sums = []
    for (e, tr, ids, v, base), h in zip(views, heads):
        r = rng.random()
        sums.append(np.full(tr.M, -1, np.int32) if r < 0.2 else sm.summary(v, h) if r < 0.3
                    else sm.summary(v, rng.randrange(h + 1)))
    return heads, sums


def _assert_batch_equals_single(views, heads, sums):
    engs = [x[0] for x in views]
    k0 = engs[0].stats()["kernel_launches"]
    index, cols = E.batch_sync_reply(engs, heads, sums)
    launches = engs[0].stats()["kernel_launches"] - k0
    bs = E.batch_sync_summary(engs, heads)
    for (e, tr, ids, v, _), h, S, bi, bc, s in zip(views, heads, sums, index, cols, bs):
        si, sc = e.sync_reply(h, S)
        assert np.array_equal(bi, si) and np.array_equal(bi, sm.bfs_reply(v, h, S))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(bc, sc))
        assert np.array_equal(s, e.sync_summary(h))
    return launches


def test_batch_equals_single_and_launches():
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = random.Random(9)
    views = _views([(4, 4), (16, 16), (33, 24), (64, 24), (16, n_sm + 3 - 68)], 9)
    counts = {}
    for B in (1, 16, 64, n_sm + 3):
        sel = views[:B] if B <= 64 else views
        heads, sums = _batch_case(sel, rng)
        counts[B] = _assert_batch_equals_single(sel, heads, sums)
    assert set(counts.values()) == {3}, counts


def test_large_view_beside_small_ones():
    base = traces.gossip_np(64, 1 << 18, seed=10)
    big, bids = ingested(base)
    vb = sm.View(base)
    small = _views([(16, 6)], 10)
    views = [(big, base, bids, vb, base)] + small
    rng = random.Random(10)
    heads, sums = _batch_case(views, rng)
    heads[0], sums[0] = base.N - 1, np.full(64, -1, np.int32)    # a fresh requester catches up: the whole view
    _assert_batch_equals_single(views, heads, sums)


def _raw_batch(engs, heads, sums, cap, sentinel=0x5a):
    B = len(engs)
    S = np.ascontiguousarray(np.concatenate(sums), np.int32)
    h = np.ascontiguousarray(heads, np.int32)
    offs, cnt = np.full(B + 1, -7, np.int32), np.full(B, -7, np.int32)
    n = max(cap, 1)
    outs = [np.full(n, -7, np.int32), np.full((n, 32), sentinel, np.uint8), np.full((n, 32), sentinel, np.uint8),
            np.full((n, 32), sentinel, np.uint8), np.full(n, -7, np.int32), np.full(n, -7.0), np.full((n, 64), sentinel, np.uint8)]
    rc = engs[0]._lib.sw_batch_sync_reply(E._handles(engs), B, E._ptr(h), E._ptr(S), cap, E._ptr(offs), E._ptr(cnt),
                                          *[E._ptr(a) for a in outs])
    return rc, offs, cnt, outs


def test_capacity_then_retry():
    views = _views([(16, 5)], 11)
    engs = [x[0] for x in views]
    heads = [x[1].N - 1 for x in views]
    sums = [np.full(16, -1, np.int32)] * 5
    exp = [len(sm.bfs_reply(x[3], h, s)) for x, h, s in zip(views, heads, sums)]
    rc, offs, cnt, outs = _raw_batch(engs, heads, sums, sum(exp) - 1)
    assert rc == -5 and cnt.tolist() == exp
    assert (offs == -7).all() and (outs[0] == -7).all() and (outs[1] == 0x5a).all() and (outs[6] == 0x5a).all()
    rc, offs, cnt, outs = _raw_batch(engs, heads, sums, sum(exp))
    assert rc == 0 and cnt.tolist() == exp and offs.tolist() == np.cumsum([0] + exp).tolist()
    e = engs[0]
    idx, cn = np.full(4, -7, np.int32), C.c_int32(-7)
    rc = e._lib.sw_sync_reply(e._h, heads[0], E._ptr(sums[0]), 3, E._ptr(idx), C.byref(cn), *[None] * 6)
    assert rc == -5 and cn.value == exp[0] and (idx == -7).all()


def test_refusals_write_nothing():
    views = _views([(16, 3)], 12)
    engs = [x[0] for x in views]
    heads = [x[1].N - 1 for x in views]
    sums = [np.full(16, -1, np.int32)] * 3

    def refused(engs, heads, sums, code=-1):
        rc, offs, cnt, outs = _raw_batch(engs, heads, sums, 4096)
        assert rc == code and (offs == -7).all() and (cnt == -7).all() and (outs[0] == -7).all()

    refused([engs[0], engs[1], engs[0]], heads, sums)                       # repeated engine
    refused(engs, [heads[0], engs[1].n_divided, heads[2]], sums)             # head not divided
    refused(engs, [heads[0], -1, heads[2]], sums)                            # head out of range
    bad = [s.copy() for s in sums]
    bad[2][5] = -2
    refused(engs, heads, bad)                                                # summary entry < -1
    rc = engs[0]._lib.sw_batch_sync_reply(E._handles(engs), 0, *[None] * 2, 0, *[None] * 9)
    assert rc == -1
    arr = (C.c_void_p * 2)(engs[0]._h, None)
    S = np.zeros(32, np.int32)
    rc = engs[0]._lib.sw_batch_sync_reply(C.cast(arr, C.c_void_p), 2, E._ptr(np.array(heads[:2], np.int32)), E._ptr(S),
                                          16, E._ptr(np.zeros(3, np.int32)), E._ptr(np.zeros(2, np.int32)), *[None] * 7)
    assert rc == -1
    out = np.full(16, -7, np.int32)
    assert engs[0]._lib.sw_sync_summary(engs[0]._h, engs[0].n_divided, E._ptr(out)) == -1 and (out == -7).all()


def test_rounds_ahead_and_pending_appends(monkeypatch):
    """A view whose round stream has a piece in flight (M <= 64, calls of 2048 events) answers, and its rounds stay
    those of a twin that never answered; appends beyond the head do not change the reply."""
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "1")
    tr = traces.gossip(32, 20000, seed=13)
    ids = chain_ids(tr)
    p0, p1 = parent_ids(tr, ids)
    a, b = E.Engine(32, tr.N), E.Engine(32, tr.N)
    for x in (a, b):
        x.ingest(ids, p0, p1, tr.creator, tr.t, tr.sig)
    v = sm.View(tr)
    S = sm.summary(v, 5000)
    for first in range(0, tr.N, 2048):
        n = min(2048, tr.N - first)
        for x in (a, b):
            x.divide_rounds(first, n)
        h = first + n - 1
        assert np.array_equal(a.sync_reply(h, S, rows=False), sm.bfs_reply(v, h, S))
        assert np.array_equal(a.sync_summary(h), sm.summary(v, h))
    assert np.array_equal(a.rounds(), b.rounds()) and np.array_equal(a.witness_flags(), b.witness_flags())
    # appends beyond the head: the second half arrives after the first is divided
    c, cid = ingested(tr, n=tr.N // 2)
    c.ingest(ids[tr.N // 2:], p0[tr.N // 2:], p1[tr.N // 2:], tr.creator[tr.N // 2:], tr.t[tr.N // 2:], tr.sig[tr.N // 2:])
    h = tr.N // 2 - 1
    check_reply(c, tr, cid, v, h, S)


def test_signed_gossip_full_batched_turn():
    """16 views of a signed gossip; each turn every view asks another view (a derangement, so the responders are
    distinct) and the whole turn runs batched: summaries, replies, verified ingest, divide, fame, order.  A twin set
    is fed the replies built in Python from the same views' host graphs.  Both end with the same events, id maps and
    consensus results, and sampled views equal the oracle's replay of their events."""
    import test_gpu_verify as tv
    M, B = 8, 16
    pks, bursts = tv._gossip(M, 700, seed=14)
    evs = {x[0]: x for b in bursts for x in b}
    order = [x for b in bursts for x in b]
    rng = random.Random(14)
    sets = []
    for _ in range(2):
        engs = [E.Engine(M, 2048) for _ in range(B)]
        for e in engs:
            e.set_member_keys(pks)
        sets.append(engs)
    # view v starts with the first 40 (v + 1) events of the gossip (closed under parents): what the others lack
    # reaches them only through the turns' replies
    for v in range(B):
        seed_items = order[:40 * (v + 1)]
        for engs in sets:
            engs[v].ingest(*tv._cols(seed_items), [x[2] for x in seed_items], [x[3] for x in seed_items])
    zero = bytes(32)

    def py_reply(e, head, S):
        """ask_sync over the view's host graph: BFS from head over parents the requester lacks."""
        ids = [bytes(x) for x in e.ids()]
        hgt = e.heights()
        at = {h: i for i, h in enumerate(ids)}
        seen, q = {head}, [head]
        while q:
            u = q.pop(0)
            ev = evs[ids[u]][1]
            for p in ev.p:
                i = at[p]
                c = evs[p][4]
                if i not in seen and (S[c] < 0 or hgt[i] > S[c]):
                    seen.add(i)
                    q.append(i)
        return [evs[ids[i]] for i in sorted(seen)]

    for turn in range(12):
        perm = list(range(B))
        while any(p == i for i, p in enumerate(perm)):
            rng.shuffle(perm)
        for k, engs in enumerate(sets):
            for e in engs:
                if e.n_divided < e.n_events:
                    e.divide_rounds(e.n_divided, e.n_events - e.n_divided)
            heads = [e.n_divided - 1 for e in engs]
            sums = E.batch_sync_summary(engs, heads)
            resp = [engs[p] for p in perm]
            if k == 0:
                _, cols = E.batch_sync_reply(resp, [heads[p] for p in perm], sums)
                items = [[evs[bytes(h)] for h in c[0]] for c in cols]
            else:
                items = [py_reply(engs[p], heads[p], s) for p, s in zip(perm, sums)]
            batches = [tuple(tv._cols(it)) + ([x[2] for x in it], [x[3] for x in it]) for it in items]
            E.batch_ingest(engs, batches)
        for a, b in zip(*sets):
            assert np.array_equal(a.ids(), b.ids()) and np.array_equal(a.heights(), b.heights())
    for engs in sets:
        for e in engs:
            if e.n_divided < e.n_events:
                e.divide_rounds(e.n_divided, e.n_events - e.n_divided)
        ncs = E.batch_decide_fame(engs)
        E.batch_find_order(engs, ncs)
    for a, b in zip(*sets):
        ra, rb = a.results(), b.results()
        for k in ra:
            assert np.array_equal(ra[k], rb[k]), k
    assert min(e.n_events for e in sets[0]) > 40 * B / 2
    # sampled views against the oracle's replay of the same events in the same index order
    from oracle_engine import OracleEngine
    import util
    for v in (0, 7, 15):
        e = sets[0][v]
        ids = [bytes(x) for x in e.ids()]
        at = {h: i for i, h in enumerate(ids)}
        rows = [evs[h] for h in ids]
        par = lambda k: np.array([at[x[1].p[k]] if x[1].p else -1 for x in rows], np.int32)
        o = OracleEngine(M, len(rows))
        o.append(par(0), par(1), np.array([x[4] for x in rows], np.int32), np.array([x[1].t for x in rows]),
                 np.frombuffer(b"".join(x[1].s for x in rows), np.uint8))
        o.divide_rounds(0, len(rows))
        o.find_order(o.decide_fame())
        util.assert_same(o.results(), e.results(), what="view %d" % v)
        o.close()
