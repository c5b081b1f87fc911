"""tests/gossip_model.py checked without a GPU: every reply the model's views send equals ask_sync's BFS and the closed
form the engine's kernels select (tests/sync_model.py), every request equals the summary of the requester's head, each
view's trace replays through the oracle to a consistent order, and the schedules reach the cases the GPU loop
(tests/test_gpu_gossip_loop.py) is there for, counted."""
import numpy as np
import pytest

pytest.importorskip("nacl.bindings")

import gossip_model as gm
import sync_model as sm

CASES = {
    # two gossips, a quarter of the replies tampered: every tamper kind, drops and their dependants, refused heads
    "m4_g2_tampered": dict(M=4, G=2, turns=100, seed=3, tamper=0.2),
    # two members apart from the rest for 15 turns, then a catch-up reply
    "m5_apart": dict(M=5, G=1, turns=60, seed=4, apart=([0, 1], 15)),
}


def _run(M, G, turns, seed, tamper=0.0, apart=None):
    s = gm.make_schedule(M, G, turns, seed, tamper, apart)
    g = gm.Gossip(s)
    g.start()
    return s, g, [g.turn() for _ in range(turns)]


@pytest.fixture(scope="module", params=list(CASES))
def run(request):
    return (request.param,) + _run(**CASES[request.param])


def test_replies_and_requests(run):
    name, s, g, turns = run
    sizes = [[1] for _ in g.views]
    n_checked = 0
    for k, vt in enumerate(turns):
        before = [sm.View(x.trace(sum(sizes[v]))) for v, x in enumerate(g.views)]
        heads = {}
        for v, x in enumerate(g.views):                        # the head before the turn: the last own event so far
            own = [i for i, h in enumerate(x.arrival[:sum(sizes[v])]) if x.hg[h].c == x.pk]
            heads[v] = own[-1]
        for v, t in enumerate(vt):
            view_v = before[v]
            assert np.array_equal(t.request, sm.summary(view_v, heads[v])), (name, k, v)
            p = t.peer
            view_p = before[p]
            idx = np.array([g.views[p].index[h] for h, _ in t.reply], np.int32)
            assert idx[-1] == heads[p]
            assert np.array_equal(idx, sm.bfs_reply(view_p, heads[p], t.request)), (name, k, v)
            assert np.array_equal(idx, sm.closed_reply(view_p, heads[p], t.request)), (name, k, v)
            n_checked += 1
        for v, t in enumerate(vt):
            sizes[v].append(len(t.added) + (t.new is not None))
    assert n_checked == len(turns) * len(g.views)
    assert [x.sizes for x in g.views] == sizes


def test_arrivals_and_new_events(run):
    name, s, g, turns = run
    for vt in turns:
        for v, t in enumerate(vt):
            x = g.views[v]
            got = x.arrival[t.first:t.first + len(t.added) + (t.new is not None)]
            assert got == t.added + ([t.new[0]] if t.new else [])
            have = set(x.arrival[:t.first + len(t.added)])
            for i in t.new_rows:                           # what the view dropped was tampered or depends on a drop
                h, ev = t.delivered[i]
                if h not in have:
                    assert t.delivered[i] != t.reply[i] or any(p not in have for p in ev.p)
            if t.new:
                h, ev = t.new
                assert ev.p == (x.arrival[max(j for j in range(t.first) if x.hg[x.arrival[j]].c == x.pk)], t.reply[-1][0])
                assert gm.event_id(ev) == h


def test_oracle_replay_is_consistent(run):
    name, s, g, turns = run
    ordered = 0
    for v, x in enumerate(g.views):
        tr = x.trace()
        r = gm.replay(tr, x.sizes)
        gm.check_replay(r)
        assert (r["round"] >= 0).all()
        assert len(r["new_c"]) == len(x.sizes)
        ordered += r["transactions"].size
    assert ordered > 0, name


def test_schedules_reach_their_cases(run):
    name, s, g, turns = run
    cov = g.cov + gm.time_cases(s)
    print("%s: %s" % (name, " ".join("%s=%d" % kv for kv in sorted(cov.items()))))
    need = ["repeated_responders", "non_integral", "equal_times", "last_bit_times"]
    if name == "m4_g2_tampered":
        # known rows: after a refused head the request still names the old head, so the next reply resends what the
        # view entered in that turn
        need += ["known_rows", "tampered_sig", "tampered_msg", "tampered_id", "tampered_head", "dropped",
                 "dropped_dependants", "zero_event_views"]
    missing = [c for c in need if cov[c] == 0]
    assert not missing, "%s no longer reaches %s" % (name, missing)
    if name == "m5_apart":
        k = CASES[name]["apart"][1]
        caught_up = max(len(turns[k][v].reply) for v in CASES[name]["apart"][0])
        assert caught_up > 2 * k, caught_up
