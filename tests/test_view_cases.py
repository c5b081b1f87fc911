"""The node views of tests/view_cases.py are what a node holds, and each reaches the sizes it is there for.  Oracle and
model only (no GPU): a change of traces.node_view, a generator or a schedule that breaks a view or shrinks a case fails
here.  Run with -rA or -s to see each case's sizes."""
import numpy as np
import pytest

import view_cases as vc
import shape_cases as sc


def _base_index(base, view):
    """The base index of every view event (signatures are distinct)."""
    key = {bytes(s): i for i, s in enumerate(base.sig)}
    return np.array([key[bytes(s)] for s in view.sig], np.int64)


def _ancestors(base, x):
    seen = np.zeros(base.N, bool)
    seen[x] = True
    p0, p1 = base.p0.tolist(), base.p1.tolist()
    for i in range(x, -1, -1):
        if seen[i] and p0[i] >= 0:
            seen[p0[i]] = seen[p1[i]] = True
    return np.flatnonzero(seen)


def check_view(base, X, view, sizes):
    """view is a valid arrival order of X's knowledge: topological, fork-free as sw_append validates it, exactly the
    ancestors of X's last event, every call ends with X's own event, t and sig those of the base event."""
    N = view.N
    assert sum(sizes) == N and min(sizes) >= 1
    i = np.arange(N)
    assert np.all(view.p0 < i) and np.all(view.p1 < i)
    head = [-1] * view.M
    p0, p1, cr = view.p0.tolist(), view.p1.tolist(), view.creator.tolist()
    for h in range(N):
        c = cr[h]
        if p0[h] < 0:
            assert p1[h] < 0 and head[c] < 0, "event %d: a second root of member %d" % (h, c)
        else:
            assert p1[h] >= 0 and cr[p0[h]] == c and cr[p1[h]] != c
            assert head[c] == p0[h], "event %d: the self-parent is not member %d's latest event (fork)" % (h, c)
        head[c] = h
    ends = np.cumsum(sizes) - 1
    assert np.all(view.creator[ends] == X), "a call does not end with the node's own event"
    bi = _base_index(base, view)
    chain = np.flatnonzero(base.creator == X)
    assert bi[-1] == chain[-1]
    assert np.array_equal(np.sort(bi), _ancestors(base, chain[-1]))
    assert np.array_equal(bi[ends], chain), "call j does not end with X's j-th event"
    for col in ("p0", "p1"):
        v, b = getattr(view, col), getattr(base, col)[bi]
        assert np.array_equal(np.where(v >= 0, bi[np.maximum(v, 0)], -1), b)
    assert np.array_equal(view.creator, base.creator[bi])
    assert np.array_equal(view.t, base.t[bi]) and np.array_equal(view.sig, base.sig[bi])


@pytest.mark.parametrize("name", list(vc.CASES))
def test_view_is_what_the_node_holds(name):
    from swirld_b200 import traces
    case = vc.CASES[name]
    base = getattr(traces, case.gen)(**case.kw)
    view, sizes = case.view()
    check_view(base, case.node, view, sizes)
    assert sum(case.calls()) == view.N
    if not case.resident:                                # (merged syncs end with the last one's own event too)
        assert np.all(view.creator[np.cumsum(case.calls()) - 1] == case.node)


def test_node_views_of_every_member():
    """node_views(base) is node_view(base, X) for every X, from one can_see pass; a node sees its own events in order."""
    from swirld_b200 import traces
    base = traces.partition(6, 3000, seed=9, split=3, start=500, end=2000)
    views = traces.node_views(base)
    assert len(views) == base.M
    for X, (view, sizes) in enumerate(views):
        v1, s1 = traces.node_view(base, X)
        assert sizes == s1 and np.array_equal(view.p1, v1.p1) and np.array_equal(view.sig, v1.sig)
        check_view(base, X, view, sizes)
    rows = traces.can_see_rows(base)
    import oracle as orc
    o = orc.Oracle(base.M)
    o.append(base)
    o.divide_rounds(0, base.N)
    assert np.array_equal(rows, o.can_see())


@pytest.mark.parametrize("name", list(vc.CASES))
def test_case_exceeds_its_sizes(name):
    case = vc.CASES[name]
    tr = case.trace()
    s = vc.view_sizes(case, tr)
    o = sc.sizes(case.as_case(), tr)
    s.update({k: o[k] for k in ("run", "ring_gap", "behind", "segment")})
    s.update(o["oracle"].coverage())
    if case.resident:
        slow, row = vc.slow_sizes(case, tr)
        s.update(slow)
        assert np.array_equal(row, o["oracle"].can_see()), name + ": the scan model differs from the oracle"
    print("%s: N=%d calls=%d %s" % (name, tr.N, len(case.calls()), " ".join("%s=%d" % (k, s[k]) for k in sorted(s))))
    assert not vc.missing(case, s), "%s no longer exceeds %s" % (name, vc.missing(case, s))
