"""swirld_verify.cuh's field, encoding, scalar, double-scalar and hash functions value for value against exact Python
integers (tests/arith_cases.py), at their carry, canonicalisation and byte-position edges.  Every family runs on the
host build of tests/verify_harness.py without a GPU; the same assertions run on the sm_90a build on the GPU, whose
outputs must also equal the host build's byte for byte.

Field outputs are checked for their value mod p and for their limbs: every output limb stays below
arith_cases.LIMB_BOUND (2^52), which fe_sub's precondition asks of its operands."""
import numpy as np
import pytest

import arith_cases as ac
import verify_cases as vc
import verify_harness as vh

P, L = ac.P, ac.L


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    if vh.nvcc() is None:
        pytest.skip("nvcc not available")
    return vh.Harness(vh.compile_lib(tmp_path_factory.mktemp("arith_host"), device=False), device=False)


@pytest.fixture(scope="module")
def device(tmp_path_factory):
    return vh.Harness(vh.compile_lib(tmp_path_factory.mktemp("arith_device"), device=True), device=True)


def _rows(bs, width=32):
    return np.frombuffer(b"".join(bs), np.uint8).reshape(-1, width)


def _ints(a):
    return [int.from_bytes(r.tobytes(), "little") for r in a]


MAX_LIMB = {}                                  # the largest output limb seen per operation and build


def _limbs_ok(h, op, out, want):
    """out: (n, 5) limbs; want: exact values mod p."""
    mx = int(out.max()) if out.size else 0
    key = ("device" if h.device else "host", op)
    MAX_LIMB[key] = max(MAX_LIMB.get(key, 0), mx)
    assert mx < ac.LIMB_BOUND, (op, hex(mx))
    bad = [i for i, (o, w) in enumerate(zip(out, want)) if ac.value(o) % P != w % P]
    assert not bad, (op, [(i, [hex(int(x)) for x in out[i]], hex(want[i] % P)) for i in bad[:5]])


# ---------------------------------------------------------------- families: each returns its raw outputs
def field(h):
    got = {}
    a, b, va, vb = ac.field_pairs()
    for op, f in (("fe_add", lambda x, y: x + y), ("fe_sub", lambda x, y: x - y), ("fe_mul", lambda x, y: x * y)):
        got[op] = out = h.fe_binary(op, a, b)
        _limbs_ok(h, op, out, [f(x, y) for x, y in zip(va, vb)])
    x, vx = ac.field_inputs()
    for op, f in (("fe_sq", lambda v: v * v), ("fe_neg", lambda v: -v),
                  ("fe_invert", lambda v: pow(v, P - 2, P)), ("fe_pow22523", lambda v: pow(v, (P - 5) // 8, P))):
        got[op] = out = h.fe_unary(op, x)
        _limbs_ok(h, op, out, [f(v) for v in vx])
    # fe_invert of 0 and of p (both 0) and of p - 1 (itself), as values the field meets
    for v, want in ((0, 0), (P, 0), (P - 1, P - 1)):
        assert ac.value(h.fe_unary("fe_invert", np.array([ac.limbs_of(v)], np.uint64))[0]) % P == want, v
    # 1000 squarings in one chain
    chain = [2, 3, P - 1, ac.D, ac.SQRTM1, (1 << 255) - 1, (1 << 51) - 19]
    got["fe_sqn"] = out = h.fe_sqn(np.array([ac.limbs_of(v) for v in chain], np.uint64), 1000)
    _limbs_ok(h, "fe_sqn", out, [pow(v, 1 << 1000, P) for v in chain])
    # fe_tobytes: exactly x mod p, whatever the limbs
    got["fe_tobytes"] = tb = h.fe_tobytes(x)
    bad = [i for i, (o, v) in enumerate(zip(tb, vx)) if o.tobytes() != ac.fe_bytes(v)]
    assert not bad, [(i, [hex(int(l)) for l in x[i]], tb[i].tobytes().hex()) for i in bad[:5]]
    got["fe_iszero"] = z = h.fe_flag("fe_iszero", x)
    assert list(z) == [int(v % P == 0) for v in vx]
    got["fe_isneg"] = s = h.fe_flag("fe_isneg", x)
    assert list(s) == [(v % P) & 1 for v in vx]
    # fe_frombytes: bit 255 ignored, a value >= p kept as it is, limbs exact
    vals = ac.field_values()
    enc = _rows([v.to_bytes(32, "little") for v in vals] + [(v | (1 << 255)).to_bytes(32, "little") for v in vals])
    got["fe_frombytes"] = fb = h.fe_frombytes(enc)
    assert [list(map(int, r)) for r in fb] == [ac.limbs_of(v) for v in vals + vals]
    return got


def encodings(h):
    got = {}
    encs = ac.encodings()
    s = _rows(encs)
    got["y_canonical"] = yc = h.y_canonical(s)
    bad = [e.hex() for e, c in zip(encs, yc) if bool(c) != (ac.y_raw(e) < P)]
    assert not bad, bad[:5]
    pts = [vc.dec(e) for e in encs]
    # every lowered byte position has a y that decodes, with either sign
    for i in range(1, 31):
        assert any(p is not None for e, p in zip(encs, pts) if e[i] == 0xfe and ac.y_raw(e) < P), i
    for neg in (0, 1):
        ok, out = h.ge_decode(s, np.full(len(encs), neg, np.uint8))
        got["ge_decode_%d" % neg] = (ok, out * ok[:, None])
        for e, p, o, q in zip(encs, pts, ok, out):
            assert bool(o) == (p is not None), e.hex()
            if p is not None:
                assert q.tobytes() == vc.enc(ac.negate(p) if neg else p), (e.hex(), neg)
    # the key path: y < p, decodes, [8]A != O; then [1..15](-A)
    ok, tab, t_ok = h.point_table(s)
    got["point_table"] = (ok, tab * ok[:, None, None], t_ok * ok[:, None])
    n_acc = 0
    for e, p, o, t, tk in zip(encs, pts, ok, tab, t_ok):
        want = ac.y_raw(e) < P and p is not None and not ac.small_order(ac.ext(p))
        assert bool(o) == want, e.hex()
        if want:
            n_acc += 1
            assert [r.tobytes() for r in t] == ac.table(ac.negate(p)), e.hex()
            assert tk.all(), e.hex()
    assert n_acc > 100
    return got


def scalars(h):
    got = {}
    vals = ac.sc_canonical_values()
    got["sc_canonical"] = c = h.sc_canonical(_rows([v.to_bytes(32, "little") for v in vals]))
    assert [bool(x) for x in c] == [v < L for v in vals], [hex(v) for v, x in zip(vals, c) if bool(x) != (v < L)]
    vals = ac.sc_reduce_values()
    got["sc_reduce512"] = r = h.sc_reduce512(_rows([v.to_bytes(64, "little") for v in vals], 64))
    bad = [hex(v) for v, x in zip(vals, _ints(r)) if x != v % L]
    assert not bad, bad[:5]
    return got


_CASES = {}


def _cached(fn):
    if fn not in _CASES:
        _CASES[fn] = fn()
    return _CASES[fn]


def double_scalar(h):
    rows = _cached(ac.double_scalar_cases)
    S = _rows([s.to_bytes(32, "little") for s, *_ in rows])
    k = _rows([x.to_bytes(32, "little") for _, x, *_ in rows])
    a_ok, q, small, verdict = h.double_scalar(S, k, _rows([r[2] for r in rows]), _rows([r[3] for r in rows]))
    assert a_ok.all()
    bad = [(hex(s), hex(x), A.hex()) for (s, x, A, _, Q, *_), g in zip(rows, q) if g.tobytes() != Q]
    assert not bad, (len(bad), bad[:5])
    assert [bool(x) for x in small] == [r[5] for r in rows]
    bad = [(hex(s), hex(x), A.hex(), R.hex()) for (s, x, A, R, _, _, want), g in zip(rows, verdict) if bool(g) != want]
    assert not bad, (len(bad), bad[:5])
    assert any(r[5] for r in rows) and any(ac.y_raw(r[3]) >= P for r in rows)       # small Q, and y + p aliases
    return {"q": q, "small": small, "verdict": verdict}


def verdicts(h):
    """crypto_sign_verify_detached as the two kernels compose it, on every family of verify_cases, against libsodium."""
    cases = _cached(vc.build)
    got = h.verify(_rows([c.sig for c in cases], 64), _rows([c.pk for c in cases]), *vh.packed([c.msg for c in cases]))
    bad = [(i, c.family) for i, (c, g) in enumerate(zip(cases, got)) if bool(g) != c.ok_sig]
    assert not bad, bad[:20]
    return {"verify": got}


def hashes(h):
    buf, off, ln, sha, b2 = ac.hash_cases()
    got = {}
    for op, want in (("sha512", sha), ("blake2b_256", b2)):
        got[op] = out = h.hash(op, buf, off, ln)
        bad = [(n, o) for n, o, g, w in zip(ln, off, out, want) if g.tobytes() != w]
        assert not bad, (op, bad[:10])
    return got


FAMILIES = [field, encodings, scalars, double_scalar, hashes, verdicts]


@pytest.mark.parametrize("family", FAMILIES, ids=lambda f: f.__name__)
def test_host_build(host, family):
    family(host)


_HOST = {}


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES, ids=lambda f: f.__name__)
def test_device_build(host, device, family):
    got = family(device)
    if family.__name__ not in _HOST:
        _HOST[family.__name__] = family(host)
    want = _HOST[family.__name__]
    assert got.keys() == want.keys()
    for k in got:
        g, w = (got[k], want[k]) if isinstance(got[k], tuple) else ((got[k],), (want[k],))
        for x, y in zip(g, w):
            assert x.dtype == y.dtype and np.array_equal(x, y), (family.__name__, k)
