"""swirld_sign.cuh on the host (`-x c++` build of sign_harness.py), value for value against PyNaCl's libsodium and
exact Python integers; and the source-level constant-time check on the -DSWV_CT_TRACE build."""
import hashlib
import random

import numpy as np
import pytest

import sign_harness as SH
from verify_harness import nvcc

nacl = pytest.importorskip("nacl.bindings")

L = 2 ** 252 + 27742317777372353535851937790883648493
IDENTITY = bytes([1] + [0] * 31)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    if nvcc() is None:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("sign_host")
    return SH.SignHarness(SH.compile_lib(d, False), False), SH.compile_lib(d, False, trace=True)


@pytest.fixture(scope="module")
def h(libs):
    return libs[0]


def le(x, n=32):
    return x.to_bytes(n, "little")


def arr(bs, w):
    return np.frombuffer(b"".join(bs), np.uint8).reshape(-1, w).copy()


def base_enc(x):
    x %= L
    return IDENTITY if x == 0 else nacl.crypto_scalarmult_ed25519_base_noclamp(le(x))


def all_eights():
    """Scalars whose digits 0..62 all recode to -8 (the most negative digit; +8 occurs only at the top), top digit 1..8."""
    return [top * 16 ** 63 - 8 * sum(16 ** i for i in range(63)) for top in (1, 4, 7, 8)]


def test_expand(h):
    rng = random.Random(1)
    seeds = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(64)] + [bytes(32), b"\xff" * 32]
    a, prefix = h.expand(arr(seeds, 32))
    for i, s in enumerate(seeds):
        az = bytearray(hashlib.sha512(s).digest())
        az[0] &= 248; az[31] &= 127; az[31] |= 64
        assert bytes(a[i]) == bytes(az[:32]) and bytes(prefix[i]) == bytes(az[32:])


def test_recode(h):
    rng = random.Random(2)
    xs = [0, 1, L - 1, 2 ** 255 - 1, 2 ** 254 + 2 ** 253 + 248] + all_eights() + [rng.randrange(2 ** 255) for _ in range(500)]
    e = h.recode(arr([le(x) for x in xs], 32)).astype(np.int64)
    for i, x in enumerate(xs):
        assert sum(int(d) * 16 ** j for j, d in enumerate(e[i])) == x
        assert e[i, :63].min() >= -8 and e[i, :63].max() <= 7 and 0 <= e[i, 63] <= 8
    for i, x in enumerate(all_eights()):
        assert set(e[5 + i, :63].tolist()) == {-8}


def test_table(h):
    tab = h.table()
    for k in range(32):
        for j in range(8):
            assert bytes(tab[k, j]) == base_enc((j + 1) * 256 ** k), (k, j)


def test_base_mult(h):
    rng = random.Random(3)
    xs = [0, 1, 2, 8, 16, L - 1, L - 8] + all_eights() + [rng.randrange(L) for _ in range(200)] + \
         [rng.randrange(2 ** 254, 2 ** 255) & ~7 for _ in range(50)]
    a = arr([le(x) for x in xs], 32)
    want = [base_enc(x) for x in xs]
    for got in [h.base_mult(a)] + [h.lanes_mult(a, lanes) for lanes in (1, 2, 4, 8, 16, 32)]:
        assert [bytes(r) for r in got] == want


def test_reduce(h):
    rng = random.Random(4)
    xs = [0, L - 1, L, 2 * L - 1, 2 * L, 2 ** 512 - 1, 2 ** 512 - L, 2 ** 252, 2 ** 253 - 1, 2 ** 256, 2 ** 511]
    xs += [k * L + d for k in (1, 2, 3, 2 ** 64, 2 ** 128 + 7, (2 ** 512 - 1) // L) for d in (-1, 0, 1) if 0 <= k * L + d < 2 ** 512]
    xs += [rng.randrange(2 ** 512) for _ in range(500)]
    got = h.reduce(arr([le(x, 64) for x in xs], 64))
    for i, x in enumerate(xs):
        assert int.from_bytes(bytes(got[i]), "little") == x % L, hex(x)
    mu = 2 ** 512 // L
    assert mu < 2 ** 260          # the five words of mu_words; their value is checked by the reductions above


def test_muladd(h):
    rng = random.Random(5)
    ks = [0, 1, L - 1] + [rng.randrange(L) for _ in range(300)]
    As = [0, 1, 2 ** 255 - 8] + [rng.randrange(2 ** 254, 2 ** 255) & ~7 for _ in range(300)]
    rs = [0, L - 1, L - 1] + [rng.randrange(L) for _ in range(300)]
    got = h.muladd(arr([le(x) for x in ks], 32), arr([le(x) for x in As], 32), arr([le(x) for x in rs], 32))
    for i, (k, a, r) in enumerate(zip(ks, As, rs)):
        s = bytes(got[i])
        assert int.from_bytes(s, "little") == (r + k * a) % L
        want = nacl.crypto_core_ed25519_scalar_add(nacl.crypto_core_ed25519_scalar_mul(le(k), le(a % L)), le(r))
        assert s == want


def signing_case(n_keys=200, seed=6):
    """200 seeded keys and messages of every length 0..300 (SHA-512 padding edges of both hashes included)."""
    rng = random.Random(seed)
    seeds = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(n_keys)]
    msgs, who = [], []
    for ln in list(range(301)) + [79, 80, 81, 207, 208, 209, 47, 48, 49, 175, 176, 177]:
        msgs.append(bytes(rng.randrange(256) for _ in range(ln)))
        who.append(rng.randrange(n_keys))
    for k in range(n_keys):                          # every key signs at least once
        msgs.append(bytes(rng.randrange(256) for _ in range(150)))
        who.append(k)
    return seeds, msgs, who


def test_sign(h):
    seeds, msgs, who = signing_case()
    sk = h.signing_key(arr(seeds, 32))
    kp = [nacl.crypto_sign_seed_keypair(s) for s in seeds]
    assert [bytes(r[64:]) for r in sk] == [pk for pk, _ in kp]
    buf, off = SH._packed(msgs)
    sig = h.sign(sk[who], buf, off[:-1], np.diff(off))
    for i, m in enumerate(msgs):
        pk, s = kp[who[i]]
        assert bytes(sig[i]) == nacl.crypto_sign(m, s)[:64], (i, len(m))
        nacl.crypto_sign_open(bytes(sig[i]) + m, pk)


def test_sign_events_host(h):
    """The kernel's arithmetic (the lanes' partial combs summed), its signature copied into the preimage and hashed."""
    seeds, msgs, who = signing_case(20, 7)
    msgs = msgs[::7]
    who = [w % 20 for w in who[::7]]
    sk = h.signing_key(arr(seeds, 32))
    pres = [b"<" + m + bytes(64) + b">" for m in msgs]
    at = [1 + len(m) for m in msgs]
    for lanes in (1, 8):
        sig, ids = h.sign_events(lanes, sk[who], msgs, pres, at)
        for i, m in enumerate(msgs):
            s = nacl.crypto_sign(m, nacl.crypto_sign_seed_keypair(seeds[who[i]])[1])[:64]
            assert bytes(sig[i]) == s
            assert bytes(ids[i]) == hashlib.blake2b(b"<" + m + s + b">", digest_size=32).digest()


def test_constant_time_trace(libs):
    """The table rows and entries read and the loop trip counts of key expansion, [a]B and a signature are the same
    for 1000 random keys and messages of one length (the host build runs one lane; the kernel's shuffle offsets are
    the constants LANES/2 .. 1)."""
    lib = SH.C.CDLL(libs[1])
    rng = random.Random(8)
    first = None
    for _ in range(1000):
        seed = bytes(rng.randrange(256) for _ in range(32))
        msg = bytes(rng.randrange(256) for _ in range(150))
        tr = SH.trace_sign(lib, seed, msg)
        if first is None:
            first = tr
            kinds = tr >> 40
            assert (kinds == 1).sum() == 2 * 64 * 8        # [a]B and [r]B: 64 lookups of all 8 entries each
        assert np.array_equal(tr, first)
