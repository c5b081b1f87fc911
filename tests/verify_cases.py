"""Signature and id cases for the verify kernels (swirld_verify.cuh), deterministic from seeds, each with libsodium's
verdict (PyNaCl's bundled libsodium, crypto_sign_open) and hashlib's BLAKE2b-256 digest.

Families: valid signatures over messages of every length 0..320 and real event shapes, tampered bits, malleated S,
keys libsodium refuses (every encoding of every small-order point, non-points, y >= p) and mixed-order keys, small-order
and negated R, and random bytes.  A small pure-Python model of the curve finds the torsion points; nothing in it is on
the path under test.
"""
from __future__ import annotations

import hashlib
import pickle
import random
from collections import namedtuple

from nacl import bindings as nb
from nacl import exceptions as nexc

P = 2 ** 255 - 19
L = 2 ** 252 + 27742317777372353535851937790883648493
D = -121665 * pow(121666, P - 2, P) % P
SQRTM1 = pow(2, (P - 1) // 4, P)

Event = namedtuple("Event", "d p t c s")                  # the reference's event tuple (swirld.py:91-92)
Case = namedtuple("Case", "family pk sig msg pre id ok_sig ok_id")


def blake(b: bytes) -> bytes:
    return hashlib.blake2b(b, digest_size=32).digest()


def nacl_ok(sig: bytes, msg: bytes, pk: bytes) -> bool:
    try:
        nb.crypto_sign_open(sig + msg, pk)
        return True
    except nexc.CryptoError:
        return False


# ---- a small model of the curve (test side only)
def sqrt_mod(a):
    """A square root of a mod p, or None (p = 5 mod 8)."""
    a %= P
    x = pow(a, (P + 3) // 8, P)
    if x * x % P == a:
        return x
    x = x * SQRTM1 % P
    return x if x * x % P == a else None


def add(p1, p2):
    (x1, y1), (x2, y2) = p1, p2
    t = D * x1 * x2 * y1 * y2 % P
    return ((x1 * y2 + y1 * x2) * pow(1 + t, P - 2, P) % P, (y1 * y2 + x1 * x2) * pow(1 - t, P - 2, P) % P)


def enc(pt, sign=None, alias=False):
    x, y = pt
    v = y + (P if alias else 0)
    s = (x & 1) if sign is None else sign
    return (v | (s << 255)).to_bytes(32, "little")


def dec(b):
    v = int.from_bytes(b, "little")
    y, s = (v & ((1 << 255) - 1)) % P, v >> 255
    x = sqrt_mod((y * y - 1) * pow(D * y * y + 1, P - 2, P))
    if x is None:
        return None
    if (x & 1) != s:
        x = -x % P
    return (x, y)


def torsion():
    """The eight points of order dividing 8: identity, (0, -1), (+-sqrt(-1), 0) and the four of order 8 (x^2 = -y^2,
    d y^4 + 2 y^2 - 1 = 0)."""
    pts = [(0, 1), (0, P - 1), (SQRTM1, 0), (P - SQRTM1, 0)]
    r = sqrt_mod(1 + D)
    for yy in ((-1 + r) * pow(D, P - 2, P) % P, (-1 - r) * pow(D, P - 2, P) % P):
        y = sqrt_mod(yy)
        if y is None:
            continue
        for yv in (y, P - y):
            x = yv * SQRTM1 % P
            pts += [(x, yv), (P - x, yv)]
    assert len(pts) == 8
    for pt in pts:
        q = pt
        for _ in range(3):
            q = add(q, q)
        assert q == (0, 1)
    return pts


def small_order_encodings():
    """Every 32-byte encoding of a point of order dividing 8: canonical y, y + p where it fits in 255 bits, each with
    both sign bits."""
    out = set()
    for pt in torsion():
        for alias in (False, True):
            if alias and pt[1] + P >= 2 ** 255:
                continue
            for s in (0, 1):
                out.add(enc(pt, s, alias))
    return sorted(out)


def order8_point():
    return next(pt for pt in torsion() if pt[0] != 0 and pt[1] != 0)


# ---- signing
class Keys:
    def __init__(self, rng):
        self.rng = rng

    def seeded(self):
        pk, sk = nb.crypto_sign_seed_keypair(self.rng.randbytes(32))
        return pk, sk

    def scalar(self):
        return self.rng.randrange(1, L)


def sign(sk, msg):
    return nb.crypto_sign(msg, sk)[:64]


def base_mul(s: int) -> bytes:
    return nb.crypto_scalarmult_ed25519_base_noclamp(s.to_bytes(32, "little"))


def challenge(R, A, msg):
    return int.from_bytes(hashlib.sha512(R + A + msg).digest(), "little") % L


def case(family, pk, sig, msg, pre=None, id_=None):
    pre = bytes(pre if pre is not None else msg[:40] + b"pre")
    id_ = blake(pre) if id_ is None else id_
    return Case(family, bytes(pk), bytes(sig), bytes(msg), pre, bytes(id_), nacl_ok(sig, msg, pk), blake(pre) == id_)


def flip(b, bit):
    a = bytearray(b)
    a[bit >> 3] ^= 1 << (bit & 7)
    return bytes(a)


def event_shapes(rng, pk, sk, n):
    """(msg, preimage, id) of events as the reference makes them: msg = dumps((d, p, t, pk)), id = BLAKE2b of
    dumps(Event(d, p, t, pk, sig)) (swirld.py:88-95)."""
    out = []
    for j in range(n):
        d = None if j % 2 == 0 else [rng.randbytes(rng.randrange(0, 40)) for _ in range(rng.randrange(1, 4))]
        p = () if j % 5 == 0 else (rng.randbytes(32), rng.randbytes(32))
        t = 1.7e9 + rng.random() * 1e6
        msg = pickle.dumps((d, p, t, pk))
        sig = sign(sk, msg)
        pre = pickle.dumps(Event(d, p, t, pk, sig))
        out.append((msg, sig, pre, blake(pre)))
    return out


def build(seed=1):
    rng = random.Random(seed)
    keys = Keys(rng)
    cases = []
    signers = [keys.seeded() for _ in range(8)]

    # 1. valid: every message length 0..320 (SHA-512 input 64 + len crosses the padding edges at 47/48 and 175/176),
    # BLAKE2b preimages at its block edges, and event-shaped messages and ids
    for n in range(321):
        pk, sk = signers[n % len(signers)]
        m = rng.randbytes(n)
        cases.append(case("valid", pk, sign(sk, m), m, pre=rng.randbytes(n % 300)))
    for n in (0, 1, 127, 128, 129, 255, 256, 257, 384, 1000):
        pk, sk = signers[n % len(signers)]
        m = rng.randbytes(64)
        cases.append(case("valid", pk, sign(sk, m), m, pre=rng.randbytes(n)))
    for pk, sk in signers[:4]:
        for msg, sig, pre, id_ in event_shapes(rng, pk, sk, 6):
            cases.append(case("event", pk, sig, msg, pre, id_))

    # 2. tampering: one bit of R, of S, of the message, of the preimage, of the id; another member's key
    for j in range(24):
        pk, sk = signers[j % len(signers)]
        msg, sig, pre, id_ = event_shapes(rng, pk, sk, 1)[0]
        cases.append(case("tamper_r", pk, flip(sig, rng.randrange(256)), msg, pre, id_))
        cases.append(case("tamper_s", pk, flip(sig, 256 + rng.randrange(253)), msg, pre, id_))
        cases.append(case("tamper_msg", pk, sig, flip(msg, rng.randrange(8 * len(msg))), pre, id_))
        cases.append(case("tamper_pre", pk, sig, msg, flip(pre, rng.randrange(8 * len(pre))), id_))
        cases.append(case("tamper_id", pk, sig, msg, pre, flip(id_, rng.randrange(256))))
        cases.append(case("other_key", signers[(j + 1) % len(signers)][0], sig, msg, pre, id_))

    # 3. malleated S: S + L, S = L, bit 255 set, S = L - 1
    for j in range(6):
        pk, sk = signers[j]
        m = rng.randbytes(40 + j)
        sig = sign(sk, m)
        R, S = sig[:32], int.from_bytes(sig[32:], "little")
        for s2 in (S + L, L, S | (1 << 255), L - 1, S):
            cases.append(case("malleate_s", pk, R + s2.to_bytes(32, "little"), m))

    # 4. keys: every encoding of every small-order point (with signatures whose equation holds: R = [s]B, S = s), "-0",
    # a y with no square root, y >= p, and mixed-order keys A + T8
    for A in small_order_encodings() + [(1 | (1 << 255)).to_bytes(32, "little")]:
        for _ in range(2):
            s = keys.scalar()
            m = rng.randbytes(33)
            cases.append(case("key_small", A, base_mul(s) + s.to_bytes(32, "little"), m))
        pk, sk = signers[0]
        m = rng.randbytes(20)
        cases.append(case("key_small", A, sign(sk, m), m))
    y = 2
    bad = []
    while len(bad) < 3:
        if sqrt_mod((y * y - 1) * pow(D * y * y + 1, P - 2, P)) is None:
            bad.append(y)
        y += 1
    for y in bad + [P, P + 2, P + 5, P + 18, 2 ** 255 - 1]:
        for s in (0, 1):
            A = (y | (s << 255)).to_bytes(32, "little")
            pk, sk = signers[1]
            m = rng.randbytes(25)
            cases.append(case("key_bad", A, sign(sk, m), m))
    T8 = order8_point()
    for j in range(16):
        a = keys.scalar()
        Apt = add(dec(base_mul(a)), T8 if j % 2 == 0 else torsion()[2])
        A = enc(Apt)
        for _ in range(3):
            r = keys.scalar()
            R = base_mul(r)
            m = rng.randbytes(30)
            k = challenge(R, A, m)
            cases.append(case("key_mixed", A, R + ((r + k * a) % L).to_bytes(32, "little"), m))

    # 5. R: every small-order encoding; the identity with an equation that holds ([S]B - [k]A = O); -R of a valid one
    for R in small_order_encodings():
        a = keys.scalar()
        A = base_mul(a)
        m = rng.randbytes(28)
        k = challenge(R, A, m)
        cases.append(case("r_small", A, R + (k * a % L).to_bytes(32, "little"), m))
        cases.append(case("r_small", A, R + keys.scalar().to_bytes(32, "little"), m))
    for j in range(8):
        pk, sk = signers[j]
        m = rng.randbytes(50)
        sig = sign(sk, m)
        cases.append(case("r_neg", pk, flip(sig, 255), m))

    # 6. random signatures and keys
    for j in range(64):
        pk = rng.randbytes(32) if j % 2 else signers[j % 8][0]
        m = rng.randbytes(rng.randrange(0, 200))
        sig = bytearray(rng.randbytes(64))
        if j % 4 == 0:
            sig[63] &= 0x0f                                # S < 2^252 < L: canonical, so the equation decides
        cases.append(case("random", pk, bytes(sig), m))

    # (the families below draw from their own generator, so the ones above stay what they were)
    rng = random.Random(seed + 1000)
    # 7. ground: valid signatures whose S or k has four zero nibbles at nibble w..w+3 (w = 59: S or k < 2^236, the
    # top 16 bits below 2^252 clear), found by grinding the message, about 2^16 tries each
    for which in ("S", "k"):
        for w in (59, 30, 0):
            a = rng.randrange(1, L)
            A = base_mul(a)
            r = rng.randrange(1, L)
            R = base_mul(r)
            pre = rng.randbytes(20)
            for ctr in range(1 << 24):
                m = pre + ctr.to_bytes(4, "little")
                k = challenge(R, A, m)
                S = (r + k * a) % L
                if (((S if which == "S" else k) >> (4 * w)) & 0xFFFF) == 0:
                    break
            cases.append(case("ground", A, R + S.to_bytes(32, "little"), m))

    # 8. s_high: canonical S in [2^252, L) (the top nibble is 1, k's is almost surely 0) with random R; no such S of a
    # valid signature can be found, so libsodium refuses every one
    for j in range(12):
        pk = signers[j % len(signers)][0]
        S = (1 << 252) + [0, 1, L - (1 << 252) - 1][j] if j < 3 else (1 << 252) + rng.randrange(L - (1 << 252))
        R = base_mul(rng.randrange(1, L)) if j % 2 else rng.randbytes(32)
        cases.append(case("s_high", pk, R + S.to_bytes(32, "little"), rng.randbytes(40)))

    # 9. long_msg: valid signatures over messages whose SHA-512 length needs more than 16 bits
    for n in ((1 << 16) - 1, 1 << 16, (1 << 16) + 1, 1 << 20):
        pk, sk = signers[n % len(signers)]
        m = rng.randbytes(n)
        cases.append(case("long_msg", pk, sign(sk, m), m))
    return cases
