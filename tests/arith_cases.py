"""Inputs at the carry, canonicalisation and byte-position edges of swirld_verify.cuh's arithmetic, each with its exact
value from Python integers: the field mod p on raw radix-2^51 limbs, point encodings, scalars mod L, the
double-scalar product [S]B + [k](-A) and the two hashes.  CPU only; tests/test_verify_arith.py runs them through
both builds of tests/verify_harness.py.

The random operands of the verdict tests (tests/verify_cases.py) reach an edge like "limb 0 is exactly 2^51 after the
carry" or "S is at least 2^252" about once in 2^40 or more; these cases reach every such edge on purpose."""
from __future__ import annotations

import hashlib
import itertools
import random

import numpy as np

import verify_cases as vc

P, L, D, SQRTM1 = vc.P, vc.L, vc.D, vc.SQRTM1
M51 = (1 << 51) - 1

# The bound every field operation's output limbs must stay below.  fe_sub(a, b) computes a + 4p - b limb by limb and
# is exact only while b's limbs are below 2^53; any output may become the b of an fe_sub (or both operands of an
# fe_add whose sum then goes there), so outputs must stay below half that.  The limbs the operations leave are a
# little above 2^51 at most (limb 0 or 1, after the wrap-around carry times 19), far below.
LIMB_BOUND = (1 << 53) // 2

# limb values at the edges of the carries: 2^51 - 19 plus the 19 of a wrapped carry is exactly 2^51; fe_add and
# fe_sub leave limbs up to 2^51 + 73 on reduced operands
EDGE_LIMBS = (0, 1, M51 - 18, M51, 1 << 51, (1 << 51) + 73)


# ---------------------------------------------------------------- the field
def limbs_of(x: int) -> list[int]:
    """x < 2^255 as five limbs below 2^51."""
    assert 0 <= x < 1 << 255
    return [(x >> (51 * i)) & M51 for i in range(5)]


def value(limbs) -> int:
    return sum(int(l) << (51 * i) for i, l in enumerate(limbs))


def field_values() -> list[int]:
    """Values below 2^255: the small ones, (p +- 1) / 2, p - 2, p - 1, every value from p to 2^255 - 1 (all 19 of
    them: fe_frombytes keeps them as they are), 2^(51 i) +- 1 at each limb boundary, d and sqrt(-1)."""
    vals = [0, 1, 2, 19, (P - 1) // 2, (P + 1) // 2, P - 2, P - 1] + list(range(P, 1 << 255))
    for i in range(1, 6):
        vals += [(1 << (51 * i)) - 1] + ([(1 << (51 * i)) + 1] if i < 5 else [])
    vals += [D, SQRTM1, P - D, P - SQRTM1]
    rng = random.Random(1)
    vals += [rng.getrandbits(255) for _ in range(16)]
    return list(dict.fromkeys(vals))


def field_inputs():
    """(limb vectors, their values): every value of field_values() as canonical limbs, then every vector of five
    limbs drawn from EDGE_LIMBS (6^5 of them)."""
    vecs = [limbs_of(x) for x in field_values()] + [list(t) for t in itertools.product(EDGE_LIMBS, repeat=5)]
    a = np.array(vecs, np.uint64)
    return a, [value(v) for v in vecs]


def field_pairs():
    """Operand pairs for the binary operations: every value against every value, and every edge vector against
    zero, one, p - 1, itself, and another edge vector."""
    a, vals = field_inputs()
    nv = len(field_values())
    idx = [(i, j) for i in range(nv) for j in range(nv)]
    n = len(a)
    special = [vals.index(0), vals.index(1), vals.index(P - 1)]
    for i in range(nv, n):
        idx += [(i, s) for s in special] + [(s, i) for s in special]
        idx += [(i, i), (i, nv + (7 * i + 3) % (n - nv))]
    ia, ib = np.array(idx).T
    return a[ia], a[ib], [vals[i] for i in ia], [vals[i] for i in ib]


def fe_bytes(x: int) -> bytes:
    return (x % P).to_bytes(32, "little")


# ---------------------------------------------------------------- encodings
P_BYTES = P.to_bytes(32, "little")                   # ed ff .. ff 7f


def with_byte(b: bytes, i: int, v: int) -> bytes:
    a = bytearray(b)
    a[i] = v
    return bytes(a)


def y_encodings() -> list[bytes]:
    """y (bit 255 clear) at the edges of y < p: 0, +-1, +-2; p's pattern with one byte i in 1..30 lowered to 0xfe and
    byte 0 anywhere in 0xed..0xff (all below p); byte 0 = 0xec, 0xed, 0xee with every other byte p's (p - 1, p,
    p + 1); every value from p to 2^255 - 1."""
    ys = [y.to_bytes(32, "little") for y in (0, 1, P - 1, 2, P - 2)]
    for i in range(1, 31):
        for b0 in range(0xed, 0x100):
            ys.append(with_byte(with_byte(P_BYTES, i, 0xfe), 0, b0))
    ys += [with_byte(P_BYTES, 0, b0) for b0 in (0xec, 0xed, 0xee)]
    ys += [y.to_bytes(32, "little") for y in range(P + 2, 1 << 255)]
    return list(dict.fromkeys(ys))


def encodings() -> list[bytes]:
    """Every y of y_encodings() with both sign bits."""
    return [with_byte(y, 31, y[31] | s) for y in y_encodings() for s in (0, 0x80)]


def y_raw(s: bytes) -> int:
    return int.from_bytes(s, "little") & ((1 << 255) - 1)


def negate(pt):
    return (-pt[0] % P, pt[1])


# ---------------------------------------------------------------- points in extended coordinates (X : Y : Z : T)
def ext(pt):
    x, y = pt
    return (x, y, 1, x * y % P)


IDENT = (0, 1, 1, 0)


def padd(p, q):
    """Hisil-Wong-Carter-Dawson addition for a = -1 (complete)."""
    X1, Y1, Z1, T1 = p
    X2, Y2, Z2, T2 = q
    A = (Y1 - X1) * (Y2 - X2) % P
    B = (Y1 + X1) * (Y2 + X2) % P
    Cc = 2 * D * T1 * T2 % P
    Dd = 2 * Z1 * Z2 % P
    E, F, G, H = B - A, Dd - Cc, Dd + Cc, B + A
    return (E * F % P, G * H % P, F * G % P, E * H % P)


def affine(p):
    X, Y, Z, _ = p
    zi = pow(Z, P - 2, P)
    return (X * zi % P, Y * zi % P)


def pneg(p):
    X, Y, Z, T = p
    return (-X % P, Y, Z, -T % P)


def small_order(p) -> bool:
    for _ in range(3):
        p = padd(p, p)
    return p[0] == 0 and p[1] == p[2]


class Multiples:
    """[s]P for any s < 2^256 from the 256 doublings of P."""

    def __init__(self, p):
        self.dbl = [p]
        for _ in range(255):
            self.dbl.append(padd(self.dbl[-1], self.dbl[-1]))

    def __call__(self, s):
        acc = IDENT
        for i in range(256):
            if s >> i & 1:
                acc = padd(acc, self.dbl[i])
        return acc


def base_point():
    return vc.dec(vc.base_mul(1))


def table(pt) -> list[bytes]:
    """enc([1..15] pt)"""
    out, acc = [], ext(pt)
    for _ in range(15):
        out.append(vc.enc(affine(acc)))
        acc = padd(acc, ext(pt))
    return out


# ---------------------------------------------------------------- scalars
def sc_canonical_values() -> list[int]:
    """At L: L - 1, L, L + 1, L with one 64-bit word one more or one less (word 2 of L is 0: one more only); and
    2^252 +- 1, 2^253 - 1, 2^256 - 1, 0."""
    vals = [0, L - 1, L, L + 1, (1 << 252) - 1, (1 << 252) + 1, (1 << 253) - 1, (1 << 256) - 1]
    for w in range(4):
        vals.append(L + (1 << (64 * w)))
        if (L >> (64 * w)) & ((1 << 64) - 1):
            vals.append(L - (1 << (64 * w)))
    return vals


def sc_reduce_values() -> list[int]:
    """kL - 1, kL, kL + 1 for k = 1, 2, 2^128 and the largest k with kL < 2^512; 2^i and 2^i - 1 for every i < 512;
    2^512 - 1."""
    vals = []
    for k in (1, 2, 1 << 128, ((1 << 512) - 1) // L):
        vals += [k * L - 1, k * L, k * L + 1]
    for i in range(512):
        vals += [1 << i, (1 << i) - 1]
    vals.append((1 << 512) - 1)
    vals = list(dict.fromkeys(vals))
    assert all(0 <= v < 1 << 512 for v in vals)
    return vals


def scalars() -> list[int]:
    """Scalars below L for the double-scalar product: 0, 1, 15, 16, 17, 16^j for every nibble position, L - 1,
    2^252 - 1, values in [2^252, L) (the top nibble is 1 and k's is almost always 0), runs of zero nibbles and of 0xF
    nibbles at several positions."""
    rng = random.Random(5)
    vals = [0, 1, 15, 16, 17, L - 1, L - 2, (1 << 252) - 1]
    vals += [16 ** j for j in range(63)]
    vals += [1 << 252, (1 << 252) + 1, (1 << 252) + 15] + [(1 << 252) + rng.randrange(L - (1 << 252)) for _ in range(5)]
    for lo, n in ((0, 8), (7, 5), (28, 12), (50, 13), (59, 4)):
        run = ((1 << (4 * n)) - 1) << (4 * lo)
        vals.append(run)                                                    # a run of 0xF alone
        vals.append(rng.randrange(1 << 252) & ~run)                         # a run of zeros
        vals.append(rng.randrange(1 << 252) | run)                          # a run of 0xF in random nibbles
    vals = list(dict.fromkeys(v for v in vals if v < L))
    return vals


def keys():
    """Points A for the double-scalar product, as (name, encoding): B and -B (S = k gives the identity with A = B),
    random keys, the first two mixed-order keys of verify_cases (A + T, T of order 8 and of order 4), and edge keys:
    accepted keys whose y is p's pattern with one byte lowered."""
    rng = random.Random(9)
    out = [("B", vc.base_mul(1)), ("-B", vc.enc(negate(base_point())))]
    out += [("random", vc.base_mul(rng.randrange(1, L))) for _ in range(3)]
    mixed = list(dict.fromkeys(c.pk for c in vc.build() if c.family == "key_mixed"))
    out += [("mixed", A) for A in mixed[:2]]
    edge = [s for s in encodings() if y_raw(s) < P and vc.dec(s) is not None and not small_order(ext(vc.dec(s)))]
    out += [("edge", edge[j]) for j in (0, len(edge) // 2, len(edge) - 1)]
    return out


def double_scalar_cases():
    """Rows (S, k, A, R, Q, small, verdict): Q = enc([S]B + [k](-A)), small = [8]Q is the identity, and the verdict
    of signature_equation on (R, S).  For each A and scalar: (S, 0), (0, k), (S, k = S), (S, k reversed) and (S, k
    shuffled); each with R = Q (accepted exactly when Q is not of small order), R with its sign bit flipped, and,
    where Q's y < 19, R as y + p (both refused)."""
    sc = scalars()
    rng = random.Random(13)
    shuf = sc[:]
    rng.shuffle(shuf)
    pairs = [(s, 0) for s in sc] + [(0, k) for k in sc] + list(zip(sc, sc)) + list(zip(sc, sc[::-1])) + list(zip(sc, shuf))
    mB = Multiples(ext(base_point()))
    sB = {s: mB(s) for s in sc}
    rows = []
    for _, A in keys():
        mA = Multiples(pneg(ext(vc.dec(A))))
        kA = {k: mA(k) for k in sc}
        for s, k in pairs:
            q = padd(sB[s], kA[k])
            x, y = affine(q)
            R = vc.enc((x, y))
            small = small_order(q)
            rows.append((s, k, A, R, R, small, not small))
            rows.append((s, k, A, vc.enc((x, y), sign=1 - (x & 1)), R, small, False))
            if y < 19:
                rows.append((s, k, A, vc.enc((x, y), alias=True), R, small, False))
    return rows


# ---------------------------------------------------------------- hashes
HASH_LENGTHS = list(range(401)) + [(1 << 16) - 1, 1 << 16, (1 << 16) + 1, 1 << 20]


def hash_cases():
    """(buffer, offsets, lengths, sha512 digests, blake2b-256 digests): every length of HASH_LENGTHS at byte offsets
    0..7 into one shared buffer."""
    buf = np.frombuffer(random.Random(17).randbytes((1 << 20) + 64), np.uint8)
    off = [o for n in HASH_LENGTHS for o in range(8)]
    ln = [n for n in HASH_LENGTHS for _ in range(8)]
    raw = buf.tobytes()
    sha = [hashlib.sha512(raw[o:o + n]).digest() for o, n in zip(off, ln)]
    b2 = [vc.blake(raw[o:o + n]) for o, n in zip(off, ln)]
    return buf, off, ln, sha, b2
