"""The field, group and hash functions of swirld_verify.cuh, built for the host with nvcc (no device needed), against
libsodium (PyNaCl) and hashlib on every family of tests/verify_cases.py: verdict for verdict, digest for digest.
The library runs the same functions on the GPU only; this build (tests/verify_harness.py) exists to check them."""
import hashlib
import random

import numpy as np
import pytest

import verify_cases as vc
import verify_harness as vh


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if vh.nvcc() is None:
        pytest.skip("nvcc not available")
    return vh.Harness(vh.compile_lib(tmp_path_factory.mktemp("verify_host"), device=False), device=False)


@pytest.fixture(scope="module")
def cases():
    return vc.build()


def _rows(bs, width):
    return np.frombuffer(b"".join(bs), np.uint8).reshape(-1, width)


def _digests(lib, op, msgs):
    return [d.tobytes() for d in lib.hash(op, *vh.packed(msgs))]


def test_sha512_every_length(lib):
    ns = list(range(0, 400)) + [1000, 4096]
    msgs = [bytes((7 * i + n) & 0xff for i in range(n)) for n in ns]
    for n, m, d in zip(ns, msgs, _digests(lib, "sha512", msgs)):
        assert d == hashlib.sha512(m).digest(), n


def test_blake2b_every_length(lib):
    ns = list(range(0, 400)) + [1000, 4096]
    msgs = [bytes((5 * i + n) & 0xff for i in range(n)) for n in ns]
    for n, m, d in zip(ns, msgs, _digests(lib, "blake2b_256", msgs)):
        assert d == vc.blake(m), n


def test_reduce_mod_l(lib):
    rng = random.Random(3)
    vals = [0, 1, vc.L - 1, vc.L, vc.L + 1, 2 ** 512 - 1, 2 ** 256, vc.L * vc.L] + [rng.getrandbits(512) for _ in range(200)]
    out = lib.sc_reduce512(_rows([v.to_bytes(64, "little") for v in vals], 64))
    for v, o in zip(vals, out):
        assert int.from_bytes(o.tobytes(), "little") == v % vc.L, v


def test_key_verdicts(lib, cases):
    """What libsodium says about a key alone: a key is refused exactly when no signature under it verifies; every key
    of the cases that signed a valid message is accepted."""
    small = vc.small_order_encodings()
    good = sorted({c.pk for c in cases if c.ok_sig})
    ok = lib.point_table(_rows(small + good, 32))[0]
    for A, o in zip(small + good, ok):
        assert bool(o) == (A in good), A.hex()


def test_every_family_against_libsodium(lib, cases):
    buf, off, ln = vh.packed([c.msg for c in cases])
    got = lib.verify(_rows([c.sig for c in cases], 64), _rows([c.pk for c in cases], 32), buf, off, ln)
    bad = [(i, c.family, bool(g), c.ok_sig) for i, (c, g) in enumerate(zip(cases, got)) if bool(g) != c.ok_sig]
    ids = _digests(lib, "blake2b_256", [c.pre for c in cases])
    for i, (c, d) in enumerate(zip(cases, ids)):
        assert (d == c.id) == c.ok_id, (i, c.family)
    assert not bad, bad[:20]
    fams = {c.family for c in cases}
    assert {"valid", "event", "tamper_r", "tamper_s", "tamper_msg", "tamper_pre", "tamper_id", "other_key",
            "malleate_s", "key_small", "key_bad", "key_mixed", "r_small", "r_neg", "random", "ground", "s_high",
            "long_msg"} <= fams
