"""The field, group and hash functions of swirld_verify.cuh, built for the host with nvcc (no device needed), against
libsodium (PyNaCl) and hashlib on every family of tests/verify_cases.py: verdict for verdict, digest for digest.
The library runs the same functions on the GPU only; this build exists to check them."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess

import pytest

import verify_cases as vc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "py-swirld_b200", "csrc")

SHIM = r'''
#include "swirld_verify.cuh"
extern "C" {
int swv_key(const uint8_t *pk, swv::gc *tab) { return swv::point_table(pk, true, true, tab); }
void swv_sha512(const uint8_t *in, int64_t len, uint8_t *out) {
    swv::sha512(out, len, [&](int64_t i) -> uint8_t { return in[i]; });
}
void swv_blake2b(const uint8_t *in, int64_t len, uint8_t *out) {
    swv::blake2b_256(out, len, [&](int64_t i) -> uint8_t { return in[i]; });
}
void swv_reduce(const uint8_t *h, uint8_t *out) { swv::sc_reduce512(out, h); }
// crypto_sign_verify_detached, as the two kernels compute it
int swv_verify(const uint8_t *sig, const uint8_t *pk, const uint8_t *msg, int64_t len) {
    static swv::gc btab[swv::TAB];
    static bool have_b = false;
    if (!have_b) { uint8_t b[32]; swv::base_encoding(b); swv::point_table(b, false, false, btab); have_b = true; }
    swv::gc atab[swv::TAB];
    if (!swv::point_table(pk, true, true, atab) || !swv::sc_canonical(sig + 32)) return 0;
    uint8_t k[32];
    swv::challenge(k, sig, pk, msg, len);
    return swv::signature_equation(sig, k, btab, atab);
}
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("verify_host")
    src, so = d / "shim.cu", d / "libverify_host.so"
    src.write_text(SHIM)
    # -x c++: the host build alone (no device code is compiled, and none is needed to call these functions)
    subprocess.check_call([nvcc, "-x", "c++", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-Wno-unknown-pragmas",
                           "-I", CSRC, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.swv_key.argtypes = [C.c_char_p, C.c_void_p]
    L.swv_sha512.argtypes = [C.c_char_p, C.c_int64, C.c_char_p]
    L.swv_blake2b.argtypes = [C.c_char_p, C.c_int64, C.c_char_p]
    L.swv_reduce.argtypes = [C.c_char_p, C.c_char_p]
    L.swv_verify.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64]
    return L


@pytest.fixture(scope="module")
def cases():
    return vc.build()


def _digest(fn, data, n):
    out = C.create_string_buffer(n)
    fn(data, len(data), out)
    return out.raw


def test_sha512_every_length(lib):
    for n in list(range(0, 400)) + [1000, 4096]:
        m = bytes((7 * i + n) & 0xff for i in range(n))
        assert _digest(lib.swv_sha512, m, 64) == hashlib.sha512(m).digest(), n


def test_blake2b_every_length(lib):
    for n in list(range(0, 400)) + [1000, 4096]:
        m = bytes((5 * i + n) & 0xff for i in range(n))
        assert _digest(lib.swv_blake2b, m, 32) == vc.blake(m), n


def test_reduce_mod_l(lib):
    import random
    rng = random.Random(3)
    vals = [0, 1, vc.L - 1, vc.L, vc.L + 1, 2 ** 512 - 1, 2 ** 256, vc.L * vc.L] + [rng.getrandbits(512) for _ in range(200)]
    for v in vals:
        out = C.create_string_buffer(32)
        lib.swv_reduce(v.to_bytes(64, "little"), out)
        assert int.from_bytes(out.raw, "little") == v % vc.L, v


def test_key_verdicts(lib, cases):
    """What libsodium says about a key alone: a key is refused exactly when no signature under it verifies; every key
    of the cases that signed a valid message is accepted."""
    tab = C.create_string_buffer(15 * 4 * 5 * 8)
    good = {c.pk for c in cases if c.ok_sig}
    for A in vc.small_order_encodings():
        assert lib.swv_key(A, tab) == 0, A.hex()
    for pk in good:
        assert lib.swv_key(pk, tab) == 1, pk.hex()


def test_every_family_against_libsodium(lib, cases):
    bad = []
    for i, c in enumerate(cases):
        got = bool(lib.swv_verify(c.sig, c.pk, c.msg, len(c.msg)))
        if got != c.ok_sig:
            bad.append((i, c.family, got, c.ok_sig))
        assert (_digest(lib.swv_blake2b, c.pre, 32) == c.id) == c.ok_id, (i, c.family)
    assert not bad, bad[:20]
    fams = {c.family for c in cases}
    assert {"valid", "event", "tamper_r", "tamper_s", "tamper_msg", "tamper_pre", "tamper_id", "other_key",
            "malleate_s", "key_small", "key_bad", "key_mixed", "r_small", "r_neg", "random"} <= fams
