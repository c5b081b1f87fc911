"""One C++ source over swirld_verify.cuh whose extern "C" entry points each apply one swv:: function to arrays of n
inputs, built two ways: `-x c++` for the host (no device needed), and with the library's nvcc flags for sm_90a, where
each entry point runs a grid-stride kernel on device pointers.  `Harness` calls either build with numpy arrays and
returns numpy arrays, so one set of assertions can check both and the two builds can be compared byte for byte.

Field elements cross the boundary as their five raw 64-bit limbs (radix 2^51, exactly as swv::fe holds them), so a
test sees the limbs an operation leaves and not only their value."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "py-swirld_b200", "csrc")

SOURCE = r'''
#include "swirld_verify.cuh"
#ifdef __CUDACC__
#include <cuda_runtime.h>
template <class F> __global__ void __launch_bounds__(128) k_each(int n, F f) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) f(i);
}
#endif
// f(0) .. f(n - 1): a grid-stride kernel on the device build, a loop on the host build; 0 or the CUDA error
template <class F> int each(int n, F f) {
#ifdef __CUDACC__
    if (n <= 0) return 0;
    const int blocks = n / 128 + 1 < 2048 ? n / 128 + 1 : 2048;
    k_each<<<blocks, 128>>>(n, f);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
#else
    for (int i = 0; i < n; i++) f(i);
    return 0;
#endif
}
#define EACH(body) return each(n, [=] __host__ __device__ (int i) { body; })
#define EXPORT extern "C" int
using swv::fe; using swv::ge; using swv::gc; using swv::u64;

SWV_HD fe ld(const u64 *p, int i) { fe h; for (int j = 0; j < 5; j++) h.v[j] = p[5 * i + j]; return h; }
SWV_HD void st(u64 *p, int i, const fe &h) { for (int j = 0; j < 5; j++) p[5 * i + j] = h.v[j]; }
// the encoding of a cached point (Y + X, Y - X, Z, 2dT), and whether its 2dT is 2d XY / Z
SWV_HDI bool cached_encode(uint8_t *s, const gc &c) {
    const fe X2 = swv::fe_sub(c.YpX, c.YmX), Y2 = swv::fe_add(c.YpX, c.YmX);          // 2X, 2Y
    const fe zi = swv::fe_invert(swv::fe_add(c.Z, c.Z));
    swv::fe_tobytes(s, swv::fe_mul(Y2, zi));
    s[31] ^= (uint8_t)(swv::fe_isneg(swv::fe_mul(X2, zi)) << 7);
    return swv::fe_iszero(swv::fe_sub(swv::fe_mul(swv::fe_add(c.T2d, c.T2d), c.Z), swv::fe_mul(swv::fe_d(), swv::fe_mul(X2, Y2))));
}

// ---- the field, on raw limbs
EXPORT t_fe_add(int n, const u64 *a, const u64 *b, u64 *o) { EACH(st(o, i, swv::fe_add(ld(a, i), ld(b, i)))); }
EXPORT t_fe_sub(int n, const u64 *a, const u64 *b, u64 *o) { EACH(st(o, i, swv::fe_sub(ld(a, i), ld(b, i)))); }
EXPORT t_fe_mul(int n, const u64 *a, const u64 *b, u64 *o) { EACH(st(o, i, swv::fe_mul(ld(a, i), ld(b, i)))); }
EXPORT t_fe_sq(int n, const u64 *a, u64 *o) { EACH(st(o, i, swv::fe_sq(ld(a, i)))); }
EXPORT t_fe_sqn(int n, int k, const u64 *a, u64 *o) { EACH(st(o, i, swv::fe_sqn(ld(a, i), k))); }
EXPORT t_fe_neg(int n, const u64 *a, u64 *o) { EACH(st(o, i, swv::fe_neg(ld(a, i)))); }
EXPORT t_fe_invert(int n, const u64 *a, u64 *o) { EACH(st(o, i, swv::fe_invert(ld(a, i)))); }
EXPORT t_fe_pow22523(int n, const u64 *a, u64 *o) { EACH(st(o, i, swv::fe_pow22523(ld(a, i)))); }
EXPORT t_fe_frombytes(int n, const uint8_t *s, u64 *o) { EACH(st(o, i, swv::fe_frombytes(s + 32 * i))); }
EXPORT t_fe_tobytes(int n, const u64 *a, uint8_t *o) { EACH(swv::fe_tobytes(o + 32 * i, ld(a, i))); }
EXPORT t_fe_iszero(int n, const u64 *a, uint8_t *o) { EACH(o[i] = swv::fe_iszero(ld(a, i))); }
EXPORT t_fe_isneg(int n, const u64 *a, uint8_t *o) { EACH(o[i] = swv::fe_isneg(ld(a, i))); }

// ---- encodings
EXPORT t_y_canonical(int n, const uint8_t *s, uint8_t *o) { EACH(o[i] = swv::y_canonical(s + 32 * i)); }
// ok[i], and the encoding of the decoded point (negated when negate[i])
EXPORT t_ge_decode(int n, const uint8_t *s, const uint8_t *negate, uint8_t *ok, uint8_t *o) {
    EACH(ge p; ok[i] = swv::ge_decode(p, s + 32 * i, negate[i] != 0); if (ok[i]) swv::ge_encode(o + 32 * i, p));
}
// the key path of sw_set_member_keys: libsodium's verdict on the key, and [1..15](-A) as 15 encodings with, per
// entry, whether its 2dT agrees with X and Y
EXPORT t_point_table(int n, const uint8_t *s, uint8_t *ok, uint8_t *o, uint8_t *t_ok) {
    EACH(gc tab[swv::TAB]; ok[i] = swv::point_table(s + 32 * i, true, true, tab);
         if (ok[i]) for (int j = 0; j < swv::TAB; j++) t_ok[swv::TAB * i + j] = cached_encode(o + 32 * (swv::TAB * i + j), tab[j]));
}

// ---- scalars
EXPORT t_sc_canonical(int n, const uint8_t *s, uint8_t *o) { EACH(o[i] = swv::sc_canonical(s + 32 * i)); }
EXPORT t_sc_reduce512(int n, const uint8_t *h, uint8_t *o) { EACH(swv::sc_reduce512(o + 32 * i, h + 64 * i)); }

// ---- the double-scalar product: Q = [S]B + [k](-A) as double_scalar computes it (A decoded without the key checks),
// enc(Q), whether [8]Q = O, and signature_equation's verdict on (R, S)
EXPORT t_double_scalar(int n, const uint8_t *S, const uint8_t *k, const uint8_t *A, const uint8_t *R, uint8_t *a_ok,
                       uint8_t *q, uint8_t *small, uint8_t *verdict) {
    EACH(gc btab[swv::TAB]; gc atab[swv::TAB]; uint8_t b[32]; uint8_t sig[64];
         swv::base_encoding(b); swv::point_table(b, false, false, btab);
         a_ok[i] = swv::point_table(A + 32 * i, true, false, atab);
         if (a_ok[i]) {
             ge Q;
             swv::double_scalar(Q, S + 32 * i, k + 32 * i, btab, atab);
             swv::ge_encode(q + 32 * i, Q);
             small[i] = swv::ge_small_order(Q);
             for (int j = 0; j < 32; j++) { sig[j] = R[32 * i + j]; sig[32 + j] = S[32 * i + j]; }
             verdict[i] = swv::signature_equation(sig, k + 32 * i, btab, atab);
         });
}

// ---- crypto_sign_verify_detached of (sig, pk, buf[off[i] .. off[i] + len[i])), as the two kernels compute it
EXPORT t_verify(int n, const uint8_t *sig, const uint8_t *pk, const uint8_t *buf, const int64_t *off, const int64_t *len,
                uint8_t *o) {
    EACH(gc btab[swv::TAB]; gc atab[swv::TAB]; uint8_t b[32]; uint8_t k[32];
         const uint8_t *s = sig + 64 * i; const uint8_t *A = pk + 32 * i;
         swv::base_encoding(b); swv::point_table(b, false, false, btab);
         o[i] = swv::point_table(A, true, true, atab) && swv::sc_canonical(s + 32);
         if (o[i]) { swv::challenge(k, s, A, buf + off[i], len[i]); o[i] = swv::signature_equation(s, k, btab, atab); });
}

// ---- hashes of buf[off[i] .. off[i] + len[i])
EXPORT t_sha512(int n, const uint8_t *buf, const int64_t *off, const int64_t *len, uint8_t *o) {
    EACH(const uint8_t *p = buf + off[i]; swv::sha512(o + 64 * i, len[i], [&](int64_t j) -> uint8_t { return p[j]; }));
}
EXPORT t_blake2b_256(int n, const uint8_t *buf, const int64_t *off, const int64_t *len, uint8_t *o) {
    EACH(const uint8_t *p = buf + off[i]; swv::blake2b_256(o + 32 * i, len[i], [&](int64_t j) -> uint8_t { return p[j]; }));
}
'''


def nvcc() -> str | None:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


def compile_lib(out_dir, device: bool) -> str:
    """The harness as a shared library in out_dir: the host build, or (device=True) the sm_90a build."""
    from swirld_b200 import build
    out_dir = str(out_dir)
    src = os.path.join(out_dir, "harness.cu" if device else "harness.cpp")
    so = os.path.join(out_dir, "libharness_%s.so" % ("device" if device else "host"))
    with open(src, "w") as f:
        f.write(SOURCE)
    if device:
        cmd = [nvcc()] + build.NVCC_FLAGS + ["--extended-lambda"]
    else:
        cmd = [nvcc(), "-x", "c++", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-Wno-unknown-pragmas"]
    subprocess.check_call(cmd + ["-I", CSRC, "-o", so, src])
    return so


class Harness:
    """The entry points of SOURCE on numpy arrays, through the host build (device=False) or the device build."""

    def __init__(self, so: str, device: bool):
        self.lib = C.CDLL(so)
        self.device = device
        if device:
            import torch
            self.torch = torch

    def _call(self, name, n, ints, ins, outs):
        """ins: numpy arrays; outs: (shape, dtype) pairs; returns the outputs as numpy arrays."""
        fn = getattr(self.lib, "t_" + name)
        fn.restype = C.c_int
        if n == 0:
            return [np.zeros(s, d) for s, d in outs]
        if self.device:
            t = self.torch
            dins = [t.from_numpy(np.array(a, copy=True)).cuda() for a in ins]
            douts = [t.zeros(s, dtype=t.from_numpy(np.zeros(0, d)).dtype, device="cuda") for s, d in outs]
            ptrs = [C.c_void_p(x.data_ptr()) for x in dins + douts]
            rc = fn(C.c_int(n), *[C.c_int(k) for k in ints], *ptrs)
            assert rc == 0, "%s: CUDA error %d" % (name, rc)
            return [x.cpu().numpy() for x in douts]
        hins = [np.ascontiguousarray(a) for a in ins]
        houts = [np.zeros(s, d) for s, d in outs]
        ptrs = [C.c_void_p(a.ctypes.data) for a in hins + houts]
        rc = fn(C.c_int(n), *[C.c_int(k) for k in ints], *ptrs)
        assert rc == 0, name
        return houts

    # ---- field: limbs are (n, 5) uint64 arrays
    def fe_binary(self, op, a, b):
        return self._call(op, len(a), (), [a, b], [((len(a), 5), np.uint64)])[0]

    def fe_unary(self, op, a):
        return self._call(op, len(a), (), [a], [((len(a), 5), np.uint64)])[0]

    def fe_sqn(self, a, k):
        return self._call("fe_sqn", len(a), (k,), [a], [((len(a), 5), np.uint64)])[0]

    def fe_frombytes(self, s):
        return self._call("fe_frombytes", len(s), (), [s], [((len(s), 5), np.uint64)])[0]

    def fe_tobytes(self, a):
        return self._call("fe_tobytes", len(a), (), [a], [((len(a), 32), np.uint8)])[0]

    def fe_flag(self, op, a):
        return self._call(op, len(a), (), [a], [((len(a),), np.uint8)])[0]

    # ---- encodings and scalars: byte strings are (n, 32) or (n, 64) uint8 arrays
    def y_canonical(self, s):
        return self._call("y_canonical", len(s), (), [s], [((len(s),), np.uint8)])[0]

    def ge_decode(self, s, negate):
        n = len(s)
        return self._call("ge_decode", n, (), [s, negate], [((n,), np.uint8), ((n, 32), np.uint8)])

    def point_table(self, s):
        n = len(s)
        return self._call("point_table", n, (), [s], [((n,), np.uint8), ((n, 15, 32), np.uint8), ((n, 15), np.uint8)])

    def sc_canonical(self, s):
        return self._call("sc_canonical", len(s), (), [s], [((len(s),), np.uint8)])[0]

    def sc_reduce512(self, h):
        return self._call("sc_reduce512", len(h), (), [h], [((len(h), 32), np.uint8)])[0]

    def double_scalar(self, S, k, A, R):
        n = len(S)
        return self._call("double_scalar", n, (), [S, k, A, R],
                          [((n,), np.uint8), ((n, 32), np.uint8), ((n,), np.uint8), ((n,), np.uint8)])

    def verify(self, sig, pk, buf, off, ln):
        n = len(off)
        return self._call("verify", n, (), [sig, pk, buf, np.asarray(off, np.int64), np.asarray(ln, np.int64)],
                          [((n,), np.uint8)])[0]

    def hash(self, op, buf, off, ln):
        n, d = len(off), 64 if op == "sha512" else 32
        return self._call(op, n, (), [buf, np.asarray(off, np.int64), np.asarray(ln, np.int64)], [((n, d), np.uint8)])[0]


def packed(chunks):
    """(one buffer, offsets, lengths) of byte strings laid end to end (the buffer never empty)."""
    off = np.cumsum([0] + [len(c) for c in chunks[:-1]]).astype(np.int64) if chunks else np.zeros(0, np.int64)
    buf = np.frombuffer(b"".join(chunks) + b"\0", np.uint8)
    return buf, off, np.array([len(c) for c in chunks], np.int64)
