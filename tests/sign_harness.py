"""One C++ source over swirld_sign.cuh whose extern "C" entry points apply one sws:: function to arrays of n inputs, built
as verify_harness.py builds its source: `-x c++` for the host, or with the library's sm_90a flags, where each entry
point runs a grid-stride kernel (and `sign_events` launches the library's own k_sign_events) on device pointers.  A
third build, the host one with -DSWV_CT_TRACE, records the access pattern of a signature (`trace_sign`).

Points cross the boundary as their 32-byte encodings; scalars as 32 little-endian bytes."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from verify_harness import CSRC, nvcc

SOURCE = r'''
#include "swirld_sign.cuh"
#include <cstring>
#ifdef __CUDACC__
#include <cuda_runtime.h>
template <class F> __global__ void __launch_bounds__(128) k_each(int n, F f) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) f(i);
}
#endif
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

// the comb table, made once: by k_sign_table on the device build, by the same rows on the host
static gc *table() {
    static gc *tab = nullptr;
    if (tab) return tab;
#ifdef __CUDACC__
    cudaMalloc(&tab, sizeof(gc) * sws::ROWS * sws::COLS);
    k_sign_table<<<1, 32>>>(tab);
    cudaDeviceSynchronize();
#else
    static gc h[sws::ROWS * sws::COLS];
    for (int k = 0; k < sws::ROWS; k++) sws::table_row(h + sws::COLS * k, k);
    tab = h;
#endif
    return tab;
}
SWV_HDI void cached_encode(uint8_t *s, const gc &c) {     // (Y + X, Y - X, Z, 2dT) -> enc(X / Z, Y / Z)
    const fe X2 = swv::fe_sub(c.YpX, c.YmX), Y2 = swv::fe_add(c.YpX, c.YmX);
    const fe zi = swv::fe_invert(swv::fe_add(c.Z, c.Z));
    swv::fe_tobytes(s, swv::fe_mul(Y2, zi));
    s[31] ^= (uint8_t)(swv::fe_isneg(swv::fe_mul(X2, zi)) << 7);
}
// [a]B summed from the partials of `lanes` lanes (lanes = 1: base_mult's own path)
SWV_HDI ge lanes_mult(const uint8_t *a, const gc *tab, int lanes) {
    int8_t e[64];
    sws::recode16(e, a);
    ge P = swv::ge_identity(), Q = swv::ge_identity();
    for (int l = 0; l < lanes; l++) {
        ge p, q;
        sws::comb_partial(p, q, e, tab, l, lanes);
        P = swv::ge_add(P, swv::ge_cached(p));
        Q = swv::ge_add(Q, swv::ge_cached(q));
    }
    return sws::comb_finish(P, Q);
}

EXPORT t_expand(int n, const uint8_t *seed, uint8_t *a, uint8_t *prefix) { EACH(sws::expand_key(a + 32 * i, prefix + 32 * i, seed + 32 * i)); }
EXPORT t_recode(int n, const uint8_t *a, int8_t *e) { EACH(sws::recode16(e + 64 * i, a + 32 * i)); }
// every table entry's encoding, entry (k, j) at [k * 8 + j - 1]
EXPORT t_table(int n, uint8_t *o) { const gc *tab = table(); EACH(cached_encode(o + 32 * i, tab[i])); }
EXPORT t_base_mult(int n, const uint8_t *a, uint8_t *o) { const gc *tab = table(); EACH(swv::ge_encode(o + 32 * i, sws::base_mult(a + 32 * i, tab))); }
EXPORT t_lanes_mult(int n, int lanes, const uint8_t *a, uint8_t *o) {
    const gc *tab = table();
    EACH(swv::ge_encode(o + 32 * i, lanes_mult(a + 32 * i, tab, lanes)));
}
EXPORT t_reduce(int n, const uint8_t *h, uint8_t *o) { EACH(u64 r[4]; sws::reduce_bytes(r, h + 64 * i); sws::words_to_bytes(o + 32 * i, r, 4)); }
EXPORT t_muladd(int n, const uint8_t *k, const uint8_t *a, const uint8_t *r, uint8_t *o) {
    EACH(u64 kw[4]; u64 aw[4]; u64 rw[4]; u64 s[4];
         for (int j = 0; j < 4; j++) { kw[j] = swv::ld64(k + 32 * i + 8 * j); aw[j] = swv::ld64(a + 32 * i + 8 * j); rw[j] = swv::ld64(r + 32 * i + 8 * j); }
         sws::sc_muladd(s, kw, aw, rw); sws::words_to_bytes(o + 32 * i, s, 4));
}
// the signing key a || prefix || A of a seed, A = enc([a]B)
EXPORT t_signing_key(int n, const uint8_t *seed, uint8_t *sk) {
    const gc *tab = table();
    EACH(uint8_t *k = sk + sws::SK_BYTES * i; sws::expand_key(k, k + 32, seed + 32 * i); swv::ge_encode(k + 64, sws::base_mult(k, tab)));
}
// crypto_sign_detached of buf[off[i] .. off[i] + len[i]) by the signing key sk[i], in one thread
EXPORT t_sign(int n, const uint8_t *sk, const uint8_t *buf, const int64_t *off, const int64_t *len, uint8_t *sig) {
    const gc *tab = table();
    EACH(sws::sign(sig + 64 * i, sk + sws::SK_BYTES * i, buf + off[i], len[i], tab));
}
// k_sign_events<lanes> (device build) or its arithmetic (host build: the lanes' partials summed in order): event i is
// signed by sk[i]; pre is a copy, the signature lands in it at sig_at[i]
EXPORT t_sign_events(int n, int lanes, const uint8_t *sk, const uint8_t *msg, const int64_t *moff, const uint8_t *pre_in,
                     const int64_t *poff, const int64_t *sig_at, uint8_t *sig, uint8_t *ids) {
    const gc *tab = table();
#ifdef __CUDACC__
    const uint8_t **keys = nullptr;
    int32_t *set = nullptr;
    uint8_t *pre = nullptr;
    int64_t pn = 0;
    cudaMemcpy(&pn, poff + n, 8, cudaMemcpyDeviceToHost);
    cudaMalloc(&keys, sizeof(void *) * n); cudaMalloc(&set, 4 * n); cudaMalloc(&pre, pn + 1);
    cudaMemcpy(pre, pre_in, pn, cudaMemcpyDeviceToDevice);
    int rc = each(n, [=] __device__ (int i) { keys[i] = sk + sws::SK_BYTES * i; set[i] = i; });
    if (rc) return rc;
    const int groups = 128 / lanes, blocks = (n + groups - 1) / groups;
    if (lanes == 1) k_sign_events<1><<<blocks, 128>>>(n, set, keys, tab, msg, moff, pre, poff, sig_at, sig, ids);
    else if (lanes == 8) k_sign_events<8><<<blocks, 128>>>(n, set, keys, tab, msg, moff, pre, poff, sig_at, sig, ids);
    else return -1;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaFree(keys); cudaFree(set); cudaFree(pre);
    return (int)e;
#else
    std::vector<uint8_t> pre(pre_in, pre_in + poff[n]);
    for (int i = 0; i < n; i++) {
        const uint8_t *k = sk + sws::SK_BYTES * i, *m = msg + moff[i];
        const int64_t len = moff[i + 1] - moff[i];
        u64 r[4];
        uint8_t rb[32], *s = sig + 64 * i, *p = pre.data() + poff[i];
        sws::nonce(r, k + 32, m, len);
        sws::words_to_bytes(rb, r, 4);
        swv::ge_encode(s, lanes_mult(rb, tab, lanes));
        sws::sign_scalar(s + 32, s, k, k + 64, r, m, len);
        memcpy(p + sig_at[i], s, 64);
        swv::blake2b_256(ids + 32 * i, poff[i + 1] - poff[i], [&](int64_t j) -> uint8_t { return p[j]; });
    }
    return 0;
#endif
}
#ifdef SWV_CT_TRACE
// the trace of key expansion, [a]B and one signature of msg[0..len) by seed: its length, and its first `cap` entries
EXPORT t_trace_sign(const uint8_t *seed, const uint8_t *msg, int64_t len, long long *out, int cap) {
    sws::ct_trace().clear();
    uint8_t sk[sws::SK_BYTES], sig[64];
    sws::expand_key(sk, sk + 32, seed);
    swv::ge_encode(sk + 64, sws::base_mult(sk, table()));
    sws::sign(sig, sk, msg, len, table());
    const int m = (int)sws::ct_trace().size();
    for (int i = 0; i < m && i < cap; i++) out[i] = sws::ct_trace()[i];
    return m;
}
#endif
'''


def compile_lib(out_dir, device: bool, trace: bool = False) -> str:
    """The harness as a shared library in out_dir: the host build (with the access trace when `trace`), or the sm_90a
    build (device=True)."""
    from swirld_b200 import build
    out_dir = str(out_dir)
    tag = "device" if device else "trace" if trace else "host"
    src = os.path.join(out_dir, "sign_%s.%s" % (tag, "cu" if device else "cpp"))
    so = os.path.join(out_dir, "libsign_%s.so" % tag)
    with open(src, "w") as f:
        f.write(SOURCE if device else "#include <vector>\n" + SOURCE)
    if device:
        cmd = [nvcc()] + build.NVCC_FLAGS + ["--extended-lambda"]
    else:
        cmd = [nvcc(), "-x", "c++", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-Wno-unknown-pragmas"]
        if trace:
            cmd += ["-DSWV_CT_TRACE"]
    subprocess.check_call(cmd + ["-I", CSRC, "-o", so, src])
    return so


class SignHarness:
    """The entry points of SOURCE on numpy arrays, through the host build (device=False) or the device build."""

    def __init__(self, so: str, device: bool):
        self.lib = C.CDLL(so)
        self.device = device
        if device:
            import torch
            self.torch = torch

    def _call(self, name, n, ints, ins, outs):
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

    def expand(self, seeds):
        n = len(seeds)
        return self._call("expand", n, (), [seeds], [((n, 32), np.uint8), ((n, 32), np.uint8)])

    def recode(self, a):
        return self._call("recode", len(a), (), [a], [((len(a), 64), np.int8)])[0]

    def table(self):
        return self._call("table", 256, (), [], [((256, 32), np.uint8)])[0].reshape(32, 8, 32)

    def base_mult(self, a):
        return self._call("base_mult", len(a), (), [a], [((len(a), 32), np.uint8)])[0]

    def lanes_mult(self, a, lanes):
        return self._call("lanes_mult", len(a), (lanes,), [a], [((len(a), 32), np.uint8)])[0]

    def reduce(self, h):
        return self._call("reduce", len(h), (), [h], [((len(h), 32), np.uint8)])[0]

    def muladd(self, k, a, r):
        return self._call("muladd", len(k), (), [k, a, r], [((len(k), 32), np.uint8)])[0]

    def signing_key(self, seeds):
        return self._call("signing_key", len(seeds), (), [seeds], [((len(seeds), 96), np.uint8)])[0]

    def sign(self, sk, buf, off, ln):
        n = len(off)
        return self._call("sign", n, (), [sk, buf, np.asarray(off, np.int64), np.asarray(ln, np.int64)],
                          [((n, 64), np.uint8)])[0]

    def sign_events(self, lanes, sk, msgs, pres, sig_at):
        """(sig, ids) of events signed by sk[i] (n x 96), msgs[i] signed, pres[i] with the signature at sig_at[i]."""
        n = len(msgs)
        mb, mo = _packed(msgs)
        pb, po = _packed(pres)
        return self._call("sign_events", n, (lanes,), [sk, mb, mo, pb, po, np.asarray(sig_at, np.int64)],
                          [((n, 64), np.uint8), ((n, 32), np.uint8)])


def _packed(items):
    """(buffer, n+1 offsets) of byte strings laid end to end (the buffer never empty)."""
    off = np.zeros(len(items) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in items])
    return np.frombuffer(b"".join(items) + b"\0", np.uint8), off


def trace_sign(lib, seed: bytes, msg: bytes) -> np.ndarray:
    """The access trace (SWV_CT_TRACE build) of expanding `seed`, [a]B and signing `msg`."""
    fn = lib.t_trace_sign
    fn.restype = C.c_int
    cap = 1 << 16
    out = np.zeros(cap, np.int64)
    m = fn(C.c_char_p(seed), C.c_char_p(msg), C.c_int64(len(msg)), C.c_void_p(out.ctypes.data), C.c_int(cap))
    assert 0 < m <= cap
    return out[:m].copy()
