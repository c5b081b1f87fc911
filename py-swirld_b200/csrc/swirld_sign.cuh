// swirld_sign.cuh -- a node's own new event (swirld.py:82-95, 139-144) on the GPU: the Ed25519 signature libsodium's
// deterministic crypto_sign_detached makes (RFC 8032), byte for byte, and the event's BLAKE2b-256 id.
//
//   az = SHA-512(seed); a = az[0..32) clamped, prefix = az[32..64)
//   r = SHA-512(prefix || M) mod L, R = enc([r]B); k = SHA-512(R || A || M) mod L, S = (r + k a) mod L; sig = R || S
//
// Built on swv::'s field, group, encodings and hashes, whose behaviour this file does not change.  a, prefix, r, [r]B
// before its encoding, and S before it is written are secret, so everything that touches them is constant time: no
// branch, loop bound, shared or global address or shuffle source lane depends on them.
//   - [r]B is a fixed-base comb.  r is recoded into 64 signed radix-16 digits e_i in [-8, 8] with arithmetic carries,
//     and  [r]B = 16 * sum_k e_{2k+1} 256^k B  +  sum_k e_{2k} 256^k B,  each term read from row k of a table of
//     j 256^k B (32 rows x 8 entries, cached form).  A lookup reads all 8 entries of its row and keeps one by masks,
//     then negates by a masked swap; a zero digit keeps the identity and still adds it.
//   - Scalars mod L (the 512-bit nonce and challenge, and r + k a) go through a Barrett reduction with a fixed number
//     of word operations and two masked subtractions.  swv::sc_reduce512 is bit-serial and branches on its input, so
//     it stays with verification.
// With SWV_CT_TRACE (host builds only) every table row and entry read, every secret-adjacent loop's trip count and
// every shuffle offset is appended to sws::ct_trace(), so a test can check the access pattern does not depend on keys.
#pragma once
#include "swirld_verify.cuh"

#ifdef SWV_CT_TRACE
#include <vector>
namespace sws { inline std::vector<long long> &ct_trace() { static std::vector<long long> t; return t; } }
#define SWS_CT(kind, a, b) sws::ct_trace().push_back(((long long)(kind) << 40) | ((long long)(a) << 20) | (long long)(b))
#else
#define SWS_CT(kind, a, b) ((void)0)
#endif

namespace sws {

using swv::fe; using swv::ge; using swv::gc; using swv::u64; using swv::u128;
constexpr int ROWS = 32, COLS = 8;        // the comb table: ROWS x COLS entries, j 256^k B at [k * COLS + j - 1]
constexpr int SK_BYTES = 96;              // an expanded signing key on the device: a || prefix || A

// ---------------------------------------------------------------- masks
SWV_HD u64 mask_of(u64 bit) { return 0 - bit; }                       // 0 / 1 -> no bits / all bits
SWV_HD u64 eq_small(u64 a, u64 b) { return ((a ^ b) - 1) >> 63; }     // 1 when a == b (a, b < 2^63)
SWV_HD void fe_cmov(fe &f, const fe &g, u64 m) { for (int i = 0; i < 5; i++) f.v[i] ^= m & (f.v[i] ^ g.v[i]); }
SWV_HD void gc_cmov(gc &t, const gc &u, u64 m) { fe_cmov(t.YpX, u.YpX, m); fe_cmov(t.YmX, u.YmX, m); fe_cmov(t.Z, u.Z, m); fe_cmov(t.T2d, u.T2d, m); }
SWV_HD gc gc_identity() { return gc{swv::fe_small(1), swv::fe_small(1), swv::fe_small(1), swv::fe_small(0)}; }

// ---------------------------------------------------------------- the comb
// 64 signed digits of a (32 bytes, a[31] <= 127): a = sum e_i 16^i, e_i in [-8, 7] for i < 63, e_63 in [0, 8]
SWV_HDI void recode16(int8_t *e, const uint8_t *a) {
    for (int i = 0; i < 32; i++) { e[2 * i] = (int8_t)(a[i] & 15); e[2 * i + 1] = (int8_t)(a[i] >> 4); }
    int carry = 0;
    SWS_CT(2, 1, 63);
    for (int i = 0; i < 63; i++) {
        const int x = e[i] + carry;                      // in [0, 16]
        carry = (x + 8) >> 4;                            // 1 when x >= 8
        e[i] = (int8_t)(x - (carry << 4));
    }
    e[63] = (int8_t)(e[63] + carry);
}
// e (in [-8, 8]) times row k's point, from row[0..COLS) = [1..8] 256^k B: every entry read, one kept by masks
SWV_HDI gc select(const gc *row, int k, int e) {
    const u64 neg = (u64)((unsigned)e >> 31);            // 1 when e < 0
    const u64 ab = (u64)((e ^ -(int)neg) + (int)neg);    // |e|
    gc t = gc_identity();
    for (int j = 0; j < COLS; j++) {
        SWS_CT(1, k, j);
        gc_cmov(t, row[j], mask_of(eq_small(ab, (u64)(j + 1))));
    }
    const gc m{t.YmX, t.YpX, t.Z, swv::fe_neg(t.T2d)};   // -(x, y) = (-x, y)
    gc_cmov(t, m, mask_of(neg));
    return t;
}
// Rows [lane * 32/lanes, (lane + 1) * 32/lanes) of the comb: P = sum e_{2k+1} 256^k B, Q = sum e_{2k} 256^k B
SWV_HDI void comb_partial(ge &P, ge &Q, const int8_t *e, const gc *tab, int lane, int lanes) {
    P = Q = swv::ge_identity();
    const int per = ROWS / lanes;
    SWS_CT(2, 0, per);
    for (int q = 0; q < per; q++) {
        const int k = lane * per + q;
        P = swv::ge_add(P, select(tab + COLS * k, k, e[2 * k + 1]));
        Q = swv::ge_add(Q, select(tab + COLS * k, k, e[2 * k]));
    }
}
// 16 P + Q
SWV_HDI ge comb_finish(const ge &P, const ge &Q) {
    const ge h = swv::ge_dbl(swv::ge_dbl(swv::ge_dbl(swv::ge_dbl(P))));
    return swv::ge_add(h, swv::ge_cached(Q));
}
// [a]B for a 32-byte a with a[31] <= 127, in one thread
SWV_HDI ge base_mult(const uint8_t *a, const gc *tab) {
    int8_t e[64];
    recode16(e, a);
    ge P, Q;
    comb_partial(P, Q, e, tab, 0, 1);
    return comb_finish(P, Q);
}
// [1..8] base in cached form (row k of the table holds base = 256^k B)
SWV_HDI void comb_row(gc *row, const ge &base) {
    const gc c = swv::ge_cached(base);
    ge acc = base;
    row[0] = c;
    for (int j = 1; j < COLS; j++) { acc = swv::ge_add(acc, c); row[j] = swv::ge_cached(acc); }
}
// Row k of the table, from the base point's encoding and 8k doublings
SWV_HDI void table_row(gc *row, int k) {
    uint8_t b[32];
    swv::base_encoding(b);
    ge p;
    swv::ge_decode(p, b, false);
    for (int i = 0; i < 8 * k; i++) p = swv::ge_dbl(p);
    comb_row(row, p);
}

// ---------------------------------------------------------------- scalars mod L, constant time
SWV_HD void L5(u64 *l) { swv::L_words(l); l[4] = 0; }
// floor(2^512 / L), five little-endian words (checked against exact integers by the tests)
SWV_HD void mu_words(u64 *m) {
    m[0] = 0xed9ce5a30a2c131bull; m[1] = 0x2106215d086329a7ull; m[2] = 0xffffffffffffffebull; m[3] = 0xffffffffffffffffull;
    m[4] = 0xfull;
}
// d = a - b over n words; returns the borrow out
SWV_HD u64 sub_words(u64 *d, const u64 *a, const u64 *b, int n) {
    u64 borrow = 0;
    for (int i = 0; i < n; i++) {
        const u128 t = (u128)a[i] - b[i] - borrow;
        d[i] = (u64)t;
        borrow = (u64)(t >> 64) & 1;
    }
    return borrow;
}
// x (8 words, any value below 2^512) mod L into r (4 words).  Barrett (HAC 14.42, b = 2^64, k = 4):
// q3 = ((x >> 192) mu) >> 320 is at most 2 below x / L, so r1 - q3 L mod 2^320 is in [0, 3L): two masked subtractions.
SWV_HDI void sc_reduce_ct(u64 *r, const u64 *x) {
    u64 mu[5], l[5], q2[10] = {0}, r2[5] = {0}, t[5];
    mu_words(mu);
    L5(l);
    for (int i = 0; i < 5; i++) {                         // q2 = q1 mu, q1 = x[3..8)
        u64 c = 0;
        for (int j = 0; j < 5; j++) {
            const u128 p = (u128)x[3 + i] * mu[j] + q2[i + j] + c;
            q2[i + j] = (u64)p;
            c = (u64)(p >> 64);
        }
        q2[i + 5] = c;
    }
    const u64 *q3 = q2 + 5;
    for (int i = 0; i < 5; i++) {                         // r2 = q3 L mod 2^320
        u64 c = 0;
        for (int j = 0; i + j < 5; j++) {
            const u128 p = (u128)q3[i] * l[j] + r2[i + j] + c;
            r2[i + j] = (u64)p;
            c = (u64)(p >> 64);
        }
    }
    sub_words(t, x, r2, 5);                               // r1 - r2 mod 2^320
    SWS_CT(2, 2, 2);
    for (int s = 0; s < 2; s++) {
        u64 d[5];
        const u64 keep = mask_of(sub_words(d, t, l, 5)); // all bits when t < L
        for (int i = 0; i < 5; i++) t[i] = (t[i] & keep) | (d[i] & ~keep);
    }
    for (int i = 0; i < 4; i++) r[i] = t[i];
}
SWV_HD void words_to_bytes(uint8_t *s, const u64 *w, int n) { for (int i = 0; i < 8 * n; i++) s[i] = (uint8_t)(w[i >> 3] >> (8 * (i & 7))); }
SWV_HDI void reduce_bytes(u64 *r, const uint8_t *h) {    // 64 little-endian bytes mod L
    u64 x[8];
    for (int i = 0; i < 8; i++) x[i] = swv::ld64(h + 8 * i);
    sc_reduce_ct(r, x);
}
// (r + k a) mod L: k, r < L and a < 2^256 as 4 words each, so the sum stays below 2^510
SWV_HDI void sc_muladd(u64 *s, const u64 *k, const u64 *a, const u64 *r) {
    u64 x[8] = {0};
    for (int i = 0; i < 4; i++) {
        u64 c = 0;
        for (int j = 0; j < 4; j++) {
            const u128 p = (u128)k[i] * a[j] + x[i + j] + c;
            x[i + j] = (u64)p;
            c = (u64)(p >> 64);
        }
        x[i + 4] = c;
    }
    u64 c = 0;
    for (int i = 0; i < 8; i++) {
        const u128 p = (u128)x[i] + (i < 4 ? r[i] : 0) + c;
        x[i] = (u64)p;
        c = (u64)(p >> 64);
    }
    sc_reduce_ct(s, x);
}

// ---------------------------------------------------------------- keys and signatures
// libsodium's expansion of a 32-byte seed: a = SHA-512(seed)[0..32) clamped, prefix = SHA-512(seed)[32..64)
SWV_HDI void expand_key(uint8_t *a, uint8_t *prefix, const uint8_t *seed) {
    uint8_t az[64];
    swv::sha512(az, 32, [&](int64_t i) -> uint8_t { return seed[i]; });
    for (int i = 0; i < 32; i++) { a[i] = az[i]; prefix[i] = az[32 + i]; }
    a[0] &= 248;
    a[31] &= 127;
    a[31] |= 64;
}
// r = SHA-512(prefix || M) mod L
SWV_HDI void nonce(u64 *r, const uint8_t *prefix, const uint8_t *msg, int64_t len) {
    uint8_t h[64];
    swv::sha512(h, 32 + len, [&](int64_t i) -> uint8_t { return i < 32 ? prefix[i] : msg[i - 32]; });
    reduce_bytes(r, h);
}
// k = SHA-512(R || A || M) mod L
SWV_HDI void challenge(u64 *k, const uint8_t *R, const uint8_t *A, const uint8_t *msg, int64_t len) {
    uint8_t h[64];
    swv::sha512(h, 64 + len, [&](int64_t i) -> uint8_t { return i < 32 ? R[i] : i < 64 ? A[i - 32] : msg[i - 64]; });
    reduce_bytes(k, h);
}
// S = (r + k a) mod L as 32 bytes, k from R and the message
SWV_HDI void sign_scalar(uint8_t *S, const uint8_t *R, const uint8_t *a, const uint8_t *A, const u64 *r,
                         const uint8_t *msg, int64_t len) {
    u64 k[4], aw[4], s[4];
    challenge(k, R, A, msg, len);
    for (int i = 0; i < 4; i++) aw[i] = swv::ld64(a + 8 * i);
    sc_muladd(s, k, aw, r);
    words_to_bytes(S, s, 4);
}
// The whole signature in one thread: sig = R || S over msg[0..len) by the key sk = a || prefix || A
SWV_HDI void sign(uint8_t *sig, const uint8_t *sk, const uint8_t *msg, int64_t len, const gc *tab) {
    u64 r[4];
    uint8_t rb[32];
    nonce(r, sk + 32, msg, len);
    words_to_bytes(rb, r, 4);
    swv::ge_encode(sig, base_mult(rb, tab));
    sign_scalar(sig + 32, sig, sk, sk + 64, r, msg, len);
}

}  // namespace sws

#ifdef __CUDACC__
// ---------------------------------------------------------------- kernels
// The comb table: thread k writes row k, [1..8] 256^k B
__global__ void k_sign_table(swv::gc *__restrict__ tab) {
    if (threadIdx.x < sws::ROWS) sws::table_row(tab + sws::COLS * threadIdx.x, threadIdx.x);
}

// A signing key from libsodium's 64-byte secret key in[0..64) = seed || pk: ok[0] = 1 when [a]B encodes to pk, and then
// sk = a || prefix || pk; else nothing is written but ok[0] = 0.
__global__ void k_sign_key(const uint8_t *__restrict__ in, const swv::gc *__restrict__ tab, uint8_t *__restrict__ sk,
                           uint8_t *__restrict__ ok) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint8_t a[32], prefix[32], enc[32];
    sws::expand_key(a, prefix, in);
    swv::ge_encode(enc, sws::base_mult(a, tab));
    uint8_t x = 0;
    for (int i = 0; i < 32; i++) x |= enc[i] ^ in[32 + i];
    ok[0] = x == 0;
    if (x == 0)                                        // (the verdict is public: the caller learns it)
        for (int i = 0; i < 32; i++) { sk[i] = a[i]; sk[32 + i] = prefix[i]; sk[64 + i] = in[32 + i]; }
}

// u64 limbs of a point from lane (lane ^ o) of the group
__device__ __forceinline__ swv::ge shfl_ge(const swv::ge &p, int o, unsigned mask, int width) {
    swv::ge q;
    for (int j = 0; j < 5; j++) {
        q.X.v[j] = __shfl_xor_sync(mask, p.X.v[j], o, width);
        q.Y.v[j] = __shfl_xor_sync(mask, p.Y.v[j], o, width);
        q.Z.v[j] = __shfl_xor_sync(mask, p.Z.v[j], o, width);
        q.T.v[j] = __shfl_xor_sync(mask, p.T.v[j], o, width);
    }
    return q;
}

// Event i's signature and id, by a group of LANES lanes: every lane hashes, each takes ROWS / LANES rows of the comb,
// the partial sums meet by __shfl_xor_sync (fixed offsets), and lane 0 writes sig_out[i], copies it into the preimage
// at sig_at[i] and writes id_out[i] = BLAKE2b-256(preimage).  Event i is signed by the key keys[set[i]] (set null:
// keys[0]); a key is a || prefix || A on the device.
template <int LANES>
__global__ void __launch_bounds__(128) k_sign_events(int n, const int32_t *__restrict__ set, const uint8_t *const *__restrict__ keys,
                                                     const swv::gc *__restrict__ tab, const uint8_t *__restrict__ msg,
                                                     const int64_t *__restrict__ msg_off, uint8_t *__restrict__ pre,
                                                     const int64_t *__restrict__ pre_off, const int64_t *__restrict__ sig_at,
                                                     uint8_t *__restrict__ sig_out, uint8_t *__restrict__ id_out) {
    const int lane = threadIdx.x % LANES;
    const unsigned mask = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1) << ((threadIdx.x & 31) & ~(LANES - 1));
    const int stride = gridDim.x * blockDim.x / LANES;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) / LANES; i < n; i += stride) {
        const uint8_t *sk = keys[set ? set[i] : 0];
        const int64_t m0 = msg_off[i], len = msg_off[i + 1] - m0;
        const uint8_t *m = msg + m0;
        swv::u64 r[4];
        uint8_t rb[32], sig[64];
        sws::nonce(r, sk + 32, m, len);
        sws::words_to_bytes(rb, r, 4);
        int8_t e[64];
        sws::recode16(e, rb);
        swv::ge P, Q;
        sws::comb_partial(P, Q, e, tab, lane, LANES);
        for (int o = LANES / 2; o > 0; o >>= 1) {
            P = swv::ge_add(P, swv::ge_cached(shfl_ge(P, o, mask, LANES)));
            Q = swv::ge_add(Q, swv::ge_cached(shfl_ge(Q, o, mask, LANES)));
        }
        swv::ge_encode(sig, sws::comb_finish(P, Q));
        sws::sign_scalar(sig + 32, sig, sk, sk + 64, r, m, len);
        if (lane == 0) {
            uint8_t *s = sig_out + 64 * (size_t)i, *p = pre + pre_off[i];
            for (int j = 0; j < 64; j++) s[j] = p[sig_at[i] + j] = sig[j];
            swv::blake2b_256(id_out + 32 * (size_t)i, pre_off[i + 1] - pre_off[i], [&](int64_t j) -> uint8_t { return p[j]; });
        }
    }
}
#endif
