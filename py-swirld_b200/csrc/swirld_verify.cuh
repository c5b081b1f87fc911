// swirld_verify.cuh -- is_valid_event's crypto (swirld.py:97-103) on the GPU: Ed25519 signature verification with
// libsodium's verdicts (crypto_sign_verify_detached, >= 1.0.18 without ED25519_COMPAT) and BLAKE2b-256 event ids.
//
// Field GF(2^255 - 19) in radix 2^51 (five 64-bit limbs, 64 x 64 -> 128-bit products through unsigned __int128, which
// nvcc lowers to mul.lo / mul.hi on the device); points on -x^2 + y^2 = 1 + d x^2 y^2 in extended coordinates
// (X : Y : Z : T), x = X/Z, y = Y/Z, xy = T/Z.  Everything is public data, so nothing here is constant time: this is
// verification only.  The field, group and hash functions are __host__ __device__ and compute the same values on both
// sides (no intrinsics), so a host build of this header can check them against libsodium without a GPU; the library
// itself runs them on the device only.
//
// A signature (R, S) by key A over M is accepted exactly when
//   - S < L (canonical), and A's y is < p (canonical), A decodes to a curve point and [8]A != O (not of small order);
//   - with k = SHA-512(R || A || M) mod L, the point Q = [S]B - [k]A encodes to R byte for byte, and [8]Q != O.
// The last test is libsodium's refusal of an R whose y (sign bit ignored, aliases y + p included) is that of a
// small-order point: when R is the canonical encoding of Q, R names a point of small order exactly when Q is one, and
// any other R (non-canonical, off the curve) never equals an encoding, so it fails the byte comparison anyway.
// Small order is tested from the group itself -- three doublings reach the identity -- so no list of torsion encodings
// is written down.  The only literal curve constants are p (through 19 and the limb masks), d, sqrt(-1), L and the
// base point's encoding; the tables of multiples of B and of every member's -A are computed on the device.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif
#define SWV_HD __host__ __device__ __forceinline__
#define SWV_HDI __host__ __device__ inline

namespace swv {

typedef unsigned __int128 u128;
typedef uint64_t u64;
constexpr u64 M51 = (1ull << 51) - 1;
constexpr int TAB = 15;           // a table holds [1..15]P: scalars are read four bits at a time

// ---------------------------------------------------------------- GF(2^255 - 19)
struct fe { u64 v[5]; };

SWV_HD fe fe_words(u64 w0, u64 w1, u64 w2, u64 w3) {     // a 255-bit value given as 4 little-endian words
    fe h;
    h.v[0] = w0 & M51;
    h.v[1] = ((w0 >> 51) | (w1 << 13)) & M51;
    h.v[2] = ((w1 >> 38) | (w2 << 26)) & M51;
    h.v[3] = ((w2 >> 25) | (w3 << 39)) & M51;
    h.v[4] = (w3 >> 12) & M51;
    return h;
}
SWV_HD u64 ld64(const uint8_t *b) {
    u64 r = 0;
    for (int i = 7; i >= 0; i--) r = (r << 8) | b[i];
    return r;
}
// 32 bytes, bit 255 ignored; a value >= p is kept as it is (it is congruent to value - p)
SWV_HD fe fe_frombytes(const uint8_t *s) { return fe_words(ld64(s), ld64(s + 8), ld64(s + 16), ld64(s + 24)); }
SWV_HD fe fe_small(u64 x) { return fe{{x, 0, 0, 0, 0}}; }

SWV_HD fe fe_d() { return fe_words(0x75eb4dca135978a3ull, 0x00700a4d4141d8abull, 0x8cc740797779e898ull, 0x52036cee2b6ffe73ull); }
SWV_HD fe fe_sqrtm1() { return fe_words(0xc4ee1b274a0ea0b0ull, 0x2f431806ad2fe478ull, 0x2b4d00993dfbd7a7ull, 0x2b8324804fc1df0bull); }

SWV_HD void fe_carry(fe &h) {      // limbs back below 2^51 (limb 0: plus a little)
    u64 c;
    c = h.v[0] >> 51; h.v[0] &= M51; h.v[1] += c;
    c = h.v[1] >> 51; h.v[1] &= M51; h.v[2] += c;
    c = h.v[2] >> 51; h.v[2] &= M51; h.v[3] += c;
    c = h.v[3] >> 51; h.v[3] &= M51; h.v[4] += c;
    c = h.v[4] >> 51; h.v[4] &= M51; h.v[0] += 19 * c;
}
SWV_HD fe fe_add(const fe &a, const fe &b) {
    fe r;
    for (int i = 0; i < 5; i++) r.v[i] = a.v[i] + b.v[i];
    fe_carry(r);
    return r;
}
SWV_HD fe fe_sub(const fe &a, const fe &b) {     // a + 4p - b: no limb goes negative while b's limbs are < 2^53
    fe r;
    r.v[0] = a.v[0] + 0x1FFFFFFFFFFFB4ull - b.v[0];
    for (int i = 1; i < 5; i++) r.v[i] = a.v[i] + 0x1FFFFFFFFFFFFCull - b.v[i];
    fe_carry(r);
    return r;
}
SWV_HD fe fe_neg(const fe &a) { return fe_sub(fe_small(0), a); }
SWV_HDI fe fe_mul(const fe &a, const fe &b) {
    const u64 a0 = a.v[0], a1 = a.v[1], a2 = a.v[2], a3 = a.v[3], a4 = a.v[4];
    const u64 b0 = b.v[0], b1 = b.v[1], b2 = b.v[2], b3 = b.v[3], b4 = b.v[4];
    const u64 c1 = 19 * b1, c2 = 19 * b2, c3 = 19 * b3, c4 = 19 * b4;     // 2^255 = 19 (mod p)
    u128 t0 = (u128)a0 * b0 + (u128)a1 * c4 + (u128)a2 * c3 + (u128)a3 * c2 + (u128)a4 * c1;
    u128 t1 = (u128)a0 * b1 + (u128)a1 * b0 + (u128)a2 * c4 + (u128)a3 * c3 + (u128)a4 * c2;
    u128 t2 = (u128)a0 * b2 + (u128)a1 * b1 + (u128)a2 * b0 + (u128)a3 * c4 + (u128)a4 * c3;
    u128 t3 = (u128)a0 * b3 + (u128)a1 * b2 + (u128)a2 * b1 + (u128)a3 * b0 + (u128)a4 * c4;
    u128 t4 = (u128)a0 * b4 + (u128)a1 * b3 + (u128)a2 * b2 + (u128)a3 * b1 + (u128)a4 * b0;
    fe r;
    t1 += (u64)(t0 >> 51); r.v[0] = (u64)t0 & M51;
    t2 += (u64)(t1 >> 51); r.v[1] = (u64)t1 & M51;
    t3 += (u64)(t2 >> 51); r.v[2] = (u64)t2 & M51;
    t4 += (u64)(t3 >> 51); r.v[3] = (u64)t3 & M51;
    r.v[4] = (u64)t4 & M51;
    r.v[0] += 19 * (u64)(t4 >> 51);
    r.v[1] += r.v[0] >> 51; r.v[0] &= M51;
    return r;
}
SWV_HD fe fe_sq(const fe &a) { return fe_mul(a, a); }
SWV_HDI fe fe_sqn(fe a, int n) { for (int i = 0; i < n; i++) a = fe_sq(a); return a; }

// the canonical representative, as 32 little-endian bytes (bit 255 clear)
SWV_HDI void fe_tobytes(uint8_t *s, const fe &a) {
    fe h = a;
    fe_carry(h);
    fe_carry(h);                                            // h < 2^255, limbs < 2^51
    u64 q = (h.v[0] + 19) >> 51;                            // q = 1 exactly when h >= p
    q = (h.v[1] + q) >> 51; q = (h.v[2] + q) >> 51; q = (h.v[3] + q) >> 51; q = (h.v[4] + q) >> 51;
    h.v[0] += 19 * q;                                       // h + 19q - 2^255 q, the 2^255 dropped by the mask below
    u64 c;
    c = h.v[0] >> 51; h.v[0] &= M51; h.v[1] += c;
    c = h.v[1] >> 51; h.v[1] &= M51; h.v[2] += c;
    c = h.v[2] >> 51; h.v[2] &= M51; h.v[3] += c;
    c = h.v[3] >> 51; h.v[3] &= M51; h.v[4] += c;
    h.v[4] &= M51;
    const u64 w[4] = {h.v[0] | (h.v[1] << 51), (h.v[1] >> 13) | (h.v[2] << 38),
                      (h.v[2] >> 26) | (h.v[3] << 25), (h.v[3] >> 39) | (h.v[4] << 12)};
    for (int i = 0; i < 32; i++) s[i] = (uint8_t)(w[i >> 3] >> (8 * (i & 7)));
}
SWV_HDI bool fe_iszero(const fe &a) {
    uint8_t s[32];
    fe_tobytes(s, a);
    uint8_t x = 0;
    for (int i = 0; i < 32; i++) x |= s[i];
    return x == 0;
}
SWV_HDI bool fe_isneg(const fe &a) {      // the parity of the canonical value: the sign bit of an encoding
    uint8_t s[32];
    fe_tobytes(s, a);
    return s[0] & 1;
}
// z^(2^252 - 3) = z^((p - 5) / 8), and z^(p - 2) = 1/z, through z^(2^250 - 1)
SWV_HDI fe fe_pow250(const fe &z, fe &z11) {
    const fe z2 = fe_sq(z);
    const fe z9 = fe_mul(fe_sqn(z2, 2), z);
    z11 = fe_mul(z9, z2);
    const fe z5 = fe_mul(fe_sq(z11), z9);                   // 2^5 - 1
    const fe z10 = fe_mul(fe_sqn(z5, 5), z5);               // 2^10 - 1
    const fe z20 = fe_mul(fe_sqn(z10, 10), z10);
    const fe z40 = fe_mul(fe_sqn(z20, 20), z20);
    const fe z50 = fe_mul(fe_sqn(z40, 10), z10);
    const fe z100 = fe_mul(fe_sqn(z50, 50), z50);
    const fe z200 = fe_mul(fe_sqn(z100, 100), z100);
    return fe_mul(fe_sqn(z200, 50), z50);                   // 2^250 - 1
}
SWV_HDI fe fe_pow22523(const fe &z) { fe z11; return fe_mul(fe_sqn(fe_pow250(z, z11), 2), z); }
SWV_HDI fe fe_invert(const fe &z) { fe z11; return fe_mul(fe_sqn(fe_pow250(z, z11), 5), z11); }

// ---------------------------------------------------------------- the group
struct ge { fe X, Y, Z, T; };
struct gc { fe YpX, YmX, Z, T2d; };        // a point as the addend of ge_add wants it: (Y + X, Y - X, Z, 2dT)

SWV_HD ge ge_identity() { return ge{fe_small(0), fe_small(1), fe_small(1), fe_small(0)}; }
SWV_HD gc ge_cached(const ge &p) {
    const fe d = fe_d();
    return gc{fe_add(p.Y, p.X), fe_sub(p.Y, p.X), p.Z, fe_mul(p.T, fe_add(d, d))};
}
// p + q (Hisil-Wong-Carter-Dawson, a = -1; complete, so it also doubles and adds the identity)
SWV_HDI ge ge_add(const ge &p, const gc &q) {
    const fe A = fe_mul(fe_add(p.Y, p.X), q.YpX);
    const fe B = fe_mul(fe_sub(p.Y, p.X), q.YmX);
    const fe C = fe_mul(p.T, q.T2d);
    fe D = fe_mul(p.Z, q.Z);
    D = fe_add(D, D);
    const fe X3 = fe_sub(A, B), Y3 = fe_add(A, B), Z3 = fe_add(D, C), T3 = fe_sub(D, C);
    return ge{fe_mul(X3, T3), fe_mul(Y3, Z3), fe_mul(Z3, T3), fe_mul(X3, Y3)};
}
// 2p (T of the input is not read)
SWV_HDI ge ge_dbl(const ge &p) {
    const fe XX = fe_sq(p.X), YY = fe_sq(p.Y);
    fe B = fe_sq(p.Z);
    B = fe_add(B, B);
    const fe AA = fe_sq(fe_add(p.X, p.Y));
    const fe Y3 = fe_add(YY, XX), Z3 = fe_sub(YY, XX), X3 = fe_sub(AA, Y3), T3 = fe_sub(B, Z3);
    return ge{fe_mul(X3, T3), fe_mul(Y3, Z3), fe_mul(Z3, T3), fe_mul(X3, Y3)};
}
SWV_HDI bool ge_small_order(const ge &p) {     // [8]p is the identity
    const ge q = ge_dbl(ge_dbl(ge_dbl(p)));
    return fe_iszero(q.X) && fe_iszero(fe_sub(q.Y, q.Z));
}
SWV_HDI void ge_encode(uint8_t *s, const ge &p) {
    const fe zi = fe_invert(p.Z);
    fe_tobytes(s, fe_mul(p.Y, zi));
    s[31] ^= (uint8_t)(fe_isneg(fe_mul(p.X, zi)) << 7);
}
// y (bit 255 cleared) < p
SWV_HD bool y_canonical(const uint8_t *s) {
    if ((s[31] & 0x7f) != 0x7f || s[0] < 0xed) return true;
    for (int i = 1; i < 31; i++) if (s[i] != 0xff) return true;
    return false;
}
// The point with y = s (mod p) and x of the sign bit s[31] >> 7, negated when `negate`; false when x^2 has no root.
// x = 0 with the sign bit set decodes to x = 0 (as libsodium's decoder does; only y = +-1, of small order, get there).
SWV_HDI bool ge_decode(ge &p, const uint8_t *s, bool negate) {
    const fe y = fe_frombytes(s), one = fe_small(1);
    const fe yy = fe_sq(y);
    const fe u = fe_sub(yy, one), v = fe_add(fe_mul(yy, fe_d()), one);   // x^2 = u / v
    const fe v3 = fe_mul(fe_sq(v), v);
    fe x = fe_mul(fe_mul(fe_pow22523(fe_mul(fe_mul(fe_sq(v3), v), u)), v3), u);   // u v^3 (u v^7)^((p-5)/8)
    const fe vxx = fe_mul(fe_sq(x), v);
    if (!fe_iszero(fe_sub(vxx, u))) {
        if (!fe_iszero(fe_add(vxx, u))) return false;
        x = fe_mul(x, fe_sqrtm1());
    }
    if (fe_isneg(x) != (bool)((s[31] >> 7) ^ (negate ? 1 : 0))) x = fe_neg(x);
    p = ge{x, y, one, fe_mul(x, y)};
    return true;
}
// The base point's encoding: y = 4/5, x even
SWV_HD void base_encoding(uint8_t *s) {
    for (int i = 0; i < 32; i++) s[i] = 0x66;
    s[0] = 0x58;
}
// What libsodium says about a key alone, and [1..TAB](sign P) into tab, P the point of `enc` (the tab is written only
// when the key is accepted; a refused key's signatures all fail before any table is read)
SWV_HDI bool point_table(const uint8_t *enc, bool negate, bool check, gc *tab) {
    ge p;
    if (check && !y_canonical(enc)) return false;
    if (!ge_decode(p, enc, negate)) return false;
    if (check && ge_small_order(p)) return false;
    const gc c = ge_cached(p);
    ge acc = p;
    tab[0] = c;
    for (int j = 1; j < TAB; j++) { acc = ge_add(acc, c); tab[j] = ge_cached(acc); }
    return true;
}

// ---------------------------------------------------------------- scalars mod L = 2^252 + 27742317777372353535851937790883648493
SWV_HD void L_words(u64 *l) {
    l[0] = 0x5812631a5cf5d3edull; l[1] = 0x14def9dea2f79cd6ull; l[2] = 0; l[3] = 0x1000000000000000ull;
}
SWV_HD bool ge_words(const u64 *a, const u64 *b) {      // a >= b, 4 words
    for (int i = 3; i >= 0; i--) if (a[i] != b[i]) return a[i] > b[i];
    return true;
}
SWV_HD bool sc_canonical(const uint8_t *s) {            // S < L (all 256 bits)
    u64 w[4], l[4];
    for (int i = 0; i < 4; i++) w[i] = ld64(s + 8 * i);
    L_words(l);
    return !ge_words(w, l);
}
// a 512-bit little-endian value mod L, one bit at a time (variable time; a few thousand operations)
SWV_HDI void sc_reduce512(uint8_t *out, const uint8_t *h) {
    u64 r[4] = {0, 0, 0, 0}, l[4];
    L_words(l);
    for (int i = 511; i >= 0; i--) {
        r[3] = (r[3] << 1) | (r[2] >> 63); r[2] = (r[2] << 1) | (r[1] >> 63);
        r[1] = (r[1] << 1) | (r[0] >> 63); r[0] = (r[0] << 1) | ((h[i >> 3] >> (i & 7)) & 1);
        if (ge_words(r, l)) {
            u64 borrow = 0;
            for (int j = 0; j < 4; j++) {
                const u64 d = r[j] - l[j] - borrow;
                borrow = (r[j] < l[j] + borrow) || (l[j] + borrow < l[j]);
                r[j] = d;
            }
        }
    }
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(r[i >> 3] >> (8 * (i & 7)));
}

// ---------------------------------------------------------------- SHA-512 (FIPS 180-4)
#define SWV_SHA512_K                                                                                    \
    0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull,         \
    0x3956c25bf348b538ull, 0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull,         \
    0xd807aa98a3030242ull, 0x12835b0145706fbeull, 0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull,         \
    0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull, 0xc19bf174cf692694ull,         \
    0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,         \
    0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull,         \
    0x983e5152ee66dfabull, 0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull,         \
    0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull, 0x06ca6351e003826full, 0x142929670a0e6e70ull,         \
    0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull, 0x53380d139d95b3dfull,         \
    0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,         \
    0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull,         \
    0xd192e819d6ef5218ull, 0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull,         \
    0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull, 0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull,         \
    0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull, 0x682e6ff3d6b2b8a3ull,         \
    0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,         \
    0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull,         \
    0xca273eceea26619cull, 0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull,         \
    0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull, 0x113f9804bef90daeull, 0x1b710b35131c471bull,         \
    0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull, 0x431d67c49c100d4cull,         \
    0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull
#ifdef __CUDACC__
__constant__ u64 c_sha512_k[80] = {SWV_SHA512_K};     // every thread reads the same round's constant
#endif
static const u64 h_sha512_k[80] = {SWV_SHA512_K};
SWV_HD u64 sha512_k(int t) {
#ifdef __CUDA_ARCH__
    return c_sha512_k[t];
#else
    return h_sha512_k[t];
#endif
}
// SHA-512 and BLAKE2b start from the same eight words
SWV_HD u64 iv(int i) {
    const u64 v[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                      0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    return v[i];
}
SWV_HD u64 rotr(u64 x, int n) { return (x >> n) | (x << (64 - n)); }

SWV_HDI void sha512_block(u64 *h, u64 *w) {
    u64 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
    for (int t0 = 0; t0 < 80; t0 += 16) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            if (t0) {                                         // w[j] becomes W[t0 + j]
                const u64 w15 = w[(j + 1) & 15], w2 = w[(j + 14) & 15];
                w[j] += (rotr(w15, 1) ^ rotr(w15, 8) ^ (w15 >> 7)) + w[(j + 9) & 15] +
                        (rotr(w2, 19) ^ rotr(w2, 61) ^ (w2 >> 6));
            }
            const u64 t1 = k + (rotr(e, 14) ^ rotr(e, 18) ^ rotr(e, 41)) + ((e & f) ^ (~e & g)) + sha512_k(t0 + j) + w[j];
            const u64 t2 = (rotr(a, 28) ^ rotr(a, 34) ^ rotr(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
            k = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += k;
}
// SHA-512 of the `len` bytes byte(0) .. byte(len - 1)
template <class Byte>
SWV_HDI void sha512(uint8_t *out, int64_t len, const Byte &byte) {
    u64 h[8], w[16];
    for (int i = 0; i < 8; i++) h[i] = iv(i);
    const int64_t nb = (len + 17 + 127) / 128;                // the 0x80 byte and the 128-bit length fit in the last block
    for (int64_t b = 0; b < nb; b++) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            u64 x = 0;
            for (int q = 0; q < 8; q++) {
                const int64_t i = b * 128 + 8 * j + q;
                const uint8_t v = i < len ? byte(i) : i == len ? 0x80 : 0;
                x = (x << 8) | v;
            }
            w[j] = x;
        }
        if (b == nb - 1) w[15] = (u64)len << 3, w[14] = (u64)len >> 61;
        sha512_block(h, w);
    }
    for (int i = 0; i < 64; i++) out[i] = (uint8_t)(h[i >> 3] >> (56 - 8 * (i & 7)));
}

// ---------------------------------------------------------------- BLAKE2b-256, unkeyed (RFC 7693)
SWV_HD void b2_g(u64 *v, int a, int b, int c, int d, u64 x, u64 y) {
    v[a] = v[a] + v[b] + x; v[d] = rotr(v[d] ^ v[a], 32);
    v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 24);
    v[a] = v[a] + v[b] + y; v[d] = rotr(v[d] ^ v[a], 16);
    v[c] = v[c] + v[d];     v[b] = rotr(v[b] ^ v[c], 63);
}
SWV_HDI void b2_compress(u64 *h, const u64 *m, u64 t, bool last) {
    // the message schedule: row r lists its 16 word indices, one per nibble, lowest first
    const u64 sigma[10] = {0xfedcba9876543210ull, 0x357b20c16df984aeull, 0x491763eadf250c8bull, 0x8f04a562ebcd1397ull,
                           0xd386cb1efa427509ull, 0x91ef57d438b0a6c2ull, 0xb8293670a4def15cull, 0xa2684f05931ce7bdull,
                           0x5a417d2c803b9ef6ull, 0x0dc3e9bf5167482aull};
    u64 v[16];
    for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = iv(i); }
    v[12] ^= t;
    if (last) v[14] = ~v[14];
#pragma unroll
    for (int r = 0; r < 12; r++) {
        const u64 s = sigma[r % 10];
#define SWV_M(j) m[(s >> (4 * (j))) & 15]
        b2_g(v, 0, 4, 8, 12, SWV_M(0), SWV_M(1));
        b2_g(v, 1, 5, 9, 13, SWV_M(2), SWV_M(3));
        b2_g(v, 2, 6, 10, 14, SWV_M(4), SWV_M(5));
        b2_g(v, 3, 7, 11, 15, SWV_M(6), SWV_M(7));
        b2_g(v, 0, 5, 10, 15, SWV_M(8), SWV_M(9));
        b2_g(v, 1, 6, 11, 12, SWV_M(10), SWV_M(11));
        b2_g(v, 2, 7, 8, 13, SWV_M(12), SWV_M(13));
        b2_g(v, 3, 4, 9, 14, SWV_M(14), SWV_M(15));
#undef SWV_M
    }
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}
// BLAKE2b with a 32-byte digest of byte(0) .. byte(len - 1): the last block (the only one, zero-filled, when len is 0;
// a full one when len is a multiple of 128) is compressed with the final flag and the byte count len
template <class Byte>
SWV_HDI void blake2b_256(uint8_t *out, int64_t len, const Byte &byte) {
    u64 h[8], m[16];
    for (int i = 0; i < 8; i++) h[i] = iv(i);
    h[0] ^= 0x01010000ull | 32;                               // digest length 32, no key, fanout 1, depth 1
    const int64_t nb = len > 0 ? (len + 127) / 128 : 1;
    for (int64_t b = 0; b < nb; b++) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            u64 x = 0;
            for (int q = 7; q >= 0; q--) {
                const int64_t i = b * 128 + 8 * j + q;
                x = (x << 8) | (i < len ? byte(i) : 0);
            }
            m[j] = x;
        }
        const bool last = b == nb - 1;
        b2_compress(h, m, last ? (u64)len : (u64)(b + 1) * 128, last);
    }
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(h[i >> 3] >> (8 * (i & 7)));
}

// ---------------------------------------------------------------- one event
// k = SHA-512(R || A || M) mod L
SWV_HDI void challenge(uint8_t *k, const uint8_t *R, const uint8_t *A, const uint8_t *msg, int64_t len) {
    uint8_t h[64];
    sha512(h, 64 + len, [&](int64_t i) -> uint8_t { return i < 32 ? R[i] : i < 64 ? A[i - 32] : msg[i - 64]; });
    sc_reduce512(k, h);
}
SWV_HD int nibble(const uint8_t *s, int w) { return (s[w >> 1] >> (4 * (w & 1))) & 15; }
// [S]B + [k](-A), Btab = [1..15]B, Atab = [1..15](-A).  Four bits of both scalars per step: four doublings, then at
// most one addition from each table.
SWV_HD void double_scalar(ge &acc, const uint8_t *S, const uint8_t *k, const gc *Btab, const gc *Atab) {
    acc = ge_identity();
    bool started = false;
    for (int w = 63; w >= 0; w--) {
        if (started) { acc = ge_dbl(acc); acc = ge_dbl(acc); acc = ge_dbl(acc); acc = ge_dbl(acc); }
        const int s = nibble(S, w), a = nibble(k, w);
        if (s) { acc = ge_add(acc, Btab[s - 1]); started = true; }
        if (a) { acc = ge_add(acc, Atab[a - 1]); started = true; }
    }
}
// Does [S]B + [k](-A) encode to R, and is it not of small order?  S < L is checked by the caller.
SWV_HDI bool signature_equation(const uint8_t *sig, const uint8_t *k, const gc *Btab, const gc *Atab) {
    ge acc;
    double_scalar(acc, sig + 32, k, Btab, Atab);
    uint8_t enc[32];
    ge_encode(enc, acc);
    for (int i = 0; i < 32; i++) if (enc[i] != sig[i]) return false;
    return !ge_small_order(acc);
}

}  // namespace swv

#ifdef __CUDACC__
// ---------------------------------------------------------------- kernels
// [1..15]P of `count` points: the members' keys negated, with libsodium's verdict on each key alone (keys != null),
// or the base point (keys == null, count 1)
__global__ void k_verify_tables(int count, const uint8_t *__restrict__ keys, uint8_t *__restrict__ key_ok,
                                swv::gc *__restrict__ tab) {
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < count; m += gridDim.x * blockDim.x) {
        if (keys) {
            key_ok[m] = swv::point_table(keys + 32 * (size_t)m, true, true, tab + (size_t)swv::TAB * m);
        } else {
            uint8_t b[32];
            swv::base_encoding(b);
            swv::point_table(b, false, false, tab);
        }
    }
}

// Where an event's key set comes from: one set for every event of the launch (by value: the single-view calls), or a
// device array of the node-views' sets, event i's being Kv[set[i]] (sw_batch_ingest_verified).  A set is the members'
// keys (32 bytes each), libsodium's verdict on each key alone and [1..15](-A) per member.
struct KeySet { const uint8_t *keys; const uint8_t *key_ok; const swv::gc *Atab; };
__device__ __forceinline__ const KeySet &key_set(const KeySet &K, const int32_t *, int) { return K; }
__device__ __forceinline__ const KeySet &key_set(const KeySet *Kv, const int32_t *set, int i) { return Kv[set[i]]; }

// The byte-serial half: k = SHA-512(R || A || M) mod L into k_out, and bit 1 of flags (the id is BLAKE2b-256 of the
// preimage); bit 0 is cleared here and set by k_verify_curve.
template <class Keys>
__global__ void __launch_bounds__(256) k_verify_hash(int n, const int32_t *__restrict__ creator, const int32_t *__restrict__ set,
                                                     Keys K, const uint8_t *__restrict__ sig, const uint8_t *__restrict__ msg,
                                                     const int64_t *__restrict__ msg_off, const uint8_t *__restrict__ pre,
                                                     const int64_t *__restrict__ pre_off, const uint8_t *__restrict__ ids,
                                                     uint8_t *__restrict__ k_out, uint8_t *__restrict__ flags) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int64_t m0 = msg_off[i], p0 = pre_off[i];
        const uint8_t *A = key_set(K, set, i).keys + 32 * (size_t)creator[i];
        swv::challenge(k_out + 32 * (size_t)i, sig + 64 * (size_t)i, A, msg + m0, msg_off[i + 1] - m0);
        uint8_t dg[32];
        const uint8_t *p = pre + p0;
        swv::blake2b_256(dg, pre_off[i + 1] - p0, [&](int64_t j) -> uint8_t { return p[j]; });
        const uint8_t *id = ids + 32 * (size_t)i;
        uint8_t x = 0;
        for (int j = 0; j < 32; j++) x |= dg[j] ^ id[j];
        flags[i] = x == 0 ? 2 : 0;
    }
}

// The curve half: bit 0 of flags for events whose key and S libsodium accepts and whose equation holds.
template <class Keys>
__global__ void __launch_bounds__(128) k_verify_curve(int n, const int32_t *__restrict__ creator, const int32_t *__restrict__ set,
                                                      Keys K, const uint8_t *__restrict__ sig, const swv::gc *__restrict__ Btab,
                                                      const uint8_t *__restrict__ k, uint8_t *__restrict__ flags) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = creator[i];
        const KeySet &ks = key_set(K, set, i);
        const uint8_t *s = sig + 64 * (size_t)i;
        if (ks.key_ok[c] && swv::sc_canonical(s + 32) &&
            swv::signature_equation(s, k + 32 * (size_t)i, Btab, ks.Atab + (size_t)swv::TAB * c))
            flags[i] |= 1;
    }
}
#endif
