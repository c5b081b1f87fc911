// swirld_stream.cuh -- divide_rounds at the reference's own cadence: one sync per call, a handful of new
// events (Node.main, swirld.py:319-328).  The batch kernels (blocked can_see scan, round kernel, finish
// kernels: ~15 launches) are built for thousands of events per call; here ONE launch of ONE CTA does the
// whole of swirld.py:193-222 for the few new events, in arrival order, with the reference's own per-event
// structure (row merge, strongly-sees count against the witnesses of round r, promotion, witness
// registration) -- one thread per member column, the O(M^2) count as M coalesced row reads per event:
//
//   row(h)    = max(row(p0), row(p1)), own column := h                      swirld.py:203-205, 220
//   r         = max(round[p0], round[p1])                                    :200
//   hits[c_]  = stake of the members c whose latest seen event k (>= Wf_r[c]) sees Wf_r[c_]   :207-214
//   round[h]  = r + [ #{c_ : hits[c_] > 2T/3} > 2T/3 ]                      :216-219
//   witness, W / Wf tables, seen-mask SM(h), and for a witness decide_fame's strongly-seen set S (:245-254)
//
// It also keeps what the batch kernels need should a later call be a big one (per-member ring of recent events,
// event counts, can_see carry heads), so the two paths can be mixed freely on one engine.
#pragma once
#include "swirld_kernels.cuh"

struct StreamParams {
    int M, first, n, Rcap, NJ;
    const int32_t *p0, *p1, *creator, *seq;
    int32_t *row, *round;
    uint8_t *wit;
    int32_t *W, *Wf;
    u64 *SM, *S;                // M <= 64 path
    unsigned *SMw, *Sw;         // wide path
    uint8_t *coin;
    const uint8_t *sig;
    const i64 *stake;
    i64 tot2;
    int32_t *scal;
    int32_t *ctot, *gchain, *carry;
    int ring;
};

// sum over the CTA (all threads call it)
__device__ __forceinline__ i64 st_block_sum(i64 v, i64 *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    i64 s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[w];
    return s;
}

template <bool WIDE>
__device__ __forceinline__ void stream_divide(const StreamParams &P) {
    extern __shared__ int st_smem[];
    const int M = P.M, c = threadIdx.x, lane = c & 31;
    i64 *stake_s = reinterpret_cast<i64 *>(st_smem);       // [M]
    i64 *red = stake_s + M;                                // [32]
    int *pre = reinterpret_cast<int *>(red + 32);          // [M] merged row before the own column is set
    int *Wr = pre + M;                                     // [M] Wf_r, then W[round h]
    int *kk = Wr + M;                                      // [M] live member -> its latest seen event, else -1
    unsigned *words = reinterpret_cast<unsigned *>(kk + M);   // [32] ballot words
    const bool col = c < M;
    const i64 thr = P.tot2 / 3;
    if (col) stake_s[c] = P.stake[c];
    int max_round = P.scal[SC_MAX_ROUND];
    __syncthreads();
    for (int h = P.first; h < P.first + P.n; h++) {
        const int a = P.p0[h], b = P.p1[h], cr = P.creator[h], sq = P.seq[h];
        const bool root = a < 0;
        int v = -1;
        if (col && !root) v = max(P.row[(size_t)a * M + c], P.row[(size_t)b * M + c]);
        const int mine = c == cr ? h : v;
        if (col) { pre[c] = v; P.row[(size_t)h * M + c] = mine; }
        int rh = 0;
        bool witness = true;
        if (!root) {
            const int ra = P.round[a], r = max(ra, P.round[b]);
            const int wv = col ? P.Wf[(size_t)r * M + c] : -1;
            const bool live = col && wv >= 0 && v >= wv;
            if (col) { Wr[c] = wv; kk[c] = live ? v : -1; }
            const i64 lv = st_block_sum(live ? stake_s[c] : 0, red);       // (also: pre / Wr / kk are visible)
            bool promoted = false;
            if (lv > thr) {                                               // hits[c_] <= stake of the live members
                i64 hits = 0;
                if (col && wv >= 0) {
#pragma unroll 4
                    for (int m = 0; m < M; m++) {
                        const int k = kk[m];
                        if (k >= 0 && P.row[(size_t)k * M + c] >= wv) hits += stake_s[m];
                    }
                }
                promoted = (i64)__syncthreads_count(hits > thr) > thr;   // a COUNT of members against the STAKE threshold (quirk Q3)
            }
            rh = r + (promoted ? 1 : 0);
            witness = rh > ra;
            if (c == 0) {
                P.round[h] = rh; P.wit[h] = witness ? 1 : 0;
                if (witness) {
                    if (rh >= P.Rcap - 1) atomicMin(&P.scal[SC_ERR], -5);
                    else {
                        P.W[(size_t)rh * M + cr] = h;
                        for (int r2 = ra + 1; r2 <= rh; r2++) P.Wf[(size_t)r2 * M + cr] = h;
                    }
                }
            }
        } else if (c == 0) {
            P.round[h] = 0; P.wit[h] = 1;
            P.W[cr] = h; P.Wf[cr] = h;
        }
        if (rh >= P.Rcap - 1) { __syncthreads(); continue; }
        max_round = max(max_round, rh);
        __syncthreads();                                                  // the tables of round rh hold h now
        // ---- seen-mask SM(h) against the witnesses of its own round
        {
            const int w = col ? P.W[(size_t)rh * M + c] : -1;
            const unsigned bal = __ballot_sync(0xffffffffu, col && w >= 0 && mine >= w);
            if (lane == 0) words[c >> 5] = bal;
            if (col) kk[c] = mine;                                        // the FINAL row of h (own column = h)
            __syncthreads();
            if (WIDE) { if (c < P.NJ) P.SMw[(size_t)h * P.NJ + c] = c < (int)((M + 31) >> 5) ? words[c] : 0u; }
            else if (c == 0) P.SM[h] = (u64)words[0] | (M > 32 ? (u64)words[1] << 32 : 0ull);
        }
        // ---- a witness: coin bit, and decide_fame's strongly-seen set over the round before (quirk Q15)
        if (witness) {
            if (c == 0) P.coin[(size_t)rh * M + cr] = P.sig[(size_t)h * 64] >> 7;
            if (rh >= 1) {
                i64 hits = 0;
                if (col) {
                    for (int m = 0; m < M; m++) {
                        const int k = kk[m];
                        if (k < 0 || P.round[k] != rh - 1) continue;
                        const bool bit = WIDE ? (P.SMw[(size_t)k * P.NJ + (c >> 5)] >> (c & 31)) & 1 : (P.SM[k] >> c) & 1;
                        if (bit) hits += stake_s[m];
                    }
                }
                __syncthreads();
                const unsigned bal = __ballot_sync(0xffffffffu, col && hits > thr);
                if (lane == 0) words[c >> 5] = bal;
                __syncthreads();
                if (WIDE) { if (c < P.NJ) P.Sw[((size_t)rh * M + cr) * P.NJ + c] = c < (int)((M + 31) >> 5) ? words[c] : 0u; }
                else if (c == 0) P.S[(size_t)rh * M + cr] = (u64)words[0] | (M > 32 ? (u64)words[1] << 32 : 0ull);
            }
        }
        if (c == 0) {                                                     // what the batch kernels keep per member
            P.gchain[(size_t)cr * P.ring + (sq & (P.ring - 1))] = h;
            P.ctot[cr] = sq + 1;
            P.carry[cr] = h;
        }
        __syncthreads();                                                  // row / round / masks of h before the next event reads them
    }
    if (c == 0 && P.n > 0) P.scal[SC_MAX_ROUND] = max_round;
}

// One CTA per node-view: sw_batch_divide_rounds puts every view's call of a handful of events in one launch.  The
// views share M (so the thread count and the dynamic shared memory); stakes and coin periods are per view.
template <bool WIDE, class Src>
__global__ void __launch_bounds__(1024) k_stream_divide(Src s) { stream_divide<WIDE>(params(s)); }
SW_SRC_INSTANCES_OF(k_stream_divide, StreamParams, false) SW_SRC_INSTANCES_OF(k_stream_divide, StreamParams, true)

// the event columns of a small append arrive as ONE packed block: scatter it to the SoA columns
struct UnpackParams {
    int base, n;
    const uint8_t *stage;       // [p0 n][p1 n][creator n][seq n][height n] int32, [t n] f64, [sig n][64], [stale n]
    int32_t *p0, *p1, *creator, *seq, *height;
    double *t;
    uint8_t *sig, *stale;
};
__host__ __device__ inline size_t unpack_off_t(int n) { return (size_t)20 * n + ((8 - (20 * (size_t)n) % 8) % 8); }
__host__ __device__ inline size_t unpack_bytes(int n) { return unpack_off_t(n) + (size_t)8 * n + (size_t)64 * n + n; }
__device__ __forceinline__ void unpack(const UnpackParams &P) {
    const int n = P.n;
    const int32_t *ints = reinterpret_cast<const int32_t *>(P.stage);
    const double *tt = reinterpret_cast<const double *>(P.stage + unpack_off_t(n));
    const uint8_t *sg = reinterpret_cast<const uint8_t *>(tt + n), *stl = sg + (size_t)64 * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        P.p0[P.base + i] = ints[i]; P.p1[P.base + i] = ints[n + i]; P.creator[P.base + i] = ints[2 * n + i];
        P.seq[P.base + i] = ints[3 * n + i]; P.height[P.base + i] = ints[4 * n + i];
        P.t[P.base + i] = tt[i]; P.stale[P.base + i] = stl[i];
    }
    for (int i = threadIdx.x; i < 64 * n; i += blockDim.x) P.sig[(size_t)P.base * 64 + i] = sg[i];
}
// one CTA per node-view: sw_batch_append's views all point `stage` into one packed block
template <class Src> __global__ void k_unpack(Src s) { unpack(params(s)); }
SW_SRC_INSTANCES(k_unpack, UnpackParams)
